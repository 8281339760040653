from dance_b200.modules.graphsc import *  # noqa: F401,F403
from dance_b200.modules.graphsc import GraphSC  # noqa: F401
