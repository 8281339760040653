"""dance_b200 — H100-native (sm_90a) implementation of the GNN message-passing hot path of
OmicsML/dance: hand-written CUDA kernels behind a C-ABI (include/dance_b200.h), driven by
thin Python classes that keep the reference's operator / model API."""
__version__ = "0.1.0"
