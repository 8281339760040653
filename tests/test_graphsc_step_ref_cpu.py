"""The float64 restatement of graph-sc's training (tests/graphsc_ref.py) against the reference's own ``GraphSC.fit`` on the dgl
surface of tests/graphsc_ref.py, with the device's dropout masks injected into both, at ≤ 1e-10.

Cases: agg sum / mean, n_layers 1 / 2, n_hidden 0 / 1 (and 2), hidden_bn, dropout 0 / 0.1, edges renormalised or not, and
batch sizes that leave a short last batch, one of them a single cell.  Needs the reference sources."""
import numpy as np
import pytest
import torch

import graphsc_ref as R
from oracle import ref_loader

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="needs the reference sources")

BASE = dict(agg="sum", activation="relu", in_feats=8, n_hidden=1, hidden_dim=12, hidden_1=10, hidden_2=0, dropout=0.1, n_layers=1,
            hidden_relu=False, hidden_bn=False)
CASES = {
    "default": (BASE, True, 16),
    "mean": (dict(BASE, agg="mean"), True, 16),
    "no_hidden": (dict(BASE, n_hidden=0, dropout=0.0), False, 16),
    "two_layers": (dict(BASE, n_layers=2, activation="leaky_relu"), True, 12),
    "bn_relu": (dict(BASE, n_hidden=2, hidden_2=6, hidden_bn=True, hidden_relu=True, activation="gelu"), False, 13),
    "single_last": (dict(BASE, n_layers=2, agg="mean"), True, 20),                   # 41 cells: batches 20, 20, 1
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_restatement_matches_reference_fit(case):
    cfg, normalize, bs = CASES[case]
    ref = ref_loader.graphsc()
    gd = R.synthetic_graph(41, 30, 8, seed=0, normalize_edges=normalize)
    out = R.run_reference_fit(ref, cfg, gd, R.init_state(cfg, 1), fit_seed=2, epochs=2, lr=1e-2, batch_size=bs, drop_seed=7)
    assert all(sum(len(b) for b in out["batches"][e * -(-41 // bs):(e + 1) * -(-41 // bs)]) == 41 for e in range(2))
    graph = R.csr_by_destination(gd)
    losses, z, sd = R.fit(out["init"], dict(cfg, stride=1 + cfg["hidden_bn"] + cfg["hidden_relu"]), graph, out["batches"], None,
                          1e-2, R.device_masks(7, cfg["dropout"]))
    assert np.abs(losses - out["losses"]).max() <= 1e-10
    assert np.abs(z.numpy() - out["z"]).max() <= 1e-10
    for k, v in out["final"].items():
        # a bias in front of a BatchNorm has an exact gradient of 0: Adam steps it by rounding noise, which differs with the order
        # of the sums; it moves no output, only the running mean that tracks it
        noisy = cfg["hidden_bn"] and k.startswith("encoder.") and (k.endswith(".bias") and f"encoder.{int(k.split('.')[1]) + 1}.running_mean" in out["final"] or
                                      k.endswith("running_mean"))
        assert (sd[k].double() - v.double()).abs().max().item() <= (1e-6 if noisy else 1e-10), k


def test_short_last_batches_are_kept():
    torch.manual_seed(0)
    g = R.dgl_lite.Graph(torch.arange(5), torch.arange(5), 5)
    loader = R.DataLoader(g, torch.arange(5), R.MultiLayerFullNeighborSampler(1), batch_size=2, shuffle=True, drop_last=False,
                          num_workers=1)
    assert [len(seeds) for _, seeds, _ in loader] == [2, 2, 1]
