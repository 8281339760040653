"""The masked GAT restatement (tests/gat_dropout_ref.py) against the reference's own Graph_AE run in train() mode with the same
dropout masks (tests/golden/graph_ae_gat_dropout.npz, from tests/make_golden_gat_dropout.py).  No GPU needed."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import rel_err
from gat_dropout_ref import fixture_masks, graph_ae_gat_forward, scaled_mask


def _graph(golden):
    g = golden("knn_graph")
    n, k = g["knn_idx"].shape
    edge_index = torch.from_numpy(np.stack([np.repeat(np.arange(n), k), g["knn_idx"].reshape(-1)]).astype(np.int64))
    adj = sp.csr_matrix((np.ones(len(g["adj_indices"])), g["adj_indices"], g["adj_indptr"]), shape=(n, n))
    labels = torch.from_numpy((adj + sp.eye(n)).toarray()).float()
    return torch.from_numpy(g["X"]), edge_index, labels


@pytest.mark.parametrize("tag", ["proj", "ident"])
def test_masked_port_matches_reference_train_step(golden, tag):
    """Forward, loss, every gradient and the weights after one Adam step, with the fixture's masks at all three sites."""
    X, edge_index, labels = _graph(golden)
    gg = golden("graph_ae_gat_dropout")
    sd = {k[len(tag) + 6:]: torch.from_numpy(gg[k]).requires_grad_() for k in gg.files if k.startswith(f"{tag}.init.")}
    masks = fixture_masks(gg, tag, torch.float32)
    z = graph_ae_gat_forward(X, edge_index, sd, masks)
    assert rel_err(z.detach().numpy(), gg[f"{tag}.z"]) < 1e-6
    loss = torch.nn.functional.binary_cross_entropy_with_logits(z @ z.t(), labels)
    assert abs(loss.item() - float(gg[f"{tag}.loss"])) < 1e-6 * float(gg[f"{tag}.loss"])
    opt = torch.optim.Adam(sd.values(), lr=1e-2)
    opt.zero_grad()
    loss.backward()
    for k, v in sd.items():
        if f"{tag}.grad.{k}" in gg.files:
            assert rel_err(v.grad.numpy(), gg[f"{tag}.grad.{k}"]) < 1e-5, k
        else:   # identity skip: skip_proj is never read
            assert tag == "ident" and k.endswith("skip_proj.weight") and v.grad is None, k
    opt.step()
    for k, v in sd.items():
        assert rel_err(v.detach().numpy(), gg[f"{tag}.after.{k}"]) < 1e-6, k
    if tag == "ident":
        for l in range(2):
            k = f"gat.gat_net.{l}.skip_proj.weight"
            assert np.array_equal(gg[f"{tag}.after.{k}"], gg[f"{tag}.init.{k}"])


def test_masks_follow_the_drop_probability(golden):
    gg = golden("graph_ae_gat_dropout")
    keep = np.concatenate([gg[k].reshape(-1) for k in gg.files if ".mask." in k])
    p = float(gg["proj.p"])
    assert abs(keep.mean() - (1 - p)) < 6 * np.sqrt(p * (1 - p) / keep.size)
    m = scaled_mask(torch.tensor([True, False]), p)
    assert m.tolist() == [1 / (1 - p), 0.0] and scaled_mask(torch.tensor([True]), 1.0).tolist() == [0.0]


def test_unit_masks_equal_the_plain_restatement(golden):
    """All-ones masks (p = 0) give oracle.port's dropout-free restatement bit for bit, forward and gradients."""
    from oracle import port
    X, edge_index, labels = _graph(golden)
    gg = golden("graph_ae_gat")
    outs = []
    for masks in (None, "ones"):
        sd = {k[len("init."):]: torch.from_numpy(gg[k]).double().requires_grad_() for k in gg.files if k.startswith("init.")}
        x = X.double()
        if masks is None:
            z = port.graph_ae_gat_forward(x, edge_index, sd)
        else:
            m = []
            h_in = [x.shape[1], sd["gat.gat_net.1.linear_proj.weight"].shape[1]]
            for l in range(2):
                W = sd[f"gat.gat_net.{l}.linear_proj.weight"].shape[0]
                m.append({"input": torch.ones(x.shape[0], h_in[l], dtype=torch.float64),
                          "proj": torch.ones(x.shape[0], W, dtype=torch.float64),
                          "attn": torch.ones(edge_index.shape[1], 2, dtype=torch.float64)})
            z = graph_ae_gat_forward(x, edge_index, sd, m)
        torch.nn.functional.binary_cross_entropy_with_logits(z @ z.t(), labels.double()).backward()
        outs.append((z.detach(), {k: v.grad for k, v in sd.items()}))
    assert torch.equal(outs[0][0], outs[1][0])
    for k in outs[0][1]:
        assert torch.equal(outs[0][1][k], outs[1][1][k]), k
