"""The float64 GraphSCI step restatement (oracle/graphsci_step_ref.py) without a GPU: against the fixture the reference's own code
recorded (dropout 0), against the reference's GNNModel / AEModel / get_loss / evaluate run in float64 with dropout 0.1 and
recorded keep-masks (when the reference tree is present), and a check that a wrong mask site or stale BatchNorm statistics
would move its result far beyond the tolerance that pins it."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import graphsci_step_ref as R
from oracle import ref_loader

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="reference sources not present")

TOL = 1e-4          # tests/test_gpu_graphsci.py: the fixture was recorded in float32
PIN = 1e-10         # restatement against the reference's own code, both in float64
COEF = dict(le=1.3, la=0.7, ke=2.0, ka=0.9)


def _fixture_inputs(g):
    """What GraphSCI.fit hands to its first train() call on the fixture (graphsci.py:240-277)."""
    X, Xl, mask = g["X"], g["Xl"], g["mask"]
    n, G = X.shape
    test_idx = np.setdiff1d(np.arange(n), g["train_idx"])
    train_mask, valid_mask = mask.copy(), ~mask
    train_mask[test_idx] = False
    valid_mask[test_idx] = False
    Xraw = torch.from_numpy(X).double()
    counts = Xraw.sum(1)
    sf = counts / torch.median(counts)
    params = {f"{s}.{k[len(f'init.{s}.'):]}": torch.from_numpy(g[k]) for s in ("aemodel", "gnnmodel") for k in g.files
              if k.startswith(f"init.{s}.")}
    running = {k: (torch.from_numpy(g[f"init.aemodel.{k}.running_mean"]), torch.from_numpy(g[f"init.aemodel.{k}.running_var"]))
               for k in R.BN_KEYS}
    return dict(params=params, running=running, X=torch.from_numpy(Xl * mask).double(), Xraw=Xraw, sf=sf,
                graph=R.GeneGraph(g["src"], g["dst"], G, "cpu"), train_mask=torch.from_numpy(train_mask),
                valid_mask=torch.from_numpy(valid_mask))


def _masks(g, p=0.1, seed=0):
    """Keep-masks scaled by 1/(1 − p) for every dropout site, at the fixture's shapes."""
    n, G = g["X"].shape
    shapes = {"feat": (G, n), "h1": (G, R.H1), "h2_mean": (G, R.H2), "h2_log_std": (G, R.H2), "X": (n, G), "enc.1": (n, G),
              "enc.5": (n, R.H1)}
    shapes.update({h: (n, R.H2) for h in R.HEADS})
    gen = torch.Generator().manual_seed(seed)
    return {s: (torch.rand(shapes[s], generator=gen, dtype=torch.float64) >= p).double() / (1 - p) for s in R.SITES}


def _step(g, masks=None, **coef):
    a = _fixture_inputs(g)
    eps = torch.from_numpy(g["eps"][:2]).double()
    return R.train_step(a["params"], a["running"], a["X"], a["Xraw"], a["sf"], a["graph"], a["train_mask"], a["valid_mask"],
                        eps_train=eps[0], eps_eval=eps[1], masks=masks, **(coef or dict(le=1, la=1, ke=1, ka=1)))


def test_restatement_reproduces_fixture(golden):
    """Dropout 0, unit loss weights: the first epoch's losses, every gradient and the updated running statistics."""
    g = golden("graphsci")
    ref = _step(g)
    got = np.array([ref["losses"][k] for k in ("loss_adj", "loss_exp", "kl", "train_loss", "valid_loss")])
    assert np.allclose(got, g["e1.losses"], rtol=TOL), (got, g["e1.losses"])
    gmax = max(np.abs(g[k]).max() for k in g.files if k.startswith("grad."))
    seen = set()
    for k in g.files:
        if not k.startswith("grad.") or ".dec_log_std." in k:
            continue
        name = k[len("grad."):]
        seen.add(name)
        mine = ref["grads"][name].numpy()
        if np.abs(g[k]).max() < 1e-6 * gmax:
            # biases in front of a BatchNorm: the exact gradient is zero, the float32 fixture holds rounding noise
            assert np.abs(mine).max() < 1e-5 * gmax, name
        else:
            assert rel_err(mine, g[k]) < 5e-4, name
    assert seen == set(R.PARAMS)
    for key, (rm, rv) in ref["running"].items():
        assert rel_err(rm, g[f"e1.aemodel.{key}.running_mean"]) < TOL, key
        assert rel_err(rv, g[f"e1.aemodel.{key}.running_var"]) < TOL, key


def _reference_step(g, masks, le, la, ke, ka, monkeypatch, tmp_path):
    """The reference's own pieces in float64: train-mode GNN / AE forward, get_loss, evaluate (eval mode, the running statistics
    the train forward just updated), backward.  F.dropout hands out ``masks`` in call order; torch.normal is mean + std·ε."""
    from oracle import dgl_lite
    ref = ref_loader.graphsci()
    a = _fixture_inputs(g)
    n, G = g["X"].shape
    monkeypatch.chdir(tmp_path)                    # GraphSCI.__init__ creates ./graphsci
    drawn = []

    def dropout(x, p=0.5, training=True, inplace=False):
        if not training:
            return x
        site = R.SITES[len(drawn)]
        drawn.append(site)
        assert tuple(x.shape) == tuple(masks[site].shape), (site, x.shape)
        return x * masks[site]

    eps = iter(torch.from_numpy(g["eps"][:2]).double())
    monkeypatch.setattr(torch.nn.functional, "dropout", dropout)
    monkeypatch.setattr(torch, "normal", lambda mean, std: mean + std * next(eps))
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        m = ref.GraphSCI(num_cells=n, num_genes=G, dataset="pin", dropout=0.1)
        for scope in ("aemodel", "gnnmodel"):
            getattr(m, scope).load_state_dict({k[len(f"init.{scope}."):]: torch.from_numpy(g[k]) for k in g.files
                                               if k.startswith(f"init.{scope}.")})
        gr = dgl_lite.Graph(g["src"], g["dst"], G)
        gr.ndata["feat"] = a["X"].t().contiguous()
        m.adj, m.size_factors = a["graph"].adj, a["sf"]
        m.gnnmodel.train()
        m.aemodel.train()
        z, ls, mu = m.gnnmodel(gr)
        z_exp, mean, disp, pi = m.aemodel(a["X"], z, m.size_factors)
        losses = m.get_loss(a["Xraw"], m.adj, z, ls, mu, z_exp, mean, disp, pi, a["train_mask"], le, la, ke, ka)
        assert drawn == list(R.SITES)
        valid, _, z_exp_eval = m.evaluate(a["X"], a["Xraw"], gr, a["valid_mask"], le, la, ke, ka)
        assert drawn == list(R.SITES)              # evaluate runs in eval mode: no further masks
        losses[-1].backward()
    finally:
        torch.set_default_dtype(default)
    out = {"losses": dict(zip(R.LOSSES, (float(v) for v in losses))), "z_exp": z_exp_eval.detach()}
    out["losses"]["valid_loss"] = float(valid)
    out["grads"] = {f"{s}.{k}": p.grad for s in ("aemodel", "gnnmodel") for k, p in getattr(m, s).named_parameters() if p.grad is not None}
    sd = m.aemodel.state_dict()
    out["running"] = {k: (sd[f"{k}.running_mean"], sd[f"{k}.running_var"]) for k in R.BN_KEYS}
    return out


def _assert_agree(got, want, tol):
    for k, v in want["losses"].items():
        assert abs(got["losses"][k] - v) <= tol * abs(v), (k, got["losses"][k], v)
    assert set(got["grads"]) == set(want["grads"])
    gmax = max(float(v.abs().max()) for v in want["grads"].values())
    for k, v in want["grads"].items():
        # a bias in front of a BatchNorm has an exact gradient of zero: bounded against the gradient scale
        assert float((got["grads"][k] - v).abs().max()) <= tol * max(float(v.abs().max()), gmax * 1e-3) or rel_err(got["grads"][k], v) <= tol, k
    for k, (rm, rv) in want["running"].items():
        assert rel_err(got["running"][k][0], rm) <= tol and rel_err(got["running"][k][1], rv) <= tol, k
    assert rel_err(got["z_exp"], want["z_exp"]) <= tol


@needs_ref
def test_restatement_matches_reference_with_dropout(golden, monkeypatch, tmp_path):
    """Dropout 0.1 at every one of the ten sites, two independent masks into dec_mean, non-unit loss weights."""
    g = golden("graphsci")
    masks = _masks(g)
    want = _reference_step(g, masks, monkeypatch=monkeypatch, tmp_path=tmp_path, **COEF)
    got = _step(g, masks, **COEF)
    _assert_agree(got, want, PIN)


def _distance(a, b):
    """Largest relative difference over the losses and the gradients of two restated steps."""
    d = max(abs(a["losses"][k] - b["losses"][k]) / abs(b["losses"][k]) for k in b["losses"])
    return max(d, max(rel_err(a["grads"][k], b["grads"][k]) for k in b["grads"] if float(b["grads"][k].abs().max()) > 1e-12))


def test_mask_sites_and_eval_statistics_are_pinned(golden):
    """A restatement that swapped the two dec_mean masks, or that evaluated the validation loss with the running statistics from
    before the step, lands far outside the tolerance the reference pins it to."""
    g = golden("graphsci")
    masks = _masks(g)
    base = _step(g, masks, **COEF)
    swapped = dict(masks, h2_mean=masks["h2_log_std"], h2_log_std=masks["h2_mean"])
    assert _distance(_step(g, swapped, **COEF), base) > 1e6 * PIN
    for a, b in (("enc.5", "dec_pi"), ("dec_disp", "dec_mean")):
        assert _distance(_step(g, dict(masks, **{a: masks[b], b: masks[a]}), **COEF), base) > 1e6 * PIN, (a, b)
    a = _fixture_inputs(g)
    eps = torch.from_numpy(g["eps"][1]).double()
    stale, _ = R.evaluate(a["params"], a["running"], a["X"], a["Xraw"], a["sf"], a["graph"], a["valid_mask"], eps=eps, **COEF)
    assert abs(float(stale) - base["losses"]["valid_loss"]) > 1e6 * PIN * abs(base["losses"]["valid_loss"])
