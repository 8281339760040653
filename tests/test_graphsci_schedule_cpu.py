"""GraphSCI's choice of training schedule (modules/graphsci.py: choose_schedule) and a float64 restatement of the lean
schedule's backward algebra against autograd (no GPU needed).

The lean schedule never stores the heads' BatchNorm outputs, their loss gradients or any dropout mask: each head's BatchNorm
backward is formed from two column sums of the loss gradient and written over that head's pre-BatchNorm buffer, the
multiply layer's ReLU-with-dropout backward reads only its dropped output h_d, and a freed head buffer takes the multiply
layer's gradient.  The restatement below runs those steps in the schedule's order on five named buffers and must give
autograd's gradients."""
import pytest
import torch
import torch.nn.functional as F

from dance_b200.modules import graphsci

GiB = 2**30
H100 = 80 * GiB


@pytest.mark.parametrize("cells,want", [(20_000, "materialise"), (200_000, "materialise"), (500_000, "lean")])
def test_schedule_at_configuration_3_sizes(cells, want):
    assert graphsci.choose_schedule(cells, 3000, H100) == want


def test_schedule_is_monotone_in_cells():
    for genes in (1000, 3000, 10000):
        for mem in (40 * GiB, H100, 141 * 10**9):
            picks = [graphsci.choose_schedule(n, genes, mem) for n in range(1000, 2_000_001, 1000)]
            first_lean = picks.index("lean") if "lean" in picks else len(picks)
            assert all(p == "materialise" for p in picks[:first_lean]) and all(p == "lean" for p in picks[first_lean:])


def test_schedule_estimates():
    # the lean schedule keeps 5 [cells, genes] matrices of its own against 25, plus the caller's
    for n, g in ((1000, 100), (500_000, 3000)):
        lean, mat = graphsci.schedule_bytes("lean", n, g), graphsci.schedule_bytes("materialise", n, g)
        assert mat - lean == 4 * n * g * 20
    assert graphsci.schedule_bytes("lean", 500_000, 3000) < graphsci.HEADROOM * H100 < graphsci.schedule_bytes("materialise", 500_000, 3000)


def test_schedule_override(monkeypatch):
    class M:
        N, G, device = 500_000, 3000, None
    monkeypatch.setattr(graphsci, "SCHEDULE", "materialise")
    assert graphsci.GraphSCI.schedule(M()) == "materialise"
    monkeypatch.setattr(graphsci, "SCHEDULE", "lean")
    assert graphsci.GraphSCI.schedule(M()) == "lean"
    monkeypatch.setattr(graphsci, "SCHEDULE", "fast")
    with pytest.raises(ValueError):
        graphsci.GraphSCI.schedule(M())


def _act_loss(y):
    """A smooth stand-in for the ZINB / MSE loss of the three heads' BatchNorm outputs, and its elementwise gradient."""
    w = torch.linspace(-1, 1, y[0].numel(), dtype=torch.float64).view_as(y[0])
    loss = sum((w * torch.tanh(yk) + 0.3 * (k + 1) * yk * yk).sum() for k, yk in enumerate(y))
    grads = [w * (1 - torch.tanh(yk)**2) + 0.6 * (k + 1) * yk for k, yk in enumerate(y)]
    return loss, grads


@pytest.mark.parametrize("p", [0.0, 0.3])
def test_lean_backward_algebra_against_autograd(p):
    torch.manual_seed(0)
    n, g, h = 40, 12, 8
    dt = torch.float64
    X = torch.rand(n, g, dtype=dt)
    keep = lambda shape: (torch.rand(shape, dtype=dt) >= p).to(dt) / (1 - p)       # noqa: E731
    mX, m1, mh = keep((n, g)), keep((n, g)), [keep((n, h)) for _ in range(3)]
    zf = torch.randn(g, g, dtype=dt).requires_grad_()
    b0 = torch.randn(g, dtype=dt).requires_grad_()
    enc = torch.rand(n, h, dtype=dt)                                   # the encoder's output, fed to the heads
    W = [torch.randn(g, h, dtype=dt).requires_grad_() for _ in range(3)]
    b = [torch.randn(g, dtype=dt).requires_grad_() for _ in range(3)]
    gamma = [(1 + 0.1 * torch.randn(g, dtype=dt)).requires_grad_() for _ in range(3)]
    beta = [(0.1 * torch.randn(g, dtype=dt)).requires_grad_() for _ in range(3)]
    eps = 1e-5

    # autograd: the materialising schedule's algebra.  The heads read the (dropped) multiply-layer output through a fixed
    # projection P so that its gradient path runs through every head, as dh = Σ_k dpre_k·W_k does through the encoder.
    Pm = torch.randn(g, h, dtype=dt) / g
    leaves = [zf, b0, *W, *b, *gamma, *beta]
    h0 = torch.relu((X * mX) @ zf + b0)
    hd = h0 * m1
    inp = [(hd @ Pm + enc) * mh[k] for k in range(3)]
    y = [F.batch_norm(inp[k] @ W[k].t() + b[k], None, None, gamma[k], beta[k], True, 0.0, eps) for k in range(3)]
    loss, _ = _act_loss(y)
    want = dict(zip(("zf", "b0", "W0", "W1", "W2", "b0h", "b1h", "b2h", "g0", "g1", "g2", "be0", "be1", "be2"),
                    torch.autograd.grad(loss, leaves)))

    # the lean schedule, on five named [n, g] buffers
    with torch.no_grad():
        buf = {}
        buf["scratch"] = X * mX                                          # X_d
        buf["h_d"] = torch.relu(buf["scratch"] @ zf + b0) * m1            # h0 with the enc.1 dropout applied in place
        inp = [(buf["h_d"] @ Pm + enc) * mh[k] for k in range(3)]
        for k in range(3):
            buf[f"pre{k}"] = inp[k] @ W[k].t() + b[k]
        stats = [(buf[f"pre{k}"].mean(0), (buf[f"pre{k}"].var(0, unbiased=False) + eps).rsqrt()) for k in range(3)]
        xh = [(buf[f"pre{k}"] - stats[k][0]) * stats[k][1] for k in range(3)]
        _, gy = _act_loss([xh[k] * gamma[k] + beta[k] for k in range(3)])
        got = {}
        for k in range(3):      # two column sums, then dpre over pre in place
            sg, sgx = gy[k].sum(0), (gy[k] * xh[k]).sum(0)
            buf[f"pre{k}"].copy_(gamma[k] * stats[k][1] * (gy[k] - sg / n - xh[k] * sgx / n))
            got[f"g{k}"], got[f"be{k}"] = sgx, sg
        dh = torch.zeros(n, g, dtype=dt)
        for k in range(3):      # heads backward: weight gradient, bias gradient, input gradient (dropout redrawn)
            dpre = buf[f"pre{k}"]
            got[f"W{k}"], got[f"b{k}h"] = dpre.t() @ inp[k], dpre.sum(0)
            dh += ((dpre @ W[k]) * mh[k]) @ Pm.t()
        for k in (1, 2):
            del buf[f"pre{k}"]
        buf["pre0"].copy_(dh)                                            # the multiply layer's gradient in a freed head buffer
        buf["pre0"].mul_(m1)                                             # dropout redrawn on the gradient
        buf["pre0"].mul_((buf["h_d"] > 0).to(dt))                        # ReLU backward from h_d alone
        got["b0"] = buf["pre0"].sum(0)
        got["zf"] = buf["scratch"].t() @ buf["pre0"]                     # scratch still holds X_d
    for k, v in want.items():
        assert torch.allclose(got[k], v, rtol=1e-10, atol=1e-10 * float(v.abs().max()) + 1e-12), k
    # where the forward dropped an element h_d is 0, so the ReLU mask alone already zeroes it
    assert bool(((buf["h_d"] > 0) <= (m1 > 0)).all())
