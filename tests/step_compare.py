"""Comparison helpers of the engine-step tests (test infrastructure): worst-row error, views of a flat parameter buffer, float64
Adam on given gradients."""
import torch


def row_rel_err(a, ref):
    """Worst row of ‖a_i − ref_i‖ / ‖ref_i‖.  Rows whose reference norm is below 1e-3 of the RMS row
    norm are measured against that floor instead, so that a near-zero row does not turn rounding into a large ratio."""
    a = torch.as_tensor(a).double()
    ref = torch.as_tensor(ref).double().to(a.device)
    a, ref = a.reshape(a.shape[0], -1), ref.reshape(ref.shape[0], -1)
    den = ref.norm(dim=1)
    floor = 1e-3 * float(den.pow(2).mean().sqrt())
    return float(((a - ref).norm(dim=1) / den.clamp(min=max(floor, 1e-300))).max())


def adam_reference(flat0, grads, lr):
    """float64 torch.optim.Adam (the engines' defaults: betas 0.9 / 0.999, eps 1e-8, no weight decay) over the flat parameter
    vector, applied to the given sequence of gradients."""
    p = flat0.double().clone().requires_grad_()
    opt = torch.optim.Adam([p], lr=lr)
    for g in grads:
        p.grad = g.double()
        opt.step()
    return p.detach()


def param_views(params, flat):
    """The named parameters of a FlatParams, as views into a copy `flat` of its flat buffer."""
    base = params.flat.storage_offset()
    return {k: flat[v.storage_offset() - base:v.storage_offset() - base + v.numel()].view(v.shape) for k, v in params.p.items()}
