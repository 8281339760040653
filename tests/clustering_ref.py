"""Float64 restatements of the clustering kernels (csrc/dec.cu, csrc/em.cu), written from the formulas those kernels cite:
SpaGCN's DEC head (spagcn.py:391-425), one Lloyd step of k-means (scgnn2.py:186) and scGNN's regulariser weights, Cell-type loss
and L1 term (scgnn2.py:716-752, 1268-1274, 1316-1326).  Every function takes torch tensors (any device) or numpy arrays, computes
in float64 from the float32 values it is given, and stands alone: nothing here imports the library."""
import numpy as np
import torch

F64 = torch.float64


def sq_dist(X, C):
    """‖x_i − c_j‖² [n, k] in float64, summed over the columns one at a time in one fixed order: two equal rows of C give
    bit-equal columns, and integer-valued inputs give exact distances."""
    X, C = X.to(F64), C.to(F64)
    D = torch.zeros((X.shape[0], C.shape[0]), dtype=F64, device=X.device)
    for c in range(X.shape[1]):
        D += (X[:, c:c + 1] - C[:, c])**2
    return D


# ---- DEC head ---------------------------------------------------------------------------------------------------------------
def dec_t(d2, alpha):
    return 1.0 / ((1.0 + d2 / alpha) + 1e-8)


def dec_q(d2, alpha):
    """q_ij = u_ij / Σ_j u_ij with u = t^(α+1) / 2, t = 1 / ((1 + d²/α) + 1e-8)."""
    u = dec_t(d2, alpha)**(alpha + 1.0) / 2.0
    return u / u.sum(1, keepdim=True)


def dec_target(q):
    """p = q² / colsum(q), row-normalised."""
    p = q**2 / q.sum(0)
    return p / p.sum(1, keepdim=True)


def dec_loss_terms(p, q):
    """p·log(p / (q + 1e-6)); the loss is their row sums' mean."""
    return p * torch.log(p / (q + 1e-6))


def dec_dl_dd2(d2, p, alpha, n):
    """Closed form of c = ∂L/∂d² for the rows of ``d2`` (L divides by the full row count ``n``), and the same expression with
    every term taken by magnitude before the one subtraction in it: ∂L/∂u_j = (g_j − Σ_k g_k q_k) / S with g = ∂L/∂q.  Returns
    (c, c_abs), c_abs ≥ |c|."""
    t = dec_t(d2, alpha)
    u = t**(alpha + 1.0) / 2.0
    S = u.sum(1, keepdim=True)
    q = u / S
    g = -p / (n * (q + 1e-6))
    gq = (g * q).sum(1, keepdim=True)
    du_dd2 = -(alpha + 1.0) / (2.0 * alpha) * t**(alpha + 2.0)
    return (g - gq) / S * du_dd2, (g.abs() + gq.abs()) / S * du_dd2.abs()


def dec_reference(z, mu, p, alpha, max_elems=1 << 25):
    """The DEC head in float64 over row chunks of at most ``max_elems`` (rows·K·h) elements, so that 200 000 × 64 × 256 fits.

    ``z`` [n, h], ``mu`` [K, h] and ``p`` [n, K] are the kernels' float32 operands.  c = ∂L/∂d² comes from float64 autograd of
    the loss with respect to d², then dz_i = 2 Σ_j c_ij (z_i − μ_j) and dμ_j = −2 Σ_i c_ij (z_i − μ_j).  Error scales per element:
    scale_dz[i, c] = Σ_j c̄_ij |z_ic − μ_jc| and scale_dmu[j, c] = Σ_i of the same terms, with c̄ the magnitude form of
    :func:`dec_dl_dd2`.  Returns a dict with q, loss, loss_abs (mean_i Σ_j |p·log(p/(q+1e-6))|), dz, dmu, scale_dz, scale_dmu."""
    n, h = z.shape
    K = mu.shape[0]
    dev = z.device
    mu64 = mu.to(F64)
    q_all = torch.empty((n, K), dtype=F64, device=dev)
    dz = torch.empty((n, h), dtype=F64, device=dev)
    scale_dz = torch.empty_like(dz)
    dmu = torch.zeros((K, h), dtype=F64, device=dev)
    scale_dmu = torch.zeros_like(dmu)
    loss = loss_abs = 0.0
    step = max(1, max_elems // (K * h))
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        z64, p64 = z[r0:r1].to(F64), p[r0:r1].to(F64)
        d2 = sq_dist(z64, mu64).requires_grad_()
        q = dec_q(d2, alpha)
        terms = dec_loss_terms(p64, q)
        c, = torch.autograd.grad(terms.sum() / n, d2)
        terms = terms.detach()
        loss += float(terms.sum()) / n
        loss_abs += float(terms.abs().sum()) / n
        q_all[r0:r1] = q.detach()
        _, c_abs = dec_dl_dd2(d2.detach(), p64, alpha, n)
        diff = z64[:, None, :] - mu64[None]
        dz[r0:r1] = 2.0 * torch.einsum("ij,ijc->ic", c, diff)
        dmu -= 2.0 * torch.einsum("ij,ijc->jc", c, diff)
        diff.abs_()
        scale_dz[r0:r1] = torch.einsum("ij,ijc->ic", c_abs, diff)
        scale_dmu += torch.einsum("ij,ijc->jc", c_abs, diff)
    return dict(q=q_all, loss=loss, loss_abs=loss_abs, dz=dz, dmu=dmu, scale_dz=scale_dz, scale_dmu=scale_dmu)


# ---- k-means ----------------------------------------------------------------------------------------------------------------
def nearest_two(D):
    """(best, second best, index of the best: the lowest index among equal minima) of each row of a distance matrix."""
    top = torch.topk(D, min(2, D.shape[1]), dim=1, largest=False).values
    best = top[:, 0]
    second = top[:, 1] if D.shape[1] > 1 else torch.full_like(best, float("inf"))
    first = (D == best[:, None]).to(torch.int8).argmax(1)
    return best, second, first


def lloyd_update(X, C, labels):
    """New centres = the float64 mean of each cluster's points under the given labels; an empty cluster keeps its centre.
    Returns (centres float64 [k, d], counts int64 [k])."""
    k = C.shape[0]
    lab = labels.long()
    sums = torch.zeros((k, X.shape[1]), dtype=F64, device=X.device).index_add_(0, lab, X.to(F64))
    counts = torch.bincount(lab, minlength=k)
    new = C.to(F64).clone()
    nz = counts > 0
    new[nz] = sums[nz] / counts[nz, None].to(F64)
    return new, counts


def lloyd_stats(D, labels, prev_labels, C_old, C_new):
    """The step's statistics: inertia Σ_i ‖x_i − C_old[label_i]‖² (float64 distances ``D`` to the old centres), ‖C_new − C_old‖²
    and the number of labels that differ from ``prev_labels``."""
    lab = labels.long()
    inertia = float(D.gather(1, lab[:, None]).sum())
    shift2 = float(((C_new.to(F64) - C_old.to(F64))**2).sum())
    return inertia, shift2, int((labels.long() != prev_labels.long()).sum())


def lloyd_loop(X, C0, max_iter=300):
    """Float64 Lloyd iterations from C0 until no label changes or the centres stop moving (ops.kmeans with tol = 0), then one
    more assignment.  Returns (labels, iterations, smallest relative gap between the best and second-best centre seen)."""
    X = X.to(F64)
    C = C0.to(F64).clone()
    prev = torch.full((X.shape[0], ), -1, dtype=torch.long, device=X.device)
    min_gap = float("inf")

    def assign(C):
        nonlocal min_gap
        best, second, lab = nearest_two(sq_dist(X, C))
        min_gap = min(min_gap, float(((second - best) / best.clamp_min(1e-300)).min()))
        return lab

    it = 0
    for it in range(1, max_iter + 1):
        lab = assign(C)
        changed = int((lab != prev).sum())
        C_new, _ = lloyd_update(X, C, lab)
        shift2 = float(((C_new - C)**2).sum())
        C, prev = C_new, lab
        if changed == 0 or shift2 <= 0.0:
            break
    return assign(C), it, min_gap


# ---- scGNN regulariser, Cell-type loss, L1 ----------------------------------------------------------------------------------
def _rows(rowptr):
    rowptr = np.asarray(rowptr, dtype=np.int64)
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))


def regu_weights(rowptr, colidx, labels, n_clusters):
    """w_j = deg_j · Σ_{i ∈ cluster(j)} 1/deg_i, deg = row length without the diagonal entry; a zero-degree row adds nothing
    and a label outside [0, n_clusters) gives w = 0."""
    rows, colidx, labels = _rows(rowptr), np.asarray(colidx), np.asarray(labels, dtype=np.int64)
    n = len(rowptr) - 1
    deg = np.bincount(rows[colidx != rows], minlength=n).astype(np.float64)
    return _cluster_weights(deg, deg, labels, n_clusters)


def regu_weights_weighted(rowptr, colidx, vals, labels, n_clusters):
    """The weighted, directed form: w_j = colsum_j · Σ_{i ∈ cluster(j)} 1/rowsum_i over the off-diagonal entries; a row whose
    sum is zero adds nothing."""
    rows, colidx, vals = _rows(rowptr), np.asarray(colidx), np.asarray(vals, dtype=np.float64)
    n = len(rowptr) - 1
    off = colidx != rows
    rowsum = np.bincount(rows[off], weights=vals[off], minlength=n)
    colsum = np.bincount(colidx[off], weights=vals[off], minlength=n)
    return _cluster_weights(rowsum, colsum, np.asarray(labels, dtype=np.int64), n_clusters)


def _cluster_weights(rowsum, colsum, labels, n_clusters):
    ok = (labels >= 0) & (labels < n_clusters)
    inv = np.divide(1.0, rowsum, out=np.zeros_like(rowsum), where=rowsum != 0)
    per = np.bincount(labels[ok], weights=inv[ok], minlength=n_clusters)
    return np.where(ok, colsum * per[np.where(ok, labels, 0)], 0.0)


def celltype_loss_grad(recon, target, x_dropout, row_weight, relu_mask):
    """loss = Σ_i w_i Σ_g (r − x)² + ‖(xd − r)[xd ≠ 0]‖ over the first cols_orig columns, and its gradient with respect to r:
    2 w_i (r − x) − [xd ≠ 0] (xd − r) / ‖·‖ (the second term is 0 when the norm is 0), zeroed where r ≤ 0 under ``relu_mask``.
    Returns (loss, grad, grad_abs): grad_abs sums the magnitudes of the gradient's terms."""
    r, x, xd, w = (torch.as_tensor(a).to(F64) for a in (recon, target, x_dropout, row_weight))
    co = xd.shape[1]
    a = 2.0 * w[:, None] * (r - x)
    m = xd != 0
    v = torch.where(m, xd - r[:, :co], torch.zeros_like(xd))
    nrm = float(torch.sqrt((v**2).sum()))
    b = torch.zeros_like(r)
    if nrm > 0:
        b[:, :co] = v / nrm
    grad, grad_abs = a - b, a.abs() + b.abs()
    if relu_mask:
        keep = r > 0
        grad, grad_abs = torch.where(keep, grad, 0.0), torch.where(keep, grad_abs, 0.0)
    loss = float((w[:, None] * (r - x)**2).sum()) + nrm
    return loss, grad, grad_abs


def l1_grad_add(param, grad, coef):
    """(grad + coef·sign(p) in float32, with sign 0 for +0 and −0, and coef·Σ|p| in float64)."""
    p = torch.as_tensor(param)
    s = (p > 0).to(torch.float32) - (p < 0).to(torch.float32)
    return torch.as_tensor(grad) + np.float32(coef) * s, float(coef) * float(p.to(F64).abs().sum())
