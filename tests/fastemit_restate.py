"""fp64 restatement of the FastEmit gradient of csrc/loss.cu, and its independent oracle (TEST INFRASTRUCTURE).

grad_fastemit()   d S / d logits by the branches of the gradient kernels with fastemit_lambda = lam
                  (include/edgedict_b200.h, eb_rnnt_loss_bwd_fe); at lam = 0 the operations of
                  loss_restate.grad_formula, so the same bits
surrogate_grad()  the same gradient by torch autograd (fp64, any device) of the surrogate
                      S_b = -log P_b - lam sum_{t < T_b, u < U_b - 1} sg(gamma(t,u)) y(t,u),
                      y(t,u) = log_softmax(x(t,u))[label[u]],  gamma(t,u) = exp(alpha(t,u) + y(t,u) + beta(t,u+1) - log P_b)
                  with log P_b from an alpha recursion that autograd differentiates; nothing of the kernels' formula

Lengths are clamped as the kernels clamp them (loss_restate.lengths)."""
import math

import torch

from tests import loss_restate as lr

f64 = torch.float64


def grad_fastemit(a, b, d, ll, lpl, x, labels, xlen, ylen, blank, lam, terms=False):
    """g [B,T,U,V] fp64 from alpha, beta, denom, lpl [B,T,U], ll [B] and the logits x [B,T,U,V], zero on padded cells:
        g_v = exp(c_all + x_v) - [v = blank] exp(c_blank + x_v) - [v = label[u]] exp(c_lab + x_v)
    with loss_restate.grad_formula's c_blank, and on the cells u < U_b - 1, for lam > 0,
        c_all = d + logaddexp(a + b - ll, log lam + a + beta(t,u+1) + lpl - ll),   c_lab = a - ll + d + beta(t,u+1) + log1p(lam)
    (grad_formula's c_all = a + b - ll + d and c_lab elsewhere, and everywhere at lam = 0).
    With terms=True also returns the terms and their exponents' operand magnitudes (as grad_formula does), with the
    FastEmit parts: mag_q = |log lam| + |a| + |beta(t,u+1)| + |lpl| + |ll|, |L| of the logaddexp, and fe (the cells
    where the FastEmit branch ran)."""
    a, b, d, ll, lpl, x = a.to(f64), b.to(f64), d.to(f64), ll.to(f64), lpl.to(f64), x.to(f64)
    B, T, U = a.shape
    dev = a.device
    valid = lr.valid_cells(xlen, ylen, T, U, dev)
    Tn, Un = lr.lengths(xlen, ylen, T, U, dev)
    Tn, Un = Tn[:, None, None], Un[:, None, None]
    ll = ll[:, None, None]
    ninf = torch.full_like(a, -math.inf)
    zero = torch.zeros_like(a)
    t_idx = torch.arange(T, device=dev)[None, :, None]
    u_idx = torch.arange(U, device=dev)[None, None, :]
    has_lab = valid & (u_idx < Un - 1)
    b_next_u = torch.cat([b[:, :, 1:], ninf[:, :, :1]], dim=2)
    fe = has_lab & (lam > 0)
    c_all = torch.where(valid, a + b - ll + d, ninf)
    L = zero
    if lam > 0:
        p = a + b - ll
        q = math.log(lam) + a + b_next_u + lpl - ll
        L = torch.where(fe, torch.logaddexp(p, q), zero)
        c_all = torch.where(fe, d + L, c_all)
    main = torch.exp(c_all[..., None] + x)
    g = main.clone()
    b_next_t = torch.cat([b[:, 1:], ninf[:, :1]], dim=1)
    last = (t_idx == Tn - 1) & (u_idx == Un - 1)
    c_blank = torch.where(t_idx < Tn - 1, a - ll + d + b_next_t, torch.where(last, a - ll + d, ninf))
    c_blank = torch.where(valid, c_blank, ninf)
    corr_b = torch.exp(c_blank + x[..., blank])
    g[..., blank] -= corr_b
    mag_all = torch.where(valid, a.abs() + b.abs() + ll.abs() + d.abs(), zero)
    mag_b = torch.where(valid, a.abs() + ll.abs() + d.abs() + torch.where(t_idx < Tn - 1, b_next_t.abs(), zero), zero)
    absum = main.clone()
    absum[..., blank] += corr_b
    corr_l = mag_l = None
    if U > 1:
        lab = torch.as_tensor(labels, device=dev).long()[:, None, :, None].expand(B, T, U - 1, 1)
        c_lab = torch.where(has_lab, a - ll + d + b_next_u, ninf)
        if lam > 0:
            c_lab = c_lab + math.log1p(lam)
        c_lab = c_lab[:, :, :U - 1]
        xl = torch.gather(x[:, :, :U - 1], 3, lab)
        corr_l = torch.exp(c_lab[..., None] + xl)
        g[:, :, :U - 1].scatter_add_(3, lab, -corr_l)
        absum[:, :, :U - 1].scatter_add_(3, lab, corr_l)
        mag_l = torch.where(has_lab, a.abs() + ll.abs() + d.abs() + b_next_u.abs(), zero)
    g[~valid] = 0
    if not terms:
        return g
    absum[~valid] = 0
    mag_q = torch.where(fe, abs(math.log(lam)) + a.abs() + b_next_u.abs() + lpl.abs() + ll.abs(), zero) \
        if lam > 0 else zero
    return g, dict(absum=absum, main=main.where(valid[..., None], 0.0), mag_all=mag_all, mag_b=mag_b,
                   corr_b=corr_b.where(valid, 0.0), corr_l=corr_l, mag_l=mag_l, mag_q=mag_q, L=L.abs(), fe=fe)


def _alpha_ll(y_blank, y_lab, Tb, Ub):
    """log P of one utterance from its blank / label log-probs [T, U] by the alpha recursion, differentiable."""
    ninf = y_blank.new_tensor(-math.inf)
    al = [[None] * Ub for _ in range(Tb)]
    for t in range(Tb):
        for u in range(Ub):
            if t == 0 and u == 0:
                al[t][u] = y_blank.new_zeros(())
                continue
            stay = al[t - 1][u] + y_blank[t - 1, u] if t > 0 else ninf
            emit = al[t][u - 1] + y_lab[t, u - 1] if u > 0 else ninf
            al[t][u] = torch.logaddexp(stay, emit)
    return al[Tb - 1][Ub - 1] + y_blank[Tb - 1, Ub - 1]


def surrogate_grad(x, labels, xlen, ylen, blank, lam, weights=None):
    """(d sum_b w_b S_b / d x [B,T,U,V] fp64, -log P [B] fp64) by autograd; w_b = weights[b] (default 1).  An
    utterance without frames (T_b = 0) has no alignment: cost +inf and a zero gradient."""
    x = x.detach().to(f64).clone().requires_grad_(True)
    B, T, U, V = x.shape
    Tn, Un = lr.lengths(xlen, ylen, T, U, "cpu")
    y = torch.log_softmax(x, -1)
    total = x.new_zeros(())
    costs = []
    for bi in range(B):
        Tb, Ub = int(Tn[bi]), int(Un[bi])
        if Tb == 0:
            costs.append(math.inf)
            continue
        yb = y[bi, :Tb, :Ub, blank]
        lab = torch.as_tensor(labels[bi][:Ub - 1], device=x.device).long()
        yl = torch.zeros(Tb, Ub, dtype=f64, device=x.device)
        if Ub > 1:
            yl = torch.cat([torch.gather(y[bi, :Tb, :Ub - 1], 2, lab[None, :, None].expand(Tb, Ub - 1, 1))[..., 0],
                            yl[:, :1]], dim=1)
        logp = _alpha_ll(yb, yl, Tb, Ub)
        s = -logp
        if lam > 0 and Ub > 1:
            with torch.no_grad():
                xl_ = torch.tensor([Tb], dtype=torch.int32)
                yl_ = torch.tensor([Ub - 1], dtype=torch.int32)
                al, be, llf, _ = lr.lattice(yb[None], yl[None], xl_, yl_)
                gamma = torch.exp(al[0, :, :Ub - 1] + yl[:, :Ub - 1] + be[0, :, 1:] - llf[0])
            s = s - lam * (gamma * yl[:, :Ub - 1]).sum()
        w = 1.0 if weights is None else float(weights[bi])
        total = total + w * s
        costs.append(float(-logp.detach()))
    if total.requires_grad:
        total.backward()
    g = x.grad if x.grad is not None else torch.zeros_like(x)
    return g.detach(), torch.tensor(costs, dtype=f64)
