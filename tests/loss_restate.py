"""fp64 restatements of the RNN-T loss kernels of csrc/loss.cu, in torch on any device (TEST INFRASTRUCTURE).

lattice()       alphas, betas, ll_fwd, ll_bwd from the per-cell log-probs lpb = log p(blank), lpl = log p(label[u]),
                one anti-diagonal at a time for the whole batch
grad_formula()  d loss / d logits from a lattice, the statistics and the logits, by the branches of the gradient kernels

Both clamp the lengths as the kernels do (include/edgedict_b200.h): utterance b has the cells t < T_b = min(max(xlen,
0), maxT), u < U_b = min(max(ylen, 0), maxU - 1) + 1.  tests/test_loss_host.py pins them to the C oracle
(oracle/rnnt_loss_oracle.c)."""
import math

import numpy as np
import torch

f64 = torch.float64


def planted_labels(rng, B, U, V, blank):
    """Random labels != blank [B, U-1] int32, with columns 127, 128, V - 1 and the two neighbours of the blank planted in
    every row (label capture at chunk and tile edges)."""
    if U == 1:
        return np.zeros((B, 0), np.int32)
    r = rng.randint(0, V - 1, size=(B, U - 1))
    lab = r + (r >= blank)
    special = [c for c in (127, 128, V - 1, blank - 1, blank + 1) if 0 <= c < V and c != blank]
    for b in range(B):
        for i, c in enumerate(special[b % len(special):] + special[:b % len(special)]):
            if i < U - 1:
                lab[b, (i + b) % (U - 1)] = c
    return lab.astype(np.int32)


def lengths(xlen, ylen, T, U, device):
    """Clamped (T_b, U_b) as int64 tensors on `device`."""
    Tn = torch.as_tensor(xlen, device=device).long().clamp(0, T)
    Un = (torch.as_tensor(ylen, device=device).long().clamp(min=0) + 1).clamp(max=U)
    return Tn, Un


def valid_cells(xlen, ylen, T, U, device):
    """[B, T, U] bool: the cells the loss reads."""
    Tn, Un = lengths(xlen, ylen, T, U, device)
    t = torch.arange(T, device=device)[None, :, None]
    u = torch.arange(U, device=device)[None, None, :]
    return (t < Tn[:, None, None]) & (u < Un[:, None, None])


def _diagonal(n, T, U, device):
    u = torch.arange(U, device=device)
    u = u[(n - u >= 0) & (n - u < T)]
    return n - u, u


def lattice(lpb, lpl, xlen, ylen, need_beta=True):
    """(alphas, betas, ll_fwd, ll_bwd) in fp64 from lpb, lpl [B, T, U]:
        alpha(0,0) = 0, alpha(t,u) = logaddexp(alpha(t-1,u) + lpb(t-1,u), alpha(t,u-1) + lpl(t,u-1))
        beta(T_b-1,U_b-1) = lpb(T_b-1,U_b-1), beta(t,u) = logaddexp(beta(t+1,u) + lpb(t,u), beta(t,u+1) + lpl(t,u))
        ll_fwd = alpha(T_b-1,U_b-1) + lpb(T_b-1,U_b-1), ll_bwd = beta(0,0); both -inf when T_b = 0.
    A term that leaves the utterance's cells is -inf.  Padded cells of alphas / betas are NaN; betas is None without
    need_beta.  lpb / lpl of padded cells are never used."""
    lpb, lpl = lpb.to(f64), lpl.to(f64)
    B, T, U = lpb.shape
    dev = lpb.device
    Tn, Un = lengths(xlen, ylen, T, U, dev)
    valid = valid_cells(xlen, ylen, T, U, dev)
    ninf = -math.inf
    al = torch.full((B, T, U), ninf, dtype=f64, device=dev)
    al[:, 0, 0] = 0.0
    for n in range(1, T + U - 1):
        t, u = _diagonal(n, T, U, dev)
        tp, up = (t - 1).clamp(min=0), (u - 1).clamp(min=0)
        stay = torch.where(t > 0, al[:, tp, u] + lpb[:, tp, u], ninf)
        emit = torch.where(u > 0, al[:, t, up] + lpl[:, t, up], ninf)
        al[:, t, u] = torch.logaddexp(stay, emit)
    bi = torch.arange(B, device=dev)
    has = Tn > 0
    tl, ul = (Tn - 1).clamp(min=0), Un - 1
    ll_fwd = torch.where(has, al[bi, tl, ul] + lpb[bi, tl, ul], ninf)
    al = torch.where(valid, al, math.nan)
    if not need_beta:
        return al, None, ll_fwd, None
    be = torch.full((B, T, U), ninf, dtype=f64, device=dev)
    Tb, Ub = Tn[:, None], Un[:, None]
    for n in range(T + U - 2, -1, -1):
        t, u = _diagonal(n, T, U, dev)
        tn, un = (t + 1).clamp(max=T - 1), (u + 1).clamp(max=U - 1)
        stay = torch.where(t < Tb - 1, be[:, tn, u] + lpb[:, t, u], ninf)
        emit = torch.where(u < Ub - 1, be[:, t, un] + lpl[:, t, u], ninf)
        last = (t == Tb - 1) & (u == Ub - 1)
        be[:, t, u] = torch.where(last, lpb[:, t, u], torch.logaddexp(stay, emit))
    ll_bwd = torch.where(has, be[:, 0, 0], ninf)
    be = torch.where(valid, be, math.nan)
    return al, be, ll_fwd, ll_bwd


def grad_formula(a, b, d, ll, x, labels, xlen, ylen, blank, terms=False):
    """g [B,T,U,V] fp64 from alpha, beta, denom [B,T,U], ll [B] and the logits x [B,T,U,V], zero on padded cells:
        g_v = exp(c_all + x_v) - [v = blank] exp(c_blank + x_v) - [v = label[u]] exp(c_lab + x_v)
        c_all   = a + b - ll + d
        c_blank = a - ll + d + beta(t+1, u) if t < T_b - 1, a - ll + d at the last cell (T_b-1, U_b-1), else no term
        c_lab   = a - ll + d + beta(t, u+1)  if u < U_b - 1
    With terms=True also returns the three exponentials |.| summed per element (main + blank + label terms) and the
    exponents' operand magnitudes, from which a caller bounds the rounding of each term."""
    a, b, d, ll, x = a.to(f64), b.to(f64), d.to(f64), ll.to(f64), x.to(f64)
    B, T, U = a.shape
    dev = a.device
    valid = valid_cells(xlen, ylen, T, U, dev)
    Tn, Un = lengths(xlen, ylen, T, U, dev)
    Tn, Un = Tn[:, None, None], Un[:, None, None]
    ll = ll[:, None, None]
    ninf = torch.full_like(a, -math.inf)
    zero = torch.zeros_like(a)
    c_all = torch.where(valid, a + b - ll + d, ninf)
    main = torch.exp(c_all[..., None] + x)
    g = main.clone()
    t_idx = torch.arange(T, device=dev)[None, :, None]
    u_idx = torch.arange(U, device=dev)[None, None, :]
    b_next_t = torch.cat([b[:, 1:], ninf[:, :1]], dim=1)
    last = (t_idx == Tn - 1) & (u_idx == Un - 1)
    c_blank = torch.where(t_idx < Tn - 1, a - ll + d + b_next_t, torch.where(last, a - ll + d, ninf))
    c_blank = torch.where(valid, c_blank, ninf)
    corr_b = torch.exp(c_blank + x[..., blank])
    g[..., blank] -= corr_b
    # |operands| of each exponent, for the caller's rounding bound
    mag_all = torch.where(valid, a.abs() + b.abs() + ll.abs() + d.abs(), zero)
    mag_b = torch.where(valid, a.abs() + ll.abs() + d.abs() + torch.where(t_idx < Tn - 1, b_next_t.abs(), zero), zero)
    absum = main.clone()
    absum[..., blank] += corr_b
    corr_l = None
    if U > 1:
        lab = torch.as_tensor(labels, device=dev).long()[:, None, :, None].expand(B, T, U - 1, 1)
        b_next_u = torch.cat([b[:, :, 1:], ninf[:, :, :1]], dim=2)
        has_lab = valid & (u_idx < Un - 1)
        c_lab = torch.where(has_lab, a - ll + d + b_next_u, ninf)[:, :, :U - 1]
        xl = torch.gather(x[:, :, :U - 1], 3, lab)
        corr_l = torch.exp(c_lab[..., None] + xl)
        g[:, :, :U - 1].scatter_add_(3, lab, -corr_l)
        absum[:, :, :U - 1].scatter_add_(3, lab, corr_l)
        mag_l = torch.where(has_lab, a.abs() + ll.abs() + d.abs() + b_next_u.abs(), zero)
    g[~valid] = 0
    if not terms:
        return g
    absum[~valid] = 0
    return g, dict(absum=absum, main=main.where(valid[..., None], 0.0), mag_all=mag_all, mag_b=mag_b,
                   corr_b=corr_b.where(valid, 0.0), corr_l=corr_l, mag_l=mag_l if U > 1 else None)
