"""Vectorised fp64 restatements of the pruned RNN-T loss's kernels (csrc/pruned.cu and the band entries of csrc/loss.cu
and csrc/gemm_tc.cu), in torch on any device (TEST INFRASTRUCTURE).  tests/pruned_oracle.py says the same things cell by
cell with autograd; these reach the bench shapes (T' = 500, U+1 = 257, V = 4096) on the device.
tests/test_pruned_restate_host.py pins each function here to pruned_oracle.

simple_lse()    N(t,u) = logsumexp_v(am[t] + lm[u]), chunked over t
simple_grad()   d am, d lm of the trivial joiner's loss, teacher-forced on a loss workspace (the kernel's own)
band_rule()     s_begin and nopath of include/edgedict_b200.h's band rule, scores summed in fp32 in ascending u
live_rows()     the padding rule: which band rows are live, and their cells
band_stats()    denom / lpb / lpl of band rows scattered to their cells, -inf on every other valid cell
band_grad()     d loss / d logits of the band rows from a lattice (loss_restate.grad_formula's branches, per band row)
band_reduce()   dep / ddp of band-row d(pre-activation)

Lengths are clamped as the kernels clamp them: T_b = min(max(xlen, 0), maxT), U_b = min(max(ylen, 0), maxU - 1) + 1."""
import math

import torch

from tests import loss_restate as lr

f64 = torch.float64
NINF = -math.inf


def simple_lse(am, lm, xlen, ylen, max_bytes=1 << 30):
    """N [B, T, U] fp64 on valid cells (NaN elsewhere), from am [B, T, V] and lm [B, U, V]; no temporary over
    max_bytes."""
    am, lm = am.to(f64), lm.to(f64)
    B, T, V = am.shape
    U = lm.shape[1]
    N = torch.full((B, T, U), math.nan, dtype=f64, device=am.device)
    tc = max(1, max_bytes // (8 * U * V))
    for b in range(B):
        for t0 in range(0, T, tc):
            N[b, t0:t0 + tc] = torch.logsumexp(am[b, t0:t0 + tc, None, :] + lm[b, None, :, :], -1)
    return N.where(lr.valid_cells(xlen, ylen, T, U, am.device), math.nan)


def _gamma(a, be, lpb, lpl, ll, Tn, Un):
    """(occ exponent a + be - ll, gamma_blank, gamma_emit) [B, T, U] fp64, zero / -inf off the valid cells."""
    B, T, U = a.shape
    dev = a.device
    t = torch.arange(T, device=dev)[None, :, None]
    u = torch.arange(U, device=dev)[None, None, :]
    Tb, Ub = Tn[:, None, None], Un[:, None, None]
    valid = (t < Tb) & (u < Ub)
    llb = ll[:, None, None]
    be_t = torch.cat([be[:, 1:], torch.full_like(be[:, :1], NINF)], 1)
    be_u = torch.cat([be[:, :, 1:], torch.full_like(be[:, :, :1], NINF)], 2)
    gb = torch.where(t < Tb - 1, torch.exp(a + lpb + be_t - llb),
                     torch.where((t == Tb - 1) & (u == Ub - 1), torch.exp(a + lpb - llb), 0.0))
    ge = torch.where(u < Ub - 1, torch.exp(a + lpl + be_u - llb), 0.0)
    return valid, torch.where(valid, a + be - llb, NINF), torch.where(valid, gb, 0.0), torch.where(valid, ge, 0.0)


def simple_grad(am, lm, labels, xlen, ylen, blank, a, be, d, lpb, lpl, ll, scale, max_bytes=1 << 30):
    """(dam [B,T,V], dlm [B,U,V], sum of |terms| of each) fp64 from the header's formula (eb_rnnt_simple_bwd) on the
    workspace arrays a, be, d, lpb, lpl [B, T, U] and ll [B] (upcast), times scale [B]:
        dam[t,v] = sum_u exp(a + be - ll + d + am[t,v] + lm[u,v]) - [v = blank] sum_u gb - sum_u [v = y_u] ge
    and dlm the same over t.  Zero rows for t >= T_b, u >= U_b and T_b = 0."""
    am, lm = am.to(f64), lm.to(f64)
    a, be, d, lpb, lpl, ll = (x.to(f64) for x in (a, be, d, lpb, lpl, ll))
    B, T, V = am.shape
    U = lm.shape[1]
    dev = am.device
    Tn, Un = lr.lengths(xlen, ylen, T, U, dev)
    valid, occ, gb, ge = _gamma(a, be, lpb, lpl, ll, Tn, Un)
    c_all = torch.where(valid, occ + d, NINF)
    dam = torch.zeros(B, T, V, dtype=f64, device=dev)
    dlm = torch.zeros(B, U, V, dtype=f64, device=dev)
    tc = max(1, max_bytes // (8 * U * V))
    for b in range(B):
        for t0 in range(0, T, tc):
            E = torch.exp(c_all[b, t0:t0 + tc, :, None] + am[b, t0:t0 + tc, None, :] + lm[b, None, :, :])
            dam[b, t0:t0 + tc] += E.sum(1)
            dlm[b] += E.sum(0)
    abs_am, abs_lm = dam.clone(), dlm.clone()
    dam[:, :, blank] -= gb.sum(2)
    dlm[:, :, blank] -= gb.sum(1)
    abs_am[:, :, blank] += gb.sum(2)
    abs_lm[:, :, blank] += gb.sum(1)
    if U > 1:
        lab = torch.as_tensor(labels, device=dev).long()
        gel = ge[:, :, :U - 1]
        dam.scatter_add_(2, lab[:, None, :].expand(B, T, U - 1), -gel)
        abs_am.scatter_add_(2, lab[:, None, :].expand(B, T, U - 1), gel)
        dlm[:, :U - 1].scatter_add_(2, lab[:, :, None], -gel.sum(1)[:, :, None])
        abs_lm[:, :U - 1].scatter_add_(2, lab[:, :, None], gel.sum(1)[:, :, None])
    sc = torch.as_tensor(scale, dtype=f64, device=dev)[:, None, None]
    rows_t = (torch.arange(T, device=dev)[None, :] < Tn[:, None])[..., None]
    rows_u = (torch.arange(U, device=dev)[None, :] < Un[:, None])[..., None] & (Tn > 0)[:, None, None]
    z = torch.zeros((), dtype=f64, device=dev)
    return (torch.where(rows_t, dam * sc, z), torch.where(rows_u, dlm * sc, z),
            torch.where(rows_t, abs_am * sc.abs(), z), torch.where(rows_u, abs_lm * sc.abs(), z))


def band_rule(occ, xlen, ylen, R, occ64=None):
    """(s_begin [B, T] int32, nopath [B] int32, margin [B, T] fp64) of the band rule on the occupancy occ [B, T, U]
    fp32: window scores summed in fp32 in ascending u, argmax with ties to the lowest s, then the two passes.  margin is
    the fp64 score of the chosen window minus the best window whose fp64 score differs from it (inf when there is none:
    windows with equal fp64 scores hold the same nonzero cells, so their fp32 sums tie too), on occ64 (default occ in
    fp64); frames t >= T_b get inf."""
    B, T, U = occ.shape
    dev = occ.device
    occ64 = occ.to(f64) if occ64 is None else occ64.to(f64)
    s_out = torch.zeros(B, T, dtype=torch.int32)
    nop = torch.zeros(B, dtype=torch.int32)
    margin = torch.full((B, T), math.inf, dtype=f64)
    Tn, Un = lr.lengths(xlen, ylen, T, U, "cpu")
    for b in range(B):
        tn, un = int(Tn[b]), int(Un[b])
        if tn == 0:
            continue
        rb = min(R, un)
        S = un - rb
        o = occ[b, :tn, :un].float()
        sc = torch.zeros(tn, S + 1, dtype=torch.float32, device=dev)
        sc64 = torch.zeros(tn, S + 1, dtype=f64, device=dev)
        for k in range(rb):
            sc = sc + o[:, k:k + S + 1]
            sc64 = sc64 + occ64[b, :tn, k:k + S + 1]
        best = torch.zeros(tn, dtype=torch.long, device=dev)
        bs = sc[:, 0].clone()
        for s in range(1, S + 1):
            up = sc[:, s] > bs
            best = torch.where(up, s, best)
            bs = torch.where(up, sc[:, s], bs)
        if S > 0:
            chosen = sc64.gather(1, best[:, None])[:, 0]
            other = sc64.masked_fill(sc64 == chosen[:, None], NINF).max(1).values
            margin[b, :tn] = (chosen - other).cpu()
        s = best.tolist()
        s[0] = 0
        for t in range(1, tn):
            s[t] = min(max(s[t], s[t - 1]), s[t - 1] + rb - 1)
        s[tn - 1] = S
        for t in range(tn - 2, -1, -1):
            s[t] = max(s[t], s[t + 1] - (rb - 1))
        s_out[b, :tn] = torch.tensor(s, dtype=torch.int32)
        nop[b] = int(s[0] > 0)
    return s_out, nop, margin


def live_rows(s_begin, nopath, xlen, ylen, T, U, R, loss=True):
    """(live [B, T, R] bool, u [B, T, R] long) of the padding rule: row r of frame t holds cell u = s_begin[b, t] + r
    when t < T_b, r < min(R, U_b), s_begin >= 0 and u < U_b, and (loss entries) nopath[b] = 0."""
    s = torch.as_tensor(s_begin).long()
    dev = s.device
    Tn, Un = lr.lengths(xlen, ylen, T, U, dev)
    t = torch.arange(T, device=dev)[None, :, None]
    r = torch.arange(R, device=dev)[None, None, :]
    u = s[:, :, None] + r
    Ub = Un[:, None, None]
    live = (t < Tn[:, None, None]) & (r < torch.clamp(Ub, max=R)) & (s[:, :, None] >= 0) & (u < Ub)
    if loss:
        live &= ~torch.as_tensor(nopath, device=dev).bool()[:, None, None]
    return live, u


def _scatter_cells(vals, live, u, U, fill):
    """[B, T, U] with vals [B, T, R] at the live rows' cells, fill elsewhere."""
    B, T, R = vals.shape
    out = torch.full((B, T, U + 1), fill, dtype=vals.dtype, device=vals.device)   # padding rows land in column U
    out.scatter_(2, torch.where(live, u, U), torch.where(live, vals, fill))
    return out[..., :U]


def band_stats(x, labels, xlen, ylen, s_begin, nopath, U, blank):
    """(denom, lpb, lpl [B, T, U] fp64, live [B, T, R]) of band-row logits x [B, T, R, V]: each live row's -logsumexp,
    log p(blank), log p(label[u]) (denom for u = U_b - 1) at its cell, -inf on every other valid cell, NaN off them."""
    x = x.to(f64)
    B, T, R, V = x.shape
    dev = x.device
    live, u = live_rows(torch.as_tensor(s_begin, device=dev), torch.as_tensor(nopath, device=dev), xlen, ylen, T, U,
                        R)
    lse = torch.logsumexp(x, -1)
    d = -lse
    pb = x[..., blank] - lse
    Tn, Un = lr.lengths(xlen, ylen, T, U, dev)
    uu = torch.where(live, u, 0)
    has_lab = live & (u < Un[:, None, None] - 1)
    if U > 1:
        lab = torch.as_tensor(labels, device=dev).long()
        y = lab.gather(1, uu.clamp(max=U - 2).view(B, -1)).view(B, T, R)
        pl = torch.where(has_lab, x.gather(3, y[..., None])[..., 0] - lse, d)
    else:
        pl = d
    valid = lr.valid_cells(xlen, ylen, T, U, dev)
    out = []
    for v in (d, pb, pl):
        c = _scatter_cells(v, live, u, U, NINF)
        out.append(torch.where(valid, c, math.nan))
    return out[0], out[1], out[2], live


def band_grad(a, be, d, ll, x, labels, xlen, ylen, s_begin, nopath, U, blank, scale=None, terms=False):
    """d loss / d logits [B, T, R, V] fp64 of band rows x from a full [B, T, U] lattice (a, be, d, ll [B]): each live
    row gets loss_restate.grad_formula's value for its cell, padding rows 0.  With terms=True also the per-element sum
    of |terms| and the exponents' operand magnitudes (as grad_formula returns them, per band row)."""
    x = x.to(f64)
    a, be, d, ll = a.to(f64), be.to(f64), d.to(f64), ll.to(f64)
    B, T, R, V = x.shape
    dev = x.device
    live, u = live_rows(torch.as_tensor(s_begin, device=dev), torch.as_tensor(nopath, device=dev), xlen, ylen, T, U,
                        R)
    Tn, Un = lr.lengths(xlen, ylen, T, U, dev)
    uu = torch.where(live, u, 0)
    t = torch.arange(T, device=dev)[None, :, None].expand(B, T, R)
    Tb, Ub = Tn[:, None, None], Un[:, None, None]
    g2 = lambda A: A.gather(2, uu)                                    # noqa: E731  [B, T, U] -> [B, T, R]
    be_t = torch.cat([be[:, 1:], torch.full_like(be[:, :1], NINF)], 1)
    be_u = torch.cat([be[:, :, 1:], torch.full_like(be[:, :, :1], NINF)], 2)
    ar, br, dr, btr, bur = g2(a), g2(be), g2(d), g2(be_t), g2(be_u)
    llr = ll[:, None, None]
    ninf = torch.full_like(ar, NINF)
    c_all = torch.where(live, ar + br - llr + dr, ninf)
    last = (t == Tb - 1) & (uu == Ub - 1)
    c_blank = torch.where(live & (t < Tb - 1), ar - llr + dr + btr, torch.where(live & last, ar - llr + dr, ninf))
    has_lab = live & (uu < Ub - 1)
    c_lab = torch.where(has_lab, ar - llr + dr + bur, ninf)
    main = torch.exp(c_all[..., None] + x)
    g = main.clone()
    corr_b = torch.exp(c_blank + x[..., blank])
    g[..., blank] -= corr_b
    absum = main.clone()
    absum[..., blank] += corr_b
    corr_l = torch.zeros_like(ar)
    y = torch.zeros_like(uu)
    if U > 1:
        lab = torch.as_tensor(labels, device=dev).long()
        y = lab.gather(1, uu.clamp(max=U - 2).view(B, -1)).view(B, T, R)
        corr_l = torch.exp(c_lab + x.gather(3, y[..., None])[..., 0])
        g.scatter_add_(3, y[..., None], -corr_l[..., None])
        absum.scatter_add_(3, y[..., None], corr_l[..., None])
    if scale is not None:
        sc = torch.as_tensor(scale, dtype=f64, device=dev)[:, None, None, None]
        g, absum = g * sc, absum * sc.abs()
    g = torch.where(live[..., None], g, 0.0)
    if not terms:
        return g
    z = torch.zeros_like(ar)
    # (an exponent of -inf gives an exact 0 term: magnitude 0)
    mag_all = torch.where(torch.isfinite(c_all), ar.abs() + br.abs() + llr.abs() + dr.abs(), z)
    mag_b = torch.where(torch.isfinite(c_blank), ar.abs() + llr.abs() + dr.abs() + torch.where(t < Tb - 1, btr.abs(), z),
                        z)
    mag_l = torch.where(torch.isfinite(c_lab), ar.abs() + llr.abs() + dr.abs() + bur.abs(), z)
    return g, dict(absum=torch.where(live[..., None], absum, 0.0), main=torch.where(live[..., None], main, 0.0),
                   corr_b=torch.where(live, corr_b, z), corr_l=torch.where(has_lab, corr_l, z), y=y, has_lab=has_lab,
                   mag_all=mag_all, mag_b=mag_b, mag_l=mag_l, live=live)


def band_reduce(dpre, s_begin, xlen, ylen, U):
    """(dep [B, T, J], ddp [B, U, J], |dep| terms, |ddp| terms) fp64 of band-row d(pre-activation) dpre [B, T, R, J]:
    dep sums the live rows of a frame, ddp the live rows that hold cell (t, u) over t (no nopath: the reduction sees
    whatever the gradient wrote there)."""
    dpre = dpre.to(f64)
    B, T, R, J = dpre.shape
    dev = dpre.device
    s = torch.as_tensor(s_begin, device=dev)
    live, u = live_rows(s, torch.zeros(B, dtype=torch.int32, device=dev), xlen, ylen, T, U, R, loss=False)
    x = torch.where(live[..., None], dpre, 0.0)
    dep = x.sum(2)
    adep = x.abs().sum(2)
    idx = (torch.arange(B, device=dev)[:, None, None] * U + torch.where(live, u, 0)).view(-1)
    ddp = torch.zeros(B * U, J, dtype=f64, device=dev).index_add_(0, idx, x.view(-1, J)).view(B, U, J)
    addp = torch.zeros(B * U, J, dtype=f64, device=dev).index_add_(0, idx, x.abs().view(-1, J)).view(B, U, J)
    return dep, ddp, adep, addp
