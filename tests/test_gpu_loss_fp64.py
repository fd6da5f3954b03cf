"""Kernel-level fp64 parity of the fp32 / fp64 RNN-T loss of csrc/loss.cu, the path of the fp32-mode training step,
the bf16 fallback, warprnnt_pytorch.RNNTLoss, the compute_rnnt_loss[_fp64] C ABI and forced alignment:

    rnnt_denom_kernel    denom = -logsumexp, lpb = log p(blank), lpl = log p(label[u]) per valid cell (4-wide VEC
                         variant, and the scalar one for V % 4 != 0 or logits not 16-byte aligned)
    rnnt_lattice_kernel  alpha / beta wavefronts, ll_fwd / ll_bwd (PF = 8 ring; the wide kernel with a shallower ring
                         for blocks the PF = 8 kernel cannot launch: U+1 > 896 in fp32, > 544 in fp64 on sm_90a)
    rnnt_grad_kernel     d loss / d logits: fp32 out (VEC / scalar), bf16 out from fp32 logits (VEC / scalar), fp64 out

The C entries are called directly, into NaN-prefilled workspaces and outputs.  References are fp64: torch on the device
for the statistics, tests/loss_restate.py (pinned to the C oracle by tests/test_loss_host.py) for the lattice and the
gradient formula, teacher-forced on the kernel's own inputs, and oracle.loss for end-to-end costs and gradients.  Every
bar comes from the error model in its test's docstring; every measured figure is printed next to its bar (pytest -s).
eps is the unit roundoff of the compute type: 2^-24 (fp32), 2^-53 (fp64).

The shape matrix (CASES) names the code path each case reaches.  The file runs in about 30 s on an H100."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import loss as ol
from tests import loss_restate as lr

pytestmark = pytest.mark.gpu

f32, f64, bf16 = torch.float32, torch.float64, torch.bfloat16
NAN = float("nan")
EPS = {f32: 2.0 ** -24, f64: 2.0 ** -53}
# relative error of the exponential the statistics / main gradient term use: ex2.approx.ftz (2^-22) in fp32, exp
# (1 ulp) in fp64; and of the accurate expf / exp of the corrections (2 ulp / 1 ulp)
EXP_FAST = {f32: 2.0 ** -22, f64: 2.0 ** -52}
EXP_ACC = {f32: 2.0 ** -23, f64: 2.0 ** -52}
# largest exponent error bound (delta_lat) at which the end-to-end gradient bar still constrains the gradient: each term
# within 6.5 % of its value, so a dropped correction or a wrong scale still exceeds it
E2E_GRAD_MAX_DELTA = 2.0 ** -4

# name: (B, T, U, V, blank, xlen, ylen, dtype, offset)   offset: logits start one element past a 16-byte boundary
CASES = {
    # statistics and gradient: VEC variant, V = 1024 (8 chunks per lane), ragged with xlen = 1 and ylen = 0
    "f32_v1024_vec": (3, 20, 9, 1024, 0, [20, 11, 1], [8, 3, 0], f32, 0),
    # VEC, V % 128 != 0 (lanes with one chunk fewer), blank = V - 1
    "f32_v1000_blank_last": (2, 13, 7, 1000, 999, [13, 6], [6, 2], f32, 0),
    # VEC, V < 128: idle lanes; blank in the middle
    "f32_v72_blank_mid": (3, 11, 6, 72, 35, [11, 11, 4], [5, 0, 5], f32, 0),
    # scalar variant by V % 4 != 0: masked tail of the last chunk
    "f32_v29_scalar": (2, 9, 8, 29, 5, [9, 7], [7, 4], f32, 0),
    # scalar variant by alignment: V % 4 == 0 but logits (and gradients) 4 bytes past a 16-byte boundary
    "f32_v256_offset_scalar": (2, 10, 6, 256, 128, [10, 8], [5, 5], f32, 1),
    # maxU = 1 with labels = NULL
    "f32_v200_maxU1": (2, 17, 1, 200, 199, [17, 9], [0, 0], f32, 0),
    # lattice: anti-diagonal counts 39 / 40 / 41 around the PF = 8 ring, a T = 1 utterance with ylen = 0
    "f32_u32_ring": (4, 10, 32, 6, 1, [10, 9, 8, 1], [31, 31, 31, 0], f32, 0),
    "f32_u33": (3, 9, 33, 4, 3, [9, 8, 7], [32, 32, 5], f32, 0),
    # the widest block of the PF = 8 kernel in fp32 (896 threads), diagonal counts 913 / 912 / 911 and 105; the first
    # block of the wide kernel (PF = 4), 913 / 912 / 911 and 304; the widest, 1041 / 1040 / 1039 and 1 (T = 1, ylen = 0)
    "f32_u896": (4, 18, 896, 3, 0, [18, 17, 16, 5], [895, 895, 895, 100], f32, 0),
    "f32_u897_wide": (4, 17, 897, 3, 0, [17, 16, 15, 4], [896, 896, 896, 300], f32, 0),
    "f32_u1024_wide": (4, 18, 1024, 3, 2, [18, 17, 16, 1], [1023, 1023, 1023, 0], f32, 0),
    # T = 1 for every utterance
    "f32_t1": (2, 1, 6, 7, 3, [1, 1], [5, 0], f32, 0),
    # T' = 4000 at small U: the accumulation bar over 4000 diagonals
    "f32_t4000": (2, 4000, 3, 5, 4, [4000, 3999], [2, 1], f32, 0),
    # fp64: VEC, scalar by V % 4, scalar by alignment (8 bytes past), idle lanes
    "f64_v1024_vec": (3, 12, 7, 1024, 511, [12, 5, 1], [6, 6, 0], f64, 0),
    "f64_v29_scalar": (2, 9, 5, 29, 28, [9, 4], [4, 1], f64, 0),
    "f64_v136_offset_scalar": (2, 8, 5, 136, 0, [8, 6], [4, 3], f64, 1),
    "f64_v72_maxU1": (2, 9, 1, 72, 7, [9, 3], [0, 0], f64, 0),
    # fp64 lattice: the widest PF = 8 block (544 threads), diagonal counts 553 / 552 / 551 and 13; the first block of
    # the wide kernel (PF = 2), 553 / 552 / 551 and 203; the widest, 1032 / 1031 and 1 (T = 1, ylen = 0)
    "f64_u544": (4, 10, 544, 3, 1, [10, 9, 8, 3], [543, 543, 543, 10], f64, 0),
    "f64_u545_wide": (4, 9, 545, 3, 1, [9, 8, 7, 3], [544, 544, 544, 200], f64, 0),
    "f64_u1024_wide": (3, 9, 1024, 3, 0, [9, 8, 1], [1023, 1023, 0], f64, 0),
    "f64_t1000": (2, 1000, 4, 5, 2, [1000, 999], [3, 2], f64, 0),
}


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _buffer(shape, dtype, offset, fill=NAN):
    """A tensor of `shape` starting `offset` elements into a fresh allocation (offset 1: not 16-byte aligned)."""
    n = int(np.prod(shape))
    buf = torch.full((n + offset,), fill, dtype=dtype, device="cuda")
    return buf[offset:].view(shape)


def _make_case(name):
    B, T, U, V, blank, xl, yl, dt, off = CASES[name]
    seed = sum(map(ord, name))
    rng = np.random.RandomState(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = _buffer((B, T, U, V), dt, off)
    X.copy_(torch.randn(B, T, U, V, device="cuda", generator=g, dtype=f64) * 3)   # |X| up to ~15
    lab = lr.planted_labels(rng, B, U, V, blank)
    xlen, ylen = np.asarray(xl, np.int32), np.asarray(yl, np.int32)
    valid = lr.valid_cells(xlen, ylen, T, U, "cuda")
    return dict(name=name, B=B, T=T, U=U, V=V, blank=blank, dt=dt, off=off, X=X, lab=lab, xlen=xlen, ylen=ylen,
                valid=valid, lab_d=torch.as_tensor(lab, device="cuda") if U > 1 else None,
                xlen_d=torch.as_tensor(xlen, device="cuda"), ylen_d=torch.as_tensor(ylen, device="cuda"))


def _ws(c):
    ds = 8 if c["dt"] == f64 else 4
    n = _lib().eb_rnnt_workspace_bytes(c["B"], c["T"], c["U"], ds) // ds
    return torch.full((n,), NAN, dtype=c["dt"], device="cuda")


def _views(c, ws):
    B, n = c["B"], c["B"] * c["T"] * c["U"]
    sh = (B, c["T"], c["U"])
    return dict(denom=ws[:n].view(sh), lpb=ws[n:2 * n].view(sh), lpl=ws[2 * n:3 * n].view(sh),
                alphas=ws[3 * n:4 * n].view(sh), betas=ws[4 * n:5 * n].view(sh),
                ll_fwd=ws[5 * n:5 * n + B], ll_bwd=ws[5 * n + B:5 * n + 2 * B])


def _fwd(c, X=None, ws=None, need_beta=1, xlen=None, ylen=None):
    X = c["X"] if X is None else X
    ws = _ws(c) if ws is None else ws
    costs = torch.full((c["B"],), NAN, dtype=c["dt"], device="cuda")
    rc = _lib().eb_rnnt_loss_fwd(_p(X), _p(c["lab_d"]), _p(c["xlen_d"] if xlen is None else xlen),
                                 _p(c["ylen_d"] if ylen is None else ylen), c["B"], c["T"], c["U"], c["V"],
                                 c["blank"], 8 if c["dt"] == f64 else 4, _p(ws), _p(costs), need_beta, _stream())
    assert rc == 0, rc
    return costs, ws


def _bwd(c, ws, out, X=None, gscale=None, host_scale=1.0, xlen=None, ylen=None):
    X = c["X"] if X is None else X
    per_batch = int(gscale is not None and gscale.numel() > 1)
    rc = _lib().eb_rnnt_loss_bwd(_p(X), _p(out), int(out.dtype == bf16), _p(c["lab_d"]),
                                 _p(c["xlen_d"] if xlen is None else xlen), _p(c["ylen_d"] if ylen is None else ylen),
                                 c["B"], c["T"], c["U"], c["V"], c["blank"], 8 if c["dt"] == f64 else 4, _p(ws),
                                 _p(gscale), per_batch, float(host_scale), _stream())
    assert rc == 0, rc
    return out


def _out(c, dtype=None):
    return _buffer(tuple(c["X"].shape), dtype or c["dt"], c["off"])


def _gather_lab(c, A):
    """A[b, t, u, label[b, u]] for u < U-1, [B, T, U] with the last column 0."""
    B, T, U = c["B"], c["T"], c["U"]
    out = torch.zeros(B, T, U, dtype=A.dtype, device="cuda")
    if U > 1:
        idx = c["lab_d"].long()[:, None, :, None].expand(B, T, U - 1, 1)
        out[:, :, :U - 1] = torch.gather(A[:, :, :U - 1], 3, idx)[..., 0]
    return out


def _stat_bar(c, X):
    """Per-cell bar of denom (see test_statistics); X fp64 [B,T,U,V]."""
    dt, V = c["dt"], c["V"]
    eps = EPS[dt]
    m = X.max(-1).values
    lse = torch.logsumexp(X, -1)
    R = (torch.softmax(X, -1) * (m[..., None] - X)).sum(-1)
    spread = m - X.min(-1).values
    chunks = -(-V // 128)
    return ((1 + chunks) * EXP_FAST[dt] + eps * (3 * R + 3 * spread + 2 * chunks + 16 + 2 * math.log(V) + lse.abs()),
            lse)


def _lattice_bar(c, ref, forward, M):
    """(steps + 1) eps (3 M_b + 6) per cell: steps = t + u (alphas) or the steps to the last cell (betas)."""
    B, T, U = c["B"], c["T"], c["U"]
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], T, U, "cuda")
    t = torch.arange(T, device="cuda")[None, :, None]
    u = torch.arange(U, device="cuda")[None, None, :]
    steps = (t + u) if forward else (Tn[:, None, None] - 1 - t) + (Un[:, None, None] - 1 - u)
    return (steps + 1).double() * EPS[c["dt"]] * (3 * M[:, None, None] + 6)


def _e2e_bars(c, x, smax):
    """(per-utterance cost bar, bound on the error of an exponent of the gradient) of the chain on the fp64 logits x,
    with smax the largest bar of a log-prob: the lattice's bar of (b) at M from the exact fp64 lattice, plus smax for
    each of the T_b + U_b - 1 log-probs of a path (the lattice passes input errors on as a weighted mean)."""
    lse = torch.logsumexp(x, -1)
    al, be, _, _ = lr.lattice(x[..., c["blank"]] - lse, _gather_lab(c, x) - lse, c["xlen_d"], c["ylen_d"])
    M = torch.maximum(al.nan_to_num(0).abs().amax((1, 2)), be.nan_to_num(0).abs().amax((1, 2)))
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], c["T"], c["U"], "cuda")
    bar_c = (Tn + Un).double() * (EPS[c["dt"]] * (3 * M + 6) + smax)
    # an exponent a + b - ll + d: three lattice values and one statistic
    return bar_c, 3 * float(bar_c.max()) + smax


def _smax(c, x, valid):
    bar_s, lse = _stat_bar(c, x)
    return float((bar_s + EPS[c["dt"]] * (x.abs().amax(-1) + lse.abs()))[valid].max())


def _ratio(err, bar, mask=None):
    r = err / bar
    if mask is not None:
        r = r[mask]
    return float(r.max()) if r.numel() else 0.0


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    c = _make_case(request.param)
    costs, ws = _fwd(c)
    c["costs"], c["ws"] = costs, ws
    torch.cuda.synchronize()
    return c


def test_statistics(case):
    """(a) denom, lpb, lpl of rnnt_denom_kernel against log_softmax of the logits in fp64, per valid cell.

    Error model, per row: each lane sums exp(x - m) of its 4-wide chunks with a running max.  A term's relative error
    is the exponential's (EXP_FAST) plus the rounding of x - m and of its scaling to base 2, 2 eps |x - m|, so the
    sum's is EXP_FAST + 3 eps R, R = sum_v p_v (max - x_v); each of the <= ceil(V/128) rescalings by exp(m - m') adds
    EXP_FAST + eps |m - m'| (together <= chunks EXP_FAST + eps spread, spread = max - min), and the additions of the
    lane and of the warp reduction add eps each (2 chunks + 8).  log s is good to 2 eps log V + 1 ulp; -m - log s
    rounds once (eps |denom|).  Bar on denom:
        (1 + chunks) EXP_FAST + eps (3 R + 3 spread + 2 chunks + 16 + 2 log V + |denom|),
    and on lpb / lpl = denom + x one rounding more: + eps |lp|.  A masked tail counted as exp(0 - m), a blank or
    label taken from the wrong column, or a lane's chunk dropped exceed it by orders of magnitude.
    Padded cells stay NaN, and the lattice part of the workspace is written only where (b) says."""
    c = case
    X = c["X"].double()
    valid = c["valid"]
    w = _views(c, c["ws"])
    bar_d, lse = _stat_bar(c, X)
    eps = EPS[c["dt"]]
    ref_b = X[..., c["blank"]] - lse
    ref_l = _gather_lab(c, X) - lse
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], c["T"], c["U"], "cuda")
    has_lab = valid & (torch.arange(c["U"], device="cuda")[None, None, :] < Un[:, None, None] - 1)
    r_d = _ratio((w["denom"].double() + lse).abs(), bar_d, valid)
    r_b = _ratio((w["lpb"].double() - ref_b).abs(), bar_d + eps * ref_b.abs(), valid)
    r_l = _ratio((w["lpl"].double() - ref_l).abs(), bar_d + eps * ref_l.abs(), has_lab)
    print("%s: denom err/bar %.3f, lpb %.3f, lpl %.3f (bar at |denom| max: %.1e)"
          % (c["name"], r_d, r_b, r_l, float(bar_d[valid].max())))
    assert r_d <= 1 and r_b <= 1 and r_l <= 1, (r_d, r_b, r_l)
    for k in ("denom", "lpb", "lpl"):
        assert bool(w[k][~valid].isnan().all()), k
    assert not bool(w["lpl"][has_lab].isnan().any())


def test_lattice_teacher_forced(case):
    """(b) alphas, betas, ll_fwd, ll_bwd against the fp64 lattice (loss_restate.lattice) on the kernel's own lpb / lpl.

    Error model: a cell is lse2(emit, stay) of two sums pred + lp.  Each addition rounds (eps |.|, and a term's rounding
    reaches the result weighted by its share exp(term - result), so by eps (|result| + 1/e)); expf / log1pf (fp32, 2 ulp
    each) or exp / log1p (fp64) add <= 4 eps absolute; the final addition eps |result|.  lse2 passes its inputs' errors
    on as a weighted mean, so errors add along the path: after n steps <= n eps (3 M + 5), M the largest |alpha| or
    |beta| of the utterance.  Bar per cell: (n + 1) eps (3 M + 6), n = t + u for alphas, the steps to (T_b-1, U_b-1)
    for betas; ll_fwd and ll_bwd with n = T_b + U_b - 1.  A broken prefetch carry, a lost __syncthreads or a wrong
    diagonal buffer exceed it at once.  Padded cells stay NaN.  need_beta = 0 gives the same cost bits and leaves betas
    and ll_bwd NaN."""
    c = case
    w = _views(c, c["ws"])
    al, be, llf, llb = lr.lattice(w["lpb"], w["lpl"], c["xlen_d"], c["ylen_d"])
    valid = c["valid"]
    M = torch.maximum(al.nan_to_num(0).abs().amax((1, 2)), be.nan_to_num(0).abs().amax((1, 2)))
    r_a = _ratio((w["alphas"].double() - al).abs(), _lattice_bar(c, al, True, M), valid)
    r_be = _ratio((w["betas"].double() - be).abs(), _lattice_bar(c, be, False, M), valid)
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], c["T"], c["U"], "cuda")
    bar_ll = (Tn + Un).double() * EPS[c["dt"]] * (3 * M + 6)
    r_f = float(((w["ll_fwd"].double() - llf).abs() / bar_ll).max())
    r_bw = float(((w["ll_bwd"].double() - llb).abs() / bar_ll).max())
    print("%s: alphas err/bar %.3f, betas %.3f, ll_fwd %.3f, ll_bwd %.3f (M %.1f, ll bar %.1e)"
          % (c["name"], r_a, r_be, r_f, r_bw, float(M.max()), float(bar_ll.max())))
    assert r_a <= 1 and r_be <= 1 and r_f <= 1 and r_bw <= 1, (r_a, r_be, r_f, r_bw)
    for k in ("alphas", "betas"):
        assert bool(w[k][~valid].isnan().all()), k
    assert torch.equal(c["costs"], -w["ll_fwd"])
    costs_nb, ws_nb = _fwd(c, need_beta=0)
    v = _views(c, ws_nb)
    bits = torch.int64 if c["dt"] == f64 else torch.int32
    assert torch.equal(costs_nb.view(bits), c["costs"].view(bits))
    assert torch.equal(v["alphas"].view(bits), w["alphas"].view(bits))
    assert bool(v["betas"].isnan().all()) and bool(v["ll_bwd"].isnan().all())


def _grad_bar(c, terms, x, sc, out_dtype):
    """Per-element bar of the gradient (see test_gradient_teacher_forced)."""
    dt = c["dt"]
    eps = EPS[dt]
    blank, B, T, U = c["blank"], c["B"], c["T"], c["U"]
    ax = x.abs()
    bar = terms["main"] * (EXP_FAST[dt] + eps * (5 * terms["mag_all"][..., None] + 2 * ax))
    bar[..., blank] += terms["corr_b"] * (EXP_ACC[dt] + eps * (5 * terms["mag_b"] + 2 * ax[..., blank]))
    if U > 1:
        lab = c["lab_d"].long()[:, None, :, None].expand(B, T, U - 1, 1)
        xl = torch.gather(ax[:, :, :U - 1], 3, lab)
        e = terms["corr_l"] * (EXP_ACC[dt] + eps * (5 * terms["mag_l"][:, :, :U - 1, None] + 2 * xl))
        bar[:, :, :U - 1].scatter_add_(3, lab, e)
    bar = (bar + 2 * eps * terms["absum"]) * sc.abs()
    return bar


def _check_grad(c, g, ref, bar, out_dtype, tag):
    valid = c["valid"]
    eps = EPS[c["dt"]]
    tiny = 2.0 ** -120 if c["dt"] == f32 else 2.0 ** -1000       # flush-to-zero of the fp32 exponentials
    bar = bar + eps * ref.abs() + tiny
    if out_dtype == bf16:
        bar = bar + 2.0 ** -8 * (ref.abs() + bar)               # one rounding to 8 significant bits
    err = (g.double() - ref).abs()
    r = _ratio(err, bar, valid)
    print("%s [%s]: grad err/bar %.3f" % (c["name"], tag, r))
    assert r <= 1, (tag, r)
    assert bool((g[~valid] == 0).all()) and not bool(g.isnan().any()), tag


def test_gradient_teacher_forced(case):
    """(c) rnnt_grad_kernel on the kernel's own workspace against grad_formula (loss_restate) in fp64.

    Error model: the exponent c_all + x = a + b - ll + d + x is summed in the compute type: each of its four additions
    rounds by eps times a partial sum, <= eps (|a| + |b| + |ll| + |d| + |x|) each, plus the scaling to base 2 of
    ex2.approx (eps |c_all + x|): relative error of the main term <= EXP_FAST + eps (5 mag + 2 |x|), mag = |a| + |b|
    + |ll| + |d|; the blank and label corrections likewise with the accurate exponential (EXP_ACC) and their own
    operands.  The two subtractions and the scaling round by eps |.|.  Bar per element:
        |sc| (sum over the row's terms of |term| delta_term + 2 eps sum |term|) + eps |ref|
    (plus 2^-8 (|ref| + bar) for bf16 output, 2^-120 for fp32 flush-to-zero).  A dropped or misplaced correction, a
    correction on a cell without one (small occupancy included: the bar scales with the terms of that element), or a
    scale of the wrong utterance exceed it.
    Variants: output in the compute type (VEC or scalar as the case selects), bf16 output from fp32 logits, scales
    gscale None / [1] / [B] with mixed signs times host_scale.  In place and out of place give the same bits; padded
    cells are exactly 0; nothing is NaN."""
    c = case
    B, dt = c["B"], c["dt"]
    w = _views(c, c["ws"])
    x = c["X"].double()
    ref, terms = lr.grad_formula(w["alphas"], w["betas"], w["denom"], w["ll_fwd"], x, c["lab"], c["xlen_d"],
                                 c["ylen_d"], c["blank"], terms=True)
    signs = torch.tensor([(-1.5) ** (b + 1) for b in range(B)], dtype=dt, device="cuda")
    variants = [("1", None, 1.0), ("host 0.37, gscale[1] = -1.5", torch.tensor([-1.5], dtype=dt, device="cuda"), 0.37),
                ("host 0.25, gscale[B] mixed signs", signs, 0.25), ("host 1, gscale[B] mixed signs", signs, 1.0)]
    outs = [dt] + ([bf16] if dt == f32 else [])
    for od in outs:
        for tag, gs, hs in variants:
            g = _bwd(c, c["ws"], _out(c, od), gscale=gs, host_scale=hs)
            # the kernel's scale: host_scale * gscale[b or 0] in the compute type
            gsv = gs if gs is not None else torch.ones(1, dtype=dt, device="cuda")
            sc = (torch.tensor(hs, dtype=dt, device="cuda") * gsv).double().expand(B)[:, None, None, None]
            _check_grad(c, g, ref * sc, _grad_bar(c, terms, x, sc, od), od, "%s out, %s" % (od, tag))
    # in place over a copy of the logits: the same bits as out of place
    g = _bwd(c, c["ws"], _out(c))
    xi = _buffer(tuple(c["X"].shape), dt, c["off"])
    xi.copy_(c["X"])
    _bwd(c, c["ws"], xi, X=xi)
    bits = torch.int64 if dt == f64 else torch.int32
    assert torch.equal(g.view(bits), xi.view(bits)), "in place and out of place differ"


def test_end_to_end_against_oracle(case):
    """(c, d) Costs and gradient of the chain against oracle.loss.logits in fp64.

    Error model: the cost carries the lattice's error (bar of b with the true M) plus the statistics' on each of the
    T_b + U_b - 1 log-probs of a path (bar of a).  Each exponent of the gradient carries, on top of (c)'s rounding, the
    errors of alpha, beta, ll and denom, together at most delta_lat (their bars' maxima), so each term is off by a
    factor within exp(+-delta_lat): bar_e2e = bar_c + sum |term| expm1(delta_lat).  That bounds anything only while
    delta_lat is small; the gradient is asserted end to end where delta_lat <= E2E_GRAD_MAX_DELTA and printed otherwise
    (the wide and long fp32 cases, where |alpha|, |beta| reach the hundreds).  (c) checks every case's gradient
    teacher-forced."""
    c = case
    x = c["X"].double()
    costs_o, g_o = ol.logits(x.cpu().numpy(), c["lab"], c["xlen"], c["ylen"], blank=c["blank"], dtype=np.float64)
    costs_o, g_o = torch.as_tensor(costs_o, device="cuda"), torch.as_tensor(g_o, device="cuda")
    bar_c, delta_lat = _e2e_bars(c, x, _smax(c, x, c["valid"]))
    r_c = float(((c["costs"].double() - costs_o).abs() / bar_c).max())
    print("%s: costs err/bar %.3f (bar %.1e)" % (c["name"], r_c, float(bar_c.max())))
    assert r_c <= 1, r_c
    w = _views(c, c["ws"])
    ref, terms = lr.grad_formula(w["alphas"], w["betas"], w["denom"], w["ll_fwd"], x, c["lab"], c["xlen_d"],
                                 c["ylen_d"], c["blank"], terms=True)
    one = torch.ones(c["B"], 1, 1, 1, dtype=f64, device="cuda")
    g = _bwd(c, c["ws"], _out(c))
    bar = _grad_bar(c, terms, x, one, c["dt"]) + terms["absum"] * math.expm1(delta_lat)
    if delta_lat <= E2E_GRAD_MAX_DELTA:
        _check_grad(c, g, g_o, bar, c["dt"], "end to end vs oracle, delta_lat %.1e" % delta_lat)
    else:
        r = _ratio((g.double() - g_o).abs(), bar + EPS[c["dt"]] * g_o.abs(), c["valid"])
        print("%s [end to end vs oracle]: not asserted, delta_lat %.2f; err/bar %.3f" % (c["name"], delta_lat, r))


def test_repeatable_bits(case):
    """(f) A second forward and backward on the same inputs gives the same bits: costs, the whole workspace (with its
    untouched NaN prefill) and the gradient."""
    c = case
    costs, ws = _fwd(c)
    bits = torch.int64 if c["dt"] == f64 else torch.int32
    assert torch.equal(costs.view(bits), c["costs"].view(bits))
    assert torch.equal(ws.view(bits), c["ws"].view(bits))
    g1 = _bwd(c, c["ws"], _out(c, c["dt"]))
    g2 = _bwd(c, ws, _out(c, c["dt"]))
    assert torch.equal(g1.view(bits), g2.view(bits))


# ---- (d) warp-transducer compatible C ABI ----------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [f32, f64])
def test_compat_abi_ragged_blank_not_zero(dt):
    """(d) compute_rnnt_loss / compute_rnnt_loss_fp64 on a ragged problem with blank != 0 (35 of 72, 28 of 29) against
    oracle.loss.logits in fp64, with the bars of test_end_to_end_against_oracle for its own statistics (costs) and
    the same bits as eb_rnnt_loss_fwd / _bwd (whose gradient test_end_to_end_against_oracle checks on this case).  A
    forward-only call leaves the poisoned gradient buffer untouched."""
    c = _make_case("f32_v72_blank_mid" if dt == f32 else "f64_v29_scalar")
    B, T, U, V = c["X"].shape
    L = _lib()
    sz = C.c_size_t(0)
    assert L.get_workspace_size(T, U, B, True, C.byref(sz), c["X"].element_size()) == 0
    ws = torch.full((sz.value,), 255, dtype=torch.uint8, device="cuda")
    fn = L.compute_rnnt_loss if dt == f32 else L.compute_rnnt_loss_fp64
    npdt = np.float32 if dt == f32 else np.float64
    opt = ol.RnntOptions(loc=1, num_threads=0, stream=_stream(), blank_label=c["blank"], maxT=T, maxU=U,
                         batch_first=True)
    x = c["X"].double()
    costs_o, _ = ol.logits(x.cpu().numpy(), c["lab"], c["xlen"], c["ylen"], blank=c["blank"], want_grads=False,
                           dtype=np.float64)
    bar_c, _ = _e2e_bars(c, x, _smax(c, x, c["valid"]))
    bar_c = bar_c.cpu().numpy()
    for want in (True, False):
        grads = torch.full_like(c["X"], 7.0)
        costs = np.full(B, np.nan, npdt)
        st = fn(C.c_void_p(_p(c["X"])), C.c_void_p(_p(grads)) if want else None, C.c_void_p(_p(c["lab_d"])),
                C.c_void_p(_p(c["ylen_d"])), C.c_void_p(_p(c["xlen_d"])), V, B, costs.ctypes.data_as(C.c_void_p),
                C.c_void_p(ws.data_ptr()), opt)
        assert st == 0, st
        torch.cuda.synchronize()
        ref_costs, ws_ref = _fwd(c)
        assert np.array_equal(costs, ref_costs.cpu().numpy()), (costs, ref_costs)   # the same kernels, same bits
        r = float(np.max(np.abs(costs - costs_o) / bar_c))
        print("compat %s want_grads=%d: costs err/bar %.3f" % (dt, want, r))
        assert r <= 1, r
        if want:
            g_ref = _bwd(c, ws_ref, _out(c))
            bits = torch.int64 if dt == f64 else torch.int32
            assert torch.equal(grads.view(bits), g_ref.view(bits))
        else:
            assert bool((grads == 7.0).all())


# ---- (e) production shape ------------------------------------------------------------------------------------------
def test_production_shape_against_fp64():
    """(e) B=32, T'=500, U+1=129, V=1024 fp32 (the workload of the fp32-mode training step) against fp64 on the device,
    one utterance at a time where the fp64 copies are large (0.5 GB per utterance):
      - statistics per valid cell against log_softmax of the logits in fp64, the bar of test_statistics;
      - alphas, betas, ll_fwd, ll_bwd teacher-forced on the kernel's own lpb / lpl, the bar of
        test_lattice_teacher_forced;
      - the gradient (gscale = [1], host_scale = 1/B, as JointLoss runs it) teacher-forced on the kernel's own workspace,
        the bar of test_gradient_teacher_forced;
      - costs end to end against the fp64 lattice of the fp64 log-probs, the cost bar of test_end_to_end_against_oracle.
    The gradient is not compared end to end here: with |alpha|, |beta| in the thousands, the fp32 lattice's own bar
    (about 0.5 on an exponent) leaves no useful bound on exp(exponent)."""
    B, T, U, V, blank = 32, 500, 129, 1024, 0
    g = torch.Generator(device="cuda").manual_seed(1)
    X = torch.randn(B, T, U, V, device="cuda", generator=g)
    lab = torch.randint(1, V, (B, U - 1), device="cuda", dtype=torch.int32, generator=g)
    xl = torch.randint(T // 2, T + 1, (B,), device="cuda", dtype=torch.int32, generator=g)
    yl = torch.randint(U // 2, U, (B,), device="cuda", dtype=torch.int32, generator=g)
    xl[0], yl[0] = T, U - 1
    valid = lr.valid_cells(xl, yl, T, U, "cuda")
    c = dict(name="production", B=B, T=T, U=U, V=V, blank=blank, dt=f32, off=0, X=X, lab=lab.cpu().numpy(),
             xlen=xl.cpu().numpy(), ylen=yl.cpu().numpy(), lab_d=lab, xlen_d=xl, ylen_d=yl, valid=valid)
    costs, ws = _fwd(c)
    grads = _bwd(c, ws, torch.empty_like(X), gscale=torch.ones(1, device="cuda"), host_scale=1.0 / B)
    w = _views(c, ws)
    Tn, Un = lr.lengths(xl, yl, T, U, "cuda")
    has_lab = valid & (torch.arange(U, device="cuda")[None, None, :] < Un[:, None, None] - 1)
    eps = EPS[f32]

    def one(b, **kw):
        return dict(c, B=1, lab=c["lab"][b:b + 1], lab_d=lab[b:b + 1], xlen=c["xlen"][b:b + 1],
                    ylen=c["ylen"][b:b + 1], xlen_d=xl[b:b + 1], ylen_d=yl[b:b + 1], valid=valid[b:b + 1], **kw)

    # statistics against fp64, and the exact fp64 log-probs for the end-to-end costs
    lpb, lpl = torch.empty(B, T, U, dtype=f64, device="cuda"), torch.empty(B, T, U, dtype=f64, device="cuda")
    r_s, smax = 0.0, 0.0
    for b in range(B):
        cb, x = one(b), X[b:b + 1].double()
        bar_d, lse = _stat_bar(cb, x)
        ref_b, ref_l = x[..., blank] - lse, _gather_lab(cb, x) - lse
        vb, lb = valid[b:b + 1], has_lab[b:b + 1]
        r_s = max(r_s, _ratio((w["denom"][b:b + 1].double() + lse).abs(), bar_d, vb),
                  _ratio((w["lpb"][b:b + 1].double() - ref_b).abs(), bar_d + eps * ref_b.abs(), vb),
                  _ratio((w["lpl"][b:b + 1].double() - ref_l).abs(), bar_d + eps * ref_l.abs(), lb))
        smax = max(smax, _smax(cb, x, vb))
        lpb[b], lpl[b] = ref_b[0], ref_l[0]
        del x, bar_d, lse, ref_b, ref_l
    # lattice teacher-forced on the kernel's own log-probs
    al, be, llf, llb = lr.lattice(w["lpb"], w["lpl"], xl, yl)
    M = torch.maximum(al.nan_to_num(0).abs().amax((1, 2)), be.nan_to_num(0).abs().amax((1, 2)))
    r_a = _ratio((w["alphas"].double() - al).abs(), _lattice_bar(c, al, True, M), valid)
    r_be = _ratio((w["betas"].double() - be).abs(), _lattice_bar(c, be, False, M), valid)
    bar_ll = (Tn + Un).double() * eps * (3 * M + 6)
    r_ll = max(float(((w["ll_fwd"].double() - llf).abs() / bar_ll).max()),
               float(((w["ll_bwd"].double() - llb).abs() / bar_ll).max()))
    del al, be
    # costs end to end: the fp64 lattice of the fp64 log-probs
    al, be, llf64, _ = lr.lattice(lpb, lpl, xl, yl)
    M64 = torch.maximum(al.nan_to_num(0).abs().amax((1, 2)), be.nan_to_num(0).abs().amax((1, 2)))
    del al, be, lpb, lpl
    bar_c = (Tn + Un).double() * (eps * (3 * M64 + 6) + smax)              # as _e2e_bars
    r_c = float(((costs.double() + llf64).abs() / bar_c).max())
    # gradient teacher-forced on the kernel's own workspace
    r_g = 0.0
    sc = torch.full((1, 1, 1, 1), 1.0 / B, dtype=f64, device="cuda")       # host_scale * gscale[0], exact in fp32
    for b in range(B):
        cb, x = one(b), X[b:b + 1].double()
        ref, terms = lr.grad_formula(w["alphas"][b:b + 1], w["betas"][b:b + 1], w["denom"][b:b + 1],
                                     w["ll_fwd"][b:b + 1], x, cb["lab"], cb["xlen_d"], cb["ylen_d"], blank, terms=True)
        ref = ref * sc
        bar = _grad_bar(cb, terms, x, sc, f32) + eps * ref.abs() + 2.0 ** -120
        r_g = max(r_g, _ratio((grads[b:b + 1].double() - ref).abs(), bar, valid[b:b + 1]))
        assert bool((grads[b:b + 1][~valid[b:b + 1]] == 0).all())
        del x, ref, terms, bar
    print("production: statistics err/bar %.3f, alphas %.3f, betas %.3f, ll %.3f, grad %.3f (teacher-forced); "
          "costs end to end %.3f (bar %.1e, costs %.1f..%.1f)"
          % (r_s, r_a, r_be, r_ll, r_g, r_c, float(bar_c.max()), float(-llf64.max()), float(-llf64.min())))
    assert max(r_s, r_a, r_be, r_ll, r_g, r_c) <= 1, (r_s, r_a, r_be, r_ll, r_g, r_c)


# ---- (f) bitwise invariants ----------------------------------------------------------------------------------------
def _embed_problem(dt, V=64, T=20, U=30, blank=3, seed=5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rng = np.random.RandomState(seed)
    X = torch.randn(1, T, U, V, device="cuda", generator=g, dtype=f64).to(dt) * 3
    lab = lr.planted_labels(rng, 1, U, V, blank)
    return X, lab


def _run(X, lab, xlen, ylen, blank, dt):
    B, T, U, V = X.shape
    c = dict(B=B, T=T, U=U, V=V, blank=blank, dt=dt, off=0, X=X,
             lab_d=torch.as_tensor(lab, device="cuda") if U > 1 else None,
             xlen_d=torch.as_tensor(np.asarray(xlen, np.int32), device="cuda"),
             ylen_d=torch.as_tensor(np.asarray(ylen, np.int32), device="cuda"))
    costs, ws = _fwd(c)
    g = _bwd(c, ws, torch.full_like(X, NAN), gscale=torch.ones(1, dtype=dt, device="cuda"), host_scale=1.0)
    torch.cuda.synchronize()
    return costs, _views(c, ws), g


@pytest.mark.parametrize("dt", [f32, f64])
@pytest.mark.parametrize("maxT, maxU", [(27, 40), (27, 1024)])
def test_utterance_bits_independent_of_batch_and_padding(dt, maxT, maxU):
    """(f) An utterance (T = 20, U+1 = 30, V = 64) alone, and embedded as utterance 1 of 3 with other neighbours and
    larger maxT / maxU padding: the same bits for its cost, ll_fwd / ll_bwd, its workspace cells and its gradient rows.
    maxU = 1024 also crosses from the PF = 8 lattice kernel (alone) to the wide one (embedded)."""
    X1, lab1 = _embed_problem(dt)
    T, U, V = X1.shape[1:]
    costs1, w1, g1 = _run(X1, lab1, [T], [U - 1], 3, dt)
    g = torch.Generator(device="cuda").manual_seed(9)
    X = (torch.randn(3, maxT, maxU, V, device="cuda", generator=g, dtype=f64) * 3).to(dt)
    X[1, :T, :U] = X1[0]
    lab = np.random.RandomState(2).randint(0, V - 1, size=(3, maxU - 1))
    lab = (lab + (lab >= 3)).astype(np.int32)
    lab[1, :U - 1] = lab1[0]
    costs, w, gr = _run(X, lab, [maxT, T, 11], [maxU - 1, U - 1, 7], 3, dt)
    bits = torch.int64 if dt == f64 else torch.int32
    eq = lambda a, b: torch.equal(a.contiguous().view(bits), b.contiguous().view(bits))
    assert eq(costs[1:2], costs1)
    for k in ("denom", "lpb", "lpl", "alphas", "betas"):
        assert eq(w[k][1, :T, :U], w1[k][0]), k
    assert eq(w["ll_fwd"][1:2], w1["ll_fwd"]) and eq(w["ll_bwd"][1:2], w1["ll_bwd"])
    assert eq(gr[1, :T, :U], g1[0])
    assert bool((gr[1, T:] == 0).all()) and bool((gr[1, :, U:] == 0).all())


@pytest.mark.parametrize("dt", [f32, f64])
def test_no_frames_and_over_long_lengths(dt):
    """(f) xlen = 0: cost +inf, ll_fwd = ll_bwd = -inf, a zero gradient and no workspace cell written, whatever its
    neighbours are (first, middle or last utterance).  Over-long lengths (xlen > maxT, ylen >= maxU, negative ones) give
    the same bits as the clamped lengths."""
    B, T, U, V, blank = 3, 14, 9, 40, 6
    g = torch.Generator(device="cuda").manual_seed(21)
    X = (torch.randn(B, T, U, V, device="cuda", generator=g, dtype=f64) * 3).to(dt)
    lab = lr.planted_labels(np.random.RandomState(4), B, U, V, blank)
    bits = torch.int64 if dt == f64 else torch.int32
    eq = lambda a, b: torch.equal(a.contiguous().view(bits), b.contiguous().view(bits))
    full = _run(X, lab, [14, 10, 7], [8, 5, 3], blank, dt)
    for z in range(B):
        xl = [14, 10, 7]
        xl[z] = 0
        costs, w, gr = _run(X, lab, xl, [8, 5, 3], blank, dt)
        assert float(costs[z]) == math.inf and float(w["ll_fwd"][z]) == -math.inf
        assert float(w["ll_bwd"][z]) == -math.inf
        assert bool((gr[z] == 0).all())
        for k in ("denom", "lpb", "lpl", "alphas", "betas"):
            assert bool(w[k][z].isnan().all()), (z, k)
        for b in range(B):
            if b != z:
                assert eq(costs[b], full[0][b]) and eq(gr[b], full[2][b]), (z, b)
                for k in ("denom", "lpb", "lpl", "alphas", "betas"):
                    assert eq(w[k][b], full[1][k][b]), (z, b, k)
    # over-long and negative lengths against their clamped values
    clamped = _run(X, lab, [14, 0, 7], [8, 0, 8], blank, dt)
    over = _run(X, lab, [14 + 9, -3, 7], [8 + 40, -5, 9], blank, dt)
    assert eq(clamped[0], over[0]) and eq(clamped[2], over[2])
    for k in ("denom", "lpb", "lpl", "alphas", "betas", "ll_fwd", "ll_bwd"):
        assert torch.equal(clamped[1][k].nan_to_num(), over[1][k].nan_to_num()), k


def test_fused_statistics_clamp_lengths():
    """(f) eb_joint_logits_lse decodes the valid cells with the same clamp: over-long lengths give the bits of the
    clamped ones, in the logits and in the statistics, and the lattice over them (eb_rnnt_loss_lattice) too."""
    from edgedict_b200 import ops
    B, T, U, V, J, blank = 2, 13, 7, 136, 64, 2
    g = torch.Generator(device="cuda").manual_seed(3)
    hid = (torch.rand(B * T * U, J, device="cuda", generator=g) * 2 - 1).to(bf16)
    w2 = (torch.randn(V, J, device="cuda", generator=g) * 0.6).to(bf16)
    b2 = torch.randn(V, device="cuda", generator=g)
    lab = torch.as_tensor(lr.planted_labels(np.random.RandomState(1), B, U, V, blank), device="cuda")
    res = []
    for xl, yl in (([13, 5], [6, 6]), ([13 + 4, 5], [6 + 9, 6])):
        xl, yl = torch.tensor(xl, dtype=torch.int32, device="cuda"), torch.tensor(yl, dtype=torch.int32, device="cuda")
        l16, ws = ops.joint_logits_lse(hid, w2, b2, lab, xl, yl, B, T, U, blank)
        n = B * T * U
        ws.view(f32)[3 * n:].fill_(NAN)
        wsf = ws.view(f32).clone()
        wsf[:3 * n] = torch.where(lr.valid_cells([13, 5], [6, 6], T, U, "cuda").reshape(-1).repeat(3),
                                  wsf[:3 * n], 0.0)
        costs = torch.full((B,), NAN, device="cuda")
        assert _lib().eb_rnnt_loss_lattice(_p(xl), _p(yl), B, T, U, _p(wsf), _p(costs), 1, _stream()) == 0
        torch.cuda.synchronize()
        res.append((l16, wsf, costs))
    assert torch.equal(res[0][0].view(torch.int16), res[1][0].view(torch.int16))
    assert torch.equal(res[0][1].nan_to_num().view(torch.int32), res[1][1].nan_to_num().view(torch.int32))
    assert torch.equal(res[0][2].view(torch.int32), res[1][2].view(torch.int32))


def test_wide_lattice_through_every_entry():
    """U+1 = 1024 through RNNTLoss (fp32, the drop-in module) and eb_rnnt_loss_lattice (the bf16 fused path's lattice),
    which launched no kernel at this width before the wide instantiation: RNNTLoss costs against the oracle (the cost
    bar of test_end_to_end_against_oracle), and the lattice-only entry on the statistics of eb_rnnt_loss_fwd gives the
    bits of eb_rnnt_loss_fwd's own lattice."""
    from edgedict_b200.warprnnt_pytorch import RNNTLoss
    c = _make_case("f32_u1024_wide")
    costs_o, _ = ol.logits(c["X"].double().cpu().numpy(), c["lab"], c["xlen"], c["ylen"], blank=c["blank"],
                           want_grads=False, dtype=np.float64)
    a = c["X"].clone().requires_grad_(True)
    out = RNNTLoss(blank=c["blank"], reduction="none")(a, c["lab_d"], c["xlen_d"], c["ylen_d"])
    out.sum().backward()
    x = c["X"].double()
    bar_c, _ = _e2e_bars(c, x, _smax(c, x, c["valid"]))
    r = float(np.max(np.abs(out.detach().double().cpu().numpy() - costs_o) / bar_c.cpu().numpy()))
    print("RNNTLoss at U+1 = 1024: costs err/bar %.3f" % r)
    assert r <= 1 and bool(torch.isfinite(a.grad).all())
    costs, ws = _fwd(c)
    ws2 = ws.clone()
    n = c["B"] * c["T"] * c["U"]
    ws2[3 * n:] = NAN
    costs2 = torch.full((c["B"],), NAN, device="cuda")
    assert _lib().eb_rnnt_loss_lattice(_p(c["xlen_d"]), _p(c["ylen_d"]), c["B"], c["T"], c["U"], _p(ws2), _p(costs2),
                                       1, _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(ws2.view(torch.int32), ws.view(torch.int32)) and torch.equal(costs2, costs)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_joint_loss_at_full_width(precision):
    """JointLoss (joint GEMMs, loss and gradient as one autograd node) at U+1 = 1024, the widest lattice.
    fp32 mode (eb_rnnt_loss_fwd / _bwd on fp32 logits): costs against oracle.loss.logits of the joint computed in fp64
    from the same operands, within the 1e-4 relative loss bar of the fp32 mode's model check (smoke()).  bf16 mode: the
    fused path (eb_joint_logits_lse, eb_rnnt_loss_lattice, eb_rnnt_loss_bwd_bf16) against the unfused bf16 path (fp32
    logits through eb_rnnt_loss_fwd) on the same bf16 operands, within the bars of test_gpu_model.py's fused-vs-unfused
    check (costs 2e-3, gradients 6e-2 relative); every gradient finite."""
    from edgedict_b200 import functional as Fn
    B, T, U, E, D, J, V, blank = 2, 5, 1024, 16, 16, 64, 64, 0
    g = torch.Generator().manual_seed(17)
    h_enc, h_dec = torch.randn(B, T, E, generator=g), torch.randn(B, U, D, generator=g)
    w1, b1 = torch.randn(J, E + D, generator=g) / 6, torch.randn(J, generator=g) / 6
    w2, b2 = torch.randn(V, J, generator=g) / 6, torch.randn(V, generator=g) / 6
    labels = torch.randint(1, V, (B, U - 1), generator=g, dtype=torch.int32)
    xl = torch.tensor([T, T - 2], dtype=torch.int32)
    yl = torch.tensor([U - 1, U - 300], dtype=torch.int32)
    rel = lambda a, b: float((a - b).norm() / b.norm())

    def run(fused):
        saved = Fn.FUSE_JOINT_LSE
        Fn.FUSE_JOINT_LSE = fused
        try:
            ins = [t.clone().cuda().requires_grad_(True) for t in (h_enc, h_dec, w1, b1, w2, b2)]
            loss, costs = Fn.JointLoss.apply(*ins, labels.cuda(), xl.cuda(), yl.cuda(), blank, precision)
            loss.backward()
        finally:
            Fn.FUSE_JOINT_LSE = saved
        grads = [t.grad.double().cpu() for t in ins]
        assert all(bool(torch.isfinite(gr).all()) for gr in grads)
        return costs.double().cpu(), grads

    if precision == "fp32":
        costs, _ = run(True)
        he, hd, W1, B1, W2, B2 = (t.double() for t in (h_enc, h_dec, w1, b1, w2, b2))
        hid = torch.tanh((he @ W1[:, :E].t() + B1)[:, :, None] + (hd @ W1[:, E:].t())[:, None])
        X = hid @ W2.t() + B2
        costs_o, _ = ol.logits(X.numpy(), labels.numpy(), xl.numpy(), yl.numpy(), blank=blank, want_grads=False,
                               dtype=np.float64)
        r = float(np.max(np.abs(costs.numpy() - costs_o) / np.abs(costs_o)))
        print("JointLoss fp32 at U+1 = 1024: costs rel err %.2e (bar 1e-4)" % r)
        assert r <= 1e-4, r
    else:
        c0, g0 = run(False)
        c1, g1 = run(True)
        r = rel(c1, c0)
        rg = max(rel(a, b) for a, b in zip(g1, g0))
        print("JointLoss bf16 at U+1 = 1024: fused vs unfused costs rel %.2e (bar 2e-3), gradients %.2e (bar 6e-2)"
              % (r, rg))
        assert r <= 2e-3 and rg <= 6e-2, (r, rg)
