"""Kernel-level fp64 parity of the pruned RNN-T loss (csrc/pruned.cu, the band entries of csrc/loss.cu and the LSE_BAND
epilogue of csrc/gemm_tc.cu), one section per C entry:

    eb_rnnt_simple_stats         N(t,u) in product form, the direct log-sum-exp on fallback cells (P < 1e-25)
    eb_rnnt_simple_bwd           d am / d lm: two fp32 GEMMs, then per row the fallback, blank and label terms
    eb_rnnt_band_choice          the band rule on the device's own occupancy, and on exact synthetic occupancies
    eb_joint_band_hidden_fwd     tanh rows of the bands, fp32 (tanhf) and bf16 (tanh.approx)
    eb_rnnt_band_loss_fwd        band-row statistics (VEC / scalar), the -inf fill and the lattice
    eb_joint_band_logits_lse     the logits GEMM's statistics epilogue over band rows, + eb_rnnt_band_lattice
    eb_rnnt_band_loss_bwd[_bf16_db]  band-row d logits (fp32, in place, bf16) and the bias gradient
    eb_joint_band_dpre_reduce    dep / ddp of band-row d(pre-activation)

The C entries are called directly, into NaN-prefilled workspaces and outputs.  References are fp64
(tests/pruned_restate.py, pinned to tests/pruned_oracle.py by tests/test_pruned_restate_host.py), teacher-forced on
the kernels' own inputs.  Every bar comes from the error model in its test's docstring and every measured err/bar is
printed (pytest -s).  eps = 2^-24, the fp32 unit roundoff; gamma_n = n eps / (1 - n eps).  The shape matrices name the
code path each case reaches.  Out-of-range starts are chosen so that even kernels that ignore the padding rule read
only inside their buffers: no negative start on utterance 0, no start past maxU - R on the last utterance."""
import math

import numpy as np
import pytest
import torch

from tests import loss_restate as lr
from tests import pruned_restate as pr

pytestmark = pytest.mark.gpu

f32, f64, bf16, i32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
NAN = float("nan")
EPS = 2.0 ** -24
EXP_FAST = 2.0 ** -22            # ex2.approx.ftz
EXP_ACC = 2.0 ** -23             # expf / logf / tanhf: 2 ulp


def gam(n):
    return n * EPS / (1 - n * EPS)


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ratio(err, bar, mask=None):
    r = err / bar
    if mask is not None:
        r = r[mask]
    return float(r.max()) if r.numel() else 0.0


def _ws(B, T, U):
    n = _lib().eb_rnnt_workspace_bytes(B, T, U, 4) // 4
    return torch.full((n,), NAN, dtype=f32, device="cuda")


def _views(ws, B, T, U):
    n = B * T * U
    sh = (B, T, U)
    return dict(denom=ws[:n].view(sh), lpb=ws[n:2 * n].view(sh), lpl=ws[2 * n:3 * n].view(sh),
                alphas=ws[3 * n:4 * n].view(sh), betas=ws[4 * n:5 * n].view(sh), ll=ws[5 * n:5 * n + B])


def _lens(xl, yl):
    return torch.tensor(xl, dtype=i32, device="cuda"), torch.tensor(yl, dtype=i32, device="cuda")


# ---------------------------------------------------------------------------------------------------------------------
# 1 / 2 / 3a: the simple loss.  name: (B, T, U, V, blank, xlen, ylen, plant)
#   plant: rows with a peak of +56 / +57.5 / +60 / +70 at different tokens in am and lm: products above, near and below
#   1e-25 (fallback cells), in the second chunk (t >= 256, u = 256) where the shape has one, and at the final cell
#   (T - 1, 256) whose occupancy is 1 in every utterance with T_b = T and U_b = 257
SIMPLE = {
    # bench shape at B = 2: T' = 500 (dlm's t-chunk loop: 256 + 244), V = 1024 (4 v0 passes), U+1 = 129
    "bench_u129_v1024": (2, 500, 129, 1024, 0, [500, 317], [128, 64], True),
    # U+1 = 257, V = 4096: dam's u-chunk loop (256 + 1) and 16 v0 passes
    "bench_u257_v4096": (1, 500, 257, 4096, 0, [500], [256], True),
    # chunk edges: T_b = 513 / 256 / 257, U_b = 257 / 256 / 1, T_b = 0; V = 29, blank = V - 1
    "edges_v29": (4, 513, 257, 29, 28, [513, 256, 257, 0], [256, 255, 0, 9], True),
    # V = 1000 (v0 tail), xlen = 1, ylen = 0
    "ragged_v1000": (3, 40, 20, 1000, 999, [40, 1, 33], [19, 0, 7], False),
}


def _simple_case(name):
    B, T, U, V, blank, xl, yl, plant = SIMPLE[name]
    seed = sum(map(ord, name))
    g = torch.Generator(device="cuda").manual_seed(seed)
    am = torch.randn(B, T, V, device="cuda", generator=g) * 1.5
    lm = torch.randn(B, U, V, device="cuda", generator=g) * 1.5
    if plant:
        for k, off in enumerate((56.0, 57.5, 60.0, 70.0)):
            ts = [t for t in (3 + k, 257 + k, 300 + 3 * k) + ((T - 1,) if k == 3 else ()) if t < T]
            us = [u for u in (2 + k, 120 + k, 253 + k) if u < U]
            am[:, ts, 5 + k] += off
            lm[:, us, 11 + k] += off
    rng = np.random.RandomState(seed)
    lab = lr.planted_labels(rng, B, U, V, blank)
    xlen, ylen = _lens(xl, yl)
    c = dict(name=name, B=B, T=T, U=U, V=V, blank=blank, am=am, lm=lm, xlen=xlen, ylen=ylen,
             lab=torch.as_tensor(lab, device="cuda") if U > 1 else None)
    c["ws"], c["scratch"] = _simple_fwd(c)
    return c


def _simple_fwd(c, am=None, lm=None, lab=None, xlen=None, ylen=None, B=None):
    am = c["am"] if am is None else am
    lm = c["lm"] if lm is None else lm
    B = c["B"] if B is None else B
    T, U, V = c["T"], c["U"], c["V"]
    ws = _ws(B, T, U)
    scratch = torch.full((_lib().eb_rnnt_simple_scratch_bytes(B, T, U, V) // 4,), NAN, dtype=f32, device="cuda")
    args = (c["lab"] if lab is None else lab, c["xlen"] if xlen is None else xlen, c["ylen"] if ylen is None else ylen)
    assert _lib().eb_rnnt_simple_stats(_p(am), _p(lm), *map(_p, args), B, T, U, V, c["blank"], _p(scratch), _p(ws),
                                       _st()) == 0
    costs = torch.full((B,), NAN, dtype=f32, device="cuda")
    assert _lib().eb_rnnt_loss_lattice(_p(args[1]), _p(args[2]), B, T, U, _p(ws), _p(costs), 1, _st()) == 0
    return ws, scratch


def _prod(c):
    """The scratch's product P [B, T, U] (eb_rnnt_simple_scratch_bytes layout)."""
    B, T, U, V = c["B"], c["T"], c["U"], c["V"]
    o = B * T * V + B * U * V + B * T + B * U
    return c["scratch"][o:o + B * T * U].view(B, T, U)


@pytest.fixture(scope="module", params=list(SIMPLE))
def simple(request):
    c = _simple_case(request.param)
    torch.cuda.synchronize()
    return c


def test_simple_stats(simple):
    """(1) denom / lpb / lpl per valid cell against N = logsumexp_v(am[t] + lm[u]) in fp64.

    Product cells, N = amax + lmax + log P: each term of P = sum_v exp(am - amax) exp(lm - lmax) carries expf (2 ulp)
    and the rounding of its argument (eps |x - max|) twice, the fp32 GEMM sums V positive terms (gamma_V relative),
    logf adds 2 ulp of |log P| plus eps, and the two additions eps (|amax| + |lmax| + |N|):
        bar = gamma_V + 4 EXP_ACC + eps (max|am - amax| + max|lm - lmax|) + eps (2 |log P| + 2) + 2 eps (|amax| + |lmax|
              + |N|).
    Fallback cells (the online log-sum-exp over V in ascending v): each step rounds the running sum (eps) and its two
    exponentials (2 ulp + eps |x - m|): bar = V (eps + 2 EXP_ACC) + eps (2 spread + 2 |m| + 2 |log s| + |N|).
    lpb / lpl add a[k] + l[k]: + 2 eps (|am_k| + |lm_k| + |lp|).  Padded cells stay NaN; fallback cells exist on both
    sides of the threshold where the case plants them (t >= 256, u = 256)."""
    c = simple
    B, T, U, V, blank = c["B"], c["T"], c["U"], c["V"], c["blank"]
    w = _views(c["ws"], B, T, U)
    valid = lr.valid_cells(c["xlen"], c["ylen"], T, U, "cuda")
    N = pr.simple_lse(c["am"], c["lm"], c["xlen"], c["ylen"])
    am, lm = c["am"].double(), c["lm"].double()
    amax, lmax = am.amax(-1), lm.amax(-1)
    P = _prod(c).double()
    fb = ~(P >= 1e-25)
    spr_a, spr_l = (am - amax[..., None]).abs().amax(-1), (lm - lmax[..., None]).abs().amax(-1)
    bar_p = (gam(V) + 4 * EXP_ACC + EPS * (spr_a[:, :, None] + spr_l[:, None, :]) + EPS * (2 * P.log().abs() + 2)
             + 2 * EPS * (amax[:, :, None].abs() + lmax[:, None, :].abs() + N.abs()))
    m = amax[:, :, None] + lmax[:, None, :]
    spread = (am.amax(-1) - am.amin(-1))[:, :, None] + (lm.amax(-1) - lm.amin(-1))[:, None, :]
    bar_f = V * (EPS + 2 * EXP_ACC) + EPS * (2 * spread + 2 * m.abs() + 2 * (N - m).abs() + N.abs())
    bar = torch.where(fb, bar_f, bar_p)
    r_d = _ratio((w["denom"].double() + N).abs(), bar, valid)
    ref_b = am[:, :, None, blank] + lm[:, None, :, blank] - N
    ab = am[:, :, None, blank].abs() + lm[:, None, :, blank].abs()
    r_b = _ratio((w["lpb"].double() - ref_b).abs(), bar + 2 * EPS * (ab + ref_b.abs()), valid)
    r_l = 0.0
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], T, U, "cuda")
    if U > 1:
        lab = c["lab"].long()
        xa = torch.gather(am, 2, lab[:, None, :].expand(B, T, U - 1))
        xl = torch.gather(lm[:, :U - 1], 2, lab[:, :, None])[:, None, :, 0]
        ref_l = xa + xl - N[:, :, :U - 1]
        has = valid[:, :, :U - 1] & (torch.arange(U - 1, device="cuda")[None, None, :] < Un[:, None, None] - 1)
        r_l = _ratio((w["lpl"][:, :, :U - 1].double() - ref_l).abs(),
                     bar[:, :, :U - 1] + 2 * EPS * (xa.abs() + xl.abs() + ref_l.abs()), has)
    nfb = int((fb & valid).sum())
    print("%s: denom err/bar %.3f, lpb %.3f, lpl %.3f; %d fallback cells, %d product cells with P < 1e-24"
          % (c["name"], r_d, r_b, r_l, nfb, int((~fb & valid & (P < 1e-24)).sum())))
    assert r_d <= 1 and r_b <= 1 and r_l <= 1, (r_d, r_b, r_l)
    for k in ("denom", "lpb", "lpl"):
        assert bool(w[k][~valid].isnan().all()), k
    if c["name"] in ("bench_u257_v4096", "edges_v29"):
        t = torch.arange(T, device="cuda")[None, :, None]
        u = torch.arange(U, device="cuda")[None, None, :]
        assert bool((fb & valid & (t >= 256)).any()) and bool((fb & valid & (u >= 256)).any())
        assert bool((~fb & valid & (P < 1e-24)).any())


def _simple_bwd(c, gscale, host_scale, B=None, am=None, lm=None, lab=None, xlen=None, ylen=None, ws=None, sc=None):
    B = c["B"] if B is None else B
    am = c["am"] if am is None else am
    lm = c["lm"] if lm is None else lm
    dam = torch.full_like(am, NAN)
    dlm = torch.full_like(lm, NAN)
    per = int(gscale is not None and gscale.numel() > 1)
    args = (c["lab"] if lab is None else lab, c["xlen"] if xlen is None else xlen, c["ylen"] if ylen is None else ylen)
    assert _lib().eb_rnnt_simple_bwd(_p(am), _p(lm), *map(_p, args), B, c["T"], c["U"], c["V"], c["blank"],
                                     _p(c["scratch"] if sc is None else sc), _p(c["ws"] if ws is None else ws),
                                     _p(gscale), per, float(host_scale), _p(dam), _p(dlm), _st()) == 0
    return dam, dlm


def test_simple_bwd(simple):
    """(2) d am / d lm per element against the header's formula on the kernel's own workspace (teacher-forced).

    Each term exp(a + be - ll + d + am + lm) is formed as exp(am - amax) G exp(lm - lmax) or directly: its relative
    error is expf's (2 ulp, three of them) plus the rounding of its exponent's sums, <= 8 eps mag with mag the largest
    |a| + |be| + |ll| + |d| + |amax| + |lmax| + |lpb| + |lpl| of the row's cells, plus eps |x - max| of each exp(x -
    max) (the row spreads); the GEMM over K = U (d am) or T (d lm) adds gamma_K.  The gamma sums and the subtractions
    round by eps per term.  So per element
        bar = |scale| sum|terms| (gamma_K + 3 EXP_ACC + 8 eps mag + eps (spread_a + spread_l) + gamma_K) + eps |ref|.
    The bar is on sum|terms|, not |result|: occupancy and gamma terms cancel.  Scales: gscale NULL, [1] and [B] with
    negative entries times host_scale = 1/B.  Rows t >= T_b, u >= U_b and every row of a T_b = 0 utterance are exactly
    0; row sums are ~0 within the sum of their bars."""
    c = simple
    B, T, U, V, blank = c["B"], c["T"], c["U"], c["V"], c["blank"]
    w = _views(c["ws"], B, T, U)
    valid = lr.valid_cells(c["xlen"], c["ylen"], T, U, "cuda")
    a, be, d, lpb, lpl = (w[k].double().where(valid, 0.0) for k in ("alphas", "betas", "denom", "lpb", "lpl"))
    a = a.where(valid, -math.inf)
    ll = w["ll"].double()
    one = torch.ones(B, dtype=f64, device="cuda")
    ref_a, ref_l, abs_a, abs_l = pr.simple_grad(c["am"], c["lm"], c["lab"], c["xlen"], c["ylen"], blank, a, be, d, lpb,
                                                lpl, ll, one)
    am, lm = c["am"].double(), c["lm"].double()
    amax, lmax = am.amax(-1), lm.amax(-1)
    mag = (a.abs() + be.abs() + ll.abs()[:, None, None] + d.abs() + lpb.abs() + lpl.abs()).where(valid, 0.0) + \
        amax.abs()[:, :, None] + lmax.abs()[:, None, :]
    mag = mag.where(valid, 0.0)
    spr_a, spr_l = (am - amax[..., None]).abs().amax(-1), (lm - lmax[..., None]).abs().amax(-1)
    base = 3 * EXP_ACC + EPS * (spr_a.amax(1) + spr_l.amax(1))[:, None]
    rel_a = (2 * gam(U) + base + 8 * EPS * mag.amax(2))[..., None]
    rel_l = (2 * gam(T) + base + 8 * EPS * mag.amax(1))[..., None]
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], T, U, "cuda")
    rows_t = torch.arange(T, device="cuda")[None, :] < Tn[:, None]
    rows_u = (torch.arange(U, device="cuda")[None, :] < Un[:, None]) & (Tn > 0)[:, None]
    gs = torch.tensor([1.5, -0.75, 2.0, -1.25][:B], device="cuda")
    for tag, gscale in (("gscale NULL", None), ("gscale [1]", torch.tensor([0.5], device="cuda")),
                        ("gscale [B]", gs)):
        hs = 1.0 / B
        dam, dlm = _simple_bwd(c, gscale, hs)
        s = torch.ones(B, dtype=f64, device="cuda") if gscale is None else gscale.double().expand(B)
        s = (s * hs)[:, None, None]
        ra, rl = ref_a * s, ref_l * s
        bar_a = abs_a * s.abs() * rel_a + EPS * ra.abs() + 2.0 ** -126
        bar_l = abs_l * s.abs() * rel_l + EPS * rl.abs() + 2.0 ** -126
        r_a = _ratio((dam.double() - ra).abs(), bar_a, rows_t[..., None].expand_as(ra))
        r_l = _ratio((dlm.double() - rl).abs(), bar_l, rows_u[..., None].expand_as(rl))
        rs_a = _ratio(dam.double().sum(-1).abs(), bar_a.sum(-1), rows_t)
        rs_l = _ratio(dlm.double().sum(-1).abs(), bar_l.sum(-1), rows_u)
        print("%s [%s]: dam err/bar %.3f, dlm %.3f; row sums dam %.3f, dlm %.3f"
              % (c["name"], tag, r_a, r_l, rs_a, rs_l))
        assert r_a <= 1 and r_l <= 1 and rs_a <= 1 and rs_l <= 1, (tag, r_a, r_l, rs_a, rs_l)
        assert bool(dam[~rows_t].eq(0).all()) and bool(dlm[~rows_u].eq(0).all()), tag
        assert not bool(dam.isnan().any()) and not bool(dlm.isnan().any())
    d2 = _simple_bwd(c, gs, 1.0 / B)
    assert torch.equal(d2[0], dam) and torch.equal(d2[1], dlm)                 # bitwise repeatable


def _occ_bar(w, valid, B):
    """(occ fp32 as the kernel forms it, fp64 occupancy, its per-cell error bar): expf(a + be - ll) with two fp32
    additions (eps (|a| + |be| + |ll|) each) and 2 ulp."""
    a, be, ll = w["alphas"], w["betas"], w["ll"][:, None, None]
    occ = torch.exp((a + be) - ll).where(valid, 0.0)
    a64, be64, ll64 = a.double(), be.double(), ll.double()
    o64 = torch.exp(a64 + be64 - ll64).where(valid, 0.0)
    bar = o64 * (EXP_ACC + 2 * EPS * (a64.abs() + be64.abs() + ll64.abs())).where(valid, 0.0)
    return occ, o64, bar


@pytest.mark.parametrize("R", [2, 5, 64])
def test_band_choice_on_device_occupancy(simple, R):
    """(3a) s_begin / nopath against the rule on the device's own simple workspace.  The fp64 score of a window is
    within sum_window bar(occ) + Rb eps score of the kernel's fp32 score; where every frame's margin (best minus second
    best fp64 score) exceeds twice that, the argmaxes agree and s_begin must match exactly.  Utterances with a frame
    below the bar are reported and skipped, as the CTC beam test does with near-ties."""
    c = simple
    B, T, U = c["B"], c["T"], c["U"]
    w = _views(c["ws"], B, T, U)
    valid = lr.valid_cells(c["xlen"], c["ylen"], T, U, "cuda")
    occ, o64, obar = _occ_bar(w, valid, B)
    s_ref, nop_ref, margin = pr.band_rule(occ, c["xlen"].cpu(), c["ylen"].cpu(), R, occ64=o64)
    s_dev = torch.full((B, T), -7, dtype=i32, device="cuda")
    nop = torch.full((B,), -7, dtype=i32, device="cuda")
    assert _lib().eb_rnnt_band_choice(_p(c["xlen"]), _p(c["ylen"]), B, T, U, R, _p(c["ws"]), _p(s_dev), _p(nop),
                                      _st()) == 0
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], T, U, "cpu")
    skipped, matched, worst = 0, 0, 0.0
    for b in range(B):
        rb = min(R, int(Un[b]))
        bar_t = (obar[b].sum(-1) * 1 + rb * EPS * o64[b].sum(-1) + 2.0 ** -126).cpu() * 2
        tn = int(Tn[b])
        if tn and bool((margin[b, :tn] <= bar_t[:tn]).any()):
            skipped += 1
            matched += int(s_dev[b].cpu().tolist() == s_ref[b].tolist())
            continue
        if tn:
            worst = max(worst, float((bar_t[:tn] / margin[b, :tn]).max()))
        assert s_dev[b].cpu().tolist() == s_ref[b].tolist() and int(nop[b]) == int(nop_ref[b]), b
    print("%s R=%d: band choice exact on %d of %d utterances (%d with a frame under the margin bar, %d of them equal "
          "anyway; largest bar/margin elsewhere %.3g)" % (c["name"], R, B - skipped, B, skipped, matched, worst))


# name: (T, U, R, xlen, ylen)  synthetic 0 / 1 occupancies
SYNTH = {
    "ties_r3": (40, 12, 3, [40, 17, 1, 0], [11, 11, 5, 3]),
    "r_ge_ub_and_ub1": (30, 9, 8, [30, 25, 12], [3, 0, 8]),
    "nopath": (6, 40, 4, [6, 6], [39, 10]),
    "t513": (513, 20, 5, [513, 300], [19, 7]),
    "maxT_12288": (12288, 6, 2, [12288, 7000], [5, 2]),
}


@pytest.mark.parametrize("name", list(SYNTH))
def test_band_choice_synthetic(name):
    """(3b) s_begin / nopath on synthetic workspaces with alpha + beta - ll in {0, -inf} (ll = 0): every expf gives
    exactly 1 or 0, the scores are exact integers, and the rule is compared without a bar: exact ties (the lowest s
    must win), R >= U_b, U_b = 1 (Rb = 1), nopath, T_b > 256 (several frames per thread) and maxT = 12288 (48 KB of
    dynamic shared memory)."""
    T, U, R, xl, yl = SYNTH[name]
    B = len(xl)
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    on = torch.rand(B, T, U, device="cuda", generator=g) < 0.3
    if name == "ties_r3":
        on[0, :, :] = False
        on[0, :, 2] = on[0, :, 5] = True                        # windows at s = 0..2 and 3..5 tie with one cell each
        on[1, ::2] = True                                        # every window full: ties everywhere
    xlen, ylen = _lens(xl, yl)
    valid = lr.valid_cells(xlen, ylen, T, U, "cuda")
    ws = _ws(B, T, U)
    w = _views(ws, B, T, U)
    w["alphas"].copy_(torch.where(on & valid, 0.0, -math.inf))
    w["betas"].copy_(torch.where(valid, 0.0, NAN))
    w["ll"].zero_()
    s_dev = torch.full((B, T), -7, dtype=i32, device="cuda")
    nop = torch.full((B,), -7, dtype=i32, device="cuda")
    assert _lib().eb_rnnt_band_choice(_p(xlen), _p(ylen), B, T, U, R, _p(ws), _p(s_dev), _p(nop), _st()) == 0
    occ = (on & valid).float()
    s_ref, nop_ref, _ = pr.band_rule(occ, xlen.cpu(), ylen.cpu(), R)
    assert torch.equal(s_dev.cpu(), s_ref) and torch.equal(nop.cpu(), nop_ref)
    print("%s: exact; nopath %s" % (name, nop.tolist()))
    if name == "nopath":
        assert nop.tolist() == [1, 0]


# ---------------------------------------------------------------------------------------------------------------------
# band rows.  name: (B, T, U, R, V, J, blank, xlen, ylen, offset)
BAND = {
    # bench shapes at small B: T' = 500, U+1 = 129, V = 1024, J = 640, R = 4 / 8; ragged with a nopath utterance
    "bench_r4": (3, 500, 129, 4, 1024, 640, 0, [500, 480, 3], [128, 100, 60], 0),
    "bench_r8_blank_last": (2, 500, 129, 8, 1024, 640, 1023, [500, 211], [128, 128], 0),
    # U+1 = 257, V = 4096, R = 5
    "bench_u257_v4096_r5": (1, 500, 257, 5, 4096, 640, 0, [500], [256], 0),
    # V = 1000 (GEMM tile tail), R >= U_b mixed with R < U_b, xlen = 0 / 1, ylen = 0
    "v1000_mixed": (5, 40, 30, 8, 1000, 64, 3, [40, 40, 1, 0, 25], [29, 4, 6, 5, 0], 0),
    # scalar loss kernels: V = 29 (odd, V % 4 != 0); V = 256 at a 4-byte offset; R = 2 and 64
    "v29_r2": (3, 30, 12, 2, 29, 16, 28, [30, 20, 9], [11, 11, 0], 0),
    "v256_offset_r64": (2, 20, 70, 64, 256, 32, 128, [20, 13], [69, 30], 1),
    # 40000 band rows: 313 row blocks of the logits GEMM, >= 2 per CTA
    "rows_40k_r20": (4, 500, 40, 20, 1024, 64, 0, [500, 500, 433, 250], [39, 30, 39, 10], 0),
}


def _band_case(name):
    B, T, U, R, V, J, blank, xl, yl, off = BAND[name]
    seed = sum(map(ord, name))
    rng = np.random.RandomState(seed)
    gc = torch.Generator().manual_seed(seed)
    xlen, ylen = _lens(xl, yl)
    Tn, Un = lr.lengths(xl, yl, T, U, "cpu")
    s = torch.zeros(B, T, dtype=i32)
    nop = torch.zeros(B, dtype=i32)
    for b in range(B):
        tn, un = int(Tn[b]), int(Un[b])
        if tn:
            sb, np_, _ = pr.band_rule(torch.rand(1, tn, un, generator=gc), [tn], [un - 1], R)
            s[b, :tn], nop[b] = sb[0, :tn], np_[0]
    lab = lr.planted_labels(rng, B, U, V, blank)
    c = dict(name=name, B=B, T=T, U=U, R=R, V=V, J=J, blank=blank, off=off, xlen=xlen, ylen=ylen, xl=xl, yl=yl,
             s=s.cuda(), nop=nop.cuda(), lab=torch.as_tensor(lab, device="cuda"))
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.full((B * T * R * V + off,), NAN, dtype=f32, device="cuda")[off:].view(B, T, R, V)
    X.copy_(torch.randn(B, T, R, V, device="cuda", generator=g) * 3)
    c["X"] = X
    return c


def _band_fwd(c, X=None, s=None, nop=None, xlen=None, ylen=None, B=None):
    B = c["B"] if B is None else B
    T, U, R, V = c["T"], c["U"], c["R"], c["V"]
    ws = _ws(B, T, U)
    costs = torch.full((B,), NAN, dtype=f32, device="cuda")
    assert _lib().eb_rnnt_band_loss_fwd(
        _p(c["X"] if X is None else X), _p(c["lab"][:B] if X is None else c["lab_b"]),
        _p(c["xlen"] if xlen is None else xlen), _p(c["ylen"] if ylen is None else ylen),
        _p(c["s"] if s is None else s), _p(c["nop"] if nop is None else nop), B, T, U, R, V, c["blank"], _p(ws),
        _p(costs), 1, _st()) == 0
    return costs, ws


def _dense_of(c, X):
    """[B, T, U, V] zeros with the live band rows of X at their cells."""
    B, T, U, R, V = c["B"], c["T"], c["U"], c["R"], c["V"]
    live, u = pr.live_rows(c["s"], c["nop"], c["xlen"], c["ylen"], T, U, R)
    D = torch.zeros(B, T, U, X.shape[-1], dtype=X.dtype, device="cuda")
    bi, ti, ri = live.nonzero(as_tuple=True)
    D[bi, ti, u[bi, ti, ri]] = X[bi, ti, ri]
    return D, live, u


def _stat_bar(X, V):
    """test_gpu_loss_fp64's per-row bar of denom for the 4-wide lane chunks of denom_row, on X fp64 [..., V]."""
    m = X.amax(-1)
    lse = torch.logsumexp(X, -1)
    Rm = (torch.softmax(X, -1) * (m[..., None] - X)).sum(-1)
    spread = m - X.amin(-1)
    chunks = -(-V // 128)
    return (1 + chunks) * EXP_FAST + EPS * (3 * Rm + 3 * spread + 2 * chunks + 16 + 2 * math.log(V) + lse.abs())


def _lattice_check(c, w, costs, tag):
    """alphas / betas / costs against loss_restate.lattice on the kernel's own lpb / lpl: (n + 1) eps (3 M + 6) per
    cell (test_gpu_loss_fp64's lattice model); nopath and T_b = 0 utterances cost +inf."""
    B, T, U = c["B"], c["T"], c["U"]
    al, be, llf, _ = lr.lattice(w["lpb"], w["lpl"], c["xlen"], c["ylen"])
    fin = torch.isfinite(llf)
    M = torch.maximum(al.nan_to_num(0, neginf=0).abs().amax((1, 2)), be.nan_to_num(0, neginf=0).abs().amax((1, 2)))
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], T, U, "cuda")
    bar = (Tn + Un).double() * EPS * (3 * M + 6)
    r = _ratio((w["ll"].double() - llf).abs(), bar, fin)
    print("%s [%s]: ll_fwd err/bar %.3f" % (c["name"], tag, r))
    assert r <= 1, r
    assert torch.equal(torch.isfinite(costs), fin)
    assert bool(costs[~fin].eq(math.inf).all())
    return fin


@pytest.fixture(scope="module", params=list(BAND))
def band(request):
    c = _band_case(request.param)
    c["costs"], c["ws"] = _band_fwd(c)
    torch.cuda.synchronize()
    return c


def test_band_loss_fwd(band):
    """(5) eb_rnnt_band_loss_fwd: statistics of each live band row against log_softmax in fp64 with the dense loss's
    statistics bar (test_gpu_loss_fp64: (1 + chunks) EXP_FAST + eps (3 R + 3 spread + 2 chunks + 16 + 2 log V +
    |denom|), + eps |lp| for lpb / lpl); bitwise the statistics eb_rnnt_loss_fwd gives a dense tensor holding the band
    rows at their cells; every other valid cell exactly -inf (all of a nopath utterance's), padded cells NaN; costs and
    ll against the lattice restatement on the kernel's own statistics."""
    c = band
    B, T, U, R, V = c["B"], c["T"], c["U"], c["R"], c["V"]
    w = _views(c["ws"], B, T, U)
    d, pb, pl, live = pr.band_stats(c["X"].double(), c["lab"], c["xlen"], c["ylen"], c["s"], c["nop"], U, c["blank"])
    valid = lr.valid_cells(c["xlen"], c["ylen"], T, U, "cuda")
    fill = valid & torch.isneginf(d)
    cell = valid & ~fill
    bar_rows = _stat_bar(c["X"].double(), V)
    bar = pr._scatter_cells(bar_rows, live, pr.live_rows(c["s"], c["nop"], c["xlen"], c["ylen"], T, U, R)[1], U, 1.0)
    r = [_ratio((w[k].double() - ref).abs(), bar + EPS * ref.abs(), cell)
         for k, ref in (("denom", d), ("lpb", pb), ("lpl", pl))]
    print("%s: band statistics err/bar denom %.3f lpb %.3f lpl %.3f (%d live rows, %d fill cells)"
          % (c["name"], *r, int(live.sum()), int(fill.sum())))
    assert max(r) <= 1, r
    for k in ("denom", "lpb", "lpl"):
        assert bool(w[k][fill].eq(-math.inf).all()), k
        assert bool(w[k][~valid].isnan().all()), k
    if B * T * U * V <= 200_000_000:
        D, _, _ = _dense_of(c, c["X"])
        wsd = _ws(B, T, U)
        cd = torch.empty(B, dtype=f32, device="cuda")
        assert _lib().eb_rnnt_loss_fwd(_p(D), _p(c["lab"]), _p(c["xlen"]), _p(c["ylen"]), B, T, U, V, c["blank"], 4,
                                       _p(wsd), _p(cd), 1, _st()) == 0
        wd = _views(wsd, B, T, U)
        for k in ("denom", "lpb", "lpl"):
            assert torch.equal(w[k][cell].view(i32), wd[k][cell].view(i32)), k
    fin = _lattice_check(c, w, c["costs"], "fp32")
    assert not bool(fin[c["nop"].bool()].any())


def test_band_loss_negative_and_past_the_end_starts():
    """(5, padding rule) starts outside [0, U_b - Rb]: a negative start on the only frame of utterance 2 (Rb = 7) and on
    frames 0..1 of utterance 4 (Rb = 1) makes every cell of those frames -inf in a NaN-prefilled workspace, so their
    costs are the restated +inf; a start past the end on the last
    frame of utterance 1 (R >= U_b) makes row 4 padding while its path survives.  Every cost matches the lattice
    restatement on the restated statistics within the lattice bar plus the statistics bar along a path."""
    c = _band_case("v1000_mixed")
    B, T, U, V = c["B"], c["T"], c["U"], c["V"]
    s = c["s"].clone()
    s[2, 0] = -1
    s[4, :2] = -1
    s[1, T - 1] = 1
    c["s"] = s
    costs, ws = _band_fwd(c)
    w = _views(ws, B, T, U)
    valid = lr.valid_cells(c["xlen"], c["ylen"], T, U, "cuda")
    d, pb, pl, live = pr.band_stats(c["X"].double(), c["lab"], c["xlen"], c["ylen"], s, c["nop"], U, c["blank"])
    assert not bool(live[4, :2].any()) and not bool(live[2, 0].any())
    assert live[1, T - 1].tolist()[:5] == [True] * 4 + [False]
    assert bool(w["denom"][2, 0][valid[2, 0]].eq(-math.inf).all())
    assert bool(w["denom"][4, :2][valid[4, :2]].eq(-math.inf).all())
    assert torch.equal(torch.isneginf(w["denom"]) & valid, torch.isneginf(d) & valid)
    _, _, llf, _ = lr.lattice(pb, pl, c["xlen"], c["ylen"])
    ref = -llf
    assert torch.equal(torch.isfinite(costs), torch.isfinite(ref)) and float(costs[2]) == float(costs[4]) == math.inf
    fin = torch.isfinite(ref)
    Tn, Un = lr.lengths(c["xlen"], c["ylen"], T, U, "cuda")
    smax = float(_stat_bar(c["X"].double(), V).max()) * 2
    bar = (Tn + Un).double() * (EPS * (3 * ref.abs().nan_to_num(0, posinf=0) + 6) + smax)
    r = _ratio((costs.double() - ref).abs(), bar, fin)
    print("negative / past-the-end starts: cost err/bar %.3f" % r)
    assert r <= 1


def test_band_logits_lse_and_lattice(band):
    """(6) eb_joint_band_logits_lse + eb_rnnt_band_lattice (bf16 mode).  logits16 against the fp64 product of the bf16
    operands: gamma_J sum_j |h w| + |b| eps, then one bf16 rounding (2^-8 relative).  Statistics against log_softmax of
    the fp64 logits with the dense statistics bar plus gamma_J max_v sum_j |h w| (a logit's error reaches the
    log-sum-exp as a weighted mean).  Bitwise: logits16 and the statistics are those eb_joint_logits_lse gives a dense
    hidden16 that holds the same rows at their cells; the lattice's fill and costs as in (5)."""
    c = band
    B, T, U, R, V, J = c["B"], c["T"], c["U"], c["R"], c["V"], c["J"]
    if V % 8 or J % 8:
        pytest.skip("bf16 mode needs V % 8 == 0 and J % 8 == 0")
    g = torch.Generator(device="cuda").manual_seed(7)
    h16 = torch.tanh(torch.randn(B, T, R, J, device="cuda", generator=g)).to(bf16)
    live, u = pr.live_rows(c["s"], c["nop"], c["xlen"], c["ylen"], T, U, R, loss=False)
    h16[~live] = 0
    w16 = (torch.randn(V, J, device="cuda", generator=g) / math.sqrt(J)).to(bf16)
    b2 = torch.randn(V, device="cuda", generator=g) * 0.1
    lg16 = torch.full((B, T, R, V), NAN, dtype=bf16, device="cuda")
    ws = _ws(B, T, U)
    w = _views(ws, B, T, U)
    n = B * T * U
    assert _lib().eb_joint_band_logits_lse(_p(h16), _p(w16), _p(b2), _p(lg16), _p(c["lab"]), _p(c["xlen"]),
                                           _p(c["ylen"]), _p(c["s"]), _p(ws[:n]), _p(ws[n:2 * n]), _p(ws[2 * n:3 * n]),
                                           B, T, U, R, V, J, c["blank"], _st()) == 0
    costs = torch.full((B,), NAN, dtype=f32, device="cuda")
    assert _lib().eb_rnnt_band_lattice(_p(c["xlen"]), _p(c["ylen"]), _p(c["s"]), _p(c["nop"]), B, T, U, R, _p(ws),
                                       _p(costs), 1, _st()) == 0
    x = (h16.double().view(-1, J) @ w16.double().t() + b2.double()).view(B, T, R, V)
    ax = (h16.double().abs().view(-1, J) @ w16.double().abs().t()).view(B, T, R, V)
    bar_x = gam(J) * ax + EPS * b2.double().abs() + 2.0 ** -8 * x.abs() + 2.0 ** -133
    r_x = _ratio((lg16.double() - x).abs(), bar_x)
    d, pb, pl, lv = pr.band_stats(x, c["lab"], c["xlen"], c["ylen"], c["s"], c["nop"], U, c["blank"])
    valid = lr.valid_cells(c["xlen"], c["ylen"], T, U, "cuda")
    cell = valid & ~torch.isneginf(d)
    bar_rows = _stat_bar(x, V) + gam(J) * ax.amax(-1) * 2 + 2 * EPS * b2.abs().max()
    bar = pr._scatter_cells(bar_rows, lv, u, U, 1.0)
    r = [_ratio((w[k].double() - ref).abs(), bar + EPS * ref.abs(), cell)
         for k, ref in (("denom", d), ("lpb", pb), ("lpl", pl))]
    print("%s: logits16 err/bar %.3f; statistics denom %.3f lpb %.3f lpl %.3f" % (c["name"], r_x, *r))
    assert r_x <= 1 and max(r) <= 1, (r_x, r)
    fill = valid & torch.isneginf(d)
    assert bool(w["denom"][fill].eq(-math.inf).all()) and bool(w["denom"][~valid].isnan().all())
    _lattice_check(c, w, costs, "bf16")
    if B * T * U * V <= 600_000_000:
        D16, live, u = _dense_of(c, h16)
        ld = torch.empty(B, T, U, V, dtype=bf16, device="cuda")
        wsd = _ws(B, T, U)
        assert _lib().eb_joint_logits_lse(_p(D16), _p(w16), _p(b2), _p(ld), _p(c["lab"]), _p(c["xlen"]),
                                          _p(c["ylen"]), _p(wsd[:n]), _p(wsd[n:2 * n]), _p(wsd[2 * n:3 * n]), B, T, U,
                                          V, J, c["blank"], _st()) == 0
        wd = _views(wsd, B, T, U)
        for k in ("denom", "lpb", "lpl"):
            assert torch.equal(w[k][cell].view(i32), wd[k][cell].view(i32)), k
        bi, ti, ri = live.nonzero(as_tuple=True)
        assert torch.equal(lg16[bi, ti, ri].view(torch.int16), ld[bi, ti, u[bi, ti, ri]].view(torch.int16))


def _grad_bar(terms, x, blank, sc):
    """test_gpu_loss_fp64's per-element gradient bar on band rows."""
    ax = x.abs()
    bar = terms["main"] * (EXP_FAST + EPS * (5 * terms["mag_all"][..., None] + 2 * ax))
    bar[..., blank] += terms["corr_b"] * (EXP_ACC + EPS * (5 * terms["mag_b"] + 2 * ax[..., blank]))
    y = terms["y"]
    e = terms["corr_l"] * (EXP_ACC + EPS * (5 * terms["mag_l"] + 2 * ax.gather(3, y[..., None])[..., 0]))
    bar.scatter_add_(3, y[..., None], e[..., None])
    return (bar + 2 * EPS * terms["absum"]) * sc.abs()[:, None, None, None]


def test_band_loss_bwd(band):
    """(7) eb_rnnt_band_loss_bwd (fp32 out, in place, bf16 out) and eb_rnnt_band_loss_bwd_bf16_db against the band
    gradient (pruned_restate.band_grad, grad_formula per band row) on the kernel's own workspace, with the dense
    gradient's per-element bar (test_gpu_loss_fp64: each term's exponent rounding and exponential, 2 eps sum|terms|,
    eps |ref|, one bf16 rounding for bf16 out).  Bitwise: each equals the dense eb_rnnt_loss_bwd /
    eb_rnnt_loss_bwd_bf16_db on the scattered dense logits with the same band workspace, at the band cells; db equals
    eb_colsum of the written gradients bitwise and is within the fp64 column sum's bar (sum of the row bars + gamma_rows
    sum |g|).  Padding rows and nopath utterances are exactly 0."""
    c = band
    B, T, U, R, V, blank = c["B"], c["T"], c["U"], c["R"], c["V"], c["blank"]
    w = _views(c["ws"], B, T, U)
    gs = torch.tensor([1.0, -0.5, 2.0, 0.75, -1.5][:B], device="cuda")
    hs = 1.0 / B
    sc = gs.double() * hs
    X = c["X"]
    g_ref, terms = pr.band_grad(w["alphas"].double(), w["betas"].double(), w["denom"].double(), w["ll"].double(),
                                X.double(), c["lab"], c["xlen"], c["ylen"], c["s"], c["nop"], U, blank, scale=sc,
                                terms=True)
    live = terms["live"]
    bar = _grad_bar(terms, X.double(), blank, sc) + EPS * g_ref.abs() + 2.0 ** -120

    def run(out, logits):
        assert _lib().eb_rnnt_band_loss_bwd(_p(logits), _p(out), int(out.dtype == bf16), _p(c["lab"]), _p(c["xlen"]),
                                            _p(c["ylen"]), _p(c["s"]), _p(c["nop"]), B, T, U, R, V, blank, _p(c["ws"]),
                                            _p(gs), 1, hs, _st()) == 0
        return out

    off = c["off"]
    g32 = run(torch.full((B * T * R * V + off,), NAN, dtype=f32, device="cuda")[off:].view(B, T, R, V), X)
    g16 = run(torch.full((B, T, R, V), NAN, dtype=bf16, device="cuda"), X)
    Xi = X.clone()
    run(Xi, Xi)
    assert torch.equal(Xi, g32)
    r32 = _ratio((g32.double() - g_ref).abs(), bar)
    bar16 = bar + 2.0 ** -8 * (g_ref.abs() + bar)
    r16 = _ratio((g16.double() - g_ref).abs(), bar16)
    assert bool(g32[~live].eq(0).all()) and bool(g16[~live].eq(0).all())
    assert not bool(g32.isnan().any())
    msg = "%s: d logits err/bar fp32 %.3f, bf16 %.3f" % (c["name"], r32, r16)
    assert r32 <= 1 and r16 <= 1, (r32, r16)
    if B * T * U * V <= 200_000_000:
        D, _, u = _dense_of(c, X)
        gd = torch.empty_like(D)
        assert _lib().eb_rnnt_loss_bwd(_p(D), _p(gd), 0, _p(c["lab"]), _p(c["xlen"]), _p(c["ylen"]), B, T, U, V,
                                       blank, 4, _p(c["ws"]), _p(gs), 1, hs, _st()) == 0
        bi, ti, ri = live.nonzero(as_tuple=True)
        assert torch.equal(g32[bi, ti, ri], gd[bi, ti, u[bi, ti, ri]])
    if V % 8 == 0 and off == 0:
        X16 = X.to(bf16)
        G16 = X16.clone()
        part = torch.empty(512 * V, dtype=f32, device="cuda")
        db = torch.zeros(V, dtype=f32, device="cuda")
        assert _lib().eb_rnnt_band_loss_bwd_bf16_db(_p(G16), _p(G16), _p(c["lab"]), _p(c["xlen"]), _p(c["ylen"]),
                                                    _p(c["s"]), _p(c["nop"]), B, T, U, R, V, blank, _p(c["ws"]),
                                                    _p(gs), 1, hs, _p(part), _p(db), _st()) == 0
        g_ref16, t16 = pr.band_grad(w["alphas"].double(), w["betas"].double(), w["denom"].double(), w["ll"].double(),
                                    X16.double(), c["lab"], c["xlen"], c["ylen"], c["s"], c["nop"], U, blank, scale=sc,
                                    terms=True)
        b16 = _grad_bar(t16, X16.double(), blank, sc) + EPS * g_ref16.abs() + 2.0 ** -120
        b16 = b16 + 2.0 ** -8 * (g_ref16.abs() + b16)
        rdb16 = _ratio((G16.double() - g_ref16).abs(), b16)
        assert bool(G16[~live].eq(0).all()) and rdb16 <= 1, rdb16
        cs = torch.zeros(V, dtype=f32, device="cuda")
        assert _lib().eb_colsum(_p(G16), 1, _p(cs), B * T * R, V, _st()) == 0
        assert torch.equal(db.view(i32), cs.view(i32))
        rows = B * T * R
        db_ref = g_ref16.sum((0, 1, 2))
        bar_db = b16.sum((0, 1, 2)) + gam(rows) * G16.double().abs().sum((0, 1, 2)) + 2.0 ** -120
        rdb = _ratio((db.double() - db_ref).abs(), bar_db)
        msg += ", bf16_db %.3f, db %.3f" % (rdb16, rdb)
        assert rdb <= 1, rdb
        # bitwise the dense bf16 entry on the scattered logits, at the band cells
        if B * T * U * V <= 200_000_000:
            D16, _, u = _dense_of(c, X16)
            part2 = torch.empty(512 * V, dtype=f32, device="cuda")
            db2 = torch.zeros(V, dtype=f32, device="cuda")
            assert _lib().eb_rnnt_loss_bwd_bf16_db(_p(D16), _p(D16), _p(c["lab"]), _p(c["xlen"]), _p(c["ylen"]), B, T,
                                                   U, V, blank, _p(c["ws"]), _p(gs), 1, hs, _p(part2), _p(db2),
                                                   _st()) == 0
            bi, ti, ri = live.nonzero(as_tuple=True)
            assert torch.equal(G16[bi, ti, ri].view(torch.int16), D16[bi, ti, u[bi, ti, ri]].view(torch.int16))
    print(msg)


@pytest.mark.parametrize("bf16_mode", [False, True])
@pytest.mark.parametrize("name", ["bench_r4", "v256_offset_r64", "v29_r2"])
def test_band_hidden_fwd(name, bf16_mode):
    """(4) eb_joint_band_hidden_fwd against tanh(ep + dp[s + r]) in fp64, with out-of-range starts (negative on
    utterance >= 1, past the end short of maxU - R on the last).  fp32 (tanhf): 2 ulp of |h| plus the sum's rounding
    eps |e + d| times (1 - h^2).  bf16 (tanh.approx.f32, max relative error 2^-10.987 per the PTX ISA) then one bf16
    rounding (2^-8 relative).  Padding rows are exactly 0."""
    B, T, U, R, V, J, blank, xl, yl, _ = BAND[name]
    J = max(J, 8)
    c = _band_case(name)
    s = c["s"].clone()
    if B > 1:
        s[1, :2] = -1
        s[B - 1, 0] = max(0, U - R)                          # at most maxU - R: every row it would read lies inside dp
    g = torch.Generator(device="cuda").manual_seed(3)
    ep = torch.randn(B, T, J, device="cuda", generator=g)
    dp = torch.randn(B, U, J, device="cuda", generator=g)
    xlen, ylen = c["xlen"], c["ylen"]
    hid = torch.full((B, T, R, J), NAN, dtype=bf16 if bf16_mode else f32, device="cuda")
    assert _lib().eb_joint_band_hidden_fwd(_p(ep), _p(dp), _p(xlen), _p(ylen), _p(s), _p(hid), int(bf16_mode), B, T,
                                           U, R, J, _st()) == 0
    live, u = pr.live_rows(s, c["nop"], xlen, ylen, T, U, R, loss=False)
    uu = torch.where(live, u, 0)
    pre = ep.double()[:, :, None, :] + torch.stack([dp.double()[b][uu[b]] for b in range(B)])
    h = torch.tanh(pre)
    if bf16_mode:
        bar = (2.0 ** -10.987 + 2.0 ** -8) * 1.001 * h.abs() + (1 - h * h) * EPS * pre.abs() + 2.0 ** -126
    else:
        bar = 2 * EXP_ACC * h.abs() + (1 - h * h) * EPS * pre.abs() + 2.0 ** -149
    r = _ratio((hid.double() - h).abs(), bar, live[..., None].expand_as(h))
    print("%s [%s]: hidden err/bar %.3f (%d padding rows)" % (name, "bf16" if bf16_mode else "fp32", r,
                                                               int((~live).sum())))
    assert r <= 1, r
    assert bool(hid[~live].eq(0).all())


# name: (B, T, U, R, J, xlen, ylen)
REDUCE = {
    "t500_u257_r2_j640": (2, 500, 257, 2, 640, [500, 300], [256, 255]),
    "t500_u129_r64_j640": (2, 500, 129, 64, 640, [500, 77], [128, 20]),
    "t257_u40_r5_j24": (3, 257, 40, 5, 24, [257, 256, 1], [39, 0, 39]),
}


@pytest.mark.parametrize("bf16_mode", [False, True])
@pytest.mark.parametrize("name", list(REDUCE))
def test_band_dpre_reduce(name, bf16_mode):
    """(8) eb_joint_band_dpre_reduce against pruned_restate.band_reduce on the same dpre (fp32: dx (1 - h^2) formed in
    fp64 from the fp32 operands; bf16: dx itself).  Bar per element gamma_n sum|terms| with n the number of terms
    (R for dep, T for ddp), plus 3 eps per term of the fp32 product.  Rows u >= U_b are 0; padding rows carry garbage
    and must not reach dep or ddp, including rows past U_b and frames with a negative start (utterance 1, frames
    0..1, monotone)."""
    B, T, U, R, J, xl, yl = REDUCE[name]
    xlen, ylen = _lens(xl, yl)
    Tn, Un = lr.lengths(xl, yl, T, U, "cpu")
    gc = torch.Generator().manual_seed(sum(map(ord, name)))
    s = torch.zeros(B, T, dtype=i32)
    for b in range(B):
        tn, un = int(Tn[b]), int(Un[b])
        if tn:
            sb, _, _ = pr.band_rule(torch.rand(1, tn, un, generator=gc), [tn], [un - 1], R)
            s[b, :tn] = sb[0, :tn]
    s[1, :2] = -1
    s[0, int(Tn[0]) - 1] = int(Un[0]) - 1                    # past the end on the last frame of utterance 0
    s = s.cuda()
    g = torch.Generator(device="cuda").manual_seed(5)
    dx = torch.randn(B, T, R, J, device="cuda", generator=g)
    hid = torch.tanh(torch.randn(B, T, R, J, device="cuda", generator=g))
    if bf16_mode:
        dx = dx.to(bf16)
        hid_arg, dpre = None, dx.double()
    else:
        hid_arg, dpre = hid, dx.double() * (1 - hid.double() ** 2)
    dep = torch.full((B, T, J), NAN, dtype=f32, device="cuda")
    ddp = torch.full((B, U, J), NAN, dtype=f32, device="cuda")
    assert _lib().eb_joint_band_dpre_reduce(_p(dx), _p(hid_arg), int(bf16_mode), _p(xlen), _p(ylen), _p(s), _p(dep),
                                            _p(ddp), B, T, U, R, J, _st()) == 0
    rdep, rddp, adep, addp = pr.band_reduce(dpre, s, xlen, ylen, U)
    extra = 0.0 if bf16_mode else 3 * EPS
    bdep = (gam(R) + extra) * adep + 2.0 ** -149
    bddp = (gam(T) + extra) * addp + 2.0 ** -149
    r1 = _ratio((dep.double() - rdep).abs(), bdep)
    r2 = _ratio((ddp.double() - rddp).abs(), bddp)
    print("%s [%s]: dep err/bar %.3f, ddp %.3f" % (name, "bf16" if bf16_mode else "fp32", r1, r2))
    assert r1 <= 1 and r2 <= 1, (r1, r2)
    rows_u = torch.arange(U, device="cuda")[None, :] >= Un.cuda()[:, None]
    assert bool(ddp[rows_u].eq(0).all()) and bool(dep[1, :2].eq(0).all())


def test_batch_independence_and_repeatability():
    """(9) every entry bitwise repeatable (run twice), and the simple loss, the band choice and the band loss
    bitwise batch-independent: an utterance alone equals its rows of the batch."""
    c = _simple_case("ragged_v1000")
    B, T, U = c["B"], c["T"], c["U"]
    ws2, _ = _simple_fwd(c)
    assert torch.equal(ws2.view(i32), c["ws"].view(i32))
    R = 4
    s_all = torch.empty(B, T, dtype=i32, device="cuda")
    n_all = torch.empty(B, dtype=i32, device="cuda")
    assert _lib().eb_rnnt_band_choice(_p(c["xlen"]), _p(c["ylen"]), B, T, U, R, _p(c["ws"]), _p(s_all), _p(n_all),
                                      _st()) == 0
    wa = _views(c["ws"], B, T, U)
    for b in range(B):
        sl = slice(b, b + 1)
        ws1, _ = _simple_fwd(c, am=c["am"][sl].contiguous(), lm=c["lm"][sl].contiguous(), lab=c["lab"][sl].contiguous(),
                             xlen=c["xlen"][sl].contiguous(), ylen=c["ylen"][sl].contiguous(), B=1)
        w1 = _views(ws1, 1, T, U)
        for k in ("denom", "lpb", "lpl", "alphas", "betas", "ll"):
            assert torch.equal(w1[k].view(i32), wa[k][sl].view(i32)), (b, k)
        s1 = torch.empty(1, T, dtype=i32, device="cuda")
        n1 = torch.empty(1, dtype=i32, device="cuda")
        assert _lib().eb_rnnt_band_choice(_p(c["xlen"][sl]), _p(c["ylen"][sl]), 1, T, U, R, _p(ws1), _p(s1), _p(n1),
                                          _st()) == 0
        assert torch.equal(s1, s_all[sl]) and torch.equal(n1, n_all[sl])
    bc = _band_case("v1000_mixed")
    costs2, ws2 = _band_fwd(bc)
    costs, ws = _band_fwd(bc)
    assert torch.equal(costs.view(i32), costs2.view(i32)) and torch.equal(ws.view(i32), ws2.view(i32))
    for b in range(bc["B"]):
        sl = slice(b, b + 1)
        bc["lab_b"] = bc["lab"][sl].contiguous()
        c1, w1 = _band_fwd(bc, X=bc["X"][sl].contiguous(), s=bc["s"][sl].contiguous(), nop=bc["nop"][sl].contiguous(),
                           xlen=bc["xlen"][sl].contiguous(), ylen=bc["ylen"][sl].contiguous(), B=1)
        assert torch.equal(c1.view(i32), costs[sl].view(i32)), b
    print("batch independence and repeatability: bitwise")
