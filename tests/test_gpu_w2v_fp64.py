"""Per-element fp64 parity and bitwise invariants of every csrc/w2v.cu kernel, each through its C entry point
(``_lib``), into NaN-prefilled outputs (int outputs prefilled with -7).

The error model and every bar are in tests/w2v_restate.py's docstring.  Each kernel is teacher-forced: logits_fwd is
checked on the xh / yh that normalize wrote, logits_bwd on the kernel's own A, AC, xh, yh, xn and yn, quant_bwd on the
kernel's own s, p and coef, so a failure names one kernel and one element.  Copies, selections and integer outputs are
restated bit for bit: the row copies against host indexing, ``scale`` against fp32 ``x * (g * alpha)``, k0 / k against
the kernels' lane maps (the first-index argmax without NaN), st, X and q from the kernel's own s, counts against a
bincount and CE's correct count against the restated rule on the same fp32 logits.

A NaN logit in quant_fwd makes p (and s) NaN over its (row, group) (the sum is NaN); the k0 (k) reported is where
lane 0's butterfly ends (``w2v_restate.lane_arg``): a NaN a lane meets first sticks there and wins only if that lane is
lane 0's, a NaN later in a lane's slice is skipped.  A lane holding NaN neither takes nor hands on a pair, so the lanes
can end on different indices and that group's X and q are not pinned.  torch.argmax would return the NaN's index; the
engine's quantizer rows are never NaN.

A masked candidate (c > 0 whose logit is -inf because it equals the positive) passes no gradient: the reference's
``logits[1:][neg_is_pos] = -inf`` is an index_put whose backward is zero there.  The forward's saved cosine is -inf at
those candidates too, and that is how the backward knows them.  ``test_masked_candidates_pass_no_gradient``
feeds a dense upstream gradient that is nonzero at every masked candidate.

``pytest -s`` prints the worst err/bar of every check and where it occurs; DESIGN.md section 2 records the figures.  The
case tables reach every loop trip count the kernels have, asserted in ``test_reach``."""
import math

import numpy as np
import pytest
import torch

from tests import w2v_restate as rs

pytestmark = pytest.mark.gpu

f32, f64, i32 = torch.float32, torch.float64, torch.int32
DEV = "cuda"
NAN = float("nan")
EPS = 1e-8              # torch.cosine_similarity's eps (ops.COS_EPS)
TEMP = 0.1

ROW_CASES = [(2, 7, 1, 1), (3, 5, 5, 33), (2, 40, 9, 33), (4, 1000, 900, 640)]      # (B, T, M, D)
SQ_N = [1, 5, 1023, 1024, 1025, 4096, 4097, 3_000_001]
QUANT_CASES = [(7, 1, 1, 3), (40, 2, 31, 5), (33, 4, 32, 8), (50, 1, 33, 1), (300, 2, 320, 64), (20, 4, 1100, 33),
               (9, 2, 70, 4)]                                                     # (N, G, V, vd)
STATS_CASES = [(5, 1, 1), (3, 2, 7), (300, 2, 320), (700, 2, 320), (10, 4, 300), (50, 1, 1100)]   # (N, G, V)
BWD_CASES = [(3, 1, 1), (9, 4, 33), (40, 2, 320), (5, 1, 1100)]                  # (N, G, V)
FWD_CASES = [(2, 5, 1, 1), (2, 9, 31, 100), (3, 40, 32, 100), (2, 33, 33, 1), (2, 30, 512, 100), (1, 50, 513, 7),
             (2, 20, 640, 100), (2, 12, 1030, 100)]                               # (B, M, D, K)
BWDL_D = [1, 511, 512, 513, 1023, 1024, 1025, 1030, 1537]
CE_CASES = [(2, 1, 1), (33, 1, 31), (101, 4, 8), (101, 3, 11), (2, 2, 17), (33, 24, 450)]   # (C, B, M)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_cap():
    """grid_for's cap in threads: SMs x 32 blocks x 256 threads."""
    return sms() * 32 * 256


# ---- calls and buffers -------------------------------------------------------------------------------------------------
def call(name, *args):
    from edgedict_b200._lib import lib
    a = [x.data_ptr() if torch.is_tensor(x) else x for x in args]
    rc = getattr(lib(), name)(*a, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, (name, rc)


def nanf(*shape):
    return torch.full(shape, NAN, dtype=f32, device=DEV)


def negi(*shape):
    return torch.full(shape, -7, dtype=i32, device=DEV)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(*shape, g, scale=1.0):
    return torch.randn(shape, generator=g, device=DEV) * scale


def bits(x):
    return x.view(i32) if x.dtype == f32 else x


def same_bits(a, b):
    """Bit for bit, except that any NaN equals any NaN (payloads are not part of any contract here)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype != f32:
        return torch.equal(a, b)
    nan = a.isnan()
    return torch.equal(nan, b.isnan()) and torch.equal(bits(a.contiguous())[~nan], bits(b.contiguous())[~nan])


WORST = {}


def check(what, got, want, b):
    """got (fp32) within b of want (fp64) per element; NaN and infinities exactly where want has them."""
    got, want, b = got.to(f64), want.to(f64).to(got.device), b.to(f64).to(got.device)
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    assert torch.equal(got.isnan(), want.isnan()), (what, "NaN mismatch", int((got.isnan() != want.isnan()).sum()))
    inf = want.isinf()
    assert torch.equal(got.isinf(), inf) and torch.equal(got[inf], want[inf]), (what, "infinity mismatch")
    ok = torch.isfinite(want)
    r = torch.where(ok, (got - want).abs() / b, torch.zeros_like(got))
    worst = float(r.max()) if r.numel() else 0.0
    at = tuple(int(i) for i in np.unravel_index(int(r.argmax()), tuple(r.shape))) if r.numel() else ()
    WORST[what] = max(WORST.get(what, 0.0), worst)
    print("%-24s worst err/bar %.3f at %s" % (what, worst, at))
    assert worst <= 1.0, (what, worst, at, float(got[at]), float(want[at]), float(b[at]))


def check_scalar(what, got, want, b):
    check(what, torch.tensor([float(got)], dtype=f64), torch.tensor([float(want)], dtype=f64),
          torch.tensor([float(b)], dtype=f64))


# ---- row copies ------------------------------------------------------------------------------------------------------
def masks(B, T, M, seed):
    """[B, T] bool with M masked frames per row; row 0 masks frame 0 and row B - 1 frame T - 1."""
    rng = np.random.RandomState(seed)
    mask = np.zeros((B, T), bool)
    for b in range(B):
        pick = rng.choice(T, M, replace=False)
        forced = 0 if b == 0 else T - 1 if b == B - 1 else None
        if forced is not None and forced not in pick:
            pick[0] = forced
        mask[b, pick] = True
    idx = torch.nonzero(torch.from_numpy(mask))[:, 1].view(B, M)
    inv = torch.full((B, T), -1, dtype=i32)
    for b in range(B):
        inv[b, idx[b]] = torch.arange(M, dtype=i32)
    return torch.from_numpy(mask).to(DEV), idx.to(DEV, i32), inv.to(DEV)


def run_rows(B, T, M, D, seed):
    mask, idx, inv = masks(B, T, M, seed)
    g = gen(seed)
    x = randn(B, T, D, g=g)
    x.view(-1)[::7] = -0.0
    emb = randn(D, g=g)
    out = {}
    out["mask"] = o = nanf(B, T, D)
    call("eb_w2v_mask_fwd", x, emb, inv, o, B * T, D)
    want = x.clone()
    want[mask] = emb
    assert same_bits(o, want), "mask_fwd"
    out["keep"] = o = nanf(B, T, D)
    call("eb_w2v_keep_rows", x, inv, o, B * T, D)
    want = x.clone()
    want[mask] = 0.0
    assert same_bits(o, want), "keep_rows"
    out["gather"] = o = nanf(B, M, D)
    call("eb_w2v_gather", x, idx, o, B, T, M, D)
    assert same_bits(o, x[mask].view(B, M, D)), "gather"
    src = randn(B, M, D, g=g)
    out["scatter"] = o = nanf(B, T, D)
    call("eb_w2v_scatter", src, inv, o, B, T, M, D)
    want = torch.zeros(B, T, D, device=DEV)
    want[mask] = src.view(-1, D)
    assert same_bits(o, want), "scatter"
    return out


@pytest.mark.parametrize("B,T,M,D", ROW_CASES)
def test_row_copies_bitwise(B, T, M, D):
    run_rows(B, T, M, D, 11 + T)


# ---- sq_mean, scale ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SQ_N)
def test_sq_mean(n):
    x = randn(n, g=gen(n), scale=3.0)
    out = nanf(1)
    call("eb_w2v_sq_mean", x, n, out)
    want, b = rs.sq_mean(x)
    check_scalar("sq_mean", out[0], want, b)


@pytest.mark.parametrize("n", [1, 1000, 2 * 1024 * 1024 + 77])
def test_scale_bitwise(n):
    g = gen(n)
    x = randn(n, g=g)
    gs = randn(1, g=g)
    alpha = 2.0 / 3.0 / n
    out = nanf(n)
    call("eb_w2v_scale", x, gs, alpha, n, out)
    assert same_bits(out, rs.scale(x, gs, alpha))
    call("eb_w2v_scale", x, gs, alpha, 0, out)              # n = 0: nothing launched, nothing written
    assert same_bits(out, rs.scale(x, gs, alpha))


# ---- quant_fwd -------------------------------------------------------------------------------------------------------
def quant_inputs(N, G, V, vd, seed):
    g = gen(seed)
    l = randn(N, G * V, g=g, scale=3.0)
    lv = l.view(N, G, V)
    if N >= 5:
        lv[0, 0] = 0.5                                        # all equal: k0 = 0
        if V > 1:
            lv[1, 0, min(3, V - 1)] = lv[1, 0, V - 1] = 20.0  # tie across lanes (or one lane at V = 4, 33)
        if V > 35:
            lv[2, 0, 3] = lv[2, 0, 35] = 20.0                 # tie within lane 3
        lv[4] *= 10.0                                         # a wide row: large |d|
    noise = -torch.empty(N, G * V, device=DEV).exponential_(generator=g).log()
    if N >= 4:
        noise.view(N, G, V)[3, 0] = 1.0 - lv[3, 0]            # z nearly equal: ties in s
    vars = torch.rand(G * V, vd, generator=g, device=DEV)
    return l, noise, vars


def run_quant(l, noise, vars, G, tau):
    N, GV = l.shape
    V, vd = GV // G, vars.shape[1]
    o = dict(q=nanf(N, G * vd), p=nanf(N, GV), s=nanf(N, GV), X=nanf(N, GV), k0=negi(N, G), k=negi(N, G),
             st=nanf(N, G))
    call("eb_w2v_quant_fwd", l, noise, vars, N, G, V, vd, tau, o["q"], o["p"], o["s"], o["X"], o["k0"], o["k"],
         o["st"])
    return o


def check_quant(l, noise, vars, G, tau, o, tag=""):
    N, GV = l.shape
    V, vd = GV // G, vars.shape[1]
    want = rs.quant_fwd(l, noise, vars, G, tau)
    assert torch.equal(o["k0"].long(), want["k0"].long()), "k0: the lane argmax"
    fin = torch.isfinite(l.view(N, G, V)).all(-1)
    assert torch.equal(o["k0"].long()[fin], l.view(N, G, V).argmax(-1)[fin]), "k0: the first-index argmax"
    check("quant p" + tag, o["p"], want["p"], want["p_bar"])
    grp = torch.arange(G, device=DEV)[None]
    vg = vars.view(G, V, vd)
    if noise is None:
        assert torch.equal(o["k"], o["k0"]), "eval: k = k0"
        assert same_bits(o["st"], torch.ones(N, G, device=DEV)), "eval: st = 1"
        assert o["s"].isnan().all(), "eval: s is not written"
        k, st = o["k0"].long(), o["st"]
    else:
        check("quant s" + tag, o["s"], want["s"], want["s_bar"])
        s32 = o["s"].view(N * G, V)
        k = o["k"].long()
        assert torch.equal(k.view(-1).cpu(), rs.lane_arg(s32.cpu().numpy())), "k: the lane argmax of the kernel's s"
        assert torch.equal(k.view(-1), s32.argmax(-1)), "k: the first-index argmax of the kernel's s"
        clear = want["gap"] > want["gap_bar"]
        assert torch.equal(k[clear], want["k"][clear]), "k: the fp64 argmax where the gap is above the bar"
        sk = s32.gather(-1, k.view(-1, 1)).view(N, G)
        st = o["st"]
        assert same_bits(st, (1 - sk) + sk), "st = (1 - s_k) + s_k in fp32"
    # a group with a NaN logit leaves the lanes disagreeing on the index: X and q are pinned where none is NaN
    X = torch.zeros(N, G, V, device=DEV)
    X.scatter_(-1, k[..., None], st[..., None])
    assert same_bits(o["X"].view(N, G, V)[fin], X[fin]), "X"
    vk = vg[grp, k]                                           # [N, G, vd]
    q = vk if noise is None else st[..., None] * vk
    assert same_bits(o["q"].view(N, G, vd)[fin], q[fin]), "q"
    return want


@pytest.mark.parametrize("noisy", [True, False])
@pytest.mark.parametrize("N,G,V,vd", QUANT_CASES)
def test_quant_fwd(N, G, V, vd, noisy):
    l, noise, vars = quant_inputs(N, G, V, vd, 100 + V)
    noise = noise if noisy else None
    o = run_quant(l, noise, vars, G, 1.7)
    check_quant(l, noise, vars, G, 1.7, o)


def test_quant_fwd_nan_logits():
    """NaN logits: p NaN over the group, k0 where the lane map ends, the other groups untouched."""
    N, G, V, vd = 4, 2, 70, 4
    l, noise, vars = quant_inputs(N, G, V, vd, 7)
    lv = l.view(N, G, V)
    lv[0, 0, 0] = NAN                                        # lane 0's first element: sticks, and lane 0 wins
    lv[1, 0, 37] = NAN                                       # lane 5's second element: skipped
    lv[2, 0, 5] = NAN                                        # lane 5's first element: sticks in lane 5 only
    lv[2, 0, 40] = 50.0
    lv[3, 0, 69] = NAN
    lv[3, 0, 0] = 50.0
    for nz in (noise, None):
        o = run_quant(l, nz, vars, G, 1.7)
        check_quant(l, nz, vars, G, 1.7, o, " nan")
        assert o["p"].view(N, G, V)[:, 0].isnan().all() and not o["p"].view(N, G, V)[:, 1].isnan().any()
    assert o["k0"][:, 0].tolist() == [0, int(lv[1, 0].nan_to_num(-1e30).argmax()), 40, 0]


# ---- quant_stats -----------------------------------------------------------------------------------------------------
def stats_inputs(N, G, V, seed):
    g = gen(seed)
    p = torch.softmax(randn(N, G, V, g=g, scale=2.0), -1)
    p[:, :, :: 3] = 0.0                                      # psum columns exactly 0 (a = 0)
    psum = p.sum(0).reshape(-1).contiguous()
    k0 = torch.randint(0, V, (N, G), generator=g, device=DEV, dtype=i32)
    k0[k0 == V // 2] = 0                                     # columns never chosen
    return psum, k0


def run_stats(psum, k0, N, G, V):
    o = dict(out=nanf(2), coef=nanf(G * V), counts=negi(G * V))
    call("eb_w2v_quant_stats", psum, k0, N, G, V, o["out"], o["coef"], o["counts"])
    return o


def check_stats(psum, k0, N, G, V, o):
    want = rs.quant_stats(psum, k0, N, G, V)
    assert torch.equal(o["counts"].long(), want["counts"]), "counts"
    check_scalar("stats prob_ppl", o["out"][0], want["pp"], want["pp_bar"])
    check_scalar("stats code_ppl", o["out"][1], want["cp"], want["cp_bar"])
    check("stats coef", o["coef"], want["coef"], want["coef_bar"])


@pytest.mark.parametrize("N,G,V", STATS_CASES)
def test_quant_stats(N, G, V):
    psum, k0 = stats_inputs(N, G, V, 200 + N)
    assert (psum == 0).any()
    check_stats(psum, k0, N, G, V, run_stats(psum, k0, N, G, V))


# ---- quant_bwd -------------------------------------------------------------------------------------------------------
def run_qbwd(ds, s, p, coef, gppl, N, G, V, tau):
    dl = nanf(N, G * V)
    call("eb_w2v_quant_bwd", ds, s, p, coef, gppl, N, G, V, tau, dl)
    return dl


def qbwd_inputs(N, G, V, seed):
    """The kernel's own s, p (quant_fwd) and coef (quant_stats), a dense dsoft and g_ppl."""
    l, noise, vars = quant_inputs(N, G, V, 2, seed)
    o = run_quant(l, noise, vars, G, 1.7)
    psum = o["p"].sum(0).contiguous()
    coef = run_stats(psum, o["k0"], N, G, V)["coef"]
    g = gen(seed + 1)
    return randn(N, G * V, g=g), o["s"], o["p"], coef, torch.tensor([-2.5], device=DEV)


@pytest.mark.parametrize("mode", ["dsoft", "g_ppl", "both"])
@pytest.mark.parametrize("N,G,V", BWD_CASES)
def test_quant_bwd(N, G, V, mode):
    ds, s, p, coef, gppl = qbwd_inputs(N, G, V, 300 + V)
    ds = ds if mode != "g_ppl" else None
    gppl = gppl if mode != "dsoft" else None
    dl = run_qbwd(ds, s, p, coef, gppl, N, G, V, 1.7)
    want, b = rs.quant_bwd(ds, s, p, coef, gppl, N, G, V, 1.7)
    check("quant_bwd " + mode, dl, want, b)


# ---- normalize + logits_fwd, logits_bwd ------------------------------------------------------------------------------
def logits_inputs(B, M, D, K, seed):
    g = gen(seed)
    xp, yp = randn(B, M, D, g=g), randn(B, M, D, g=g)
    neg = torch.randint(0, M, (B, M, K), generator=g, device=DEV, dtype=i32)
    neg[0, 1 % M, 0] = 1 % M                                 # neg == m
    if M >= 8:
        yp[0, 5] = yp[0, 3]                                  # equal rows: masked both ways
        neg[0, 3, 0], neg[0, 5, K - 1] = 5, 3
        yp[B - 1, 7] = -yp[B - 1, 2]                         # a row's negation is not equal
        neg[B - 1, 2, 0] = 7
        xp[0, 1] = 0.0                                       # zero rows
        yp[0, 2] = 0.0
        xp[B - 1, 4] *= 1e-12                                # below eps: the clamp
        yp[B - 1, 6] *= 1e-12
    return xp, yp, neg


def run_lfwd(xp, yp, neg, temp=TEMP):
    B, M, D = xp.shape
    K = neg.shape[-1]
    o = dict(xh=nanf(B, M, D), yh=nanf(B, M, D), xn=nanf(B, M), yn=nanf(B, M), cos=nanf(K + 1, B, M),
             logits=nanf(K + 1, B, M))
    call("eb_w2v_logits_fwd", xp, yp, neg, B, M, D, K, temp, EPS, o["xh"], o["yh"], o["xn"], o["yn"], o["cos"],
         o["logits"])
    return o


def check_lfwd(xp, yp, neg, o, temp=TEMP):
    for r, h, n, t in ((xp, "xh", "xn", "x"), (yp, "yh", "yn", "y")):
        wh, bh, wn, bn = rs.normalize(r, EPS)
        check("normalize %sn" % t, o[n], wn, bn)
        check("normalize %sh" % t, o[h], wh, bh)
    cos, cb, lo, lb = rs.logits_fwd(o["xh"], o["yh"], yp, neg, temp)
    check("logits_fwd cos", o["cos"], cos, cb)
    check("logits_fwd logits", o["logits"], lo, lb)
    return lo.isinf()


@pytest.mark.parametrize("B,M,D,K", FWD_CASES)
def test_logits_fwd(B, M, D, K):
    xp, yp, neg = logits_inputs(B, M, D, K, 400 + D)
    masked = check_lfwd(xp, yp, neg, run_lfwd(xp, yp, neg))
    assert masked[1:, 0, 1 % M].any()                        # neg == m is masked
    if M >= 8:
        assert masked[1, 0, 3] and masked[K, 0, 5] and not masked[1, B - 1, 2]


def run_lbwd(dlog, f, xp, yp, neg, temp=TEMP):
    B, M, D = xp.shape
    K = neg.shape[-1]
    o = dict(A=nanf(B, M, M), AC=nanf(B, M, M), dx=nanf(B, M, D), dy=nanf(B, M, D))
    call("eb_w2v_logits_bwd", dlog, f["cos"], neg, f["xh"], f["yh"], xp, yp, f["xn"], f["yn"], B, M, D, K,
         temp, EPS, o["A"], o["AC"], o["dx"], o["dy"])
    return o


def check_lbwd(dlog, f, xp, yp, neg, o, temp=TEMP):
    masked = f["logits"].isinf()
    assert torch.equal(f["cos"].isinf(), masked)
    A, bA, AC, bAC = rs.logits_a(dlog, f["cos"], neg, masked)
    check("logits_bwd A", o["A"], A, bA)
    check("logits_bwd AC", o["AC"], AC, bAC)
    dx, bx, dy, by = rs.logits_bwd(o["A"], o["AC"], f["xh"], f["yh"], xp, yp, f["xn"], f["yn"], temp, EPS)
    check("logits_bwd dxp", o["dx"], dx, bx)
    check("logits_bwd dyp", o["dy"], dy, by)


@pytest.mark.parametrize("D", BWDL_D)
def test_logits_bwd(D):
    B, M, K = 2, 20, 30
    xp, yp, neg = logits_inputs(B, M, D, K, 500 + D)
    f = run_lfwd(xp, yp, neg)
    dlog = randn(K + 1, B, M, g=gen(D))
    check_lbwd(dlog, f, xp, yp, neg, run_lbwd(dlog, f, xp, yp, neg))


def test_masked_candidates_pass_no_gradient():
    """A dense upstream gradient, nonzero at every masked candidate: A / AC leave them out, and dxp / dyp are bit for
    bit those of the same gradient with the masked entries zeroed."""
    B, M, D, K = 2, 20, 600, 30
    xp, yp, neg = logits_inputs(B, M, D, K, 77)
    f = run_lfwd(xp, yp, neg)
    masked = f["logits"].isinf()
    assert int(masked.sum()) >= 4
    dlog = randn(K + 1, B, M, g=gen(78)) + 3.0
    assert (dlog[masked] != 0).all()
    o = run_lbwd(dlog, f, xp, yp, neg)
    check_lbwd(dlog, f, xp, yp, neg, o)
    z = run_lbwd(torch.where(masked, torch.zeros_like(dlog), dlog), f, xp, yp, neg)
    for k in ("A", "AC", "dx", "dy"):
        assert same_bits(o[k], z[k]), k


# ---- ce --------------------------------------------------------------------------------------------------------------
def ce_inputs(C, B, M, seed):
    lo = randn(C, B, M, g=gen(seed), scale=5.0)

    def row(i):
        m, b = divmod(i, B)
        return lo[:, b, m]
    n = B * M
    if n >= 6:
        row(0).fill_(0.25)                                   # all equal: argmax and argmin 0, not correct
        r = row(1)
        r[0] = r[C - 1] = 20.0                               # a tie for the maximum with candidate 0: correct
        r = row(2)
        r[0] = r[1] = -20.0                                  # a tie for the minimum with candidate 0
        if C > 2:
            r = row(3)
            r[0] = 30.0
            r[1:min(4, C - 1) + 1] = -math.inf               # -inf negatives
            r = row(4)
            r[1:] = 0.0
            r[0] = 1.0                                       # others all equal: argmin 1
            r = row(5)
            r[1] = r[C - 1] = 40.0                           # a tie for the maximum without candidate 0
    return lo


def run_ce(lo):
    C, B, M = lo.shape
    o = dict(grad=nanf(C, B, M), out=nanf(2))
    call("eb_w2v_ce", lo, B, M, C, o["grad"], o["out"])
    return o


def check_ce(lo, o):
    want = rs.ce(lo)
    check("ce grad", o["grad"], want["grad"], want["grad_bar"])
    check_scalar("ce loss", o["out"][0], want["loss"], want["loss_bar"])
    assert float(o["out"][1]) == want["correct"], (float(o["out"][1]), want["correct"])
    return want


@pytest.mark.parametrize("C,B,M", CE_CASES)
def test_ce(C, B, M):
    lo = ce_inputs(C, B, M, 600 + C + M)
    want = check_ce(lo, run_ce(lo))
    if B * M >= 6:
        rows = lo.permute(2, 1, 0).reshape(B * M, C)
        assert 0 < want["correct"] < B * M or B * M < 32
        assert rows[1].argmax() == 0 and rows[0].argmax() == 0 and rows[0].argmin() == 0


# ---- the cli model's head shapes -------------------------------------------------------------------------------------
_CLI = {}


def cli_shapes():
    """cli/pretrain_wav2vec.py's model (test_gpu_wav2vec.py's test_cli_shape_against_the_oracle) on 24 utterances of
    14 s: T frames, M masked frames per utterance, embed and final dims."""
    if not _CLI:
        from edgedict_b200.rnnt import wav2vec as w2v
        from tests.test_gpu_wav2vec import CLI_FE
        torch.manual_seed(0)
        m = w2v.Wav2Vec(frontend_params=CLI_FE, front_bias=False, quantize_input=False, quantize_targets=True,
                        input_size=128, enc_hidden_size=512, enc_layers=4, enc_dropout=0.1, enc_proj_size=512,
                        num_negatives=100)
        B, T = 24, m.frontend.output_length(14 * 16000)
        np.random.seed(3)
        mask = w2v.compute_mask_indices((B, T), None, m.mask_prob, m.mask_length, m.mask_selection, m.mask_other,
                                        min_masks=2, min_space=m.mask_min_space)
        torch.manual_seed(4)
        M = int(mask[0].sum())
        neg = w2v.sample_negative_indices(B, M, 100).view(B, M, 100)
        _CLI.update(B=B, T=T, M=M, C=128, D=m.final_proj.out_features, G=m.quantizer.groups,
                    V=m.quantizer.num_vars, vd=m.quantizer.vars.shape[-1], K=100, neg=neg.to(DEV, i32))
    return _CLI


def test_cli_head_shapes():
    c = cli_shapes()
    B, T, M, D, G, V, vd, K = (c[k] for k in ("B", "T", "M", "D", "G", "V", "vd", "K"))
    assert (B, D, G, V, K) == (24, 128, 2, 320, 100)          # final_dim defaults to the 128-wide embedding
    print("cli head: B %d T %d M %d N %d vd %d" % (B, T, M, B * M, vd))
    run_rows(B, T, M, c["C"], 21)
    run_rows(B, T, M, D, 22)
    x = randn(B * T * c["C"], g=gen(23))
    out = nanf(1)
    call("eb_w2v_sq_mean", x, x.numel(), out)
    check_scalar("sq_mean cli", out[0], *rs.sq_mean(x))
    N = B * M
    l, noise, vars = quant_inputs(N, G, V, vd, 24)
    o = run_quant(l, noise, vars, G, 1.9)
    check_quant(l, noise, vars, G, 1.9, o, " cli")
    psum = o["p"].sum(0).contiguous()
    st = run_stats(psum, o["k0"], N, G, V)
    check_stats(psum, o["k0"], N, G, V, st)
    ds = randn(N, G * V, g=gen(25))
    gp = torch.tensor([0.7], device=DEV)
    dl = run_qbwd(ds, o["s"], o["p"], st["coef"], gp, N, G, V, 1.9)
    check("quant_bwd cli", dl, *rs.quant_bwd(ds, o["s"], o["p"], st["coef"], gp, N, G, V, 1.9))
    g = gen(26)
    xp, yp, neg = randn(B, M, D, g=g), randn(B, M, D, g=g), c["neg"]
    f = run_lfwd(xp, yp, neg)
    check_lfwd(xp, yp, neg, f)
    ce = run_ce(f["logits"])
    check_ce(f["logits"], ce)
    lb = run_lbwd(ce["grad"], f, xp, yp, neg)
    check_lbwd(ce["grad"], f, xp, yp, neg, lb)


# ---- bitwise invariants ----------------------------------------------------------------------------------------------
def test_repeated_launches_are_bitwise_equal():
    c = cli_shapes()
    B, M, D, G, V, vd = (c[k] for k in ("B", "M", "D", "G", "V", "vd"))
    runs = []
    for _ in range(2):
        r = run_rows(4, 1000, 900, 640, 31)
        x = randn(3_000_001, g=gen(32))
        out = nanf(1)
        call("eb_w2v_sq_mean", x, x.numel(), out)
        r["sq"] = out
        l, noise, vars = quant_inputs(B * M, G, V, vd, 33)
        q = run_quant(l, noise, vars, G, 1.9)
        r.update({"q" + k: v for k, v in q.items()})
        st = run_stats(q["p"].sum(0).contiguous(), q["k0"], B * M, G, V)
        r.update({"st" + k: v for k, v in st.items()})
        r["dl"] = run_qbwd(l, q["s"], q["p"], st["coef"], torch.tensor([0.7], device=DEV), B * M, G, V, 1.9)
        xp, yp, neg = randn(B, M, D, g=gen(34)), randn(B, M, D, g=gen(35)), c["neg"]
        f = run_lfwd(xp, yp, neg)
        r.update({"f" + k: v for k, v in f.items()})
        ce = run_ce(f["logits"])
        r.update({"ce" + k: v for k, v in ce.items()})
        r.update({"b" + k: v for k, v in run_lbwd(ce["grad"], f, xp, yp, neg).items()})
        runs.append(r)
    for k in runs[0]:
        assert same_bits(runs[0][k], runs[1][k]), k


def test_rows_are_independent_of_the_batch():
    """Per-row outputs of normalize, logits_fwd, quant_fwd / bwd and CE's gradient, and dxp / dyp of one utterance, are
    the same bits alone and inside the batch."""
    c = cli_shapes()
    B, M, D, G, V, vd = (c[k] for k in ("B", "M", "D", "G", "V", "vd"))
    N = B * M
    l, noise, vars = quant_inputs(N, G, V, vd, 41)
    q = run_quant(l, noise, vars, G, 1.9)
    coef = run_stats(q["p"].sum(0).contiguous(), q["k0"], N, G, V)["coef"]
    ds = randn(N, G * V, g=gen(42))
    gp = torch.tensor([0.7], device=DEV)
    dl = run_qbwd(ds, q["s"], q["p"], coef, gp, N, G, V, 1.9)
    sl = slice(37, 37 + 50)
    q1 = run_quant(l[sl].contiguous(), noise[sl].contiguous(), vars, G, 1.9)
    for k in ("q", "p", "s", "X", "k0", "k", "st"):
        assert same_bits(q1[k], q[k][sl]), "quant_fwd " + k
    # g_ppl / N is formed from the call's N: pass the batch's N so the rows' arithmetic is the same
    dl1 = torch.full((50, G * V), NAN, device=DEV)
    call("eb_w2v_quant_bwd", ds[sl].contiguous(), q1["s"], q1["p"], coef, None, 50, G, V, 1.9, dl1)
    dl0 = run_qbwd(ds, q["s"], q["p"], coef, None, N, G, V, 1.9)
    assert same_bits(dl1, dl0[sl]), "quant_bwd (dsoft) rows"
    assert not same_bits(dl0, dl)
    xp, yp, neg = randn(B, M, D, g=gen(43)), randn(B, M, D, g=gen(44)), c["neg"]
    f = run_lfwd(xp, yp, neg)
    ce = run_ce(f["logits"])
    lb = run_lbwd(ce["grad"], f, xp, yp, neg)
    b = 5
    one = lambda t: t[b:b + 1].contiguous()                  # noqa: E731
    f1 = run_lfwd(one(xp), one(yp), one(neg))
    for k in ("xh", "yh", "xn", "yn"):
        assert same_bits(f1[k], f[k][b:b + 1]), "normalize " + k
    for k in ("cos", "logits"):
        assert same_bits(f1[k], f[k][:, b:b + 1]), "logits_fwd " + k
    ce1 = run_ce(f1["logits"])
    assert same_bits(ce1["grad"], ce["grad"][:, b:b + 1]), "ce grad"
    lb1 = run_lbwd(ce1["grad"], f1, one(xp), one(yp), one(neg))
    for k in ("A", "AC", "dx", "dy"):
        assert same_bits(lb1[k], lb[k][b:b + 1]), "logits_bwd " + k


# ---- reach -----------------------------------------------------------------------------------------------------------
def test_reach():
    """The case tables reach every loop trip count and branch named in the error model."""
    cap = grid_cap()
    assert any(B * M * D >= 2 * cap and B * T * D >= 2 * cap for B, T, M, D in ROW_CASES)   # two grid-stride trips
    assert {1, 33} <= {D for *_, D in ROW_CASES} and any(M == T for _, T, M, _ in ROW_CASES)
    assert any(M == 1 for _, _, M, _ in ROW_CASES)
    assert any(n < 1024 for n in SQ_N) and any(n % 1024 == 0 for n in SQ_N) and any(n % 1024 == 1 for n in SQ_N)
    assert max(SQ_N) > 1024 * 1024
    Vs = {V for _, _, V, _ in QUANT_CASES}
    assert {1, 31, 32, 33, 320, 1100} <= Vs and {G for _, G, _, _ in QUANT_CASES} == {1, 2, 4}
    assert any(N * G > 1024 for N, G, V in STATS_CASES) and any(G * V > 1024 for N, G, V in STATS_CASES)
    assert any(V > 1024 for _, _, V in STATS_CASES)
    assert {1, 33, 320, 1100} <= {V for _, _, V in BWD_CASES}
    assert {1, 31, 32, 33, 512, 513, 640, 1030} <= {D for _, _, D, _ in FWD_CASES}
    assert {1, 100} <= {K for *_, K in FWD_CASES}
    passes = {-(-D // 512) for D in BWDL_D}                   # logits_bwd's 512-column passes
    assert passes >= {1, 2, 3, 4}
    assert all(any(D == k * 512 + e for D in BWDL_D) for k in (1, 2) for e in (-1, 0, 1))
    assert {2, 33, 101} <= {C for C, _, _ in CE_CASES}
    assert {1, 31, 32, 33} <= {B * M for _, B, M in CE_CASES} and max(B * M for _, B, M in CE_CASES) >= 10000
