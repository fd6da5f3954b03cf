"""Per-element fp64 parity and bitwise invariants of the raw-waveform front end's kernels (csrc/conv.cu) and of the GEMM
entries its backward uses, each through its C entry point.

    eb_conv1d_bf16          conv_tc_kernel<BN, BKC>: all nine tile configurations (BN = 128 / 32 / 16 by N, BKC =
                            64 / 32 / 16 by C), strides 1 ... 5, 1 ... 10 taps, the dX phase form (s = 1, row0 < 0), a
                            persistent grid with >= 3 tiles per CTA, tiles that change column, reads past x_rows
    eb_gn_stats / _apply    per-utterance GELU statistics and the padded, normalised conv operand (fp32 and bf16)
    eb_gn_bwd               the GroupNorm + GELU backward: dgamma / dbeta / db partials, dy and / or dy16
    eb_conv1d_first_fwd/_dw the first layer (C_in = 1)
    eb_gemm_f32_splitk      the fp32 weight-gradient GEMM of the strided convs, its slices summed by eb_colsum
    eb_gemm_bf16            at the bf16 dW layout of functional.FrontEndStack (MN-major dY, overlapping xp rows)

Error model.  bf16 operands are drawn as bf16, so they are exact in fp64 and every bf16 x bf16 product is exact in fp32.
  conv1d_bf16   the raw product P (no bias) against the exact convolution S of the bf16 operands (fp64):
                |P - S| <= taps C UTC (|X| * |W|) + TINY, UTC = 2^-23 per tensor-core add.  Bitwise: P + bias =
                fp32(P + bias); a negative row0 equals the same call on a buffer with those zero rows written in front;
                rows [m0, M) equal the call on the view advanced by m0 operand rows (by m0 + row0 rows with row0 = 0
                when row0 < 0: the rows above then hold data, not zeros); repeated launches; a 128-wide W
                equals four 32-wide and eight 16-wide slices (m64n128 / m64n32 / m64n16 accumulate alike).
  GELU          exact in fp64 (erf).  The kernel's fp32 GELU 0.5 x (1 + erff(x / sqrt 2)) is off by at most
                0.5 |x| (2^-22 + 3 U24) + U24 |g| (erff 2 ulp, the argument's and the sum's roundings, the product's);
                its derivative Phi(x) + x phi(x) by 0.5 (2^-22 + 3 U24) + |x| phi(x) (2^-22 + (x^2 / 2 + 3) U24)
                + U24 |g'| (expf 2 ulp, the rounded argument -x^2 / 2 scaled by exp, three roundings).
  gn_stats      fp64 partial sums of the fp32 GELU: mean within sum dg / n + U24 |mean|, the variance within
                sum 2 |g - mean| dg / n plus the fp64 summation (E[g^2] - E[g]^2 in fp64 holds at mean / std ~ 1e3),
                rstd within half the variance's relative error + U24.
  gn_apply      teacher-forced on the kernel's mean / rstd: (g - mean) rstd gamma + beta, four roundings and dg; the
                padding rows exactly 0; the bf16 output bitwise bf16_rn of the fp32 output; gamma = beta = None
                bitwise gamma = 1, beta = 0.
  gn_bwd        teacher-forced on the kernel's mean / rstd: dy = rstd (dz gamma - S1/n - xh S2/n) GELU'(y), with the
                errors of xh, of the fp64 sums S1, S2 (from the fp32 xh) and of GELU' propagated, plus five roundings;
                dgamma, dbeta, db: the chains over a split plus the row lanes and the slice sum, n_add = rows per split
                + slices + 16 at U24, the totals taken in eb_colsum's order (`_colsum_order`) from the kernel's own
                partials; dy16 bitwise bf16_rn(dy); dy the same bits with or without dy16; rows t >= T of the dy
                buffers untouched.
  first layer   forward an fmaf chain of k terms from the bias: k U24 (|b| + sum |w x|); dW / db the chain over a
                split and the split reduction, (rows per split + splits + 8) U24 sum |dy x|, and ops.conv1d_first_dw
                bitwise `_colsum_order` of the kernel's partials.
  f32 split-K   every slice bitwise eb_gemm_f32 over its k range; the total within (kchunk + slices + 8) U24 (|A| @ |B|)
                and ops.gemm_f32_rows bitwise `_colsum_order` of the slices.
  bf16 dW       test_gpu_gemm_fp64's bar: (K + splits) UTC (|A| @ |B|).

Every output goes into a NaN-prefilled buffer with a guard row (or guard columns) behind it, inputs that must not be
read are NaN, and every bar-based check prints its worst err/bar (pytest -s); DESIGN.md section 2 records the measured
figures."""
import math

import pytest
import torch

from tests.test_gpu_gemm_fp64 import TINY, U24, UTC, _n_add, _plan, _report, _same
from tests.test_gpu_glue_fp64 import _colsum_order

pytestmark = pytest.mark.gpu

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
NAN = float("nan")
U22 = 2.0 ** -22          # 2 ulp relative: erff, expf
SENT = -7.0               # sentinel of buffers a kernel must leave alone


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


def _ok(st, name):
    assert st == 0, "%s: status %d" % (name, st)
    torch.cuda.synchronize()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---- eb_conv1d_bf16 ---------------------------------------------------------------------------------------------------
def _tile(N, C):
    bn = 128 if N % 128 == 0 else (32 if N % 32 == 0 else 16)
    return bn, 64 if C % 64 == 0 else (32 if C % 32 == 0 else 16)


def _conv_call(name, x16, x_rows, s, C, row0, w16, taps, N, M, bias=None, ldc=None, col0=0, x_off=0):
    """One eb_conv1d_bf16 into a NaN-filled [M + 1, ldc] buffer at column col0; checks that nothing outside rows
    [0, M) x columns [col0, col0 + N) was written and returns that block."""
    ldc = ldc or N
    buf = torch.full((M + 1, ldc), NAN, device=DEV)
    _ok(_lib().eb_conv1d_bf16(x16.data_ptr() + 2 * x_off, x_rows, s, C, row0, _p(w16), taps, N, _p(bias),
                              buf.data_ptr() + 4 * col0, ldc, M, _stream()), name)
    assert bool(torch.isnan(buf[M]).all()), name + ": a store past the last row"
    assert bool(torch.isnan(buf[:, :col0]).all()) and bool(torch.isnan(buf[:, col0 + N:]).all()), \
        name + ": a store outside the written columns"
    return buf[:M, col0:col0 + N]


def _conv_ref(x16, x_rows, s, C, row0, w16, taps, M):
    """(S, |X| * |W|) in fp64: out[m, n] = sum_j sum_c X[m + row0 + j // s, j % s, c] W[n, j C + c], zero outside
    [0, x_rows)."""
    X = x16[:x_rows * s * C].view(x_rows, s, C).double()
    lo = max(0, -row0)
    hi = max(0, M + row0 + (taps - 1) // s - x_rows)
    Xp = torch.zeros(lo + x_rows + hi, s, C, dtype=f64, device=DEV)
    Xp[lo:lo + x_rows] = X
    m = torch.arange(M, device=DEV)
    A = torch.cat([Xp[m + row0 + j // s + lo, j % s] for j in range(taps)], 1)
    W = w16.double()
    return A @ W.t(), A.abs() @ W.abs().t()


def _conv_case(name, nsm):
    """name -> (M, N, C, s, taps, row0, x_rows or None (all rows the conv reads), ldc or None, col0)."""
    many = BM_CONV * 3 * nsm + 77                              # >= 3 tiles per CTA at 128-wide tiles
    return {
        "bn128-bkc64-s2-t3": (517, 128, 128, 2, 3, 0, None, None, 0),
        "bn128-bkc32-s5-t10": (129, 128, 32, 5, 10, 0, None, None, 0),
        "bn128-bkc16-s4-t8": (63, 256, 16, 4, 8, 0, None, None, 0),
        "bn32-bkc64-s3-t2": (64, 32, 64, 3, 2, 0, None, None, 0),                       # taps < s
        "bn32-bkc32-dx-t4": (65, 96, 32, 1, 4, -3, None, 3 * 96, 96),                  # dX phase, dxp layout
        "bn32-bkc16-M1": (1, 32, 48, 1, 1, 0, None, None, 0),
        "bn16-bkc64-s4-t1": (255, 48, 192, 4, 1, 0, None, None, 0),                     # M % 128 = 127
        "bn16-bkc32-cut": (257, 16, 96, 2, 9, 0, 200, None, 0),                         # M % 128 = 1, TMA zero fill
        "bn16-bkc16-dx-t2": (200, 80, 16, 1, 2, -1, None, 2 * 80, 80),
        "many-bn128-bkc64": (many, 128, 128, 2, 3, 0, None, None, 0),
        # 5 / 7 column tiles: with the grid at #SMs a CTA's tiles change column (checked below)
        "many-cols-bn32-bkc32-dx-cut": (BM_CONV * _cdiv(3 * nsm, 5) + 5, 160, 32, 1, 7, -6,
                                        BM_CONV * _cdiv(3 * nsm, 5) - 50, 2 * 160, 160),
        "many-cols-bn16-bkc16-s5-t6": (BM_CONV * _cdiv(3 * nsm, 7) - 3, 112, 16, 5, 6, 0, None, None, 0),
    }[name]


BM_CONV = 128
CONV_CASES = ["bn128-bkc64-s2-t3", "bn128-bkc32-s5-t10", "bn128-bkc16-s4-t8", "bn32-bkc64-s3-t2", "bn32-bkc32-dx-t4",
              "bn32-bkc16-M1", "bn16-bkc64-s4-t1", "bn16-bkc32-cut", "bn16-bkc16-dx-t2", "many-bn128-bkc64",
              "many-cols-bn32-bkc32-dx-cut", "many-cols-bn16-bkc16-s5-t6"]


def _conv_operands(M, N, C, s, taps, row0, x_rows, seed):
    need = max(1, M + row0 + (taps - 1) // s)
    x_rows = x_rows or need
    g = _gen(seed)
    x16 = torch.randn(x_rows * s * C, device=DEV, generator=g).bfloat16()
    w16 = (torch.randn(N, taps * C, device=DEV, generator=g) * 0.2).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)
    return x16, x_rows, w16, bias, need


@pytest.mark.parametrize("name", CONV_CASES)
def test_conv1d_bf16(name):
    nsm = _nsm()
    M, N, C, s, taps, row0, x_rows, ldc, col0 = _conv_case(name, nsm)
    bn, bkc = _tile(N, C)
    tiles = _cdiv(M, BM_CONV) * (N // bn)
    if name.startswith("many"):
        assert tiles >= 3 * nsm, (name, tiles)
    if name.startswith("many-cols"):
        assert N // bn > 1 and nsm % (N // bn) != 0, "the tiles of a CTA must change column"
    x16, x_rows, w16, bias, need = _conv_operands(M, N, C, s, taps, row0, x_rows, M + N + C + taps)
    if "cut" in name:
        assert x_rows < need
    print("  %-30s BN %d, BKC %d, %d tiles over %d CTAs, x_rows %d of %d read" % (name, bn, bkc, tiles,
                                                                                  min(tiles, nsm), x_rows, need))
    P = _conv_call(name, x16, x_rows, s, C, row0, w16, taps, N, M, ldc=ldc, col0=col0)
    S, R = _conv_ref(x16, x_rows, s, C, row0, w16, taps, M)
    _report(name, "raw", P, S, taps * C * UTC * R)
    _same(name + " repeated launch", _conv_call(name, x16, x_rows, s, C, row0, w16, taps, N, M, ldc=ldc, col0=col0), P)
    _same(name + " + bias", _conv_call(name, x16, x_rows, s, C, row0, w16, taps, N, M, bias, ldc, col0), P + bias)
    if row0 < 0:                       # the negative row offset reads zeros: write them in front instead
        z = torch.cat([torch.zeros(-row0 * s * C, dtype=bf16, device=DEV), x16])
        _same(name + " row0 < 0 vs explicit zero rows", _conv_call(name, z, x_rows - row0, s, C, 0, w16, taps, N, M),
              P)
    m0 = M // 3
    if m0 > 0:                         # the view starts at operand row m0 + row0 (row0 < 0: the rows above are real)
        adv, r0 = m0 + min(row0, 0), max(row0, 0)
        _same(name + " rows [%d, M) vs the advanced view" % m0,
              _conv_call(name, x16, x_rows - adv, s, C, r0, w16, taps, N, M - m0, x_off=adv * s * C), P[m0:])
    if N % 128 == 0:                   # the k16 order does not depend on the tile width
        for w in (32, 16):
            for j in range(N // w):
                Pj = _conv_call(name, x16, x_rows, s, C, row0, w16[j * w:(j + 1) * w], taps, w, M)
                _same("%s %d-wide slice %d vs the %d-wide tile" % (name, w, j, bn), Pj, P[:, j * w:(j + 1) * w])


def test_conv1d_bf16_strides_and_taps():
    """s = 1 ... 5 against taps = 1 ... 10 (taps < s included), and at s = 1 the dX phase form row0 = -(taps - 1)."""
    M, N, C = 70, 32, 32
    worst = 0.0
    for s in range(1, 6):
        for taps in range(1, 11):
            for row0 in ((0, -(taps - 1)) if s == 1 and taps > 1 else (0,)):
                name = "sweep s%d t%d row0 %d" % (s, taps, row0)
                x16, x_rows, w16, _, _ = _conv_operands(M, N, C, s, taps, row0, None, 100 * s + taps)
                P = _conv_call(name, x16, x_rows, s, C, row0, w16, taps, N, M)
                S, R = _conv_ref(x16, x_rows, s, C, row0, w16, taps, M)
                err = (P.double() - S).abs()
                r = float((err / (taps * C * UTC * R + TINY)).max())
                assert r <= 1.0, (name, r)
                worst = max(worst, r)
    print("  %-44s worst err/bar %.3g" % ("conv sweep s 1-5 x taps 1-10", worst))


# ---- GELU error model ---------------------------------------------------------------------------------------------------
def _gelu_ref(y):
    """(g, bound on |g_kernel - g|, g', bound on |g'_kernel - g'|) for fp32 y, in fp64."""
    x = y.double()
    e = torch.erf(x / math.sqrt(2.0))
    g = 0.5 * x * (1 + e)
    dg = 0.5 * x.abs() * (U22 + 3 * U24) + U24 * g.abs()
    phi = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    gg = 0.5 * (1 + e) + x * phi
    dgg = 0.5 * (U22 + 3 * U24) + x.abs() * phi * (U22 + (0.5 * x * x + 3) * U24) + U24 * gg.abs()
    return g, dg, gg, dgg


# ---- eb_gn_stats / eb_gn_apply / eb_gn_bwd ----------------------------------------------------------------------------
# (name, B, T, C, k, s, extra rows of ustride, input kind, affine): C = 24 / 40 leave lanes idle, 320 a second, partial
# channel block; T < the row lanes (T = 5 at C = 16, T = 1 at C = 128), >= 3 row splits with a ragged last one (rows per
# split 32768 / C), ustride > T C as the blocks pass it (Q C_out), B = 32; mean / std ~ 1e3; a variance comparable to eps
GN_CASES = [("c16-T5", 3, 5, 16, 3, 2, 0, "normal", True), ("c24-splits", 2, 4196, 24, 3, 2, 7, "normal", False),
            ("c40-offset", 4, 1000, 40, 2, 2, 0, "offset", True), ("c128-B32", 32, 700, 128, 3, 2, 5, "normal", True),
            ("c256-var-eps", 5, 300, 256, 4, 2, 0, "small", True), ("c320-offset", 3, 333, 320, 3, 2, 2, "offset", True),
            ("c512", 2, 150, 512, 2, 2, 1, "normal", False), ("c128-T1", 2, 1, 128, 2, 3, 0, "normal", True)]
EPS = 1e-5


def _gn_inputs(B, T, C, extra, kind, seed):
    """y [B, ustride] (NaN beyond T C), gamma, beta."""
    g = _gen(seed)
    ustride = (T + extra) * C
    y = torch.full((B, ustride), NAN, device=DEV)
    v = torch.randn(B, T * C, device=DEV, generator=g)
    if kind == "offset":
        v = 1e3 + v
    elif kind == "small":
        v = 0.004 * v
    else:
        v = v * (0.5 + torch.rand(B, 1, device=DEV, generator=g)) * 2 + 0.3
    y[:, :T * C] = v
    gamma = 0.5 + torch.rand(C, device=DEV, generator=g)
    beta = torch.rand(C, device=DEV, generator=g) - 0.5
    return y, ustride, gamma, beta


def _rps(C):
    return int(_lib().eb_conv_rows_per_split(C))


def _gn_stats(y, ustride, B, T, C):
    from edgedict_b200 import ops
    dpart = torch.full((ops._gn_slices(B, T, C)[1], 2), NAN, dtype=f64, device=DEV)
    mean, rstd = torch.full((B + 1,), NAN, device=DEV), torch.full((B + 1,), NAN, device=DEV)
    _ok(_lib().eb_gn_stats(_p(y), ustride, B, T, C, _p(dpart), _p(mean), _p(rstd), EPS, _stream()), "eb_gn_stats")
    assert math.isnan(float(mean[B])) and math.isnan(float(rstd[B]))
    return mean[:B], rstd[:B]


def _check_stats(name, y, B, T, C, mean, rstd):
    """mean / rstd against fp64 of the exact GELU; returns (g, dg) [B, T C]."""
    g, dg, _, _ = _gelu_ref(y[:, :T * C])
    n = T * C
    mu = g.mean(1)
    var = ((g - mu[:, None]) ** 2).mean(1)
    chain = min(T, _rps(C)) + 16 + _cdiv(T, _rps(C))
    dmu = dg.sum(1) / n + U24 * mu.abs() + chain * 2.0 ** -53 * g.abs().mean(1)
    dvar = (2 * (g - mu[:, None]).abs() * dg).sum(1) / n + 4 * chain * 2.0 ** -53 * ((g * g).mean(1) + mu * mu)
    rs = 1 / torch.sqrt(var + EPS)
    _report(name, "mean", mean, mu, dmu)
    _report(name, "rstd", rstd, rs, rs * (0.5 * dvar / (var + EPS) + U24))
    return g, dg


def _apply(y, ustride, B, T, C, mean, rstd, gamma, beta, k, s, out_bf16):
    p, Q = k - 1, _cdiv(k - 1 + T, s)
    total = B * Q * s + _cdiv(k, s) * s
    out = torch.full(((total + 1) * C,), NAN, dtype=bf16 if out_bf16 else f32, device=DEV)
    _ok(_lib().eb_gn_apply(_p(y), ustride, B, T, C, _p(mean), _p(rstd), _p(gamma), _p(beta), _p(out), int(out_bf16), p,
                           Q * s, total, _stream()), "eb_gn_apply")
    assert bool(torch.isnan(out[total * C:].float()).all()), "eb_gn_apply: a store past the last row"
    return out[:total * C].view(total, C), Q * s


@pytest.mark.parametrize("name,B,T,C,k,s,extra,kind,affine", GN_CASES, ids=[c[0] for c in GN_CASES])
def test_gn_stats_and_apply(name, B, T, C, k, s, extra, kind, affine):
    y, ustride, gamma, beta = _gn_inputs(B, T, C, extra, kind, B * T + C)
    if not affine:
        gamma = beta = None
    print("  %-30s %d row splits of %d, %d channel blocks" % (name, _cdiv(T, _rps(C)), _rps(C), _cdiv(C, 256)))
    mean, rstd = _gn_stats(y, ustride, B, T, C)
    g, dg = _check_stats(name, y, B, T, C, mean, rstd)
    out, rpu = _apply(y, ustride, B, T, C, mean, rstd, gamma, beta, k, s, False)
    out16, _ = _apply(y, ustride, B, T, C, mean, rstd, gamma, beta, k, s, True)
    _same(name + " bf16 output vs bf16_rn(fp32 output)", out16, out.bfloat16())
    # teacher-forced on the kernel's own statistics
    ga = gamma.double() if gamma is not None else torch.ones(C, dtype=f64, device=DEV)
    be = beta.double() if beta is not None else torch.zeros(C, dtype=f64, device=DEV)
    gt, dgt = g.view(B, T, C), dg.view(B, T, C)
    d = gt - mean.double()[:, None, None]
    r = rstd.double()[:, None, None]
    ref = d * r * ga + be
    bar = dgt * r * ga.abs() + 4 * U24 * (d * r * ga).abs() + U24 * be.abs()
    rows = torch.arange(out.shape[0], device=DEV)
    b, u = rows // rpu, rows % rpu - (k - 1)
    valid = (b < B) & (u >= 0) & (u < T)
    _report(name, "apply", out[valid].view(B, T, C), ref, bar)
    _same(name + " padding rows are 0", out[~valid], torch.zeros_like(out[~valid]))
    if affine:
        ones, zeros = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
        plain, _ = _apply(y, ustride, B, T, C, mean, rstd, None, None, k, s, False)
        _same(name + " gamma = beta = None vs 1 / 0", plain,
              _apply(y, ustride, B, T, C, mean, rstd, ones, zeros, k, s, False)[0])


def _gn_bwd_call(y, ustride, B, T, C, mean, rstd, gamma, dz, dz_off, dz_ustride, want_dy, want_dy16, want_db, dy_off,
                 dy_ustride):
    from edgedict_b200 import ops
    ns, nd = ops._gn_slices(B, T, C)
    pg, pb = torch.full((ns + 1, C), NAN, device=DEV), torch.full((ns + 1, C), NAN, device=DEV)
    pdb = torch.full((ns + 1, C), NAN, device=DEV) if want_db else None
    dpart = torch.full((nd, 2), NAN, dtype=f64, device=DEV)
    n = dy_off + B * dy_ustride + C
    dy = torch.full((n,), SENT, device=DEV) if want_dy else None
    dy16 = torch.full((n,), SENT, dtype=bf16, device=DEV) if want_dy16 else None

    def at(t, off):
        return None if t is None else t.data_ptr() + off * t.element_size()

    _ok(_lib().eb_gn_bwd(_p(y), ustride, B, T, C, _p(mean), _p(rstd), _p(gamma), at(dz, dz_off), dz_ustride, _p(pg),
                         _p(pb), _p(dpart), at(dy, dy_off), at(dy16, dy_off), dy_ustride, _p(pdb), _stream()), "eb_gn_bwd")
    for t, nm in ((pg, "pg"), (pb, "pb"), (pdb, "pdb")):
        if t is not None:
            assert bool(torch.isnan(t[ns]).all()) and bool(torch.isfinite(t[:ns]).all()), "eb_gn_bwd " + nm
    return pg[:ns], pb[:ns], None if pdb is None else pdb[:ns], dy, dy16


@pytest.mark.parametrize("name,B,T,C,k,s,extra,kind,affine", GN_CASES, ids=[c[0] for c in GN_CASES])
def test_gn_bwd(name, B, T, C, k, s, extra, kind, affine):
    y, ustride, gamma, _ = _gn_inputs(B, T, C, extra, kind, B * T + C)
    if not affine:
        gamma = None
    mean, rstd = _gn_stats(y, ustride, B, T, C)
    gdz = _gen(T * C + 1)
    # dz as FrontEndStack passes it: the dX buffer of the conv above, k - 1 rows in, Q s rows per utterance; the rows
    # beyond T are NaN (never read)
    Q = _cdiv(k - 1 + T, s)
    dz_off, dz_ustride = (k - 1) * C, Q * s * C
    dzv = torch.randn(B, T, C, device=DEV, generator=gdz)
    dz = torch.full((dz_off + B * dz_ustride,), NAN, device=DEV)
    dz[dz_off:].view(B, dz_ustride)[:, :T * C] = dzv.view(B, T * C)
    # dy as the block below reads it: one lead row, two spare rows per utterance (they must keep their contents)
    dy_off, dy_ustride = C, (T + 2) * C
    args = (y, ustride, B, T, C, mean, rstd, gamma, dz, dz_off, dz_ustride)
    runs = {lab: _gn_bwd_call(*args, *want, dy_off, dy_ustride)
            for lab, want in (("dy", (1, 0, 1)), ("dy16", (0, 1, 0)), ("both", (1, 1, 1)), ("dy, no db", (1, 0, 0)))}
    pg, pb, pdb, dy, dy16 = runs["both"]
    for lab, (pg2, pb2, pdb2, dy2, dy162) in runs.items():
        _same("%s %s: dgamma partials" % (name, lab), pg2, pg)
        _same("%s %s: dbeta partials" % (name, lab), pb2, pb)
        if pdb2 is not None:
            _same("%s %s: db partials" % (name, lab), pdb2, pdb)
        if dy2 is not None:
            _same("%s %s: dy" % (name, lab), dy2, dy)
        if dy162 is not None:
            _same("%s %s: dy16" % (name, lab), dy162, dy16)
    valid = torch.zeros(dy.numel(), dtype=torch.bool, device=DEV)
    valid[dy_off:dy_off + B * dy_ustride].view(B, dy_ustride)[:, :T * C] = True
    _same(name + " dy outside the T rows untouched", dy[~valid], torch.full_like(dy[~valid], SENT))
    _same(name + " dy16 outside the T rows untouched", dy16[~valid], torch.full_like(dy16[~valid], SENT))
    _same(name + " dy16 vs bf16_rn(dy)", dy16[valid], dy[valid].bfloat16())
    # teacher-forced fp64
    g, dg, gg, dgg = (t.view(B, T, C) for t in _gelu_ref(y[:, :T * C]))
    m, r = mean.double()[:, None, None], rstd.double()[:, None, None]
    ga = gamma.double() if gamma is not None else torch.ones(C, dtype=f64, device=DEV)
    d = dzv.double()
    xh = (g - m) * r
    dxh = r * (dg + U24 * (g - m).abs()) + U24 * xh.abs()
    n = T * C
    A = d * ga
    m1 = A.sum((1, 2), keepdim=True) / n
    m2 = (A * xh).sum((1, 2), keepdim=True) / n
    dm1 = U24 * m1.abs()
    dm2 = (A.abs() * dxh).sum((1, 2), keepdim=True) / n + U24 * m2.abs()
    inner = A - m1 - xh * m2
    inner_abs = A.abs() + m1.abs() + xh.abs() * m2.abs()
    dinner = 3 * U24 * inner_abs + dm1 + m2.abs() * dxh + xh.abs() * dm2
    ref = r * inner * gg
    bar = r * (dinner * (gg.abs() + dgg) + inner.abs() * dgg) + 2 * U24 * ref.abs()
    got = dy[dy_off:dy_off + B * dy_ustride].view(B, dy_ustride)[:, :T * C].view(B, T, C)
    _report(name, "dy", got, ref, bar)
    ns = pg.shape[0]
    n_add = (min(T, _rps(C)) + ns + 16) * U24
    zero = torch.zeros(C, device=DEV)
    _report(name, "dgamma", _colsum_order(pg, zero).to(DEV), (d * xh).sum((0, 1)),
            (d.abs() * dxh).sum((0, 1)) + n_add * (d * xh).abs().sum((0, 1)))
    _report(name, "dbeta", _colsum_order(pb, zero).to(DEV), d.sum((0, 1)), n_add * d.abs().sum((0, 1)))
    _report(name, "db", _colsum_order(pdb, zero).to(DEV), ref.sum((0, 1)), bar.sum((0, 1)) + n_add * ref.abs().sum((0, 1)))


# ---- the first layer ---------------------------------------------------------------------------------------------------
# (name, B, L, C, k, s, bias): (L + k - 2) % s != 0 wherever s > 1; B T rows over many 256-row splits, the last ragged
FIRST_CASES = [("k10-s5-c32", 3, 4003, 32, 10, 5, True), ("k8-s4-c16", 2, 3001, 16, 8, 4, False),
               ("k2-s1-c512", 2, 777, 512, 2, 1, True), ("k10-s4-c512", 1, 4101, 512, 10, 4, False),
               ("k2-s5-c16", 4, 1234, 16, 2, 5, True), ("k8-s1-c32", 3, 999, 32, 8, 1, False)]


@pytest.mark.parametrize("name,B,L,C,k,s,with_bias", FIRST_CASES, ids=[c[0] for c in FIRST_CASES])
def test_conv1d_first(name, B, L, C, k, s, with_bias):
    from edgedict_b200 import ops
    T = (L + k - 2) // s + 2 - k
    assert s == 1 or (L + k - 2) % s != 0
    g = _gen(L + C)
    x = torch.randn(B, L, device=DEV, generator=g)
    w = torch.randn(C, k, device=DEV, generator=g) * 0.3
    b = torch.randn(C, device=DEV, generator=g) if with_bias else None
    y = torch.full((B * T * C + C,), NAN, device=DEV)
    _ok(_lib().eb_conv1d_first_fwd(_p(x), _p(w), _p(b), _p(y), B, L, C, k, s, T, _stream()), "eb_conv1d_first_fwd")
    assert bool(torch.isnan(y[B * T * C:]).all()), name + ": a store past the output"
    # taps: xt[b, t, j] = x[b, t s + j - (k - 1)], 0 outside [0, L)
    xp = torch.zeros(B, (k - 1) + (T - 1) * s + k, dtype=f64, device=DEV)
    xp[:, k - 1:k - 1 + L] = x.double()[:, :xp.shape[1] - (k - 1)]
    xt = xp.unfold(1, k, s)[:, :T]                                            # [B, T, k]
    wd = w.double()
    bd = b.double() if b is not None else torch.zeros(C, dtype=f64, device=DEV)
    ref = xt @ wd.t() + bd
    _report(name, "fwd", y[:B * T * C].view(B, T, C), ref, k * U24 * (xt.abs() @ wd.abs().t() + bd.abs()))
    dy = torch.randn(B, T, C, device=DEV, generator=g)
    rows = B * T
    rps = max(256, _cdiv(rows, 1024))                                         # ops.conv1d_first_dw's split
    ns = _cdiv(rows, rps)
    assert ns >= 3 and rows % rps, (name, rows, rps)
    part = torch.full((ns + 1, (k + 1) * C), NAN, device=DEV)
    _ok(_lib().eb_conv1d_first_dw(_p(x), _p(dy), _p(part), ns, rps, B, L, C, k, s, T, _stream()), "eb_conv1d_first_dw")
    assert bool(torch.isnan(part[ns]).all())
    tot = _colsum_order(part[:ns], torch.zeros((k + 1) * C)).view(k + 1, C)
    dw, db = ops.conv1d_first_dw(x, dy, k, s)
    _same(name + " dW vs the colsum order of its partials", dw.cpu(), tot[:k].t().contiguous())
    _same(name + " db vs the colsum order of its partials", db.cpu(), tot[k].contiguous())
    d = dy.double().view(rows, C)
    xr = torch.cat([xt.reshape(rows, k), torch.ones(rows, 1, dtype=f64, device=DEV)], 1)   # [rows, k + 1]
    n_add = (rps + ns + 8) * U24
    _report(name, "dW, db", tot.to(DEV), xr.t() @ d, n_add * (xr.abs().t() @ d.abs()))


# ---- eb_gemm_f32_splitk ------------------------------------------------------------------------------------------------
def _splitk_case(name):
    """name -> (A storage, sam, sak, B storage, sbk, sbn, M, N, K, kchunk): A(m, k) = A[m sam + k sak],
    B(k, n) = B[k sbk + n sbn]."""
    g = _gen(len(name))
    if name == "plain-K%16":
        M, N, K = 70, 90, 4 * 1024 + 7
        A, B = torch.randn(M * K, device=DEV, generator=g), torch.randn(K * N, device=DEV, generator=g)
        return A, K, 1, B, N, 1, M, N, K, 1024
    # the dW strides of FrontEndStack's fp32 mode: A = dY [rows, C_out] from the lead row (sam = 1, sak = C_out),
    # B = the padded operand as overlapping rows (sbk = s C_in, sbn = 1), N = k C_in
    Cout, Cin, k, s, K, kchunk = {"dw-ragged": (48, 32, 3, 2, 5 * 1000 + 333, 1000),
                                  "dw-ops-rule": (128, 128, 3, 2, 140000, None)}[name]
    kchunk = kchunk or max(1024, _cdiv(K, 128))                             # ops.gemm_f32_rows's rule
    A = torch.randn(K * Cout, device=DEV, generator=g)
    B = torch.randn((K - 1) * s * Cin + k * Cin, device=DEV, generator=g)
    return A, 1, Cout, B, s * Cin, 1, Cout, k * Cin, K, kchunk


@pytest.mark.parametrize("name", ["plain-K%16", "dw-ragged", "dw-ops-rule"])
def test_gemm_f32_splitk(name):
    from edgedict_b200 import ops
    A, sam, sak, B, sbk, sbn, M, N, K, kchunk = _splitk_case(name)
    nz = _cdiv(K, kchunk)
    assert K % kchunk and nz >= 3
    part = torch.full((nz + 1, M * N), NAN, device=DEV)
    _ok(_lib().eb_gemm_f32_splitk(_p(A), sam, sak, _p(B), sbk, sbn, _p(part), M, N, K, kchunk, _stream()), name)
    assert bool(torch.isnan(part[nz]).all()), name + ": a store past the last slice"
    for z in range(nz):
        k0, kz = z * kchunk, min(kchunk, K - z * kchunk)
        one = torch.full((M + 1, N), NAN, device=DEV)
        _ok(_lib().eb_gemm_f32(A.data_ptr() + 4 * k0 * sak, sam, sak, B.data_ptr() + 4 * k0 * sbk, sbk, sbn, _p(one), N,
                               None, M, N, kz, 1.0, 0.0, _stream()), "eb_gemm_f32")
        _same("%s slice %d vs eb_gemm_f32 over k [%d, %d)" % (name, z, k0, k0 + kz), part[z].view(M, N), one[:M])
    tot = _colsum_order(part[:nz], torch.zeros(M * N)).view(M, N)
    if sam == 1 and kchunk == max(1024, _cdiv(K, 128)):
        _same(name + " ops.gemm_f32_rows vs the colsum order of its slices",
              ops.gemm_f32_rows(A, 0, sam, sak, B, sbk, sbn, M, N, K).cpu(), tot)
    Al = A.as_strided((M, K), (sam, sak)).double()
    Bl = B.as_strided((K, N), (sbk, sbn)).double()
    print("  %-30s %d slices of %d" % (name, nz, kchunk))
    _report(name, "total", tot.to(DEV), Al @ Bl, (kchunk + nz + 8) * U24 * (Al.abs() @ Bl.abs()))


# ---- eb_gemm_bf16 at the dW layout -------------------------------------------------------------------------------------
def test_gemm_bf16_dw_layout():
    """FrontEndStack's bf16 dW: part d = dY^T (MN-major, [B Q, C_out]) times the padded operand from row d s on, read
    as [B Q, s C_in] rows of pitch s C_in (MN-major), for d < ceil(k / s); K = B Q takes split-K."""
    from edgedict_b200 import ops
    Cout, Cin, k, s, K = 128, 128, 3, 2, 8000
    nd = _cdiv(k, s)
    g = _gen(K)
    dy16 = torch.randn(K * Cout, device=DEV, generator=g).bfloat16()
    xp16 = torch.randn((K + nd) * s * Cin, device=DEV, generator=g).bfloat16()
    M, N = Cout, s * Cin
    _, ks = _plan(M, N, K)
    assert ks > 1, "the dW product must take split-K"
    Ad = dy16.view(K, Cout).double()
    for d in range(nd):
        P = ops.gemm_bf16(dy16, 1, xp16[d * s * Cin:], 1, M, N, K)
        Bd = xp16[d * s * Cin:d * s * Cin + K * N].view(K, N).double()
        _report("bf16 dW part %d (%d splits)" % (d, ks), "raw", P, Ad.t() @ Bd, _n_add(K, ks) * UTC * (Ad.abs().t() @ Bd.abs()))
