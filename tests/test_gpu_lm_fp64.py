"""Per-element fp64 parity and bitwise invariants of the language model's loss kernels, the path `functional.LMLoss`
runs on every LMModel training step:

    eb_lm_logits_ce   gemm_tc.cu, LSE_ROWS epilogue: logits16 = bf16(h . w^T + b), and from the fp32 accumulators each
                      row's lse and target logit (tlogit)                                          (bf16 mode)
    eb_lm_ce_rows     lm.cu: the same row statistics of fp32 logits, one warp per row              (fp32 mode)
    eb_lm_ce_loss     lm.cu: per-token costs, their fixed-order sum and count, the loss and the gradient scale
    eb_lm_ce_bwd      lm.cu: d logits, fp32 or bf16, in place or not, 16-byte vectorised or scalar

Every C entry is called directly into NaN-prefilled outputs with guard elements behind them, and every check is
teacher-forced on the outputs of the kernel before it, so a failure names one kernel and one element.  u = U24 = 2^-24
is the fp32 unit roundoff.  Each check prints its worst err/bar and where it occurs (pytest -s); DESIGN.md section 2
records the measured figures.

(a) eb_lm_logits_ce.  P is the raw fp32 product of the same bf16 operands from eb_gemm_bf16, the same bits on every tile
configuration (test_gpu_gemm_fp64.py), and x = fp32(P + b) the fp32 logits the epilogue sees.  Bitwise:
logits16 = bf16_rn(x), tlogit = x[r, t] for t in [0, V) and +0 otherwise.  The lse against fp64 logsumexp(x): a
thread owns 32 columns of each 128-wide column tile (two chains of 16) and keeps a running max nm.  A term
ex2(fma(x, L, -fl(nm L))) (L = fp32 log2 e) is off by the ex2.approx error EXP_FAST, the rounding of nm L (u |nm|,
|nm| <= |m| + (m - x)), the FMA's rounding and L's own (2 u (m - x)); weighted by the softmax p that is
EXP_FAST + u (|m| + 3 R), R = sum_v p_v (m - x_v).  Each of the T_n - 1 per-tile rescales and the two quad merges
costs EXP_FAST, one product rounding and 3 u |dm| (subtraction, scaling by L, L), sum |dm| <= spread = max - min per
level; the chains add 16 + 1 + T_n roundings and the merges 2 more.  So the sum s = sum exp(x - m) is within
    eps_s = (T_n + 2) EXP_FAST + u (|m| + 3 R + 9 spread + 2 T_n + 24)
relative, and lse = m + logf(s) within  eps_s + 2 u log(s) + u |lse|  (logf 1 ulp, the final add).  The |m| term is the
epilogue's own: it computes exp(x - m) without forming x - m.  The large-offset case shows that the bar without it
fails, and the power check shows that the lse of the bf16-rounded logits misses the bar by more than 8x: the test tells
statistics of the accumulators from statistics of the stored logits.

(b) eb_lm_ce_rows.  tlogit is the input element bitwise.  The lse: each term expf(fl(x - m)) is off by 2 ulp (EXPF,
2^-22) and u (m - x); a lane adds ceil(V/32) terms and the warp 5 more:
    eps_s = EXPF + u (R + ceil(V/32) + 5),  lse within  eps_s + 2 u log(s) + u |lse|.
No |m| term: the row pass subtracts first, and the large-offset case passes this bar.

(c) eb_lm_ce_loss on the kernel's own lse and tlogit: cost = fp32(lse - tlogit) bitwise for a valid target, +0 for
ignore_index, NaN for any other target outside [0, V).  The loss against fsum(costs) / n (mean) or fsum(costs) (sum),
within one fp32 ulp (the kernel sums in fp64); scale is bitwise float32(1 / n) or 1; n counts every target that is not
ignored.  Everything ignored: the mean is NaN and its scale +inf.  M = 0.

(d) eb_lm_ce_bwd on the kernel's own logits (fp32, or the bf16 logits16) and lse.  With gs = fp32(g scale), the kernel's
own product, ref = gs (exp(l - lse) - [k = t]).  fl(l - lse) costs u |l - lse| relative in the exponential, expf 2 ulp,
the subtraction and the product one rounding each:
    |grad - ref| <= |gs| (e (u |l - lse| + EXPF) + 2 u |e - [k = t]|) (1 + 2^-20) + TINY,   e = exp(l - lse),
plus half a bf16 ulp of |ref| + bar in bf16.  Ignored rows are +0 with the sign bit clear, also under scale = +inf and
a negative g; rows with an out-of-range target are all NaN; neither changes any other row's bits.

(e) Bitwise invariants: a row's lse, tlogit and logits16 in its full batch and in a prefix batch of m rows (m not a
multiple of 128); permuted targets change only tlogit; int32 and int64 targets give the same outputs; the gradient in
place and out of place, vectorised (4 fp32 / 8 bf16 per access) and scalar (one element off alignment), with a scalar g
and with g broadcast per row; repeated launches.

(f) functional.LMLoss for each reduction and precision: the loss (or the costs) and db = colsum(d logits) are the bits
of the kernels called one by one.

Targets hit columns 0, 127, 128, 255, 256 and V - 1, ignore_index 0 (the LM's pad) and -100, and out-of-range values
-1, V, 2^31 and 2^32 + 7 (int64; in the int32 run the last two read 2^31 - 1).  Every case runs with int32 and int64
targets.  The file runs in about 15 s on an H100."""
import math

import numpy as np
import pytest
import torch

from tests.test_gpu_gemm_fp64 import TINY, U24, _gemm, _same, worst
from tests.test_gpu_joint_loss_fused import _bf16_ulp
from tests.test_gpu_loss_fp64 import EXP_FAST

pytestmark = pytest.mark.gpu

bf16, f32, f64, i32, i64 = torch.bfloat16, torch.float32, torch.float64, torch.int32, torch.int64
DEV = "cuda"
NAN = float("nan")
EXPF = 2.0 ** -22         # expf: 2 ulp
TILE_N = 128              # column tile of the LSE epilogue
IGNORES = (0, -100)


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Buf:
    """A NaN-filled allocation holding a tensor of `shape` `off` elements in, with `off` guard elements before it and a
    guard row (or 4 elements) behind it."""

    def __init__(self, shape, dtype, off=0):
        self.n = int(np.prod(shape))
        self.off = off
        self.flat = torch.full((2 * off + self.n + (shape[-1] if len(shape) > 1 else 4),), NAN, dtype=dtype, device=DEV)
        self.t = self.flat[off:off + self.n].view(shape)

    def guards_ok(self, name):
        f = self.flat.float()
        assert bool(f[:self.off].isnan().all()) and bool(f[self.off + self.n:].isnan().all()), \
            name + ": a store outside the output"


def _check(name, label, got, ref, bar, mask=None):
    """Prints the worst err/bar of `got` against its fp64 value over `mask` (all elements by default), then asserts it."""
    got = got.double()
    if mask is None:
        mask = torch.ones_like(got, dtype=torch.bool)
    elif mask.dim() < got.dim():                                       # a row mask
        mask = mask[:, None].expand_as(got)
    assert bool(torch.isfinite(got[mask]).all()), "%s %s: non-finite output" % (name, label)
    if not bool(mask.any()):
        return 0.0
    err = torch.where(mask, (got - ref).abs(), torch.zeros_like(got))
    ratio, idx, e, b = worst(err, torch.where(mask, bar, torch.ones_like(bar)))
    print("  %-24s %-34s worst err/bar %.3g at %s (err %.3g, bar %.3g)" % (name, label, ratio, idx, e, b))
    assert ratio <= 1.0, "%s %s: err/bar %.3g at %s" % (name, label, ratio, idx)
    return ratio


def _max_ratio(err, bar):
    return float((err / bar).max())


# ---- targets ----------------------------------------------------------------------------------------------------------
def _specials(V):
    """Target values every case plants: tile-edge columns (those >= V are out of range there), V - 1, the two
    ignore_index values and out-of-range values."""
    return [0, 127, 128, 255, 256, V - 1, -100, -1, V, 2 ** 31, 2 ** 32 + 7]


def _targets(M, V, seed):
    """(int64, int32) targets [M]: uniform in [0, V), every 13th row a special value, the last row V - 1 and the one
    before it 2^32 + 7.  The int32 copy reads 2^31 - 1 where int64 holds 2^31 or 2^32 + 7 (out of range either way)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, V, (M,), generator=g, dtype=i64)
    sp = _specials(V)
    r = torch.arange(M)
    sel = r % 13 == 5
    t[sel] = torch.tensor(sp, dtype=i64)[(r[sel] // 13) % len(sp)]
    t[M - 1] = V - 1
    if M > 2:
        t[M - 2] = 2 ** 32 + 7
    return t.to(DEV), t.clamp(max=2 ** 31 - 1).to(i32).to(DEV)


def _classes(t, V, ignore):
    """(valid, ignored, out of range) row masks of targets t under ignore_index."""
    ign = t == ignore
    inr = (t >= 0) & (t < V)
    return inr & ~ign, ign, ~inr & ~ign


# ---- (a) the logits GEMM with its cross-entropy epilogue --------------------------------------------------------------
def _gcases(nsm):
    """name -> (M, V, K, bias, offset of logits16 in bf16 elements, logit scale, common logit offset)"""
    return {
        "bench": (32768, 1024, 1024, True, 0, 3.0, 0.0),                   # DESIGN section 4b's production shape
        "many_row_blocks": (2 * nsm * 128 + 165, 1024, 64, True, 0, 3.0, 0.0),   # every CTA >= 2 row blocks, partial last
        "v520": (1000, 520, 128, True, 0, 3.0, 0.0),                        # partial last column tile, staged TMA store
        "v136_k72": (700, 136, 72, True, 0, 3.0, 0.0),                      # K tail, a second column tile 8 wide
        "v72_k8": (300, 72, 8, True, 0, 3.0, 0.0),                          # V < one tile: threads owning no column
        "v517": (400, 517, 64, True, 0, 3.0, 0.0),                          # V % 8 != 0: row-wise register stores
        "unaligned": (300, 264, 64, True, 2, 3.0, 0.0),                     # logits16 4 bytes off: 2-wide register stores
        "nobias": (500, 384, 96, False, 0, 3.0, 0.0),
        "m1": (1, 1024, 64, True, 0, 3.0, 0.0),
        "offset": (8000, 1024, 64, True, 0, 1.0, 1024.0),                   # bias + 2^10: the |m| term of the lse bar
    }


GCASES = list(_gcases(132))


def _logits_ce(c, h, t, t64, M=None):
    """eb_lm_logits_ce into guarded NaN-filled buffers: (logits16, lse, tlogit)."""
    M = c["M"] if M is None else M
    V, K = c["V"], c["K"]
    lg, ls, tl = Buf((M, V), bf16, c["off"]), Buf((M,), f32), Buf((M,), f32)
    rc = _lib().eb_lm_logits_ce(_p(h), _p(c["w"]), _p(c["bias"]), _p(lg.t), _p(t), t64, _p(ls.t), _p(tl.t), M, V, K,
                                _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    for b, k in ((lg, "logits16"), (ls, "lse"), (tl, "tlogit")):
        b.guards_ok("%s %s" % (c["name"], k))
    return lg.t, ls.t, tl.t


def _epilogue_lse_bar(x, with_m=True):
    """The lse bar of (a) per row of the fp32 logits x (as fp64 [M, V]), and the fp64 lse."""
    V = x.shape[1]
    m = x.max(1).values
    lse = torch.logsumexp(x, 1)
    R = (torch.softmax(x, 1) * (m[:, None] - x)).sum(1)
    spread = m - x.min(1).values
    tn = -(-V // TILE_N)
    eps_s = (tn + 2) * EXP_FAST[f32] + U24 * ((m.abs() if with_m else 0) + 3 * R + 9 * spread + 2 * tn + 24)
    eps_s = eps_s + V * 2.0 ** -126                                    # ex2.approx.ftz flushes terms below 2^-126
    return eps_s + 2 * U24 * (lse - m) + U24 * lse.abs() + TINY, lse


@pytest.fixture(scope="module", params=GCASES)
def gcase(request):
    name = request.param
    M, V, K, has_b, off, scale, offset = _gcases(_nsm())[name]
    seed = sum(map(ord, name))
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = (torch.rand(M, K, device=DEV, generator=g) * 2 - 1).to(bf16)
    w = (torch.randn(V, K, device=DEV, generator=g) * (scale * math.sqrt(3.0 / K))).to(bf16)
    bias = torch.randn(V, device=DEV, generator=g) + offset if has_b else None
    t64, t32 = _targets(M, V, seed)
    c = dict(name=name, M=M, V=V, K=K, off=off, h=h, w=w, bias=bias, t64=t64, t32=t32)
    P = _gemm(name + " raw", h, 0, w, 0, M, V, K)
    c["x"] = P + bias if has_b else P                                  # the epilogue's fp32 logits
    c["logits16"], c["lse"], c["tlogit"] = _logits_ce(c, h, t64, 1)
    c["run32"] = _logits_ce(c, h, t32, 0)
    return c


def test_logits_ce_parity(gcase):
    """(a) logits16 and tlogit bitwise from the fp32 logits x = fp32(P + b); the lse within the epilogue's bar (module
    docstring), which the lse of the bf16-rounded logits misses by more than 8x, and which needs its |m| term in the
    large-offset case."""
    c = gcase
    M, V, name = c["M"], c["V"], c["name"]
    x = c["x"]
    _same(name + " logits16", c["logits16"], x.to(bf16))
    t = c["t64"]
    inr = (t >= 0) & (t < V)
    want = torch.zeros(M, dtype=f32, device=DEV)
    want[inr] = x[inr.nonzero()[:, 0], t[inr]]
    _same(name + " tlogit", c["tlogit"], want)                         # +0 (sign bit clear) outside [0, V)
    x64 = x.double()
    bar, lse = _epilogue_lse_bar(x64)
    _check(name, "lse vs fp64 logsumexp(x)", c["lse"], lse, bar)
    err = (c["lse"].double() - lse).abs()
    bar_nom, _ = _epilogue_lse_bar(x64, with_m=False)
    r_nom = _max_ratio(err, bar_nom)
    lse16 = torch.logsumexp(x.to(bf16).double(), 1)
    r16 = _max_ratio((lse16 - lse).abs(), bar)
    print("  %-24s without the |m| term: err/bar %.3g; bf16 logits' lse: %.3g x the bar; |m| max %.1f"
          % (name, r_nom, r16, float(x64.max(1).values.abs().max())))
    if M > 1:
        assert r16 >= 8.0, "the lse bar does not tell the accumulators from the bf16 logits: %.3g" % r16
    if name == "offset":
        assert r_nom > 1.0, "the |m| term is not needed at |m| ~ 2^10: %.3g" % r_nom


def test_logits_ce_invariants(gcase):
    """(e) int32 targets give the int64 run's bits; a repeated launch, a prefix batch of m rows (m % 128 != 0) and
    permuted targets give the same logits16 and lse bits, and tlogit follows the targets."""
    c = gcase
    M, V, name = c["M"], c["V"], c["name"]
    for k, a, b in zip(("logits16", "lse", "tlogit"), c["run32"], (c["logits16"], c["lse"], c["tlogit"])):
        _same("%s int32 vs int64 targets: %s" % (name, k), a, b)
    for k, a, b in zip(("logits16", "lse", "tlogit"), _logits_ce(c, c["h"], c["t64"], 1),
                       (c["logits16"], c["lse"], c["tlogit"])):
        _same("%s repeated launch: %s" % (name, k), a, b)
    if M > 1:
        m = (5 * M) // 8 or 1
        if m % 128 == 0:
            m -= 1
        for k, a, b in zip(("logits16", "lse", "tlogit"), _logits_ce(c, c["h"][:m], c["t64"][:m], 1, M=m),
                           (c["logits16"], c["lse"], c["tlogit"])):
            _same("%s first %d rows alone: %s" % (name, m, k), a, b[:m])
    perm = c["t64"][torch.randperm(M, generator=torch.Generator().manual_seed(M)).to(DEV)]
    lg, ls, tl = _logits_ce(c, c["h"], perm, 1)
    _same(name + " permuted targets: logits16", lg, c["logits16"])
    _same(name + " permuted targets: lse", ls, c["lse"])
    inr = (perm >= 0) & (perm < V)
    want = torch.zeros(M, dtype=f32, device=DEV)
    want[inr] = c["x"][inr.nonzero()[:, 0], perm[inr]]
    _same(name + " permuted targets: tlogit", tl, want)


# ---- (b) the fp32 row pass ------------------------------------------------------------------------------------------
def _rcases(nsm):
    """name -> (M, V, common logit offset): M above the 16 x #SMs x 8-row grid, so that the grid-stride loop runs."""
    big = 16 * nsm * 8 + 37
    return {"v1": (big, 1, 0.0), "v31": (big, 31, 0.0), "v33": (big, 33, 0.0), "v517": (big, 517, 0.0),
            "v520": (big, 520, 0.0), "v1024": (big, 1024, 0.0), "v1024_offset": (4000, 1024, 1024.0)}


RCASES = list(_rcases(132))


def _ce_rows(c, t, t64):
    ls, tl = Buf((c["M"],), f32), Buf((c["M"],), f32)
    rc = _lib().eb_lm_ce_rows(_p(c["x"]), _p(t), t64, _p(ls.t), _p(tl.t), c["M"], c["V"], _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    ls.guards_ok(c["name"] + " lse")
    tl.guards_ok(c["name"] + " tlogit")
    return ls.t, tl.t


@pytest.fixture(scope="module", params=RCASES)
def rcase(request):
    name = request.param
    M, V, offset = _rcases(_nsm())[name]
    seed = sum(map(ord, name)) + 1
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, V, device=DEV, generator=g) * 3 + offset
    t64, t32 = _targets(M, V, seed)
    c = dict(name="rows-" + name, M=M, V=V, x=x, t64=t64, t32=t32)
    c["lse"], c["tlogit"] = _ce_rows(c, t64, 1)
    c["run32"] = _ce_rows(c, t32, 0)
    return c


def test_ce_rows_parity(rcase):
    """(b) tlogit is the input element bitwise (+0 outside [0, V)); the lse within the row pass's bar, which has no |m|
    term; int32 targets and a repeated launch give the same bits."""
    c = rcase
    M, V, name, x = c["M"], c["V"], c["name"], c["x"]
    t = c["t64"]
    inr = (t >= 0) & (t < V)
    want = torch.zeros(M, dtype=f32, device=DEV)
    want[inr] = x[inr.nonzero()[:, 0], t[inr]]
    _same(name + " tlogit", c["tlogit"], want)
    x64 = x.double()
    m = x64.max(1).values
    lse = torch.logsumexp(x64, 1)
    R = (torch.softmax(x64, 1) * (m[:, None] - x64)).sum(1)
    eps_s = EXPF + U24 * (R + -(-V // 32) + 5)
    _check(name, "lse vs fp64 logsumexp(x)", c["lse"], lse, eps_s + 2 * U24 * (lse - m) + U24 * lse.abs() + TINY)
    for k, a, b in zip(("lse", "tlogit"), c["run32"], (c["lse"], c["tlogit"])):
        _same("%s int32 vs int64 targets: %s" % (name, k), a, b)
    for k, a, b in zip(("lse", "tlogit"), _ce_rows(c, t, 1), (c["lse"], c["tlogit"])):
        _same("%s repeated launch: %s" % (name, k), a, b)


# ---- (c) the loss kernel ----------------------------------------------------------------------------------------------
def _ce_loss(lse, tl, t, t64, ignore, M, V, mean, with_cost=True):
    """eb_lm_ce_loss into guarded buffers: (cost or None, loss [1], scale [1])."""
    cost = Buf((max(M, 1),), f32) if with_cost else None
    loss, scale = Buf((1,), f32), Buf((1,), f32)
    rc = _lib().eb_lm_ce_loss(_p(lse), _p(tl), _p(t), t64, ignore, M, V, int(mean), _p(cost.t) if cost else None,
                              _p(loss.t), _p(scale.t), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    for b, k in ((cost, "cost"), (loss, "loss"), (scale, "scale")):
        if b is not None:
            b.guards_ok("loss kernel " + k)
    if M == 0 and cost is not None:
        assert bool(cost.t.isnan().all()), "M = 0: a cost was written"
    return (cost.t[:M] if cost else None), loss.t, scale.t


def _f32_bits(v):
    return torch.tensor([v], dtype=f64).to(f32).to(DEV)


def _check_loss(c):
    """(c) on the statistics of case c, for both ignore_index values, both reductions and both target widths."""
    M, V, name = c["M"], c["V"], c["name"]
    lse, tl = c["lse"], c["tlogit"]
    for ignore in IGNORES:
        valid, ign, oor = _classes(c["t64"], V, ignore)
        n = int((~ign).sum())
        clean = torch.where(oor, torch.full_like(c["t64"], ignore), c["t64"])
        n_clean = int(valid.sum())
        for mean in (1, 0):
            tag = "%s ignore %d %s" % (name, ignore, "mean" if mean else "sum")
            cost, loss, scale = _ce_loss(lse, tl, c["t64"], 1, ignore, M, V, mean)
            want = torch.where(valid, lse - tl, torch.zeros_like(lse))
            _same(tag + " costs", cost[~oor], want[~oor])
            assert bool(cost[oor].isnan().all()), tag + ": a cost of an out-of-range target is not NaN"
            assert bool(loss.isnan().all()) == bool(oor.any()), tag + ": NaN costs must make the loss NaN"
            _same(tag + " scale", scale, _f32_bits(1.0 / n) if mean else torch.ones(1, device=DEV))
            for k, a, b in zip(("cost", "loss", "scale"), _ce_loss(lse, tl, c["t32"], 0, ignore, M, V, mean),
                               (cost, loss, scale)):
                _same("%s int32 targets: %s" % (tag, k), a, b)
            # without out-of-range targets: the sum within one fp32 ulp of fsum
            cost_c, loss_c, scale_c = _ce_loss(lse, tl, clean, 1, ignore, M, V, mean)
            _same(tag + " costs, out-of-range targets ignored", cost_c[valid], cost[valid])
            if mean and n_clean == 0:
                assert bool(loss_c.isnan().all()) and float(scale_c) == math.inf, tag
                continue
            s = math.fsum(cost_c.double().cpu().tolist())
            ref = s / n_clean if mean else s
            ulp = float(np.spacing(np.float32(abs(ref))))
            err = abs(float(loss_c) - ref)
            print("  %-24s %-34s err/ulp %.3g (loss %.9g)" % (tag, "loss vs fsum", err / ulp, ref))
            assert err <= ulp, (tag, float(loss_c), ref)
            _same(tag + " scale (clean)", scale_c, _f32_bits(1.0 / n_clean) if mean else torch.ones(1, device=DEV))
            _, loss_n, scale_n = _ce_loss(lse, tl, clean, 1, ignore, M, V, mean, with_cost=False)
            _same(tag + " loss without cost", loss_n, loss_c)
            _same(tag + " scale without cost", scale_n, scale_c)


def test_ce_loss_on_epilogue_statistics(gcase):
    _check_loss(gcase)


def test_ce_loss_on_row_statistics(rcase):
    _check_loss(rcase)


def test_ce_loss_edges():
    """(c) every target ignored: mean NaN with scale +inf, sum 0 with scale 1, every cost +0; M = 0 alike, with null
    statistics and no cost written."""
    M, V = 300, 50
    lse = torch.randn(M, device=DEV)
    tl = torch.randn(M, device=DEV)
    for t64 in (1, 0):
        t = torch.full((M,), -100, dtype=i64 if t64 else i32, device=DEV)
        cost, loss, scale = _ce_loss(lse, tl, t, t64, -100, M, V, 1)
        assert bool(loss.isnan().all()) and float(scale) == math.inf
        _same("all ignored costs", cost, torch.zeros(M, device=DEV))
        cost, loss, scale = _ce_loss(lse, tl, t, t64, -100, M, V, 0)
        _same("all ignored, sum: loss", loss, torch.zeros(1, device=DEV))
        _same("all ignored, sum: scale", scale, torch.ones(1, device=DEV))
    _, loss, scale = _ce_loss(None, None, None, 1, 0, 0, V, 1)
    assert bool(loss.isnan().all()) and float(scale) == math.inf
    _, loss, scale = _ce_loss(None, None, None, 1, 0, 0, V, 0)
    _same("M = 0, sum: loss", loss, torch.zeros(1, device=DEV))
    _same("M = 0, sum: scale", scale, torch.ones(1, device=DEV))


# ---- (d) the gradient kernel ------------------------------------------------------------------------------------------
def _ce_bwd(logits, lse, t, t64, ignore, g, g_per_row, scale, off=0, in_place=False):
    """eb_lm_ce_bwd on a copy of logits placed `off` elements into a guarded allocation (off = 1: the scalar path), into
    a guarded NaN-filled output at the same offset or in place over the copy.  Returns d logits."""
    M, V = logits.shape
    src = Buf((M, V), logits.dtype, off)
    src.t.copy_(logits)
    dst = src if in_place else Buf((M, V), logits.dtype, off)
    rc = _lib().eb_lm_ce_bwd(_p(src.t), _p(dst.t), int(logits.dtype == bf16), _p(lse), _p(t), t64, ignore, M, V, _p(g),
                             g_per_row, _p(scale), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    dst.guards_ok("gradient")
    if not in_place:
        _same("gradient: the logits operand was written", src.t, logits)
    return dst.t


def _grad_ref(logits, lse, t, valid, gs):
    """(ref, bar) of (d) in fp64 on valid rows (zeros elsewhere); gs [M] the kernel's fp32 g * scale."""
    M, V = logits.shape
    d = logits.double() - lse.double()[:, None]
    e = torch.exp(d)
    onehot = torch.zeros(M, V, dtype=f64, device=DEV)
    rows = valid.nonzero()[:, 0]
    onehot[rows, t[valid]] = 1.0
    q = e - onehot
    gsd = gs.double()[:, None]
    ref = gsd * q
    bar = gsd.abs() * (e * (U24 * d.abs() + EXPF) + 2 * U24 * q.abs()) * (1 + 2.0 ** -20) + TINY
    if logits.dtype == bf16:
        bar = bar + 0.5 * _bf16_ulp(ref.abs() + bar)
    return ref, bar


def _check_grad(c, logits):
    """(d) and the gradient's invariants of (e) on case c's own logits (fp32 x, or logits16) and lse."""
    M, V, name = c["M"], c["V"], c["name"] + (" bf16" if logits.dtype == bf16 else " fp32")
    lse = c["lse"]
    vec = 8 if logits.dtype == bf16 else 4
    gen = torch.Generator(device=DEV).manual_seed(M + V)
    g_row = torch.randn(M, device=DEV, generator=gen)                  # mixed signs
    g1 = torch.tensor([0.75], device=DEV)
    for ignore in IGNORES:
        tag = "%s ignore %d" % (name, ignore)
        t = c["t64"]
        valid, ign, oor = _classes(t, V, ignore)
        n = int((~ign).sum())
        sc = _f32_bits(1.0 / n)
        # per-row g, scale set
        gr = _ce_bwd(logits, lse, t, 1, ignore, g_row, 1, sc)
        ref, bar = _grad_ref(logits, lse, t, valid, g_row * sc)
        path = "vec %d" % vec if V % vec == 0 else "scalar"
        _check(tag, "g per row, scale (%s)" % path, gr, ref, bar, valid)
        assert bool((gr[ign].view(torch.int16 if logits.dtype == bf16 else i32) == 0).all()), tag + ": ignored row != +0"
        assert bool(gr[oor].isnan().all()), tag + ": out-of-range row not NaN"
        # scalar g, no scale
        gsc = _ce_bwd(logits, lse, t, 1, ignore, g1, 0, None)
        ref1, bar1 = _grad_ref(logits, lse, t, valid, g1.expand(M))
        _check(tag, "g scalar, no scale (%s)" % path, gsc, ref1, bar1, valid)
        # bitwise: int32 targets, the scalar path, in place, g broadcast per row, a repeated launch
        _same(tag + " int32 targets", _ce_bwd(logits, lse, c["t32"], 0, ignore, g_row, 1, sc), gr)
        _same(tag + " scalar path (one element off)", _ce_bwd(logits, lse, t, 1, ignore, g_row, 1, sc, off=1), gr)
        _same(tag + " in place", _ce_bwd(logits, lse, t, 1, ignore, g_row, 1, sc, in_place=True), gr)
        _same(tag + " g broadcast per row", _ce_bwd(logits, lse, t, 1, ignore, g1.expand(M).contiguous(), 1, None),
              gsc)
        _same(tag + " repeated launch", _ce_bwd(logits, lse, t, 1, ignore, g_row, 1, sc), gr)
        # other rows keep their bits when the ignored / out-of-range rows get valid targets
        if bool((ign | oor).any()):
            tv = torch.where(ign | oor, torch.full_like(t, V // 2), t)
            if ignore == V // 2:
                tv = torch.where(ign | oor, torch.full_like(t, V - 1), t)
            g2 = _ce_bwd(logits, lse, tv, 1, ignore, g_row, 1, sc)
            _same(tag + " valid rows beside ignored / out-of-range rows", gr[valid], g2[valid])
        # scale = +inf and a negative g: ignored rows still +0, sign bit clear
        inf = torch.tensor([math.inf], device=DEV)
        gi = _ce_bwd(logits, lse, t, 1, ignore, -g_row.abs() - 1, 1, inf, off=0)
        assert bool((gi[ign].view(torch.int16 if logits.dtype == bf16 else i32) == 0).all()), \
            tag + ": an ignored row under scale = +inf is not +0"
        assert bool(gi[oor].isnan().all())


def test_ce_bwd_bf16(gcase):
    _check_grad(gcase, gcase["logits16"])


def test_ce_bwd_fp32(rcase):
    _check_grad(rcase, rcase["x"])


def test_ce_bwd_paths_reached():
    """The case tables reach both gradient variants in both precisions, a partial last row block, a CTA with two row
    blocks and V below one column tile."""
    nsm = _nsm()
    gc, rc = _gcases(nsm), _rcases(nsm)
    assert any(v[1] % 8 == 0 for v in gc.values()) and any(v[1] % 8 for v in gc.values())
    assert any(v[1] % 4 == 0 for v in rc.values()) and any(v[1] % 4 for v in rc.values())
    M = gc["many_row_blocks"][0]
    assert -(-M // 128) >= 2 * nsm and M % 128
    assert gc["v72_k8"][1] < TILE_N and gc["unaligned"][1] % 8 == 0 and gc["unaligned"][4] * 2 % 16
    assert all(v[0] > 16 * nsm * 8 for k, v in rc.items() if k != "v1024_offset")


# ---- (f) the chain as LMLoss runs it --------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("reduction", ["mean", "sum", "none"])
def test_lmloss_chain_bits(precision, reduction):
    """(f) functional.LMLoss: the loss (or costs) and db are the bits of eb_lm_logits_ce / eb_lm_ce_rows,
    eb_lm_ce_loss, eb_lm_ce_bwd (in place, with LMLoss's g and scale) and eb_colsum called one by one."""
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    M, K, V, ignore = 777, 64, 520, 0
    g = torch.Generator(device=DEV).manual_seed(M + len(reduction) + len(precision))
    x = torch.randn(M, K, device=DEV, generator=g)
    w = 0.3 * torch.randn(V, K, device=DEV, generator=g)
    b = (0.1 * torch.randn(V, device=DEV, generator=g)).requires_grad_(True)
    t = torch.randint(0, V, (M,), device=DEV, generator=g)
    t[::9] = ignore
    go = torch.randn(M, device=DEV, generator=g) if reduction == "none" else torch.ones((), device=DEV)
    out = Fn.LMLoss.apply(x, w, b, t, ignore, reduction, precision)
    out.backward(go)
    L = _lib()
    lse, tl = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    if precision == "bf16":
        logits = torch.empty(M, V, dtype=bf16, device=DEV)
        assert L.eb_lm_logits_ce(_p(ops.cast_bf16(x)), _p(ops.cast_bf16(w)), _p(b), _p(logits), _p(t), 1, _p(lse),
                                 _p(tl), M, V, K, _stream()) == 0
    else:
        logits = ops.mm_nt(x, w, b.detach(), "fp32")
        assert L.eb_lm_ce_rows(_p(logits), _p(t), 1, _p(lse), _p(tl), M, V, _stream()) == 0
    cost, loss, scale = torch.empty(M, device=DEV), torch.empty((), device=DEV), torch.empty(1, device=DEV)
    assert L.eb_lm_ce_loss(_p(lse), _p(tl), _p(t), 1, ignore, M, V, int(reduction == "mean"), _p(cost), _p(loss),
                           _p(scale), _stream()) == 0
    _same("LMLoss %s %s output" % (precision, reduction), out.detach(), cost if reduction == "none" else loss)
    gv = go.reshape(-1).contiguous()
    assert L.eb_lm_ce_bwd(_p(logits), _p(logits), int(precision == "bf16"), _p(lse), _p(t), 1, ignore, M, V, _p(gv),
                          int(gv.numel() > 1), _p(scale), _stream()) == 0
    _same("LMLoss %s %s db" % (precision, reduction), b.grad, ops.colsum(logits))
