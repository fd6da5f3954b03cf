"""Per-element fp64 parity and bitwise invariants of the dense GEMMs, in every configuration.

    eb_gemm_bf16 / eb_gemm_bf16_ex   wgmma, 128 x 256 and 128 x 128 tiles, the co-resident 128 x 128 / 3-stage /
                                     112-register configuration (EB_GEMM_CORESIDENT), split-K with splitk_reduce_kernel,
                                     the n_inner and round-robin tile schedules; fp32 / bf16 output, bias, accumulate
    eb_gemm_bf16_dtanh               the tanh' epilogue
    eb_joint_logits_lse              its bf16 logits (the softmax statistics are pinned by test_gpu_joint_loss_fused.py)
    eb_gemm_f32                      the fp32 CUDA-core GEMM of the parity mode and the front end

Error model.  The bf16 operands are drawn as bf16, so their fp64 values are exact, and every bf16 x bf16 product is exact
in fp32.  The only rounding of the raw product P (fp32 output, no bias, no accumulate) is the fp32 accumulation:
  |P - S| <= n_add u_acc (|A| @ |B|) + TINY,   S the exact product (fp64; its own rounding, ~K 2^-53, is negligible),
n_add = K products through wgmma plus one add per split-K partial (`_n_add`), u_acc = UTC = 2^-23 per add (the tensor
core aligns the addends and may truncate: one ulp, not half).  eb_gemm_f32 runs one FMA chain per element in k order:
K roundings of U24 = 2^-24, plus the roundings of alpha, bias and beta.

Everything else is checked BITWISE against torch fp32 arithmetic on the kernel's own P, because the epilogue code fixes
the order of its roundings:
  + bias                 P + bias
  accumulate             (P + bias) + C_before
  bf16 out               bf16_rn(P + bias)
  bf16 out + accumulate  bf16_rn((P + bias) + float(C16_before))
  dtanh                  bf16_rn(P * fp32(1 - h^2))   (h bf16: h^2 is exact in fp32, so FMA contraction changes nothing)
  logits16 of the LSE    bf16_rn(P + b2)
  split-K                C_before (or 0) plus the partial tiles one by one in split order; partial s is the same GEMM
                         over k-blocks [s kb_per, (s+1) kb_per) run as its own call, with the bias in partial 0 only
A given output element accumulates the same k16 steps in the same order whatever the tile, so P is also bitwise the same
on the 128 x 256 tile, the 128 x 128 tile and the co-resident configuration, under both tile schedules and on every
launch.  Every output is written into a NaN-prefilled buffer with a guard row behind it: a tile the schedule never
visits, or a store past the last row, fails the test.

Which configuration a shape takes is decided by plan() in gemm_tc.cu; `_plan` restates it and is pinned to the library
through eb_gemm_bf16_partials (the split count depends on the tile width).  The worst-case summation bound is loose
(random signs give ~sqrt(n_add)); every raw-product check prints its worst err/bar next to where it occurs (pytest -s),
and DESIGN.md section 2 records the measured figures.  The file runs in about 15 s on an H100."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
UTC = 2.0 ** -23          # per add of a tensor-core fp32 accumulation
U24 = 2.0 ** -24          # fp32 unit roundoff, round to nearest (the FMA chains of gemm_simt.cu)
TINY = 2.0 ** -120        # absolute floor of every bar
BM, BK = 128, 64          # gemm_tc.cu: rows of a tile, k per k-block
CORESIDENT = 1            # include/edgedict_b200.h EB_GEMM_CORESIDENT
FIXED_K = 2               # EB_GEMM_FIXED_K


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


@pytest.fixture(autouse=True)
def _default_tile_choice():
    if os.environ.get("EDGEDICT_GEMM_BN", "0") not in ("", "0"):
        pytest.skip("EDGEDICT_GEMM_BN overrides the tile width that _plan restates")


# ---- error bookkeeping ------------------------------------------------------------------------------------------------
def worst(err, bar):
    """(largest err / bar, index of that element, its err, its bar); err == 0 counts as 0 whatever the bar."""
    r = torch.where(err == 0, torch.zeros_like(err), err / bar.clamp_min(1e-300))
    k = int(torch.argmax(r.reshape(-1)))
    idx = tuple(int(i) for i in np.unravel_index(k, tuple(r.shape)))
    return float(r.reshape(-1)[k]), idx, float(err.reshape(-1)[k]), float(bar.reshape(-1)[k])


def _report(name, label, got, ref, bar):
    """Prints the worst err/bar of one output against its fp64 value, then asserts it."""
    got = got.double()
    assert torch.isfinite(got).all(), "%s %s: non-finite output" % (name, label)
    ratio, idx, e, b = worst((got - ref).abs(), bar + TINY)
    print("  %-44s %-10s worst err/bar %.3g at %s (err %.3g, bar %.3g)" % (name, label, ratio, idx, e, b))
    assert ratio <= 1.0, "%s %s: err/bar %.3g at %s, kernel %r, fp64 %r" % (name, label, ratio, idx, float(got[idx]),
                                                                            float(ref[idx]))


def _bits(x):
    return x.view(torch.int32) if x.dtype == f32 else x.view(torch.int16)


def _same(name, got, want):
    """Bit-for-bit equality, naming the first differing element."""
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    d = _bits(got) != _bits(want)
    if bool(d.any()):
        idx = tuple(int(i) for i in torch.nonzero(d)[0])
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r, want %r"
                             % (name, int(d.sum()), d.numel(), idx, float(got[idx]), float(want[idx])))


# ---- plan() restated --------------------------------------------------------------------------------------------------
def _choose_ksplit(out_tiles, nkb, workers, r):
    ksplit, best = 1, -1.0
    for ks in range(1, min(nkb // 16, 64) + 1):
        items = out_tiles * ks
        waves = _cdiv(items, workers)
        score = items / (waves * workers) / (1.0 + r * ks / nkb)
        if score > best:
            best, ksplit = score, ks
    return ksplit


def _plan(M, N, K, c16=0, acc=0, flags=0):
    """plan() in gemm_tc.cu: (tile width, planned split count).  The split count needs a workspace: without one there is
    no split.  (gemm_dispatch also narrows the tile of the tanh' epilogue to 128.)"""
    nsm = _nsm()
    num_m, nkb = _cdiv(M, BM), _cdiv(K, BK)
    wide_tiles = num_m * (N // 256)
    wide = N % 256 == 0 and (wide_tiles >= nsm or (not c16 and nkb >= 64 and wide_tiles >= 8))
    if not wide and N % 256 == 128 and N >= 512 and num_m >= 4 * nsm and acc == 0:
        wide = True
    low = bool(flags & CORESIDENT)
    if low:
        wide = False
    fixed = bool(flags & FIXED_K)            # the tile width follows N alone and K is never split
    if fixed:
        wide = N % 256 == 0
    bn = 256 if wide else 128
    out_tiles = num_m * _cdiv(N, bn)
    ks = 1
    if not low and not fixed and not c16 and nkb >= 64 and out_tiles < nsm:
        ks = _choose_ksplit(out_tiles, nkb, nsm, 32.0 if bn == 256 else 16.0)
    return bn, ks


def _n_inner(M, N, bn, ksplit):
    """Sched::n_inner of gemm_tc_kernel: ksplit == 1 and num_m >= 2 x the grid (one CTA per SM, at most one per item)."""
    num_m = _cdiv(M, BM)
    grid = min(num_m * _cdiv(N, bn) * ksplit, _nsm())
    return ksplit == 1 and num_m >= 2 * grid


def _partials(a_mn, c16, acc, M, N, K, flags=0):
    return int(_lib().eb_gemm_bf16_partials(a_mn, c16, acc, M, N, K, flags))


def _config(a_mn, M, N, K, c16=0, acc=0, flags=0):
    """(tile width, planned split count, n_inner) of a product, with the split count checked against the library."""
    bn, ks = _plan(M, N, K, c16, acc, flags)
    assert _partials(a_mn, c16, acc, M, N, K, flags) == (ks * M * N if ks > 1 else 0), "_plan disagrees with plan()"
    return bn, ks, _n_inner(M, N, bn, 1)


def _n_add(K, ksplit=1):
    """Longest fp32 summation chain of one output element: K products through wgmma, then one add per split partial."""
    return K + (ksplit if ksplit > 1 else 0)


# ---- operands and calls -----------------------------------------------------------------------------------------------
def _operands(M, N, K, kind, seed):
    """Logical bf16 A [M,K] and B [N,K] (C = A B^T)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, device=DEV, generator=g)
    b = torch.randn(N, K, device=DEV, generator=g)
    if kind == "wide":             # magnitudes 2^-20 ... 2^20 in one contraction
        a = a * torch.exp2(torch.randint(-20, 21, (M, K), device=DEV, generator=g).float())
        b = b * torch.exp2(torch.randint(-20, 21, (N, K), device=DEV, generator=g).float())
    elif kind == "zeros":          # exact-zero rows of A and of B: exact-zero rows and columns of C
        a[torch.arange(M, device=DEV) % 5 == 2] = 0
        b[torch.arange(N, device=DEV) % 7 == 3] = 0
    elif kind == "cancel":         # the second half of the contraction cancels the first, except two small terms
        h = K // 2
        a[:, h:2 * h] = -a[:, :h]
        b[:, h:2 * h] = b[:, :h]
        a[:, h - 1] = torch.randn(M, device=DEV, generator=g) * 2.0 ** -12
        a[:, 2 * h - 1] = torch.randn(M, device=DEV, generator=g) * 2.0 ** -12
    else:
        assert kind == "normal", kind
    return a.bfloat16(), b.bfloat16()


def _store(x, mn):
    """Storage of a logical [rows, K] operand: K-major as is, MN-major as [K, rows]."""
    return x.t().contiguous() if mn else x.contiguous()


def _out(M, N, dtype, init=None):
    """[M+1, N] NaN-filled buffer: rows [0, M) are the output (prefilled with `init` for accumulate), row M a guard."""
    buf = torch.full((M + 1, N), float("nan"), dtype=dtype, device=DEV)
    if init is not None:
        buf[:M] = init
    return buf


def _guard(name, buf, M):
    assert bool(torch.isnan(buf[M].float()).all()), name + ": a store went past the last row"


def _gemm(name, A, a_mn, B, b_mn, M, N, K, dtype=f32, bias=None, init=None, flags=0, ws=None, aux=None):
    """One eb_gemm_bf16_ex (or eb_gemm_bf16_dtanh when aux is given) call into a guarded buffer; returns C [M, N]."""
    buf = _out(M, N, dtype, init)
    L = _lib()
    if aux is not None:
        st = L.eb_gemm_bf16_dtanh(_p(A), a_mn, _p(B), b_mn, _p(buf), _p(aux), M, N, K, _stream())
    else:
        st = L.eb_gemm_bf16_ex(_p(A), a_mn, _p(B), b_mn, _p(buf), int(dtype == bf16), _p(bias), int(init is not None),
                               M, N, K, flags, _p(ws), 0 if ws is None else ws.numel(), _stream())
    assert st == 0, "%s: status %d" % (name, st)
    torch.cuda.synchronize()
    _guard(name, buf, M)
    return buf[:M]


class Case:
    """A product of logical bf16 operands in one storage layout."""

    def __init__(self, name, M, N, K, a_mn, b_mn, kind="normal", seed=0):
        self.name, self.M, self.N, self.K, self.a_mn, self.b_mn = name, M, N, K, a_mn, b_mn
        self.a, self.b = _operands(M, N, K, kind, seed)
        self.A, self.B = _store(self.a, a_mn), _store(self.b, b_mn)
        self.S = self.a.double() @ self.b.double().t()
        self.R = self.a.double().abs() @ self.b.double().abs().t()

    def gemm(self, label, **kw):
        return _gemm("%s %s" % (self.name, label), self.A, self.a_mn, self.B, self.b_mn, self.M, self.N, self.K, **kw)

    def check_raw(self, label, P, ksplit=1):
        _report(self.name, label, P, self.S, _n_add(self.K, ksplit) * UTC * self.R)


def _relations(c, P, flags=0, tag=""):
    """The bitwise epilogue relations on the raw product P of case c (bias, accumulate, bf16 out, dtanh)."""
    M, N = c.M, c.N
    g = torch.Generator(device=DEV).manual_seed(M * 131 + N)
    bias = torch.randn(N, device=DEV, generator=g)
    c0 = torch.randn(M, N, device=DEV, generator=g)
    c16 = torch.randn(M, N, device=DEV, generator=g).bfloat16()
    n = c.name + tag
    _same(n + " + bias", c.gemm("bias", bias=bias, flags=flags), P + bias)
    _same(n + " accumulate", c.gemm("acc", bias=bias, init=c0, flags=flags), (P + bias) + c0)
    _same(n + " accumulate, no bias", c.gemm("acc", init=c0, flags=flags), P + c0)
    _same(n + " bf16", c.gemm("bf16", dtype=bf16, bias=bias, flags=flags), (P + bias).to(bf16))
    _same(n + " bf16 no bias", c.gemm("bf16", dtype=bf16, flags=flags), P.to(bf16))
    _same(n + " bf16 accumulate", c.gemm("bf16 acc", dtype=bf16, bias=bias, init=c16, flags=flags),
          ((P + bias) + c16.float()).to(bf16))
    if N % 4 == 0 and flags == 0:
        h = torch.tanh(torch.randn(M, N, device=DEV, generator=g)).bfloat16()
        hf = h.float()
        _same(n + " dtanh", c.gemm("dtanh", dtype=bf16, aux=h), (P * (1 - hf * hf)).to(bf16))


def _slices_match(c, P, tag=""):
    """P bitwise equals the same A against 128-column slices of B (128 x 128 tiles)."""
    for j in range(_cdiv(c.N, 128)):
        n0, n1 = 128 * j, min(c.N, 128 * j + 128)
        Bj = c.B[n0:n1] if not c.b_mn else c.B[:, n0:n1].contiguous()     # K-major: a pointer offset
        Pj = _gemm("%s slice %d" % (c.name, j), c.A, c.a_mn, Bj, c.b_mn, c.M, n1 - n0, c.K)
        _same("%s%s: 128-column slice %d vs the full product" % (c.name, tag, j), Pj, P[:, n0:n1])


# ---- 1 / 3: the shape matrix ------------------------------------------------------------------------------------------
def _matrix():
    """Every layout against every M and N it admits (the contiguous dimension of an operand is a multiple of 8), with the
    K values and operand kinds cycled through them."""
    Ms_k = [1, 8, 63, 64, 65, 127, 129]                  # M < 64: the second consumer warpgroup owns no rows
    Ms_mn = [8, 64, 136, 192, 264, 128]                  # MN-major A: 128 k + r, r in (0, 64]: its second TMA box is empty
    Ns_k = [1, 3, 5, 127, 8, 24, 120, 136, 384, 640, 1024]   # odd N: the scalar stores
    Ns_mn = [8, 24, 120, 136, 384, 640, 1024]
    Ks = [8, 24, 72, 120, 184, 640]                      # < one k-block, 64 n + 8 / 64 n + 56 tails, the joint's J
    kinds = ["normal", "wide", "zeros", "cancel"]
    out = []
    for a_mn in (0, 1):
        for b_mn in (0, 1):
            Ms, Ns = (Ms_mn if a_mn else Ms_k), (Ns_mn if b_mn else Ns_k)
            for i in range(max(len(Ms), len(Ns))):
                M, N = Ms[i % len(Ms)], Ns[i % len(Ns)]
                K = Ks[(i + 2 * a_mn + b_mn) % len(Ks)]
                kind = kinds[(i + a_mn) % len(kinds)]
                out.append(("%s%s-M%d-N%d-K%d-%s" % ("t" if a_mn else "n", "n" if b_mn else "t", M, N, K, kind),
                            M, N, K, a_mn, b_mn, kind))
    return out


MATRIX = _matrix()


@pytest.mark.parametrize("name,M,N,K,a_mn,b_mn,kind", MATRIX, ids=[m[0] for m in MATRIX])
def test_gemm_bf16_shape_matrix(name, M, N, K, a_mn, b_mn, kind):
    c = Case(name, M, N, K, a_mn, b_mn, kind, seed=len(name) + M + N + K)
    bn, ks, _ = _config(a_mn, M, N, K)
    assert bn == 128 and ks == 1, "the matrix holds small products: 128-wide tiles, no split"
    P = c.gemm("raw")
    c.check_raw("raw", P)
    _same(name + " repeated launch", c.gemm("raw"), P)
    _relations(c, P)
    if not a_mn and not b_mn:
        Pl = c.gemm("co-resident", flags=CORESIDENT)
        _same(name + " co-resident vs default", Pl, P)
        _relations(c, P, flags=CORESIDENT, tag=" (co-resident)")


# ---- 2: configurations: tile widths, co-resident, schedules -----------------------------------------------------------
def _config_case(name, nsm):
    """name -> (M, N, K, a_mn, b_mn, expected tile width, expected n_inner), with the shapes derived from the SM count.
    Layout letters as in ops.gemm_bf16's names: A K-major 'n' / MN-major 't', then B K-major 't' / MN-major 'n'."""
    wide_m = BM * _cdiv(nsm, 4) - 40                     # N = 1024: >= #SMs wide tiles, ragged last row block
    sched_m = BM * (2 * nsm - 1)                         # 2 x #SMs row blocks
    table = {
        # plan(): N % 256 == 0 and wide_tiles >= #SMs
        "wide-nt": (wide_m, 1024, 136, 0, 0, 256, False),
        "wide-nn": (wide_m, 1024, 184, 0, 1, 256, False),
        "wide-tn": (wide_m, 1024, 72, 1, 1, 256, False),
        "wide-tt": (wide_m, 1024, 640, 1, 0, 256, False),
        # plan(): fp32 output, >= 64 k-blocks, >= 8 wide tiles (no workspace: no split)
        "wide-wgrad-tn": (1024, 256, 64 * 64 + 8, 1, 1, 256, False),
        # plan(): N % 256 == 128, N >= 512, >= 4 x #SMs row blocks, no accumulate; n_inner (num_m >= 2 x #SMs)
        "wide-overhang-nt": (BM * 4 * nsm + 77, 640, 64, 0, 0, 256, True),
        # the layer wavefront's per-chunk input GEMM (B = 32 rows x 12 frames, 4H = 4096, I = 1024)
        "coresident-wavefront-nt": (32 * 12, 4096, 1024, 0, 0, 128, False),
        # > #SMs narrow tiles, round robin, ragged last row block
        "many-tiles-nt": (BM * 40 + 17, 640, 72, 0, 0, 128, False),
        # just below / at 2 x #SMs row blocks: round robin / n_inner (the pair is compared row by row)
        "sched-rr-nt": (sched_m - 5, 384, 120, 0, 0, 128, False),
        "sched-ninner-nt": (sched_m + 3, 384, 120, 0, 0, 128, True),
        "sched-rr-tt": (sched_m - 8, 136, 24, 1, 0, 128, False),
        "sched-ninner-tt": (sched_m + 8, 136, 24, 1, 0, 128, True),
    }
    return table[name]


CONFIG_CASES = ["wide-nt", "wide-nn", "wide-tn", "wide-tt", "wide-wgrad-tn", "wide-overhang-nt",
                "coresident-wavefront-nt", "many-tiles-nt", "sched-ninner-nt", "sched-ninner-tt"]


@pytest.mark.parametrize("name", CONFIG_CASES)
def test_gemm_bf16_configurations(name):
    """The configuration plan() picks for the shape, then the same product on 128-column slices of B (128 x 128 tiles),
    in the co-resident configuration (K-major operands), and for the schedule cases on fewer row blocks (the other
    schedule): all bitwise equal.  The epilogue relations hold on the configuration's own raw product."""
    M, N, K, a_mn, b_mn, want_bn, want_inner = _config_case(name, _nsm())
    bn, ks, inner = _config(a_mn, M, N, K)
    assert (bn, inner) == (want_bn, want_inner), (name, bn, inner)
    c = Case(name, M, N, K, a_mn, b_mn, "normal", seed=M + N)
    P = c.gemm("raw")
    c.check_raw("raw", P)
    _same(name + " repeated launch", c.gemm("raw"), P)
    if bn == 256:
        _slices_match(c, P)
    if not a_mn and not b_mn:
        _same(name + " co-resident vs default", c.gemm("co-resident", flags=CORESIDENT), P)
    if name.startswith("sched-"):
        other = name.replace("ninner", "rr")
        M2 = _config_case(other, _nsm())[0]
        assert _n_inner(M2, N, 128, 1) != inner
        A2 = c.A[:M2] if not a_mn else c.A[:, :M2].contiguous()
        P2 = _gemm(other, A2, a_mn, c.B, b_mn, M2, N, K)
        _same("%s vs %s (first %d rows)" % (other, name, M2), P2, P[:M2])
    _relations(c, P)


# ---- 1: split-K -------------------------------------------------------------------------------------------------------
def _split_sum(c, ksplit, bias=None, init=None):
    """C_before (or 0) plus the partial tiles in split order; partial s is its own no-split call on the K-slice of
    k-blocks [s kb_per, (s+1) kb_per), with the bias in partial 0 only (an empty split adds zeros)."""
    nkb = _cdiv(c.K, BK)
    kb_per = _cdiv(nkb, ksplit)
    v = init.clone() if init is not None else torch.zeros(c.M, c.N, device=DEV)
    for s in range(ksplit):
        k0, k1 = s * kb_per * BK, min(c.K, (s + 1) * kb_per * BK)
        if k0 >= c.K:
            part = torch.zeros(c.M, c.N, device=DEV) + (bias if s == 0 else 0)
        else:
            part = _gemm("%s partial %d" % (c.name, s), _store(c.a[:, k0:k1], c.a_mn), c.a_mn,
                         _store(c.b[:, k0:k1], c.b_mn), c.b_mn, c.M, c.N, k1 - k0, bias=bias if s == 0 else None)
        v = v + part
    return v


def _split_case(name):
    """name -> (M, N, K, a_mn, b_mn, workspace splits or None for the planned count)"""
    return {
        "splitk-tn": (320, 384, 64 * 97, 1, 1, None),                 # the weight-gradient layout
        "splitk-nt": (200, 136, 64 * 80 + 56, 0, 0, None),
        "splitk-wide-tn": (1024, 256, 64 * 64 + 8, 1, 1, None),       # 128 x 256 tiles, 8 of them
        "splitk-empty-last-nt": (128, 128, 64 * 400 - 8, 0, 0, 21),   # 21 splits of 20 k-blocks over 400: the last is empty
        "splitk-shrunk-tt": (256, 384, 64 * 150, 1, 0, 3),            # a workspace for 3 of the planned splits
    }[name]


SPLIT_CASES = ["splitk-tn", "splitk-nt", "splitk-wide-tn", "splitk-empty-last-nt", "splitk-shrunk-tt"]


@pytest.mark.parametrize("name", SPLIT_CASES)
def test_gemm_bf16_split_k(name):
    """fp32-output products with a long contraction and few tiles split K: the split product within the fp64 bar (one
    more add per split), and bitwise the split-order sum of its partials run as separate calls, with and without bias and
    accumulate; repeated launches give the same bits."""
    M, N, K, a_mn, b_mn, want = _split_case(name)
    bn, planned, _ = _config(a_mn, M, N, K)
    assert planned > 1, name + " must take the split-K path"
    floats = _partials(a_mn, 0, 0, M, N, K)
    if want is not None:
        assert planned >= want
        floats = want * M * N + M * N - 1                 # fit = floats // (M N)
    ws = torch.empty(floats, device=DEV)
    ksplit = min(planned, floats // (M * N))
    nkb = _cdiv(K, BK)
    kb_per = _cdiv(nkb, ksplit)
    empty = (ksplit - 1) * kb_per >= nkb
    assert empty == (name == "splitk-empty-last-nt"), (name, ksplit, kb_per, nkb)
    c = Case(name, M, N, K, a_mn, b_mn, "normal", seed=K)
    print("  %-44s tile %d, %d splits of %d k-blocks over %d" % (name, bn, ksplit, kb_per, nkb))
    P = c.gemm("split", ws=ws)
    c.check_raw("split", P, ksplit)
    _same(name + " repeated launch", c.gemm("split", ws=ws), P)
    _same(name + " vs its partials", P, _split_sum(c, ksplit))
    g = torch.Generator(device=DEV).manual_seed(N)
    bias = torch.randn(N, device=DEV, generator=g)
    c0 = torch.randn(M, N, device=DEV, generator=g)
    _same(name + " + bias vs its partials", c.gemm("split bias", bias=bias, ws=ws), _split_sum(c, ksplit, bias))
    _same(name + " accumulate vs its partials", c.gemm("split acc", bias=bias, init=c0, ws=ws),
          _split_sum(c, ksplit, bias, c0))
    # no workspace: one chain over all of K
    c.check_raw("no split", c.gemm("no split"))


# ---- EB_GEMM_FIXED_K: the serial encoder backward's dgrad GEMM ----------------------------------------------------------
# (name, M, N, K): A K-major, B MN-major (dG [rows, 4H] times W_ih [4H, I]).  N = 1024 at M = 300 would be split at the
# default plan (12 wide tiles, 64 k-blocks); FIXED_K keeps one chain over K.
FIXED_K_CASES = [("fixedk-M300-N1024-K4096", 300, 1024, 4096), ("fixedk-M200-N240-K4096", 200, 240, 4096),
                 ("fixedk-M129-N640-K72", 129, 640, 72)]


@pytest.mark.parametrize("name,M,N,K", FIXED_K_CASES, ids=[c[0] for c in FIXED_K_CASES])
def test_gemm_bf16_fixed_k(name, M, N, K):
    """EB_GEMM_FIXED_K: the tile width follows N alone (256 when N % 256 == 0) and K is never split.  The raw product is
    within the fp64 bar of one chain over K, and the epilogue relations hold on it."""
    bn, ks, _ = _config(0, M, N, K, flags=FIXED_K)
    assert (bn, ks) == (256 if N % 256 == 0 else 128, 1), (name, bn, ks)
    c = Case(name, M, N, K, 0, 1, "normal", seed=M + N + K)
    P = c.gemm("raw", flags=FIXED_K)
    c.check_raw("raw", P)
    _same(name + " repeated launch", c.gemm("raw", flags=FIXED_K), P)
    _relations(c, P, flags=FIXED_K, tag=" (fixed K)")


@pytest.mark.parametrize("N", [1024, 240])
def test_gemm_bf16_fixed_k_equals_coresident_row_blocks(N):
    """The invariant both encoder backward schedules rest on: the serial schedule's whole-layer dgrad GEMM (FIXED_K, A
    K-major, B MN-major, accumulated onto fp32 C) is bitwise the chunked schedule's co-resident GEMMs (B transposed to
    K-major) on row blocks accumulated onto the same C: one row, blocks that are not a multiple of 128, and the
    wavefront's group sizes at B = 32 (3 x 168 and 2 x 168 + 160 frames, 3 x 84 on the reduced axis)."""
    K = 4096
    blocks = [1, 77, 333, 32 * 504, 32 * 496, 32 * 252]
    M = sum(blocks)
    g = torch.Generator(device=DEV).manual_seed(N)
    A = (torch.randn(M, K, device=DEV, generator=g) * 0.1).bfloat16()
    Bt = (torch.randn(N, K, device=DEV, generator=g) / 32).bfloat16()         # W_ih^T: [I, 4H], K-major
    Bn = Bt.t().contiguous()                                                  # W_ih: [4H, I], MN-major
    C0 = torch.randn(M, N, device=DEV, generator=g)
    assert _partials(0, 0, 1, M, N, K, FIXED_K) == 0
    whole = _gemm("fixed-K whole", A, 0, Bn, 1, M, N, K, init=C0, flags=FIXED_K)
    a = 0
    for n in blocks:
        part = _gemm("co-resident rows [%d, %d)" % (a, a + n), A[a:a + n], 0, Bt, 0, n, N, K, init=C0[a:a + n],
                     flags=CORESIDENT)
        _same("N%d: co-resident rows [%d, %d) vs fixed-K whole" % (N, a, a + n), part, whole[a:a + n])
        a += n


# ---- the joint's logits ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T,U,V,J,with_b2", [(2, 37, 5, 333, 640, True), (3, 20, 9, 1024, 640, False),
                                               (4, 150, 30, 1024, 640, True), (1, 7, 3, 136, 72, True)])
def test_joint_logits_lse_logits16(B, T, U, V, J, with_b2):
    """eb_joint_logits_lse's bf16 logits are bf16_rn(P + b2), P the plain GEMM of the same operands (K-major B)."""
    M = B * T * U
    name = "lse-B%d-T%d-U%d-V%d-J%d" % (B, T, U, V, J)
    c = Case(name, M, V, J, 0, 0, "normal", seed=M + V)
    g = torch.Generator(device=DEV).manual_seed(V)
    b2 = torch.randn(V, device=DEV, generator=g) if with_b2 else None
    xlen = torch.randint(1, T + 1, (B,), device=DEV, generator=g, dtype=torch.int32)
    ylen = torch.randint(0, U, (B,), device=DEV, generator=g, dtype=torch.int32)
    labels = torch.randint(1, V, (B, max(U - 1, 1)), device=DEV, generator=g, dtype=torch.int32)
    stats = [torch.zeros(M, device=DEV) for _ in range(3)]
    buf = _out(M, V, bf16)
    st = _lib().eb_joint_logits_lse(_p(c.A), _p(c.B), _p(b2), _p(buf), _p(labels), _p(xlen), _p(ylen), *map(_p, stats),
                                    B, T, U, V, J, 0, _stream())
    assert st == 0
    torch.cuda.synchronize()
    _guard(name, buf, M)
    P = c.gemm("raw")
    c.check_raw("raw", P)
    _same(name + " logits16", buf[:M], (P + b2 if with_b2 else P).to(bf16))


# ---- every configuration is reached by a named case --------------------------------------------------------------------
def test_every_configuration_is_reached():
    """From the parametrisation and plan(): both tile widths, the co-resident configuration, both schedules, split-K
    with and without an empty last split, odd N, M < 64, MN-major A with its second row box empty, bf16 + accumulate and
    dtanh (run by every matrix and configuration case)."""
    nsm = _nsm()
    seen = set()
    for name in CONFIG_CASES + [n.replace("ninner", "rr") for n in CONFIG_CASES if n.startswith("sched-ninner")]:
        M, N, K, a_mn, b_mn, _, _ = _config_case(name, nsm)
        bn, _, inner = _config(a_mn, M, N, K)
        seen.add("tile %d" % bn)
        seen.add("n_inner" if inner else "round robin")
        if not a_mn and not b_mn:
            seen.add("co-resident")
        if N % 4 == 0:
            seen.add("dtanh")
    for _, M, N, K, a_mn, b_mn, _ in MATRIX:
        if N % 2:
            seen.add("odd N")
        if M < 64:
            seen.add("M < 64")
        if a_mn and 0 < M % 128 <= 64:
            seen.add("MN-major A, empty second box")
        seen.add("bf16 accumulate")
    for name in SPLIT_CASES:
        M, N, K, a_mn, b_mn, want = _split_case(name)
        if _partials(a_mn, 0, 0, M, N, K) > 0:
            seen.add("split-K")
            ks = want or _partials(a_mn, 0, 0, M, N, K) // (M * N)
            if (ks - 1) * _cdiv(_cdiv(K, BK), ks) >= _cdiv(K, BK):
                seen.add("empty last split")
    need = {"tile 128", "tile 256", "co-resident", "n_inner", "round robin", "split-K", "empty last split", "odd N",
            "M < 64", "MN-major A, empty second box", "bf16 accumulate", "dtanh"}
    assert need <= seen, need - seen


# ---- 4: the fp32 GEMM -------------------------------------------------------------------------------------------------
def _f32(A, sam, sak, B, sbk, sbn, M, N, K, bias=None, alpha=1.0, beta=0.0, init=None, ldc=None):
    """eb_gemm_f32 into a NaN-filled [M+1, ldc] buffer; returns the buffer."""
    ldc = ldc or N
    buf = torch.full((M + 1, ldc), float("nan"), device=DEV)
    if init is not None:
        buf[:M, :N] = init
    st = _lib().eb_gemm_f32(_p(A), sam, sak, _p(B), sbk, sbn, _p(buf), ldc, _p(bias), M, N, K, alpha, beta, _stream())
    assert st == 0
    torch.cuda.synchronize()
    return buf


def _f32_layouts(a, b):
    """The four stride layouts of logical fp32 A [M,K], B [K,N]: (label, A storage, sam, sak, B storage, sbk, sbn)."""
    M, K = a.shape
    N = b.shape[1]
    at, bt = a.t().contiguous(), b.t().contiguous()
    return [("A[M,K] B[K,N]", a, K, 1, b, N, 1), ("A[M,K] B[N,K]", a, K, 1, bt, 1, K),
            ("A[K,M] B[K,N]", at, 1, M, b, N, 1), ("A[K,M] B[N,K]", at, 1, M, bt, 1, K)]


@pytest.mark.parametrize("M,N,K", [(1, 1, 1), (37, 5, 17), (65, 70, 33), (130, 129, 7), (70, 200, 515), (3, 66, 1000)])
def test_gemm_f32_per_element_and_layouts(M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M * N + K)
    a = torch.randn(M, K, device=DEV, generator=g)
    b = torch.randn(K, N, device=DEV, generator=g)
    a[:, K // 2] *= 2.0 ** 20                              # one column of large terms
    S = a.double() @ b.double()
    R = a.double().abs() @ b.double().abs()
    name = "f32-M%d-N%d-K%d" % (M, N, K)
    lay = _f32_layouts(a, b)
    P = None
    for label, A, sam, sak, B, sbk, sbn in lay:
        buf = _f32(A, sam, sak, B, sbk, sbn, M, N, K)
        _guard(name, buf, M)
        if P is None:
            P = buf[:M].clone()
            _report(name, "raw", P, S, K * U24 * R)
        else:
            _same("%s %s vs %s" % (name, label, lay[0][0]), buf[:M], P)
    A, sam, sak, B, sbk, sbn = lay[0][1:]
    bias = torch.randn(N, device=DEV, generator=g)
    c0 = torch.randn(M, N, device=DEV, generator=g)
    _same(name + " + bias", _f32(A, sam, sak, B, sbk, sbn, M, N, K, bias=bias)[:M], P + bias)
    _same(name + " beta 1", _f32(A, sam, sak, B, sbk, sbn, M, N, K, beta=1.0, init=c0)[:M], P + c0)
    _same(name + " bias, beta 1", _f32(A, sam, sak, B, sbk, sbn, M, N, K, bias=bias, beta=1.0, init=c0)[:M],
          (P + bias) + c0)
    # ldc > N: columns [N, ldc) and the guard row untouched
    buf = _f32(A, sam, sak, B, sbk, sbn, M, N, K, bias=bias, beta=1.0, init=c0, ldc=N + 3)
    _same(name + " ldc > N", buf[:M, :N], (P + bias) + c0)
    assert bool(torch.isnan(buf[:, N:]).all()) and bool(torch.isnan(buf[M]).all()), name + ": store outside [M, N)"
    # general alpha / beta: fp64 bar with the roundings of alpha * acc, + bias and + beta * C
    alpha, beta = 0.37, -0.61
    got = _f32(A, sam, sak, B, sbk, sbn, M, N, K, bias=bias, alpha=alpha, beta=beta, init=c0)[:M]
    bd, cd = bias.double(), c0.double()
    ref = alpha * S + bd + beta * cd
    bar = abs(alpha) * K * U24 * R + 3 * U24 * (abs(alpha) * S.abs() + bd.abs() + abs(beta) * cd.abs())
    _report(name, "alpha-beta", got, ref, bar)


@pytest.mark.parametrize("hop,K,N,M", [(160, 400, 402, 37), (16, 48, 10, 130), (1, 5, 3, 70)])
def test_gemm_f32_overlapping_view(hop, K, N, M):
    """The front end's framing view (A(m,k) = x[m hop + k], hop < K: rows overlap) gives bitwise the product of its
    materialised copy, and is within the fp64 bar."""
    g = torch.Generator(device=DEV).manual_seed(hop + K)
    x = torch.randn((M - 1) * hop + K, device=DEV, generator=g)
    b = torch.randn(K, N, device=DEV, generator=g)
    frames = x.as_strided((M, K), (hop, 1)).contiguous()
    name = "f32-frames-hop%d-K%d" % (hop, K)
    got = _f32(x, hop, 1, b, N, 1, M, N, K)
    _guard(name, got, M)
    want = _f32(frames, K, 1, b, N, 1, M, N, K)
    _same(name + " view vs copy", got[:M], want[:M])
    _report(name, "raw", got[:M], frames.double() @ b.double(), K * U24 * (frames.double().abs() @ b.double().abs()))
