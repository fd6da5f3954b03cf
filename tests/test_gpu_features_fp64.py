"""Per-element fp64 parity and bitwise invariants of the per-utterance entries of csrc/frontend.cu, each through its C
entry point, and of the composed batch transform against its fp64 restatement on the module's own tables.  (The
equal-length entries eb_fe_preemph_pad, eb_fe_power, eb_fe_log_stack, eb_fe_mask and the framing-view eb_gemm_f32 are
pinned by test_gpu_glue_fp64.py and test_gpu_gemm_fp64.py.)

Error model.  The build uses no fast-math (IEEE division), but nvcc contracts a*b + c into one FMA.  u = 2^-24.

  eb_fe_preemph_pad_lens  reflect without edge repeat at each utterance's own L_b, zero from L_b + 2 pad to Lp:
                          bitwise without pre-emphasis; with it x_r - p x_{r-1} is one FMA or a product and a
                          difference, so |err| <= 2u (|x_r| + |p x_{r-1}|) (the glue test's bar).  Samples x[b, L_b:]
                          are NaN and the output must not change; with every L_b = L it is bitwise eb_fe_preemph_pad.
  eb_fe_log               logf(fl(x + off)): the add is one IEEE rounding (restated exactly in torch fp32), logf is
                          within ULP_LOGF = 1 ulp of the exact log of that sum (CUDA C++ Programming Guide); the test
                          measures the worst ulp count and prints it.  Mel values 1e-8 ... 1e-4 pin the offset itself:
                          there log(x + 1e-6) and log(x + 1e-20) differ by far more than the bar.
  eb_fe_finish            static channel: logf(fl(v + 1e-20f)) within 1 ulp of the exact log of the sum, or bitwise
                          when take_log = 0; frames >= ceil(L_b / hop) (use_mask) exactly 0.  d1, d2, the stacking index
                          out[b, t, s Cd + j C + c], the pad_to_divisible=False drop (after the deltas: frames [Fs, F)
                          feed the last kept frames' deltas) and the zero rows t >= T_b: BITWISE against
                          features_fp64.finish32 on the kernel's own static values, because (2 (p2 - m2) + (p1 - m1)) /
                          10 rounds the same with or without FMA contraction (2 x is exact) and the division is IEEE.
                          If the library is ever built with --use_fast_math this stops holding and these tests fail.
  eb_fe_deltas            bitwise against the same restatement, at every clamp pattern (F = 1, 2, 3, 5) and a long F.
  the composed chain      ops.fe_batch (build_batch_transform's test module) against features_fp64.chain on the module's
                          own fp32 tables, under the bar propagated stage by stage (features_fp64's docstring).

Every output goes into a NaN-prefilled buffer with guard elements behind it, and inputs that must not be read are NaN.
Each bar-based check prints its worst err/bar (pytest -s); DESIGN.md section 2 records the measured figures."""
import numpy as np
import pytest
import torch

from tests import features_fp64 as X

pytestmark = pytest.mark.gpu

f32, f64 = torch.float32, torch.float64
DEV = "cuda"
U24 = X.U24
G = 40                       # guard elements behind every flat output


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ok(st, name):
    assert st == 0, "%s: status %d" % (name, st)
    torch.cuda.synchronize()


def _bits(x):
    return x.contiguous().view(torch.int32)


def _same(name, got, want):
    """Bit-for-bit equality, naming the first differing element."""
    got, want = torch.as_tensor(got).cpu(), torch.as_tensor(want).cpu()
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    d = _bits(got) != _bits(want)
    if bool(d.any()):
        idx = tuple(int(i) for i in torch.nonzero(d)[0])
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r, want %r"
                             % (name, int(d.sum()), d.numel(), idx, float(got[idx]), float(want[idx])))


def _nan(n):
    return torch.full((n + G,), float("nan"), dtype=f32, device=DEV)


def _guard(name, buf, n):
    assert bool(torch.isnan(buf[n:]).all()), name + ": a store went past the end of the output"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ulp32(y):
    """The fp32 ulp at |y| (y fp64)."""
    return torch.from_numpy(np.spacing(np.abs(y.cpu().numpy()).astype(np.float32)).astype(np.float64))


def _cint(v):
    import ctypes
    return (ctypes.c_int * len(v))(*[int(i) for i in v])


# ---- eb_fe_preemph_pad_lens -------------------------------------------------------------------------------------------
def _padded_ref(x, lens, Lp, pad, p):
    """fp64 rows of the kernel's output (reflect without edge repeat at L_b, zero from L_b + 2 pad), their bar, and the
    fp32 rows without pre-emphasis."""
    B = x.shape[0]
    xd = x.double().cpu().numpy()
    ref, bar, raw = np.zeros((B, Lp)), np.zeros((B, Lp)), np.zeros((B, Lp), np.float32)
    i = np.arange(Lp)
    for b, Lb in enumerate(lens):
        r = i - pad
        r = np.where(r < 0, -r, r)
        r = np.where(r >= Lb, 2 * (Lb - 1) - r, r)
        inside = i < Lb + 2 * pad
        r = np.where(inside, r, 0)
        xr = xd[b, r]
        prev = np.where(r > 0, xd[b, np.maximum(r - 1, 0)], 0.0)
        ref[b] = np.where(inside, xr - p * prev, 0.0)
        bar[b] = np.where(inside, 2 * U24 * (np.abs(xr) + np.abs(p * prev)), 0.0)
        raw[b] = np.where(inside, xr, 0.0).astype(np.float32)
    return torch.from_numpy(ref), torch.from_numpy(bar), torch.from_numpy(raw)


# (name, L, pad, hop, lens): L_b = pad + 1 (the shortest reflect), L_b = L, L_b + 2 pad a multiple of hop, B = 1
PAD_CASES = [("shortest-reflect", 1000, 256, 200, [257, 1000, 600]),
             ("multiple-of-hop", 1200, 200, 200, [800, 1200, 333, 201]),
             ("B1", 777, 256, 160, [777]),
             ("B1-shortest", 300, 256, 100, [257]),
             ("pad-1", 50, 1, 7, [2, 50, 13])]


@pytest.mark.parametrize("name,L,pad,hop,lens", PAD_CASES, ids=[c[0] for c in PAD_CASES])
def test_preemph_pad_lens(name, L, pad, hop, lens):
    B = len(lens)
    Lp = -(-(L + 2 * pad) // hop) * hop
    x = torch.randn(B, L, device=DEV, generator=_gen(L + pad))
    xs = x.clone()
    for b, Lb in enumerate(lens):
        xs[b, Lb:] = float("nan")                          # past L_b: never read
    lens_dev = torch.tensor(lens, dtype=torch.int32, device=DEV)
    p = float(np.float32(0.97))
    ref, bar, raw = _padded_ref(x, lens, Lp, pad, p)
    Lib = _lib()
    outs = {}
    for use_pre in (0, 1):
        for src, tag in ((xs, "NaN past L_b"), (x, "clean")):
            xb = _nan(B * Lp)
            _ok(Lib.eb_fe_preemph_pad_lens(_p(src), _cint(lens), _p(lens_dev), _p(xb), B, L, Lp, pad, 0.97, use_pre,
                                           _stream()), "eb_fe_preemph_pad_lens")
            _guard(name, xb, B * Lp)
            outs[use_pre, tag] = xb[:B * Lp].view(B, Lp).cpu()
        _same("%s pre%d: NaN past L_b changes nothing" % (name, use_pre), outs[use_pre, "NaN past L_b"],
              outs[use_pre, "clean"])
    _same(name + " reflect at L_b, no pre-emphasis", outs[0, "clean"], raw)
    X.report(name + " reflect at L_b, pre-emphasis", outs[1, "clean"], ref, bar)


@pytest.mark.parametrize("use_pre", [0, 1])
def test_preemph_pad_lens_equal_lengths_is_preemph_pad(use_pre):
    B, L, pad, hop = 3, 4000, 256, 200
    Lp = -(-(L + 2 * pad) // hop) * hop
    x = torch.randn(B, L, device=DEV, generator=_gen(5))
    a, b = _nan(B * Lp), _nan(B * Lp)
    Lib = _lib()
    lens = [L] * B
    _ok(Lib.eb_fe_preemph_pad_lens(_p(x), _cint(lens), _p(torch.tensor(lens, dtype=torch.int32, device=DEV)), _p(a),
                                   B, L, Lp, pad, 0.97, use_pre, _stream()), "eb_fe_preemph_pad_lens")
    _ok(Lib.eb_fe_preemph_pad(_p(x), _p(b), B, L, Lp, pad, 0.97, use_pre, _stream()), "eb_fe_preemph_pad")
    _same("preemph_pad_lens at L_b = L vs preemph_pad", a, b)


# ---- eb_fe_log --------------------------------------------------------------------------------------------------------
def test_fe_log():
    n = 3 * 256 * 97 + 5                                   # not a multiple of the block
    g = _gen(11)
    x = torch.exp(torch.empty(n, device=DEV).uniform_(np.log(1e-12), np.log(1e6), generator=g))
    x[: n // 4] = torch.exp(torch.empty(n // 4, device=DEV).uniform_(np.log(1e-8), np.log(1e-4), generator=g))
    x[::101] = 0.0                                          # log(0 + offset)
    xb = _nan(n)
    xb[:n] = x
    _ok(_lib().eb_fe_log(_p(xb), n, 1e-6, _stream()), "eb_fe_log")
    _guard("fe_log", xb, n)
    z = (x + np.float32(1e-6)).double().cpu()              # the fp32 add, exactly as the kernel rounds it
    ref = torch.log(z)
    got = xb[:n].double().cpu()
    ulps = float(((got - ref).abs() / _ulp32(ref)).max())
    print("  fe_log: logf measured worst %.3g ulp (bar %g ulp)" % (ulps, X.ULP_LOGF))
    bar = X.ULP_LOGF * _ulp32(ref)
    X.report("fe_log log(x + 1e-6)", got, ref, bar)
    # the offset is pinned: 1e-20 in its place would miss the bar by orders of magnitude over the small mel values
    other = torch.log((x + np.float32(1e-20)).double().cpu())
    assert int(((other - ref).abs() > 1e3 * bar).sum()) > n // 8


# ---- eb_fe_finish -----------------------------------------------------------------------------------------------------
# (name, C, hop, n_stack, take_log, use_mask, delta, pad_to_divisible, lens): hop divides L_b (the mask takes the last
# frame), L_b < hop (F_b = 1), frames dropped by pad_to_divisible=False, T_b = 1 and T_b = 0 in a ragged batch
FINISH_CASES = [
    ("log-mask-n1-delta", 40, 200, 1, 1, 1, 1, 1, [4000, 3999, 200, 199]),
    ("log-mask-n3-delta-drop", 40, 200, 3, 1, 1, 1, 0, [4000, 3999, 1000, 450]),
    ("log-mask-n2-delta-drop", 40, 200, 2, 1, 1, 1, 0, [4200, 2000, 401]),
    ("log-mask-n3-static", 80, 200, 3, 1, 1, 0, 1, [2400, 2399, 601]),
    ("log-nomask-n1-static", 5, 160, 1, 1, 0, 0, 1, [1600, 321]),
    ("nolog-n2-delta", 13, 100, 2, 0, 0, 1, 1, [1000, 777, 50]),
    ("nolog-n2-delta-drop", 20, 100, 2, 0, 0, 1, 0, [1234, 999, 250]),
    ("nolog-mask-n3-delta-drop-T0", 7, 100, 3, 0, 1, 1, 0, [700, 599, 300, 150]),
]


def _geometry(lens, hop, n, use_mask, ptd):
    F = [1 + L // hop for L in lens]
    seq = [-(-L // hop) if use_mask else f for L, f in zip(lens, F)]
    Fs = [f if ptd else f - f % n for f in F]
    T = [-(-f // n) if ptd else f // n for f in F]
    return F, seq, Fs, T


def _finish(feat, lens, R, hop, C, n, t_out, take_log, use_mask, delta, ptd, name):
    B = len(lens)
    W = C * (3 if delta else 1) * n
    ob = _nan(B * t_out * W)
    _ok(_lib().eb_fe_finish(_p(feat), _p(ob), _cint(lens), _p(torch.tensor(lens, dtype=torch.int32, device=DEV)), B, R,
                            hop, C, n, t_out, take_log, use_mask, delta, ptd, _stream()), "eb_fe_finish")
    _guard(name, ob, B * t_out * W)
    return ob[:B * t_out * W].view(B, t_out, W).cpu()


@pytest.mark.parametrize("name,C,hop,n,take_log,use_mask,delta,ptd,lens", FINISH_CASES, ids=[c[0] for c in FINISH_CASES])
def test_fe_finish(name, C, hop, n, take_log, use_mask, delta, ptd, lens):
    B = len(lens)
    F, seq, Fs, T = _geometry(lens, hop, n, use_mask, ptd)
    R = max(F) + 2
    g = _gen(len(name) * 7 + C)
    if take_log:
        feat = torch.exp(4 * torch.randn(B, R, C, device=DEV, generator=g))
        feat[:, ::3, ::4] = 0.0                            # log(0 + 1e-20)
    else:
        feat = torch.randn(B, R, C, device=DEV, generator=g)
    for b in range(B):
        feat[b, seq[b]:] = float("nan")                    # masked frames and the unused slots are never read
    planted = feat.cpu().numpy()
    # the kernel's static values of every frame < F_b: a pad_to_divisible, one-frame, static-only launch
    stat = _finish(feat, lens, R, hop, C, 1, max(F), take_log, use_mask, 0, 1, name + " statics")
    for b in range(B):
        _same("%s b%d statics are +0 from frame %d" % (name, b, seq[b]), stat[b, seq[b]:],
              torch.zeros(max(F) - seq[b], C))
        v = torch.from_numpy(planted[b, :seq[b]])
        if take_log:
            ref = torch.log((v + np.float32(1e-20)).double())
            X.report("%s b%d static logf(v + 1e-20f)" % (name, b), stat[b, :seq[b]], ref,
                     X.ULP_LOGF * _ulp32(ref))
        else:
            _same("%s b%d static copy" % (name, b), stat[b, :seq[b]], v)
    t_out = max(T) + 1                                      # every utterance has zero rows behind it
    out = _finish(feat, lens, R, hop, C, n, t_out, take_log, use_mask, delta, ptd, name)
    for b in range(B):
        want = X.finish32(stat[b, :F[b]].numpy(), F[b], Fs[b], n, t_out, delta)
        _same("%s b%d F%d Fs%d T%d vs finish32" % (name, b, F[b], Fs[b], T[b]), out[b], torch.from_numpy(want))
        _same("%s b%d rows t >= T_b are +0" % (name, b), out[b, T[b]:], torch.zeros(t_out - T[b], out.shape[2]))


@pytest.mark.parametrize("F", [1, 2, 3, 5, 4099])
def test_fe_deltas(F):
    B, C = 2, 7 if F < 4099 else 80
    g = _gen(F)
    feat = torch.randn(B, F, C, device=DEV, generator=g) * torch.exp(torch.randn(1, 1, C, device=DEV, generator=g))
    n = B * F * 3 * C
    ob = _nan(n)
    _ok(_lib().eb_fe_deltas(_p(feat), _p(ob), B, F, C, _stream()), "eb_fe_deltas")
    _guard("fe_deltas", ob, n)
    out = ob[:n].view(B, F, 3 * C).cpu()
    for b in range(B):
        want = X.finish32(feat[b].cpu().numpy(), F, F, 1, F, True)
        _same("fe_deltas F%d b%d vs finish32" % (F, b), out[b], torch.from_numpy(want))


# ---- the composed chain on the module's own tables --------------------------------------------------------------------
def speech_like(lens, seed):
    g = torch.Generator().manual_seed(seed)
    L = max(lens)
    t = torch.arange(L) / 16000.0
    x = torch.zeros(len(lens), L)
    for b, n in enumerate(lens):
        env = 0.5 + 0.5 * torch.sin(2 * np.pi * 3.0 * t[:n] + b)
        x[b, :n] = 0.05 * torch.randn(n, generator=g) + env * (0.4 * torch.sin(2 * np.pi * (150.0 + 40 * b) * t[:n]) +
                                                               0.1 * torch.sin(2 * np.pi * 2500.0 * t[:n]))
    return x


CHAIN_CASES = [("logfbank", 512, 400, True, 3, False), ("logfbank", 512, 320, False, 1, True),
               ("mfcc", 512, 400, True, 2, True), ("mfcc", 400, 400, True, 3, False),
               ("melspec", 512, 400, True, 3, True), ("melspec", 400, 400, False, 1, False)]


@pytest.mark.parametrize("ft,n_fft,win,delta,ds,ptd", CHAIN_CASES)
def test_chain_on_the_module_tables(ft, n_fft, win, delta, ds, ptd):
    from edgedict_b200.rnnt.features import build_batch_transform
    lens = [48000, 30117, 12800, 7201, 601]
    x = speech_like(lens, 11).to(DEV)
    _, test, _ = build_batch_transform(ft, 40, n_fft=n_fft, win_length=win, hop_length=200, delta=delta,
                                       downsample=ds, pad_to_divisible=ptd, dither=0)
    test = test.to(DEV)
    got, xlen = test(x, lens)
    basis, fbT, dct, pre = X.module_tables(test)
    val, bar, ok = X.chain(x, lens, ft, basis, fbT, n_fft, 200, ds, delta, ptd, preemph=pre, dct=dct)
    assert got.shape == val.shape
    X.report("chain %s n_fft %d win %d d%d ds%d p%d (module tables)" % (ft, n_fft, win, delta, ds, ptd), got, val,
             bar, ok)
