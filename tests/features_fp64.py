"""The batched feature transform (ops.fe_batch -> csrc/frontend.cu) restated twice (TEST INFRASTRUCTURE):

* ``chain``: in fp64 from the module's own fp32 tables (DFT basis, filterbank, DCT matrix, fp32(0.97)), with a
  per-element first-order bound on the device's distance from it, propagated stage by stage;
* ``finish32`` / ``deltas32``: eb_fe_finish / eb_fe_deltas in numpy float32, in frontend.cuh's order of operations.

Error model of ``chain`` (u = 2^-24; every bound is per element and first order).
  pre-emphasis  xp = x_r - p x_{r-1}: e_xp = 2u (|x_r| + |p x_{r-1}|) (the product and the difference, or one FMA).
  DFT           eb_gemm_f32 runs one FMA chain per output in k order from 0 (alpha = 1, no bias), so its n_fft roundings
                are each relative to the partial sum s_k they produce: e_spec = u sum_k |s_k| + |B| . e_xp.  This is
                the n_fft u sum |xp||B| bound with each term replaced by the partial sum it bounds (|s_k| <= sum_j<=k
                |xp_j B_j|); random signs make it ~sqrt(n_fft) times tighter.
  power         P = re^2 + im^2: e_P = 2|re| e_re + e_re^2 + 2|im| e_im + e_im^2 + 2u P.
  mel           M = P @ fb: e_M = u sum_k s_k + fb . e_P (P, fb >= 0: the partial sums are non-negative).
  log           y = logf(fl(M + off)), off = fp32(1e-20) (logfbank) or fp32(1e-6) (MFCC):
                e_y = e_M / (M + off - e_M) + u (the add) + ULP_LOGF 2^-23 |y| (logf).  Where e_M >= (M + off) / 2 the
                bound says nothing; those elements (and every output they feed) are counted and left unasserted.
  DCT           c = y @ D: e_c = u sum_k |s_k| + |D| . e_y.
  deltas        d = (2 (p2 - m2) + (p1 - m1)) / 10: e_d = (2 (e_p2 + e_m2) + e_p1 + e_m1) / 10 plus four roundings, each
                at most u (2 (|p2| + |m2|) + |p1| + |m1|) / 10; d2 likewise from d1 and e_d1.
  mask, stacking, the pad_to_divisible drop and the zero rows are exact.
The fp64 evaluation itself (~1e-16 relative) is negligible against these bars.

Table mode (``tables_err``).  Compared with an oracle built on exact tables (tests/features_batch_oracle.py) or with
the reference's own features, the module's fp32 tables are a second source of distance.  Their effect is propagated
through the same linearisation: the DFT basis is an fp64 formula rounded once (|dB| <= u |B|, a property of the code,
not measured, so that a wrong window is not absorbed), fp32(0.97) is within u of 0.97, fp32(off) within u off of off;
the filterbank and DCT tables' distances from the oracle's are measured per element on the host.
"""
import numpy as np
import torch

U24 = 2.0 ** -24
ULP_LOGF = 1.0           # CUDA logf: maximum error 1 ulp (CUDA C++ Programming Guide, single-precision functions)
LOG_OFF = {"logfbank": float(np.float32(1e-20)), "mfcc": float(np.float32(1e-6))}
EXACT_OFF = {"logfbank": 1e-20, "mfcc": 1e-6}


def fma_chain(a, b, chunk_bytes=1 << 30):
    """(a @ b, sum_k |s_k|) in fp64, s_k = sum_{j <= k} a[:, j] b[j, :]: the product and the sum of the partial sums an
    FMA chain in k order rounds."""
    K, N = b.shape
    rows = max(1, chunk_bytes // (8 * K * N))
    out, acc = [], []
    for i in range(0, a.shape[0], rows):
        s = (a[i:i + rows, :, None] * b[None]).cumsum(1)
        out.append(s[:, -1])
        acc.append(s.abs().sum(1))
    return torch.cat(out), torch.cat(acc)


def _frames(x, Lb, n_fft, hop, F, p, p_err):
    """Frames [F, n_fft] of one utterance's pre-emphasised, reflect-padded row (fp64) and their e_xp."""
    pad = n_fft // 2
    dev = x.device
    r = torch.arange(Lb + 2 * pad, device=dev) - pad
    r = torch.where(r < 0, -r, r)
    r = torch.where(r >= Lb, 2 * (Lb - 1) - r, r)
    xr = x[r]
    if p is None:
        xp, e = xr, torch.zeros_like(xr)
    else:
        prev = torch.where(r > 0, x[(r - 1).clamp_min(0)], torch.zeros_like(xr))
        xp = xr - p * prev
        e = 2 * U24 * (xr.abs() + (p * prev).abs()) + p_err * prev.abs()
    idx = torch.arange(F, device=dev)[:, None] * hop + torch.arange(n_fft, device=dev)[None, :]
    return xp[idx], e[idx]


def _log(M, e_M, off, off_err):
    y = torch.log(M + off)
    ok = e_M < 0.5 * (M + off)
    e_y = e_M / (M + off - e_M).clamp_min(1e-300) + U24 + ULP_LOGF * 2.0 ** -23 * y.abs() + off_err / (M + off)
    return y, e_y, ok


def _delta(s, e, ok):
    F = s.shape[0]
    i = torch.arange(F, device=s.device)
    p2, m2, p1, m1 = (torch.clamp(i + k, 0, F - 1) for k in (2, -2, 1, -1))
    d = (2 * (s[p2] - s[m2]) + (s[p1] - s[m1])) / 10
    mag = 2 * (s[p2].abs() + s[m2].abs()) + s[p1].abs() + s[m1].abs()
    e_d = (2 * (e[p2] + e[m2]) + e[p1] + e[m1]) / 10 + 4 * U24 * mag / 10
    return d, e_d, ok[p2] & ok[m2] & ok[p1] & ok[m1]


def _stack(v, F, Fs, n, T):
    """Frames [F, Cd] -> rows [T, n Cd]: frame t n + s at row t, block s; zero past Fs (Downsample)."""
    out = torch.zeros(T * n, v.shape[1], dtype=v.dtype, device=v.device)
    k = min(Fs, T * n)
    out[:k] = v[:k]
    return out.reshape(T, n * v.shape[1])


def chain(x, lens, ft, basis, fbT, n_fft, hop, n_stack, delta, ptd, preemph=None, dct=None, tables_err=None):
    """fp64 features of x [B, L] (fp32, any device) at per-utterance lens, from the given fp32 tables, as
    build_batch_transform's module computes them; returns (value, bar, ok) [B, T_max, W] (ok: the bar holds there)
    and the per-stage figures.  tables_err: None (the device's own tables) or dict(basis, fb, dct, preemph, offset) of
    the tables' distances from the exact ones (module docstring)."""
    dev = x.device
    x = x.double()
    B_ = basis.double().to(dev)
    fb = fbT.double().to(dev)
    D = dct.double().to(dev) if dct is not None else None
    te = tables_err or {}
    eB = te.get("basis", torch.zeros_like(B_)).to(dev)
    efb = te.get("fb", torch.zeros_like(fb)).to(dev)
    eD = te.get("dct", torch.zeros_like(D)).to(dev) if D is not None else None
    p = float(np.float32(preemph)) if preemph is not None else None
    p_err = te.get("preemph", 0.0)
    off_err = te.get("offset", 0.0)
    nb = n_fft // 2 + 1
    vals, bars, oks, Ts = [], [], [], []
    for b, Lb in enumerate(int(v) for v in lens):
        F = 1 + Lb // hop
        Fs = F if ptd else F - F % n_stack
        T = -(-F // n_stack) if ptd else F // n_stack
        fr, efr = _frames(x[b], Lb, n_fft, hop, F, p, p_err)
        spec, S1 = fma_chain(fr, B_)
        e_spec = U24 * S1 + efr @ B_.abs() + fr.abs() @ eB
        re, im, e_re, e_im = spec[:, :nb], spec[:, nb:], e_spec[:, :nb], e_spec[:, nb:]
        P = re * re + im * im
        e_P = 2 * re.abs() * e_re + e_re ** 2 + 2 * im.abs() * e_im + e_im ** 2 + 2 * U24 * P
        M, S2 = fma_chain(P, fb)
        e_M = U24 * S2 + e_P @ fb + P @ efb
        if ft == "mfcc":
            y, e_y, ok = _log(M, e_M, LOG_OFF[ft], off_err * LOG_OFF[ft])
            s, S3 = fma_chain(y, D)
            e_s = U24 * S3 + e_y @ D.abs() + y.abs() @ eD
            ok = ok.all(1, keepdim=True).expand_as(s)
        elif ft == "logfbank":
            s, e_s, ok = _log(M, e_M, LOG_OFF[ft], off_err * LOG_OFF[ft])
            seq = -(-Lb // hop)
            s, e_s, ok = s.clone(), e_s.clone(), ok.clone()
            s[seq:], e_s[seq:], ok[seq:] = 0, 0, True
        else:
            s, e_s, ok = M, e_M, torch.ones_like(M, dtype=torch.bool)
        if delta:
            d1, e1, ok1 = _delta(s, e_s, ok)
            d2, e2, ok2 = _delta(d1, e1, ok1)
            s, e_s, ok = torch.cat([s, d1, d2], 1), torch.cat([e_s, e1, e2], 1), torch.cat([ok, ok1, ok2], 1)
        vals.append(_stack(s, F, Fs, n_stack, T))
        bars.append(_stack(e_s, F, Fs, n_stack, T))
        oks.append(_stack((~ok).double(), F, Fs, n_stack, T) < 0.5)      # the zero slots past Fs are exact
        Ts.append(T)
    W = vals[0].shape[1]
    Tm = max(Ts)
    out = [torch.zeros(len(lens), Tm, W, dtype=torch.float64, device=dev) for _ in range(3)]
    for b in range(len(lens)):
        out[0][b, :Ts[b]], out[1][b, :Ts[b]] = vals[b], bars[b]
        out[2][b] = True
        out[2][b, :Ts[b]] = oks[b]
    return out[0], out[1], out[2] > 0.5


def module_tables(module):
    """(basis, fbT, dct, preemph) a build_batch_transform test module's features hand to ops.fe_batch."""
    f = module.features
    name = type(f).__name__
    if name == "FilterbankFeatures":
        return f.dft_basis, f.fb_t, None, f.preemph
    mel = f.MelSpectrogram if name == "MFCC" else f
    return mel.spectrogram.dft_basis, mel.mel_scale.fb, (f.dct_mat if name == "MFCC" else None), None


def tables_err(ft, basis, fbT, dct, n_fft, n_ch, preemph):
    """The fp32 tables' distances from the exact ones the oracle uses (module docstring, table mode)."""
    from tests import features_batch_oracle as O
    if ft == "logfbank":
        fb_exact = O.F.slaney_mel_filterbank(O.SR, n_fft, n_ch).astype(np.float64).T
    else:
        fb_exact = O.htk_mel_filterbank(n_fft, O.MFCC_N_MELS if ft == "mfcc" else n_ch)
    te = dict(basis=U24 * basis.double().cpu().abs(),
              fb=(fbT.double().cpu() - torch.from_numpy(fb_exact)).abs(),
              offset=U24)
    if dct is not None:
        te["dct"] = (dct.double().cpu() - torch.from_numpy(O.create_dct(dct.shape[1], dct.shape[0]))).abs()
    if preemph is not None:
        te["preemph"] = abs(float(np.float32(preemph)) - preemph)
    return te


def report(name, got, ref, bar, ok=None, extra=None):
    """Asserts |got - ref| <= bar (+ extra) wherever ok; prints the worst err/bar, where it occurs and how many elements
    had no bound; returns the worst ratio."""
    got = torch.as_tensor(np.asarray(got) if not torch.is_tensor(got) else got).double().cpu()
    ref = torch.as_tensor(np.asarray(ref) if not torch.is_tensor(ref) else ref).double().cpu()
    bar = bar.double().cpu() + 2.0 ** -126
    if extra is not None:
        bar = bar + torch.as_tensor(np.asarray(extra) if not torch.is_tensor(extra) else extra).double().cpu()
    ok = torch.ones_like(bar, dtype=torch.bool) if ok is None else ok.cpu()
    assert got.shape == ref.shape == bar.shape, (name, got.shape, ref.shape, bar.shape)
    assert torch.isfinite(got).all(), name + ": non-finite output"
    err = (got - ref).abs()
    r = torch.where(ok & (err > 0), err / bar, torch.zeros_like(err))
    k = int(torch.argmax(r.reshape(-1)))
    idx = tuple(int(i) for i in np.unravel_index(k, tuple(r.shape)))
    ratio = float(r.reshape(-1)[k])
    print("  %-58s worst err/bar %.3g at %s (err %.3g, bar %.3g); %d unbounded" %
          (name, ratio, idx, float(err[idx]), float(bar[idx]), int((~ok).sum())))
    assert ratio <= 1.0, "%s: err/bar %.3g at %s, got %r, want %r" % (name, ratio, idx, float(got[idx]), float(ref[idx]))
    return ratio


# ---- float32 restatement of eb_fe_finish / eb_fe_deltas (frontend.cuh) ----------------------------------------------
def deltas32(s):
    """fe_delta1 over every frame of s [F, C] float32: (2 (p2 - m2) + (p1 - m1)) / 10 with replicate edges at F - 1.
    2 x is exact, so an FMA contraction of 2 (p2 - m2) + (p1 - m1) rounds as the separate add does; the division is
    IEEE (the library is built without --use_fast_math)."""
    s = np.asarray(s, np.float32)
    F = s.shape[0]
    i = np.arange(F)
    g = lambda k: s[np.clip(i + k, 0, F - 1)]
    return (np.float32(2) * (g(2) - g(-2)) + (g(1) - g(-1))) / np.float32(10)


def finish32(statics, F, Fs, n_stack, T, delta):
    """One utterance of eb_fe_finish from its static values [F, C] float32 (already logged and masked, as fe_static
    returns them): [static | d1 | d2] per frame, stacked n_stack frames per row, zero from frame Fs, T rows."""
    s = np.asarray(statics, np.float32)[:F]
    if delta:
        d1 = deltas32(s)
        s = np.concatenate([s, d1, deltas32(d1)], axis=1)
    out = np.zeros((T * n_stack, s.shape[1]), np.float32)
    k = min(Fs, T * n_stack)
    out[:k] = s[:k]
    return out.reshape(T, n_stack * s.shape[1])
