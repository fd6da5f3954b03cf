"""Teacher-forced fp64 parity of the recurrent LSTM kernels, per step and per element.

    forward   eb_lstm_c4_fwd (wgmma, clusters of 4), eb_lstm_tc_fwd (mma.sync), eb_lstm_seq_fwd (fp32)
    BPTT      eb_lstm_tc_bwd, eb_lstm_tc_bwd_chunks (clusters of 8 / 4 / 2), eb_lstm_c4_bwd (CTA-private bf16 saves,
              clusters of 8 / 4), eb_lstm_c4_bwd_chunks (K split over clusters of 16), eb_lstm_seq_bwd (fp32)

Every rounding on the recurrent path is visible from outside the kernel: the bf16 h_{t-1} a forward step multiplies is
what the kernel writes to hprev16[:, t] (c4) or y16[:, t-1] (tc; the fp32 kernel exchanges y itself), the cell state
stays fp32 and is saved, and the bf16 dG_t a BPTT step exchanges is what it writes to dg16.  The fp64 references below
therefore compute step t from the kernel's own inputs to step t (teacher forcing): errors do not compound over t, the
bar of step t covers only what step t does, and a failure names one (batch row, step, gate, unit).  Only the dc carry
of BPTT is recursed in fp64 (elementwise, contracting with f <= 1), with its bar recursed alongside.

Error model (first order, per element; the absolute terms scale with the operand magnitudes):
  pre-activation  n_add u_acc sum_k |h_k||w_k| + 2^-24 (|s| + |xg|): n_add is the longest fp32 summation chain of the
                  kernel (`_n_add`), u_acc = 2^-23 per add for tensor-core accumulation (the alignment of the addends
                  may truncate: one ulp, not half) and 2^-24 for the fp32 FMA chains of lstm.cu;
  gates           sigma' |dpre| + EPS_ACT, tanh' |dpre| + EPS_ACT (EPS_ACT: absolute error of the gate nonlinearities,
                  measured by test_gate_nonlinearity_error);
  c, h            propagated through c = f c' + i g and h = o tanh(c), plus the fp32 roundings of each operation;
  BPTT            dh = dy + dg16_{t+1} W with the bar of the pre-activation; 1 - tanh(c)^2 carries the ABSOLUTE error
                  2 |tanh c| EPS_ACT (it loses all relative precision for |c| > ~4); then through the four gate-gradient
                  formulas.  dg16 may differ from the fp64 value by the error bar plus half a bf16 ulp (the fp32 value
                  may sit on the other side of a rounding boundary), and the share of elements whose bits differ from
                  bf16_rn(dG_ref) must stay below FRAC_DIFF.

The worst-case summation bound is loose (random signs give ~sqrt(n_add) instead of n_add: the dh0 checks measure 0.02 of
it at most); every test prints the worst err/bar ratio next to where it occurs (pytest -s), and DESIGN.md section 2
records the measured figures.  The file runs in about 10 s on an H100."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
U24 = 2.0 ** -24          # fp32 unit roundoff, round to nearest
UTC = 2.0 ** -23          # per add of a tensor-core fp32 accumulation
EPS_FAST = 3e-7           # |fsig - sigmoid|, |ftanh - tanh| (ex2.approx + rcp.approx; lstm_c4.cu, lstm_tc.cu): 1.1e-7 / 2.1e-7 measured
EPS_LIBM = 1.5e-7         # expf / tanhf of the fp32 kernels (lstm.cu): 8.9e-8 / 6.7e-8 measured
FRAC_DIFF = 0.01          # share of dg16 elements != bf16_rn(dG_ref); 0.0016 measured at most
TINY = 2.0 ** -120         # absolute floor of every bar: fp32 intermediates underflow (and flush) below ~2^-126
SAT = [20.0, 44.0, 44.5, 45.0, 87.0, 87.5, 88.0, 88.5, 89.0, 89.5, 90.0, 1e4]   # |xg| planted by the saturation tests


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---- error bookkeeping ------------------------------------------------------------------------------------------------
def _bf16_ulp(x):
    """Spacing of bf16 numbers (8 significant bits) at |x| >= 2^-126, fp64."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


def worst(err, bar):
    """(largest err / bar, index of that element, its err, its bar); err == 0 counts as 0 whatever the bar."""
    r = torch.where(err == 0, torch.zeros_like(err), err / bar.clamp_min(1e-300))
    k = int(torch.argmax(r.reshape(-1)))
    idx = tuple(int(i) for i in np.unravel_index(k, tuple(r.shape)))
    return float(r.reshape(-1)[k]), idx, float(err.reshape(-1)[k]), float(bar.reshape(-1)[k])


def _report(name, items):
    """items: (label, kernel value, fp64 value, bar) with matching shapes.  Prints every ratio, then asserts them all."""
    bad = []
    for label, got, ref, bar in items:
        got = got.double()
        assert torch.isfinite(got).all(), "%s %s: non-finite output" % (name, label)
        bar = bar + TINY
        ratio, idx, e, b = worst((got - ref).abs(), bar)
        print("  %-34s %-6s worst err/bar %.3g at %s (err %.3g, bar %.3g)" % (name, label, ratio, idx, e, b))
        if ratio > 1.0:
            bad.append("%s: err/bar %.3g at %s, kernel %r, fp64 %r" % (label, ratio, idx, float(got[idx]), float(ref[idx])))
    assert not bad, name + ": " + "; ".join(bad)


# ---- fp64 references --------------------------------------------------------------------------------------------------
def fwd_ref(xg, w, hin, cin, n_add, u_acc, eps, dpre_in=0.0, dcin=0.0):
    """Teacher-forced forward, every step at once.  xg [B,T,4H], w [4H,H] (the values the kernel multiplies), hin [B,T,H]
    the h_{t-1} operand of each step as the kernel used it (bf16(h0) / hprev16 / y16 / y), cin [B,T,H] the c_{t-1} the
    kernel carried (c0, then its fp32 cell save).  dpre_in [B,T,4H] and dcin [B,T,H] are bars the pre-activation and
    c_{t-1} already carry (0 when every input is the kernel's own).  Returns {name: (value, bar)} for gates [B,T,4,H],
    c and y [B,T,H]."""
    xg, w, hin, cin = (a.to(f64) for a in (xg, w, hin, cin))
    B, T, H4 = xg.shape
    H = H4 // 4
    s = hin @ w.t()
    pre = (xg + s).view(B, T, 4, H)
    dpre = (n_add * u_acc * (hin.abs() @ w.abs().t()) + U24 * (s.abs() + xg.abs()) + dpre_in).view(B, T, 4, H)
    sg = torch.sigmoid(pre)
    tg = torch.tanh(pre)
    is_g = (torch.arange(4, device=pre.device) == 2).view(1, 1, 4, 1)
    act = torch.where(is_g, tg, sg)
    slope = torch.where(is_g, 1 - tg * tg, sg * (1 - sg))
    dact = slope * dpre + eps + U24 * act.abs()
    i, f, g, o = act.unbind(2)
    di, df, dg, do = dact.unbind(2)
    c = f * cin + i * g
    dc = df * cin.abs() + f * dcin + di * g.abs() + i * dg + 2 * U24 * ((f * cin).abs() + (i * g).abs())
    tc = torch.tanh(c)
    y = o * tc
    dy = do * tc.abs() + o * ((1 - tc * tc) * dc + eps) + 2 * U24 * y.abs()
    return dict(gates=(act, dact), c=(c, dc), y=(y, dy), pre=pre)


def bwd_ref(dy, gates, cseq, c0, w, dgq, dhT, dcT, n_add, u_acc, eps):
    """Teacher-forced BPTT.  dy [B,T,H]; gates [B,T,4H] and cseq [B,T,H] as the kernel read them (eb_lstm_c4_bwd reads
    bf16 gates: pass those values); c0 / dhT / dcT [B,H] or None; w [4H,H]; dgq [B,T,4H] the dG the kernel exchanged
    (its dg16, or its fp32 dgates).  dh_t = dy_t + dgq_{t+1} W (dhT at T-1) is the kernel's own input to step t; the dc
    carry is recursed in fp64 with its bar.  Returns {name: (value, bar)} for dG [B,T,4,H], dh0 and dc0 [B,H]."""
    dy, gates, cseq, w, dgq = (a.to(f64) for a in (dy, gates, cseq, w, dgq))
    B, T, H = dy.shape
    i, f, g, o = gates.view(B, T, 4, H).unbind(2)
    z = torch.zeros(B, H, dtype=f64, device=dy.device)
    c0 = z if c0 is None else c0.to(f64)
    cprev = torch.cat([c0[:, None], cseq[:, :-1]], 1)
    dh, ddh = dy.clone(), U24 * dy.abs()
    if T > 1:
        r = dgq[:, 1:] @ w
        dh[:, :-1] += r
        ddh[:, :-1] += n_add * u_acc * (dgq[:, 1:].abs() @ w.abs()) + U24 * r.abs()
    if dhT is not None:
        dh[:, -1] += dhT.to(f64)
        ddh[:, -1] += U24 * dhT.to(f64).abs()
    tc = torch.tanh(cseq)
    k = 1 - tc * tc
    dk = 2 * tc.abs() * eps + U24 * (tc * tc + k)          # absolute: 1 - tc*tc cancels for |c| > ~4
    e = dh * o * k
    de = ddh * o * k + (dh * o).abs() * dk + 2 * U24 * e.abs()
    dct, ddct = torch.empty_like(dy), torch.empty_like(dy)
    dc = z if dcT is None else dcT.to(f64)
    ddc = torch.zeros_like(z)
    for t in range(T - 1, -1, -1):
        x = dc + e[:, t]
        dct[:, t] = x
        ddct[:, t] = ddc + de[:, t] + U24 * x.abs()
        dc = x * f[:, t]
        ddc = ddct[:, t] * f[:, t] + U24 * dc.abs()
    ai = dct * g * i * (1 - i)
    af = dct * cprev * f * (1 - f)
    ag = dct * i * (1 - g * g)
    ao = dh * tc * o * (1 - o)
    bi = ddct * (g * i * (1 - i)).abs() + 4 * U24 * ai.abs()
    bf = ddct * (cprev * f * (1 - f)).abs() + 4 * U24 * af.abs()
    bg = ddct * (i * (1 - g * g)).abs() + 2 * U24 * (dct * i).abs() * g * g + 4 * U24 * ag.abs()
    bo = ddh * (tc * o * (1 - o)).abs() + (dh * o * (1 - o)).abs() * eps + 4 * U24 * ao.abs()
    dG = torch.stack([ai, af, ag, ao], 2)
    dGb = torch.stack([bi, bf, bg, bo], 2)
    dh0 = dgq[:, 0] @ w
    dh0b = n_add * u_acc * (dgq[:, 0].abs() @ w.abs())
    return dict(dG=(dG, dGb), dh0=(dh0, dh0b), dc0=(dc, ddc))


def _n_add(kernel, H, cs=0):
    """Longest fp32 summation chain of one pre-activation / one dh element."""
    if kernel == "c4_fwd":        # H/4 products per CTA (wgmma), then own + 3 received partial tiles, + xg
        return H // 4 + 4 + 1
    if kernel == "tc_fwd":        # each of 8 warps: ceil(H/128) k16 steps, then the 8 warp partials, + xg
        return 16 * -(-H // 128) + 8 + 1
    if kernel == "tc_bwd":        # 4H/CS contraction rows per CTA over 8 warps, 8 warp partials, CS CTA partials
        cs = cs or 4              # the software-reduction fallback runs the CS = 4 decomposition
        return 16 * -(-(4 * H // cs) // 128) + 8 + cs
    if kernel == "c4_bwd":        # 4H/CS per CTA (wgmma), then CS partials
        return 4 * H // cs + cs
    if kernel == "seq":           # fp32 FMA chains of lstm.cu: at most the whole contraction, + the K-split partials
        return 4 * H + 8
    raise ValueError(kernel)


def _check_fwd(name, r, w, xg, kernel, eps, u_acc):
    B, T, H = r["y"].shape
    ref = fwd_ref(xg, w, r["hin"], r["cin"], _n_add(kernel, H), u_acc, eps)
    _report(name, [("gates", r["gates"].view(B, T, 4, H), *ref["gates"]),
                   ("c", r["cseq"], *ref["c"]),
                   ("y", r["y"], *ref["y"])])
    return ref


def _check_bwd(name, ref, dg, dh0, dc0, bf16_out=True):
    """dg [B,T,4H] (bf16 dg16, or fp32 dgates), dh0 / dc0 [B,H] fp32 against bwd_ref's output."""
    val, bar = ref["dG"]
    B, T, _, H = val.shape
    dg = dg.view(B, T, 4, H)
    if bf16_out:
        # rounding is monotone: the bf16 value of anything within the bar lies in [bf16_rn(ref - bar), bf16_rn(ref + bar)]
        lo, hi = (val - bar).to(f32).to(bf16).double(), (val + bar).to(f32).to(bf16).double()
        d = dg.double()
        outside = int(((d < lo) | (d > hi)).sum())
        frac = float((dg != val.to(f32).to(bf16)).double().mean())
        print("  %-34s dg16 bits != bf16_rn(dG_ref): %.4f of the elements (bar %.3g), %d outside the rounded bar"
              % (name, frac, FRAC_DIFF, outside))
        bar = bar + 0.5 * _bf16_ulp(val.abs() + bar)
    _report(name, [("dG", dg, val, bar), ("dh0", dh0, *ref["dh0"]), ("dc0", dc0, *ref["dc0"])])
    if bf16_out:
        assert outside == 0, "%s: %d dg16 elements are not a rounding of a value within the bar" % (name, outside)
        assert frac <= FRAC_DIFF, "%s: %.4f of dg16 differs from bf16_rn(dG_ref)" % (name, frac)


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _plant(x, gen, frac, values):
    """Overwrite a random `frac` of x with entries of `values`, random sign."""
    m = torch.rand(x.shape, device=DEV, generator=gen) < frac
    v = torch.tensor(values, device=DEV, dtype=x.dtype)
    pick = v[torch.randint(0, len(values), x.shape, device=DEV, generator=gen)]
    sign = torch.where(torch.rand(x.shape, device=DEV, generator=gen) < 0.5, -1.0, 1.0).to(x.dtype)
    return torch.where(m, pick * sign, x)


def fwd_inputs(B, T, H, seed, init, sat=False):
    """w [4H,H] fp32 ~ U(-1/sqrt(H), 1/sqrt(H)), xg ~ N(0, 1), h0 / c0 ~ N(0, 1/4) or None.  sat: 10 % of xg at the
    values of SAT and c0 up to +-50."""
    gen = _gen(seed)
    w = (torch.rand(4 * H, H, device=DEV, generator=gen) * 2 - 1) / math.sqrt(H)
    xg = torch.randn(B, T, 4 * H, device=DEV, generator=gen)
    h0 = c0 = None
    if init:
        h0 = torch.randn(B, H, device=DEV, generator=gen) * 0.5
        c0 = torch.randn(B, H, device=DEV, generator=gen) * 0.5
    if sat:
        xg = _plant(xg, gen, 0.1, SAT)
        c0 = (torch.rand(B, H, device=DEV, generator=gen) * 2 - 1) * 50
        h0 = torch.randn(B, H, device=DEV, generator=gen) * 0.5
    return w, xg, h0, c0


def synthetic_saves(B, T, H, seed, sat=False):
    """gates in (0, 1) (g in (-1, 1)), cells ~ N(0, 1), dy ~ N(0, 1); sat: exact 0 / 1 / -1 gates and |c| up to 50."""
    gen = _gen(seed)
    gates = torch.sigmoid(torch.randn(B, T, 4 * H, device=DEV, generator=gen) * 2)
    gates[..., 2 * H:3 * H] = torch.tanh(torch.randn(B, T, H, device=DEV, generator=gen) * 2)
    cseq = torch.randn(B, T, H, device=DEV, generator=gen)
    if sat:
        sig = _plant(gates, gen, 0.1, [0.0, 1.0]).abs()
        gates = torch.where(torch.rand(gates.shape, device=DEV, generator=gen) < 0.5, sig, gates)
        gates[..., 2 * H:3 * H] = _plant(gates[..., 2 * H:3 * H], gen, 0.1, [1.0])
        cseq = _plant(cseq, gen, 0.2, [5.0, 9.0, 20.0, 50.0])
    return gates.contiguous(), cseq


def bwd_grads(B, T, H, seed, init):
    gen = _gen(seed)
    dy = torch.randn(B, T, H, device=DEV, generator=gen)
    if not init:
        return dy, None, None, None
    return (dy, torch.randn(B, H, device=DEV, generator=gen) * 0.5, torch.randn(B, H, device=DEV, generator=gen),
            torch.randn(B, H, device=DEV, generator=gen))


def _shift(first, seq):
    """[first, seq[:, 0], ..., seq[:, T-2]] along t."""
    return torch.cat([first[:, None].to(seq.dtype), seq[:, :-1]], 1)


def _zeros_bh(B, H, dtype=f32):
    return torch.zeros(B, H, dtype=dtype, device=DEV)


# ---- kernel runners ---------------------------------------------------------------------------------------------------
def _c4_fwd_ok(H):
    return _lib().eb_lstm_c4_max_clusters(H, 0) >= H // 32


def c4_decode_gates(gsave, B, T, H):
    """CTA-private gate save -> [B,T,4H] bf16.  Per 32-row batch tile: [T][H/8 CTAs][128 threads] records of 8 bf16
    (i0 i1 f0 f1 g0 g1 o0 o1); thread tid is batch row tid >> 2 and units 8 cta + 2 (tid & 3) + {0, 1}."""
    nt = -(-B // 32)
    g = gsave.view(bf16).view(nt, T, H // 8, 32, 4, 4, 2)           # tile, t, cta, row, up, gate, pair
    return g.permute(0, 3, 1, 5, 2, 4, 6).reshape(nt * 32, T, 4 * H)[:B]


def c4_decode_cells(csave, B, T, H):
    """CTA-private cell save (float2 per thread, same record order) -> [B,T,H] fp32."""
    nt = -(-B // 32)
    c = csave.view(f32).view(nt, T, H // 8, 32, 4, 2)                # tile, t, cta, row, up, pair
    return c.permute(0, 3, 1, 2, 4, 5).reshape(nt * 32, T, H)[:B]


def run_c4_fwd(w16, xg, h0, c0):
    """eb_lstm_c4_fwd asked for BOTH save layouts in one call."""
    from edgedict_b200 import ops
    B, T, H4 = xg.shape
    H = H4 // 4
    y = torch.empty(B, T, H, device=DEV)
    hp = torch.empty(B, T, H, dtype=bf16, device=DEV)
    hT, cT = torch.empty(B, H, device=DEV), torch.empty(B, H, device=DEV)
    gsave, csave = ops.lstm_c4_save_buffers(B, T, H, DEV)
    gstd, cstd = torch.empty(B, T, H4, device=DEV), torch.empty(B, T, H, device=DEV)
    scratch = torch.zeros(_lib().eb_lstm_c4_scratch_bytes(B, H), dtype=torch.uint8, device=DEV)
    rc = _lib().eb_lstm_c4_fwd(_p(xg), _p(w16), _p(h0), _p(c0), _p(y), _p(hp), _p(hT), _p(cT), _p(gsave), _p(csave),
                               _p(gstd), _p(cstd), _p(scratch), B, T, H, _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    c0z = c0 if c0 is not None else _zeros_bh(B, H)
    return dict(y=y, hprev16=hp, hT=hT, cT=cT, gsave=gsave, csave=csave, gates=gstd, cseq=cstd,
                hin=hp, cin=_shift(c0z, cstd))


def run_tc_fwd(w16, xg, h0, c0):
    from edgedict_b200 import ops
    B, T, H4 = xg.shape
    H = H4 // 4
    y, y16, hT, cT, gates, cseq = ops.lstm_tc_fwd(xg, w16, h0, c0, True)
    torch.cuda.synchronize()
    h0z = h0 if h0 is not None else _zeros_bh(B, H)
    c0z = c0 if c0 is not None else _zeros_bh(B, H)
    return dict(y=y, y16=y16, hT=hT, cT=cT, gates=gates, cseq=cseq,
                hin=_shift(h0z.to(bf16), y16), cin=_shift(c0z, cseq))


def run_seq_fwd(w, xg, h0, c0):
    from edgedict_b200 import ops
    B, T, H4 = xg.shape
    H = H4 // 4
    y, hT, cT, gates, cseq = ops.lstm_seq_fwd(xg, w, h0, c0, True)
    torch.cuda.synchronize()
    h0z = h0 if h0 is not None else _zeros_bh(B, H)
    c0z = c0 if c0 is not None else _zeros_bh(B, H)
    return dict(y=y, hT=hT, cT=cT, gates=gates, cseq=cseq, hin=_shift(h0z, y), cin=_shift(c0z, cseq))


def tc_cluster_size(H):
    """The cluster size eb_lstm_tc_bwd picks (lstm_tc.cu pick_cs): the largest of 8 / 4 / 2 whose clusters all fit."""
    for cs in (8, 4, 2):
        if _lib().eb_lstm_tc_max_clusters(H, cs) >= H // (8 * cs):
            return cs
    return 0


def _chunk_call(entry, dy, gates, cseq, c0, w16, dhT, dcT, lens, scratch_bytes):
    """eb_lstm_{tc,c4}_bwd_chunks over the chunk-major scatter of [B,T,...] inputs; returns dg16 [B,T,4H], dh0, dc0."""
    import ctypes
    from edgedict_b200.functional import _Chunks
    B, T, H = dy.shape
    ck = _Chunks(B, lens)
    dg = torch.full((ck.rows + 1, 4 * H), 7.0, dtype=bf16, device=DEV)      # one guard row past the buffer
    dh0, dc0 = torch.empty(B, H, device=DEV), torch.empty(B, H, device=DEV)
    arr = (ctypes.c_int * len(lens))(*lens)
    scratch = torch.zeros(scratch_bytes(B, H), dtype=torch.uint8, device=DEV)
    args = (ck.scatter(dy), ck.scatter(gates), ck.scatter(cseq), c0, w16.t().contiguous(), dhT, dcT)   # alive during the call
    rc = entry(*map(_p, args), _p(dg), _p(dh0), _p(dc0), _p(scratch), B, arr, len(lens), H, _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert (dg[ck.rows] == 7.0).all(), "write past the dg16 buffer"
    return ck.gather(dg[:ck.rows]), dh0, dc0


# ---- forward ----------------------------------------------------------------------------------------------------------
FWD_SHAPES = [(1, 1, True), (1, 37, False), (5, 1, False), (5, 37, True), (32, 2, False), (32, 37, True),
              (40, 37, False), (40, 2, True)]


def _fwd_bitwise_common(name, r):
    assert torch.equal(r["hT"], r["y"][:, -1]), name + ": hT != y[:, -1]"
    assert torch.equal(r["cT"], r["cseq"][:, -1]), name + ": cT != cseq[:, -1]"


def _c4_fwd_case(B, T, H, init, seed, sat=False):
    if not _c4_fwd_ok(H):
        pytest.skip("clusters of 4 of the lstm_c4 forward kernel are not co-resident on this GPU")
    w, xg, h0, c0 = fwd_inputs(B, T, H, seed, init, sat)
    w16 = w.to(bf16)
    r = run_c4_fwd(w16, xg, h0, c0)
    name = "c4_fwd B%d T%d H%d %s" % (B, T, H, "h0c0" if h0 is not None else "zero-init")
    # bitwise: the exchanged h is the saved hprev16, the CTA-private saves hold the standard-layout values
    h0b = (h0 if h0 is not None else _zeros_bh(B, H)).to(bf16)
    assert torch.equal(r["hprev16"][:, 0], h0b), name + ": hprev16[:, 0] != bf16(h0)"
    assert torch.equal(r["hprev16"][:, 1:], r["y"][:, :-1].to(bf16)), name + ": hprev16[:, 1:] != bf16_rn(y[:, :-1])"
    _fwd_bitwise_common(name, r)
    assert torch.equal(c4_decode_gates(r["gsave"], B, T, H), r["gates"].to(bf16)), name + ": gsave != bf16_rn(gates)"
    assert torch.equal(c4_decode_cells(r["csave"], B, T, H), r["cseq"]), name + ": csave != cseq"
    ref = _check_fwd(name, r, w16, xg, "c4_fwd", EPS_FAST, UTC)
    return r, ref, w16, xg, h0, c0


@pytest.mark.parametrize("H", [256, 512, 768, 1024])
@pytest.mark.parametrize("B,T,init", FWD_SHAPES)
def test_c4_fwd_teacher_forced(B, T, init, H):
    """eb_lstm_c4_fwd, both save layouts requested in one call.  Bitwise: hprev16[:, 0] = bf16(h0) (0 without h0),
    hprev16[:, 1:] = bf16_rn(y[:, :-1]), hT = y[:, -1], cT = cseq[:, -1], and the CTA-private saves decode to
    bf16_rn(gates_std) and cseq_std.  Per element against fwd_ref with n_add = H/4 + 4 + 1 (wgmma over the K slice of
    the CTA, the four partials of the cluster, xg) and u_acc = 2^-23."""
    _c4_fwd_case(B, T, H, init, 1000 * H + 10 * B + T)


@pytest.mark.parametrize("H", [64, 320, 512, 1024])
@pytest.mark.parametrize("B,T,init", FWD_SHAPES)
def test_tc_fwd_teacher_forced(B, T, init, H):
    """eb_lstm_tc_fwd.  Bitwise: y16 = bf16_rn(y) (y16[:, t-1] is the h_{t-1} operand of step t), hT = y[:, -1],
    cT = cseq[:, -1].  Per element against fwd_ref with n_add = 16 ceil(H/128) + 8 + 1 (each warp's k16 steps, the 8
    warp partials, xg) and u_acc = 2^-23."""
    w, xg, h0, c0 = fwd_inputs(B, T, H, 2000 * H + 10 * B + T, init)
    w16 = w.to(bf16)
    r = run_tc_fwd(w16, xg, h0, c0)
    name = "tc_fwd B%d T%d H%d %s" % (B, T, H, "h0c0" if init else "zero-init")
    assert torch.equal(r["y16"], r["y"].to(bf16)), name + ": y16 != bf16_rn(y)"
    _fwd_bitwise_common(name, r)
    _check_fwd(name, r, w16, xg, "tc_fwd", EPS_FAST, UTC)


@pytest.mark.parametrize("H", [8, 24, 320, 1024])
@pytest.mark.parametrize("B,T,init", FWD_SHAPES)
def test_seq_fwd_teacher_forced(B, T, init, H):
    """eb_lstm_seq_fwd (fp32 mode).  The exchanged h is y itself (lstm.cu writes hn to y and to the exchange buffer), so
    the harness runs with identity rounding: hin = [h0, y[:, :-1]], fp32 weights, fp32 FMA chains (u = 2^-24,
    n_add = 4H + 8 as an upper bound of the K-split chains), expf / tanhf (EPS_LIBM)."""
    w, xg, h0, c0 = fwd_inputs(B, T, H, 3000 * H + 10 * B + T, init)
    r = run_seq_fwd(w, xg, h0, c0)
    name = "seq_fwd B%d T%d H%d %s" % (B, T, H, "h0c0" if init else "zero-init")
    _fwd_bitwise_common(name, r)
    _check_fwd(name, r, w, xg, "seq", EPS_LIBM, U24)


@pytest.mark.parametrize("kernel,B,T,H", [("c4", 32, 512, 1024), ("tc", 40, 300, 512), ("seq", 5, 400, 320)])
def test_fwd_long_sequence(kernel, B, T, H):
    """One long sequence per forward kernel: teacher forcing keeps the bar of step 500 the bar of step 0."""
    if kernel == "c4":
        _c4_fwd_case(B, T, H, True, 7)
        return
    w, xg, h0, c0 = fwd_inputs(B, T, H, 8, True)
    if kernel == "tc":
        w16 = w.to(bf16)
        r = run_tc_fwd(w16, xg, h0, c0)
        assert torch.equal(r["y16"], r["y"].to(bf16))
        _check_fwd("tc_fwd long T%d H%d" % (T, H), r, w16, xg, "tc_fwd", EPS_FAST, UTC)
    else:
        r = run_seq_fwd(w, xg, h0, c0)
        _check_fwd("seq_fwd long T%d H%d" % (T, H), r, w, xg, "seq", EPS_LIBM, U24)


def _limits_exact(name, gates, pre, ftz):
    """Where the fp64 gate rounds to its limit in fp32 with a margin (within 2^-27 of 1 or -1; below 2^-127 for 0 when
    the kernel flushes denormals to zero, below 2^-151 when it keeps them), the kernel returns the limit exactly.  The
    margin keeps values at a rounding threshold, where a 1-ulp accurate function may land either side, out of the test.
    pre [B,T,4,H] fp64."""
    B, T, _, H = pre.shape
    got = gates.view(B, T, 4, H).double()
    sg, tg = torch.sigmoid(pre), torch.tanh(pre)
    is_g = (torch.arange(4, device=DEV) == 2).view(1, 1, 4, 1)
    ref = torch.where(is_g, tg, sg)
    lim = torch.where(is_g, torch.sign(pre), (pre > 0).double())
    near = torch.where(lim == 0, ref.abs() < 2.0 ** (-127 if ftz else -151), (ref - lim).abs() < 2.0 ** -27)
    n = int(near.sum())
    bad = int((near & (got != lim)).sum())
    print("  %-34s %d gates at a saturation limit, %d not exact" % (name, n, bad))
    assert n > 0 and bad == 0, name


@pytest.mark.parametrize("kernel,H", [("c4", 256), ("tc", 320), ("seq", 24)])
def test_gate_nonlinearity_error(kernel, H):
    """EPS_ACT, measured: W_hh = 0 and h0 = 0 make every pre-activation exactly xg, so the saved gates are the kernel's
    sigmoid / tanh of known fp32 arguments.  xg sweeps [-30, 30] densely plus the saturation values of SAT (|x| = 20,
    the band 87 ... 90 where fast_exp leaves the range of __fdividef, which then returns 0, and 1e4).  Every gate must
    be within EPS_ACT of the fp64 function, finite, and exactly at its limit where the fp64 value rounds to it in fp32
    (with the margin of _limits_exact).  Measured on an H100: fsig 1.1e-7, ftanh 2.1e-7 (the cancellation in
    1 - 2 / (e^2x + 1) near 0), expf-based sigmoid 8.9e-8, tanhf 6.7e-8."""
    B, T = 32, 3
    n = B * T * 4 * H
    xg = torch.linspace(-30, 30, n, device=DEV).view(B, T, 4 * H)
    xg = _plant(xg, _gen(11), 0.05, SAT).contiguous()
    w = torch.zeros(4 * H, H, device=DEV)
    h0 = torch.zeros(B, H, device=DEV)
    c0 = (torch.rand(B, H, device=DEV, generator=_gen(12)) * 2 - 1) * 50
    if kernel == "c4":
        if not _c4_fwd_ok(H):
            pytest.skip("clusters of 4 of the lstm_c4 forward kernel are not co-resident on this GPU")
        r, eps = run_c4_fwd(w.to(bf16), xg, h0, c0), EPS_FAST
    elif kernel == "tc":
        r, eps = run_tc_fwd(w.to(bf16), xg, h0, c0), EPS_FAST
    else:
        r, eps = run_seq_fwd(w, xg, h0, c0), EPS_LIBM
    pre = xg.double().view(B, T, 4, H)
    got = r["gates"].view(B, T, 4, H).double()
    assert torch.isfinite(r["gates"]).all() and torch.isfinite(r["y"]).all() and torch.isfinite(r["cseq"]).all()
    es = float((got[:, :, [0, 1, 3]] - torch.sigmoid(pre[:, :, [0, 1, 3]])).abs().max())
    et = float((got[:, :, 2] - torch.tanh(pre[:, :, 2])).abs().max())
    print("  %s gate nonlinearities: max |sigmoid err| %.3g, max |tanh err| %.3g (EPS_ACT %.3g)" % (kernel, es, et, eps))
    _limits_exact(kernel + " gates", r["gates"], pre, kernel != "seq")
    assert es <= eps and et <= eps


@pytest.mark.parametrize("kernel,H", [("c4", 256), ("c4", 1024), ("tc", 320), ("seq", 24)])
def test_fwd_saturation(kernel, H):
    """Saturated inputs: 10 % of xg at +-20, +-44 ... +-45, +-87 ... +-90 and +-1e4, |c0| up to 50.  Every output is
    finite, the gates take their exact limits where the fp64 value rounds to them in fp32 (_limits_exact), and every
    element is within the bars of the teacher-forced reference."""
    B, T = 40, 37
    if kernel == "c4":
        r, ref, *_ = _c4_fwd_case(B, T, H, True, 21, sat=True)
    else:
        w, xg, h0, c0 = fwd_inputs(B, T, H, 22, True, sat=True)
        if kernel == "tc":
            w16 = w.to(bf16)
            r = run_tc_fwd(w16, xg, h0, c0)
            ref = _check_fwd("tc_fwd saturated H%d" % H, r, w16, xg, "tc_fwd", EPS_FAST, UTC)
        else:
            r = run_seq_fwd(w, xg, h0, c0)
            ref = _check_fwd("seq_fwd saturated H%d" % H, r, w, xg, "seq", EPS_LIBM, U24)
    for k in ("y", "gates", "cseq", "hT", "cT"):
        assert torch.isfinite(r[k]).all(), k
    _limits_exact(kernel + " saturated", r["gates"], ref["pre"], kernel != "seq")


# ---- BPTT -------------------------------------------------------------------------------------------------------------
def _tc_bwd_case(B, T, H, init, saves, seed, sat=False, long_name=None):
    from edgedict_b200 import ops
    w = (torch.rand(4 * H, H, device=DEV, generator=_gen(seed)) * 2 - 1) / math.sqrt(H)
    w16 = w.to(bf16)
    if saves == "fwd":
        _, xg, h0, c0 = fwd_inputs(B, T, H, seed + 1, True, sat)
        f = run_tc_fwd(w16, xg, h0, c0)
        gates, cseq = f["gates"], f["cseq"]
        c0 = c0 if init else None
    else:
        gates, cseq = synthetic_saves(B, T, H, seed + 1, sat)
        c0 = torch.randn(B, H, device=DEV, generator=_gen(seed + 2)) if init else None
    dy, _, dhT, dcT = bwd_grads(B, T, H, seed + 3, init)
    cs = tc_cluster_size(H)
    dg, dh0, dc0 = ops.lstm_tc_bwd(dy, gates, cseq, c0, w16.t().contiguous(), dhT, dcT)
    torch.cuda.synchronize()
    ref = bwd_ref(dy, gates, cseq, c0, w16, dg, dhT, dcT, _n_add("tc_bwd", H, cs), UTC, EPS_FAST)
    name = long_name or "tc_bwd B%d T%d H%d CS%d %s %s" % (B, T, H, cs, saves, "init" if init else "zero")
    _check_bwd(name, ref, dg, dh0, dc0)


@pytest.mark.parametrize("H", [64, 256, 320, 512, 1024])
@pytest.mark.parametrize("B,T,init,saves", [(5, 37, True, "fwd"), (40, 9, False, "synthetic"), (1, 2, True, "synthetic")])
def test_tc_bwd_teacher_forced(B, T, init, saves, H):
    """eb_lstm_tc_bwd against bwd_ref: n_add = 16 ceil(4H/CS/128) + 8 + CS (each warp's k16 steps over the CTA's 4H/CS
    contraction rows, 8 warp partials, CS CTA partials), u_acc = 2^-23.  The H values reach every cluster size an H100
    picks (printed; 0 = the software reduction through L2, which runs the CS = 4 decomposition)."""
    _tc_bwd_case(B, T, H, init, saves, 4000 * H + 10 * B + T)


LENS = [(5, [1]), (40, [3, 1, 5]), (32, [1] * 8), (5, [7, 2, 1, 9, 4, 1, 3, 5]), (40, [2, 5])]


def _chunks_case(kind, B, lens, H, init, seed, sat=False):
    from edgedict_b200 import ops
    lib = _lib()
    T = sum(lens)
    w = (torch.rand(4 * H, H, device=DEV, generator=_gen(seed)) * 2 - 1) / math.sqrt(H)
    w16 = w.to(bf16)
    if sat:
        _, xg, h0, c0 = fwd_inputs(B, T, H, seed + 1, True, True)
        f = run_c4_fwd(w16, xg, h0, c0) if _c4_fwd_ok(H) and H % 256 == 0 else run_tc_fwd(w16, xg, h0, c0)
        gates, cseq = f["gates"], f["cseq"]
    else:
        gates, cseq = synthetic_saves(B, T, H, seed + 1)
        c0 = torch.randn(B, H, device=DEV, generator=_gen(seed + 2)) if init else None
    dy, _, dhT, dcT = bwd_grads(B, T, H, seed + 3, init or sat)
    if kind == "c4":
        if not ops.lstm_c4_bwd_chunks_supported(H):
            pytest.skip("clusters of 16 of the lstm_c4 BPTT kernel are not co-resident on this GPU")
        entry, sb, n_add, cs = lib.eb_lstm_c4_bwd_chunks, lib.eb_lstm_c4_scratch_bytes, _n_add("c4_bwd", H, 16), 16
    else:
        cs = tc_cluster_size(H)
        entry, sb, n_add = lib.eb_lstm_tc_bwd_chunks, lib.eb_lstm_tc_scratch_bytes, _n_add("tc_bwd", H, cs)
    dg, dh0, dc0 = _chunk_call(entry, dy, gates, cseq, c0, w16, dhT, dcT, lens, sb)
    ref = bwd_ref(dy, gates, cseq, c0, w16, dg, dhT, dcT, n_add, UTC, EPS_FAST)
    name = "%s_bwd_chunks B%d H%d CS%d %s%s" % (kind, B, H, cs, lens if len(lens) < 5 else "%d chunks" % len(lens),
                                                 " sat" if sat else "")
    _check_bwd(name, ref, dg, dh0, dc0)


@pytest.mark.parametrize("H", [256, 320, 1024])
@pytest.mark.parametrize("B,lens", LENS)
def test_tc_bwd_chunks_teacher_forced(B, lens, H):
    """eb_lstm_tc_bwd_chunks over chunk-major buffers, with c0 / dh_T / dc_T: chunk lists with length-1 chunks, odd
    lengths (the double-buffer parity flips at a chunk boundary) and 8 chunks, the most the entry takes.  dg16 is read
    back through the inverse of the scatter, and a guard row past the buffer must stay untouched."""
    _chunks_case("tc", B, lens, H, B != 32, 5000 * H + 10 * B + len(lens))


@pytest.mark.parametrize("H", [256, 512, 1024])
@pytest.mark.parametrize("B,lens", LENS)
def test_c4_bwd_chunks_teacher_forced(B, lens, H):
    """eb_lstm_c4_bwd_chunks (K split over clusters of 16), c0 / dh_T / dc_T given except at B = 32: n_add = H/4 + 16
    (wgmma over the CTA's K slice, then the 16 partials), u_acc = 2^-23.  Same chunk lists as the tc entry."""
    _chunks_case("c4", B, lens, H, B != 32, 6000 * H + 10 * B + len(lens))


def _c4_bwd_case(B, T, H, init, sat=False):
    from edgedict_b200 import ops
    cs = _lib().eb_lstm_c4_bwd_cluster(H)
    if cs == 0 or not _c4_fwd_ok(H):
        pytest.skip("clusters of the lstm_c4 BPTT kernel over CTA-private saves are not co-resident on this GPU")
    seed = 7000 * H + 10 * B + T
    w = (torch.rand(4 * H, H, device=DEV, generator=_gen(seed)) * 2 - 1) / math.sqrt(H)
    w16 = w.to(bf16)
    _, xg, h0, c0 = fwd_inputs(B, T, H, seed + 1, True, sat)
    f = run_c4_fwd(w16, xg, h0, c0)
    c0 = c0 if init or sat else None
    dy, _, dhT, dcT = bwd_grads(B, T, H, seed + 3, init or sat)
    dg, dh0, dc0 = ops.lstm_c4_bwd(dy, f["gsave"], f["csave"], c0, w16.t().contiguous(), dhT, dcT)
    torch.cuda.synchronize()
    gates = c4_decode_gates(f["gsave"], B, T, H)
    cseq = c4_decode_cells(f["csave"], B, T, H)
    ref = bwd_ref(dy, gates, cseq, c0, w16, dg, dhT, dcT, _n_add("c4_bwd", H, cs), UTC, EPS_FAST)
    _check_bwd("c4_bwd B%d T%d H%d CS%d%s" % (B, T, H, cs, " sat" if sat else ""), ref, dg, dh0, dc0)


@pytest.mark.parametrize("H", [256, 512, 768, 1024])
@pytest.mark.parametrize("B,T,init", [(5, 37, True), (40, 9, False), (1, 1, True)])
def test_c4_bwd_teacher_forced(B, T, init, H):
    """eb_lstm_c4_bwd over the CTA-private saves of eb_lstm_c4_fwd: the reference reads the same bf16-rounded gates
    (decoded from gsave) and the fp32 cells (csave); n_add = 4H/CS + CS with CS = eb_lstm_c4_bwd_cluster(H)."""
    _c4_bwd_case(B, T, H, init)


def _seq_bwd_case(B, T, H, init, saves, sat=False):
    from edgedict_b200 import ops
    seed = 8000 * H + 10 * B + T
    w = (torch.rand(4 * H, H, device=DEV, generator=_gen(seed)) * 2 - 1) / math.sqrt(H)
    if saves == "fwd":
        _, xg, h0, c0 = fwd_inputs(B, T, H, seed + 1, True, sat)
        f = run_seq_fwd(w, xg, h0, c0)
        gates, cseq = f["gates"], f["cseq"]
        c0 = c0 if init or sat else None
    else:
        gates, cseq = synthetic_saves(B, T, H, seed + 1, sat)
        c0 = torch.randn(B, H, device=DEV, generator=_gen(seed + 2)) if init else None
    dy, _, dhT, dcT = bwd_grads(B, T, H, seed + 3, init or sat)
    snap = gates.clone()
    dg, dh0, dc0 = ops.lstm_seq_bwd(dy, gates, cseq, c0, w, dhT, dcT)
    torch.cuda.synchronize()
    ref = bwd_ref(dy, snap, cseq, c0, w, dg, dhT, dcT, _n_add("seq", H), U24, EPS_LIBM)
    _check_bwd("seq_bwd B%d T%d H%d %s%s" % (B, T, H, saves, " sat" if sat else ""), ref, dg, dh0, dc0, bf16_out=False)


@pytest.mark.parametrize("H", [8, 24, 320, 1024])
@pytest.mark.parametrize("B,T,init,saves", [(5, 37, True, "fwd"), (40, 9, False, "synthetic"), (1, 1, True, "synthetic")])
def test_seq_bwd_teacher_forced(B, T, init, saves, H):
    """eb_lstm_seq_bwd (fp32): dgates are written in place over the gates, so the reference reads a snapshot; the
    exchanged dG is the fp32 dgates itself (identity rounding), n_add = 4H + 8, u = 2^-24, EPS_LIBM."""
    _seq_bwd_case(B, T, H, init, saves)


@pytest.mark.parametrize("kernel", ["tc", "tc_chunks", "c4_chunks", "c4", "seq"])
def test_bwd_saturation(kernel):
    """BPTT over the saves of a saturated forward (10 % of xg at +-20 ... +-1e4, |c0| up to 50: gates at exactly 0 / 1,
    cells far beyond the range where 1 - tanh(c)^2 keeps any relative precision) and, for the tc kernel, synthetic
    saves with exact 0 / 1 / -1 gates and cells up to +-50.  Every gradient is finite and within the same bars."""
    if kernel == "tc":
        _tc_bwd_case(40, 37, 320, True, "fwd", 91, sat=True, long_name="tc_bwd saturated fwd saves H320")
        _tc_bwd_case(40, 37, 1024, True, "synthetic", 92, sat=True, long_name="tc_bwd saturated synthetic H1024")
    elif kernel == "tc_chunks":
        _chunks_case("tc", 40, [3, 1, 5, 2], 512, True, 93, sat=True)
    elif kernel == "c4_chunks":
        _chunks_case("c4", 40, [3, 1, 5, 2], 1024, True, 94, sat=True)
    elif kernel == "c4":
        _c4_bwd_case(40, 37, 256, True, sat=True)
    else:
        _seq_bwd_case(40, 37, 24, True, "fwd", sat=True)
        _seq_bwd_case(40, 37, 320, True, "synthetic", sat=True)


@pytest.mark.parametrize("kernel", ["tc", "c4_chunks"])
def test_bwd_long_sequence(kernel):
    """One long BPTT per bf16 BPTT path that the training step runs: eb_lstm_tc_bwd at T = 300 and eb_lstm_c4_bwd_chunks
    over 8 chunks, T = 317, both at H = 1024, B = 32."""
    if kernel == "tc":
        _tc_bwd_case(32, 300, 1024, True, "fwd", 95, long_name="tc_bwd long T300 H1024")
    else:
        _chunks_case("c4", 32, [40] * 7 + [37], 1024, True, 96)
