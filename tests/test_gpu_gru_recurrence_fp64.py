"""Teacher-forced fp64 parity of the recurrent GRU kernels, per step and per element: eb_gru_seq_fwd / eb_gru_seq_bwd
(fp32) and eb_gru_tc_fwd / eb_gru_tc_bwd (bf16 tensor-core operands, fp32 accumulation and state).

Every operand of the recurrence is visible from outside: the h_{t-1} a forward step multiplies is y[:, t-1] (h0 at
t = 0) -- rounded to bf16 by the tc kernel, whose update z h_{t-1} keeps the fp32 value -- and the dgh a BPTT step
multiplies is the kernel's dgh output of the step after it (fp32, or the bf16 dgh16 of the tc kernel).  The fp64
references therefore compute step t from the kernel's own inputs to step t, so errors do not compound over t and a
failure names one (batch row, step, gate, unit).  Only the direct term dh z of dh_{t-1} = dh z + W_hh^T dgh is recursed in fp64 (elementwise, contracting with z <= 1), with its bar recursed alongside.

Error model (first order, per element; the same method as test_gpu_lstm_recurrence_fp64.py):
  recurrent sums  n_add u_acc sum_k |h_k||w_k| (fp32 kernels: n_add = 3H + 8, the FMA chain plus the K-split partials,
                  u_acc = 2^-24; tc kernels: the k16 steps of one warp plus the 8 warp partials, u_acc = 2^-23), plus
                  one rounding per further add (xg, b_hn);
  gates           sigma' |dpre| + eps, tanh' |dpre| + eps (EPS_LIBM for expf / tanhf, EPS_FAST for ex2.approx);
  n, h            propagated through n = tanh(xg_n + r gh_n) and h = (1 - z) n + z h_{t-1}, plus the fp32 roundings;
  BPTT            dh through the three gate-gradient formulas, plus their roundings.
Every test prints the worst err/bar ratio next to where it occurs (pytest -s)."""
import math

import pytest
import torch

from tests.test_gpu_lstm_recurrence_fp64 import SAT, U24, UTC, EPS_FAST, EPS_LIBM, _bf16_ulp, _plant, _report

pytestmark = pytest.mark.gpu

f32, f64 = torch.float32, torch.float64
DEV = "cuda"


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


bf16 = torch.bfloat16


def _n_add(kernel, H):
    """Longest fp32 summation chain of one recurrent sum (forward: over H, BPTT: over 3H)."""
    if kernel == "seq":
        return 3 * H + 8
    if kernel == "tc_fwd":        # each of 8 warps: ceil(H/128) k16 steps, then the 8 warp partials, + xg
        return 16 * -(-H // 128) + 8 + 1
    if kernel == "tc_bwd":        # each of 8 warps: ceil(3H/128) k16 steps, the 8 warp partials, + dh z, + dy
        return 16 * -(-(3 * H) // 128) + 8 + 2
    raise ValueError(kernel)


# ---- kernels ----------------------------------------------------------------------------------------------------------
def run_fwd(xg, w, bhn, h0):
    B, T, H3 = xg.shape
    H = H3 // 3
    L = _lib()
    y = torch.empty(B, T, H, device=DEV)
    hT = torch.empty(B, H, device=DEV)
    save = torch.empty(B, T, 4 * H, device=DEV)
    scratch = torch.zeros(L.eb_gru_scratch_bytes(B, H), dtype=torch.uint8, device=DEV)
    assert L.eb_gru_seq_fwd(_p(xg), _p(w), _p(bhn), _p(h0), _p(y), _p(hT), _p(save), _p(scratch), B, T, H,
                            _stream()) == 0
    torch.cuda.synchronize()
    return y, hT, save


def run_tc_fwd(xg, w, bhn, h0):
    B, T, H3 = xg.shape
    H = H3 // 3
    L = _lib()
    y = torch.empty(B, T, H, device=DEV)
    hT = torch.empty(B, H, device=DEV)
    save = torch.empty(B, T, 4 * H, device=DEV)
    scratch = torch.zeros(L.eb_gru_tc_scratch_bytes(B, H), dtype=torch.uint8, device=DEV)
    w16 = w.to(bf16).contiguous()
    assert L.eb_gru_tc_fwd(_p(xg), _p(w16), _p(bhn), _p(h0), _p(y), _p(hT), _p(save), _p(scratch), B, T, H,
                           _stream()) == 0
    torch.cuda.synchronize()
    return y, hT, save


def run_tc_bwd(dy, save, y, h0, w, dhT):
    B, T, H = dy.shape
    L = _lib()
    dgi = torch.empty(B, T, 3 * H, dtype=bf16, device=DEV)
    dgh = torch.empty(B, T, 3 * H, dtype=bf16, device=DEV)
    dh0 = torch.empty(B, H, device=DEV)
    scratch = torch.zeros(L.eb_gru_tc_scratch_bytes(B, H), dtype=torch.uint8, device=DEV)
    wT16 = w.t().contiguous().to(bf16)
    assert L.eb_gru_tc_bwd(_p(dy), _p(save), _p(y), _p(h0), _p(wT16), _p(dhT), _p(dgi), _p(dgh), _p(dh0), _p(scratch),
                           B, T, H, _stream()) == 0
    torch.cuda.synchronize()
    return dgi, dgh, dh0


def run_bwd(dy, save, y, h0, w, dhT):
    B, T, H = dy.shape
    L = _lib()
    dgi = torch.empty(B, T, 3 * H, device=DEV)
    dgh = torch.empty(B, T, 3 * H, device=DEV)
    dh0 = torch.empty(B, H, device=DEV)
    scratch = torch.zeros(L.eb_gru_scratch_bytes(B, H), dtype=torch.uint8, device=DEV)
    assert L.eb_gru_seq_bwd(_p(dy), _p(save), _p(y), _p(h0), _p(w), _p(dhT), _p(dgi), _p(dgh), _p(dh0), _p(scratch),
                            B, T, H, _stream()) == 0
    torch.cuda.synchronize()
    return dgi, dgh, dh0


# ---- fp64 references --------------------------------------------------------------------------------------------------
def hprev_of(y, h0):
    B, _, H = y.shape
    first = torch.zeros(B, 1, H, dtype=y.dtype, device=y.device) if h0 is None else h0[:, None].to(y.dtype)
    return torch.cat([first, y[:, :-1]], 1)


def fwd_ref(xg, w, bhn, hin, hst=None, kernel="seq", u_acc=U24, eps=EPS_LIBM, dxg=0.0):
    """Teacher-forced forward, every step at once: xg [B,T,3H], w [3H,H] (the values the kernel multiplies), bhn [H],
    hin [B,T,H] the h_{t-1} the kernel multiplied, hst the h_{t-1} of its update (default: hin).  dxg [B,T,3H] is a
    bar the xg input already carries (0 when xg is the kernel's own input).  Returns {name: (value, bar)} for r, z, n,
    gh_n and y [B,T,H]."""
    hst = hin if hst is None else hst
    xg, w, bhn, hin, hst = (a.to(f64) for a in (xg, w, bhn, hin, hst))
    B, T, H3 = xg.shape
    H = H3 // 3
    s = hin @ w.t()
    ds = _n_add(kernel, H) * u_acc * (hin.abs() @ w.abs().t())
    xr, xz, xn = xg.view(B, T, 3, H).unbind(2)
    sr, sz, sn = s.view(B, T, 3, H).unbind(2)
    dsr, dsz, dsn = ds.view(B, T, 3, H).unbind(2)
    dxr, dxz, dxn = dxg.to(f64).view(B, T, 3, H).unbind(2) if torch.is_tensor(dxg) else (dxg,) * 3
    out = {}
    gates = {}
    for name, x, sv, dv, dx in (("r", xr, sr, dsr, dxr), ("z", xz, sz, dsz, dxz)):
        pre = x + sv
        dpre = dv + dx + U24 * (sv.abs() + x.abs())
        g = torch.sigmoid(pre)
        gates[name] = g
        out[name] = (g, g * (1 - g) * dpre + eps + U24 * g)
    r, z = gates["r"], gates["z"]
    dr, dz = out["r"][1], out["z"][1]
    ghn = sn + bhn
    dghn = dsn + U24 * ghn.abs()
    out["ghn"] = (ghn, dghn)
    a = xn + r * ghn
    da = dxn + dr * ghn.abs() + r * dghn + 2 * U24 * ((r * ghn).abs() + a.abs())
    n = torch.tanh(a)
    dn = (1 - n * n) * da + eps + U24 * n.abs()
    out["n"] = (n, dn)
    y = (1 - z) * n + z * hst
    dy = dz * (n.abs() + hst.abs()) + (1 - z) * dn + 3 * U24 * (((1 - z) * n).abs() + (z * hst).abs())
    out["y"] = (y, dy)
    return out


def bwd_ref(dy, save, hin, w, dghk, dhT, kernel="seq", u_acc=U24):
    """Teacher-forced BPTT.  dy [B,T,H]; save [B,T,4H] = r|z|n|gh_n as the kernel read it; hin [B,T,H] the h_{t-1} of
    each step; w [3H,H]; dghk [B,T,3H] the kernel's own dgh (the operand of the exchanged recurrence).  dh_t =
    dy_t + z_{t+1} dh_{t+1} + dghk_{t+1} W (+ dhT at T-1), the direct term recursed in fp64 with its bar.  Returns
    {name: (value, bar)} for dgi, dgh [B,T,3,H] and dh0 [B,H]."""
    dy, save, hin, w, dghk = (a.to(f64) for a in (dy, save, hin, w, dghk))
    B, T, H = dy.shape
    r, z, n, ghn = save.view(B, T, 4, H).unbind(2)
    n_add = _n_add(kernel, H)
    rec = torch.zeros_like(dy)
    drec = torch.zeros_like(dy)
    if T > 1:
        m = dghk[:, 1:] @ w
        rec[:, :-1] = m
        drec[:, :-1] = n_add * u_acc * (dghk[:, 1:].abs() @ w.abs())
    dh_all, ddh_all = torch.empty_like(dy), torch.empty_like(dy)
    carry = torch.zeros(B, H, dtype=f64, device=dy.device) if dhT is None else dhT.to(f64)
    dcarry = torch.zeros_like(carry)
    for t in range(T - 1, -1, -1):
        # kernel: dh_rec = (dh_{t+1} z_{t+1}) + (W^T dgh_{t+1}), then dh = dy + dh_rec
        dh_rec = carry + rec[:, t]
        ddh_rec = dcarry + drec[:, t] + U24 * dh_rec.abs()
        dh = dy[:, t] + dh_rec
        ddh = ddh_rec + U24 * dh.abs()
        dh_all[:, t], ddh_all[:, t] = dh, ddh
        carry = dh * z[:, t]
        dcarry = ddh * z[:, t] + U24 * carry.abs()
    dh, ddh = dh_all, ddh_all
    dn = dh * (1 - z) * (1 - n * n)
    ddn = ddh * ((1 - z) * (1 - n * n)).abs() + 2 * U24 * (dh * (1 - z)).abs() + 4 * U24 * dn.abs()
    kz = (hin - n) * z * (1 - z)
    dzg = dh * kz
    ddz = ddh * kz.abs() + 6 * U24 * dh.abs() * (hin.abs() + n.abs()) * z * (1 - z)
    kr = ghn * r * (1 - r)
    dr = dn * kr
    ddr = ddn * kr.abs() + 6 * U24 * (dn * ghn).abs() * r * (1 - r)
    dhn = r * dn
    ddhn = r * ddn + U24 * dhn.abs()
    dgi = torch.stack([dr, dzg, dn], 2)
    dgib = torch.stack([ddr, ddz, ddn], 2)
    dgh = torch.stack([dr, dzg, dhn], 2)
    dghb = torch.stack([ddr, ddz, ddhn], 2)
    m0 = dghk[:, 0] @ w
    dh0 = carry + m0
    dh0b = dcarry + n_add * u_acc * (dghk[:, 0].abs() @ w.abs()) + U24 * dh0.abs()
    return dict(dgi=(dgi, dgib), dgh=(dgh, dghb), dh0=(dh0, dh0b))


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def gru_inputs(B, T, H, seed, init, sat=False, big_bhn=False):
    """w [3H,H] ~ U(-1/sqrt(H), 1/sqrt(H)), bhn ~ U(-1, 1), xg ~ N(0, 1), h0 ~ N(0, 1/4) or None.  sat: 10 % of xg at the
    values of SAT.  big_bhn: b_hn = +-30 with the reset pre-activation pushed to +-20 (r near 0 or 1) on half the
    elements."""
    gen = _gen(seed)
    w = (torch.rand(3 * H, H, device=DEV, generator=gen) * 2 - 1) / math.sqrt(H)
    bhn = torch.rand(H, device=DEV, generator=gen) * 2 - 1
    xg = torch.randn(B, T, 3 * H, device=DEV, generator=gen)
    h0 = torch.randn(B, H, device=DEV, generator=gen) * 0.5 if init else None
    if sat:
        xg = _plant(xg, gen, 0.1, SAT)
    if big_bhn:
        bhn = torch.where(torch.rand(H, device=DEV, generator=gen) < 0.5, -30.0, 30.0)
        xg[..., :H] = _plant(xg[..., :H], gen, 0.5, [20.0])
    return w, bhn, xg.contiguous(), h0


CASES = [  # (H, B, T, h0 / dhT, seed)
    (48, 5, 37, True, 1),
    (48, 1, 1, False, 2),
    (100, 40, 37, True, 3),
    (100, 32, 2, False, 4),
    (64, 1, 2, True, 5),
    (64, 32, 37, False, 6),
    (256, 5, 1, True, 7),
    (256, 40, 37, True, 8),
    (320, 32, 37, True, 9),
    (320, 1, 37, False, 10),
    (1024, 32, 37, True, 11),
    (1024, 5, 2, False, 12),
    (256, 32, 300, True, 13),
]


def _fwd_case(H, B, T, init, seed, tc=False, **kw):
    w, bhn, xg, h0 = gru_inputs(B, T, H, seed, init, **kw)
    if tc:
        y, hT, save = run_tc_fwd(xg, w, bhn, h0)
        hst = hprev_of(y, h0)
        ref = fwd_ref(xg, w.to(bf16), bhn, hst.to(bf16), hst, "tc_fwd", UTC, EPS_FAST)
    else:
        y, hT, save = run_fwd(xg, w, bhn, h0)
        ref = fwd_ref(xg, w, bhn, hprev_of(y, h0))
    r, z, n, ghn = save.view(B, T, 4, H).unbind(2)
    name = "gru_%s_fwd H=%d B=%d T=%d%s" % ("tc" if tc else "seq", H, B, T, " h0" if init else "")
    _report(name, [("r", r, *ref["r"]), ("z", z, *ref["z"]), ("n", n, *ref["n"]), ("gh_n", ghn, *ref["ghn"]),
                   ("y", y, *ref["y"])])
    assert torch.equal(hT, y[:, -1])
    return w, bhn, xg, h0, y, save


def _bwd_case(H, B, T, init, seed, tc=False, **kw):
    w, bhn, xg, h0, y, save = _fwd_case(H, B, T, init, seed, tc=tc, **kw)
    gen = _gen(seed + 1000)
    dy = torch.randn(B, T, H, device=DEV, generator=gen)
    dhT = torch.randn(B, H, device=DEV, generator=gen) if init else None
    if tc:
        dgi, dgh, dh0 = run_tc_bwd(dy, save, y, h0, w, dhT)
        ref = bwd_ref(dy, save, hprev_of(y, h0), w.to(bf16), dgh, dhT, "tc_bwd", UTC)
        # dgi16 / dgh16 are bf16 roundings of the fp32 values: half a bf16 ulp on top of the bar
        for k in ("dgi", "dgh"):
            val, bar = ref[k]
            ref[k] = (val, bar + 0.5 * _bf16_ulp(val.abs() + bar))
    else:
        dgi, dgh, dh0 = run_bwd(dy, save, y, h0, w, dhT)
        ref = bwd_ref(dy, save, hprev_of(y, h0), w, dgh, dhT)
    name = "gru_%s_bwd H=%d B=%d T=%d%s" % ("tc" if tc else "seq", H, B, T, " h0 dhT" if init else "")
    _report(name, [("dgi", dgi.view(B, T, 3, H), *ref["dgi"]), ("dgh", dgh.view(B, T, 3, H), *ref["dgh"]),
                   ("dh0", dh0, *ref["dh0"])])
    # the r and z slices of the two gate gradients are the same numbers
    assert torch.equal(dgi[..., :2 * H], dgh[..., :2 * H])


@pytest.mark.parametrize("H,B,T,init,seed", CASES)
def test_gru_seq_fwd_per_step(H, B, T, init, seed):
    _fwd_case(H, B, T, init, seed)


@pytest.mark.parametrize("H,B,T,init,seed", CASES)
def test_gru_seq_bwd_per_step(H, B, T, init, seed):
    _bwd_case(H, B, T, init, seed)


@pytest.mark.parametrize("H,B,T", [(64, 5, 37), (100, 32, 37), (1024, 32, 2)])
def test_gru_saturated_gate_inputs(H, B, T):
    _bwd_case(H, B, T, True, 21, sat=True)


@pytest.mark.parametrize("H,B,T", [(48, 5, 37), (256, 32, 37)])
def test_gru_large_b_hn_reset_near_zero_and_one(H, B, T):
    """b_hn sits inside the reset product: with |b_hn| = 30 and r at sigmoid(+-20), n differs by O(30) between the
    right and a wrong placement of b_hn."""
    w, bhn, xg, h0, y, save = _fwd_case(H, B, T, True, 31, big_bhn=True)
    r = save.view(B, T, 4, H)[:, :, 0]
    assert (r < 1e-8).any() and (r > 1 - 1e-7).any()
    _bwd_case(H, B, T, True, 31, big_bhn=True)


def test_gru_long_sequence_h1024():
    _bwd_case(1024, 40, 320, True, 41)


def test_gru_h0_and_dhT_reach_the_first_and_last_step():
    """h0 enters step 0's update and reset product; dhT enters step T-1's gradient; both vanish without them."""
    H, B, T = 64, 5, 3
    w, bhn, xg, h0 = gru_inputs(B, T, H, 51, True)
    y1, _, _ = run_fwd(xg, w, bhn, h0)
    y0, _, _ = run_fwd(xg, w, bhn, None)
    assert (y1[:, 0] - y0[:, 0]).abs().max() > 1e-2
    _, _, save = run_fwd(xg, w, bhn, h0)
    dy = torch.zeros(B, T, H, device=DEV)
    dhT = torch.randn(B, H, device=DEV)
    dgi, _, dh0 = run_bwd(dy, save, y1, h0, w, dhT)
    assert dgi[:, -1].abs().max() > 0 and dh0.abs().max() > 0
    dgi0, _, dh00 = run_bwd(dy, save, y1, h0, w, None)
    assert dgi0.abs().max() == 0 and dh00.abs().max() == 0


# ---- tensor-core kernels (H % 64 == 0, H <= 1024) ---------------------------------------------------------------------
TC_CASES = [  # (H, B, T, h0 / dhT, seed)
    (64, 1, 1, False, 61),
    (64, 5, 37, True, 62),
    (256, 32, 2, True, 63),
    (256, 40, 37, False, 64),
    (320, 5, 37, True, 65),
    (1024, 32, 37, True, 66),
    (1024, 40, 2, False, 67),
    (1024, 32, 300, True, 68),
]


@pytest.mark.parametrize("H,B,T,init,seed", TC_CASES)
def test_gru_tc_fwd_per_step(H, B, T, init, seed):
    _fwd_case(H, B, T, init, seed, tc=True)


@pytest.mark.parametrize("H,B,T,init,seed", TC_CASES)
def test_gru_tc_bwd_per_step(H, B, T, init, seed):
    _bwd_case(H, B, T, init, seed, tc=True)


@pytest.mark.parametrize("H,B,T", [(64, 5, 37), (1024, 32, 2)])
def test_gru_tc_saturated_gate_inputs(H, B, T):
    _bwd_case(H, B, T, True, 71, tc=True, sat=True)


def test_gru_tc_large_b_hn_reset_near_zero_and_one():
    H, B, T = 256, 32, 37
    _, _, _, _, _, save = _fwd_case(H, B, T, True, 72, tc=True, big_bhn=True)
    r = save.view(B, T, 4, H)[:, :, 0]
    assert (r < 1e-8).any() and (r > 1 - 1e-7).any()
    _bwd_case(H, B, T, True, 72, tc=True, big_bhn=True)


def test_unsupported_hidden_sizes_are_refused():
    """H = 4096 does not fit the fp32 kernels' shared memory; the tc kernels take H % 64 == 0, H <= 1024 only."""
    L = _lib()
    assert L.eb_gru_scratch_bytes(4, 4096) == 0
    P = 1 << 20
    assert L.eb_gru_seq_fwd(P, P, P, None, P, P, P, P, 4, 3, 4096, None) == 2
    assert L.eb_gru_seq_bwd(P, P, P, None, P, None, P, P, P, P, 4, 3, 4096, None) == 2
    assert L.eb_gru_tc_supported(4, 2048) == 0 and L.eb_gru_tc_supported(4, 1024) == 1
