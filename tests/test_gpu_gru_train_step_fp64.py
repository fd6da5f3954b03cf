"""Teacher-forced fp64 parity of the GRU training step, per layer and per element: functional.GRULayer, the
Encoder(module=ResLayerNormGRU) stack of CTCEncoder, CTCEncoder's output layer (Linear + LogSoftmax) and its loss
(edgedict_b200.ctc.ctc_loss on CTCLossFn), and the CTC lattice with four states per thread (2S+1 > 1024).

The recurrent kernels are pinned one by one by test_gpu_gru_recurrence_fp64.py; this file pins the code that composes
them: the input GEMM and its folded bias [b_ir + b_hr, b_iz + b_hz, b_in] (b_hn stays inside the reset product and
reaches the kernel unfolded), the h_{t-1} operand of the recurrence (bf16 for the tensor-core kernel) and of dW_hh, the
choice between dgi and dgh for each GEMM, the bf16 casts of the fp32-recurrence fallback, the bias gradients in
eb_colsum's order, LayerNorm with the residual, TimeReduction on an odd length, the sum of the dgrad GEMM and the residual
gradient, and the head's d logits with the per-utterance factor of the loss.  Every operation is captured by wrapping
its `ops` entry (`Tap`: arguments before the call, results after, cloned), and each layer is checked from the engine's
own inputs to that layer, so errors do not compound and a failure names one (batch row, step, gate, unit):

  GRULayer fwd  xg = x16 bf16(W_ih)^T + bias in fp64 with the bar of its GEMM plan (n_add 2^-23 per add, or K 2^-24 for
                the fp32 GEMM) plus one rounding of b_i + b_h, checked against the GEMM's output and passed to the
                recurrence reference (`fwd_ref`, dxg); h_{t-1} = bf16(y shifted) (tc) or y shifted (fp32 recurrence)
                with the fp32 value in the update; r, z, n, gh_n from the save and y against their bars.
  GRULayer bwd  `bwd_ref` over the whole layer with the kernel's own dgh as the recurrent operand; dgi16 / dgh16 within
                the bar plus half a bf16 ulp, every element a rounding of a value within the bar and at most FRAC_DIFF
                of them different from bf16_rn(ref) (test_gpu_train_step_fp64.check_lstm_bwd's rule); the fallback's
                casts bitwise; dx = dgi16 bf16(W_ih), dW_ih = dgi16^T x16, dW_hh = dgh16^T bf16([h0 | y[:, :-1]])
                against fp64 with the n_add u |A||B| bars of their plans; db_ih, db_hh bitwise in eb_colsum's order
                (bf16 lanes for the tc kernel's bf16 rows, colsum_kernel's for fp32 rows); dh0 within its bar.
  stack         LayerNorm mean / rstd / output teacher-forced from the saved statistics (test_gpu_glue_fp64.py's bars),
                its input y (+ the layer's input for i > 0) bitwise; TimeReduction forward and backward bitwise (zero pad
                of the odd frame); LayerNorm dz and dgamma within their bars, dbeta bitwise in its kernel's order; the
                gradient of every layer's input bitwise fl(dx_gemm + dz_residual) of the engine's two terms; the proj
                Linear's output, dx, dW per element and db bitwise.
  head          logits = bf16(enc) bf16(W)^T + b with the plan's bar; log-probs within test_gpu_ctc.py's per-element
                bar; costs, loss and d log_probs against F.ctc_loss in fp64 on the CPU of the engine's own log-probs
                (COST_REL relative, GRAD_ABS absolute; reduction 'mean': the factor 1 / (N max(tl, 1)) included);
                log-softmax backward dx = g - e^y sum g within its bar; the tovocab Linear's dW and dx per element, db
                bitwise.
  lattice       ctc_lattice_kernel<4> (S = 512 and 1023) against F.ctc_loss fp64 under every reduction and both
                values of zero_infinity, with repeated labels planted in the states only its third and fourth slots hold.

References are built in slices of batch rows (teacher forcing makes the rows independent).  Every check prints its worst
err/bar and where it occurs (pytest -s); DESIGN.md section 2 records the measured figures."""
import inspect
import math

import pytest
import torch

from tests.test_gpu_ctc import COST_REL, E6D2, GRAD_ABS, _run
from tests.test_gpu_ctc import TINY as CTC_TINY
from tests.test_gpu_gemm_fp64 import _plan, _same
from tests.test_gpu_gemm_fp64 import _n_add as gemm_n_add
from tests.test_gpu_glue_fp64 import _colsum_order, _dbeta_order, _ln_ref, ln_bwd_ref
from tests.test_gpu_gru_recurrence_fp64 import bwd_ref, fwd_ref
from tests.test_gpu_lstm_recurrence_fp64 import EPS_FAST, EPS_LIBM, FRAC_DIFF, U24, UTC, _bf16_ulp, worst
from tests.test_gpu_train_step_fp64 import Worst, _colsum_lanes, _shift, _slices

pytestmark = pytest.mark.gpu

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
ENTRIES = ("mm_nt", "mm_nn", "mm_tn", "colsum", "gru_tc_fwd", "gru_seq_fwd", "gru_tc_bwd", "gru_seq_bwd",
           "layernorm_fwd", "layernorm_bwd", "time_reduce_fwd", "time_reduce_bwd", "log_softmax_fwd",
           "log_softmax_bwd", "ctc_loss_fwd", "ctc_loss_bwd")


# ---- capture ----------------------------------------------------------------------------------------------------------
def _clone(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, (tuple, list)):
        return type(v)(_clone(a) for a in v)
    return v


class Tap:
    """Wraps the `ops` entries and records every call in order: (entry, arguments by name, result), the tensors cloned
    (arguments before the call, results after it)."""

    def __init__(self, monkeypatch, entries=ENTRIES):
        from edgedict_b200 import ops
        self.calls = []
        for e in entries:
            orig = getattr(ops, e)
            sig = inspect.signature(orig)

            def wrapped(*a, _o=orig, _e=e, _s=sig, **kw):
                ba = _s.bind(*a, **kw)
                ba.apply_defaults()
                args = {k: _clone(v) for k, v in ba.arguments.items()}
                out = _o(*a, **kw)
                self.calls.append((_e, args, _clone(out)))
                return out
            monkeypatch.setattr(ops, e, wrapped)

    def of(self, *entries):
        return [(e, a, o) for e, a, o in self.calls if e in entries]


def _layer_events(tap, L, linear_first=0):
    """Per GRU layer (forward order): its input GEMM, recurrence forward / backward, dgrad GEMM, the two weight-gradient
    GEMMs and the two column sums.  linear_first: Linear layers whose backward runs before the top GRU layer's."""
    mm_nt, rf, rb = tap.of("mm_nt"), tap.of("gru_tc_fwd", "gru_seq_fwd"), tap.of("gru_tc_bwd", "gru_seq_bwd")
    nn, tn, cs = tap.of("mm_nn"), tap.of("mm_tn"), tap.of("colsum")
    assert len(rf) == L and len(rb) == L, (len(rf), len(rb))
    out = []
    for i in range(L):
        k = L - 1 - i
        j = linear_first + k
        out.append(dict(mm=mm_nt[i], fwd=rf[i], bwd=rb[k], nn=nn[j], tn=tn[linear_first + 2 * k:linear_first + 2 * k + 2],
                        cs=cs[linear_first + 2 * k:linear_first + 2 * k + 2],
                        rec="tc" if rf[i][0] == "gru_tc_fwd" else "seq"))
        assert rb[k][0] == ("gru_tc_bwd" if out[-1]["rec"] == "tc" else "gru_seq_bwd"), (rf[i][0], rb[k][0])
    return out


# ---- bars -------------------------------------------------------------------------------------------------------------
def _gemm(precision, M, N, K):
    """(n_add, u) of one output element of C[M,N] = A[M,K] B[N,K]^T: the wgmma plan's chain at 2^-23 per add in bf16
    mode (GRULayer and Linear pass no flags), eb_gemm_f32's K-term FMA chain at 2^-24 in fp32 mode."""
    if precision == "bf16":
        return gemm_n_add(K, _plan(M, N, K)[1]), UTC
    return K, U24


def _op(t, precision):
    """The value a GEMM multiplies: bf16_rn(t) in bf16 mode, t in fp32 mode."""
    return (t if t.dtype == bf16 else t.to(bf16)).double() if precision == "bf16" else t.double()


def _ragged(B, T, gen):
    """Per-frame scale factors in [1/4, 4]: rows of very different magnitudes."""
    return torch.exp((torch.rand(B, T, 1, device=DEV, generator=gen) * 2 - 1) * math.log(4.0))


def _check_rounded(name, chk, label, got, val, bar, row0, stats):
    """got (bf16) within bar + half a bf16 ulp of val, every element a rounding of a value within the bar; counts the
    elements whose bits differ from bf16_rn(val) into stats."""
    lo, hi = (val - bar).to(f32).to(bf16).double(), (val + bar).to(f32).to(bf16).double()
    d = got.double()
    stats[0] += int(((d < lo) | (d > hi)).sum())
    stats[1] += int((got != val.to(f32).to(bf16)).sum())
    stats[2] += got.numel()
    chk.add(label, got, val, bar + 0.5 * _bf16_ulp(val.abs() + bar), row0=row0)


def _rounding_done(name, stats):
    outside, ndiff, n = stats
    frac = ndiff / max(n, 1)
    print("  %-40s dgi16 / dgh16 bits != bf16_rn(ref): %.4f of the elements (bar %.3g), %d outside the rounded bar"
          % (name, frac, FRAC_DIFF, outside))
    assert outside == 0, "%s: %d bf16 gate gradients are not a rounding of a value within the bar" % (name, outside)
    assert frac <= FRAC_DIFF, "%s: %.4f of dgi16 / dgh16 differs from bf16_rn(ref)" % (name, frac)


# ---- one GRU layer, teacher-forced ------------------------------------------------------------------------------------
def check_gru_layer(name, ev, x, w_ih, w_hh, b_ih, b_hh, precision, grads, h0=None, dh0=None, dhT=None, dy=None):
    """The forward and backward checks of one GRULayer (module docstring) from its captured events.  x [B,T,I] fp32 the
    layer's input; grads (dW_ih, dW_hh, db_ih, db_hh) as autograd returned them; h0 / dh0 (h0's gradient) / dhT / dy
    the initial state and the incoming gradients when the caller knows them.  Returns the dgrad GEMM's output [B,T,I]."""
    B, T, I = x.shape
    H = w_hh.shape[1]
    H3, M = 3 * H, B * T
    w_ih, w_hh, b_ih, b_hh = (t.detach() for t in (w_ih, w_hh, b_ih, b_hh))
    tc, bfm = ev["rec"] == "tc", precision == "bf16"
    print("  %s: recurrence %s, %s mode" % (name, ev["rec"], precision))
    assert not tc or bfm
    _, ma, xg = ev["mm"]
    _same(name + " input GEMM operand = the layer's input", ma["x"], x.reshape(M, I))
    if bfm:
        _same(name + " x16 = bf16_rn(x)", ma["x16"], x.reshape(M, I).to(bf16))
    else:
        assert ma["x16"] is None and ma["precision"] == "fp32"
    _same(name + " GEMM bias = [b_ir + b_hr, b_iz + b_hz, b_in]", ma["bias"],
          torch.cat([b_ih[:2 * H] + b_hh[:2 * H], b_ih[2 * H:]]))
    _, fa, (y, hT, save) = ev["fwd"]
    _same(name + " b_hn reaches the recurrence unfolded", fa["bhn"], b_hh[2 * H:])
    _same(name + " recurrence input = the GEMM's output", fa["xg"], xg.view(B, T, H3))
    _same(name + " hT = y[:, -1]", hT, y[:, -1])
    if h0 is None:
        assert fa["h0"] is None
        h0v = torch.zeros(B, H, device=DEV)
    else:
        _same(name + " h0 reaches the recurrence", fa["h0"], h0)
        h0v = h0
    hst = _shift(h0v, y)                                    # the fp32 h_{t-1} of the update
    # ---- forward: xg in fp64 with its GEMM's bar, then the recurrence from the kernel's own h_{t-1} ----
    wih = _op(w_ih, precision)
    bias = torch.cat([b_ih[:2 * H].double() + b_hh[:2 * H].double(), b_ih[2 * H:].double()])
    bias_bar = torch.cat([U24 * bias[:2 * H].abs(), torch.zeros(H, dtype=f64, device=DEV)])  # one rounding of b_i + b_h
    n_in, u_in = _gemm(precision, M, H3, I)
    kf, u_rec, eps = ("tc_fwd", UTC, EPS_FAST) if tc else ("seq", U24, EPS_LIBM)
    whh = w_hh.to(bf16) if tc else w_hh
    xo = _op(ma["x16"] if bfm else ma["x"], precision)
    chk = Worst(name + " fwd")
    for r0, r1 in _slices(B, T, H):
        xs = xo.view(B, T, I)[r0:r1]
        ref = xs @ wih.t() + bias
        bar = n_in * u_in * (xs.abs() @ wih.abs().t()) + U24 * ref.abs() + bias_bar
        chk.add("xg", xg.view(B, T, H3)[r0:r1], ref, bar, row0=r0)
        hin = hst[r0:r1].to(bf16) if tc else hst[r0:r1]
        out = fwd_ref(ref, whh, b_hh[2 * H:], hin, hst[r0:r1], kf, u_rec, eps, dxg=bar)
        rr, zz, nn, gg = save[r0:r1].view(r1 - r0, T, 4, H).unbind(2)
        for label, got in (("r", rr), ("z", zz), ("n", nn), ("gh_n", gg)):
            chk.add(label, got, *out[label if label != "gh_n" else "ghn"], row0=r0)
        chk.add("y", y[r0:r1], *out["y"], row0=r0)
        del xs, ref, bar, out
    chk.done()
    # ---- backward: the BPTT over the whole layer from the kernel's own dy and dgh ----
    _, ba, (dgi, dgh, dh0k) = ev["bwd"]
    _same(name + " BPTT reads the forward's save", ba["save"], save)
    _same(name + " BPTT reads the forward's y", ba["y"], y)
    if dy is not None:
        _same(name + " BPTT dy = the incoming gradient", ba["dy"], dy)
    dhk = ba["dhT"]
    if dhT is not None:
        _same(name + " BPTT dhT = hT's gradient", dhk, dhT)
    else:
        assert dhk is None or not bool(dhk.any()), name + ": nonzero dhT without a gradient for hT"
    assert dgi.dtype == dgh.dtype == (bf16 if tc else f32), (dgi.dtype, dgh.dtype)
    _same(name + " dgi[..., :2H] = dgh[..., :2H]", dgi[..., :2 * H], dgh[..., :2 * H])
    kb = "tc_bwd" if tc else "seq"
    chk = Worst(name + " BPTT")
    stats = [0, 0, 0]
    for r0, r1 in _slices(B, T, H):
        sl = slice(r0, r1)
        ref = bwd_ref(ba["dy"][sl], save[sl], hst[sl], whh, dgh[sl], None if dhk is None else dhk[sl], kb,
                      UTC if tc else U24)
        for label, got in (("dgi", dgi), ("dgh", dgh)):
            g = got[sl].view(r1 - r0, T, 3, H)
            if tc:
                _check_rounded(name, chk, label, g, *ref[label], r0, stats)
            else:
                chk.add(label, g, *ref[label], row0=r0)
        if dh0 is not None:
            chk.add("dh0", dh0[sl], *ref["dh0"], row0=r0)
        del ref
    chk.done()
    if tc:
        _rounding_done(name, stats)
    if dh0 is not None:
        _same(name + " h0's gradient = the BPTT's dh0", dh0, dh0k)
    # ---- the bulk GEMMs and the bias gradients ----
    (_, na, dx), ((_, ta1, _), (_, ta2, _)), ((_, ca1, _), (_, ca2, _)) = ev["nn"], ev["tn"], ev["cs"]
    if bfm:
        gi16, gh16 = (dgi, dgh) if tc else (dgi.to(bf16), dgh.to(bf16))
        _same(name + " dgi16 of dx", na["dy16"], gi16.view(M, H3))
        _same(name + " dgi16 of dW_ih", ta1["dy16"], gi16.view(M, H3))
        _same(name + " dgh16 of dW_hh", ta2["dy16"], gh16.view(M, H3))
        _same(name + " x16 of dW_ih", ta1["x16"], ma["x16"])
    _same(name + " dW_hh's h_{t-1} operand = [h0 | y[:, :-1]]", ta2["x"], hst.reshape(M, H))
    _same(name + " dW_hh operand at t = 0 = h0 (or zeros)", ta2["x"].view(B, T, H)[:, 0], h0v)
    dW_ih, dW_hh, db_ih, db_hh = grads
    gi, gh = _op(dgi, precision).view(M, H3), _op(dgh, precision).view(M, H3)
    hp = _op(hst.reshape(M, H), precision)
    chk = Worst(name + " grads")
    n, u = _gemm(precision, M, I, H3)
    chk.add("dx", dx, gi @ wih, n * u * (gi.abs() @ wih.abs()))
    n, u = _gemm(precision, H3, I, M)
    chk.add("dW_ih", dW_ih, gi.t() @ xo, n * u * (gi.abs().t() @ xo.abs()))
    n, u = _gemm(precision, H3, H, M)
    chk.add("dW_hh", dW_hh, gh.t() @ hp, n * u * (gh.abs().t() @ hp.abs()))
    chk.done()
    assert ca1["x"].dtype == ca2["x"].dtype == dgi.dtype, (name, "bias-gradient rows", ca1["x"].dtype)
    if tc:                            # the vectorised bf16 colsum (16-byte rows), lane order
        assert H3 % 8 == 0
        want_i, want_h = _colsum_lanes(dgi.view(M, H3)), _colsum_lanes(dgh.view(M, H3))
        order = "the lane-order column sum of dgi16 / dgh16"
    else:                             # colsum_kernel over the fp32 rows
        z = torch.zeros(H3, device=DEV)
        want_i, want_h = _colsum_order(dgi.view(M, H3), z).to(DEV), _colsum_order(dgh.view(M, H3), z).to(DEV)
        order = "colsum_kernel's order over the fp32 dgi / dgh"
    _same(name + " db_ih vs " + order, db_ih, want_i)
    _same(name + " db_hh vs " + order, db_hh, want_h)
    return dx.view(B, T, I)


# ---- 1. GRULayer ------------------------------------------------------------------------------------------------------
# (name, B, T, I, H, h0, dhT, precision, expected recurrence): B = 40 runs the tc recurrence in two batch tiles, the
# second of 8 rows; H = 48 is not a tc size (H % 64 != 0), so bf16 mode runs the fp32 recurrence and casts its outputs
LAYER_CASES = [
    ("tc-H1024-B40", 40, 33, 240, 1024, True, True, "bf16", "tc"),
    ("tc-H192-B7", 7, 29, 64, 192, True, False, "bf16", "tc"),
    ("tc-H256-B32", 32, 37, 80, 256, False, False, "bf16", "tc"),
    ("bf16-fp32-recurrence-H48", 5, 21, 24, 48, True, True, "bf16", "seq"),
    ("fp32-H100", 6, 19, 40, 100, True, True, "fp32", "seq"),
]


@pytest.mark.parametrize("name,B,T,I,H,with_h0,with_dhT,precision,rec", LAYER_CASES, ids=[c[0] for c in LAYER_CASES])
def test_gru_layer_teacher_forced(name, B, T, I, H, with_h0, with_dhT, precision, rec, monkeypatch):
    from edgedict_b200 import functional as Fn
    gen = torch.Generator(device=DEV).manual_seed(7 * H + B + T)
    k = 1 / math.sqrt(H)
    w_ih, w_hh = (((torch.rand(3 * H, n, device=DEV, generator=gen) * 2 - 1) * k).requires_grad_(True) for n in (I, H))
    b_ih, b_hh = (((torch.rand(3 * H, device=DEV, generator=gen) * 2 - 1) * k).requires_grad_(True) for _ in range(2))
    x = (torch.randn(B, T, I, device=DEV, generator=gen) * _ragged(B, T, gen)).requires_grad_(True)
    h0 = (torch.randn(B, H, device=DEV, generator=gen) * 0.5).requires_grad_(True) if with_h0 else None
    dhT = torch.randn(B, H, device=DEV, generator=gen) * 0.5 if with_dhT else None
    dy = torch.randn(B, T, H, device=DEV, generator=gen) * _ragged(B, T, gen)
    tap = Tap(monkeypatch)
    y, hT = Fn.GRULayer.apply(x, h0, w_ih, w_hh, b_ih, b_hh, precision)
    torch.autograd.backward([y, hT] if with_dhT else [y], [dy, dhT] if with_dhT else [dy])
    torch.cuda.synchronize()
    ev = _layer_events(tap, 1)[0]
    assert ev["rec"] == rec, (name, ev["rec"])
    _same(name + " output = the recurrence's y", y.detach(), ev["fwd"][2][0])
    dx = check_gru_layer(name, ev, x.detach(), w_ih, w_hh, b_ih, b_hh, precision,
                         (w_ih.grad, w_hh.grad, b_ih.grad, b_hh.grad), h0=None if h0 is None else h0.detach(),
                         dh0=None if h0 is None else h0.grad, dhT=dhT, dy=dy)
    _same(name + " x's gradient = the dgrad GEMM", x.grad, dx)


# ---- 2. Encoder(module=ResLayerNormGRU) -------------------------------------------------------------------------------
def _gru_encoder(I, H, L, P, red, precision, seed):
    from edgedict_b200.rnnt.models import Encoder, ResLayerNormGRU
    torch.manual_seed(seed)
    enc = Encoder(I, H, L, 0.0, P, module=ResLayerNormGRU, time_reductions=list(red)).cuda()
    with torch.no_grad():                 # gamma = 1, beta = 0 would hide a dropped or swapped LayerNorm parameter
        for ln in [enc.norm] + [post[0] for post in enc.lstm.projs]:
            ln.weight.uniform_(0.5, 1.5)
            ln.bias.normal_(0.0, 0.1)
    for m in enc.modules():
        m.precision = precision
    return enc


def _check_ln_fwd(nm, la, lo, z, ln):
    """LayerNorm forward of z from its captured call (arguments la, outputs lo): mean, rstd and the output
    teacher-forced from the saved statistics."""
    out, _, mean, rstd = lo
    H = z.shape[-1]
    assert la["eps"] == ln.eps
    _same(nm + " LayerNorm gamma", la["gamma"], ln.weight.detach())
    _same(nm + " LayerNorm beta", la["beta"], ln.bias.detach())
    mu, bar_mu, rs, bar_rs, tf, bar_tf, _, _ = _ln_ref(z.reshape(-1, H), mean, rstd, ln.weight.detach(),
                                                       ln.bias.detach(), ln.eps, H)
    chk = Worst(nm + " LayerNorm")
    chk.add("mean", mean, mu, bar_mu)
    chk.add("rstd", rstd, rs, bar_rs)
    chk.add("out", out.reshape(-1, H), tf, bar_tf)
    chk.done()
    return out


def _check_ln_bwd(nm, la, lo, z, gz, ln, dz_ret=False):
    """LayerNorm backward from its captured call: dz teacher-forced from the incoming gradient gz and the saved
    statistics, dgamma within its bar, dbeta bitwise in layernorm_param_grad_kernel's order."""
    (_, _, mean, rstd), (lb_args, (dz, dgam, dbet)) = lo, la
    H = z.shape[-1]
    _same(nm + " LayerNorm bwd reads the saved mean", lb_args["mean"], mean)
    _same(nm + " LayerNorm bwd reads the saved rstd", lb_args["rstd"], rstd)
    _same(nm + " LayerNorm bwd incoming gradient", lb_args["dy"], gz)
    ref, bar, _, dg, bar_dg = ln_bwd_ref(z.reshape(-1, H), mean, rstd, gz.reshape(-1, H), ln.weight.detach())
    chk = Worst(nm + " LayerNorm bwd")
    chk.add("dz", dz.reshape(-1, H), ref, bar)
    chk.add("dgamma", ln.weight.grad, dg, bar_dg)
    chk.done()
    _same(nm + " dbeta vs the parameter pass's order", ln.bias.grad.cpu(),
          torch.from_numpy(_dbeta_order(gz.reshape(-1, H), H)))
    return dz


def _check_linear(nm, fwd, bwd, x, w, b, dy, precision):
    """Linear y = x W^T + b (captured mm_nt) and its backward (captured mm_nn, mm_tn, colsum; W / b's gradients):
    per element against fp64 with the plans' bars, db bitwise in colsum_kernel's order over the fp32 dy."""
    (_, fa, y), ((_, na, dx), (_, ta, _), (_, ca, _)) = fwd, bwd
    M, K = x.shape
    N = w.shape[0]
    _same(nm + " operand = its input", fa["x"], x)
    _same(nm + " dy = its incoming gradient", na["dy"], dy)
    _same(nm + " dW's dy", ta["dy"], dy)
    _same(nm + " db's rows", ca["x"], dy)
    if precision == "bf16":
        _same(nm + " x16 = bf16_rn(x)", fa["x16"], x.to(bf16))
        _same(nm + " dy16 of dx = bf16_rn(dy)", na["dy16"], dy.to(bf16))
        _same(nm + " dy16 of dW = bf16_rn(dy)", ta["dy16"], dy.to(bf16))
        _same(nm + " x16 of dW", ta["x16"], x.to(bf16))
    xo, wo, go = _op(x, precision), _op(w.detach(), precision), _op(dy, precision)
    chk = Worst(nm)
    ref = xo @ wo.t() + b.detach().double()
    n, u = _gemm(precision, M, N, K)
    chk.add("out", y, ref, n * u * (xo.abs() @ wo.abs().t()) + U24 * ref.abs())
    n, u = _gemm(precision, M, K, N)
    chk.add("dx", dx, go @ wo, n * u * (go.abs() @ wo.abs()))
    n, u = _gemm(precision, N, K, M)
    chk.add("dW", w.grad, go.t() @ xo, n * u * (go.abs().t() @ xo.abs()))
    chk.done()
    _same(nm + " db vs colsum_kernel's order over dy", b.grad, _colsum_order(dy, torch.zeros(N, device=DEV)).to(DEV))
    return y, dx


def _tr_fwd(x):
    B, T, H = x.shape
    xp = torch.cat([x, torch.zeros(B, 1, H, device=x.device)], 1) if T % 2 else x
    return (xp[:, 0::2] + xp[:, 1::2]) * 0.5


@torch.no_grad()
def check_encoder(name, enc, x, xgrad, out, dout, tap, precision):
    """Every layer of Encoder(module=ResLayerNormGRU), forward then backward, from the captured calls."""
    gru = enc.lstm
    L = len(gru.lstms)
    red = [any(type(m).__name__ == "TimeReduction" for m in list(post)[1:]) for post in gru.projs]
    lnf, lnb = tap.of("layernorm_fwd"), tap.of("layernorm_bwd")
    trf, trb = tap.of("time_reduce_fwd"), tap.of("time_reduce_bwd")
    mm_nt, mm_nn, mm_tn, cs = tap.of("mm_nt"), tap.of("mm_nn"), tap.of("mm_tn"), tap.of("colsum")
    assert len(lnf) == len(lnb) == L + 1 and len(trf) == len(trb) == sum(red)
    assert len(mm_nt) == len(mm_nn) == L + 1 and len(mm_tn) == len(cs) == 2 * L + 1
    ev = _layer_events(tap, L, linear_first=1)
    B = x.shape[0]
    # forward
    _same(name + " input LayerNorm's operand", lnf[0][1]["x"], x)
    assert lnf[0][1]["res"] is None
    cur = _check_ln_fwd(name + " input", lnf[0][1], lnf[0][2], x, enc.norm)
    ys, zs, ins, tri = [], [], [], iter(trf)
    for i in range(L):
        nm = "%s layer %d" % (name, i)
        ins.append(cur)
        y = ev[i]["fwd"][2][0]
        la, lo = lnf[i + 1][1], lnf[i + 1][2]
        _same(nm + " LayerNorm input = the GRU output", la["x"], y)
        if i == 0:
            assert la["res"] is None, nm + ": a residual at layer 0"
            z = y
        else:
            assert la["res"] is not None, nm + ": the residual is missing"
            _same(nm + " LayerNorm residual = the layer's input", la["res"], cur)
            z = y + cur                                    # torch fp32: exactly the kernel's add
        ys.append(y)
        zs.append(z)
        cur = _check_ln_fwd(nm, la, lo, z, gru.projs[i][0])
        if red[i]:
            _, ta, (t2, _) = next(tri)
            _same(nm + " TimeReduction input", ta["x"], cur)
            _same(nm + " TimeReduction = (z[2t] + z[2t+1]) / 2 with a zero pad", t2, _tr_fwd(cur))
            cur = t2
    # backward: the proj Linear, then the layers from the top down
    P, H = enc.proj.weight.shape
    Tl = cur.shape[1]
    proj_out, g = _check_linear(name + " proj", mm_nt[L], (mm_nn[0], mm_tn[0], cs[0]), cur.reshape(-1, H),
                                enc.proj.weight, enc.proj.bias, dout.reshape(-1, P), precision)
    _same(name + " output = proj", out, proj_out.view(B, Tl, P))
    g = g.view(B, Tl, H)
    tri = iter(trb)                                        # recorded top-down
    for i in range(L - 1, -1, -1):
        nm = "%s layer %d" % (name, i)
        k = L - 1 - i
        if red[i]:
            _, ta, dxr = next(tri)
            _same(nm + " TimeReduction bwd incoming gradient", ta["dy"], g)
            Ti = ys[i].shape[1]
            _same(nm + " TimeReduction bwd = 0.5 dy, repeated", dxr, (0.5 * g).repeat_interleave(2, dim=1)[:, :Ti])
            g = dxr
        dz = _check_ln_bwd(nm, (lnb[k][1], lnb[k][2]), lnf[i + 1][2], zs[i], g, gru.projs[i][0])
        cell = gru.lstms[i]
        dx = check_gru_layer(nm, ev[i], ins[i], cell.weight_ih_l0, cell.weight_hh_l0, cell.bias_ih_l0,
                             cell.bias_hh_l0, precision, (cell.weight_ih_l0.grad, cell.weight_hh_l0.grad,
                                                          cell.bias_ih_l0.grad, cell.bias_hh_l0.grad), dy=dz)
        g = dx + dz if i else dx                           # the gradient of the layer's input: dgrad + residual
        torch.cuda.empty_cache()
    dz0 = _check_ln_bwd(name + " input", (lnb[L][1], lnb[L][2]), lnf[0][2], x, g, enc.norm)
    _same(name + " x's gradient = the input LayerNorm's dz", xgrad, dz0)


# (name, B, T, I, H, L, P, time-reduced layers, precision, expected recurrence): the E6D2 CTCEncoder encoder at one and
# two tc batch tiles (odd T, odd T' = 101 after the reduction); the tiny stack in bf16 mode on the fp32 recurrence and in
# fp32 mode
STACK_CASES = [
    ("E6D2-B32", 32, 201, 240, 1024, 6, 640, (1,), "bf16", "tc"),
    ("E6D2-B40", 40, 201, 240, 1024, 6, 640, (1,), "bf16", "tc"),
    ("tiny-bf16-fp32-recurrence", 5, 23, 24, 48, 3, 32, (1,), "bf16", "seq"),
    ("tiny-fp32", 5, 23, 24, 48, 3, 32, (1,), "fp32", "seq"),
]


@pytest.mark.parametrize("name,B,T,I,H,L,P,red,precision,rec", STACK_CASES, ids=[c[0] for c in STACK_CASES])
def test_gru_encoder_teacher_forced(name, B, T, I, H, L, P, red, precision, rec, monkeypatch):
    seed = B * 100 + T + H
    enc = _gru_encoder(I, H, L, P, red, precision, seed)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, T, I, device=DEV, generator=gen) * _ragged(B, T, gen)
    tap = Tap(monkeypatch)
    xi = x.clone().requires_grad_(True)
    out, _ = enc(xi)
    dout = torch.randn(out.shape, device=DEV, generator=gen)
    out.backward(dout)
    torch.cuda.synchronize()
    recs = {e for e, _, _ in tap.of("gru_tc_fwd", "gru_seq_fwd")}
    assert recs == {"gru_%s_fwd" % rec}, (name, recs)
    check_encoder(name, enc, x, xi.grad, out.detach(), dout, tap, precision)


# ---- 3. CTCEncoder head and loss --------------------------------------------------------------------------------------
def _vs(name, label, got, want, bar, rel=False):
    """Worst err/bar of got against want (NaN where want is NaN, equal infinities, finite elsewhere), printed with its
    index; returns the ratio."""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (name, label, got.shape, want.shape)
    assert torch.equal(torch.isnan(got), torch.isnan(want)), "%s %s: NaN pattern" % (name, label)
    inf = torch.isinf(want)
    assert torch.equal(got[inf], want[inf]), "%s %s: infinities" % (name, label)
    fin = torch.isfinite(want)
    assert bool(torch.isfinite(got[fin]).all()), "%s %s: non-finite where the reference is finite" % (name, label)
    err = torch.where(fin, got - want, torch.zeros_like(got)).abs()
    if rel:
        err = err / want.abs().clamp_min(1e-30)
    ratio, idx, e, b = worst(err, torch.full_like(err, bar))
    print("  %-40s %-12s worst err/bar %.3g at %s (err %.3g, bar %.3g)" % (name, label, ratio, idx, e, b))
    return ratio


def _ctc_problem(B, Tp, V, S, seed):
    """Ragged input lengths (the first utterance full) and target lengths, padded labels in [1, V) (blank 0), every
    utterance feasible."""
    g = torch.Generator().manual_seed(seed)
    il = torch.tensor([Tp] + [int(v) for v in torch.randint(Tp // 2, Tp + 1, (B - 1,), generator=g)])
    tl = torch.tensor([S] + [int(v) for v in torch.randint(0, S + 1, (B - 1,), generator=g)])
    tl = torch.minimum(tl, il // 2)
    ys = torch.randint(1, V, (B, S), generator=g)
    return ys, il, tl


# (name, model config, precision, B, T): V = 1024 at the E6D2 encoder, bf16; the tiny model in fp32 mode
HEAD_CASES = [("E6D2-bf16-B8", E6D2, "bf16", 8, 201, 40), ("tiny-fp32", CTC_TINY, "fp32", 4, 23, 5)]


@pytest.mark.parametrize("name,cfg,precision,B,T,S", HEAD_CASES, ids=[c[0] for c in HEAD_CASES])
def test_ctc_head_and_loss_teacher_forced(name, cfg, precision, B, T, S, monkeypatch):
    import torch.nn.functional as F
    from edgedict_b200.ctc import CTCLoss
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(B + T)
    m = CTCEncoder(**cfg).cuda().set_precision(precision)
    gen = torch.Generator(device=DEV).manual_seed(B + T)
    xs = torch.randn(B, T, cfg["input_size"], device=DEV, generator=gen) * _ragged(B, T, gen)
    tap = Tap(monkeypatch)
    lp = m(xs)
    Tp, V = lp.shape[1], lp.shape[2]
    ys, il, tl = _ctc_problem(B, Tp, V, S, B * T)
    loss = CTCLoss()(lp.transpose(0, 1), ys, il, tl)
    loss.backward()
    torch.cuda.synchronize()
    lin = m.tovocab[0]
    P = lin.weight.shape[1]
    M = B * Tp
    (_, la, logits), = tap.of("mm_nt")[-1:]
    enc = la["x"]
    assert enc.shape == (M, P)
    # log-softmax forward, per element from the engine's own logits (test_gpu_ctc.py's bar)
    (_, sa, y), = tap.of("log_softmax_fwd")
    _same(name + " log-softmax input = the logits", sa["x"].reshape(M, V), logits)
    _same(name + " log-probs = the log-softmax output", lp.detach(), y.view(B, Tp, V))
    x64 = logits.double()
    mx = x64.max(-1, keepdim=True).values
    ls = torch.log(torch.exp(x64 - mx).sum(-1, keepdim=True))
    y64 = x64 - mx - ls
    chk = Worst(name + " head")
    chk.add("log_probs", y.reshape(M, V), y64, 2 * U24 * ((x64 - mx).abs() + (V + 2) + 2 * ls.abs() + y64.abs()))
    # the loss: costs and d log_probs against F.ctc_loss in fp64 on the engine's own log-probs
    (_, fa, (costs, _)), = tap.of("ctc_loss_fwd")
    (_, ga, grad), = tap.of("ctc_loss_bwd")
    _same(name + " CTC log_probs = the (T, N, V) view of the log-probs", fa["lp"], y.view(B, Tp, V).transpose(0, 1))
    lr = y.view(B, Tp, V).transpose(0, 1).double().cpu().requires_grad_(True)
    ref_costs = F.ctc_loss(lr, ys, il, tl, reduction="none")
    ref = F.ctc_loss(lr, ys, il, tl, reduction="mean")
    ref.backward()
    worst_cost = max(_vs(name, "costs (rel)", costs, ref_costs, COST_REL, rel=True),
                     _vs(name, "loss (rel)", loss.reshape(()), ref, COST_REL, rel=True))
    worst_grad = _vs(name, "d log_probs", grad, lr.grad, GRAD_ABS)
    assert worst_cost <= 1.0 and worst_grad <= 1.0, (name, worst_cost, worst_grad)
    # log-softmax backward from the engine's own g and y
    (_, sb, dl), = tap.of("log_softmax_bwd")
    gin = grad.transpose(0, 1)
    _same(name + " log-softmax backward's g = the CTC gradient", sb["dy"], gin.contiguous())
    _same(name + " log-softmax backward's y", sb["y"], y.view(B, Tp, V))
    g64, ey = gin.double(), torch.exp(y.view(B, Tp, V).double())
    dl64 = g64 - ey * g64.sum(-1, keepdim=True)
    chk.add("dlogits", dl, dl64, 2 * U24 * (g64.abs() + dl64.abs() + ey * (V + 3) * g64.abs().sum(-1, keepdim=True)))
    chk.done()
    # the tovocab Linear: logits, dx, dW per element, db bitwise
    _check_linear(name + " tovocab", tap.of("mm_nt")[-1], (tap.of("mm_nn")[0], tap.of("mm_tn")[0], tap.of("colsum")[0]),
                  enc, lin.weight, lin.bias, dl.view(M, V), precision)


# ---- 4. the CTC lattice with four states per thread -------------------------------------------------------------------
def _lattice4_problem(N, T, V, S, blank, seed, tl, il, repeats):
    """log_probs (T, N, V), padded labels without the blank, and adjacent repeats planted at the label indices in
    `repeats` (utterance 0): their states 2j + 1 lie in the third and fourth slots of ctc_lattice_kernel<4>."""
    g = torch.Generator().manual_seed(seed)
    lp = (torch.randn(T, N, V, generator=g) * 2).log_softmax(-1)
    lab = torch.randint(0, V - 1, (N, S), generator=g)
    lab = lab + (lab >= blank).long()
    for j in repeats:
        lab[0, j + 1] = lab[0, j]
    return lp, lab, torch.tensor(il), torch.tensor(tl)


def _threads(S):
    """ctc_lattice_kernel's CTA size: four states per thread above 1024 states, rounded up to whole warps."""
    L = 2 * S + 1
    slots = 2 if L <= 1024 else 4
    return ((L + slots - 1) // slots + 31) // 32 * 32


# (name, N, T, V, S, blank, layout, target lengths, input lengths, planted repeats): 1025 states (288 threads: slots 2
# and 3 hold s >= 576), and 2047 states (512 threads: s >= 1024) with concatenated targets, blank V - 1, ragged lengths
# and one infeasible utterance (1023 labels in 900 frames)
LATTICE4_CASES = [
    ("S512-T1100", 3, 1100, 64, 512, 0, "padded", [512, 400, 512], [1100, 1100, 900], [300, 301, 450, 500]),
    ("S1023-T2100-concat-blank-last", 4, 2100, 48, 1023, 47, "concat", [1023, 700, 1023, 600],
     [2100, 1500, 900, 2000], [520, 521, 700, 900, 1000]),
]


@pytest.mark.parametrize("name,N,T,V,S,blank,layout,tl,il,repeats", LATTICE4_CASES,
                         ids=[c[0] for c in LATTICE4_CASES])
def test_ctc_lattice_four_states_per_thread(name, N, T, V, S, blank, layout, tl, il, repeats):
    assert 2 * S + 1 > 1024
    nt = _threads(S)
    assert 2 * repeats[0] + 1 >= 2 * nt, "the planted repeats must lie in the third or fourth slot"
    lp, lab, il, tl = _lattice4_problem(N, T, V, S, blank, N * T + S, tl, il, repeats)
    targets = torch.cat([lab[b, :int(n)] for b, n in enumerate(tl)]) if layout == "concat" else lab
    g = torch.Generator().manual_seed(S)
    worst_c = worst_g = 0.0
    for reduction in ("none", "mean", "sum"):
        for zero_inf in (False, True):
            go = torch.rand(N, generator=g) + 0.5 if reduction == "none" else torch.tensor(1.3)
            got, dg, ref, dr = _run(lp, targets, il, tl, blank, reduction, zero_inf, go)
            tag = "%s zero_inf=%d" % (reduction, zero_inf)
            worst_c = max(worst_c, _vs(name, tag + " costs", got, ref, COST_REL, rel=True))
            worst_g = max(worst_g, _vs(name, tag + " grad", dg, dr, GRAD_ABS))
    assert worst_c <= 1.0 and worst_g <= 1.0, (name, worst_c, worst_g)
