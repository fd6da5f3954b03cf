"""Teacher-forced fp64 parity of the composed bf16 training step, per layer and per element: the encoder stack
(functional.LSTMStack: the forward wavefront, the serial backward and the chunked backward `_backward_wave`), the bf16
LSTMLayer and the bf16 JointLoss backward (`_joint_bwd`, from the engine's own dlogits and saved hidden).

The kernels are pinned one by one by the kernel-level files; this file pins the code that composes them: the chunk-major
layouts, the bias of the input GEMM, the h_{t-1} / c_{t-1} carried across chunks and BPTT groups, the h_{t-1} operand of
dW_hh, TimeReduction on a ragged last chunk, the LayerNorm split into its dz and parameter passes, the dgrad GEMM
accumulated onto the residual gradient, the weight and bias gradients.  Each layer is checked from the engine's own inputs
to that layer, so errors do not compound through the stack and a failure names one (batch row, step, unit):

  forward   the saved x16[l], W_ih and b_ih + b_hh give xg in fp64 with the bar of its GEMM (K = I, u = 2^-23 per add, one
            rounding of the bias add), passed to the recurrence reference (`fwd_ref`) as `dpre_in`; h_{t-1} is the bf16
            operand the kernel multiplied (the c4 forward saves it, the tc forward's y16 shifted), c_{t-1} the saved cell
            state shifted -- over the whole layer, so every chunk boundary is an ordinary step.  LayerNorm + residual
            teacher-forced from the saved mean / rstd (the bars of test_gpu_glue_fp64.py), the mean and rstd themselves
            against fp64, TimeReduction propagated: (z[2t] + z[2t+1]) / 2 with the two bars and one rounding.
  backward  from the top layer down, with the backward hook `LSTMStack.collect_bwd` (the BPTT's input dy, its bf16 dG and
            d xs[l] after the dgrad GEMM, and the LayerNorm's incoming gradient): TimeReduction backward bitwise
            against its restatement (0.5 dy, repeated) and the asserted schedule and BPTT entry; the LayerNorm dz
            teacher-forced from the incoming gradient; the BPTT over the whole layer (`bwd_ref` with the hook's dy and
            dg16), dg16 within the bar plus half a bf16 ulp and its share of differing bits below FRAC_DIFF;
            d xs[l] = dy + dg16 bf16(W_ih), dW_ih = dg16^T x16, dW_hh = dg16^T h_{t-1}: fp64 with n_add u |A| |B| bars
            (n_add from the GEMM's plan, split-K included); dgamma barred.
  bitwise   everything the code only gathers, copies, casts or adds in a fixed order: y16 (the h_{t-1} operand),
            hT / cT at every chunk's last step, x16[l+1] = bf16_rn(xs[l+1]), the output and `collect`, b_ih = b_hh =
            the column sum of dg16 in eb_colsum's lane order over the CHUNK-MAJOR rows, dbeta in the LayerNorm parameter
            pass's order over the chunk-major rows.
  joint     the engine's bf16 dlogits against the fp64 C oracle (the bars of test_gpu_joint_loss_fused.py), then every
            gradient of `_joint_bwd` teacher-forced from them and the saved bf16 hidden.

References are built one layer at a time and in slices of batch rows (teacher forcing makes the rows independent), so
the peak fp64 memory stays near a few GB at the bench shape.  Every check prints its worst err/bar (pytest -s); DESIGN.md
section 2 records the measured figures.  The file runs in about 35 s on an H100."""
import math

import pytest
import torch

from tests.test_gpu_gemm_fp64 import CORESIDENT, _plan, _same
from tests.test_gpu_gemm_fp64 import _n_add as gemm_n_add
from tests.test_gpu_glue_fp64 import _colsum_order, _dbeta_order, _ln_ref, ln_bwd_ref
from tests.test_gpu_lstm_recurrence_fp64 import (EPS_FAST, EPS_LIBM, FRAC_DIFF, TINY, U24, UTC, _bf16_ulp, _n_add,
                                                 bwd_ref, fwd_ref, tc_cluster_size, worst)

pytestmark = pytest.mark.gpu

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
SLICE_BYTES = 2 ** 27       # fp64 bytes of one [rows, T, 4H] reference tensor in a batch slice


# ---- bookkeeping ------------------------------------------------------------------------------------------------------
class Worst:
    """Worst err/bar per label over the batch slices a reference is built in; `done` prints each with the index where it
    occurs ((row, step, unit) or (row, step, gate, unit)) and asserts them all."""

    def __init__(self, name):
        self.name, self.items = name, {}

    def add(self, label, got, ref, bar, row0=0):
        got = got.double()
        assert torch.isfinite(got).all(), "%s %s: non-finite output" % (self.name, label)
        ratio, idx, e, b = worst((got - ref).abs(), bar + TINY)
        cur = self.items.get(label)
        if cur is None or ratio > cur[0]:
            self.items[label] = (ratio, (idx[0] + row0,) + idx[1:], e, b, float(got[idx]), float(ref[idx]))

    def done(self):
        bad = []
        for label, (ratio, idx, e, b, g, r) in self.items.items():
            print("  %-40s %-8s worst err/bar %.3g at %s (err %.3g, bar %.3g)" % (self.name, label, ratio, idx, e, b))
            if ratio > 1.0:
                bad.append("%s: err/bar %.3g at %s, engine %r, fp64 %r" % (label, ratio, idx, g, r))
        assert not bad, self.name + ": " + "; ".join(bad)


def _slices(B, T, H):
    bs = max(1, SLICE_BYTES // (T * 4 * H * 8))
    return [(r, min(B, r + bs)) for r in range(0, B, bs)]


def _shift(first, seq):
    """[first, seq[:, 0], ..., seq[:, T-2]] along t."""
    return torch.cat([first[:, None].to(seq.dtype), seq[:, :-1]], 1)


def _colsum_lanes(x16):
    """eb_colsum of bf16 rows in its order (test_gpu_colsum_order.py), in torch fp32 on the device: lane k adds rows k,
    k + 512, ... in order, then a tree at strides 256 ... 1."""
    rows, N = x16.shape
    lanes = torch.zeros(512, N, device=x16.device)
    for r0 in range(0, rows, 512):
        blk = x16[r0:r0 + 512].float()
        lanes[:blk.shape[0]] += blk
    st = 256
    while st:
        lanes[:st] += lanes[st:2 * st]
        st //= 2
    return lanes[0]


# ---- one LSTM layer, teacher-forced -----------------------------------------------------------------------------------
def check_lstm_fwd(name, x16, w_ih, w_hh, b_ih, b_hh, hin, cin, gates, cseq, y, kernel, in_flags=0):
    """x16 [B,T,I] bf16 the input the engine multiplied; hin / cin [B,T,H] the h_{t-1} (bf16, or fp32 for the fp32
    recurrence) and c_{t-1} of every step; gates / cseq / y the engine's.  kernel: "c4_fwd", "tc_fwd" or "seq"."""
    B, T, I = x16.shape
    H = w_hh.shape[1]
    wih = w_ih.to(bf16).double()
    whh = w_hh if kernel == "seq" else w_hh.to(bf16)
    bias = (b_ih + b_hh).double()                       # the fp32 sum the engine adds in the GEMM's epilogue
    _, ks = _plan(B * T, 4 * H, I, flags=in_flags)
    n_in = gemm_n_add(I, ks)
    u_rec, eps = (U24, EPS_LIBM) if kernel == "seq" else (UTC, EPS_FAST)
    chk = Worst(name + " fwd")
    for r0, r1 in _slices(B, T, H):
        xs = x16[r0:r1].double()
        s = xs @ wih.t()
        xg = s + bias
        dxg = n_in * UTC * (xs.abs() @ wih.abs().t()) + U24 * xg.abs()
        ref = fwd_ref(xg, whh, hin[r0:r1], cin[r0:r1], _n_add(kernel, H), u_rec, eps, dpre_in=dxg)
        chk.add("gates", gates[r0:r1].view(r1 - r0, T, 4, H), *ref["gates"], row0=r0)
        chk.add("c", cseq[r0:r1], *ref["c"], row0=r0)
        chk.add("y", y[r0:r1], *ref["y"], row0=r0)
        del s, xg, dxg, ref
    chk.done()


def check_lstm_bwd(name, dy, dgq, gates, cseq, c0, w_hh, dhT, dcT, kernel, n_add, bf16_out=True):
    """The BPTT over the whole layer from the engine's dy and exchanged dG (dg16, or the fp32 dgates); returns the
    references of dh0 and dc0 as (value, bar) pairs [B,H]."""
    B, T, H = dy.shape
    w = w_hh if kernel == "seq" else w_hh.to(bf16)
    u_rec, eps = (U24, EPS_LIBM) if kernel == "seq" else (UTC, EPS_FAST)
    chk = Worst(name + " BPTT")
    outside = ndiff = 0
    dh0, dc0 = [], []
    for r0, r1 in _slices(B, T, H):
        sl = slice(r0, r1)
        ref = bwd_ref(dy[sl], gates[sl], cseq[sl], None if c0 is None else c0[sl], w, dgq[sl],
                      None if dhT is None else dhT[sl], None if dcT is None else dcT[sl], n_add, u_rec, eps)
        val, bar = ref["dG"]
        dg = dgq[sl].view(r1 - r0, T, 4, H)
        if bf16_out:
            lo, hi = (val - bar).to(f32).to(bf16).double(), (val + bar).to(f32).to(bf16).double()
            d = dg.double()
            outside += int(((d < lo) | (d > hi)).sum())
            ndiff += int((dg != val.to(f32).to(bf16)).sum())
            bar = bar + 0.5 * _bf16_ulp(val.abs() + bar)
        chk.add("dG", dg, val, bar, row0=r0)
        dh0.append(ref["dh0"])
        dc0.append(ref["dc0"])
        del ref, val, bar
    if bf16_out:
        frac = ndiff / dgq.numel()
        print("  %-40s dg16 bits != bf16_rn(dG_ref): %.4f of the elements (bar %.3g), %d outside the rounded bar"
              % (name, frac, FRAC_DIFF, outside))
        assert outside == 0, "%s: %d dg16 elements are not a rounding of a value within the bar" % (name, outside)
        assert frac <= FRAC_DIFF, "%s: %.4f of dg16 differs from bf16_rn(dG_ref)" % (name, frac)
    chk.done()
    cat = lambda parts, i: torch.cat([p[i] for p in parts], 0)
    return (cat(dh0, 0), cat(dh0, 1)), (cat(dc0, 0), cat(dc0, 1))


def check_lstm_grads(name, dg16, x16, hprev, w_ih, dW_ih, dW_hh, db_ih, db_hh, dg_rows, dy=None, dx=None):
    """dx = [dy +] dg16 bf16(W_ih) per element (dx None: not checked); dW_ih = dg16^T x16 and dW_hh = dg16^T hprev
    against fp64 with the bars of their GEMM plans; b_ih = b_hh = the colsum of dg_rows (dg16 in the engine's row
    order), bitwise.  dg16 / x16 / hprev [B,T,.] bf16."""
    B, T, H4 = dg16.shape
    I = x16.shape[2]
    H = H4 // 4
    M = B * T
    wih = w_ih.to(bf16).double()
    chk = Worst(name + " grads")
    # dx: the encoder's dgrad of layers >= 1 runs FIXED_K or co-resident (one chain over K), the plain product may split
    n_dx = gemm_n_add(H4, 1 if dy is not None else _plan(M, I, H4)[1])
    Sx = torch.zeros(H4, I, dtype=f64, device=DEV)
    Rx = torch.zeros_like(Sx)
    Sh = torch.zeros(H4, H, dtype=f64, device=DEV)
    Rh = torch.zeros_like(Sh)
    for r0, r1 in _slices(B, T, H):
        g = dg16[r0:r1].reshape(-1, H4).double()
        if dx is not None:
            p = g @ wih
            bar = n_dx * UTC * (g.abs() @ wih.abs())
            if dy is not None:
                p = p + dy[r0:r1].reshape(-1, I).double()
                bar = bar + U24 * p.abs()
            chk.add("dx", dx[r0:r1], p.view(r1 - r0, T, I), bar.view(r1 - r0, T, I), row0=r0)
            del p, bar
        xs = x16[r0:r1].reshape(-1, I).double()
        hp = hprev[r0:r1].reshape(-1, H).double()
        Sx += g.t() @ xs
        Rx += g.abs().t() @ xs.abs()
        Sh += g.t() @ hp
        Rh += g.abs().t() @ hp.abs()
        del g, xs, hp
    _, ks_ih = _plan(H4, I, M)
    _, ks_hh = _plan(H4, H, M)
    chk.add("dW_ih", dW_ih, Sx, gemm_n_add(M, ks_ih) * UTC * Rx)
    chk.add("dW_hh", dW_hh, Sh, gemm_n_add(M, ks_hh) * UTC * Rh)
    chk.done()
    if dg_rows.dtype == bf16:
        want = _colsum_lanes(dg_rows)
    else:                            # the fp32 recurrence's bias gradients sum its fp32 dgates
        want = _colsum_order(dg_rows, torch.zeros(H4, device=DEV)).to(DEV)
    _same(name + " b_ih grad vs the lane-order column sum of dG", db_ih, want)
    _same(name + " b_hh grad vs the lane-order column sum of dG", db_hh, want)


# ---- the encoder stack ------------------------------------------------------------------------------------------------
def _encoder(I, H, L, red, seed):
    from edgedict_b200.rnnt.models import ResLayerNormLSTM
    torch.manual_seed(seed)
    net = ResLayerNormLSTM(I, H, L, time_reductions=list(red)).cuda()
    with torch.no_grad():                  # gamma = 1, beta = 0 would hide a dropped or swapped LayerNorm parameter
        for post in net.projs:
            post[0].weight.uniform_(0.5, 1.5)
            post[0].bias.normal_(0.0, 0.1)
    for m in net.modules():
        m.precision = "bf16"
    params = []
    for cell, post in zip(net.lstms, net.projs):
        params += [cell.weight_ih_l0, cell.weight_hh_l0, cell.bias_ih_l0, cell.bias_hh_l0, post[0].weight, post[0].bias]
    return net, params


def _run_stack(net, params, x, seed, monkeypatch):
    """Forward + backward with both hooks on; returns what the checks read (saves cloned before backward)."""
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    coll, recs, ran = [], [], []
    monkeypatch.setattr(Fn.LSTMStack, "collect", coll)
    monkeypatch.setattr(Fn.LSTMStack, "collect_bwd", recs)
    # which schedule and which BPTT entry the backward takes: the checks name them and pick the BPTT's n_add from them
    for entry in ("lstm_c4_bwd_chunks", "lstm_tc_bwd_chunks", "lstm_tc_bwd", "lstm_c4_bwd"):
        orig = getattr(ops, entry)
        monkeypatch.setattr(ops, entry, lambda *a, _o=orig, _e=entry, **kw: (ran.append(_e), _o(*a, **kw))[1])
    wave = Fn.LSTMStack._backward_wave
    monkeypatch.setattr(Fn.LSTMStack, "_backward_wave", staticmethod(lambda *a: (ran.append("wave"), wave(*a))[1]))
    xi = x.clone().requires_grad_(True)
    out, _ = net(xi)
    gf = out.grad_fn
    assert "LSTMStack" in type(gf).__name__, "the encoder did not take the layer-wavefront path"
    reductions, eps, plan = gf.cfg
    B, T, I0, H, L, C = gf.dims
    sv = list(gf.saved_tensors)[6 * L:]
    hT, cT, sv = sv[0].clone(), sv[1].clone(), sv[2:]
    x16, sv = sv[:L], sv[L:]
    xs, sv = [None] + sv[:L - 1], sv[L - 1:]
    y, y16, gates, cseq, mean, rstd = (sv[i * L:(i + 1) * L] for i in range(6))
    gates = [g.clone() for g in gates]              # the BPTT kernels may write into the saved gates
    saves = dict(x16=[t.clone() for t in x16], xs=[None if t is None else t.clone() for t in xs],
                 y=[t.clone() for t in y], y16=[t.clone() for t in y16], gates=gates,
                 cseq=[t.clone() for t in cseq], mean=[t.clone() for t in mean], rstd=[t.clone() for t in rstd],
                 hT=hT, cT=cT)
    dout = torch.randn(out.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    out.backward(dout)
    torch.cuda.synchronize()
    assert len(recs) == L and len(coll) == L
    return dict(cfg=gf.cfg, dims=gf.dims, c4=gf.c4, out=out.detach(), dout=dout, dx=xi.grad, coll=coll, recs=recs,
                grads=[p.grad.clone() for p in params], ran=ran, **saves)


def _gather(ck, buf):
    return ck.gather(buf if buf.dim() == 2 else buf.view(-1, 1))


@torch.no_grad()
def check_stack(name, net, params, r, bptt):
    """The per-layer forward and backward checks of one LSTMStack run (module docstring)."""
    from edgedict_b200.functional import _Chunks
    reductions, eps, plan = r["cfg"]
    B, T, I0, H, L, C = r["dims"]
    ck = [_Chunks(B, lens) for lens in plan]
    fk = "c4_fwd" if r["c4"] else "tc_fwd"
    print("  %s: %d layers, chunks %s, forward %s, BPTT %s" % (name, L, plan[0], fk, bptt))
    bk, cs = bptt
    n_bwd = _n_add(bk, H, cs)
    _same(name + " output vs collect[L-1]", r["out"], r["coll"][L - 1])
    gin = r["dout"]
    for l in range(L - 1, -1, -1):       # backward order; the forward checks of layer l run first
        k, kn = ck[l], ck[l + 1]
        nm = "%s layer %d" % (name, l)
        w_ih, w_hh, b_ih, b_hh, gamma, beta = params[6 * l:6 * l + 6]
        x16 = _gather(k, r["x16"][l])
        y = _gather(k, r["y"][l])
        y16 = _gather(k, r["y16"][l])
        gates = _gather(k, r["gates"][l])
        cseq = _gather(k, r["cseq"][l])
        zero = torch.zeros(B, H, device=DEV)
        hprev = y16 if r["c4"] else _shift(zero.to(bf16), y16)
        if r["c4"]:
            _same(nm + " hprev16 = [0, bf16_rn(y[:, :-1])]", y16, _shift(zero.to(bf16), y.to(bf16)))
        else:
            _same(nm + " y16 = bf16_rn(y)", y16, y.to(bf16))
        for c in range(C):
            te = k.off[c + 1] - 1
            _same("%s hT[%d] = y at step %d" % (nm, c, te), r["hT"][l, c], y[:, te])
            _same("%s cT[%d] = c at step %d" % (nm, c, te), r["cT"][l, c], cseq[:, te])
        check_lstm_fwd(nm, x16, w_ih, w_hh, b_ih, b_hh, hprev, _shift(zero, cseq), gates, cseq, y, fk,
                       in_flags=CORESIDENT)
        # LayerNorm + residual from the saved statistics, then TimeReduction
        res = _gather(k, r["xs"][l]) if l else None
        z = (y + res if l else y).view(-1, H)
        mean, rstd = _gather(k, r["mean"][l]).view(-1), _gather(k, r["rstd"][l]).view(-1)
        mu, bar_mu, rs, bar_rs, tf, bar_tf, _, _ = _ln_ref(z, mean, rstd, gamma, beta, eps[l], H)
        chk = Worst(nm + " LayerNorm")
        chk.add("mean", mean, mu, bar_mu)
        chk.add("rstd", rstd, rs, bar_rs)
        Tl = y.shape[1]
        tf, bar_tf = tf.view(B, Tl, H), bar_tf.view(B, Tl, H)
        if reductions[l]:
            if Tl % 2:
                pad = torch.zeros(B, 1, H, dtype=f64, device=DEV)
                tf, bar_tf = torch.cat([tf, pad], 1), torch.cat([bar_tf, pad], 1)
            tf = (tf[:, 0::2] + tf[:, 1::2]) * 0.5
            bar_tf = (bar_tf[:, 0::2] + bar_tf[:, 1::2]) * 0.5 * (1 + U24) + U24 * tf.abs()
        xn = r["coll"][l]
        chk.add("xs[l+1]", xn, tf, bar_tf)
        del mu, bar_mu, rs, bar_rs, tf, bar_tf
        chk.done()
        if l + 1 < L:
            _same(nm + " saved xs[l+1] vs collect", _gather(kn, r["xs"][l + 1]), xn)
            _same(nm + " x16[l+1] = bf16_rn(xs[l+1])", _gather(kn, r["x16"][l + 1]), xn.to(bf16))
        # backward: TimeReduction, LayerNorm dz, BPTT, dgrad, weight and bias gradients, LayerNorm parameters
        rec = r["recs"][l]
        gz = gin
        if reductions[l]:
            gz = (0.5 * gin).repeat_interleave(2, dim=1)[:, :Tl]
        _same(nm + " LayerNorm's incoming gradient" + (" = TimeReduction backward" if reductions[l] else ""),
              rec["dln"], gz)
        dz, bar_dz, _, dgam, bar_dgam = ln_bwd_ref(z, mean, rstd, gz.reshape(-1, H), gamma)
        chk = Worst(nm + " LayerNorm bwd")
        chk.add("dz", rec["dy"], dz.view(B, Tl, H), bar_dz.view(B, Tl, H))
        chk.add("dgamma", r["grads"][6 * l + 4], dgam, bar_dgam)
        del dz, bar_dz
        chk.done()
        want_db = torch.from_numpy(_dbeta_order(k.scatter(gz.contiguous()), H))
        _same(nm + " dbeta vs the parameter pass's order over the chunk-major rows", r["grads"][6 * l + 5].cpu(), want_db)
        check_lstm_bwd(nm, rec["dy"], rec["dg16"], gates, cseq, None, w_hh, None, None, bk, n_bwd)
        g = r["grads"]
        dxs, dyres = (rec["dxs"], rec["dy"]) if l else (r["dx"], None)
        check_lstm_grads(nm, rec["dg16"], x16, hprev, w_ih, g[6 * l], g[6 * l + 1], g[6 * l + 2], g[6 * l + 3],
                         k.scatter(rec["dg16"]), dy=dyres, dx=dxs)
        gin = rec["dxs"]
        del x16, y, y16, gates, cseq, z, hprev
        torch.cuda.empty_cache()


def _bptt_of(entry, H):
    """(kernel, cluster size) of the BPTT entry the encoder ran: the K-split c4 kernel (clusters of 16), or the tc kernel
    (one launch over the chunks, or one per chunk) at the cluster size it picks for H."""
    return ("c4_bwd", 16) if entry == "lstm_c4_bwd_chunks" else ("tc_bwd", tc_cluster_size(H))


# (name, B, T, I, H, L, time-reduced layers, WAVEFRONT_CHUNKS, BPTT_GROUP, BPTT_WAVEFRONT, expected C, expected c4,
#  expected backward: "wave" (_backward_wave) or "serial", and the BPTT entry it calls)
STACK_CASES = [
    # the bench encoder: c4 forward, chunked backward in two groups of three chunks (168 x 5 + 160)
    ("E6D2-bench", 32, 1000, 240, 1024, 6, (1,), 6, 3, True, 6, True, "wave", "lstm_c4_bwd_chunks"),
    ("E6D2-bench-serial", 32, 1000, 240, 1024, 6, (1,), 6, 3, False, 6, True, "serial", "lstm_c4_bwd_chunks"),
    # ragged last chunk of 5 frames: TimeReduction pads one; groups of one and two chunks
    ("ragged-group1", 5, 101, 80, 1024, 3, (1,), 6, 1, True, 4, True, "wave", "lstm_c4_bwd_chunks"),
    ("ragged-group2", 5, 101, 80, 1024, 3, (1,), 6, 2, True, 4, True, "wave", "lstm_c4_bwd_chunks"),
    # C > 8: c4 forward, per-chunk lstm_tc_bwd
    ("C10-per-chunk", 8, 400, 64, 1024, 2, (0,), 10, 3, True, 10, True, "serial", "lstm_tc_bwd"),
    # c4 forward, lstm_tc_bwd_chunks
    ("H256-tc-chunks", 32, 400, 64, 256, 3, (0, 2), 6, 3, True, 6, True, "serial", "lstm_tc_bwd_chunks"),
    ("H512-tc-chunks", 40, 400, 64, 512, 3, (0, 2), 6, 3, True, 6, True, "serial", "lstm_tc_bwd_chunks"),
    # tc forward, per-chunk BPTT with the h_{t-1} operand shifted across chunks in Python
    ("H128-tc", 7, 64, 40, 128, 3, (), 2, 3, True, 2, False, "serial", "lstm_tc_bwd"),
]


@pytest.mark.parametrize("name,B,T,I,H,L,red,chunks,group,wave,C,c4,sched,entry", STACK_CASES,
                         ids=[c[0] for c in STACK_CASES])
def test_lstm_stack_teacher_forced(name, B, T, I, H, L, red, chunks, group, wave, C, c4, sched, entry, monkeypatch):
    from edgedict_b200 import functional as Fn
    monkeypatch.setattr(Fn, "WAVEFRONT_CHUNKS", chunks)
    monkeypatch.setattr(Fn, "BPTT_GROUP", group)
    monkeypatch.setattr(Fn, "BPTT_WAVEFRONT", wave)
    seed = B * 1000 + T + H
    net, params = _encoder(I, H, L, red, seed)
    x = torch.randn(B, T, I, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    r = _run_stack(net, params, x, seed + 1, monkeypatch)
    assert (r["dims"][5], r["c4"]) == (C, c4), (name, r["dims"], r["c4"])
    if name == "ragged-group1":
        assert r["cfg"][2][0] == [32, 32, 32, 5]
    ran = r["ran"]
    assert ("wave" in ran) == (sched == "wave"), (name, "backward schedule", ran)
    assert set(ran) - {"wave"} == {entry}, (name, "BPTT entries", sorted(set(ran)))
    check_stack(name, net, params, r, _bptt_of(entry, H))


def test_collect_bwd_leaves_the_gradients_unchanged(monkeypatch):
    """The backward hook only copies: with it on, the output, dx and every parameter gradient are the same bits as with
    it off, under both backward schedules."""
    from edgedict_b200 import functional as Fn
    B, T, I, H, L = 5, 101, 80, 1024, 3
    net, params = _encoder(I, H, L, (1,), 17)
    x = torch.randn(B, T, I, device=DEV, generator=torch.Generator(device=DEV).manual_seed(17))
    dout = None
    for wave in (True, False):
        monkeypatch.setattr(Fn, "BPTT_WAVEFRONT", wave)
        res = []
        for hook in (None, []):
            monkeypatch.setattr(Fn.LSTMStack, "collect_bwd", hook)
            net.zero_grad()
            xi = x.clone().requires_grad_(True)
            out, _ = net(xi)
            if dout is None:
                dout = torch.randn(out.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(18))
            out.backward(dout)
            torch.cuda.synchronize()
            assert hook is None or len(hook) == L
            res.append((out.detach(), xi.grad, [p.grad.clone() for p in params]))
        (o0, d0, g0), (o1, d1, g1) = res
        _same("wavefront %s: output, hook on vs off" % wave, o1, o0)
        _same("wavefront %s: dx, hook on vs off" % wave, d1, d0)
        for i, (a, b) in enumerate(zip(g1, g0)):
            _same("wavefront %s: gradient %d, hook on vs off" % (wave, i), a, b)


# ---- LSTMLayer in bf16 mode -------------------------------------------------------------------------------------------
# (name, B, T, I, H, with h0 / c0 / dhT / dcT, expected forward kernel, expected BPTT)
LAYER_CASES = [
    ("c4-c4bwd-H1024", 32, 60, 240, 1024, True, "c4_fwd", "c4_bwd_chunks"),
    ("c4-tcbwd-predictor", 32, 129, 256, 256, False, "c4_fwd", "tc_bwd"),
    ("tc-H192", 7, 33, 64, 192, True, "tc_fwd", "tc_bwd"),
    ("fp32-recurrence-H48", 5, 21, 24, 48, True, "seq", "seq_bwd"),
]


@pytest.mark.parametrize("name,B,T,I,H,init,fk,bk", LAYER_CASES, ids=[c[0] for c in LAYER_CASES])
def test_lstm_layer_bf16_teacher_forced(name, B, T, I, H, init, fk, bk, monkeypatch):
    """functional.LSTMLayer in bf16 mode, the same per-layer checks as the stack, plus dh0 / dc0 and the t = 0 row of the
    h_{t-1} operand of dW_hh (bf16(h0), or zeros).  The BPTT's dG is captured by wrapping the ops entry the layer calls."""
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    seed = 300 * H + T
    gen = torch.Generator(device=DEV).manual_seed(seed)
    k = 1 / math.sqrt(H)
    w_ih = ((torch.rand(4 * H, I, device=DEV, generator=gen) * 2 - 1) * k).requires_grad_(True)
    w_hh = ((torch.rand(4 * H, H, device=DEV, generator=gen) * 2 - 1) * k).requires_grad_(True)
    b_ih = ((torch.rand(4 * H, device=DEV, generator=gen) * 2 - 1) * k).requires_grad_(True)
    b_hh = ((torch.rand(4 * H, device=DEV, generator=gen) * 2 - 1) * k).requires_grad_(True)
    x = torch.randn(B, T, I, device=DEV, generator=gen).requires_grad_(True)
    h0 = c0 = dhT = dcT = None
    if init:
        h0 = (torch.randn(B, H, device=DEV, generator=gen) * 0.5).requires_grad_(True)
        c0 = (torch.randn(B, H, device=DEV, generator=gen) * 0.5).requires_grad_(True)
        dhT = torch.randn(B, H, device=DEV, generator=gen) * 0.5
        dcT = torch.randn(B, H, device=DEV, generator=gen) * 0.5
    dy = torch.randn(B, T, H, device=DEV, generator=gen)
    cap = {}
    for entry in ("lstm_c4_bwd_chunks", "lstm_tc_bwd", "lstm_seq_bwd"):
        orig = getattr(ops, entry)

        def wrapped(*a, _orig=orig, _entry=entry, **kw):
            out = _orig(*a, **kw)
            cap[_entry] = out[0].clone()
            return out
        monkeypatch.setattr(ops, entry, wrapped)
    y, hT, cT = Fn.LSTMLayer.apply(x, h0, c0, w_ih, w_hh, b_ih, b_hh, "bf16")
    gf = y.grad_fn
    x16, sh0, sc0, _, _, ysave, gates, cseq = gf.saved_tensors
    kern = "c4_fwd" if gf.c4 else "tc_fwd" if gf.tc else "seq"
    assert kern == fk, (name, kern)
    ysave, gates, cseq = ysave.clone(), gates.clone(), cseq.clone()
    yv = y.detach().clone()
    x16 = x16.view(B, T, I)
    zero = torch.zeros(B, H, device=DEV)
    h0v = zero if h0 is None else h0.detach()
    c0v = zero if c0 is None else c0.detach()
    _same(name + " hT = y[:, -1]", hT.detach(), yv[:, -1])
    _same(name + " cT = cseq[:, -1]", cT.detach(), cseq[:, -1])
    _same(name + " x16 = bf16_rn(x)", x16, x.detach().to(bf16))
    if kern == "c4_fwd":
        _same(name + " hprev16 = [bf16(h0), bf16_rn(y[:, :-1])]", ysave, _shift(h0v.to(bf16), yv.to(bf16)))
        hin = ysave
    elif kern == "tc_fwd":
        _same(name + " y16 = bf16_rn(y)", ysave, yv.to(bf16))
        hin = _shift(h0v.to(bf16), ysave)
    else:
        _same(name + " saved y", ysave, yv)
        hin = _shift(h0v, yv)
    check_lstm_fwd(name, x16, w_ih.detach(), w_hh.detach(), b_ih.detach(), b_hh.detach(), hin, _shift(c0v, cseq), gates,
                   cseq, yv, kern)
    if init:
        torch.autograd.backward([y, hT, cT], [dy, dhT, dcT])
    else:
        y.backward(dy)
    torch.cuda.synchronize()
    entry = {"c4_bwd_chunks": "lstm_c4_bwd_chunks", "tc_bwd": "lstm_tc_bwd", "seq_bwd": "lstm_seq_bwd"}[bk]
    assert list(cap) == [entry], (name, list(cap))
    dgq = cap[entry].view(B, T, 4 * H)
    if bk == "c4_bwd_chunks":
        n_add = _n_add("c4_bwd", H, 16)
    elif bk == "tc_bwd":
        n_add = _n_add("tc_bwd", H, tc_cluster_size(H))
    else:
        n_add = _n_add("seq", H)
    # (the BPTT may write over the saved gates -- the fp32 one writes its dgates there: the clone is read)
    (dh0r, dh0b), (dc0r, dc0b) = check_lstm_bwd(name, dy, dgq, gates, cseq, None if c0 is None else c0.detach(),
                                                w_hh.detach(), dhT, dcT, "seq" if bk == "seq_bwd" else bk,
                                                n_add, bf16_out=bk != "seq_bwd")
    dg16 = dgq if dgq.dtype == bf16 else dgq.to(bf16)
    hprev = hin if hin.dtype == bf16 else hin.to(bf16)
    if kern == "seq":                                # the dW_hh operand of the fp32 recurrence: bf16_rn of [h0, y]
        hprev = _shift(h0v, yv).to(bf16)
    _same(name + " h_{t-1} operand at t = 0", hprev[:, 0], h0v.to(bf16))
    check_lstm_grads(name, dg16, x16, hprev, w_ih.detach(), w_ih.grad, w_hh.grad, b_ih.grad, b_hh.grad,
                     dgq.reshape(B * T, 4 * H), dx=x.grad)
    if init:
        chk = Worst(name + " initial state")
        chk.add("dh0", h0.grad, dh0r, dh0b)
        chk.add("dc0", c0.grad, dc0r, dc0b)
        chk.done()


# ---- JointLoss backward in bf16 mode ----------------------------------------------------------------------------------
# (name, B, T, U, E, D, J, V, xlen, ylen, fused): V = 1024 takes the flipped dW2 GEMM (hid^T dl, then transposed),
# V = 1000 the other branch; fused: the logits GEMM emits the softmax statistics and bf16 logits (the headline path),
# otherwise (EDGEDICT_FUSE_LSE=0) fp32 logits, the fp32 loss and its bf16 gradient.  Every case takes the tanh' epilogue
# of the d-hidden GEMM: in bf16 mode J % 8 == 0 is required (test_joint_loss_bf16_rejects_j_not_multiple_of_8).  Ragged
# lengths leave padded cells, and the last utterance is full so that its last cell, the last row of every flat joint
# buffer, carries a gradient
JOINT_CASES = [
    ("E640-D256-J640-V1024", 3, 21, 9, 640, 256, 640, 1024, [14, 1, 21], [3, 0, 8], True),
    ("E640-D256-J640-V1000", 2, 17, 6, 640, 256, 640, 1000, [9, 17], [2, 5], True),
    ("E640-D256-J640-V1024-unfused", 3, 19, 7, 640, 256, 640, 1024, [11, 1, 19], [6, 0, 4], False),
]


def _joint_inputs(B, T, U, E, D, J, V, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    h_enc = torch.randn(B, T, E, device=DEV, generator=gen).requires_grad_(True)
    h_dec = torch.randn(B, U, D, device=DEV, generator=gen).requires_grad_(True)
    w1 = (torch.randn(J, E + D, device=DEV, generator=gen) / math.sqrt(E + D)).requires_grad_(True)
    b1 = (torch.randn(J, device=DEV, generator=gen) * 0.1).requires_grad_(True)
    w2 = (torch.randn(V, J, device=DEV, generator=gen) * (3.0 / math.sqrt(J))).requires_grad_(True)
    b2 = torch.randn(V, device=DEV, generator=gen).requires_grad_(True)
    labels = torch.randint(1, V, (B, U - 1), device=DEV, generator=gen, dtype=torch.int32)
    return h_enc, h_dec, w1, b1, w2, b2, labels


def _joint_run(name, B, T, U, E, D, J, V, xl, yl, monkeypatch, side, fused):
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    monkeypatch.setattr(Fn, "JOINT_WGRAD_SIDE", side)
    monkeypatch.setattr(Fn, "FUSE_JOINT_LSE", fused)
    h_enc, h_dec, w1, b1, w2, b2, labels = _joint_inputs(B, T, U, E, D, J, V, V + J + T)
    xlen = torch.tensor(xl, dtype=torch.int32, device=DEV)
    ylen = torch.tensor(yl, dtype=torch.int32, device=DEV)
    cap = {}
    orig_bwd, orig_dtanh, orig_reduce = Fn._joint_bwd, ops.gemm_bf16_dtanh, ops.joint_dpre_reduce

    def joint_bwd(p, dlog2, *a, **kw):
        cap["dl16"] = dlog2.clone()
        return orig_bwd(p, dlog2, *a, **kw)

    def dtanh(*a, **kw):
        out = orig_dtanh(*a, **kw)
        cap["dpre16"] = out.clone()
        return out
    def reduce(*a, **kw):
        dep, ddp = orig_reduce(*a, **kw)
        cap["dep"], cap["ddp"] = dep.clone(), ddp.clone()
        return dep, ddp
    monkeypatch.setattr(Fn, "_joint_bwd", joint_bwd)
    monkeypatch.setattr(ops, "gemm_bf16_dtanh", dtanh)
    monkeypatch.setattr(ops, "joint_dpre_reduce", reduce)
    loss, _ = Fn.JointLoss.apply(h_enc, h_dec, w1, b1, w2, b2, labels, xlen, ylen, 0, "bf16")
    sv = loss.grad_fn.saved_tensors
    hid = sv[0].clone()
    logits = sv[5].clone()          # fused: bf16, and the gradient is written over it in place
    assert logits.dtype == (bf16 if fused else f32), (name, logits.dtype)
    loss.backward()
    torch.cuda.synchronize()
    grads = [t.grad.clone() for t in (h_enc, h_dec, w1, b1, w2, b2)]
    return dict(h_enc=h_enc.detach(), h_dec=h_dec.detach(), w1=w1.detach(), w2=w2.detach(), b2=b2.detach(), hid=hid,
                logits=logits, labels=labels, cap=cap, grads=grads)


def _check_dlogits(name, r, B, T, U, V, J, xl, yl, fused):
    """The engine's bf16 dlogits against the fp64 C oracle (oracle/loss.py), with the bars of
    test_gpu_joint_loss_fused.py.  fused: against the restatement of the chained kernels (statistics of the exact
    logits X = hid16 bf16(W2)^T + b2, the exponent on the engine's bf16 logits; bars of its section (d)), and against the
    true gradient of X within the bf16-logit bar of (d).  Unfused: against oracle.loss.logits of the engine's own fp32
    logits, the exact answer for them (bars of section (c))."""
    import numpy as np
    from tests.test_gpu_joint_loss_fused import (GRAD_ABS, GRAD_FRO, _grad_errors, _oracle_logits, _restated_grad)
    from tests.test_gpu_joint_loss_fused import _bf16_ulp as ulp16
    lab = r["labels"].cpu().numpy()
    xlen, ylen = np.asarray(xl, np.int32), np.asarray(yl, np.int32)
    t = np.arange(T)[None, :, None]
    u = np.arange(U)[None, None, :]
    valid = (t < xlen[:, None, None]) & (u <= ylen[:, None, None])
    X = r["hid"].view(-1, J).double() @ r["w2"].to(bf16).double().t() + r["b2"].double()
    c = dict(B=B, T=T, U=U, blank=0, X=X.view(B, T, U, V), lab=lab, xlen=xlen, ylen=ylen, valid=valid,
             lab_d=r["labels"], xlen_d=torch.as_tensor(xlen, device=DEV), ylen_d=torch.as_tensor(ylen, device=DEV))
    g = r["cap"]["dl16"].view(B, T, U, V)
    if fused:
        ref = _restated_grad(c, r["logits"]) / B
    else:
        _, ref = _oracle_logits(c, r["logits"])
        ref = torch.as_tensor(ref, device=DEV) / B
    ratio, fro = _grad_errors(g, ref)
    print("  %-40s dl16 vs the fp64 oracle: element err / bar %.3f, Frobenius rel %.2e (bar %.0e)"
          % (name, ratio, fro, GRAD_FRO))
    assert ratio <= 1.0 and fro <= GRAD_FRO, (name, ratio, fro)
    if fused:
        _, gtrue = _oracle_logits(c, c["X"])
        gtrue = torch.as_tensor(gtrue, device=DEV) / B
        bar = ((1 + 2.0 ** -8) * torch.expm1(ulp16(c["X"])) + 2.0 ** -8) * gtrue.abs() + GRAD_ABS
        ratio_t = float(((g.double() - gtrue).abs() / bar).max())
        print("  %-40s dl16 vs the true fp64 gradient of X: element err / bar %.3f" % (name, ratio_t))
        assert ratio_t <= 1.0, (name, ratio_t)


@pytest.mark.parametrize("name,B,T,U,E,D,J,V,xl,yl,fused", JOINT_CASES, ids=[c[0] for c in JOINT_CASES])
def test_joint_loss_bwd_teacher_forced(name, B, T, U, E, D, J, V, xl, yl, fused, monkeypatch):
    """JointLoss.backward in bf16 mode.  First the engine's bf16 dlogits against the fp64 C oracle (_check_dlogits).
    Then, teacher-forced from those dlogits and the saved bf16 hidden: db2 and db1 bitwise in eb_colsum's order; dW2 per
    element (n_add from its GEMM plan); dpre16 = bf16_rn(fp32(fp32(dl16 bf16(W2)) fp32(1 - hid^2))) within the bar (the
    GEMM's, and the two fp32 roundings of the epilogue) plus half a bf16 ulp; dep = sum_u and ddp = sum_t of
    float(dpre16) bitwise; dh_enc, dh_dec, dW1[:, :E], dW1[:, E:] per element from bf16(dep), bf16(ddp); zero dlogits on
    every padded cell; the same bits with the output layer's weight gradients on the side stream (JOINT_WGRAD_SIDE) and
    without."""
    from tests.test_gpu_glue_fp64 import _seq_sums
    r = _joint_run(name, B, T, U, E, D, J, V, xl, yl, monkeypatch, True, fused)
    r0 = _joint_run(name, B, T, U, E, D, J, V, xl, yl, monkeypatch, False, fused)
    for i, (a, b) in enumerate(zip(r["grads"], r0["grads"])):
        _same("%s gradient %d: JOINT_WGRAD_SIDE on vs off" % (name, i), a, b)
    dl16, dpre16, hid = r["cap"]["dl16"], r["cap"]["dpre16"], r["hid"]
    assert dl16.dtype == bf16 and dpre16.dtype == bf16 and hid.dtype == bf16
    N = B * T * U
    dhe, dhd, dw1, db1, dw2, db2 = r["grads"]
    t = torch.arange(T, device=DEV).view(1, T, 1)
    u = torch.arange(U, device=DEV).view(1, 1, U)
    valid = (t < torch.tensor(xl, device=DEV).view(B, 1, 1)) & (u <= torch.tensor(yl, device=DEV).view(B, 1, 1))
    assert bool((dl16.view(B, T, U, V)[~valid] == 0).all()), name + ": nonzero dlogits on a padded cell"
    _check_dlogits(name, r, B, T, U, V, J, xl, yl, fused)
    _same(name + " db2 vs the lane-order column sum of dl16", db2, _colsum_lanes(dl16))
    chk = Worst(name + " joint bwd")
    dl, h = dl16.double(), hid.view(N, J).double()
    ks = _plan(J, V, N)[1] if V % 256 == 0 else _plan(V, J, N)[1]
    chk.add("dW2", dw2, dl.t() @ h, gemm_n_add(N, ks) * UTC * (dl.abs().t() @ h.abs()))
    w2_16 = r["w2"].to(bf16).double()
    P = dl @ w2_16
    one = 1 - h * h
    dpre = P * one
    bar = V * UTC * (dl.abs() @ w2_16.abs()) * one + 2 * U24 * dpre.abs()
    bar = bar + 0.5 * _bf16_ulp(dpre.abs() + bar)
    chk.add("dpre16", dpre16.view(N, J), dpre, bar)
    del P, one, dpre, bar
    dep, ddp = _seq_sums(dpre16.view(B, T, U, J))
    dep, ddp = dep.to(DEV), ddp.to(DEV)
    _same(name + " dep = sum over u of float(dpre16), in order", r["cap"]["dep"], dep)
    _same(name + " ddp = sum over t of float(dpre16), in order", r["cap"]["ddp"], ddp)
    ep16, dp16 = dep.view(B * T, J).to(bf16).double(), ddp.view(B * U, J).to(bf16).double()
    w1 = r["w1"].to(bf16).double()
    he, hd = r["h_enc"].view(B * T, E).to(bf16).double(), r["h_dec"].view(B * U, D).to(bf16).double()
    for label, a, w, got, M, K in (("dh_enc", ep16, w1[:, :E], dhe.view(B * T, E), B * T, J),
                                   ("dh_dec", dp16, w1[:, E:], dhd.view(B * U, D), B * U, J)):
        ks = _plan(M, w.shape[1], K)[1]
        chk.add(label, got, a @ w, gemm_n_add(K, ks) * UTC * (a.abs() @ w.abs()))
    for label, a, x, got in (("dW1[:, :E]", ep16, he, dw1[:, :E]), ("dW1[:, E:]", dp16, hd, dw1[:, E:])):
        ks = _plan(J, x.shape[1], a.shape[0])[1]
        chk.add(label, got, a.t() @ x, gemm_n_add(a.shape[0], ks) * UTC * (a.abs().t() @ x.abs()))
    chk.done()
    _same(name + " db1 vs colsum_kernel's order over dep", db1.cpu(),
          _colsum_order(dep.view(B * T, J), torch.zeros(J, device=DEV)))


def test_joint_loss_bf16_rejects_j_not_multiple_of_8():
    """In bf16 mode the joint's hidden is bf16 and its kernels take 16-byte rows: J % 8 != 0 is refused on the host by
    eb_joint_hidden_fwd before any backward exists (so `_joint_bwd`'s joint_hidden_bwd branch is the fp32 mode's), with
    an error rather than a fall-back."""
    from edgedict_b200 import functional as Fn
    B, T, U, E, D, J, V = 2, 5, 3, 64, 32, 100, 136
    h_enc, h_dec, w1, b1, w2, b2, labels = _joint_inputs(B, T, U, E, D, J, V, 5)
    xlen = torch.tensor([5, 3], dtype=torch.int32, device=DEV)
    ylen = torch.tensor([2, 1], dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="eb_joint_hidden_fwd"):
        Fn.JointLoss.apply(h_enc, h_dec, w1, b1, w2, b2, labels, xlen, ylen, 0, "bf16")
