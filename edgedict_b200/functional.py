"""Autograd glue: each Function's forward/backward is a short sequence of C-ABI calls
(edgedict_b200/ops.py).  torch.autograd only stitches them together -- it never differentiates
through a torch op on the hot path.

Reference semantics per Function are cited next to each class (paths relative to the reference project).
"""
import math
import numbers

import torch

from . import ops

import os

f32, bf16 = torch.float32, torch.bfloat16
# bf16 mode: the joint's output GEMM also emits the softmax statistics of the loss from its fp32 accumulators
# and writes bf16 logits; the 8 GB denominator pass disappears and the gradient pass runs in place on 4 GB
# (EDGEDICT_FUSE_LSE=0 selects the unfused fp32-logits path).
FUSE_JOINT_LSE = os.environ.get("EDGEDICT_FUSE_LSE", "1") != "0"


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


class Linear(torch.autograd.Function):
    """nn.Linear: y = x W^T + b  (rnnt/models.py:129,148,163-167)."""

    @staticmethod
    def forward(ctx, x, w, b, precision):
        shp = x.shape
        x2 = _c(x).view(-1, shp[-1])
        x16 = ops.cast_bf16(x2) if precision == "bf16" else None
        y = ops.mm_nt(x2, w, b, precision, x16=x16)
        ctx.save_for_backward(x2 if x16 is None else x16, w)
        ctx.precision, ctx.has_b, ctx.shp = precision, b is not None, shp
        return y.view(*shp[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        xs, w = ctx.saved_tensors
        p = ctx.precision
        dy2 = _c(dy).view(-1, dy.shape[-1])
        dy16 = ops.cast_bf16(dy2) if p == "bf16" else None
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = ops.mm_nn(dy2, w, p, dy16=dy16).view(ctx.shp)
        if ctx.needs_input_grad[1]:
            dw = ops.mm_tn(dy2, xs, p, dy16=dy16, x16=xs if p == "bf16" else None)
        if ctx.has_b and ctx.needs_input_grad[2]:
            db = ops.colsum(dy2)
        return dx, dw, db, None


class LayerNormRes(torch.autograd.Function):
    """y = LayerNorm(x + res) (res optional): nn.LayerNorm + the residual add of
    ResLayerNormLSTM.forward (rnnt/models.py:47,66-70,124)."""

    @staticmethod
    def forward(ctx, x, res, gamma, beta, eps):
        x = _c(x)
        res = _c(res) if res is not None else None
        y, _, mean, rstd = ops.layernorm_fwd(x, res, gamma, beta, eps)
        ctx.save_for_backward(x, res, gamma, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, res, gamma, mean, rstd = ctx.saved_tensors
        dz, dgamma, dbeta = ops.layernorm_bwd(_c(dy), x, res, gamma, mean, rstd)
        return dz, (dz if res is not None else None), dgamma, dbeta, None


class TimeReduce(torch.autograd.Function):
    """TimeReduction(2): zero-pad to even length, mean of frame pairs (rnnt/models.py:21-29)."""

    @staticmethod
    def forward(ctx, x):
        ctx.T = x.shape[1]
        y, _ = ops.time_reduce_fwd(_c(x))
        return y

    @staticmethod
    def backward(ctx, dy):
        return ops.time_reduce_bwd(_c(dy), ctx.T)


class Embedding(torch.autograd.Function):
    """nn.Embedding(padding_idx=PAD) with the optional BOS prepend of Decoder.forward
    (rnnt/models.py:150-153)."""

    @staticmethod
    def forward(ctx, ids, w, prepend_bos, bos, pad):
        ids = _c(ids)
        if ids.dtype not in (torch.int32, torch.int64):
            ids = ids.long()
        ctx.save_for_backward(ids)
        ctx.meta = (w.shape[0], prepend_bos, bos, pad)
        return ops.embedding_fwd(ids, w, prepend_bos, bos)

    @staticmethod
    def backward(ctx, dout):
        (ids,) = ctx.saved_tensors
        V, prepend_bos, bos, pad = ctx.meta
        return None, ops.embedding_bwd(ids, _c(dout), V, prepend_bos, bos, pad), None, None, None


# The K-split BPTT kernel (eb_lstm_c4_bwd_chunks) runs where it measured faster than lstm_tc_bwd on an H100 at B = 32:
# H = 1024 (6.35 - 6.49 against 7.48 - 7.67 us per step).  At H = 512 it is slower (4.98 against 4.42), at the predictor's
# H = 256 (two clusters) the two measure the same (3.90 - 4.04 against 3.89 - 4.00); those sizes keep lstm_tc_bwd.
C4_BPTT_MIN_H = 1024


def _c4_bptt(H):
    return H >= C4_BPTT_MIN_H and ops.lstm_c4_bwd_chunks_supported(H)


class LSTMLayer(torch.autograd.Function):
    """One unidirectional batch_first nn.LSTM layer (rnnt/models.py:45-46,64-65,145-147):
    bulk input GEMM + persistent recurrent kernel; backward = BPTT kernel + three bulk GEMMs."""

    @staticmethod
    def forward(ctx, x, h0, c0, w_ih, w_hh, b_ih, b_hh, precision):
        B, T, I = x.shape
        H = w_hh.shape[1]
        x2 = _c(x).view(B * T, I)
        x16 = ops.cast_bf16(x2) if precision == "bf16" else None
        bias = b_ih + b_hh
        xg = ops.mm_nt(x2, w_ih, bias, precision, x16=x16).view(B, T, 4 * H)
        h0c = _c(h0) if h0 is not None else None
        c0c = _c(c0) if c0 is not None else None
        need = any(ctx.needs_input_grad)     # (grad mode is off inside Function.forward)
        tc = precision == "bf16" and ops.lstm_tc_supported(B, H)
        c4 = precision == "bf16" and ops.lstm_c4_supported(B, H)
        if c4:
            # cluster / wgmma kernels: saves in their CTA-private layout, y16 IS the h_{t-1}-shifted copy
            y, y16, hT, cT, gates, cseq = ops.lstm_c4_fwd(xg, ops.cast_bf16(_c(w_hh)), h0c, c0c, need,
                                                          std_saves=None if ops.C4_BWD else True)
        elif tc:
            y, y16, hT, cT, gates, cseq = ops.lstm_tc_fwd(xg, ops.cast_bf16(_c(w_hh)), h0c, c0c, need)
        else:
            y, hT, cT, gates, cseq = ops.lstm_seq_fwd(xg, _c(w_hh), h0c, c0c, need)
            y16 = None
        if need:
            ctx.save_for_backward(x2 if x16 is None else x16, h0c, c0c, w_ih, w_hh, y16 if (tc or c4) else y, gates, cseq)
            ctx.precision, ctx.dims, ctx.tc, ctx.c4, ctx.c4_bwd = precision, (B, T, I, H), tc, c4, c4 and ops.C4_BWD
        return y, hT, cT

    @staticmethod
    def backward(ctx, dy, dhT, dcT):
        xs, h0, c0, w_ih, w_hh, y, gates, cseq = ctx.saved_tensors
        B, T, I, H = ctx.dims
        p = ctx.precision
        dy = _c(dy) if dy is not None else torch.zeros(B, T, H, dtype=f32, device=y.device)
        dhT = _c(dhT) if dhT is not None else None
        dcT = _c(dcT) if dcT is not None else None
        if getattr(ctx, "consumed", False):
            raise RuntimeError("LSTMLayer.backward ran twice on the same graph: the saved gates are overwritten in "
                               "place by the first pass (retain_graph is not supported by this node)")
        ctx.consumed = True
        if ctx.c4_bwd:
            dg16, dh0, dc0 = ops.lstm_c4_bwd(dy, gates, cseq, c0, ops.transpose_to_bf16(_c(w_hh)), dhT, dcT)
            dg2 = dg16.view(B * T, 4 * H)
        elif ctx.c4 and _c4_bptt(H):
            dg16, dh0, dc0 = ops.lstm_c4_bwd_chunks(dy, gates, cseq, ops.transpose_to_bf16(_c(w_hh)), [T], B,
                                                    torch.empty(B, T, 4 * H, dtype=bf16, device=dy.device), c0, dhT, dcT)
            dg2 = dg16.view(B * T, 4 * H)
        elif ctx.tc or ctx.c4:
            dg16, dh0, dc0 = ops.lstm_tc_bwd(dy, gates, cseq, c0, ops.transpose_to_bf16(_c(w_hh)), dhT, dcT)
            dg2 = dg16.view(B * T, 4 * H)
        else:
            dg, dh0, dc0 = ops.lstm_seq_bwd(dy, gates, cseq, c0, _c(w_hh), dhT, dcT)
            dg2 = dg.view(B * T, 4 * H)
            dg16 = ops.cast_bf16(dg2) if p == "bf16" else None
        dg16 = dg16.view(B * T, 4 * H) if dg16 is not None else None
        if ctx.c4:
            hp2 = y.view(B * T, H)                           # the kernel already wrote h_{t-1} for every step
        else:
            # h_{t-1} for every step: y shifted right by one frame, h0 (or zeros) in front
            hprev = torch.empty_like(y)
            hprev[:, 1:] = y[:, :-1]
            if h0 is not None:
                hprev[:, 0] = h0
            else:
                hprev[:, 0].zero_()
            hp2 = hprev.view(B * T, H)
        dx = ops.mm_nn(dg2, w_ih, p, dy16=dg16).view(B, T, I) if ctx.needs_input_grad[0] else None
        dw_ih = ops.mm_tn(dg2, xs, p, dy16=dg16, x16=xs if p == "bf16" else None)
        dw_hh = ops.mm_tn(dg2, hp2, p, dy16=dg16, x16=hp2 if hp2.dtype == bf16 else None)
        db = ops.colsum(dg2)
        return (dx, dh0 if ctx.needs_input_grad[1] else None, dc0 if ctx.needs_input_grad[2] else None,
                dw_ih, dw_hh, db, db.clone(), None)


class GRULayer(torch.autograd.Function):
    """One unidirectional batch_first nn.GRU layer (rnnt/models.py:77-116, gate order r|z|n): bulk input GEMM with
    b_hr and b_hz folded into its bias (b_hn stays inside the reset product and is added by the recurrent kernel) +
    persistent recurrent kernel; backward = BPTT kernel + three bulk GEMMs (dx, dW_ih from the input-side gate gradient
    [dr, dz, dn], dW_hh from the recurrent-side one [dr, dz, r dn]) and their column sums for the biases.  fp32 mode runs
    the fp32 recurrence (eb_gru_seq_fwd/bwd); bf16 mode runs the tensor-core recurrence (eb_gru_tc_fwd/bwd) where it is
    supported (H % 64 == 0, H <= 1024) and the fp32 one otherwise, and the three bulk GEMMs on tensor cores."""

    @staticmethod
    def forward(ctx, x, h0, w_ih, w_hh, b_ih, b_hh, precision):
        B, T, I = x.shape
        H = w_hh.shape[1]
        x2 = _c(x).view(B * T, I)
        x16 = ops.cast_bf16(x2) if precision == "bf16" else None
        bias = torch.cat([b_ih[:2 * H] + b_hh[:2 * H], b_ih[2 * H:]])
        xg = ops.mm_nt(x2, w_ih, bias, precision, x16=x16).view(B, T, 3 * H)
        h0c = _c(h0) if h0 is not None else None
        bhn = _c(b_hh[2 * H:])
        need = any(ctx.needs_input_grad)     # (grad mode is off inside Function.forward)
        tc = precision == "bf16" and ops.gru_tc_supported(B, H)
        if tc:
            y, hT, save = ops.gru_tc_fwd(xg, ops.cast_bf16(_c(w_hh)), bhn, h0c, need)
        else:
            y, hT, save = ops.gru_seq_fwd(xg, _c(w_hh), bhn, h0c, need)
        if need:
            ctx.save_for_backward(x2 if x16 is None else x16, h0c, w_ih, w_hh, y, save)
            ctx.precision, ctx.dims, ctx.tc = precision, (B, T, I, H), tc
        return y, hT

    @staticmethod
    def backward(ctx, dy, dhT):
        xs, h0, w_ih, w_hh, y, save = ctx.saved_tensors
        B, T, I, H = ctx.dims
        p = ctx.precision
        if getattr(ctx, "consumed", False):
            raise RuntimeError("GRULayer.backward ran twice on the same graph (retain_graph is not supported by this "
                               "node)")
        ctx.consumed = True
        dy = _c(dy) if dy is not None else torch.zeros(B, T, H, dtype=f32, device=y.device)
        dhT = _c(dhT) if dhT is not None else None
        if ctx.tc:
            dgi, dgh, dh0 = ops.gru_tc_bwd(dy, save, y, h0, ops.transpose_to_bf16(_c(w_hh)), dhT)
        else:
            dgi, dgh, dh0 = ops.gru_seq_bwd(dy, save, y, h0, _c(w_hh), dhT)
        dgi2, dgh2 = dgi.view(B * T, 3 * H), dgh.view(B * T, 3 * H)
        dgi16 = (dgi2 if ctx.tc else ops.cast_bf16(dgi2)) if p == "bf16" else None
        dgh16 = (dgh2 if ctx.tc else ops.cast_bf16(dgh2)) if p == "bf16" else None
        # h_{t-1} for every step: y shifted right by one frame, h0 (or zeros) in front
        hprev = torch.empty_like(y)
        hprev[:, 1:] = y[:, :-1]
        if h0 is not None:
            hprev[:, 0] = h0
        else:
            hprev[:, 0].zero_()
        hp2 = hprev.view(B * T, H)
        dx = ops.mm_nn(dgi2, w_ih, p, dy16=dgi16).view(B, T, I) if ctx.needs_input_grad[0] else None
        dw_ih = ops.mm_tn(dgi2, xs, p, dy16=dgi16, x16=xs if p == "bf16" else None)
        dw_hh = ops.mm_tn(dgh2, hp2, p, dy16=dgh16)
        return (dx, dh0 if ctx.needs_input_grad[1] else None, dw_ih, dw_hh, ops.colsum(dgi2), ops.colsum(dgh2), None)


# ---- layer-wavefront schedule of the LSTM stack ------------------------------------------------------------
# The recurrence of one layer is a chain of T grid-synchronous steps that is bound by exchange/barrier LATENCY
# (DESIGN.md section 4a): one layer's persistent kernel leaves its SMs idle most of the time.  Layer l+1 at frame t
# only needs layer l up to frame t, so the time axis is cut into chunks and layer l+1 runs chunk c on a second
# stream while layer l runs chunk c+1: two persistent kernels (the lstm_c4 forward CTA: 128 threads, <= 168 registers,
# 109 KB of shared memory at H = 1024) fit on every SM and hide each other's latency.  The per-chunk input GEMM uses the
# co-resident tile configuration (EB_GEMM_CORESIDENT) so that it fits next to the other layer's recurrent CTA.
WAVEFRONT_CHUNKS = int(os.environ.get("EDGEDICT_WAVEFRONT_CHUNKS", "6"))     # 0 disables
_wave_streams = {}


def _side_streams(device):
    st = _wave_streams.get(device)
    if st is None:
        st = _wave_streams[device] = (torch.cuda.Stream(device), torch.cuda.Stream(device))
    return st


_aux_streams = {}


def _wave_aux_streams(device):
    """Four more streams of the forward wavefront: input-projection GEMMs (two) and LayerNorm / TimeReduction (two)."""
    st = _aux_streams.get(device)
    if st is None:
        st = _aux_streams[device] = tuple(torch.cuda.Stream(device) for _ in range(4))
    return st


def wavefront_plan(T, reductions, max_chunks=None):
    """Chunk lengths per layer for the wavefront schedule, or None when T is too short to cut.
    Chunk boundaries are multiples of 2^(number of time reductions) so that TimeReduction pairs never straddle
    a boundary; only the last chunk may be ragged (its zero padding is the reference's padding of the last
    frame, rnnt/models.py:24-27).  Returns a list (len L+1) of per-chunk lengths on each layer's time axis."""
    max_chunks = WAVEFRONT_CHUNKS if max_chunks is None else max_chunks
    if max_chunks < 2:
        return None
    gran = 1 << sum(1 for r in reductions if r)
    step = -(-T // (max_chunks * gran)) * gran
    if step < 16 * gran:                     # too short to amortise the per-chunk launches
        step = 16 * gran
    lens = [min(step, T - t0) for t0 in range(0, T, step)]
    if len(lens) < 2:
        return None
    plan = [lens]
    for r in reductions:
        lens = [(n + 1) // 2 for n in lens] if r else lens
        plan.append(lens)
    return plan


class _Chunks:
    """Chunk-major storage: the [B, Tc, D] blocks of all chunks back to back in one [B*T, D] buffer.  Row-wise
    kernels (LayerNorm, casts, the bulk GEMMs of the backward pass) run on the flat buffer, time-ordered ones
    (the recurrence, TimeReduction) on one block."""

    def __init__(self, B, lens):
        self.B, self.lens = B, lens
        self.off = [0]
        for n in lens:
            self.off.append(self.off[-1] + n)
        self.rows = B * self.off[-1]

    def new(self, D, dtype, device):
        return torch.empty(self.rows, D, dtype=dtype, device=device) if D else torch.empty(self.rows, dtype=dtype, device=device)

    def blk(self, buf, c):
        a, b = self.B * self.off[c], self.B * self.off[c + 1]
        v = buf[a:b]
        return v.view(self.B, self.lens[c], buf.shape[1]) if buf.dim() == 2 else v

    def scatter(self, x):
        """[B, T, D] -> chunk-major flat buffer."""
        out = self.new(x.shape[2], x.dtype, x.device)
        for c in range(len(self.lens)):
            self.blk(out, c).copy_(x[:, self.off[c]:self.off[c + 1]])
        return out

    def gather(self, buf):
        """chunk-major flat buffer -> [B, T, D]."""
        out = torch.empty(self.B, self.off[-1], buf.shape[1], dtype=buf.dtype, device=buf.device)
        for c in range(len(self.lens)):
            out[:, self.off[c]:self.off[c + 1]].copy_(self.blk(buf, c))
        return out


BPTT_ONE_LAUNCH = __import__("os").environ.get("EDGEDICT_BPTT_ONE_LAUNCH", "1") != "0"   # one BPTT launch per layer (else per chunk)
# Chunked backward (LSTMStack._backward_wave): the BPTT of every layer runs in groups of BPTT_GROUP time chunks, and the
# input of a group (dgrad GEMM of the layer above, TimeReduction and LayerNorm backward) is prepared on other streams
# while the recurrence of the layer above is still running, so that the recurrences follow each other without the
# serial schedule's gap between layers.  Tests set it to False to take the serial schedule, which gives the same bits.
BPTT_WAVEFRONT = True
BPTT_GROUP = 3          # time chunks per BPTT launch of the chunked backward (fewer launches, each ~45 us of prologue)
_bwd_streams = {}


def _wave_bwd_streams(device):
    """Streams of the chunked backward: one for the recurrence and two for the group inputs at high priority (their
    blocks are dispatched first when a BPTT grid ends, so the next group's grid is not held up behind a GEMM), and one
    for the weight gradients at the default priority."""
    st = _bwd_streams.get(device)
    if st is None:
        st = _bwd_streams[device] = tuple(torch.cuda.Stream(device, priority=-1) for _ in range(3)) + (
            torch.cuda.Stream(device),)
    return st


class LSTMStack(torch.autograd.Function):
    """ResLayerNormLSTM.forward (rnnt/models.py:57-75) for all layers at once, bf16 tensor-core mode, zero
    initial state: per layer nn.LSTM -> LayerNorm(y + x) (no residual for layer 0) -> optional TimeReduction,
    executed as a layer wavefront over time chunks on two streams (see above).  Numerically identical to the
    layer-by-layer Functions (same kernels, same per-row / per-step arithmetic); the backward pass reuses their
    kernels on the chunk-major buffers, the BPTT kernel once per chunk with the (dh, dc) carry.
    args: x [B,T,I] fp32, cfg = (reductions, eps, plan), then per layer w_ih, w_hh, b_ih, b_hh, ln_w, ln_b.
    returns y [B,T',H], h_T [L,B,H], c_T [L,B,H] (final states: not differentiated through)."""

    collect = None      # tests: set to a list to receive every layer's output [B,T_l,H] (parity of the per-layer activations)
    # tests: set to a list to receive, per backward and per layer l = 0 .. L-1, a dict of [B,T_l,.] tensors: "dln" the
    # LayerNorm's incoming gradient (after TimeReduction backward), "dy" the BPTT's input (the LayerNorm dz, before the dgrad
    # GEMM accumulates into it), "dg16" the bf16 dG of the BPTT, "dxs" d xs[l] (dy + the dgrad GEMM; None for l = 0, whose
    # product is the returned dx).  Off (None): nothing is copied or ordered.
    collect_bwd = None

    @staticmethod
    def forward(ctx, x, cfg, *params):
        reductions, eps, plan = cfg
        L = len(reductions)
        B, T, I0 = x.shape
        dev = x.device
        H = params[1].shape[1]
        C = len(plan[0])
        need = any(ctx.needs_input_grad)
        c4 = ops.lstm_c4_supported(B, H)
        c4b = c4 and ops.C4_BWD                              # saves in lstm_c4's own layout, BPTT through lstm_c4
        ck = [_Chunks(B, lens) for lens in plan]
        P = [params[6 * l:6 * l + 6] for l in range(L)]
        wih16 = [ops.cast_bf16(_c(p[0])) for p in P]
        whh16 = [ops.cast_bf16(_c(p[1])) for p in P]
        bias = [p[2] + p[3] for p in P]
        x16 = [ck[0].scatter(ops.cast_bf16(_c(x)))] + [None] * L
        xs = [None] * (L + 1)                                # fp32 layer inputs (LayerNorm residuals), l >= 1
        y, y16, gates, cseq, mean, rstd = ([None] * L for _ in range(6))
        z = [None] * L
        for l in range(L):
            k, kn = ck[l], ck[l + 1]
            y[l] = k.new(H, f32, dev)
            y16[l] = k.new(H, bf16, dev) if (need or not c4) else None     # c4: holds h_{t-1} (the dW_hh operand)
            gates[l] = k.new(4 * H, f32, dev) if (need and not c4b) else None
            cseq[l] = k.new(H, f32, dev) if (need and not c4b) else None
            mean[l], rstd[l] = k.new(0, f32, dev), k.new(0, f32, dev)
            xs[l + 1] = kn.new(H, f32, dev)
            z[l] = k.new(H, f32, dev) if reductions[l] else xs[l + 1]
            x16[l + 1] = kn.new(H, bf16, dev) if l + 1 < L else None
        hT = torch.empty(L, C, B, H, dtype=f32, device=dev)
        cT = torch.empty(L, C, B, H, dtype=f32, device=dev)
        # Streams: the recurrence of layer l on rec[l % 2]; its input projection (xg = x W_ih^T + b, per chunk) on gem[l % 2]
        # and its LayerNorm / TimeReduction on nrm[l % 2].  The GEMM of chunk c+1 therefore runs AHEAD, under the recurrence of
        # chunk c, instead of queueing behind it (in one stream per layer parity the ~0.15 ms of GEMM + LayerNorm per chunk
        # were 20 % of the stream's time with no recurrence running); xg is double-buffered per layer.
        xgbuf = [[torch.empty(B * max(plan[l]), 4 * H, dtype=f32, device=dev) for _ in range(2)] for l in range(L)]
        c4saves = [[None] * C for _ in range(L)]               # c4: per (layer, chunk) saves in the kernels' layout

        main = torch.cuda.current_stream(dev)
        rec = _side_streams(dev)
        aux = _wave_aux_streams(dev)
        gem, nrm = aux[:2], aux[2:]
        ev = lambda: torch.cuda.Event()
        prep_done = [[ev() for _ in range(C)] for _ in range(L)]
        rec_done = [[ev() for _ in range(C)] for _ in range(L)]
        done = [[ev() for _ in range(C)] for _ in range(L)]
        for s_ in (*rec, *aux):
            s_.wait_stream(main)
        for d in range(L + C - 1):
            for l in range(max(0, d - C + 1), min(L, d + 1)):
                c = d - l
                k, kn = ck[l], ck[l + 1]
                Tc = k.lens[c]
                xg = xgbuf[l][c % 2][:B * Tc]
                with torch.cuda.stream(gem[l % 2]):
                    if l > 0:
                        gem[l % 2].wait_event(done[l - 1][c])
                    if c >= 2:
                        gem[l % 2].wait_event(rec_done[l][c - 2])          # the xg buffer is free again
                    xin = k.blk(x16[l], c)
                    ops.gemm_bf16(xin.view(B * Tc, xin.shape[2]), 0, wih16[l], 0, B * Tc, 4 * H, xin.shape[2],
                                  bias=bias[l], out=xg, flags=ops.GEMM_CORESIDENT)
                    prep_done[l][c].record(gem[l % 2])
                with torch.cuda.stream(rec[l % 2]):
                    rec[l % 2].wait_event(prep_done[l][c])
                    if c4:
                        r = ops.lstm_c4_fwd(xg.view(B, Tc, 4 * H), whh16[l], hT[l, c - 1] if c else None,
                                            cT[l, c - 1] if c else None, need,
                                            out=(k.blk(y[l], c), k.blk(y16[l], c) if need else None, hT[l, c], cT[l, c]),
                                            std_saves=None if (c4b or not need) else (k.blk(gates[l], c), k.blk(cseq[l], c)))
                        if need and c4b:
                            c4saves[l][c] = (r[4], r[5])
                            r[4].record_stream(main)
                            r[5].record_stream(main)
                    else:
                        ops.lstm_tc_fwd(xg.view(B, Tc, 4 * H), whh16[l], hT[l, c - 1] if c else None,
                                        cT[l, c - 1] if c else None, need,
                                        out=(k.blk(y[l], c), k.blk(y16[l], c), hT[l, c], cT[l, c],
                                             k.blk(gates[l], c) if need else None, k.blk(cseq[l], c) if need else None))
                    rec_done[l][c].record(rec[l % 2])
                with torch.cuda.stream(nrm[l % 2]):
                    nrm[l % 2].wait_event(rec_done[l][c])
                    res = k.blk(xs[l], c) if l else None
                    nx16 = kn.blk(x16[l + 1], c) if x16[l + 1] is not None else None
                    if reductions[l]:
                        ops.layernorm_fwd(k.blk(y[l], c), res, P[l][4], P[l][5], eps[l],
                                          out=(k.blk(z[l], c), None, k.blk(mean[l], c), k.blk(rstd[l], c)))
                        ops.time_reduce_fwd(k.blk(z[l], c), out=(kn.blk(xs[l + 1], c), nx16))
                    else:
                        ops.layernorm_fwd(k.blk(y[l], c), res, P[l][4], P[l][5], eps[l],
                                          out=(kn.blk(xs[l + 1], c), nx16, k.blk(mean[l], c), k.blk(rstd[l], c)))
                    done[l][c].record(nrm[l % 2])
        for s_ in (*rec, *aux):
            main.wait_stream(s_)
        out = ck[L].gather(xs[L])
        if LSTMStack.collect is not None:
            LSTMStack.collect.extend(ck[l + 1].gather(xs[l + 1]) for l in range(L))
        hT_last, cT_last = hT[:, C - 1].contiguous(), cT[:, C - 1].contiguous()
        if need:
            if c4b:
                gates = [torch.empty(0, device=dev)] * L
                cseq = [torch.empty(0, device=dev)] * L
            flat_saves = [t for row in c4saves for pair in row for t in pair] if c4b else []
            ctx.save_for_backward(*params, hT, cT, *x16[:L], *xs[1:L], *y, *y16, *gates, *cseq, *mean, *rstd, *flat_saves)
            ctx.cfg, ctx.dims, ctx.c4, ctx.c4b = cfg, (B, T, I0, H, L, C), c4, c4b
        ctx.mark_non_differentiable(hT_last, cT_last)
        return out, hT_last, cT_last

    @staticmethod
    def backward(ctx, dout, _dh, _dc):
        reductions, eps, plan = ctx.cfg
        B, T, I0, H, L, C = ctx.dims
        sv = list(ctx.saved_tensors)
        params, sv = sv[:6 * L], sv[6 * L:]
        hT, cT = sv[0], sv[1]
        sv = sv[2:]
        x16, sv = sv[:L], sv[L:]
        xs, sv = [None] + sv[:L - 1], sv[L - 1:]
        y, y16, gates, cseq, mean, rstd = (sv[i * L:(i + 1) * L] for i in range(6))
        c4, c4b = ctx.c4, ctx.c4b
        flat_saves = sv[6 * L:]
        if getattr(ctx, "consumed", False):
            raise RuntimeError("LSTMStack.backward ran twice on the same graph (retain_graph is not supported)")
        ctx.consumed = True
        P = [params[6 * l:6 * l + 6] for l in range(L)]
        ck = [_Chunks(B, lens) for lens in plan]
        dev = dout.device
        if BPTT_WAVEFRONT and BPTT_ONE_LAUNCH and C <= 8 and c4 and not c4b and _c4_bptt(H):
            return LSTMStack._backward_wave(ctx, dout, P, ck, hT, cT, x16, xs, y, y16, gates, cseq, mean, rstd)
        main = torch.cuda.current_stream(dev)
        side = _side_streams(dev)[0]
        side.wait_stream(main)
        g = ck[L].scatter(_c(dout))                           # d xs[L], chunk-major
        grads = [None] * (6 * L)
        hook = LSTMStack.collect_bwd
        recs = [None] * L
        for l in range(L - 1, -1, -1):
            k, kn = ck[l], ck[l + 1]
            if reductions[l]:
                gz = k.new(H, f32, dev)
                for c in range(C):
                    ops.time_reduce_bwd(kn.blk(g, c), k.lens[c], out=k.blk(gz, c))
                g = gz
            dz, dgamma, dbeta = ops.layernorm_bwd(g, y[l], xs[l], P[l][4], mean[l], rstd[l])
            if hook is not None:
                recs[l] = dict(dln=k.gather(g), dy=k.gather(dz))
            whhT16 = ops.transpose_to_bf16(_c(P[l][1]))
            dg16 = k.new(4 * H, bf16, dev)
            dh = dc = None
            if c4b:
                hprev = y16[l]                                # written by the forward kernel
                for c in range(C - 1, -1, -1):
                    gs, cs = flat_saves[2 * (l * C + c)], flat_saves[2 * (l * C + c) + 1]
                    _, dh, dc = ops.lstm_c4_bwd(k.blk(dz, c), gs, cs, cT[l, c - 1] if c else None, whhT16, dh, dc,
                                                out=k.blk(dg16, c))
            else:
                hprev = y16[l] if c4 else k.new(H, bf16, dev)  # c4 forward: h_{t-1} already written by the kernel
                one_launch = c4 and BPTT_ONE_LAUNCH and C <= 8
                if one_launch and _c4_bptt(H):                 # the kernel walks the chunk-major buffers itself
                    ops.lstm_c4_bwd_chunks(dz, gates[l], cseq[l], whhT16, k.lens, B, dg16)
                elif one_launch:
                    ops.lstm_tc_bwd_chunks(dz, gates[l], cseq[l], whhT16, k.lens, B, dg16)
                for c in (() if one_launch else range(C - 1, -1, -1)):
                    _, dh, dc = ops.lstm_tc_bwd(k.blk(dz, c), k.blk(gates[l], c), k.blk(cseq[l], c),
                                                cT[l, c - 1] if c else None, whhT16, dh, dc, out=k.blk(dg16, c))
                    if c4:
                        continue
                    hp, yc = k.blk(hprev, c), k.blk(y16[l], c)
                    hp[:, 1:] = yc[:, :-1]
                    if c:
                        hp[:, 0] = k.blk(y16[l], c - 1)[:, -1]
                    else:
                        hp[:, 0].zero_()
            # critical path to the next layer: d x = dG W_ih (+ dz: the LayerNorm residual branch, accumulated by the
            # GEMM's epilogue straight into dz)
            wih16 = ops.cast_bf16(_c(P[l][0]))
            M, I_l = dg16.shape[0], P[l][0].shape[1]
            if l > 0:
                g = ops.gemm_bf16(dg16, 0, wih16, 1, M, I_l, 4 * H, out=dz, accumulate=True, tag="gemm_bf16_nn",
                                  flags=ops.GEMM_FIXED_K)
            elif ctx.needs_input_grad[0]:
                g = ops.gemm_bf16(dg16, 0, wih16, 1, M, I_l, 4 * H, tag="gemm_bf16_nn")
            else:
                g = None
            if hook is not None:
                recs[l].update(dg16=k.gather(dg16), dxs=k.gather(g) if l > 0 else None)
            # off the critical path: the weight / bias gradients of this layer run on a side stream under the BPTT
            # recurrence of the next layer (which leaves 20 SMs idle and the tensor pipe nearly so)
            ready = torch.cuda.Event()
            ready.record(main)
            with torch.cuda.stream(side):
                side.wait_event(ready)
                grads[6 * l + 0] = ops.mm_tn(dg16, x16[l], "bf16", dy16=dg16, x16=x16[l])
                grads[6 * l + 1] = ops.mm_tn(dg16, hprev, "bf16", dy16=dg16, x16=hprev)
                db = ops.colsum(dg16)
                grads[6 * l + 2], grads[6 * l + 3] = db, db.clone()
                for t_ in (dg16, hprev):
                    t_.record_stream(side)
                for t_ in grads[6 * l:6 * l + 4]:
                    t_.record_stream(main)
            grads[6 * l + 4], grads[6 * l + 5] = dgamma, dbeta
        main.wait_stream(side)
        if hook is not None:
            hook.extend(recs)
        dxin = ck[0].gather(g) if g is not None else None
        return (dxin, None, *grads)

    @staticmethod
    def _backward_wave(ctx, dout, P, ck, hT, cT, x16, xs, y, y16, gates, cseq, mean, rstd):
        """The backward pass in reverse time, in groups of BPTT_GROUP consecutive time chunks of the forward's plan:
        group (l, q), q = NG-1 .. 0, runs its BPTT in one launch over the group's chunk segments with the (dh, dc) carry
        of group q+1.  Its input dz_l[q] is prepared on prep[l % 2] as soon as layer l+1 has finished group q: the dgrad
        GEMM of layer l+1's rows of the group accumulated into dz_{l+1} (the residual branch), TimeReduction backward,
        the dz pass of the LayerNorm backward.  Every BPTT launch runs on one stream, in the order of the diagonals of
        forward's wavefront, so the inputs of layer l are prepared under the recurrence of layer l+1 and the recurrences
        follow each other without a gap.  (Two layers' recurrences at once, as in the forward, would need two grids of a
        BPTT kernel co-resident at H = 1024: the clusters-of-16 kernel fits 14 clusters where two grids need 16, and a
        clusters-of-8 variant 30 where two need 32, on an H100 SXM -- DESIGN.md section 4a.)  The dgrad GEMM runs in the
        co-resident configuration, beside the BPTT grid's CTAs on every SM instead of on the few SMs it leaves free.
        Every kernel computes what the serial schedule's does on a row block (the dgrad GEMMs of both sum each element's
        K in one order, the LayerNorm's parameter pass runs once per layer over all rows), so the gradients are the same
        bits.  The weight, bias and LayerNorm parameter gradients wait for layer 1's last group and run under the
        recurrence of layer 0: earlier, they slow down the recurrences they run beside.  All cross-stream dependencies
        are events; one BPTT grid is in flight at a time, and it completes once all its own CTAs are resident."""
        reductions, eps, plan = ctx.cfg
        B, T, I0, H, L, C = ctx.dims
        dev = dout.device
        main = torch.cuda.current_stream(dev)
        st = _wave_bwd_streams(dev)
        rec, prep, wgs = st[0], st[1:3], st[3]
        gtop = ck[L].scatter(_c(dout))                       # d xs[L], chunk-major
        whhT16 = [ops.transpose_to_bf16(_c(p[1])) for p in P]
        wihT16 = [ops.transpose_to_bf16(_c(p[0])) for p in P]
        for s_ in st:
            s_.wait_stream(main)
        dz = [ck[l].new(H, f32, dev) for l in range(L)]      # LayerNorm dz; layer l > 0: + the dgrad GEMM = d xs[l]
        gz = [ck[l].new(H, f32, dev) if reductions[l] else None for l in range(L)]
        dg16 = [ck[l].new(4 * H, bf16, dev) for l in range(L)]
        hook = LSTMStack.collect_bwd
        dyc = [ck[l].new(H, f32, dev) for l in range(L)] if hook is not None else None
        # units of the schedule: groups of BPTT_GROUP consecutive chunks, one BPTT launch each (it walks their segments)
        G = [list(range(max(0, e - BPTT_GROUP), e)) for e in range(C, 0, -BPTT_GROUP)][::-1]
        NG = len(G)
        ev = lambda: torch.cuda.Event()
        prep_done = [[ev() for _ in range(NG)] for _ in range(L)]
        rec_done = [[ev() for _ in range(NG)] for _ in range(L)]
        carry = [(None, None)] * L
        grads = [None] * (6 * L)
        wg = []
        for d in range(L + NG - 1):
            for l in range(L - 1, -1, -1):
                q = NG - 1 - (d - (L - 1 - l))
                if not 0 <= q < NG:
                    continue
                k, kn = ck[l], ck[l + 1]
                c0, c1 = G[q][0], G[q][-1] + 1
                a, b = k.B * k.off[c0], k.B * k.off[c1]       # rows of the group on layer l's axis
                with torch.cuda.stream(prep[l % 2]):
                    if l + 1 < L:
                        prep[l % 2].wait_event(rec_done[l + 1][q])
                        an, bn = kn.B * kn.off[c0], kn.B * kn.off[c1]
                        # the co-resident configuration shares the SMs of the running BPTT grid; the same bits as the
                        # serial schedule's whole-layer GEMM (both sum each element's K in one order)
                        ops.gemm_bf16(dg16[l + 1][an:bn], 0, wihT16[l + 1], 0, bn - an, H, 4 * H, out=dz[l + 1][an:bn],
                                      accumulate=True, tag="gemm_bf16_nn", flags=ops.GEMM_CORESIDENT)
                        gin = dz[l + 1]
                    else:
                        gin = gtop
                    if reductions[l]:
                        for c in G[q]:
                            ops.time_reduce_bwd(kn.blk(gin, c), k.lens[c], out=k.blk(gz[l], c))
                    gl = gz[l] if reductions[l] else gin
                    ops.layernorm_bwd_dz(gl[a:b], y[l][a:b], xs[l][a:b] if l else None, P[l][4], mean[l][a:b],
                                         rstd[l][a:b], out=dz[l][a:b])
                    if dyc is not None:
                        # the copy is ordered before prep_done[l][q]; the BPTT of the group waits for that event and the
                        # dgrad GEMM of layer l-1 that adds into these rows waits for rec_done[l][q], recorded after it
                        dyc[l][a:b].copy_(dz[l][a:b])
                    prep_done[l][q].record(prep[l % 2])
                with torch.cuda.stream(rec):
                    rec.wait_event(prep_done[l][q])
                    _, dh, dc = ops.lstm_c4_bwd_chunks(dz[l][a:b], gates[l][a:b], cseq[l][a:b], whhT16[l],
                                                       k.lens[c0:c1], B, dg16[l][a:b], cT[l, c0 - 1] if c0 else None,
                                                       *carry[l])
                    carry[l] = (dh, dc)
                    rec_done[l][q].record(rec)
                if q == 0:
                    wg.append((l, gl))
        # off the critical path: the weight, bias and LayerNorm parameter gradients, once layers L-1 .. 1 are done (under
        # the recurrence of layer 0; earlier they would slow the recurrence of the layers they wait for)
        with torch.cuda.stream(wgs):
            for l, gl in wg:
                wgs.wait_event(rec_done[min(l, 1)][0])
                grads[6 * l + 0] = ops.mm_tn(dg16[l], x16[l], "bf16", dy16=dg16[l], x16=x16[l])
                grads[6 * l + 1] = ops.mm_tn(dg16[l], y16[l], "bf16", dy16=dg16[l], x16=y16[l])
                db = ops.colsum(dg16[l])
                grads[6 * l + 2], grads[6 * l + 3] = db, db.clone()
                grads[6 * l + 4], grads[6 * l + 5] = ops.layernorm_bwd_params(gl, y[l], xs[l], mean[l], rstd[l])
        for s_ in st:
            main.wait_stream(s_)
        for t_ in grads:
            t_.record_stream(main)
        g = None
        if ctx.needs_input_grad[0]:
            g = ops.gemm_bf16(dg16[0], 0, ops.cast_bf16(_c(P[0][0])), 1, dg16[0].shape[0], I0, 4 * H, tag="gemm_bf16_nn")
        if hook is not None:
            gls = dict(wg)
            hook.extend(dict(dln=ck[l].gather(gls[l]), dy=ck[l].gather(dyc[l]), dg16=ck[l].gather(dg16[l]),
                             dxs=ck[l].gather(dz[l]) if l else None) for l in range(L))
        dxin = ck[0].gather(g) if g is not None else None
        return (dxin, None, *grads)


def _fused_lse(precision, J, U):
    """bf16 mode takes the softmax statistics from the logits GEMM's epilogue when its tiles allow it."""
    return precision == "bf16" and FUSE_JOINT_LSE and J % 8 == 0 and U <= 1024


def joint_align(h_enc, h_dec, w1, b1, w2, b2, labels, act_lens, label_lens, blank, precision):
    """Transducer.align's joint: the logits and the loss workspace exactly as JointLoss.forward makes them, then the
    Viterbi alignment over it (ops.rnnt_viterbi).  The logits are freed before the alignment runs."""
    B, T, _ = h_enc.shape
    U = h_dec.shape[1]
    J = w1.shape[0]
    _, _, ep, dp = _joint_pre(h_enc, h_dec, w1, b1, precision)
    hid2 = ops.joint_hidden_fwd(ep, dp, precision == "bf16").view(B * T * U, J)
    del ep, dp
    if _fused_lse(precision, J, U):
        b2a = b2 if (b2.is_contiguous() and b2.data_ptr() % 16 == 0) else b2.clone()
        logits, ws = ops.joint_logits_lse(hid2, ops.cast_bf16(w2.contiguous()), b2a, labels, act_lens, label_lens,
                                          B, T, U, blank)
    else:
        logits = ops.mm_nt(hid2, w2, b2, precision, x16=hid2 if precision == "bf16" else None).view(B, T, U, -1)
        _, ws = ops.rnnt_loss_fwd(logits, labels, act_lens, label_lens, blank, need_beta=False)
    del logits, hid2
    return ops.rnnt_viterbi(act_lens, label_lens, B, T, U, ws, torch.float32)


def _joint_pre(h_enc, h_dec, w1, b1, precision):
    """ep = W1[:, :E] h_enc + b1, dp = W1[:, E:] h_dec  -- exact split of Linear(cat[e, d])."""
    B, T, E = h_enc.shape
    U, Dd = h_dec.shape[1], h_dec.shape[2]
    J = w1.shape[0]
    he2, hd2 = _c(h_enc).view(B * T, E), _c(h_dec).view(B * U, Dd)
    ep = ops.mm_nt(he2, w1[:, :E], b1, precision).view(B, T, J)
    dp = ops.mm_nt(hd2, w1[:, E:], None, precision).view(B, U, J)
    return he2, hd2, ep, dp


JOINT_WGRAD_SIDE = __import__("os").environ.get("EDGEDICT_JOINT_WGRAD_SIDE", "1") != "0"


def _joint_bwd(ctx_p, dlog2, hid, he2, hd2, w1, w2, dims, db2=None, band=None):
    """Shared backward of the joint given d logits [N_rows, V] (fp32 or bf16); db2 may already have
    been accumulated by the fused loss-gradient kernel.  band = (xlen, ylen, s_begin): the rows are the pruned loss's
    band rows (hid [B, T, R, J]), reduced onto ep / dp by the banded reduction."""
    B, T, U, E, Dd, J, V = dims
    p = ctx_p
    dl16 = dlog2 if dlog2.dtype == bf16 else (ops.cast_bf16(dlog2) if p == "bf16" else None)
    hid2 = hid.view(-1, J)

    def out_layer_grads(db2):
        if db2 is None:
            db2 = ops.colsum(dlog2)
        if p == "bf16" and V % 256 == 0:
            # compute dW2^T = hidden^T dlogits ([J, V]: 256-wide GEMM tiles divide V, not J) and flip it
            dw2 = ops.mm_tn(hid2, dl16, p, dy16=hid2, x16=dl16).t().contiguous()
        else:
            dw2 = ops.mm_tn(dlog2, hid2, p, dy16=dl16, x16=hid2 if p == "bf16" else None)
        return dw2, db2

    side = None
    if JOINT_WGRAD_SIDE and p == "bf16" and dlog2.is_cuda:
        # the output layer's weight gradient (the split-K dW2 GEMM, and the 4.2 GB column sum for db2 unless the loss
        # gradient already produced it) is off the critical path to the encoder: it runs on a side stream under the
        # d-hidden GEMM and the d-pre reductions
        main = torch.cuda.current_stream(dlog2.device)
        side = _side_streams(dlog2.device)[1]
        side.wait_stream(main)
        with torch.cuda.stream(side):
            dw2, db2 = out_layer_grads(db2)
        for t_ in (dlog2, dl16, hid2):
            if t_ is not None:
                t_.record_stream(side)
    else:
        dw2, db2 = out_layer_grads(db2)
    if p == "bf16" and J % 8 == 0 and hid.dtype == bf16:
        # tanh' applied in the d-hidden GEMM's epilogue: d(pre-activation) leaves the GEMM, then two pure reductions
        dpre = ops.gemm_bf16_dtanh(dl16, ops.cast_bf16(w2.contiguous()), True, hid2, hid2.shape[0], J, V)
        if band is None:
            dep, ddp = ops.joint_dpre_reduce(dpre.view(B, T, U, J))
        else:
            dep, ddp = ops.joint_band_dpre_reduce(dpre.view(hid.shape), None, *band, U)
    else:
        dhid = ops.mm_nn(dlog2, w2, p, dy16=dl16, out_bf16=(p == "bf16"))
        if band is None:
            dep, ddp = ops.joint_hidden_bwd(dhid.view(B, T, U, J), hid)
        else:
            dep, ddp = ops.joint_band_dpre_reduce(dhid.view(hid.shape), hid, *band, U)
    dep2, ddp2 = dep.view(B * T, J), ddp.view(B * U, J)
    w1e, w1d = w1[:, :E], w1[:, E:]
    dhe = ops.mm_nn(dep2, w1e, p).view(B, T, E)
    dhd = ops.mm_nn(ddp2, w1d, p).view(B, U, Dd)
    dw1 = torch.empty_like(w1)
    dw1[:, :E] = ops.mm_tn(dep2, he2, p)
    dw1[:, E:] = ops.mm_tn(ddp2, hd2, p)
    db1 = ops.colsum(dep2)
    if side is not None:
        main.wait_stream(side)
        dw2.record_stream(main)
        db2.record_stream(main)
    return dhe, dhd, dw1, db1, dw2, db2


class JointLogits(torch.autograd.Function):
    """Joint.forward on [B,T,E] x [B,U,D] -> logits [B,T,U,V] (rnnt/models.py:169-179)."""

    @staticmethod
    def forward(ctx, h_enc, h_dec, w1, b1, w2, b2, precision):
        B, T, E = h_enc.shape
        U, Dd = h_dec.shape[1], h_dec.shape[2]
        J, V = w1.shape[0], w2.shape[0]
        he2, hd2, ep, dp = _joint_pre(h_enc, h_dec, w1, b1, precision)
        hid = ops.joint_hidden_fwd(ep, dp, precision == "bf16")
        logits = ops.mm_nt(hid.view(B * T * U, J), w2, b2, precision, x16=hid.view(B * T * U, J) if precision == "bf16" else None)
        ctx.save_for_backward(hid, he2, hd2, w1, w2)
        ctx.precision, ctx.dims = precision, (B, T, U, E, Dd, J, V)
        return logits.view(B, T, U, V)

    @staticmethod
    def backward(ctx, dlogits):
        hid, he2, hd2, w1, w2 = ctx.saved_tensors
        B, T, U, E, Dd, J, V = ctx.dims
        dl2 = _c(dlogits).view(B * T * U, V)
        dhe, dhd, dw1, db1, dw2, db2 = _joint_bwd(ctx.precision, dl2, hid, he2, hd2, w1, w2, ctx.dims)
        return dhe, dhd, dw1, db1, dw2, db2, None


def check_fastemit_lambda(value):
    """FastEmit's lambda as a float: a real number (TypeError otherwise) that is finite and >= 0 (ValueError)."""
    if isinstance(value, bool) or not isinstance(value, numbers.Real):
        raise TypeError("fastemit_lambda must be a real number, got %s" % type(value).__name__)
    lam = float(value)
    if not math.isfinite(lam) or lam < 0:
        raise ValueError("fastemit_lambda must be finite and >= 0, got %r" % lam)
    return lam


class RNNTLossFn(torch.autograd.Function):
    """warprnnt_pytorch._RNNT (pytorch_binding/warprnnt_pytorch/__init__.py:10-50) on CUDA logits:
    costs stay on the device, the gradient kernel runs in backward with the upstream gradient
    folded in (the reference computes it eagerly and rescales it in a second pass).
    fastemit_lambda > 0 gives backward the FastEmit gradient (include/edgedict_b200.h, eb_rnnt_loss_bwd_fe); the
    costs are the plain negative log-likelihoods whatever it is."""

    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens, blank, reduction, fastemit_lambda=0.0):
        ctx.fastemit_lambda = check_fastemit_lambda(fastemit_lambda)
        acts = _c(acts)
        costs, ws = ops.rnnt_loss_fwd(acts, labels, act_lens, label_lens, blank, need_beta=True)
        B = acts.shape[0]
        ctx.save_for_backward(acts, labels, act_lens, label_lens, ws)
        ctx.blank, ctx.reduction, ctx.B = blank, reduction, B
        if reduction in ("sum", "mean"):
            costs = costs.sum().unsqueeze(-1)
            if reduction == "mean":
                costs = costs / B
        return costs

    @staticmethod
    def backward(ctx, go):
        acts, labels, act_lens, label_lens, ws = ctx.saved_tensors
        scale = 1.0 / ctx.B if ctx.reduction == "mean" else 1.0
        g = _c(go.to(acts.dtype)).view(-1)
        grads = ops.rnnt_loss_bwd(acts, labels, act_lens, label_lens, ctx.blank, ws, g, scale,
                                  fastemit_lambda=ctx.fastemit_lambda)
        return grads, None, None, None, None, None, None


class LogSoftmax(torch.autograd.Function):
    """nn.LogSoftmax(dim=-1) of CTCEncoder.tovocab (rnnt/models.py:284-287), fp32 in every precision mode."""

    @staticmethod
    def forward(ctx, x):
        y = ops.log_softmax_fwd(_c(x))
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        return ops.log_softmax_bwd(_c(dy), y)


class LMLoss(torch.autograd.Function):
    """nn.NLLLoss(ignore_index, reduction)(F.log_softmax(x W^T + b), targets) -- the reference LMModel's decoder and
    log-softmax (models.py:224-261) under cli/train_lm.py's criterion -- as one node: the log-probs are never written.
    bf16 mode: the logits GEMM writes bf16 logits and takes each row's log-sum-exp and target logit from its fp32
    accumulators (ops.lm_logits_ce); fp32 mode: the fp32 GEMM and a row pass (ops.lm_ce_rows).  The loss kernel sums
    the costs and counts the targets on the device; backward writes d logits over the saved logits (bf16 or fp32) and
    runs the three GEMMs of Linear.  x [M, K], targets [M] int32 / int64.  reduction "mean" / "sum" -> [], "none" -> the
    per-token costs [M] (0 at ignored targets).  A target outside [0, V) that is not ignore_index gives a NaN cost."""

    @staticmethod
    def forward(ctx, x, w, b, targets, ignore_index, reduction, precision):
        M, K = x.shape
        V = w.shape[0]
        targets = _c(targets)
        if precision == "bf16":
            x16 = ops.cast_bf16(_c(x))
            ba = b if (b is None or (b.is_contiguous() and b.data_ptr() % 16 == 0)) else b.clone()
            logits, lse, tl = ops.lm_logits_ce(x16, ops.cast_bf16(_c(w)), ba, targets)
            xs = x16
        else:
            xs = _c(x)
            logits = ops.mm_nt(xs, w, b, "fp32")
            lse, tl = ops.lm_ce_rows(logits, targets)
        cost, loss, scale = ops.lm_ce_loss(lse, tl, targets, ignore_index, V, reduction == "mean")
        ctx.save_for_backward(xs, w, logits, lse, targets, scale)
        ctx.meta = (precision, ignore_index, b is not None)
        return cost if reduction == "none" else loss

    @staticmethod
    def backward(ctx, go):
        xs, w, logits, lse, targets, scale = ctx.saved_tensors
        p, ignore_index, has_b = ctx.meta
        if getattr(ctx, "consumed", False):
            raise RuntimeError("LMLoss.backward ran twice on the same graph: the gradient is written in place over the "
                               "saved logits (retain_graph is not supported by this node)")
        ctx.consumed = True
        dl = ops.lm_ce_bwd(logits, lse, targets, ignore_index, _c(go.to(f32)).reshape(-1), scale, out=logits)
        dl16 = dl if p == "bf16" else None
        dx = ops.mm_nn(dl, w, p, dy16=dl16) if ctx.needs_input_grad[0] else None
        dw = ops.mm_tn(dl, xs, p, dy16=dl16, x16=xs if p == "bf16" else None) if ctx.needs_input_grad[1] else None
        db = ops.colsum(dl) if has_b and ctx.needs_input_grad[2] else None
        return dx, dw, db, None, None, None, None


class CTCLossFn(torch.autograd.Function):
    """Per-utterance CTC costs [N] of log_probs (T, N, V) (torch.nn.functional.ctc_loss with reduction='none'); the
    reductions are taken by the caller (edgedict_b200/ctc.py), and autograd hands their per-utterance factors to
    backward, where the gradient kernel applies them.  meta = (S, blank, zero_infinity)."""

    @staticmethod
    def forward(ctx, log_probs, targets, offsets, tlen, ilen, meta):
        S, blank, zero_inf = meta
        costs, ws = ops.ctc_loss_fwd(log_probs, targets, offsets, tlen, ilen, S, blank, zero_inf)
        ctx.save_for_backward(log_probs, tlen, ilen, ws)
        ctx.meta = meta
        return costs

    @staticmethod
    def backward(ctx, gcosts):
        log_probs, tlen, ilen, ws = ctx.saved_tensors
        S, blank, zero_inf = ctx.meta
        grad = ops.ctc_loss_bwd(log_probs, tlen, ilen, S, blank, zero_inf, ws, _c(gcosts.to(f32)))
        return grad, None, None, None, None, None


def _joint_loss_fwd(ctx, h_enc, h_dec, w1, b1, w2, b2, labels, act_lens, label_lens, blank, precision):
    """The joint and the RNN-T loss of JointLoss / JointCosts: costs [B] of the rows, with what backward needs saved
    on ctx."""
    B, T, E = h_enc.shape
    U, Dd = h_dec.shape[1], h_dec.shape[2]
    J, V = w1.shape[0], w2.shape[0]
    he2, hd2, ep, dp = _joint_pre(h_enc, h_dec, w1, b1, precision)
    hid = ops.joint_hidden_fwd(ep, dp, precision == "bf16")
    hid2 = hid.view(B * T * U, J)
    fused = _fused_lse(precision, J, U)
    if fused:
        # bf16 mode: the logits GEMM epilogue also produces the softmax statistics (fp32, from the
        # register accumulators) and writes bf16 logits; the denominator pass over 8 GB disappears
        b2a = b2 if (b2.is_contiguous() and b2.data_ptr() % 16 == 0) else b2.clone()
        logits, ws = ops.joint_logits_lse(hid2, ops.cast_bf16(w2.contiguous()), b2a, labels, act_lens,
                                          label_lens, B, T, U, blank)
        costs = ops.rnnt_lattice(act_lens, label_lens, B, T, U, ws)
    else:
        logits = ops.mm_nt(hid2, w2, b2, precision, x16=hid2 if precision == "bf16" else None).view(B, T, U, V)
        costs, ws = ops.rnnt_loss_fwd(logits, labels, act_lens, label_lens, blank, need_beta=True)
    ctx.save_for_backward(hid, he2, hd2, w1, w2, logits, labels, act_lens, label_lens, ws)
    ctx.precision, ctx.dims, ctx.blank = precision, (B, T, U, E, Dd, J, V), blank
    return costs


def _joint_loss_bwd(ctx, g, host_scale, lam, node):
    """The gradients (h_enc, h_dec, w1, b1, w2, b2) of _joint_loss_fwd's costs, each row's scaled by g (one element:
    every row) times host_scale, written over the saved logits."""
    hid, he2, hd2, w1, w2, logits, labels, act_lens, label_lens, ws = ctx.saved_tensors
    if getattr(ctx, "consumed", False):
        raise RuntimeError("%s.backward ran twice on the same graph: the gradient is written in place over "
                           "the saved logits (retain_graph is not supported by this node)" % node)
    ctx.consumed = True
    B, T, U, E, Dd, J, V = ctx.dims
    p = ctx.precision
    db2 = None
    if logits.dtype == bf16 and V % 8 == 0:
        # the bias gradient comes out of the gradient kernel, which holds every d logit it writes: the output layer's
        # side stream is left with dW2 alone
        dl, db2 = ops.rnnt_loss_bwd_bf16_db(logits, labels, act_lens, label_lens, ctx.blank, ws, g, host_scale,
                                            fastemit_lambda=lam)
    elif logits.dtype == bf16:
        dl = ops.rnnt_loss_bwd_bf16(logits, labels, act_lens, label_lens, ctx.blank, ws, g, host_scale,
                                    fastemit_lambda=lam)
    elif p == "bf16":
        dl = ops.rnnt_loss_bwd(logits, labels, act_lens, label_lens, ctx.blank, ws, g, host_scale, out_bf16=True,
                               fastemit_lambda=lam)
    else:
        dl = ops.rnnt_loss_bwd(logits, labels, act_lens, label_lens, ctx.blank, ws, g, host_scale, out=logits,
                               fastemit_lambda=lam)
    return _joint_bwd(p, dl.view(B * T * U, V), hid, he2, hd2, w1, w2, ctx.dims, db2)


class JointLoss(torch.autograd.Function):
    """Transducer.forward's joint + loss (rnnt/models.py:234-239) as one autograd node: logits are
    produced, consumed by the loss, and their gradient is written IN PLACE over them (fp32 mode)
    or straight to bf16 (bf16 mode) -- no autograd copy of the 8 GB tensor is ever made.
    fastemit_lambda > 0: every backward branch writes the FastEmit gradient; the loss and costs do not change."""

    @staticmethod
    def forward(ctx, h_enc, h_dec, w1, b1, w2, b2, labels, act_lens, label_lens, blank, precision, fastemit_lambda=0.0):
        ctx.fastemit_lambda = check_fastemit_lambda(fastemit_lambda)
        costs = _joint_loss_fwd(ctx, h_enc, h_dec, w1, b1, w2, b2, labels, act_lens, label_lens, blank, precision)
        ctx.mark_non_differentiable(costs)
        loss = costs.sum().unsqueeze(-1) / h_enc.shape[0]
        ctx.costs = costs
        return loss, costs

    @staticmethod
    def backward(ctx, go, _gc):
        g = _c(go.to(f32)).view(-1)
        grads = _joint_loss_bwd(ctx, g, 1.0 / ctx.dims[0], ctx.fastemit_lambda, "JointLoss")
        return (*grads, None, None, None, None, None, None)


class JointCosts(torch.autograd.Function):
    """JointLoss's joint + loss with the per-row costs [B] as the differentiable output: backward hands each row's
    upstream gradient to the loss-gradient kernel as its per-utterance scale (what minimum word error rate training
    needs, whose rows are weighted by their posteriors).  No FastEmit: on negatively weighted rows it regularises
    nothing."""

    @staticmethod
    def forward(ctx, h_enc, h_dec, w1, b1, w2, b2, labels, act_lens, label_lens, blank, precision):
        return _joint_loss_fwd(ctx, h_enc, h_dec, w1, b1, w2, b2, labels, act_lens, label_lens, blank, precision)

    @staticmethod
    def backward(ctx, gcosts):
        grads = _joint_loss_bwd(ctx, _c(gcosts.to(f32)).view(-1), 1.0, 0.0, "JointCosts")
        return (*grads, None, None, None, None, None)


class ExpectedRisk(torch.autograd.Function):
    """The expected risk of N-best lists (ops.mwer_risk_fwd): costs [B, N] fp32 (-log P of each hypothesis), errors
    and valid int32 [B, N] -> (loss [1] = mean over utterances of sum_i P_i (E_i - mean E), P the posteriors
    renormalised over the valid ranks [B, N], not differentiable).  The gradient reaches the costs alone."""

    @staticmethod
    def forward(ctx, costs, errors, valid):
        costs = _c(costs)
        loss, post, _ = ops.mwer_risk_fwd(costs, errors, valid)
        ctx.save_for_backward(costs, errors, valid)
        ctx.mark_non_differentiable(post)
        return loss, post

    @staticmethod
    def backward(ctx, gloss, _gpost):
        costs, errors, valid = ctx.saved_tensors
        return ops.mwer_risk_bwd(costs, errors, valid, gloss), None, None


class SimpleLoss(torch.autograd.Function):
    """The pruned RNN-T loss's trivial joiner (Kuang et al., Interspeech 2022): am [B, T, V], lm [B, U, V] fp32 ->
    costs [B] of the RNN-T lattice on log softmax(am[t] + lm[u]), and the loss workspace (alpha, beta, statistics)
    that the band choice reads (ops.rnnt_band_choice).  The workspace takes no gradient."""

    @staticmethod
    def forward(ctx, am, lm, labels, act_lens, label_lens, blank):
        am, lm = _c(am), _c(lm)
        costs, ws, scratch = ops.rnnt_simple_fwd(am, lm, labels, act_lens, label_lens, blank)
        ctx.save_for_backward(am, lm, labels, act_lens, label_lens, ws, scratch)
        ctx.blank = blank
        ctx.mark_non_differentiable(ws)
        return costs, ws

    @staticmethod
    def backward(ctx, gcosts, _gws):
        am, lm, labels, act_lens, label_lens, ws, scratch = ctx.saved_tensors
        dam, dlm = ops.rnnt_simple_bwd(am, lm, labels, act_lens, label_lens, ctx.blank, ws, scratch,
                                       _c(gcosts.to(f32)), 1.0)
        return dam, dlm, None, None, None, None


class RNNTBandLossFn(torch.autograd.Function):
    """The RNN-T loss restricted to bands: logits [B, T, R, V] fp32 of the band rows given by s_begin / nopath
    (ops.rnnt_band_choice) -> costs [B]; the cells outside the bands are dead ends of the lattice."""

    @staticmethod
    def forward(ctx, logits, labels, act_lens, label_lens, s_begin, nopath, U, blank):
        logits = _c(logits)
        costs, ws = ops.rnnt_band_loss_fwd(logits, labels, act_lens, label_lens, s_begin, nopath, U, blank)
        ctx.save_for_backward(logits, labels, act_lens, label_lens, s_begin, nopath, ws)
        ctx.U, ctx.blank = U, blank
        return costs

    @staticmethod
    def backward(ctx, gcosts):
        logits, labels, act_lens, label_lens, s_begin, nopath, ws = ctx.saved_tensors
        dl = ops.rnnt_band_loss_bwd(logits, labels, act_lens, label_lens, s_begin, nopath, ctx.U, ctx.blank, ws,
                                    _c(gcosts.to(f32)), 1.0)
        return dl, None, None, None, None, None, None, None


class PrunedJointLoss(torch.autograd.Function):
    """JointLoss on the pruned loss's band rows: the joint hidden, logits, statistics and gradient of the B*T*R rows
    (b, t, r) at cell (t, s_begin[b,t] + r) only.  bf16 mode takes the statistics from the logits GEMM's epilogue and
    writes the bf16 d logits and the bias gradient in place (JointLoss's fused branch); fp32 mode writes the gradient
    in place over the fp32 logits.  The backward is _joint_bwd's over the band rows, with the banded reduction."""

    @staticmethod
    def forward(ctx, h_enc, h_dec, w1, b1, w2, b2, s_begin, nopath, R, labels, act_lens, label_lens, blank, precision):
        B, T, E = h_enc.shape
        U, Dd = h_dec.shape[1], h_dec.shape[2]
        J, V = w1.shape[0], w2.shape[0]
        if precision == "bf16" and J % 8:
            raise ValueError("the pruned joint in bf16 mode needs joint_size % 8 == 0, got %d" % J)
        he2, hd2, ep, dp = _joint_pre(h_enc, h_dec, w1, b1, precision)
        hid = ops.joint_band_hidden_fwd(ep, dp, act_lens, label_lens, s_begin, R, precision == "bf16")
        del ep, dp
        hid2 = hid.view(-1, J)
        if _fused_lse(precision, J, U) and V % 8 == 0:
            # bf16 mode: the statistics come out of the logits GEMM's epilogue, as in JointLoss
            b2a = b2 if (b2.is_contiguous() and b2.data_ptr() % 16 == 0) else b2.clone()
            logits, costs, ws = ops.joint_band_logits_lse(hid, ops.cast_bf16(w2.contiguous()), b2a, labels, act_lens,
                                                          label_lens, s_begin, nopath, U, blank)
        else:
            logits = ops.mm_nt(hid2, w2, b2, precision, x16=hid2 if precision == "bf16" else None).view(B, T, R, V)
            costs, ws = ops.rnnt_band_loss_fwd(logits, labels, act_lens, label_lens, s_begin, nopath, U, blank)
        ctx.save_for_backward(hid, he2, hd2, w1, w2, logits, labels, act_lens, label_lens, s_begin, nopath, ws)
        ctx.precision, ctx.dims, ctx.blank = precision, (B, T, U, E, Dd, J, V), blank
        ctx.mark_non_differentiable(costs)
        return costs.sum().unsqueeze(-1) / B, costs

    @staticmethod
    def backward(ctx, go, _gc):
        hid, he2, hd2, w1, w2, logits, labels, act_lens, label_lens, s_begin, nopath, ws = ctx.saved_tensors
        if getattr(ctx, "consumed", False):
            raise RuntimeError("PrunedJointLoss.backward ran twice on the same graph: the gradient is written in place "
                               "over the saved logits (retain_graph is not supported by this node)")
        ctx.consumed = True
        B, T, U, E, Dd, J, V = ctx.dims
        p = ctx.precision
        g = _c(go.to(f32)).view(-1)
        db2 = None
        if logits.dtype == bf16:
            dl, db2 = ops.rnnt_band_loss_bwd_bf16_db(logits, labels, act_lens, label_lens, s_begin, nopath, U, ctx.blank,
                                                     ws, g, 1.0 / B)
        elif p == "bf16":
            dl = ops.rnnt_band_loss_bwd(logits, labels, act_lens, label_lens, s_begin, nopath, U, ctx.blank, ws, g,
                                        1.0 / B, out_bf16=True)
        else:
            dl = ops.rnnt_band_loss_bwd(logits, labels, act_lens, label_lens, s_begin, nopath, U, ctx.blank, ws, g,
                                        1.0 / B, out=logits)
        dhe, dhd, dw1, db1, dw2, db2 = _joint_bwd(p, dl.view(-1, V), hid, he2, hd2, w1, w2, ctx.dims, db2,
                                                  band=(act_lens, label_lens, s_begin))
        return dhe, dhd, dw1, db1, dw2, db2, None, None, None, None, None, None, None, None


def conv_out_len(T, k, s):
    """Output length of a FrontEnd conv (pad k - 1 on both sides, stride s, the last k - 1 outputs dropped)."""
    return (T + k - 2) // s + 2 - k


class FrontEndStack(torch.autograd.Function):
    """FrontEnd.forward (rnnt/models.py:348-360) channels-last: the first conv (C_in = 1), then per DilatedConvBlock
    (rnnt/models.py:319-334) conv(GroupNorm(1, C_in)(GELU(y))) with the trim, then LayerNorm(C_last).

    spec = (first, blocks, ln_eps): first = (k, s, C, has_bias) or None (then x is a [B, T, C] block input, which takes
    a gradient), blocks = ((k, s, C_in, C_out, has_bias, gn_eps), ...), ln_eps = the LayerNorm's eps or None (no
    LayerNorm).  params in that order: first w [, b]; per block conv w [, b], gn weight, gn bias; ln weight, ln bias.

    Each strided conv reads a padded operand buffer (csrc/conv.cu) that the GroupNorm pass writes; the backward
    rebuilds it from the saved conv outputs and per-utterance statistics instead of keeping it."""

    @staticmethod
    def forward(ctx, x, spec, precision, *params):
        first, blocks, ln_eps = spec
        bf = precision == "bf16"
        B = x.shape[0]
        it = iter(params)
        saves, meta = [], []
        if first is not None:
            k, s, C, hb = first
            w0 = next(it)
            b0 = next(it) if hb else None
            T = conv_out_len(x.shape[1], k, s)
            y = ops.conv1d_first_fwd(x, _c(w0.view(C, k)), b0, k, s, T)
        else:
            y, T, C = x, x.shape[1], x.shape[2]
        ustride = T * C
        for (k, s, Cin, Cout, hb, eps) in blocks:
            w = next(it)
            b = next(it) if hb else None
            g, be = next(it), next(it)
            mean, rstd = ops.gn_stats(y, ustride, B, T, Cin, eps)
            Q = (k - 1 + T + s - 1) // s
            rows = B * Q + (k + s - 1) // s
            xp = torch.empty(rows * s * Cin, dtype=bf16 if bf else f32, device=x.device)
            ops.gn_apply(y, ustride, B, T, Cin, mean, rstd, g, be, xp, k - 1, Q * s)
            wp = w.permute(0, 2, 1).contiguous()                       # [C_out, k, C_in]
            yo = torch.empty(B * Q, Cout, dtype=f32, device=x.device)
            if bf:
                ops.conv1d_bf16(xp, 0, rows, s, Cin, 0, ops.cast_bf16(wp), k, Cout, b, yo, 0, Cout, B * Q)
            else:
                ops.gemm_f32_at(xp, 0, s * Cin, 1, wp, 1, k * Cin, yo, 0, Cout, B * Q, Cout, k * Cin, bias=b)
            saves.append((y, mean, rstd))
            meta.append((ustride, T))
            y, ustride, T, C = yo, Q * Cout, conv_out_len(T, k, s), Cout
        out = y.view(B, -1, C)[:, :T].contiguous()
        ctx.meta, ctx.spec, ctx.precision, ctx.B, ctx.nparams = meta, spec, precision, B, len(params)
        ln_saves = ()
        if ln_eps is not None:
            lw, lb = next(it), next(it)
            pre_ln = out
            out, _, lm, lr = ops.layernorm_fwd(pre_ln, None, lw, lb, ln_eps)
            ln_saves = (pre_ln, lm, lr)
        ctx.save_for_backward(x, *params, *[t for blk in saves for t in blk], *ln_saves)
        return out

    @staticmethod
    def backward(ctx, dout):
        first, blocks, ln_eps = ctx.spec
        bf = ctx.precision == "bf16"
        B, n = ctx.B, ctx.nparams
        st = ctx.saved_tensors
        first_in, params = st[0], st[1:1 + n]
        saves = [(st[1 + n + 3 * i],) + ctx.meta[i] + st[2 + n + 3 * i:4 + n + 3 * i] for i in range(len(blocks))]
        dev = dout.device
        grads = [None] * len(params)
        # parameter index of each piece
        idx = 0
        if first is not None:
            i_first = idx
            idx += 2 if first[3] else 1
        i_blocks = []
        for blk in blocks:
            i_blocks.append(idx)
            idx += 4 if blk[4] else 3
        dz = _c(dout)
        if ln_eps is not None:
            pre_ln, lm, lr = st[1 + n + 3 * len(blocks):]
            dz, grads[idx], grads[idx + 1] = ops.layernorm_bwd(dz, pre_ln, None, params[idx], lm, lr)
        C = dz.shape[-1]
        dx_in = None
        # the gradient of the last conv output in the layout of its dY buffer: [lead + B*Q, C_out], zero rows besides
        # the T_out valid ones of each utterance, lead = k - 1 zero rows in front (the dX phase GEMMs read above row 0)
        db_next = None
        if blocks:
            k, s, Cin, Cout, hb, _ = blocks[-1]
            T = saves[-1][2]
            Q, To = (k - 1 + T + s - 1) // s, conv_out_len(T, k, s)
            dyb = torch.zeros((k - 1 + B * Q) * Cout, dtype=f32, device=dev)
            dyb[(k - 1) * Cout:].view(B, Q, Cout)[:, :To] = dz
            dy16 = ops.cast_bf16(dyb) if bf else None
            dy32 = dyb
            db_next = ops.colsum(dz.view(-1, Cout)) if hb else None
        for bi in range(len(blocks) - 1, -1, -1):
            k, s, Cin, Cout, hb, _ = blocks[bi]
            y, ustride, T, mean, rstd = saves[bi]
            pi = i_blocks[bi]
            w = params[pi]
            gi = pi + (2 if hb else 1)
            g, be = params[gi], params[gi + 1]
            if hb:
                grads[pi + 1] = db_next
            Q = (k - 1 + T + s - 1) // s
            rows = B * Q + (k + s - 1) // s
            lead = (k - 1) * Cout
            xp = torch.empty(rows * s * Cin, dtype=bf16 if bf else f32, device=dev)
            ops.gn_apply(y, ustride, B, T, Cin, mean, rstd, g, be, xp, k - 1, Q * s)
            # dW[n, j, c] = sum_m dY[m, n] X[m*s + j, c]
            if bf:
                nd = (k + s - 1) // s
                parts = [ops.gemm_bf16(dy16[lead:], 1, xp[d * s * Cin:], 1, Cout, s * Cin, B * Q) for d in range(nd)]
                dwp = torch.cat(parts, 1)[:, :k * Cin]
            else:
                dwp = ops.gemm_f32_rows(dy32, lead, 1, Cout, xp, s * Cin, 1, Cout, k * Cin, B * Q)
            grads[pi] = dwp.reshape(Cout, k, Cin).permute(0, 2, 1).contiguous()
            # dX per phase r: padded row q*s + r = sum_m dY[q - m] W[:, :, r + m*s], as a stride-1 conv over dY with the
            # taps in reverse (m' = mr - 1 - m) starting mr - 1 rows above q
            dxp = (torch.zeros if s > k else torch.empty)(B * Q * s * Cin, dtype=f32, device=dev)
            for r in range(min(s, k)):
                mr = len(range(r, k, s))
                taps = [r + (mr - 1 - m) * s for m in range(mr)]
                wr = w[:, :, taps].permute(1, 2, 0).contiguous()          # [C_in, mr, C_out]
                if bf:
                    ops.conv1d_bf16(dy16, lead, B * Q, 1, Cout, -(mr - 1), ops.cast_bf16(wr), mr, Cin, None, dxp, r * Cin,
                                    s * Cin, B * Q)
                else:
                    ops.gemm_f32_at(dy32, lead - (mr - 1) * Cout, Cout, 1, wr, 1, mr * Cout, dxp, r * Cin, s * Cin,
                                    B * Q, Cin, mr * Cout)
            # GroupNorm + GELU backward into the gradient of this block's input
            if bi > 0:
                kp, sp, _, _, hbp, _ = blocks[bi - 1]
                Tp = saves[bi - 1][2]
                Qp = (kp - 1 + Tp + sp - 1) // sp
                nxt = (kp - 1 + B * Qp) * Cin
                dy32 = None if bf else torch.zeros(nxt, dtype=f32, device=dev)
                dy16 = torch.zeros(nxt, dtype=bf16, device=dev) if bf else None
                off, dstride, want_db = (kp - 1) * Cin, Qp * Cin, hbp
            else:
                dy32, dy16 = torch.empty(B * T * Cin, dtype=f32, device=dev), None
                off, dstride, want_db = 0, T * Cin, False
            grads[gi], grads[gi + 1], db_next = ops.gn_bwd(y, ustride, B, T, Cin, mean, rstd, g, dxp, (k - 1) * Cin,
                                                           Q * s * Cin, dy32, dy16, off, dstride, want_db)
            if bi == 0:
                dx_in = dy32.view(B, T, Cin)
        if first is not None:
            k, s, C0, hb = first
            dy0 = dx_in if blocks else dz.view(B, -1, C0)
            dw0, db0 = ops.conv1d_first_dw(first_in, _c(dy0), k, s)
            grads[i_first] = dw0.view(C0, 1, k)
            if hb:
                grads[i_first + 1] = db0
            dx_in = None
        return (dx_in, None, None) + tuple(grads)


# ---- wav2vec pre-training head (rnnt/wav2vec.py, modules/softmax_vector_quantizer.py; csrc/w2v.cu) ----------------
class W2VMask(torch.autograd.Function):
    """Wav2Vec.apply_mask's ``x[mask_indices] = mask_emb`` (rnnt/wav2vec.py:165-181), out of place: x [B, T, D] with
    mask_emb in the masked rows.  Backward: the masked rows of dx are zero and d mask_emb is the column sum of the
    masked rows of dout, gathered and added in row order (eb_colsum)."""

    @staticmethod
    def forward(ctx, x, mask_emb, idx, inv):
        ctx.save_for_backward(idx, inv)
        return ops.w2v_mask_fwd(_c(x), _c(mask_emb), inv)

    @staticmethod
    def backward(ctx, dout):
        idx, inv = ctx.saved_tensors
        dout = _c(dout)
        dx = ops.w2v_keep_rows(dout, inv) if ctx.needs_input_grad[0] else None
        demb = None
        if ctx.needs_input_grad[1]:
            demb = ops.colsum(ops.w2v_gather(dout, idx).view(-1, dout.shape[-1]))
        return dx, demb, None, None


class W2VGather(torch.autograd.Function):
    """x[mask_indices].view(B, M, D) (rnnt/wav2vec.py:308, 358): the masked rows of each utterance in frame order.
    Backward writes them back and zeros elsewhere; the rows are unique, so no sum is involved."""

    @staticmethod
    def forward(ctx, x, idx, inv):
        ctx.save_for_backward(inv)
        return ops.w2v_gather(_c(x), idx)

    @staticmethod
    def backward(ctx, dy):
        (inv,) = ctx.saved_tensors
        return ops.w2v_scatter(_c(dy), inv), None, None


class W2VSqMean(torch.autograd.Function):
    """features.float().pow(2).mean() (rnnt/wav2vec.py:269), added in a fixed order by one CTA."""

    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        ctx.save_for_backward(x)
        return ops.w2v_sq_mean(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return ops.w2v_scale(x, _c(g.to(f32)).reshape(1), 2.0 / x.numel())


class W2VQuantize(torch.autograd.Function):
    """GumbelVectorQuantizer.forward after weight_proj (modules/softmax_vector_quantizer.py:140-201) for
    combine_groups=False: logits [N, G*V], vars [1, G*V, vd], noise [N, G*V] (training) or None (eval) ->
    (q [N, G*vd], prob_perplexity, code_perplexity, k [N, G] int32).  Training: q[r, g] = st * vars[g*V + k] with k the
    hard Gumbel index and st = (1 - s_k) + s_k in fp32, as torch's straight-through F.gumbel_softmax(hard=True) gives it;
    eval: q = vars[k0], k0 the clean argmax.  Backward: d soft = dq_g vars_g^T and d vars_g = X_g^T dq_g (eb_gemm_f32,
    X the straight-through matrix), then the noisy and the clean softmax Jacobians (eb_w2v_quant_bwd)."""

    @staticmethod
    def forward(ctx, logits, vars, noise, G, tau):
        logits = _c(logits)
        v2 = _c(vars).view(-1, vars.shape[-1])
        q, p, s, X, k0, k, st = ops.w2v_quant_fwd(logits, noise, v2, G, tau)
        stats, coef = ops.w2v_quant_stats(p, k0, G)
        ctx.save_for_backward(v2, p, X, coef, *([s] if s is not None else []))
        ctx.meta = (G, tau, s is not None, vars.shape)
        pp, cp = stats[0].clone(), stats[1].clone()
        ctx.mark_non_differentiable(cp, k)
        return q, pp, cp, k

    @staticmethod
    def backward(ctx, dq, dpp, _dcp, _dk):
        G, tau, noisy, vshape = ctx.meta
        v2, p, X, coef = ctx.saved_tensors[:4]
        s = ctx.saved_tensors[4] if noisy else None
        N, GV = p.shape
        V, vd = GV // G, v2.shape[1]
        dq = _c(dq)
        dsoft = None
        if ctx.needs_input_grad[0] and noisy:
            dsoft = torch.empty(N, GV, dtype=f32, device=p.device)
            for g in range(G):
                ops.gemm_f32_at(dq, g * vd, G * vd, 1, v2[g * V:(g + 1) * V], 1, vd, dsoft, g * V, GV, N, V, vd)
        dl = None
        if ctx.needs_input_grad[0]:
            dl = ops.w2v_quant_bwd(dsoft, s, p, coef, _c(dpp.to(f32)).reshape(1), G, tau)
        dvars = None
        if ctx.needs_input_grad[1]:
            dvars = torch.empty(GV, vd, dtype=f32, device=p.device)
            for g in range(G):
                ops.gemm_f32_at(X, g * V, 1, GV, dq[:, g * vd:], G * vd, 1, dvars, g * V * vd, vd, V, vd, N)
            dvars = dvars.view(vshape)
        return dl, dvars, None, None, None


class W2VLogits(torch.autograd.Function):
    """Wav2Vec.compute_preds (rnnt/wav2vec.py:381-395) with the negatives of sample_negatives as frame indices:
    xp, yp [B, M, D], neg [B, M, K] int32 -> logits [K+1, B, M] = cos(xp[b, m], candidate) / logit_temp, candidate 0 =
    yp[b, m] and candidate 1 + k = yp[b, neg[b, m, k]]; -inf (and no gradient) where a negative equals the positive in
    every element.  torch.cosine_similarity's semantics: each row over max(|row|, 1e-8), then the dot product.  The
    [K+1, B, M, D] candidate tensor is never written."""

    @staticmethod
    def forward(ctx, xp, yp, neg, temp):
        xp, yp = _c(xp), _c(yp)
        logits, saved = ops.w2v_logits_fwd(xp, yp, neg, temp)
        ctx.save_for_backward(xp, yp, neg, *saved)
        ctx.temp = temp
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        xp, yp, neg, xh, yh, xn, yn, cos = ctx.saved_tensors
        dxp, dyp = ops.w2v_logits_bwd(_c(dlogits), cos, neg, xh, yh, xp, yp, xn, yn, ctx.temp)
        return dxp, dyp, None, None


class W2VCrossEntropy(torch.autograd.Function):
    """ConstrastiveCriterion's F.cross_entropy(get_logits(x), 0, reduction='sum') and its correct count
    (rnnt/wav2vec.py:445-461, 512-523) on logits [K+1, B, M], rows in get_logits' (m, b) order -> (loss, correct)."""

    @staticmethod
    def forward(ctx, logits):
        grad, out = ops.w2v_ce(_c(logits))
        ctx.save_for_backward(grad)
        loss, correct = out[0].clone(), out[1].clone()
        ctx.mark_non_differentiable(correct)
        return loss, correct

    @staticmethod
    def backward(ctx, go, _dc):
        (grad,) = ctx.saved_tensors
        return ops.w2v_scale(grad, _c(go.to(f32)).reshape(1))
