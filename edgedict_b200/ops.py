"""Tensor-level wrappers over the C-ABI: torch supplies device memory and the current stream,
nothing else.  Every function requires CUDA tensors and raises otherwise (no fallback)."""
import torch

from ._lib import lib
from ._lib import check as _check


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("edgedict_b200 ops need CUDA tensors (got a %s tensor); there is no CPU path" % t.device)
    return t.data_ptr()


def _need(t, dtype=None, name="tensor"):
    if not t.is_cuda:
        raise RuntimeError("edgedict_b200 ops need CUDA tensors (%s is on %s); there is no CPU path" % (name, t.device))
    if dtype is not None and t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s must be contiguous" % name)
    return t


f32, bf16 = torch.float32, torch.bfloat16
COLSUM_LANES = 512           # row lanes of eb_colsum's order for bf16 rows (csrc/common.cuh)


# ---- optional per-kernel instrumentation (bench.py) ----------------------------------------------
class _Prof:
    """When enabled, every wrapped C-ABI call is bracketed by CUDA events on the launching stream
    and counted; bench.py reads `summary()` after a synchronize.  Disabled: zero overhead."""

    def __init__(self):
        self.enabled = False
        self.events = []          # (name, start, end, bytes, flops)
        self.launches = 0

    def reset(self):
        self.events, self.launches = [], 0

    def summary(self, base=None):
        """Per-name totals.  `ms` is the UNION of the call intervals (calls of one name overlap when two layers'
        kernels run on two streams in the wavefront schedule) when a `base` event recorded before the first call
        is given, else their sum; `ms_sum` is always the plain sum."""
        out, spans = {}, {}
        for name, a, b, nbytes, flops in self.events:
            d = out.setdefault(name, dict(ms=0.0, ms_sum=0.0, calls=0, bytes=0.0, flops=0.0))
            d["ms_sum"] += a.elapsed_time(b)
            d["calls"] += 1
            d["bytes"] += nbytes
            d["flops"] += flops
            if base is not None:
                spans.setdefault(name, []).append((base.elapsed_time(a), base.elapsed_time(b)))
        for name, d in out.items():
            if base is None:
                d["ms"] = d["ms_sum"]
                continue
            tot, cur_s, cur_e = 0.0, None, None
            for s0, e0 in sorted(spans[name]):
                if cur_e is None or s0 > cur_e:
                    if cur_e is not None:
                        tot += cur_e - cur_s
                    cur_s, cur_e = s0, e0
                else:
                    cur_e = max(cur_e, e0)
            if cur_e is not None:
                tot += cur_e - cur_s
            d["ms"] = tot
        return out


PROF = _Prof()


def check(rc, what):
    PROF.launches += 1            # every C-ABI call launches at least one of our kernels
    _check(rc, what)


class _timed:
    def __init__(self, name, kernels=1, nbytes=0.0, flops=0.0):
        self.name, self.k, self.nbytes, self.flops = name, kernels, nbytes, flops

    def __enter__(self):
        if PROF.enabled:
            self.a = torch.cuda.Event(enable_timing=True)
            self.a.record()
        return self

    def __exit__(self, *exc):
        PROF.launches += self.k - 1     # extra kernels beyond the one `check` counts
        if PROF.enabled:
            b = torch.cuda.Event(enable_timing=True)
            b.record()
            PROF.events.append((self.name, self.a, b, self.nbytes, self.flops))
        return False


def cast_bf16(x, out=None):
    _need(x, f32, "x")
    y = out if out is not None else torch.empty(x.shape, dtype=bf16, device=x.device)
    n = x.numel()
    if n:
        check(lib().eb_cast_bf16(_p(x), _p(y), n, _s()), "eb_cast_bf16")
    return y


def gemm_f32(A, sam, sak, B, sbk, sbn, M, N, K, bias=None, out=None, beta=0.0, alpha=1.0):
    """C[M,N] = alpha*A'B' + beta*C + bias; strided views of fp32 storage (see eb_gemm_f32)."""
    if out is None:
        out = torch.empty(M, N, dtype=f32, device=A.device)
    with _timed("gemm_f32", 1, 0.0, 2.0 * M * N * K):
        check(lib().eb_gemm_f32(_p(A), sam, sak, _p(B), sbk, sbn, _p(out), N, _p(bias), M, N, K, alpha, beta, _s()),
              "eb_gemm_f32")
    return out


GEMM_CORESIDENT = 1      # include/edgedict_b200.h EB_GEMM_CORESIDENT
GEMM_FIXED_K = 2         # EB_GEMM_FIXED_K: row blocks of a product give the bits of the whole


def gemm_bf16(A, a_mn, B, b_mn, M, N, K, bias=None, out=None, out_bf16=False, accumulate=False, tag=None, flags=0):
    if out is None:
        out = torch.empty(M, N, dtype=bf16 if out_bf16 else f32, device=A.device)
    name = tag or ("gemm_bf16_%s%s" % ("t" if a_mn else "n", "n" if b_mn else "t"))
    with _timed(name, 1, 2.0 * (M * K + N * K) + out.element_size() * M * N, 2.0 * M * N * K):
        c16 = int(out.dtype == bf16)
        # split-K workspace (partial tiles summed in a fixed order: the same bits on every run)
        nws = int(lib().eb_gemm_bf16_partials(int(a_mn), c16, int(accumulate), M, N, K, int(flags)))
        ws = torch.empty(nws, dtype=f32, device=A.device) if nws else None
        check(lib().eb_gemm_bf16_ex(_p(A), int(a_mn), _p(B), int(b_mn), _p(out), c16, _p(bias), int(accumulate), M, N, K,
                                    int(flags), _p(ws), nws, _s()), "eb_gemm_bf16")
    return out


# ---- the three GEMM shapes of a Linear layer, dispatched on precision ---------------------------
def mm_nt(x, w, bias=None, precision="fp32", x16=None, w16=None, out_bf16=False):
    """y[M,N] = x[M,K] @ w[N,K]^T + bias.  w may be a column-slice view (fp32 mode uses strides)."""
    M, K = x.shape
    N = w.shape[0]
    if precision == "bf16":
        x16 = x16 if x16 is not None else (x if x.dtype == bf16 else cast_bf16(x))
        w16 = w16 if w16 is not None else cast_bf16(w.contiguous())
        return gemm_bf16(x16, 0, w16, 0, M, N, K, bias=bias, out_bf16=out_bf16)
    _need(x, f32, "x")
    return gemm_f32(x, K, 1, w, w.stride(1), w.stride(0), M, N, K, bias=bias)


def mm_nn(dy, w, precision="fp32", dy16=None, w16=None, out_bf16=False):
    """dx[M,K] = dy[M,N] @ w[N,K]."""
    M, N = dy.shape
    K = w.shape[1]
    if precision == "bf16":
        dy16 = dy16 if dy16 is not None else (dy if dy.dtype == bf16 else cast_bf16(dy))
        w16 = w16 if w16 is not None else cast_bf16(w.contiguous())
        return gemm_bf16(dy16, 0, w16, 1, M, K, N, out_bf16=out_bf16)
    _need(dy, f32, "dy")
    return gemm_f32(dy, N, 1, w, w.stride(0), w.stride(1), M, K, N)


def mm_tn(dy, x, precision="fp32", dy16=None, x16=None, out=None, accumulate=False):
    """dw[N,K] (+)= dy[M,N]^T @ x[M,K]  (contraction over the rows)."""
    M, N = dy.shape
    K = x.shape[1]
    if precision == "bf16":
        dy16 = dy16 if dy16 is not None else (dy if dy.dtype == bf16 else cast_bf16(dy))
        x16 = x16 if x16 is not None else (x if x.dtype == bf16 else cast_bf16(x))
        return gemm_bf16(dy16, 1, x16, 1, N, K, M, out=out, accumulate=accumulate)
    _need(dy, f32, "dy")
    _need(x, f32, "x")
    return gemm_f32(dy, 1, N, x, K, 1, N, K, M, out=out, beta=1.0 if accumulate else 0.0)


def colsum(x, out=None):
    rows, N = x.shape
    if out is None:
        out = torch.zeros(N, dtype=f32, device=x.device)
    check(lib().eb_colsum(_p(x), int(x.dtype == bf16), _p(out), rows, N, _s()), "eb_colsum")
    return out


# ---- LayerNorm / TimeReduction / Embedding -------------------------------------------------------
def layernorm_fwd(x, res, gamma, beta, eps=1e-5, want_bf16=False, out=None):
    """out = (y, y16 | None, mean, rstd) preallocated (contiguous slices of larger buffers), or None."""
    H = x.shape[-1]
    rows = x.numel() // H
    if out is not None:
        y, y16, mean, rstd = out
    else:
        y = torch.empty_like(x)
        y16 = torch.empty(x.shape, dtype=bf16, device=x.device) if want_bf16 else None
        mean = torch.empty(rows, dtype=f32, device=x.device)
        rstd = torch.empty(rows, dtype=f32, device=x.device)
    check(lib().eb_layernorm_fwd(_p(x), _p(res), _p(gamma), _p(beta), _p(y), _p(y16), _p(mean), _p(rstd),
                                 rows, H, eps, _s()), "eb_layernorm_fwd")
    return y, y16, mean, rstd


def layernorm_bwd_dz(dy, x, res, gamma, mean, rstd, out):
    """The dz pass of layernorm_bwd alone, into out (rows independent: a row block gives the rows of the whole)."""
    H = x.shape[-1]
    check(lib().eb_layernorm_bwd_dz(_p(dy), _p(x), _p(res), _p(gamma), _p(mean), _p(rstd), _p(out), x.numel() // H, H,
                                    _s()), "eb_layernorm_bwd_dz")
    return out


def layernorm_bwd_params(dy, x, res, mean, rstd):
    """The parameter pass of layernorm_bwd alone: (dgamma, dbeta), the same bits as layernorm_bwd's."""
    H = x.shape[-1]
    dgamma = torch.zeros(H, dtype=f32, device=x.device)
    dbeta = torch.zeros(H, dtype=f32, device=x.device)
    check(lib().eb_layernorm_bwd_params(_p(dy), _p(x), _p(res), _p(mean), _p(rstd), _p(dgamma), _p(dbeta),
                                        x.numel() // H, H, _s()), "eb_layernorm_bwd_params")
    return dgamma, dbeta


def layernorm_bwd(dy, x, res, gamma, mean, rstd):
    H = x.shape[-1]
    rows = x.numel() // H
    dz = torch.empty_like(x)
    dgamma = torch.zeros(H, dtype=f32, device=x.device)
    dbeta = torch.zeros(H, dtype=f32, device=x.device)
    check(lib().eb_layernorm_bwd(_p(dy), _p(x), _p(res), _p(gamma), _p(mean), _p(rstd), _p(dz), _p(dgamma),
                                 _p(dbeta), rows, H, _s()), "eb_layernorm_bwd")
    return dz, dgamma, dbeta


def time_reduce_fwd(x, want_bf16=False, out=None):
    B, T, H = x.shape
    if out is not None:
        y, y16 = out
    else:
        y = torch.empty(B, (T + 1) // 2, H, dtype=f32, device=x.device)
        y16 = torch.empty(y.shape, dtype=bf16, device=x.device) if want_bf16 else None
    check(lib().eb_time_reduce_fwd(_p(x), _p(y), _p(y16), B, T, H, _s()), "eb_time_reduce_fwd")
    return y, y16


def time_reduce_bwd(dy, T, out=None):
    B, _, H = dy.shape
    dx = out if out is not None else torch.empty(B, T, H, dtype=f32, device=dy.device)
    check(lib().eb_time_reduce_bwd(_p(dy), _p(dx), B, T, H, _s()), "eb_time_reduce_bwd")
    return dx


def embedding_fwd(ids, W, prepend_bos, bos):
    B, U = ids.shape
    E = W.shape[1]
    out = torch.empty(B, U + (1 if prepend_bos else 0), E, dtype=f32, device=W.device)
    if out.numel():
        check(lib().eb_embedding_fwd(_p(ids), int(ids.dtype == torch.int64), _p(W), _p(out), None, B, U, E,
                                     int(prepend_bos), bos, _s()), "eb_embedding_fwd")
    return out


def embedding_bwd(ids, dout, V, prepend_bos, bos, pad):
    B, U = ids.shape
    E = dout.shape[-1]
    dW = torch.zeros(V, E, dtype=f32, device=dout.device)
    if dout.numel():
        with _timed("embedding_bwd"):
            check(lib().eb_embedding_bwd(_p(ids), int(ids.dtype == torch.int64), _p(dout), _p(dW), B, U, E,
                                         int(prepend_bos), bos, pad, _s()), "eb_embedding_bwd")
    return dW


# ---- LSTM recurrent part -------------------------------------------------------------------------
_scratch = {}


def _lstm_scratch(B, H, device):
    key = (B, H, device, _s())        # per stream: layers on different streams (predictor / encoder) run concurrently
    t = _scratch.get(key)
    if t is None:
        n = lib().eb_lstm_scratch_bytes(B, H)
        if n == 0:
            raise ValueError("LSTM hidden size %d not supported by the persistent kernel" % H)
        t = torch.zeros(n, dtype=torch.uint8, device=device)
        _scratch[key] = t
    return t


def lstm_seq_fwd(xg, whh, h0, c0, save):
    B, T, H4 = xg.shape
    H = H4 // 4
    dev = xg.device
    y = torch.empty(B, T, H, dtype=f32, device=dev)
    hT = torch.empty(B, H, dtype=f32, device=dev)
    cT = torch.empty(B, H, dtype=f32, device=dev)
    gates = torch.empty(B, T, H4, dtype=f32, device=dev) if save else None
    cseq = torch.empty(B, T, H, dtype=f32, device=dev) if save else None
    with _timed("lstm_seq_fwd", 1, 0.0, 2.0 * B * T * 4 * H * H):
        check(lib().eb_lstm_seq_fwd(_p(xg), _p(whh), _p(h0), _p(c0), _p(y), _p(hT), _p(cT), _p(gates), _p(cseq),
                                    _p(_lstm_scratch(B, H, dev)), B, T, H, _s()), "eb_lstm_seq_fwd")
    return y, hT, cT, gates, cseq


def lstm_seq_bwd(dy, gates, cseq, c0, whh, dhT, dcT):
    """Returns (dgates -- written IN PLACE over `gates` --, dh0, dc0)."""
    B, T, H = dy.shape
    dev = dy.device
    dh0 = torch.empty(B, H, dtype=f32, device=dev)
    dc0 = torch.empty(B, H, dtype=f32, device=dev)
    with _timed("lstm_seq_bwd", 1, 0.0, 2.0 * B * T * 4 * H * H):
        check(lib().eb_lstm_seq_bwd(_p(dy), _p(gates), _p(cseq), _p(c0), _p(whh), _p(dhT), _p(dcT), _p(gates),
                                    _p(dh0), _p(dc0), _p(_lstm_scratch(B, H, dev)), B, T, H, _s()), "eb_lstm_seq_bwd")
    return gates, dh0, dc0


# ---- GRU recurrent part --------------------------------------------------------------------------
def _gru_scratch(B, H, device):
    key = ("gru", B, H, device, _s())
    t = _scratch.get(key)
    if t is None:
        n = lib().eb_gru_scratch_bytes(B, H)
        if n == 0:
            raise ValueError("GRU hidden size %d not supported by the persistent kernel" % H)
        t = torch.zeros(n, dtype=torch.uint8, device=device)
        _scratch[key] = t
    return t


def gru_seq_fwd(xg, whh, bhn, h0, save):
    """xg [B,T,3H] (b_hr, b_hz folded in), whh [3H,H], bhn [H] -> (y, hT, save [B,T,4H] = r|z|n|gh_n or None)."""
    B, T, H3 = xg.shape
    H = H3 // 3
    dev = xg.device
    y = torch.empty(B, T, H, dtype=f32, device=dev)
    hT = torch.empty(B, H, dtype=f32, device=dev)
    sv = torch.empty(B, T, 4 * H, dtype=f32, device=dev) if save else None
    with _timed("gru_seq_fwd", 1, 0.0, 2.0 * B * T * 3 * H * H):
        check(lib().eb_gru_seq_fwd(_p(xg), _p(whh), _p(bhn), _p(h0), _p(y), _p(hT), _p(sv),
                                   _p(_gru_scratch(B, H, dev)), B, T, H, _s()), "eb_gru_seq_fwd")
    return y, hT, sv


def gru_seq_bwd(dy, save, y, h0, whh, dhT):
    """Returns (dgi, dgh [B,T,3H], dh0 [B,H])."""
    B, T, H = dy.shape
    dev = dy.device
    dgi = torch.empty(B, T, 3 * H, dtype=f32, device=dev)
    dgh = torch.empty(B, T, 3 * H, dtype=f32, device=dev)
    dh0 = torch.empty(B, H, dtype=f32, device=dev)
    with _timed("gru_seq_bwd", 1, 0.0, 2.0 * B * T * 3 * H * H):
        check(lib().eb_gru_seq_bwd(_p(dy), _p(save), _p(y), _p(h0), _p(whh), _p(dhT), _p(dgi), _p(dgh), _p(dh0),
                                   _p(_gru_scratch(B, H, dev)), B, T, H, _s()), "eb_gru_seq_bwd")
    return dgi, dgh, dh0


def gru_tc_supported(B, H):
    return bool(lib().eb_gru_tc_supported(B, H))


def _gru_tc_scratch(B, H, device):
    key = ("gru_tc", H, device, _s())
    t = _scratch.get(key)
    if t is None:
        t = torch.zeros(lib().eb_gru_tc_scratch_bytes(B, H), dtype=torch.uint8, device=device)
        _scratch[key] = t
    return t


def gru_tc_fwd(xg, whh16, bhn, h0, save):
    """bf16 tensor-core recurrence: xg [B,T,3H] fp32, whh16 [3H,H] bf16 -> (y, hT, save | None), as gru_seq_fwd."""
    B, T, H3 = xg.shape
    H = H3 // 3
    dev = xg.device
    y = torch.empty(B, T, H, dtype=f32, device=dev)
    hT = torch.empty(B, H, dtype=f32, device=dev)
    sv = torch.empty(B, T, 4 * H, dtype=f32, device=dev) if save else None
    with _timed("gru_tc_fwd", 1, 0.0, 2.0 * B * T * 3 * H * H):
        check(lib().eb_gru_tc_fwd(_p(xg), _p(whh16), _p(bhn), _p(h0), _p(y), _p(hT), _p(sv),
                                  _p(_gru_tc_scratch(B, H, dev)), B, T, H, _s()), "eb_gru_tc_fwd")
    return y, hT, sv


def gru_tc_bwd(dy, save, y, h0, whhT16, dhT):
    """Returns (dgi16, dgh16 [B,T,3H] bf16, dh0 [B,H] fp32)."""
    B, T, H = dy.shape
    dev = dy.device
    dgi = torch.empty(B, T, 3 * H, dtype=bf16, device=dev)
    dgh = torch.empty(B, T, 3 * H, dtype=bf16, device=dev)
    dh0 = torch.empty(B, H, dtype=f32, device=dev)
    with _timed("gru_tc_bwd", 1, 0.0, 2.0 * B * T * 3 * H * H):
        check(lib().eb_gru_tc_bwd(_p(dy), _p(save), _p(y), _p(h0), _p(whhT16), _p(dhT), _p(dgi), _p(dgh), _p(dh0),
                                  _p(_gru_tc_scratch(B, H, dev)), B, T, H, _s()), "eb_gru_tc_bwd")
    return dgi, dgh, dh0


def lstm_tc_supported(B, H):
    return bool(lib().eb_lstm_tc_supported(B, H))


def _lstm_tc_scratch(B, H, device):
    key = ("tc", H, device, _s())     # one exchange buffer + barrier block per stream: kernels of two layers overlap
    t = _scratch.get(key)
    if t is None:
        t = torch.zeros(lib().eb_lstm_tc_scratch_bytes(B, H), dtype=torch.uint8, device=device)
        _scratch[key] = t
    return t


def lstm_tc_fwd(xg, whh16, h0, c0, save, out=None):
    """out = (y, y16, hT, cT, gates | None, cseq | None) preallocated, or None."""
    B, T, H4 = xg.shape
    H = H4 // 4
    dev = xg.device
    if out is not None:
        y, y16, hT, cT, gates, cseq = out
    else:
        y = torch.empty(B, T, H, dtype=f32, device=dev)
        y16 = torch.empty(B, T, H, dtype=bf16, device=dev)
        hT = torch.empty(B, H, dtype=f32, device=dev)
        cT = torch.empty(B, H, dtype=f32, device=dev)
        gates = torch.empty(B, T, H4, dtype=f32, device=dev) if save else None
        cseq = torch.empty(B, T, H, dtype=f32, device=dev) if save else None
    with _timed("lstm_tc_fwd", 1, 0.0, 2.0 * B * T * 4 * H * H):
        check(lib().eb_lstm_tc_fwd(_p(xg), _p(whh16), _p(h0), _p(c0), _p(y), _p(y16), _p(hT), _p(cT), _p(gates),
                                   _p(cseq), _p(_lstm_tc_scratch(B, H, dev)), B, T, H, _s()), "eb_lstm_tc_fwd")
    return y, y16, hT, cT, gates, cseq


def lstm_tc_bwd(dy, gates, cseq, c0, whhT16, dhT, dcT, out=None):
    B, T, H = dy.shape
    dev = dy.device
    dg16 = out if out is not None else torch.empty(B, T, 4 * H, dtype=bf16, device=dev)
    dh0 = torch.empty(B, H, dtype=f32, device=dev)
    dc0 = torch.empty(B, H, dtype=f32, device=dev)
    with _timed("lstm_tc_bwd", 1, 0.0, 2.0 * B * T * 4 * H * H):
        check(lib().eb_lstm_tc_bwd(_p(dy), _p(gates), _p(cseq), _p(c0), _p(whhT16), _p(dhT), _p(dcT), _p(dg16),
                                   _p(dh0), _p(dc0), _p(_lstm_tc_scratch(B, H, dev)), B, T, H, _s()), "eb_lstm_tc_bwd")
    return dg16, dh0, dc0


def lstm_tc_bwd_chunks(dy, gates, cseq, whhT16, lens, B, out):
    """BPTT of one layer over chunk-major buffers (functional._Chunks: rows = B * sum(lens)) in ONE launch; zero initial and
    final-state gradients.  dy [rows,H] fp32, gates [rows,4H], cseq [rows,H], out = dg16 [rows,4H] bf16."""
    import ctypes
    H = dy.shape[1]
    dev = dy.device
    dh0 = torch.empty(B, H, dtype=f32, device=dev)
    dc0 = torch.empty(B, H, dtype=f32, device=dev)
    arr = (ctypes.c_int * len(lens))(*[int(n) for n in lens])
    with _timed("lstm_tc_bwd", 1, 0.0, 2.0 * B * sum(lens) * 4 * H * H):
        check(lib().eb_lstm_tc_bwd_chunks(_p(dy), _p(gates), _p(cseq), None, _p(whhT16), None, None, _p(out), _p(dh0),
                                          _p(dc0), _p(_lstm_tc_scratch(B, H, dev)), B, arr, len(lens), H, _s()),
              "eb_lstm_tc_bwd_chunks")
    return out, dh0, dc0


# ---- cluster / wgmma recurrent kernels (csrc/lstm_c4.cu) ------------------------------------------
_c4_ok = {}


def lstm_c4_supported(B, H):
    """True when eb_lstm_c4_* can run this layer: H % 256 == 0, H <= 1024 and all clusters co-resident."""
    v = _c4_ok.get(H)
    if v is None:
        v = _c4_ok[H] = bool(lib().eb_lstm_c4_supported(B, H))
    return v


def _lstm_c4_scratch(B, H, device):
    key = ("c4", H, device, _s())     # one exchange buffer + barrier block per stream: kernels of two layers overlap
    t = _scratch.get(key)
    if t is None:
        t = torch.zeros(lib().eb_lstm_c4_scratch_bytes(B, H), dtype=torch.uint8, device=device)
        _scratch[key] = t
    return t


def lstm_c4_save_buffers(B, T, H, device):
    """(gsave, csave): CTA-private layout of the forward saves (bf16 gates, fp32 cell states)."""
    return (torch.empty(lib().eb_lstm_c4_gsave_bytes(B, T, H), dtype=torch.uint8, device=device),
            torch.empty(lib().eb_lstm_c4_csave_bytes(B, T, H), dtype=torch.uint8, device=device))


C4_BWD = __import__("os").environ.get("EDGEDICT_LSTM_C4_BWD", "0") != "0"   # BPTT through lstm_c4 (else lstm_tc's kernel)


def lstm_c4_fwd(xg, whh16, h0, c0, save, out=None, std_saves=None):
    """out = (y, hprev16, hT, cT) preallocated, or None.  Returns (y, hprev16, hT, cT, gsave | None, csave | None);
    hprev16[:, t] = bf16(h_{t-1}) (frame 0 = h0) is the operand of the dW_hh GEMM.  The saves for backward are
    either the kernels' own CTA-private layout (gsave, csave: consumed by lstm_c4_bwd) or, with
    std_saves = (gates [B,T,4H] fp32, cseq [B,T,H] fp32) (or True to allocate them), the layout of lstm_tc_bwd."""
    B, T, H4 = xg.shape
    H = H4 // 4
    dev = xg.device
    if out is not None:
        y, hprev16, hT, cT = out
    else:
        y = torch.empty(B, T, H, dtype=f32, device=dev)
        hprev16 = torch.empty(B, T, H, dtype=bf16, device=dev) if save else None
        hT = torch.empty(B, H, dtype=f32, device=dev)
        cT = torch.empty(B, H, dtype=f32, device=dev)
    gsave = csave = gstd = cstd = None
    if save and std_saves is not None and std_saves is not False:
        gstd, cstd = std_saves if isinstance(std_saves, tuple) else (torch.empty(B, T, H4, dtype=f32, device=dev),
                                                                     torch.empty(B, T, H, dtype=f32, device=dev))
    elif save:
        gsave, csave = lstm_c4_save_buffers(B, T, H, dev)
    with _timed("lstm_tc_fwd", 1, 0.0, 2.0 * B * T * 4 * H * H):
        check(lib().eb_lstm_c4_fwd(_p(xg), _p(whh16), _p(h0), _p(c0), _p(y), _p(hprev16), _p(hT), _p(cT), _p(gsave),
                                   _p(csave), _p(gstd), _p(cstd), _p(_lstm_c4_scratch(B, H, dev)), B, T, H, _s()),
              "eb_lstm_c4_fwd")
    if gstd is not None:
        return y, hprev16, hT, cT, gstd, cstd
    return y, hprev16, hT, cT, gsave, csave


_c4_chunks_ok = {}


def lstm_c4_bwd_chunks_supported(H):
    """True when eb_lstm_c4_bwd_chunks can run hidden size H: H % 256 == 0, H <= 1024 and all clusters of 16 co-resident."""
    v = _c4_chunks_ok.get(H)
    if v is None:
        v = _c4_chunks_ok[H] = lib().eb_lstm_c4_bwd_chunks_cluster(H) == 16
    return v


def lstm_c4_bwd_chunks(dy, gates, cseq, whhT16, lens, B, out, c0=None, dhT=None, dcT=None):
    """lstm_tc_bwd_chunks on the K-split wgmma kernel (clusters of 16), same saves and buffers; returns (out, dh0, dc0).
    c0 / dhT / dcT [B,H] are optional (zero)."""
    import ctypes
    H = dy.shape[-1]
    dev = dy.device
    dh0 = torch.empty(B, H, dtype=f32, device=dev)
    dc0 = torch.empty(B, H, dtype=f32, device=dev)
    arr = (ctypes.c_int * len(lens))(*[int(n) for n in lens])
    with _timed("lstm_tc_bwd", 1, 0.0, 2.0 * B * sum(lens) * 4 * H * H):
        check(lib().eb_lstm_c4_bwd_chunks(_p(dy), _p(gates), _p(cseq), _p(c0), _p(whhT16), _p(dhT), _p(dcT), _p(out),
                                          _p(dh0), _p(dc0), _p(_lstm_c4_scratch(B, H, dev)), B, arr, len(lens), H, _s()),
              "eb_lstm_c4_bwd_chunks")
    return out, dh0, dc0


def lstm_c4_bwd(dy, gsave, csave, c0, whhT16, dhT, dcT, out=None):
    B, T, H = dy.shape
    dev = dy.device
    dg16 = out if out is not None else torch.empty(B, T, 4 * H, dtype=bf16, device=dev)
    dh0 = torch.empty(B, H, dtype=f32, device=dev)
    dc0 = torch.empty(B, H, dtype=f32, device=dev)
    with _timed("lstm_tc_bwd", 1, 0.0, 2.0 * B * T * 4 * H * H):
        check(lib().eb_lstm_c4_bwd(_p(dy), _p(gsave), _p(csave), _p(c0), _p(whhT16), _p(dhT), _p(dcT), _p(dg16),
                                   _p(dh0), _p(dc0), _p(_lstm_c4_scratch(B, H, dev)), B, T, H, _s()), "eb_lstm_c4_bwd")
    return dg16, dh0, dc0


def transpose_to_bf16(x):
    """x [rows, cols] (fp32 or bf16) -> bf16 [cols, rows]."""
    rows, cols = x.shape
    y = torch.empty(cols, rows, dtype=bf16, device=x.device)
    check(lib().eb_transpose_to_bf16(_p(x), int(x.dtype == bf16), _p(y), rows, cols, _s()), "eb_transpose_to_bf16")
    return y


# ---- joint + loss ----------------------------------------------------------------------------------
def joint_hidden_fwd(ep, dp, want_bf16):
    B, T, J = ep.shape
    U = dp.shape[1]
    hid = torch.empty(B, T, U, J, dtype=bf16 if want_bf16 else f32, device=ep.device)
    check(lib().eb_joint_hidden_fwd(_p(ep), _p(dp), _p(hid), int(want_bf16), B, T, U, J, _s()), "eb_joint_hidden_fwd")
    return hid


def joint_hidden_bwd(dhid, hid):
    """dhid is overwritten with d(pre-activation); returns (dep [B,T,J], ddp [B,U,J])."""
    B, T, U, J = hid.shape
    dep = torch.empty(B, T, J, dtype=f32, device=hid.device)
    ddp = torch.empty(B, U, J, dtype=f32, device=hid.device)
    check(lib().eb_joint_hidden_bwd(_p(dhid), _p(hid), int(hid.dtype == bf16), _p(dep), _p(ddp), B, T, U, J, _s()),
          "eb_joint_hidden_bwd")
    return dep, ddp


def gemm_bf16_dtanh(A16, B16, b_mn, hid16, M, N, K):
    """bf16 [M,N] = (A16 [M,K] @ B) * (1 - hid16^2)  (B16: [N,K] if not b_mn else [K,N])."""
    out = torch.empty(M, N, dtype=bf16, device=A16.device)
    with _timed("gemm_bf16_n%s" % ("n" if b_mn else "t"), 1, 2.0 * (M * K + N * K) + 4.0 * M * N, 2.0 * M * N * K):
        check(lib().eb_gemm_bf16_dtanh(_p(A16), 0, _p(B16), int(b_mn), _p(out), _p(hid16), M, N, K, _s()),
              "eb_gemm_bf16_dtanh")
    return out


def joint_dpre_reduce(dpre16):
    """dpre16 [B,T,U,J] bf16 -> (dep [B,T,J], ddp [B,U,J]) fp32."""
    B, T, U, J = dpre16.shape
    dep = torch.empty(B, T, J, dtype=f32, device=dpre16.device)
    ddp = torch.empty(B, U, J, dtype=f32, device=dpre16.device)
    check(lib().eb_joint_dpre_reduce(_p(dpre16), _p(dep), _p(ddp), B, T, U, J, _s()), "eb_joint_dpre_reduce")
    PROF.launches += 1
    return dep, ddp


def rnnt_workspace(B, T, U, dtype, device):
    n = lib().eb_rnnt_workspace_bytes(B, T, U, 8 if dtype == torch.float64 else 4)
    return torch.empty(n, dtype=torch.uint8, device=device)


def rnnt_loss_fwd(logits, labels, xlen, ylen, blank, need_beta=True):
    B, T, U, V = logits.shape
    ds = 8 if logits.dtype == torch.float64 else 4
    ws = rnnt_workspace(B, T, U, logits.dtype, logits.device)
    costs = torch.empty(B, dtype=logits.dtype, device=logits.device)
    with _timed("rnnt_loss_fwd", 3, float(ds) * B * T * U * V, 0.0):
        check(lib().eb_rnnt_loss_fwd(_p(logits), _p(labels), _p(xlen), _p(ylen), B, T, U, V, blank, ds, _p(ws),
                                     _p(costs), int(need_beta), _s()), "eb_rnnt_loss_fwd")
    return costs, ws


def rnnt_loss_bwd(logits, labels, xlen, ylen, blank, ws, gscale, host_scale, out=None, out_bf16=False,
                  fastemit_lambda=0.0):
    """d loss / d logits (fp32 / fp64, or bf16 with out_bf16), with the FastEmit gradient for fastemit_lambda > 0
    (include/edgedict_b200.h, eb_rnnt_loss_bwd_fe); at 0 the plain loss's gradient."""
    B, T, U, V = logits.shape
    ds = 8 if logits.dtype == torch.float64 else 4
    if out is None:
        out = torch.empty(logits.shape, dtype=bf16 if out_bf16 else logits.dtype, device=logits.device)
    per_batch = int(gscale is not None and gscale.numel() > 1)
    with _timed("rnnt_loss_bwd", 1, float(ds + out.element_size()) * B * T * U * V, 0.0):
        check(lib().eb_rnnt_loss_bwd_fe(_p(logits), _p(out), int(out.dtype == bf16), _p(labels), _p(xlen), _p(ylen), B,
                                        T, U, V, blank, ds, _p(ws), _p(gscale), per_batch, float(host_scale),
                                        float(fastemit_lambda), _s()), "eb_rnnt_loss_bwd_fe")
    return out


def joint_logits_lse(hid16, w2_16, b2, labels, xlen, ylen, B, T, U, blank):
    """bf16 logits [B,T,U,V] + loss workspace with denom / log p(blank) / log p(label) filled in."""
    V, J = w2_16.shape
    logits16 = torch.empty(B, T, U, V, dtype=bf16, device=hid16.device)
    ws = rnnt_workspace(B, T, U, f32, hid16.device)
    n = B * T * U
    wsf = ws.view(f32)
    N = float(n) * V
    with _timed("joint_logits_lse", 1, 2.0 * n * J + 2.0 * N, 2.0 * N * J):
        check(lib().eb_joint_logits_lse(_p(hid16), _p(w2_16), _p(b2), _p(logits16), _p(labels), _p(xlen), _p(ylen),
                                        _p(wsf[0:n]), _p(wsf[n:2 * n]), _p(wsf[2 * n:3 * n]), B, T, U, V, J, blank,
                                        _s()), "eb_joint_logits_lse")
    return logits16, ws


def rnnt_lattice(xlen, ylen, B, T, U, ws, need_beta=True):
    costs = torch.empty(B, dtype=f32, device=ws.device)
    with _timed("rnnt_loss_fwd", 2, 0.0, 0.0):
        check(lib().eb_rnnt_loss_lattice(_p(xlen), _p(ylen), B, T, U, _p(ws), _p(costs), int(need_beta), _s()),
              "eb_rnnt_loss_lattice")
    return costs


def rnnt_viterbi(xlen, ylen, B, T, U, ws, dtype):
    """Forced alignment over a loss workspace of `dtype` (fp32 / fp64) that rnnt_loss_fwd or joint_logits_lse filled.
    Returns (frames int32 [B, U-1], label_logp [B, U-1], score [B]) on the device (include/edgedict_b200.h)."""
    dev = ws.device
    dec = torch.empty(lib().eb_rnnt_align_bytes(B, T, U), dtype=torch.uint8, device=dev)
    frames = torch.empty(B, U - 1, dtype=torch.int32, device=dev)
    label_logp = torch.empty(B, U - 1, dtype=dtype, device=dev)
    score = torch.empty(B, dtype=dtype, device=dev)
    with _timed("rnnt_viterbi", 1, 0.0, 0.0):
        check(lib().eb_rnnt_viterbi(_p(xlen), _p(ylen), B, T, U, 8 if dtype == torch.float64 else 4, _p(ws),
                                    _p(dec) if dec.numel() else None, _p(frames), _p(label_logp), _p(score), _s()),
              "eb_rnnt_viterbi")
    return frames, label_logp, score


def rnnt_loss_bwd_bf16(logits16, labels, xlen, ylen, blank, ws, gscale, host_scale, fastemit_lambda=0.0):
    """In place: logits16 becomes d loss / d logits (bf16), FastEmit's for fastemit_lambda > 0."""
    B, T, U, V = logits16.shape
    per_batch = int(gscale is not None and gscale.numel() > 1)
    with _timed("rnnt_loss_bwd", 1, 4.0 * B * T * U * V, 0.0):
        check(lib().eb_rnnt_loss_bwd_bf16_fe(_p(logits16), _p(logits16), _p(labels), _p(xlen), _p(ylen), B, T, U, V,
                                             blank, _p(ws), _p(gscale), per_batch, float(host_scale),
                                             float(fastemit_lambda), _s()), "eb_rnnt_loss_bwd_bf16_fe")
    return logits16


def rnnt_loss_bwd_bf16_db(logits16, labels, xlen, ylen, blank, ws, gscale, host_scale, fastemit_lambda=0.0):
    """In place: logits16 becomes d loss / d logits (bf16), as rnnt_loss_bwd_bf16 writes them for the same
    fastemit_lambda; also returns their column sum db [V] fp32, the same bits as colsum(logits16.view(-1, V))
    afterwards.  V % 8 == 0."""
    B, T, U, V = logits16.shape
    per_batch = int(gscale is not None and gscale.numel() > 1)
    part = torch.empty(COLSUM_LANES * V, dtype=f32, device=logits16.device)
    db = torch.zeros(V, dtype=f32, device=logits16.device)
    with _timed("rnnt_loss_bwd", 2, 4.0 * B * T * U * V, 0.0):
        check(lib().eb_rnnt_loss_bwd_bf16_db_fe(_p(logits16), _p(logits16), _p(labels), _p(xlen), _p(ylen), B, T, U, V,
                                                blank, _p(ws), _p(gscale), per_batch, float(host_scale), _p(part),
                                                _p(db), float(fastemit_lambda), _s()), "eb_rnnt_loss_bwd_bf16_db_fe")
    return logits16, db


# ---- pruned RNN-T loss (csrc/pruned.cu, csrc/loss.cu; include/edgedict_b200.h) ----------------------------------
def rnnt_simple_fwd(am, lm, labels, xlen, ylen, blank):
    """The trivial joiner's loss: (costs [B], workspace with alpha, beta and the statistics of N(t,u), scratch that
    rnnt_simple_bwd reads)."""
    B, T, V = am.shape
    U = lm.shape[1]
    ws = rnnt_workspace(B, T, U, f32, am.device)
    scratch = torch.empty(lib().eb_rnnt_simple_scratch_bytes(B, T, U, V), dtype=torch.uint8, device=am.device)
    with _timed("rnnt_simple_fwd", 3 + B, 4.0 * (B * T + B * U) * V, 2.0 * B * T * U * V):
        check(lib().eb_rnnt_simple_stats(_p(am), _p(lm), _p(labels), _p(xlen), _p(ylen), B, T, U, V, blank,
                                         _p(scratch), _p(ws), _s()), "eb_rnnt_simple_stats")
    return rnnt_lattice(xlen, ylen, B, T, U, ws), ws, scratch


def rnnt_simple_bwd(am, lm, labels, xlen, ylen, blank, ws, scratch, gscale, host_scale):
    """(d am, d lm) of sum_b gscale[b] * cost_b * host_scale."""
    B, T, V = am.shape
    U = lm.shape[1]
    dam, dlm = torch.empty_like(am), torch.empty_like(lm)
    per_batch = int(gscale is not None and gscale.numel() > 1)
    with _timed("rnnt_simple_bwd", 3 + 2 * B, 8.0 * (B * T + B * U) * V, 4.0 * B * T * U * V):
        check(lib().eb_rnnt_simple_bwd(_p(am), _p(lm), _p(labels), _p(xlen), _p(ylen), B, T, U, V, blank,
                                       _p(scratch), _p(ws), _p(gscale), per_batch, float(host_scale), _p(dam), _p(dlm),
                                       _s()), "eb_rnnt_simple_bwd")
    return dam, dlm


def rnnt_band_choice(xlen, ylen, B, T, U, R, ws):
    """(s_begin [B, T] int32, nopath [B] int32) from a simple-loss workspace."""
    s_begin = torch.empty(B, T, dtype=torch.int32, device=ws.device)
    nopath = torch.empty(B, dtype=torch.int32, device=ws.device)
    with _timed("rnnt_band_choice", 1, 0.0, 0.0):
        check(lib().eb_rnnt_band_choice(_p(xlen), _p(ylen), B, T, U, R, _p(ws), _p(s_begin), _p(nopath), _s()),
              "eb_rnnt_band_choice")
    return s_begin, nopath


def joint_band_hidden_fwd(ep, dp, xlen, ylen, s_begin, R, want_bf16):
    """hidden [B, T, R, J] of the band rows (fp32, or bf16 with want_bf16)."""
    B, T, J = ep.shape
    U = dp.shape[1]
    hid = torch.empty(B, T, R, J, dtype=bf16 if want_bf16 else f32, device=ep.device)
    check(lib().eb_joint_band_hidden_fwd(_p(ep), _p(dp), _p(xlen), _p(ylen), _p(s_begin), _p(hid), int(want_bf16), B,
                                         T, U, R, J, _s()), "eb_joint_band_hidden_fwd")
    return hid


def rnnt_band_loss_fwd(logits, labels, xlen, ylen, s_begin, nopath, U, blank, need_beta=True):
    """logits [B, T, R, V] fp32 of the band rows -> (costs [B], full [B, T, U] loss workspace)."""
    B, T, R, V = logits.shape
    ws = rnnt_workspace(B, T, U, f32, logits.device)
    costs = torch.empty(B, dtype=f32, device=logits.device)
    with _timed("rnnt_band_loss_fwd", 4, 4.0 * B * T * R * V, 0.0):
        check(lib().eb_rnnt_band_loss_fwd(_p(logits), _p(labels), _p(xlen), _p(ylen), _p(s_begin), _p(nopath), B, T, U,
                                          R, V, blank, _p(ws), _p(costs), int(need_beta), _s()), "eb_rnnt_band_loss_fwd")
    return costs, ws


def joint_band_logits_lse(hid16, w2_16, b2, labels, xlen, ylen, s_begin, nopath, U, blank):
    """bf16 mode: bf16 logits [B, T, R, V] of the band rows hid16 [B, T, R, J] and their statistics from the GEMM's
    epilogue, then the fill and the lattice: (logits16, costs [B], full [B, T, U] loss workspace)."""
    B, T, R, J = hid16.shape
    V = w2_16.shape[0]
    logits16 = torch.empty(B, T, R, V, dtype=bf16, device=hid16.device)
    ws = rnnt_workspace(B, T, U, f32, hid16.device)
    n = B * T * U
    wsf = ws.view(f32)
    N = float(B * T * R) * V
    with _timed("joint_band_logits_lse", 1, 2.0 * B * T * R * J + 2.0 * N, 2.0 * N * J):
        check(lib().eb_joint_band_logits_lse(_p(hid16), _p(w2_16), _p(b2), _p(logits16), _p(labels), _p(xlen),
                                             _p(ylen), _p(s_begin), _p(wsf[0:n]), _p(wsf[n:2 * n]),
                                             _p(wsf[2 * n:3 * n]), B, T, U, R, V, J, blank, _s()),
              "eb_joint_band_logits_lse")
    costs = torch.empty(B, dtype=f32, device=hid16.device)
    with _timed("rnnt_band_lattice", 3, 0.0, 0.0):
        check(lib().eb_rnnt_band_lattice(_p(xlen), _p(ylen), _p(s_begin), _p(nopath), B, T, U, R, _p(ws), _p(costs), 1,
                                         _s()), "eb_rnnt_band_lattice")
    return logits16, costs, ws


def rnnt_band_loss_bwd_bf16_db(logits16, labels, xlen, ylen, s_begin, nopath, U, blank, ws, gscale, host_scale):
    """In place: logits16 [B, T, R, V] becomes the band rows' bf16 d logits; also returns their column sum db [V]."""
    B, T, R, V = logits16.shape
    per_batch = int(gscale is not None and gscale.numel() > 1)
    part = torch.empty(COLSUM_LANES * V, dtype=f32, device=logits16.device)
    db = torch.zeros(V, dtype=f32, device=logits16.device)
    with _timed("rnnt_band_loss_bwd", 2, 4.0 * B * T * R * V, 0.0):
        check(lib().eb_rnnt_band_loss_bwd_bf16_db(_p(logits16), _p(logits16), _p(labels), _p(xlen), _p(ylen),
                                                  _p(s_begin), _p(nopath), B, T, U, R, V, blank, _p(ws), _p(gscale),
                                                  per_batch, float(host_scale), _p(part), _p(db), _s()),
              "eb_rnnt_band_loss_bwd_bf16_db")
    return logits16, db


def rnnt_band_loss_bwd(logits, labels, xlen, ylen, s_begin, nopath, U, blank, ws, gscale, host_scale, out=None,
                       out_bf16=False):
    """d loss / d logits of the band rows: fp32 (out may be logits: in place) or bf16 with out_bf16."""
    B, T, R, V = logits.shape
    if out is None:
        out = torch.empty(logits.shape, dtype=bf16 if out_bf16 else f32, device=logits.device)
    per_batch = int(gscale is not None and gscale.numel() > 1)
    with _timed("rnnt_band_loss_bwd", 1, float(4 + out.element_size()) * B * T * R * V, 0.0):
        check(lib().eb_rnnt_band_loss_bwd(_p(logits), _p(out), int(out.dtype == bf16), _p(labels), _p(xlen), _p(ylen),
                                          _p(s_begin), _p(nopath), B, T, U, R, V, blank, _p(ws), _p(gscale), per_batch,
                                          float(host_scale), _s()), "eb_rnnt_band_loss_bwd")
    return out


def joint_band_dpre_reduce(dx, hid, xlen, ylen, s_begin, U):
    """(dep [B, T, J], ddp [B, U, J]) fp32 from the band rows' d hidden dx [B, T, R, J] fp32 with hid fp32, or from
    the bf16 d(pre-activation) dx with hid None."""
    B, T, R, J = dx.shape
    dep = torch.empty(B, T, J, dtype=f32, device=dx.device)
    ddp = torch.empty(B, U, J, dtype=f32, device=dx.device)
    with _timed("joint_band_dpre_reduce", 2, 2.0 * dx.numel() * dx.element_size(), 0.0):
        check(lib().eb_joint_band_dpre_reduce(_p(dx), _p(hid), int(dx.dtype == bf16), _p(xlen), _p(ylen), _p(s_begin),
                                              _p(dep), _p(ddp), B, T, U, R, J, _s()), "eb_joint_band_dpre_reduce")
    return dep, ddp


# ---- language-model cross-entropy (csrc/lm.cu, csrc/gemm_tc.cu) ---------------------------------------
def _targets(t):
    _need(t, None, "targets")
    if t.dtype not in (torch.int32, torch.int64):
        raise TypeError("targets must be int32 or int64, got %s" % t.dtype)
    return int(t.dtype == torch.int64)


def lm_logits_ce(hid16, w16, b, targets):
    """bf16 logits [M, V] of hid16 [M, K] @ w16[V, K]^T + b, with each row's lse and target logit (fp32 [M]) from the
    GEMM's accumulators."""
    M, K = hid16.shape
    V = w16.shape[0]
    t64 = _targets(targets)
    logits16 = torch.empty(M, V, dtype=bf16, device=hid16.device)
    lse = torch.empty(M, dtype=f32, device=hid16.device)
    tl = torch.empty(M, dtype=f32, device=hid16.device)
    with _timed("lm_logits_ce", 1, 2.0 * (M * K + V * K) + 2.0 * M * V, 2.0 * M * V * K):
        check(lib().eb_lm_logits_ce(_p(hid16), _p(w16), _p(b), _p(logits16), _p(targets), t64, _p(lse), _p(tl), M, V, K,
                                    _s()), "eb_lm_logits_ce")
    return logits16, lse, tl


def lm_ce_rows(logits, targets):
    """(lse, target logit) [M] of fp32 logit rows [M, V]."""
    _need(logits, f32, "logits")
    M, V = logits.shape
    t64 = _targets(targets)
    lse = torch.empty(M, dtype=f32, device=logits.device)
    tl = torch.empty(M, dtype=f32, device=logits.device)
    with _timed("lm_ce_rows", 1, 4.0 * M * V, 0.0):
        check(lib().eb_lm_ce_rows(_p(logits), _p(targets), t64, _p(lse), _p(tl), M, V, _s()), "eb_lm_ce_rows")
    return lse, tl


def lm_ce_loss(lse, tl, targets, ignore_index, V, mean):
    """(cost [M], loss [] , scale [1]): per-token costs, their sum or mean over non-ignored targets, and the gradient
    scale (1 or 1 / count), all on the device."""
    M = lse.shape[0]
    t64 = _targets(targets)
    cost = torch.empty(M, dtype=f32, device=lse.device)
    loss = torch.empty((), dtype=f32, device=lse.device)
    scale = torch.empty(1, dtype=f32, device=lse.device)
    with _timed("lm_ce_loss", 1, 12.0 * M, 0.0):
        check(lib().eb_lm_ce_loss(_p(lse), _p(tl), _p(targets), t64, int(ignore_index), M, V, int(mean), _p(cost),
                                  _p(loss), _p(scale), _s()), "eb_lm_ce_loss")
    return cost, loss, scale


def lm_ce_bwd(logits, lse, targets, ignore_index, g, scale=None, out=None):
    """d logits (same dtype as logits, written into `out`, which may be logits itself) of sum_r g[r] * scale * cost_r
    (g [M]) or of g * scale * sum_r cost_r (g one element)."""
    M, V = logits.shape
    t64 = _targets(targets)
    _need(g, f32, "g")
    out = torch.empty_like(logits) if out is None else out
    with _timed("lm_ce_bwd", 1, 2.0 * logits.element_size() * M * V, 0.0):
        check(lib().eb_lm_ce_bwd(_p(logits), _p(out), int(logits.dtype == bf16), _p(lse), _p(targets), t64,
                                 int(ignore_index), M, V, _p(g), int(g.numel() > 1), _p(scale), _s()), "eb_lm_ce_bwd")
    return out


# ---- CTC (csrc/ctc.cu) -------------------------------------------------------------------------------
def log_softmax_fwd(x):
    """Row log-softmax over the last dim of a contiguous fp32 tensor."""
    _need(x, f32, "x")
    y = torch.empty_like(x)
    V = x.shape[-1]
    with _timed("log_softmax_fwd", 1, 8.0 * x.numel(), 0.0):
        check(lib().eb_log_softmax_fwd(_p(x), _p(y), x.numel() // V, V, _s()), "eb_log_softmax_fwd")
    return y


def log_softmax_bwd(dy, y):
    """dx = dy - exp(y) * sum(dy) per row; contiguous fp32 tensors of one shape."""
    _need(dy, f32, "dy")
    _need(y, f32, "y")
    dx = torch.empty_like(y)
    V = y.shape[-1]
    with _timed("log_softmax_bwd", 1, 12.0 * y.numel(), 0.0):
        check(lib().eb_log_softmax_bwd(_p(dy), _p(y), _p(dx), y.numel() // V, V, _s()), "eb_log_softmax_bwd")
    return dx


def ctc_loss_fwd(lp, targets, offsets, tlen, ilen, S, blank, zero_infinity):
    """lp (T, N, V) fp32 with unit stride over V (any T / N strides); targets int32 (device, 1-D storage of the labels);
    offsets / tlen / ilen int32 [N] on the device; S >= max(tlen).  Returns (costs [N], workspace)."""
    T, N, V = lp.shape
    ws = torch.empty(lib().eb_ctc_workspace_size(N, T, S), dtype=torch.uint8, device=lp.device)
    costs = torch.empty(N, dtype=f32, device=lp.device)
    with _timed("ctc_loss_fwd", 1, 4.0 * N * T * (2 * S + 1) * 2, 0.0):
        check(lib().eb_ctc_loss_fwd(_p(lp), lp.stride(1), lp.stride(0), N, T, V, _p(targets), targets.numel(),
                                    _p(offsets), _p(tlen), _p(ilen), S, blank, int(zero_infinity), _p(ws), _p(costs),
                                    _s()), "eb_ctc_loss_fwd")
    return costs, ws


def ctc_loss_bwd(lp, tlen, ilen, S, blank, zero_infinity, ws, gscale):
    """Gradient for log_probs (same shape and strides as lp), scaled per utterance by gscale [N] (device fp32)."""
    T, N, V = lp.shape
    grad = torch.empty_like(lp)
    with _timed("ctc_loss_bwd", 1, 8.0 * lp.numel(), 0.0):
        check(lib().eb_ctc_loss_bwd(_p(lp), lp.stride(1), lp.stride(0), _p(grad), grad.stride(1), grad.stride(0), N, T,
                                    V, _p(tlen), _p(ilen), S, blank, int(zero_infinity), _p(ws), _p(gscale), _s()),
              "eb_ctc_loss_bwd")
    return grad


def ctc_greedy(lp, xlen, blank):
    """lp [B, T, V] fp32 (unit stride over V), xlen int32 [B] on the device -> one int32 device buffer
    [B*T ids | B counts | B neg-scores (fp32 bits)], so that the host needs one copy."""
    B, T, V = lp.shape
    out = torch.empty(B * T + 2 * B, dtype=torch.int32, device=lp.device)
    with _timed("ctc_greedy", 1, 4.0 * lp.numel(), 0.0):
        check(lib().eb_ctc_greedy(_p(lp), lp.stride(0), lp.stride(1), B, T, V, _p(xlen), blank, _p(out),
                                  _p(out[B * T:]), _p(out[B * T + B:]), _s()), "eb_ctc_greedy")
    return out


def ctc_align(lp, targets, offsets, tlen, ilen, S, blank):
    """lp [B, T, V] fp32 (unit stride over V, any B / T strides); targets / offsets / tlen / ilen as ctc_loss_fwd.
    Returns (alignment int32 [B, T], frame_logp fp32 [B, T]) on the device (include/edgedict_b200.h)."""
    B, T, V = lp.shape
    ws = torch.empty(lib().eb_ctc_align_workspace_size(B, T, S), dtype=torch.uint8, device=lp.device)
    alignment = torch.empty(B, T, dtype=torch.int32, device=lp.device)
    frame_logp = torch.empty(B, T, dtype=f32, device=lp.device)
    with _timed("ctc_align", 1, 4.0 * B * T * (2 * S + 1), 0.0):
        check(lib().eb_ctc_align(_p(lp), lp.stride(0), lp.stride(1), B, T, V, _p(targets), targets.numel(), _p(offsets),
                                 _p(tlen), _p(ilen), S, blank, _p(ws) if ws.numel() else None, _p(alignment),
                                 _p(frame_logp), _s()), "eb_ctc_align")
    return alignment, frame_logp


def adam_step(p, g, m, v, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0):
    check(lib().eb_adam_step(_p(p), _p(g), _p(m), _p(v), p.numel(), lr, beta1, beta2, eps, weight_decay, step,
                             grad_scale, _s()), "eb_adam_step")


def adam_step_ex(p, g, m, v, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0, sumsq=None, max_norm=0.0,
                 adamw=False):
    check(lib().eb_adam_step_ex(_p(p), _p(g), _p(m), _p(v), p.numel(), lr, beta1, beta2, eps, weight_decay, step,
                                grad_scale, _p(sumsq), float(max_norm or 0.0), int(adamw), _s()), "eb_adam_step_ex")


def sumsq(x, out):
    check(lib().eb_sumsq(_p(x), x.numel(), _p(out), _s()), "eb_sumsq")


# ---- the flat optimizers (optim.FlatOptimizer): seg / tiles are the int64 eb_opt_seg / eb_opt_tile tables, h an
# _lib.OptHyper, ctl float [2], steps int32 [groups] ------------------------------------------------------------------
def opt_seg_sumsq(g, seg, tiles, partial, segsum, total=None):
    check(lib().eb_opt_seg_sumsq(_p(g), _p(seg), seg.shape[0], _p(tiles), tiles.shape[0], _p(partial), _p(segsum),
                                 _p(total), _s()), "eb_opt_seg_sumsq")


def opt_prologue(total, grad_scale, max_norm, steps, ctl):
    check(lib().eb_opt_prologue(_p(total), float(grad_scale), float(max_norm or 0.0), steps.numel(), _p(steps),
                                _p(ctl), _s()), "eb_opt_prologue")


def opt_sgd_step(p, g, buf, seg, tiles, h, steps, ctl):
    check(lib().eb_opt_sgd_step(_p(p), _p(g), _p(buf), _p(seg), _p(tiles), tiles.shape[0], h, steps.numel(), _p(ctl),
                                _p(steps), _s()), "eb_opt_sgd_step")


def opt_sm3_step(p, g, acc, acc_new, seg, tiles, h, steps, ctl):
    check(lib().eb_opt_sm3_step(_p(p), _p(g), _p(acc), _p(acc_new), acc.numel(), _p(seg), _p(tiles), tiles.shape[0], h,
                                steps.numel(), _p(ctl), _s()), "eb_opt_sm3_step")


def opt_adamw_step(p, g, m, v, seg, tiles, h, steps, ctl):
    check(lib().eb_opt_adamw_step(_p(p), _p(g), _p(m), _p(v), _p(seg), _p(tiles), tiles.shape[0], h, steps.numel(),
                                  _p(ctl), _p(steps), _s()), "eb_opt_adamw_step")


def opt_novograd_step(p, g, m, segv, segsum, seg, tiles, h, steps, ctl):
    check(lib().eb_opt_novograd_step(_p(p), _p(g), _p(m), _p(segv), _p(segsum), _p(seg), seg.shape[0], _p(tiles),
                                     tiles.shape[0], h, steps.numel(), _p(ctl), _s()), "eb_opt_novograd_step")


# ---- log-mel front end (SURVEY 8(f) N2) ------------------------------------------------------------
def logmel_frontend(x, basis, fbT, n_fft, hop, n_mels, n_stack, preemph, take_log=True, pad_to_divisible=True):
    """x [B, L] fp32 waveform -> [B, T, n_mels*n_stack] log-mel features (see csrc/frontend.cu).
    basis [n_fft, 2*nbins] = window * (cos | -sin); fbT [nbins, n_mels]."""
    _need(x, f32, "x")
    B, L = x.shape
    nb = n_fft // 2 + 1
    pad = n_fft // 2
    R = -(-(L + 2 * pad) // hop)                       # frame slots per utterance (>= the 1 + L//hop real frames)
    Lp = R * hop
    F = 1 + L // hop
    seq_len = -(-L // hop)
    dev = x.device
    xp = torch.zeros(B * Lp + n_fft, dtype=f32, device=dev)      # tail: the last slots' windows stay in bounds
    check(lib().eb_fe_preemph_pad(_p(x), _p(xp), B, L, Lp, pad, float(preemph or 0.0), int(preemph is not None), _s()),
          "eb_fe_preemph_pad")
    rows = B * R
    spec = gemm_f32(xp, hop, 1, basis, 2 * nb, 1, rows, 2 * nb, n_fft)
    power = torch.empty(rows, nb, dtype=f32, device=dev)
    check(lib().eb_fe_power(_p(spec), _p(power), rows, nb, _s()), "eb_fe_power")
    mel = gemm_f32(power, nb, 1, fbT, n_mels, 1, rows, n_mels, nb)
    Fs = F if pad_to_divisible else F - F % n_stack
    T = -(-Fs // n_stack)
    out = torch.empty(B, T, n_mels * n_stack, dtype=f32, device=dev)
    check(lib().eb_fe_log_stack(_p(mel), _p(out), B, R, Fs, seq_len, n_mels, n_stack, T, int(take_log), _s()),
          "eb_fe_log_stack")
    return out


def fe_lengths(lens, hop, n_stack, pad_to_divisible=True):
    """Host geometry of utterances of lens samples: (frames F_b = 1 + L_b // hop, output rows T_b after stacking)."""
    F = [1 + int(n) // hop for n in lens]
    T = [-(-f // n_stack) if pad_to_divisible else f // n_stack for f in F]
    return F, T


def fe_batch(x, lens, basis, fbT, n_fft, hop, n_stack, preemph=None, dct=None, take_log=False, use_mask=False,
             delta=False, pad_to_divisible=True):
    """Per-utterance features of a padded batch (see csrc/frontend.cu).  x [B, L] fp32 waveforms whose row b holds
    lens[b] samples (lens: host int [B], n_fft//2 < lens[b] <= L); basis [n_fft, 2*nbins] = window * (cos | -sin);
    fbT [nbins, n_mels]; dct [n_mels, n_mfcc] for MFCC (log(mel + 1e-6), then the DCT).  Returns (out [B, T_max,
    C*(3 if delta)*n_stack], T int32 CPU [B]); rows t >= T[b] of utterance b are zero."""
    _need(x, f32, "x")
    for t, name in ((basis, "basis"), (fbT, "fbT"), (dct, "dct")):
        if t is not None:
            _need(t, f32, name)
    B, L = x.shape
    lens = torch.as_tensor(lens).to("cpu", torch.int32).contiguous()
    if tuple(lens.shape) != (B,):
        raise ValueError("lengths must have shape [%d], got %s" % (B, tuple(lens.shape)))
    pad = n_fft // 2
    if int(lens.min()) <= pad or int(lens.max()) > L:
        raise ValueError("every length must be in (n_fft // 2, L] = (%d, %d], got %s" % (pad, L, lens.tolist()))
    nb = n_fft // 2 + 1
    R = -(-(L + 2 * pad) // hop)                       # frame slots per utterance (>= the 1 + L_b//hop real frames)
    Lp = R * hop
    dev = x.device
    lens_dev = lens.to(dev)
    hl = lens.numpy()
    xp = torch.zeros(B * Lp + n_fft, dtype=f32, device=dev)      # tail: the last slots' windows stay in bounds
    check(lib().eb_fe_preemph_pad_lens(_p(x), hl.ctypes.data, _p(lens_dev), _p(xp), B, L, Lp, pad,
                                       float(preemph or 0.0), int(preemph is not None), _s()), "eb_fe_preemph_pad_lens")
    rows = B * R
    spec = gemm_f32(xp, hop, 1, basis, 2 * nb, 1, rows, 2 * nb, n_fft)
    power = torch.empty(rows, nb, dtype=f32, device=dev)
    check(lib().eb_fe_power(_p(spec), _p(power), rows, nb, _s()), "eb_fe_power")
    n_mels = fbT.shape[1]
    feat = gemm_f32(power, nb, 1, fbT, n_mels, 1, rows, n_mels, nb)
    if dct is not None:
        check(lib().eb_fe_log(_p(feat), feat.numel(), 1e-6, _s()), "eb_fe_log")
        feat = gemm_f32(feat, n_mels, 1, dct, dct.shape[1], 1, rows, dct.shape[1], n_mels)
    C = feat.shape[1]
    _, T = fe_lengths(hl, hop, n_stack, pad_to_divisible)
    T_max = max(T)
    out = torch.empty(B, T_max, C * (3 if delta else 1) * n_stack, dtype=f32, device=dev)
    if T_max > 0:
        check(lib().eb_fe_finish(_p(feat), _p(out), hl.ctypes.data, _p(lens_dev), B, R, hop, C, n_stack, T_max,
                                 int(take_log), int(use_mask), int(delta), int(pad_to_divisible), _s()), "eb_fe_finish")
    return out, torch.tensor(T, dtype=torch.int32)


def fe_deltas(feat):
    """CatDeltas on frame-major features: feat [B, F, C] fp32 -> [B, F, 3C] = [x, d1, d2] per frame."""
    _need(feat, f32, "feat")
    B, F, C = feat.shape
    out = torch.empty(B, F, 3 * C, dtype=f32, device=feat.device)
    if out.numel():
        check(lib().eb_fe_deltas(_p(feat), _p(out), B, F, C, _s()), "eb_fe_deltas")
    return out


def fe_mask(x, spans, axis, fill=0.0):
    """SpecAugment masking in place: x [B, D1, D2] fp32, spans int32 [B, nmask, 2] along axis 1 or 2."""
    _need(x, f32, "x")
    B, D1, D2 = x.shape
    check(lib().eb_fe_mask(_p(x), _p(spans), B, D1, D2, spans.shape[1], axis, float(fill), _s()), "eb_fe_mask")
    return x


# ---- raw-waveform front end (csrc/conv.cu) ----------------------------------------------------------------------------
def _gn_slices(B, T, C):
    """(per-channel partial slices, fp64 per-utterance partial slices) of eb_gn_stats / eb_gn_bwd."""
    rps = int(lib().eb_conv_rows_per_split(C))
    ns = B * ((T + rps - 1) // rps)
    return ns, ns * ((C + 255) // 256)


def conv1d_first_fwd(x, w, b, k, s, T):
    """y [B, T, C] = the first layer (C_in = 1) of FrontEnd on x [B, L]; w [C, k]."""
    B, L = x.shape
    C = w.shape[0]
    y = torch.empty(B, T, C, dtype=f32, device=x.device)
    with _timed("conv1d_first_fwd", 1, 4.0 * (x.numel() + y.numel()), 2.0 * y.numel() * k):
        check(lib().eb_conv1d_first_fwd(_p(x), _p(w), _p(b), _p(y), B, L, C, k, s, T, _s()), "eb_conv1d_first_fwd")
    return y


def conv1d_first_dw(x, dy, k, s):
    """(dW [C, k], db [C]) of the first layer from dy [B, T, C]: row splits summed in order."""
    B, L = x.shape
    _, T, C = dy.shape
    rows = B * T
    rps = max(256, -(-rows // 1024))
    ns = -(-rows // rps)
    part = torch.empty(ns, (k + 1) * C, dtype=f32, device=x.device)
    with _timed("conv1d_first_dw", 2, 4.0 * dy.numel(), 2.0 * dy.numel() * (k + 1)):
        check(lib().eb_conv1d_first_dw(_p(x), _p(dy), _p(part), ns, rps, B, L, C, k, s, T, _s()), "eb_conv1d_first_dw")
        tot = colsum(part)
    tot = tot.view(k + 1, C)
    return tot[:k].t().contiguous(), tot[k].contiguous()


def gn_stats(y, ustride, B, T, C, eps=1e-5):
    dpart = torch.empty(_gn_slices(B, T, C)[1], 2, dtype=torch.float64, device=y.device)
    mean = torch.empty(B, dtype=f32, device=y.device)
    rstd = torch.empty(B, dtype=f32, device=y.device)
    with _timed("gn_stats", 2, 4.0 * B * T * C):
        check(lib().eb_gn_stats(_p(y), ustride, B, T, C, _p(dpart), _p(mean), _p(rstd), eps, _s()), "eb_gn_stats")
    return mean, rstd


def gn_apply(y, ustride, B, T, C, mean, rstd, gamma, beta, out, p, rows_per_utt):
    """The padded conv operand (out: flat fp32 or bf16, a whole number of C-rows) from y."""
    total = out.numel() // C
    with _timed("gn_apply", 1, 4.0 * B * T * C + out.element_size() * out.numel()):
        check(lib().eb_gn_apply(_p(y), ustride, B, T, C, _p(mean), _p(rstd), _p(gamma), _p(beta), _p(out),
                                int(out.dtype == bf16), p, rows_per_utt, total, _s()), "eb_gn_apply")
    return out


def gn_bwd(y, ustride, B, T, C, mean, rstd, gamma, dz, dz_off, dz_ustride, dy, dy16, dy_off, dy_ustride, want_db):
    """GroupNorm(1, C) + GELU backward.  dz / dy / dy16 are flat buffers read / written from element offsets dz_off /
    dy_off.  Returns (dgamma, dbeta, db | None): db = the column sums of dy (the bias gradient of the conv below)."""
    ns, nd = _gn_slices(B, T, C)
    dev = y.device
    pg = torch.empty(ns, C, dtype=f32, device=dev)
    pb = torch.empty(ns, C, dtype=f32, device=dev)
    pdb = torch.empty(ns, C, dtype=f32, device=dev) if want_db else None
    dpart = torch.empty(nd, 2, dtype=torch.float64, device=dev)

    def at(t, off):
        return None if t is None else t.data_ptr() + off * t.element_size()

    with _timed("gn_bwd", 5, 8.0 * B * T * C + 6.0 * B * T * C):
        check(lib().eb_gn_bwd(_p(y), ustride, B, T, C, _p(mean), _p(rstd), _p(gamma), at(dz, dz_off), dz_ustride,
                              _p(pg), _p(pb), _p(dpart), at(dy, dy_off), at(dy16, dy_off), dy_ustride, _p(pdb), _s()),
              "eb_gn_bwd")
        dg, dbe = colsum(pg), colsum(pb)
        db = colsum(pdb) if want_db else None
    return dg, dbe, db


def conv1d_bf16(x16, x_off, x_rows, s, C, row0, w16, taps, N, bias, out, out_off, ldc, M):
    """out[m, n] (row pitch ldc, from element out_off) = bias + sum_j X[m + row0 + j/s][j%s] . W[n, j]  (eb_conv1d_bf16)."""
    _need(w16, bf16, "w16")
    with _timed("conv1d_bf16", 1, 2.0 * x_rows * s * C + 4.0 * M * N, 2.0 * M * N * taps * C):
        check(lib().eb_conv1d_bf16(x16.data_ptr() + 2 * x_off, x_rows, s, C, row0, _p(w16), taps, N, _p(bias),
                                   out.data_ptr() + 4 * out_off, ldc, M, _s()), "eb_conv1d_bf16")
    return out


def gemm_f32_at(A, a_off, sam, sak, B, sbk, sbn, out, out_off, ldc, M, N, K, bias=None):
    """eb_gemm_f32 on views starting at element offsets of flat fp32 storage, output row pitch ldc."""
    with _timed("gemm_f32", 1, 0.0, 2.0 * M * N * K):
        check(lib().eb_gemm_f32(A.data_ptr() + 4 * a_off, sam, sak, _p(B), sbk, sbn, out.data_ptr() + 4 * out_off, ldc,
                                _p(bias), M, N, K, 1.0, 0.0, _s()), "eb_gemm_f32")
    return out


def gemm_f32_rows(A, a_off, sam, sak, B, sbk, sbn, M, N, K):
    """[M, N] = A' B' with a long contraction (weight gradients over rows): split in slices, added in order."""
    kchunk = max(1024, -(-K // 128))
    nz = -(-K // kchunk)
    part = torch.empty(nz, M * N, dtype=f32, device=A.device)
    with _timed("gemm_f32_splitk", 2, 0.0, 2.0 * M * N * K):
        check(lib().eb_gemm_f32_splitk(A.data_ptr() + 4 * a_off, sam, sak, _p(B), sbk, sbn, _p(part), M, N, K, kchunk,
                                       _s()), "eb_gemm_f32_splitk")
        out = colsum(part)
    return out.view(M, N)


# ---- wav2vec pre-training head (csrc/w2v.cu) -----------------------------------------------------
def w2v_mask_fwd(x, mask_emb, inv):
    """x [B, T, D] with mask_emb in the masked rows (inv [B, T] int32 >= 0), out of place."""
    _need(x, f32, "x"), _need(mask_emb, f32, "mask_emb"), _need(inv, torch.int32, "inv")
    out = torch.empty_like(x)
    check(lib().eb_w2v_mask_fwd(_p(x), _p(mask_emb), _p(inv), _p(out), inv.numel(), x.shape[-1], _s()),
          "eb_w2v_mask_fwd")
    return out


def w2v_keep_rows(x, inv):
    _need(x, f32, "x"), _need(inv, torch.int32, "inv")
    out = torch.empty_like(x)
    check(lib().eb_w2v_keep_rows(_p(x), _p(inv), _p(out), inv.numel(), x.shape[-1], _s()), "eb_w2v_keep_rows")
    return out


def w2v_gather(x, idx):
    """x [B, T, D], idx [B, M] int32 -> [B, M, D]."""
    _need(x, f32, "x"), _need(idx, torch.int32, "idx")
    B, T, D = x.shape
    M = idx.shape[1]
    out = torch.empty(B, M, D, dtype=f32, device=x.device)
    check(lib().eb_w2v_gather(_p(x), _p(idx), _p(out), B, T, M, D, _s()), "eb_w2v_gather")
    return out


def w2v_scatter(x, inv):
    """x [B, M, D], inv [B, T] int32 -> [B, T, D] (zeros in unmasked rows)."""
    _need(x, f32, "x"), _need(inv, torch.int32, "inv")
    B, M, D = x.shape
    T = inv.shape[1]
    out = torch.empty(B, T, D, dtype=f32, device=x.device)
    check(lib().eb_w2v_scatter(_p(x), _p(inv), _p(out), B, T, M, D, _s()), "eb_w2v_scatter")
    return out


def w2v_sq_mean(x):
    _need(x, f32, "x")
    out = torch.empty((), dtype=f32, device=x.device)
    check(lib().eb_w2v_sq_mean(_p(x), x.numel(), _p(out), _s()), "eb_w2v_sq_mean")
    return out


def w2v_scale(x, g, alpha=1.0, out=None):
    """x * g (a device scalar) * alpha."""
    _need(x, f32, "x"), _need(g, f32, "g")
    out = torch.empty_like(x) if out is None else out
    check(lib().eb_w2v_scale(_p(x), _p(g), float(alpha), x.numel(), _p(out), _s()), "eb_w2v_scale")
    return out


def w2v_quant_fwd(logits, noise, vars, G, tau):
    """logits [N, G*V], noise like logits or None (eval), vars [G*V, vd] -> q [N, G*vd], p, s (None in eval), X,
    k0, k [N, G] int32, st [N, G]."""
    _need(logits, f32, "logits"), _need(vars, f32, "vars")
    if noise is not None:
        _need(noise, f32, "noise")
    N, GV = logits.shape
    V, vd = GV // G, vars.shape[-1]
    dev = logits.device
    q = torch.empty(N, G * vd, dtype=f32, device=dev)
    p, X = torch.empty_like(logits), torch.empty_like(logits)
    s = torch.empty_like(logits) if noise is not None else None
    k0 = torch.empty(N, G, dtype=torch.int32, device=dev)
    k = torch.empty(N, G, dtype=torch.int32, device=dev)
    st = torch.empty(N, G, dtype=f32, device=dev)
    check(lib().eb_w2v_quant_fwd(_p(logits), _p(noise), _p(vars), N, G, V, vd, float(tau), _p(q), _p(p), _p(s), _p(X),
                                 _p(k0), _p(k), _p(st), _s()), "eb_w2v_quant_fwd")
    return q, p, s, X, k0, k, st


def w2v_quant_stats(p, k0, G):
    """-> (out [2] = prob_perplexity, code_perplexity; coef [G*V])."""
    N, GV = p.shape
    psum = colsum(p)
    out = torch.empty(2, dtype=f32, device=p.device)
    coef = torch.empty(GV, dtype=f32, device=p.device)
    counts = torch.empty(GV, dtype=torch.int32, device=p.device)
    check(lib().eb_w2v_quant_stats(_p(psum), _p(k0), N, G, GV // G, _p(out), _p(coef), _p(counts), _s()),
          "eb_w2v_quant_stats")
    return out, coef


def w2v_quant_bwd(dsoft, s, p, coef, g_ppl, G, tau):
    ref = dsoft if dsoft is not None else p
    N, GV = ref.shape
    dl = torch.empty(N, GV, dtype=f32, device=ref.device)
    check(lib().eb_w2v_quant_bwd(_p(dsoft), _p(s), _p(p), _p(coef), _p(g_ppl), N, G, GV // G, float(tau), _p(dl), _s()),
          "eb_w2v_quant_bwd")
    return dl


COS_EPS = 1e-8          # torch.cosine_similarity's default eps


def w2v_logits_fwd(xp, yp, neg, temp):
    """xp, yp [B, M, D], neg [B, M, K] int32 -> logits [K+1, B, M] and the saved (xh, yh, xn, yn, cos)."""
    _need(xp, f32, "xp"), _need(yp, f32, "yp"), _need(neg, torch.int32, "neg")
    B, M, D = xp.shape
    K = neg.shape[-1]
    dev = xp.device
    xh, yh = torch.empty_like(xp), torch.empty_like(yp)
    xn = torch.empty(B, M, dtype=f32, device=dev)
    yn = torch.empty(B, M, dtype=f32, device=dev)
    cos = torch.empty(K + 1, B, M, dtype=f32, device=dev)
    logits = torch.empty(K + 1, B, M, dtype=f32, device=dev)
    check(lib().eb_w2v_logits_fwd(_p(xp), _p(yp), _p(neg), B, M, D, K, float(temp), COS_EPS, _p(xh), _p(yh), _p(xn),
                                  _p(yn), _p(cos), _p(logits), _s()), "eb_w2v_logits_fwd")
    return logits, (xh, yh, xn, yn, cos)


def w2v_logits_bwd(dlogits, cos, neg, xh, yh, xp, yp, xn, yn, temp):
    _need(dlogits, f32, "dlogits")
    B, M, D = xp.shape
    K = neg.shape[-1]
    A = torch.empty(B, M, M, dtype=f32, device=xp.device)
    AC = torch.empty_like(A)
    dxp, dyp = torch.empty_like(xp), torch.empty_like(yp)
    check(lib().eb_w2v_logits_bwd(_p(dlogits), _p(cos), _p(neg), _p(xh), _p(yh), _p(xp), _p(yp), _p(xn), _p(yn), B, M,
                                  D, K, float(temp), COS_EPS, _p(A), _p(AC), _p(dxp), _p(dyp), _s()),
          "eb_w2v_logits_bwd")
    return dxp, dyp


def w2v_ce(logits):
    """logits [C, B, M] -> (grad [C, B, M] of the summed cross-entropy, out [2] = summed loss, correct rows)."""
    _need(logits, f32, "logits")
    C, B, M = logits.shape
    grad = torch.empty_like(logits)
    out = torch.empty(2, dtype=f32, device=logits.device)
    check(lib().eb_w2v_ce(_p(logits), B, M, C, _p(grad), _p(out), _s()), "eb_w2v_ce")
    return grad, out


# ---- minimum word error rate training (csrc/mwer.cu; include/edgedict_b200.h) ------------------------------------
def edit_distance(hyp, ref, meta, meta_host, n_hyp, n_ref, word_table=None, word_chars=None, vocab=0):
    """Counts [n_hyp, 5] int32 {errors, S, D, I, reference length} of hypothesis rows hyp [n_hyp, ld_h] against
    reference rows ref [n_ref, ld_r] (int32, contiguous).  meta int32 on the device = hyp_len | ref_len | ref_index and
    meta_host the same values in host memory (eb_edit_distance checks them); word_table [n_table, 3] / word_chars
    int32 on the device select word units."""
    _need(hyp, torch.int32, "hyp")
    _need(ref, torch.int32, "ref")
    _need(meta, torch.int32, "meta")
    if meta_host.device.type != "cpu" or meta_host.dtype != torch.int32 or not meta_host.is_contiguous():
        raise ValueError("meta_host must be a contiguous int32 host tensor")
    if meta.numel() != 2 * n_hyp + n_ref or meta_host.numel() != meta.numel():
        raise ValueError("meta must hold 2 * n_hyp + n_ref entries")
    out = torch.empty(n_hyp, 5, dtype=torch.int32, device=hyp.device)
    n_table = 0
    if word_table is not None:
        _need(word_table, torch.int32, "word_table")
        _need(word_chars, torch.int32, "word_chars")
        n_table = word_table.shape[0]
    ld_h = hyp.shape[1] if hyp.dim() == 2 else 0
    ld_r = ref.shape[1] if ref.dim() == 2 else 0
    if n_hyp == 0:
        return out
    # an empty row buffer (width 0) is never read: meta stands in for its null pointer
    with _timed("edit_distance"):
        check(lib().eb_edit_distance(hyp.data_ptr() or _p(meta), ld_h, ref.data_ptr() or _p(meta), ld_r, _p(meta),
                                     meta_host.data_ptr(), n_hyp, n_ref, _p(word_table),
                                     _p(word_chars) if word_table is not None else None, n_table, vocab, _p(out), _s()),
              "eb_edit_distance")
    return out


def nbest_pack(ids, count, ref, ref_len, ld_out):
    """ids int32 [B, N, L] (a beam engine's N-best ids), count [B], ref int32 [B, S], ref_len int32 [B] -> (labels
    int32 [B*(N+1), ld_out], lens int32 [B*(N+1)], valid int32 [B, N]) (include/edgedict_b200.h, eb_nbest_pack)."""
    B, N, L = ids.shape
    _need(ids, torch.int32, "ids")
    _need(count, torch.int32, "count")
    _need(ref, torch.int32, "ref")
    _need(ref_len, torch.int32, "ref_len")
    dev = ids.device
    labels = torch.empty(B * (N + 1), ld_out, dtype=torch.int32, device=dev)
    lens = torch.empty(B * (N + 1), dtype=torch.int32, device=dev)
    valid = torch.empty(B, N, dtype=torch.int32, device=dev)
    with _timed("nbest_pack"):
        check(lib().eb_nbest_pack(_p(ids), _p(count), B, N, L, ref.data_ptr() or _p(lens), ref.shape[1], _p(ref_len),
                                  _p(labels), ld_out, _p(lens), _p(valid), _s()), "eb_nbest_pack")
    return labels, lens, valid


def mwer_risk_fwd(costs, errors, valid):
    """costs fp32 [B, N], errors / valid int32 [B, N] -> (loss [1] fp32, posteriors [B, N] fp32, risk [B] fp64)."""
    _need(costs, f32, "costs")
    _need(errors, torch.int32, "errors")
    _need(valid, torch.int32, "valid")
    B, N = costs.shape
    post = torch.empty(B, N, dtype=f32, device=costs.device)
    risk = torch.empty(B, dtype=torch.float64, device=costs.device)
    loss = torch.empty(1, dtype=f32, device=costs.device)
    with _timed("mwer_risk_fwd", 2):
        check(lib().eb_mwer_risk_fwd(_p(costs), _p(errors), _p(valid), B, N, _p(post), _p(risk), _p(loss), _s()),
              "eb_mwer_risk_fwd")
    return loss, post, risk


def mwer_risk_bwd(costs, errors, valid, gout):
    """d loss / d costs [B, N] fp32 for the upstream gradient gout (fp32, one element, on the device)."""
    B, N = costs.shape
    g = gout.to(f32).reshape(1).contiguous()
    dc = torch.empty(B, N, dtype=f32, device=costs.device)
    with _timed("mwer_risk_bwd"):
        check(lib().eb_mwer_risk_bwd(_p(costs), _p(errors), _p(valid), B, N, _p(g), _p(dc), _s()), "eb_mwer_risk_bwd")
    return dc
