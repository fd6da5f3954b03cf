// decode.cu -- streaming greedy decode as ONE persistent kernel per audio chunk (sm_90a).
//
// Replaces the Python loop of PytorchStreamDecoder.decode (rnnt/stream.py:93-120): per chunk the
// reference runs the stateful encoder, then for every encoder frame joint -> argmax(.item(): a
// host sync) -> optional predictor step.  Here the whole chunk for S concurrent streams is a
// "phase program" (built once by the host, edgedict_b200/stream_engine.py) that one cooperative
// kernel walks with a grid barrier between dependent phases -- no launch gaps, no host syncs:
//
//   LN      y = LayerNorm(x1 (+ x2))                 nn.LayerNorm + residual (models.py:47,66-70,124)
//   PAIR    y[s,t/2] = mean(x[s,t], x[s,t+1])        TimeReduction (models.py:21-29)
//   LSTM    one cell step for S streams              nn.LSTM step (models.py:45-46,145-147); the
//           x rows may come from an embedding table indexed by the last token, and the update can
//           be masked per stream (predictor advances only on non-blank, stream.py:111-116)
//   LINEAR  y = act(x1 W1^T (+ x2 W2^T) + b)         Linear / joint (models.py:129,148,163-167)
//   ARGMAX  token = argmax(logits) with the <unk> rule (stream.py:105-108: logit := 0, re-argmax); with flags 256 (a
//           continuation round of a multi-symbol frame) rows whose tok_out already holds blank stay blank
//   COPY    y = x
//   SKIP    if no row of tok_in[0..S) differs from aux2 (blank), jump over the next aux phases: a frame's round j >= 1
//           costs one read of S ints per CTA when no row is still emitting (greedy decoding with max_symbols > 1)
//   BEAM_SELECT  per utterance: log-softmax of its W rows, exact top-W of the live slots' candidates, merge of equal
//           token sequences, new slot log p / tokens / gather sources / history (Transducer.beam_search, one frame);
//           optionally with an LSTM language model's log-probs fused into the candidate values (shallow fusion); with
//           flags 512 one round of several per frame (beam search with max_symbols > 1: closed slots stay, open ones extend)
//   GATHER  y[l, r] = x1[l, src[r]] (and y2[r] = x2[src[r]]): survivors inherit their parent's predictor state
//   BEAM_FINAL  per utterance: best live slot, back-pointer walk through the history, ids and -log p written out
//   BEAM_COMMIT per stream, at the end of a streaming chunk: commit the live hypotheses' common prefix, collapse the
//           beam to its best slot when a stored suffix would outgrow its capacity (or on a flush)
//   GRU     one nn.GRU cell step for S streams (ResLayerNormGRU, models.py:77-116): CTCEncoder's streaming encoder
//   CTC_EMIT per stream: log-softmax, argmax, repeats (carried across chunks) and blanks dropped (CTCEncoder.greedy_decode)
//   FE_*    the feature transform of a chunk of raw audio (framing, direct-DFT product, power, mel / DCT products, MFCC
//           log, log / mask / deltas / stacking into the encoder input), a front-end program run by a GATHER with flags
//           1024 at the head of the chunk program, bit for bit build_batch_transform's features of each stream's window
//
// LINEAR's x1 row divisor (x1_div) lets the W rows of one utterance's beam share its encoder frame without copies.
// fp32-accurate arithmetic throughout: the north star asks for token-for-token identical greedy output, which
// bf16 (or plain tf32) near-ties would break.  The matrix products run on the tensor cores as 3xTF32 split
// products with fp32 accumulation (see tile_mma); everything else is fp32 CUDA-core code.
#include <cooperative_groups.h>
#include "frontend.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int TR = 64, TC = 32;              // tile rows (streams), tile cols
constexpr int NWARP = 8;
constexpr int RED_FLOATS = NWARP * 16 * 4 * 32;      // per-warp partial tiles [warp][16 mma tiles][4 regs][32 lanes]
constexpr int OUT_LD = TC + 1;

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void grid_sync(unsigned* ctr, unsigned target) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(ctr, 1u);
        spin_wait_ge(ctr, target);
    }
    __syncthreads();
}

// ---- fp32-accurate products on the tensor cores: x = hi + lo with hi = tf32(x), lo = tf32(x - hi); a*b is
// evaluated as a_lo*b_hi + a_hi*b_lo + a_hi*b_hi with fp32 accumulation ("3xTF32": the dropped lo*lo term is
// 2^-22 relative, below the fp32 rounding of the accumulation itself).  The decode path has to reproduce the
// reference's fp32 argmax token for token, so bf16 / plain tf32 operands are not an option; the CUDA-core
// version of this kernel spent 3.5 ms per chunk of 64 streams (8.6 GFLOP of fp32 FMAs through a shared-memory
// bound inner loop), this one streams the weights once per phase at mma.sync rate.
__device__ __forceinline__ uint32_t tf32_of(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = tf32_of(x);
    lo = tf32_of(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// four consecutive k of one row (guarded at the end of the row); CG = written earlier in this kernel (bypass L1)
template <bool CG>
__device__ __forceinline__ float4 load_k4(const float* row, int k, int K, bool vec) {
    if (vec && k + 3 < K) {
        const float4* q = reinterpret_cast<const float4*>(row + k);
        return CG ? __ldcg(q) : __ldg(q);
    }
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < K) v.x = CG ? __ldcg(row + k) : __ldg(row + k);
    if (k + 1 < K) v.y = CG ? __ldcg(row + k + 1) : __ldg(row + k + 1);
    if (k + 2 < K) v.z = CG ? __ldcg(row + k + 2) : __ldg(row + k + 2);
    if (k + 3 < K) v.w = CG ? __ldcg(row + k + 3) : __ldg(row + k + 3);
    return v;
}

// acc[mt][nt][4] += A(rows, K) * W(cols, K)^T for one K segment.  The 16-wide k steps of all segments of a tile are
// dealt round-robin to the 8 warps (step_ctr runs across segments); inside a step lane (g = lane/4, t = lane%4) loads
// k0+4t .. k0+4t+3 of its rows as ONE 16-byte load and feeds two m16n8k8 MMAs whose k slots (t, t+4) hold (k0+4t, k0+4t+1)
// resp. (k0+4t+2, k0+4t+3) -- the same permutation of k on both operands, so no shuffle or shared-memory transpose.
template <typename AF, typename BF>
__device__ __forceinline__ void tile_mma(float (&acc)[4][4][4], AF arow, BF brow, int K, int nrows, int ncols, bool avec,
                                         bool bvec, int& step_ctr) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int nmt = (nrows + 15) >> 4;
    const int nsteps = (K + 15) >> 4;
    // this warp's steps of the segment: first, then every NWARP-th
    int i = (w - (step_ctr & (NWARP - 1)) + NWARP) & (NWARP - 1);
    step_ctr += nsteps;
    if (i >= nsteps) return;
    // operand rows are fixed across the steps: resolve the pointers once
    const float* bp[4];
    const float* ap[4][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) bp[nt] = (nt * 8 + g < ncols) ? brow(nt * 8 + g) : nullptr;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
        ap[mt][0] = (mt < nmt && mt * 16 + g < nrows) ? arow(mt * 16 + g) : nullptr;
        ap[mt][1] = (mt < nmt && mt * 16 + g + 8 < nrows) ? arow(mt * 16 + g + 8) : nullptr;
    }
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 bv[4], av[4][2];
    auto fetch = [&](int step) {
        const int k = step * 16 + 4 * t;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) bv[nt] = bp[nt] ? load_k4<false>(bp[nt], k, K, bvec) : zero4;
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
            av[mt][0] = ap[mt][0] ? load_k4<true>(ap[mt][0], k, K, avec) : zero4;
            av[mt][1] = ap[mt][1] ? load_k4<true>(ap[mt][1], k, K, avec) : zero4;
        }
    };
    fetch(i);
    for (; i < nsteps; i += NWARP) {
        // split the operands of this step, then issue the loads of the next one before the MMAs (weights stream from
        // HBM: one step of latency is hidden behind 96 MMAs)
        uint32_t bh[4][4], bl[4][4], ah[4][2][4], al[4][2][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            split_tf32(bv[nt].x, bh[nt][0], bl[nt][0]);
            split_tf32(bv[nt].y, bh[nt][1], bl[nt][1]);
            split_tf32(bv[nt].z, bh[nt][2], bl[nt][2]);
            split_tf32(bv[nt].w, bh[nt][3], bl[nt][3]);
        }
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
            const float4 a0 = av[mt][0], a1 = av[mt][1];
            split_tf32(a0.x, ah[mt][0][0], al[mt][0][0]); split_tf32(a1.x, ah[mt][0][1], al[mt][0][1]);
            split_tf32(a0.y, ah[mt][0][2], al[mt][0][2]); split_tf32(a1.y, ah[mt][0][3], al[mt][0][3]);
            split_tf32(a0.z, ah[mt][1][0], al[mt][1][0]); split_tf32(a1.z, ah[mt][1][1], al[mt][1][1]);
            split_tf32(a0.w, ah[mt][1][2], al[mt][1][2]); split_tf32(a1.w, ah[mt][1][3], al[mt][1][3]);
        }
        if (i + NWARP < nsteps) fetch(i + NWARP);
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
            if (mt < nmt) {
#pragma unroll
                for (int e = 0; e < 2; ++e)
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        mma_tf32(acc[mt][nt], al[mt][e], bh[nt][2 * e], bh[nt][2 * e + 1]);
                        mma_tf32(acc[mt][nt], ah[mt][e], bl[nt][2 * e], bl[nt][2 * e + 1]);
                        mma_tf32(acc[mt][nt], ah[mt][e], bh[nt][2 * e], bh[nt][2 * e + 1]);
                    }
            }
        }
    }
}

__device__ __forceinline__ bool vec_ok(const void* base, long ld, int K) {
    return ((reinterpret_cast<uintptr_t>(base) & 15) == 0) && (ld % 4 == 0) && (K % 4 == 0);
}

// sum the 8 warps' partial tiles and lay the [64 rows][32 cols] result out row-major in `outs`
__device__ __forceinline__ void tile_reduce(float (&acc)[4][4][4], float* red, float* outs) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, tid = threadIdx.x;
    __syncthreads();                                         // previous tile's readers are done with red / outs
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) red[((w * 16 + mt * 4 + nt) * 4 + i) * 32 + lane] = acc[mt][nt][i];
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const int e = q * 256 + tid;                         // (tile, reg, lane) flat
        float s = 0.f;
#pragma unroll
        for (int ww = 0; ww < NWARP; ++ww) s += red[ww * 2048 + e];
        const int ln = e & 31, i = (e >> 5) & 3, tile = e >> 7;
        const int row = (tile >> 2) * 16 + (ln >> 2) + ((i >> 1) << 3);
        const int col = (tile & 3) * 8 + (ln & 3) * 2 + (i & 1);
        outs[row * OUT_LD + col] = s;
    }
    __syncthreads();
}

__device__ void phase_lstm(const EbPhase& p, float* red, float* outs) {
    const int S = p.S, H = p.N;
    const int ctiles = (H + 7) / 8, rtiles = (S + TR - 1) / TR;
    const int tid = threadIdx.x;
    const bool embed = p.flags & 2;
    const bool a1vec = vec_ok(p.x1, p.ldx1, p.K1), a2vec = vec_ok(p.x2, p.ldx2, p.K2);
    const bool b1vec = vec_ok(p.w1, p.ldw1, p.K1), b2vec = vec_ok(p.w2, p.ldw2, p.K2);
    for (int tile = blockIdx.x; tile < ctiles * rtiles; tile += gridDim.x) {
        const int s0 = (tile / ctiles) * TR, j0 = (tile % ctiles) * 8;
        const int nrows = min(TR, S - s0), nunits = min(8, H - j0);
        float acc[4][4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
        auto x1row = [&](int r) -> const float* {
            if (embed) {                                     // embedding row of the last token; none (zeros) below 0
                const int k = __ldcg(p.tok_in + s0 + r);
                return k < 0 ? nullptr : p.x1 + (long)k * p.ldx1;
            }
            return p.x1 + (long)(s0 + r) * p.ldx1;
        };
        auto hrow = [&](int r) -> const float* { return p.x2 + (long)(s0 + r) * p.ldx2; };
        auto w1row = [&](int n) -> const float* { return p.w1 + ((long)(n & 3) * H + j0 + (n >> 2)) * p.ldw1; };
        auto w2row = [&](int n) -> const float* { return p.w2 + ((long)(n & 3) * H + j0 + (n >> 2)) * p.ldw2; };
        int step = 0;
        tile_mma(acc, x1row, w1row, p.K1, nrows, nunits * 4, a1vec, b1vec, step);
        tile_mma(acc, hrow, w2row, p.K2, nrows, nunits * 4, a2vec, b2vec, step);
        tile_reduce(acc, red, outs);
        // 64 rows x 8 units = 512 (row, unit) pairs: two per thread
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int e = q * 256 + tid;
            const int r = e >> 3, u = e & 7;
            const int s = s0 + r;
            if (r >= nrows || u >= nunits) continue;
            const int j = j0 + u;
            const bool active = !(p.flags & 4) || (__ldcg(p.tok_in + s) != p.aux);
            float hn;
            if (active) {
                float g4[4];
#pragma unroll
                for (int g = 0; g < 4; ++g) g4[g] = outs[r * OUT_LD + u * 4 + g] + p.b1[(long)g * H + j] + p.b2[(long)g * H + j];
                const float ig = sigmoidf_(g4[0]), fg = sigmoidf_(g4[1]), gg = tanhf(g4[2]), og = sigmoidf_(g4[3]);
                const float cn = fg * __ldcg(p.c + (long)s * H + j) + ig * gg;
                p.c[(long)s * H + j] = cn;
                hn = og * tanhf(cn);
            } else {
                hn = __ldcg(p.x2 + (long)s * p.ldx2 + j);
            }
            p.y[(long)s * p.ldy + j] = hn;
            if (p.y2) p.y2[(long)s * H + j] = hn;
        }
    }
}

// GRU: one nn.GRU cell step for S rows, gate order r|z|n (w1 = W_ih [3H, K1], w2 = W_hh [3H, K2 = H], b1 = b_ih,
// b2 = b_hh, h read from x2).  LSTM's tile: each of a tile's 8 units takes 4 columns, r, z, n_x (x W_in alone) and n_h
// (h W_hn alone); the rows a column does not use are nullptr, which tile_mma reads as zeros, so a step streams the
// 3H (K1 + K2) weights once.  r and z add b1 then b2 as LSTM's gates do; n = tanh((n_x + b_in) + r (n_h + b_hn)) keeps
// b_hn inside the reset product (nn.GRU); h' = (1 - z) n + z h.
__device__ void phase_gru(const EbPhase& p, float* red, float* outs) {
    const int S = p.S, H = p.N;
    const int ctiles = (H + 7) / 8, rtiles = (S + TR - 1) / TR;
    const int tid = threadIdx.x;
    const bool a1vec = vec_ok(p.x1, p.ldx1, p.K1), a2vec = vec_ok(p.x2, p.ldx2, p.K2);
    const bool b1vec = vec_ok(p.w1, p.ldw1, p.K1), b2vec = vec_ok(p.w2, p.ldw2, p.K2);
    for (int tile = blockIdx.x; tile < ctiles * rtiles; tile += gridDim.x) {
        const int s0 = (tile / ctiles) * TR, j0 = (tile % ctiles) * 8;
        const int nrows = min(TR, S - s0), nunits = min(8, H - j0);
        float acc[4][4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
        auto x1row = [&](int r) -> const float* { return p.x1 + (long)(s0 + r) * p.ldx1; };
        auto hrow = [&](int r) -> const float* { return p.x2 + (long)(s0 + r) * p.ldx2; };
        // column n = 4 u + g: g = 0 r, 1 z, 2 n_x (W_ih rows only), 3 n_h (W_hh rows only)
        auto w1row = [&](int n) -> const float* {
            const int g = n & 3;
            return g == 3 ? nullptr : p.w1 + ((long)g * H + j0 + (n >> 2)) * p.ldw1;
        };
        auto w2row = [&](int n) -> const float* {
            const int g = n & 3;
            return g == 2 ? nullptr : p.w2 + ((long)(g == 3 ? 2 : g) * H + j0 + (n >> 2)) * p.ldw2;
        };
        int step = 0;
        tile_mma(acc, x1row, w1row, p.K1, nrows, nunits * 4, a1vec, b1vec, step);
        tile_mma(acc, hrow, w2row, p.K2, nrows, nunits * 4, a2vec, b2vec, step);
        tile_reduce(acc, red, outs);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int e = q * 256 + tid;
            const int r = e >> 3, u = e & 7;
            const int s = s0 + r;
            if (r >= nrows || u >= nunits) continue;
            const int j = j0 + u;
            const float* o = outs + r * OUT_LD + u * 4;
            const float rg = sigmoidf_(o[0] + p.b1[j] + p.b2[j]);
            const float zg = sigmoidf_(o[1] + p.b1[(long)H + j] + p.b2[(long)H + j]);
            const float ng = tanhf((o[2] + p.b1[2L * H + j]) + rg * (o[3] + p.b2[2L * H + j]));
            const float hp = __ldcg(p.x2 + (long)s * p.ldx2 + j);
            const float hn = (1.f - zg) * ng + zg * hp;
            p.y[(long)s * p.ldy + j] = hn;
            if (p.y2) p.y2[(long)s * H + j] = hn;
        }
    }
}

__device__ void phase_linear(const EbPhase& p, float* red, float* outs) {
    const int S = p.S, N = p.N;
    const int ctiles = (N + TC - 1) / TC, rtiles = (S + TR - 1) / TR;
    const int tid = threadIdx.x;
    const bool a1vec = vec_ok(p.x1, p.ldx1, p.K1), b1vec = vec_ok(p.w1, p.ldw1, p.K1);
    const bool a2vec = p.K2 > 0 && vec_ok(p.x2, p.ldx2, p.K2), b2vec = p.K2 > 0 && vec_ok(p.w2, p.ldw2, p.K2);
    for (int tile = blockIdx.x; tile < ctiles * rtiles; tile += gridDim.x) {
        const int s0 = (tile / ctiles) * TR, n0 = (tile % ctiles) * TC;
        const int nrows = min(TR, S - s0), ncols = min(TC, N - n0);
        float acc[4][4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
        auto x1row = [&](int r) -> const float* {
            return p.x1 + (long)(p.x1_div > 1 ? (s0 + r) / p.x1_div : s0 + r) * p.ldx1;
        };
        auto w1row = [&](int n) -> const float* { return p.w1 + (long)(n0 + n) * p.ldw1; };
        int step = 0;
        tile_mma(acc, x1row, w1row, p.K1, nrows, ncols, a1vec, b1vec, step);
        if (p.K2 > 0) {
            auto x2row = [&](int r) -> const float* { return p.x2 + (long)(s0 + r) * p.ldx2; };
            auto w2row = [&](int n) -> const float* { return p.w2 + (long)(n0 + n) * p.ldw2; };
            tile_mma(acc, x2row, w2row, p.K2, nrows, ncols, a2vec, b2vec, step);
        }
        tile_reduce(acc, red, outs);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int e = q * 256 + tid;
            const int r = e >> 5, c = e & 31;
            if (r >= nrows || c >= ncols) continue;
            float v = outs[r * OUT_LD + c] + (p.b1 ? p.b1[n0 + c] : 0.f);
            if (p.flags & 1) v = tanhf(v);
            p.y[(long)(s0 + r) * p.ldy + n0 + c] = v;
        }
    }
}

__device__ void phase_ln(const EbPhase& p) {
    const int lane = threadIdx.x & 31, H = p.N;
    for (int r = blockIdx.x * 8 + (threadIdx.x >> 5); r < p.S; r += gridDim.x * 8) {
        const float* x = p.x1 + (long)r * p.ldx1;
        const float* x2 = p.x2 ? p.x2 + (long)r * p.ldx2 : nullptr;
        float s = 0.f;
        for (int c = lane; c < H; c += 32) s += __ldcg(x + c) + (x2 ? __ldcg(x2 + c) : 0.f);
        const float mu = warp_sum(s) / H;
        float q = 0.f;
        for (int c = lane; c < H; c += 32) {
            float d = __ldcg(x + c) + (x2 ? __ldcg(x2 + c) : 0.f) - mu;
            q += d * d;
        }
        const float rs = rsqrtf(warp_sum(q) / H + 1e-5f);
        for (int c = lane; c < H; c += 32) {
            float z = __ldcg(x + c) + (x2 ? __ldcg(x2 + c) : 0.f);
            p.y[(long)r * p.ldy + c] = (z - mu) * rs * p.w1[c] + p.b1[c];
        }
    }
}

// (v, i) ranks above (b, bi) in torch.argmax's order: NaN above every number, then by value, ties to the lower index
__device__ __forceinline__ bool argmax_before(float v, int i, float b, int bi) {
    if (isnan(v)) return !isnan(b) || i < bi;
    if (isnan(b)) return false;
    return v > b || (v == b && i < bi);
}

__device__ void phase_argmax(const EbPhase& p) {
    const int lane = threadIdx.x & 31, V = p.N, blank = p.aux, unk = p.aux2;
    const bool cont = p.flags & 256;
    for (int s = blockIdx.x * 8 + (threadIdx.x >> 5); s < p.S; s += gridDim.x * 8) {
        // continuation round of a multi-symbol frame (flags 256): a row whose frame already ended on blank stays blank,
        // takes no argmax and adds no log p; its masked predictor phases then leave it untouched
        if (cont && __ldcg(p.tok_out + s) == blank) {
            if (lane == 0 && p.hist) p.hist[(long)s * p.hist_ld + p.hist_col] = blank;
            continue;
        }
        const float* x = p.x1 + (long)s * p.ldx1;
        int pred = -1;
        for (int pass = 0; pass < 2; ++pass) {
            // the sentinel index loses every tie, so an all -inf row gives index 0 and a lane without columns
            // (V < 32) never wins: the token is always in [0, V)
            float best = -INFINITY;
            int bi = 0x7fffffff;
            for (int v = lane; v < V; v += 32) {
                float val = __ldcg(x + v);
                if (pass == 1 && v == pred) val = 0.f;              // stream.py:107 `prob[:, pred] = 0`
                if (argmax_before(val, v, best, bi)) { best = val; bi = v; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                float ob = __shfl_xor_sync(0xffffffffu, best, o);
                int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (argmax_before(ob, oi, best, bi)) { best = ob; bi = oi; }
            }
            pred = bi;
            if (pred != unk) break;
        }
        if (p.flags & 8) {                                     // batched greedy (models.py:253-255): accumulate
            const float best = __ldcg(x + pred);               // log_softmax(x)[pred] = -log sum exp(x - max)
            float sum = 0.f;
            for (int v = lane; v < V; v += 32) sum += expf(__ldcg(x + v) - best);
            sum = warp_sum(sum);
            if (lane == 0) p.y[s] += -logf(sum);
        }
        if (lane == 0) {
            p.tok_out[s] = pred;
            if (p.hist) p.hist[(long)s * p.hist_ld + p.hist_col] = pred;
        }
    }
}

// CTC_EMIT: greedy CTC emission of one streaming chunk (CTCEncoder.greedy_decode, rnnt/models.py:294-310, carried across
// chunks), one warp per stream.  Field use: S streams, aux = n frames (row s*n + t), N = V, aux2 = blank; x1 logits
// (ldx1); y log-probs out (ldy), each row as eb_log_softmax_fwd forms it, (x - max) - log(sum exp(x - max)); tok_out [S]
// the previous frame's argmax (in / out; a negative value after a reset matches no token); hist ids [S, hist_ld] and
// tok_out2 counts [S]; y2 the running score [S] as DOUBLE, += the fp32 whole-row sum of every kept frame's log-probs;
// seq_out (optional) the argmax of every frame [S, n].  A frame is kept when its argmax (torch.argmax order over the
// log-probs: NaN first, ties to the lowest id) is not blank and differs from the previous frame's.
__device__ __noinline__ void phase_ctc_emit(const EbPhase& p) {
    const int lane = threadIdx.x & 31, V = p.N, n = p.aux, blank = p.aux2;
    double* score = reinterpret_cast<double*>(p.y2);
    for (int s = blockIdx.x * 8 + (threadIdx.x >> 5); s < p.S; s += gridDim.x * 8) {
        int prev = __ldcg(p.tok_out + s), cnt = 0;
        double acc = 0.0;
        for (int t = 0; t < n; ++t) {
            const long row = (long)s * n + t;
            const float* x = p.x1 + row * p.ldx1;
            float* lp = p.y + row * p.ldy;
            float m = -INFINITY;
            for (int v = lane; v < V; v += 32) m = fmaxf(m, __ldcg(x + v));
            m = warp_max(m);
            float e = 0.f;
            for (int v = lane; v < V; v += 32) e += expf(__ldcg(x + v) - m);
            const float ls = logf(warp_sum(e));
            float best = -INFINITY, sum = 0.f;
            int bi = 0x7fffffff;
            for (int v = lane; v < V; v += 32) {
                const float val = (__ldcg(x + v) - m) - ls;
                lp[v] = val;
                if (argmax_before(val, v, best, bi)) { best = val; bi = v; }
                sum += val;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (argmax_before(ob, oi, best, bi)) { best = ob; bi = oi; }
            }
            sum = warp_sum(sum);
            if (bi != blank && bi != prev) {
                if (lane == 0) p.hist[(long)s * p.hist_ld + cnt] = bi;
                ++cnt;
                acc += (double)sum;
            }
            if (lane == 0 && p.seq_out) p.seq_out[row] = bi;
            prev = bi;
        }
        if (lane == 0) {
            p.tok_out[s] = prev;
            p.tok_out2[s] = cnt;
            score[s] += acc;
        }
    }
}

// ---- front end: the feature transform of a streaming chunk of raw audio, at the head of the chunk program.  Each value
// is computed by frontend.cuh's expression for it, and the products keep eb_gemm_f32's order, so the model input equals
// bit for bit what build_batch_transform's module (ops.fe_batch) gives each stream's window.  Field use:
//   FE_FRAME  S streams of N samples (x1 [S, N]; x2, optional, the dither noise [S, N]; fuse = {dither, preemph}):
//             y [S, ldy] = the dithered fl(x + fl(dither * noise)), pre-emphasised (flags 1) and reflect-padded by K1
//             samples, zero past N + 2 K1;
//   FE_GEMM   y [S, N] (ldy) = A [S, K1] B [K1, N], A(m, k) = x1[(m / aux) ldx1 + (m % aux) ldx2 + k] (aux rows per
//             group: the strided frames of a padded signal, or plain rows), B(k, n) = w1[k ldw1 + n]; per output the
//             k-ascending fmaf chain from 0.f over K1 rounded up to a multiple of 16 with zero operands (sgemm_kernel's);
//   FE_POWER  y [S, N] = |X|^2 of the rows x1 [S, 2N] = [re | im];
//   FE_LOG    y [S*N] = log(x1 + 1e-6) (MFCC's log of the mel power, in place allowed);
//   FE_FINISH S streams of K1 per-frame rows x1 [S*K1, N] -> y [S, aux2, W] (ldy = aux2 * W, W = N (3 with flags 2)
//             aux): stacks of aux frames, with the log (flags 1) and deltas (flags 2); hist_ld = F frames, hist_col =
//             Fs frames kept, x1_div = the frame the seq_len mask starts at.
// They are not phases of the kernel's loop but of a front-end program that the GATHER opening a chunk program runs
// (flags 1024, fe_program).
constexpr int FE_BM = 64, FE_BN = 64, FE_BK = 16, FE_LD = FE_BM + 4;
static_assert(2 * FE_BK * FE_LD <= RED_FLOATS + TR * OUT_LD, "front-end product tiles");

__device__ __forceinline__ void fe_gemm(const EbPhase& p, float* sm) {
    float* As = sm;                                          // [FE_BK][FE_LD]: As[k][m]
    float* Bs = sm + FE_BK * FE_LD;                          // [FE_BK][FE_LD]: Bs[k][n]
    const int M = p.S, N = p.N, K = p.K1, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const int ntn = (N + FE_BN - 1) / FE_BN, ntiles = ((M + FE_BM - 1) / FE_BM) * ntn;
    const int ak = tid & 15, bk = tid >> 6, bn = tid & 63;   // A: 4 rows (tid / 16 + 16 r) at k ak; B: 4 k at col bn
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int m0 = (tile / ntn) * FE_BM, n0 = (tile % ntn) * FE_BN;
        const float* arow[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int m = m0 + ty + 16 * r;
            arow[r] = m < M ? p.x1 + (long)(m / p.aux) * p.ldx1 + (long)(m % p.aux) * p.ldx2 : nullptr;
        }
        const bool bcol = n0 + bn < N;
        float ra[4], rb[4];
        auto fetch = [&](int k0) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                ra[r] = arow[r] && k0 + ak < K ? __ldcg(arow[r] + k0 + ak) : 0.f;
                const int k = k0 + bk + 4 * r;
                rb[r] = bcol && k < K ? __ldg(p.w1 + (long)k * p.ldw1 + n0 + bn) : 0.f;
            }
        };
        float acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
        fetch(0);
        for (int k0 = 0; k0 < K; k0 += FE_BK) {
            __syncthreads();                                 // the previous step's readers are done with the tiles
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                As[ak * FE_LD + ty + 16 * r] = ra[r];
                Bs[(bk + 4 * r) * FE_LD + bn] = rb[r];
            }
            __syncthreads();
            if (k0 + FE_BK < K) fetch(k0 + FE_BK);
#pragma unroll
            for (int k = 0; k < FE_BK; ++k) {
                const float4 a4 = *reinterpret_cast<const float4*>(As + k * FE_LD + ty * 4);
                const float4 b4 = *reinterpret_cast<const float4*>(Bs + k * FE_LD + tx * 4);
                const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = m0 + ty * 4 + i;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = n0 + tx * 4 + j;
                if (m < M && n < N) p.y[(long)m * p.ldy + n] = acc[i][j];
            }
        }
    }
}

__device__ __forceinline__ void phase_fe(const EbPhase& p, float* sm) {
    const long gtid = (long)blockIdx.x * blockDim.x + threadIdx.x, gn = (long)gridDim.x * blockDim.x;
    switch (p.type) {
        case EB_PH_FE_FRAME: {
            const int L = p.N, pad = p.K1;
            const long Lp = p.ldy;
            const float dither = __ldg(p.fuse), preemph = __ldg(p.fuse + 1);
            for (long k = gtid; k < (long)p.S * Lp; k += gn) {
                const long s = k / Lp, i = k % Lp;
                const float* x = p.x1 + s * L;
                const float* nz = p.x2 ? p.x2 + s * L : nullptr;
                // FilterbankFeatures._batch: x + dither * randn_like(x), two roundings (torch's mul, then its add)
                auto sample = [&](long r) {
                    return nz ? __fadd_rn(__ldg(x + r), __fmul_rn(dither, __ldg(nz + r))) : __ldg(x + r);
                };
                p.y[k] = fe_framed_sample(sample, i, L, pad, preemph, p.flags & 1);
            }
        } break;
        case EB_PH_FE_GEMM: fe_gemm(p, sm); break;
        case EB_PH_FE_POWER:
            for (long k = gtid; k < (long)p.S * p.N; k += gn) {
                const long g = k / p.N;
                const int b = (int)(k % p.N);
                p.y[k] = fe_power_value(__ldcg(p.x1 + g * 2 * p.N + b), __ldcg(p.x1 + g * 2 * p.N + p.N + b));
            }
            break;
        case EB_PH_FE_LOG:
            for (long k = gtid; k < (long)p.S * p.N; k += gn) p.y[k] = fe_log_value(__ldcg(p.x1 + k), 1e-6f);
            break;
        case EB_PH_FE_FINISH: {
            const int C = p.N, n_frame = p.aux, Tout = p.aux2, take_log = p.flags & 1, delta = (p.flags >> 1) & 1;
            const int W = (delta ? 3 * C : C) * n_frame;
            for (long k = gtid; k < (long)p.S * Tout * W; k += gn) {
                const long s = k / ((long)Tout * W), i = k % ((long)Tout * W);
                const float* rows = p.x1 + s * p.K1 * C;
                p.y[k] = fe_finish_value([&](long e) { return __ldcg(rows + e); }, (int)(i / W), (int)(i % W),
                                         p.hist_ld, p.hist_col, p.x1_div, C, n_frame, take_log, delta);
            }
        } break;
        default: break;
    }
}

// The front-end program of a chunk (K1 phases at x1), run by the GATHER with flags 1024 that opens the chunk program:
// each phase is closed by a grid barrier on the counter tok_out (the entry zeroes it at every launch), the last one
// included.  Run from inside the __noinline__ GATHER, the front end leaves the phase loop's code as it was: any new call
// site or phase case in the loop, whose matrix phases are compiled at the register cap, costs 4 - 40 more bytes of
// spills in some of the kernel's instantiations.
__device__ __forceinline__ void fe_program(const EbPhase& head) {
    extern __shared__ __align__(16) float dsm[];
    __shared__ EbPhase ph;
    const EbPhase* prog = reinterpret_cast<const EbPhase*>(head.x1);
    unsigned* bar = reinterpret_cast<unsigned*>(head.tok_out);
    for (int i = 0; i < head.K1; ++i) {
        __syncthreads();
        if (threadIdx.x < sizeof(EbPhase) / 4)
            reinterpret_cast<int*>(&ph)[threadIdx.x] = reinterpret_cast<const int*>(prog + i)[threadIdx.x];
        __syncthreads();
        phase_fe(ph, dsm);
        grid_sync(bar, (unsigned)(i + 1) * gridDim.x);
    }
}

// ---- beam search: B utterances x W slots, row r = b*W + slot, T' = hist_ld frames.  Field use:
//   BEAM_SELECT (S = B, aux = W, N = V, aux2 = blank, hist_col = t, flags 16 = merge): x1 logits [B*W, V] (ldx1);
//     y slot log p [B*W] (in/out, dead slots -inf); tok_in frames [B]; tok_out token per row (blank for dead and
//     frozen rows, so the masked predictor skips them); src gather source row [B*W]; seq_in / seq_out token
//     sequences [B*W][T'+3] = {len, hash lo, hash hi, tokens} of frame t-1 / t (two buffers alternating by frame);
//     hist = parent slot [B,T',W] | token [B,T',W] | log p (fp32 bits) [B,T',W] | live count [B,T'], back to back.
//     Slots 0..live-1 are live.  Frozen frames (t >= frames[b]) write an identity history entry.
//     flags 32 = LM fusion: x2 LM logits [B*W, K2] (ldx2), fuse {lm_weight, length_bonus}, tok_map [V] -> LM token or
//     -1, tok_out2 LM token per row (-1 where the LM rests, its masked step's sentinel).
//   BEAM_FINAL (S = B, aux = W, aux2 = blank): y slot log p; hist; tok_out ids [B][ldy], the non-blank tokens of the
//     best live slot right-aligned in the row and -1 before them; y2 -log p of that slot [B].  N-best (all unused, so
//     zero / NULL, by the best-only program): K1 = N ranks (0: 1), tok_out ids [B*N][ldy] and y2 [B*N] per rank;
//     seq_out (optional) each token's frame [B*N][ldy] (column / ldw2, ldw2 = K columns per frame, 0: 1); tok_out2
//     (optional) the count min(N, live) [B].
//   BEAM_COMMIT (S = B streams, aux = W, N = max_pending, aux2 = max_pending - n_out, K1 = sequence row stride, K2 = the
//     row's head before its tokens (0: 3, BEAM_SELECT's {len, hash lo, hash hi}; CTC_SEQ_HEAD = 5 for CTC_BEAM's rows),
//     hist_ld = T', flags 128 = collapse unconditionally): y slot value (in/out: log p, or CTC_BEAM's ranking value);
//     hist (reads and rewrites the live count of column T'-1); seq_in / seq_out sequence rows before / after the commit
//     (distinct buffers); tok_out committed tokens [B][N]; tok_out2 committed count [B] | collapsed 0/1 [B]; src gather
//     source row [B*W]; y2 (optional, int32 [B]) each stream's last committed token, rewritten when it commits any.
//   Several symbols per frame (BEAM_SELECT flags 512, ldw2 = K rounds per frame): hist_col = t*K + j is round j of
//     frame t, hist_ld = T'*K columns.  The live count is read from and written to the last column, hist_live[b,
//     hist_ld - 1], in every round (the host sets it before the launch), and each round a row takes also records it in
//     its own column.  A round a row does not take (frozen, its frame ended, or SKIP jumped over it) writes no history:
//     the host fills parent = slot, token = blank beforehand.  BEAM_FINAL and BEAM_COMMIT need no change.
//   Contextual biasing (flags 2048, BEAM_SELECT / CTC_BEAM / BEAM_FINAL / BEAM_COMMIT; DESIGN.md 4e): ctx -> EbContext
//     {next, delta [n_states, V], pending [n_states], state[2] [B*W]}.  A non-blank candidate of slot q adds
//     delta[state(q), k] to its fusion term; each survivor's state goes to the other parity; BEAM_FINAL ranks by
//     y - pending[state], the states read from parity hist_col; BEAM_COMMIT reads the states from parity 1, collapses
//     by y - pending[state] and writes them, moved by src, to parity 0.
// They run one CTA per utterance (grid-strided over B).  They are __noinline__ so that their registers do not
// count against the tensor-core phases the streaming decode spends its time in.
constexpr int BEAM_MAX_W = EB_BEAM_MAX_W;
constexpr unsigned long long SEQ_HASH_MUL = 0x100000001b3ull;      // polynomial hash: h' = h * MUL + (token + 1)
// BEAM_SELECT's shared memory (2 x u64 + 13 x 32-bit arrays of BEAM_MAX_W, histogram, scalars) lives in the dynamic
// shared memory the matrix phases use
static_assert(BEAM_MAX_W * (2 * 8 + 13 * 4) + 256 * 4 + 8 * 4 <= (RED_FLOATS + TR * OUT_LD) * 4, "beam smem");

// order-preserving map of a float to uint32 (larger float -> larger key); -0 ranks with +0 as in a float compare
__device__ __forceinline__ uint32_t order_key(float v) {
    if (v == 0.f) v = 0.f;
    const uint32_t b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
// low half of a candidate's composite key: the lowest flat index ranks first (the map is its own inverse)
__device__ __forceinline__ unsigned tie_key(unsigned flat) { return 0xffffffffu - flat; }
// torch.logaddexp
__device__ __forceinline__ float logaddexp_(float a, float b) {
    const float m = fmaxf(a, b);
    if (m == -INFINITY) return m;
    return m + log1pf(expf(-fabsf(a - b)));
}
// s2 == s1 + [k1], exactly (rows of the sequence buffer)
__device__ bool seq_extends(const int* s2, const int* s1, int k1) {
    const int n1 = __ldcg(s1);
    if (__ldcg(s2) != n1 + 1 || __ldcg(s2 + 3 + n1) != k1) return false;
    for (int i = 0; i < n1; ++i)
        if (__ldcg(s2 + 3 + i) != __ldcg(s1 + 3 + i)) return false;
    return true;
}
// s1 + [e1] == s2 + [e2] exactly, where e < 0 appends nothing; the caller has checked that the lengths are equal
__device__ bool seq_equal_ext(const int* s1, int e1, const int* s2, int e2) {
    const int n1 = __ldcg(s1), n2 = __ldcg(s2), n = n1 + (e1 >= 0);
    for (int i = 0; i < n; ++i)
        if ((i < n1 ? __ldcg(s1 + 3 + i) : e1) != (i < n2 ? __ldcg(s2 + 3 + i) : e2)) return false;
    return true;
}

// N-gram shallow fusion (flags 4096, BEAM_SELECT / CTC_BEAM / BEAM_FINAL; DESIGN.md 4f): ng -> EbNgram.  ngram_rows
// builds, for the slots q < n with want(q), row r0 + q of the workspace: g(state(q), k) for every token k in the fp32
// order of the backoff rule.  It starts from the unigram row and, for each state of the slot's suffix chain from depth
// 1 up to state(q), does row = bo + row over all V tokens, then overwrites that state's children with their p: depth * V
// adds per slot, one pass per chain level for all slots, two __syncthreads per level.  All threads of the CTA call it;
// it ends at a __syncthreads, after which the rows are read like the logits.
template <class State, class Want>
__device__ void ngram_rows(const EbNgram* ng, long r0, int n, int V, State state, Want want, int* smax) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const int *depth = ng->depth, *suffix = ng->suffix;
    float* rows = ng->row;
    if (tid == 0) *smax = 0;
    __syncthreads();
    int dmax = 0;
    for (int q = tid; q < n; q += nt)
        if (want(q)) dmax = max(dmax, __ldg(depth + state(q)));
    if (dmax) atomicMax(smax, dmax);
    for (int q = 0; q < n; ++q) {
        if (!want(q)) continue;
        float* row = rows + (r0 + q) * V;
        for (int k = tid; k < V; k += nt) row[k] = __ldg(ng->unigram + k);
    }
    __syncthreads();
    const int D = *smax;
    for (int i = 1; i <= D; ++i)
        for (int pass = 0; pass < 2; ++pass) {           // bo + row, then the children of the level-i state
            for (int q = 0; q < n; ++q) {
                if (!want(q)) continue;
                int s = state(q), d = __ldg(depth + s);
                if (d < i) continue;
                for (; d > i; --d) s = __ldg(suffix + s);
                float* row = rows + (r0 + q) * V;
                if (pass == 0) {
                    const float b = __ldg(ng->bo + s);
                    for (int k = tid; k < V; k += nt) row[k] = __fadd_rn(b, row[k]);
                } else {
                    const int c0 = __ldg(ng->first + s), c1 = c0 + __ldg(ng->count + s);
                    for (int c = c0 + tid; c < c1; c += nt) row[__ldg(ng->tok + c)] = __ldg(ng->prob + c);
                }
            }
            __syncthreads();
        }
}
// The n-gram state after a non-blank token k in state s: the next state of the first child k found walking down the
// suffix chain from s (a binary search in each state's sorted children, at most depth(s) + 1 states), the root if none.
__device__ int ngram_next(const EbNgram* ng, int s, int k) {
    for (;;) {
        int lo = __ldg(ng->first + s), hi = lo + __ldg(ng->count + s);
        const int end = hi;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(ng->tok + mid) < k) lo = mid + 1;
            else hi = mid;
        }
        if (lo < end && __ldg(ng->tok + lo) == k) return __ldg(ng->next + lo);
        if (s == 0) return 0;
        s = __ldg(ng->suffix + s);
    }
}

// Selection: the candidates of one utterance are (slot q < live, token k) with value
//   lp = ((x[q,k] - max_q) - log sum_k exp(x[q,k] - max_q)) + logp[q],
// or with LM fusion (flags 32) lp = (a + f) + logp[q] where a is the first term above and, for k != blank,
//   f = lm_weight * ((l[q,j] - lmax_q) - log sum_i exp(l[q,i] - lmax_q)) + length_bonus   (j = tok_map[k] >= 0)
//   f = length_bonus   (j < 0),
// and f = 0 for blank (a + 0 is a bitwise, since a is never -0: lm_weight = length_bonus = 0 ranks as without LM).
// ranked by value descending, ties by the lowest flat index q*V + k.  Each candidate's 64-bit composite
// (order_key(lp) << 32 | tie_key(flat)) is unique and orders exactly so; a radix select finds the min(W, live*V)-th largest
// composite 8 bits at a time (a 256-bin shared-memory histogram per pass, stopping at the first pass whose chosen bin
// holds exactly the remaining count: 3-4 passes without exact value ties, at most 8), one more pass collects the
// survivors and a bitonic sort of those <= W composites gives the walk order.  Cost per frame and utterance: about
// 4-5 passes over live*V candidates read from L2 (W = 64, V = 1024: 64 K candidates, 256 per thread per pass) and
// O(W log^2 W) for the sort.  Merging (rule: a candidate whose token sequence equals an earlier survivor's is folded
// into it by log-add) compares survivor i with every earlier one, O(W) per thread.  Because the previous beam was
// already merged, two distinct candidates can only have equal sequences when one is the blank extension of a parent
// q2 and the other the non-blank extension seq(q1) + [k]; length and a 64-bit hash reject the rest, and a hash match
// is confirmed by an exact token-by-token comparison (seq_extends), never accepted on its own.
//
// Streaming (flags 64): the beam lives on across launches.  The live count at t = 0 is the one the previous launch left
// in the last history column (hist_live[b, T'-1], set by BEAM_COMMIT or the host), and the sequence rows have stride K1
// (max_pending + 3) whatever the frames per launch.  A row's length counts only the tokens stored since the stream's
// last commit, while its hash keeps describing the whole sequence: every slot of a stream shares the committed prefix,
// so equal whole sequences are exactly equal stored suffixes, and seq_extends and the merge stay exact.
//
// Several symbols per frame (MULTI, flags 512, K = ldw2 rounds): round j of frame t.  A slot is open when its previous
// round's token (tok_out, read before it is overwritten) is non-blank; every slot is open at round 0.  An open slot's
// candidates are its V tokens as above: blank closes it, a non-blank token keeps it open unless j = K-1.  A closed slot
// has one "stay" candidate of value logp[q] (nothing added) at flat index q*V + blank; it keeps its sequence and state,
// so it is written exactly as a blank extension.  Merging needs equal sequences AND equal closedness (an open and a
// closed hypothesis are different lattice states), and equal sequences can now come from parents with equal sequences
// (a stay and a blank extension), so the exact check is the general seq_equal_ext.  A row with no open slot at j >= 1
// has ended its frame and keeps its beam, as a frozen row does, and as SKIP does when no row is open: history, live
// count and log p unwritten, the sequences copied to seq_out (the round's state moves back from there).
template <bool MULTI>
__device__ __forceinline__ void beam_select(const EbPhase& p, float* sm) {
    const int W = p.aux, V = p.N, T = p.hist_ld, col = p.hist_col, blank = p.aux2;
    const int KR = MULTI ? p.ldw2 : 1, t = MULTI ? col / KR : col, jr = MULTI ? col % KR : 0;
    const bool last = jr == KR - 1;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x;
    const bool merge = p.flags & 16, lm = p.flags & 32, stream = p.flags & 64;
    const long BTW = (long)p.S * T * W;
    int* hpar = p.hist;
    int* htok = p.hist + BTW;
    float* hlp = reinterpret_cast<float*>(p.hist + 2 * BTW);
    int* hlive = p.hist + 3 * BTW;
    const int LS = stream ? p.K1 : T + 3;
    unsigned long long* comp = reinterpret_cast<unsigned long long*>(sm);       // [BEAM_MAX_W] (padded to 2^k)
    unsigned long long* shash = comp + BEAM_MAX_W;
    float* rowm = reinterpret_cast<float*>(shash + BEAM_MAX_W);
    float* rowls = rowm + BEAM_MAX_W;
    float* rowlp = rowls + BEAM_MAX_W;
    float* sval = rowlp + BEAM_MAX_W;
    float* smlp = sval + BEAM_MAX_W;
    int* spar = reinterpret_cast<int*>(smlp + BEAM_MAX_W);
    int* stok = spar + BEAM_MAX_W;
    int* slen = stok + BEAM_MAX_W;
    int* sfirst = slen + BEAM_MAX_W;
    int* skept = sfirst + BEAM_MAX_W;                                           // slot -> survivor index
    float* lmm = reinterpret_cast<float*>(skept + BEAM_MAX_W);                   // LM log-softmax statistics
    float* lmls = lmm + BEAM_MAX_W;
    int* sopen = reinterpret_cast<int*>(lmls + BEAM_MAX_W);                      // slot open (MULTI)
    unsigned* rhist = reinterpret_cast<unsigned*>(sopen + BEAM_MAX_W);          // [256]
    int* misc = reinterpret_cast<int*>(rhist + 256);
    // n-gram fusion (flags 4096): its states alternate as the context states do, its rows are built per frame / round
    const bool ng = p.flags & 4096;
    const EbNgram* ngd = ng ? p.ctx->ng : nullptr;
    const float lm_weight = lm ? __ldg(p.fuse) : 0.f, length_bonus = lm || ng ? __ldg(p.fuse + 1) : 0.f;
    const float ng_w = ng ? ngd->weight : 0.f;
    const float* ng_row = ng ? ngd->row : nullptr;
    const int* nst_in = ng ? ngd->state[MULTI ? 0 : t & 1] : nullptr;
    int* nst_out = ng ? ngd->state[MULTI ? 1 : (t & 1) ^ 1] : nullptr;
    // contextual biasing (flags 2048): the slots' automaton states alternate as the sequence rows do
    const bool cx = p.flags & 2048;
    const int* cnext = cx ? p.ctx->next : nullptr;
    const float* cdelta = cx ? p.ctx->delta : nullptr;
    const int* cst_in = cx ? p.ctx->state[MULTI ? 0 : t & 1] : nullptr;
    int* cst_out = cx ? p.ctx->state[MULTI ? 1 : (t & 1) ^ 1] : nullptr;
    for (int b = blockIdx.x; b < p.S; b += gridDim.x) {
        const long r0 = (long)b * W, h0 = ((long)b * T + col) * W;
        const int nlive = MULTI ? __ldcg(hlive + (long)b * T + T - 1)
                                : t > 0 ? __ldcg(hlive + (long)b * T + t - 1) : stream ? __ldcg(hlive + (long)b * T + T - 1) : 1;
        __syncthreads();                                     // the previous utterance is done with shared memory
        int nopen = nlive;
        if (MULTI) {
            if (tid == 0) misc[5] = 0;
            __syncthreads();
            int open = 0;
            for (int q = tid; q < nlive; q += nt) {
                sopen[q] = jr == 0 || __ldcg(p.tok_out + r0 + q) != blank;
                open += sopen[q];
            }
            if (open) atomicAdd(&misc[5], open);
            __syncthreads();
            nopen = misc[5];
            if (t >= __ldg(p.tok_in + b) || nopen == 0) {   // frozen, or the frame has ended: the beam stays as it is
                for (int s = tid; s < W; s += nt) {
                    p.tok_out[r0 + s] = blank;
                    p.src[r0 + s] = (int)(r0 + s);
                    if (lm) p.tok_out2[r0 + s] = -1;
                    if (cx) cst_out[r0 + s] = __ldcg(cst_in + r0 + s);
                    if (ng) nst_out[r0 + s] = __ldcg(nst_in + r0 + s);
                }
                for (int s = 0; s < nlive; ++s) {
                    const int* ps = p.seq_in + (r0 + s) * LS;
                    int* d = p.seq_out + (r0 + s) * LS;
                    const int n = __ldcg(ps) + 3;
                    for (int i = tid; i < n; i += nt) d[i] = __ldcg(ps + i);
                }
                continue;
            }
        } else if (t >= __ldg(p.tok_in + b)) {               // frozen: the beam stays, the predictor rests
            for (int j = tid; j < W; j += nt) {
                hpar[h0 + j] = j;
                htok[h0 + j] = blank;
                hlp[h0 + j] = __ldcg(p.y + r0 + j);
                p.tok_out[r0 + j] = blank;
                p.src[r0 + j] = (int)(r0 + j);
                if (lm) p.tok_out2[r0 + j] = -1;
                if (cx) cst_out[r0 + j] = __ldcg(cst_in + r0 + j);   // the state BEAM_FINAL reads stays current
                if (ng) nst_out[r0 + j] = __ldcg(nst_in + r0 + j);
            }
            if (tid == 0) hlive[(long)b * T + t] = nlive;
            continue;
        }
        // per-row log-softmax statistics (warp per row)
        for (int q = warp; q < nlive; q += nt >> 5) {
            if (MULTI && !sopen[q]) {                        // a stay needs only the slot's log p
                if (lane == 0) rowlp[q] = __ldcg(p.y + r0 + q);
                continue;
            }
            const float* x = p.x1 + (r0 + q) * p.ldx1;
            float m = -INFINITY;
            for (int k = lane; k < V; k += 32) m = fmaxf(m, __ldcg(x + k));
            m = warp_max(m);
            float s = 0.f;
            for (int k = lane; k < V; k += 32) s += expf(__ldcg(x + k) - m);
            s = warp_sum(s);
            if (lane == 0) {
                rowm[q] = m;
                rowls[q] = logf(s);
                rowlp[q] = __ldcg(p.y + r0 + q);
            }
            if (lm) {
                const float* l = p.x2 + (r0 + q) * p.ldx2;
                float lmx = -INFINITY;
                for (int k = lane; k < p.K2; k += 32) lmx = fmaxf(lmx, __ldcg(l + k));
                lmx = warp_max(lmx);
                float ls = 0.f;
                for (int k = lane; k < p.K2; k += 32) ls += expf(__ldcg(l + k) - lmx);
                ls = warp_sum(ls);
                if (lane == 0) {
                    lmm[q] = lmx;
                    lmls[q] = logf(ls);
                }
            }
        }
        __syncthreads();
        if (ng)                                              // g(state(q), .) of every slot with candidates
            ngram_rows(ngd, r0, nlive, V, [&](int q) { return __ldcg(nst_in + r0 + q); },
                       [&](int q) { return !MULTI || sopen[q]; }, misc + 6);
        // the one expression every pass ranks by; d = the delta row of slot q's context state
        auto composite = [&](int q, int k, const float* x, const float* d) -> unsigned long long {
            float v = (__ldcg(x + k) - rowm[q]) - rowls[q];
            if (lm || cx || ng) {
                float f = 0.f;
                if (k != blank) {
                    if (lm) {
                        const int j = __ldg(p.tok_map + k);
                        f = j >= 0 ? lm_weight * ((__ldcg(p.x2 + (r0 + q) * p.ldx2 + j) - lmm[q]) - lmls[q]) +
                                         length_bonus
                                   : length_bonus;
                    } else if (ng) {
                        f = length_bonus;
                    }
                    if (ng) f = __fadd_rn(f, __fmul_rn(ng_w, __ldcg(ng_row + (r0 + q) * V + k)));
                    if (cx) f = lm || ng ? f + __ldg(d + k) : __ldg(d + k);
                }
                v = v + f;
            }
            v = v + rowlp[q];
            return ((unsigned long long)order_key(v) << 32) | tie_key((unsigned)(q * V + k));
        };
        // a closed slot's (MULTI) one candidate, its stay: value logp[q], flat index q*V + blank
        auto stay = [&](int q) -> unsigned long long {
            return ((unsigned long long)order_key(rowlp[q]) << 32) | tie_key((unsigned)(q * V + blank));
        };
        auto drow = [&](int q) -> const float* { return cx ? cdelta + (long)__ldcg(cst_in + r0 + q) * V : nullptr; };
        const int nsel = (int)min((long)W, (long)nopen * V + (nlive - nopen));
        unsigned need = nsel;
        unsigned long long prefix = 0, mask = 0;
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int i = tid; i < 256; i += nt) rhist[i] = 0;
            __syncthreads();
            for (int q = 0; q < nlive; ++q) {
                const float* x = p.x1 + (r0 + q) * p.ldx1;
                if (MULTI && !sopen[q]) {                    // a closed slot: its stay alone
                    const unsigned long long c = stay(q);
                    if (tid == 0 && (c & mask) == prefix) atomicAdd(&rhist[(c >> shift) & 255], 1u);
                    continue;
                }
                const float* d = drow(q);
                for (int k = tid; k < V; k += nt) {
                    const unsigned long long c = composite(q, k, x, d);
                    if ((c & mask) == prefix) atomicAdd(&rhist[(c >> shift) & 255], 1u);
                }
            }
            __syncthreads();
            if (warp == 0) {                                 // lane l owns bins 255-8l .. 248-8l, scanned from the top
                unsigned cnt[8], s = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    cnt[i] = rhist[255 - 8 * lane - i];
                    s += cnt[i];
                }
                unsigned inc = s;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
                    if (lane >= o) inc += v;
                }
                unsigned above = inc - s;
                if (above < need && need <= inc) {
                    int i = 0;
                    while (above + cnt[i] < need) above += cnt[i++];
                    misc[0] = 255 - 8 * lane - i;
                    misc[1] = (int)above;
                    misc[2] = (int)cnt[i];
                }
            }
            __syncthreads();
            need -= (unsigned)misc[1];
            prefix |= (unsigned long long)misc[0] << shift;
            mask |= 0xffull << shift;
            if ((unsigned)misc[2] == need) break;            // every candidate under this prefix survives
        }
        if (tid == 0) misc[3] = 0;
        __syncthreads();
        for (int q = 0; q < nlive; ++q) {
            const float* x = p.x1 + (r0 + q) * p.ldx1;
            if (MULTI && !sopen[q]) {
                const unsigned long long c = stay(q);
                if (tid == 0 && (c & mask) >= prefix) {
                    const int i = atomicAdd(&misc[3], 1);
                    if (i < nsel) comp[i] = c;
                }
                continue;
            }
            const float* d = drow(q);
            for (int k = tid; k < V; k += nt) {
                const unsigned long long c = composite(q, k, x, d);
                if ((c & mask) >= prefix) {
                    const int i = atomicAdd(&misc[3], 1);
                    if (i < nsel) comp[i] = c;               // exactly nsel pass; the guard keeps smem safe regardless
                }
            }
        }
        int P = 1;
        while (P < nsel) P <<= 1;
        for (int i = nsel + tid; i < P; i += nt) comp[i] = 0;
        __syncthreads();
        for (int kk = 2; kk <= P; kk <<= 1)                  // bitonic sort, descending
            for (int jj = kk >> 1; jj > 0; jj >>= 1) {
                for (int i = tid; i < P; i += nt) {
                    const int l = i ^ jj;
                    if (l > i) {
                        const unsigned long long a = comp[i], c = comp[l];
                        if ((i & kk) == 0 ? a < c : a > c) {
                            comp[i] = c;
                            comp[l] = a;
                        }
                    }
                }
                __syncthreads();
            }
        // survivors in walk order: parent, token, value, and the length / hash of the extended sequence
        for (int i = tid; i < nsel; i += nt) {
            const unsigned long long c = comp[i];
            const unsigned f = tie_key((unsigned)c);
            const int q = (int)(f / V), k = (int)(f % V);
            const int* ps = p.seq_in + (r0 + q) * LS;
            int len = __ldcg(ps);
            unsigned long long h = (unsigned)__ldcg(ps + 1) | ((unsigned long long)(unsigned)__ldcg(ps + 2) << 32);
            if (k != blank) {
                ++len;
                h = h * SEQ_HASH_MUL + (unsigned)(k + 1);
            }
            spar[i] = q;
            stok[i] = k;
            sval[i] = key_value((unsigned)(c >> 32));
            slen[i] = len;
            shash[i] = h;
        }
        if (tid == 0) misc[4] = 0;
        __syncthreads();
        for (int i = tid; i < nsel; i += nt) {
            int first = i;
            if (MULTI && merge) {                            // same sequence and same closedness
                const bool ic = stok[i] == blank || last;
                for (int j = 0; j < i; ++j) {
                    if ((stok[j] == blank || last) != ic || slen[j] != slen[i] || shash[j] != shash[i]) continue;
                    if (seq_equal_ext(p.seq_in + (r0 + spar[i]) * LS, stok[i] != blank ? stok[i] : -1,
                                      p.seq_in + (r0 + spar[j]) * LS, stok[j] != blank ? stok[j] : -1)) {
                        first = j;
                        break;
                    }
                }
            } else if (merge) {
                const bool ib = stok[i] == blank;
                for (int j = 0; j < i; ++j) {
                    if ((stok[j] == blank) == ib || slen[j] != slen[i] || shash[j] != shash[i]) continue;
                    const int q2 = ib ? spar[i] : spar[j], q1 = ib ? spar[j] : spar[i], k1 = ib ? stok[j] : stok[i];
                    if (seq_extends(p.seq_in + (r0 + q2) * LS, p.seq_in + (r0 + q1) * LS, k1)) {
                        first = j;
                        break;
                    }
                }
            }
            sfirst[i] = first;
        }
        __syncthreads();
        for (int i = tid; i < nsel; i += nt) {
            if (sfirst[i] != i) continue;
            int slot = 0;
            for (int j = 0; j < i; ++j) slot += sfirst[j] == j;
            float lp = sval[i];
            for (int j = i + 1; j < nsel; ++j)               // fold in walk order, as the host loop did
                if (sfirst[j] == i) lp = logaddexp_(lp, sval[j]);
            smlp[i] = lp;
            skept[slot] = i;
            atomicAdd(&misc[4], 1);
        }
        __syncthreads();
        const int nkept = misc[4];
        for (int s = tid; s < W; s += nt) {
            const long h = h0 + s, r = r0 + s;
            if (s < nkept) {
                const int i = skept[s], k = stok[i];
                p.y[r] = smlp[i];
                p.tok_out[r] = k;
                if (lm) p.tok_out2[r] = k != blank ? __ldg(p.tok_map + k) : -1;
                p.src[r] = (int)(r0 + spar[i]);
                hpar[h] = spar[i];
                htok[h] = k;
                hlp[h] = smlp[i];
                int* d = p.seq_out + r * LS;
                d[0] = slen[i];
                d[1] = (int)(unsigned)shash[i];
                d[2] = (int)(unsigned)(shash[i] >> 32);
                if (cx) {
                    const int cs = __ldcg(cst_in + r0 + spar[i]);
                    cst_out[r] = k != blank ? __ldg(cnext + (long)cs * V + k) : cs;
                }
                if (ng) {
                    const int ns = __ldcg(nst_in + r0 + spar[i]);
                    nst_out[r] = k != blank ? ngram_next(ngd, ns, k) : ns;
                }
            } else {
                p.y[r] = -INFINITY;
                p.tok_out[r] = blank;
                if (lm) p.tok_out2[r] = -1;
                if (cx) cst_out[r] = 0;
                if (ng) nst_out[r] = 0;
                p.src[r] = (int)r;
                hpar[h] = s;
                htok[h] = blank;
                hlp[h] = -INFINITY;
            }
        }
        if (tid == 0) {
            hlive[(long)b * T + col] = nkept;
            if (MULTI) hlive[(long)b * T + T - 1] = nkept;  // the live count the next round reads
        }
        for (int s = 0; s < nkept; ++s) {                    // token sequences of the new beam
            const int i = skept[s], len = slen[i];
            const int* ps = p.seq_in + (r0 + spar[i]) * LS + 3;
            int* d = p.seq_out + (r0 + s) * LS + 3;
            for (int j = tid; j < len; j += nt) d[j] = (stok[i] != blank && j == len - 1) ? stok[i] : __ldcg(ps + j);
        }
    }
}

// one call site in the kernel, as before the multi-symbol rounds: a second one costs the matrix phases spills
__device__ __noinline__ void phase_beam_select(const EbPhase& p, float* sm) {
    if (p.flags & 512) beam_select<true>(p, sm);
    else beam_select<false>(p, sm);
}

__device__ __noinline__ void phase_gather(const EbPhase& p) {
    if (p.flags & 1024) {                                    // a chunk's front end: no gather
        fe_program(p);
        return;
    }
    const long gtid = (long)blockIdx.x * blockDim.x + threadIdx.x, gn = (long)gridDim.x * blockDim.x;
    const int S = p.S, N = p.N;
    for (long e = gtid; e < (long)p.aux * S * N; e += gn) {
        const long lr = e / N;
        const int c = (int)(e - lr * N), r = (int)(lr % S);
        p.y[e] = __ldcg(p.x1 + ((lr - r) + __ldcg(p.src + r)) * N + c);
    }
    if (p.x2)
        for (long e = gtid; e < (long)S * p.K2; e += gn) {
            const int r = (int)(e / p.K2), c = (int)(e % p.K2);
            p.y2[e] = __ldcg(p.x2 + (long)__ldcg(p.src + r) * p.K2 + c);
        }
}

// Chunk end of the streaming beam, one CTA per stream.  The live slots' stored suffixes (seq_in) share a longest common
// prefix of c tokens; no later frame can change it, since every future hypothesis extends a current one, so it is
// committed: written to tok_out row b and dropped from every live suffix (seq_out).  If a suffix then still holds more
// than aux2 = max_pending - n_out tokens (or flags 128: always), the beam collapses: the best live slot (highest y,
// lowest slot on ties, as BEAM_FINAL) commits its whole suffix and becomes slot 0, the only live one, keeping its y.
// src receives the gather sources that move each kept slot's state (predictor / LM, or CTC's pb | pnb | f) into place
// (identity without a collapse), tok_out2[b] the committed count and tok_out2[S + b] whether the beam collapsed.  The
// row head (K2) is copied unchanged: the hashes describe the whole sequence, committed part included.  With y2, the last
// token committed is kept per stream: a CTC slot whose stored suffix is empty takes it as its last token.
// Contextual biasing (flags 2048): the slots' automaton states are read from ctx->state[1], a collapse ranks by
// y - pending[state] (BEAM_FINAL's value and tie rule; the kept slot keeps its y and its state), and each slot's state
// moves to ctx->state[0] by the same gather sources as the rest of its state.
__device__ __noinline__ void phase_beam_commit(const EbPhase& p, float* sm) {
    const int W = p.aux, T = p.hist_ld, LS = p.K1, HEAD = p.K2 > 0 ? p.K2 : 3;
    int* last = reinterpret_cast<int*>(p.y2);
    const int tid = threadIdx.x, nt = blockDim.x;
    int* hlive = p.hist + 3 * (long)p.S * T * W;
    int* misc = reinterpret_cast<int*>(sm);
    const bool cx = p.flags & 2048;
    for (int b = blockIdx.x; b < p.S; b += gridDim.x) {
        const long r0 = (long)b * W;
        const int nlive = __ldcg(hlive + (long)b * T + T - 1);
        const int* seq0 = p.seq_in + r0 * LS;
        __syncthreads();                                     // the previous stream is done with shared memory
        if (tid == 0) {
            misc[0] = 0x7fffffff;                            // shortest live suffix
            misc[1] = 0;                                     // longest live suffix
            misc[4] = 0x7fffffff;                            // first position where two live suffixes differ
        }
        __syncthreads();
        for (int s = tid; s < nlive; s += nt) {
            const int len = __ldcg(p.seq_in + (r0 + s) * LS);
            atomicMin(&misc[0], len);
            atomicMax(&misc[1], len);
        }
        __syncthreads();
        const int lmin = misc[0];
        for (long e = tid; e < (long)(nlive - 1) * lmin; e += nt) {
            const int s = 1 + (int)(e / lmin), j = (int)(e % lmin);
            if (__ldcg(p.seq_in + (r0 + s) * LS + HEAD + j) != __ldcg(seq0 + HEAD + j)) atomicMin(&misc[4], j);
        }
        __syncthreads();
        const int c = min(lmin, misc[4]);
        const bool collapse = (p.flags & 128) || misc[1] - c > p.aux2;
        if (collapse && tid < 32) {                          // logp.argmax() over the live slots
            float best = -INFINITY;
            int bi = -1;
            for (int j = tid; j < nlive; j += 32) {
                float v = __ldcg(p.y + r0 + j);
                if (cx) v = v - __ldg(p.ctx->pending + __ldcg(p.ctx->state[1] + r0 + j));
                if (bi < 0 || v > best) { best = v; bi = j; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (oi >= 0 && (bi < 0 || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
            }
            if (tid == 0) {
                misc[2] = bi;
                misc[3] = __float_as_int(cx && bi >= 0 ? __ldcg(p.y + r0 + bi) : best);   // the kept slot's y
            }
        }
        __syncthreads();
        const int best = collapse ? misc[2] : 0, nkeep = collapse ? 1 : nlive;
        const int* bs = p.seq_in + (r0 + best) * LS;
        const int ncommit = collapse ? __ldcg(bs) : c;
        int* out = p.tok_out + (long)b * p.N;
        for (int j = tid; j < ncommit; j += nt) out[j] = __ldcg(bs + HEAD + j);
        for (long e = tid; e < (long)nkeep * LS; e += nt) {  // kept slot s: {length - ncommit, hash, shifted tokens}
            const int s = (int)(e / LS), j = (int)(e % LS);
            const int* ps = p.seq_in + (r0 + (collapse ? best : s)) * LS;
            const int len = __ldcg(ps) - ncommit;
            if (j >= len + HEAD) continue;
            p.seq_out[(r0 + s) * LS + j] = j == 0 ? len : j < HEAD ? __ldcg(ps + j) : __ldcg(ps + j + ncommit);
        }
        for (int s = tid; s < W; s += nt) {
            p.src[r0 + s] = (int)(r0 + (s == 0 ? best : s));
            if (collapse) p.y[r0 + s] = s == 0 ? __int_as_float(misc[3]) : -INFINITY;
            if (cx) p.ctx->state[0][r0 + s] = __ldcg(p.ctx->state[1] + r0 + (s == 0 ? best : s));
        }
        if (tid == 0) {
            p.tok_out2[b] = ncommit;
            p.tok_out2[p.S + b] = collapse;
            hlive[(long)b * T + T - 1] = nkeep;
            if (last && ncommit > 0) last[b] = __ldcg(bs + HEAD + ncommit - 1);
        }
    }
}

// The N best live slots of each utterance (N = K1, 0 read as 1), ranked by value descending, lowest slot on ties
// (logp.argmax() at rank 0, -0 with +0): the 64-bit composites order_key(value) << 32 | tie_key(slot) of the live
// slots, bitonic-sorted in shared memory as BEAM_SELECT sorts its survivors, by the CTA's first warp (up to 32 keys
// per lane and step at W = 1024; with all 256 threads eb_decode_run_ctc spills 4 bytes more).  Lane n walks rank n's
// back-pointers (then n + 32, ...) over the hist_ld columns and writes its non-blank tokens right-aligned in row
// b*N + n of tok_out (-1 before them), with seq_out set each token's frame (column / ldw2, ldw2 = K rounds per frame, 0 read as 1) in the same positions, and
// y2[b*N + n] = -value; tok_out2, when set, gets the count min(N, live) per utterance.  Ranks at or past the count hold
// ids and frames -1 and y2 = +inf.  The walk is one dependent load per column, as for N = 1.
__device__ __noinline__ void phase_beam_final(const EbPhase& p) {
    extern __shared__ __align__(16) float dsm[];
    unsigned long long* comp = reinterpret_cast<unsigned long long*>(dsm);     // [BEAM_MAX_W]
    const int W = p.aux, T = p.hist_ld, blank = p.aux2, lane = threadIdx.x & 31;
    const long BTW = (long)p.S * T * W;
    const int* hpar = p.hist;
    const int* htok = p.hist + BTW;
    const int* hlive = p.hist + 3 * BTW;
    if (threadIdx.x >= 32) return;                           // one warp: with the whole CTA the CTC entry spills more
    // the ranking value: y, with n-gram fusion (flags 4096) y + w*e(state), with contextual biasing (flags 2048) then
    // - pending[state], the states from parity hist_col
    const bool cx = p.flags & 2048;
    const float* cpend = cx ? p.ctx->pending : nullptr;
    const int* cst = cx ? p.ctx->state[p.hist_col & 1] : nullptr;
    const float* nend = p.flags & 4096 ? p.ctx->ng->end : nullptr;
    const int* nst = nend ? p.ctx->ng->state[p.hist_col & 1] : nullptr;
    const float ng_w = nend ? p.ctx->ng->weight : 0.f;
    auto value = [&](long r) -> float {
        float v = __ldcg(p.y + r);
        if (nend) v = __fadd_rn(v, __fmul_rn(ng_w, __ldg(nend + __ldcg(nst + r))));
        return cx ? v - __ldg(cpend + __ldcg(cst + r)) : v;
    };
    for (int b = blockIdx.x; b < p.S; b += gridDim.x) {
        const int nlive = T == 0 ? 1 : __ldcg(hlive + (long)b * T + T - 1);
        int P = 1;
        while (P < nlive) P <<= 1;
        __syncwarp();                                        // the previous utterance is done with shared memory
        for (int i = lane; i < P; i += 32)
            comp[i] = i < nlive ? ((unsigned long long)order_key(value((long)b * W + i)) << 32) | tie_key(i) : 0;
        __syncwarp();
        for (int kk = 2; kk <= P; kk <<= 1)                  // bitonic sort, descending
            for (int jj = kk >> 1; jj > 0; jj >>= 1) {
                for (int i = lane; i < P; i += 32) {
                    const int l = i ^ jj;
                    if (l > i) {
                        const unsigned long long a = comp[i], c = comp[l];
                        if ((i & kk) == 0 ? a < c : a > c) {
                            comp[i] = c;
                            comp[l] = a;
                        }
                    }
                }
                __syncwarp();
            }
        const int NB = p.K1 > 0 ? p.K1 : 1, KR = p.ldw2 > 0 ? p.ldw2 : 1, cnt = min(NB, nlive);
        for (int n = lane; n < NB; n += 32) {
            const long row = (long)b * NB + n;
            int* ids = p.tok_out + row * p.ldy;
            int* fr = p.seq_out ? p.seq_out + row * p.ldy : nullptr;
            int pos = T;
            if (n < cnt) {
                const int top = (int)tie_key((unsigned)comp[n]);
                int slot = top;
                for (int tt = T - 1; tt >= 0; --tt) {
                    const long h = ((long)b * T + tt) * W + slot;
                    const int k = __ldcg(htok + h);
                    if (k != blank) {
                        ids[--pos] = k;
                        if (fr) fr[pos] = tt / KR;
                    }
                    slot = __ldcg(hpar + h);
                }
                p.y2[row] = -value((long)b * W + top);         // the value itself: -0 stays -0, as argmax gave it
            } else {
                p.y2[row] = INFINITY;
            }
            for (int j = 0; j < pos; ++j) {
                ids[j] = -1;
                if (fr) fr[j] = -1;
            }
        }
        if (p.tok_out2 && lane == 0) p.tok_out2[b] = cnt;
    }
}

// ---- CTC prefix beam search (CTCBeamEngine, Hannun et al. 2014): B utterances x W slots, row r = b*W + slot, T' =
// hist_ld frames.  Field use of CTC_BEAM:
//   S = B, N = V, aux = W, aux2 = blank, hist_col = first frame t0, ldw1 = frames this phase runs (>= 1), K1 = LS =
//   T' + 5; x1 log-probs [B, T', V] contiguous; tok_in frames [B]; c per-slot state [2 parities][pb | pnb | f][B*W]
//   (frame t reads parity t&1 and writes the other); seq_out token rows [2 parities][B*W][LS] = {len, hash lo, hash hi,
//   parent hash lo, parent hash hi, tokens} (the parent hash is the hash of the prefix without its last token); y the
//   ranking value (pb (+) pnb) + f of each slot [B*W] (dead slots -inf), what BEAM_FINAL picks by; hist as BEAM_SELECT's,
//   a stay recorded with token blank; src the parent row [B*W].  Flag 32 (LM fusion): x2 / ldx2 / K2 LM logits, fuse,
//   tok_map and tok_out2 (LM token of each new slot, -1 for a stay) as BEAM_SELECT's.  Flag 64 (streaming): K1 =
//   max_pending + 5, the live count at t = 0 from hist_live[b, T'-1], y2 the last committed token [B] (int32, read).
// A frame t < frames[b] of one utterance, for its live slots q (prefix l, last token e or none), with (+) = logaddexp_:
//   stay       pb' = (pb (+) pnb) + y[blank], pnb' = pnb + y[e] (-inf for the empty prefix), f' = f;
//   extension  by a non-blank c: pb' = -inf, pnb' = (c == e ? pb : pb (+) pnb) + y[c], f' = f + fusion term;
//   merge      when l + c is the prefix of another live slot q2 (q2's prefix minus its last token is l: length, hash,
//              then an exact token comparison, never the hash alone), that extension is no candidate of its own: its
//              pnb' is log-added into q2's stay pnb' after q2's own repeat term;
//   ranking    by (pb' (+) pnb') + f' descending, ties to the lowest flat index q*V + k (a stay at k = blank), the same
//              64-bit composites, radix select and bitonic sort as BEAM_SELECT; min(W, candidates) survive.
// The previous beam holds distinct prefixes, so the merge is the only way two candidates can share one.  An extension's
// value is pnb' + f', which is (-inf (+) pnb') + f' bit for bit for every non-NaN pnb'.  Frames t >= frames[b] write an
// identity history entry and touch no state: a frozen utterance is never read again.  NaN log-probs are outside the
// contract; a NaN value gets a composite like any other (order_key keeps every key distinct), so the select still ends
// after at most 8 passes and reads nothing out of bounds.  Without an LM nothing runs between frames, and one phase
// walks all frames of its utterances with no grid barrier; with an LM the program runs one frame per phase.
// Streaming (flags 64, CTCStreamBeamEngine): the beam lives on across launches, as BEAM_SELECT's does.  The live count at
// t = 0 is the one the previous launch left in the last history column (hist_live[b, T'-1], where BEAM_COMMIT reads and
// rewrites it), K1 = max_pending + 5 whatever the frames per launch, and a row stores only the tokens since the stream's
// last commit while its hash and parent hash keep describing the whole prefix, so the merge test stays exact (every
// live slot of a stream shares the committed part, and no slot shorter than it is live).  y2 (int32 [B]) holds each
// stream's last committed token, -1 before any: a slot whose stored suffix is empty takes it as its last token e, so the
// stay's repeat term and the extension rule see the real last token across a commit.  Without the flag e is -1 there,
// which is the same thing at the start of an utterance.
constexpr int CTC_SEQ_HEAD = 5;
// CTC_BEAM's shared memory (2 x u64 + 11 x 32-bit arrays of BEAM_MAX_W, histogram, scalars, the context and n-gram
// states) in the dynamic shared memory
static_assert(BEAM_MAX_W * (2 * 8 + 13 * 4) + 256 * 4 + 8 * 4 <= (RED_FLOATS + TR * OUT_LD) * 4, "ctc beam smem");

template <bool NG>
__device__ __noinline__ void ctc_beam(const EbPhase& p, float* sm) {
    const int W = p.aux, V = p.N, T = p.hist_ld, blank = p.aux2, LS = p.K1;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x;
    const bool lm = p.flags & 32, stream = p.flags & 64;
    const long R = (long)p.S * W, BTW = R * T;
    int* hpar = p.hist;
    int* htok = p.hist + BTW;
    float* hlp = reinterpret_cast<float*>(p.hist + 2 * BTW);
    int* hlive = p.hist + 3 * BTW;
    unsigned long long* comp = reinterpret_cast<unsigned long long*>(sm);       // [BEAM_MAX_W] (padded to 2^k)
    unsigned long long* shash = comp + BEAM_MAX_W;                             // prefix hash
    float* sA = reinterpret_cast<float*>(shash + BEAM_MAX_W);                   // pb (+) pnb
    float* sB = sA + BEAM_MAX_W;                                                // pb
    float* sf = sB + BEAM_MAX_W;                                                // f
    float* sstay = sf + BEAM_MAX_W;                                             // the stay's value
    float* lmm = sstay + BEAM_MAX_W;                                            // LM log-softmax statistics
    float* lmls = lmm + BEAM_MAX_W;
    int* se = reinterpret_cast<int*>(lmls + BEAM_MAX_W);                        // last token, -1 for the empty prefix
    int* slen = se + BEAM_MAX_W;
    int* mpar = slen + BEAM_MAX_W;                                              // slot whose extension merges in, or -1
    int* chead = mpar + BEAM_MAX_W;                                             // slots merging from this one: a list
    int* cnext = chead + BEAM_MAX_W;
    unsigned* rhist = reinterpret_cast<unsigned*>(cnext + BEAM_MAX_W);          // [256]
    int* misc = reinterpret_cast<int*>(rhist + 256);
    int* sst = misc + 8;                                                        // context state of each slot
    int* sng = sst + BEAM_MAX_W;                                                // n-gram state of each slot
    const bool ng = NG;                                                         // n-gram fusion (flags 4096)
    const EbNgram* ngd = ng ? p.ctx->ng : nullptr;
    const float ng_w = ng ? ngd->weight : 0.f;
    const float* ng_row = ng ? ngd->row : nullptr;
    int* const* ng_state = ng ? ngd->state : nullptr;                           // parity t & 1, as c and seq_out
    const float lm_weight = lm ? __ldg(p.fuse) : 0.f, length_bonus = lm || ng ? __ldg(p.fuse + 1) : 0.f;
    const bool cx = p.flags & 2048;                                             // contextual biasing
    const int* ctx_next = cx ? p.ctx->next : nullptr;
    const float* ctx_delta = cx ? p.ctx->delta : nullptr;
    int* const* ctx_state = cx ? p.ctx->state : nullptr;                        // parity t & 1, as c and seq_out
    for (int b = blockIdx.x; b < p.S; b += gridDim.x) {
        const long r0 = (long)b * W;
        const int frames = __ldg(p.tok_in + b);
        const int e0 = stream ? __ldcg(reinterpret_cast<const int*>(p.y2) + b) : -1;   // last token of an empty suffix
        for (int t = p.hist_col; t < p.hist_col + p.ldw1; ++t) {
            __syncthreads();                                 // the previous frame's shared and global writes are done
            const long h0 = ((long)b * T + t) * W;
            const int nlive = t > 0 ? __ldcg(hlive + (long)b * T + t - 1) : stream ? __ldcg(hlive + (long)b * T + T - 1) : 1;
            if (t >= frames) {                               // frozen: the beam stays, the LM rests
                for (int j = tid; j < W; j += nt) {
                    hpar[h0 + j] = j;
                    htok[h0 + j] = blank;
                    hlp[h0 + j] = __ldcg(p.y + r0 + j);
                    p.src[r0 + j] = (int)(r0 + j);
                    if (lm) p.tok_out2[r0 + j] = -1;
                    if (cx) ctx_state[(t + 1) & 1][r0 + j] = __ldcg(ctx_state[t & 1] + r0 + j);
                    if (ng) ng_state[(t + 1) & 1][r0 + j] = __ldcg(ng_state[t & 1] + r0 + j);
                }
                if (tid == 0) hlive[(long)b * T + t] = nlive;
                continue;
            }
            const float* st_in = p.c + (t & 1) * 3 * R;
            float* st_out = p.c + ((t + 1) & 1) * 3 * R;
            const int* seq_in = p.seq_out + (t & 1) * R * LS;
            int* seq_out = p.seq_out + ((t + 1) & 1) * R * LS;
            const float* y = p.x1 + ((long)b * T + t) * V;
            if (tid < 8) misc[tid] = 0;
            for (int q = tid; q < nlive; q += nt) {
                const float pb = __ldcg(st_in + r0 + q), pnb = __ldcg(st_in + R + r0 + q);
                const int* ps = seq_in + (r0 + q) * LS;
                const int len = __ldcg(ps);
                sA[q] = logaddexp_(pb, pnb);
                sB[q] = pb;
                sf[q] = __ldcg(st_in + 2 * R + r0 + q);
                slen[q] = len;
                shash[q] = (unsigned)__ldcg(ps + 1) | ((unsigned long long)(unsigned)__ldcg(ps + 2) << 32);
                se[q] = len > 0 ? __ldcg(ps + CTC_SEQ_HEAD + len - 1) : e0;
                chead[q] = -1;
                if (cx) sst[q] = __ldcg(ctx_state[t & 1] + r0 + q);
                if (ng) sng[q] = __ldcg(ng_state[t & 1] + r0 + q);
            }
            __syncthreads();
            if (ng)                                          // g(state(q), .) of every live slot
                ngram_rows(ngd, r0, nlive, V, [&](int q) { return sng[q]; }, [](int) { return true; }, misc + 7);
            // merges: the slot whose prefix is slot q2's minus its last token
            for (int q2 = tid; q2 < nlive; q2 += nt) {
                int par = -1;
                const int len = slen[q2];
                if (len > 0) {
                    const int* s2 = seq_in + (r0 + q2) * LS;
                    const unsigned long long ph =
                        (unsigned)__ldcg(s2 + 3) | ((unsigned long long)(unsigned)__ldcg(s2 + 4) << 32);
                    for (int q = 0; q < nlive && par < 0; ++q) {
                        if (slen[q] != len - 1 || shash[q] != ph) continue;
                        const int* s1 = seq_in + (r0 + q) * LS + CTC_SEQ_HEAD;
                        bool eq = true;
                        for (int i = 0; i < len - 1 && eq; ++i) eq = __ldcg(s1 + i) == __ldcg(s2 + CTC_SEQ_HEAD + i);
                        if (eq) par = q;
                    }
                }
                mpar[q2] = par;
                if (par >= 0) {
                    cnext[q2] = atomicExch(&chead[par], q2);
                    atomicAdd(&misc[6], 1);
                }
            }
            __syncthreads();
            // the stay of slot q, with the extension that merges into it
            auto stay_of = [&](int q, float& pb2, float& pnb2) {
                const int e = se[q], par = mpar[q];
                pb2 = sA[q] + __ldg(y + blank);
                pnb2 = e >= 0 ? __ldcg(st_in + R + r0 + q) + __ldg(y + e) : -INFINITY;
                if (par >= 0) pnb2 = logaddexp_(pnb2, (e == se[par] ? sB[par] : sA[par]) + __ldg(y + e));
            };
            for (int q = tid; q < nlive; q += nt) {
                float pb2, pnb2;
                stay_of(q, pb2, pnb2);
                sstay[q] = logaddexp_(pb2, pnb2) + sf[q];
            }
            if (lm)                                          // per-row LM log-softmax statistics (warp per row)
                for (int q = warp; q < nlive; q += nt >> 5) {
                    const float* l = p.x2 + (r0 + q) * p.ldx2;
                    float lmx = -INFINITY;
                    for (int k = lane; k < p.K2; k += 32) lmx = fmaxf(lmx, __ldcg(l + k));
                    lmx = warp_max(lmx);
                    float ls = 0.f;
                    for (int k = lane; k < p.K2; k += 32) ls += expf(__ldcg(l + k) - lmx);
                    ls = warp_sum(ls);
                    if (lane == 0) {
                        lmm[q] = lmx;
                        lmls[q] = logf(ls);
                    }
                }
            __syncthreads();
            // extension (q, k), k != blank: pnb' and f'
            auto ext_of = [&](int q, int k, float& pnb2, float& f2) {
                pnb2 = (k == se[q] ? sB[q] : sA[q]) + __ldg(y + k);
                f2 = sf[q];
                if (lm) {
                    const int j = __ldg(p.tok_map + k);
                    f2 = f2 + (j >= 0 ? lm_weight * ((__ldcg(p.x2 + (r0 + q) * p.ldx2 + j) - lmm[q]) - lmls[q]) +
                                            length_bonus
                                      : length_bonus);
                } else if (ng) {
                    f2 = f2 + length_bonus;
                }
                if (ng) f2 = __fadd_rn(f2, __fmul_rn(ng_w, __ldcg(ng_row + (r0 + q) * V + k)));
                if (cx) f2 = f2 + __ldg(ctx_delta + (long)sst[q] * V + k);
            };
            // candidate flat index e = q*V + k; false when it merged into a live slot's stay
            auto cand = [&](long e, unsigned long long& c) -> bool {
                const int q = (int)(e / V), k = (int)(e - (long)q * V);
                float v;
                if (k == blank) {
                    v = sstay[q];
                } else {
                    for (int q2 = chead[q]; q2 >= 0; q2 = cnext[q2])
                        if (se[q2] == k) return false;
                    float pnb2, f2;
                    ext_of(q, k, pnb2, f2);
                    v = pnb2 + f2;
                }
                c = ((unsigned long long)order_key(v) << 32) | tie_key((unsigned)e);
                return true;
            };
            const long ncand = (long)nlive * V;
            const int nsel = (int)min((long)W, ncand - misc[6]);
            unsigned need = nsel;
            unsigned long long prefix = 0, mask = 0;
            for (int shift = 56; shift >= 0; shift -= 8) {
                for (int i = tid; i < 256; i += nt) rhist[i] = 0;
                __syncthreads();
                for (long e = tid; e < ncand; e += nt) {
                    unsigned long long c;
                    if (cand(e, c) && (c & mask) == prefix) atomicAdd(&rhist[(c >> shift) & 255], 1u);
                }
                __syncthreads();
                if (warp == 0) {                             // lane l owns bins 255-8l .. 248-8l, scanned from the top
                    unsigned cnt[8], s = 0;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        cnt[i] = rhist[255 - 8 * lane - i];
                        s += cnt[i];
                    }
                    unsigned inc = s;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
                        if (lane >= o) inc += v;
                    }
                    unsigned above = inc - s;
                    if (above < need && need <= inc) {
                        int i = 0;
                        while (above + cnt[i] < need) above += cnt[i++];
                        misc[0] = 255 - 8 * lane - i;
                        misc[1] = (int)above;
                        misc[2] = (int)cnt[i];
                    }
                }
                __syncthreads();
                need -= (unsigned)misc[1];
                prefix |= (unsigned long long)misc[0] << shift;
                mask |= 0xffull << shift;
                if ((unsigned)misc[2] == need) break;        // every candidate under this prefix survives
            }
            for (long e = tid; e < ncand; e += nt) {
                unsigned long long c;
                if (cand(e, c) && (c & mask) >= prefix) {
                    const int i = atomicAdd(&misc[3], 1);
                    if (i < nsel) comp[i] = c;               // exactly nsel pass; the guard keeps smem safe regardless
                }
            }
            int P = 1;
            while (P < nsel) P <<= 1;
            for (int i = nsel + tid; i < P; i += nt) comp[i] = 0;
            __syncthreads();
            for (int kk = 2; kk <= P; kk <<= 1)              // bitonic sort, descending
                for (int jj = kk >> 1; jj > 0; jj >>= 1) {
                    for (int i = tid; i < P; i += nt) {
                        const int l = i ^ jj;
                        if (l > i) {
                            const unsigned long long a = comp[i], c = comp[l];
                            if ((i & kk) == 0 ? a < c : a > c) {
                                comp[i] = c;
                                comp[l] = a;
                            }
                        }
                    }
                    __syncthreads();
                }
            // the new beam in walk order
            for (int s = tid; s < W; s += nt) {
                const long r = r0 + s, h = h0 + s;
                if (s < nsel) {
                    const unsigned f = tie_key((unsigned)comp[s]);
                    const int q = (int)(f / V), k = (int)(f % V);
                    float pb2, pnb2, f2, v;
                    if (k == blank) {
                        stay_of(q, pb2, pnb2);
                        f2 = sf[q];
                        v = sstay[q];
                    } else {
                        pb2 = -INFINITY;
                        ext_of(q, k, pnb2, f2);
                        v = pnb2 + f2;
                    }
                    st_out[r] = pb2;
                    st_out[R + r] = pnb2;
                    st_out[2 * R + r] = f2;
                    if (cx) ctx_state[(t + 1) & 1][r] = k == blank ? sst[q] : __ldg(ctx_next + (long)sst[q] * V + k);
                    if (ng) ng_state[(t + 1) & 1][r] = k == blank ? sng[q] : ngram_next(ngd, sng[q], k);
                    p.y[r] = v;
                    p.src[r] = (int)(r0 + q);
                    if (lm) p.tok_out2[r] = k != blank ? __ldg(p.tok_map + k) : -1;
                    hpar[h] = q;
                    htok[h] = k;
                    hlp[h] = v;
                } else {
                    st_out[r] = -INFINITY;
                    st_out[R + r] = -INFINITY;
                    st_out[2 * R + r] = 0.f;
                    if (cx) ctx_state[(t + 1) & 1][r] = 0;
                    if (ng) ng_state[(t + 1) & 1][r] = 0;
                    p.y[r] = -INFINITY;
                    p.src[r] = (int)r;
                    if (lm) p.tok_out2[r] = -1;
                    hpar[h] = s;
                    htok[h] = blank;
                    hlp[h] = -INFINITY;
                }
            }
            if (tid == 0) hlive[(long)b * T + t] = nsel;
            for (int s = 0; s < nsel; ++s) {                 // token rows of the new beam
                const unsigned f = tie_key((unsigned)comp[s]);
                const int q = (int)(f / V), k = (int)(f % V), len = slen[q];
                const bool ext = k != blank;
                const int* ps = seq_in + (r0 + q) * LS;
                int* d = seq_out + (r0 + s) * LS;
                const unsigned long long hn = shash[q] * SEQ_HASH_MUL + (unsigned)(k + 1);
                for (int j = tid; j < CTC_SEQ_HEAD + len + ext; j += nt) {
                    int v;
                    if (j >= CTC_SEQ_HEAD) v = j - CTC_SEQ_HEAD < len ? __ldcg(ps + j) : k;
                    else if (!ext) v = __ldcg(ps + j);
                    else if (j == 0) v = len + 1;
                    else if (j < 3) v = (int)(unsigned)((j == 1 ? hn : hn >> 32));
                    else v = (int)(unsigned)((j == 3 ? shash[q] : shash[q] >> 32));
                    d[j] = v;
                }
            }
        }
    }
}

// One call site in the kernel and two __noinline__ instantiations behind it: a program without n-gram fusion runs a
// body compiled without the term.  With the term's flag tests in one body the offline CTC beam without an n-gram model
// measured 12 % slower than before (W = 4 / 8 / 16, DESIGN.md 4f).
__device__ __noinline__ void phase_ctc_beam(const EbPhase& p, float* sm) {
    if (p.flags & 4096) ctc_beam<true>(p, sm);
    else ctc_beam<false>(p, sm);
}

// SKIP: does any row of tok_in[0..S) differ from aux2 (blank)?  tok_in is final at the preceding grid barrier, so every
// thread of every CTA gets the same answer.
__device__ __noinline__ bool phase_skip_live(const EbPhase& p) {
    int live = 0;
    for (int s = threadIdx.x; s < p.S; s += blockDim.x) live |= __ldcg(p.tok_in + s) != p.aux2;
    return __syncthreads_or(live);
}

// the phase loader copies the struct as 32-bit words, one per thread of the 256-thread CTA
static_assert(sizeof(EbPhase) % 4 == 0 && sizeof(EbPhase) / 4 <= 256, "EbPhase loader");

// Two instantiations: CTC = false runs every phase but CTC_BEAM (which it skips), CTC = true adds CTC_BEAM.  Any reachable
// call to phase_ctc_beam, whatever the call site, takes this kernel from 12 / 16 to 44 / 136 bytes of spill stores / loads,
// some of them inside the matrix phases' tile loops; the programs that do not search CTC beams keep the kernel without it.
// A third, CTC_STREAM = true (eb_decode_run_ctc_stream), adds GRU and CTC_EMIT, the phases of a streaming CTC chunk, and
// skips LSTM (with it, 28 / 52 bytes of spills instead of 16 / 28); the other two skip GRU and CTC_EMIT like any unknown
// type, so their code and registers are what they were without these phases.
// A fourth, GRU_RNNT = true (eb_decode_run_gru_rnnt), is the default one plus GRU: the phases of a streaming GRU
// transducer chunk (GRU encoder, LSTM predictor and LM, greedy and beam frames).  It skips CTC_BEAM and CTC_EMIT.
// A fifth, CTC_STREAM_BEAM = true (eb_decode_run_ctc_stream_beam), holds the phases of a streaming CTC beam chunk: the
// GRU encoder, CTC_EMIT for the log-probs, CTC_BEAM, the LM's LSTM step, GATHER and BEAM_COMMIT.  It has to be a kernel
// of its own: with CTC_BEAM reachable from any of the four above, their matrix phases would pay its spills.  It skips
// ARGMAX, BEAM_SELECT and BEAM_FINAL, which no CTC program uses: with them, 68 / 200 bytes of spills instead of 36 / 148.
template <bool CTC, bool CTC_STREAM, bool GRU_RNNT, bool CTC_STREAM_BEAM>
__global__ void __launch_bounds__(256) decode_program_kernel(const EbPhase* __restrict__ prog, int nphase, unsigned* bar) {
    extern __shared__ __align__(16) float dsm[];
    float* red = dsm;                                        // [8 warps][2048]
    float* outs = dsm + RED_FLOATS;                          // [64][33]
    __shared__ EbPhase ph;
    // the next phase index lives in shared memory: a loop-carried register that SKIP could change costs the matrix
    // phases (compiled at the 255-register cap) extra spills
    __shared__ int next;
    unsigned epoch = 0;
    for (int i = 0; i < nphase; i = next) {
        __syncthreads();
        if (threadIdx.x < sizeof(EbPhase) / 4)
            reinterpret_cast<int*>(&ph)[threadIdx.x] = reinterpret_cast<const int*>(prog + i)[threadIdx.x];
        if (threadIdx.x == 0) next = i + 1;
        __syncthreads();
        const long gtid = (long)blockIdx.x * blockDim.x + threadIdx.x, gn = (long)gridDim.x * blockDim.x;
        switch (ph.type) {
            case EB_PH_LN: phase_ln(ph); break;
            case EB_PH_PAIR: {
                const int H = ph.N, n2 = ph.aux / 2;                // x1 [S, n, H] -> y [S, n/2, H]
                for (long k = gtid; k < (long)ph.S * n2 * H; k += gn) {
                    const int c = (int)(k % H);
                    const long st = k / H;
                    const int t2 = (int)(st % n2), s = (int)(st / n2);
                    const float* x = ph.x1 + ((long)s * ph.aux + 2 * t2) * H + c;
                    ph.y[k] = 0.5f * (__ldcg(x) + __ldcg(x + H));
                }
            } break;
            case EB_PH_LSTM:
                if constexpr (!CTC_STREAM) phase_lstm(ph, red, outs);
                break;
            case EB_PH_LINEAR: phase_linear(ph, red, outs); break;
            case EB_PH_ARGMAX:
                if constexpr (!CTC_STREAM_BEAM) phase_argmax(ph);
                break;
            case EB_PH_COPY:
                for (long k = gtid; k < (long)ph.S * ph.N; k += gn) ph.y[k] = __ldcg(ph.x1 + k);
                break;
            case EB_PH_BEAM_SELECT:
                if constexpr (!CTC_STREAM_BEAM) phase_beam_select(ph, dsm);
                break;
            case EB_PH_CTC_BEAM:
                if constexpr (CTC || CTC_STREAM_BEAM) phase_ctc_beam(ph, dsm);
                break;
            case EB_PH_GATHER: phase_gather(ph); break;
            case EB_PH_BEAM_FINAL:
                if constexpr (!CTC_STREAM_BEAM) phase_beam_final(ph);
                break;
            case EB_PH_BEAM_COMMIT: phase_beam_commit(ph, dsm); break;
            case EB_PH_SKIP:
                // writes nothing, so it takes no grid barrier (and no epoch) of its own, and neither do the phases it
                // skips: every CTA counts the same barriers
                if (!phase_skip_live(ph) && threadIdx.x == 0) next = i + 1 + ph.aux;
                __syncthreads();                             // every thread reads the same next
                continue;
            default:
                if constexpr (CTC_STREAM || CTC_STREAM_BEAM) {
                    if (ph.type == EB_PH_GRU) phase_gru(ph, red, outs);
                    else if (ph.type == EB_PH_CTC_EMIT) phase_ctc_emit(ph);
                } else if constexpr (GRU_RNNT) {
                    if (ph.type == EB_PH_GRU) phase_gru(ph, red, outs);
                }
                break;
        }
        ++epoch;
        if (i + 1 < nphase) grid_sync(bar, epoch * gridDim.x);
        // redundant after grid_sync, but it costs nothing beside the grid barrier, and with it ptxas keeps this kernel's
        // spills at 12 / 16 bytes (stores / loads); without it they grow to 20 / 28
        __syncthreads();
    }
}

}  // namespace

template <bool CTC, bool CTC_STREAM, bool GRU_RNNT, bool CTC_STREAM_BEAM = false>
int decode_run(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream) {
    if (!phases_dev || nphase <= 0 || !barrier_dev) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    EB_CUDA(cudaMemsetAsync(barrier_dev, 0, 8, st));        // the phase loop's barrier counter and fe_program's
    int grid = eb_num_sms();
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    const EbPhase* prog = reinterpret_cast<const EbPhase*>(phases_dev);
    unsigned* bar = reinterpret_cast<unsigned*>(barrier_dev);
    void* args[] = {(void*)&prog, (void*)&nphase, (void*)&bar};
    const size_t smem = sizeof(float) * (RED_FLOATS + TR * OUT_LD);
    EB_CUDA(cudaFuncSetAttribute(decode_program_kernel<CTC, CTC_STREAM, GRU_RNNT, CTC_STREAM_BEAM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem));
    EB_CUDA(cudaLaunchCooperativeKernel((void*)decode_program_kernel<CTC, CTC_STREAM, GRU_RNNT, CTC_STREAM_BEAM>, dim3(grid), dim3(256), args, smem,
                                        st));
    return EB_OK;
}

EB_API int eb_decode_run(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream) {
    return decode_run<false, false, false>(phases_dev, nphase, barrier_dev, max_ctas, stream);
}

EB_API int eb_decode_run_ctc(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream) {
    return decode_run<true, false, false>(phases_dev, nphase, barrier_dev, max_ctas, stream);
}

EB_API int eb_decode_run_ctc_stream(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream) {
    return decode_run<false, true, false>(phases_dev, nphase, barrier_dev, max_ctas, stream);
}

EB_API int eb_decode_run_gru_rnnt(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream) {
    return decode_run<false, false, true>(phases_dev, nphase, barrier_dev, max_ctas, stream);
}

EB_API int eb_decode_run_ctc_stream_beam(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas,
                                         void* stream) {
    return decode_run<false, false, false, true>(phases_dev, nphase, barrier_dev, max_ctas, stream);
}

EB_API int eb_decode_phase_size(void) { return (int)sizeof(EbPhase); }
