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
//   ARGMAX  token = argmax(logits) with the <unk> rule (stream.py:105-108: logit := 0, re-argmax)
//   COPY    y = x
//
// fp32-accurate arithmetic throughout: the north star asks for token-for-token identical greedy output, which
// bf16 (or plain tf32) near-ties would break.  The matrix products run on the tensor cores as 3xTF32 split
// products with fp32 accumulation (see tile_mma); everything else is fp32 CUDA-core code.
#include <cooperative_groups.h>
#include "common.cuh"
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
            if (embed) return p.x1 + (long)__ldcg(p.tok_in + s0 + r) * p.ldx1;     // embedding row of the last token
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
        auto x1row = [&](int r) -> const float* { return p.x1 + (long)(s0 + r) * p.ldx1; };
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

__device__ void phase_argmax(const EbPhase& p) {
    const int lane = threadIdx.x & 31, V = p.N, blank = p.aux, unk = p.aux2;
    (void)blank;
    for (int s = blockIdx.x * 8 + (threadIdx.x >> 5); s < p.S; s += gridDim.x * 8) {
        const float* x = p.x1 + (long)s * p.ldx1;
        int pred = -1;
        for (int pass = 0; pass < 2; ++pass) {
            float best = -INFINITY;
            int bi = 0x7fffffff;
            for (int v = lane; v < V; v += 32) {
                float val = __ldcg(x + v);
                if (pass == 1 && v == pred) val = 0.f;              // stream.py:107 `prob[:, pred] = 0`
                if (val > best) { best = val; bi = v; }             // strict >: first index wins ties
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                float ob = __shfl_xor_sync(0xffffffffu, best, o);
                int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
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

__global__ void __launch_bounds__(256) decode_program_kernel(const EbPhase* __restrict__ prog, int nphase, unsigned* bar) {
    extern __shared__ __align__(16) float dsm[];
    float* red = dsm;                                        // [8 warps][2048]
    float* outs = dsm + RED_FLOATS;                          // [64][33]
    __shared__ EbPhase ph;
    unsigned epoch = 0;
    for (int i = 0; i < nphase; ++i) {
        __syncthreads();
        if (threadIdx.x < sizeof(EbPhase) / 4)
            reinterpret_cast<int*>(&ph)[threadIdx.x] = reinterpret_cast<const int*>(prog + i)[threadIdx.x];
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
            case EB_PH_LSTM: phase_lstm(ph, red, outs); break;
            case EB_PH_LINEAR: phase_linear(ph, red, outs); break;
            case EB_PH_ARGMAX: phase_argmax(ph); break;
            case EB_PH_COPY:
                for (long k = gtid; k < (long)ph.S * ph.N; k += gn) ph.y[k] = __ldcg(ph.x1 + k);
                break;
            default: break;
        }
        ++epoch;
        if (i + 1 < nphase) grid_sync(bar, epoch * gridDim.x);
    }
}

}  // namespace

EB_API int eb_decode_run(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream) {
    if (!phases_dev || nphase <= 0 || !barrier_dev) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    EB_CUDA(cudaMemsetAsync(barrier_dev, 0, 4, st));
    int grid = eb_num_sms();
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    const EbPhase* prog = reinterpret_cast<const EbPhase*>(phases_dev);
    unsigned* bar = reinterpret_cast<unsigned*>(barrier_dev);
    void* args[] = {(void*)&prog, (void*)&nphase, (void*)&bar};
    const size_t smem = sizeof(float) * (RED_FLOATS + TR * OUT_LD);
    EB_CUDA(cudaFuncSetAttribute(decode_program_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    EB_CUDA(cudaLaunchCooperativeKernel((void*)decode_program_kernel, dim3(grid), dim3(256), args, smem, st));
    return EB_OK;
}

EB_API int eb_decode_phase_size(void) { return (int)sizeof(EbPhase); }
