// conv.cu -- the raw-waveform front end (FrontEnd, rnnt/models.py:313-365): causal strided 1-D convolutions, exact GELU
// and GroupNorm(1, C), channels-last throughout.
//
// Operand layout.  Each strided conv (kernel k, stride s, p = k - 1) reads its input from a padded buffer: per utterance
// Q*s rows of C_in (p zero rows, the T input rows, zeros up to a multiple of s), then ceil(k/s)*s zero rows after the
// last utterance.  Output row m = b*Q + t takes tap j from padded row m*s + j, so the convolution is a GEMM on the
// overlapping row view (row pitch s*C_in, K = k*C_in) and no im2col is written.  Rows t >= T_out of each utterance are
// computed and never used.  In bf16 mode the same buffer is a 3-D tensor map {C_in, s, rows}: tap j of output tile t0 is
// the box at (c0, j mod s, t0 + j div s), and the view does not overlap.
//
//   eb_conv1d_first_fwd / _dw : the first layer (C_in = 1) as a CUDA-core direct convolution; dW and db over row splits.
//   eb_gn_stats               : per-utterance mean / rstd of GELU(y) over all C x T (padded frames included), fp64 sums.
//   eb_gn_apply               : the normalised, affine operand of the next conv into its padded buffer (fp32 or bf16).
//   eb_gn_bwd                 : GroupNorm + GELU backward: dgamma, dbeta, the conv-input gradient and its bias gradient.
//   eb_conv1d_bf16            : out[m] = bias + sum_j X[m*s + j] . W[:, j, :]^T, TMA + wgmma, fp32 accumulation; with
//                               s = 1 and a negative row offset it is also the phase GEMM of dX.
// Every reduction is written as partial slices summed in slice order (eb_colsum): no float atomics, the same bits on
// every run.
#include <cuda.h>
#include "common.cuh"
#include "sm90.cuh"
#include "../../include/edgedict_b200.h"

namespace {

__device__ __forceinline__ float gelu(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad(float x) {
    const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
    return cdf + x * 0.39894228040143268f * expf(-0.5f * x * x);
}

// ---- first layer -------------------------------------------------------------------------------------------------------
// y[b, t, c] = bias[c] + sum_j w[c, j] x[b, t*s + j - p]   (x = 0 outside [0, L))
__global__ void first_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                 float* __restrict__ y, int B, int L, int C, int k, int s, int T) {
    const long n = (long)B * T * C;
    const int p = k - 1;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long bt = i / C;
        const int t = (int)(bt % T), b = (int)(bt / T);
        const float* xb = x + (long)b * L;
        float acc = bias ? bias[c] : 0.f;
        for (int j = 0; j < k; ++j) {
            const long u = (long)t * s + j - p;
            if (u >= 0 && u < L) acc = fmaf(w[c * k + j], xb[u], acc);
        }
        y[i] = acc;
    }
}

// part[split][j][c] (j = k: the bias) = sum over the split's rows of dy[row, c] * x(row, j), rows in order
__global__ void first_dw_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ part,
                                int B, int L, int C, int k, int s, int T, long rows_per_split) {
    const long rows = (long)B * T;
    const long r0 = blockIdx.x * rows_per_split, r1 = min(rows, r0 + rows_per_split);
    const int p = k - 1, n = (k + 1) * C;
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        const int j = e / C, c = e % C;
        float acc = 0.f;
        for (long r = r0; r < r1; ++r) {
            const int t = (int)(r % T), b = (int)(r / T);
            const long u = (long)t * s + j - p;
            const float xv = j == k ? 1.f : ((u >= 0 && u < L) ? x[(long)b * L + u] : 0.f);
            acc = fmaf(dy[r * C + c], xv, acc);
        }
        part[(long)blockIdx.x * n + e] = acc;
    }
}

// ---- GroupNorm(1, C) over GELU ---------------------------------------------------------------------------------------
// Blocks of 256 threads over (row split, utterance, channel block): thread (r, cl) owns channel cb*cw + cl and rows
// t0 + r, t0 + r + rp, ... of the split, rp = 256 / cw row lanes of cw = min(C, 256) channels.
constexpr int GN_THREADS = 256;

struct GnGeo {
    int cw, rp, c, r;
    bool on;
    __device__ GnGeo(int C) {
        cw = C < GN_THREADS ? C : GN_THREADS;
        rp = GN_THREADS / cw;
        c = blockIdx.z * cw + (int)threadIdx.x % cw;
        r = (int)threadIdx.x / cw;
        on = (int)threadIdx.x < rp * cw && c < C;
    }
};

// fixed-order sum of two doubles over the block (tree over thread index); thread 0 holds the result
__device__ void block_sum2(double& a, double& b, double* sh) {
    sh[threadIdx.x] = a;
    sh[GN_THREADS + threadIdx.x] = b;
    __syncthreads();
    for (int o = GN_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            sh[threadIdx.x] += sh[threadIdx.x + o];
            sh[GN_THREADS + threadIdx.x] += sh[GN_THREADS + threadIdx.x + o];
        }
        __syncthreads();
    }
    a = sh[0];
    b = sh[GN_THREADS];
    __syncthreads();
}

// dpart[(b*nsplit + split)*gz + z] = (sum g, sum g^2) of g = GELU(y) over the block's elements
__global__ void __launch_bounds__(GN_THREADS)
gn_stats_kernel(const float* __restrict__ y, long ustride, int T, int C, int rows_per_split, double2* __restrict__ dpart) {
    __shared__ double sh[2 * GN_THREADS];
    const GnGeo g(C);
    const int b = blockIdx.y, t0 = blockIdx.x * rows_per_split, t1 = min(T, t0 + rows_per_split);
    double s1 = 0.0, s2 = 0.0;
    if (g.on) {
        const float* yb = y + (long)b * ustride + g.c;
        for (int t = t0 + g.r; t < t1; t += g.rp) {
            const double v = gelu(yb[(long)t * C]);
            s1 += v;
            s2 += v * v;
        }
    }
    block_sum2(s1, s2, sh);
    if (threadIdx.x == 0) dpart[((long)b * gridDim.x + blockIdx.x) * gridDim.z + blockIdx.z] = make_double2(s1, s2);
}

// mean / rstd of utterance b from its nparts partials, in order (biased variance, as GroupNorm)
__global__ void gn_finalize_kernel(const double2* __restrict__ dpart, int nparts, int B, double n, float eps,
                                   float* __restrict__ mean, float* __restrict__ rstd) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    double s1 = 0.0, s2 = 0.0;
    for (int i = 0; i < nparts; ++i) { s1 += dpart[(long)b * nparts + i].x; s2 += dpart[(long)b * nparts + i].y; }
    const double m = s1 / n, var = fmax(s2 / n - m * m, 0.0);
    mean[b] = (float)m;
    rstd[b] = (float)(1.0 / sqrt(var + (double)eps));
}

// padded operand row r (b = r / rows_per_utt, u = r % rows_per_utt): (GELU(y[b, u - p]) - mean_b) * rstd_b * gamma + beta
// for p <= u < p + T, else 0 (the conv padding, the stride round-up and the tail after the last utterance)
template <typename OUT>
__global__ void gn_apply_kernel(const float* __restrict__ y, long ustride, int B, int T, int C,
                                const float* __restrict__ mean, const float* __restrict__ rstd,
                                const float* __restrict__ gamma, const float* __restrict__ beta, OUT* __restrict__ out,
                                int p, long rows_per_utt, long total_rows) {
    const long n = total_rows * C;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long r = i / C;
        const long b = r / rows_per_utt, u = r % rows_per_utt - p;
        float v = 0.f;
        if (b < B && u >= 0 && u < T) {
            const float gv = gelu(y[b * ustride + u * C + c]);
            v = (gv - mean[b]) * rstd[b] * (gamma ? gamma[c] : 1.f) + (beta ? beta[c] : 0.f);
        }
        if constexpr (sizeof(OUT) == 2) out[i] = __float2bfloat16(v);
        else out[i] = v;
    }
}

// store the block's per-channel sums (row lanes added in order) to part[slot][c]; the channel blocks of a (split,
// utterance) share the slot, each writing its own channels
__device__ void chan_store(float v, const GnGeo& g, float* sh, float* __restrict__ part, long slot, int C) {
    sh[threadIdx.x] = v;
    __syncthreads();
    if ((int)threadIdx.x < g.cw && g.c < C) {
        float a = 0.f;
        for (int r = 0; r < g.rp; ++r) a += sh[r * g.cw + threadIdx.x];
        part[slot * C + g.c] = a;
    }
    __syncthreads();
}

// pass A: with x^ = (GELU(y) - mean) rstd and dz the gradient of the affine output:
//   pg[slot][c] = sum dz x^,  pb[slot][c] = sum dz  (slot = b*nsplit + split),
//   dpart[slot*gz + z] = (sum dz gamma, sum dz gamma x^) of the utterance, one per channel block z
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_sums_kernel(const float* __restrict__ y, long ustride, int T, int C, const float* __restrict__ mean,
                   const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ dz,
                   long dz_ustride, int rows_per_split, float* __restrict__ pg, float* __restrict__ pb,
                   double2* __restrict__ dpart) {
    __shared__ double sh[2 * GN_THREADS];
    const GnGeo g(C);
    const int b = blockIdx.y, t0 = blockIdx.x * rows_per_split, t1 = min(T, t0 + rows_per_split);
    const float mu = mean[b], rs = rstd[b];
    float sg = 0.f, sb = 0.f;
    double s1 = 0.0, s2 = 0.0;
    if (g.on) {
        const float ga = gamma ? gamma[g.c] : 1.f;
        const float* yb = y + (long)b * ustride + g.c;
        const float* db = dz + (long)b * dz_ustride + g.c;
        for (int t = t0 + g.r; t < t1; t += g.rp) {
            const float xh = (gelu(yb[(long)t * C]) - mu) * rs, d = db[(long)t * C];
            sg = fmaf(d, xh, sg);
            sb += d;
            const double dx = (double)d * ga;
            s1 += dx;
            s2 += dx * xh;
        }
    }
    const long slot = (long)b * gridDim.x + blockIdx.x;
    float* shf = reinterpret_cast<float*>(sh);
    chan_store(sg, g, shf, pg, slot, C);
    chan_store(sb, g, shf, pb, slot, C);
    block_sum2(s1, s2, sh);
    if (threadIdx.x == 0) dpart[slot * gridDim.z + blockIdx.z] = make_double2(s1, s2);
}

// pass B: dy = rstd (dz gamma - S1/N - x^ S2/N) GELU'(y) into the conv-output gradient buffers (fp32 and / or bf16),
// and the per-channel partial sums of dy (the bias gradient of the conv below) into pdb[slot][c]
template <bool BF>
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_dy_kernel(const float* __restrict__ y, long ustride, int T, int C, const float* __restrict__ mean,
                 const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ dz,
                 long dz_ustride, int rows_per_split, const double2* __restrict__ dpart, int nparts, double n,
                 float* __restrict__ dy, __nv_bfloat16* __restrict__ dy16, long dy_ustride, float* __restrict__ pdb) {
    __shared__ float sh[GN_THREADS];
    __shared__ float coef[2];
    const GnGeo g(C);
    const int b = blockIdx.y, t0 = blockIdx.x * rows_per_split, t1 = min(T, t0 + rows_per_split);
    if (threadIdx.x == 0) {
        double s1 = 0.0, s2 = 0.0;
        for (int i = 0; i < nparts; ++i) { s1 += dpart[(long)b * nparts + i].x; s2 += dpart[(long)b * nparts + i].y; }
        coef[0] = (float)(s1 / n);
        coef[1] = (float)(s2 / n);
    }
    __syncthreads();
    const float mu = mean[b], rs = rstd[b], m1 = coef[0], m2 = coef[1];
    float sdb = 0.f;
    if (g.on) {
        const float ga = gamma ? gamma[g.c] : 1.f;
        const float* yb = y + (long)b * ustride + g.c;
        const float* db = dz + (long)b * dz_ustride + g.c;
        const long ob = (long)b * dy_ustride + g.c;
        for (int t = t0 + g.r; t < t1; t += g.rp) {
            const float yv = yb[(long)t * C];
            const float xh = (gelu(yv) - mu) * rs;
            const float v = rs * (db[(long)t * C] * ga - m1 - xh * m2) * gelu_grad(yv);
            if (dy) dy[ob + (long)t * C] = v;
            if (BF) dy16[ob + (long)t * C] = __float2bfloat16(v);
            sdb += v;
        }
    }
    if (pdb) chan_store(sdb, g, sh, pdb, (long)b * gridDim.x + blockIdx.x, C);
}

// ---- strided conv on the tensor cores (bf16 operands, fp32 accumulation) -------------------------------------------
// Tile 128 rows x BN columns; two consumer warpgroups (64 rows each) and a TMA producer warp; k-iterations run over
// (tap j, channel chunk of BKC) in that order.  BKC = 64 / 32 / 16 channels: operand rows of 128 / 64 / 32 B in the
// matching TMA swizzle, so that channel counts of 16 and 32 need no padding.
constexpr int CBM = 128, CTHREADS = 2 * 128 + 32, CSTAGES = 4;

template <int BN, int BKC> struct ConvCfg {
    static constexpr int ROWB = BKC * 2;                           // bytes per operand row = the swizzle span
    static constexpr int A_BYTES = CBM * ROWB, B_BYTES = BN * ROWB;
    static constexpr int STAGE_BYTES = (A_BYTES + B_BYTES + 1023) / 1024 * 1024;
    static constexpr int SMEM_BYTES = 1024 + CSTAGES * STAGE_BYTES + 256;
    static constexpr uint64_t LAYOUT = BKC == 64 ? 1 : (BKC == 32 ? 2 : 3);   // descriptor: SW128 / SW64 / SW32
    static constexpr CUtensorMapSwizzle SWZ =
        BKC == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (BKC == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
};

// K-major swizzled operand: 8-row groups 8 * row bytes apart
__device__ __forceinline__ uint64_t conv_desc(uint32_t saddr, uint32_t sbo, uint64_t layout) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32) |
           (layout << 62);
}

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t da, uint64_t db) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %10, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(1));
}

template <int BN>
__device__ __forceinline__ void conv_mma(float (&acc)[BN / 2], uint64_t ad, uint64_t bd) {
    if constexpr (BN == 128) wgmma_m64n128k16<0, 0>(acc, ad, bd, 1);
    else if constexpr (BN == 32) wgmma_m64n32k16<0, 0>(acc, ad, bd, 1);
    else wgmma_m64n16k16(acc, ad, bd);
}

// out[m, n] = bias[n] + sum_{j < taps} sum_c X[m + row0 + j / s, j % s, c] W[n, j * C + c]   (m < M, n < N)
template <int BN, int BKC>
__global__ void __launch_bounds__(CTHREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tma_x, const __grid_constant__ CUtensorMap tma_w,
               float* __restrict__ out, long ldc, const float* __restrict__ bias, long M, int N, int C, int s, int taps,
               int row0) {
    using Cf = ConvCfg<BN, BKC>;
    constexpr int NACC = BN / 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + CSTAGES * Cf::STAGE_BYTES);
    const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + CSTAGES);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long num_m = (M + CBM - 1) / CBM;
    const int num_n = N / BN;
    const long tiles = num_m * num_n;
    const int nkc = C / BKC, nk = taps * nkc;

    if (threadIdx.x == 0) {
        for (int i = 0; i < CSTAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_w) : "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                const int m0 = (int)((tile / num_n) * CBM), n0 = (int)(tile % num_n) * BN;
                for (int kk = 0; kk < nk; ++kk) {
                    const int j = kk / nkc, c0 = (kk % nkc) * BKC;
                    mbar_wait(empty0 + 8 * stage, phase ^ 1);
                    const uint32_t sa = smem_u32(smem + stage * Cf::STAGE_BYTES), sb = sa + Cf::A_BYTES;
                    const uint32_t fb = full0 + 8 * stage;
                    mbar_expect_tx(fb, Cf::A_BYTES + Cf::B_BYTES);   // rows outside the buffer arrive as zeros
                    tma_load_3d(sa, &tma_x, c0, j % s, m0 + row0 + j / s, fb);
                    tma_load_2d(sb, &tma_w, j * C + c0, n0, fb);
                    if (++stage == CSTAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    const int wg = warp >> 2;
    const int r_in = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
    float acc[NACC];
    int stage = 0;
    uint32_t phase = 0;
    for (long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const long m0 = (tile / num_n) * CBM;
        const int n0 = (int)(tile % num_n) * BN;
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kk = 0; kk < nk; ++kk) {
            mbar_wait(full0 + 8 * stage, phase);
            const uint32_t sa = smem_u32(smem + stage * Cf::STAGE_BYTES) + (uint32_t)wg * 64u * Cf::ROWB;
            const uint32_t sb = smem_u32(smem + stage * Cf::STAGE_BYTES) + Cf::A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BKC / 16; ++k)
                conv_mma<BN>(acc, conv_desc(sa + 32 * k, 8 * Cf::ROWB, Cf::LAYOUT),
                             conv_desc(sb + 32 * k, 8 * Cf::ROWB, Cf::LAYOUT));
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
            prev = stage;
            if (++stage == CSTAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const long row = m0 + r_in + 8 * h;
            if (row >= M) continue;
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
                const int col = n0 + 8 * i + cq;
                float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
                if (bias) { v0 += __ldg(bias + col); v1 += __ldg(bias + col + 1); }
                *reinterpret_cast<float2*>(out + row * ldc + col) = make_float2(v0, v1);
            }
        }
    }
}

template <int BN, int BKC>
int conv_tc_launch(const void* x16, long x_rows, int s, int C, int row0, const void* w16, int taps, int N,
                   const float* bias, float* out, long ldc, long M, cudaStream_t st) {
    using Cf = ConvCfg<BN, BKC>;
    EncodeTiledFn enc = get_encode();
    if (!enc) return EB_ERR_CUDA;
    CUtensorMap tx, tw;
    const cuuint64_t xd[3] = {(cuuint64_t)C, (cuuint64_t)s, (cuuint64_t)x_rows};
    const cuuint64_t xs[2] = {(cuuint64_t)C * 2, (cuuint64_t)s * C * 2};
    const cuuint32_t xb[3] = {BKC, 1, CBM}, e3[3] = {1, 1, 1};
    const cuuint64_t wd[2] = {(cuuint64_t)taps * C, (cuuint64_t)N};
    const cuuint64_t ws[1] = {(cuuint64_t)taps * C * 2};
    const cuuint32_t wb[2] = {BKC, BN}, e2[2] = {1, 1};
    if (enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(x16), xd, xs, xb, e3, CU_TENSOR_MAP_INTERLEAVE_NONE,
            Cf::SWZ, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS ||
        enc(&tw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w16), wd, ws, wb, e2, CU_TENSOR_MAP_INTERLEAVE_NONE,
            Cf::SWZ, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
        fprintf(stderr, "[edgedict_b200] cuTensorMapEncodeTiled failed (conv)\n");
        return EB_ERR_CUDA;
    }
    auto kern = conv_tc_kernel<BN, BKC>;
    static bool attr_done = false;
    if (!attr_done) {
        EB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cf::SMEM_BYTES));
        attr_done = true;
    }
    const long tiles = ((M + CBM - 1) / CBM) * (N / BN);
    const int grid = (int)(tiles < eb_num_sms() ? tiles : eb_num_sms());
    kern<<<grid, CTHREADS, Cf::SMEM_BYTES, st>>>(tx, tw, out, ldc, bias, M, N, C, s, taps, row0);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

template <int BN>
int conv_tc_bkc(const void* x16, long x_rows, int s, int C, int row0, const void* w16, int taps, int N,
                const float* bias, float* out, long ldc, long M, cudaStream_t st) {
    if (C % 64 == 0) return conv_tc_launch<BN, 64>(x16, x_rows, s, C, row0, w16, taps, N, bias, out, ldc, M, st);
    if (C % 32 == 0) return conv_tc_launch<BN, 32>(x16, x_rows, s, C, row0, w16, taps, N, bias, out, ldc, M, st);
    return conv_tc_launch<BN, 16>(x16, x_rows, s, C, row0, w16, taps, N, bias, out, ldc, M, st);
}

int ew_blocks(long n) {
    const long b = (n + 255) / 256, cap = 8L * eb_num_sms();
    return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

int gn_cblocks(int C) { return (C + GN_THREADS - 1) / GN_THREADS; }

}  // namespace

EB_API int eb_conv_rows_per_split(int C) {
    if (C <= 0) return 0;
    const int r = 32768 / C;
    return r < 1 ? 1 : r;
}

EB_API int eb_conv1d_first_fwd(const float* x, const float* w, const float* bias, float* y, int B, int L, int C, int k,
                               int s, int T, void* stream) {
    if (!x || !w || !y || B <= 0 || L <= 0 || C <= 0 || k < 2 || s <= 0 || T <= 0 || T != (L + k - 2) / s + 2 - k)
        return EB_ERR_INVALID;
    first_fwd_kernel<<<ew_blocks((long)B * T * C), 256, 0, (cudaStream_t)stream>>>(x, w, bias, y, B, L, C, k, s, T);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_conv1d_first_dw(const float* x, const float* dy, float* part, int nsplit, long rows_per_split, int B,
                              int L, int C, int k, int s, int T, void* stream) {
    if (!x || !dy || !part || B <= 0 || L <= 0 || C <= 0 || k < 2 || s <= 0 || T <= 0 || rows_per_split <= 0 ||
        nsplit != (int)(((long)B * T + rows_per_split - 1) / rows_per_split))
        return EB_ERR_INVALID;
    const int n = (k + 1) * C;
    const int threads = n < 1024 ? (n + 31) / 32 * 32 : 1024;
    first_dw_kernel<<<nsplit, threads, 0, (cudaStream_t)stream>>>(x, dy, part, B, L, C, k, s, T, rows_per_split);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_gn_stats(const float* y, long ustride, int B, int T, int C, double* dpart, float* mean, float* rstd,
                       float eps, void* stream) {
    if (!y || !dpart || !mean || !rstd || B <= 0 || T <= 0 || C <= 0 || ustride < (long)T * C) return EB_ERR_INVALID;
    const int rps = eb_conv_rows_per_split(C), ns = (T + rps - 1) / rps, gz = gn_cblocks(C);
    cudaStream_t st = (cudaStream_t)stream;
    gn_stats_kernel<<<dim3(ns, B, gz), GN_THREADS, 0, st>>>(y, ustride, T, C, rps, (double2*)dpart);
    EB_CHECK_LAUNCH();
    gn_finalize_kernel<<<(B + 127) / 128, 128, 0, st>>>((const double2*)dpart, ns * gz, B, (double)T * C, eps, mean, rstd);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_gn_apply(const float* y, long ustride, int B, int T, int C, const float* mean, const float* rstd,
                       const float* gamma, const float* beta, void* out, int out_bf16, int p, long rows_per_utt,
                       long total_rows, void* stream) {
    if (!y || !mean || !rstd || !out || B <= 0 || T <= 0 || C <= 0 || p < 0 || rows_per_utt < p + T ||
        total_rows < B * rows_per_utt || ustride < (long)T * C)
        return EB_ERR_INVALID;
    const int g = ew_blocks(total_rows * C);
    cudaStream_t st = (cudaStream_t)stream;
    if (out_bf16)
        gn_apply_kernel<__nv_bfloat16><<<g, 256, 0, st>>>(y, ustride, B, T, C, mean, rstd, gamma, beta,
                                                          (__nv_bfloat16*)out, p, rows_per_utt, total_rows);
    else
        gn_apply_kernel<float><<<g, 256, 0, st>>>(y, ustride, B, T, C, mean, rstd, gamma, beta, (float*)out, p,
                                                  rows_per_utt, total_rows);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_gn_bwd(const float* y, long ustride, int B, int T, int C, const float* mean, const float* rstd,
                     const float* gamma, const float* dz, long dz_ustride, float* pg, float* pb, double* dpart,
                     float* dy, void* dy16, long dy_ustride, float* pdb, void* stream) {
    if (!y || !mean || !rstd || !dz || !pg || !pb || !dpart || (!dy && !dy16) || B <= 0 || T <= 0 || C <= 0 ||
        ustride < (long)T * C || dz_ustride < (long)T * C || dy_ustride < (long)T * C)
        return EB_ERR_INVALID;
    const int rps = eb_conv_rows_per_split(C), ns = (T + rps - 1) / rps, gz = gn_cblocks(C);
    const dim3 grid(ns, B, gz);
    cudaStream_t st = (cudaStream_t)stream;
    gn_bwd_sums_kernel<<<grid, GN_THREADS, 0, st>>>(y, ustride, T, C, mean, rstd, gamma, dz, dz_ustride, rps, pg, pb,
                                                    (double2*)dpart);
    EB_CHECK_LAUNCH();
    if (dy16)
        gn_bwd_dy_kernel<true><<<grid, GN_THREADS, 0, st>>>(y, ustride, T, C, mean, rstd, gamma, dz, dz_ustride, rps,
                                                           (const double2*)dpart, ns * gz, (double)T * C, dy,
                                                           (__nv_bfloat16*)dy16, dy_ustride, pdb);
    else
        gn_bwd_dy_kernel<false><<<grid, GN_THREADS, 0, st>>>(y, ustride, T, C, mean, rstd, gamma, dz, dz_ustride, rps,
                                                            (const double2*)dpart, ns * gz, (double)T * C, dy, nullptr,
                                                            dy_ustride, pdb);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_conv1d_bf16(const void* x16, long x_rows, int s, int C, int row0, const void* w16, int taps, int N,
                          const float* bias, float* out, long ldc, long M, void* stream) {
    if (!x16 || !w16 || !out || x_rows <= 0 || s <= 0 || C <= 0 || C % 16 || taps <= 0 || N <= 0 || N % 16 ||
        M <= 0 || M > INT32_MAX || x_rows > INT32_MAX || ldc < N || ldc % 2)
        return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(x16) & 15) || (reinterpret_cast<uintptr_t>(w16) & 15) ||
        (reinterpret_cast<uintptr_t>(out) & 7) || (bias && (reinterpret_cast<uintptr_t>(bias) & 7)))
        return EB_ERR_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    if (N % 128 == 0) return conv_tc_bkc<128>(x16, x_rows, s, C, row0, w16, taps, N, bias, out, ldc, M, st);
    if (N % 32 == 0) return conv_tc_bkc<32>(x16, x_rows, s, C, row0, w16, taps, N, bias, out, ldc, M, st);
    return conv_tc_bkc<16>(x16, x_rows, s, C, row0, w16, taps, N, bias, out, ldc, M, st);
}
