// lm.cu -- the cross-entropy of the language model's output layer (LMModel.loss, edgedict_b200/models.py): what
// nn.NLLLoss(ignore_index) computes on top of the reference's F.log_softmax(decoder(output)) (models.py:224-261), without
// the [rows, V] log-probs ever being written.
//   1. lm_ce_rows_kernel   fp32 mode: one warp per row of fp32 logits, lse = max + log(sum exp(x - max)) (expf / logf,
//                          fixed order) and the target's logit.  bf16 mode takes both from the logits GEMM's epilogue
//                          instead (eb_lm_logits_ce, csrc/gemm_tc.cu).
//   2. lm_ce_loss_kernel   one CTA: per-row costs lse - logit[target], the count of targets that are not ignored and
//                          the sum, in a fixed order (no atomics), the loss and the gradient scale left on the device.
//   3. lm_ce_grad_kernel   one warp per row: d logits = g * scale * (exp(l - lse) - [k == target]), 0 on ignored rows,
//                          fp32 or bf16, in place over the logits.
// A target that is neither ignore_index nor in [0, V) is never used as an index: its cost and its row of d logits are
// NaN.  Nothing here synchronises with the host or allocates.
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int WARPS = 8;
constexpr int LOSS_THREADS = 1024;

__device__ __forceinline__ long long target_at(const void* t, int t64, long r) {
    return t64 ? static_cast<const long long*>(t)[r] : (long long)static_cast<const int*>(t)[r];
}

inline int row_grid(long rows) {
    const long blocks = (rows + WARPS - 1) / WARPS;
    const long cap = (long)eb_num_sms() * 16;
    return (int)(blocks < cap ? blocks : cap);
}

__global__ void __launch_bounds__(WARPS * 32)
lm_ce_rows_kernel(const float* __restrict__ x, const void* __restrict__ targets, int t64, long rows, int V,
                  float* __restrict__ lse, float* __restrict__ tlogit) {
    const int lane = threadIdx.x & 31;
    for (long r = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * WARPS) {
        const float* xr = x + r * V;
        float m = -INFINITY;
        for (int v = lane; v < V; v += 32) m = fmaxf(m, xr[v]);
        m = warp_max(m);
        float s = 0.f;
        for (int v = lane; v < V; v += 32) s += expf(xr[v] - m);
        s = warp_sum(s);
        if (lane == 0) {
            const long long t = target_at(targets, t64, r);
            lse[r] = m + logf(s);
            tlogit[r] = (t >= 0 && t < V) ? xr[t] : 0.f;
        }
    }
}

__global__ void __launch_bounds__(LOSS_THREADS)
lm_ce_loss_kernel(const float* __restrict__ lse, const float* __restrict__ tlogit, const void* __restrict__ targets,
                  int t64, long long ignore, long rows, int V, int mean, float* __restrict__ cost,
                  float* __restrict__ loss, float* __restrict__ scale) {
    __shared__ double sh[33];
    double s = 0.0, n = 0.0;
    for (long r = threadIdx.x; r < rows; r += blockDim.x) {
        const long long t = target_at(targets, t64, r);
        float c = 0.f;
        if (t != ignore) {
            n += 1.0;
            c = (t >= 0 && t < V) ? lse[r] - tlogit[r] : NAN;
        }
        if (cost) cost[r] = c;
        s += (double)c;
    }
    s = block_sum(s, sh);
    n = block_sum(n, sh);
    if (threadIdx.x == 0) {
        loss[0] = mean ? (float)(s / n) : (float)s;          // all ignored: 0 / 0, NaN, as torch's mean
        scale[0] = mean ? (float)(1.0 / n) : 1.f;
    }
}

// VEC consecutive elements of a row as floats (VEC = 1, or 4 fp32 / 8 bf16 in one 16-byte access)
template <typename T, int VEC>
__device__ __forceinline__ void ld_vec(const T* p, float* f) {
    if constexpr (VEC == 1) {
        if constexpr (sizeof(T) == 2) f[0] = __bfloat162float(*p); else f[0] = (float)*p;
    } else if constexpr (sizeof(T) == 2) {
        const uint4 u = *reinterpret_cast<const uint4*>(p);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 x = __bfloat1622float2(h[i]); f[2 * i] = x.x; f[2 * i + 1] = x.y; }
    } else {
        const float4 u = *reinterpret_cast<const float4*>(p);
        f[0] = u.x; f[1] = u.y; f[2] = u.z; f[3] = u.w;
    }
}
template <typename T, int VEC>
__device__ __forceinline__ void st_vec(T* p, const float* f) {
    if constexpr (VEC == 1) {
        if constexpr (sizeof(T) == 2) *p = __float2bfloat16(f[0]); else *p = f[0];
    } else if constexpr (sizeof(T) == 2) {
        uint4 u;
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
        *reinterpret_cast<uint4*>(p) = u;
    } else {
        *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
    }
}

template <typename T, int VEC>
__global__ void __launch_bounds__(WARPS * 32)
lm_ce_grad_kernel(const T* logits, T* grad, const float* __restrict__ lse, const void* __restrict__ targets, int t64,
                  long long ignore, long rows, int V, const float* __restrict__ g, int g_per_row,
                  const float* __restrict__ scale) {
    const int lane = threadIdx.x & 31;
    const float sc = scale ? scale[0] : 1.f;
    for (long r = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * WARPS) {
        const long long t = target_at(targets, t64, r);
        const bool ign = t == ignore;
        // (an ignored row is written as zeros, not as 0 * g: the mean's scale is +inf when every row is ignored)
        const float gs = ign ? 0.f : ((t >= 0 && t < V) ? g[g_per_row ? r : 0] * sc : NAN);
        const float ls = lse[r];
        const T* lr = logits + r * V;
        T* dr = grad + r * V;
        for (int v = VEC * lane; v < V; v += 32 * VEC) {
            float f[VEC];
            ld_vec<T, VEC>(lr + v, f);
#pragma unroll
            for (int i = 0; i < VEC; ++i) f[i] = ign ? 0.f : gs * (expf(f[i] - ls) - (v + i == t ? 1.f : 0.f));
            st_vec<T, VEC>(dr + v, f);
        }
    }
}

template <typename T>
void launch_grad(const void* logits, void* grad, const float* lse, const void* targets, int t64, long long ignore,
                 long rows, int V, const float* g, int g_per_row, const float* scale, cudaStream_t st) {
    constexpr int VEC = sizeof(T) == 2 ? 8 : 4;
    const bool vec = V % VEC == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(grad) & 15) == 0;
    const T* l = static_cast<const T*>(logits);
    T* d = static_cast<T*>(grad);
    if (vec)
        lm_ce_grad_kernel<T, VEC><<<row_grid(rows), WARPS * 32, 0, st>>>(l, d, lse, targets, t64, ignore, rows, V, g,
                                                                           g_per_row, scale);
    else
        lm_ce_grad_kernel<T, 1><<<row_grid(rows), WARPS * 32, 0, st>>>(l, d, lse, targets, t64, ignore, rows, V, g,
                                                                         g_per_row, scale);
}

}  // namespace

EB_API int eb_lm_ce_rows(const float* logits, const void* targets, int targets_int64, float* lse, float* tlogit, long M,
                         int V, void* stream) {
    if (!logits || !targets || !lse || !tlogit || M < 0 || V <= 0) return EB_ERR_INVALID;
    if (M == 0) return EB_OK;
    lm_ce_rows_kernel<<<row_grid(M), WARPS * 32, 0, (cudaStream_t)stream>>>(logits, targets, targets_int64 ? 1 : 0, M,
                                                                            V, lse, tlogit);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_lm_ce_loss(const float* lse, const float* tlogit, const void* targets, int targets_int64,
                         long ignore_index, long M, int V, int mean, float* cost, float* loss, float* scale,
                         void* stream) {
    if ((M > 0 && (!lse || !tlogit || !targets)) || !loss || !scale || M < 0 || V <= 0) return EB_ERR_INVALID;
    lm_ce_loss_kernel<<<1, LOSS_THREADS, 0, (cudaStream_t)stream>>>(lse, tlogit, targets, targets_int64 ? 1 : 0,
                                                                    ignore_index, M, V, mean ? 1 : 0, cost, loss, scale);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_lm_ce_bwd(const void* logits, void* grad, int bf16, const float* lse, const void* targets,
                        int targets_int64, long ignore_index, long M, int V, const float* g, int g_per_row,
                        const float* scale, void* stream) {
    if (!logits || !grad || !lse || !targets || !g || M < 0 || V <= 0) return EB_ERR_INVALID;
    if (M == 0) return EB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int t64 = targets_int64 ? 1 : 0;
    if (bf16)
        launch_grad<__nv_bfloat16>(logits, grad, lse, targets, t64, ignore_index, M, V, g, g_per_row, scale, st);
    else
        launch_grad<float>(logits, grad, lse, targets, t64, ignore_index, M, V, g, g_per_row, scale, st);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
