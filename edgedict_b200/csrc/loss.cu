// loss.cu -- RNN-Transducer loss for sm_90a.
//
// Replaces the reference's GPU path  warp-transducer/include/detail/gpu_rnnt.h:82-215
// (memset + reduce_max + reduce_exp + alphas + betas + grad + D2H, three host syncs) with
//
//   1. rnnt_denom_kernel   one warp per (b,t,u) row: one streaming 128-bit pass over the logits,
//                          writes -logsumexp and the two log-probs the lattice needs
//                          (blank, label[u]) as compact [B,T,U] arrays        (reads 1*s*N bytes)
//   2. rnnt_lattice_kernel alpha and beta wavefronts concurrently (grid = B x 2), each touching
//                          2 floats per cell instead of V-strided gathers      (latency bound)
//   3. rnnt_grad_kernel    one warp per row: re-reads the logits, writes d loss / d logits
//                          (fp32 or bf16, optionally in place), zero on padded cells, scaled
//                          by the upstream gradient on the device               (2*s*N bytes)
//
// and, for forced alignment, rnnt_viterbi_kernel: the alpha wavefront with max in place of
// log-add and a decision byte per cell, then the backtrace in the same CTA (eb_rnnt_viterbi).
//
// No host synchronisation anywhere except in the warp-transducer compatible entry point
// compute_rnnt_loss(), whose contract returns costs in HOST memory (include/rnnt.h).
//
// Arithmetic follows include/detail/gpu_rnnt_kernel.h:5-179 and rnnt_helper.h:17-24.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <type_traits>

#include "common.cuh"
#include "../../include/rnnt.h"
#include "../../include/edgedict_b200.h"

namespace {

template <typename T> struct M;
template <> struct M<float> {
    static __device__ __forceinline__ float exp_fast(float x) { return fast_exp(x); }
    static __device__ __forceinline__ float exp_acc(float x) { return expf(x); }
    static __device__ __forceinline__ float log_acc(float x) { return logf(x); }
    static __device__ __forceinline__ float log1p_acc(float x) { return log1pf(x); }
    static __device__ __forceinline__ float ninf() { return -INFINITY; }
};
template <> struct M<double> {
    static __device__ __forceinline__ double exp_fast(double x) { return exp(x); }
    static __device__ __forceinline__ double exp_acc(double x) { return exp(x); }
    static __device__ __forceinline__ double log_acc(double x) { return log(x); }
    static __device__ __forceinline__ double log1p_acc(double x) { return log1p(x); }
    static __device__ __forceinline__ double ninf() { return -(double)INFINITY; }
};

template <typename T>
__device__ __forceinline__ T lse2(T a, T b) {   // rnnt_helper.h:17-24
    if (a == M<T>::ninf()) return b;
    if (b == M<T>::ninf()) return a;
    return (a > b) ? M<T>::log1p_acc(M<T>::exp_acc(b - a)) + a : M<T>::log1p_acc(M<T>::exp_acc(a - b)) + b;
}

// The lengths every kernel here uses: the valid cells of utterance b are t < Tn, u < Un, which never leave its own
// [maxT, maxU] block whatever xlen / ylen hold (include/edgedict_b200.h).
__device__ __forceinline__ int clamp_T(int xlen, int maxT) { return min(max(xlen, 0), maxT); }
__device__ __forceinline__ int clamp_U(int ylen, int maxU) { return min(max(ylen, 0) + 1, maxU); }

// 4-wide row access; VEC=true requires V % 4 == 0 (row starts are then 16-byte aligned for fp32)
template <typename T, bool VEC> struct Row4 {
    static __device__ __forceinline__ void load(const T* row, int v, int V, T (&x)[4]) {
        if (VEC) {
            if (sizeof(T) == 4) {
                float4 q;
                asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                             : "=f"(q.x), "=f"(q.y), "=f"(q.z), "=f"(q.w) : "l"(row + v));
                x[0] = q.x; x[1] = q.y; x[2] = q.z; x[3] = q.w;
            } else {
                const double2* p = reinterpret_cast<const double2*>(row + v);
                double2 a = p[0], b = p[1];
                x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) x[i] = (v + i < V) ? row[v + i] : M<T>::ninf();
        }
    }
};

// bf16 logits (written by the fused joint GEMM epilogue): 4 values per 8-byte load
template <bool VEC> struct Row4<__nv_bfloat16, VEC> {
    static __device__ __forceinline__ void load(const __nv_bfloat16* row, int v, int V, float (&x)[4]) {
        if (VEC) {
            const uint2 q = *reinterpret_cast<const uint2*>(row + v);
            const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.x));
            const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.y));
            x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y;
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) x[i] = (v + i < V) ? __bfloat162float(row[v + i]) : -INFINITY;
        }
    }
};

// ---------------------------------------------------------------------------------------------
// 1. denominators + (blank, label) gather
// ---------------------------------------------------------------------------------------------
// One warp's statistics of one row of V logits: d = -logsumexp and the blank / label logits xb, xl (0 where absent).
// rnnt_denom_kernel and rnnt_band_denom_kernel share it, so a band row and the same dense cell get the same bits.
template <typename T, bool VEC>
__device__ __forceinline__ void denom_row(const T* row, int lane, int V, int blank, int lab, T& d, T& xb_out,
                                          T& xl_out) {
    // online max / sum-exp over this lane's 4-wide chunks
    T m = M<T>::ninf(), s = 0, xb = 0, xl = 0;
    for (int v = lane * 4; v < V; v += 128) {
        T x[4];
        Row4<T, VEC>::load(row, v, V, x);
        T cm = fmax(fmax(x[0], x[1]), fmax(x[2], x[3]));
        T nm = fmax(m, cm);
        T acc = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            acc += M<T>::exp_fast(x[i] - nm);       // exp(-inf) = 0 for the masked tail
            if (v + i == blank) xb = x[i];
            if (v + i == lab) xl = x[i];
        }
        s = s * M<T>::exp_fast(m - nm) + acc;       // m = -inf on first chunk => s*0
        m = nm;
    }
    T gm = warp_max(m);
    s *= M<T>::exp_fast(m - gm);
    s = warp_sum(s);
    d = -gm - M<T>::log_acc(s);
    // the lane that saw the blank / label column owns the value: reduce by sum of one-hot
    xb_out = warp_sum(xb);
    xl_out = warp_sum(xl);
}

template <typename T, bool VEC, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
rnnt_denom_kernel(const T* __restrict__ logits, const int* __restrict__ labels,
                  const int* __restrict__ xlen, const int* __restrict__ ylen,
                  T* __restrict__ denom, T* __restrict__ lpb, T* __restrict__ lpl,
                  int B, int maxT, int maxU, int V, int blank) {
    const int lane = threadIdx.x & 31;
    const long ncells = (long)B * maxT * maxU;
    const long wstride = (long)gridDim.x * WARPS;
    for (long cell = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); cell < ncells; cell += wstride) {
        const int u = (int)(cell % maxU);
        const long bt = cell / maxU;
        const int t = (int)(bt % maxT);
        const int b = (int)(bt / maxT);
        const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
        if (t >= Tn || u >= Un) continue;                // padded cell: never read
        const T* row = logits + cell * (long)V;
        const int lab = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
        T d, xb, xl;
        denom_row<T, VEC>(row, lane, V, blank, lab, d, xb, xl);
        if (lane == 0) {
            denom[cell] = d;
            lpb[cell] = d + xb;
            lpl[cell] = d + xl;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 2. alpha / beta wavefronts.  grid = (B, 2): y == 0 -> alphas, y == 1 -> betas.
//    blockDim.x = maxU rounded up to a warp.  Thread u walks its own column t = n - u, with the log-probs of the
//    next PF diagonals in flight in registers.  An utterance without frames (Tn = 0) has no diagonal: ll = -inf.
// ---------------------------------------------------------------------------------------------
template <typename T, int PF>
__device__ __forceinline__ void lattice_body(const T* __restrict__ lpb, const T* __restrict__ lpl,
                                             const int* __restrict__ xlen, const int* __restrict__ ylen,
                                             T* __restrict__ alphas, T* __restrict__ betas,
                                             T* __restrict__ ll_fwd, T* __restrict__ ll_bwd,
                                             int maxT, int maxU, int do_beta) {
    extern __shared__ unsigned char sm_raw[];
    T* sh = reinterpret_cast<T*>(sm_raw);               // [2][blockDim.x]
    const int b = blockIdx.x, u = threadIdx.x;
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    const long base = (long)b * maxT * maxU;
    const T* pb = lpb + base;
    const T* pl = lpl + base;
    const int ND = Tn > 0 ? Tn + Un - 1 : 0;             // number of anti-diagonals
    const bool act = u < Un;
    const int W = blockDim.x;
    if (blockIdx.y == 0) {
        T* al = alphas + base;
        T self = M<T>::ninf();                           // alpha(t-1,u)
        // register prefetch ring: values for iterations n0 .. n0+PF-1
        T cb[PF], cl[PF], nb[PF], nl[PF];
#pragma unroll
        for (int i = 0; i < PF; ++i) {
            int t = i - u;
            cb[i] = (act && t >= 1 && t < Tn) ? pb[(long)(t - 1) * maxU + u] : T(0);
            cl[i] = (act && u >= 1 && t >= 0 && t < Tn) ? pl[(long)t * maxU + u - 1] : T(0);
        }
        for (int n0 = 0; n0 < ND; n0 += PF) {
#pragma unroll
            for (int i = 0; i < PF; ++i) {               // issue next block's loads early
                int t = n0 + PF + i - u;
                nb[i] = (act && t >= 1 && t < Tn) ? pb[(long)(t - 1) * maxU + u] : T(0);
                nl[i] = (act && u >= 1 && t >= 0 && t < Tn) ? pl[(long)t * maxU + u - 1] : T(0);
            }
#pragma unroll
            for (int i = 0; i < PF; ++i) {
                const int n = n0 + i;
                if (n < ND) {
                    const int t = n - u;
                    if (act && t >= 0 && t < Tn) {
                        T a;
                        if (n == 0) a = 0;
                        else {
                            T stay = (t > 0) ? self + cb[i] : M<T>::ninf();
                            T emit = (u > 0) ? sh[((n - 1) & 1) * W + u - 1] + cl[i] : M<T>::ninf();
                            a = lse2(emit, stay);
                        }
                        al[(long)t * maxU + u] = a;
                        self = a;
                        sh[(n & 1) * W + u] = a;
                    }
                }
                __syncthreads();
            }
#pragma unroll
            for (int i = 0; i < PF; ++i) { cb[i] = nb[i]; cl[i] = nl[i]; }
        }
        if (u == Un - 1) ll_fwd[b] = Tn > 0 ? self + pb[(long)(Tn - 1) * maxU + Un - 1] : M<T>::ninf();
    } else {
        if (!do_beta) return;
        T* be = betas + base;
        T self = M<T>::ninf();                           // beta(t+1,u)
        T cb[PF], cl[PF], nb[PF], nl[PF];
#pragma unroll
        for (int i = 0; i < PF; ++i) {
            int t = (ND - 1 - i) - u;
            bool ok = act && t >= 0 && t < Tn;
            cb[i] = ok ? pb[(long)t * maxU + u] : T(0);
            cl[i] = (ok && u < Un - 1) ? pl[(long)t * maxU + u] : T(0);
        }
        for (int n0 = 0; n0 < ND; n0 += PF) {
#pragma unroll
            for (int i = 0; i < PF; ++i) {
                int t = (ND - 1 - (n0 + PF + i)) - u;
                bool ok = act && t >= 0 && t < Tn;
                nb[i] = ok ? pb[(long)t * maxU + u] : T(0);
                nl[i] = (ok && u < Un - 1) ? pl[(long)t * maxU + u] : T(0);
            }
#pragma unroll
            for (int i = 0; i < PF; ++i) {
                const int k = n0 + i;                    // k-th step, diagonal n = ND-1-k
                if (k < ND) {
                    const int n = ND - 1 - k;
                    const int t = n - u;
                    if (act && t >= 0 && t < Tn) {
                        T v;
                        if (k == 0) v = cb[i];           // (T-1, U-1): log p(blank)
                        else {
                            T stay = (t < Tn - 1) ? self + cb[i] : M<T>::ninf();
                            T emit = (u < Un - 1) ? sh[((k - 1) & 1) * W + u + 1] + cl[i] : M<T>::ninf();
                            v = lse2(emit, stay);
                        }
                        be[(long)t * maxU + u] = v;
                        self = v;
                        sh[(k & 1) * W + u] = v;
                    }
                }
                __syncthreads();
            }
#pragma unroll
            for (int i = 0; i < PF; ++i) { cb[i] = nb[i]; cl[i] = nl[i]; }
        }
        if (u == 0) ll_bwd[b] = self;                    // -inf when Tn = 0: no cell was written
    }
}

// The kernel for blocks of up to the thread count its registers allow (896 fp32 / 544 fp64 threads with ptxas of
// CUDA 12.9), and the one for wider blocks: a shallower ring in the registers a 1024-thread block leaves.  The ring's
// depth only moves loads earlier, so both give the same bits.
template <typename T>
__global__ void rnnt_lattice_kernel(const T* __restrict__ lpb, const T* __restrict__ lpl,
                                    const int* __restrict__ xlen, const int* __restrict__ ylen,
                                    T* __restrict__ alphas, T* __restrict__ betas,
                                    T* __restrict__ ll_fwd, T* __restrict__ ll_bwd,
                                    int maxT, int maxU, int do_beta) {
    lattice_body<T, 8>(lpb, lpl, xlen, ylen, alphas, betas, ll_fwd, ll_bwd, maxT, maxU, do_beta);
}

template <typename T> constexpr int LATTICE_WIDE_PF = sizeof(T) == 8 ? 2 : 4;

template <typename T>
__global__ void __launch_bounds__(1024)
rnnt_lattice_wide_kernel(const T* __restrict__ lpb, const T* __restrict__ lpl,
                         const int* __restrict__ xlen, const int* __restrict__ ylen,
                         T* __restrict__ alphas, T* __restrict__ betas,
                         T* __restrict__ ll_fwd, T* __restrict__ ll_bwd,
                         int maxT, int maxU, int do_beta) {
    lattice_body<T, LATTICE_WIDE_PF<T>>(lpb, lpl, xlen, ylen, alphas, betas, ll_fwd, ll_bwd, maxT, maxU, do_beta);
}

// ---------------------------------------------------------------------------------------------
// 2b. Viterbi alignment: the alpha wavefront with max in place of log-add, in fp64, one decision
//    byte per cell (1: emit, 0: stay; an exact tie takes stay), then a backtrace in the same CTA.
//    grid = B, blockDim.x = maxU rounded up to a warp.  The decisions live in shared memory after
//    the two delta diagonals when dec == nullptr (rows == maxT), else at dec + b*maxT*maxU and the
//    backtrace stages them `rows` rows at a time; row stride maxU.
// ---------------------------------------------------------------------------------------------
template <typename T, int PF>
__global__ void __launch_bounds__(1024) rnnt_viterbi_kernel(const T* __restrict__ lpb, const T* __restrict__ lpl,
                                    const int* __restrict__ xlen, const int* __restrict__ ylen,
                                    unsigned char* __restrict__ dec_global, int* __restrict__ frames,
                                    T* __restrict__ label_logp, T* __restrict__ score, int maxT, int maxU,
                                    int rows) {
    extern __shared__ double dsm[];
    const int W = blockDim.x;
    double* sh = dsm;                                    // [2][W] delta of the last two diagonals
    int* fr = reinterpret_cast<int*>(dsm + 2 * W);       // [W] frame of each label, from the backtrace
    int* pos = fr + W;                                   // [2] the backtrace's (t, u) between bands
    unsigned char* stage = reinterpret_cast<unsigned char*>(pos + 2);   // [rows][maxU] decision bytes
    const int b = blockIdx.x, u = threadIdx.x;
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    const long base = (long)b * maxT * maxU;
    unsigned char* dec = dec_global ? dec_global + base : stage;
    const T* pb = lpb + base;
    const T* pl = lpl + base;
    const int ND = Tn + Un - 1;
    const bool act = u < Un;
    double self = -INFINITY;                             // delta(t-1,u)
    T cb[PF], cl[PF], nb[PF], nl[PF];
#pragma unroll
    for (int i = 0; i < PF; ++i) {
        int t = i - u;
        cb[i] = (act && t >= 1 && t < Tn) ? pb[(long)(t - 1) * maxU + u] : T(0);
        cl[i] = (act && u >= 1 && t >= 0 && t < Tn) ? pl[(long)t * maxU + u - 1] : T(0);
    }
    for (int n0 = 0; n0 < ND; n0 += PF) {
#pragma unroll
        for (int i = 0; i < PF; ++i) {
            int t = n0 + PF + i - u;
            nb[i] = (act && t >= 1 && t < Tn) ? pb[(long)(t - 1) * maxU + u] : T(0);
            nl[i] = (act && u >= 1 && t >= 0 && t < Tn) ? pl[(long)t * maxU + u - 1] : T(0);
        }
#pragma unroll
        for (int i = 0; i < PF; ++i) {
            const int n = n0 + i;
            if (n < ND) {
                const int t = n - u;
                if (act && t >= 0 && t < Tn) {
                    double d = 0.0;
                    if (n > 0) {
                        const double stay = (t > 0) ? self + (double)cb[i] : -INFINITY;
                        const double emit = (u > 0) ? sh[((n - 1) & 1) * W + u - 1] + (double)cl[i] : -INFINITY;
                        const bool e = emit > stay;
                        d = e ? emit : stay;
                        dec[(long)t * maxU + u] = e;
                    }
                    self = d;
                    sh[(n & 1) * W + u] = d;
                }
            }
            __syncthreads();
        }
#pragma unroll
        for (int i = 0; i < PF; ++i) { cb[i] = nb[i]; cl[i] = nl[i]; }
    }
    if (u == 0) {
        if (Tn == 0) {
            score[b] = T(-INFINITY);
        } else {
            // self of thread 0 is delta(Tn-1, 0); the corner's delta sits in the last diagonal's buffer
            const double last = sh[((ND - 1) & 1) * W + Un - 1];
            score[b] = (T)(last + (double)pb[(long)(Tn - 1) * maxU + Un - 1]);
        }
    }
    // Backtrace by thread 0 over the decisions in shared memory.  When they are in the caller's buffer (rows < maxT),
    // the CTA first copies the band of the `rows` rows at and below the current t into shared memory, so the walk
    // makes no dependent global load; a band's rows are contiguous bytes.  t and u are the same in every thread.
    int t = Tn - 1, v = Tn > 0 ? Un - 1 : 0;
    while (v > 0) {
        const int lo = max(0, t - rows + 1);
        if (dec_global) {
            block_copy_bytes(stage, dec + (long)lo * maxU, (t - lo + 1) * maxU, u, W);
            __syncthreads();
        }
        if (u == 0) {
            while (v > 0 && t >= lo) {                   // at t == 0 only emit is possible
                if (t == 0 || stage[(t - lo) * maxU + v]) fr[--v] = t;
                else --t;
            }
            pos[0] = t;
            pos[1] = v;
        }
        __syncthreads();
        t = pos[0];
        v = pos[1];
        __syncthreads();                                 // every thread has read pos before the next band
    }
    __syncthreads();
    for (int k = u; k < maxU - 1; k += W) {
        const long o = (long)b * (maxU - 1) + k;
        if (k < Un - 1 && Tn > 0) {
            frames[o] = fr[k];
            label_logp[o] = pl[(long)fr[k] * maxU + k];
        } else {
            frames[o] = -1;
            label_logp[o] = (k < Un - 1) ? T(-INFINITY) : T(0);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 3. gradient wrt logits (gpu_rnnt_kernel.h:143-179), fused zero-fill of padded cells, upstream
//    gradient and 1/B scaling applied on the device.
// ---------------------------------------------------------------------------------------------
template <typename TO> struct Store4;
template <> struct Store4<float> {
    static __device__ __forceinline__ void st(float* p, const float (&g)[4]) {
        asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                     :: "l"(p), "f"(g[0]), "f"(g[1]), "f"(g[2]), "f"(g[3]) : "memory");
    }
};
template <> struct Store4<double> {
    static __device__ __forceinline__ void st(double* p, const double (&g)[4]) {
        reinterpret_cast<double2*>(p)[0] = make_double2(g[0], g[1]);
        reinterpret_cast<double2*>(p)[1] = make_double2(g[2], g[3]);
    }
};
template <> struct Store4<__nv_bfloat16> {
    static __device__ __forceinline__ void st(__nv_bfloat16* p, const float (&g)[4]) {
        __nv_bfloat162 a = __floats2bfloat162_rn(g[0], g[1]);
        __nv_bfloat162 b = __floats2bfloat162_rn(g[2], g[3]);
        uint2 q;
        q.x = *reinterpret_cast<uint32_t*>(&a);
        q.y = *reinterpret_cast<uint32_t*>(&b);
        *reinterpret_cast<uint2*>(p) = q;
    }
};

// FastEmit (Yu et al., ICASSP 2021): the gradient of the surrogate -log P - lambda sum sg(gamma) log p(label | t,u),
// gamma the occupancy of the emit edge, which scales the gradient along every label edge by (1 + lambda) and leaves
// the cost alone.  Per cell with a label (u < U-1) it changes two row scalars (include/edgedict_b200.h):
//   c_all = d + logaddexp(a + beta - ll, log lambda + a + beta(t,u+1) + lpl - ll),   c_lab += log1p(lambda)
// so the per-element work is unchanged.  The kernels take it as a template flag: FE = false is the plain loss's
// arithmetic, and never reads lpl.
template <typename T>
struct FastEmit {
    const T* lpl;                                         // log p(label[u] | t,u) of the loss workspace
    T log_lam, log1p_lam;
};

template <typename T, typename TO, bool VEC, int WARPS, typename TI = T, bool FE = false>
__global__ void __launch_bounds__(WARPS * 32)
rnnt_grad_kernel(const TI* logits, TO* grads, const int* __restrict__ labels,
                 const int* __restrict__ xlen, const int* __restrict__ ylen,
                 const T* __restrict__ denom, const T* __restrict__ alphas,
                 const T* __restrict__ betas, const T* __restrict__ ll_fwd,
                 const T* __restrict__ gscale, int gscale_per_batch, T hscale,
                 int B, int maxT, int maxU, int V, int blank, FastEmit<T> fe) {
    const int lane = threadIdx.x & 31;
    const long ncells = (long)B * maxT * maxU;
    const long wstride = (long)gridDim.x * WARPS;
    for (long cell = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); cell < ncells; cell += wstride) {
        const int u = (int)(cell % maxU);
        const long bt = cell / maxU;
        const int t = (int)(bt % maxT);
        const int b = (int)(bt / maxT);
        const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
        const TI* row = logits + cell * (long)V;
        TO* orow = grads + cell * (long)V;
        if (t >= Tn || u >= Un) {                         // padded: zero, logits never read
            for (int v = lane * 4; v < V; v += 128) {
                if (VEC) {
                    const T z[4] = {0, 0, 0, 0};
                    Store4<TO>::st(orow + v, z);
                } else {
                    for (int i = 0; i < 4 && v + i < V; ++i) orow[v + i] = TO(T(0));
                }
            }
            continue;
        }
        const T sc = hscale * (gscale ? gscale[gscale_per_batch ? b : 0] : T(1));
        const T a = alphas[cell], bt_ = betas[cell], ll = ll_fwd[b], d = denom[cell];
        const int lab = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
        // scalar pieces shared by the row
        T c_all = a + bt_ - ll + d;                       // exp(c_all + x_v) = exp(a+b+logp-ll)
        T c_blank = M<T>::ninf();                         // log-factor subtracted at v == blank
        if (t < Tn - 1) c_blank = a - ll + d + betas[cell + maxU];
        else if (u == Un - 1) c_blank = a - ll + d;
        T c_lab = (lab >= 0) ? a - ll + d + betas[cell + 1] : M<T>::ninf();
        if (FE && lab >= 0) {
            c_all = d + lse2(a + bt_ - ll, fe.log_lam + a + betas[cell + 1] + fe.lpl[cell] - ll);
            c_lab += fe.log1p_lam;
        }
        for (int v = lane * 4; v < V; v += 128) {
            T x[4];
            Row4<TI, VEC>::load(row, v, V, x);
            T g[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                T gr = M<T>::exp_fast(c_all + x[i]);
                if (v + i == blank) gr -= M<T>::exp_acc(c_blank + x[i]);
                if (v + i == lab) gr -= M<T>::exp_acc(c_lab + x[i]);
                g[i] = gr * sc;
            }
            if (VEC) {
                Store4<TO>::st(orow + v, g);
            } else {
                for (int i = 0; i < 4 && v + i < V; ++i) orow[v + i] = TO(g[i]);
            }
        }
    }
}

// bf16 logits -> bf16 gradients (in place allowed), the fused-joint path: 8 values per lane and iteration (one 16-byte
// load, one 16-byte store); the rare blank / label corrections are applied outside the unrolled exponentials.  Same
// arithmetic as rnnt_grad_kernel (gpu_rnnt_kernel.h:143-179).  GradRow holds what a cell's row shares, grad_bf16x8
// turns 8 logits of it into 8 gradients: the kernel below and rnnt_grad_db_bf16x8_kernel share both, so their d logits
// are the same bits.
struct GradRow {
    float c2, c_blank, c_lab, sc;
    int lab;
    bool pad;                                             // padded cell: zero gradient, logits never read
};

__device__ __forceinline__ void cell_btu(long cell, int maxT, int maxU, int& b, int& t, int& u) {
    u = (int)(cell % maxU);
    const long bt = cell / maxU;
    t = (int)(bt % maxT);
    b = (int)(bt / maxT);
}

// What the row of cell (b, t, u) reads from the workspace, given its clamped lengths Tn, Un.  The loads are kept
// apart from the arithmetic (grad_row) so that a thread can issue those of several cells before it waits for any.
struct GradLoads {
    float a, bt_, ll, d, gs, b_next, b_lab, lpl;
    int lab;
};

template <bool FE>
__device__ __forceinline__ GradLoads grad_loads(long cell, int b, int t, int u, int Tn, int Un,
                                                const int* __restrict__ labels, const float* __restrict__ denom,
                                                const float* __restrict__ alphas, const float* __restrict__ betas,
                                                const float* __restrict__ ll_fwd, const float* __restrict__ gscale,
                                                int gscale_per_batch, int maxU, const FastEmit<float>& fe) {
    GradLoads l;
    l.gs = gscale ? gscale[gscale_per_batch ? b : 0] : 1.f;
    l.a = alphas[cell]; l.bt_ = betas[cell]; l.ll = ll_fwd[b]; l.d = denom[cell];
    l.lab = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
    l.b_next = (t < Tn - 1) ? betas[cell + maxU] : 0.f;
    l.b_lab = (u < Un - 1) ? betas[cell + 1] : 0.f;
    l.lpl = (FE && u < Un - 1) ? fe.lpl[cell] : 0.f;
    return l;
}

template <bool FE>
__device__ __forceinline__ GradRow grad_row(const GradLoads& l, int t, int u, int Tn, int Un, float hscale,
                                            const FastEmit<float>& fe) {
    GradRow r;
    r.pad = t >= Tn || u >= Un;
    r.sc = hscale * l.gs;
    r.lab = l.lab;
    float c_all = l.a + l.bt_ - l.ll + l.d;
    r.c_blank = -INFINITY;
    if (t < Tn - 1) r.c_blank = l.a - l.ll + l.d + l.b_next;
    else if (u == Un - 1) r.c_blank = l.a - l.ll + l.d;
    r.c_lab = (r.lab >= 0) ? l.a - l.ll + l.d + l.b_lab : -INFINITY;
    if (FE && r.lab >= 0) {                               // the same arithmetic as rnnt_grad_kernel's FastEmit branch
        c_all = l.d + lse2(l.a + l.bt_ - l.ll, fe.log_lam + l.a + l.b_lab + l.lpl - l.ll);
        r.c_lab += fe.log1p_lam;
    }
    constexpr float LOG2E = 1.4426950408889634f;
    r.c2 = c_all * LOG2E;
    return r;
}

// the gradients of the 8 bf16 logits q at columns v .. v+7 of a valid cell, packed as bf16
__device__ __forceinline__ uint4 grad_bf16x8(uint4 q, int v, const GradRow& r, int blank) {
    constexpr float LOG2E = 1.4426950408889634f;
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    float x[8], g[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
        x[2 * i] = f.x; x[2 * i + 1] = f.y;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = fast_ex2(fmaf(x[i], LOG2E, r.c2));
    const unsigned ib = (unsigned)(blank - v), il = (unsigned)(r.lab - v);
    if (ib < 8u || il < 8u) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if ((unsigned)i == ib) g[i] -= expf(r.c_blank + x[i]);
            if ((unsigned)i == il) g[i] -= expf(r.c_lab + x[i]);
        }
    }
    uint32_t ow[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        __nv_bfloat162 pk = __floats2bfloat162_rn(g[2 * i] * r.sc, g[2 * i + 1] * r.sc);
        ow[i] = *reinterpret_cast<uint32_t*>(&pk);
    }
    return make_uint4(ow[0], ow[1], ow[2], ow[3]);
}

template <int WARPS, bool FE>
__global__ void __launch_bounds__(WARPS * 32)
rnnt_grad_bf16x8_kernel(const __nv_bfloat16* logits, __nv_bfloat16* grads, const int* __restrict__ labels,
                        const int* __restrict__ xlen, const int* __restrict__ ylen, const float* __restrict__ denom,
                        const float* __restrict__ alphas, const float* __restrict__ betas,
                        const float* __restrict__ ll_fwd, const float* __restrict__ gscale, int gscale_per_batch,
                        float hscale, int B, int maxT, int maxU, int V, int blank, FastEmit<float> fe) {
    const int lane = threadIdx.x & 31;
    const long ncells = (long)B * maxT * maxU;
    const long wstride = (long)gridDim.x * WARPS;
    for (long cell = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); cell < ncells; cell += wstride) {
        int b, t, u;
        cell_btu(cell, maxT, maxU, b, t, u);
        const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
        const bool pad = t >= Tn || u >= Un;
        const GradRow r = grad_row<FE>(pad ? GradLoads{} : grad_loads<FE>(cell, b, t, u, Tn, Un, labels, denom, alphas,
                                                                          betas, ll_fwd, gscale, gscale_per_batch, maxU,
                                                                          fe),
                                       t, u, Tn, Un, hscale, fe);
        const __nv_bfloat16* row = logits + cell * (long)V;
        __nv_bfloat16* orow = grads + cell * (long)V;
        if (r.pad) {
            for (int v = lane * 8; v < V; v += 256) *reinterpret_cast<uint4*>(orow + v) = make_uint4(0u, 0u, 0u, 0u);
            continue;
        }
        // logits and grads may be the same buffer: all four 16-byte loads of a group are issued before the first
        // store, otherwise the possible aliasing serialises load -> store -> load and one row costs four DRAM
        // round trips
        for (int v0 = lane * 8; v0 < V; v0 += 1024) {
            uint4 qq[4];
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (v0 + k * 256 < V) qq[k] = *reinterpret_cast<const uint4*>(row + v0 + k * 256);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int v = v0 + k * 256;
                if (v >= V) break;
                *reinterpret_cast<uint4*>(orow + v) = grad_bf16x8(qq[k], v, r, blank);
            }
        }
    }
}

// The same d logits, and the bias gradient db[c] += sum over rows of the bf16 d logits in eb_colsum's order
// (COLSUM_LANES, common.cuh), without a second pass over them.  Thread (k, q) owns row lane k and the 8 columns
// v = 8q .. 8q+7: it walks the cells k, k + COLSUM_LANES, ... in order, adding each bf16 gradient it stores (the zeros
// of padded cells included) to its own fp32 accumulators, so each (lane, column) sum receives exactly eb_colsum's rows
// in eb_colsum's order.  The lane sums go to part[k * V + v], and colsum_lanes_finish adds them with eb_colsum's tree.
// That leaves COLSUM_LANES * V / 8 threads (16 warps per SM at V = 1024 on 132 SMs), so each thread keeps the loads
// of DB_ROWS cells in flight; as in rnnt_grad_bf16x8_kernel, all of them are issued before the first store.
constexpr int DB_THREADS = 128, DB_ROWS = 4;
template <bool FE>
__global__ void __launch_bounds__(DB_THREADS, 4)
rnnt_grad_db_bf16x8_kernel(const __nv_bfloat16* logits, __nv_bfloat16* grads, const int* __restrict__ labels,
                           const int* __restrict__ xlen, const int* __restrict__ ylen, const float* __restrict__ denom,
                           const float* __restrict__ alphas, const float* __restrict__ betas,
                           const float* __restrict__ ll_fwd, const float* __restrict__ gscale, int gscale_per_batch,
                           float hscale, int B, int maxT, int maxU, int V, int blank, float* __restrict__ part,
                           FastEmit<float> fe) {
    const int V8 = V / 8;
    const int tid = blockIdx.x * DB_THREADS + threadIdx.x;
    if (tid >= COLSUM_LANES * V8) return;
    const int k = tid / V8, v = (tid - k * V8) * 8;
    const long ncells = (long)B * maxT * maxU;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long c0 = k; c0 < ncells; c0 += (long)DB_ROWS * COLSUM_LANES) {
        // the lengths of all DB_ROWS cells first, then their rows and logits: one dependent round trip per group
        int bi[DB_ROWS], ti[DB_ROWS], ui[DB_ROWS], Tn[DB_ROWS], Un[DB_ROWS];
#pragma unroll
        for (int i = 0; i < DB_ROWS; ++i) {
            const long cell = c0 + (long)i * COLSUM_LANES;
            cell_btu(cell < ncells ? cell : ncells - 1, maxT, maxU, bi[i], ti[i], ui[i]);
            Tn[i] = clamp_T(xlen[bi[i]], maxT);
            Un[i] = cell < ncells ? clamp_U(ylen[bi[i]], maxU) : 0;          // (a cell past the end: padded)
        }
        GradLoads l[DB_ROWS];
        uint4 q[DB_ROWS];
#pragma unroll
        for (int i = 0; i < DB_ROWS; ++i) {
            const long cell = c0 + (long)i * COLSUM_LANES;
            const long cl = cell < ncells ? cell : ncells - 1;
            l[i] = grad_loads<FE>(cl, bi[i], ti[i], ui[i], Tn[i], Un[i], labels, denom, alphas, betas, ll_fwd, gscale,
                                  gscale_per_batch, maxU, fe);
            if (ti[i] < Tn[i] && ui[i] < Un[i]) q[i] = *reinterpret_cast<const uint4*>(logits + cell * (long)V + v);
        }
#pragma unroll
        for (int i = 0; i < DB_ROWS; ++i) {
            const long cell = c0 + (long)i * COLSUM_LANES;
            if (cell >= ncells) break;
            const GradRow r = grad_row<FE>(l[i], ti[i], ui[i], Tn[i], Un[i], hscale, fe);
            const uint4 g = r.pad ? make_uint4(0u, 0u, 0u, 0u) : grad_bf16x8(q[i], v, r, blank);
            *reinterpret_cast<uint4*>(grads + cell * (long)V + v) = g;
            const uint32_t w[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[j]));
                acc[2 * j] += f.x;
                acc[2 * j + 1] += f.y;
            }
        }
    }
    float* o = part + (long)k * V + v;
    *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

template <typename T>
struct Workspace {
    T *denom, *lpb, *lpl, *alphas, *betas, *ll_fwd, *ll_bwd;
    static size_t bytes(int B, int maxT, int maxU) {
        return sizeof(T) * ((size_t)B * maxT * maxU * 5 + 2 * (size_t)B);
    }
    Workspace(void* ws, int B, int maxT, int maxU) {
        const size_t n = (size_t)B * maxT * maxU;
        T* p = reinterpret_cast<T*>(ws);
        denom = p; lpb = p + n; lpl = p + 2 * n; alphas = p + 3 * n; betas = p + 4 * n;
        ll_fwd = p + 5 * n; ll_bwd = ll_fwd + B;
    }
};

// alpha / beta launch: the PF = 8 kernel when its register count lets a block of maxU threads (rounded up to a warp)
// launch, else the wide one.  The limit comes from the compiled kernel, queried once per device.
template <typename T>
int launch_lattice(const Workspace<T>& w, const int* xlen, const int* ylen, int B, int maxT, int maxU, int need_beta,
                   cudaStream_t st) {
    // per device, each slot written once with the value any racing writer also computes
    static std::atomic<int> cache[64];
    int dev;
    EB_CUDA(cudaGetDevice(&dev));
    int narrow_max = dev < 64 ? cache[dev].load(std::memory_order_relaxed) : 0;
    if (!narrow_max) {
        cudaFuncAttributes a;
        EB_CUDA(cudaFuncGetAttributes(&a, rnnt_lattice_kernel<T>));
        narrow_max = a.maxThreadsPerBlock;
        if (dev < 64) cache[dev].store(narrow_max, std::memory_order_relaxed);
    }
    const int threads = ((maxU + 31) / 32) * 32;
    const size_t smem = 2 * threads * sizeof(T);
    if (threads <= narrow_max)
        rnnt_lattice_kernel<T><<<dim3(B, 2), threads, smem, st>>>(w.lpb, w.lpl, xlen, ylen, w.alphas, w.betas,
                                                                  w.ll_fwd, w.ll_bwd, maxT, maxU, need_beta);
    else
        rnnt_lattice_wide_kernel<T><<<dim3(B, 2), threads, smem, st>>>(w.lpb, w.lpl, xlen, ylen, w.alphas, w.betas,
                                                                       w.ll_fwd, w.ll_bwd, maxT, maxU, need_beta);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

inline int row_grid(long ncells, int warps) {
    long blocks = (ncells + warps - 1) / warps;
    long cap = (long)eb_num_sms() * 16;                  // grid-stride above 16 CTAs/SM
    return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

// The problem description every loss entry validates before it launches anything: the kernels dereference the
// lengths (and the labels, for maxU > 1) on the device, and a blank outside [0, V) would silently skip its term.
inline bool bad_problem(const int* labels, const int* xlen, const int* ylen, int B, int maxT, int maxU, int V,
                        int blank) {
    return (!labels && maxU > 1) || !xlen || !ylen || B <= 0 || maxT <= 0 || maxU <= 0 || V <= 0 || blank < 0 ||
           blank >= V || maxU > 1024;
}

// fastemit_lambda must be a finite lambda >= 0 (NaN fails the comparison)
inline bool bad_lambda(double lam) { return !(lam >= 0.0) || !std::isfinite(lam); }

// f(std::true_type) for lambda > 0, the FastEmit instantiation of a gradient kernel; f(std::false_type) at lambda = 0,
// the plain loss's kernel, which runs the same instructions as before FastEmit existed.
template <typename T, typename F>
void with_fastemit(const T* lpl, double lam, F&& f) {
    if (lam > 0.0) f(std::true_type{}, FastEmit<T>{lpl, (T)std::log(lam), (T)std::log1p(lam)});
    else f(std::false_type{}, FastEmit<T>{nullptr, T(0), T(0)});
}

template <typename T>
int loss_fwd(const T* logits, const int* labels, const int* xlen, const int* ylen, int B, int maxT,
             int maxU, int V, int blank, void* ws, int need_beta, cudaStream_t st) {
    if (!logits || !ws || bad_problem(labels, xlen, ylen, B, maxT, maxU, V, blank)) return EB_ERR_INVALID;
    Workspace<T> w(ws, B, maxT, maxU);
    const long ncells = (long)B * maxT * maxU;
    constexpr int WARPS = 8;
    const bool vec = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
    if (vec)
        rnnt_denom_kernel<T, true, WARPS><<<row_grid(ncells, WARPS), WARPS * 32, 0, st>>>(
            logits, labels, xlen, ylen, w.denom, w.lpb, w.lpl, B, maxT, maxU, V, blank);
    else
        rnnt_denom_kernel<T, false, WARPS><<<row_grid(ncells, WARPS), WARPS * 32, 0, st>>>(
            logits, labels, xlen, ylen, w.denom, w.lpb, w.lpl, B, maxT, maxU, V, blank);
    EB_CHECK_LAUNCH();
    return launch_lattice<T>(w, xlen, ylen, B, maxT, maxU, need_beta, st);
}

template <typename T, typename TO>
int loss_bwd(const T* logits, TO* grads, const int* labels, const int* xlen, const int* ylen, int B,
             int maxT, int maxU, int V, int blank, void* ws, const T* gscale, int per_batch,
             T hscale, double lam, cudaStream_t st) {
    if (!logits || !grads || !ws || bad_problem(labels, xlen, ylen, B, maxT, maxU, V, blank) || bad_lambda(lam))
        return EB_ERR_INVALID;
    Workspace<T> w(ws, B, maxT, maxU);
    const long ncells = (long)B * maxT * maxU;
    constexpr int WARPS = 8;
    const bool vec = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(grads) & 15) == 0);
    with_fastemit(w.lpl, lam, [&](auto fe_on, const FastEmit<T>& fe) {
        constexpr bool FE = decltype(fe_on)::value;
        if (vec)
            rnnt_grad_kernel<T, TO, true, WARPS, T, FE><<<row_grid(ncells, WARPS), WARPS * 32, 0, st>>>(
                logits, grads, labels, xlen, ylen, w.denom, w.alphas, w.betas, w.ll_fwd, gscale,
                per_batch, hscale, B, maxT, maxU, V, blank, fe);
        else
            rnnt_grad_kernel<T, TO, false, WARPS, T, FE><<<row_grid(ncells, WARPS), WARPS * 32, 0, st>>>(
                logits, grads, labels, xlen, ylen, w.denom, w.alphas, w.betas, w.ll_fwd, gscale,
                per_batch, hscale, B, maxT, maxU, V, blank, fe);
    });
    EB_CHECK_LAUNCH();
    return EB_OK;
}

template <typename T>
__global__ void neg_copy_kernel(const T* ll, T* costs, int B) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) costs[i] = -ll[i];
}

template <typename T>
rnntStatus_t compat_entry(const T* acts, T* grads, const int* labels, const int* label_lengths,
                          const int* input_lengths, int V, int B, T* costs, void* workspace,
                          rnntOptions o) {
    // argument validation mirrors src/rnnt_entrypoint.cpp:49-59
    if (!acts || (!labels && o.maxU > 1) || !label_lengths || !input_lengths || !costs || !workspace || V <= 0 ||
        B <= 0 || o.maxT <= 0 || o.maxU <= 0)
        return RNNT_STATUS_INVALID_VALUE;
    if (o.loc != RNNT_GPU) {
        // The reference prints a diagnostic when the requested location is not compiled in
        // (rnnt_entrypoint.cpp:86-88).  This library is GPU-only by design: no CPU fallback.
        fprintf(stderr, "CPU execution requested, but edgedict_b200 is a GPU-only (sm_90a) build\n");
        return RNNT_STATUS_EXECUTION_FAILED;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(o.stream);
    int rc = loss_fwd<T>(acts, labels, input_lengths, label_lengths, B, o.maxT, o.maxU, V,
                         o.blank_label, workspace, grads != nullptr, st);
    if (rc == EB_ERR_INVALID) return RNNT_STATUS_INVALID_VALUE;
    if (rc != EB_OK) return RNNT_STATUS_EXECUTION_FAILED;
    if (grads) {
        rc = loss_bwd<T, T>(acts, grads, labels, input_lengths, label_lengths, B, o.maxT, o.maxU, V,
                            o.blank_label, workspace, nullptr, 0, T(1), 0.0, st);
        if (rc != EB_OK) return RNNT_STATUS_EXECUTION_FAILED;
    }
    Workspace<T> w(workspace, B, o.maxT, o.maxU);
    if (cudaMemcpyAsync(costs, w.ll_fwd, sizeof(T) * B, cudaMemcpyDeviceToHost, st) != cudaSuccess)
        return RNNT_STATUS_MEMOPS_FAILED;
    if (cudaStreamSynchronize(st) != cudaSuccess) return RNNT_STATUS_EXECUTION_FAILED;
    for (int i = 0; i < B; ++i) costs[i] = -costs[i];   // gpu_rnnt.h:209-213
    return RNNT_STATUS_SUCCESS;
}

// ---------------------------------------------------------------------------------------------
// 4. Pruned RNN-T (include/edgedict_b200.h, eb_rnnt_band_loss_fwd): band rows m = (b*maxT + t)*R + r hold the
//    logits of cell (b, t, u = s_begin[b,t] + r) for r < Rb = min(R, U_b).  The statistics of a band row go to that
//    cell of a full [B, maxT, maxU] workspace (the same bits rnnt_denom_kernel writes for the same logits), every other
//    valid cell gets -inf, and the unchanged lattice runs on it.  The gradient of a band row is rnnt_grad_kernel's.
// ---------------------------------------------------------------------------------------------
struct Band {
    const int* s_begin;                                   // [B, maxT]
    const int* nopath;                                    // [B]: 1 when the bands hold no path (cost +inf)
    int R;
};

// the cell of band row m, or false for a padding row (band_row_live, or an utterance without a band path)
__device__ __forceinline__ bool band_cell(long m, const Band& bd, const int* xlen, const int* ylen, int maxT, int maxU,
                                          int& b, int& t, int& u, int& Tn, int& Un) {
    const int r = (int)(m % bd.R);
    const long bt = m / bd.R;
    t = (int)(bt % maxT);
    b = (int)(bt / maxT);
    Tn = clamp_T(xlen[b], maxT);
    Un = clamp_U(ylen[b], maxU);
    if (t >= Tn || r >= min(bd.R, Un) || bd.nopath[b]) return false;
    const int s = bd.s_begin[bt];
    u = s + r;
    return band_row_live(t, Tn, Un, bd.R, s, r);
}

template <bool VEC, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
rnnt_band_denom_kernel(const float* __restrict__ logits, const int* __restrict__ labels,
                       const int* __restrict__ xlen, const int* __restrict__ ylen, Band bd,
                       float* __restrict__ denom, float* __restrict__ lpb, float* __restrict__ lpl,
                       int B, int maxT, int maxU, int V, int blank) {
    const int lane = threadIdx.x & 31;
    const long nrows = (long)B * maxT * bd.R;
    const long wstride = (long)gridDim.x * WARPS;
    for (long m = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); m < nrows; m += wstride) {
        int b, t, u, Tn, Un;
        if (!band_cell(m, bd, xlen, ylen, maxT, maxU, b, t, u, Tn, Un)) continue;
        const long cell = ((long)b * maxT + t) * maxU + u;
        const int lab = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
        float d, xb, xl;
        denom_row<float, VEC>(logits + m * (long)V, lane, V, blank, lab, d, xb, xl);
        if (lane == 0) {
            denom[cell] = d;
            lpb[cell] = d + xb;
            lpl[cell] = d + xl;
        }
    }
}

// -inf statistics for the valid cells that no live band row holds (all of them when the bands hold no path, and every
// cell of a frame whose start is negative)
__global__ void rnnt_band_fill_kernel(const int* __restrict__ xlen, const int* __restrict__ ylen, Band bd,
                                      float* __restrict__ denom, float* __restrict__ lpb, float* __restrict__ lpl,
                                      int B, int maxT, int maxU) {
    const long ncells = (long)B * maxT * maxU;
    for (long cell = (long)blockIdx.x * blockDim.x + threadIdx.x; cell < ncells; cell += (long)gridDim.x * blockDim.x) {
        int b, t, u;
        cell_btu(cell, maxT, maxU, b, t, u);
        const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
        if (t >= Tn || u >= Un) continue;
        const int s = bd.s_begin[(long)b * maxT + t];
        if (bd.nopath[b] || u < s || !band_row_live(t, Tn, Un, bd.R, s, u - s)) {
            denom[cell] = -INFINITY;
            lpb[cell] = -INFINITY;
            lpl[cell] = -INFINITY;
        }
    }
}

// rnnt_grad_kernel (FE = false) on band rows: the row scalars of cell (t, s_begin + r), zero on padding rows
template <typename TO, bool VEC, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
rnnt_band_grad_kernel(const float* logits, TO* grads, const int* __restrict__ labels,
                      const int* __restrict__ xlen, const int* __restrict__ ylen, Band bd,
                      const float* __restrict__ denom, const float* __restrict__ alphas,
                      const float* __restrict__ betas, const float* __restrict__ ll_fwd,
                      const float* __restrict__ gscale, int gscale_per_batch, float hscale,
                      int B, int maxT, int maxU, int V, int blank) {
    const int lane = threadIdx.x & 31;
    const long nrows = (long)B * maxT * bd.R;
    const long wstride = (long)gridDim.x * WARPS;
    for (long m = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); m < nrows; m += wstride) {
        int b, t, u, Tn, Un;
        const float* row = logits + m * (long)V;
        TO* orow = grads + m * (long)V;
        if (!band_cell(m, bd, xlen, ylen, maxT, maxU, b, t, u, Tn, Un)) {
            for (int v = lane * 4; v < V; v += 128) {
                if (VEC) {
                    const float z[4] = {0, 0, 0, 0};
                    Store4<TO>::st(orow + v, z);
                } else {
                    for (int i = 0; i < 4 && v + i < V; ++i) orow[v + i] = TO(0.f);
                }
            }
            continue;
        }
        const long cell = ((long)b * maxT + t) * maxU + u;
        const float sc = hscale * (gscale ? gscale[gscale_per_batch ? b : 0] : 1.f);
        const float a = alphas[cell], bt_ = betas[cell], ll = ll_fwd[b], d = denom[cell];
        const int lab = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
        const float c_all = a + bt_ - ll + d;
        float c_blank = -INFINITY;
        if (t < Tn - 1) c_blank = a - ll + d + betas[cell + maxU];
        else if (u == Un - 1) c_blank = a - ll + d;
        const float c_lab = (lab >= 0) ? a - ll + d + betas[cell + 1] : -INFINITY;
        for (int v = lane * 4; v < V; v += 128) {
            float x[4];
            Row4<float, VEC>::load(row, v, V, x);
            float g[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float gr = fast_exp(c_all + x[i]);
                if (v + i == blank) gr -= expf(c_blank + x[i]);
                if (v + i == lab) gr -= expf(c_lab + x[i]);
                g[i] = gr * sc;
            }
            if (VEC) {
                Store4<TO>::st(orow + v, g);
            } else {
                for (int i = 0; i < 4 && v + i < V; ++i) orow[v + i] = TO(g[i]);
            }
        }
    }
}

// rnnt_grad_db_bf16x8_kernel over band rows: the same row scalars (grad_loads / grad_row) and d logits (grad_bf16x8)
// at the band row's cell, zero on padding rows, and the bias gradient's lane sums over the band rows in eb_colsum's
// order.  Thread (k, q) walks the rows k, k + COLSUM_LANES, ... for the 8 columns 8q .. 8q+7.
__global__ void __launch_bounds__(DB_THREADS)
rnnt_band_grad_db_bf16x8_kernel(const __nv_bfloat16* logits, __nv_bfloat16* grads, const int* __restrict__ labels,
                                const int* __restrict__ xlen, const int* __restrict__ ylen, Band bd,
                                const float* __restrict__ denom, const float* __restrict__ alphas,
                                const float* __restrict__ betas, const float* __restrict__ ll_fwd,
                                const float* __restrict__ gscale, int gscale_per_batch, float hscale, int B, int maxT,
                                int maxU, int V, int blank, float* __restrict__ part) {
    const int V8 = V / 8;
    const int tid = blockIdx.x * DB_THREADS + threadIdx.x;
    if (tid >= COLSUM_LANES * V8) return;
    const int k = tid / V8, v = (tid - k * V8) * 8;
    const long nrows = (long)B * maxT * bd.R;
    const FastEmit<float> fe{nullptr, 0.f, 0.f};
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long m = k; m < nrows; m += COLSUM_LANES) {
        int b, t, u, Tn, Un;
        uint4 g = make_uint4(0u, 0u, 0u, 0u);
        if (band_cell(m, bd, xlen, ylen, maxT, maxU, b, t, u, Tn, Un)) {
            const long cell = ((long)b * maxT + t) * maxU + u;
            const GradRow r = grad_row<false>(grad_loads<false>(cell, b, t, u, Tn, Un, labels, denom, alphas, betas,
                                                                ll_fwd, gscale, gscale_per_batch, maxU, fe),
                                              t, u, Tn, Un, hscale, fe);
            g = grad_bf16x8(*reinterpret_cast<const uint4*>(logits + m * (long)V + v), v, r, blank);
        }
        *reinterpret_cast<uint4*>(grads + m * (long)V + v) = g;
        const uint32_t w[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[j]));
            acc[2 * j] += f.x;
            acc[2 * j + 1] += f.y;
        }
    }
    float* o = part + (long)k * V + v;
    *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// what every band entry checks before it launches anything
inline bool bad_band(const int* s_begin, const int* nopath, int R) {
    return !s_begin || !nopath || R < 2 || R > 64;
}

}  // namespace

// ------------------------------ warp-transducer compatible C ABI ------------------------------
extern "C" {

__attribute__((visibility("default"))) int get_warprnnt_version() { return 1; }

__attribute__((visibility("default"))) const char* rnntGetStatusString(rnntStatus_t status) {
    switch (status) {
        case RNNT_STATUS_SUCCESS: return "no error";
        case RNNT_STATUS_MEMOPS_FAILED: return "cuda memcpy or memset failed";
        case RNNT_STATUS_INVALID_VALUE: return "invalid value";
        case RNNT_STATUS_EXECUTION_FAILED: return "execution failed";
        default: return "unknown error";
    }
}

__attribute__((visibility("default"))) rnntStatus_t
compute_rnnt_loss(const float* const activations, float* gradients, const int* const flat_labels,
                  const int* const label_lengths, const int* const input_lengths, int alphabet_size,
                  int minibatch, float* costs, void* workspace, rnntOptions options) {
    return compat_entry<float>(activations, gradients, flat_labels, label_lengths, input_lengths,
                               alphabet_size, minibatch, costs, workspace, options);
}

__attribute__((visibility("default"))) rnntStatus_t
compute_rnnt_loss_fp64(const double* const activations, double* gradients,
                       const int* const flat_labels, const int* const label_lengths,
                       const int* const input_lengths, int alphabet_size, int minibatch,
                       double* costs, void* workspace, rnntOptions options) {
    return compat_entry<double>(activations, gradients, flat_labels, label_lengths, input_lengths,
                                alphabet_size, minibatch, costs, workspace, options);
}

__attribute__((visibility("default"))) rnntStatus_t
get_workspace_size(int maxT, int maxU, int minibatch, bool gpu, size_t* size_bytes,
                   size_t dtype_size) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0 || !size_bytes) return RNNT_STATUS_INVALID_VALUE;
    (void)gpu;  // only the GPU location exists in this build; same size either way
    *size_bytes = dtype_size * ((size_t)minibatch * maxT * maxU * 5 + 2 * (size_t)minibatch);
    return RNNT_STATUS_SUCCESS;
}

}  // extern "C"

// ------------------------------ device-resident (no host sync) ABI ----------------------------
EB_API size_t eb_rnnt_workspace_bytes(int B, int maxT, int maxU, int dtype_size) {
    return (size_t)dtype_size * ((size_t)B * maxT * maxU * 5 + 2 * (size_t)B);
}

EB_API int eb_rnnt_loss_fwd(const void* logits, const int* labels, const int* xlen, const int* ylen,
                            int B, int maxT, int maxU, int V, int blank, int dtype_size,
                            void* workspace, void* costs_dev, int need_beta, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc;
    if (dtype_size == 4) {
        rc = loss_fwd<float>((const float*)logits, labels, xlen, ylen, B, maxT, maxU, V, blank,
                             workspace, need_beta, st);
        if (rc) return rc;
        if (costs_dev) {
            Workspace<float> w(workspace, B, maxT, maxU);
            neg_copy_kernel<float><<<(B + 127) / 128, 128, 0, st>>>(w.ll_fwd, (float*)costs_dev, B);
        }
    } else if (dtype_size == 8) {
        rc = loss_fwd<double>((const double*)logits, labels, xlen, ylen, B, maxT, maxU, V, blank,
                              workspace, need_beta, st);
        if (rc) return rc;
        if (costs_dev) {
            Workspace<double> w(workspace, B, maxT, maxU);
            neg_copy_kernel<double><<<(B + 127) / 128, 128, 0, st>>>(w.ll_fwd, (double*)costs_dev, B);
        }
    } else {
        return EB_ERR_INVALID;
    }
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_rnnt_loss_bwd_fe(const void* logits, void* grads, int grads_bf16, const int* labels,
                               const int* xlen, const int* ylen, int B, int maxT, int maxU, int V,
                               int blank, int dtype_size, void* workspace, const void* gscale_dev,
                               int gscale_per_batch, double host_scale, double fastemit_lambda, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (dtype_size == 4) {
        if (grads_bf16)
            return loss_bwd<float, __nv_bfloat16>((const float*)logits, (__nv_bfloat16*)grads, labels,
                                                  xlen, ylen, B, maxT, maxU, V, blank, workspace,
                                                  (const float*)gscale_dev, gscale_per_batch,
                                                  (float)host_scale, fastemit_lambda, st);
        return loss_bwd<float, float>((const float*)logits, (float*)grads, labels, xlen, ylen, B, maxT,
                                      maxU, V, blank, workspace, (const float*)gscale_dev,
                                      gscale_per_batch, (float)host_scale, fastemit_lambda, st);
    }
    if (dtype_size == 8 && !grads_bf16)
        return loss_bwd<double, double>((const double*)logits, (double*)grads, labels, xlen, ylen, B,
                                        maxT, maxU, V, blank, workspace, (const double*)gscale_dev,
                                        gscale_per_batch, host_scale, fastemit_lambda, st);
    return EB_ERR_INVALID;
}

EB_API int eb_rnnt_loss_bwd(const void* logits, void* grads, int grads_bf16, const int* labels,
                            const int* xlen, const int* ylen, int B, int maxT, int maxU, int V,
                            int blank, int dtype_size, void* workspace, const void* gscale_dev,
                            int gscale_per_batch, double host_scale, void* stream) {
    return eb_rnnt_loss_bwd_fe(logits, grads, grads_bf16, labels, xlen, ylen, B, maxT, maxU, V, blank, dtype_size,
                               workspace, gscale_dev, gscale_per_batch, host_scale, 0.0, stream);
}

// Lattice only: denom / lpb / lpl of the workspace were already produced by eb_joint_logits_lse.
EB_API int eb_rnnt_loss_lattice(const int* xlen, const int* ylen, int B, int maxT, int maxU, void* workspace,
                                float* costs_dev, int need_beta, void* stream) {
    if (!xlen || !ylen || !workspace || B <= 0 || maxT <= 0 || maxU <= 0 || maxU > 1024) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Workspace<float> w(workspace, B, maxT, maxU);
    const int rc = launch_lattice<float>(w, xlen, ylen, B, maxT, maxU, need_beta, st);
    if (rc) return rc;
    if (costs_dev) neg_copy_kernel<float><<<(B + 127) / 128, 128, 0, st>>>(w.ll_fwd, costs_dev, B);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

namespace {

constexpr size_t ALIGN_SMEM_MAX = 227 * 1024;           // opt-in dynamic shared memory per CTA on sm_90
// frames of the prefetch ring: 1024 threads leave 64 registers each, which eight fp64 pairs in flight would overrun
template <typename T> constexpr int VITERBI_PF = sizeof(T) == 8 ? 4 : 8;

// rows of decisions the backtrace stages at a time when they do not all fit in shared memory
constexpr size_t ALIGN_STAGE_BYTES = 64 * 1024;

// dynamic shared memory of rnnt_viterbi_kernel: delta [2][W] doubles, frames [W] ints, (t, u) and [rows][maxU] decision
// bytes: all maxT rows when they fit (the decisions then live there), else a staging band of the caller's buffer.  The
// kernel has no static shared memory, so the whole opt-in limit is available to this buffer.
inline size_t viterbi_smem(int maxT, int maxU, int* rows) {
    const size_t W = ((size_t)maxU + 31) / 32 * 32;
    const size_t fixed = W * (2 * sizeof(double) + sizeof(int)) + 2 * sizeof(int);
    *rows = fixed + (size_t)maxT * maxU <= ALIGN_SMEM_MAX ? maxT : (int)(ALIGN_STAGE_BYTES / maxU);
    return fixed + (size_t)*rows * maxU;
}

template <typename T>
int viterbi(const int* xlen, const int* ylen, int B, int maxT, int maxU, void* ws, unsigned char* decisions,
            int* frames, void* label_logp, void* score, cudaStream_t st) {
    int rows;
    const size_t smem = viterbi_smem(maxT, maxU, &rows);
    const bool in_smem = rows == maxT;
    if (!in_smem && !decisions) return EB_ERR_INVALID;
    Workspace<T> w(ws, B, maxT, maxU);
    EB_CUDA(cudaFuncSetAttribute(rnnt_viterbi_kernel<T, VITERBI_PF<T>>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rnnt_viterbi_kernel<T, VITERBI_PF<T>><<<B, ((maxU + 31) / 32) * 32, smem, st>>>(
        w.lpb, w.lpl, xlen, ylen, in_smem ? nullptr : decisions, frames, (T*)label_logp, (T*)score, maxT, maxU, rows);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

}  // namespace

EB_API size_t eb_rnnt_align_bytes(int B, int maxT, int maxU) {
    if (B <= 0 || maxT <= 0 || maxU <= 0 || maxU > 1024) return 0;
    int rows;
    viterbi_smem(maxT, maxU, &rows);
    return rows == maxT ? 0 : (size_t)B * maxT * maxU;
}

EB_API int eb_rnnt_viterbi(const int* xlen, const int* ylen, int B, int maxT, int maxU, int dtype_size,
                           const void* workspace, void* decisions, int* frames, void* label_logp, void* score,
                           void* stream) {
    if (!xlen || !ylen || !workspace || ((!frames || !label_logp) && maxU > 1) || !score || B <= 0 || maxT <= 0 ||
        maxU <= 0 || maxU > 1024)
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    void* ws = const_cast<void*>(workspace);
    unsigned char* dec = reinterpret_cast<unsigned char*>(decisions);
    if (dtype_size == 4) return viterbi<float>(xlen, ylen, B, maxT, maxU, ws, dec, frames, label_logp, score, st);
    if (dtype_size == 8) return viterbi<double>(xlen, ylen, B, maxT, maxU, ws, dec, frames, label_logp, score, st);
    return EB_ERR_INVALID;
}

// Gradient wrt bf16 logits, written as bf16 (grads16 may alias logits16: in place).
EB_API int eb_rnnt_loss_bwd_bf16_fe(const void* logits16, void* grads16, const int* labels, const int* xlen,
                                    const int* ylen, int B, int maxT, int maxU, int V, int blank, void* workspace,
                                    const float* gscale_dev, int gscale_per_batch, double host_scale,
                                    double fastemit_lambda, void* stream) {
    if (!logits16 || !grads16 || !workspace || bad_problem(labels, xlen, ylen, B, maxT, maxU, V, blank) ||
        bad_lambda(fastemit_lambda))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Workspace<float> w(workspace, B, maxT, maxU);
    const long ncells = (long)B * maxT * maxU;
    constexpr int WARPS = 8;
    const bool vec = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits16) & 7) == 0) &&
                     ((reinterpret_cast<uintptr_t>(grads16) & 7) == 0);
    const __nv_bfloat16* in = reinterpret_cast<const __nv_bfloat16*>(logits16);
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(grads16);
    const bool vec8 = (V % 8 == 0) && ((reinterpret_cast<uintptr_t>(logits16) & 15) == 0) &&
                      ((reinterpret_cast<uintptr_t>(grads16) & 15) == 0);
    with_fastemit(w.lpl, fastemit_lambda, [&](auto fe_on, const FastEmit<float>& fe) {
        constexpr bool FE = decltype(fe_on)::value;
        if (vec8)
            rnnt_grad_bf16x8_kernel<WARPS, FE><<<row_grid(ncells, WARPS), WARPS * 32, 0, st>>>(
                in, out, labels, xlen, ylen, w.denom, w.alphas, w.betas, w.ll_fwd, gscale_dev, gscale_per_batch,
                (float)host_scale, B, maxT, maxU, V, blank, fe);
        else if (vec)
            rnnt_grad_kernel<float, __nv_bfloat16, true, WARPS, __nv_bfloat16, FE>
                <<<row_grid(ncells, WARPS), WARPS * 32, 0, st>>>(
                    in, out, labels, xlen, ylen, w.denom, w.alphas, w.betas, w.ll_fwd, gscale_dev, gscale_per_batch,
                    (float)host_scale, B, maxT, maxU, V, blank, fe);
        else
            rnnt_grad_kernel<float, __nv_bfloat16, false, WARPS, __nv_bfloat16, FE>
                <<<row_grid(ncells, WARPS), WARPS * 32, 0, st>>>(
                    in, out, labels, xlen, ylen, w.denom, w.alphas, w.betas, w.ll_fwd, gscale_dev, gscale_per_batch,
                    (float)host_scale, B, maxT, maxU, V, blank, fe);
    });
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_rnnt_loss_bwd_bf16(const void* logits16, void* grads16, const int* labels, const int* xlen,
                                 const int* ylen, int B, int maxT, int maxU, int V, int blank, void* workspace,
                                 const float* gscale_dev, int gscale_per_batch, double host_scale, void* stream) {
    return eb_rnnt_loss_bwd_bf16_fe(logits16, grads16, labels, xlen, ylen, B, maxT, maxU, V, blank, workspace,
                                    gscale_dev, gscale_per_batch, host_scale, 0.0, stream);
}

// The same d logits as eb_rnnt_loss_bwd_bf16's 16-byte kernel, and db_accum[c] += sum over the B*maxT*maxU rows of
// them in eb_colsum's order.  db_part: fp32 scratch of COLSUM_LANES * V.
EB_API int eb_rnnt_loss_bwd_bf16_db_fe(const void* logits16, void* grads16, const int* labels, const int* xlen,
                                       const int* ylen, int B, int maxT, int maxU, int V, int blank, void* workspace,
                                       const float* gscale_dev, int gscale_per_batch, double host_scale,
                                       float* db_part, float* db_accum, double fastemit_lambda, void* stream) {
    if (!logits16 || !grads16 || !workspace || !db_part || !db_accum ||
        bad_problem(labels, xlen, ylen, B, maxT, maxU, V, blank) || bad_lambda(fastemit_lambda) || V % 8 ||
        ((reinterpret_cast<uintptr_t>(logits16) | reinterpret_cast<uintptr_t>(grads16) |
          reinterpret_cast<uintptr_t>(db_part)) & 15))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Workspace<float> w(workspace, B, maxT, maxU);
    const int threads = COLSUM_LANES * (V / 8);
    with_fastemit(w.lpl, fastemit_lambda, [&](auto fe_on, const FastEmit<float>& fe) {
        rnnt_grad_db_bf16x8_kernel<decltype(fe_on)::value><<<(threads + DB_THREADS - 1) / DB_THREADS, DB_THREADS, 0, st>>>(
            reinterpret_cast<const __nv_bfloat16*>(logits16), reinterpret_cast<__nv_bfloat16*>(grads16), labels, xlen,
            ylen, w.denom, w.alphas, w.betas, w.ll_fwd, gscale_dev, gscale_per_batch, (float)host_scale, B, maxT, maxU,
            V, blank, db_part, fe);
    });
    EB_CHECK_LAUNCH();
    return colsum_lanes_finish(db_part, db_accum, V, st);
}

EB_API int eb_rnnt_loss_bwd_bf16_db(const void* logits16, void* grads16, const int* labels, const int* xlen,
                                    const int* ylen, int B, int maxT, int maxU, int V, int blank, void* workspace,
                                    const float* gscale_dev, int gscale_per_batch, double host_scale, float* db_part,
                                    float* db_accum, void* stream) {
    return eb_rnnt_loss_bwd_bf16_db_fe(logits16, grads16, labels, xlen, ylen, B, maxT, maxU, V, blank, workspace,
                                       gscale_dev, gscale_per_batch, host_scale, db_part, db_accum, 0.0, stream);
}

// debugging / test access to the lattice (device pointers into the workspace)
EB_API int eb_rnnt_workspace_views(void* workspace, int B, int maxT, int maxU, int dtype_size,
                                   void** denom, void** alphas, void** betas, void** ll_fwd,
                                   void** ll_bwd) {
    if (dtype_size == 4) {
        Workspace<float> w(workspace, B, maxT, maxU);
        *denom = w.denom; *alphas = w.alphas; *betas = w.betas; *ll_fwd = w.ll_fwd; *ll_bwd = w.ll_bwd;
    } else {
        Workspace<double> w(workspace, B, maxT, maxU);
        *denom = w.denom; *alphas = w.alphas; *betas = w.betas; *ll_fwd = w.ll_fwd; *ll_bwd = w.ll_bwd;
    }
    return EB_OK;
}

EB_API int eb_rnnt_band_loss_fwd(const float* logits, const int* labels, const int* xlen, const int* ylen,
                                 const int* s_begin, const int* nopath, int B, int maxT, int maxU, int R, int V,
                                 int blank, void* workspace, float* costs_dev, int need_beta, void* stream) {
    if (!logits || !workspace || bad_problem(labels, xlen, ylen, B, maxT, maxU, V, blank) ||
        bad_band(s_begin, nopath, R))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Workspace<float> w(workspace, B, maxT, maxU);
    const Band bd{s_begin, nopath, R};
    const long nrows = (long)B * maxT * R;
    constexpr int WARPS = 8;
    if (V % 4 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0)
        rnnt_band_denom_kernel<true, WARPS><<<row_grid(nrows, WARPS), WARPS * 32, 0, st>>>(
            logits, labels, xlen, ylen, bd, w.denom, w.lpb, w.lpl, B, maxT, maxU, V, blank);
    else
        rnnt_band_denom_kernel<false, WARPS><<<row_grid(nrows, WARPS), WARPS * 32, 0, st>>>(
            logits, labels, xlen, ylen, bd, w.denom, w.lpb, w.lpl, B, maxT, maxU, V, blank);
    EB_CHECK_LAUNCH();
    return eb_rnnt_band_lattice(xlen, ylen, s_begin, nopath, B, maxT, maxU, R, workspace, costs_dev, need_beta, stream);
}

EB_API int eb_rnnt_band_lattice(const int* xlen, const int* ylen, const int* s_begin, const int* nopath, int B,
                                int maxT, int maxU, int R, void* workspace, float* costs_dev, int need_beta,
                                void* stream) {
    if (!xlen || !ylen || !workspace || B <= 0 || maxT <= 0 || maxU <= 0 || maxU > 1024 || bad_band(s_begin, nopath, R))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Workspace<float> w(workspace, B, maxT, maxU);
    const Band bd{s_begin, nopath, R};
    const long ncells = (long)B * maxT * maxU;
    rnnt_band_fill_kernel<<<(int)std::min<long>((ncells + 255) / 256, (long)eb_num_sms() * 16), 256, 0, st>>>(
        xlen, ylen, bd, w.denom, w.lpb, w.lpl, B, maxT, maxU);
    EB_CHECK_LAUNCH();
    const int rc = launch_lattice<float>(w, xlen, ylen, B, maxT, maxU, need_beta, st);
    if (rc) return rc;
    if (costs_dev) neg_copy_kernel<float><<<(B + 127) / 128, 128, 0, st>>>(w.ll_fwd, costs_dev, B);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_rnnt_band_loss_bwd_bf16_db(const void* logits16, void* grads16, const int* labels, const int* xlen,
                                         const int* ylen, const int* s_begin, const int* nopath, int B, int maxT,
                                         int maxU, int R, int V, int blank, void* workspace, const float* gscale_dev,
                                         int gscale_per_batch, double host_scale, float* db_part, float* db_accum,
                                         void* stream) {
    if (!logits16 || !grads16 || !workspace || !db_part || !db_accum ||
        bad_problem(labels, xlen, ylen, B, maxT, maxU, V, blank) || bad_band(s_begin, nopath, R) || V % 8 ||
        ((reinterpret_cast<uintptr_t>(logits16) | reinterpret_cast<uintptr_t>(grads16) |
          reinterpret_cast<uintptr_t>(db_part)) & 15))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Workspace<float> w(workspace, B, maxT, maxU);
    const int threads = COLSUM_LANES * (V / 8);
    rnnt_band_grad_db_bf16x8_kernel<<<(threads + DB_THREADS - 1) / DB_THREADS, DB_THREADS, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(logits16), reinterpret_cast<__nv_bfloat16*>(grads16), labels, xlen,
        ylen, Band{s_begin, nopath, R}, w.denom, w.alphas, w.betas, w.ll_fwd, gscale_dev, gscale_per_batch,
        (float)host_scale, B, maxT, maxU, V, blank, db_part);
    EB_CHECK_LAUNCH();
    return colsum_lanes_finish(db_part, db_accum, V, st);
}

EB_API int eb_rnnt_band_loss_bwd(const float* logits, void* grads, int grads_bf16, const int* labels,
                                 const int* xlen, const int* ylen, const int* s_begin, const int* nopath, int B,
                                 int maxT, int maxU, int R, int V, int blank, void* workspace,
                                 const float* gscale_dev, int gscale_per_batch, double host_scale, void* stream) {
    if (!logits || !grads || !workspace || bad_problem(labels, xlen, ylen, B, maxT, maxU, V, blank) ||
        bad_band(s_begin, nopath, R) || (grads_bf16 && (reinterpret_cast<uintptr_t>(grads) & 1)))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Workspace<float> w(workspace, B, maxT, maxU);
    const Band bd{s_begin, nopath, R};
    const long nrows = (long)B * maxT * R;
    constexpr int WARPS = 8;
    const int grid = row_grid(nrows, WARPS);
    const bool vec = V % 4 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(grads) & (grads_bf16 ? 7 : 15)) == 0;
    auto launch = [&](auto* g, auto vec_on) {
        using TO = std::remove_pointer_t<decltype(g)>;
        rnnt_band_grad_kernel<TO, decltype(vec_on)::value, WARPS><<<grid, WARPS * 32, 0, st>>>(
            logits, g, labels, xlen, ylen, bd, w.denom, w.alphas, w.betas, w.ll_fwd, gscale_dev, gscale_per_batch,
            (float)host_scale, B, maxT, maxU, V, blank);
    };
    if (grads_bf16) {
        if (vec) launch((__nv_bfloat16*)grads, std::true_type{});
        else launch((__nv_bfloat16*)grads, std::false_type{});
    } else {
        if (vec) launch((float*)grads, std::true_type{});
        else launch((float*)grads, std::false_type{});
    }
    EB_CHECK_LAUNCH();
    return EB_OK;
}
