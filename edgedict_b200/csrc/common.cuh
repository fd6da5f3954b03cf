// common.cuh -- shared device/host helpers for the edgedict_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>

#define EB_OK 0
#define EB_ERR_INVALID 2
#define EB_ERR_CUDA 3

#define EB_API extern "C" __attribute__((visibility("default")))

// Launch-error check only (no sync): keeps every entry point asynchronous on its stream.
#define EB_CHECK_LAUNCH()                                                             \
    do {                                                                              \
        cudaError_t e__ = cudaGetLastError();                                         \
        if (e__ != cudaSuccess) {                                                     \
            fprintf(stderr, "[edgedict_b200] %s:%d CUDA error: %s\n", __FILE__,       \
                    __LINE__, cudaGetErrorString(e__));                               \
            return EB_ERR_CUDA;                                                       \
        }                                                                             \
    } while (0)

#define EB_CUDA(call)                                                                 \
    do {                                                                              \
        cudaError_t e__ = (call);                                                     \
        if (e__ != cudaSuccess) {                                                     \
            fprintf(stderr, "[edgedict_b200] %s:%d CUDA error: %s\n", __FILE__,       \
                    __LINE__, cudaGetErrorString(e__));                               \
            return EB_ERR_CUDA;                                                       \
        }                                                                             \
    } while (0)

static inline int eb_num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// n bytes from global to shared memory by threads tid = 0 .. nt-1, sixteen independent loads in flight per thread
// before their stores (a plain byte loop waits out one global load latency per byte it copies)
__device__ __forceinline__ void block_copy_bytes(unsigned char* dst, const unsigned char* src, int n, int tid, int nt) {
    constexpr int K = 16;
    for (int i0 = tid; i0 < n; i0 += K * nt) {
        unsigned char r[K];
#pragma unroll
        for (int k = 0; k < K; ++k) r[k] = i0 + k * nt < n ? src[i0 + k * nt] : 0;
#pragma unroll
        for (int k = 0; k < K; ++k)
            if (i0 + k * nt < n) dst[i0 + k * nt] = r[k];
    }
}

// block-wide sum for blockDim.x <= 1024 (result valid in every thread)
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* sh /* >= 33 entries */) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) sh[w] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    T r = (threadIdx.x < nw) ? sh[threadIdx.x] : T(0);
    if (w == 0) {
        r = warp_sum(r);
        if (lane == 0) sh[32] = r;
    }
    __syncthreads();
    return sh[32];
}

// Spin until *ctr >= target (acquire).  A protocol bug or a CTA that was never scheduled must fail
// loudly instead of hanging the GPU: after ~4 s of spinning the kernel traps.
__device__ __forceinline__ void spin_wait_ge(const unsigned* ctr, unsigned target) {
    unsigned v;
    long long t0 = 0;
    unsigned spins = 0;
    while (true) {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        if (v >= target) break;
        if ((++spins & 0xFFFF) == 0) {
            const long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 8000000000LL) {
                printf("[edgedict_b200] grid barrier timeout: block %d saw %u, wants %u\n", blockIdx.x, v, target);
                __trap();
            }
        }
    }
}

// eb_colsum's order for bf16 rows (elementwise.cu): row lane k of COLSUM_LANES adds rows k, k + COLSUM_LANES, ... in
// order from 0.f, then a fixed tree (at stride st = COLSUM_LANES / 2, ..., 1, lane k < st adds lane k + st) adds the lane
// sums, and out[c] += the total.  colsum_lanes_finish runs that tree over lane sums part[k * N + c] that a producer
// summed in that order itself (the loss gradient, loss.cu): the same bits as eb_colsum over the same rows.
constexpr int COLSUM_LANES = 512;
int colsum_lanes_finish(const float* part, float* out, int N, cudaStream_t st);

// The pruned RNN-T loss's padding rule (include/edgedict_b200.h): band row r of frame t, whose band starts at symbol
// position s, holds cell (t, s + r) when t < T_b, r < min(R, U_b), s >= 0 and s + r < U_b; every other row is padding.
// A frame with a negative start has no live row.  The loss entries also treat every row of a nopath utterance as padding.
__device__ __forceinline__ bool band_row_live(int t, int Tn, int Un, int R, int s, int r) {
    return t < Tn && r < min(R, Un) && s + r < Un && s >= 0;
}

// exp through ex2.approx.ftz: FMUL + MUFU.  (__expf without -ftz=true is ex2.approx WITHOUT flush-to-zero, which
// the compiler guards with a range test and two conditional multiplies per call: 3 extra instructions per element
// in the streaming softmax loops.)  Results below 1.2e-38 flush to zero, irrelevant for softmax sums.
__device__ __forceinline__ float fast_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float fast_exp(float x) { return fast_ex2(x * 1.4426950408889634f); }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// streaming (read-once) 128-bit load / store that do not pollute L1
__device__ __forceinline__ float4 ld_stream_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_f4(float* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
