// gemm_simt.cu -- fp32 CUDA-core GEMM used by the fp32 (parity) mode of every Linear /
// LSTM-input projection of the path (nn.Linear / nn.LSTM input GEMMs in rnnt/models.py:45-46,
// 129,148,163-167).  Exact fp32 FMA accumulation so that the parity tests can hold the
// reference's torch-CPU fp32 results to 1e-3 relative; the bf16 tensor-core path lives in
// gemm_tc.cu.
//
//   C[m,n] = alpha * sum_k A(m,k) * B(k,n) + beta * C[m,n] + bias[n]
//   A(m,k) = A[m*sam + k*sak],  B(k,n) = B[k*sbk + n*sbn],  C row-major with leading dim ldc.
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;

__global__ void __launch_bounds__(256)
sgemm_kernel(const float* __restrict__ A, long sam, long sak, const float* __restrict__ B, long sbk,
             long sbn, float* __restrict__ C, long ldc, const float* __restrict__ bias, int M, int N,
             int K, float alpha, float beta, int kchunk = 0, long ldz = 0) {
    // split-K (blockIdx.z): slice z contracts k in [z*kchunk, (z+1)*kchunk) into its own C slice z*ldz apart
    if (kchunk > 0) {
        const long z = blockIdx.z;
        A += z * kchunk * sak;
        B += z * kchunk * sbk;
        C += z * ldz;
        K = min((long)kchunk, (long)K - z * kchunk);
    }
    __shared__ float As[2][BK][BM + 4];
    __shared__ float Bs[2][BK][BN + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;   // M (can be millions) on grid.x
    const int ty = tid / 16, tx = tid % 16;           // 16 x 16 threads, each 4x4 outputs
    const bool a_kc = (sak == 1), b_nc = (sbn == 1);  // contiguous direction of each operand
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    float ra[4], rb[4];
    auto fetch = [&](int k0) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            int i = tid + r * 256;                    // 0..1023 over the 64x16 tile
            int am, ak, bk, bn;
            if (a_kc) { am = i / BK; ak = i % BK; } else { ak = i / BM; am = i % BM; }
            if (b_nc) { bk = i / BN; bn = i % BN; } else { bn = i / BK; bk = i % BK; }
            ra[r] = (m0 + am < M && k0 + ak < K) ? A[(long)(m0 + am) * sam + (long)(k0 + ak) * sak] : 0.f;
            rb[r] = (n0 + bn < N && k0 + bk < K) ? B[(long)(k0 + bk) * sbk + (long)(n0 + bn) * sbn] : 0.f;
        }
    };
    auto stash = [&](int buf) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            int i = tid + r * 256;
            int am, ak, bk, bn;
            if (a_kc) { am = i / BK; ak = i % BK; } else { ak = i / BM; am = i % BM; }
            if (b_nc) { bk = i / BN; bn = i % BN; } else { bn = i / BK; bk = i % BK; }
            As[buf][ak][am] = ra[r];
            Bs[buf][bk][bn] = rb[r];
        }
    };
    const int nk = (K + BK - 1) / BK;
    fetch(0);
    stash(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) fetch((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float4 a4 = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM]);
            float4 b4 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * TN]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) stash(buf ^ 1);
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        int m = m0 + ty * TM + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            int n = n0 + tx * TN + j;
            if (n >= N) continue;
            float v = alpha * acc[i][j];
            if (bias) v += bias[n];
            if (beta != 0.f) v += beta * C[(long)m * ldc + n];
            C[(long)m * ldc + n] = v;
        }
    }
}

}  // namespace

EB_API int eb_gemm_f32(const float* A, long sam, long sak, const float* B, long sbk, long sbn, float* C,
                       long ldc, const float* bias, int M, int N, int K, float alpha, float beta,
                       void* stream) {
    if (!A || !B || !C || M <= 0 || N <= 0 || K <= 0) return EB_ERR_INVALID;
    dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN);
    sgemm_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(A, sam, sak, B, sbk, sbn, C,
                                                                           ldc, bias, M, N, K, alpha, beta);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

// C = A B as eb_gemm_f32 (alpha 1, no bias), its contraction split into ceil(K / kchunk) slices: slice z writes
// part[z] ([M, N], row-major) and the caller adds the slices in slice order (eb_colsum).  For the weight gradients of the
// front end's convolutions, whose K (rows) runs to about a million against a 128 x 384 output.
EB_API int eb_gemm_f32_splitk(const float* A, long sam, long sak, const float* B, long sbk, long sbn, float* part,
                              int M, int N, int K, int kchunk, void* stream) {
    if (!A || !B || !part || M <= 0 || N <= 0 || K <= 0 || kchunk <= 0) return EB_ERR_INVALID;
    const int nz = (K + kchunk - 1) / kchunk;
    if (nz > 65535) return EB_ERR_INVALID;
    dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, nz);
    sgemm_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(A, sam, sak, B, sbk, sbn, part, N, nullptr,
                                                                           M, N, K, 1.f, 0.f, kchunk, (long)M * N);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
