// elementwise.cu -- bandwidth-bound glue kernels of the RNN-T path (sm_90a).
//
//   layernorm fwd/bwd (+ fused residual add)      nn.LayerNorm in rnnt/models.py:47,124 and the
//                                                 `xs = xs + xs_next` of rnnt/models.py:66-69
//   time reduction fwd/bwd                        TimeReduction.forward, rnnt/models.py:21-29
//   embedding gather / scatter-add (BOS prepend)  Decoder.forward, rnnt/models.py:150-153
//   joint hidden tanh(e_t + d_u) fwd/bwd          Joint.forward, rnnt/models.py:169-179 with the
//                                                 first Linear split as W1e*e + W1d*d + b1
//   column sums (bias gradients), casts, Adam     torch autograd / torch.optim.Adam in
//                                                 cli/baseline.py:141-156,239-245
#include <cooperative_groups.h>
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace cg = cooperative_groups;

namespace {

// ------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, H <= 32*MAXV*... generic loop; two-pass mean/var in registers
// when the row fits (H <= 2048), otherwise three passes over global.
// ------------------------------------------------------------------------------------------
constexpr int LN_WARPS = 8;

template <int PL>   // PL = values per lane kept in registers; H <= 32*PL
__global__ void __launch_bounds__(LN_WARPS * 32)
layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ res,
                     const float* __restrict__ gamma, const float* __restrict__ beta,
                     float* __restrict__ y, __nv_bfloat16* __restrict__ y16,
                     float* __restrict__ mean, float* __restrict__ rstd, long rows, int H, float eps) {
    const int lane = threadIdx.x & 31;
    const long wstride = (long)gridDim.x * LN_WARPS;
    for (long r = (long)blockIdx.x * LN_WARPS + (threadIdx.x >> 5); r < rows; r += wstride) {
        const float* xr = x + r * H;
        const float* rr = res ? res + r * H : nullptr;
        float v[PL];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < PL; ++i) {
            int c = lane + i * 32;
            v[i] = 0.f;
            if (c < H) {
                float t = xr[c];
                if (rr) t += rr[c];
                v[i] = t;
                s += t;
            }
        }
        const float mu = warp_sum(s) / H;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < PL; ++i) {
            int c = lane + i * 32;
            if (c < H) { float d = v[i] - mu; q += d * d; }
        }
        const float rs = rsqrtf(warp_sum(q) / H + eps);
        if (lane == 0) {
            if (mean) mean[r] = mu;
            if (rstd) rstd[r] = rs;
        }
#pragma unroll
        for (int i = 0; i < PL; ++i) {
            int c = lane + i * 32;
            if (c < H) {
                float o = (v[i] - mu) * rs * gamma[c] + beta[c];
                y[r * H + c] = o;
                if (y16) y16[r * H + c] = __float2bfloat16(o);
            }
        }
    }
}

// dz = rstd * (g - mean(g) - xhat * mean(g*xhat)), g = dy*gamma
template <int PL>
__global__ void __launch_bounds__(LN_WARPS * 32)
layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                     const float* __restrict__ res, const float* __restrict__ gamma,
                     const float* __restrict__ mean, const float* __restrict__ rstd,
                     float* __restrict__ dz, long rows, int H) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long wstride = (long)gridDim.x * LN_WARPS;
    for (long r = (long)blockIdx.x * LN_WARPS + w; r < rows; r += wstride) {
        const float mu = mean[r], rs = rstd[r];
        float xh[PL], g[PL];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < PL; ++i) {
            int c = lane + i * 32;
            xh[i] = 0.f; g[i] = 0.f;
            if (c < H) {
                float z = x[r * H + c];
                if (res) z += res[r * H + c];
                xh[i] = (z - mu) * rs;
                g[i] = dy[r * H + c] * gamma[c];
                s1 += g[i];
                s2 += g[i] * xh[i];
            }
        }
        s1 = warp_sum(s1) / H;
        s2 = warp_sum(s2) / H;
#pragma unroll
        for (int i = 0; i < PL; ++i) {
            int c = lane + i * 32;
            if (c < H) dz[r * H + c] = rs * (g[i] - s1 - xh[i] * s2);
        }
    }
}

// dz for H % 128 == 0, H <= 1024: one warp per row, 128-bit accesses, NV float4 per lane.  The parameter gradients are
// summed by layernorm_param_grad_kernel in a fixed order, so that they are the same bits on every run.
constexpr int LNB_WARPS = 4;
template <int NV>
__global__ void __launch_bounds__(LNB_WARPS * 32)
layernorm_bwd_fused_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ res,
                           const float* __restrict__ gamma, const float* __restrict__ mean,
                           const float* __restrict__ rstd, float* __restrict__ dz, long rows, int H) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int H4 = H >> 2;
    const long wstride = (long)gridDim.x * LNB_WARPS;
    const float inv_h = 1.f / (float)H;
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    for (long r = (long)blockIdx.x * LNB_WARPS + w; r < rows; r += wstride) {
        const float mu = mean[r], rs = rstd[r];
        const float4* dy4 = reinterpret_cast<const float4*>(dy + r * H);
        const float4* x4 = reinterpret_cast<const float4*>(x + r * H);
        const float4* r4 = res ? reinterpret_cast<const float4*>(res + r * H) : nullptr;
        float4 d[NV], xh[NV];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = lane + i * 32;
            d[i] = make_float4(0.f, 0.f, 0.f, 0.f); xh[i] = d[i];
            if (c < H4) {
                d[i] = dy4[c];
                float4 z = x4[c];
                if (r4) { const float4 q = r4[c]; z.x += q.x; z.y += q.y; z.z += q.z; z.w += q.w; }
                xh[i] = make_float4((z.x - mu) * rs, (z.y - mu) * rs, (z.z - mu) * rs, (z.w - mu) * rs);
                const float4 gm = __ldg(g4 + c);
                const float4 g = make_float4(d[i].x * gm.x, d[i].y * gm.y, d[i].z * gm.z, d[i].w * gm.w);
                s1 += (g.x + g.y) + (g.z + g.w);
                s2 += (g.x * xh[i].x + g.y * xh[i].y) + (g.z * xh[i].z + g.w * xh[i].w);
            }
        }
        s1 = warp_sum(s1) * inv_h;
        s2 = warp_sum(s2) * inv_h;
        float4* dz4 = reinterpret_cast<float4*>(dz + r * H);
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = lane + i * 32;
            if (c < H4) {
                const float4 gm = __ldg(g4 + c);
                dz4[c] = make_float4(rs * (d[i].x * gm.x - s1 - xh[i].x * s2), rs * (d[i].y * gm.y - s1 - xh[i].y * s2),
                                     rs * (d[i].z * gm.z - s1 - xh[i].z * s2), rs * (d[i].w * gm.w - s1 - xh[i].w * s2));
            }
        }
    }
}

// dgamma[c] += sum_r dy*xhat ; dbeta[c] += sum_r dy.  One CTA per 8 columns (one 32-byte sector of a row); thread (c, k)
// of the 8 x 128 block sums the rows k, k+128, ... of column c and a fixed-shape tree adds the 128 lanes of a column:
// a fixed summation order, so the parameter gradients are the same bits on every run.
__global__ void __launch_bounds__(1024) layernorm_param_grad_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                                     const float* __restrict__ res,
                                                                     const float* __restrict__ mean,
                                                                     const float* __restrict__ rstd, float* __restrict__ dgamma,
                                                                     float* __restrict__ dbeta, long rows, int H) {
    __shared__ float sg[128][9], sb[128][9];
    const int cx = threadIdx.x & 7, k = threadIdx.x >> 3;
    const int c = blockIdx.x * 8 + cx;
    float ag = 0.f, ab = 0.f;
    if (c < H) {
        for (long r = k; r < rows; r += 128) {
            float z = x[r * H + c];
            if (res) z += res[r * H + c];
            const float d = dy[r * H + c];
            ag += d * (z - mean[r]) * rstd[r];
            ab += d;
        }
    }
    sg[k][cx] = ag;
    sb[k][cx] = ab;
    __syncthreads();
#pragma unroll 1
    for (int st = 64; st > 0; st >>= 1) {
        if (k < st) { sg[k][cx] += sg[k + st][cx]; sb[k][cx] += sb[k + st][cx]; }
        __syncthreads();
    }
    if (k == 0 && c < H) {
        dgamma[c] += sg[0][cx];
        dbeta[c] += sb[0][cx];
    }
}

// ------------------------------------------------------------------------------------------
__global__ void time_reduce_fwd_kernel(const float* __restrict__ x, float* __restrict__ y,
                                       __nv_bfloat16* __restrict__ y16, int B, int T, int H) {
    const int T2 = (T + 1) / 2;
    const long n = (long)B * T2 * H;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        int c = (int)(i % H);
        long bt = i / H;
        int t2 = (int)(bt % T2);
        int b = (int)(bt / T2);
        float a = x[((long)b * T + 2 * t2) * H + c];
        float bb = (2 * t2 + 1 < T) ? x[((long)b * T + 2 * t2 + 1) * H + c] : 0.f;   // zero pad
        float o = (a + bb) * 0.5f;
        y[i] = o;
        if (y16) y16[i] = __float2bfloat16(o);
    }
}
__global__ void time_reduce_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B,
                                       int T, int H) {
    const int T2 = (T + 1) / 2;
    const long n = (long)B * T * H;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        int c = (int)(i % H);
        long bt = i / H;
        int t = (int)(bt % T);
        int b = (int)(bt / T);
        dx[i] = 0.5f * dy[((long)b * T2 + t / 2) * H + c];
    }
}

// ------------------------------------------------------------------------------------------
// Embedding.  ids [B,U] (int32 or int64); out [B,U+prepend,E]; position 0 = BOS row if prepend.
// ------------------------------------------------------------------------------------------
template <typename I>
__global__ void embedding_fwd_kernel(const I* __restrict__ ids, const float* __restrict__ W,
                                     float* __restrict__ out, __nv_bfloat16* __restrict__ out16,
                                     int B, int U, int E, int prepend, int bos) {
    const int U1 = U + prepend;
    const long n = (long)B * U1 * E;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        int e = (int)(i % E);
        long bu = i / E;
        int u = (int)(bu % U1);
        int b = (int)(bu / U1);
        long id = (prepend && u == 0) ? bos : (long)ids[(long)b * U + u - prepend];
        float v = W[id * E + e];
        out[i] = v;
        if (out16) out16[i] = __float2bfloat16(v);
    }
}
// dW[id] += sum of dout over the positions with that id.  The warp of the FIRST position of an id owns its row and adds
// the positions in order (no atomics: the same bits on every run).  Both walks read 32 consecutive positions per step
// (one coalesced load of ids and a ballot): a warp whose id occurs earlier stops at the first 32-position step that holds
// it, and the owner walks the positions from its own in n / 32 steps, adding only the rows of the matches, lowest first.
// E is walked by the lanes, EMB_EC columns per lane and pass.
constexpr int EMB_EC = 4;
template <typename I>
__device__ __forceinline__ long emb_id(const I* ids, long pos, int U, int U1, int prepend, int bos) {
    const long b = pos / U1;
    const int u = (int)(pos % U1);
    return (prepend && u == 0) ? bos : (long)ids[b * U + u - prepend];
}
template <typename I>
__global__ void embedding_bwd_kernel(const I* __restrict__ ids, const float* __restrict__ dout,
                                     float* __restrict__ dW, int B, int U, int E, int prepend,
                                     int bos, int pad) {
    const int U1 = U + prepend;
    const long n = (long)B * U1;
    const int lane = threadIdx.x & 31;
    for (long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += ((long)gridDim.x * blockDim.x) >> 5) {
        const long id = emb_id(ids, i, U, U1, prepend, bos);
        if (id == pad) continue;                              // padding_idx row gets no gradient
        bool first = true;
        for (long j0 = 0; j0 < i; j0 += 32) {
            const long j = j0 + lane;
            if (__any_sync(0xffffffffu, j < i && emb_id(ids, j, U, U1, prepend, bos) == id)) { first = false; break; }
        }
        if (!first) continue;
        for (int e0 = 0; e0 < E; e0 += 32 * EMB_EC) {
            float acc[EMB_EC];
#pragma unroll
            for (int c = 0; c < EMB_EC; ++c) acc[c] = 0.f;
            for (long j0 = i; j0 < n; j0 += 32) {
                const long j = j0 + lane;
                unsigned m = __ballot_sync(0xffffffffu, j < n && emb_id(ids, j, U, U1, prepend, bos) == id);
                while (m) {
                    const float* dr = dout + (j0 + __ffs(m) - 1) * E;
                    m &= m - 1;
#pragma unroll
                    for (int c = 0; c < EMB_EC; ++c) {
                        const int e = e0 + lane + 32 * c;
                        if (e < E) acc[c] += dr[e];
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < EMB_EC; ++c) {
                const int e = e0 + lane + 32 * c;
                if (e < E) dW[id * E + e] += acc[c];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Joint hidden: h[b,t,u,:] = tanh(ep[b,t,:] + dp[b,u,:])   (ep already carries b1)
// one CTA per (b,t): ep row staged in registers, loops over u; J % 4 == 0 fast path.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float tanh_fast(float x) {     // MUFU.TANH, rel. error ~2^-11: below bf16 resolution
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
}

// fp32 hidden (parity mode): exact tanhf, one CTA per (b,t)
__global__ void joint_hidden_fwd_f32_kernel(const float* __restrict__ ep, const float* __restrict__ dp,
                                            float* __restrict__ hid, int T, int U, int J) {
    const long bt = blockIdx.x;
    const int b = (int)(bt / T);
    const float* e = ep + bt * J;
    const float* d = dp + (long)b * U * J;
    float* o = hid + bt * (long)U * J;
    for (int i = threadIdx.x; i < U * J; i += blockDim.x) o[i] = tanhf(e[i % J] + d[i]);
}

// bf16 hidden (bench mode): each thread owns 8 consecutive j (one 16-byte store per u), e_t kept
// in registers for the whole u loop; J % 8 == 0
__global__ void joint_hidden_fwd_bf16_kernel(const float* __restrict__ ep, const float* __restrict__ dp,
                                             __nv_bfloat16* __restrict__ hid, int T, int U, int J) {
    const long bt = blockIdx.x;
    const int b = (int)(bt / T);
    const int J8 = J / 8;
    for (int q = threadIdx.x; q < J8; q += blockDim.x) {
        const float4 e0 = *reinterpret_cast<const float4*>(ep + bt * J + q * 8);
        const float4 e1 = *reinterpret_cast<const float4*>(ep + bt * J + q * 8 + 4);
        const float* d = dp + (long)b * U * J + q * 8;
        __nv_bfloat16* o = hid + bt * (long)U * J + q * 8;
#pragma unroll 4
        for (int u = 0; u < U; ++u) {
            const float4 d0 = *reinterpret_cast<const float4*>(d + (long)u * J);
            const float4 d1 = *reinterpret_cast<const float4*>(d + (long)u * J + 4);
            uint4 v;
            v.x = pack_bf16(tanh_fast(e0.x + d0.x), tanh_fast(e0.y + d0.y));
            v.y = pack_bf16(tanh_fast(e0.z + d0.z), tanh_fast(e0.w + d0.w));
            v.z = pack_bf16(tanh_fast(e1.x + d1.x), tanh_fast(e1.y + d1.y));
            v.w = pack_bf16(tanh_fast(e1.z + d1.z), tanh_fast(e1.w + d1.w));
            *reinterpret_cast<uint4*>(o + (long)u * J) = v;
        }
    }
}

// dpre = dh * (1 - h^2) written in place over dh; dep[b,t,:] = sum_u dpre
__global__ void joint_hidden_bwd_t_f32_kernel(float* __restrict__ dh, const float* __restrict__ hid,
                                              float* __restrict__ dep, int T, int U, int J) {
    const long bt = blockIdx.x;
    float* g = dh + bt * (long)U * J;
    const float* h = hid + bt * (long)U * J;
    for (int j = threadIdx.x; j < J; j += blockDim.x) {
        float acc = 0.f;
        for (int u = 0; u < U; ++u) {
            float hv = h[(long)u * J + j];
            float pv = g[(long)u * J + j] * (1.f - hv * hv);
            g[(long)u * J + j] = pv;
            acc += pv;
        }
        dep[bt * J + j] = acc;
    }
}
__global__ void joint_hidden_bwd_t_bf16_kernel(__nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ hid,
                                               float* __restrict__ dep, int T, int U, int J) {
    const long bt = blockIdx.x;
    const int J8 = J / 8;
    for (int q = threadIdx.x; q < J8; q += blockDim.x) {
        __nv_bfloat16* g = dh + bt * (long)U * J + q * 8;
        const __nv_bfloat16* h = hid + bt * (long)U * J + q * 8;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int u = 0; u < U; ++u) {
            const uint4 hv = *reinterpret_cast<const uint4*>(h + (long)u * J);
            uint4 gv = *reinterpret_cast<const uint4*>(g + (long)u * J);
            const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w};
            uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 hf = unpack_bf16(hw[i]), gf = unpack_bf16(gw[i]);
                const float p0 = gf.x * (1.f - hf.x * hf.x), p1 = gf.y * (1.f - hf.y * hf.y);
                acc[2 * i] += p0;
                acc[2 * i + 1] += p1;
                gw[i] = pack_bf16(p0, p1);
            }
            *reinterpret_cast<uint4*>(g + (long)u * J) = make_uint4(gw[0], gw[1], gw[2], gw[3]);
        }
        float* o = dep + bt * J + q * 8;
        *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
}
// dep[b,t,:] = sum_u dpre[b,t,u,:] for dpre already produced by the d-hidden GEMM epilogue (eb_gemm_bf16_dtanh)
__global__ void joint_dep_reduce_bf16_kernel(const __nv_bfloat16* __restrict__ dpre, float* __restrict__ dep, int U, int J) {
    const long bt = blockIdx.x;
    const int J8 = J / 8;
    for (int q = threadIdx.x; q < J8; q += blockDim.x) {
        const __nv_bfloat16* g = dpre + bt * (long)U * J + q * 8;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
        for (int u = 0; u < U; ++u) {
            const uint4 gv = *reinterpret_cast<const uint4*>(g + (long)u * J);
            const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 gf = unpack_bf16(gw[i]);
                acc[2 * i] += gf.x;
                acc[2 * i + 1] += gf.y;
            }
        }
        float* o = dep + bt * J + q * 8;
        *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
}
// ddp[b,u,:] = sum_t dpre[b,t,u,:]   one CTA per (b,u)
__global__ void joint_hidden_bwd_u_f32_kernel(const float* __restrict__ dpre, float* __restrict__ ddp, int T,
                                              int U, int J) {
    const int b = blockIdx.x / U, u = blockIdx.x % U;
    const float* g = dpre + ((long)b * T * U + u) * J;
    for (int j = threadIdx.x; j < J; j += blockDim.x) {
        float acc = 0.f;
        for (int t = 0; t < T; ++t) acc += g[(long)t * U * J + j];
        ddp[((long)b * U + u) * J + j] = acc;
    }
}
// bf16: one CTA per (b,u) sums all of T in order (no cross-CTA atomics: the same bits on every run)
__global__ void joint_hidden_bwd_u_bf16_kernel(const __nv_bfloat16* __restrict__ dpre, float* __restrict__ ddp,
                                               int T, int U, int J) {
    const int b = blockIdx.x / U, u = blockIdx.x % U;
    const int t0 = 0, t1 = T;
    const int J8 = J / 8;
    for (int q = threadIdx.x; q < J8; q += blockDim.x) {
        const __nv_bfloat16* g = dpre + ((long)b * T * U + u) * J + q * 8;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int t = t0; t < t1; ++t) {
            const uint4 gv = *reinterpret_cast<const uint4*>(g + (long)t * U * J);
            const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 gf = unpack_bf16(gw[i]);
                acc[2 * i] += gf.x;
                acc[2 * i + 1] += gf.y;
            }
        }
        float* o = ddp + ((long)b * U + u) * J + q * 8;
        *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
}

// ------------------------------------------------------------------------------------------
// column sums out[c] (+)= sum_r x[r,c].  One CTA owns a slab of columns over ALL rows: its row lanes sum strided rows,
// then a fixed-shape tree in shared memory adds the lanes -- no cross-CTA atomics, the same bits on every run.
// ------------------------------------------------------------------------------------------
template <int RL, int CW>                      // RL row lanes x CW columns per CTA, RL * CW threads
__device__ __forceinline__ float colsum_tree(float (*sh)[CW + 1], float v, int k, int cx) {
    sh[k][cx] = v;
    __syncthreads();
#pragma unroll 1
    for (int st = RL / 2; st > 0; st >>= 1) {
        if (k < st) sh[k][cx] += sh[k + st][cx];
        __syncthreads();
    }
    return sh[0][cx];
}
template <typename TI>
__global__ void __launch_bounds__(1024) colsum_kernel(const TI* __restrict__ x, float* __restrict__ out, long rows, int N) {
    __shared__ float sh[32][33];
    const int cx = threadIdx.x & 31, k = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + cx;
    float acc = 0.f;
    if (c < N)
        for (long r = k; r < rows; r += 32) acc += (float)x[r * N + c];
    const float t = colsum_tree<32, 32>(sh, acc, k, cx);
    if (k == 0 && c < N) out[c] += t;
}

// bf16 rows with N % 8 == 0: a slab of 16 columns is summed by 512 row lanes (two threads of 8 columns per lane, one
// 16-byte load per row each, eight row loads in flight); lane k adds rows k, k + 512, k + 1024, ... in order, then a
// fixed-shape tree adds the 512 lane sums.  The lanes of a slab are spread over a cluster of COLSUM_CL CTAs so that the
// 4 GB column sum of the joint's d logits (N = 1024: 64 slabs) streams from every SM instead of 64, and so that a CTA
// needs only 8.7 KB of shared memory: it fits beside a CTA of the joint's d-hidden GEMM (198 KB), under which this sum
// runs.  The first tree levels add lane sums across the cluster through distributed shared memory, the rest run in the
// CTA of rank 0.  Same additions in the same order as one CTA of 512 lanes: the same bits.
constexpr int COLSUM_CL = 4, COLSUM_CTA_LANES = COLSUM_LANES / COLSUM_CL;   // (the tree below assumes 4)
__global__ void __cluster_dims__(1, COLSUM_CL, 1) __launch_bounds__(2 * COLSUM_CTA_LANES)
colsum_bf16_vec_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, long rows, int N) {
    __shared__ float sh[COLSUM_CTA_LANES][17];
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned rank = cluster.block_rank();
    const int half = threadIdx.x & 1, kl = threadIdx.x >> 1, k = (int)rank * COLSUM_CTA_LANES + kl;
    const int c0 = blockIdx.x * 16 + half * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c0 < N) {
        const __nv_bfloat16* p = x + (long)k * N + c0;
        const long step = (long)COLSUM_LANES * N;
        long r = k;
        for (; r + 7 * COLSUM_LANES < rows; r += 8 * COLSUM_LANES) {
            uint4 v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = *reinterpret_cast<const uint4*>(p + q * step);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const uint32_t w[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
                    acc[2 * i] += f.x;
                    acc[2 * i + 1] += f.y;
                }
            }
            p += 8 * step;
        }
        for (; r < rows; r += COLSUM_LANES, p += step) {
            const uint4 v = *reinterpret_cast<const uint4*>(p);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
                acc[2 * i] += f.x;
                acc[2 * i + 1] += f.y;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) sh[kl][half * 8 + i] = acc[i];
    // the tree of colsum_tree<512, 16> (at stride st, lane k < st adds lane k + st), its first two levels across the
    // cluster: stride 256 adds rank r + 2 to rank r, stride 128 adds rank 1 to rank 0
    cluster.sync();
    if (rank < 2) {
        const float* peer = cluster.map_shared_rank(&sh[0][0], rank + 2);
        for (int e = threadIdx.x; e < COLSUM_CTA_LANES * 16; e += blockDim.x) sh[e >> 4][e & 15] += peer[(e >> 4) * 17 + (e & 15)];
    }
    cluster.sync();
    if (rank == 0) {
        const float* peer = cluster.map_shared_rank(&sh[0][0], 1);
        for (int e = threadIdx.x; e < COLSUM_CTA_LANES * 16; e += blockDim.x) sh[e >> 4][e & 15] += peer[(e >> 4) * 17 + (e & 15)];
    }
    cluster.sync();                                          // (a CTA's shared memory stays valid until its peers have read it)
    if (rank != 0) return;
#pragma unroll 1
    for (int st = COLSUM_CTA_LANES / 2; st > 0; st >>= 1) {
        for (int e = threadIdx.x; e < st * 16; e += blockDim.x) sh[e >> 4][e & 15] += sh[(e >> 4) + st][e & 15];
        __syncthreads();
    }
    if (threadIdx.x < 16 && blockIdx.x * 16 + (int)threadIdx.x < N) out[blockIdx.x * 16 + threadIdx.x] += sh[0][threadIdx.x];
}

// colsum_tree<COLSUM_LANES, 16> over lane sums in global memory (common.cuh): one CTA per 16 columns
__global__ void __launch_bounds__(COLSUM_LANES) colsum_lanes_finish_kernel(const float* __restrict__ part,
                                                                           float* __restrict__ out, int N) {
    __shared__ float sh[COLSUM_LANES][17];
    const int c0 = blockIdx.x * 16;
    for (int e = threadIdx.x; e < COLSUM_LANES * 16; e += blockDim.x)
        sh[e >> 4][e & 15] = c0 + (e & 15) < N ? part[(long)(e >> 4) * N + c0 + (e & 15)] : 0.f;
    __syncthreads();
#pragma unroll 1
    for (int st = COLSUM_LANES / 2; st > 0; st >>= 1) {
        for (int e = threadIdx.x; e < st * 16; e += blockDim.x) sh[e >> 4][e & 15] += sh[(e >> 4) + st][e & 15];
        __syncthreads();
    }
    if (threadIdx.x < 16 && c0 + (int)threadIdx.x < N) out[c0 + threadIdx.x] += sh[0][threadIdx.x];
}

__global__ void cast_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long n) {
    long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const long stride = (long)gridDim.x * blockDim.x * 4;
    for (; i + 3 < n; i += stride) {
        float4 v = *reinterpret_cast<const float4*>(x + i);
        __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        uint2 q;
        q.x = *reinterpret_cast<uint32_t*>(&a);
        q.y = *reinterpret_cast<uint32_t*>(&b);
        *reinterpret_cast<uint2*>(y + i) = q;
    }
    if (i < n) for (long k = i; k < n && k < i + 4; ++k) y[k] = __float2bfloat16(x[k]);
}

// y[c, r] = x[r, c]  (bf16 or fp32 -> bf16), 32x32 tiles through shared memory.  Column tiles on x, row tiles on y,
// looped with stride gridDim.y: gridDim.y is capped at 65535, so rows beyond 65535 * 32 take more than one pass.
template <typename TI>
__global__ void transpose_to_bf16_kernel(const TI* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                         long rows, long cols) {
    __shared__ float tile[32][33];
    const long c0 = (long)blockIdx.x * 32;
    for (long r0 = (long)blockIdx.y * 32; r0 < rows; r0 += (long)gridDim.y * 32) {
        for (int i = threadIdx.y; i < 32; i += blockDim.y) {
            long r = r0 + i, c = c0 + threadIdx.x;
            tile[i][threadIdx.x] = (r < rows && c < cols) ? (float)x[r * cols + c] : 0.f;
        }
        __syncthreads();
        for (int i = threadIdx.y; i < 32; i += blockDim.y) {
            long c = c0 + i, r = r0 + threadIdx.x;
            if (r < rows && c < cols) y[c * rows + r] = __float2bfloat16(tile[threadIdx.x][i]);
        }
        __syncthreads();                                   // the tile is refilled by the next pass
    }
}

// Adam (torch.optim.Adam semantics, no amsgrad): flat fp32 bucket
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long n, float lr, float b1, float b2, float eps,
                            float wd, float bc1, float bc2, float gscale) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        float gi = g[i] * gscale;
        if (wd != 0.f) gi += wd * p[i];
        float mi = b1 * m[i] + (1.f - b1) * gi;
        float vi = b2 * v[i] + (1.f - b2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        float denom = sqrtf(vi) / sqrtf(bc2) + eps;
        p[i] -= (lr / bc1) * (mi / denom);
    }
}

// Adam / AdamW over the flat bucket with the gradient clip and the loss-scale handling folded in (SURVEY 8(f) N3):
//   gscale      = 1 / loss_scale (and 1 / accumulation steps): every gradient is multiplied by it;
//   sumsq       = device scalar holding sum(g^2) of the UNSCALED bucket (eb_sumsq), or null: no clip, no overflow test;
//   max_norm>0  : torch.nn.utils.clip_grad_norm_ semantics, coef = max_norm / (norm + 1e-6) applied when < 1
//                 (cli/baseline.py:239-245);
//   a non-finite norm (overflow under loss scaling) skips the update entirely, as apex's scaler does;
//   adamw       : the reference's own AdamW (modules/optimizer.py:283-290): p -= lr*sqrt(bc2)/bc1 * (wd*p + m/(sqrt(v)+eps));
//                 else torch.optim.Adam with L2 weight decay added to the gradient.
__global__ void adam_ex_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                               float* __restrict__ v, long n, float lr, float b1, float b2, float eps, float wd,
                               float bc1, float bc2, float gscale, const float* __restrict__ sumsq, float max_norm,
                               int adamw) {
    float coef = gscale;
    if (sumsq) {
        const float norm = sqrtf(*sumsq) * fabsf(gscale);
        if (!isfinite(norm)) return;
        if (max_norm > 0.f) {
            const float c = max_norm / (norm + 1e-6f);
            if (c < 1.f) coef *= c;
        }
    }
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        float gi = g[i] * coef;
        const float pi = p[i];
        if (!adamw && wd != 0.f) gi += wd * pi;
        const float mi = b1 * m[i] + (1.f - b1) * gi;
        const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        if (adamw) p[i] = pi - (lr * sqrtf(bc2) / bc1) * (wd * pi + mi / (sqrtf(vi) + eps));
        else p[i] = pi - (lr / bc1) * (mi / (sqrtf(vi) / sqrtf(bc2) + eps));
    }
}

__global__ void sumsq_kernel(const float* __restrict__ x, long n, float* __restrict__ out) {
    __shared__ float sh[33];
    float acc = 0.f;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        acc += x[i] * x[i];
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) atomicAdd(out, acc);
}

inline int ew_grid(long n, int threads) {
    long b = (n + threads - 1) / threads;
    long cap = (long)eb_num_sms() * 32;
    return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

EB_API int eb_layernorm_fwd(const float* x, const float* res, const float* gamma, const float* beta,
                            float* y, void* y_bf16, float* mean, float* rstd, long rows, int H,
                            float eps, void* stream) {
    if (!x || !gamma || !beta || !y || rows <= 0 || H <= 0 || H > 2048) return EB_ERR_INVALID;
    long blocks = (rows + LN_WARPS - 1) / LN_WARPS;
    long cap = (long)eb_num_sms() * 8;
    int grid = (int)(blocks < cap ? blocks : cap);
#define LN_FWD(PL) layernorm_fwd_kernel<PL><<<grid, LN_WARPS * 32, 0, ST(stream)>>>( \
        x, res, gamma, beta, y, (__nv_bfloat16*)y_bf16, mean, rstd, rows, H, eps)
    if (H <= 256) LN_FWD(8); else if (H <= 512) LN_FWD(16); else if (H <= 1024) LN_FWD(32); else LN_FWD(64);
#undef LN_FWD
    EB_CHECK_LAUNCH();
    return EB_OK;
}

// The two passes of eb_layernorm_bwd, for callers that run them apart (the layer wavefront of the LSTM stack's backward:
// dz per time chunk on the critical path, the parameter gradients once per layer beside it).  Rows are independent in
// the dz pass and the parameter pass sums in a fixed order over all rows it is given, so dz of a row block is the same
// bits as the rows of a whole-buffer call, and the parameter pass over the whole buffer is the same bits as inside it.
EB_API int eb_layernorm_bwd_dz(const float* dy, const float* x, const float* res, const float* gamma, const float* mean,
                               const float* rstd, float* dz, long rows, int H, void* stream) {
    if (!dy || !x || !gamma || !mean || !rstd || !dz || rows <= 0 || H <= 0 || H > 2048) return EB_ERR_INVALID;
    const bool vec_ok = H % 128 == 0 && H <= 1024 &&
                        ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dz) |
                          reinterpret_cast<uintptr_t>(gamma) | (res ? reinterpret_cast<uintptr_t>(res) : 0)) & 15) == 0;
    if (vec_ok) {
        long blocks_f = (rows + LNB_WARPS - 1) / LNB_WARPS;
        long cap_f = (long)eb_num_sms() * 3;
        const int grid_f = (int)(blocks_f < cap_f ? blocks_f : cap_f);
#define LN_BWDF(NV) layernorm_bwd_fused_kernel<NV><<<grid_f, LNB_WARPS * 32, 0, ST(stream)>>>( \
        dy, x, res, gamma, mean, rstd, dz, rows, H)
        if (H <= 128) LN_BWDF(1); else if (H <= 256) LN_BWDF(2); else if (H <= 512) LN_BWDF(4); else LN_BWDF(8);
#undef LN_BWDF
    } else {
        long blocks = (rows + LN_WARPS - 1) / LN_WARPS;
        long cap = (long)eb_num_sms() * 8;
        int grid = (int)(blocks < cap ? blocks : cap);
#define LN_BWD(PL) layernorm_bwd_kernel<PL><<<grid, LN_WARPS * 32, 0, ST(stream)>>>( \
        dy, x, res, gamma, mean, rstd, dz, rows, H)
        if (H <= 256) LN_BWD(8); else if (H <= 512) LN_BWD(16); else if (H <= 1024) LN_BWD(32); else LN_BWD(64);
#undef LN_BWD
    }
    EB_CHECK_LAUNCH();
    return EB_OK;
}

// dgamma += sum_r dy*xhat, dbeta += sum_r dy (the caller zeroes them)
EB_API int eb_layernorm_bwd_params(const float* dy, const float* x, const float* res, const float* mean,
                                   const float* rstd, float* dgamma, float* dbeta, long rows, int H, void* stream) {
    if (!dy || !x || !mean || !rstd || !dgamma || !dbeta || rows <= 0 || H <= 0 || H > 2048) return EB_ERR_INVALID;
    layernorm_param_grad_kernel<<<(H + 7) / 8, 1024, 0, ST(stream)>>>(dy, x, res, mean, rstd, dgamma, dbeta, rows, H);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_layernorm_bwd(const float* dy, const float* x, const float* res, const float* gamma,
                            const float* mean, const float* rstd, float* dz, float* dgamma,
                            float* dbeta, long rows, int H, void* stream) {
    if (!dy || !x || !gamma || !mean || !rstd || !dz || !dgamma || !dbeta || rows <= 0 || H <= 0 || H > 2048)
        return EB_ERR_INVALID;
    const int st = eb_layernorm_bwd_dz(dy, x, res, gamma, mean, rstd, dz, rows, H, stream);
    if (st != EB_OK) return st;
    return eb_layernorm_bwd_params(dy, x, res, mean, rstd, dgamma, dbeta, rows, H, stream);
}

EB_API int eb_time_reduce_fwd(const float* x, float* y, void* y_bf16, int B, int T, int H, void* stream) {
    if (B < 0 || T < 0 || H < 0) return EB_ERR_INVALID;
    long n = (long)B * ((T + 1) / 2) * H;
    if (n == 0) return EB_OK;
    if (!x || !y) return EB_ERR_INVALID;
    time_reduce_fwd_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(x, y, (__nv_bfloat16*)y_bf16, B, T, H);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
EB_API int eb_time_reduce_bwd(const float* dy, float* dx, int B, int T, int H, void* stream) {
    if (B < 0 || T < 0 || H < 0) return EB_ERR_INVALID;
    long n = (long)B * T * H;
    if (n == 0) return EB_OK;
    if (!dy || !dx) return EB_ERR_INVALID;
    time_reduce_bwd_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(dy, dx, B, T, H);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_embedding_fwd(const void* ids, int ids_are_int64, const float* W, float* out,
                            void* out_bf16, int B, int U, int E, int prepend_bos, int bos, void* stream) {
    if (B < 0 || U < 0 || E < 0 || (prepend_bos && bos < 0)) return EB_ERR_INVALID;
    long n = (long)B * (U + (prepend_bos ? 1 : 0)) * E;
    if (n == 0) return EB_OK;
    if (!W || !out || (U > 0 && !ids)) return EB_ERR_INVALID;    // U = 0 (priming): ids is never read
    if (ids_are_int64)
        embedding_fwd_kernel<long long><<<ew_grid(n, 256), 256, 0, ST(stream)>>>(
            (const long long*)ids, W, out, (__nv_bfloat16*)out_bf16, B, U, E, prepend_bos ? 1 : 0, bos);
    else
        embedding_fwd_kernel<int><<<ew_grid(n, 256), 256, 0, ST(stream)>>>(
            (const int*)ids, W, out, (__nv_bfloat16*)out_bf16, B, U, E, prepend_bos ? 1 : 0, bos);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
EB_API int eb_embedding_bwd(const void* ids, int ids_are_int64, const float* dout, float* dW, int B,
                            int U, int E, int prepend_bos, int bos, int pad, void* stream) {
    if (B < 0 || U < 0 || E < 0 || (prepend_bos && bos < 0)) return EB_ERR_INVALID;
    const long npos = (long)B * (U + (prepend_bos ? 1 : 0));
    if (npos == 0 || E == 0) return EB_OK;
    if (!dout || !dW || (U > 0 && !ids)) return EB_ERR_INVALID;
    const long n = npos * 32;                                // one warp per position
    if (ids_are_int64)
        embedding_bwd_kernel<long long><<<ew_grid(n, 256), 256, 0, ST(stream)>>>(
            (const long long*)ids, dout, dW, B, U, E, prepend_bos ? 1 : 0, bos, pad);
    else
        embedding_bwd_kernel<int><<<ew_grid(n, 256), 256, 0, ST(stream)>>>(
            (const int*)ids, dout, dW, B, U, E, prepend_bos ? 1 : 0, bos, pad);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_joint_hidden_fwd(const float* ep, const float* dp, void* hidden, int hidden_bf16, int B,
                               int T, int U, int J, void* stream) {
    if (!ep || !dp || !hidden) return EB_ERR_INVALID;
    if (hidden_bf16) {       // 16-byte loads of ep / dp and stores of hidden
        if (J % 8 || ((reinterpret_cast<uintptr_t>(ep) | reinterpret_cast<uintptr_t>(dp) |
                       reinterpret_cast<uintptr_t>(hidden)) & 15))
            return EB_ERR_INVALID;
        joint_hidden_fwd_bf16_kernel<<<B * T, 96, 0, ST(stream)>>>(ep, dp, (__nv_bfloat16*)hidden, T, U, J);
    } else {
        joint_hidden_fwd_f32_kernel<<<B * T, 256, 0, ST(stream)>>>(ep, dp, (float*)hidden, T, U, J);
    }
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_joint_hidden_bwd(void* dhidden_inout, const void* hidden, int is_bf16, float* dep,
                               float* ddp, int B, int T, int U, int J, void* stream) {
    if (!dhidden_inout || !hidden || !dep || !ddp) return EB_ERR_INVALID;
    if (is_bf16) {           // 16-byte accesses of every operand
        if (J % 8 || ((reinterpret_cast<uintptr_t>(dhidden_inout) | reinterpret_cast<uintptr_t>(hidden) |
                       reinterpret_cast<uintptr_t>(dep) | reinterpret_cast<uintptr_t>(ddp)) & 15))
            return EB_ERR_INVALID;
        joint_hidden_bwd_t_bf16_kernel<<<B * T, 96, 0, ST(stream)>>>(
            (__nv_bfloat16*)dhidden_inout, (const __nv_bfloat16*)hidden, dep, T, U, J);
        EB_CHECK_LAUNCH();
        joint_hidden_bwd_u_bf16_kernel<<<B * U, 96, 0, ST(stream)>>>((const __nv_bfloat16*)dhidden_inout, ddp, T, U, J);
    } else {
        joint_hidden_bwd_t_f32_kernel<<<B * T, 256, 0, ST(stream)>>>(
            (float*)dhidden_inout, (const float*)hidden, dep, T, U, J);
        EB_CHECK_LAUNCH();
        joint_hidden_bwd_u_f32_kernel<<<B * U, 256, 0, ST(stream)>>>((const float*)dhidden_inout, ddp, T, U, J);
    }
    EB_CHECK_LAUNCH();
    return EB_OK;
}

// The two broadcast reductions of the joint's first layer when d(pre-activation) [B,T,U,J] (bf16) already exists:
// dep[b,t,:] = sum_u, ddp[b,u,:] = sum_t  (backward of the e_t + d_u broadcast add of Joint.forward).
EB_API int eb_joint_dpre_reduce(const void* dpre16, float* dep, float* ddp, int B, int T, int U, int J, void* stream) {
    if (!dpre16 || !dep || !ddp || B <= 0 || T <= 0 || U <= 0 || J <= 0 || J % 8 ||
        ((reinterpret_cast<uintptr_t>(dpre16) | reinterpret_cast<uintptr_t>(dep) | reinterpret_cast<uintptr_t>(ddp)) & 15))
        return EB_ERR_INVALID;
    joint_dep_reduce_bf16_kernel<<<B * T, 96, 0, ST(stream)>>>((const __nv_bfloat16*)dpre16, dep, U, J);
    EB_CHECK_LAUNCH();
    joint_hidden_bwd_u_bf16_kernel<<<B * U, 96, 0, ST(stream)>>>((const __nv_bfloat16*)dpre16, ddp, T, U, J);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_colsum(const void* x, int x_bf16, float* out, long rows, int N, void* stream) {
    if (!x || !out || rows <= 0 || N <= 0) return EB_ERR_INVALID;
    if (x_bf16 && N % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0)
        colsum_bf16_vec_kernel<<<dim3((N + 15) / 16, COLSUM_CL), 2 * COLSUM_CTA_LANES, 0, ST(stream)>>>((const __nv_bfloat16*)x, out, rows, N);
    else if (x_bf16)
        colsum_kernel<__nv_bfloat16><<<(N + 31) / 32, 1024, 0, ST(stream)>>>((const __nv_bfloat16*)x, out, rows, N);
    else
        colsum_kernel<float><<<(N + 31) / 32, 1024, 0, ST(stream)>>>((const float*)x, out, rows, N);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

int colsum_lanes_finish(const float* part, float* out, int N, cudaStream_t st) {
    colsum_lanes_finish_kernel<<<(N + 15) / 16, COLSUM_LANES, 0, st>>>(part, out, N);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_cast_bf16(const float* x, void* y, long n, void* stream) {
    if (n <= 0) return EB_OK;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 7)) return EB_ERR_INVALID;
    cast_bf16_kernel<<<ew_grid((n + 3) / 4, 256), 256, 0, ST(stream)>>>(x, (__nv_bfloat16*)y, n);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_transpose_to_bf16(const void* x, int x_bf16, void* y, long rows, long cols, void* stream) {
    if (rows < 0 || cols < 0 || (cols + 31) / 32 > 0x7fffffffL) return EB_ERR_INVALID;
    if (rows == 0 || cols == 0) return EB_OK;
    if (!x || !y) return EB_ERR_INVALID;
    const long row_tiles = (rows + 31) / 32;
    dim3 grid((unsigned)((cols + 31) / 32), (unsigned)(row_tiles < 65535 ? row_tiles : 65535));
    if (x_bf16)
        transpose_to_bf16_kernel<__nv_bfloat16><<<grid, dim3(32, 8), 0, ST(stream)>>>(
            (const __nv_bfloat16*)x, (__nv_bfloat16*)y, rows, cols);
    else
        transpose_to_bf16_kernel<float><<<grid, dim3(32, 8), 0, ST(stream)>>>((const float*)x, (__nv_bfloat16*)y, rows, cols);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_adam_step(float* p, const float* g, float* m, float* v, long n, float lr, float beta1,
                        float beta2, float eps, float weight_decay, int step, float grad_scale,
                        void* stream) {
    if (!p || !g || !m || !v || n <= 0 || step < 1) return EB_ERR_INVALID;
    float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
    adam_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(p, g, m, v, n, lr, beta1, beta2, eps,
                                                         weight_decay, bc1, bc2, grad_scale);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_adam_step_ex(float* p, const float* g, float* m, float* v, long n, float lr, float beta1, float beta2,
                           float eps, float weight_decay, int step, float grad_scale, const float* sumsq,
                           float max_norm, int adamw, void* stream) {
    if (!p || !g || !m || !v || n <= 0 || step < 1) return EB_ERR_INVALID;
    float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
    adam_ex_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2,
                                                            grad_scale, sumsq, max_norm, adamw);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_sumsq(const float* x, long n, float* out_accum, void* stream) {
    if (n < 0 || !out_accum) return EB_ERR_INVALID;
    if (n == 0) return EB_OK;
    if (!x) return EB_ERR_INVALID;
    sumsq_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(x, n, out_accum);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
