// pruned.cu -- the pruned RNN-T loss's own kernels (Kuang et al., "Pruned RNN-T for fast, memory-efficient ASR
// training", Interspeech 2022), for sm_90a:
//
//   1. simple statistics       the trivial joiner's N(t,u) = logsumexp_v(am[t,v] + lm[u,v]) in product form,
//                              amax[t] + lmax[u] + log(exp(am - amax) . exp(lm - lmax)^T), one fp32 GEMM per utterance;
//                              a cell whose product falls below SIMPLE_MIN_P is recomputed by a direct log-sum-exp.
//                              Written as denom / lpb / lpl of a loss workspace that eb_rnnt_loss_lattice runs on.
//   2. simple backward         d am = exp(am - amax) * (G . exp(lm - lmax)), d lm = exp(lm - lmax) * (G^T . exp(am -
//                              amax)), G(t,u) = occ(t,u) exp(amax + lmax - N), two fp32 GEMMs per utterance, then one
//                              pass per row adding the direct terms of the fallback cells and the blank / label terms
//   3. band_choice_kernel      s_begin[b, t], the first symbol position of frame t's band of Rb, one CTA per utterance
//   4. band_hidden_kernel      tanh(ep[b,t] + dp[b, s_begin + r]) over the band rows, fp32 (tanhf) or bf16 (tanh.approx)
//   5. band_dep/ddp_kernel     d ep and d dp from d(pre-activation) of the band rows; the frames whose band covers a
//                              symbol position are a contiguous range (the bands are monotone), so d dp is a gather
//
// The band rows' statistics and gradient live in loss.cu, next to the dense kernels whose row code they share.
// The formulas, lengths and bounds are in include/edgedict_b200.h.
#include <cmath>

#include "common.cuh"
#include "../../include/edgedict_b200.h"

#define ST(s) reinterpret_cast<cudaStream_t>(s)

namespace {

__device__ __forceinline__ int clamp_T(int xlen, int maxT) { return min(max(xlen, 0), maxT); }
__device__ __forceinline__ int clamp_U(int ylen, int maxU) { return min(max(ylen, 0) + 1, maxU); }

// the loss workspace's arrays (loss.cu, Workspace<float>)
struct Ws {
    float *denom, *lpb, *lpl, *alphas, *betas, *ll_fwd;
    __host__ __device__ Ws(void* ws, int B, int maxT, int maxU) {
        const size_t n = (size_t)B * maxT * maxU;
        float* p = reinterpret_cast<float*>(ws);
        denom = p; lpb = p + n; lpl = p + 2 * n; alphas = p + 3 * n; betas = p + 4 * n; ll_fwd = p + 5 * n;
    }
};

// ---------------------------------------------------------------------------------------------
// 1. simple-loss statistics.  All products have positive terms, so the fp32 GEMM keeps its relative accuracy down to
//    where terms underflow: below SIMPLE_MIN_P the mass exp(am - amax) exp(lm - lmax) lost to underflow (at most V
//    terms of 2^-126) could matter, and the cell takes the direct log-sum-exp instead.  A cell whose rows peak at
//    different tokens far apart lands there, so a finite N never comes out +-inf.
// ---------------------------------------------------------------------------------------------
constexpr float SIMPLE_MIN_P = 1e-25f;

// the scratch of the simple loss (include/edgedict_b200.h, eb_rnnt_simple_scratch_bytes)
struct SimpleScratch {
    float *ea, *el, *amax, *lmax, *prod, *G;              // [B,T,V], [B,U,V], [B,T], [B,U], [B,T,U], [B,T,U]
    __host__ __device__ SimpleScratch(void* p, int B, int T, int U, int V) {
        float* f = reinterpret_cast<float*>(p);
        ea = f; f += (size_t)B * T * V;
        el = f; f += (size_t)B * U * V;
        amax = f; f += (size_t)B * T;
        lmax = f; f += (size_t)B * U;
        prod = f; f += (size_t)B * T * U;
        G = f;
    }
    static size_t bytes(int B, int T, int U, int V) {
        return sizeof(float) * ((size_t)B * T * V + (size_t)B * U * V + (size_t)B * T + (size_t)B * U +
                                2 * (size_t)B * T * U);
    }
};

// one warp per row of am (rows < nA) or lm: its max and exp(x - max)
constexpr int SW = 8;                                      // warps per CTA
__global__ void __launch_bounds__(SW * 32)
simple_exp_rows_kernel(const float* __restrict__ am, const float* __restrict__ lm, SimpleScratch sc, long nA,
                       long nrows, int V) {
    const int lane = threadIdx.x & 31;
    for (long row = (long)blockIdx.x * SW + (threadIdx.x >> 5); row < nrows; row += (long)gridDim.x * SW) {
        const bool is_a = row < nA;
        const long r = is_a ? row : row - nA;
        const float* x = (is_a ? am : lm) + r * V;
        float* e = (is_a ? sc.ea : sc.el) + r * V;
        float m = -INFINITY;
        for (int v = lane; v < V; v += 32) m = fmaxf(m, x[v]);
        m = warp_max(m);
        for (int v = lane; v < V; v += 32) e[v] = expf(x[v] - m);
        if (lane == 0) (is_a ? sc.amax : sc.lmax)[r] = m;
    }
}

// N(t,u) by a direct online log-sum-exp over v in ascending order (the fallback)
__device__ float direct_lse(const float* a, const float* l, int V) {
    float m = -INFINITY, s = 0.f;
    for (int v = 0; v < V; ++v) {
        const float x = a[v] + l[v];
        const float nm = fmaxf(m, x);
        s = (m == -INFINITY ? 0.f : s * expf(m - nm)) + expf(x - nm);
        m = nm;
    }
    return m + logf(s);
}

// one thread per cell: N from the product (or the fallback), then denom / lpb / lpl
__global__ void simple_stats_kernel(const float* __restrict__ am, const float* __restrict__ lm,
                                    const int* __restrict__ labels, const int* __restrict__ xlen,
                                    const int* __restrict__ ylen, SimpleScratch sc, Ws w, int B, int maxT, int maxU,
                                    int V, int blank) {
    const long ncells = (long)B * maxT * maxU;
    for (long cell = (long)blockIdx.x * blockDim.x + threadIdx.x; cell < ncells; cell += (long)gridDim.x * blockDim.x) {
        const int u = (int)(cell % maxU);
        const long bt = cell / maxU;
        const int t = (int)(bt % maxT), b = (int)(bt / maxT);
        const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
        if (t >= Tn || u >= Un) continue;
        const long bu = (long)b * maxU + u;
        const float* a = am + bt * V;
        const float* l = lm + bu * V;
        const float P = sc.prod[cell];
        const float N = P >= SIMPLE_MIN_P ? sc.amax[bt] + sc.lmax[bu] + logf(P) : direct_lse(a, l, V);
        const float d = -N;
        const int lab = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
        w.denom[cell] = d;
        w.lpb[cell] = d + a[blank] + l[blank];
        w.lpl[cell] = lab >= 0 ? d + a[lab] + l[lab] : d;
    }
}

// ---------------------------------------------------------------------------------------------
// 2. simple-loss backward.  With a = alpha, be = beta, ll = ll_fwd[b], d = -N of cell (t,u):
//      c_all(t,u) = a + be - ll + d                     occ(t,u) * softmax_v = exp(c_all + am[t,v] + lm[u,v])
//      gb(t,u)    = exp(a + lpb + beta(t+1,u) - ll)     (t < T-1; exp(a + lpb - ll) at the final cell; else 0)
//      ge(t,u)    = exp(a + lpl + beta(t,u+1) - ll)     (u < U-1; else 0)
//    G(t,u) = exp(c_all + amax[t] + lmax[u]) on product cells (0 on fallback and padded cells), so that
//    sum_u occ softmax_v = exp(am - amax)[t,v] (G . exp(lm - lmax))[t,v] + the fallback cells' direct terms;
//    d am[t,v] = that - [v = blank] sum_u gb - sum_u [v = y_u] ge, d lm the same over t; both scaled by
//    host_scale * gscale.  The per-cell scalars of the finishing passes are staged CH at a time in shared memory.
// ---------------------------------------------------------------------------------------------
constexpr int CH = 256;
struct CellScalars { float c_all, gb, ge; int fallback; };

__device__ __forceinline__ CellScalars cell_scalars(const Ws& w, const SimpleScratch& sc, long cell, int t, int u,
                                                    int Tn, int Un, int maxU, float ll) {
    const float a = w.alphas[cell], d = w.denom[cell];
    CellScalars c;
    c.c_all = a + w.betas[cell] - ll + d;
    c.gb = (t < Tn - 1) ? expf(a + w.lpb[cell] + w.betas[cell + maxU] - ll)
                        : (u == Un - 1 ? expf(a + w.lpb[cell] - ll) : 0.f);
    c.ge = (u < Un - 1) ? expf(a + w.lpl[cell] + w.betas[cell + 1] - ll) : 0.f;
    c.fallback = !(sc.prod[cell] >= SIMPLE_MIN_P);
    return c;
}

__global__ void simple_g_kernel(const int* __restrict__ xlen, const int* __restrict__ ylen, Ws w, SimpleScratch sc,
                                int B, int maxT, int maxU) {
    const long ncells = (long)B * maxT * maxU;
    for (long cell = (long)blockIdx.x * blockDim.x + threadIdx.x; cell < ncells; cell += (long)gridDim.x * blockDim.x) {
        const int u = (int)(cell % maxU);
        const long bt = cell / maxU;
        const int t = (int)(bt % maxT), b = (int)(bt / maxT);
        const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
        float g = 0.f;
        if (t < Tn && u < Un && sc.prod[cell] >= SIMPLE_MIN_P)
            g = expf(w.alphas[cell] + w.betas[cell] - w.ll_fwd[b] + w.denom[cell] + sc.amax[bt] +
                     sc.lmax[(long)b * maxU + u]);
        sc.G[cell] = g;
    }
}

// one CTA per (b, t): d am[b, t, :] in place over the product (G . exp(lm - lmax))[t, :]
__global__ void __launch_bounds__(256, 1)
simple_dam_kernel(const float* __restrict__ am, const float* __restrict__ lm, const int* __restrict__ labels,
                  const int* __restrict__ xlen, const int* __restrict__ ylen, Ws w, SimpleScratch sc,
                  const float* __restrict__ gscale, int per_batch, float hscale, float* __restrict__ dam, int maxT,
                  int maxU, int V, int blank) {
    __shared__ CellScalars cs[CH];
    __shared__ int lab[CH];
    const long bt = blockIdx.x;
    const int t = (int)(bt % maxT), b = (int)(bt / maxT);
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    float* o = dam + bt * V;
    if (t >= Tn) {
        for (int v = threadIdx.x; v < V; v += blockDim.x) o[v] = 0.f;
        return;
    }
    const float g = hscale * (gscale ? gscale[per_batch ? b : 0] : 1.f);
    const float ll = w.ll_fwd[b];
    const float* a = am + bt * V;
    const float* ea = sc.ea + bt * V;
    const float* l = lm + (long)b * maxU * V;
    for (int v0 = 0; v0 < V; v0 += blockDim.x) {
        const int v = v0 + threadIdx.x;
        float acc = v < V ? ea[v] * o[v] : 0.f, gbs = 0.f;
        for (int u0 = 0; u0 < Un; u0 += CH) {
            const int n = min(CH, Un - u0);
            __syncthreads();
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const int u = u0 + i;
                cs[i] = cell_scalars(w, sc, bt * maxU + u, t, u, Tn, Un, maxU, ll);
                lab[i] = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
            }
            __syncthreads();
            for (int i = 0; i < n; ++i) {
                const CellScalars c = cs[i];
                gbs += c.gb;
                if (v < V) {
                    if (c.fallback) acc += expf(c.c_all + a[v] + l[(long)(u0 + i) * V + v]);
                    if (v == lab[i]) acc -= c.ge;
                }
            }
        }
        if (v < V) o[v] = (acc - (v == blank ? gbs : 0.f)) * g;
    }
}

// one CTA per (b, u): d lm[b, u, :] in place over the product (G^T . exp(am - amax))[u, :]
__global__ void __launch_bounds__(256, 1)
simple_dlm_kernel(const float* __restrict__ am, const float* __restrict__ lm, const int* __restrict__ labels,
                  const int* __restrict__ xlen, const int* __restrict__ ylen, Ws w, SimpleScratch sc,
                  const float* __restrict__ gscale, int per_batch, float hscale, float* __restrict__ dlm, int maxT,
                  int maxU, int V, int blank) {
    __shared__ CellScalars cs[CH];
    const long bu = blockIdx.x;
    const int u = (int)(bu % maxU), b = (int)(bu / maxU);
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    float* o = dlm + bu * V;
    if (u >= Un || Tn == 0) {
        for (int v = threadIdx.x; v < V; v += blockDim.x) o[v] = 0.f;
        return;
    }
    const float g = hscale * (gscale ? gscale[per_batch ? b : 0] : 1.f);
    const float ll = w.ll_fwd[b];
    const int lab = (u < Un - 1) ? labels[b * (maxU - 1) + u] : -1;
    const float* l = lm + bu * V;
    const float* el = sc.el + bu * V;
    const float* a = am + (long)b * maxT * V;
    for (int v0 = 0; v0 < V; v0 += blockDim.x) {
        const int v = v0 + threadIdx.x;
        float acc = v < V ? el[v] * o[v] : 0.f, gbs = 0.f, ges = 0.f;
        for (int t0 = 0; t0 < Tn; t0 += CH) {
            const int n = min(CH, Tn - t0);
            __syncthreads();
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const int t = t0 + i;
                cs[i] = cell_scalars(w, sc, ((long)b * maxT + t) * maxU + u, t, u, Tn, Un, maxU, ll);
            }
            __syncthreads();
            for (int i = 0; i < n; ++i) {
                const CellScalars c = cs[i];
                gbs += c.gb;
                ges += c.ge;
                if (c.fallback && v < V) acc += expf(c.c_all + a[(long)(t0 + i) * V + v] + l[v]);
            }
        }
        if (v < V) o[v] = (acc - (v == blank ? gbs : 0.f) - (v == lab ? ges : 0.f)) * g;
    }
}

// ---------------------------------------------------------------------------------------------
// 3. band choice: one CTA per utterance; thread t scores frame t's windows, thread 0 then runs the two passes over
//    the frames in shared memory
// ---------------------------------------------------------------------------------------------
__global__ void band_choice_kernel(const int* __restrict__ xlen, const int* __restrict__ ylen, Ws w, int maxT,
                                   int maxU, int R, int* __restrict__ s_begin, int* __restrict__ nopath) {
    extern __shared__ int sb[];                            // [maxT]
    const int b = blockIdx.x;
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    const int Rb = min(R, Un), S = Un - Rb;                // windows s = 0 .. S
    const float ll = w.ll_fwd[b];
    for (int t = threadIdx.x; t < Tn; t += blockDim.x) {
        const long c0 = ((long)b * maxT + t) * maxU;
        int best = 0;
        float best_score = 0.f;
        for (int s = 0; s <= S; ++s) {
            float sc = 0.f;
            for (int u = s; u < s + Rb; ++u) sc += expf(w.alphas[c0 + u] + w.betas[c0 + u] - ll);
            if (s == 0 || sc > best_score) { best = s; best_score = sc; }
        }
        sb[t] = best;
    }
    __syncthreads();
    if (threadIdx.x == 0 && Tn > 0) {
        int prev = 0;
        sb[0] = 0;
        for (int t = 1; t < Tn; ++t) {
            prev = min(max(sb[t], prev), prev + Rb - 1);
            sb[t] = prev;
        }
        sb[Tn - 1] = S;
        for (int t = Tn - 2; t >= 0; --t) sb[t] = max(sb[t], sb[t + 1] - (Rb - 1));
        nopath[b] = sb[0] > 0;
    } else if (threadIdx.x == 0) {
        nopath[b] = 0;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < maxT; t += blockDim.x) s_begin[(long)b * maxT + t] = t < Tn ? sb[t] : 0;
}

// ---------------------------------------------------------------------------------------------
// 4. band hidden rows: one CTA per (b, t), zero padding rows (band_row_live)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float tanh_fast(float x) {     // MUFU.TANH, as eb_joint_hidden_fwd's bf16 kernel
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <bool BF16>
__global__ void band_hidden_kernel(const float* __restrict__ ep, const float* __restrict__ dp,
                                   const int* __restrict__ xlen, const int* __restrict__ ylen,
                                   const int* __restrict__ s_begin, void* __restrict__ hid, int maxT, int maxU, int R,
                                   int J) {
    const long bt = blockIdx.x;
    const int t = (int)(bt % maxT), b = (int)(bt / maxT);
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    const int s = s_begin[bt];
    const float* e = ep + bt * J;
    const float* d = dp + (long)b * maxU * J;
    for (int i = threadIdx.x; i < R * J; i += blockDim.x) {
        const int r = i / J, j = i - r * J;
        const bool live = band_row_live(t, Tn, Un, R, s, r);
        if (BF16) {
            reinterpret_cast<__nv_bfloat16*>(hid)[bt * R * J + i] =
                __float2bfloat16_rn(live ? tanh_fast(e[j] + d[(long)(s + r) * J + j]) : 0.f);
        } else {
            reinterpret_cast<float*>(hid)[bt * R * J + i] = live ? tanhf(e[j] + d[(long)(s + r) * J + j]) : 0.f;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 5. banded d-pre reduction.  dpre = dh * (1 - h^2) for fp32 d hidden (h given), or the bf16 d(pre-activation) of
//    eb_gemm_bf16_dtanh (h = NULL).
// ---------------------------------------------------------------------------------------------
template <bool BF16>
__device__ __forceinline__ float dpre_at(const void* dx, const float* h, long i) {
    if (BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(dx)[i]);
    const float hv = h[i];
    return reinterpret_cast<const float*>(dx)[i] * (1.f - hv * hv);
}

// dep[b,t,:] = sum over the live rows r of dpre[b,t,r,:] in ascending r; one CTA per (b, t)
template <bool BF16>
__global__ void band_dep_kernel(const void* __restrict__ dx, const float* __restrict__ h,
                                const int* __restrict__ xlen, const int* __restrict__ ylen,
                                const int* __restrict__ s_begin, float* __restrict__ dep, int maxT, int maxU, int R,
                                int J) {
    const long bt = blockIdx.x;
    const int t = (int)(bt % maxT), b = (int)(bt / maxT);
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    const int s = s_begin[bt];
    for (int j = threadIdx.x; j < J; j += blockDim.x) {
        float acc = 0.f;
        for (int r = 0; r < R; ++r)
            if (band_row_live(t, Tn, Un, R, s, r)) acc += dpre_at<BF16>(dx, h, (bt * R + r) * J + j);
        dep[bt * J + j] = acc;
    }
}

// ddp[b,u,:] = sum over the frames t whose band covers u, in ascending t, of dpre[b,t,u - s_begin[t],:]; one CTA per
// (b, u).  With s[t] non-decreasing over t < T_b, {t : s[t] <= u < s[t] + Rb} = [first t with s[t] > u - Rb, first t
// with s[t] > u): two binary searches.  A frame with a negative start has no live row and adds nothing.
template <bool BF16>
__global__ void band_ddp_kernel(const void* __restrict__ dx, const float* __restrict__ h,
                                const int* __restrict__ xlen, const int* __restrict__ ylen,
                                const int* __restrict__ s_begin, float* __restrict__ ddp, int maxT, int maxU, int R,
                                int J) {
    const long bu = blockIdx.x;
    const int u = (int)(bu % maxU), b = (int)(bu / maxU);
    const int Tn = clamp_T(xlen[b], maxT), Un = clamp_U(ylen[b], maxU);
    const int Rb = min(R, Un);
    const int* s = s_begin + (long)b * maxT;
    auto first_above = [&](int x) {                       // first t < Tn with s[t] > x (Tn if none)
        int lo = 0, hi = Tn;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (s[mid] > x) hi = mid; else lo = mid + 1;
        }
        return lo;
    };
    const int t0 = u < Un ? first_above(u - Rb) : 0, t1 = u < Un ? first_above(u) : 0;
    for (int j = threadIdx.x; j < J; j += blockDim.x) {
        float acc = 0.f;
        for (int t = t0; t < t1; ++t)
            if (band_row_live(t, Tn, Un, R, s[t], u - s[t]))
                acc += dpre_at<BF16>(dx, h, ((((long)b * maxT + t) * R) + u - s[t]) * J + j);
        ddp[bu * J + j] = acc;
    }
}

inline bool bad_lengths(const int* xlen, const int* ylen, int B, int maxT, int maxU) {
    return !xlen || !ylen || B <= 0 || maxT <= 0 || maxU <= 0 || maxU > 1024;
}
inline bool bad_R(int R) { return R < 2 || R > 64; }
inline int grid_cap(long n, int per) {
    const long blocks = (n + per - 1) / per, cap = (long)eb_num_sms() * 16;
    return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}
constexpr int BAND_CHOICE_MAX_T = 48 * 1024 / 4;          // s_begin of one utterance in static-size shared memory

}  // namespace

EB_API size_t eb_rnnt_simple_scratch_bytes(int B, int maxT, int maxU, int V) {
    return SimpleScratch::bytes(B, maxT, maxU, V);
}

EB_API int eb_rnnt_simple_stats(const float* am, const float* lm, const int* labels, const int* xlen, const int* ylen,
                                int B, int maxT, int maxU, int V, int blank, void* scratch, void* workspace,
                                void* stream) {
    if (!am || !lm || !scratch || !workspace || (!labels && maxU > 1) || bad_lengths(xlen, ylen, B, maxT, maxU) ||
        V <= 0 || blank < 0 || blank >= V)
        return EB_ERR_INVALID;
    cudaStream_t st = ST(stream);
    const SimpleScratch sc(scratch, B, maxT, maxU, V);
    const long nA = (long)B * maxT, nrows = nA + (long)B * maxU;
    simple_exp_rows_kernel<<<grid_cap(nrows, SW), SW * 32, 0, st>>>(am, lm, sc, nA, nrows, V);
    EB_CHECK_LAUNCH();
    for (int b = 0; b < B; ++b) {                       // prod[b] = exp(am - amax)[b] . exp(lm - lmax)[b]^T  [T, U]
        const int rc = eb_gemm_f32(sc.ea + (size_t)b * maxT * V, V, 1, sc.el + (size_t)b * maxU * V, 1, V,
                                   sc.prod + (size_t)b * maxT * maxU, maxU, nullptr, maxT, maxU, V, 1.f, 0.f, stream);
        if (rc) return rc;
    }
    simple_stats_kernel<<<grid_cap((long)B * maxT * maxU, 256), 256, 0, st>>>(
        am, lm, labels, xlen, ylen, sc, Ws(workspace, B, maxT, maxU), B, maxT, maxU, V, blank);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_rnnt_simple_bwd(const float* am, const float* lm, const int* labels, const int* xlen, const int* ylen,
                              int B, int maxT, int maxU, int V, int blank, void* scratch, const void* workspace,
                              const float* gscale_dev, int gscale_per_batch, double host_scale, float* dam,
                              float* dlm, void* stream) {
    if (!am || !lm || !scratch || !workspace || !dam || !dlm || (!labels && maxU > 1) ||
        bad_lengths(xlen, ylen, B, maxT, maxU) || V <= 0 || blank < 0 || blank >= V)
        return EB_ERR_INVALID;
    cudaStream_t st = ST(stream);
    const SimpleScratch sc(scratch, B, maxT, maxU, V);
    const Ws w(const_cast<void*>(workspace), B, maxT, maxU);
    simple_g_kernel<<<grid_cap((long)B * maxT * maxU, 256), 256, 0, st>>>(xlen, ylen, w, sc, B, maxT, maxU);
    EB_CHECK_LAUNCH();
    for (int b = 0; b < B; ++b) {
        const float* G = sc.G + (size_t)b * maxT * maxU;
        // dam[b] = G [T, U] . exp(lm - lmax)[b] [U, V];  dlm[b] = G^T [U, T] . exp(am - amax)[b] [T, V]
        int rc = eb_gemm_f32(G, maxU, 1, sc.el + (size_t)b * maxU * V, V, 1, dam + (size_t)b * maxT * V, V, nullptr,
                             maxT, V, maxU, 1.f, 0.f, stream);
        if (!rc) rc = eb_gemm_f32(G, 1, maxU, sc.ea + (size_t)b * maxT * V, V, 1, dlm + (size_t)b * maxU * V, V,
                                  nullptr, maxU, V, maxT, 1.f, 0.f, stream);
        if (rc) return rc;
    }
    simple_dam_kernel<<<B * maxT, 256, 0, st>>>(am, lm, labels, xlen, ylen, w, sc, gscale_dev, gscale_per_batch,
                                                (float)host_scale, dam, maxT, maxU, V, blank);
    simple_dlm_kernel<<<B * maxU, 256, 0, st>>>(am, lm, labels, xlen, ylen, w, sc, gscale_dev, gscale_per_batch,
                                                (float)host_scale, dlm, maxT, maxU, V, blank);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_rnnt_band_choice(const int* xlen, const int* ylen, int B, int maxT, int maxU, int R,
                               const void* workspace, int* s_begin, int* nopath, void* stream) {
    if (!workspace || !s_begin || !nopath || bad_lengths(xlen, ylen, B, maxT, maxU) || bad_R(R) ||
        maxT > BAND_CHOICE_MAX_T)
        return EB_ERR_INVALID;
    band_choice_kernel<<<B, 256, maxT * sizeof(int), ST(stream)>>>(
        xlen, ylen, Ws(const_cast<void*>(workspace), B, maxT, maxU), maxT, maxU, R, s_begin, nopath);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_joint_band_hidden_fwd(const float* ep, const float* dp, const int* xlen, const int* ylen,
                                    const int* s_begin, void* hidden, int hidden_bf16, int B, int maxT, int maxU,
                                    int R, int J, void* stream) {
    if (!ep || !dp || !s_begin || !hidden || bad_lengths(xlen, ylen, B, maxT, maxU) || bad_R(R) || J <= 0 ||
        (hidden_bf16 && (reinterpret_cast<uintptr_t>(hidden) & 15)))
        return EB_ERR_INVALID;
    if (hidden_bf16)
        band_hidden_kernel<true><<<B * maxT, 256, 0, ST(stream)>>>(ep, dp, xlen, ylen, s_begin, hidden, maxT, maxU, R,
                                                                   J);
    else
        band_hidden_kernel<false><<<B * maxT, 256, 0, ST(stream)>>>(ep, dp, xlen, ylen, s_begin, hidden, maxT, maxU,
                                                                    R, J);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_joint_band_dpre_reduce(const void* dx, const float* hidden, int is_bf16, const int* xlen,
                                     const int* ylen, const int* s_begin, float* dep, float* ddp, int B, int maxT,
                                     int maxU, int R, int J, void* stream) {
    if (!dx || !s_begin || !dep || !ddp || (!is_bf16 && !hidden) || bad_lengths(xlen, ylen, B, maxT, maxU) ||
        bad_R(R) || J <= 0 || (is_bf16 && (reinterpret_cast<uintptr_t>(dx) & 15)))
        return EB_ERR_INVALID;
    if (is_bf16) {
        band_dep_kernel<true><<<B * maxT, 256, 0, ST(stream)>>>(dx, nullptr, xlen, ylen, s_begin, dep, maxT, maxU, R,
                                                              J);
        band_ddp_kernel<true><<<B * maxU, 256, 0, ST(stream)>>>(dx, nullptr, xlen, ylen, s_begin, ddp, maxT, maxU, R,
                                                                J);
    } else {
        band_dep_kernel<false><<<B * maxT, 256, 0, ST(stream)>>>(dx, hidden, xlen, ylen, s_begin, dep, maxT, maxU, R,
                                                               J);
        band_ddp_kernel<false><<<B * maxU, 256, 0, ST(stream)>>>(dx, hidden, xlen, ylen, s_begin, ddp, maxT, maxU, R,
                                                                 J);
    }
    EB_CHECK_LAUNCH();
    return EB_OK;
}
