// w2v.cu -- the wav2vec pre-training head (rnnt/wav2vec.py, modules/softmax_vector_quantizer.py): span mask and row
// gathers, the features penalty, the Gumbel vector quantizer and its perplexities, the cosine contrastive logits and
// the InfoNCE cross-entropy, forward and backward.
//
// Masked frames are given per utterance as idx [B, M] (ascending frame numbers, the row-major order of x[mask]) and
// inv [B, T] (m for a masked frame, -1 otherwise).  Every reduction adds in a fixed order (warp trees over fixed lane
// maps, loops in index order): no float atomics, the same bits on every run.  No entry reads device memory on the host.
//
//   eb_w2v_mask_fwd      : out = x with mask_emb in the masked rows.
//   eb_w2v_keep_rows     : out = x with the masked rows zeroed (the mask's backward).
//   eb_w2v_gather        : out[b, m] = x[b, idx[b, m]].
//   eb_w2v_scatter       : out[b, t] = x[b, inv[b, t]] or 0 (the gather's backward, a plain write: rows are unique).
//   eb_w2v_sq_mean       : out = sum(x^2) / n, one CTA.       eb_w2v_scale: out = x * g[0] * alpha.
//   eb_w2v_quant_fwd     : per (row, group): clean argmax k0 and softmax p, noisy soft s = softmax((l + g) / tau), hard
//                          k = argmax s (first on ties), st = (1 - s_k) + s_k in fp32, the straight-through matrix X
//                          (st at k, 0 elsewhere) and q = st * vars[k]; eval (noise NULL): X one-hot at k0, q = vars[k0].
//   eb_w2v_quant_stats   : one CTA: the perplexities from sum_r p and the counts of k0, and the coefficients
//                          d prob_ppl / d avg_probs.
//   eb_w2v_quant_bwd     : d logits = (1/tau) J_s d_soft + (g_ppl / N) J_p coef, J the softmax Jacobians.
//   eb_w2v_logits_fwd    : cosine logits [K+1, B, M] / logit_temp, -inf where a negative equals the positive (there
//                          the saved cosine is -inf too: it carries the mask to the backward).
//   eb_w2v_logits_bwd    : the dense per-utterance weights A, AC [B, M, M], then dxp and dyp; a masked candidate (-inf
//                          cosine) contributes nothing, as the reference's index_put of -inf passes no gradient.
//   eb_w2v_ce            : one CTA: InfoNCE cross-entropy (target 0) over the rows (m, b), its unscaled gradient,
//                          the summed loss and the count of correct rows.
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace {

#define ST(s) reinterpret_cast<cudaStream_t>(s)

__global__ void mask_fwd_kernel(const float* __restrict__ x, const float* __restrict__ emb, const int* __restrict__ inv,
                                float* __restrict__ out, long rows, int D, int zero) {
    const long n = rows * D;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long r = i / D;
        out[i] = inv[r] >= 0 ? (zero ? 0.f : emb[i - r * D]) : x[i];
    }
}

__global__ void gather_kernel(const float* __restrict__ x, const int* __restrict__ idx, float* __restrict__ out, int B,
                              int T, int M, int D) {
    const long n = (long)B * M * D;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long bm = i / D;
        const int d = (int)(i - bm * D), b = (int)(bm / M);
        out[i] = x[((long)b * T + idx[bm]) * D + d];
    }
}

__global__ void scatter_kernel(const float* __restrict__ x, const int* __restrict__ inv, float* __restrict__ out, int B,
                               int T, int M, int D) {
    const long n = (long)B * T * D;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long bt = i / D;
        const int d = (int)(i - bt * D), b = (int)(bt / T), m = inv[bt];
        out[i] = m >= 0 ? x[((long)b * M + m) * D + d] : 0.f;
    }
}

// one CTA of 1024: thread t adds elements t, t + 1024, ... in order, then the fixed block tree
__global__ void __launch_bounds__(1024) sq_mean_kernel(const float* __restrict__ x, long n, float* __restrict__ out) {
    __shared__ float sh[33];
    float acc = 0.f;
    for (long i = threadIdx.x; i < n; i += blockDim.x) acc = fmaf(x[i], x[i], acc);
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) out[0] = acc / (float)n;
}

__global__ void scale_kernel(const float* __restrict__ x, const float* __restrict__ g, float alpha, long n,
                             float* __restrict__ out) {
    const float s = g[0] * alpha;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        out[i] = x[i] * s;
}

// argmax / max over a warp's strided slice: first index on ties (index order breaks value ties)
__device__ __forceinline__ void warp_argmax(float& v, int& k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int ok = __shfl_xor_sync(0xffffffffu, k, o);
        if (ov > v || (ov == v && ok < k)) { v = ov; k = ok; }
    }
}
__device__ __forceinline__ void warp_argmin(float& v, int& k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int ok = __shfl_xor_sync(0xffffffffu, k, o);
        if (ov < v || (ov == v && ok < k)) { v = ov; k = ok; }
    }
}

// one warp per (row r, group g); logits / noise / p / s / X rows are [N, G*V]
__global__ void quant_fwd_kernel(const float* __restrict__ logits, const float* __restrict__ noise,
                                 const float* __restrict__ vars, int N, int G, int V, int vd, float tau,
                                 float* __restrict__ q, float* __restrict__ p, float* __restrict__ s,
                                 float* __restrict__ X, int* __restrict__ k0_out, int* __restrict__ k_out,
                                 float* __restrict__ st_out) {
    const int lane = threadIdx.x & 31;
    const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= (long)N * G) return;
    const int g = (int)(w % G);
    const long base = w * V;                         // (r * G + g) * V
    const float* l = logits + base;
    float mx = -INFINITY;
    int k0 = 0x7fffffff;
    for (int v = lane; v < V; v += 32)
        if (l[v] > mx || k0 == 0x7fffffff) { mx = l[v]; k0 = v; }
    warp_argmax(mx, k0);
    float sum = 0.f;
    for (int v = lane; v < V; v += 32) sum += expf(l[v] - mx);
    sum = warp_sum(sum);
    for (int v = lane; v < V; v += 32) p[base + v] = expf(l[v] - mx) / sum;
    int k = k0;
    float stv = 1.f;
    if (noise) {
        const float* gn = noise + base;
        float zm = -INFINITY;
        for (int v = lane; v < V; v += 32) zm = fmaxf(zm, (l[v] + gn[v]) / tau);
        zm = warp_max(zm);
        float zs = 0.f;
        for (int v = lane; v < V; v += 32) zs += expf((l[v] + gn[v]) / tau - zm);
        zs = warp_sum(zs);
        float sm = -INFINITY;
        int sk = 0x7fffffff;
        for (int v = lane; v < V; v += 32) {
            const float sv = expf((l[v] + gn[v]) / tau - zm) / zs;
            s[base + v] = sv;
            if (sv > sm || sk == 0x7fffffff) { sm = sv; sk = v; }
        }
        warp_argmax(sm, sk);
        k = sk;
        stv = __fadd_rn(__fsub_rn(1.f, sm), sm);     // the reference's y_hard - y_soft.detach() + y_soft at k
    }
    for (int v = lane; v < V; v += 32) X[base + v] = v == k ? stv : 0.f;
    const float* vr = vars + ((long)g * V + k) * vd;
    float* qr = q + w * vd;                          // q [N, G*vd]: row r, group g
    for (int d = lane; d < vd; d += 32) qr[d] = noise ? stv * vr[d] : vr[d];
    if (lane == 0) {
        k0_out[w] = k0;
        k_out[w] = k;
        st_out[w] = stv;
    }
}

// one CTA: psum [G*V] = sum_r p, k0 [N*G] -> out = {prob_ppl, code_ppl}, coef [G*V] = d prob_ppl / d avg_probs
__global__ void __launch_bounds__(1024) quant_stats_kernel(const float* __restrict__ psum, const int* __restrict__ k0,
                                                           int N, int G, int V, float* __restrict__ out,
                                                           float* __restrict__ coef, int* __restrict__ counts) {
    __shared__ float sh[33];
    for (int i = threadIdx.x; i < G * V; i += blockDim.x) counts[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < N * G; i += blockDim.x) atomicAdd(&counts[(i % G) * V + k0[i]], 1);   // integers
    __syncthreads();
    float pp = 0.f, cp = 0.f;
    for (int g = 0; g < G; ++g) {
        float hp = 0.f, hc = 0.f;
        for (int v = threadIdx.x; v < V; v += blockDim.x) {
            const float a = psum[g * V + v] / (float)N;
            const float c = (float)counts[g * V + v] / (float)N;
            hp += a * logf(a + 1e-7f);
            hc += c * logf(c + 1e-7f);
        }
        hp = block_sum(hp, sh);
        hc = block_sum(hc, sh);
        const float ep = expf(-hp);
        pp += ep;
        cp += expf(-hc);
        for (int v = threadIdx.x; v < V; v += blockDim.x) {
            const float a = psum[g * V + v] / (float)N;
            coef[g * V + v] = -ep * (logf(a + 1e-7f) + a / (a + 1e-7f));
        }
    }
    if (threadIdx.x == 0) {
        out[0] = pp;
        out[1] = cp;
    }
}

// one warp per (row, group): dl = (1/tau) s (ds - <s, ds>) + (g_ppl / N) p (c - <p, c>)
__global__ void quant_bwd_kernel(const float* __restrict__ dsoft, const float* __restrict__ s,
                                 const float* __restrict__ p, const float* __restrict__ coef,
                                 const float* __restrict__ g_ppl, int N, int G, int V, float tau,
                                 float* __restrict__ dl) {
    const int lane = threadIdx.x & 31;
    const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= (long)N * G) return;
    const int g = (int)(w % G);
    const long base = w * V;
    const float* c = coef + (long)g * V;
    float a = 0.f, b = 0.f;
    for (int v = lane; v < V; v += 32) {
        if (dsoft) a += s[base + v] * dsoft[base + v];
        if (g_ppl) b += p[base + v] * c[v];
    }
    a = warp_sum(a);
    b = warp_sum(b);
    const float gp = g_ppl ? g_ppl[0] / (float)N : 0.f;
    for (int v = lane; v < V; v += 32) {
        float r = 0.f;
        if (dsoft) r = s[base + v] * (dsoft[base + v] - a) / tau;
        if (g_ppl) r += gp * (p[base + v] * (c[v] - b));
        dl[base + v] = r;
    }
}

// one warp per row of x (rows < nx) or y: n = |row|, h = row / max(n, eps)
__global__ void normalize_kernel(const float* __restrict__ x, const float* __restrict__ y, long nx, long ny, int D,
                                 float eps, float* __restrict__ xh, float* __restrict__ yh, float* __restrict__ xn,
                                 float* __restrict__ yn) {
    const int lane = threadIdx.x & 31;
    const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= nx + ny) return;
    const bool isx = w < nx;
    const long r = isx ? w : w - nx;
    const float* src = (isx ? x : y) + r * D;
    float* dst = (isx ? xh : yh) + r * D;
    float ss = 0.f;
    for (int d = lane; d < D; d += 32) ss = fmaf(src[d], src[d], ss);
    ss = warp_sum(ss);
    const float n = sqrtf(ss), c = fmaxf(n, eps);
    for (int d = lane; d < D; d += 32) dst[d] = src[d] / c;
    if (lane == 0) (isx ? xn : yn)[r] = n;
}

// one warp per (b, m): candidates c = 0 (the positive, row m) and c = 1 + k (row neg[b, m, k])
__global__ void logits_fwd_kernel(const float* __restrict__ xh, const float* __restrict__ yh,
                                  const float* __restrict__ y, const int* __restrict__ neg, int B, int M, int D, int K,
                                  float temp, float* __restrict__ cosv, float* __restrict__ logits) {
    const int lane = threadIdx.x & 31;
    const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= (long)B * M) return;
    const int b = (int)(w / M), m = (int)(w % M);
    const float* xr = xh + w * D;
    const float* ypos = y + w * D;
    const long BM = (long)B * M;
    for (int c = 0; c <= K; ++c) {
        const int j = c == 0 ? m : neg[w * K + c - 1];
        const long jr = (long)b * M + j;
        const float* yr = yh + jr * D;
        const float* yraw = y + jr * D;
        float acc = 0.f;
        bool same = true;
        for (int d = lane; d < D; d += 32) {
            acc = fmaf(xr[d], yr[d], acc);
            same = same && (yraw[d] == ypos[d]);
        }
        acc = warp_sum(acc);
        same = __all_sync(0xffffffffu, same);
        const bool masked = c > 0 && same;
        cosv[c * BM + w] = masked ? -INFINITY : acc;
        logits[c * BM + w] = masked ? -INFINITY : acc / temp;
    }
}

// one thread per (b, r): A[b, r, j] = sum of dlogit over the unmasked candidates of row r that are row j (k order,
// the positive first); AC the same sum of dlogit * cos
__global__ void logits_bwd_a_kernel(const float* __restrict__ dlog, const float* __restrict__ cosv,
                                    const int* __restrict__ neg, int B, int M, int K, float* __restrict__ A,
                                    float* __restrict__ AC) {
    const long w = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= (long)B * M) return;
    const long BM = (long)B * M;
    float* a = A + w * M;
    float* ac = AC + w * M;
    for (int j = 0; j < M; ++j) a[j] = ac[j] = 0.f;
    const int m = (int)(w % M);
    for (int c = 0; c <= K; ++c) {
        if (c > 0 && cosv[c * BM + w] == -INFINITY) continue;       // masked: no gradient
        const int j = c == 0 ? m : neg[w * K + c - 1];
        const float g = dlog[c * BM + w];
        a[j] += g;
        ac[j] += g * cosv[c * BM + w];
    }
}

// warps 0 .. BM-1: dx of row r; warps BM .. 2BM-1: dy of row j.  u = row / |row| (the raw norm: torch's clamp is not
// seen by autograd), c = max(|row|, eps):
//   dx_r = (sum_j A[r, j] yh_j - (sum_j AC[r, j]) ux_r) / (temp c_r),  dy_j = (sum_r A[r, j] xh_r - (sum_r AC[r, j]) uy_j) / (temp c_j)
__global__ void logits_bwd_kernel(const float* __restrict__ A, const float* __restrict__ AC,
                                  const float* __restrict__ xh, const float* __restrict__ yh,
                                  const float* __restrict__ x, const float* __restrict__ y,
                                  const float* __restrict__ xn, const float* __restrict__ yn, int B, int M, int D,
                                  float temp, float eps, float* __restrict__ dx, float* __restrict__ dy) {
    const int lane = threadIdx.x & 31;
    const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long BM = (long)B * M;
    if (w >= 2 * BM) return;
    const bool isx = w < BM;
    const long row = isx ? w : w - BM;
    const int b = (int)(row / M), i = (int)(row % M);
    const float* other = isx ? yh : xh;
    const float* self = (isx ? x : y) + row * D;
    float* out = (isx ? dx : dy) + row * D;
    const float n = (isx ? xn : yn)[row];
    const float c = fmaxf(n, eps);
    // lane-owned accumulators over d = lane + 32 t, up to D = 32 * 16 in registers, further chunks in passes
    for (int d0 = 0; d0 < D; d0 += 32 * 16) {
        float acc[16];
#pragma unroll
        for (int t = 0; t < 16; ++t) acc[t] = 0.f;
        float sc = 0.f;
        for (int o = 0; o < M; ++o) {
            const long ai = isx ? ((long)b * M + i) * M + o : ((long)b * M + o) * M + i;
            const float a = A[ai];
            sc += AC[ai];
            const float* orow = other + ((long)b * M + o) * D;
#pragma unroll
            for (int t = 0; t < 16; ++t) {
                const int d = d0 + lane + 32 * t;
                if (d < D) acc[t] = fmaf(a, orow[d], acc[t]);
            }
        }
#pragma unroll
        for (int t = 0; t < 16; ++t) {
            const int d = d0 + lane + 32 * t;
            if (d < D) {
                const float u = n > 0.f ? self[d] / n : 0.f;
                out[d] = (acc[t] - sc * u) / c / temp;
            }
        }
    }
}

// one CTA of 1024; row i = m * B + b of the [K+1, B, M] logits; warp w takes rows w, w + 32, ...
__global__ void __launch_bounds__(1024) ce_kernel(const float* __restrict__ logits, int B, int M, int C,
                                                  float* __restrict__ grad, float* __restrict__ out) {
    __shared__ float shl[32], shc[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long BM = (long)B * M;
    float lsum = 0.f, csum = 0.f;
    for (long i = wid; i < BM; i += 32) {
        const int m = (int)(i / B), b = (int)(i % B);
        const long col = (long)b * M + m;
        float mx = -INFINITY, mn = INFINITY;
        int kx = 0x7fffffff, kn = 0x7fffffff;
        for (int c = lane; c < C; c += 32) {
            const float v = logits[c * BM + col];
            if (v > mx || kx == 0x7fffffff) { mx = v; kx = c; }
            if (v < mn || kn == 0x7fffffff) { mn = v; kn = c; }
        }
        warp_argmax(mx, kx);
        warp_argmin(mn, kn);
        float se = 0.f;
        for (int c = lane; c < C; c += 32) se += expf(logits[c * BM + col] - mx);
        se = warp_sum(se);
        const float lse = mx + logf(se);
        for (int c = lane; c < C; c += 32)
            grad[c * BM + col] = expf(logits[c * BM + col] - lse) - (c == 0 ? 1.f : 0.f);
        lsum += lse - logits[col];
        csum += (kx == 0 && kn != 0) ? 1.f : 0.f;
    }
    if (lane == 0) {
        shl[wid] = lsum;
        shc[wid] = csum;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float l = 0.f, c = 0.f;
        for (int w = 0; w < 32; ++w) {
            l += shl[w];
            c += shc[w];
        }
        out[0] = l;
        out[1] = c;
    }
}

inline int grid_for(long n, int threads) {
    long b = (n + threads - 1) / threads;
    long cap = (long)eb_num_sms() * 32;
    return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

inline int warp_blocks(long warps) { return (int)((warps * 32 + 255) / 256); }

}  // namespace

EB_API int eb_w2v_mask_fwd(const float* x, const float* mask_emb, const int* inv, float* out, long rows, int D,
                           void* stream) {
    if (!x || !mask_emb || !inv || !out || rows <= 0 || D <= 0) return EB_ERR_INVALID;
    mask_fwd_kernel<<<grid_for(rows * D, 256), 256, 0, ST(stream)>>>(x, mask_emb, inv, out, rows, D, 0);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_keep_rows(const float* x, const int* inv, float* out, long rows, int D, void* stream) {
    if (!x || !inv || !out || rows <= 0 || D <= 0) return EB_ERR_INVALID;
    mask_fwd_kernel<<<grid_for(rows * D, 256), 256, 0, ST(stream)>>>(x, x, inv, out, rows, D, 1);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_gather(const float* x, const int* idx, float* out, int B, int T, int M, int D, void* stream) {
    if (!x || !idx || !out || B <= 0 || T <= 0 || M <= 0 || M > T || D <= 0) return EB_ERR_INVALID;
    gather_kernel<<<grid_for((long)B * M * D, 256), 256, 0, ST(stream)>>>(x, idx, out, B, T, M, D);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_scatter(const float* x, const int* inv, float* out, int B, int T, int M, int D, void* stream) {
    if (!x || !inv || !out || B <= 0 || T <= 0 || M <= 0 || M > T || D <= 0) return EB_ERR_INVALID;
    scatter_kernel<<<grid_for((long)B * T * D, 256), 256, 0, ST(stream)>>>(x, inv, out, B, T, M, D);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_sq_mean(const float* x, long n, float* out, void* stream) {
    if (!x || !out || n <= 0) return EB_ERR_INVALID;
    sq_mean_kernel<<<1, 1024, 0, ST(stream)>>>(x, n, out);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_scale(const float* x, const float* g, float alpha, long n, float* out, void* stream) {
    if (!x || !g || !out || n < 0) return EB_ERR_INVALID;
    if (n == 0) return EB_OK;
    scale_kernel<<<grid_for(n, 256), 256, 0, ST(stream)>>>(x, g, alpha, n, out);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_quant_fwd(const float* logits, const float* noise, const float* vars, int N, int G, int V, int vd,
                            float tau, float* q, float* p, float* s, float* X, int* k0, int* k, float* st,
                            void* stream) {
    if (!logits || !vars || !q || !p || !X || !k0 || !k || !st || N <= 0 || G <= 0 || V <= 0 || vd <= 0 ||
        (noise && (!s || !(tau > 0.f))))
        return EB_ERR_INVALID;
    quant_fwd_kernel<<<warp_blocks((long)N * G), 256, 0, ST(stream)>>>(logits, noise, vars, N, G, V, vd, tau, q, p, s,
                                                                       X, k0, k, st);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_quant_stats(const float* psum, const int* k0, int N, int G, int V, float* out, float* coef,
                              int* counts, void* stream) {
    if (!psum || !k0 || !out || !coef || !counts || N <= 0 || G <= 0 || V <= 0) return EB_ERR_INVALID;
    quant_stats_kernel<<<1, 1024, 0, ST(stream)>>>(psum, k0, N, G, V, out, coef, counts);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_quant_bwd(const float* dsoft, const float* s, const float* p, const float* coef, const float* g_ppl,
                            int N, int G, int V, float tau, float* dlogits, void* stream) {
    if (!dlogits || N <= 0 || G <= 0 || V <= 0 || (dsoft && (!s || !(tau > 0.f))) || (g_ppl && (!p || !coef)))
        return EB_ERR_INVALID;
    quant_bwd_kernel<<<warp_blocks((long)N * G), 256, 0, ST(stream)>>>(dsoft, s, p, coef, g_ppl, N, G, V, tau,
                                                                       dlogits);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_logits_fwd(const float* xp, const float* yp, const int* neg, int B, int M, int D, int K, float temp,
                             float eps, float* xh, float* yh, float* xn, float* yn, float* cosv, float* logits,
                             void* stream) {
    if (!xp || !yp || !neg || !xh || !yh || !xn || !yn || !cosv || !logits || B <= 0 || M <= 1 || D <= 0 || K <= 0 ||
        temp == 0.f || !(eps >= 0.f))
        return EB_ERR_INVALID;
    const long BM = (long)B * M;
    normalize_kernel<<<warp_blocks(2 * BM), 256, 0, ST(stream)>>>(xp, yp, BM, BM, D, eps, xh, yh, xn, yn);
    EB_CHECK_LAUNCH();
    logits_fwd_kernel<<<warp_blocks(BM), 256, 0, ST(stream)>>>(xh, yh, yp, neg, B, M, D, K, temp, cosv, logits);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_logits_bwd(const float* dlogits, const float* cosv, const int* neg, const float* xh, const float* yh,
                             const float* xp, const float* yp, const float* xn, const float* yn, int B, int M, int D,
                             int K, float temp, float eps, float* A, float* AC, float* dxp, float* dyp, void* stream) {
    if (!dlogits || !cosv || !neg || !xh || !yh || !xp || !yp || !xn || !yn || !A || !AC || !dxp || !dyp || B <= 0 ||
        M <= 1 || D <= 0 || K <= 0 || temp == 0.f || !(eps >= 0.f))
        return EB_ERR_INVALID;
    const long BM = (long)B * M;
    logits_bwd_a_kernel<<<(int)((BM + 127) / 128), 128, 0, ST(stream)>>>(dlogits, cosv, neg, B, M, K, A, AC);
    EB_CHECK_LAUNCH();
    logits_bwd_kernel<<<warp_blocks(2 * BM), 256, 0, ST(stream)>>>(A, AC, xh, yh, xp, yp, xn, yn, B, M, D, temp, eps,
                                                                   dxp, dyp);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_w2v_ce(const float* logits, int B, int M, int C, float* grad, float* out, void* stream) {
    if (!logits || !grad || !out || B <= 0 || M <= 0 || C <= 1) return EB_ERR_INVALID;
    ce_kernel<<<1, 1024, 0, ST(stream)>>>(logits, B, M, C, grad, out);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
