// optim.cu -- the reference trainers' optimizers over the flat parameter / gradient buckets (sm_90a):
//
//   eb_opt_sgd_step        torch.optim.SGD (momentum, L2 weight decay)      cli/train.py:135-140, cli/baseline.py:141-146
//   eb_opt_sm3_step        SM3 (momentum = beta = 0)                        modules/optimizer.py:36-189
//   eb_opt_adamw_step      AdamW                                            modules/optimizer.py:237-292
//   eb_opt_novograd_step   Novograd (grad_averaging = False)                modules/optimizer.py:335-399
//   eb_opt_seg_sumsq       per-tensor sum(g^2) in a fixed order; the clip norm and Novograd's per-tensor norm
//   eb_opt_prologue        the clip coefficient, the overflow skip and the per-group step counters, on the device
//
// The bucket is described by a segment table (one eb_opt_seg per tensor) and a tile table.  A tile is a contiguous
// range of one tensor, cut from the tensor's own shape only (whole rows of its last dimension, or pieces of one row),
// so every per-tile partial and therefore every per-tensor sum is independent of where the tensor sits in the bucket.
// Every kernel walks the tile table grid-stride, one tile per block at a time.
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int OPT_THREADS = 256;
constexpr int SM3_COLS = 4096;     // smem column maxima per tile (the tile table's column cap, optim.py mirrors it)
constexpr int SM3_ROWS = 1024;     // smem row maxima per tile (the tile table's row cap)

// ctl[0] = the gradient coefficient (grad_scale x clip), ctl[1] != 0: skip this step
__global__ void prologue_kernel(const float* __restrict__ total, float gscale, float max_norm, int ngroups,
                                int* __restrict__ steps, float* __restrict__ ctl) {
    float coef = gscale, skip = 0.f;
    if (total) {
        const float norm = sqrtf(*total) * fabsf(gscale);
        if (!isfinite(norm)) skip = 1.f;
        else if (max_norm > 0.f) {
            const float c = max_norm / (norm + 1e-6f);            // torch.nn.utils.clip_grad_norm_
            if (c < 1.f) coef *= c;
        }
    }
    ctl[0] = coef;
    ctl[1] = skip;
    if (skip == 0.f)
        for (int g = 0; g < ngroups; ++g) steps[g] += 1;
}

// partial[t] = sum of g^2 over tile t, in a fixed thread assignment and a fixed tree
__global__ void __launch_bounds__(OPT_THREADS)
seg_sumsq_partial_kernel(const float* __restrict__ g, const eb_opt_seg* __restrict__ seg,
                         const eb_opt_tile* __restrict__ tiles, int ntiles, float* __restrict__ partial) {
    __shared__ float sh[33];
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const eb_opt_tile tl = tiles[t];
        const float* x = g + seg[tl.seg].off + tl.start;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        long j = threadIdx.x;
        for (; j + 3 * OPT_THREADS < tl.len; j += 4 * OPT_THREADS) {
            const float x0 = x[j], x1 = x[j + OPT_THREADS], x2 = x[j + 2 * OPT_THREADS], x3 = x[j + 3 * OPT_THREADS];
            a0 += x0 * x0; a1 += x1 * x1; a2 += x2 * x2; a3 += x3 * x3;
        }
        for (; j < tl.len; j += OPT_THREADS) a0 += x[j] * x[j];
        const float s = block_sum((a0 + a1) + (a2 + a3), sh);
        if (threadIdx.x == 0) partial[t] = s;
    }
}

// segsum[s] = the partials of tensor s summed in tile order (fp64); total = the segments summed in order (fp64)
__global__ void __launch_bounds__(1024)
seg_sumsq_reduce_kernel(const eb_opt_seg* __restrict__ seg, int nseg, const float* __restrict__ partial,
                        float* __restrict__ segsum, float* __restrict__ total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int s = w; s < nseg; s += nw) {
        double a = 0.0;
        for (long t = seg[s].tile_begin + lane; t < seg[s].tile_end; t += 32) a += (double)partial[t];
        a = warp_sum(a);
        if (lane == 0) segsum[s] = (float)a;
    }
    if (!total) return;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0;
        for (int s = 0; s < nseg; ++s) a += (double)segsum[s];
        *total = (float)a;
    }
}

// torch.optim.SGD: d = g + wd p; buf = d on the group's first step, else mu buf + d; p -= lr buf (mu = 0: p -= lr d)
__global__ void __launch_bounds__(OPT_THREADS)
sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf,
           const eb_opt_seg* __restrict__ seg, const eb_opt_tile* __restrict__ tiles, int ntiles,
           const __grid_constant__ eb_opt_hyper h, const float* __restrict__ ctl, const int* __restrict__ steps) {
    if (ctl[1] != 0.f) return;
    const float coef = ctl[0];
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const eb_opt_tile tl = tiles[t];
        const eb_opt_seg sg = seg[tl.seg];
        const int grp = (int)sg.group;
        const float lr = (float)h.lr[grp], wd = (float)h.wd[grp], mu = (float)h.b1[grp];
        const bool first = steps[grp] <= 1;
        const long base = sg.off + tl.start;
        for (long j = threadIdx.x; j < tl.len; j += OPT_THREADS) {
            const long i = base + j;
            const float pi = p[i];
            float d = g[i] * coef;
            if (wd != 0.f) d = d + wd * pi;
            if (mu != 0.f) {
                d = first ? d : mu * buf[i] + d;
                buf[i] = d;
            }
            p[i] = pi - lr * d;
        }
    }
}

// the reference's AdamW: m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2, p -= lr sqrt(bc2)/bc1 (wd p + m / (sqrt(v) + eps)),
// the step size formed in fp64 from the group's device step counter as the reference forms it in Python
__global__ void __launch_bounds__(OPT_THREADS)
adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
             const eb_opt_seg* __restrict__ seg, const eb_opt_tile* __restrict__ tiles, int ntiles,
             const __grid_constant__ eb_opt_hyper h, const float* __restrict__ ctl, const int* __restrict__ steps) {
    if (ctl[1] != 0.f) return;
    const float coef = ctl[0];
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const eb_opt_tile tl = tiles[t];
        const eb_opt_seg sg = seg[tl.seg];
        const int grp = (int)sg.group;
        const double b1d = h.b1[grp], b2d = h.b2[grp];
        const double k = (double)steps[grp];
        const float step_size = (float)(h.lr[grp] * sqrt(1.0 - pow(b2d, k)) / (1.0 - pow(b1d, k)));
        const float b1 = (float)b1d, b2 = (float)b2d, c1 = (float)(1.0 - b1d), c2 = (float)(1.0 - b2d);
        const float wd = (float)h.wd[grp], eps = (float)h.eps[grp];
        const long base = sg.off + tl.start;
        for (long j = threadIdx.x; j < tl.len; j += OPT_THREADS) {
            const long i = base + j;
            const float gi = g[i] * coef, pi = p[i];
            const float mi = b1 * m[i] + c1 * gi;
            const float vi = b2 * v[i] + c2 * (gi * gi);
            m[i] = mi;
            v[i] = vi;
            p[i] = pi - step_size * (wd * pi + mi / (sqrtf(vi) + eps));
        }
    }
}

// Novograd, per tensor: n = sum (coef g)^2 = coef^2 segsum, v = (v == 0) ? n : b2 v + (1-b2) n
__global__ void novograd_v_kernel(const float* __restrict__ segsum, const eb_opt_seg* __restrict__ seg, int nseg,
                                  const __grid_constant__ eb_opt_hyper h, const float* __restrict__ ctl,
                                  float* __restrict__ segv) {
    if (ctl[1] != 0.f) return;
    const float coef = ctl[0];
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < nseg; s += gridDim.x * blockDim.x) {
        const int grp = (int)seg[s].group;
        const float n = (coef * coef) * segsum[s], v = segv[s];
        segv[s] = v == 0.f ? n : (float)h.b2[grp] * v + (float)(1.0 - h.b2[grp]) * n;
    }
}

// Novograd, per element: g' = g / (sqrt(v) + eps) + wd p, m = b1 m + g', p -= lr m
__global__ void __launch_bounds__(OPT_THREADS)
novograd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                const float* __restrict__ segv, const eb_opt_seg* __restrict__ seg,
                const eb_opt_tile* __restrict__ tiles, int ntiles, const __grid_constant__ eb_opt_hyper h,
                const float* __restrict__ ctl) {
    if (ctl[1] != 0.f) return;
    const float coef = ctl[0];
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const eb_opt_tile tl = tiles[t];
        const eb_opt_seg sg = seg[tl.seg];
        const int grp = (int)sg.group;
        const float lr = (float)h.lr[grp], wd = (float)h.wd[grp], b1 = (float)h.b1[grp];
        const float denom = sqrtf(segv[tl.seg]) + (float)h.eps[grp];
        const long base = sg.off + tl.start;
        for (long j = threadIdx.x; j < tl.len; j += OPT_THREADS) {
            const long i = base + j;
            const float pi = p[i];
            float gi = (g[i] * coef) / denom;
            if (wd != 0.f) gi = gi + wd * pi;
            const float mi = b1 * m[i] + gi;
            m[i] = mi;
            p[i] = pi - lr * mi;
        }
    }
}

// SM3 (beta = 0).  The tensor is viewed as [R, C] with C its last dimension (1 for a scalar); accumulator `last` is
// indexed by the column, every other accumulator i by (row / rs_i) % n_i.  u = min_i acc_i + g^2,
// p -= lr g / sqrt(u + eps), new acc_i = max of u over every dimension except i.  The maxima go through the tile's
// shared-memory column and row maxima (reduced within the warp first) and then one global atomicMax per column and
// per row and dimension.  u >= 0, so the float's bit pattern orders like the float and the maxima are exact and
// independent of their order.  acc_new is zeroed by the entry; a skipped step copies acc into it instead.
__device__ __forceinline__ void smem_max_warp(unsigned* sh, int key, unsigned bits, bool active) {
    const unsigned mask = __match_any_sync(0xffffffffu, active ? key : -1);
    const unsigned mx = __reduce_max_sync(mask, bits);
    if (active && (threadIdx.x & 31) == __ffs(mask) - 1) atomicMax(sh + key, mx);
}

__global__ void __launch_bounds__(OPT_THREADS)
sm3_kernel(float* __restrict__ p, const float* __restrict__ g, const float* __restrict__ acc,
           float* __restrict__ acc_new, long nacc, const eb_opt_seg* __restrict__ seg,
           const eb_opt_tile* __restrict__ tiles, int ntiles, const __grid_constant__ eb_opt_hyper h,
           const float* __restrict__ ctl) {
    if (ctl[1] != 0.f) {
        for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nacc; i += (long)gridDim.x * blockDim.x)
            acc_new[i] = acc[i];
        return;
    }
    __shared__ unsigned colmax[SM3_COLS];
    __shared__ unsigned rowmax[SM3_ROWS];
    __shared__ float rowacc[SM3_ROWS];                        // min over the row dimensions' accumulators, per row
    const float coef = ctl[0];
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const eb_opt_tile tl = tiles[t];
        const eb_opt_seg* sg = seg + tl.seg;                  // read in place: rank-dependent indexing
        const int grp = (int)sg->group;
        const int last = sg->rank > 1 ? (int)sg->rank - 1 : 0;
        const int len = (int)tl.len, ncols = (int)tl.ncols, nrows = len / ncols;
        const float lr = (float)h.lr[grp], eps = (float)h.eps[grp];
        long rs[3] = {1, 1, 1};                               // row stride of every dimension but the last
#pragma unroll
        for (int d = 2; d >= 0; --d)
            if (d < last - 1) rs[d] = rs[d + 1] * sg->shape[d + 1];
        for (int i = threadIdx.x; i < ncols; i += OPT_THREADS) colmax[i] = 0u;
        for (int r = threadIdx.x; r < nrows; r += OPT_THREADS) {
            rowmax[r] = 0u;
            const long row = tl.r0 + r;
            float a = INFINITY;
#pragma unroll
            for (int d = 0; d < 3; ++d)
                if (d < last) a = fminf(a, acc[sg->acc[d] + (row / rs[d]) % sg->shape[d]]);
            rowacc[r] = a;
        }
        __syncthreads();
        const float* acc_last = acc + sg->acc[last] + tl.c0;
        const float* gt = g + sg->off + tl.start;
        float* pt = p + sg->off + tl.start;
        const int n_iter = (len + OPT_THREADS - 1) / OPT_THREADS * OPT_THREADS;     // whole warps: warp reductions
        for (int j = threadIdx.x; j < n_iter; j += OPT_THREADS) {
            const bool active = j < len;
            const int rr = active ? j / ncols : 0, cc = active ? j - rr * ncols : 0;
            unsigned ubits = 0u;
            if (active) {
                const float a = fminf(acc_last[cc], rowacc[rr]);
                const float gi = gt[j] * coef;
                const float u = a + gi * gi;
                ubits = __float_as_uint(u);
                const float upd = (1.f / sqrtf(u + eps)) * gi;
                pt[j] = pt[j] - lr * upd;
            }
            smem_max_warp(colmax, cc, ubits, active);
            if (last > 0) smem_max_warp(rowmax, rr, ubits, active);
        }
        __syncthreads();
        unsigned* out_last = reinterpret_cast<unsigned*>(acc_new + sg->acc[last] + tl.c0);
        for (int c = threadIdx.x; c < ncols; c += OPT_THREADS) atomicMax(out_last + c, colmax[c]);
        if (last > 0)
            for (int r = threadIdx.x; r < nrows; r += OPT_THREADS) {
                const long row = tl.r0 + r;
#pragma unroll
                for (int d = 0; d < 3; ++d)
                    if (d < last)
                        atomicMax(reinterpret_cast<unsigned*>(acc_new + sg->acc[d] + (row / rs[d]) % sg->shape[d]),
                                  rowmax[r]);
            }
        __syncthreads();                                      // the maxima are refilled by the next tile
    }
}

inline int opt_grid(int ntiles) {
    const int cap = eb_num_sms() * 8;
    return ntiles < cap ? ntiles : cap;
}

inline bool groups_ok(const eb_opt_seg* seg, const eb_opt_tile* tiles, int ntiles, int ngroups) {
    return seg && tiles && ntiles > 0 && ngroups >= 1 && ngroups <= EB_OPT_MAX_GROUPS;
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

EB_API int eb_opt_seg_sumsq(const float* g, const eb_opt_seg* seg, int nseg, const eb_opt_tile* tiles, int ntiles,
                            float* partial, float* segsum, float* total, void* stream) {
    if (!g || !seg || !tiles || !partial || !segsum || nseg <= 0 || ntiles <= 0) return EB_ERR_INVALID;
    seg_sumsq_partial_kernel<<<opt_grid(ntiles), OPT_THREADS, 0, ST(stream)>>>(g, seg, tiles, ntiles, partial);
    EB_CHECK_LAUNCH();
    seg_sumsq_reduce_kernel<<<1, 1024, 0, ST(stream)>>>(seg, nseg, partial, segsum, total);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_opt_prologue(const float* total, float grad_scale, float max_norm, int ngroups, int* steps, float* ctl,
                           void* stream) {
    if (!steps || !ctl || ngroups < 1 || ngroups > EB_OPT_MAX_GROUPS || max_norm < 0.f) return EB_ERR_INVALID;
    prologue_kernel<<<1, 1, 0, ST(stream)>>>(total, grad_scale, max_norm, ngroups, steps, ctl);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_opt_sgd_step(float* p, const float* g, float* buf, const eb_opt_seg* seg, const eb_opt_tile* tiles,
                           int ntiles, eb_opt_hyper h, int ngroups, const float* ctl, const int* steps, void* stream) {
    if (!p || !g || !ctl || !steps || !groups_ok(seg, tiles, ntiles, ngroups)) return EB_ERR_INVALID;
    for (int k = 0; k < ngroups; ++k)
        if (h.b1[k] != 0.0 && !buf) return EB_ERR_INVALID;
    sgd_kernel<<<opt_grid(ntiles), OPT_THREADS, 0, ST(stream)>>>(p, g, buf, seg, tiles, ntiles, h, ctl, steps);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_opt_sm3_step(float* p, const float* g, const float* acc, float* acc_new, long nacc,
                           const eb_opt_seg* seg, const eb_opt_tile* tiles, int ntiles, eb_opt_hyper h, int ngroups,
                           const float* ctl, void* stream) {
    if (!p || !g || !acc || !acc_new || nacc <= 0 || !ctl || !groups_ok(seg, tiles, ntiles, ngroups))
        return EB_ERR_INVALID;
    EB_CUDA(cudaMemsetAsync(acc_new, 0, (size_t)nacc * sizeof(float), ST(stream)));
    sm3_kernel<<<opt_grid(ntiles), OPT_THREADS, 0, ST(stream)>>>(p, g, acc, acc_new, nacc, seg, tiles, ntiles, h, ctl);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_opt_adamw_step(float* p, const float* g, float* m, float* v, const eb_opt_seg* seg,
                             const eb_opt_tile* tiles, int ntiles, eb_opt_hyper h, int ngroups, const float* ctl,
                             const int* steps, void* stream) {
    if (!p || !g || !m || !v || !ctl || !steps || !groups_ok(seg, tiles, ntiles, ngroups)) return EB_ERR_INVALID;
    adamw_kernel<<<opt_grid(ntiles), OPT_THREADS, 0, ST(stream)>>>(p, g, m, v, seg, tiles, ntiles, h, ctl, steps);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_opt_novograd_step(float* p, const float* g, float* m, float* segv, const float* segsum,
                                const eb_opt_seg* seg, int nseg, const eb_opt_tile* tiles, int ntiles,
                                eb_opt_hyper h, int ngroups, const float* ctl, void* stream) {
    if (!p || !g || !m || !segv || !segsum || !ctl || nseg <= 0 || !groups_ok(seg, tiles, ntiles, ngroups))
        return EB_ERR_INVALID;
    novograd_v_kernel<<<(nseg + 255) / 256, 256, 0, ST(stream)>>>(segsum, seg, nseg, h, ctl, segv);
    EB_CHECK_LAUNCH();
    novograd_kernel<<<opt_grid(ntiles), OPT_THREADS, 0, ST(stream)>>>(p, g, m, segv, seg, tiles, ntiles, h, ctl);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
