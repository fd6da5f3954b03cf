// ctc.cu -- the CTC head, loss and greedy decode of CTCEncoder (rnnt/models.py:272-310) for sm_90a.
//
//   1. ctc_log_softmax_fwd_kernel  one warp per row: max, sum of exp(x - max), y = x - max - log(sum); two
//                                  reductions in a fixed order (the tovocab LogSoftmax)
//   2. ctc_log_softmax_bwd_kernel  one warp per row: dx = g - exp(y) * sum(g)
//   3. ctc_lattice_kernel          grid (N, 2): alpha (y = 0) and beta (y = 1) of one utterance over the extended
//                                  label sequence l' = (blank, l1, blank, ..., lS, blank), two states per thread (four
//                                  above 1024 states), the states double-buffered in shared memory, one barrier per
//                                  frame; the frame's log-probs are prefetched CTC_PF frames ahead into registers
//   4. ctc_grad_kernel             grid (T, N): the gradient torch's ctc_loss returns for log_probs,
//                                  exp(lp_v) - sum_{s: l'_s = v} exp(alpha_t(s) + beta_t(s) + nll - lp_v), the states of
//                                  one label summed in increasing s (the lattice kernel links them)
//   5. ctc_greedy_kernel           one CTA per utterance: per-frame argmax, repeats and blanks dropped, the reference's
//                                  whole-row score
//   ctc_viterbi_kernel             forced alignment: the alpha recurrence of 3. with max in place of log-add, one
//                                  back-pointer byte per (t, s), then the backtrace in the same CTA
//
// Arithmetic follows torch's CPU ctc_loss (aten/src/ATen/native/LossCTC.cpp): alpha and beta include the frame's
// emission, a step log-adds its (up to) three predecessors around their maximum, nll = -log p from alpha.  The lattice
// and the label terms of the gradient run in fp64 (inputs and outputs are fp32): |alpha| grows to thousands over a long
// utterance, and fp32 rounding of values that size would move exp(alpha + beta + nll - lp) by ~1e-3 relative.
// Nothing here synchronises with the host or allocates.
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int CTC_MAX_S = 1023;                          // 2S+1 <= 2047 states: four per thread of a 512-thread CTA
constexpr int CTC_PF = 8;                                 // frames of log-probs in flight per state

// log(exp(a) + exp(b) + exp(c)) as torch's ctc_loss computes it: around the maximum, -inf when all three are
__device__ __forceinline__ double lse3(double a, double b, double c) {
    const double m = fmax(a, fmax(b, c));
    if (m == -INFINITY) return -INFINITY;
    return log(exp(a - m) + exp(b - m) + exp(c - m)) + m;
}

__device__ __forceinline__ double lse2(double a, double b) {
    if (a == -INFINITY) return b;
    if (b == -INFINITY) return a;
    const double m = fmax(a, b);
    return log(exp(a - m) + exp(b - m)) + m;
}

// ---------------------------------------------------------------------------------------------
// 1./2. row log-softmax
// ---------------------------------------------------------------------------------------------
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
ctc_log_softmax_fwd_kernel(const float* x, float* y, long rows, int V) {   // y may alias x
    const int lane = threadIdx.x & 31;
    for (long r = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * WARPS) {
        const float* xr = x + r * V;
        float* yr = y + r * V;
        float m = -INFINITY;
        for (int v = lane; v < V; v += 32) m = fmaxf(m, xr[v]);
        m = warp_max(m);
        float s = 0.f;
        for (int v = lane; v < V; v += 32) s += expf(xr[v] - m);
        const float ls = logf(warp_sum(s));
        for (int v = lane; v < V; v += 32) yr[v] = (xr[v] - m) - ls;
    }
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
ctc_log_softmax_bwd_kernel(const float* dy, const float* y, float* dx, long rows, int V) {   // dx may alias dy
    const int lane = threadIdx.x & 31;
    for (long r = (long)blockIdx.x * WARPS + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * WARPS) {
        const float* gr = dy + r * V;
        const float* yr = y + r * V;
        float* dr = dx + r * V;
        float s = 0.f;
        for (int v = lane; v < V; v += 32) s += gr[v];
        s = warp_sum(s);
        for (int v = lane; v < V; v += 32) dr[v] = gr[v] - expf(yr[v]) * s;
    }
}

// ---------------------------------------------------------------------------------------------
// 3. alpha / beta
// ---------------------------------------------------------------------------------------------
struct CtcWs {
    double *alphas, *betas, *ll_fwd, *ll_bwd;            // [N][T][Lmax] x2, [N] x2
    int *lab, *nxt, *first;                              // [N][Lmax] x3: l'_s, next state with l'_s, first of its label
    static size_t bytes(int N, int T, int S) {
        const size_t L = 2 * (size_t)S + 1;
        return 8 * (2 * (size_t)N * T * L + 2 * (size_t)N) + 4 * 3 * (size_t)N * L;
    }
    CtcWs(void* ws, int N, int T, int S) {
        const size_t L = 2 * (size_t)S + 1, n = (size_t)N * T * L;
        double* p = reinterpret_cast<double*>(ws);
        alphas = p; betas = p + n; ll_fwd = p + 2 * n; ll_bwd = ll_fwd + N;
        lab = reinterpret_cast<int*>(ll_bwd + N); nxt = lab + (size_t)N * L; first = nxt + (size_t)N * L;
    }
};

// the utterance's lengths, clamped so that nothing is read outside the log-probs or the label rows
__device__ __forceinline__ void ctc_lens(const int* in_len, const int* tg_len, int b, int T, int S, int& Tb, int& L) {
    Tb = min(max(in_len[b], 0), T);
    L = 2 * min(max(tg_len[b], 0), S) + 1;
}

template <int SLOTS>                                     // states per thread: 2 up to 1024 states, else 4
__global__ void __launch_bounds__(512)
ctc_lattice_kernel(const float* __restrict__ lp, long sn, long st, int T, int V, const int* __restrict__ targets,
                   long ntargets, const int* __restrict__ tg_off, const int* __restrict__ tg_len,
                   const int* __restrict__ in_len, int S, int blank, int zero_inf, CtcWs w, float* __restrict__ costs) {
    extern __shared__ double sm[];
    const int Lmax = 2 * S + 1;
    double* buf = sm;                                    // [2][Lmax]
    int* lab = reinterpret_cast<int*>(sm + 2 * Lmax);   // [Lmax]
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    int Tb, L;
    ctc_lens(in_len, tg_len, b, T, S, Tb, L);
    const long off = tg_off[b];
    for (int s = tid; s < L; s += nt) {
        int c = blank;
        if (s & 1) {
            const long i = off + (s >> 1);
            c = (i >= 0 && i < ntargets) ? targets[i] : -1;   // an index outside the targets: no emission
        }
        lab[s] = c;
    }
    __syncthreads();
    // per slot k (state s = tid + k*nt): its label column (-1: none, never read) and its skip transition
    int col[SLOTS];
    bool skip[SLOTS];
#pragma unroll
    for (int k = 0; k < SLOTS; ++k) {
        const int s = tid + k * nt;
        const int c = s < L ? lab[s] : -1;
        col[k] = (c >= 0 && c < V) ? c : -1;
        if (blockIdx.y == 0)                             // s-2 -> s: s a label state whose label differs from l'_{s-2}
            skip[k] = s < L && (s & 1) && s >= 2 && lab[s] != lab[s - 2];
        else                                             // s+2 -> s in the reversed lattice
            skip[k] = s + 2 < L && (s & 1) && lab[s + 2] != lab[s];
    }
    const float* row0 = lp + (long)b * sn;
    double* base = (blockIdx.y == 0 ? w.alphas : w.betas) + (long)b * T * Lmax;
    const bool fwd = blockIdx.y == 0;
    // frame of step n: n (alpha) or Tb-1-n (beta)
#define CTC_EMIT(k, n) ((col[k] >= 0 && (n) < Tb) ? __ldg(row0 + (long)(fwd ? (n) : Tb - 1 - (n)) * st + col[k]) : -INFINITY)
    float e[SLOTS][CTC_PF], en[SLOTS][CTC_PF];
#pragma unroll
    for (int k = 0; k < SLOTS; ++k)
#pragma unroll
        for (int i = 0; i < CTC_PF; ++i) e[k][i] = CTC_EMIT(k, i);
    for (int n0 = 0; n0 < Tb; n0 += CTC_PF) {
#pragma unroll
        for (int k = 0; k < SLOTS; ++k)
#pragma unroll
            for (int i = 0; i < CTC_PF; ++i) en[k][i] = CTC_EMIT(k, n0 + CTC_PF + i);
#pragma unroll
        for (int i = 0; i < CTC_PF; ++i) {
            const int n = n0 + i;
            if (n >= Tb) break;                          // uniform across the CTA
            const double* pv = buf + ((n - 1) & 1) * Lmax;
            double* cur = buf + (n & 1) * Lmax;
#pragma unroll
            for (int k = 0; k < SLOTS; ++k) {
                const int s = tid + k * nt;
                if (s >= L) continue;
                double v;
                if (fwd) {
                    if (n == 0) v = (s <= 1) ? e[k][i] : -INFINITY;
                    else v = lse3(pv[s], s >= 1 ? pv[s - 1] : -INFINITY, skip[k] ? pv[s - 2] : -INFINITY) + e[k][i];
                } else {
                    if (n == 0) v = (s >= L - 2) ? e[k][i] : -INFINITY;
                    else v = lse3(pv[s], s + 1 < L ? pv[s + 1] : -INFINITY, skip[k] ? pv[s + 2] : -INFINITY) + e[k][i];
                }
                cur[s] = v;
                base[(long)(fwd ? n : Tb - 1 - n) * Lmax + s] = v;
            }
            __syncthreads();
        }
#pragma unroll
        for (int k = 0; k < SLOTS; ++k)
#pragma unroll
            for (int i = 0; i < CTC_PF; ++i) e[k][i] = en[k][i];
    }
#undef CTC_EMIT
    if (tid == 0) {
        const double* last = buf + ((Tb - 1) & 1) * Lmax;
        double ll;
        if (Tb == 0) ll = (L == 1) ? 0.0 : -INFINITY;    // empty input: only the empty target has a path
        else if (fwd) ll = lse2(last[L - 1], L >= 2 ? last[L - 2] : -INFINITY);
        else ll = lse2(last[0], L >= 2 ? last[1] : -INFINITY);
        if (fwd) {
            w.ll_fwd[b] = ll;
            costs[b] = (zero_inf && ll == -INFINITY) ? 0.f : (float)-ll;
        } else {
            w.ll_bwd[b] = ll;
        }
    }
    if (fwd) return;
    // the beta CTA links the states of each label for the gradient: nxt[s] = the next state with label l'_s (-1: none),
    // first[s] = 1 when no earlier state has it.  Labels outside [0, V) belong to no chain.
    int* lb = w.lab + (long)b * Lmax;
    int* nx = w.nxt + (long)b * Lmax;
    int* fs = w.first + (long)b * Lmax;
    for (int s = tid; s < L; s += nt) {
        const int c = lab[s];
        const bool ok = c >= 0 && c < V;
        int q = -1;
        bool first = ok;
        if (ok) {
            for (int s2 = s + 1; s2 < L; ++s2)
                if (lab[s2] == c) { q = s2; break; }
            for (int s2 = s - 1; s2 >= 0 && first; --s2) first = lab[s2] != c;
        }
        lb[s] = c;
        nx[s] = q;
        fs[s] = first;
    }
}

// ---------------------------------------------------------------------------------------------
// 3b. Viterbi alignment: the alpha recurrence of ctc_lattice_kernel with max in place of log-add, in fp64, and one
//     back-pointer byte per (t, s): how many states back the best predecessor lies (0, 1 or 2).  Predecessors are
//     taken in the order s, s-1, s-2, a later one replacing the current only when strictly greater.  At the last frame
//     the last label state L-2 wins unless the final blank L-1 is strictly greater.  Then one thread walks the
//     back-pointers and writes alignment[b, t]; every thread fills frame_logp[b, t] from it.  grid = N; the
//     back-pointers live in shared memory after the states when bp == nullptr, else at bp + b*T*Lmax.
// ---------------------------------------------------------------------------------------------
template <int SLOTS>
__global__ void __launch_bounds__(512, 1)
ctc_viterbi_kernel(const float* __restrict__ lp, long sn, long st, int T, int V, const int* __restrict__ targets,
                   long ntargets, const int* __restrict__ tg_off, const int* __restrict__ tg_len,
                   const int* __restrict__ in_len, int S, int blank, unsigned char* __restrict__ bp_global,
                   int rows, int* __restrict__ alignment, float* __restrict__ frame_logp) {
    extern __shared__ double sm[];
    const int Lmax = 2 * S + 1;
    double* buf = sm;                                    // [2][Lmax]
    int* lab = reinterpret_cast<int*>(sm + 2 * Lmax);   // [Lmax]
    int* ctl = lab + Lmax;                               // [4]: feasible, walk, t, s (no static shared memory)
    unsigned char* stage = reinterpret_cast<unsigned char*>(ctl + 4);   // [rows][Lmax] back-pointer bytes
    unsigned char* bp = bp_global ? bp_global + (long)blockIdx.x * T * Lmax : stage;
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    int Tb, L;
    ctc_lens(in_len, tg_len, b, T, S, Tb, L);
    const long off = tg_off[b];
    for (int s = tid; s < L; s += nt) {
        int c = blank;
        if (s & 1) {
            const long i = off + (s >> 1);
            c = (i >= 0 && i < ntargets) ? targets[i] : -1;
        }
        lab[s] = c;
    }
    __syncthreads();
    int col[SLOTS];
    bool skip[SLOTS];
#pragma unroll
    for (int k = 0; k < SLOTS; ++k) {
        const int s = tid + k * nt;
        const int c = s < L ? lab[s] : -1;
        col[k] = (c >= 0 && c < V) ? c : -1;
        skip[k] = s < L && (s & 1) && s >= 2 && lab[s] != lab[s - 2];
    }
    const float* row0 = lp + (long)b * sn;
#define CTC_EMIT(k, n) ((col[k] >= 0 && (n) < Tb) ? __ldg(row0 + (long)(n) * st + col[k]) : -INFINITY)
    float e[SLOTS][CTC_PF], en[SLOTS][CTC_PF];
#pragma unroll
    for (int k = 0; k < SLOTS; ++k)
#pragma unroll
        for (int i = 0; i < CTC_PF; ++i) e[k][i] = CTC_EMIT(k, i);
    for (int n0 = 0; n0 < Tb; n0 += CTC_PF) {
#pragma unroll
        for (int k = 0; k < SLOTS; ++k)
#pragma unroll
            for (int i = 0; i < CTC_PF; ++i) en[k][i] = CTC_EMIT(k, n0 + CTC_PF + i);
#pragma unroll
        for (int i = 0; i < CTC_PF; ++i) {
            const int n = n0 + i;
            if (n >= Tb) break;                          // uniform across the CTA
            const double* pv = buf + ((n - 1) & 1) * Lmax;
            double* cur = buf + (n & 1) * Lmax;
#pragma unroll
            for (int k = 0; k < SLOTS; ++k) {
                const int s = tid + k * nt;
                if (s >= L) continue;
                double v;
                if (n == 0) {
                    v = (s <= 1) ? (double)e[k][i] : -INFINITY;
                } else {
                    double best = pv[s];
                    int back = 0;
                    if (s >= 1 && pv[s - 1] > best) { best = pv[s - 1]; back = 1; }
                    if (skip[k] && pv[s - 2] > best) { best = pv[s - 2]; back = 2; }
                    v = best + (double)e[k][i];
                    bp[(long)n * Lmax + s] = (unsigned char)back;
                }
                cur[s] = v;
            }
            __syncthreads();
        }
#pragma unroll
        for (int k = 0; k < SLOTS; ++k)
#pragma unroll
            for (int i = 0; i < CTC_PF; ++i) e[k][i] = en[k][i];
    }
#undef CTC_EMIT
    int* al = alignment + (long)b * T;
    float* fl = frame_logp + (long)b * T;
    if (tid == 0) {
        bool ok = Tb > 0;
        int s = 0;
        if (ok) {
            const double* last = buf + ((Tb - 1) & 1) * Lmax;
            s = L - 1;
            if (L >= 2 && !(last[L - 1] > last[L - 2])) s = L - 2;
            ok = last[s] > -INFINITY;
        }
        ctl[0] = ok || (Tb == 0 && L == 1);              // an empty input aligns only the empty target
        ctl[1] = ok;
        ctl[2] = Tb - 1;
        ctl[3] = s;
    }
    __syncthreads();
    const int ok = ctl[0];
    // Backtrace by thread 0 over the back-pointers in shared memory.  When they are in the caller's buffer
    // (rows < T), the CTA first copies the band of the `rows` frames at and below the current t into shared memory, so
    // the walk makes no dependent global load; a band's frames are contiguous bytes.  t is the same in every thread.
    int t = ctl[1] ? ctl[2] : -1;
    while (t >= 0) {
        const int lo = max(0, t - rows + 1);
        if (bp_global) {
            block_copy_bytes(stage, bp + (long)lo * Lmax, (t - lo + 1) * Lmax, tid, nt);
            __syncthreads();
        }
        if (tid == 0) {
            int s = ctl[3];
            for (; t >= lo; --t) {
                al[t] = lab[s];
                if (t > 0) s -= stage[(t - lo) * Lmax + s];
            }
            ctl[2] = t;
            ctl[3] = s;
        }
        __syncthreads();
        t = ctl[2];
        __syncthreads();                                 // every thread has read t before the next band
    }
    for (int t = tid; t < T; t += nt) {
        if (!ok) {
            al[t] = -1;
            fl[t] = -INFINITY;
        } else if (t < Tb) {
            fl[t] = __ldg(row0 + (long)t * st + al[t]);
        } else {
            al[t] = -1;
            fl[t] = 0.f;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 4. gradient
// ---------------------------------------------------------------------------------------------
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
ctc_grad_kernel(const float* __restrict__ lp, long sn, long st, float* __restrict__ grad, long gn, long gt, int T,
                int V, const int* __restrict__ tg_len, const int* __restrict__ in_len, int S, int zero_inf,
                CtcWs w, const float* __restrict__ gscale) {
    const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int Lmax = 2 * S + 1;
    int Tb, L;
    ctc_lens(in_len, tg_len, b, T, S, Tb, L);
    const float* row = lp + (long)b * sn + (long)t * st;
    float* g = grad + (long)b * gn + (long)t * gt;
    const double nll = -w.ll_fwd[b];
    if (t >= Tb || (zero_inf && nll == INFINITY)) {
        for (int v = tid; v < V; v += THREADS) g[v] = 0.f;
        return;
    }
    const float sc = gscale ? gscale[b] : 1.f;
    // exp(lp_v) - exp(-inf + nll - lp_v) for a column of no state: torch's NaN when nll is not finite
    const float none = nll < INFINITY ? 0.f : NAN;
    for (int v = tid; v < V; v += THREADS) g[v] = (expf(row[v]) - none) * sc;
    __syncthreads();                                     // the label columns below overwrite these stores
    const long cell = ((long)b * T + t) * Lmax;
    const double* al = w.alphas + cell;
    const double* be = w.betas + cell;
    const int* lb = w.lab + (long)b * Lmax;
    const int* nx = w.nxt + (long)b * Lmax;
    const int* fs = w.first + (long)b * Lmax;
    for (int s = tid; s < L; s += THREADS) {
        if (!fs[s]) continue;
        double acc = -INFINITY;
        for (int q = s; q >= 0; q = nx[q]) acc = lse2(acc, al[q] + be[q]);   // increasing s
        const int c = lb[s];
        const double x = row[c];
        g[c] = (float)((exp(x) - exp(acc + nll - x)) * (double)sc);
    }
}

// ---------------------------------------------------------------------------------------------
// 5. greedy decode
// ---------------------------------------------------------------------------------------------
// torch.argmax order: NaN wins, ties go to the lowest index
__device__ __forceinline__ bool argmax_before(float v, int i, float b, int bi) {
    if (isnan(v)) return !isnan(b) || i < bi;
    if (isnan(b)) return false;
    return v > b || (v == b && i < bi);
}

constexpr int GREEDY_THREADS = 256;

__global__ void __launch_bounds__(GREEDY_THREADS)
ctc_greedy_kernel(const float* __restrict__ lp, long sb, long st, int T, int V, const int* __restrict__ xlen, int blank,
                  int* __restrict__ ids, int* __restrict__ counts, float* __restrict__ nscore) {
    constexpr int W = GREEDY_THREADS / 32;
    __shared__ int am[GREEDY_THREADS];
    __shared__ float rs[GREEDY_THREADS];
    __shared__ int wcnt[W];
    __shared__ double wsum[W];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Tk = min(max(xlen[b], 0), T);              // the reference slices [:xlen] of the T frames
    const float* row0 = lp + (long)b * sb;
    int prev = -1, cnt = 0;
    double score = 0.0;
    for (int t0 = 0; t0 < Tk; t0 += GREEDY_THREADS) {
        for (int i = warp; i < GREEDY_THREADS && t0 + i < Tk; i += W) {
            const float* row = row0 + (long)(t0 + i) * st;
            float best = -INFINITY, sum = 0.f;
            int bi = 0x7fffffff;
            for (int v = lane; v < V; v += 32) {
                const float x = row[v];
                if (argmax_before(x, v, best, bi)) { best = x; bi = v; }
                sum += x;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (argmax_before(ob, oi, best, bi)) { best = ob; bi = oi; }
            }
            sum = warp_sum(sum);
            if (lane == 0) { am[i] = bi; rs[i] = sum; }
        }
        __syncthreads();
        const int t = t0 + tid;
        const int c = t < Tk ? am[tid] : -1;
        const int p = tid ? (t < Tk ? am[tid - 1] : -1) : prev;
        const bool keep = t < Tk && c != blank && (t == 0 || c != p);
        // compaction: exclusive prefix count of `keep` over the CTA; score: kept whole-row sums in a fixed order
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        const double part = warp_sum(keep ? (double)rs[tid] : 0.0);
        if (lane == 0) { wcnt[warp] = __popc(bal); wsum[warp] = part; }
        __syncthreads();
        int before = cnt, total = 0;
        double chunk = 0.0;
#pragma unroll
        for (int q = 0; q < W; ++q) {
            if (q < warp) before += wcnt[q];
            total += wcnt[q];
            chunk += wsum[q];
        }
        if (keep) ids[(long)b * T + before + __popc(bal & ((1u << lane) - 1u))] = c;
        score += chunk;
        cnt += total;
        prev = am[GREEDY_THREADS - 1];                   // read only when the next chunk exists (then this one is full)
        __syncthreads();
    }
    if (tid == 0) {
        counts[b] = cnt;
        nscore[b] = -(float)score;
    }
}

inline int row_grid(long rows, int warps) {
    const long blocks = (rows + warps - 1) / warps;
    const long cap = (long)eb_num_sms() * 16;
    return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

// shared by the loss entries: a problem the kernels can index without reading outside any buffer
inline bool bad_ctc(const float* lp, const int* tg_len, const int* in_len, int N, int T, int V, int S, int blank,
                    const void* ws) {
    return !lp || !tg_len || !in_len || !ws || N <= 0 || N > 65535 || T < 0 || V <= 0 || S < 0 ||
           S > CTC_MAX_S || blank < 0 || blank >= V;
}

}  // namespace

EB_API int eb_log_softmax_fwd(const float* x, float* y, long rows, int V, void* stream) {
    if (!x || !y || rows < 0 || V <= 0) return EB_ERR_INVALID;
    if (rows == 0) return EB_OK;
    constexpr int WARPS = 8;
    ctc_log_softmax_fwd_kernel<WARPS><<<row_grid(rows, WARPS), WARPS * 32, 0, (cudaStream_t)stream>>>(x, y, rows, V);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_log_softmax_bwd(const float* dy, const float* y, float* dx, long rows, int V, void* stream) {
    if (!dy || !y || !dx || rows < 0 || V <= 0) return EB_ERR_INVALID;
    if (rows == 0) return EB_OK;
    constexpr int WARPS = 8;
    ctc_log_softmax_bwd_kernel<WARPS><<<row_grid(rows, WARPS), WARPS * 32, 0, (cudaStream_t)stream>>>(dy, y, dx, rows, V);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API size_t eb_ctc_workspace_size(int N, int T, int S) {
    if (N <= 0 || T < 0 || S < 0 || S > CTC_MAX_S) return 0;
    return CtcWs::bytes(N, T, S);
}

EB_API int eb_ctc_loss_fwd(const float* log_probs, long stride_n, long stride_t, int N, int T, int V, const int* targets,
                           long ntargets, const int* target_offsets, const int* target_lengths, const int* input_lengths,
                           int S, int blank, int zero_infinity, void* workspace, float* costs, void* stream) {
    if (bad_ctc(log_probs, target_lengths, input_lengths, N, T, V, S, blank, workspace) || !target_offsets || !costs ||
        ntargets < 0 || (!targets && ntargets > 0))
        return EB_ERR_INVALID;
    const int Lmax = 2 * S + 1;
    const int slots = Lmax <= 1024 ? 2 : 4;
    const int threads = ((Lmax + slots - 1) / slots + 31) / 32 * 32;
    const size_t smem = 2 * Lmax * sizeof(double) + Lmax * sizeof(int);
    CtcWs w(workspace, N, T, S);
    if (Lmax <= 1024)
        ctc_lattice_kernel<2><<<dim3(N, 2), threads, smem, (cudaStream_t)stream>>>(
            log_probs, stride_n, stride_t, T, V, targets, ntargets, target_offsets, target_lengths, input_lengths, S,
            blank, zero_infinity, w, costs);
    else
        ctc_lattice_kernel<4><<<dim3(N, 2), threads, smem, (cudaStream_t)stream>>>(
            log_probs, stride_n, stride_t, T, V, targets, ntargets, target_offsets, target_lengths, input_lengths, S,
            blank, zero_infinity, w, costs);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_ctc_loss_bwd(const float* log_probs, long stride_n, long stride_t, float* grad, long grad_stride_n,
                           long grad_stride_t, int N, int T, int V, const int* target_lengths, const int* input_lengths,
                           int S, int blank, int zero_infinity, const void* workspace, const float* gscale, void* stream) {
    if (bad_ctc(log_probs, target_lengths, input_lengths, N, T, V, S, blank, workspace) || !grad ||
        (const void*)grad == (const void*)log_probs)
        return EB_ERR_INVALID;
    if (T == 0) return EB_OK;
    CtcWs w(const_cast<void*>(workspace), N, T, S);
    constexpr int THREADS = 256;
    ctc_grad_kernel<THREADS><<<dim3(T, N), THREADS, 0, (cudaStream_t)stream>>>(
        log_probs, stride_n, stride_t, grad, grad_stride_n, grad_stride_t, T, V, target_lengths, input_lengths, S,
        zero_infinity, w, gscale);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

namespace {

constexpr size_t ALIGN_SMEM_MAX = 227 * 1024;           // opt-in dynamic shared memory per CTA on sm_90

// frames of back-pointers the backtrace stages at a time when they do not all fit in shared memory
constexpr size_t ALIGN_STAGE_BYTES = 64 * 1024;

// dynamic shared memory of ctc_viterbi_kernel: states [2][Lmax] doubles, labels [Lmax] ints, four control ints and
// [rows][Lmax] back-pointer bytes: all T frames when they fit (the back-pointers then live there), else a staging band
// of the caller's buffer.  The kernel has no static shared memory, so the whole opt-in limit is available to this
// buffer.
inline size_t ctc_viterbi_smem(int T, int S, int* rows) {
    const size_t L = 2 * (size_t)S + 1;
    const size_t fixed = L * (2 * sizeof(double) + sizeof(int)) + 4 * sizeof(int);
    *rows = fixed + (size_t)T * L <= ALIGN_SMEM_MAX ? T : (int)(ALIGN_STAGE_BYTES / L);
    return fixed + (size_t)*rows * L;
}

}  // namespace

EB_API size_t eb_ctc_align_workspace_size(int B, int T, int S) {
    if (B <= 0 || T < 0 || S < 0 || S > CTC_MAX_S) return 0;
    int rows;
    ctc_viterbi_smem(T, S, &rows);
    return rows == T ? 0 : (size_t)B * T * (2 * (size_t)S + 1);
}

EB_API int eb_ctc_align(const float* log_probs, long stride_b, long stride_t, int B, int T, int V, const int* targets,
                        long ntargets, const int* tg_off, const int* tg_len, const int* in_len, int S, int blank,
                        void* workspace, int* alignment, float* frame_logp, void* stream) {
    if (!log_probs || !tg_off || !tg_len || !in_len || !alignment || !frame_logp || B <= 0 || B > 65535 || T < 0 ||
        V <= 0 || S < 0 || S > CTC_MAX_S || blank < 0 || blank >= V || ntargets < 0 || (!targets && ntargets > 0) ||
        stride_b < 0 || stride_t < 0)
        return EB_ERR_INVALID;
    int rows;
    const size_t smem = ctc_viterbi_smem(T, S, &rows);
    const bool in_smem = rows == T;
    if (!in_smem && !workspace) return EB_ERR_INVALID;
    if (T == 0) return EB_OK;
    unsigned char* bp = in_smem ? nullptr : reinterpret_cast<unsigned char*>(workspace);
    const int Lmax = 2 * S + 1;
    const int slots = Lmax <= 1024 ? 2 : 4;
    const int threads = ((Lmax + slots - 1) / slots + 31) / 32 * 32;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (Lmax <= 1024) {
        EB_CUDA(cudaFuncSetAttribute(ctc_viterbi_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ctc_viterbi_kernel<2><<<B, threads, smem, st>>>(log_probs, stride_b, stride_t, T, V, targets, ntargets, tg_off,
                                                        tg_len, in_len, S, blank, bp, rows, alignment, frame_logp);
    } else {
        EB_CUDA(cudaFuncSetAttribute(ctc_viterbi_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ctc_viterbi_kernel<4><<<B, threads, smem, st>>>(log_probs, stride_b, stride_t, T, V, targets, ntargets, tg_off,
                                                        tg_len, in_len, S, blank, bp, rows, alignment, frame_logp);
    }
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_ctc_greedy(const float* log_probs, long stride_b, long stride_t, int B, int T, int V, const int* xlen,
                         int blank, int* ids, int* counts, float* neg_score, void* stream) {
    if (!log_probs || !xlen || !ids || !counts || !neg_score || B <= 0 || T < 0 || V <= 0) return EB_ERR_INVALID;
    ctc_greedy_kernel<<<B, GREEDY_THREADS, 0, (cudaStream_t)stream>>>(log_probs, stride_b, stride_t, T, V, xlen, blank,
                                                                      ids, counts, neg_score);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
