// lstm.cu -- persistent-RNN LSTM layer, fp32 (parity mode), sm_90a.
//
// Replaces the recurrent half of nn.LSTM (rnnt/models.py:45-46,64-65 encoder layers,
// :145-147,154-155 predictor): the input projection W_ih*x + b_ih + b_hh for all timesteps is a
// bulk GEMM done by the caller (xg, [B,T,4H], gate order i|f|g|o as in PyTorch); this kernel
// runs the T sequential cell steps in ONE launch:
//
//   * grid = ceil(H / HS) CTAs (<= #SMs, cooperative launch), CTA k owns hidden units
//     [k*HS, (k+1)*HS) -- all four gates of a unit live in the same thread, so the cell
//     update c' = s(f)c + s(i)tanh(g), h' = s(o)tanh(c') is thread-local;
//   * the CTA's slice of W_hh (4*HS rows x H) is loaded into shared memory ONCE and stays
//     there for all T steps (fp32: 16*HS*H bytes, 114 KB at H=1024/HS=7);
//   * h_{t-1} is exchanged through a transposed [H][Bp] global buffer (L2 resident, 128 KB)
//     that every CTA streams through a cp.async double buffer; one grid-wide barrier
//     (monotonic counter, release/acquire) per timestep;
//   * backward (BPTT) mirrors it with the W_hh column slice resident in shared memory and the
//     gate-gradient vector dG_t exchanged through a [4H][Bp] buffer.
//
// Saved for backward: post-activation gates [B,T,4H] and cell states [B,T,H].
//
// The GRU layer (nn.GRU, gate order r|z|n; gru_fwd_kernel / gru_bwd_kernel below) runs on the same design with three
// gate rows per unit and the same helpers.
#include <cooperative_groups.h>
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int KC = 128;        // k-rows per staged chunk
constexpr int BT = 32;         // batch tile (lanes of the exchange buffer row)

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// all threads of every CTA call this; `target` = number of arrivals that must have happened
__device__ __forceinline__ void grid_arrive(unsigned* ctr) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(ctr, 1u);
}
__device__ __forceinline__ void grid_wait(const unsigned* ctr, unsigned target) {
    if (threadIdx.x == 0) {
        spin_wait_ge(ctr, target);
    }
    __syncthreads();
}

// acc[g][i] += sum_k W[(k*HS + j)*NG + g] * X[k][bg*4 + i]   over this thread's share of K.
// X (global, [K][Bp], batch tile offset already applied by the caller via xcol0) is staged
// chunk by chunk through `stage` ([2][KC][BT] floats).  All threads of the CTA must call.
template <int NG>
__device__ __forceinline__ void staged_matmul(const float* __restrict__ Wsm, const float* __restrict__ X,
                                              int K, int HS, int Bp, int xcol0, float* stage,
                                              float (&acc)[NG][4], int j, int bg, int ks, int KS,
                                              bool active) {
    const int nchunks = (K + KC - 1) / KC;
    const int tid = threadIdx.x, nthr = blockDim.x;
    auto issue = [&](int c, int buf) {
        const int k0 = c * KC;
        const int rows = min(KC, K - k0);
        float* dst = stage + buf * (KC * BT);
        for (int i = tid; i < rows * (BT / 4); i += nthr) {
            int r = i / (BT / 4), q = i % (BT / 4);
            cp_async16(dst + r * BT + q * 4, X + (long)(k0 + r) * Bp + xcol0 + q * 4);
        }
        cp_async_commit();
    };
    issue(0, 0);
    for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) { issue(c + 1, (c + 1) & 1); cp_async_wait<1>(); }
        else cp_async_wait<0>();
        __syncthreads();
        if (active) {
            const int k0 = c * KC;
            const int rows = min(KC, K - k0);
            const int per = (rows + KS - 1) / KS;
            const int ka = ks * per, kb = min(rows, ka + per);
            const float* xs = stage + (c & 1) * (KC * BT) + bg * 4;
            const float* ws = Wsm + ((long)k0 * HS + j) * NG;
#pragma unroll 4
            for (int k = ka; k < kb; ++k) {
                const float4 x4 = *reinterpret_cast<const float4*>(xs + k * BT);
                const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
                float wv[NG];
                if (NG == 4) {
                    const float4 w4 = *reinterpret_cast<const float4*>(ws + (long)k * HS * 4);
                    wv[0] = w4.x; wv[1 % NG] = w4.y; wv[2 % NG] = w4.z; wv[3 % NG] = w4.w;
                } else if (NG == 3) {
                    const float* w3 = ws + (long)k * HS * 3;
                    wv[0] = w3[0]; wv[1 % NG] = w3[1]; wv[2 % NG] = w3[2];
                } else {
                    wv[0] = ws[(long)k * HS];
                }
#pragma unroll
                for (int g = 0; g < NG; ++g)
#pragma unroll
                    for (int i = 0; i < 4; ++i) acc[g][i] = fmaf(wv[g], xv[i], acc[g][i]);
            }
        }
        __syncthreads();
    }
}

struct FwdP {
    const float* xg; const float* whh; const float* h0; const float* c0;
    float* y; float* hT; float* cT; float* gates; float* cseq;
    float* hbuf; unsigned* bar;
    int B, T, H, HS, KS, Bp;
};

__global__ void lstm_fwd_kernel(FwdP p) {
    extern __shared__ __align__(16) float smf[];
    const int H = p.H, HS = p.HS, KS = p.KS, B = p.B, T = p.T, Bp = p.Bp;
    float* Wsm = smf;                                   // [H][HS][4]
    float* stage = Wsm + (size_t)H * HS * 4;            // [2][KC][BT]
    float* red = stage + 2 * KC * BT;                   // [KS][HS*8][16]
    const int tid = threadIdx.x;
    const int per_ks = HS * 8;
    const int ks = tid / per_ks, rem = tid % per_ks, jl = rem / 8, bg = rem % 8;
    const int j = blockIdx.x * HS + jl;                 // global hidden unit
    const bool unit_ok = j < H;
    const unsigned ncta = gridDim.x;
    // resident weight slice: Wsm[(k*HS + jl)*4 + g] = W_hh[g*H + j][k]
    for (int i = tid; i < H * HS * 4; i += blockDim.x) {
        int g = i & 3, jj = (i >> 2) % HS, k = (i >> 2) / HS;
        int ju = blockIdx.x * HS + jj;
        Wsm[i] = (ju < H) ? p.whh[((long)g * H + ju) * H + k] : 0.f;
    }
    // prologue: publish h_{-1} (h0) into hbuf[1], running cell state into cT
    float* hb[2] = {p.hbuf, p.hbuf + (size_t)H * Bp};
    if (ks == 0 && unit_ok) {
        for (int b = bg; b < Bp; b += 8) {
            float hv = (b < B && p.h0) ? p.h0[(long)b * H + j] : 0.f;
            hb[1][(long)j * Bp + b] = hv;
            if (b < B) p.cT[(long)b * H + j] = p.c0 ? p.c0[(long)b * H + j] : 0.f;
        }
    }
    grid_arrive(p.bar);
    unsigned epoch = 1;
    const int nbt = (B + BT - 1) / BT;
    for (int t = 0; t < T; ++t) {
        const float* hprev = hb[(t + 1) & 1];
        float* hnext = hb[t & 1];
        for (int bt = 0; bt < nbt; ++bt) {
            const int b0 = bt * BT + bg * 4;
            // prefetch this thread's input-projected gate pre-activations (independent of h)
            float px[4][4];
            if (ks == 0) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int g = 0; g < 4; ++g)
                        px[g][i] = (unit_ok && b0 + i < B)
                                       ? __ldg(p.xg + ((long)(b0 + i) * T + t) * 4 * H + (long)g * H + j) : 0.f;
            }
            if (bt == 0) grid_wait(p.bar, epoch * ncta);
            float acc[4][4];
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[g][i] = 0.f;
            staged_matmul<4>(Wsm, hprev, H, HS, Bp, bt * BT, stage, acc, jl, bg, ks, KS, true);
            if (KS > 1) {
                float* r = red + ((size_t)ks * per_ks + rem) * 16;
#pragma unroll
                for (int g = 0; g < 4; ++g)
#pragma unroll
                    for (int i = 0; i < 4; ++i) r[g * 4 + i] = acc[g][i];
                __syncthreads();
            }
            if (ks == 0 && unit_ok) {
                for (int s = 1; s < KS; ++s) {
                    const float* r = red + ((size_t)s * per_ks + rem) * 16;
#pragma unroll
                    for (int g = 0; g < 4; ++g)
#pragma unroll
                        for (int i = 0; i < 4; ++i) acc[g][i] += r[g * 4 + i];
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int b = b0 + i;
                    if (b >= B) continue;
                    const float ig = sigmoidf_(acc[0][i] + px[0][i]);
                    const float fg = sigmoidf_(acc[1][i] + px[1][i]);
                    const float gg = tanhf(acc[2][i] + px[2][i]);
                    const float og = sigmoidf_(acc[3][i] + px[3][i]);
                    const float cp = p.cT[(long)b * H + j];
                    const float cn = fg * cp + ig * gg;
                    const float hn = og * tanhf(cn);
                    p.cT[(long)b * H + j] = cn;
                    p.y[((long)b * T + t) * H + j] = hn;
                    hnext[(long)j * Bp + b] = hn;
                    if (p.gates) {
                        float* gp = p.gates + ((long)b * T + t) * 4 * H + j;
                        gp[0] = ig; gp[H] = fg; gp[2 * (long)H] = gg; gp[3 * (long)H] = og;
                    }
                    if (p.cseq) p.cseq[((long)b * T + t) * H + j] = cn;
                    if (t == T - 1) p.hT[(long)b * H + j] = hn;
                }
            }
            if (KS > 1) __syncthreads();   // red reused by the next batch tile
        }
        grid_arrive(p.bar);
        ++epoch;
    }
}

struct BwdP {
    const float* dy; const float* gates; const float* cseq; const float* c0; const float* whh;
    const float* dhT; const float* dcT;
    float* dgates; float* dh0; float* dc0;   // dh0/dc0 double as the running dh_rec / dc_rec state
    float* gbuf; unsigned* bar;
    int B, T, H, HS, KS, Bp;
};

__global__ void lstm_bwd_kernel(BwdP p) {
    extern __shared__ __align__(16) float smf[];
    const int H = p.H, HS = p.HS, KS = p.KS, B = p.B, T = p.T, Bp = p.Bp;
    const int H4 = 4 * H;
    float* Wsm = smf;                                   // [4H][HS]   Wsm[r*HS + jl] = W_hh[r][j]
    float* stage = Wsm + (size_t)H4 * HS;
    float* red = stage + 2 * KC * BT;                   // [KS][HS*8][4]
    const int tid = threadIdx.x;
    const int per_ks = HS * 8;
    const int ks = tid / per_ks, rem = tid % per_ks, jl = rem / 8, bg = rem % 8;
    const int j = blockIdx.x * HS + jl;
    const bool unit_ok = j < H;
    const unsigned ncta = gridDim.x;
    for (int i = tid; i < H4 * HS; i += blockDim.x) {
        int jj = i % HS, r = i / HS;
        int ju = blockIdx.x * HS + jj;
        Wsm[i] = (ju < H) ? p.whh[(long)r * H + ju] : 0.f;
    }
    float* gb[2] = {p.gbuf, p.gbuf + (size_t)H4 * Bp};
    // running states: dh0 <- dhT (or 0), dc0 <- dcT (or 0)
    if (ks == 0 && unit_ok) {
        for (int b = bg; b < B; b += 8) {
            p.dh0[(long)b * H + j] = p.dhT ? p.dhT[(long)b * H + j] : 0.f;
            p.dc0[(long)b * H + j] = p.dcT ? p.dcT[(long)b * H + j] : 0.f;
        }
    }
    __syncthreads();
    unsigned epoch = 0;
    const int nbt = (B + BT - 1) / BT;
    for (int t = T - 1; t >= 0; --t) {
        float* gcur = gb[t & 1];
        // phase A: gate gradients of step t for the owned units
        if (ks == 0 && unit_ok) {
            for (int b = bg; b < B; b += 8) {
                const long bt = (long)b * T + t;
                const float* gp = p.gates + bt * H4 + j;
                const float ig = gp[0], fg = gp[H], gg = gp[2 * (long)H], og = gp[3 * (long)H];
                const float ct = p.cseq[bt * H + j];
                const float cprev = (t > 0) ? p.cseq[(bt - 1) * H + j] : (p.c0 ? p.c0[(long)b * H + j] : 0.f);
                const float tc = tanhf(ct);
                const float dh = p.dy[bt * H + j] + p.dh0[(long)b * H + j];
                const float dc = p.dc0[(long)b * H + j] + dh * og * (1.f - tc * tc);
                const float dai = dc * gg * ig * (1.f - ig);
                const float daf = dc * cprev * fg * (1.f - fg);
                const float dag = dc * ig * (1.f - gg * gg);
                const float dao = dh * tc * og * (1.f - og);
                p.dc0[(long)b * H + j] = dc * fg;
                float* dg = p.dgates + bt * H4 + j;
                dg[0] = dai; dg[H] = daf; dg[2 * (long)H] = dag; dg[3 * (long)H] = dao;
                gcur[((long)0 * H + j) * Bp + b] = dai;
                gcur[((long)1 * H + j) * Bp + b] = daf;
                gcur[((long)2 * H + j) * Bp + b] = dag;
                gcur[((long)3 * H + j) * Bp + b] = dao;
            }
        }
        grid_arrive(p.bar);
        ++epoch;
        grid_wait(p.bar, epoch * ncta);
        // phase B: dh_rec[b, j] = sum_r dG_t[b, r] * W_hh[r, j]
        for (int bt = 0; bt < nbt; ++bt) {
            float acc[1][4] = {{0.f, 0.f, 0.f, 0.f}};
            staged_matmul<1>(Wsm, gcur, H4, HS, Bp, bt * BT, stage, acc, jl, bg, ks, KS, true);
            if (KS > 1) {
                float* r = red + ((size_t)ks * per_ks + rem) * 4;
#pragma unroll
                for (int i = 0; i < 4; ++i) r[i] = acc[0][i];
                __syncthreads();
            }
            if (ks == 0 && unit_ok) {
                for (int s = 1; s < KS; ++s) {
                    const float* r = red + ((size_t)s * per_ks + rem) * 4;
#pragma unroll
                    for (int i = 0; i < 4; ++i) acc[0][i] += r[i];
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int b = bt * BT + bg * 4 + i;
                    if (b < B) p.dh0[(long)b * H + j] = acc[0][i];
                }
            }
            __syncthreads();
        }
    }
}

// ---- GRU layer (torch.nn.GRU, gate order r|z|n), the same persistent design with three gate rows per unit --------
// xg [B,T,3H] = W_ih x + b_ih + (b_hr | b_hz | 0): b_hn cannot be folded into the input GEMM because it sits inside the
// reset product, n = tanh(xg_n + r (W_hn h + b_hn)); the kernel adds it to the recurrent n-row sum.  Saved for backward
// per (row, step): r | z | n | gh_n  ([B,T,4H]); h_{t-1} comes from y (shifted by one step) or h0.
struct GruFwdP {
    const float* xg; const float* whh; const float* bhn; const float* h0;
    float* y; float* hT; float* save;
    float* hbuf; unsigned* bar;
    int B, T, H, HS, KS, Bp;
};

// floats of a CTA's resident weight slice, rounded up so that the cp.async stage behind it stays 16-byte aligned
__host__ __device__ inline size_t gru_wsm_floats(int H, int HS) { return ((size_t)3 * H * HS + 3) & ~(size_t)3; }

__global__ void gru_fwd_kernel(GruFwdP p) {
    extern __shared__ __align__(16) float smf[];
    const int H = p.H, HS = p.HS, KS = p.KS, B = p.B, T = p.T, Bp = p.Bp;
    const long H3 = 3 * (long)H;
    float* Wsm = smf;                                   // [H][HS][3]
    float* stage = Wsm + gru_wsm_floats(H, HS);         // [2][KC][BT]
    float* red = stage + 2 * KC * BT;                   // [KS][HS*8][12]
    const int tid = threadIdx.x;
    const int per_ks = HS * 8;
    const int ks = tid / per_ks, rem = tid % per_ks, jl = rem / 8, bg = rem % 8;
    const int j = blockIdx.x * HS + jl;
    const bool unit_ok = j < H;
    const unsigned ncta = gridDim.x;
    // resident weight slice: Wsm[(k*HS + jl)*3 + g] = W_hh[g*H + j][k]
    for (int i = tid; i < H * HS * 3; i += blockDim.x) {
        int g = i % 3, jj = (i / 3) % HS, k = (i / 3) / HS;
        int ju = blockIdx.x * HS + jj;
        Wsm[i] = (ju < H) ? p.whh[((long)g * H + ju) * H + k] : 0.f;
    }
    float* hb[2] = {p.hbuf, p.hbuf + (size_t)H * Bp};
    if (ks == 0 && unit_ok) {
        for (int b = bg; b < Bp; b += 8) hb[1][(long)j * Bp + b] = (b < B && p.h0) ? p.h0[(long)b * H + j] : 0.f;
    }
    const float bn = (unit_ok && p.bhn) ? p.bhn[j] : 0.f;
    grid_arrive(p.bar);
    unsigned epoch = 1;
    const int nbt = (B + BT - 1) / BT;
    for (int t = 0; t < T; ++t) {
        const float* hprev = hb[(t + 1) & 1];
        float* hnext = hb[t & 1];
        for (int bt = 0; bt < nbt; ++bt) {
            const int b0 = bt * BT + bg * 4;
            float px[3][4];
            if (ks == 0) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int g = 0; g < 3; ++g)
                        px[g][i] = (unit_ok && b0 + i < B) ? __ldg(p.xg + ((long)(b0 + i) * T + t) * H3 + (long)g * H + j) : 0.f;
            }
            if (bt == 0) grid_wait(p.bar, epoch * ncta);
            float acc[3][4];
#pragma unroll
            for (int g = 0; g < 3; ++g)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[g][i] = 0.f;
            staged_matmul<3>(Wsm, hprev, H, HS, Bp, bt * BT, stage, acc, jl, bg, ks, KS, true);
            if (KS > 1) {
                float* r = red + ((size_t)ks * per_ks + rem) * 12;
#pragma unroll
                for (int g = 0; g < 3; ++g)
#pragma unroll
                    for (int i = 0; i < 4; ++i) r[g * 4 + i] = acc[g][i];
                __syncthreads();
            }
            if (ks == 0 && unit_ok) {
                for (int s = 1; s < KS; ++s) {
                    const float* r = red + ((size_t)s * per_ks + rem) * 12;
#pragma unroll
                    for (int g = 0; g < 3; ++g)
#pragma unroll
                        for (int i = 0; i < 4; ++i) acc[g][i] += r[g * 4 + i];
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int b = b0 + i;
                    if (b >= B) continue;
                    const float rg = sigmoidf_(acc[0][i] + px[0][i]);
                    const float zg = sigmoidf_(acc[1][i] + px[1][i]);
                    const float ghn = acc[2][i] + bn;
                    const float ng = tanhf(px[2][i] + rg * ghn);
                    const float hp = __ldcg(hprev + (long)j * Bp + b);   // written by this thread (or the prologue)
                    const float hn = (1.f - zg) * ng + zg * hp;
                    p.y[((long)b * T + t) * H + j] = hn;
                    hnext[(long)j * Bp + b] = hn;
                    if (p.save) {
                        float* sp = p.save + ((long)b * T + t) * 4 * H + j;
                        sp[0] = rg; sp[H] = zg; sp[2 * (long)H] = ng; sp[3 * (long)H] = ghn;
                    }
                    if (t == T - 1) p.hT[(long)b * H + j] = hn;
                }
            }
            if (KS > 1) __syncthreads();
        }
        grid_arrive(p.bar);
        ++epoch;
    }
}

// BPTT: per step the owned (unit, row) pairs form
//   dn = dh (1-z)(1-n^2),  dz = dh (h_{t-1} - n) z(1-z),  dr = dn gh_n r(1-r)
//   dgi = [dr, dz, dn] (input side: dx, dW_ih, db_ih),  dgh = [dr, dz, r dn] (recurrent side: dW_hh, db_hh)
// and dh_{t-1} = dh z + W_hh^T dgh, with dgh exchanged through a [3H][Bp] buffer.
struct GruBwdP {
    const float* dy; const float* save; const float* y; const float* h0; const float* whh; const float* dhT;
    float* dgi; float* dgh; float* dh0;     // dh0 doubles as the running dh_rec state
    float* gbuf; unsigned* bar;
    int B, T, H, HS, KS, Bp;
};

__global__ void gru_bwd_kernel(GruBwdP p) {
    extern __shared__ __align__(16) float smf[];
    const int H = p.H, HS = p.HS, KS = p.KS, B = p.B, T = p.T, Bp = p.Bp;
    const int H3 = 3 * H;
    float* Wsm = smf;                                   // [3H][HS]   Wsm[r*HS + jl] = W_hh[r][j]
    float* stage = Wsm + gru_wsm_floats(H, HS);
    float* red = stage + 2 * KC * BT;                   // [KS][HS*8][4]
    const int tid = threadIdx.x;
    const int per_ks = HS * 8;
    const int ks = tid / per_ks, rem = tid % per_ks, jl = rem / 8, bg = rem % 8;
    const int j = blockIdx.x * HS + jl;
    const bool unit_ok = j < H;
    const unsigned ncta = gridDim.x;
    for (int i = tid; i < H3 * HS; i += blockDim.x) {
        int jj = i % HS, r = i / HS;
        int ju = blockIdx.x * HS + jj;
        Wsm[i] = (ju < H) ? p.whh[(long)r * H + ju] : 0.f;
    }
    float* gb[2] = {p.gbuf, p.gbuf + (size_t)H3 * Bp};
    if (ks == 0 && unit_ok) {
        for (int b = bg; b < B; b += 8) p.dh0[(long)b * H + j] = p.dhT ? p.dhT[(long)b * H + j] : 0.f;
    }
    __syncthreads();
    unsigned epoch = 0;
    const int nbt = (B + BT - 1) / BT;
    for (int t = T - 1; t >= 0; --t) {
        float* gcur = gb[t & 1];
        // phase A: gate gradients of step t; dh0 <- the direct term dh z of dh_{t-1}
        if (ks == 0 && unit_ok) {
            for (int b = bg; b < B; b += 8) {
                const long bt = (long)b * T + t;
                const float* sp = p.save + bt * 4 * H + j;
                const float rg = sp[0], zg = sp[H], ng = sp[2 * (long)H], ghn = sp[3 * (long)H];
                const float hp = (t > 0) ? p.y[(bt - 1) * H + j] : (p.h0 ? p.h0[(long)b * H + j] : 0.f);
                const float dh = p.dy[bt * H + j] + p.dh0[(long)b * H + j];
                const float dn = dh * (1.f - zg) * (1.f - ng * ng);
                const float dz = dh * (hp - ng) * zg * (1.f - zg);
                const float dr = dn * ghn * rg * (1.f - rg);
                const float dhn = rg * dn;
                p.dh0[(long)b * H + j] = dh * zg;
                float* gi = p.dgi + bt * H3 + j;
                gi[0] = dr; gi[H] = dz; gi[2 * (long)H] = dn;
                float* gh = p.dgh + bt * H3 + j;
                gh[0] = dr; gh[H] = dz; gh[2 * (long)H] = dhn;
                gcur[((long)0 * H + j) * Bp + b] = dr;
                gcur[((long)1 * H + j) * Bp + b] = dz;
                gcur[((long)2 * H + j) * Bp + b] = dhn;
            }
        }
        grid_arrive(p.bar);
        ++epoch;
        grid_wait(p.bar, epoch * ncta);
        // phase B: dh_{t-1}[b, j] = sum_r dgh_t[b, r] W_hh[r, j] + dh z
        for (int bt = 0; bt < nbt; ++bt) {
            float acc[1][4] = {{0.f, 0.f, 0.f, 0.f}};
            staged_matmul<1>(Wsm, gcur, H3, HS, Bp, bt * BT, stage, acc, jl, bg, ks, KS, true);
            if (KS > 1) {
                float* r = red + ((size_t)ks * per_ks + rem) * 4;
#pragma unroll
                for (int i = 0; i < 4; ++i) r[i] = acc[0][i];
                __syncthreads();
            }
            if (ks == 0 && unit_ok) {
                for (int s = 1; s < KS; ++s) {
                    const float* r = red + ((size_t)s * per_ks + rem) * 4;
#pragma unroll
                    for (int i = 0; i < 4; ++i) acc[0][i] += r[i];
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int b = bt * BT + bg * 4 + i;
                    if (b < B) p.dh0[(long)b * H + j] = acc[0][i] + p.dh0[(long)b * H + j];
                }
            }
            __syncthreads();
        }
    }
}

struct Plan { int HS, KS, ncta, threads, Bp; size_t smem_f, smem_b; };

inline bool make_plan(int B, int H, Plan& pl) {
    const int sms = eb_num_sms();
    int HS = (H + sms - 1) / sms;
    if (HS < 1) HS = 1;
    pl.HS = HS;
    pl.ncta = (H + HS - 1) / HS;
    int KS = 256 / (HS * 8);
    if (KS < 1) KS = 1;
    if (KS > 8) KS = 8;
    pl.KS = KS;
    pl.threads = HS * 8 * KS;
    pl.Bp = ((B + BT - 1) / BT) * BT;
    pl.smem_f = sizeof(float) * ((size_t)H * HS * 4 + 2 * KC * BT + (size_t)KS * HS * 8 * 16);
    pl.smem_b = sizeof(float) * ((size_t)4 * H * HS + 2 * KC * BT + (size_t)KS * HS * 8 * 4);
    return pl.threads <= 1024 && pl.smem_f <= 220 * 1024 && pl.smem_b <= 220 * 1024;
}

inline bool make_gru_plan(int B, int H, Plan& pl) {
    make_plan(B, H, pl);
    pl.smem_f = sizeof(float) * (gru_wsm_floats(H, pl.HS) + 2 * KC * BT + (size_t)pl.KS * pl.HS * 8 * 12);
    pl.smem_b = sizeof(float) * (gru_wsm_floats(H, pl.HS) + 2 * KC * BT + (size_t)pl.KS * pl.HS * 8 * 4);
    return pl.threads <= 1024 && pl.smem_f <= 220 * 1024 && pl.smem_b <= 220 * 1024;
}

}  // namespace

// scratch: hbuf/gbuf exchange buffers + barrier word.  Bytes needed (caller allocates, zeroed once):
EB_API size_t eb_lstm_scratch_bytes(int B, int H) {
    Plan pl;
    if (!make_plan(B, H, pl)) return 0;
    return sizeof(float) * (size_t)2 * 4 * H * pl.Bp + 256;
}

EB_API int eb_lstm_seq_fwd(const float* xg, const float* whh, const float* h0, const float* c0, float* y,
                           float* hT, float* cT, float* gates_save, float* cseq_save, void* scratch,
                           int B, int T, int H, void* stream) {
    if (!xg || !whh || !y || !hT || !cT || !scratch || B <= 0 || T <= 0 || H <= 0) return EB_ERR_INVALID;
    Plan pl;
    if (!make_plan(B, H, pl)) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FwdP p;
    p.xg = xg; p.whh = whh; p.h0 = h0; p.c0 = c0; p.y = y; p.hT = hT; p.cT = cT;
    p.gates = gates_save; p.cseq = cseq_save;
    p.bar = reinterpret_cast<unsigned*>(scratch);
    p.hbuf = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + 256);
    p.B = B; p.T = T; p.H = H; p.HS = pl.HS; p.KS = pl.KS; p.Bp = pl.Bp;
    // zero the barrier and the (padded) exchange buffers
    EB_CUDA(cudaMemsetAsync(scratch, 0, 256 + sizeof(float) * (size_t)2 * H * pl.Bp, st));
    EB_CUDA(cudaFuncSetAttribute(lstm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_f));
    void* args[] = {&p};
    EB_CUDA(cudaLaunchCooperativeKernel((void*)lstm_fwd_kernel, dim3(pl.ncta), dim3(pl.threads), args,
                                        pl.smem_f, st));
    return EB_OK;
}

EB_API int eb_lstm_seq_bwd(const float* dy, const float* gates, const float* cseq, const float* c0,
                           const float* whh, const float* dhT, const float* dcT, float* dgates,
                           float* dh0, float* dc0, void* scratch, int B, int T, int H, void* stream) {
    if (!dy || !gates || !cseq || !whh || !dgates || !dh0 || !dc0 || !scratch) return EB_ERR_INVALID;
    Plan pl;
    if (!make_plan(B, H, pl)) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    BwdP p;
    p.dy = dy; p.gates = gates; p.cseq = cseq; p.c0 = c0; p.whh = whh; p.dhT = dhT; p.dcT = dcT;
    p.dgates = dgates; p.dh0 = dh0; p.dc0 = dc0;
    p.bar = reinterpret_cast<unsigned*>(scratch);
    p.gbuf = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + 256);
    p.B = B; p.T = T; p.H = H; p.HS = pl.HS; p.KS = pl.KS; p.Bp = pl.Bp;
    EB_CUDA(cudaMemsetAsync(scratch, 0, 256 + sizeof(float) * (size_t)2 * 4 * H * pl.Bp, st));
    EB_CUDA(cudaFuncSetAttribute(lstm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_b));
    void* args[] = {&p};
    EB_CUDA(cudaLaunchCooperativeKernel((void*)lstm_bwd_kernel, dim3(pl.ncta), dim3(pl.threads), args,
                                        pl.smem_b, st));
    return EB_OK;
}

// ---- GRU entry points ----------------------------------------------------------------------------------------------
EB_API size_t eb_gru_scratch_bytes(int B, int H) {
    if (B <= 0 || H <= 0) return 0;
    Plan pl;
    if (!make_gru_plan(B, H, pl)) return 0;
    return sizeof(float) * (size_t)2 * 3 * H * pl.Bp + 256;
}

EB_API int eb_gru_seq_fwd(const float* xg, const float* whh, const float* bhn, const float* h0, float* y, float* hT,
                          float* save, void* scratch, int B, int T, int H, void* stream) {
    if (!xg || !whh || !y || !hT || !scratch || B <= 0 || T <= 0 || H <= 0) return EB_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(scratch) & 15) return EB_ERR_INVALID;     // the exchange buffer is pulled in 16 B
    Plan pl;
    if (!make_gru_plan(B, H, pl)) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    GruFwdP p;
    p.xg = xg; p.whh = whh; p.bhn = bhn; p.h0 = h0; p.y = y; p.hT = hT; p.save = save;
    p.bar = reinterpret_cast<unsigned*>(scratch);
    p.hbuf = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + 256);
    p.B = B; p.T = T; p.H = H; p.HS = pl.HS; p.KS = pl.KS; p.Bp = pl.Bp;
    EB_CUDA(cudaMemsetAsync(scratch, 0, 256 + sizeof(float) * (size_t)2 * H * pl.Bp, st));
    EB_CUDA(cudaFuncSetAttribute(gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_f));
    void* args[] = {&p};
    EB_CUDA(cudaLaunchCooperativeKernel((void*)gru_fwd_kernel, dim3(pl.ncta), dim3(pl.threads), args, pl.smem_f, st));
    return EB_OK;
}

EB_API int eb_gru_seq_bwd(const float* dy, const float* save, const float* y, const float* h0, const float* whh,
                          const float* dhT, float* dgi, float* dgh, float* dh0, void* scratch, int B, int T, int H,
                          void* stream) {
    if (!dy || !save || !y || !whh || !dgi || !dgh || !dh0 || !scratch || B <= 0 || T <= 0 || H <= 0)
        return EB_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(scratch) & 15) return EB_ERR_INVALID;
    Plan pl;
    if (!make_gru_plan(B, H, pl)) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    GruBwdP p;
    p.dy = dy; p.save = save; p.y = y; p.h0 = h0; p.whh = whh; p.dhT = dhT;
    p.dgi = dgi; p.dgh = dgh; p.dh0 = dh0;
    p.bar = reinterpret_cast<unsigned*>(scratch);
    p.gbuf = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + 256);
    p.B = B; p.T = T; p.H = H; p.HS = pl.HS; p.KS = pl.KS; p.Bp = pl.Bp;
    EB_CUDA(cudaMemsetAsync(scratch, 0, 256 + sizeof(float) * (size_t)2 * 3 * H * pl.Bp, st));
    EB_CUDA(cudaFuncSetAttribute(gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_b));
    void* args[] = {&p};
    EB_CUDA(cudaLaunchCooperativeKernel((void*)gru_bwd_kernel, dim3(pl.ncta), dim3(pl.threads), args, pl.smem_b, st));
    return EB_OK;
}
