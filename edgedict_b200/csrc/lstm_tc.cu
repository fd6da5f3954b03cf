// lstm_tc.cu -- persistent-RNN LSTM layer on tensor cores (bf16 operands, fp32 accumulate / state),
// the bf16-mode replacement of lstm.cu for H % 64 == 0, H <= 1024 (all BASELINE configs).
//
// Forward (one launch for all T steps, H/8 CTAs x 256 threads):
//   * CTA k owns hidden units [8k, 8k+8): 32 gate rows of W_hh arranged as two m16 tiles
//     (i|f) and (g|o), so that after mma.sync.m16n8k16 one thread holds all four gates of a
//     (unit, batch) pair and the cell update is thread-local;
//   * W_hh is held in REGISTERS as mma A-fragments for the whole sequence: each of the 8 warps
//     owns a K-range of H/8 columns (<= 8 k-steps x 2 m-tiles x 4 regs = 64 registers);
//   * h_{t-1} (bf16, [batch][H]) is exchanged through an L2-resident double buffer; each warp
//     pulls only its own K-range with cp.async and feeds ldmatrix B-fragments; the 8 partial
//     accumulators are summed through shared memory; one grid barrier per timestep whose
//     release (one 16-byte store per batch row + ONE thread's fence + atomic) is issued before
//     the non-critical stores (y, saved gates, cell states) so that they overlap the wait.
// Backward (BPTT): 2-D decomposition: a group of CS CTAs owns 8*CS hidden units and splits the 4H
//   gate rows (the contraction) CS ways; W_hh^T A-fragments in registers (64 regs for any CS at
//   H=1024); partial [8*CS units x batch] tiles are reduce-scattered
//     CLUSTER = true : across a thread-block cluster through DISTRIBUTED SHARED MEMORY behind one
//                      hardware cluster barrier (CS = 8, 4 or 2, the largest that is co-resident);
//     CLUSTER = false: through L2 behind a per-group software barrier (always launchable);
//   the owning threads then run the gate-gradient math for step t-1 (inputs prefetched during the
//   wait) with dh/dc carried in registers, and publish dG_t in bf16.
//
// Semantics: nn.LSTM cell, gate order i|f|g|o (rnnt/models.py:45-46 -> torch.nn.LSTM).
#include <cooperative_groups.h>
#include <stdlib.h>
#include "common.cuh"
#include "sm90.cuh"
#include "../../include/edgedict_b200.h"

namespace cg = cooperative_groups;

namespace {

#ifndef EB_LSTM_MINB
#define EB_LSTM_MINB 2           // CTAs per SM the FORWARD kernel is compiled for (<= 128 registers / thread): the
#endif                           // kernels of two LAYERS are co-resident on every SM in the wavefront schedule
constexpr int NW = 8;            // warps per CTA
constexpr int UPC = 8;           // hidden units finalised per CTA
constexpr int PAD = 8;           // bf16 elements of row padding (16 B) -> conflict-free ldmatrix
constexpr int NB = 32;           // widest batch tile (rows of the exchange buffers)
constexpr size_t TC_HDR = 16384; // scratch: [0,8192) grid barrier counters (one per K slice, 1 KB apart: the L2 slice hash uses address
                                 // bits 8 and 10-27, so counters 128 B apart share slices), [8192,16384) per-group barriers
constexpr int CTR_STRIDE = 256;  // uints between two slice counters

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_row) {
    unsigned a = (unsigned)__cvta_generic_to_shared(smem_row);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t ldg_u32(const __nv_bfloat16* p) {
    return *reinterpret_cast<const uint32_t*>(p);
}
// bf16-mode gate nonlinearities: ex2.approx + rcp.approx (abs. error measured at most 1.1e-7 for the
// sigmoid and 2.1e-7 for the tanh, whose 1 - 2/(e^2x + 1) cancels near 0; far below the bf16 rounding
// of the exchanged h); the fp32 parity kernels in lstm.cu keep expf/tanhf.
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.f, 1.f + fast_exp(-x)); }
__device__ __forceinline__ float fast_tanh(float x) { return 1.f - __fdividef(2.f, fast_exp(2.f * x) + 1.f); }

// one warp copies its K-range (cpr 16-byte chunks per row, NB rows) of the exchange buffer into a
// padded shared tile.  No integer division in the common case (cpr divides 32).
__device__ __forceinline__ void warp_pull(__nv_bfloat16* dst, int dst_ld, const __nv_bfloat16* src, int src_ld,
                                          int cpr, int nrows) {
    const int l = threadIdx.x & 31;
    if (cpr > 0 && (cpr % 8) == 0 && (nrows % 4) == 0) {
        // 128-byte column blocks, four rows per instruction (eight lanes read one full line of a row): the access pattern
        // that halved the pull latency of the lstm_c4 forward kernel
        const int r0 = l >> 3, c0 = l & 7;
        for (int cb = 0; cb < cpr; cb += 8)
            for (int r = r0; r < nrows; r += 4)
                cp_async16(dst + (size_t)r * dst_ld + (cb + c0) * 8, src + (size_t)r * src_ld + (cb + c0) * 8);
    } else if (cpr > 0 && (32 % cpr) == 0) {
        const int rstep = 32 / cpr;
        int r = l / cpr;
        const int q = l % cpr;
        __nv_bfloat16* d = dst + (size_t)r * dst_ld + q * 8;
        const __nv_bfloat16* g = src + (size_t)r * src_ld + q * 8;
        for (; r < nrows; r += rstep) {
            cp_async16(d, g);
            d += (size_t)rstep * dst_ld;
            g += (size_t)rstep * src_ld;
        }
    } else {
        for (int i = l; i < nrows * cpr; i += 32) {
            const int r = i / cpr, q = i % cpr;
            cp_async16(dst + (size_t)r * dst_ld + q * 8, src + (size_t)r * src_ld + q * 8);
        }
    }
    cp_async_wait_all();
    __syncwarp();
}

// Grid barrier = monotonic counter: every CTA adds 1 after publishing (one thread: fence + atomic),
// ONE thread per CTA polls with ld.acquire.gpu, then a block barrier.  (A poller per warp contends on the
// counter line; one flag per producer with st.release and vector polls costs more polls per step.)
// B fragments for one k-step and all four batch n-tiles out of a padded [NB][ld] bf16 tile
template <int NT>
__device__ __forceinline__ void load_b(uint32_t (&b01)[4], uint32_t (&b23)[4], const __nv_bfloat16* tile, int ld,
                                       int kstep) {
    const int l = threadIdx.x & 31;
    const int mrow = (l & 7) + ((l >> 4) & 1) * 8;
    const int mk = kstep * 16 + ((l >> 3) & 1) * 8;
    ldmatrix_x4(b01, tile + (size_t)mrow * ld + mk);
    if (NT > 2) ldmatrix_x4(b23, tile + (size_t)(16 + mrow) * ld + mk);
}

struct FwdP {
    const float* xg;              // [B,T,4H] fp32
    const __nv_bfloat16* whh;     // [4H,H] bf16
    const float* h0; const float* c0;
    float* y; __nv_bfloat16* y16; float* hT; float* cT; float* gates; float* cseq;
    __nv_bfloat16* hx;            // [2][NB][H] exchange
    unsigned* bar;
    int B, T, H;
};

// One batch tile of up to NBT = 32 rows per launch.  (Two independent 16-row halves co-resident on every SM would each be
// as latency-bound as the whole; pairing DIFFERENT layers is what pays: functional.LSTMStack.)
constexpr int NBT = NB;
__global__ void __launch_bounds__(NW * 32, EB_LSTM_MINB) lstm_tc_fwd_kernel(FwdP p) {
    constexpr int NT = NBT / 8;                              // batch n-tiles
    constexpr int SL = NT * 8;                               // accumulator slots per thread
    extern __shared__ __align__(16) unsigned char smraw[];
    const int H = p.H, B = p.B, T = p.T;
    const int HP = H + PAD;
    __nv_bfloat16* hs = reinterpret_cast<__nv_bfloat16*>(smraw);                 // [NBT][HP]
    float* red = reinterpret_cast<float*>(smraw + (size_t)NBT * HP * 2);         // [NW][SL][32]
    __nv_bfloat16* sh_h = reinterpret_cast<__nv_bfloat16*>(red + NW * SL * 32);   // [NBT][UPC]
    // next step's input pre-activations are prefetched with cp.async into a per-thread shared slot: no
    // registers are held across the grid barrier (a register prefetch is spilled at the 128-register
    // budget of the two-CTAs-per-SM build, and the spill store waits for the DRAM round trip)
    float* pxs = reinterpret_cast<float*>(sh_h + NBT * UPC) + threadIdx.x;         // [4][NW*32]
    const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
    const int j0 = blockIdx.x * UPC;
    const unsigned ncta = gridDim.x;
    const int nks = H / 16;
    const int ksper = (nks + NW - 1) / NW;                   // <= 8
    const int ks0 = w * ksper;
    const int myks = max(0, min(ksper, nks - ks0));
    const size_t xstride = (size_t)NBT * H;

    // resident A fragments: afr[mt][ks][4]; mt 0 = rows (i: 0-7, f: 8-15), mt 1 = (g, o)
    uint32_t afr[2][8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            const int k = (ks0 + ks) * 16 + (l & 3) * 2;
            const int u = j0 + (l >> 2);
            const __nv_bfloat16* rlo = p.whh + ((long)(mt * 2 + 0) * H + u) * H + k;   // gate i / g
            const __nv_bfloat16* rhi = p.whh + ((long)(mt * 2 + 1) * H + u) * H + k;   // gate f / o
            const bool ok = ks < myks;
            afr[mt][ks][0] = ok ? ldg_u32(rlo) : 0u;
            afr[mt][ks][1] = ok ? ldg_u32(rhi) : 0u;
            afr[mt][ks][2] = ok ? ldg_u32(rlo + 8) : 0u;
            afr[mt][ks][3] = ok ? ldg_u32(rhi + 8) : 0u;
        }

    // the (unit, batch) pair this thread finalises every step
    const int ju = l >> 2;
    const int bb = (w >> 1) * 8 + (l & 3) * 2 + (w & 1);
    const int j = j0 + ju;
    const bool own = (w >> 1) < NT && bb < B;
    float c_state = (own && p.c0) ? p.c0[(long)bb * H + j] : 0.f;
    if (own) p.hx[xstride + (long)bb * H + j] = __float2bfloat16(p.h0 ? p.h0[(long)bb * H + j] : 0.f);
    __syncthreads();
    if (tid == 0) { __threadfence(); atomicAdd(p.bar, 1u); }
    unsigned epoch = 1;

    // element offsets of this thread's (batch row, unit) pair in the [B,T,H] and [B,T,4H] tensors: advance by
    // one frame per step (two offsets instead of five pointers: the kernel lives at 128 registers)
    long oh = (long)bb * T * H + j;
    long og4 = (long)bb * T * 4 * H + j;
    if (own) {
#pragma unroll
        for (int g = 0; g < 4; ++g) cp_async4(pxs + g * (NW * 32), p.xg + og4 + (long)g * H);
    }

    for (int t = 0; t < T; ++t) {
        const __nv_bfloat16* hprev = p.hx + ((t + 1) & 1) * xstride;
        __nv_bfloat16* hnext = p.hx + (t & 1) * xstride;
        // grid barrier, wait side: ONE poller per CTA (8 pollers per CTA cost ~1.1 us/step of L2 contention on
        // the counter line), then a block barrier
        if (tid == 0) spin_wait_ge(p.bar, epoch * ncta);
        __syncthreads();
        // pull this warp's K-range of h_{t-1}: NB rows x (myks*16) bf16
        warp_pull(hs + ks0 * 16, HP, hprev + ks0 * 16, H, myks * 2, NBT);
        float acc[2][NT][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            if (ks < myks) {
                uint32_t b01[4], b23[4];
                load_b<NT>(b01, b23, hs, HP, ks0 + ks);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    mma_bf16(acc[mt][0], afr[mt][ks], b01[0], b01[1]);
                    mma_bf16(acc[mt][1], afr[mt][ks], b01[2], b01[3]);
                    if (NT > 2) {
                        mma_bf16(acc[mt][NT - 2], afr[mt][ks], b23[0], b23[1]);
                        mma_bf16(acc[mt][NT - 1], afr[mt][ks], b23[2], b23[3]);
                    }
                }
            }
        }
        // partials -> shared: red[w][slot][lane], slot = nt*8 + mt*4 + i
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) red[(w * SL + nt * 8 + mt * 4 + i) * 32 + l] = acc[mt][nt][i];
        __syncthreads();
        float ig = 0.f, fg = 0.f, gg = 0.f, og = 0.f, hn = 0.f;
        if ((w >> 1) < NT) {   // nt = w>>1, batch offset = w&1 -> slots (i: mt0,off) (f: mt0,2+off) (g: mt1,off) (o: mt1,2+off)
            const int nt = w >> 1, off = w & 1;
            float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int sw = 0; sw < NW; ++sw) {
                const float* r = red + (size_t)(sw * SL + nt * 8) * 32 + l;
                s[0] += r[(0 + off) * 32];
                s[1] += r[(2 + off) * 32];
                s[2] += r[(4 + off) * 32];
                s[3] += r[(6 + off) * 32];
            }
            cp_async_wait_all();                             // (already drained by warp_pull)
            float px[4];
#pragma unroll
            for (int g = 0; g < 4; ++g) px[g] = own ? pxs[g * (NW * 32)] : 0.f;
            ig = fast_sigmoid(s[0] + px[0]);
            fg = fast_sigmoid(s[1] + px[1]);
            gg = fast_tanh(s[2] + px[2]);
            og = fast_sigmoid(s[3] + px[3]);
            c_state = fg * c_state + ig * gg;
            hn = og * fast_tanh(c_state);
            sh_h[bb * UPC + ju] = __float2bfloat16(own ? hn : 0.f);
        }
        __syncthreads();
        if (w == 0) {   // publish h_t: one 16-byte store per batch row, then a single fence + arrive
            if (l < NBT) *reinterpret_cast<uint4*>(hnext + (size_t)l * H + j0) = *reinterpret_cast<const uint4*>(sh_h + l * UPC);
            __syncwarp();
            if (l == 0) { __threadfence(); atomicAdd(p.bar, 1u); }
        }
        ++epoch;
        // everything below overlaps the other CTAs' progress towards the barrier
        if (own) {
            p.y[oh] = hn;
            if (p.y16) p.y16[oh] = __float2bfloat16(hn);
            if (p.gates) { float* g_p = p.gates + og4; g_p[0] = ig; g_p[H] = fg; g_p[2 * (long)H] = gg; g_p[3 * (long)H] = og; }
            if (p.cseq) p.cseq[oh] = c_state;
            if (t == T - 1) { p.hT[(long)bb * H + j] = hn; p.cT[(long)bb * H + j] = c_state; }
        }
        oh += H; og4 += 4 * (long)H;
        if (t + 1 < T && own) {
#pragma unroll
            for (int g = 0; g < 4; ++g) cp_async4(pxs + g * (NW * 32), p.xg + og4 + (long)g * H);
        }
    }
}

// ------------------------------------------------------------------------------------------------
struct BwdP {
    const float* dy; const float* gates; const float* cseq; const float* c0;
    const __nv_bfloat16* whhT;    // [H,4H] bf16 = W_hh^T
    const float* dhT; const float* dcT;
    __nv_bfloat16* dg16;          // [B,T,4H] bf16 gate-preactivation gradients (output)
    float* dh0; float* dc0;
    __nv_bfloat16* gx;            // [2][NB][4H] exchange
    unsigned* bar;
    unsigned* gbar;               // per-group counters (non-cluster variant)
    float* pglob;                 // [H/(8*CS)][CS][8*CS][NB] partial tiles in L2 (non-cluster variant)
    long long* trace; int trace_steps;   // debug: clock64 stamps of CTA 0 (eb_lstm_tc_set_trace)
    int B, T, H;
    // time axis in segments (chunk-major storage of the layer wavefront, functional._Chunks): segment c covers steps
    // [seg_off[c], seg_off[c+1]) and is a contiguous [Btot, len_c, D] block at row Btot * seg_off[c]; one segment = [B,T,D]
    int b0, Btot, nseg;
    int seg_off[9];
    int wpoll;                    // every warp polls the barrier counter itself (default; EDGEDICT_LSTM_WPOLL bit 1): the pull of a warp
                                  // starts when IT sees the counter, no block barrier behind a single poller
};
#define TC_STAMP(step, s)                                                                          \
    do {                                                                                           \
        if (p.trace && blockIdx.x == 0 && tid == 0 && (step) < p.trace_steps) p.trace[(size_t)(step) * 16 + (s)] = clock64(); \
    } while (0)
long long* g_tc_trace = nullptr;
int g_tc_trace_steps = 0;

// REMAP selects the phase-A thread -> (unit, batch row) map:
//   true  (default): unit = lane / 4, row = 4 * warp + lane % 4, the forward kernel's map: the 8 units of a row are one sector, a
//          warp-wide load of a saved gate touches 4 sectors, and -- what counts on the critical path -- the exchange store of a warp
//          is 4 rows x 64 contiguous bytes instead of 32 rows x 8 bytes: fewer write transactions to fence before the barrier;
//   false (EDGEDICT_LSTM_BWD_REMAP=0): unit = warp, row = lane: 32 sectors per load for 4 useful bytes each.
template <int CS, bool CLUSTER, bool REMAP = false>
__global__ void __launch_bounds__(NW * 32, 1) lstm_tc_bwd_kernel(BwdP p) {
    constexpr int MT = CS / 2;                               // m16 tiles: 8*CS units
    constexpr int JS = 8 * CS;                               // units per group
    constexpr int KSMAX = 32 / CS;                           // k-steps per warp at H = 1024
    constexpr int SLOTS = MT * 16;                           // accumulator registers per thread
    extern __shared__ __align__(16) unsigned char smraw[];
    const int H = p.H, B = p.B, T = p.T, H4 = 4 * H;
    const int KR = H4 / CS;                                  // gate rows (contraction) per CTA
    const int KP = KR + PAD;
    __nv_bfloat16* gs = reinterpret_cast<__nv_bfloat16*>(smraw);                 // [NB][KP]
    float* red = reinterpret_cast<float*>(smraw + (size_t)NB * KP * 2);          // [NW][SLOTS][32]
    float* part = red + NW * SLOTS * 32;                                         // [2][JS][NB] (step parity)
    __nv_bfloat16* sg = reinterpret_cast<__nv_bfloat16*>(part + 2 * JS * NB);    // [NB][4][UPC]  (gate-major, for dg16)
    float* pgs = reinterpret_cast<float*>(sg + NB * 4 * UPC) + threadIdx.x;      // [4][NW*32] cp.async prefetch slots (gates)
    // cluster variant: the peers' partial tiles of this CTA's 8 units arrive here as bulk DSMEM copies that complete
    // on `rbar` ([2 step parities][CS sources][UPC][NB]; the slot of the own rank is unused)
    float* recvp = reinterpret_cast<float*>(sg + NB * 4 * UPC) + 4 * NW * 32;
    uint64_t* rbar_p = reinterpret_cast<uint64_t*>(recvp + 2 * CS * UPC * NB);
    const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
    const int rs = blockIdx.x % CS;                          // K slice (= cluster rank)
    const int js = blockIdx.x / CS;                          // unit group
    const int r0 = rs * KR;
    const unsigned ncta = gridDim.x;
    const int nks = KR / 16;
    const int ksper = (nks + NW - 1) / NW;                   // <= KSMAX
    const int ks0 = w * ksper;
    const int myks = max(0, min(ksper, nks - ks0));
    const size_t xstride = (size_t)NB * H4;
    auto rowof = [&](int b, int t) -> long {                 // row of (batch b of this tile, step t) in the saved tensors
        int c = 0;
        while (c + 1 < p.nseg && t >= p.seg_off[c + 1]) ++c;
        const int lo = p.seg_off[c];
        return (long)p.Btot * lo + (long)(p.b0 + b) * (p.seg_off[c + 1] - lo) + (t - lo);
    };

    // The contraction index is ordered unit-major, r' = 4*j + g, so that a K-slice is produced by a
    // contiguous range of CTAs (8 units x 4 gates each):  A(m = unit u, k = r') = W_hh[g*H + j, u]
    // = whhT[u][g*H + j].  Consecutive k of a fragment register are gates (g, g+1) of the same j.
    uint32_t afr[MT][KSMAX][4];
    auto wpair = [&](int u, int rp) -> uint32_t {            // (r', r'+1), r' even
        const int jj = rp >> 2, g = rp & 3;
        const unsigned short lo = *reinterpret_cast<const unsigned short*>(p.whhT + (long)u * H4 + (long)g * H + jj);
        const unsigned short hi = *reinterpret_cast<const unsigned short*>(p.whhT + (long)u * H4 + (long)(g + 1) * H + jj);
        return (uint32_t)lo | ((uint32_t)hi << 16);
    };
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int ks = 0; ks < KSMAX; ++ks) {
            const int k = r0 + (ks0 + ks) * 16 + (l & 3) * 2;
            const int u = js * JS + mt * 16 + (l >> 2);
            const bool ok = ks < myks;
            afr[mt][ks][0] = ok ? wpair(u, k) : 0u;
            afr[mt][ks][1] = ok ? wpair(u + 8, k) : 0u;
            afr[mt][ks][2] = ok ? wpair(u, k + 8) : 0u;
            afr[mt][ks][3] = ok ? wpair(u + 8, k + 8) : 0u;
        }

    // phase-A ownership (see REMAP above): unit = js*JS + rs*8 + uu, batch row = bb
    const int uu = REMAP ? (l >> 2) : w;
    const int bb = REMAP ? (w * 4 + (l & 3)) : l;
    const int j = js * JS + rs * UPC + uu;
    const bool own = bb < B;
    float dh = (own && p.dhT) ? p.dhT[(long)bb * H + j] : 0.f;
    float dc = (own && p.dcT) ? p.dcT[(long)bb * H + j] : 0.f;
    unsigned epoch = 0;
    // grid barrier per K slice (see lstm_c4.cu): this CTA consumes slice rs of dG_t, produced by the ncta/CS CTAs that
    // own the units [rs*H/CS, (rs+1)*H/CS); it arrives on the counter of the slice its own units belong to
    const unsigned nprod = ncta / CS;
    unsigned* const my_ctr = p.bar + ((js * JS + rs * UPC) / (H / CS)) * CTR_STRIDE;
    const unsigned* const wait_ctr = p.bar + rs * CTR_STRIDE;
    const uint32_t rbar = smem_u32(rbar_p);
    if (CLUSTER) {
        if (tid == 0) {
            mbar_init(rbar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        cluster_sync_all();                                  // every peer's mbarrier exists before a copy completes on it
    }

    // prefetched inputs of the gate-gradient math: gates i,f,g,o, c_t, c_{t-1}, dy_t
    // (the four gates go through cp.async + shared memory, see the forward kernel; c_t, c_{t-1}, dy_t in registers)
    float in4 = 0.f, in5 = 0.f, in6 = 0.f;
#define EB_PREFETCH(tt)                                                                                   \
    if (own && (tt) >= 0) {                                                                               \
        const long bt_ = rowof(bb, (tt));                                                                 \
        const float* gp_ = p.gates + bt_ * H4 + j;                                                        \
        _Pragma("unroll") for (int g_ = 0; g_ < 4; ++g_) cp_async4(pgs + g_ * (NW * 32), gp_ + (long)g_ * H); \
        in4 = __ldg(p.cseq + bt_ * H + j);                                                                \
        in5 = ((tt) > 0) ? __ldg(p.cseq + rowof(bb, (tt) - 1) * H + j) : (p.c0 ? p.c0[(long)bb * H + j] : 0.f); \
        in6 = __ldg(p.dy + bt_ * H + j);                                                                  \
    }
    EB_PREFETCH(T - 1)

    for (int t = T - 1; t >= 0; --t) {
        __nv_bfloat16* gcur = p.gx + (t & 1) * xstride;
        TC_STAMP(T - 1 - t, 0);
        // ---- phase A: gate gradients of step t for the owned (unit, batch)
        {
            float da[4] = {0.f, 0.f, 0.f, 0.f};
            if (own) {
                cp_async_wait_all();                         // (already drained by warp_pull, except at t = T-1)
                const float ig = pgs[0], fg = pgs[NW * 32], gg = pgs[2 * NW * 32], og = pgs[3 * NW * 32];
                const float tc = fast_tanh(in4);
                const float dht = in6 + dh;
                const float dct = dc + dht * og * (1.f - tc * tc);
                da[0] = dct * gg * ig * (1.f - ig);
                da[1] = dct * in5 * fg * (1.f - fg);
                da[2] = dct * ig * (1.f - gg * gg);
                da[3] = dht * tc * og * (1.f - og);
                dc = dct * fg;
            }
            // exchange buffer (unit-major, r' = 4*j + g): the four gates of (unit j, batch row bb) are 8
            // contiguous bytes -> ONE direct store per thread, no staging and no extra block barrier on the
            // critical path (rows bb >= B carry zeros)
            __nv_bfloat162 lo = __floats2bfloat162_rn(da[0], da[1]), hi = __floats2bfloat162_rn(da[2], da[3]);
            uint2 pk;
            pk.x = *reinterpret_cast<uint32_t*>(&lo);
            pk.y = *reinterpret_cast<uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(gcur + (size_t)bb * H4 + (size_t)j * 4) = pk;
            // gate-major staging for dG_t (weight-gradient GEMMs), stored after the barrier arrival
            sg[(bb * 4 + 0) * UPC + uu] = __low2bfloat16(lo);
            sg[(bb * 4 + 1) * UPC + uu] = __high2bfloat16(lo);
            sg[(bb * 4 + 2) * UPC + uu] = __low2bfloat16(hi);
            sg[(bb * 4 + 3) * UPC + uu] = __high2bfloat16(hi);
        }
        __syncthreads();
        ++epoch;
        TC_STAMP(T - 1 - t, 1);
        if (tid == 0) { __threadfence(); atomicAdd(my_ctr, 1u); }
        TC_STAMP(T - 1 - t, 2);
        if (tid < NB * 4) {   // off the critical path: dG_t in the standard gate-major layout, 16-byte stores
            const int b = tid >> 2, c = tid & 3;
            const int jb = js * JS + rs * UPC;
            if (b < B) *reinterpret_cast<uint4*>(p.dg16 + (size_t)rowof(b, t) * H4 + (size_t)c * H + jb) =
                *reinterpret_cast<const uint4*>(sg + (b * 4 + c) * UPC);
        }
        EB_PREFETCH(t - 1)                                   // overlaps the wait
        if (p.wpoll) {
            if (l == 0) spin_wait_ge(wait_ctr, epoch * nprod);
            __syncwarp();
        } else {
            if (tid == 0) spin_wait_ge(wait_ctr, epoch * nprod);  // one poller per CTA (see forward kernel)
            TC_STAMP(T - 1 - t, 3);
            __syncthreads();
        }
        TC_STAMP(T - 1 - t, 4);
        // ---- phase B: partial dh_rec[unit (JS), batch] over this CTA's K-slice of dG_t
        // (staggering the warps' pulls by 64-192 cycles lets warp 0 start its HMMAs 900 cycles earlier but leaves the step unchanged:
        //  the last warp's range arrives when it did before -- measured, removed)
        warp_pull(gs + ks0 * 16, KP, gcur + r0 + ks0 * 16, H4, myks * 2, NB);
        TC_STAMP(T - 1 - t, 5);
        float acc[MT][4][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KSMAX; ++ks) {
            if (ks < myks) {
                uint32_t b01[4], b23[4];
                load_b<4>(b01, b23, gs, KP, ks0 + ks);
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    mma_bf16(acc[mt][0], afr[mt][ks], b01[0], b01[1]);
                    mma_bf16(acc[mt][1], afr[mt][ks], b01[2], b01[3]);
                    mma_bf16(acc[mt][2], afr[mt][ks], b23[0], b23[1]);
                    mma_bf16(acc[mt][3], afr[mt][ks], b23[2], b23[3]);
                }
            }
        }
        TC_STAMP(T - 1 - t, 6);
        // cross-warp reduction: red[w][slot][lane], slot = mt*16 + nt*4 + i
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) red[(w * SLOTS + mt * 16 + nt * 4 + i) * 32 + l] = acc[mt][nt][i];
        __syncthreads();
        TC_STAMP(T - 1 - t, 7);
        // SLOTS/NW slots per thread: slot -> (mt = slot/16, nt = (slot/4)%4, i = slot%4)
#pragma unroll
        for (int q = 0; q < SLOTS / NW; ++q) {
            const int slot = w * (SLOTS / NW) + q;
            float s = 0.f;
#pragma unroll
            for (int sw = 0; sw < NW; ++sw) s += red[(sw * SLOTS + slot) * 32 + l];
            const int mt = slot >> 4, nt = (slot >> 2) & 3, i = slot & 3;
            const int unit = mt * 16 + (l >> 2) + (i >> 1) * 8;
            const int bcol = nt * 8 + (l & 3) * 2 + (i & 1);
            if (CLUSTER) part[((t & 1) * JS + unit) * NB + bcol] = s;
            else p.pglob[((((size_t)(t & 1) * gridDim.x / CS + js) * CS + rs) * JS + unit) * NB + bcol] = s;
        }
        TC_STAMP(T - 1 - t, 8);
        if (CLUSTER) {
            // reduce-scatter of the partial tiles: each CTA hands the three 1 KB slices of its tile that belong to its
            // peers to the copy engine (DSMEM bulk copies completing on the destination's mbarrier) and adds the three
            // it receives to its own slice.  (cluster.sync() + remote loads measured 1780 cycles per step here.)
            fence_proxy_async_smem();
            __syncthreads();
            const uint32_t ph = (uint32_t)((T - 1 - t) & 1);
            if (tid == 0) mbar_expect_tx(rbar, (CS - 1) * UPC * NB * 4);
            if (tid < CS && tid != rs)
                bulk_s2c(map_to_rank(smem_u32(recvp + (((t & 1) * CS + rs) * UPC) * NB), (uint32_t)tid),
                         smem_u32(part + ((t & 1) * JS + tid * UPC) * NB), UPC * NB * 4, map_to_rank(rbar, (uint32_t)tid));
            TC_STAMP(T - 1 - t, 9);
            mbar_wait_cluster(rbar, ph);
            float s = part[((t & 1) * JS + rs * UPC + uu) * NB + bb];
#pragma unroll
            for (int c = 0; c < CS; ++c)
                if (c != rs) s += recvp[(((t & 1) * CS + c) * UPC + uu) * NB + bb];
            dh = s;                                          // dh_rec for (unit j, batch l) at step t-1
            TC_STAMP(T - 1 - t, 10);
            // `part` / `recvp` are double buffered by step parity: a buffer is rewritten two steps later, and the grid
            // barrier in between is passed only after every CTA of the cluster has consumed it.
        } else {
            __syncthreads();
            if (tid == 0) {
                __threadfence();
                atomicAdd(p.gbar + js, 1u);
                spin_wait_ge(p.gbar + js, (unsigned)CS * (unsigned)(T - t));
            }
            __syncthreads();
            float s = 0.f;
#pragma unroll
            for (int c = 0; c < CS; ++c)
                s += __ldcg(p.pglob + ((((size_t)(t & 1) * gridDim.x / CS + js) * CS + c) * JS + rs * UPC + uu) * NB + bb);
            dh = s;
        }
    }
#undef EB_PREFETCH
    if (own) {
        p.dh0[(long)bb * H + j] = dh;
        p.dc0[(long)bb * H + j] = dc;
    }
    if (CLUSTER) cluster_sync_all();                         // no CTA exits while a copy may still target its smem
}

inline bool tc_ok(int B, int H) { return H % 64 == 0 && H <= 1024 && B >= 1; }

template <int CS>
size_t bwd_smem(int H) {
    return (size_t)NB * (4 * H / CS + PAD) * 2 + sizeof(float) * (NW * (CS / 2) * 16 * 32 + 2 * 8 * CS * NB) + NB * 4 * UPC * 2 +
           sizeof(float) * 4 * NW * 32 + sizeof(float) * 2 * CS * UPC * NB + 16;
}

inline bool bwd_remap() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("EDGEDICT_LSTM_BWD_REMAP"); v = (e && atoi(e) == 0) ? 0 : 1; }
    return v == 1;
}

template <int CS>
int max_clusters(int H) {
    auto kern = lstm_tc_bwd_kernel<CS, true>;
    const size_t smem = bwd_smem<CS>(H);
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        (void)cudaGetLastError();
        return -2;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(H / 8);
    cfg.blockDim = dim3(NW * 32);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = CS; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) { (void)cudaGetLastError(); return -3; }
    return n;
}

template <int CS>
bool launch_cluster(const BwdP& p, int H, cudaStream_t st) {
    auto kern = bwd_remap() ? lstm_tc_bwd_kernel<CS, true, true> : lstm_tc_bwd_kernel<CS, true, false>;
    const size_t smem = bwd_smem<CS>(H);
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        (void)cudaGetLastError();
        return false;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(H / 8);
    cfg.blockDim = dim3(NW * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeClusterDimension;
    attrs[0].val.clusterDim.x = CS; attrs[0].val.clusterDim.y = 1; attrs[0].val.clusterDim.z = 1;
    attrs[1].id = cudaLaunchAttributeCooperative;
    attrs[1].val.cooperative = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = 2;
    if (cudaLaunchKernelEx(&cfg, kern, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    return true;
}

// cluster size to use for hidden size H: largest of 8/4/2 whose H/(8*CS) clusters are co-resident;
// 0 = software (L2) reduction.  EDGEDICT_LSTM_CLUSTER=<0|2|4|8> overrides.
int pick_cs(int H) {
    static int cache[17];          // index H/64
    static bool init = false;
    if (!init) { for (int& c : cache) c = -1; init = true; }
    int& c = cache[H / 64];
    if (c >= 0) return c;
    const char* e = getenv("EDGEDICT_LSTM_CLUSTER");
    if (e) {
        const int v = atoi(e);
        c = (v == 8 || v == 4 || v == 2) ? v : 0;
        return c;
    }
    if (max_clusters<8>(H) >= H / 64) c = 8;
    else if (max_clusters<4>(H) >= H / 32) c = 4;
    else if (max_clusters<2>(H) >= H / 16) c = 2;
    else c = 0;
    return c;
}

// ---- GRU layer on tensor cores (nn.GRU, gate order r|z|n; bf16 operands, fp32 accumulation and state) -------------
// Forward: CTA k owns the 16 hidden units [16k, 16k+16) as three m16 tiles of W_hh rows -- (r|z of units 0-7),
// (r|z of units 8-15), (n of units 0-15) -- held in registers as A fragments (each warp a K-range of H/8 columns:
// 3 x 8 x 4 = 96 registers at H = 1024); h_{t-1} is exchanged in bf16 as in lstm_tc_fwd_kernel, the fp32 state stays in
// registers of the thread that owns the (unit, batch row) pair, and b_hn is added to the n-row sum inside the reset
// product.  Saves r | z | n | gh_n (fp32, [B,T,4H]) as the fp32 kernel does.
// BPTT: CTA k owns the same 16 units, now as the output rows of dh_rec = W_hh^T dgh; the contraction runs over all 3H
// rows of dgh (each warp a K-range of 3H/8 rows: 24 k-steps x 4 = 96 registers at H = 1024).  dgh_t is exchanged in
// bf16 ([NB][3H], gate-major), the direct term dh z is carried in fp32 registers.
constexpr int GU = 16;           // hidden units per CTA
constexpr int GRS = 33;          // padded lane stride of the cross-warp reduction buffer

// the caller has pulled this warp's K-range into `tile`; the warp's partial products -> red[w][slot][lane],
// slot = (mt * 4 + nt) * 4 + i
template <int MT, int KSM>
__device__ __forceinline__ void gru_contract(const uint32_t (&afr)[MT][KSM][4], const __nv_bfloat16* tile, int ld,
                                             int ks0, int myks, float* red) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    float acc[MT][4][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KSM; ++ks) {
        if (ks < myks) {
            uint32_t b01[4], b23[4];
            load_b<4>(b01, b23, tile, ld, ks0 + ks);
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                mma_bf16(acc[mt][0], afr[mt][ks], b01[0], b01[1]);
                mma_bf16(acc[mt][1], afr[mt][ks], b01[2], b01[3]);
                mma_bf16(acc[mt][2], afr[mt][ks], b23[0], b23[1]);
                mma_bf16(acc[mt][3], afr[mt][ks], b23[2], b23[3]);
            }
        }
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) red[(w * MT * 16 + (mt * 4 + nt) * 4 + i) * GRS + l] = acc[mt][nt][i];
}

// sum over the 8 warps of the accumulator element at (tile mt, tile row `row` 0-15, batch column b)
__device__ __forceinline__ float gru_red_sum(const float* red, int MT, int mt, int row, int b) {
    const int lane = (row & 7) * 4 + ((b & 7) >> 1);
    const int slot = (mt * 4 + (b >> 3)) * 4 + (row >> 3) * 2 + (b & 1);
    float s = 0.f;
#pragma unroll
    for (int sw = 0; sw < NW; ++sw) s += red[(sw * MT * 16 + slot) * GRS + lane];
    return s;
}

struct GruFwdP {
    const float* xg;              // [B,T,3H] fp32 (b_hr, b_hz folded in)
    const __nv_bfloat16* whh;     // [3H,H] bf16
    const float* bhn; const float* h0;
    float* y; float* hT; float* save;
    __nv_bfloat16* hx;            // [2][NB][H] exchange
    unsigned* bar;
    int B, T, H;
};

__global__ void __launch_bounds__(NW * 32, 1) gru_tc_fwd_kernel(GruFwdP p) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int H = p.H, B = p.B, T = p.T;
    const long H3 = 3 * (long)H;
    const int HP = H + PAD;
    __nv_bfloat16* hs = reinterpret_cast<__nv_bfloat16*>(smraw);                 // [NB][HP]
    float* red = reinterpret_cast<float*>(smraw + (size_t)NB * HP * 2);          // [NW][48][GRS]
    __nv_bfloat16* sh_h = reinterpret_cast<__nv_bfloat16*>(red + NW * 48 * GRS);  // [NB][GU]
    const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
    const int j0 = blockIdx.x * GU;
    const unsigned ncta = gridDim.x;
    const int nks = H / 16;
    const int ksper = (nks + NW - 1) / NW;                   // <= 8
    const int ks0 = w * ksper;
    const int myks = max(0, min(ksper, nks - ks0));
    const size_t xstride = (size_t)NB * H;

    // A fragments: tile mt rows lo (fragment row l/4) and hi (l/4 + 8) as W_hh rows
    uint32_t afr[3][8][4];
#pragma unroll
    for (int mt = 0; mt < 3; ++mt)
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            const int k = (ks0 + ks) * 16 + (l & 3) * 2;
            const int u = l >> 2;
            const long rlo = mt == 2 ? 2 * (long)H + j0 + u : (long)j0 + mt * 8 + u;
            const long rhi = mt == 2 ? 2 * (long)H + j0 + 8 + u : (long)H + j0 + mt * 8 + u;
            const bool ok = ks < myks;
            afr[mt][ks][0] = ok ? ldg_u32(p.whh + rlo * H + k) : 0u;
            afr[mt][ks][1] = ok ? ldg_u32(p.whh + rhi * H + k) : 0u;
            afr[mt][ks][2] = ok ? ldg_u32(p.whh + rlo * H + k + 8) : 0u;
            afr[mt][ks][3] = ok ? ldg_u32(p.whh + rhi * H + k + 8) : 0u;
        }

    // the two (unit, batch row) pairs this thread finalises every step: (w, l) and (w + 8, l)
    const int bb = l;
    const bool own = bb < B;
    float h_state[2], bn[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const int j = j0 + w + 8 * q;
        h_state[q] = (own && p.h0) ? p.h0[(long)bb * H + j] : 0.f;
        bn[q] = p.bhn ? p.bhn[j] : 0.f;
        if (own) p.hx[xstride + (long)bb * H + j] = __float2bfloat16(h_state[q]);
    }
    __syncthreads();
    if (tid == 0) { __threadfence(); atomicAdd(p.bar, 1u); }
    unsigned epoch = 1;

    for (int t = 0; t < T; ++t) {
        const __nv_bfloat16* hprev = p.hx + ((t + 1) & 1) * xstride;
        __nv_bfloat16* hnext = p.hx + (t & 1) * xstride;
        float px[2][3];                                      // input pre-activations, loaded before the wait
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int g = 0; g < 3; ++g)
                px[q][g] = own ? __ldg(p.xg + ((long)bb * T + t) * H3 + (long)g * H + j0 + w + 8 * q) : 0.f;
        if (tid == 0) spin_wait_ge(p.bar, epoch * ncta);
        __syncthreads();
        warp_pull(hs + ks0 * 16, HP, hprev + ks0 * 16, H, myks * 2, NB);
        gru_contract<3, 8>(afr, hs, HP, ks0, myks, red);
        __syncthreads();
        float rg[2], zg[2], ng[2], ghn[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int u = w + 8 * q;                         // tile rows: r, z in tile u/8, n in tile 2
            rg[q] = fast_sigmoid(gru_red_sum(red, 3, q, w, bb) + px[q][0]);
            zg[q] = fast_sigmoid(gru_red_sum(red, 3, q, 8 + w, bb) + px[q][1]);
            ghn[q] = gru_red_sum(red, 3, 2, u, bb) + bn[q];
            ng[q] = fast_tanh(px[q][2] + rg[q] * ghn[q]);
            h_state[q] = (1.f - zg[q]) * ng[q] + zg[q] * h_state[q];
            sh_h[bb * GU + u] = __float2bfloat16(own ? h_state[q] : 0.f);
        }
        __syncthreads();
        if (w == 0) {   // publish h_t: two 16-byte stores per batch row, then a single fence + arrive
            const uint4* src = reinterpret_cast<const uint4*>(sh_h + l * GU);
            uint4* dst = reinterpret_cast<uint4*>(hnext + (size_t)l * H + j0);
            dst[0] = src[0];
            dst[1] = src[1];
            __syncwarp();
            if (l == 0) { __threadfence(); atomicAdd(p.bar, 1u); }
        }
        ++epoch;
        if (own) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int j = j0 + w + 8 * q;
                const long row = (long)bb * T + t;
                p.y[row * H + j] = h_state[q];
                if (p.save) {
                    float* sp = p.save + row * 4 * H + j;
                    sp[0] = rg[q]; sp[H] = zg[q]; sp[2 * (long)H] = ng[q]; sp[3 * (long)H] = ghn[q];
                }
                if (t == T - 1) p.hT[(long)bb * H + j] = h_state[q];
            }
        }
    }
}

struct GruBwdP {
    const float* dy; const float* save; const float* y; const float* h0;
    const __nv_bfloat16* whhT;    // [H,3H] bf16 = W_hh^T
    const float* dhT;
    __nv_bfloat16* dgi16; __nv_bfloat16* dgh16;   // [B,T,3H] bf16 out
    float* dh0;
    __nv_bfloat16* gx;            // [2][NB][3H] exchange
    unsigned* bar;
    int B, T, H;
};

__global__ void __launch_bounds__(NW * 32, 1) gru_tc_bwd_kernel(GruBwdP p) {
    constexpr int KSM = 24;                                  // k-steps per warp at H = 1024: 3H / 16 / NW
    extern __shared__ __align__(16) unsigned char smraw[];
    const int H = p.H, B = p.B, T = p.T;
    const int H3 = 3 * H;
    const int KP = H3 + PAD;
    __nv_bfloat16* gs = reinterpret_cast<__nv_bfloat16*>(smraw);                 // [NB][KP]
    float* red = reinterpret_cast<float*>(smraw + (size_t)NB * KP * 2);          // [NW][16][GRS]
    __nv_bfloat16* sg = reinterpret_cast<__nv_bfloat16*>(red + NW * 16 * GRS);    // [NB][3][GU]
    const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
    const int j0 = blockIdx.x * GU;
    const unsigned ncta = gridDim.x;
    const int nks = H3 / 16;
    const int ksper = (nks + NW - 1) / NW;                   // <= KSM
    const int ks0 = w * ksper;
    const int myks = max(0, min(ksper, nks - ks0));
    const size_t xstride = (size_t)NB * H3;

    // A(m = unit u, k = gate row r) = W_hh[r, j0 + u] = whhT[j0 + u][r]: consecutive k are contiguous in whhT
    uint32_t afr[1][KSM][4];
#pragma unroll
    for (int ks = 0; ks < KSM; ++ks) {
        const int k = (ks0 + ks) * 16 + (l & 3) * 2;
        const long ulo = j0 + (l >> 2), uhi = ulo + 8;
        const bool ok = ks < myks;
        afr[0][ks][0] = ok ? ldg_u32(p.whhT + ulo * H3 + k) : 0u;
        afr[0][ks][1] = ok ? ldg_u32(p.whhT + uhi * H3 + k) : 0u;
        afr[0][ks][2] = ok ? ldg_u32(p.whhT + ulo * H3 + k + 8) : 0u;
        afr[0][ks][3] = ok ? ldg_u32(p.whhT + uhi * H3 + k + 8) : 0u;
    }

    const int bb = l;
    const bool own = bb < B;
    float dh_rec[2];                                         // dh_{t} minus dy_t: dh_{t+1} z_{t+1} + W_hh^T dgh_{t+1}
#pragma unroll
    for (int q = 0; q < 2; ++q) dh_rec[q] = (own && p.dhT) ? p.dhT[(long)bb * H + j0 + w + 8 * q] : 0.f;
    unsigned epoch = 0;

    for (int t = T - 1; t >= 0; --t) {
        __nv_bfloat16* gcur = p.gx + (t & 1) * xstride;
        float carry[2];
        // phase A: gate gradients of step t for the owned pairs
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int u = w + 8 * q, j = j0 + u;
            float dr = 0.f, dz = 0.f, dn = 0.f, dhn = 0.f;
            carry[q] = 0.f;
            if (own) {
                const long row = (long)bb * T + t;
                const float* sp = p.save + row * 4 * H + j;
                const float rg = sp[0], zg = sp[H], ng = sp[2 * (long)H], ghn = sp[3 * (long)H];
                const float hp = (t > 0) ? p.y[(row - 1) * H + j] : (p.h0 ? p.h0[(long)bb * H + j] : 0.f);
                const float dh = p.dy[row * H + j] + dh_rec[q];
                dn = dh * (1.f - zg) * (1.f - ng * ng);
                dz = dh * (hp - ng) * zg * (1.f - zg);
                dr = dn * ghn * rg * (1.f - rg);
                dhn = rg * dn;
                carry[q] = dh * zg;
                __nv_bfloat16* gi = p.dgi16 + row * H3 + j;
                __nv_bfloat16* gh = p.dgh16 + row * H3 + j;
                gi[0] = gh[0] = __float2bfloat16(dr);
                gi[H] = gh[H] = __float2bfloat16(dz);
                gi[2 * (long)H] = __float2bfloat16(dn);
                gh[2 * (long)H] = __float2bfloat16(dhn);
            }
            sg[(bb * 3 + 0) * GU + u] = __float2bfloat16(dr);
            sg[(bb * 3 + 1) * GU + u] = __float2bfloat16(dz);
            sg[(bb * 3 + 2) * GU + u] = __float2bfloat16(dhn);
        }
        __syncthreads();
        if (tid < NB * 3 * 2) {   // publish dgh_t: rows b, gates g, two 16-byte halves of the 16 units
            const int b = tid / 6, g = (tid >> 1) % 3, half = tid & 1;
            *reinterpret_cast<uint4*>(gcur + (size_t)b * H3 + (size_t)g * H + j0 + half * 8) =
                *reinterpret_cast<const uint4*>(sg + (b * 3 + g) * GU + half * 8);
        }
        __syncthreads();
        ++epoch;
        if (tid == 0) {
            __threadfence();
            atomicAdd(p.bar, 1u);
            spin_wait_ge(p.bar, epoch * ncta);
        }
        __syncthreads();
        // phase B: dh_rec = dh z + W_hh^T dgh_t for the owned pairs
        warp_pull(gs + ks0 * 16, KP, gcur + ks0 * 16, H3, myks * 2, NB);
        gru_contract<1, KSM>(afr, gs, KP, ks0, myks, red);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 2; ++q) dh_rec[q] = carry[q] + gru_red_sum(red, 1, 0, w + 8 * q, bb);
    }
    if (own) {
#pragma unroll
        for (int q = 0; q < 2; ++q) p.dh0[(long)bb * H + j0 + w + 8 * q] = dh_rec[q];
    }
}

inline size_t gru_tc_fwd_smem(int H) {
    return (size_t)NB * (H + PAD) * 2 + sizeof(float) * NW * 48 * GRS + NB * GU * 2;
}
inline size_t gru_tc_bwd_smem(int H) {
    return (size_t)NB * (3 * H + PAD) * 2 + sizeof(float) * NW * 16 * GRS + NB * 3 * GU * 2;
}

}  // namespace

// debug: clock64 stamps of CTA 0 of the BPTT kernel for the first `steps` steps of subsequent launches ([steps][16] int64)
EB_API int eb_lstm_tc_set_trace(void* dev_buf, int steps) {
    g_tc_trace = reinterpret_cast<long long*>(dev_buf);
    g_tc_trace_steps = dev_buf ? steps : 0;
    return EB_OK;
}

EB_API int eb_lstm_tc_supported(int B, int H) { return tc_ok(B, H) ? 1 : 0; }

EB_API size_t eb_lstm_tc_scratch_bytes(int B, int H) {
    if (!tc_ok(B, H)) return 0;
    return TC_HDR + sizeof(__nv_bfloat16) * (size_t)2 * NB * 4 * H + sizeof(float) * (size_t)2 * (H / 8) * 64 * NB;
}

// co-resident clusters of `cs` CTAs of the BPTT kernel (diagnostic + path selection)
EB_API int eb_lstm_tc_max_clusters(int H, int cs) {
    if (H % 64 || H > 1024) return -1;
    if (cs == 8) return max_clusters<8>(H);
    if (cs == 4) return max_clusters<4>(H);
    if (cs == 2) return max_clusters<2>(H);
    return -1;
}

// xg [B,T,4H] fp32; whh16 [4H,H] bf16.  B > 32 is processed in batch tiles of 32 (independent
// utterances), one launch per tile.
EB_API int eb_lstm_tc_fwd(const float* xg, const void* whh16, const float* h0, const float* c0, float* y,
                          void* y16, float* hT, float* cT, float* gates_save, float* cseq_save,
                          void* scratch, int B, int T, int H, void* stream) {
    if (!xg || !whh16 || !y || !hT || !cT || !scratch || T <= 0 || !tc_ok(B, H)) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t smem = (size_t)NBT * (H + PAD) * 2 + sizeof(float) * NW * (NBT / 8) * 8 * 32 + NBT * UPC * 2 +
                        sizeof(float) * 4 * NW * 32;
    EB_CUDA(cudaFuncSetAttribute(lstm_tc_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int b0 = 0; b0 < B; b0 += NB) {
        const int nb = (B - b0 < NB) ? (B - b0) : NB;
        FwdP p;
        p.xg = xg + (size_t)b0 * T * 4 * H;
        p.whh = reinterpret_cast<const __nv_bfloat16*>(whh16);
        p.h0 = h0 ? h0 + (size_t)b0 * H : nullptr;
        p.c0 = c0 ? c0 + (size_t)b0 * H : nullptr;
        p.y = y + (size_t)b0 * T * H;
        p.y16 = y16 ? reinterpret_cast<__nv_bfloat16*>(y16) + (size_t)b0 * T * H : nullptr;
        p.hT = hT + (size_t)b0 * H;
        p.cT = cT + (size_t)b0 * H;
        p.gates = gates_save ? gates_save + (size_t)b0 * T * 4 * H : nullptr;
        p.cseq = cseq_save ? cseq_save + (size_t)b0 * T * H : nullptr;
        p.bar = reinterpret_cast<unsigned*>(scratch);
        p.hx = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<char*>(scratch) + TC_HDR);
        p.B = nb; p.T = T; p.H = H;
        EB_CUDA(cudaMemsetAsync(scratch, 0, TC_HDR + sizeof(__nv_bfloat16) * (size_t)2 * NB * H, st));
        void* args[] = {&p};
        EB_CUDA(cudaLaunchCooperativeKernel((void*)lstm_tc_fwd_kernel, dim3(H / UPC), dim3(NW * 32), args, smem, st));
    }
    return EB_OK;
}

static int tc_bwd_impl(const float* dy, const float* gates, const float* cseq, const float* c0,
                       const void* whhT16, const float* dhT, const float* dcT, void* dg16, float* dh0,
                       float* dc0, void* scratch, int B, int T, int H, const int* lens, int nseg, void* stream);

// whhT16 [H,4H] bf16 (W_hh transposed).  dg16 [B,T,4H] bf16 out; dh0/dc0 [B,H] fp32 out.
EB_API int eb_lstm_tc_bwd(const float* dy, const float* gates, const float* cseq, const float* c0,
                          const void* whhT16, const float* dhT, const float* dcT, void* dg16, float* dh0,
                          float* dc0, void* scratch, int B, int T, int H, void* stream) {
    return tc_bwd_impl(dy, gates, cseq, c0, whhT16, dhT, dcT, dg16, dh0, dc0, scratch, B, T, H, &T, 1, stream);
}

// The same recurrence over a time axis stored chunk-major (the layer wavefront's buffers): chunk c, chunk_lens[c] steps,
// is a contiguous [B, chunk_lens[c], D] block and the blocks follow each other -- ONE launch walks all chunks (T = their
// sum) instead of one launch per chunk with the (dh, dc) carry through memory.  nchunks <= 8; chunk_lens is a host array.
EB_API int eb_lstm_tc_bwd_chunks(const float* dy, const float* gates, const float* cseq, const float* c0,
                                 const void* whhT16, const float* dhT, const float* dcT, void* dg16, float* dh0,
                                 float* dc0, void* scratch, int B, const int* chunk_lens, int nchunks, int H,
                                 void* stream) {
    if (!chunk_lens || nchunks < 1 || nchunks > 8) return EB_ERR_INVALID;
    long T = 0;
    for (int c = 0; c < nchunks; ++c) {
        if (chunk_lens[c] <= 0) return EB_ERR_INVALID;
        T += chunk_lens[c];
    }
    if (T > 0x7fffffffL) return EB_ERR_INVALID;
    return tc_bwd_impl(dy, gates, cseq, c0, whhT16, dhT, dcT, dg16, dh0, dc0, scratch, B, (int)T, H, chunk_lens, nchunks,
                       stream);
}

static int tc_bwd_impl(const float* dy, const float* gates, const float* cseq, const float* c0,
                       const void* whhT16, const float* dhT, const float* dcT, void* dg16, float* dh0,
                       float* dc0, void* scratch, int B, int T, int H, const int* lens, int nseg, void* stream) {
    if (!dy || !gates || !cseq || !whhT16 || !dg16 || !dh0 || !dc0 || !scratch || T <= 0 || !tc_ok(B, H))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int cs = pick_cs(H);
    char* base = reinterpret_cast<char*>(scratch);
    for (int b0 = 0; b0 < B; b0 += NB) {
        const int nb = (B - b0 < NB) ? (B - b0) : NB;
        BwdP p;
        p.dy = dy; p.gates = gates; p.cseq = cseq;           // batch tile and time segments are applied by rowof()
        p.b0 = b0; p.Btot = B; p.nseg = nseg;
        p.seg_off[0] = 0;
        for (int c = 0; c < 8; ++c) p.seg_off[c + 1] = c < nseg ? p.seg_off[c] + lens[c] : T;
        p.c0 = c0 ? c0 + (size_t)b0 * H : nullptr;
        p.whhT = reinterpret_cast<const __nv_bfloat16*>(whhT16);
        p.dhT = dhT ? dhT + (size_t)b0 * H : nullptr;
        p.dcT = dcT ? dcT + (size_t)b0 * H : nullptr;
        p.dg16 = reinterpret_cast<__nv_bfloat16*>(dg16);
        p.dh0 = dh0 + (size_t)b0 * H;
        p.dc0 = dc0 + (size_t)b0 * H;
        p.bar = reinterpret_cast<unsigned*>(base);
        p.gbar = reinterpret_cast<unsigned*>(base + 8192);
        p.gx = reinterpret_cast<__nv_bfloat16*>(base + TC_HDR);
        p.pglob = reinterpret_cast<float*>(base + TC_HDR + sizeof(__nv_bfloat16) * (size_t)2 * NB * 4 * H);
        p.B = nb; p.T = T; p.H = H;
        p.trace = g_tc_trace; p.trace_steps = g_tc_trace_steps;
        { static int wp = -1; if (wp < 0) { const char* e = getenv("EDGEDICT_LSTM_WPOLL"); wp = e ? atoi(e) : 3; } p.wpoll = wp & 2; }
        EB_CUDA(cudaMemsetAsync(scratch, 0, TC_HDR + sizeof(__nv_bfloat16) * (size_t)2 * NB * 4 * H, st));
        bool launched = false;
        if (cs == 8) launched = launch_cluster<8>(p, H, st);
        else if (cs == 4) launched = launch_cluster<4>(p, H, st);
        else if (cs == 2) launched = launch_cluster<2>(p, H, st);
        if (!launched) {
            // software reduce-scatter through L2: plain cooperative grid, always co-resident
            auto kern = bwd_remap() ? lstm_tc_bwd_kernel<4, false, true> : lstm_tc_bwd_kernel<4, false, false>;
            const size_t smem = bwd_smem<4>(H);
            EB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            void* args[] = {&p};
            EB_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(H / 8), dim3(NW * 32), args, smem, st));
        }
    }
    return EB_OK;
}

// ---- GRU entry points (bf16 mode; H % 64 == 0, H <= 1024) -------------------------------------------------------------
static inline bool gru_tc_ok(int B, int H) { return H > 0 && tc_ok(B, H); }

EB_API int eb_gru_tc_supported(int B, int H) { return gru_tc_ok(B, H) ? 1 : 0; }

EB_API size_t eb_gru_tc_scratch_bytes(int B, int H) {
    if (!gru_tc_ok(B, H)) return 0;
    return TC_HDR + sizeof(__nv_bfloat16) * (size_t)2 * NB * 3 * H;
}

// xg [B,T,3H] fp32 (b_hr, b_hz folded in); whh16 [3H,H] bf16; bhn [H] fp32 (NULL: zero).  B > 32: batch tiles of 32.
EB_API int eb_gru_tc_fwd(const float* xg, const void* whh16, const float* bhn, const float* h0, float* y, float* hT,
                         float* save, void* scratch, int B, int T, int H, void* stream) {
    if (!xg || !whh16 || !y || !hT || !scratch || T <= 0 || !gru_tc_ok(B, H)) return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(whh16) & 3) || (reinterpret_cast<uintptr_t>(scratch) & 15)) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t smem = gru_tc_fwd_smem(H);
    EB_CUDA(cudaFuncSetAttribute(gru_tc_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int b0 = 0; b0 < B; b0 += NB) {
        const int nb = (B - b0 < NB) ? (B - b0) : NB;
        GruFwdP p;
        p.xg = xg + (size_t)b0 * T * 3 * H;
        p.whh = reinterpret_cast<const __nv_bfloat16*>(whh16);
        p.bhn = bhn;
        p.h0 = h0 ? h0 + (size_t)b0 * H : nullptr;
        p.y = y + (size_t)b0 * T * H;
        p.hT = hT + (size_t)b0 * H;
        p.save = save ? save + (size_t)b0 * T * 4 * H : nullptr;
        p.bar = reinterpret_cast<unsigned*>(scratch);
        p.hx = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<char*>(scratch) + TC_HDR);
        p.B = nb; p.T = T; p.H = H;
        EB_CUDA(cudaMemsetAsync(scratch, 0, TC_HDR + sizeof(__nv_bfloat16) * (size_t)2 * NB * H, st));
        void* args[] = {&p};
        EB_CUDA(cudaLaunchCooperativeKernel((void*)gru_tc_fwd_kernel, dim3(H / GU), dim3(NW * 32), args, smem, st));
    }
    return EB_OK;
}

// whhT16 [H,3H] bf16 (W_hh transposed); dgi16 / dgh16 [B,T,3H] bf16 out; dh0 [B,H] fp32 out.
EB_API int eb_gru_tc_bwd(const float* dy, const float* save, const float* y, const float* h0, const void* whhT16,
                         const float* dhT, void* dgi16, void* dgh16, float* dh0, void* scratch, int B, int T, int H,
                         void* stream) {
    if (!dy || !save || !y || !whhT16 || !dgi16 || !dgh16 || !dh0 || !scratch || T <= 0 || !gru_tc_ok(B, H))
        return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(whhT16) & 3) || (reinterpret_cast<uintptr_t>(scratch) & 15)) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t smem = gru_tc_bwd_smem(H);
    EB_CUDA(cudaFuncSetAttribute(gru_tc_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int b0 = 0; b0 < B; b0 += NB) {
        const int nb = (B - b0 < NB) ? (B - b0) : NB;
        GruBwdP p;
        p.dy = dy + (size_t)b0 * T * H;
        p.save = save + (size_t)b0 * T * 4 * H;
        p.y = y + (size_t)b0 * T * H;
        p.h0 = h0 ? h0 + (size_t)b0 * H : nullptr;
        p.whhT = reinterpret_cast<const __nv_bfloat16*>(whhT16);
        p.dhT = dhT ? dhT + (size_t)b0 * H : nullptr;
        p.dgi16 = reinterpret_cast<__nv_bfloat16*>(dgi16) + (size_t)b0 * T * 3 * H;
        p.dgh16 = reinterpret_cast<__nv_bfloat16*>(dgh16) + (size_t)b0 * T * 3 * H;
        p.dh0 = dh0 + (size_t)b0 * H;
        p.bar = reinterpret_cast<unsigned*>(scratch);
        p.gx = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<char*>(scratch) + TC_HDR);
        p.B = nb; p.T = T; p.H = H;
        EB_CUDA(cudaMemsetAsync(scratch, 0, TC_HDR + sizeof(__nv_bfloat16) * (size_t)2 * NB * 3 * H, st));
        void* args[] = {&p};
        EB_CUDA(cudaLaunchCooperativeKernel((void*)gru_tc_bwd_kernel, dim3(H / GU), dim3(NW * 32), args, smem, st));
    }
    return EB_OK;
}
