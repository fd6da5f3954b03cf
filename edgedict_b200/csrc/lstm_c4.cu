// lstm_c4.cu -- persistent-RNN LSTM layer on wgmma tensor cores inside thread-block clusters (bf16 operands,
// fp32 accumulate / state): the bf16-mode recurrent kernels for H % 256 == 0, H <= 1024 (the encoder and predictor
// sizes of every BASELINE config except E4D1, which keeps lstm_tc.cu).
//
// Semantics: nn.LSTM cell, gate order i|f|g|o (rnnt/models.py:45-46 -> torch.nn.LSTM), one launch for all T steps.
//
// Decomposition (forward).  H/8 CTAs in clusters of 4.  Cluster g owns hidden units [32g, 32g+32) = 128 gate rows;
// the CTA of cluster rank r (a) finalises units [32g+8r, 32g+8r+8) and (b) contracts over the K slice
// [r*H/4, (r+1)*H/4) of h_{t-1} for ALL 128 gate rows of its cluster:
//   * its W_hh slice [128 x H/4] bf16 (64 KB at H = 1024) is staged ONCE into shared memory in the canonical
//     K-major 128B-swizzle layout and stays there for the whole sequence -- no weight lives in registers;
//   * per step the CTA waits on the grid barrier of its K slice, pulls the slice of h_{t-1} (32 x H/4 bf16 = 16 KB,
//     a quarter of what a full-K design pulls) into swizzled shared memory and its warpgroup issues wgmma
//     (M64 N32 K16), accumulator [128 gate rows x 32 batch] fp32 in registers;
//   * the four 32-row blocks of the accumulator are the partial sums destined to the four CTAs of the cluster: they
//     are staged in shared memory and the three remote ones are pushed into the peers' shared memory by DSMEM bulk
//     copies that complete on the destination's mbarrier -- no cluster-wide barrier;
//   * every CTA adds the four partials of its own 8 units, applies the gates thread-locally (two (unit, batch)
//     pairs per thread, cell state in registers), publishes h_t in bf16 (16 B per batch row) and arrives on the
//     grid barrier; y, the h_{t-1}-shifted bf16 copy for the weight-gradient GEMM and the saved gates / cell
//     states leave after the arrival, as full 16-byte / 8-byte coalesced stores in a CTA-private layout.
// Backward (BPTT): the same structure with the roles of the operands swapped: a cluster of CS CTAs owns 8*CS units;
// rank r contracts over the K slice [r*4H/CS, ...) of dG_t (wgmma M64 N32 K16: rows = units), and the gate-gradient
// math of step t-1 runs on the owning threads with dh/dc in registers.  CS = 16 (eb_lstm_c4_bwd_chunks, fp32
// standard-layout saves) is the forward's K-split design: a 16 KB pull per CTA and step, partial dh reduce-scattered
// with bulk DSMEM copies, one barrier counter per K slice.  CS = 8 / 4 (eb_lstm_c4_bwd, CTA-private bf16 saves; for
// CS = 4 rows 32-63 are discarded) push the partial dh tiles with st.shared::cluster behind one grid-wide counter.  The
// exchange buffer orders the contraction index unit-major, k' = 4*unit + gate (the layout of lstm_tc.cu), so that a
// thread publishes the eight gate gradients of its two units with one 16-byte store.
#include <cuda.h>
#include <stdlib.h>
#include "common.cuh"
#include "sm90.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int NB = 32;            // batch tile (rows of the exchange buffers, N of the MMA)
constexpr int UPC = 8;            // hidden units finalised per CTA
constexpr int RP = 36;            // floats per row of the DSMEM receive tiles (16-byte aligned, conflict-free)
// forward receive / staging tiles: [src or dest][32 rows][32 floats], 16-byte chunk c of row r stored at chunk c ^ (r & 7)
__device__ __forceinline__ int swz(int row, int b) { return row * 32 + ((((b >> 2) ^ (row & 7)) << 2) | (b & 3)); }
constexpr int NGT = 128;          // gate threads (warps 0-3, one warpgroup); backward: warp 4 = barrier poller / TMA
constexpr int NTHR = 160;
constexpr size_t C4_HDR = 16384;  // scratch: grid barrier counters, one per K slice (up to 16), 1 KB apart (different L2 slices)
constexpr int CTR_STRIDE = 256;   // uints between two slice counters

// debug stamps: slot s of step `step` <- clock64() (CTA 0 only; the pointer is null in production)
__device__ __forceinline__ long long gtimer() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// trace_steps > 0: clock64 stamps of CTA 0, [step][16].  trace_steps < 0: globaltimer stamps of EVERY CTA for the first
// -trace_steps steps, [step][cta][16] (skew between CTAs).
#define C4_STAMP(step, s)                                                                          \
    do {                                                                                           \
        if (p.trace) {                                                                             \
            if (p.trace_steps > 0) {                                                               \
                if (blockIdx.x == 0 && (step) < p.trace_steps) p.trace[(size_t)(step) * 16 + (s)] = clock64(); \
            } else if ((step) < -p.trace_steps)                                                    \
                p.trace[((size_t)(step) * gridDim.x + blockIdx.x) * 16 + (s)] = gtimer();          \
        }                                                                                          \
    } while (0)
long long* g_trace = nullptr;
int g_trace_steps = 0;

__device__ __forceinline__ float fsig(float x) { return __fdividef(1.f, 1.f + fast_exp(-x)); }
__device__ __forceinline__ float ftanh(float x) { return 1.f - __fdividef(2.f, fast_exp(2.f * x) + 1.f); }
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack2(uint32_t v) {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v));
}
__device__ __forceinline__ uint32_t cluster_id_x() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void named_bar_gate() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------
struct C4FwdP {
    const float* xg;              // [B,T,4H] fp32 input pre-activations (W_ih x + b_ih + b_hh)
    const __nv_bfloat16* whh;     // [4H,H] bf16
    const float* h0; const float* c0;
    float* y;                     // [B,T,H] fp32
    __nv_bfloat16* hprev16;       // [B,T,H] bf16: h_{t-1} (frame 0 = h0) -- operand of the dW_hh GEMM; may be null
    float* hT; float* cT;
    uint4* gsave;                 // [T][H/8][128] post-activation gates, bf16 (i0 i1 f0 f1 g0 g1 o0 o1); may be null
    float2* csave;                // [T][H/8][128] cell states; may be null
    __nv_bfloat16* hx;            // [2][NB][H] exchange
    unsigned* bar;                // grid barrier counters (one per K slice)
    long long* trace;             // debug: [steps][16] clock64 stamps of CTA 0 (eb_lstm_c4_set_trace), else null
    int trace_steps;
    float* gates_std; float* cseq_std;   // optional saves in the layout of eb_lstm_tc_bwd: [B,T,4H] gates, [B,T,H] cells (fp32)
    int wpoll;                    // every warp polls the barrier counter itself instead of one poller + block barrier
                                  // (EDGEDICT_LSTM_WPOLL bit 0 = this kernel, bit 1 = the BPTT kernel)
    int B, T, H;
};

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(saddr), "l"(gmem) : "memory");
}

// The CTA is one warpgroup.  Its W_hh slice [128 gate rows x H/4] stays in shared memory for the whole sequence; per step
// the warpgroup issues H/64 x 2 wgmma (M64 N32 K16: gate rows [0,64) and [64,128) against the 32 batch rows of h_{t-1}).
// Three CTAs per SM fit the register budget (168 per thread); two fit the shared memory at H = 1024.
__global__ void __launch_bounds__(NGT, 3) lstm_c4_fwd_kernel(C4FwdP p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int H = p.H, B = p.B, T = p.T;
    const int KS = H >> 2, NA = KS >> 6;                     // K slice per CTA, 64-wide swizzle atoms in it
    const int NC = H / UPC;
    const int CPR = KS >> 3;                                 // 16-byte chunks per row of the h slice (8 .. 32)
    const int NLD = CPR >> 2;                                // chunks per thread and step: 32 rows * CPR / 128
    uint8_t* sA = smem;                                      // [NA][128 rows][128 B]   W_hh slice, resident
    uint8_t* sB = sA + NA * 16384;                           // [NA][32 rows][128 B]    h_{t-1} slice of the step
    float* stage = reinterpret_cast<float*>(sB + 16384);     // [4 dest][32 rows][32]   outgoing partial tiles (swz)
    float* recv = stage + 4 * 1024;                          // [3 src][32 rows][32]    incoming partial tiles (swz)
    uint64_t* bars = reinterpret_cast<uint64_t*>(recv + 3 * 1024);
    const uint32_t rbar = smem_u32(bars);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t rank = cluster_ctarank();
    const int grp = (int)cluster_id_x();
    const int cta = grp * 4 + (int)rank;                     // owner of units [8 cta, 8 cta + 8)
    const unsigned ncta = gridDim.x;

    // W_hh slice -> shared (row m = 32*dest_rank + 8*gate + unit; K-major, 128B swizzle)
    for (int idx = tid; idx < 128 * CPR; idx += NGT) {
        const int m = idx / CPR, cc = idx - m * CPR;
        const int q = m >> 5, gate = (m >> 3) & 3, u = m & 7;
        const uint4 v = *reinterpret_cast<const uint4*>(p.whh + ((size_t)gate * H + 32 * grp + 8 * q + u) * H +
                                                        (size_t)rank * KS + cc * 8);
        const int a = cc >> 3, c = cc & 7;
        *reinterpret_cast<uint4*>(sA + a * 16384 + m * 128 + ((c ^ (m & 7)) << 4)) = v;
    }
    if (tid == 0) {
        mbar_init(rbar, 1);                                  // one local arrive.expect_tx per step + 3 x 4 KB of copies
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    fence_proxy_async();                                     // the A tile was written through the generic proxy
    __syncthreads();
    cluster_sync_all();                                      // peers' mbarriers exist before any copy completes on them

    const int b = tid >> 2, up = tid & 3;
    const int j = cta * UPC + 2 * up;
    const bool own = b < B;
    const size_t xstride = (size_t)NB * H;
    float c0v = 0.f, c1v = 0.f;
    {
        float h0a = 0.f, h0b = 0.f;
        if (own && p.h0) { h0a = p.h0[(size_t)b * H + j]; h0b = p.h0[(size_t)b * H + j + 1]; }
        if (own && p.c0) { c0v = p.c0[(size_t)b * H + j]; c1v = p.c0[(size_t)b * H + j + 1]; }
        const uint32_t hp = pack2(h0a, h0b);
        *reinterpret_cast<uint32_t*>(p.hx + xstride + (size_t)b * H + j) = hp;
        if (own && p.hprev16) *reinterpret_cast<uint32_t*>(p.hprev16 + (size_t)b * T * H + j) = hp;
    }
    __syncthreads();
    // Grid barrier per K SLICE: the CTA of rank r only consumes the h units of slice r, produced by the NC/4 CTAs
    // [r*NC/4, (r+1)*NC/4): it waits for those arrivals alone (counter r, 1 KB apart).  Every cluster consumes
    // all four slices, so no CTA can run a step ahead of any producer and the double-buffered exchange stays safe.
    const unsigned nprod = ncta >> 2;
    unsigned* const my_ctr = p.bar + (cta / (int)nprod) * CTR_STRIDE;
    const unsigned* const wait_ctr = p.bar + rank * CTR_STRIDE;
    if (tid == 0) { __threadfence(); atomicAdd(my_ctr, 1u); }
    const float* xgp = p.xg + (size_t)b * T * 4 * H + j;
    float2 xr[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) xr[g] = own ? __ldg(reinterpret_cast<const float2*>(xgp + (size_t)g * H)) : make_float2(0.f, 0.f);
    size_t oy = (size_t)b * T * H + j;
    // thread d < 4 (d != rank) hands the partial tile destined to CTA d to the copy engine
    const uint32_t dst = (uint32_t)(tid & 3);
    const uint32_t slot_at_dst = (rank < dst) ? rank : rank - 1;                  // my slot in CTA dst's recv
    const uint32_t push_dst = map_to_rank(smem_u32(recv) + slot_at_dst * 4096u, dst);
    const uint32_t rbar_dst = map_to_rank(rbar, dst);
    const int ro0 = swz(2 * up, b), ro1 = swz(2 * up + 1, b);     // (row & 7) is the same for every gate / source
    const float* own_tile = stage + rank * 1024;
    const uint32_t sa = smem_u32(sA), sb = smem_u32(sB);
    // pull map: chunk q = i*128 + tid of the [32 rows][CPR chunks] slice (CPR divides 128 or is 24)
    const bool regular = (NGT % CPR) == 0;
    const int cc0 = tid % CPR, rw0 = tid / CPR, rstep = NGT / CPR;
    // accumulator fragment rows of this thread: m = 64*mi + 16*warp + lane/4 + 8*h -> destination m/32, row m%32
    const int frow = 16 * (warp & 1) + (lane >> 2), fcol = 2 * (lane & 3);

    for (int t = 0; t < T; ++t) {
        const uint32_t ph = (uint32_t)(t & 1);
        // ---- grid barrier: every producer of my K slice has published h_{t-1}
        if (p.wpoll) {
            if (lane == 0) spin_wait_ge(wait_ctr, (unsigned)(t + 1) * nprod);
            __syncwarp();
        } else {
            if (tid == 0) spin_wait_ge(wait_ctr, (unsigned)(t + 1) * nprod);
            __syncthreads();
        }
        if (tid == 0) C4_STAMP(t, 0);
        // ---- A. pull this CTA's K slice of h_{t-1} (L2 -> swizzled shared tile)
        {
            const __nv_bfloat16* src = p.hx + (size_t)((t + 1) & 1) * xstride + (size_t)rank * KS;
            // cp.async straight into the swizzled tile
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (i < NLD) {
                    int row, cc;
                    if (regular) { row = rw0 + i * rstep; cc = cc0; }
                    else { const int q = i * NGT + tid; row = q / CPR; cc = q - row * CPR; }
                    cp_async16(sb + (uint32_t)((cc >> 3) * 4096 + row * 128 + (((cc & 7) ^ (row & 7)) << 4)), src + (size_t)row * H + cc * 8);
                }
            }
            asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
            fence_proxy_async_smem();
            __syncthreads();
        }
        if (tid == 0) { C4_STAMP(t, 1); mbar_expect_tx(rbar, 3 * 4096); }
        // ---- B. partial gate pre-activations of the cluster's 128 gate rows over my K slice
        float acc0[16], acc1[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
        wgmma_fence();
        for (int a = 0; a < NA; ++a) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t bd = make_desc(sb + a * 4096 + k * 32, 16, 1024);
                wgmma_m64n32k16<0, 0>(acc0, make_desc(sa + a * 16384 + k * 32, 16, 1024), bd, 1);
                wgmma_m64n32k16<0, 0>(acc1, make_desc(sa + a * 16384 + 8192 + k * 32, 16, 1024), bd, 1);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        if (tid == 0) C4_STAMP(t, 2);
        // ---- C. reduce the partial tiles across the cluster: stage the four 32-row blocks (block q = the partial sums
        // of CTA q's 32 gate rows), hand the three remote ones to the copy engine (DSMEM bulk copies complete on the
        // destination's mbarrier)
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
            const float* accv = mi ? acc1 : acc0;
            float* tile = stage + (2 * mi + (warp >> 1)) * 1024;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    *reinterpret_cast<float2*>(tile + swz(frow + 8 * h, 8 * i + fcol)) =
                        make_float2(accv[4 * i + 2 * h], accv[4 * i + 2 * h + 1]);
        }
        fence_proxy_async_smem();
        __syncthreads();                                     // every partial tile is staged
        if (tid < 4 && dst != rank) bulk_s2c(push_dst, smem_u32(stage) + dst * 4096u, 4096u, rbar_dst);
        if (tid == 0) C4_STAMP(t, 3);
        mbar_wait_cluster(rbar, ph);
        if (tid == 0) C4_STAMP(t, 4);
        float pre[4][2];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            float s0 = own_tile[g * 256 + ro0], s1 = own_tile[g * 256 + ro1];
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                s0 += recv[s * 1024 + g * 256 + ro0];
                s1 += recv[s * 1024 + g * 256 + ro1];
            }
            pre[g][0] = s0 + xr[g].x;
            pre[g][1] = s1 + xr[g].y;
        }
        const float i0 = fsig(pre[0][0]), i1 = fsig(pre[0][1]);
        const float f0 = fsig(pre[1][0]), f1 = fsig(pre[1][1]);
        const float g0 = ftanh(pre[2][0]), g1 = ftanh(pre[2][1]);
        const float o0 = fsig(pre[3][0]), o1 = fsig(pre[3][1]);
        c0v = f0 * c0v + i0 * g0;
        c1v = f1 * c1v + i1 * g1;
        float hn0 = o0 * ftanh(c0v), hn1 = o1 * ftanh(c1v);
        if (!own) { hn0 = 0.f; hn1 = 0.f; }
        const uint32_t hp = pack2(hn0, hn1);
        *reinterpret_cast<uint32_t*>(p.hx + (size_t)(t & 1) * xstride + (size_t)b * H + j) = hp;
        if (tid == 0) C4_STAMP(t, 5);
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            atomicAdd(my_ctr, 1u);
            C4_STAMP(t, 6);
        }
        // everything below overlaps the other CTAs' progress towards the barrier
        if (own) {
            *reinterpret_cast<float2*>(p.y + oy) = make_float2(hn0, hn1);
            if (p.hprev16 && t + 1 < T) *reinterpret_cast<uint32_t*>(p.hprev16 + oy + H) = hp;
            const size_t si = ((size_t)t * NC + cta) * NGT + tid;
            if (p.gsave) p.gsave[si] = make_uint4(pack2(i0, i1), pack2(f0, f1), pack2(g0, g1), pack2(o0, o1));
            if (p.csave) p.csave[si] = make_float2(c0v, c1v);
            if (p.gates_std) {
                float* gp = p.gates_std + oy * 4 - 3 * (size_t)j;          // ((b*T + t) * 4H) + j
                *reinterpret_cast<float2*>(gp) = make_float2(i0, i1);
                *reinterpret_cast<float2*>(gp + H) = make_float2(f0, f1);
                *reinterpret_cast<float2*>(gp + 2 * (size_t)H) = make_float2(g0, g1);
                *reinterpret_cast<float2*>(gp + 3 * (size_t)H) = make_float2(o0, o1);
            }
            if (p.cseq_std) *reinterpret_cast<float2*>(p.cseq_std + oy) = make_float2(c0v, c1v);
            if (t == T - 1) {
                *reinterpret_cast<float2*>(p.hT + (size_t)b * H + j) = make_float2(hn0, hn1);
                *reinterpret_cast<float2*>(p.cT + (size_t)b * H + j) = make_float2(c0v, c1v);
            }
        }
        oy += H;
        xgp += 4 * (size_t)H;
        if (t + 1 < T && own) {
#pragma unroll
            for (int g = 0; g < 4; ++g) xr[g] = __ldg(reinterpret_cast<const float2*>(xgp + (size_t)g * H));
        }
    }
    __syncthreads();
    cluster_sync_all();                                      // no CTA exits while a peer may still address its smem
}

// ---------------------------------------------------------------------------------------------------------
struct C4BwdP {
    const float* dy;              // [B,T,H] fp32
    const uint4* gsave; const float2* csave;   // forward saves (layout above)
    const float* gates; const float* cseq;     // STD: fp32 saves in the layout of eb_lstm_tc_bwd ([rows,4H], [rows,H])
    const float* c0;
    const __nv_bfloat16* whhT;    // [H,4H] bf16 = W_hh^T
    const float* dhT; const float* dcT;
    __nv_bfloat16* dg16;          // [B,T,4H] bf16 gate-preactivation gradients (output, standard layout)
    float* dh0; float* dc0;
    __nv_bfloat16* gx;            // [2][NB][4H] exchange, contraction index k' = 4*unit + gate
    unsigned* bar;
    long long* trace;             // debug stamps (eb_lstm_c4_set_trace), else null
    int trace_steps;
    int B, T, H;
    // STD: time axis in segments, as eb_lstm_tc_bwd_chunks: segment c covers steps [seg_off[c], seg_off[c+1]) and is a
    // contiguous [Btot, len_c, D] block at row Btot * seg_off[c]; dy / gates / cseq / dg16 are addressed by rows, the
    // batch tile starts at row b0
    int b0, Btot, nseg;
    int seg_off[9];
};

__device__ __forceinline__ void st_cluster_f2(uint32_t caddr, float a, float b) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1,%2};" :: "r"(caddr), "f"(a), "f"(b) : "memory");
}

// Warps 0-3 (one warpgroup): gate-gradient math of the owned (unit, batch) pairs and the wgmma of the step; warp 4: grid
// barrier poller and TMA producer of the dG_t slice.
//   CS = 4 / 8: one M = 64 wgmma block, partial dh pushed with st.shared::cluster, one grid-wide barrier counter.
//   CS = 16: the forward's K-split design.  The cluster owns 128 units = two M = 64 blocks; rank r keeps the W_hh^T slice
//     [128 units x H/4] (64 KB at H = 1024) and pulls only its K slice of dG_t (16 KB: a quarter of CS = 4's pull per CTA,
//     2 MB per step over the grid instead of 8).  The [128 x 32] fp32 partial tile is staged as 16 blocks of 1 KB, the 15
//     remote ones leave as DSMEM bulk copies that complete on the destination's mbarrier, and the owner adds the 16
//     partials of its 8 units in rank order.  Slice r of the contraction is produced by the CTAs [r*NC/16, (r+1)*NC/16):
//     one barrier counter per slice, 1 KB apart.
// STD selects the inputs: fp32 gates / cells in eb_lstm_tc_bwd's layout over a segmented time axis (the saves the layer
// wavefront keeps) instead of the CTA-private bf16 saves of eb_lstm_c4_fwd.
template <int CS, bool STD>
__global__ void __launch_bounds__(NTHR, CS == 4 ? 1 : 2) lstm_c4_bwd_kernel(const __grid_constant__ CUtensorMap gmap, C4BwdP p) {
    constexpr bool KS16 = CS == 16;
    constexpr int MR = 8 * CS;                               // valid accumulator rows (units of the cluster)
    constexpr int APITCH = MR * 128;                         // bytes between the 64-wide K atoms of the A tile
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int H = p.H, B = p.B, T = p.T, H4 = 4 * H;
    const int KSL = H4 / CS, NA = KSL >> 6;
    uint8_t* sA = smem;                                      // [NA][MR rows][128 B]  (M = 64 MMA: for CS = 4 rows 32-63 of
    uint8_t* sB = sA + (size_t)NA * APITCH;                  //  an atom alias the next atom / the B tile: discarded rows)
    // CS < 16: [CS src][8 units][RP];  CS = 16: [15 src][8 units][32 batch] (swz), the slot of the own rank is skipped
    float* recv = reinterpret_cast<float*>(sB + NA * 4096);
    float* stage = recv + (KS16 ? 15 * 256 : CS * 8 * RP);   // CS = 16: [16 dest][8 units][32 batch] (swz) outgoing partials
    uint64_t* bars = reinterpret_cast<uint64_t*>(stage + (KS16 ? 16 * 256 : 0));
    const uint32_t full0 = smem_u32(bars), rbar = smem_u32(bars + 5);
    const uint32_t bfree = smem_u32(bars + 6);               // CS = 16: the wgmma of the step has read the B tile
    const uint32_t sfree = smem_u32(bars + 7);               // CS = 16: all 15 destinations have consumed my partials
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t rank = cluster_ctarank();
    const int grp = (int)cluster_id_x();
    const int cta = grp * CS + (int)rank;
    const int NC = H / UPC;
    const unsigned ncta = gridDim.x;
    // grid barrier: CS = 16 waits for the producers of its K slice only (see the forward kernel), else for every CTA
    const unsigned nprod = KS16 ? ncta / CS : ncta;
    unsigned* const my_ctr = p.bar + (KS16 ? (cta / (int)nprod) * CTR_STRIDE : 0);
    const unsigned* const wait_ctr = p.bar + (KS16 ? rank * CTR_STRIDE : 0);
    const int NQB = KS16 ? NA : 4, NQ = NA / NQB;            // TMA barriers, atoms per barrier (CS = 16: NA <= 4)

    // W_hh^T slice -> shared: A[row = unit i of the cluster][k' = 4*u + gate] = W_hh[gate*H + u][MR*grp + i]
    {
        const int cpr = KSL >> 3;
        for (int idx = tid; idx < MR * cpr; idx += NTHR) {
            const int i = idx / cpr, cc = idx - i * cpr;
            const int u = ((int)rank * KSL + cc * 8) >> 2;   // the chunk holds the four gates of units u, u+1
            const unsigned short* src = reinterpret_cast<const unsigned short*>(p.whhT + (size_t)(MR * grp + i) * H4 + u);
            auto w2 = [&](int du, int g) {                   // gates g, g+1 of unit u+du
                return (uint32_t)src[(size_t)g * H + du] | ((uint32_t)src[(size_t)(g + 1) * H + du] << 16);
            };
            uint4 v;
            v.x = w2(0, 0);
            v.y = w2(0, 2);
            v.z = w2(1, 0);
            v.w = w2(1, 2);
            const int a = cc >> 3, c = cc & 7;
            *reinterpret_cast<uint4*>(sA + (size_t)a * APITCH + i * 128 + ((c ^ (i & 7)) << 4)) = v;
        }
    }
    if (tid == 0) {
        for (int a = 0; a < 4; ++a) mbar_init(full0 + 8 * a, 1);
        if (KS16) {
            mbar_init(rbar, 1);                              // one local arrive.expect_tx per step + 15 x 1 KB of copies
            mbar_init(bfree, 1);
            mbar_init(sfree, CS - 1);
        } else {
            mbar_init(rbar, CS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&gmap) : "memory");
    }
    fence_proxy_async();
    __syncthreads();
    cluster_sync_all();
    const size_t xstride = (size_t)NB * H4;

    if (warp < 4) {
        const int b = tid >> 2, up = tid & 3;
        const int j = cta * UPC + 2 * up;
        const bool own = b < B;
        // STD: row of (batch row b of this tile, step t) in the segmented [rows, D] tensors
        auto rowof = [&](int t) -> size_t {
            int c = 0;
            while (c + 1 < p.nseg && t >= p.seg_off[c + 1]) ++c;
            const int lo = p.seg_off[c];
            return (size_t)p.Btot * lo + (size_t)(p.b0 + b) * (p.seg_off[c + 1] - lo) + (t - lo);
        };
        const float2 c0v = (own && p.c0) ? make_float2(p.c0[(size_t)b * H + j], p.c0[(size_t)b * H + j + 1]) : make_float2(0.f, 0.f);
        float dh0v = 0.f, dh1v = 0.f, dc0v = 0.f, dc1v = 0.f;
        if (own && p.dhT) { dh0v = p.dhT[(size_t)b * H + j]; dh1v = p.dhT[(size_t)b * H + j + 1]; }
        if (own && p.dcT) { dc0v = p.dcT[(size_t)b * H + j]; dc1v = p.dcT[(size_t)b * H + j + 1]; }
        // M = 64 accumulator fragment: rows 16*warp + lane/4 + 8*h (h = 0, 1) = units of destination rank 2*warp + h
        const int frow = 16 * warp + (lane >> 2), fcol = 2 * (lane & 3);
        const bool push0 = frow < MR, push1 = frow + 8 < MR;
        const uint32_t rslot = smem_u32(recv) + (uint32_t)((rank * 8 + (frow & 7)) * RP + fcol) * 4u;
        const uint32_t dst0 = (!KS16 && push0) ? map_to_rank(rslot, (uint32_t)(frow >> 3)) : 0u;
        const uint32_t dst1 = (!KS16 && push1) ? map_to_rank(rslot, (uint32_t)((frow + 8) >> 3)) : 0u;
        const uint32_t rbar0 = (!KS16 && push0) ? map_to_rank(rbar, (uint32_t)(2 * warp)) : 0u;
        const uint32_t rbar1 = (!KS16 && push1) ? map_to_rank(rbar, (uint32_t)(2 * warp + 1)) : 0u;
        const float* rbase = recv + (2 * up) * RP + b;
        // CS = 16: thread d < 16 (d != rank) hands the partial block of CTA d to the copy engine and tells CTA d when
        // the block CTA d sent it has been consumed
        const uint32_t dst = (uint32_t)(tid & 15);
        const bool pusher = KS16 && tid < 16 && dst != rank;
        const uint32_t push_dst = pusher ? map_to_rank(smem_u32(recv) + ((rank < dst) ? rank : rank - 1) * 1024u, dst) : 0u;
        const uint32_t rbar_dst = pusher ? map_to_rank(rbar, dst) : 0u;
        const uint32_t sfree_dst = pusher ? map_to_rank(sfree, dst) : 0u;
        const int ro0 = swz(2 * up, b), ro1 = swz(2 * up + 1, b);
        const uint32_t sa = smem_u32(sA), sb = smem_u32(sB);
        // prefetched inputs of step t: gates, c_t (cur), c_{t-1} (prv), dy_t
        const size_t sstep = (size_t)NC * NGT;
        size_t si = ((size_t)(T - 1) * NC + cta) * NGT + tid;
        size_t oy = ((size_t)b * T + (T - 1)) * H + j;
        uint4 gq = make_uint4(0u, 0u, 0u, 0u);
        float2 g4[4] = {};
        float2 ccur = make_float2(0.f, 0.f), cprv = make_float2(0.f, 0.f), dyv = make_float2(0.f, 0.f);
        if (own) {
            if constexpr (STD) {
                const size_t r = rowof(T - 1);
#pragma unroll
                for (int g = 0; g < 4; ++g) g4[g] = __ldg(reinterpret_cast<const float2*>(p.gates + r * H4 + (size_t)g * H + j));
                ccur = __ldg(reinterpret_cast<const float2*>(p.cseq + r * H + j));
                cprv = (T > 1) ? __ldg(reinterpret_cast<const float2*>(p.cseq + rowof(T - 2) * H + j)) : c0v;
                dyv = __ldg(reinterpret_cast<const float2*>(p.dy + r * H + j));
            } else {
                gq = p.gsave[si];
                ccur = p.csave[si];
                cprv = (T > 1) ? p.csave[si - sstep] : c0v;
                dyv = *reinterpret_cast<const float2*>(p.dy + oy);
            }
        }

        for (int t = T - 1; t >= 0; --t) {
            const int e = T - 1 - t;
            if (tid == 0) C4_STAMP(e, 0);
            // ---- gate gradients of step t for the owned pairs
            uint4 pk = make_uint4(0u, 0u, 0u, 0u);          // dG_t of units (j, j+1), gate-major pairs: i, f, g, o
            if (own) {
                float2 ig, fg, gg, og;
                if constexpr (STD) {
                    ig = g4[0]; fg = g4[1]; gg = g4[2]; og = g4[3];
                } else {
                    ig = unpack2(gq.x); fg = unpack2(gq.y); gg = unpack2(gq.z); og = unpack2(gq.w);
                }
                const float tc0 = ftanh(ccur.x), tc1 = ftanh(ccur.y);
                const float dht0 = dyv.x + dh0v, dht1 = dyv.y + dh1v;
                const float dct0 = dc0v + dht0 * og.x * (1.f - tc0 * tc0);
                const float dct1 = dc1v + dht1 * og.y * (1.f - tc1 * tc1);
                pk.x = pack2(dct0 * gg.x * ig.x * (1.f - ig.x), dct1 * gg.y * ig.y * (1.f - ig.y));
                pk.y = pack2(dct0 * cprv.x * fg.x * (1.f - fg.x), dct1 * cprv.y * fg.y * (1.f - fg.y));
                pk.z = pack2(dct0 * ig.x * (1.f - gg.x * gg.x), dct1 * ig.y * (1.f - gg.y * gg.y));
                pk.w = pack2(dht0 * tc0 * og.x * (1.f - og.x), dht1 * tc1 * og.y * (1.f - og.y));
                dc0v = dct0 * fg.x;
                dc1v = dct1 * fg.y;
            }
            // exchange (k' = 4*unit + gate): i_j f_j | g_j o_j | i_j+1 f_j+1 | g_j+1 o_j+1
            *reinterpret_cast<uint4*>(p.gx + (size_t)(t & 1) * xstride + (size_t)b * H4 + 4 * j) =
                make_uint4(__byte_perm(pk.x, pk.y, 0x5410), __byte_perm(pk.z, pk.w, 0x5410),
                           __byte_perm(pk.x, pk.y, 0x7632), __byte_perm(pk.z, pk.w, 0x7632));
            fence_proxy_async();
            named_bar_gate();
            if (tid == 0) { __threadfence(); atomicAdd(my_ctr, 1u); C4_STAMP(e, 1); }
            // CS = 16: every gate thread has read the partials of step t+1 out of recv: their senders may overwrite it
            if (KS16 && pusher && e > 0) mbar_arrive_cluster(sfree_dst);
            // off the critical path: dG_t in the standard gate-major layout, inputs of step t-1
            if (own) {
                __nv_bfloat16* dgp = p.dg16 + (STD ? rowof(t) * H4 : ((size_t)b * T + t) * H4) + j;
                *reinterpret_cast<uint32_t*>(dgp) = pk.x;
                *reinterpret_cast<uint32_t*>(dgp + H) = pk.y;
                *reinterpret_cast<uint32_t*>(dgp + 2 * (size_t)H) = pk.z;
                *reinterpret_cast<uint32_t*>(dgp + 3 * (size_t)H) = pk.w;
                if (t > 0) {
                    ccur = cprv;
                    if constexpr (STD) {
                        const size_t r = rowof(t - 1);
#pragma unroll
                        for (int g = 0; g < 4; ++g) g4[g] = __ldg(reinterpret_cast<const float2*>(p.gates + r * H4 + (size_t)g * H + j));
                        cprv = (t > 1) ? __ldg(reinterpret_cast<const float2*>(p.cseq + rowof(t - 2) * H + j)) : c0v;
                        dyv = __ldg(reinterpret_cast<const float2*>(p.dy + r * H + j));
                    } else {
                        si -= sstep;
                        oy -= H;
                        gq = p.gsave[si];
                        cprv = (t > 1) ? p.csave[si - sstep] : c0v;
                        dyv = *reinterpret_cast<const float2*>(p.dy + oy);
                    }
                }
            }
            // ---- dh_rec of step t-1: the cluster's units against my K slice of dG_t, as each part of it lands
            const uint32_t ph = (uint32_t)(e & 1);
            if constexpr (KS16) {
                float acc0[16], acc1[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
                for (int q = 0; q < NQB; ++q) {
                    mbar_wait(full0 + 8 * q, ph);
                    if (tid == 0 && q == 0) C4_STAMP(e, 2);
                    wgmma_fence();
                    for (int a = q * NQ; a < (q + 1) * NQ; ++a) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint64_t bd = make_desc(sb + a * 4096 + k * 32, 16, 1024);
                            wgmma_m64n32k16<0, 0>(acc0, make_desc(sa + a * APITCH + k * 32, 16, 1024), bd, 1);
                            wgmma_m64n32k16<0, 0>(acc1, make_desc(sa + a * APITCH + 8192 + k * 32, 16, 1024), bd, 1);
                        }
                    }
                    wgmma_commit();
                }
                wgmma_wait<0>();
                wgmma_fence_regs(acc0);
                wgmma_fence_regs(acc1);
                if (tid == 0) C4_STAMP(e, 3);
                // the copies of the previous step have been consumed by every destination: stage is free
                if (e > 0) mbar_wait_cluster(sfree, (uint32_t)((e - 1) & 1));
                // block d = rows [8d, 8d+8) of the accumulator = the partial dh of CTA d's units
#pragma unroll
                for (int mi = 0; mi < 2; ++mi) {
                    const float* accv = mi ? acc1 : acc0;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float* tile = stage + (8 * mi + 2 * warp + h) * 256;
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            *reinterpret_cast<float2*>(tile + swz(lane >> 2, 8 * i + fcol)) =
                                make_float2(accv[4 * i + 2 * h], accv[4 * i + 2 * h + 1]);
                    }
                }
                fence_proxy_async_smem();
                named_bar_gate();                            // every block is staged, the B tile is read
                if (tid == 0) { mbar_arrive(bfree); mbar_expect_tx(rbar, 15 * 1024); }
                if (pusher) bulk_s2c(push_dst, smem_u32(stage) + dst * 1024u, 1024u, rbar_dst);
                if (tid == 0) C4_STAMP(e, 4);
                mbar_wait_cluster(rbar, ph);
                if (tid == 0) C4_STAMP(e, 5);
                // ranks [0, 8) and [8, 16) in order, then the two halves: the summation order of lstm_tc_bwd with clusters
                // of 2 (16 k16 steps per warp, 8 warps, 2 CTAs), which is what an H100 runs, so the two kernels agree
                float s[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
                for (int src = 0; src < CS; ++src) {
                    const float* tl = (src == (int)rank) ? stage + rank * 256 : recv + (src < (int)rank ? src : src - 1) * 256;
                    s[src >> 3][0] += tl[ro0];
                    s[src >> 3][1] += tl[ro1];
                }
                dh0v = s[0][0] + s[1][0];
                dh1v = s[0][1] + s[1][1];
            } else {
                float acc[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[i] = 0.f;
                for (int q = 0; q < 4; ++q) {
                    mbar_wait(full0 + 8 * q, ph);
                    wgmma_fence();
                    for (int a = q * NQ; a < (q + 1) * NQ; ++a) {
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            wgmma_m64n32k16<0, 0>(acc, make_desc(sa + a * APITCH + k * 32, 16, 1024),
                                                  make_desc(sb + a * 4096 + k * 32, 16, 1024), 1);
                    }
                    wgmma_commit();
                }
                wgmma_wait<0>();
                wgmma_fence_regs(acc);
                // partial dh tiles -> the owning CTAs' shared memory (DSMEM), one release arrival per destination
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (push0) st_cluster_f2(dst0 + i * 32, acc[4 * i], acc[4 * i + 1]);
                    if (push1) st_cluster_f2(dst1 + i * 32, acc[4 * i + 2], acc[4 * i + 3]);
                }
                __syncwarp();
                if (lane == 0) {
                    if (push0) mbar_arrive_cluster(rbar0);
                    if (push1) mbar_arrive_cluster(rbar1);
                }
                mbar_wait_cluster(rbar, ph);
                float s0 = 0.f, s1 = 0.f;
#pragma unroll
                for (int src = 0; src < CS; ++src) {
                    s0 += rbase[(src * 8) * RP];
                    s1 += rbase[(src * 8 + 1) * RP];
                }
                dh0v = s0;
                dh1v = s1;
            }
        }
        if (own) {
            *reinterpret_cast<float2*>(p.dh0 + (size_t)b * H + j) = make_float2(dh0v, dh1v);
            *reinterpret_cast<float2*>(p.dc0 + (size_t)b * H + j) = make_float2(dc0v, dc1v);
        }
    } else if (lane == 0) {
        const uint32_t sb = smem_u32(sB);
        const int k0 = (int)rank * KSL;
        for (int t = T - 1; t >= 0; --t) {
            const int e = T - 1 - t;
            spin_wait_ge(wait_ctr, (unsigned)(e + 1) * nprod);   // every producer of my K slice has published dG_t
            C4_STAMP(e, 8);
            // CS = 16 (the slice's producers need not include this CTA): the previous step's wgmma is done with the B tile
            if (KS16 && e > 0) mbar_wait(bfree, (uint32_t)((e - 1) & 1));
            fence_proxy_async();
            const int row0 = (t & 1) * NB;
            for (int q = 0; q < NQB; ++q) {
                mbar_expect_tx(full0 + 8 * q, 4096u * NQ);
                for (int a = q * NQ; a < (q + 1) * NQ; ++a)
                    tma_load_2d(sb + a * 4096, &gmap, k0 + a * 64, row0, full0 + 8 * q);
            }
        }
    }
    __syncthreads();
    cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------------
inline bool c4_shape_ok(int B, int H) { return B >= 1 && H % 256 == 0 && H <= 1024; }

inline size_t fwd_smem(int H) {
    const int NA = H / 256;
    return 1024 + (size_t)NA * 16384 + 16384 + 7 * 4096 + 128;
}
template <int CS> size_t bwd_smem(int H) {
    const int NA = 4 * H / CS / 64;
    // CS = 16: A + B tiles, 15 receive and 16 staging blocks of 1 KB: 111 KB at H = 1024, two CTAs per SM
    if (CS == 16) return 1024 + (size_t)NA * (16384 + 4096) + 31 * 1024 + 128;
    // + one B-tile-sized tail: for CS = 4 the discarded accumulator rows 32-63 of the last atom read past the A tile
    return 1024 + (size_t)NA * (8 * CS * 128 + 4096) + (CS == 4 ? 4096 : 0) + sizeof(float) * CS * 8 * RP + 128;
}

template <typename K>
int max_clusters_of(K kern, int grid, int cs, size_t smem, int nthr = NTHR) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
        (cs > 8 && cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess)) {
        (void)cudaGetLastError();
        return -2;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(nthr);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cs; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) { (void)cudaGetLastError(); return -3; }
    return n;
}

template <typename K, typename... A>
bool launch_clustered(K kern, int grid, int nthr, int cs, size_t smem, cudaStream_t st, const A&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(nthr);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeClusterDimension;
    attrs[0].val.clusterDim.x = cs; attrs[0].val.clusterDim.y = 1; attrs[0].val.clusterDim.z = 1;
    attrs[1].id = cudaLaunchAttributeCooperative;
    attrs[1].val.cooperative = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = 2;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args...);
    if (e != cudaSuccess) {
        fprintf(stderr, "[edgedict_b200] lstm_c4 cluster launch failed: %s\n", cudaGetErrorString(e));
        (void)cudaGetLastError();
        return false;
    }
    return true;
}

// cluster size of the BPTT kernel over the fp32 standard-layout saves (eb_lstm_c4_bwd_chunks): 16 when all H/128 clusters
// of 16 are co-resident (non-portable cluster size), else 0 (eb_lstm_tc_bwd_chunks runs the layer)
int kbwd_cs(int H) {
    static int cache[5] = {-1, -1, -1, -1, -1};              // index H/256
    int& c = cache[H / 256];
    if (c < 0) c = max_clusters_of(lstm_c4_bwd_kernel<16, true>, H / 8, 16, bwd_smem<16>(H)) >= H / 128 ? 16 : 0;
    return c;
}

// cluster size of the BPTT kernel over the CTA-private saves (eb_lstm_c4_bwd): 8 when H/64 clusters of 8 are co-resident,
// else 4, else 0 (unsupported).  EDGEDICT_LSTM_C4_BWD_CS=<4|8> overrides.
int bwd_cs(int H) {
    static int cache[5] = {-1, -1, -1, -1, -1};              // index H/256
    int& c = cache[H / 256];
    if (c >= 0) return c;
    int want = 0;
    const char* e = getenv("EDGEDICT_LSTM_C4_BWD_CS");
    if (e) want = atoi(e);
    c = 0;
    if ((want == 0 || want == 8) && H % 512 == 0 &&
        max_clusters_of(lstm_c4_bwd_kernel<8, false>, H / 8, 8, bwd_smem<8>(H)) >= H / 64) c = 8;
    else if ((want == 0 || want == 4) && max_clusters_of(lstm_c4_bwd_kernel<4, false>, H / 8, 4, bwd_smem<4>(H)) >= H / 32) c = 4;
    return c;
}

int fwd_max_clusters(int H) { return max_clusters_of(lstm_c4_fwd_kernel, H / 8, 4, fwd_smem(H), NGT); }

bool fwd_ok(int H) {
    static int cache[5] = {-1, -1, -1, -1, -1};
    int& c = cache[H / 256];
    if (c < 0) c = fwd_max_clusters(H) >= H / 32 ? 1 : 0;
    return c == 1;
}

}  // namespace

// 1 when the cluster/wgmma recurrent kernels can run this layer (shape + co-residency of all clusters)
EB_API int eb_lstm_c4_supported(int B, int H) {
    static int off = -1;
    if (off < 0) { const char* e = getenv("EDGEDICT_LSTM_C4"); off = (e && atoi(e) == 0) ? 1 : 0; }
    if (off || !c4_shape_ok(B, H)) return 0;
    return (fwd_ok(H) && bwd_cs(H) > 0) ? 1 : 0;
}

// debug: clock64 stamps of CTA 0 for the first `steps` steps of subsequent launches ([steps][16] int64; null = off)
EB_API int eb_lstm_c4_set_trace(void* dev_buf, int steps) {
    g_trace = reinterpret_cast<long long*>(dev_buf);
    g_trace_steps = dev_buf ? steps : 0;
    return EB_OK;
}

// diagnostic: co-resident clusters of the kernels (which: 0 forward / clusters of 4; 4, 8 or 16 backward with that cluster
// size, 16 = the kernel of eb_lstm_c4_bwd_chunks)
EB_API int eb_lstm_c4_max_clusters(int H, int which) {
    if (H % 256 || H > 1024 || H <= 0) return -1;
    if (which == 0) return fwd_max_clusters(H);
    if (which == 4) return max_clusters_of(lstm_c4_bwd_kernel<4, false>, H / 8, 4, bwd_smem<4>(H));
    if (which == 8) return max_clusters_of(lstm_c4_bwd_kernel<8, false>, H / 8, 8, bwd_smem<8>(H));
    if (which == 16) return max_clusters_of(lstm_c4_bwd_kernel<16, true>, H / 8, 16, bwd_smem<16>(H));
    return -1;
}

EB_API int eb_lstm_c4_bwd_cluster(int H) { return (H % 256 == 0 && H <= 1024 && H > 0) ? bwd_cs(H) : 0; }

EB_API int eb_lstm_c4_bwd_chunks_cluster(int H) { return (H % 256 == 0 && H <= 1024 && H > 0) ? kbwd_cs(H) : 0; }

EB_API size_t eb_lstm_c4_scratch_bytes(int B, int H) {
    if (!c4_shape_ok(B, H)) return 0;
    // forward: [2][32][H/8][4] 8-byte exchange words = 256 H bytes; backward: [2][32][4H] bf16 = 512 H bytes
    return C4_HDR + (size_t)512 * H;
}

// bytes of the forward saves for backward: gates (bf16) and cell states (fp32) of all batch tiles
EB_API size_t eb_lstm_c4_gsave_bytes(int B, int T, int H) { return (size_t)((B + NB - 1) / NB) * T * (H / UPC) * NGT * 16; }
EB_API size_t eb_lstm_c4_csave_bytes(int B, int T, int H) { return (size_t)((B + NB - 1) / NB) * T * (H / UPC) * NGT * 8; }

// xg [B,T,4H] fp32; whh16 [4H,H] bf16.  y [B,T,H] fp32; hprev16 [B,T,H] bf16 (h_{t-1}; optional); gsave / csave as sized
// above (optional).  B > 32 runs as batch tiles of 32 (independent utterances), one launch per tile.
EB_API int eb_lstm_c4_fwd(const float* xg, const void* whh16, const float* h0, const float* c0, float* y,
                          void* hprev16, float* hT, float* cT, void* gsave, void* csave, float* gates_std,
                          float* cseq_std, void* scratch, int B, int T, int H, void* stream) {
    if (!xg || !whh16 || !y || !hT || !cT || !scratch || T <= 0 || !c4_shape_ok(B, H)) return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(whh16) & 15) || (reinterpret_cast<uintptr_t>(xg) & 7) || (reinterpret_cast<uintptr_t>(y) & 7))
        return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t smem = fwd_smem(H);
    EB_CUDA(cudaFuncSetAttribute(lstm_c4_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    char* base = reinterpret_cast<char*>(scratch);
    const size_t tile_save = (size_t)T * (H / UPC) * NGT;
    for (int b0 = 0, tile = 0; b0 < B; b0 += NB, ++tile) {
        C4FwdP p;
        p.xg = xg + (size_t)b0 * T * 4 * H;
        p.whh = reinterpret_cast<const __nv_bfloat16*>(whh16);
        p.h0 = h0 ? h0 + (size_t)b0 * H : nullptr;
        p.c0 = c0 ? c0 + (size_t)b0 * H : nullptr;
        p.y = y + (size_t)b0 * T * H;
        p.hprev16 = hprev16 ? reinterpret_cast<__nv_bfloat16*>(hprev16) + (size_t)b0 * T * H : nullptr;
        p.hT = hT + (size_t)b0 * H;
        p.cT = cT + (size_t)b0 * H;
        p.gsave = gsave ? reinterpret_cast<uint4*>(gsave) + tile * tile_save : nullptr;
        p.csave = csave ? reinterpret_cast<float2*>(csave) + tile * tile_save : nullptr;
        p.hx = reinterpret_cast<__nv_bfloat16*>(base + C4_HDR);
        p.bar = reinterpret_cast<unsigned*>(base);
        p.B = (B - b0 < NB) ? (B - b0) : NB; p.T = T; p.H = H;
        p.trace = g_trace; p.trace_steps = g_trace_steps;
        p.gates_std = gates_std ? gates_std + (size_t)b0 * T * 4 * H : nullptr;
        { static int wp = -1; if (wp < 0) { const char* e = getenv("EDGEDICT_LSTM_WPOLL"); wp = e ? atoi(e) : 3; } p.wpoll = wp & 1; }
        p.cseq_std = cseq_std ? cseq_std + (size_t)b0 * T * H : nullptr;
        EB_CUDA(cudaMemsetAsync(scratch, 0, C4_HDR, st));
        if (!launch_clustered(lstm_c4_fwd_kernel, H / UPC, NGT, 4, smem, st, p)) return EB_ERR_CUDA;
    }
    return EB_OK;
}

// whhT16 [H,4H] bf16 (W_hh transposed).  dg16 [B,T,4H] bf16 out; dh0/dc0 [B,H] fp32 out.
EB_API int eb_lstm_c4_bwd(const float* dy, const void* gsave, const void* csave, const float* c0, const void* whhT16,
                          const float* dhT, const float* dcT, void* dg16, float* dh0, float* dc0, void* scratch,
                          int B, int T, int H, void* stream) {
    if (!dy || !gsave || !csave || !whhT16 || !dg16 || !dh0 || !dc0 || !scratch || T <= 0 || !c4_shape_ok(B, H))
        return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(whhT16) & 3) || (reinterpret_cast<uintptr_t>(dy) & 7) || (reinterpret_cast<uintptr_t>(dg16) & 3))
        return EB_ERR_INVALID;
    const int cs = bwd_cs(H);
    if (cs == 0) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    char* base = reinterpret_cast<char*>(scratch);
    CUtensorMap gmap;
    if (!make_map(&gmap, base + C4_HDR, (uint64_t)4 * H, (uint64_t)2 * NB, NB)) {
        fprintf(stderr, "[edgedict_b200] cuTensorMapEncodeTiled failed (lstm_c4 bwd)\n");
        return EB_ERR_CUDA;
    }
    const size_t tile_save = (size_t)T * (H / UPC) * NGT;
    for (int b0 = 0, tile = 0; b0 < B; b0 += NB, ++tile) {
        C4BwdP p;
        p.dy = dy + (size_t)b0 * T * H;
        p.gsave = reinterpret_cast<const uint4*>(gsave) + tile * tile_save;
        p.csave = reinterpret_cast<const float2*>(csave) + tile * tile_save;
        p.c0 = c0 ? c0 + (size_t)b0 * H : nullptr;
        p.whhT = reinterpret_cast<const __nv_bfloat16*>(whhT16);
        p.dhT = dhT ? dhT + (size_t)b0 * H : nullptr;
        p.dcT = dcT ? dcT + (size_t)b0 * H : nullptr;
        p.dg16 = reinterpret_cast<__nv_bfloat16*>(dg16) + (size_t)b0 * T * 4 * H;
        p.dh0 = dh0 + (size_t)b0 * H;
        p.dc0 = dc0 + (size_t)b0 * H;
        p.gx = reinterpret_cast<__nv_bfloat16*>(base + C4_HDR);
        p.bar = reinterpret_cast<unsigned*>(base);
        p.gates = p.cseq = nullptr;
        p.trace = g_trace; p.trace_steps = g_trace_steps;
        p.B = (B - b0 < NB) ? (B - b0) : NB; p.T = T; p.H = H;
        p.b0 = 0; p.Btot = p.B; p.nseg = 1;
        for (int c = 0; c < 9; ++c) p.seg_off[c] = c ? T : 0;
        EB_CUDA(cudaMemsetAsync(scratch, 0, C4_HDR, st));
        bool ok;
        if (cs == 8) {
            const size_t smem = bwd_smem<8>(H);
            EB_CUDA(cudaFuncSetAttribute(lstm_c4_bwd_kernel<8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ok = launch_clustered(lstm_c4_bwd_kernel<8, false>, H / UPC, NTHR, 8, smem, st, gmap, p);
        } else {
            const size_t smem = bwd_smem<4>(H);
            EB_CUDA(cudaFuncSetAttribute(lstm_c4_bwd_kernel<4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ok = launch_clustered(lstm_c4_bwd_kernel<4, false>, H / UPC, NTHR, 4, smem, st, gmap, p);
        }
        if (!ok) return EB_ERR_CUDA;
    }
    return EB_OK;
}

// The BPTT of eb_lstm_tc_bwd_chunks (same arguments, same fp32 standard-layout saves, e.g. eb_lstm_c4_fwd's gates_std /
// cseq_std) on the K-split wgmma kernel in clusters of 16: H % 256 == 0, H <= 1024, and eb_lstm_c4_bwd_chunks_cluster(H)
// == 16 (all clusters co-resident), else EB_ERR_INVALID.  One launch per batch tile of 32 walks all chunks.
EB_API int eb_lstm_c4_bwd_chunks(const float* dy, const float* gates, const float* cseq, const float* c0,
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
    if (!dy || !gates || !cseq || !whhT16 || !dg16 || !dh0 || !dc0 || !scratch || !c4_shape_ok(B, H)) return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(whhT16) & 3) || (reinterpret_cast<uintptr_t>(dy) & 7) ||
        (reinterpret_cast<uintptr_t>(gates) & 7) || (reinterpret_cast<uintptr_t>(cseq) & 7) ||
        (reinterpret_cast<uintptr_t>(dg16) & 3))
        return EB_ERR_INVALID;
    if (kbwd_cs(H) != 16) return EB_ERR_INVALID;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    char* base = reinterpret_cast<char*>(scratch);
    CUtensorMap gmap;
    if (!make_map(&gmap, base + C4_HDR, (uint64_t)4 * H, (uint64_t)2 * NB, NB)) {
        fprintf(stderr, "[edgedict_b200] cuTensorMapEncodeTiled failed (lstm_c4 bwd)\n");
        return EB_ERR_CUDA;
    }
    const size_t smem = bwd_smem<16>(H);
    EB_CUDA(cudaFuncSetAttribute(lstm_c4_bwd_kernel<16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    EB_CUDA(cudaFuncSetAttribute(lstm_c4_bwd_kernel<16, true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    for (int b0 = 0; b0 < B; b0 += NB) {
        C4BwdP p;
        p.dy = dy; p.gates = gates; p.cseq = cseq;           // batch tile and time segments: row addressing in the kernel
        p.gsave = nullptr; p.csave = nullptr;
        p.b0 = b0; p.Btot = B; p.nseg = nchunks;
        p.seg_off[0] = 0;
        for (int c = 0; c < 8; ++c) p.seg_off[c + 1] = c < nchunks ? p.seg_off[c] + chunk_lens[c] : (int)T;
        p.c0 = c0 ? c0 + (size_t)b0 * H : nullptr;
        p.whhT = reinterpret_cast<const __nv_bfloat16*>(whhT16);
        p.dhT = dhT ? dhT + (size_t)b0 * H : nullptr;
        p.dcT = dcT ? dcT + (size_t)b0 * H : nullptr;
        p.dg16 = reinterpret_cast<__nv_bfloat16*>(dg16);
        p.dh0 = dh0 + (size_t)b0 * H;
        p.dc0 = dc0 + (size_t)b0 * H;
        p.gx = reinterpret_cast<__nv_bfloat16*>(base + C4_HDR);
        p.bar = reinterpret_cast<unsigned*>(base);
        p.trace = g_trace; p.trace_steps = g_trace_steps;
        p.B = (B - b0 < NB) ? (B - b0) : NB; p.T = (int)T; p.H = H;
        EB_CUDA(cudaMemsetAsync(scratch, 0, C4_HDR, st));
        if (!launch_clustered(lstm_c4_bwd_kernel<16, true>, H / UPC, NTHR, 16, smem, st, gmap, p)) return EB_ERR_CUDA;
    }
    return EB_OK;
}
