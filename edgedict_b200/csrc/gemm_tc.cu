// gemm_tc.cu -- bf16 tensor-core GEMM for sm_90a: TMA -> shared (128B swizzle) -> wgmma.mma_async (fp32
// accumulators in registers) -> epilogue from the accumulator fragments.  Hand-written PTX, no CUTLASS.
//
// Used in bf16 mode for every dense contraction of the RNN-T path:
//   LSTM input projections  xg = X * W_ih^T          (rnnt/models.py:45-46 -> nn.LSTM)
//   encoder/predictor projections, joint W1 halves   (rnnt/models.py:129,148,163)
//   joint logits            logits = tanh(.) * W2^T  (rnnt/models.py:165, 2.7 TFLOP at E6D2)
//   and their dgrad / wgrad counterparts (operands read MN-major, no transposes materialised).
//
// Kernel anatomy (one CTA per SM, persistent over output tiles of 128 x 128 / 128 x 256, BK = 64):
//   warps 0-7   two consumer warpgroups: warpgroup g issues the wgmma (M64 N128|256 K16) of rows [64g, 64g+64) of the
//               tile, four per stage; one stage of MMAs stays in flight and the stage before it is handed back to the
//               producer.  At the end of the tile the warpgroup applies the epilogue (bias, + C, tanh', softmax
//               statistics) to its own accumulators and stores them.  Staged-C configuration (SC: bf16 C written
//               whole, 128-wide tile): the warpgroup converts its 64 x 128 half to bf16 into a swizzled shared tile,
//               one thread hands it to a TMA store and the warpgroup goes on to the next tile's MMAs while it drains.
//   warp 8      TMA producer: cp.async.bulk.tensor.2d into a STAGES-deep ring, mbarrier expect_tx.  It runs ahead into
//               the next tile while the consumers are in the epilogue.  SC with a tanh' operand: it also loads the
//               tile's 128 x 128 block of that operand into the staging tile once the consumers have started the tile,
//               so the load lands under the MMAs; the epilogue reads it there and overwrites it with C in place.
#include <cuda.h>
#include <stdlib.h>
#include "common.cuh"
#include "sm90.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int BM = 128, BK = 64, UMMA_K = 16;
constexpr int A_BYTES = BM * BK * 2;
constexpr int NTHREADS = 2 * 128 + 32;                       // two consumer warpgroups + the producer warp

// Debug trace (eb_gemm_tc_set_trace): clock64 stamps of CTA 0 for its first trace_tiles work items, [item][8] int64.
// Consumer thread 0: [0] tile start, [1] its first `full` wait satisfied, [2] the last wgmma_wait<0>, [3] epilogue end,
// [4] cycles spent in its `full` waits, [6] the staging tile ready (staged-C epilogue: its previous stores have read it,
// and the tanh' operand has landed); the producer: [5] cycles spent in its `empty` waits for that item.
constexpr int TRACE_SLOTS = 8;
long long* g_trace = nullptr;
int g_trace_tiles = 0;

// Tile width BN_ = 128 (6 stages) or 256 (4 stages): ~193 KB of shared memory either way.
// LOW_ = "co-resident" configuration: 3 stages of the narrow tile (97 KB of shared memory), so that a GEMM CTA fits on an
// SM next to one CTA of a persistent recurrent kernel (lstm_c4.cu) -- used by the layer-wavefront schedule of the encoder
// stack, where the input GEMM of one layer runs under the recurrence of another.
// SC_ = staged-C configuration: 5 stages + the 32 KB staging tile, the shared memory of the 6-stage one, so that the
// joint's d-hidden GEMM still leaves room on each SM for a CTA of the bias column sum that runs beside it.
template <int BN_, bool LOW_ = false, bool SC_ = false> struct Cfg {
    static_assert(!SC_ || (BN_ == 128 && !LOW_), "the staged-C epilogue is built for the full-size 128-wide tile");
    static constexpr int STAGES = LOW_ ? 3 : (BN_ == 256 ? 4 : (SC_ ? 5 : 6));
    static constexpr int B_BYTES = BN_ * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int X_BYTES = SC_ ? BM * BN_ * 2 : 0;    // staging tile: [warpgroup][64-column half][64 rows][128 B]
    static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + X_BYTES + 256;
};

// Persistent tile schedule (identical in the producer and the consumers).  Work item j of CTA b:
//   split-K (weight gradients): K-split major -- the CTAs running concurrently stream the SAME rows
//     of both operands, so the operand k-blocks are shared in L2 while hot;
//   otherwise, when there are many more row blocks than CTAs: one CTA walks all column tiles of its
//     row block back to back -- the A tile is re-read from L2 instead of being fetched from HBM again
//     after eviction by the output stream;
//   else the plain round-robin over output tiles.
struct Sched {
    long num_m; int num_n; int ksplit; long out_tiles; bool n_inner;
    unsigned wid, nw;                                        // this worker (CTA) and the number of workers
    __device__ __forceinline__ bool get(long j, long& m_blk, int& n_blk, int& ks) const {
        if (n_inner) {
            const long grp = (long)wid + (j / num_n) * nw;
            if (grp >= num_m) return false;
            m_blk = grp; n_blk = (int)(j % num_n); ks = 0;
            return true;
        }
        const long wi = (long)wid + j * nw;
        if (wi >= out_tiles * ksplit) return false;
        const long tile = wi % out_tiles;
        ks = (int)(wi / out_tiles);
        m_blk = tile / num_n; n_blk = (int)(tile % num_n);
        return true;
    }
};

// Optional fused epilogue of the joint's output GEMM (rows = lattice cells (b,t,u), columns = vocabulary):
// while the logits tile leaves the accumulators, each thread keeps an online (max, sum-exp) of its two rows over
// its columns of the whole vocabulary across the consecutive column tiles of its row block, plus the blank and label
// logits; the four threads that share a row merge them at the end -- everything rnnt_denom_kernel would otherwise
// re-read the logits for.
// LSE_ROWS is the same epilogue for the language model's output layer (eb_lm_logits_ce): row r has its own target
// targets[r], denom[r] receives the row's log-sum-exp and lpl[r] the target's logit (0 for a target outside [0, N),
// which is never used to index anything).
// LSE_BAND is LSE_RNNT over the pruned loss's band rows m = (b*maxT + t)*R + r (eb_joint_band_logits_lse): row m holds
// cell (t, u = s_begin[b*maxT + t] + r), targets = s_begin and targets64 = R; padding rows (band_row_live) write
// nothing.
constexpr int LSE_NONE = 0, LSE_RNNT = 1, LSE_ROWS = 2, LSE_BAND = 3;
struct LseArgs {
    const int* labels; const int* xlen; const int* ylen;     // [B,maxU-1], [B], [B]
    float* denom; float* lpb; float* lpl;                     // [B*maxT*maxU] each (loss workspace)
    int maxT, maxU, blank;
    // (not LSE) optional epilogue multiplier for bf16 outputs: C = (A B) * (1 - aux^2), aux bf16 [M,N] -- the tanh'
    // of the joint's hidden layer applied where d hidden is produced (eb_gemm_bf16_dtanh)
    const __nv_bfloat16* aux;
    const void* targets; int targets64;                       // LSE_ROWS: [M] int32 or int64
};

__device__ __forceinline__ void st_bf16x2(__nv_bfloat16* p, float a, float b) {
    *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(a, b);
}

// ---- staged-C epilogue (SC)
// Byte offset of the thread's column pair of fragment column group i (tile columns 8i + cq, + 1) in row rr of its
// warpgroup's staging tile.  The TMA 128B swizzle: 64-column halves of 8 KB, 128 B per row, the 16-byte chunk c of row r
// at chunk c ^ (r % 8).  The 8 rows of a warp store land in 8 different chunks: no bank conflicts.
__device__ __forceinline__ uint32_t x_off(int rr, int i, int lane) {
    return (uint32_t)((i >> 3) * 8192 + rr * 128 + (((i & 7) ^ (rr & 7)) << 4) + 4 * (lane & 3));
}
__device__ __forceinline__ void st_shared_bf16x2(uint32_t a, float x, float y) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(x, y);
    asm volatile("st.shared.b32 [%0], %1;" :: "r"(a), "r"(*reinterpret_cast<const uint32_t*>(&v)) : "memory");
}
__device__ __forceinline__ float2 ld_shared_bf16x2(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v));
}
__device__ __forceinline__ void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" :: "r"(1 + wg) : "memory"); }
// the warpgroup's staging tile is free: its previous TMA stores have read it
__device__ __forceinline__ void x_acquire(int wg, bool leader) {
    if (leader) bulk_wait_read<0>();
    wg_bar_sync(wg);
}
// the warpgroup's 64 x 128 half tile [r0, r0 + 64) x [n0, n0 + 128) leaves by TMA; rows >= M and columns >= N are clipped
__device__ __forceinline__ void x_store(const CUtensorMap* map, uint32_t xw, int wg, bool leader, long r0, int n0, long M,
                                        int N) {
    fence_proxy_async_smem();                                // the st.shared above -> the TMA engine's reads
    wg_bar_sync(wg);
    if (leader) {
        if (r0 < M) {
            tma_store_2d(map, xw, n0, (int)r0);
            if (n0 + 64 < N) tma_store_2d(map, xw + 8192, n0 + 64, (int)r0);
        }
        bulk_commit();
    }
}

// A_MN / B_MN: operand stored with its M (resp. N) index contiguous ("MN-major"), else K contiguous.
//   K-major tile in smem : [rows][64 k] bf16, 128 B per row, 128B swizzle; SBO = 1024 (8 rows)
//   MN-major tile in smem: [64 k][64 mn] bf16 boxes of 8 KB, 128 B per k-row; SBO = 1024 (8 k-rows), LBO = 8192
// LOW_ is also capped to 112 registers per thread (two CTAs' worth per SM): the register file has to hold a recurrent
// CTA beside it as well.
// SC: staged-C epilogue (bf16 C, no accumulation, ksplit = 1, N % 8 == 0; tma_c / tma_x: C and lse.aux with 64 x 64
// boxes), else tma_c / tma_x are unused.
template <bool A_MN, bool B_MN, int BN_, int LSE = LSE_NONE, bool LOW_ = false, bool SC = false>
__global__ void __launch_bounds__(NTHREADS, LOW_ ? 2 : 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
               const __grid_constant__ CUtensorMap tma_c, const __grid_constant__ CUtensorMap tma_x,
               void* __restrict__ Cout, int c_bf16, const float* __restrict__ bias, int accumulate,
               long M, int N, long K, int ksplit, LseArgs lse = LseArgs(), float* __restrict__ part = nullptr,
               long long* trace = nullptr, int trace_tiles = 0) {
    using C_ = Cfg<BN_, LOW_, SC>;
    constexpr int BN = BN_, STAGES = C_::STAGES, STAGE_BYTES = C_::STAGE_BYTES, NACC = BN / 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* tiles = smem;
    const uint32_t xtile = smem_u32(smem + STAGES * STAGE_BYTES);   // SC staging tile (1024-aligned)
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + C_::X_BYTES);
    // bars: full[S], empty[S], xfull, xempty (SC with a tanh' operand: the operand has landed in the staging tile / the
    // staging tile's stores have read it)
    const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + STAGES);
    const uint32_t xfull = smem_u32(bars + 2 * STAGES), xempty = xfull + 8;
    const bool has_x = SC && lse.aux != nullptr;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long num_m = (M + BM - 1) / BM;
    const int num_n = (N + BN - 1) / BN;
    Sched sch;
    sch.num_m = num_m; sch.num_n = num_n; sch.ksplit = ksplit; sch.out_tiles = num_m * num_n;
    sch.wid = blockIdx.x; sch.nw = gridDim.x;
    sch.n_inner = LSE || ((ksplit == 1) && (num_m >= 2L * sch.nw));   // LSE needs a row block's tiles back to back
    const int nkb_total = (int)((K + BK - 1) / BK);
    const int kb_per = (nkb_total + ksplit - 1) / ksplit;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 8); }   // 8 consumer warps
        if (SC) { mbar_init(xfull, 1); mbar_init(xempty, 2); }                                          // 2 store leaders
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_b) : "memory");
        if (SC) asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_c) : "memory");
        if (has_x) asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_x) : "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0; uint32_t phase = 0;
            long mb; int nb, ksx;
            // out-of-range rows / columns / k arrive as zeros and still count their bytes
            constexpr uint32_t TX = A_BYTES + C_::B_BYTES;
            for (long jj = 0; sch.get(jj, mb, nb, ksx); ++jj) {
                const int kb0 = ksx * kb_per, kb1 = min(nkb_total, kb0 + kb_per);
                const int m0 = (int)mb * BM, n0 = nb * BN;
                // the tanh' operand of this tile: loaded once the wait for k-block kb0 + STAGES has shown that the
                // consumers are into the tile, so that waiting for the staging tile does not stall the ring
                const int kbx = min(kb0 + STAGES, kb1 - 1);
                const bool tr = trace && blockIdx.x == 0 && jj < trace_tiles;
                long long twait = 0;
                for (int kb = kb0; kb < kb1; ++kb) {
                    const long long tw = tr ? clock64() : 0;
                    mbar_wait(empty0 + 8 * stage, phase ^ 1);
                    if (tr) twait += clock64() - tw;
                    const uint32_t sa = smem_u32(tiles + stage * STAGE_BYTES), sb = sa + A_BYTES;
                    const uint32_t fb = full0 + 8 * stage;
                    mbar_expect_tx(fb, TX);
                    if (!A_MN) tma_load_2d(sa, &tma_a, kb * BK, m0, fb);
                    else { tma_load_2d(sa, &tma_a, m0, kb * BK, fb); tma_load_2d(sa + 8192, &tma_a, m0 + 64, kb * BK, fb); }
                    if (!B_MN) tma_load_2d(sb, &tma_b, kb * BK, n0, fb);
                    else {
#pragma unroll
                        for (int bx = 0; bx < BN / 64; ++bx) tma_load_2d(sb + bx * 8192, &tma_b, n0 + bx * 64, kb * BK, fb);
                    }
                    if (has_x && kb == kbx) {
                        if (jj > 0) mbar_wait(xempty, (uint32_t)(jj - 1) & 1u);   // the previous tile's stores read it
                        mbar_expect_tx(xfull, C_::X_BYTES);
#pragma unroll
                        for (int q = 0; q < 4; ++q)                  // [warpgroup q / 2][64-column half q % 2]
                            tma_load_2d(xtile + q * 8192, &tma_x, n0 + 64 * (q & 1), m0 + 64 * (q >> 1), xfull);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
                if (tr) trace[jj * TRACE_SLOTS + 5] = twait;
            }
        }
        return;
    }

    // ---- consumers
    const int wg = warp >> 2;                                // rows [64 wg, 64 wg + 64) of the tile
    const int r_in = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // tile row of fragment row h = 0 (h = 1: + 8)
    const int cq = 2 * (lane & 3);                           // column of the thread's pair inside each 8-column group
    float* Cf = reinterpret_cast<float*>(Cout);
    __nv_bfloat16* const Ch = reinterpret_cast<__nv_bfloat16*>(Cout);
    const bool vec2 = (N % 2) == 0;
    const uint32_t xw = xtile + (uint32_t)wg * 16384u;       // SC: this warpgroup's 64 rows of the staging tile
    const bool leader = threadIdx.x == 128 * wg;             // SC: issues and waits for the warpgroup's TMA stores
    uint32_t xph = 0;
    float acc[NACC];
    int stage = 0; uint32_t phase = 0;
    long mb; int nb, ks;
    float rm[2] = {-INFINITY, -INFINITY}, rs[2] = {0.f, 0.f}, xb[2] = {0.f, 0.f}, xl[2] = {0.f, 0.f};   // LSE row statistics
    int lab[2] = {-1, -1};
    bool cell_ok[2] = {false, false};
    for (long jj = 0; sch.get(jj, mb, nb, ks); ++jj) {
        const int kb0 = ks * kb_per, kb1 = min(nkb_total, kb0 + kb_per);
        const long m0 = mb * BM;
        const int n0 = nb * BN;
        long long* const tr = (trace && blockIdx.x == 0 && threadIdx.x == 0 && jj < trace_tiles) ? trace + jj * TRACE_SLOTS
                                                                                                  : nullptr;
        long long twait = 0;
        if (tr) tr[0] = clock64();
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            const long long tw = tr ? clock64() : 0;
            mbar_wait(full0 + 8 * stage, phase);
            if (tr) {
                const long long t = clock64();
                twait += t - tw;
                if (kb == kb0) tr[1] = t;
            }
            const uint32_t sa = smem_u32(tiles + stage * STAGE_BYTES) + (uint32_t)wg * 8192u, sb = smem_u32(tiles + stage * STAGE_BYTES) + A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k) {
                const uint64_t ad = A_MN ? make_desc(sa + k * 2048, 8192, 1024) : make_desc(sa + k * 32, 16, 1024);
                const uint64_t bd = B_MN ? make_desc(sb + k * 2048, 8192, 1024) : make_desc(sb + k * 32, 16, 1024);
                if constexpr (BN == 256) wgmma_m64n256k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, ad, bd, 1);
                else wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, ad, bd, 1);
            }
            wgmma_commit();
            wgmma_wait<1>();                                 // the previous stage's MMAs have retired: hand it back
            if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
            // the previous tile's stores have read the staging tile: the producer may load this tile's tanh' operand
            if (has_x && kb == kb0 && jj > 0 && leader) { bulk_wait_read<0>(); mbar_arrive(xempty); }
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (tr) { tr[2] = clock64(); tr[4] = twait; }
        if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);

        if constexpr (LSE) {
            constexpr float LOG2E = 1.4426950408889634f;
            // The bias of the thread's 32 columns, shared by its two rows: all loads issued here, unconditionally (a
            // column past N reads bias[N - 1] and is never used), so that their latency overlaps and is paid once.
            // Loaded under a `col < N` branch at the point of use, each load's latency was exposed in turn.
            float bb[BN / 4];
            if (bias) {
#pragma unroll
                for (int i = 0; i < BN / 4; ++i) bb[i] = __ldg(bias + min(n0 + 8 * (i >> 1) + cq + (i & 1), N - 1));
            } else {
#pragma unroll
                for (int i = 0; i < BN / 4; ++i) bb[i] = 0.f;
            }
            if (nb == 0) {                                   // new row block: reset, decode (b,t,u) of my two rows
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    rm[h] = -INFINITY; rs[h] = 0.f; xb[h] = 0.f; xl[h] = 0.f; lab[h] = -1; cell_ok[h] = false;
                    const long cell = m0 + r_in + 8 * h;
                    if constexpr (LSE == LSE_ROWS) {
                        if (cell < M) {
                            const long t = lse.targets64 ? static_cast<const long long*>(lse.targets)[cell]
                                                         : (long)static_cast<const int*>(lse.targets)[cell];
                            lab[h] = (t >= 0 && t < N) ? (int)t : -1;
                            cell_ok[h] = true;
                        }
                    } else if constexpr (LSE == LSE_BAND) {
                        if (cell < M) {
                            const int R = lse.targets64;
                            const long bt = cell / R;
                            const int r = (int)(cell % R);
                            const int t = (int)(bt % lse.maxT), b = (int)(bt / lse.maxT);
                            const int Tn = min(max(lse.xlen[b], 0), lse.maxT);
                            const int Un = min(max(lse.ylen[b], 0) + 1, lse.maxU);
                            const int s = static_cast<const int*>(lse.targets)[bt], u = s + r;
                            cell_ok[h] = band_row_live(t, Tn, Un, R, s, r);
                            if (cell_ok[h] && u < Un - 1) lab[h] = lse.labels[b * (lse.maxU - 1) + u];
                        }
                    } else if (cell < M) {
                        const int u = (int)(cell % lse.maxU);
                        const long bt = cell / lse.maxU;
                        const int t = (int)(bt % lse.maxT), b = (int)(bt / lse.maxT);
                        const int Tn = min(max(lse.xlen[b], 0), lse.maxT);       // clamped as in loss.cu
                        const int Un = min(max(lse.ylen[b], 0) + 1, lse.maxU);
                        cell_ok[h] = t < Tn && u < Un;
                        if (cell_ok[h] && u < Un - 1) lab[h] = lse.labels[b * (lse.maxU - 1) + u];
                    }
                }
            }
            if constexpr (SC) x_acquire(wg, leader);
            if (tr) tr[6] = clock64();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                // add the bias here (the statistics are over logits = acc + b2), then the online softmax
                float cm = -INFINITY;
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    const int col = n0 + 8 * i + cq;
                    float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
                    v0 = col < N ? v0 + bb[2 * i] : -INFINITY;
                    v1 = col + 1 < N ? v1 + bb[2 * i + 1] : -INFINITY;
                    acc[4 * i + 2 * h] = v0; acc[4 * i + 2 * h + 1] = v1;
                    cm = fmaxf(cm, fmaxf(v0, v1));
                    if (col == lse.blank) xb[h] = v0;
                    if (col + 1 == lse.blank) xb[h] = v1;
                    if (col == lab[h]) xl[h] = v0;
                    if (col + 1 == lab[h]) xl[h] = v1;
                }
                const float nm = fmaxf(rm[h], cm);
                if (nm != -INFINITY) {                       // (a thread may own no column of a narrow vocabulary)
                    const float nml = nm * LOG2E;
                    float a0 = 0.f, a1 = 0.f;                // exp(v - nm) = ex2(v*log2e - nm*log2e): FFMA + MUFU + FADD
#pragma unroll
                    for (int i = 0; i < BN / 8; ++i) {
                        a0 += fast_ex2(fmaf(acc[4 * i + 2 * h], LOG2E, -nml));
                        a1 += fast_ex2(fmaf(acc[4 * i + 2 * h + 1], LOG2E, -nml));
                    }
                    rs[h] = rs[h] * fast_ex2((rm[h] - nm) * LOG2E) + (a0 + a1);
                    rm[h] = nm;
                }
                const long row = m0 + r_in + 8 * h;
                if constexpr (SC) {
                    const int rr = r_in - 64 * wg + 8 * h;
#pragma unroll
                    for (int i = 0; i < BN / 8; ++i) st_shared_bf16x2(xw + x_off(rr, i, lane), acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
                } else if (row < M) {
#pragma unroll
                    for (int i = 0; i < BN / 8; ++i) {
                        const int col = n0 + 8 * i + cq;
                        __nv_bfloat16* cp = Ch + row * N + col;
                        if (vec2 && col + 1 < N) st_bf16x2(cp, acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
                        else {
                            if (col < N) cp[0] = __float2bfloat16(acc[4 * i + 2 * h]);
                            if (col + 1 < N) cp[1] = __float2bfloat16(acc[4 * i + 2 * h + 1]);
                        }
                    }
                }
            }
            if constexpr (SC) x_store(&tma_c, xw, wg, leader, m0 + 64 * wg, n0, M, N);
            if (nb == num_n - 1) {                           // whole vocabulary seen: merge the quad, publish
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int o = 1; o <= 2; o <<= 1) {
                        const float m2 = __shfl_xor_sync(0xffffffffu, rm[h], o), s2 = __shfl_xor_sync(0xffffffffu, rs[h], o);
                        xb[h] += __shfl_xor_sync(0xffffffffu, xb[h], o);
                        xl[h] += __shfl_xor_sync(0xffffffffu, xl[h], o);
                        const float m = fmaxf(rm[h], m2);
                        rs[h] = (rm[h] == -INFINITY ? 0.f : rs[h] * fast_ex2((rm[h] - m) * LOG2E)) +
                                (m2 == -INFINITY ? 0.f : s2 * fast_ex2((m2 - m) * LOG2E));
                        rm[h] = m;
                    }
                    if constexpr (LSE == LSE_ROWS) {
                        if ((lane & 3) == 0 && cell_ok[h]) {
                            const long row = m0 + r_in + 8 * h;
                            lse.denom[row] = rm[h] + logf(rs[h]);
                            lse.lpl[row] = xl[h];
                        }
                    } else if ((lane & 3) == 0 && cell_ok[h]) {
                        long cell = m0 + r_in + 8 * h;
                        if constexpr (LSE == LSE_BAND) {
                            const long bt = cell / lse.targets64;
                            cell = bt * lse.maxU + static_cast<const int*>(lse.targets)[bt] + (int)(cell % lse.targets64);
                        }
                        const float d = -(rm[h] + logf(rs[h]));
                        lse.denom[cell] = d;
                        lse.lpb[cell] = d + xb[h];
                        lse.lpl[cell] = d + xl[h];
                    }
                }
            }
        } else if constexpr (SC) {
            // the register path's arithmetic in its order (bias, then tanh'), every row and column of the tile: the TMA
            // store clips what lies outside C
            if (has_x) { mbar_wait(xfull, xph); xph ^= 1; }   // (implies the previous stores have read the tile)
            else x_acquire(wg, leader);
            if (tr) tr[6] = clock64();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int rr = r_in - 64 * wg + 8 * h;
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    const int col = n0 + 8 * i + cq;
                    float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
                    if (bias && col < N) { v0 += __ldg(bias + col); v1 += __ldg(bias + col + 1); }
                    const uint32_t a = xw + x_off(rr, i, lane);
                    if (has_x) {
                        const float2 hh = ld_shared_bf16x2(a);
                        v0 *= 1.f - hh.x * hh.x; v1 *= 1.f - hh.y * hh.y;
                    }
                    st_shared_bf16x2(a, v0, v1);
                }
            }
            x_store(&tma_c, xw, wg, leader, m0 + 64 * wg, n0, M, N);
        } else {
            const bool add_bias = bias && ks == 0;
            // split-K: each split stores its partial tile in its own slice of the workspace (splitk_reduce_kernel adds
            // the slices in split order -- no atomics, the same bits on every run)
            if (ksplit > 1) Cf = part + (long)ks * M * N;
            const int acc_c = ksplit > 1 ? 0 : accumulate;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const long row = m0 + r_in + 8 * h;
                if (row >= M) continue;
                // tanh' epilogue (eb_gemm_bf16_dtanh, always on the 128-wide tile): the row's aux operands are all loaded
                // before its first store.  The compiler cannot move a load of aux above a store to C (they may alias), so
                // loads placed between the stores waited one HBM round trip per 8 columns.  The other tiles have no
                // registers to spare for this and keep the loads in place.
                constexpr bool PRE = BN == 128 && !LOW_;
                __nv_bfloat162 hx[PRE ? BN / 8 : 1];
                if constexpr (PRE) {
                    if (c_bf16 && lse.aux) {
#pragma unroll
                        for (int i = 0; i < BN / 8; ++i) {
                            const int col = n0 + 8 * i + cq;
                            const long off = row * N + col;
                            hx[i] = __floats2bfloat162_rn(0.f, 0.f);
                            if (col + 1 < N && vec2) hx[i] = __ldg(reinterpret_cast<const __nv_bfloat162*>(lse.aux + off));
                            else if (col < N) {
                                hx[i].x = lse.aux[off];
                                if (col + 1 < N) hx[i].y = lse.aux[off + 1];
                            }
                        }
                    }
                }
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    const int col = n0 + 8 * i + cq;
                    if (col >= N) break;
                    const bool two = col + 1 < N, pair = two && vec2;
                    float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
                    if (add_bias) { v0 += __ldg(bias + col); if (two) v1 += __ldg(bias + col + 1); }
                    const long off = row * N + col;
                    if (c_bf16) {
                        __nv_bfloat16* cp = Ch + off;
                        if (lse.aux) {
                            float h0, h1 = 0.f;
                            if constexpr (PRE) {
                                const float2 hh = __bfloat1622float2(hx[i]);
                                h0 = hh.x;
                                if (two) h1 = hh.y;
                            } else if (pair) {
                                const float2 hh = __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(lse.aux + off)));
                                h0 = hh.x; h1 = hh.y;
                            } else {
                                h0 = __bfloat162float(lse.aux[off]);
                                if (two) h1 = __bfloat162float(lse.aux[off + 1]);
                            }
                            v0 *= 1.f - h0 * h0; v1 *= 1.f - h1 * h1;
                        }
                        if (pair) {
                            if (accumulate) {
                                const float2 o = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(cp));
                                v0 += o.x; v1 += o.y;
                            }
                            st_bf16x2(cp, v0, v1);
                        } else {
                            if (accumulate) { v0 += __bfloat162float(cp[0]); if (two) v1 += __bfloat162float(cp[1]); }
                            cp[0] = __float2bfloat16(v0);
                            if (two) cp[1] = __float2bfloat16(v1);
                        }
                    } else {
                        float* cp = Cf + off;
                        if (pair) {
                            if (acc_c) { const float2 o = *reinterpret_cast<const float2*>(cp); v0 += o.x; v1 += o.y; }
                            *reinterpret_cast<float2*>(cp) = make_float2(v0, v1);
                        } else {
                            if (acc_c) { v0 += cp[0]; if (two) v1 += cp[1]; }
                            cp[0] = v0;
                            if (two) cp[1] = v1;
                        }
                    }
                }
            }
        }
        if (tr) tr[3] = clock64();
    }
    if constexpr (SC) {
        if (leader) bulk_wait<0>();                          // the staging tile stays valid until the last store is done
    }
}

// C[i] = (accumulate ? C[i] : 0) + part[0][i] + part[1][i] + ...: the split-K partial tiles added in split order
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int ksplit, long mn, float* __restrict__ C, int accumulate) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < mn; i += (long)gridDim.x * blockDim.x) {
        float v = accumulate ? C[i] : 0.f;
        for (int s = 0; s < ksplit; ++s) v += part[(long)s * mn + i];
        C[i] = v;
    }
}

// split-K (weight gradients: few output tiles, contraction over up to millions of rows).  The persistent grid
// processes tiles*ksplit work items in waves of one per CTA; a ragged last wave idles most of the machine, so ksplit is
// chosen to fill whole waves: maximise  wave efficiency / (1 + r * ksplit / nkb):  items / (waves * workers) against the
// cost of one more partial tile per split, r k-blocks of MMA time.  Partial tiles go to a caller-provided workspace.
int choose_ksplit(long out_tiles, long nkb, long workers, double r) {
    int ksplit = 1;
    long cap = nkb / 16;
    if (cap > 64) cap = 64;
    double best = -1.0;
    for (long ks = 1; ks <= cap; ++ks) {
        const long items = out_tiles * ks;
        const long waves = (items + workers - 1) / workers;
        const double score = (double)items / (double)(waves * workers) / (1.0 + r * (double)ks / (double)nkb);
        if (score > best) { best = score; ksplit = (int)ks; }
    }
    return ksplit;
}

// Whether a product takes the staged-C epilogue (SC): bf16 C written whole by one K split, its rows (and those of the
// tanh' operand) 16-byte aligned as a tensor map needs.  The caller adds: 128-wide tile, not co-resident.
bool staged_c(const void* C, int c_bf16, int accumulate, int N, int ksplit, const void* aux) {
    return c_bf16 && !accumulate && ksplit == 1 && N % 8 == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0 &&
           (reinterpret_cast<uintptr_t>(aux) & 15) == 0;
}

// C (and the tanh' operand) as TMA-store / load maps: [M][N] bf16, 64 x 64 boxes (one per 64 x 64 quarter of a
// warpgroup's half tile), 128B swizzle
bool make_c_maps(CUtensorMap* tc, CUtensorMap* tx, const void* C, const void* aux, long M, int N) {
    return make_map(tc, C, (uint64_t)N, (uint64_t)M, 64) && (!aux || make_map(tx, aux, (uint64_t)N, (uint64_t)M, 64));
}

const CUtensorMap kNoMap = {};

// one persistent launch over `work` items, at most one CTA per SM; tc / tx: the SC maps (SC instantiations only)
template <bool A_MN, bool B_MN, int BN_, int LSE, bool LOW_, bool SC = false>
int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const CUtensorMap* tx, void* C,
                  int c_bf16, const float* bias, int accumulate, long M, int N, long K, int ksplit, long work,
                  const LseArgs& ea, cudaStream_t st, float* part = nullptr) {
    using C_ = Cfg<BN_, LOW_, SC>;
    auto kern = gemm_tc_kernel<A_MN, B_MN, BN_, LSE, LOW_, SC>;
    static bool attr_done = false;
    if (!attr_done) {
        EB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C_::SMEM_BYTES));
        attr_done = true;
    }
    const int grid = (int)(work < eb_num_sms() ? work : eb_num_sms());
    kern<<<grid, NTHREADS, C_::SMEM_BYTES, st>>>(ta, tb, tc ? *tc : kNoMap, tx ? *tx : kNoMap, C, c_bf16, bias,
                                                 accumulate, M, N, K, ksplit, ea, part, g_trace, g_trace_tiles);
    EB_CHECK_LAUNCH();
    if (ksplit > 1) {
        const long mn = M * (long)N;
        const long blocks = (mn + 255) / 256, cap = 4L * eb_num_sms();
        splitk_reduce_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(part, ksplit, mn, (float*)C, accumulate);
        EB_CHECK_LAUNCH();
    }
    return EB_OK;
}

// tc non-null: the SC epilogue (128-wide tile only)
template <bool A_MN, bool B_MN, int BN_>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const CUtensorMap* tx, void* C,
           int c_bf16, const float* bias, int accumulate, long M, int N, long K, int ksplit, float* part,
           cudaStream_t st, const void* aux = nullptr) {
    LseArgs ea = LseArgs();
    ea.aux = reinterpret_cast<const __nv_bfloat16*>(aux);
    const long out_tiles = ((M + BM - 1) / BM) * ((N + BN_ - 1) / BN_);
    if constexpr (BN_ == 128) {
        if (tc)
            return launch_kernel<A_MN, B_MN, BN_, LSE_NONE, false, true>(ta, tb, tc, tx, C, c_bf16, bias, accumulate, M, N,
                                                                      K, ksplit, out_tiles * ksplit, ea, st, part);
    }
    return launch_kernel<A_MN, B_MN, BN_, LSE_NONE, false>(ta, tb, nullptr, nullptr, C, c_bf16, bias, accumulate, M, N, K,
                                                        ksplit, out_tiles * ksplit, ea, st, part);
}

// Tile width and split-K factor of a product (the one decision shared by eb_gemm_bf16_partials and the launch).
void plan(int a_mn_major, int c_bf16, int accumulate, long M, int N, long K, int flags, bool& wide, int& ksplit) {
    const bool low = (flags & EB_GEMM_CORESIDENT) != 0;
    static int force_bn = -1;
    if (force_bn < 0) { const char* e = getenv("EDGEDICT_GEMM_BN"); force_bn = e ? atoi(e) : 0; }
    // 256-wide tiles when they tile N exactly and there is enough work to fill the machine with them
    const long wide_tiles = ((M + BM - 1) / BM) * (N / 256);
    // (split-K weight gradients take their parallelism from K: the wide tile only has to exist a few times -- it
    //  moves 48 KB of operands per 128x256x64 block where two narrow tiles move 64 KB)
    wide = (N % 256 == 0) && (wide_tiles >= eb_num_sms() || (!c_bf16 && (K + BK - 1) / BK >= 64 && wide_tiles >= 8));
    // N = 256 k + 128 with many row blocks: wide tiles with a half-empty last column tile move 20 % fewer operand bytes
    // than 128-wide tiles for 20 % more (idle anyway) MMA issue
    if (!wide && N % 256 == 128 && N >= 512 && (M + BM - 1) / BM >= 4L * eb_num_sms() && accumulate == 0) wide = true;
    if (force_bn == 128) wide = false;
    if (force_bn == 256 && N % 128 == 0) wide = true;
    if (low) wide = false;
    // fixed K order: the plan depends on N alone, so that a product computed in row blocks gives the bits of the whole
    const bool fixed = (flags & EB_GEMM_FIXED_K) != 0;
    if (fixed) wide = N % 256 == 0;
    (void)a_mn_major;
    const int BN = wide ? 256 : 128;
    const long out_tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
    const long nkb = (K + BK - 1) / BK;
    ksplit = 1;
    if (!low && !fixed && !c_bf16 && nkb >= 64 && out_tiles < eb_num_sms())
        ksplit = choose_ksplit(out_tiles, nkb, eb_num_sms(), BN == 256 ? 32.0 : 16.0);
}

// co-resident configuration (see Cfg): plain nt GEMM, narrow tile, no split-K
int launch_low(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int c_bf16, const float* bias, int accumulate,
               long M, int N, long K, cudaStream_t st) {
    const long tiles = ((M + BM - 1) / BM) * ((N + 127) / 128);
    return launch_kernel<false, false, 128, LSE_NONE, true>(ta, tb, nullptr, nullptr, C, c_bf16, bias, accumulate, M, N, K,
                                                         1, tiles, LseArgs(), st);
}

template <int LSE>
int launch_lse(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, void* C, const float* bias, long M,
               int N, long K, const LseArgs& lse, cudaStream_t st) {
    if (tc)
        return launch_kernel<false, false, 128, LSE, false, true>(ta, tb, tc, nullptr, C, 1, bias, 0, M, N, K, 1,
                                                                  (M + BM - 1) / BM, lse, st);
    return launch_kernel<false, false, 128, LSE, false>(ta, tb, nullptr, nullptr, C, 1, bias, 0, M, N, K, 1,
                                                        (M + BM - 1) / BM, lse, st);
}

}  // namespace

// Joint output layer fused with the softmax statistics of the RNN-T loss (bf16 mode):
//   logits16[cell, v] = bf16(hidden16[cell, :] . W2_16[v, :] + b2[v]),  cell = (b*maxT + t)*maxU + u
//   denom[cell] = -logsumexp_v(logits fp32),  lpb/lpl[cell] = log p(blank), log p(label[u])   (valid cells only)
// replaces Joint's second Linear (rnnt/models.py:165) + reduce_max/reduce_exp (reduce.h:45-104) + the
// gathers of compute_alphas/betas (gpu_rnnt_kernel.h:5-9) without re-reading the logits.
EB_API int eb_joint_logits_lse(const void* hidden16, const void* w2_16, const float* b2, void* logits16,
                               const int* labels, const int* xlen, const int* ylen, float* denom, float* lpb,
                               float* lpl, int B, int maxT, int maxU, int V, int J, int blank, void* stream) {
    if (!hidden16 || !w2_16 || !logits16 || !xlen || !ylen || !denom || !lpb || !lpl || (!labels && maxU > 1) ||
        B <= 0 || maxT <= 0 || maxU <= 0 || V <= 0 || J <= 0 || J % 8 || blank < 0 || blank >= V)
        return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(hidden16) & 15) || (reinterpret_cast<uintptr_t>(w2_16) & 15) ||
        (b2 && (reinterpret_cast<uintptr_t>(b2) & 15)))
        return EB_ERR_INVALID;
    const long M = (long)B * maxT * maxU;
    // 128-wide tiles: the softmax statistics of a 256-wide tile do not fit the registers beside its accumulators
    CUtensorMap ta, tb, tc;
    const bool sc = staged_c(logits16, 1, 0, V, 1, nullptr);
    if (!make_map(&ta, hidden16, (uint64_t)J, (uint64_t)M, 128) || !make_map(&tb, w2_16, (uint64_t)J, (uint64_t)V, 128) ||
        (sc && !make_c_maps(&tc, nullptr, logits16, nullptr, M, V))) {
        fprintf(stderr, "[edgedict_b200] cuTensorMapEncodeTiled failed\n");
        return EB_ERR_CUDA;
    }
    LseArgs lse;
    lse.labels = labels; lse.xlen = xlen; lse.ylen = ylen; lse.denom = denom; lse.lpb = lpb; lse.lpl = lpl;
    lse.maxT = maxT; lse.maxU = maxU; lse.blank = blank; lse.aux = nullptr;
    lse.targets = nullptr; lse.targets64 = 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return launch_lse<LSE_RNNT>(ta, tb, sc ? &tc : nullptr, logits16, b2, M, V, J, lse, st);
}

// The same epilogue over the pruned loss's band rows (LSE_BAND): logits16 [B*maxT*R, V], and the statistics of band
// row m = (b*maxT + t)*R + r at cell (t, s_begin[b*maxT + t] + r) of the [B, maxT, maxU] workspace arrays (valid band
// rows only; include/edgedict_b200.h).
EB_API int eb_joint_band_logits_lse(const void* hidden16, const void* w2_16, const float* b2, void* logits16,
                                    const int* labels, const int* xlen, const int* ylen, const int* s_begin,
                                    float* denom, float* lpb, float* lpl, int B, int maxT, int maxU, int R, int V, int J,
                                    int blank, void* stream) {
    if (!hidden16 || !w2_16 || !logits16 || !xlen || !ylen || !s_begin || !denom || !lpb || !lpl ||
        (!labels && maxU > 1) || B <= 0 || maxT <= 0 || maxU <= 0 || maxU > 1024 || R < 2 || R > 64 || V <= 0 ||
        J <= 0 || J % 8 || blank < 0 || blank >= V)
        return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(hidden16) & 15) || (reinterpret_cast<uintptr_t>(w2_16) & 15) ||
        (b2 && (reinterpret_cast<uintptr_t>(b2) & 15)) || (reinterpret_cast<uintptr_t>(logits16) & 3))
        return EB_ERR_INVALID;
    const long M = (long)B * maxT * R;
    CUtensorMap ta, tb, tc;
    const bool sc = staged_c(logits16, 1, 0, V, 1, nullptr);
    if (!make_map(&ta, hidden16, (uint64_t)J, (uint64_t)M, 128) || !make_map(&tb, w2_16, (uint64_t)J, (uint64_t)V, 128) ||
        (sc && !make_c_maps(&tc, nullptr, logits16, nullptr, M, V))) {
        fprintf(stderr, "[edgedict_b200] cuTensorMapEncodeTiled failed\n");
        return EB_ERR_CUDA;
    }
    LseArgs lse;
    lse.labels = labels; lse.xlen = xlen; lse.ylen = ylen; lse.denom = denom; lse.lpb = lpb; lse.lpl = lpl;
    lse.maxT = maxT; lse.maxU = maxU; lse.blank = blank; lse.aux = nullptr;
    lse.targets = s_begin; lse.targets64 = R;
    return launch_lse<LSE_BAND>(ta, tb, sc ? &tc : nullptr, logits16, b2, M, V, J, lse,
                                reinterpret_cast<cudaStream_t>(stream));
}

// The language model's output layer with the statistics of its cross-entropy (LMModel.loss, bf16 mode): the joint's
// epilogue above with one target per row (LSE_ROWS).
//   logits16[r, v] = bf16(hidden16[r, :] . w16[v, :] + b[v]),  lse[r] = logsumexp_v(logits fp32),
//   tlogit[r] = the fp32 logit of targets[r] when it lies in [0, V), else 0
EB_API int eb_lm_logits_ce(const void* hidden16, const void* w16, const float* b, void* logits16, const void* targets,
                           int targets_int64, float* lse, float* tlogit, long M, int V, int K, void* stream) {
    if (!hidden16 || !w16 || !logits16 || !targets || !lse || !tlogit || M <= 0 || V <= 0 || K <= 0 || K % 8 ||
        M > INT32_MAX)
        return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(hidden16) & 15) || (reinterpret_cast<uintptr_t>(w16) & 15) ||
        (b && (reinterpret_cast<uintptr_t>(b) & 15)) || (reinterpret_cast<uintptr_t>(logits16) & 3))
        return EB_ERR_INVALID;
    CUtensorMap ta, tb, tc;
    const bool sc = staged_c(logits16, 1, 0, V, 1, nullptr);
    if (!make_map(&ta, hidden16, (uint64_t)K, (uint64_t)M, 128) || !make_map(&tb, w16, (uint64_t)K, (uint64_t)V, 128) ||
        (sc && !make_c_maps(&tc, nullptr, logits16, nullptr, M, V))) {
        fprintf(stderr, "[edgedict_b200] cuTensorMapEncodeTiled failed\n");
        return EB_ERR_CUDA;
    }
    LseArgs a = LseArgs();
    a.denom = lse; a.lpl = tlogit; a.blank = -1; a.targets = targets; a.targets64 = targets_int64 ? 1 : 0;
    return launch_lse<LSE_ROWS>(ta, tb, sc ? &tc : nullptr, logits16, b, M, V, K, a, reinterpret_cast<cudaStream_t>(stream));
}

// debug: per-tile clock64 stamps of CTA 0 of subsequent wgmma GEMM launches ([tiles][8] int64, see TRACE_SLOTS; null = off)
EB_API int eb_gemm_tc_set_trace(void* dev_buf, int tiles) {
    g_trace = reinterpret_cast<long long*>(dev_buf);
    g_trace_tiles = dev_buf ? tiles : 0;
    return EB_OK;
}

EB_API int eb_gemm_bf16(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C, int c_bf16,
                        const float* bias, int accumulate, long M, int N, long K, void* stream) {
    return eb_gemm_bf16_ex(A, a_mn_major, B, b_mn_major, C, c_bf16, bias, accumulate, M, N, K, 0, nullptr, 0, stream);
}

static int gemm_dispatch(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C, int c_bf16,
                         const float* bias, int accumulate, long M, int N, long K, int flags, const void* aux,
                         float* partials, long partial_floats, void* stream);

// floats of split-K workspace eb_gemm_bf16_ex can use for this product (0: it runs without split-K)
EB_API long eb_gemm_bf16_partials(int a_mn_major, int c_bf16, int accumulate, long M, int N, long K, int flags) {
    if (M <= 0 || N <= 0 || K <= 0) return 0;
    bool wide;
    int ksplit;
    plan(a_mn_major, c_bf16, accumulate, M, N, K, flags, wide, ksplit);
    return ksplit > 1 ? (long)ksplit * M * N : 0;
}

EB_API int eb_gemm_bf16_ex(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C, int c_bf16,
                           const float* bias, int accumulate, long M, int N, long K, int flags, float* partials,
                           long partial_floats, void* stream) {
    return gemm_dispatch(A, a_mn_major, B, b_mn_major, C, c_bf16, bias, accumulate, M, N, K, flags, nullptr, partials,
                         partial_floats, stream);
}

// C16[M,N] = bf16( (A B) * (1 - hid16^2) ): the joint's d hidden GEMM with tanh' applied in the epilogue (Joint.forward's
// Tanh, rnnt/models.py:164): d(pre-activation) leaves the GEMM directly, one pass over the 2.6 GB tensor less.
EB_API int eb_gemm_bf16_dtanh(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C16,
                              const void* hid16, long M, int N, long K, void* stream) {
    if (!hid16 || (reinterpret_cast<uintptr_t>(hid16) & 7) || (reinterpret_cast<uintptr_t>(C16) & 7) || N % 4) return EB_ERR_INVALID;
    return gemm_dispatch(A, a_mn_major, B, b_mn_major, C16, 1, nullptr, 0, M, N, K, 0, hid16, nullptr, 0, stream);
}

static int gemm_dispatch(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C, int c_bf16,
                         const float* bias, int accumulate, long M, int N, long K, int flags, const void* aux,
                         float* partials, long partial_floats, void* stream) {
    if (!A || !B || !C || M <= 0 || N <= 0 || K <= 0) return EB_ERR_INVALID;
    const bool low = (flags & EB_GEMM_CORESIDENT) != 0;
    if (low && (a_mn_major || b_mn_major)) return EB_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return EB_ERR_INVALID;
    // the epilogue stores column pairs as one float2 / __nv_bfloat162 whenever N is even
    if (reinterpret_cast<uintptr_t>(C) & (c_bf16 ? 3 : 7)) return EB_ERR_INVALID;
    // contiguous dimension must keep row pitches 16-byte aligned
    if ((a_mn_major ? M : K) % 8 || (b_mn_major ? (long)N : K) % 8) return EB_ERR_INVALID;
    bool wide;
    int ksplit;
    plan(a_mn_major, c_bf16, accumulate, M, N, K, flags, wide, ksplit);
    // the tanh' epilogue (eb_gemm_bf16_dtanh: the joint's d-hidden GEMM, N = 640) runs on 128-wide tiles, which have the
    // registers to load a row's aux operands ahead of its stores (the 128 x 256 tile's epilogue waits for each load in
    // turn); bf16 output never splits K, so this only changes the tile width
    if (aux) wide = false;
    // split-K needs its workspace: with less (or none) the split count shrinks to what fits, down to no split
    if (ksplit > 1) {
        const long fit = (partials && (reinterpret_cast<uintptr_t>(partials) & 7) == 0) ? partial_floats / (M * (long)N) : 0;
        if (fit < ksplit) ksplit = fit > 1 ? (int)fit : 1;
    }
    CUtensorMap ta, tb, tc, tx;
    const bool sc = !low && !wide && staged_c(C, c_bf16, accumulate, N, ksplit, aux);
    bool ok = a_mn_major ? make_map(&ta, A, (uint64_t)M, (uint64_t)K, 64) : make_map(&ta, A, (uint64_t)K, (uint64_t)M, 128);
    ok = ok && (b_mn_major ? make_map(&tb, B, (uint64_t)N, (uint64_t)K, 64)
                           : make_map(&tb, B, (uint64_t)K, (uint64_t)N, wide ? 256 : 128));
    ok = ok && (!sc || make_c_maps(&tc, &tx, C, aux, M, N));
    if (!ok) {
        fprintf(stderr, "[edgedict_b200] cuTensorMapEncodeTiled failed\n");
        return EB_ERR_CUDA;
    }
    const CUtensorMap* pc = sc ? &tc : nullptr;
    const CUtensorMap* px = sc && aux ? &tx : nullptr;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (low) return launch_low(ta, tb, C, c_bf16, bias, accumulate, M, N, K, st);
#define EB_GO(AM, BMN)                                                                                            \
    return wide ? launch<AM, BMN, 256>(ta, tb, nullptr, nullptr, C, c_bf16, bias, accumulate, M, N, K, ksplit,    \
                                       partials, st, aux)                                                         \
                : launch<AM, BMN, 128>(ta, tb, pc, px, C, c_bf16, bias, accumulate, M, N, K, ksplit, partials, st, aux)
    if (a_mn_major) {
        if (b_mn_major) { EB_GO(true, true); }
        EB_GO(true, false);
    }
    if (b_mn_major) { EB_GO(false, true); }
    EB_GO(false, false);
#undef EB_GO
}
