// mwer.cu -- minimum word error rate training (Prabhavalkar et al., ICASSP 2018) for sm_90a: the edit distance between
// hypothesis and reference rows, the packing of a beam engine's N-best lists into label rows, and the expected risk over
// an N-best list.
//
//   1. edit_distance_kernel  one CTA per (hypothesis, reference) pair: optionally the word segmentation of both rows
//                            (word ids by exact comparison of the words' characters, a 64-bit hash as pre-filter), then
//                            the Levenshtein recurrence as an anti-diagonal wavefront over three diagonals in shared
//                            memory; each cell packs {distance, S, D, I} in 64 bits, so the counts ride along the chosen
//                            predecessor and no backtrace is stored
//   2. nbest_pack_kernel     one CTA per output row: right-aligned N-best ids -> left-aligned label rows, lengths and the
//                            validity mask, the reference row after the N hypotheses of each utterance
//   3. mwer_risk_kernel      one CTA per utterance: renormalised posteriors and the risk in fp64, in rank order
//      mwer_loss_kernel      the mean of the per-utterance risks, in utterance order
//      mwer_risk_bwd_kernel  one CTA per utterance: d loss / d costs from the same fp64 values as the forward
#include "common.cuh"
#include "../../include/edgedict_b200.h"

namespace {

constexpr int ED_THREADS = 256;
typedef unsigned long long u64;
// a DP cell: distance in bits 48..63, substitutions 0..15, deletions 16..31, insertions 32..47 (each <= 8192)
constexpr u64 ED_DIST = 1ull << 48, ED_SUB = ED_DIST | 1ull, ED_DEL = ED_DIST | (1ull << 16),
              ED_INS = ED_DIST | (1ull << 32);

struct WordTab {
    const int* tab;      // [n][3]: char offset, char count, class
    const int* chars;
    int n;
};

// {char offset, chars the token adds to a word, closes a word}: separators and dropped ids add no characters, and an
// id outside the table counts as dropped
__device__ __forceinline__ int3 unit_info(const WordTab& w, int id) {
    if (id < 0 || id >= w.n) return make_int3(0, 0, 0);
    const int* e = w.tab + 3 * (long)id;
    const int cls = __ldg(e + 2);
    const bool adds = cls == EB_WORD_INSIDE || cls == EB_WORD_END;
    return make_int3(__ldg(e), adds ? max(__ldg(e + 1), 0) : 0, cls == EB_WORD_END || cls == EB_WORD_SEP);
}

// the exact comparison of two words of len characters each, starting at tokens pa of sa and pb of sb
__device__ bool words_equal(const int* sa, int pa, const int* sb, int pb, int len, const WordTab& w) {
    int ka = 0, na = 0, oa = 0, kb = 0, nb = 0, ob = 0;
    --pa;
    --pb;
    for (int i = 0; i < len; ++i) {
        while (ka == na) {
            const int3 t = unit_info(w, __ldg(sa + ++pa));
            oa = t.x, na = t.y, ka = 0;
        }
        while (kb == nb) {
            const int3 t = unit_info(w, __ldg(sb + ++pb));
            ob = t.x, nb = t.y, kb = 0;
        }
        if (__ldg(w.chars + oa + ka) != __ldg(w.chars + ob + kb)) return false;
        ++ka, ++kb;
    }
    return true;
}

// The words of seq[0, L): a word starts at a token that adds characters while no word is open; it takes every later
// token's characters up to and including the first token that closes it (a word end or a separator).  Writes each
// word's first token, character count and hash; returns the word count.  Every thread of the CTA calls it.
__device__ int segment_words(const int* seq, int L, const WordTab& w, u64* hash, int* start, int* clen, int* sh) {
    const int tid = threadIdx.x;
    const int chunk = (L + ED_THREADS - 1) / ED_THREADS, p0 = min(tid * chunk, L), p1 = min(p0 + chunk, L);
    // state after the chunk: -1 no token that adds characters or closes, 0 a word open, 1 closed
    int last = -1;
    for (int p = p0; p < p1; ++p) {
        const int3 t = unit_info(w, __ldg(seq + p));
        if (t.z) last = 1;
        else if (t.y > 0) last = 0;
    }
    sh[tid] = last;
    __syncthreads();
    int open = 0;
    for (int q = tid - 1; q >= 0; --q)
        if (sh[q] >= 0) {
            open = sh[q] == 0;
            break;
        }
    int starts = 0;
    for (int p = p0, o = open; p < p1; ++p) {
        const int3 t = unit_info(w, __ldg(seq + p));
        if (t.y > 0 && !o) ++starts;
        if (t.z) o = 0;
        else if (t.y > 0) o = 1;
    }
    __syncthreads();
    sh[tid] = starts;
    __syncthreads();
    int k = 0, total = 0;
    for (int q = 0; q < ED_THREADS; ++q) {
        if (q < tid) k += sh[q];
        total += sh[q];
    }
    for (int p = p0, o = open; p < p1; ++p) {
        const int3 t = unit_info(w, __ldg(seq + p));
        if (t.y > 0 && !o) {
            u64 h = 1469598103934665603ull;                 // FNV-1a over the code points
            int n = 0;
            for (int r = p; r < L; ++r) {
                const int3 u = unit_info(w, __ldg(seq + r));
                for (int c = 0; c < u.y; ++c) h = (h ^ (unsigned)__ldg(w.chars + u.x + c)) * 1099511628211ull;
                n += u.y;
                if (u.z) break;
            }
            hash[k] = h, start[k] = p, clen[k] = n;
            ++k;
        }
        if (t.z) o = 0;
        else if (t.y > 0) o = 1;
    }
    __syncthreads();
    return total;
}

// meta: hyp_len [n_hyp] | ref_len [n_ref] | ref_index [n_hyp]
__global__ void __launch_bounds__(ED_THREADS) edit_distance_kernel(const int* __restrict__ hyp, long ld_h,
                                                                   const int* __restrict__ ref, long ld_r,
                                                                   const int* __restrict__ meta, int n_hyp, int n_ref,
                                                                   WordTab w, int word, int cap_h, int cap_r,
                                                                   int* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int pair = blockIdx.x, tid = threadIdx.x;
    const int r = meta[n_hyp + n_ref + pair];
    if (r < 0 || r >= n_ref) {                            // refused on the host; never read outside the buffers
        if (tid < 5) out[5 * (long)pair + tid] = -1;
        return;
    }
    int Lh = min(max(meta[pair], 0), cap_h), Lr = min(max(meta[n_hyp + r], 0), cap_r);
    const int* hs = hyp + pair * ld_h;
    const int* rs = ref + r * ld_r;
    int* sh = reinterpret_cast<int*>(smem);                          // [ED_THREADS]
    int* uh = sh + ED_THREADS;                                       // [cap_h] hypothesis units
    int* ur = uh + cap_h;                                            // [cap_r] reference units
    unsigned char* region = smem + (((ED_THREADS + cap_h + cap_r) * 4 + 15) & ~15);
    if (word) {
        u64* hash_r = reinterpret_cast<u64*>(region);
        u64* hash_h = hash_r + cap_r;
        int* start_r = reinterpret_cast<int*>(hash_h + cap_h);
        int* start_h = start_r + cap_r;
        int* clen_r = start_h + cap_h;
        int* clen_h = clen_r + cap_r;
        Lr = segment_words(rs, Lr, w, hash_r, start_r, clen_r, sh);
        Lh = segment_words(hs, Lh, w, hash_h, start_h, clen_h, sh);
        // a reference word's unit is the index of the first reference word equal to it; a hypothesis word takes the
        // unit of the first reference word equal to it, -1 when there is none
        for (int i = tid; i < Lr; i += ED_THREADS) {
            int k = 0;
            while (k < i && !(hash_r[k] == hash_r[i] && clen_r[k] == clen_r[i] &&
                              words_equal(rs, start_r[k], rs, start_r[i], clen_r[i], w)))
                ++k;
            ur[i] = k;
        }
        for (int j = tid; j < Lh; j += ED_THREADS) {
            int k = 0;
            while (k < Lr && !(hash_r[k] == hash_h[j] && clen_r[k] == clen_h[j] &&
                               words_equal(rs, start_r[k], hs, start_h[j], clen_h[j], w)))
                ++k;
            uh[j] = k < Lr ? k : -1;
        }
    } else {
        for (int j = tid; j < Lh; j += ED_THREADS) uh[j] = __ldg(hs + j);
        for (int i = tid; i < Lr; i += ED_THREADS) ur[i] = __ldg(rs + i);
    }
    __syncthreads();
    // D[i][j]: the first i reference units against the first j hypothesis units, on anti-diagonal d = i + j at index i
    u64* dg = reinterpret_cast<u64*>(region);
    const int ld = cap_r + 1;
    for (int d = 0; d <= Lr + Lh; ++d) {
        u64* cur = dg + (d % 3) * ld;
        const u64* p1 = dg + ((d + 2) % 3) * ld;                     // d - 1
        const u64* p2 = dg + ((d + 1) % 3) * ld;                     // d - 2
        for (int i = max(0, d - Lh) + tid; i <= min(Lr, d); i += ED_THREADS) {
            const int j = d - i;
            u64 v;
            if (i == 0) v = (u64)j * ED_INS;
            else if (j == 0) v = (u64)i * ED_DEL;
            else {
                const u64 dia = p2[i - 1] + (ur[i - 1] == uh[j - 1] ? 0ull : ED_SUB);
                const u64 del = p1[i - 1] + ED_DEL, ins = p1[i] + ED_INS;
                const unsigned a = (unsigned)(dia >> 48), b = (unsigned)(del >> 48), c = (unsigned)(ins >> 48);
                v = (a <= b && a <= c) ? dia : (b <= c ? del : ins);     // the diagonal on ties, then the deletion
            }
            cur[i] = v;
        }
        __syncthreads();
    }
    if (tid == 0) {
        const u64 v = dg[((Lr + Lh) % 3) * ld + Lr];
        int* o = out + 5 * (long)pair;
        o[0] = (int)(v >> 48);
        o[1] = (int)(v & 0xffff);
        o[2] = (int)((v >> 16) & 0xffff);
        o[3] = (int)((v >> 32) & 0xffff);
        o[4] = Lr;
    }
}

constexpr int PACK_THREADS = 128;

__global__ void __launch_bounds__(PACK_THREADS) nbest_pack_kernel(const int* __restrict__ ids,
                                                                  const int* __restrict__ count, int N, int L,
                                                                  const int* __restrict__ ref, int ld_ref,
                                                                  const int* __restrict__ ref_len,
                                                                  int* __restrict__ labels, int ld_out,
                                                                  int* __restrict__ lens, int* __restrict__ valid) {
    __shared__ int first;
    const int row = blockIdx.x, b = row / (N + 1), i = row % (N + 1), tid = threadIdx.x;
    int* lab = labels + (long)row * ld_out;
    const int* src;
    int n;
    if (i == N) {
        src = ref + (long)b * ld_ref;
        n = min(max(ref_len[b], 0), min(ld_ref, ld_out));
    } else {
        const int cnt = min(max(count[b], 0), N);
        if (tid == 0) valid[b * N + i] = i < cnt;
        if (tid == 0) first = L;
        __syncthreads();
        src = ids + ((long)b * N + i) * L;
        if (i < cnt)
            for (int k = tid; k < L; k += PACK_THREADS)
                if (src[k] >= 0 && (k == 0 || src[k - 1] < 0)) atomicMin(&first, k);
        __syncthreads();
        n = i < cnt ? min(L - first, ld_out) : 0;
        src += first;
    }
    for (int k = tid; k < ld_out; k += PACK_THREADS) lab[k] = k < n ? src[k] : 0;
    if (tid == 0) lens[row] = n;
}

// The posteriors and the risk of utterance b, in fp64 and rank order: m = max of -c over the valid ranks, P_i =
// exp(-c_i - m) / sum_j exp(-c_j - m), Ebar = mean of the valid errors, risk = sum_i P_i (E_i - Ebar).
__device__ double utterance_risk(const float* c, const int* e, const int* valid, int N, double* post, double* ebar) {
    double m = -INFINITY;
    int n = 0;
    long esum = 0;
    for (int i = 0; i < N; ++i)
        if (valid[i]) m = fmax(m, -(double)c[i]), ++n, esum += e[i];
    double z = 0.0;
    for (int i = 0; i < N; ++i)
        if (valid[i]) z += exp(-(double)c[i] - m);
    *ebar = n ? (double)esum / n : 0.0;
    double risk = 0.0;
    for (int i = 0; i < N; ++i) {
        post[i] = valid[i] ? exp(-(double)c[i] - m) / z : 0.0;
        if (valid[i]) risk += post[i] * ((double)e[i] - *ebar);
    }
    return risk;
}

__global__ void mwer_risk_kernel(const float* __restrict__ costs, const int* __restrict__ errors,
                                 const int* __restrict__ valid, int N, float* __restrict__ post,
                                 double* __restrict__ risk) {
    __shared__ double p[EB_BEAM_MAX_W];
    const int b = blockIdx.x;
    const long o = (long)b * N;
    __shared__ double rb;
    if (threadIdx.x == 0) {
        double ebar;
        rb = utterance_risk(costs + o, errors + o, valid + o, N, p, &ebar);
        risk[b] = rb;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) post[o + i] = (float)p[i];
}

__global__ void mwer_loss_kernel(const double* __restrict__ risk, int B, float* __restrict__ loss) {
    double s = 0.0;
    for (int b = 0; b < B; ++b) s += risk[b];
    *loss = (float)(s / B);
}

// d loss / d c_i = -P_i (E_i - sum_j P_j E_j) / B * g, with sum_j P_j E_j taken as Ebar + risk: equal errors give 0
__global__ void mwer_risk_bwd_kernel(const float* __restrict__ costs, const int* __restrict__ errors,
                                     const int* __restrict__ valid, int B, int N, const float* __restrict__ gout,
                                     float* __restrict__ dcosts) {
    __shared__ double p[EB_BEAM_MAX_W];
    __shared__ double ebar, rb;
    const int b = blockIdx.x;
    const long o = (long)b * N;
    if (threadIdx.x == 0) rb = utterance_risk(costs + o, errors + o, valid + o, N, p, &ebar);
    __syncthreads();
    const double g = (double)*gout / B;
    for (int i = threadIdx.x; i < N; i += blockDim.x)
        dcosts[o + i] = valid[o + i] ? (float)(-(p[i] * (((double)errors[o + i] - ebar) - rb)) * g) : 0.0f;
}

}  // namespace

EB_API size_t eb_edit_distance_smem_bytes(int cap_h, int cap_r, int word) {
    if (cap_h < 0 || cap_r < 0 || cap_h > EB_EDIT_MAX_UNITS || cap_r > EB_EDIT_MAX_UNITS) return 0;
    size_t head = ((size_t)(ED_THREADS + cap_h + cap_r) * 4 + 15) & ~(size_t)15;
    size_t dp = (size_t)3 * (cap_r + 1) * 8, wm = word ? (size_t)16 * (cap_h + cap_r) : 0;
    return head + (dp > wm ? dp : wm);
}

EB_API int eb_edit_distance(const int* hyp, long ld_h, const int* ref, long ld_r, const int* meta,
                            const int* meta_host, int n_hyp, int n_ref, const int* word_table, const int* word_chars,
                            int n_table, int vocab, int* out, void* stream) {
    if (!hyp || !ref || !meta || !meta_host || !out || n_hyp < 0 || n_ref < 0 || (n_hyp > 0 && n_ref == 0) ||
        ld_h < 0 || ld_r < 0)
        return EB_ERR_INVALID;
    const int word = word_table != nullptr;
    if (word && (!word_chars || n_table < vocab || vocab < 0)) return EB_ERR_INVALID;
    int cap_h = 0, cap_r = 0;
    for (int i = 0; i < n_hyp; ++i) {
        const int n = meta_host[i], r = meta_host[n_hyp + n_ref + i];
        if (n < 0 || n > EB_EDIT_MAX_UNITS || n > ld_h || r < 0 || r >= n_ref) return EB_ERR_INVALID;
        cap_h = n > cap_h ? n : cap_h;
    }
    for (int i = 0; i < n_ref; ++i) {
        const int n = meta_host[n_hyp + i];
        if (n < 0 || n > EB_EDIT_MAX_UNITS || n > ld_r) return EB_ERR_INVALID;
        cap_r = n > cap_r ? n : cap_r;
    }
    if (n_hyp == 0) return EB_OK;
    const size_t smem = eb_edit_distance_smem_bytes(cap_h, cap_r, word);
    EB_CUDA(cudaFuncSetAttribute(edit_distance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    edit_distance_kernel<<<n_hyp, ED_THREADS, smem, (cudaStream_t)stream>>>(
        hyp, ld_h, ref, ld_r, meta, n_hyp, n_ref, WordTab{word_table, word_chars, n_table}, word, cap_h, cap_r, out);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_nbest_pack(const int* ids, const int* count, int B, int N, int L, const int* ref, int ld_ref,
                         const int* ref_len, int* labels, int ld_out, int* lens, int* valid, void* stream) {
    if (!ids || !count || !ref || !ref_len || !labels || !lens || !valid || B < 0 || N < 1 || N > EB_BEAM_MAX_W ||
        L < 1 || ld_ref < 0 || ld_out < L || ld_out < ld_ref)
        return EB_ERR_INVALID;
    if (B == 0) return EB_OK;
    nbest_pack_kernel<<<B * (N + 1), PACK_THREADS, 0, (cudaStream_t)stream>>>(ids, count, N, L, ref, ld_ref, ref_len,
                                                                               labels, ld_out, lens, valid);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_mwer_risk_fwd(const float* costs, const int* errors, const int* valid, int B, int N, float* post,
                            double* risk, float* loss, void* stream) {
    if (!costs || !errors || !valid || !post || !risk || !loss || B < 1 || N < 1 || N > EB_BEAM_MAX_W)
        return EB_ERR_INVALID;
    mwer_risk_kernel<<<B, 128, 0, (cudaStream_t)stream>>>(costs, errors, valid, N, post, risk);
    EB_CHECK_LAUNCH();
    mwer_loss_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(risk, B, loss);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_mwer_risk_bwd(const float* costs, const int* errors, const int* valid, int B, int N, const float* gout,
                            float* dcosts, void* stream) {
    if (!costs || !errors || !valid || !gout || !dcosts || B < 1 || N < 1 || N > EB_BEAM_MAX_W) return EB_ERR_INVALID;
    mwer_risk_bwd_kernel<<<B, 128, 0, (cudaStream_t)stream>>>(costs, errors, valid, B, N, gout, dcosts);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
