// frontend.cu -- log-mel front end (SURVEY 8(f) row N2: the step before the hot path), fp32.
//
// Reference: rnnt/features.py:126-164 (FilterbankFeatures.forward: pre-emphasis -> torch.stft(center, reflect,
// hann of win_length centred in n_fft) -> power -> mel matmul -> log(x + 1e-20) -> zero frames >= ceil(L/hop)) and
// rnnt/transforms.py:37-51 (Downsample: stack n_frame consecutive frames, zero-pad to a multiple).
//
// Decomposition (all on the caller's stream):
//   K1 fe_preemph_pad   : x[B,L] -> xp[B,Lp]  pre-emphasised, reflect-padded by n_fft/2, rows padded with zeros
//                         to Lp = multiple of hop, so that frame g = b*(Lp/hop) + f of the FLAT buffer starts at
//                         g*hop: the framing is a strided view (row stride hop), never materialised;
//   G1 eb_gemm_f32      : spec[g, 0:NB | NB:2NB] = frames[g, :] @ (window * cos | -window * sin)   (direct DFT as an
//                         exact-fp32 GEMM: n_fft = 512 is a 512-deep contraction, 0.4 GFLOP per second of audio);
//   K2 fe_power         : P[g,k] = re^2 + im^2;
//   G2 eb_gemm_f32      : mel[g,m] = P[g,:] @ fb[m,:]^T;
//   K3 fe_log_stack     : out[b,t,s*n_mels+m] = log(mel[g(b, t*n_frame+s), m] + 1e-20), zero for masked / padded
//                         frames -- directly in the [B, T, n_mels*n_frame] layout Encoder.forward consumes.
//
// Per-utterance lengths (a padded batch, as rnnt/dataset.py:202-240 collates the reference's per-utterance features):
// K1 and K3 take a device int32 lens[B] (nullptr: every utterance is L long).  Utterance b then reflects at its own
// L_b, has F_b = 1 + L_b/hop frames and T_b = ceil(F_b/n) (or floor) output rows, and rows t >= T_b are zero.  K3 also
// computes CatDeltas (rnnt/transforms.py:10-16: torchaudio compute_deltas twice, window 5, replicate edge at F_b - 1)
// and writes [static | d1 | d2] per stacked frame, the channel order Downsample's reshape gives.  The MFCC path adds
// fe_log (log(mel + 1e-6)) and one more eb_gemm_f32 against the orthonormal DCT-II matrix before K3.
#include "frontend.cuh"
#include "../../include/edgedict_b200.h"

namespace {

// row b of x is L samples apart; its first lens[b] (or L) are the utterance
__global__ void fe_preemph_pad_kernel(const float* __restrict__ x, const int* __restrict__ lens, float* __restrict__ xp,
                                      int L, long Lp, int pad, float preemph, int use_preemph) {
    const int b = blockIdx.y;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Lp) return;
    const int Lb = lens ? lens[b] : L;
    const float* row = x + (long)b * L;
    xp[(long)b * Lp + i] = fe_framed_sample([&](long r) { return row[r]; }, i, Lb, pad, preemph, use_preemph);
}

__global__ void fe_power_kernel(const float* __restrict__ spec, float* __restrict__ pw, long rows, int NB) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * NB) return;
    const long g = i / NB;
    const int k = (int)(i % NB);
    pw[i] = fe_power_value(spec[g * 2 * NB + k], spec[g * 2 * NB + NB + k]);
}

// feat [B*R, C] per-frame rows -> out[b, t, s*Cd + j*C + c] (Cd = C * (delta ? 3 : 1); j = 0 static, 1 d1, 2 d2) for
// frame f = t*n_frame + s < F_stack, zero elsewhere.  lens == nullptr: every utterance has F_stack = F = n_frames
// frames and its mask at seq_len; else utterance b has F = 1 + lens[b]/hop, its mask at ceil(lens[b]/hop) (use_mask)
// or none, and F_stack = F (pad_div) or F - F % n_frame.
__global__ void fe_finish_kernel(const float* __restrict__ feat, float* __restrict__ out, const int* __restrict__ lens,
                                 int R, int n_frames, int seq_len, int hop, int use_mask, int pad_div, int C,
                                 int n_frame, int Tout, int take_log, int delta) {
    const int b = blockIdx.y;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int W = (delta ? 3 * C : C) * n_frame;
    if (i >= (long)Tout * W) return;
    int F = n_frames, Fs = n_frames, seq = seq_len;
    if (lens) {
        const int Lb = lens[b];
        F = 1 + Lb / hop;
        seq = use_mask ? (Lb + hop - 1) / hop : F;
        Fs = pad_div ? F : F - F % n_frame;
    }
    const float* rows = feat + (long)b * R * C;
    out[(long)b * Tout * W + i] = fe_finish_value([&](long k) { return __ldg(rows + k); }, (int)(i / W), (int)(i % W), F,
                                                  Fs, seq, C, n_frame, take_log, delta);
}

__global__ void fe_log_kernel(float* __restrict__ x, long n, float offset) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = fe_log_value(x[i], offset);
}

// SpecAugment masking (rnnt/transforms.py:53-147): x [B, D1, D2]; spans [B, nmask, 2] = [start, end) along dim `axis`
// (1: frequency rows, 2: time columns); masked elements := fill.
__global__ void fe_mask_kernel(float* __restrict__ x, const int* __restrict__ spans, int nmask, int D1, int D2, int axis,
                               float fill) {
    const int b = blockIdx.y;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)D1 * D2) return;
    const int pos = axis == 1 ? (int)(i / D2) : (int)(i % D2);
    const int* sp = spans + (long)b * nmask * 2;
    bool hit = false;
    for (int m = 0; m < nmask; ++m) hit = hit || (pos >= sp[2 * m] && pos < sp[2 * m + 1]);
    if (hit) x[(long)b * D1 * D2 + i] = fill;
}

}  // namespace

EB_API int eb_fe_mask(float* x, const int* spans, int B, int D1, int D2, int nmask, int axis, float fill, void* stream) {
    if (!x || !spans || B <= 0 || D1 <= 0 || D2 <= 0 || nmask <= 0 || (axis != 1 && axis != 2)) return EB_ERR_INVALID;
    dim3 grid((unsigned)(((long)D1 * D2 + 255) / 256), B);
    fe_mask_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, spans, nmask, D1, D2, axis, fill);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_fe_preemph_pad(const float* x, float* xp, int B, int L, long Lp, int pad, float preemph,
                             int use_preemph, void* stream) {
    if (!x || !xp || B <= 0 || L <= 1 || pad < 0 || pad >= L || Lp < (long)L + 2 * pad) return EB_ERR_INVALID;
    dim3 grid((unsigned)((Lp + 255) / 256), B);
    fe_preemph_pad_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, nullptr, xp, L, Lp, pad, preemph,
                                                                                    use_preemph);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_fe_power(const float* spec, float* power, long rows, int nbins, void* stream) {
    if (!spec || !power || rows <= 0 || nbins <= 0) return EB_ERR_INVALID;
    const long n = rows * nbins;
    fe_power_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(spec, power, rows, nbins);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_fe_log_stack(const float* mel, float* out, int B, int rows_per_utt, int n_frames, int seq_len,
                           int n_mels, int n_stack, int t_out, int take_log, void* stream) {
    if (!mel || !out || B <= 0 || rows_per_utt < n_frames || n_frames <= 0 || n_mels <= 0 || n_stack <= 0 ||
        t_out <= 0)
        return EB_ERR_INVALID;
    const long per = (long)t_out * n_mels * n_stack;
    dim3 grid((unsigned)((per + 255) / 256), B);
    fe_finish_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(mel, out, nullptr, rows_per_utt, n_frames,
                                                                               seq_len, 1, 0, 1, n_mels, n_stack, t_out,
                                                                               take_log, 0);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

// Host-side checks of the per-utterance lengths (lens, on the host; lens_dev holds the same values on the device).
static bool fe_lens_ok(const int* lens, int B, int lo, int hi) {
    for (int b = 0; b < B; ++b)
        if (lens[b] <= lo || lens[b] > hi) return false;
    return true;
}

EB_API int eb_fe_preemph_pad_lens(const float* x, const int* lens, const int* lens_dev, float* xp, int B, int L, long Lp,
                                  int pad, float preemph, int use_preemph, void* stream) {
    if (!x || !lens || !lens_dev || !xp || B <= 0 || L <= 1 || pad < 0 || Lp < (long)L + 2 * pad) return EB_ERR_INVALID;
    if (!fe_lens_ok(lens, B, pad, L)) return EB_ERR_INVALID;       // torch's reflect pad needs pad < L_b
    dim3 grid((unsigned)((Lp + 255) / 256), B);
    fe_preemph_pad_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, lens_dev, xp, L, Lp, pad, preemph,
                                                                                    use_preemph);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_fe_log(float* x, long n, float offset, void* stream) {
    if (!x || n <= 0 || !(offset > 0.f)) return EB_ERR_INVALID;
    fe_log_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, n, offset);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_fe_finish(const float* feat, float* out, const int* lens, const int* lens_dev, int B, int rows_per_utt,
                        int hop, int n_ch, int n_stack, int t_out, int take_log, int use_mask, int delta,
                        int pad_to_divisible, void* stream) {
    if (!feat || !out || !lens || !lens_dev || B <= 0 || rows_per_utt <= 0 || hop <= 0 || n_ch <= 0 || n_stack <= 0 ||
        t_out <= 0)
        return EB_ERR_INVALID;
    for (int b = 0; b < B; ++b) {
        if (lens[b] <= 0) return EB_ERR_INVALID;
        const int F = 1 + lens[b] / hop;
        const int T = pad_to_divisible ? (F + n_stack - 1) / n_stack : F / n_stack;
        if (F > rows_per_utt || T > t_out) return EB_ERR_INVALID;
    }
    const int W = n_ch * (delta ? 3 : 1) * n_stack;
    dim3 grid((unsigned)(((long)t_out * W + 255) / 256), B);
    fe_finish_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(feat, out, lens_dev, rows_per_utt, 0, 0, hop,
                                                                               use_mask, pad_to_divisible, n_ch, n_stack,
                                                                               t_out, take_log, delta);
    EB_CHECK_LAUNCH();
    return EB_OK;
}

EB_API int eb_fe_deltas(const float* feat, float* out, int B, int n_frames, int n_ch, void* stream) {
    if (!feat || !out || B <= 0 || n_frames <= 0 || n_ch <= 0) return EB_ERR_INVALID;
    dim3 grid((unsigned)(((long)n_frames * 3 * n_ch + 255) / 256), B);
    fe_finish_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(feat, out, nullptr, n_frames, n_frames,
                                                                               n_frames, 1, 0, 1, n_ch, 1, n_frames, 0, 1);
    EB_CHECK_LAUNCH();
    return EB_OK;
}
