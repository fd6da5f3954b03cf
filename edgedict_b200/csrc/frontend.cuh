// frontend.cuh -- the per-element arithmetic of the log-mel front end, shared by frontend.cu's batch kernels and the
// front-end phases of the streaming decode kernel (decode.cu), so that a stream engine fed raw audio computes bit for
// bit the features build_batch_transform's module gives the same window.  Every function here is one element of one
// step; the callers only decide which elements a thread computes and where the operands live.
#pragma once
#include "common.cuh"

namespace {

// Sample i of an utterance's pre-emphasised, reflect-padded row (features.py:126-164: pre-emphasis, then torch.stft's
// reflect padding by `pad` = n_fft / 2 on each side), zero at and past Lb + 2 pad.  x(r) reads raw sample r < Lb.
template <typename X>
__device__ __forceinline__ float fe_framed_sample(X x, long i, int Lb, int pad, float preemph, int use_preemph) {
    float v = 0.f;
    if (i < (long)Lb + 2 * pad) {
        long r = i - pad;                               // reflect (no edge repeat): -1 -> 1, L -> L-2
        if (r < 0) r = -r;
        if (r >= Lb) r = 2L * (Lb - 1) - r;
        v = x(r);
        if (use_preemph && r > 0) v -= preemph * x(r - 1);
    }
    return v;
}

// |X_k|^2 from bin k's real and imaginary parts (a direct-DFT row is [re 0..NB-1 | im 0..NB-1])
__device__ __forceinline__ float fe_power_value(float re, float im) { return re * re + im * im; }

// Static feature of frame f (< F), channel c: the optional log(x + 1e-20) of features.py:155-156, zero from frame `seq`
// on (features.py:160-164; seq = F when there is no mask).  rows(k) reads element k of the utterance's [F, C] rows.
template <typename R>
__device__ __forceinline__ float fe_static(R rows, int f, int c, int C, int seq, int take_log) {
    if (f >= seq) return 0.f;
    const float v = rows((long)f * C + c);
    return take_log ? logf(v + 1e-20f) : v;
}

__device__ __forceinline__ int fe_clamp(int f, int F) { return f < 0 ? 0 : (f >= F ? F - 1 : f); }

// torchaudio compute_deltas (window 5, replicate padding): d[f] = sum_{k=-2..2} k x[clamp(f+k, 0, F-1)] / 10
template <typename R>
__device__ float fe_delta1(R rows, int f, int c, int C, int seq, int F, int take_log) {
    const float m2 = fe_static(rows, fe_clamp(f - 2, F), c, C, seq, take_log);
    const float m1 = fe_static(rows, fe_clamp(f - 1, F), c, C, seq, take_log);
    const float p1 = fe_static(rows, fe_clamp(f + 1, F), c, C, seq, take_log);
    const float p2 = fe_static(rows, fe_clamp(f + 2, F), c, C, seq, take_log);
    return (2.f * (p2 - m2) + (p1 - m1)) / 10.f;
}

template <typename R>
__device__ float fe_delta2(R rows, int f, int c, int C, int seq, int F, int take_log) {
    const float m2 = fe_delta1(rows, fe_clamp(f - 2, F), c, C, seq, F, take_log);
    const float m1 = fe_delta1(rows, fe_clamp(f - 1, F), c, C, seq, F, take_log);
    const float p1 = fe_delta1(rows, fe_clamp(f + 1, F), c, C, seq, F, take_log);
    const float p2 = fe_delta1(rows, fe_clamp(f + 2, F), c, C, seq, F, take_log);
    return (2.f * (p2 - m2) + (p1 - m1)) / 10.f;
}

// Element w of output row t of one utterance whose per-frame rows [F, C] rows(k) reads: frame f = t*n_frame + s of
// the stacked row, channel block j (0 static, 1 d1, 2 d2, with Cd = C * (delta ? 3 : 1)); zero for f >= Fs (the frames
// Downsample keeps), the seq_len mask from frame seq on.
template <typename R>
__device__ __forceinline__ float fe_finish_value(R rows, int t, int w, int F, int Fs, int seq,
                                                 int C, int n_frame, int take_log, int delta) {
    const int Cd = delta ? 3 * C : C;
    const int s = w / Cd, j = (w % Cd) / C, c = w % C;
    const int f = t * n_frame + s;
    float v = 0.f;
    if (f < Fs) {
        if (j == 0) v = fe_static(rows, f, c, C, seq, take_log);
        else if (j == 1) v = fe_delta1(rows, f, c, C, seq, F, take_log);
        else v = fe_delta2(rows, f, c, C, seq, F, take_log);
    }
    return v;
}

__device__ __forceinline__ float fe_log_value(float x, float offset) { return logf(x + offset); }

}  // namespace
