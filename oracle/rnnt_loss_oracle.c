/*
 * oracle/rnnt_loss_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of the RNN-Transducer forward-backward loss that the
 * reference vendors in warp-transducer.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference leg may load this file's
 * shared object; the product path (edgedict_b200/csrc) never links it.
 *
 * Parity pin: checked against the reference's known-answer vectors
 * (warp-transducer/tests/test_cpu.cpp:12-179, pytorch_binding/test/test.py:51-161)
 * in tests/test_oracle_loss.py, and against oracle/_ref/libwarprnnt_ref.so
 * (the reference's own CPU library, tests/golden/ref_loss.npz) on random
 * problems.
 *
 * What follows what:
 *   lse2_*            <- include/detail/rnnt_helper.h:17-24  (log_sum_exp via log1p(exp))
 *   row_log_softmax_* <- what warprnnt_pytorch/__init__.py:95-98 asks torch to do
 *                        before the CPU library is called
 *   lattice_*         <- include/detail/cpu_rnnt.h:115-128 (blank/label gather),
 *                        :175-212 (alphas), :214-270 (betas + grads wrt log-probs)
 *   logits_grad_*     <- include/detail/gpu_rnnt_kernel.h:143-179 (dense gradient wrt
 *                        logits, the semantics of the reference's GPU entry point)
 *
 * Layout everywhere: acts[((b*maxT + t)*maxU + u)*V + v]  (include/rnnt.h:75-80),
 * labels[b*(maxU-1) + u]  (cpu_rnnt.h:299).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_DEFINE(T, SFX, EXPF, LOGF, LOG1PF, NEGINF)                                   \
                                                                                            \
static T lse2_##SFX(T a, T b) {                                                             \
    if (a == NEGINF) return b;                                                              \
    if (b == NEGINF) return a;                                                              \
    return (a > b) ? (T)(LOG1PF(EXPF(b - a)) + a) : (T)(LOG1PF(EXPF(a - b)) + b);           \
}                                                                                           \
                                                                                            \
/* out[r, :] = x[r, :] - logsumexp(x[r, :]) ; also returns -logsumexp in denom if !NULL */  \
void oracle_row_log_softmax_##SFX(const T* x, T* out, T* denom, long rows, int V) {         \
    for (long r = 0; r < rows; ++r) {                                                       \
        const T* xr = x + r * (long)V;                                                      \
        T m = xr[0];                                                                        \
        for (int v = 1; v < V; ++v) if (xr[v] > m) m = xr[v];                               \
        T s = 0;                                                                            \
        for (int v = 0; v < V; ++v) s += EXPF(xr[v] - m);                                   \
        T d = -m - LOGF(s);                                                                 \
        if (denom) denom[r] = d;                                                            \
        if (out) { T* o = out + r * (long)V; for (int v = 0; v < V; ++v) o[v] = xr[v] + d; }\
    }                                                                                       \
}                                                                                           \
                                                                                            \
/* One utterance.  lp2[(t*U+u)*2 + {0,1}] = log p(blank | t,u), log p(label[u] | t,u).      \
 * alphas/betas are [T*U].  Returns log-likelihood from the forward pass; *ll_b gets the    \
 * backward one (cpu_rnnt.h:167-170 compares them).                                         */ \
static T lattice_##SFX(const T* lp2, int Tn, int U, T* alphas, T* betas, T* ll_b) {         \
    alphas[0] = 0;                                                                          \
    for (int t = 0; t < Tn; ++t)                                                            \
        for (int u = 0; u < U; ++u) {                                                       \
            if (u == 0 && t > 0)                                                            \
                alphas[t * U] = alphas[(t - 1) * U] + lp2[((t - 1) * U) * 2];               \
            if (t == 0 && u > 0)                                                            \
                alphas[u] = alphas[u - 1] + lp2[(u - 1) * 2 + 1];                           \
            if (t > 0 && u > 0) {                                                           \
                T stay = alphas[(t - 1) * U + u] + lp2[((t - 1) * U + u) * 2];              \
                T emit = alphas[t * U + u - 1] + lp2[(t * U + u - 1) * 2 + 1];              \
                alphas[t * U + u] = lse2_##SFX(emit, stay);                                 \
            }                                                                               \
        }                                                                                   \
    T ll = alphas[(Tn - 1) * U + U - 1] + lp2[((Tn - 1) * U + U - 1) * 2];                  \
    if (betas) {                                                                            \
        betas[(Tn - 1) * U + U - 1] = lp2[((Tn - 1) * U + U - 1) * 2];                      \
        for (int t = Tn - 1; t >= 0; --t)                                                   \
            for (int u = U - 1; u >= 0; --u) {                                              \
                if (u == U - 1 && t < Tn - 1)                                               \
                    betas[t * U + U - 1] = betas[(t + 1) * U + U - 1] + lp2[(t * U + U - 1) * 2]; \
                if (t == Tn - 1 && u < U - 1)                                               \
                    betas[t * U + u] = betas[t * U + u + 1] + lp2[(t * U + u) * 2 + 1];     \
                if (t < Tn - 1 && u < U - 1) {                                              \
                    T stay = betas[(t + 1) * U + u] + lp2[(t * U + u) * 2];                 \
                    T emit = betas[t * U + u + 1] + lp2[(t * U + u) * 2 + 1];               \
                    betas[t * U + u] = lse2_##SFX(emit, stay);                              \
                }                                                                           \
            }                                                                               \
        if (ll_b) *ll_b = betas[0];                                                         \
    }                                                                                       \
    return ll;                                                                              \
}                                                                                           \
                                                                                            \
/* CPU-entry-point semantics (acts are LOG-PROBS; grads wrt log-probs, sparse).             \
 * grads may be NULL (score_forward, cpu_rnnt.h:306-338).  alphas_out/betas_out optional    \
 * [B*maxT*maxU] dumps (row stride maxU) for debugging kernels.  Returns 0.                 */ \
int oracle_rnnt_logprobs_##SFX(const T* log_probs, T* grads, const int* labels,             \
                               const int* label_lengths, const int* input_lengths,          \
                               int V, int B, int maxT, int maxU, int blank, T* costs,       \
                               T* alphas_out, T* betas_out) {                               \
    T* lp2 = (T*)malloc(sizeof(T) * (size_t)maxT * maxU * 2);                               \
    T* al = (T*)malloc(sizeof(T) * (size_t)maxT * maxU);                                    \
    T* be = (T*)malloc(sizeof(T) * (size_t)maxT * maxU);                                    \
    for (int b = 0; b < B; ++b) {                                                           \
        const int Tn = input_lengths[b], U = label_lengths[b] + 1;                          \
        const long per = (long)maxT * maxU * V;                                             \
        const T* lp = log_probs + b * per;                                                  \
        const int* lab = labels + b * (maxU - 1);                                           \
        for (int t = 0; t < Tn; ++t)                                                        \
            for (int u = 0; u < U; ++u) {                                                   \
                long cell = ((long)t * maxU + u) * V;                                       \
                lp2[(t * U + u) * 2] = lp[cell + blank];                                    \
                if (u < U - 1) lp2[(t * U + u) * 2 + 1] = lp[cell + lab[u]];                \
            }                                                                               \
        T llb = 0;                                                                          \
        T ll = lattice_##SFX(lp2, Tn, U, al, grads ? be : NULL, &llb);                      \
        costs[b] = -ll;                                                                     \
        if (grads) {                                                                        \
            T* g = grads + b * per;                                                         \
            memset(g, 0, sizeof(T) * (size_t)per);                                          \
            /* cpu_rnnt.h:252-267 uses the BACKWARD log-likelihood as normaliser */         \
            for (int t = 0; t < Tn; ++t)                                                    \
                for (int u = 0; u < U; ++u) {                                               \
                    long cell = ((long)t * maxU + u) * V;                                   \
                    if (t < Tn - 1)                                                         \
                        g[cell + blank] = -EXPF(lp2[(t * U + u) * 2] + (al[t * U + u] +     \
                                                be[(t + 1) * U + u]) - llb);                \
                    if (u < U - 1)                                                          \
                        g[cell + lab[u]] = -EXPF(lp2[(t * U + u) * 2 + 1] + (al[t * U + u] +\
                                                 be[t * U + u + 1]) - llb);                 \
                }                                                                           \
            g[((long)(Tn - 1) * maxU + U - 1) * V + blank] =                                \
                -EXPF(lp2[((Tn - 1) * U + U - 1) * 2] + al[(Tn - 1) * U + U - 1] - llb);    \
        }                                                                                   \
        for (int t = 0; t < Tn; ++t)                                                        \
            for (int u = 0; u < U; ++u) {                                                   \
                if (alphas_out) alphas_out[((long)b * maxT + t) * maxU + u] = al[t * U + u];\
                if (betas_out && grads) betas_out[((long)b * maxT + t) * maxU + u] = be[t * U + u]; \
            }                                                                               \
    }                                                                                       \
    free(lp2); free(al); free(be);                                                          \
    return 0;                                                                               \
}                                                                                           \
                                                                                            \
/* GPU-entry-point semantics (acts are raw LOGITS; grads wrt logits, dense, zero on padded  \
 * cells; normaliser is the FORWARD log-likelihood, gpu_rnnt.h:198-200).                    */ \
int oracle_rnnt_logits_##SFX(const T* logits, T* grads, const int* labels,                  \
                             const int* label_lengths, const int* input_lengths,            \
                             int V, int B, int maxT, int maxU, int blank, T* costs) {       \
    T* lp2 = (T*)malloc(sizeof(T) * (size_t)maxT * maxU * 2);                               \
    T* al = (T*)malloc(sizeof(T) * (size_t)maxT * maxU);                                    \
    T* be = (T*)malloc(sizeof(T) * (size_t)maxT * maxU);                                    \
    T* den = (T*)malloc(sizeof(T) * (size_t)maxT * maxU);                                   \
    for (int b = 0; b < B; ++b) {                                                           \
        const int Tn = input_lengths[b], U = label_lengths[b] + 1;                          \
        const long per = (long)maxT * maxU * V;                                             \
        const T* x = logits + b * per;                                                      \
        const int* lab = labels + b * (maxU - 1);                                           \
        oracle_row_log_softmax_##SFX(x, NULL, den, (long)maxT * maxU, V);                   \
        for (int t = 0; t < Tn; ++t)                                                        \
            for (int u = 0; u < U; ++u) {                                                   \
                long col = (long)t * maxU + u;                                              \
                lp2[(t * U + u) * 2] = den[col] + x[col * V + blank];                       \
                if (u < U - 1) lp2[(t * U + u) * 2 + 1] = den[col] + x[col * V + lab[u]];   \
            }                                                                               \
        T llb = 0;                                                                          \
        T ll = lattice_##SFX(lp2, Tn, U, al, grads ? be : NULL, &llb);                      \
        costs[b] = -ll;                                                                     \
        if (!grads) continue;                                                               \
        T* g = grads + b * per;                                                             \
        memset(g, 0, sizeof(T) * (size_t)per);                                              \
        for (int t = 0; t < Tn; ++t)                                                        \
            for (int u = 0; u < U; ++u) {                                                   \
                long col = (long)t * maxU + u;                                              \
                T a = al[t * U + u], bt = be[t * U + u];                                    \
                for (int v = 0; v < V; ++v) {                                               \
                    T logpk = den[col] + x[col * V + v];                                    \
                    T gr = EXPF(a + bt + logpk - ll);                                       \
                    if (v == blank && t == Tn - 1 && u == U - 1) gr -= EXPF(a + logpk - ll);\
                    if (v == blank && t < Tn - 1) gr -= EXPF(a + logpk - ll + be[(t + 1) * U + u]); \
                    if (u < U - 1 && v == lab[u]) gr -= EXPF(a + logpk - ll + be[t * U + u + 1]);   \
                    g[col * V + v] = gr;                                                    \
                }                                                                           \
            }                                                                               \
    }                                                                                       \
    free(lp2); free(al); free(be); free(den);                                               \
    return 0;                                                                               \
}

ORACLE_DEFINE(float, f32, expf, logf, log1pf, (-INFINITY))
ORACLE_DEFINE(double, f64, exp, log, log1p, (-(double)INFINITY))
