/* include/edgedict_b200.h -- C ABI of libedgedict_b200.so (sm_90a).
 *
 * Plain pointers and sizes only; every pointer is a DEVICE pointer unless its name ends in
 * _host; every call is asynchronous on `stream` (a cudaStream_t passed as void*) and returns
 * 0 on success, 2 for invalid arguments, 3 for a CUDA error.  No call allocates memory:
 * callers own all buffers (same ownership rule as warp-transducer, README.md:36-37).
 *
 * Each entry point names the piece of the reference it replaces (paths relative to the
 * root of the reference project).  The reference has no FFI for the model path (it calls torch.nn modules),
 * so those entry points mirror the module boundaries of rnnt/models.py.
 */
#pragma once
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- RNN-T loss, device-resident costs, no host sync ------------------------------------
 * replaces warp-transducer/include/detail/gpu_rnnt.h:82-215 (GpuRNNT::compute_cost_and_score)
 * and warprnnt_pytorch/__init__.py:10-50 (_RNNT.forward/backward).
 *   logits [B,maxT,maxU,V] (dtype_size 4|8), labels [B,maxU-1] int32, xlen/ylen [B] int32, 1 <= maxU <= 1024.
 * Lengths (eb_rnnt_loss_fwd / _bwd / _lattice / _bwd_bf16 and eb_joint_logits_lse alike): utterance b has the cells
 *   t < T = min(max(xlen[b], 0), maxT), u < U = min(max(ylen[b], 0), maxU-1) + 1, the same clamp as eb_rnnt_viterbi;
 *   no kernel reads or writes a cell, a label or a gradient row of b outside them, other than zero-filling the
 *   gradient of its padded cells.
 * T = 0 has no alignment: ll_fwd = ll_bwd = -inf (cost +inf) and a zero gradient. */
size_t eb_rnnt_workspace_bytes(int B, int maxT, int maxU, int dtype_size);
int eb_rnnt_loss_fwd(const void* logits, const int* labels, const int* xlen, const int* ylen,
                     int B, int maxT, int maxU, int V, int blank, int dtype_size,
                     void* workspace, void* costs_dev /* [B], may be NULL */, int need_beta,
                     void* stream);
/* grads = d(sum_b gscale[b]*cost_b)/d logits * host_scale; grads may alias logits (in place);
 * grads_bf16: write bf16 instead of fp32 (dtype_size 4 only). */
int eb_rnnt_loss_bwd(const void* logits, void* grads, int grads_bf16, const int* labels,
                     const int* xlen, const int* ylen, int B, int maxT, int maxU, int V, int blank,
                     int dtype_size, void* workspace, const void* gscale_dev /* [1]|[B]|NULL */,
                     int gscale_per_batch, double host_scale, void* stream);
/* bf16-mode fused path: the joint's output GEMM writes bf16 logits AND the softmax statistics
 * (eb_joint_logits_lse below), then only the lattice runs, and the gradient is taken on bf16 logits. */
int eb_rnnt_loss_lattice(const int* xlen, const int* ylen, int B, int maxT, int maxU, void* workspace,
                         float* costs_dev, int need_beta, void* stream);
int eb_rnnt_loss_bwd_bf16(const void* logits16, void* grads16, const int* labels, const int* xlen, const int* ylen,
                          int B, int maxT, int maxU, int V, int blank, void* workspace, const float* gscale_dev,
                          int gscale_per_batch, double host_scale, void* stream);
/* The same d logits as eb_rnnt_loss_bwd_bf16 (V % 8 == 0; logits16, grads16, db_part 16-byte aligned, else
 * EB_ERR_INVALID), and db_accum[c] += the column sum of the bf16 d logits over all B*maxT*maxU rows, the same bits as
 * eb_colsum on them.  db_part: fp32 scratch of 512 * V. */
int eb_rnnt_loss_bwd_bf16_db(const void* logits16, void* grads16, const int* labels, const int* xlen, const int* ylen,
                             int B, int maxT, int maxU, int V, int blank, void* workspace, const float* gscale_dev,
                             int gscale_per_batch, double host_scale, float* db_part, float* db_accum, void* stream);
/* FastEmit (Yu et al., ICASSP 2021): the three backward entries above with fastemit_lambda = lambda >= 0 (finite, else
 * EB_ERR_INVALID before any launch); each of those is the _fe entry with lambda = 0, whose gradient is the same bits.
 * The gradient is that of the surrogate
 *   S_b = -log P_b - lambda sum_{t < T, u < U-1} sg(gamma(t,u)) y(t,u),  y(t,u) = log p(label[u] | t,u),
 *   gamma(t,u) = exp(alpha(t,u) + y(t,u) + beta(t,u+1) - log P_b)   (the occupancy of the emit edge; sg: no gradient),
 * which scales the gradient along every label-emitting edge by (1 + lambda).  With a = alpha(t,u), beta = beta(t,u),
 * d = denom(t,u), ll = ll_fwd[b] and lpl = lpl(t,u) of the workspace, the cells u < U-1 of the gradient become
 *   g_v = exp(c_all + x_v) - [v = blank] exp(c_blank + x_v) - [v = label[u]] exp(c_lab + x_v),
 *   c_all = d + logaddexp(a + beta - ll, log lambda + a + beta(t,u+1) + lpl - ll),
 *   c_lab = a - ll + d + beta(t,u+1) + log1p(lambda),
 * and everything else is the plain loss's gradient: c_blank, the cells u = U-1, zero on padded cells and for T = 0, and
 * the scaling by host_scale * gscale.  Every valid row still sums to zero.  lambda changes no cost: costs and the
 * workspace are those of eb_rnnt_loss_fwd / eb_joint_logits_lse + eb_rnnt_loss_lattice, which take no lambda. */
int eb_rnnt_loss_bwd_fe(const void* logits, void* grads, int grads_bf16, const int* labels, const int* xlen,
                        const int* ylen, int B, int maxT, int maxU, int V, int blank, int dtype_size, void* workspace,
                        const void* gscale_dev, int gscale_per_batch, double host_scale, double fastemit_lambda,
                        void* stream);
int eb_rnnt_loss_bwd_bf16_fe(const void* logits16, void* grads16, const int* labels, const int* xlen, const int* ylen,
                             int B, int maxT, int maxU, int V, int blank, void* workspace, const float* gscale_dev,
                             int gscale_per_batch, double host_scale, double fastemit_lambda, void* stream);
int eb_rnnt_loss_bwd_bf16_db_fe(const void* logits16, void* grads16, const int* labels, const int* xlen,
                                const int* ylen, int B, int maxT, int maxU, int V, int blank, void* workspace,
                                const float* gscale_dev, int gscale_per_batch, double host_scale, float* db_part,
                                float* db_accum, double fastemit_lambda, void* stream);
int eb_rnnt_workspace_views(void* workspace, int B, int maxT, int maxU, int dtype_size,
                            void** denom, void** alphas, void** betas, void** ll_fwd, void** ll_bwd);
/* Forced (Viterbi) alignment over a workspace that eb_rnnt_loss_fwd (any need_beta) or eb_joint_logits_lse filled;
 * dtype_size 4 or 8 as it was filled, 1 <= maxU <= 1024.  The workspace holds lpb = log p(blank) and lpl =
 * log p(label u) for cell (b, t, u) at [(b*maxT + t)*maxU + u] of its second and third n = B*maxT*maxU arrays.  With
 * T = min(xlen[b], maxT), U = min(ylen[b], maxU-1) + 1 and delta in fp64:
 *   delta(0,0) = 0;  delta(t,u) = max(stay, emit), stay = delta(t-1,u) + lpb(t-1,u), emit = delta(t,u-1) + lpl(t,u-1),
 *   a term -inf when it leaves the lattice; on an exact tie the cell takes stay.
 *   score[b] = delta(T-1,U-1) + lpb(T-1,U-1), rounded to the workspace's dtype.
 * The best path is backtraced from (T-1, U-1): frames [B, maxU-1] int32 holds the frame t at which label u is emitted
 * (the step (t,u) -> (t,u+1)) and label_logp [B, maxU-1] (workspace dtype) lpl(t,u); past ylen[b] they are -1 and 0
 * (both may be NULL when maxU = 1).
 * T = 0 has no alignment: score -inf, frames -1 and label_logp -inf for every label (the loss: cost +inf).
 * decisions: eb_rnnt_align_bytes(B, maxT, maxU) bytes of scratch, NULL allowed when that is 0 (the decisions then stay
 * in shared memory).  No host synchronisation. */
size_t eb_rnnt_align_bytes(int B, int maxT, int maxU);
int eb_rnnt_viterbi(const int* xlen, const int* ylen, int B, int maxT, int maxU, int dtype_size, const void* workspace,
                    void* decisions, int* frames, void* label_logp, void* score, void* stream);

/* ---- CTC: CTCEncoder's head, loss and greedy decode (csrc/ctc.cu) ------------------------------
 * replaces tovocab's LogSoftmax and greedy_decode of CTCEncoder (rnnt/models.py:272-310) and torch.nn.CTCLoss.
 * eb_log_softmax_fwd: y[r,:] = x[r,:] - logsumexp(x[r,:]) over contiguous rows of V floats (y may alias x);
 * eb_log_softmax_bwd: dx = dy - exp(y) * sum(dy) per row (dx may alias dy).  Fixed reduction order: bitwise repeatable.
 * eb_ctc_loss_fwd: log_probs element (n, t, v) at log_probs[n*stride_n + t*stride_t + v] (torch's (T, N, C) layout or
 * the transposed [N, T, V] view); the labels of utterance n are targets[target_offsets[n] + k], k < target_lengths[n]
 * (padded (N, S) rows: offset n*S; concatenated: the running sum), ntargets the size of `targets`.  S >= every
 * target length, 0 <= S <= 1023 (2S+1 lattice states); lengths are clamped to [0, T] / [0, S], and a label outside
 * [0, V) (or an index outside `targets`) has no emission, so nothing outside the buffers is read.  costs [N] = -log p
 * (+inf when no alignment exists; 0 then when zero_infinity).  workspace: eb_ctc_workspace_size(N, T, S) bytes,
 * 8-byte aligned (0: unsupported sizes).
 * eb_ctc_loss_bwd (after the forward, same workspace): grad (strides grad_stride_n / _t, not aliasing log_probs) =
 * gscale[n] * (exp(lp) - sum_{s: l'_s = v} exp(alpha_t(s) + beta_t(s) + nll - lp_v)), the gradient torch's ctc_loss
 * returns for log_probs; zero for t >= input_lengths[n], and for the whole utterance when zero_infinity and its cost is
 * +inf.  gscale [N] may be NULL (1).  The states of one label are summed in increasing s: every value is bitwise
 * repeatable and independent of the other utterances of the batch.  alpha / beta are computed and kept in fp64.
 * eb_ctc_greedy: log_probs [B, T, V] (strides stride_b / stride_t); per frame t < min(xlen[b], T) the argmax in
 * torch.argmax order (NaN first, ties to the lowest index); frames equal to the previous frame's argmax and blanks are
 * dropped: ids [B, T] row b holds counts[b] ids; neg_score[b] = -(sum of the WHOLE log-prob rows of the kept frames),
 * the reference's score. */
int eb_log_softmax_fwd(const float* x, float* y, long rows, int V, void* stream);
int eb_log_softmax_bwd(const float* dy, const float* y, float* dx, long rows, int V, void* stream);
size_t eb_ctc_workspace_size(int N, int T, int S);
int eb_ctc_loss_fwd(const float* log_probs, long stride_n, long stride_t, int N, int T, int V, const int* targets,
                    long ntargets, const int* target_offsets, const int* target_lengths, const int* input_lengths,
                    int S, int blank, int zero_infinity, void* workspace, float* costs, void* stream);
int eb_ctc_loss_bwd(const float* log_probs, long stride_n, long stride_t, float* grad, long grad_stride_n,
                    long grad_stride_t, int N, int T, int V, const int* target_lengths, const int* input_lengths,
                    int S, int blank, int zero_infinity, const void* workspace, const float* gscale, void* stream);
int eb_ctc_greedy(const float* log_probs, long stride_b, long stride_t, int B, int T, int V, const int* xlen, int blank,
                  int* ids, int* counts, float* neg_score, void* stream);
/* eb_ctc_align: forced (Viterbi) alignment.  log_probs [B, T, V] at log_probs[b*stride_b + t*stride_t + v] (strides
 * >= 0); targets, offsets and lengths as eb_ctc_loss_fwd, 0 <= S <= 1023, lengths clamped the same way.  Over the
 * extended sequence l' of L = 2*tg_len+1 states, with delta in fp64 and e_t(s) = log_probs[b, t, l'_s]:
 *   delta_0(s) = e_0(s) for s <= 1;  delta_t(s) = max(delta_{t-1}(s), delta_{t-1}(s-1), delta_{t-1}(s-2) when l'_s is
 *   a label different from l'_{s-2}) + e_t(s), the predecessors taken in that order, a later one replacing the current
 *   only when strictly greater.  The path ends in the last label state L-2 unless the final blank L-1 is strictly
 *   greater.  alignment [B, T] int32 = l'_s of the path's state at frame t and frame_logp [B, T] its log-prob, -1 and 0
 *   for t >= in_len[b].  An utterance with no alignment (too short for its labels and repeats, a label outside [0, V))
 *   gets -1 and -inf for every frame.  workspace: eb_ctc_align_workspace_size(B, T, S) bytes of back-pointers, NULL
 *   allowed when that is 0 (they then stay in shared memory).  No host synchronisation. */
size_t eb_ctc_align_workspace_size(int B, int T, int S);
int eb_ctc_align(const float* log_probs, long stride_b, long stride_t, int B, int T, int V, const int* targets,
                 long ntargets, const int* tg_off, const int* tg_len, const int* in_len, int S, int blank, void* workspace,
                 int* alignment, float* frame_logp, void* stream);

/* ---- fp32 GEMM (parity mode of every Linear / LSTM input projection) ----------------------
 * replaces the cuBLAS/MKL calls behind nn.Linear and nn.LSTM's input GEMM (rnnt/models.py:45-46,
 * 129,148,163-167).  C = alpha*A'B' + beta*C + bias[n], A'(m,k)=A[m*sam+k*sak],
 * B'(k,n)=B[k*sbk+n*sbn]. */
int eb_gemm_f32(const float* A, long sam, long sak, const float* B, long sbk, long sbn, float* C,
                long ldc, const float* bias, int M, int N, int K, float alpha, float beta,
                void* stream);

/* ---- bf16 tensor-core GEMM (wgmma + TMA), fp32 accumulate ----------------------------------
 * same call sites in bf16 mode.  A: [M,K] (a_mn_major=0, K contiguous) or [K,M] (a_mn_major=1);
 * B: [N,K] (b_mn_major=0) or [K,N] (b_mn_major=1); C row-major [M,N] fp32 or bf16;
 * C = A*B (+ bias[n]) (+ C when accumulate).  A and B 16-byte aligned, contiguous dim % 8 == 0; C 8-byte aligned
 * (fp32) or 4-byte aligned (bf16), the width of the epilogue's paired stores. */
int eb_gemm_bf16(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C, int c_bf16,
                 const float* bias, int accumulate, long M, int N, long K, void* stream);

/* eb_gemm_bf16 with launch flags and a split-K workspace.  EB_GEMM_CORESIDENT (A and B K-major only): a 97 KB,
 * 112-register configuration that shares an SM with one CTA of a persistent recurrent kernel (eb_lstm_c4_fwd), used by
 * the layer-wavefront schedule of the encoder stack (functional.LSTMStack).  fp32-output products with few output tiles
 * split K across CTAs: every split writes its partial tile into `partials` (8-byte aligned, `partial_floats` floats;
 * eb_gemm_bf16_partials says how many it can use) and the splits are added in a fixed order, so the result is the same
 * bits on every run.  With a smaller workspace the split count shrinks to what fits (NULL / 0: no split; eb_gemm_bf16
 * passes none). */
#define EB_GEMM_CORESIDENT 1
/* EB_GEMM_FIXED_K: the tile width follows N alone (256 when N % 256 == 0) and K is never split, so every element's K
 * order is independent of M: a product computed in row blocks gives the bits of the whole product. */
#define EB_GEMM_FIXED_K 2
long eb_gemm_bf16_partials(int a_mn_major, int c_bf16, int accumulate, long M, int N, long K, int flags);
int eb_gemm_bf16_ex(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C, int c_bf16,
                    const float* bias, int accumulate, long M, int N, long K, int flags, float* partials,
                    long partial_floats, void* stream);
/* debug: per-tile clock64 stamps of CTA 0 of the wgmma GEMM ([tiles][8] int64: tile start, first operand stage ready,
 * last MMA retired, epilogue end, consumer operand-wait cycles, producer empty-wait cycles; NULL = off) */
int eb_gemm_tc_set_trace(void* dev_buf, int tiles);

/* C16[M,N] = bf16((A B) * (1 - hid16[M,N]^2)): the joint's d-hidden GEMM with the derivative of Joint.forward's Tanh
 * (rnnt/models.py:164) applied in the epilogue, so that d(pre-activation) leaves the GEMM directly. */
int eb_gemm_bf16_dtanh(const void* A, int a_mn_major, const void* B, int b_mn_major, void* C16, const void* hid16,
                       long M, int N, long K, void* stream);

/* joint output layer + softmax statistics in one GEMM (bf16 mode): replaces the second Linear of Joint
 * (rnnt/models.py:165) together with reduce_max/reduce_exp (warp-transducer reduce.h:45-104) and the
 * blank/label gathers of the lattice kernels.  denom/lpb/lpl: the first three arrays of the loss workspace, written
 * for the valid cells of the loss's length rule above. */
int eb_joint_logits_lse(const void* hidden16, const void* w2_16, const float* b2, void* logits16, const int* labels,
                        const int* xlen, const int* ylen, float* denom, float* lpb, float* lpl, int B, int maxT,
                        int maxU, int V, int J, int blank, void* stream);

/* ---- language model: the output layer's cross-entropy (csrc/lm.cu, csrc/gemm_tc.cu) -------------------------------
 * replaces decoder + F.log_softmax of the reference's LMModel (models.py:224-261) under cli/train_lm.py's
 * nn.NLLLoss(ignore_index); the [M, V] log-probs are never written.  targets [M] int32 or int64 (targets_int64).
 * eb_lm_logits_ce (bf16 mode): logits16[r, v] = bf16(hidden16[r, :] . w16[v, :] + b[v]) (hidden16 [M, K], w16 [V, K]
 *   bf16, b [V] fp32 or NULL, all 16-byte aligned, K % 8 == 0), with lse[r] = logsumexp_v of the fp32 logits and
 *   tlogit[r] = the fp32 logit of targets[r] (0 when the target lies outside [0, V)) from the GEMM's accumulators.
 * eb_lm_ce_rows (fp32 mode): lse and tlogit of contiguous fp32 logit rows [M, V] (expf / logf, fixed order).
 * eb_lm_ce_loss: cost[r] = lse[r] - tlogit[r], 0 where targets[r] == ignore_index, NaN where the target is neither
 *   ignore_index nor in [0, V) (never used as an index); cost may be NULL.  loss[0] = sum of the costs (mean = 0) or
 *   that sum over the count of non-ignored targets (mean = 1: NaN when every target is ignored), and scale[0] = 1 or
 *   1 / count, the factor of eb_lm_ce_bwd.  One CTA sums in a fixed order: bitwise repeatable, no atomics.
 * eb_lm_ce_bwd: grad[r, k] = g[r or 0] * scale[0] * (exp(logits[r, k] - lse[r]) - [k == targets[r]]) (scale NULL: 1,
 *   g [M] when g_per_row else [1], both device fp32), 0 on ignored rows, NaN on rows with an out-of-range target.
 *   logits and grad both bf16 (bf16 = 1) or both fp32; grad may alias logits (in place).
 * No host synchronisation. */
int eb_lm_logits_ce(const void* hidden16, const void* w16, const float* b, void* logits16, const void* targets,
                    int targets_int64, float* lse, float* tlogit, long M, int V, int K, void* stream);
int eb_lm_ce_rows(const float* logits, const void* targets, int targets_int64, float* lse, float* tlogit, long M, int V,
                  void* stream);
int eb_lm_ce_loss(const float* lse, const float* tlogit, const void* targets, int targets_int64, long ignore_index,
                  long M, int V, int mean, float* cost, float* loss, float* scale, void* stream);
int eb_lm_ce_bwd(const void* logits, void* grad, int bf16, const float* lse, const void* targets, int targets_int64,
                 long ignore_index, long M, int V, const float* g, int g_per_row, const float* scale, void* stream);

/* ---- LSTM layer, recurrent part (persistent kernel) ---------------------------------------
 * replaces the time loop of nn.LSTM (rnnt/models.py:45-46,64-65,145-147,154-155).
 * xg [B,T,4H] = W_ih x + b_ih + b_hh (gate order i|f|g|o); whh [4H,H]; h0/c0 may be NULL (zeros).
 * gates_save [B,T,4H] / cseq_save [B,T,H] may be NULL for inference.  scratch: zero-size-checked
 * by eb_lstm_scratch_bytes(B,H). */
size_t eb_lstm_scratch_bytes(int B, int H);
int eb_lstm_seq_fwd(const float* xg, const float* whh, const float* h0, const float* c0, float* y,
                    float* hT, float* cT, float* gates_save, float* cseq_save, void* scratch, int B,
                    int T, int H, void* stream);
/* BPTT: dgates [B,T,4H] (may alias gates) = d loss / d gate pre-activations; dh0/dc0 [B,H] out. */
int eb_lstm_seq_bwd(const float* dy, const float* gates, const float* cseq, const float* c0,
                    const float* whh, const float* dhT, const float* dcT, float* dgates, float* dh0,
                    float* dc0, void* scratch, int B, int T, int H, void* stream);

/* ---- GRU layer, recurrent part (persistent kernel, fp32) ------------------------------------
 * replaces the time loop of nn.GRU (rnnt/models.py:77-116, ResLayerNormGRU), gate order r|z|n:
 *   r = s(xg_r + W_hr h), z = s(xg_z + W_hz h), n = tanh(xg_n + r (W_hn h + b_hn)), h' = (1-z) n + z h.
 * xg [B,T,3H] = W_ih x + b_ih + (b_hr | b_hz | 0); whh [3H,H]; bhn [H] (NULL: zero); h0 may be NULL (zeros).
 * save [B,T,4H] = r | z | n | gh_n (gh_n = W_hn h + b_hn), may be NULL for inference.
 * scratch: eb_gru_scratch_bytes(B,H) bytes, 16-byte aligned (0: H not supported). */
size_t eb_gru_scratch_bytes(int B, int H);
int eb_gru_seq_fwd(const float* xg, const float* whh, const float* bhn, const float* h0, float* y, float* hT,
                   float* save, void* scratch, int B, int T, int H, void* stream);
/* BPTT: y [B,T,H] the forward output (h_{t-1} of step t is y[:, t-1], h0 at t = 0), dhT may be NULL.
 * dgi [B,T,3H] = [dr, dz, dn] (input side: dx, dW_ih, db_ih), dgh [B,T,3H] = [dr, dz, r dn] (recurrent side:
 * dW_hh, db_hh), dh0 [B,H] = d loss / d h0. */
int eb_gru_seq_bwd(const float* dy, const float* save, const float* y, const float* h0, const float* whh,
                   const float* dhT, float* dgi, float* dgh, float* dh0, void* scratch, int B, int T, int H,
                   void* stream);

/* ---- GRU layer on tensor cores (bf16 mode; H % 64 == 0, H <= 1024) ----------------------------
 * same contract as eb_gru_seq_fwd/bwd with bf16 recurrent operands (fp32 accumulation, fp32 state): whh16 [3H,H] bf16,
 * whhT16 [H,3H] bf16 (= W_hh^T), both 4-byte aligned; dgi16 / dgh16 [B,T,3H] bf16 out.  scratch:
 * eb_gru_tc_scratch_bytes(B,H) bytes, 16-byte aligned. */
int eb_gru_tc_supported(int B, int H);
size_t eb_gru_tc_scratch_bytes(int B, int H);
int eb_gru_tc_fwd(const float* xg, const void* whh16, const float* bhn, const float* h0, float* y, float* hT,
                  float* save, void* scratch, int B, int T, int H, void* stream);
int eb_gru_tc_bwd(const float* dy, const float* save, const float* y, const float* h0, const void* whhT16,
                  const float* dhT, void* dgi16, void* dgh16, float* dh0, void* scratch, int B, int T, int H,
                  void* stream);

/* ---- LSTM layer on tensor cores (bf16 mode; H % 64 == 0, H <= 1024) ---------------------------
 * same contract as eb_lstm_seq_fwd/bwd with bf16 recurrent operands (fp32 accumulation, fp32 cell
 * state): whh16 [4H,H] bf16, whhT16 [H,4H] bf16 (= W_hh^T), y16 optional bf16 copy of y, dg16
 * [B,T,4H] bf16 gate-preactivation gradients. */
int eb_lstm_tc_supported(int B, int H);
size_t eb_lstm_tc_scratch_bytes(int B, int H);
int eb_lstm_tc_set_trace(void* dev_buf, int steps);     /* debug: per-stage clock64 stamps of CTA 0 of the BPTT kernel */
int eb_lstm_tc_max_clusters(int H, int cluster_size);   /* co-resident clusters of the BPTT kernel (diagnostic) */
int eb_lstm_tc_fwd(const float* xg, const void* whh16, const float* h0, const float* c0, float* y, void* y16,
                   float* hT, float* cT, float* gates_save, float* cseq_save, void* scratch, int B, int T,
                   int H, void* stream);
int eb_lstm_tc_bwd(const float* dy, const float* gates, const float* cseq, const float* c0,
                   const void* whhT16, const float* dhT, const float* dcT, void* dg16, float* dh0, float* dc0,
                   void* scratch, int B, int T, int H, void* stream);
/* eb_lstm_tc_bwd over a time axis stored chunk-major (functional.LSTMStack's wavefront buffers): chunk c is a contiguous
 * [B, chunk_lens[c], D] block, the blocks follow each other; one launch walks all chunks (T = sum of chunk_lens,
 * nchunks <= 8, chunk_lens a HOST array) instead of one launch per chunk with the (dh, dc) carry through memory. */
int eb_lstm_tc_bwd_chunks(const float* dy, const float* gates, const float* cseq, const float* c0,
                          const void* whhT16, const float* dhT, const float* dcT, void* dg16, float* dh0, float* dc0,
                          void* scratch, int B, const int* chunk_lens, int nchunks, int H, void* stream);

/* ---- LSTM layer on wgmma tensor cores inside thread-block clusters (bf16 mode; H % 256 == 0, H <= 1024) ------
 * csrc/lstm_c4.cu: W_hh slices resident in shared memory, h / dG exchanged through L2 with TMA pulls, partial gate
 * sums reduced across a cluster through distributed shared memory.  Same cell semantics as eb_lstm_tc_* with a
 * CTA-private layout of the forward saves:
 *   gsave: post-activation gates in bf16, csave: cell states in fp32, sizes from eb_lstm_c4_{g,c}save_bytes;
 *   hprev16 [B,T,H] bf16 = h_{t-1} for every step (frame 0 = h0): the operand of the dW_hh GEMM (optional).
 * eb_lstm_c4_supported also checks that all clusters of a launch are co-resident (cooperative cluster launch). */
int eb_lstm_c4_supported(int B, int H);
int eb_lstm_c4_max_clusters(int H, int which);        /* diagnostic: co-resident clusters (0 fwd, 4 / 8 / 16 bwd) */
int eb_lstm_c4_bwd_cluster(int H);                      /* cluster size the BPTT kernel uses (8 / 4), 0 = cannot run */
int eb_lstm_c4_set_trace(void* dev_buf, int steps);     /* debug: per-stage clock64 stamps of CTA 0 ([steps][16] int64) */
size_t eb_lstm_c4_scratch_bytes(int B, int H);
size_t eb_lstm_c4_gsave_bytes(int B, int T, int H);
size_t eb_lstm_c4_csave_bytes(int B, int T, int H);
int eb_lstm_c4_fwd(const float* xg, const void* whh16, const float* h0, const float* c0, float* y, void* hprev16,
                   float* hT, float* cT, void* gsave, void* csave, float* gates_std, float* cseq_std, void* scratch,
                   int B, int T, int H, void* stream);   /* gates_std / cseq_std: optional saves in eb_lstm_tc_bwd's layout */
int eb_lstm_c4_bwd(const float* dy, const void* gsave, const void* csave, const float* c0, const void* whhT16,
                   const float* dhT, const float* dcT, void* dg16, float* dh0, float* dc0, void* scratch, int B,
                   int T, int H, void* stream);
/* eb_lstm_tc_bwd_chunks on the wgmma kernel: same arguments and fp32 standard-layout saves (eb_lstm_c4_fwd's gates_std /
 * cseq_std), scratch sized by eb_lstm_c4_scratch_bytes.  The contraction is split over clusters of 16 CTAs (non-portable
 * cluster size); it runs when eb_lstm_c4_bwd_chunks_cluster(H) == 16 (all H/128 clusters co-resident), else returns
 * EB_ERR_INVALID.  Only the summation order of dh = W_hh^T dG differs from eb_lstm_tc_bwd_chunks. */
int eb_lstm_c4_bwd_chunks_cluster(int H);
int eb_lstm_c4_bwd_chunks(const float* dy, const float* gates, const float* cseq, const float* c0,
                          const void* whhT16, const float* dhT, const float* dcT, void* dg16, float* dh0, float* dc0,
                          void* scratch, int B, const int* chunk_lens, int nchunks, int H, void* stream);
/* ---- LayerNorm(x + res) fwd/bwd, TimeReduction, Embedding -------------------------------
 * rnnt/models.py:47,66-69,124 ; :21-29 ; :150-153.  *_bf16 outputs are optional side copies.
 * LayerNorm: rows > 0 and 0 < H <= 2048.  Time reduction and embedding: negative sizes are EB_ERR_INVALID, an empty
 * output is a no-op, and ids may be NULL when U == 0 (the BOS-only priming input). */
int eb_layernorm_fwd(const float* x, const float* res, const float* gamma, const float* beta, float* y,
                     void* y_bf16, float* mean, float* rstd, long rows, int H, float eps, void* stream);
int eb_layernorm_bwd(const float* dy, const float* x, const float* res, const float* gamma,
                     const float* mean, const float* rstd, float* dz, float* dgamma_accum,
                     float* dbeta_accum, long rows, int H, void* stream);
/* the two passes of eb_layernorm_bwd apart: dz (rows independent) and the parameter gradients (fixed order over rows) */
int eb_layernorm_bwd_dz(const float* dy, const float* x, const float* res, const float* gamma, const float* mean,
                        const float* rstd, float* dz, long rows, int H, void* stream);
int eb_layernorm_bwd_params(const float* dy, const float* x, const float* res, const float* mean, const float* rstd,
                            float* dgamma_accum, float* dbeta_accum, long rows, int H, void* stream);
int eb_time_reduce_fwd(const float* x, float* y, void* y_bf16, int B, int T, int H, void* stream);
int eb_time_reduce_bwd(const float* dy, float* dx, int B, int T, int H, void* stream);
int eb_embedding_fwd(const void* ids, int ids_are_int64, const float* W, float* out, void* out_bf16,
                     int B, int U, int E, int prepend_bos, int bos, void* stream);
int eb_embedding_bwd(const void* ids, int ids_are_int64, const float* dout, float* dW_accum, int B,
                     int U, int E, int prepend_bos, int bos, int pad, void* stream);

/* ---- Joint network pieces (rnnt/models.py:169-179) --------------------------------------
 * hidden[b,t,u,:] = tanh(ep[b,t,:] + dp[b,u,:]) with ep = W1e*h_enc + b1, dp = W1d*h_dec.
 * bf16 (hidden_bf16 / is_bf16 = 1, tanh.approx): J % 8 == 0 and every pointer 16-byte aligned, else EB_ERR_INVALID.
 * In the bf16 backward ddp sums the stored (bf16-rounded) dpre over t, while dep sums the unrounded fp32 products
 * dh * (1 - h^2) over u: the two reductions do not see the same addends. */
int eb_joint_hidden_fwd(const float* ep, const float* dp, void* hidden, int hidden_bf16, int B, int T,
                        int U, int J, void* stream);
int eb_joint_hidden_bwd(void* dhidden_inout, const void* hidden, int is_bf16, float* dep, float* ddp,
                        int B, int T, int U, int J, void* stream);
/* the same two reductions when d(pre-activation) [B,T,U,J] bf16 is already available (eb_gemm_bf16_dtanh);
 * J % 8 == 0 and dpre16, dep, ddp 16-byte aligned, else EB_ERR_INVALID */
int eb_joint_dpre_reduce(const void* dpre16, float* dep, float* ddp, int B, int T, int U, int J, void* stream);

/* ---- pruned RNN-T loss (Kuang et al., Interspeech 2022) ----------------------------------------
 * Lengths as the RNN-T loss above: utterance b has T_b = min(max(xlen[b], 0), maxT) frames and U_b = min(max(ylen[b],
 * 0), maxU-1) + 1 symbol positions; 1 <= maxU <= 1024.  R is the prune range, 2 <= R <= 64, and Rb = min(R, U_b).
 * Every entry below returns EB_ERR_INVALID before any launch for R outside [2, 64], maxU > 1024, a missing pointer or a
 * misaligned bf16 pointer, and none synchronises with the host.
 *
 * Trivial-joiner ("simple") loss on am [B, maxT, V] and lm [B, maxU, V] fp32:
 *   N(t,u) = log sum_v exp(am[t,v] + lm[u,v]),  lpb = am[t,blank] + lm[u,blank] - N,  lpl = am[t,y_u] + lm[u,y_u] - N.
 * eb_rnnt_simple_stats writes denom = -N, lpb and lpl of a dtype_size-4 loss workspace (eb_rnnt_workspace_bytes) for
 * the valid cells; eb_rnnt_loss_lattice on that workspace then gives alpha, beta and the costs.  N is taken in product
 * form, amax[t] + lmax[u] + log(exp(am - amax) . exp(lm - lmax)^T) with one fp32 GEMM per utterance, and a cell whose
 * product is below 1e-25 (where terms lost to underflow could matter) is recomputed by a direct log-sum-exp over v in
 * ascending order, so a finite N never comes out +-inf.  scratch: eb_rnnt_simple_scratch_bytes, filled by
 * eb_rnnt_simple_stats and read by eb_rnnt_simple_bwd.  eb_rnnt_simple_bwd, from that workspace (need_beta = 1), writes
 * with occ = exp(alpha + beta - ll), gamma_blank(t,u) = exp(alpha + lpb + beta(t+1,u) - ll) (alpha + lpb - ll at the
 * final cell) and gamma_emit(t,u) = exp(alpha + lpl + beta(t,u+1) - ll):
 *   dam[t,v] = sum_u occ * softmax_v(am[t] + lm[u]) - sum_u [v = y_u] gamma_emit - [v = blank] sum_u gamma_blank,
 *   dlm[u,v] = the same summed over t,
 * times host_scale * gscale ([1] or [B] with gscale_per_batch, or NULL for 1); zero for t >= T_b, u >= U_b and T_b = 0.
 * The occupancy terms are exp(am - amax) * (G . exp(lm - lmax)) and exp(lm - lmax) * (G^T . exp(am - amax)) with
 * G(t,u) = occ exp(amax + lmax - N), two fp32 GEMMs per utterance; the fallback cells' terms are added directly.  Fixed
 * order, no atomics: the same bits on every run. */
size_t eb_rnnt_simple_scratch_bytes(int B, int maxT, int maxU, int V);
int eb_rnnt_simple_stats(const float* am, const float* lm, const int* labels, const int* xlen, const int* ylen, int B,
                         int maxT, int maxU, int V, int blank, void* scratch, void* workspace, void* stream);
int eb_rnnt_simple_bwd(const float* am, const float* lm, const int* labels, const int* xlen, const int* ylen, int B,
                       int maxT, int maxU, int V, int blank, void* scratch, const void* workspace,
                       const float* gscale_dev, int gscale_per_batch, double host_scale, float* dam, float* dlm,
                       void* stream);
/* Band choice from the simple loss's workspace (alpha, beta, ll_fwd), per utterance:
 *   1. score(t,s) = sum_{u=s}^{s+Rb-1} occ(t,u) in ascending u in fp32, s in [0, U_b - Rb]; s*(t) = its argmax, ties to
 *      the lowest s;
 *   2. s[0] = 0, s[t] = min(max(s*(t), s[t-1]), s[t-1] + Rb - 1);
 *   3. s[T_b-1] = U_b - Rb, then s[t] = max(s[t], s[t+1] - (Rb - 1)) for t = T_b-2 down to 0;
 *   4. nopath[b] = s[0] > 0 (the bands hold no path: U_b - Rb > (T_b - 1)(Rb - 1));
 *   5. s_begin[b, t] = s[t] for t < T_b, 0 for t >= T_b.
 * s_begin [B, maxT] int32, nopath [B] int32; maxT <= 12288. */
int eb_rnnt_band_choice(const int* xlen, const int* ylen, int B, int maxT, int maxU, int R, const void* workspace,
                        int* s_begin, int* nopath, void* stream);
/* Band rows m = (b*maxT + t)*R + r, r < R: row m is cell (t, u = s_begin[b,t] + r) when t < T_b, r < Rb, s_begin[b,t]
 * >= 0 and u < U_b (and, for the loss entries, nopath[b] = 0), else a padding row.  So every row of a frame with a
 * negative start is padding, and so is each row past U_b; eb_rnnt_band_choice only writes starts in [0, U_b - Rb].
 * eb_joint_band_hidden_fwd: hidden[m, :] = tanh(ep[b,t,:] + dp[b,u,:]) ([B*maxT*R, J]; ep [B, maxT, J], dp [B, maxU,
 *   J] fp32), fp32 with tanhf, or bf16 with tanh.approx (hidden_bf16 = 1, hidden 16-byte aligned); padding rows zero.
 * eb_rnnt_band_loss_fwd: the statistics of each valid band row of logits [B*maxT*R, V] fp32 (the same per-row
 *   arithmetic as eb_rnnt_loss_fwd, so a row gets the bits its cell would get there) go to cell (t, u) of a full
 *   [B, maxT, maxU] fp32 loss workspace; every other valid cell gets denom = lpb = lpl = -inf (all of them when
 *   nopath[b]), then the lattice of eb_rnnt_loss_lattice runs: costs_dev[b] = -ll (+inf when nopath[b] or T_b = 0).
 * eb_rnnt_band_loss_bwd: d loss / d logits of the band rows, each row eb_rnnt_loss_bwd's gradient of its cell (lambda
 *   = 0), fp32 (grads may alias logits) or bf16 (grads_bf16); zero on padding rows. */
int eb_joint_band_hidden_fwd(const float* ep, const float* dp, const int* xlen, const int* ylen, const int* s_begin,
                             void* hidden, int hidden_bf16, int B, int maxT, int maxU, int R, int J, void* stream);
int eb_rnnt_band_loss_fwd(const float* logits, const int* labels, const int* xlen, const int* ylen,
                          const int* s_begin, const int* nopath, int B, int maxT, int maxU, int R, int V, int blank,
                          void* workspace, float* costs_dev, int need_beta, void* stream);
/* eb_rnnt_band_lattice: the -inf fill and the lattice of eb_rnnt_band_loss_fwd alone, for band statistics that
 *   eb_joint_band_logits_lse wrote.  Run it after them: it also clears the band cells of an utterance with nopath[b].
 * eb_joint_band_logits_lse: eb_joint_logits_lse's GEMM and statistics epilogue over the band rows of hidden16
 *   [B*maxT*R, J] (bf16 mode): bf16 logits16 [B*maxT*R, V] and the statistics of each valid band row at its cell, the
 *   bits eb_joint_logits_lse gives the same row (J % 8 == 0, 16-byte aligned hidden16 / w2_16 / b2).
 * eb_rnnt_band_loss_bwd_bf16_db: eb_rnnt_loss_bwd_bf16_db (lambda = 0) over the band rows, in place allowed: bf16 d
 *   logits with the row scalars of the band row's cell, zero on padding rows, and db_accum[c] += their column sum in
 *   eb_colsum's order (V % 8 == 0, 16-byte aligned pointers; db_part: fp32 scratch of 512 * V).
 * Every band entry follows the padding rule above; a valid cell that no live row holds gets -inf statistics. */
int eb_rnnt_band_lattice(const int* xlen, const int* ylen, const int* s_begin, const int* nopath, int B, int maxT,
                         int maxU, int R, void* workspace, float* costs_dev, int need_beta, void* stream);
int eb_joint_band_logits_lse(const void* hidden16, const void* w2_16, const float* b2, void* logits16,
                             const int* labels, const int* xlen, const int* ylen, const int* s_begin, float* denom,
                             float* lpb, float* lpl, int B, int maxT, int maxU, int R, int V, int J, int blank,
                             void* stream);
int eb_rnnt_band_loss_bwd_bf16_db(const void* logits16, void* grads16, const int* labels, const int* xlen,
                                  const int* ylen, const int* s_begin, const int* nopath, int B, int maxT, int maxU,
                                  int R, int V, int blank, void* workspace, const float* gscale_dev,
                                  int gscale_per_batch, double host_scale, float* db_part, float* db_accum,
                                  void* stream);
int eb_rnnt_band_loss_bwd(const float* logits, void* grads, int grads_bf16, const int* labels, const int* xlen,
                          const int* ylen, const int* s_begin, const int* nopath, int B, int maxT, int maxU, int R,
                          int V, int blank, void* workspace, const float* gscale_dev, int gscale_per_batch,
                          double host_scale, void* stream);
/* Banded d-pre reduction: dpre = dx * (1 - hidden^2) for fp32 d hidden dx (is_bf16 = 0), or dx itself, the bf16
 * d(pre-activation) of eb_gemm_bf16_dtanh (is_bf16 = 1, hidden NULL, dx 16-byte aligned), over band rows as above:
 *   dep[b,t,:] = sum_{r < Rb} dpre[m(b,t,r), :] in ascending r (zero for t >= T_b),
 *   ddp[b,u,:] = sum over the t < T_b with s_begin[t] <= u < s_begin[t] + Rb, in ascending t, of dpre[m(b,t,u -
 *                s_begin[t]), :] (zero for u >= U_b),
 * each over the live rows only (padding rows are skipped, whatever dx holds there).  Precondition: s_begin[b, t] is
 * non-decreasing over t < T_b (as eb_rnnt_band_choice writes it), so those t are a contiguous range found by binary
 * search: one thread sums each output, no atomics.  It is not checked (that would need a device sync). */
int eb_joint_band_dpre_reduce(const void* dx, const float* hidden, int is_bf16, const int* xlen, const int* ylen,
                              const int* s_begin, float* dep, float* ddp, int B, int maxT, int maxU, int R, int J,
                              void* stream);

/* ---- streaming greedy decode: one persistent kernel per audio chunk -----------------------------
 * replaces PytorchStreamDecoder.decode's Python loop (rnnt/stream.py:93-120).  The host builds a
 * phase program once (edgedict_b200/stream_engine.py) and launches it per chunk; see decode.cu. */
enum { EB_PH_LN = 0, EB_PH_PAIR = 1, EB_PH_LSTM = 2, EB_PH_LINEAR = 3, EB_PH_ARGMAX = 4, EB_PH_COPY = 5,
       EB_PH_BEAM_SELECT = 6, EB_PH_GATHER = 7, EB_PH_BEAM_FINAL = 8, EB_PH_BEAM_COMMIT = 9, EB_PH_SKIP = 10,
       EB_PH_CTC_BEAM = 11, EB_PH_GRU = 12, EB_PH_CTC_EMIT = 13, EB_PH_FE_FRAME = 14, EB_PH_FE_GEMM = 15,
       EB_PH_FE_POWER = 16, EB_PH_FE_LOG = 17, EB_PH_FE_FINISH = 18 };
/* The backoff tables of a token n-gram model (flag 4096; edgedict_b200/ngram.py builds them from an ARPA file), the
 * n-gram state of every slot [B*W] in two parities beside the token sequences, and a row workspace: the CTA that owns
 * an utterance builds there, per frame (or round), g(state(q), k) for all N tokens of each slot q it scores. */
typedef struct EbNgram {
    const float* unigram;     /* [N]: ln P(k), the <unk> fill applied */
    const float* bo;          /* [n_states]: backoff weight */
    const int32_t* suffix;    /* [n_states]: longest proper suffix that is a state (the root, 0, for itself) */
    const int32_t* depth;     /* [n_states]: suffix links to the root (at most 7) */
    const int32_t* first;     /* [n_states]: first child */
    const int32_t* count;     /* [n_states]: number of children */
    const int32_t* tok;       /* [n_children]: token, ascending within a state */
    const float* prob;        /* [n_children]: g(state, tok) */
    const int32_t* next;      /* [n_children]: the state after tok */
    const float* end;         /* [n_states]: e(state) = g(state, </s>), or NULL without </s> */
    int32_t* state[2];        /* per-slot state, parity 0 / 1 */
    float* row;               /* [B*W, N] workspace */
    float weight;             /* ngram_weight */
    int32_t pad_;
} EbNgram;
/* The phrase automaton of contextual biasing (flag 2048; edgedict_b200/context.py builds it): dense tables over
 * n_states states and the N tokens of the phase, and the automaton state of every slot [B*W] in two parities, beside
 * the token sequences. */
typedef struct EbContext {
    const int32_t* next;      /* [n_states, N]: the state after a non-blank token */
    const float* delta;       /* [n_states, N]: the increment a non-blank token adds to a candidate's value */
    const float* pending;     /* [n_states]: boost * the state's length, what BEAM_FINAL takes back */
    int32_t* state[2];        /* per-slot state, parity 0 / 1 */
    const EbNgram* ng;        /* the n-gram model under flag 4096 (the fields above unused without flag 2048) */
} EbContext;
typedef struct EbPhase {
    int32_t type, S, K1, K2, N, flags, ldx1, ldx2, ldw1, ldw2, ldy, aux, aux2, hist_ld, hist_col, x1_div;
    const float *x1, *x2, *w1, *w2, *b1, *b2;
    float *y, *y2, *c;
    const int32_t* tok_in;
    int32_t* tok_out;
    int32_t* hist;
    const int32_t* seq_in;
    int32_t *seq_out, *src;
    const float* fuse;
    const int32_t* tok_map;
    int32_t* tok_out2;
    const EbContext* ctx;
} EbPhase;
/* flags: 1 = tanh epilogue (LINEAR); 2 = x1 rows are embedding rows indexed by tok_in, a negative token reading as a
 *            zero row (LSTM);
 *        4 = masked update: streams whose tok_in equals aux (blank, or -1 for a language model) keep their state (LSTM);
 *        8 = ARGMAX also accumulates log_softmax(x)[argmax] into y[s] (batched greedy decode);
 *       16 = BEAM_SELECT folds hypotheses with equal token sequences (log-add);
 *       32 = BEAM_SELECT fuses a language model into the candidate values (shallow fusion): x2 [B*W, K2] (ldx2) holds
 *            the LM logits of each slot, fuse = {lm_weight, length_bonus} on the device, tok_map [N] maps a token to
 *            its LM token (-1: not scored by the LM), and tok_out2 [B*W] receives each new slot's LM token (-1 when the
 *            LM does not step: blank, unmapped, empty slot or frozen utterance).
 *       64 = BEAM_SELECT streams: the beam carries over from the previous launch (live count at t = 0 read from the
 *            last history column, hist_live[b, hist_ld - 1]) and the token-sequence rows have stride K1 (max_pending + 3)
 *            and hold only the tokens since the stream's last commit (length = that count; the hash still covers the
 *            whole sequence).  The offline beam search does not set it.  CTC_BEAM streams with the same flag (rows of
 *            stride K1 = max_pending + 5, hashes and parent hashes of the whole prefix) and reads y2 as int32 [S], each
 *            stream's last committed token (-1 before any), the last token of a slot whose stored suffix is empty.
 *      128 = BEAM_COMMIT collapses every stream's beam to its best slot unconditionally (a flush).
 *      256 = ARGMAX continuation (round j >= 1 of a multi-symbol greedy frame): a row whose tok_out already holds aux
 *            (blank: its frame ended) writes blank to its hist column, takes no argmax and adds nothing under flag 8;
 *            the other rows run the plain ARGMAX, <unk> rule included.
 *      512 = BEAM_SELECT runs round j of several per frame (beam search with max_symbols K = ldw2 > 1): hist_col =
 *            t*K + j over hist_ld = T'*K columns; a slot whose previous round's tok_out is blank is closed and has one
 *            candidate, its stay (value log p, flat index slot*N + blank); a non-blank token at j = K-1 closes; only
 *            hypotheses of equal closedness merge; the live count lives in the last history column; a row with no open
 *            slot (or frozen) keeps its beam and writes no history.
 *     2048 = contextual biasing (BEAM_SELECT, CTC_BEAM, BEAM_FINAL, BEAM_COMMIT): ctx points to an EbContext.  A
 *            candidate that
 *            appends a non-blank token k to slot q adds delta[state(q), k] to its value (BEAM_SELECT: inside the fusion
 *            term f, for k != blank; CTC_BEAM: to the extension's f'), and each survivor's state (next[state(q), k], or
 *            state(q) for blank, a stay or a frozen frame) is written to the other parity: BEAM_SELECT reads parity
 *            t & 1 (parity 0 under flag 512), CTC_BEAM parity t & 1, as their sequence rows.  BEAM_FINAL ranks and writes
 *            y - pending[state] with the state from parity hist_col.  BEAM_COMMIT reads the states from parity 1,
 *            collapses to the live slot of highest y - pending[state] (lowest slot on ties; it keeps its y and state)
 *            and writes every slot's state, moved by src, to parity 0.
 *     4096 = n-gram shallow fusion (BEAM_SELECT, CTC_BEAM, BEAM_FINAL): ctx->ng points to an EbNgram and fuse[1] holds the
 *            length bonus even without flag 32.  A candidate that appends a non-blank token k to slot q adds w*g(state(q),
 *            k), unfused by __fmul_rn / __fadd_rn, right after the LM term (BEAM_SELECT: f = f0 + w*g, f0 the LM term or
 *            the length bonus, then + delta under 2048; CTC_BEAM: f' = ((f + f0) + w*g) + delta), and each survivor's
 *            state is written to the other parity exactly where the context state is.  BEAM_FINAL ranks and writes
 *            (y + w*e(state)) - pending, the state from parity hist_col (no w*e term when end is NULL).
 * SKIP (no flags, writes nothing, no grid barrier): when no row of tok_in[0..S) differs from aux2 (blank), every CTA
 * jumps over the next aux phases.  It reads only data final at the preceding barrier, so all CTAs take the same branch.
 * BEAM_COMMIT (streaming beam, after a chunk's last frame, one CTA per stream): commits the common prefix of the live
 * slots' stored suffixes to tok_out [S, N] with the count in tok_out2[s] (tok_out2[S + s] = 1 when the beam collapsed),
 * shifts the suffixes left into seq_out, and, when a suffix still exceeds aux2 tokens or on flags 128, collapses the beam
 * to its best slot by y; src receives the gather sources that move the kept slots' state into place.  K2 is the rows'
 * head before their tokens (0 for BEAM_SELECT's 3, 5 for CTC_BEAM's); y2, when set, int32 [S], receives each stream's
 * last committed token whenever it commits any.
 *     1024 = GATHER runs a front-end program instead of gathering: the K1 phases at x1 (an EbPhase array), each closed
 *            by a grid barrier on the counter tok_out, which the decode entries zero at every launch (barrier_dev holds
 *            two counters, 8 bytes).  Its phases are FE_* only; they compute a chunk's features from raw audio:
 *   FE_FRAME  S streams of N samples x1 (x2: optional dither noise [S, N]; fuse = {dither, preemph} on the device) ->
 *             y [S, ldy]: fl(x + fl(dither * noise)), pre-emphasised with flags 1, reflect-padded by K1 samples, zeros
 *             after;
 *   FE_GEMM   y [S, N] (ldy) = A [S, K1] B [K1, N] with A(m, k) = x1[(m / aux) ldx1 + (m % aux) ldx2 + k] and
 *             B(k, n) = w1[k ldw1 + n], each output eb_gemm_f32's k-ascending fmaf chain from 0;
 *   FE_POWER  y [S, N] = re^2 + im^2 of x1 rows [S, 2N] = [re | im];
 *   FE_LOG    y [S*N] = log(x1 + 1e-6);
 *   FE_FINISH x1 [S*K1, N] per-frame rows of S streams -> y [S, aux2, W] (W = N (3 with flags 2) aux): aux frames
 *             stacked per row, log(x + 1e-20) with flags 1, deltas with flags 2; hist_ld = frames F, hist_col = frames
 *             kept Fs, x1_div = the first masked frame.
 *            Each value is frontend.cu's expression for it, so the features equal eb_fe_* / eb_gemm_f32's bit for bit.
 * x1_div (LINEAR): row r of x1 is x1[r / x1_div] (0 or 1: row r), the encoder frame a beam's W rows share.
 * Beam search (batched, W slots per utterance, row r = b*W + slot; see decode.cu for the field use of each phase):
 * at most EB_BEAM_MAX_W slots per utterance.  BEAM_FINAL writes the K1 = N best live slots of each utterance (0 reads
 * as 1: the best one alone), ranked by value descending, lowest slot on ties: ids [B*N][ldy] in tok_out, -value [B*N] in
 * y2, and, when set, each token's frame (history column / ldw2, 0 read as 1) in seq_out and min(N, live) [B] in
 * tok_out2.  Ranks past the count hold ids and frames -1 and +inf.
 * CTC_BEAM (CTC prefix beam search over log-probs, one CTA per utterance; see decode.cu for the field use): frames
 * hist_col .. hist_col + ldw1 - 1 in one phase; each slot carries log P(prefix, ends in blank / non-blank) and a fusion
 * term in an engine-owned state buffer (c), an extension that reaches another live slot's prefix is log-added into that
 * slot's stay before the ranking, the history is BEAM_SELECT's (a stay recorded as blank) and BEAM_FINAL reads it.
 * Programs with CTC_BEAM run through eb_decode_run_ctc. */
#define EB_BEAM_MAX_W 1024
int eb_decode_phase_size(void);
int eb_decode_run(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream);
/* eb_decode_run with CTC_BEAM phases: the same kernel in an instantiation that also runs CTC_BEAM (eb_decode_run skips
 * them: the extra phase costs the matrix phases register spills, which the other programs do not pay). */
int eb_decode_run_ctc(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream);
/* Streaming CTC (stream_engine.CTCStreamEngine, see decode.cu for the field use):
 * GRU       one nn.GRU cell step for S rows (gate order r|z|n): w1 = W_ih [3N, K1], w2 = W_hh [3N, K2], b1 = b_ih,
 *           b2 = b_hh, h from x2; y (ldy) = h', y2 (optional, [S, N]) a copy.  No flags.
 * CTC_EMIT  greedy CTC emission of a chunk, one warp per stream: S streams of aux frames (logits x1 row s*aux + t), V = N,
 *           blank = aux2; per frame the log-probs y = (x - max) - log(sum exp(x - max)), their argmax in torch.argmax
 *           order (NaN first, ties to the lowest id); a frame equal to the previous frame's argmax (tok_out [S], carried
 *           across launches; negative after a reset) or to blank is dropped; the kept ids go to hist [S, hist_ld] with
 *           their count in tok_out2 [S]; y2, a DOUBLE [S], accumulates the whole-row log-prob sum of every kept frame;
 *           seq_out (optional) [S, aux] receives every frame's argmax.
 * eb_decode_run and eb_decode_run_ctc skip both; programs with them run through eb_decode_run_ctc_stream, the kernel
 * in a third instantiation (the two others keep their code and registers), which skips LSTM and CTC_BEAM. */
int eb_decode_run_ctc_stream(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream);
/* Streaming GRU transducer (stream_engine.GRUStreamEngine / GRUStreamBeamEngine): the kernel in a fourth instantiation,
 * eb_decode_run's plus GRU, so one program holds a GRU encoder, an LSTM predictor and LM, and the greedy and beam frame
 * phases.  It skips CTC_BEAM and CTC_EMIT; the three other instantiations keep their code and registers. */
int eb_decode_run_gru_rnnt(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream);
/* Streaming CTC beam search (stream_engine.CTCStreamBeamEngine): the kernel in a fifth instantiation with GRU, LINEAR,
 * CTC_EMIT, CTC_BEAM (streaming, flag 64), LSTM (the fused LM's step), GATHER, COPY and BEAM_COMMIT.  It skips ARGMAX,
 * BEAM_SELECT and BEAM_FINAL; the four other instantiations keep their code and registers. */
int eb_decode_run_ctc_stream_beam(const void* phases_dev, int nphase, void* barrier_dev, int max_ctas, void* stream);

/* ---- reductions, casts, optimizer -------------------------------------------------------- */
int eb_colsum(const void* x, int x_bf16, float* out_accum, long rows, int N, void* stream);
int eb_cast_bf16(const float* x, void* y, long n, void* stream);
/* eb_transpose_to_bf16: y [cols, rows] = x^T for any rows, cols >= 0 (an empty matrix is a no-op). */
int eb_transpose_to_bf16(const void* x, int x_bf16, void* y, long rows, long cols, void* stream);
int eb_adam_step(float* p, const float* g, float* m, float* v, long n, float lr, float beta1,
                 float beta2, float eps, float weight_decay, int step, float grad_scale, void* stream);
/* Adam / AdamW with gradient clip and loss-scale handling on the device (no host read of the norm):
 * sumsq = device scalar sum(g^2) of the unscaled bucket (eb_sumsq) or NULL; max_norm > 0 clips like
 * torch.nn.utils.clip_grad_norm_ (cli/baseline.py:239-245); a non-finite norm skips the step (loss-scale overflow);
 * adamw = 1 selects the reference's AdamW update (modules/optimizer.py:283-290). */
int eb_adam_step_ex(float* p, const float* g, float* m, float* v, long n, float lr, float beta1, float beta2,
                    float eps, float weight_decay, int step, float grad_scale, const float* sumsq, float max_norm,
                    int adamw, void* stream);
int eb_sumsq(const float* x, long n, float* out_accum, void* stream);

/* ---- the reference trainers' optimizers over the flat buckets (optim.FlatOptimizer), csrc/optim.cu -------------------
 * seg [nseg]: one entry per tensor: bucket offset, numel, rank (<= 4), parameter group, its tiles [tile_begin, tile_end),
 *             shape, and for SM3 the offsets of its accumulators in the accumulator bucket (rank 0 and 1: one).
 * tiles      : contiguous ranges [start, start + len) of one tensor (seg) cut from its own shape: whole rows of its last
 *              dimension (ncols = the last dimension) or one piece of a row; r0 / c0 = the tile's first row / column.
 * h          : the per-group hyperparameters, by value: lr, weight decay, b1 (SGD: momentum), b2, eps.
 * ctl [2]    : written by eb_opt_prologue: ctl[0] = grad_scale x the clip coefficient, ctl[1] != 0: the step is skipped.
 * steps [ngroups]: the device step counters; eb_opt_prologue advances them only when the step is taken.
 * eb_opt_seg_sumsq : partial [ntiles] = per-tile sum g^2, segsum [nseg] = the tiles of each tensor summed in order,
 *                    total (optional) = the tensors summed in order: no float atomics, bitwise repeatable.
 * eb_opt_prologue  : total (optional, the unscaled sum g^2): with it, a non-finite norm skips the step and max_norm > 0
 *                    clips like torch.nn.utils.clip_grad_norm_.
 * eb_opt_sgd_step  : torch.optim.SGD; buf [n] may be NULL when every group's momentum is 0.
 * eb_opt_sm3_step  : SM3 with beta = 0: reads acc [nacc], writes the new accumulators into acc_new [nacc] (zeroed here;
 *                    a skipped step copies acc).  The caller swaps the two.
 * eb_opt_adamw_step: the reference's AdamW; bias corrections from the device step counters.
 * eb_opt_novograd_step: Novograd; segv [nseg] = the per-tensor second moment, segsum from eb_opt_seg_sumsq. */
#define EB_OPT_MAX_GROUPS 16
typedef struct { long long off, numel, rank, group, tile_begin, tile_end, shape[4], acc[4]; } eb_opt_seg;
typedef struct { long long seg, start, len, r0, c0, ncols; } eb_opt_tile;
typedef struct { double lr[EB_OPT_MAX_GROUPS], wd[EB_OPT_MAX_GROUPS], b1[EB_OPT_MAX_GROUPS], b2[EB_OPT_MAX_GROUPS],
                 eps[EB_OPT_MAX_GROUPS]; } eb_opt_hyper;
int eb_opt_seg_sumsq(const float* g, const eb_opt_seg* seg, int nseg, const eb_opt_tile* tiles, int ntiles,
                     float* partial, float* segsum, float* total, void* stream);
int eb_opt_prologue(const float* total, float grad_scale, float max_norm, int ngroups, int* steps, float* ctl,
                    void* stream);
int eb_opt_sgd_step(float* p, const float* g, float* buf, const eb_opt_seg* seg, const eb_opt_tile* tiles, int ntiles,
                    eb_opt_hyper h, int ngroups, const float* ctl, const int* steps, void* stream);
int eb_opt_sm3_step(float* p, const float* g, const float* acc, float* acc_new, long nacc, const eb_opt_seg* seg,
                    const eb_opt_tile* tiles, int ntiles, eb_opt_hyper h, int ngroups, const float* ctl, void* stream);
int eb_opt_adamw_step(float* p, const float* g, float* m, float* v, const eb_opt_seg* seg, const eb_opt_tile* tiles,
                      int ntiles, eb_opt_hyper h, int ngroups, const float* ctl, const int* steps, void* stream);
int eb_opt_novograd_step(float* p, const float* g, float* m, float* segv, const float* segsum, const eb_opt_seg* seg,
                         int nseg, const eb_opt_tile* tiles, int ntiles, eb_opt_hyper h, int ngroups,
                         const float* ctl, void* stream);

/* ---- log-mel front end (the step before the path; SURVEY 8(f) N2) ------------------------------
 * replaces FilterbankFeatures.forward (rnnt/features.py:126-164) + Downsample (rnnt/transforms.py:37-51).
 * eb_fe_preemph_pad : x[B,L] -> xp[B,Lp]: pre-emphasis (features.py:137-141) and the reflect padding of
 *                     torch.stft(center=True) by `pad` = n_fft/2 samples; positions >= L+2*pad are zero.  With Lp a
 *                     multiple of hop, frame g = b*(Lp/hop)+f starts at flat offset g*hop, so the STFT is
 *                     eb_gemm_f32 on a strided view (sam = hop) against the windowed DFT basis [n_fft, 2*nbins].
 * eb_fe_power       : spec[rows, re(nbins) | im(nbins)] -> power[rows, nbins]  (features.py:149)
 * eb_fe_log_stack   : mel[B*rows_per_utt, n_mels] -> out[B, t_out, n_mels*n_stack]: log(x + 1e-20)
 *                     (features.py:155-156), zero for frames >= seq_len (features.py:160-164) and for the
 *                     stacking pad (transforms.py:41-45); out is the [B,T,F] layout Encoder.forward takes. */
int eb_fe_preemph_pad(const float* x, float* xp, int B, int L, long Lp, int pad, float preemph,
                      int use_preemph, void* stream);
int eb_fe_power(const float* spec, float* power, long rows, int nbins, void* stream);
int eb_fe_log_stack(const float* mel, float* out, int B, int rows_per_utt, int n_frames, int seq_len,
                    int n_mels, int n_stack, int t_out, int take_log, void* stream);
/* Per-utterance features of a padded batch (rnnt/transforms.py:165-203 applied to each x[b, :L_b] alone, then
 * rnnt/dataset.py:202-240's zero padding).  Lengths come twice: `lens` on the host, checked before any launch, and
 * `lens_dev`, the same int32 [B] values on the device, read by the kernels.
 * eb_fe_preemph_pad_lens : eb_fe_preemph_pad with row b reflected at its own L_b (x rows stay L apart) and zero from
 *                          L_b + 2*pad on; every L_b must satisfy pad < L_b <= L (torch's reflect pad refuses L_b <= pad).
 * eb_fe_log              : x := log(x + offset) in place (the MFCC's log(mel + 1e-6), torchaudio MFCC log_mels=True).
 * eb_fe_finish           : feat[B*rows_per_utt, n_ch] per-frame rows -> out[B, t_out, n_ch*(delta ? 3 : 1)*n_stack]:
 *                          per utterance the optional log(x + 1e-20), the mask from frame ceil(L_b/hop) on (use_mask),
 *                          CatDeltas' [x, d1, d2] (compute_deltas twice, window 5, replicate edge at F_b - 1 with
 *                          F_b = 1 + L_b/hop), Downsample's stacking of n_stack frames, and zeros from
 *                          T_b = ceil(F_b/n_stack) (floor unless pad_to_divisible) on.  Needs F_b <= rows_per_utt and
 *                          T_b <= t_out.
 * eb_fe_deltas           : CatDeltas on feat [B, n_frames, n_ch] -> out [B, n_frames, 3*n_ch] (eb_fe_finish's arithmetic
 *                          with every utterance n_frames long, no log, no mask, no stacking). */
int eb_fe_preemph_pad_lens(const float* x, const int* lens, const int* lens_dev, float* xp, int B, int L, long Lp,
                           int pad, float preemph, int use_preemph, void* stream);
int eb_fe_log(float* x, long n, float offset, void* stream);
int eb_fe_finish(const float* feat, float* out, const int* lens, const int* lens_dev, int B, int rows_per_utt, int hop,
                 int n_ch, int n_stack, int t_out, int take_log, int use_mask, int delta, int pad_to_divisible,
                 void* stream);
int eb_fe_deltas(const float* feat, float* out, int B, int n_frames, int n_ch, void* stream);
/* SpecAugment masks (rnnt/transforms.py:53-147) in place on x [B, D1, D2]: spans int32 [B, nmask, 2] = [start, end)
 * along axis 1 (frequency) or 2 (time); masked elements := fill. */
int eb_fe_mask(float* x, const int* spans, int B, int D1, int D2, int nmask, int axis, float fill, void* stream);

/* ---- raw-waveform front end: FrontEnd (rnnt/models.py:313-365), csrc/conv.cu ------------------------------------
 * Activations channels-last.  y buffers are [B][rows][C] fp32 with `ustride` elements between utterances, the T valid
 * rows first.  A strided conv (k, s, p = k - 1) over an input of T rows reads a padded operand buffer of Q = ceil((p+T)/s)
 * rows of s*C_in per utterance (p zero rows, the input, zeros) plus ceil(k/s) zero rows of s*C_in at the end; its output
 * row b*Q + t is valid for t < T_out = floor((T + k - 2) / s) + 2 - k.
 * eb_conv_rows_per_split : rows of a [T, C] utterance per partial slice in eb_gn_stats / eb_gn_bwd.  With
 *                          ns = B * ceil(T / rows): the per-channel partials (pg, pb, pdb) have ns slices of C, the fp64
 *                          per-utterance partials (dpart) ns * ceil(C / 256) slices of 2.
 * eb_conv1d_first_fwd    : the first layer (C_in = 1): y[b, t, c] = bias[c] + sum_j w[c, j] x[b, t*s + j - p], T as above.
 * eb_conv1d_first_dw     : part[z][j][c] (j = k: the bias) over rows [z*rows_per_split, ...) of the B*T rows of dy;
 *                          dW, db = the slices summed in order (eb_colsum).
 * eb_gn_stats            : mean / rstd of GELU(y) per utterance over all T x C (GroupNorm(1, C), biased variance, eps),
 *                          fp64 partial sums in dpart [slices][2].
 * eb_gn_apply            : out row r = b*rows_per_utt + u (r < total_rows): (GELU(y[b, u-p]) - mean) rstd gamma + beta
 *                          for p <= u < p + T, else 0; out fp32 or bf16.
 * eb_gn_bwd              : dz (gradient of eb_gn_apply's valid rows, dz_ustride apart) -> pg / pb [slices][C] partials
 *                          of dgamma / dbeta, dy = d y (fp32 and / or bf16, dy_ustride apart), pdb [slices][C] partials
 *                          of sum dy (NULL: none); dpart [slices][2] fp64 scratch.
 * eb_conv1d_bf16         : out[m, n] (row pitch ldc) = bias[n] + sum_{j<taps} sum_c X[m + row0 + j/s][j%s][c] W[n][j*C + c]
 *                          on the tensor cores (TMA + wgmma, fp32 accumulation); X bf16 [x_rows][s][C], W bf16
 *                          [N][taps*C]; rows outside [0, x_rows) read as zeros.  C % 16 == 0, N % 16 == 0. */
int eb_conv_rows_per_split(int C);
int eb_conv1d_first_fwd(const float* x, const float* w, const float* bias, float* y, int B, int L, int C, int k, int s,
                        int T, void* stream);
int eb_conv1d_first_dw(const float* x, const float* dy, float* part, int nsplit, long rows_per_split, int B, int L,
                       int C, int k, int s, int T, void* stream);
int eb_gn_stats(const float* y, long ustride, int B, int T, int C, double* dpart, float* mean, float* rstd, float eps,
                void* stream);
int eb_gn_apply(const float* y, long ustride, int B, int T, int C, const float* mean, const float* rstd,
                const float* gamma, const float* beta, void* out, int out_bf16, int p, long rows_per_utt,
                long total_rows, void* stream);
int eb_gn_bwd(const float* y, long ustride, int B, int T, int C, const float* mean, const float* rstd,
              const float* gamma, const float* dz, long dz_ustride, float* pg, float* pb, double* dpart, float* dy,
              void* dy16, long dy_ustride, float* pdb, void* stream);
int eb_conv1d_bf16(const void* x16, long x_rows, int s, int C, int row0, const void* w16, int taps, int N,
                   const float* bias, float* out, long ldc, long M, void* stream);
/* eb_gemm_f32 (alpha 1, beta 0, no bias) with the contraction split in slices of kchunk: part[z] = [M, N] of slice z */
int eb_gemm_f32_splitk(const float* A, long sam, long sak, const float* B, long sbk, long sbn, float* part, int M,
                       int N, int K, int kchunk, void* stream);

/* ---- wav2vec pre-training head: Wav2Vec / ConstrastiveCriterion (rnnt/wav2vec.py), GumbelVectorQuantizer
 * (modules/softmax_vector_quantizer.py), csrc/w2v.cu.  Masked frames per utterance: idx int32 [B, M] (ascending frame
 * numbers) and inv int32 [B, T] (m of a masked frame, -1 otherwise).  Fixed-order reductions, no float atomics.
 * eb_w2v_mask_fwd    : out[r] = inv[r] >= 0 ? mask_emb : x[r] over rows = B*T rows of D (x[mask] = mask_emb, out of place).
 * eb_w2v_keep_rows   : out[r] = inv[r] >= 0 ? 0 : x[r].
 * eb_w2v_gather      : out[b, m] = x[b, idx[b, m]];  eb_w2v_scatter: out[b, t] = inv[b, t] >= 0 ? x[b, inv[b, t]] : 0.
 * eb_w2v_sq_mean     : out[0] = sum(x^2) / n (one CTA, fixed order).  eb_w2v_scale: out = x * g[0] * alpha (may alias).
 * eb_w2v_quant_fwd   : logits, noise (NULL: eval), p, s, X [N, G*V], vars [G*V, vd], q [N, G*vd], k0, k, st [N*G]:
 *                      k0 = argmax logits, p = softmax(logits), s = softmax((logits + noise) / tau), k = argmax s (first
 *                      on ties), st = (1 - s_k) + s_k (fp32), X = st at k and 0 elsewhere, q[r, g] = st * vars[g*V + k].
 *                      Eval: k = k0, st = 1, q = vars[k0] exactly; s is not written.
 * eb_w2v_quant_stats : psum [G*V] = sum_r p, k0 -> out[0] = prob_perplexity, out[1] = code_perplexity, coef [G*V] =
 *                      d prob_perplexity / d mean_r p; counts int [G*V] scratch.
 * eb_w2v_quant_bwd   : dlogits = (1/tau) s (dsoft - <s, dsoft>) + (g_ppl[0] / N) p (coef - <p, coef>) per (row, group);
 *                      dsoft or g_ppl may be NULL (that term is dropped).
 * eb_w2v_logits_fwd  : xp, yp [B, M, D], neg int32 [B, M, K] (frames of the same utterance) -> xh, yh (rows over
 *                      max(|row|, eps)), xn, yn [B*M] (|row|), cosv and logits [K+1, B, M]: candidate 0 is row m of yp,
 *                      candidate 1 + k row neg[b, m, k]; logits = cos / temp, -inf where a negative equals yp[b, m]
 *                      (cosv is -inf there too: it marks the masked candidates for the backward).
 * eb_w2v_logits_bwd  : dlogits, cosv (the forward's) [K+1, B, M] -> dxp, dyp; A, AC [B, M, M] scratch.  A masked
 *                      candidate (c > 0 with a -inf cosv) passes no gradient, whatever its dlogit.
 * eb_w2v_ce          : logits [C, B, M], rows (m, b) -> grad (softmax - onehot(0)), out[0] = sum of lse - logit 0,
 *                      out[1] = rows whose argmax is 0 and argmin is not (first index on ties). */
int eb_w2v_mask_fwd(const float* x, const float* mask_emb, const int* inv, float* out, long rows, int D, void* stream);
int eb_w2v_keep_rows(const float* x, const int* inv, float* out, long rows, int D, void* stream);
int eb_w2v_gather(const float* x, const int* idx, float* out, int B, int T, int M, int D, void* stream);
int eb_w2v_scatter(const float* x, const int* inv, float* out, int B, int T, int M, int D, void* stream);
int eb_w2v_sq_mean(const float* x, long n, float* out, void* stream);
int eb_w2v_scale(const float* x, const float* g, float alpha, long n, float* out, void* stream);
int eb_w2v_quant_fwd(const float* logits, const float* noise, const float* vars, int N, int G, int V, int vd,
                     float tau, float* q, float* p, float* s, float* X, int* k0, int* k, float* st, void* stream);
int eb_w2v_quant_stats(const float* psum, const int* k0, int N, int G, int V, float* out, float* coef, int* counts,
                       void* stream);
int eb_w2v_quant_bwd(const float* dsoft, const float* s, const float* p, const float* coef, const float* g_ppl, int N,
                     int G, int V, float tau, float* dlogits, void* stream);
int eb_w2v_logits_fwd(const float* xp, const float* yp, const int* neg, int B, int M, int D, int K, float temp,
                      float eps, float* xh, float* yh, float* xn, float* yn, float* cosv, float* logits, void* stream);
int eb_w2v_logits_bwd(const float* dlogits, const float* cosv, const int* neg, const float* xh, const float* yh,
                      const float* xp, const float* yp, const float* xn, const float* yn, int B, int M, int D, int K,
                      float temp, float eps, float* A, float* AC, float* dxp, float* dyp, void* stream);
int eb_w2v_ce(const float* logits, int B, int M, int C, float* grad, float* out, void* stream);

/* Minimum word error rate training (csrc/mwer.cu).
 * eb_edit_distance: Levenshtein distance of n_hyp pairs, one CTA each.  Hypothesis row p is hyp[p*ld_h + k] and
 * reference row r is ref[r*ld_r + k] (int32 ids, left-aligned); meta (device) = hyp_len [n_hyp] | ref_len [n_ref] |
 * ref_index [n_hyp] (pair p compares hypothesis p with reference ref_index[p]) and meta_host the same values in host
 * memory, which are checked and sized before the launch.  out [n_hyp][5] int32 = {errors, substitutions, deletions,
 * insertions, reference length}, all in units.  Units are the ids, or, with word_table [n_table][3] = {char offset,
 * char count, class} and word_chars (code points), words: ids of class EB_WORD_DROP (and ids outside [0, n_table)) are
 * removed, a separator adds no characters, and a word is a maximal run of characters closed by a word end (whose
 * characters it includes), a separator or the end of the row; two words are equal iff their characters are (a hash
 * pre-filters, the comparison is exact).  D[i][j] over the first i reference and j hypothesis units takes the diagonal
 * step on ties, else the deletion D[i-1][j] + 1 if it is not above the insertion D[i][j-1] + 1; S, D and I are carried
 * along the chosen predecessor.  EB_ERR_INVALID before any launch for a missing pointer, a length below 0, above its
 * row or above EB_EDIT_MAX_UNITS, a ref_index outside [0, n_ref), or a word table with n_table < vocab (the ids the
 * rows may hold).
 * eb_nbest_pack: a beam engine's N-best ids [B][N][L] (right-aligned, -1 before the tokens) and count [B], and the
 * references ref [B][ld_ref] of ref_len [B] -> labels [B*(N+1)][ld_out] left-aligned and zero-padded, lens [B*(N+1)]:
 * row b*(N+1)+i is rank i (length 0 at or past count[b]), row b*(N+1)+N the reference; valid [B][N] = i < count[b].
 * ld_out >= max(L, ld_ref).
 * eb_mwer_risk_fwd: costs c [B][N] (-log P(y_i | x)), errors E [B][N], valid [B][N] (nonzero: a hypothesis), N <=
 * EB_BEAM_MAX_W; per utterance in fp64 and rank order P_i = softmax over the valid i of -c_i (0 elsewhere), Ebar = the
 * mean valid E, risk[b] = sum_i P_i (E_i - Ebar); post [B][N] = P (fp32), loss [1] = sum_b risk[b] / B (fp64 sum in
 * utterance order).  eb_mwer_risk_bwd: dcosts [B][N] = -P_i ((E_i - Ebar) - risk[b]) / B * gout[0] from the same fp64
 * values, 0 for invalid ranks: an utterance of one valid rank, or of equal errors, gives exactly 0. */
#define EB_EDIT_MAX_UNITS 4096
#define EB_WORD_INSIDE 0
#define EB_WORD_END 1
#define EB_WORD_SEP 2
#define EB_WORD_DROP 3
size_t eb_edit_distance_smem_bytes(int cap_h, int cap_r, int word);
int eb_edit_distance(const int* hyp, long ld_h, const int* ref, long ld_r, const int* meta, const int* meta_host,
                     int n_hyp, int n_ref, const int* word_table, const int* word_chars, int n_table, int vocab,
                     int* out, void* stream);
int eb_nbest_pack(const int* ids, const int* count, int B, int N, int L, const int* ref, int ld_ref, const int* ref_len,
                  int* labels, int ld_out, int* lens, int* valid, void* stream);
int eb_mwer_risk_fwd(const float* costs, const int* errors, const int* valid, int B, int N, float* post, double* risk,
                     float* loss, void* stream);
int eb_mwer_risk_bwd(const float* costs, const int* errors, const int* valid, int B, int N, const float* gout,
                     float* dcosts, void* stream);

#ifdef __cplusplus
}
#endif
