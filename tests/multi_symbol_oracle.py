"""CPU restatement of greedy decoding with up to K symbols per encoder frame (``max_symbols``), on the pieces of
oracle/model_torch.py.  At K = 1 both functions are oracle.model_torch's own greedy_decode / stream_decode, unchanged.

The rule, per row and encoder frame: round 0 is the one-symbol frame (joint, argmax, predictor step on non-blank);
round j >= 1 runs only when round j-1 emitted a non-blank token.  The frame ends at the first blank or after K non-blank
tokens, in which case the predictor has stepped on the K-th.  log p sums every round taken."""
import torch
import torch.nn.functional as F

from oracle import model_torch as mt


@torch.no_grad()
def greedy_decode(sd, xs, xlen, max_symbols=1, blank=mt.NUL, time_reductions=(1,), fast=False):
    """mt.greedy_decode with K = max_symbols: (id arrays of K entries per frame, blank for rounds not taken, truncated
    to the first xlen frames; -sum log p over all frames)."""
    K = max_symbols
    if K == 1:
        return mt.greedy_decode(sd, xs, xlen, blank, time_reductions, fast)
    h_enc, _ = mt.encoder(sd, xs, None, time_reductions, fast=fast)
    B, T = xs.shape[0], h_enc.shape[1]
    h_dec, (hp, cp) = mt.decoder(sd, torch.zeros(B, 0, dtype=torch.long), None, fast=fast)
    h_dec, hp, cp = h_dec.clone(), hp.clone(), cp.clone()
    seq = torch.full((B, T * K), blank, dtype=torch.long)
    lp = torch.zeros(B, dtype=h_enc.dtype)
    for t in range(T):
        live = torch.ones(B, dtype=torch.bool)
        for j in range(K):
            p, pred = F.log_softmax(mt.joint(sd, h_enc[:, t], h_dec[:, 0]), 1).max(1)
            seq[live, t * K + j] = pred[live]
            lp[live] += p[live]
            live = live & (pred != blank)
            if not live.any():
                break
            nd, (hn, cn) = mt.decoder(sd, pred[:, None], (hp, cp), fast=fast)
            h_dec[live] = nd[live]
            hp[:, live] = hn[:, live]
            cp[:, live] = cn[:, live]
    return [s[:int(n) * K].numpy() for s, n in zip(seq, xlen)], -lp


@torch.no_grad()
def stream_decode(sd, st, chunk, unk_id=mt.UNK, time_reductions=(1,), fast=False, max_symbols=1):
    """mt.stream_decode with K = max_symbols: the emitted (non-blank) ids of one chunk, with the <unk> rule in every
    round."""
    K = max_symbols
    if K == 1:
        return mt.stream_decode(sd, st, chunk, unk_id, time_reductions, fast)
    enc, (st.enc_h, st.enc_c) = mt.encoder(sd, chunk, (st.enc_h, st.enc_c), time_reductions, fast=fast)
    out = []
    for k in range(enc.shape[1]):
        for _ in range(K):
            prob = mt.joint(sd, enc[:, k], st.dec_x[:, 0])
            pred = int(prob.argmax(-1))
            if pred == unk_id:
                prob[:, pred] = 0
                pred = int(prob.argmax(-1))
            if pred == mt.NUL:
                break
            st.dec_x, (st.dec_h, st.dec_c) = mt.decoder(sd, torch.full((1, 1), pred), (st.dec_h, st.dec_c), fast=fast)
            out.append(pred)
    return out
