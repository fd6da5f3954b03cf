"""fp64-capable torch restatement of CTCEncoder (rnnt/models.py:272-310) -- TEST INFRASTRUCTURE.

``sd``: {reference state_dict key -> tensor} of a CTCEncoder (``model.*`` = Encoder with ResLayerNormGRU, ``tovocab.0.*``
= the output Linear).  The encoder is oracle.model_torch.encoder_gru.  Pinned by tests/test_oracle_ctc.py against
tests/golden/ctc_tiny.npz, which the reference's own CTCEncoder produced.
"""
import torch
import torch.nn.functional as F

from . import model_torch as mt

NUL = 0


def ctc_encoder_forward(sd, xs, time_reductions=(1,)):
    """CTCEncoder.forward: xs [B, T, F] -> log-probs [B, T', V] (dtype of sd / xs)."""
    h, _ = mt.encoder_gru(sd, xs, None, time_reductions, pre="model.")
    return F.log_softmax(F.linear(h, sd["tovocab.0.weight"], sd["tovocab.0.bias"]), -1)


def greedy_from_logprobs(logprobs, xlen, blank=NUL):
    """CTCEncoder.greedy_decode after the forward pass, line for line: argmax per frame (torch.max), a frame is kept when
    it is not blank and differs from the previous frame, truncation to xlen[b] frames (not scaled to T'), and the score
    sums the WHOLE log-prob rows of the kept frames.  Returns (list of int64 arrays, -score [B])."""
    _, y_seq = logprobs.max(dim=-1)
    unique = F.pad(y_seq[:, 1:] != y_seq[:, :-1], [1, 0, 0, 0], value=True)
    masks = (y_seq != blank) & unique
    ids, log_p = [], []
    for seq, lp, n, mask in zip(y_seq, logprobs, xlen, masks):
        n = int(n)
        mask = mask[:n]
        ids.append(seq[:n][mask].numpy().astype("int64"))
        log_p.append(lp[:n][mask].sum())
    return ids, -torch.stack(log_p)


@torch.no_grad()
def ctc_greedy_decode(sd, xs, xlen, blank=NUL, time_reductions=(1,)):
    """CTCEncoder.greedy_decode."""
    return greedy_from_logprobs(ctc_encoder_forward(sd, xs, time_reductions), xlen, blank)
