"""Forced alignment of a transducer: for a known transcript, the single best path through the RNN-T lattice (Viterbi), so
that each label gets the encoder frame at which it is emitted.

``rnnt_forced_align`` takes the inputs ``RNNTLoss`` takes (raw joint logits); ``Transducer.align`` runs the model
itself.  ``edgedict_b200.ctc.forced_align`` is the CTC counterpart.  The recurrence, the tie rule and the output layout
are stated with ``eb_rnnt_viterbi`` in include/edgedict_b200.h.
"""
import torch

from . import ops
from .warprnnt_pytorch import certify_inputs

__all__ = ["rnnt_forced_align"]


@torch.no_grad()
def rnnt_forced_align(acts, labels, act_lens, label_lens, blank=0):
    """Viterbi alignment of raw logits acts [B, T, U+1, V] (fp32 or fp64, CUDA), labels int32 [B, U], lengths int32
    [B], with ``certify_inputs``' checks and errors and then RNNTLoss's (RuntimeError for CPU acts, TypeError for
    another dtype).

    Returns, on the device, (frames int32 [B, U]: the frame at which label u is emitted, -1 past label_lens[b];
    label_logp [B, U] in acts' dtype: log p(label u) at that frame, 0 past label_lens[b]; score [B]: the log-prob of
    the best path, blank at the last frame included).  On an exact tie a lattice cell takes the blank ("stay") step."""
    certify_inputs(acts, labels, act_lens, label_lens)
    if not acts.is_cuda:
        raise RuntimeError("edgedict_b200 rnnt_forced_align is CUDA-only (sm_90a); got CPU activations")
    if acts.dtype not in (torch.float32, torch.float64):
        raise TypeError("unsupported data type {} (float32/float64 only)".format(acts.dtype))
    dev = acts.device
    B, T, U = acts.shape[:3]
    xl, yl = act_lens.to(dev), label_lens.to(dev)
    _, ws = ops.rnnt_loss_fwd(acts, labels.to(dev), xl, yl, blank, need_beta=False)
    return ops.rnnt_viterbi(xl, yl, B, T, U, ws, acts.dtype)
