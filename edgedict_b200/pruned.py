"""Pruned RNN-T loss (Kuang et al., "Pruned RNN-T for fast, memory-efficient ASR training", Interspeech 2022).

    costs, ws = rnnt_loss_simple(am, lm, labels, act_lens, label_lens, reduction="none", return_workspace=True)
    s_begin, no_path = prune_ranges(ws, act_lens, label_lens, prune_range)
    pruned = rnnt_loss_pruned(band_logits, labels, act_lens, label_lens, s_begin, no_path)

am [B, T, V] and lm [B, U+1, V] are the trivial joiner's projections, band_logits [B, T, R, V] the real joint's
logits at the cells (t, s_begin[b, t] + r).  The formulas and length rules are those of include/edgedict_b200.h.
Every argument is checked before any device work, as warprnnt_pytorch.rnnt_loss checks its own.
"""
import torch

from . import functional as Fn
from . import ops


def _check_common(labels, act_lens, label_lens, B, T, U, V, blank, reduction):
    for name, t in (("labels", labels), ("act_lens", act_lens), ("label_lens", label_lens)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.int32:
            raise TypeError("%s must be an int32 tensor" % name)
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor; there is no CPU path" % name)
    if labels.dim() != 2 or labels.shape[0] != B or labels.shape[1] != U - 1:
        raise ValueError("labels must be [B, U-1] = [%d, %d], got %s" % (B, U - 1, tuple(labels.shape)))
    if act_lens.shape != (B,) or label_lens.shape != (B,):
        raise ValueError("act_lens and label_lens must be [B] = [%d]" % B)
    if not 1 <= U <= 1024:
        raise ValueError("U (max label length + 1) must be in [1, 1024], got %d" % U)
    if T < 1:
        raise ValueError("T must be >= 1")
    if not 0 <= blank < V:
        raise ValueError("blank must be in [0, %d), got %d" % (V, blank))
    if reduction not in ("none", "sum", "mean"):
        raise ValueError("reduction must be 'none', 'sum' or 'mean', got %r" % (reduction,))


def check_prune_range(R):
    """The prune range as an int in [2, 64] (TypeError / ValueError otherwise)."""
    if isinstance(R, bool) or not isinstance(R, int):
        raise TypeError("prune_range must be an int, got %r" % (R,))
    if not 2 <= R <= 64:
        raise ValueError("prune_range must be in [2, 64], got %d" % R)
    return R


def _reduce(costs, reduction):
    if reduction == "none":
        return costs
    return costs.sum() if reduction == "sum" else costs.mean()


def rnnt_loss_simple(am, lm, labels, act_lens, label_lens, blank=0, reduction="mean", return_workspace=False):
    """The trivial joiner's RNN-T loss on log softmax(am[b, t] + lm[b, u]); with return_workspace also the loss
    workspace that prune_ranges reads."""
    for name, t in (("am", am), ("lm", lm)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.dim() != 3:
            raise TypeError("%s must be a 3-d float32 tensor" % name)
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor; there is no CPU path" % name)
    B, T, V = am.shape
    if lm.shape[0] != B or lm.shape[2] != V:
        raise ValueError("lm must be [B, U, V] with am's B = %d and V = %d, got %s" % (B, V, tuple(lm.shape)))
    _check_common(labels, act_lens, label_lens, B, T, lm.shape[1], V, blank, reduction)
    costs, ws = Fn.SimpleLoss.apply(am, lm, labels, act_lens, label_lens, blank)
    out = _reduce(costs, reduction)
    return (out, ws) if return_workspace else out


def prune_ranges(ws, act_lens, label_lens, prune_range, T, U):
    """(s_begin [B, T] int32, no_path [B] int32): each frame's band of min(prune_range, U_b) symbol positions from the
    simple loss's workspace; no_path[b] = 1 when the bands of utterance b hold no path."""
    R = check_prune_range(prune_range)
    if not isinstance(ws, torch.Tensor) or ws.dtype != torch.uint8 or not ws.is_cuda:
        raise TypeError("ws must be the CUDA uint8 workspace of rnnt_loss_simple")
    for name, t in (("act_lens", act_lens), ("label_lens", label_lens)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or t.dim() != 1:
            raise TypeError("%s must be a 1-d int32 tensor" % name)
        if t.device != ws.device:
            raise RuntimeError("%s must be on ws's device %s" % (name, ws.device))
    B = act_lens.shape[0]
    if label_lens.shape != (B,):
        raise ValueError("act_lens and label_lens must both be [B]")
    if ws.numel() != ops.lib().eb_rnnt_workspace_bytes(B, T, U, 4):
        raise ValueError("ws is not the workspace of a [%d, %d, %d] simple loss" % (B, T, U))
    if T > 12288:
        raise ValueError("T must be <= 12288 for the band choice, got %d" % T)
    return ops.rnnt_band_choice(act_lens, label_lens, B, T, U, R, ws)


def rnnt_loss_pruned(logits, labels, act_lens, label_lens, s_begin, no_path, blank=0, reduction="mean"):
    """The RNN-T loss on the band rows logits [B, T, R, V] fp32; +inf for an utterance whose bands hold no path."""
    if not isinstance(logits, torch.Tensor) or logits.dtype != torch.float32 or logits.dim() != 4:
        raise TypeError("logits must be a 4-d float32 tensor [B, T, R, V]")
    if not logits.is_cuda:
        raise RuntimeError("logits must be a CUDA tensor; there is no CPU path")
    B, T, R, V = logits.shape
    check_prune_range(R)
    U = labels.shape[1] + 1 if isinstance(labels, torch.Tensor) and labels.dim() == 2 else 0
    _check_common(labels, act_lens, label_lens, B, T, U, V, blank, reduction)
    if s_begin.dtype != torch.int32 or s_begin.shape != (B, T) or no_path.dtype != torch.int32 or no_path.shape != (B,):
        raise ValueError("s_begin must be int32 [B, T] and no_path int32 [B]")
    return _reduce(Fn.RNNTBandLossFn.apply(logits, labels, act_lens, label_lens, s_begin, no_path, U, blank), reduction)
