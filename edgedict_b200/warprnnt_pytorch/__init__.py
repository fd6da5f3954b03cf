"""Drop-in for the reference's ``warprnnt_pytorch`` package
(warp-transducer/pytorch_binding/warprnnt_pytorch/__init__.py:1-141): same ``RNNTLoss`` /
``rnnt_loss`` signatures, same input certification and error types, same 'mean' = sum/B
semantics -- but CUDA-only: CPU activations raise instead of silently taking a slow path, and
the native status code is checked (the reference's binding drops it, binding.cpp:46-80)."""
import torch
from torch.nn import Module

from ..functional import RNNTLossFn, check_fastemit_lambda

__all__ = ['rnnt_loss', 'RNNTLoss']


def _check_type(var, t, name):
    if var.dtype is not t:
        raise TypeError("{} must be {}".format(name, t))


def _check_contiguous(var, name):
    if not var.is_contiguous():
        raise ValueError("{} must be contiguous".format(name))


def _check_dim(var, dim, name):
    if len(var.shape) != dim:
        raise ValueError("{} must be {}D".format(name, dim))


def certify_inputs(log_probs, labels, lengths, label_lengths):
    """Same checks, in the same order, as __init__.py:115-140 of the reference binding."""
    _check_type(labels, torch.int32, "labels")
    _check_type(label_lengths, torch.int32, "label_lengths")
    _check_type(lengths, torch.int32, "lengths")
    _check_contiguous(log_probs, "log_probs")
    _check_contiguous(labels, "labels")
    _check_contiguous(label_lengths, "label_lengths")
    _check_contiguous(lengths, "lengths")
    if lengths.shape[0] != log_probs.shape[0]:
        raise ValueError("must have a length per example.")
    if label_lengths.shape[0] != log_probs.shape[0]:
        raise ValueError("must have a label length per example.")
    _check_dim(log_probs, 4, "log_probs")
    _check_dim(labels, 2, "labels")
    _check_dim(lengths, 1, "lenghts")
    _check_dim(label_lengths, 1, "label_lenghts")
    max_T = torch.max(lengths)
    max_U = torch.max(label_lengths)
    T, U = log_probs.shape[1:3]
    if T != max_T:
        raise ValueError("Input length mismatch")
    if U != max_U + 1:
        raise ValueError("Output length mismatch")


def rnnt_loss(acts, labels, act_lens, label_lens, blank=0, reduction='mean', fastemit_lambda=0.0):
    """acts [B,T,U+1,V] raw logits on CUDA (fp32 or fp64); labels [B,U] int32; lengths int32.

    fastemit_lambda: FastEmit's regularisation weight (Yu et al., ICASSP 2021), a finite real >= 0.  Above 0 the
    gradient along every label-emitting edge of the lattice is scaled by (1 + fastemit_lambda), which teaches a
    streaming transducer to emit its tokens earlier (include/edgedict_b200.h, eb_rnnt_loss_bwd_fe).  It acts in the
    backward pass only: the returned costs are the plain negative log-likelihoods, bit for bit those of 0."""
    fastemit_lambda = check_fastemit_lambda(fastemit_lambda)
    certify_inputs(acts, labels, act_lens, label_lens)
    if not acts.is_cuda:
        raise RuntimeError("edgedict_b200.warprnnt_pytorch is CUDA-only (sm_90a); got CPU activations")
    if acts.dtype not in (torch.float32, torch.float64):
        raise TypeError("unsupported data type {} (float32/float64 only, as in binding.cpp:46-80)".format(acts.dtype))
    dev = acts.device
    return RNNTLossFn.apply(acts, labels.to(dev), act_lens.to(dev), label_lens.to(dev), blank, reduction,
                            fastemit_lambda)


class RNNTLoss(Module):
    """RNNTLoss(blank=0, reduction='mean', fastemit_lambda=0.0): 'none' | 'sum' | 'mean' (= sum / batch size);
    fastemit_lambda as in rnnt_loss (backward only, the costs do not change)."""

    def __init__(self, blank=0, reduction='mean', fastemit_lambda=0.0):
        super(RNNTLoss, self).__init__()
        self.blank = blank
        self.reduction = reduction
        self.fastemit_lambda = check_fastemit_lambda(fastemit_lambda)

    def forward(self, acts, labels, act_lens, label_lens):
        return rnnt_loss(acts, labels, act_lens, label_lens, self.blank, self.reduction, self.fastemit_lambda)
