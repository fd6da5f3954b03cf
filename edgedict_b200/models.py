"""H100-native mirror of the reference's top-level ``models.py`` language model, ``LMModel`` (models.py:224-261): the
LSTM LM that ``cli/train_lm.py`` trains and every beam search here fuses (``lm=``).

Same constructor, errors, submodules, ``init_weights`` / ``init_hidden``, ``forward`` return value and ``state_dict``
keys as the reference, so ``cli/train_lm.py`` runs on this module after ``from edgedict_b200.models import LMModel``.
As in ``edgedict_b200.rnnt.models``, the ``nn.Embedding`` / ``nn.LSTM`` / ``nn.Linear`` objects are PARAMETER
CONTAINERS ONLY (identical default initialisation, built in the reference's order, so one ``torch.manual_seed`` gives
the reference's weights bit for bit); all arithmetic goes through libedgedict_b200.so (edgedict_b200/functional.py).
CUDA tensors are mandatory.  ``set_precision("fp32" | "bf16")`` and ``torch.autocast('cuda')`` select the arithmetic
as in ``rnnt/models.py``.
"""
import operator

import torch
import torch.nn.functional as F
from torch import nn

from . import functional as Fn
from .rnnt.models import _precision, _set_precision

_REDUCTIONS = ("mean", "sum", "none")


class LMModel(nn.Module):
    """The reference's LMModel: embedding -> dropout -> nn.LSTM(nlayers, inter-layer dropout) -> dropout -> Linear ->
    log-softmax, on the engine's kernels (Fn.Embedding without a padding row, one Fn.LSTMLayer per layer, Fn.Linear,
    Fn.LogSoftmax).  Dropout is torch's F.dropout and is active only in ``training`` mode.  ``loss`` is the fused
    training path: the output layer, the log-softmax and nn.NLLLoss in one autograd node."""

    def __init__(self, ntoken, ninp, nhid, nlayers, dropout=0.5, tie_weights=False):
        super().__init__()
        self.ntoken = ntoken
        self.drop = nn.Dropout(dropout)
        self.encoder = nn.Embedding(ntoken, ninp)
        self.rnn = nn.LSTM(ninp, nhid, nlayers, dropout=dropout, batch_first=True)
        self.decoder = nn.Linear(nhid, ntoken)
        if tie_weights:
            if nhid != ninp:
                raise ValueError('When using the tied flag, nhid must be equal to emsize')
            self.decoder.weight = self.encoder.weight
        self.init_weights()
        self.nhid = nhid
        self.rnn_type = 'LSTM'
        self.nlayers = nlayers

    def init_weights(self):
        initrange = 0.1
        nn.init.uniform_(self.encoder.weight, -initrange, initrange)
        nn.init.zeros_(self.decoder.weight)
        nn.init.uniform_(self.decoder.weight, -initrange, initrange)

    def init_hidden(self, bsz):
        weight = next(self.parameters())
        return (weight.new_zeros(self.nlayers, bsz, self.nhid),
                weight.new_zeros(self.nlayers, bsz, self.nhid))

    def set_precision(self, precision):
        return _set_precision(self, precision)

    def _trunk(self, input, hidden):
        """Embedding, the LSTM layers and the dropouts: (output [B, S, nhid], (h, c) [L, B, nhid])."""
        p = _precision(self)
        x = Fn.Embedding.apply(input, self.encoder.weight, False, 0, -1)     # -1: no padding row
        x = F.dropout(x, self.drop.p, self.training)
        hs, cs = (None, None) if hidden is None else hidden
        out_h, out_c = [], []
        for k in range(self.nlayers):
            w = [getattr(self.rnn, n % k) for n in ("weight_ih_l%d", "weight_hh_l%d", "bias_ih_l%d", "bias_hh_l%d")]
            x, hT, cT = Fn.LSTMLayer.apply(x, None if hs is None else hs[k], None if cs is None else cs[k],
                                           w[0], w[1], w[2], w[3], p)
            if k < self.nlayers - 1:
                x = F.dropout(x, self.rnn.dropout, self.training)            # nn.LSTM's inter-layer dropout
            out_h.append(hT)
            out_c.append(cT)
        x = F.dropout(x, self.drop.p, self.training)
        return x, (torch.stack(out_h, 0), torch.stack(out_c, 0))

    def forward(self, input, hidden=None):
        """input [B, S] token ids, hidden (h0, c0) [L, B, nhid] or None (zeros) -> (log-probs [B*S, ntoken] fp32,
        (h, c) [L, B, nhid]), the reference's return value.  The log-softmax is fp32 in both precision modes."""
        x, hidden = self._trunk(input, hidden)
        lin = self.decoder
        decoded = Fn.Linear.apply(x, lin.weight, lin.bias, _precision(self)).view(-1, self.ntoken)
        return Fn.LogSoftmax.apply(decoded), hidden

    def loss(self, input, targets, hidden=None, ignore_index=0, reduction="mean"):
        """nn.NLLLoss(ignore_index=ignore_index, reduction=reduction)(self(input, hidden)[0], targets.flatten()), with
        the output layer, the log-softmax and the loss in one autograd node: the [B*S, ntoken] log-probs are never
        written, and no step reads anything back to the host.  reduction "mean" (over the targets that are not
        ignore_index; NaN when all are, as torch), "sum" -> a 0-d tensor, "none" -> the per-token costs [B*S], 0 at
        ignored positions (perplexity, sentence scores).  A target that is not ignore_index and lies outside
        [0, ntoken) is never used as an index: it makes that token's cost NaN (and so a mean or sum NaN) and its
        gradient row NaN, where torch raises.  bf16 mode takes the log-sum-exp from the logits GEMM's fp32
        accumulators and differentiates through bf16 logits; it needs ntoken and nhid to be multiples of 8
        (ValueError otherwise)."""
        if reduction not in _REDUCTIONS:
            raise ValueError("reduction must be one of %s, got %r" % (_REDUCTIONS, reduction))
        if not isinstance(targets, torch.Tensor) or targets.dtype not in (torch.int32, torch.int64):
            raise TypeError("targets must be an int32 or int64 tensor")
        if targets.numel() != input.numel():
            raise ValueError("targets must have one entry per input token (%d), got %d" % (input.numel(),
                                                                                           targets.numel()))
        ignore_index = operator.index(ignore_index)
        if _precision(self) == "bf16" and (self.ntoken % 8 or self.nhid % 8):
            raise ValueError("bf16 mode needs ntoken and nhid to be multiples of 8 (the rows of the bf16 GEMM operands "
                             "are 16-byte aligned), got %d and %d; use fp32 mode" % (self.ntoken, self.nhid))
        x, _ = self._trunk(input, hidden)
        lin = self.decoder
        return Fn.LMLoss.apply(x.reshape(-1, x.shape[-1]), lin.weight, lin.bias, targets.reshape(-1), ignore_index,
                               reduction, _precision(self))
