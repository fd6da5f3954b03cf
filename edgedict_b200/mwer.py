"""Minimum word error rate training and error rates on the device.

  * ``edit_distance`` -- batched Levenshtein counts (errors, substitutions, deletions, insertions, reference length) of
    hypothesis rows against reference rows, in tokens or, with a ``word_table``, in words (csrc/mwer.cu).
  * ``word_table`` -- the table that makes the units words: built on the host from the reference's ``CharTokenizer``
    (``id2token``) or ``HuggingFaceTokenizer`` (CharBPE, ``</w>`` word ends), or from a plain list of pieces.
  * ``error_rate`` -- corpus-level errors over reference units: ``jiwer.wer`` on a batch of decoded texts, computed from
    the ids.
  * ``expected_risk`` -- the MWER loss over N-best costs (Prabhavalkar et al., ICASSP 2018): the mean over utterances of
    sum_i P_i (E_i - mean E), P the posteriors renormalised over each N-best list.

``Transducer.mwer_loss`` and ``CTCEncoder.mwer_loss`` (rnnt/models.py) put these together with the beam engines.

Words.  A word is a maximal non-empty run of characters, closed by a token that ends a word (CharBPE's ``</w>``
suffix, whose characters it includes), a separator (``CharTokenizer``'s space) or the end of the sequence; dropped ids
(0-3 and anything ``decode`` removes) vanish without closing a word.  Two words are equal iff their characters are, so
two tokenisations of one word are one word.  This is what ``decode`` followed by jiwer's default transform
(RemoveMultipleSpaces, Strip, ReduceToListOfListOfWords) gives when the only whitespace in the vocabulary is the
separator: word-level errors are jiwer's WER numerator and the reference length its denominator.

Every argument is checked on the host before any device work; lengths given as device tensors are copied to the host
for that.
"""
import numbers
import operator

import torch

from . import functional as Fn
from . import ops

MAX_UNITS = 4096                  # EB_EDIT_MAX_UNITS: tokens per sequence
INSIDE, END, SEP, DROP = 0, 1, 2, 3
SPECIAL_IDS = (0, 1, 2, 3)        # NUL, PAD, BOS, UNK (rnnt/tokenizer.py)


class WordTable:
    """Per token id {character offset, character count, class} (int32 [V, 3]) and the characters (int32 code points)
    that ``edit_distance`` segments words with; ``vocab_size`` = V ids are covered.  Built by ``word_table``."""

    def __init__(self, entries, chars):
        self.entries = entries
        self.chars = chars
        self.vocab_size = entries.shape[0]
        self._dev = {}

    def device(self, device):
        """(entries, chars) on ``device``, uploaded once."""
        key = torch.device(device)
        if key not in self._dev:
            self._dev[key] = (self.entries.to(key), self.chars.to(key))
        return self._dev[key]


def word_table(source, end_suffix=None, separators=None, dropped=SPECIAL_IDS):
    """The WordTable of a tokenizer or of a list of pieces.

      * the reference's ``CharTokenizer`` (has ``id2token``): one character per id, the space token a separator;
      * its ``HuggingFaceTokenizer`` (``.tokenizer.get_vocab()``): CharBPE pieces, ``</w>`` ends a word and is not a
        character, no separator;
      * a list of pieces (None: an id ``decode`` drops): ``end_suffix`` marks word ends (default none), ``separators``
        are the pieces that separate words (default a space).
    Ids in ``dropped`` (default 0-3, the special tokens both tokenizers remove) and ids without a piece are dropped."""
    if hasattr(source, "id2token"):
        pieces = list(source.id2token)
    elif hasattr(source, "tokenizer") and hasattr(source.tokenizer, "get_vocab"):
        vocab = source.tokenizer.get_vocab()
        pieces = [None] * (max(vocab.values()) + 1 if vocab else 0)
        for piece, i in vocab.items():
            pieces[i] = piece
        end_suffix = "</w>" if end_suffix is None else end_suffix
        separators = () if separators is None else separators
    elif isinstance(source, (list, tuple)):
        pieces = list(source)
    else:
        raise TypeError("word_table takes a CharTokenizer, a HuggingFaceTokenizer or a list of pieces, got %s"
                        % type(source).__name__)
    separators = (" ",) if separators is None else tuple(separators)
    if end_suffix is not None and (not isinstance(end_suffix, str) or not end_suffix):
        raise ValueError("end_suffix must be a non-empty string or None, got %r" % (end_suffix,))
    dropped = {operator.index(i) for i in dropped}
    if not pieces:
        raise ValueError("word_table needs at least one piece")
    entries, chars = [], []
    for i, piece in enumerate(pieces):
        if piece is not None and not isinstance(piece, str):
            raise TypeError("piece %d must be a string or None, got %s" % (i, type(piece).__name__))
        if piece is None or i in dropped:
            entries.append((0, 0, DROP))
        elif piece in separators:
            entries.append((0, 0, SEP))
        else:
            cls = INSIDE
            if end_suffix is not None and piece.endswith(end_suffix):
                cls, piece = END, piece[:-len(end_suffix)]
            entries.append((len(chars), len(piece), cls))
            chars.extend(ord(c) for c in piece)
    return WordTable(torch.tensor(entries, dtype=torch.int32).reshape(-1, 3),
                     torch.tensor(chars or [0], dtype=torch.int32))


def _host_ints(x, n, name):
    if isinstance(x, torch.Tensor):
        if x.is_floating_point() or x.is_complex() or x.dtype == torch.bool:
            raise TypeError("%s must hold integers, got %s" % (name, x.dtype))
        x = x.detach().reshape(-1).cpu().to(torch.int64)
    else:
        x = torch.tensor([operator.index(v) for v in x], dtype=torch.int64)
    if x.numel() != n:
        raise ValueError("%s must have %d entries, got %d" % (name, n, x.numel()))
    return x


def _rows(x, name):
    if not isinstance(x, torch.Tensor):
        raise TypeError("%s must be a tensor" % name)
    if x.dim() != 2:
        raise ValueError("%s must be [rows, length], got shape %s" % (name, tuple(x.shape)))
    if x.is_floating_point() or x.is_complex() or x.dtype == torch.bool:
        raise TypeError("%s must hold integer ids, got %s" % (name, x.dtype))
    return x


def _check_lens(lens, width, name):
    if lens.numel() and (int(lens.min()) < 0 or int(lens.max()) > min(width, MAX_UNITS)):
        raise ValueError("%s must lie in [0, min(row length %d, %d)], got %s" % (name, width, MAX_UNITS, lens.tolist()))


def check_word_table(table, vocab=0):
    """None or a WordTable covering ids [0, vocab); raises TypeError / ValueError."""
    if table is None:
        return None
    if not isinstance(table, WordTable):
        raise TypeError("word_table must be a mwer.WordTable (see mwer.word_table), got %s" % type(table).__name__)
    if table.vocab_size < vocab:
        raise ValueError("the word table covers %d ids, the vocabulary has %d" % (table.vocab_size, vocab))
    return table


def _meta(hyp_lens, ref_lens, ref_index, device):
    host = torch.cat([hyp_lens, ref_lens, ref_index]).to(torch.int32)
    staged = torch.empty(host.shape, dtype=torch.int32, pin_memory=True)
    staged.copy_(host)
    return staged.to(device, non_blocking=True), staged


def _distance(hyp, hyp_lens, ref, ref_lens, ref_index, table, vocab):
    """ops.edit_distance on checked host lengths / index (int64 tensors) and int32 rows on the device."""
    meta, meta_host = _meta(hyp_lens, ref_lens, ref_index, hyp.device)
    wt, wc = table.device(hyp.device) if table is not None else (None, None)
    return ops.edit_distance(hyp, ref, meta, meta_host, hyp.shape[0], ref.shape[0], wt, wc, vocab)


def edit_distance(hyp, hyp_lens, ref, ref_lens, ref_index=None, word_table=None):
    """Levenshtein counts of hypothesis rows against reference rows, on the device.

      * hyp [n_hyp, Lh], ref [n_ref, Lr]: integer ids on one CUDA device, left-aligned, row i holding its first
        hyp_lens[i] / ref_lens[i] ids (each length in [0, min(row length, 4096)]);
      * ref_index: n_hyp integers in [0, n_ref), the reference of each hypothesis (default: row i against row i);
      * word_table: None (units are tokens) or a ``word_table(...)`` (units are words; ids outside the table count as
        dropped).

    Returns int32 [n_hyp, 5] on the device: errors = S + D + I, substitutions S, deletions D, insertions I and the
    reference length, in units.  Ties between alignments of equal distance go to the substitution (or hit), then the
    deletion, then the insertion, cell by cell of the DP."""
    hyp, ref = _rows(hyp, "hyp"), _rows(ref, "ref")
    table = check_word_table(word_table)
    n_hyp, n_ref = hyp.shape[0], ref.shape[0]
    hl = _host_ints(hyp_lens, n_hyp, "hyp_lens")
    rl = _host_ints(ref_lens, n_ref, "ref_lens")
    _check_lens(hl, hyp.shape[1], "hyp_lens")
    _check_lens(rl, ref.shape[1], "ref_lens")
    if ref_index is None:
        if n_hyp != n_ref:
            raise ValueError("without ref_index hyp and ref need as many rows, got %d and %d" % (n_hyp, n_ref))
        ri = torch.arange(n_hyp, dtype=torch.int64)
    else:
        ri = _host_ints(ref_index, n_hyp, "ref_index")
        if ri.numel() and (int(ri.min()) < 0 or int(ri.max()) >= n_ref):
            raise ValueError("ref_index must lie in [0, %d), got %s" % (n_ref, ri.tolist()))
    if not hyp.is_cuda or not ref.is_cuda or hyp.device != ref.device:
        raise RuntimeError("edit_distance needs hyp and ref on one CUDA device (there is no CPU path)")
    hyp = hyp.to(torch.int32).contiguous()
    ref = ref.to(torch.int32).contiguous()
    return _distance(hyp, hl, ref, rl, ri, table, table.vocab_size if table is not None else 0)


def error_rate(hyp, hyp_lens, ref, ref_lens, ref_index=None, word_table=None):
    """Corpus-level error rate of a batch, sum of errors over sum of reference lengths (``jiwer.wer`` over the decoded
    texts with a word table, the token error rate without): ``edit_distance``'s arguments, a float.  Raises ValueError
    when the references hold no unit."""
    counts = edit_distance(hyp, hyp_lens, ref, ref_lens, ref_index, word_table)
    errors, units = (int(v) for v in counts[:, [0, 4]].sum(0, dtype=torch.int64).cpu())
    if units == 0:
        raise ValueError("the references hold no unit: the error rate is undefined")
    return errors / units


def expected_risk(costs, errors, valid=None):
    """The MWER loss of N-best lists: costs [B, N] fp32 CUDA (-log P(y_i | x), differentiable), errors [B, N] integers
    (the edit distances of the hypotheses), valid [B, N] (nonzero: rank i exists; default all).  Returns (loss [1] =
    mean over b of sum_i P_i (E_i - Ebar_b), posteriors [B, N]), P = softmax of -c over the valid ranks and Ebar the
    plain mean of their errors; an utterance with one valid rank gives 0.  N <= 1024."""
    from .stream_engine import BEAM_MAX_W
    if not isinstance(costs, torch.Tensor) or not isinstance(errors, torch.Tensor):
        raise TypeError("costs and errors must be tensors")
    if costs.dtype != torch.float32:
        raise TypeError("costs must be float32, got %s" % costs.dtype)
    if costs.dim() != 2 or costs.shape[0] < 1 or not 1 <= costs.shape[1] <= BEAM_MAX_W:
        raise ValueError("costs must be [B >= 1, 1 <= N <= %d], got shape %s" % (BEAM_MAX_W, tuple(costs.shape)))
    for t, name in ((errors, "errors"), (valid, "valid")):
        if t is None:
            continue
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a tensor" % name)
        if t.is_floating_point() or t.is_complex():
            raise TypeError("%s must hold integers, got %s" % (name, t.dtype))
        if t.shape != costs.shape:
            raise ValueError("%s must have costs' shape %s, got %s" % (name, tuple(costs.shape), tuple(t.shape)))
    if not costs.is_cuda or errors.device != costs.device or (valid is not None and valid.device != costs.device):
        raise RuntimeError("expected_risk needs costs, errors and valid on one CUDA device (there is no CPU path)")
    v = torch.ones_like(errors, dtype=torch.int32) if valid is None else valid.to(torch.int32).contiguous()
    return Fn.ExpectedRisk.apply(costs, errors.to(torch.int32).contiguous(), v)


def check_ce_weight(value):
    """The weight of the reference row's loss in a MWER loss: a finite real >= 0."""
    if isinstance(value, bool) or not isinstance(value, numbers.Real):
        raise TypeError("ce_weight must be a real number, got %s" % type(value).__name__)
    w = float(value)
    if not w >= 0 or w == float("inf"):
        raise ValueError("ce_weight must be finite and >= 0, got %r" % w)
    return w


def nbest_rows(buf, B, N, L, ys, ylen, table=None, vocab=0):
    """A beam engine's N-best output ``buf`` (stream_engine.final_outputs' layout) and the references ys int32 [B, S]
    (device) of ylen (host int64 [B]) -> (labels int32 [B*(N+1), Umax], row lengths int32 on the device and int64 on
    the host, valid int32 [B, N], errors int32 [B, N], count int32 [B]).  Row b*(N+1)+i is rank i, row b*(N+1)+N the
    reference (eb_nbest_pack); errors are each rank's edit distance to its reference, in words with ``table``.  One
    device-to-host copy: the row lengths, for Umax."""
    n = B * N * L
    ids, count = buf[:n].view(B, N, L), buf[2 * n + B * N:]
    ref_len = ylen.to(torch.int32).pin_memory().to(ys.device, non_blocking=True)
    labels, lens, valid = ops.nbest_pack(ids, count, ys, ref_len, max(L, ys.shape[1]))
    lens_h = lens.cpu().to(torch.int64)
    if int(lens_h.max()) > MAX_UNITS:
        raise ValueError("edit distances take rows of at most %d tokens, got %d" % (MAX_UNITS, int(lens_h.max())))
    R = B * (N + 1)
    ref_rows = torch.arange(R, dtype=torch.int64) // (N + 1) * (N + 1) + N
    counts = _distance(labels, lens_h, labels, lens_h, ref_rows, table, vocab)
    errors = counts[:, 0].view(B, N + 1)[:, :N].contiguous()
    return labels[:, :int(lens_h.max())].contiguous(), lens, lens_h, valid, errors, count.clone()
