"""CTC loss on the engine: ``CTCLoss`` / ``ctc_loss`` with the signature and semantics of ``torch.nn.CTCLoss`` /
``torch.nn.functional.ctc_loss``, computed by this library's kernels (csrc/ctc.cu).

Unlike torch's CUDA ctc_loss, the backward pass is deterministic: the gradient of every utterance is bitwise the same on
every run and does not depend on the other utterances of the batch, so it may run under
``torch.use_deterministic_algorithms(True)``.

Accepted inputs:
  * log_probs: fp32 CUDA tensor (T, N, C), or (T, C) for one unbatched utterance.  Any strides over T and N (the
    ``.transpose(0, 1)`` view of a [N, T, C] tensor is used without a copy).  Other dtypes raise TypeError, CPU tensors
    RuntimeError: there is no fallback.
  * targets: integer tensor, padded (N, S) or the labels of all utterances concatenated (sum(target_lengths),);
    (S,) for an unbatched input.  Labels are expected in [0, C) and different from blank.  A label outside [0, C) gives
    the utterance no alignment (cost +inf).
  * input_lengths / target_lengths: integer tensors or sequences with one entry per utterance (a scalar when
    unbatched).  They are read on the host; every length is checked there, before anything is launched.
  * target lengths up to 1023.

reduction: 'none' (per-utterance costs), 'sum', or 'mean' (each cost divided by max(target_length, 1), then the mean over
the batch).  zero_infinity sets infinite costs (no alignment exists) and their gradients to zero.
"""
import operator

import torch
from torch import nn

from . import functional as Fn
from . import ops

MAX_TARGET_LENGTH = 1023          # 2S+1 lattice states, at most 2047


def _lengths(x, n, name):
    if isinstance(x, torch.Tensor):
        if x.is_floating_point() or x.is_complex() or x.dtype == torch.bool:
            raise TypeError("%s must hold integers, got %s" % (name, x.dtype))
        x = x.detach().reshape(-1).cpu().to(torch.int64)
    else:
        if not hasattr(x, "__len__"):
            x = [x]
        x = torch.tensor([operator.index(v) for v in x], dtype=torch.int64)
    if x.numel() != n:
        raise ValueError("%s must have one entry per utterance (%d), got %d" % (name, n, x.numel()))
    return x


def _targets_and_lengths(targets, input_lengths, target_lengths, N, T):
    """The host checks of the lengths and the target layout -> (input lengths, target lengths, offsets, S)."""
    il = _lengths(input_lengths, N, "input_lengths")
    tl = _lengths(target_lengths, N, "target_lengths")
    if bool((il < 0).any()) or bool((il > T).any()):
        raise ValueError("input_lengths must lie in [0, T = %d], got %s" % (T, il.tolist()))
    if bool((tl < 0).any()):
        raise ValueError("target_lengths must be >= 0, got %s" % tl.tolist())
    if targets.dim() == 2:
        if targets.shape[0] != N:
            raise ValueError("padded targets must have %d rows, got %d" % (N, targets.shape[0]))
        if bool((tl > targets.shape[1]).any()):
            raise ValueError("target_lengths exceed the padded target length %d" % targets.shape[1])
        offsets = torch.arange(N, dtype=torch.int64) * targets.shape[1]
    elif targets.dim() == 1:
        if int(tl.sum()) != targets.numel():
            raise ValueError("concatenated targets hold %d labels, target_lengths sum to %d"
                             % (targets.numel(), int(tl.sum())))
        offsets = torch.cumsum(tl, 0) - tl
    else:
        raise ValueError("targets must be (N, S) or 1-D, got shape %s" % (tuple(targets.shape),))
    S = int(tl.max())
    if S > MAX_TARGET_LENGTH:
        raise ValueError("target lengths above %d are not supported, got %d" % (MAX_TARGET_LENGTH, S))
    return il, tl, offsets, S


def ctc_loss(log_probs, targets, input_lengths, target_lengths, blank=0, reduction="mean", zero_infinity=False):
    """torch.nn.functional.ctc_loss on the engine's kernels; see the module docstring."""
    if not isinstance(log_probs, torch.Tensor) or not isinstance(targets, torch.Tensor):
        raise TypeError("log_probs and targets must be tensors")
    if log_probs.dtype != torch.float32:
        raise TypeError("edgedict_b200 ctc_loss takes fp32 log_probs, got %s (there is no fallback)" % log_probs.dtype)
    if reduction not in ("none", "mean", "sum"):
        raise ValueError("reduction must be 'none', 'mean' or 'sum', got %r" % (reduction,))
    if targets.is_floating_point() or targets.is_complex() or targets.dtype == torch.bool:
        raise TypeError("targets must hold integers, got %s" % targets.dtype)
    unbatched = log_probs.dim() == 2
    if unbatched:
        if targets.dim() != 1:
            raise ValueError("an unbatched (T, C) input takes 1-D targets, got shape %s" % (tuple(targets.shape),))
        log_probs, targets = log_probs.unsqueeze(1), targets.unsqueeze(0)
    elif log_probs.dim() != 3:
        raise ValueError("log_probs must be (T, N, C) or (T, C), got shape %s" % (tuple(log_probs.shape),))
    T, N, V = log_probs.shape
    if T < 1 or N < 1 or V < 1:
        raise ValueError("log_probs must not be empty, got shape %s"
                         % (tuple(log_probs.shape),))
    blank = operator.index(blank)
    if not 0 <= blank < V:
        raise ValueError("blank must lie in [0, %d), got %d" % (V, blank))
    il, tl, offsets, S = _targets_and_lengths(targets, input_lengths, target_lengths, N, T)
    if not log_probs.is_cuda:                  # checked last: every argument error above is found without a GPU
        raise RuntimeError("edgedict_b200 ctc_loss needs CUDA log_probs (got a %s tensor); there is no CPU path"
                           % log_probs.device)
    dev = log_probs.device
    lens = torch.empty(3, N, dtype=torch.int32, pin_memory=True)
    lens[0], lens[1], lens[2] = offsets, tl, il
    lens = lens.to(dev, non_blocking=True)
    tg = targets.reshape(-1).to(device=dev, dtype=torch.int32).contiguous()
    if log_probs.stride(-1) != 1:
        log_probs = log_probs.contiguous()
    costs = Fn.CTCLossFn.apply(log_probs, tg, lens[0], lens[1], lens[2], (S, blank, bool(zero_infinity)))
    if reduction == "mean":
        costs = (costs / lens[1].clamp(min=1).to(costs.dtype)).mean()
    elif reduction == "sum":
        costs = costs.sum()
    elif unbatched:
        costs = costs[0]
    return costs


class CTCLoss(nn.Module):
    """torch.nn.CTCLoss on the engine's kernels (see ctc_loss)."""

    def __init__(self, blank=0, reduction="mean", zero_infinity=False):
        super().__init__()
        self.blank, self.reduction, self.zero_infinity = blank, reduction, zero_infinity

    def forward(self, log_probs, targets, input_lengths, target_lengths):
        return ctc_loss(log_probs, targets, input_lengths, target_lengths, self.blank, self.reduction,
                        self.zero_infinity)


def forced_align(log_probs, targets, input_lengths, target_lengths, blank=0):
    """Forced (Viterbi) alignment of known transcripts, batched: torchaudio.functional.forced_align's signature and
    return, for a whole batch in one kernel launch (csrc/ctc.cu).

      * log_probs: fp32 CUDA tensor [B, T, V] of log-softmax rows, batch first (what ``CTCEncoder.forward`` returns),
        any strides over B and T.
      * targets: integer tensor, padded (B, S) or all labels concatenated (sum(target_lengths),), as in ``ctc_loss``;
        S up to 1023.
      * input_lengths / target_lengths: integers or integer tensors, one per utterance, read on the host.

    Returns (alignments [B, T] in targets' dtype, scores [B, T] fp32), on the device.  Frame t < input_lengths[b]
    holds the label (or blank) the best path emits there and its log-prob; later frames hold -1 and 0.  An utterance
    without any alignment (its input too short for its labels and repeats, or a label outside [0, V)) holds -1 and -inf
    in every frame.  The path maximises the sum of the frame log-probs, accumulated in fp64; ties between predecessors
    go to the state itself, then s-1, then s-2, and the path ends in the last label unless the final blank is strictly
    better (include/edgedict_b200.h, eb_ctc_align).  Arguments are checked on the host before any launch, with
    ``ctc_loss``'s errors and order; CPU log_probs raise RuntimeError."""
    if not isinstance(log_probs, torch.Tensor) or not isinstance(targets, torch.Tensor):
        raise TypeError("log_probs and targets must be tensors")
    if log_probs.dtype != torch.float32:
        raise TypeError("edgedict_b200 forced_align takes fp32 log_probs, got %s (there is no fallback)" % log_probs.dtype)
    if targets.is_floating_point() or targets.is_complex() or targets.dtype == torch.bool:
        raise TypeError("targets must hold integers, got %s" % targets.dtype)
    if log_probs.dim() != 3:
        raise ValueError("log_probs must be [B, T, V], got shape %s" % (tuple(log_probs.shape),))
    B, T, V = log_probs.shape
    if T < 1 or B < 1 or V < 1:
        raise ValueError("log_probs must not be empty, got shape %s" % (tuple(log_probs.shape),))
    blank = operator.index(blank)
    if not 0 <= blank < V:
        raise ValueError("blank must lie in [0, %d), got %d" % (V, blank))
    il, tl, offsets, S = _targets_and_lengths(targets, input_lengths, target_lengths, B, T)
    if not log_probs.is_cuda:
        raise RuntimeError("edgedict_b200 forced_align needs CUDA log_probs (got a %s tensor); there is no CPU path"
                           % log_probs.device)
    dev = log_probs.device
    lens = torch.empty(3, B, dtype=torch.int32, pin_memory=True)
    lens[0], lens[1], lens[2] = offsets, tl, il
    lens = lens.to(dev, non_blocking=True)
    tg = targets.reshape(-1).to(device=dev, dtype=torch.int32).contiguous()
    if log_probs.stride(-1) != 1:
        log_probs = log_probs.contiguous()
    with torch.no_grad():
        alignment, scores = ops.ctc_align(log_probs, tg, lens[0], lens[1], lens[2], S, blank)
    return alignment.to(targets.dtype), scores


# beam_search keeps the program of its last call (one engine: its log-prob copy [B, T, V], history [B, T, W] x 3,
# token rows [2, B*W, T + 5], state and, with an LM, the LM's weights on the device); free_beam_search() releases it
_beam_engines = {}


def free_beam_search():
    """Release the device memory beam_search keeps for its next call with the same shapes and LM."""
    _beam_engines.clear()


def beam_search(log_probs, input_lengths, beam_width, blank=0, *, lm=None, lm_weight=0.0, length_bonus=0.0, lm_bos=1,
                lm_token_map=None, nbest=None, context=None, ngram=None, ngram_weight=0.0):
    """CTC prefix beam search (Hannun et al., 2014) on the device, optionally with shallow fusion of the reference's
    LSTM language model (LMModel, or its state_dict).  ``CTCEncoder.beam_search`` states the rule.

      * log_probs: fp32 CUDA tensor [B, T, V] of log-softmax rows, batch first (what ``CTCEncoder.forward`` returns),
        any strides.  ``ctc_loss``'s (T, N, C) layout is not taken as such: pass its ``.transpose(0, 1)``.
      * input_lengths: integers or an integer tensor, one per utterance, in log-prob frames, each in [0, T].
      * beam_width: W in [1, 1024]; blank in [0, V).
      * lm, lm_weight, length_bonus, lm_bos, lm_token_map: as ``Transducer.beam_search``'s fusion arguments.

    Returns (list of B int64 arrays: the best prefix of each utterance, -score [B] on the device: its negated
    (pb (+) pnb) + f).  Every argument is checked on the host before any device work (TypeError / ValueError, and
    RuntimeError for CPU log_probs: there is no CPU path).  One persistent kernel launch (stream_engine.CTCBeamEngine)
    and one device-to-host copy of the ids.  The engine stays resident for the next call with the same shapes and LM
    (about 4·B·T·(V + 4·W) bytes and the LM's weights); ``free_beam_search()`` releases it.

    N-best lists: ``nbest`` = N (an integer in [1, W]) returns instead a list of B lists of
    ``stream_engine.Hypothesis(tokens, frames, nlogp)``, best first: the live prefixes at the end of the search, ranked
    by (pb (+) pnb) + f descending (lowest slot on ties, the rule the best-only call picks by), min(N, live) of them.
    nlogp is the negated (pb (+) pnb) + f, and entry 0 of each list is bitwise the best-only call's ids and score.
    ``frames`` gives each token's log-prob frame: the frame of the extension that put it into the prefix, on the path
    the history recorded (an extension merged into another prefix's stay adds no token to it), so frames are strictly
    increasing.  An utterance of length 0 gives one empty hypothesis with nlogp 0.  Still one device-to-host copy;
    ``nbest`` is part of the engine cache key.

    Contextual biasing: ``context`` is an ``edgedict_b200.context.ContextGraph`` over the V tokens with this blank (a
    ValueError otherwise, before any device work).  An extension of a prefix in automaton state s by c adds the
    graph's increment delta(s, c) to the fusion term: f' = (f + LM term) + delta (f' = f + delta without an LM); a stay
    adds nothing and keeps the state.  The final ranking and every returned score use (pb (+) pnb) + f - P(s), P(s)
    the pending bonus of the partial match, so a phrase earns its bonus only once it completes.  An empty graph (or
    None) gives the search without context bit for bit; the graph's fingerprint is part of the engine cache key.

    N-gram shallow fusion: ``ngram`` is an ``edgedict_b200.ngram.NgramLM`` over the V tokens with this blank (a
    ValueError otherwise, before any device work), ``ngram_weight`` = w finite.  Each prefix carries the model's state h
    (the start state first); an extension by c adds w g(h, c) after the LM term, f' = ((f + T_LM) + w g) + delta, T_LM
    the LM term or, without an LM, ``length_bonus`` (legal with an ngram alone); a stay keeps the state and adds
    nothing.  The final ranking and every returned score use ((pb (+) pnb) + f + w e(h)) - P(s), e(h) the model's
    end-of-sentence term (absent without </s>).  The model's fingerprint, w and the length bonus are part of the
    engine cache key."""
    import numbers
    from .context import check_context, context_cache_key
    from .ngram import check_ngram, check_ngram_weight, ngram_cache_key
    from .stream_engine import BEAM_MAX_W, CTCBeamEngine, check_lm_args, check_nbest, lm_cache_key, nbest_lists
    if not isinstance(log_probs, torch.Tensor):
        raise TypeError("log_probs must be a tensor")
    if log_probs.dtype != torch.float32:
        raise TypeError("edgedict_b200 ctc beam_search takes fp32 log_probs, got %s (there is no fallback)"
                        % log_probs.dtype)
    if log_probs.dim() != 3:
        raise ValueError("log_probs must be [B, T, V], got shape %s" % (tuple(log_probs.shape),))
    B, T, V = log_probs.shape
    if B < 1 or T < 1 or V < 1:
        raise ValueError("log_probs must not be empty, got shape %s" % (tuple(log_probs.shape),))
    if isinstance(beam_width, bool) or not isinstance(beam_width, numbers.Integral):
        raise TypeError("beam_width must be an integer, got %r" % (beam_width,))
    W = int(beam_width)
    if not 1 <= W <= BEAM_MAX_W:
        raise ValueError("beam_width must be in [1, %d], got %d" % (BEAM_MAX_W, W))
    if W * V >= 2 ** 31:
        raise ValueError("beam_width x V must stay below 2^31, got %d x %d" % (W, V))
    N = 0 if nbest is None else check_nbest(nbest, W)
    blank = operator.index(blank)
    if not 0 <= blank < V:
        raise ValueError("blank must lie in [0, %d), got %d" % (V, blank))
    il = _lengths(input_lengths, B, "input_lengths")
    if bool((il < 0).any()) or bool((il > T).any()):
        raise ValueError("input_lengths must lie in [0, T = %d], got %s" % (T, il.tolist()))
    model = check_ngram(ngram, V, blank)
    ng_w = check_ngram_weight(model, ngram_weight)
    fusion = check_lm_args(lm, V, lm_weight, length_bonus, lm_bos, lm_token_map, ngram=model is not None)
    graph = check_context(context, V, blank)
    if not log_probs.is_cuda:
        raise RuntimeError("edgedict_b200 ctc beam_search needs CUDA log_probs (got a %s tensor); there is no CPU path"
                           % log_probs.device)
    dev = log_probs.device
    key = (B, T, V, W, N, blank, dev, lm_cache_key(fusion), context_cache_key(graph),
           ngram_cache_key(model, ng_w, length_bonus))
    eng = _beam_engines.get(key)
    if eng is None:
        _beam_engines.clear()                                  # one resident program is enough
        eng = _beam_engines[key] = CTCBeamEngine(B, T, V, W, blank, lm=lm, lm_weight=lm_weight,
                                                 length_bonus=length_bonus, lm_bos=lm_bos, lm_token_map=lm_token_map,
                                                 device=dev, nbest=N, context=graph, ngram=model,
                                                 ngram_weight=ng_w)
    lens = torch.empty(B, dtype=torch.int32, pin_memory=True)
    lens.copy_(il)
    with torch.no_grad():
        if N:
            return nbest_lists(eng.run(log_probs, lens.to(dev, non_blocking=True)), B, N, T)
        ids, nlogp = eng.run(log_probs, lens.to(dev, non_blocking=True))
        ids = ids.cpu().numpy()
    return [row[row >= 0].astype("int64") for row in ids], nlogp.clone()


class CTCStreamDecoder:
    """Streaming CTC decoding of a ``CTCEncoder`` with ``PytorchStreamDecoder``'s surface (rnnt/stream.py:15-120):
    ``reset()``, ``decode(frame) -> str``, ``flush() -> str``, ``reset_profile()``, the ``encoder_elapsed`` /
    ``decoder_elapsed`` / ``joint_elapsed`` lists and ``tokenizer``.  ``decode`` runs one persistent kernel launch per
    chunk (one stream) and returns the text of the ids that became final in that chunk, ``'</w>'`` turned into a space.

    Greedy (``beam_width=None``, stream_engine.CTCStreamEngine): the ids of all chunks together are
    ``CTCEncoder.greedy_decode``'s on the concatenated frames (a token held across a chunk boundary is emitted once), and
    ``flush()`` returns ``""``.  Beam search (``beam_width`` = W, stream_engine.CTCStreamBeamEngine): a chunk's text is
    the common prefix of all live prefixes that became final in it, never revised; ``flush()`` returns the rest of the
    best prefix, and decoding goes on from it.  ``lm``, ``lm_weight``, ``length_bonus``, ``lm_bos`` and
    ``lm_token_map`` fuse the reference's LSTM LM as ``CTCEncoder.beam_search`` does; ``max_pending`` bounds the
    uncommitted tokens a prefix may hold before the beam collapses to its best prefix.  ``context`` (an
    edgedict_b200.context.ContextGraph over the model's vocabulary and blank; beam search only) biases the search as
    in ``CTCEncoder.beam_search``: each prefix carries its phrase-automaton state across chunks and commits, and the
    text of ``decode`` plus ``flush`` is that of the offline biased best prefix.

    ``transform`` maps a chunk of audio to log-mel features [1, F, n] (the reference's feature transform), on the host
    before each chunk; when it is build_batch_transform's test module (a BatchTransform), ``decode`` uploads the
    window's audio instead and the engine computes those features in its launch, bit for bit what the module gives the
    window (``frames_per_chunk`` is then ignored: the first window builds the program);
    ``tokenizer`` is the reference's HuggingFaceTokenizer (``tokenizer.tokenizer.id_to_token``).  A chunk whose frame
    count differs from the previous one's (a short last chunk), or weights that moved (``.to()``, an optimizer's flat
    bucket), rebuild the program and carry the state (the beam included) over; only ``reset()`` starts a new utterance.
    Chunks must hold an even number of frames before each time reduction.  Every argument is checked before any device
    work."""

    def __init__(self, model, transform, tokenizer, device="cuda", frames_per_chunk=None, *, beam_width=None, lm=None,
                 lm_weight=0.0, length_bonus=0.0, lm_bos=1, lm_token_map=None, max_pending=64, context=None):
        import numbers
        from .context import check_context
        from .rnnt.models import CTCEncoder
        from .stream_engine import BEAM_MAX_W, check_lm_args, check_stream_shape
        if not isinstance(model, CTCEncoder):
            raise TypeError("CTCStreamDecoder decodes a CTCEncoder, got %s" % type(model).__name__)
        self._beam = None
        if beam_width is not None:
            if isinstance(beam_width, bool) or not isinstance(beam_width, numbers.Integral):
                raise TypeError("beam_width must be an integer or None, got %r" % (beam_width,))
            W, V = int(beam_width), model.tovocab[0].weight.shape[0]
            if not 1 <= W <= BEAM_MAX_W:
                raise ValueError("beam_width must be in [1, %d], got %d" % (BEAM_MAX_W, W))
            if W * V >= 2 ** 31:
                raise ValueError("beam_width x V must stay below 2^31, got %d x %d" % (W, V))
            check_lm_args(lm, V, lm_weight, length_bonus, lm_bos, lm_token_map)
            check_context(context, V, model.blank)
            P = operator.index(max_pending)
            if frames_per_chunk is not None:
                _, _, T = check_stream_shape(model.model, 1, frames_per_chunk)
                if P < T:
                    raise ValueError("max_pending (%d) must be at least the encoder frames per chunk (%d)" % (P, T))
            self._beam = dict(W=W, lm=lm, lm_weight=lm_weight, length_bonus=length_bonus, lm_bos=lm_bos,
                              lm_token_map=lm_token_map, max_pending=P, context=context)
        elif lm is not None or lm_weight != 0.0 or length_bonus != 0.0 or lm_token_map is not None:
            raise ValueError("lm, lm_weight, length_bonus and lm_token_map need beam_width")
        elif context is not None:
            raise ValueError("context needs beam_width: greedy decoding has no contextual biasing")
        self.device = torch.device(device)
        self.transform, self.tokenizer = transform, tokenizer
        model.eval()
        model.to(self.device)
        self.model = model
        self._engine = None
        self._frames = frames_per_chunk
        from .rnnt.features import BatchTransform
        self._device_fe = isinstance(transform, BatchTransform)    # the features run inside the decode launch
        self.reset_profile()
        if frames_per_chunk is not None and not self._device_fe:
            self._build(operator.index(frames_per_chunk))

    def reset_profile(self):
        self.encoder_elapsed = []
        self.decoder_elapsed = []
        self.joint_elapsed = []

    def _build(self, n):
        from .stream_engine import CTCStreamBeamEngine, CTCStreamEngine
        st = self._engine.state() if self._engine is not None else None
        fe = dict(frontend=self.transform, samples_per_chunk=n) if self._device_fe else {}
        frames = None if self._device_fe else n                # n: the window's samples with a device front end
        if self._beam is None:
            self._engine = CTCStreamEngine(self.model, 1, frames, blank=self.model.blank, state=st, **fe)
        else:
            b = dict(self._beam)
            self._engine = CTCStreamBeamEngine(self.model, 1, frames, b.pop("W"), blank=self.model.blank, state=st,
                                               **b, **fe)
        self._frames = n

    def _text(self, ids, counts):
        return "".join(self.tokenizer.tokenizer.id_to_token(int(k)).replace('</w>', ' ')
                       for k in ids[0, :int(counts[0])].tolist())

    @torch.no_grad()
    def reset(self):
        if self._engine is not None:
            self._engine.reset()

    @torch.no_grad()
    def decode(self, frame):
        import time
        from .stream_engine import param_fingerprint
        start = time.time()
        if self._device_fe:                                        # the window's audio, transformed in the launch
            xs = torch.as_tensor(frame).to(self.device, torch.float32).reshape(1, -1)
        else:
            xs = self.transform(frame).transpose(1, 2).to(self.device, non_blocking=True)   # [1, n, F] log-mel
        if self._engine is None or xs.shape[1] != self._frames or \
                self._engine.fingerprint != param_fingerprint(self.model):
            self._build(xs.shape[1])
        ids, counts = self._engine.step(xs)                        # one D2H per chunk
        self.encoder_elapsed.append(time.time() - start)
        return self._text(ids, counts)

    @torch.no_grad()
    def flush(self):
        """The rest of the best prefix (beam search), after which decoding continues from it; ``""`` for greedy
        decoding, whose every id is final when its chunk is decoded."""
        if self._beam is None or self._engine is None:
            return ""
        ids, counts, _ = self._engine.flush()
        return self._text(ids, counts)
