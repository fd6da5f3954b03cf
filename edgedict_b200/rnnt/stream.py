"""H100-native mirror of the reference's streaming decoder interface (rnnt/stream.py:15-120).

``PytorchStreamDecoder(FLAGS)`` keeps the reference's attributes and methods -- ``reset()``,
``decode(frame) -> str``, ``reset_profile()``, ``encoder_elapsed / decoder_elapsed /
joint_elapsed``, ``tokenizer`` -- so ``stream.py`` / ``youtube_live.py`` /
``cli/openvino_wav_inference.py`` drive it unchanged, but ``decode`` is ONE persistent-kernel
launch per chunk (edgedict_b200/stream_engine.py) instead of a Python loop with a host sync per
encoder frame.  With ``beam_width`` it decodes by streaming beam search instead (optionally with a fused LSTM
language model): ``decode`` returns the text that became final in that chunk and ``flush()`` the rest.
The BPE tokenizer is a host-side component, taken from the caller (``tokenizer=``) or, like the reference, built
from FLAGS when the reference's ``rnnt.tokenizer`` is importable.  The feature transform runs on the device, in the
same launch as the decode, when ``transform`` is build_batch_transform's test module (a BatchTransform): ``decode``
then uploads the window of raw audio and the engine's front end computes, bit for bit, what that module gives the
window.  Any other ``transform`` (a callable mapping a window to [1, F, n] features, or, with ``transform=None``, the
reference's ``rnnt.transforms.build_transform`` from FLAGS) runs on the host before each chunk, as in the reference.
"""
import operator
import os
import time

import torch

from .features import BatchTransform
from .models import ResLayerNormGRU, Transducer, convert_lightning2normal
from .tokenizer import NUL, BOS, UNK
from ..context import check_context
from ..stream_engine import BEAM_MAX_W, GRUStreamBeamEngine, GRUStreamEngine, StreamBeamEngine, StreamEngine, \
    check_lm_args, check_max_symbols, param_fingerprint


class StreamTransducerDecoder:
    def reset_profile(self):
        self.encoder_elapsed = []
        self.decoder_elapsed = []
        self.joint_elapsed = []

    def reset(self):
        raise NotImplementedError()

    def decode(self, frame):
        raise NotImplementedError()


class PytorchStreamDecoder(StreamTransducerDecoder):
    """``beam_width=None`` decodes greedily, as the reference does.  With a beam width W, every chunk runs the streaming
    beam search of stream_engine.StreamBeamEngine (``merge``, ``lm``, ``lm_weight``, ``length_bonus``, ``lm_bos`` and
    ``lm_token_map`` as in Transducer.beam_search; ``max_pending`` caps the uncommitted tokens a hypothesis stores).
    ``decode`` then returns the text of the tokens that became final in that chunk: the common prefix of all live
    hypotheses, which no later audio can change, so returned text is never revised.  ``flush()`` returns the rest of
    the best hypothesis and continues decoding from it; call it at the end of an utterance or a segment.  Without a
    forced collapse (a suffix outgrowing ``max_pending``), everything ``decode`` returned plus ``flush()`` is the
    best hypothesis of Transducer.beam_search over the same encoder frames.  The beam does not apply the reference's
    ``<unk>`` rule, which belongs to greedy argmax decoding; Transducer.beam_search does not apply it either.

    ``context`` (an edgedict_b200.context.ContextGraph over the transducer's vocabulary, blank NUL; beam search only)
    biases the streaming beam towards its phrases, as Transducer.beam_search(context=...) biases the offline one: each
    hypothesis carries its phrase-automaton state across chunks and commits, so a phrase may straddle them, and the text
    of ``decode`` plus ``flush`` is that of the offline biased best hypothesis over the same encoder frames.  Every
    rebuilt engine (another chunk length, moved weights) takes the same graph and the carried states.

    ``max_symbols`` = K (1 to 16, greedy decoding only) lets each encoder frame emit up to K symbols: the frame repeats
    joint -> argmax (with the ``<unk>`` rule) -> predictor step until a blank or K non-blank tokens.

    A transducer with a GRU encoder (``Transducer(module_type='GRU')``; from FLAGS, ``enc_type='GRU'`` as
    cli/lightning.py --enc_type GRU trains it) streams through stream_engine.GRUStreamEngine / GRUStreamBeamEngine,
    greedily or by beam search, with the same ``decode`` / ``flush`` / ``max_symbols`` / beam and LM arguments.  The
    reference cannot stream such a model (its decode hands an LSTM's (h, c) to the GRU stack): this is an addition, not
    a mirror of rnnt/stream.py."""

    def __init__(self, FLAGS, transducer=None, transform=None, tokenizer=None, device="cuda",
                 frames_per_chunk=None, input_size=None, *, beam_width=None, merge=True, lm=None, lm_weight=0.0,
                 length_bonus=0.0, lm_bos=1, lm_token_map=None, max_pending=64, max_symbols=1, context=None):
        self._max_symbols = check_max_symbols(max_symbols)
        if beam_width is not None and self._max_symbols != 1:
            raise ValueError("max_symbols > 1 is a greedy decoding option; the beam search emits one symbol per frame")
        if beam_width is None and context is not None:
            raise ValueError("context needs beam_width: greedy decoding has no contextual biasing")
        self.FLAGS = FLAGS
        self.device = torch.device(device)
        if tokenizer is None:
            from rnnt.tokenizer import HuggingFaceTokenizer        # the reference's own host-side class
            tokenizer = HuggingFaceTokenizer(cache_dir='BPE-' + str(FLAGS.bpe_size), vocab_size=FLAGS.bpe_size)
            assert tokenizer.tokenizer is not None
        self.tokenizer = tokenizer
        if transform is None:
            from rnnt.transforms import build_transform             # log-mel front end (host side)
            _, transform, input_size = build_transform(
                feature_type=FLAGS.feature, feature_size=FLAGS.feature_size, n_fft=FLAGS.n_fft,
                win_length=FLAGS.win_length, hop_length=FLAGS.hop_length, delta=FLAGS.delta, cmvn=FLAGS.cmvn,
                downsample=FLAGS.downsample, pad_to_divisible=False, T_mask=FLAGS.T_mask,
                T_num_mask=FLAGS.T_num_mask, F_mask=FLAGS.F_mask, F_num_mask=FLAGS.F_num_mask)
        elif isinstance(transform, BatchTransform):
            input_size = transform.input_size if input_size is None else input_size
        elif input_size is None and transducer is None:
            # a caller-supplied transform: the feature width follows the flagfile (rnnt/transforms.py:30-51)
            input_size = FLAGS.feature_size * FLAGS.downsample * (3 if getattr(FLAGS, "delta", False) else 1)
        self.transform = transform
        self._device_fe = isinstance(transform, BatchTransform)    # the features run inside the decode launch
        if transducer is None:
            logdir = os.path.join('logs', FLAGS.name)
            model_path = os.path.join(logdir, 'models', FLAGS.model_name)
            if not os.path.exists(model_path):
                model_path = os.path.join(logdir, FLAGS.model_name)
            checkpoint = torch.load(model_path, lambda storage, loc: storage)
            transducer = Transducer(
                vocab_embed_size=FLAGS.vocab_embed_size, vocab_size=self.tokenizer.vocab_size,
                input_size=input_size, enc_hidden_size=FLAGS.enc_hidden_size, enc_layers=FLAGS.enc_layers,
                enc_dropout=FLAGS.enc_dropout, enc_proj_size=FLAGS.enc_proj_size,
                dec_hidden_size=FLAGS.dec_hidden_size, dec_layers=FLAGS.dec_layers, dec_dropout=FLAGS.dec_dropout,
                dec_proj_size=FLAGS.dec_proj_size, joint_size=FLAGS.joint_size,
                module_type=getattr(FLAGS, "enc_type", "LSTM"), output_loss=False)
            transducer.load_state_dict(convert_lightning2normal(checkpoint)['model'])
        transducer.eval()
        transducer.to(self.device)
        self.encoder, self.decoder, self.joint = transducer.encoder, transducer.decoder, transducer.joint
        self._transducer = transducer
        self._unk = self._token_id('<unk>')
        self._beam = None
        if beam_width is not None:
            W = operator.index(beam_width)
            if not 1 <= W <= BEAM_MAX_W:
                raise ValueError("beam_width must be in [1, %d], got %d" % (BEAM_MAX_W, W))
            check_lm_args(lm, transducer.joint.joint[2].weight.shape[0], lm_weight, length_bonus, lm_bos, lm_token_map)
            check_context(context, transducer.joint.joint[2].weight.shape[0], NUL)
            self._beam = dict(W=W, merge=bool(merge), lm=lm, lm_weight=lm_weight, length_bonus=length_bonus,
                              lm_bos=lm_bos, lm_token_map=lm_token_map, max_pending=operator.index(max_pending),
                              context=context)
        self._engine = None
        self._frames = frames_per_chunk
        self.reset_profile()
        if frames_per_chunk is not None and not self._device_fe:   # a device front end builds for its first window
            self._build(frames_per_chunk)

    def _token_id(self, token):
        try:
            i = self.tokenizer.tokenizer.token_to_id(token)
            return UNK if i is None else int(i)
        except Exception:
            return UNK

    def _build(self, n):
        # a different chunk length (a short last chunk, a changed block size) or re-homed weights need a new phase
        # program, NOT a new utterance: the recurrent state moves over (rnnt/stream.py:94-120 carries it across
        # arbitrary chunk lengths); only reset() starts from the primed zero state.  n counts frames, or with a device
        # front end the window's samples.
        st = self._engine.state() if self._engine is not None else None
        gru = isinstance(self.encoder.lstm, ResLayerNormGRU)
        fe = dict(frontend=self.transform, samples_per_chunk=n) if self._device_fe else {}
        frames = None if self._device_fe else n
        if self._beam is None:
            self._engine = (GRUStreamEngine if gru else StreamEngine)(self._transducer, 1, frames, unk_id=self._unk,
                                                                      blank=NUL, state=st,
                                                                      max_symbols=self._max_symbols, **fe)
        else:
            self._engine = (GRUStreamBeamEngine if gru else StreamBeamEngine)(self._transducer, 1, frames, blank=NUL,
                                                                              state=st, **self._beam, **fe)
        self._frames = n

    @torch.no_grad()
    def reset(self):
        if self._engine is not None:
            self._engine.reset()

    @torch.no_grad()
    def decode(self, frame):
        start = time.time()
        if self._device_fe:                                         # the window's audio, transformed in the launch
            xs = torch.as_tensor(frame).to(self.device, torch.float32).reshape(1, -1)
        else:
            xs = self.transform(frame).transpose(1, 2).to(self.device, non_blocking=True)   # [1, n, F], stream.py:96
        if self._engine is None or xs.shape[1] != self._frames or \
                self._engine.fingerprint != param_fingerprint(self._transducer):
            self._build(xs.shape[1])
        if self._beam is not None:
            ids, counts = self._engine.step(xs)                     # one D2H per chunk
            self.encoder_elapsed.append(time.time() - start)
            self.joint_elapsed += [0.0] * self._engine.n_out      # fused into the chunk kernel
            return self._text(ids[0, :int(counts[0])].tolist())
        ids = self._engine.step(xs)[0].tolist()                     # one D2H per chunk
        self.encoder_elapsed.append(time.time() - start)
        tokens = []
        for pred in ids:
            self.joint_elapsed.append(0.0)                          # fused into the chunk kernel
            if pred != NUL:
                self.decoder_elapsed.append(0.0)
                seq = self.tokenizer.tokenizer.id_to_token(pred)
                tokens.append(seq.replace('</w>', ' '))
        return "".join(tokens)

    def _text(self, ids):
        tokens = []
        for pred in ids:
            self.decoder_elapsed.append(0.0)
            tokens.append(self.tokenizer.tokenizer.id_to_token(pred).replace('</w>', ' '))
        return "".join(tokens)

    @torch.no_grad()
    def flush(self):
        """Beam search: the text of the best hypothesis' tokens not yet returned by ``decode``; decoding continues
        from that hypothesis.  Greedy decoding returns every token at once, so there is nothing to flush: ""."""
        if self._beam is None or self._engine is None:
            return ""
        ids, counts, _ = self._engine.flush()
        return self._text(ids[0, :int(counts[0])].tolist())
