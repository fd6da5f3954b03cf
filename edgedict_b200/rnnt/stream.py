"""H100-native mirror of the reference's streaming decoder interface (rnnt/stream.py:15-120).

``PytorchStreamDecoder(FLAGS)`` keeps the reference's attributes and methods -- ``reset()``,
``decode(frame) -> str``, ``reset_profile()``, ``encoder_elapsed / decoder_elapsed /
joint_elapsed``, ``tokenizer`` -- so ``stream.py`` / ``youtube_live.py`` /
``cli/openvino_wav_inference.py`` drive it unchanged, but ``decode`` is ONE persistent-kernel
launch per chunk (edgedict_b200/stream_engine.py) instead of a Python loop with a host sync per
encoder frame.  The feature transform and the BPE tokenizer are host-side components outside the
hot path: they are taken from the caller (``transform=``, ``tokenizer=``) or, like the reference,
built from FLAGS when the reference's ``rnnt.transforms`` / ``rnnt.tokenizer`` are importable.
"""
import os
import time

import torch

from .models import Transducer, convert_lightning2normal
from .tokenizer import NUL, BOS, UNK
from ..stream_engine import StreamEngine, param_fingerprint


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
    def __init__(self, FLAGS, transducer=None, transform=None, tokenizer=None, device="cuda",
                 frames_per_chunk=None, input_size=None):
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
        elif input_size is None and transducer is None:
            # a caller-supplied transform: the feature width follows the flagfile (rnnt/transforms.py:30-51)
            input_size = FLAGS.feature_size * FLAGS.downsample * (3 if getattr(FLAGS, "delta", False) else 1)
        self.transform = transform
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
                dec_proj_size=FLAGS.dec_proj_size, joint_size=FLAGS.joint_size, output_loss=False)
            transducer.load_state_dict(convert_lightning2normal(checkpoint)['model'])
        transducer.eval()
        transducer.to(self.device)
        self.encoder, self.decoder, self.joint = transducer.encoder, transducer.decoder, transducer.joint
        self._transducer = transducer
        self._unk = self._token_id('<unk>')
        self._engine = None
        self._frames = frames_per_chunk
        self.reset_profile()
        if frames_per_chunk is not None:
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
        # arbitrary chunk lengths); only reset() starts from the primed zero state
        st = self._engine.state() if self._engine is not None else None
        self._engine = StreamEngine(self._transducer, 1, n, unk_id=self._unk, blank=NUL, state=st)
        self._frames = n

    @torch.no_grad()
    def reset(self):
        if self._engine is not None:
            self._engine.reset()

    @torch.no_grad()
    def decode(self, frame):
        start = time.time()
        xs = self.transform(frame).transpose(1, 2)                  # [1, n, F] log-mel, as stream.py:96
        if self._engine is None or xs.shape[1] != self._frames or \
                self._engine.fingerprint != param_fingerprint(self._transducer):
            self._build(xs.shape[1])
        ids = self._engine.step(xs.to(self.device, non_blocking=True))[0].tolist()   # one D2H per chunk
        self.encoder_elapsed.append(time.time() - start)
        tokens = []
        for pred in ids:
            self.joint_elapsed.append(0.0)                          # fused into the chunk kernel
            if pred != NUL:
                self.decoder_elapsed.append(0.0)
                seq = self.tokenizer.tokenizer.id_to_token(pred)
                tokens.append(seq.replace('</w>', ' '))
        return "".join(tokens)
