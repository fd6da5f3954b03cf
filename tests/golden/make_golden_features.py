"""Generates tests/golden/features_tiny.npz with the REFERENCE's own feature transforms (only possible where its
sources are):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_features.py

* module: ``rnnt.transforms.build_transform`` of $EDGEDICT_REFERENCE on torch CPU fp32, applied per utterance as
  rnnt/dataset.py:103 does (``transform(x[:1])[0].T`` on the unpadded waveform) and collated by its ``seq_collate``;
* input: B = 3 waveforms of unequal lengths (one a multiple of the hop, so logfbank's frame mask bites);
* configurations: every feature type with and without deltas, each at (n_fft, downsample, pad_to_divisible) =
  (512, 1, True), (400, 3, True) and (512, 3, False), win 400, hop 200, feature_size 20, FilterbankFeatures' dither 0;
  and two train transforms with SpecAugment masks, drawn after ``random.seed(MASK_SEED)``.

Two stand-ins let the reference import and run with this torch:
* ``librosa`` is not installed.  Only FilterbankFeatures calls it (``librosa.filters.mel``, Slaney scale, Slaney area
  normalisation); torchaudio's ``melscale_fbanks(norm='slaney', mel_scale='slaney')`` computes the same published
  formula, the substitution tests/test_oracle_features.py pins.
* torch now requires ``return_complex`` in ``torch.stft``; rnnt/features.py:101-123 expects the old real [..., 2]
  return, so a call without it gets ``view_as_real(stft(..., return_complex=True))``.

The committed fixture is what the tests see; nothing at test time reads the reference.
"""
import os
import random
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LENS = (3517, 2800, 2003)
SIZE, WIN, HOP = 20, 400, 200
GEOMS = [(512, 1, True), (400, 3, True), (512, 3, False)]
CONFIGS = [(ft, delta) + g for ft in ("logfbank", "mfcc", "melspec") for delta in (False, True) for g in GEOMS]
MASKED = [dict(ft="mfcc", delta=True, n_fft=512, ds=3, ptd=True, T_mask=3, T_num_mask=2, F_mask=8, F_num_mask=2),
          dict(ft="logfbank", delta=False, n_fft=400, ds=1, ptd=True, T_mask=4, T_num_mask=2, F_mask=5, F_num_mask=1)]
MASK_SEED = 1234


def tag(ft, delta, n_fft, ds, ptd):
    return "%s.d%d.n%d.ds%d.p%d" % (ft, int(delta), n_fft, ds, int(ptd))


def reference_build_transform():
    if "librosa" not in sys.modules:
        import torchaudio
        lib = sys.modules["librosa"] = types.ModuleType("librosa")
        lib.filters = types.SimpleNamespace(mel=lambda sr, n_fft, n_mels=128, fmin=0.0, fmax=None: (
            torchaudio.functional.melscale_fbanks(1 + n_fft // 2, float(fmin), float(fmax or sr / 2.0), n_mels, sr,
                                                  norm="slaney", mel_scale="slaney").T.numpy()))
        stft = torch.stft

        def old_stft(*a, **kw):
            if "return_complex" in kw:
                return stft(*a, **kw)
            return torch.view_as_real(stft(*a, return_complex=True, **kw))
        torch.stft = old_stft
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    from rnnt.transforms import build_transform  # (the reference)
    from rnnt.dataset import zero_pad_concat  # (the reference)
    return build_transform, zero_pad_concat


def per_utterance(tf, x, zero_pad_concat):
    feats = [tf(x[b:b + 1, :n].clone())[0].T for b, n in enumerate(LENS)]
    return zero_pad_concat(feats).numpy(), np.array([len(f) for f in feats], dtype=np.int32)


def main():
    build_transform, zero_pad_concat = reference_build_transform()
    g = torch.Generator().manual_seed(5)
    t = torch.arange(max(LENS)) / 16000.0
    x = torch.zeros(len(LENS), max(LENS))
    for b, n in enumerate(LENS):
        x[b, :n] = (0.1 * torch.randn(max(LENS), generator=g) + 0.4 * torch.sin(2 * np.pi * 300.0 * (b + 1) * t))[:n]
    save = dict(x=x.numpy(), lens=np.array(LENS, dtype=np.int32), size=np.int64(SIZE), win=np.int64(WIN),
                hop=np.int64(HOP), mask_seed=np.int64(MASK_SEED))
    for ft, delta, n_fft, ds, ptd in CONFIGS:
        _, test, input_size = build_transform(ft, SIZE, n_fft=n_fft, win_length=WIN, hop_length=HOP, delta=delta,
                                              downsample=ds, pad_to_divisible=ptd)
        if ft == "logfbank":
            test[0].dither = 0
        k = tag(ft, delta, n_fft, ds, ptd)
        save[k + ".xs"], save[k + ".xlen"] = per_utterance(test, x, zero_pad_concat)
        save[k + ".input_size"] = np.int64(input_size)
        print(k, save[k + ".xs"].shape, save[k + ".xlen"])
    for i, c in enumerate(MASKED):
        train, _, _ = build_transform(c["ft"], SIZE, n_fft=c["n_fft"], win_length=WIN, hop_length=HOP,
                                      delta=c["delta"], downsample=c["ds"], pad_to_divisible=c["ptd"],
                                      T_mask=c["T_mask"], T_num_mask=c["T_num_mask"], F_mask=c["F_mask"],
                                      F_num_mask=c["F_num_mask"])
        if c["ft"] == "logfbank":
            train[0].dither = 0
        random.seed(MASK_SEED)
        save["masked%d.xs" % i], save["masked%d.xlen" % i] = per_utterance(train, x, zero_pad_concat)
        save["masked%d.cfg" % i] = np.array([c["ft"], int(c["delta"]), c["n_fft"], c["ds"], int(c["ptd"]), c["T_mask"],
                                            c["T_num_mask"], c["F_mask"], c["F_num_mask"]]).astype(str)
        print("masked%d" % i, c["ft"], save["masked%d.xs" % i].shape)
    np.savez_compressed(os.path.join(HERE, "features_tiny.npz"), **save)


if __name__ == "__main__":
    main()
    print("features_tiny.npz", os.path.getsize(os.path.join(HERE, "features_tiny.npz")) // 1024, "KiB")
