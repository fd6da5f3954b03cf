"""fp64 numpy restatement of every feature transform the reference's ``build_transform`` builds (rnnt/transforms.py:
165-203), applied per utterance and collated as the reference's data loader does (TEST INFRASTRUCTURE; the product
path is edgedict_b200/csrc/frontend.cu).

* ``mfcc``: torchaudio.transforms.MFCC(n_mfcc, log_mels=True, melkwargs={n_fft, win_length, hop_length}) -- the
  power spectrogram of torch.stft(center=True, reflect) with a periodic Hann window of win_length centred in n_fft, the
  HTK mel filterbank (norm=None, n_mels=128, f_max = sr/2), log(mel + 1e-6), the orthonormal DCT-II.
* ``melspec``: torchaudio.transforms.MelSpectrogram(n_mels=feature_size, ...): the same spectrogram and mel steps, no log.
* ``logfbank``: oracle/features_np.filterbank_features (the reference's FilterbankFeatures, dither 0).
* ``delta``: CatDeltas (transforms.py:10-16): torchaudio.functional.compute_deltas twice (window 5, replicate edge).
* per utterance: rnnt/dataset.py:103 transforms x[b, :L_b] alone; seq_collate / zero_pad_concat (dataset.py:202-240)
  pads the [T_b, C] features with zeros and returns xlen = T_b.

PINNED against torchaudio in tests/test_features_batch_host.py (where it is importable) and against the reference's
own transform in tests/golden/features_tiny.npz.
"""
import random

import numpy as np

from oracle import features_np as F

SR = 16000
MFCC_N_MELS = 128                     # torchaudio's default: build_transform's melkwargs do not set n_mels


def hann_periodic(win_length):
    """torch.hann_window(win_length) (periodic=True, torchaudio's window_fn)."""
    n = np.arange(win_length, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * n / win_length)


def htk_mel_filterbank(n_fft, n_mels, sr=SR, f_min=0.0, f_max=None):
    """torchaudio.functional.melscale_fbanks(1 + n_fft//2, f_min, f_max, n_mels, sr, norm=None, mel_scale='htk')
    -> fp64 [1 + n_fft//2, n_mels]."""
    f_max = sr / 2.0 if f_max is None else f_max
    freqs = np.linspace(0.0, sr // 2, 1 + n_fft // 2)
    hz_to_mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)
    m = np.linspace(hz_to_mel(f_min), hz_to_mel(f_max), n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m / 2595.0) - 1.0)
    f_diff = np.diff(f_pts)
    slopes = f_pts[None, :] - freqs[:, None]
    return np.maximum(0.0, np.minimum(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:]))


def create_dct(n_mfcc, n_mels):
    """torchaudio.functional.create_dct(n_mfcc, n_mels, norm='ortho') -> fp64 [n_mels, n_mfcc]."""
    n = np.arange(n_mels, dtype=np.float64)
    k = np.arange(n_mfcc, dtype=np.float64)[:, None]
    dct = np.cos(np.pi / n_mels * (n + 0.5) * k)
    dct[0] *= 1.0 / np.sqrt(2.0)
    return (dct * np.sqrt(2.0 / n_mels)).T


def power_spectrogram(x, n_fft, win_length, hop_length):
    """torchaudio Spectrogram(power=2) of x [B, L] -> [B, 1 + n_fft//2, 1 + L//hop]."""
    return F.stft_power(np.asarray(x, np.float64), n_fft, hop_length, win_length, hann_periodic(win_length))


def melspec(x, n_mels, n_fft=400, win_length=None, hop_length=None):
    win_length = win_length or n_fft
    hop_length = hop_length or win_length // 2
    p = power_spectrogram(x, n_fft, win_length, hop_length)
    return np.einsum("km,bkf->bmf", htk_mel_filterbank(n_fft, n_mels), p)


def mfcc(x, n_mfcc, n_fft=400, win_length=None, hop_length=None):
    if n_mfcc > MFCC_N_MELS:
        raise ValueError("Cannot select more MFCC coefficients than # mel bins")
    mel = np.log(melspec(x, MFCC_N_MELS, n_fft, win_length, hop_length) + 1e-6)
    return np.einsum("mc,bmf->bcf", create_dct(n_mfcc, MFCC_N_MELS), mel)


def logfbank(x, n_filt, n_fft=512, win_length=400, hop_length=200):
    return F.filterbank_features(x, win_length=win_length, hop_length=hop_length, n_fft=n_fft, n_filt=n_filt,
                                 dtype=np.float64)


def compute_deltas(feat, win_length=5):
    """torchaudio.functional.compute_deltas on [B, C, F]: replicate padding along time."""
    n = (win_length - 1) // 2
    denom = n * (n + 1) * (2 * n + 1) / 3
    Fn = feat.shape[-1]
    out = np.zeros_like(feat, dtype=np.float64)
    for k in range(-n, n + 1):
        out += k * feat[..., np.clip(np.arange(Fn) + k, 0, Fn - 1)]
    return out / denom


def cat_deltas(feat):
    d1 = compute_deltas(feat)
    return np.concatenate([feat, d1, compute_deltas(d1)], axis=1)


def transform(x, feature_type, feature_size, n_fft=512, win_length=400, hop_length=200, delta=False, downsample=1,
              pad_to_divisible=True):
    """build_transform(...)[1] (the test transform) on x [B, L] -> [B, C, T] in the reference's layout."""
    args = dict(n_fft=n_fft, win_length=win_length, hop_length=hop_length)
    if feature_type == "mfcc":
        f = mfcc(x, feature_size, **args)
    elif feature_type == "melspec":
        f = melspec(x, feature_size, **args)
    elif feature_type == "logfbank":
        f = logfbank(x, feature_size, **args)
    else:
        raise NotImplementedError(feature_type)
    if delta:
        f = cat_deltas(f)
    if downsample > 1:
        f = F.downsample(f, downsample, pad_to_divisible)
    return f


def seq_collate(feats):
    """zero_pad_concat of per-utterance [T_b, C] features -> ([B, T_max, C], xlen int32)."""
    xlen = np.array([len(f) for f in feats], dtype=np.int32)
    xs = np.zeros((len(feats), xlen.max()) + feats[0].shape[1:], dtype=np.float64)
    for b, f in enumerate(feats):
        xs[b, :len(f)] = f
    return xs, xlen


def batch_transform(x, lens, feature_type, feature_size, **kw):
    """The reference's data path: transform(x[b:b+1, :L_b])[0].T per utterance (dataset.py:103), then seq_collate."""
    return seq_collate([transform(x[b:b + 1, :n], feature_type, feature_size, **kw)[0].T for b, n in enumerate(lens)])


def reference_spans(T, n_ch, T_mask=0, T_num_mask=0, F_mask=0, F_num_mask=0):
    """The python `random` draws of TimeMasking then FrequencyMasking (transforms.py:53-147) when the dataset
    transforms each utterance alone, utterance after utterance: ([B][T_num_mask][2], [B][F_num_mask][2])."""
    tsp, fsp = [], []
    for Tb in T:
        row = []
        if T_mask > 0 and T_num_mask > 0:
            for _ in range(T_num_mask):                 # TimeMasking.forward on [1, n_ch, T_b]
                start = random.randrange(0, Tb)
                end = start + random.randrange(0, T_mask)
                row.append((start, end))
        tsp.append(row)
        row = []
        if F_mask > 0 and F_num_mask > 0:
            for _ in range(F_num_mask):                 # FrequencyMasking.forward on [1, n_ch, T_b]
                start = random.randrange(0, n_ch)
                end = start + random.randrange(0, F_mask)
                row.append((start, end))
        fsp.append(row)
    return tsp, fsp


def apply_spans(xs, tsp, fsp):
    """Zero the spans in the collated [B, T, C] features (masked_fill with 0 on each utterance)."""
    xs = xs.copy()
    for b in range(xs.shape[0]):
        for s, e in tsp[b]:
            xs[b, s:e, :] = 0
        for s, e in fsp[b]:
            xs[b, :, s:e] = 0
    return xs


def frame_power(x, n_fft, win_length, hop_length):
    """Total power sum_k P[k, f] of every frame of x [B, L] (periodic window) -> [B, 1 + L//hop]."""
    return power_spectrogram(x, n_fft, win_length, hop_length).sum(axis=1)
