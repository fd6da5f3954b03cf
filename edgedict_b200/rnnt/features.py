"""H100-native mirror of the reference's log-mel front end (``rnnt/features.py`` + the feature part of
``rnnt/transforms.py``): same class names, constructor arguments and output layouts, arithmetic in
csrc/frontend.cu (pre-emphasis / reflect padding, direct-DFT GEMM, power, mel GEMM, log + frame stacking).

The mel filterbank table is generated here with the Slaney formula librosa 0.7.2 implements
(``librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)``, rnnt/features.py:76-80) -- librosa itself is not a
dependency.  Buffers keep the reference's names and shapes (``fb`` [1, n_filt, n_fft/2+1], ``window`` [win_length]).
"""
import math

import numpy as np
import torch
from torch import nn

from .. import ops


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(sr, n_fft, n_mels, fmin=0.0, fmax=None):
    """Slaney-scale, area-normalised triangular filters (float32 [n_mels, n_fft//2 + 1])."""
    fmax = sr / 2.0 if fmax is None else fmax
    nb = 1 + n_fft // 2
    freqs = np.linspace(0.0, sr / 2.0, nb)
    edges = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    width = np.diff(edges)
    ramps = edges[:, None] - freqs[None, :]
    rising = -ramps[:-2] / width[:-1, None]
    falling = ramps[2:] / width[1:, None]
    w = np.maximum(0.0, np.minimum(rising, falling))
    w *= (2.0 / (edges[2:] - edges[:-2]))[:, None]
    return w.astype(np.float32)


class FilterbankFeatures(nn.Module):
    """rnnt/features.py:33-176 (window='hann', normalize='none'; the per-feature normalisations are not used by
    any BASELINE flagfile).  forward(x [B, L]) -> [B, n_filt, 1 + L//hop]; `dither` adds N(0, dither^2) noise in
    place like the reference (features.py:133-134) -- set 0 for reproducible features."""

    def __init__(self, sample_rate=16000, win_length=320, hop_length=160, n_fft=512, window="hann",
                 normalize="none", log=True, dither=1e-5, pad_to=0, max_duration=16.7, preemph=0.97, n_filt=64,
                 f_min=0, f_max=None):
        super().__init__()
        if window != "hann" or normalize not in ("none", None) or pad_to != 0:
            raise NotImplementedError("edgedict_b200 front end: window='hann', normalize='none', pad_to=0")
        self.win_length, self.hop_length = win_length, hop_length
        self.n_fft = n_fft or 2 ** math.ceil(math.log2(win_length))
        self.log, self.dither, self.n_filt, self.preemph = log, dither, n_filt, preemph
        f_max = f_max or sample_rate / 2
        self.register_buffer("fb", torch.tensor(mel_filterbank(sample_rate, self.n_fft, n_filt, f_min, f_max)).unsqueeze(0))
        self.register_buffer("window", torch.hann_window(win_length, periodic=False))
        # windowed DFT basis [n_fft, 2*nbins]: (w cos | -w sin), window centred in n_fft as torch.stft pads it
        n = np.arange(self.n_fft, dtype=np.float64)[:, None]
        k = np.arange(self.n_fft // 2 + 1, dtype=np.float64)[None, :]
        w = np.zeros(self.n_fft)
        left = (self.n_fft - win_length) // 2
        w[left:left + win_length] = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) / (win_length - 1))
        ang = 2.0 * np.pi * ((n * k) % self.n_fft) / self.n_fft
        basis = np.concatenate([w[:, None] * np.cos(ang), -w[:, None] * np.sin(ang)], axis=1)
        self.register_buffer("dft_basis", torch.tensor(basis, dtype=torch.float32), persistent=False)
        self.register_buffer("fb_t", self.fb[0].t().contiguous(), persistent=False)
        max_length = 1 + math.ceil((max_duration * sample_rate - win_length) / hop_length)
        self.max_length = max_length + (16 - (max_length % 16))

    def get_seq_len(self, seq_len):
        return torch.ceil(seq_len.float() / self.hop_length).int()

    def _features(self, x, n_stack, pad_to_divisible=True):
        if self.dither > 0:
            x += self.dither * torch.randn_like(x)
        return ops.logmel_frontend(x.contiguous(), self.dft_basis, self.fb_t, self.n_fft, self.hop_length, self.n_filt,
                                   n_stack, self.preemph, self.log, pad_to_divisible)

    @torch.no_grad()
    def forward(self, x):
        return self._features(x, 1).transpose(1, 2)


class Downsample(nn.Module):
    """rnnt/transforms.py:30-51 on [B, C, F] -> [B, C*n_frame, ceil(F/n_frame)] (a strided copy; when it directly
    follows FilterbankFeatures, LogMelFrontend does both in one pass)."""

    def __init__(self, n_frame, pad_to_divisible=True):
        super().__init__()
        self.n_frame, self.pad_to_divisible = n_frame, pad_to_divisible

    @torch.no_grad()
    def forward(self, feat):
        feat = feat.transpose(1, 2)
        B, F, C = feat.shape
        if self.pad_to_divisible:
            feat = nn.functional.pad(feat, [0, 0, 0, (self.n_frame - F % self.n_frame) % self.n_frame, 0, 0])
        else:
            feat = feat[:, :F - F % self.n_frame]
        return feat.reshape(B, -1, C * self.n_frame).transpose(1, 2)


class LogMelFrontend(nn.Module):
    """build_transform('logfbank', feature_size, downsample=n) of rnnt/transforms.py:165-203 (test transform) fused:
    waveform [B, L] -> model input [B, T, feature_size*n] in one pass over the frames."""

    def __init__(self, feature_size=80, n_fft=512, win_length=400, hop_length=200, downsample=3, pad_to_divisible=True,
                 dither=1e-5, **kw):
        super().__init__()
        self.fbank = FilterbankFeatures(n_filt=feature_size, n_fft=n_fft, win_length=win_length, hop_length=hop_length,
                                        dither=dither, **kw)
        self.downsample, self.pad_to_divisible = downsample, pad_to_divisible
        self.input_size = feature_size * downsample

    @torch.no_grad()
    def forward(self, x):
        return self.fbank._features(x, self.downsample, self.pad_to_divisible)


class _SpanMasking(nn.Module):
    """SpecAugment masking of rnnt/transforms.py:53-147 on the [B, C, T] feature layout.  The spans are drawn on the
    host with python's `random` in exactly the reference's order (per utterance, per mask: start = randrange(dim),
    end = start + randrange(max_width)), so `random.seed(s)` reproduces the reference's masks; they are applied by
    one kernel (eb_fe_mask) instead of a boolean mask tensor + masked_fill."""
    axis = 2

    def __init__(self, max_width, num_masks, use_mean=False):
        super().__init__()
        self.max_width, self.num_masks, self.use_mean = max_width, num_masks, use_mean

    @torch.no_grad()
    def forward(self, x):
        import random
        fill = float(x.mean()) if self.use_mean else 0.0
        dim = x.shape[self.axis]
        spans = []
        for _ in range(x.shape[0]):
            row = []
            for _ in range(self.num_masks):
                start = random.randrange(0, dim)
                row.append((start, start + random.randrange(0, self.max_width)))
            spans.append(row)
        if self.num_masks == 0:
            return x
        sp = torch.tensor(spans, dtype=torch.int32).to(x.device, non_blocking=True)
        out = x.contiguous().clone()                      # masked_fill is out of place in the reference
        return ops.fe_mask(out, sp, self.axis, fill)

    def __repr__(self):
        return "%s(max_width=%d,num_masks=%d,use_mean=%s)" % (self.__class__.__name__, self.max_width, self.num_masks,
                                                               self.use_mean)


class TimeMasking(_SpanMasking):
    """rnnt/transforms.py:102-147: `mask[i, :, start:end] = 1` on the last (time) axis."""
    axis = 2


class FrequencyMasking(_SpanMasking):
    """rnnt/transforms.py:53-99: `mask[i, start:end, :] = 1` on the channel axis."""
    axis = 1


def build_transform(feature_type, feature_size, n_fft=512, win_length=400, hop_length=200, delta=False, cmvn=False,
                    downsample=1, T_mask=0, T_num_mask=0, F_mask=0, F_num_mask=0, pad_to_divisible=True):
    """rnnt/transforms.py:165-203 for feature_type='logfbank' without deltas (every BASELINE flagfile); returns
    (transform_train, transform_test, input_size) producing the reference's [B, C, T] layout; the train transform
    appends the SpecAugment time / frequency masks exactly where the reference does (transforms.py:195-199)."""
    if feature_type != "logfbank" or delta:
        raise NotImplementedError("edgedict_b200 front end implements feature_type='logfbank', delta=False")
    mods = [FilterbankFeatures(n_filt=feature_size, n_fft=n_fft, win_length=win_length, hop_length=hop_length)]
    input_size = feature_size
    if downsample > 1:
        mods.append(Downsample(downsample, pad_to_divisible))
        input_size *= downsample
    test = nn.Sequential(*mods)
    train_mods = list(mods)
    if T_mask > 0 and T_num_mask > 0:
        train_mods.append(TimeMasking(T_mask, T_num_mask))
    if F_mask > 0 and F_num_mask > 0:
        train_mods.append(FrequencyMasking(F_mask, F_num_mask))
    train = nn.Sequential(*train_mods) if len(train_mods) > len(mods) else test
    return train, test, input_size
