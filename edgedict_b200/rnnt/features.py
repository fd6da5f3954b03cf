"""H100-native mirror of the reference's feature transforms (``rnnt/features.py`` + ``rnnt/transforms.py``, and the
torchaudio ``MFCC`` / ``MelSpectrogram`` modules ``build_transform`` builds): same class names, constructor arguments
and output layouts, arithmetic in csrc/frontend.cu (pre-emphasis / reflect padding, direct-DFT GEMM, power, mel GEMM,
log, DCT GEMM, deltas + frame stacking).

``build_batch_transform`` runs the same transforms per utterance over a padded batch: utterance b of length L_b gets
what the reference's transform computes on x[b, :L_b] alone, collated as rnnt/dataset.py's ``seq_collate`` pads it.

The mel filterbank table is generated here with the Slaney formula librosa 0.7.2 implements
(``librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)``, rnnt/features.py:76-80) -- librosa itself is not a
dependency.  Buffers keep the reference's names and shapes (``fb`` [1, n_filt, n_fft/2+1], ``window`` [win_length]).
``MFCC`` / ``MelSpectrogram`` use torchaudio's HTK filterbank (norm=None), periodic Hann window and orthonormal DCT-II,
generated here too, under torchaudio's buffer names (``window``, ``fb`` [n_fft/2+1, n_mels], ``dct_mat``).
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


def htk_mel_filterbank(sr, n_fft, n_mels, f_min=0.0, f_max=None):
    """torchaudio.functional.melscale_fbanks(n_fft//2 + 1, f_min, f_max, n_mels, sr, norm=None, mel_scale='htk'):
    triangular filters on the HTK mel scale, float32 [n_fft//2 + 1, n_mels], evaluated in fp32 in torchaudio's order so
    that the filters that cover no bin (many mels, a short FFT) are all zero exactly where torchaudio's are."""
    f_max = sr / 2.0 if f_max is None else f_max
    freqs = torch.linspace(0, sr // 2, 1 + n_fft // 2)
    m = torch.linspace(2595.0 * math.log10(1.0 + f_min / 700.0), 2595.0 * math.log10(1.0 + f_max / 700.0), n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.max(torch.zeros(1), torch.min(down, up))


def dct_ortho(n_mfcc, n_mels):
    """torchaudio.functional.create_dct(n_mfcc, n_mels, norm='ortho'): orthonormal DCT-II, float32 [n_mels, n_mfcc]."""
    n = np.arange(n_mels, dtype=np.float64)
    k = np.arange(n_mfcc, dtype=np.float64)[:, None]
    dct = np.cos(np.pi / n_mels * (n + 0.5) * k)
    dct[0] *= 1.0 / np.sqrt(2.0)
    dct *= np.sqrt(2.0 / n_mels)
    return np.ascontiguousarray(dct.T, dtype=np.float32)


def dft_basis(n_fft, win_length, periodic):
    """Windowed DFT basis [n_fft, 2*nbins] = (w cos | -w sin): a Hann window of win_length (periodic, as
    torch.hann_window's default, or symmetric) centred in n_fft as torch.stft pads it."""
    n = np.arange(n_fft, dtype=np.float64)[:, None]
    k = np.arange(n_fft // 2 + 1, dtype=np.float64)[None, :]
    w = np.zeros(n_fft)
    left = (n_fft - win_length) // 2
    w[left:left + win_length] = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) /
                                                   (win_length if periodic else win_length - 1))
    ang = 2.0 * np.pi * ((n * k) % n_fft) / n_fft
    basis = np.concatenate([w[:, None] * np.cos(ang), -w[:, None] * np.sin(ang)], axis=1)
    return torch.tensor(basis, dtype=torch.float32)


def _full_lengths(x):
    return torch.full((x.shape[0],), x.shape[1], dtype=torch.int32)


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
        self.register_buffer("dft_basis", dft_basis(self.n_fft, win_length, periodic=False), persistent=False)
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

    def _batch(self, x, lens, n_stack, delta, pad_to_divisible):
        if self.dither > 0:
            x = x + self.dither * torch.randn_like(x)
        return ops.fe_batch(x.contiguous(), lens, self.dft_basis, self.fb_t, self.n_fft, self.hop_length, n_stack,
                            self.preemph, take_log=self.log, use_mask=True, delta=delta,
                            pad_to_divisible=pad_to_divisible)

    @torch.no_grad()
    def forward(self, x):
        return self._features(x, 1).transpose(1, 2)


class Spectrogram(nn.Module):
    """The window holder of torchaudio.transforms.Spectrogram (periodic Hann, center=True, reflect padding, power 2);
    the arithmetic runs inside MelSpectrogram / MFCC."""

    def __init__(self, n_fft=400, win_length=None, hop_length=None):
        super().__init__()
        self.n_fft = n_fft
        self.win_length = win_length if win_length is not None else n_fft
        self.hop_length = hop_length if hop_length is not None else self.win_length // 2
        self.register_buffer("window", torch.hann_window(self.win_length))
        self.register_buffer("dft_basis", dft_basis(n_fft, self.win_length, periodic=True), persistent=False)


class MelScale(nn.Module):
    """The filterbank holder of torchaudio.transforms.MelScale (HTK scale, norm=None): ``fb`` [n_stft, n_mels]."""

    def __init__(self, n_mels=128, sample_rate=16000, f_min=0.0, f_max=None, n_stft=201):
        super().__init__()
        self.n_mels = n_mels
        self.register_buffer("fb", htk_mel_filterbank(sample_rate, 2 * (n_stft - 1), n_mels, f_min, f_max))


class MelSpectrogram(nn.Module):
    """torchaudio.transforms.MelSpectrogram for the arguments build_transform passes (rnnt/transforms.py:183-185):
    forward(x [B, L]) -> mel power [B, n_mels, 1 + L//hop], no log, no mask, no pre-emphasis.  CUDA only."""

    def __init__(self, sample_rate=16000, n_fft=400, win_length=None, hop_length=None, f_min=0.0, f_max=None,
                 n_mels=128):
        super().__init__()
        self.spectrogram = Spectrogram(n_fft, win_length, hop_length)
        self.mel_scale = MelScale(n_mels, sample_rate, f_min, f_max, n_fft // 2 + 1)
        self.n_fft, self.hop_length, self.n_mels = n_fft, self.spectrogram.hop_length, n_mels

    def _batch(self, x, lens, n_stack, delta, pad_to_divisible, dct=None):
        return ops.fe_batch(x.contiguous(), lens, self.spectrogram.dft_basis, self.mel_scale.fb, self.n_fft,
                            self.hop_length, n_stack, dct=dct, delta=delta, pad_to_divisible=pad_to_divisible)

    @torch.no_grad()
    def forward(self, x):
        return self._batch(x, _full_lengths(x), 1, False, True)[0].transpose(1, 2)


class MFCC(nn.Module):
    """torchaudio.transforms.MFCC(n_mfcc, log_mels=True, melkwargs) as build_transform builds it (rnnt/transforms.py:
    179-181): the MelSpectrogram (n_mels 128 unless melkwargs sets it), log(mel + 1e-6), the orthonormal DCT-II to
    n_mfcc coefficients.  forward(x [B, L]) -> [B, n_mfcc, 1 + L//hop].  CUDA only."""

    def __init__(self, sample_rate=16000, n_mfcc=40, dct_type=2, norm="ortho", log_mels=False, melkwargs=None):
        super().__init__()
        if dct_type != 2 or norm != "ortho" or not log_mels:
            raise NotImplementedError("edgedict_b200 MFCC: dct_type=2, norm='ortho', log_mels=True")
        self.n_mfcc = n_mfcc
        self.MelSpectrogram = MelSpectrogram(sample_rate=sample_rate, **(melkwargs or {}))
        if n_mfcc > self.MelSpectrogram.n_mels:
            raise ValueError("Cannot select more MFCC coefficients than # mel bins")
        self.register_buffer("dct_mat", torch.tensor(dct_ortho(n_mfcc, self.MelSpectrogram.n_mels)))

    def _batch(self, x, lens, n_stack, delta, pad_to_divisible):
        return self.MelSpectrogram._batch(x, lens, n_stack, delta, pad_to_divisible, dct=self.dct_mat)

    @torch.no_grad()
    def forward(self, x):
        return self._batch(x, _full_lengths(x), 1, False, True)[0].transpose(1, 2)


class CatDeltas(nn.Module):
    """rnnt/transforms.py:10-16: [B, C, F] -> [B, 3C, F] = [x, d1, d2] with torchaudio's compute_deltas (window 5,
    replicate padding) applied twice.  CUDA only."""

    @torch.no_grad()
    def forward(self, feat):
        return ops.fe_deltas(feat.transpose(1, 2).contiguous()).transpose(1, 2)


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


def _feature_module(feature_type, feature_size, n_fft, win_length, hop_length, **kw):
    args = dict(n_fft=n_fft, win_length=win_length, hop_length=hop_length)
    if feature_type == "mfcc":
        return MFCC(n_mfcc=feature_size, log_mels=True, melkwargs=args)
    if feature_type == "melspec":
        return MelSpectrogram(n_mels=feature_size, **args)
    if feature_type == "logfbank":
        return FilterbankFeatures(n_filt=feature_size, **args, **kw)
    raise NotImplementedError("edgedict_b200 front end implements feature_type 'mfcc', 'melspec' and 'logfbank'")


def build_transform(feature_type, feature_size, n_fft=512, win_length=400, hop_length=200, delta=False, cmvn=False,
                    downsample=1, T_mask=0, T_num_mask=0, F_mask=0, F_num_mask=0, pad_to_divisible=True):
    """rnnt/transforms.py:165-203: returns (transform_train, transform_test, input_size) with the reference's module
    sequence (features, CatDeltas, Downsample; the train transform appends the SpecAugment time / frequency masks
    exactly where the reference does, transforms.py:195-199), in the reference's [B, C, T] layout.  ``cmvn`` is
    ignored, as in the reference."""
    mods = [_feature_module(feature_type, feature_size, n_fft, win_length, hop_length)]
    input_size = feature_size
    if delta:
        mods.append(CatDeltas())
        input_size *= 3
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


def draw_utterance_spans(T, n_ch, T_mask=0, T_num_mask=0, F_mask=0, F_num_mask=0):
    """The SpecAugment spans the reference draws when its dataset transforms each utterance alone (rnnt/dataset.py:
    103 with num_workers=0): per utterance b, its time masks (start = randrange(T[b]) on its OWN length) and then its
    frequency masks (start = randrange(n_ch)), each end = start + randrange(max_width).  Returns (time spans, frequency
    spans) as nested lists [B][n][2]; a kind of mask the transform does not append draws nothing."""
    import random
    t_on, f_on = T_mask > 0 and T_num_mask > 0, F_mask > 0 and F_num_mask > 0
    tsp, fsp = [], []
    for Tb in T:
        row = []
        for _ in range(T_num_mask if t_on else 0):
            start = random.randrange(0, Tb)
            row.append((start, start + random.randrange(0, T_mask)))
        tsp.append(row)
        row = []
        for _ in range(F_num_mask if f_on else 0):
            start = random.randrange(0, n_ch)
            row.append((start, start + random.randrange(0, F_mask)))
        fsp.append(row)
    return tsp, fsp


class BatchTransform(nn.Module):
    """build_batch_transform's module: forward(x [B, L] fp32 CUDA, lengths [B]) -> (xs [B, T_max, input_size] fp32
    CUDA, xlen int32 CPU [B]).  Utterance b gets what the reference's transform computes on x[b, :lengths[b]] alone,
    in the model-input layout, and rows t >= xlen[b] are zero: seq_collate (rnnt/dataset.py:223-240) of the
    per-utterance features.  With masks, the spans are drawn by draw_utterance_spans, in the reference's order."""

    def __init__(self, features, delta, downsample, pad_to_divisible, input_size, T_mask=0, T_num_mask=0, F_mask=0,
                 F_num_mask=0):
        super().__init__()
        self.features = features
        self.delta, self.downsample, self.pad_to_divisible = bool(delta), max(int(downsample), 1), pad_to_divisible
        self.input_size = input_size
        self.T_mask, self.T_num_mask, self.F_mask, self.F_num_mask = T_mask, T_num_mask, F_mask, F_num_mask

    @torch.no_grad()
    def forward(self, x, lengths):
        xs, xlen = self.features._batch(x, lengths, self.downsample, self.delta, self.pad_to_divisible)
        tsp, fsp = draw_utterance_spans(xlen.tolist(), xs.shape[2], self.T_mask, self.T_num_mask, self.F_mask,
                                        self.F_num_mask)
        for spans, axis in ((tsp, 1), (fsp, 2)):
            if spans and spans[0]:
                ops.fe_mask(xs, torch.tensor(spans, dtype=torch.int32).to(xs.device), axis, 0.0)
        return xs, xlen

    def extra_repr(self):
        return "delta=%s, downsample=%d, pad_to_divisible=%s, T_mask=%d, T_num_mask=%d, F_mask=%d, F_num_mask=%d" % (
            self.delta, self.downsample, self.pad_to_divisible, self.T_mask, self.T_num_mask, self.F_mask,
            self.F_num_mask)


def build_batch_transform(feature_type, feature_size, n_fft=512, win_length=400, hop_length=200, delta=False,
                          cmvn=False, downsample=1, T_mask=0, T_num_mask=0, F_mask=0, F_num_mask=0,
                          pad_to_divisible=True, dither=1e-5):
    """build_transform's transforms per utterance over a padded batch: returns (train, test, input_size), each module
    mapping (x [B, L], lengths [B]) to (xs [B, T_max, input_size], xlen int32 CPU), see BatchTransform.  ``dither``
    is logfbank's FilterbankFeatures dither (0 for reproducible features); ``cmvn`` is ignored, as in the reference."""
    kw = dict(dither=dither) if feature_type == "logfbank" else {}
    features = _feature_module(feature_type, feature_size, n_fft, win_length, hop_length, **kw)
    input_size = feature_size * (3 if delta else 1) * max(downsample, 1)
    test = BatchTransform(features, delta, downsample, pad_to_divisible, input_size)
    train = BatchTransform(features, delta, downsample, pad_to_divisible, input_size, T_mask, T_num_mask, F_mask,
                           F_num_mask)
    return train, test, input_size
