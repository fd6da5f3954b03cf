"""numpy restatement of the log-mel front end (TEST INFRASTRUCTURE -- only tests/, smoke() and the bench
baseline may import this; the product path is edgedict_b200/csrc/frontend.cu).

Follows rnnt/features.py:33-152 (FilterbankFeatures: dither -> pre-emphasis -> torch.stft -> power -> mel
matmul -> log(x + 1e-20) -> mask) and rnnt/transforms.py:30-51 (Downsample = frame stacking).

Third-party arithmetic outside the reference project (SURVEY 8c):
  * torch.stft as the reference calls it (torch==1.4: center=True, pad_mode='reflect', onesided, window of
    win_length zero-padded symmetrically to n_fft).  PINNED in tests/test_oracle_features.py against this
    container's torch.stft (same arguments, return_complex=True).
  * librosa.filters.mel (librosa==0.7.2, requirements.txt; htk=False, norm=1 i.e. Slaney area normalisation):
    librosa is absent here, its published algorithm is restated in slaney_mel_filterbank().  PINNED against
    torchaudio.functional.melscale_fbanks(norm='slaney', mel_scale='slaney') -- an independent implementation of
    the same formula; parity against librosa itself is UNPINNED.
"""
import numpy as np


def hann_window(win_length, dtype=np.float64):
    """torch.hann_window(win_length, periodic=False) (features.py:74-75)."""
    n = np.arange(win_length, dtype=np.float64)
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * n / (win_length - 1))).astype(dtype)


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mel = f / f_sp
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, mel)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def slaney_mel_filterbank(sr, n_fft, n_mels, fmin=0.0, fmax=None):
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) of librosa 0.7.2 -> float32 [n_mels, 1 + n_fft//2]
    (features.py:76-80)."""
    fmax = sr / 2.0 if fmax is None else fmax
    nb = 1 + n_fft // 2
    fftfreqs = np.linspace(0.0, sr / 2.0, nb)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, nb))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0.0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    return (w * enorm[:, None]).astype(np.float32)


def preemphasis(x, coeff):
    """features.py:137-141."""
    return np.concatenate([x[:, :1], x[:, 1:] - coeff * x[:, :-1]], axis=1)


def stft_power(x, n_fft, hop_length, win_length, window):
    """|torch.stft|^2 with the torch==1.4 defaults the reference relies on (features.py:121-124,146):
    -> [B, 1 + n_fft//2, 1 + L//hop]."""
    pad = n_fft // 2
    xp = np.pad(x, ((0, 0), (pad, pad)), mode="reflect")
    wfull = np.zeros(n_fft, dtype=x.dtype)
    left = (n_fft - win_length) // 2
    wfull[left:left + win_length] = window
    nfr = 1 + (xp.shape[1] - n_fft) // hop_length
    idx = np.arange(n_fft)[None, :] + hop_length * np.arange(nfr)[:, None]
    frames = xp[:, idx] * wfull[None, None, :]
    spec = np.fft.rfft(frames, axis=-1)
    return (spec.real ** 2 + spec.imag ** 2).transpose(0, 2, 1)


def filterbank_features(x, sample_rate=16000, win_length=320, hop_length=160, n_fft=512, n_filt=64, preemph=0.97,
                        log=True, f_min=0.0, f_max=None, dtype=np.float32):
    """FilterbankFeatures.forward (features.py:126-176) with dither=0, normalize='none', pad_to=0.
    x [B, L] -> [B, n_filt, 1 + L//hop]."""
    x = np.asarray(x, dtype=dtype)
    L = x.shape[1]
    seq_len = int(np.ceil(L / hop_length))                       # get_seq_len on x.shape[1] (features.py:128)
    if preemph is not None:
        x = preemphasis(x, dtype(preemph))
    p = stft_power(x, n_fft, hop_length, win_length, hann_window(win_length, dtype)).astype(dtype)
    fb = slaney_mel_filterbank(sample_rate, n_fft, n_filt, f_min, f_max).astype(dtype)
    y = np.einsum("mk,bkf->bmf", fb, p)
    if log:
        y = np.log(y + dtype(1e-20))
    y[:, :, seq_len:] = 0                                        # features.py:160-164
    return y.astype(dtype)


def downsample(feat, n_frame, pad_to_divisible=True):
    """transforms.Downsample.forward (transforms.py:37-51): [B, C, F] -> [B, C*n_frame, ceil(F/n_frame)]."""
    feat = feat.transpose(0, 2, 1)
    B, F, C = feat.shape
    if pad_to_divisible:
        pad = (n_frame - F % n_frame) % n_frame
        feat = np.pad(feat, ((0, 0), (0, pad), (0, 0)))
    else:
        F = F - F % n_frame
        feat = feat[:, :F]
    return feat.reshape(B, -1, C * n_frame).transpose(0, 2, 1)


def logmel_frontend(x, n_filt=80, n_fft=512, win_length=400, hop_length=200, downsample_n=3, **kw):
    """build_transform('logfbank', 80, downsample=3) as flagfiles/E6D2.txt configures it (transforms.py:165-203,
    test transform: no SpecAugment masks) -> model input layout [B, T, n_filt * downsample_n]."""
    f = filterbank_features(x, win_length=win_length, hop_length=hop_length, n_fft=n_fft, n_filt=n_filt, **kw)
    if downsample_n > 1:
        f = downsample(f, downsample_n)
    return np.ascontiguousarray(f.transpose(0, 2, 1))
