"""Throughput of the per-utterance feature transforms over a padded batch (build_batch_transform -> csrc/frontend.cu):
B = 32 utterances of 8 - 16 s at 16 kHz, for logfbank, mfcc and melspec (80 channels), with and without deltas, at
downsample = 3, with and without the SpecAugment masks (T_mask 50 x 2, F_mask 27 x 2).  Reports audio-seconds per second
and peak device memory.

The comparison is a torch restatement of the reference's data path: each utterance transformed alone (torch.stft ->
power -> mel matmul -> log / DCT -> compute_deltas -> Downsample -> masks, rnnt/dataset.py:103), then zero_pad_concat.
It runs on CUDA and on one CPU thread; the CPU figure is what the data-loader workers spend on the features this path
replaces.  Neither torchaudio nor the reference is needed: the tables come from edgedict_b200.rnnt.features.

    python scripts/bench_features.py [--rounds 5] [--cpu-utts 4]
"""
import argparse
import json
import os
import random
import sys
import time

import torch

sys.path.insert(0, os.getcwd())
from edgedict_b200.rnnt import features as Fm  # noqa: E402

B, SR, C, DS = 32, 16000, 80, 3
MASKS = dict(T_mask=50, T_num_mask=2, F_mask=27, F_num_mask=2)


def torch_reference(ft, delta, masks, device):
    """Per-utterance torch restatement: f(x [L], ...) -> [T_b, C * (3 if delta) * DS]."""
    mod = Fm.build_transform(ft, C, delta=delta, downsample=DS)[1][0]
    if ft == "logfbank":
        win, fb, pre, hop = mod.window, mod.fb[0], mod.preemph, mod.hop_length
        n_fft, win_len = mod.n_fft, mod.win_length
    else:
        mel = mod.MelSpectrogram if ft == "mfcc" else mod
        win, fb, pre, hop = mel.spectrogram.window, mel.mel_scale.fb.t(), None, mel.hop_length
        n_fft, win_len = mel.n_fft, mel.spectrogram.win_length
    dct = mod.dct_mat.t().to(device) if ft == "mfcc" else None
    win, fb = win.to(device), fb.contiguous().to(device)
    kern = torch.arange(-2, 3, dtype=torch.float32, device=device)

    def deltas(f):                                        # compute_deltas on [C, F]: replicate pad, conv, / 10
        p = torch.nn.functional.pad(f[None], (2, 2), mode="replicate")[0]
        return torch.nn.functional.conv1d(p[:, None], kern.view(1, 1, 5))[:, 0] / 10

    def one(x):
        L = x.shape[0]
        if pre is not None:
            x = torch.cat([x[:1], x[1:] - pre * x[:-1]])
        s = torch.stft(x, n_fft, hop, win_len, win, center=True, pad_mode="reflect", return_complex=True)
        f = fb @ (s.real ** 2 + s.imag ** 2)
        if ft == "logfbank":
            f = torch.log(f + 1e-20)
            f[:, -(-L // hop):] = 0
        elif ft == "mfcc":
            f = dct @ torch.log(f + 1e-6)
        if delta:
            d1 = deltas(f)
            f = torch.cat([f, d1, deltas(d1)])
        f = f.t()
        f = torch.nn.functional.pad(f, (0, 0, 0, (DS - f.shape[0] % DS) % DS)).reshape(-1, f.shape[1] * DS)
        if masks:
            for _ in range(MASKS["T_num_mask"]):
                s0 = random.randrange(0, f.shape[0])
                f[s0:s0 + random.randrange(0, MASKS["T_mask"])] = 0
            for _ in range(MASKS["F_num_mask"]):
                s0 = random.randrange(0, f.shape[1])
                f[:, s0:s0 + random.randrange(0, MASKS["F_mask"])] = 0
        return f

    def run(x, lens):
        feats = [one(x[b, :n]) for b, n in enumerate(lens)]
        out = torch.zeros(len(feats), max(len(f) for f in feats), feats[0].shape[1], device=device)
        for b, f in enumerate(feats):
            out[b, :len(f)] = f
        return out
    return run


def cuda_time(fn, rounds):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(rounds):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / rounds, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cpu-utts", type=int, default=4, help="utterances timed on one CPU thread (scaled to B)")
    a = ap.parse_args()
    g = torch.Generator().manual_seed(0)
    lens = [int(SR * (8 + 8 * float(v))) for v in torch.rand(B, generator=g)]
    x = 0.1 * torch.randn(B, max(lens), generator=g)
    xc = x.cuda()
    audio = sum(lens) / SR
    torch.set_num_threads(1)
    for ft in ("logfbank", "mfcc", "melspec"):
        for delta in (False, True):
            for masks in (False, True):
                train, test, n = Fm.build_batch_transform(ft, C, delta=delta, downsample=DS, dither=0,
                                                          **(MASKS if masks else {}))
                mod = (train if masks else test).cuda()
                ms, mem = cuda_time(lambda: mod(xc, lens), a.rounds)
                ref = torch_reference(ft, delta, masks, "cuda")
                ms_ref, mem_ref = cuda_time(lambda: ref(xc, lens), a.rounds)
                cpu = torch_reference(ft, delta, masks, "cpu")
                k = a.cpu_utts
                t0 = time.perf_counter()
                cpu(x[:k], lens[:k])
                s_cpu = time.perf_counter() - t0
                cpu_rate = sum(lens[:k]) / SR / s_cpu
                print(json.dumps(dict(feature=ft, delta=delta, downsample=DS, masks=masks, batch=B,
                                      audio_sec=round(audio, 1), input_size=n, ms=round(ms, 3),
                                      audio_sec_per_sec=round(audio / ms * 1e3, 1), peak_mib=round(mem, 1),
                                      torch_cuda_ms=round(ms_ref, 3),
                                      torch_cuda_audio_sec_per_sec=round(audio / ms_ref * 1e3, 1),
                                      torch_cuda_peak_mib=round(mem_ref, 1),
                                      torch_cpu_1thread_audio_sec_per_sec=round(cpu_rate, 1))), flush=True)


if __name__ == "__main__":
    main()
