#!/usr/bin/env python
"""Streaming from raw audio: 64 streams x 250 windows of 1320 samples (E6D2: win 320 + hop 200 x (3 x 2 - 1), advancing
by 1200 = 75 ms; each window gives 7 log-mel frames, 6 stacked by 3 into the [64, 2, 240] chunk of bench_stream.py),
through bench_stream.py's E6D2_LARGE transducer (StreamEngine) and bench_ctc_stream.py's GRU CTCEncoder (CTCStreamEngine).
Three arms per model, alternated round by round so that they see the same clocks and neighbours:

  fused:    the engine built with build_batch_transform's test module: the window's audio goes up, and the features run
            as front-end phases inside the one decode launch;
  separate: the same module on the device as its own launches (BatchTransform(audio, lengths)), then ``step``;
  cpu:      (transducer only) a torch CPU restatement of the reference's FilterbankFeatures per window on one thread
            (pre-emphasis, torch.stft, power, mel, log, mask, Downsample), then ``step``.

Per chunk the latency runs from the host audio to the ids on the host.  A separate profiler run gives the decode
kernel's time with and without the front end (the engine fed features), hence the front end's share of the fused
launch.  Prints one JSON line with the card (name, power limit) read in the same run.

  python scripts/bench_stream_audio.py [--rounds N] [--chunks C] [--cpu-chunks K] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_ctc_stream import CFG, LARGE, card                      # noqa: E402
from edgedict_b200.rnnt.features import build_batch_transform     # noqa: E402
from edgedict_b200.rnnt.models import CTCEncoder, Transducer      # noqa: E402
from edgedict_b200.stream_engine import CTCStreamEngine, StreamEngine   # noqa: E402

S, L, ADV, HOP, WIN, NFFT = 64, 1320, 1200, 200, 320, 512
WINDOW_SEC = ADV / 16000.0


class CpuFbank:
    """The reference's FilterbankFeatures (rnnt/features.py:126-164, dither 0) and Downsample(3, pad_to_divisible=False)
    restated in torch on the CPU, one window at a time."""

    def __init__(self, tr):
        f = tr.features
        self.fb, self.window, self.preemph = f.fb[0].cpu().clone(), f.window.cpu().clone(), f.preemph

    def __call__(self, x):                                   # x [1, L] -> [1, T, 240]
        x = torch.cat((x[:, :1], x[:, 1:] - self.preemph * x[:, :-1]), 1)
        spec = torch.stft(x, NFFT, hop_length=HOP, win_length=WIN, center=True, window=self.window,
                          return_complex=True)
        feat = torch.log(torch.matmul(self.fb, spec.abs().pow(2)) + 1e-20)
        seq = -(-x.shape[1] // HOP)
        feat[:, :, seq:] = 0
        F = feat.shape[2]
        feat = feat[:, :, :F - F % 3].transpose(1, 2)
        return feat.reshape(1, -1, feat.shape[2] * 3)


def build_models():
    torch.manual_seed(10)
    rnnt = Transducer(output_loss=False, **LARGE).eval()
    with torch.no_grad():
        for p in rnnt.parameters():
            p.mul_(2.0)
    torch.manual_seed(11)
    ctc = CTCEncoder(**CFG).eval()
    return rnnt.cuda(), ctc.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunks", type=int, default=250)
    ap.add_argument("--cpu-chunks", type=int, default=25)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this path")
    a = ap.parse_args()
    torch.set_num_threads(1)
    _, tr, _ = build_batch_transform("logfbank", 80, n_fft=NFFT, win_length=WIN, hop_length=HOP, downsample=3,
                                     pad_to_divisible=False, dither=0)
    tr = tr.cuda()
    cpu_fe = CpuFbank(tr)
    rnnt, ctc = build_models()
    g = torch.Generator().manual_seed(0)
    audio = (0.1 * torch.randn(a.chunks, S, L, generator=g)).pin_memory()
    lens = [L] * S
    host = torch.zeros(S * 4, dtype=torch.int32).pin_memory()
    arms = {}
    for name, model, cls in (("rnnt", rnnt, StreamEngine), ("ctc", ctc, CTCStreamEngine)):
        fused = cls(model, S, None, frontend=tr, samples_per_chunk=L)
        plain = cls(model, S, 2)
        arms[name] = (fused, plain)

    def to_host(out):
        ids = out[0] if isinstance(out, tuple) else out
        host[:ids.numel()].copy_(ids.reshape(-1), non_blocking=True)
        torch.cuda.current_stream().synchronize()

    def run(name, arm, n):
        fused, plain = arms[name]
        fused.reset()
        plain.reset()
        lat = []
        t_all = time.perf_counter()
        for i in range(n):
            t0 = time.perf_counter()
            if arm == "fused":
                out = fused.step(audio[i].cuda(non_blocking=True))
            elif arm == "separate":
                out = plain.step(tr(audio[i].cuda(non_blocking=True), lens)[0])
            else:
                xs = torch.cat([cpu_fe(audio[i, s:s + 1]) for s in range(S)])
                out = plain.step(xs.pin_memory().cuda(non_blocking=True))
            to_host(out)
            lat.append(time.perf_counter() - t0)
        wall = time.perf_counter() - t_all
        lat = np.array(lat) * 1e3
        return dict(audio_sec_per_sec=round(S * n * WINDOW_SEC / wall, 1),
                    p50_ms=round(float(np.percentile(lat, 50)), 3), p99_ms=round(float(np.percentile(lat, 99)), 3))

    for name in arms:                                       # warm every shape
        for arm in ("fused", "separate"):
            run(name, arm, 3)
    run("rnnt", "cpu", 2)
    torch.cuda.synchronize()
    # the two arms decode the same features: the same ids
    same = {}
    for name, (fused, plain) in arms.items():
        fused.reset()
        plain.reset()
        ok = True
        for i in range(20):
            x = audio[i].cuda()
            u, v = fused.step(x), plain.step(tr(x, lens)[0])
            u, v = (u[0], v[0]) if isinstance(u, tuple) else (u, v)
            ok = ok and torch.equal(u.cpu(), v.cpu())
        same[name] = ok
    rounds = []
    for r in range(a.rounds):
        row = {}
        for name in arms:
            for arm in ("fused", "separate"):
                row["%s_%s" % (name, arm)] = run(name, arm, a.chunks)
        row["rnnt_cpu"] = run("rnnt", "cpu", a.cpu_chunks)
        rounds.append(row)
    # front-end share of the fused launch, from kernel times in a profiler run of its own
    from torch.profiler import ProfilerActivity, profile
    share = {}
    for name, (fused, plain) in arms.items():
        x = audio[0].cuda()
        xs = tr(x, lens)[0]
        torch.cuda.synchronize()
        times = {}
        for arm, eng, inp in (("fused", fused, x), ("plain", plain, xs)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(50):
                    eng.step(inp)
                torch.cuda.synchronize()
            ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "decode_program_kernel" in e.name]
            times[arm] = float(np.median([e.device_time_total for e in ks]))
        share[name] = dict(fused_kernel_us=round(times["fused"], 1), features_in_kernel_us=round(times["plain"], 1),
                           front_end_share=round(1.0 - times["plain"] / times["fused"], 4))
    res = dict(bench="stream_audio", card=card(), streams=S, window_samples=L, advance_samples=ADV,
               chunks=a.chunks, cpu_chunks=a.cpu_chunks, torch_threads=torch.get_num_threads(),
               same_ids_fused_vs_separate=same, rounds=rounds, front_end_share=share)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
