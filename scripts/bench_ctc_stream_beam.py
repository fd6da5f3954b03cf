#!/usr/bin/env python
"""Streaming CTC prefix beam search at E6D2 shape: bench_ctc_stream.py's workload (the GRU CTCEncoder, 6 x 1024 GRU
layers, time reduction after layer 1, proj 640, V = 1024, input 240; 64 streams x 250 chunks of [64, 2, 240] log-mel
frames, one encoder output frame per chunk) through CTCStreamBeamEngine, one persistent kernel launch and one
device-to-host copy per chunk.

  python scripts/bench_ctc_stream_beam.py [--rounds N] [--chunks C]

Audio convention: E6D2, one input frame = 37.5 ms, so a chunk of 2 frames is 75 ms and a run is 64 x 250 x 75 ms = 1200
audio-seconds.  Arms, alternated in every round so that all see the same clocks and neighbours: greedy CTCStreamEngine
(the anchor), the beam at W = 1 / 4 / 8, and W = 4 with an LMModel(1024, 64, 1024, 2)-shaped LM fused (lm_weight 0.5,
length_bonus 0.5).  The head's weights are scaled x 32 so that the log-probs are peaked, as a trained model's are.  Per
chunk the latency runs from the call to the committed ids on the host.  Prints one JSON line with the card (name, power
limit) read in the same run, and per arm and round audio-sec/sec, chunk latency p50 / p99, the tokens committed before
the final flush, the tokens the flush adds, and the forced collapses."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_ctc_stream import CFG, F, FRAME_SEC, N, S, card   # noqa: E402  the same workload and card query


def run_arm(step, reset, flush, chunks):
    import torch
    reset()
    lat, toks = [], 0
    t_all = time.perf_counter()
    for i in range(chunks.shape[0]):
        t0 = time.perf_counter()
        toks += step(chunks[i].cuda(non_blocking=True))
        torch.cuda.current_stream().synchronize()
        lat.append(time.perf_counter() - t0)
    wall = time.perf_counter() - t_all
    lat = np.array(lat) * 1e3
    return dict(wall_s=round(wall, 4), p50_ms=round(float(np.percentile(lat, 50)), 3),
                p99_ms=round(float(np.percentile(lat, 99)), 3), tokens_before_flush=int(toks),
                tokens_at_flush=int(flush()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunks", type=int, default=250)
    a = ap.parse_args()
    import torch
    from edgedict_b200.rnnt.models import CTCEncoder
    from edgedict_b200.stream_engine import CTCStreamBeamEngine, CTCStreamEngine
    assert torch.cuda.is_available(), "bench_ctc_stream_beam.py measures on the GPU"
    torch.manual_seed(0)
    m = CTCEncoder(**CFG).cuda().eval()
    with torch.no_grad():
        m.tovocab[0].weight.mul_(32.0)
    torch.manual_seed(1)
    lm = torch.nn.Module()
    lm.encoder = torch.nn.Embedding(1024, 64)
    lm.rnn = torch.nn.LSTM(64, 1024, 2, batch_first=True)
    lm.decoder = torch.nn.Linear(1024, 1024)
    lm = lm.cuda().eval()
    g = torch.Generator().manual_seed(0)
    chunks = torch.randn(a.chunks, S, N, F, generator=g).pin_memory()
    greedy = CTCStreamEngine(m, S, N)
    engines = dict(greedy=greedy)
    for W in (1, 4, 8):
        engines["beam_w%d" % W] = CTCStreamBeamEngine(m, S, N, W)
    engines["beam_w4_lm"] = CTCStreamBeamEngine(m, S, N, 4, lm=lm, lm_weight=0.5, length_bonus=0.5)

    def arm(e):
        def step(x):
            return int(e.step(x)[1].sum())

        def flush():
            return 0 if e is greedy else int(e.flush()[1].sum())
        return step, e.reset, flush

    arms = {k: arm(e) for k, e in engines.items()}
    for step, reset, _ in arms.values():                      # warm-up
        reset()
        for i in range(3):
            step(chunks[i].cuda(non_blocking=True))
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, (step, reset, flush) in arms.items():
            res[k].append(run_arm(step, reset, flush, chunks))
            res[k][-1]["forced_collapses"] = getattr(engines[k], "n_collapses", 0)
            if hasattr(engines[k], "n_collapses"):
                engines[k].n_collapses = 0
    audio = S * a.chunks * N * FRAME_SEC
    for k in res:
        for r in res[k]:
            r["audio_sec_per_sec"] = round(audio / r["wall_s"], 1)
    print(json.dumps(dict(card=card(), streams=S, chunks=a.chunks, frames_per_chunk=N,
                          audio_convention="E6D2: 37.5 ms per input frame, %.0f ms per chunk" % (N * FRAME_SEC * 1e3),
                          audio_sec=audio, phases_per_chunk={k: e.n_chunk_phases for k, e in engines.items()},
                          rounds=res)))


if __name__ == "__main__":
    main()
