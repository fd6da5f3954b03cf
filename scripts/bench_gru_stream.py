#!/usr/bin/env python
"""Streaming GRU transducer at E6D2_LARGE shape: bench_stream.py's workload with the encoder a GRU stack
(``Transducer(module_type='GRU')``: 6 x 1024 GRU layers, time reduction after layer 1, proj 640, predictor 512 x 2,
joint 640, V = 1024, input 240, weights x 2), 64 streams x 250 chunks of [64, 2, 240] log-mel frames, 120 ms of audio
per chunk (bench_stream.py's convention), one persistent kernel launch per chunk through eb_decode_run_gru_rnnt.

  python scripts/bench_gru_stream.py [--rounds N] [--chunks C]

Arms, alternated in every round so that all of them see the same clocks and neighbours:
  gru_greedy:  GRUStreamEngine, max_symbols 1;
  gru_beam4:   GRUStreamBeamEngine, W = 4;
  gru_beam4_lm: GRUStreamBeamEngine, W = 4, fused with an LMModel(1024, 64, 1024, 2)-shaped LM (weights x 2);
  lstm_greedy: StreamEngine on bench_stream.py's LSTM model, the anchor.
Per chunk the latency runs from the call to the tokens on the host.  Prints one JSON line with the card (name, power
limit) read in the same run, audio-sec/sec, chunk latency p50 / p99 per arm and round, and the tokens emitted."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

S, N, F = 64, 2, 240
CHUNK_SEC = 0.120
LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def model(module_type):
    import torch
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(10)
    m = Transducer(output_loss=False, module_type=module_type, **LARGE).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)                       # random-init weights emit only blanks; scale up so symbols appear
    return m.cuda()


def lm_module():
    import torch
    import torch.nn as nn

    class LMModel(nn.Module):                 # the reference's LMModel layout: encoder, rnn, decoder
        def __init__(self, ntoken, ninp, nhid, nlayers):
            super().__init__()
            self.encoder = nn.Embedding(ntoken, ninp)
            self.rnn = nn.LSTM(ninp, nhid, nlayers, batch_first=True)
            self.decoder = nn.Linear(nhid, ntoken)

    torch.manual_seed(3)
    lm = LMModel(1024, 64, 1024, 2).eval()
    with torch.no_grad():
        for p in lm.parameters():
            p.mul_(2.0)
    return lm.cuda()


def run_arm(step, pinned, n):
    """-> (wall s, per-chunk latency ms, tokens emitted)"""
    import torch
    step.reset()
    torch.cuda.synchronize()
    lat, toks = [], 0
    t_all = time.perf_counter()
    for i in range(n):
        t0 = time.perf_counter()
        toks += step(pinned[i])
        lat.append(time.perf_counter() - t0)
    return time.perf_counter() - t_all, np.array(lat) * 1e3, toks


class Greedy:
    def __init__(self, eng):
        import torch
        self.eng = eng
        self.host = torch.zeros(S, eng.n_out * eng.max_symbols, dtype=torch.int32).pin_memory()

    def reset(self):
        self.eng.reset()

    def __call__(self, chunk):
        import torch
        out = self.eng.step(chunk.cuda(non_blocking=True))
        self.host.copy_(out, non_blocking=True)
        torch.cuda.current_stream().synchronize()           # the tokens are on the host: end of the chunk
        return int((self.host != 0).sum())


class Beam:
    def __init__(self, eng):
        self.eng = eng

    def reset(self):
        self.eng.reset()

    def __call__(self, chunk):
        _, counts = self.eng.step(chunk.cuda(non_blocking=True))   # committed ids on the host
        return int(counts.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunks", type=int, default=250)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from edgedict_b200.stream_engine import GRUStreamBeamEngine, GRUStreamEngine, StreamEngine
    gru, lstm, lm = model("GRU"), model("LSTM"), lm_module()
    chunks = torch.randn(a.chunks, S, N, F, generator=torch.Generator().manual_seed(0))
    pinned = chunks.pin_memory()
    arms = dict(gru_greedy=Greedy(GRUStreamEngine(gru, S, N)),
                gru_beam4=Beam(GRUStreamBeamEngine(gru, S, N, 4)),
                gru_beam4_lm=Beam(GRUStreamBeamEngine(gru, S, N, 4, lm=lm, lm_weight=0.3, length_bonus=0.5)),
                lstm_greedy=Greedy(StreamEngine(lstm, S, N)))
    for arm in arms.values():                                  # warm-up: module load, first launches
        run_arm(arm, pinned, 3)
    res = {k: [] for k in arms}
    for r in range(a.rounds):
        for k, arm in arms.items():
            wall, lat, toks = run_arm(arm, pinned, a.chunks)
            audio = S * a.chunks * CHUNK_SEC
            res[k].append(dict(audio_sec_per_sec=round(audio / wall, 1), p50_ms=round(float(np.percentile(lat, 50)), 3),
                               p99_ms=round(float(np.percentile(lat, 99)), 3), tokens=toks))
    out = dict(config="E6D2_LARGE GRU transducer streaming, %d streams x %d chunks of [%d, %d, %d], %.0f ms per chunk"
               % (S, a.chunks, S, N, F, CHUNK_SEC * 1e3), card=card(), rounds=res,
               phases_per_chunk={k: arm.eng.n_chunk_phases for k, arm in arms.items()})
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
