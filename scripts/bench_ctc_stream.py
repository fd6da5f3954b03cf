#!/usr/bin/env python
"""Streaming greedy CTC at E6D2 shape: bench_ctc.py's CTCEncoder (6 x 1024 GRU layers, time reduction after layer 1,
proj 640, V = 1024, input 240), 64 streams x 250 chunks of [64, 2, 240] log-mel frames through CTCStreamEngine (one
persistent kernel launch and one device-to-host copy per chunk).

  python scripts/bench_ctc_stream.py [--rounds N] [--chunks C]

Audio convention: E6D2, one input frame = 37.5 ms (hop 200 x downsample 3 at 16 kHz), so a chunk of 2 frames is 75 ms
and the run is 64 x 250 x 75 ms = 1200 audio-seconds.  Anchors, alternated with it in every round so that all arms see
the same clocks and neighbours:
  transducer: StreamEngine on bench_stream.py's workload (E6D2_LARGE transducer, weights x 2, 64 streams, [64, 2, 240]
              chunks; the same kernel with LSTM cells, joint, argmax and predictor);
  torch:      the same CTC chunk restated in torch on the GPU, batched over the 64 streams: LayerNorm, per layer cuDNN
              nn.GRU from the carried h, residual LayerNorm, time reduction, projection, head, log_softmax, argmax and
              the carried collapse, one device-to-host copy.
Per chunk the latency runs from the call to the ids on the host.  Prints one JSON line with the card (name, power limit)
read in the same run, audio-sec/sec, chunk latency p50 / p99 per arm and round, and the emitted tokens."""
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
FRAME_SEC = 0.0375
CFG = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0, proj_size=640)
LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


class TorchChunk:
    """The CTC chunk restated in torch (cuDNN GRU), all streams batched, state carried between chunks."""

    def __init__(self, m):
        import torch
        import torch.nn as nn
        enc = m.model
        self.norm, self.proj, self.head = enc.norm, enc.proj, m.tovocab[0]
        self.lns = [p[0] for p in enc.lstm.projs]
        self.red = enc.lstm.time_reductions
        self.grus = []
        for g in enc.lstm.lstms:
            q = nn.GRU(g.input_size, g.hidden_size, 1, batch_first=True).to(g.weight_ih_l0.device)
            q.load_state_dict(g.state_dict())
            self.grus.append(q.eval())
        self.blank = m.blank
        self.h = torch.zeros(len(self.grus), S, enc.lstm.hidden_size, device=m.tovocab[0].weight.device)
        self.prev = torch.full((S,), -1, dtype=torch.long, device=self.h.device)

    def step(self, x):
        import torch
        import torch.nn.functional as Fn
        with torch.no_grad():
            x = Fn.layer_norm(x, (x.shape[-1],), self.norm.weight, self.norm.bias, 1e-5)
            hs = []
            for i, (g, ln) in enumerate(zip(self.grus, self.lns)):
                y, h = g(x, self.h[i:i + 1])
                hs.append(h)
                x = Fn.layer_norm(y if i == 0 else x + y, (y.shape[-1],), ln.weight, ln.bias, 1e-5)
                if i in self.red:
                    x = x.view(S, -1, 2, x.shape[-1]).mean(2)
            self.h = torch.cat(hs, 0)
            lp = Fn.log_softmax(self.head(self.proj(x)), -1)
            am = lp.argmax(-1)
            prev = torch.cat([self.prev[:, None], am[:, :-1]], 1)
            keep = (am != self.blank) & (am != prev)
            self.prev = am[:, -1]
            return torch.where(keep, am, -1).cpu()


def run_arm(step, reset, chunks):
    import torch
    reset()
    lat, toks = [], 0
    t_all = time.perf_counter()
    for i in range(chunks.shape[0]):
        t0 = time.perf_counter()
        out = step(chunks[i].cuda(non_blocking=True))
        torch.cuda.current_stream().synchronize()
        lat.append(time.perf_counter() - t0)
        toks += out
    wall = time.perf_counter() - t_all
    lat = np.array(lat) * 1e3
    return dict(wall_s=round(wall, 4), p50_ms=round(float(np.percentile(lat, 50)), 3),
                p99_ms=round(float(np.percentile(lat, 99)), 3), tokens=int(toks))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunks", type=int, default=250)
    a = ap.parse_args()
    import torch
    from edgedict_b200.rnnt.models import CTCEncoder, Transducer
    from edgedict_b200.stream_engine import CTCStreamEngine, StreamEngine
    assert torch.cuda.is_available(), "bench_ctc_stream.py measures on the GPU"
    torch.manual_seed(0)
    m = CTCEncoder(**CFG).cuda().eval()
    torch.manual_seed(10)
    tr = Transducer(output_loss=False, **LARGE).eval()
    with torch.no_grad():
        for p in tr.parameters():
            p.mul_(2.0)
    tr.cuda()
    g = torch.Generator().manual_seed(0)
    chunks = torch.randn(a.chunks, S, N, F, generator=g).pin_memory()
    ctc = CTCStreamEngine(m, S, N)
    trd = StreamEngine(tr, S, N)
    ref = TorchChunk(m)

    def ctc_step(x):
        ids, cnt = ctc.step(x)
        return int(cnt.sum())

    def trd_step(x):
        return int((trd.step(x).cpu() != 0).sum())

    def torch_step(x):
        return int((ref.step(x) >= 0).sum())

    def torch_reset():
        ref.h.zero_()
        ref.prev.fill_(-1)

    arms = dict(ctc_stream=(ctc_step, ctc.reset), transducer_stream=(trd_step, trd.reset),
                torch_cudnn_gru=(torch_step, torch_reset))
    for step, reset in arms.values():                         # warm-up
        reset()
        for i in range(3):
            step(chunks[i].cuda(non_blocking=True))
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, (step, reset) in arms.items():
            res[k].append(run_arm(step, reset, chunks))
    audio = S * a.chunks * N * FRAME_SEC
    for k in res:
        for r in res[k]:
            r["audio_sec_per_sec"] = round(audio / r["wall_s"], 1)
    # how often the torch restatement's per-chunk ids agree with the engine's (cuDNN's products are not fp32-accurate)
    ctc.reset()
    torch_reset()
    same = total = 0
    for i in range(min(a.chunks, 50)):
        ids, cnt = ctc.step(chunks[i].cuda())
        r = ref.step(chunks[i].cuda())
        for s in range(S):
            want = [int(v) for v in r[s] if v >= 0]
            same += ids[s, :int(cnt[s])].tolist() == want
            total += 1
    print(json.dumps(dict(card=card(), streams=S, chunks=a.chunks, frames_per_chunk=N,
                          audio_convention="E6D2: 37.5 ms per input frame, %.0f ms per chunk" % (N * FRAME_SEC * 1e3),
                          audio_sec=audio, ctc_phases_per_chunk=ctc.n_chunk_phases, rounds=res,
                          torch_restatement_chunk_agreement=round(same / max(total, 1), 4))))


if __name__ == "__main__":
    main()
