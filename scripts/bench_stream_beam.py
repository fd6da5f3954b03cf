"""Streaming beam search on bench_stream.py's workload: E6D2_LARGE, 64 concurrent synthetic 30-s streams (250 chunks of
[64, 2, 240] log-mel = 120 ms of audio each), one persistent decode launch per chunk.  Greedy StreamEngine is the
anchor; StreamBeamEngine runs W = 1, 4, 8 without an LM and W = 4 with an LMModel(1024, 64, 1024, 2)-shaped LM.  The
configurations are warmed up, then timed in alternation over several rounds.  Per configuration: RTF, audio-s/s,
per-chunk latency p50/p99 (H2D of the chunk, the launch, the D2H of the committed tokens), forced collapses and
committed tokens (including each stream's final flush).  Prints one JSON line with the card's name and power limit."""
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.getcwd())
from edgedict_b200.rnnt.models import Transducer
from edgedict_b200.stream_engine import StreamBeamEngine, StreamEngine

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
S, CHUNKS, CHUNK_SEC, ROUNDS = 64, 250, 0.120, 3


def card():
    """Name and power limit of the device torch runs on, found by its PCI bus id, else by its UUID
    (CUDA_VISIBLE_DEVICES renumbers devices for torch, not for nvidia-smi)."""
    pr = torch.cuda.get_device_properties(torch.cuda.current_device())
    bus = (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)

    def smi(*args):
        try:
            return subprocess.run(["nvidia-smi", "--format=csv,noheader"] + list(args), capture_output=True,
                                  text=True, timeout=30).stdout
        except (OSError, subprocess.SubprocessError):
            return ""
    q = smi("--query-gpu=pci.bus_id,name,power.limit")
    for line in q.splitlines():
        m = re.match(r"\s*([0-9A-Fa-f]+):([0-9A-Fa-f]+):([0-9A-Fa-f]+)\.[0-9A-Fa-f]+\s*,(.*)", line)
        if m and tuple(int(m.group(i), 16) for i in (1, 2, 3)) == bus:
            return m.group(4).strip()
    uuid = str(getattr(pr, "uuid", ""))
    if uuid:
        q = smi("--query-gpu=name,power.limit", "-i", uuid if uuid.startswith("GPU-") else "GPU-" + uuid).strip()
        if q and "," in q:
            return q
    print("card: no nvidia-smi row for bus %s / uuid %s: %r" % (bus, uuid, q), file=sys.stderr)
    return pr.name + ", power limit not readable"


def main():
    torch.manual_seed(10)
    model = Transducer(output_loss=False, **LARGE).eval()
    with torch.no_grad():
        for p in model.parameters():
            p.mul_(2.0)                   # random-init weights emit only blanks; scale up so symbols appear
    model.cuda()
    torch.manual_seed(11)
    lm = torch.nn.Module()                # LMModel(1024, 64, 1024, 2): embedding 64, 2 x LSTM 1024, decoder 1024
    lm.encoder, lm.rnn = torch.nn.Embedding(1024, 64), torch.nn.LSTM(64, 1024, 2, batch_first=True)
    lm.decoder = torch.nn.Linear(1024, 1024)
    lm = lm.cuda().eval()
    g = torch.Generator().manual_seed(0)
    pinned = torch.randn(CHUNKS, S, 2, 240, generator=g).pin_memory()
    greedy_host = torch.zeros(S, 1, dtype=torch.int32).pin_memory()

    def greedy_step(eng, x):
        greedy_host.copy_(eng.step(x), non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return int((greedy_host != 0).sum())

    def beam_step(eng, x):
        _, counts = eng.step(x)
        return int(counts.sum())

    configs = [("greedy", StreamEngine(model, S, 2), greedy_step)]
    for W in (1, 4, 8):
        configs.append(("beam W=%d" % W, StreamBeamEngine(model, S, 2, W), beam_step))
    configs.append(("beam W=4 + LM", StreamBeamEngine(model, S, 2, 4, lm=lm, lm_weight=0.3, length_bonus=0.5),
                    beam_step))
    for _, eng, stepf in configs:                                  # warm-up
        for i in range(5):
            stepf(eng, pinned[i].cuda(non_blocking=True))
        eng.reset()
    torch.cuda.synchronize()
    stats = {name: dict(lat=[], wall=0.0, tokens=0, collapses=0) for name, _, _ in configs}
    for _ in range(ROUNDS):
        for name, eng, stepf in configs:
            st = stats[name]
            eng.reset()
            c0 = getattr(eng, "n_collapses", 0)
            torch.cuda.synchronize()
            t_all = time.perf_counter()
            for i in range(CHUNKS):
                t0 = time.perf_counter()
                st["tokens"] += stepf(eng, pinned[i].cuda(non_blocking=True))
                st["lat"].append(time.perf_counter() - t0)
            st["wall"] += time.perf_counter() - t_all
            if isinstance(eng, StreamBeamEngine):
                st["collapses"] += eng.n_collapses - c0
                st["tokens"] += int(eng.flush()[1].sum())
    audio = S * CHUNKS * CHUNK_SEC * ROUNDS
    out = {}
    for name, st in stats.items():
        lat = np.array(st["lat"]) * 1e3
        out[name] = dict(rtf=round(st["wall"] / audio, 6), audio_sec_per_sec=round(audio / st["wall"], 1),
                         chunk_latency_ms=dict(p50=round(float(np.percentile(lat, 50)), 3),
                                               p99=round(float(np.percentile(lat, 99)), 3)),
                         forced_collapses=st["collapses"] // ROUNDS, committed_tokens=st["tokens"] // ROUNDS)
    res = dict(config="E6D2_LARGE streaming, %d streams x %d chunks x 120 ms, %d alternated rounds"
               % (S, CHUNKS, ROUNDS), card=card(), results=out)
    print(json.dumps(res))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
