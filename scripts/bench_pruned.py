#!/usr/bin/env python
"""The pruned RNN-T loss against the full loss at the E6D2 shape: B = 32, T = 1000 -> T' = 500, U = 128 labels, V = 1024,
bf16 mode, and one memory-bound shape (V = 4096, U = 256).

  python scripts/bench_pruned.py [--rounds N] [--reps K] [--ranges 4,5,8]

Per shape and arm (full, prune_range = R), alternated within every round so all arms see the same clocks:
  step : a bf16 Transducer training step (forward + backward), ms per step;
  peak : peak device memory of one step, GB;
and, for the pruned arms, the stages of the joint + loss from ops' CUDA-event instrumentation over one step:
simple loss (forward + backward), band choice, band-row GEMMs, loss gradient.  Prints one JSON line with the card
(name, power limit, max SM clock) read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T = 32, 1000
E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0,
            dec_proj_size=256, joint_size=640)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ranges", default="4,5,8")
    a = ap.parse_args()
    import torch
    from edgedict_b200 import ops
    from edgedict_b200.rnnt.models import Transducer
    assert torch.cuda.is_available(), "bench_pruned.py measures on the GPU"
    dev = torch.device("cuda")
    ranges = [int(x) for x in a.ranges.split(",")]
    out = dict(card=card(), B=B, T=T, T_out=(T + 1) // 2, shapes={})
    for U, V in ((128, 1024), (256, 4096)):
        g = torch.Generator(device=dev).manual_seed(0)
        ys = torch.randint(1, V, (B, U), dtype=torch.int32, device=dev, generator=g)
        xs = torch.randn(B, T, E6D2["input_size"], device=dev, generator=g)
        xlen = torch.full((B,), T, dtype=torch.int32)
        ylen = torch.full((B,), U, dtype=torch.int32)
        models = {}
        for R in [None] + ranges:
            torch.manual_seed(0)
            m = Transducer(**dict(E6D2, vocab_size=V), prune_range=R).to(dev)
            m.set_precision("bf16")
            models["full" if R is None else "R%d" % R] = m

        def step(m):
            m.zero_grad(set_to_none=True)
            m(xs, ys, xlen, ylen).backward()

        res = {k: dict(step_ms=[]) for k in models}
        for k, m in list(models.items()):                 # warm-up, peak memory and the stage split
            try:
                step(m)
            except torch.cuda.OutOfMemoryError:
                res[k] = "out of memory"
                del models[k]
                torch.cuda.empty_cache()
                continue
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            step(m)
            torch.cuda.synchronize()
            res[k]["peak_GB"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
            ops.PROF.reset()
            ops.PROF.enabled = True
            step(m)
            torch.cuda.synchronize()
            ops.PROF.enabled = False
            prof = ops.PROF.summary()
            res[k]["stages_ms"] = {n: round(d["ms"], 3) for n, d in prof.items()
                                   if n.startswith(("rnnt_", "joint_", "gemm_bf16"))}
        for _ in range(a.rounds):
            for k, m in models.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    step(m)
                e1.record()
                torch.cuda.synchronize()
                res[k]["step_ms"].append(round(e0.elapsed_time(e1) / a.reps, 2))
        out["shapes"]["U%d_V%d" % (U, V)] = res
        del models
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
