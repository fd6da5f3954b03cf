#!/usr/bin/env python
"""GRU encoder stack at E6D2 dims (6 x 1024 GRU layers, time reduction after layer 1, input 240, B = 32, T = 1000):
forward + backward on the engine (ResLayerNormGRU -> functional.GRULayer: eb_gru_seq_fwd / eb_gru_seq_bwd in fp32 mode,
eb_gru_tc_fwd / eb_gru_tc_bwd in bf16 mode) against the nn.GRU / nn.LayerNorm path through cuDNN on the same weights
and inputs.

  python scripts/bench_gru.py [--rounds N] [--reps K]

  fp32: the engine in fp32 mode against cuDNN in fp32 (TF32 off: torch.backends.cudnn.allow_tf32 = False);
  bf16: the engine in bf16 mode against cuDNN under torch.autocast(dtype=bfloat16).

The engine and cuDNN alternate within each round (K timed encoder forward + backward passes each, after a warm-up), so
both see the same clocks and neighbours.  Prints one JSON line: the card (name, power limit) read in the same run, ms per
encoder forward + backward for every round, and the engine's per-kernel time in us per recurrent step (ops.PROF).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, F, H, L = 32, 1000, 240, 1024, 6
REDUCTIONS = (1,)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def cudnn_encoder(enc, xs):
    """The nn.GRU path on the engine's parameters: LayerNorm -> per layer nn.GRU, residual, LayerNorm, time reduction."""
    import torch
    from torch import nn
    x = nn.functional.layer_norm(xs, (xs.shape[-1],), enc.norm.weight, enc.norm.bias, enc.norm.eps)
    for i, (gru, post) in enumerate(zip(enc.lstm.lstms, enc.lstm.projs)):
        y, _ = gru(x)
        x = y if i == 0 else x + y
        ln = post[0]
        x = nn.functional.layer_norm(x, (x.shape[-1],), ln.weight, ln.bias, ln.eps)
        if i in REDUCTIONS:
            if x.shape[1] % 2:
                x = nn.functional.pad(x, [0, 0, 0, 1])
            x = x.reshape(x.shape[0], -1, 2, x.shape[-1]).mean(2)
    return nn.functional.linear(x, enc.proj.weight, enc.proj.bias)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    from edgedict_b200 import ops
    from edgedict_b200.rnnt.models import Encoder, ResLayerNormGRU, _set_precision
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    enc = Encoder(F, H, L, 0.0, 640, module=ResLayerNormGRU, time_reductions=list(REDUCTIONS)).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    xs = torch.randn(B, T, F, device=dev, generator=g)
    gout = torch.randn(B, (T + 1) // 2, 640, device=dev, generator=g)
    params = list(enc.parameters())

    def engine(precision):
        _set_precision(enc, precision)
        out, _ = enc(xs)
        torch.autograd.backward(out, gout)

    def cudnn(precision):
        if precision == "bf16":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = cudnn_encoder(enc, xs)
        else:
            out = cudnn_encoder(enc, xs)
        torch.autograd.backward(out.float(), gout)

    def timed(fn, precision):
        for p in params:
            p.grad = None
        torch.cuda.synchronize()
        a0, b0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record()
        for _ in range(a.reps):
            fn(precision)
        b0.record()
        torch.cuda.synchronize()
        return a0.elapsed_time(b0) / a.reps

    res = {"card": card(), "dims": dict(B=B, T=T, F=F, H=H, L=L, reductions=REDUCTIONS), "reps": a.reps}
    steps = sum(T if i <= max(REDUCTIONS) else (T + 1) // 2 for i in range(L))   # recurrent steps per pass
    for precision in ("fp32", "bf16"):
        engine(precision), cudnn(precision)                                           # warm-up
        rounds = []
        for _ in range(a.rounds):
            rounds.append(dict(engine_ms=round(timed(engine, precision), 2), cudnn_ms=round(timed(cudnn, precision), 2)))
        ops.PROF.reset()
        ops.PROF.enabled = True
        engine(precision)
        torch.cuda.synchronize()
        ops.PROF.enabled = False
        prof = {k: round(1000.0 * v["ms"] / steps, 2) for k, v in ops.PROF.summary().items() if k.startswith("gru_")}
        res[precision] = dict(rounds=rounds, engine_us_per_step=prof)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
