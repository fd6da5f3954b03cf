#!/usr/bin/env python
"""FastEmit's cost at the E6D2 shape: B = 32, T = 1000 -> T' = 500, U = 128 labels (U+1 = 129), V = 1024.

  python scripts/bench_fastemit.py [--rounds N] [--reps K] [--lam L]

Three comparisons of fastemit_lambda = 0 against fastemit_lambda = L (default 0.01), each alternated within every round
(K timed calls per arm after a warm-up), so both arms see the same clocks and neighbours:
  bf16_db : eb_rnnt_loss_bwd_bf16_db_fe in place over bf16 logits, the gradient kernel of the bf16 training step;
  fp32    : eb_rnnt_loss_bwd_fe, fp32 logits to fp32 d logits out of place, the gradient kernel of the fp32 mode;
  step    : a bf16 Transducer training step (forward + backward) with model.fastemit_lambda set per arm.
The per-element work of the kernels does not depend on lambda (two extra row scalars per cell), so the arms should
differ by no more than the spread across rounds.  Prints one JSON line: the card (name, power limit, max SM clock) read
in the same run and ms per call for every round.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, U, V = 32, 1000, 128, 1024
E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0,
            dec_proj_size=256, joint_size=640)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--lam", type=float, default=0.01)
    a = ap.parse_args()
    import torch
    from edgedict_b200 import ops
    from edgedict_b200.rnnt.models import Transducer
    assert torch.cuda.is_available(), "bench_fastemit.py measures on the GPU"
    dev = torch.device("cuda")
    Tp = (T + 1) // 2

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    def alternate(arms, reps):
        res = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                res[k].append(round(timed(fn, reps), 3))
        return res

    # the kernels, over one workspace filled from random fp32 logits [B, T', U+1, V]
    g = torch.Generator(device=dev).manual_seed(0)
    ys = torch.randint(1, V, (B, U), dtype=torch.int32, device=dev, generator=g)
    xl = torch.full((B,), Tp, dtype=torch.int32, device=dev)
    yl = torch.full((B,), U, dtype=torch.int32, device=dev)
    acts = torch.randn(B, Tp, U + 1, V, device=dev, generator=g)
    _, ws = ops.rnnt_loss_fwd(acts, ys, xl, yl, 0, need_beta=True)
    gs = torch.ones(1, device=dev)
    grads = torch.empty_like(acts)
    l16 = acts.to(torch.bfloat16)

    def fp32(lam):
        return lambda: ops.rnnt_loss_bwd(acts, ys, xl, yl, 0, ws, gs, 1.0 / B, out=grads, fastemit_lambda=lam)

    def bf16_db(lam):
        # in place, as JointLoss runs it: the d logits of one call are the logits of the next, which changes nothing the
        # kernel's time depends on
        return lambda: ops.rnnt_loss_bwd_bf16_db(l16, ys, xl, yl, 0, ws, gs, 1.0 / B, fastemit_lambda=lam)

    res = alternate({"bf16_db_lam0": bf16_db(0.0), "bf16_db_lam": bf16_db(a.lam)}, a.reps)
    res.update(alternate({"fp32_lam0": fp32(0.0), "fp32_lam": fp32(a.lam)}, a.reps))
    del acts, grads, l16, ws
    torch.cuda.empty_cache()

    # a bf16 training step of the E6D2 transducer
    torch.manual_seed(0)
    m = Transducer(**E6D2).to(dev)
    m.set_precision("bf16")
    xs = torch.randn(B, T, E6D2["input_size"], device=dev)
    xlen = torch.full((B,), T, dtype=torch.int32)
    ylen = torch.full((B,), U, dtype=torch.int32)

    def step(lam):
        def run():
            m.fastemit_lambda = lam
            m.zero_grad(set_to_none=True)
            m(xs, ys, xlen, ylen).backward()
        return run

    res.update(alternate({"step_bf16_lam0": step(0.0), "step_bf16_lam": step(a.lam)}, max(1, a.reps // 5)))
    print(json.dumps(dict(card=card(), B=B, T=T, T_out=Tp, U=U, V=V, lam=a.lam, reps=a.reps,
                          step_reps=max(1, a.reps // 5), ms=res)))


if __name__ == "__main__":
    main()
