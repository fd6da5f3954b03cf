"""Step time of the flat-bucket optimizers (edgedict_b200.optim) against torch restatements of the reference's classes.

    python scripts/bench_optim.py [--steps 50] [--warmup 10] [--out results.json]

Parameter sets: the E6D2 transducer (bench.py's configuration, 55 tensors), and cli/train.py's raw-waveform FrontEnd
plus the transducer on its 128 features.  Gradients are filled from a seed.  For every optimizer it reports the median
step time (CUDA events, after warm-up), the bytes of optimizer state, the bytes one step must move (parameters read and
written, gradients read, state read and written, one more gradient read for a per-tensor or clip norm) and the
achieved bandwidth against the H100 SXM data sheet's 3.35 TB/s.  Anchors: torch.optim.SGD(foreach=True) and
(fused=True), and torch.optim.AdamW(fused=True) as a speed anchor only (its update differs from the reference's).
The torch restatements below follow modules/optimizer.py's operations, per tensor, as the reference runs them.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from edgedict_b200 import optim                          # noqa: E402
from edgedict_b200.rnnt.models import FrontEnd, Transducer   # noqa: E402

E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0,
            dec_proj_size=256, joint_size=640)
E6D2_FE = dict(E6D2, input_size=128, enc_time_reductions=[])
TRAIN_FE = [(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3
HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable: %s" % e


# ---- torch restatements of the reference's classes (per tensor, as modules/optimizer.py runs them) -----------------
class RefSM3(torch.optim.Optimizer):
    def __init__(self, params, lr=0.1, eps=1e-30):
        super().__init__(params, dict(lr=lr, eps=eps))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            for p in group["params"]:
                grad, state = p.grad, self.state[p]
                r = grad.dim()
                if not state:
                    state["step"] = 0
                    shapes = [grad.shape] if r <= 1 else [[1] * i + [grad.shape[i]] + [1] * (r - 1 - i)
                                                         for i in range(r)]
                    state["acc"] = [torch.zeros(s, device=grad.device) for s in shapes]
                accs = state["acc"]
                update = accs[0].clone()
                for a in accs[1:]:
                    update = torch.min(update, a)
                update.addcmul_(grad, grad)
                for i, a in enumerate(accs):
                    nu = update
                    if r > 1:
                        for d in range(r):
                            if d != i:
                                nu = nu.max(dim=d, keepdim=True).values
                    a.copy_(nu)
                update.add_(group["eps"]).rsqrt_().mul_(grad)
                p.sub_(update, alpha=group["lr"])
                state["step"] += 1


class RefAdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                grad, state = p.grad, self.state[p]
                if not state:
                    state["step"], state["m"], state["v"] = 0, torch.zeros_like(p), torch.zeros_like(p)
                m, v = state["m"], state["v"]
                state["step"] += 1
                m.mul_(b1).add_(grad, alpha=1 - b1)
                v.mul_(b2).addcmul_(grad, grad, value=1 - b2)
                denom = v.sqrt().add_(group["eps"])
                step_size = group["lr"] * math.sqrt(1 - b2 ** state["step"]) / (1 - b1 ** state["step"])
                p.add_(torch.mul(p, group["weight_decay"]).addcdiv_(m, denom), alpha=-step_size)


class RefNovograd(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.95, 0.0), eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                grad, state = p.grad, self.state[p]
                if not state:
                    state["step"], state["m"] = 0, torch.zeros_like(p)
                    state["v"] = torch.zeros([], device=p.device)
                m, v = state["m"], state["v"]
                state["step"] += 1
                norm = torch.sum(torch.pow(grad, 2))
                if v == 0:                                     # the reference's host sync, per tensor per step
                    v.copy_(norm)
                else:
                    v.mul_(b2).add_(norm, alpha=1 - b2)
                grad.div_(v.sqrt().add_(group["eps"]))
                if group["weight_decay"] != 0:
                    grad.add_(p, alpha=group["weight_decay"])
                m.mul_(b1).add_(grad)
                p.add_(m, alpha=-group["lr"])


# ---- the runs ---------------------------------------------------------------------------------------------------------
def param_set(name):
    torch.manual_seed(0)
    if name == "E6D2":
        mods = [Transducer(**E6D2)]
    else:
        mods = [Transducer(**E6D2_FE), FrontEnd(TRAIN_FE, bias=True)]
    return [p.detach().clone() for m in mods for p in m.parameters()]


def fresh(ps):
    return [p.to("cuda").requires_grad_(True) for p in ps]


def fill_grads(params, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
        p.grad.copy_(torch.randn(p.shape, generator=g, device="cuda") * 1e-3)


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def state_bytes(opt):
    if isinstance(opt, optim.FlatOptimizer):
        sd = [opt.momentum_buffer] if isinstance(opt, optim.SGD) else \
            opt._acc[:1] if isinstance(opt, optim.SM3) else [opt.exp_avg, opt.exp_avg_sq]
        return sum(t.numel() * 4 for t in sd if t is not None)
    total = 0
    for st in opt.state.values():
        for v in st.values():
            for t in (v if isinstance(v, list) else [v]):
                if torch.is_tensor(t):
                    total += t.numel() * t.element_size()
    return total


# per-element fp32 streams one step moves: p read + write, g read, state read + write; + a gradient read for a norm
STREAMS = {"sgd": 5, "sm3": 3, "adamw": 7, "novograd": 6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim.py needs a CUDA device")
    rows = []
    for pset in ("E6D2", "FrontEnd+E6D2"):
        base = param_set(pset)
        n = sum(p.numel() for p in base)
        variants = [
            ("sgd", "engine SGD(momentum=0.9)", lambda ps: optim.SGD(ps, lr=1e-3, momentum=0.9), {}),
            ("sgd", "engine SGD(momentum=0.9) + clip", lambda ps: optim.SGD(ps, lr=1e-3, momentum=0.9),
             dict(max_norm=1.0)),
            ("sgd", "torch SGD(momentum=0.9, foreach=True)",
             lambda ps: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, foreach=True), None),
            ("sgd", "torch SGD(momentum=0.9, fused=True)",
             lambda ps: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, fused=True), None),
            ("sm3", "engine SM3", lambda ps: optim.SM3(ps, lr=0.1), {}),
            ("sm3", "torch restatement of the reference's SM3", lambda ps: RefSM3(ps, lr=0.1), None),
            ("adamw", "engine AdamW(wd=1e-5)", lambda ps: optim.AdamW(ps, lr=1e-3, weight_decay=1e-5), {}),
            ("adamw", "torch restatement of the reference's AdamW",
             lambda ps: RefAdamW(ps, lr=1e-3, weight_decay=1e-5), None),
            ("adamw", "torch AdamW(fused=True) (speed anchor; different formula)",
             lambda ps: torch.optim.AdamW(ps, lr=1e-3, weight_decay=1e-5, fused=True), None),
            ("novograd", "engine Novograd(wd=1e-3)", lambda ps: optim.Novograd(ps, lr=1e-3, weight_decay=1e-3), {}),
            ("novograd", "torch restatement of the reference's Novograd",
             lambda ps: RefNovograd(ps, lr=1e-3, weight_decay=1e-3), None),
        ]
        for kind, name, make, kw in variants:
            params = fresh(base)
            fill_grads(params, 7)
            opt = make(params)
            if isinstance(opt, optim.FlatOptimizer):
                fill_grads(params, 7)                  # the bucket's gradients

                def step(opt=opt, kw=kw):
                    opt.step(**kw)
            else:
                def step(opt=opt):
                    opt.step()
            ms = time_steps(step, args.steps, args.warmup)
            streams = STREAMS[kind] + (1 if kw and kw.get("max_norm") else 0)
            moved = streams * 4 * n
            row = dict(params=pset, numel=n, optimizer=name, step_ms=round(ms, 4),
                       state_bytes=state_bytes(opt), step_bytes=moved,
                       achieved_TBps=round(moved / (ms * 1e-3) / 1e12, 3),
                       share_of_3p35TBps=round(moved / (ms * 1e-3) / HBM, 3))
            print(json.dumps(row), flush=True)
            rows.append(row)
            del opt, params
            torch.cuda.empty_cache()
    result = dict(card=card(), steps=args.steps, warmup=args.warmup, rows=rows)
    print(json.dumps(dict(card=result["card"])))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
