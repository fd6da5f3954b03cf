#!/usr/bin/env python
"""CTC on the engine at E6D2 shape: a GRU CTCEncoder (6 x 1024 GRU layers, time reduction after layer 1, proj 640,
V = 1024, input 240), B = 32, T = 1000 -> T' = 500, S = 128 labels per utterance.

  python scripts/bench_ctc.py [--rounds N] [--reps K]

Three comparisons, each alternated within every round (K timed calls per arm after a warm-up), so both arms see the same
clocks and neighbours:
  loss : CTC loss forward + backward on the same log-probs [T', B, V], edgedict_b200.ctc.ctc_loss against torch's CUDA
         F.ctc_loss (reduction 'mean');
  step : the full training step (forward, loss, backward) in fp32 and in bf16 mode;
  greedy: CTCEncoder.greedy_decode (encoder + head + eb_ctc_greedy + one copy) against the reference's torch decode
         (rnnt/models.py:294-310: max, masks, a per-utterance loop with one copy each) after the engine's forward, and
         the decode stage alone (both arms from the same log-probs).
Prints one JSON line: the card (name, power limit) read in the same run and ms per call for every round.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, S = 32, 1000, 128
CFG = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0, proj_size=640)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def reference_decode(logprobs, xlen, blank):
    """rnnt/models.py:297-310 on the device log-probs, as the reference runs it."""
    import torch
    import torch.nn.functional as F
    logprob, y_seq = logprobs.max(dim=-1)
    unique = F.pad(y_seq[:, 1:] != y_seq[:, :-1], [1, 0, 0, 0], value=True).bool()
    masks = ((y_seq != blank).int() * unique.int()).bool()
    out, log_p = [], []
    for seq, lp, n, mask in zip(y_seq, logprobs, xlen, masks):
        mask = mask[:n]
        out.append(seq[:n][mask].cpu().numpy())
        log_p.append(lp[:n][mask].sum())
    return out, -torch.stack(log_p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from edgedict_b200.ctc import CTCLoss, ctc_loss
    from edgedict_b200.rnnt.models import CTCEncoder
    assert torch.cuda.is_available(), "bench_ctc.py measures on the GPU"
    torch.manual_seed(0)
    dev = torch.device("cuda")
    m = CTCEncoder(**CFG).to(dev)
    xs = torch.randn(B, T, CFG["input_size"], device=dev)
    Tp = (T + 1) // 2
    ys = torch.randint(1, CFG["vocab_size"], (B, S), device=dev)
    il = torch.full((B,), Tp, dtype=torch.long)
    tl = torch.full((B,), S, dtype=torch.long)
    xlen = torch.full((B,), T, dtype=torch.long)
    with torch.no_grad():
        lp_btv = m(xs)
    lp = lp_btv.transpose(0, 1).contiguous()              # [T', B, V], the layout both loss arms get

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.reps

    def loss_ours():
        x = lp.detach().requires_grad_()
        ctc_loss(x, ys, il, tl).backward()

    def loss_torch():
        x = lp.detach().requires_grad_()
        F.ctc_loss(x, ys, il, tl).backward()

    crit = CTCLoss()

    def step(precision):
        def run():
            m.set_precision(precision)
            m.zero_grad(set_to_none=True)
            crit(m(xs).transpose(0, 1), ys, il, tl).backward()
        return run

    def greedy_ours():
        m.set_precision("fp32")
        m.greedy_decode(xs, xlen)

    def greedy_reference():
        m.set_precision("fp32")
        with torch.no_grad():
            reference_decode(m(xs), xlen, m.blank)

    from edgedict_b200 import ops
    xl_dev = xlen.to(torch.int32).clamp(max=Tp).to(dev)

    def decode_ours():
        ops.ctc_greedy(lp_btv, xl_dev, 0).cpu()

    def decode_reference():
        reference_decode(lp_btv, xlen, 0)

    arms = dict(loss_ours=loss_ours, loss_torch=loss_torch, step_fp32=step("fp32"), step_bf16=step("bf16"),
                greedy_ours=greedy_ours, greedy_reference=greedy_reference, decode_ours=decode_ours,
                decode_reference=decode_reference)
    res = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            res[k].append(round(timed(fn), 3))
    # the two loss arms on the same log-probs: how far apart the values are
    x1, x2 = lp.detach().requires_grad_(), lp.detach().requires_grad_()
    l1, l2 = ctc_loss(x1, ys, il, tl), F.ctc_loss(x2, ys, il, tl)
    (l1 + l2).backward()
    print(json.dumps(dict(card=card(), B=B, T=T, T_out=Tp, S=S, V=CFG["vocab_size"], reps=a.reps, ms=res,
                          loss_rel_diff=abs(float(l1.detach()) - float(l2.detach())) / abs(float(l2.detach())),
                          grad_max_abs_diff=float((x1.grad - x2.grad).abs().max()))))


if __name__ == "__main__":
    main()
