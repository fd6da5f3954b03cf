#!/usr/bin/env python
"""Language-model training at cli/train_lm.py's shape: LMModel(1024, 64, 1024, 2) (dropout 0.5, train mode), B = 256,
S = 64 and 128 synthetic tokens, about 10 % of the targets padding (trailing 0s, ignored by NLLLoss(ignore_index=0)).

  python scripts/bench_lm.py [--rounds N] [--steps K] [--warmup W]

A step is cli/train_lm.py's: forward, loss, backward, clip_grad_norm_(1.0), Adam.  Arms, alternated within every round
(K timed steps per arm after W warm-up steps), so all see the same clocks and neighbours:
  torch        : a torch restatement of the reference's LMModel (nn.Embedding, nn.LSTM on cuDNN, nn.Linear,
                 F.log_softmax, nn.NLLLoss), torch.optim.Adam and clip_grad_norm_, fp32 -- the reference's own step;
  dropin_fp32  : edgedict_b200.models.LMModel(input) + nn.NLLLoss, FlatAdam(max_norm=1.0), fp32 mode;
  fused_fp32   : LMModel.loss (output layer + cross-entropy in one node), FlatAdam(max_norm=1.0), fp32 mode;
  dropin_bf16, fused_bf16 : the same in bf16 mode.
Also per S: an eval pass (no gradients, per-token costs) in tokens per second for torch and the fused arms, the peak
device memory of one training step per arm, and the per-kernel split of one step of each fused arm (ops._timed: the
recurrence is lstm_*; "other" is the step time no timed kernel covers).  Prints one JSON line with the card (name,
power limit) read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NTOKEN, NINP, NHID, NLAYERS, B = 1024, 64, 1024, 2, 256


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def torch_lm():
    """The reference's LMModel (models.py:224-261), restated: its sources are not needed to run this benchmark."""
    import torch.nn as nn
    import torch.nn.functional as F

    class RefLM(nn.Module):
        def __init__(self):
            super().__init__()
            self.drop = nn.Dropout(0.5)
            self.encoder = nn.Embedding(NTOKEN, NINP)
            self.rnn = nn.LSTM(NINP, NHID, NLAYERS, dropout=0.5, batch_first=True)
            self.decoder = nn.Linear(NHID, NTOKEN)
            nn.init.uniform_(self.encoder.weight, -0.1, 0.1)
            nn.init.zeros_(self.decoder.weight)
            nn.init.uniform_(self.decoder.weight, -0.1, 0.1)

        def forward(self, x, hidden):
            out, hidden = self.rnn(self.drop(self.encoder(x)), hidden)
            return F.log_softmax(self.decoder(self.drop(out)).view(-1, NTOKEN), dim=-1), hidden

    return RefLM()


def batch(S, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    tg = torch.randint(2, NTOKEN, (B, S), generator=g)
    lens = S - (torch.rand(B, generator=g) * 0.2 * S).long()          # mean 10 % padding
    tg[torch.arange(S)[None] >= lens[:, None]] = 0
    inp = torch.cat([torch.ones(B, 1, dtype=torch.long), tg[:, :-1]], 1)
    return inp.cuda(), tg.cuda()


def make_arms():
    import torch
    import torch.nn as nn
    from edgedict_b200.models import LMModel
    from edgedict_b200.optim import FlatAdam
    crit = nn.NLLLoss(ignore_index=0)
    arms = {}
    torch.manual_seed(0)
    ref = torch_lm().cuda().train()
    opt = torch.optim.Adam(ref.parameters(), lr=1e-4)

    def torch_step(inp, tg, ref=ref, opt=opt):
        ref.zero_grad()
        logp, _ = ref(inp, None)
        loss = crit(logp, tg.flatten())
        loss.backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 1.0)
        opt.step()
        return loss

    def torch_eval(inp, tg, ref=ref):
        with torch.no_grad():
            logp, _ = ref.eval()(inp, None)
            ref.train()
            return nn.functional.nll_loss(logp, tg.flatten(), ignore_index=0, reduction="none")

    arms["torch"] = (torch_step, torch_eval, ref)
    for prec in ("fp32", "bf16"):
        for kind in ("dropin", "fused"):
            torch.manual_seed(0)
            m = LMModel(NTOKEN, NINP, NHID, NLAYERS).cuda().train().set_precision(prec)
            o = FlatAdam(m, lr=1e-4)

            def step(inp, tg, m=m, o=o, fused=kind == "fused"):
                o.zero_grad()
                loss = m.loss(inp, tg) if fused else crit(m(inp)[0], tg.flatten())
                loss.backward()
                o.step(max_norm=1.0)
                return loss

            def ev(inp, tg, m=m):
                with torch.no_grad():
                    out = m.eval().loss(inp, tg, reduction="none")
                    m.train()
                    return out

            arms["%s_%s" % (kind, prec)] = (step, ev if kind == "fused" else None, m)
    return arms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seq", type=int, nargs="*", default=[64, 128])
    a = ap.parse_args()
    import torch
    from edgedict_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_lm.py needs a CUDA device")
    arms = make_arms()
    res = dict(card=card(), model=[NTOKEN, NINP, NHID, NLAYERS], B=B, rounds=a.rounds, steps=a.steps, by_S={})
    for S in a.seq:
        inp, tg = batch(S, S)
        r = dict(pad_fraction=float((tg == 0).float().mean()), step_ms={k: [] for k in arms}, eval_tok_s={},
                 peak_mb={}, split={})
        for k, (step, _, _) in arms.items():
            for _ in range(a.warmup):
                step(inp, tg)
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k, (step, _, _) in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    step(inp, tg)
                e1.record()
                torch.cuda.synchronize()
                r["step_ms"][k].append(round(e0.elapsed_time(e1) / a.steps, 3))
        for k, (step, ev, _) in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            step(inp, tg)
            torch.cuda.synchronize()
            r["peak_mb"][k] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
            if ev is None:
                continue
            ev(inp, tg)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                ev(inp, tg)
            e1.record()
            torch.cuda.synchronize()
            r["eval_tok_s"][k] = round(B * S * a.steps / (e0.elapsed_time(e1) / 1e3))
        for k in ("fused_fp32", "fused_bf16"):
            step = arms[k][0]
            ops.PROF.reset()
            ops.PROF.enabled = True
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(inp, tg)
            e1.record()
            torch.cuda.synchronize()
            ops.PROF.enabled = False
            total = e0.elapsed_time(e1)
            sp = {n: round(d["ms_sum"], 3) for n, d in sorted(ops.PROF.summary().items(), key=lambda x: -x[1]["ms_sum"])}
            rec = sum(v for n, v in sp.items() if n.startswith("lstm"))
            sp["other"] = round(total - sum(sp.values()), 3)
            r["split"][k] = dict(step_ms=round(total, 3), recurrence_share=round(rec / total, 3), kernels=sp)
        r["step_ms_median"] = {k: sorted(v)[len(v) // 2] for k, v in r["step_ms"].items()}
        res["by_S"][S] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
