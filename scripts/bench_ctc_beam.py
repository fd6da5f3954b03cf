#!/usr/bin/env python
"""CTC prefix beam search on the engine at scripts/bench_ctc.py's shape: a GRU CTCEncoder (6 x 1024 GRU layers, time
reduction after layer 1, proj 640, V = 1024, input 240), B = 32, T = 1000 -> T' = 500.

  python scripts/bench_ctc_beam.py [--rounds N] [--reps K] [--loop-utts U]

Arms, alternated within every round (K timed calls per arm after a warm-up, CUDA events around them):
  decode_W{1,4,8,16}       edgedict_b200.ctc.beam_search on the same device log-probs, no LM (the decode stage alone:
                           the copy into the engine, one persistent launch, one device-to-host copy of the ids);
  decode_lm_W{4,8}         the same with an LMModel(1024, 64, 1024, 2)-shaped LM, lm_weight 0.5, length_bonus 0.5;
  e2e_W{4,8}, e2e_lm_W4    CTCEncoder.beam_search (forward in fp32 mode, then the search);
  greedy_decode, greedy_e2e   ops.ctc_greedy on the log-probs (and one copy), and CTCEncoder.greedy_decode: the anchor.
The per-utterance Python loop it replaces (tests/ctc_beam_oracle.py's restatement, numpy fp32, W = 4) is timed on U
utterances with a host clock and reported per utterance.
Prints one JSON line: the card (name, power limit) read in the same run, ms per call for every round and the medians.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T = 32, 1000
CFG = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0, proj_size=640)


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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-utts", type=int, default=2)
    a = ap.parse_args()
    import numpy as np
    import torch
    from edgedict_b200 import ctc, ops
    from edgedict_b200.rnnt.models import CTCEncoder
    from tests.ctc_beam_oracle import prefix_beam_search
    assert torch.cuda.is_available(), "bench_ctc_beam.py measures on the GPU"
    torch.manual_seed(0)
    dev = torch.device("cuda")
    m = CTCEncoder(**CFG).to(dev)
    with torch.no_grad():
        m.tovocab[0].weight.mul_(8.0)            # peaked log-probs, as a trained model gives
    lm = torch.nn.Module()
    lm.encoder = torch.nn.Embedding(1024, 64)
    lm.rnn = torch.nn.LSTM(64, 1024, 2, batch_first=True)
    lm.decoder = torch.nn.Linear(1024, 1024)
    lm = lm.to(dev).eval()
    xs = torch.randn(B, T, CFG["input_size"], device=dev)
    xlen = torch.full((B,), T, dtype=torch.long)
    with torch.no_grad():
        lp = m(xs)
    Tp = lp.shape[1]
    lens = [Tp] * B
    xl_dev = torch.full((B,), Tp, dtype=torch.int32, device=dev)
    fuse = dict(lm=lm, lm_weight=0.5, length_bonus=0.5)

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

    arms = {}
    for W in (1, 4, 8, 16):
        arms["decode_W%d" % W] = (lambda W=W: ctc.beam_search(lp, lens, W))
    for W in (4, 8):
        arms["decode_lm_W%d" % W] = (lambda W=W: ctc.beam_search(lp, lens, W, **fuse))
        arms["e2e_W%d" % W] = (lambda W=W: m.beam_search(xs, xlen, W=W))
    arms["e2e_lm_W4"] = lambda: m.beam_search(xs, xlen, W=4, **fuse)
    arms["greedy_decode"] = lambda: ops.ctc_greedy(lp, xl_dev, 0).cpu()
    arms["greedy_e2e"] = lambda: m.greedy_decode(xs, xlen)
    res = {k: [] for k in arms}
    # every arm in every round rebuilds its engine once (one resident program): the warm-up call of timed() pays it
    for _ in range(a.rounds):
        for k, fn in arms.items():
            res[k].append(round(timed(fn), 3))
    host = lp[:a.loop_utts].cpu().numpy()
    t0 = time.perf_counter()
    for b in range(a.loop_utts):
        prefix_beam_search(host[b], Tp, 4, 0, dtype=np.float32)
    loop_ms = (time.perf_counter() - t0) * 1e3 / a.loop_utts
    ids4, _ = ctc.beam_search(lp, lens, 4)
    ref4 = prefix_beam_search(host[0], Tp, 4, 0, dtype=np.float32)[0]
    print(json.dumps(dict(card=card(), B=B, T=T, T_out=Tp, V=CFG["vocab_size"], reps=a.reps, ms=res,
                          median_ms={k: statistics.median(v) for k, v in res.items()},
                          python_loop_W4_ms_per_utt=round(loop_ms, 1),
                          python_loop_W4_ms_per_batch_est=round(loop_ms * B, 1),
                          utt0_ids_equal_restatement=tuple(ids4[0].tolist()) == tuple(ref4),
                          mean_len_W4=float(np.mean([len(i) for i in ids4])))))


if __name__ == "__main__":
    main()
