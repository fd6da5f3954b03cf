#!/usr/bin/env python
"""N-best beam search against the best-only call, at the shapes of scripts/bench_beam.py and scripts/bench_ctc_beam.py.

  python scripts/bench_nbest.py [--reps K] [--rounds R]

Arms, alternated within every round (K timed calls each after a warm-up, CUDA events around them, one device
synchronise at the end):
  rnnt_W{4,8}, rnnt_nbest_W{4,8}         E6D2_LARGE Transducer.beam_search (weights x 2), B = 32 x 500 input frames
                                          (30 s of audio, T' = 250), without and with nbest = W;
  rnnt_lm_W{4,8}, rnnt_lm_nbest_W{4,8}   the same with a random LMModel(1024, 64, 1024, 2)-shaped LM fused;
  ctc_W{4,8,16}, ctc_nbest_W{4,8,16}     edgedict_b200.ctc.beam_search on the log-probs of bench_ctc_beam.py's GRU
                                          CTCEncoder (B = 32, T = 1000 -> T' = 500), without and with nbest = W.
Each model keeps one resident engine, so the N-best calls go through a shallow copy of the model with its own cache.
The BEAM_FINAL phase is then timed alone: a one-phase program over the history the last search left, best-only and
N-best, launched 20 times under torch.profiler (kernel time per launch, launch overhead excluded).
Prints one JSON line with the card (name, power limit) read in the same run."""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
CTC_CFG = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0, proj_size=640)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from edgedict_b200 import ctc
    from edgedict_b200.rnnt.models import CTCEncoder, Transducer
    from edgedict_b200 import stream_engine as se
    assert torch.cuda.is_available(), "bench_nbest.py measures on the GPU"
    dev = torch.device("cuda")

    torch.manual_seed(10)
    rnnt = Transducer(output_loss=False, **LARGE).eval()
    with torch.no_grad():
        for p in rnnt.parameters():
            p.mul_(2.0)
    rnnt.cuda()
    g = torch.Generator().manual_seed(0)
    xs = torch.randn(32, 500, 240, generator=g).cuda()
    xlen = torch.full((32,), 500, dtype=torch.int32)
    torch.manual_seed(11)
    lm = torch.nn.Module()
    lm.encoder = torch.nn.Embedding(1024, 64)
    lm.rnn = torch.nn.LSTM(64, 1024, 2, batch_first=True)
    lm.decoder = torch.nn.Linear(1024, 1024)
    lm = lm.eval().cuda()
    fuse = dict(lm=lm, lm_weight=0.5, length_bonus=1.0)
    models = {k: copy.copy(rnnt) for k in ("plain", "nbest", "lm", "lm_nbest")}

    torch.manual_seed(0)
    cm = CTCEncoder(**CTC_CFG).to(dev)
    with torch.no_grad():
        cm.tovocab[0].weight.mul_(8.0)
        lp = cm(torch.randn(32, 1000, 240, device=dev))
    lens = [lp.shape[1]] * 32

    arms = {}
    for W in (4, 8):
        arms["rnnt_W%d" % W] = lambda W=W: models["plain"].beam_search(xs, xlen, W=W)
        arms["rnnt_nbest_W%d" % W] = lambda W=W: models["nbest"].beam_search(xs, xlen, W=W, nbest=W)
        arms["rnnt_lm_W%d" % W] = lambda W=W: models["lm"].beam_search(xs, xlen, W=W, **fuse)
        arms["rnnt_lm_nbest_W%d" % W] = lambda W=W: models["lm_nbest"].beam_search(xs, xlen, W=W, nbest=W, **fuse)
    for W in (4, 8, 16):
        arms["ctc_W%d" % W] = lambda W=W: ctc.beam_search(lp, lens, W)
        arms["ctc_nbest_W%d" % W] = lambda W=W: ctc.beam_search(lp, lens, W, nbest=W)

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

    ms = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            ms[k].append(round(timed(fn), 2))
    med = {k: statistics.median(v) for k, v in ms.items()}

    # head check at the measured shape: entry 0 of every list is the best-only result, bit for bit
    ids, nlp = models["plain"].beam_search(xs, xlen, W=8)
    hyps = models["nbest"].beam_search(xs, xlen, W=8, nbest=8)
    head_ok = all(hyps[b][0].tokens.tolist() == ids[b] and
                  torch.tensor(hyps[b][0].nlogp, dtype=torch.float32).view(torch.int32).item() ==
                  nlp[b:b + 1].view(torch.int32).item() for b in range(32))

    # BEAM_FINAL alone, over the history the last N-best search of each engine left
    def final_program(eng, N, y, K):
        keep = (eng.nbest, eng.ids, eng.nlogp, eng.nbest_frames, eng.nbest_count)
        if N == 0:
            se.final_outputs(eng, eng.ids.shape[0], 0, eng.ids.shape[-1])
        ph = se.final_phase(eng, eng.W, y, K)
        out = se._upload([ph], eng.dev), (eng.ids, eng.nlogp)       # the buffers the phase writes stay referenced
        eng.nbest, eng.ids, eng.nlogp, eng.nbest_frames, eng.nbest_count = keep
        return out

    def kernel_us(entry, prog, bar):
        from torch.profiler import ProfilerActivity, profile
        for _ in range(3):
            se._launch(entry, prog, 1, bar, 0)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                se._launch(entry, prog, 1, bar, 0)
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "decode_program_kernel" in e.key]
        tot = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ev)
        return round(tot / max(1, sum(e.count for e in ev)), 1)

    final_us = {}
    reng = next(iter(models["nbest"]._beam_engines.values()))
    ceng = next(iter(ctc._beam_engines.values()))
    for tag, eng, y, K, entry in (("rnnt_W%d" % reng.W, reng, reng.logp, reng.max_symbols, "eb_decode_run"),
                                  ("ctc_W%d" % ceng.W, ceng, ceng.score, 1, "eb_decode_run_ctc")):
        for N in (0, eng.W):
            (prog, _bufs) = final_program(eng, N, y, K)
            final_us["%s_N%d" % (tag, N)] = kernel_us(entry, prog, eng._bar)

    print(json.dumps(dict(card=card(), reps=a.reps, rounds=a.rounds, rnnt_shape="E6D2_LARGE B=32 T=500 (T'=250)",
                          ctc_shape="GRU CTCEncoder B=32 T=1000 (T'=%d)" % lp.shape[1], ms=ms, median_ms=med,
                          nbest_over_best_only={k[:k.rindex("_W")].replace("_nbest", "") + k[k.rindex("_W"):]:
                                                round(med[k] / med[k.replace("_nbest", "")], 3)
                                                for k in med if "_nbest" in k},
                          beam_final_kernel_us=final_us, rnnt_W8_head_equals_best_only=head_ok)))


if __name__ == "__main__":
    main()
