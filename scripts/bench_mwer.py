#!/usr/bin/env python
"""Minimum word error rate training steps against the plain training step, and the edit distance alone.

  python scripts/bench_mwer.py [--reps K] [--rounds R]

Arms (CUDA events, K calls per arm after a warm-up, arms alternated within every round):
  * E6D2 Transducer in bf16 (bench.py's model), T = 1000 input frames (T' = 500), U = 128 reference tokens, W = N = 4,
    B = 16 and 32: ``mwer_loss(...).backward()`` against ``forward(...).backward()``.  The joint's output bias favours
    blank by +4 so that the random model's beam emits few tokens, as a trained model's hypotheses are about as long as
    the reference: the joint then covers B*(N+1) rows x 500 x 129 (Umax is printed).  The step is split into the stages
    timed on their own (encoder forward, beam search, pack + edit distance) and, by difference, the predictor + joint +
    loss forward and the backward; peak memory of one step.
  * The GRU CTCEncoder at scripts/bench_ctc.py's shape (B = 32, T = 1000, S = 128, V = 1024) in bf16: the same split.
  * eb_edit_distance alone on 32 x 4 pairs of 128 and 1024 tokens, in tokens and in words (CharTokenizer-style table,
    one separator in 6 tokens), against the one-thread Python restatement (tests/mwer_oracle.py) per pair.
Prints one JSON line with the card (name, power limit) read in the same run."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0,
            dec_proj_size=256, joint_size=640)
CTC_CFG = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0, proj_size=640)
T, U, W = 1000, 128, 4


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    import torch
    from edgedict_b200 import mwer
    from edgedict_b200.rnnt.models import CTCEncoder, Transducer, _ctc_frames, scale_length
    from edgedict_b200.stream_engine import BeamEngine, CTCBeamEngine
    from tests import mwer_oracle as mo
    assert torch.cuda.is_available(), "bench_mwer.py measures on the GPU"
    dev = torch.device("cuda")
    out = dict(card=card(), reps=a.reps, rounds=a.rounds)

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

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        return round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)

    # ---- transducer --------------------------------------------------------------------------------------------------
    torch.manual_seed(0)
    m = Transducer(**E6D2).to(dev)
    with torch.no_grad():
        m.joint.joint[2].bias[m.blank] += 4.0
    m.set_precision("bf16")
    for B in (16, 32):
        xs = torch.randn(B, T, E6D2["input_size"], device=dev)
        ys = torch.randint(4, E6D2["vocab_size"], (B, U), dtype=torch.int32, device=dev)
        xlen, ylen = torch.full((B,), T), torch.full((B,), U)

        def plain():
            m.zero_grad(set_to_none=True)
            m(xs, ys, xlen, ylen).backward()

        def step():
            m.zero_grad(set_to_none=True)
            m.mwer_loss(xs, ys, xlen, ylen, W=W).backward()

        def fwd():
            with torch.no_grad():
                m.mwer_loss(xs, ys, xlen, ylen, W=W)

        def enc():
            with torch.no_grad():
                m.encoder(xs)

        with torch.no_grad():
            h_enc, _ = m.encoder(xs)
        xl = scale_length(h_enc.shape[1], xlen).to(torch.int32).to(dev)
        eng = BeamEngine(m, B, h_enc.shape[1], W, merge=True, nbest=W)
        buf = eng.run(h_enc, xl)

        def beam():
            eng.run(h_enc, xl)

        def rows():
            mwer.nbest_rows(buf, B, W, eng.ids.shape[-1], ys, ylen, None, E6D2["vocab_size"])

        r = {k: [] for k in ("plain", "mwer_step", "mwer_fwd", "encoder", "beam", "pack_edit_distance")}
        for _ in range(a.rounds):
            for k, fn in (("plain", plain), ("mwer_step", step), ("mwer_fwd", fwd), ("encoder", enc), ("beam", beam),
                          ("pack_edit_distance", rows)):
                r[k].append(round(timed(fn), 2))
        best = {k: min(v) for k, v in r.items()}
        out["rnnt_B%d" % B] = dict(
            ms=r, umax=mwer.nbest_rows(buf, B, W, eng.ids.shape[-1], ys, ylen)[0].shape[1],
            predictor_joint_loss_fwd_ms_by_difference=round(best["mwer_fwd"] - best["encoder"] - best["beam"]
                                                            - best["pack_edit_distance"], 2),
            backward_ms_by_difference=round(best["mwer_step"] - best["mwer_fwd"], 2),
            peak_gib=dict(plain=peak(plain), mwer=peak(step)))
        del eng, buf, h_enc
        torch.cuda.empty_cache()
    del m
    torch.cuda.empty_cache()

    # ---- CTC ---------------------------------------------------------------------------------------------------------
    torch.manual_seed(0)
    B = 32
    c = CTCEncoder(**CTC_CFG).to(dev)
    c.set_precision("bf16")
    xs = torch.randn(B, T, CTC_CFG["input_size"], device=dev)
    ys = torch.randint(4, CTC_CFG["vocab_size"], (B, U), dtype=torch.int32, device=dev)
    xlen, ylen = torch.full((B,), T), torch.full((B,), U)
    from edgedict_b200.ctc import ctc_loss

    def cplain():
        c.zero_grad(set_to_none=True)
        lp = c(xs)
        ctc_loss(lp.transpose(0, 1), ys, _ctc_frames(lp.shape[1], xlen, B), ylen).backward()

    def cstep():
        c.zero_grad(set_to_none=True)
        c.mwer_loss(xs, ys, xlen, ylen, W=W).backward()

    def cfwd():
        with torch.no_grad():
            c.mwer_loss(xs, ys, xlen, ylen, W=W)

    def cenc():
        with torch.no_grad():
            c(xs)

    with torch.no_grad():
        lp = c(xs)
    frames = _ctc_frames(lp.shape[1], xlen, B).to(torch.int32).to(dev)
    ceng = CTCBeamEngine(B, lp.shape[1], CTC_CFG["vocab_size"], W, device=dev, nbest=W)
    cbuf = ceng.run(lp, frames)

    def cbeam():
        ceng.run(lp, frames)

    def crows():
        mwer.nbest_rows(cbuf, B, W, lp.shape[1], ys, ylen, None, CTC_CFG["vocab_size"])

    r = {k: [] for k in ("plain", "mwer_step", "mwer_fwd", "encoder", "beam", "pack_edit_distance")}
    for _ in range(a.rounds):
        for k, fn in (("plain", cplain), ("mwer_step", cstep), ("mwer_fwd", cfwd), ("encoder", cenc), ("beam", cbeam),
                      ("pack_edit_distance", crows)):
            r[k].append(round(timed(fn), 2))
    best = {k: min(v) for k, v in r.items()}
    out["ctc_gru_B32"] = dict(ms=r, umax=mwer.nbest_rows(cbuf, B, W, lp.shape[1], ys, ylen)[0].shape[1],
                              loss_fwd_ms_by_difference=round(best["mwer_fwd"] - best["encoder"] - best["beam"]
                                                              - best["pack_edit_distance"], 2),
                              backward_ms_by_difference=round(best["mwer_step"] - best["mwer_fwd"], 2),
                              peak_gib=dict(plain=peak(cplain), mwer=peak(cstep)))
    del c, ceng, cbuf, lp
    torch.cuda.empty_cache()

    # ---- edit distance alone ------------------------------------------------------------------------------------------
    rng = random.Random(0)
    pieces = ["<nul>", "<pad>", "<bos>", "<unk>", " "] + [chr(ord("a") + k) for k in range(26)]
    table = mwer.word_table(pieces)
    ed = {}
    for L in (128, 1024):
        ref = [[rng.choice(range(4, 31)) if rng.random() > 1 / 6 else 4 for _ in range(L)] for _ in range(32)]
        hyp = [[t if rng.random() > 0.1 else rng.choice(range(4, 31)) for t in ref[k // 4]] for k in range(128)]
        h = torch.tensor(hyp, dtype=torch.int32, device=dev)
        rr = torch.tensor(ref, dtype=torch.int32, device=dev)
        hl, rl, idx = [L] * 128, [L] * 32, [k // 4 for k in range(128)]
        for unit, tab in (("tokens", None), ("words", table)):
            ms = min(timed(lambda: mwer.edit_distance(h, hl, rr, rl, idx, tab)) for _ in range(a.rounds))
            npy = 8 if L == 128 else 1
            t0 = time.perf_counter()
            for k in range(npy):
                if tab is None:
                    mo.levenshtein(ref[idx[k]], hyp[k])
                else:
                    ents, chs = tab.entries.tolist(), tab.chars.tolist()
                    mo.levenshtein(mo.words(ref[idx[k]], ents, chs), mo.words(hyp[k], ents, chs))
            py_pair_ms = (time.perf_counter() - t0) * 1e3 / npy
            ed["%s_%d" % (unit, L)] = dict(device_ms_128_pairs=round(ms, 3),
                                           python_one_thread_ms_per_pair=round(py_pair_ms, 2),
                                           python_128_pairs_ms_extrapolated=round(128 * py_pair_ms, 1))
    out["edit_distance"] = ed
    print(json.dumps(out))


if __name__ == "__main__":
    main()
