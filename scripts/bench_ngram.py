#!/usr/bin/env python
"""N-gram shallow fusion in the device beam searches: the cost of the n-gram term, arms alternated per round.

  python scripts/bench_ngram.py [--lib PARENT.so] [--rounds R] [--out FILE]

The ARPA files are made here, in a temporary directory, from a seeded Zipf / Markov token corpus over V = 1024
(token 3-grams of about 10^5 entries and 4-grams of about 10^6, counts turned into discounted log10 probabilities with
one backoff weight per history).  Reported per model: host load-and-compile time (NgramLM) and table bytes.

Arms (one run each per round, CUDA events around it, the order reversed every other round):
  rnnt W{4,8} lm{0,1} ng{0,3,4}   BeamEngine (the device part of Transducer.beam_search) over B = 32 x 30 s of
                                   E6D2_LARGE encoder output (T' = 250, weights x 2), with and without an
                                   LMModel(1024, 64, 1024, 2)-shaped LM (lm_weight 0.5, length_bonus 3), without the
                                   n-gram and with the 3-gram / 4-gram (ngram_weight 0.3);
  ctc W{4,8,16} ng{0,3,4}          CTCBeamEngine, the decode stage of ctc.beam_search, at bench_ctc_beam.py's shape
                                   (B = 32, T' = 500, V = 1024) on random log-probs (3 randn, log-softmax), and at
                                   W = 4 with the LM.
With --lib (a build of the parent commit: the same EbPhase layout) every no-n-gram arm also runs through that library
in the same process; the outputs are compared bit for bit and the two are timed as arms of their own.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
B, T_RNNT, T_CTC, V = 32, 250, 500, 1024


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable: %s" % e


def make_arpa(path, order, n_tokens, seed, D=0.7):
    """An ARPA file of ``order`` over tokens 1..V-1 (0 is blank) and </s> from a Zipf / Markov corpus of about
    n_tokens tokens: absolute-discounted relative frequencies, backoff log10 -0.4 for every history."""
    rng = np.random.default_rng(seed)
    nt = V - 1
    zipf = 1.0 / np.arange(1, nt + 1) ** 1.1
    zipf /= zipf.sum()
    shift = rng.integers(0, nt, size=nt)
    toks = np.empty(n_tokens, dtype=np.int64)
    cur = int(rng.integers(nt))
    draws = rng.choice(nt, size=n_tokens, p=zipf)
    for i in range(n_tokens):                                  # next token: a Zipf draw shifted by the current one
        cur = (draws[i] + shift[cur]) % nt
        toks[i] = cur + 1
    sent = np.where(rng.random(n_tokens) < 0.05, V, toks)      # V: </s>, which also starts the next sentence
    words = lambda k: "</s>" if k == V else str(k)
    with open(path, "w") as fh:
        grams = []
        for m in range(1, order + 1):
            keys = np.stack([sent[j:len(sent) - m + 1 + j] for j in range(m)], 1)
            if m > 1:
                keys = keys[(keys[:, :-1] != V).all(1)]        # </s> only last
            u, c = np.unique(keys, axis=0, return_counts=True)
            hist = {}
            for row, cnt in zip(map(tuple, u[:, :-1]), c):
                hist[row] = hist.get(row, 0) + cnt
            p = np.array([max(cnt - D, 0.1) / hist[tuple(r[:-1])] for r, cnt in zip(u, c)])
            grams.append((u, np.log10(p)))
        fh.write("\\data\\\n")
        for m, (u, _) in enumerate(grams, 1):
            fh.write("ngram %d=%d\n" % (m, len(u) + (m == 1)))
        for m, (u, lp) in enumerate(grams, 1):
            fh.write("\n\\%d-grams:\n" % m)
            if m == 1:
                fh.write("-99\t<s>\t-0.4\n")
            bo = "\t-0.4" if m < order else ""
            fh.write("".join("%.6f\t%s%s\n" % (x, " ".join(words(k) for k in r), bo if r[-1] != V else "")
                             for r, x in zip(u, lp)))
        fh.write("\n\\end\\\n")
    return sum(len(u) for u, _ in grams)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import edgedict_b200.stream_engine as se
    from edgedict_b200.ngram import NgramLM
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import BeamEngine, CTCBeamEngine
    assert torch.cuda.is_available(), "bench_ngram.py measures on the GPU"
    other = None
    if args.lib:
        other = C.CDLL(os.path.abspath(args.lib))
        for n in ("eb_decode_run", "eb_decode_run_ctc"):
            getattr(other, n).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
            getattr(other, n).restype = C.c_int
        assert other.eb_decode_phase_size() == C.sizeof(se.EbPhase), "--lib must have this EbPhase layout"
    own_launch = se._launch

    def run(eng, h, lens, parent=False):
        if not parent:
            return eng.run(h, lens)

        def launch(entry, prog, nphase, bar, max_ctas):
            rc = getattr(other, entry)(prog.data_ptr(), nphase, bar.data_ptr(), max_ctas,
                                       torch.cuda.current_stream().cuda_stream)
            assert rc == 0, (entry, rc)
        se._launch = launch
        try:
            return eng.run(h, lens)
        finally:
            se._launch = own_launch

    models, host = {0: None}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for order, n_tok in ((3, 60000), (4, 400000)):
            path = os.path.join(tmp, "m%d.arpa" % order)
            entries = make_arpa(path, order, n_tok, seed=order)
            t0 = time.perf_counter()
            models[order] = NgramLM(path, V)
            host[order] = dict(arpa_entries=entries, load_s=round(time.perf_counter() - t0, 2),
                               states=models[order].n_states, children=models[order].n_children,
                               table_bytes=models[order].nbytes)
    torch.manual_seed(10)
    model = Transducer(output_loss=False, **LARGE).eval()
    with torch.no_grad():
        for p in model.parameters():
            p.mul_(2.0)
        model.joint.joint[2].bias[0] += 3.0            # about half the frames emit (bench_beam_multi_symbol.py)
    model.cuda()
    torch.manual_seed(11)
    lm = torch.nn.Module()
    lm.encoder, lm.rnn, lm.decoder = torch.nn.Embedding(1024, 64), torch.nn.LSTM(64, 1024, 2, batch_first=True), \
        torch.nn.Linear(1024, 1024)
    with torch.no_grad():
        for p in lm.parameters():
            p.mul_(3.0)
    lm = lm.eval().cuda()
    g = torch.Generator().manual_seed(0)
    h_enc = torch.randn(B, T_RNNT, 640, generator=g).cuda()
    fr_rnnt = torch.full((B,), T_RNNT, dtype=torch.int32, device="cuda")
    lp = (3.0 * torch.randn(B, T_CTC, V, generator=g)).log_softmax(-1).cuda()
    fr_ctc = torch.full((B,), T_CTC, dtype=torch.int32, device="cuda")

    arms = {}
    for W in (4, 8):
        for use_lm in (False, True):
            kw = dict(lm=lm, lm_weight=0.5, length_bonus=3.0) if use_lm else {}
            for n, ng in models.items():
                t0 = time.perf_counter()
                eng = BeamEngine(model, B, T_RNNT, W, ngram=ng, ngram_weight=0.3 if ng else 0.0, **kw)
                arms["rnnt_W%d_lm%d_ng%d" % (W, use_lm, n)] = (eng, h_enc, fr_rnnt, False)
                if n == 0 and other is not None:
                    arms["rnnt_W%d_lm%d_ng0_parent" % (W, use_lm)] = (eng, h_enc, fr_rnnt, True)
    for W in (4, 8, 16):
        for n, ng in models.items():
            eng = CTCBeamEngine(B, T_CTC, V, W, ngram=ng, ngram_weight=0.3 if ng else 0.0, device="cuda")
            arms["ctc_W%d_ng%d" % (W, n)] = (eng, lp, fr_ctc, False)
            if n == 0 and other is not None:
                arms["ctc_W%d_ng0_parent" % W] = (eng, lp, fr_ctc, True)
    for n, ng in models.items():                           # W = 4 with the LM: the program runs the LM's matrix phases
        eng = CTCBeamEngine(B, T_CTC, V, 4, lm=lm, lm_weight=0.5, length_bonus=3.0, ngram=ng,
                            ngram_weight=0.3 if ng else 0.0, device="cuda")
        arms["ctc_W4_lm1_ng%d" % n] = (eng, lp, fr_ctc, False)
        if n == 0 and other is not None:
            arms["ctc_W4_lm1_ng0_parent"] = (eng, lp, fr_ctc, True)

    same_bits = {}
    for name, (eng, h, lens, parent) in arms.items():      # warm-up, and the parent's bits against this tree's
        out = [t.clone() for t in run(eng, h, lens, parent)]
        if parent:
            mine = run(eng, h, lens)
            same_bits[name] = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(out, mine))
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = {k: [] for k in arms}
    names = list(arms)
    for r in range(args.rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            eng, h, lens, parent = arms[name]
            ev[0].record()
            run(eng, h, lens, parent)
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]))
    res = dict(card=card(), host=host, rounds=args.rounds, same_bits_as_parent=same_bits,
               ms_median={k: round(statistics.median(v), 2) for k, v in times.items()},
               ms_min={k: round(min(v), 2) for k, v in times.items()})
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
