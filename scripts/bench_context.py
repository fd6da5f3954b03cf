#!/usr/bin/env python
"""Contextual biasing in the device beam searches: the cost of the phrase automaton's term, arms alternated per round.

  python scripts/bench_context.py [--lib PARENT.so] [--rounds R] [--out FILE]
  python scripts/bench_context.py --stream [--lib PARENT.so] [--rounds R] [--chunks C] [--out FILE]

Arms (one run each per round, CUDA events around it, the order reversed every other round):
  rnnt W{4,8} lm{0,1} ctx{0,100,1000,5000}   BeamEngine (the device part of Transducer.beam_search) over B = 32 x 30 s
                                              of E6D2_LARGE encoder output (T' = 250, weights x 2), with and without
                                              an LMModel(1024, 64, 1024, 2)-shaped LM (lm_weight 0.5, length_bonus 3),
                                              and graphs of 0 / 100 / 1000 / 5000 random 2-6-token phrases (boost 1.5);
  ctc W{4,8,16} ctx{0,100,1000,5000}          CTCBeamEngine, the decode stage of ctc.beam_search, at
                                              bench_ctc_beam.py's shape (B = 32, T' = 500, V = 1024) on random
                                              log-probs (3 randn, log-softmax).
With --lib (a build of the parent commit, whose EbPhase lacks the trailing ctx pointer) every no-context arm also runs
through that library, its program repacked into the parent's layout, and the outputs are compared bit for bit.

--stream measures the streaming beams instead, each stream carrying its automaton state across chunks:
  srnnt W{4,8} lm{0,1} ctx{0,100,1000,5000}  StreamBeamEngine on bench_stream_beam.py's workload: E6D2_LARGE (weights
                                              x 2), 64 streams x C chunks of [64, 2, 240] log-mel (120 ms each), W = 4
                                              and 8, and W = 4 with the LMModel(1024, 64, 1024, 2)-shaped LM
                                              (lm_weight 0.3, length_bonus 0.5);
  sctc W{4,8} ctx{0,100,1000,5000}            CTCStreamBeamEngine on bench_ctc_stream_beam.py's workload (the E6D2 GRU
                                              CTCEncoder, head x 32, 64 streams x C chunks of 2 frames = 75 ms).
Per arm: audio-sec/sec and chunk latency p50 / p99 (the call to the committed ids on the host), over all rounds.  With
--lib (here a build of the commit before streaming context, the same EbPhase) the no-context arms also run through that
library in the same process: committed ids and flushed scores compared bit for bit, and timed as arms of their own.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
B, T_RNNT, T_CTC, V = 32, 250, 500, 1024
PHRASES = (0, 100, 1000, 5000)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--stream", action="store_true")
    ap.add_argument("--chunks", type=int, default=250)
    args = ap.parse_args()
    if args.stream:
        return stream_main(args)
    import torch
    import edgedict_b200.stream_engine as se
    from edgedict_b200.context import ContextGraph
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import BeamEngine, CTCBeamEngine
    assert torch.cuda.is_available(), "bench_context.py measures on the GPU"
    new_size = C.sizeof(se.EbPhase)
    old_size = new_size - C.sizeof(C.c_void_p)            # the parent's EbPhase: no ctx

    other = None
    if args.lib:
        other = C.CDLL(os.path.abspath(args.lib))
        for n in ("eb_decode_run", "eb_decode_run_ctc"):
            getattr(other, n).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
            getattr(other, n).restype = C.c_int
        assert other.eb_decode_phase_size() == old_size, "--lib must be a build with the parent's EbPhase"
    own_launch = se._launch

    def run(eng, h, lens, parent=False):
        if not parent:
            return eng.run(h, lens)
        old = eng.__dict__.get("_old_prog")
        if old is None:
            old = eng._old_prog = eng._prog.view(eng.nphase, new_size)[:, :old_size].contiguous()

        def launch(entry, prog, nphase, bar, max_ctas):
            rc = getattr(other, entry)(old.data_ptr(), nphase, bar.data_ptr(), max_ctas,
                                       torch.cuda.current_stream().cuda_stream)
            assert rc == 0, (entry, rc)
        se._launch = launch
        try:
            return eng.run(h, lens)
        finally:
            se._launch = own_launch

    rng = random.Random(5)
    graphs = {n: ContextGraph([[rng.randrange(1, V) for _ in range(rng.randint(2, 6))] for _ in range(n)], V, 1.5)
              for n in PHRASES}
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
            for n in PHRASES:
                eng = BeamEngine(model, B, T_RNNT, W, context=graphs[n] if n else None, **kw)
                arms["rnnt_W%d_lm%d_ctx%d" % (W, use_lm, n)] = (eng, h_enc, fr_rnnt, False)
                if n == 0 and other is not None:
                    arms["rnnt_W%d_lm%d_ctx0_parent" % (W, use_lm)] = (eng, h_enc, fr_rnnt, True)
    for W in (4, 8, 16):
        for n in PHRASES:
            eng = CTCBeamEngine(B, T_CTC, V, W, context=graphs[n] if n else None, device="cuda")
            arms["ctc_W%d_ctx%d" % (W, n)] = (eng, lp, fr_ctc, False)
            if n == 0 and other is not None:
                arms["ctc_W%d_ctx0_parent" % W] = (eng, lp, fr_ctc, True)

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
    res = dict(card=card(), rounds=args.rounds, states={n: graphs[n].n_states for n in PHRASES},
               ms={k: dict(min=round(min(v), 3), median=round(sorted(v)[len(v) // 2], 3), max=round(max(v), 3))
                   for k, v in times.items()},
               parent_same_bits=same_bits)
    for k, v in res["ms"].items():
        print("%-28s %8.2f %8.2f %8.2f ms" % (k, v["min"], v["median"], v["max"]), file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


def stream_main(args):
    import time

    import numpy as np
    import torch
    import edgedict_b200.stream_engine as se
    from edgedict_b200.context import ContextGraph
    from edgedict_b200.rnnt.models import CTCEncoder, Transducer
    from edgedict_b200.stream_engine import CTCStreamBeamEngine, StreamBeamEngine
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    from bench_ctc_stream import CFG, F, FRAME_SEC, N, S   # the streaming CTC workload
    assert torch.cuda.is_available(), "bench_context.py measures on the GPU"
    C_ = args.chunks
    other = None
    if args.lib:
        other = C.CDLL(os.path.abspath(args.lib))
        for n in ("eb_decode_run", "eb_decode_run_ctc_stream_beam"):
            getattr(other, n).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
            getattr(other, n).restype = C.c_int
        assert other.eb_decode_phase_size() == C.sizeof(se.EbPhase), "--lib must share this tree's EbPhase"
    own_launch = se._launch

    def parent_launch(entry, prog, nphase, bar, max_ctas):
        rc = getattr(other, entry)(prog.data_ptr(), nphase, bar.data_ptr(), max_ctas,
                                   torch.cuda.current_stream().cuda_stream)
        assert rc == 0, (entry, rc)

    rng = random.Random(5)
    graphs = {n: ContextGraph([[rng.randrange(1, V) for _ in range(rng.randint(2, 6))] for _ in range(n)], V, 1.5)
              for n in PHRASES if n}
    torch.manual_seed(10)
    model = Transducer(output_loss=False, **LARGE).eval()
    with torch.no_grad():
        for p in model.parameters():
            p.mul_(2.0)
    model.cuda()
    torch.manual_seed(11)
    lm = torch.nn.Module()
    lm.encoder, lm.rnn = torch.nn.Embedding(1024, 64), torch.nn.LSTM(64, 1024, 2, batch_first=True)
    lm.decoder = torch.nn.Linear(1024, 1024)
    lm = lm.cuda().eval()
    torch.manual_seed(0)
    cm = CTCEncoder(**CFG).cuda().eval()
    with torch.no_grad():
        cm.tovocab[0].weight.mul_(32.0)
    g = torch.Generator().manual_seed(0)
    x_rnnt = torch.randn(C_, 64, 2, 240, generator=g).pin_memory()
    x_ctc = torch.randn(C_, S, N, F, generator=g).pin_memory()

    arms = {}                                              # name -> (engine, chunks, seconds of audio, parent)
    for W, use_lm in ((4, False), (8, False), (4, True)):
        kw = dict(lm=lm, lm_weight=0.3, length_bonus=0.5) if use_lm else {}
        for n in PHRASES:
            eng = StreamBeamEngine(model, 64, 2, W, context=graphs.get(n), **kw)
            arms["srnnt_W%d_lm%d_ctx%d" % (W, use_lm, n)] = (eng, x_rnnt, 64 * C_ * 0.120, False)
            if n == 0 and other is not None:
                arms["srnnt_W%d_lm%d_ctx0_parent" % (W, use_lm)] = (eng, x_rnnt, 64 * C_ * 0.120, True)
    for W in (4, 8):
        for n in PHRASES:
            eng = CTCStreamBeamEngine(cm, S, N, W, context=graphs.get(n))
            arms["sctc_W%d_ctx%d" % (W, n)] = (eng, x_ctc, S * C_ * N * FRAME_SEC, False)
            if n == 0 and other is not None:
                arms["sctc_W%d_ctx0_parent" % W] = (eng, x_ctc, S * C_ * N * FRAME_SEC, True)

    def committed(ids, counts):
        return [ids[s, :int(counts[s])].tolist() for s in range(ids.shape[0])]

    def run(eng, xs, parent, lat=None):
        """The whole utterance: reset, every chunk, flush.  Untimed (lat None): -> (committed ids per chunk and
        stream, the flush's committed ids per stream and -log p bits); timed: the chunk latencies go to lat."""
        se._launch = parent_launch if parent else own_launch
        try:
            eng.reset()
            outs = []
            for i in range(xs.shape[0]):
                t0 = time.perf_counter()
                ids, counts = eng.step(xs[i].cuda(non_blocking=True))
                if lat is not None:
                    lat.append(time.perf_counter() - t0)
                else:
                    outs.append(committed(ids, counts))
            ids, counts, nlp = eng.flush()
            return None if lat is not None else (outs, (committed(ids, counts), nlp.view(torch.int32).tolist()))
        finally:
            se._launch = own_launch

    same_bits = {}
    for name, (eng, xs, _, parent) in arms.items():        # warm-up, and the parent's bits against this tree's
        if parent:
            a, fa = run(eng, xs[:40], True)
            b, fb = run(eng, xs[:40], False)
            same_bits[name] = a == b and fa == fb and sum(len(x) for c in a for x in c) > 0
        else:
            run(eng, xs[:10], False)
    torch.cuda.synchronize()
    stats = {k: dict(lat=[], wall=0.0, audio=0.0) for k in arms}
    names = list(arms)
    for r in range(args.rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            eng, xs, audio, parent = arms[name]
            st = stats[name]
            t_all = time.perf_counter()
            run(eng, xs, parent, st["lat"])
            torch.cuda.synchronize()
            st["wall"] += time.perf_counter() - t_all
            st["audio"] += audio
    out = {}
    for k, st in stats.items():
        lat = np.array(st["lat"]) * 1e3
        out[k] = dict(audio_sec_per_sec=round(st["audio"] / st["wall"], 1),
                      chunk_latency_ms=dict(p50=round(float(np.percentile(lat, 50)), 3),
                                            p99=round(float(np.percentile(lat, 99)), 3)))
        print("%-28s %9.1f audio-s/s  p50 %7.3f  p99 %7.3f ms" % (k, out[k]["audio_sec_per_sec"],
                                                                   out[k]["chunk_latency_ms"]["p50"],
                                                                   out[k]["chunk_latency_ms"]["p99"]), file=sys.stderr)
    res = dict(card=card(), rounds=args.rounds, chunks=C_, states={n: graphs[n].n_states for n in graphs},
               results=out, parent_same_bits=same_bits)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
