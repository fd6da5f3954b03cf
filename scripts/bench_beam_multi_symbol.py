"""Beam search with up to K = max_symbols symbols per encoder frame, variants alternated in one process:
  - batched (BeamEngine, the device part of Transducer.beam_search) over B = 32 x 30 s of E6D2_LARGE encoder output
    (T' = 250): W = 4 / 8, K = 1 / 2 / 4, with and without an LMModel(1024, 64, 1024, 2)-shaped LM (lm_weight 0.5,
    length_bonus 3), timed with CUDA events;
  - streaming (StreamBeamEngine), 64 streams x 250 chunks of [2, 240] log-mel = 120 ms each, W = 4, K = 1 / 2:
    audio-sec/sec.
Random weights (x 2, as bench_stream.py) with two emission profiles set by shifting joint[2].bias[blank]:
  realistic  + 3 (the shift of test_gpu_multi_symbol's E6D2_LARGE cases: about half the frames emit);
  worst      blank at -1e4: every open slot emits in every round, so every frame takes K rounds.
Reports tokens of the best hypotheses per utterance-frame, rounds taken per frame, and the card's name and power limit.
With --lib OTHER.so (a build of another commit with the same EbPhase layout) the K = 1 batched programs are also run
through that library's eb_decode_run, alternated with this tree's, and their outputs compared bitwise.
  python scripts/bench_beam_multi_symbol.py [--lib OTHER.so] [out.json]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import torch
sys.path.insert(0, os.getcwd())
from edgedict_b200.rnnt.models import Transducer
import edgedict_b200.stream_engine as se
from edgedict_b200.stream_engine import BeamEngine, StreamBeamEngine

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
B, T_OUT, UTT_SEC, REPS = 32, 250, 30.0, 3
S, CHUNKS, CHUNK_SEC = 64, 250, 0.120
PROFILES = dict(realistic=3.0, worst=-1e4)

ap = argparse.ArgumentParser()
ap.add_argument("--lib", default=None)
ap.add_argument("out", nargs="?", default=None)
args = ap.parse_args()
assert torch.cuda.is_available(), "needs a CUDA device"
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip().splitlines()
card = dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)
other = None
if args.lib:
    other = C.CDLL(os.path.abspath(args.lib))
    other.eb_decode_run.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    other.eb_decode_run.restype = C.c_int
own_lib = se.lib

torch.manual_seed(10)
model = Transducer(output_loss=False, **LARGE).eval()
with torch.no_grad():
    for p in model.parameters():
        p.mul_(2.0)
model.cuda()
bias = model.joint.joint[2].bias                      # the engines read it in place
bias0 = float(bias[0])
torch.manual_seed(11)
lm = torch.nn.Module()
lm.encoder, lm.rnn, lm.decoder = torch.nn.Embedding(1024, 64), torch.nn.LSTM(64, 1024, 2, batch_first=True), \
    torch.nn.Linear(1024, 1024)
with torch.no_grad():
    for p in lm.parameters():
        p.mul_(3.0)
lm = lm.eval().cuda()
g = torch.Generator().manual_seed(0)
h_enc = torch.randn(B, T_OUT, 640, generator=g).cuda()
frames = torch.full((B,), T_OUT, dtype=torch.int32, device="cuda")
pinned = torch.randn(CHUNKS, S, 2, 240, generator=g).pin_memory()

batched = {}
for W in (4, 8):
    for K in (1, 2, 4):
        for use_lm in (False, True):
            kw = dict(lm=lm, lm_weight=0.5, length_bonus=3.0) if use_lm else {}
            batched[(W, K, use_lm)] = BeamEngine(model, B, T_OUT, W, max_symbols=K, **kw)
streams = {K: StreamBeamEngine(model, S, 2, 4, max_symbols=K, max_pending=64) for K in (1, 2)}


def run_batched(eng, lib=None):
    """BeamEngine.run, launched through this tree's library or through ``lib``."""
    if lib is None:
        return eng.run(h_enc, frames)
    se.lib = lambda: lib
    try:
        return eng.run(h_enc, frames)
    finally:
        se.lib = own_lib


def rounds_taken(eng):
    """Rounds the utterances took per frame, from the history's live counts (0: a round not taken)."""
    K = eng.max_symbols
    if K == 1:
        return 1.0
    live = eng.hist_live.view(eng.B, eng.T, K).clone()
    live[:, -1, -1] = 1                               # the last column holds the final live count
    return float((live > 0).sum()) / (eng.B * eng.T)


res = dict(card=card, batched={}, stream={}, other_lib=args.lib)
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for prof, shift in PROFILES.items():
    with torch.no_grad():
        bias[0] = bias0 + shift
    for key, eng in batched.items():                  # warm-up
        run_batched(eng)
    torch.cuda.synchronize()
    times = {}
    for rep in range(REPS):
        for key, eng in batched.items():
            libs = [("this", None)] + ([("other", other)] if other is not None and key[1] == 1 else [])
            for name, lib in (libs if rep % 2 == 0 else libs[::-1]):
                ev[0].record()
                ids, nlp = run_batched(eng, lib)
                ev[1].record()
                torch.cuda.synchronize()
                times.setdefault((key, name), []).append(ev[0].elapsed_time(ev[1]))
                if name == "other":
                    mine = [t.clone() for t in run_batched(eng)]
                    assert torch.equal(ids, mine[0]) and torch.equal(nlp.view(torch.int32), mine[1].view(torch.int32))
    for (key, name), ts in times.items():
        W, K, use_lm = key
        eng = batched[key]
        run_batched(eng)
        ntok = int((eng.ids >= 0).sum())
        r = dict(W=W, K=K, lm=use_lm, lib=name, ms=sorted(ts), tokens_per_frame=ntok / (B * T_OUT),
                 rounds_per_frame=rounds_taken(eng), audio_sec_per_sec=B * UTT_SEC / (min(ts) / 1e3))
        res["batched"].setdefault(prof, []).append(r)
        print("%s batched W=%d K=%d lm=%d %s: %.1f-%.1f ms, %.3f tokens/frame, %.2f rounds/frame"
              % (prof, W, K, use_lm, name, min(ts), max(ts), r["tokens_per_frame"], r["rounds_per_frame"]), flush=True)
    # streaming: K alternated chunk by chunk
    for K, eng in streams.items():
        eng.reset()
        eng.step(pinned[0])
    tot = {K: 0.0 for K in streams}
    ntok = {K: 0 for K in streams}
    for K, eng in streams.items():
        eng.reset()
    for c in range(CHUNKS):
        for K, eng in (streams.items() if c % 2 == 0 else list(streams.items())[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ids, counts = eng.step(pinned[c])
            tot[K] += time.perf_counter() - t0
            ntok[K] += int(counts.sum())
    for K in streams:
        r = dict(K=K, W=4, seconds=tot[K], audio_sec_per_sec=S * CHUNKS * CHUNK_SEC / tot[K],
                 committed_tokens=ntok[K], collapses=streams[K].n_collapses)
        res["stream"].setdefault(prof, []).append(r)
        print("%s stream W=4 K=%d: %.0f audio-sec/sec, %d tokens committed, %d collapses"
              % (prof, K, r["audio_sec_per_sec"], ntok[K], r["collapses"]), flush=True)
with torch.no_grad():
    bias[0] = bias0
print(json.dumps(card))
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
