"""Greedy decoding with up to K = max_symbols symbols per encoder frame, K = 1 / 2 / 4 alternated in one process:
  - E6D2_LARGE streaming (StreamEngine), 64 streams x 250 chunks of [2, 240] log-mel = 120 ms each: audio-sec/sec and
    chunk latency p50 / p99 (H2D of the chunk, the kernel, D2H of the tokens);
  - batched greedy decode (GreedyEngine, the device part of Transducer.greedy_decode) over B = 32 x 30 s of encoder
    output (T' = 250), timed with CUDA events.
Random weights (x 2, as bench_stream.py) need a controlled emission profile, set by shifting joint[2].bias[blank]:
  realistic  a shift found by bisection so that about a third of the streaming frames emit in round 0;
  worst      blank at -inf: every round emits, so K rounds cost about K frames.
Reports non-blank tokens per round and the SKIPs taken (a round j >= 1 that no row reached), with the card's name and
power limit.  python scripts/bench_multi_symbol.py [out.json]"""
import json, os, subprocess, sys, time
import numpy as np
import torch
sys.path.insert(0, os.getcwd())
from edgedict_b200.rnnt.models import Transducer
from edgedict_b200.stream_engine import GreedyEngine, StreamEngine

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
S, CHUNKS, CHUNK_SEC, KS, REPS = 64, 250, 0.120, (1, 2, 4), 2
B, UTT_SEC, T_OUT = 32, 30.0, 250

assert torch.cuda.is_available(), "needs a CUDA device"
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip().splitlines()
card = dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)
torch.manual_seed(10)
model = Transducer(output_loss=False, **LARGE).eval()
with torch.no_grad():
    for p in model.parameters():
        p.mul_(2.0)
model.cuda()
bias = model.joint.joint[2].bias                      # the engines read it in place
bias0 = float(bias[0])
g = torch.Generator().manual_seed(0)
pinned = torch.randn(CHUNKS, S, 2, 240, generator=g).pin_memory()
stream = {K: StreamEngine(model, S, 2, max_symbols=K) for K in KS}
host = {K: torch.zeros(S, K, dtype=torch.int32).pin_memory() for K in KS}


def run_stream(K, n=CHUNKS):
    eng, h = stream[K], host[K]
    eng.reset()
    torch.cuda.synchronize()
    lat, toks = [], []
    t_all = time.perf_counter()
    for i in range(n):
        t0 = time.perf_counter()
        out = eng.step(pinned[i].cuda(non_blocking=True))
        h.copy_(out, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        lat.append(time.perf_counter() - t0)
        toks.append(h.clone())
    return time.perf_counter() - t_all, np.array(lat) * 1e3, torch.stack(toks).numpy()     # [n, S, K]


def rounds(toks, K):
    """non-blank tokens per round and SKIPs taken (round j >= 1 reached by no row) over frames [..., rows, K]"""
    t = toks.reshape(-1, toks.shape[-2], K)
    nb = (t != 0)
    return nb.sum((0, 1)).tolist(), int((~nb[:, :, :K - 1].any(1)).sum())


def set_blank(v):
    with torch.no_grad():
        bias[0] = v


def calibrate():
    """blank bias for ~1/3 non-blank frames in round 0 of the streaming run (first 40 chunks, K = 2)"""
    lo, hi = bias0 - 4.0, bias0 + 12.0                 # shift up = more blank
    for _ in range(14):
        mid = 0.5 * (lo + hi)
        set_blank(mid)
        frac = float((run_stream(2, 40)[2][..., 0] != 0).mean())
        lo, hi = (mid, hi) if frac > 1 / 3 else (lo, mid)
    return 0.5 * (lo + hi)


E = model.encoder.proj.weight.shape[0]
h_enc = (torch.randn(B, T_OUT, E, generator=g) * 2).cuda()
greedy = {K: GreedyEngine(model, B, T_OUT, max_symbols=K) for K in KS}


def run_greedy(K, reps=5):
    eng = greedy[K]
    eng.run(h_enc)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.run(h_enc)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return ms, eng.hist.cpu().numpy().reshape(B, T_OUT, K).transpose(1, 0, 2)


for K in KS:                                           # warm up every program
    run_stream(K, 3)
    greedy[K].run(h_enc)
torch.cuda.synchronize()
res = dict(card=card, config="E6D2_LARGE; streaming %d streams x %d chunks x 120 ms; greedy B=%d x %g s (T'=%d)"
           % (S, CHUNKS, B, UTT_SEC, T_OUT), profiles={})
for name in ("realistic", "worst"):
    set_blank(calibrate() if name == "realistic" else float("-inf"))
    prof = dict(blank_bias=float(bias[0]), stream={K: [] for K in KS}, greedy={K: [] for K in KS})
    for rep in range(REPS):
        for K in KS:
            wall, lat, toks = run_stream(K)
            per_round, skips = rounds(toks, K)
            prof["stream"][K].append(dict(
                audio_sec_per_sec=round(S * CHUNKS * CHUNK_SEC / wall, 1),
                chunk_latency_ms=dict(p50=round(float(np.percentile(lat, 50)), 3),
                                      p99=round(float(np.percentile(lat, 99)), 3)),
                nonblank_per_round=per_round, frames=CHUNKS * S, skips_taken=skips,
                skips_possible=CHUNKS * (K - 1), phases_per_chunk=stream[K].n_chunk_phases))
            ms, toks = run_greedy(K)
            per_round, skips = rounds(toks, K)
            prof["greedy"][K].append(dict(
                ms_min=round(min(ms), 3), ms_median=round(float(np.median(ms)), 3),
                audio_sec_per_sec=round(B * UTT_SEC / (min(ms) / 1e3), 1), nonblank_per_round=per_round,
                frames=B * T_OUT, skips_taken=skips, skips_possible=T_OUT * (K - 1), phases=greedy[K].nphase))
    for part in ("stream", "greedy"):
        key = "audio_sec_per_sec"
        best = {K: max(r[key] for r in prof[part][K]) for K in KS}
        prof[part + "_k4_over_k1_time"] = round(best[1] / best[4], 3)
    res["profiles"][name] = prof
set_blank(bias0)
print(json.dumps(res))
if len(sys.argv) > 1:
    json.dump(res, open(sys.argv[1], "w"), indent=1)
