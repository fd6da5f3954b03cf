"""BASELINE.json configs[3]: E6D2_LARGE streaming greedy decode, 64 concurrent synthetic 30-s streams
(250 chunks of [64, 2, 240] log-mel = 120 ms of audio each) through the persistent decode kernel:
RTF, per-chunk latency p50/p99, and the CPU reference loop (one stream, as the reference runs it)."""
import json, os, sys, time
import numpy as np
import torch
sys.path.insert(0, os.getcwd())
from edgedict_b200.rnnt.models import Transducer
from edgedict_b200.stream_engine import StreamEngine
from oracle import model_torch as mt

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
S, CHUNKS, CHUNK_SEC = 64, 250, 0.120
torch.manual_seed(10)
model = Transducer(output_loss=False, **LARGE).eval()
with torch.no_grad():
    for p in model.parameters():
        p.mul_(2.0)                       # random-init weights emit only blanks; scale up so symbols appear
sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
model.cuda()
g = torch.Generator().manual_seed(0)
chunks = torch.randn(CHUNKS, S, 2, 240, generator=g)
pinned = chunks.pin_memory()
eng = StreamEngine(model, S, 2)
for i in range(3):
    eng.step(pinned[i].cuda(non_blocking=True))
torch.cuda.synchronize()
eng.reset()
lat, toks = [], []
host = torch.zeros(S, 1, dtype=torch.int32).pin_memory()
t_all = time.perf_counter()
for i in range(CHUNKS):
    t0 = time.perf_counter()
    out = eng.step(pinned[i].cuda(non_blocking=True))        # H2D of the chunk + one kernel
    host.copy_(out, non_blocking=True)
    torch.cuda.current_stream().synchronize()                 # tokens are on the host: end of the chunk
    lat.append(time.perf_counter() - t0)
    toks.append(host.clone())
wall = time.perf_counter() - t_all
toks = torch.stack(toks)                                      # [chunks, S, 1]
lat = np.array(lat) * 1e3
# CPU reference loop on stream 0 (bounded: first 40 chunks), token-for-token check + timing
st = mt.StreamState(sd)
ref, t0 = [], time.perf_counter()
NREF = 40
for i in range(NREF):
    o = mt.stream_decode(sd, st, chunks[i, 0:1], fast=True)
    ref.append(o[0] if o else 0)
cpu_s = time.perf_counter() - t0
match = [int(toks[i, 0, 0]) for i in range(NREF)] == ref
res = dict(config="E6D2_LARGE streaming greedy, %d streams x %d chunks x 120 ms" % (S, CHUNKS),
           audio_sec=S * CHUNKS * CHUNK_SEC, wall_s=round(wall, 4), rtf=round(wall / (S * CHUNKS * CHUNK_SEC), 6),
           audio_sec_per_sec=round(S * CHUNKS * CHUNK_SEC / wall, 1), chunk_latency_ms=dict(p50=round(float(np.percentile(lat, 50)), 3),
           p99=round(float(np.percentile(lat, 99)), 3), max=round(float(lat.max()), 3)), phases_per_chunk=eng.n_chunk_phases,
           nonblank_tokens=int((toks != 0).sum()), token_for_token_vs_cpu_loop_stream0=bool(match),
           cpu_reference=dict(streams=1, chunks=NREF, sec_per_chunk=round(cpu_s / NREF, 5),
                              audio_sec_per_sec=round(NREF * CHUNK_SEC / cpu_s, 2), threads=torch.get_num_threads()))
print(json.dumps(res))
if len(sys.argv) > 1:
    json.dump(res, open(sys.argv[1], "w"), indent=1)
