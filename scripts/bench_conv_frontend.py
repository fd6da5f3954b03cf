"""Measures the raw-waveform front end (FrontEnd with cli/train.py's parameters) on the engine against a torch/cuDNN
restatement of the reference's module, and its share of a full bf16 step with an E6D2-shaped transducer behind it.

    python scripts/bench_conv_frontend.py [--rounds 10] [--B 32] [--seconds 14]

Workload: B = 32 utterances of up to 14 s at 16 kHz (audio_max_length=14), lengths spread over the top 10 %, zero-padded
as seq_collate pads them.  Arms, alternated within each round: engine fp32, engine bf16, the torch restatement
(tests/frontend_oracle.py) in fp32 with cuDNN's default TF32 convolutions, and the same under
torch.use_deterministic_algorithms(True).  Prints one JSON line with median times, the engine's per-kernel split
(ops._timed), peak memory, and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from edgedict_b200 import ops                                  # noqa: E402
from edgedict_b200.rnnt.models import FrontEnd, Transducer, frontend_lengths   # noqa: E402
from tests import frontend_oracle as fo                        # noqa: E402

TRAIN = [(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3
E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=128, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, enc_time_reductions=[], dec_hidden_size=256, dec_layers=2,
            dec_dropout=0.0, dec_proj_size=256, joint_size=640)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        return "nvidia-smi unavailable: %s" % e


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def median(v):
    v = sorted(v)
    return round(v[len(v) // 2], 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=14.0)
    ap.add_argument("--U", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_frontend.py measures on a CUDA device; none is present")
    dev = torch.device("cuda")
    L = int(a.seconds * 16000)
    g = torch.Generator().manual_seed(0)
    lens = (L * (0.9 + 0.1 * torch.rand(a.B, generator=g))).long()
    lens[0] = L
    x = torch.zeros(a.B, L)
    for b, n in enumerate(lens.tolist()):
        x[b, :n] = 0.3 * torch.randn(n, generator=g)
    x = x.to(dev)

    torch.manual_seed(1)
    fe32 = FrontEnd(TRAIN, bias=True).to(dev).set_precision("fp32")
    fe16 = FrontEnd(TRAIN, bias=True).to(dev).set_precision("bf16")
    fe16.load_state_dict(fe32.state_dict())
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in fe32.state_dict().items()}
    R = None

    def engine(m):
        return lambda: m(x)

    def torch_ref():
        return fo.forward(sd, x, TRAIN)

    def fwd_bwd(f, params):
        def run():
            for p in params:
                p.grad = None
            out = f()
            (out * R).sum().backward()
        return run

    with torch.no_grad():
        R = torch.randn(fe32(x).shape, device=dev)
    arms = {
        "engine_fp32": (engine(fe32), list(fe32.parameters()), False),
        "engine_bf16": (engine(fe16), list(fe16.parameters()), False),
        "torch_cudnn_tf32": (torch_ref, list(sd.values()), False),
        "torch_cudnn_deterministic": (torch_ref, list(sd.values()), True),
    }
    res = {k: dict(fwd_ms=[], fwd_bwd_ms=[]) for k in arms}
    prev = torch.are_deterministic_algorithms_enabled()
    for r in range(a.rounds + 2):                # two warm-up rounds
        for name, (f, params, det) in arms.items():
            torch.use_deterministic_algorithms(det)
            with torch.no_grad():
                tf = timed(f)
            tb = timed(fwd_bwd(f, params))
            if r >= 2:
                res[name]["fwd_ms"].append(tf)
                res[name]["fwd_bwd_ms"].append(tb)
    torch.use_deterministic_algorithms(prev)
    out = {}
    for name, (f, params, det) in arms.items():
        torch.use_deterministic_algorithms(det)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fwd_bwd(f, params)()
        torch.cuda.synchronize()
        out[name] = dict(fwd_ms=median(res[name]["fwd_ms"]), fwd_bwd_ms=median(res[name]["fwd_bwd_ms"]),
                         peak_mem_mb=round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1))
    torch.use_deterministic_algorithms(prev)

    kernels = {}
    for name, m in (("engine_fp32", fe32), ("engine_bf16", fe16)):
        ops.PROF.enabled = True
        ops.PROF.reset()
        fwd_bwd(engine(m), list(m.parameters()))()
        torch.cuda.synchronize()
        ops.PROF.enabled = False
        kernels[name] = {k: round(v["ms_sum"], 3) for k, v in sorted(ops.PROF.summary().items(),
                                                                     key=lambda kv: -kv[1]["ms_sum"])}

    # a full bf16 step: front end + E6D2-shaped transducer (input_size 128, no time reduction) + loss + backward
    torch.manual_seed(2)
    model = Transducer(**E6D2).to(dev).set_precision("bf16")
    ys = torch.randint(4, 1024, (a.B, a.U), generator=g, dtype=torch.int32).to(dev)
    ylen = torch.full((a.B,), a.U, dtype=torch.int32)

    def step():
        for p in list(model.parameters()) + list(fe16.parameters()):
            p.grad = None
        feats = fe16(x)
        xlen = frontend_lengths(lens, feats.shape[1])
        loss = model(feats[:, :int(xlen.max())].contiguous(), ys, xlen, ylen)
        loss.backward()

    def fe_only():
        fwd_bwd(engine(fe16), list(fe16.parameters()))()

    st, fs = [], []
    for r in range(a.rounds + 2):
        t1, t2 = timed(step), timed(fe_only)
        if r >= 2:
            st.append(t1)
            fs.append(t2)
    full = dict(step_ms=median(st), frontend_fwd_bwd_ms=median(fs))
    full["frontend_share"] = round(full["frontend_fwd_bwd_ms"] / full["step_ms"], 3)
    T = int(fe16(x).shape[1])
    print(json.dumps(dict(metric="FrontEnd fwd / fwd+bwd ms, cli/train.py parameters", card=card(),
                          workload="B=%d up to %.0f s (lengths 90-100 %%), T_out=%d, full step E6D2-shaped bf16 U=%d"
                          % (a.B, a.seconds, T, a.U), arms=out, kernels_ms=kernels, full_step=full,
                          rounds=a.rounds)))


if __name__ == "__main__":
    main()
