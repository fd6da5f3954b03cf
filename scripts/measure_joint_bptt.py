#!/usr/bin/env python
"""Where the bf16 E6D2 training step (B=32, T=1000, U=128, V=1024) spends the time between the start of the joint's
backward and the first encoder BPTT kernel, and how much the BPTT recurrence slows down with joint-backward work
running beside it.  These are the figures that decide whether running the joint's backward under the top encoder
layer's BPTT (time-chunked) can pay off.

  python scripts/measure_joint_bptt.py [--out DIR] [--reps N]

Prints one JSON line:
- `card`: GPU name and power limit, read in the same run;
- `profile`: one training step under torch.profiler (after warm-up steps): the interval from the first loss-gradient
  kernel to the first `lstm_c4_bwd_kernel`, the kernels inside it per stream, and every BPTT launch with its time per
  step.  The Chrome trace is written to DIR/joint_bptt_step.pt.trace.json;
- `bptt`: the top layer's BPTT (eb_lstm_c4_bwd_chunks over the wavefront's chunk lengths) timed with CUDA events,
  alone and with a co-resident-configuration GEMM of the joint's d-hidden shape (one time chunk of rows) and the bf16
  loss-gradient kernel over one time chunk looping on a second stream;
- `chunk_work`: those two side kernels alone, per chunk;
- `max_clusters_c4_bwd16`: eb_lstm_c4_max_clusters(1024, 16), the co-resident clusters of 16 of the BPTT kernel.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0,
            dec_proj_size=256, joint_size=640)
B, T, U, V, J, H = 32, 1000, 128, 1024, 640, 1024


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def profile_step(out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from edgedict_b200.optim import FlatAdam
    from edgedict_b200.rnnt.models import Transducer
    dev = torch.device("cuda", 0)
    torch.manual_seed(10)
    model = Transducer(**E6D2).to(dev)
    model.set_precision("bf16")
    opt = FlatAdam(model, lr=5e-4)
    g = torch.Generator(device=dev).manual_seed(10)
    xs = torch.randn(B, T, 240, device=dev, generator=g)
    ys = torch.randint(4, V, (B, U), device=dev, dtype=torch.int32, generator=g)
    xlen = torch.full((B,), T, dtype=torch.int32)
    ylen = torch.full((B,), U, dtype=torch.int32)

    def step():
        opt.zero_grad()
        loss = model(xs, ys, xlen, ylen)
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    path = os.path.join(out_dir, "joint_bptt_step.pt.trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    t_first, t_last = ev[0]["ts"], max(e["ts"] + e["dur"] for e in ev)
    g0 = next(e for e in ev if "rnnt_grad" in e["name"])
    b0 = next(e for e in ev if "lstm_c4_bwd_kernel" in e["name"] and e["ts"] > g0["ts"])
    t0, t1 = g0["ts"], b0["ts"]
    inside = {}
    for e in ev:
        if e["ts"] + e["dur"] <= t0 or e["ts"] >= t1:
            continue
        name = e["name"].replace("(anonymous namespace)::", "").split("(")[0][:90]
        key = "%s | stream %s" % (name, e["args"].get("stream"))
        d = inside.setdefault(key, dict(calls=0, us=0.0, first_start_us=round(e["ts"] - t0, 1)))
        d["calls"] += 1
        d["us"] = round(d["us"] + e["dur"], 1)
    bptt = [e for e in ev if "lstm_c4_bwd_kernel" in e["name"]]
    steps = [T // 2] * 4 + [T] * 2                                  # layers 5 .. 0 (time reduction after layer 1)
    return dict(step_kernel_span_ms=round((t_last - t_first) / 1e3, 3),
                grad_start_to_first_bptt_ms=round((t1 - t0) / 1e3, 3),
                grad_stream=g0["args"].get("stream"), bptt_stream=b0["args"].get("stream"),
                kernels_in_interval=dict(sorted(inside.items(), key=lambda kv: kv[1]["first_start_us"])),
                bptt_launches=[dict(ms=round(e["dur"] / 1e3, 3), us_per_step=round(e["dur"] / n, 3) if n else None,
                                    stream=e["args"].get("stream"))
                               for e, n in zip(bptt, steps + [0] * max(0, len(bptt) - len(steps)))])


def bptt_contention(reps):
    import torch
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    from edgedict_b200._lib import lib
    dev = torch.device("cuda", 0)
    f32, bf16 = torch.float32, torch.bfloat16
    plan = Fn.wavefront_plan(T, [False, True, False, False, False, False])
    lens = plan[-1]
    Tp = sum(lens)
    g = torch.Generator(device=dev).manual_seed(5)
    rows = B * Tp
    dz = torch.randn(rows, H, device=dev, generator=g) * 1e-2
    gates = torch.rand(rows, 4 * H, device=dev, generator=g)
    cseq = torch.randn(rows, H, device=dev, generator=g)
    whhT16 = ops.transpose_to_bf16(torch.randn(4 * H, H, device=dev, generator=g) * 0.03)
    dg16 = torch.empty(rows, 4 * H, dtype=bf16, device=dev)

    Tc = max(lens)
    M = B * Tc * (U + 1)
    dl16 = (torch.randn(M, V, device=dev, generator=g) * 1e-3).to(bf16)
    w2T16 = (torch.randn(J, V, device=dev, generator=g) * 0.03).to(bf16)          # W2^T, K-major for the co-resident tile
    dpre = torch.empty(M, J, dtype=bf16, device=dev)
    logits = (torch.randn(B, Tc, U + 1, V, device=dev, generator=g)).to(bf16)
    ws = ops.rnnt_workspace(B, Tc, U + 1, f32, dev)
    ws.view(f32).fill_(-7.0)                                                      # finite statistics: timing only
    labels = torch.randint(1, V, (B, U), device=dev, dtype=torch.int32, generator=g)
    xl = torch.full((B,), Tc, dtype=torch.int32, device=dev)
    yl = torch.full((B,), U, dtype=torch.int32, device=dev)
    gsc = torch.ones(B, device=dev)

    def bptt():
        ops.lstm_c4_bwd_chunks(dz, gates, cseq, whhT16, lens, B, dg16)

    def side_gemm():
        ops.gemm_bf16(dl16, 0, w2T16, 0, M, J, V, out=dpre, flags=ops.GEMM_CORESIDENT)

    def side_grad():
        ops.rnnt_loss_bwd_bf16(logits, labels, xl, yl, 0, ws, gsc, 1.0 / B)

    def timed(fn, n, stream=None):
        s = stream or torch.cuda.current_stream()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(s):
            a.record()
            for _ in range(n):
                fn()
            b.record()
        return a, b

    for fn in (bptt, side_gemm, side_grad):
        fn()
    torch.cuda.synchronize()
    res = {}
    a, b = timed(bptt, reps)
    torch.cuda.synchronize()
    alone = a.elapsed_time(b) / reps
    res["alone_ms"] = round(alone, 3)
    res["alone_us_per_step"] = round(alone * 1e3 / Tp, 3)
    chunk = {}
    for name, fn in (("coresident_dhidden_gemm", side_gemm), ("grad_bf16", side_grad)):
        a, b = timed(fn, 10)
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / 10
        chunk[name] = dict(ms=round(ms, 3), rows=M)
    chunk["rows_per_chunk"] = M
    chunk["bptt_chunk_ms_alone"] = round(alone * Tc / Tp, 3)
    side = torch.cuda.Stream(dev)
    for label, fns in (("with_gemm", (side_gemm,)), ("with_grad", (side_grad,)), ("with_gemm_and_grad", (side_gemm, side_grad))):
        per = sum(chunk[n]["ms"] for n, f in (("coresident_dhidden_gemm", side_gemm), ("grad_bf16", side_grad)) if f in fns)
        n_side = int(alone * reps / per) + 2                     # keep the side stream busy for the whole BPTT window
        torch.cuda.synchronize()
        sa, sb = timed(lambda: [f() for f in fns], n_side, side)
        a, b = timed(bptt, reps)
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / reps
        side_ms = sa.elapsed_time(sb)
        res[label] = dict(ms=round(ms, 3), us_per_step=round(ms * 1e3 / Tp, 3), slowdown=round(ms / alone, 3),
                          side_ms_total=round(side_ms, 2), side_iters=n_side,
                          side_ms_per_iter=round(side_ms / n_side, 3))
    res["lens"] = lens
    return res, chunk, int(lib().eb_lstm_c4_max_clusters(H, 16))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the trace (default: a new temporary directory)")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs an H100"
    if args.out is None:
        import tempfile
        args.out = tempfile.mkdtemp(prefix="joint_bptt_")
    os.makedirs(args.out, exist_ok=True)
    out = dict(card=card())
    out["profile"] = profile_step(args.out)
    torch.cuda.empty_cache()
    out["bptt"], out["chunk_work"], out["max_clusters_c4_bwd16"] = bptt_contention(args.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
