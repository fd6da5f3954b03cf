#!/usr/bin/env python
"""The encoder backward of the bf16 E6D2 training step (6 x 1024 LSTM layers, time reduction after layer 1, B = 32,
T = 1000) under the chunked schedule (functional.LSTMStack._backward_wave: BPTT in groups of time chunks, group inputs
prepared under the layer above) and under the serial schedule (one layer after another), alternated in one process.

  python scripts/measure_bptt_wavefront.py [--reps N] [--out DIR]

Prints one JSON line:
- `card`: GPU name and power limit, read in the same run;
- `k16_clusters`: eb_lstm_c4_max_clusters(1024, 16), the co-resident clusters of 16 of the BPTT kernel (two grids would
  need 16);
- `encoder_bwd_ms`: wall time of the stack's backward (CUDA events on the calling stream, which waits for every stream
  of the schedule), per schedule: every rep, min, median, max;
- `chunks`: one chunked backward with CUDA events around every BPTT launch: per layer and group the stream, the start
  and end (ms from the start of the backward), the BPTT interval, its time per step, and the gap on its stream since
  the previous BPTT launch there ended;
- `serial_layers`: the same for the serial schedule (one launch per layer).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, I0, H, L = 32, 1000, 240, 1024, 6


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        return "nvidia-smi unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    from edgedict_b200._lib import lib
    from edgedict_b200.rnnt.models import ResLayerNormLSTM
    assert torch.cuda.is_available(), "needs a GPU"
    torch.manual_seed(0)
    net = ResLayerNormLSTM(I0, H, L, time_reductions=[1]).cuda()
    for m in net.modules():
        m.precision = "bf16"
    x = torch.randn(B, T, I0, device="cuda")
    w = torch.randn(B, T // 2, H, device="cuda")
    main_st = torch.cuda.current_stream()

    stamps = []
    orig = ops.lstm_c4_bwd_chunks

    def traced(dy, *a, **kw):
        st = torch.cuda.current_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        r = orig(dy, *a, **kw)
        e1.record(st)
        stamps.append((st.cuda_stream, dy.numel() // (B * H), e0, e1))
        return r

    def backward_ms(wave, trace=False):
        Fn.BPTT_WAVEFRONT = wave
        net.zero_grad()
        y, _ = net(x)
        loss = (y * w).sum()
        torch.cuda.synchronize()
        stamps.clear()
        ops.lstm_c4_bwd_chunks = traced if trace else orig
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(main_st)
        loss.backward()
        b.record(main_st)
        torch.cuda.synchronize()
        ops.lstm_c4_bwd_chunks = orig
        Fn.BPTT_WAVEFRONT = True
        rows = []
        if trace:
            last = {}
            for i, (sid, steps, e0, e1) in enumerate(stamps):
                s, e = a.elapsed_time(e0), a.elapsed_time(e1)
                rows.append(dict(i=i, stream=sid % 1000, steps=steps, start_ms=round(s, 3), end_ms=round(e, 3),
                                 bptt_ms=round(e - s, 3), us_per_step=round((e - s) * 1e3 / steps, 2),
                                 gap_ms=round(s - last[sid], 3) if sid in last else None))
                last[sid] = e
        return a.elapsed_time(b), rows

    for wave in (True, False, True, False):      # warm-up: module loads, allocator, occupancy queries
        backward_ms(wave)
    res = {True: [], False: []}
    for _ in range(args.reps):
        for wave in (True, False):
            res[wave].append(backward_ms(wave)[0])
    _, chunks = backward_ms(True, trace=True)
    _, serial = backward_ms(False, trace=True)
    # layer / group of each chunked launch, in issue order (diagonals from the top layer and the last group)
    plan = Fn.wavefront_plan(T, [False, True] + [False] * (L - 2))
    C = len(plan[0])
    NG = -(-C // Fn.BPTT_GROUP)
    order = [(l, NG - 1 - (d - (L - 1 - l))) for d in range(L + NG - 1) for l in range(L - 1, -1, -1)
             if 0 <= NG - 1 - (d - (L - 1 - l)) < NG]
    if len(order) == len(chunks):
        for r, (l, q) in zip(chunks, order):
            r["layer"], r["group"] = l, q
    for r, l in zip(serial, range(L - 1, -1, -1)):
        r["layer"] = l

    def summ(v):
        s = sorted(v)
        return dict(reps=[round(t, 3) for t in v], min=round(s[0], 3), median=round(s[len(s) // 2], 3),
                    max=round(s[-1], 3))

    L_ = lib()
    out = dict(card=card(), shape="E6D2 encoder B=%d T=%d H=%d L=%d, reduction after layer 1, C=%d" % (B, T, H, L, C),
               k16_clusters=int(L_.eb_lstm_c4_max_clusters(H, 16)),
               encoder_bwd_ms=dict(chunked=summ(res[True]), serial=summ(res[False])),
               chunks=chunks, serial_layers=serial)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bptt_wavefront.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
