#!/usr/bin/env python
"""The joint's three 2.7 TFLOP products of the bf16 E6D2 training step, timed alone at the step's shapes
(B=32, T'=500, U+1=129: M = 2,064,000 lattice rows, J = 640, V = 1024):
- `logits_lse`: eb_joint_logits_lse, hidden [M,J] x W2^T -> bf16 logits [M,V] + the loss's softmax statistics;
- `dhidden`:    eb_gemm_bf16_dtanh, d logits [M,V] x W2 [V,J] -> bf16 (.) * (1 - hidden^2) [M,J];
- `dw2`:        hidden^T d logits -> fp32 [J,V] (split-K, what ops.mm_tn runs for dW2^T), the anchor: its epilogue is
                the fp32 split-K one.

  python scripts/bench_joint_gemm.py [--lib OTHER.so] [--rounds R] [--iters N] [--warmup W]

With --lib, a second build of the library (e.g. of another commit) is loaded beside this tree's and the two are timed in
alternation, round by round, on the same inputs; the outputs of the two are also compared bitwise.  Each kernel time is
the median over N launches, each between its own pair of CUDA events, after W warm-up launches.  Prints the card's
name and power limit read in the same run, a table, and one JSON line.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, U1, V, J = 32, 500, 129, 1024, 640
M = B * T * U1
FLOP = 2.0 * M * V * J


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def load(path):
    from edgedict_b200._lib import SIGNATURES
    h = ctypes.CDLL(os.path.abspath(path))
    for name in ("eb_joint_logits_lse", "eb_gemm_bf16_dtanh", "eb_gemm_bf16_ex", "eb_gemm_bf16_partials"):
        res, args = SIGNATURES[name]
        fn = getattr(h, name)
        fn.restype = res
        fn.argtypes = args
    return h


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=None, help="a second libedgedict_b200.so to time in alternation with this tree's")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from edgedict_b200._lib import LIB_PATH
    assert torch.cuda.is_available(), "bench_joint_gemm.py times CUDA kernels: it needs a GPU"
    dev = torch.device("cuda", 0)
    bf16, f32 = torch.bfloat16, torch.float32
    libs = [("this", load(LIB_PATH))]
    if args.lib:
        libs.insert(0, ("other", load(args.lib)))

    g = torch.Generator(device=dev).manual_seed(7)
    hid = (torch.rand(M, J, device=dev, generator=g) * 2 - 1).to(bf16)          # tanh outputs
    w2 = (torch.randn(V, J, device=dev, generator=g) * 0.04).to(bf16)
    b2 = torch.randn(V, device=dev, generator=g) * 0.1
    dl = (torch.randn(M, V, device=dev, generator=g) * 1e-3).to(bf16)
    labels = torch.randint(1, V, (B, U1 - 1), device=dev, dtype=torch.int32, generator=g)
    xlen = torch.full((B,), T, device=dev, dtype=torch.int32)
    ylen = torch.full((B,), U1 - 1, device=dev, dtype=torch.int32)
    out = {name: dict(logits=torch.empty(M, V, dtype=bf16, device=dev), stats=torch.empty(3, M, dtype=f32, device=dev),
                      dpre=torch.empty(M, J, dtype=bf16, device=dev), dw2=torch.empty(J, V, dtype=f32, device=dev))
           for name, _ in libs}
    nws = max(int(h.eb_gemm_bf16_partials(1, 0, 0, J, V, M, 0)) for _, h in libs)
    ws = torch.empty(max(nws, 1), dtype=f32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    p = lambda t: ctypes.c_void_p(t.data_ptr())

    def kernels(h, o):
        s = o["stats"]
        return {
            "logits_lse": lambda: h.eb_joint_logits_lse(p(hid), p(w2), p(b2), p(o["logits"]), p(labels), p(xlen),
                                                        p(ylen), p(s[0]), p(s[1]), p(s[2]), B, T, U1, V, J, 0, st),
            "dhidden": lambda: h.eb_gemm_bf16_dtanh(p(dl), 0, p(w2), 1, p(o["dpre"]), p(hid), M, J, V, st),
            "dw2": lambda: h.eb_gemm_bf16_ex(p(hid), 1, p(dl), 1, p(o["dw2"]), 0, None, 0, J, V, M, 0, p(ws), nws, st),
        }

    def time_one(fn):
        for _ in range(args.warmup):
            assert fn() == 0
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
        for a, b in ev:
            a.record()
            assert fn() == 0
            b.record()
        torch.cuda.synchronize()
        return statistics.median(a.elapsed_time(b) for a, b in ev)

    the_card = card()
    print("card:", the_card)
    res = {name: {k: [] for k in ("logits_lse", "dhidden", "dw2")} for name, _ in libs}
    fns = {name: kernels(h, out[name]) for name, h in libs}
    for r in range(args.rounds):
        for k in ("logits_lse", "dhidden", "dw2"):       # the libraries back to back per kernel: the same card state
            for name, _ in libs:
                ms = time_one(fns[name][k])
                res[name][k].append(ms)
                print("round %d  %-10s  %-5s  %8.3f ms  %6.1f TFLOP/s" % (r, k, name, ms, FLOP / ms * 1e-9))
    same = None
    if len(libs) == 2:
        a, b = out["other"], out["this"]
        same = {k: bool(torch.equal(a[k], b[k])) for k in a}
        print("bitwise identical outputs:", same)
    summary = {name: {k: dict(ms=v, tflops=[round(FLOP / x * 1e-9, 1) for x in v]) for k, v in d.items()}
               for name, d in res.items()}
    print(json.dumps(dict(card=the_card, shapes=dict(M=M, J=J, V=V), flop_per_product=FLOP, iters=args.iters,
                          results=summary, bitwise_identical=same)))


if __name__ == "__main__":
    main()
