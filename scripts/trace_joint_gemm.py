#!/usr/bin/env python
"""Where a tile of the joint's logits+LSE and d-hidden GEMMs spends its cycles, at the bf16 E6D2 training step's shapes
(the shapes and inputs of scripts/bench_joint_gemm.py).  One warm launch of each product with eb_gemm_tc_set_trace on
records clock64 stamps of CTA 0 for its first --tiles work items; per tile this prints

  total    tile start to epilogue end (consumer warpgroup 0)
  wait     cycles its `full` waits took: the MMAs waiting for operands to land
  mma      the rest of the k-loop up to the last wgmma_wait<0>: issuing and retiring the MMAs
  epi      the epilogue (bias, softmax statistics / tanh', bf16 conversion, the staged TMA store issue), of which
  epi_wait waiting for the staging tile (its previous TMA stores to have read it; d-hidden: the tanh' operand to land)
  p_empty  cycles the producer warp waited for a free ring stage while it loaded that work item

and the medians over the tiles after the first (which starts cold).

  python scripts/trace_joint_gemm.py [--lib OTHER.so] [--tiles N]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_joint_gemm import B, T, U1, V, J, M, card  # noqa: E402

SLOTS = 8


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=None, help="trace this libedgedict_b200.so instead of this tree's")
    ap.add_argument("--tiles", type=int, default=48)
    args = ap.parse_args()

    import torch
    from edgedict_b200._lib import LIB_PATH, SIGNATURES
    assert torch.cuda.is_available(), "trace_joint_gemm.py reads clock64 stamps of CUDA kernels: it needs a GPU"
    h = ctypes.CDLL(os.path.abspath(args.lib or LIB_PATH))
    for name in ("eb_joint_logits_lse", "eb_gemm_bf16_dtanh", "eb_gemm_tc_set_trace"):
        res, argt = SIGNATURES[name]
        fn = getattr(h, name)
        fn.restype, fn.argtypes = res, argt

    dev = torch.device("cuda", 0)
    bf16, f32 = torch.bfloat16, torch.float32
    g = torch.Generator(device=dev).manual_seed(7)
    hid = (torch.rand(M, J, device=dev, generator=g) * 2 - 1).to(bf16)
    w2 = (torch.randn(V, J, device=dev, generator=g) * 0.04).to(bf16)
    b2 = torch.randn(V, device=dev, generator=g) * 0.1
    dl = (torch.randn(M, V, device=dev, generator=g) * 1e-3).to(bf16)
    labels = torch.randint(1, V, (B, U1 - 1), device=dev, dtype=torch.int32, generator=g)
    xlen = torch.full((B,), T, device=dev, dtype=torch.int32)
    ylen = torch.full((B,), U1 - 1, device=dev, dtype=torch.int32)
    logits = torch.empty(M, V, dtype=bf16, device=dev)
    stats = torch.empty(3, M, dtype=f32, device=dev)
    dpre = torch.empty(M, J, dtype=bf16, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    prods = {
        "logits_lse": lambda: h.eb_joint_logits_lse(p(hid), p(w2), p(b2), p(logits), p(labels), p(xlen), p(ylen),
                                                    p(stats[0]), p(stats[1]), p(stats[2]), B, T, U1, V, J, 0, st),
        "dhidden": lambda: h.eb_gemm_bf16_dtanh(p(dl), 0, p(w2), 1, p(dpre), p(hid), M, J, V, st),
    }
    buf = torch.zeros(args.tiles, SLOTS, dtype=torch.int64, device=dev)
    the_card = card()
    print("card:", the_card)
    out = {}
    for name, fn in prods.items():
        for _ in range(3):
            assert fn() == 0
        buf.zero_()
        assert h.eb_gemm_tc_set_trace(p(buf), args.tiles) == 0
        try:
            assert fn() == 0
            torch.cuda.synchronize()
        finally:
            h.eb_gemm_tc_set_trace(None, 0)
        s = buf.cpu().tolist()
        rows = []
        print("\n%s: CTA 0, cycles per tile" % name)
        print("%5s %8s %8s %8s %8s %8s %8s" % ("tile", "total", "wait", "mma", "epi", "epi_wait", "p_empty"))
        for i, t in enumerate(s):
            if t[0] == 0 or t[3] == 0:
                break
            r = dict(total=t[3] - t[0], wait=t[4], mma=t[2] - t[0] - t[4], epi=t[3] - t[2], epi_wait=t[6] - t[2],
                     p_empty=t[5])
            rows.append(r)
            print("%5d %8d %8d %8d %8d %8d %8d" % (i, r["total"], r["wait"], r["mma"], r["epi"], r["epi_wait"],
                                                   r["p_empty"]))
        warm = rows[1:] or rows
        med = {k: statistics.median(r[k] for r in warm) for k in ("total", "wait", "mma", "epi", "epi_wait", "p_empty")}
        print("median (tiles 1..%d): " % (len(rows) - 1) + "  ".join("%s %d" % kv for kv in med.items()))
        out[name] = dict(median=med, tiles=rows)
    print(json.dumps(dict(card=the_card, shapes=dict(M=M, J=J, V=V), medians={k: v["median"] for k, v in out.items()})))


if __name__ == "__main__":
    main()
