"""BASELINE.json configs[4]: joint + rnnt_loss isolation sweep, T' in {250,500,1000,2000} x U in {64,128,256},
V=1024, B=32 halved until fp32 logits + bf16 gradients (6N bytes) fit in 60 GB of the H100's 80 GB: HBM GB/s of the loss kernels against the
measured copy bandwidth, the joint logits GEMM beside it, and the loss checked against the oracle on a
sub-problem small enough for the CPU.  Run on an H100:  python scripts/bench_sweep.py [out.json]"""
import json, os, sys
import numpy as np
import torch
sys.path.insert(0, os.getcwd())
from edgedict_b200 import ops
from oracle import loss as ol

peaks = json.load(open("MEASURED_PEAKS.json")) if os.path.exists("MEASURED_PEAKS.json") else {"hbm_gbs": 3350.0}   # H100 SXM data sheet
HBM = peaks["hbm_gbs"]
V, J = 1024, 640
rows = []
torch.manual_seed(10)
w2 = (torch.randn(V, J, device="cuda") / 25).bfloat16()
b2 = torch.zeros(V, device="cuda")
for T in (250, 500, 1000, 2000):
    for U in (64, 128, 256):
        U1 = U + 1
        B = 32
        while B > 1 and 6 * B * T * U1 * V > 60e9:
            B //= 2
        g = torch.Generator(device="cuda").manual_seed(T * 1000 + U)
        hid = torch.randn(B * T * U1, J, device="cuda", generator=g).mul_(0.5).bfloat16()
        logits = torch.empty(B * T * U1, V, device="cuda")
        lab = torch.randint(1, V, (B, U), device="cuda", dtype=torch.int32, generator=g)
        xl = torch.full((B,), T, device="cuda", dtype=torch.int32)
        yl = torch.full((B,), U, device="cuda", dtype=torch.int32)
        grads = torch.empty(B, T, U1, V, device="cuda", dtype=torch.bfloat16)
        l4 = logits.view(B, T, U1, V)

        def step():
            ops.gemm_bf16(hid, 0, w2, 0, B * T * U1, V, J, bias=b2, out=logits)
            costs, ws = ops.rnnt_loss_fwd(l4, lab, xl, yl, 0)
            ops.rnnt_loss_bwd(l4, lab, xl, yl, 0, ws, None, 1.0 / B, out=grads)
            return costs
        for _ in range(2):
            costs = step()
        torch.cuda.synchronize()
        ops.PROF.reset(); ops.PROF.enabled = True
        n = 3
        for _ in range(n):
            costs = step()
        torch.cuda.synchronize()
        pr = ops.PROF.summary(); ops.PROF.enabled = False
        ms = {k: v["ms"] / n for k, v in pr.items()}
        N = B * T * U1 * V
        loss_ms = ms["rnnt_loss_fwd"] + ms["rnnt_loss_bwd"]
        alg = (4 + 4 + 2) * N                                  # read, read, write bf16
        # oracle check on the first utterance cropped to 24 x 12 cells
        sub = l4[:1, :24, :12].contiguous()
        c_s, _ = ops.rnnt_loss_fwd(sub, lab[:1, :11].contiguous(), torch.tensor([24], dtype=torch.int32, device="cuda"),
                                   torch.tensor([11], dtype=torch.int32, device="cuda"), 0)
        c_o, _ = ol.logits(sub.cpu().numpy(), lab[:1, :11].cpu().numpy(), [24], [11], want_grads=False, dtype=np.float64)
        rel = float(abs(c_s.cpu().numpy()[0] - c_o[0]) / abs(c_o[0]))
        r = dict(T=T, U=U, B=B, logits_gb=round(4 * N / 1e9, 2), denom_lattice_ms=round(ms["rnnt_loss_fwd"], 3),
                 grad_ms=round(ms["rnnt_loss_bwd"], 3), loss_gbs=round(alg / loss_ms / 1e6, 1),
                 loss_frac_hbm=round(alg / loss_ms / 1e6 / HBM, 3), joint_gemm_ms=round(ms["gemm_bf16_nt"], 3),
                 joint_gemm_tflops=round(2.0 * B * T * U1 * V * J / ms["gemm_bf16_nt"] / 1e9, 1),
                 joint_plus_loss_gbs=round((alg + 4 * N) / (loss_ms + ms["gemm_bf16_nt"]) / 1e6, 1),
                 loss_rel_err_vs_oracle=float("%.2e" % rel), finite=bool(torch.isfinite(costs).all()))
        # ---- the path bench.py runs (bf16 mode): logits GEMM with the softmax statistics in its epilogue (bf16 logits),
        # lattice, in-place bf16 gradient.  SURVEY 8(d): 4*s*N with the GEMM inside the region, s = 2.
        del logits, grads, l4
        torch.cuda.empty_cache()

        def fused():
            lg, ws = ops.joint_logits_lse(hid, w2, b2, lab, xl, yl, B, T, U1, 0)
            costs = ops.rnnt_lattice(xl, yl, B, T, U1, ws)
            ops.rnnt_loss_bwd_bf16(lg, lab, xl, yl, 0, ws, None, 1.0 / B)
            return costs
        for _ in range(2):
            cf = fused()
        torch.cuda.synchronize()
        ops.PROF.reset(); ops.PROF.enabled = True
        for _ in range(n):
            cf = fused()
        torch.cuda.synchronize()
        pr = ops.PROF.summary(); ops.PROF.enabled = False
        fm = {k: v["ms"] / n for k, v in pr.items()}
        f_ms = fm["joint_logits_lse"] + fm["rnnt_loss_fwd"] + fm["rnnt_loss_bwd"]
        # loss of the fused path against the C oracle on utterance 0 cropped to 24 x 12 cells (logits from the same
        # bf16 operands, accumulated in fp64 on the host)
        idx = (torch.arange(24, device="cuda")[:, None] * U1 + torch.arange(12, device="cuda")[None, :]).reshape(-1)
        hs = hid[idx].contiguous()
        one = lambda v: torch.tensor([v], dtype=torch.int32, device="cuda")
        lgs, wss = ops.joint_logits_lse(hs, w2, b2, lab[:1, :11].contiguous(), one(24), one(11), 1, 24, 12, 0)
        cs = ops.rnnt_lattice(one(24), one(11), 1, 24, 12, wss)
        ref_logits = (hs.double().cpu() @ w2.double().cpu().t()).view(1, 24, 12, V).numpy()
        co, _ = ol.logits(ref_logits, lab[:1, :11].cpu().numpy(), [24], [11], want_grads=False, dtype=np.float64)
        r.update(fused_gemm_lse_ms=round(fm["joint_logits_lse"], 3), fused_lattice_ms=round(fm["rnnt_loss_fwd"], 3),
                 fused_grad_ms=round(fm["rnnt_loss_bwd"], 3), fused_total_ms=round(f_ms, 3),
                 fused_gbs=round(4 * 2 * N / f_ms / 1e6, 1), fused_frac_hbm=round(4 * 2 * N / f_ms / 1e6 / HBM, 3),
                 fused_grad_gbs=round(2 * 2 * N / fm["rnnt_loss_bwd"] / 1e6, 1),
                 fused_gemm_tflops=round(2.0 * N * J / fm["joint_logits_lse"] / 1e9, 1),
                 fused_loss_rel_err_vs_oracle=float("%.2e" % (abs(float(cs[0]) - co[0]) / abs(co[0]))),
                 fused_finite=bool(torch.isfinite(cf).all()))
        rows.append(r)
        print(json.dumps(r), flush=True)
        del hid
        torch.cuda.empty_cache()
if len(sys.argv) > 1:
    json.dump(dict(hbm_peak_gbs=HBM, rows=rows), open(sys.argv[1], "w"), indent=1)
