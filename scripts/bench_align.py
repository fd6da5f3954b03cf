#!/usr/bin/env python
"""Forced alignment at E6D2 shape: B = 32, T = 1000 -> T' = 500, U = 128 labels, V = 1024.

  python scripts/bench_align.py [--rounds N] [--reps K]

Four comparisons, each alternated within every round (K timed calls per arm after a warm-up), so all arms see the same
clocks and neighbours:
  model  : Transducer.align (encoder, predictor, joint, statistics, Viterbi, one copy of the frames) in fp32 and bf16
           mode, against Transducer.forward (the loss) without gradients on the same batch;
  stage  : the Viterbi + backtrace alone (eb_rnnt_viterbi) over a filled loss workspace, against the alpha lattice
           (eb_rnnt_loss_lattice, need_beta = 0) on the same workspace and against a batched torch restatement on the
           GPU, one max-plus step per anti-diagonal and a host backtrace (what a user would write without this);
  staged : the same two stages where the decisions / back-pointers exceed shared memory and the backtrace stages them
           from the caller's buffer (T' = 1000, U+1 = 256; CTC T = 2000, S = 511), against the α lattice of the loss
           at the same shapes;
  ctc    : edgedict_b200.ctc.forced_align over [32, 500, 1024] log-probs with S = 128 (scripts/bench_ctc.py's shape),
           against torchaudio's forced_align looped over the 32 utterances on CUDA and on the CPU (an arm is skipped
           when torchaudio or its CUDA op is absent).
Prints one JSON line: the card (name, power limit) read in the same run, ms per call for every round, and whether the
restatements chose the same paths.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, U, V, S = 32, 1000, 128, 1024, 128
E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0,
            dec_proj_size=256, joint_size=640)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                       # the measurement itself does not depend on it
        q = "nvidia-smi unavailable: %s" % e
    return q


def torch_viterbi(lpb, lpl):
    """Transducer Viterbi as a user would batch it in torch: full-length utterances, fp64 delta, one max-plus step per
    anti-diagonal on the device, then the decisions copied to the host and backtraced there.  Same tie rule as the
    kernel (stay unless emit is strictly greater)."""
    import numpy as np
    import torch
    Bn, Tn, Un = lpb.shape
    b64, l64 = lpb.double(), lpl.double()
    d = torch.full((Bn, Tn, Un), -float("inf"), dtype=torch.float64, device=lpb.device)
    emit_won = torch.zeros((Bn, Tn, Un), dtype=torch.bool, device=lpb.device)
    d[:, 0, 0] = 0
    ninf = torch.tensor(-float("inf"), dtype=torch.float64, device=lpb.device)
    for n in range(1, Tn + Un - 1):
        u = torch.arange(max(0, n - Tn + 1), min(n, Un - 1) + 1, device=lpb.device)
        t = n - u
        tm, um = (t - 1).clamp(min=0), (u - 1).clamp(min=0)
        stay = torch.where(t > 0, d[:, tm, u] + b64[:, tm, u], ninf)
        emit = torch.where(u > 0, d[:, t, um] + l64[:, t, um], ninf)
        e = emit > stay
        d[:, t, u] = torch.where(e, emit, stay)
        emit_won[:, t, u] = e
    score = d[:, Tn - 1, Un - 1] + b64[:, Tn - 1, Un - 1]
    dec = emit_won.cpu().numpy()
    frames = np.zeros((Bn, Un - 1), np.int32)
    for b in range(Bn):
        t, u = Tn - 1, Un - 1
        while u > 0:
            if t == 0 or dec[b, t, u]:
                u -= 1
                frames[b, u] = t
            else:
                t -= 1
    return frames, score


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    from edgedict_b200 import ctc, ops
    from edgedict_b200.rnnt.models import Transducer
    assert torch.cuda.is_available(), "bench_align.py measures on the GPU"
    torch.manual_seed(0)
    dev = torch.device("cuda")
    m = Transducer(**E6D2).to(dev)
    xs = torch.randn(B, T, E6D2["input_size"], device=dev)
    ys = torch.randint(1, V, (B, U), dtype=torch.int32, device=dev)
    xlen = torch.full((B,), T, dtype=torch.int32)
    ylen = torch.full((B,), U, dtype=torch.int32)
    Tp = (T + 1) // 2

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.reps

    def align(precision):
        def run():
            m.set_precision(precision)
            m.align(xs, ys, xlen, ylen)
        return run

    def loss(precision):
        def run():
            m.set_precision(precision)
            with torch.no_grad():
                m(xs, ys, xlen, ylen)
        return run

    model_arms = dict(align_fp32=align("fp32"), loss_fp32=loss("fp32"), align_bf16=align("bf16"),
                      loss_bf16=loss("bf16"))
    res = {k: [] for k in model_arms}
    for _ in range(a.rounds):
        for k, fn in model_arms.items():
            res[k].append(round(timed(fn), 3))
    torch.cuda.empty_cache()

    # the stage alone, over one workspace filled from random logits [B, T', U+1, V]
    xl = torch.full((B,), Tp, dtype=torch.int32, device=dev)
    yl = ylen.to(dev)
    acts = torch.randn(B, Tp, U + 1, V, device=dev)
    _, ws = ops.rnnt_loss_fwd(acts, ys, xl, yl, 0, need_beta=False)
    del acts
    torch.cuda.empty_cache()
    n = B * Tp * (U + 1)
    wsf = ws.view(torch.float32)
    lpb, lpl = wsf[n:2 * n].view(B, Tp, U + 1), wsf[2 * n:3 * n].view(B, Tp, U + 1)
    stage_arms = dict(viterbi=lambda: ops.rnnt_viterbi(xl, yl, B, Tp, U + 1, ws, torch.float32),
                      lattice_alpha=lambda: ops.rnnt_lattice(xl, yl, B, Tp, U + 1, ws, need_beta=False),
                      viterbi_torch=lambda: torch_viterbi(lpb, lpl))
    res.update({k: [] for k in stage_arms})
    for _ in range(a.rounds):
        for k, fn in stage_arms.items():
            res[k].append(round(timed(fn), 3))
    frames, _, score = ops.rnnt_viterbi(xl, yl, B, Tp, U + 1, ws, torch.float32)
    tf, ts = torch_viterbi(lpb, lpl)
    stage_same = dict(frames_equal=bool((frames.cpu().numpy() == tf).all()),
                      score_equal=bool(torch.equal(score, ts.float())))
    del ws, wsf, lpb, lpl
    torch.cuda.empty_cache()

    # decisions too large for shared memory (T' = 1000, U+1 = 256): the backtrace stages them from the caller's buffer
    Tg, Ug = 1000, 256
    wsg = torch.empty(ops.lib().eb_rnnt_workspace_bytes(B, Tg, Ug, 4), dtype=torch.uint8, device=dev)
    ng = B * Tg * Ug
    wsg.view(torch.float32)[ng:3 * ng] = -torch.rand(2 * ng, device=dev, generator=torch.Generator(dev).manual_seed(2))
    xg = torch.full((B,), Tg, dtype=torch.int32, device=dev)
    yg = torch.full((B,), Ug - 1, dtype=torch.int32, device=dev)
    global_arms = dict(viterbi_staged=lambda: ops.rnnt_viterbi(xg, yg, B, Tg, Ug, wsg, torch.float32),
                       lattice_alpha_staged_shape=lambda: ops.rnnt_lattice(xg, yg, B, Tg, Ug, wsg, need_beta=False))
    # CTC back-pointers too large for shared memory (T = 2000, S = 511), against the loss's lattice at the same shape
    Tc, Sc = 2000, 511
    lpc = torch.randn(B, Tc, V, device=dev).log_softmax(-1)
    tgc = torch.randint(1, V, (B, Sc), device=dev)
    ilc = torch.full((B,), Tc, dtype=torch.long)
    tlc = torch.full((B,), Sc, dtype=torch.long)
    tg32c = tgc.to(torch.int32).reshape(-1).contiguous()
    offc = (torch.arange(B, dtype=torch.int32, device=dev) * Sc)
    tlc32 = torch.full((B,), Sc, dtype=torch.int32, device=dev)
    ilc32 = torch.full((B,), Tc, dtype=torch.int32, device=dev)
    global_arms.update(
        ctc_align_staged=lambda: ctc.forced_align(lpc, tgc, ilc, tlc)[0].cpu(),
        ctc_loss_fwd_staged_shape=lambda: ops.ctc_loss_fwd(lpc.transpose(0, 1), tg32c, offc, tlc32, ilc32, Sc, 0, False))
    res.update({k: [] for k in global_arms})
    for _ in range(a.rounds):
        for k, fn in global_arms.items():
            res[k].append(round(timed(fn), 3))
    del wsg, lpc
    torch.cuda.empty_cache()

    # CTC at bench_ctc.py's shape
    g = torch.Generator(device=dev).manual_seed(1)
    lp = torch.randn(B, Tp, V, device=dev, generator=g).log_softmax(-1)
    tg = torch.randint(1, V, (B, S), device=dev, generator=g)
    il = torch.full((B,), Tp, dtype=torch.long)
    tl = torch.full((B,), S, dtype=torch.long)
    ctc_arms = dict(ctc_ours=lambda: ctc.forced_align(lp, tg, il, tl)[0].cpu())
    skipped = {}
    try:
        import torchaudio.functional as TAF
        tg32, lp_cpu, tg_cpu = tg.to(torch.int32), lp.cpu(), tg.to(torch.int32).cpu()

        def ta_loop(x, y):
            return [TAF.forced_align(x[b:b + 1], y[b:b + 1], blank=0)[0].cpu() for b in range(B)]

        try:
            ta_loop(lp, tg32)
            ctc_arms["ctc_torchaudio_cuda"] = lambda: ta_loop(lp, tg32)
        except Exception as e:
            skipped["ctc_torchaudio_cuda"] = str(e)[:200]
        ctc_arms["ctc_torchaudio_cpu"] = lambda: ta_loop(lp_cpu, tg_cpu)
    except Exception as e:
        skipped["torchaudio"] = str(e)[:200]
    res.update({k: [] for k in ctc_arms})
    for _ in range(a.rounds):
        for k, fn in ctc_arms.items():
            res[k].append(round(timed(fn), 3))
    ctc_same = None
    if "ctc_torchaudio_cpu" in ctc_arms:
        ours = ctc.forced_align(lp, tg, il, tl)[0].cpu()
        theirs = torch.cat(ta_loop(lp_cpu, tg_cpu))
        same = (ours == theirs).all(dim=1)
        # where the paths differ: both paths' log-probs summed in fp64 (ours is the fp64 optimum)
        lp64, fr = lp_cpu.double(), torch.arange(Tp)
        ctc_same = dict(equal=int(same.sum()), differing=[
            dict(utt=b, ours_fp64=float(lp64[b, fr, ours[b].long()].sum()),
                 torchaudio_fp64=float(lp64[b, fr, theirs[b].long()].sum())) for b in range(B) if not bool(same[b])])
    print(json.dumps(dict(card=card(), B=B, T=T, T_out=Tp, U=U, V=V, S=S, reps=a.reps, ms=res,
                          stage_matches_torch_restatement=stage_same,
                          ctc_utterances_equal_to_torchaudio_cpu=ctc_same, skipped=skipped)))


if __name__ == "__main__":
    main()
