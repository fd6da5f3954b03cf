#!/usr/bin/env python
"""bench.py -- headline benchmark of BASELINE.json:

  metric  audio-sec/sec, E6D2 training step (encoder LSTM stack -> predictor -> joint -> rnnt_loss,
          forward + backward + Adam), B=32 per GPU, T=1000 frames (37.5 ms each), U=128, V=1024.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]
  torchrun --nproc-per-node N bench.py --gpus N ...        (one rank per GPU, NCCL)

"ours": the H100 engine in bf16 mode (wgmma GEMMs, fp32 accumulate / fp32 recurrent state),
weak scaling (B=32 per GPU), one all-reduce of the flat gradient bucket per step; the line also carries
`strong_scaling` (BASELINE configs[2]: global B=256 as 8/N accumulation micro-steps of 32 per GPU, one all-reduce
per optimizer step -- the reference's sub_batch mechanism, cli/baseline.py:214-237) and `parity_probe` (loss of the
bf16 bench mode against the fp32 parity mode of the same weights).  `--scaling strong` makes the strong-scaling
figure the headline instead.
"reference": the reference's own CPU path restated in oracle/model_torch.py (torch-CPU fp32,
nn.LSTM's ATen kernel) + the reference's compiled warp-transducer CPU library (oracle/_ref) on the SAME config:
the B=32 step is executed the way the reference itself runs a large batch on a small device, as accumulation
sub-batches of the same utterance shape (T=1000, U=128); each timed "step" is one sub-batch (a bounded sample:
1/16 of the optimizer step), the optimizer update is applied every 16th sub-batch inside the timed region.
Prints ONE JSON line on rank 0.

--dump-outputs DIR (ours): after the timed steps of the headline leg, rank 0 writes what the last of them computed --
loss.npy (the step's loss) and a fixed, seeded sample of the flat gradient and parameter buckets after the optimizer
update (grads_sample.npy, params_sample.npy; sample_index.npy holds the bucket positions) -- so that two builds can be
compared output for output on identical seeded inputs.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FRAME_SEC = 0.0375          # E6D2: downsample 3 x hop 200 / 16 kHz (flagfiles/E6D2.txt:28,31)
E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6,
            enc_dropout=0.0, enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0,
            dec_proj_size=256, joint_size=640)
B, T, U, V = 32, 1000, 128, 1024
GLOBAL_B = 256              # BASELINE configs[2]


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=d["hbm_gbs"], tf_burst=d["bf16_tflops"], tf_sus=d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                    src="measured")
    # NVIDIA's H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s -- bounds, not reached figures
    return dict(hbm=3350.0, tf_burst=989.0, tf_sus=989.0, src="H100 SXM data sheet")


DUMP_SAMPLE = 1 << 21       # bucket elements sampled per dumped array: 32 MB in all with the float64 positions


def dump_outputs(path, loss, opt):
    """The headline leg's last step, as float arrays: loss, and a seeded sample of the gradient / parameter buckets."""
    import numpy as np
    import torch
    os.makedirs(path, exist_ok=True)
    n = opt.flat_grads.numel()
    g = torch.Generator().manual_seed(1234)
    idx = torch.randperm(n, generator=g)[:min(n, DUMP_SAMPLE)].sort().values
    di = idx.to(opt.flat_grads.device)
    np.save(os.path.join(path, "loss.npy"), np.array([float(loss)], dtype=np.float64))
    np.save(os.path.join(path, "grads_sample.npy"), opt.flat_grads[di].cpu().numpy().astype(np.float32))
    np.save(os.path.join(path, "params_sample.npy"), opt.flat_params[di].cpu().numpy().astype(np.float32))
    np.save(os.path.join(path, "sample_index.npy"), idx.numpy().astype(np.float64))


class ClockSampler:
    FIELDS = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None
        self.t0 = self.t1 = None

    # nvidia-smi is started BEFORE the warm-up and stopped after the last leg: its start-up (NVML initialisation, a driver lock)
    # and its teardown each stalled kernel launches for 50 - 100 ms when they fell inside a timed region (one step in ~10 % of the
    # runs: 55 ms instead of 46).  The rows are time-stamped as they arrive; the report uses those inside [begin(), end()].
    def begin(self):
        self.t0 = time.time()

    def end(self):
        self.t1 = time.time()

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.FIELDS,
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")] + [time.time()])

    def stop(self):
        if self.proc is None:
            return None
        self.proc.terminate()
        if self.t0 is not None and self.t1 is not None:
            inside = [r for r in self.rows if self.t0 <= r[-1] <= self.t1 + 0.25]     # (a row describes the 200 ms before it)
            if inside:
                self.rows = inside
        sm = sorted(int(r[0]) for r in self.rows if r and r[0].isdigit())
        if not sm:
            return None
        reasons = []
        for i, name in enumerate(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap")):
            if any(len(r) > 2 + i and r[2 + i].lower().startswith("active") for r in self.rows):
                reasons.append(name)
        mx = [int(r[1]) for r in self.rows if len(r) > 1 and r[1].isdigit()]
        return dict(sm_mhz=sm[len(sm) // 2], sm_max_mhz=max(mx) if mx else None, reasons=reasons, samples=len(sm))


def run_ours(args):
    import torch
    from edgedict_b200 import dist as ed
    from edgedict_b200 import ops
    from edgedict_b200.optim import FlatAdam
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200._lib import lib
    lib()                                             # fail loudly if the CUDA library is missing
    rank, world, local = ed.init_from_env("nccl")
    assert world == args.gpus, "launch with torchrun --nproc-per-node %d" % args.gpus
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    torch.manual_seed(10)
    model = Transducer(**E6D2).to(dev)
    model.set_precision(args.precision)
    opt = FlatAdam(model, lr=5e-4)
    ed.broadcast_bucket(opt.flat_params)
    g = torch.Generator(device=dev).manual_seed(10 + rank)
    xs = torch.randn(B, T, 240, device=dev, generator=g)
    ys = torch.randint(4, V, (B, U), device=dev, dtype=torch.int32, generator=g)
    xlen = torch.full((B,), T, dtype=torch.int32)
    ylen = torch.full((B,), U, dtype=torch.int32)
    # pinned host copies for the end-to-end leg
    hx, hy = xs.cpu().pin_memory(), ys.cpu().pin_memory()

    strong = args.scaling == "strong"
    micro = max(1, GLOBAL_B // (B * world))           # configs[2]: B=256 global -> 8/N micro-steps of 32 per GPU
    if strong:
        assert B * world * micro == GLOBAL_B, "strong scaling needs N in {1, 2, 4, 8}"

    def step(x, y, n_micro=None):
        """One optimizer step: n_micro accumulation micro-steps (gradients add up in the flat bucket), ONE all-reduce,
        one fused Adam launch with the 1/n_micro scale folded in."""
        n_micro = (micro if strong else 1) if n_micro is None else n_micro
        opt.zero_grad()
        for _ in range(n_micro):
            loss = model(x, y, xlen, ylen)
            loss.backward()
        ed.allreduce_bucket(opt.flat_grads, world)
        opt.step(grad_scale=1.0 / n_micro)
        return loss

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()                                            # (see ClockSampler: outside every timed region)
    min_warm = int(os.environ.get("EB_BENCH_MIN_WARMUP", "3"))       # only lowered for ncu captures
    for _ in range(max(args.warmup, min_warm)):
        loss = step(xs, ys)
    barrier()
    first_loss = float(loss.detach())
    probe = parity_probe(model, dev) if rank == 0 else None
    barrier()

    # ---- leg 1: inputs resident in HBM, per-kernel events on --------------------------------------
    ops.PROF.reset()
    ops.PROF.enabled = True
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler.begin()
    e0.record()
    for _ in range(args.steps):
        loss = step(xs, ys)
    e1.record()
    barrier()
    sampler.end()
    ms_dev = ed.max_over_ranks(e0.elapsed_time(e1), dev) / args.steps
    prof = ops.PROF.summary(base=e0)
    launches = ops.PROF.launches // args.steps
    ops.PROF.enabled = False
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss.detach(), opt)

    # ---- leg 2: end to end through the public API with host buffers --------------------------------
    # Every step's inputs are copied from pinned host memory and every step's loss is read back on the host,
    # all inside the timed region, software-pipelined the way a training loop is written: the upload of step
    # i+1 is issued on a copy stream while step i computes, and the loss of step i is read (a blocking event
    # wait + host read) after step i+1 has been enqueued, so the device never idles behind the host.
    copy_stream = torch.cuda.Stream(dev)
    main_stream = torch.cuda.current_stream(dev)
    hl = [torch.zeros(1).pin_memory() for _ in range(2)]
    lev = [torch.cuda.Event() for _ in range(2)]
    host_losses = []

    def upload():
        with torch.cuda.stream(copy_stream):
            x = hx.to(dev, non_blocking=True)
            y = hy.to(dev, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return x, y, ev

    for _ in range(2):                                  # warm the copy stream's allocator pool (untimed)
        x, y, ev = upload()
        main_stream.wait_event(ev)
        x.record_stream(main_stream)
        y.record_stream(main_stream)
        step(x, y)
    barrier()
    import time as _time
    step_wall = []
    e0.record()
    nxt = upload()
    for i in range(args.steps):
        _t0 = _time.perf_counter()
        x, y, ev = nxt
        main_stream.wait_event(ev)
        x.record_stream(main_stream)
        y.record_stream(main_stream)
        if i + 1 < args.steps:
            nxt = upload()
        loss = step(x, y)
        hl[i % 2].copy_(loss.detach(), non_blocking=True)
        lev[i % 2].record(main_stream)
        if i > 0:
            lev[(i - 1) % 2].synchronize()
            host_losses.append(float(hl[(i - 1) % 2]))
        step_wall.append(round((_time.perf_counter() - _t0) * 1e3, 2))
    lev[(args.steps - 1) % 2].synchronize()
    host_losses.append(float(hl[(args.steps - 1) % 2]))
    e1.record()
    barrier()
    ms_e2e = ed.max_over_ranks(e0.elapsed_time(e1), dev) / args.steps
    last_loss = host_losses[-1]
    assert len(host_losses) == args.steps

    # ---- leg 3: BASELINE configs[2] strong scaling (global B=256), two optimizer steps after one warm-up
    strong_ms = None
    if not strong and B * world * micro == GLOBAL_B:
        step(xs, ys, micro)
        barrier()
        e0.record()
        for _ in range(2):
            step(xs, ys, micro)
        e1.record()
        barrier()
        strong_ms = ed.max_over_ranks(e0.elapsed_time(e1), dev) / 2

    if rank != 0:
        return None
    clocks = sampler.stop()                                        # after the last timed leg
    pk = peaks()
    audio = world * B * T * FRAME_SEC * (micro if strong else 1)
    kern = {}
    for name, d in prof.items():
        ms = d["ms"] / args.steps
        kern[name] = dict(ms_per_step=round(ms, 4), ms_sum_per_step=round(d["ms_sum"] / args.steps, 4),
                          calls_per_step=d["calls"] / args.steps,
                          share=round(ms / ms_dev, 4),
                          gbs=round(d["bytes"] / args.steps / ms / 1e6, 1) if d["bytes"] else None,
                          tflops=round(d["flops"] / args.steps / ms / 1e9, 2) if d["flops"] else None)
    top = max(kern, key=lambda k: kern[k]["ms_per_step"])
    hbm_kernels = ("rnnt_loss_bwd", "rnnt_loss_fwd")
    kern = {k: v for k, v in kern.items() if v["ms_per_step"] > 0}
    if top in hbm_kernels:
        ach = kern[top]["gbs"]
        roof = dict(kernel=top, bound="hbm", achieved=ach, peak=pk["hbm"], unit="GB/s", frac=round(ach / pk["hbm"], 4))
    else:
        ach = kern[top]["tflops"] or 0.0
        roof = dict(kernel=top, bound="tensor", achieved=ach, peak=pk["tf_sus"], unit="TFLOP/s",
                    frac=round(ach / pk["tf_sus"], 4))
    if top.startswith("lstm_tc"):
        # SURVEY 8(d): the recurrent critical path is latency-, not throughput-bound -- report it per timestep
        cell_steps = 2 * T + (E6D2["enc_layers"] - 2) * (T // 2) + E6D2["dec_layers"] * (U + 1)
        roof["us_per_timestep"] = round(kern[top]["ms_per_step"] * 1e3 / cell_steps, 3)
        roof["timesteps"] = cell_steps
        roof["note"] = ("grid-synchronous recurrence: one exchange + barrier per timestep, %d sequential steps per "
                        "training step; the tensor-pipe fraction is what the dependency chain leaves, the figure "
                        "to track is us_per_timestep" % cell_steps)
    roof["peak_source"] = pk["src"] + (" (sustained)" if roof["bound"] == "tensor" else "")
    # the BASELINE.json side metric: joint+loss HBM fraction on the algorithmic bytes of SURVEY 8(d)
    n_logits = B * (T // 2) * (U + 1) * V
    if "joint_logits_lse" in kern:
        # fused bf16 path, joint GEMM inside the region: SURVEY 8(d) counts 4*s*N with the GEMM included (logits
        # written by the epilogue, read for the denominators, read + gradient written by the gradient pass), s = 2
        # for the bf16 logits this path materialises.  The denominators come out of the GEMM epilogue, so the
        # kernels actually move 3*s*N; the achieved figure is still algorithmic bytes / time.
        jl_keys = ("joint_logits_lse", "rnnt_loss_fwd", "rnnt_loss_bwd")
        jl_bytes = 4 * 2 * n_logits
        note = ("s=2 (bf16 logits), joint GEMM + lattice + in-place gradient; algorithmic 4*s*N (GEMM included), moved "
                "3*s*N: the softmax statistics come out of the GEMM epilogue")
    else:
        jl_keys = hbm_kernels
        jl_bytes = (4 + 4 + (2 if args.precision == "bf16" else 4)) * n_logits
        note = "s=4 logits; denominator pass + lattice + gradient (joint GEMM not included)"
    jl_ms = sum(kern[k]["ms_per_step"] for k in jl_keys if k in kern)
    joint_loss = dict(algorithmic_gb=round(jl_bytes / 1e9, 2), ms=round(jl_ms, 3),
                      gbs=round(jl_bytes / jl_ms / 1e6, 1), frac_hbm=round(jl_bytes / jl_ms / 1e6 / pk["hbm"], 4),
                      what=note)
    out = dict(metric="audio-sec/sec E6D2 B=32 T=1000 U=128 V=1024 training step", value=round(audio / ms_dev * 1e3, 1),
               unit="audio-sec/sec", n_gpus=world, steps=args.steps, warmup=max(args.warmup, 3),
               ms_per_step=round(ms_dev, 3), higher_is_better=True, scaling="strong" if strong else "weak", vs_baseline=None,
               dtype="bf16" if args.precision == "bf16" else "f32", data="synthetic",
               config=dict(workload="E6D2 (6x1024 LSTM enc / 2x256 pred / joint 640 / V=1024) fwd+loss+bwd+Adam, "
                                    "B=32/GPU T=1000 U=128 (configs[1]); frame=37.5 ms",
                           global_batch=B * world * (micro if strong else 1), seq_len=T, parallelism="dp%d" % world,
                           micro_steps_per_optimizer_step=micro if strong else 1,
                           l2="inputs >> L2: 4.2 GB of bf16 logits (8.45 GB with EDGEDICT_FUSE_LSE=0) streamed per step"),
               e2e=dict(value=round(audio / ms_e2e * 1e3, 1), unit="audio-sec/sec",
                        h2d_bytes_per_step=hx.numel() * 4 + hy.numel() * 4, d2h_bytes_per_step=4,
                        ms_per_step=round(ms_e2e, 3), host_ms_per_iteration=step_wall),
               gpu_launches=launches, clocks=clocks, roofline=roof, joint_loss_hbm=joint_loss, kernels=kern,
               loss_first=round(first_loss, 4), loss_last=round(last_loss, 4), parity_probe=probe)
    if strong_ms is not None:
        out["strong_scaling"] = dict(global_batch=GLOBAL_B, micro_steps=micro, ms_per_optimizer_step=round(strong_ms, 3),
                                     value=round(GLOBAL_B * T * FRAME_SEC / strong_ms * 1e3, 1), unit="audio-sec/sec",
                                     what="BASELINE configs[2]: 8/N accumulation micro-steps of B=32 per GPU, one "
                                          "all-reduce + one Adam launch per optimizer step")
    return out


def parity_probe(model, dev):
    """Loss of the bf16 bench mode against the fp32 parity mode (same weights, same inputs) on a probe batch of the
    benchmark's hidden sizes: the figure tests/test_gpu_parity_bf16.py asserts against the CPU oracle."""
    import torch
    g = torch.Generator(device=dev).manual_seed(123)
    xs = torch.randn(4, 200, 240, device=dev, generator=g)
    ys = torch.randint(4, V, (4, 32), device=dev, dtype=torch.int32, generator=g)
    xlen = torch.tensor([200, 200, 171, 150], dtype=torch.int32)
    ylen = torch.tensor([32, 25, 32, 17], dtype=torch.int32)
    with torch.no_grad():
        l16 = float(model(xs, ys, xlen, ylen))
        model.set_precision("fp32")
        l32 = float(model(xs, ys, xlen, ylen))
        model.set_precision("bf16")
    return dict(shape="E6D2 B=4 T=200 U=32 ragged", loss_bf16=round(l16, 5), loss_fp32=round(l32, 5),
                rel_err=abs(l16 - l32) / abs(l32), bar=1e-3)


REF_SUB_B = 2               # utterances per accumulation sub-batch of the CPU arm (same T, U as the GPU arm)


def run_reference(steps, warmup, sub_b=REF_SUB_B):
    """The reference's CPU path (oracle port of rnnt/models.py + compiled warp-transducer CPU loss) on the bench
    config: B=32 T=1000 U=128 executed as 32/sub_b accumulation sub-batches of identical shape, the reference's own
    mechanism for batches that do not fit a device (cli/baseline.py:214-237).  One timed "step" = one sub-batch
    (forward + loss + backward into the accumulated gradients); the Adam update runs once every 32/sub_b
    sub-batches, inside the timed region.  audio-sec/sec = sub_b * T * 37.5 ms / seconds per sub-batch."""
    import torch
    from oracle import loss as ol
    from oracle import model_torch as mt
    from edgedict_b200.rnnt.models import Transducer          # parameter container only (same init)
    # torch's CPU LSTM / GEMM kernels and the OpenMP loss stop scaling (and then degrade badly: 5x slower
    # at 128 threads than at 8 on the GPU box's host) well before a big host's core count: use at most 32
    cores = min(os.cpu_count() or 1, 32)
    torch.set_num_threads(cores)
    os.environ["OMP_NUM_THREADS"] = str(cores)
    ol.NUM_THREADS = cores
    torch.manual_seed(10)
    shell = Transducer(**E6D2)
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in shell.state_dict().items()}
    optim = torch.optim.Adam(list(sd.values()), lr=5e-4)
    n_sub = B // sub_b
    torch.manual_seed(10)
    xs = torch.randn(sub_b, T, 240)
    ys = torch.randint(4, V, (sub_b, U), dtype=torch.int32)
    xlen, ylen = torch.full((sub_b,), T, dtype=torch.int32), torch.full((sub_b,), U, dtype=torch.int32)
    done = [0]

    def one():
        if done[0] % n_sub == 0:
            optim.zero_grad()
        loss = mt.transducer_loss(sd, xs, ys, xlen, ylen, fast=True, use_ref=True) / n_sub
        loss.backward()
        done[0] += 1
        if done[0] % n_sub == 0:
            optim.step()
        return float(loss.detach()) * n_sub

    for _ in range(warmup):
        one()
    t0 = time.perf_counter()
    for _ in range(steps):
        one()
    dt = (time.perf_counter() - t0) / steps
    val = sub_b * T * FRAME_SEC / dt
    kind = "reference" if ol.have_ref() else "port"
    if kind == "port":
        print("bench.py: oracle/_ref/libwarprnnt_ref.so is not built: the CPU baseline's loss runs this project's C "
              "oracle, NOT the reference's warp-transducer library", file=sys.stderr)
    sample = ("E6D2 B=32 T=1000 U=128 V=1024 fwd+loss+bwd+Adam fp32 as %d accumulation sub-batches of B=%d T=%d U=%d; "
              "%d sub-batch(es) timed (%.1f s each), optimizer step every %d" % (n_sub, sub_b, T, U, steps, dt, n_sub))
    return dict(value=round(val, 3), unit="audio-sec/sec", cores=cores,
                kind=kind + " (warp-transducer CPU lib compiled from the reference; model = torch-CPU port "
                            "calling the same ATen LSTM kernel as nn.LSTM)" if kind == "reference" else
                "port (oracle/_ref not built: loss from this project's C oracle, not the reference's library; model = "
                "torch-CPU port calling the same ATen LSTM kernel as nn.LSTM)", sample=sample), dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--scaling", default="weak", choices=["weak", "strong"])
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's loss and seeded gradient / parameter samples as DIR/<name>.npy")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    if args.impl == "reference":
        if rank != 0:
            return
        # a sub-batch of the full-size utterances takes several seconds on the host: keep the whole run within minutes
        steps, warmup = min(args.steps, 8), min(args.warmup, 1)
        cb, dt = run_reference(steps, warmup)
        print(json.dumps(dict(impl="reference", metric="audio-sec/sec E6D2 B=32 T=1000 U=128 V=1024 training step",
                              value=cb["value"], unit="audio-sec/sec", n_gpus=args.gpus, steps=steps,
                              warmup=warmup, requested_steps=args.steps, requested_warmup=args.warmup,
                              ms_per_step=round(dt * 1e3 * (B // REF_SUB_B), 1), higher_is_better=True,
                              scaling="weak", vs_baseline=None, dtype="f32", data="synthetic",
                              config=dict(workload="E6D2 (6x1024 LSTM enc / 2x256 pred / joint 640 / V=1024) fwd+loss+bwd+Adam, "
                                                   "B=32/GPU T=1000 U=128 (configs[1]); frame=37.5 ms",
                                          global_batch=B, seq_len=T, parallelism="host cores",
                                          sub_batches_timed=steps, sub_batches_warmup=warmup,
                                          how=cb["sample"]),
                              cpu_baseline=cb, gpu_launches=0,
                              e2e=dict(value=cb["value"], unit="audio-sec/sec", h2d_bytes_per_step=0,
                                       d2h_bytes_per_step=0))))
        return
    out = run_ours(args)
    import torch.distributed as dist
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()
    if out is None:
        return
    if args.gpus == 1 and not args.no_cpu_baseline:
        cb, _ = run_reference(2, 1)          # 1 warm-up + 2 timed sub-batches of the full-size utterances
        out["cpu_baseline"] = cb
    print(json.dumps(out))


if __name__ == "__main__":
    main()
