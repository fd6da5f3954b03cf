"""Measures one wav2vec pre-training sub-batch (forward + backward) at cli/pretrain_wav2vec.py's shape on the engine in
bf16 and fp32 mode, against a torch/cuDNN restatement of the reference's step kept in this script.

    python scripts/bench_wav2vec.py [--rounds 5] [--B 24] [--seconds 14]

Workload: B = 24 utterances of 14 s at 16 kHz; FrontEnd [(10,5,32)] + [(3,2,128)]*4 + [(2,2,128)]*3 without bias,
input_size 128, a 4 x 512 LSTM encoder with proj 512, K = 100 negatives, G = 2 groups of V = 320 codes, mask_prob 0.15,
mask_length 10; loss weights (0.1, 10) and the CLI's log keys.  Each round runs the three arms in turn with the same
seeds and reports, per arm, the whole step and the head alone (mask -> cross-entropy: everything but the front end and
the encoder, timed as the step minus front end and encoder forward + backward run on their own).  Prints one JSON
line with median times and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from edgedict_b200.rnnt import wav2vec as w2v            # noqa: E402

FE = [(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:
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


class TorchRef(torch.nn.Module):
    """The reference's step in plain torch (cuDNN LSTM, torch convolutions, torch quantizer, logits and loss) on the
    engine model's weights: rnnt/wav2vec.py and modules/softmax_vector_quantizer.py restated for the benchmark."""

    def __init__(self, m):
        super().__init__()
        self.m = m
        enc = m.encoder
        self.lstms = torch.nn.ModuleList()
        for cell in enc.lstm.lstms:
            l = torch.nn.LSTM(cell.input_size, cell.hidden_size, 1, batch_first=True).cuda()
            l.load_state_dict(cell.state_dict())
            self.lstms.append(l)

    def frontend(self, x):
        fe = self.m.frontend
        c = fe.conv1
        y = F.conv1d(x[:, None], c.weight, c.bias, stride=c.stride, padding=c.padding)[:, :, :-c.padding[0]]
        for blk in fe.encode:
            y = F.gelu(y)
            y = F.group_norm(y, 1, blk.gn.weight, blk.gn.bias, blk.gn.eps)
            y = F.conv1d(y, blk.conv.weight, blk.conv.bias, stride=blk.conv.stride, padding=blk.conv.padding)
            y = y[:, :, :-blk.conv.padding[0]]
        y = y.transpose(1, 2)
        return F.layer_norm(y, (y.shape[-1],), fe.layer_norm.weight, fe.layer_norm.bias, fe.layer_norm.eps)

    def encoder(self, x):
        enc = self.m.encoder
        x = F.layer_norm(x, (x.shape[-1],), enc.norm.weight, enc.norm.bias, enc.norm.eps)
        for i, (l, post) in enumerate(zip(self.lstms, enc.lstm.projs)):
            y, _ = l(x)
            ln = post[0]
            x = F.layer_norm(y + (x if i else 0), (y.shape[-1],), ln.weight, ln.bias, ln.eps)
        return F.linear(x, enc.proj.weight, enc.proj.bias)

    def head(self, features, x, mask, neg):
        m, q = self.m, self.m.quantizer
        B, T, C = features.shape
        fpen = features.float().pow(2).mean()
        xin = features.clone()
        xin[mask] = m.mask_emb
        y = features[mask].view(B, -1, C)
        M = y.shape[1]
        l = F.linear(y.reshape(-1, C), q.weight_proj.weight, q.weight_proj.bias).view(B * M * q.groups, -1)
        k = l.argmax(-1)
        hard = torch.zeros_like(l).scatter_(-1, k[:, None], 1.0).view(B * M, q.groups, -1).mean(0)
        cp = torch.exp(-(hard * torch.log(hard + 1e-7)).sum(-1)).sum()
        avg = torch.softmax(l.view(B * M, q.groups, -1), -1).mean(0)
        pp = torch.exp(-(avg * torch.log(avg + 1e-7)).sum(-1)).sum()
        s = F.gumbel_softmax(l, tau=q.curr_temp, hard=True).view(B * M, -1)
        yq = (s.unsqueeze(-1) * q.vars).view(B * M, q.groups, q.num_vars, -1).sum(-2).view(B, M, -1)
        yq = F.linear(yq, m.project_q.weight, m.project_q.bias)
        negs = yq.reshape(-1, yq.shape[-1])[(neg + torch.arange(B, device=neg.device)[:, None] * M).view(-1)]
        negs = negs.view(B, M, m.n_negatives, -1).permute(2, 0, 1, 3)
        xm = F.linear(x[mask].view(B, M, -1), m.final_proj.weight, m.final_proj.bias)
        same = (yq == negs).all(-1)
        logits = torch.cosine_similarity(xm.float(), torch.cat([yq[None], negs]).float(), dim=-1) / m.logit_temp
        logits[1:][same] = float("-inf")
        rows = logits.transpose(0, 2).reshape(-1, logits.shape[0])
        ce = F.cross_entropy(rows, rows.new_zeros(rows.shape[0], dtype=torch.long), reduction="sum")
        n = rows.shape[0]
        loss = ce + 0.1 * ((q.num_vars * q.groups - pp) / (q.num_vars * q.groups)) * n + 10.0 * fpen * n
        return loss, xin, cp

    def step(self, audio, mask, neg):
        features = self.frontend(audio)
        B, T, C = features.shape
        xin = features.clone()
        xin[mask] = self.m.mask_emb
        x = self.encoder(xin)
        loss, _, cp = self.head(features, x, mask, neg)
        loss.backward()
        float(loss), float(cp)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--B", type=int, default=24)
    ap.add_argument("--seconds", type=float, default=14.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wav2vec.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = w2v.Wav2Vec(frontend_params=FE, front_bias=False, quantize_input=False, quantize_targets=True,
                        input_size=128, enc_hidden_size=512, enc_layers=4, enc_dropout=0.0, enc_proj_size=512,
                        num_negatives=100).to(dev)
    crit = w2v.ConstrastiveCriterion(infonce=True, loss_weights=[0.1, 10.0],
                                     log_keys=["prob_perplexity", "code_perplexity", "temp"])
    ref = TorchRef(model)
    audio = 0.3 * torch.randn(a.B, int(a.seconds * 16000), device=dev)
    T = model.frontend.output_length(audio.shape[1])

    def engine(precision, parts=False):
        model.set_precision(precision)
        model.zero_grad(set_to_none=True)
        if parts:                                  # front end + encoder alone, forward and backward
            f = model.frontend(audio)
            x, _ = model.encoder(f)
            (f.sum() + x.sum()).backward()
            return
        np.random.seed(1)
        torch.manual_seed(1)
        loss, _, log = crit(model, audio)
        loss.backward()

    def torch_arm(parts=False):
        ref.zero_grad(set_to_none=True)
        if parts:
            f = ref.frontend(audio)
            x = ref.encoder(f)
            (f.sum() + x.sum()).backward()
            return
        np.random.seed(1)
        torch.manual_seed(1)
        mask = torch.from_numpy(w2v.compute_mask_indices((a.B, T), None, 0.15, 10, "static", 0.0, min_masks=2,
                                                         min_space=1)).to(dev)
        M = int(mask[0].sum())
        neg = w2v.sample_negative_indices(a.B, M, 100).to(dev)
        ref.step(audio, mask, neg)

    arms = {"engine_bf16": (lambda: engine("bf16"), lambda: engine("bf16", True)),
            "engine_fp32": (lambda: engine("fp32"), lambda: engine("fp32", True)),
            "torch_cudnn": (torch_arm, lambda: torch_arm(True))}
    for full, part in arms.values():               # warm-up
        full(), part(), full(), part()
    times = {k: dict(step=[], frontend_encoder=[]) for k in arms}
    for _ in range(a.rounds):
        for k, (full, part) in arms.items():
            times[k]["step"].append(timed(full))
            times[k]["frontend_encoder"].append(timed(part))
    out = dict(card=card(), B=a.B, seconds=a.seconds, frames=T, rounds=a.rounds)
    for k, d in times.items():
        st, fe = median(d["step"]), median(d["frontend_encoder"])
        out[k] = dict(step_ms=st, frontend_encoder_ms=fe, head_ms=round(st - fe, 3))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
