"""Wav2vec pre-training on the GPU: every w2v.cu stage teacher-forced against fp64 (tests/wav2vec_oracle.py), the full
fp32-mode step against the reference (tests/golden/wav2vec_tiny.npz) with its spans, negatives and Gumbel noise replayed,
eval mode, bf16 mode, bitwise repeatability, the single readback per criterion call, cli/pretrain_wav2vec.py's full
shape, features_only and a few optimizer steps."""
import os
import warnings

import numpy as np
import pytest
import torch

from tests import wav2vec_oracle as wo
from tests.test_wav2vec_host import CONFIGS, audio, golden, recorded_noise, sample, seeded

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
f64 = torch.float64
CLI_FE = [(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ---- kernels, teacher-forced ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,G,V,vd", [(300, 2, 320, 64), (37, 3, 20, 5)])
def test_quantizer_against_fp64(N, G, V, vd):
    from edgedict_b200 import functional as Fn
    g = torch.Generator().manual_seed(N)
    logits = (3 * torch.randn(N, G * V, generator=g)).to(dev).requires_grad_()
    noise = -torch.empty(N, G * V).exponential_(generator=g).log().to(dev)
    vars = torch.rand(1, G * V, vd, generator=g).to(dev).requires_grad_()
    tau = 1.7
    q, pp, cp, k = Fn.W2VQuantize.apply(logits, vars, noise, G, tau)
    s = torch.softmax((logits.detach() + noise).view(N, G, V) / tau, -1)
    # k: the first maximum of the engine's own s; st and q bit for bit from it
    lq, pq, cq, kq, st = wo.quantize(logits.detach().double().cpu(), vars.detach()[0].double().cpu(),
                                     noise.double().cpu(), G, tau)
    assert torch.equal(k.cpu().long(), kq), "hard indices"
    sk = s.gather(-1, k.long()[..., None])[..., 0]
    st32 = (1 - sk) + sk
    want_q = st32[..., None] * vars.detach()[0].view(G, V, vd)[torch.arange(G, device=dev), k.long()]
    assert torch.equal(q.view(N, G, vd), want_q), "q = st * vars[k] exactly"
    assert abs(float(pp.detach()) - float(pq)) < 1e-5 * float(pq) and abs(float(cp) - float(cq)) < 1e-6 * float(cq)
    R = torch.randn(N, G * vd, generator=g).to(dev)
    (((q * R).sum()) + 3.0 * pp).backward()
    L = logits.detach().double().cpu().requires_grad_()
    Vv = vars.detach()[0].double().cpu().requires_grad_()
    q2, pp2, _, _, _ = wo.quantize(L, Vv, noise.double().cpu(), G, tau)
    ((q2 * R.double().cpu()).sum() + 3.0 * pp2).backward()
    assert rel(logits.grad, L.grad) < 1e-4
    assert rel(vars.grad[0], Vv.grad) < 1e-5


def test_quantizer_eval_is_the_codebook_row():
    from edgedict_b200 import functional as Fn
    g = torch.Generator().manual_seed(5)
    N, G, V, vd = 50, 2, 32, 8
    logits = torch.randn(N, G * V, generator=g).to(dev)
    vars = torch.rand(1, G * V, vd, generator=g).to(dev)
    q, _, _, k = Fn.W2VQuantize.apply(logits, vars, None, G, 2.0)
    k0 = logits.view(N, G, V).argmax(-1)
    assert torch.equal(k.long(), k0)
    assert torch.equal(q.view(N, G, vd), vars[0].view(G, V, vd)[torch.arange(G, device=dev), k0])


@pytest.mark.parametrize("B,M,D,K", [(3, 50, 128, 100), (2, 70, 40, 9), (1, 300, 64, 30)])
def test_logits_against_fp64(B, M, D, K):
    from edgedict_b200 import functional as Fn
    g = torch.Generator().manual_seed(M)
    xp = torch.randn(B, M, D, generator=g)
    yp = torch.randn(B, M, D, generator=g)
    yp[0, 5] = yp[0, 3]                                   # duplicate rows: -inf both ways
    yp[B - 1, 7] = yp[B - 1, 2]
    xp[0, 1] *= 1e-10                                     # clamped norms
    yp[0, 9] *= 1e-10
    neg = torch.randint(0, M, (B, M, K), generator=g)
    neg[0, 3, :4] = 5
    neg[0, 5, 0] = 3
    neg[B - 1, 2, -1] = 7
    neg[0, 0, :] = 9                                      # one index repeated K times
    xg, yg = xp.to(dev).requires_grad_(), yp.to(dev).requires_grad_()
    out = Fn.W2VLogits.apply(xg, yg, neg.to(dev, torch.int32), 0.1)
    X, Y = xp.double().requires_grad_(), yp.double().requires_grad_()
    want = wo.contrastive_logits(X, Y, neg, 0.1)
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(out).cpu(), fin)
    assert int((~fin).sum()) >= 6
    assert float((out.cpu().double()[fin] - want[fin]).abs().max()) < 1e-5 / 0.1
    R = torch.randn(out.shape, generator=g).double()
    R = torch.where(fin, R, torch.zeros_like(R))
    (out * R.to(dev).float()).sum().backward()
    (torch.where(fin, want, torch.zeros_like(want)) * R).sum().backward()
    assert rel(xg.grad, X.grad) < 2e-5
    assert rel(yg.grad, Y.grad) < 2e-5


def test_cross_entropy_against_fp64():
    from edgedict_b200 import functional as Fn
    g = torch.Generator().manual_seed(9)
    C, B, M = 101, 4, 33
    lo = 5 * torch.randn(C, B, M, generator=g)
    lo[3:7, 1, 2] = -float("inf")
    lo[:, 2, 5] = 0.25                                    # all equal: argmax and argmin are 0, not correct
    lo[0, 0, :5] = 100.0
    x = lo.to(dev).requires_grad_()
    loss, correct = Fn.W2VCrossEntropy.apply(x)
    X = lo.double().requires_grad_()
    want, wc = wo.cross_entropy(X)
    assert int(correct) == wc
    assert abs(float(loss) - float(want)) < 1e-5 * float(want)
    (2.5 * loss).backward()
    (2.5 * want).backward()
    assert rel(x.grad, X.grad) < 1e-5


def test_mask_and_gathers():
    from edgedict_b200 import functional as Fn
    g = torch.Generator().manual_seed(2)
    B, T, D, M = 3, 40, 24, 9
    mask = np.zeros((B, T), bool)
    for b in range(B):
        mask[b, np.sort(np.random.RandomState(b).choice(T, M, replace=False))] = True
    idx = wo.frames(mask)
    inv = torch.full((B, T), -1, dtype=torch.int32)
    for b in range(B):
        inv[b, idx[b]] = torch.arange(M, dtype=torch.int32)
    x = torch.randn(B, T, D, generator=g).to(dev).requires_grad_()
    emb = torch.rand(D, generator=g).to(dev).requires_grad_()
    idd, ivd = idx.to(dev, torch.int32), inv.to(dev)
    out = Fn.W2VMask.apply(x, emb, idd, ivd)
    want = x.detach().clone()
    want[torch.as_tensor(mask, device=dev)] = emb.detach()
    assert torch.equal(out, want)
    y = Fn.W2VGather.apply(x, idd, ivd)
    assert torch.equal(y, x.detach()[torch.as_tensor(mask, device=dev)].view(B, M, D))
    R1, R2 = torch.randn(B, T, D, generator=g).to(dev), torch.randn(B, M, D, generator=g).to(dev)
    ((out * R1).sum() + (y * R2).sum() + 4.0 * Fn.W2VSqMean.apply(x)).backward()
    mk = torch.as_tensor(mask, device=dev)[..., None]
    dx = torch.where(mk, torch.zeros_like(R1), R1)
    dx[mk[..., 0]] += R2.view(-1, D)
    Xd = x.detach().double()
    dx = dx.double() + 4.0 * 2 * Xd / Xd.numel()
    assert rel(x.grad, dx) < 1e-6
    assert rel(emb.grad, R1.double()[mk[..., 0]].sum(0)) < 1e-6
    assert abs(float(Fn.W2VSqMean.apply(x)) - float(Xd.pow(2).mean())) < 1e-6 * float(Xd.pow(2).mean())


# ---- the full step against the reference --------------------------------------------------------------------------
def replay(tag, z, model, crit, eval_=False):
    """One criterion call with the fixture's seeds and recorded Gumbel noise (the one test hook)."""
    from edgedict_b200.rnnt import wav2vec as w2v
    pre = "cli.eval." if eval_ else tag + "."
    seed = int(z[tag + ".seed"])
    noises = [] if eval_ else [n.to(dev) for n in recorded_noise(z, pre)]
    x = audio(z).to(dev)
    real = w2v.gumbel_noise

    def recorded(logits):
        n = noises.pop(0)
        assert n.shape == logits.shape
        return n
    w2v.gumbel_noise = recorded
    try:
        np.random.seed(seed + (1 if eval_ else 0))
        torch.manual_seed(seed + (2000 if eval_ else 1000))
        res = {}
        h = model.register_forward_hook(lambda m, i, o: res.update(o))
        out = crit(model, x)
        h.remove()
    finally:
        w2v.gumbel_noise = real
    assert not noises
    return out, res


def criterion(z, tag):
    from edgedict_b200.rnnt.wav2vec import ConstrastiveCriterion
    return ConstrastiveCriterion(infonce=True, loss_weights=list(z[tag + ".weights"]),
                                 log_keys=[str(k) for k in z["log_keys"]])


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_fp32_step_matches_the_reference(tag):
    z = golden()
    model = seeded(tag, z).to(dev)
    (loss, ss, log), res = replay(tag, z, model, criterion(z, tag))
    want = torch.from_numpy(z[tag + ".logits"])
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(res["x"]).cpu(), fin)
    assert float((res["x"].detach().cpu()[fin] - want[fin]).abs().max()) < 2e-3
    names = [str(k) for k in z[tag + ".log_names"]]
    assert list(log) == names
    for k, v in zip(names, z[tag + ".log_values"]):
        if k in ("correct", "count", "ntokens", "sample_size"):
            assert log[k] == int(v), k
        else:
            assert abs(log[k] - v) <= 2e-4 * max(1.0, abs(v)), (k, log[k], v)
    assert abs(float(loss) - float(z[tag + ".loss"])) <= 2e-4 * abs(float(z[tag + ".loss"]))
    loss.backward()
    no_grad = {str(k) for k in z[tag + ".no_grad"]}
    for k, p in model.named_parameters():
        if k in no_grad:
            assert p.grad is None, k
            continue
        assert rel(sample(p.grad.detach().cpu()), torch.from_numpy(z[tag + ".grad." + k])) < 2e-3, k


def test_eval_step_matches_the_reference():
    z = golden()
    model = seeded("cli", z).to(dev).eval()
    with torch.no_grad():
        (loss, ss, log), res = replay("cli", z, model, criterion(z, "cli"), eval_=True)
    assert torch.equal(res["targets"].cpu(), torch.from_numpy(z["cli.eval.targets"]))
    want = torch.from_numpy(z["cli.eval.logits"])
    fin = torch.isfinite(want)
    assert float((res["x"].cpu()[fin] - want[fin]).abs().max()) < 2e-3
    for k, v in zip([str(k) for k in z["cli.eval.log_names"]], z["cli.eval.log_values"]):
        assert abs(log[k] - v) <= 2e-4 * max(1.0, abs(v)), (k, log[k], v)


# Measured on one H100 80GB HBM3 at a 700 W power limit: loss rel 6.1e-6, worst gradient-norm rel 6.0e-3.
def test_bf16_step_within_bars():
    z = golden()
    ref = seeded("cli", z).to(dev)
    (l32, _, _), _ = replay("cli", z, ref, criterion(z, "cli"))
    l32.backward()
    model = seeded("cli", z).to(dev)
    model.set_precision("bf16")
    (l16, _, log), _ = replay("cli", z, model, criterion(z, "cli"))
    l16.backward()
    r = abs(float(l16) - float(l32)) / abs(float(l32))
    worst = 0.0
    for (k, p), (_, q) in zip(model.named_parameters(), ref.named_parameters()):
        if q.grad is not None:
            worst = max(worst, abs(float(p.grad.norm()) - float(q.grad.norm())) / (float(q.grad.norm()) + 1e-12))
    print("bf16: loss rel %.2e, worst gradient-norm rel %.2e" % (r, worst))
    assert r < 1e-3 and worst < 3e-2


def test_step_is_bitwise_repeatable():
    z = golden()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        outs = []
        for _ in range(2):
            model = seeded("qin", z).to(dev)
            torch.manual_seed(5)
            np.random.seed(5)
            loss, _, log = criterion(z, "qin")(model, audio(z).to(dev))
            loss.backward()
            outs.append((loss.detach().clone(), log, [p.grad.clone() for p in model.parameters() if p.grad is not None]))
        assert torch.equal(outs[0][0], outs[1][0]) and outs[0][1] == outs[1][1]
        for a, b in zip(outs[0][2], outs[1][2]):
            assert torch.equal(a, b)
    finally:
        torch.use_deterministic_algorithms(prev)


def test_one_readback_per_criterion_call():
    z = golden()
    model = seeded("cli", z).to(dev)
    crit = criterion(z, "cli")
    x = audio(z).to(dev)
    crit(model, x)                                        # warm-up: library load, pinned pool
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            loss, _, _ = crit(model, x)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    syncs = [str(r.message) for r in rec if "synchroniz" in str(r.message).lower()]
    assert len(syncs) == 1, syncs


def test_cli_shape_against_the_oracle():
    """cli/pretrain_wav2vec.py's model (4 x 512 LSTM, K = 100, G = 2, V = 320) on 24 utterances of 14 s: finite, and the
    head's logits, loss and logging values against the fp64 restatement fed the engine's own front-end and encoder
    outputs, spans, negatives and noise."""
    from edgedict_b200.rnnt import wav2vec as w2v
    torch.manual_seed(0)
    model = w2v.Wav2Vec(frontend_params=CLI_FE, front_bias=False, quantize_input=False, quantize_targets=True,
                        input_size=128, enc_hidden_size=512, enc_layers=4, enc_dropout=0.1, enc_proj_size=512,
                        num_negatives=100).to(dev)
    crit = w2v.ConstrastiveCriterion(infonce=True, loss_weights=[0.1, 10.0],
                                     log_keys=["prob_perplexity", "code_perplexity", "temp"])
    x = 0.3 * torch.randn(24, 14 * 16000, device=dev)
    got, noises = {}, []
    real = w2v.gumbel_noise

    def keep(logits):
        n = real(logits)
        noises.append(n)
        return n
    hooks = [model.frontend.register_forward_hook(lambda m, i, o: got.__setitem__("fe", o.detach())),
             model.encoder.register_forward_hook(lambda m, i, o: got.__setitem__("enc", o[0].detach())),
             model.register_forward_hook(lambda m, i, o: got.__setitem__("x", o["x"].detach()))]
    w2v.gumbel_noise = keep
    try:
        np.random.seed(3)
        torch.manual_seed(4)
        loss, ss, log = crit(model, x)
    finally:
        w2v.gumbel_noise = real
        for h in hooks:
            h.remove()
    loss.backward()
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)
    B, T = 24, got["fe"].shape[1]
    np.random.seed(3)
    mask = w2v.compute_mask_indices((B, T), None, 0.15, 10, "static", 0.0, min_masks=2, min_space=1)
    torch.manual_seed(4)
    M = int(mask[0].sum())
    neg = w2v.sample_negative_indices(B, M, 100)
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    idx = wo.frames(mask)
    fe = got["fe"].double().cpu()
    logits, want_loss, want = wo.head(sd, wo.gather(fe, idx), wo.gather(got["enc"].double().cpu(), idx),
                                      fe.pow(2).mean(), neg, noises[0].double().cpu(), 2, model.quantizer.curr_temp,
                                      0.1, [0.1, 10.0])
    fin = torch.isfinite(logits)
    assert torch.equal(torch.isfinite(got["x"]).cpu(), fin)
    assert float((got["x"].cpu().double()[fin] - logits[fin]).abs().max()) < 1e-3
    assert abs(float(loss) - float(want_loss)) < 1e-4 * float(want_loss)
    for k in ("loss_0", "loss_1", "loss_2", "prob_perplexity", "code_perplexity"):
        assert abs(log[k] - float(want[k])) < 1e-4 * max(1.0, abs(float(want[k]))), k
    assert abs(log["correct"] - want["correct"]) <= 2


def test_features_only_and_gru():
    z = golden()
    for tag in ("cli", "gru"):
        model = seeded(tag, z).to(dev)
        x = audio(z).to(dev)
        out = model(x, mask=False, features_only=True)
        enc, _ = model.encoder(model.frontend(x))
        assert torch.equal(out["x"], enc) and out["padding_mask"] is None
        np.random.seed(1)
        out2 = model(x, features_only=True)
        assert out2["x"].shape == enc.shape and not torch.equal(out2["x"], enc)


def test_flat_adamw_lowers_the_loss():
    from edgedict_b200.optim import FlatAdamW
    z = golden()
    model = seeded("cli", z).to(dev)
    opt = FlatAdamW(model, lr=3e-3)
    crit = criterion(z, "cli")
    x = audio(z).to(dev)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        np.random.seed(0)
        torch.manual_seed(0)
        loss, _, _ = crit(model, x)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0], losses
