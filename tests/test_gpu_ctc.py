"""CTC on the engine (csrc/ctc.cu, edgedict_b200.ctc, CTCEncoder) against fp64 references:

* loss, per-utterance costs and the gradient for log_probs against torch.nn.functional.ctc_loss in fp64 on the CPU, over
  a matrix of batch sizes, lengths, vocabularies, target layouts, blanks, reductions and zero_infinity; repeated labels
  with just-feasible and infeasible lengths; the transposed [B, T, V] view and the unbatched (T, C) form;
* bitwise repeatability and batch independence of costs and gradients;
* the row log-softmax forward and backward per element against fp64, within a rounding-error bound;
* CTCEncoder against the fp64 oracle (oracle/ctc.py) and the reference's fixture (tests/golden/ctc_tiny.npz), in fp32 and
  bf16 mode; greedy_decode including NaN and tied rows.

Bars: costs relative COST_REL, gradients absolute GRAD_ABS (after the upstream factor).  They started from the RNN-T loss
kernels' bars (1e-5, 2e-4) and sit about 14x above the worst cases measured on an H100 (7.1e-8 and 1.44e-7: the lattice
runs in fp64); every test prints its measured worst case ("[ctc] ..." lines; DESIGN.md section 2 records them)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_oracle_ctc import load_ctc_tiny
from tests.util import rel_err

pytestmark = pytest.mark.gpu

f64 = torch.float64
COST_REL = 1e-6
GRAD_ABS = 2e-6
U = 2.0 ** -24


def _note(what, value, bar):
    print("  [ctc] %-58s worst %.3g  bar %.3g  (%.3f of the bar)" % (what, value, bar, value / bar))


def _problem(B, T, V, S, seed, blank=0, ragged=True, short_inputs=True):
    g = torch.Generator().manual_seed(seed)
    lp = (torch.randn(T, B, V, generator=g) * 2).log_softmax(-1)
    lab = torch.randint(0, V - 1, (B, S), generator=g)
    lab = lab + (lab >= blank).long()                    # labels in [0, V) without the blank
    tl = torch.full((B,), S, dtype=torch.long)
    il = torch.full((B,), T, dtype=torch.long)
    if ragged and B > 1:
        tl[1:] = torch.randint(0, S + 1, (B - 1,), generator=g)
        if short_inputs:
            il[1:] = torch.randint(1, T + 1, (B - 1,), generator=g)
    return lp, lab, il, tl


def _cmp(got, want, rel=False):
    """NaN where the reference is NaN, equal infinities, and the worst abs (or relative) error elsewhere."""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    inf = torch.isinf(want)
    assert torch.equal(got[inf], want[inf])
    fin = torch.isfinite(want)
    if not bool(fin.any()):
        return 0.0
    err = (got[fin] - want[fin]).abs()
    if rel:
        err = err / want[fin].abs().clamp_min(1e-30)
    return float(err.max())


def _run(lp, targets, il, tl, blank, reduction, zero_inf, go, layout="tnv"):
    """(engine loss, grad as [T, N, V]) and (reference loss, grad) for one call."""
    from edgedict_b200.ctc import ctc_loss
    lr = lp.double().requires_grad_()
    ref = F.ctc_loss(lr, targets.long(), il, tl, blank, reduction, zero_inf)
    ref.backward(go.double())
    if layout == "btv":                                  # CTCEncoder's output, passed as .transpose(0, 1)
        le = lp.transpose(0, 1).contiguous().cuda().requires_grad_()
        got = ctc_loss(le.transpose(0, 1), targets.cuda(), il, tl, blank, reduction, zero_inf)
        got.backward(go.float().cuda())
        return got, le.grad.transpose(0, 1), ref, lr.grad
    le = lp.cuda().requires_grad_()
    got = ctc_loss(le, targets.cuda(), il, tl, blank, reduction, zero_inf)
    got.backward(go.float().cuda())
    return got, le.grad, ref, lr.grad


def _concat(lab, tl):
    return torch.cat([lab[b, :int(n)] for b, n in enumerate(tl)])


# (B, T, V, S, seed, blank, layout, short inputs)
CASES = {
    "T1_S0": (1, 1, 2, 0, 1, 0, "padded", False),
    "T1_S1": (1, 1, 3, 1, 2, 0, "padded", False),
    "tiny_concat": (3, 17, 11, 6, 3, 0, "concat", True),
    "tiny_blank_last": (3, 17, 11, 6, 4, 10, "padded", True),
    "B64": (64, 60, 29, 12, 5, 0, "padded", True),
    "B64_concat_blank_last": (64, 45, 7, 9, 6, 6, "concat", True),
    "odd_V1023": (8, 200, 1023, 80, 7, 0, "concat", True),
    "V2_repeats": (3, 300, 2, 100, 8, 0, "padded", True),
    "S_above_T": (5, 20, 6, 15, 9, 0, "padded", False),
    "T1000_V1024_S256": (4, 1000, 1024, 256, 10, 0, "padded", True),
    "btv_view": (6, 150, 97, 30, 11, 0, "btv", True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_ctc_loss_matches_torch_fp64(case):
    B, T, V, S, seed, blank, layout, short = CASES[case]
    lp, lab, il, tl = _problem(B, T, V, S, seed, blank, short_inputs=short)
    targets = _concat(lab, tl) if layout == "concat" else lab
    g = torch.Generator().manual_seed(seed + 100)
    worst_c = worst_g = 0.0
    for reduction in ("none", "mean", "sum"):
        for zero_inf in (False, True):
            go = torch.rand(B, generator=g) + 0.5 if reduction == "none" else torch.tensor(1.3)
            got, dg, ref, dr = _run(lp, targets, il, tl, blank, reduction, zero_inf, go,
                                    "btv" if layout == "btv" else "tnv")
            worst_c = max(worst_c, _cmp(got, ref, rel=True))
            worst_g = max(worst_g, _cmp(dg, dr))
    _note("%s costs (rel)" % case, worst_c, COST_REL)
    _note("%s gradient (abs)" % case, worst_g, GRAD_ABS)
    assert worst_c <= COST_REL and worst_g <= GRAD_ABS


@pytest.mark.parametrize("reduction", ["none", "mean", "sum"])
def test_ctc_loss_unbatched(reduction):
    lp, lab, il, tl = _problem(1, 40, 13, 9, 21)
    go = torch.tensor(0.7)
    from edgedict_b200.ctc import CTCLoss
    lr = lp[:, 0].double().requires_grad_()
    ref = F.ctc_loss(lr, lab[0], il[0], tl[0], reduction=reduction)
    ref.backward(go.double())
    le = lp[:, 0].cuda().requires_grad_()
    got = CTCLoss(reduction=reduction)(le, lab[0].cuda(), int(il[0]), torch.tensor(int(tl[0])))
    got.backward(go.cuda())
    assert got.shape == ref.shape
    ec, eg = _cmp(got, ref, rel=True), _cmp(le.grad, lr.grad)
    _note("unbatched %s" % reduction, max(ec / COST_REL, eg / GRAD_ABS), 1.0)
    assert ec <= COST_REL and eg <= GRAD_ABS


@pytest.mark.parametrize("T", [7, 8, 9])
@pytest.mark.parametrize("zero_inf", [False, True])
def test_repeated_labels_feasibility(T, zero_inf):
    """l = (a, a, a, b, b): 5 labels and 3 adjacent repeats need T >= 8; at T = 7 no alignment exists (+inf)."""
    V = 6
    g = torch.Generator().manual_seed(T)
    lp = torch.randn(T, 2, V, generator=g).log_softmax(-1)
    targets = torch.tensor([[2, 2, 2, 4, 4], [3, 3, 1, 1, 0]])
    il, tl = torch.tensor([T, T]), torch.tensor([5, 4])
    got, dg, ref, dr = _run(lp, targets, il, tl, 0, "none", zero_inf, torch.tensor([1.0, 0.5]))
    assert bool(torch.isinf(ref[0])) == (T < 8 and not zero_inf)
    ec, eg = _cmp(got, ref, rel=True), _cmp(dg, dr)
    _note("repeats T=%d zero_infinity=%s" % (T, zero_inf), max(ec / COST_REL, eg / GRAD_ABS), 1.0)
    assert ec <= COST_REL and eg <= GRAD_ABS


def test_out_of_range_labels_have_no_alignment():
    """A label outside [0, V) is never read: the utterance gets +inf, the others are unaffected."""
    from edgedict_b200.ctc import ctc_loss
    lp, lab, il, tl = _problem(3, 30, 9, 5, 31, ragged=False)
    bad = lab.clone()
    bad[1, 2] = 9
    bad[2, 0] = -5
    costs = ctc_loss(lp.cuda(), bad.cuda(), il, tl, reduction="none").cpu()
    ref = F.ctc_loss(lp.double(), lab, il, tl, reduction="none")
    assert torch.isinf(costs[1:]).all() and rel_err(costs[0], ref[0]) <= COST_REL


def _engine_costs_grads(lp, lab, il, tl, go, layout="tnv"):
    from edgedict_b200.ctc import ctc_loss
    le = lp.cuda().requires_grad_()
    c = ctc_loss(le, lab.cuda(), il, tl, reduction="none")
    c.backward(go.cuda())
    return c.detach().cpu(), le.grad.cpu()


def test_costs_and_gradients_are_bitwise_repeatable_and_batch_independent():
    lp, lab, il, tl = _problem(5, 400, 300, 60, 41)
    go = torch.rand(5, generator=torch.Generator().manual_seed(1)) + 0.5
    c1, g1 = _engine_costs_grads(lp, lab, il, tl, go)
    c2, g2 = _engine_costs_grads(lp, lab, il, tl, go)
    assert torch.equal(c1, c2) and torch.equal(g1, g2)
    for b in (0, 3):                                     # utterance b alone, then in another batch
        c, gr = _engine_costs_grads(lp[:, b:b + 1].contiguous(), lab[b:b + 1], il[b:b + 1], tl[b:b + 1], go[b:b + 1])
        assert torch.equal(c[0], c1[b]) and torch.equal(gr[:, 0], g1[:, b])
        perm = [b, 4 - b if b != 2 else 1]
        c, gr = _engine_costs_grads(lp[:, perm].contiguous(), lab[perm], il[perm], tl[perm], go[perm])
        assert torch.equal(c[0], c1[b]) and torch.equal(gr[:, 0], g1[:, b])


def test_ctc_loss_runs_under_deterministic_algorithms():
    from edgedict_b200.ctc import ctc_loss
    lp, lab, il, tl = _problem(2, 30, 8, 5, 51)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        le = lp.cuda().requires_grad_()
        ctc_loss(le, lab.cuda(), il, tl).backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.isfinite(le.grad).all()


# ---- row log-softmax --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,V", [(1, 1), (7, 2), (33, 1023), (500, 1024), (3, 5000)])
def test_log_softmax_forward_and_backward_per_element(rows, V):
    """Bound per element (u = 2^-24): forward u (|x - m| + (V + 2) + 2 |log s| + |y|), backward
    u (|g| + |dx| + exp(y) (V + 3) sum|g|), both doubled; the inputs of the fp64 restatement are the kernel's own fp32
    inputs."""
    from edgedict_b200 import ops
    g = torch.Generator().manual_seed(rows * 7 + V)
    x = torch.randn(rows, V, generator=g) * 4
    y = ops.log_softmax_fwd(x.cuda()).cpu()
    x64 = x.double()
    m = x64.max(-1, keepdim=True).values
    ls = torch.log(torch.exp(x64 - m).sum(-1, keepdim=True))
    y64 = x64 - m - ls
    bar = 2 * U * ((x64 - m).abs() + (V + 2) + 2 * ls.abs() + y64.abs())
    ef = float(((y.double() - y64).abs() / bar).max())
    dy = torch.randn(rows, V, generator=g)
    dx = ops.log_softmax_bwd(dy.cuda(), y.cuda()).cpu()
    g64, ey = dy.double(), torch.exp(y.double())
    dx64 = g64 - ey * g64.sum(-1, keepdim=True)
    bar_b = 2 * U * (g64.abs() + dx64.abs() + ey * (V + 3) * g64.abs().sum(-1, keepdim=True))
    eb = float(((dx.double() - dx64).abs() / bar_b).max())
    _note("log_softmax rows=%d V=%d fwd err/bar" % (rows, V), ef, 1.0)
    _note("log_softmax rows=%d V=%d bwd err/bar" % (rows, V), eb, 1.0)
    assert ef <= 1.0 and eb <= 1.0
    assert torch.equal(ops.log_softmax_fwd(x.cuda()).cpu(), y)


# ---- greedy decode ----------------------------------------------------------------------------------------------------
def _decode(lp, xlen, blank):
    from edgedict_b200 import ops
    B, T = lp.shape[0], lp.shape[1]
    out = ops.ctc_greedy(lp.cuda(), torch.as_tensor(xlen, dtype=torch.int32).clamp(0, T).cuda(), blank).cpu()
    ids, counts = out[:B * T].view(B, T), out[B * T:B * T + B]
    return [ids[b, :int(counts[b])].numpy() for b in range(B)], out[B * T + B:].view(torch.float32)


@pytest.mark.parametrize("blank", [0, 36])
def test_greedy_kernel_matches_reference_decode_with_nan_and_ties(blank):
    from oracle.ctc import greedy_from_logprobs
    B, T, V = 4, 600, 37
    g = torch.Generator().manual_seed(61 + blank)
    lp = (torch.randn(B, T, V, generator=g) * 3).log_softmax(-1)
    lp[:, ::3, blank] += 6.0                              # plenty of blanks
    lp[0, 240:275] = lp[0, 240]                          # one argmax repeated across the 256-frame chunk boundary
    lp[0, 100, 5] = lp[0, 100, 9] = lp[0, 100].max() + 1  # exact ties: the lowest id wins
    lp[2, 300, [7, 30]] = lp[2, 300].max() + 1
    lp[1, 10, 3] = float("nan")                           # NaN wins the argmax
    lp[1, 11, [2, 7]] = float("nan")
    lp[3, 50:60] = 0.0                                    # all-equal rows: id 0
    xlen = [600, 513, 900, 257]
    ids, nscore = _decode(lp, xlen, blank)
    want_ids, want_score = greedy_from_logprobs(lp, xlen, blank)
    for got, want in zip(ids, want_ids):
        assert got.tolist() == want.tolist()
    e = _cmp(nscore, want_score, rel=True)
    _note("greedy score blank=%d (rel)" % blank, e, 1e-5)
    assert e <= 1e-5
    ids0, _ = _decode(lp, [0, 1, 0, 0], blank)
    first = int(lp[1, 0].argmax())
    assert [i.tolist() for i in ids0] == [[], [] if first == blank else [first], [], []]


# ---- CTCEncoder -------------------------------------------------------------------------------------------------------
def _engine_model(cfg, sd, precision="fp32"):
    from edgedict_b200.rnnt.models import CTCEncoder
    m = CTCEncoder(**cfg)
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    return m.cuda().set_precision(precision)


def test_ctc_encoder_reproduces_the_reference_fixture():
    z, cfg, sd = load_ctc_tiny()
    m = _engine_model(cfg, sd).eval()
    xs = torch.as_tensor(z["xs"]).cuda()
    with torch.no_grad():
        lp = m(xs)
    e = rel_err(lp.cpu(), z["logprobs"])
    ids, nlp = m.greedy_decode(xs, torch.as_tensor(z["xlen"]))
    for got, row, n in zip(ids, z["greedy_ids"], z["greedy_counts"]):
        assert got.dtype == np.int64 and got.tolist() == row[:n].tolist()
    es = rel_err(nlp.cpu(), z["greedy_nlp"])
    _note("fixture log-probs (rel)", e, 2e-5)
    _note("fixture greedy score (rel)", es, 1e-5)
    assert e <= 2e-5 and es <= 1e-5
    with torch.no_grad():
        m.tovocab[0].bias[0] += 100.0
    ids, nlp = m.greedy_decode(xs, z["xlen"].tolist())
    assert all(len(i) == 0 for i in ids) and torch.equal(nlp.cpu(), torch.as_tensor(z["blank_bias_nlp"]))


TINY = dict(vocab_size=40, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0, proj_size=32)
E6D2 = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0, proj_size=640)


def _norm_err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a.norm() - b.norm()).abs() / (b.norm() + 1e-30))


@pytest.mark.parametrize("precision,dims", [("fp32", "tiny"), ("bf16", "e6d2")])
def test_ctc_encoder_training_step_matches_oracle(precision, dims):
    from edgedict_b200.ctc import CTCLoss
    from edgedict_b200.rnnt.models import CTCEncoder
    from oracle import ctc as oc
    cfg, B, T, S = (TINY, 3, 23, 5) if dims == "tiny" else (E6D2, 2, 200, 20)
    torch.manual_seed(71)
    m = CTCEncoder(**cfg).cuda().set_precision(precision)
    g = torch.Generator().manual_seed(72)
    xs = torch.randn(B, T, cfg["input_size"], generator=g)
    Tp = (T + 1) // 2
    ys = torch.randint(1, cfg["vocab_size"], (B, S), generator=g)
    il, tl = torch.tensor([Tp] + [Tp - 3] * (B - 1)), torch.tensor([S] + [S - 2] * (B - 1))
    sd = {k: v.detach().cpu().double().requires_grad_() for k, v in m.state_dict().items()}
    lr = oc.ctc_encoder_forward(sd, xs.double())
    ref = F.ctc_loss(lr.transpose(0, 1), ys, il, tl)
    ref.backward()
    lp = m(xs.cuda())
    loss = CTCLoss()(lp.transpose(0, 1), ys, il, tl)
    loss.backward()
    el = rel_err(loss.detach().cpu(), ref.detach())
    ef = rel_err(lp.detach().cpu(), lr.detach())
    worst = (0.0, "")
    for k, p in m.named_parameters():
        e = rel_err(p.grad.cpu(), sd[k].grad) if precision == "fp32" else _norm_err(p.grad, sd[k].grad)
        worst = max(worst, (e, k))
    print("  [ctc] CTCEncoder %s %s: loss %.3g, log-probs %.3g, worst gradient %.3g (%s)"
          % (precision, dims, el, ef, worst[0], worst[1]))
    if precision == "fp32":
        assert el < 1e-4 and ef < 1e-4 and worst[0] < 1e-3
    else:
        assert el < 1e-3 and worst[0] < 2e-2
