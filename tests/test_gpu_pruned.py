"""The pruned RNN-T loss on the device against the fp64 oracle (tests/pruned_oracle.py): the simple loss and its
gradients, the band choice on the device's own occupancy, the band-row loss and gradient in fp32 and bf16, the banded
reduction, the full-band identity with the default path and the subset property, and Transducer(prune_range)."""
import math

import numpy as np
import pytest
import torch

from tests import pruned_oracle as po

pytestmark = pytest.mark.gpu
f64 = torch.float64
i32 = torch.int32


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _problem(seed, B, T, U, V, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    am = torch.randn(B, T, V, generator=g) * scale
    lm = torch.randn(B, U, V, generator=g) * scale
    labels = torch.randint(1, V, (B, U - 1), generator=g, dtype=i32)
    xlen = torch.randint(1, T + 1, (B,), generator=g, dtype=i32)
    ylen = torch.randint(0, U, (B,), generator=g, dtype=i32)
    xlen[0], ylen[0] = T, U - 1
    return am, lm, labels, xlen, ylen


def _simple_dev(am, lm, labels, xlen, ylen, blank, weights):
    from edgedict_b200 import functional as Fn
    a = am.cuda().requires_grad_(True)
    l = lm.cuda().requires_grad_(True)
    costs, ws = Fn.SimpleLoss.apply(a, l, labels.cuda(), xlen.cuda(), ylen.cuda(), blank)
    (costs * weights.cuda()).sum().backward()
    return costs.detach(), ws, a.grad, l.grad


@pytest.mark.parametrize("case", ["ragged", "underflow", "no_frames"])
def test_simple_loss_matches_fp64_oracle(case):
    blank = 2
    if case == "ragged":
        am, lm, labels, xlen, ylen = _problem(1, 3, 7, 5, 33)
    elif case == "underflow":
        # row maxima at different tokens, more than 100 apart: exp(am - amax) . exp(lm - lmax) would underflow
        am, lm, labels, xlen, ylen = _problem(2, 2, 6, 4, 40)
        am[:, :, 3] += 150.0
        lm[:, :, 7] += 150.0
    else:
        am, lm, labels, xlen, ylen = _problem(3, 3, 5, 4, 16)
        xlen[1] = 0
    weights = torch.tensor([0.7, -0.3, 1.3][:am.shape[0]])
    costs, _, dam, dlm = _simple_dev(am, lm, labels, xlen, ylen, blank, weights)
    a64, l64 = am.double().requires_grad_(True), lm.double().requires_grad_(True)
    ref = po.simple_costs(a64, l64, labels.long(), xlen, ylen, blank)
    fin = torch.isfinite(ref)
    (ref[fin] * weights.double()[fin]).sum().backward()
    assert torch.equal(torch.isfinite(costs.cpu()), fin)
    # fp32 error model: a sum of ~V * T * U rounded terms of magnitude |cost|
    assert _rel(costs.cpu()[fin], ref.detach()[fin]) < 2e-5
    assert _rel(dam, a64.grad) < 5e-5 and _rel(dlm, l64.grad) < 5e-5, (_rel(dam, a64.grad), _rel(dlm, l64.grad))
    # bitwise repeatable
    c2, _, dam2, dlm2 = _simple_dev(am, lm, labels, xlen, ylen, blank, weights)
    assert torch.equal(c2.view(i32), costs.view(i32)) and torch.equal(dam2, dam) and torch.equal(dlm2, dlm)


def _occ(ws, B, T, U):
    w = ws.view(torch.float32)
    n = B * T * U
    al, be, ll = w[3 * n:4 * n].view(B, T, U), w[4 * n:5 * n].view(B, T, U), w[5 * n:5 * n + B]
    return torch.exp(al + be - ll.view(B, 1, 1)).cpu()


@pytest.mark.parametrize("shape, R", [((3, 9, 6, 20), 3), ((2, 4, 30, 12), 5), ((2, 3, 40, 10), 4), ((4, 50, 20, 24), 8)])
def test_band_choice_is_the_rule_on_the_device_occupancy(shape, R):
    """Exact s_begin of the rule applied to the device's fp32 occupancy; long U with short T reaches the no-path case."""
    from edgedict_b200 import ops
    B, T, U, V = shape
    am, lm, labels, xlen, ylen = _problem(7 + R, B, T, U, V, scale=2.0)
    costs, ws, _, _ = _simple_dev(am, lm, labels, xlen, ylen, 0, torch.ones(B))
    s_begin, nopath = ops.rnnt_band_choice(xlen.cuda(), ylen.cuda(), B, T, U, R, ws)
    occ = _occ(ws, B, T, U)
    for b in range(B):
        Tn, Un = po.lengths(xlen[b], ylen[b], T, U)
        s, np_ = po.band_rule(occ[b, :Tn, :Un], Tn, Un, R)
        assert s_begin[b, :Tn].tolist() == s and bool(nopath[b]) == np_, (b, s_begin[b].tolist(), s)
        assert s_begin[b, Tn:].eq(0).all()
    if shape == (2, 3, 40, 10):
        assert bool(nopath.any())


def _bands(B, T, U, R, xlen, ylen, seed):
    g = torch.Generator().manual_seed(seed)
    s = torch.zeros(B, T, dtype=i32)
    nop = torch.zeros(B, dtype=i32)
    for b in range(B):
        Tn, Un = po.lengths(xlen[b], ylen[b], T, U)
        sb, np_ = po.band_rule(torch.rand(Tn, Un, generator=g), Tn, Un, R)
        s[b, :Tn] = torch.tensor(sb, dtype=i32)
        nop[b] = int(np_)
    return s, nop


@pytest.mark.parametrize("V", [32, 29])
def test_band_loss_kernels_match_fp64_oracle(V):
    """Costs and d logits of band rows in fp32 (in place and not) and bf16 against the fp64 oracle; padding rows zero,
    valid rows sum to ~0."""
    from edgedict_b200 import ops, pruned
    B, T, U, R, blank = 3, 8, 6, 3, 1
    _, _, labels, xlen, ylen = _problem(11, B, T, U, V)
    s, nop = _bands(B, T, U, R, xlen, ylen, 3)
    g = torch.Generator().manual_seed(4)
    logits = torch.randn(B, T, R, V, generator=g) * 2
    x = logits.cuda().requires_grad_(True)
    costs = pruned.rnnt_loss_pruned(x, labels.cuda(), xlen.cuda(), ylen.cuda(), s.cuda(), nop.cuda(), blank,
                                    reduction="none")
    w = torch.tensor([0.5, 1.5, -1.0])
    (costs * w.cuda()).sum().backward()
    x64 = logits.double().requires_grad_(True)
    ref = po.pruned_costs(x64, labels.long(), xlen, ylen, s.tolist(), U, blank)
    (ref * w.double()).sum().backward()
    fin = torch.isfinite(ref.detach())
    assert torch.equal(torch.isfinite(costs.detach()).cpu(), fin)         # +inf exactly where the bands hold no path
    assert _rel(costs.detach().cpu()[fin], ref.detach()[fin]) < 1e-5
    assert _rel(x.grad, x64.grad) < 1e-5
    assert x.grad[nop.cuda().bool()].eq(0).all()
    # padding rows zero, valid rows sum to ~0
    for b in range(B):
        Tn, Un = po.lengths(xlen[b], ylen[b], T, U)
        assert x.grad[b, Tn:].eq(0).all() and x.grad[b, :, min(R, Un):].eq(0).all()
    assert float(x.grad.double().sum(-1).abs().max()) < 1e-5
    # in place and bf16 through the ops entries
    lg = logits.cuda()
    c2, ws = ops.rnnt_band_loss_fwd(lg, labels.cuda(), xlen.cuda(), ylen.cuda(), s.cuda(), nop.cuda(), U, blank)
    gw = w.cuda()
    d16 = ops.rnnt_band_loss_bwd(lg, labels.cuda(), xlen.cuda(), ylen.cuda(), s.cuda(), nop.cuda(), U, blank, ws, gw,
                                 1.0, out_bf16=True)
    ops.rnnt_band_loss_bwd(lg, labels.cuda(), xlen.cuda(), ylen.cuda(), s.cuda(), nop.cuda(), U, blank, ws, gw, 1.0,
                           out=lg)
    assert torch.equal(lg, x.grad) and torch.equal(d16, x.grad.to(torch.bfloat16))


def _joint_inputs(seed, B, T, U, E, D, J, V):
    g = torch.Generator().manual_seed(seed)
    he = torch.randn(B, T, E, generator=g)
    hd = torch.randn(B, U, D, generator=g)
    w1 = torch.randn(J, E + D, generator=g) / math.sqrt(E + D)
    b1 = torch.randn(J, generator=g) * 0.1
    w2 = torch.randn(V, J, generator=g) / math.sqrt(J)
    b2 = torch.randn(V, generator=g) * 0.1
    return [t.cuda() for t in (he, hd, w1, b1, w2, b2)]


def _run(fn, params, *args):
    ps = [p.clone().requires_grad_(True) for p in params]
    loss, costs = fn.apply(*ps, *args)
    loss.backward()
    return costs.detach(), [p.grad for p in ps]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_full_band_is_the_full_loss_bitwise(precision):
    """Transducer(prune_range=R) with R >= max U_b: the band choice gives every frame the whole column and the pruned
    cost is bitwise the default Transducer's (bf16 mode: both through the logits GEMM's statistics epilogue); with the
    simple loss's scale at 0 every shared parameter's gradient agrees within the parity bars."""
    base, inputs = _model()
    pr, _ = _model(prune_range=8)                           # ys has 7 labels: max U_b = 8
    pr.load_state_dict(base.state_dict(), strict=False)
    pr.simple_loss_scale = 0.0
    base.set_precision(precision)
    pr.set_precision(precision)
    _, g_base = _step(base, inputs)
    c_base = base.last_costs.clone()
    _, g_pr = _step(pr, inputs)
    assert torch.equal(pr.last_costs.view(i32), c_base.view(i32)), (pr.last_costs, c_base)
    tol = 1e-4 if precision == "fp32" else 2e-2
    errs = {k: _rel(g_pr[k], g_base[k]) for k in g_base}
    assert max(errs.values()) < tol, errs


@pytest.mark.parametrize("R", [2, 4, 8])
def test_pruned_cost_is_at_least_the_full_cost(R):
    from edgedict_b200 import functional as Fn, ops
    B, T, U, E, D, J, V = 4, 12, 10, 16, 8, 24, 32
    _, _, labels, xlen, ylen = _problem(30 + R, B, T, U, V)
    params = _joint_inputs(31 + R, B, T, U, E, D, J, V)
    lab, xl, yl = labels.cuda(), xlen.cuda(), ylen.cuda()
    c_full, _ = _run(Fn.JointLoss, params, lab, xl, yl, 0, "fp32")
    am, lm, _, _, _ = _problem(32 + R, B, T, U, V)
    _, ws, _, _ = _simple_dev(am, lm, labels, xlen, ylen, 0, torch.ones(B))
    s, nop = ops.rnnt_band_choice(xl, yl, B, T, U, R, ws)
    c_pr, _ = _run(Fn.PrunedJointLoss, params, s, nop, R, lab, xl, yl, 0, "fp32")
    slack = c_full.abs() * 2.0 ** -23
    assert bool((c_pr >= c_full - slack).all()), (c_pr, c_full)


@pytest.mark.parametrize("bf16", [False, True])
def test_banded_reduction(bf16):
    """dep / ddp against an fp64 restatement, and bitwise independent of the other utterances and of padding."""
    from edgedict_b200 import ops
    B, T, U, R, J = 3, 10, 8, 4, 16
    _, _, _, xlen, ylen = _problem(40, B, T, U, 8)
    s, _ = _bands(B, T, U, R, xlen, ylen, 41)
    g = torch.Generator().manual_seed(42)
    dx = torch.randn(B, T, R, J, generator=g)
    hid = torch.tanh(torch.randn(B, T, R, J, generator=g))
    for b in range(B):                                      # padding rows are zero, as the kernels upstream write them
        Tn, Un = po.lengths(xlen[b], ylen[b], T, U)
        dx[b, Tn:] = 0
        dx[b, :, min(R, Un):] = 0
    if bf16:
        dd = dx.to(torch.bfloat16).cuda()
        dep, ddp = ops.joint_band_dpre_reduce(dd, None, xlen.cuda(), ylen.cuda(), s.cuda(), U)
        dpre = dd.double().cpu()
    else:
        dep, ddp = ops.joint_band_dpre_reduce(dx.cuda(), hid.cuda(), xlen.cuda(), ylen.cuda(), s.cuda(), U)
        dpre = dx.double() * (1 - hid.double() ** 2)
    rdep, rddp = po.band_reduce(dpre, s.tolist(), xlen, ylen, U)
    assert _rel(dep, rdep) < 1e-6 and _rel(ddp, rddp) < 1e-6
    # utterance 1 alone, and with garbage in another utterance
    one = slice(1, 2)
    args = (dd[one].contiguous(), None) if bf16 else (dx[one].cuda(), hid[one].cuda())
    dep1, ddp1 = ops.joint_band_dpre_reduce(*args, xlen[one].cuda(), ylen[one].cuda(), s[one].cuda(), U)
    assert torch.equal(dep1, dep[one]) and torch.equal(ddp1, ddp[one])


TINY = dict(vocab_embed_size=16, vocab_size=64, input_size=24, enc_hidden_size=48, enc_layers=2, enc_dropout=0,
            enc_proj_size=40, dec_hidden_size=32, dec_layers=1, dec_dropout=0, dec_proj_size=24, joint_size=56)


def _model(**kw):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(5)
    m = Transducer(**TINY, **kw).cuda()
    g = torch.Generator().manual_seed(6)
    xs = torch.randn(4, 20, 24, generator=g).cuda()
    ys = torch.randint(4, 64, (4, 7), dtype=i32, generator=g).cuda()
    xlen, ylen = torch.tensor([20, 20, 15, 9], dtype=i32), torch.tensor([7, 5, 7, 2], dtype=i32)
    return m, (xs, ys, xlen, ylen)


def _step(m, inputs):
    m.zero_grad()
    loss = m(*inputs)
    loss.backward()
    return loss.detach(), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_transducer_pruned_step(precision):
    """Transducer(prune_range=5): the loss is simple_loss_scale * mean(simple) + pruned_loss_scale * mean(pruned),
    the joint's and the simple projections' gradients match an fp64 restatement on the model's own encoder outputs,
    every parameter gets a gradient, and two runs are bitwise equal."""
    from edgedict_b200 import functional as Fn
    from edgedict_b200.rnnt.models import _precision
    m, inputs = _model(prune_range=5)
    m.set_precision(precision)
    l0, g0 = _step(m, inputs)
    sc, pc = m.last_simple_costs, m.last_costs
    assert torch.allclose(l0, 0.5 * sc.mean() + pc.mean(), rtol=1e-6)
    assert set(g0) == {k for k, _ in m.named_parameters()}
    l1, g1 = _step(m, inputs)
    assert torch.equal(l0, l1) and all(torch.equal(g0[k], g1[k]) for k in g0)
    # fp64 restatement of the heads on the same encoder / predictor outputs
    xs, ys, xlen, ylen = inputs
    with torch.no_grad():
        h_enc, h_dec = m._encode(xs, ys, xlen, ylen)
    from edgedict_b200.rnnt.models import scale_length
    xl = scale_length(h_enc.shape[1], xlen).to(i32)
    U = h_dec.shape[1]
    lab = ys[:, :U - 1].cpu().long()
    he, hd = h_enc.double().cpu(), h_dec.double().cpu()
    P = {k: p.detach().double().cpu().requires_grad_(True) for k, p in m.named_parameters()
         if k.startswith(("simple_", "joint."))}
    am = he @ P["simple_am_proj.weight"].t() + P["simple_am_proj.bias"]
    lmp = hd @ P["simple_lm_proj.weight"].t() + P["simple_lm_proj.bias"]
    simple = po.simple_costs(am, lmp, lab, xl, ylen, 0)
    # the bands the model chose: its own projections, in its precision, on the same encoder outputs
    p = _precision(m)
    with torch.no_grad():
        am_dev = Fn.Linear.apply(h_enc, m.simple_am_proj.weight, m.simple_am_proj.bias, p)
        lm_dev = Fn.Linear.apply(h_dec, m.simple_lm_proj.weight, m.simple_lm_proj.bias, p)
        s_dev = Fn.SimpleLoss.apply(am_dev, lm_dev, ys[:, :U - 1].contiguous(), xl.cuda(), ylen.cuda(), 0)[1]
    from edgedict_b200 import ops
    s, nop = ops.rnnt_band_choice(xl.cuda(), ylen.cuda(), 4, h_enc.shape[1], U, 5, s_dev)
    w1, b1 = P["joint.joint.0.weight"], P["joint.joint.0.bias"]
    w2, b2 = P["joint.joint.2.weight"], P["joint.joint.2.bias"]
    E = he.shape[2]
    sl = s.cpu().long()
    idx = (sl[:, :, None] + torch.arange(5)[None, None]).clamp(max=U - 1)
    dp = hd @ w1[:, E:].t()
    dpb = torch.stack([dp[b][idx[b]] for b in range(4)])
    hidden = torch.tanh((he @ w1[:, :E].t() + b1)[:, :, None] + dpb)
    band_logits = hidden @ w2.t() + b2
    pruned = po.pruned_costs(band_logits, lab, xl, ylen, sl.tolist(), U, 0)
    loss = 0.5 * simple.mean() + pruned.mean()
    loss.backward()
    tol = 2e-3 if precision == "fp32" else 6e-2
    assert abs(float(l0) - float(loss)) <= tol * abs(float(loss))
    errs = {k: _rel(g0[k], P[k].grad) for k in P}
    assert max(errs.values()) < tol, errs


def test_transducer_pruned_scales_and_fastemit():
    m, inputs = _model(prune_range=4)
    m.pruned_loss_scale = 0.0                          # the pruned joint is skipped
    m.zero_grad()
    loss = m(*inputs)
    assert m.last_costs is None
    assert torch.allclose(loss, 0.5 * m.last_simple_costs.mean())
    loss.backward()
    assert m.joint.joint[2].weight.grad is None
    m.fastemit_lambda = 0.01
    with pytest.raises(ValueError):
        m(*inputs)
