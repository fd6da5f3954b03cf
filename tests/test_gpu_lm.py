"""The language model on the engine (edgedict_b200.models.LMModel): forward against the reference's own outputs, the
fused loss (LMModel.loss: the output GEMM with its cross-entropy epilogue, csrc/gemm_tc.cu + csrc/lm.cu) and every
gradient against the fp64 restatement (tests/lm_train_oracle.py) and against the drop-in path, its invariants, and a
trained module driving the device beam searches."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import lm_train_oracle as lo

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# tensor-core shapes: nhid a multiple of 256 (the cluster recurrence), V and K multiples of 8; M = B*S = 96 and V = 520
# leave partial row and column tiles
SHAPES = {"untied": (64, 256, 512, False), "tied": (256, 256, 512, True), "ragged": (64, 256, 520, False)}


def model(ntoken, ninp, nhid, nlayers=2, tie=False, seed=0, precision="fp32"):
    from edgedict_b200.models import LMModel
    torch.manual_seed(seed)
    m = LMModel(ntoken, ninp, nhid, nlayers, dropout=0.0, tie_weights=tie).cuda()
    return m.set_precision(precision)


def batch(V, B=8, S=12, seed=1, pad=0.15):
    """Tokens in [1, V), a <bos> = 1 column in front, and about `pad` of the targets 0 (trailing, as seq_collate pads)."""
    g = torch.Generator().manual_seed(seed)
    tg = torch.randint(1, V, (B, S), generator=g)
    lens = S - (torch.rand(B, generator=g) * 2 * pad * S).long()
    tg[torch.arange(S)[None] >= lens[:, None]] = 0
    inp = torch.cat([torch.ones(B, 1, dtype=torch.long), tg[:, :-1]], 1)
    return inp, tg


def grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters()}


def zero(m):
    for p in m.parameters():
        p.grad = None


def sd_of(m):
    return {k: v.detach().cpu().double().numpy() for k, v in m.state_dict().items()}


def fixture(tag):
    z = np.load(os.path.join(GOLDEN, "lm_train_tiny.npz"))
    p = tag + ".sd."
    return z, {k[len(p):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(p)}


@pytest.mark.parametrize("tag", ["u", "t"])
def test_forward_matches_the_reference(tag):
    from edgedict_b200.models import LMModel
    z, sd = fixture(tag)
    ninp, nhid = sd["encoder.weight"].shape[1], sd["rnn.weight_hh_l0"].shape[1]
    m = LMModel(int(z["ntoken"]), ninp, nhid, 2, dropout=0.0, tie_weights=tag == "t")
    m.load_state_dict(sd)
    m = m.cuda().eval()
    inp = torch.from_numpy(z["inputs"]).cuda()
    with torch.no_grad():
        logp, (h, c) = m(inp, m.init_hidden(inp.shape[0]))
    assert logp.shape == (inp.numel(), int(z["ntoken"])) and logp.dtype == torch.float32
    np.testing.assert_allclose(logp.cpu().numpy(), z[tag + ".logp"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(h.cpu().numpy(), z[tag + ".h"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(c.cpu().numpy(), z[tag + ".c"], rtol=0, atol=1e-5)
    hid = (torch.from_numpy(z[tag + ".h0"]).cuda(), torch.from_numpy(z[tag + ".c0"]).cuda())
    with torch.no_grad():
        logp, (h, c) = m(inp, hid)
    np.testing.assert_allclose(logp.cpu().numpy(), z[tag + ".logp_h0"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(h.cpu().numpy(), z[tag + ".h_h0"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(c.cpu().numpy(), z[tag + ".c_h0"], rtol=0, atol=1e-5)
    # the fused loss on the fixture's padded batch: the reference's NLLLoss(ignore_index=0) value
    loss = m.train().loss(inp, torch.from_numpy(z["targets"]).cuda())
    assert abs(float(loss.detach()) - float(z[tag + ".loss"])) < 1e-5


def test_forward_matches_the_fusion_fixture():
    from edgedict_b200.models import LMModel
    z = np.load(os.path.join(GOLDEN, "lm_tiny.npz"))
    m = LMModel(16, 6, 10, 2, dropout=0.5)
    m.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd.")})
    m = m.cuda().eval()
    toks = torch.from_numpy(z["tokens"]).long().cuda()
    with torch.no_grad():
        logp, (h, c) = m(toks, None)
    np.testing.assert_allclose(logp.view(3, 7, 16).cpu().numpy(), z["logp"], rtol=0, atol=5e-5)
    np.testing.assert_allclose(h.cpu().numpy(), z["h"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(c.cpu().numpy(), z["c"], rtol=0, atol=1e-5)


# fp32: the fp32 GEMMs and recurrence; bf16: bf16 operands with fp32 accumulation throughout (relative to the largest
# gradient element of each parameter)
TOL = {"fp32": (2e-6, 2e-4), "bf16": (1e-2, 4e-2)}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_loss_and_gradients_against_fp64(shape, precision):
    ninp, nhid, V, tie = SHAPES[shape]
    m = model(V, ninp, nhid, tie=tie, precision=precision)
    inp, tg = batch(V)
    want, wg = lo.loss_and_grads(sd_of(m), inp.numpy(), tg.numpy(), tied=tie)
    loss = m.loss(inp.cuda(), tg.cuda())
    loss.backward()
    assert loss.shape == () and loss.dtype == torch.float32
    tl, tg_ = TOL[precision]
    assert abs(float(loss.detach()) - want) <= tl * abs(want), (float(loss.detach()), want)
    got = grads(m)
    assert set(got) == set(wg)
    for k, g in got.items():
        ref = wg[k]
        err = np.abs(g.cpu().double().numpy() - ref).max() / np.abs(ref).max()
        assert err <= tg_, (k, err)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("reduction", ["mean", "sum", "none"])
def test_loss_equals_the_drop_in_path(precision, reduction):
    ninp, nhid, V, _ = SHAPES["untied"]
    m = model(V, ninp, nhid, precision=precision)
    inp, tg = batch(V)
    inp, tg = inp.cuda(), tg.cuda()
    h0 = tuple(0.3 * torch.randn(2, inp.shape[0], nhid, device="cuda") for _ in range(2))
    gw = torch.rand(inp.numel(), device="cuda") if reduction == "none" else None
    logp, _ = m(inp, h0)
    ref = F.nll_loss(logp, tg.flatten(), ignore_index=0, reduction=reduction)
    (ref if gw is None else (ref * gw).sum()).backward()
    rg = grads(m)
    zero(m)
    got = m.loss(inp, tg, h0, reduction=reduction)
    (got if gw is None else (got * gw).sum()).backward()
    assert got.shape == ref.shape
    tl, tg_ = (1e-6, 1e-5) if precision == "fp32" else (1e-2, 4e-2)
    np.testing.assert_allclose(got.detach().cpu().numpy(), ref.detach().cpu().numpy(), rtol=tl, atol=tl)
    if reduction == "none":
        assert (got[tg.flatten() == 0] == 0).all()
    for k, g in grads(m).items():
        err = float((g - rg[k]).abs().max() / rg[k].abs().max())
        assert err <= tg_, (k, err)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_ignored_positions_do_not_move_any_gradient(precision):
    """New tokens at the padded positions change the logits there (and the LSTM state after the sequence's end) but no
    gradient, bit for bit; the costs of those positions are 0 and every other cost is unchanged."""
    ninp, nhid, V, _ = SHAPES["untied"]
    m = model(V, ninp, nhid, precision=precision)
    inp, tg = batch(V, pad=0.3)
    pad = (tg == 0)
    pad_in = torch.zeros_like(pad)
    pad_in[:, 1:] = pad[:, :-1]                                  # inputs that only feed ignored positions
    assert pad_in.any()
    out = []
    for seed in (0, 1):
        g = torch.Generator().manual_seed(seed)
        x = torch.where(pad_in, torch.randint(1, V, inp.shape, generator=g), inp)
        zero(m)
        cost = m.loss(x.cuda(), tg.cuda(), reduction="none")
        cost.sum().backward()
        out.append((cost.detach(), grads(m)))
    assert torch.equal(out[0][0], out[1][0])
    assert (out[0][0][pad.flatten().cuda()] == 0).all()
    for k in out[0][1]:
        assert torch.equal(out[0][1][k], out[1][1][k]), k


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_tied_weight_gradient_is_the_sum_of_both_uses(precision):
    ninp, nhid, V, _ = SHAPES["tied"]
    tied = model(V, ninp, nhid, tie=True, seed=3, precision=precision)
    untied = model(V, ninp, nhid, tie=False, seed=3, precision=precision)
    untied.load_state_dict(tied.state_dict())
    inp, tg = batch(V)
    for m in (tied, untied):
        m.loss(inp.cuda(), tg.cuda()).backward()
    gt, gu = grads(tied), grads(untied)
    assert "decoder.weight" not in gt
    both = gu["encoder.weight"] + gu["decoder.weight"]
    assert float((gt["encoder.weight"] - both).abs().max()) <= 1e-6 * float(both.abs().max())
    for k in gt:
        if k != "encoder.weight":
            assert torch.equal(gt[k], gu[k]), k


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_two_identical_steps_are_bitwise_identical(precision):
    ninp, nhid, V, _ = SHAPES["untied"]
    m = model(V, ninp, nhid, precision=precision)
    inp, tg = batch(V, B=40, S=20)
    runs = []
    for _ in range(2):
        zero(m)
        loss = m.loss(inp.cuda(), tg.cuda())
        loss.backward()
        runs.append((loss.detach().clone(), grads(m)))
    assert torch.equal(runs[0][0], runs[1][0])
    for k in runs[0][1]:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("dtype", [torch.int64, torch.int32])
def test_out_of_range_targets_give_nan_costs(precision, dtype):
    ninp, nhid, V, _ = SHAPES["untied"]
    m = model(V, ninp, nhid, precision=precision)
    inp, tg = batch(V)
    bad = tg.clone()
    bad[0, 2], bad[3, 4], bad[5, 0] = V, -7, 2 ** 30
    cost = m.loss(inp.cuda(), bad.to(dtype).cuda(), reduction="none")
    ref = m.loss(inp.cuda(), tg.to(dtype).cuda(), reduction="none").detach()
    nan = torch.zeros_like(tg, dtype=torch.bool)
    nan[0, 2] = nan[3, 4] = nan[5, 0] = True
    nan = nan.flatten().cuda()
    assert torch.isnan(cost[nan]).all()
    assert torch.equal(cost[~nan].detach(), ref[~nan])
    assert torch.isnan(m.loss(inp.cuda(), bad.to(dtype).cuda()))
    # with ignore_index = -100 the padded 0s are ordinary targets, and -100 itself is ignored
    pads = tg.clone()
    pads[tg == 0] = -100
    want = m.loss(inp.cuda(), tg.to(dtype).cuda(), ignore_index=V + 5)
    got = m.loss(inp.cuda(), tg.to(dtype).cuda(), ignore_index=-100)
    assert torch.isfinite(got) and torch.equal(got, want)
    got = m.loss(inp.cuda(), pads.to(dtype).cuda(), ignore_index=-100)
    got = float(got.detach())
    assert abs(got - float(ref.sum()) / int((tg != 0).sum())) <= 1e-6 * abs(got)
    # all ignored: torch's NaN mean, zero gradients
    zero(m)
    loss = m.loss(inp.cuda(), torch.zeros_like(tg).to(dtype).cuda())
    loss.backward()
    assert torch.isnan(loss)
    assert all(float(g.abs().max()) == 0 for g in grads(m).values())


def test_a_few_flat_adam_steps_lower_the_loss():
    from edgedict_b200.optim import FlatAdam
    ninp, nhid, V, _ = SHAPES["untied"]
    m = model(V, ninp, nhid, precision="bf16")
    m.train()
    inp, tg = batch(V, B=32, S=16)
    inp, tg = inp.cuda(), tg.cuda()
    opt = FlatAdam(m, lr=1e-2)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = m.loss(inp, tg)
        loss.backward()
        opt.step(max_norm=1.0)
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0] - 0.05, losses


def test_a_trained_module_drives_the_beam_searches():
    """Train a few steps, then: the state_dict gives the fp64 restatement's log-probs (what loading it into the
    reference's LMModel gives); fused into Transducer.beam_search and ctc.beam_search, the module gives the searches'
    fp32 restatements run with the trained weights, which differ from those run with the initial ones; the module and
    its state_dict give the same results."""
    from edgedict_b200 import ctc
    from edgedict_b200.optim import FlatAdam
    from edgedict_b200.rnnt.models import Transducer
    from tests import ctc_beam_oracle as cbo
    from tests import lm_oracle
    V = 64
    m = model(V, 32, 64, seed=4)
    init = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    m.train()
    inp, tg = batch(V, B=8, S=10)
    opt = FlatAdam(m, lr=3e-2)
    for _ in range(5):
        opt.zero_grad()
        m.loss(inp.cuda(), tg.cuda()).backward()
        opt.step(max_norm=1.0)
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    assert any(not torch.equal(sd[k], init[k]) for k in sd)
    m.eval()
    with torch.no_grad():
        logp, _ = m(inp.cuda(), None)
    want, _, _ = lo.forward(sd, inp.numpy())
    np.testing.assert_allclose(logp.cpu().numpy(), want, rtol=0, atol=5e-5)

    torch.manual_seed(5)
    t = Transducer(vocab_embed_size=16, vocab_size=V, input_size=24, enc_hidden_size=32, enc_layers=2, enc_dropout=0,
                   enc_proj_size=24, dec_hidden_size=32, dec_layers=1, dec_dropout=0, dec_proj_size=24,
                   joint_size=32, output_loss=False)
    tsd = {k: v.detach().clone() for k, v in t.state_dict().items()}
    t = t.cuda()
    xs = torch.randn(2, 20, 24)
    kw = dict(lm_weight=1.0, length_bonus=3.0)            # (the bonus makes the untrained transducer emit tokens)
    ids, nlp = t.beam_search(xs.cuda(), W=4, lm=m, **kw)
    rids, rlp = lm_oracle.beam_search(tsd, xs, W=4, lm_sd=sd, **kw)
    assert ids == rids and all(len(r) > 0 for r in ids)
    assert float((nlp.cpu().double() - rlp.double()).abs().max() / rlp.double().abs().max()) < 1e-4
    _, ilp = lm_oracle.beam_search(tsd, xs, W=4, lm_sd=init, **kw)
    assert float((ilp.double() - rlp.double()).abs().max()) > 1e-3       # the trained weights reach the search
    ids2, nlp2 = t.beam_search(xs.cuda(), W=4, lm=sd, **kw)
    assert ids2 == ids and torch.equal(nlp2, nlp)

    lp = torch.log_softmax(torch.randn(2, 15, V), -1)
    got = ctc.beam_search(lp.cuda(), [15, 11], 4, lm=m, **kw)
    rids, rs, _ = cbo.batch_search(lp.numpy(), [15, 11], 4, 0, dtype=np.float32, lm_sd=sd, **kw)
    assert all(np.array_equal(x, y) for x, y in zip(got[0], rids))
    assert np.allclose(got[1].double().cpu().numpy(), rs, rtol=1e-5)
    _, irs, _ = cbo.batch_search(lp.numpy(), [15, 11], 4, 0, dtype=np.float32, lm_sd=init, **kw)
    assert np.abs(irs - rs).max() > 1e-3
    b = ctc.beam_search(lp.cuda(), [15, 11], 4, lm=sd, **kw)
    assert all(np.array_equal(x, y) for x, y in zip(got[0], b[0])) and torch.equal(got[1], b[1])


@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_autocast_selects_the_bf16_path(reduction):
    """Under torch.autocast('cuda') an fp32-mode module runs what set_precision('bf16') runs, bit for bit."""
    ninp, nhid, V, _ = SHAPES["untied"]
    inp, tg = batch(V)
    inp, tg = inp.cuda(), tg.cuda()
    out = []
    for ac in (False, True):
        m = model(V, ninp, nhid, precision="fp32" if ac else "bf16")
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
            with torch.no_grad():
                logp, (h, c) = m(inp)
            loss = m.loss(inp, tg, reduction=reduction)
        loss.sum().backward()
        out.append((logp, h, c, loss.detach(), grads(m)))
    for a, b in zip(out[0][:4], out[1][:4]):
        assert torch.equal(a, b)
    for k in out[0][4]:
        assert torch.equal(out[0][4][k], out[1][4][k]), k
    ref = model(V, ninp, nhid, precision="fp32")
    with torch.no_grad():
        assert not torch.equal(ref(inp)[0], out[0][0])                 # (fp32 mode is another computation)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_loss_kernels_at_an_odd_vocabulary(precision):
    """V = 517: the row-wise fp32 stores of the logits GEMM's epilogue (no staged TMA store, V % 8 != 0) and the scalar
    gradient kernel, against fp64 on the same hidden rows and weights.  The whole loss at V = 517 in fp32 mode."""
    from edgedict_b200 import ops
    M, K, V = 200, 64, 517
    g = torch.Generator().manual_seed(9)
    x = torch.randn(M, K, generator=g)
    w = 0.2 * torch.randn(V, K, generator=g)
    b = 0.1 * torch.randn(V, generator=g)
    t = torch.randint(0, V, (M,), generator=g)
    t[::7] = 0
    xd, wd, bd, td = x.cuda(), w.cuda(), b.cuda(), t.cuda()
    if precision == "bf16":
        xq, wq = x.bfloat16().double(), w.bfloat16().double()
        logits, lse, tl = ops.lm_logits_ce(ops.cast_bf16(xd), ops.cast_bf16(wd), bd, td)
    else:
        xq, wq = x.double(), w.double()
        logits = ops.mm_nt(xd, wd, bd, "fp32")
        lse, tl = ops.lm_ce_rows(logits, td)
    ref = xq @ wq.T + b.double()
    rlse = torch.logsumexp(ref, 1)
    tol = 1e-5 if precision == "fp32" else 1e-4
    assert float((lse.cpu().double() - rlse).abs().max()) < tol
    assert float((tl.cpu().double() - ref[torch.arange(M), t]).abs().max()) < tol
    if precision == "bf16":
        assert float((logits.cpu().double() - ref).abs().max()) <= float(ref.abs().max()) * 2 ** -8
    cost, loss, scale = ops.lm_ce_loss(lse, tl, td, 0, V, True)
    keep = t != 0
    rcost = torch.where(keep, rlse - ref[torch.arange(M), t], torch.zeros(()).double())
    assert float((cost.cpu().double() - rcost).abs().max()) < tol
    gs = torch.rand(M, generator=g)
    d = ops.lm_ce_bwd(logits, lse, td, 0, gs.cuda(), None, out=logits)
    rd = torch.softmax(ref, 1)
    rd[torch.arange(M), t] -= 1
    rd = rd * (gs.double() * keep)[:, None]
    assert float((d.cpu().double() - rd).abs().max()) < (1e-6 if precision == "fp32" else 4e-3)
    assert (d[~keep.cuda()] == 0).all()
    if precision == "fp32":
        m = model(V, 64, 256)
        inp, tgt = batch(V)
        want, wg = lo.loss_and_grads(sd_of(m), inp.numpy(), tgt.numpy())
        m.loss(inp.cuda(), tgt.cuda()).backward()
        for k, gk in grads(m).items():
            assert np.abs(gk.cpu().double().numpy() - wg[k]).max() <= 2e-4 * np.abs(wg[k]).max(), k
    else:
        m = model(V, 64, 256, precision="bf16")
        with pytest.raises(ValueError):
            m.loss(*[z.cuda() for z in batch(V)])


def test_embedding_gradient_at_a_language_model_batch():
    """B = 64, S = 128: 8192 positions over a 512-token vocabulary (the padding token 0 at ~15 % of them), every
    gradient of a training step against fp64, the embedding's included."""
    ninp, nhid, V, _ = SHAPES["untied"]
    m = model(V, ninp, nhid, precision="fp32")
    inp, tg = batch(V, B=64, S=128)
    want, wg = lo.loss_and_grads(sd_of(m), inp.numpy(), tg.numpy())
    m.loss(inp.cuda(), tg.cuda()).backward()
    got = grads(m)
    for k, g in got.items():
        err = np.abs(g.cpu().double().numpy() - wg[k]).max() / np.abs(wg[k]).max()
        assert err <= 2e-4, (k, err)
    assert int(torch.count_nonzero(got["encoder.weight"].abs().sum(1))) > V // 2    # most rows receive a gradient
