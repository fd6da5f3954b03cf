"""The raw-waveform front end on the device (FrontEnd, DilatedConvBlock: csrc/conv.cu) against the fp64 restatement
(tests/frontend_oracle.py) and the reference's own outputs (tests/golden/frontend_tiny.npz): per block teacher-forced
and end to end in fp32 mode; in bf16 mode within bf16 bars of exact fp64 and, element by element, against the
restatement of bf16 mode's roundings (the residual is fp32 accumulation and rare bf16 rounding-boundary flips; a wiring
mistake in the backward permutes or regroups terms and shows up near 1); both modes at a production shape (8 utterances
of up to 14 s); the padded-frame GroupNorm semantics, bitwise repeatable steps, a full FrontEnd + Transducer step
against oracle.model_torch, and loading wav2vec-shaped weights."""
import os

import numpy as np
import pytest
import torch
from torch import nn

from tests import frontend_oracle as fo

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TRAIN = [(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3
DFLT = [(10, 5, 16)] + [(8, 4, 32)] + [(4, 2, 128)] * 3
SAMPLE_ABOVE, SAMPLE_STEP = 4096, 31          # tests/golden/make_golden_frontend.py


# max-relative error of bf16 mode against the rounding restatement, per block and end to end (7 blocks: a rounding-
# boundary flip in an early block carries through the later ones); measured worst 2.5e-4 and 6.5e-3 on an H100
BF16_BAR_BLOCK, BF16_BAR = 1e-3, 3e-2


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double().to(torch.as_tensor(a).device)
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _against_rounding(name, got, ref, bar=BF16_BAR):
    """Max-relative error of one bf16-mode output against the rounding restatement, printed and asserted."""
    r = _rel(got, ref)
    print("  %-40s max-relative error vs the bf16 rounding restatement %.3g" % (name, r))
    assert r < bar, (name, r)


def _frontend(params, bias, seed, precision="fp32"):
    from edgedict_b200.rnnt.models import FrontEnd
    torch.manual_seed(seed)
    return FrontEnd(params, bias=bias).cuda().set_precision(precision)


def _fixture(tag):
    z = np.load(os.path.join(GOLDEN, "frontend_tiny.npz"))
    params = [tuple(int(v) for v in r) for r in z[tag + ".params"]]
    return z, params, bool(z[tag + ".bias"]), int(z[tag + ".seed"])


def _sd_cpu(m):
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("tag", ["train", "pre", "dflt"])
def test_fp32_matches_the_reference_fixture_and_fp64(tag):
    z, params, bias, seed = _fixture(tag)
    m = _frontend(params, bias, seed)
    x = torch.as_tensor(z["x"]).cuda()
    out = m(x)
    (out * torch.as_tensor(z[tag + ".R"]).cuda()).sum().backward()
    assert out.shape == z[tag + ".out"].shape
    assert _rel(out.detach(), z[tag + ".out"]) < 1e-4
    ref_out, ref_g = fo.forward_and_grads(_sd_cpu(m), z["x"], params, z[tag + ".R"])
    assert _rel(out.detach(), ref_out) < 1e-4
    for k, p in m.named_parameters():
        g = p.grad.detach().cpu().reshape(-1)
        r = ref_g[k].reshape(-1)
        assert _rel(g, r) < 1e-3, k
        want = z[tag + ".grad." + k]
        got = g if g.numel() <= SAMPLE_ABOVE else g[::SAMPLE_STEP]
        assert _rel(got, want) < 1e-3, k


# (C_in, C_out, k, s, bias, T): every (k, s) of the reference configurations, C_in of 16, 32 and 128, odd sizes in
# fp32 mode, C_in > 256 (two channel blocks in the GroupNorm passes), row counts that leave partial 128-row tiles
BLOCKS = [(16, 32, 8, 4, True, 301), (32, 128, 3, 2, True, 517), (128, 128, 3, 2, False, 260),
          (128, 128, 2, 2, True, 133), (128, 128, 4, 2, True, 97), (32, 16, 10, 5, False, 211),
          (24, 40, 3, 2, True, 77), (128, 48, 2, 3, True, 50), (320, 64, 3, 2, True, 90)]


def _block(cin, cout, k, s, bias, seed, precision="fp32"):
    from edgedict_b200.rnnt.models import DilatedConvBlock
    torch.manual_seed(seed)
    blk = DilatedConvBlock(cin, cout, k, stride=s, bias=bias)
    with torch.no_grad():
        blk.gn.weight.uniform_(0.5, 1.5)
        blk.gn.bias.uniform_(-0.5, 0.5)
    return blk.cuda().set_precision(precision)


def _block_ref(blk, x, R, s, rnd=None):
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in blk.state_dict().items()}
    xr = x.detach().cpu().double().requires_grad_(True)
    out = fo.block(xr, sd["conv.weight"], sd.get("conv.bias"), sd["gn.weight"], sd["gn.bias"], s, blk.gn.eps, rnd)
    (out * R.cpu().double()).sum().backward()
    return out.detach(), {k: v.grad for k, v in sd.items()}, xr.grad


@pytest.mark.parametrize("cin,cout,k,s,bias,T", BLOCKS)
def test_block_fp32_teacher_forced_against_fp64(cin, cout, k, s, bias, T):
    blk = _block(cin, cout, k, s, bias, seed=cin + cout + k)
    g = torch.Generator().manual_seed(T)
    x = (torch.randn(3, cin, T, generator=g) * 2.0 + 0.3).cuda().requires_grad_(True)
    out = blk(x)
    R = torch.randn(out.shape, generator=g).cuda()
    (out * R).sum().backward()
    ref, ref_g, ref_dx = _block_ref(blk, x, R, s)
    assert out.shape == ref.shape
    assert _rel(out.detach(), ref) < 1e-4
    assert _rel(x.grad, ref_dx) < 1e-3
    for kk, p in blk.named_parameters():
        assert _rel(p.grad, ref_g[kk]) < 1e-3, kk


@pytest.mark.parametrize("cin,cout,k,s,bias,T", [b for b in BLOCKS if b[0] % 16 == 0 and b[1] % 16 == 0])
def test_block_bf16_against_fp64(cin, cout, k, s, bias, T):
    blk = _block(cin, cout, k, s, bias, seed=cin + cout + k, precision="bf16")
    g = torch.Generator().manual_seed(T)
    x = (torch.randn(3, cin, T, generator=g) * 2.0 + 0.3).cuda().requires_grad_(True)
    out = blk(x)
    R = torch.randn(out.shape, generator=g).cuda()
    (out * R).sum().backward()
    ref, ref_g, ref_dx = _block_ref(blk, x, R, s)
    assert _rel(out.detach(), ref) < 2e-2
    assert abs(float(x.grad.double().norm()) / float(ref_dx.norm()) - 1) < 2e-2
    for kk, p in blk.named_parameters():
        assert abs(float(p.grad.double().norm()) / float(ref_g[kk].norm()) - 1) < 2e-2, kk
    # element by element against the restatement of bf16 mode's roundings
    ref, ref_g, ref_dx = _block_ref(blk, x, R, s, rnd=True)
    name = "block %d-%d k%d s%d T%d" % (cin, cout, k, s, T)
    _against_rounding(name + " out", out.detach(), ref, BF16_BAR_BLOCK)
    _against_rounding(name + " dx", x.grad, ref_dx, BF16_BAR_BLOCK)
    for kk, p in blk.named_parameters():
        _against_rounding(name + " " + kk, p.grad, ref_g[kk], BF16_BAR_BLOCK)


def test_block_follows_the_modules_groupnorm_eps():
    blk = _block(32, 32, 3, 2, True, seed=7)
    blk.gn.eps = 0.05
    g = torch.Generator().manual_seed(8)
    x = (0.05 * torch.randn(2, 32, 60, generator=g)).cuda().requires_grad_(True)   # variance comparable to eps
    out = blk(x)
    R = torch.randn(out.shape, generator=g).cuda()
    (out * R).sum().backward()
    ref, ref_g, ref_dx = _block_ref(blk, x, R, 2)
    assert _rel(out.detach(), ref) < 1e-4
    assert _rel(x.grad, ref_dx) < 1e-3
    for kk, p in blk.named_parameters():
        assert _rel(p.grad, ref_g[kk]) < 1e-3, kk


def test_in_place_parameter_change_before_backward_is_detected():
    m = _frontend(DFLT, True, 9)
    out = m(0.3 * torch.randn(2, 6000, device="cuda"))
    with torch.no_grad():
        m.encode[0].conv.weight.mul_(2.0)
    with pytest.raises(RuntimeError, match="inplace"):
        out.sum().backward()


def test_first_layer_alone_against_fp64():
    m = _frontend([(10, 5, 32)], True, 3)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(4, 3333, generator=g)
    out = m(x.cuda())
    R = torch.randn(out.shape, generator=g)
    (out * R.cuda()).sum().backward()
    ref, ref_g = fo.forward_and_grads(_sd_cpu(m), x, [(10, 5, 32)], R)
    assert _rel(out.detach(), ref) < 1e-4
    for k, p in m.named_parameters():
        assert _rel(p.grad, ref_g[k]) < 1e-3, k


@pytest.mark.parametrize("params", [TRAIN, DFLT], ids=["train", "dflt"])
def test_bf16_end_to_end_within_bf16_bars(params):
    m = _frontend(params, True, 21, "bf16")
    g = torch.Generator().manual_seed(6)
    x = torch.zeros(3, 24000)
    for b, n in enumerate((24000, 21000, 17000)):
        x[b, :n] = 0.3 * torch.randn(n, generator=g)
    out = m(x.cuda())
    R = torch.randn(out.shape, generator=g)
    (out * R.cuda()).sum().backward()
    ref, ref_g = fo.forward_and_grads(_sd_cpu(m), x, params, R)
    assert _rel(out.detach(), ref) < 5e-2
    for k, p in m.named_parameters():
        assert abs(float(p.grad.double().norm()) / float(ref_g[k].norm()) - 1) < 2e-2, k
    ref, ref_g = fo.forward_and_grads(_sd_cpu(m), x, params, R, bf16=True)
    name = "end to end %s" % ("train" if params is TRAIN else "dflt")
    _against_rounding(name + " out", out.detach(), ref)
    for k, p in m.named_parameters():
        _against_rounding(name + " " + k, p.grad, ref_g[k])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_production_shape_against_fp64_on_the_device(precision):
    """cli/train.py's parameters on 8 utterances of up to 14 s (ragged): about 10 tiles per CTA in the first block's
    forward conv and dX, many row splits in every reduction.  The output and every gradient per element against fp64
    computed on the device: exact fp64 in fp32 mode, the rounding restatement in bf16 mode."""
    m = _frontend(TRAIN, True, 70, precision)
    g = torch.Generator(device="cuda").manual_seed(71)
    lens = [224000, 215000, 198000, 180500, 160000, 143999, 120000, 96000]
    x = torch.zeros(len(lens), lens[0], device="cuda")
    for b, n in enumerate(lens):
        x[b, :n] = 0.3 * torch.randn(n, device="cuda", generator=g)
    out = m(x)
    R = torch.randn(out.shape, device="cuda", generator=g)
    (out * R).sum().backward()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    bf = precision == "bf16"
    ref, ref_g = fo.forward_and_grads(sd, x, TRAIN, R, bf16=bf)
    check = _against_rounding if bf else (lambda n, a, b: _against_fp64(n, a, b, 1e-4 if n.endswith("out") else 1e-3))
    check("production %s out" % precision, out.detach(), ref)
    for k, p in m.named_parameters():
        check("production %s %s" % (precision, k), p.grad, ref_g[k])


def _against_fp64(name, got, ref, bar):
    r = _rel(got, ref)
    print("  %-40s max-relative error vs fp64 %.3g" % (name, r))
    assert r < bar, (name, r)


def test_groupnorm_statistics_include_padded_frames():
    m = _frontend(DFLT, True, 8)
    g = torch.Generator().manual_seed(9)
    short = 0.3 * torch.randn(1, 4000, generator=g)
    batch = torch.zeros(2, 9000)
    batch[0, :4000] = short[0]
    batch[1] = 0.3 * torch.randn(9000, generator=g)
    with torch.no_grad():
        alone = m(short.cuda()).cpu()
        together = m(batch.cuda()).cpu()
    sd = _sd_cpu(m)
    ref_alone = fo.forward(fo_sd(sd), short.double(), DFLT)
    ref_together = fo.forward(fo_sd(sd), batch.double(), DFLT)
    assert _rel(alone, ref_alone) < 1e-4 and _rel(together, ref_together) < 1e-4
    T = alone.shape[1]
    # the same utterance gives other frames when the batch's longer utterance pads it
    assert float((together[0, :T] - alone[0]).abs().max()) > 1e-2


def fo_sd(sd):
    return {k: v.double() for k, v in sd.items()}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_bitwise_repeatable_under_deterministic_algorithms(precision):
    m = _frontend(TRAIN, True, 30, precision)
    g = torch.Generator().manual_seed(31)
    x = (0.3 * torch.randn(4, 20000, generator=g)).cuda()
    runs = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            for p in m.parameters():
                p.grad = None
            out = m(x)
            (out * out).sum().backward()
            runs.append([out.detach().clone()] + [p.grad.clone() for p in m.parameters()])
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def _step_inputs():
    g = torch.Generator().manual_seed(41)
    lens = torch.tensor([16000, 14500, 13000])
    x = torch.zeros(3, 16000)
    for b, n in enumerate(lens.tolist()):
        x[b, :n] = 0.3 * torch.randn(n, generator=g)
    ys = torch.randint(4, 40, (3, 5), generator=g, dtype=torch.int32)
    ylen = torch.tensor([5, 3, 4], dtype=torch.int32)
    return x, lens, ys, ylen


TCFG = dict(vocab_embed_size=16, vocab_size=40, input_size=128, enc_hidden_size=64, enc_layers=2, enc_dropout=0,
            enc_proj_size=48, enc_time_reductions=[], dec_hidden_size=32, dec_layers=1, dec_dropout=0,
            dec_proj_size=48, joint_size=40)


def _models(precision):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(50)
    fe = _frontend(TRAIN, True, 51, precision)
    torch.manual_seed(52)
    model = Transducer(**TCFG).cuda().set_precision(precision)
    return fe, model


def _engine_step(fe, model, x, lens, ys, ylen):
    from edgedict_b200.rnnt.models import frontend_lengths
    out = fe(x.cuda())
    xlen = frontend_lengths(lens, out.shape[1])
    xs = out[:, :int(xlen.max())].contiguous()
    return model(xs, ys.cuda(), xlen, ylen)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_full_step_bitwise_repeatable_under_deterministic_algorithms(precision):
    x, lens, ys, ylen = _step_inputs()
    fe, model = _models(precision)
    params = list(model.parameters()) + list(fe.parameters())
    runs = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            for p in params:
                p.grad = None
            loss = _engine_step(fe, model, x, lens, ys, ylen)
            loss.backward()
            runs.append([loss.detach().clone()] + [p.grad.clone() for p in params])
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_full_step_fp32_against_model_torch_and_bf16_loss():
    from edgedict_b200.rnnt.models import frontend_lengths
    from oracle import model_torch as mt
    x, lens, ys, ylen = _step_inputs()
    fe, model = _models("fp32")
    loss = _engine_step(fe, model, x, lens, ys, ylen)
    loss.backward()
    loss = loss.detach()
    sd_fe = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in fe.state_dict().items()}
    sd_m = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    out = fo.forward(sd_fe, x, TRAIN)
    xlen = frontend_lengths(lens, out.shape[1])
    ref = mt.transducer_loss(sd_m, out[:, :int(xlen.max())].contiguous(), ys, xlen, ylen, time_reductions=())
    ref.backward()
    ref = ref.detach()
    assert abs(float(loss) - float(ref)) / abs(float(ref)) < 1e-4
    for mod, sd in ((fe, sd_fe), (model, sd_m)):
        for k, p in mod.named_parameters():
            assert _rel(p.grad, sd[k].grad) < 2e-3, k
    fe16, m16 = _models("bf16")
    loss16 = _engine_step(fe16, m16, x, lens, ys, ylen).detach()
    assert abs(float(loss16) - float(loss)) / abs(float(loss)) < 1e-3


def test_flat_adam_steps_frontend_and_transducer_together():
    from edgedict_b200.optim import FlatAdam
    x, lens, ys, ylen = _step_inputs()
    fe, model = _models("bf16")
    before = [p.detach().clone() for p in list(model.parameters()) + list(fe.parameters())]
    opt = FlatAdam(nn.ModuleList([model, fe]), lr=1e-3)
    losses = []
    for _ in range(3):
        opt.zero_grad()
        loss = _engine_step(fe, model, x, lens, ys, ylen)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    after = list(model.parameters()) + list(fe.parameters())
    assert all(not torch.equal(a, b) for a, b in zip(before, after))
    assert losses[-1] < losses[0]


def test_loading_wav2vec_frontend_weights():
    from edgedict_b200.rnnt.models import FrontEnd
    torch.manual_seed(60)
    src = FrontEnd(TRAIN, bias=False)
    ckpt = {"frontend." + k: v.clone() for k, v in src.state_dict().items()}
    ckpt["encoder.proj.weight"] = torch.zeros(1)          # other keys of a wav2vec checkpoint pass by
    fe = FrontEnd(TRAIN, bias=False)
    front = fe.state_dict()
    for key, tensor in ckpt.items():                      # cli/train.py's load_pretrained_model
        if "frontend." in key:
            front[key.replace("frontend.", "")] = tensor
    fe.load_state_dict(front)
    fe = fe.cuda()
    g = torch.Generator().manual_seed(61)
    x = 0.3 * torch.randn(2, 9000, generator=g)
    with torch.no_grad():
        out = fe(x.cuda()).cpu()
    ref = fo.forward(fo_sd(src.state_dict()), x.double(), TRAIN)
    assert _rel(out, ref) < 1e-4
