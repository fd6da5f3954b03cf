"""End-to-end parity of the H100 engine (edgedict_b200.rnnt.models) against the golden fixtures
produced by the reference itself (tests/golden/*.npz) and against the oracle restatements."""
import numpy as np
import pytest
import torch

from tests.util import load_tiny, load_e4d1, e4d1_inputs, E4D1_CFG, rel_err

pytestmark = pytest.mark.gpu

# north_star: "loss and encoder activations within 1e-3 rel fp32"
TOL = 1e-3


def _tiny_model(output_loss=True):
    from edgedict_b200.rnnt.models import Transducer
    z, cfg, sd, pg = load_tiny()
    m = Transducer(output_loss=output_loss, **cfg)
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    return m.cuda(), z, pg


def test_tiny_forward_matches_reference_fixture():
    m, z, _ = _tiny_model(False)
    xs, ys = torch.as_tensor(z["xs"]).cuda(), torch.as_tensor(z["ys"]).cuda()
    with torch.no_grad():
        h_enc, (eh, ec) = m.encoder(xs)
        h_dec, (dh, dc) = m.decoder(ys)
        logits = m.joint(h_enc, h_dec)
    assert rel_err(h_enc.cpu(), z["h_enc"]) < 1e-5 and rel_err(h_dec.cpu(), z["h_dec"]) < 1e-5
    assert rel_err(eh.cpu(), z["enc_h"]) < 1e-5 and rel_err(ec.cpu(), z["enc_c"]) < 1e-5
    assert rel_err(dh.cpu(), z["dec_h"]) < 1e-5 and rel_err(dc.cpu(), z["dec_c"]) < 1e-5
    assert rel_err(logits.cpu(), z["logits"]) < 1e-5
    out = m(xs, ys, torch.as_tensor(z["xlen"]), torch.as_tensor(z["ylen"]))
    assert rel_err(out.detach().cpu(), z["logits"]) < 1e-5   # output_loss=False returns logits


def test_tiny_loss_and_all_parameter_gradients():
    m, z, pg = _tiny_model(True)
    xs, ys = torch.as_tensor(z["xs"]).cuda(), torch.as_tensor(z["ys"]).cuda()
    loss = m(xs, ys, torch.as_tensor(z["xlen"]), torch.as_tensor(z["ylen"]))
    assert rel_err(loss.detach().cpu(), z["loss"]) < 1e-5
    loss.backward()
    for k, p in m.named_parameters():
        assert rel_err(p.grad.cpu(), pg[k]) < TOL, k


def test_tiny_unfused_path_joint_plus_rnntloss_module():
    """cli/lightning.py:83-91 style: output_loss=False, loss applied by the caller."""
    from edgedict_b200.warprnnt_pytorch import RNNTLoss
    m, z, pg = _tiny_model(False)
    xs, ys = torch.as_tensor(z["xs"]).cuda(), torch.as_tensor(z["ys"]).cuda()
    xlen, ylen = torch.as_tensor(z["xlen"]), torch.as_tensor(z["ylen"])
    logits = m(xs, ys, xlen, ylen)
    xl = m.scale_length(logits, xlen)
    loss = RNNTLoss(blank=0)(logits, ys, xl.cuda(), ylen.cuda())
    assert rel_err(loss.detach().cpu(), z["loss"]) < 1e-5
    loss.backward()
    for k, p in m.named_parameters():
        assert rel_err(p.grad.cpu(), pg[k]) < TOL, k


def test_tiny_greedy_decode_token_for_token():
    m, z, _ = _tiny_model(False)
    m.eval()
    ids, nlp = m.greedy_decode(torch.as_tensor(z["xs"]).cuda(), torch.as_tensor(z["xlen"]))
    for got, want in zip(ids, z["greedy_ids"]):
        assert (got == want[:len(got)]).all()
    assert rel_err(nlp.cpu(), z["greedy_nlp"]) < 1e-4


def test_tiny_stateful_encoder_chunks_equal_full_sequence():
    """Streaming contract (rnnt/stream.py:97-98): feeding chunks with carried (h, c) reproduces the
    per-chunk outputs of the reference loop; checked against the oracle restatement."""
    from oracle import model_torch as mt
    m, z, _ = _tiny_model(False)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    chunks = torch.as_tensor(z["stream_chunks"])
    st = None
    eh = ec = None
    with torch.no_grad():
        hid = None
        ref_hid = None
        for i in range(6):
            ch = chunks[i:i + 1]
            out, hid = m.encoder(ch.cuda(), hid)
            ref, ref_hid = mt.encoder(sd, ch, ref_hid)
            assert rel_err(out.cpu(), ref) < 1e-5


def _e4d1():
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(10)
    m = Transducer(**E4D1_CFG)
    return m.cuda(), load_e4d1()


@pytest.mark.parametrize("tag,xl,yl", [("full", [200, 200], [40, 40]), ("ragged", [200, 180], [40, 33])])
def test_e4d1_config_matches_reference_fixture(tag, xl, yl):
    """BASELINE.json configs[0]: E4D1 forward + rnnt_loss, B=2 T=200 U=40."""
    m, z = _e4d1()
    xs, ys = e4d1_inputs()
    assert abs(float(xs.double().sum()) - float(z["xs_sum"])) < 1e-6 and (ys.numpy() == z["ys"]).all()
    xlen, ylen = torch.tensor(xl, dtype=torch.int32), torch.tensor(yl, dtype=torch.int32)
    with torch.no_grad():
        h_enc, _ = m.encoder(xs.cuda())
        h_dec, _ = m.decoder(ys[:, :max(yl)].cuda())
        logits = m.joint(h_enc, h_dec)
    assert rel_err(h_enc.cpu(), z[tag + ".h_enc"]) < TOL
    assert rel_err(h_dec.cpu(), z[tag + ".h_dec"]) < TOL
    assert rel_err(logits[:, ::9, ::5, ::16].cpu(), z[tag + ".logits_sub"]) < TOL
    loss = m(xs.cuda(), ys.cuda(), xlen, ylen)
    assert rel_err(loss.detach().cpu(), z[tag + ".loss"]) < 1e-4
    loss.backward()
    for k, p in m.named_parameters():
        g = p.grad.double().cpu()
        want = float(z[tag + ".pgrad_norm." + k])
        assert abs(float(g.norm()) - want) <= TOL * want + 1e-7, k
        head = z[tag + ".pgrad_head." + k]
        assert np.abs(g.reshape(-1)[:32].numpy() - head).max() <= TOL * (np.abs(head).max() + want / np.sqrt(g.numel()) + 1e-9), k


def test_e4d1_greedy_decode_identical():
    m, z = _e4d1()
    m.eval()
    xs, _ = e4d1_inputs()
    ids, nlp = m.greedy_decode(xs.cuda(), torch.tensor([200, 200]))
    assert (np.stack(ids) == z["greedy_ids"]).all()
    assert rel_err(nlp.cpu(), z["greedy_nlp"]) < 1e-4


def test_bf16_mode_close_to_fp32_mode():
    """bf16 tensor-core mode (bench mode): same engine, GEMM operands rounded to bf16.  Documented
    tolerance: loss within 2e-2 relative of the fp32 path on the tiny-but-aligned config."""
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(5)
    cfg = dict(vocab_embed_size=16, vocab_size=64, input_size=24, enc_hidden_size=48, enc_layers=3,
               enc_dropout=0, enc_proj_size=40, dec_hidden_size=32, dec_layers=2, dec_dropout=0,
               dec_proj_size=24, joint_size=56)
    m = Transducer(**cfg).cuda()
    xs = torch.randn(4, 20, 24).cuda()
    ys = torch.randint(4, 64, (4, 7), dtype=torch.int32).cuda()
    xlen, ylen = torch.tensor([20, 20, 15, 9], dtype=torch.int32), torch.tensor([7, 5, 7, 2], dtype=torch.int32)
    l32 = m(xs, ys, xlen, ylen)
    l32.backward()
    g32 = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    m.set_precision("bf16")
    l16 = m(xs, ys, xlen, ylen)
    l16.backward()
    assert abs(float(l16.detach()) - float(l32.detach())) / float(l32.detach()) < 2e-2
    for k, p in m.named_parameters():
        assert rel_err(p.grad.cpu(), g32[k].cpu()) < 0.15, k
    m.zero_grad()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        m.set_precision("fp32")
        l_ac = m(xs, ys, xlen, ylen)                    # autocast selects the bf16 engine
    assert abs(float(l_ac.detach()) - float(l16.detach())) < 1e-6 * abs(float(l16.detach())) + 1e-6


@pytest.mark.parametrize("B,T,U,E,D,J,V", [(2, 40, 9, 32, 24, 64, 1024), (3, 17, 5, 16, 16, 56, 64), (2, 130, 3, 40, 24, 72, 256)])
def test_fused_joint_lse_path_matches_unfused_bf16_path(B, T, U, E, D, J, V):
    """bf16 mode: the logits GEMM whose epilogue also emits the softmax statistics (+ bf16 logits, in-place
    bf16 gradient) against the unfused bf16 path (fp32 logits, separate denominator kernel)."""
    from edgedict_b200 import functional as Fn
    g = torch.Generator().manual_seed(B * 100 + T)
    h_enc, h_dec = torch.randn(B, T, E, generator=g), torch.randn(B, U, D, generator=g)
    w1, b1 = torch.randn(J, E + D, generator=g) / 6, torch.randn(J, generator=g) / 6
    w2, b2 = torch.randn(V, J, generator=g) / 6, torch.randn(V, generator=g) / 6
    labels = torch.randint(1, V, (B, U - 1), generator=g, dtype=torch.int32)
    xl = torch.full((B,), T, dtype=torch.int32)
    yl = torch.full((B,), U - 1, dtype=torch.int32)
    if B > 1:
        xl[1], yl[1] = max(1, T - 7), max(0, U - 3)
    res = []
    for fused in (False, True):
        Fn.FUSE_JOINT_LSE = fused
        ins = [t.clone().cuda().requires_grad_(True) for t in (h_enc, h_dec, w1, b1, w2, b2)]
        loss, costs = Fn.JointLoss.apply(*ins, labels.cuda(), xl.cuda(), yl.cuda(), 0, "bf16")
        loss.backward()
        res.append((loss.detach().cpu(), costs.cpu(), [t.grad.cpu() for t in ins]))
    Fn.FUSE_JOINT_LSE = True
    (l0, c0, g0), (l1, c1, g1) = res
    assert rel_err(c1, c0) < 2e-3           # same bf16 operands; statistics from fp32 accumulators on both sides
    for a, b, name in zip(g1, g0, "h_enc h_dec w1 b1 w2 b2".split()):
        assert rel_err(a, b) < 6e-2, name   # gradient softmax evaluated on bf16-rounded logits in the fused path


@pytest.mark.parametrize("B,T,L,red,H", [(3, 70, 3, (1,), 64), (2, 133, 4, (0, 2), 128), (33, 48, 2, (1,), 64)])
def test_layer_wavefront_stack_matches_layer_by_layer(B, T, L, red, H):
    """functional.LSTMStack (time-chunked layer wavefront on two streams, chunk-major buffers, chunked BPTT with
    the (dh, dc) carry) against the layer-by-layer Functions: same kernels and arithmetic, so outputs, final
    states and every gradient agree to fp32 round-off of the bulk GEMMs' different summation splits."""
    from edgedict_b200 import functional as Fn
    from edgedict_b200.rnnt.models import ResLayerNormLSTM
    torch.manual_seed(T)
    net = ResLayerNormLSTM(40, H, L, time_reductions=list(red)).cuda()
    for m in net.modules():
        m.precision = "bf16"
    x = torch.randn(B, T, 40).cuda()
    w = torch.randn(B, T, H).cuda()
    res = []
    for chunks in (0, 4):
        Fn.WAVEFRONT_CHUNKS = chunks
        net.zero_grad()
        xi = x.clone().requires_grad_(True)
        y, (hT, cT) = net(xi)
        assert (Fn.wavefront_plan(T, [i in red for i in range(L)]) is not None) == (chunks > 0)
        (y * w[:, :y.shape[1]]).sum().backward()
        res.append((y.detach().cpu(), hT.detach().cpu(), cT.detach().cpu(), xi.grad.cpu(), [p.grad.cpu().clone() for p in net.parameters()]))
    Fn.WAVEFRONT_CHUNKS = int(__import__("os").environ.get("EDGEDICT_WAVEFRONT_CHUNKS", "6"))
    (y0, h0, c0, dx0, g0), (y1, h1, c1, dx1, g1) = res
    assert y0.shape == y1.shape
    assert rel_err(y1, y0) < 1e-5 and rel_err(h1, h0) < 1e-5 and rel_err(c1, c0) < 1e-5
    assert rel_err(dx1, dx0) < 2e-3
    for a, b, (name, _) in zip(g1, g0, net.named_parameters()):
        assert rel_err(a, b) < 2e-3, name
