"""The GRU encoder on the engine (functional.GRULayer, ResLayerNormGRU): one layer against torch.nn.GRU in fp64 on the
CPU, and the whole Transducer(module_type='GRU') against oracle.model_torch.encoder_gru + the oracle's predictor, joint
and loss, in fp32 and bf16 mode."""
import pytest
import torch

from tests.util import rel_err

pytestmark = pytest.mark.gpu

f64 = torch.float64
TINY = dict(vocab_embed_size=16, vocab_size=64, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0,
            enc_proj_size=40, dec_hidden_size=32, dec_layers=1, dec_dropout=0, dec_proj_size=24, joint_size=56)
E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
            enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0, dec_proj_size=256, joint_size=640)


def _norm_err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a.norm() - b.norm()).abs() / (b.norm() + 1e-30))


# ---- one layer against nn.GRU ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("I,H,B,T,carry", [(24, 48, 3, 17, True), (64, 64, 5, 37, False), (96, 256, 32, 40, True),
                                           (256, 1024, 2, 23, True)])
def test_gru_layer_matches_nn_gru_fp64(precision, I, H, B, T, carry):
    from edgedict_b200 import functional as Fn
    torch.manual_seed(H + T)
    ref = torch.nn.GRU(I, H, 1, batch_first=True).double()
    with torch.no_grad():
        ref.bias_hh_l0.uniform_(-1, 1)                         # b_hn matters: make it as large as the rest
    x = torch.randn(B, T, I, dtype=f64)
    h0 = torch.randn(B, H, dtype=f64) * 0.5 if carry else None
    gy = torch.randn(B, T, H, dtype=f64)
    ghT = torch.randn(B, H, dtype=f64) if carry else None
    # fp64 CPU reference
    xr = x.clone().requires_grad_()
    h0r = h0.clone().requires_grad_() if carry else None
    yr, hr = ref(xr, None if h0r is None else h0r[None])
    lr = (yr * gy).sum() + ((hr[0] * ghT).sum() if carry else 0)
    lr.backward()
    # engine
    params = [p.detach().float().cuda().requires_grad_() for p in
              (ref.weight_ih_l0, ref.weight_hh_l0, ref.bias_ih_l0, ref.bias_hh_l0)]
    xe = x.float().cuda().requires_grad_()
    h0e = h0.float().cuda().requires_grad_() if carry else None
    ye, he = Fn.GRULayer.apply(xe, h0e, *params, precision)
    le = (ye * gy.float().cuda()).sum() + ((he * ghT.float().cuda()).sum() if carry else 0)
    le.backward()
    got = dict(y=ye, hT=he, dx=xe.grad, dw_ih=params[0].grad, dw_hh=params[1].grad, db_ih=params[2].grad,
               db_hh=params[3].grad)
    want = dict(y=yr, hT=hr[0], dx=xr.grad, dw_ih=ref.weight_ih_l0.grad, dw_hh=ref.weight_hh_l0.grad,
                db_ih=ref.bias_ih_l0.grad, db_hh=ref.bias_hh_l0.grad)
    if carry:
        got["dh0"], want["dh0"] = h0e.grad, h0r.grad
    for k in got:
        e = rel_err(got[k].detach().cpu(), want[k].detach())
        print("  GRULayer %s I=%d H=%d B=%d T=%d %-6s max err / max |ref| %.3g, norm %.3g"
              % (precision, I, H, B, T, k, e, _norm_err(got[k].detach(), want[k].detach())))
        if precision == "fp32":
            assert e < 1e-4, k
        else:
            assert e < 3e-2 and _norm_err(got[k].detach(), want[k].detach()) < 2e-2, k


def test_gru_layer_refuses_a_second_backward():
    from edgedict_b200 import functional as Fn
    H = 64
    params = [(torch.randn(*s, device="cuda") * 0.1).requires_grad_() for s in ((3 * H, 32), (3 * H, H), (3 * H,),
                                                                                (3 * H,))]
    x = torch.randn(2, 5, 32, device="cuda", requires_grad=True)
    y, _ = Fn.GRULayer.apply(x, None, *params, "fp32")
    y.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="twice"):
        y.sum().backward()


# ---- the whole model against the oracle -----------------------------------------------------------------------------
def _model(cfg, seed, precision):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(seed)
    m = Transducer(module_type="GRU", **cfg).cuda()
    m.set_precision(precision)
    return m


def _oracle_loss_and_grads(m, xs, ys, xlen, ylen):
    from oracle import model_torch as mt
    sd = {k: v.detach().cpu().double().requires_grad_() for k, v in m.state_dict().items()}
    x = xs[:, :int(xlen.max())].double()
    y = ys[:, :int(ylen.max())]
    h_enc, _ = mt.encoder_gru(sd, x)
    h_dec, _ = mt.decoder(sd, y)
    logits = mt.joint(sd, h_enc, h_dec)
    xl = mt.scale_length(logits.shape[1], xlen)
    loss = mt.rnnt_loss(logits, y.int(), xl, ylen.int(), 0, "mean", use_ref=False)
    loss.backward()
    return loss.detach(), h_enc.detach(), {k: v.grad for k, v in sd.items() if v.grad is not None}


def _inputs(cfg, B, T, U, xlen, ylen, seed):
    g = torch.Generator().manual_seed(seed)
    xs = torch.randn(B, T, cfg["input_size"], generator=g)
    ys = torch.randint(1, cfg["vocab_size"], (B, U), generator=g, dtype=torch.int32)
    return xs, ys, torch.tensor(xlen), torch.tensor(ylen)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("dims", ["tiny", "e6d2"])
def test_transducer_gru_loss_and_gradients_match_oracle(precision, dims):
    if dims == "tiny":
        cfg, B, T, U, xlen, ylen = TINY, 3, 23, 6, [23, 17, 9], [6, 4, 2]
    else:
        cfg, B, T, U, xlen, ylen = E6D2, 2, 200, 32, [200, 157], [32, 21]
    m = _model(cfg, 5, precision)
    xs, ys, xl, yl = _inputs(cfg, B, T, U, xlen, ylen, 7)
    want_loss, want_enc, want_g = _oracle_loss_and_grads(m, xs, ys, xl, yl)
    loss = m(xs.cuda(), ys.cuda(), xl, yl)
    loss.backward()
    with torch.no_grad():
        h_enc, _ = m.encoder(xs[:, :int(xl.max())].cuda())
    el = rel_err(loss.detach().cpu(), want_loss)
    ee = rel_err(h_enc.cpu(), want_enc)
    print("  Transducer GRU %s %s: loss %.3g, h_enc %.3g" % (dims, precision, el, ee))
    worst = (0.0, "")
    for k, p in m.named_parameters():
        e = rel_err(p.grad.cpu(), want_g[k]) if precision == "fp32" else _norm_err(p.grad, want_g[k])
        worst = max(worst, (e, k))
        if precision == "fp32":
            assert e < 1e-3, k
        else:
            assert e < 2e-2, k
    print("  worst gradient error %.3g (%s)" % worst)
    if precision == "fp32":
        assert el < 1e-4 and ee < 1e-3
    else:
        assert el < 1e-3


def test_gru_encoder_carried_hiddens_match_oracle():
    from oracle import model_torch as mt
    m = _model(TINY, 9, "fp32").eval()
    xs = torch.randn(2, 11, TINY["input_size"])
    h_in = torch.randn(TINY["enc_layers"], 2, TINY["enc_hidden_size"]) * 0.5
    with torch.no_grad():
        out, hs = m.encoder(xs.cuda(), h_in.cuda())
    sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    ref, rh = mt.encoder_gru(sd, xs.double(), h_in.double())
    assert hs.shape == (TINY["enc_layers"], 2, TINY["enc_hidden_size"])
    assert rel_err(out.cpu(), ref) < 1e-5 and rel_err(hs.cpu(), rh) < 1e-5
    # a chunk fed with the state of the previous chunk continues the sequence (even lengths: the time reduction pairs
    # the same frames)
    xa, xb = torch.randn(2, 12, TINY["input_size"]).cuda(), torch.randn(2, 12, TINY["input_size"]).cuda()
    with torch.no_grad():
        full, hf = m.encoder(torch.cat([xa, xb], 1))
        first, h1 = m.encoder(xa)
        second, h2 = m.encoder(xb, h1)
    assert rel_err(torch.cat([first, second], 1).cpu(), full.cpu()) < 1e-5
    assert rel_err(h2.cpu(), hf.cpu()) < 1e-5


def test_gru_gradients_are_bitwise_repeatable():
    runs = []
    for _ in range(2):
        m = _model(TINY, 11, "fp32")
        xs, ys, xl, yl = _inputs(TINY, 3, 23, 6, [23, 17, 9], [6, 4, 2], 13)
        m(xs.cuda(), ys.cuda(), xl, yl).backward()
        runs.append({k: p.grad.clone() for k, p in m.named_parameters()})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_gru_beam_width_one_is_greedy_decode():
    m = _model(TINY, 17, "fp32").eval()
    xs = torch.randn(3, 23, TINY["input_size"]).cuda()
    full = torch.full((3,), 23)
    ids, nlp = m.greedy_decode(xs, full)
    seqs, blp = m.beam_search(xs, None, W=1)
    for got, want in zip(seqs, ids):
        assert got == [int(t) for t in want if t != 0]
    assert rel_err(blp.cpu(), nlp.cpu()) < 1e-4


def test_stream_engine_refuses_a_gru_encoder():
    from edgedict_b200.stream_engine import StreamEngine
    m = _model(TINY, 19, "fp32").eval()
    with pytest.raises(ValueError, match="LSTM"):
        StreamEngine(m, 2, 2)
