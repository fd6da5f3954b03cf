"""Shallow fusion of the reference's LSTM language model without a GPU: the LM restatement against the reference's
own LMModel (tests/golden/lm_tiny.npz), the fused restatement of the beam at zero weights, the argument checks of
Transducer.beam_search (before any device work) and the EbPhase layout the decode kernel shares with ctypes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import lm_oracle as lo
from tests.util import load_tiny

HERE = os.path.dirname(os.path.abspath(__file__))
SMALL = dict(vocab_embed_size=32, vocab_size=96, input_size=40, enc_hidden_size=64, enc_layers=2, enc_dropout=0.0,
             enc_proj_size=80, dec_hidden_size=64, dec_layers=2, dec_dropout=0.0, dec_proj_size=72, joint_size=88)


def load_lm():
    z = np.load(os.path.join(HERE, "golden", "lm_tiny.npz"))
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd.")}
    return z, sd


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_lm_step_reproduces_the_reference(dtype):
    z, sd = load_lm()
    sd = {k: v.to(dtype) for k, v in sd.items()}
    toks = torch.from_numpy(z["tokens"]).long()
    B, U = toks.shape
    L, H = z["h"].shape[0], z["h"].shape[2]
    h = c = torch.zeros(L, B, H, dtype=dtype)
    for u in range(U):
        lp, (h, c) = lo.lm_step(sd, toks[:, u], (h, c))
        np.testing.assert_allclose(lp.numpy(), z["logp"][:, u], rtol=0, atol=1e-6)
    np.testing.assert_allclose(h.numpy(), z["h"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(c.numpy(), z["c"], rtol=0, atol=1e-6)


def _lm_for_tiny():
    """The fixture LM over the tiny transducer's 16 tokens."""
    _, sd = load_lm()
    return sd


@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 4, 20])
def test_restatement_at_zero_weights_is_the_plain_beam(W, merge):
    from oracle import model_torch as mt
    z, cfg, sd, _ = load_tiny()
    sd = {k: torch.as_tensor(v) for k, v in sd.items()}
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    want, wlp = mt.beam_search(sd, xs, xlen, W=W, merge=merge)
    got, glp = lo.beam_search(sd, xs, xlen, W=W, merge=merge, lm_sd=_lm_for_tiny(), lm_weight=0.0, length_bonus=0.0)
    assert got == want
    assert torch.equal(glp, wlp)
    # and the LM does move the result once it has weight
    got2, glp2 = lo.beam_search(sd, xs, xlen, W=W, merge=merge, lm_sd=_lm_for_tiny(), lm_weight=1.0, length_bonus=0.5)
    assert got2 != want or not torch.equal(glp2, wlp)


def _cpu_model():
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(0)
    return Transducer(output_loss=False, **SMALL)


def _lm_sd(ntok=96, ninp=8, nhid=12, L=2):
    g = torch.Generator().manual_seed(5)
    r = lambda *s: torch.randn(*s, generator=g)
    sd = {"encoder.weight": r(ntok, ninp), "decoder.weight": r(ntok, nhid), "decoder.bias": r(ntok)}
    for k in range(L):
        sd.update({"rnn.weight_ih_l%d" % k: r(4 * nhid, ninp if k == 0 else nhid),
                   "rnn.weight_hh_l%d" % k: r(4 * nhid, nhid), "rnn.bias_ih_l%d" % k: r(4 * nhid),
                   "rnn.bias_hh_l%d" % k: r(4 * nhid)})
    return sd


class _LM(torch.nn.Module):
    def __init__(self, ntok=96, ninp=8, nhid=12, L=2, **lstm_kw):
        super().__init__()
        self.encoder = torch.nn.Embedding(ntok, ninp)
        self.rnn = torch.nn.LSTM(ninp, nhid, L, **dict(dict(batch_first=True), **lstm_kw))
        self.decoder = torch.nn.Linear(nhid, ntok)


def _drop(sd, k):
    sd = dict(sd)
    del sd[k]
    return sd


def _with(sd, k, v):
    sd = dict(sd)
    sd[k] = v
    return sd


BAD = [
    ("not a module", dict(lm=[1, 2]), TypeError),
    ("module without an LSTM", dict(lm=torch.nn.Linear(3, 3)), TypeError),
    ("not batch_first", dict(lm=_LM(batch_first=False)), ValueError),
    ("bidirectional", dict(lm=_LM(bidirectional=True)), ValueError),
    ("proj_size", dict(lm=_LM(proj_size=4)), ValueError),
    ("output over other tokens", dict(lm=_with(_lm_sd(), "decoder.weight", torch.zeros(90, 12))), ValueError),
    ("missing key", dict(lm=_drop(_lm_sd(), "rnn.bias_hh_l1")), ValueError),
    ("extra key", dict(lm=_with(_lm_sd(), "rnn.weight_hr_l0", torch.zeros(12, 12))), ValueError),
    ("no layer", dict(lm={"encoder.weight": torch.zeros(96, 8), "decoder.weight": torch.zeros(96, 12),
                          "decoder.bias": torch.zeros(96)}), ValueError),
    ("wrong hidden shape", dict(lm=_with(_lm_sd(), "rnn.weight_hh_l1", torch.zeros(48, 11))), ValueError),
    ("wrong input size", dict(lm=_with(_lm_sd(), "rnn.weight_ih_l0", torch.zeros(48, 9))), ValueError),
    ("integer weights", dict(lm=_with(_lm_sd(), "decoder.bias", torch.zeros(96, dtype=torch.int64))), TypeError),
    ("ntoken != V without a map", dict(lm=_lm_sd(ntok=50)), ValueError),
    ("map of the wrong length", dict(lm=_lm_sd(ntok=50), lm_token_map=torch.zeros(95, dtype=torch.int64)),
     ValueError),
    ("map out of range", dict(lm=_lm_sd(ntok=50), lm_token_map=torch.full((96,), 50)), ValueError),
    ("map below -1", dict(lm=_lm_sd(ntok=50), lm_token_map=torch.full((96,), -2)), ValueError),
    ("float map", dict(lm=_lm_sd(ntok=50), lm_token_map=torch.zeros(96)), TypeError),
    ("lm_weight inf", dict(lm=_lm_sd(), lm_weight=float("inf")), ValueError),
    ("lm_weight nan", dict(lm=_lm_sd(), lm_weight=float("nan")), ValueError),
    ("length_bonus -inf", dict(lm=_lm_sd(), length_bonus=float("-inf")), ValueError),
    ("lm_weight a string", dict(lm=_lm_sd(), lm_weight="1"), TypeError),
    ("lm_bos = ntoken", dict(lm=_lm_sd(), lm_bos=96), ValueError),
    ("lm_bos negative", dict(lm=_lm_sd(), lm_bos=-1), ValueError),
    ("lm_bos a float", dict(lm=_lm_sd(), lm_bos=1.0), TypeError),
    ("weights without an lm", dict(lm_weight=0.5), ValueError),
    ("map without an lm", dict(lm_token_map=torch.arange(96)), ValueError),
]


@pytest.mark.parametrize("what,kw,exc", BAD, ids=[b[0] for b in BAD])
def test_beam_search_lm_arguments_checked_before_any_device_work(what, kw, exc):
    """A CPU model gets the argument error, not the encoder's or a device error."""
    m = _cpu_model()
    xs = torch.zeros(1, 4, SMALL["input_size"])
    with pytest.raises(exc):
        m.beam_search(xs, None, W=2, **kw)


def test_good_lm_arguments_pass_the_checks():
    from edgedict_b200.stream_engine import check_lm_args
    for lm in (_lm_sd(), _LM(), _LM(L=1)):
        sd, lw, lb, bos, tmap = check_lm_args(lm, 96, 0.5, 1, 1, None)
        assert (lw, lb, bos) == (0.5, 1.0, 1) and torch.equal(tmap, torch.arange(96))
    tm = torch.full((96,), -1, dtype=torch.int32)
    tm[4:54] = torch.arange(50)
    assert torch.equal(check_lm_args(_lm_sd(ntok=50), 96, 0.0, 0.0, 49, tm)[4], tm.long())
    assert check_lm_args(None, 96, 0.0, 0.0, 1, None) is None


def test_ebphase_layout_matches_the_library():
    from edgedict_b200 import build
    from edgedict_b200._lib import lib
    from edgedict_b200.stream_engine import EbPhase
    build.build()
    assert C.sizeof(EbPhase) == lib().eb_decode_phase_size()
    assert C.sizeof(EbPhase) % 4 == 0 and C.sizeof(EbPhase) // 4 <= 256    # the kernel's word-per-thread loader
