"""The language model without a GPU: the fp64 restatement of a training step (tests/lm_train_oracle.py) against the
reference's own LMModel (tests/golden/lm_train_tiny.npz, lm_tiny.npz), the engine's LMModel construction against the
reference's seeded weights, the refusals of ``LMModel`` / ``LMModel.loss`` before any device work, and the argument
checks of the C entries."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import lm_train_oracle as lo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VARIANTS = {"u": dict(ninp=8, nhid=12, seed=5, tie_weights=False), "t": dict(ninp=12, nhid=12, seed=6, tie_weights=True)}


def fixture(tag):
    z = np.load(os.path.join(GOLDEN, "lm_train_tiny.npz"))
    p = tag + ".sd."
    sd = {k[len(p):]: z[k] for k in z.files if k.startswith(p)}
    p = tag + ".grad."
    grads = {k[len(p):]: z[k] for k in z.files if k.startswith(p)}
    return z, sd, grads


@pytest.mark.parametrize("tag", ["u", "t"])
def test_restatement_reproduces_the_reference_forward(tag):
    z, sd, _ = fixture(tag)
    logp, (h, c), _ = lo.forward(sd, z["inputs"])
    np.testing.assert_allclose(logp, z[tag + ".logp"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(h, z[tag + ".h"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(c, z[tag + ".c"], rtol=0, atol=1e-6)
    logp, (h, c), _ = lo.forward(sd, z["inputs"], (z[tag + ".h0"], z[tag + ".c0"]))
    np.testing.assert_allclose(logp, z[tag + ".logp_h0"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(h, z[tag + ".h_h0"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(c, z[tag + ".c_h0"], rtol=0, atol=1e-6)


@pytest.mark.parametrize("tag", ["u", "t"])
def test_restatement_reproduces_the_reference_loss_and_gradients(tag):
    z, sd, grads = fixture(tag)
    assert (z["targets"] == 0).any(), "the padded batch must exercise ignore_index"
    loss, got = lo.loss_and_grads(sd, z["inputs"], z["targets"], tied=tag == "t")
    assert abs(loss - float(z[tag + ".loss"])) < 1e-6
    assert set(got) == set(grads)
    for k, g in grads.items():
        np.testing.assert_allclose(got[k], g, rtol=0, atol=1e-6 * max(1.0, np.abs(g).max()), err_msg=k)


def test_restatement_nll_matches_torch():
    g = torch.Generator().manual_seed(0)
    logp = torch.log_softmax(torch.randn(9, 7, generator=g, dtype=torch.float64), -1)
    t = torch.tensor([0, 3, 6, 0, 1, 2, 5, 4, 0])
    for red in ("mean", "sum", "none"):
        want = torch.nn.NLLLoss(ignore_index=0, reduction=red)(logp, t).numpy()
        np.testing.assert_allclose(lo.nll(logp.numpy(), t.numpy(), 0, red), want, rtol=1e-15, atol=0)


@pytest.mark.parametrize("tag", ["u", "t"])
def test_construction_under_the_seed_gives_the_reference_weights(tag):
    from edgedict_b200.models import LMModel
    z, sd, _ = fixture(tag)
    v = VARIANTS[tag]
    torch.manual_seed(v["seed"])
    m = LMModel(int(z["ntoken"]), v["ninp"], v["nhid"], 2, dropout=0.0, tie_weights=v["tie_weights"])
    got = m.state_dict()
    assert list(got) == [str(k) for k in z[tag + ".keys"]]
    for k, t in got.items():
        assert np.array_equal(t.numpy(), sd[k]), k
    if v["tie_weights"]:
        assert m.decoder.weight is m.encoder.weight
    assert [k for k, _ in m.named_parameters()] == sorted(fixture(tag)[2], key=list(got).index)


def test_construction_matches_the_fusion_fixture():
    from edgedict_b200.models import LMModel
    z = np.load(os.path.join(GOLDEN, "lm_tiny.npz"))
    torch.manual_seed(77)
    m = LMModel(16, 6, 10, 2, dropout=0.5)
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(4.0)
    for k, t in m.state_dict().items():
        assert np.array_equal(t.numpy(), z["sd." + k]), k


def test_interface_surface():
    from edgedict_b200.models import LMModel
    from edgedict_b200.stream_engine import lm_state_dict
    with pytest.raises(ValueError):
        LMModel(10, 8, 12, 2, tie_weights=True)
    m = LMModel(10, 8, 12, 3, dropout=0.25)
    assert (m.ntoken, m.nhid, m.nlayers, m.rnn_type) == (10, 12, 3, "LSTM")
    assert m.drop.p == 0.25 and m.rnn.dropout == 0.25 and m.rnn.batch_first and m.encoder.padding_idx is None
    h, c = m.init_hidden(5)
    assert h.shape == c.shape == (3, 5, 12) and not h.any() and not c.any()
    sd = lm_state_dict(m)                                # accepted as a fusion LM as it stands
    assert set(sd) == set(m.state_dict())
    assert m.set_precision("bf16") is m and m.precision == "bf16"


@pytest.mark.parametrize("bad, exc", [
    (dict(reduction="batchmean"), ValueError),
    (dict(targets=torch.zeros(2, 3)), TypeError),
    (dict(targets=[[1, 2, 3], [1, 2, 3]]), TypeError),
    (dict(targets=torch.zeros(2, 4, dtype=torch.long)), ValueError),
    (dict(ignore_index=0.5), TypeError),
])
def test_loss_refuses_bad_arguments_before_the_device(bad, exc):
    from edgedict_b200.models import LMModel
    m = LMModel(10, 8, 8, 1, dropout=0.0)
    a = dict(input=torch.ones(2, 3, dtype=torch.long), targets=torch.ones(2, 3, dtype=torch.long))
    a.update(bad)
    with pytest.raises(exc):
        m.loss(**a)


def test_cpu_module_is_refused():
    from edgedict_b200.models import LMModel
    m = LMModel(10, 8, 8, 1, dropout=0.0)
    with pytest.raises(RuntimeError):
        m.loss(torch.ones(2, 3, dtype=torch.long), torch.ones(2, 3, dtype=torch.long))


def test_entry_points_refuse_bad_arguments_before_touching_the_device():
    from edgedict_b200._lib import lib
    L = lib()
    fk = ctypes.c_void_p(256)                # never dereferenced: every call below must return before any launch
    al = ctypes.c_void_p(4096)               # 16-byte aligned, for the checks that come after the alignment rule
    mis = ctypes.c_void_p(4104)

    def ce(**kw):
        a = dict(h=al, w=al, b=al, o=al, t=fk, t64=0, lse=fk, tl=fk, M=8, V=16, K=16)
        a.update(kw)
        return L.eb_lm_logits_ce(a["h"], a["w"], a["b"], a["o"], a["t"], a["t64"], a["lse"], a["tl"], a["M"], a["V"],
                                 a["K"], None)

    for kw in (dict(K=12), dict(K=0), dict(M=0), dict(V=0), dict(h=None), dict(w=None), dict(o=None), dict(t=None),
               dict(lse=None), dict(tl=None), dict(h=mis), dict(w=mis), dict(b=ctypes.c_void_p(4100)),
               dict(o=ctypes.c_void_p(4098)), dict(M=1 << 31)):
        assert ce(**kw) == 2, kw

    assert L.eb_lm_ce_rows(None, fk, 0, fk, fk, 8, 16, None) == 2
    assert L.eb_lm_ce_rows(fk, None, 0, fk, fk, 8, 16, None) == 2
    assert L.eb_lm_ce_rows(fk, fk, 0, fk, fk, 8, 0, None) == 2
    assert L.eb_lm_ce_rows(fk, fk, 0, fk, fk, -1, 16, None) == 2
    assert L.eb_lm_ce_rows(fk, fk, 0, fk, fk, 0, 16, None) == 0          # nothing to do, nothing launched

    def loss(**kw):
        a = dict(lse=fk, tl=fk, t=fk, M=8, V=16, loss=fk, scale=fk)
        a.update(kw)
        return L.eb_lm_ce_loss(a["lse"], a["tl"], a["t"], 0, 0, a["M"], a["V"], 1, None, a["loss"], a["scale"], None)

    for kw in (dict(lse=None), dict(tl=None), dict(t=None), dict(loss=None), dict(scale=None), dict(M=-1), dict(V=0)):
        assert loss(**kw) == 2, kw

    def bwd(**kw):
        a = dict(l=fk, d=fk, lse=fk, t=fk, M=8, V=16, g=fk)
        a.update(kw)
        return L.eb_lm_ce_bwd(a["l"], a["d"], 1, a["lse"], a["t"], 0, 0, a["M"], a["V"], a["g"], 0, None, None)

    for kw in (dict(l=None), dict(d=None), dict(lse=None), dict(t=None), dict(g=None), dict(M=-1), dict(V=0)):
        assert bwd(**kw) == 2, kw
    assert bwd(M=0) == 0


def test_bf16_mode_refuses_vocabularies_its_gemm_cannot_take():
    from edgedict_b200.models import LMModel
    m = LMModel(10, 8, 8, 1, dropout=0.0).set_precision("bf16")
    with pytest.raises(ValueError):
        m.loss(torch.ones(2, 3, dtype=torch.long), torch.ones(2, 3, dtype=torch.long))
