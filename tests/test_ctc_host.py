"""CTCEncoder's parameters and the CTC argument checks, without a GPU: the state_dict keys, shapes and GRU layout equal the
reference's (tests/golden/ctc_tiny.npz), and every malformed argument is refused on the host (Python) or by the C ABI
before anything is launched."""
import ctypes

import pytest
import torch

from tests.test_oracle_ctc import load_ctc_tiny


def test_ctc_encoder_state_dict_matches_reference():
    from edgedict_b200.rnnt.models import CTCEncoder, ResLayerNormGRU
    _, cfg, sd = load_ctc_tiny()
    m = CTCEncoder(**cfg)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == {k: tuple(v.shape) for k, v in sd.items()}
    assert isinstance(m.model.lstm, ResLayerNormGRU)
    H = cfg["enc_hidden_size"]
    assert got["model.lstm.lstms.0.weight_hh_l0"] == (3 * H, H)          # GRU gates r|z|n, not the LSTM's 4H
    assert list(m.tovocab[0].weight.shape) == [cfg["vocab_size"], cfg["proj_size"]]
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})    # a reference checkpoint loads strictly


def test_encoder_default_module_is_unchanged():
    from edgedict_b200.rnnt.models import Encoder, ResLayerNormLSTM
    assert isinstance(Encoder(8, 16, 1, 0, 8).lstm, ResLayerNormLSTM)


def _args(**kw):
    T, N, V, S = 6, 2, 5, 3
    a = dict(log_probs=torch.randn(T, N, V).log_softmax(-1), targets=torch.randint(1, V, (N, S)),
             input_lengths=[T, T - 1], target_lengths=[S, 2], blank=0, reduction="mean")
    a.update(kw)
    return a


@pytest.mark.parametrize("bad, exc", [
    (dict(log_probs=torch.randn(6, 2, 5, dtype=torch.float64)), TypeError),
    (dict(log_probs=torch.randn(6, 2, 5).half()), TypeError),
    (dict(log_probs=torch.randn(6, 2, 5, 1)), ValueError),
    (dict(log_probs=torch.randn(6)), ValueError),
    (dict(log_probs=torch.randn(0, 2, 5)), ValueError),
    (dict(targets=torch.ones(2, 3)), TypeError),
    (dict(targets=torch.ones(2, 3, 1, dtype=torch.long)), ValueError),
    (dict(targets=torch.ones(3, 3, dtype=torch.long)), ValueError),
    (dict(target_lengths=[4, 2]), ValueError),                           # above the padded length
    (dict(target_lengths=[-1, 2]), ValueError),
    (dict(target_lengths=[3]), ValueError),
    (dict(target_lengths=torch.tensor([3.0, 2.0])), TypeError),
    (dict(input_lengths=[7, 6]), ValueError),                            # above T
    (dict(input_lengths=[6, -1]), ValueError),
    (dict(input_lengths=[6, 6, 6]), ValueError),
    (dict(targets=torch.ones(6, dtype=torch.long)), ValueError),         # concatenated: 6 labels, lengths sum to 5
    (dict(blank=5), ValueError),
    (dict(blank=-1), ValueError),
    (dict(reduction="avg"), ValueError),
    (dict(log_probs=torch.randn(6, 5), targets=torch.ones(2, 3, dtype=torch.long), input_lengths=6, target_lengths=3),
     ValueError),                                                        # unbatched input, batched targets
    (dict(log_probs=torch.randn(1100, 1, 5), targets=torch.ones(1, 1024, dtype=torch.long), input_lengths=[1100],
          target_lengths=[1024]), ValueError),                           # S >= 1024
    (dict(), RuntimeError),                                              # a valid call on CPU tensors: no CPU path
])
def test_ctc_loss_refuses_bad_arguments_on_the_host(bad, exc):
    from edgedict_b200.ctc import ctc_loss
    with pytest.raises(exc):
        ctc_loss(**_args(**bad))


def test_ctc_loss_module_and_unbatched_reach_the_device_check():
    from edgedict_b200.ctc import CTCLoss
    with pytest.raises(RuntimeError, match="CUDA"):
        CTCLoss(blank=1, reduction="sum")(torch.randn(6, 5), torch.tensor([2, 3]), 6, 2)
    with pytest.raises(RuntimeError, match="CUDA"):        # concatenated targets, S = 1023 is accepted
        CTCLoss()(torch.randn(2100, 1, 5), torch.ones(1023, dtype=torch.long), [2100], [1023])


def test_ctc_entry_points_refuse_bad_arguments_before_touching_the_device():
    from edgedict_b200._lib import lib
    L = lib()
    fake = ctypes.c_void_p(256)          # never dereferenced: every call below must return before any launch
    assert L.eb_ctc_workspace_size(2, 10, 1024) == 0
    assert L.eb_ctc_workspace_size(0, 10, 3) == 0
    assert L.eb_ctc_workspace_size(2, 10, 1023) > 0

    def fwd(**kw):
        a = dict(lp=fake, N=2, T=10, V=5, targets=fake, nt=6, off=fake, tl=fake, il=fake, S=3, blank=0, ws=fake,
                 costs=fake)
        a.update(kw)
        return L.eb_ctc_loss_fwd(a["lp"], 5, 10, a["N"], a["T"], a["V"], a["targets"], a["nt"], a["off"], a["tl"],
                                 a["il"], a["S"], a["blank"], 0, a["ws"], a["costs"], None)

    for kw in (dict(S=1024), dict(S=-1), dict(blank=5), dict(blank=-1), dict(N=0), dict(N=70000), dict(T=-1),
               dict(V=0), dict(lp=None), dict(off=None), dict(tl=None), dict(il=None), dict(ws=None), dict(costs=None),
               dict(targets=None), dict(nt=-1)):
        assert fwd(**kw) == 2, kw

    def bwd(**kw):
        a = dict(lp=fake, g=ctypes.c_void_p(512), N=2, S=3, blank=0)
        a.update(kw)
        return L.eb_ctc_loss_bwd(a["lp"], 5, 10, a["g"], 5, 10, a["N"], 10, 5, fake, fake, a["S"], a["blank"], 0, fake,
                                 None, None)

    for kw in (dict(S=1024), dict(blank=7), dict(N=0), dict(g=None), dict(g=fake), dict(lp=None)):
        assert bwd(**kw) == 2, kw
    assert L.eb_ctc_greedy(fake, 50, 5, 0, 10, 5, fake, 0, fake, fake, fake, None) == 2
    assert L.eb_ctc_greedy(fake, 50, 5, 2, 10, 5, None, 0, fake, fake, fake, None) == 2
    assert L.eb_log_softmax_fwd(fake, fake, 4, 0, None) == 2
    assert L.eb_log_softmax_bwd(fake, None, fake, 4, 5, None) == 2
