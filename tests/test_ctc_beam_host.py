"""CTC prefix beam search without a GPU: every malformed argument of edgedict_b200.ctc.beam_search and
CTCEncoder.beam_search is refused on the host before any device work, and the CPU restatement (tests/ctc_beam_oracle.py)
equals a brute-force enumeration of prefixes when the beam holds them all."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import ctc_beam_oracle as cbo


def _lp(B=2, T=5, V=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, V, generator=g).log_softmax(-1)


@pytest.mark.parametrize("kw, exc", [
    (dict(log_probs=[[0.0]]), TypeError),
    (dict(log_probs=_lp().double()), TypeError),
    (dict(log_probs=_lp()[0]), ValueError),
    (dict(log_probs=torch.zeros(2, 0, 4)), ValueError),
    (dict(beam_width=0), ValueError),
    (dict(beam_width=1025), ValueError),
    (dict(beam_width=2.0), TypeError),
    (dict(beam_width=True), TypeError),
    (dict(blank=4), ValueError),
    (dict(blank=-1), ValueError),
    (dict(input_lengths=[5]), ValueError),
    (dict(input_lengths=[5, 6]), ValueError),
    (dict(input_lengths=[5, -1]), ValueError),
    (dict(input_lengths=torch.tensor([5.0, 5.0])), TypeError),
    (dict(lm_weight=0.5), ValueError),                           # fusion arguments need an lm
    (dict(lm_token_map=torch.arange(4)), ValueError),
    (dict(), RuntimeError),                                      # CPU log_probs: there is no CPU path
])
def test_beam_search_rejects_bad_arguments_on_the_host(kw, exc):
    from edgedict_b200 import ctc
    a = dict(log_probs=_lp(), input_lengths=[5, 3], beam_width=4, blank=0)
    a.update(kw)
    with pytest.raises(exc):
        ctc.beam_search(a.pop("log_probs"), a.pop("input_lengths"), a.pop("beam_width"), **a)


def test_beam_search_checks_the_lm_on_the_host():
    from edgedict_b200 import ctc
    lm = {"encoder.weight": torch.zeros(4, 3)}
    with pytest.raises(ValueError):
        ctc.beam_search(_lp(), [5, 5], 4, lm=lm)
    with pytest.raises(TypeError):
        ctc.beam_search(_lp(), [5, 5], 4, lm=object())


def test_ctc_encoder_beam_search_checks_before_the_forward():
    from edgedict_b200.rnnt.models import CTCEncoder
    m = CTCEncoder(vocab_size=6, input_size=4, enc_hidden_size=8, enc_layers=1, enc_dropout=0.0, proj_size=4)
    xs = torch.randn(1, 3, 4)
    with pytest.raises(ValueError):
        m.beam_search(xs, W=0)
    with pytest.raises(ValueError):
        m.beam_search(xs, W=2, length_bonus=1.0)


@pytest.mark.parametrize("V, T, blank", [(2, 6, 0), (3, 6, 0), (3, 5, 2), (4, 4, 1)])
def test_restatement_without_pruning_equals_brute_force(V, T, blank):
    """With W >= the number of prefixes nothing is pruned: every prefix of at most T tokens is in the final beam with
    exp(pb (+) pnb) = P(prefix), the CTC forward probability (and F.ctc_loss), and the best is the brute-force argmax."""
    y = _lp(1, T, V, seed=V * 10 + T)[0].double()
    prefixes = cbo.all_prefixes(V, T, blank)
    W = len(prefixes)
    seq, nscore, beam, _ = cbo.prefix_beam_search(y.numpy(), T, W, blank)
    got = {p: np.logaddexp(pb, pnb) for p, pb, pnb, _ in beam}
    assert len(beam) == W and set(got) == set(prefixes)
    want = {p: cbo.prefix_logprob(y.numpy(), p, blank) for p in prefixes}
    close = lambda a, b: a == b or abs(a - b) <= 1e-10 * (1 + abs(b))      # infeasible prefixes: -inf on both sides
    for p in prefixes:
        assert close(got[p], want[p]), (p, got[p], want[p])
        if p:
            ref = -F.ctc_loss(y[:, None], torch.tensor([p]), [T], [len(p)], blank=blank, reduction="none")
            assert close(float(ref), want[p])
    best = max(prefixes, key=lambda p: want[p])
    assert seq == best and abs(-nscore - want[best]) <= 1e-10 * (1 + abs(want[best]))


def test_restatement_fp32_follows_fp64():
    lp = _lp(3, 12, 7, seed=5)
    a_ids, a_s, _ = cbo.batch_search(lp.numpy(), [12, 9, 0], 4, 0, dtype=np.float64)
    b_ids, b_s, _ = cbo.batch_search(lp.numpy(), [12, 9, 0], 4, 0, dtype=np.float32)
    assert all(np.array_equal(a, b) for a, b in zip(a_ids, b_ids))
    assert np.allclose(a_s, b_s, rtol=1e-5) and a_s[2] == 0 and len(a_ids[2]) == 0


def test_restatement_merges_repeated_prefixes():
    """A peaked utterance 'a a _ a': the extension of 'a' by 'a' (via blank) must fold into an existing beam entry."""
    V, T = 3, 8
    y = np.full((T, V), np.log(0.05))
    for t, k in enumerate([1, 1, 0, 1, 2, 2, 0, 1]):
        y[t, k] = np.log(0.9)
    _, _, _, merges = cbo.prefix_beam_search(y, T, 8, 0)
    assert sum(m > 0 for m in merges[1:]) >= T - 2


def test_free_beam_search_releases_the_resident_engine():
    from edgedict_b200 import ctc
    ctc._beam_engines["k"] = object()
    ctc.free_beam_search()
    assert ctc._beam_engines == {}
