"""N-best beam search without a GPU: the restatement (tests/nbest_oracle.py) against brute-force enumeration on tiny
problems where the beam prunes nothing, and every malformed ``nbest`` refused on the host before any device work."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import ctc_beam_oracle as cbo
from tests import nbest_oracle as no

TINY = dict(vocab_embed_size=8, vocab_size=4, input_size=6, enc_hidden_size=8, enc_layers=1, enc_dropout=0.0,
            enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0.0, dec_proj_size=8, joint_size=8)


def _lp(B=2, T=5, V=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, V, generator=g).log_softmax(-1)


def _tiny_transducer(seed):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(seed)
    m = Transducer(output_loss=False, **TINY).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(3.0)
    return {k: v.detach().double() for k, v in m.state_dict().items()}


# ---- the restatement against brute force ------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_ctc_oracle_is_every_prefix_by_exact_probability(seed):
    """V = 3, T = 4: 31 prefixes, W = 32 keeps them all.  The list is every prefix of non-zero probability, each
    scored by the CTC forward algorithm, ranked by it (the -inf candidates the beam also keeps rank last).  Without
    pruning a prefix enters the beam at the first frame it is a candidate, at -inf when it ends in a repeat, so token
    i entered at frame i; the path with those frames has log p at most the prefix's."""
    V, T = 3, 4
    y = _lp(1, T, V, seed)[0].double().numpy()
    got = no.ctc_nbest(y, T, 32, dtype=np.float64)
    prefixes = cbo.all_prefixes(V, T)
    exact = {p: cbo.prefix_logprob(y, p) for p in prefixes}
    reachable = [p for p in prefixes if np.isfinite(exact[p])]
    assert sorted(h[0] for h in got if np.isfinite(h[2])) == sorted(reachable)
    for tokens, frames, nlogp in got[:len(reachable)]:
        assert abs(-nlogp - exact[tokens]) < 1e-12 * max(1.0, abs(exact[tokens]))
        assert frames == tuple(range(len(tokens)))
        assert no.ctc_path_logprob(y, tokens, frames) <= exact[tokens] + 1e-12
    assert [h[2] for h in got] == sorted(h[2] for h in got)


def test_ctc_oracle_head_and_scores_are_prefix_beam_search():
    """The ranked list's head is prefix_beam_search's result, and the list is its final beam, in fp32 and with an LM."""
    from tests.test_oracle_lm import load_lm
    _, lsd = load_lm()
    lp = _lp(2, 6, 16, seed=3)
    for kw in ({}, dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5)):
        for W in (1, 3, 8):
            for b in range(2):
                got = no.ctc_nbest(lp[b].numpy(), 6 - 2 * b, W, **kw)
                seq, nlp, beam, _ = cbo.prefix_beam_search(lp[b].numpy(), 6 - 2 * b, W, dtype=np.float32, **kw)
                assert got[0][0] == seq and got[0][2] == nlp
                assert sorted(h[0] for h in got) == sorted(h[0] for h in beam)


@pytest.mark.parametrize("seed", [0, 1])
def test_transducer_oracle_is_every_sequence_by_exact_probability(seed):
    """V = 4 (3 tokens), T' = 3, K = 1 with merge and W = 64 >= the 40 reachable sequences: the list is every
    sequence of at most 3 tokens, each scored by the fp64 sum over its alignments, ranked by that score."""
    sd = _tiny_transducer(seed)
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(1, 3, TINY["enc_proj_size"], generator=g, dtype=torch.float64)
    got = no.transducer_nbest(sd, h, [3], 64, K=1, merge=True)[0]
    seqs = no.all_sequences(4, 3)
    assert sorted(x[0] for x in got) == sorted(seqs)
    for tokens, frames, nlogp in got:
        ref = no.transducer_sequence_logprob(sd, h[0], 3, tokens)
        assert abs(-nlogp - ref) < 1e-9, tokens
        assert all(0 <= f < 3 for f in frames) and list(frames) == sorted(set(frames))
        assert no.transducer_path_logprob(sd, h[0], 3, tokens, frames) <= ref + 1e-12
    nl = [x[2] for x in got]
    assert nl == sorted(nl)


def test_transducer_oracle_without_merge_scores_its_own_path():
    """merge = False, no LM, K = 1 and 2: each hypothesis is one lattice path, and its score is that path's log p."""
    sd = _tiny_transducer(4)
    g = torch.Generator().manual_seed(4)
    h = torch.randn(1, 4, TINY["enc_proj_size"], generator=g, dtype=torch.float64)
    for K in (1, 2):
        got = no.transducer_nbest(sd, h, [4], 6, K=K, merge=False)[0]
        assert len(got) == 6
        for tokens, frames, nlogp in got:
            assert abs(-nlogp - no.transducer_path_logprob(sd, h[0], 4, tokens, frames, K)) < 1e-9


def test_ctc_path_logprob_sums_to_the_prefix():
    """The brute-force path sum: over every frame assignment of a prefix the path probabilities add up to the CTC
    forward algorithm's."""
    import itertools
    y = _lp(1, 5, 3, 7)[0].double().numpy()
    for p in [(), (1,), (1, 2), (2, 2), (1, 2, 1)]:
        tot = [no.ctc_path_logprob(y, p, fr) for fr in itertools.combinations(range(5), len(p))]
        assert abs(np.logaddexp.reduce(tot + [-np.inf]) - cbo.prefix_logprob(y, p)) < 1e-12


# ---- refusals before device work -------------------------------------------------------------------------------------
BAD = [(True, TypeError), (2.0, TypeError), ("2", TypeError), (0, ValueError), (-1, ValueError), (5, ValueError)]


@pytest.mark.parametrize("bad, exc", BAD)
def test_ctc_beam_search_refuses_bad_nbest(bad, exc):
    from edgedict_b200 import ctc
    with pytest.raises(exc):
        ctc.beam_search(_lp(), [5, 3], 4, nbest=bad)
    with pytest.raises(RuntimeError):                            # a good one: the CPU tensor is what is refused
        ctc.beam_search(_lp(), [5, 3], 4, nbest=4)


@pytest.mark.parametrize("bad, exc", BAD)
def test_ctc_encoder_refuses_bad_nbest_before_the_forward(bad, exc):
    from edgedict_b200.rnnt.models import CTCEncoder
    m = CTCEncoder(vocab_size=6, input_size=4, enc_hidden_size=8, enc_layers=1, enc_dropout=0.0, proj_size=4)
    with pytest.raises(exc):
        m.beam_search(torch.randn(1, 3, 4), W=4, nbest=bad)


@pytest.mark.parametrize("bad, exc", BAD)
def test_transducer_refuses_bad_nbest_before_the_encoder(bad, exc):
    from edgedict_b200.rnnt.models import Transducer
    m = Transducer(output_loss=False, **TINY)
    with pytest.raises(exc):
        m.beam_search(torch.randn(1, 4, TINY["input_size"]), W=4, nbest=bad)


@pytest.mark.parametrize("bad, exc", [b for b in BAD if b[0] != 0] + [(None, TypeError)])
def test_engines_refuse_bad_nbest(bad, exc):
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import BeamEngine, CTCBeamEngine
    m = Transducer(output_loss=False, **TINY)
    with pytest.raises(exc):
        BeamEngine(m, 1, 3, 4, nbest=bad)
    with pytest.raises(exc):
        CTCBeamEngine(1, 3, 4, 4, nbest=bad, device="cpu")
    for ok in (0, 1, 4):                                         # accepted: the CPU device is what is refused
        with pytest.raises(RuntimeError):
            BeamEngine(m, 1, 3, 4, nbest=ok)
        with pytest.raises(RuntimeError):
            CTCBeamEngine(1, 3, 4, 4, nbest=ok, device="cpu")
