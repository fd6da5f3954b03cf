"""Contextual biasing on the host (no GPU): the ContextGraph tables against the brute-force restatement of their
definition (tests/context_oracle.py), the banked bonus along random sequences, every refusal before device work and
the content fingerprint."""
import random

import numpy as np
import pytest
import torch

from edgedict_b200.context import MAX_TABLE, ContextGraph, check_context
from tests import context_oracle as co


def _phrase_sets():
    rng = random.Random(7)
    sets = [
        [[1, 2, 3], [2, 3], [3], [2, 3, 4, 5]],            # nested: suffixes that are phrases
        [[1, 2], [1, 2, 3, 4], [1, 2, 3]],                  # prefixes of each other
        [[1, 1, 1], [1, 1], [2, 1, 1, 2]],                  # repeated tokens, overlaps
        [[4, 5, 4, 5, 6], [5, 4, 5], [4, 5]],               # self-overlapping
        [[2, 3], [2, 3], [3, 2, 3]],                         # duplicates collapse
    ]
    for _ in range(6):
        V = rng.choice([4, 5, 7])
        sets.append([[rng.randrange(1, V) for _ in range(rng.randint(1, 5))] for _ in range(rng.randint(1, 8))])
    return sets


@pytest.mark.parametrize("i", range(11))
@pytest.mark.parametrize("beta", [0.0, 0.75, 1.3])
def test_tables_equal_brute_force(i, beta):
    phrases = _phrase_sets()[i]
    V = max(max(p) for p in phrases) + 2
    g = ContextGraph(phrases, V, beta)
    ref = co.brute_tables(phrases, V, beta)
    index = {s: n for n, s in enumerate(g.nodes)}
    assert len(index) == g.n_states == len({tuple(p[:j]) for p in phrases for j in range(len(p) + 1)})
    assert g.next.shape == g.delta.shape == (g.n_states, V) and g.next.dtype == np.int32
    assert g.delta.dtype == np.float32 and g.pending.dtype == np.float32
    for n, s in enumerate(g.nodes):
        assert g.pending[n] == np.float32(beta) * np.float32(len(s))
        assert g.next[n, 0] == n and g.delta[n, 0] == 0.0            # blank: identity, nothing added
        for k in range(1, V):
            u, d = ref[s, k]
            assert g.nodes[g.next[n, k]] == u, (s, k)
            assert g.delta[n, k] == d, (s, k, g.delta[n, k], d)


@pytest.mark.parametrize("i", range(11))
def test_sum_of_increments_minus_pending_is_the_banked_bonus(i):
    phrases = _phrase_sets()[i]
    V = max(max(p) for p in phrases) + 2
    beta = 0.625
    g = ContextGraph(phrases, V, beta)
    rng = random.Random(i)
    toks = sorted({k for p in phrases for k in p}) + [V - 1]
    for _ in range(60):
        seq = [rng.choice(toks + [0]) for _ in range(rng.randint(0, 14))]
        s, tot = 0, 0.0
        for k in seq:
            s, d = g.step(s, k)
            tot += d
        want = co.banked(phrases, seq, beta)
        assert abs((tot - float(g.pending[s])) - want) <= 1e-5 * (1 + want), (seq, tot, want)


def test_prefix_phrase_completes_first_and_resets():
    g = ContextGraph([[1, 2], [1, 2, 3]], 5, 1.0)
    s, d1 = g.step(0, 1)
    s, d2 = g.step(s, 2)
    assert s == 0 and d1 == 1.0 and d2 == 1.0                           # [1, 2] completes, the state resets
    s, d3 = g.step(s, 3)
    assert s == 0 and d3 == 0.0                                          # [1, 2, 3] cannot complete after it


def test_empty_graph_and_duplicates():
    g = ContextGraph([], 8, 2.0)
    assert g.n_states == 1 and len(g) == 0 and g.to("cpu") is None
    assert check_context(g, 8, 0) is None and check_context(None, 8, 0) is None
    assert ContextGraph([[1, 2], (1, 2), np.array([1, 2])], 8, 1.0).phrases == [(1, 2)]


@pytest.mark.parametrize("args, exc", [
    (([[0, 1]], 8, 1.0), ValueError),                  # blank
    (([[1, -1]], 8, 1.0), ValueError),                 # negative
    (([[1, 8]], 8, 1.0), ValueError),                  # out of range
    (([[]], 8, 1.0), ValueError),                      # empty phrase
    (([[1]], 8, float("inf")), ValueError),
    (([[1]], 8, float("nan")), ValueError),
    (([[1]], 8, -0.5), ValueError),
    (([[1]], 8, "1"), TypeError),
    (([[1]], 8, True), TypeError),
    (([[1.5]], 8, 1.0), TypeError),
    (("ab", 8, 1.0), TypeError),
    ((["ab"], 8, 1.0), TypeError),
    (([[1]], 0, 1.0), ValueError),
    (([[1]], 8.0, 1.0), TypeError),
    (([[1]], 8, 1.0, 8), ValueError),                  # blank outside [0, V)
])
def test_refusals(args, exc):
    with pytest.raises(exc):
        ContextGraph(*args)


def test_table_cap():
    V = 4096
    n_ok = MAX_TABLE // V - 1
    ContextGraph([[k] for k in range(1, n_ok)], V, 1.0)   # the root and n_ok - 1 one-token phrases: under the cap
    with pytest.raises(ValueError, match="2\\^24"):
        ContextGraph([[1 + (k % (V - 1)), 1 + (k // (V - 1))] for k in range(MAX_TABLE // V + 1)], V, 1.0)


def test_check_context_refusals():
    g = ContextGraph([[1, 2]], 8, 1.0)
    assert check_context(g, 8, 0) is g
    with pytest.raises(ValueError):
        check_context(g, 9, 0)
    with pytest.raises(ValueError):
        check_context(ContextGraph([[1, 2]], 8, 1.0, blank=3), 8, 0)
    with pytest.raises(TypeError):
        check_context([[1, 2]], 8, 0)


def test_fingerprint_follows_content():
    a = ContextGraph([[1, 2], [3]], 8, 1.0)
    assert a.fingerprint == ContextGraph([[3], [1, 2], [1, 2]], 8, 1.0).fingerprint
    others = [ContextGraph([[1, 2], [4]], 8, 1.0), ContextGraph([[1, 2], [3]], 8, 1.5),
              ContextGraph([[1, 2], [3]], 9, 1.0), ContextGraph([[1, 2, 3]], 8, 1.0),
              ContextGraph([[1], [2, 3]], 8, 1.0)]
    assert len({a.fingerprint} | {o.fingerprint for o in others}) == 1 + len(others)


def test_refusals_come_before_device_work(monkeypatch):
    """The public entries refuse a mismatched graph before touching the model or the device: no CUDA call is made."""
    from edgedict_b200 import ctc
    from edgedict_b200.rnnt.models import CTCEncoder, Transducer

    def boom(*a, **k):
        raise AssertionError("device work before the context check")

    class Boom(torch.nn.Module):
        forward = staticmethod(boom)
    g = ContextGraph([[1, 2]], 7, 1.0)
    m = Transducer(output_loss=False, vocab_embed_size=4, vocab_size=8, input_size=6, enc_hidden_size=8,
                   enc_layers=1, enc_dropout=0.0, enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0.0,
                   dec_proj_size=8, joint_size=8)
    monkeypatch.setattr(m, "encoder", Boom())
    with pytest.raises(ValueError, match="vocab_size"):
        m.beam_search(torch.zeros(1, 4, 6), W=2, context=g)
    with pytest.raises(TypeError):
        m.beam_search(torch.zeros(1, 4, 6), W=2, context=[[1, 2]])
    c = CTCEncoder(vocab_size=8, input_size=6, enc_hidden_size=8, enc_layers=1, enc_dropout=0.0, proj_size=8)
    monkeypatch.setattr(c, "forward", boom)
    with pytest.raises(ValueError, match="vocab_size"):
        c.beam_search(torch.zeros(1, 4, 6), W=2, context=g)
    with pytest.raises(ValueError, match="vocab_size"):
        ctc.beam_search(torch.zeros(1, 4, 8), [4], 2, context=g)     # CPU log-probs: refused before the CUDA check
