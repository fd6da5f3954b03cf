"""Contextual biasing in the streaming beams, without a GPU: the restatement of BEAM_COMMIT with flag 2048 against
brute force, the streaming CTC restatement with a graph against the offline one (tests/context_oracle.py) and against
the plain streaming restatement at boost 0, and every refusal of a ``context`` argument, before any device work."""
import numpy as np
import pytest
import torch

from edgedict_b200.context import ContextGraph
from tests import beam_phases_restate as rs
from tests import context_oracle as co
from tests import context_stream_oracle as cso
from tests.ctc_stream_beam_oracle import CTCStreamBeamRestatement


def _commit_case(rng, S, W, live, flush):
    P, T, HEAD = 12, 2, 3
    LS = P + HEAD
    R = S * W
    seq = np.zeros((R, LS), dtype=np.int32)
    hist = np.zeros(3 * S * T * W + S * T, dtype=np.int32)
    _, _, _, hlive = rs.hist_views(hist, S, T, W)
    for b in range(S):
        hlive[b, T - 1] = live
        for s in range(live):
            n = int(rng.integers(0, 6))
            seq[b * W + s, 0] = n
            seq[b * W + s, HEAD:HEAD + n] = rng.integers(1, 4, size=n)
    n_states = 5
    d = dict(y=(-0.5 * rng.integers(0, 8, size=R)).astype(np.float32), hist=hist, seq_in=seq,
             seq_out=np.zeros_like(seq), tok_out=np.zeros(S * P, dtype=np.int32),
             tok_out2=np.zeros(2 * S, dtype=np.int32), src=np.zeros(R, dtype=np.int32),
             ctx_pending=(0.5 * rng.integers(0, 5, size=n_states)).astype(np.float32),
             ctx_state=np.stack([np.zeros(R, dtype=np.int32), rng.integers(0, n_states, size=R).astype(np.int32)]))
    p = dict(S=S, N=P, aux=W, aux2=1, K1=LS, K2=0, hist_ld=T, flags=2048 | (128 if flush else 0))
    return p, d


@pytest.mark.parametrize("flush", [False, True])
def test_commit_restatement_ranks_collapses_by_value_minus_pending(flush):
    rng = np.random.default_rng(3 + flush)
    for _ in range(50):
        S, W = 3, 4
        live = int(rng.integers(1, W + 1))
        p, d = _commit_case(rng, S, W, live, flush)
        y0, st1 = d["y"].copy(), d["ctx_state"][1].copy()
        cso.beam_commit(p, d)
        for b in range(S):
            r0 = b * W
            v = [float(y0[r0 + j]) - float(d["ctx_pending"][st1[r0 + j]]) for j in range(live)]
            if d["tok_out2"][S + b]:
                best = max(range(live), key=lambda j: (v[j], -j))        # the first of equal maxima
                assert d["src"][r0] == r0 + best
                assert d["y"][r0] == y0[r0 + best]                       # the kept slot keeps its own y
                assert np.isneginf(d["y"][r0 + 1:r0 + W]).all()
            else:
                assert np.array_equal(d["y"][r0:r0 + W], y0[r0:r0 + W])
            assert np.array_equal(d["ctx_state"][0][r0:r0 + W], st1[d["src"][r0:r0 + W]])
        # zero pending bonuses: the plain phase
        p2, d2 = _commit_case(np.random.default_rng(9), S, W, live, flush)
        d2["ctx_pending"][:] = 0
        plain = {k: v.copy() for k, v in d2.items()}
        cso.beam_commit(p2, d2)
        rs.beam_commit(dict(p2, flags=p2["flags"] & ~2048), plain)
        for k in ("y", "seq_out", "tok_out", "tok_out2", "src"):
            assert np.array_equal(d2[k].view(np.int32), plain[k].view(np.int32)), k


def _lp(seed, T, V):
    g = torch.Generator().manual_seed(seed)
    return (2.5 * torch.randn(T, V, generator=g, dtype=torch.float64)).log_softmax(-1).numpy()


@pytest.mark.parametrize("seed", range(4))
def test_ctc_stream_restatement_is_the_offline_biased_search(seed):
    """Chunks of 1-3 frames with a generous max_pending: the committed tokens plus the flush are the best prefix of
    tests/context_oracle.ctc_nbest over the whole utterance, and its -score, with phrases straddling the chunks."""
    V, T, W = 7, 18, 4
    lp = _lp(seed, T, V)
    best = co.ctc_nbest(lp, T, W, ContextGraph([], V, 1.0), dtype=np.float64)[0]
    graph = ContextGraph([list(best[0][i:i + 3]) for i in range(0, max(len(best[0]) - 2, 1), 2)] + [[1, 2], [3, 4]],
                         V, 1.25)
    want = co.ctc_nbest(lp, T, W, graph, dtype=np.float64)[0]
    r = cso.CTCContextStream(W, graph, max_pending=64)
    got, t = [], 0
    for n in [1, 3, 2, 1, 2, 3, 1, 2, 3]:
        got += r.chunk(lp[t:t + n])
        t += n
    assert t == T
    rest, score = r.flush()
    assert tuple(got + rest) == want[0]
    assert abs(score - want[2]) <= 1e-9 * max(1.0, abs(want[2]))
    assert r.n_collapses == 0


def test_ctc_stream_restatement_at_boost_zero_is_the_plain_one():
    V, T, W = 7, 24, 3
    lp = _lp(11, T, V)
    graph = ContextGraph([[1, 2], [2, 3, 4], [5]], V, 0.0)
    a = cso.CTCContextStream(W, graph, max_pending=2)
    b = CTCStreamBeamRestatement(W, max_pending=2)
    for t in range(0, T, 2):
        assert a.chunk(lp[t:t + 2]) == b.chunk(lp[t:t + 2])
    assert a.flush() == b.flush()
    assert a.n_collapses == b.n_collapses > 0


# ---- refusals, before any device work ----------------------------------------------------------------------------------
def _cpu_transducer():
    from edgedict_b200.rnnt.models import Transducer
    from tests.test_gpu_beam_engine import SMALL
    torch.manual_seed(0)
    return Transducer(output_loss=False, **SMALL)


def _cpu_ctc():
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(0)
    return CTCEncoder(vocab_size=40, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0, proj_size=32)


class _Tok:
    class tokenizer:
        @staticmethod
        def token_to_id(t):
            return None


def test_stream_engines_refuse_a_mismatched_context():
    from edgedict_b200.stream_engine import CTCStreamBeamEngine, GRUStreamBeamEngine, StreamBeamEngine
    cuda_before = torch.cuda.is_initialized()
    m = _cpu_transducer()
    V = m.joint.joint[2].weight.shape[0]
    for bad, exc in ((ContextGraph([[1, 2]], V + 1, 1.0), ValueError), (ContextGraph([[1, 2]], V, 1.0, blank=3),
                                                                         ValueError), ([[1, 2]], TypeError)):
        with pytest.raises(exc):
            StreamBeamEngine(m, 1, 4, 4, context=bad)
        with pytest.raises(exc):
            GRUStreamBeamEngine(m, 1, 4, 4, context=bad)
    c = _cpu_ctc()
    with pytest.raises(ValueError, match="vocab_size"):
        CTCStreamBeamEngine(c, 1, 4, 4, context=ContextGraph([[1, 2]], 41, 1.0))
    with pytest.raises(ValueError, match="blank"):
        CTCStreamBeamEngine(c, 1, 4, 4, blank=2, context=ContextGraph([[1, 3]], 40, 1.0))
    # a matching graph gets as far as the device check
    with pytest.raises(RuntimeError, match="CUDA"):
        StreamBeamEngine(m, 1, 4, 4, context=ContextGraph([[1, 2]], V, 1.0))
    assert torch.cuda.is_initialized() == cuda_before


def test_stream_decoders_refuse_context_without_a_beam_and_mismatched_graphs():
    from edgedict_b200.ctc import CTCStreamDecoder
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    cuda_before = torch.cuda.is_initialized()
    m = _cpu_transducer()
    V = m.joint.joint[2].weight.shape[0]
    good = ContextGraph([[1, 2]], V, 1.0)
    with pytest.raises(ValueError, match="beam_width"):
        PytorchStreamDecoder(FLAGS=None, transducer=m, transform=lambda f: f, tokenizer=_Tok(), device="cpu",
                             context=good)
    for bad in (ContextGraph([[1, 2]], V + 3, 1.0), ContextGraph([[1, 2]], V, 1.0, blank=5)):
        with pytest.raises(ValueError):
            PytorchStreamDecoder(FLAGS=None, transducer=m, transform=lambda f: f, tokenizer=_Tok(), device="cpu",
                                 beam_width=4, context=bad)
    c = _cpu_ctc()
    with pytest.raises(ValueError, match="beam_width"):
        CTCStreamDecoder(c, None, None, device="cuda", context=ContextGraph([[1, 2]], 40, 1.0))
    for bad in (ContextGraph([[1, 2]], 39, 1.0), ContextGraph([[1, 2]], 40, 1.0, blank=3)):
        with pytest.raises(ValueError):
            CTCStreamDecoder(c, None, None, device="cuda", beam_width=4, context=bad)
    with pytest.raises(TypeError):
        CTCStreamDecoder(c, None, None, device="cuda", beam_width=4, context=[[1, 2]])
    assert torch.cuda.is_initialized() == cuda_before
