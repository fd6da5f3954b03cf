"""Contextual biasing in the streaming beams (StreamBeamEngine, GRUStreamBeamEngine, CTCStreamBeamEngine with
``context``; decode.cu flag 2048 in BEAM_COMMIT; PytorchStreamDecoder / CTCStreamDecoder(context=...)):

* chunking is invisible: the committed ids of every chunk plus the flush are the offline biased search's best
  hypothesis on the concatenated per-chunk encoder output (or log-probs), -log p bit for bit, with phrases that
  straddle chunks and commits;
* forced collapses against the CPU restatement (tests/context_stream_oracle.py), which ranks a collapse by
  value - pending and moves the automaton state with the slot;
* BEAM_COMMIT alone, teacher-forced, through every decode entry and max_ctas, equal to the restatement word for word;
* bitwise invariants, state() / load_state() and its refusals, the boost, and the two decoders."""
import random

import numpy as np
import pytest
import torch

from edgedict_b200.context import ContextGraph
from oracle import model_torch as mt
from tests import context_oracle as co
from tests import context_stream_oracle as cso
from tests.test_gpu_beam_engine import SMALL
from tests.test_gpu_beam_lm import _lm_module
from tests.test_gpu_beam_phases_fp64 import F_CONTEXT, F_FLUSH, _commit_inputs, _compare, _restate, _run_all
from tests.test_gpu_ctc_stream_beam import TINY as CTC_TINY
from tests.test_gpu_ctc_stream_beam import _model as _ctc_model
from tests.test_gpu_stream_beam import _tiny
from tests.test_oracle_lm import load_lm

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bits(t):
    return t.contiguous().view(torch.int32)


def _transducer(enc, seed=4):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(seed)
    m = Transducer(output_loss=False, module_type=enc, **SMALL).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)
    return m.to(DEV)


def _stream(m, chunks, W, gru=False, max_ctas=0, **kw):
    """The chunks (a list of [S, n, F]) through (GRU)StreamBeamEngine, rebuilt with the carried state whenever the
    chunk length changes.  -> (committed ids per chunk and stream, flushed ids per stream, -log p [S], the
    concatenated encoder output [S, T', E], the engine)."""
    from edgedict_b200.stream_engine import GRUStreamBeamEngine, StreamBeamEngine
    cls = GRUStreamBeamEngine if gru else StreamBeamEngine
    eng, per, enc = None, [], []
    S = chunks[0].shape[0]
    for c in chunks:
        if eng is None or eng.n != c.shape[1]:
            eng = cls(m, S, c.shape[1], W, state=None if eng is None else eng.state(), max_ctas=max_ctas, **kw)
        ids, counts = eng.step(c.to(DEV))
        per.append([ids[s, :int(counts[s])].tolist() for s in range(S)])
        enc.append(eng.enc_out.clone())
    ids, counts, nlp = eng.flush()
    return per, [ids[s, :int(counts[s])].tolist() for s in range(S)], nlp, torch.cat(enc, 1), eng


def _joined(per, fl):
    return [sum((c[s] for c in per), []) + fl[s] for s in range(len(fl))]


def _offline(m, enc, W, **kw):
    from edgedict_b200.stream_engine import BeamEngine
    S, T = enc.shape[0], enc.shape[1]
    eng = BeamEngine(m, S, T, W, **kw)
    ids, nlp = eng.run(enc, torch.full((S,), T, dtype=torch.int32, device=DEV))
    return [[int(k) for k in r if k >= 0] for r in ids.cpu().numpy()], nlp.cpu()


def _chunks(S, lens, F, seed, scale=1.5):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(S, n, F, generator=g) * scale for n in lens]


def _phrases_from(hyps, V, seed, n_random=20, lo=2, hi=5):
    """Phrases cut from the given token sequences (windows of lo..hi tokens, so matches span several chunks of one
    output frame) plus random ones over [1, V)."""
    rng = random.Random(seed)
    out = []
    for h in hyps:
        for _ in range(3):
            if len(h) >= lo:
                n = rng.randint(lo, min(hi, len(h)))
                i = rng.randrange(len(h) - n + 1)
                out.append(h[i:i + n])
    out += [[rng.randrange(1, V) for _ in range(rng.randint(lo, hi))] for _ in range(n_random)]
    return out


def _graph_for(m, chunks, W, V, beta, seed, gru=False, **kw):
    """A graph whose phrases come from the unbiased search's N-best over the same audio."""
    from edgedict_b200.stream_engine import BeamEngine
    _, _, _, enc, _ = _stream(m, chunks, W, gru=gru, **kw)
    S, T = enc.shape[0], enc.shape[1]
    from edgedict_b200.stream_engine import nbest_lists
    be = BeamEngine(m, S, T, max(W, 2), nbest=max(W, 2), **kw)
    out = be.run(enc, torch.full((S,), T, dtype=torch.int32, device=DEV))
    lists = nbest_lists(out, S, max(W, 2), be.ids.shape[-1])
    hyps = [h.tokens.tolist() for lst in lists for h in lst[1:]]
    return ContextGraph(_phrases_from(hyps, V, seed), V, beta)


LENS = {"2": [2] * 12, "mixed": [4, 2, 6, 2, 4, 2, 4]}


# ---- 1. chunking is invisible ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens", sorted(LENS))
@pytest.mark.parametrize("lm", [False, True])
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 4, 8])
def test_transducer_chunking_is_invisible(W, merge, K, lm, lens):
    m = _transducer("LSTM")
    V = SMALL["vocab_size"]
    kw = dict(merge=merge, max_symbols=K)
    if lm:
        kw.update(lm=_lm_module(V, 16, 48, 2, 4.0, seed=1).to(DEV), lm_weight=0.4, length_bonus=0.3)
    chunks = _chunks(3, LENS[lens], SMALL["input_size"], seed=W * 7 + K + len(lens))
    graph = _graph_for(m, chunks, W, V, 1.5, seed=W + K, **kw)
    per, fl, nlp, enc, eng = _stream(m, chunks, W, max_pending=256, context=graph, **kw)
    want, wlp = _offline(m, enc, W, context=graph, **kw)
    got = _joined(per, fl)
    hits = sum(co.banked(graph.phrases, g, 1.0) > 0 for g in got)
    print("W=%d merge=%s K=%d lm=%s lens=%s: %d tokens, %d committed before the flush, %d streams complete a "
          "phrase" % (W, merge, K, lm, lens, sum(map(len, got)), sum(len(x) for c in per for x in c), hits))
    assert eng.n_collapses == 0
    assert got == want
    assert torch.equal(_bits(nlp), _bits(wlp))
    assert sum(map(len, got)) > 0


@pytest.mark.parametrize("lm", [False, True])
@pytest.mark.parametrize("W", [1, 4, 8])
def test_gru_transducer_chunking_is_invisible(W, lm):
    m = _transducer("GRU", seed=6)
    V = SMALL["vocab_size"]
    kw = dict(lm=_lm_module(V, 16, 48, 2, 4.0, seed=1).to(DEV), lm_weight=0.4, length_bonus=0.3) if lm else {}
    chunks = _chunks(2, LENS["mixed"], SMALL["input_size"], seed=W + 40)
    graph = _graph_for(m, chunks, W, V, 2.0, seed=W, gru=True, **kw)
    per, fl, nlp, enc, eng = _stream(m, chunks, W, gru=True, context=graph, **kw)
    want, wlp = _offline(m, enc, W, context=graph, **kw)
    assert eng.n_collapses == 0
    assert _joined(per, fl) == want
    assert torch.equal(_bits(nlp), _bits(wlp))


def _ctc_stream(m, S, lens, xs, W, max_ctas=0, **kw):
    from edgedict_b200.stream_engine import CTCStreamBeamEngine
    eng, per, lps, t0 = None, [], [], 0
    for n in lens:
        if eng is None or eng.n != n:
            eng = CTCStreamBeamEngine(m, S, n, W, state=None if eng is None else eng.state(), max_ctas=max_ctas, **kw)
        ids, cnt = eng.step(xs[:, t0:t0 + n])
        t0 += n
        per.append([ids[s, :int(cnt[s])].tolist() for s in range(S)])
        lps.append(eng.logprobs.view(S, eng.n_out, -1).clone())
    ids, cnt, nscore = eng.flush()
    return per, [ids[s, :int(cnt[s])].tolist() for s in range(S)], nscore, torch.cat(lps, 1), eng


def _ctc_offline(lp, W, **kw):
    from edgedict_b200.stream_engine import CTCBeamEngine
    B, T, V = lp.shape
    ids, nlp = CTCBeamEngine(B, T, V, W, device=DEV, **kw).run(lp, torch.full((B,), T, dtype=torch.int32, device=DEV))
    ids = ids.cpu()
    return [r[r >= 0].tolist() for r in ids], nlp.cpu().clone()


def _ctc_setup(S, seed, lens):
    m = _ctc_model(CTC_TINY, seed, scale=2.0)
    g = torch.Generator().manual_seed(seed)
    xs = torch.randn(S, sum(lens), CTC_TINY["input_size"], generator=g).to(DEV)
    return m, xs


def _ctc_graph(m, S, lens, xs, W, beta, seed, **kw):
    from edgedict_b200 import ctc
    _, _, _, lp, _ = _ctc_stream(m, S, lens, xs, W, **kw)
    N = max(W, 2)
    lists = ctc.beam_search(lp, [lp.shape[1]] * S, N, nbest=N, **kw)
    hyps = [h.tokens.tolist() for lst in lists for h in lst[1:]]
    return ContextGraph(_phrases_from(hyps, CTC_TINY["vocab_size"], seed), CTC_TINY["vocab_size"], beta)


@pytest.mark.parametrize("lm", [False, True])
@pytest.mark.parametrize("lens", [[2] * 10, [4, 2, 6, 2, 4]])
@pytest.mark.parametrize("S", [3, 70])
def test_ctc_chunking_is_invisible(S, lens, lm):
    V = CTC_TINY["vocab_size"]
    m, xs = _ctc_setup(S, 21 + len(lens), lens)
    kw = dict(lm=_lm_module(V, 8, 12, 2, 3.0, seed=5), lm_weight=0.6, length_bonus=0.3) if lm else {}
    W = 4
    graph = _ctc_graph(m, S, lens, xs, W, 1.5, seed=S, **kw)
    per, fl, nscore, lp, eng = _ctc_stream(m, S, lens, xs, W, context=graph, **kw)
    want, wlp = _ctc_offline(lp, W, context=graph, **kw)
    got = [sum((c[s] for c in per), []) + fl[s] for s in range(S)]
    hits = sum(co.banked(graph.phrases, g, 1.0) > 0 for g in got)
    print("S=%d lens=%s lm=%s: %d tokens, %d streams complete a phrase" % (S, lens, lm, sum(map(len, got)), hits))
    assert eng.n_collapses == 0
    assert got == want
    assert torch.equal(_bits(nscore), _bits(wlp))
    assert sum(map(len, got)) > 0


# ---- 2. forced collapses against the restatement ----------------------------------------------------------------------
@pytest.mark.parametrize("lm", [False, True])
def test_transducer_forced_collapses_match_restatement(lm):
    m, z, sd = _tiny()
    V = sd["joint.joint.2.weight"].shape[0]
    chunks = [torch.as_tensor(np.concatenate(z["stream_chunks"][i:i + 2], 0)[None]) for i in range(0, 40, 2)]
    kw, okw = {}, {}
    if lm:
        lsd = load_lm()[1]
        kw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5)
        okw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5)
    W, P = 4, 4
    _, _, _, enc, _ = _stream(m, chunks, W, max_pending=P, **kw)
    h_enc, _ = mt.encoder(sd, torch.cat(chunks, 1), None)
    base, _ = _offline(m, enc, W, **kw)
    graph = ContextGraph(_phrases_from([base[0]], V, seed=3, n_random=5), V, 1.0)
    per, fl, nlp, _, eng = _stream(m, chunks, W, max_pending=P, context=graph, **kw)
    wper, wfl, wnlp, wcol = cso.transducer_stream(sd, h_enc[0], [c.shape[1] // 2 for c in chunks], W, P, graph, **okw)
    print("lm=%s: %d forced collapses (restatement %d), flush -log p %.6f / %.6f"
          % (lm, eng.n_collapses, wcol, float(nlp[0]), wnlp))
    assert [c[0] for c in per] == wper
    assert fl[0] == wfl
    assert eng.n_collapses == wcol > 0
    assert abs(float(nlp[0]) - wnlp) <= 1e-4 * max(1.0, abs(wnlp))


@pytest.mark.parametrize("lm", [False, True])
def test_ctc_forced_collapses_match_restatement(lm):
    V = CTC_TINY["vocab_size"]
    lens = [2] * 16
    m, xs = _ctc_setup(2, 31, lens)
    kw, okw = {}, {}
    if lm:
        mod = _lm_module(V, 8, 12, 2, 3.0, seed=5)
        kw = dict(lm=mod, lm_weight=0.6, length_bonus=0.3)
        okw = dict(lm_sd={k: v.detach().float() for k, v in mod.state_dict().items()}, lm_weight=0.6,
                   length_bonus=0.3)
    graph = _ctc_graph(m, 2, lens, xs, 4, 1.5, seed=7, **kw)
    P = 2
    per, fl, nscore, lp, eng = _ctc_stream(m, 2, lens, xs, 4, max_pending=P, context=graph, **kw)
    lpc = lp.cpu().numpy()
    n_out = lp.shape[1] // len(lens)
    for s in range(2):
        r = cso.CTCContextStream(4, graph, max_pending=P, dtype=np.float32, **okw)
        for i in range(len(lens)):
            assert r.chunk(lpc[s, i * n_out:(i + 1) * n_out]) == per[i][s], ("stream", s, "chunk", i)
        rest, wscore = r.flush()
        assert rest == fl[s]
        assert abs(float(nscore[s]) - wscore) <= 1e-5 * max(1.0, abs(wscore))
        print("stream %d: %d forced collapses" % (s, r.n_collapses))
    assert eng.n_collapses > 0


# ---- 3. BEAM_COMMIT alone, teacher-forced --------------------------------------------------------------------------------
COMMIT_CASES = [(3, 1, 3, 1, "common"), (3, 4, 5, 4, "flush"), (5, 31, 3, 31, "edge"), (5, 32, 5, 32, "tie"),
                (3, 256, 3, 256, "edge"), (3, 257, 5, 257, "tie"), (2, 1024, 3, 1024, "tie"),
                (2, 1024, 5, 1000, "flush"), (150, 4, 5, 4, "edge")]


@pytest.mark.parametrize("S,W,head,live,mode", COMMIT_CASES)
def test_beam_commit_context_exact(S, W, head, live, mode):
    """Flag 2048 with and without flag 128: states in parity 1, pending bonuses that reorder the raw y (the best slot's
    raw y is not the highest), and ties in y - pending (the lowest slot wins, -0 with +0)."""
    for flush in (False, True):
        for with_last in (False, True):
            p, host = _commit_inputs(S, W, head, live, mode if mode != "flush" else "common", S * 17 + W + head, with_last)
            rng = np.random.default_rng(S + W + head + flush)
            n_states, R = 9, S * W
            pend = (0.25 * rng.integers(0, 13, size=n_states)).astype(np.float32)
            st = np.stack([np.full(R, 5, dtype=np.int32), rng.integers(0, n_states, size=R).astype(np.int32)])
            y = host["y"]
            for b in range(S):
                n = min(live, W)
                r0 = b * W
                top = r0 + int(np.argmax(y[r0:r0 + n]))
                st[1, top] = n_states - 1                       # the raw best pays the largest pending bonus
                pend[n_states - 1] = 16.0                       # more than the spread of y
                if mode == "tie" and n >= 3:                    # equal y - pending in two slots, -0 and +0
                    st[1, r0 + n - 2], st[1, r0 + n - 1] = 0, 0
                    y[r0 + n - 2], y[r0 + n - 1] = -0.0, 0.0
                    pend[0] = 0.0
            p["flags"] = F_CONTEXT | (F_FLUSH if flush or mode in ("flush", "tie") else 0)
            host.update(ctx_next=np.zeros((n_states, 4), dtype=np.int32), ctx_delta=np.zeros((n_states, 4),
                        dtype=np.float32), ctx_pending=pend, ctx_state=st)
            got = _run_all("commit", p, host)
            want, _ = _restate(cso.beam_commit, p, host)
            _compare("commit+ctx W=%d head=%d %s flush=%s" % (W, head, mode, flush), got, want)
            if p["flags"] & F_FLUSH:
                src = want["src"].reshape(S, W)[:, 0] - np.arange(S) * W
                raw = [int(np.argmax(host["y"][b * W:b * W + min(live, W)])) for b in range(S)]
                moved = sum(int(a != b) for a, b in zip(src, raw))
                print("  S=%d W=%d %s: %d of %d collapses keep a slot other than the raw best" % (S, W, mode, moved, S))
                if min(live, W) > 1:
                    assert moved > 0


# ---- 4. bitwise invariants ------------------------------------------------------------------------------------------------
def test_streams_ctas_and_repeats_are_bitwise_invariant():
    m = _transducer("LSTM", seed=8)
    V = SMALL["vocab_size"]
    chunks = _chunks(4, [2] * 10, SMALL["input_size"], seed=5)
    graph = _graph_for(m, chunks, 4, V, 1.5, seed=2)
    ref = _stream(m, chunks, 4, context=graph)
    for mc in (1, 3, 0):
        again = _stream(m, chunks, 4, context=graph, max_ctas=mc)
        assert again[0] == ref[0] and again[1] == ref[1] and torch.equal(_bits(again[2]), _bits(ref[2])), mc
    for s in range(4):
        alone = _stream(m, [c[s:s + 1] for c in chunks], 4, context=graph)
        assert [c[0] for c in alone[0]] == [c[s] for c in ref[0]] and alone[1][0] == ref[1][s]
        assert torch.equal(_bits(alone[2]), _bits(ref[2][s:s + 1]))
    # CTC
    lens = [2] * 8
    mc_, xs = _ctc_setup(3, 9, lens)
    g2 = _ctc_graph(mc_, 3, lens, xs, 4, 1.5, seed=4)
    ref = _ctc_stream(mc_, 3, lens, xs, 4, context=g2)
    for mc in (1, 3, 0):
        again = _ctc_stream(mc_, 3, lens, xs, 4, context=g2, max_ctas=mc)
        assert again[0] == ref[0] and again[1] == ref[1] and torch.equal(_bits(again[2]), _bits(ref[2])), mc
    for s in range(3):
        alone = _ctc_stream(mc_, 1, lens, xs[s:s + 1], 4, context=g2)
        assert [c[0] for c in alone[0]] == [c[s] for c in ref[0]] and alone[1][0] == ref[1][s]
        assert torch.equal(_bits(alone[2]), _bits(ref[2][s:s + 1]))


# ---- 5. state() / load_state() ---------------------------------------------------------------------------------------------
def test_rebuilt_run_continues_bitwise_and_bad_states_are_refused():
    from edgedict_b200.stream_engine import CTCStreamBeamEngine, StreamBeamEngine
    m = _transducer("LSTM", seed=9)
    V = SMALL["vocab_size"]
    chunks = _chunks(2, [4] * 6, SMALL["input_size"], seed=12)
    graph = _graph_for(m, chunks, 4, V, 1.5, seed=5)
    whole = _stream(m, chunks, 4, context=graph)
    # 4-frame chunks, with the engine rebuilt for 2-frame chunks over chunks 2 and 3 and back
    cut = chunks[:2] + [chunks[2][:, :2], chunks[2][:, 2:], chunks[3][:, :2], chunks[3][:, 2:]] + chunks[4:]
    split = _stream(m, cut, 4, context=graph)
    assert _joined(*split[:2]) == _joined(*whole[:2])
    assert torch.equal(_bits(split[2]), _bits(whole[2]))
    assert split[4].n_collapses == 0

    eng = StreamBeamEngine(m, 2, 4, 4, context=graph)
    eng.step(chunks[0].to(DEV))
    st = eng.state()
    other = ContextGraph(graph.phrases[:-1], V, 1.5)
    plain = StreamBeamEngine(m, 2, 4, 4)
    plain.step(chunks[0].to(DEV))
    target = StreamBeamEngine(m, 2, 4, 4, context=graph)
    before = target.state()
    bad = dict(st, ctx_state=st["ctx_state"].clone())
    bad["ctx_state"][0] = graph.n_states
    for what, s, eng_ in (("other graph", st, StreamBeamEngine(m, 2, 4, 4, context=other)),
                          ("state without context", plain.state(), target),
                          ("context state into a plain engine", st, plain),
                          ("out-of-range automaton state", bad, target)):
        keep = eng_.state()
        with pytest.raises(ValueError):
            eng_.load_state(s)
        now = eng_.state()
        for k, v in keep.items():                               # nothing was written
            if isinstance(v, torch.Tensor):
                assert torch.equal(v.cpu(), now[k].cpu()), (what, k)
    target.load_state(st)                                       # the right one loads
    assert torch.equal(target.state()["ctx_state"], st["ctx_state"])
    assert before["ctx_state"].abs().sum() == 0

    lens = [2] * 4
    mc_, xs = _ctc_setup(2, 3, lens)
    g2 = _ctc_graph(mc_, 2, lens, xs, 4, 1.5, seed=4)
    ce = CTCStreamBeamEngine(mc_, 2, 2, 4, context=g2)
    ce.step(xs[:, :2])
    cst = ce.state()
    with pytest.raises(ValueError):
        CTCStreamBeamEngine(mc_, 2, 2, 4).load_state(cst)
    with pytest.raises(ValueError):
        CTCStreamBeamEngine(mc_, 2, 2, 4, context=ContextGraph(g2.phrases[1:], CTC_TINY["vocab_size"], 1.5)) \
            .load_state(cst)
    bad = dict(cst, ctx_state=cst["ctx_state"].clone())
    bad["ctx_state"][0] = -1
    with pytest.raises(ValueError, match="outside"):
        CTCStreamBeamEngine(mc_, 2, 2, 4, context=g2).load_state(bad)


# ---- 6. the boost ---------------------------------------------------------------------------------------------------------
def test_boost_lifts_a_phrase_into_the_stream_and_zero_boost_changes_nothing():
    from edgedict_b200.stream_engine import BeamEngine, nbest_lists
    m, z, sd = _tiny()
    V = sd["joint.joint.2.weight"].shape[0]
    chunks = [torch.as_tensor(c[None]) for c in z["stream_chunks"]]
    W = 8
    _, _, _, enc, _ = _stream(m, chunks, W, max_pending=256)
    T = enc.shape[1]
    lists = nbest_lists(BeamEngine(m, 1, T, W, nbest=W).run(enc, torch.tensor([T], dtype=torch.int32,
                                                                              device=DEV)), 1, W, T)[0]
    target = next(tuple(h.tokens.tolist()) for h in lists[1:] if len(h.tokens))
    h_enc, _ = mt.encoder(sd, torch.cat(chunks, 1), None)
    lifted = None
    for beta in (0.25, 0.5, 1.0, 2.0, 4.0):
        graph = ContextGraph([list(target)], V, beta)
        if co.transducer_nbest(sd, h_enc, [h_enc.shape[1]], W, graph)[0][0][0] == target:
            lifted = graph
            break
    assert lifted is not None
    per, fl, _, _, _ = _stream(m, chunks, W, max_pending=256, context=lifted)
    assert tuple(_joined(per, fl)[0]) == target
    base = _stream(m, chunks, W, max_pending=256)
    zero = _stream(m, chunks, W, max_pending=256, context=ContextGraph([list(target)], V, 0.0))
    assert zero[0] == base[0] and zero[1] == base[1]
    assert torch.equal(_bits(zero[2]), _bits(base[2]))


# ---- 7. the decoders --------------------------------------------------------------------------------------------------------
class _Tok:
    vocab_size = 16

    class tokenizer:
        @staticmethod
        def id_to_token(i):
            return "<unk>" if i == 3 else "t%d</w>" % i

        @staticmethod
        def token_to_id(t):
            return 3 if t == "<unk>" else None


def _text(ids):
    return "".join("<unk>" if t == 3 else "t%d " % t for t in ids)


def test_decoders_give_the_offline_biased_text():
    from edgedict_b200.ctc import CTCStreamDecoder
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    m, z, sd = _tiny()
    V = sd["joint.joint.2.weight"].shape[0]
    xs = torch.as_tensor(z["stream_chunks"]).reshape(1, -1, 12)
    lists = m.beam_search(xs.to(DEV), None, W=4, nbest=4)[0]
    other = [h.tokens.tolist()[:3] for h in lists[1:] if len(h.tokens) >= 2]
    graph = ContextGraph(other + [[5, 6], [7, 8, 9]], V, 2.0)
    dec = PytorchStreamDecoder(FLAGS=None, transducer=m, transform=lambda f: f.transpose(1, 2), tokenizer=_Tok(),
                               beam_width=4, context=graph)
    # mixed chunk lengths: the decoder rebuilds its engine with the carried state and the same graph
    parts, t0 = [], 0
    for n in [2, 4, 2, 6, 2] * 8:
        if t0 >= xs.shape[1]:
            break
        parts.append(dec.decode(xs[:, t0:t0 + n]))
        t0 += n
    text = "".join(parts) + dec.flush()
    best, _ = m.beam_search(xs.to(DEV), None, W=4, context=graph)
    assert text == _text(best[0]) and len(text) > 0

    cm = _ctc_model(CTC_TINY, 13, scale=2.0)
    Vc = CTC_TINY["vocab_size"]
    g = torch.Generator().manual_seed(2)
    cx = torch.randn(1, 24, CTC_TINY["input_size"], generator=g)
    graph = ContextGraph([[1, 2], [3, 4, 5], [6, 7]], Vc, 1.5)
    cdec = CTCStreamDecoder(cm, lambda f: f.transpose(1, 2), _Tok(), beam_width=4, context=graph)
    parts = [cdec.decode(cx[:, i:i + n]) for i, n in ((0, 4), (4, 2), (6, 6), (12, 4), (16, 8))]
    text = "".join(parts) + cdec.flush()
    from edgedict_b200.stream_engine import CTCStreamBeamEngine
    ref = CTCStreamBeamEngine(cm, 1, 24, 4)
    ref.step(cx.to(DEV))
    from edgedict_b200 import ctc
    ids, _ = ctc.beam_search(ref.logprobs.view(1, ref.n_out, -1), [ref.n_out], 4, blank=cm.blank, context=graph)
    assert text == "".join(_Tok.tokenizer.id_to_token(int(k)).replace("</w>", " ") for k in ids[0])
