"""Contextual biasing on the device (decode.cu flag 2048 in BEAM_SELECT, CTC_BEAM and BEAM_FINAL; edgedict_b200/context.py):
no context and an empty graph are the plain search bit for bit, the biased lists equal the restatement
(tests/context_oracle.py) and, when nothing is pruned, the exhaustive ranking by log p + banked bonus; the effect of
the boost, merging, the bitwise invariants, graphs swapped in one process and a graph near the table cap."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from edgedict_b200.context import MAX_TABLE, ContextGraph
from oracle import model_torch as mt
from tests import context_oracle as co
from tests import ctc_beam_oracle as cbo
from tests import nbest_oracle as no
from tests.test_gpu_beam_engine import SMALL, _scaled_model
from tests.test_gpu_beam_lm import _lm_module
from tests.test_gpu_nbest import TINY, _bits, _check_structure, _lists_equal, _same_list, _tiny
from tests.test_oracle_lm import load_lm

pytestmark = pytest.mark.gpu


def _random_graph(V, n, beta, seed, lo=1, hi=4):
    rng = random.Random(seed)
    return ContextGraph([[rng.randrange(1, V) for _ in range(rng.randint(lo, hi))] for _ in range(n)], V, beta)


def _same_output(a, b):
    if isinstance(a, list):
        return all(_lists_equal(x, y) for x, y in zip(a, b)) and len(a) == len(b)
    ids_a, nl_a = a
    ids_b, nl_b = b
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(ids_a, ids_b)) and \
        torch.equal(nl_a.view(torch.int32), nl_b.view(torch.int32))


# ---- 1. no context / an empty graph: the plain search, bit for bit -----------------------------------------------------
@pytest.mark.parametrize("enc", ["LSTM", "GRU"])
@pytest.mark.parametrize("with_lm", [False, True])
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("K", [1, 2])
def test_transducer_without_context_is_unchanged(K, merge, with_lm, enc):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(4)
    m = Transducer(output_loss=False, module_type=enc, **SMALL).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)
    m.cuda()
    kw = dict(lm=_lm_module(96, 16, 48, 2, 4.0, seed=1).cuda(), lm_weight=0.4, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(K)
    xs = torch.randn(3, 30, SMALL["input_size"], generator=g).cuda()
    xlen = torch.tensor([30, 17, 0])
    empty = ContextGraph([], SMALL["vocab_size"], 2.0)
    for extra in ({}, dict(nbest=4)):
        base = m.beam_search(xs, xlen, W=4, merge=merge, max_symbols=K, **kw, **extra)
        for ctx in (None, empty):
            got = m.beam_search(xs, xlen, W=4, merge=merge, max_symbols=K, context=ctx, **kw, **extra)
            assert _same_output(got, base), (ctx, extra)


@pytest.mark.parametrize("with_lm", [False, True])
def test_ctc_without_context_is_unchanged(with_lm):
    from edgedict_b200 import ctc
    _, lsd = load_lm()
    kw = dict(lm=lsd, lm_weight=0.5, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(5)
    lp = (3.0 * torch.randn(4, 30, 16, generator=g)).log_softmax(-1).cuda()
    lens = [30, 17, 0, 25]
    empty = ContextGraph([], 16, 1.0)
    for extra in ({}, dict(nbest=4)):
        base = ctc.beam_search(lp, lens, 4, **kw, **extra)
        for ctx in (None, empty):
            assert _same_output(ctc.beam_search(lp, lens, 4, context=ctx, **kw, **extra), base), (ctx, extra)


# ---- 2. with phrases: the restatement ---------------------------------------------------------------------------------
@pytest.mark.parametrize("K, merge, with_lm", [(1, True, False), (1, False, False), (2, True, False),
                                               (1, True, True), (2, True, True)])
def test_transducer_matches_restatement(K, merge, with_lm):
    """Tiny model, ragged batch, bar 1e-4 relative as test_gpu_nbest.py; W = 1 / 4 / 16 with nbest = W."""
    m, z, sd = _tiny()
    _, lsd = load_lm()
    V = sd["joint.joint.2.weight"].shape[0]
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    okw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    dkw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    h, _ = mt.encoder(sd, xs, None)
    fr = [min(h.shape[1], int(mt.scale_length(h.shape[1], xlen)[b])) for b in range(xs.shape[0])]
    graph = _random_graph(V, 12, 1.25, seed=K + 2 * merge)
    for W in (1, 4, 16):
        want = co.transducer_nbest(sd, h, fr, W, graph, K=K, merge=merge, **okw)
        got = m.beam_search(xs.cuda(), xlen, W=W, merge=merge, max_symbols=K, nbest=W, context=graph, **dkw)
        ids, nlp = m.beam_search(xs.cuda(), xlen, W=W, merge=merge, max_symbols=K, context=graph, **dkw)
        for b in range(len(fr)):
            _same_list(got[b], want[b], 1e-4, (W, b))
            _check_structure(got[b], fr[b], K, W, W, len(want[b]), merge)
            assert got[b][0].tokens.tolist() == ids[b] and _bits(got[b][0].nlogp) == _bits(nlp[b].item())


@pytest.mark.parametrize("with_lm", [False, True])
def test_ctc_matches_restatement(with_lm):
    """V = 16, ragged batch with a length-0 utterance, W = 1 / 4 / 16; bar 1e-5 relative as test_gpu_nbest.py."""
    from edgedict_b200 import ctc
    _, lsd = load_lm()
    kw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    dkw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    g = torch.Generator().manual_seed(7)
    lp = (3.0 * torch.randn(3, 24, 16, generator=g)).log_softmax(-1)
    lens = [24, 15, 0]
    graph = _random_graph(16, 20, 0.9, seed=3)
    for W in (1, 4, 16):
        want = co.ctc_batch_nbest(lp.numpy(), lens, W, graph, **kw)
        got = ctc.beam_search(lp.cuda(), lens, W, nbest=W, context=graph, **dkw)
        ids, nlp = ctc.beam_search(lp.cuda(), lens, W, context=graph, **dkw)
        for b in range(3):
            _same_list(got[b], want[b], 1e-5, (W, b))
            _check_structure(got[b], max(lens[b], 1), 1, W, W, len(want[b]), True, ctc=True)
            assert np.array_equal(got[b][0].tokens, ids[b]) and _bits(got[b][0].nlogp) == _bits(nlp[b].item())


# ---- 3. exhaustive: nothing pruned, the ranking by log p + banked --------------------------------------------------------
def _check_exhaustive(hyps, refs_of, bar_of):
    refs = []
    for x in hyps:
        ref = refs_of(tuple(x.tokens.tolist()))
        bar = bar_of(x, ref)
        if ref == -np.inf:
            assert x.nlogp == np.inf
        else:
            assert abs(-x.nlogp - ref) <= bar, (x, ref)
        refs.append((ref, bar))
    for (r1, b1), (r2, b2) in zip(refs, refs[1:]):
        assert r1 >= r2 or r2 - r1 <= 2 * max(b1, b2)


@pytest.mark.parametrize("V, T", [(3, 6), (4, 5)])
def test_ctc_exhaustive_ranking(V, T):
    from edgedict_b200 import ctc
    prefixes = cbo.all_prefixes(V, T)
    W = len(prefixes)
    g = torch.Generator().manual_seed(V * 100 + T)
    lp = (1.5 * torch.randn(1, T, V, generator=g)).log_softmax(-1)
    phrases = [[1, 2], [2, 2, 1], [V - 1]]
    graph = ContextGraph(phrases, V, 1.5)
    hyps = ctc.beam_search(lp.cuda(), [T], W, nbest=W, context=graph)[0]
    assert sorted(tuple(h.tokens.tolist()) for h in hyps) == sorted(prefixes)
    ymax = float(lp[0].abs().max())

    def ref(p):
        lpp = (-float(F.ctc_loss(lp[0].double()[:, None], torch.tensor([p]), [T], [len(p)], reduction="none"))
               if p else float(lp[0, :, 0].double().sum()))
        return lpp + co.banked(phrases, p, 1.5)
    _check_exhaustive(hyps, ref, lambda x, r: 2.0 ** -20 * T * (1 + abs(r) + ymax + 1.5 * T))


@pytest.mark.parametrize("seed", [0, 1])
def test_transducer_exhaustive_ranking(seed):
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import BeamEngine, nbest_lists
    torch.manual_seed(seed)
    m = Transducer(output_loss=False, **TINY).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(3.0)
    sd64 = {k: v.detach().double() for k, v in m.state_dict().items()}
    m.cuda()
    g = torch.Generator().manual_seed(seed)
    T = 4
    h = torch.randn(1, T, TINY["enc_proj_size"], generator=g)
    seqs = no.all_sequences(4, T)
    W = 4 * len(no.all_sequences(4, T - 1))
    phrases = [[1, 2], [3, 3], [2, 1, 3]]
    graph = ContextGraph(phrases, 4, 1.25)
    eng = BeamEngine(m, 1, T, W, nbest=W, context=graph)
    hyps = nbest_lists(eng.run(h.cuda(), torch.tensor([T], dtype=torch.int32).cuda()), 1, W, T)[0]
    assert sorted(tuple(x.tokens.tolist()) for x in hyps) == sorted(seqs)

    def ref(p):
        return no.transducer_sequence_logprob(sd64, h[0].double(), T, p) + co.banked(phrases, p, 1.25)
    _check_exhaustive(hyps, ref, lambda x, r: 2.0 ** -20 * (T + len(x.tokens)) * (1 + abs(r) + 1.25 * T))


# ---- 4. effect of the boost --------------------------------------------------------------------------------------------
def test_boost_lifts_a_phrase_and_zero_boost_changes_nothing():
    from edgedict_b200 import ctc
    g = torch.Generator().manual_seed(11)
    lp = (2.0 * torch.randn(1, 20, 12, generator=g)).log_softmax(-1)
    W = 8
    base = ctc.beam_search(lp.cuda(), [20], W, nbest=W)[0]
    target = tuple(base[2].tokens.tolist())
    assert target
    lifted = None
    for beta in (0.25, 0.5, 1.0, 2.0, 4.0):                 # the least boost the restatement says suffices
        graph = ContextGraph([list(target)], 12, beta)
        if co.ctc_nbest(lp[0].numpy(), 20, W, graph)[0][0] == target:
            lifted = graph
            break
    assert lifted is not None
    got = ctc.beam_search(lp.cuda(), [20], W, nbest=W, context=lifted)[0]
    assert tuple(got[0].tokens.tolist()) == target
    zero = ctc.beam_search(lp.cuda(), [20], W, nbest=W, context=ContextGraph([list(target)], 12, 0.0))[0]
    assert [tuple(h.tokens.tolist()) for h in zero] == [tuple(h.tokens.tolist()) for h in base]
    assert [h.nlogp for h in zero] == [h.nlogp for h in base]

    m, z, sd = _tiny()
    xs, xlen = torch.as_tensor(z["xs"]).cuda(), torch.as_tensor(z["xlen"])
    V = sd["joint.joint.2.weight"].shape[0]
    base = m.beam_search(xs, xlen, W=W, nbest=W)
    b = next(i for i in range(len(base)) if len(base[i]) > 2 and len(base[i][2].tokens))
    target = tuple(base[b][2].tokens.tolist())
    h, _ = mt.encoder(sd, torch.as_tensor(z["xs"]), None)
    fr = [min(h.shape[1], int(mt.scale_length(h.shape[1], xlen)[i])) for i in range(xs.shape[0])]
    lifted = None
    for beta in (0.25, 0.5, 1.0, 2.0, 4.0):
        graph = ContextGraph([list(target)], V, beta)
        if co.transducer_nbest(sd, h[b:b + 1], fr[b:b + 1], W, graph)[0][0][0] == target:
            lifted = graph
            break
    assert lifted is not None
    assert tuple(m.beam_search(xs, xlen, W=W, nbest=W, context=lifted)[b][0].tokens.tolist()) == target
    zero = m.beam_search(xs, xlen, W=W, nbest=W, context=ContextGraph([list(target)], V, 0.0))
    for x, y in zip(zero, base):
        assert [tuple(h.tokens.tolist()) for h in x] == [tuple(h.tokens.tolist()) for h in y]
        assert [h.nlogp for h in x] == [h.nlogp for h in y]


# ---- 5. merging, invariants, graph swaps, a graph near the cap ----------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2])
def test_merge_folds_exactly_equal_sequences(K):
    """With merge the biased list holds distinct sequences; each equals the unmerged search's best copy or a log-add
    of its copies, so the merged list's sequences are those of the unmerged list with duplicates removed among the
    ones that survive in both."""
    m = _scaled_model(SMALL, seed=4)
    g = torch.Generator().manual_seed(6)
    h = torch.randn(3, 12, SMALL["enc_proj_size"], generator=g).cuda()
    graph = _random_graph(SMALL["vocab_size"], 40, 1.0, seed=9, hi=3)
    from edgedict_b200.stream_engine import BeamEngine, nbest_lists
    lens = torch.tensor([12, 7, 10], dtype=torch.int32).cuda()
    for merge in (True, False):
        eng = BeamEngine(m, 3, 12, 8, merge=merge, max_symbols=K, nbest=8, context=graph)
        hyps = nbest_lists(eng.run(h, lens), 3, 8, 12 * K)
        for b in range(3):
            seqs = [tuple(x.tokens.tolist()) for x in hyps[b]]
            if merge:
                assert len(set(seqs)) == len(seqs)
            else:
                assert len(set(seqs)) <= len(seqs)


@pytest.mark.parametrize("K", [1, 2])
def test_transducer_batch_invariance_repeatability_and_cta_count(K):
    from edgedict_b200.stream_engine import BeamEngine, nbest_lists
    m = _scaled_model(SMALL, seed=4)
    kw = dict(lm=_lm_module(96, 16, 48, 2, 4.0, seed=3).cuda(), lm_weight=0.7, length_bonus=0.3)
    graph = _random_graph(SMALL["vocab_size"], 60, 1.0, seed=K, hi=3)
    g = torch.Generator().manual_seed(2)
    T, W = 20, 6
    h = torch.randn(4, T, SMALL["enc_proj_size"], generator=g).cuda()
    lens = [20, 11, 1, 0]
    eng = BeamEngine(m, 4, T, W, max_symbols=K, nbest=W, context=graph, **kw)
    buf = eng.run(h, torch.tensor(lens, dtype=torch.int32).cuda()).clone()
    assert torch.equal(buf, eng.run(h, torch.tensor(lens, dtype=torch.int32).cuda()))
    for ctas in (1, 3):
        eng.max_ctas = ctas
        assert torch.equal(buf, eng.run(h, torch.tensor(lens, dtype=torch.int32).cuda())), ctas
    full = nbest_lists(buf, 4, W, T * K)
    for b, n in enumerate(lens[:3]):
        one = BeamEngine(m, 1, n, W, max_symbols=K, nbest=W, context=graph, **kw)
        alone = nbest_lists(one.run(h[b:b + 1, :n].contiguous(), torch.tensor([n], dtype=torch.int32).cuda()), 1,
                            W, max(n * K, 1))
        assert _lists_equal(alone[0], full[b]), b


def test_ctc_batch_invariance_repeatability_and_cta_count():
    from edgedict_b200.stream_engine import CTCBeamEngine, nbest_lists
    g = torch.Generator().manual_seed(3)
    T, V, W = 28, 40, 8
    lp = (3.0 * torch.randn(4, T, V, generator=g)).log_softmax(-1).cuda()
    lens = torch.tensor([28, 11, 0, 20], dtype=torch.int32).cuda()
    graph = _random_graph(V, 80, 0.8, seed=4, hi=3)
    eng = CTCBeamEngine(4, T, V, W, nbest=W, device="cuda", context=graph)
    buf = eng.run(lp, lens).clone()
    assert torch.equal(buf, eng.run(lp, lens))
    for ctas in (1, 3):
        eng.max_ctas = ctas
        assert torch.equal(buf, eng.run(lp, lens)), ctas
    full = nbest_lists(buf, 4, W, T)
    for b in (0, 1, 3):
        n = int(lens[b])
        one = CTCBeamEngine(1, n, V, W, nbest=W, device="cuda", context=graph)
        alone = nbest_lists(one.run(lp[b:b + 1, :n], lens[b:b + 1]), 1, W, n)
        assert _lists_equal(alone[0], full[b]), b


def test_graphs_swapped_in_one_process():
    from edgedict_b200 import ctc
    g = torch.Generator().manual_seed(8)
    lp = (2.0 * torch.randn(2, 20, 16, generator=g)).log_softmax(-1)
    A = _random_graph(16, 15, 1.0, seed=1)
    Bg = _random_graph(16, 15, 1.0, seed=2)
    ra = ctc.beam_search(lp.cuda(), [20, 14], 4, nbest=4, context=A)
    rb = ctc.beam_search(lp.cuda(), [20, 14], 4, nbest=4, context=Bg)
    ra2 = ctc.beam_search(lp.cuda(), [20, 14], 4, nbest=4, context=A)
    assert _same_output(ra, ra2)
    for graph, got in ((A, ra), (Bg, rb)):
        want = co.ctc_batch_nbest(lp.numpy(), [20, 14], 4, graph)
        for b in range(2):
            _same_list(got[b], want[b], 1e-5, b)
    m, z, sd = _tiny()
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    V = sd["joint.joint.2.weight"].shape[0]
    A, Bg = _random_graph(V, 10, 1.0, seed=5), _random_graph(V, 10, 1.0, seed=6)
    h, _ = mt.encoder(sd, xs, None)
    fr = [min(h.shape[1], int(mt.scale_length(h.shape[1], xlen)[b])) for b in range(xs.shape[0])]
    outs = [m.beam_search(xs.cuda(), xlen, W=4, nbest=4, context=c) for c in (A, Bg, A)]
    assert _same_output(outs[0], outs[2])
    for graph, got in ((A, outs[0]), (Bg, outs[1])):
        want = co.transducer_nbest(sd, h, fr, 4, graph)
        for b in range(len(fr)):
            _same_list(got[b], want[b], 1e-4, b)


def test_graph_near_the_cap():
    """About 2000 phrases of 2-6 tokens over V = 2048: n_states x V within 15 % of 2^24.  The phrases' tokens are
    made likely in the log-probs so that the automaton leaves the root."""
    from edgedict_b200 import ctc
    V, T = 2048, 24
    rng = random.Random(12)
    phrases = [[rng.randrange(1, V) for _ in range(rng.randint(2, 6))] for _ in range(2000)]
    graph = ContextGraph(phrases, V, 1.0)
    assert 0.85 * MAX_TABLE <= graph.n_states * V <= MAX_TABLE
    g = torch.Generator().manual_seed(13)
    lp = 2.0 * torch.randn(2, T, V, generator=g)
    for b in range(2):
        t = 0
        for ph in phrases[3 * b:3 * b + 3]:
            for k in ph:
                if t < T:
                    lp[b, t, k] += 6.0
                    t += 1
    lp = lp.log_softmax(-1)
    want = co.ctc_batch_nbest(lp.numpy(), [T, T - 5], 4, graph)
    got = ctc.beam_search(lp.cuda(), [T, T - 5], 4, nbest=4, context=graph)
    for b in range(2):
        _same_list(got[b], want[b], 1e-5, b)
