"""N-gram shallow fusion in the device beam searches (edgedict_b200/ngram.py, decode.cu flag 4096): unchanged
without a model, a zero weight changes nothing, the transducer and CTC lists against the host restatement
(tests/ngram_oracle.py), batch invariance, repeatability and CTA-count independence, the direction of the effect,
and a large model."""
import numpy as np
import pytest
import torch

from edgedict_b200.context import ContextGraph
from edgedict_b200.ngram import NgramLM
from oracle import model_torch as mt
from tests import ngram_oracle as no
from tests.test_gpu_beam_engine import SMALL
from tests.test_gpu_beam_lm import _lm_module
from tests.test_gpu_context import _random_graph, _same_output
from tests.test_gpu_nbest import _bits, _check_structure, _same_list, _tiny
from tests.test_oracle_lm import load_lm

pytestmark = pytest.mark.gpu


def _ngram(tmp_path, V, order, seed, n_sent=80, max_len=10, blank=0):
    m = no.estimate(no.corpus(seed, V, n_sent, max_len, blank=blank), order, V, blank=blank)
    return NgramLM(no.write_arpa(str(tmp_path / ("m%d_%d_%d.arpa" % (V, order, seed))), m), V, blank=blank)


# ---- 1. without a model: the plain search, bit for bit ---------------------------------------------------------------
@pytest.mark.parametrize("enc", ["LSTM", "GRU"])
@pytest.mark.parametrize("with_lm", [False, True])
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("K", [1, 2])
def test_transducer_without_ngram_is_unchanged(K, merge, with_lm, enc):
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
    for extra in ({}, dict(nbest=4)):
        base = m.beam_search(xs, xlen, W=4, merge=merge, max_symbols=K, **kw, **extra)
        got = m.beam_search(xs, xlen, W=4, merge=merge, max_symbols=K, ngram=None, ngram_weight=0.0, **kw, **extra)
        assert _same_output(got, base), extra


@pytest.mark.parametrize("with_lm", [False, True])
def test_ctc_without_ngram_is_unchanged(with_lm):
    from edgedict_b200 import ctc
    _, lsd = load_lm()
    kw = dict(lm=lsd, lm_weight=0.5, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(5)
    lp = (3.0 * torch.randn(4, 30, 16, generator=g)).log_softmax(-1).cuda()
    lens = [30, 17, 0, 25]
    for extra in ({}, dict(nbest=4)):
        base = ctc.beam_search(lp, lens, 4, **kw, **extra)
        assert _same_output(ctc.beam_search(lp, lens, 4, ngram=None, **kw, **extra), base), extra


# ---- 2. weight 0: the same ids and -log p -----------------------------------------------------------------------------
def test_zero_weight_changes_nothing(tmp_path):
    from edgedict_b200 import ctc
    g = torch.Generator().manual_seed(6)
    lp = (3.0 * torch.randn(3, 24, 16, generator=g)).log_softmax(-1).cuda()
    lens = [24, 11, 0]
    ng = _ngram(tmp_path, 16, 3, seed=1)
    graph = _random_graph(16, 10, 0.7, seed=2)
    for ctx in (None, graph):
        ids0, nl0 = ctc.beam_search(lp, lens, 8, context=ctx)
        ids1, nl1 = ctc.beam_search(lp, lens, 8, context=ctx, ngram=ng, ngram_weight=0.0)
        assert all(np.array_equal(a, b) for a, b in zip(ids0, ids1))
        assert torch.equal(nl0, nl1)
    m, z, sd = _tiny()
    V = sd["joint.joint.2.weight"].shape[0]
    ngt = _ngram(tmp_path, V, 3, seed=3, blank=m.blank)
    xs, xlen = torch.as_tensor(z["xs"]).cuda(), torch.as_tensor(z["xlen"])
    for K in (1, 2):
        ids0, nl0 = m.beam_search(xs, xlen, W=4, max_symbols=K)
        ids1, nl1 = m.beam_search(xs, xlen, W=4, max_symbols=K, ngram=ngt, ngram_weight=0.0)
        assert ids0 == ids1 and torch.equal(nl0, nl1)


# ---- 3. the restatement ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K, merge, ctx, order", [(1, True, False, 3), (1, False, False, 2), (2, True, False, 3),
                                                  (1, True, True, 3), (2, False, True, 4)])
def test_transducer_matches_restatement(tmp_path, K, merge, ctx, order):
    """Tiny model, ragged batch, W = 1 / 4 / 16 with nbest = W; bar 1e-4 relative as test_gpu_nbest.py."""
    m, z, sd = _tiny()
    V = sd["joint.joint.2.weight"].shape[0]
    ng = _ngram(tmp_path, V, order, seed=K + 2 * merge, blank=m.blank)
    graph = _random_graph(V, 12, 1.25, seed=K) if ctx else None
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    h, _ = mt.encoder(sd, xs, None)
    fr = [min(h.shape[1], int(mt.scale_length(h.shape[1], xlen)[b])) for b in range(xs.shape[0])]
    kw = dict(ngram=ng, ngram_weight=0.75, length_bonus=0.5, context=graph)
    for W in (1, 4, 16):
        want = no.transducer_nbest(sd, h, fr, W, ng, 0.75, K=K, merge=merge, blank=m.blank, length_bonus=0.5,
                                   graph=graph)
        got = m.beam_search(xs.cuda(), xlen, W=W, merge=merge, max_symbols=K, nbest=W, **kw)
        ids, nlp = m.beam_search(xs.cuda(), xlen, W=W, merge=merge, max_symbols=K, **kw)
        for b in range(len(fr)):
            _same_list(got[b], want[b], 1e-4, (W, b))
            _check_structure(got[b], fr[b], K, W, W, len(want[b]), merge)
            assert got[b][0].tokens.tolist() == ids[b] and _bits(got[b][0].nlogp) == _bits(nlp[b].item())


@pytest.mark.parametrize("ctx, order", [(False, 2), (False, 4), (True, 3)])
def test_ctc_matches_restatement(tmp_path, ctx, order):
    """V = 16, ragged batch with a length-0 utterance, W = 1 / 4 / 16; bar 1e-5 relative as test_gpu_nbest.py."""
    from edgedict_b200 import ctc
    g = torch.Generator().manual_seed(7)
    lp = (3.0 * torch.randn(3, 24, 16, generator=g)).log_softmax(-1)
    lens = [24, 15, 0]
    ng = _ngram(tmp_path, 16, order, seed=order)
    graph = _random_graph(16, 20, 0.9, seed=3) if ctx else None
    for W in (1, 4, 16):
        want = [no.ctc_nbest(lp[b].numpy(), lens[b], W, ng, 0.6, length_bonus=0.25, graph=graph) for b in range(3)]
        kw = dict(ngram=ng, ngram_weight=0.6, length_bonus=0.25, context=graph)
        got = ctc.beam_search(lp.cuda(), lens, W, nbest=W, **kw)
        ids, nlp = ctc.beam_search(lp.cuda(), lens, W, **kw)
        for b in range(3):
            _same_list(got[b], want[b], 1e-5, (W, b))
            _check_structure(got[b], max(lens[b], 1), 1, W, W, len(want[b]), True, ctc=True)
            assert np.array_equal(got[b][0].tokens, ids[b]) and _bits(got[b][0].nlogp) == _bits(nlp[b].item())


# ---- 4. exhaustive ranking on tiny V and T ---------------------------------------------------------------------------------
def test_ctc_exhaustive_ranking(tmp_path):
    """W = V^T keeps every prefix: the N-best list is every distinct collapsed sequence ranked by its score."""
    import itertools
    from edgedict_b200 import ctc
    V, T = 3, 5
    ng = _ngram(tmp_path, V, 3, seed=11, n_sent=20, max_len=5)
    g = torch.Generator().manual_seed(8)
    lp = (2.0 * torch.randn(1, T, V, generator=g)).log_softmax(-1)
    W = min(V ** T, 64)
    got = ctc.beam_search(lp.cuda(), [T], W, nbest=W, ngram=ng, ngram_weight=0.5)[0]
    y = lp[0].double().numpy()
    tot = {}
    for path in itertools.product(range(V), repeat=T):
        seq, prev = [], -1
        for k in path:
            if k != 0 and k != prev:
                seq.append(k)
            prev = k
        tot[tuple(seq)] = np.logaddexp(tot.get(tuple(seq), -np.inf), sum(y[t, k] for t, k in enumerate(path)))
    ref = {}
    for seq, v in tot.items():
        s, lm = ng.start, 0.0
        for k in seq:
            s, gk = ng.step(s, k)
            lm += gk
        ref[seq] = v + 0.5 * (lm + float(ng.end[s]))
    fin = [h for h in got if np.isfinite(h.nlogp)]          # prefixes no path reaches stay in the beam at -inf
    assert len(fin) == len(ref) and {tuple(h.tokens.tolist()) for h in fin} == set(ref)
    for h in fin:
        v = ref[tuple(h.tokens.tolist())]
        assert abs(-h.nlogp - v) <= 1e-4 * (1 + abs(v))
    best = max(ref.values())
    assert ref[tuple(got[0].tokens.tolist())] >= best - 1e-4 * (1 + abs(best))


# ---- 5. batch invariance, repeatability, CTA count ----------------------------------------------------------------------
def test_batch_invariance_repeatability_and_cta_count(tmp_path):
    from edgedict_b200.stream_engine import BeamEngine, CTCBeamEngine, nbest_lists
    ng = _ngram(tmp_path, 16, 3, seed=12)
    g = torch.Generator().manual_seed(9)
    lp = (3.0 * torch.randn(5, 20, 16, generator=g)).log_softmax(-1).cuda()
    lens = torch.tensor([20, 3, 17, 0, 20], dtype=torch.int32).cuda()
    outs = []
    for mc in (0, 1, 3, 17):
        e = CTCBeamEngine(5, 20, 16, 8, ngram=ng, ngram_weight=0.7, length_bonus=0.2, max_ctas=mc, nbest=4)
        for _ in range(2):
            outs.append(e.run(lp, lens).clone())
    assert all(torch.equal(o, outs[0]) for o in outs)
    full = nbest_lists(outs[0], 5, 4, 20)
    for b in range(5):
        e1 = CTCBeamEngine(1, 20, 16, 8, ngram=ng, ngram_weight=0.7, length_bonus=0.2, nbest=4)
        one = nbest_lists(e1.run(lp[b:b + 1], lens[b:b + 1]), 1, 4, 20)[0]
        assert len(one) == len(full[b]) and all(
            np.array_equal(x.tokens, y.tokens) and _bits(x.nlogp) == _bits(y.nlogp) for x, y in zip(one, full[b]))
    m, z, sd = _tiny()
    V = sd["joint.joint.2.weight"].shape[0]
    ngt = _ngram(tmp_path, V, 3, seed=13, blank=m.blank)
    h = mt.encoder(sd, torch.as_tensor(z["xs"]), None)[0].cuda()
    fr = torch.full((h.shape[0],), h.shape[1], dtype=torch.int32).cuda()
    res = []
    for mc in (0, 1, 3, 17):
        e = BeamEngine(m, h.shape[0], h.shape[1], 4, blank=m.blank, max_ctas=mc, ngram=ngt, ngram_weight=0.5,
                       max_symbols=2, nbest=4)
        res.append(e.run(h, fr).clone())
        res.append(e.run(h, fr).clone())
    assert all(torch.equal(r, res[0]) for r in res)


# ---- 6. effect ---------------------------------------------------------------------------------------------------------
def test_weight_lifts_the_sequence_the_model_prefers(tmp_path):
    """Two tokens equally likely to the acoustics at every frame: with the n-gram, the best hypothesis follows the
    model's preferred continuation, and a larger weight raises the model's share of the score."""
    from edgedict_b200 import ctc
    text = ("\\data\\\nngram 1=3\nngram 2=2\n\n\\1-grams:\n-0.5\t1\t-0.3\n-0.5\t2\t-0.3\n-0.6\t</s>\n\n"
            "\\2-grams:\n-0.05\t1 2\n-0.05\t2 1\n\n\\end\\\n")
    p = tmp_path / "alt.arpa"
    p.write_text(text)
    ng = NgramLM(str(p), 3)
    T = 6
    lp = torch.full((1, T, 3), -30.0)
    lp[0, :, 1] = lp[0, :, 2] = np.log(0.5)
    lp[0, :, 0] = -1.0
    lp = lp.log_softmax(-1).cuda()
    ids0, _ = ctc.beam_search(lp, [T], 8)
    ids, _ = ctc.beam_search(lp, [T], 8, ngram=ng, ngram_weight=2.0)
    seq = ids[0].tolist()
    assert len(seq) >= 2 and all(a != b for a, b in zip(seq, seq[1:]))      # 1 2 1 2 ...: the model's alternation


# ---- 7. a large model ----------------------------------------------------------------------------------------------------
def test_large_model_decodes(tmp_path):
    """A 3-gram over V = 1024 with about 10^5 children decodes, and agrees with the host walk on its best list."""
    from edgedict_b200 import ctc
    V = 1024
    ng = _ngram(tmp_path, V, 3, seed=21, n_sent=6000, max_len=20)
    assert ng.n_children > 50000
    g = torch.Generator().manual_seed(10)
    lp = (2.0 * torch.randn(2, 40, V, generator=g)).log_softmax(-1)
    got = ctc.beam_search(lp.cuda(), [40, 31], 4, nbest=4, ngram=ng, ngram_weight=0.5)
    for b, n in enumerate((40, 31)):
        want = no.ctc_nbest(lp[b].numpy(), n, 4, ng, 0.5)
        _same_list(got[b], want, 1e-5, b)
