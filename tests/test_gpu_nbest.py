"""N-best beam search on the device (``beam_search(nbest=N)``: BEAM_FINAL's ranked walk in csrc/decode.cu, nbest_lists
in stream_engine): the head of every list is the best-only call bit for bit, the whole list is the restatement's
(tests/nbest_oracle.py), the exact search when nothing is pruned, the frames form a real lattice path, the structure of
the lists, and the bitwise invariants of the best-only output."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_torch as mt
from tests import ctc_beam_oracle as cbo
from tests import nbest_oracle as no
from tests.test_gpu_beam_engine import SMALL, _scaled_model
from tests.test_gpu_beam_lm import _lm_module
from tests.test_oracle_lm import load_lm
from tests.util import load_tiny, to_t

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24


def _bits(x):
    return int(np.float32(x).view(np.int32))


def _tiny():
    from edgedict_b200.rnnt.models import Transducer
    z, cfg, sd, _ = load_tiny()
    sd = dict(to_t(sd))
    m = Transducer(output_loss=False, **cfg)
    m.load_state_dict(sd)
    return m.cuda().eval(), z, sd


def _check_structure(hyps, frames_b, K, W, N, live, merge, ctc=False):
    assert len(hyps) == min(N, live)
    seqs = [tuple(h.tokens.tolist()) for h in hyps]
    for h in hyps:
        f = h.frames.tolist()
        assert len(f) == len(h.tokens) and all(0 <= x < frames_b for x in f)
        assert f == sorted(f) and all(f.count(x) <= K for x in set(f))
        if K == 1 or ctc:
            assert len(set(f)) == len(f)
    if merge:
        assert len(set(seqs)) == len(seqs)
    nl = [h.nlogp for h in hyps]
    assert nl == sorted(nl)


# ---- 1. the head is the best-only call, bit for bit -------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["LSTM", "GRU"])
@pytest.mark.parametrize("with_lm", [False, True])
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("K", [1, 2, 4])
def test_transducer_head_is_the_best_only_call(K, merge, with_lm, enc):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(4)
    m = Transducer(output_loss=False, module_type=enc, **SMALL).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)
        m.joint.joint[2].bias[0] += 1.0
    m.cuda()
    kw = dict(lm=_lm_module(96, 16, 48, 2, 4.0, seed=1).cuda(), lm_weight=0.4, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(K)
    xs = torch.randn(4, 40, SMALL["input_size"], generator=g).cuda()
    xlen = torch.tensor([40, 23, 0, 31])
    for W in (1, 4, 7):
        ids, nlp = m.beam_search(xs, xlen, W=W, merge=merge, max_symbols=K, **kw)
        hyps = m.beam_search(xs, xlen, W=W, merge=merge, max_symbols=K, nbest=W, **kw)
        assert len(hyps) == 4
        for b in range(4):
            assert hyps[b][0].tokens.tolist() == ids[b], (W, b)
            assert _bits(hyps[b][0].nlogp) == _bits(nlp[b].item()), (W, b)
        assert len(hyps[2]) == 1 and len(hyps[2][0].tokens) == 0 and hyps[2][0].nlogp == 0.0
        assert sum(len(i) for i in ids) > 0 or with_lm


@pytest.mark.parametrize("with_lm", [False, True])
def test_ctc_head_is_the_best_only_call(with_lm):
    from edgedict_b200 import ctc
    _, lsd = load_lm()
    kw = dict(lm=lsd, lm_weight=0.5, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(5)
    lp = (3.0 * torch.randn(4, 30, 16, generator=g)).log_softmax(-1).cuda()
    lens = [30, 17, 0, 25]
    for W in (1, 4, 16):
        ids, nlp = ctc.beam_search(lp, lens, W, **kw)
        hyps = ctc.beam_search(lp, lens, W, nbest=W, **kw)
        for b in range(4):
            assert np.array_equal(hyps[b][0].tokens, ids[b]), (W, b)
            assert _bits(hyps[b][0].nlogp) == _bits(nlp[b].item()), (W, b)
        assert len(hyps[2]) == 1 and len(hyps[2][0].tokens) == 0 and hyps[2][0].nlogp == 0.0


def test_ctc_encoder_head_is_the_best_only_call():
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(2)
    m = CTCEncoder(vocab_size=32, input_size=12, enc_hidden_size=32, enc_layers=2, enc_dropout=0.0,
                   proj_size=24).cuda().eval()
    xs = torch.randn(3, 20, 12).cuda()
    ids, nlp = m.beam_search(xs, [20, 9, 14], W=4)
    hyps = m.beam_search(xs, [20, 9, 14], W=4, nbest=3)
    for b in range(3):
        assert np.array_equal(hyps[b][0].tokens, ids[b]) and _bits(hyps[b][0].nlogp) == _bits(nlp[b].item())
        assert 1 <= len(hyps[b]) <= 3


# ---- 2. the whole list is the restatement's ---------------------------------------------------------------------------
def _same_list(got, want, rtol, tag):
    assert [tuple(h.tokens.tolist()) for h in got] == [w[0] for w in want], tag
    assert [tuple(h.frames.tolist()) for h in got] == [w[1] for w in want], tag
    for h, w in zip(got, want):
        if np.isinf(w[2]):
            assert h.nlogp == w[2], tag
        else:
            assert abs(h.nlogp - w[2]) <= rtol * abs(w[2]), (tag, h.nlogp, w[2])


@pytest.mark.parametrize("K, merge, with_lm", [(1, True, False), (1, False, False), (2, True, False),
                                               (2, False, False), (1, True, True), (2, True, True)])
def test_transducer_list_matches_restatement(K, merge, with_lm):
    """Tiny model, ragged batch; bar 1e-4 relative as the best-only restatement tests of the transducer beam."""
    m, z, sd = _tiny()
    _, lsd = load_lm()
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    okw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    dkw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    h, _ = mt.encoder(sd, xs, None)
    fr = [min(h.shape[1], int(mt.scale_length(h.shape[1], xlen)[b])) for b in range(xs.shape[0])]
    for W in (4, 8):
        want = no.transducer_nbest(sd, h, fr, W, K=K, merge=merge, **okw)
        got = m.beam_search(xs.cuda(), xlen, W=W, merge=merge, max_symbols=K, nbest=W, **dkw)
        for b in range(len(fr)):
            _same_list(got[b], want[b], 1e-4, (W, b))
            _check_structure(got[b], fr[b], K, W, W, len(want[b]), merge)


@pytest.mark.parametrize("with_lm", [False, True])
def test_ctc_list_matches_restatement(with_lm):
    """V = 16, ragged batch with a length-0 utterance, W = 4 / 16; bar 1e-5 relative as test_gpu_ctc_beam.py."""
    from edgedict_b200 import ctc
    _, lsd = load_lm()
    kw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    dkw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    g = torch.Generator().manual_seed(7)
    lp = (3.0 * torch.randn(3, 24, 16, generator=g)).log_softmax(-1)
    lens = [24, 15, 0]
    for W in (4, 16):
        want = no.ctc_batch_nbest(lp.numpy(), lens, W, **kw)
        got = ctc.beam_search(lp.cuda(), lens, W, nbest=W, **dkw)
        for b in range(3):
            _same_list(got[b], want[b], 1e-5, (W, b))
            _check_structure(got[b], max(lens[b], 1), 1, W, W, len(want[b]), True, ctc=True)


# ---- 3. exact search when nothing is pruned ---------------------------------------------------------------------------
@pytest.mark.parametrize("V, T", [(2, 6), (3, 6), (4, 5)])
def test_ctc_exact_without_pruning(V, T):
    """W = the number of prefixes: the list is every prefix, ordered by F.ctc_loss in fp64 except for swaps inside
    twice test_exact_without_pruning's bar 2^-20 T (1 + |log p| + max|y|); token i entered at frame i."""
    from edgedict_b200 import ctc
    prefixes = cbo.all_prefixes(V, T)
    W = len(prefixes)
    g = torch.Generator().manual_seed(V * 100 + T)
    lp = (1.5 * torch.randn(2, T, V, generator=g)).log_softmax(-1)
    hyps = ctc.beam_search(lp.cuda(), [T, T], W, nbest=W)
    for b in range(2):
        assert sorted(tuple(h.tokens.tolist()) for h in hyps[b]) == sorted(prefixes)
        ymax = float(lp[b].abs().max())
        refs = []
        for h in hyps[b]:
            p = tuple(h.tokens.tolist())
            assert h.frames.tolist() == list(range(len(p)))
            ref = (-float(F.ctc_loss(lp[b].double()[:, None], torch.tensor([p]), [T], [len(p)], reduction="none"))
                   if p else float(lp[b, :, 0].double().sum()))
            bar = 2.0 ** -20 * T * (1 + abs(ref) + ymax)
            if ref == -np.inf:
                assert h.nlogp == np.inf
            else:
                assert abs(-h.nlogp - ref) <= bar, (p, h.nlogp, ref)
            refs.append((ref, bar))
        for (r1, b1), (r2, b2) in zip(refs, refs[1:]):
            assert r1 >= r2 or r2 - r1 <= 2 * max(b1, b2)


TINY = dict(vocab_embed_size=8, vocab_size=4, input_size=6, enc_hidden_size=8, enc_layers=1, enc_dropout=0.0,
            enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0.0, dec_proj_size=8, joint_size=8)


@pytest.mark.parametrize("seed", [0, 1])
def test_transducer_exact_without_pruning(seed):
    """V = 4 (3 tokens), T' = 4, K = 1 with merge.  The selection takes the top W candidates before it merges, so W =
    160, the candidates of the last frame (40 hypotheses x 4 tokens), keeps all 121 sequences of at most 4 tokens.  The
    list is every sequence, each scored by the fp64 sum over its alignments within 2^-20 (T' + U) (1 + |log p|), in that
    order except for swaps inside twice the bar."""
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
    eng = BeamEngine(m, 1, T, W, nbest=W)
    hyps = nbest_lists(eng.run(h.cuda(), torch.tensor([T], dtype=torch.int32).cuda()), 1, W, T)[0]
    assert sorted(tuple(x.tokens.tolist()) for x in hyps) == sorted(seqs)
    refs = []
    for x in hyps:
        ref = no.transducer_sequence_logprob(sd64, h[0].double(), T, tuple(x.tokens.tolist()))
        bar = 2.0 ** -20 * (T + len(x.tokens)) * (1 + abs(ref))
        assert abs(-x.nlogp - ref) <= bar, (x, ref)
        refs.append((ref, bar))
    for (r1, b1), (r2, b2) in zip(refs, refs[1:]):
        assert r1 >= r2 or r2 - r1 <= 2 * max(b1, b2)


# ---- 4. the frames are a real path ------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2])
def test_frames_are_a_lattice_path(K):
    """merge = False, no LM: each hypothesis is one path of the K-symbol lattice, and nlogp is the fp32 sum of its
    steps' log-softmax values.  The path rebuilt from (tokens, frames) in fp64 must give it within 2^-20 per step,
    (T' + U) steps, times (1 + |log p|): a wrong frame moves the sum by a whole log-prob, orders above the bar."""
    m, z, sd = _tiny()
    sd64 = {k: v.double() for k, v in sd.items()}
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    h, _ = mt.encoder(sd64, xs.double(), None)
    fr = [min(h.shape[1], int(mt.scale_length(h.shape[1], xlen)[b])) for b in range(xs.shape[0])]
    hyps = m.beam_search(xs.cuda(), xlen, W=8, merge=False, max_symbols=K, nbest=8)
    worst = 0.0
    for b in range(len(fr)):
        for x in hyps[b]:
            ref = no.transducer_path_logprob(sd64, h[b], fr[b], x.tokens.tolist(), x.frames.tolist(), K)
            bar = 2.0 ** -20 * (fr[b] + len(x.tokens)) * (1 + abs(ref))
            worst = max(worst, abs(-x.nlogp - ref) / bar)
            assert abs(-x.nlogp - ref) <= bar, (b, x, ref)
    print("K=%d: worst err/bar %.3g" % (K, worst))


# ---- 5. structure, counts and the ranks past them ---------------------------------------------------------------------
@pytest.mark.parametrize("K, merge", [(1, True), (2, True), (4, False)])
def test_counts_and_ranks_past_the_count(K, merge):
    from edgedict_b200.stream_engine import BeamEngine, nbest_lists
    m = _scaled_model(SMALL, seed=4)
    g = torch.Generator().manual_seed(2)
    h = torch.randn(4, 9, SMALL["enc_proj_size"], generator=g).cuda()
    frames = [9, 1, 0, 5]
    W, N = 8, 6
    eng = BeamEngine(m, 4, 9, W, merge=merge, max_symbols=K, nbest=N)
    buf = eng.run(h, torch.tensor(frames, dtype=torch.int32).cuda())
    hyps = nbest_lists(buf, 4, N, 9 * K)
    for b in range(4):
        live = int(eng.hist_live[b, -1])
        cnt = int(eng.nbest_count[b])
        assert cnt == min(N, live)
        _check_structure(hyps[b], max(frames[b], 1), K, W, N, live, merge)
        assert bool((eng.ids[b, cnt:] == -1).all()) and bool((eng.nbest_frames[b, cnt:] == -1).all())
        assert bool(torch.isinf(eng.nlogp[b, cnt:]).all()) and bool((eng.nlogp[b, cnt:] > 0).all())
    assert int(eng.nbest_count[2]) == 1


# ---- 6. determinism ---------------------------------------------------------------------------------------------------
def _lists_equal(a, b):
    return len(a) == len(b) and all(np.array_equal(x.tokens, y.tokens) and np.array_equal(x.frames, y.frames)
                                    and _bits(x.nlogp) == _bits(y.nlogp) for x, y in zip(a, b))


@pytest.mark.parametrize("with_lm", [False, True])
@pytest.mark.parametrize("K", [1, 2])
def test_transducer_batch_invariance_repeatability_and_cta_count(K, with_lm):
    from edgedict_b200.stream_engine import BeamEngine, nbest_lists
    m = _scaled_model(SMALL, seed=4)
    kw = dict(lm=_lm_module(96, 16, 48, 2, 4.0, seed=3).cuda(), lm_weight=0.7, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(2)
    T, W = 30, 6
    h = torch.randn(5, T, SMALL["enc_proj_size"], generator=g).cuda()
    lens = [30, 17, 1, 26, 0]
    eng = BeamEngine(m, 5, T, W, max_symbols=K, nbest=W, **kw)
    buf = eng.run(h, torch.tensor(lens, dtype=torch.int32).cuda()).clone()
    assert torch.equal(buf, eng.run(h, torch.tensor(lens, dtype=torch.int32).cuda()))
    for ctas in (1, 3):
        eng.max_ctas = ctas
        assert torch.equal(buf, eng.run(h, torch.tensor(lens, dtype=torch.int32).cuda())), ctas
    full = nbest_lists(buf, 5, W, T * K)
    for b, n in enumerate(lens[:4]):
        one = BeamEngine(m, 1, n, W, max_symbols=K, nbest=W, **kw)
        alone = nbest_lists(one.run(h[b:b + 1, :n].contiguous(), torch.tensor([n], dtype=torch.int32).cuda()), 1,
                            W, max(n * K, 1))
        assert _lists_equal(alone[0], full[b]), b


def test_ctc_batch_invariance_repeatability_and_cta_count():
    from edgedict_b200.stream_engine import CTCBeamEngine, nbest_lists
    g = torch.Generator().manual_seed(3)
    T, V, W = 28, 40, 8
    lp = (3.0 * torch.randn(4, T, V, generator=g)).log_softmax(-1).cuda()
    lens = torch.tensor([28, 11, 0, 20], dtype=torch.int32).cuda()
    eng = CTCBeamEngine(4, T, V, W, nbest=W, device="cuda")
    buf = eng.run(lp, lens).clone()
    assert torch.equal(buf, eng.run(lp, lens))
    for ctas in (1, 3):
        eng.max_ctas = ctas
        assert torch.equal(buf, eng.run(lp, lens)), ctas
    full = nbest_lists(buf, 4, W, T)
    for b in (0, 1, 3):
        n = int(lens[b])
        one = CTCBeamEngine(1, n, V, W, nbest=W, device="cuda")
        alone = nbest_lists(one.run(lp[b:b + 1, :n], lens[b:b + 1]), 1, W, n)
        assert _lists_equal(alone[0], full[b]), b


def test_best_only_program_is_unchanged_by_the_nbest_fields():
    """nbest = 0 leaves K1, ldw2, seq_out and tok_out2 of BEAM_FINAL zero / NULL, the program built before N-best."""
    from edgedict_b200.stream_engine import EbPhase, PH_BEAM_FINAL, BeamEngine, CTCBeamEngine
    m = _scaled_model(SMALL, seed=4)
    for eng in (BeamEngine(m, 2, 5, 4, max_symbols=2), CTCBeamEngine(2, 5, 8, 4, device="cuda")):
        raw = eng._prog.cpu().numpy().tobytes()
        ph = (EbPhase * eng.nphase).from_buffer_copy(raw)[eng.nphase - 1]
        assert ph.type == PH_BEAM_FINAL and ph.K1 == 0 and ph.ldw2 == 0
        assert ph.seq_out is None and ph.tok_out2 is None
