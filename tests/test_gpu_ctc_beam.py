"""CTC prefix beam search on the device (edgedict_b200.ctc.beam_search, CTCEncoder.beam_search, stream_engine.CTCBeamEngine,
CTC_BEAM of csrc/decode.cu): exact prefix probabilities when nothing is pruned, parity with the CPU restatement
(tests/ctc_beam_oracle.py) with and without LM fusion, bitwise invariants, and the model-level entry point."""
import numpy as np
import pytest
import torch

from tests import ctc_beam_oracle as cbo
from tests.test_gpu_beam_lm import _lm_module, _perm_map

pytestmark = pytest.mark.gpu


def _lp(B, T, V, seed, scale=3.0):
    """Peaked random log-probs [B, T, V] (fp32, CPU)."""
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(B, T, V, generator=g)).log_softmax(-1)


def _engine(B, T, V, W, blank=0, **kw):
    from edgedict_b200.stream_engine import CTCBeamEngine
    return CTCBeamEngine(B, T, V, W, blank, device="cuda", **kw)


def _run(eng, lp, lengths):
    ids, nlp = eng.run(lp.cuda(), torch.as_tensor(lengths, dtype=torch.int32).cuda())
    ids = ids.cpu().numpy()
    return [r[r >= 0].astype(np.int64) for r in ids], nlp.cpu().clone()


def _same(ids_a, ids_b):
    return len(ids_a) == len(ids_b) and all(np.array_equal(a, b) for a, b in zip(ids_a, ids_b))


@pytest.mark.parametrize("V, T", [(2, 6), (3, 6), (4, 5)])
def test_exact_without_pruning(V, T):
    """W = the number of prefixes of at most T tokens (7 / 127 / 364), so nothing is pruned: every final hypothesis'
    pb (+) pnb must be log P(prefix), F.ctc_loss in fp64 on the CPU.  Bar: each frame adds at most a few fp32 roundings
    of log-adds and sums of magnitude <= the running |log p| plus |y|, so |error| <= 2^-20 * T * (1 + |log p| + max|y|)
    (a factor ~8 above 4 roundings per frame).  The best must be the brute-force argmax unless the two best prefixes lie
    within twice that bar."""
    import torch.nn.functional as F
    prefixes = cbo.all_prefixes(V, T)
    W = len(prefixes)
    lp = _lp(2, T, V, seed=V * 100 + T, scale=1.5)
    eng = _engine(2, T, V, W)
    ids, nlp = _run(eng, lp, [T, T])
    worst = 0.0
    for b in range(2):
        hy = eng.hypotheses(b)
        assert sorted(h[0] for h in hy) == sorted(prefixes)
        ymax = float(lp[b].abs().max())
        want = {}
        for p, pb, pnb, f in hy:
            got = float(cbo.logadd(np.float64(pb), np.float64(pnb)))
            if p:
                ref = -float(F.ctc_loss(lp[b].double()[:, None], torch.tensor([p]), [T], [len(p)],
                                        reduction="none"))
            else:
                ref = float(lp[b, :, 0].double().sum())
            want[p] = ref
            if ref == -np.inf:
                assert got == -np.inf, (p, got)
                continue
            bar = 2.0 ** -20 * T * (1 + abs(ref) + ymax)
            worst = max(worst, abs(got - ref) / bar)
            assert abs(got - ref) <= bar, (p, got, ref)
            assert f == 0.0
        top = sorted(want.values(), reverse=True)
        best = max(prefixes, key=lambda p: want[p])
        if top[0] - top[1] > 2 * 2.0 ** -20 * T * (1 + abs(top[0]) + ymax):
            assert tuple(ids[b].tolist()) == best
    print("  [ctc beam] exact V=%d T=%d W=%d: worst err/bar %.3g" % (V, T, W, worst))


@pytest.mark.parametrize("V", [2, 77, 1024])
@pytest.mark.parametrize("blank_last", [False, True])
@pytest.mark.parametrize("W", [1, 4, 16, 64])
def test_matches_restatement(W, blank_last, V):
    """Ragged batch (full length, a shorter one, length 0): ids equal to the fp32 restatement and -score within 1e-5
    relative; length 0 gives the empty prefix and score 0."""
    T = 30 if V < 1024 else 16
    blank = V - 1 if blank_last else 0
    lp = _lp(3, T, V, seed=W * 7 + V + blank)
    lengths = [T, T - 7, 0]
    ids, nlp = _run(_engine(3, T, V, W, blank), lp, lengths)
    rids, rs, _ = cbo.batch_search(lp.numpy(), lengths, W, blank, dtype=np.float32)
    assert _same(ids, rids)
    assert len(ids[2]) == 0 and float(nlp[2]) == 0.0
    assert np.allclose(nlp.double().numpy(), rs, rtol=1e-5, atol=0)


def test_infeasible_tokens_and_blank_only_rows():
    """-inf entries: token 3 is never possible, and frames 4 .. 7 allow only blank; -inf candidates still fill the beam."""
    B, T, V = 2, 14, 6
    lp = _lp(B, T, V, seed=9)
    lp[:, :, 3] = -np.inf
    lp[:, 4:8, :] = -np.inf
    lp[:, 4:8, 0] = 0.0
    lp[1, :, 1:] = -np.inf                                   # utterance 1: only blank is ever finite
    lp[1, :, 0] = 0.0
    for W in (4, 40):
        ids, nlp = _run(_engine(B, T, V, W), lp, [T, T])
        rids, rs, _ = cbo.batch_search(lp.numpy(), [T, T], W, 0, dtype=np.float32)
        assert _same(ids, rids) and np.allclose(nlp.double().numpy(), rs, rtol=1e-5)
        assert all(3 not in i for i in ids) and len(ids[1]) == 0 and float(nlp[1]) == 0.0


def test_merges_into_live_slots():
    """Peaked utterances of repeated tokens: an extension of one slot reaches another live slot's prefix in most frames
    (counted by the restatement), and the ids and scores still match."""
    B, T, V = 3, 40, 5
    g = torch.Generator().manual_seed(11)
    lab = torch.randint(1, 3, (B, T // 4), generator=g).repeat_interleave(4, 1)
    lab[:, 3::8] = 0
    lp = torch.full((B, T, V), -4.0).scatter_(2, lab[..., None], 0.0)
    lp = (lp + 0.5 * torch.randn(B, T, V, generator=g)).log_softmax(-1)
    ids, nlp = _run(_engine(B, T, V, 8), lp, [T] * B)
    rids, rs, merges = cbo.batch_search(lp.numpy(), [T] * B, 8, 0, dtype=np.float32)
    assert _same(ids, rids) and np.allclose(nlp.double().numpy(), rs, rtol=1e-5)
    frames_with_merge = sum(sum(m > 0 for m in mg) for mg in merges)
    print("  [ctc beam] frames with a merge: %d of %d" % (frames_with_merge, B * T))
    assert frames_with_merge > 0.6 * B * T


def test_exact_ties_go_to_the_lowest_flat_index():
    """Rows of exactly equal finite log-probs, so that many candidates tie exactly: the lowest flat index q*V + k (a stay
    at k = blank) must win in the selection, and the lowest slot in the final pick.  Utterance 0 has uniform rows, so
    at W = 1 with blank 0 the stay of the empty prefix beats every extension of equal value and the result is empty,
    while with blank V - 1 the extension by token 0 ranks first and then stays; utterance 1 has rows of three distinct
    values."""
    B, T, V = 2, 12, 6
    g = torch.Generator().manual_seed(51)
    lp = torch.full((B, T, V), -float(np.log(V)), dtype=torch.float32)
    lp[1] = torch.randint(0, 3, (T, V), generator=g).float().log_softmax(-1)
    for blank in (0, V - 1):
        for W in (1, 3, 8, 40):
            ids, nlp = _run(_engine(B, T, V, W, blank), lp, [T, T])
            rids, rs, _ = cbo.batch_search(lp.numpy(), [T, T], W, blank, dtype=np.float32)
            assert _same(ids, rids), (blank, W)
            assert np.allclose(nlp.double().numpy(), rs, rtol=1e-5)
            if W == 1:                                   # the stay of the empty prefix at flat index blank: with
                assert ids[0].tolist() == ([] if blank == 0 else [0])   # blank = V - 1, token 0's extension ranks first


def _lm_cases():
    return [(lw, lb, mapped) for lw in (0.3, 1.0) for lb in (0.0, 0.5) for mapped in (False, True)]


def test_lm_fusion_matches_restatement():
    """Tiny LM (16 tokens) over V = 16 log-probs, identity and permuting maps with two unscored tokens, lm_weight 0.3 / 1,
    length_bonus 0 / 0.5, W = 1 / 4 / 8: ids equal to the fp32 restatement (LM through lm_oracle), -score within 1e-5;
    the LM changes the ids in most cases."""
    B, T, V = 3, 24, 16
    lm = _lm_module(V, 8, 12, 2, 3.0, seed=5)
    sd32 = {k: v.detach().float() for k, v in lm.state_dict().items()}
    lp = _lp(B, T, V, seed=21, scale=1.0)
    lengths = [T, T - 5, 9]
    changed = total = 0
    for W in (1, 4, 8):
        base, _ = _run(_engine(B, T, V, W), lp, lengths)
        for lw, lb, mapped in _lm_cases():
            tmap = _perm_map(V, V) if mapped else None
            eng = _engine(B, T, V, W, lm=lm, lm_weight=lw, length_bonus=lb, lm_token_map=tmap)
            ids, nlp = _run(eng, lp, lengths)
            rids, rs, _ = cbo.batch_search(lp.numpy(), lengths, W, 0, dtype=np.float32, lm_sd=sd32, lm_weight=lw,
                                           length_bonus=lb, lm_map=tmap)
            assert _same(ids, rids), (W, lw, lb, mapped)
            assert np.allclose(nlp.double().numpy(), rs, rtol=1e-5), (W, lw, lb, mapped)
            changed += not _same(ids, base)
            total += 1
    print("  [ctc beam] LM changed the ids in %d of %d cases" % (changed, total))
    assert changed > total // 2


def test_lm_fusion_large_lm():
    """An LMModel(1024, 64, 1024, 2)-shaped LM over V = 1024, W = 4: ids equal to the fp32 restatement."""
    B, T, V = 2, 12, 1024
    lm = _lm_module(V, 64, 1024, 2, 2.0, seed=6)
    sd32 = {k: v.detach().float() for k, v in lm.state_dict().items()}
    lp = _lp(B, T, V, seed=22, scale=1.0)
    ids, nlp = _run(_engine(B, T, V, 4, lm=lm, lm_weight=0.5, length_bonus=0.5), lp, [T, T - 3])
    rids, rs, _ = cbo.batch_search(lp.numpy(), [T, T - 3], 4, 0, dtype=np.float32, lm_sd=sd32, lm_weight=0.5,
                                   length_bonus=0.5)
    assert _same(ids, rids) and np.allclose(nlp.double().numpy(), rs, rtol=1e-5)


def test_lm_zero_weights_and_state_dict_are_bitwise():
    from edgedict_b200 import ctc
    B, T, V = 3, 20, 16
    lm = _lm_module(V, 8, 12, 2, 3.0, seed=7).cuda()
    lp = _lp(B, T, V, seed=23, scale=1.0).cuda()
    a_ids, a_s = ctc.beam_search(lp, [T, 11, 0], 4)
    b_ids, b_s = ctc.beam_search(lp, [T, 11, 0], 4, lm=lm, lm_weight=0.0, length_bonus=0.0)
    assert _same(a_ids, b_ids) and torch.equal(a_s, b_s)
    c_ids, c_s = ctc.beam_search(lp, [T, 11, 0], 4, lm=lm, lm_weight=0.7, length_bonus=0.2)
    d_ids, d_s = ctc.beam_search(lp, [T, 11, 0], 4, lm=lm.state_dict(), lm_weight=0.7, length_bonus=0.2)
    assert _same(c_ids, d_ids) and torch.equal(c_s, d_s)


def test_bitwise_invariants():
    """Batch invariance (an utterance alone and inside a batch), repeatability, max_ctas 0 / 1 / 3 / 17, and the no-LM
    program of one phase for all frames equal to one frame per phase (and to 7 frames per phase)."""
    B, T, V, W = 5, 33, 77, 8
    lp = _lp(B, T, V, seed=31)
    lengths = [T, 20, 33, 0, 5]
    ref = _run(_engine(B, T, V, W), lp, lengths)
    assert _same(_run(_engine(B, T, V, W), lp, lengths)[0], ref[0])
    for mc in (1, 3, 17):
        ids, s = _run(_engine(B, T, V, W, max_ctas=mc), lp, lengths)
        assert _same(ids, ref[0]) and torch.equal(s, ref[1])
    for n in (1, 7):
        ids, s = _run(_engine(B, T, V, W, frames_per_phase=n), lp, lengths)
        assert _same(ids, ref[0]) and torch.equal(s, ref[1])
    for b in (0, 2, 4):
        ids, s = _run(_engine(1, T, V, W), lp[b:b + 1], lengths[b:b + 1])
        assert np.array_equal(ids[0], ref[0][b]) and torch.equal(s[0], ref[1][b])
    lm = _lm_module(V, 8, 12, 1, 3.0, seed=8)
    a = _run(_engine(B, T, V, W, lm=lm, lm_weight=0.5), lp, lengths)
    for mc in (1, 3):
        ids, s = _run(_engine(B, T, V, W, lm=lm, lm_weight=0.5, max_ctas=mc), lp, lengths)
        assert _same(ids, a[0]) and torch.equal(s, a[1])
    ids, s = _run(_engine(1, T, V, W, lm=lm, lm_weight=0.5), lp[1:2], lengths[1:2])
    assert np.array_equal(ids[0], a[0][1]) and torch.equal(s[0], a[1][1])


TINY = dict(vocab_size=40, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0, proj_size=32)
E6D2 = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0, proj_size=640)


def test_ctc_encoder_beam_search_tiny_matches_oracle():
    """CTCEncoder.beam_search on the tiny config against oracle/ctc.py's fp64 forward and the fp64 restatement."""
    from edgedict_b200.rnnt.models import CTCEncoder
    from oracle import ctc as oc
    torch.manual_seed(41)
    m = CTCEncoder(**TINY).cuda()
    with torch.no_grad():
        m.tovocab[0].weight.mul_(4.0)
    xs = torch.randn(3, 30, TINY["input_size"])
    sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    lr = oc.ctc_encoder_forward(sd, xs.double())
    ids, nlp = m.beam_search(xs.cuda(), None, W=6)
    rids, rs, _ = cbo.batch_search(lr.numpy(), [lr.shape[1]] * 3, 6, 0)
    assert _same(ids, rids) and np.allclose(nlp.double().cpu().numpy(), rs, rtol=1e-5)


def test_ctc_encoder_beam_search_scales_xlen():
    """xlen is in input frames and is scaled to T' (time reduction 2): the result is ctc.beam_search on the forward's
    log-probs with scale_length's lengths."""
    from edgedict_b200 import ctc
    from edgedict_b200.rnnt.models import CTCEncoder, scale_length
    torch.manual_seed(42)
    m = CTCEncoder(**TINY).cuda()
    xs = torch.randn(3, 30, TINY["input_size"]).cuda()
    xlen = torch.tensor([30, 21, 6])
    ids, nlp = m.beam_search(xs, xlen, W=4)
    with torch.no_grad():
        lp = m(xs)
    frames = scale_length(lp.shape[1], xlen)
    assert lp.shape[1] == 15 and frames.tolist() == [15, 11, 3]
    rids, rs = ctc.beam_search(lp, frames, 4)
    assert _same(ids, rids) and torch.equal(nlp, rs)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_ctc_encoder_beam_search_e6d2(precision):
    """E6D2 dims (GRU 1024 x 6, proj 640, V = 1024), B = 4, T = 200 (T' = 100), W = 8, in fp32 and bf16 mode, against the
    fp64 restatement run on the device's own log-probs.  Near-tie margin: the bar of test_exact_without_pruning,
    2^-20 * T' * (1 + |best| + max|y|), the fp32 error the search can accumulate on a hypothesis' value.  Wherever the
    fp64 search's two best final hypotheses lie further apart than that, the ids must be equal and -score within 1e-5
    relative; at least one utterance must be outside the margin.  The fp32 restatement (the kernel's arithmetic) must
    give the same ids everywhere."""
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(43)
    m = CTCEncoder(**E6D2).cuda().set_precision(precision)
    with torch.no_grad():
        m.tovocab[0].weight.mul_(32.0)                   # peaked log-probs, as a trained model gives
    xs = torch.randn(4, 200, E6D2["input_size"]).cuda()
    ids, nlp = m.beam_search(xs, W=8)
    with torch.no_grad():
        lp = m(xs).cpu()
    Tp = lp.shape[1]
    rids, rs, _ = cbo.batch_search(lp.numpy(), [Tp] * 4, 8, 0, dtype=np.float32)
    assert _same(ids, rids) and np.allclose(nlp.double().cpu().numpy(), rs, rtol=1e-5)
    checked = 0
    for b in range(4):
        seq, ds, beam, _ = cbo.prefix_beam_search(lp[b].numpy(), Tp, 8, 0, dtype=np.float64)
        tot = sorted((float(cbo.logadd(np.float64(pb), np.float64(pnb))) + f for _, pb, pnb, f in beam), reverse=True)
        margin = 2.0 ** -20 * Tp * (1 + abs(tot[0]) + float(lp[b].abs().max()))
        print("  [ctc beam] E6D2 %s utterance %d: best two %.4g apart, margin %.3g" % (precision, b, tot[0] - tot[1], margin))
        if len(tot) > 1 and tot[0] - tot[1] <= margin:
            continue
        checked += 1
        assert tuple(ids[b].tolist()) == seq, b
        assert abs(float(nlp[b]) - ds) <= 1e-5 * abs(ds)
    print("  [ctc beam] E6D2 %s: %d of 4 utterances outside the near-tie margin, ids equal to fp64" % (precision, checked))
    assert checked >= 1
