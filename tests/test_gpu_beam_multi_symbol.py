"""Beam search with up to K = max_symbols symbols per encoder frame (BEAM_SELECT flag 512 of csrc/decode.cu,
stream_engine.beam_frame, BeamEngine / StreamBeamEngine / Transducer.beam_search(max_symbols=K)) against the CPU
restatement in tests/beam_multi_symbol_oracle.py: K = 1 is the one-symbol program bit for bit, W = 1 is greedy with K,
LM fusion, batch / CTA-count invariance, streaming against the offline search, forced collapses, argument checks."""
import numpy as np
import pytest
import torch

from tests import beam_multi_symbol_oracle as bo
from tests import lm_oracle as lo
from tests import multi_symbol_oracle as mo
from tests.test_gpu_beam_engine import LARGE, SMALL, _scaled_model
from tests.test_gpu_beam_lm import _lm_module, _perm_map
from tests.test_oracle_lm import load_lm
from tests.util import load_tiny, to_t

SHIFTS = (0.0, 1.0, 5.0)                 # blank-bias shifts: rounds stop at different points


def _tiny(shift=0.0):
    from edgedict_b200.rnnt.models import Transducer
    z, cfg, sd, _ = load_tiny()
    sd = dict(to_t(sd))
    b = sd["joint.joint.2.bias"].clone()
    b[0] += shift
    sd["joint.joint.2.bias"] = b
    m = Transducer(output_loss=False, **cfg)
    m.load_state_dict(sd)
    return m.cuda().eval(), z, sd


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---- CPU: the restatement ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 4])
def test_restatement_k1_is_the_one_symbol_beam(W, merge):
    _, lsd = load_lm()
    z, cfg, sd, _ = load_tiny()
    sd = to_t(sd)
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    for kw, okw in (({}, {}), (dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5),) * 2):
        want, wlp = lo.beam_search(sd, xs, xlen, W=W, merge=merge, **okw)
        got, glp = bo.beam_search(sd, xs, xlen, W=W, max_symbols=1, merge=merge, **kw)
        assert got == want and torch.equal(glp, wlp)


@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("shift", SHIFTS)
def test_restatement_width_one_is_greedy(K, shift):
    z, cfg, sd, _ = load_tiny()
    sd = dict(to_t(sd))
    sd["joint.joint.2.bias"] = sd["joint.joint.2.bias"].clone()
    sd["joint.joint.2.bias"][0] += shift
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    got, glp = bo.beam_search(sd, xs, xlen, W=1, max_symbols=K)
    want, _ = mo.greedy_decode(sd, xs, xlen, max_symbols=K)
    fr = _frames(sd, xs, xlen)
    for b in range(len(got)):
        assert got[b] == [int(k) for k in want[b][:fr[b] * K] if k != 0], b


def _frames(sd, xs, xlen):
    from oracle import model_torch as mt
    h, _ = mt.encoder(sd, xs, None)
    return [min(h.shape[1], int(mt.scale_length(h.shape[1], xlen)[b])) for b in range(xs.shape[0])]


def test_max_symbols_checked_before_device_work():
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import BeamEngine, StreamBeamEngine
    torch.manual_seed(0)
    m = Transducer(output_loss=False, **SMALL)                # on the CPU: device work would fail differently
    xs = torch.zeros(1, 4, SMALL["input_size"])
    for bad, err in ((0, ValueError), (17, ValueError), (2.0, TypeError), (True, TypeError), (None, TypeError)):
        with pytest.raises(err):
            m.beam_search(xs, None, W=2, max_symbols=bad)
        with pytest.raises(err):
            BeamEngine(m, 1, 2, 2, max_symbols=bad)
        with pytest.raises(err):
            StreamBeamEngine(m, 1, 4, 2, max_symbols=bad)
    with pytest.raises(ValueError, match="max_pending"):     # a chunk of n_out = 2 frames at K = 3 adds up to 6 tokens
        StreamBeamEngine(m, 1, 4, 2, max_pending=5, max_symbols=3)
    with pytest.raises(RuntimeError, match="CUDA"):           # the arguments are fine: the device is what is missing
        StreamBeamEngine(m, 1, 4, 2, max_pending=6, max_symbols=3)


# ---- K = 1 is the one-symbol program ---------------------------------------------------------------------------------
def _fields(eng, n):
    """The program phase for phase: every integer field, and which pointers are set (the buffers are the engine's)."""
    from edgedict_b200.stream_engine import EbPhase
    raw = (eng._prog if hasattr(eng, "_prog") else eng._chunk).cpu().numpy().tobytes()
    arr = (EbPhase * n).from_buffer_copy(raw)
    ints = [f for f, _ in EbPhase._fields_[:16]]
    ptrs = [f for f, _ in EbPhase._fields_[16:]]
    return [tuple(getattr(p, f) for f in ints) + tuple(getattr(p, f) is None for f in ptrs) for p in arr]


@pytest.mark.gpu
@pytest.mark.parametrize("with_lm", [False, True])
def test_k1_is_the_one_symbol_program(with_lm):
    from edgedict_b200.stream_engine import BeamEngine, StreamBeamEngine
    m = _scaled_model(SMALL, seed=4)
    kw = dict(lm=_lm_module(96, 16, 48, 2, 4.0, seed=1).cuda(), lm_weight=0.7, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(2)
    h = torch.randn(5, 23, SMALL["enc_proj_size"], generator=g).cuda()
    frames = torch.tensor([23, 11, 1, 20, 0], dtype=torch.int32).cuda()
    a, b = BeamEngine(m, 5, 23, 4, **kw), BeamEngine(m, 5, 23, 4, max_symbols=1, **kw)
    assert a.nphase == b.nphase and _fields(a, a.nphase) == _fields(b, b.nphase)
    ia, na = (t.clone() for t in a.run(h, frames))
    ib, nb = b.run(h, frames)
    assert torch.equal(ia, ib) and torch.equal(_bits(na), _bits(nb))
    a, b = StreamBeamEngine(m, 3, 4, 4, **kw), StreamBeamEngine(m, 3, 4, 4, max_symbols=1, **kw)
    assert a.n_chunk_phases == b.n_chunk_phases
    assert _fields(a, a.n_chunk_phases) == _fields(b, b.n_chunk_phases)
    for c in [torch.randn(3, 4, SMALL["input_size"], generator=g) for _ in range(6)]:
        (ia, ca), (ib, cb) = a.step(c.cuda()), b.step(c.cuda())
        assert torch.equal(ia, ib) and torch.equal(ca, cb)
    (ia, ca, na), (ib, cb, nb) = a.flush(), b.flush()
    assert torch.equal(ia, ib) and torch.equal(_bits(na), _bits(nb))


# ---- against the restatement -----------------------------------------------------------------------------------------
def _check(m, sd, xs, xlen, W, K, merge, **lm):
    okw = {} if not lm else dict(lm_sd=lm["lm_sd"], lm_weight=lm["lm_weight"], length_bonus=lm["length_bonus"],
                                 lm_map=lm.get("lm_map"))
    dkw = {} if not lm else dict(lm=lm["lm_sd"], lm_weight=lm["lm_weight"], length_bonus=lm["length_bonus"],
                                 lm_token_map=lm.get("lm_map"))
    stats = {}
    want, wlp = bo.beam_search(sd, xs, xlen, W=W, max_symbols=K, merge=merge, stats=stats, **okw)
    got, glp = m.beam_search(xs.cuda(), xlen, W=W, merge=merge, max_symbols=K, **dkw)
    err = float(np.max(np.abs(glp.cpu().numpy() - wlp.numpy()) / np.abs(wlp.numpy())))
    assert got == want
    assert err < 1e-4
    return got, stats.get("rounds", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("shift", SHIFTS)
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("K", [2, 3, 4])
def test_beam_matches_restatement(K, merge, shift):
    """Tiny model, ragged batch, W = 1 / 4 / 8 / 20 (20 > V: a short first round)."""
    m, z, sd = _tiny(shift)
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    changed = 0
    for W in (1, 4, 8, 20):
        got, rounds = _check(m, sd, xs, xlen, W, K, merge)
        one, _ = m.beam_search(xs.cuda(), xlen, W=W, merge=merge)
        changed += got != one
        print("K=%d merge=%s shift=%g W=%d: %d rounds taken, %d tokens (%d at K = 1)"
              % (K, merge, shift, W, rounds, sum(map(len, got)), sum(map(len, one))))
    assert changed > 0, "K > 1 should change the result somewhere"


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 4])
def test_random_model_rows_stop_at_different_rounds(K):
    """B = 9 random utterances on the SMALL model with the blank bias raised: every frame where every slot closes in
    round 0 is a SKIP, and rows end their frames in different rounds."""
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(3)
    m = Transducer(output_loss=False, **SMALL).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)
        m.joint.joint[2].bias[0] += 2.0
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m.cuda()
    g = torch.Generator().manual_seed(K)
    xs = torch.randn(9, 24, SMALL["input_size"], generator=g)
    xlen = torch.randint(8, 25, (9,), generator=g)
    from edgedict_b200.stream_engine import BeamEngine
    for W in (1, 4):
        got, rounds = _check(m, sd, xs, xlen, W, K, True)
        fr = _frames(sd, xs, xlen)
        print("K=%d W=%d: %d tokens, %d rounds of %d" % (K, W, sum(map(len, got)), rounds, sum(fr) * K))
        assert sum(fr) < rounds < sum(fr) * K                # some frames stop early, some take a second round
        # each utterance alone: a round j >= 1 it does not take is a SKIP of the whole launch (the column keeps the
        # fill, live count 0; the last column holds the final live count)
        h, _ = m.encoder(xs.cuda())
        skipped = 0
        for i in range(9):
            eng = BeamEngine(m, 1, fr[i], W, max_symbols=K)
            eng.run(h[i:i + 1, :fr[i]].contiguous(), torch.tensor([fr[i]], dtype=torch.int32).cuda())
            skipped += int((eng.hist_live.view(-1, K)[:, 1:].flatten()[:-1] == 0).sum())
        print("  rounds j >= 1 skipped: %d" % skipped)
        assert skipped > 0


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("shift", SHIFTS)
def test_width_one_is_greedy(K, shift):
    m, z, sd = _tiny(shift)
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    got, _ = m.beam_search(xs.cuda(), xlen, W=1, max_symbols=K)
    ids, _ = m.greedy_decode(xs.cuda(), xlen, max_symbols=K)
    fr = _frames(sd, xs, xlen)
    for b in range(len(got)):
        assert got[b] == [int(k) for k in ids[b][:fr[b] * K] if k != 0], b


@pytest.mark.gpu
@pytest.mark.parametrize("mapped", [False, True])
@pytest.mark.parametrize("K", [2, 4])
def test_fused_beam_matches_restatement(K, mapped):
    m, z, sd = _tiny(1.0)
    _, lsd = load_lm()
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    tmap = _perm_map(16, lsd["encoder.weight"].shape[0]) if mapped else None
    for W in (1, 4, 8):
        for merge in (True, False):
            _check(m, sd, xs, xlen, W, K, merge, lm_sd=lsd, lm_weight=0.3, length_bonus=0.5, lm_map=tmap)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 4])
def test_zero_lm_weights_are_bitwise_the_plain_beam(K):
    m = _scaled_model(SMALL, seed=4)
    g = torch.Generator().manual_seed(2)
    xs = torch.randn(5, 60, SMALL["input_size"], generator=g).cuda()
    xlen = torch.tensor([60, 41, 7, 52, 30])
    for W in (1, 4):
        plain, plp = m.beam_search(xs, xlen, W=W, max_symbols=K)
        fused, flp = m.beam_search(xs, xlen, W=W, max_symbols=K, lm=_lm_module(96, 16, 48, 2, 4.0, seed=1).cuda())
        assert fused == plain and torch.equal(_bits(flp), _bits(plp))
        assert sum(map(len, plain)) > 0


# ---- invariance ------------------------------------------------------------------------------------------------------
def _run(m, h, frames, W, K, **kw):
    from edgedict_b200.stream_engine import BeamEngine
    eng = BeamEngine(m, h.shape[0], h.shape[1], W, max_symbols=K, **kw)
    ids, nlp = eng.run(h, frames)
    return eng, [[int(k) for k in r if k >= 0] for r in ids.cpu().numpy()], nlp.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("with_lm", [False, True])
@pytest.mark.parametrize("K", [2, 4])
def test_batch_invariance_repeatability_and_cta_count(K, with_lm):
    m = _scaled_model(SMALL, seed=4)
    kw = dict(lm=_lm_module(96, 16, 48, 2, 4.0, seed=3).cuda(), lm_weight=0.7, length_bonus=0.3) if with_lm else {}
    g = torch.Generator().manual_seed(2)
    T = 37
    h = torch.randn(5, T, SMALL["enc_proj_size"], generator=g).cuda()
    lens = [37, 20, 1, 33, 0]
    frames = torch.tensor(lens, dtype=torch.int32).cuda()
    for W in (1, 4, 6):
        eng, ids, nlp = _run(m, h, frames, W, K, **kw)
        hist = eng.hist.clone()
        ids2, nlp2 = eng.run(h, frames)
        assert torch.equal(hist, eng.hist) and torch.equal(_bits(nlp), _bits(nlp2))
        assert ids[4] == [] and float(nlp[4]) == 0.0
        for ctas in (1, 3):
            eng.max_ctas = ctas
            ids3, nlp3 = eng.run(h, frames)
            assert torch.equal(hist, eng.hist) and torch.equal(_bits(nlp), _bits(nlp3)), ctas
        for b, n in enumerate(lens[:4]):
            _, ids1, nlp1 = _run(m, h[b:b + 1, :n].contiguous(), torch.tensor([n], dtype=torch.int32).cuda(), W, K,
                                 **kw)
            assert ids1[0] == ids[b], (W, b)
            assert _bits(nlp1).item() == _bits(nlp[b:b + 1]).item(), (W, b)
        print("K=%d W=%d lm=%s: %d symbols" % (K, W, with_lm, sum(map(len, ids))))
        assert sum(map(len, ids)) > 0 or with_lm              # this LM term holds the SMALL model at blank


# ---- streaming -------------------------------------------------------------------------------------------------------
def _ids(ids, counts, s):
    return ids[s, :int(counts[s])].tolist()


def _stream(m, chunks, W, K, max_pending=256, **kw):
    from edgedict_b200.stream_engine import StreamBeamEngine
    eng, per, enc = None, [], []
    S = chunks[0].shape[0]
    for c in chunks:
        if eng is None or eng.n != c.shape[1]:
            eng = StreamBeamEngine(m, S, c.shape[1], W, max_pending=max_pending, max_symbols=K,
                                   state=None if eng is None else eng.state(), **kw)
        ids, counts = eng.step(c.cuda())
        per.append([_ids(ids, counts, s) for s in range(S)])
        enc.append(eng.enc_out.clone())
    ids, counts, nlp = eng.flush()
    fl = [_ids(ids, counts, s) for s in range(S)]
    return [sum((c[s] for c in per), []) + fl[s] for s in range(S)], nlp, torch.cat(enc, 1), eng


def _offline(m, enc, W, K, **kw):
    S, T = enc.shape[0], enc.shape[1]
    _, ids, nlp = _run(m, enc, torch.full((S,), T, dtype=torch.int32, device="cuda"), W, K, **kw)
    return ids, nlp.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("with_lm", [False, True])
@pytest.mark.parametrize("K", [2, 4])
def test_chunking_is_invisible_to_the_search(K, with_lm):
    m, z, sd = _tiny(1.0)
    kw = dict(lm=load_lm()[1], lm_weight=0.3, length_bonus=0.5) if with_lm else {}
    g = torch.Generator().manual_seed(K)
    chunks = [torch.randn(3, n, 12, generator=g) * 1.5 for n in [4, 2, 6, 2, 4, 2, 6, 2]]
    for W in (1, 4, 8):
        got, nlp, enc, eng = _stream(m, chunks, W, K, **kw)
        want, wlp = _offline(m, enc, W, K, **kw)
        assert eng.n_collapses == 0 and got == want, W
        assert torch.equal(_bits(nlp), _bits(wlp)), W
        assert sum(map(len, got)) > 0


@pytest.mark.gpu
def test_chunking_is_invisible_to_the_search_e6d2_large():
    m = _scaled_model(LARGE, seed=10)
    with torch.no_grad():
        m.joint.joint[2].bias[0] += 3.0
    g = torch.Generator().manual_seed(3)
    chunks = [torch.randn(2, n, 240, generator=g) for n in [2, 4, 2, 2, 6, 2] * 4]
    got, nlp, enc, eng = _stream(m, chunks, 4, 2)
    want, wlp = _offline(m, enc, 4, 2)
    one, _ = _offline(m, enc, 4, 1)
    print("E6D2_LARGE W=4 K=2: %d tokens (%d at K = 1)" % (sum(map(len, got)), sum(map(len, one))))
    assert eng.n_collapses == 0 and got == want
    assert torch.equal(_bits(nlp), _bits(wlp))
    assert sum(map(len, got)) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("with_lm", [False, True])
@pytest.mark.parametrize("K", [2, 3])
def test_forced_collapse_matches_restatement(K, with_lm):
    """max_pending = n_out * K + 2 forces collapses; the committed ids of every chunk and the live hypotheses after it
    match the restatement."""
    from edgedict_b200.stream_engine import StreamBeamEngine
    m, z, sd = _tiny(-1.0)
    kw, okw = {}, {}
    if with_lm:
        lsd = load_lm()[1]
        kw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5)
        okw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5)
    chunks = [torch.as_tensor(np.concatenate(z["stream_chunks"][i:i + 2], 0)[None]) for i in range(0, 40, 2)]
    n_out = chunks[0].shape[1] // 2
    P = n_out * K + 2
    want, wlive = bo.stream_search(sd, torch.cat(chunks, 1), [n_out] * len(chunks), 4, P, K, **okw)
    eng = StreamBeamEngine(m, 1, chunks[0].shape[1], 4, max_pending=P, max_symbols=K, **kw)
    done = []
    for i, c in enumerate(chunks):
        ids, counts = eng.step(c.cuda())
        got = _ids(ids, counts, 0)
        assert got == want[i], ("chunk", i, got, want[i])
        done += got
        live = int(eng.hist_live[0, -1])
        seqs = eng.seqs[0].cpu().numpy()
        assert [done + seqs[s, 3:3 + seqs[s, 0]].tolist() for s in range(live)] == wlive[i], ("chunk", i)
    print("K=%d lm=%s: %d forced collapses over %d chunks, %d tokens" % (K, with_lm, eng.n_collapses, len(chunks),
                                                                         len(done)))
    assert eng.n_collapses > 0


# ---- per round against fp64 ------------------------------------------------------------------------------------------
def _check_round(fv, fb, flats, keys, W, merge, V, par, tok, lp, live, where):
    """test_gpu_beam_engine._check_frame over an explicit candidate list (flat index slot*V + token, fp64 value fv,
    bar fb, merge key): candidates ranked beyond their bars must be ranked so, near-ties may go either way, and each
    survivor's log p must lie within the bars of the log-add of its merge group."""
    N, m = fv.size, min(W, fv.size)
    lo, hi = fv - fb, fv + fb
    above = N - np.searchsorted(np.sort(lo), hi, side="right")
    maybe = N - np.searchsorted(np.sort(hi), lo, side="left") - 1
    out, sure = above >= m, maybe < m
    index = {f: i for i, f in enumerate(flats)}
    assert 1 <= live <= m, (where, "live count", live, m)
    kd = []
    for s in range(live):
        f = int(par[s]) * V + int(tok[s])
        assert f in index, (where, "slot", s, "is no candidate of this round", divmod(f, V))
        kd.append(index[f])
    for s, c in enumerate(kd):
        assert not out[c], (where, "slot", s, "survivor cannot be in the top W")
        for s2 in range(s):
            assert not lo[c] > hi[kd[s2]], (where, "slot", s, "ranked below a worse survivor", s2)
    kseq = [keys[c] for c in kd]
    if merge:
        assert len(set(kseq)) == live, (where, "equal hypotheses left unmerged")
        rep = {q: c for q, c in zip(kseq, kd)}
        for c in np.flatnonzero(sure):
            r = rep.get(keys[c])
            assert r is not None, (where, "sure candidate missing", divmod(flats[c], V))
            assert not lo[c] > hi[r], (where, "merge kept the later of", divmod(flats[c], V), divmod(flats[r], V))
        cand = [c for c in np.flatnonzero(~out) if keys[c] in rep]
    else:
        assert live == m and set(np.flatnonzero(sure).tolist()) <= set(kd), (where, "top W")
        cand = kd
    worst = 0.0
    for s, c in enumerate(kd):
        grp = [x for x in cand if keys[x] == kseq[s]] if merge else [c]
        low = np.logaddexp.reduce([fv[x] for x in grp if sure[x] or x == c])
        high = np.logaddexp.reduce([fv[x] for x in grp])
        bar = max(fb[x] for x in grp) + 4 * 2.0 ** -24 * (abs(high) + 1)
        err = max(low - lp[s], lp[s] - high, 0.0)
        worst = max(worst, err / bar)
        assert err <= bar, (where, "slot", s, "log p", float(lp[s]), "fp64", low, high, "bar", bar)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("merge", [True, False])
def test_beam_rounds_teacher_forced_fp64(merge):
    """Every round of the device beam against fp64 from the device's own beam after the previous round (its sequences
    and open / closed state from the history, its fp32 slot log p), at E6D2_LARGE dims, W = 4, K = 2, with the setting
    and the bars of test_gpu_beam_engine.test_beam_teacher_forced_fp64 (frames presented twice, output layer x 3, blank
    bias raised to about half the mass).  An open slot's candidates carry that test's bar; a closed slot's stay is its
    fp32 log p exactly.  A merge key is (sequence, open), so stays, last-round closes and merges across closedness are
    all checked; the predictor is recomputed in fp64 from the sequences."""
    from edgedict_b200.rnnt.tokenizer import BOS
    from edgedict_b200.stream_engine import BeamEngine
    from tests.test_gpu_beam_engine import U32, _dec64
    m = _scaled_model(LARGE, seed=10)
    B, blank, W, K = 4, m.blank, 4, 2
    g = torch.Generator().manual_seed(1)
    xs = torch.randn(B, 60, 240, generator=g).cuda()
    with torch.no_grad():
        h_enc, _ = m.encoder(xs)
        h_enc = h_enc[:, torch.arange(2 * h_enc.shape[1], device="cuda") // 2].contiguous()
        m.joint.joint[2].weight.mul_(3.0)
        m.joint.joint[2].bias.mul_(3.0)
        d0, _ = m.decoder(torch.zeros(B, 0, dtype=torch.long, device="cuda"))
        z0 = m.joint(h_enc[:, :8].reshape(-1, h_enc.shape[2]), d0[:, 0].repeat_interleave(8, 0))
        lse_rest = torch.cat([z0[:, :blank], z0[:, blank + 1:]], 1).logsumexp(1)
        m.joint.joint[2].bias[blank] += float((lse_rest - z0[:, blank]).median())
    T = h_enc.shape[1]
    frames = torch.tensor([T, T, T - 17, T], dtype=torch.int32)
    eng = BeamEngine(m, B, T, W, merge=merge, max_symbols=K)
    ids, nlp = eng.run(h_enc, frames.cuda())
    torch.cuda.synchronize()
    hpar, htok = eng.hist_parent.cpu().numpy(), eng.hist_token.cpu().numpy()
    hlp, hlive = eng.hist_logp.cpu().numpy().astype(np.float64), eng.hist_live.cpu().numpy()
    ids, dec_final = ids.cpu().numpy(), eng.dec_x[0].double()

    sd64 = {k: v.detach().double() for k, v in m.state_dict().items()}
    Ld, Hd = m.decoder.lstm.num_layers, m.decoder.lstm.hidden_size
    w1, b1 = sd64["joint.joint.0.weight"], sd64["joint.joint.0.bias"]
    w2, b2 = sd64["joint.joint.2.weight"], sd64["joint.joint.2.bias"]
    J, V, E = w1.shape[0], w2.shape[0], h_enc.shape[2]
    D = w1.shape[1] - E
    c1, c2 = U32 * (np.sqrt((E + D + 1) / 2) + 4), U32 * (np.sqrt((J + 1) / 2) + 4)
    rss = lambda x, w: (x * x) @ (w * w).t()
    step = _dec64(sd64, Ld)
    zs = torch.zeros(Ld, 1, Hd, dtype=torch.float64, device="cuda")
    x0, mag0, hh, cc = step(torch.tensor([BOS], device="cuda"), zs, zs)
    cache = {(): (x0[0], mag0[0], hh[:, 0], cc[:, 0])}
    he64 = h_enc.double()
    worst, pred_worst, n = 0.0, 0.0, dict(stays=0, stay_kept=0, second=0, last_close=0, mixed_keys=0, merges=0)
    for b in range(B):
        seqs, lps = [()], np.zeros(1)
        for t in range(T):
            opened = [True] * len(seqs)
            for j in range(K):
                col = t * K + j
                where = "utterance %d frame %d round %d" % (b, t, j)
                taken = t < int(frames[b]) and any(opened)
                if not taken:                      # the beam stays; the column holds what the host filled in
                    assert (hpar[b, col] == np.arange(W)).all() and (htok[b, col] == blank).all(), where
                    if col != T * K - 1:
                        assert hlive[b, col] == 0, where
                    continue
                live = int(hlive[b, col])
                last = j == K - 1
                oq = [q for q in range(len(seqs)) if opened[q]]
                fv, fb, flats, keys = [], [], [], []
                if oq:
                    d = torch.stack([cache[seqs[q]][0] for q in oq])
                    dd = 2.0 ** -16 * torch.stack([cache[seqs[q]][1] for q in oq])
                    x = torch.cat([he64[b, t].expand(len(oq), -1), d], 1)
                    u = x @ w1.t() + b1
                    h = u.tanh()
                    du = c1 * (rss(x, w1) + b1 * b1).sqrt() + rss(dd, w1[:, E:]).sqrt()
                    dh = (1 - h * h) * du + 2 * U32 * h.abs()
                    zz = h @ w2.t() + b2
                    dz = c2 * (rss(h, w2) + b2 * b2).sqrt() + rss(dh, w2).sqrt()
                    lse = torch.logsumexp(zz, 1, keepdim=True)
                    zmax = zz.max(1, keepdim=True).values
                    lpq = torch.as_tensor(lps[oq], device="cuda")[:, None]
                    v = (zz - lse + lpq).cpu().numpy()
                    beta = (6 * (dz + dz.max(1, keepdim=True).values) + V * U32 +
                            3 * U32 * ((zz - zmax).abs() + lse.abs() + lpq.abs())).cpu().numpy()
                for q in range(len(seqs)):
                    if opened[q]:
                        i = oq.index(q)
                        fv.append(v[i])
                        fb.append(beta[i])
                        flats += [q * V + k for k in range(V)]
                        keys += [(seqs[q] + ((k,) if k != blank else ()), k != blank and not last) for k in range(V)]
                    else:
                        fv.append(np.array([lps[q]]))
                        fb.append(np.zeros(1))
                        flats.append(q * V + blank)
                        keys.append((seqs[q], False))
                        n["stays"] += 1
                fv, fb = np.concatenate(fv), np.concatenate(fb)
                n["mixed_keys"] += len({k[0] for k in keys}) < len(set(keys))
                worst = max(worst, _check_round(fv, fb, flats, keys, W, merge, V, hpar[b, col], htok[b, col],
                                                hlp[b, col], live, where))
                new, nopen = [], []
                for s in range(live):
                    q, k = int(hpar[b, col, s]), int(htok[b, col, s])
                    emits = opened[q] and k != blank
                    assert emits or k == blank, (where, "a closed slot took a token")
                    new.append(seqs[q] + ((k,) if emits else ()))
                    nopen.append(emits and not last)
                    n["stay_kept"] += not opened[q]
                    n["second"] += emits and j > 0
                    n["last_close"] += emits and last
                n["merges"] += merge and live < min(W, len(flats))
                todo = sorted(set(s for s in new if s not in cache))
                if todo:
                    prev = [cache[s[:-1]] for s in todo]
                    hx, mg, h2, c2_ = step(torch.tensor([s[-1] for s in todo], device="cuda"),
                                           torch.stack([p[2] for p in prev], 1), torch.stack([p[3] for p in prev], 1))
                    for i, s in enumerate(todo):
                        cache[s] = (hx[i], mg[i], h2[:, i], c2_[:, i])
                seqs, lps, opened = new, hlp[b, col, :live], nopen
        best = int(np.argmax(lps))
        assert [int(k) for k in ids[b] if k >= 0] == list(seqs[best]), ("utterance %d result" % b)
        assert float(nlp[b]) == -float(lps[best])
        for s, sq in enumerate(seqs):
            e = ((dec_final[b * W + s] - cache[sq][0]).abs() / (2.0 ** -16 * cache[sq][1])).max().item()
            pred_worst = max(pred_worst, e)
    print("merge=%s: worst err/bar %.3f, predictor err/budget %.3f, %s" % (merge, worst, pred_worst, n))
    assert pred_worst <= 1.0
    assert n["stays"] > 0 and n["stay_kept"] > 0 and n["second"] > 0 and n["last_close"] > 0
    assert n["merges"] > 0 or not merge


@pytest.mark.gpu
@pytest.mark.parametrize("with_lm", [False, True])
def test_state_moves_between_symbol_caps(with_lm):
    """A K = 1 beam carried into a K = 3 engine whose bound (max_pending - n_out * 3) forces the load-time collapse,
    then back to K = 1: committed ids per chunk and the live hypotheses equal the restatement with K per chunk."""
    from edgedict_b200.stream_engine import StreamBeamEngine
    m, z, sd = _tiny(-1.0)
    kw, okw = {}, {}
    if with_lm:
        lsd = load_lm()[1]
        kw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5)
        okw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5)
    chunks = [torch.as_tensor(np.concatenate(z["stream_chunks"][i:i + 2], 0)[None]) for i in range(0, 40, 2)]
    n_out, P = chunks[0].shape[1] // 2, 7
    Ks = [1] * 6 + [3] * 8 + [1] * 6
    want, wlive = bo.stream_search(sd, torch.cat(chunks, 1), [n_out] * len(chunks), 4, P, Ks, **okw)
    eng, done, at_load = None, [], 0
    for i, (c, K) in enumerate(zip(chunks, Ks)):
        if eng is None or eng.max_symbols != K:
            eng = StreamBeamEngine(m, 1, c.shape[1], 4, max_pending=P, max_symbols=K,
                                   state=None if eng is None else eng.state(), **kw)
            at_load += eng.n_collapses
        ids, counts = eng.step(c.cuda())
        got = _ids(ids, counts, 0)
        assert got == want[i], ("chunk", i, got, want[i])
        done += got
        live = int(eng.hist_live[0, -1])
        seqs = eng.seqs[0].cpu().numpy()
        assert [done + seqs[s, 3:3 + seqs[s, 0]].tolist() for s in range(live)] == wlive[i], ("chunk", i)
    print("lm=%s: %d collapses when the K = 3 engine took over, %d tokens" % (with_lm, at_load, len(done)))
    assert at_load > 0
