"""Streaming GRU transducers on the device (stream_engine.GRUStreamEngine / GRUStreamBeamEngine,
PytorchStreamDecoder on a ``Transducer(module_type='GRU')``; csrc/decode.cu through eb_decode_run_gru_rnnt):

* the reference's fixture (tests/golden/gru_rnnt_tiny.npz) streamed greedily gives its offline ids per frame;
* token for token against the CPU restatement (tests/gru_stream_oracle.py): many streams with the <unk> rule firing,
  max_symbols rounds, and E6D2_LARGE dims with 64 streams;
* the streaming beam: chunking invisible against BeamEngine over the same encoder frames, with and without an LM; W = 1
  against the greedy stream; forced collapses against the beam restatement on encoder_gru; Transducer.beam_search;
* state carried across rebuilds, refused across encoder kinds; bitwise invariances over max_ctas and streams;
* the new kernel instantiation computes the shared phases bit for bit as the other instantiations do."""
import numpy as np
import pytest
import torch

from tests.gru_stream_oracle import GRUStreamRestatement
from tests.test_gpu_beam_engine import LARGE
from tests.test_gpu_stream_beam import _chunks, _ids, _joined, _offline
from tests.test_gru_stream_host import MIXED, Tok, load_gru_rnnt_tiny
from tests.test_oracle_lm import load_lm

pytestmark = pytest.mark.gpu

CTAS = (0, 1, 3, 17)


def _tiny(sd_edit=None):
    from edgedict_b200.rnnt.models import Transducer
    z, cfg, sd = load_gru_rnnt_tiny()
    sd = {k: v.clone() for k, v in sd.items()}
    if sd_edit is not None:
        sd_edit(sd)
    m = Transducer(output_loss=False, module_type="GRU", **cfg)
    m.load_state_dict(sd)
    return m.cuda().eval(), z, sd


def _xs(z):
    return torch.as_tensor(z["xs"])[None]                      # [1, 96, 12]


def _greedy(eng, chunks):
    return [eng.step(c.cuda()).cpu().clone() for c in chunks]


def _decoder(m, **kw):
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    return PytorchStreamDecoder(FLAGS=None, transducer=m, transform=lambda f: f.transpose(1, 2), tokenizer=Tok(), **kw)


def _text(ids):
    return "".join("<unk>" if t == 3 else "t%d " % t for t in ids)


# ---- 1. the reference's fixture --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 4])
def test_fixture_streamed_greedily(n):
    from edgedict_b200.stream_engine import GRUStreamEngine
    m, z, _ = _tiny()
    xs = _xs(z)
    eng = GRUStreamEngine(m, 1, n)
    assert "enc_c" not in eng.state()
    got = sum((eng.step(xs[:, t:t + n].cuda())[0].tolist() for t in range(0, xs.shape[1], n)), [])
    assert got == z["greedy_ids"].tolist()


def test_fixture_through_the_stream_decoder_mixed_chunks():
    m, z, _ = _tiny()
    xs = _xs(z)
    dec = _decoder(m)
    text, t0 = "", 0
    for n in MIXED:
        text += dec.decode(xs[:, t0:t0 + n])
        t0 += n
    assert text == _text([int(k) for k in z["greedy_ids"] if k != 0])
    assert len(dec.encoder_elapsed) == len(MIXED)
    assert len(dec.joint_elapsed) == len(z["greedy_ids"])
    assert len(dec.decoder_elapsed) == int((z["greedy_ids"] != 0).sum())
    assert dec.flush() == ""


# ---- 2. / 3. many streams, the <unk> rule, max_symbols ---------------------------------------------------------------
def _raise_unk(unk):
    def edit(sd):
        b = sd["joint.joint.2.bias"]
        b[unk] = float(b.max()) + 1.0
    return edit


@pytest.mark.parametrize("S", [3, 70])
@pytest.mark.parametrize("n", [2, 4])
def test_many_streams_with_the_unk_rule(S, n):
    from edgedict_b200.stream_engine import GRUStreamEngine
    unk = 9
    m, z, sd = _tiny(_raise_unk(unk))
    chunks = _chunks(S, [n] * 10, 12, seed=S * 10 + n)
    eng = GRUStreamEngine(m, S, n, unk_id=unk)
    got = _greedy(eng, chunks)
    rs = GRUStreamRestatement(sd, S, unk_id=unk)
    for ci, c in enumerate(chunks):
        want = rs.step(c)
        assert torch.equal(got[ci].long(), want), ("chunk", ci, np.argwhere((got[ci].long() != want).numpy())[:5])
    print("S=%d n=%d: the <unk> rule fired %d times, smallest top-2 margin %.3g" % (S, n, rs.hit_unk, min(rs.margins)))
    assert rs.hit_unk > 0 and sum(int((g != 0).sum()) for g in got) > 0
    eng.reset()                                                # reset() reproduces the first chunk's output
    assert torch.equal(eng.step(chunks[0].cuda()).cpu(), got[0])


@pytest.mark.parametrize("K", [2, 4])
def test_max_symbols_against_the_restatement(K):
    from edgedict_b200.stream_engine import GRUStreamEngine
    unk = 9
    m, z, sd = _tiny(_raise_unk(unk))
    S, n = 5, 4
    chunks = _chunks(S, [n] * 8, 12, seed=K)
    got = _greedy(GRUStreamEngine(m, S, n, unk_id=unk, max_symbols=K), chunks)
    rs = GRUStreamRestatement(sd, S, unk_id=unk, max_symbols=K)
    multi = 0
    for ci, c in enumerate(chunks):
        want = rs.step(c)
        assert torch.equal(got[ci].long(), want), ("chunk", ci)
        multi += int((want.view(S, -1, K)[:, :, 1] != 0).sum())
    print("K=%d: %d frames emitted a second symbol" % (K, multi))
    assert multi > 0
    one = _greedy(GRUStreamEngine(m, S, n, unk_id=unk, max_symbols=1), chunks)
    default = _greedy(GRUStreamEngine(m, S, n, unk_id=unk), chunks)
    assert all(torch.equal(a, b) for a, b in zip(one, default))


# ---- 4. E6D2_LARGE with a GRU encoder ----------------------------------------------------------------------------------
def _large_gru(seed=10):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(seed)
    m = Transducer(output_loss=False, module_type="GRU", **LARGE).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)                       # random-init weights emit only blanks; scale up so symbols appear
    return m


def test_e6d2_large_64_streams_token_for_token():
    """E6D2_LARGE dims with a GRU encoder (H = 1024 x 6, F = 240, predictor 512 x 2, joint 640, V = 1024), 64 streams x
    24 chunks of 2 frames against the restatement batched over the streams, exact."""
    from edgedict_b200.stream_engine import GRUStreamEngine
    S, CHUNKS = 64, 24
    m = _large_gru()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m.cuda()
    chunks = list(torch.randn(CHUNKS, S, 2, 240, generator=torch.Generator().manual_seed(0)))
    got = torch.stack(_greedy(GRUStreamEngine(m, S, 2), chunks))[:, :, 0].long()
    rs = GRUStreamRestatement(sd, S, fast=True)
    want = torch.stack([rs.step(c) for c in chunks])[:, :, 0]
    print("E6D2_LARGE GRU: %d non-blank tokens, smallest top-2 logit margin %.3g, <unk> rule fired %d times"
          % (int((want != 0).sum()), min(rs.margins), rs.hit_unk))
    assert int((want != 0).sum()) > 50
    assert torch.equal(got, want), "streams differ at %s" % (np.argwhere((got != want).numpy())[:5].tolist(),)


# ---- 5. the streaming beam -------------------------------------------------------------------------------------------
def _stream_beam(m, chunks, W, merge=True, max_pending=256, **kw):
    """tests/test_gpu_stream_beam._stream on GRUStreamBeamEngine."""
    from edgedict_b200.stream_engine import GRUStreamBeamEngine
    eng, per, enc = None, [], []
    S = chunks[0].shape[0]
    for c in chunks:
        if eng is None or eng.n != c.shape[1]:
            eng = GRUStreamBeamEngine(m, S, c.shape[1], W, merge=merge, max_pending=max_pending,
                                      state=None if eng is None else eng.state(), **kw)
        ids, counts = eng.step(c.cuda())
        per.append([_ids(ids, counts, s) for s in range(S)])
        enc.append(eng.enc_out.clone())
    ids, counts, nlp = eng.flush()
    return per, [_ids(ids, counts, s) for s in range(S)], nlp, torch.cat(enc, 1), eng


def _lm_kw(lm):
    return dict(lm=load_lm()[1], lm_weight=0.3, length_bonus=0.5) if lm else {}


@pytest.mark.parametrize("lm", [False, True])
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 4, 8])
def test_beam_chunking_is_invisible_to_the_search(W, merge, lm):
    m, z, sd = _tiny()
    chunks = _chunks(3, [4, 2, 6, 2, 4, 2, 6, 2], 12, seed=W + 2 * merge)
    kw = _lm_kw(lm)
    per, fl, nlp, enc, eng = _stream_beam(m, chunks, W, merge, **kw)
    want, wlp = _offline(m, enc, W, merge, **kw)
    got = _joined(per, fl)
    print("W=%d merge=%s lm=%s: %d tokens, %d committed before the flush" % (W, merge, lm, sum(map(len, got)),
                                                                           sum(len(x) for c in per for x in c)))
    assert eng.n_collapses == 0 and got == want
    assert torch.equal(nlp.view(torch.int32), wlp.view(torch.int32))
    assert sum(map(len, got)) > 0


def test_beam_width_one_is_the_greedy_stream_without_unk_rule():
    from edgedict_b200.stream_engine import GRUStreamBeamEngine, GRUStreamEngine
    m, z, sd = _tiny()
    S, n = 4, 4
    chunks = _chunks(S, [n] * 12, 12, seed=5)
    greedy = GRUStreamEngine(m, S, n, unk_id=-1)
    beam = GRUStreamBeamEngine(m, S, n, 1, max_pending=n // 2)
    total = 0
    for i, c in enumerate(chunks):
        g = greedy.step(c.cuda()).cpu().numpy()
        ids, counts = beam.step(c.cuda())
        for s in range(S):
            assert _ids(ids, counts, s) == [int(k) for k in g[s] if k != 0], ("chunk", i, "stream", s)
            total += int(counts[s])
    assert total > 0 and beam.n_collapses == 0


@pytest.mark.parametrize("lm", [False, True])
@pytest.mark.parametrize("merge", [True, False])
def test_beam_forced_collapse_matches_restatement(merge, lm, monkeypatch):
    """max_pending = n_out + 2 forces collapses.  The restatement is beam_multi_symbol_oracle.stream_search with its
    encoder the GRU one (oracle.model_torch.encoder_gru)."""
    from oracle import model_torch as mt
    from tests import beam_multi_symbol_oracle as bo
    from edgedict_b200.stream_engine import GRUStreamBeamEngine
    m, z, sd = _tiny()
    monkeypatch.setattr(mt, "encoder", lambda sd_, xs, hiddens=None, *a, **k: (mt.encoder_gru(sd_, xs)[0], None))
    xs = _xs(z)
    n = 4
    P = n // 2 + 2
    okw = dict(lm_sd=load_lm()[1], lm_weight=0.3, length_bonus=0.5) if lm else {}
    want, _ = bo.stream_search(sd, xs, [n // 2] * (xs.shape[1] // n), 4, P, merge=merge, **okw)
    eng = GRUStreamBeamEngine(m, 1, n, 4, merge=merge, max_pending=P, **_lm_kw(lm))
    for i, t in enumerate(range(0, xs.shape[1], n)):
        ids, counts = eng.step(xs[:, t:t + n].cuda())
        assert _ids(ids, counts, 0) == want[i], ("chunk", i)
    print("merge=%s lm=%s: %d forced collapses, %d tokens committed" % (merge, lm, eng.n_collapses, sum(map(len, want))))
    assert eng.n_collapses > 0


def test_beam_matches_transducer_beam_search():
    """The fixture streamed in chunks of 4 with W = 4: the committed ids plus the flush are Transducer.beam_search's
    best hypothesis over the whole utterance, text through PytorchStreamDecoder included."""
    m, z, _ = _tiny()
    xs = _xs(z)
    best, _ = m.beam_search(xs.cuda(), None, W=4)
    per, fl, _, _, eng = _stream_beam(m, [xs[:, t:t + 4] for t in range(0, 96, 4)], 4)
    assert eng.n_collapses == 0 and _joined(per, fl)[0] == list(best[0]) and len(best[0]) > 0
    dec = _decoder(m, beam_width=4)
    parts = [dec.decode(xs[:, t:t + 4]) for t in range(0, 96, 4)]
    assert "".join(parts) + dec.flush() == _text(best[0])
    assert sum(map(len, parts)) > 0 and len(dec.encoder_elapsed) == 24
    dec.reset()
    assert "".join(dec.decode(xs[:, t:t + 4]) for t in range(0, 96, 4)) + dec.flush() == _text(best[0])


# ---- 6. state --------------------------------------------------------------------------------------------------------
def test_greedy_state_survives_rebuilds_and_refuses_the_other_kind():
    from edgedict_b200.stream_engine import GRUStreamEngine, StreamEngine, param_fingerprint
    from tests.test_gpu_stream import _tiny as lstm_tiny
    m, z, sd = _tiny()
    lens = [4, 4, 2, 6, 2, 4]
    chunks = _chunks(1, lens, 12, seed=7)
    rs = GRUStreamRestatement(sd, 1)
    want = [[int(k) for k in rs.step(c)[0] if k != 0] for c in chunks]
    eng, got = None, []
    for i, c in enumerate(chunks):
        if i == 3:                                   # re-home the weights mid-utterance
            for p in m.parameters():
                p.data = p.data.clone()
        if eng is None or eng.n != c.shape[1] or eng.fingerprint != param_fingerprint(m):
            eng = GRUStreamEngine(m, 1, c.shape[1], state=None if eng is None else eng.state())
        got.append([t for t in eng.step(c.cuda())[0].tolist() if t != 0])
    assert got == want and sum(map(len, got)) > 0
    assert set(eng.state()) == {"enc_h", "dec_h", "dec_c", "dec_x", "tok"}
    lstm = StreamEngine(lstm_tiny()[0], 1, 2)
    with pytest.raises(ValueError, match="state keys"):
        lstm.load_state(eng.state())
    with pytest.raises(ValueError, match="state keys"):
        eng.load_state(lstm.state())
    with pytest.raises(ValueError, match="state keys"):
        GRUStreamEngine(m, 1, 2, state=lstm.state())
    with pytest.raises(ValueError, match="has shape"):     # one stream's state is not broadcast to four
        StreamEngine(lstm_tiny()[0], 4, 2, state=lstm.state())
    with pytest.raises(ValueError, match="has shape"):
        GRUStreamEngine(m, 4, 2).load_state(eng.state())


@pytest.mark.parametrize("with_lm", [False, True])
def test_beam_state_survives_rebuilds_and_refuses_the_other_kind(with_lm):
    from edgedict_b200.stream_engine import GRUStreamBeamEngine, StreamBeamEngine, param_fingerprint
    from tests.test_gpu_stream import _tiny as lstm_tiny
    m, z, sd = _tiny()
    kw = _lm_kw(with_lm)
    chunks = _chunks(1, [4, 4, 2, 6, 2, 4], 12, seed=7)
    eng, got = None, []
    for i, c in enumerate(chunks):
        if i == 3:
            for p in m.parameters():
                p.data = p.data.clone()
        if eng is None or eng.n != c.shape[1] or eng.fingerprint != param_fingerprint(m):
            eng = GRUStreamBeamEngine(m, 1, c.shape[1], 4, state=None if eng is None else eng.state(), **kw)
        ids, counts = eng.step(c.cuda())
        got += _ids(ids, counts, 0)
    assert "enc_c" not in eng.state()
    ids, counts, nlp = eng.flush()
    got += _ids(ids, counts, 0)
    one = GRUStreamBeamEngine(m, 1, 2, 4, **kw)
    want = []
    for c in chunks:
        for j in range(0, c.shape[1], 2):
            ids, counts = one.step(c[:, j:j + 2].cuda())
            want += _ids(ids, counts, 0)
    ids, counts, wlp = one.flush()
    want += _ids(ids, counts, 0)
    assert got == want and len(got) > 0
    assert torch.equal(nlp.view(torch.int32), wlp.view(torch.int32))
    lstm = StreamBeamEngine(lstm_tiny()[0], 1, 2, 4, **kw)
    with pytest.raises(ValueError, match="state keys"):
        lstm.load_state(eng.state())
    with pytest.raises(ValueError, match="state keys"):
        eng.load_state(lstm.state())
    # reset() reproduces the first chunk's commits
    one.reset()
    first = [_ids(*one.step(chunks[0][:, j:j + 2].cuda()), 0) for j in (0, 2)]
    one.reset()
    assert [_ids(*one.step(chunks[0][:, j:j + 2].cuda()), 0) for j in (0, 2)] == first


# ---- 7. invariances --------------------------------------------------------------------------------------------------
def test_outputs_do_not_depend_on_the_grid():
    from edgedict_b200.stream_engine import GRUStreamBeamEngine, GRUStreamEngine
    m, z, sd = _tiny(_raise_unk(9))
    chunks = _chunks(5, [4] * 6, 12, seed=11)
    first = None
    for mc in CTAS:
        g = GRUStreamEngine(m, 5, 4, unk_id=9, max_ctas=mc, max_symbols=2)
        greedy = _greedy(g, chunks)
        b = GRUStreamBeamEngine(m, 5, 4, 4, max_pending=4, max_ctas=mc, **_lm_kw(True))
        beam = [b.step(c.cuda()) for c in chunks] + [b.flush()]
        st = {k: v.cpu() for k, v in list(g.state().items()) + [("b_" + k, v) for k, v in b.state().items()]}
        if first is None:
            first = greedy, beam, st
            continue
        assert all(torch.equal(x, y) for x, y in zip(first[0], greedy)), mc
        for x, y in zip(first[1], beam):
            assert all(torch.equal(u, v) for u, v in zip(x, y)), mc
        for k, v in st.items():
            assert torch.equal(v.view(torch.int32) if v.is_floating_point() else v,
                               first[2][k].view(torch.int32) if v.is_floating_point() else first[2][k]), (mc, k)


def test_streams_are_independent_bitwise():
    from edgedict_b200.stream_engine import GRUStreamEngine
    m, z, sd = _tiny(_raise_unk(9))
    chunks = _chunks(5, [4] * 10, 12, seed=9)
    got = _greedy(GRUStreamEngine(m, 5, 4, unk_id=9), chunks)
    per, fl, nlp, _, eng = _stream_beam(m, chunks, 4, max_pending=4)
    assert eng.n_collapses > 0
    for s in range(5):
        one = _greedy(GRUStreamEngine(m, 1, 4, unk_id=9), [c[s:s + 1] for c in chunks])
        assert all(torch.equal(a[s], b[0]) for a, b in zip(got, one)), s
        per1, fl1, nlp1, _, _ = _stream_beam(m, [c[s:s + 1] for c in chunks], 4, max_pending=4)
        assert [c[0] for c in per1] == [c[s] for c in per] and fl1[0] == fl[s], s
        assert nlp1.view(torch.int32)[0] == nlp.view(torch.int32)[s], s


# ---- 8. the shared phases in the new instantiation ---------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def test_lstm_stream_programs_give_the_same_bits_through_the_new_entry():
    """StreamEngine's (greedy, K = 2) and StreamBeamEngine's (with an LM) programs on an LSTM transducer, launched
    through eb_decode_run_gru_rnnt instead of eb_decode_run: the same outputs and states, bit for bit."""
    from edgedict_b200.stream_engine import StreamBeamEngine, StreamEngine
    from tests.test_gpu_stream import _tiny as lstm_tiny
    m = lstm_tiny()[0]
    chunks = _chunks(3, [4] * 8, 12, seed=13)
    runs = []
    for entry in ("eb_decode_run", "eb_decode_run_gru_rnnt"):
        g = StreamEngine(m, 3, 4, unk_id=3, max_symbols=2)
        b = StreamBeamEngine(m, 3, 4, 4, max_pending=4, **_lm_kw(True))
        g.RUN = b.RUN = entry
        g.reset()
        b.reset()
        out = [g.step(c.cuda()).cpu().clone() for c in chunks]
        out += [t for c in chunks for t in b.step(c.cuda())] + list(b.flush())
        st = [v.cpu() for v in g.state().values()] + [v.cpu() for v in b.state().values()]
        runs.append((out, st, b.n_collapses))
    (o1, s1, n1), (o2, s2, n2) = runs
    assert n1 == n2 and n1 > 0
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(o1, o2))
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(s1, s2))


def test_one_phase_gru_ln_linear_programs_match_the_ctc_stream_instantiation():
    from edgedict_b200._lib import check, lib
    from edgedict_b200.stream_engine import EbPhase, PH_GRU, PH_LINEAR, PH_LN, _ptr, _upload
    gen = torch.Generator().manual_seed(3)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, generator=gen) * sc).cuda()
    S, H, I, N = 70, 100, 240, 72
    x, h = rnd(S, I), rnd(S, H, sc=0.5)
    wih, whh, bih, bhh = rnd(3 * H, I, sc=0.1), rnd(3 * H, H, sc=0.1), rnd(3 * H, sc=0.5), rnd(3 * H, sc=0.5)
    lw, lb, w, b = rnd(I), rnd(I), rnd(N, I, sc=0.1), rnd(N)
    outs = []
    for entry in ("eb_decode_run_ctc_stream", "eb_decode_run_gru_rnnt"):
        y, y2, yl, ylin = (torch.full(s, float("nan"), device="cuda") for s in ((S, H), (S, H), (S, I), (S, N)))
        progs = [[EbPhase(type=PH_GRU, S=S, N=H, K1=I, K2=H, x1=_ptr(x), ldx1=I, x2=_ptr(h), ldx2=H, w1=_ptr(wih),
                          ldw1=I, w2=_ptr(whh), ldw2=H, b1=_ptr(bih), b2=_ptr(bhh), y=_ptr(y), ldy=H, y2=_ptr(y2))],
                 [EbPhase(type=PH_LN, S=S, N=I, x1=_ptr(x), ldx1=I, w1=_ptr(lw), b1=_ptr(lb), y=_ptr(yl), ldy=I)],
                 [EbPhase(type=PH_LINEAR, S=S, N=N, K1=I, x1=_ptr(x), ldx1=I, w1=_ptr(w), ldw1=I, b1=_ptr(b),
                          y=_ptr(ylin), ldy=N, flags=1)]]
        bar = torch.zeros(64, dtype=torch.int32, device="cuda")
        for p in progs:
            t = _upload(p, "cuda")
            check(getattr(lib(), entry)(t.data_ptr(), 1, bar.data_ptr(), 0, torch.cuda.current_stream().cuda_stream),
                  entry)
        torch.cuda.synchronize()
        outs.append([y, y2, yl, ylin])
    for a, b in zip(*outs):
        assert not torch.isnan(a).any()
        assert torch.equal(_bits(a), _bits(b))
