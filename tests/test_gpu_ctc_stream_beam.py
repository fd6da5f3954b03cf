"""Streaming CTC prefix beam search on the device (stream_engine.CTCStreamBeamEngine, ctc.CTCStreamDecoder(beam_width=...);
csrc/decode.cu CTC_BEAM with flag 64 and BEAM_COMMIT on CTC rows, through eb_decode_run_ctc_stream_beam):

* chunking is invisible: the committed ids of every chunk plus flush() are CTCBeamEngine.run's on the engine's own
  concatenated log-probs, with -score bitwise equal, with and without an LM, through state-carrying rebuilds;
* the concatenated chunks against CTCEncoder.beam_search (fp32 mode) and the fp64 restatement;
* commit and collapse, chunk by chunk and slot by slot, against the restatement (tests/ctc_stream_beam_oracle.py);
* a token held across a chunk boundary is committed once, and again after a blank;
* stream independence, carried state, refusal of the greedy engine's state, and the decoder's text."""
import numpy as np
import pytest
import torch

from tests import ctc_beam_oracle as cbo
from tests.ctc_stream_beam_oracle import CTCStreamBeamRestatement
from tests.test_gpu_beam_lm import _lm_module, _perm_map

pytestmark = pytest.mark.gpu

DEV = "cuda"
TINY = dict(vocab_size=40, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0, proj_size=32)
E6D2 = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0, proj_size=640)
MUL = 0x100000001b3


def _model(cfg, seed, scale=1.0, head=1.0):
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(seed)
    m = CTCEncoder(**cfg).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(scale)
        m.tovocab[0].weight.mul_(head)
    return m.to(DEV)


def _lm_kw(lm, V):
    if lm is None:
        return {}
    mod = _lm_module(V, 8, 12, 2, 3.0, seed=5)
    return dict(lm=mod, lm_weight=0.6, length_bonus=0.3, lm_token_map=_perm_map(V, V) if lm == "permuted" else None)


def _stream(m, S, lens, xs, W, rehome_at=None, **kw):
    """xs [S, sum(lens), F] through CTCStreamBeamEngine, rebuilt with the carried state at every change of chunk length
    (and after re-homing the weights before chunk rehome_at).  -> (committed ids per chunk and stream, flushed ids per
    stream, -score [S], log-probs [S, T', V], engine)."""
    from edgedict_b200.stream_engine import CTCStreamBeamEngine, param_fingerprint
    eng, per, lps, t0 = None, [], [], 0
    for ci, n in enumerate(lens):
        if ci == rehome_at:
            with torch.no_grad():
                for p in m.parameters():
                    p.data = p.data.clone()
        if eng is None or eng.n != n or eng.fingerprint != param_fingerprint(m):
            eng = CTCStreamBeamEngine(m, S, n, W, state=None if eng is None else eng.state(), **kw)
        ids, cnt = eng.step(xs[:, t0:t0 + n])
        t0 += n
        per.append([ids[s, :int(cnt[s])].tolist() for s in range(S)])
        lps.append(eng.logprobs.view(S, eng.n_out, -1).clone())
    ids, cnt, nscore = eng.flush()
    return per, [ids[s, :int(cnt[s])].tolist() for s in range(S)], nscore, torch.cat(lps, 1), eng


def _joined(per, rest, s):
    return [k for chunk in per for k in chunk[s]] + rest[s]


def _offline(lp, W, **kw):
    from edgedict_b200.stream_engine import CTCBeamEngine
    B, T, V = lp.shape
    eng = CTCBeamEngine(B, T, V, W, device=DEV, **kw)
    ids, nlp = eng.run(lp, torch.full((B,), T, dtype=torch.int32, device=DEV))
    ids = ids.cpu()
    return [r[r >= 0].tolist() for r in ids], nlp.cpu().clone()


# ---- 1. chunking is invisible to the search -----------------------------------------------------------------------------
@pytest.mark.parametrize("S", [3, 70])
@pytest.mark.parametrize("lens", [[2] * 8, [4] * 4, [2, 4, 2, 6, 2], "rehome"])
@pytest.mark.parametrize("lm", [None, "identity", "permuted"])
def test_chunks_plus_flush_equal_the_offline_search_bitwise(S, lens, lm):
    rehome = lens == "rehome"
    lens = [4, 2, 2, 6, 2] if rehome else lens
    m = _model(TINY, 1, scale=3.0)
    xs = torch.randn(S, sum(lens), TINY["input_size"], generator=torch.Generator().manual_seed(S + len(lens))).to(DEV)
    kw = _lm_kw(lm, TINY["vocab_size"])
    committed = 0
    for W in (1, 4, 8):
        per, rest, nscore, lp, eng = _stream(m, S, lens, xs, W, rehome_at=3 if rehome else None, **kw)
        want, wn = _offline(lp, W, **kw)
        for s in range(S):
            assert _joined(per, rest, s) == want[s], (W, s)
        assert torch.equal(nscore, wn), W
        assert eng.n_collapses == 0
        committed += sum(len(c[s]) for c in per for s in range(S))
    assert committed > 0, "nothing was committed before the flush"


def test_e6d2_one_frame_per_chunk_with_lm_bitwise():
    """E6D2 dims, 64 streams x 16 chunks of 2 input frames (every frame a chunk boundary), W = 4 with an
    LMModel(1024, 64, 1024, 2)-shaped LM."""
    S, C, V = 64, 16, 1024
    m = _model(E6D2, 3, head=32.0)
    lm = _lm_module(V, 64, 1024, 2, 2.0, seed=6)
    kw = dict(lm=lm, lm_weight=0.5, length_bonus=0.5)
    xs = torch.randn(S, 2 * C, 240, generator=torch.Generator().manual_seed(4)).to(DEV)
    per, rest, nscore, lp, eng = _stream(m, S, [2] * C, xs, 4, **kw)
    want, wn = _offline(lp, 4, **kw)
    for s in range(S):
        assert _joined(per, rest, s) == want[s], s
    assert torch.equal(nscore, wn) and eng.n_collapses == 0
    n = sum(len(c[s]) for c in per for s in range(S))
    print("  e6d2 W=4 + LM: %d tokens committed before the flush, %d at it" % (n, sum(map(len, rest))))
    assert n > S


# ---- 2. against fp64 ----------------------------------------------------------------------------------------------------
def test_against_model_beam_search_and_fp64():
    from oracle import ctc as oc
    S, W, lens = 3, 4, [2, 4, 2, 6, 4, 2]
    m = _model(TINY, 5, scale=3.0)
    xs = torch.randn(S, sum(lens), TINY["input_size"], generator=torch.Generator().manual_seed(6)).to(DEV)
    per, rest, nscore, lp, _ = _stream(m, S, lens, xs, W)
    m.set_precision("fp32")
    ids, nlp = m.beam_search(xs, W=W)
    sd = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    lr = oc.ctc_encoder_forward(sd, xs.double().cpu())
    for s in range(S):
        seq, ds, beam, _ = cbo.prefix_beam_search(lr[s].numpy(), lr.shape[1], W, 0)
        tot = sorted((float(cbo.logadd(np.float64(pb), np.float64(pnb))) + f for _, pb, pnb, f in beam), reverse=True)
        assert len(tot) < 2 or tot[0] - tot[1] > 1e-4, "a near-tie between the two best prefixes"
        got = _joined(per, rest, s)
        assert got == ids[s].tolist() and tuple(got) == seq, s
        assert abs(float(nscore[s]) - float(nlp[s])) <= 1e-5 * abs(float(nlp[s]))
        assert abs(float(nscore[s]) - ds) <= 1e-5 * abs(ds)


# ---- 3. commit and collapse against the restatement ---------------------------------------------------------------------
def _hash(seq):
    h = 0
    for k in seq:
        h = (h * MUL + k + 1) & 0xffffffffffffffff
    return h


def _close(a, b):
    return a == b or abs(a - b) <= 1e-5 * max(1.0, abs(b))


@pytest.mark.parametrize("lm", [None, "identity"])
def test_commit_and_collapse_against_the_restatement(lm):
    from edgedict_b200.stream_engine import CTCStreamBeamEngine
    S, W, n, C, V = 3, 4, 2, 16, TINY["vocab_size"]
    m = _model(TINY, 7, scale=2.0)
    kw = _lm_kw(lm, V)
    rkw = {}
    if lm:
        rkw = dict(lm_sd={k: v.detach().float() for k, v in kw["lm"].state_dict().items()},
                   lm_weight=kw["lm_weight"], length_bonus=kw["length_bonus"])
    eng = CTCStreamBeamEngine(m, S, n, W, max_pending=2, **kw)           # n_out = 1: suffixes of at most 1 after a commit
    P, T = eng.max_pending, eng.n_out
    rs = [CTCStreamBeamRestatement(W, max_pending=P, dtype=np.float32, **rkw) for _ in range(S)]
    xs = torch.randn(C + 1, S, 2 * n, TINY["input_size"], generator=torch.Generator().manual_seed(8)).to(DEV)

    def check():
        for s in range(S):
            hy = eng.hypotheses(s)
            assert len(hy) == len(rs[s].hyps)
            for (suf, pb, pnb, f, h, ph), want in zip(hy, rs[s].hyps):
                whole = rs[s].committed + suf
                assert whole == want["seq"] and len(suf) <= P - T
                assert h == _hash(whole)
                if whole:
                    assert ph == _hash(whole[:-1])
                assert _close(pb, float(want["pb"])) and _close(pnb, float(want["pnb"])) and _close(f, float(want["f"]))

    for c in range(C):
        ids, cnt = eng.step(xs[c, :, :n])
        lp = eng.logprobs.view(S, T, V).cpu().numpy()
        for s in range(S):
            assert ids[s, :int(cnt[s])].tolist() == rs[s].chunk(lp[s]), (c, s)
        check()
    assert eng.n_collapses == sum(r.n_collapses for r in rs) > 0
    # a longer chunk after load_state: a carried suffix of 1 exceeds the new bound max_pending - 2 = 0
    eng2 = CTCStreamBeamEngine(m, S, 2 * n, W, max_pending=2, state=eng.state(), **kw)
    pending = [r.commit(eng2.n_out) for r in rs]
    assert eng2.n_collapses == sum(r.collapsed for r in rs) > 0
    ids, cnt = eng2.step(xs[C])
    lp = eng2.logprobs.view(S, eng2.n_out, V).cpu().numpy()
    for s in range(S):
        assert ids[s, :int(cnt[s])].tolist() == pending[s] + rs[s].chunk(lp[s]), s
    eng, T = eng2, eng2.n_out
    check()


# ---- 4. a repeat across a chunk boundary --------------------------------------------------------------------------------
@pytest.mark.parametrize("W, max_pending", [(1, 64), (4, 1)])
def test_built_head_holds_and_repeats_across_chunk_boundaries(W, max_pending):
    """tovocab weight 0, so the logits are the bias; one output frame per chunk.  W = 1 commits its whole prefix after
    every chunk, W = 4 with max_pending 1 collapses every chunk: either way each chunk starts from an empty stored suffix
    and the carried last token.  Token 5 over two chunks is committed once, again after a blank chunk."""
    from edgedict_b200.stream_engine import CTCStreamBeamEngine
    m = _model(TINY, 2)
    lin = m.tovocab[0]
    with torch.no_grad():
        lin.weight.zero_()
    eng = CTCStreamBeamEngine(m, 2, 2, W, max_pending=max_pending)
    xs = torch.randn(2, 2, TINY["input_size"], device=DEV)
    seq = []
    for tok in (5, 5, 0, 5, 9, 5):
        with torch.no_grad():                                 # in place: the program reads the weights where they are
            lin.bias.zero_()
            lin.bias[tok] = 4.0
        ids, cnt = eng.step(xs)
        assert int(cnt[0]) == int(cnt[1])
        seq.append(ids[0, :int(cnt[0])].tolist())
    assert seq == [[5], [], [], [5], [9], [5]]
    assert eng.last.tolist() == [5, 5]


# ---- 5. independence and state ------------------------------------------------------------------------------------------
def test_streams_are_independent_and_states_are_refused_across_kinds():
    from edgedict_b200.stream_engine import CTCStreamBeamEngine, CTCStreamEngine
    S, W, n, C = 5, 4, 4, 6
    m = _model(TINY, 9, scale=3.0)
    kw = _lm_kw("identity", TINY["vocab_size"])
    xs = torch.randn(S, n * C, TINY["input_size"], generator=torch.Generator().manual_seed(10)).to(DEV)
    per, rest, nscore, _, eng = _stream(m, S, [n] * C, xs, W, **kw)
    for s in (0, 3):
        p1, r1, n1, _, _ = _stream(m, 1, [n] * C, xs[s:s + 1], W, **kw)
        assert [c[0] for c in p1] == [c[s] for c in per] and r1[0] == rest[s]
        assert torch.equal(n1[0], nscore[s])
    with pytest.raises(ValueError, match="state keys"):
        CTCStreamEngine(m, S, n, state=eng.state())
    with pytest.raises(ValueError, match="state keys"):
        CTCStreamBeamEngine(m, S, n, W, state=CTCStreamEngine(m, S, n).state(), **kw)
    with pytest.raises(ValueError, match="state keys"):                   # a beam without the LM
        CTCStreamBeamEngine(m, S, n, W, state=eng.state())


# ---- 6. the decoder ------------------------------------------------------------------------------------------------------
class _Tok:
    class tokenizer:
        @staticmethod
        def id_to_token(i):
            return "t%d</w>" % i


def test_stream_decoder_beam_text():
    from edgedict_b200 import ctc
    from edgedict_b200.ctc import CTCStreamDecoder
    m = _model(TINY, 11, scale=3.0)
    lens = [2, 2, 4, 6, 2]
    xs = torch.randn(1, sum(lens), TINY["input_size"], generator=torch.Generator().manual_seed(12)).to(DEV)
    dec = CTCStreamDecoder(m, lambda f: f, _Tok, device=DEV, beam_width=4)
    texts, lps, t0 = [], [], 0
    for n in lens:
        texts.append(dec.decode(xs[:, t0:t0 + n].transpose(1, 2)))
        lps.append(dec._engine.logprobs.view(1, dec._engine.n_out, -1).clone())
        t0 += n
    texts.append(dec.flush())
    ids, _ = ctc.beam_search(torch.cat(lps, 1), [sum(lens) // 2], 4)
    assert "".join(texts) == "".join("t%d " % k for k in ids[0].tolist())
    # greedy: today's decoder, with flush() == ""
    g = CTCStreamDecoder(m, lambda f: f, _Tok, device=DEV)
    gt, t0 = [], 0
    for n in lens:
        gt.append(g.decode(xs[:, t0:t0 + n].transpose(1, 2)))
        t0 += n
    assert g.flush() == ""
    m.set_precision("fp32")
    want, _ = m.greedy_decode(xs, torch.tensor([sum(lens)]))
    assert "".join(gt) == "".join("t%d " % k for k in want[0].tolist())
