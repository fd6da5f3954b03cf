"""Streaming beam search (stream_engine.StreamBeamEngine: BEAM_SELECT's streaming mode, flag 64, and BEAM_COMMIT of
csrc/decode.cu; PytorchStreamDecoder(beam_width=...)).  Cutting the audio into chunks must not change the search: the
committed tokens of every chunk plus the flush are BeamEngine's result over the same encoder frames, bit for bit.
The commit and collapse rule is checked against a CPU restatement, W = 1 against the greedy stream, and the argument
checks without a GPU."""
import numpy as np
import pytest
import torch

from tests import lm_oracle as lo
from tests.test_gpu_beam_engine import LARGE, SMALL, _scaled_model, _tiny
from tests.test_gpu_beam_lm import _perm_map
from tests.test_oracle_lm import _lm_sd, load_lm

HASH_MUL, MASK64 = 0x100000001b3, (1 << 64) - 1


def _ids(ids, counts, s):
    return ids[s, :int(counts[s])].tolist()


def _stream(m, chunks, W, merge=True, max_pending=256, **kw):
    """Run the chunks (a list of [S, n, F]) through StreamBeamEngine, rebuilding it with the carried state whenever
    the chunk length changes.  -> (committed ids per chunk and stream, flushed ids per stream, -log p [S], the
    concatenated per-chunk encoder output [S, T', E], the engine)."""
    from edgedict_b200.stream_engine import StreamBeamEngine
    eng, per, enc = None, [], []
    S = chunks[0].shape[0]
    for c in chunks:
        if eng is None or eng.n != c.shape[1]:
            eng = StreamBeamEngine(m, S, c.shape[1], W, merge=merge, max_pending=max_pending,
                                   state=None if eng is None else eng.state(), **kw)
        ids, counts = eng.step(c.cuda())
        per.append([_ids(ids, counts, s) for s in range(S)])
        enc.append(eng.enc_out.clone())
    ids, counts, nlp = eng.flush()
    return per, [_ids(ids, counts, s) for s in range(S)], nlp, torch.cat(enc, 1), eng


def _offline(m, enc, W, merge=True, **kw):
    from edgedict_b200.stream_engine import BeamEngine
    S, T = enc.shape[0], enc.shape[1]
    eng = BeamEngine(m, S, T, W, merge=merge, **kw)
    ids, nlp = eng.run(enc, torch.full((S,), T, dtype=torch.int32, device="cuda"))
    return [[int(k) for k in r if k >= 0] for r in ids.cpu().numpy()], nlp.cpu()


def _joined(per, fl):
    return [sum((c[s] for c in per), []) + fl[s] for s in range(len(fl))]


def _chunks(S, lens, F, seed, scale=1.5):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(S, n, F, generator=g) * scale for n in lens]


LENS = {"2": [2] * 14, "4": [4] * 7, "mixed": [4, 2, 6, 2, 4, 2, 6, 2]}


@pytest.mark.gpu
@pytest.mark.parametrize("lens", sorted(LENS))
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 4, 8])
def test_chunking_is_invisible_to_the_search(W, merge, lens):
    """Committed ids of every chunk plus the flush equal BeamEngine.run over the concatenated per-chunk encoder output:
    ids identical, -log p bitwise (both run the same phases on the same rows).  Mixed lengths go through the
    state-carrying rebuild."""
    m, z, sd = _tiny()
    chunks = _chunks(3, LENS[lens], sd["encoder.norm.weight"].shape[0], seed=len(lens) * 10 + W)
    per, fl, nlp, enc, eng = _stream(m, chunks, W, merge)
    want, wlp = _offline(m, enc, W, merge)
    got = _joined(per, fl)
    print("W=%d merge=%s lens=%s: %s, committed before the flush %d of %d tokens"
          % (W, merge, lens, got, sum(len(x) for c in per for x in c), sum(map(len, got))))
    assert eng.n_collapses == 0
    assert got == want
    assert torch.equal(nlp.view(torch.int32), wlp.view(torch.int32))
    assert sum(map(len, got)) > 0


@pytest.mark.gpu
def test_chunking_is_invisible_to_the_search_e6d2_large():
    m = _scaled_model(LARGE, seed=10)
    chunks = _chunks(2, [2, 4, 2, 2, 6, 2] * 5, 240, seed=3, scale=1.0)
    per, fl, nlp, enc, eng = _stream(m, chunks, 4)
    want, wlp = _offline(m, enc, 4)
    got = _joined(per, fl)
    print("E6D2_LARGE W=4: %d tokens, %d committed before the flush"
          % (sum(map(len, got)), sum(len(x) for c in per for x in c)))
    assert eng.n_collapses == 0 and got == want
    assert torch.equal(nlp.view(torch.int32), wlp.view(torch.int32))
    assert sum(map(len, got)) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("lm", [None, "identity", "permuted"])
def test_stream_matches_restatement(lm):
    """The tiny fixture's 40 stream chunks as one stream against the CPU restatement on the whole utterance:
    ids equal, -log p within 1e-4."""
    m, z, sd = _tiny()
    kw, okw = {}, {}
    if lm is not None:
        _, lsd = load_lm()
        tmap = _perm_map(16, lsd["encoder.weight"].shape[0]) if lm == "permuted" else None
        kw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5, lm_token_map=tmap)
        okw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5, lm_map=tmap)
    chunks = [torch.as_tensor(c[None]) for c in z["stream_chunks"]]
    for W in (1, 4):
        per, fl, nlp, _, _ = _stream(m, chunks, W, **kw)
        want, wlp = lo.beam_search(sd, torch.cat(chunks, 1), None, W=W, **okw)
        got = _joined(per, fl)
        err = abs(float(nlp[0]) - float(wlp[0])) / abs(float(wlp[0]))
        print("lm=%s W=%d: %s, rel err %.2e" % (lm, W, got[0], err))
        assert got == want
        assert err < 1e-4


# ---- CPU restatement of the streaming beam: lm_oracle.beam_search's frame (with or without the LM), then the commit
# and collapse rule at each chunk end, and before a chunk whose n_out outgrows the bound the beam was left under

def _seq_hash(seq):
    h = 0
    for k in seq:
        h = (h * HASH_MUL + k + 1) & MASK64
    return h


def _restate_stream(sd, xs, chunk_out, W, max_pending, merge=True, blank=0, lm_sd=None, lm_weight=0.0,
                    length_bonus=0.0, lm_bos=1):
    """-> (committed ids per chunk, the live hypotheses' full sequences after each chunk)"""
    import torch.nn.functional as F
    from oracle import model_torch as mt
    V = sd["joint.joint.2.weight"].shape[0]
    h_enc, _ = mt.encoder(sd, xs, None)
    dec_x, (dh, dc) = mt.decoder(sd, torch.zeros(1, 0, dtype=torch.long), None)
    hyps = [dict(seq=[], lp=torch.zeros(()), x=dec_x[0, 0], h=dh[:, 0], c=dc[:, 0])]
    if lm_sd is not None:
        llp, (lh, lc) = lo.lm_prime(lm_sd, lm_bos)
        hyps[0].update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
    done, t, per, live = 0, 0, [], []

    def commit(n_out):
        nonlocal hyps, done
        pend = [h["seq"][done:] for h in hyps]
        c = 0
        while all(len(p) > c and p[c] == pend[0][c] for p in pend):
            c += 1
        out = pend[0][:c]
        done += c
        if max(len(p) for p in pend) - c > max_pending - n_out:
            best = max(range(len(hyps)), key=lambda i: (float(hyps[i]["lp"]), -i))
            out += hyps[best]["seq"][done:]
            done = len(hyps[best]["seq"])
            hyps = [hyps[best]]
        return out

    for n_out in chunk_out:
        out = commit(n_out)                   # a no-op unless n_out grew
        for _ in range(n_out):
            cand = []
            for qi, hy in enumerate(hyps):
                a = F.log_softmax(mt.joint(sd, h_enc[0, t][None], hy["x"][None])[0], 0)
                if lm_sd is not None:
                    a = a + lo.fusion_term(hy["llp"].to(a.dtype), V, blank, lm_weight, length_bonus)
                lp = a + hy["lp"]
                cand += [(float(lp[k]), qi, k, lp[k]) for k in range(lp.shape[0])]
            cand.sort(key=lambda c: (-c[0], c[1], c[2]))
            new, seen = [], {}
            for _, qi, k, lpk in cand[:W]:
                hy = hyps[qi]
                seq = hy["seq"] + ([k] if k != blank else [])
                if merge and tuple(seq) in seen:
                    seen[tuple(seq)]["lp"] = torch.logaddexp(seen[tuple(seq)]["lp"], lpk)
                    continue
                nh = dict(hy, seq=seq, lp=lpk)
                if k != blank:
                    nx, (h2, c2) = mt.decoder(sd, torch.full((1, 1), k), (hy["h"][:, None], hy["c"][:, None]))
                    nh.update(x=nx[0, 0], h=h2[:, 0], c=c2[:, 0])
                    if lm_sd is not None:
                        llp, (lh, lc) = lo.lm_step(lm_sd, torch.tensor([k]), (hy["lh"][:, None], hy["lc"][:, None]))
                        nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
                seen[tuple(seq)] = nh
                new.append(nh)
            hyps = new
            t += 1
        per.append(out + commit(n_out))
        live.append([h["seq"] for h in hyps])
    return per, live


def _check_commits(m, sd, chunks, W, P, merge=True, lm=False):
    """Stream one utterance (chunks [1, n, F], the engine rebuilt with the carried state whenever n changes) and check
    every chunk's committed ids against the restatement, and after every chunk the engine's live slots: committed
    tokens + stored suffix (at most max_pending - n_out long) equal the restatement's hypotheses, and the stored
    hash is that of the whole sequence, so the committed tokens are a prefix of every live hypothesis.
    -> (forced collapses, those of them made when a rebuilt engine took over the beam, tokens committed)"""
    from edgedict_b200.stream_engine import StreamBeamEngine
    kw, okw = {}, {}
    if lm:
        lsd = load_lm()[1]
        kw = dict(lm=lsd, lm_weight=0.3, length_bonus=0.5)
        okw = dict(lm_sd=lsd, lm_weight=0.3, length_bonus=0.5)
    outs = [ch.shape[1] // 2 for ch in chunks]
    want, wlive = _restate_stream(sd, torch.cat(chunks, 1), outs, W, P, merge, **okw)
    eng, done, collapses, at_load = None, [], 0, 0
    for i, c in enumerate(chunks):
        if eng is None or eng.n != c.shape[1]:
            if eng is not None:
                collapses += eng.n_collapses
            eng = StreamBeamEngine(m, 1, c.shape[1], W, merge=merge, max_pending=P,
                                   state=None if eng is None else eng.state(), **kw)
            at_load += eng.n_collapses
        ids, counts = eng.step(c.cuda())
        got = _ids(ids, counts, 0)
        assert got == want[i], ("chunk", i, got, want[i])
        done += got
        live = int(eng.hist_live[0, -1])
        seqs = eng.seqs[0].cpu().numpy()
        full = []
        for s in range(live):
            row = seqs[s]
            assert 0 <= row[0] <= P - eng.n_out, ("chunk", i, "slot", s, "suffix length", row[0])
            sq = done + row[3:3 + row[0]].tolist()
            assert (int(row[1]) & 0xffffffff) | ((int(row[2]) & 0xffffffff) << 32) == _seq_hash(sq), ("hash", i, s)
            full.append(sq)
        assert full == wlive[i], ("chunk", i)
    return collapses + eng.n_collapses, at_load, len(done)


@pytest.mark.gpu
@pytest.mark.parametrize("lm", [False, True])
@pytest.mark.parametrize("merge", [True, False])
def test_forced_collapse_matches_restatement(merge, lm):
    """max_pending = n_out + 2 forces collapses (with an LM, the collapse also moves the LM state and logits)."""
    m, z, sd = _tiny()
    chunks = [torch.as_tensor(np.concatenate(z["stream_chunks"][i:i + 2], 0)[None]) for i in range(0, 40, 2)]
    collapses, _, n = _check_commits(m, sd, chunks, 4, 4, merge, lm)
    print("merge=%s lm=%s: %d forced collapses over %d chunks, %d tokens committed" % (merge, lm, collapses,
                                                                                      len(chunks), n))
    assert collapses > 0


@pytest.mark.gpu
@pytest.mark.parametrize("lm", [False, True])
def test_longer_chunks_keep_the_suffix_bound(lm):
    """Chunks of 2 frames (n_out 1) then 6 frames (n_out 3) with max_pending = 3: a beam left under the bound of the
    short chunks (suffixes up to 2 tokens) would outgrow its rows in a long chunk; the rebuilt engine first brings it
    under its own bound (max_pending - 3 = 0, a collapse) and returns those tokens with the next chunk."""
    m, z, sd = _tiny()
    ch = torch.as_tensor(z["stream_chunks"]).reshape(1, -1, 12)
    lens = [2, 2, 2, 6, 2, 2, 6, 6, 2, 4, 2, 6, 2, 2, 6, 6, 2, 2, 2, 6, 2, 2, 6]
    assert sum(lens) == ch.shape[1]
    cuts = np.cumsum([0] + lens)
    chunks = [ch[:, a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    collapses, at_load, n = _check_commits(m, sd, chunks, 4, 3, True, lm)
    print("lm=%s: %d forced collapses (%d when a rebuilt engine took over) over %d chunks, %d tokens committed"
          % (lm, collapses, at_load, len(chunks), n))
    assert at_load > 0


@pytest.mark.gpu
def test_width_one_is_the_greedy_stream_without_unk_rule():
    """W = 1 commits, chunk by chunk, exactly the non-blank tokens of StreamEngine with the <unk> rule off."""
    from edgedict_b200.stream_engine import StreamBeamEngine, StreamEngine
    m, z, sd = _tiny()
    S, n = 4, 4
    chunks = _chunks(S, [n] * 12, 12, seed=5)
    greedy = StreamEngine(m, S, n, unk_id=-1)
    beam = StreamBeamEngine(m, S, n, 1, max_pending=n // 2)
    total = 0
    for i, c in enumerate(chunks):
        g = greedy.step(c.cuda()).cpu().numpy()
        ids, counts = beam.step(c.cuda())
        for s in range(S):
            assert _ids(ids, counts, s) == [int(k) for k in g[s] if k != 0], ("chunk", i, "stream", s)
            total += int(counts[s])
    assert total > 0 and beam.n_collapses == 0


@pytest.mark.gpu
def test_streams_are_independent_bitwise():
    """S = 5 streams of different audio (with collapses): each stream's output is bitwise its S = 1 output."""
    m, z, sd = _tiny()
    chunks = _chunks(5, [4] * 10, 12, seed=9)
    per, fl, nlp, _, eng = _stream(m, chunks, 4, max_pending=4)
    assert eng.n_collapses > 0
    for s in range(5):
        per1, fl1, nlp1, _, _ = _stream(m, [c[s:s + 1] for c in chunks], 4, max_pending=4)
        assert [c[0] for c in per1] == [c[s] for c in per], s
        assert fl1[0] == fl[s], s
        assert nlp1.view(torch.int32)[0] == nlp.view(torch.int32)[s], s


@pytest.mark.gpu
@pytest.mark.parametrize("with_lm", [False, True])
def test_state_survives_chunk_length_change_and_rehomed_weights(with_lm):
    """A chunk of another length or re-homed parameter storage rebuilds the program but continues the beam, predictor
    and LM state: the result is the single-length run's, bitwise."""
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import StreamBeamEngine, param_fingerprint
    from tests.util import load_tiny
    _, cfg, sd, _ = load_tiny()
    m = Transducer(output_loss=False, **cfg)
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    m = m.cuda().eval()
    kw = dict(lm=load_lm()[1], lm_weight=0.5, length_bonus=0.3) if with_lm else {}
    lens = [4, 4, 2, 6, 2, 4]
    g = torch.Generator().manual_seed(7)
    chunks = [torch.randn(1, n, cfg["input_size"], generator=g) * 1.5 for n in lens]
    eng, got = None, []
    for i, c in enumerate(chunks):
        if i == 3:                                   # re-home the weights mid-utterance
            for p in m.parameters():
                p.data = p.data.clone()
        if eng is None or eng.n != c.shape[1] or eng.fingerprint != param_fingerprint(m):
            eng = StreamBeamEngine(m, 1, c.shape[1], 4, state=None if eng is None else eng.state(), **kw)
        ids, counts = eng.step(c.cuda())
        got += _ids(ids, counts, 0)
    ids, counts, nlp = eng.flush()
    got += _ids(ids, counts, 0)
    one = StreamBeamEngine(m, 1, 2, 4, **kw)
    want = []
    for c in chunks:
        for j in range(0, c.shape[1], 2):
            ids, counts = one.step(c[:, j:j + 2].cuda())
            want += _ids(ids, counts, 0)
    ids, counts, wlp = one.flush()
    want += _ids(ids, counts, 0)
    print("lm=%s: %s" % (with_lm, got))
    assert got == want and len(got) > 0
    assert torch.equal(nlp.view(torch.int32), wlp.view(torch.int32))


@pytest.mark.gpu
def test_stream_decoder_beam_interface():
    """PytorchStreamDecoder(beam_width=4) with injected transform and tokenizer: decode returns str, the decode texts
    plus flush() are the offline best hypothesis' text, and reset() starts over."""
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    m, z, _ = _tiny()

    class Tok:
        vocab_size = 16

        class tokenizer:
            @staticmethod
            def id_to_token(i):
                return "<unk>" if i == 3 else "t%d</w>" % i

            @staticmethod
            def token_to_id(t):
                return 3 if t == "<unk>" else None

    dec = PytorchStreamDecoder(FLAGS=None, transducer=m, transform=lambda f: f.transpose(1, 2), tokenizer=Tok(),
                               beam_width=4)
    parts = [dec.decode(torch.as_tensor(ch[None])) for ch in z["stream_chunks"]]
    assert all(isinstance(p, str) for p in parts)
    text = "".join(parts) + dec.flush()
    best, _ = m.beam_search(torch.as_tensor(z["stream_chunks"]).reshape(1, -1, 12).cuda(), None, W=4)
    want = "".join("<unk>" if t == 3 else "t%d " % t for t in best[0])
    assert text == want and len(text) > 0
    assert sum(map(len, parts)) > 0                   # text arrives before the flush
    assert len(dec.encoder_elapsed) == len(z["stream_chunks"])
    dec.reset()
    again = "".join(dec.decode(torch.as_tensor(ch[None])) for ch in z["stream_chunks"]) + dec.flush()
    assert again == text


# ---- argument checks, no GPU

def _cpu(module_type="LSTM"):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(0)
    return Transducer(output_loss=False, module_type=module_type, **SMALL)


@pytest.mark.parametrize("what,args,kw", [
    ("W = 0", (1, 4, 0), {}),
    ("W too large", (1, 4, 1025), {}),
    ("max_pending < n_out", (1, 8, 4), dict(max_pending=3)),
    ("lm_weight without lm", (1, 4, 4), dict(lm_weight=0.5)),
    ("malformed lm state_dict", (1, 4, 4), dict(lm={"encoder.weight": torch.zeros(3, 2)})),
    ("lm of another vocabulary without a map", (1, 4, 4), dict(lm=_lm_sd(ntok=50))),
    ("lm_bos out of range", (1, 4, 4), dict(lm=_lm_sd(), lm_bos=96)),
    ("odd chunk before a time reduction", (1, 3, 4), {}),
    ("no streams", (0, 4, 4), {}),
])
def test_stream_beam_arguments_checked_before_any_device_work(what, args, kw):
    """A CPU model gets the ValueError, not the engine's 'needs a CUDA device' error."""
    from edgedict_b200.stream_engine import StreamBeamEngine
    with pytest.raises(ValueError):
        StreamBeamEngine(_cpu(), *args, **kw)


def test_stream_beam_refuses_a_gru_encoder():
    from edgedict_b200.stream_engine import StreamBeamEngine
    with pytest.raises(ValueError, match="LSTM encoder"):
        StreamBeamEngine(_cpu("GRU"), 1, 4, 4)


def test_stream_beam_needs_a_cuda_model():
    from edgedict_b200.stream_engine import StreamBeamEngine
    with pytest.raises(RuntimeError, match="CUDA"):
        StreamBeamEngine(_cpu(), 1, 4, 4)


def test_stream_decoder_checks_beam_arguments():
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder

    class Tok:
        class tokenizer:
            @staticmethod
            def token_to_id(t):
                return None

    for kw in (dict(beam_width=0), dict(beam_width=2, lm_weight=1.0)):
        with pytest.raises(ValueError):
            PytorchStreamDecoder(FLAGS=None, transducer=_cpu(), transform=lambda f: f, tokenizer=Tok(), device="cpu",
                                 **kw)
