"""Greedy decoding with up to K = max_symbols symbols per encoder frame: the ARGMAX continuation flag and the SKIP phase
of the decode program (csrc/decode.cu), GreedyEngine / Transducer.greedy_decode and StreamEngine /
PytorchStreamDecoder against the CPU restatement in tests/multi_symbol_oracle.py, batch invariance, a teacher-forced
fp64 check at E6D2_LARGE dims, and the argument checks.  K = 1 must be the one-symbol program, bit for bit."""
import numpy as np
import pytest
import torch

from tests import multi_symbol_oracle as mo
from tests.util import E4D1_CFG, e4d1_inputs, load_e4d1, load_tiny, rel_err, to_t

f32, f64, i32 = torch.float32, torch.float64, torch.int32
DEV = "cuda"


def _shift_blank(sd, shift):
    sd = dict(sd)
    b = sd["joint.joint.2.bias"].clone()
    b[0] += shift
    sd["joint.joint.2.bias"] = b
    return sd


def _tiny_sd(shift=0.0):
    z, cfg, sd, _ = load_tiny()
    return z, cfg, _shift_blank(to_t(sd), shift)


def _model(cfg, sd):
    from edgedict_b200.rnnt.models import Transducer
    m = Transducer(output_loss=False, **cfg)
    m.load_state_dict(sd)
    return m.cuda().eval()


def _e4d1_sd():
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(10)
    m = Transducer(**E4D1_CFG)
    return {k: v.detach().clone() for k, v in m.state_dict().items() if not k.startswith("loss")}


# ---- CPU: the restatement and the argument checks ----------------------------------------------------------------------
def test_oracle_k1_reproduces_reference_fixtures():
    z, _, sd = _tiny_sd()
    ids, nlp = mo.greedy_decode(sd, torch.as_tensor(z["xs"]), z["xlen"], max_symbols=1)
    for i, row in zip(ids, z["greedy_ids"]):
        assert (i == row[:len(i)]).all()
    assert rel_err(nlp, z["greedy_nlp"]) < 1e-5
    e = load_e4d1()
    xs, _ = e4d1_inputs()
    ids, nlp = mo.greedy_decode(_e4d1_sd(), xs, torch.tensor([200, 200]), max_symbols=1, fast=True)
    assert (np.stack(ids) == e["greedy_ids"]).all()
    assert rel_err(nlp, e["greedy_nlp"]) < 1e-4


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("shift", [1.0, 5.0])
def test_oracle_multi_symbol_equals_batch1_loop(K, shift):
    """The batched restatement against a plain per-utterance loop of the rule."""
    import torch.nn.functional as F
    from oracle import model_torch as mt
    z, _, sd = _tiny_sd(shift)
    xs = torch.as_tensor(z["xs"])
    ids, nlp = mo.greedy_decode(sd, xs, z["xlen"], max_symbols=K)
    h_enc, _ = mt.encoder(sd, xs)
    rounds = set()
    for b in range(xs.shape[0]):
        x, (h, c) = mt.decoder(sd, torch.zeros(1, 0, dtype=torch.long), None)
        seq, lp = [], 0.0
        for t in range(h_enc.shape[1]):
            row = [0] * K
            for j in range(K):
                p, k = F.log_softmax(mt.joint(sd, h_enc[b:b + 1, t], x[:, 0]), 1).max(1)
                row[j], lp = int(k), lp + float(p)
                if int(k) == 0:
                    break
                x, (h, c) = mt.decoder(sd, k[:, None], (h, c))
            rounds.add(j)
            seq += row
        assert ids[b].tolist() == seq[:int(z["xlen"][b]) * K], b
        assert abs(float(nlp[b]) + lp) < 1e-4 * abs(lp)
    assert len(rounds) > 1, "every frame stopped in the same round"


def test_max_symbols_checked_before_device_work():
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    from edgedict_b200.stream_engine import GreedyEngine, StreamEngine, check_max_symbols
    _, cfg, sd = _tiny_sd()
    m = Transducer(output_loss=False, **cfg)                 # on the CPU: any device work would fail differently
    m.load_state_dict(sd)
    xs = torch.zeros(1, 4, cfg["input_size"])
    for bad, err in ((0, ValueError), (17, ValueError), (-1, ValueError), (2.0, TypeError), ("2", TypeError),
                     (True, TypeError), (None, TypeError)):
        with pytest.raises(err):
            check_max_symbols(bad)
        with pytest.raises(err):
            m.greedy_decode(xs, torch.tensor([4]), max_symbols=bad)
        with pytest.raises(err):
            GreedyEngine(m, 1, 2, max_symbols=bad)
        with pytest.raises(err):
            StreamEngine(m, 1, 2, max_symbols=bad)
        with pytest.raises(err):
            PytorchStreamDecoder(None, transducer=m, transform=lambda f: f, tokenizer=object(), device="cpu",
                                 max_symbols=bad)
    assert check_max_symbols(1) == 1 and check_max_symbols(np.int64(16)) == 16
    with pytest.raises(RuntimeError, match="CUDA"):           # the arguments are fine: the device is what is missing
        GreedyEngine(m, 1, 2)
    with pytest.raises(ValueError):
        PytorchStreamDecoder(None, transducer=m, transform=lambda f: f, tokenizer=object(), device="cpu",
                             beam_width=4, max_symbols=2)


# ---- phase level ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("V,unk,logp", [(33, 3, False), (1025, 3, False), (1025, -1, True), (31, -1, True)])
def test_argmax_continuation_phase(V, unk, logp):
    """ARGMAX with F_CONT against the plain ARGMAX on the same logits: rows whose tok_out holds blank stay blank with
    a blank hist entry and their log p bitwise unchanged; the other rows get the plain phase's token, hist and log p
    bitwise, <unk> rule included."""
    from edgedict_b200.stream_engine import EbPhase, F_CONT, F_LOGP, PH_ARGMAX, _ptr
    from tests.test_gpu_decode_fp64 import _argmax_rows, _bits, _run_all
    gen = torch.Generator().manual_seed(V + unk)
    x = torch.cat([_argmax_rows(V, max(unk, 3), gen), torch.randn(30, V, generator=gen) * 3]).to(DEV)   # S = 70
    S, HL, col, blank = x.shape[0], 4, 2, 0
    tok0 = torch.randint(1, V, (S,), generator=gen).int().to(DEV)
    tok0[::3] = blank
    y0 = (torch.randn(S, generator=gen) * 5).to(DEV)
    outs = {}
    for cont in (False, True):
        tok, hist, y = tok0.clone(), torch.full((S, HL), -7, dtype=i32, device=DEV), y0.clone()
        ph = EbPhase(type=PH_ARGMAX, S=S, N=V, flags=(F_CONT if cont else 0) | (F_LOGP if logp else 0), x1=_ptr(x),
                     ldx1=V, aux=blank, aux2=unk, tok_out=_ptr(tok), hist=_ptr(hist), hist_ld=HL, hist_col=col,
                     y=_ptr(y))

        def reset():
            tok.copy_(tok0)
            hist.fill_(-7)
            y.copy_(y0)

        outs[cont] = _run_all([ph], [tok, hist, y], reset)
    (tp, hp, yp), (tc, hc, yc) = outs[False], outs[True]
    done, live = tok0 == blank, tok0 != blank
    assert (tc[done] == blank).all() and (hc[done, col] == blank).all(), "finished rows"
    assert torch.equal(_bits(yc[done]), _bits(y0[done])), "finished rows' log p changed"
    assert torch.equal(tc[live], tp[live]) and torch.equal(hc[live], hp[live]), "live rows differ from ARGMAX"
    assert torch.equal(_bits(yc[live]), _bits(yp[live])), "live rows' log p differs from ARGMAX"
    assert (hc[:, [0, 1, 3]] == -7).all(), "hist columns"
    if not logp:
        assert torch.equal(_bits(yc), _bits(y0)), "y written without F_LOGP"


@pytest.mark.gpu
@pytest.mark.parametrize("live_row", [None, 69])
def test_skip_phase(live_row):
    """S = 70 (two row tiles): SKIP over two COPYs when every token is blank, none when one row (in the last tile) is
    live.  A chain of dependent COPYs after it checks that every CTA counts the same grid barriers."""
    from edgedict_b200.stream_engine import EbPhase, PH_COPY, PH_SKIP, _ptr
    from tests.test_gpu_decode_fp64 import _bits, _run_all
    S, N, blank = 70, 300, 0
    gen = torch.Generator().manual_seed(1)
    tok = torch.full((S,), blank, dtype=i32, device=DEV)
    if live_row is not None:
        tok[live_row] = 5
    a = torch.randn(S, N, generator=gen).to(DEV)
    bufs = [torch.empty(S, N, device=DEV) for _ in range(6)]
    cp = lambda s, d: EbPhase(type=PH_COPY, S=S, N=N, x1=_ptr(s), y=_ptr(d))
    prog = [cp(a, bufs[0]), EbPhase(type=PH_SKIP, S=S, aux=2, aux2=blank, tok_in=_ptr(tok)), cp(bufs[0], bufs[1]),
            cp(bufs[1], bufs[2]), cp(bufs[0], bufs[3]), cp(bufs[3], bufs[4]), cp(bufs[4], bufs[5]),
            EbPhase(type=PH_SKIP, S=S, aux=5, aux2=blank, tok_in=_ptr(tok)), cp(bufs[5], bufs[0])]   # jumps past the end

    def reset():
        for b in bufs:
            b.fill_(float("nan"))

    got = _run_all(prog, bufs, reset)
    for k in (0, 3, 4, 5):
        assert torch.equal(_bits(got[k]), _bits(a)), "buffer %d" % k
    for k in (1, 2):
        if live_row is None:
            assert torch.isnan(got[k]).all(), "skipped COPY %d ran" % k
        else:
            assert torch.equal(_bits(got[k]), _bits(a)), "COPY %d did not run" % k


# ---- GreedyEngine / greedy_decode ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_greedy_k1_is_the_one_symbol_program():
    from edgedict_b200.stream_engine import GreedyEngine
    from tests.test_gpu_decode_fp64 import _bits
    z, cfg, sd = _tiny_sd(1.0)
    m = _model(cfg, sd)
    g = torch.Generator().manual_seed(2)
    h = torch.randn(70, 9, m.encoder.proj.weight.shape[0], generator=g).to(DEV)
    a, b = GreedyEngine(m, 70, 9), GreedyEngine(m, 70, 9, max_symbols=1)
    assert a.nphase == b.nphase and a.hist.shape == b.hist.shape
    ha, la = (t.clone() for t in a.run(h))
    hb, lb = b.run(h)
    assert torch.equal(ha, hb) and torch.equal(_bits(la), _bits(lb))
    xs, xlen = torch.as_tensor(z["xs"]).cuda(), torch.as_tensor(z["xlen"])
    ia, na = m.greedy_decode(xs, xlen)
    ib, nb = m.greedy_decode(xs, xlen, max_symbols=1)
    assert all((p == q).all() for p, q in zip(ia, ib)) and torch.equal(_bits(na), _bits(nb))


def _greedy_vs_oracle(m, sd, xs, xlen, K, fast=False):
    ids, nlp = m.greedy_decode(xs.cuda(), xlen, max_symbols=K)
    want, wnlp = mo.greedy_decode(sd, xs, xlen, max_symbols=K, fast=fast)
    for b, (p, q) in enumerate(zip(ids, want)):
        assert p.shape == q.shape and (p == q).all(), "row %d: first difference at %s" % (b, np.argwhere(p != q)[:3])
    assert rel_err(nlp.cpu(), wnlp) < 1e-4
    return np.concatenate([i.reshape(-1, K) for i in ids])


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 4, 16])
@pytest.mark.parametrize("shift", [0.0, 1.0, 5.0])
def test_greedy_tiny_vs_oracle(K, shift):
    z, cfg, sd = _tiny_sd(shift)
    m = _model(cfg, sd)
    _greedy_vs_oracle(m, sd, torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"]), K)
    g = torch.Generator().manual_seed(K)                     # B = 70: two row tiles, mixed stopping rounds
    xs = torch.randn(70, 14, cfg["input_size"], generator=g) * 1.5
    xlen = torch.randint(8, 15, (70,), generator=g)
    xlen[0] = 14
    _greedy_vs_oracle(m, sd, xs, xlen, K)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 4, 16])
def test_greedy_e4d1_vs_oracle(K):
    """E4D1 in fp32 mode: at random init every frame emits in every round, so each frame takes all K rounds."""
    sd = _e4d1_sd()
    m = _model(E4D1_CFG, sd)
    xs, _ = e4d1_inputs()
    a = _greedy_vs_oracle(m, sd, xs, torch.tensor([200, 170]), K, fast=True)
    assert (a != 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 3, 16])
def test_greedy_forced_emission_takes_k_rounds(K):
    """Blank bias at -1e4: no frame ends on blank, so every frame takes exactly K rounds and the predictor steps on
    every token."""
    z, cfg, sd = _tiny_sd(-1e4)
    m = _model(cfg, sd)
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    a = _greedy_vs_oracle(m, sd, xs, xlen, K)
    assert (a != 0).all()


@pytest.mark.gpu
def test_greedy_mixed_rows_and_batch_invariance():
    """B = 70 rows that stop at different rounds; each row decoded alone gives the same ids and log p, bitwise."""
    from edgedict_b200.stream_engine import GreedyEngine
    from tests.test_gpu_decode_fp64 import _bits
    _, cfg, sd = _tiny_sd(1.0)
    m = _model(cfg, sd)
    K, B, T = 4, 70, 10
    g = torch.Generator().manual_seed(4)
    h = (torch.randn(B, T, m.encoder.proj.weight.shape[0], generator=g) * 2).to(DEV)
    eng = GreedyEngine(m, B, T, max_symbols=K)
    hist, lp = (t.clone() for t in eng.run(h))
    taken = 1 + (hist.view(B, T, K)[:, :, :K - 1] != 0).sum(2)        # rounds each frame took
    counts = torch.bincount(taken.flatten().cpu(), minlength=K + 1)
    print("  rounds taken per frame (1..K):", counts[1:].tolist())
    assert (counts[1:] > 0).sum() >= 2, "rows should stop at different rounds"
    one = GreedyEngine(m, 1, T, max_symbols=K)
    for b in range(B):
        h1, l1 = one.run(h[b:b + 1])
        assert torch.equal(h1[0], hist[b]) and torch.equal(_bits(l1), _bits(lp[b:b + 1])), "row %d" % b


@pytest.mark.gpu
def test_greedy_engine_teacher_forced_large():
    """E6D2_LARGE dims (weights x 2, blank bias + 3 so that about half the frames emit), B = 70, T' = 6, K = 4: each
    frame and round in fp64 from the engine's own hist, with test_greedy_engine_teacher_forced's bars: every token lies
    in the fp64 argmax set of its logits' bar, rows stop exactly at their first blank or after K tokens, skipped
    rounds hold blank, and the predictor steps exactly for the non-blank tokens."""
    from edgedict_b200.rnnt.tokenizer import BOS
    from edgedict_b200.stream_engine import GreedyEngine
    from tests.test_gpu_decode_fp64 import LARGE, _Pred, _scaled, may_win
    model = _scaled(LARGE, seed=10)
    with torch.no_grad():
        model.joint.joint[2].bias[0] += 3.0
    B, T, K = 70, 6, 4
    E = model.encoder.proj.weight.shape[0]
    g = torch.Generator().manual_seed(9)
    h_enc = (torch.randn(B, T, E, generator=g) * 2).to(DEV)
    eng = GreedyEngine(model, B, T, max_symbols=K)
    hist = eng.run(h_enc)[0].clone().view(B, T, K)
    P = _Pred(model)
    Ld, Hd = model.decoder.lstm.num_layers, model.decoder.lstm.hidden_size
    z0 = torch.zeros(Ld, B, Hd, dtype=f64, device=DEV)
    st, dx, ddx = P.step(torch.full((B,), BOS, dtype=i32, device=DEV), (z0, z0, z0, z0))
    und, per_round = [0] * T, [0] * K
    for t in range(T):
        live = torch.ones(B, dtype=torch.bool, device=DEV)
        for j in range(K):
            tok = hist[:, t, j]
            assert (tok[~live] == 0).all(), "frame %d round %d: a finished row holds a token" % (t, j)
            if not live.any():
                continue
            hid, dhid = P.joint(h_enc[:, t], dx, ddx)
            zz, dz = P.logits(hid, dhid)
            ok = may_win(zz, dz, -1).gather(1, tok.long()[:, None])[:, 0]
            assert ok[live].all(), "frame %d round %d rows %s: token outside the fp64 argmax set" % (
                t, j, (live & ~ok).nonzero().flatten()[:5].tolist())
            und[t] += int((may_win(zz, dz, -1).sum(1) > 1)[live].sum())
            per_round[j] += int(live.sum())
            step = live & (tok != 0)
            if step.any():
                nst, nx, ndx = P.step(torch.where(step, tok, torch.zeros_like(tok)), st)
                st = tuple(torch.where(step[None, :, None], a, b) for a, b in zip(nst, st))
                dx, ddx = torch.where(step[:, None], nx, dx), torch.where(step[:, None], ndx, ddx)
            live = step
    # the predictor's bars are propagated worst-case from round to round (its state is recomputed, not read back), so
    # at these dims many tokens lie inside their logits' bar: the count is reported, the stop rule is checked exactly
    print("  large teacher-forced: rows live per round %s of %d; inside the logits' bar per frame: %s" % (
        per_round, B * T, und))
    assert per_round[1] > 0 and per_round[0] > per_round[1]


# ---- StreamEngine / PytorchStreamDecoder ----------------------------------------------------------------------------------
def _stream_vs_oracle(m, sd, chunks, K, unk, S):
    """chunks [C, S, n, F]: every stream's non-blank tokens of every chunk against mo.stream_decode."""
    from edgedict_b200.stream_engine import StreamEngine
    from oracle import model_torch as mt
    n = chunks.shape[2]
    eng = StreamEngine(m, S, n, unk_id=unk, max_symbols=K)
    got = np.stack([eng.step(c.cuda()).cpu().numpy().copy() for c in chunks])        # [C, S, n_out * K]
    assert got.shape[2] == eng.n_out * K
    for s in range(S):
        st = mt.StreamState(sd)
        for ci in range(chunks.shape[0]):
            want = mo.stream_decode(sd, st, chunks[ci, s:s + 1], unk_id=unk, max_symbols=K, fast=True)
            row = got[ci, s].reshape(-1, K)
            for f in row:                                    # within a frame, blanks only after the last token
                nz = np.flatnonzero(f)
                assert nz.size == 0 or nz[-1] == nz.size - 1, (s, ci, row)
            assert [int(t) for t in row.flatten() if t != 0] == want, (s, ci)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("K,n,unk", [(2, 2, 11), (4, 4, 11), (3, 2, 3)])
def test_stream_many_streams_vs_oracle(K, n, unk):
    """70 streams with independent state; for unk != 3 that token's joint bias is raised so that the <unk> rule fires;
    the blank bias is raised by 1 so that frames stop at different rounds."""
    z, cfg, sd = _tiny_sd(1.0)
    if unk != 3:
        b = sd["joint.joint.2.bias"]
        b[unk] = float(b.max()) + 1.0
    m = _model(cfg, sd)
    g = torch.Generator().manual_seed(K * 10 + n)
    chunks = torch.randn(8, 70, n, cfg["input_size"], generator=g) * 1.5
    got = _stream_vs_oracle(m, sd, chunks, K, unk, 70)
    assert (got != 0).any() and (got == 0).any()


@pytest.mark.gpu
def test_stream_state_across_chunk_length_rebuild():
    """Chunks of 4, 4, 2, 6, 2 frames through PytorchStreamDecoder with K = 3: each length change rebuilds the engine
    with the carried state and the same max_symbols; the text equals the restatement's tokens."""
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    from oracle import model_torch as mt
    z, cfg, sd = _tiny_sd(1.0)
    m = _model(cfg, sd)

    class Tok:
        vocab_size = 16

        class tokenizer:
            @staticmethod
            def id_to_token(i):
                return "t%d</w>" % i

            @staticmethod
            def token_to_id(t):
                return 3 if t == "<unk>" else None

    dec = PytorchStreamDecoder(FLAGS=None, transducer=m, transform=lambda f: f.transpose(1, 2), tokenizer=Tok(),
                               max_symbols=3)
    g = torch.Generator().manual_seed(7)
    chunks = [torch.randn(1, n, cfg["input_size"], generator=g) for n in (4, 4, 2, 6, 2, 4)]
    st = mt.StreamState(sd)
    engine, rebuilds = None, 0
    for c in chunks:
        text = dec.decode(c)
        rebuilds += dec._engine is not engine
        engine = dec._engine
        assert dec._engine.max_symbols == 3
        want = mo.stream_decode(sd, st, c, max_symbols=3)
        assert text == "".join("t%d " % t for t in want)
    assert rebuilds == 5


@pytest.mark.gpu
def test_stream_e6d2_large_64_streams():
    """E6D2_LARGE (weights x 2, blank bias + 3), 64 streams, chunks of 2 log-mel frames, K = 4: every stream token for
    token against the restatement."""
    from tests.test_gpu_decode_fp64 import LARGE, _scaled
    model = _scaled(LARGE, seed=10)
    with torch.no_grad():
        model.joint.joint[2].bias[0] += 3.0
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(0)
    chunks = torch.randn(4, 64, 2, 240, generator=g)
    got = _stream_vs_oracle(model, sd, chunks, 4, 3, 64)
    print("  large stream: non-blank per round", (got.reshape(-1, 4) != 0).sum(0).tolist())
    assert (got[..., 1] != 0).sum() > 0
