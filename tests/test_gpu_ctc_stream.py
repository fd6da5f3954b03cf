"""Streaming greedy CTC on the device (stream_engine.CTCStreamEngine, ctc.CTCStreamDecoder; csrc/decode.cu GRU and
CTC_EMIT through eb_decode_run_ctc_stream):

* the GRU phase alone, teacher-forced, against fp64 per element, with test_gpu_decode_fp64's error model for the 3xTF32
  products (`_n_add` over the K segments) propagated through the cell as test_gpu_gru_recurrence_fp64's fwd_ref does
  (EPS_LIBM for expf / tanhf, the r * gh_n product, the h update); the power check against plain TF32, NaN-prefilled
  outputs and bitwise equal outputs for max_ctas 0 / 1 / 3 / 17;
* the emission phase alone against a host restatement on its own log-probs, bitwise: ties, NaN rows, -inf rows,
  all-equal rows and a repeat carried across the launch boundary;
* whole chunks at E6D2 dims, layer by layer, against fp64 from the engine's own buffers;
* token for token against the CPU restatement (tests/ctc_stream_oracle.py) and against CTCEncoder.greedy_decode on the
  concatenated frames, the reference's fixture included; bitwise invariances.

pytest -s prints the worst err/bar of every phase and shape; DESIGN.md's verification table records them."""
import numpy as np
import pytest
import torch

from tests.ctc_stream_oracle import CTCStreamRestatement
from tests.test_gpu_decode_fp64 import CTAS, _adversarial, _bits, _n_add, _nan, _power, linear_ref, ln_ref
from tests.test_gpu_lstm_recurrence_fp64 import EPS_LIBM, SAT, U24, UTC, _report
from tests.test_oracle_ctc import load_ctc_tiny

pytestmark = pytest.mark.gpu

f32, f64, i32 = torch.float32, torch.float64, torch.int32
DEV = "cuda"
TINY = dict(vocab_size=40, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0, proj_size=32)
E6D2 = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0, proj_size=640)


def _run(phases, max_ctas=0):
    from edgedict_b200._lib import check, lib
    from edgedict_b200.stream_engine import EbPhase
    arr = (EbPhase * len(phases))(*phases)
    prog = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(DEV)
    bar = torch.zeros(64, dtype=i32, device=DEV)
    check(lib().eb_decode_run_ctc_stream(prog.data_ptr(), len(phases), bar.data_ptr(), max_ctas,
                                         torch.cuda.current_stream().cuda_stream), "eb_decode_run_ctc_stream")
    torch.cuda.synchronize()


def _run_all(phases, outs, reset):
    """test_gpu_decode_fp64._run_all through eb_decode_run_ctc_stream: every max_ctas of CTAS gives the same bits."""
    first = None
    for mc in CTAS:
        reset()
        _run(phases, mc)
        snap = [o.clone() for o in outs]
        if first is None:
            first = snap
            continue
        for k, (a, b) in enumerate(zip(first, snap)):
            assert torch.equal(_b(a), _b(b)), "output %d: max_ctas=%d differs from the full grid" % (k, mc)
    return first


def _b(t):
    """The bits of a float32 / float64 tensor (NaN equal to itself), integers as they are."""
    return t.contiguous().view(torch.int64) if t.dtype == f64 else _bits(t)


# ---- GRU phase ----------------------------------------------------------------------------------------------------------
def gru_ref(x, wih, h, whh, bih, bhh):
    """One GRU phase step in fp64 with its bar: r, z from one accumulator over both products plus b_ih then b_hh; n_x and
    n_h from their own columns; n = tanh((n_x + b_in) + r (n_h + b_hn)); y = (1 - z) n + z h."""
    x, wih, h, whh, bih, bhh = (a.double() for a in (x, wih, h, whh, bih, bhh))
    H = whh.shape[1]
    na = _n_add(wih.shape[1], whh.shape[1]) * UTC
    gi, gh = x @ wih.t(), h @ whh.t()
    ai, ah = x.abs() @ wih.abs().t(), h.abs() @ whh.abs().t()
    part = lambda t, g: t[:, g * H:(g + 1) * H]
    gates = []
    for g in (0, 1):
        acc = part(gi, g) + part(gh, g)
        pre = acc + part(bih[None], g) + part(bhh[None], g)
        dpre = na * (part(ai, g) + part(ah, g)) + 2 * U24 * (acc.abs() + part(bih[None], g).abs() + pre.abs())
        s = torch.sigmoid(pre)
        gates.append((s, s * (1 - s) * dpre + EPS_LIBM + U24 * s))
    (r, dr), (z, dz) = gates
    xn = part(gi, 2) + bih[2 * H:]
    dxn = na * part(ai, 2) + U24 * xn.abs()
    hn = part(gh, 2) + bhh[2 * H:]
    dhn = na * part(ah, 2) + U24 * hn.abs()
    a = xn + r * hn
    da = dxn + dr * hn.abs() + r * dhn + 2 * U24 * ((r * hn).abs() + a.abs())
    n = torch.tanh(a)
    dn = (1 - n * n) * da + EPS_LIBM + U24 * n.abs()
    y = (1 - z) * n + z * h
    dy = dz * (n.abs() + h.abs()) + (1 - z) * dn + 3 * U24 * (((1 - z) * n).abs() + (z * h).abs())
    return y, dy, r


# S, H, K1, mode.  plain: dense rows; strided: the encoder's x1 = X + t K1 (ldx1 = 3 K1) and h = y_{t-1} (ldx2 = 3 H);
# sat: 10 % of the biases at the saturation values; bhn30: b_hn = +-30 with the reset pre-activation at +-20.
GRU_CASES = [
    (1, 48, 48, "plain"),
    (7, 100, 240, "strided"),
    (64, 1024, 1024, "plain"),
    (130, 100, 240, "strided"),
    (130, 1024, 240, "plain"),
    (64, 48, 240, "sat"),
    (130, 100, 100, "sat"),
    (7, 1024, 1024, "bhn30"),
    (70, 48, 48, "bhn30"),
]


@pytest.mark.parametrize("S,H,K1,mode", GRU_CASES)
def test_gru_phase(S, H, K1, mode):
    from edgedict_b200.stream_engine import EbPhase, PH_GRU, _ptr
    gen = torch.Generator().manual_seed(S * 7 + H + K1 + len(mode))
    rnd = lambda *s, sc=1.0: (torch.randn(*s, generator=gen) * sc).to(DEV)
    G = 3 * H
    wih, whh = rnd(G, K1, sc=1.5 / K1 ** 0.5), rnd(G, H, sc=1.5 / H ** 0.5)
    bih, bhh = rnd(G, sc=0.5), rnd(G, sc=0.5)
    scale = 2.0 ** -round(np.log2(0.3 * (K1 + H)))           # the adversarial pre-activation stays O(1)
    for g in range(3):                                        # unit 0: every gate row
        wih[g * H] = _adversarial(K1, scale, gen).to(DEV)
        whh[g * H] = _adversarial(H, scale, gen).to(DEV)
    if mode == "sat":
        sat = torch.tensor(SAT, device=DEV)
        pick = torch.rand(2, G, generator=gen).to(DEV) < 0.1
        vals = sat[torch.randint(0, len(SAT), (2, G), generator=gen).to(DEV)] * \
            torch.where(torch.rand(2, G, generator=gen).to(DEV) < 0.5, -1.0, 1.0)
        bih = torch.where(pick[0], vals[0], bih)
        bhh = torch.where(pick[1], vals[1], bhh)
    if mode == "bhn30":
        bhh[2 * H:] = torch.where(torch.rand(H, generator=gen).to(DEV) < 0.5, -30.0, 30.0)
        bih[:H] = torch.where(torch.rand(H, generator=gen).to(DEV) < 0.5, -20.0, 20.0)
    ni, t = (3, 1) if mode == "strided" else (1, 0)
    X = rnd(S, ni, K1)
    X[0, t] = _adversarial(K1, 1.0, gen).to(DEV)
    Y = rnd(S, ni, H) * 0.7
    hsrc = Y[:, t - 1] if mode == "strided" else rnd(S, H) * 0.7
    hsrc[0] = _adversarial(H, 1.0, gen).to(DEV)
    if mode == "strided":
        Y[:, t - 1] = hsrc
        x2, ldx2 = Y.view(-1)[(t - 1) * H:], ni * H
    else:
        x2, ldx2 = hsrc, H
    x1, ldx1 = X.view(-1)[t * K1:], ni * K1
    ybuf = _nan(S, ni * H + 3)
    y2 = _nan(S, H)
    ph = EbPhase(type=PH_GRU, S=S, N=H, K1=K1, K2=H, x1=_ptr(x1), ldx1=ldx1, x2=_ptr(x2), ldx2=ldx2, w1=_ptr(wih),
                 ldw1=K1, w2=_ptr(whh), ldw2=H, b1=_ptr(bih), b2=_ptr(bhh), y=_ptr(ybuf, t * H), ldy=ni * H + 3,
                 y2=_ptr(y2))

    def reset():
        ybuf.fill_(float("nan"))
        y2.fill_(float("nan"))

    yb, y2g = _run_all([ph], [ybuf, y2], reset)
    y = yb[:, t * H:(t + 1) * H]
    assert torch.isnan(torch.cat([yb[:, :t * H], yb[:, (t + 1) * H:]], 1)).all(), "GRU wrote outside its y columns"
    assert torch.equal(_bits(y2g), _bits(y)), "y2 is not a bitwise copy of y"
    xv = X[:, t]
    yr, dy, r = gru_ref(xv, wih, hsrc, whh, bih, bhh)
    if mode == "bhn30":
        assert (r < 1e-8).any() and (r > 1 - 1e-7).any()
    name = "gru S=%d H=%d K1=%d %s" % (S, H, K1, mode)
    _report(name, [("y", y, yr, dy)])
    pre_bar = _n_add(K1, H) * UTC * (torch.cat([xv, hsrc], 1).double().abs() @
                                     torch.cat([wih, whh], 1).double().abs().t())
    _power(name, [(xv, wih), (hsrc, whh)], pre_bar)


# ---- CTC_EMIT phase ---------------------------------------------------------------------------------------------------------
def _emit_phase(S, n, V, blank, logits, lp, prev, out, score, am):
    from edgedict_b200.stream_engine import EbPhase, PH_CTC_EMIT, _ptr
    return EbPhase(type=PH_CTC_EMIT, S=S, N=V, aux=n, aux2=blank, x1=_ptr(logits), ldx1=V, y=_ptr(lp), ldy=V,
                   tok_out=_ptr(prev), hist=_ptr(out), hist_ld=n, tok_out2=_ptr(out, S * n), y2=_ptr(score),
                   seq_out=_ptr(am))


def _host_emit(lp, prev, blank):
    """The collapse on the host from the device's log-probs [S, n, V]: torch.argmax per frame, prev [S] carried."""
    am = torch.argmax(lp.cpu(), -1)
    rows = lp.double().sum(-1).cpu()
    ids, sc, prev = [], [], prev.clone()
    for s in range(lp.shape[0]):
        out, acc = [], 0.0
        for t in range(lp.shape[1]):
            c = int(am[s, t])
            if c != blank and c != int(prev[s]):
                out.append(c)
                acc += float(rows[s, t])
            prev[s] = c
        ids.append(out)
        sc.append(acc)
    return am, ids, torch.tensor(sc, dtype=f64), prev


@pytest.mark.parametrize("V,blank", [(1, 0), (33, 0), (40, 7), (1024, 0), (1025, 1024)])
def test_emit_phase_against_host_restatement(V, blank):
    nan, inf = float("nan"), float("inf")
    S, n = 70, 4
    gen = torch.Generator().manual_seed(V + blank)
    x = torch.randn(S, n, V, generator=gen) * 3
    x[:, :, :min(V, 4)] += 2.0 * torch.randint(0, 2, (S, n, min(V, 4)), generator=gen)   # frequent repeats
    if V > 1:
        for s in range(0, 10):                                # exact ties inside a lane and across lanes
            a, d = s % min(V, 5), (1, 32, 64)[s % 3]
            if a + d < V:
                x[s, 1, a] = x[s, 1, a + d] = x[s, 1].max() + 1.0
    x[10, 0] = nan
    x[11, 2] = -inf
    x[12, 1, V // 2] = nan
    x[13, 3] = 0.25                                           # all equal: the lowest id
    x[14, :] = x[14, 0]                                       # one row repeated over the chunk
    x[15, 1] = -inf
    x[15, 1, V - 1] = 1.0
    logits = x.to(DEV).reshape(S * n, V)
    lp, out = _nan(S * n, V), torch.full((S * n + S,), -9, dtype=i32, device=DEV)
    am = torch.full((S, n), -9, dtype=i32, device=DEV)
    prev0 = torch.randint(-1, V, (S,), generator=gen).to(DEV, i32)
    prev0[16] = int(torch.argmax(x[16, 0]))                   # a repeat carried across the launch boundary
    score0 = (torch.randn(S, generator=gen, dtype=f64) * 10).to(DEV)
    prev, score = prev0.clone(), score0.clone()
    ph = _emit_phase(S, n, V, blank, logits, lp, prev, out, score, am)

    def reset():
        lp.fill_(nan)
        out.fill_(-9)
        am.fill_(-9)
        prev.copy_(prev0)
        score.copy_(score0)

    lpg, outg, amg, prevg, scg = _run_all([ph], [lp, out, am, prev, score], reset)
    want_am, want_ids, want_sc, want_prev = _host_emit(lpg.view(S, n, V), prev0.cpu().long(), blank)
    assert torch.equal(amg.cpu().long(), want_am), "per-frame argmax"
    assert torch.equal(prevg.cpu().long(), want_prev), "carried argmax"
    counts = outg[S * n:].cpu()
    ids = outg[:S * n].view(S, n).cpu()
    for s in range(S):
        assert counts[s] == len(want_ids[s]) and ids[s, :counts[s]].tolist() == want_ids[s], "stream %d" % s
    assert int(counts[16]) == 0 or ids[16, 0] != prev0[16], "the carried repeat was emitted again"
    got = scg.cpu() - score0.cpu()
    fin = torch.isfinite(want_sc)
    assert torch.equal(torch.isnan(got), torch.isnan(want_sc))
    rel = float(((got[fin] - want_sc[fin]).abs() / want_sc[fin].abs().clamp_min(1e-30)).max()) if fin.any() else 0.0
    print("  emit V=%d blank=%d: score rel err %.3g, %d ids" % (V, blank, rel, int(counts.sum())))
    assert rel <= 1e-5
    # the log-probs against fp64 where the row is finite: (x - m) - log(sum exp(x - m)) in fp32
    xd = logits.double().cpu()
    ok = torch.isfinite(xd).all(1)
    ref = torch.log_softmax(xd[ok], 1)
    m = xd[ok].max(1, keepdim=True).values
    bar = 4 * U24 * ((xd[ok] - m).abs() + ref.abs()) + (-(-V // 32) + 6) * U24 + 2.0 ** -22
    _report("emit logp V=%d" % V, [("lp", lpg.cpu()[ok], ref, bar)])
    assert torch.equal(torch.isnan(lpg.cpu()[~ok]), torch.isnan(torch.log_softmax(xd[~ok].float(), 1)))


# ---- engines ------------------------------------------------------------------------------------------------------------------
def _model(cfg, seed, scale=1.0):
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(seed)
    m = CTCEncoder(**cfg).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(scale)
    return m.to(DEV)


def _sd(m):
    return {k: v.detach() for k, v in m.state_dict().items()}


def _margins(lp):
    top = lp.double().topk(2, -1).values if lp.shape[-1] > 1 else None
    return None if top is None else top[..., 0] - top[..., 1]


def _stream_tokens(m, S, lens, xs, max_ctas=0, rehome_at=None, blank=0):
    """Stream xs [S, sum(lens), F] through CTCStreamEngine with the state-carrying rebuild at every change of chunk
    length (and after re-homing the weights before chunk rehome_at).  -> (ids per stream, per-frame argmax [S, T'],
    log-probs [S, T', V], score)."""
    from edgedict_b200.stream_engine import CTCStreamEngine, param_fingerprint
    eng, ids, ams, lps, t0 = None, [[] for _ in range(S)], [], [], 0
    for ci, n in enumerate(lens):
        if ci == rehome_at:
            with torch.no_grad():
                for p in m.parameters():
                    p.data = p.data.clone()
            assert eng.fingerprint != param_fingerprint(m)
        if eng is None or eng.n != n or eng.fingerprint != param_fingerprint(m):
            eng = CTCStreamEngine(m, S, n, blank=blank, max_ctas=max_ctas, state=None if eng is None else eng.state())
        got, cnt = eng.step(xs[:, t0:t0 + n])
        t0 += n
        for s in range(S):
            ids[s] += got[s, :int(cnt[s])].tolist()
        ams.append(eng.argmax.clone())
        lps.append(eng.logprobs.view(S, eng.n_out, -1).clone())
    return ids, torch.cat(ams, 1), torch.cat(lps, 1), eng.score().clone(), eng


@pytest.mark.parametrize("S", [3, 70])
@pytest.mark.parametrize("lens", [[2] * 8, [4] * 4, [2, 4, 6, 2, 2], "rehome"])
def test_tiny_token_for_token_against_restatement(S, lens):
    rehome = lens == "rehome"
    lens = [4, 2, 2, 6, 2] if rehome else lens
    m = _model(TINY, 1, scale=3.0)
    sd = {k: v.double().cpu() for k, v in _sd(m).items()}
    T = sum(lens)
    xs = torch.randn(S, T, TINY["input_size"], generator=torch.Generator().manual_seed(S + T)).to(DEV)
    ids, am, lp, score, _ = _stream_tokens(m, S, lens, xs, rehome_at=3 if rehome else None)
    rs = CTCStreamRestatement(sd, S, 0, device=DEV)
    want = [[] for _ in range(S)]
    lps = []
    t0 = 0
    for n in lens:
        out, l, _ = rs.step(xs[:, t0:t0 + n].double())
        t0 += n
        lps.append(l)
        for s in range(S):
            want[s] += out[s]
    ref = torch.cat(lps, 1)
    mg = _margins(ref)
    assert float(mg.min()) > 1e-4, "a near-tie: the fp32 and fp64 argmax may differ"
    assert ids == want
    assert sum(map(len, ids)) > S
    assert torch.allclose(score.cpu(), rs.score, rtol=1e-5, atol=1e-5)
    print("  tiny S=%d %s: %d ids, worst |lp - fp64| %.3g" % (S, lens, sum(map(len, ids)),
                                                             float((lp.double() - ref).abs().max())))


def test_built_head_holds_and_repeats_across_chunk_boundaries():
    """tovocab weight 0, so the logits are the bias: token 5 over two chunks is emitted once; after a blank chunk it is
    emitted again; a chunk of token 9 then 5 emits both."""
    from edgedict_b200.stream_engine import CTCStreamEngine
    m = _model(TINY, 2)
    lin = m.tovocab[0]
    with torch.no_grad():
        lin.weight.zero_()
    eng = CTCStreamEngine(m, 2, 2)
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


def test_e6d2_token_for_token_with_boundary_repeats():
    """E6D2 dims, 64 streams x 24 chunks of 2 input frames (one output frame per chunk, so every repeat is a chunk
    boundary), against the restatement in fp64; the head's bias favours a few tokens so that frames repeat."""
    S, C = 64, 24
    m = _model(E6D2, 3)
    with torch.no_grad():
        m.tovocab[0].bias[[0, 5, 9, 17]] += 2.5
    sd = {k: v.double() for k, v in _sd(m).items()}
    xs = torch.randn(S, 2 * C, 240, generator=torch.Generator().manual_seed(4)).to(DEV)
    ids, am, lp, score, _ = _stream_tokens(m, S, [2] * C, xs)
    rs = CTCStreamRestatement(sd, S, 0, device=DEV)
    want, lps = [[] for _ in range(S)], []
    for c in range(C):
        out, l, _ = rs.step(xs[:, 2 * c:2 * c + 2].double())
        lps.append(l)
        for s in range(S):
            want[s] += out[s]
    ref = torch.cat(lps, 1)
    mg = _margins(ref)
    near = int((mg < 1e-4).sum())
    ref_am = ref.argmax(-1).cpu()
    clear = (mg >= 1e-4).cpu()
    assert torch.equal(am.cpu().long()[clear], ref_am[clear])
    n_ids = sum(map(len, ids))
    rep = int(((ref_am[:, 1:] == ref_am[:, :-1]) & (ref_am[:, 1:] != 0)).sum())
    # a stream with a frame inside the near-tie margin may legitimately take the other token: compare the rest
    whole = clear.all(1)
    print("  e6d2: %d ids, %d collapsed repeats across chunk boundaries, %d near-tie frames, %d of %d streams compared"
          % (n_ids, rep, near, int(whole.sum()), S))
    assert n_ids > 50 and rep >= 1 and int(whole.sum()) >= S - 4
    for s in range(S):
        if whole[s]:
            assert ids[s] == want[s], "stream %d" % s
            assert abs(float(score[s]) - float(rs.score[s])) <= 1e-5 * abs(float(rs.score[s])), "stream %d score" % s


def test_offline_equivalence_tiny_and_fixture():
    """The concatenated chunks through CTCEncoder.greedy_decode (fp32 mode): the same ids and the score within 1e-5
    relative.  Then the reference's fixture: its first 14 of 15 frames in even chunks follow its first 7 log-prob
    frames."""
    m = _model(TINY, 5, scale=3.0)
    S, lens = 9, [2, 4, 2, 6, 4, 2]
    T = sum(lens)
    xs = torch.randn(S, T, TINY["input_size"], generator=torch.Generator().manual_seed(6)).to(DEV)
    ids, am, lp, score, _ = _stream_tokens(m, S, lens, xs)
    m.set_precision("fp32")
    with torch.no_grad():
        off = m(xs)
    assert float(_margins(off).min()) > 1e-4
    want, nlp = m.greedy_decode(xs, torch.full((S,), T))
    assert [w.tolist() for w in want] == ids
    assert torch.allclose(score.float(), -nlp, rtol=1e-5, atol=0)
    z, cfg, sd = load_ctc_tiny()
    from edgedict_b200.rnnt.models import CTCEncoder
    fm = CTCEncoder(**cfg).to(DEV).eval()
    fm.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    xf = torch.as_tensor(z["xs"]).to(DEV)[:, :14]
    fix = torch.as_tensor(z["logprobs"][:, :7])
    assert float(_margins(fix).min()) > 1e-5
    for lens in ([2] * 7, [4, 4, 6], [14]):
        ids, am, _, _, _ = _stream_tokens(fm, 4, lens, xf)
        assert torch.equal(am.cpu().long(), fix.argmax(-1)), lens
        a = fix.argmax(-1)
        for s in range(4):
            keep = [int(a[s, t]) for t in range(7) if a[s, t] != 0 and (t == 0 or a[s, t] != a[s, t - 1])]
            assert ids[s] == keep


def test_e6d2_chunk_layer_by_layer_fp64():
    """Each chunk against fp64 recomputed from the engine's own buffers: the input LN, every layer's GRU steps (x from
    the layer below, h_{t-1} from the layer's own y), the LN (+ residual), the time reduction (bitwise), the projection,
    the logits and the log-probs; the ids equal the fp64 argmax wherever the top-2 margin exceeds the logits' bar."""
    from edgedict_b200.stream_engine import CTCStreamEngine
    S, n, C = 64, 2, 3
    m = _model(E6D2, 7)
    sd = {k: v.double() for k, v in _sd(m).items()}
    enc = m.model
    L, red = len(enc.lstm.lstms), enc.lstm.time_reductions
    xs = torch.randn(C, S, n, 240, generator=torch.Generator().manual_seed(8)).to(DEV)
    eng = CTCStreamEngine(m, S, n)
    worst, decided, frames = {}, 0, 0
    for ci in range(C):
        st0 = eng.state()
        eng.step(xs[ci])
        items = []
        a0r, da0 = ln_ref(xs[ci].reshape(S * n, -1), sd["model.norm.weight"], sd["model.norm.bias"])
        items.append(("a0", eng.a0.view(S * n, -1), a0r, da0))
        X, ni, bi = eng.a0, n, 0
        for i in range(L):
            yL, zL = eng._bufs[bi], eng._bufs[bi + 1]
            bi += 2
            g = lambda nm: sd["model.lstm.lstms.%d.%s_l0" % (i, nm)]
            for t in range(ni):
                hin = st0["enc_h"][i] if t == 0 else yL[:, t - 1]
                yr, dy, _ = gru_ref(X[:, t], g("weight_ih"), hin, g("weight_hh"), g("bias_ih"), g("bias_hh"))
                items.append(("L%d y t%d" % (i, t), yL[:, t], yr, dy))
            assert torch.equal(_bits(eng.enc_h[i]), _bits(yL[:, ni - 1])), "enc_h is not the last step's y"
            H = yL.shape[2]
            z32 = (yL + X) if i > 0 else yL
            zr, dz = ln_ref(z32.reshape(-1, H), sd["model.lstm.projs.%d.0.weight" % i],
                            sd["model.lstm.projs.%d.0.bias" % i])
            items.append(("L%d ln" % i, zL.reshape(-1, H), zr, dz))
            X = zL
            if i in red:
                zp = eng._bufs[bi]
                bi += 1
                assert torch.equal(_bits(zp), _bits(0.5 * (zL[:, 0::2] + zL[:, 1::2]))), "PAIR"
                X, ni = zp, ni // 2
        er, de = linear_ref(X.reshape(S * ni, -1), sd["model.proj.weight"], sd["model.proj.bias"])
        items.append(("enc_out", eng.enc_out.reshape(S * ni, -1), er, de))
        zr, dz = linear_ref(eng.enc_out.reshape(S * ni, -1), sd["tovocab.0.weight"], sd["tovocab.0.bias"])
        items.append(("logits", eng.logits, zr, dz))
        lg = eng.logits.double()
        lpr = torch.log_softmax(lg, 1)
        m_ = lg.max(1, keepdim=True).values
        V = lg.shape[1]
        items.append(("logp", eng.logprobs, lpr,
                      4 * U24 * ((lg - m_).abs() + lpr.abs()) + (-(-V // 32) + 6) * U24 + 2.0 ** -22))
        top = zr.topk(2, 1)
        clear = (top.values[:, 0] - top.values[:, 1]) > 2 * dz.max(1).values + 8 * U24 * lpr.abs().max(1).values
        got = eng.argmax.view(-1).long()
        assert torch.equal(got[clear], top.indices[clear, 0]), "chunk %d: an argmax outside the logits' bar" % ci
        decided, frames = decided + int(clear.sum()), frames + clear.numel()
        for label, gv, ref, bar in items:
            ratio = float(((gv.double() - ref).abs() / (bar + 2.0 ** -120)).max())
            if label not in worst or ratio > worst[label][0]:
                worst[label] = (ratio, gv.clone(), ref, bar)
    _report("ctc stream e6d2 S=%d n=%d" % (S, n), [(k, v[1], v[2], v[3]) for k, v in worst.items()])
    print("  ctc stream e6d2: %d of %d frames decided outside the logits' bar" % (decided, frames))
    assert decided >= frames * 0.9


def test_invariances():
    """Streams independent of each other, repeated runs and reset() equal to a fresh engine, max_ctas 1 / 3 / all: every
    output bitwise."""
    from edgedict_b200.stream_engine import CTCStreamEngine
    m = _model(TINY, 9, scale=3.0)
    S, n, C = 70, 4, 3
    xs = torch.randn(C, S, n, TINY["input_size"], generator=torch.Generator().manual_seed(10)).to(DEV)

    def run(eng, xs):
        outs = []
        for c in range(xs.shape[0]):
            ids, cnt = eng.step(xs[c])
            outs.append((ids, cnt, eng.logprobs.clone(), eng.enc_h.clone()))
        return outs, eng.score().clone()

    def emitted(ids, cnt):                                   # the entries past a stream's count are not written
        return torch.where(torch.arange(ids.shape[1])[None] < cnt[:, None], ids, -1)

    def same(a, b, streams=slice(None)):
        (oa, sa), (ob, sb) = a, b
        assert torch.equal(_b(sa[streams]), _b(sb[streams]))
        for (i1, c1, l1, h1), (i2, c2, l2, h2) in zip(oa, ob):
            assert torch.equal(c1[streams], c2[streams])
            assert torch.equal(emitted(i1, c1)[streams], emitted(i2, c2)[streams])
            assert torch.equal(_bits(l1.view(S, -1)[streams]), _bits(l2.view(S, -1)[streams]))
            assert torch.equal(_bits(h1[:, streams]), _bits(h2[:, streams]))

    eng = CTCStreamEngine(m, S, n)
    base = run(eng, xs)
    eng.reset()
    same(base, run(eng, xs))                                  # reset() then the same chunks
    same(base, run(CTCStreamEngine(m, S, n), xs))             # a fresh engine
    for mc in (1, 3):
        same(base, run(CTCStreamEngine(m, S, n, max_ctas=mc), xs))
    xs2 = xs.clone()
    xs2[:, 5] = torch.randn(C, n, TINY["input_size"], device=DEV) * 3
    other = run(CTCStreamEngine(m, S, n), xs2)
    keep = torch.arange(S) != 5
    same(base, other, keep)
    sub = run(CTCStreamEngine(m, 1, n), xs[:, 11:12])
    for (i1, c1, l1, _), (i2, c2, l2, _) in zip(base[0], sub[0]):
        assert torch.equal(emitted(i1, c1)[11:12], emitted(i2, c2)) and torch.equal(c1[11:12], c2)
        assert torch.equal(_bits(l1.view(S, -1)[11:12]), _bits(l2.view(1, -1)))


def test_stream_decoder_text():
    """CTCStreamDecoder: the text of each chunk's ids with '</w>' as a space; a change of chunk length rebuilds and
    carries the state, so the texts together are greedy_decode's ids."""
    from edgedict_b200.ctc import CTCStreamDecoder

    class Tok:
        class tokenizer:
            @staticmethod
            def id_to_token(i):
                return "t%d</w>" % i

    m = _model(TINY, 11, scale=3.0)
    lens = [2, 2, 4, 6, 2]
    xs = torch.randn(1, sum(lens), TINY["input_size"], generator=torch.Generator().manual_seed(12)).to(DEV)
    dec = CTCStreamDecoder(m, lambda f: f, Tok, device=DEV)
    texts, t0 = [], 0
    for n in lens:
        texts.append(dec.decode(xs[:, t0:t0 + n].transpose(1, 2)))
        t0 += n
    assert len(dec.encoder_elapsed) == len(lens)
    m.set_precision("fp32")
    want, _ = m.greedy_decode(xs, torch.tensor([sum(lens)]))
    assert "".join(texts) == "".join("t%d " % k for k in want[0].tolist())
    dec.reset()
    dec.reset_profile()
    assert dec.decode(xs[:, :2].transpose(1, 2)) == texts[0] and len(dec.encoder_elapsed) == 1
