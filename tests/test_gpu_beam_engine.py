"""Batched beam search on the device (stream_engine.BeamEngine, the BEAM_SELECT / GATHER / BEAM_FINAL phases of
csrc/decode.cu): against the CPU restatement, frame by frame against fp64, batch invariance, repeatability and the
argument checks of Transducer.beam_search."""
import numpy as np
import pytest
import torch

from tests.util import load_tiny, rel_err

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
U32 = 2.0 ** -24


def _tiny(sd_edit=None):
    from edgedict_b200.rnnt.models import Transducer
    z, cfg, sd, _ = load_tiny()
    sd = {k: torch.as_tensor(v).clone() for k, v in sd.items()}
    if sd_edit is not None:
        sd_edit(sd)
    m = Transducer(output_loss=False, **cfg)
    m.load_state_dict(sd)
    return m.cuda().eval(), z, sd


def _scaled_model(cfg, seed):
    """Random-init weights x 2 (as scripts/bench_stream.py): at x 1 the joint emits blanks only."""
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(seed)
    m = Transducer(output_loss=False, **cfg).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)
    return m.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 2, 4, 8, 16, 20])
def test_beam_matches_restatement_ragged(W, merge):
    """Three utterances of different lengths in one batch; W = 20 > V = 16 exercises the short first frame."""
    from oracle import model_torch as mt
    m, z, sd = _tiny()
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    want, wlp = mt.beam_search(sd, xs, xlen, W=W, merge=merge)
    got, glp = m.beam_search(xs.cuda(), xlen, W=W, merge=merge)
    err = float(np.max(np.abs(glp.cpu().numpy() - wlp.numpy()) / np.abs(wlp.numpy())))
    print("W=%d merge=%s: ids %s, -logp %s, max rel err %.2e" % (W, merge, got, glp.cpu().numpy(), err))
    assert got == want
    assert err < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 3])
def test_beam_exact_ties_go_to_the_lowest_index(W):
    """Tokens 5 and 9 get identical rows in the output layer and the largest bias: every frame holds exact value ties,
    which the selection breaks by the lowest flat index (slot * V + token), as the restatement's sort does."""
    from oracle import model_torch as mt

    def tie(sd):
        w, b = sd["joint.joint.2.weight"], sd["joint.joint.2.bias"]
        w[9] = w[5]
        b[5] = b[9] = float(b.max()) + 4.0

    m, z, sd = _tiny(tie)
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    want, wlp = mt.beam_search(sd, xs, xlen, W=W)
    got, glp = m.beam_search(xs.cuda(), xlen, W=W)
    print("W=%d: ids %s" % (W, got))
    assert got == want
    assert rel_err(glp.cpu(), wlp) < 1e-4
    if W == 1:                                       # greedy: the tie goes to token 5 at every frame
        assert any(5 in s for s in got) and not any(9 in s for s in got)


def _dec64(sd64, Ld):
    emb, wp, bp = sd64["decoder.embed.weight"], sd64["decoder.proj.weight"], sd64["decoder.proj.bias"]

    def step(tok, h, c):
        """One fp64 predictor step for tokens [n] from (h, c) [Ld, n, Hd] -> (dec_x, |W_p||h| + |b_p|, h, c)."""
        x, hs, cs = emb[tok], [], []
        for k in range(Ld):
            g = x @ sd64["decoder.lstm.weight_ih_l%d" % k].t() + sd64["decoder.lstm.bias_ih_l%d" % k] + \
                h[k] @ sd64["decoder.lstm.weight_hh_l%d" % k].t() + sd64["decoder.lstm.bias_hh_l%d" % k]
            i, f, gg, o = g.chunk(4, 1)
            ck = f.sigmoid() * c[k] + i.sigmoid() * gg.tanh()
            x = o.sigmoid() * ck.tanh()
            hs.append(x)
            cs.append(ck)
        return x @ wp.t() + bp, x.abs() @ wp.abs().t() + bp.abs(), torch.stack(hs), torch.stack(cs)
    return step


def _check_frame(v, beta, seqs, W, merge, blank, par, tok, lp, live, where):
    """Check the device's survivors of one frame against fp64 candidate values v [n, V] with bars beta [n, V].

    Candidates whose fp64 ranking is decided beyond the bars must be ranked as fp64 ranks them; candidates within the
    bars of each other may go either way, and the device's choice stands.  Returns (worst err / bar of the survivor
    log p, whether the frame held such a near-tie)."""
    n, V = v.shape
    fv, fb = v.ravel(), beta.ravel()
    N, m = fv.size, min(W, fv.size)
    lo, hi = fv - fb, fv + fb
    above = N - np.searchsorted(np.sort(lo), hi, side="right")            # candidates surely better than c
    maybe = N - np.searchsorted(np.sort(hi), lo, side="left") - 1         # candidates possibly better than c
    out, sure = above >= m, maybe < m
    key = lambda c: seqs[c // V] + ((int(c % V),) if c % V != blank else ())
    assert 1 <= live <= m, (where, "live count", live, m)
    kd = [int(par[s]) * V + int(tok[s]) for s in range(live)]
    for s, c in enumerate(kd):
        assert 0 <= par[s] < n and not out[c], (where, "slot", s, "survivor cannot be in the top W")
        for s2 in range(s):
            assert not lo[c] > hi[kd[s2]], (where, "slot", s, "ranked below a worse survivor", s2)
    kseq = [key(c) for c in kd]
    if merge:
        assert len(set(kseq)) == live, (where, "equal sequences left unmerged")
        rep = {q: c for q, c in zip(kseq, kd)}
        for c in np.flatnonzero(sure):
            r = rep.get(key(c))
            assert r is not None, (where, "sure candidate missing", divmod(int(c), V))
            assert not lo[c] > hi[r], (where, "merge kept the later of", divmod(int(c), V), divmod(r, V))
        cand = [c for c in np.flatnonzero(~out) if key(c) in rep]
        assert len(cand) >= m and len(set(kd) | set(np.flatnonzero(sure).tolist())) <= m, (where, "beam size")
    else:
        assert live == m and set(np.flatnonzero(sure).tolist()) <= set(kd), (where, "top W")
        cand = kd
    worst = 0.0
    for s, c in enumerate(kd):
        grp = [x for x in cand if key(x) == kseq[s]] if merge else [c]
        low = np.logaddexp.reduce([fv[x] for x in grp if sure[x] or x == c])
        high = np.logaddexp.reduce([fv[x] for x in grp])
        bar = max(fb[x] for x in grp) + 4 * U32 * (abs(high) + 1)
        err = max(low - lp[s], lp[s] - high, 0.0)
        worst = max(worst, err / bar)
        assert err <= bar, (where, "slot", s, "log p", float(lp[s]), "fp64", low, high, "bar", bar)
    return worst, bool((~out & ~sure).sum() > 1)


@pytest.mark.gpu
@pytest.mark.parametrize("W,merge", [(4, True), (8, True), (4, False)])
def test_beam_teacher_forced_fp64(W, merge):
    """Every frame of the device beam against fp64, starting from the device's own beam at t-1 (its sequences, from
    the history's back-pointers, and its fp32 slot log p).  E6D2_LARGE dims, weights x 2, B = 4, T' = 100, one
    ragged utterance.  So that hypotheses which differ only in the timing of a symbol meet and merge, every encoder
    frame is presented twice, the output layer is sharpened (x 3) and the blank bias raised until blank takes about
    half of the mass at the first frames.

    Error model of a candidate value lp = log_softmax(z)[k] + logp[q] (u = 2^-24), a 6-sigma bar of independent
    roundings (a sum of K fp32 terms p_i errs by about u sqrt(K/2) |p|_2, the 3xTF32 products by 4 u |p|_2 more):
    - predictor output d: |dd_i| <= 2^-16 (|W_p||h| + |b_p|)_i, a budget for the fp32 LSTM chain over the sequence,
      checked against the device's predictor outputs of the final beam;
    - joint hidden pre-activation, K = E + D + 1 terms: du = u (sqrt(K/2) + 4) |W_1 * x|_2 (+) |W_1,dec * dd|_2;
      tanh: dh = (1 - h^2) du + 2 u |h|;
    - logits, J + 1 terms: dz = u (sqrt(J/2) + 4) |W_2 * h|_2 (+) |W_2 * dh|_2  ((+): root sum of squares);
    - log-softmax: the max and the log-sum-exp move by at most max dz + V u, and the three fp32 operations of
      ((z - max) - lse) + logp round by at most 3 u (|z - max| + |lse| + |logp|).
    A merged survivor adds 4 u (|lp| + 1) for the log-adds.  The predictor is recomputed in fp64 from the token
    sequences, so a survivor that inherited the wrong state, or stepped on a blank, fails."""
    from edgedict_b200.rnnt.tokenizer import BOS
    from edgedict_b200.stream_engine import BeamEngine
    m = _scaled_model(LARGE, seed=10)
    B, blank = 4, m.blank
    g = torch.Generator().manual_seed(1)
    xs = torch.randn(B, 100, 240, generator=g).cuda()
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
    frames = torch.tensor([T, T, T - 27, T], dtype=torch.int32)
    eng = BeamEngine(m, B, T, W, merge=merge)
    ids, nlp = eng.run(h_enc, frames.cuda())
    torch.cuda.synchronize()
    hpar, htok = eng.hist_parent.cpu().numpy(), eng.hist_token.cpu().numpy()
    hlp, hlive = eng.hist_logp.cpu().numpy().astype(np.float64), eng.hist_live.cpu().numpy()
    ids, dec_final = ids.cpu().numpy(), eng.dec_x[T & 1].double()

    sd64 = {k: v.detach().double() for k, v in m.state_dict().items()}
    Ld, Hd = m.decoder.lstm.num_layers, m.decoder.lstm.hidden_size
    w1, b1 = sd64["joint.joint.0.weight"], sd64["joint.joint.0.bias"]
    w2, b2 = sd64["joint.joint.2.weight"], sd64["joint.joint.2.bias"]
    J, V, E = w1.shape[0], w2.shape[0], h_enc.shape[2]
    D = w1.shape[1] - E
    c1, c2 = U32 * (np.sqrt((E + D + 1) / 2) + 4), U32 * (np.sqrt((J + 1) / 2) + 4)
    rss = lambda x, w: (x * x) @ (w * w).t()                                # sum_i (w_ji x_i)^2
    step = _dec64(sd64, Ld)
    zs = torch.zeros(Ld, 1, Hd, dtype=torch.float64, device="cuda")
    x0, mag0, hh, cc = step(torch.tensor([BOS], device="cuda"), zs, zs)
    cache = {(): (x0[0], mag0[0], hh[:, 0], cc[:, 0])}
    he64 = h_enc.double()
    worst, near, merges, pred_worst = 0.0, 0, 0, 0.0
    for b in range(B):
        seqs, lps = [()], np.zeros(1)
        for t in range(T):
            where = "utterance %d frame %d" % (b, t)
            live = int(hlive[b, t])
            if t >= int(frames[b]):
                assert live == len(seqs) and (hpar[b, t, :live] == np.arange(live)).all(), where
                assert (htok[b, t, :live] == blank).all() and (hlp[b, t, :live] == lps).all(), where
                continue
            d = torch.stack([cache[s][0] for s in seqs])
            dd = 2.0 ** -16 * torch.stack([cache[s][1] for s in seqs])
            x = torch.cat([he64[b, t].expand(len(seqs), -1), d], 1)
            u = x @ w1.t() + b1
            h = u.tanh()
            du = c1 * (rss(x, w1) + b1 * b1).sqrt() + rss(dd, w1[:, E:]).sqrt()
            dh = (1 - h * h) * du + 2 * U32 * h.abs()
            zz = h @ w2.t() + b2
            dz = c2 * (rss(h, w2) + b2 * b2).sqrt() + rss(dh, w2).sqrt()
            lse = torch.logsumexp(zz, 1, keepdim=True)
            zmax = zz.max(1, keepdim=True).values
            lpq = torch.as_tensor(lps, device="cuda")[:, None]
            v = zz - lse + lpq
            beta = 6 * (dz + dz.max(1, keepdim=True).values) + V * U32 + \
                3 * U32 * ((zz - zmax).abs() + lse.abs() + lpq.abs())
            w, nt = _check_frame(v.cpu().numpy(), beta.cpu().numpy(), seqs, W, merge, blank, hpar[b, t],
                                 htok[b, t], hlp[b, t], live, where)
            worst, near = max(worst, w), near + nt
            new = [seqs[hpar[b, t, s]] + ((int(htok[b, t, s]),) if htok[b, t, s] != blank else ()) for s in range(live)]
            merges += bool(merge and live < min(W, len(seqs) * V))
            todo = sorted(set(s for s in new if s not in cache))
            if todo:
                prev = [cache[s[:-1]] for s in todo]
                hx, mg, h2, c2_ = step(torch.tensor([s[-1] for s in todo], device="cuda"),
                                       torch.stack([p[2] for p in prev], 1), torch.stack([p[3] for p in prev], 1))
                for i, s in enumerate(todo):
                    cache[s] = (hx[i], mg[i], h2[:, i], c2_[:, i])
            seqs, lps = new, hlp[b, t, :live]
        best = int(np.argmax(lps))
        assert [int(k) for k in ids[b] if k >= 0] == list(seqs[best]), ("utterance %d result" % b)
        assert float(nlp[b]) == -float(lps[best])
        for s, sq in enumerate(seqs):              # the device's predictor output of the final beam vs the budget
            e = ((dec_final[b * W + s] - cache[sq][0]).abs() / (2.0 ** -16 * cache[sq][1])).max().item()
            pred_worst = max(pred_worst, e)
    print("W=%d merge=%s: worst err/bar %.3f, predictor err/budget %.3f, %d frames with a near-tie, %d frames "
          "merged, %d predictor states" % (W, merge, worst, pred_worst, near, merges, len(cache)))
    assert pred_worst <= 1.0
    assert len(cache) > 1 and (merges > 0 or not merge)


def _engine_run(m, h_enc, frames, W, merge=True):
    from edgedict_b200.stream_engine import BeamEngine
    eng = BeamEngine(m, h_enc.shape[0], h_enc.shape[1], W, merge=merge)
    ids, nlp = eng.run(h_enc, frames)
    return eng, [[int(k) for k in r if k >= 0] for r in ids.cpu().numpy()], nlp.clone()


SMALL = dict(vocab_embed_size=32, vocab_size=96, input_size=40, enc_hidden_size=64, enc_layers=2, enc_dropout=0.0,
             enc_proj_size=80, dec_hidden_size=64, dec_layers=2, dec_dropout=0.0, dec_proj_size=72, joint_size=88)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 4, 6])
def test_beam_batch_invariance_bitwise(W):
    """Each utterance decoded alone (its own T' = its length) gives the ids and the -log p bits it gets inside a
    batch of 5 of different lengths: rows never interact, and a row's 3xTF32 sums do not depend on its tile."""
    m = _scaled_model(SMALL, seed=4)
    g = torch.Generator().manual_seed(2)
    T = 37
    h_enc = torch.randn(5, T, SMALL["enc_proj_size"], generator=g).cuda()
    lens = [37, 20, 1, 33, 9]
    _, ids, nlp = _engine_run(m, h_enc, torch.tensor(lens, dtype=torch.int32).cuda(), W)
    for b, n in enumerate(lens):
        _, ids1, nlp1 = _engine_run(m, h_enc[b:b + 1, :n].contiguous(), torch.tensor([n], dtype=torch.int32).cuda(), W)
        assert ids1[0] == ids[b], b
        assert nlp1.view(torch.int32).item() == nlp[b:b + 1].view(torch.int32).item(), b
    print("W=%d: %d symbols, -logp %s" % (W, sum(map(len, ids)), nlp.cpu().numpy()))
    assert sum(map(len, ids)) > 0


@pytest.mark.gpu
def test_beam_repeatable_bitwise():
    m = _scaled_model(SMALL, seed=5)
    g = torch.Generator().manual_seed(3)
    h_enc = torch.randn(6, 29, SMALL["enc_proj_size"], generator=g).cuda()
    frames = torch.tensor([29, 3, 17, 29, 0, 11], dtype=torch.int32).cuda()
    eng, ids, nlp = _engine_run(m, h_enc, frames, 8)
    hist = eng.hist.clone()
    ids2, nlp2 = eng.run(h_enc, frames)
    assert torch.equal(hist, eng.hist)
    assert [[int(k) for k in r if k >= 0] for r in ids2.cpu().numpy()] == ids
    assert torch.equal(nlp.view(torch.int32), nlp2.view(torch.int32))
    assert ids[4] == [] and float(nlp[4]) == 0.0                       # no frame: the empty hypothesis, log p = 0
    print("ids lengths %s, merges in %d frames" % ([len(s) for s in ids], int((eng.hist_live < 8).sum())))


def test_beam_width_checked_before_any_device_work():
    """W < 1 is rejected before the encoder runs: a CPU model gets the ValueError, not a device error."""
    from edgedict_b200.rnnt.models import Transducer
    m = Transducer(output_loss=False, **SMALL)
    xs = torch.zeros(1, 4, SMALL["input_size"])
    for W in (0, -3):
        with pytest.raises(ValueError):
            m.beam_search(xs, None, W=W)


@pytest.mark.gpu
def test_beam_engine_rebuilt_after_parameters_move():
    m, z, sd = _tiny()
    xs = torch.as_tensor(z["xs"]).cuda()
    a, alp = m.beam_search(xs, None, W=4)
    eng = next(iter(m._beam_engines.values()))
    with torch.no_grad():
        for p in m.parameters():
            p.data = p.data.clone()                  # same values, new storage (what FlatAdam's bucketing does)
    b, blp = m.beam_search(xs, None, W=4)
    assert next(iter(m._beam_engines.values())) is not eng
    assert a == b and torch.equal(alp, blp)
    with torch.no_grad():
        for p in m.parameters():
            p.data = p.data.clone() * 0.5
    c, _ = m.beam_search(xs, None, W=4)
    from oracle import model_torch as mt
    want, _ = mt.beam_search({k: v.detach().cpu() for k, v in m.state_dict().items()}, xs.cpu(), None, W=4)
    assert c == want
