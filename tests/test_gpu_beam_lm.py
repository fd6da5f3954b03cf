"""Beam search with shallow fusion of an LSTM language model on the device (Transducer.beam_search(lm=...),
stream_engine.BeamEngine, BEAM_SELECT flag 32 of csrc/decode.cu): against the CPU restatement (tests/lm_oracle.py),
bitwise against lm=None at zero weights, frame by frame against fp64, batch invariance, repeatability, the two forms
of the LM and the engine cache."""
import numpy as np
import pytest
import torch

from tests import lm_oracle as lo
from tests.test_gpu_beam_engine import LARGE, SMALL, U32, _check_frame, _dec64, _scaled_model, _tiny
from tests.test_oracle_lm import load_lm


def _perm_map(V, ntok):
    """A permutation of the LM's tokens with two tokens the LM does not score."""
    m = (torch.arange(V) * 5 + 3) % ntok
    m[2] = m[7] = -1
    return m


def _lm_module(ntok, ninp, nhid, L, scale, seed):
    """An LMModel-shaped module (reference models.py:224-261), weights x ``scale`` so that the LM term matters."""
    torch.manual_seed(seed)
    lm = torch.nn.Module()
    lm.encoder = torch.nn.Embedding(ntok, ninp)
    lm.rnn = torch.nn.LSTM(ninp, nhid, L, batch_first=True)
    lm.decoder = torch.nn.Linear(nhid, ntok)
    with torch.no_grad():
        for p in lm.parameters():
            p.mul_(scale)
    return lm.eval()


@pytest.mark.gpu
@pytest.mark.parametrize("mapped", [False, True])
@pytest.mark.parametrize("lm_weight,length_bonus", [(0.3, 0.0), (0.3, 0.5), (1.0, 0.0), (1.0, 0.5)])
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 4, 20])
def test_fused_beam_matches_restatement(W, merge, lm_weight, length_bonus, mapped):
    """The tiny transducer and the tiny fixture LM (16 tokens each), ragged batch of three.  W = 1 is fused greedy;
    W = 20 > V exercises the short first frame."""
    m, z, sd = _tiny()
    _, lsd = load_lm()
    xs, xlen = torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"])
    V = sd["joint.joint.2.weight"].shape[0]
    tmap = _perm_map(V, lsd["encoder.weight"].shape[0]) if mapped else None
    kw = dict(lm_weight=lm_weight, length_bonus=length_bonus)
    want, wlp = lo.beam_search(sd, xs, xlen, W=W, merge=merge, lm_sd=lsd, lm_map=tmap, **kw)
    got, glp = m.beam_search(xs.cuda(), xlen, W=W, merge=merge, lm=lsd, lm_token_map=tmap, **kw)
    plain, _ = m.beam_search(xs.cuda(), xlen, W=W, merge=merge)
    err = float(np.max(np.abs(glp.cpu().numpy() - wlp.numpy()) / np.abs(wlp.numpy())))
    print("W=%d merge=%s lm_weight=%g bonus=%g map=%s: ids %s (without LM %s), -logp %s, max rel err %.2e"
          % (W, merge, lm_weight, length_bonus, mapped, got, plain, glp.cpu().numpy(), err))
    assert got == want
    assert err < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("W", [1, 4, 8])
def test_zero_weights_are_bitwise_the_plain_beam(W, merge):
    """lm_weight = length_bonus = 0 runs the whole LM path (priming, gathers, masked steps, logits, statistics) and
    must give the ids and the -log p bits of lm=None, with the identity map and with a map."""
    m = _scaled_model(SMALL, seed=4)
    g = torch.Generator().manual_seed(2)
    xs = torch.randn(5, 60, SMALL["input_size"], generator=g).cuda()
    xlen = torch.tensor([60, 41, 7, 52, 30])
    plain, plp = m.beam_search(xs, xlen, W=W, merge=merge)
    lm = _lm_module(96, 16, 48, 2, 4.0, seed=1).cuda()
    fused, flp = m.beam_search(xs, xlen, W=W, merge=merge, lm=lm)
    assert fused == plain and torch.equal(flp.view(torch.int32), plp.view(torch.int32))
    lm50 = _lm_module(50, 16, 48, 1, 4.0, seed=2)
    fused, flp = m.beam_search(xs, xlen, W=W, merge=merge, lm=lm50.state_dict(), lm_token_map=_perm_map(96, 50))
    assert fused == plain and torch.equal(flp.view(torch.int32), plp.view(torch.int32))
    moved, _ = m.beam_search(xs, xlen, W=W, merge=merge, lm=lm, lm_weight=1.0, length_bonus=0.5)
    print("W=%d merge=%s: %d symbols without LM, %d with lm_weight 1 / bonus 0.5"
          % (W, merge, sum(map(len, plain)), sum(map(len, moved))))
    assert sum(map(len, plain)) > 0


def _lm64(lsd64):
    L = (len(lsd64) - 3) // 4
    emb, wd, bd = lsd64["encoder.weight"], lsd64["decoder.weight"], lsd64["decoder.bias"]

    def step(tok, h, c):
        """One fp64 LM step for tokens [n] from (h, c) [L, n, H] -> (logits, |W_d||h| + |b_d|, h, c)."""
        x, hs, cs = emb[tok], [], []
        for k in range(L):
            g = x @ lsd64["rnn.weight_ih_l%d" % k].t() + lsd64["rnn.bias_ih_l%d" % k] + \
                h[k] @ lsd64["rnn.weight_hh_l%d" % k].t() + lsd64["rnn.bias_hh_l%d" % k]
            i, f, gg, o = g.chunk(4, 1)
            ck = f.sigmoid() * c[k] + i.sigmoid() * gg.tanh()
            x = o.sigmoid() * ck.tanh()
            hs.append(x)
            cs.append(ck)
        return x @ wd.t() + bd, x.abs() @ wd.abs().t() + bd.abs(), torch.stack(hs), torch.stack(cs)
    return step, L


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_fused_beam_teacher_forced_fp64(W):
    """Every frame of the fused device beam against fp64, from the device's own beam at t-1 (its sequences from the
    history, its fp32 slot values).  E6D2_LARGE dims as in test_gpu_beam_engine.test_beam_teacher_forced_fp64 (frames
    presented twice, sharpened output layer, raised blank bias) and an LM of cli/train_lm.py's shape
    LMModel(1024, 64, 1024, 2), weights x 3, lm_weight 0.5 and length_bonus 3 (about what offsets the LM's mean
    log-prob, so that both blank and symbols survive).

    The fp64 value of candidate (q, k) is (a + f) + logp[q] with the LM log-probs of slot q recomputed in fp64 from
    its token sequence.  Its bar is the acoustic bar of the plain test plus |lm_weight| times the LM log-prob bar:
    - LM logits l (3xTF32 LSTM chain and LINEAR, as the predictor): |dl_i| <= 2^-16 (|W_d||h| + |b_d|)_i, a budget
      checked against the device's LM logits of the final beam;
    - fp32 log-softmax over ntoken: max dl + ntoken u for the statistics, 3 u (|l - max| + |lse|) for the roundings;
    - and 3 u (|a| + |f|) for forming (a + f)."""
    from edgedict_b200.rnnt.tokenizer import BOS
    from edgedict_b200.stream_engine import BeamEngine
    m = _scaled_model(LARGE, seed=10)
    B, blank, lm_weight, bonus = 4, m.blank, 0.5, 3.0
    lm = _lm_module(1024, 64, 1024, 2, 3.0, seed=11).cuda()
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
    eng = BeamEngine(m, B, T, W, lm=lm, lm_weight=lm_weight, length_bonus=bonus)
    ids, nlp = eng.run(h_enc, frames.cuda())
    torch.cuda.synchronize()
    hpar, htok = eng.hist_parent.cpu().numpy(), eng.hist_token.cpu().numpy()
    hlp, hlive = eng.hist_logp.cpu().numpy().astype(np.float64), eng.hist_live.cpu().numpy()
    ids, dec_final, lm_final = ids.cpu().numpy(), eng.dec_x[T & 1].double(), eng.lm_logits.double()

    sd64 = {k: v.detach().double() for k, v in m.state_dict().items()}
    lsd64 = {k: v.detach().double() for k, v in lm.state_dict().items()}
    Ld, Hd = m.decoder.lstm.num_layers, m.decoder.lstm.hidden_size
    w1, b1 = sd64["joint.joint.0.weight"], sd64["joint.joint.0.bias"]
    w2, b2 = sd64["joint.joint.2.weight"], sd64["joint.joint.2.bias"]
    J, V, E = w1.shape[0], w2.shape[0], h_enc.shape[2]
    D = w1.shape[1] - E
    c1, c2 = U32 * (np.sqrt((E + D + 1) / 2) + 4), U32 * (np.sqrt((J + 1) / 2) + 4)
    rss = lambda x, w: (x * x) @ (w * w).t()
    step = _dec64(sd64, Ld)
    lstep, Ll = _lm64(lsd64)
    Hl = lsd64["rnn.weight_hh_l0"].shape[1]
    zs, zl = (torch.zeros(n, 1, h, dtype=torch.float64, device="cuda") for n, h in ((Ld, Hd), (Ll, Hl)))
    x0, mag0, hh, cc = step(torch.tensor([BOS], device="cuda"), zs, zs)
    l0, lmag0, lh0, lc0 = lstep(torch.tensor([1], device="cuda"), zl, zl)
    cache = {(): (x0[0], mag0[0], hh[:, 0], cc[:, 0])}
    lcache = {(): (l0[0], lmag0[0], lh0[:, 0], lc0[:, 0])}
    he64 = h_enc.double()
    worst, near, merges, pred_worst, lm_worst, lm_moves = 0.0, 0, 0, 0.0, 0.0, 0
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
            a = zz - lse
            beta = 6 * (dz + dz.max(1, keepdim=True).values) + V * U32 + \
                3 * U32 * ((zz - zmax).abs() + lse.abs() + lpq.abs())
            # the LM term (identity map: the LM's sequence is the slot's token sequence)
            ll = torch.stack([lcache[s][0] for s in seqs])
            dl = 2.0 ** -16 * torch.stack([lcache[s][1] for s in seqs])
            llse = torch.logsumexp(ll, 1, keepdim=True)
            lmlp = ll - llse
            lbar = dl + dl.max(1, keepdim=True).values + ll.shape[1] * U32 + \
                3 * U32 * ((ll - ll.max(1, keepdim=True).values).abs() + llse.abs())
            f = lm_weight * lmlp + bonus
            f[:, blank] = 0.0
            fbar = abs(lm_weight) * lbar
            fbar[:, blank] = 0.0
            v = (a + f) + lpq
            beta = beta + fbar + 3 * U32 * (a.abs() + f.abs())
            lm_moves += int(((a + lpq).argmax(1) != v.argmax(1)).sum())
            w, nt = _check_frame(v.cpu().numpy(), beta.cpu().numpy(), seqs, W, True, blank, hpar[b, t],
                                 htok[b, t], hlp[b, t], live, where)
            worst, near = max(worst, w), near + nt
            new = [seqs[hpar[b, t, s]] + ((int(htok[b, t, s]),) if htok[b, t, s] != blank else ()) for s in range(live)]
            merges += bool(live < min(W, len(seqs) * V))
            todo = sorted(set(s for s in new if s not in cache))
            if todo:
                prev, lprev = [cache[s[:-1]] for s in todo], [lcache[s[:-1]] for s in todo]
                tk = torch.tensor([s[-1] for s in todo], device="cuda")
                hx, mg, h2, c2_ = step(tk, torch.stack([p[2] for p in prev], 1), torch.stack([p[3] for p in prev], 1))
                lx, lmg, lh2, lc2 = lstep(tk, torch.stack([p[2] for p in lprev], 1),
                                          torch.stack([p[3] for p in lprev], 1))
                for i, s in enumerate(todo):
                    cache[s] = (hx[i], mg[i], h2[:, i], c2_[:, i])
                    lcache[s] = (lx[i], lmg[i], lh2[:, i], lc2[:, i])
            seqs, lps = new, hlp[b, t, :live]
        best = int(np.argmax(lps))
        assert [int(k) for k in ids[b] if k >= 0] == list(seqs[best]), ("utterance %d result" % b)
        assert float(nlp[b]) == -float(lps[best])
        for s, sq in enumerate(seqs):              # the device's predictor output and LM logits of the final beam
            e = ((dec_final[b * W + s] - cache[sq][0]).abs() / (2.0 ** -16 * cache[sq][1])).max().item()
            pred_worst = max(pred_worst, e)
            e = ((lm_final[b * W + s] - lcache[sq][0]).abs() / (2.0 ** -16 * lcache[sq][1])).max().item()
            lm_worst = max(lm_worst, e)
    print("W=%d: worst err/bar %.3f, predictor err/budget %.3f, LM logits err/budget %.3f, %d frames with a "
          "near-tie, %d frames merged, %d states, %d rows whose best candidate the LM changed"
          % (W, worst, pred_worst, lm_worst, near, merges, len(cache), lm_moves))
    assert pred_worst <= 1.0 and lm_worst <= 1.0
    assert len(cache) > 1 and merges > 0 and lm_moves > 0


def _run(m, h_enc, frames, W, **kw):
    from edgedict_b200.stream_engine import BeamEngine
    eng = BeamEngine(m, h_enc.shape[0], h_enc.shape[1], W, **kw)
    ids, nlp = eng.run(h_enc, frames)
    return eng, [[int(k) for k in r if k >= 0] for r in ids.cpu().numpy()], nlp.clone()


FUSE = dict(lm_weight=0.7, length_bonus=0.3)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 4, 6])
def test_fused_beam_batch_invariance_bitwise(W):
    m = _scaled_model(SMALL, seed=4)
    lm = _lm_module(96, 16, 48, 2, 4.0, seed=3).cuda()
    g = torch.Generator().manual_seed(2)
    T = 37
    h_enc = torch.randn(5, T, SMALL["enc_proj_size"], generator=g).cuda()
    lens = [37, 20, 1, 33, 9]
    _, ids, nlp = _run(m, h_enc, torch.tensor(lens, dtype=torch.int32).cuda(), W, lm=lm, **FUSE)
    for b, n in enumerate(lens):
        _, ids1, nlp1 = _run(m, h_enc[b:b + 1, :n].contiguous(), torch.tensor([n], dtype=torch.int32).cuda(), W,
                             lm=lm, **FUSE)
        assert ids1[0] == ids[b], b
        assert nlp1.view(torch.int32).item() == nlp[b:b + 1].view(torch.int32).item(), b
    print("W=%d: %d symbols, -logp %s" % (W, sum(map(len, ids)), nlp.cpu().numpy()))
    assert sum(map(len, ids)) > 0


@pytest.mark.gpu
def test_fused_beam_repeatable_bitwise():
    m = _scaled_model(SMALL, seed=5)
    lm = _lm_module(96, 16, 48, 2, 4.0, seed=4).cuda()
    g = torch.Generator().manual_seed(3)
    h_enc = torch.randn(6, 29, SMALL["enc_proj_size"], generator=g).cuda()
    frames = torch.tensor([29, 3, 17, 29, 0, 11], dtype=torch.int32).cuda()
    eng, ids, nlp = _run(m, h_enc, frames, 8, lm=lm, **FUSE)
    hist, lml = eng.hist.clone(), eng.lm_logits.clone()
    ids2, nlp2 = eng.run(h_enc, frames)
    assert torch.equal(hist, eng.hist) and torch.equal(lml, eng.lm_logits)
    assert [[int(k) for k in r if k >= 0] for r in ids2.cpu().numpy()] == ids
    assert torch.equal(nlp.view(torch.int32), nlp2.view(torch.int32))
    assert ids[4] == [] and float(nlp[4]) == 0.0                       # no frame: the empty hypothesis, score 0


@pytest.mark.gpu
def test_module_and_state_dict_give_the_same_bits():
    """The module on the device (read in place), its state_dict on the host (copied into the engine), and a module
    with tied input / output embeddings (LMModel(tie_weights=True)) against its untied copy."""
    m = _scaled_model(SMALL, seed=6)
    g = torch.Generator().manual_seed(4)
    xs = torch.randn(3, 50, SMALL["input_size"], generator=g).cuda()
    lm = _lm_module(96, 24, 24, 2, 4.0, seed=5)
    sd_host = {k: v.clone() for k, v in lm.state_dict().items()}
    a, alp = m.beam_search(xs, None, W=4, lm=lm.cuda(), **FUSE)
    b, blp = m.beam_search(xs, None, W=4, lm=sd_host, **FUSE)
    assert a == b and torch.equal(alp.view(torch.int32), blp.view(torch.int32))
    lm.decoder.weight = lm.encoder.weight                             # tied, as LMModel(tie_weights=True)
    c, clp = m.beam_search(xs, None, W=4, lm=lm, **FUSE)
    untied = {k: v.detach().cpu().clone() for k, v in lm.state_dict().items()}
    d, dlp = m.beam_search(xs, None, W=4, lm=untied, **FUSE)
    assert c == d and torch.equal(clp.view(torch.int32), dlp.view(torch.int32))
    print("ids %s / tied %s" % (a, c))


@pytest.mark.gpu
def test_engine_rebuilt_after_lm_parameters_move():
    m, z, sd = _tiny()
    _, lsd = load_lm()
    lm = _lm_module(16, 6, 10, 2, 1.0, seed=0)
    lm.load_state_dict(lsd)
    lm.cuda()
    xs = torch.as_tensor(z["xs"]).cuda()
    a, alp = m.beam_search(xs, None, W=4, lm=lm, **FUSE)
    eng = next(iter(m._beam_engines.values()))
    m.beam_search(xs, None, W=4, lm=lm, **FUSE)
    assert next(iter(m._beam_engines.values())) is eng                # same LM, same engine
    with torch.no_grad():
        for p in lm.parameters():
            p.data = p.data.clone()                                   # same values, new storage
    b, blp = m.beam_search(xs, None, W=4, lm=lm, **FUSE)
    assert next(iter(m._beam_engines.values())) is not eng
    assert a == b and torch.equal(alp, blp)
    with torch.no_grad():
        for p in lm.parameters():
            p.data = p.data.clone() * 0.5
    c, clp = m.beam_search(xs, None, W=4, lm=lm, **FUSE)
    want, _ = lo.beam_search(sd, xs.cpu(), None, W=4, lm_sd={k: v.cpu() for k, v in lm.state_dict().items()}, **FUSE)
    assert c == want
    eng = next(iter(m._beam_engines.values()))
    m.beam_search(xs, None, W=4, lm=lm, lm_weight=0.2, length_bonus=0.3)
    assert next(iter(m._beam_engines.values())) is not eng           # the weights are part of the key
