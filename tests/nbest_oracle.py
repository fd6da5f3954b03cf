"""CPU restatement of the N-best beam searches (``beam_search(nbest=N)``): the whole final beam of the transducer beam
(any max_symbols K, merge, LM fusion) and of the CTC prefix beam, ranked as BEAM_FINAL ranks it (value descending,
lowest slot on ties), with the encoder frame at which each token entered each hypothesis.  Also the brute-force sums
the exact-search tests compare against.

The transducer frames come from tests/beam_multi_symbol_oracle.py's ``frame``: every hypothesis it returns is a copy
of its parent's dict, so a frame list carried in the dict is the parent's, and the tokens a hypothesis gained during
frame t are exactly those past the end of that list.  The CTC search carries the frames itself; its arithmetic is
tests/ctc_beam_oracle.py's prefix_beam_search, statement for statement."""
import itertools

import numpy as np
import torch
import torch.nn.functional as F

from oracle import model_torch as mt
from tests import beam_multi_symbol_oracle as bo
from tests.ctc_beam_oracle import logadd
from tests.lm_oracle import fusion_term, lm_prime, lm_step


def ranked(values):
    """Slot indices ordered by value descending, lowest slot on ties (-0 ties with +0, as in a float compare)."""
    return sorted(range(len(values)), key=lambda i: (-float(values[i]), i))


@torch.no_grad()
def transducer_nbest(sd, h_enc, frames, W, K=1, merge=True, blank=mt.NUL, lm_sd=None, lm_weight=0.0,
                     length_bonus=0.0, lm_bos=1, lm_map=None):
    """h_enc [B, T', E], frames: the encoder frames each utterance decodes -> per utterance the ranked final beam,
    [(tokens tuple, frames tuple, nlogp float)]."""
    out = []
    for b in range(h_enc.shape[0]):
        hyps = [dict(bo.start(sd, lm_sd, lm_bos), fr=[])]
        for t in range(int(frames[b])):
            hyps = bo.frame(sd, hyps, h_enc[b, t], W, K, merge, blank, lm_sd, lm_weight, length_bonus, lm_map)
            hyps = [dict(h, fr=h["fr"] + [t] * (len(h["seq"]) - len(h["fr"]))) for h in hyps]
        lps = [float(h["lp"]) for h in hyps]
        out.append([(tuple(hyps[i]["seq"]), tuple(hyps[i]["fr"]), -lps[i]) for i in ranked(lps)])
    return out


def ctc_nbest(y, n, W, blank=0, dtype=np.float32, lm_sd=None, lm_weight=0.0, length_bonus=0.0, lm_bos=1,
              lm_map=None):
    """One utterance: y [T, V] log-probs, its first n frames -> the ranked final beam [(prefix tuple, frames tuple,
    -score)], score = (pb (+) pnb) + f.  A prefix's last token has the frame of the extension that created it; a
    stay (merged extensions included) keeps the frames."""
    y = np.asarray(y, dtype=dtype)
    V = y.shape[1]
    ninf = dtype(-np.inf)
    hyps = [dict(seq=(), fr=(), pb=dtype(0.0), pnb=ninf, f=dtype(0.0))]
    if lm_sd is not None:
        llp, (lh, lc) = lm_prime(lm_sd, lm_bos)
        hyps[0].update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
        tmap = torch.arange(V) if lm_map is None else torch.as_tensor(lm_map).long()
    k_all = np.arange(V)
    for t in range(n):
        yt = y[t]
        index = {h["seq"]: q for q, h in enumerate(hyps)}
        nq = len(hyps)
        vals = np.empty((nq, V), dtype=dtype)
        pnbx = np.empty((nq, V), dtype=dtype)
        fx = np.empty((nq, V), dtype=dtype)
        valid = np.ones((nq, V), dtype=bool)
        A = [logadd(h["pb"], h["pnb"]) for h in hyps]
        for q, h in enumerate(hyps):
            e = h["seq"][-1] if h["seq"] else -1
            pnbx[q] = np.where(k_all == e, h["pb"], A[q]) + yt
            if lm_sd is not None:
                fz = fusion_term(h["llp"].to(torch.float64 if dtype == np.float64 else torch.float32), V, blank,
                                 lm_weight, length_bonus, lm_map).numpy().astype(dtype)
                fx[q] = h["f"] + fz
            else:
                fx[q] = h["f"]
            vals[q] = pnbx[q] + fx[q]
        stay = []
        for q, h in enumerate(hyps):
            e = h["seq"][-1] if h["seq"] else -1
            pb2 = A[q] + yt[blank]
            pnb2 = h["pnb"] + yt[e] if e >= 0 else ninf
            par = index.get(h["seq"][:-1]) if h["seq"] else None
            if par is not None:
                pnb2 = logadd(pnb2, pnbx[par, e])
                valid[par, e] = False
            stay.append((dtype(pb2), dtype(pnb2)))
            vals[q, blank] = logadd(pb2, pnb2) + h["f"]
        flat = np.arange(nq * V)
        v = vals.reshape(-1)
        ok = valid.reshape(-1)
        flat, v = flat[ok], v[ok]
        v = np.where(v == 0, dtype(0.0), v)
        order = np.lexsort((flat, -v))[:W]
        new = []
        for i in order:
            q, k = divmod(int(flat[i]), V)
            h = hyps[q]
            if k == blank:
                nh = dict(h, pb=stay[q][0], pnb=stay[q][1])
            else:
                nh = dict(h, seq=h["seq"] + (k,), fr=h["fr"] + (t,), pb=ninf, pnb=pnbx[q, k], f=fx[q, k])
                if lm_sd is not None and int(tmap[k]) >= 0:
                    llp, (lh, lc) = lm_step(lm_sd, tmap[k:k + 1], (h["lh"][:, None], h["lc"][:, None]))
                    nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
            new.append(nh)
        hyps = new
    tot = [logadd(h["pb"], h["pnb"]) + h["f"] for h in hyps]
    return [(hyps[i]["seq"], hyps[i]["fr"], -float(tot[i])) for i in ranked(tot)]


def ctc_batch_nbest(lp, lengths, W, blank=0, **kw):
    """ctc_nbest over a batch lp [B, T, V]."""
    return [ctc_nbest(np.asarray(lp[b]), int(lengths[b]), W, blank, **kw) for b in range(lp.shape[0])]


# ---- brute force: every path of a tiny problem -----------------------------------------------------------------------
def ctc_path_logprob(y, tokens, frames, blank=0):
    """fp64 log p of the CTC paths that emit ``tokens`` with token i first emitted at frames[i] (its run of repeats may
    go on; a blank or another token ends it), over the frames of y [n, V]."""
    y = np.asarray(y, dtype=np.float64)
    n = y.shape[0]
    # state per frame: (index of the last token entered, whether the path still repeats it); -1 before any token
    alpha = {(-1, False): 0.0}
    for t in range(n):
        nxt = {}
        for (i, rep), a in alpha.items():
            opts = []
            if i + 1 < len(tokens) and frames[i + 1] == t:
                if not (rep and tokens[i + 1] == tokens[i]):         # a repeat enters only after a blank
                    opts = [((i + 1, True), y[t, tokens[i + 1]])]
            else:
                opts = [((i, False), y[t, blank])]
                if rep:
                    opts.append(((i, True), y[t, tokens[i]]))
            for s, v in opts:
                nxt[s] = np.logaddexp(nxt.get(s, -np.inf), a + v)
        alpha = nxt
    return float(np.logaddexp.reduce([a for (i, _), a in alpha.items() if i == len(tokens) - 1] or [-np.inf]))


def transducer_sequence_logprob(sd64, h_enc, n, tokens, blank=mt.NUL):
    """fp64 log of the sum over every alignment with at most one symbol per frame (a frame emits one token or blank)
    of ``tokens`` over the first n frames of h_enc [T', E] (fp64 state dict sd64)."""
    U = len(tokens)
    if U > n:
        return -np.inf
    ys = torch.tensor([list(tokens)], dtype=torch.long)
    d, _ = mt.decoder(sd64, ys, None)                        # [1, U + 1, D]: the predictor after 0 .. U tokens
    z = mt.joint(sd64, h_enc[:n, None, :].expand(n, U + 1, -1).reshape(-1, h_enc.shape[1]),
                 d[0][None].expand(n, U + 1, -1).reshape(-1, d.shape[2]))
    lp = F.log_softmax(z.double(), -1).view(n, U + 1, -1)
    a = torch.full((U + 1,), -np.inf, dtype=torch.float64)
    a[0] = 0.0
    for t in range(n):
        b = a + lp[t, :, blank]
        if U:
            emit = a[:-1] + lp[t, torch.arange(U), ys[0]]
            b[1:] = torch.logaddexp(b[1:], emit)
        a = b
    return float(a[U])


def transducer_path_logprob(sd64, h_enc, n, tokens, frames, K=1, blank=mt.NUL):
    """fp64 log p of one path of the K-symbol lattice over the first n frames of h_enc [T', E]: at frame t the tokens
    whose frame is t in order, then blank unless K tokens were emitted."""
    ys = torch.tensor([list(tokens)], dtype=torch.long)
    d, _ = mt.decoder(sd64, ys, None)
    total, u = 0.0, 0
    for t in range(n):
        j = 0
        while u < len(tokens) and frames[u] == t:
            lp = F.log_softmax(mt.joint(sd64, h_enc[t][None], d[0, u][None])[0].double(), 0)
            total += float(lp[tokens[u]])
            u += 1
            j += 1
        if j < K:
            lp = F.log_softmax(mt.joint(sd64, h_enc[t][None], d[0, u][None])[0].double(), 0)
            total += float(lp[blank])
    assert u == len(tokens)
    return total


def all_sequences(V, n, blank=0):
    """Every token sequence of at most n non-blank tokens."""
    syms = [k for k in range(V) if k != blank]
    return [p for L in range(n + 1) for p in itertools.product(syms, repeat=L)]
