"""CPU restatement of the CTC prefix beam search of CTCEncoder.beam_search / edgedict_b200.ctc.beam_search (decode.cu,
CTC_BEAM), in fp64 or fp32, with the LM through tests/lm_oracle.py's lm_step / fusion_term, and a brute-force
enumeration of prefixes for tiny problems.  The oracle of tests/test_ctc_beam_host.py and tests/test_gpu_ctc_beam.py."""
import itertools

import numpy as np
import torch

from tests.lm_oracle import fusion_term, lm_prime, lm_step


def logadd(a, b):
    """The kernel's log-add, elementwise: m + log1p(exp(-|a - b|)) with m = max(a, b), and -inf when m is -inf."""
    a, b = np.asarray(a), np.asarray(b)
    m = np.maximum(a, b)
    with np.errstate(invalid="ignore", over="ignore"):
        r = m + np.log1p(np.exp(-np.abs(a - b)))
    return np.where(m == -np.inf, m, r).astype(np.result_type(a, b))


def prefix_beam_search(y, n, W, blank=0, dtype=np.float64, lm_sd=None, lm_weight=0.0, length_bonus=0.0, lm_bos=1,
                       lm_map=None):
    """One utterance: y [T, V] log-probs, its first n frames.  Returns (prefix tuple, -score, final beam, merges per
    frame): the final beam is [(prefix, pb, pnb, f)] in slot order.  ``dtype`` is the arithmetic (with an LM the LM's
    weights' dtype is the LM's arithmetic)."""
    y = np.asarray(y, dtype=dtype)
    V = y.shape[1]
    ninf = dtype(-np.inf)
    hyps = [dict(seq=(), pb=dtype(0.0), pnb=ninf, f=dtype(0.0))]
    if lm_sd is not None:
        llp, (lh, lc) = lm_prime(lm_sd, lm_bos)
        hyps[0].update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
        tmap = torch.arange(V) if lm_map is None else torch.as_tensor(lm_map).long()
    merges = []
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
        nmerge = 0
        for q, h in enumerate(hyps):
            e = h["seq"][-1] if h["seq"] else -1
            pb2 = A[q] + yt[blank]
            pnb2 = h["pnb"] + yt[e] if e >= 0 else ninf
            par = index.get(h["seq"][:-1]) if h["seq"] else None
            if par is not None:
                pnb2 = logadd(pnb2, pnbx[par, e])
                valid[par, e] = False
                nmerge += 1
            stay.append((dtype(pb2), dtype(pnb2)))
            vals[q, blank] = logadd(pb2, pnb2) + h["f"]
        merges.append(nmerge)
        flat = np.arange(nq * V)
        v = vals.reshape(-1)
        ok = valid.reshape(-1)
        flat, v = flat[ok], v[ok]
        v = np.where(v == 0, dtype(0.0), v)                     # -0 ranks with +0, as order_key does
        order = np.lexsort((flat, -v))[:W]
        new = []
        for i in order:
            q, k = divmod(int(flat[i]), V)
            h = hyps[q]
            if k == blank:
                nh = dict(h, pb=stay[q][0], pnb=stay[q][1])
            else:
                nh = dict(h, seq=h["seq"] + (k,), pb=ninf, pnb=pnbx[q, k], f=fx[q, k])
                if lm_sd is not None and int(tmap[k]) >= 0:
                    llp, (lh, lc) = lm_step(lm_sd, tmap[k:k + 1], (h["lh"][:, None], h["lc"][:, None]))
                    nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
            nh["val"] = vals[q, k]
            new.append(nh)
        hyps = new
    tot = [logadd(h["pb"], h["pnb"]) + h["f"] for h in hyps]
    best = max(range(len(hyps)), key=lambda j: (tot[j], -j))
    beam = [(h["seq"], float(h["pb"]), float(h["pnb"]), float(h["f"])) for h in hyps]
    return hyps[best]["seq"], -float(tot[best]), beam, merges


def batch_search(lp, lengths, W, blank=0, **kw):
    """prefix_beam_search over a batch lp [B, T, V] -> (list of int64 arrays, -score [B] float64, merges per
    utterance)."""
    ids, sc, mg = [], [], []
    for b in range(lp.shape[0]):
        seq, s, _, m = prefix_beam_search(np.asarray(lp[b]), int(lengths[b]), W, blank, **kw)
        ids.append(np.array(seq, dtype=np.int64))
        sc.append(s)
        mg.append(m)
    return ids, np.array(sc), mg


def prefix_logprob(y, prefix, blank=0):
    """log P(prefix | y) in fp64: the CTC forward algorithm over the extended label sequence."""
    y = np.asarray(y, dtype=np.float64)
    ext = [blank]
    for c in prefix:
        ext += [c, blank]
    S = len(ext)
    a = np.full(S, -np.inf)
    a[0] = y[0, blank]
    if S > 1:
        a[1] = y[0, ext[1]]
    for t in range(1, y.shape[0]):
        b = a.copy()
        b[1:] = np.logaddexp(b[1:], a[:-1])
        for s in range(2, S):
            if ext[s] != blank and ext[s] != ext[s - 2]:
                b[s] = np.logaddexp(b[s], a[s - 2])
        a = b + y[t, ext]
    return np.logaddexp(a[-1], a[-2]) if S > 1 else a[-1]


def all_prefixes(V, T, blank=0):
    """Every prefix of at most T non-blank tokens."""
    syms = [k for k in range(V) if k != blank]
    return [p for L in range(T + 1) for p in itertools.product(syms, repeat=L)]
