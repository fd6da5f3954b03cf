"""CPU restatement of contextual biasing (edgedict_b200/context.py, decode.cu flag 2048).

- ``brute_step`` / ``banked``: the automaton's definition on token strings, by suffix matching over the phrase set,
  with no trie, no failure links and no tables;
- ``transducer_nbest`` / ``ctc_nbest``: tests/nbest_oracle.py's two searches with the bias term where the device adds
  it (transducer: f = f_LM + delta for k != blank, value (a + f) + logp; CTC: f' = (f + LM term) + delta) and the final
  ranking by value - pending[state]."""
import numpy as np
import torch

from oracle import model_torch as mt
from tests import beam_multi_symbol_oracle as bo
from tests.ctc_beam_oracle import logadd
from tests.lm_oracle import fusion_term, lm_prime, lm_step
from tests.nbest_oracle import ranked


def brute_step(phrases, string, k):
    """(next string, banked amount in tokens or 0) of appending k to the state string ``string``: u = the longest
    suffix of string + (k,) that is a prefix of some phrase; if a suffix of u is a phrase, the longest one c completes
    (|c| banked, next state empty), else the next state is u."""
    phrases = set(map(tuple, phrases))
    prefixes = {p[:i] for p in phrases for i in range(len(p) + 1)}
    x = tuple(string) + (k,)
    u = next(x[i:] for i in range(len(x) + 1) if x[i:] in prefixes)
    c = next((u[i:] for i in range(len(u)) if u[i:] in phrases), None)
    return ((), len(c)) if c is not None else (u, 0)


def brute_tables(phrases, V, beta, blank=0):
    """{(state string, k): (next string, delta)} for every trie node and non-blank k, by brute_step, delta in float32
    as the definition states it: (completes ? beta |c| : beta |u|) - beta |s|."""
    phrases = set(map(tuple, phrases))
    nodes = sorted({p[:i] for p in phrases for i in range(len(p) + 1)})
    b = np.float32(beta)
    out = {}
    for s in nodes:
        for k in range(V):
            if k == blank:
                continue
            u, c = brute_step(phrases, s, k)
            gain = b * np.float32(c) if c else b * np.float32(len(u))
            out[s, k] = (u, np.float32(gain - b * np.float32(len(s))))
    return out


def banked(phrases, seq, beta, blank=0):
    """fp64 bonus banked by the token sequence ``seq`` (blanks skipped): beta times the length of every completion."""
    s, tot = (), 0.0
    for k in seq:
        if k == blank:
            continue
        s, c = brute_step(phrases, s, k)
        tot += beta * c
    return tot


@torch.no_grad()
def transducer_nbest(sd, h_enc, frames, W, graph, K=1, merge=True, blank=mt.NUL, lm_sd=None, lm_weight=0.0,
                     length_bonus=0.0, lm_bos=1, lm_map=None):
    """tests/nbest_oracle.transducer_nbest with the bias term of ``graph`` (a ContextGraph; tests/
    beam_multi_symbol_oracle.frame's rounds, f = f_LM + delta): per utterance the final beam ranked by
    value - pending[state], [(tokens, frames, -(value - pending))]."""
    V = sd["joint.joint.2.weight"].shape[0]
    tmap = torch.arange(V) if lm_map is None else torch.as_tensor(lm_map).long()
    nxt, dlt, pend = graph.next, torch.from_numpy(graph.delta), graph.pending
    out = []
    for b in range(h_enc.shape[0]):
        hyps = [dict(bo.start(sd, lm_sd, lm_bos), fr=[], cs=0)]
        for t in range(int(frames[b])):
            hyps = [dict(h, open=True) for h in hyps]
            for j in range(K):
                if not any(h["open"] for h in hyps):
                    break
                last = j == K - 1
                cand = []
                for qi, hy in enumerate(hyps):
                    if not hy["open"]:
                        cand.append((float(hy["lp"]), qi, blank, hy["lp"]))
                        continue
                    a = torch.log_softmax(mt.joint(sd, h_enc[b, t][None], hy["x"][None])[0], 0)
                    d = dlt[hy["cs"]].clone()
                    d[blank] = 0.0
                    if lm_sd is not None:
                        f = fusion_term(hy["llp"].to(a.dtype), V, blank, lm_weight, length_bonus, lm_map) + d
                    else:
                        f = d
                    lp = (a + f) + hy["lp"]
                    cand += [(float(lp[k]), qi, k, lp[k]) for k in range(V)]
                cand.sort(key=lambda c: (-c[0], c[1], c[2]))
                new, seen = [], {}
                for _, qi, k, lpk in cand[:W]:
                    hy = hyps[qi]
                    emits = hy["open"] and k != blank
                    seq = hy["seq"] + [k] if emits else hy["seq"]
                    key = (tuple(seq), emits and not last)
                    if merge and key in seen:
                        seen[key]["lp"] = torch.logaddexp(seen[key]["lp"], lpk)
                        continue
                    nh = dict(hy, seq=seq, lp=lpk, open=emits and not last)
                    if emits:
                        nx, (h2, c2) = mt.decoder(sd, torch.full((1, 1), k), (hy["h"][:, None], hy["c"][:, None]))
                        nh.update(x=nx[0, 0], h=h2[:, 0], c=c2[:, 0], cs=int(nxt[hy["cs"], k]))
                        if lm_sd is not None and int(tmap[k]) >= 0:
                            llp, (lh, lc) = lm_step(lm_sd, tmap[k:k + 1], (hy["lh"][:, None], hy["lc"][:, None]))
                            nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
                    seen[key] = nh
                    new.append(nh)
                hyps = new
            hyps = [dict(h, open=False, fr=h["fr"] + [t] * (len(h["seq"]) - len(h["fr"]))) for h in hyps]
        vals = [np.float32(float(h["lp"])) - pend[h["cs"]] for h in hyps]
        out.append([(tuple(hyps[i]["seq"]), tuple(hyps[i]["fr"]), -float(vals[i])) for i in ranked(vals)])
    return out


def ctc_nbest(y, n, W, graph, blank=0, dtype=np.float32, lm_sd=None, lm_weight=0.0, length_bonus=0.0, lm_bos=1,
              lm_map=None):
    """tests/nbest_oracle.ctc_nbest with the bias term of ``graph``: f' = (f + LM term) + delta for an extension, the
    final ranking by (pb (+) pnb) + f - pending[state] -> [(prefix, frames, -(that))]."""
    y = np.asarray(y, dtype=dtype)
    V = y.shape[1]
    ninf = dtype(-np.inf)
    nxt, dlt, pend = graph.next, graph.delta.astype(dtype), graph.pending.astype(dtype)
    hyps = [dict(seq=(), fr=(), pb=dtype(0.0), pnb=ninf, f=dtype(0.0), cs=0)]
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
                fx[q] = (h["f"] + fz) + dlt[h["cs"]]
            else:
                fx[q] = h["f"] + dlt[h["cs"]]
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
                nh = dict(h, seq=h["seq"] + (k,), fr=h["fr"] + (t,), pb=ninf, pnb=pnbx[q, k], f=fx[q, k],
                          cs=int(nxt[h["cs"], k]))
                if lm_sd is not None and int(tmap[k]) >= 0:
                    llp, (lh, lc) = lm_step(lm_sd, tmap[k:k + 1], (h["lh"][:, None], h["lc"][:, None]))
                    nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
            new.append(nh)
        hyps = new
    tot = [dtype(logadd(h["pb"], h["pnb"]) + h["f"]) - pend[h["cs"]] for h in hyps]
    return [(hyps[i]["seq"], hyps[i]["fr"], -float(tot[i])) for i in ranked(tot)]


def ctc_batch_nbest(lp, lengths, W, graph, blank=0, **kw):
    """ctc_nbest over a batch lp [B, T, V]."""
    return [ctc_nbest(np.asarray(lp[b]), int(lengths[b]), W, graph, blank, **kw) for b in range(lp.shape[0])]
