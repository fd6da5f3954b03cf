"""Host oracle for edgedict_b200.ngram: a small estimator that writes ARPA files (interpolated absolute discounting
with normalised backoff weights over seeded random token corpora), the backoff rule restated over the n-gram
dictionary with no CSR and no suffix links, and the CTC / transducer beam searches with the n-gram term (the
restatements of tests/context_oracle.py with f = (f0 + w g) + delta and the final value (y + w e) - pending)."""
import math

import numpy as np
import torch

from oracle import model_torch as mt
from tests import beam_multi_symbol_oracle as bo
from tests.ctc_beam_oracle import logadd
from tests.nbest_oracle import ranked

f32 = np.float32
LN10 = math.log(10.0)
BOS, EOS = "<s>", "</s>"


def corpus(seed, V, n_sent, max_len, blank=0, zipf=1.3):
    """Seeded sentences of token ids in [0, V) without blank, drawn from a Zipf-weighted Markov chain."""
    rng = np.random.default_rng(seed)
    toks = np.array([k for k in range(V) if k != blank])
    base = 1.0 / np.arange(1, len(toks) + 1) ** zipf
    trans = np.stack([np.roll(base, int(s)) for s in rng.integers(0, len(toks), size=len(toks))])
    trans /= trans.sum(1, keepdims=True)
    out = []
    for _ in range(n_sent):
        i = int(rng.integers(len(toks)))
        s = []
        for _ in range(int(rng.integers(1, max_len + 1))):
            s.append(int(toks[i]))
            i = int(rng.choice(len(toks), p=trans[i]))
        out.append(s)
    return out


def estimate(sentences, order, V, blank=0, D=0.5):
    """{m: {words tuple: (log10 p, log10 bo or None)}} of an interpolated absolute-discounting model of ``order`` over
    the tokens (decimal words) and </s>, <s> as history only.  Unigrams are add-one over every token and </s>, so the
    model sums to 1 over them in every history."""
    vocab = [str(k) for k in range(V) if k != blank] + [EOS]
    cnt = [dict() for _ in range(order + 1)]
    for s in sentences:
        w = [BOS] + [str(k) for k in s] + [EOS]
        for i in range(1, len(w)):
            for m in range(1, order + 1):
                if i - m + 1 < 0:
                    break
                g = tuple(w[i - m + 1:i + 1])
                cnt[m][g] = cnt[m].get(g, 0) + 1
    ctx = {}                                                  # history -> (total count, distinct continuations)
    for m in range(2, order + 1):
        for g, c in cnt[m].items():
            t, n = ctx.get(g[:-1], (0, 0))
            ctx[g[:-1]] = (t + c, n + 1)
    N1 = sum(c for g, c in cnt[1].items())
    uni = {(w,): (cnt[1].get((w,), 0) + 1) / (N1 + len(vocab)) for w in vocab}
    interp = dict(uni)

    def P(h, w):                                              # the interpolated model, fp64
        if not h:
            return uni[(w,)]
        if h not in ctx:
            return P(h[1:], w)
        t, n = ctx[h]
        return max(cnt[len(h) + 1].get(h + (w,), 0) - D, 0) / t + D * n / t * P(h[1:], w)

    model = {1: {}}
    for m in range(2, order + 1):
        model[m] = {}
        for g in cnt[m]:
            interp[g] = P(g[:-1], g[-1])
    arpa = {m: {g: p for g, p in interp.items() if len(g) == m} for m in range(1, order + 1)}

    # the backoff weight of a history is its interpolation weight D n / t: with it the backoff rule over the entries
    # is the interpolated model itself, so every history's distribution sums to 1
    bos = {h: D * n / t for h, (t, n) in ctx.items()}
    for m in range(1, order + 1):
        for g, p in arpa[m].items():
            model[m][g] = (math.log10(p), math.log10(bos[g]) if m < order and g in bos else None)
    model[1][(BOS,)] = (-99.0, math.log10(bos[(BOS,)]) if (BOS,) in bos else None)
    return model


def write_arpa(path, model):
    """Write {m: {words: (log10 p, log10 bo or None)}} as an ARPA file."""
    n = max(model)
    with open(path, "w") as fh:
        fh.write("\\data\\\n")
        for m in range(1, n + 1):
            fh.write("ngram %d=%d\n" % (m, len(model[m])))
        for m in range(1, n + 1):
            fh.write("\n\\%d-grams:\n" % m)
            for g, (p, b) in sorted(model[m].items()):
                fh.write("%r\t%s" % (p, " ".join(g)) + ("\t%r" % b if b is not None else "") + "\n")
        fh.write("\n\\end\\\n")
    return path


class Brute:
    """The rule of edgedict_b200.ngram over the parsed entries, with no tables: ``prob`` / ``bo`` {words tuple: value}
    with <s> / </s> as their strings and tokens as ints."""

    def __init__(self, model, V, dtype=np.float32, vocab=None):
        self.dtype, self.V = dtype, V
        word = (lambda w: int(w)) if vocab is None else {w: i for i, w in enumerate(vocab) if w}.get
        self.prob, self.bo = {}, {}
        self.unk = None
        for m, ents in model.items():
            for g, (p, b) in ents.items():
                if g == ("<unk>",):
                    self.unk = dtype(p * LN10)
                    continue
                key = tuple(w if w in (BOS, EOS) else word(w) for w in g)
                if None in key:
                    continue
                self.prob[key] = dtype(p * LN10)
                if b is not None:
                    self.bo[key] = dtype(b * LN10)
        self.order = max(model)
        st = {()}
        for k in self.prob:
            if len(k) < self.order and k[-1] != EOS:
                st.add(k)
            for j in range(1, len(k)):
                st.add(k[:j])
        self.states = st

    def g(self, h, k):
        d = self.dtype
        if h + (k,) in self.prob:
            return self.prob[h + (k,)]
        if not h:
            return self.unk if self.unk is not None else d(-100.0 * LN10)
        suf = next(h[j:] for j in range(1, len(h) + 1) if h[j:] in self.states)
        return d(self.bo.get(h, d(0.0)) + self.g(suf, k))

    def next(self, h, k):
        s = h + (k,)
        return next(s[j:] for j in range(len(s) + 1) if s[j:] in self.states)


# ---- the searches with the n-gram term ---------------------------------------------------------------------------------
def _ngram_row(ng, s, V):
    """g(s, k) for every k and the next state of every k, from ng.step (the host table walk)."""
    row = np.zeros(V, dtype=f32)
    nxt = np.zeros(V, dtype=np.int64)
    for k in range(V):
        nxt[k], row[k] = ng.step(s, k)
    return row, nxt


def _end(ng, s):
    return f32(0.0) if ng.end is None else ng.end[s]


def ctc_nbest(y, n, W, ng, w, blank=0, length_bonus=0.0, graph=None):
    """CTC prefix beam search (tests/context_oracle.ctc_nbest without an LM) with the n-gram term:
    f' = ((f + length_bonus) + w g) + delta, final ((pb (+) pnb) + f + w e) - pending -> [(prefix, frames, -that)]."""
    y = np.asarray(y, dtype=f32)
    V = y.shape[1]
    ninf = f32(-np.inf)
    w, lb = f32(w), f32(length_bonus)
    hyps = [dict(seq=(), fr=(), pb=f32(0.0), pnb=ninf, f=f32(0.0), cs=0, ns=ng.start)]
    for t in range(n):
        yt = y[t]
        index = {h["seq"]: q for q, h in enumerate(hyps)}
        nq = len(hyps)
        vals = np.empty((nq, V), dtype=f32)
        pnbx = np.empty((nq, V), dtype=f32)
        fx = np.empty((nq, V), dtype=f32)
        nxt = []
        valid = np.ones((nq, V), dtype=bool)
        A = [logadd(h["pb"], h["pnb"]) for h in hyps]
        for q, h in enumerate(hyps):
            e = h["seq"][-1] if h["seq"] else -1
            pnbx[q] = np.where(np.arange(V) == e, h["pb"], A[q]) + yt
            g, nx = _ngram_row(ng, h["ns"], V)
            nxt.append(nx)
            fq = ((h["f"] + lb).astype(f32) + (w * g).astype(f32)).astype(f32)
            if graph is not None:
                fq = (fq + graph.delta[h["cs"]]).astype(f32)
            fx[q] = fq
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
            stay.append((f32(pb2), f32(pnb2)))
            vals[q, blank] = logadd(pb2, pnb2) + h["f"]
        flat = np.arange(nq * V)
        ok = valid.reshape(-1)
        flat, v = flat[ok], vals.reshape(-1)[ok]
        v = np.where(v == 0, f32(0.0), v)
        order = np.lexsort((flat, -v))[:W]
        new = []
        for i in order:
            q, k = divmod(int(flat[i]), V)
            h = hyps[q]
            if k == blank:
                new.append(dict(h, pb=stay[q][0], pnb=stay[q][1]))
            else:
                new.append(dict(h, seq=h["seq"] + (k,), fr=h["fr"] + (t,), pb=ninf, pnb=pnbx[q, k], f=fx[q, k],
                                ns=int(nxt[q][k]), cs=int(graph.next[h["cs"], k]) if graph is not None else 0))
        hyps = new
    tot = []
    for h in hyps:
        v = f32(f32(logadd(h["pb"], h["pnb"]) + h["f"]) + f32(w * _end(ng, h["ns"])) if ng.end is not None else
                f32(logadd(h["pb"], h["pnb"]) + h["f"]))
        tot.append(f32(v - graph.pending[h["cs"]]) if graph is not None else v)
    return [(hyps[i]["seq"], hyps[i]["fr"], -float(tot[i])) for i in ranked(tot)]


@torch.no_grad()
def transducer_nbest(sd, h_enc, frames, W, ng, w, K=1, merge=True, blank=mt.NUL, length_bonus=0.0, graph=None):
    """tests/context_oracle.transducer_nbest without an LM, with the n-gram term: f = (length_bonus + w g) + delta for
    a non-blank k, final (value + w e) - pending -> per utterance [(tokens, frames, -that)]."""
    V = sd["joint.joint.2.weight"].shape[0]
    w, lb = f32(w), f32(length_bonus)
    out = []
    for b in range(h_enc.shape[0]):
        hyps = [dict(bo.start(sd, None, 1), fr=[], cs=0, ns=ng.start)]
        for t in range(int(frames[b])):
            hyps = [dict(h, open=True) for h in hyps]
            for j in range(K):
                if not any(h["open"] for h in hyps):
                    break
                last = j == K - 1
                cand, nxts = [], {}
                for qi, hy in enumerate(hyps):
                    if not hy["open"]:
                        cand.append((float(hy["lp"]), qi, blank, hy["lp"]))
                        continue
                    a = torch.log_softmax(mt.joint(sd, h_enc[b, t][None], hy["x"][None])[0], 0)
                    g, nx = _ngram_row(ng, hy["ns"], V)
                    nxts[qi] = nx
                    f = ((lb + (w * g).astype(f32)).astype(f32))
                    if graph is not None:
                        f = (f + graph.delta[hy["cs"]]).astype(f32)
                    f[blank] = 0.0
                    lp = (a + torch.from_numpy(f)) + hy["lp"]
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
                        nh.update(x=nx[0, 0], h=h2[:, 0], c=c2[:, 0], ns=int(nxts[qi][k]),
                                  cs=int(graph.next[hy["cs"], k]) if graph is not None else 0)
                    seen[key] = nh
                    new.append(nh)
                hyps = new
            hyps = [dict(h, open=False, fr=h["fr"] + [t] * (len(h["seq"]) - len(h["fr"]))) for h in hyps]
        vals = []
        for h in hyps:
            v = np.float32(float(h["lp"]))
            if ng.end is not None:
                v = f32(v + f32(w * _end(ng, h["ns"])))
            vals.append(f32(v - graph.pending[h["cs"]]) if graph is not None else v)
        out.append([(tuple(hyps[i]["seq"]), tuple(hyps[i]["fr"]), -float(vals[i])) for i in ranked(vals)])
    return out
