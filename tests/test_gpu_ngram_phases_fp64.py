"""One-phase parity of the beam phases with n-gram fusion (decode.cu flag 4096): BEAM_SELECT (with and without
several-symbol rounds), CTC_BEAM and BEAM_FINAL, each run alone as a one-phase program on the planted inputs of
tests/test_gpu_beam_phases_fp64.py's exact regime plus planted n-gram tables, and compared word for word with the host
restatement tests/beam_phases_restate.py.

The restatement needs no n-gram code of its own.  In the exact regime every fp32 operation of the phase is exact
(dyadic logits, log p, weights, table values and increments), so the n-gram and context terms may be regrouped: the
two automata are restated as one product automaton, state z = n-gram state * n_ctx + context state, whose increment
for a non-blank k is (f0 + w g(ns, k)) + delta(cs, k) (f0 the length bonus without an LM, else 0 with the LM term added
by the restatement itself), whose next state pairs the two next states, and whose pending bonus is
pending(cs) - w e(ns).  g and the next states are computed here from the planted tables by the rule of
edgedict_b200/ngram.py (the chain of suffix links from the root, bo + row, the children; the first child found walking
down the chain).  Values, survivors, history planes, sequence rows and both parities of the n-gram (and context)
states must match bit for bit.  Each program runs at max_ctas in {0, 1, 3, 17} through every decode entry that
compiles the phase, and all runs must agree bitwise."""
import numpy as np
import pytest
import torch

from tests import beam_phases_restate as rs
from tests.test_gpu_beam_phases_fp64 import (ENTRIES, CTAS, DEV, F_CONTEXT, F_LM, F_MERGE, F_ROUNDS, _compare,
                                             _ctc_inputs, _launch, _restate, _select_inputs, _words, rs as _rs)

pytestmark = pytest.mark.gpu
F_NGRAM = 4096
NG_KEYS = ("ng_unigram", "ng_bo", "ng_suffix", "ng_depth", "ng_first", "ng_count", "ng_tok", "ng_prob", "ng_next",
           "ng_end")


def _ng_tables(rng, V, blank, n_states=9, with_end=True):
    """A planted model: states 1.. with suffix links to earlier states (depth <= 3), dyadic unigram / bo / p / end,
    each state's children a random sorted token subset (no blank) with random next states."""
    suffix, depth = [0], [0]
    for s in range(1, n_states):
        cand = [u for u in range(s) if depth[u] < 3]
        u = int(rng.choice(cand))
        suffix.append(u)
        depth.append(depth[u] + 1)
    toks = [k for k in range(V) if k != blank]
    first, count, tok, prob, nxt = [], [], [], [], []
    for s in range(n_states):
        n = int(rng.integers(0, min(len(toks), 6) + 1)) if s else min(len(toks), int(rng.integers(1, 40)))
        ks = sorted(int(k) for k in rng.choice(toks, size=n, replace=False))
        first.append(len(tok))
        count.append(n)
        tok += ks
        prob += list(-0.25 * rng.integers(0, 33, size=n))
        nxt += list(rng.integers(0, n_states, size=n))
    f32, i32 = np.float32, np.int32
    return dict(ng_unigram=(-0.25 * rng.integers(1, 40, size=V)).astype(f32),
                ng_bo=np.where(np.arange(n_states) == 0, 0, -0.25 * rng.integers(0, 9, size=n_states)).astype(f32),
                ng_suffix=np.array(suffix, i32), ng_depth=np.array(depth, i32), ng_first=np.array(first, i32),
                ng_count=np.array(count, i32), ng_tok=np.array(tok + [0], i32), ng_prob=np.array(prob + [0], f32),
                ng_next=np.array(nxt + [0], i32),
                ng_end=(-0.25 * rng.integers(1, 17, size=n_states)).astype(f32) if with_end else None)


def _g_next(t, s, k):
    """(g(s, k), next state) by the rule, from the planted tables."""
    chain = [s]
    while chain[-1] != 0:
        chain.append(int(t["ng_suffix"][chain[-1]]))

    def child(u):
        lo, n = int(t["ng_first"][u]), int(t["ng_count"][u])
        hit = np.flatnonzero(t["ng_tok"][lo:lo + n] == k)
        return lo + int(hit[0]) if hit.size else -1
    v = t["ng_unigram"][k]
    for u in reversed(chain[:-1]):
        v = np.float32(t["ng_bo"][u] + v)
        c = child(u)
        if c >= 0:
            v = t["ng_prob"][c]
    for u in chain:
        c = child(u)
        if c >= 0:
            return v, int(t["ng_next"][c])
    return v, 0


def _add_ngram(rng, p, host, V, R, pin, w, lb):
    blank = p["aux2"]
    t = _ng_tables(rng, V, blank, with_end=bool(rng.integers(0, 4)))
    host.update(t)
    st = np.full((2, R), -3, dtype=np.int32)
    st[pin] = rng.integers(0, len(t["ng_bo"]), size=R)
    host["ng_state"] = st
    host["ng_row"] = np.full((R, V), np.nan, dtype=np.float32)
    host["ng_w"] = np.float32(w)
    if not p["flags"] & F_LM:
        host["fuse"] = np.array([0.0, lb], dtype=np.float32)
    p["flags"] |= F_NGRAM


def _run_all(kind, p, host):
    """tests/test_gpu_beam_phases_fp64._run_all with the EbNgram descriptor (ng_* tables, state, row, weight) in the
    EbContext, the n-gram state and the row reset before every run."""
    from edgedict_b200.stream_engine import EbNgram, EbPhase, _ptr
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in host.items()
           if v is not None and k != "ng_w"}
    fields = dict(p)
    for k, t in dev.items():
        if not k.startswith("ctx_") and not k.startswith("ng_"):
            fields[k] = _ptr(t)
    st = dev["ng_state"]
    d = EbNgram(*[_ptr(dev.get(k)) for k in NG_KEYS], st[0].data_ptr(), st[1].data_ptr(), dev["ng_row"].data_ptr(),
                float(host["ng_w"]), 0)
    ngd = torch.frombuffer(bytearray(bytes(d)), dtype=torch.uint8).to(DEV)
    cx = [0] * 5
    if "ctx_next" in dev:
        cs = dev["ctx_state"]
        cx = [dev["ctx_next"].data_ptr(), dev["ctx_delta"].data_ptr(), dev["ctx_pending"].data_ptr(),
              cs[0].data_ptr(), cs[1].data_ptr()]
    desc = torch.tensor(cx + [ngd.data_ptr()], dtype=torch.int64).to(DEV)
    fields["ctx"] = desc.data_ptr()
    ph = EbPhase(**fields)
    first = None
    for entry in ENTRIES[kind]:
        for mc in CTAS:
            for k, t in dev.items():
                t.copy_(torch.from_numpy(np.ascontiguousarray(host[k])))
            _launch(entry, ph, mc)
            snap = {k: t.cpu().numpy() for k, t in dev.items()}
            if first is None:
                first = snap
                continue
            for k in first:
                bad = np.flatnonzero(_words(first[k]).ravel() != _words(snap[k]).ravel())
                assert bad.size == 0, "%s: %s max_ctas=%d differs at %s" % (k, entry, mc, bad[:4].tolist())
    return first


def _product(p, host, V, lb):
    """The restatement's inputs: the product automaton as one context automaton (flag 2048, no 4096)."""
    t = host
    NS = len(t["ng_bo"])
    w = np.float32(t["ng_w"])
    cx = "ctx_next" in t
    NC = len(t["ctx_pending"]) if cx else 1
    cnext = t["ctx_next"] if cx else np.zeros((1, V), np.int32)
    cdelta = t["ctx_delta"] if cx else np.zeros((1, V), np.float32)
    cpend = t["ctx_pending"] if cx else np.zeros(1, np.float32)
    f0 = np.float32(0.0 if p["flags"] & F_LM else lb)
    nz = NS * NC
    nxt = np.zeros((nz, V), np.int32)
    dl = np.zeros((nz, V), np.float32)
    pend = np.zeros(nz, np.float32)
    for ns in range(NS):
        gk = [_g_next(t, ns, k) for k in range(V)]
        g = np.array([a for a, _ in gk], np.float32)
        nn = np.array([b for _, b in gk], np.int64)
        e = t["ng_end"][ns] if t["ng_end"] is not None else np.float32(0.0)
        for cs in range(NC):
            z = ns * NC + cs
            dl[z] = ((f0 + w * g).astype(np.float32) + cdelta[cs]).astype(np.float32)
            nxt[z] = nn * NC + cnext[cs]
            pend[z] = np.float32(cpend[cs] - np.float32(w * e))
    cst = t["ctx_state"] if cx else np.zeros_like(t["ng_state"])
    z = np.where((t["ng_state"] >= 0) & (cst >= 0), t["ng_state"] * NC + cst, -3).astype(np.int32)
    d = {k: v for k, v in host.items() if not k.startswith("ng_") and not k.startswith("ctx_")}
    d.update(ctx_next=nxt, ctx_delta=dl, ctx_pending=pend, ctx_state=z)
    q = dict(p)
    q["flags"] = (q["flags"] & ~F_NGRAM) | F_CONTEXT
    return q, d, NC, cx


def _split(want, NC, cx):
    z = want.pop("ctx_state")
    for k in ("ctx_next", "ctx_delta", "ctx_pending"):
        want.pop(k, None)
    want["ng_state"] = np.where(z >= 0, z // NC, -3).astype(np.int32)
    if cx:
        want["ctx_state"] = np.where(z >= 0, z % NC, -3).astype(np.int32)
    return want


SELECT_CASES = [
    (3, 2, 3, F_MERGE, 2, "mid"), (5, 31, 33, F_MERGE, 31, "mid"), (4, 32, 33, F_MERGE | F_LM, 7, "frozen"),
    (4, 33, 1024, F_MERGE | F_CONTEXT, 33, "mid"), (3, 256, 3, F_MERGE | F_LM | F_CONTEXT, 256, "ninf"),
    (2, 1024, 33, F_MERGE | F_CONTEXT, 1024, "t0"), (4, 8, 33, F_MERGE | F_ROUNDS, 8, "r0"),
    (4, 16, 33, F_MERGE | F_ROUNDS | F_LM | F_CONTEXT, 16, "rmid"), (4, 8, 3, F_MERGE | F_ROUNDS | F_CONTEXT, 8, "rdone"),
    (4, 33, 33, F_ROUNDS, 30, "rlast"),
]


@pytest.mark.parametrize("S,W,V,flags,live,mode", SELECT_CASES)
def test_beam_select_ngram_exact(S, W, V, flags, live, mode):
    p, host, _ = _select_inputs(S, W, V, flags, live, mode, seed=S * 7919 + W * 31 + V + flags + len(mode) + 1)
    rng = np.random.default_rng(W + V)
    multi = flags & F_ROUNDS
    pin = 0 if multi else p["hist_col"] & 1
    _add_ngram(rng, p, host, V, S * W, pin, 0.5, -0.75)
    got = _run_all("select", p, host)
    q, d, NC, cx = _product(p, host, V, -0.75)
    want, folded = _restate(rs.beam_select, q, d)
    want = _split(want, NC, cx)
    n = S * p["hist_ld"] * W
    fold = dict(y=folded, hist=[2 * n + (r // W * p["hist_ld"] + p["hist_col"]) * W + r % W for r in folded])
    _compare("ngram select W=%d V=%d flags=%d %s" % (W, V, flags, mode), got, want, fold)


CTC_CASES = [
    (3, 2, 3, 0, 2, 3, "levels"), (4, 31, 33, 0, 31, 1, "ties"), (4, 32, 33, F_LM, 32, 1, "levels"),
    (4, 33, 33, F_CONTEXT, 20, 3, "frozen"), (3, 256, 1024, F_CONTEXT | F_LM, 256, 1, "levels"),
    (2, 1024, 33, 0, 1024, 2, "levels"), (140, 4, 33, F_CONTEXT, 4, 2, "frozen"),
]


@pytest.mark.parametrize("S,W,V,flags,live,n,mode", CTC_CASES)
def test_ctc_beam_ngram_exact(S, W, V, flags, live, n, mode):
    p, host, _ = _ctc_inputs(S, W, V, flags, live, n, mode, seed=S * 31 + W * 7 + V + flags + n + 1)
    rng = np.random.default_rng(W * 3 + V)
    _add_ngram(rng, p, host, V, S * W, p["hist_col"] & 1, 0.5, 0.25)
    got = _run_all("ctc", p, host)
    q, d, NC, cx = _product(p, host, V, 0.25)
    want, folded = _restate(rs.ctc_beam, q, d)
    want = _split(want, NC, cx)
    T, R = p["hist_ld"], S * W
    last_t = {}
    for t, r in folded:
        last_t.setdefault(r, set()).add(t)
    fold = dict(y=[r for r, ts in last_t.items() if max(ts) == p["hist_col"] + n - 1],
                hist=[2 * S * T * W + (r // W * T + t) * W + r % W for t, r in folded],
                c=[par * 3 * R + pl * R + r for t, r in folded for par in (0, 1) for pl in (0, 1)])
    _compare("ngram ctc W=%d V=%d flags=%d n=%d %s" % (W, V, flags, n, mode), got, want, fold)


@pytest.mark.parametrize("S,W,T,N,K,cx", [(3, 4, 6, 0, 1, False), (5, 32, 9, 4, 1, True), (2, 1024, 3, 32, 2, True),
                                          (4, 7, 8, 7, 3, False)])
def test_beam_final_ngram_exact(S, W, T, N, K, cx):
    rng = np.random.default_rng(S * 5 + W + T + N + K)
    blank, R, NB = 0, S * W, max(N, 1)
    hist = np.zeros(3 * S * T * W + S * T, dtype=np.int32)
    hpar, htok, _, hlive = _rs.hist_views(hist, S, T, W)
    for b in range(S):
        prev = 1
        for t in range(T):
            nl = W if t == T - 1 else int(rng.integers(1, W + 1))
            hpar[b, t] = rng.integers(0, prev, size=W)
            htok[b, t] = np.where(rng.random(W) < 0.4, blank, rng.integers(1, 900, size=W))
            hlive[b, t] = nl
            prev = nl
    y = (-0.25 * rng.integers(0, 12, size=R)).astype(np.float32)
    ldy = T + 2
    host = dict(y=y, hist=hist, tok_out=np.full(S * NB * ldy, -9, dtype=np.int32),
                y2=np.full(S * NB, np.nan, dtype=np.float32),
                seq_out=np.full(S * NB * ldy, -9, dtype=np.int32) if N else None,
                tok_out2=np.full(S, -9, dtype=np.int32) if N else None)
    par = int(rng.integers(0, 2))
    p = dict(type=8, S=S, aux=W, aux2=blank, hist_ld=T, ldy=ldy, K1=N, ldw2=K, hist_col=par + 2, flags=0)
    if cx:
        host.update(ctx_next=np.zeros((5, 1), np.int32), ctx_delta=np.zeros((5, 1), np.float32),
                    ctx_pending=(0.25 * rng.integers(0, 17, size=5)).astype(np.float32))
        st = np.full((2, R), -3, dtype=np.int32)
        st[par] = rng.integers(0, 5, size=R)
        host["ctx_state"] = st
        p["flags"] |= F_CONTEXT
    _add_ngram(rng, p, host, 1, R, par, 0.5, 0.0)
    host.pop("fuse", None)
    host["ng_end"] = (-0.25 * rng.integers(1, 17, size=len(host["ng_bo"]))).astype(np.float32)
    got = _run_all("final", p, host)
    q, d, NC, cxx = _product(p, host, 1, 0.0)
    want, _ = _restate(rs.beam_final, q, d)
    want = _split(want, NC, cxx)
    _compare("ngram final W=%d T=%d N=%d K=%d" % (W, T, N, K), got, want)
