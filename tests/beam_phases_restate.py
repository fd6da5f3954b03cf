"""Host restatement of the beam phases of the decode program (csrc/decode.cu): BEAM_SELECT (plain, merge, LM fusion,
streaming, several symbols per frame, contextual biasing, frozen rows), CTC_BEAM (frames per phase, LM fusion,
streaming, contextual biasing), BEAM_COMMIT, BEAM_FINAL (N-best, frames, pending bonus) and GATHER (aux planes, the x2
operand).  Each function takes the phase's fields (a dict, the names of EbPhase) and host copies of the buffers the
phase reads and writes (numpy arrays, the device layout), and writes into those copies what the phase's contract says
it writes, so a whole buffer compares with the device's, sentinels included.

The contract is the field-use comments in decode.cu and include/edgedict_b200.h, stated independently of the kernel's
algorithm: the top min(W, candidates) by sorting (value descending, then the lowest flat index, with -0 ranking as +0;
BEAM_SELECT's survivors carry the value of their rank key, so a -0 comes back as +0), not a radix select and a bitonic sort; merges by comparing whole token sequences, not hashes; the sequence hash
h' = h * 0x100000001b3 + (k + 1) in Python integers mod 2^64.

Arithmetic is fp32 in the order the contract states ((x - max) - lse, then + fusion term, then + log p).  It is the
device's bit for bit where every such operation is exact (the exact regime of tests/test_gpu_beam_phases_fp64.py).
Two things are not exact on any inputs and are flagged instead: the log-softmax statistics (computed in fp64 and
rounded; exactly 0 when a row's maximum is unique and every other entry underflows in expf) and a log-add whose
expf term does not underflow (logaddexp_, whose log1pf / expf the host does not reproduce to the bit).  Every
function returns the positions whose value went through such a log-add."""
import numpy as np

MUL = 0x100000001b3
M64 = (1 << 64) - 1
f32 = np.float32
NINF = f32(-np.inf)


def order_key(v):
    """decode.cu's order_key over a float32 array as int64: larger float -> larger key, -0 with +0."""
    v = np.where(np.asarray(v, dtype=f32) == 0, f32(0), np.asarray(v, dtype=f32)).astype(f32)
    b = v.view(np.uint32).astype(np.int64)
    return np.where(b & 0x80000000, (~b) & 0xffffffff, b | 0x80000000)


def ranked(values, flat):
    """Indices of the candidates in rank order: value descending, then flat index ascending."""
    return np.lexsort((np.asarray(flat, dtype=np.int64), -order_key(values)))


def logadd(a, b):
    """logaddexp_ in fp32: (value, exact) where exact tells that the expf term underflowed to 0 (or m = -inf), so
    the device's value is m bit for bit."""
    a, b = f32(a), f32(b)
    m = max(a, b)
    if m == NINF:
        return m, True
    with np.errstate(over="ignore", under="ignore"):
        e = np.exp(-np.abs(f32(a - b)), dtype=f32)
    return f32(m + np.log1p(e, dtype=f32)), bool(e == 0)


def log_softmax_stats(x):
    """(max, log sum exp(x - max)) of one fp32 row: exact when the maximum is unique and every other entry lies
    more than 104 below it."""
    x = np.asarray(x, dtype=f32)
    m = x.max()
    if m == NINF:
        return m, f32(np.nan)
    return m, f32(np.log(np.exp((x - m).astype(np.float64)).sum()))


def hash_words(h):
    """A 64-bit hash as the two int32 words of a sequence row."""
    lo, hi = h & 0xffffffff, h >> 32
    return [lo - (1 << 32) if lo >= 1 << 31 else lo, hi - (1 << 32) if hi >= 1 << 31 else hi]


def row_hash(row, at=1):
    return (int(row[at]) & 0xffffffff) | ((int(row[at + 1]) & 0xffffffff) << 32)


def ext_hash(h, k):
    return (h * MUL + k + 1) & M64


def seq_hash(tokens, h=0):
    for k in tokens:
        h = ext_hash(h, int(k))
    return h


def hist_views(hist, S, T, W):
    """The four planes of a history buffer (int32 flat): parent, token [S,T,W], log p (fp32) [S,T,W], live [S,T]."""
    n = S * T * W
    return (hist[:n].reshape(S, T, W), hist[n:2 * n].reshape(S, T, W), hist[2 * n:3 * n].view(f32).reshape(S, T, W),
            hist[3 * n:3 * n + S * T].reshape(S, T))


def _fusion(p, d, r, ks, cs):
    """The fusion term of non-blank tokens ks of row r (LM: lm_weight * LM log p + length_bonus, or length_bonus for
    an unmapped token; then + the context increment of state cs), fp32 in that order, or None without either."""
    lm, cx = p["flags"] & 32, p["flags"] & 2048
    if not (lm or cx):
        return None
    f = np.zeros(len(ks), dtype=f32)
    if lm:
        lw, lb = (f32(v) for v in d["fuse"][:2])
        l = d["x2"][r, :p["K2"]]
        lmx, lmls = log_softmax_stats(l)
        j = d["tok_map"][ks]
        g = f32(lw * ((l[np.maximum(j, 0)] - lmx) - lmls)) + lb
        f = np.where(j >= 0, g, lb).astype(f32)
    if cx:
        dr = d["ctx_delta"][cs, ks]
        f = (f + dr).astype(f32) if lm else dr.astype(f32)
    return f


def beam_select(p, d):
    """BEAM_SELECT.  d: x1 [R, ldx1], y [R], tok_in [S], tok_out [R], src [R], seq_in / seq_out [R, LS] (int32),
    hist (int32 flat), and with flags 32 x2 [R, ldx2], fuse, tok_map, tok_out2; with 2048 ctx_next / ctx_delta
    [n, V], ctx_state [2, R].  Returns the set of rows r whose y (and history log p) is a log-add fold."""
    S, W, V, T, col, blank, fl = p["S"], p["aux"], p["N"], p["hist_ld"], p["hist_col"], p["aux2"], p["flags"]
    multi, merge, lm, stream, cx = fl & 512, fl & 16, fl & 32, fl & 64, fl & 2048
    KR = p["ldw2"] if multi else 1
    t, jr = (col // KR, col % KR) if multi else (col, 0)
    last = jr == KR - 1
    LS = p["K1"] if stream else T + 3
    hpar, htok, hlp, hlive = hist_views(d["hist"], S, T, W)
    y, tok_out, src, sin, sout = d["y"], d["tok_out"], d["src"], d["seq_in"].reshape(-1, LS), d["seq_out"].reshape(-1, LS)
    cin = cout = None
    if cx:
        cin, cout = (d["ctx_state"][0], d["ctx_state"][1]) if multi else (d["ctx_state"][t & 1], d["ctx_state"][(t & 1) ^ 1])
    folded = set()
    for b in range(S):
        r0 = b * W
        rows = np.arange(r0, r0 + W)
        nlive = int(hlive[b, T - 1] if multi else hlive[b, t - 1] if t > 0 else hlive[b, T - 1] if stream else 1)
        if multi:
            opn = [jr == 0 or int(tok_out[r0 + q]) != blank for q in range(nlive)]
            nopen = sum(opn)
            if t >= d["tok_in"][b] or nopen == 0:               # the beam stays: no history, no y
                tok_out[rows], src[rows] = blank, rows
                if lm:
                    d["tok_out2"][rows] = -1
                if cx:
                    cout[rows] = cin[rows]
                for s in range(nlive):
                    n = int(sin[r0 + s, 0]) + 3
                    sout[r0 + s, :n] = sin[r0 + s, :n]
                continue
        elif t >= d["tok_in"][b]:                              # frozen: an identity history entry
            hpar[b, col], htok[b, col], hlp[b, col] = np.arange(W), blank, y[rows]
            tok_out[rows], src[rows] = blank, rows
            if lm:
                d["tok_out2"][rows] = -1
            if cx:
                cout[rows] = cin[rows]
            hlive[b, col] = nlive
            continue
        else:
            opn, nopen = [True] * nlive, nlive
        vals, flats = [], []
        ks = np.arange(V)
        for q in range(nlive):
            r = r0 + q
            if not opn[q]:                                    # a closed slot's stay
                vals.append(np.array([y[r]], dtype=f32))
                flats.append(np.array([q * V + blank]))
                continue
            x = d["x1"][r, :V]
            m, ls = log_softmax_stats(x)
            a = ((x - m) - ls).astype(f32)
            f = _fusion(p, d, r, ks, int(cin[r]) if cx else 0)
            if f is not None:
                a = (a + np.where(ks != blank, f, f32(0))).astype(f32)
            vals.append((a + y[r]).astype(f32))
            flats.append(q * V + ks)
        vals, flats = np.concatenate(vals), np.concatenate(flats)
        nsel = min(W, nopen * V + (nlive - nopen))
        sel = ranked(vals, flats)[:nsel]
        qs, kk = flats[sel] // V, flats[sel] % V
        vs = np.where(vals[sel] == 0, f32(0), vals[sel]).astype(f32)   # the rank key's value: -0 comes back +0

        def seq(i):
            q, k = int(qs[i]), int(kk[i])
            toks = tuple(int(v) for v in sin[r0 + q, 3:3 + int(sin[r0 + q, 0])])
            return toks + ((k,) if k != blank else ())

        seqs = [seq(i) for i in range(nsel)]
        closed = [int(k) == blank or last for k in kk]
        first = list(range(nsel))
        if merge:                                             # the earliest survivor of the same sequence (and closedness)
            seen = {}
            for i in range(nsel):
                first[i] = seen.setdefault((seqs[i], closed[i] if multi else None), i)
        kept = [i for i in range(nsel) if first[i] == i]
        for s in range(W):
            r = r0 + s
            if s < len(kept):
                i = kept[s]
                q, k = int(qs[i]), int(kk[i])
                lp, fold = vs[i], False
                for j in range(i + 1, nsel):
                    if first[j] == i:
                        lp, ex = logadd(lp, vs[j])
                        fold |= not ex
                if fold:
                    folded.add(r)
                y[r], tok_out[r], src[r] = lp, k, r0 + q
                if lm:
                    d["tok_out2"][r] = d["tok_map"][k] if k != blank else -1
                hpar[b, col, s], htok[b, col, s], hlp[b, col, s] = q, k, lp
                h = row_hash(sin[r0 + q])
                if k != blank:
                    h = ext_hash(h, k)
                n = len(seqs[i])
                sout[r, :3] = [n] + hash_words(h)
                sout[r, 3:3 + n] = seqs[i]
                if cx:
                    cs = int(cin[r0 + q])
                    cout[r] = d["ctx_next"][cs, k] if k != blank else cs
            else:
                y[r], tok_out[r], src[r] = NINF, blank, r
                if lm:
                    d["tok_out2"][r] = -1
                if cx:
                    cout[r] = 0
                hpar[b, col, s], htok[b, col, s], hlp[b, col, s] = s, blank, NINF
        hlive[b, col] = len(kept)
        if multi:
            hlive[b, T - 1] = len(kept)
    return folded


def gather(p, d):
    """GATHER: y[l, r, :] = x1[l, src[r], :] for the aux planes of S rows of N floats, and y2[r] = x2[src[r]] (K2
    floats) when x2 is set."""
    S, N, aux = p["S"], p["N"], p["aux"]
    src = d["src"]
    d["y"][:aux * S * N] = d["x1"][:aux * S * N].reshape(aux, S, N)[:, src, :].ravel()
    if d.get("x2") is not None:
        K2 = p["K2"]
        d["y2"][:S * K2] = d["x2"].reshape(-1, K2)[src].ravel()


def beam_final(p, d):
    """BEAM_FINAL.  d: y [R], hist, tok_out (int32 flat, rows of ldy), y2 [S*N], optional seq_out (frames, rows of
    ldy) and tok_out2 [S]; with flags 2048 ctx_pending [n] and ctx_state [2, R] (parity hist_col & 1)."""
    S, W, T, blank, ldy = p["S"], p["aux"], p["hist_ld"], p["aux2"], p["ldy"]
    NB, KR = max(p.get("K1", 0), 1), max(p.get("ldw2", 0), 1)
    hpar, htok, _, hlive = hist_views(d["hist"], S, T, W)
    for b in range(S):
        nlive = 1 if T == 0 else int(hlive[b, T - 1])
        v = d["y"][b * W:b * W + nlive].astype(f32)
        if p.get("flags", 0) & 2048:
            v = (v - d["ctx_pending"][d["ctx_state"][p["hist_col"] & 1][b * W:b * W + nlive]]).astype(f32)
        order = ranked(v, np.arange(nlive))
        cnt = min(NB, nlive)
        for n in range(NB):
            row = b * NB + n
            ids = d["tok_out"][row * ldy:row * ldy + ldy]
            fr = d["seq_out"][row * ldy:row * ldy + ldy] if d.get("seq_out") is not None else None
            pos = T
            if n < cnt:
                slot = int(order[n])
                for tt in range(T - 1, -1, -1):
                    k = int(htok[b, tt, slot])
                    if k != blank:
                        pos -= 1
                        ids[pos] = k
                        if fr is not None:
                            fr[pos] = tt // KR
                    slot = int(hpar[b, tt, slot])
                d["y2"][row] = -v[order[n]]
            else:
                d["y2"][row] = f32(np.inf)
            ids[:pos] = -1
            if fr is not None:
                fr[:pos] = -1
        if d.get("tok_out2") is not None:
            d["tok_out2"][b] = cnt


def beam_commit(p, d):
    """BEAM_COMMIT.  d: y [R], hist, seq_in / seq_out [R, K1] (int32), tok_out [S, N], tok_out2 [2S], src [R],
    optional y2 (int32 [S], the last committed token)."""
    S, W, T, LS, aux2 = p["S"], p["aux"], p["hist_ld"], p["K1"], p["aux2"]
    HEAD = p["K2"] if p["K2"] > 0 else 3
    _, _, _, hlive = hist_views(d["hist"], S, T, W)
    sin, sout, y = d["seq_in"].reshape(-1, LS), d["seq_out"].reshape(-1, LS), d["y"]
    for b in range(S):
        r0 = b * W
        nlive = int(hlive[b, T - 1])
        lens = sin[r0:r0 + nlive, 0].astype(int)
        lmin = int(lens.min())
        c = lmin
        for j in range(lmin):
            if (sin[r0:r0 + nlive, HEAD + j] != sin[r0, HEAD + j]).any():
                c = j
                break
        collapse = bool(p["flags"] & 128) or int(lens.max()) - c > aux2
        best = int(np.argmax(y[r0:r0 + nlive])) if collapse else 0       # the first of equal maxima, -0 with +0
        bval = y[r0 + best]
        bs = sin[r0 + best]
        ncommit = int(bs[0]) if collapse else c
        d["tok_out"][b * p["N"]:b * p["N"] + ncommit] = bs[HEAD:HEAD + ncommit]
        nkeep = 1 if collapse else nlive
        for s in range(nkeep):
            ps = sin[r0 + (best if collapse else s)]
            n = int(ps[0]) - ncommit
            sout[r0 + s, 0] = n
            sout[r0 + s, 1:HEAD] = ps[1:HEAD]
            sout[r0 + s, HEAD:HEAD + n] = ps[HEAD + ncommit:HEAD + ncommit + n]
        d["src"][r0:r0 + W] = r0 + np.arange(W)
        d["src"][r0] = r0 + best
        if collapse:
            y[r0 + 1:r0 + W] = NINF
            y[r0] = bval
        d["tok_out2"][b], d["tok_out2"][S + b] = ncommit, int(collapse)
        hlive[b, T - 1] = nkeep
        if d.get("y2") is not None and ncommit > 0:
            d["y2"][b] = bs[HEAD + ncommit - 1]


def ctc_beam(p, d):
    """CTC_BEAM over frames hist_col .. hist_col + ldw1 - 1.  d: x1 [S, T, V], tok_in [S], c [2, 3, R], seq_out
    [2, R, K1] (int32), y [R], src [R], hist; flags 32: x2, fuse, tok_map, tok_out2; flags 64: y2 (int32 [S], the last
    committed token); flags 2048: ctx_next / ctx_delta [n, V], ctx_state [2, R].  Returns the set of (frame, row)
    whose values went through a log-add that is not exact."""
    S, W, V, T, blank, LS, fl = p["S"], p["aux"], p["N"], p["hist_ld"], p["aux2"], p["K1"], p["flags"]
    lm, stream, cx = fl & 32, fl & 64, fl & 2048
    R = S * W
    hpar, htok, hlp, hlive = hist_views(d["hist"], S, T, W)
    c, seqs, yv, src = d["c"].reshape(2, 3, R), d["seq_out"].reshape(2, R, LS), d["y"], d["src"]
    cst = d["ctx_state"] if cx else None
    folded = set()
    ks = np.arange(V)
    for b in range(S):
        r0 = b * W
        rows = np.arange(r0, r0 + W)
        e0 = int(d["y2"][b]) if stream else -1
        taint = set()                                         # rows whose state carries a folded value
        for t in range(p["hist_col"], p["hist_col"] + p["ldw1"]):
            nlive = int(hlive[b, t - 1] if t > 0 else hlive[b, T - 1] if stream else 1)
            if t >= d["tok_in"][b]:                            # frozen
                hpar[b, t], htok[b, t], hlp[b, t] = np.arange(W), blank, yv[rows]
                src[rows] = rows
                if lm:
                    d["tok_out2"][rows] = -1
                if cx:
                    cst[(t + 1) & 1][rows] = cst[t & 1][rows]
                hlive[b, t] = nlive
                folded |= {(t, r) for r in taint}
                continue
            si, so = c[t & 1], c[(t + 1) & 1]
            qin, qout = seqs[t & 1], seqs[(t + 1) & 1]
            y = d["x1"][b, t, :V].astype(f32)
            live = range(nlive)
            pb = [si[0, r0 + q] for q in live]
            pnb = [si[1, r0 + q] for q in live]
            f = [si[2, r0 + q] for q in live]
            A, exA = zip(*[logadd(pb[q], pnb[q]) for q in live])
            toks = [tuple(int(v) for v in qin[r0 + q, 5:5 + int(qin[r0 + q, 0])]) for q in live]
            se = [tk[-1] if tk else e0 for tk in toks]
            st = [int(cst[t & 1][r0 + q]) for q in live] if cx else [0] * nlive
            index = {}
            for q in live:
                index.setdefault(toks[q], q)
            par = [index.get(toks[q2][:-1], -1) if toks[q2] else -1 for q2 in live]
            merged = {(par[q2], se[q2]) for q2 in live if par[q2] >= 0}
            inexact = [not exA[q] or r0 + q in taint for q in live]

            def stay(q):
                e = se[q]
                pb2 = f32(A[q] + y[blank])
                pnb2 = f32(pnb[q] + y[e]) if e >= 0 else NINF
                bad = inexact[q]
                if par[q] >= 0:
                    pq = par[q]
                    pnb2, ex = logadd(pnb2, f32((pb[pq] if e == se[pq] else A[pq]) + y[e]))
                    bad |= not ex or (e != se[pq] and inexact[pq])
                return pb2, pnb2, bad

            # every candidate (q, k) of the live slots: a stay at k = blank, extensions elsewhere, [nlive, V]
            PB2, PNB2 = np.full((nlive, V), NINF, dtype=f32), np.empty((nlive, V), dtype=f32)
            F2, BAD = np.empty((nlive, V), dtype=f32), np.zeros((nlive, V), dtype=bool)
            ok = np.ones((nlive, V), dtype=bool)
            nolm = dict(p, flags=fl & ~2048)
            for q in live:
                PNB2[q] = np.where(ks == se[q], pb[q], A[q]).astype(f32) + y
                F2[q] = f[q]
                if lm:                                        # + the LM term, then + the context increment
                    F2[q] = (F2[q] + _fusion(nolm, d, r0 + q, ks, 0)).astype(f32)
                if cx:
                    F2[q] = (F2[q] + d["ctx_delta"][st[q]]).astype(f32)
                BAD[q] = inexact[q]
                pb2, pnb2, bad = stay(q)
                v, ex = logadd(pb2, pnb2)
                PB2[q, blank], PNB2[q, blank], F2[q, blank], BAD[q, blank] = pb2, pnb2, f[q], bad or not ex
            VAL = (PNB2 + F2).astype(f32)
            for q in live:
                VAL[q, blank] = f32(logadd(PB2[q, blank], PNB2[q, blank])[0] + f[q])
            for q, k in merged:                               # merged into a live slot's stay: no candidate
                ok[q, k] = False
            flat = np.flatnonzero(ok.ravel())
            vals = VAL.ravel()[flat]
            nsel = min(W, len(vals))
            order = flat[ranked(vals, flat)[:nsel]]
            for s in range(W):
                r, hc = r0 + s, (b, t, s)
                if s < nsel:
                    q, k = divmod(int(order[s]), V)
                    pb2, pnb2, f2, bad = PB2[q, k], PNB2[q, k], F2[q, k], BAD[q, k]
                    v = VAL[q, k]
                    so[0, r], so[1, r], so[2, r] = pb2, pnb2, f2
                    if cx:
                        cst[(t + 1) & 1][r] = st[q] if k == blank else d["ctx_next"][st[q], k]
                    yv[r], src[r] = v, r0 + q
                    if lm:
                        d["tok_out2"][r] = d["tok_map"][k] if k != blank else -1
                    hpar[hc], htok[hc], hlp[hc] = q, k, v
                    if bad:
                        folded.add((t, r))
                    row = qin[r0 + q]
                    n = int(row[0])
                    if k == blank:
                        qout[r, :5 + n] = row[:5 + n]
                    else:
                        h = row_hash(row)
                        qout[r, :5] = [n + 1] + hash_words(ext_hash(h, k)) + hash_words(h)
                        qout[r, 5:5 + n] = row[5:5 + n]
                        qout[r, 5 + n] = k
                else:
                    so[0, r], so[1, r], so[2, r] = NINF, NINF, f32(0)
                    if cx:
                        cst[(t + 1) & 1][r] = 0
                    yv[r], src[r] = NINF, r
                    if lm:
                        d["tok_out2"][r] = -1
                    hpar[hc], htok[hc], hlp[hc] = s, blank, NINF
            hlive[b, t] = nsel
            taint = {r for tt, r in folded if tt == t}
    return folded
