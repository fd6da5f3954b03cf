"""CPU restatements of forced (Viterbi) alignment in numpy fp64, written from the recurrences stated with
eb_rnnt_viterbi and eb_ctc_align in include/edgedict_b200.h, not from the kernels.

Each cell's value is one fp64 add of an fp64 predecessor and a log-prob widened to fp64, so these functions give the
kernels' values bit for bit.  Ties:
  * transducer: a cell takes "stay" (blank from t-1) unless "emit" (label from u-1) is strictly greater;
  * CTC: predecessors in the order s, s-1, s-2, a later one replacing the current only when strictly greater; the path
    ends in the last label state unless the final blank state is strictly greater.
"""
import numpy as np

NINF = -np.inf


def rnnt_viterbi(lpb, lpl):
    """lpb, lpl [T, U+1] (one utterance, already cut to its lengths) -> (frames int64 [U], label_logp [U] in lpl's
    dtype, score fp64).  frames[u] is the t of the step (t, u) -> (t, u+1).  T = 0: (-1, -inf, -inf)."""
    T, U1 = lpb.shape
    if T == 0:
        return np.full(U1 - 1, -1, np.int64), np.full(U1 - 1, NINF, lpl.dtype), NINF
    b64, l64 = lpb.astype(np.float64), lpl.astype(np.float64)
    d = np.full((T, U1), NINF)
    emit_won = np.zeros((T, U1), bool)
    d[0, 0] = 0.0
    # anti-diagonal n holds the cells t + u = n: both predecessors lie on diagonal n - 1
    for n in range(1, T + U1 - 1):
        u = np.arange(max(0, n - T + 1), min(n, U1 - 1) + 1)
        t = n - u
        stay = np.where(t > 0, d[np.maximum(t - 1, 0), u] + b64[np.maximum(t - 1, 0), u], NINF)
        emit = np.where(u > 0, d[t, np.maximum(u - 1, 0)] + l64[t, np.maximum(u - 1, 0)], NINF)
        e = emit > stay
        d[t, u] = np.where(e, emit, stay)
        emit_won[t, u] = e
    score = d[T - 1, U1 - 1] + b64[T - 1, U1 - 1]
    frames = np.zeros(U1 - 1, np.int64)
    t, u = T - 1, U1 - 1
    while u > 0:
        if t == 0 or emit_won[t, u]:
            u -= 1
            frames[u] = t
        else:
            t -= 1
    return frames, lpl[frames, np.arange(U1 - 1)], score


def ctc_extended(labels, blank):
    ext = [blank]
    for c in labels:
        ext += [int(c), blank]
    return np.array(ext, np.int64)


def ctc_viterbi(lp, labels, blank):
    """lp [T, V] (one utterance, cut to its input length), labels [S] -> (alignment int64 [T], frame_logp [T] in lp's
    dtype, score fp64).  No alignment: (-1, -inf, -inf) throughout; T = 0 with no labels: empty arrays, score 0."""
    T, V = lp.shape
    ext = ctc_extended(labels, blank)
    L = len(ext)
    none = (np.full(T, -1, np.int64), np.full(T, NINF, lp.dtype), NINF)
    if T == 0:
        return (np.zeros(0, np.int64), np.zeros(0, lp.dtype), 0.0) if L == 1 else none
    ok = (ext >= 0) & (ext < V)
    lp64 = lp.astype(np.float64)
    e = np.where(ok[None, :], lp64[:, np.clip(ext, 0, V - 1)], NINF)          # [T, L]
    skip = np.zeros(L, bool)
    skip[2:] = (np.arange(2, L) % 2 == 1) & (ext[2:] != ext[:-2])
    d = np.full(L, NINF)
    d[:min(2, L)] = e[0, :min(2, L)]
    back = np.zeros((T, L), np.int64)
    for t in range(1, T):
        best, bk = d.copy(), np.zeros(L, np.int64)
        c1 = np.concatenate([[NINF], d[:-1]])
        m = c1 > best
        best[m], bk[m] = c1[m], 1
        c2 = np.where(skip, np.concatenate([[NINF, NINF], d[:-2]])[:L], NINF)
        m = c2 > best
        best[m], bk[m] = c2[m], 2
        d = best + e[t]
        back[t] = bk
    s = L - 1
    if L >= 2 and not d[L - 1] > d[L - 2]:
        s = L - 2
    score = d[s]
    if not score > NINF:
        return none
    path = np.zeros(T, np.int64)
    for t in range(T - 1, -1, -1):
        path[t] = s
        s -= back[t, s]
    align = ext[path]
    return align, lp[np.arange(T), align], score


# ---- brute force over every alignment, for tiny sizes ----------------------------------------------------------------
def rnnt_all_paths(lpb, lpl):
    """Every monotone lattice path as (frames, score summed in path order in fp64)."""
    T, U1 = lpb.shape
    out = []

    def walk(t, u, acc, frames):
        if t == T - 1 and u == U1 - 1:
            out.append((tuple(frames), acc + float(lpb[t, u])))
            return
        if t + 1 < T:
            walk(t + 1, u, acc + float(lpb[t, u]), frames)
        if u + 1 < U1:
            walk(t, u + 1, acc + float(lpl[t, u]), frames + [t])

    walk(0, 0, 0.0, [])
    return out


def ctc_all_paths(lp, labels, blank):
    """Every valid CTC state path as (frame labels, score summed in frame order in fp64)."""
    T, V = lp.shape
    ext = ctc_extended(labels, blank)
    L = len(ext)
    out = []

    def walk(t, s, acc, seq):
        if not 0 <= ext[s] < V:
            return
        acc = acc + float(lp[t, ext[s]])
        seq = seq + [int(ext[s])]
        if t == T - 1:
            if s >= L - 2:
                out.append((tuple(seq), acc))
            return
        for k in (0, 1, 2):
            n = s + k
            if n >= L or (k == 2 and not (n % 2 == 1 and ext[n] != ext[s])):
                continue
            walk(t + 1, n, acc, seq)

    for s0 in range(min(2, L)):
        walk(0, s0, 0.0, [])
    return out
