"""CPU checks of the beam-phase restatement (tests/beam_phases_restate.py), which tests/test_gpu_beam_phases_fp64.py
compares the device phases with: BEAM_SELECT frame by frame against exhaustive enumeration of every alignment, with
and without pruning; CTC_BEAM frame by frame against tests/ctc_beam_oracle.py's prefix beam search; BEAM_FINAL and
BEAM_COMMIT against brute force; the ranking rule and the sequence hash."""
import itertools

import numpy as np
import pytest

from tests import beam_phases_restate as rs
from tests.ctc_beam_oracle import prefix_beam_search


def test_ranking_rule():
    """Value descending, the lowest flat index on ties, -0 with +0, -inf last."""
    v = np.array([0.0, -0.0, 1.0, -np.inf, 1.0, -1.0, -0.0], dtype=np.float32)
    assert rs.ranked(v, np.arange(7)).tolist() == [2, 4, 0, 1, 6, 5, 3]
    assert rs.ranked(v, np.arange(7)[::-1]).tolist() == [4, 2, 6, 1, 0, 5, 3]


def test_hash_is_the_64_bit_polynomial():
    toks = [5, 0, 4098, 7]
    h = 0
    for k in toks:
        h = (h * 0x100000001b3 + k + 1) % 2 ** 64
    assert rs.seq_hash(toks) == h
    lo, hi = rs.hash_words(h)
    assert rs.row_hash(np.array([4, lo, hi], dtype=np.int32)) == h


def _row_logits(t, seq, V):
    """A deterministic logit row for frame t and hypothesis seq (the joint's output depends on both)."""
    rng = np.random.default_rng(abs(hash((t,) + seq)) % 2 ** 32)
    return (rng.standard_normal(V) * 1.5).astype(np.float32)


def _select_frames(V, W, T, merge, blank=0):
    """T frames of BEAM_SELECT from the empty hypothesis through the restatement; returns the beam per frame as
    {seq: log p} and the buffers of the last frame."""
    R, LS = W, T + 3
    seq = np.zeros((2, R, LS), dtype=np.int32)
    hist = np.zeros(3 * T * W + T, dtype=np.int32)
    y = np.full(R, -np.inf, dtype=np.float32)
    y[0] = 0.0
    beams = []
    for t in range(T):
        _, _, _, hl = rs.hist_views(hist, 1, T, W)
        live = 1 if t == 0 else int(hl[0, t - 1])
        x = np.zeros((R, V), dtype=np.float32)
        for q in range(live):
            x[q] = _row_logits(t, tuple(seq[t & 1, q, 3:3 + seq[t & 1, q, 0]]), V)
        d = dict(x1=x, y=y, tok_in=np.array([T], dtype=np.int32), tok_out=np.zeros(R, dtype=np.int32),
                 src=np.zeros(R, dtype=np.int32), seq_in=seq[t & 1], seq_out=seq[(t + 1) & 1], hist=hist)
        rs.beam_select(dict(S=1, N=V, aux=W, aux2=blank, flags=16 if merge else 0, hist_ld=T, hist_col=t), d)
        n = int(hl[0, t])
        beams.append({tuple(seq[(t + 1) & 1, s, 3:3 + seq[(t + 1) & 1, s, 0]]): float(y[s]) for s in range(n)})
    return beams


def _enumerate(V, T, blank=0):
    """Every hypothesis after each frame with its log p summed over all alignments (at most one symbol per frame)."""
    out, cur = [], {(): 0.0}
    for t in range(T):
        nxt = {}
        for s, lp in cur.items():
            x = _row_logits(t, s, V).astype(np.float64)
            ls = x - np.logaddexp.reduce(x)
            for k in range(V):
                s2 = s + ((k,) if k != blank else ())
                nxt[s2] = np.logaddexp(nxt.get(s2, -np.inf), lp + ls[k])
        out.append(nxt)
        cur = nxt
    return out


@pytest.mark.parametrize("V,T", [(2, 5), (3, 4), (4, 3)])
def test_select_merge_equals_enumeration_without_pruning(V, T):
    """W above the number of hypotheses: the merged beam holds every token sequence with its total log p."""
    W = sum(V ** k for k in range(T + 1))
    for got, want in zip(_select_frames(V, W, T, merge=True), _enumerate(V, T)):
        assert set(got) == set(want)
        for s, v in want.items():
            assert abs(got[s] - v) <= 1e-5 * (1 + abs(v)), (s, got[s], v)


@pytest.mark.parametrize("V,W", [(3, 2), (4, 5), (2, 3)])
def test_select_pruned_frame_is_the_top_w(V, W):
    """Each frame of a pruned search: the survivors are the top W candidates of the previous beam by (value, flat
    index), merged by sequence, as brute force over the candidates states it."""
    T = 4
    beams = _select_frames(V, W, T, merge=True)
    prev = {(): 0.0}
    for t, got in enumerate(beams):
        cands = []
        for q, (s, lp) in enumerate(prev.items()):
            x = _row_logits(t, s, V).astype(np.float64)
            ls = x - np.logaddexp.reduce(x)
            cands += [(lp + ls[k], -(q * V + k), s + ((k,) if k else ())) for k in range(V)]
        top = sorted(cands, reverse=True)[:W]
        want = {}
        for v, _, s in top:
            want[s] = np.logaddexp(want.get(s, -np.inf), v)
        assert set(got) == set(want), t
        for s in want:
            assert abs(got[s] - want[s]) <= 1e-5 * (1 + abs(want[s]))
        prev = got


@pytest.mark.parametrize("V,W,T", [(3, 4, 5), (5, 8, 6), (4, 64, 4), (2, 1, 6)])
def test_ctc_beam_frames_equal_the_oracle(V, W, T):
    """CTC_BEAM over T frames, one frame per phase and all in one phase, against prefix_beam_search in fp32:
    the same prefixes in the same slots, pb / pnb within the log-add rounding."""
    rng = np.random.default_rng(V * 100 + W + T)
    y = rng.standard_normal((T, V)) * 2
    y = (y - np.logaddexp.reduce(y, axis=1, keepdims=True)).astype(np.float32)
    _, _, beam, _ = prefix_beam_search(y, T, W, 0, dtype=np.float32)
    for n in (1, T):
        R, LS = W, T + 5
        c = np.zeros((2, 3, R), dtype=np.float32)
        c[0, :2] = -np.inf
        c[0, 0, 0] = 0.0
        d = dict(x1=y[None], tok_in=np.array([T], dtype=np.int32), c=c, seq_out=np.zeros((2, R, LS), dtype=np.int32),
                 y=np.full(R, -np.inf, dtype=np.float32), src=np.zeros(R, dtype=np.int32),
                 hist=np.zeros(3 * T * W + T, dtype=np.int32))
        for t0 in range(0, T, n):
            rs.ctc_beam(dict(S=1, N=V, aux=W, aux2=0, flags=0, hist_ld=T, hist_col=t0, ldw1=n, K1=LS), d)
        _, _, _, hl = rs.hist_views(d["hist"], 1, T, W)
        live = int(hl[0, T - 1])
        rows = d["seq_out"][T & 1]
        got = [(tuple(rows[s, 5:5 + rows[s, 0]]), d["c"][T & 1, 0, s], d["c"][T & 1, 1, s]) for s in range(live)]
        assert [g[0] for g in got] == [b[0] for b in beam]
        for (_, pb, pnb), (_, opb, opnb, _) in zip(got, beam):
            for a, b in ((pb, opb), (pnb, opnb)):
                assert (a == b == -np.inf) or abs(a - b) <= 1e-5 * (1 + abs(b))
        for s, (tk, _, _) in enumerate(got):                  # the row head: hash of the prefix and of its parent
            assert rs.row_hash(rows[s]) == rs.seq_hash(tk) and (not tk or rs.row_hash(rows[s], 3) == rs.seq_hash(tk[:-1]))


def test_final_against_brute_force():
    """BEAM_FINAL on a random history: each rank's walk, frames and -value equal a direct back-pointer walk of the
    slots sorted by (value - pending) with the lowest slot on ties."""
    rng = np.random.default_rng(3)
    S, W, T, N, K = 2, 6, 5, 4, 2
    hist = np.zeros(3 * S * T * W + S * T, dtype=np.int32)
    hp, ht, _, hl = rs.hist_views(hist, S, T, W)
    hp[:] = rng.integers(0, W, size=hp.shape)
    ht[:] = rng.integers(0, 4, size=ht.shape)
    hl[:] = W
    y = (0.5 * rng.integers(-4, 1, size=S * W)).astype(np.float32)
    st = rng.integers(0, 3, size=(2, S * W)).astype(np.int32)
    pend = np.array([0.0, 0.5, 1.0], dtype=np.float32)
    d = dict(y=y, hist=hist, tok_out=np.zeros(S * N * T, dtype=np.int32), y2=np.zeros(S * N, dtype=np.float32),
             seq_out=np.zeros(S * N * T, dtype=np.int32), tok_out2=np.zeros(S, dtype=np.int32), ctx_pending=pend,
             ctx_state=st)
    rs.beam_final(dict(S=S, aux=W, aux2=0, hist_ld=T, ldy=T, K1=N, ldw2=K, flags=2048, hist_col=1), d)
    for b in range(S):
        val = [float(y[b * W + s]) - float(pend[st[1, b * W + s]]) for s in range(W)]
        order = sorted(range(W), key=lambda s: (-val[s], s))[:N]
        for n, s0 in enumerate(order):
            toks, frs, s = [], [], s0
            for t in range(T - 1, -1, -1):
                if ht[b, t, s]:
                    toks.insert(0, int(ht[b, t, s]))
                    frs.insert(0, t // K)
                s = hp[b, t, s]
            row = d["tok_out"][(b * N + n) * T:(b * N + n + 1) * T]
            assert row.tolist() == [-1] * (T - len(toks)) + toks
            assert d["seq_out"][(b * N + n) * T:(b * N + n + 1) * T].tolist() == [-1] * (T - len(toks)) + frs
            assert d["y2"][b * N + n] == -val[s0]
        assert d["tok_out2"][b] == N


@pytest.mark.parametrize("flush", [False, True])
def test_commit_keeps_every_sequence(flush):
    """BEAM_COMMIT: committed tokens + each kept slot's new suffix is the slot's old suffix; the common prefix is the
    longest one; a collapse keeps the first best slot alone."""
    rng = np.random.default_rng(5 + flush)
    S, W, P, T, HEAD = 3, 5, 12, 2, 3
    LS = P + HEAD
    seq = np.full((S * W, LS), -9, dtype=np.int32)
    hist = np.zeros(3 * S * T * W + S * T, dtype=np.int32)
    _, _, _, hl = rs.hist_views(hist, S, T, W)
    old = {}
    for b in range(S):
        hl[b, T - 1] = W
        pre = list(rng.integers(0, 9, size=3))
        for s in range(W):
            tk = pre + list(rng.integers(0, 9, size=rng.integers(0, 6)))
            seq[b * W + s, :HEAD + len(tk)] = [len(tk), 11, 12] + tk
            old[b * W + s] = tk
    y = np.array([0.0, -1.0, 0.0, -2.0, -3.0] * S, dtype=np.float32)
    d = dict(y=y, hist=hist, seq_in=seq, seq_out=np.full_like(seq, -9), tok_out=np.full(S * P, -9, dtype=np.int32),
             tok_out2=np.zeros(2 * S, dtype=np.int32), src=np.zeros(S * W, dtype=np.int32))
    rs.beam_commit(dict(S=S, N=P, aux=W, aux2=P - 3, K1=LS, K2=0, hist_ld=T, flags=128 if flush else 0), d)
    for b in range(S):
        n, col = int(d["tok_out2"][b]), bool(d["tok_out2"][S + b])
        com = d["tok_out"][b * P:b * P + n].tolist()
        assert col == flush
        keep = [0] if col else list(range(W))
        for s in keep:
            r = b * W + s
            src = b * W + (0 if col else s)                    # the first of the tied best slots 0 and 2
            suf = d["seq_out"][r, HEAD:HEAD + d["seq_out"][r, 0]].tolist()
            assert com + suf == old[src] and d["seq_out"][r, 1:3].tolist() == [11, 12]
        if not col:
            seqs = [old[b * W + s] for s in range(W)]
            c = len(com)
            assert all(x[:c] == com for x in seqs)
            assert min(map(len, seqs)) == c or len({x[c] for x in seqs}) > 1
