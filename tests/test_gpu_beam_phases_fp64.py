"""One-phase parity of the beam phases of the decode program (csrc/decode.cu): BEAM_SELECT, CTC_BEAM, BEAM_COMMIT,
BEAM_FINAL and GATHER, each run alone as a one-phase program on planted inputs and compared, whole buffer by whole
buffer, with the host restatement tests/beam_phases_restate.py.

Two regimes.
  exact    logit rows whose maximum 0 is unique and whose other entries are multiples of 1/4 at or below -110 (so
           expf underflows to 0 and the log-softmax statistics are exactly (0, 0)), LM rows likewise, dyadic log p,
           lm_weight, length_bonus, context increments and pending bonuses, and for CTC_BEAM slot states with pb or
           pnb at -inf and levels 120 apart (so logaddexp_ returns its larger operand).  Every fp32 operation of the
           phase is then exact and every output word must equal the restatement's bit for bit: values, tokens,
           parents, gather sources, the four history planes, every sequence-row word, both context parities, CTC's
           pb | pnb | f, BEAM_FINAL's ids, frames, -value and count, BEAM_COMMIT's tokens, counts, collapse flags,
           last token and shifted rows.  The one exception is a value that folds two candidates by a log-add whose
           expf term does not underflow (a merge of near-equal values): it must lie within FOLD_ULP ulp of the
           log1pf term and of the result, FOLD_ULP 2^-24 (1 + |value|) (the sum can cancel: -0.5 (+) -0.5 = 0.19).
  general  Gaussian, peaked and near-uniform logits into BEAM_SELECT, against fp64 candidate values with first-order
           bars (the max and log-sum-exp move by about V u, plus the three roundings of ((z - m) - ls) + lp), the
           selection checked by the ambiguity rule of test_gpu_beam_engine._check_frame.

Planted in the exact regime: exact value ties across slots and tokens, -0 against +0, fewer finite candidates than
W, a pair of rows whose stored (len, hash) words match but whose tokens differ (must not merge), frozen utterances
beside live ones, several-symbol rounds at j = 0, a middle round and K-1 with open and closed slots mixed, a round
where no slot is open, streaming rows with a short stored suffix, BEAM_COMMIT's empty shortest suffix, a suffix of
exactly aux2 tokens against aux2 + 1, a collapse between tied values.

Every output buffer is filled with a sentinel (NaN bits, or -7 / -9 for int words) before each run, so a word the
phase should not write, or fails to write, shows.  Each program runs at max_ctas in {0, 1, 3, 17} and through every
decode entry that compiles the phase, and all runs must give the same bits.  pytest -s prints the worst fold err /
bar and the general regime's worst err / bar for each shape."""
import numpy as np
import pytest
import torch

from tests import beam_phases_restate as rs
from tests.test_gpu_beam_engine import _check_frame

pytestmark = pytest.mark.gpu

DEV = "cuda"
CTAS = (0, 1, 3, 17)
ALL = ("eb_decode_run", "eb_decode_run_ctc", "eb_decode_run_gru_rnnt", "eb_decode_run_ctc_stream",
       "eb_decode_run_ctc_stream_beam")
ENTRIES = dict(select=ALL[:3], final=ALL[:3], ctc=("eb_decode_run_ctc", "eb_decode_run_ctc_stream_beam"),
               commit=ALL, gather=ALL)
FOLD_ULP = 4
U32 = 2.0 ** -24
F_MERGE, F_LM, F_STREAM, F_FLUSH, F_ROUNDS, F_CONTEXT = 16, 32, 64, 128, 512, 2048
NAN_BITS = -0x400000          # 0xffc00000: a NaN as an int32 word


# ---- running one-phase programs --------------------------------------------------------------------------------------
def _launch(entry, ph, max_ctas):
    from edgedict_b200._lib import check, lib
    from edgedict_b200.stream_engine import EbPhase
    prog = torch.frombuffer(bytearray(bytes((EbPhase * 1)(ph))), dtype=torch.uint8).to(DEV)
    bar = torch.zeros(64, dtype=torch.int32, device=DEV)
    check(getattr(lib(), entry)(prog.data_ptr(), 1, bar.data_ptr(), max_ctas,
                                torch.cuda.current_stream().cuda_stream), entry)
    torch.cuda.synchronize()


def _words(a):
    return a.view(np.int32) if a.dtype == np.float32 else a


def _run_all(kind, p, host):
    """Build the phase from the fields p and the host buffers ``host`` (name -> numpy array; EbPhase pointer fields
    by name, plus ctx_* for the context descriptor), run it through every entry of ENTRIES[kind] at every max_ctas
    from the same initial buffers, check that all runs agree bitwise and return the outputs as numpy arrays."""
    from edgedict_b200.stream_engine import EbPhase, _ptr
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in host.items() if v is not None}
    fields = dict(p)
    for k, t in dev.items():
        if not k.startswith("ctx_"):
            fields[k] = _ptr(t)
    if "ctx_next" in dev:                                    # the descriptor context_program uploads
        st = dev["ctx_state"]
        desc = torch.tensor([dev["ctx_next"].data_ptr(), dev["ctx_delta"].data_ptr(), dev["ctx_pending"].data_ptr(),
                             st[0].data_ptr(), st[1].data_ptr()], dtype=torch.int64).to(DEV)
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
                assert bad.size == 0, "%s: %s max_ctas=%d differs from %s max_ctas=0 at %s" % (
                    k, entry, mc, ENTRIES[kind][0], bad[:4].tolist())
    return first


def _compare(name, got, want, fold_rows=None):
    """Every buffer bitwise, except the float words listed by fold_rows (per buffer name: flat indices), values that
    went through a log-add whose expf term does not underflow: within FOLD_ULP ulp of the log1pf term and of the
    result, FOLD_ULP 2^-24 (1 + |value|).  Returns the worst err / bar of those."""
    worst = 0.0
    for k, w in want.items():
        if w is None or k not in got:
            continue
        g = got[k]
        diff = _words(g).ravel() != _words(w).ravel()
        tol = (fold_rows or {}).get(k)
        if tol is not None and len(tol):
            idx = np.asarray(sorted(tol), dtype=np.int64)
            gi, wi = (a.ravel().view(np.float32)[idx].astype(np.float64) for a in (g, w))
            fin = np.isfinite(wi)
            with np.errstate(invalid="ignore"):               # -inf - -inf: the bitwise branch decides
                err = np.where(fin, np.abs(gi - wi), np.where(gi == wi, 0.0, np.inf))
            ratio = err / (FOLD_ULP * U32 * (1 + np.abs(np.where(fin, wi, 0.0))))
            assert (ratio <= 1).all(), "%s: %s folded values beyond the bar at %s: device %s, restatement %s" % (
                name, k, idx[ratio > 1][:4].tolist(), gi[ratio > 1][:4].tolist(), wi[ratio > 1][:4].tolist())
            worst = max(worst, float(ratio.max()))
            diff[idx] = False
        bad = np.flatnonzero(diff)
        assert bad.size == 0, "%s: %s differs at flat %s: device %s, restatement %s" % (
            name, k, bad[:6].tolist(), g.ravel()[bad[:6]].tolist(), w.ravel()[bad[:6]].tolist())
    return worst


def _restate(fn, p, host):
    d = {k: (None if v is None else v.copy()) for k, v in host.items()}
    folded = fn(p, d)
    return d, folded


# ---- planted inputs ----------------------------------------------------------------------------------------------------
def _logit_rows(rng, n, V, ninf_frac=0.0):
    """Rows with a unique maximum 0 and the other entries multiples of 1/4 in [-126, -110] (many exact ties)."""
    x = -(110.0 + 0.25 * rng.integers(0, 65, size=(n, V))).astype(np.float32)
    if ninf_frac:
        x[rng.random((n, V)) < ninf_frac] = -np.inf
    x[np.arange(n), rng.integers(0, V, size=n)] = 0.0
    return x


def _distinct_seqs(rng, n, V, blank, maxlen, tree=True):
    """n distinct token sequences (no blank), about half of them one token longer than an earlier one (so blank and
    non-blank extensions meet).  Fewer when V and maxlen admit fewer."""
    toks = [k for k in range(V) if k != blank]
    out, seen = [], set()
    for _ in range(20 * n + 20):
        if len(out) == n:
            break
        if tree and out and rng.random() < 0.5:
            base = out[rng.integers(len(out))]
            s = base + (int(rng.choice(toks)),) if len(base) < maxlen else base
        else:
            s = tuple(int(v) for v in rng.choice(toks, size=rng.integers(0, maxlen + 1)))
        if s not in seen:
            seen.add(s)
            out.append(s)
    return out


def _ctx_tables(rng, V, n_states=7):
    return dict(ctx_next=rng.integers(0, n_states, size=(n_states, V)).astype(np.int32),
                ctx_delta=(0.5 * rng.integers(-8, 9, size=(n_states, V))).astype(np.float32),
                ctx_pending=(0.25 * rng.integers(0, 17, size=n_states)).astype(np.float32)), n_states


def _hist(S, T, W):
    h = np.full(3 * S * T * W + S * T, -7, dtype=np.int32)
    h[2 * S * T * W:3 * S * T * W] = NAN_BITS
    return h


# ---- BEAM_SELECT ---------------------------------------------------------------------------------------------------------
# (S, W, V, flags, live, mode); live: the live slot count of every utterance (capped at W), mode: "mid" a frame t > 0,
# "t0" the first frame, "frozen" some utterances past their length, "ninf" -inf logits (fewer finite candidates than W),
# "r0" / "rmid" / "rlast" several-symbol rounds j = 0, 1, K-1 of K = 3, "rdone" a round with no open slot in one row.
SELECT_CASES = [
    (3, 1, 2, 0, 1, "mid"), (3, 2, 3, F_MERGE, 2, "mid"), (5, 31, 33, F_MERGE, 31, "mid"),
    (4, 32, 33, F_MERGE | F_LM, 7, "frozen"), (4, 33, 1024, F_MERGE | F_CONTEXT, 33, "mid"),
    (3, 255, 2, F_MERGE, 200, "mid"), (3, 256, 3, F_MERGE | F_LM | F_CONTEXT, 256, "ninf"),
    (3, 257, 33, 0, 257, "mid"), (2, 511, 1024, F_MERGE | F_STREAM, 300, "mid"),
    (2, 1000, 4099, F_MERGE | F_LM, 1000, "mid"), (2, 1024, 33, F_MERGE | F_CONTEXT | F_STREAM, 1024, "t0"),
    (2, 1024, 3, F_MERGE, 5, "mid"), (150, 4, 33, F_MERGE | F_CONTEXT, 4, "frozen"),
    (4, 8, 33, F_MERGE | F_ROUNDS, 8, "r0"), (4, 16, 33, F_MERGE | F_ROUNDS | F_LM | F_CONTEXT, 16, "rmid"),
    (4, 33, 33, F_MERGE | F_ROUNDS, 30, "rlast"), (4, 8, 3, F_MERGE | F_ROUNDS | F_CONTEXT, 8, "rdone"),
    (3, 256, 1024, F_MERGE | F_ROUNDS | F_STREAM, 256, "rmid"), (2, 1024, 33, F_ROUNDS | F_MERGE, 1024, "rlast"),
]


def _select_inputs(S, W, V, flags, live, mode, seed):
    rng = np.random.default_rng(seed)
    blank, R = int(rng.integers(0, V)), S * W
    multi, stream = flags & F_ROUNDS, flags & F_STREAM
    K = 3 if multi else 1
    Tf = 8                                                    # frames
    t = 0 if mode == "t0" else 5
    j = dict(r0=0, rmid=1, rlast=2, rdone=1).get(mode, 0)
    col, T = (t * K + j, Tf * K) if multi else (t, Tf)
    maxlen = 5 if stream else col                             # a hypothesis holds at most one token per column
    LS = maxlen + 8 if stream else T + 3                      # a streaming row: stride K1, the stored suffix only
    y = np.full(R, -np.inf, dtype=np.float32)
    seq = np.full((R, LS), -9, dtype=np.int32)
    hist = _hist(S, T, W)
    _, _, _, hlive = rs.hist_views(hist, S, T, W)
    tok_out = np.full(R, -9, dtype=np.int32)
    x = _logit_rows(rng, R, V, ninf_frac=0.9 if mode == "ninf" else 0.0)
    nl = []
    for b in range(S):
        first = t == 0 and not stream and not multi
        seqs = [()] if first else _distinct_seqs(rng, min(live, W), V, blank, maxlen)
        n = len(seqs)
        nl.append(n)
        h0 = int(rng.integers(0, 2 ** 63)) if stream else 0  # the committed prefix's hash
        index = {sq: s for s, sq in enumerate(seqs)}
        for s, sq in enumerate(seqs):
            seq[b * W + s, :3 + len(sq)] = [len(sq)] + rs.hash_words(rs.seq_hash(sq, h0)) + list(sq)
            q1 = index.get(sq[:-1]) if sq else None
            if q1 is not None:                                # q1 + [k] and the blank extension of q meet: merges
                for row, top in ((b * W + q1, sq[-1]), (b * W + s, blank)):
                    x[row] = np.where(x[row] == 0, np.float32(-110), x[row])
                    x[row, top] = 0.0
        y[b * W:b * W + n] = -0.25 * rng.integers(0, 33, size=n)
        y[b * W] = 0.0
        if n > 1:
            y[b * W + 1] = -0.0                               # -0 against +0
        if multi:
            hlive[b, T - 1] = n
            if j:                                             # open (non-blank last round) and closed slots mixed
                tok_out[b * W:b * W + n] = np.where(rng.random(n) < 0.5, blank, (blank + 1) % V)
                if mode == "rdone" and b == 1:
                    tok_out[b * W:b * W + n] = blank
        elif t > 0:
            hlive[b, t - 1] = n
        elif stream:
            hlive[b, T - 1] = n
        # a stored (len, hash) collision: slot c's words equal those of slot a's extension by k, its tokens differ.
        # c has no live parent or child, so no true merge depends on its hash: to the phase this is a 64-bit collision.
        lone = [c for c, sq in enumerate(seqs) if sq and sq[:-1] not in index and
                not any(o[:-1] == sq for o in seqs if o)]
        if flags & F_MERGE and lone and V >= 3:
            c = lone[0]
            a = next((a for a, sq in enumerate(seqs) if len(sq) == len(seqs[c]) - 1), None)
            if a is not None:
                k = next(v for v in range(V) if v != blank)
                seq[b * W + c, 1:3] = rs.hash_words(rs.ext_hash(rs.row_hash(seq[b * W + a]), k))
                for row, top in ((b * W + a, k), (b * W + c, blank)):   # both candidates at the top of the frame
                    x[row] = np.where(x[row] == 0, np.float32(-110), x[row])
                    x[row, top] = 0.0
                y[b * W + c] = 0.0
    frames = np.full(S, Tf, dtype=np.int32)
    if mode == "frozen":
        frames[::2] = rng.integers(0, t + 1, size=len(frames[::2]))
    if mode == "rmid" and S > 2:
        frames[2] = t                                         # frame ended for this row: frozen in a round
    host = dict(x1=x, y=y, tok_in=frames, tok_out=tok_out, src=np.full(R, -9, dtype=np.int32), seq_in=seq,
                seq_out=np.full((R, LS), -9, dtype=np.int32), hist=hist)
    p = dict(type=6, S=S, N=V, aux=W, aux2=blank, flags=flags, ldx1=V, hist_ld=T, hist_col=col, K1=LS if stream else 0,
             ldw2=K if multi else 0)
    if flags & F_LM:
        K2 = int(rng.integers(2, 40))
        host.update(x2=_logit_rows(rng, R, K2), fuse=np.array([0.5, 0.25], dtype=np.float32),
                    tok_map=np.where(rng.random(V) < 0.2, -1, rng.integers(0, K2, size=V)).astype(np.int32),
                    tok_out2=np.full(R, -9, dtype=np.int32))
        p.update(K2=K2, ldx2=K2)
    if flags & F_CONTEXT:
        tabs, ns = _ctx_tables(rng, V)
        host.update(tabs)
        st = np.full((2, R), -3, dtype=np.int32)
        pin = 0 if multi else t & 1
        st[pin] = rng.integers(0, ns, size=R)
        host["ctx_state"] = st
    return p, host, nl


@pytest.mark.parametrize("S,W,V,flags,live,mode", SELECT_CASES)
def test_beam_select_exact(S, W, V, flags, live, mode):
    p, host, nl = _select_inputs(S, W, V, flags, live, mode, seed=S * 7919 + W * 31 + V + flags + len(mode))
    got = _run_all("select", p, host)
    want, folded = _restate(rs.beam_select, p, host)
    n = S * p["hist_ld"] * W
    fold = dict(y=folded, hist=[2 * n + (r // W * p["hist_ld"] + p["hist_col"]) * W + r % W for r in folded])
    worst = _compare("select W=%d V=%d flags=%d %s" % (W, V, flags, mode), got, want, fold)
    _, _, _, hl = rs.hist_views(want["hist"], S, p["hist_ld"], W)
    merged = int(sum(min(W, nl[b] * V) - hl[b, p["hist_col"]] for b in range(S) if hl[b, p["hist_col"]] > 0))
    print("  select S=%d W=%d V=%d flags=%d %s: live %s.., %d merged candidates, %d folds, worst fold err/bar %.2f"
          % (S, W, V, flags, mode, nl[:3], merged, len(folded), worst))


# ---- CTC_BEAM ---------------------------------------------------------------------------------------------------------------
# (S, W, V, flags, live, frames per phase, mode): "levels" slot states 120 apart (merges exact), "ties" equal levels
# (ties across slots), "frozen" some utterances ending inside the phase
CTC_CASES = [
    (3, 1, 2, 0, 1, 1, "levels"), (3, 2, 3, 0, 2, 3, "levels"), (4, 31, 33, 0, 31, 1, "ties"),
    (4, 32, 33, F_LM, 32, 1, "levels"), (4, 33, 33, F_CONTEXT, 20, 3, "frozen"),
    (3, 255, 3, 0, 255, 1, "levels"), (3, 256, 1024, F_CONTEXT | F_LM, 256, 1, "levels"),
    (3, 257, 33, F_STREAM, 100, 3, "levels"), (2, 511, 1024, F_STREAM | F_CONTEXT, 511, 1, "levels"),
    (2, 1000, 4099, 0, 1000, 1, "ties"), (2, 1024, 33, F_STREAM, 1024, 2, "levels"),
    (2, 1024, 2, 0, 40, 3, "levels"), (140, 4, 33, F_CONTEXT, 4, 2, "frozen"),
]


def _ctc_inputs(S, W, V, flags, live, n, mode, seed):
    rng = np.random.default_rng(seed)
    blank, R = int(rng.integers(0, V)), S * W
    stream = flags & F_STREAM
    T, t0 = 8, 4
    maxlen = 5 if stream else t0                              # a prefix holds at most one token per frame
    LS = maxlen + n + 8 if stream else T + 5
    c = np.full((2, 3, R), np.nan, dtype=np.float32)
    seqs = np.full((2, R, LS), -9, dtype=np.int32)
    hist = _hist(S, T, W)
    _, _, _, hlive = rs.hist_views(hist, S, T, W)
    pin = t0 & 1
    y2 = np.full(S, -5, dtype=np.int32)
    nl = []
    for b in range(S):
        sq = _distinct_seqs(rng, min(live, W), V, blank, maxlen, tree=mode != "ties")
        nl.append(len(sq))
        hlive[b, t0 - 1] = len(sq)
        h0 = int(rng.integers(0, 2 ** 63)) if stream else 0
        y2[b] = int(rng.choice([k for k in range(V) if k != blank])) if stream and b % 2 == 0 else -1
        for s, tk in enumerate(sq):
            r = b * W + s
            ph = rs.seq_hash(tk[:-1], h0) if tk else int(rng.integers(0, 2 ** 63))
            seqs[pin, r, :5 + len(tk)] = [len(tk)] + rs.hash_words(rs.seq_hash(tk, h0)) + rs.hash_words(ph) + list(tk)
            level = 0.0 if mode == "ties" else -120.0 * s
            v = np.float32(level - 0.25 * rng.integers(0, 9))
            if rng.random() < 0.5:
                c[pin, :2, r] = (-np.inf, v)                 # pb = -inf: pb (+) pnb = pnb exactly
            else:
                c[pin, :2, r] = (v, -np.inf)
            c[pin, 2, r] = -0.25 * rng.integers(0, 5)
        # a stored parent-hash match whose tokens differ: slot 1 claims slot 0 as its parent
        # (its true parent is not live, so no true merge depends on the planted words)
        if len(sq) >= 2 and len(sq[1]) == len(sq[0]) + 1 and sq[1][:-1] not in sq:
            seqs[pin, b * W + 1, 3:5] = seqs[pin, b * W, 1:3]
    x = _logit_rows(rng, S * T, V).reshape(S, T, V)
    if n > 1 or mode == "levels":
        x[:, :, blank] = -np.inf                              # stays keep pb = -inf: the next frame stays exact
    frames = np.full(S, T, dtype=np.int32)
    if mode == "frozen":
        frames[::2] = t0 + rng.integers(0, n, size=len(frames[::2]))
    yv = np.full(R, np.nan, dtype=np.float32)
    host = dict(x1=x, tok_in=frames, c=c, seq_out=seqs, y=yv, src=np.full(R, -9, dtype=np.int32), hist=hist,
                y2=y2 if stream else None)
    p = dict(type=11, S=S, N=V, aux=W, aux2=blank, flags=flags, hist_ld=T, hist_col=t0, ldw1=n, K1=LS)
    if flags & F_LM:
        K2 = int(rng.integers(2, 40))
        host.update(x2=_logit_rows(rng, R, K2), fuse=np.array([0.5, -0.75], dtype=np.float32),
                    tok_map=np.where(rng.random(V) < 0.2, -1, rng.integers(0, K2, size=V)).astype(np.int32),
                    tok_out2=np.full(R, -9, dtype=np.int32))
        p.update(K2=K2, ldx2=K2)
    if flags & F_CONTEXT:
        tabs, ns = _ctx_tables(rng, V)
        host.update(tabs)
        st = np.full((2, R), -3, dtype=np.int32)
        st[pin] = rng.integers(0, ns, size=R)
        host["ctx_state"] = st
    return p, host, nl


@pytest.mark.parametrize("S,W,V,flags,live,n,mode", CTC_CASES)
def test_ctc_beam_exact(S, W, V, flags, live, n, mode):
    p, host, nl = _ctc_inputs(S, W, V, flags, live, n, mode, seed=S * 31 + W * 7 + V + flags + n)
    got = _run_all("ctc", p, host)
    want, folded = _restate(rs.ctc_beam, p, host)
    T, R = p["hist_ld"], S * W
    last_t = {}
    for t, r in folded:
        last_t.setdefault(r, set()).add(t)
    fold = dict(y=[r for r, ts in last_t.items() if max(ts) == p["hist_col"] + n - 1],
                hist=[2 * S * T * W + (r // W * T + t) * W + r % W for t, r in folded],
                c=[par * 3 * R + pl * R + r for t, r in folded for par in (0, 1) for pl in (0, 1)])
    worst = _compare("ctc W=%d V=%d flags=%d n=%d %s" % (W, V, flags, n, mode), got, want, fold)
    print("  ctc S=%d W=%d V=%d flags=%d frames/phase=%d %s: live %s.., %d folds, worst fold err/bar %.2f"
          % (S, W, V, flags, n, mode, nl[:3], len(folded), worst))


# ---- BEAM_COMMIT --------------------------------------------------------------------------------------------------------
# (S, W, head, live, mode): "common" a shared prefix, "empty" one live suffix empty, "edge" the longest suffix past the
# common prefix exactly aux2 on even streams and aux2 + 1 on odd ones, "flush" flags 128, "tie" a collapse between
# equal best values (and -0 / +0)
COMMIT_CASES = [
    (3, 1, 3, 1, "common"), (3, 2, 5, 2, "empty"), (5, 31, 3, 31, "edge"), (5, 32, 5, 32, "tie"),
    (4, 33, 3, 20, "flush"), (3, 255, 5, 255, "common"), (3, 256, 3, 256, "edge"), (3, 257, 5, 257, "tie"),
    (2, 511, 3, 511, "empty"), (2, 1000, 5, 1000, "edge"), (2, 1024, 3, 1024, "common"), (2, 1024, 5, 1024, "tie"),
    (150, 4, 5, 4, "edge"),
]


def _commit_inputs(S, W, head, live, mode, seed, with_last):
    rng = np.random.default_rng(seed)
    P, T, R = 24, 3, S * W
    LS = P + head
    aux2 = 10
    seq = np.full((R, LS), -9, dtype=np.int32)
    y = np.full(R, np.nan, dtype=np.float32)
    hist = _hist(S, T, W)
    _, _, _, hlive = rs.hist_views(hist, S, T, W)
    for b in range(S):
        n = min(live, W)
        hlive[b, T - 1] = n
        c0 = int(rng.integers(0, 6))
        pre = rng.integers(0, 50, size=c0)
        lens = rng.integers(c0, c0 + aux2 + 1, size=n)
        if mode == "empty":
            lens[n // 2] = 0
        if mode == "edge":
            lens[:] = np.minimum(lens, c0 + aux2 - 1)
            lens[n - 1] = c0 + aux2 + (b & 1)                 # exactly aux2 past the prefix, or aux2 + 1
        for s in range(n):
            toks = np.concatenate([pre, rng.integers(0, 50, size=P)])[:lens[s]]
            if s > 0 and lens[s] > c0:
                toks[c0] = 50 + s % 7                        # the suffixes part at c0 (some rows agree there)
            seq[b * W + s, :head + lens[s]] = np.concatenate(
                [[lens[s]], rng.integers(-2 ** 31, 2 ** 31, size=head - 1), toks]).astype(np.int32)
        y[b * W:b * W + n] = -0.25 * rng.integers(0, 40, size=n)
        if mode == "tie":                                     # the best value twice, -0 first
            y[b * W:b * W + n] -= 0.25
            y[b * W + n // 3], y[b * W + n - 1] = -0.0, 0.0
    host = dict(y=y, hist=hist, seq_in=seq, seq_out=np.full((R, LS), -9, dtype=np.int32),
                tok_out=np.full(S * P, -9, dtype=np.int32), tok_out2=np.full(2 * S, -9, dtype=np.int32),
                src=np.full(R, -9, dtype=np.int32),
                y2=np.where(np.arange(S) % 3 == 0, -1, 7).astype(np.int32) if with_last else None)
    p = dict(type=9, S=S, N=P, aux=W, aux2=aux2, K1=LS, K2=head if head != 3 else 0, hist_ld=T,
             flags=F_FLUSH if mode in ("flush", "tie") else 0)
    return p, host


@pytest.mark.parametrize("S,W,head,live,mode", COMMIT_CASES)
def test_beam_commit_exact(S, W, head, live, mode):
    for with_last in (False, True):
        p, host = _commit_inputs(S, W, head, live, mode, S * 13 + W + head + len(mode), with_last)
        got = _run_all("commit", p, host)
        want, _ = _restate(rs.beam_commit, p, host)
        _compare("commit W=%d head=%d %s" % (W, head, mode), got, want)
    col = want["tok_out2"][S:]
    print("  commit S=%d W=%d head=%d %s: committed %s.., collapsed %d of %d" % (
        S, W, head, mode, want["tok_out2"][:4].tolist(), int(col.sum()), S))
    if mode == "edge":
        assert col[0::2].sum() == 0 and col[1::2].all(), "the collapse bound"


# ---- BEAM_FINAL ----------------------------------------------------------------------------------------------------------
# (S, W, T, N (0: best only), K rounds per frame (0: 1), live, context)
FINAL_CASES = [
    (3, 1, 5, 0, 0, 1, False), (3, 2, 5, 2, 0, 2, True), (5, 31, 7, 5, 2, 31, False), (5, 32, 6, 32, 0, 32, True),
    (4, 33, 6, 33, 3, 20, False), (3, 255, 4, 40, 0, 255, True), (3, 256, 4, 256, 2, 256, False),
    (3, 257, 4, 3, 0, 257, True), (2, 511, 3, 511, 0, 511, False), (2, 1000, 3, 70, 2, 1000, True),
    (2, 1024, 3, 1024, 0, 1024, False), (2, 1024, 3, 1024, 3, 600, True), (150, 4, 5, 4, 2, 4, True),
    (3, 8, 0, 3, 0, 1, False),
]


@pytest.mark.parametrize("S,W,T,N,K,live,cx", FINAL_CASES)
def test_beam_final_exact(S, W, T, N, K, live, cx):
    rng = np.random.default_rng(S * 5 + W + T + N + K + live)
    blank, R, NB = 0, S * W, max(N, 1)
    hist = np.zeros(3 * S * T * W + S * T, dtype=np.int32)
    hpar, htok, hlp, hlive = rs.hist_views(hist, S, T, W)
    for b in range(S):
        prev = 1
        for t in range(T):
            nl = min(W, live) if t == T - 1 else int(rng.integers(1, W + 1))
            hpar[b, t] = rng.integers(0, prev, size=W)
            htok[b, t] = np.where(rng.random(W) < 0.4, blank, rng.integers(1, 900, size=W))
            hlive[b, t] = nl
            prev = nl
    y = np.full(R, -np.inf, dtype=np.float32)
    nlv = min(W, live) if T else 1
    for b in range(S):
        y[b * W:b * W + nlv] = -0.25 * rng.integers(0, 12, size=nlv)   # many ties
        y[b * W + nlv // 2] = -0.0
    ldy = T + 2
    host = dict(y=y, hist=hist, tok_out=np.full(S * NB * ldy, -9, dtype=np.int32),
                y2=np.full(S * NB, np.nan, dtype=np.float32),
                seq_out=np.full(S * NB * ldy, -9, dtype=np.int32) if N else None,
                tok_out2=np.full(S, -9, dtype=np.int32) if N else None)
    p = dict(type=8, S=S, aux=W, aux2=blank, hist_ld=T, ldy=ldy, K1=N, ldw2=K)
    if cx:
        tabs, ns = _ctx_tables(rng, 5)
        host.update(tabs)
        st = np.full((2, R), -3, dtype=np.int32)
        par = int(rng.integers(0, 2))
        st[par] = rng.integers(0, ns, size=R)
        host["ctx_state"] = st
        p.update(flags=F_CONTEXT, hist_col=par + 2)
    got = _run_all("final", p, host)
    want, _ = _restate(rs.beam_final, p, host)
    _compare("final W=%d T=%d N=%d K=%d" % (W, T, N, K), got, want)
    print("  final S=%d W=%d T=%d N=%d K=%d live=%d context=%s: best -value %s.." % (
        S, W, T, N, K, live, cx, want["y2"][:3].tolist()))


# ---- GATHER -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,N,aux,K2", [(1, 1, 1, 0), (33, 5, 4, 0), (257, 64, 2, 33), (1024, 3, 6, 640),
                                         (2048, 512, 4, 1)])
def test_gather_exact(R, N, aux, K2):
    rng = np.random.default_rng(R + N + aux + K2)
    x1 = rng.standard_normal(aux * R * N).astype(np.float32)
    x1[::7] = -0.0
    src = (np.arange(R) // 4 * 4 + rng.integers(0, 4, size=R)).clip(0, R - 1).astype(np.int32)   # within a beam
    src[::5] = np.arange(R)[::5]
    host = dict(x1=x1, y=np.full(aux * R * N + 3, np.nan, dtype=np.float32), src=src,
                x2=rng.standard_normal(R * K2).astype(np.float32) if K2 else None,
                y2=np.full(R * K2 + 3, np.nan, dtype=np.float32) if K2 else None)
    p = dict(type=7, S=R, N=N, aux=aux, K2=K2)
    got = _run_all("gather", p, host)
    want, _ = _restate(rs.gather, p, host)
    _compare("gather R=%d N=%d aux=%d K2=%d" % (R, N, aux, K2), got, want)


# ---- BEAM_SELECT, general regime ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,V,kind,merge", [(4, 33, "gauss", True), (32, 1024, "peaked", True),
                                             (64, 4099, "uniform", False), (256, 1024, "gauss", True),
                                             (1024, 1024, "peaked", False), (1000, 33, "uniform", True)])
def test_beam_select_general_fp64(W, V, kind, merge):
    """Logits N(0, 3^2), peaked (N(0, 1) with one entry +8 per row) or near-uniform (N(0, 1e-3^2)); slot log p from
    -20 to 0.  fp64 values and bars as test_beam_teacher_forced_fp64's log-softmax terms."""
    rng = np.random.default_rng(W + V + len(kind))
    S, blank, t, T = 3, 0, 2, 4
    R = S * W
    x = (rng.standard_normal((R, V)) * dict(gauss=3.0, peaked=1.0, uniform=1e-3)[kind]).astype(np.float32)
    if kind == "peaked":
        x[np.arange(R), rng.integers(0, V, size=R)] += 8.0
    y = np.full(R, -np.inf, dtype=np.float32)
    seq = np.full((R, T + 3), -9, dtype=np.int32)
    hist = _hist(S, T, W)
    _, _, _, hl = rs.hist_views(hist, S, T, W)
    allseqs = []
    for b in range(S):
        sq = _distinct_seqs(rng, W, V, blank, t)
        allseqs.append(sq)
        hl[b, t - 1] = len(sq)
        for s, tk in enumerate(sq):
            seq[b * W + s, :3 + len(tk)] = [len(tk)] + rs.hash_words(rs.seq_hash(tk)) + list(tk)
        y[b * W:b * W + len(sq)] = np.sort(-20 * rng.random(len(sq)))[::-1]
    host = dict(x1=x, y=y, tok_in=np.full(S, T, dtype=np.int32), tok_out=np.full(R, -9, dtype=np.int32),
                src=np.full(R, -9, dtype=np.int32), seq_in=seq, seq_out=np.full((R, T + 3), -9, dtype=np.int32),
                hist=hist)
    p = dict(type=6, S=S, N=V, aux=W, aux2=blank, flags=F_MERGE if merge else 0, ldx1=V, hist_ld=T, hist_col=t)
    got = _run_all("select", p, host)
    hpar, htok, hlp, hlv = rs.hist_views(got["hist"], S, T, W)
    worst, near = 0.0, 0
    for b in range(S):
        n = len(allseqs[b])
        z = x[b * W:b * W + n].astype(np.float64)
        zmax = z.max(1, keepdims=True)
        lse = zmax + np.log(np.exp(z - zmax).sum(1, keepdims=True))
        lp = y[b * W:b * W + n].astype(np.float64)[:, None]
        v = z - lse + lp
        beta = V * U32 * 2 + 3 * U32 * (np.abs(z - zmax) + np.abs(lse - zmax) + np.abs(lp)) + 4 * U32
        live = int(hlv[b, t])
        w, nt = _check_frame(v, beta, allseqs[b], W, merge, blank, hpar[b, t], htok[b, t],
                             hlp[b, t].astype(np.float64), live, "utterance %d" % b)
        worst, near = max(worst, w), near + nt
        assert np.array_equal(got["y"][b * W:b * W + live].view(np.int32), hlp[b, t, :live].view(np.int32))
    print("  select general W=%d V=%d %s merge=%s: worst err/bar %.3f, %d utterances with a near-tie" % (
        W, V, kind, merge, worst, near))
