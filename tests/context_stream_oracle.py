"""CPU restatement of contextual biasing in the streaming beams (decode.cu flag 2048 in BEAM_COMMIT; the engines
StreamBeamEngine and CTCStreamBeamEngine with ``context``).

- ``beam_commit``: BEAM_COMMIT's contract with the flag, on the device layout (tests/beam_phases_restate.py's
  beam_commit with the collapse ranked by y - pending[state] from parity 1, the kept slot keeping its y, and every
  slot's state moved to parity 0 by the gather sources);
- ``transducer_stream``: one stream of the transducer beam (K = 1, tests/context_oracle.transducer_nbest's frame:
  f = f_LM + delta for k != blank) with the chunk-end rule, a collapse picking the best of value - pending[state];
- ``CTCContextStream``: tests/ctc_stream_beam_oracle.py's streaming CTC restatement with f' = (f + LM term) + delta for
  an extension, the state carried by each prefix, and collapses and the flush by (pb (+) pnb) + f - pending[state]."""
import numpy as np
import torch

from oracle import model_torch as mt
from tests import beam_multi_symbol_oracle as bo
from tests import beam_phases_restate as rs
from tests.ctc_beam_oracle import logadd
from tests.ctc_stream_beam_oracle import CTCStreamBeamRestatement, common_prefix
from tests.lm_oracle import fusion_term, lm_step

f32 = np.float32


def beam_commit(p, d):
    """BEAM_COMMIT with flags 2048.  d: rs.beam_commit's buffers plus ctx_pending [n] and ctx_state [2, R]."""
    S, W = p["S"], p["aux"]
    y0 = d["y"].copy()
    st = d["ctx_state"]
    with np.errstate(invalid="ignore"):
        d["y"] = (y0 - d["ctx_pending"][st[1]]).astype(f32)    # what a collapse ranks by
    rs.beam_commit(p, d)
    y = y0.copy()
    for b in range(S):
        r0 = b * W
        if d["tok_out2"][S + b]:                                  # the kept slot keeps its own y
            y[r0 + 1:r0 + W] = rs.NINF
            y[r0] = y0[d["src"][r0]]
    d["y"] = y
    st[0] = st[1][d["src"]]


@torch.no_grad()
def transducer_stream(sd, h_enc, chunk_out, W, max_pending, graph, merge=True, blank=mt.NUL, lm_sd=None,
                      lm_weight=0.0, length_bonus=0.0, lm_bos=1):
    """One stream: encoder output h_enc [T', E] cut into chunks of chunk_out frames.  -> (committed tokens per chunk,
    the flushed rest, -(value - pending) of the flushed hypothesis, forced collapses)."""
    V = sd["joint.joint.2.weight"].shape[0]
    nxt, dlt, pend = graph.next, torch.from_numpy(graph.delta), graph.pending
    hyps = [dict(bo.start(sd, lm_sd, lm_bos), cs=0)]
    done, t, per, collapses = 0, 0, [], 0

    def value(h):
        return f32(float(h["lp"])) - pend[h["cs"]]

    def commit(n_out, flush=False):
        nonlocal hyps, done, collapses
        pend_seqs = [tuple(h["seq"][done:]) for h in hyps]
        c = len(common_prefix(pend_seqs))
        out = list(pend_seqs[0][:c])
        done += c
        if flush or max(len(s) for s in pend_seqs) - c > max_pending - n_out:
            best = max(range(len(hyps)), key=lambda i: (value(hyps[i]), -i))
            out += hyps[best]["seq"][done:]
            done = len(hyps[best]["seq"])
            hyps = [hyps[best]]
            collapses += not flush
        return out

    for n_out in chunk_out:
        out = commit(n_out)
        for _ in range(n_out):
            cand = []
            for qi, hy in enumerate(hyps):
                a = torch.log_softmax(mt.joint(sd, h_enc[t][None], hy["x"][None])[0], 0)
                d = dlt[hy["cs"]].clone()
                d[blank] = 0.0
                f = fusion_term(hy["llp"].to(a.dtype), V, blank, lm_weight, length_bonus) + d if lm_sd is not None \
                    else d
                lp = (a + f) + hy["lp"]
                cand += [(float(lp[k]), qi, k, lp[k]) for k in range(V)]
            cand.sort(key=lambda c: (-c[0], c[1], c[2]))
            new, seen = [], {}
            for _, qi, k, lpk in cand[:W]:
                hy = hyps[qi]
                seq = hy["seq"] + [k] if k != blank else hy["seq"]
                if merge and tuple(seq) in seen:
                    seen[tuple(seq)]["lp"] = torch.logaddexp(seen[tuple(seq)]["lp"], lpk)
                    continue
                nh = dict(hy, seq=seq, lp=lpk)
                if k != blank:
                    nx, (h2, c2) = mt.decoder(sd, torch.full((1, 1), k), (hy["h"][:, None], hy["c"][:, None]))
                    nh.update(x=nx[0, 0], h=h2[:, 0], c=c2[:, 0], cs=int(nxt[hy["cs"], k]))
                    if lm_sd is not None:
                        llp, (lh, lc) = lm_step(lm_sd, torch.tensor([k]), (hy["lh"][:, None], hy["lc"][:, None]))
                        nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
                seen[tuple(seq)] = nh
                new.append(nh)
            hyps = new
            t += 1
        per.append(out + commit(n_out))
    rest = commit(0, flush=True)
    return per, rest, -float(value(hyps[0])), collapses


class CTCContextStream(CTCStreamBeamRestatement):
    """CTCStreamBeamRestatement with the ContextGraph ``graph``: every hypothesis carries its automaton state ``cs``;
    an extension by c != blank adds delta[cs, c] after the LM term and moves the state to next[cs, c]; a stay keeps
    both.  ``scores()`` (the collapse ranking and the flush) is (pb (+) pnb) + f - pending[cs]."""

    def __init__(self, W, graph, **kw):
        super().__init__(W, **kw)
        self.graph = graph
        self.hyps[0]["cs"] = 0

    def frame(self, yt):
        dt, blank, hyps = self.dtype, self.blank, self.hyps
        yt = np.asarray(yt, dtype=dt)
        V = yt.shape[0]
        ninf = dt(-np.inf)
        k_all = np.arange(V)
        nxt, dlt = self.graph.next, self.graph.delta.astype(dt)
        index = {h["seq"]: q for q, h in enumerate(hyps)}
        nq = len(hyps)
        vals, pnbx, fx = (np.empty((nq, V), dtype=dt) for _ in range(3))
        valid = np.ones((nq, V), dtype=bool)
        A = [logadd(h["pb"], h["pnb"]) for h in hyps]
        for q, h in enumerate(hyps):
            e = h["seq"][-1] if h["seq"] else -1
            pnbx[q] = np.where(k_all == e, h["pb"], A[q]) + yt
            if self.lm_sd is not None:
                fz = fusion_term(h["llp"].to(torch.float64 if dt == np.float64 else torch.float32), V, blank,
                                 self.lm_weight, self.length_bonus, self.lm_map).numpy().astype(dt)
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
            stay.append((dt(pb2), dt(pnb2)))
            vals[q, blank] = logadd(pb2, pnb2) + h["f"]
        flat = np.arange(nq * V)
        v, ok = vals.reshape(-1), valid.reshape(-1)
        flat, v = flat[ok], v[ok]
        v = np.where(v == 0, dt(0.0), v)
        tmap = None if self.lm_sd is None else (torch.arange(V) if self.lm_map is None
                                                else torch.as_tensor(self.lm_map).long())
        new = []
        for i in np.lexsort((flat, -v))[:self.W]:
            q, k = divmod(int(flat[i]), V)
            h = hyps[q]
            if k == blank:
                nh = dict(h, pb=stay[q][0], pnb=stay[q][1])
            else:
                nh = dict(h, seq=h["seq"] + (k,), pb=ninf, pnb=pnbx[q, k], f=fx[q, k], cs=int(nxt[h["cs"], k]))
                if tmap is not None and int(tmap[k]) >= 0:
                    llp, (lh, lc) = lm_step(self.lm_sd, tmap[k:k + 1], (h["lh"][:, None], h["lc"][:, None]))
                    nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
            new.append(nh)
        self.hyps = new

    def scores(self):
        pend = self.graph.pending.astype(self.dtype)
        return [logadd(h["pb"], h["pnb"]) + h["f"] - pend[h["cs"]] for h in self.hyps]
