"""CPU restatement of the streaming CTC prefix beam search of stream_engine.CTCStreamBeamEngine (decode.cu, CTC_BEAM with
flag 64, then BEAM_COMMIT on CTC rows at every chunk end), in fp64 or fp32, with the LM through tests/lm_oracle.py.

Each hypothesis holds its WHOLE prefix, so the last token of a prefix is always its real last token; the engine stores
only the suffix since the stream's last commit and carries the last committed token instead.  The per-frame rule is
tests/ctc_beam_oracle.py's prefix_beam_search, restated here one frame at a time so that a beam can be carried; the
chunk end is BEAM_COMMIT's rule: commit the longest common prefix of the live prefixes, and when an uncommitted suffix
still holds more than max_pending - n_out tokens (or on a flush) collapse the beam to its best hypothesis (highest
(pb (+) pnb) + f, lowest slot on ties) and commit all of it."""
import numpy as np
import torch

from tests.ctc_beam_oracle import logadd
from tests.lm_oracle import fusion_term, lm_prime, lm_step


def common_prefix(seqs):
    """The longest common prefix of the tuples ``seqs``."""
    n = min(len(s) for s in seqs)
    for i in range(n):
        if any(s[i] != seqs[0][i] for s in seqs):
            return seqs[0][:i]
    return seqs[0][:n]


class CTCStreamBeamRestatement:
    """One stream.  ``chunk(y)`` runs the frames y [n_out, V] and the chunk end, returning the committed tokens;
    ``flush()`` returns the rest of the best prefix and its -score.  ``hyps`` is the live beam in slot order (dicts
    with the whole prefix ``seq``, ``pb``, ``pnb``, ``f``), ``committed`` every token committed so far."""

    def __init__(self, W, blank=0, max_pending=64, dtype=np.float64, lm_sd=None, lm_weight=0.0, length_bonus=0.0,
                 lm_bos=1, lm_map=None):
        self.W, self.blank, self.P, self.dtype = W, blank, max_pending, dtype
        self.lm_sd, self.lm_weight, self.length_bonus, self.lm_map = lm_sd, lm_weight, length_bonus, lm_map
        self.hyps = [dict(seq=(), pb=dtype(0.0), pnb=dtype(-np.inf), f=dtype(0.0))]
        if lm_sd is not None:
            llp, (lh, lc) = lm_prime(lm_sd, lm_bos)
            self.hyps[0].update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
        self.committed = ()
        self.n_collapses = 0

    def frame(self, yt):
        """One frame of prefix_beam_search's rule over the carried beam."""
        dt, blank, hyps = self.dtype, self.blank, self.hyps
        yt = np.asarray(yt, dtype=dt)
        V = yt.shape[0]
        ninf = dt(-np.inf)
        k_all = np.arange(V)
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
            stay.append((dt(pb2), dt(pnb2)))
            vals[q, blank] = logadd(pb2, pnb2) + h["f"]
        flat = np.arange(nq * V)
        v, ok = vals.reshape(-1), valid.reshape(-1)
        flat, v = flat[ok], v[ok]
        v = np.where(v == 0, dt(0.0), v)                        # -0 ranks with +0, as order_key does
        tmap = None if self.lm_sd is None else (torch.arange(V) if self.lm_map is None
                                                else torch.as_tensor(self.lm_map).long())
        new = []
        for i in np.lexsort((flat, -v))[:self.W]:
            q, k = divmod(int(flat[i]), V)
            h = hyps[q]
            if k == blank:
                nh = dict(h, pb=stay[q][0], pnb=stay[q][1])
            else:
                nh = dict(h, seq=h["seq"] + (k,), pb=ninf, pnb=pnbx[q, k], f=fx[q, k])
                if tmap is not None and int(tmap[k]) >= 0:
                    llp, (lh, lc) = lm_step(self.lm_sd, tmap[k:k + 1], (h["lh"][:, None], h["lc"][:, None]))
                    nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
            new.append(nh)
        self.hyps = new

    def scores(self):
        return [logadd(h["pb"], h["pnb"]) + h["f"] for h in self.hyps]

    def commit(self, n_out, flush=False):
        """The chunk end for chunks of n_out frames: -> the tokens committed (a list); sets ``collapsed``."""
        c0 = len(self.committed)
        seqs = [h["seq"] for h in self.hyps]
        c = len(common_prefix(seqs))
        self.collapsed = flush or max(len(s) for s in seqs) - c > self.P - n_out
        if self.collapsed:
            tot = self.scores()
            best = max(range(len(self.hyps)), key=lambda j: (tot[j], -j))
            self.hyps = [self.hyps[best]]
            c = len(self.hyps[0]["seq"])
            self.n_collapses += not flush
        out = list(self.hyps[0]["seq"][c0:c])
        self.committed = self.hyps[0]["seq"][:c]
        return out

    def chunk(self, y):
        """Frames y [n_out, V], then the chunk end."""
        for yt in np.asarray(y):
            self.frame(yt)
        return self.commit(len(y))

    def flush(self):
        """-> (the rest of the best prefix, -score of that prefix); decoding continues from it."""
        out = self.commit(0, flush=True)
        return out, -float(self.scores()[0])
