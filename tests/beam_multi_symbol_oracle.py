"""CPU restatement of beam search with up to K symbols per encoder frame (Transducer.beam_search(max_symbols=K)), on
the pieces of oracle/model_torch.py and tests/lm_oracle.py.  Per utterance and encoder frame, rounds j = 0 .. K-1:

- every hypothesis is open at round 0;
- an open hypothesis q offers every token k at (a_q[k] + f_q[k]) + lp[q] (f the LM term, absent without an LM):
  blank closes it, a non-blank k extends the sequence and stays open unless j = K-1;
- a closed hypothesis offers one "stay" of value lp[q], ranked as flat index q*V + blank;
- the W best candidates survive (ties to the lowest flat index); with ``merge`` a candidate folds into an earlier
  survivor by log-add when both the sequence and the closedness are equal;
- a survivor that took a non-blank token steps the predictor (and the LM when it maps the token);
- the frame ends after round K-1 or when no hypothesis is open.

At K = 1 this is lm_oracle.beam_search, step for step."""
import torch
import torch.nn.functional as F

from oracle import model_torch as mt
from tests import lm_oracle as lo


def start(sd, lm_sd=None, lm_bos=1):
    """The one hypothesis every utterance starts from: empty sequence, log p 0, predictor (and LM) primed."""
    dec_x, (dh, dc) = mt.decoder(sd, torch.zeros(1, 0, dtype=torch.long), None)
    hy = dict(seq=[], lp=torch.zeros(()), x=dec_x[0, 0], h=dh[:, 0], c=dc[:, 0], open=False)
    if lm_sd is not None:
        llp, (lh, lc) = lo.lm_prime(lm_sd, lm_bos)
        hy.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
    return hy


def frame(sd, hyps, h_t, W, K, merge=True, blank=mt.NUL, lm_sd=None, lm_weight=0.0, length_bonus=0.0, lm_map=None,
          stats=None):
    """One encoder frame (h_t [E]) of the search from the hypotheses ``hyps`` -> the new hypotheses.  ``stats``, a dict,
    counts the rounds taken under 'rounds'."""
    V = sd["joint.joint.2.weight"].shape[0]
    tmap = torch.arange(V) if lm_map is None else torch.as_tensor(lm_map).long()
    hyps = [dict(h, open=True) for h in hyps]
    for j in range(K):
        if not any(h["open"] for h in hyps):
            break
        if stats is not None:
            stats["rounds"] = stats.get("rounds", 0) + 1
        last = j == K - 1
        cand = []
        for qi, hy in enumerate(hyps):
            if not hy["open"]:
                cand.append((float(hy["lp"]), qi, blank, hy["lp"]))
                continue
            a = F.log_softmax(mt.joint(sd, h_t[None], hy["x"][None])[0], 0)
            if lm_sd is not None:
                a = a + lo.fusion_term(hy["llp"].to(a.dtype), V, blank, lm_weight, length_bonus, lm_map)
            lp = a + hy["lp"]
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
                nh.update(x=nx[0, 0], h=h2[:, 0], c=c2[:, 0])
                if lm_sd is not None and int(tmap[k]) >= 0:
                    llp, (lh, lc) = lo.lm_step(lm_sd, tmap[k:k + 1], (hy["lh"][:, None], hy["lc"][:, None]))
                    nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
            seen[key] = nh
            new.append(nh)
        hyps = new
    return [dict(h, open=False) for h in hyps]


@torch.no_grad()
def beam_search(sd, xs, xlen=None, W=4, max_symbols=1, merge=True, blank=mt.NUL, time_reductions=(1,), lm_sd=None,
                lm_weight=0.0, length_bonus=0.0, lm_bos=1, lm_map=None, h_enc=None, stats=None):
    """-> (best non-blank ids per utterance, -log p [B]) as Transducer.beam_search(max_symbols=K).  ``h_enc`` [B, T', E]
    replaces the encoder output of xs."""
    if h_enc is None:
        h_enc, _ = mt.encoder(sd, xs, None, time_reductions)
    outs, nlps = [], []
    for b in range(h_enc.shape[0]):
        Tn = h_enc.shape[1]
        frames = Tn if xlen is None else min(Tn, int(mt.scale_length(Tn, xlen)[b]))
        hyps = [start(sd, lm_sd, lm_bos)]
        for t in range(frames):
            hyps = frame(sd, hyps, h_enc[b, t], W, max_symbols, merge, blank, lm_sd, lm_weight, length_bonus, lm_map,
                         stats)
        best = max(hyps, key=lambda h: float(h["lp"]))
        outs.append(best["seq"])
        nlps.append(-best["lp"])
    return outs, torch.stack(nlps)


@torch.no_grad()
def stream_search(sd, xs, chunk_out, W, max_pending, max_symbols=1, merge=True, blank=mt.NUL, lm_sd=None,
                  lm_weight=0.0, length_bonus=0.0, lm_bos=1):
    """One stream (xs [1, T, F]) cut into chunks of chunk_out encoder frames each, as StreamBeamEngine(max_symbols=K):
    the frames above, then at each chunk end the commit of the live hypotheses' common prefix and, when a stored
    suffix still exceeds max_pending - n_out * K tokens, the collapse to the best hypothesis (highest log p, lowest slot
    on ties).  ``max_symbols`` may also be a list, one K per chunk: an engine rebuilt for another K continues the beam
    (StreamBeamEngine.load_state), and the chunk-end rule then runs once under the new bound.
    -> (committed ids per chunk, the live hypotheses' full sequences after each chunk)"""
    Ks = list(max_symbols) if isinstance(max_symbols, (list, tuple)) else [max_symbols] * len(chunk_out)
    h_enc, _ = mt.encoder(sd, xs, None)
    hyps = [start(sd, lm_sd, lm_bos)]
    done, t, per, live = 0, 0, [], []

    def commit(n_out, K):
        nonlocal hyps, done
        pend = [h["seq"][done:] for h in hyps]
        c = 0
        while all(len(p) > c and p[c] == pend[0][c] for p in pend):
            c += 1
        out = pend[0][:c]
        done += c
        if max(len(p) for p in pend) - c > max_pending - n_out * K:
            best = max(range(len(hyps)), key=lambda i: (float(hyps[i]["lp"]), -i))
            out += hyps[best]["seq"][done:]
            done = len(hyps[best]["seq"])
            hyps = [hyps[best]]
        return out

    for n_out, K in zip(chunk_out, Ks):
        out = commit(n_out, K)                # a no-op unless n_out * K grew
        for _ in range(n_out):
            hyps = frame(sd, hyps, h_enc[0, t], W, K, merge, blank, lm_sd, lm_weight, length_bonus)
            t += 1
        per.append(out + commit(n_out, K))
        live.append([h["seq"] for h in hyps])
    return per, live
