"""CPU restatement of beam search with shallow fusion of the reference's LSTM language model (LMModel, reference
models.py:224-261), the oracle of tests/test_oracle_lm.py and tests/test_gpu_beam_lm.py.  It builds on
oracle/model_torch.py's encoder / predictor / joint and follows its ``beam_search`` step for step, adding the LM term
Transducer.beam_search documents."""
import torch
import torch.nn.functional as F

from oracle import model_torch as mt


def lm_step(lm_sd, tok, hidden):
    """One token of LMModel.forward (eval mode: no dropout) for a batch: tok [B] -> (log_softmax of the logits
    [B, ntoken], (h, c) [L, B, H]).  ``lm_sd`` is its state_dict; the dtype of the weights (fp32 / fp64) is the
    arithmetic."""
    h0, c0 = hidden
    L = mt._n(lm_sd, "rnn.weight_ih_l%d")
    x = F.embedding(torch.as_tensor(tok).long(), lm_sd["encoder.weight"])[:, None]
    nh, nc = [], []
    for k in range(L):
        x, h, c = mt.lstm_layer(x, h0[k], c0[k], *(lm_sd["rnn.%s_l%d" % (n, k)]
                                                   for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
        nh.append(h)
        nc.append(c)
    logits = F.linear(x[:, 0], lm_sd["decoder.weight"], lm_sd["decoder.bias"])
    return F.log_softmax(logits, -1), (torch.stack(nh), torch.stack(nc))


def lm_prime(lm_sd, lm_bos, n=1):
    """LM log-probs and state of n hypotheses after the <bos> step from zeros."""
    L, H = mt._n(lm_sd, "rnn.weight_ih_l%d"), lm_sd["rnn.weight_hh_l0"].shape[1]
    z = lm_sd["encoder.weight"].new_zeros(L, n, H)
    return lm_step(lm_sd, torch.full((n,), lm_bos), (z, z))


def fusion_term(llp, V, blank, lm_weight, length_bonus, lm_map=None):
    """f [V] of one hypothesis whose LM log-probs are llp [ntoken]: lm_weight * llp[map(k)] + length_bonus for a mapped
    non-blank k, length_bonus for an unmapped one, 0 for blank."""
    tmap = torch.arange(V) if lm_map is None else torch.as_tensor(lm_map).long()
    f = torch.where(tmap >= 0, lm_weight * llp[tmap.clamp(min=0)] + length_bonus,
                    torch.full((V,), length_bonus, dtype=llp.dtype))
    f[blank] = 0.0
    return f


@torch.no_grad()
def beam_search(sd, xs, xlen=None, W=4, blank=mt.NUL, merge=True, time_reductions=(1,), lm_sd=None, lm_weight=0.0,
                length_bonus=0.0, lm_bos=1, lm_map=None):
    """oracle.model_torch.beam_search with the LM fused: candidate value (a + f) + lp (fusion_term), each
    hypothesis' LM primed with lm_bos and stepped on map(k) when it emits a non-blank k with map(k) >= 0.  Without
    ``lm_sd`` it is model_torch.beam_search."""
    if lm_sd is None:
        return mt.beam_search(sd, xs, xlen, W=W, blank=blank, merge=merge, time_reductions=time_reductions)
    V = sd["joint.joint.2.weight"].shape[0]
    tmap = torch.arange(V) if lm_map is None else torch.as_tensor(lm_map).long()
    h_enc_all, _ = mt.encoder(sd, xs, None, time_reductions)
    outs, nlps = [], []
    for b in range(xs.shape[0]):
        Tn = h_enc_all.shape[1]
        frames = Tn if xlen is None else min(Tn, int(mt.scale_length(Tn, xlen)[b]))
        dec_x, (dh, dc) = mt.decoder(sd, torch.zeros(1, 0, dtype=torch.long), None)
        llp, (lh, lc) = lm_prime(lm_sd, lm_bos)
        hyps = [dict(seq=[], lp=torch.zeros(()), x=dec_x[0, 0], h=dh[:, 0], c=dc[:, 0], llp=llp[0], lh=lh[:, 0],
                     lc=lc[:, 0])]
        for t in range(frames):
            cand = []
            for qi, hy in enumerate(hyps):
                a = F.log_softmax(mt.joint(sd, h_enc_all[b, t][None], hy["x"][None])[0], 0)
                lp = (a + fusion_term(hy["llp"].to(a.dtype), V, blank, lm_weight, length_bonus, lm_map)) + hy["lp"]
                cand += [(float(lp[k]), qi, k, lp[k]) for k in range(lp.shape[0])]
            cand.sort(key=lambda c: (-c[0], c[1], c[2]))
            new, seen = [], {}
            for _, qi, k, lpk in cand[:W]:
                hy = hyps[qi]
                seq = hy["seq"] + ([k] if k != blank else [])
                key = tuple(seq)
                if merge and key in seen:
                    seen[key]["lp"] = torch.logaddexp(seen[key]["lp"], lpk)
                    continue
                nh = dict(hy, seq=seq, lp=lpk)
                if k != blank:
                    nx, (h2, c2) = mt.decoder(sd, torch.full((1, 1), k), (hy["h"][:, None], hy["c"][:, None]))
                    nh.update(x=nx[0, 0], h=h2[:, 0], c=c2[:, 0])
                    if int(tmap[k]) >= 0:
                        llp, (lh, lc) = lm_step(lm_sd, tmap[k:k + 1], (hy["lh"][:, None], hy["lc"][:, None]))
                        nh.update(llp=llp[0], lh=lh[:, 0], lc=lc[:, 0])
                seen[key] = nh
                new.append(nh)
            hyps = new
        best = max(hyps, key=lambda h: float(h["lp"]))
        outs.append(best["seq"])
        nlps.append(-best["lp"])
    return outs, torch.stack(nlps)
