"""A torch-fp64 restatement, on the CPU, of the pruned RNN-T loss (include/edgedict_b200.h): the trivial joiner's loss,
the band rule, and the RNN-T loss on band rows.  Everything is written from the definitions, cell by cell, with autograd
giving the gradients."""
import math

import torch

f64 = torch.float64
NINF = -math.inf
# the log-probability of the cells outside the bands: finite, so that autograd through logaddexp stays NaN-free, and
# small enough that no path through such a cell carries weight in fp64
DEAD = -1e30


def lengths(xlen, ylen, T, U):
    """(T_b, U_b) with the loss's clamp."""
    return min(max(int(xlen), 0), T), min(max(int(ylen), 0), U - 1) + 1


def lattice(lpb, lpl, Tn, Un):
    """(alpha, beta, log P) of the RNN-T lattice on lpb / lpl [>= Tn, >= Un] (-inf allowed); log P = -inf for Tn = 0."""
    if Tn == 0:
        return None, None, torch.tensor(NINF, dtype=f64)
    ninf = torch.tensor(NINF, dtype=f64)
    al = [[None] * Un for _ in range(Tn)]
    for t in range(Tn):
        for u in range(Un):
            if t == 0 and u == 0:
                al[t][u] = torch.zeros((), dtype=f64)
                continue
            stay = al[t - 1][u] + lpb[t - 1, u] if t > 0 else ninf
            emit = al[t][u - 1] + lpl[t, u - 1] if u > 0 else ninf
            al[t][u] = torch.logaddexp(stay, emit)
    be = [[None] * Un for _ in range(Tn)]
    for t in reversed(range(Tn)):
        for u in reversed(range(Un)):
            if t == Tn - 1 and u == Un - 1:
                be[t][u] = lpb[t, u]
                continue
            stay = be[t + 1][u] + lpb[t, u] if t < Tn - 1 else ninf
            emit = be[t][u + 1] + lpl[t, u] if u < Un - 1 else ninf
            be[t][u] = torch.logaddexp(stay, emit)
    ll = al[Tn - 1][Un - 1] + lpb[Tn - 1, Un - 1]
    return torch.stack([torch.stack(r) for r in al]), torch.stack([torch.stack(r) for r in be]), ll


def _lp_cells(logp, lab, blank, Un):
    """lpb, lpl [T, Un] from log-probs [T, Un, V]."""
    lpb = logp[:, :, blank]
    lpl = torch.stack([logp[:, u, lab[u]] if u < Un - 1 else torch.zeros_like(logp[:, u, 0]) for u in range(Un)], 1)
    return lpb, lpl


def simple_costs(am, lm, labels, xlen, ylen, blank):
    """Costs [B] of the trivial joiner: the RNN-T lattice on log softmax(am[t] + lm[u])."""
    B, T, V = am.shape
    U = lm.shape[1]
    out = []
    for b in range(B):
        Tn, Un = lengths(xlen[b], ylen[b], T, U)
        if Tn == 0:
            out.append(torch.tensor(math.inf, dtype=f64))
            continue
        logp = torch.log_softmax(am[b, :Tn, None, :] + lm[b, None, :Un, :], -1)
        lpb, lpl = _lp_cells(logp, labels[b], blank, Un)
        out.append(-lattice(lpb, lpl, Tn, Un)[2])
    return torch.stack(out)


def band_rule(occ, Tn, Un, R):
    """(s [Tn] ints, no_path) from the occupancy occ [Tn, Un] (fp32 tensor: scores summed in ascending u in fp32)."""
    Rb = min(R, Un)
    S = Un - Rb
    s = []
    for t in range(Tn):
        best, best_sc = 0, None
        for s0 in range(S + 1):
            sc = torch.zeros((), dtype=occ.dtype)
            for u in range(s0, s0 + Rb):
                sc = sc + occ[t, u]
            if best_sc is None or bool(sc > best_sc):
                best, best_sc = s0, sc
        s.append(best)
    if Tn == 0:
        return [], False
    s[0] = 0
    for t in range(1, Tn):
        s[t] = min(max(s[t], s[t - 1]), s[t - 1] + Rb - 1)
    s[Tn - 1] = S
    for t in range(Tn - 2, -1, -1):
        s[t] = max(s[t], s[t + 1] - (Rb - 1))
    return s, s[0] > 0


def live(s, r, Un):
    """The padding rule for row r < min(R, U_b) of a frame t < T_b that starts at s: it holds cell s + r when s >= 0 and
    s + r < U_b (a frame with a negative start has no live row)."""
    return s >= 0 and s + r < Un


def pruned_costs(band_logits, labels, xlen, ylen, s_begin, U, blank):
    """Costs [B] of the RNN-T loss on band rows [B, T, R, V]: cell (t, s_begin[b][t] + r) for the live rows r < Rb,
    every other cell -inf; +inf when the bands hold no path."""
    B, T, R, V = band_logits.shape
    out = []
    for b in range(B):
        Tn, Un = lengths(xlen[b], ylen[b], T, U)
        Rb = min(R, Un)
        if Tn == 0:
            out.append(torch.tensor(math.inf, dtype=f64))
            continue
        logp = torch.log_softmax(band_logits[b], -1)
        lpb = [[torch.tensor(DEAD, dtype=f64)] * Un for _ in range(Tn)]
        lpl = [[torch.tensor(DEAD, dtype=f64)] * Un for _ in range(Tn)]
        for t in range(Tn):
            for r in range(Rb):
                u = int(s_begin[b][t]) + r
                if not live(int(s_begin[b][t]), r, Un):
                    continue
                lpb[t][u] = logp[t, r, blank]
                if u < Un - 1:
                    lpl[t][u] = logp[t, r, labels[b][u]]
        lpb = torch.stack([torch.stack(x) for x in lpb])
        lpl = torch.stack([torch.stack(x) for x in lpl])
        cost = -lattice(lpb, lpl, Tn, Un)[2]
        out.append(cost if float(cost.detach()) < -DEAD / 2 else torch.tensor(math.inf, dtype=f64))    # no band path
    return torch.stack(out)


def full_costs(logits, labels, xlen, ylen, blank):
    """Costs [B] of the plain RNN-T loss on logits [B, T, U, V]."""
    B, T, U, V = logits.shape
    out = []
    for b in range(B):
        Tn, Un = lengths(xlen[b], ylen[b], T, U)
        if Tn == 0:
            out.append(torch.tensor(math.inf, dtype=f64))
            continue
        logp = torch.log_softmax(logits[b, :Tn, :Un], -1)
        lpb, lpl = _lp_cells(logp, labels[b], blank, Un)
        out.append(-lattice(lpb, lpl, Tn, Un)[2])
    return torch.stack(out)


def band_reduce(dpre, s_begin, xlen, ylen, U):
    """(dep [B, T, J], ddp [B, U, J]) fp64 of band-row d(pre-activation) dpre [B, T, R, J]."""
    B, T, R, J = dpre.shape
    dep = torch.zeros(B, T, J, dtype=f64)
    ddp = torch.zeros(B, U, J, dtype=f64)
    for b in range(B):
        Tn, Un = lengths(xlen[b], ylen[b], T, U)
        Rb = min(R, Un)
        for t in range(Tn):
            for r in range(Rb):
                if not live(int(s_begin[b][t]), r, Un):
                    continue
                dep[b, t] += dpre[b, t, r]
                ddp[b, int(s_begin[b][t]) + r] += dpre[b, t, r]
    return dep, ddp
