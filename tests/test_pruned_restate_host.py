"""tests/pruned_restate.py pinned to tests/pruned_oracle.py (autograd, cell by cell) at small shapes, on the CPU: the
simple loss's statistics and teacher-forced gradients, the band rule, the padding rule (negative and past-the-end
starts), the band statistics and gradient through loss_restate, and the banded reduction."""
import math

import numpy as np
import pytest
import torch

from tests import loss_restate as lr
from tests import pruned_oracle as po
from tests import pruned_restate as pr

f64 = torch.float64
i32 = torch.int32


def _problem(seed, B, T, U, V):
    g = torch.Generator().manual_seed(seed)
    am = torch.randn(B, T, V, generator=g, dtype=f64) * 2
    lm = torch.randn(B, U, V, generator=g, dtype=f64) * 2
    labels = torch.randint(1, V, (B, max(U - 1, 0)), generator=g, dtype=i32)
    return am, lm, labels


# (B, T, U, V, xlen, ylen): ragged with xlen = 0 and 1, ylen = 0, and one full utterance
SIMPLE = [(4, 6, 5, 9, [6, 0, 1, 4], [4, 2, 0, 3]), (2, 3, 1, 7, [3, 2], [0, 0])]


@pytest.mark.parametrize("shape", SIMPLE)
def test_simple_lse_and_grad_match_autograd(shape):
    B, T, U, V, xl, yl = shape
    am, lm, labels = _problem(1, B, T, U, V)
    blank = 2
    xlen, ylen = torch.tensor(xl, dtype=i32), torch.tensor(yl, dtype=i32)
    N = pr.simple_lse(am, lm, xlen, ylen, max_bytes=8 * U * V * 2)          # two frames per chunk
    valid = lr.valid_cells(xlen, ylen, T, U, "cpu")
    ref = torch.logsumexp(am[:, :, None] + lm[:, None], -1)
    assert torch.allclose(N[valid], ref[valid], rtol=0, atol=1e-12) and bool(N[~valid].isnan().all())
    # exact fp64 workspace from the definitions, then the teacher-forced gradient against autograd of the cost
    lpb = am[:, :, None, blank] + lm[:, None, :, blank] - ref
    lab = labels.long()
    lpl = torch.zeros_like(lpb)
    if U > 1:
        lpl[:, :, :U - 1] = torch.gather(am, 2, lab[:, None, :].expand(B, T, U - 1)) + \
            torch.gather(lm[:, :U - 1], 2, lab[:, :, None])[:, None, :, 0] - ref[:, :, :U - 1]
    a, be, ll, _ = lr.lattice(lpb, lpl, xlen, ylen)
    w = torch.tensor([0.7, -0.3, 1.3, 2.0][:B], dtype=f64)
    dam, dlm, aam, alm = pr.simple_grad(am, lm, labels, xlen, ylen, blank, a.nan_to_num(0), be.nan_to_num(0),
                                        -ref, lpb, lpl, ll, w, max_bytes=8 * U * V)
    a64, l64 = am.clone().requires_grad_(True), lm.clone().requires_grad_(True)
    cost = po.simple_costs(a64, l64, lab, xlen, ylen, blank)
    fin = torch.isfinite(cost)
    (cost[fin] * w[fin]).sum().backward()
    assert torch.allclose(dam, a64.grad, rtol=0, atol=1e-12), float((dam - a64.grad).abs().max())
    assert torch.allclose(dlm, l64.grad, rtol=0, atol=1e-12), float((dlm - l64.grad).abs().max())
    assert bool((aam >= dam.abs() - 1e-12).all()) and bool((alm >= dlm.abs() - 1e-12).all())


def test_band_rule_matches_oracle_and_breaks_ties_low():
    B, T, U, R = 5, 9, 8, 3
    g = torch.Generator().manual_seed(3)
    occ = torch.rand(B, T, U, generator=g)
    occ[1, :, :] = 0.25                                      # every window ties: the lowest s wins
    xlen = torch.tensor([9, 9, 0, 1, 3], dtype=i32)
    ylen = torch.tensor([7, 7, 4, 0, 7], dtype=i32)          # utterance 4: no path through bands of 3
    s, nop, margin = pr.band_rule(occ, xlen, ylen, R)
    for b in range(B):
        Tn, Un = po.lengths(xlen[b], ylen[b], T, U)
        ref, np_ = po.band_rule(occ[b, :Tn, :Un], Tn, Un, R)
        assert s[b, :Tn].tolist() == ref and bool(nop[b]) == np_
        assert bool(s[b, Tn:].eq(0).all())
    assert bool(margin[1, :9].isinf().all()) and bool(nop[4])   # equal fp64 scores are exact ties, not near-ties
    assert bool(margin[3].isinf().all())                     # U_b = 1: one window


def _band_case(seed, B, T, U, R, V, xl, yl):
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(1, V, (B, U - 1), generator=g, dtype=i32)
    xlen, ylen = torch.tensor(xl, dtype=i32), torch.tensor(yl, dtype=i32)
    s = torch.zeros(B, T, dtype=i32)
    nop = torch.zeros(B, dtype=i32)
    for b in range(B):
        Tn, Un = po.lengths(xl[b], yl[b], T, U)
        sb, np_ = po.band_rule(torch.rand(Tn, Un, generator=g), Tn, Un, R)
        s[b, :Tn] = torch.tensor(sb, dtype=i32)
        nop[b] = int(np_)
    x = torch.randn(B, T, R, V, generator=g, dtype=f64) * 2
    return labels, xlen, ylen, s, nop, x


def test_band_loss_and_grad_match_autograd_with_out_of_range_starts():
    B, T, U, R, V, blank = 4, 7, 6, 3, 11, 1
    labels, xlen, ylen, s, nop, x = _band_case(5, B, T, U, R, V, [7, 7, 5, 4], [5, 5, 4, 5])
    s[1, 6] = 4                                              # past the end on the last frame: rows 4 + 2 >= U_b padding
    s[2, 0] = -1                                             # a negative start: the frame has no live row, cost +inf
    live, u = pr.live_rows(s, nop, xlen, ylen, T, U, R)
    assert not bool(live[2, 0].any()) and live[1, 6].tolist() == [True, True, False]
    d, pb, pl, _ = pr.band_stats(x, labels, xlen, ylen, s, nop, U, blank)
    a, be, ll, _ = lr.lattice(pb, pl, xlen, ylen)
    cost = torch.where(nop.bool() | torch.isneginf(ll), math.inf, -ll)
    x64 = x.clone().requires_grad_(True)
    ref = po.pruned_costs(x64, labels.long(), xlen, ylen, s.tolist(), U, blank)
    assert torch.equal(torch.isfinite(cost), torch.isfinite(ref.detach())) and not bool(torch.isfinite(cost[2]))
    fin = torch.isfinite(cost)
    assert torch.allclose(cost[fin], ref.detach()[fin], rtol=1e-13, atol=0)
    w = torch.tensor([0.5, 1.5, -1.0, 2.0], dtype=f64)
    (ref[fin] * w[fin]).sum().backward()
    g = pr.band_grad(a.nan_to_num(0), be.nan_to_num(0), d.nan_to_num(0), ll, x, labels, xlen, ylen, s, nop, U, blank,
                     scale=w)
    assert torch.allclose(g[fin], x64.grad[fin], rtol=0, atol=1e-12), float((g[fin] - x64.grad[fin]).abs().max())
    assert bool(g[~live].eq(0).all())
    # band_grad is grad_formula's value at each live row's cell
    dense = torch.zeros(B, T, U, V, dtype=f64)
    bi, ti, ri = live.nonzero(as_tuple=True)
    dense[bi, ti, u[bi, ti, ri]] = x[bi, ti, ri]
    gd = lr.grad_formula(a.nan_to_num(0), be.nan_to_num(0), d.nan_to_num(0), ll, dense, labels, xlen, ylen, blank)
    g1 = pr.band_grad(a.nan_to_num(0), be.nan_to_num(0), d.nan_to_num(0), ll, x, labels, xlen, ylen, s, nop, U, blank)
    ok = fin[bi]
    assert torch.equal(g1[bi, ti, ri][ok], gd[bi, ti, u[bi, ti, ri]][ok])


def test_band_reduce_matches_oracle_with_out_of_range_starts():
    B, T, U, R, J = 3, 8, 7, 4, 5
    _, xlen, ylen, s, _, _ = _band_case(9, B, T, U, R, 3, [8, 6, 8], [6, 3, 6])
    s[2, :2] = -2                                            # negative starts on the first frames (monotone)
    s[0, 7] = 5                                              # past the end on the last frame
    g = torch.Generator().manual_seed(10)
    dpre = torch.randn(B, T, R, J, generator=g, dtype=f64)
    dep, ddp, adep, addp = pr.band_reduce(dpre, s, xlen, ylen, U)
    rdep, rddp = po.band_reduce(dpre, s.tolist(), xlen, ylen, U)
    assert torch.allclose(dep, rdep, rtol=0, atol=1e-13) and torch.allclose(ddp, rddp, rtol=0, atol=1e-13)
    assert bool(dep[2, :2].eq(0).all()) and bool((adep >= dep.abs()).all()) and bool((addp >= ddp.abs()).all())


def test_live_rows_rule():
    s = torch.tensor([[0, -1, 3, 5]], dtype=i32)
    live, u = pr.live_rows(s, torch.zeros(1, dtype=i32), np.array([3]), np.array([5]), 4, 7, 3)
    # frame 1 starts below 0, frame 2 holds u = 3, 4, 5 < U_b = 6, frame 3 lies past T_b = 3
    assert live.tolist() == [[[True] * 3, [False] * 3, [True] * 3, [False] * 3]]
    live, _ = pr.live_rows(s, torch.ones(1, dtype=i32), [3], [5], 4, 7, 3)
    assert not bool(live.any())
    live, _ = pr.live_rows(torch.tensor([[4]], dtype=i32), torch.zeros(1, dtype=i32), [1], [4], 1, 7, 3)
    assert live.tolist() == [[[True, False, False]]]
