"""Pins the fp64 restatements of tests/loss_restate.py, which the GPU loss tests compare the kernels with, to the C oracle
(oracle/rnnt_loss_oracle.c): the anti-diagonal lattice against the oracle's alphas, betas and costs, and the gradient
formula against the oracle's gradient wrt logits.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import loss as ol
from tests import loss_restate as lr

# name: (B, T, U, V, blank, xlen, ylen)
CASES = {
    "ragged_blank0": (3, 9, 6, 7, 0, [9, 4, 1], [5, 2, 0]),
    "blank_mid": (2, 13, 8, 11, 5, [13, 7], [7, 4]),
    "blank_last_u1": (2, 6, 1, 5, 4, [6, 3], [0, 0]),
    "t1": (2, 1, 5, 6, 2, [1, 1], [4, 0]),
    "long_t": (2, 70, 3, 4, 1, [70, 33], [2, 1]),
}


def _problem(name):
    B, T, U, V, blank, xl, yl = CASES[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    x = rng.randn(B, T, U, V) * 2
    r = rng.randint(0, V - 1, size=(B, U - 1))
    lab = (r + (r >= blank)).astype(np.int32)
    return x, lab, np.asarray(xl, np.int32), np.asarray(yl, np.int32), blank


@pytest.mark.parametrize("name", list(CASES))
def test_lattice_restatement_matches_oracle(name):
    x, lab, xl, yl, blank = _problem(name)
    B, T, U, V = x.shape
    lp, _ = ol.log_softmax(x, dtype=np.float64)
    costs, _, al_o, be_o = ol.logprobs(lp, lab, xl, yl, blank=blank, dtype=np.float64, want_lattice=True)
    t = torch.as_tensor(lp)
    lpb = t[..., blank]
    lpl = torch.zeros(B, T, U, dtype=torch.float64)
    if U > 1:
        lpl[:, :, :U - 1] = torch.gather(t[:, :, :U - 1], 3, torch.as_tensor(lab).long()[:, None, :, None]
                                         .expand(B, T, U - 1, 1))[..., 0]
    valid = lr.valid_cells(xl, yl, T, U, "cpu")
    lpb = lpb.where(valid, float("nan"))                     # padded log-probs must not be read
    lpl = lpl.where(valid, float("nan"))
    al, be, llf, llb = lr.lattice(lpb, lpl, torch.as_tensor(xl), torch.as_tensor(yl))
    v = valid.numpy()
    assert np.allclose(al.numpy()[v], al_o[v], rtol=1e-13, atol=1e-12)
    assert np.allclose(be.numpy()[v], be_o[v], rtol=1e-13, atol=1e-12)
    assert bool(al[~valid].isnan().all()) and bool(be[~valid].isnan().all())
    assert np.allclose(-llf.numpy(), costs, rtol=1e-13) and np.allclose(-llb.numpy(), costs, rtol=1e-13)
    al2, be2, llf2, llb2 = lr.lattice(lpb, lpl, torch.as_tensor(xl), torch.as_tensor(yl), need_beta=False)
    assert be2 is None and llb2 is None and torch.equal(llf2, llf)


@pytest.mark.parametrize("name", list(CASES))
def test_grad_restatement_matches_oracle(name):
    x, lab, xl, yl, blank = _problem(name)
    B, T, U, V = x.shape
    costs, g_o = ol.logits(x, lab, xl, yl, blank=blank, dtype=np.float64)
    lp, den = ol.log_softmax(x, dtype=np.float64)
    _, _, al, be = ol.logprobs(lp, lab, xl, yl, blank=blank, dtype=np.float64, want_lattice=True)
    g = lr.grad_formula(torch.as_tensor(al), torch.as_tensor(be), torch.as_tensor(den), -torch.as_tensor(costs),
                        torch.as_tensor(x), lab, xl, yl, blank)
    assert np.allclose(g.numpy(), g_o, rtol=1e-10, atol=1e-13)
    g2, terms = lr.grad_formula(torch.as_tensor(al), torch.as_tensor(be), torch.as_tensor(den),
                                -torch.as_tensor(costs), torch.as_tensor(x), lab, xl, yl, blank, terms=True)
    assert torch.equal(g, g2) and bool((terms["absum"] >= g2.abs() * (1 - 1e-12)).all())


def test_lengths_are_clamped_and_no_frames_is_minus_inf():
    """Over-long lengths give the lattice of the clamped ones; xlen = 0 gives ll = -inf and no valid cell."""
    x, lab, xl, yl, blank = _problem("ragged_blank0")
    B, T, U, V = x.shape
    lp = torch.as_tensor(ol.log_softmax(x, dtype=np.float64)[0])
    lpb, lpl = lp[..., blank], lp[..., 1]
    ref = lr.lattice(lpb, lpl, torch.tensor([T, 4, 0]), torch.tensor([U - 1, 2, 3]))
    got = lr.lattice(lpb, lpl, torch.tensor([T + 5, 4, -2]), torch.tensor([U + 7, 2, 3]))
    for r, g in zip(ref, got):
        assert torch.equal(r.nan_to_num(), g.nan_to_num())
    assert float(ref[2][2]) == -np.inf and float(ref[3][2]) == -np.inf
    assert not bool(lr.valid_cells([T, 4, 0], [U - 1, 2, 3], T, U, "cpu")[2].any())
