"""FastEmit without a GPU: the fp64 restatement of the kernels' FastEmit branches (tests/fastemit_restate.py) against
torch autograd of the FastEmit surrogate on the CPU, the argument checks of the three FastEmit C entries, and the
Python argument checks of RNNTLoss / rnnt_loss / Transducer, which all run before any device work."""
import math

import numpy as np
import pytest
import torch

from tests import fastemit_restate as fr
from tests import loss_restate as lr

f64 = torch.float64
LAMBDAS = [0.0, 1e-3, 0.01, 0.5]

# name: (B, T, U, V, blank, xlen, ylen)
PROBLEMS = {
    # ragged lengths, blank in the middle, an utterance with T_b = 1
    "ragged_blank_mid": (3, 6, 5, 9, 4, [6, 4, 1], [4, 2, 3]),
    # U_b = 1 (no labels) beside a full utterance, blank = V - 1
    "no_labels": (2, 5, 4, 7, 6, [5, 3], [3, 0]),
    # T_b = 0 first and in the middle: cost +inf and a zero gradient
    "no_frames": (3, 4, 4, 6, 2, [0, 4, 0], [2, 3, 1]),
    # every utterance T_b = 1
    "t1": (2, 1, 5, 8, 1, [1, 1], [4, 2]),
}


def _problem(name):
    B, T, U, V, blank, xl, yl = PROBLEMS[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    x = torch.as_tensor(rng.randn(B, T, U, V) * 2.5, dtype=f64)
    lab = lr.planted_labels(rng, B, U, V, blank)
    return x, lab, np.asarray(xl, np.int32), np.asarray(yl, np.int32), blank


def _stats(x, lab, xlen, ylen, blank):
    """Exact fp64 statistics and lattice: denom, lpl, alphas, betas, ll_fwd."""
    B, T, U, V = x.shape
    d = -torch.logsumexp(x, -1)
    lpb = x[..., blank] + d
    lpl = torch.zeros(B, T, U, dtype=f64)
    if U > 1:
        idx = torch.as_tensor(lab).long()[:, None, :, None].expand(B, T, U - 1, 1)
        lpl[:, :, :U - 1] = torch.gather(x[:, :, :U - 1], 3, idx)[..., 0] + d[:, :, :U - 1]
    al, be, llf, _ = lr.lattice(lpb, lpl, xlen, ylen)
    return d, lpl, al, be, llf


@pytest.mark.parametrize("lam", LAMBDAS)
@pytest.mark.parametrize("name", list(PROBLEMS))
def test_restatement_matches_surrogate_autograd(name, lam):
    """grad_fastemit on the exact fp64 lattice against autograd of S_b with per-utterance weights (mixed signs), within
    1e-12 of the largest gradient element; every valid row sums to zero; padded cells and T_b = 0 utterances are 0."""
    x, lab, xlen, ylen, blank = _problem(name)
    B = x.shape[0]
    d, lpl, al, be, llf = _stats(x, lab, xlen, ylen, blank)
    w = torch.tensor([(-1.5) ** (b + 1) for b in range(B)], dtype=f64)
    g = fr.grad_fastemit(al.nan_to_num(0), be.nan_to_num(0), d, llf, lpl, x, lab, xlen, ylen, blank, lam)
    g = g * w[:, None, None, None]
    g_o, costs = fr.surrogate_grad(x, lab, xlen, ylen, blank, lam, weights=w)
    scale = float(g_o.abs().max())
    err = float((g - g_o).abs().max()) / scale
    valid = lr.valid_cells(xlen, ylen, x.shape[1], x.shape[2], "cpu")
    rows = g.sum(-1)[valid].abs().max() / scale
    print("%s lam=%g: restatement vs autograd max err %.2e of max |g|, row sums %.1e" % (name, lam, err, rows))
    assert err <= 1e-12, err
    assert float(rows) <= 1e-13
    assert bool((g[~valid] == 0).all())
    Tn, _ = lr.lengths(xlen, ylen, x.shape[1], x.shape[2], "cpu")
    for b in range(B):
        if int(Tn[b]) == 0:
            assert bool((g[b] == 0).all()) and math.isinf(float(costs[b]))
    # the cost does not depend on lambda: the surrogate's log P is the plain one
    assert torch.allclose(costs[torch.isfinite(costs)], -llf[torch.isfinite(llf)], rtol=1e-13, atol=0)


@pytest.mark.parametrize("name", list(PROBLEMS))
def test_restatement_at_zero_is_grad_formula(name):
    """lam = 0 runs loss_restate.grad_formula's operations: the same bits, terms included."""
    x, lab, xlen, ylen, blank = _problem(name)
    d, lpl, al, be, llf = _stats(x, lab, xlen, ylen, blank)
    a, b = al.nan_to_num(0), be.nan_to_num(0)
    g0, t0 = lr.grad_formula(a, b, d, llf, x, lab, xlen, ylen, blank, terms=True)
    g1, t1 = fr.grad_fastemit(a, b, d, llf, lpl, x, lab, xlen, ylen, blank, 0.0, terms=True)
    assert torch.equal(g0, g1)
    for k in t0:
        if t0[k] is not None:
            assert torch.equal(t0[k], t1[k]), k


def test_fastemit_changes_the_gradient_but_only_on_label_rows():
    """lam > 0 moves the gradient of the cells with a label and leaves the cells u = U_b - 1 as they were."""
    x, lab, xlen, ylen, blank = _problem("ragged_blank_mid")
    d, lpl, al, be, llf = _stats(x, lab, xlen, ylen, blank)
    a, b = al.nan_to_num(0), be.nan_to_num(0)
    g0 = fr.grad_fastemit(a, b, d, llf, lpl, x, lab, xlen, ylen, blank, 0.0)
    g1 = fr.grad_fastemit(a, b, d, llf, lpl, x, lab, xlen, ylen, blank, 0.01)
    _, Un = lr.lengths(xlen, ylen, x.shape[1], x.shape[2], "cpu")
    for bi in range(x.shape[0]):
        u_last = int(Un[bi]) - 1
        assert torch.equal(g0[bi, :, u_last], g1[bi, :, u_last])
        if u_last > 0:
            assert not torch.equal(g0[bi, :, :u_last], g1[bi, :, :u_last])


@pytest.fixture(scope="module")
def built():
    from edgedict_b200 import build
    return build.build()


def test_c_entries_reject_bad_lambda_before_touching_the_device(built):
    """eb_rnnt_loss_bwd_fe / _bf16_fe / _bf16_db_fe: a negative, NaN or infinite lambda is EB_ERR_INVALID (2), checked
    before any CUDA call; so are the checks the entries share with their siblings."""
    from edgedict_b200._lib import lib
    L = lib()
    p = 1 << 20                                               # a plausible, aligned, never dereferenced address
    args = (p, p, p, 2, 3, 4, 8, 0)                           # labels, xlen, ylen, B, maxT, maxU, V, blank
    for lam in (-1e-3, -1.0, -math.inf, math.inf, math.nan):
        for dtype_size, out_bf16 in ((4, 0), (4, 1), (8, 0)):
            assert L.eb_rnnt_loss_bwd_fe(p, p, out_bf16, *args, dtype_size, p, None, 0, 1.0, lam, None) == 2, lam
        assert L.eb_rnnt_loss_bwd_bf16_fe(p, p, *args, p, None, 0, 1.0, lam, None) == 2, lam
        assert L.eb_rnnt_loss_bwd_bf16_db_fe(p, p, *args, p, None, 0, 1.0, p, p, lam, None) == 2, lam
    # the shared problem checks still apply with a valid lambda
    bad = (p, None, p, 2, 3, 4, 8, 0)                         # no xlen
    assert L.eb_rnnt_loss_bwd_fe(p, p, 0, *bad, 4, p, None, 0, 1.0, 0.01, None) == 2
    assert L.eb_rnnt_loss_bwd_bf16_fe(p, p, *bad, p, None, 0, 1.0, 0.01, None) == 2
    assert L.eb_rnnt_loss_bwd_bf16_db_fe(p, p, *args[:6], 12, 0, p, None, 0, 1.0, p, p, 0.01, None) == 2   # V % 8
    assert L.eb_rnnt_loss_bwd_fe(p, p, 1, *args, 8, p, None, 0, 1.0, 0.01, None) == 2      # bf16 out of fp64


BAD_VALUES = [(-0.1, ValueError), (math.nan, ValueError), (math.inf, ValueError), (-math.inf, ValueError),
              ("0.1", TypeError), (None, TypeError), (torch.tensor(0.1), TypeError), (1j, TypeError),
              (True, TypeError)]


@pytest.mark.parametrize("value, exc", BAD_VALUES)
def test_python_checks(value, exc):
    """RNNTLoss, rnnt_loss and Transducer refuse a bad lambda before any device work (here: CPU tensors, which the
    loss would otherwise refuse with its CUDA-only RuntimeError)."""
    from edgedict_b200.functional import check_fastemit_lambda
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.warprnnt_pytorch import RNNTLoss, rnnt_loss
    from tests.util import E4D1_CFG
    with pytest.raises(exc):
        check_fastemit_lambda(value)
    with pytest.raises(exc):
        RNNTLoss(fastemit_lambda=value)
    acts = torch.zeros(2, 4, 3, 5)
    labels = torch.zeros(2, 2, dtype=torch.int32)
    tl = torch.tensor([4, 4], dtype=torch.int32)
    ul = torch.tensor([2, 2], dtype=torch.int32)
    with pytest.raises(exc):
        rnnt_loss(acts, labels, tl, ul, fastemit_lambda=value)
    with pytest.raises(exc):
        Transducer(fastemit_lambda=value, **E4D1_CFG)
    m = Transducer(**E4D1_CFG)
    m.fastemit_lambda = value                                 # a trainer's ramp that went wrong: caught at forward
    with pytest.raises(exc):
        m(torch.zeros(2, 8, E4D1_CFG["input_size"]), torch.zeros(2, 3, dtype=torch.int32), tl, ul)


def test_python_accepts_and_stores_lambda():
    """A valid lambda is kept as a float; Transducer's is a plain attribute outside the state_dict; the reference's
    positional arguments of RNNTLoss are unchanged."""
    import numpy as np
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.warprnnt_pytorch import RNNTLoss
    from tests.util import E4D1_CFG
    for v in (0, 0.0, 1e-3, 2, np.float32(0.25), np.float64(0.5)):
        assert RNNTLoss(fastemit_lambda=v).fastemit_lambda == float(v)
    crit = RNNTLoss(3, 'sum')
    assert (crit.blank, crit.reduction, crit.fastemit_lambda) == (3, 'sum', 0.0)
    m = Transducer(fastemit_lambda=0.01, **E4D1_CFG)
    assert m.fastemit_lambda == 0.01 and isinstance(m.fastemit_lambda, float)
    sd = Transducer(**E4D1_CFG).state_dict()
    assert list(m.state_dict().keys()) == list(sd.keys())
    assert Transducer(**E4D1_CFG).fastemit_lambda == 0.0
