"""The pruned RNN-T loss without a GPU: the fp64 oracle (tests/pruned_oracle.py) against the plain RNN-T loss, the
subset property, the band rule's invariants, and the argument checks of the C entries and of the Python API, which all
run before any device work."""
import math

import numpy as np
import pytest
import torch

from tests import pruned_oracle as po

f64 = torch.float64


def _case(seed, B, T, U, V):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, T, U, V, generator=g, dtype=f64) * 2
    labels = torch.randint(1, V, (B, U - 1), generator=g)
    xlen = torch.randint(1, T + 1, (B,), generator=g)
    ylen = torch.randint(0, U, (B,), generator=g)
    xlen[0], ylen[0] = T, U - 1
    return logits, labels, xlen, ylen


def test_full_band_pruned_loss_is_the_rnnt_loss():
    """With R >= max U_b every band is the whole column: the pruned cost is the oracle/loss.py RNN-T cost."""
    from oracle import loss as oracle_loss
    logits, labels, xlen, ylen = _case(0, 3, 5, 4, 6)
    B, T, U, V = logits.shape
    s_begin = [[0] * T for _ in range(B)]
    pc = po.pruned_costs(logits, labels, xlen, ylen, s_begin, U, 0)
    ref, _ = oracle_loss.logits(logits.numpy(), labels.numpy(), xlen.numpy(), ylen.numpy(), 0, want_grads=False,
                                dtype=np.float64)
    np.testing.assert_allclose(pc.numpy(), ref, rtol=1e-12)
    np.testing.assert_allclose(po.full_costs(logits, labels, xlen, ylen, 0).numpy(), ref, rtol=1e-12)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("R", [2, 3])
def test_pruned_cost_is_at_least_the_full_cost(seed, R):
    logits, labels, xlen, ylen = _case(seed, 2, 6, 5, 5)
    B, T, U, V = logits.shape
    full = po.full_costs(logits, labels, xlen, ylen, 0)
    g = torch.Generator().manual_seed(100 + seed)
    s_all, band = [], torch.zeros(B, T, R, V, dtype=f64)
    for b in range(B):
        Tn, Un = po.lengths(xlen[b], ylen[b], T, U)
        occ = torch.rand(Tn, Un, generator=g).float()
        s, nopath = po.band_rule(occ, Tn, Un, R)
        s = s + [0] * (T - Tn)
        s_all.append(s)
        for t in range(Tn):
            for r in range(min(R, Un)):
                band[b, t, r] = logits[b, t, s[t] + r]
    pc = po.pruned_costs(band, labels, xlen, ylen, s_all, U, 0)
    assert bool((pc >= full - 1e-12).all()), (pc, full)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("Tn,Un,R", [(8, 5, 2), (6, 9, 4), (3, 12, 5), (10, 2, 4), (1, 3, 4), (5, 1, 2)])
def test_band_rule_invariants(seed, Tn, Un, R):
    g = torch.Generator().manual_seed(seed)
    occ = torch.rand(Tn, Un, generator=g).float() ** 4
    s, nopath = po.band_rule(occ, Tn, Un, R)
    Rb = min(R, Un)
    assert nopath == (Un - Rb > (Tn - 1) * (Rb - 1))
    if nopath:
        return
    assert s[0] == 0 and s[-1] == Un - Rb
    for t in range(1, Tn):
        assert 0 <= s[t] - s[t - 1] <= Rb - 1
    assert all(0 <= x <= Un - Rb for x in s)


def test_band_rule_follows_the_occupancy():
    """An occupancy concentrated on a diagonal puts each band around it."""
    Tn, Un, R = 9, 9, 3
    occ = torch.zeros(Tn, Un)
    for t in range(Tn):
        occ[t, t] = 1.0
    s, nopath = po.band_rule(occ, Tn, Un, R)
    assert not nopath
    assert all(x <= t <= x + R - 1 for t, x in enumerate(s))


@pytest.fixture(scope="module")
def built():
    from edgedict_b200 import build
    return build.build()


def test_c_entries_reject_bad_arguments_before_touching_the_device(built):
    """Every pruned entry returns EB_ERR_INVALID (2) for R outside [2, 64], maxU > 1024, missing pointers and
    misaligned bf16 pointers, before any CUDA call."""
    from edgedict_b200._lib import lib
    L = lib()
    p = 1 << 20
    for R in (1, 0, 65, -3):
        assert L.eb_rnnt_band_choice(p, p, 2, 3, 4, R, p, p, p, None) == 2
        assert L.eb_joint_band_hidden_fwd(p, p, p, p, p, p, 0, 2, 3, 4, R, 8, None) == 2
        assert L.eb_rnnt_band_loss_fwd(p, p, p, p, p, p, 2, 3, 4, R, 8, 0, p, p, 1, None) == 2
        assert L.eb_rnnt_band_loss_bwd(p, p, 0, p, p, p, p, p, 2, 3, 4, R, 8, 0, p, None, 0, 1.0, None) == 2
        assert L.eb_joint_band_dpre_reduce(p, p, 0, p, p, p, p, p, 2, 3, 4, R, 8, None) == 2
    assert L.eb_rnnt_band_choice(p, p, 2, 3, 1025, 4, p, p, p, None) == 2
    assert L.eb_rnnt_band_loss_fwd(p, p, p, p, p, p, 2, 3, 1025, 4, 8, 0, p, p, 1, None) == 2
    assert L.eb_rnnt_simple_stats(p, p, p, p, p, 2, 3, 1025, 8, 0, p, p, None) == 2
    assert L.eb_rnnt_simple_stats(p, p, p, p, p, 2, 3, 4, 8, 8, p, p, None) == 2           # blank >= V
    assert L.eb_rnnt_simple_bwd(p, p, p, p, p, 2, 3, 4, 8, 0, None, p, None, 0, 1.0, p, p, None) == 2  # scratch
    assert L.eb_rnnt_band_loss_fwd(p, p, p, p, None, p, 2, 3, 4, 4, 8, 0, p, p, 1, None) == 2   # no s_begin
    assert L.eb_rnnt_band_loss_bwd(p, p + 1, 1, p, p, p, p, p, 2, 3, 4, 4, 8, 0, p, None, 0, 1.0, None) == 2
    assert L.eb_joint_band_hidden_fwd(p, p, p, p, p, p + 2, 1, 2, 3, 4, 4, 8, None) == 2      # bf16 misaligned
    assert L.eb_joint_band_dpre_reduce(p + 2, None, 1, p, p, p, p, p, 2, 3, 4, 4, 8, None) == 2
    assert L.eb_joint_band_dpre_reduce(p, None, 0, p, p, p, p, p, 2, 3, 4, 4, 8, None) == 2   # fp32 needs hidden


def test_python_api_checks_arguments_first():
    from edgedict_b200 import pruned
    am = torch.zeros(2, 3, 5)
    lm = torch.zeros(2, 4, 5)
    i32 = torch.int32
    lab, xl, yl = torch.zeros(2, 3, dtype=i32), torch.ones(2, dtype=i32), torch.ones(2, dtype=i32)
    with pytest.raises(TypeError):
        pruned.rnnt_loss_simple(am.double(), lm, lab, xl, yl)
    with pytest.raises(RuntimeError):                       # CPU tensors: no CPU path
        pruned.rnnt_loss_simple(am, lm, lab, xl, yl)
    with pytest.raises(TypeError):
        pruned.rnnt_loss_pruned(torch.zeros(2, 3, 4), lab, xl, yl, None, None)
    for R in (1, 65):
        with pytest.raises(ValueError):
            pruned.check_prune_range(R)
    with pytest.raises(TypeError):
        pruned.check_prune_range(4.0)


def test_transducer_pruned_arguments():
    from edgedict_b200.rnnt.models import Transducer
    kw = dict(vocab_embed_size=8, vocab_size=16, input_size=8, enc_hidden_size=8, enc_layers=1, enc_dropout=0,
              enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0, dec_proj_size=8, joint_size=8)
    base = Transducer(**kw)
    pr = Transducer(**kw, prune_range=5)
    assert set(pr.state_dict()) - set(base.state_dict()) == {"simple_am_proj.weight", "simple_am_proj.bias",
                                                           "simple_lm_proj.weight", "simple_lm_proj.bias"}
    assert not any(k.startswith("simple_") for k in base.state_dict())
    with pytest.raises(ValueError):
        Transducer(**kw, prune_range=5, fastemit_lambda=0.01)
    with pytest.raises(ValueError):
        Transducer(**kw, prune_range=1)
