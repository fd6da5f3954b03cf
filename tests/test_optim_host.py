"""CPU-side checks of the flat-bucket optimizers (edgedict_b200.optim.SGD / SM3 / AdamW / Novograd): the fp64 oracle
against the reference's recorded steps (tests/golden/optim_tiny.npz), constructor validation with the reference's
messages, the refused options, and the C entries' argument checks.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

from tests import optim_oracle as oo
from tests.util import rel_err

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def z():
    return np.load(os.path.join(HERE, "golden", "optim_tiny.npz"))


@pytest.mark.parametrize("case", sorted(oo.HYPER))
def test_oracle_matches_reference_fixture(z, case):
    init, grads, groups, hyp, _ = oo.fixture(z, case)
    out = oo.run(oo.KIND[case], init, list(zip(grads, hyp)), groups)
    for step, (ps, st) in enumerate(out, 1):
        for i, p in enumerate(ps):
            assert rel_err(p, z["%s.p.%d.%d" % (case, step, i)]) < 1e-5, (case, step, i)
            want = oo.fixture_state(z, case, step, i)
            if case == "sgd":
                assert set(want) == {"momentum_buffer"}
            else:
                assert set(want) == set(st[i]), (set(want), set(st[i]))
            for k, v in want.items():
                assert np.shape(v) == np.shape(st[i][k]), (case, k)
                assert rel_err(st[i][k], v) < 1e-5, (case, step, i, k)


def _cpu_params():
    return [torch.zeros(3, requires_grad=True), torch.zeros(2, 2, requires_grad=True)]


@pytest.mark.parametrize("make,msg", [
    (lambda o, p: o.SGD(p, lr=-1.0), "Invalid learning rate: -1.0"),
    (lambda o, p: o.SGD(p, momentum=-0.5), "Invalid momentum value: -0.5"),
    (lambda o, p: o.SGD(p, weight_decay=-1.0), "Invalid weight_decay value: -1.0"),
    (lambda o, p: o.SM3(p, lr=-0.1), "Invalid learning rate: -0.1"),
    (lambda o, p: o.SM3(p, momentum=1.0), "Invalid momentum: 1.0"),
    (lambda o, p: o.SM3(p, beta=-0.1), "Invalid beta: -0.1"),
    (lambda o, p: o.SM3(p, eps=-1.0), "Invalid eps: -1.0"),
    (lambda o, p: o.AdamW(p, lr=-1.0), "Invalid learning rate: -1.0"),
    (lambda o, p: o.AdamW(p, eps=-1.0), "Invalid epsilon value: -1.0"),
    (lambda o, p: o.AdamW(p, betas=(1.0, 0.9)), "Invalid beta parameter at index 0: 1.0"),
    (lambda o, p: o.AdamW(p, betas=(0.9, 1.5)), "Invalid beta parameter at index 1: 1.5"),
    (lambda o, p: o.Novograd(p, lr=-1.0), "Invalid learning rate: -1.0"),
    (lambda o, p: o.Novograd(p, betas=(0.9, -0.1)), "Invalid beta parameter at index 1: -0.1"),
])
def test_hyperparameters_are_checked_first_with_the_reference_messages(make, msg):
    from edgedict_b200 import optim
    with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)")):
        make(optim, _cpu_params())


@pytest.mark.parametrize("make,option", [
    (lambda o, p: o.SGD(p, momentum=0.9, dampening=0.1), "dampening"),
    (lambda o, p: o.SGD(p, momentum=0.9, nesterov=True), "nesterov"),
    (lambda o, p: o.SGD(p, maximize=True), "maximize"),
    (lambda o, p: o.SGD(p, differentiable=True), "differentiable"),
    (lambda o, p: o.SM3(p, momentum=0.5), "momentum"),
    (lambda o, p: o.SM3(p, beta=0.5), "beta"),
    (lambda o, p: o.AdamW(p, amsgrad=True), "amsgrad"),
    (lambda o, p: o.Novograd(p, amsgrad=True), "amsgrad"),
    (lambda o, p: o.Novograd(p, grad_averaging=True), "grad_averaging"),
    (lambda o, p: o.AdamW([{"params": p[:1]}, {"params": p[1:], "amsgrad": True}]), "amsgrad"),
])
def test_refused_options_name_the_option(make, option):
    from edgedict_b200 import optim
    with pytest.raises(ValueError, match=option):
        make(optim, _cpu_params())


def test_structural_refusals_and_cpu_parameters():
    from edgedict_b200 import optim
    with pytest.raises(ValueError, match="rank <= 4"):
        optim.SGD([torch.zeros(1, 1, 1, 1, 2, requires_grad=True)])
    with pytest.raises(ValueError, match="at most 16"):
        optim.AdamW([{"params": [torch.zeros(2, requires_grad=True)]} for _ in range(17)])
    p = torch.zeros(3, requires_grad=True)
    with pytest.raises(ValueError, match="more than one parameter group"):
        optim.SM3([{"params": [p]}, {"params": [p]}])
    with pytest.raises(RuntimeError, match="CUDA"):
        optim.SGD([p], lr=0.1, foreach=True, fused=False)        # foreach / fused are accepted; the device is not


@pytest.fixture(scope="module")
def built():
    from edgedict_b200 import build
    return build.build()


def test_entry_points_reject_bad_arguments_before_touching_the_device(built):
    from edgedict_b200._lib import OptHyper, lib
    L = lib()
    p = 1 << 20                                               # a plausible, aligned, never dereferenced address
    h = OptHyper()
    assert L.eb_opt_seg_sumsq(None, p, 1, p, 1, p, p, None, None) == 2
    assert L.eb_opt_seg_sumsq(p, p, 0, p, 1, p, p, None, None) == 2
    assert L.eb_opt_seg_sumsq(p, p, 1, p, -1, p, p, None, None) == 2
    assert L.eb_opt_seg_sumsq(p, p, 1, p, 1, None, p, None, None) == 2
    assert L.eb_opt_prologue(None, 1.0, 0.0, 0, p, p, None) == 2                  # no groups
    assert L.eb_opt_prologue(None, 1.0, 0.0, 17, p, p, None) == 2                 # more than 16 groups
    assert L.eb_opt_prologue(None, 1.0, -1.0, 1, p, p, None) == 2                 # max_norm < 0
    assert L.eb_opt_prologue(None, 1.0, 0.0, 1, None, p, None) == 2
    assert L.eb_opt_sgd_step(None, p, None, p, p, 1, h, 1, p, p, None) == 2
    assert L.eb_opt_sgd_step(p, p, None, p, p, -1, h, 1, p, p, None) == 2
    h.b1[0] = 0.9
    assert L.eb_opt_sgd_step(p, p, None, p, p, 1, h, 1, p, p, None) == 2          # momentum without a buffer
    assert L.eb_opt_sm3_step(p, p, p, None, 8, p, p, 1, h, 1, p, None) == 2
    assert L.eb_opt_sm3_step(p, p, p, p, -8, p, p, 1, h, 1, p, None) == 2
    assert L.eb_opt_sm3_step(p, p, p, p, 8, p, p, 1, h, 0, p, None) == 2
    assert L.eb_opt_adamw_step(p, p, p, None, p, p, 1, h, 1, p, p, None) == 2
    assert L.eb_opt_adamw_step(p, p, p, p, p, None, 1, h, 1, p, p, None) == 2
    assert L.eb_opt_novograd_step(p, p, p, p, None, p, 1, p, 1, h, 1, p, None) == 2
    assert L.eb_opt_novograd_step(p, p, p, p, p, p, -1, p, 1, h, 1, p, None) == 2
