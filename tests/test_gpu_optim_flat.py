"""The flat-bucket optimizers (edgedict_b200.optim.SGD / SM3 / AdamW / Novograd, csrc/optim.cu) on the device: parity
with the fp64 oracle (tests/optim_oracle.py) and with the reference's recorded steps (tests/golden/optim_tiny.npz),
checkpoint continuity, schedulers, the overflow skip, bitwise invariants, and AdamW against FlatAdamW."""
import io
import os

import numpy as np
import pytest
import torch

from tests import optim_oracle as oo
from tests.util import rel_err

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(oo.HYPER)


@pytest.fixture(scope="module")
def z():
    return np.load(os.path.join(HERE, "golden", "optim_tiny.npz"))


def _params(init):
    return [torch.tensor(np.asarray(x), dtype=torch.float32, device="cuda", requires_grad=True) for x in init]


def _make(case, params, groups, lr, order=None):
    from edgedict_b200 import optim
    cls, kw, _ = oo.HYPER[case]
    order = list(range(len(params))) if order is None else order
    if case == "adamw2":
        g0 = [params[i] for i in order if groups[i] == 0]
        g1 = [params[i] for i in order if groups[i] == 1]
        return getattr(optim, cls)([{"params": g0}, {"params": g1, "weight_decay": 0.0}], lr=lr, **kw)
    return getattr(optim, cls)([params[i] for i in order], lr=lr, **kw)


def _step(opt, params, grads, lr, scale=1.0, **kw):
    for g in opt.param_groups:
        g["lr"] = lr
    opt.zero_grad()
    for p, g in zip(params, grads):
        p.grad.copy_(torch.as_tensor(np.asarray(g) * scale))
    opt.step(**kw)


def _state_by_param(opt, params):
    """state_dict() keyed by the index into ``params``."""
    sd = opt.state_dict()
    order = [p for g in opt.param_groups for p in g["params"]]
    return {next(i for i, q in enumerate(params) if q is order[k]): v for k, v in sd["state"].items()}


def _lr(z, case, step):
    return float(z["%s.lr" % case][0 if step <= oo.LR_CHANGE else 1])


@pytest.mark.parametrize("variant", ["plain", "grad_scale", "clip_active", "clip_inactive"])
@pytest.mark.parametrize("case", CASES)
def test_parity_with_oracle_and_reference(z, case, variant):
    init, grads, groups, hyp, _ = oo.fixture(z, case)
    scale, kw, okw = 1.0, {}, {}
    if variant == "grad_scale":
        scale, kw, okw = 4.0, dict(grad_scale=0.25), dict(grad_scale=0.25)
    elif variant == "clip_active":
        kw = okw = dict(max_norm=1.0)
    elif variant == "clip_inactive":
        kw = okw = dict(max_norm=1e6)
    params = _params(init)
    opt = _make(case, params, groups, _lr(z, case, 1))
    want = oo.run(oo.KIND[case], init, [([g * scale for g in gs], h) for gs, h in zip(grads, hyp)], groups, **okw)
    for step in range(1, oo.NSTEPS + 1):
        _step(opt, params, grads[step - 1], _lr(z, case, step), scale, **kw)
        ops, ost = want[step - 1]
        st = _state_by_param(opt, params)
        for i, p in enumerate(params):
            got = p.detach().cpu().numpy()
            assert rel_err(got, ops[i]) < 2e-5, (case, variant, step, i)
            for k, v in st[i].items():
                if torch.is_tensor(v):
                    assert tuple(v.shape) == np.shape(ost[i][k]), (k, v.shape)
                    assert rel_err(v.cpu().numpy(), ost[i][k]) < 2e-5, (case, variant, step, i, k)
                else:
                    assert v == ost[i][k], (k, v)
            if variant != "clip_active":
                assert rel_err(got, z["%s.p.%d.%d" % (case, step, i)]) < 5e-5, (case, variant, step, i)
                for k, v in oo.fixture_state(z, case, step, i).items():
                    mine = st[i][k]
                    mine = mine.cpu().numpy() if torch.is_tensor(mine) else mine
                    assert rel_err(mine, v) < 5e-5, (case, variant, step, i, k)


@pytest.mark.parametrize("case", CASES)
def test_checkpoint_from_reference_continues(z, case):
    """The reference's step-3 parameters and state_dict, loaded into a fresh optimizer, continue like the reference."""
    init, grads, groups, hyp, _ = oo.fixture(z, case)
    params = _params([z["%s.p.3.%d" % (case, i)] for i in range(len(init))])
    opt = _make(case, params, groups, _lr(z, case, 1))
    sd = opt.state_dict()
    order = [p for g in opt.param_groups for p in g["params"]]
    idx = [next(i for i, q in enumerate(params) if q is p) for p in order]
    sd["state"] = {k: {kk: (torch.tensor(v) if np.ndim(v) or kk.startswith(("exp_avg_sq", "acc")) else float(v))
                       for kk, v in oo.fixture_state(z, case, 3, i).items()} for k, i in enumerate(idx)}
    opt.load_state_dict(sd)
    for step in range(4, oo.NSTEPS + 1):
        _step(opt, params, grads[step - 1], _lr(z, case, step))
        for i, p in enumerate(params):
            assert rel_err(p.detach().cpu().numpy(), z["%s.p.%d.%d" % (case, step, i)]) < 5e-5, (case, step, i)
    if case != "sgd":
        assert all(st["step"] == oo.NSTEPS for st in opt.state_dict()["state"].values())


@pytest.mark.parametrize("case", CASES)
def test_state_dict_roundtrip_continues_bitwise(z, case):
    init, grads, groups, hyp, _ = oo.fixture(z, case)
    params = _params(init)
    opt = _make(case, params, groups, _lr(z, case, 1))
    for step in range(1, 4):
        _step(opt, params, grads[step - 1], _lr(z, case, step), max_norm=5.0)
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    size = buf.tell()
    buf.seek(0)
    loaded = torch.load(buf, weights_only=False)
    assert size < 4 * opt.n * 4 + 65536                        # compact tensors, not views of the whole bucket
    params2 = [p.detach().clone().requires_grad_(True) for p in params]
    opt2 = _make(case, params2, groups, _lr(z, case, 1))
    opt2.load_state_dict(loaded)
    for step in range(4, oo.NSTEPS + 1):
        for o, ps in ((opt, params), (opt2, params2)):
            _step(o, ps, grads[step - 1], _lr(z, case, step), max_norm=5.0)
    assert torch.equal(opt.flat_params, opt2.flat_params)
    a, b = opt.state_dict()["state"], opt2.state_dict()["state"]
    for k in a:
        for kk, v in a[k].items():
            assert (torch.equal(v, b[k][kk]) if torch.is_tensor(v) else v == b[k][kk]), (k, kk)


def test_load_state_dict_mismatches_raise(z):
    init, _, groups, _, _ = oo.fixture(z, "adamw2")
    params = _params(init)
    opt = _make("adamw2", params, groups, 1e-3)
    sd = opt.state_dict()
    with pytest.raises(ValueError, match="number of parameter groups"):
        opt.load_state_dict(dict(sd, param_groups=sd["param_groups"][:1]))
    bad = dict(sd, param_groups=[dict(sd["param_groups"][0], params=[0]), sd["param_groups"][1]])
    with pytest.raises(ValueError, match="size"):
        opt.load_state_dict(bad)
    st = {0: {"step": 1, "exp_avg": torch.zeros(3, 3), "exp_avg_sq": torch.zeros(5, 9)}}
    with pytest.raises(ValueError, match="shape"):
        opt.load_state_dict(dict(sd, state=st))
    with pytest.raises(ValueError, match="amsgrad"):
        opt.load_state_dict(dict(sd, param_groups=[dict(g, amsgrad=True) for g in sd["param_groups"]]))
    with pytest.raises(RuntimeError, match="add_param_group"):
        opt.add_param_group({"params": [torch.zeros(2, device="cuda", requires_grad=True)]})


def test_schedulers_reach_the_next_step():
    from edgedict_b200 import optim
    p = torch.zeros(8, device="cuda", requires_grad=True)
    opt = optim.SGD([p], lr=1.0)
    lam = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.25 * (e + 1))
    opt.zero_grad()
    p.grad.fill_(1.0)
    opt.step()
    assert torch.all(p.detach() == -0.25)
    lam.step()
    opt.step()
    assert torch.all(p.detach() == -0.75)
    plateau = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, factor=0.5, patience=0)
    plateau.step(1.0)
    plateau.step(1.0)
    assert opt.param_groups[0]["lr"] == 0.25
    opt.step()
    assert torch.all(p.detach() == -1.0)
    opt.param_groups[0]["lr"] = 0.125                          # the warm-up write of cli/train.py
    opt.step()
    assert torch.all(p.detach() == -1.125)


@pytest.mark.parametrize("case", CASES)
def test_overflow_skip_leaves_everything_unchanged(z, case):
    init, grads, groups, _, _ = oo.fixture(z, case)
    params = _params(init)
    opt = _make(case, params, groups, _lr(z, case, 1))
    _step(opt, params, grads[0], _lr(z, case, 1))
    before_p = opt.flat_params.clone()
    before = opt.state_dict()
    steps = opt._steps.clone()
    opt.zero_grad()
    params[2].grad[1, 1] = float("inf")
    opt.step(grad_scale=1.0 / 1024, check_overflow=True)
    assert torch.equal(before_p, opt.flat_params)
    assert torch.equal(steps, opt._steps)
    after = opt.state_dict()
    for k, st in before["state"].items():
        for kk, v in st.items():
            assert (torch.equal(v, after["state"][k][kk]) if torch.is_tensor(v) else v == after["state"][k][kk])
    _step(opt, params, grads[1], _lr(z, case, 2))                # the next finite step is taken as step 2
    if case != "sgd":
        assert all(st["step"] == 2 for st in opt.state_dict()["state"].values())


@pytest.mark.parametrize("case", CASES)
def test_bitwise_invariants(z, case):
    init, grads, groups, _, _ = oo.fixture(z, case)

    def run(order=None, split=False, **kw):
        params = _params(init)
        if split:     # one group cut in two with the same hyperparameters
            from edgedict_b200 import optim
            cls, ckw, _ = oo.HYPER[case]
            opt = getattr(optim, cls)([{"params": params[:2]}, {"params": params[2:]}], lr=_lr(z, case, 1), **ckw)
        else:
            opt = _make(case, params, groups, _lr(z, case, 1), order)
        for step in range(1, oo.NSTEPS + 1):
            _step(opt, params, grads[step - 1], _lr(z, case, step), **kw)
        return [p.detach().clone() for p in params]

    a, b = run(max_norm=3.0), run(max_norm=3.0)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    plain = run()
    perm = run(order=list(reversed(range(len(init)))))
    assert all(torch.equal(x, y) for x, y in zip(plain, perm))
    if case != "adamw2":
        assert all(torch.equal(x, y) for x, y in zip(plain, run(split=True)))


def test_adamw_matches_flat_adamw():
    from edgedict_b200.optim import AdamW, FlatAdamW
    torch.manual_seed(2)
    net = torch.nn.Sequential(torch.nn.Linear(13, 7), torch.nn.Tanh(), torch.nn.Linear(7, 5)).cuda()
    net2 = torch.nn.Sequential(torch.nn.Linear(13, 7), torch.nn.Tanh(), torch.nn.Linear(7, 5)).cuda()
    net2.load_state_dict(net.state_dict())
    a = AdamW(net.parameters(), lr=3e-3, weight_decay=1e-2)
    b = FlatAdamW(net2, lr=3e-3, weight_decay=1e-2)
    for step in range(1, 6):
        gen = torch.Generator().manual_seed(100 + step)
        gs = [torch.randn(p.shape, generator=gen).cuda() for p in net.parameters()]
        a.zero_grad()
        b.zero_grad()
        for p, q, g in zip(net.parameters(), net2.parameters(), gs):
            p.grad.copy_(g)
            q.grad.copy_(g)
        a.step()
        b.step()
        for p, q in zip(net.parameters(), net2.parameters()):
            assert rel_err(p.detach().cpu(), q.detach().cpu()) < 1e-6, step


def test_sm3_large_shapes_against_oracle():
    """Tiles of many rows, rows longer than one tile, rank 3 and 4: the shared-memory maxima and their flush."""
    from edgedict_b200.optim import SM3
    gen = torch.Generator().manual_seed(5)
    shapes = [(300, 77), (3, 9000), (20000,), (17, 5, 33), (4, 3, 5, 7), (2048, 1)]
    init = [torch.randn(s, generator=gen).numpy() for s in shapes]
    params = _params(init)
    opt = SM3(params, lr=0.05)
    gsteps = [[torch.randn(s, generator=gen).numpy() for s in shapes] for _ in range(3)]
    want = oo.run("sm3", init, [(g, [dict(lr=0.05, eps=1e-30)]) for g in gsteps], [0] * len(shapes))
    for step, gs in enumerate(gsteps):
        _step(opt, params, gs, 0.05)
        for i, p in enumerate(params):
            assert rel_err(p.detach().cpu().numpy(), want[step][0][i]) < 2e-5, (step, shapes[i])
    st = _state_by_param(opt, params)
    for i in range(len(shapes)):
        for k, v in st[i].items():
            if torch.is_tensor(v):
                assert rel_err(v.cpu().numpy(), want[-1][1][i][k]) < 2e-5, (shapes[i], k)


def test_greedy_decode_runs_after_rehoming():
    from edgedict_b200.optim import SGD
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(3)
    model = Transducer(vocab_embed_size=16, vocab_size=64, input_size=24, enc_hidden_size=48, enc_layers=2,
                       enc_dropout=0, enc_proj_size=40, dec_hidden_size=32, dec_layers=1, dec_dropout=0,
                       dec_proj_size=24, joint_size=56).cuda()
    xs = torch.randn(2, 15, 24, device="cuda")
    xlen = torch.tensor([15, 11], dtype=torch.int32)
    before = model.greedy_decode(xs, xlen)
    opt = SGD(list(model.parameters()), lr=0.1)
    after = model.greedy_decode(xs, xlen)
    assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(before[0], after[0]))
    opt.zero_grad()
    opt.step()                                                 # zero gradients: the weights keep their values
    again = model.greedy_decode(xs, xlen)
    assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(before[0], again[0]))
