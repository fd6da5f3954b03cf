"""CPU-side checks of the flat-bucket optimizers (edgedict_b200.optim.SGD / SM3 / AdamW / Novograd): the fp64 oracle
against the reference's recorded steps (tests/golden/optim_tiny.npz), constructor validation with the reference's
messages, the refused options, the C entries' argument checks, the bucket's segment and tile tables, and the one-step
fp64 restatement of tests/optim_restate.py pinned against the oracle.  No GPU needed."""
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


# ---- the bucket tables (optim.bucket_tables) and the fp64 one-step restatement (tests/optim_restate.py) ---------------
from tests import optim_restate as rs          # noqa: E402

TABLE_SHAPES = ([(2, c) for c in (1, 3, 4, 5, 767, 768, 769, 1024, 4095, 4096, 4097, 8192, 8193)] +
                [(r, 1) for r in (1023, 1024, 1025, 2049)] + [(1025, 16), (964, 17), (1024, 16), (963, 17)] +
                [(), (1,), (5,), (6,), (7,), (8193,), (140000,), (33 * 1024 + 100, 1), (3, 1, 5), (1, 4, 6),
                 (2, 3, 1, 5), (3, 2, 4, 7), (1, 1, 1, 1), (0,), (0, 5), (3, 0, 2), (2, 1, 0, 3), (3, 3), (5, 7, 9)])


def test_tile_table_covers_every_element_once_within_the_sm3_caps():
    from edgedict_b200.optim import TILE_COLS, TILE_ELEMS, TILE_ROWS, bucket_tables
    seg, tiles, offs, n, nacc = bucket_tables([TABLE_SHAPES[0::2], TABLE_SHAPES[1::2]])
    shapes = TABLE_SHAPES[0::2] + TABLE_SHAPES[1::2]
    assert n == sum((int(np.prod(s)) + 3) // 4 * 4 for s in shapes)
    for i, (row, s) in enumerate(zip(seg, shapes)):
        k = int(np.prod(s))
        C = s[-1] if s else 1
        assert row[0] == offs[i] and offs[i] % 4 == 0
        mine = tiles[row[4]:row[5]]
        assert all(t[0] == i for t in mine)
        covered = 0
        for t in mine:
            _, start, ln, r0, c0, ncols = t
            assert ncols > 0 and ln > 0 and ln % ncols == 0            # sm3_kernel: nrows = len / ncols
            assert ncols <= TILE_COLS and ln // ncols <= TILE_ROWS and ln <= TILE_ELEMS
            assert start == covered                                    # in order, no gap, no overlap
            assert start == r0 * C + c0 and 0 <= c0 and c0 + ncols <= C
            assert c0 == 0 and ncols == C if C <= TILE_COLS else ln == ncols
            covered += ln
        assert covered == k, (s, covered)
    assert tiles == [t for row in seg for t in tiles[row[4]:row[5]]] and seg[-1][5] == len(tiles)
    assert bucket_tables([[(0,), (0, 3)], [(2, 0, 1)]])[1] == []              # an all-empty bucket has no tile


def _header_fields(name):
    src = open(os.path.join(HERE, "..", "include", "edgedict_b200.h")).read()
    import re
    body = re.search(r"typedef struct \{ long long ([^;]*); \} %s;" % name, src).group(1)
    out = []
    for f in body.split(","):
        f = f.strip()
        m = re.fullmatch(r"(\w+)\[(\d+)\]", f)
        out += ["%s%d" % (m.group(1), d) for d in range(int(m.group(2)))] if m else [f]
    return out


def test_table_rows_follow_the_c_structs_field_order():
    from edgedict_b200.optim import bucket_tables
    assert _header_fields("eb_opt_seg") == ["off", "numel", "rank", "group", "tile_begin", "tile_end", "shape0",
                                            "shape1", "shape2", "shape3", "acc0", "acc1", "acc2", "acc3"]
    assert _header_fields("eb_opt_tile") == ["seg", "start", "len", "r0", "c0", "ncols"]
    seg, tiles, _, _, nacc = bucket_tables([[(5,), (3, 4, 2)], [(), (2, 5000)]])
    f = _header_fields("eb_opt_seg")
    rows = [dict(zip(f, r)) for r in seg]
    assert rows[1] == dict(off=8, numel=24, rank=3, group=0, tile_begin=1, tile_end=2, shape0=3, shape1=4, shape2=2,
                           shape3=0, acc0=5, acc1=8, acc2=12, acc3=0)
    assert rows[2]["acc0"] == 14 and rows[2]["numel"] == 1 and rows[2]["group"] == 1
    assert rows[3]["acc0"] == 15 and rows[3]["acc1"] == 17 and nacc == 5017
    assert [dict(zip(_header_fields("eb_opt_tile"), t)) for t in tiles[3:]] == [
        dict(seg=3, start=s, len=k, r0=r, c0=c, ncols=k) for r in (0, 1) for c, k in ((0, 4096), (4096, 904))
        for s in [r * 5000 + c]]


def test_sumsq_terms_reads_the_loop_bounds():
    assert rs.sumsq_terms(1) == (1, False)
    assert rs.sumsq_terms(768) == (3, False)
    assert rs.sumsq_terms(769) == (3, True)                    # thread 0 takes one body trip, thread 1 three tail
    assert rs.sumsq_terms(1024) == (1, True)
    assert rs.sumsq_terms(1025) == (2, True)                   # thread 0: one trip, then element 1024
    assert rs.sumsq_terms(16384) == (16, True)
    assert rs.sumsq_terms(4096 + 768) == (7, True)             # 4 trips, then 3 tail elements of thread 0 (j < 4864)


@pytest.mark.parametrize("case", sorted(oo.HYPER))
def test_restatement_chained_matches_the_oracle_and_the_fixture(z, case):
    """Six one-step restatements chained on their own fp64 outputs reproduce tests/optim_oracle.run (to fp64 rounding)
    and the reference's recorded steps."""
    from edgedict_b200.optim import bucket_tables
    init, grads, groups, hyp, two = oo.fixture(z, case)
    kind = oo.KIND[case]
    ng = 2 if two else 1
    order = [[i for i in range(len(init)) if groups[i] == gi] for gi in range(ng)]
    flat = [i for o in order for i in o]
    seg, tiles, offs, n, nacc = bucket_tables([[np.shape(init[i]) for i in o] for o in order])
    L = rs.Layout(seg, tiles, n, "cpu")

    def bucket(arrs):
        b = torch.full((n,), float("nan"), dtype=torch.float64)
        for k, i in enumerate(flat):
            b[offs[k]:offs[k] + np.size(init[i])] = torch.as_tensor(np.asarray(arrs[i], dtype=np.float64)).reshape(-1)
        return b

    def scatter(vals):
        b = torch.full((n,), float("nan"), dtype=torch.float64)
        b[L.pos] = vals
        return b

    want = oo.run(kind, init, list(zip(grads, hyp)), groups)
    p = bucket(init)
    st = {k: torch.zeros(n, dtype=torch.float64) for k in ("buf", "m", "v")}
    segv = torch.zeros(len(seg), dtype=torch.float64)
    acc = torch.zeros(nacc, dtype=torch.float64)
    for step in range(1, oo.NSTEPS + 1):
        h = {k: [hg[kk] for hg in hyp[step - 1]] for k, kk in (("lr", "lr"), ("wd", "wd"), ("b1", "b1"), ("b2", "b2"),
                                                             ("eps", "eps"))}
        g = bucket(grads[step - 1])
        steps = [step] * ng
        if kind == "sgd":
            out, _ = rs.sgd(L, p, g, st["buf"], h, steps, 1.0)
            st["buf"] = scatter(out["buf"][0])
        elif kind == "adamw":
            out = rs.adamw(L, p, g, st["m"], st["v"], h, steps, 1.0)
            st["m"], st["v"] = scatter(out["m"][0]), scatter(out["v"][0])
        elif kind == "novograd":
            _, _, ssum, _ = rs.seg_sumsq(L, g)
            segv, _ = rs.novograd_v(seg, ssum, segv, h, 1.0)
            out = rs.novograd(L, p, g, st["m"], segv, h, 1.0)
            st["m"] = scatter(out["m"][0])
        else:
            out, _ = rs.sm3(L, p, g, acc, nacc, h, 1.0)
            acc = out["acc"][0]
        p = scatter(out["p"][0])
        wp, ws = want[step - 1]
        for k, i in enumerate(flat):
            mine = p[offs[k]:offs[k] + np.size(init[i])].numpy().reshape(np.shape(init[i]))
            np.testing.assert_allclose(mine, wp[i], rtol=1e-12, atol=1e-15)
            assert rel_err(mine, z["%s.p.%d.%d" % (case, step, i)]) < 1e-5, (case, step, i)
            if kind == "novograd":
                assert abs(float(segv[k]) - float(ws[i]["exp_avg_sq"])) <= 1e-12 * abs(float(ws[i]["exp_avg_sq"]))
            if kind == "sm3" and np.ndim(init[i]) >= 2:
                for d, nd in enumerate(np.shape(init[i])):
                    a0 = seg[k][10 + d]
                    np.testing.assert_array_equal(acc[a0:a0 + nd].numpy(), ws[i]["accumulator_%d" % d].reshape(-1))
