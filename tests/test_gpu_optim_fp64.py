"""Per-element fp64 parity and bitwise invariants of every csrc/optim.cu kernel, each through its C entry point
(``ops.opt_*``), on bucket tables built by ``optim.bucket_tables`` (the builder ``FlatOptimizer`` uses).

Error model.  The build uses no fast-math: division and sqrtf are IEEE, but nvcc may contract a*b + c into one FMA, which
only removes a rounding.  u = 2^-24 is the fp32 unit roundoff.  Each kernel is teacher-forced: it reads fp32 p, g and
state, the ctl / steps the prologue wrote, and the hyperparameters as the C ABI receives them (fp64, converted to fp32
by the kernel: each conversion is one rounding).  The restatement (tests/optim_restate.py) is one step in fp64 from the
same values; an element's bar is k u M, M the expression on absolute values and k the number of fp32 roundings in it,
counted without contraction (an upper bound), times 1 + 2^-10 for the second-order terms, plus k 2^-149:

  eb_opt_seg_sumsq   partial, per tile: (m + 12) u sum g^2, m the most squares one accumulator sums (read off the loop
                     bounds: four-accumulator body trips plus tail trips), 12 the levels after it ((a0 + a1) + (a2 + a3),
                     two five-level warp_sums).  segsum: its tiles' bars, the fp64 adds and one rounding to fp32.  The
                     fp64 lane-strided sum of the kernel's own partials (lane l takes tiles l, l + 32, ..., then a xor
                     butterfly 16 ... 1) and total (the segsums added in order in fp64) involve no multiply, so they are
                     restated in that order and asserted bit for bit.
  eb_opt_prologue    ctl[0] = gs min(1, max_norm / (sqrt(total) |gs| + 1e-6)) from the kernel's total: 6 roundings
                     (sqrtf, x |gs|, fp32(1e-6), the add, the division, coef x c) relative to |ctl[0]|; the skip flag
                     exactly !isfinite(fp32(sqrtf(total) |gs|)); the counters advance by exactly 1, or not at all on a skip;
                     total = NULL gives ctl[0] = gs bit for bit.
  eb_opt_sgd_step    buf 7 roundings (first step 4), p 3 from the kernel's buf, or 7 where momentum is 0.
  eb_opt_adamw_step  m 6, v 8, p 10 from the kernel's m and v with the step size formed in fp64 from the counter.
  eb_opt_novograd    segv 2 (v == 0: n = coef^2 segsum) or 7, from the kernel's segsum; m 11 from the kernel's segv; p 3
                     from the kernel's m.
  eb_opt_sm3_step    u = min acc + (coef g)^2: 4 roundings of non-negative terms (2 when coef = 1, where coef g is
                     exact); the maxima are exact selections, so a new accumulator carries u's bar at the maximum, and at
                     coef = 1 it is within 1 ulp of fp32(the fp64 maximum) (each u is fp32(a + g^2) or fp32(a +
                     fp32(g^2)): at most 1.5 ulp from the exact value, so at most 1 ulp from its rounding; max is monotone).
                     p: u's k, + eps and fp32(eps) halved through sqrtf, then 6 more: k + 8.

Every buffer has G NaN guard elements at both ends; the bucket's pads (each tensor rounded up to 4 elements) hold NaN in
p, g and every state; pure outputs are NaN-prefilled.  After each call the guards and pads are still NaN, and an output is
NaN exactly where its restatement is.  Each barred check prints its worst err/bar (pytest -s); DESIGN.md section 2
records the measured figures.  The case tables reach every loop trip count, and the reach is asserted (``test_reach``)."""
import math

import numpy as np
import pytest
import torch

from tests import optim_restate as rs

pytestmark = pytest.mark.gpu

f32, f64, i32 = torch.float32, torch.float64, torch.int32
DEV = "cuda"
G = 64
NAN = float("nan")
NG = 16

# the edges of the tile table: last dimensions around the main loop (768), a warp row, the column cap (4096) and one
# piece of a row (C > 4096: c0 != 0); the row cap (C = 1, 16, 17); ranks 0 - 4 with dimensions of size 1; numel % 4 in
# {1, 2, 3}; empty tensors among the others; tensors of more than 32 tiles
EDGE = ([(2, c) for c in (1, 3, 4, 5, 767, 768, 769, 1024, 4095, 4096, 4097, 8192, 8193)] + [(8193,)] +
        [(r, 1) for r in (1023, 1024, 1025, 2049)] + [(1025, 16), (964, 17)] +
        [(), (0,), (5,), (6,), (0, 5), (7,), (3, 1, 5), (1, 4, 6), (3, 0, 2), (2, 3, 1, 5), (3, 2, 4, 7), (1, 1, 1, 1),
         (5, 7, 9), (33 * 1024 + 100, 1), (140000,), (3, 3)])
SMALL = [(3,), (2, 2), (1, 5), (), (6,), (2, 1, 3)]


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid(ntiles):
    return min(ntiles, 8 * sms())


def e6d2_shapes():
    from edgedict_b200.rnnt.models import Transducer
    from scripts.bench_optim import E6D2
    with torch.device("meta"):
        model = Transducer(**E6D2)
    return [tuple(p.shape) for p in model.parameters()]


class Bucket:
    def __init__(self, group_shapes, keys=None):
        from edgedict_b200.optim import bucket_tables
        self.group_shapes = group_shapes
        self.shapes = [tuple(s) for gs in group_shapes for s in gs]
        self.keys = list(range(len(self.shapes))) if keys is None else keys
        self.seg, self.tiles, self.offs, self.n, self.nacc = bucket_tables(group_shapes)
        self.ngroups = len(group_shapes)
        self.L = rs.Layout(self.seg, self.tiles, self.n, DEV)
        self.seg_t = torch.tensor(self.seg, dtype=torch.int64, device=DEV)
        self.tiles_t = torch.tensor(self.tiles, dtype=torch.int64, device=DEV)
        self.cov = self.L.covered()

    def acc_len(self, i):
        s = self.shapes[i]
        return max(int(np.prod(s)), 1) if len(s) <= 1 else sum(s)


def round_robin(shapes, ngroups=NG):
    gs = [[] for _ in range(ngroups)]
    for i, s in enumerate(shapes):
        gs[i % ngroups].append(s)
    return gs


_BUCKETS = {}


def bucket(name):
    if name not in _BUCKETS:
        if name == "edge":
            many = [SMALL[i % len(SMALL)] for i in range(2 * 8 * sms() + 40)]
            _BUCKETS[name] = Bucket(round_robin(EDGE + many))
        elif name == "e6d2":      # the wav2vec-style split: matrices decayed, vectors not
            sh = e6d2_shapes()
            _BUCKETS[name] = Bucket([[s for s in sh if len(s) >= 2], [s for s in sh if len(s) < 2]])
        elif name == "skip":      # nacc > grid x 256: the skipped SM3 step's copy strides
            _BUCKETS[name] = Bucket(round_robin(EDGE[:20] + [(300000,)], 3))
    return _BUCKETS[name]


# ---- buffers ---------------------------------------------------------------------------------------------------------
def guarded(n, dtype=f32, fill=NAN):
    return torch.full((n + 2 * G,), fill, dtype=dtype, device=DEV)


def view(full):
    return full[G:-G]


def bucket_buf(B, vals):
    full = guarded(B.n)
    if vals is not None:
        view(full)[B.L.pos] = vals
    return full


def bits(x):
    return x.view(torch.int32) if x.dtype == f32 else x


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def check_frame(B, full, what, n=None):
    assert full[:G].isnan().all() and full[-G:].isnan().all(), (what, "guard written")
    if n is None:
        assert view(full)[~B.cov].isnan().all(), (what, "pad written")


WORST = {}


def check(what, got, want, bar):
    """got (fp32) within bar of want (fp64) per element; NaN exactly where want is NaN; infinities equal."""
    got = got.to(f64)
    assert torch.equal(got.isnan(), want.isnan()), (what, "NaN where the restatement has none, or the reverse",
                                                    int((got.isnan() != want.isnan()).sum()))
    inf = want.isinf()
    assert torch.equal(got[inf], want[inf]), (what, "infinity")
    ok = torch.isfinite(want)
    if not ok.any():
        return 0.0
    r = float(((got[ok] - want[ok]).abs() / bar[ok]).max())
    WORST[what] = max(WORST.get(what, 0.0), r)
    print("%-28s worst err/bar %.3f" % (what, r))
    assert r <= 1.0, (what, r)
    return r


def ophyper(h):
    from edgedict_b200._lib import OptHyper
    o = OptHyper()
    for k in ("lr", "wd", "b1", "b2", "eps"):
        for i, x in enumerate(h[k]):
            getattr(o, k)[i] = x
    return o


# ---- per-group hyperparameters: distinct in every group and field -------------------------------------------------
def hyper(kind, ngroups=NG):
    i = np.arange(NG)
    h = dict(lr=list(10.0 ** (-3 + 2 * i / 15)), wd=[0.0 if k % 3 == 0 else 1e-4 * (k + 1) for k in i],
             b1=list(0.5 + 0.03 * i), b2=list(0.99 + 0.0006 * i), eps=list(1e-8 * (i + 1)))
    if kind == "sgd":
        h["b1"] = [0.0 if k % 4 == 1 else (0.9 if k == 0 else 0.5 + 0.03 * k) for k in i]
        h["b2"], h["eps"] = [0.0] * NG, [0.0] * NG
    elif kind == "adamw":
        h["b1"][3] = 0.0
        h["eps"][5] = 1.0                                         # eps dominates sqrt(v)
    elif kind == "novograd":
        h["b2"] = [0.0 if k % 2 == 0 else 0.25 + 0.04 * k for k in i]        # b2 = 0: the reference's default
    elif kind == "sm3":
        h["wd"], h["b1"], h["b2"] = [0.0] * NG, [0.0] * NG, [0.0] * NG
        h["eps"] = [1e-30 if k % 2 == 0 else 1e-8 * (k + 1) for k in i]
    return {k: [float(x) for x in v[:ngroups]] for k, v in h.items()}


COUNTERS = [1, 2, 1000, 1, 5, 3, 1, 7, 2, 50, 1, 4, 9, 1, 2, 11]      # after the prologue; unequal across groups


# ---- seeded per-tensor data: a tensor's values depend on (seed, its key) only, not on where it sits ---------------
def draw(B, seed, zero_grad=()):
    L = B.L
    out = {k: torch.empty(L.pos.numel(), dtype=f32, device=DEV) for k in ("p", "g", "buf", "m", "v")}
    acc = torch.zeros(B.nacc, dtype=f32, device=DEV)
    segv = torch.zeros(len(B.seg), dtype=f32, device=DEV)
    cum = 0
    for i, (row, key) in enumerate(zip(B.seg, B.keys)):
        k = row[1]
        gen = torch.Generator(device=DEV).manual_seed(seed * 100003 + key)
        sc = 10.0 ** (4 * torch.rand(5, generator=gen, device=DEV) - 2)
        r = torch.randn(5, max(k, 1), generator=gen, device=DEV)
        sl = slice(cum, cum + k)
        out["p"][sl] = r[0, :k] * sc[0]
        out["g"][sl] = 0.0 if key in zero_grad else r[1, :k] * sc[1]
        out["buf"][sl] = r[2, :k] * sc[2]
        out["m"][sl] = r[3, :k] * sc[3]
        out["v"][sl] = r[4, :k] ** 2 * sc[4] ** 2
        na = B.acc_len(i)
        a = torch.floor(torch.randn(na, generator=gen, device=DEV).abs() * 4) / 4 * sc[1] ** 2   # ties and zeros
        acc[row[10]:row[10] + na] = a
        segv[i] = 0.0 if key % 2 == 0 else float(r[4, 0] ** 2 * sc[1] ** 2 * max(k, 1))
        cum += k
    out["acc"], out["segv"] = acc, segv
    return out


class Step:
    """One step of ``kind`` through the C entries on guarded buffers: seg_sumsq (when clipping or for Novograd), the
    prologue, the update.  Keeps the inputs (``before``), the outputs, coef = ctl[0] and the counters after."""

    def __init__(self, B, D, kind, h, counters, gs=0.75, clip=True, check_overflow=False, tiles=None, no_buf=False):
        from edgedict_b200 import ops
        self.B, self.kind, self.h = B, kind, h
        self.buf = {"p": bucket_buf(B, D["p"]), "g": bucket_buf(B, D["g"])}
        first = torch.tensor(counters, device=DEV)[B.L.egroup] <= 1
        if kind == "sgd" and not no_buf:
            self.buf["buf"] = bucket_buf(B, torch.where(first, NAN, D["buf"]))     # never read on a first step
        if kind in ("adamw", "novograd"):
            self.buf["m"] = bucket_buf(B, D["m"])
        if kind == "adamw":
            self.buf["v"] = bucket_buf(B, D["v"])
        if kind == "novograd":
            self.buf["segv"] = guarded(len(B.seg))
            view(self.buf["segv"]).copy_(D["segv"])
        if kind == "sm3":
            self.buf["acc"] = guarded(B.nacc)
            view(self.buf["acc"]).copy_(D["acc"])
            self.buf["acc_new"] = guarded(B.nacc)
        self.before = {k: v.clone() for k, v in self.buf.items()}
        self.partial, self.segsum, self.total = guarded(len(B.tiles)), guarded(len(B.seg)), guarded(1)
        self.ctl = guarded(2)
        self.steps = guarded(B.ngroups, i32, -777)
        view(self.steps).copy_(torch.tensor(counters[:B.ngroups], dtype=i32) - 1)
        clip = clip or check_overflow
        gv = view(self.buf["g"])
        if clip or kind == "novograd":
            ops.opt_seg_sumsq(gv, B.seg_t, B.tiles_t, view(self.partial), view(self.segsum),
                              view(self.total) if clip else None)
        max_norm = 0.0
        if clip and not check_overflow:
            max_norm = 0.5 * math.sqrt(float(view(self.total)[0])) * abs(gs)             # clip active: c ~ 0.5
        ops.opt_prologue(view(self.total) if clip else None, gs, max_norm, view(self.steps), view(self.ctl))
        tl = B.tiles_t if tiles is None else tiles
        hp = ophyper(h)
        v = {k: view(x) for k, x in self.buf.items()}
        if kind == "sgd":
            ops.opt_sgd_step(v["p"], v["g"], v.get("buf"), B.seg_t, tl, hp, view(self.steps), view(self.ctl))
        elif kind == "adamw":
            ops.opt_adamw_step(v["p"], v["g"], v["m"], v["v"], B.seg_t, tl, hp, view(self.steps), view(self.ctl))
        elif kind == "novograd":
            ops.opt_novograd_step(v["p"], v["g"], v["m"], v["segv"], view(self.segsum), B.seg_t, tl, hp,
                                  view(self.steps), view(self.ctl))
        else:
            ops.opt_sm3_step(v["p"], v["g"], v["acc"], v["acc_new"], B.seg_t, tl, hp, view(self.steps),
                             view(self.ctl))
        torch.cuda.synchronize()
        self.coef = float(view(self.ctl)[0])
        self.skipped = float(view(self.ctl)[1]) != 0.0
        self.counters = view(self.steps).tolist()

    def out(self, k):
        return view(self.buf[k])

    def inp(self, k):
        return view(self.before[k])

    def at(self, k):
        return self.out(k)[self.B.L.pos]

    def check_frames(self):
        B = self.B
        for k, full in self.buf.items():
            check_frame(B, full, (self.kind, k), n=None if k in ("p", "g", "buf", "m", "v") else 0)
        for full in (self.partial, self.segsum, self.total, self.ctl):
            check_frame(B, full, (self.kind, "sumsq/ctl"), n=0)
        assert (self.steps[:G] == -777).all() and (self.steps[-G:] == -777).all()
        assert same_bits(self.out("g"), self.inp("g")), "g written"

    def check_restatement(self, tag):
        """Every output of the step against its fp64 restatement, teacher-forced as the module docstring states."""
        B, L, h, coef, cn = self.B, self.B.L, self.h, self.coef, self.counters
        self.check_frames()
        p, g = self.inp("p").double(), self.inp("g").double()
        if self.kind == "sgd":
            has = "buf" in self.buf
            buf = self.inp("buf").double() if has else torch.zeros_like(p)
            out, has_mu = rs.sgd(L, p, g, buf, h, cn, coef, buf_new=self.out("buf").double() if has else None)
            if has:
                check(tag + " sgd buf", self.at("buf")[has_mu], out["buf"][0][has_mu], out["buf"][1][has_mu])
                assert same_bits(self.at("buf")[~has_mu], self.inp("buf")[L.pos][~has_mu]), "buf of momentum 0"
            check(tag + " sgd p", self.at("p"), *out["p"])
        elif self.kind == "adamw":
            out = rs.adamw(L, p, g, self.inp("m").double(), self.inp("v").double(), h, cn, coef,
                           m_new=self.out("m").double(), v_new=self.out("v").double())
            for k in ("m", "v", "p"):
                check(tag + " adamw " + k, self.at(k), *out[k])
        elif self.kind == "novograd":
            segsum = view(self.segsum).double()
            want, b = rs.novograd_v(B.seg, segsum, self.inp("segv").double(), h, coef)
            check(tag + " novograd segv", self.out("segv"), want, b)
            out = rs.novograd(L, p, g, self.inp("m").double(), self.out("segv"), h, coef, m_new=self.out("m").double())
            for k in ("m", "p"):
                check(tag + " novograd " + k, self.at(k), *out[k])
        else:
            out, _ = rs.sm3(L, p, g, self.inp("acc"), B.nacc, h, coef)
            check(tag + " sm3 acc", self.out("acc_new"), *out["acc"])
            check(tag + " sm3 p", self.at("p"), *out["p"])
            assert same_bits(self.out("acc"), self.inp("acc")), "acc written"
        return out


KINDS = ["sgd", "adamw", "novograd", "sm3"]


# ---- reach ---------------------------------------------------------------------------------------------------------
def test_reach():
    """The case tables reach what the kernels' loops and branches depend on."""
    B = bucket("edge")
    nt = len(B.tiles)
    assert nt >= 2 * grid(nt) and grid(nt) == 8 * sms()               # every block runs at least two tiles
    assert len(B.seg) > 32                                            # the reduce kernel's warps loop over segments
    assert max(r[5] - r[4] for r in B.seg) > 32                       # its lanes loop over a tensor's tiles
    reach = [rs.sumsq_terms(t[2])[1] for t in B.tiles]
    assert any(reach) and not all(reach)                              # tiles in the four-accumulator body and tail-only
    assert any(t[4] != 0 for t in B.tiles)                            # pieces of one row
    assert max(t[2] // t[5] for t in B.tiles) == 1024                 # the row cap
    assert B.ngroups == NG and len(set(COUNTERS)) > 1
    assert {len(s) for s in B.shapes} == {0, 1, 2, 3, 4}
    assert {int(np.prod(s)) % 4 for s in B.shapes} == {0, 1, 2, 3} and any(np.prod(s) == 0 for s in B.shapes)
    E = bucket("e6d2")
    assert len(E.tiles) == 3088 and len(E.seg) == 55 and len(E.tiles) > 2 * grid(len(E.tiles))
    assert max(r[5] - r[4] for r in E.seg) == 256
    S = bucket("skip")
    assert S.nacc > grid(len(S.tiles)) * 256


# ---- eb_opt_seg_sumsq ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["edge", "e6d2"])
def test_seg_sumsq(name):
    from edgedict_b200 import ops
    B = bucket(name)
    D = draw(B, 11)
    g = bucket_buf(B, D["g"])
    partial, segsum, total = guarded(len(B.tiles)), guarded(len(B.seg)), guarded(1)
    ops.opt_seg_sumsq(view(g), B.seg_t, B.tiles_t, view(partial), view(segsum), view(total))
    tsum, tbar, ssum, sbar = rs.seg_sumsq(B.L, view(g))
    check(name + " sumsq partial", view(partial), tsum, tbar)
    check(name + " sumsq segsum", view(segsum), ssum, sbar)
    order, tot = rs.segsum_in_order(B.seg, view(partial).cpu().numpy())
    assert np.array_equal(view(segsum).cpu().numpy().view(np.int32), order.view(np.int32))
    assert view(total).cpu().numpy().view(np.int32)[0] == np.float32(tot).view(np.int32)
    for full in (g, partial, segsum, total):
        check_frame(B, full, "sumsq", n=0)
    assert view(g)[~B.cov].isnan().all()
    # repeated launches, and total = NULL leaves total alone
    p2, s2, t2 = guarded(len(B.tiles)), guarded(len(B.seg)), guarded(1)
    ops.opt_seg_sumsq(view(g), B.seg_t, B.tiles_t, view(p2), view(s2), None)
    assert same_bits(p2, partial) and same_bits(s2, segsum) and t2.isnan().all()


# ---- eb_opt_prologue -----------------------------------------------------------------------------------------------
PROLOGUE = [   # (total, grad_scale, max_norm)
    (0.0, 0.5, 1.0), (1e-44, 1.0, 1e-7), (1e-44, 2.0, 0.0), (math.inf, 1.0, 1.0), (NAN, 1.0, 0.0),
    (4.0, 0.5, 0.999), (4.0, 0.5, 1.001), (4.0, -0.5, 0.25), (123.5, 1.0 / 1024, 0.01), (3e38, 1e20, 1.0),
    (3e38, 1.0, 1.0), (None, 0.3, 0.0), (None, -2.0, 5.0), (2.5e5, 3.0, 0.0),
]


@pytest.mark.parametrize("ngroups", [1, 2, 16])
def test_prologue(ngroups):
    from edgedict_b200 import ops
    for total, gs, max_norm in PROLOGUE:
        tot = guarded(1)
        if total is not None:
            view(tot)[0] = total
        ctl, steps = guarded(2), guarded(ngroups, i32, -777)
        init = torch.arange(ngroups, dtype=i32) * 3 + 2
        view(steps).copy_(init)
        ops.opt_prologue(view(tot) if total is not None else None, gs, max_norm, view(steps), view(ctl))
        c = view(ctl).cpu().numpy()
        gs32, mn32 = np.float32(gs), np.float32(max_norm)
        case = (total, gs, max_norm, ngroups)
        if total is None:
            skip = False
            assert c[0].view(np.int32) == gs32.view(np.int32), case
        else:
            t32 = np.float32(view(tot)[0].item())
            with np.errstate(over="ignore", invalid="ignore"):
                norm32 = np.float32(np.sqrt(t32)) * np.float32(abs(gs32))
            skip = not np.isfinite(norm32)
            if skip or mn32 == 0:
                assert c[0].view(np.int32) == gs32.view(np.int32), case
            else:
                cc = float(mn32) / (math.sqrt(float(t32)) * abs(float(gs32)) + 1e-6)
                want = float(gs32) * min(1.0, cc)
                assert abs(float(c[0]) - want) <= rs.bar(6, abs(want)), (case, float(c[0]), want)
        assert c[1] == (1.0 if skip else 0.0), case
        assert torch.equal(view(steps).cpu(), init + (0 if skip else 1)), case
        assert (steps[:G] == -777).all() and (steps[-G:] == -777).all()
        check_frame(None, ctl, "ctl", n=0)


# ---- the update kernels, one step, per element ---------------------------------------------------------------------
@pytest.mark.parametrize("name", ["edge", "e6d2"])
@pytest.mark.parametrize("kind", KINDS)
def test_step_per_element(kind, name):
    B = bucket(name)
    h = hyper(kind, B.ngroups)
    s = Step(B, draw(B, 23), kind, h, COUNTERS[:B.ngroups], gs=0.75, clip=True)
    assert not s.skipped and s.coef < 0.75 * 0.6                       # the clip is active
    assert s.counters == COUNTERS[:B.ngroups]
    s.check_restatement(name)


def test_sgd_without_buffer():
    """Every group's momentum 0: buf = NULL; p -= lr (coef g + wd p)."""
    B = bucket("edge")
    h = hyper("sgd")
    h["b1"] = [0.0] * NG
    s = Step(B, draw(B, 29), "sgd", h, COUNTERS, gs=1.5, clip=False, no_buf=True)
    assert s.coef == 1.5
    s.check_restatement("edge nobuf")


def test_sm3_accumulators_at_unit_scale():
    """gs = 1, no clip: g' = g exactly, and every new accumulator is within 1 ulp of fp32(the fp64 maximum)."""
    for name in ("edge", "e6d2"):
        B = bucket(name)
        s = Step(B, draw(B, 31), "sm3", hyper("sm3", B.ngroups), COUNTERS[:B.ngroups], gs=1.0, clip=False)
        assert s.coef == 1.0
        out = s.check_restatement(name + " gs=1")
        want32 = out["acc"][0].float()
        d = (s.out("acc_new").view(torch.int32).long() - want32.view(torch.int32).long()).abs()
        assert int(d.max()) <= 1, name
        print("%s sm3 accumulators: %d of %d bit for bit, the rest 1 ulp" % (name, int((d == 0).sum()), d.numel()))


def test_novograd_zero_gradient_then_nonzero():
    """A tensor whose gradient is all zero keeps v = 0; its next nonzero step takes v = n."""
    B = bucket("edge")
    zero = {1, 4, 7, 30}                                   # keys of tensors with zero gradients at the first step
    h = hyper("novograd")
    D = draw(B, 37, zero_grad=zero)
    D["segv"][:] = 0.0
    s1 = Step(B, D, "novograd", h, COUNTERS, gs=0.5, clip=True)
    s1.check_restatement("edge zero-grad")
    v1 = s1.out("segv")
    zi = [i for i, k in enumerate(B.keys) if k in zero and B.seg[i][1] > 0]
    assert all(float(v1[i]) == 0.0 for i in zi) and all(float(v1[i]) > 0 for i in range(len(B.seg))
                                                        if B.keys[i] not in zero and B.seg[i][1] > 0)
    D2 = draw(B, 38)
    D2["segv"], D2["p"], D2["m"] = v1.clone(), s1.at("p").clone(), s1.at("m").clone()
    s2 = Step(B, D2, "novograd", h, [c + 1 for c in COUNTERS], gs=0.5, clip=True)
    s2.check_restatement("edge after zero-grad")
    want_n = s2.coef ** 2 * view(s2.segsum).double()
    for i in zi:
        assert abs(float(s2.out("segv")[i]) - float(want_n[i])) <= rs.bar(2, float(want_n[i]))


@pytest.mark.parametrize("kind", KINDS)
def test_nonfinite_gradients(kind):
    """A NaN or +-inf gradient element, no overflow check: NaN (and infinities) exactly where the restatement has them."""
    B = bucket("edge")
    D = draw(B, 41)
    gcov = D["g"]
    for i, val in ((0, NAN), (13, math.inf), (26, -math.inf), (40, NAN)):
        row = B.seg[i]
        if row[1] == 0:
            continue
        first = int((B.L.pos == row[0]).nonzero()[0])
        gcov[first + row[1] // 2] = val
    s = Step(B, D, kind, hyper(kind), COUNTERS, gs=1.0, clip=False)
    assert not s.skipped
    s.check_restatement("edge nonfinite")


@pytest.mark.parametrize("kind", KINDS)
def test_skipped_step_changes_nothing(kind):
    """check_overflow with an inf gradient: ctl[1] = 1, every buffer and counter bit-identical; SM3 copies acc."""
    B = bucket("skip")
    D = draw(B, 43)
    D["g"][5] = math.inf
    s = Step(B, D, kind, hyper(kind, B.ngroups), COUNTERS[:B.ngroups], gs=0.5, check_overflow=True)
    assert s.skipped and s.counters == [c - 1 for c in COUNTERS[:B.ngroups]]
    s.check_frames()
    for k in s.buf:
        if k != "acc_new":
            assert same_bits(s.out(k), s.inp(k)), (kind, k)
    if kind == "sm3":
        assert same_bits(s.out("acc_new"), s.inp("acc"))


# ---- bitwise invariants --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_repeated_launches_same_bits(kind):
    B = bucket("edge")
    D = draw(B, 47)
    a = Step(B, D, kind, hyper(kind), COUNTERS)
    b = Step(B, D, kind, hyper(kind), COUNTERS)
    for k in a.buf:
        assert same_bits(a.buf[k], b.buf[k]), k
    for x, y in ((a.partial, b.partial), (a.segsum, b.segsum), (a.total, b.total), (a.ctl, b.ctl)):
        assert same_bits(x, y)


X = [(300, 77), (5000,), (3, 4, 5, 7), (1025, 3), (2, 8193), ()]          # the tensors that move


def _x_outputs(B, s, idx):
    """Per moved tensor: its p, state, partials, segsum (and SM3 accumulators, Novograd segv), as bits."""
    out = []
    for i in idx:
        row = B.seg[i]
        sl = slice(row[0], row[0] + row[1])
        d = {k: bits(s.out(k)[sl]).clone() for k in ("p", "buf", "m", "v") if k in s.buf}
        d["partial"] = bits(view(s.partial)[row[4]:row[5]]).clone()
        d["segsum"] = bits(view(s.segsum)[i:i + 1]).clone()
        if "segv" in s.buf:
            d["segv"] = bits(s.out("segv")[i:i + 1]).clone()
        if "acc_new" in s.buf:
            d["acc"] = bits(s.out("acc_new")[row[10]:row[10] + B.acc_len(i)]).clone()
        out.append(d)
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_tensor_bits_do_not_depend_on_position(kind):
    """The X tensors alone in group 0, then behind 2 x grid filler tiles (another block, another grid-stride trip), with
    other neighbours, in group 9 with group 0's hyperparameters: the same bits.  ctl is formed with total = NULL, so
    the coefficient does not depend on the bucket."""
    nf = 2 * 8 * sms() + 5
    keys_x = [10 ** 6 + k for k in range(len(X))]
    A = Bucket([X], keys=keys_x)
    filler = [SMALL[i % len(SMALL)] for i in range(nf)]
    gs9 = [filler[:nf // 2]] + [[] for _ in range(8)] + [filler[nf // 2:nf] + X[:3] + [(7, 7)] + X[3:] + [(3, 5)]]
    keys = list(range(nf)) + keys_x[:3] + [2 * 10 ** 6] + keys_x[3:] + [2 * 10 ** 6 + 1]
    B = Bucket(gs9, keys=keys)
    h = hyper(kind)
    hB = {k: list(v[:10]) for k, v in h.items()}
    for k in hB:
        hB[k][9] = h[k][0]
    cA, cB = [COUNTERS[2]], [COUNTERS[0]] + [1] * 8 + [COUNTERS[2]]
    ia = list(range(len(X)))
    ib = [i for i, k in enumerate(B.keys) if k in keys_x]
    assert [B.keys[i] for i in ib] == keys_x and B.seg[ib[0]][4] > 2 * grid(len(B.tiles)) - 10
    sa = Step(A, draw(A, 53), kind, {k: v[:1] for k, v in h.items()}, cA, gs=0.8, clip=False)
    sb = Step(B, draw(B, 53), kind, hB, cB, gs=0.8, clip=False)
    if kind != "novograd":       # the partials are formed only for Novograd when nothing clips: form them for both
        from edgedict_b200 import ops
        for s, Bk in ((sa, A), (sb, B)):
            ops.opt_seg_sumsq(s.out("g"), Bk.seg_t, Bk.tiles_t, view(s.partial), view(s.segsum), None)
    for da, db in zip(_x_outputs(A, sa, ia), _x_outputs(B, sb, ib)):
        for k in da:
            assert torch.equal(da[k], db[k]), (kind, k)


def test_sm3_maxima_do_not_depend_on_order():
    """Permuting the rows of a tensor permutes its row accumulators and leaves its column accumulators bit-identical;
    reversing the tile order changes no accumulator and no parameter."""
    shapes = [(1500, 33), (40, 4100), (6, 5, 700), (33 * 1024 + 100, 1)]
    B = Bucket([shapes])
    h = hyper("sm3", 1)
    D = draw(B, 59)
    s = Step(B, D, "sm3", h, [1], gs=1.0, clip=False)
    r = Step(B, D, "sm3", h, [1], gs=1.0, clip=False, tiles=B.tiles_t.flip(0).contiguous())
    assert same_bits(s.out("acc_new"), r.out("acc_new")) and same_bits(s.out("p"), r.out("p"))
    perm = torch.randperm(shapes[0][0], generator=torch.Generator().manual_seed(3)).to(DEV)
    D2 = {k: v.clone() for k, v in D.items()}
    row = B.seg[0]
    R, C = shapes[0]
    n0 = R * C
    for k in ("p", "g"):
        D2[k][:n0] = D[k][:n0].view(R, C)[perm].reshape(-1)
    D2["acc"][row[10]:row[10] + R] = D["acc"][row[10]:row[10] + R][perm]
    q = Step(B, D2, "sm3", h, [1], gs=1.0, clip=False)
    a, b = s.out("acc_new"), q.out("acc_new")
    assert same_bits(b[row[10]:row[10] + R], a[row[10]:row[10] + R][perm])
    assert same_bits(b[row[11]:row[11] + C], a[row[11]:row[11] + C])
    assert same_bits(b[row[11] + C:], a[row[11] + C:])


# ---- through the classes, at E6D2 ----------------------------------------------------------------------------------
def _class_opt(kind, params):
    from edgedict_b200 import optim
    mats, vecs = [p for p in params if p.dim() >= 2], [p for p in params if p.dim() < 2]
    if kind == "sgd":
        return optim.SGD([{"params": mats, "weight_decay": 1e-4}, {"params": vecs}], lr=0.01, momentum=0.9)
    if kind == "adamw":
        return optim.AdamW([{"params": mats, "weight_decay": 1e-2}, {"params": vecs, "lr": 3e-4}], lr=1e-3)
    if kind == "novograd":
        return optim.Novograd([{"params": mats, "weight_decay": 1e-3}, {"params": vecs}], lr=1e-3, betas=(0.95, 0.5))
    return optim.SM3([{"params": mats}, {"params": vecs, "lr": 0.05}], lr=0.1)


def _class_hyper(opt):
    h = {k: [] for k in ("lr", "wd", "b1", "b2", "eps")}
    for g in opt.param_groups:
        for k, x in zip(h, opt._hyper(g)):
            h[k].append(float(x))
    return h


def _restate_class_step(kind, opt, B, p0, sd, gflat):
    """The class's step against the restatement, teacher-forced from state_dict() before the step."""
    n = B.n
    order = [p for g in opt.param_groups for p in g["params"]]
    st = sd["state"]
    coef = float(opt._ctl[0])
    steps = opt._steps.tolist()
    h = _class_hyper(opt)

    def flat(key, default=0.0):
        x = torch.full((n,), default, dtype=f64, device=DEV)
        for i, p in enumerate(order):
            v = st.get(i, {}).get(key)
            if v is not None:
                x[B.offs[i]:B.offs[i] + p.numel()] = v.reshape(-1).double()
        return x

    L = B.L
    if kind == "sgd":
        out, has = rs.sgd(L, p0, gflat, flat("momentum_buffer", NAN), h, steps, coef, buf_new=opt.momentum_buffer)
        check("class sgd buf", opt.momentum_buffer[L.pos], *out["buf"])
    elif kind == "adamw":
        out = rs.adamw(L, p0, gflat, flat("exp_avg"), flat("exp_avg_sq"), h, steps, coef, m_new=opt.exp_avg,
                       v_new=opt.exp_avg_sq)
        check("class adamw m", opt.exp_avg[L.pos], *out["m"])
        check("class adamw v", opt.exp_avg_sq[L.pos], *out["v"])
    elif kind == "novograd":
        v0 = torch.tensor([float(st.get(i, {}).get("exp_avg_sq", 0.0)) for i in range(len(order))], dtype=f64,
                          device=DEV)
        want, b = rs.novograd_v(B.seg, opt._segsum.double(), v0, h, coef)
        check("class novograd segv", opt.exp_avg_sq, want, b)
        out = rs.novograd(L, p0, gflat, flat("exp_avg"), opt.exp_avg_sq, h, coef, m_new=opt.exp_avg)
        check("class novograd m", opt.exp_avg[L.pos], *out["m"])
    else:
        acc = torch.zeros(B.nacc, dtype=f64, device=DEV)
        for i, p in enumerate(order):
            row, s = B.seg[i], st.get(i, {})
            for d in range(max(p.dim(), 1)):
                a = s.get("accumulator_%d" % d)
                if a is not None:
                    acc[row[10 + d]:row[10 + d] + a.numel()] = a.reshape(-1).double()
        out, _ = rs.sm3(L, p0, gflat, acc, B.nacc, h, coef)
        check("class sm3 acc", opt._acc[opt._cur], *out["acc"])
    check("class %s p" % kind, opt.flat_params[L.pos], *out["p"])


@pytest.mark.parametrize("kind", KINDS)
def test_classes_at_e6d2(kind):
    """Three clipped steps of each class over the E6D2 parameters, each teacher-forced from state_dict()."""
    sh = e6d2_shapes()
    gen = torch.Generator(device=DEV).manual_seed(61)
    params = [(torch.randn(s, generator=gen, device=DEV) * 0.05).requires_grad_(True) for s in sh]
    opt = _class_opt(kind, params)
    groups = [[tuple(p.shape) for p in g["params"]] for g in opt.param_groups]
    B = Bucket(groups)
    assert torch.equal(B.seg_t, opt._seg) and torch.equal(B.tiles_t, opt._tiles)
    order = [p for g in opt.param_groups for p in g["params"]]
    for step in range(3):
        sd = opt.state_dict()
        p0 = opt.flat_params.double()
        opt.zero_grad()
        for p in order:
            p.grad.copy_(torch.randn(p.shape, generator=gen, device=DEV) * 10.0 ** (step - 1))
        opt.step(grad_scale=0.5, max_norm=1.0)
        assert float(opt._ctl[0]) < 0.5                             # the clip is active
        _restate_class_step(kind, opt, B, p0, sd, opt.flat_grads.double())
    assert opt._steps.tolist() == [3, 3]


def test_adamw_loaded_unequal_counters():
    """load_state_dict with step 3 in one group and 40 in the other: each group's bias corrections use its own."""
    sh = e6d2_shapes()
    gen = torch.Generator(device=DEV).manual_seed(67)
    params = [(torch.randn(s, generator=gen, device=DEV) * 0.05).requires_grad_(True) for s in sh]
    opt = _class_opt("adamw", params)
    order = [p for g in opt.param_groups for p in g["params"]]
    for _ in range(3):
        opt.zero_grad()
        for p in order:
            p.grad.copy_(torch.randn(p.shape, generator=gen, device=DEV))
        opt.step()
    sd = opt.state_dict()
    nmat = len(opt.param_groups[0]["params"])
    for i in range(nmat, len(order)):
        sd["state"][i]["step"] = 40
    opt.load_state_dict(sd)
    assert opt._steps.tolist() == [3, 40]
    B = Bucket([[tuple(p.shape) for p in g["params"]] for g in opt.param_groups])
    sd = opt.state_dict()
    p0 = opt.flat_params.double()
    opt.zero_grad()
    for p in order:
        p.grad.copy_(torch.randn(p.shape, generator=gen, device=DEV))
    opt.step()
    assert opt._steps.tolist() == [4, 41]
    _restate_class_step("adamw", opt, B, p0, sd, opt.flat_grads.double())
    ss = rs.adamw_step_size(_class_hyper(opt), [4, 41])
    assert abs(ss[1] / rs.adamw_step_size(_class_hyper(opt), [4, 4])[1] - 1) > 0.1     # the counters matter


@pytest.mark.parametrize("kind", KINDS)
def test_bucket_of_empty_tensors(kind):
    """Every tensor empty: no tile, so step() runs the prologue (the counters advance) and launches no update."""
    params = [torch.zeros(s, device=DEV, requires_grad=True) for s in [(0,), (0, 3), (2, 0, 4)]]
    opt = _class_opt(kind, params)
    assert opt._ntiles == 0
    opt.zero_grad()
    opt.step()
    opt.step(max_norm=1.0)
    torch.cuda.synchronize()
    assert opt._steps.tolist() == [2, 2][:len(opt.param_groups)]
    assert float(opt.grad_norm()) == 0.0
