"""FastEmit on the device: kernel-level fp64 parity and bitwise invariants of the three FastEmit entries of csrc/loss.cu
(eb_rnnt_loss_bwd_fe, eb_rnnt_loss_bwd_bf16_fe, eb_rnnt_loss_bwd_bf16_db_fe), RNNTLoss end to end against autograd of
the FastEmit surrogate, and Transducer's fastemit_lambda in both precision modes.

The C entries are called directly, into NaN-prefilled outputs.  The reference is tests/fastemit_restate.py
(grad_fastemit, pinned to autograd of the surrogate by tests/test_fastemit_host.py), teacher-forced on the kernel's own
workspace.  The bf16-logit kernels run on a workspace that eb_rnnt_loss_fwd filled from the fp32 values of the same bf16
logits.  Every bar comes from the error model of test_teacher_forced_parity, and every measured figure is printed next
to its bar (pytest -s).  eps is the unit roundoff of the compute type: 2^-24 (fp32, also for bf16 logits), 2^-53 (fp64).

The shape matrix (CASES) names the kernel variant each case reaches."""
import math

import numpy as np
import pytest
import torch

from tests import fastemit_restate as fr
from tests import loss_restate as lr
from tests.util import rel_err

pytestmark = pytest.mark.gpu

f32, f64, bf16 = torch.float32, torch.float64, torch.bfloat16
NAN = float("nan")
EPS = {f32: 2.0 ** -24, f64: 2.0 ** -53}
# the exponentials: ex2.approx.ftz (2^-22) for the main term in fp32, expf (2 ulp) for the corrections and the
# logaddexp; exp / log1p (1 ulp) in fp64
EXP_FAST = {f32: 2.0 ** -22, f64: 2.0 ** -52}
EXP_ACC = {f32: 2.0 ** -23, f64: 2.0 ** -52}
LAMBDAS = [0.01, 0.5]

# name: (B, T, U, V, blank, xlen, ylen, logits dtype, offset)   offset: logits one element past a 16-byte boundary
CASES = {
    # fp32 logits, VEC (V % 4 == 0); fp32 and bf16 out; ragged with T_b = 1 and ylen = 0
    "f32_v1024_vec": (3, 12, 9, 1024, 0, [12, 7, 1], [8, 3, 0], f32, 0),
    # fp32 scalar by V % 4 != 0
    "f32_v29_scalar": (2, 9, 8, 29, 5, [9, 7], [7, 4], f32, 0),
    # fp32 scalar by alignment
    "f32_v256_offset_scalar": (2, 10, 6, 256, 128, [10, 8], [5, 5], f32, 1),
    # the wide lattice kernel (U+1 > 896)
    "f32_u1024_wide": (3, 5, 1024, 3, 2, [5, 4, 1], [1023, 700, 0], f32, 0),
    # fp64 VEC and scalar
    "f64_v1024_vec": (3, 8, 7, 1024, 511, [8, 5, 1], [6, 6, 0], f64, 0),
    "f64_v29_scalar": (2, 9, 5, 29, 28, [9, 4], [4, 1], f64, 0),
    # bf16 logits in place: the 16-byte kernel and the one with the bias gradient (V % 8 == 0)
    "bf16_v1024_x8": (3, 12, 9, 1024, 0, [12, 7, 1], [8, 3, 0], bf16, 0),
    "bf16_v1000_x8_blank_last": (2, 11, 7, 1000, 999, [11, 6], [6, 2], bf16, 0),
    # bf16 logits, V % 8 != 0: the 4-wide and the scalar rnnt_grad_kernel on bf16 logits
    "bf16_v68_vec4": (3, 10, 6, 68, 35, [10, 10, 4], [5, 0, 5], bf16, 0),
    "bf16_v29_scalar": (2, 9, 8, 29, 5, [9, 7], [7, 4], bf16, 0),
    # bf16 with the bias gradient at the widest lattice
    "bf16_u1024_wide_db": (2, 4, 1024, 8, 0, [4, 3], [1023, 511], bf16, 0),
}


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _buffer(shape, dtype, offset, fill=NAN):
    n = int(np.prod(shape))
    buf = torch.full((n + offset,), fill, dtype=dtype, device="cuda")
    return buf[offset:].view(shape)


def _make(name):
    B, T, U, V, blank, xl, yl, dt, off = CASES[name]
    seed = sum(map(ord, name))
    rng = np.random.RandomState(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = _buffer((B, T, U, V), dt, off)
    X.copy_(torch.randn(B, T, U, V, device="cuda", generator=g, dtype=f64) * 3)
    cdt = f64 if dt == f64 else f32                             # the compute type of the kernels
    Xc = X if dt != bf16 else X.float()                          # what eb_rnnt_loss_fwd reads
    lab = lr.planted_labels(rng, B, U, V, blank)
    xlen, ylen = np.asarray(xl, np.int32), np.asarray(yl, np.int32)
    c = dict(name=name, B=B, T=T, U=U, V=V, blank=blank, dt=dt, cdt=cdt, off=off, X=X, Xc=Xc, lab=lab, xlen=xlen,
             ylen=ylen, valid=lr.valid_cells(xlen, ylen, T, U, "cuda"),
             lab_d=torch.as_tensor(lab, device="cuda") if U > 1 else None,
             xlen_d=torch.as_tensor(xlen, device="cuda"), ylen_d=torch.as_tensor(ylen, device="cuda"))
    c["costs"], c["ws"] = _fwd(c)
    return c


def _fwd(c, Xc=None, xlen=None, ylen=None):
    Xc = c["Xc"] if Xc is None else Xc
    ds = 8 if c["cdt"] == f64 else 4
    B = Xc.shape[0]
    ws = torch.full((_lib().eb_rnnt_workspace_bytes(B, c["T"], c["U"], ds) // ds,), NAN, dtype=c["cdt"], device="cuda")
    costs = torch.full((B,), NAN, dtype=c["cdt"], device="cuda")
    rc = _lib().eb_rnnt_loss_fwd(_p(Xc), _p(c["lab_d"]), _p(c["xlen_d"] if xlen is None else xlen),
                                 _p(c["ylen_d"] if ylen is None else ylen), B, c["T"], c["U"], c["V"], c["blank"], ds,
                                 _p(ws), _p(costs), 1, _stream())
    assert rc == 0, rc
    return costs, ws


def _views(c, ws, B=None):
    B = c["B"] if B is None else B
    n = B * c["T"] * c["U"]
    sh = (B, c["T"], c["U"])
    return dict(denom=ws[:n].view(sh), lpb=ws[n:2 * n].view(sh), lpl=ws[2 * n:3 * n].view(sh),
                alphas=ws[3 * n:4 * n].view(sh), betas=ws[4 * n:5 * n].view(sh), ll_fwd=ws[5 * n:5 * n + B])


def _args(c, B=None, xlen=None, ylen=None, lab=None):
    return (_p(c["lab_d"] if lab is None else lab), _p(c["xlen_d"] if xlen is None else xlen),
            _p(c["ylen_d"] if ylen is None else ylen), c["B"] if B is None else B, c["T"], c["U"], c["V"], c["blank"])


def bwd(c, kind, lam, ws=None, X=None, out=None, gscale=None, host_scale=1.0, old=False, **kw):
    """One gradient call into a NaN-prefilled output (or `out`, X = out for in place).  kind: "out" (eb_rnnt_loss_bwd_fe
    in the compute type), "out_bf16" (fp32 logits, bf16 out), "bf16" (eb_rnnt_loss_bwd_bf16_fe), "db"
    (eb_rnnt_loss_bwd_bf16_db_fe; returns (grads, db)).  old=True calls the entry without _fe (lam must be 0)."""
    L = _lib()
    ws = c["ws"] if ws is None else ws
    X = c["X"] if X is None else X
    B = X.shape[0]
    od = {"out": c["cdt"], "out_bf16": bf16, "bf16": bf16, "db": bf16}[kind]
    if out is None:
        out = _buffer(tuple(X.shape), od, c["off"])
    per_batch = int(gscale is not None and gscale.numel() > 1)
    a = _args(c, B=B, **kw)
    tail = (_p(gscale), per_batch, float(host_scale))
    if kind in ("out", "out_bf16"):
        ds = 8 if c["cdt"] == f64 else 4
        head = (_p(X), _p(out), int(kind == "out_bf16")) + a + (ds, _p(ws)) + tail
        rc = L.eb_rnnt_loss_bwd(*head, _stream()) if old else L.eb_rnnt_loss_bwd_fe(*head, lam, _stream())
    elif kind == "bf16":
        head = (_p(X), _p(out)) + a + (_p(ws),) + tail
        rc = L.eb_rnnt_loss_bwd_bf16(*head, _stream()) if old else L.eb_rnnt_loss_bwd_bf16_fe(*head, lam, _stream())
    else:
        part = torch.full((512 * c["V"],), NAN, device="cuda")
        db = torch.zeros(c["V"], device="cuda")
        head = (_p(X), _p(out)) + a + (_p(ws),) + tail + (_p(part), _p(db))
        rc = L.eb_rnnt_loss_bwd_bf16_db(*head, _stream()) if old else L.eb_rnnt_loss_bwd_bf16_db_fe(*head, lam,
                                                                                                    _stream())
    assert rc == 0, (kind, rc)
    return (out, db) if kind == "db" else out


def _kinds(c):
    if c["dt"] == f32:
        return ["out", "out_bf16"]
    if c["dt"] == f64:
        return ["out"]
    return ["bf16", "db"] if c["V"] % 8 == 0 else ["bf16"]


def _bar(c, t, x, sc, lam):
    """Per-element bar of the gradient (see test_teacher_forced_parity)."""
    cdt = c["cdt"]
    eps = EPS[cdt]
    blank, B, T, U = c["blank"], c["B"], c["T"], c["U"]
    ax = x.abs()
    d_plain = EXP_FAST[cdt] + eps * (5 * t["mag_all"][..., None] + 2 * ax)
    d_fe = EXP_FAST[cdt] + EXP_ACC[cdt] + eps * (5 * t["mag_all"] + 6 * t["mag_q"] + 4 * t["L"] + 4)[..., None] \
        + 2 * eps * ax
    bar = t["main"] * torch.where(t["fe"][..., None], d_fe, d_plain)
    bar[..., blank] += t["corr_b"] * (EXP_ACC[cdt] + eps * (5 * t["mag_b"] + 2 * ax[..., blank]))
    if U > 1:
        lab = c["lab_d"].long()[:, None, :, None].expand(B, T, U - 1, 1)
        xl = torch.gather(ax[:, :, :U - 1], 3, lab)
        e = t["corr_l"] * (EXP_ACC[cdt] + eps * (5 * t["mag_l"][:, :, :U - 1, None] + 2 * xl + 3 * math.log1p(lam)))
        bar[:, :, :U - 1].scatter_add_(3, lab, e)
    return (bar + 2 * eps * t["absum"]) * sc.abs()


def _ratio(err, bar, mask):
    r = (err / bar)[mask]
    return float(r.max()) if r.numel() else 0.0


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    c = _make(request.param)
    torch.cuda.synchronize()
    return c


def test_teacher_forced_parity(case):
    """Every FastEmit kernel variant against grad_fastemit on the kernel's own workspace (its denom, alphas, betas,
    ll_fwd and lpl), lambda in {0.01, 0.5}, scales gscale None and [B] with mixed signs times host_scale 0.25.

    Error model.  The plain terms keep the bar of test_gpu_loss_fp64.test_gradient_teacher_forced: the main term's
    relative error is EXP_FAST + eps (5 mag + 2 |x|), mag = |a| + |b| + |ll| + |d|, and each correction's is EXP_ACC +
    eps (5 mag_c + 2 |x|).  On a FastEmit cell the main exponent is d + L + x, L = logaddexp(p, q):
      p = a + b - ll rounds twice, <= 2 eps mag;  q = log lam + a + beta(t,u+1) + lpl - ll rounds four times and starts
      from log lam rounded to the compute type, <= 5 eps mag_q, mag_q = |log lam| + |a| + |beta(t,u+1)| + |lpl| + |ll|;
      lse2 passes its inputs' errors on as a weighted mean and adds its exponential's (EXP_ACC absolute on a value
      <= 1, which log1p passes on with slope <= 1), its log1p's (<= 2 eps absolute) and its last addition's (eps |L|);
      d + L and + x (or the base-2 scaling and fma of the 16-byte kernels) round by eps (|d| + |L|) and 2 eps |c + x|;
    so its relative error is <= EXP_FAST + EXP_ACC + eps (5 mag + 6 mag_q + 4 |L| + 4 + 2 |x|).  The label correction
    adds log1p(lam) rounded to the compute type and one more addition: + 3 eps log1p(lam).  Bar per element:
        |sc| (sum over the row's terms of |term| delta_term + 2 eps sum |term|) + eps |ref|
    (+ 2^-8 (|ref| + bar) for bf16 output, 2^-120 for fp32 flush-to-zero).  Dropping the lambda term from c_all or
    log1p(lam) from c_lab moves a label row's elements by about lam times the emit share, far outside it.
    Padded cells are exactly 0 and nothing is NaN; in place gives the bits of out of place."""
    c = case
    B, cdt = c["B"], c["cdt"]
    w = _views(c, c["ws"])
    x = c["X"].double()
    valid = c["valid"]
    signs = torch.tensor([(-1.5) ** (b + 1) for b in range(B)], dtype=cdt, device="cuda")
    for lam in LAMBDAS:
        ref, terms = fr.grad_fastemit(w["alphas"], w["betas"], w["denom"], w["ll_fwd"], w["lpl"], x, c["lab"],
                                      c["xlen_d"], c["ylen_d"], c["blank"], lam, terms=True)
        for kind in _kinds(c):
            for gs, hs in ((None, 1.0), (signs, 0.25)):
                g = bwd(c, kind, lam, gscale=gs, host_scale=hs)
                if kind == "db":
                    g = g[0]
                gsv = gs if gs is not None else torch.ones(1, dtype=cdt, device="cuda")
                sc = (torch.tensor(hs, dtype=cdt, device="cuda") * gsv).double().expand(B)[:, None, None, None]
                r = ref * sc
                bar = _bar(c, terms, x, sc, lam) + EPS[cdt] * r.abs() + (2.0 ** -120 if cdt == f32 else 2.0 ** -1000)
                if g.dtype == bf16:
                    bar = bar + 2.0 ** -8 * (r.abs() + bar)
                ratio = _ratio((g.double() - r).abs(), bar, valid)
                print("%s lam=%g %s scale=%s: grad err/bar %.3f" % (c["name"], lam, kind, "1" if gs is None else
                                                                     "0.25*gscale[B]", ratio))
                assert ratio <= 1, (kind, lam, ratio)
                assert bool((g[~valid] == 0).all()) and not bool(g.isnan().any()), kind
        # in place over a copy of the logits gives the bits of out of place
        for kind in _kinds(c):
            if kind == "out_bf16":
                continue
            g = bwd(c, kind, lam)
            g = g[0] if kind == "db" else g
            xi = _buffer(tuple(c["X"].shape), c["dt"], c["off"])
            xi.copy_(c["X"])
            bwd(c, kind, lam, X=xi, out=xi)
            assert torch.equal(g.view(torch.uint8), xi.view(torch.uint8)), (kind, lam)


def test_bitwise_invariants(case):
    """lambda = 0 through each _fe entry gives the bits of its sibling without _fe; the 16-byte bf16 kernel and the one
    with the bias gradient give the same d logits for every lambda, and db_accum is eb_colsum of those d logits, bit for
    bit; a second call gives the same bits."""
    c = case
    gs = torch.tensor([(-1.5) ** (b + 1) for b in range(c["B"])], dtype=c["cdt"], device="cuda")
    for kind in _kinds(c):
        a = bwd(c, kind, 0.0, gscale=gs, host_scale=0.25)
        b = bwd(c, kind, 0.0, gscale=gs, host_scale=0.25, old=True)
        if kind == "db":
            assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
            a, b = a[0], b[0]
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), kind
    for lam in [0.0] + LAMBDAS:
        for kind in _kinds(c):
            g1 = bwd(c, kind, lam, gscale=gs, host_scale=0.25)
            g2 = bwd(c, kind, lam, gscale=gs, host_scale=0.25)
            if kind == "db":
                assert torch.equal(g1[1].view(torch.int32), g2[1].view(torch.int32))
                g1, g2 = g1[0], g2[0]
            assert torch.equal(g1.view(torch.uint8), g2.view(torch.uint8)), (kind, lam)
        if "db" in _kinds(c):
            g8 = bwd(c, "bf16", lam, gscale=gs, host_scale=0.25)
            gd, db = bwd(c, "db", lam, gscale=gs, host_scale=0.25)
            assert torch.equal(g8.view(torch.int16), gd.view(torch.int16)), lam
            ref = torch.zeros(c["V"], device="cuda")
            assert _lib().eb_colsum(_p(gd), 1, _p(ref), gd.numel() // c["V"], c["V"], _stream()) == 0
            torch.cuda.synchronize()
            assert torch.equal(db.view(torch.int32), ref.view(torch.int32)), lam
    if c["cdt"] == f64:
        _row_sums(c)


def _row_sums(c):
    """fp64: every valid row of d logits sums to zero within the sum of its elements' bars plus what the workspace's own
    rounding leaves of the identity beta = logaddexp(stay, emit) and of sum_v exp(x_v + d) = 1: each term off by a
    factor within exp(+-delta_ws), delta_ws = 2 (T_b + U_b) eps (3 M + 6) + 8 V eps, M the largest |alpha|, |beta|."""
    w = _views(c, c["ws"])
    x = c["X"].double()
    eps = EPS[f64]
    M = float(torch.maximum(w["alphas"][c["valid"]].abs().max(), w["betas"][c["valid"]].abs().max()))
    delta_ws = 2 * (c["T"] + c["U"]) * eps * (3 * M + 6) + 8 * c["V"] * eps
    for lam in LAMBDAS:
        _, terms = fr.grad_fastemit(w["alphas"], w["betas"], w["denom"], w["ll_fwd"], w["lpl"], x, c["lab"],
                                    c["xlen_d"], c["ylen_d"], c["blank"], lam, terms=True)
        one = torch.ones(c["B"], 1, 1, 1, dtype=f64, device="cuda")
        bar = (_bar(c, terms, x, one, lam) + terms["absum"] * math.expm1(delta_ws)).sum(-1)
        g = bwd(c, "out", lam)
        r = _ratio(g.sum(-1).abs(), bar, c["valid"])
        print("%s lam=%g: fp64 row sums err/bar %.3f" % (c["name"], lam, r))
        assert r <= 1, r


@pytest.mark.parametrize("name", ["f32_v1024_vec", "f64_v29_scalar", "bf16_v1024_x8", "bf16_v68_vec4"])
def test_utterance_bits_independent_of_batch_and_padding(name):
    """An utterance alone and as utterance 1 of 3 in a batch with more frames: the same bits of its d logits rows at
    lambda = 0.5 through every kind of its case, and zero on the rows the longer batch adds."""
    c = _make(name)
    T, U, V = c["T"], c["U"], c["V"]
    T2 = T + 3
    g = torch.Generator(device="cuda").manual_seed(7)
    X2 = (torch.randn(3, T2, U, V, device="cuda", generator=g, dtype=f64) * 3).to(c["dt"])
    X2[1, :T] = c["X"][0]
    lab2 = np.concatenate([c["lab"][1:2], c["lab"][0:1], c["lab"][1:2]]) if U > 1 else c["lab"]
    xl2 = torch.tensor([T2, int(c["xlen"][0]), T2 - 1], dtype=torch.int32, device="cuda")
    yl2 = torch.tensor([U - 1, int(c["ylen"][0]), U - 2], dtype=torch.int32, device="cuda")
    lab2_d = torch.as_tensor(np.ascontiguousarray(lab2), device="cuda") if U > 1 else None
    c2 = dict(c, B=3, T=T2, X=X2, Xc=X2 if c["dt"] != bf16 else X2.float(), lab_d=lab2_d, xlen_d=xl2, ylen_d=yl2,
              off=0)
    _, ws2 = _fwd(c2)
    one = dict(c, B=1, X=c["X"][0:1].contiguous(), off=0, xlen_d=c["xlen_d"][:1], ylen_d=c["ylen_d"][:1],
               lab_d=c["lab_d"][:1] if U > 1 else None)
    one["Xc"] = one["X"] if c["dt"] != bf16 else one["X"].float()
    _, ws1 = _fwd(one)
    for kind in _kinds(c):
        g1 = bwd(one, kind, 0.5, ws=ws1)
        gb = bwd(c2, kind, 0.5, ws=ws2)
        if kind == "db":
            g1, gb = g1[0], gb[0]
        assert torch.equal(gb[1, :T].contiguous().view(torch.uint8), g1[0].contiguous().view(torch.uint8)), kind
        assert bool((gb[1, T:] == 0).all()), kind


@pytest.mark.parametrize("lam", [0.01, 0.5])
@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
def test_rnnt_loss_end_to_end_fp64(reduction, lam):
    """RNNTLoss(fastemit_lambda=lam, reduction) on fp64 logits against autograd of the surrogate S_b in fp64 on the
    CPU, with per-utterance upstream gradients of mixed signs ('none') or a scalar one ('sum', 'mean' = sum / B).  Bar:
    each term of the gradient off by a factor within exp(+-delta), delta = 4 (T + U) eps (3 M + 6) + 16 V eps (the fp64
    chain's lattice and statistics); the costs are bitwise those of lam = 0."""
    from edgedict_b200.warprnnt_pytorch import RNNTLoss
    B, T, U, V, blank = 4, 7, 5, 9, 3
    rng = np.random.RandomState(11)
    x = torch.as_tensor(rng.randn(B, T, U, V) * 2.5, dtype=f64)
    lab = lr.planted_labels(rng, B, U, V, blank)
    xlen, ylen = np.asarray([7, 5, 1, 6], np.int32), np.asarray([4, 2, 3, 0], np.int32)
    up = torch.tensor([0.7, -1.3, 2.0, 0.4], dtype=f64)

    def run(lam_):
        a = x.cuda().requires_grad_(True)
        out = RNNTLoss(blank=blank, reduction=reduction, fastemit_lambda=lam_)(
            a, torch.as_tensor(lab, device="cuda"), torch.as_tensor(xlen, device="cuda"),
            torch.as_tensor(ylen, device="cuda"))
        (out * (up.cuda() if reduction == "none" else up[0].cuda())).sum().backward()
        return out.detach(), a.grad
    out0, _ = run(0.0)
    out, g = run(lam)
    assert torch.equal(out.view(torch.int64), out0.view(torch.int64))
    wts = up if reduction == "none" else torch.full((B,), float(up[0]) / (B if reduction == "mean" else 1), dtype=f64)
    g_o, costs = fr.surrogate_grad(x, lab, xlen, ylen, blank, lam, weights=wts)
    # the exact fp64 lattice, for M and the |terms| of the restatement
    d = -torch.logsumexp(x, -1)
    lpl = torch.zeros_like(d)
    idx = torch.as_tensor(lab).long()[:, None, :, None].expand(B, T, U - 1, 1)
    lpl[:, :, :U - 1] = torch.gather(x[:, :, :U - 1], 3, idx)[..., 0] + d[:, :, :U - 1]
    al, be, llf, _ = lr.lattice(x[..., blank] + d, lpl, xlen, ylen)
    M = float(torch.maximum(al.nan_to_num(0).abs().max(), be.nan_to_num(0).abs().max()))
    delta = 4 * (T + U) * EPS[f64] * (3 * M + 6) + 16 * V * EPS[f64]
    _, terms = fr.grad_fastemit(al, be, d, llf, lpl, x, lab, xlen, ylen, blank, lam, terms=True)
    bar = terms["absum"] * math.expm1(delta) * wts.abs()[:, None, None, None] + 1e-300
    r = float(((g.cpu() - g_o).abs() / bar).max())
    rc = float(((out.cpu().view(-1) - (costs if reduction == "none" else
                                        (costs.sum() / (B if reduction == "mean" else 1)).view(1))).abs()).max())
    print("RNNTLoss %s lam=%g: grad err/bar %.3f (delta %.1e), costs max |err| %.1e" % (reduction, lam, r, delta, rc))
    assert r <= 1, r
    assert rc <= 1e-12 * float(costs.abs().sum())


TINY = dict(vocab_embed_size=16, vocab_size=64, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0,
            enc_proj_size=40, dec_hidden_size=32, dec_layers=2, dec_dropout=0, dec_proj_size=24, joint_size=56)


def _model(V):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(5)
    m = Transducer(**dict(TINY, vocab_size=V)).cuda()
    g = torch.Generator().manual_seed(V)
    xs = torch.randn(4, 20, 24, generator=g).cuda()
    ys = torch.randint(4, V, (4, 7), dtype=torch.int32, generator=g).cuda()
    xlen, ylen = torch.tensor([20, 20, 15, 9], dtype=torch.int32), torch.tensor([7, 5, 7, 2], dtype=torch.int32)
    return m, (xs, ys, xlen, ylen)


def _step(m, inputs):
    m.zero_grad()
    loss = m(*inputs)
    costs = m.last_costs.clone()
    loss.backward()
    return loss.detach(), costs, {k: p.grad.clone() for k, p in m.named_parameters()}


@pytest.mark.parametrize("precision, V", [("fp32", 64), ("bf16", 64), ("fp32", 68)])
def test_transducer_fastemit(precision, V):
    """Transducer(fastemit_lambda) in fp32 and bf16 mode; in bf16 mode V = 64 reaches the gradient kernel with the bias
    gradient, and V = 68 (V % 8 != 0) runs the fp32 mode's 4-wide gradient kernel.  A bf16-mode Transducer with
    V % 8 != 0 does not train at any lambda (the output layer's bf16 weight-gradient GEMM needs rows of 16 bytes), so
    JointLoss's bf16 branch without the bias gradient is checked through its kernels above (bf16_v68_vec4,
    bf16_v29_scalar).  The loss and last_costs are bitwise those of lambda = 0; the parameter gradients
    match the same model's joint logits fed to RNNTLoss(fastemit_lambda) within test_gpu_model.py's tolerances (fp32
    1e-3, bf16 6e-2 as its fused-against-unfused check); lambda > 0 moves them; and setting model.fastemit_lambda between
    steps takes effect at the next forward."""
    from edgedict_b200.warprnnt_pytorch import RNNTLoss
    lam = 0.5
    m, inputs = _model(V)
    m.set_precision(precision)
    xs, ys, xlen, ylen = inputs
    l0, c0, g0 = _step(m, inputs)
    m.fastemit_lambda = lam                                      # a ramp: the next forward uses it
    l1, c1, g1 = _step(m, inputs)
    assert torch.equal(l1.view(torch.int32), l0.view(torch.int32)) and torch.equal(c1.view(torch.int32),
                                                                                  c0.view(torch.int32))
    moved = max(rel_err(g1[k].cpu(), g0[k].cpu()) for k in g0)
    # the same weights, the loss outside the model
    m.output_loss = False
    m.zero_grad()
    logits = m(xs, ys, xlen, ylen).float()
    xl = m.scale_length(logits, xlen)
    loss = RNNTLoss(blank=0, fastemit_lambda=lam)(logits, ys[:, :int(ylen.max())].contiguous(), xl.cuda(),
                                                  ylen.cuda())
    loss.backward()
    tol = 1e-3 if precision == "fp32" else 6e-2
    errs = {k: rel_err(g1[k].cpu(), p.grad.cpu()) for k, p in m.named_parameters()}
    m.output_loss = True
    print("Transducer %s V=%d lam=%g: gradients vs joint + RNNTLoss max rel %.2e (bar %.0e), moved by lambda %.2e; "
          "loss rel to unfused %.2e" % (precision, V, lam, max(errs.values()), tol, moved,
                                         abs(float(loss) - float(l1)) / float(l1)))
    assert max(errs.values()) < tol, errs
    assert moved > 1e-3, moved
    # a model built with the lambda gives what the ramped one gave
    from edgedict_b200.rnnt.models import Transducer
    m2 = Transducer(fastemit_lambda=lam, **dict(TINY, vocab_size=V)).cuda()
    m2.load_state_dict(m.state_dict())
    m2.set_precision(precision)
    l2, c2, g2 = _step(m2, inputs)
    assert torch.equal(c2.view(torch.int32), c1.view(torch.int32))
    r2 = max(rel_err(g2[k].cpu(), g1[k].cpu()) for k in g1)
    print("  built with lambda vs ramped: max rel %.2e" % r2)
    assert r2 <= 1e-6, r2
