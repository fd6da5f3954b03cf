"""Per-element fp64 parity and bitwise invariants of the glue kernels: csrc/elementwise.cu (LayerNorm, time reduction,
embedding, the joint's broadcast tanh and its reductions, column sums, casts, the transpose, Adam / AdamW, the sum of
squares) and csrc/frontend.cu (the log-mel front end and the SpecAugment masks), each through its C entry point.

Error model.  The build uses no fast-math: division and sqrtf are IEEE, but nvcc contracts a*b + c into one FMA.  So a
result is checked BITWISE wherever the kernel only gathers, copies, adds in an order its code fixes, scales by 0.5 or
rounds to nearest (the reference restates that order in torch / numpy fp32), and against fp64 under a PER-ELEMENT BAR
wherever a multiply feeds an add or a transcendental is involved, because FMA contraction is not visible from Python.
u = 2^-24 is the fp32 unit roundoff; a chain of n fp32 additions is off by at most n u (sum of |terms|).

  eb_layernorm_fwd   z = fp32(x + res) is restated exactly (torch fp32); mean: each lane adds <= PL values, then 5
                     butterfly levels and a division by H: |mean - mu| <= (PL + 5) u sum|z| / H + u |mu|.  rstd: the
                     two-pass variance from the kernel's own mean (sum (z - mean)^2 = S2 + H dmu^2 exactly), n_add u per
                     square and add, the division and + eps (2 u), rsqrtf 2 ulp (2^-22 relative), halved through the
                     square root.  y teacher-forced from the kernel's mean / rstd: (z - mean) rstd gamma + beta, four
                     roundings of the product and two of the sum; end to end against fp64 LayerNorm with the mean and
                     rstd bars propagated.  y_bf16 = bf16_rn(y), NULL mean / rstd, repeated launches: bitwise.
  eb_layernorm_bwd   dz teacher-forced from the kernel's mean / rstd, both dz kernels (vectorised: H % 128 == 0, H <=
                     1024, 16-byte aligned; generic otherwise): xhat 2 u, g = dy gamma u, the two row sums with
                     ceil(H/32) + 8 roundings (both kernels' chains) plus the division, five roundings of the final
                     expression.  dbeta bitwise (thread (c, k) adds rows k, k + 128, ..., then a 64 ... 1 tree); dgamma
                     barred (its products contract into the chain) and the same bits whichever dz kernel ran.
  eb_time_reduce_*   bitwise: (x[2t] + x[2t+1]) * 0.5 with a zero pad, and 0.5 dy (torch autograd of the same).
  eb_embedding_*     forward a bitwise gather; backward bitwise: each id's positions added in position order from 0,
                     then += into dW (no gradient for the pad id).
  eb_joint_hidden_*  fp32 tanhf of fp32(e + d): 2 ulp (2^-22 relative).  bf16 tanh.approx.f32: its relative error 2^-11
                     (PTX ISA) is below an eighth of a bf16 ulp, so |h16 - tanh z| <= half a bf16 ulp + 2^-11 |tanh z|
                     (asserted with 2^-10.98), i.e. h16 is within one bf16 ulp of bf16_rn(tanh z).  Backward fp32: dpre = dh (1 - h h), three roundings; dep / ddp the sequential
                     sums of the kernel's dpre, bitwise.  Backward bf16: h^2 is exact for bf16 h, so the stored dpre16 is
                     bitwise bf16_rn(fp32(dh fp32(1 - h^2))) and ddp the sequential sum over t of float(dpre16); dep sums
                     the UNROUNDED products over u and the product may contract into that add: barred, (U + 2) u.
  eb_joint_dpre_reduce  bitwise sequential fp32 sums of float(dpre16), u in order and t in order.
  eb_colsum          bitwise: lane k of 32 adds rows k, k + 32, ..., then a 16 ... 1 tree, += into out (fp32 and the
                     generic bf16 path; the vectorised bf16 path is pinned by test_gpu_colsum_order.py).
  eb_cast_bf16, eb_transpose_to_bf16   bitwise against torch's round-to-nearest-even .bfloat16().
  eb_adam_step(_ex)  teacher-forced one step in fp64 with the hyper-parameters as the kernel receives them (fp32 lr, betas,
                     eps, wd; the host's fp32 bc = 1 - powf(beta, step)); m, v and the update d = p_new - p_old barred
                     from the roundings of each expression (bar relative to |d|, not |p|: p is drawn at the scale of
                     the update); a non-finite sum of squares leaves p, m, v bitwise untouched.
  eb_sumsq           atomics across blocks: barred, (strided chain + block tree + one add per block) u sum x^2.
  eb_fe_*            preemph_pad without pre-emphasis and log_stack without the log bitwise; v - p x[r-1] two roundings;
                     re^2 + im^2 two roundings; logf 1 ulp (barred at 2); the masks bitwise.

Every output goes into a NaN-prefilled buffer with guard elements (or rows) behind it, and inputs that must not be read
(the unused frame slots of the front end) are NaN.  Each bar-based check prints its worst err/bar (pytest -s); DESIGN.md
section 2 records the measured figures."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
U24 = 2.0 ** -24
TINY = 2.0 ** -126
G = 40                       # guard elements behind every flat output


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ok(st, name):
    assert st == 0, "%s: status %d" % (name, st)
    torch.cuda.synchronize()


# ---- error bookkeeping ------------------------------------------------------------------------------------------------
def _report(name, got, ref, bar):
    """Prints the worst err/bar of one output against its fp64 value, then asserts it."""
    got, ref, bar = got.double().cpu(), ref.double().cpu(), bar.double().cpu() + TINY
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), name + ": non-finite output"
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bar)
    k = int(torch.argmax(r.reshape(-1)))
    idx = tuple(int(i) for i in np.unravel_index(k, tuple(r.shape)))
    ratio = float(r.reshape(-1)[k])
    print("  %-52s worst err/bar %.3g at %s (err %.3g, bar %.3g)" % (name, ratio, idx, float(err[idx]), float(bar[idx])))
    assert ratio <= 1.0, "%s: err/bar %.3g at %s, kernel %r, fp64 %r" % (name, ratio, idx, float(got[idx]),
                                                                        float(ref[idx]))


def _bits(x):
    return x.view(torch.int32) if x.dtype == f32 else x.view(torch.int16)


def _same(name, got, want):
    """Bit-for-bit equality, naming the first differing element."""
    got, want = got.cpu(), want.cpu()
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    d = _bits(got) != _bits(want)
    if bool(d.any()):
        idx = tuple(int(i) for i in torch.nonzero(d)[0])
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r, want %r"
                             % (name, int(d.sum()), d.numel(), idx, float(got[idx]), float(want[idx])))


def _nan(n, dtype=f32):
    """Flat NaN buffer of n outputs plus G guard elements."""
    return torch.full((n + G,), float("nan"), dtype=dtype, device=DEV)


def _guard(name, buf, n):
    assert bool(torch.isnan(buf[n:].float()).all()), name + ": a store went past the end of the output"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---- LayerNorm forward ------------------------------------------------------------------------------------------------
def _pl(H):
    return 8 if H <= 256 else 16 if H <= 512 else 32 if H <= 1024 else 64


def _ln_fwd(x, res, gamma, beta, rows, H, eps, y16=False, stats=True, guard_rows=1):
    """eb_layernorm_fwd into [guard_rows + rows + guard_rows, H] NaN buffers (a slice in the middle, as the chunk-major
    `out=` slices of the encoder), mean / rstd likewise; returns (y, y16, mean, rstd) and checks every guard."""
    L = _lib()
    yb = torch.full(((rows + 2 * guard_rows) * H,), float("nan"), device=DEV)
    y = yb[guard_rows * H:(guard_rows + rows) * H]
    y16b = torch.full(((rows + 2 * guard_rows) * H,), float("nan"), dtype=bf16, device=DEV) if y16 else None
    y16v = y16b[guard_rows * H:(guard_rows + rows) * H] if y16 else None
    mb = torch.full((rows + 2 * guard_rows,), float("nan"), device=DEV)
    rb = torch.full((rows + 2 * guard_rows,), float("nan"), device=DEV)
    mean, rstd = mb[guard_rows:guard_rows + rows], rb[guard_rows:guard_rows + rows]
    st = L.eb_layernorm_fwd(_p(x), _p(res), _p(gamma), _p(beta), _p(y), _p(y16v), _p(mean) if stats else None,
                            _p(rstd) if stats else None, rows, H, eps, _stream())
    _ok(st, "eb_layernorm_fwd")
    for b, n in ((yb, H), (mb, 1), (rb, 1)) + (((y16b, H),) if y16 else ()):
        g = guard_rows * n
        assert bool(torch.isnan(b[:g].float()).all() and torch.isnan(b[b.numel() - g:].float()).all()), \
            "layernorm_fwd wrote a neighbouring row"
    if not stats:
        assert bool(torch.isnan(mb).all() and torch.isnan(rb).all())
    return y.view(rows, H), (y16v.view(rows, H) if y16 else None), mean, rstd


# (name, rows, H, residual, offset, scale): x = offset + scale N(0, 1).  The register tier PL = 8 / 16 / 32 / 64 follows
# from H; rows > 8 x 8 x #SMs (the grid cap) runs the grid-stride loop; a large common offset defeats a one-pass
# variance; a small scale makes eps a visible part of the variance
LN_FWD_CASES = [
    ("PL8-H1", 5, 1, False, 0.0, 1.0),
    ("PL8-H31-res", 37, 31, True, 0.0, 1.0),
    ("PL8-H200-small", 64, 200, False, 0.0, 0.01),
    ("PL8-H256-gridstride-res", 9000, 256, True, 0.0, 1.0),
    ("PL16-H257", 40, 257, False, 0.0, 1.0),
    ("PL16-H512-offset", 33, 512, True, 1e3, 1.0),
    ("PL32-H513-res", 20, 513, True, 0.0, 1.0),
    ("PL32-H1000-offset", 50, 1000, False, 1e3, 1.0),
    ("PL32-H1024-gridstride", 8600, 1024, False, 0.0, 1.0),
    ("PL64-H1025-res", 17, 1025, True, 0.0, 1.0),
    ("PL64-H2047-offset-res", 9, 2047, True, 1e3, 1.0),
    ("PL64-H2048-gridstride-res", 8500, 2048, True, 0.0, 1.0),
]


def _ln_inputs(rows, H, with_res, offset, seed, scale=1.0):
    g = _gen(seed)
    x = torch.randn(rows, H, device=DEV, generator=g) * scale + offset
    res = torch.randn(rows, H, device=DEV, generator=g) * 0.5 if with_res else None
    gamma = 1.0 + 0.5 * torch.randn(H, device=DEV, generator=g)
    beta = 0.3 * torch.randn(H, device=DEV, generator=g)
    return x, res, gamma, beta


def _ln_ref(z, mean_k, rstd_k, gamma, beta, eps, H):
    """fp64 LayerNorm of z and the bars of the kernel's mean, rstd and y (module docstring), on the device of z."""
    zd = z.double()
    mk, rk = mean_k.double(), rstd_k.double()
    gd, bd = gamma.double(), beta.double()
    n_add = _pl(H) + 5
    mu = zd.mean(1)
    bar_mu = n_add * U24 * zd.abs().sum(1) / H + U24 * mu.abs()
    dmu = mk - mu
    S2 = ((zd - mu[:, None]) ** 2).sum(1)
    var = S2 / H
    rs = 1.0 / torch.sqrt(var + eps)
    # the kernel's two-pass variance is of sum (z - mean_k)^2 = S2 + H dmu^2 (exactly): n_add roundings of it, its
    # distance H dmu^2 from S2, the division and + eps
    e_var = (n_add * U24 * (S2 + H * dmu ** 2) + H * dmu ** 2) / H + 2 * U24 * (var + eps)
    bar_rs = rs * (0.5 * e_var / (var + eps) + 2.0 ** -22)
    tf = (zd - mk[:, None]) * rk[:, None] * gd + bd
    t = (zd - mk[:, None]).abs() * rk[:, None] * gd.abs()
    bar_tf = 4 * U24 * t + 2 * U24 * tf.abs()
    y = (zd - mu[:, None]) * rs[:, None] * gd + bd
    bar_y = bar_tf + gd.abs() * (rk[:, None] * bar_mu[:, None] + (zd - mu[:, None]).abs() * bar_rs[:, None])
    return mu, bar_mu, rs, bar_rs, tf, bar_tf, y, bar_y


@pytest.mark.parametrize("name,rows,H,with_res,offset,scale", LN_FWD_CASES, ids=[c[0] for c in LN_FWD_CASES])
def test_layernorm_fwd(name, rows, H, with_res, offset, scale):
    eps = 1e-5
    x, res, gamma, beta = _ln_inputs(rows, H, with_res, offset, seed=rows + H, scale=scale)
    z = x + res if with_res else x                       # torch fp32: exactly the kernel's add
    y, y16, mean, rstd = _ln_fwd(x, res, gamma, beta, rows, H, eps, y16=True)
    mu, bar_mu, rs, bar_rs, tf, bar_tf, yr, bar_y = _ln_ref(z, mean, rstd, gamma, beta, eps, H)
    _report(name + " mean", mean, mu, bar_mu)
    _report(name + " rstd", rstd, rs, bar_rs)
    _report(name + " y (teacher-forced)", y, tf, bar_tf)
    _report(name + " y (fp64 LayerNorm)", y, yr, bar_y)
    _same(name + " y_bf16", y16, y.bfloat16())
    y2, _, _, _ = _ln_fwd(x, res, gamma, beta, rows, H, eps, stats=False)
    _same(name + " y with NULL mean / rstd", y2, y)
    y3, _, m3, r3 = _ln_fwd(x, res, gamma, beta, rows, H, eps)
    _same(name + " repeated launch", y3, y)
    _same(name + " repeated launch mean", m3, mean)
    _same(name + " repeated launch rstd", r3, rstd)


def test_layernorm_rejects_h_over_2048():
    x = torch.zeros(4, 2049, device=DEV)
    g = torch.ones(2049, device=DEV)
    assert _lib().eb_layernorm_fwd(_p(x), None, _p(g), _p(g), _p(x), None, None, None, 4, 2049, 1e-5, _stream()) == 2
    assert _lib().eb_layernorm_bwd(_p(x), _p(x), None, _p(g), _p(g), _p(g), _p(x), _p(g), _p(g), 4, 2049,
                                   _stream()) == 2


# ---- LayerNorm backward -----------------------------------------------------------------------------------------------
def _ln_bwd_vec(H, ptrs):
    """eb_layernorm_bwd's choice of the vectorised dz kernel."""
    return H % 128 == 0 and H <= 1024 and all(p % 16 == 0 for p in ptrs if p)


def _offset_copy(t, off):
    """A copy of t whose storage starts `off` floats into a fresh allocation."""
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=DEV)
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _dbeta_order(dy, H):
    """layernorm_param_grad_kernel's dbeta in its order, numpy fp32: lane k adds rows k, k + 128, ... from 0, then the
    tree at strides 64 ... 1."""
    d = dy.cpu().numpy().astype(np.float32)
    rows = d.shape[0]
    nb = -(-rows // 128)
    pad = np.zeros((nb * 128, H), np.float32)
    pad[:rows] = d
    acc = np.zeros((128, H), np.float32)
    for i in range(nb):
        acc = acc + pad[i * 128:(i + 1) * 128]
    st = 64
    while st:
        acc[:st] = acc[:st] + acc[st:2 * st]
        st >>= 1
    return acc[0]


def ln_bwd_ref(z, mean_k, rstd_k, dy, gamma, dg0=None):
    """Teacher-forced fp64 LayerNorm backward from the kernel's mean / rstd, on the device of the inputs (module
    docstring): (dz, its bar, the magnitude sum |g| + |s1| + |xhat s2| of each dz, dgamma = dg0 + sum dy xhat, its bar)."""
    zd, mk, rk, dyd, gd = (t.double() for t in (z, mean_k, rstd_k, dy, gamma))
    rows, H = zd.shape
    xh = (zd - mk[:, None]) * rk[:, None]
    gg = dyd * gd
    s1 = gg.mean(1, keepdim=True)
    s2 = (gg * xh).mean(1, keepdim=True)
    dz = rk[:, None] * (gg - s1 - xh * s2)
    n_add = -(-H // 32) + 8
    e1 = (n_add + 3) * U24 * gg.abs().mean(1, keepdim=True)
    e2 = (n_add + 6) * U24 * (gg * xh).abs().mean(1, keepdim=True)
    mag = gg.abs() + s1.abs() + (xh * s2).abs()
    bar = rk[:, None] * (5 * U24 * mag + e1 + xh.abs() * e2) + U24 * dz.abs()
    dg0 = torch.zeros(H, dtype=torch.float64, device=zd.device) if dg0 is None else dg0.double()
    dgam = dg0 + (dyd * xh).sum(0)
    bar_dgam = (3 + -(-rows // 128) + 8) * U24 * (dyd * xh).abs().sum(0) + U24 * (dg0.abs() + dgam.abs())
    return dz, bar, mag, dgam, bar_dgam


# (name, rows, H, residual): H % 128 == 0 and H <= 1024 reach both dz kernels (aligned vs a view offset by one float);
# rows < 128 and rows % 128 != 0 (the param-grad row lanes), H % 8 != 0 (the last CTA's partial column group),
# rows > 4 x 3 x #SMs (the vectorised kernel's grid-stride loop)
LN_BWD_CASES = [
    ("H128-rows37-res", 37, 128, True),
    ("H256-rows300", 300, 256, False),
    ("H384-rows2000-res", 2000, 384, True),
    ("H512-rows5", 5, 512, False),
    ("H1024-rows129-res", 129, 1024, True),
    ("H100-rows77", 77, 100, True),
    ("H1-rows3", 3, 1, False),
    ("H1500-rows50-res", 50, 1500, True),
    ("H2048-rows20", 20, 2048, False),
    ("H2047-rows130", 130, 2047, True),
]


@pytest.mark.parametrize("name,rows,H,with_res", LN_BWD_CASES, ids=[c[0] for c in LN_BWD_CASES])
def test_layernorm_bwd(name, rows, H, with_res):
    eps = 1e-5
    x, res, gamma, beta = _ln_inputs(rows, H, with_res, 0.0, seed=7 * rows + H)
    g = _gen(rows * H + 1)
    dy = torch.randn(rows, H, device=DEV, generator=g)
    _, _, mean, rstd = _ln_fwd(x, res, gamma, beta, rows, H, eps)     # the kernel's own statistics
    dg0 = torch.randn(H, device=DEV, generator=g)
    db0 = torch.randn(H, device=DEV, generator=g)
    z = (x + res if with_res else x).double().cpu()
    rk = rstd.double().cpu()
    # teacher-forced fp64 dz and its bar; dgamma teacher-forced, barred
    dz_tf, bar_tf, mag, dgam_tf, bar_dgam = ln_bwd_ref(z, mean.cpu(), rstd.cpu(), dy.cpu(), gamma.cpu(), dg0.cpu())
    # end to end: fp64 torch.layer_norm autograd
    zr = z.clone().requires_grad_(True)
    torch.nn.functional.layer_norm(zr, (H,), gamma.double().cpu(), None, eps).backward(dy.double().cpu())
    dz_e2e = zr.grad
    bar_e2e = 4 * bar_tf + 64 * U24 * rk[:, None] * mag
    # dbeta bitwise in the kernel's order
    dbeta_want = torch.from_numpy(db0.cpu().numpy() + _dbeta_order(dy, H))

    L = _lib()
    variants = [("aligned", 0)] + ([("x offset by one float", 1)] if H % 128 == 0 and H <= 1024 else [])
    results = {}
    for label, off in variants:
        xv = _offset_copy(x, off) if off else x
        dzb = _nan(rows * H)
        dgb, dbb = _nan(H), _nan(H)
        dgb[:H], dbb[:H] = dg0, db0
        vec = _ln_bwd_vec(H, [dy.data_ptr(), xv.data_ptr(), dzb.data_ptr(), gamma.data_ptr(),
                              res.data_ptr() if with_res else 0])
        assert vec == (H % 128 == 0 and H <= 1024 and off == 0), (name, label)
        kern = "vectorised" if vec else "generic"
        st = L.eb_layernorm_bwd(_p(dy), _p(xv), _p(res), _p(gamma), _p(mean), _p(rstd), _p(dzb), _p(dgb), _p(dbb),
                                rows, H, _stream())
        _ok(st, "eb_layernorm_bwd")
        for b, n in ((dzb, rows * H), (dgb, H), (dbb, H)):
            _guard(name, b, n)
        dz = dzb[:rows * H].view(rows, H)
        _report("%s dz %s (teacher-forced)" % (name, kern), dz, dz_tf, bar_tf)
        _report("%s dz %s (fp64 autograd)" % (name, kern), dz, dz_e2e, bar_e2e)
        _report("%s dgamma (%s)" % (name, kern), dgb[:H], dgam_tf, bar_dgam)
        _same("%s dbeta (%s) vs its summation order" % (name, kern), dbb[:H], dbeta_want)
        results[kern] = dgb[:H].clone()
    if len(results) == 2:
        _same(name + " dgamma: vectorised vs generic dz kernel", results["vectorised"], results["generic"])


@pytest.mark.parametrize("H,off", [(1024, 0), (1024, 1), (1000, 0)], ids=["H1024-vectorised", "H1024-offset-generic",
                                                                          "H1000-generic"])
@pytest.mark.parametrize("with_res", [False, True])
def test_layernorm_bwd_split_entry_points(H, off, with_res):
    """The two halves of eb_layernorm_bwd that the chunked encoder backward calls separately: eb_layernorm_bwd_dz on row
    sub-ranges (one row, a ragged block, the wavefront's group sizes) gives bitwise the matching rows of eb_layernorm_bwd's
    dz, on the vectorised kernel (H = 1024, aligned) and the generic one (x offset by one float, or H % 128 != 0); and
    eb_layernorm_bwd_params over all rows gives bitwise its dgamma / dbeta."""
    rows, eps = 2300, 1e-5
    x, res, gamma, beta = _ln_inputs(rows, H, with_res, 0.0, seed=H + off + 3 * with_res)
    dy = torch.randn(rows, H, device=DEV, generator=_gen(rows + H))
    _, _, mean, rstd = _ln_fwd(x, res, gamma, beta, rows, H, eps)
    xv = _offset_copy(x, off) if off else x
    L = _lib()
    dz = _nan(rows * H)
    dg, db = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    _ok(L.eb_layernorm_bwd(_p(dy), _p(xv), _p(res), _p(gamma), _p(mean), _p(rstd), _p(dz), _p(dg), _p(db), rows, H,
                           _stream()), "eb_layernorm_bwd")
    dz = dz[:rows * H].view(rows, H)
    vec = _ln_bwd_vec(H, [dy.data_ptr(), xv.data_ptr(), dz.data_ptr(), gamma.data_ptr(), res.data_ptr() if with_res else 0])
    assert vec == (H == 1024 and off == 0)
    name = "layernorm_bwd H%d %s%s" % (H, "vectorised" if vec else "generic", " res" if with_res else "")
    blocks = [(0, 1), (1, 127), (128, 32 * 5 + 3), (291, 5 * 96), (771, 1529)]      # a partition of the rows
    assert blocks[-1][0] + blocks[-1][1] == rows
    for a, n in blocks:
        out = _nan(n * H)
        r = res[a:a + n] if with_res else None
        _ok(L.eb_layernorm_bwd_dz(_p(dy[a:a + n]), _p(xv[a:a + n]), _p(r), _p(gamma), _p(mean[a:a + n]),
                                  _p(rstd[a:a + n]), _p(out), n, H, _stream()), "eb_layernorm_bwd_dz")
        _guard(name, out, n * H)
        _same("%s dz rows [%d, %d)" % (name, a, a + n), out[:n * H].view(n, H), dz[a:a + n])
    dg2, db2 = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    _ok(L.eb_layernorm_bwd_params(_p(dy), _p(xv), _p(res), _p(mean), _p(rstd), _p(dg2), _p(db2), rows, H, _stream()),
        "eb_layernorm_bwd_params")
    _same(name + " dgamma of the parameter pass", dg2, dg)
    _same(name + " dbeta of the parameter pass", db2, db)


# ---- time reduction ---------------------------------------------------------------------------------------------------
def _tr_ref(x):
    B, T, H = x.shape
    xp = torch.cat([x, torch.zeros(B, 1, H)], 1) if T % 2 else x
    return (xp[:, 0::2] + xp[:, 1::2]) * 0.5


@pytest.mark.parametrize("B,T,H", [(3, 1, 5), (2, 7, 33), (4, 10, 64), (1, 2, 1), (3, 1001, 1024)])
def test_time_reduce(B, T, H):
    """(3, 1001, 1024): 1.5 M outputs, 3 M gradient elements, past ew_grid's cap of 32 x #SMs blocks of 256."""
    L = _lib()
    g = _gen(B * T * H)
    x = torch.randn(B, T, H, device=DEV, generator=g)
    T2 = (T + 1) // 2
    n = B * T2 * H
    yb, y16b = _nan(n), _nan(n, bf16)
    _ok(L.eb_time_reduce_fwd(_p(x), _p(yb), _p(y16b), B, T, H, _stream()), "eb_time_reduce_fwd")
    _guard("time_reduce y", yb, n)
    _guard("time_reduce y16", y16b, n)
    y = yb[:n].view(B, T2, H)
    _same("time_reduce y", y, _tr_ref(x.cpu()))
    _same("time_reduce y_bf16", y16b[:n].view(B, T2, H), y.bfloat16())
    yb2 = _nan(n)
    _ok(L.eb_time_reduce_fwd(_p(x), _p(yb2), None, B, T, H, _stream()), "eb_time_reduce_fwd")
    _same("time_reduce y without y_bf16", yb2[:n].view(B, T2, H), y)
    dy = torch.randn(B, T2, H, device=DEV, generator=g)
    dxb = _nan(B * T * H)
    _ok(L.eb_time_reduce_bwd(_p(dy), _p(dxb), B, T, H, _stream()), "eb_time_reduce_bwd")
    _guard("time_reduce dx", dxb, B * T * H)
    xr = x.cpu().requires_grad_(True)
    _tr_ref(xr).backward(dy.cpu())
    _same("time_reduce dx vs autograd of the zero-pad reference", dxb[:B * T * H].view(B, T, H), xr.grad)


# ---- embedding --------------------------------------------------------------------------------------------------------
def _emb_positions(ids, prepend, bos):
    B, U = ids.shape
    flat = ids.cpu().long()
    if prepend:
        flat = torch.cat([torch.full((B, 1), bos, dtype=torch.long), flat], 1)
    return flat.reshape(-1)


def _emb_bwd_ref(pos_ids, dout, dW0, pad):
    """Each id's positions added in position order from 0 (np.add.accumulate is sequential), then += into dW."""
    d = dout.reshape(len(pos_ids), -1).cpu().numpy().astype(np.float32)
    W = dW0.cpu().numpy().astype(np.float32).copy()
    ids = pos_ids.numpy()
    for i in np.unique(ids):
        if i == pad:
            continue
        acc = np.add.accumulate(d[ids == i], axis=0, dtype=np.float32)[-1]
        W[i] = W[i] + acc
    return torch.from_numpy(W)


def _emb_ids(name, B, U, V, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (B, U), generator=g)
    if name == "late-first":
        # positions 0 ... 39 hold only the ids 0, 1 and 3: ids 4 ... V-1 first occur past position 32 (the second
        # lane-strided step of the first-owner scan)
        ids.view(-1)[:40] = torch.tensor([0, 1, 3])[torch.randint(0, 3, (40,), generator=g)]
    return ids


# (name, B, U, V, E, prepend, bos, pad): every id recurs more than 32 times in "many" / "late-first"; pad == bos; U = 0;
# more positions than one grid-stride pass of ew_grid's 32 x #SMs blocks (8 x 32 x #SMs warps)
EMB_CASES = [
    ("many", 4, 60, 7, 33, True, 2, 1),
    ("late-first", 3, 80, 9, 40, True, 2, 1),
    ("pad-is-bos", 3, 50, 6, 16, True, 1, 1),
    ("no-prepend", 5, 17, 11, 64, False, 2, 0),
    ("priming-U0", 4, 0, 5, 24, True, 2, 1),
    ("gridstride", None, None, 5, 3, True, 2, 1),
]


@pytest.mark.parametrize("int64", [0, 1])
@pytest.mark.parametrize("name,B,U,V,E,prepend,bos,pad", EMB_CASES, ids=[c[0] for c in EMB_CASES])
def test_embedding(name, B, U, V, E, prepend, bos, pad, int64):
    if name == "gridstride":
        B, U = 8, 32 * _nsm() + 500                       # > 256 x #SMs positions
    L = _lib()
    ids = _emb_ids(name, B, U, V, seed=V * 100 + E)
    pos = _emb_positions(ids, prepend, bos)
    if name in ("many", "late-first"):
        assert int(torch.bincount(pos[pos != pad]).max()) > 32
    if name == "late-first":
        first = {int(i): int(torch.nonzero(pos == i)[0]) for i in torch.unique(pos)}
        assert max(first.values()) > 40
    g = _gen(V + E)
    W = torch.randn(V, E, device=DEV, generator=g)
    idsd = ids.to(DEV, torch.int64 if int64 else torch.int32)
    npos = B * (U + (1 if prepend else 0))
    n = npos * E
    ob, o16b = _nan(n), _nan(n, bf16)
    _ok(L.eb_embedding_fwd(_p(idsd) if U else None, int64, _p(W), _p(ob), _p(o16b), B, U, E, int(prepend), bos,
                           _stream()), "eb_embedding_fwd")
    _guard(name + " out", ob, n)
    _guard(name + " out_bf16", o16b, n)
    want = W.cpu()[pos].reshape(B, -1, E)
    _same(name + " gather", ob[:n].view(B, -1, E), want)
    _same(name + " out_bf16", o16b[:n].view(B, -1, E), want.bfloat16())
    dout = torch.randn(npos, E, device=DEV, generator=g)
    dW0 = torch.randn(V, E, device=DEV, generator=g)
    dWb = _nan(V * E)
    dWb[:V * E] = dW0.reshape(-1)
    _ok(L.eb_embedding_bwd(_p(idsd) if U else None, int64, _p(dout), _p(dWb), B, U, E, int(prepend), bos, pad,
                           _stream()), "eb_embedding_bwd")
    _guard(name + " dW", dWb, V * E)
    _same(name + " dW vs the sequential per-id sums", dWb[:V * E].view(V, E), _emb_bwd_ref(pos, dout, dW0, pad))


# ---- joint hidden -----------------------------------------------------------------------------------------------------
def _seq_sums(d):
    """(sum over u in order, sum over t in order) of d [B,T,U,J] as fp32, each from 0, on the CPU."""
    d = d.float().cpu()
    B, T, U, J = d.shape
    dep, ddp = torch.zeros(B, T, J), torch.zeros(B, U, J)
    for u in range(U):
        dep = dep + d[:, :, u]
    for s in range(T):
        ddp = ddp + d[:, s]
    return dep, ddp


def _ulp_bf16(t):
    """bf16 ulp at |t| (2^(e - 7) for |t| in [2^e, 2^(e+1)))."""
    _, e = torch.frexp(t.abs())
    return torch.ldexp(torch.ones_like(t), (e - 8).to(torch.int32))


# (B, T, U, J): U J > 256 and odd J (fp32 only), J = 8, J = 776 and 1024 (> 96 x 8 columns: a thread's q loop runs
# twice), U = 1
JOINT_CASES = [(2, 3, 40, 777), (1, 2, 1, 8), (2, 3, 5, 776), (1, 2, 3, 1024), (3, 4, 1, 16), (2, 5, 7, 8)]


@pytest.mark.parametrize("B,T,U,J", JOINT_CASES)
def test_joint_hidden(B, T, U, J):
    L = _lib()
    g = _gen(B * T * U * J)
    ep = torch.randn(B, T, J, device=DEV, generator=g)
    dp = torch.randn(B, U, J, device=DEV, generator=g)
    z = ep[:, :, None, :] + dp[:, None, :, :]             # torch fp32: exactly the kernel's add
    t = torch.tanh(z.double().cpu())
    n = B * T * U * J
    name = "joint B%d T%d U%d J%d" % (B, T, U, J)
    # fp32: tanhf
    hb = _nan(n)
    _ok(L.eb_joint_hidden_fwd(_p(ep), _p(dp), _p(hb), 0, B, T, U, J, _stream()), "eb_joint_hidden_fwd")
    _guard(name, hb, n)
    h = hb[:n].view(B, T, U, J)
    _report(name + " fp32 tanhf", h, t, 2.0 ** -22 * t.abs())
    # fp32 backward: dpre in place, dep / ddp the sequential sums of the kernel's own dpre
    dh = torch.randn(B, T, U, J, device=DEV, generator=g)
    dhb = _nan(n)
    dhb[:n] = dh.reshape(-1)
    depb, ddpb = _nan(B * T * J), _nan(B * U * J)
    _ok(L.eb_joint_hidden_bwd(_p(dhb), _p(h), 0, _p(depb), _p(ddpb), B, T, U, J, _stream()), "eb_joint_hidden_bwd")
    for b, k in ((dhb, n), (depb, B * T * J), (ddpb, B * U * J)):
        _guard(name + " bwd", b, k)
    dpre = dhb[:n].view(B, T, U, J)
    hd, dhd = h.double().cpu(), dh.double().cpu()
    _report(name + " fp32 dpre", dpre, dhd * (1 - hd * hd), 3 * U24 * dhd.abs() * (1 + hd * hd))
    dep, ddp = _seq_sums(dpre)
    _same(name + " fp32 dep (sum over u)", depb[:B * T * J].view(B, T, J), dep)
    _same(name + " fp32 ddp (sum over t)", ddpb[:B * U * J].view(B, U, J), ddp)
    if J % 8:
        return
    # bf16: tanh.approx, then RN to bf16
    hb16 = _nan(n, bf16)
    _ok(L.eb_joint_hidden_fwd(_p(ep), _p(dp), _p(hb16), 1, B, T, U, J, _stream()), "eb_joint_hidden_fwd bf16")
    _guard(name + " bf16", hb16, n)
    h16 = hb16[:n].view(B, T, U, J)
    # half a bf16 ulp for the rounding plus 2^-11 |t| for tanh.approx (2^-10.98 as a margin): within one ulp of
    # bf16_rn(tanh z), measured against the exact fp64 value (torch's fp64 -> bf16 conversion rounds twice)
    _report(name + " bf16 tanh.approx, RN to bf16", h16, t, 0.5 * _ulp_bf16(t) + 2.0 ** -10.98 * t.abs())
    # bf16 backward: dpre16 bitwise, ddp bitwise over t of the stored dpre16, dep barred (unrounded products)
    dh16 = torch.randn(B, T, U, J, device=DEV, generator=g).bfloat16()
    dhb16 = _nan(n, bf16)
    dhb16[:n] = dh16.reshape(-1)
    depb, ddpb = _nan(B * T * J), _nan(B * U * J)
    _ok(L.eb_joint_hidden_bwd(_p(dhb16), _p(h16), 1, _p(depb), _p(ddpb), B, T, U, J, _stream()),
        "eb_joint_hidden_bwd bf16")
    for b, k in ((dhb16, n), (depb, B * T * J), (ddpb, B * U * J)):
        _guard(name + " bf16 bwd", b, k)
    hf, gf = h16.float(), dh16.float()
    p32 = gf * (1 - hf * hf)                               # hf^2 exact: one rounding of 1 - h^2, one of the product
    d16 = dhb16[:n].view(B, T, U, J)
    _same(name + " bf16 dpre16", d16, p32.to(bf16))
    _, ddp = _seq_sums(d16)
    _same(name + " bf16 ddp (sum over t of the stored dpre16)", ddpb[:B * U * J].view(B, U, J), ddp)
    pd = gf.double().cpu() * (1 - hf.double().cpu() ** 2)
    _report(name + " bf16 dep (unrounded products)", depb[:B * T * J].view(B, T, J), pd.sum(2),
            (U + 2) * U24 * pd.abs().sum(2))


@pytest.mark.parametrize("B,T,U,J", [(1, 1, 5, 8), (2, 3, 1, 16), (1, 4, 3, 8), (2, 5, 3, 776), (1, 3, 4, 1024),
                                     (2, 500, 129, 640)])
def test_joint_dpre_reduce(B, T, U, J):
    """T = 1, U = 1, J = 8, J > 768 and the E6D2-like joint (B = 2, T' = 500, U + 1 = 129, J = 640)."""
    g = _gen(B + T + U + J)
    dpre = torch.randn(B, T, U, J, device=DEV, generator=g).bfloat16()
    depb, ddpb = _nan(B * T * J), _nan(B * U * J)
    _ok(_lib().eb_joint_dpre_reduce(_p(dpre), _p(depb), _p(ddpb), B, T, U, J, _stream()), "eb_joint_dpre_reduce")
    _guard("dpre_reduce dep", depb, B * T * J)
    _guard("dpre_reduce ddp", ddpb, B * U * J)
    dep, ddp = _seq_sums(dpre)
    _same("dpre_reduce dep (u in order)", depb[:B * T * J].view(B, T, J), dep)
    _same("dpre_reduce ddp (t in order)", ddpb[:B * U * J].view(B, U, J), ddp)


# ---- column sums ------------------------------------------------------------------------------------------------------
def _colsum_order(x, out0):
    """colsum_kernel's order, numpy fp32: lane k of 32 adds rows k, k + 32, ... from 0, a 16 ... 1 tree, += into out."""
    d = x.float().cpu().numpy()
    rows, N = d.shape
    nb = -(-rows // 32)
    pad = np.zeros((nb * 32, N), np.float32)
    pad[:rows] = d
    acc = np.zeros((32, N), np.float32)
    for i in range(nb):
        acc = acc + pad[i * 32:(i + 1) * 32]
    st = 16
    while st:
        acc[:st] = acc[:st] + acc[st:2 * st]
        st >>= 1
    return torch.from_numpy(out0.cpu().numpy() + acc[0])


# (name, dtype, rows, N, byte offset of x): every case takes colsum_kernel (fp32, or bf16 with N % 8 != 0 or a view
# that is not 16-byte aligned)
COLSUM_CASES = [("f32-r5-N37", f32, 5, 37, 0), ("f32-r100-N33", f32, 100, 33, 0), ("f32-r1000-N70", f32, 1000, 70, 0),
                ("bf16-r7-N13", bf16, 7, 13, 0), ("bf16-r300-N100", bf16, 300, 100, 0),
                ("bf16-r257-N64-offset2", bf16, 257, 64, 2), ("bf16-r31-N8-offset2", bf16, 31, 8, 2)]


@pytest.mark.parametrize("name,dtype,rows,N,off", COLSUM_CASES, ids=[c[0] for c in COLSUM_CASES])
def test_colsum_generic(name, dtype, rows, N, off):
    g = _gen(rows * N)
    x = (torch.randn(rows, N, device=DEV, generator=g) * 3).to(dtype)
    if off:
        x = _offset_copy(x, off // x.element_size())
        assert x.data_ptr() % 16 != 0
    out0 = torch.randn(N, device=DEV, generator=g)
    ob = _nan(N)
    ob[:N] = out0
    _ok(_lib().eb_colsum(_p(x), int(dtype == bf16), _p(ob), rows, N, _stream()), "eb_colsum")
    _guard(name, ob, N)
    _same(name + " vs colsum_kernel's order", ob[:N], _colsum_order(x, out0))


# ---- casts and the transpose ------------------------------------------------------------------------------------------
def _special_f32():
    bits = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800001,  # +-0, +-inf, NaNs
            0x00000001, 0x80000001, 0x007FFFFF, 0x00008000, 0x00018000, 0x00400000,             # subnormals, ties
            0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,                                     # ties: even / odd
            0x3F808001, 0x3F807FFF, 0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000, 0xFF7FFFFF,  # largest finite
            0x00800000, 0x80800000, 0x3F800000, 0x4B800000]
    v = torch.tensor(np.array(bits, dtype=np.uint32).view(np.int32), dtype=torch.int32).view(f32)
    return v


def _same_bf16_nan(name, got, x):
    want = x.cpu().bfloat16()
    got = got.cpu()
    nan = torch.isnan(x.cpu())
    assert bool(torch.isnan(got[nan].float()).all()), name + ": NaN not kept"
    _same(name, got[~nan], want[~nan])


@pytest.mark.parametrize("n", [1, 2, 3, 5, 6, 7, 28, 29, 30, 31, None])
def test_cast_bf16(n):
    """n % 4 = 1, 2, 3 tails, and (None) n past the grid-stride cap of 32 x #SMs blocks of 256 x 4 elements."""
    if n is None:
        n = 32 * _nsm() * 1024 * 2 + 3
    g = _gen(n)
    x = torch.randn(n, device=DEV, generator=g) * torch.exp2(torch.randint(-140, 128, (n,), device=DEV, generator=g)
                                                             .float())
    sp = _special_f32().to(DEV)
    k = min(n, sp.numel())
    x[:k] = sp[:k]
    x[n - k:] = sp[sp.numel() - k:]
    yb = _nan(n, bf16)
    _ok(_lib().eb_cast_bf16(_p(x), _p(yb), n, _stream()), "eb_cast_bf16")
    _guard("cast_bf16", yb, n)
    _same_bf16_nan("cast_bf16 n=%d" % n, yb[:n], x)


def test_cast_bf16_rejects_misaligned():
    x = torch.zeros(64, device=DEV)
    y = torch.zeros(64, dtype=bf16, device=DEV)
    assert _lib().eb_cast_bf16(_p(x[1:]), _p(y), 8, _stream()) == 2        # x 4-byte aligned
    assert _lib().eb_cast_bf16(_p(x), _p(y[1:]), 8, _stream()) == 2        # y 2-byte aligned


@pytest.mark.parametrize("dtype", [f32, bf16])
@pytest.mark.parametrize("rows,cols", [(37, 45), (1, 70), (70, 1), (1000, 37), (64, 96), (65535 * 32 + 37, 3)])
def test_transpose_to_bf16(rows, cols, dtype):
    """rows > 65535 x 32: more row tiles than gridDim.y holds."""
    g = _gen(rows + cols)
    x = torch.randn(rows, cols, device=DEV, generator=g).to(dtype)
    n = rows * cols
    yb = _nan(n, bf16)
    _ok(_lib().eb_transpose_to_bf16(_p(x), int(dtype == bf16), _p(yb), rows, cols, _stream()), "eb_transpose_to_bf16")
    _guard("transpose", yb, n)
    _same("transpose %dx%d %s" % (rows, cols, dtype), yb[:n].view(cols, rows), x.t().bfloat16())


# ---- Adam / AdamW -----------------------------------------------------------------------------------------------------
def _f(v):
    return float(np.float32(v))


def _bc(beta, step):
    return float(np.float32(1.0) - np.power(np.float32(beta), np.float32(step)))


def _adam_ref(p, g, m, v, lr, b1, b2, eps, wd, step, gscale, sumsq, max_norm, adamw):
    """fp64 Adam / AdamW step with the fp32 hyper-parameters the kernel receives, and the bars of m, v and the update
    (module docstring).  Returns None when the step is skipped."""
    lr, b1, b2, eps, wd, gscale = map(_f, (lr, b1, b2, eps, wd, gscale))
    bc1, bc2 = _bc(b1, step), _bc(b2, step)
    coef, e_coef = gscale, 0.0
    if sumsq is not None:
        norm = math.sqrt(sumsq) * abs(gscale)
        if not math.isfinite(norm):
            return None
        if max_norm > 0:
            c = _f(max_norm) / (norm + 1e-6)
            if c < 1:
                coef, e_coef = gscale * c, 6 * U24
    u = U24
    pd, gd, md, vd = (t.double().cpu() for t in (p, g, m, v))
    gi = gd * coef
    e_gi = (e_coef + 2 * u) * gi.abs()
    if not adamw and wd != 0:
        e_gi = e_gi + 2 * u * (wd * pd).abs()
        gi = gi + wd * pd
    a1, a2 = 1.0 - b1, 1.0 - b2                            # exact in fp32 (Sterbenz)
    mn = b1 * md + a1 * gi
    vn = b2 * vd + a2 * gi * gi
    e_m = 3 * u * (b1 * md.abs() + a1 * gi.abs()) + a1 * e_gi
    e_v = 4 * u * (b2 * vd + a2 * gi * gi) + a2 * 2 * gi.abs() * e_gi
    sv = torch.sqrt(vn)
    rel_sv = u + 0.5 * e_v / vn.clamp_min(1e-300)
    if adamw:
        D = sv + eps
        rel_D = (rel_sv * sv + u * D) / D
        q = mn / D
        inner = wd * pd + q
        e_inner = 2 * u * (wd * pd).abs() + (e_m / mn.abs().clamp_min(1e-300) + rel_D + u) * q.abs() \
            + u * inner.abs()
        k = lr * math.sqrt(bc2) / bc1
        step_v = k * inner
        e_step = 6 * u * step_v.abs() + k * e_inner
    else:
        D = sv / math.sqrt(bc2) + eps
        rel_D = ((rel_sv + 3 * u) * sv / math.sqrt(bc2) + u * D) / D
        q = mn / D
        k = lr / bc1
        step_v = k * q
        e_step = 5 * u * step_v.abs() + k * (e_m / mn.abs().clamp_min(1e-300) + rel_D) * q.abs()
    pn = pd - step_v
    # 2x: a margin over the first-order sum of the roundings; the fp32 subtraction p - step adds u |p_new|
    return pn, mn, vn, 2 * e_step + u * pn.abs(), 2 * e_m, 2 * e_v


def _adam_state(n, seed, scale_p):
    g = _gen(seed)
    p = torch.randn(n, device=DEV, generator=g) * scale_p
    gr = torch.randn(n, device=DEV, generator=g) * torch.exp2(torch.randint(-6, 7, (n,), device=DEV, generator=g)
                                                              .float())
    m = torch.randn(n, device=DEV, generator=g) * 0.5
    v = torch.rand(n, device=DEV, generator=g) * 2.0 + 1e-3
    return p, gr, m, v


# (name, n, adamw, wd, gscale, sumsq: None / "clip" (c < 1) / "noclip" (c >= 1) / "inf" / "nan", max_norm, legacy entry)
ADAM_CASES = [
    ("adam-wd0", 1000, 0, 0.0, 1.0, None, 0.0, False),
    ("adam-l2", 1000, 0, 0.1, 1.0, None, 0.0, False),
    ("adamw", 1000, 1, 0.1, 1.0, None, 0.0, False),
    ("adam-gscale-neg", 777, 0, 0.0, -0.37, None, 0.0, False),
    ("adam-clip", 1000, 0, 0.0, 0.5, "clip", 1.0, False),
    ("adamw-clip-l2", 1000, 1, 0.05, 2.0, "clip", 1.0, False),
    ("adam-noclip", 1000, 0, 0.0, 0.5, "noclip", 1.0, False),
    ("adam-norm-no-maxnorm", 513, 0, 0.01, -1.5, "noclip", 0.0, False),
    ("adam-gridstride", None, 0, 0.01, 0.25, "clip", 1.0, False),
    ("adamw-gridstride", None, 1, 0.01, 1.0, None, 0.0, False),
    ("legacy-adam", 1001, 0, 0.0, 0.5, None, 0.0, True),
    ("legacy-adam-l2", 1001, 0, 0.1, 1.0, None, 0.0, True),
]


@pytest.mark.parametrize("step", [1, 2, 10, 1000, 100000])
@pytest.mark.parametrize("name,n,adamw,wd,gscale,mode,max_norm,legacy", ADAM_CASES, ids=[c[0] for c in ADAM_CASES])
def test_adam_step(name, n, adamw, wd, gscale, mode, max_norm, legacy, step):
    if n is None:
        n = 32 * _nsm() * 256 * 2 + 77                       # past ew_grid's cap
    lr, b1, b2, eps = 1e-2, 0.9, 0.999, 1e-8
    p, g, m, v = _adam_state(n, seed=n + step, scale_p=lr)
    sumsq = None
    if mode is not None:
        s = float((g.double() ** 2).sum())
        norm = math.sqrt(s) * abs(gscale)
        if mode == "clip":
            max_norm = 0.3 * norm
        elif mode == "noclip" and max_norm > 0:
            max_norm = 2.0 * norm                            # c = 2: a clip applied here would halve the gradient
        sumsq = torch.tensor([s], device=DEV, dtype=f32)
    ref = _adam_ref(p, g, m, v, lr, b1, b2, eps, wd, step, gscale, float(sumsq) if sumsq is not None else None,
                    max_norm, adamw)
    p0 = p.clone()
    pb, mb, vb = _nan(n), _nan(n), _nan(n)
    pb[:n], mb[:n], vb[:n] = p, m, v
    L = _lib()
    if legacy:
        st = L.eb_adam_step(_p(pb), _p(g), _p(mb), _p(vb), n, lr, b1, b2, eps, wd, step, gscale, _stream())
    else:
        st = L.eb_adam_step_ex(_p(pb), _p(g), _p(mb), _p(vb), n, lr, b1, b2, eps, wd, step, gscale, _p(sumsq),
                               max_norm, adamw, _stream())
    _ok(st, name)
    for b in (pb, mb, vb):
        _guard(name, b, n)
    pn, mn, vn, e_p, e_m, e_v = ref
    tag = "%s step %d" % (name, step)
    _report(tag + " update p_new - p", pb[:n].double() - p0.double(), pn - p0.double().cpu(), e_p)
    _report(tag + " m", mb[:n], mn, e_m)
    _report(tag + " v", vb[:n], vn, e_v)


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
@pytest.mark.parametrize("adamw,max_norm", [(0, 1.0), (1, 0.0), (0, 0.0)])
def test_adam_nonfinite_norm_skips(bad, adamw, max_norm):
    n = 1000
    p, g, m, v = _adam_state(n, seed=3, scale_p=1.0)
    sumsq = torch.tensor([bad], device=DEV)
    pb, mb, vb = p.clone(), m.clone(), v.clone()
    _ok(_lib().eb_adam_step_ex(_p(pb), _p(g), _p(mb), _p(vb), n, 1e-2, 0.9, 0.999, 1e-8, 0.01, 5, 0.5, _p(sumsq),
                               max_norm, adamw, _stream()), "eb_adam_step_ex")
    _same("skip p", pb, p)
    _same("skip m", mb, m)
    _same("skip v", vb, v)


def test_adam_vs_torch_optim():
    """Not a bar on the kernel: the size of the difference from torch.optim.Adam, which computes the bias corrections
    in double from the unrounded betas, while the C ABI passes the betas as float (float(0.999) = 0.99900001...).  At
    step 1 from a non-zero state, bc2 = 1 - beta2 differs by 1.3e-5 relative, i.e. about 6e-6 in the update."""
    n, lr = 4096, 1e-2
    p, g, m, v = _adam_state(n, seed=11, scale_p=lr)
    pt = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([pt], lr=lr, betas=(0.9, 0.999), eps=1e-8, foreach=False)
    opt.state[pt] = {"step": torch.tensor(0.0), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
    pt.grad = g.clone()
    opt.step()
    pk, mk, vk = p.clone(), m.clone(), v.clone()
    _ok(_lib().eb_adam_step_ex(_p(pk), _p(g), _p(mk), _p(vk), n, lr, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None, 0.0, 0,
                               _stream()), "eb_adam_step_ex")
    dt = (pt.detach().double() - p.double()).cpu()
    dk = (pk.double() - p.double()).cpu()
    big = dt.abs() > 0.01 * dt.abs().max()                 # (where m is near zero, the update has no relative digits)
    rel = float(((dk - dt).abs() / dt.abs())[big].max())
    print("  adam vs torch.optim.Adam, step 1: max relative difference of the update %.3g" % rel)
    assert rel < 1e-4


# ---- sum of squares ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1000, 256 * 7 + 3, None])
def test_sumsq(n):
    """Accumulates into out; n not a multiple of the block, and (None) past ew_grid's cap."""
    if n is None:
        n = 32 * _nsm() * 256 * 3 + 17
    g = _gen(n)
    x = torch.randn(n, device=DEV, generator=g)
    out = torch.tensor([3.25, float("nan")], device=DEV)
    _ok(_lib().eb_sumsq(_p(x), n, _p(out), _stream()), "eb_sumsq")
    assert bool(torch.isnan(out[1]))
    grid = min(max(-(-n // 256), 1), 32 * _nsm())
    n_add = -(-n // (grid * 256)) + 1 + 10 + grid + 1
    s = (x.double() ** 2).sum().cpu()
    _report("sumsq n=%d" % n, out[:1], s.view(1) + 3.25, (n_add * U24 * (s + 3.25)).view(1))


# ---- front end --------------------------------------------------------------------------------------------------------
def _reflect_ref(x, L, Lp, pad):
    """The kernel's padded row: reflect without edge repeat at both ends, zero from L + 2 pad to Lp; and the index r."""
    i = np.arange(Lp)
    r = i - pad
    r = np.where(r < 0, -r, r)
    r = np.where(r >= L, 2 * (L - 1) - r, r)
    inside = i < L + 2 * pad
    return np.where(inside, r, 0), inside


@pytest.mark.parametrize("B,L,pad,extra", [(3, 2, 1, 5), (2, 50, 49, 0), (1, 400, 256, 160), (4, 1000, 8, 7)])
def test_fe_preemph_pad(B, L, pad, extra):
    Lp = L + 2 * pad + extra
    g = _gen(L * 7 + pad)
    x = torch.randn(B, L, device=DEV, generator=g)
    r, inside = _reflect_ref(x, L, Lp, pad)
    xc = x.cpu().numpy()
    want = np.where(inside[None, :], xc[:, r], np.float32(0)).astype(np.float32)
    Lib = _lib()
    xb = _nan(B * Lp)
    _ok(Lib.eb_fe_preemph_pad(_p(x), _p(xb), B, L, Lp, pad, 0.97, 0, _stream()), "eb_fe_preemph_pad")
    _guard("preemph_pad", xb, B * Lp)
    _same("preemph_pad (no pre-emphasis)", xb[:B * Lp].view(B, Lp), torch.from_numpy(want))
    p = 0.97
    xb = _nan(B * Lp)
    _ok(Lib.eb_fe_preemph_pad(_p(x), _p(xb), B, L, Lp, pad, p, 1, _stream()), "eb_fe_preemph_pad")
    _guard("preemph_pad", xb, B * Lp)
    xd = x.double().cpu().numpy()
    pf = _f(p)
    prev = np.where(r > 0, xd[:, np.maximum(r - 1, 0)], 0.0)
    ref = np.where(inside[None, :], xd[:, r] - pf * prev, 0.0)
    bar = np.where(inside[None, :], 2 * U24 * (np.abs(xd[:, r]) + np.abs(pf * prev)), 0.0)
    _report("preemph_pad B%d L%d pad%d (pre-emphasis)" % (B, L, pad), xb[:B * Lp].view(B, Lp), torch.from_numpy(ref),
            torch.from_numpy(bar))


@pytest.mark.parametrize("rows,nb", [(1, 1), (37, 257), (1000, 201)])
def test_fe_power(rows, nb):
    g = _gen(rows + nb)
    spec = torch.randn(rows, 2 * nb, device=DEV, generator=g) * 10
    pb = _nan(rows * nb)
    _ok(_lib().eb_fe_power(_p(spec), _p(pb), rows, nb, _stream()), "eb_fe_power")
    _guard("power", pb, rows * nb)
    s = spec.double().cpu()
    ref = s[:, :nb] ** 2 + s[:, nb:] ** 2
    _report("power rows%d nb%d" % (rows, nb), pb[:rows * nb].view(rows, nb), ref, 2 * U24 * ref * (1 + 4 * U24))


# (B, rows_per_utt, n_frames, seq_len, n_mels, n_stack, t_out): rows_per_utt > n_frames (the unused slots are NaN, never
# read), seq_len < n_frames (masked frames), t_out n_stack > n_frames (the stacking pad)
LOGSTACK_CASES = [(2, 13, 10, 8, 5, 3, 4), (3, 6, 6, 6, 7, 1, 6), (1, 20, 17, 20, 40, 4, 5), (2, 9, 1, 1, 3, 2, 1)]


@pytest.mark.parametrize("B,R,F,seq_len,n_mels,n_stack,t_out", LOGSTACK_CASES)
def test_fe_log_stack(B, R, F, seq_len, n_mels, n_stack, t_out):
    g = _gen(B * R + n_mels)
    mel = torch.exp(3 * torch.randn(B, R, n_mels, device=DEV, generator=g))
    mel[:, :, 0] = 0.0                                     # log(0 + 1e-20)
    mel[:, F:] = float("nan")                              # slots past n_frames are never read
    W = n_mels * n_stack
    n = B * t_out * W
    m = mel.cpu()
    t = torch.arange(t_out)[:, None] * n_stack + torch.arange(W)[None, :] // n_mels          # frame f of (t, c)
    c_m = torch.arange(W)[None, :] % n_mels
    valid = (t < F) & (t < seq_len)
    Lib = _lib()
    for take_log in (0, 1):
        ob = _nan(n)
        _ok(Lib.eb_fe_log_stack(_p(mel), _p(ob), B, R, F, seq_len, n_mels, n_stack, t_out, take_log, _stream()),
            "eb_fe_log_stack")
        _guard("log_stack", ob, n)
        got = ob[:n].view(B, t_out, W).cpu()
        src = m[:, t.clamp_max(R - 1), c_m.expand_as(t)]
        if not take_log:
            want = torch.where(valid[None], src, torch.zeros(()))
            _same("log_stack (no log)", got, want)
        else:
            z = (torch.where(valid[None], src, torch.ones(())) + 1e-20).double()     # fp32 add, then fp64 log
            ref = torch.where(valid[None], torch.log(z), torch.zeros((), dtype=f64))
            _same("log_stack zeros outside the frames", got[~valid.expand_as(got)],
                  torch.zeros(int((~valid.expand_as(got)).sum())))
            _report("log_stack B%d R%d F%d (log)" % (B, R, F), got, ref, 2.0 ** -22 * ref.abs())


# (name, axis, spans per utterance [start, end)): overlapping spans, start == end (a width-0 draw), end > D (the host
# draws start + randrange(max_width)), start > end (empty), fill != 0
MASK_CASES = [
    ("time-overlap", 2, [[[3, 9], [7, 12], [20, 20]], [[0, 1], [40, 90], [5, 2]]]),
    ("freq-edges", 1, [[[0, 4], [4, 4], [10, 16]], [[15, 30], [2, 3], [9, 8]]]),
    ("time-none", 2, [[[5, 5], [0, 0], [7, 3]], [[0, 77], [0, 0], [0, 0]]]),
]


@pytest.mark.parametrize("fill", [0.0, -3.5])
@pytest.mark.parametrize("name,axis,spans", MASK_CASES, ids=[c[0] for c in MASK_CASES])
def test_fe_mask(name, axis, spans, fill):
    B, D1, D2 = 2, 16, 77
    g = _gen(len(name))
    x = torch.randn(B, D1, D2, device=DEV, generator=g)
    sp = torch.tensor(spans, dtype=torch.int32)
    n = B * D1 * D2
    xb = _nan(n)
    xb[:n] = x.reshape(-1)
    _ok(_lib().eb_fe_mask(_p(xb), _p(sp.to(DEV)), B, D1, D2, sp.shape[1], axis, fill, _stream()), "eb_fe_mask")
    _guard(name, xb, n)
    D = D1 if axis == 1 else D2
    pos = torch.arange(D)
    hit = ((pos[None, None, :] >= sp[:, :, 0:1]) & (pos[None, None, :] < sp[:, :, 1:2])).any(1)     # [B, D]
    mask = hit[:, :, None].expand(B, D1, D2) if axis == 1 else hit[:, None, :].expand(B, D1, D2)
    want = torch.where(mask, torch.full((), fill), x.cpu())
    _same("%s fill %g" % (name, fill), xb[:n].view(B, D1, D2), want)
