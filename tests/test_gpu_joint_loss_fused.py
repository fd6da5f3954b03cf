"""Kernel-level fp64 parity of the fused joint-loss path of the bf16 mode, the path JointLoss takes on every training
step of the headline:

    eb_joint_logits_lse    logits16 = bf16(hid16 . w2_16^T + b2), and from the fp32 accumulators the softmax statistics
                           denom = -logsumexp, lpb = log p(blank), lpl = log p(label[u]) of every valid cell
    eb_rnnt_loss_lattice   alpha / beta wavefronts over those statistics, costs = -ll
    eb_rnnt_loss_bwd_bf16  d loss / d logits, bf16, in place over the logits (16-byte, 4-wide and scalar variants)

Inputs are hid16 [B*T*U, J] bf16 (tanh-range values), w2_16 [V, J] bf16 and an fp32 bias b2.  X = hid16 @ w2_16^T + b2
in fp64 (on the device, torch float64) is the exact logit of the same operands; X16 = bf16(X).  References come from
the C oracle (oracle/loss.py) in fp64 and from torch fp64.  Every bar is derived from an error model stated in the
test's docstring; every measured figure is printed next to its bar (pytest -s).

The shape matrix (CASES) names the code path each case reaches: tile edges of the 128-wide column tiles, the K tail,
narrow and odd vocabularies, the blank and the labels outside the first tile, no bias, no labels, ragged lengths and a
problem large enough that every CTA of the persistent GEMM handles at least two row blocks.  The file runs in about
10 s on an H100."""
import math

import numpy as np
import pytest
import torch

from oracle import loss as ol
from tests import loss_restate as lr

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
NAN = float("nan")

# |g - ref| <= GRAD_REL |ref| + GRAD_ABS element-wise, ||g - ref||_F / ||ref||_F <= GRAD_FRO (sections c and d)
GRAD_REL, GRAD_ABS, GRAD_FRO = 2.0 ** -8, 2e-4, 5e-3
STAT_ABS = 1e-4           # denom / lpb / lpl (section a)
COST_REL = 1e-5           # costs and ll_fwd vs ll_bwd (section b): the bar of the fp32 loss path


def _many_row_blocks_T(B, U):
    """maxT such that B*T*U cells make more than 2 x (SM count) row blocks of 128: every CTA of the persistent LSE
    GEMM (grid = one CTA per SM) then starts the statistics of a second row block (the reset at nb == 0)."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    rows = 2 * nsm * 128 + 128 + 37                           # and a partial last row block
    return -(-rows // (B * U))


# name: (B, T, U, V, J, blank, xlen, ylen, bias)      (T = None: computed by _many_row_blocks_T)
CASES = {
    # bench shape (V = 1024, J = 640, blank = 0): 16-byte gradient kernel; ragged, xlen = 1 and ylen = 0
    "v1024_bench": (3, 24, 21, 1024, 640, 0, [24, 17, 1], [20, 11, 0], True),
    # last column tile 104 wide; x8 gradient with V % 256 != 0; blank in the last tile
    "v1000_blank_last": (2, 19, 13, 1000, 128, 999, [19, 12], [12, 5], True),
    # one full tile plus an 8-wide tile; blank = 128 opens the second tile; K tail (J = 64 + 8)
    "v136_blank128_j72": (2, 23, 11, 136, 72, 128, [23, 9], [10, 10], True),
    # vocabulary narrower than one tile (threads owning no column); a single partial k-block; blank = V - 1
    "v72_j8": (3, 15, 9, 72, 8, 71, [15, 15, 4], [8, 0, 8], True),
    # V % 8 != 0: 4-wide bf16 gradient path; no bias
    "v12_nobias": (2, 17, 7, 12, 64, 0, [17, 11], [6, 3], False),
    # odd V: scalar stores in the epilogue, scalar gradient path; blank in the middle
    "v29_odd": (2, 13, 8, 29, 40, 5, [13, 7], [7, 4], True),
    # maxU = 1 with labels = NULL: no label anywhere; V = 128 + 72
    "v200_maxU1_nolabels": (2, 31, 1, 200, 64, 199, [31, 20], [0, 0], True),
    # B = 1, blank = 128
    "v256_b1": (1, 37, 6, 256, 96, 128, [37], [5], True),
    # every CTA handles >= 2 row blocks; ragged so that the valid-cell decode is reset too
    "v136_many_row_blocks": (8, None, 33, 136, 64, 3, None, None, True),
}


def _make_case(name):
    B, T, U, V, J, blank, xl, yl, bias = CASES[name]
    seed = sum(map(ord, name))
    rng = np.random.RandomState(seed)
    if T is None:
        T = _many_row_blocks_T(B, U)
        xl = [T] + list(rng.randint(1, T + 1, size=B - 1))
        yl = [U - 1] + list(rng.randint(0, U, size=B - 1))
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = B * T * U
    hid = (torch.rand(n, J, device="cuda", generator=g) * 2 - 1).to(bf16)
    # logits of standard deviation ~3 (|X| up to ~15, -logsumexp ~ -10)
    w2 = (torch.randn(V, J, device="cuda", generator=g) * (3.0 * math.sqrt(3.0 / J))).to(bf16)
    b2 = torch.randn(V, device="cuda", generator=g) if bias else None
    X = hid.double() @ w2.double().t()
    if bias:
        X += b2.double()
    lab = lr.planted_labels(rng, B, U, V, blank)
    xlen, ylen = np.asarray(xl, np.int32), np.asarray(yl, np.int32)
    t = np.arange(T)[None, :, None]
    u = np.arange(U)[None, None, :]
    valid = (t < xlen[:, None, None]) & (u <= ylen[:, None, None])
    return dict(name=name, B=B, T=T, U=U, V=V, J=J, blank=blank, hid=hid, w2=w2, b2=b2, X=X.view(B, T, U, V),
                lab=lab, xlen=xlen, ylen=ylen, valid=valid,
                lab_d=torch.as_tensor(lab, device="cuda") if U > 1 else None,
                xlen_d=torch.as_tensor(xlen, device="cuda"), ylen_d=torch.as_tensor(ylen, device="cuda"))


def _lib():
    from edgedict_b200._lib import lib
    return lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ws(c):
    n = _lib().eb_rnnt_workspace_bytes(c["B"], c["T"], c["U"], 4) // 4
    return torch.full((n,), NAN, dtype=torch.float32, device="cuda")


def _views(c, ws):
    B, n = c["B"], c["B"] * c["T"] * c["U"]
    sh = (B, c["T"], c["U"])
    return dict(denom=ws[:n].view(sh), lpb=ws[n:2 * n].view(sh), lpl=ws[2 * n:3 * n].view(sh),
                alphas=ws[3 * n:4 * n].view(sh), betas=ws[4 * n:5 * n].view(sh),
                ll_fwd=ws[5 * n:5 * n + B], ll_bwd=ws[5 * n + B:5 * n + 2 * B])


def _lse(c, ws):
    """eb_joint_logits_lse into a NaN-prefilled logits buffer and workspace."""
    B, T, U, V, J = c["B"], c["T"], c["U"], c["V"], c["J"]
    n = B * T * U
    logits = torch.full((B, T, U, V), NAN, dtype=bf16, device="cuda")
    rc = _lib().eb_joint_logits_lse(_p(c["hid"]), _p(c["w2"]), _p(c["b2"]), _p(logits), _p(c["lab_d"]),
                                    _p(c["xlen_d"]), _p(c["ylen_d"]), _p(ws[:n]), _p(ws[n:2 * n]),
                                    _p(ws[2 * n:3 * n]), B, T, U, V, J, c["blank"], _stream())
    assert rc == 0, rc
    return logits


def _lattice(c, ws, need_beta=1):
    costs = torch.full((c["B"],), NAN, dtype=torch.float32, device="cuda")
    rc = _lib().eb_rnnt_loss_lattice(_p(c["xlen_d"]), _p(c["ylen_d"]), c["B"], c["T"], c["U"], _p(ws), _p(costs),
                                     need_beta, _stream())
    assert rc == 0, rc
    return costs


def _loss_fwd_f32(c, ws, logits):
    """The fp32 loss (statistics + lattice) of eb_rnnt_loss_fwd on [B,T,U,V] fp32 logits into the workspace."""
    costs = torch.empty(c["B"], dtype=torch.float32, device="cuda")
    rc = _lib().eb_rnnt_loss_fwd(_p(logits), _p(c["lab_d"]), _p(c["xlen_d"]), _p(c["ylen_d"]), c["B"], c["T"], c["U"],
                                 c["V"], c["blank"], 4, _p(ws), _p(costs), 1, _stream())
    assert rc == 0, rc
    return costs


def _bwd_bf16(c, ws, logits16, out, gscale=None, host_scale=1.0):
    per_batch = int(gscale is not None and gscale.numel() > 1)
    rc = _lib().eb_rnnt_loss_bwd_bf16(_p(logits16), _p(out), _p(c["lab_d"]), _p(c["xlen_d"]), _p(c["ylen_d"]),
                                      c["B"], c["T"], c["U"], c["V"], c["blank"], _p(ws), _p(gscale), per_batch,
                                      float(host_scale), _stream())
    assert rc == 0, rc
    return out


def _chain(c):
    """The path as JointLoss runs it: statistics + logits, lattice, gradient in place over the logits with the
    upstream gradient of loss = costs.sum() / B (gscale = [1], host_scale = 1 / B)."""
    ws = _ws(c)
    logits = _lse(c, ws)
    r = dict(logits=logits.clone(), ws_lse=ws.clone())
    r["costs"] = _lattice(c, ws)
    r["ws"] = ws.clone()
    gs = torch.ones(1, dtype=torch.float32, device="cuda")
    r["grad"] = _bwd_bf16(c, ws, logits, logits, gs, 1.0 / c["B"])
    torch.cuda.synchronize()
    return r


def _oracle_logits(c, x, want_grads=True):
    """oracle.loss.logits in fp64 on the [B,T,U,V] logits x (torch tensor, any float dtype)."""
    return ol.logits(x.double().cpu().numpy(), c["lab"], c["xlen"], c["ylen"], blank=c["blank"],
                     want_grads=want_grads, dtype=np.float64)


def _bf16_ulp(x):
    """Spacing of bf16 numbers (8 significant bits) at |x|, fp64."""
    _, e = torch.frexp(x.abs())
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


def _grad_errors(g, ref):
    """(max over elements of |g - ref| / (GRAD_REL |ref| + GRAD_ABS), Frobenius relative error)."""
    g = g.double()
    d = (g - ref).abs()
    ratio = float((d / (GRAD_REL * ref.abs() + GRAD_ABS)).max())
    fro = float(torch.linalg.vector_norm(g - ref) / torch.linalg.vector_norm(ref))
    return ratio, fro


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    c = _make_case(request.param)
    c["run"] = _chain(c)
    return c


def test_lse_statistics_and_bf16_logits(case):
    """(a) eb_joint_logits_lse against fp64 statistics of X.

    Error model of the statistics: the GEMM accumulates J bf16 products in fp32 (2^-24 relative per add, a random walk
    of ~sqrt(J) 2^-24 |X| on a logit: ~2e-5 at J = 640, |X| ~ 15), the online sum-exp uses ex2.approx (2^-22 relative)
    over V terms in fp32 and one logf (~1e-6 on |denom| ~ 10).  Bar: absolute 1e-4.  A wrong row-block reset, a lost
    quad merge, statistics taken before the bias or a padded column counted as exp(0 - max) exceed it.

    Error model of the logits: the fp32 accumulator is rounded once to bf16, so |L16 - X| <= 1/2 ulp_bf16(X) plus the
    fp32 accumulation error, which may push the rounding across one boundary: one ulp, plus J 2^-24 sum_j |h_j w_j| + |b|
    for values near zero where the accumulation error dominates.  More than that is an error.

    Cells the kernel must not write (padded cells, and the lattice part of the workspace) still hold the NaN prefill."""
    c, r = case, case["run"]
    B, T, U, V, blank = c["B"], c["T"], c["U"], c["V"], c["blank"]
    X = c["X"]
    valid = torch.as_tensor(c["valid"], device="cuda")
    lse = torch.logsumexp(X, dim=-1)
    w = _views(c, r["ws_lse"])
    err_d = float((w["denom"].double() + lse)[valid].abs().max())
    err_b = float((w["lpb"].double() - (X[..., blank] - lse))[valid].abs().max())
    err_l = 0.0
    if U > 1:
        lab = torch.as_tensor(c["lab"], device="cuda").long()                 # [B, U-1]
        xl = torch.gather(X[:, :, :U - 1, :], 3, lab[:, None, :, None].expand(B, T, U - 1, 1))[..., 0]
        has_lab = valid[:, :, :U - 1] & (torch.arange(U - 1, device="cuda")[None, None, :] <
                                         torch.as_tensor(c["ylen"], device="cuda")[:, None, None])
        if bool(has_lab.any()):
            err_l = float((w["lpl"][:, :, :U - 1].double() - (xl - lse[:, :, :U - 1]))[has_lab].abs().max())
    print("%s: denom err %.2e, lpb err %.2e, lpl err %.2e (bar %.0e); |denom| max %.1f"
          % (c["name"], err_d, err_b, err_l, STAT_ABS, float(lse[valid].abs().max())))
    assert err_d <= STAT_ABS and err_b <= STAT_ABS and err_l <= STAT_ABS, (err_d, err_b, err_l)
    # padded cells of the statistics, and everything past them, are never written
    pad = ~valid
    for k in ("denom", "lpb", "lpl"):
        assert bool(w[k][pad].isnan().all()), k
    n = B * T * U
    assert bool(r["ws_lse"][3 * n:].isnan().all())
    # bf16 logits: within one ulp of X (plus the fp32 accumulation bound near zero), every row written
    L16 = r["logits"].double()
    S = c["hid"].double().abs() @ c["w2"].double().abs().t()
    if c["b2"] is not None:
        S += c["b2"].double().abs()
    bound = _bf16_ulp(X) + c["J"] * 2.0 ** -24 * S.view(B, T, U, V)
    ratio = float(((L16 - X).abs() / bound).max())
    print("%s: bf16 logits max |L16 - X| / (ulp + accumulation bound) = %.3f (bar 1)" % (c["name"], ratio))
    assert not bool(L16.isnan().any())
    assert ratio <= 1.0, ratio


def test_lattice_costs_over_fused_statistics(case):
    """(b) eb_rnnt_loss_lattice on the statistics of (a) against oracle.loss.logits(X) in fp64.

    Error model: the lattice adds ~T + U log-probabilities in fp32 with lse2 (log1pf / expf, ~1 ulp each), on statistics
    good to ~1e-6: relative error a few 1e-7 on the cost.  Bar: relative 1e-5, the bar of the fp32 loss path
    (test_gpu_loss.py).  ll_fwd and ll_bwd sum the same lattice in two orders: same bar.  need_beta = 0 must not change
    the forward pass: the same cost bits."""
    c, r = case, case["run"]
    costs = r["costs"].double().cpu().numpy()
    ref, _ = _oracle_logits(c, c["X"], want_grads=False)
    rel = float(np.max(np.abs(costs - ref) / np.abs(ref)))
    w = _views(c, r["ws"])
    llf, llb = w["ll_fwd"].double(), w["ll_bwd"].double()
    rel_fb = float(((llf - llb).abs() / llf.abs()).max())
    print("%s: costs rel err %.2e, ll_fwd vs ll_bwd rel %.2e (bar %.0e); costs %s"
          % (c["name"], rel, rel_fb, COST_REL, np.array2string(ref[:3], precision=2)))
    assert rel <= COST_REL and rel_fb <= COST_REL, (rel, rel_fb)
    ws = r["ws_lse"].clone()
    costs_nb = _lattice(c, ws, need_beta=0)
    assert torch.equal(costs_nb.view(torch.int32), r["costs"].view(torch.int32))
    nb = _views(c, ws)
    assert bool(nb["betas"].isnan().all()) and bool(nb["ll_bwd"].isnan().all())     # need_beta = 0: no beta pass


def test_bf16_gradient_kernel_in_isolation(case):
    """(c) eb_rnnt_loss_bwd_bf16 on X16 = bf16(X), with the workspace filled by the fp32 loss on X16.float(): the
    statistics and the exponent both see X16, so oracle.loss.logits(X16) in fp64 is the exact answer.

    Error model: the fp32 lattice (|alpha + beta - ll| up to ~1e3, a few fp32 ulps: ~1e-4 relative in the exponent
    at worst) and one rounding of the result to bf16 (< 2^-8 relative).  Bars: |g - ref| <= 2^-8 |ref| + 2e-4 per
    element, Frobenius relative error <= 5e-3 (bf16 rounding alone gives ~1.1e-3 rms).  The rounding reaches 2^-8
    relative just above a power of two, so a worst element near 0.8-0.97 of its bar is the expected figure; the 2e-4
    absolute term is the room left for the lattice.  Padded cells are exactly 0.
    In place and out of place give the same bits.  host_scale and gscale ([1], and [B] with mixed signs) scale the
    result."""
    c = case
    B = c["B"]
    X16 = c["X"].to(bf16)
    ws = _ws(c)
    _loss_fwd_f32(c, ws, X16.float())
    _, gref = _oracle_logits(c, X16)
    gref = torch.as_tensor(gref, device="cuda")
    pad = torch.as_tensor(~c["valid"], device="cuda")
    out = _bwd_bf16(c, ws, X16, torch.full_like(X16, NAN))
    x_ip = X16.clone()
    _bwd_bf16(c, ws, x_ip, x_ip)
    assert torch.equal(out.view(torch.int16), x_ip.view(torch.int16)), "in-place and out-of-place differ"
    assert bool((out[pad] == 0).all()) and not bool(out.isnan().any())
    signs = torch.tensor([(-1.5) ** (b + 1) for b in range(B)], dtype=torch.float32, device="cuda")
    variants = [("1", None, 1.0, 1.0),
                ("host 0.37, gscale[1] = -1.5", torch.tensor([-1.5], device="cuda"), 0.37,
                 torch.tensor(-1.5 * 0.37, dtype=torch.float64, device="cuda")),
                ("host 0.25, gscale[B] mixed signs", signs, 0.25, signs.double()[:, None, None, None] * 0.25)]
    for tag, gs, hs, scale in variants:
        g = out if gs is None else _bwd_bf16(c, ws, X16, torch.full_like(X16, NAN), gs, hs)
        ref = gref * scale
        ratio, fro = _grad_errors(g, ref)
        print("%s [%s]: grad element err / bar %.3f, Frobenius rel %.2e (bar %.0e)" % (c["name"], tag, ratio, fro,
                                                                                       GRAD_FRO))
        assert ratio <= 1.0 and fro <= GRAD_FRO, (tag, ratio, fro)
        assert bool((g[pad] == 0).all())


def _restated_grad(c, L16):
    """fp64 restatement of what the chained kernels compute: alpha, beta and ll from log_softmax(X) through
    oracle.loss.logprobs, the exponent on the bf16 logits L16 the GEMM wrote, the branches of loss.cu's gradient kernels:
        g_v = exp(a + b - ll + d + x_v) - [v = blank] exp(c_blank + x_v) - [v = label[u]] exp(c_lab + x_v)
        c_blank = a - ll + d + beta(t+1, u) if t < T_b - 1, a - ll + d at the last cell, else no term
        c_lab   = a - ll + d + beta(t, u+1)  if u < U_b - 1"""
    lp, den = ol.log_softmax(c["X"].cpu().numpy(), dtype=np.float64)
    costs, _, al, be = ol.logprobs(lp, c["lab"], c["xlen"], c["ylen"], blank=c["blank"], dtype=np.float64,
                                   want_lattice=True)
    del lp
    dev = lambda a: torch.as_tensor(a, device="cuda")
    return _grad_formula(c, dev(al), dev(be), dev(den), -dev(costs), L16.double())


def _grad_formula(c, a, b, d, ll, x):
    """g [B,T,U,V] fp64 from alpha, beta, denom [B,T,U], ll [B] and the logits x, zero on padded cells
    (loss_restate.grad_formula)."""
    return lr.grad_formula(a, b, d, ll, x, c["lab"], c["xlen_d"], c["ylen_d"], c["blank"])


def test_chained_path_as_joint_loss_runs_it(case):
    """(d) The chain (a) -> (b) -> in-place gradient, with JointLoss's scales (gscale = [1], host_scale = 1/B).

    Against the fp64 restatement of the kernels (_restated_grad, the exponent on the bf16 logits the GEMM wrote): the
    statistics of (a) (<1e-4 absolute), the fp32 lattice and one bf16 rounding: the bars of (c).

    Against the true gradient oracle.loss.logits(X): the kernel's exponent sees L16 = X + delta, |delta_v| <=
    ulp_bf16(X_v) <= 2^-7 |X_v| (test a), and every term of g_v carries the same factor exp(delta_v), so
        |g_v - g_true_v| <= ((1 + 2^-8) expm1(ulp_bf16(X_v)) + 2^-8) |g_true_v| + 2e-4.
    The Frobenius figure printed documents how far the headline path's gradient is from the exact one."""
    c, r = case, case["run"]
    B = c["B"]
    pad = torch.as_tensor(~c["valid"], device="cuda")
    g = r["grad"]
    assert not bool(g.isnan().any()) and bool((g[pad] == 0).all())
    ref = _restated_grad(c, r["logits"]) / B
    ratio, fro = _grad_errors(g, ref)
    print("%s: chained grad vs restatement: element err / bar %.3f, Frobenius rel %.2e (bar %.0e)"
          % (c["name"], ratio, fro, GRAD_FRO))
    assert ratio <= 1.0 and fro <= GRAD_FRO, (ratio, fro)
    _, gtrue = _oracle_logits(c, c["X"])
    gtrue = torch.as_tensor(gtrue, device="cuda") / B
    X = c["X"]
    bar = ((1 + 2.0 ** -8) * torch.expm1(_bf16_ulp(X)) + 2.0 ** -8) * gtrue.abs() + GRAD_ABS
    d = (g.double() - gtrue).abs()
    ratio_t = float((d / bar).max())
    fro_t = float(torch.linalg.vector_norm(g.double() - gtrue) / torch.linalg.vector_norm(gtrue))
    print("%s: chained grad vs true fp64 gradient: element err / bar %.3f, Frobenius rel %.2e"
          % (c["name"], ratio_t, fro_t))
    assert ratio_t <= 1.0, ratio_t


def test_chain_is_bitwise_repeatable(case):
    """(e) A second run of the chain on the same inputs gives the same bits: logits, the whole workspace (statistics,
    lattice, likelihoods and the untouched NaN prefill), costs and gradients (DESIGN.md section 6)."""
    c, r = case, case["run"]
    r2 = _chain(c)
    for k, view in (("logits", torch.int16), ("ws_lse", torch.int32), ("costs", torch.int32), ("ws", torch.int32),
                    ("grad", torch.int16)):
        assert torch.equal(r[k].view(view), r2[k].view(view)), k
