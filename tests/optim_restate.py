"""fp64 restatement of ONE step of each csrc/optim.cu kernel over a flat bucket, teacher-forced from the kernel's fp32
inputs, with the per-element bar of tests/test_gpu_optim_fp64.py's error model.

Every function takes float64 tensors in the bucket's layout (length n, pads ignored), the per-group hyperparameters as
the C ABI receives them (fp64: ``dict(lr=[..], wd=[..], b1=[..], b2=[..], eps=[..])``), the device step counters the
prologue wrote and the gradient coefficient ctl[0].  It returns, for every element a tile covers (``Layout.pos``), the
fp64 value and its bar.  Where a later expression reads a state the kernel also wrote (p reads the new momentum, m, v
or segv), the caller may pass the kernel's own value (``*_new``), so each bar covers one expression's roundings.
The bars are ``bar(k, M)``: k roundings, M the expression evaluated on absolute values.  Works on any device (the
host tests pin it against tests/optim_oracle.py on the CPU)."""
import math

import numpy as np
import torch

f64, i64 = torch.float64, torch.int64
U24 = 2.0 ** -24
TINY = 2.0 ** -149            # the absolute error of one rounding into the subnormal range
OPT_THREADS = 256


def bar(k, M):
    """k fp32 roundings, each off by at most u = 2^-24 relative to a term bounded by M; 2^-10 covers the O(k^2 u^2)
    second-order terms (k <= 40 here) and k TINY a rounding that lands below the normal range."""
    return k * U24 * M * (1 + 2.0 ** -10) + k * TINY


def sumsq_terms(length):
    """The largest number of squares one accumulator of seg_sumsq_partial_kernel sums over a tile of ``length``
    elements (thread t: a0 .. a3 take j, j + 256, j + 512, j + 768 for j = t, t + 1024, ... while j + 768 < length,
    then a0 takes the rest, stride 256), and whether the tile reaches the four-accumulator body."""
    t = np.arange(OPT_THREADS)
    main = np.where(t + 3 * OPT_THREADS < length, (length - 1 - 3 * OPT_THREADS - t) // (4 * OPT_THREADS) + 1, 0)
    j = t + main * 4 * OPT_THREADS
    tail = np.where(j < length, (length - 1 - j) // OPT_THREADS + 1, 0)
    return int((main + tail).max()), bool(main.max() > 0)


SUMSQ_TREE = 12     # (a0 + a1) + (a2 + a3): 2, warp_sum: 5, the block's second warp_sum: 5


class Layout:
    """Per-element maps of a bucket built from its eb_opt_seg / eb_opt_tile rows: pos (the bucket position of every
    element a tile covers, in tile order), etile, eseg, egroup, and acc_idx [.., 4] (SM3: the accumulator of each
    dimension, -1 where the rank has none)."""

    def __init__(self, seg, tiles, n, device):
        self.seg, self.tiles, self.n, self.device = seg, tiles, n, device
        self.nseg, self.ntiles = len(seg), len(tiles)
        sg = torch.tensor(seg, dtype=i64).reshape(-1, 14).to(device)
        tl = torch.tensor(tiles, dtype=i64).reshape(-1, 6).to(device)
        lens = tl[:, 2]
        first = torch.cumsum(lens, 0) - lens
        total = int(lens.sum())
        self.etile = torch.repeat_interleave(torch.arange(self.ntiles, device=device), lens)
        k = torch.arange(total, device=device)
        self.eseg = tl[self.etile, 0]
        j = tl[self.etile, 1] + k - first[self.etile]            # index within the tensor
        self.pos = sg[self.eseg, 0] + j
        self.egroup = sg[self.eseg, 3]
        rank, shape, acc = sg[self.eseg, 2], sg[self.eseg, 6:10], sg[self.eseg, 10:14]
        self.acc_idx = torch.full((total, 4), -1, dtype=i64, device=device)
        low = rank <= 1
        self.acc_idx[low, 0] = acc[low, 0] + j[low]
        stride = torch.ones_like(j)
        for d in range(3, -1, -1):
            on = (rank > d) & ~low
            idx = (j // stride) % shape[:, d].clamp(min=1)
            self.acc_idx[on, d] = acc[on, d] + idx[on]
            stride = torch.where(on, stride * shape[:, d], stride)
        self.seg_group = sg[:, 3]

    def per_elem(self, h, key):
        return torch.tensor(h[key], dtype=f64, device=self.device)[self.egroup]

    def covered(self):
        m = torch.zeros(self.n, dtype=torch.bool, device=self.device)
        m[self.pos] = True
        return m


def _at(L, x):
    return x.to(f64)[L.pos]


def seg_sumsq(L, g):
    """(per-tile fp64 sum g^2 and its bar, per-segment fp64 sum g^2 and its bar).  A tile: (m + 12) roundings, m the
    accumulator's count of squares (``sumsq_terms``); a segment: its tiles' bars, the fp64 adds (2^-52 each) and the
    final rounding to fp32."""
    sq = _at(L, g) ** 2
    tsum = torch.zeros(L.ntiles, dtype=f64, device=L.device).index_add_(0, L.etile, sq)
    ssum = torch.zeros(L.nseg, dtype=f64, device=L.device).index_add_(0, L.eseg, sq)
    terms = {}
    m = torch.tensor([terms.setdefault(t[2], sumsq_terms(t[2])[0]) for t in L.tiles], dtype=f64, device=L.device)
    tbar = bar(m + SUMSQ_TREE, tsum)
    tseg = torch.tensor([t[0] for t in L.tiles], dtype=i64, device=L.device)
    nt = torch.tensor([s[5] - s[4] for s in L.seg], dtype=f64, device=L.device)
    sbar = torch.zeros(L.nseg, dtype=f64, device=L.device).index_add_(0, tseg, tbar) + bar(1, ssum) + \
        nt * 2.0 ** -52 * ssum
    return tsum, tbar, ssum, sbar


def segsum_in_order(seg, partial):
    """seg_sumsq_reduce_kernel's order, bit for bit: lane l of a warp adds (double) partial[t] for t = tile_begin + l,
    + 32, ... from 0.0, then five xor-butterfly levels 16 ... 1; rounded to fp32.  total: the segsums added in order in
    fp64, rounded to fp32."""
    partial = np.asarray(partial, dtype=np.float32).astype(np.float64)
    lanes = np.arange(32)
    out = np.empty(len(seg), dtype=np.float32)
    for s, row in enumerate(seg):
        a = np.zeros(32)
        for t in range(row[4], row[5]):
            a[(t - row[4]) % 32] += partial[t]
        for o in (16, 8, 4, 2, 1):
            a = a + a[lanes ^ o]
        out[s] = np.float32(a[0])
    tot = 0.0
    for x in out.astype(np.float64):
        tot += x
    return out, np.float32(tot)


def sgd(L, p, g, buf, h, steps, coef, buf_new=None):
    """d = coef g + wd p (4 roundings: coef g, fp32(wd), wd p, the add); buf = d on the group's first step (counter
    <= 1), else mu buf + d (3 more: fp32(mu), the product, the add); p -= lr buf teacher-forced from the kernel's buf
    (3: fp32(lr), the product, the subtraction), or p -= lr d where mu = 0 (4 + 3).  Returns {key: (want, bar)} and
    the mask of elements whose group has momentum."""
    p, g, buf = _at(L, p), _at(L, g), _at(L, buf)
    lr, wd, mu = L.per_elem(h, "lr"), L.per_elem(h, "wd"), L.per_elem(h, "b1")
    first = torch.as_tensor(steps, device=L.device)[L.egroup] <= 1
    gc = g * coef
    d, Md = gc + wd * p, gc.abs() + wd * p.abs()
    b = torch.where(first, d, mu * buf + d)
    Mb = torch.where(first, Md, mu * buf.abs() + Md)
    bn = b if buf_new is None else _at(L, buf_new)
    has_mu = mu != 0
    pw = torch.where(has_mu, p - lr * bn, p - lr * d)
    pbar = torch.where(has_mu, bar(3, p.abs() + lr * bn.abs()), bar(7, p.abs() + lr * Md))
    return {"buf": (b, bar(7, Mb)), "p": (pw, pbar)}, has_mu


def adamw_step_size(h, steps):
    """Per group: lr sqrt(1 - b2^k) / (1 - b1^k) in fp64 from the group's counter k, as the kernel forms it."""
    return [h["lr"][i] * math.sqrt(1.0 - h["b2"][i] ** k) / (1.0 - h["b1"][i] ** k) for i, k in enumerate(steps)]


def adamw(L, p, g, m, v, h, steps, coef, m_new=None, v_new=None):
    """m = b1 m + (1-b1) coef g: 6 roundings (coef g, fp32(b1), fp32(1-b1), two products, the add); v = b2 v +
    (1-b2) (coef g)^2: 8 (coef g counts twice through the square, the square, fp32(b2), fp32(1-b2), two products, the
    add); p -= ss (wd p + m / (sqrt(v) + eps)) teacher-forced from the kernel's m and v, ss the fp64 step size: 10
    (fp32(ss), fp32(wd), wd p, sqrtf, fp32(eps), + eps, the division, the add, ss x, the subtraction)."""
    p, g, m, v = _at(L, p), _at(L, g), _at(L, m), _at(L, v)
    b1, b2, wd, eps = (L.per_elem(h, k) for k in ("b1", "b2", "wd", "eps"))
    ss = torch.tensor(adamw_step_size(h, steps), dtype=f64, device=L.device)[L.egroup]
    gc = g * coef
    mw, Mm = b1 * m + (1 - b1) * gc, b1 * m.abs() + (1 - b1) * gc.abs()
    vw, Mv = b2 * v + (1 - b2) * gc * gc, b2 * v.abs() + (1 - b2) * gc * gc
    mn = mw if m_new is None else _at(L, m_new)
    vn = vw if v_new is None else _at(L, v_new)
    q = mn / (vn.sqrt() + eps)
    pw = p - ss * (wd * p + q)
    Mp = p.abs() + ss * (wd * p.abs() + q.abs())
    return {"m": (mw, bar(6, Mm)), "v": (vw, bar(8, Mv)), "p": (pw, bar(10, Mp))}


def novograd_v(seg, segsum, segv, h, coef):
    """Per tensor: n = coef^2 segsum (2 roundings: coef coef, x segsum); v == 0: n, else b2 v + (1-b2) n (5 more:
    fp32(b2), fp32(1-b2), two products, the add).  segsum, segv: float64 tensors [nseg]."""
    grp = torch.tensor([s[3] for s in seg], dtype=i64, device=segsum.device)
    b2 = torch.tensor(h["b2"], dtype=f64, device=segsum.device)[grp]
    n = coef * coef * segsum
    zero = segv == 0
    want = torch.where(zero, n, b2 * segv + (1 - b2) * n)
    b = torch.where(zero, bar(2, n.abs()), bar(7, b2 * segv.abs() + (1 - b2) * n.abs()))
    return want, b


def novograd(L, p, g, m, segv_new, h, coef, m_new=None):
    """Teacher-forced from the kernel's segv: g' = coef g / (sqrt(v) + eps) + wd p, m = b1 m + g': 11 roundings
    (sqrtf, fp32(eps), + eps, coef g, the division, fp32(wd), wd p, the add, fp32(b1), b1 m, the add); p -= lr m
    teacher-forced from the kernel's m: 3."""
    p, g, m = _at(L, p), _at(L, g), _at(L, m)
    lr, wd, b1, eps = (L.per_elem(h, k) for k in ("lr", "wd", "b1", "eps"))
    denom = segv_new.to(f64)[L.eseg].sqrt() + eps
    gc = g * coef
    gp, Mg = gc / denom + wd * p, gc.abs() / denom + wd * p.abs()
    mw, Mm = b1 * m + gp, b1 * m.abs() + Mg
    mn = mw if m_new is None else _at(L, m_new)
    return {"m": (mw, bar(11, Mm)), "p": (p - lr * mn, bar(3, p.abs() + lr * mn.abs()))}


def sm3(L, p, g, acc, nacc, h, coef):
    """u = min_i acc_i + (coef g)^2: 4 roundings of a sum of non-negative terms (coef g twice through the square, the
    square, the add; with coef = 1 the product is exact and 2 remain); new acc_i = the max of u over every other
    dimension: the selection is exact, so its bar is u's bar at the maximum, and an empty tensor's accumulators stay 0;
    p -= lr coef g / sqrt(u + eps): u's k roundings and two more (fp32(eps), + eps) halve through sqrtf, then sqrtf,
    1 / x, coef g (coef != 1), x gi, fp32(lr), lr x and the subtraction: at most k + 8.
    Returns ({"acc": (want [nacc], bar), "p": (want, bar)}, u)."""
    p, g, acc = _at(L, p), _at(L, g), acc.to(f64)
    lr, eps = L.per_elem(h, "lr"), L.per_elem(h, "eps")
    a = torch.full_like(p, math.inf)
    for d in range(4):
        on = L.acc_idx[:, d] >= 0
        a[on] = torch.minimum(a[on], acc[L.acc_idx[on, d]])
    gc = g * coef
    u = a + gc * gc
    new = torch.zeros(nacc, dtype=f64, device=L.device)
    isnan = torch.zeros(nacc, dtype=f64, device=L.device)
    for d in range(4):
        on = L.acc_idx[:, d] >= 0
        new.scatter_reduce_(0, L.acc_idx[on, d], u[on].nan_to_num(nan=0.0, posinf=math.inf), "amax")
        isnan.scatter_reduce_(0, L.acc_idx[on, d], u[on].isnan().to(f64), "amax")
    new[isnan > 0] = math.nan
    k_acc = 2 if coef == 1.0 else 4
    r = (u + eps).sqrt()
    pw = p - lr * gc / r
    pbar = bar(k_acc + 8, p.abs() + lr * gc.abs() / r)
    return {"acc": (new, bar(k_acc, new)), "p": (pw, pbar)}, u
