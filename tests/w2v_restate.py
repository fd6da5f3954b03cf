"""fp64 restatement of each csrc/w2v.cu kernel, fed the kernel's own fp32 inputs, with the per-element bar of
tests/test_gpu_w2v_fp64.py's error model.  Pinned to tests/wav2vec_oracle.py by tests/test_wav2vec_host.py.

Error model.  The build uses no fast-math: ``+ - * /`` and sqrtf are correctly rounded (at most u = 2^-24 relative),
expf is within 2 ulp and logf within 1 ulp; one ulp is at most 2u relative, so expf is at most 4u and logf at most 2u
relative.  nvcc may contract a*b + c into one fmaf, which only removes a rounding, so every bar counts the roundings
without contraction.  A chain of n adds of terms t_i is off by at most (n - 1) u sum |t_i| (fmaf chains: n u).  The lane
maps fix the chain lengths:

  warp reduction over n elements:  ceil(n / 32) sequential adds per lane, then 5 shuffle adds;
  block_sum (1024 threads):        the per-thread chain, then 5 adds (warp) and 5 adds (across warps);
  the CE loss:                     each warp's chain over its rows (w, w + 32, ...), then 32 ordered adds;
  logits_bwd:                      an fmaf chain of length M per output element, and sc, a chain of M adds.

Per kernel (d = l - max, L = log(a + 1e-7f), all quantities of the fp64 restatement):

  sq_mean     out = S / n, S = sum x^2:         (ceil(n / 1024) + 10 + 2) u S / n   (the chain, the tree, fp32(n), /).
  scale       bit for bit fp32 x * (g * alpha).
  softmax     p = e^d / sum e^d (quant_fwd's p and s; s from the kernel's z = fl(fl(l + g) / tau)): e^d is off by
              (|d| + 4) u (the rounding of d, expf), the sum by (ceil(V/32) + 5 + 4 + max|d|) u, the division by u.
  quant_stats H = sum_v a L (a = psum / N; per term a (4 |L| + 2) u: a, a + 1e-7f, logf, the product; then the
              chain ceil(V/1024) + 10), ppl = sum_g expf(-H_g): each off by (bar_H + 4u) relative, G - 1 adds;
              coef = -e (L + a / (a + 1e-7f)): e (bar_H + 4u) |L + r| + e ((2 |L| + 2) u + 3u r + 2u |L + r|).
  quant_bwd   a = <s, ds>, b = <p, c>: (ceil(V/32) + 6) u sum |.|;  dl = s (ds - a) / tau + (g / N) p (c - b):
              |s| (bar_a + 3u |ds - a|) / tau + |g / N| |p| (bar_b + 4u |c - b|) + u |dl|.
  normalize   n = sqrtf(ss), ss an fmaf chain (ceil(D/32) + 5) u ss: n off by (ceil(D/32) + 5) u / 2 + u relative,
              h = x / max(n, eps) by that and u more.
  logits_fwd  cos = <xh, yh> over the kernel's xh, yh: (ceil(D/32) + 5) u sum |xh yh|; logits = cos / temp: bar_cos /
              |temp| + u |logit|; both -inf where c > 0 and the candidate row equals the positive row in every element
              (the saved cos carries the mask to the backward).
  logits_bwd  A[r, j] = sum of dlogit over the unmasked candidates of row r that are row j (c order): (n_j - 1) u
              sum |g|; AC the same of dlogit * cos: n_j u sum |g cos|.  From the kernel's A, AC, xh, yh, xn, yn:
              dx = (acc - sc u) / c / temp, acc an fmaf chain of M, sc a chain of M adds, u = x / n:
              (M u sum |A yh| + |u| ((M - 1) u sum |AC| + 2u |sc|) + u |acc - sc u|) / (c |temp|) + 2u |dx|.
  ce          lse = mx + logf(se): bar_lse = (ceil(C/32) + 9 + max|d|) u + 2u |log se| + u |lse|;  grad = expf(l - lse)
              - [c = 0]: e (bar_lse + u |l - lse| + 4u) + u |grad|;  loss: the rows' bar_lse + u (lse - l0), then the
              chain (ceil(BM / 32) + 32) u sum of the row losses.

Every bar is multiplied by 1 + 2^-10 for the second-order terms, and k 2^-149 covers a rounding into the subnormal
range.  Integer outputs, selections (argmax, max) and copies have no bar: they are restated bit for bit."""
import math

import numpy as np
import torch

f32, f64 = torch.float32, torch.float64
U = 2.0 ** -24
TINY = 2.0 ** -149
EPS_P = float(np.float32(1e-7))          # the kernel's 1e-7f
SENTINEL = 0x7fffffff


def bar(x):
    """A first-order bound (already in units of u) with the second-order margin and the subnormal floor."""
    return x * (1 + 2.0 ** -10) + 16 * TINY


def ceil_div(a, b):
    return -(-a // b)


# ---- selections: the kernels' lane maps, NaN semantics included --------------------------------------------------
def lane_arg(v, largest=True):
    """The index the kernels' warp argmax (argmin) ends at in lane 0 for each row of v [R, n] (numpy float32): lane l
    scans v[l], v[l + 32], ... keeping the first strict improvement (its first element always), then a xor butterfly
    16 ... 1 takes the partner's pair when it is strictly better, or equal with a smaller index.  Comparisons with NaN
    are false, so a NaN a lane meets first sticks in that lane, and a lane holding NaN never takes its partner's pair
    nor hands its NaN on; without NaN this is the first-index argmax (argmin)."""
    v = np.asarray(v, np.float32)
    R, n = v.shape
    better = (lambda a, b: a > b) if largest else (lambda a, b: a < b)
    mx = np.full((R, 32), -np.inf if largest else np.inf, np.float32)
    k = np.full((R, 32), SENTINEL, np.int64)
    with np.errstate(invalid="ignore"):
        for t in range(ceil_div(n, 32)):
            lanes = np.arange(32)
            idx = lanes + 32 * t
            ok = idx < n
            x = np.where(ok[None], v[:, np.minimum(idx, n - 1)], np.nan)
            take = ok[None] & (better(x, mx) | (k == SENTINEL))
            mx = np.where(take, x, mx)
            k = np.where(take, idx[None], k)
        for o in (16, 8, 4, 2, 1):
            p = np.arange(32) ^ o
            ov, ok = mx[:, p], k[:, p]
            take = better(ov, mx) | ((ov == mx) & (ok < k))
            mx, k = np.where(take, ov, mx), np.where(take, ok, k)
    return torch.from_numpy(k[:, 0].copy())


# ---- sq_mean, scale ---------------------------------------------------------------------------------------------------
def sq_mean(x):
    x = x.to(f64).reshape(-1)
    n = x.numel()
    S = float((x * x).sum())
    return S / n, bar((ceil_div(n, 1024) + 12) * U * S / n)


def scale(x, g, alpha):
    """fp32 x * (g * alpha), alpha as the C ABI receives it (float)."""
    return x * (g.reshape(()) * torch.tensor(alpha, dtype=f32, device=x.device))


# ---- quantizer ---------------------------------------------------------------------------------------------------------
def softmax(z, V):
    """Rows z [R, V] (fp32 values) -> (softmax in fp64, bar) for quant_fwd's warp-per-row softmax."""
    z = z.to(f64)
    d = z - z.max(-1, keepdim=True).values
    e = d.exp()
    S = e.sum(-1, keepdim=True)
    p = e / S
    dmax = d.abs().max(-1, keepdim=True).values
    rel = (d.abs() + 4) + (ceil_div(V, 32) + 9 + dmax) + 1
    return p, bar(rel * U * p)


def noisy_z(logits, noise, tau):
    """The kernel's fp32 z = fl(fl(l + g) / tau), tau as the C ABI receives it (float)."""
    return (logits.float() + noise.float()) / torch.tensor(tau, dtype=f32, device=logits.device)


def quant_fwd(logits, noise, vars, G, tau):
    """logits, noise [N, G*V] fp32 -> dict of the restated outputs: k0 (lane argmax of the logits), p and its bar, and
    with noise: z (fp32), s and its bar from z, k (lane argmax of the fp64 s), the fp64 top-two gap of s."""
    N, GV = logits.shape
    V = GV // G
    l = logits.reshape(N * G, V)
    out = dict(k0=lane_arg(l.cpu().numpy()).to(logits.device).view(N, G))
    out["p"], out["p_bar"] = (t.reshape(N, GV) for t in softmax(l, V))
    if noise is not None:
        z = noisy_z(logits, noise, tau).reshape(N * G, V)
        s, sb = softmax(z, V)
        out["z"], out["s"], out["s_bar"] = z.reshape(N, GV), s.reshape(N, GV), sb.reshape(N, GV)
        top = s.topk(min(2, V), -1)
        out["k"] = top.indices[:, 0].view(N, G)
        gap = top.values[:, 0] - top.values[:, 1] if V > 1 else torch.full_like(top.values[:, 0], math.inf)
        out["gap"] = gap.view(N, G)
        out["gap_bar"] = (sb.max(-1).values * 2).view(N, G)
    return out


def entropy_terms(a, V):
    """a [G, V] (fp64, the exact psum / N or count / N) -> (H [G], bar [G], L) of the kernel's sum_v a log(a + 1e-7f)."""
    L = torch.log(a + EPS_P)
    H = (a * L).sum(-1)
    per = (a * (4 * L.abs() + 2)).sum(-1)
    chain = (ceil_div(V, 1024) + 10) * (a * L).abs().sum(-1)
    return H, bar((per + chain) * U), L


def quant_stats(psum, k0, N, G, V):
    """psum [G*V] fp32, k0 [N*G] -> dict counts (exact), pp, cp, coef (fp64) and their bars."""
    counts = torch.zeros(G, V, dtype=torch.int64, device=psum.device)
    k0 = k0.reshape(N, G).long()
    for g in range(G):
        counts[g] = torch.bincount(k0[:, g], minlength=V)
    a = psum.to(f64).view(G, V) / N
    c = counts.to(f64) / N
    out = dict(counts=counts.reshape(-1))
    Hp, bHp, L = entropy_terms(a, V)
    Hc, bHc, _ = entropy_terms(c, V)
    ep, ec = torch.exp(-Hp), torch.exp(-Hc)
    out["pp"], out["cp"] = ep.sum(), ec.sum()
    out["pp_bar"] = bar((ep * (bHp / U + 4)).sum() * U + (G - 1) * U * ep.sum())
    out["cp_bar"] = bar((ec * (bHc / U + 4)).sum() * U + (G - 1) * U * ec.sum())
    r = a / (a + EPS_P)
    coef = -ep[:, None] * (L + r)
    eH = bHp[:, None] + 4 * U
    out["coef"] = coef.reshape(-1)
    out["coef_bar"] = bar(ep[:, None] * (eH * (L + r).abs() + U * (2 * L.abs() + 2 + 3 * r + 2 * (L + r).abs()))).reshape(-1)
    return out


def quant_bwd(dsoft, s, p, coef, g_ppl, N, G, V, tau):
    """-> (dl [N, G*V] fp64, bar).  dsoft or g_ppl may be None (that term is dropped); tau and g_ppl / N as the kernel
    forms them (fp32 tau; g / N is one rounding, in the bar)."""
    ref = dsoft if dsoft is not None else p
    dev = ref.device
    tau = float(np.float32(tau))
    m = ceil_div(V, 32) + 6
    dl = torch.zeros(N * G, V, dtype=f64, device=dev)
    b_ = torch.zeros_like(dl)
    if dsoft is not None:
        sv, dv = s.to(f64).view(N * G, V), dsoft.to(f64).view(N * G, V)
        a = (sv * dv).sum(-1, keepdim=True)
        ba = m * U * (sv * dv).abs().sum(-1, keepdim=True)
        t1 = sv * (dv - a) / tau
        dl = dl + t1
        b_ = b_ + sv.abs() * (ba + 3 * U * (dv - a).abs()) / tau
    if g_ppl is not None:
        gp = float(g_ppl.reshape(-1)[0]) / N
        pv = p.to(f64).view(N * G, V)
        cv = coef.to(f64).view(G, V).repeat(N, 1)
        b = (pv * cv).sum(-1, keepdim=True)
        bb = m * U * (pv * cv).abs().sum(-1, keepdim=True)
        t2 = gp * (pv * (cv - b))
        dl = dl + t2
        b_ = b_ + abs(gp) * pv.abs() * (bb + 4 * U * (cv - b).abs())
    b_ = b_ + U * dl.abs()
    return dl.view(N, G * V), bar(b_).view(N, G * V)


# ---- cosine logits -----------------------------------------------------------------------------------------------------
def normalize(x, eps):
    """Rows x [..., D] fp32 -> (h, h bar, n, n bar) with h = x / max(n, eps), n = |x|, eps as the kernel's float."""
    eps = float(np.float32(eps))
    x = x.to(f64)
    D = x.shape[-1]
    ss = (x * x).sum(-1)
    n = ss.sqrt()
    nrel = (ceil_div(D, 32) + 5) * U / 2 + U
    c = n.clamp_min(eps)
    h = x / c[..., None]
    return h, bar((nrel + U) * h.abs()), n, bar(nrel * n)


def same_rows(y, neg):
    """[K+1, B, M] bool: candidate c > 0 equals the positive row in every element (float ==, as the kernel compares)."""
    B, M, D = y.shape
    K = neg.shape[-1]
    out = torch.zeros(K + 1, B, M, dtype=torch.bool, device=y.device)
    for b in range(B):
        cand = y[b][neg[b].long().reshape(-1)].view(M, K, D)
        out[1:, b] = (cand == y[b][:, None]).all(-1).T
    return out


def logits_fwd(xh, yh, y, neg, temp):
    """From the kernel's xh, yh (and the raw y for the equality test) -> (cos, cos bar, logits, logits bar), all
    [K+1, B, M]; cos and logits are -inf where masked."""
    B, M, D = xh.shape
    K = neg.shape[-1]
    temp = float(np.float32(temp))
    X, Y = xh.to(f64), yh.to(f64)
    rows = torch.cat([torch.arange(M, device=neg.device).view(1, M, 1).expand(B, M, 1), neg.long()], -1)   # [B, M, K+1]
    cand = torch.stack([Y[b][rows[b]] for b in range(B)])                                   # [B, M, K+1, D]
    prod = X[:, :, None] * cand
    cos = prod.sum(-1).permute(2, 0, 1)
    cb = bar((ceil_div(D, 32) + 5) * U * prod.abs().sum(-1).permute(2, 0, 1))
    lo = cos / temp
    lb = bar(cb / abs(temp) + U * lo.abs())
    masked = same_rows(y, neg)
    lo = torch.where(masked, torch.full_like(lo, -math.inf), lo)
    cos = torch.where(masked, torch.full_like(cos, -math.inf), cos)
    return cos, cb, lo, lb


def logits_a(dlog, cosv, neg, masked):
    """dlog, cosv [K+1, B, M] fp32, masked [K+1, B, M] -> (A, A bar, AC, AC bar) [B, M, M]: the unmasked candidates'
    dlogit (and dlogit * cos) summed per row they are."""
    K1, B, M = dlog.shape
    dev = dlog.device
    zero = torch.zeros_like(dlog, dtype=f64)
    g = torch.where(masked, zero, dlog.to(f64)).permute(1, 2, 0)                             # [B, M, K+1]
    gc = g * torch.where(masked, zero, cosv.to(f64)).permute(1, 2, 0)
    rows = torch.cat([torch.arange(M, device=dev).view(1, M, 1).expand(B, M, 1), neg.long()], -1)
    live = (~masked).permute(1, 2, 0).to(f64)
    z = torch.zeros(B, M, M, dtype=f64, device=dev)
    A = z.clone().scatter_add_(2, rows, g)
    AC = z.clone().scatter_add_(2, rows, gc)
    cnt = z.clone().scatter_add_(2, rows, live)
    sa = z.clone().scatter_add_(2, rows, g.abs())
    sac = z.clone().scatter_add_(2, rows, gc.abs())
    return A, bar((cnt - 1).clamp_min(0) * U * sa), AC, bar(cnt * U * sac)


def logits_bwd(A, AC, xh, yh, x, y, xn, yn, temp, eps):
    """From the kernel's A, AC, xh, yh, xn, yn and the raw rows -> (dx, dx bar, dy, dy bar) [B, M, D]."""
    B, M, D = x.shape
    temp, eps = float(np.float32(temp)), float(np.float32(eps))
    A, AC = A.to(f64), AC.to(f64)

    def side(W, WC, other, self_, n):
        n = n.to(f64)[..., None]
        acc = W @ other.to(f64)
        sacc = W.abs() @ other.to(f64).abs()
        sc = WC.sum(-1, keepdim=True)
        ssc = WC.abs().sum(-1, keepdim=True)
        u = torch.where(n > 0, self_.to(f64) / torch.where(n > 0, n, torch.ones_like(n)), torch.zeros_like(n))
        c = n.clamp_min(eps)
        diff = acc - sc * u
        out = diff / c / temp
        b = (M * U * sacc + u.abs() * ((M - 1) * U * ssc + 2 * U * sc.abs()) + U * diff.abs()) / (c * abs(temp))
        return out, bar(b + 2 * U * out.abs())

    dx, bx = side(A, AC, yh, x, xn)
    dy, by = side(A.transpose(1, 2), AC.transpose(1, 2), xh, y, yn)
    return dx, bx, dy, by


# ---- InfoNCE cross-entropy -------------------------------------------------------------------------------------------
def ce(logits):
    """logits [C, B, M] fp32 -> dict grad, grad bar [C, B, M], loss, loss bar, correct (the restated rule on the same
    fp32 logits: lane argmax 0 and lane argmin not 0)."""
    C, B, M = logits.shape
    rows32 = logits.permute(2, 1, 0).reshape(B * M, C)          # row i = m * B + b
    rows = rows32.to(f64)
    mx = rows.max(-1, keepdim=True).values
    d = rows - mx
    se = d.exp().sum(-1, keepdim=True)
    dmax = torch.where(torch.isfinite(d), d.abs(), torch.zeros_like(d)).max(-1, keepdim=True).values
    lse = mx + se.log()
    blse = (ceil_div(C, 32) + 9 + dmax) * U + 2 * U * se.log().abs() + U * lse.abs()
    e = (rows - lse).exp()
    onehot = torch.zeros_like(rows)
    onehot[:, 0] = 1
    grad = e - onehot
    diff = torch.where(torch.isfinite(rows), (rows - lse).abs(), torch.zeros_like(rows))
    gb = bar(e * (blse + U * diff + 4 * U) + U * grad.abs())
    rl = (lse - rows[:, :1])[:, 0]
    R = ceil_div(B * M, 32)
    loss = rl.sum()
    lb = bar((blse[:, 0] + U * rl.abs()).sum() + (R + 32) * U * rl.abs().sum())
    r32 = rows32.cpu().numpy()
    kx, kn = lane_arg(r32, True), lane_arg(r32, False)
    correct = int(((kx == 0) & (kn != 0)).sum())

    def back(t):
        return t.view(M, B, C).permute(2, 1, 0)
    return dict(grad=back(grad), grad_bar=back(gb), loss=float(loss), loss_bar=float(lb), correct=correct)
