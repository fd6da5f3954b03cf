"""fp64 restatement of the four flat-bucket optimizers' update rules (edgedict_b200.optim), written from their semantics:

* SGD (torch.optim.SGD, dampening 0): d = g + wd p; buf = d on the first step, mu buf + d after it; p -= lr buf.
* SM3 (beta = momentum = 0): per dimension i an accumulator acc_i broadcast along every other dimension (rank 0 and 1:
  one of the tensor's shape); u = min_i acc_i + g^2; acc_i = max of u over every other dimension;
  p -= lr g / sqrt(u + eps).
* AdamW: m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2, p -= lr sqrt(1-b2^t)/(1-b1^t) (wd p + m / (sqrt(v) + eps)).
* Novograd: per tensor n = sum g^2, v = n if v == 0 else b2 v + (1-b2) n; g' = g / (sqrt(v) + eps) + wd p,
  m = b1 m + g', p -= lr m.

g is the scaled gradient: grad_scale g, times clip_grad_norm_'s max_norm / (norm + 1e-6) when that is below 1 (the norm
over every tensor).  Every parameter takes every step (no None gradients).  State keys are the reference classes'.
"""
import math

import numpy as np


def _coef(grads, grad_scale, max_norm):
    c = grad_scale
    if max_norm:
        norm = math.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in grads)) * abs(grad_scale)
        k = max_norm / (norm + 1e-6)
        if k < 1:
            c *= k
    return c


def _max_except(u, d):
    axes = tuple(a for a in range(u.ndim) if a != d)
    return u.max(axis=axes, keepdims=True) if axes else u.copy()


def run(kind, params, grad_steps, groups, grad_scale=1.0, max_norm=None, state=None, t0=0):
    """params: list of arrays; grad_steps: list of (grads, [per-group hyper dict]); groups: group index per parameter.
    Hyper dict keys: lr, wd, b1, b2, eps.  Returns (params, state) after every step, state {i: {key: value}}."""
    p = [np.asarray(x, dtype=np.float64).copy() for x in params]
    st = {i: {k: (np.asarray(v, dtype=np.float64).copy() if not isinstance(v, (int, float)) else v)
              for k, v in s.items()} for i, s in (state or {}).items()}
    out = []
    t = t0
    for grads, hyper in grad_steps:
        t += 1
        c = _coef(grads, grad_scale, max_norm)
        for i, (x, g0) in enumerate(zip(p, grads)):
            h = hyper[groups[i]]
            g = np.asarray(g0, dtype=np.float64) * c
            s = st.setdefault(i, {})
            if kind == "sgd":
                d = g + h["wd"] * x
                if h["b1"] != 0:
                    d = d.copy() if "momentum_buffer" not in s else h["b1"] * s["momentum_buffer"] + d
                    s["momentum_buffer"] = d
                p[i] = x - h["lr"] * d
            elif kind == "sm3":
                r = x.ndim
                if r <= 1:
                    u = s.get("accumulator_0", np.zeros(x.shape)) + g * g
                    s["accumulator_0"] = u.copy()
                else:
                    a = np.full(x.shape, np.inf)
                    for d in range(r):
                        a = np.minimum(a, s.get("accumulator_%d" % d, np.zeros([1] * d + [x.shape[d]] +
                                                                            [1] * (r - 1 - d))))
                    u = a + g * g
                    for d in range(r):
                        s["accumulator_%d" % d] = _max_except(u, d)
                s["step"], s["momentum_buffer"] = t, 0.
                p[i] = x - h["lr"] * g / np.sqrt(u + h["eps"])
            elif kind == "adamw":
                m = h["b1"] * s.get("exp_avg", 0.0) + (1 - h["b1"]) * g
                v = h["b2"] * s.get("exp_avg_sq", 0.0) + (1 - h["b2"]) * g * g
                s["exp_avg"], s["exp_avg_sq"], s["step"] = m, v, t
                step_size = h["lr"] * math.sqrt(1 - h["b2"] ** t) / (1 - h["b1"] ** t)
                p[i] = x - step_size * (h["wd"] * x + m / (np.sqrt(v) + h["eps"]))
            elif kind == "novograd":
                n = float((g * g).sum())
                v = float(s.get("exp_avg_sq", 0.0))
                v = n if v == 0 else h["b2"] * v + (1 - h["b2"]) * n
                gp = g / (math.sqrt(v) + h["eps"]) + h["wd"] * x
                m = h["b1"] * s.get("exp_avg", 0.0) + gp
                s["exp_avg"], s["exp_avg_sq"], s["step"] = m, np.float64(v), t
                p[i] = x - h["lr"] * m
            else:
                raise ValueError(kind)
        out.append(([x.copy() for x in p], {i: dict(s) for i, s in st.items()}))
    return out


# ---- the cases of tests/golden/optim_tiny.npz (tests/golden/make_golden_optim.py) --------------------------------------
KIND = {"sgd": "sgd", "sm3": "sm3", "adamw": "adamw", "adamw2": "adamw", "novograd": "novograd"}
HYPER = {   # case -> the engine class name, its constructor kwargs, and the oracle's per-group hyperparameters
    "sgd": ("SGD", dict(momentum=0.9, weight_decay=1e-2), dict(wd=1e-2, b1=0.9, b2=0.0, eps=0.0)),
    "sm3": ("SM3", dict(), dict(wd=0.0, b1=0.0, b2=0.0, eps=1e-30)),
    "adamw": ("AdamW", dict(weight_decay=1e-2), dict(wd=1e-2, b1=0.9, b2=0.999, eps=1e-8)),
    "adamw2": ("AdamW", dict(weight_decay=5e-2), dict(wd=5e-2, b1=0.9, b2=0.999, eps=1e-8)),
    "novograd": ("Novograd", dict(weight_decay=1e-3), dict(wd=1e-3, b1=0.95, b2=0.0, eps=1e-8)),
}
NSTEPS, LR_CHANGE = 6, 3


def fixture(z, case):
    """(init params, grads per step, group index per parameter, [per-group hyper] per step, two groups) of a case."""
    n = len(z["shapes"])
    init = [z["init.%d" % i] for i in range(n)]
    grads = [[z["grad.%d.%d" % (s, i)] for i in range(n)] for s in range(1, NSTEPS + 1)]
    two = case == "adamw2"
    groups = [0 if (two and init[i].ndim >= 2) else (1 if two else 0) for i in range(n)]
    base = HYPER[case][2]
    lr1, lr2 = (float(x) for x in z["%s.lr" % case])
    hyp = []
    for s in range(1, NSTEPS + 1):
        lr = lr1 if s <= LR_CHANGE else lr2
        hs = [dict(base, lr=lr)]
        if two:
            hs.append(dict(base, lr=lr, wd=0.0))
        hyp.append(hs)
    return init, grads, groups, hyp, two


def fixture_state(z, case, step, i):
    pre = "%s.s.%d.%d." % (case, step, i)
    return {k[len(pre):]: z[k] for k in z.files if k.startswith(pre)}
