"""fp64 numpy restatement of one training step of the reference's LMModel (models.py:224-261, dropout off) under
cli/train_lm.py's nn.NLLLoss(ignore_index): the forward pass, the loss and the gradient of every parameter by hand-written
backpropagation.  The oracle of tests/test_lm_host.py (against the reference's own gradients, lm_train_tiny.npz) and of
tests/test_gpu_lm.py (against the engine at tensor-core shapes)."""
import numpy as np


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def _layers(sd):
    L = 0
    while "rnn.weight_ih_l%d" % L in sd:
        L += 1
    return L


def forward(sd, inputs, hidden=None):
    """sd: {key: array} (a state_dict), inputs [B, S] ints, hidden (h0, c0) [L, B, H] or None -> (log-probs [B*S, V],
    (h, c) [L, B, H], cache for ``backward``)."""
    sd = {k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}
    inputs = np.asarray(inputs, dtype=np.int64)
    B, S = inputs.shape
    L = _layers(sd)
    H = sd["rnn.weight_hh_l0"].shape[1]
    x = sd["encoder.weight"][inputs]
    cache = dict(sd=sd, inputs=inputs, xs=[], hs=[], cs=[], gates=[])
    hT, cT = [], []
    for k in range(L):
        wih, whh = sd["rnn.weight_ih_l%d" % k], sd["rnn.weight_hh_l%d" % k]
        b = sd["rnn.bias_ih_l%d" % k] + sd["rnn.bias_hh_l%d" % k]
        h = np.zeros((B, H)) if hidden is None else np.asarray(hidden[0][k], dtype=np.float64)
        c = np.zeros((B, H)) if hidden is None else np.asarray(hidden[1][k], dtype=np.float64)
        hs, cs, gs = [h], [c], []
        for t in range(S):
            z = x[:, t] @ wih.T + h @ whh.T + b
            i, f, g, o = _sig(z[:, :H]), _sig(z[:, H:2 * H]), np.tanh(z[:, 2 * H:3 * H]), _sig(z[:, 3 * H:])
            c = f * c + i * g
            h = o * np.tanh(c)
            hs.append(h)
            cs.append(c)
            gs.append((i, f, g, o))
        cache["xs"].append(x)
        cache["hs"].append(hs)
        cache["cs"].append(cs)
        cache["gates"].append(gs)
        x = np.stack(hs[1:], 1)
        hT.append(h)
        cT.append(c)
    y = x.reshape(B * S, H)
    logits = y @ sd["decoder.weight"].T + sd["decoder.bias"]
    m = logits.max(1, keepdims=True)
    lse = m + np.log(np.exp(logits - m).sum(1, keepdims=True))
    cache["y"] = y
    cache["logp"] = logits - lse
    return logits - lse, (np.stack(hT), np.stack(cT)), cache


def nll(logp, targets, ignore_index=0, reduction="mean"):
    """nn.NLLLoss on fp64 log-probs; out-of-range targets are not handled (torch raises)."""
    t = np.asarray(targets, dtype=np.int64).reshape(-1)
    keep = t != ignore_index
    cost = np.where(keep, -logp[np.arange(len(t)), np.where(keep, t, 0)], 0.0)
    if reduction == "none":
        return cost
    return cost.sum() / keep.sum() if reduction == "mean" else cost.sum()


def loss_and_grads(sd, inputs, targets, ignore_index=0, tied=False):
    """(mean NLL, {parameter name: gradient}) of one step; with ``tied`` the decoder's weight is the embedding and its
    gradient is the sum of both uses, under ``encoder.weight`` (named_parameters of a tied LMModel)."""
    logp, _, cache = forward(sd, inputs)
    sd = cache["sd"]
    t = np.asarray(targets, dtype=np.int64).reshape(-1)
    keep = t != ignore_index
    n = keep.sum()
    loss = nll(logp, t, ignore_index)
    dlog = np.exp(logp)
    dlog[np.arange(len(t)), np.where(keep, t, 0)] -= 1.0
    dlog *= keep[:, None] / n
    grads = {"decoder.weight": dlog.T @ cache["y"], "decoder.bias": dlog.sum(0)}
    B, S = cache["inputs"].shape
    dx = (dlog @ sd["decoder.weight"]).reshape(B, S, -1)
    L = _layers(sd)
    H = sd["rnn.weight_hh_l0"].shape[1]
    for k in range(L - 1, -1, -1):
        wih, whh = sd["rnn.weight_ih_l%d" % k], sd["rnn.weight_hh_l%d" % k]
        x, hs, cs, gs = cache["xs"][k], cache["hs"][k], cache["cs"][k], cache["gates"][k]
        dwih, dwhh, db = np.zeros_like(wih), np.zeros_like(whh), np.zeros(4 * H)
        dxin = np.zeros_like(x)
        dh, dc = np.zeros((B, H)), np.zeros((B, H))
        for s in range(S - 1, -1, -1):
            i, f, g, o = gs[s]
            dh = dh + dx[:, s]
            tc = np.tanh(cs[s + 1])
            do = dh * tc
            dc = dc + dh * o * (1 - tc * tc)
            dz = np.concatenate([dc * g * i * (1 - i), dc * cs[s] * f * (1 - f), dc * i * (1 - g * g),
                                 do * o * (1 - o)], 1)
            dwih += dz.T @ x[:, s]
            dwhh += dz.T @ hs[s]
            db += dz.sum(0)
            dxin[:, s] = dz @ wih
            dh = dz @ whh
            dc = dc * f
        grads.update({"rnn.weight_ih_l%d" % k: dwih, "rnn.weight_hh_l%d" % k: dwhh, "rnn.bias_ih_l%d" % k: db,
                      "rnn.bias_hh_l%d" % k: db.copy()})
        dx = dxin
    demb = np.zeros_like(sd["encoder.weight"])
    np.add.at(demb, cache["inputs"].reshape(-1), dx.reshape(B * S, -1))
    grads["encoder.weight"] = demb
    if tied:
        grads["encoder.weight"] = demb + grads.pop("decoder.weight")
    return loss, grads
