"""fp64 torch restatement of the wav2vec pre-training head (rnnt/wav2vec.py:264-528 and
modules/softmax_vector_quantizer.py:140-201): the masked-row gathers, the Gumbel quantizer given its noise, the cosine
logits given the negatives, the InfoNCE cross-entropy, the penalties and the logging values.  Gradients come from torch
autograd in fp64.  Pinned to the reference by tests/test_wav2vec_host.py (tests/golden/wav2vec_tiny.npz)."""
import torch

f64 = torch.float64


def frames(mask):
    """[B, T] bool mask (same count per row) -> idx [B, M] int64, ascending (the order of x[mask])."""
    mask = torch.as_tensor(mask)
    B = mask.shape[0]
    return torch.nonzero(mask)[:, 1].view(B, -1)


def gather(x, idx):
    return torch.stack([x[b, idx[b]] for b in range(x.shape[0])])


def quantize(logits, vars, noise, G, tau):
    """logits [N, G*V], vars [G*V, vd], noise [N, G*V] (None: eval) -> (q [N, G*vd], prob_ppl, code_ppl, k [N, G],
    st [N, G] or None).  st is the fp32 straight-through value (1 - s_k) + s_k of the fp32 soft probabilities; q uses it,
    as the reference's forward does."""
    N, GV = logits.shape
    V = GV // G
    l = logits.view(N, G, V)
    k0 = l.argmax(-1)
    hard = torch.zeros_like(l).scatter_(-1, k0[..., None], 1.0)
    hp = hard.mean(0)
    cp = torch.exp(-(hp * torch.log(hp + 1e-7)).sum(-1)).sum()
    avg = torch.softmax(l, -1).mean(0)
    pp = torch.exp(-(avg * torch.log(avg + 1e-7)).sum(-1)).sum()
    vg = vars.view(G, V, -1)
    if noise is None:
        q = torch.einsum("ngv,gvd->ngd", hard, vg)
        return q.reshape(N, -1), pp, cp, k0, None
    s = torch.softmax((l + noise.view(N, G, V)) / tau, -1)
    k = s.argmax(-1)
    s32 = s.detach().float()
    sk = s32.gather(-1, k[..., None])[..., 0]
    st = ((1 - sk) + sk).to(f64)
    onehot = torch.zeros_like(s).scatter_(-1, k[..., None], 1.0)
    # straight-through: forward value st at k (0 elsewhere), gradient of s
    X = onehot * st[..., None] + (s - s.detach())
    q = torch.einsum("ngv,gvd->ngd", X, vg)
    return q.reshape(N, -1), pp, cp, k, st


def contrastive_logits(xp, yp, neg, temp, eps=1e-8):
    """xp, yp [B, M, D], neg [B, M, K] -> logits [K+1, B, M] with torch.cosine_similarity's semantics (each row over
    max(|row|, eps), the clamp invisible to autograd) and -inf where a negative equals the positive."""
    B, M, D = xp.shape
    K = neg.shape[-1]
    negs = torch.stack([yp[b, neg[b].reshape(-1)].view(M, K, D) for b in range(B)]).permute(2, 0, 1, 3)
    cand = torch.cat([yp[None], negs], 0)

    def unit(v):
        n = torch.linalg.vector_norm(v, dim=-1, keepdim=True)
        return v / (n.detach().clamp_min(eps) + (n - n.detach()))       # the clamped value, the norm's gradient

    cos = (unit(xp)[None] * unit(cand)).sum(-1)
    logits = cos / temp
    same = (yp[None] == negs).all(-1)
    return torch.where(torch.cat([torch.zeros_like(same[:1]), same], 0), torch.full_like(logits, -float("inf")), logits)


def cross_entropy(logits):
    """logits [K+1, B, M] -> (summed InfoNCE loss over rows (m, b), correct count)."""
    rows = logits.transpose(0, 2).reshape(-1, logits.shape[0])
    loss = torch.nn.functional.cross_entropy(rows, torch.zeros(rows.shape[0], dtype=torch.long), reduction="sum")
    mx, mn = rows.argmax(-1) == 0, rows.argmin(-1) == 0
    return loss, int(mx.sum() - (mx & mn).sum())


def head(sd, y, xenc, fpen, neg, noise, G, tau, temp, weights):
    """The cli configuration's head (quantize_targets, embed == input_size): sd the state_dict (fp64 tensors, requires_grad
    where gradients are wanted), y the front end's output and xenc the encoder's output at the masked frames [B, M, C]
    and [B, M, P] (``gather(x, frames(mask))``), fpen the features penalty -> (logits, loss, logging values {loss,
    loss_0, loss_1, loss_2, correct, prob_perplexity, code_perplexity})."""
    B, M = y.shape[0], y.shape[1]
    lq = y.reshape(B * M, -1) @ sd["quantizer.weight_proj.weight"].T + sd["quantizer.weight_proj.bias"]
    vars = sd["quantizer.vars"][0]
    q, pp, cp, _, _ = quantize(lq, vars, noise, G, tau)
    yp = (q @ sd["project_q.weight"].T + sd["project_q.bias"]).view(B, M, -1)
    xp = xenc @ sd["final_proj.weight"].T + sd["final_proj.bias"]
    logits = contrastive_logits(xp, yp, torch.as_tensor(neg).view(B, M, -1), temp)
    ce, correct = cross_entropy(logits)
    n = B * M
    num_vars = vars.shape[0]
    p1 = weights[0] * ((num_vars - pp) / num_vars) * n
    p2 = weights[1] * fpen * n
    loss = ce + p1 + p2
    return logits, loss, dict(loss=loss, loss_0=ce, loss_1=p1, loss_2=p2, correct=correct, prob_perplexity=pp,
                              code_perplexity=cp)
