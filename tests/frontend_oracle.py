"""fp64 functional restatement of the reference's FrontEnd (rnnt/models.py:313-365) in torch: F.conv1d with padding
k - 1 and the last k - 1 outputs dropped, exact GELU, GroupNorm(1, C) over the whole padded utterance, LayerNorm over
channels.  Runs on the CPU in float64 unless told otherwise.

`forward_and_grads(..., bf16=True)` restates the engine's bf16 mode (functional.FrontEndStack): the same fp64
arithmetic with bf16 roundings where the engine rounds.
  forward   each block's conv operand (the GroupNorm output) and conv weight are rounded to bf16; the bias is added
            unrounded; the first layer, the conv outputs, the statistics and the LayerNorm stay exact.
  backward  the gradient of each block's conv output is rounded to bf16 before it enters the dW and dX products (the
            bf16 dY operand); the bias gradient is taken from the unrounded gradient; dX, the GroupNorm / GELU
            backward and the first layer's dW stay exact.
The roundings are identities in the other direction (a rounded operand passes its gradient through unchanged), so with
`rounding=False` the restatement is, bit for bit, the plain one."""
import torch
import torch.nn.functional as F

EPS = 1e-5


def conv_len(T, k, s):
    return (T + k - 2) // s + 2 - k


def _bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


class _RoundFwd(torch.autograd.Function):
    """Forward: round to bf16 (when on).  Backward: identity."""

    @staticmethod
    def forward(ctx, t, on):
        return _bf16(t) if on else t.clone()

    @staticmethod
    def backward(ctx, g):
        return g, None


class _RoundBwd(torch.autograd.Function):
    """Forward: identity.  Backward: the gradient rounded to bf16 (when on)."""

    @staticmethod
    def forward(ctx, t, on):
        ctx.on = on
        return t.clone()

    @staticmethod
    def backward(ctx, g):
        return (_bf16(g) if ctx.on else g), None


def conv(x, w, b, s, rnd=None):
    """x [B, C_in, T] -> [B, C_out, conv_len(T)] (CausalConv1d / DilatedConvBlock.conv and the trim); the bias is added
    after the product.  rnd (bool): the bf16 roundings of the module docstring, applied when True."""
    k = w.shape[-1]
    if rnd is not None:
        x, w = _RoundFwd.apply(x, rnd), _RoundFwd.apply(w, rnd)
    y = F.conv1d(x, w, None, stride=s, padding=k - 1)[:, :, :-(k - 1)].contiguous()
    if rnd is not None:
        y = _RoundBwd.apply(y, rnd)
    return y if b is None else y + b[:, None]


def block(x, w, b, gn_w, gn_b, s, eps=EPS, rnd=None):
    """DilatedConvBlock.forward: conv(GroupNorm(1, C_in, eps)(GELU(x))), x [B, C_in, T]."""
    return conv(F.group_norm(F.gelu(x), 1, gn_w, gn_b, eps), w, b, s, rnd)


def forward(sd, x, frontend_params, blocks_out=None, rnd=None):
    """FrontEnd.forward on x [B, L]: [B, T, C_last].  sd: name -> tensor (the module's state_dict keys); blocks_out, if
    a list, receives each block's input [B, C, T] (the first conv's output, then every block's); rnd as in block()."""
    y = conv(x[:, None], sd["conv1.weight"], sd.get("conv1.bias"), frontend_params[0][1])
    for i, (_, s, _) in enumerate(frontend_params[1:]):
        if blocks_out is not None:
            blocks_out.append(y)
        p = "encode.%d." % i
        y = block(y, sd[p + "conv.weight"], sd.get(p + "conv.bias"), sd[p + "gn.weight"], sd[p + "gn.bias"], s,
                  rnd=rnd)
    y = y.transpose(1, 2)
    return F.layer_norm(y, (y.shape[-1],), sd["layer_norm.weight"], sd["layer_norm.bias"], EPS)


def forward_and_grads(sd, x, frontend_params, R, dtype=torch.float64, bf16=False, rounding=True):
    """(out, {name: d sum(out * R) / d param}) in `dtype`; bf16: the bf16-mode restatement (rounding=False keeps its
    structure with every rounding an identity)."""
    p = {k: torch.as_tensor(v).to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    x = torch.as_tensor(x).to(dtype)
    out = forward(p, x, frontend_params, rnd=rounding if bf16 else None)
    (out * torch.as_tensor(R).to(dtype)).sum().backward()
    return out.detach(), {k: v.grad for k, v in p.items()}
