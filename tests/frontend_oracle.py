"""fp64 functional restatement of the reference's FrontEnd (rnnt/models.py:313-365) in torch: F.conv1d with padding
k - 1 and the last k - 1 outputs dropped, exact GELU, GroupNorm(1, C) over the whole padded utterance, LayerNorm over
channels.  Runs on the CPU in float64 unless told otherwise."""
import torch
import torch.nn.functional as F

EPS = 1e-5


def conv_len(T, k, s):
    return (T + k - 2) // s + 2 - k


def conv(x, w, b, s):
    """x [B, C_in, T] -> [B, C_out, conv_len(T)] (CausalConv1d / DilatedConvBlock.conv and the trim)."""
    k = w.shape[-1]
    return F.conv1d(x, w, b, stride=s, padding=k - 1)[:, :, :-(k - 1)]


def block(x, w, b, gn_w, gn_b, s, eps=EPS):
    """DilatedConvBlock.forward: conv(GroupNorm(1, C_in, eps)(GELU(x))), x [B, C_in, T]."""
    return conv(F.group_norm(F.gelu(x), 1, gn_w, gn_b, eps), w, b, s)


def forward(sd, x, frontend_params, blocks_out=None):
    """FrontEnd.forward on x [B, L]: [B, T, C_last].  sd: name -> tensor (the module's state_dict keys); blocks_out, if
    a list, receives each block's input [B, C, T] (the first conv's output, then every block's)."""
    y = conv(x[:, None], sd["conv1.weight"], sd.get("conv1.bias"), frontend_params[0][1])
    for i, (_, s, _) in enumerate(frontend_params[1:]):
        if blocks_out is not None:
            blocks_out.append(y)
        p = "encode.%d." % i
        y = block(y, sd[p + "conv.weight"], sd.get(p + "conv.bias"), sd[p + "gn.weight"], sd[p + "gn.bias"], s)
    y = y.transpose(1, 2)
    return F.layer_norm(y, (y.shape[-1],), sd["layer_norm.weight"], sd["layer_norm.bias"], EPS)


def forward_and_grads(sd, x, frontend_params, R, dtype=torch.float64):
    """(out, {name: d sum(out * R) / d param}) in `dtype`."""
    p = {k: torch.as_tensor(v).to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    x = torch.as_tensor(x).to(dtype)
    out = forward(p, x, frontend_params)
    (out * torch.as_tensor(R).to(dtype)).sum().backward()
    return out.detach(), {k: v.grad for k, v in p.items()}
