"""fp64 CPU statement of the depthwise 1-D convolution and its three gradients, written as the explicit sums.

    y[b, d, l]  = bias[d] + sum_{k<K} w[d, k] * u[b, d, l - P + k]        (u = 0 outside [0, L)),  0 <= l < Lout
    du[b, d, i] = sum_{k<K} w[d, k] * dout[b, d, i + P - k]                (dout = 0 outside [0, Lout)),  0 <= i < L
    dw[d, k]    = sum_{b, l} dout[b, d, l] * u[b, d, l - P + k]
    dbias[d]    = sum_{b, l} dout[b, d, l]

with Lout = L + 2P - K + 1: torch.nn.Conv1d(D, D, K, groups=D, padding=P).  Layouts as in FlashDepthWiseConv1d: BHL takes
u (B, D, L) and w (D, K), BLH takes u (B, L, D) and w (K, D); results come back in the caller's layouts.
"""
import torch


def _to_bhl(u, w, is_bhl):
    u = u.detach().to(torch.float64)
    w = w.detach().to(torch.float64)
    return (u, w) if is_bhl else (u.transpose(1, 2), w.t())


def _from_bhl(x, is_bhl):
    return x if is_bhl else x.transpose(1, 2).contiguous()


def dw_forward(u, w, bias, padding, is_bhl=True):
    """y in float64, in the input's layout."""
    u, w = _to_bhl(u, w, is_bhl)
    K, P, L = w.shape[1], padding, u.shape[-1]
    Lout = L + 2 * P - K + 1
    up = torch.nn.functional.pad(u, (P, P))                        # up[..., j] = u[..., j - P]
    y = bias.detach().to(torch.float64)[None, :, None].expand(u.shape[0], -1, Lout).clone()
    for k in range(K):
        y += w[:, k, None] * up[..., k:k + Lout]
    return _from_bhl(y, is_bhl)


def dw_grads(dout, u, w, padding, is_bhl=True):
    """(du, dw, dbias) in float64: du in the input's layout, dw in the weight's layout."""
    u, w = _to_bhl(u, w, is_bhl)
    dout = dout.detach().to(torch.float64)
    dout = dout if is_bhl else dout.transpose(1, 2)
    K, P, L = w.shape[1], padding, u.shape[-1]
    Lout = dout.shape[-1]
    dp = torch.nn.functional.pad(dout, (K - 1 - P, K - 1 - P))     # dp[..., j] = dout[..., j - (K - 1 - P)]
    du = torch.zeros_like(u)
    for k in range(K):
        du += w[:, k, None] * dp[..., K - 1 - k:K - 1 - k + L]
    up = torch.nn.functional.pad(u, (P, P))
    dw = torch.stack([(dout * up[..., k:k + Lout]).sum(dim=(0, 2)) for k in range(K)], dim=1)   # (D, K)
    dbias = dout.sum(dim=(0, 2))
    return _from_bhl(du, is_bhl), (dw if is_bhl else dw.t().contiguous()), dbias
