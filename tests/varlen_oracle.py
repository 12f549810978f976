"""Packed documents for the tests: seeded cu_seqlens tables and the fp64 per-document statement of the depthwise
convolution (FlashDepthWiseConv1d.forward(u, cu_seqlens)).

A document [o, e) of row b is convolved alone: its output is the first e - o outputs of the plain convolution run on
u[b, :, o:e], and its gradients are those of that output, i.e. of the plain convolution with dout zero past e - o."""
import numpy as np
import torch

from oracle.dwconv_oracle import dw_forward, dw_grads


def make_cu(B, L, seed, lengths=(0, 1, 2, 5, 63, 64, 65, 127, 300, 1000)):
    """int32 offsets (CPU) of rows of length L cut into documents drawn from `lengths` (and at seeded random lengths);
    every row start is an offset, the last document of a row takes what is left."""
    rng = np.random.default_rng(seed)
    cu = [0]
    for b in range(B):
        t = 0
        while t < L:
            n = int(rng.choice(lengths)) if rng.random() < 0.7 else int(rng.integers(1, L + 1))
            n = min(n, L - t)
            cu.append(b * L + t + n)
            t += n
    return torch.tensor(cu, dtype=torch.int32)


def row_docs(cu, L):
    """(b, o, e) of every non-empty document, [o, e) inside row b."""
    c = [int(x) for x in cu]
    return [(s // L, s % L, t - (s // L) * L) for s, t in zip(c[:-1], c[1:]) if t > s]


def _slice(x, b, o, e, is_bhl):
    return x[b:b + 1, :, o:e] if is_bhl else x[b:b + 1, o:e, :]


def dw_forward_docs(u, w, bias, P, cu, is_bhl=True):
    """y (float64, u's layout and shape): each document through dw_forward alone."""
    L = u.shape[-1] if is_bhl else u.shape[1]
    y = torch.zeros(u.shape, dtype=torch.float64)
    for b, o, e in row_docs(cu, L):
        if e > o:
            yd = dw_forward(_slice(u, b, o, e, is_bhl), w, bias, P, is_bhl)
            _slice(y, b, o, e, is_bhl).copy_(_slice(yd, 0, 0, e - o, is_bhl))
    return y


def dw_grads_docs(dout, u, w, P, cu, is_bhl=True):
    """(du, dw, dbias) in float64: each document through dw_grads alone with dout zero past its length; dw and dbias
    summed over the documents."""
    L = u.shape[-1] if is_bhl else u.shape[1]
    K = w.shape[1] if is_bhl else w.shape[0]
    du = torch.zeros(u.shape, dtype=torch.float64)
    dw = torch.zeros(w.shape, dtype=torch.float64)
    db = torch.zeros(w.shape[0] if is_bhl else w.shape[1], dtype=torch.float64)
    for b, o, e in row_docs(cu, L):
        if e == o:
            continue
        n = e - o
        Lout = n + 2 * P - K + 1
        dd = _slice(dout, b, o, e, is_bhl).to(torch.float64)
        pad = (0, Lout - n) if is_bhl else (0, 0, 0, Lout - n)
        a, g, c = dw_grads(torch.nn.functional.pad(dd, pad), _slice(u, b, o, e, is_bhl), w, P, is_bhl)
        _slice(du, b, o, e, is_bhl).copy_(a)
        dw += g
        db += c
    return du, dw, db
