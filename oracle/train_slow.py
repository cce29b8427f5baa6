"""Restatements of main.lua's training path for arch 'slow' (KITTI) -- TEST INFRASTRUCTURE.

* :func:`init_weights_slow`: the reset() draws of main.lua:663-695 line by line on ``preprocess.MT19937``: net_tr's
  convolutions, its nn.Linear layers (weight (out, in), then bias, U(-1/sqrt(in), +1/sqrt(in))), then net_te's
  convolutions constructed anew, whose draws are discarded when the weights are tied.
* :func:`step64_slow`: one forward / backward of net_tr + BCECriterion2 (main.lua:663-677, 848-870) in float64 autograd.
"""
import math

import numpy as np

from .train import init_weights, uniform


def init_linear(g, n_in, n_out):
    """nn.Linear(n_in, n_out):reset(), one draw at a time -> (W (out, in), b (out,)) float32"""
    stdv = 1 / math.sqrt(n_in)
    w = np.array([uniform(g, -stdv, stdv) for _ in range(n_out * n_in)]).astype(np.float32).reshape(n_out, n_in)
    b = np.array([uniform(g, -stdv, stdv) for _ in range(n_out)]).astype(np.float32)
    return w, b


def init_weights_slow(g, l1, fm, l2, nh2):
    """-> (tower, head); `g` is left where main.lua's per-sample draws start"""
    tower = init_weights(g, l1, fm)
    head = []
    for i in range(l2):
        head.append(init_linear(g, 2 * fm if i == 0 else nh2, nh2))
    head.append(init_linear(g, nh2, 1))
    init_weights(g, l1, fm)                                    # net_te's convolutions: drawn, then tied away
    return tower, head


def step64_slow(patches, tower, head, inter=False, device=None):
    """net_tr + BCECriterion2 in float64 autograd: patches (2 bs, 1, ws, ws) with ws = 1 + 2 len(tower); rows r of the
    reshape are patches 2r, 2r + 1 with targets 0, 1, 0, 1, ... -> (loss, [(gW, gb)] tower, [(gW, gb)] head, sigmoid).
    With `inter`, a fifth item: a dict of float64 numpy arrays, "z" and "dz" (each convolution's output, before its
    ReLU, and dLoss/dz), "rows" (bs, 2 fm), "rows_grad" (dLoss/drows), "fc" and "fc_grad" (each Linear's output before
    its ReLU or the Sigmoid, and dLoss/d that output) and "sigmoid".  `device` is where torch computes (default the CPU)."""
    import torch

    x = torch.as_tensor(np.asarray(patches), dtype=torch.float64, device=device)
    ps = [torch.tensor(np.asarray(a, np.float64), requires_grad=True, device=device)
          for wb in list(tower) + list(head) for a in wb]
    h, zs, fcs = x, [], []
    for i in range(len(tower)):
        zs.append(torch.nn.functional.conv2d(h, ps[2 * i], ps[2 * i + 1]))
        h = torch.relu(zs[-1])
    bs = x.shape[0] // 2
    h = rows = h.reshape(bs, -1)                                # nn.Reshape(bs, 2 fm)
    o = 2 * len(tower)
    for j in range(len(head)):
        h = h @ ps[o + 2 * j].T + ps[o + 2 * j + 1]
        fcs.append(h)
        if j < len(head) - 1:
            h = torch.relu(h)
    y = torch.sigmoid(h).reshape(-1)
    t = torch.tensor([r % 2 for r in range(bs)], dtype=torch.float64, device=device)
    eps = 1e-12
    loss = -((torch.log(y + eps) * t + torch.log(1 - y + eps) * (1 - t)) / bs).sum()
    grads = [a.cpu().numpy() for a in torch.autograd.grad(loss, ps + (zs + [rows] + fcs if inter else []))]
    pairs = [(grads[2 * i], grads[2 * i + 1]) for i in range(len(ps) // 2)]
    out = float(loss.detach()), pairs[:len(tower)], pairs[len(tower):], y.detach().cpu().numpy()
    if not inter:
        return out
    np64 = lambda a: a.detach().cpu().numpy()
    nz = len(ps) + len(zs)
    return out + (dict(z=[np64(a) for a in zs], dz=grads[len(ps):nz], rows=np64(rows), rows_grad=grads[nz],
                       fc=[np64(a) for a in fcs], fc_grad=grads[nz + 1:], sigmoid=out[3]),)
