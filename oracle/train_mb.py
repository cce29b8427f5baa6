"""Restatement of main.lua's Middlebury training draws and patches (dataset mb) -- TEST INFRASTRUCTURE.

* :func:`sample_params_mb`: main.lua:791-841 for one sample, one draw at a time on ``preprocess.MT19937``: the uniforms
  of :791-818 (oracle/train.py's sample_params), then light, exp, the d_exp test, exp_ only when it passes, the d_light
  test.  ``torch.random()`` is one 32-bit output of the generator; ``%`` is Lua's on non-negative integers.
* :func:`sample_patches_mb`: the four patches of one sample (:843-846) from ragged sources ``X[img][light]`` of shape
  (n_exp, 2, H, W), through oracle/train.py's warp_affine.
"""
from . import train as ot


def sample_params_mb(g, o, n_light, n_exp):
    """-> (sample_params' dict, light, exp, light_, exp_) for an image with n_light light groups j >= 2 and n_exp
    exposures in each (1-based light >= 2 and exp, as main.lua indexes X[img])"""
    p = ot.sample_params(g, o)
    light = g.random() % n_light + 2                     # (torch.random() % (#X[img] - 1)) + 2
    exp = g.random() % n_exp + 1
    light_, exp_ = light, exp
    if ot.uniform(g) < o["d_exp"]:
        exp_ = g.random() % n_exp + 1
    if ot.uniform(g) < o["d_light"]:
        light_ = max(2, light - 1)
    return p, light, exp, light_, exp_


def sample_patches_mb(p, row, X, light, exp, light_, exp_, ws):
    """X[light] (n_exp, 2, H, W) float32 for the sample's image -> its four (ws, ws) patches"""
    x0 = X[light][exp - 1, 0]
    x1 = X[light_][exp_ - 1, 1]
    return ot.sample_patches(p, row, x0, x1, ws)
