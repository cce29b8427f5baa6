"""GPU: the fused pipeline's sgm2 schedule (mccnn_sgm2_ckpt: forward scans that store line-state checkpoints, backward
scans that recompute the forward values from them) against the 11-pass kernels (mccnn_sgm2_band, pass mask 15, zeroed
accumulator), bit for bit, NaN positions and signs of zeros included: every (K, VEC) instantiation, image sizes on both
sides of the checkpoint spacing (16 columns, 8 rows), both directions with StereoJoin's NaN triangle, the class-tie
images of tests/dispatch_cases.py, the fall-back to the 11-pass kernels when the scratch is too small, and the bench
shape."""
import ctypes
import importlib.util
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, rowband  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("dispatch_cases", os.path.join(ROOT, "tests", "dispatch_cases.py"))
dc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(dc)

CK_H, CK_V = 16, 8          # sgm.cu SGM_CK_H / SGM_CK_V


def dev():
    return torch.device("cuda:0")


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


def same(a, b, what=""):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    if not np.array_equal(a, b, equal_nan=True):
        bad = ~((a == b) | (np.isnan(a) & np.isnan(b)))
        raise AssertionError("%s: %d / %d elements differ, first %s: got %s want %s" % (
            what, bad.sum(), bad.size, np.argwhere(bad)[:5].tolist(), a[bad][:5], b[bad][:5]))
    z = b == 0
    assert np.array_equal(np.signbit(a[z]), np.signbit(b[z])), what + ": signs of zeros differ"


def ckpt_bytes(H, W, D):
    return (H * -(-W // CK_H) + W * -(-H // CK_V)) * 32 * dc.sgm_k(D) * 4


def run_both(iL, iR, cost, params, direction, scratch_bytes=None):
    """(new, old, scratch before, scratch after): mccnn_sgm2_ckpt into a NaN-filled output, mccnn_sgm2_band into zeros"""
    H, W, D = cost.shape
    lib = adcensus.lib()
    need = lib.mccnn_sgm2_ckpt_bytes(H, W, D)
    assert need == ckpt_bytes(H, W, D)
    nbytes = need if scratch_bytes is None else scratch_bytes
    scratch = torch.full((need // 4 + 4,), 7.0, device=dev())
    before = scratch.clone()
    new = torch.full_like(cost, float("nan"))
    rc = lib.mccnn_sgm2_ckpt(vp(iL), vp(iR), vp(cost), vp(new), vp(scratch), nbytes, H, W, D, *params, direction,
                             adcensus._stream(cost))
    assert rc == 0, rc
    old = torch.zeros_like(cost)
    pi1, pi2, tau_so, alpha1, q1, q2 = params
    opt = SimpleNamespace(pi1=pi1, pi2=pi2, tau_so=tau_so, alpha1=alpha1, sgm_q1=q1, sgm_q2=q2)
    rowband.CudaOps(dev()).sgm_band(iL, iR, cost, old, H, W, 0, 0, opt, direction, 15, True)
    torch.cuda.synchronize()
    return new, old, before, scratch


def inputs(H, W, D, params, direction, seed=0):
    c = dc.SGMCase(H, W, D, 0, 0, params, dc.sgm_k(D), False)
    x0, x1, vol = dc.sgm_inputs(c, direction, seed)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    return cu(x0), cu(x1), cu(vol)


# (H, W, D, params): D picks (K, VEC) (D % 4 != 0 runs the scalar variant); H and W below, on, one above and off the
# checkpoint spacing
CASES = [
    (1, 2, 1, dc.SGM_TIE),
    (1, 1, 129, dc.SGM_TIE),
    (7, 15, 31, dc.SGM_TIE),
    (8, 16, 40, dc.SGM_TIE),
    (9, 17, 64, dc.SGM_TEN),
    (21, 37, 99, dc.SGM_TIE),
    (16, 33, 128, dc.SGM_TIE),
    (17, 48, 250, dc.SGM_TIE),
    (24, 49, 256, dc.SGM_TEN),
    (25, 50, 301, dc.SGM_TIE),
    (13, 70, 512, dc.SGM_TIE),
    (40, 15, 228, dc.SGM_TIE),
]


@pytest.mark.parametrize("direction", [-1, 1])
@pytest.mark.parametrize("H,W,D,params", CASES, ids=["H%dW%dD%d_tau%g" % (c[0], c[1], c[2], c[3][2]) for c in CASES])
def test_ckpt_schedule_matches_11_pass_kernels(H, W, D, params, direction):
    iL, iR, cost = inputs(H, W, D, params, direction)
    new, old, before, after = run_both(iL, iR, cost, params, direction)
    same(new, old, "checkpoint schedule")
    if W > CK_H or H > CK_V:
        assert not torch.equal(before, after), "no checkpoint written"


@pytest.mark.parametrize("direction", [-1, 1])
def test_too_small_scratch_runs_the_11_pass_kernels(direction):
    H, W, D = 20, 45, 128
    iL, iR, cost = inputs(H, W, D, dc.SGM_TIE, direction)
    new, old, before, after = run_both(iL, iR, cost, dc.SGM_TIE, direction, scratch_bytes=ckpt_bytes(H, W, D) - 1)
    same(new, old, "fall-back")
    assert torch.equal(before, after), "the fall-back wrote into the scratch"


@pytest.mark.parametrize("direction", [-1, 1])
def test_bench_shape(direction):
    H, W, D = 370, 1226, 228
    g = torch.Generator(device=dev()).manual_seed(5 + direction)
    iL, iR = (torch.randint(0, 5, (2, H, W), device=dev(), generator=g) * 0.25).float()
    cost = (torch.randint(0, 64, (H, W, D), device=dev(), generator=g) * 0.125).float()
    d, x = torch.arange(D, device=dev())[None, :], torch.arange(W, device=dev())[:, None]
    cost[:, (x < d) if direction < 0 else (x >= W - d)] = float("nan")
    new, old, _, _ = run_both(iL, iR, cost, (1.32, 24.25, 0.25, 2.0, 3.0, 2.0), direction)
    same(new, old, "bench shape")
