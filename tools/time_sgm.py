"""Time the fused pipeline's sgm2 phase at the bench shape, the 11-pass kernels (mccnn_sgm2_band, pass mask 15, zeroed
accumulator: classes, selectors, hpair, down, up) against the checkpoint schedule (mccnn_sgm2_ckpt: classes, selectors,
forward, backward horizontal, backward vertical).  The two alternate in one process, L2 flushed before each call, CUDA
events around each; then one torch.profiler pass gives each launch's time.  Prints the algorithmic bytes
(V = 4·D·H·W: 11V, against 7V plus the checkpoints written and read once), the card and its power limit."""
import argparse
import ctypes
import json
import os
import re
import subprocess
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, rowband  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=20)
ap.add_argument("--D", type=int, default=228)
ap.add_argument("--H", type=int, default=370)
ap.add_argument("--W", type=int, default=1226)
ap.add_argument("--direction", type=int, default=-1)
a = ap.parse_args()

dev = torch.device("cuda:0")
lib = adcensus.lib()
H, W, D = a.H, a.W, a.D
prm = (1.32, 24.25, 0.08, 2.0, 3.0, 2.0)          # the kitti accurate_cbca4 preset's pi1, pi2, tau_so, alpha1, q1, q2
opt = SimpleNamespace(pi1=prm[0], pi2=prm[1], tau_so=prm[2], alpha1=prm[3], sgm_q1=prm[4], sgm_q2=prm[5])
g = torch.Generator(device=dev).manual_seed(0)
iL, iR = torch.rand((2, H, W), device=dev, generator=g)
cost = torch.rand((H, W, D), device=dev, generator=g) * 4
d, x = torch.arange(D, device=dev)[None, :], torch.arange(W, device=dev)[:, None]
cost[:, (x < d) if a.direction < 0 else (x >= W - d)] = float("nan")
out_old, out_new = torch.empty_like(cost), torch.empty_like(cost)
ck_bytes = lib.mccnn_sgm2_ckpt_bytes(H, W, D)
scratch = torch.empty(ck_bytes // 4, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
ops = rowband.CudaOps(dev)
st = adcensus._stream(cost)


def old():
    out_old.zero_()                                # outside the timed window (below): the pipeline's accumulator needs no zeroing
    ev[0].record()
    ops.sgm_band(iL, iR, cost, out_old, H, W, 0, 0, opt, a.direction, 15, True)
    ev[1].record()


def new():
    ev[0].record()
    rc = lib.mccnn_sgm2_ckpt(ctypes.c_void_p(iL.data_ptr()), ctypes.c_void_p(iR.data_ptr()), ctypes.c_void_p(cost.data_ptr()),
                             ctypes.c_void_p(out_new.data_ptr()), ctypes.c_void_p(scratch.data_ptr()), ck_bytes, H, W, D, *prm,
                             a.direction, st)
    ev[1].record()
    assert rc == 0, rc


def timed(fn):
    flush.zero_()
    fn()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1])


ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for fn in (old, new, old, new):
    timed(fn)
t_old, t_new = [], []
for _ in range(a.rounds):
    t_old.append(timed(old))
    t_new.append(timed(new))
same = torch.equal(out_old.nan_to_num(7.5), out_new.nan_to_num(7.5)) and torch.equal(out_old.isnan(), out_new.isnan())

# launch by launch: one profiled call of each, L2 flushed before it
from torch.profiler import ProfilerActivity, profile  # noqa: E402

per_kernel = {}
for name, fn in (("old", old), ("new", new)):
    flush.zero_()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = [(e.name, e.device_time_total / 1000) for e in prof.events() if e.device_time_total > 0 and "elementwise" not in e.name
          and "fill" not in e.name.lower()]
    per_kernel[name] = [((re.findall(r"\w+_kernel", n) or [n[:40]])[0], round(t, 4)) for n, t in ks]

V = 4 * D * H * W
try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except (OSError, subprocess.SubprocessError, IndexError):
    smi = "nvidia-smi unavailable"
t_old.sort()
t_new.sort()
med = lambda t: t[len(t) // 2]
print(json.dumps({
    "card": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "shape": [H, W, D], "direction": a.direction, "rounds": a.rounds,
    "bit_identical": bool(same),
    "old_ms": {"median": round(med(t_old), 4), "min": round(t_old[0], 4), "max": round(t_old[-1], 4)},
    "new_ms": {"median": round(med(t_new), 4), "min": round(t_new[0], 4), "max": round(t_new[-1], 4)},
    "old_GB": round(11 * V / 1e9, 3), "new_GB": round((7 * V + 2 * ck_bytes) / 1e9, 3), "checkpoint_MB": round(ck_bytes / 1e6, 1),
    "old_TBps": round(11 * V / med(t_old) / 1e9, 3), "new_TBps": round((7 * V + 2 * ck_bytes) / med(t_new) / 1e9, 3),
    "per_kernel_ms": per_kernel,
}, indent=1))
