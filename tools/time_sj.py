"""Time StereoJoin at the bench size (L2 flushed between launches): the pitched form the fused pipeline runs vs the operator
on contiguous tensors."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--D", type=int, default=228)
ap.add_argument("--H", type=int, default=370)
ap.add_argument("--W", type=int, default=1226)
ap.add_argument("--C", type=int, default=64)
a = ap.parse_args()
dev = torch.device("cuda:0")
lib = adcensus.lib()
D, H, W, C = a.D, a.H, a.W, a.C
ld = (W + 3) // 4 * 4
g = torch.Generator(device=dev).manual_seed(0)
fL = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev, generator=g), dim=0)
fR = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev, generator=g), dim=0)
oL = torch.empty((D, H, ld), device=dev)
oR = torch.empty((D, H, ld), device=dev)
cL = torch.empty((1, D, H, W), device=dev)
cR = torch.empty((1, D, H, W), device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
s = adcensus._stream(fL)


def timeit(fn):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(a.iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


valid = 4 * H * (D * W - D * (D - 1) // 2)
bytes_alg = 2 * 4 * C * H * W + 2 * valid
med, mn = timeit(lambda: lib.mccnn_stereo_join_pitched(fL.data_ptr(), fR.data_ptr(), oL.data_ptr(), oR.data_ptr(), C, D, H, W,
                                                       ld, s))
print("StereoJoin pitched : median %.4f ms  min %.4f ms  %.0f GB/s (algorithmic 2F + 2 valid)" % (med, mn, bytes_alg / med / 1e6))
med, mn = timeit(lambda: lib.adcensus_StereoJoin(fL.data_ptr(), fR.data_ptr(), cL.data_ptr(), cR.data_ptr(), C, D, H, W, s))
print("StereoJoin operator: median %.4f ms  min %.4f ms  %.0f GB/s (algorithmic 2F + 2 valid)" % (med, mn, bytes_alg / med / 1e6))
