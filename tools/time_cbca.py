"""Time one CBCA iteration at the bench size on pitched volumes (L2 flushed between launches):
constant-work TMA kernel vs the exact kernel.  Prints ms and GB/s of the algorithmic 2V + 32HW bytes."""
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
ap.add_argument("--L1", type=int, default=5)
ap.add_argument("--tau1", type=float, default=0.13)
a = ap.parse_args()
dev = torch.device("cuda:0")
lib = adcensus.lib()
D, H, W = a.D, a.H, a.W
ld = (W + 3) // 4 * 4
g = torch.Generator(device=dev).manual_seed(0)
img = torch.randn((2, 1, H, W), device=dev, generator=g)
x0c = torch.empty((1, 4, H, W), device=dev)
x1c = torch.empty((1, 4, H, W), device=dev)
adcensus.cross(img[0:1], x0c, a.L1, a.tau1)
adcensus.cross(img[1:2], x1c, a.L1, a.tau1)
vin = torch.randn((D, H, ld), device=dev, generator=g)
xs = torch.arange(ld, device=dev)[None, None, :]
ds = torch.arange(D, device=dev)[:, None, None]
vin[(xs < ds).expand(D, H, ld)] = float("nan")
vout = torch.empty_like(vin)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
s = adcensus._stream(vin)


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


bytes_alg = 2 * 4 * D * H * W + 32 * H * W
med, mn = timeit(lambda: lib.mccnn_cbca_fast_pitched(x0c.data_ptr(), x1c.data_ptr(), vin.data_ptr(), vout.data_ptr(), D, H, W, ld,
                                                     -1, max(a.L1, 2), s))
print("cbca_tma   L1=%d: median %.4f ms  min %.4f ms  %.0f GB/s (algorithmic)" % (a.L1, med, mn, bytes_alg / med / 1e6))
if ld == W or True:
    vc = vin[:, :, :W].contiguous()[None]
    oc = torch.empty_like(vc)
    med, mn = timeit(lambda: lib.adcensus_cbca_ex(x0c.data_ptr(), x1c.data_ptr(), vc.data_ptr(), oc.data_ptr(), D, H, W, -1,
                                                  max(a.L1, 2), s))
    print("cbca exact L1=%d: median %.4f ms  min %.4f ms  %.0f GB/s (algorithmic)" % (a.L1, med, mn, bytes_alg / med / 1e6))
