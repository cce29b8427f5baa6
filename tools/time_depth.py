"""Time depth, the point cloud and the depth metrics of one KITTI-sized pair (mc-cnn_b200/depth.py, DESIGN §20) next to the
stereo method of predict_kitti.py's loop, on the GPU, with CUDA events.

    python tools/time_depth.py [--rounds 20] [--json out.json]

At 375 x 1242 with D 228 (predict_kitti's disp_max) and the kitti 'fast' preset: StereoPipeline.run_shape on random unit
features (the stereo method's share of a pair, without the feature tower), then depth.depth, depth.point_cloud (count, its
one int64 read-back, fill), the cloud with its device-to-host copy, and depth.metrics against one ground truth (with its
read-back), alternating in one process after a warm-up.  Prints the card's name and power limit with the medians (ms).
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, depth, pipeline  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_confidence import card, timed  # noqa: E402

H, W, C, D = 375, 1242, 64, 228
CAL = dataio.Calib(721.5377, 609.5593, 172.854, 0.5371657, 0.0, W, H)    # KITTI 2012's calib/000000.txt


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    dev = torch.device("cuda:0")
    name, power = card()
    g = torch.Generator(device=dev).manual_seed(0)
    fL = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev, generator=g), dim=0)
    fR = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev, generator=g), dim=0)
    iL = torch.randn((H, W), device=dev, generator=g)
    iR = torch.randn((H, W), device=dev, generator=g)
    disp = torch.empty((H, W), device=dev)
    sp = pipeline.StereoPipeline(C, D, H, W, pipeline.make_params("kitti", "fast"))
    sp.run_shape(fL, fR, iL, iR, disp=disp)
    d = torch.rand((H, W), device=dev, generator=g) * 200       # a dense map with valid depths everywhere
    gt = torch.where(torch.rand((H, W), device=dev, generator=g) < 0.3, d + 5 * torch.rand((H, W), device=dev, generator=g),
                     torch.zeros_like(d))
    left = torch.randint(0, 256, (H, W), device=dev, dtype=torch.uint8, generator=g)
    ops = {"run_shape": lambda: sp.run_shape(fL, fR, iL, iR, disp=disp),
           "depth": lambda: depth.depth(d, CAL),
           "cloud": lambda: depth.point_cloud(d, CAL, left),
           "cloud_d2h": lambda: depth.point_cloud(d, CAL, left).data.cpu(),
           "metrics": lambda: depth.metrics(d, gt, CAL)}
    for fn in ops.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    t = {k: [] for k in ops}
    for _ in range(a.rounds):
        for k, fn in ops.items():
            t[k].append(timed(fn))
    sp.close()
    out = {"card": name, "power_limit": power, "rounds": a.rounds, "shape": [H, W, D]}
    out.update({k: statistics.median(v) for k, v in t.items()})
    per_pair = out["depth"] + out["cloud_d2h"] + 2 * out["metrics"]      # depth PNG, PLY, noc and occ scores
    out["depth_share_of_run_shape"] = per_pair / out["run_shape"]
    print("card: %s, power limit %s" % (name, power))
    print("%dx%d D %d, ms: run_shape %.3f  depth %.4f  cloud %.4f  cloud+d2h %.4f  metrics %.4f  (depth + cloud + 2 metrics "
          "= %.1f%% of run_shape)" % (H, W, D, out["run_shape"], out["depth"], out["cloud"], out["cloud_d2h"], out["metrics"],
                                     100 * out["depth_share_of_run_shape"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
