"""Time the margin confidence and the LR map in the fused pipeline, and the sparse-map / sparsification-count kernels
(mc-cnn_b200/confidence.py, DESIGN §19), on the GPU, with CUDA events.

    python tools/time_confidence.py [--rounds 10] [--json out.json]

At bench.py's k228 (kitti accurate_cbca4, 370 x 1226, D 228) and k70 (kitti fast, D 70) workloads: run_shape without conf,
with conf, and with conf and lr, alternating in one process after a warm-up, each variant timed per call; then sparsify and
the counts on a 375 x 1242 map.  Prints the card's name and power limit with the numbers (medians over the rounds, ms).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import confidence, pipeline  # noqa: E402

WORKLOADS = {"k228": ("accurate_cbca4", 228), "k70": ("fast", 70)}
H, W, C = 370, 1226, 64


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    dev = torch.device("cuda:0")
    name, power = card()
    out = {"card": name, "power_limit": power, "rounds": a.rounds}
    g = torch.Generator(device=dev).manual_seed(0)
    fL = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev, generator=g), dim=0)
    fR = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev, generator=g), dim=0)
    iL = torch.randn((H, W), device=dev, generator=g)
    iR = torch.randn((H, W), device=dev, generator=g)
    disp, conf, lr = (torch.empty((H, W), device=dev) for _ in range(3))
    for key, (preset, D) in WORKLOADS.items():
        sp = pipeline.StereoPipeline(C, D, H, W, pipeline.make_params("kitti", preset))
        variants = {"plain": lambda: sp.run_shape(fL, fR, iL, iR, disp=disp),
                    "conf": lambda: sp.run_shape(fL, fR, iL, iR, disp=disp, conf=conf),
                    "conf_lr": lambda: sp.run_shape(fL, fR, iL, iR, disp=disp, conf=conf, lr=lr)}
        for fn in variants.values():
            for _ in range(a.warmup):
                fn()
        torch.cuda.synchronize()
        t = {k: [] for k in variants}
        for _ in range(a.rounds):
            for k, fn in variants.items():
                t[k].append(timed(fn))
        out[key] = {k: statistics.median(v) for k, v in t.items()}
        sp.run_shape(fL, fR, iL, iR, disp=disp)
        n0 = sp.launches_per_run
        sp.run_shape(fL, fR, iL, iR, disp=disp, conf=conf)
        out[key]["launches_plain_conf"] = [n0, sp.launches_per_run]
        sp.close()
    h, w = 375, 1242
    d = torch.rand((h, w), device=dev, generator=g) * 200
    c = torch.rand((h, w), device=dev, generator=g)
    gt = torch.where(torch.rand((h, w), device=dev, generator=g) < 0.3, d + 5 * torch.rand((h, w), device=dev, generator=g),
                     torch.zeros_like(d))
    ops = {"sparsify": lambda: confidence.sparsify(d, c, 0.5, 0.0), "counts": lambda: confidence.counts(d, c, gt, 3.0)}
    for fn in ops.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    out["map_375x1242"] = {k: statistics.median(timed(fn) for _ in range(a.rounds)) for k, fn in ops.items()}
    print("card: %s, power limit %s" % (name, power))
    for key in WORKLOADS:
        r = out[key]
        print("%s run_shape ms: plain %.3f  conf %.3f  conf+lr %.3f  launches plain/conf %s" % (key, r["plain"], r["conf"],
                                                                                                r["conf_lr"], r["launches_plain_conf"]))
    print("375x1242 map ms (counts includes its device-to-host read-back): sparsify %.3f  counts %.3f"
          % (out["map_375x1242"]["sparsify"], out["map_375x1242"]["counts"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
