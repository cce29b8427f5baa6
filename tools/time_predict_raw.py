"""Time the raw-drive tools at KITTI size (mc-cnn_b200/predict_raw.py, depth_eval.evaluate_raw; DESIGN §21) on the GPU.

    python tools/time_predict_raw.py [--frames 12] [--arch census] [--disp_max 228] [--rounds 50] [--json out.json]

A seeded synthetic drive of 375 x 1242 grey pairs with ~120k-point scans is written to a temporary directory.  Reported:
the frames per second of predict_raw's loop writing the disparity PNGs, and of depth_eval's raw predict loop (the loop
plus the scoring), each timed over the whole drive after one warm-up pass; the median time of one mccnn_velo_depth_map call
(CUDA events) and of one frame's scoring (the projection, the disparity of the scan's depth, depth.metrics and its
read-back; host clock around a synchronised call); and that scoring's share of a frame of the raw predict loop.  The
card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, depth, depth_eval, predict_raw, synth  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_confidence import card, timed  # noqa: E402

H, W = 375, 1242


def kitti_scan(rng, n=120000):
    """a Velodyne-like sweep: all around, 1-80 m (about a quarter of it lands in the left image)"""
    r = rng.uniform(1, 80, n)
    a = rng.uniform(-np.pi, np.pi, n)
    return np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-3, 2, n), rng.uniform(0, 1, n)], 1).astype(np.float32)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--arch", default="census", choices=("census", "ad"))
    ap.add_argument("--disp_max", type=int, default=228)
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    name, power = card()
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        drive, _ = synth.write_kitti_drive(tmp, n=a.frames, H=H, W=W, seed=0, every=1)
        rng = np.random.default_rng(0)
        for k in range(a.frames):                       # full sweeps in place of the synthetic scene's points
            scan = np.concatenate([dataio.read_velodyne(dataio.raw_file(drive, dataio.RAW_SCAN, k))[:60000], kitti_scan(rng, 60000)])
            scan.astype("<f4").tofile(dataio.raw_file(drive, dataio.RAW_SCAN, k))
        frames = predict_raw.drive_frames([drive], velodyne=True)
        kw = dict(disp_max=a.disp_max, device=0, verbose=False)

        def loop(out):
            t0 = time.perf_counter()
            predict_raw.predict_raw("kitti", a.arch, [drive], out=os.path.join(tmp, out), disp=True, **kw)
            return time.perf_counter() - t0

        def scored():
            t0 = time.perf_counter()
            depth_eval.evaluate_raw("kitti", a.arch, frames, **kw)
            return time.perf_counter() - t0

        loop("warm")
        scored()
        t_loop, t_scored = loop("timed"), scored()

        cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
        scan = dataio.read_velodyne(dataio.raw_file(drive, dataio.RAW_SCAN, 0))
        pts = torch.from_numpy(scan).to(dev)
        pred = torch.rand((H, W), device=dev) * 100
        ops = {"velo_depth": lambda: depth.velo_depth(pts, cal, H, W),
               "score_frame": lambda: depth.metrics(pred, depth_eval.lidar_gt(scan, cal, H, W, dev), cal)}
        for fn in ops.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        t = {k: [] for k in ops}
        for _ in range(a.rounds):
            for k, fn in ops.items():
                t[k].append(timed(fn))
    n = len(frames)
    out = {"card": name, "power_limit": power, "shape": [H, W, a.disp_max], "arch": a.arch, "frames": n,
           "scan_points": int(len(scan)), "predict_raw_fps": n / t_loop, "raw_predict_fps": n / t_scored}
    out.update({k + "_ms": statistics.median(v) for k, v in t.items()})
    out["score_share_of_frame"] = out["score_frame_ms"] / (1e3 * t_scored / n)
    print("card: %s, power limit %s" % (name, power))
    print("%dx%d D %d %s, %d frames: predict_raw %.2f frames/s, raw predict + score %.2f frames/s; velo_depth %.4f ms per "
          "%d-point scan, scoring %.4f ms per frame (%.1f%% of a frame)"
          % (H, W, a.disp_max, a.arch, n, out["predict_raw_fps"], out["raw_predict_fps"], out["velo_depth_ms"],
             out["scan_points"], out["score_frame_ms"], 100 * out["score_share_of_frame"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
