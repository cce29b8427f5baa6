"""Time world-frame fusion at KITTI size (mc-cnn_b200/fusion.py, csrc/fusion.cu; DESIGN §23) on the GPU.

    python tools/time_fusion.py [--sizes 0,1000000,10000000] [--rounds 20] [--frames 8] [--json out.json]

Reported: the median time of one Fusion.add of a 375 x 1242 disparity map (random disparities 5-120 px, 10% holes) into an
empty table and into tables of about each size in --sizes (the map is added at a pose whose voxels the table already holds,
so the table keeps its size while every add merges it whole); the median time of Fusion.cloud() at each size; and, on a
synthetic posed drive of --frames 375 x 1242 frames with census at D 228, the frames per second of fuse_raw's loop
(fusion.fuse_drive) against predict_raw -disp's, each timed over the whole drive after one warm-up pass.  Each call is
timed on the host clock around work that ends in a device synchronise (add reads one int64 back).  The card's name and
power limit are read in the same run.
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
from mccnn_b200 import dataio, fusion, predict_raw, synth  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_confidence import card  # noqa: E402

H, W = 375, 1242
KITTI = dataio.Calib(721.5377, 609.5593, 172.854, 0.5372, 0.0, None, None)
VOXEL = 0.01


def frame(rng, dev):
    d = rng.uniform(5, 120, (H, W)).astype(np.float32)
    d[rng.random((H, W)) < 0.1] = np.nan
    return torch.from_numpy(d).to(dev), torch.from_numpy(rng.integers(0, 256, (H, W), dtype=np.uint8)).to(dev)


def pose(k):
    P = np.eye(4)
    P[0, 3] = 200.0 * k                 # frames 200 m apart share no voxel
    return P


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    name, power = card()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    d, img = frame(rng, dev)
    out = {"card": name, "power_limit": power, "shape": [H, W], "voxel": VOXEL, "add_ms": {}, "cloud_ms": {}, "voxels": {}}

    def empty_add():
        with fusion.Fusion(VOXEL) as fu:
            return host_ms(lambda: fu.add(d, KITTI, img, pose(0)))

    empty_add()
    out["add_ms"]["empty"] = statistics.median(empty_add() for _ in range(a.rounds))
    for target in (int(s) for s in a.sizes.split(",") if s):
        with fusion.Fusion(VOXEL) as fu:
            k = 0
            while fu.stats.voxels < target:
                fill_d, fill_img = frame(rng, dev)
                fu.add(fill_d, KITTI, fill_img, pose(k + 1))
                k += 1
            fu.add(d, KITTI, img, pose(0))                       # the timed frame's voxels, once
            n = fu.stats.voxels
            t_add = [host_ms(lambda: fu.add(d, KITTI, img, pose(0))) for _ in range(a.rounds)]
            assert fu.stats.voxels == n
            fu.cloud()
            t_cloud = [host_ms(lambda: fu.cloud()) for _ in range(a.rounds)]
        out["voxels"][str(target)] = n
        out["add_ms"][str(target)] = statistics.median(t_add)
        out["cloud_ms"][str(target)] = statistics.median(t_cloud)
        torch.cuda.empty_cache()

    with tempfile.TemporaryDirectory() as tmp:
        drive, _, _, _ = synth.write_kitti_posed_drive(tmp, n=a.frames, H=H, W=W)
        kw = dict(disp_max=228, device=0, verbose=False)

        def predict(o):
            t0 = time.perf_counter()
            predict_raw.predict_raw("kitti", "census", [drive], out=os.path.join(tmp, o), disp=True, **kw)
            return time.perf_counter() - t0

        def fuse(o):
            t0 = time.perf_counter()
            fusion.fuse_drive("kitti", "census", [drive], out=os.path.join(tmp, o), voxel=0.05, **kw)
            return time.perf_counter() - t0

        predict("warm_p")
        fuse("warm_f")
        t_pred, t_fuse = predict("timed_p"), fuse("timed_f")
    out["frames"] = a.frames
    out["predict_raw_fps"] = a.frames / t_pred
    out["fuse_raw_fps"] = a.frames / t_fuse
    print("card: %s, power limit %s" % (name, power))
    print("add of a %dx%d map (voxel %g m): empty table %.3f ms; %s" % (
        H, W, VOXEL, out["add_ms"]["empty"],
        "; ".join("%d voxels %.3f ms, cloud() %.3f ms" % (out["voxels"][k], out["add_ms"][k], out["cloud_ms"][k])
                  for k in out["voxels"])))
    print("census D 228, %d-frame posed drive: predict_raw -disp %.2f frames/s, fuse_raw %.2f frames/s"
          % (a.frames, out["predict_raw_fps"], out["fuse_raw_fps"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
