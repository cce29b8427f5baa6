"""Time the photometric term of tracking at KITTI size (mc-cnn_b200/track.py, csrc/track.cu; DESIGN §26) on the GPU.

    python tools/time_track_photometric.py [--rounds 20] [--frames 8] [--json out.json]

Reported, on a synthetic posed drive of --frames 375 x 1242 frames (synth.write_kitti_posed_drive), voxel 0.05 m and the
default truncation: the median time of one mccnn_track_step reduce at each level with gates (the joint step) against one
without (read-backs included); the median tracking cost of a frame, TSDF.render at the previous pose plus Tracker.track,
without and with the term (lambda 0.01, both intensity pyramids included); and the frames per second of fuse_raw -mesh
-poses track's loop (fusion.fuse_drive) with census at D 228, without and with -photometric 0.01, each over the whole
drive after one warm-up pass.  Each call is timed on the host clock around work that ends in a device synchronise.  The
card's name and power limit are read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, fusion, synth, track  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_confidence import card  # noqa: E402

H, W = 375, 1242
VOXEL = 0.05
LAMBDA = 0.01


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    name, power = card()
    dev = torch.device("cuda:0")
    out = {"card": name, "power_limit": power, "shape": [H, W], "voxel": VOXEL, "frames": a.frames, "photometric": LAMBDA}
    with tempfile.TemporaryDirectory() as tmp:
        drive, disps, _, _ = synth.write_kitti_posed_drive(tmp, n=a.frames, H=H, W=W)
        cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
        poses = dataio.raw_poses(drive, range(a.frames))
        lefts = [np.asarray(Image.open(dataio.raw_file(drive, dataio.RAW_LEFT, k))) for k in range(a.frames)]
        d = [torch.from_numpy(x).to(dev) for x in disps]
        L = [torch.from_numpy(x).to(dev) for x in lefts]
        last = a.frames - 1
        with fusion.TSDF(VOXEL) as ts, track.Tracker(H, W) as geo, track.Tracker(H, W, photometric=LAMBDA) as pho:
            for k in range(last):
                ts.add(d[k], cal, lefts[k], poses[k])
            Z = ts.render(cal, poses[last - 1], H, W)
            for tr in (geo, pho):
                tr.source(d[last], cal)
                tr.model(Z, cal)
            pho.intensity("source", L[last])
            pho.intensity("reference", L[last - 1])
            T = track.rigid_inv(poses[last - 1]) @ poses[last]
            cos_t = math.cos(math.radians(track.THETA))
            gates = (track.GRAD_MIN, track.RHO)
            for level in range(track.LEVELS):
                delta = track.DELTA[track.LEVELS - 1 - level]
                for key, fn in (("step_ms", lambda: geo.step(level, T, delta, cos_t)),
                                ("step_joint_ms", lambda: pho.step(level, T, delta, cos_t, gates))):
                    fn()
                    out["%s_level%d" % (key, level)] = statistics.median(host_ms(fn) for _ in range(a.rounds))
            pred = track.predict("track", poses[:last])

            def frame(tr, **images):
                Zp = ts.render(cal, poses[last - 1], H, W)
                return tr.track(d[last], cal, Zp, poses[last - 1], pred, **images)

            for key, tr, images in (("track_frame_ms", geo, {}),
                                    ("track_frame_photometric_ms", pho, dict(left=L[last], ref_left=L[last - 1]))):
                frame(tr, **images)
                out[key] = statistics.median(host_ms(lambda: frame(tr, **images)) for _ in range(a.rounds))
        torch.cuda.empty_cache()
        kw = dict(disp_max=228, device=0, verbose=False, mesh=True, poses="track")

        def fuse(o, **extra):
            t0 = time.perf_counter()
            fusion.fuse_drive("kitti", "census", [drive], out=os.path.join(tmp, o), voxel=VOXEL, **kw, **extra)
            return time.perf_counter() - t0

        fuse("warm_t")
        fuse("warm_p", photometric=LAMBDA)
        out.update(fuse_track_fps=a.frames / fuse("timed_t"), fuse_photometric_fps=a.frames / fuse("timed_p", photometric=LAMBDA))
    print("card: %s, power limit %s" % (name, power))
    for level in range(track.LEVELS):
        print("reduce step at %dx%d level %d: geometric %.3f ms, joint %.3f ms" % (
            H, W, level, out["step_ms_level%d" % level], out["step_joint_ms_level%d" % level]))
    print("tracking one frame, render included: %.3f ms geometric, %.3f ms with the photometric term" % (
        out["track_frame_ms"], out["track_frame_photometric_ms"]))
    print("census D 228, %d-frame posed drive, fuse_raw -mesh -poses track: %.2f frames/s, -photometric %g %.2f frames/s" % (
        a.frames, out["fuse_track_fps"], LAMBDA, out["fuse_photometric_fps"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
