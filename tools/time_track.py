"""Time frame-to-model tracking at KITTI size (mc-cnn_b200/track.py, csrc/track.cu; DESIGN §25) on the GPU.

    python tools/time_track.py [--rounds 20] [--frames 8] [--json out.json]

Reported, on a synthetic posed drive of --frames 375 x 1242 frames (synth.write_kitti_posed_drive), voxel 0.05 m and the
default truncation: the median time of one gate-less (geometric) mccnn_track_step reduce at each level (its read-back
included); the median tracking cost of a frame, TSDF.render at the previous pose plus Tracker.track (both pyramids and
every ICP step); and the frames per second of fuse_raw -mesh -poses track's loop against -poses oxts's (fusion.fuse_drive)
with census at D 228, each over the whole drive after one warm-up pass, with the tracked drive's errors against its OXTS
poses.  Each call is timed on the host clock around work that ends in a device synchronise.  The card's name and power
limit are read in the same run.
"""
import argparse
import contextlib
import io
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
    out = {"card": name, "power_limit": power, "shape": [H, W], "voxel": VOXEL, "frames": a.frames}
    with tempfile.TemporaryDirectory() as tmp:
        drive, disps, _, _ = synth.write_kitti_posed_drive(tmp, n=a.frames, H=H, W=W)
        cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
        poses = dataio.raw_poses(drive, range(a.frames))
        lefts = [np.asarray(Image.open(dataio.raw_file(drive, dataio.RAW_LEFT, k))) for k in range(a.frames)]
        d = [torch.from_numpy(x).to(dev) for x in disps]
        with fusion.TSDF(VOXEL) as ts, track.Tracker(H, W) as tr:
            for k in range(a.frames - 1):
                ts.add(d[k], cal, lefts[k], poses[k])
            last = a.frames - 1
            Z = ts.render(cal, poses[last - 1], H, W)
            tr.source(d[last], cal)
            tr.model(Z, cal)
            T = track.rigid_inv(poses[last - 1]) @ poses[last]
            cos_t = math.cos(math.radians(track.THETA))
            for level in range(track.LEVELS):
                tr.step(level, T, track.DELTA[track.LEVELS - 1 - level], cos_t)
                t = [host_ms(lambda: tr.step(level, T, track.DELTA[track.LEVELS - 1 - level], cos_t)) for _ in range(a.rounds)]
                out["step_ms_level%d" % level] = statistics.median(t)

            def frame():
                Zp = ts.render(cal, poses[last - 1], H, W)
                return tr.track(d[last], cal, Zp, poses[last - 1], track.predict("track", poses[:last]))

            frame()
            out["track_frame_ms"] = statistics.median(host_ms(frame) for _ in range(a.rounds))
            out["render_ms"] = statistics.median(host_ms(lambda: ts.render(cal, poses[last - 1], H, W)) for _ in range(a.rounds))
        torch.cuda.empty_cache()
        kw = dict(disp_max=228, device=0, verbose=False, mesh=True)

        def fuse(o, **extra):
            t0 = time.perf_counter()
            r = fusion.fuse_drive("kitti", "census", [drive], out=os.path.join(tmp, o), voxel=VOXEL, **kw, **extra)
            return time.perf_counter() - t0, r

        fuse("warm_o")
        fuse("warm_t", poses="track")
        t_oxts, _ = fuse("timed_o")
        t_track, _ = fuse("timed_t", poses="track")
        with contextlib.redirect_stdout(io.StringIO()):
            _, r = fuse("traj", poses="track", traj=True)
        out.update(fuse_oxts_fps=a.frames / t_oxts, fuse_track_fps=a.frames / t_track, census_ate=r[0].traj.ate,
                   census_rpe_t=r[0].traj.rpe_t, census_rpe_r=r[0].traj.rpe_r, lost=r[0].lost)
    print("card: %s, power limit %s" % (name, power))
    print("reduce step at %dx%d: level 0 %.3f ms, level 1 %.3f ms, level 2 %.3f ms" % (
        H, W, out["step_ms_level0"], out["step_ms_level1"], out["step_ms_level2"]))
    print("tracking one frame, render included: %.3f ms (render alone %.3f ms)" % (out["track_frame_ms"], out["render_ms"]))
    print("census D 228, %d-frame posed drive, fuse_raw -mesh: -poses oxts %.2f frames/s, -poses track %.2f frames/s" % (
        a.frames, out["fuse_oxts_fps"], out["fuse_track_fps"]))
    print("census -poses track against OXTS: ate %.5f m, rpe_t %.5f m, rpe_r %.5f deg, lost %d" % (
        out["census_ate"], out["census_rpe_t"], out["census_rpe_r"], out["lost"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
