"""Time the truncated signed distance field at KITTI size (mc-cnn_b200/fusion.py's TSDF, csrc/tsdf.cu; DESIGN §24) on the
GPU.

    python tools/time_tsdf.py [--bricks 20000] [--rounds 10] [--frames 8] [--json out.json]

Reported, on a synthetic posed drive of --frames 375 x 1242 frames (synth.write_kitti_posed_drive with scans), voxel 0.05 m
and the default truncation: the median time of one TSDF.add of a frame's exact disparities into the drive's field (a small
table) and into a table grown to about --bricks bricks by frames far away (a large table: every add integrates every
brick); the median mesh() time with its vertex and face counts and the median render() time per frame, both on the
drive's field; the pool bytes of the drive's field; and the frames per second of fuse_raw -mesh's loop against fuse_raw's
(fusion.fuse_drive) with census at D 228, each over the whole drive after one warm-up pass, then the stereo and fused
lidar_abs_rel and lidar_a1 means of fuse_raw -mesh -score.  Each call is timed on the host clock around work that ends in a
device synchronise.  The card's name and power limit are read in the same run.
"""
import argparse
import contextlib
import io
import json
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
from mccnn_b200 import dataio, fusion, synth  # noqa: E402

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
    ap.add_argument("--bricks", type=int, default=20000)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    name, power = card()
    dev = torch.device("cuda:0")
    out = {"card": name, "power_limit": power, "shape": [H, W], "voxel": VOXEL, "frames": a.frames}
    with tempfile.TemporaryDirectory() as tmp:
        drive, disps, _, _ = synth.write_kitti_posed_drive(tmp, n=a.frames, H=H, W=W, velodyne=True)
        cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
        poses = dataio.raw_poses(drive, range(a.frames))
        lefts = [np.asarray(Image.open(dataio.raw_file(drive, dataio.RAW_LEFT, k))) for k in range(a.frames)]
        d = [torch.from_numpy(x).to(dev) for x in disps]
        with fusion.TSDF(VOXEL) as ts:
            for k in range(a.frames):
                ts.add(d[k], cal, lefts[k], poses[k])
            small = ts.stats.bricks
            t_small = [host_ms(lambda: ts.add(d[0], cal, lefts[0], poses[0])) for _ in range(a.rounds)]
            m = ts.mesh()
            t_mesh = [host_ms(lambda: ts.mesh()) for _ in range(a.rounds)]
            ts.render(cal, poses[0], H, W)
            t_render = [host_ms(lambda: ts.render(cal, poses[k % a.frames], H, W)) for k in range(a.rounds)]
            out.update(small_bricks=small, add_small_ms=statistics.median(t_small), mesh_ms=statistics.median(t_mesh),
                       vertices=m.n, faces=int(m.faces.shape[0]), render_ms=statistics.median(t_render),
                       pool_bytes=ts.stats.pool_bytes, bricks=ts.stats.bricks)
        with fusion.TSDF(VOXEL) as ts:
            k = 0
            while ts.stats.bricks < a.bricks:
                P = poses[k % a.frames].copy()
                P[0, 3] += 200.0 * (k + 1)              # far apart: every frame brings its own bricks
                ts.add(d[k % a.frames], cal, lefts[k % a.frames], P)
                k += 1
            ts.add(d[0], cal, lefts[0], poses[0])
            big = ts.stats.bricks
            t_big = [host_ms(lambda: ts.add(d[0], cal, lefts[0], poses[0])) for _ in range(a.rounds)]
            assert ts.stats.bricks == big
            out.update(large_bricks=big, add_large_ms=statistics.median(t_big))
        torch.cuda.empty_cache()
        kw = dict(disp_max=228, device=0, verbose=False)

        def fuse(o, **extra):
            t0 = time.perf_counter()
            r = fusion.fuse_drive("kitti", "census", [drive], out=os.path.join(tmp, o), voxel=VOXEL, **kw, **extra)
            return time.perf_counter() - t0, r

        fuse("warm_f")
        fuse("warm_m", mesh=True)
        t_fuse, _ = fuse("timed_f")
        t_mesh_loop, _ = fuse("timed_m", mesh=True)
        with contextlib.redirect_stdout(io.StringIO()):
            _, r = fuse("scored", mesh=True, score=True)
        mean = r[0].scores.mean
        cols = fusion.SCORE_COLUMNS
        out.update(fuse_raw_fps=a.frames / t_fuse, fuse_raw_mesh_fps=a.frames / t_mesh_loop,
                   stereo_abs_rel=mean[cols.index("stereo_lidar_abs_rel")], stereo_a1=mean[cols.index("stereo_lidar_a1")],
                   fused_abs_rel=mean[cols.index("fused_lidar_abs_rel")], fused_a1=mean[cols.index("fused_lidar_a1")])
    print("card: %s, power limit %s" % (name, power))
    print("add of a %dx%d frame (voxel %g m): %d bricks %.3f ms; %d bricks %.3f ms" % (
        H, W, VOXEL, out["small_bricks"], out["add_small_ms"], out["large_bricks"], out["add_large_ms"]))
    print("mesh %.3f ms (%d vertices, %d faces); render %.3f ms per frame; pool %d bytes for %d bricks" % (
        out["mesh_ms"], out["vertices"], out["faces"], out["render_ms"], out["pool_bytes"], out["bricks"]))
    print("census D 228, %d-frame posed drive: fuse_raw %.2f frames/s, fuse_raw -mesh %.2f frames/s" % (
        a.frames, out["fuse_raw_fps"], out["fuse_raw_mesh_fps"]))
    print("-score means: stereo lidar_abs_rel %.4f a1 %.4f; fused lidar_abs_rel %.4f a1 %.4f" % (
        out["stereo_abs_rel"], out["stereo_a1"], out["fused_abs_rel"], out["fused_a1"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
