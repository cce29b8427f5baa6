"""Fuse each KITTI raw drive's stereo depth into one world-frame point cloud, posed by the drive's OXTS records (an
addition beyond the reference).

    python tools/fuse_raw.py kitti census -drive /data/raw/2011_09_26/2011_09_26_drive_0002_sync -out O -voxel 0.1 \\
        [-min_frames 2] [-max_depth 40] [-every k] [-confidence -density p] [-disp_max 228] [-gpu 1] [-net_fname N]

Each frame of each drive is predicted with the presets of `dataset` (kitti or kitti2015), in frame order on one GPU, and
added to the drive's voxel map (edge -voxel metres) at its pose: the frame's GPS/IMU record ``oxts/data/%010d.txt`` and the
date directory's calib_imu_to_velo.txt, calib_velo_to_cam.txt and calib_cam_to_cam.txt.  The world frame is the rectified
left camera of the drive's first fused frame.  ``O/<drive>/fused.ply`` gets one vertex per voxel seen by at least
-min_frames frames: the mean of its points and of their colours.  -max_depth drops farther pixels, -density p keeps the
ceil(p H W) most confident pixels of each map (with -confidence).  The line ``<date>/<drive> <frame>`` is printed for each
frame, then one summary line per drive.  Refused before any GPU work: _extract drives, a missing OXTS or calibration file,
an existing fused.ply, and running under torchrun with more than one process.  -gpu is 1-based as in main.lua.  See
mc-cnn_b200/fusion.py.

    python tools/fuse_raw.py kitti census -drive D -out O -voxel 0.1 -mesh [-trunc 0.4] [-score [-crop garg] [-min_depth 1]]

-mesh runs the same frames into a truncated signed distance field (DESIGN §24, truncation -trunc metres, 4 -voxel by
default, at most 256 -voxel) and writes ``O/<drive>/mesh.ply`` instead: a triangle mesh of its zero level set over the voxels seen by at least
-min_frames frames, then one summary line per drive.  -score (with -mesh) then renders the field at each fused frame's
pose and scores it against that frame's Velodyne scan as depth_eval.py raw does (-crop none|garg|eigen, -min_depth,
max_depth 80 m), next to the frame's own stereo depth: one line per frame, the stereo then the fused lidar_* values, then
the line of means.  Refused as well: -trunc not finite, below -voxel or above 256 -voxel, -trunc or -score without -mesh, an existing
mesh.ply, and -score on a drive whose frames lack scans.

    python tools/fuse_raw.py kitti census -drive D -out O -voxel 0.05 -mesh -poses track|refine [-traj] [-score]

-poses track (with -mesh) poses each frame after the drive's first by tracking it against the field rendered at the
previous frame's pose (DESIGN §25): projective point-to-plane ICP on three levels, predicted by constant velocity, so the
drive needs no oxts/.  -poses refine predicts by the OXTS increment instead.  A frame tracking loses prints
``<date>/<drive> <frame> lost``, keeps its prediction and is not integrated.  ``O/<drive>/poses.txt`` gets the poses
(KITTI odometry format).  -traj (which needs oxts/) prints one line per drive against the OXTS poses: ate, rpe_t, rpe_r,
t_err (%) and r_err (deg/m) over 100 .. 800 m segments, and their count.  -score scores renders at the tracked poses.
Refused as well: -poses track or refine without -mesh, -traj without them, and an existing poses.txt.

    python tools/fuse_raw.py kitti census -drive D -out O -voxel 0.05 -mesh -poses track -photometric 0.01 [-rho 30] \\
        [-grad_min 2]

-photometric lambda (metres per grey level; 0, the default, is off) adds a photometric term to the tracking (DESIGN §26):
each frame's left image is aligned to the previous frame's, which fixes motion along a street whose surfaces' normals all
lie across it.  -rho (grey levels) and -grad_min (grey levels per pixel) gate its pixels.  Refused as well: -photometric
without -poses track or refine, and a -photometric, -rho or -grad_min that is not a finite number >= 0.
"""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="fuse_raw.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=("kitti", "kitti2015"))
    ap.add_argument("arch", choices=("fast", "slow", "census", "ad"))
    ap.add_argument("-net_fname", default="")
    ap.add_argument("-drive", action="append", default=[], help="a drive directory <date>/<date>_drive_<nnnn>_sync; repeatable")
    ap.add_argument("-out", default="out")
    ap.add_argument("-voxel", type=float, required=True, help="the voxel edge in metres")
    ap.add_argument("-min_frames", type=int, default=1, help="write the voxels seen by at least this many frames")
    ap.add_argument("-max_depth", type=float, default=None, help="drop pixels farther than this many metres")
    ap.add_argument("-confidence", action="store_true", help="compute each map's margin confidence (for -density)")
    ap.add_argument("-density", type=float, default=None, help="with -confidence: keep this share of each map's pixels, in (0, 1]")
    ap.add_argument("-every", type=int, default=1)
    ap.add_argument("-disp_max", type=int, default=228)
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    ap.add_argument("-mesh", action="store_true", help="fuse into a truncated signed distance field and write mesh.ply")
    ap.add_argument("-trunc", type=float, default=None, help="with -mesh: the truncation in metres (default 4 -voxel)")
    ap.add_argument("-score", action="store_true", help="with -mesh: score the field's depth at each frame against its scan")
    ap.add_argument("-crop", choices=("none", "garg", "eigen"), default="none", help="with -score: the crop rectangle")
    ap.add_argument("-min_depth", type=float, default=1e-3, help="with -score: the nearest scored depth in metres")
    ap.add_argument("-poses", choices=("oxts", "track", "refine"), default="oxts",
                    help="the frames' poses: the OXTS records, or tracked against the field (with -mesh)")
    ap.add_argument("-traj", action="store_true", help="with -poses track or refine: print the trajectory's errors against OXTS")
    ap.add_argument("-photometric", type=float, default=None,
                    help="with -poses track or refine: the photometric term's weight in metres per grey level (0: off)")
    ap.add_argument("-rho", type=float, default=30.0, help="with -photometric: the largest residual of an inlier, grey levels")
    ap.add_argument("-grad_min", type=float, default=2.0, help="with -photometric: the smallest gradient of an inlier")
    return ap


def parse_args(argv=None):
    """Refuses what cannot run before any file or GPU is touched."""
    args = parser().parse_args(argv)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("fuse_raw.py: fusion adds the frames in order on one GPU; run it as one process, not under torchrun")
    if args.arch in ("fast", "slow") and not args.net_fname:
        raise SystemExit("fuse_raw.py: arch '%s' needs -net_fname" % args.arch)
    if not args.drive:
        raise SystemExit("fuse_raw.py: give at least one -drive")
    if not (math.isfinite(args.voxel) and args.voxel > 0):
        raise SystemExit("fuse_raw.py: -voxel must be a finite length > 0 in metres")
    if args.min_frames < 1:
        raise SystemExit("fuse_raw.py: -min_frames must be at least 1")
    if args.max_depth is not None and not args.max_depth > 0:
        raise SystemExit("fuse_raw.py: -max_depth must be > 0")
    if args.density is not None:
        if not args.confidence:
            raise SystemExit("fuse_raw.py: -density ranks pixels by their confidence; it needs -confidence")
        if not 0 < args.density <= 1:
            raise SystemExit("fuse_raw.py: -density must be in (0, 1]")
    if args.every < 1:
        raise SystemExit("fuse_raw.py: -every must be at least 1")
    if args.disp_max < 1:
        raise SystemExit("fuse_raw.py: -disp_max must be at least 1")
    if args.gpu < 1:
        raise SystemExit("fuse_raw.py: -gpu is 1-based")
    if args.trunc is not None and not args.mesh:
        raise SystemExit("fuse_raw.py: -trunc is the distance field's truncation; it needs -mesh")
    if args.score and not args.mesh:
        raise SystemExit("fuse_raw.py: -score renders the distance field; it needs -mesh")
    if args.trunc is not None and not (math.isfinite(args.trunc) and args.voxel <= args.trunc <= 256 * args.voxel):
        raise SystemExit("fuse_raw.py: -trunc must be a finite length in metres, from -voxel to 256 -voxel")
    if args.poses != "oxts" and not args.mesh:
        raise SystemExit("fuse_raw.py: -poses %s tracks each frame against the distance field; it needs -mesh" % args.poses)
    if args.traj and args.poses == "oxts":
        raise SystemExit("fuse_raw.py: -traj compares tracked poses with OXTS; it needs -poses track or refine")
    if args.photometric is not None and args.poses == "oxts":
        raise SystemExit("fuse_raw.py: -photometric weighs a term of the tracking; it needs -poses track or refine")
    for name in ("photometric", "rho", "grad_min"):
        v = getattr(args, name)
        if v is not None and not (math.isfinite(v) and v >= 0):
            raise SystemExit("fuse_raw.py: -%s must be a finite number >= 0" % name)
    if args.score and not 0 < args.min_depth <= 80.0:
        raise SystemExit("fuse_raw.py: -min_depth must be in (0, 80]")
    for d in args.drive:
        if not os.path.isdir(d):
            raise SystemExit("fuse_raw.py: %s is not a directory" % d)
    return args


def main(argv=None):
    args = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200.fusion import fuse_drive

    fuse_drive(args.dataset, args.arch, args.drive, net_fname=args.net_fname or None, out=args.out, voxel=args.voxel,
               min_frames=args.min_frames, max_depth=args.max_depth, every=args.every, confidence=args.confidence,
               density=args.density, disp_max=args.disp_max, device=args.gpu - 1,
               **(dict(mesh=True, trunc=args.trunc, score=args.score, crop=args.crop, min_depth=args.min_depth,
                       poses=args.poses, traj=args.traj) if args.mesh else {}),
               **(dict(photometric=args.photometric, rho=args.rho, grad_min=args.grad_min) if args.photometric else {}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
