"""Run the stereo method over whole KITTI raw drives: disparity, depth and point clouds per frame (an addition beyond the
reference).

    python tools/predict_raw.py kitti fast -net_fname N -drive /data/raw/2011_09_26/2011_09_26_drive_0002_sync -out O \\
        [-disp] [-depth] [-ply] [-confidence [-density p]] [-every k] [-disp_max 228] [-gpu 1]
    torchrun --nproc-per-node 8 tools/predict_raw.py kitti census -drive D1 -drive D2 -out O -disp

Each frame of each drive (the grey pair image_00 / image_01) is predicted with the presets of `dataset` (kitti or
kitti2015) and written under ``O/<drive>/``: -disp ``disp/%010d.png`` (KITTI's PNG16), -depth ``depth/%010d.png``
(KITTI's depth format), -ply ``points/%010d.ply``, -confidence ``conf/%010d.bin`` (the margin confidence, raw float32).
-density p keeps the ceil(p H W) most confident pixels of each map.  -every k takes every k-th frame.  The calibration
comes from the drive's date directory (calib_cam_to_cam.txt).  A drive whose output directory is not empty is refused.
Under torchrun the frames go round-robin over the processes.  The line ``<date>/<drive> <frame>`` is printed for each
frame, in order.  -gpu is 1-based as in main.lua.  See mc-cnn_b200/predict_raw.py.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="predict_raw.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=("kitti", "kitti2015"))
    ap.add_argument("arch", choices=("fast", "slow", "census", "ad"))
    ap.add_argument("-net_fname", default="")
    ap.add_argument("-drive", action="append", default=[], help="a drive directory <date>/<date>_drive_<nnnn>_sync; repeatable")
    ap.add_argument("-out", default="out")
    ap.add_argument("-disp", action="store_true", help="write O/<drive>/disp/%%010d.png")
    ap.add_argument("-depth", action="store_true", help="write O/<drive>/depth/%%010d.png")
    ap.add_argument("-ply", action="store_true", help="write O/<drive>/points/%%010d.ply")
    ap.add_argument("-confidence", action="store_true", help="write O/<drive>/conf/%%010d.bin")
    ap.add_argument("-density", type=float, default=None, help="with -confidence: keep this share of each map's pixels, in (0, 1]")
    ap.add_argument("-every", type=int, default=1)
    ap.add_argument("-disp_max", type=int, default=228)
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def parse_args(argv=None):
    """Refuses what cannot run before any file or GPU is touched."""
    args = parser().parse_args(argv)
    if args.arch in ("fast", "slow") and not args.net_fname:
        raise SystemExit("predict_raw.py: arch '%s' needs -net_fname" % args.arch)
    if not args.drive:
        raise SystemExit("predict_raw.py: give at least one -drive")
    if not (args.disp or args.depth or args.ply or args.confidence):
        raise SystemExit("predict_raw.py: nothing to write; ask for -disp, -depth, -ply or -confidence")
    if args.density is not None:
        if not args.confidence:
            raise SystemExit("predict_raw.py: -density ranks pixels by their confidence; it needs -confidence")
        if not 0 < args.density <= 1:
            raise SystemExit("predict_raw.py: -density must be in (0, 1]")
    if args.every < 1:
        raise SystemExit("predict_raw.py: -every must be at least 1")
    if args.disp_max < 1:
        raise SystemExit("predict_raw.py: -disp_max must be at least 1")
    if args.gpu < 1:
        raise SystemExit("predict_raw.py: -gpu is 1-based")
    for d in args.drive:
        if not os.path.isdir(d):
            raise SystemExit("predict_raw.py: %s is not a directory" % d)
    return args


def main(argv=None):
    args = parse_args(argv)
    import torch.distributed as dist

    import mccnn_b200  # noqa: F401
    from mccnn_b200.predict_raw import predict_raw

    world = int(os.environ.get("WORLD_SIZE", "1"))
    device = args.gpu - 1
    if world > 1:
        # one index per frame crosses between processes: gloo on the host is enough
        dist.init_process_group("gloo")
        device = int(os.environ.get("LOCAL_RANK", "0"))
    try:
        predict_raw(args.dataset, args.arch, args.drive, net_fname=args.net_fname or None, out=args.out, disp=args.disp,
                    depth=args.depth, ply=args.ply, confidence=args.confidence, density=args.density, every=args.every,
                    disp_max=args.disp_max, device=device)
    finally:
        if world > 1:
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
