"""Score KITTI training pairs with the devkits' metrics: background interpolation, then D1 (2015) or Out / Avg (2012).

    python tools/kitti_eval.py predict kitti -net_fname net/net_kitti_fast_-a_train_all.t7 -data_root /data [-out O]
    python tools/kitti_eval.py predict kitti2015 -net_fname N -data_root /data [-arch fast|slow|census|ad] [-disp_max 228] \\
        [-gpu 1] [-out O]
    python tools/kitti_eval.py score kitti2015 O -data_root /data [-gpu 1]
    torchrun --nproc-per-node 8 tools/kitti_eval.py predict kitti -net_fname N -data_root /data

`predict` runs the net over every raw training pair (predict_kitti.py test's loop) and scores each map on the GPU; with -out
it also writes the maps in submission layout (``O/%06d_10.png``, ``O/disp_0/%06d_10.png`` for kitti2015).  `score` scores
such a directory.  Both print one tab-separated line per pair (0-based index, then the rates: kitti Out-Noc at 2, 3, 4,
5 px, Out-All at 2, 3, 4, 5 px, Avg-Noc, Avg-All, density; kitti2015 D1-bg, D1-fg, D1-all against disp_noc_0, the same
against disp_occ_0, density), then the devkit's table of the pixel-weighted totals.  Rates are fractions, Avg in px.  The
training ground truth (disp_noc and disp_occ, plus obj_map for kitti2015) is read from ``<data_root>/data.kitti/unzip`` or
``data.kitti2015/unzip``.  -gpu is 1-based as in main.lua.  See mc-cnn_b200/kitti_eval.py.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="kitti_eval.py", description=__doc__.splitlines()[0])
    sub = ap.add_subparsers(dest="action", required=True)
    p = sub.add_parser("predict", help="run a net over the training pairs and score each map")
    p.add_argument("dataset", choices=("kitti", "kitti2015"))
    p.add_argument("-net_fname", default="")
    p.add_argument("-arch", choices=("fast", "slow", "census", "ad"), default="fast")
    p.add_argument("-data_root", default=".")
    p.add_argument("-disp_max", type=int, default=228)
    p.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    p.add_argument("-out", default=None, help="also write the maps here, in submission layout")
    p.add_argument("-density", type=float, default=None,
                   help="keep this share of each map's pixels, the most confident ones, in (0, 1]")
    s = sub.add_parser("score", help="score PNG16 maps in submission layout")
    s.add_argument("dataset", choices=("kitti", "kitti2015"))
    s.add_argument("pred_dir")
    s.add_argument("-data_root", default=".")
    s.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def parse_args(argv=None):
    """Refuses what cannot run before any file or GPU is touched."""
    args = parser().parse_args(argv)
    if args.gpu < 1:
        raise SystemExit("kitti_eval.py: -gpu is 1-based")
    if args.action == "predict":
        if args.arch in ("fast", "slow") and not args.net_fname:
            raise SystemExit("kitti_eval.py: arch '%s' needs -net_fname" % args.arch)
        if args.disp_max < 1:
            raise SystemExit("kitti_eval.py: -disp_max must be at least 1")
        if args.density is not None and not 0 < args.density <= 1:
            raise SystemExit("kitti_eval.py: -density must be in (0, 1]")
    elif not os.path.isdir(args.pred_dir):
        raise SystemExit("kitti_eval.py: %s is not a directory" % args.pred_dir)
    return args


def main(argv=None):
    args = parse_args(argv)
    import torch.distributed as dist

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import kitti_eval

    world = int(os.environ.get("WORLD_SIZE", "1"))
    device = args.gpu - 1
    if world > 1:
        # only a few counts per pair cross between processes: gloo on the host is enough
        dist.init_process_group("gloo")
        device = int(os.environ.get("LOCAL_RANK", "0"))
    try:
        if args.action == "predict":
            kitti_eval.evaluate_training(args.dataset, args.net_fname or None, args.arch, data_root=args.data_root,
                                         disp_max=args.disp_max, out=args.out, device=device, density=args.density)
        else:
            kitti_eval.score_dir(args.dataset, args.pred_dir, data_root=args.data_root, device=device)
    finally:
        if world > 1:
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
