"""Score the stereo method's depth on the KITTI 2012 / 2015 and MiddEval3 training pairs: AbsRel, SqRel, RMSE, RMSE log and
the delta < 1.25^k rates (an addition beyond the reference).

    python tools/depth_eval.py predict kitti -net_fname net/net_kitti_fast_-a_train_all.t7 -data_root /data
    python tools/depth_eval.py predict mb -arch census -data_root /data [-gpu 1]
    python tools/depth_eval.py score kitti2015 O -data_root /data [-source disp|depth]
    torchrun --nproc-per-node 8 tools/depth_eval.py predict kitti -net_fname N -data_root /data

`predict` runs the net over every training pair (KITTI: the raw pairs at -disp_max, as predict_kitti.py test; MiddEval3:
the trainingH grey pairs at each scene's ndisp) and scores each map's depth on the GPU.  `score` scores the maps the other
tools wrote under O: KITTI disparity PNGs in submission layout or, with -source depth, predict_kitti.py -depth's
``O/depth_0/%06d_10.png``; MiddEval3 ``O/trainingH/<scene>/disp0*.pfm``.  Both print one tab-separated line per pair
(index or scene, then abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3, n, coverage against KITTI's noc and occ ground truth,
or MiddEval3's disp0GT.pfm), then the line of means.  The calibration comes from beside the images (KITTI 2015: the
calibration archive unpacked into data.kitti2015/unzip).  -gpu is 1-based as in main.lua.  See mc-cnn_b200/depth_eval.py.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="depth_eval.py", description=__doc__.splitlines()[0])
    sub = ap.add_subparsers(dest="action", required=True)
    p = sub.add_parser("predict", help="run a net over the training pairs and score each map's depth")
    p.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    p.add_argument("-net_fname", default="")
    p.add_argument("-arch", choices=("fast", "slow", "census", "ad"), default="fast")
    p.add_argument("-data_root", default=".")
    p.add_argument("-disp_max", type=int, default=228, help="KITTI only; MiddEval3 uses each scene's ndisp")
    p.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    s = sub.add_parser("score", help="score written disparity or depth maps")
    s.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    s.add_argument("pred_dir")
    s.add_argument("-data_root", default=".")
    s.add_argument("-source", choices=("disp", "depth"), default="disp")
    s.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def parse_args(argv=None):
    """Refuses what cannot run before any file or GPU is touched."""
    args = parser().parse_args(argv)
    if args.gpu < 1:
        raise SystemExit("depth_eval.py: -gpu is 1-based")
    if args.action == "predict":
        if args.arch in ("fast", "slow") and not args.net_fname:
            raise SystemExit("depth_eval.py: arch '%s' needs -net_fname" % args.arch)
        if args.disp_max < 1:
            raise SystemExit("depth_eval.py: -disp_max must be at least 1")
    else:
        if not os.path.isdir(args.pred_dir):
            raise SystemExit("depth_eval.py: %s is not a directory" % args.pred_dir)
        if args.dataset == "mb" and args.source == "depth":
            raise SystemExit("depth_eval.py: MiddEval3 maps are scored from disparity PFMs only")
    return args


def main(argv=None):
    args = parse_args(argv)
    import torch.distributed as dist

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import depth_eval

    world = int(os.environ.get("WORLD_SIZE", "1"))
    device = args.gpu - 1
    if world > 1:
        # a few numbers per pair cross between processes: gloo on the host is enough
        dist.init_process_group("gloo")
        device = int(os.environ.get("LOCAL_RANK", "0"))
    try:
        if args.action == "predict":
            depth_eval.evaluate_training(args.dataset, args.net_fname or None, args.arch, data_root=args.data_root,
                                         disp_max=args.disp_max, device=device)
        else:
            depth_eval.score_dir(args.dataset, args.pred_dir, data_root=args.data_root, source=args.source, device=device)
    finally:
        if world > 1:
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
