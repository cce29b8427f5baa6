"""Score the stereo method's depth on the KITTI 2012 / 2015 and MiddEval3 training pairs: AbsRel, SqRel, RMSE, RMSE log and
the delta < 1.25^k rates (an addition beyond the reference).

    python tools/depth_eval.py predict kitti -net_fname net/net_kitti_fast_-a_train_all.t7 -data_root /data
    python tools/depth_eval.py predict mb -arch census -data_root /data [-gpu 1]
    python tools/depth_eval.py score kitti2015 O -data_root /data [-source disp|depth]
    torchrun --nproc-per-node 8 tools/depth_eval.py predict kitti -net_fname N -data_root /data
    python tools/depth_eval.py raw predict kitti fast -net_fname N -drive D [-drive D2 ...] | -list FILE [-data_root R] \
        [-min_depth 1e-3] [-max_depth 80] [-crop garg|eigen|none] [-every k] [-disp_max 228]
    python tools/depth_eval.py raw score O -drive D ... | -list FILE [-source disp|depth]

`predict` runs the net over every training pair (KITTI: the raw pairs at -disp_max, as predict_kitti.py test; MiddEval3:
the trainingH grey pairs at each scene's ndisp) and scores each map's depth on the GPU.  `score` scores the maps the other
tools wrote under O: KITTI disparity PNGs in submission layout or, with -source depth, predict_kitti.py -depth's
``O/depth_0/%06d_10.png``; MiddEval3 ``O/trainingH/<scene>/disp0*.pfm``.  Both print one tab-separated line per pair
(index or scene, then abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3, n, coverage against KITTI's noc and occ ground truth,
or MiddEval3's disp0GT.pfm), then the line of means.  The calibration comes from beside the images (KITTI 2015: the
calibration archive unpacked into data.kitti2015/unzip).  -gpu is 1-based as in main.lua.  See mc-cnn_b200/depth_eval.py.

`raw` scores KITTI raw drives against their Velodyne scans projected into the left grey camera (DESIGN §21): `raw
predict` runs the net over the frames (every frame with a scan of each -drive, or the ``<date>/<drive> <frame>`` lines of
-list, relative to -data_root), `raw score` reads predict_raw.py's ``O/<drive>/disp/%010d.png`` (or, with -source depth,
``depth/%010d.png``).  Both print ``<date>/<drive> <frame>`` and the lidar_ metrics per frame, then the line of means.
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
    r = sub.add_parser("raw", help="KITTI raw drives scored against their projected Velodyne scans")
    rsub = r.add_subparsers(dest="raw_action", required=True)
    rp = rsub.add_parser("predict", help="run a net over the frames and score each map's depth")
    rp.add_argument("dataset", choices=("kitti", "kitti2015"))
    rp.add_argument("arch", choices=("fast", "slow", "census", "ad"))
    rp.add_argument("-net_fname", default="")
    rp.add_argument("-disp_max", type=int, default=228)
    rs = rsub.add_parser("score", help="score the maps predict_raw.py wrote")
    rs.add_argument("pred_dir")
    rs.add_argument("-source", choices=("disp", "depth"), default="disp")
    for q in (rp, rs):
        q.add_argument("-drive", action="append", default=[], help="a drive directory; repeatable")
        q.add_argument("-list", default=None, help="a split file of '<date>/<drive> <frame>' lines")
        q.add_argument("-data_root", default=".", help="where the -list lines' dates are")
        q.add_argument("-every", type=int, default=1, help="with -drive: every k-th frame")
        q.add_argument("-min_depth", type=float, default=1e-3)
        q.add_argument("-max_depth", type=float, default=80.0)
        q.add_argument("-crop", choices=("none", "garg", "eigen"), default="none")
        q.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def parse_args(argv=None):
    """Refuses what cannot run before any file or GPU is touched."""
    args = parser().parse_args(argv)
    if args.gpu < 1:
        raise SystemExit("depth_eval.py: -gpu is 1-based")
    if args.action == "raw":
        if bool(args.drive) == bool(args.list):
            raise SystemExit("depth_eval.py: raw takes -drive (one or more) or -list, not both")
        if args.list and not os.path.isfile(args.list):
            raise SystemExit("depth_eval.py: %s is not a file" % args.list)
        if args.every < 1:
            raise SystemExit("depth_eval.py: -every must be at least 1")
        if args.list and args.every != 1:
            raise SystemExit("depth_eval.py: -every applies to -drive; a -list names its frames")
        if not 0 < args.min_depth <= args.max_depth:
            raise SystemExit("depth_eval.py: need 0 < -min_depth <= -max_depth")
        for d in args.drive:
            if not os.path.isdir(d):
                raise SystemExit("depth_eval.py: %s is not a directory" % d)
        import mccnn_b200  # noqa: F401
        from mccnn_b200.predict_raw import check_synced

        try:
            check_synced(args.drive)
        except ValueError as e:
            raise SystemExit("depth_eval.py: %s" % e)
        if args.raw_action == "predict":
            if args.arch in ("fast", "slow") and not args.net_fname:
                raise SystemExit("depth_eval.py: arch '%s' needs -net_fname" % args.arch)
            if args.disp_max < 1:
                raise SystemExit("depth_eval.py: -disp_max must be at least 1")
        elif not os.path.isdir(args.pred_dir):
            raise SystemExit("depth_eval.py: %s is not a directory" % args.pred_dir)
    elif args.action == "predict":
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
        if args.action == "raw":
            from mccnn_b200 import predict_raw

            frames = (predict_raw.read_list(args.list, args.data_root) if args.list else
                      predict_raw.drive_frames(args.drive, args.every, velodyne=True))
            kw = dict(min_depth=args.min_depth, max_depth=args.max_depth, crop=args.crop, device=device)
            if args.raw_action == "predict":
                depth_eval.evaluate_raw(args.dataset, args.arch, frames, net_fname=args.net_fname or None,
                                        disp_max=args.disp_max, **kw)
            else:
                depth_eval.score_raw(frames, args.pred_dir, source=args.source, **kw)
        elif args.action == "predict":
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
