"""main.lua's command line for a trained network: the non-training actions.

    python tools/run_main.py kitti fast -a test_te -net_fname net/net_kitti_fast_-a_train_all.t7
    python tools/run_main.py kitti2015 slow -a submit -net_fname N -data_root /data -out out
    python tools/run_main.py mb census -a test_te -rect imperfect -color gray
    python tools/run_main.py kitti fast -a time -net_fname N [-tiny]
    python tools/run_main.py kitti census -a predict -left L.png -right R.png -disp_max 70
    python tools/run_main.py kitti fast -a test_te -net_fname N -sm_skip sgm          # or -sm_terminate cbca1, ...
    python tools/run_main.py kitti census -a predict -left L.png -right R.png -disp_max 70 -confidence
    python tools/run_main.py kitti census -a predict -left L.png -right R.png -disp_max 70 -calib calib/000000.txt -ply
    python tools/run_main.py kitti census -a predict -left L.png -right R.png -disp_max 70 -rectify intrinsics.yml \
        -rectify extrinsics.yml -ply

Option names are main.lua's (-gpu is 1-based as there); -L1 ... -blur_t override the stereo method's preset
(main.lua:70-295); -sm_terminate / -sm_skip stop after / leave out one step of it (main.lua:953-1082; unknown step
names, and steps that do no work with these parameters, are refused).  Datasets are read relative to -data_root (default: the working directory), as main.lua reads them
relative to its own.  -confidence (an addition beyond the reference, -a predict only) also writes conf.bin, the margin
confidence of each pixel, and with the LR check lr.bin, main.lua:1056's outlier map (mc-cnn_b200/confidence.py).
-calib FILE (also an addition, -a predict only; KITTI 2012 calib/%06d.txt, KITTI 2015 calib_cam_to_cam/%06d.txt or a
MiddEval3 calib.txt, by dataset) also writes depth.bin, the metric depth of each pixel in metres (NaN = none), and with -ply
points.ply, the coloured point cloud; -max_depth M drops depths past M metres, and -density p (with -confidence) keeps only
the ceil(p H W) most confident pixels in both (mc-cnn_b200/depth.py).  -rectify FILE [-rectify FILE2] (also an addition,
-a predict only, instead of -calib) takes raw views of a calibrated rig: OpenCV FileStorage YAML files holding M1/K1, D1,
M2/K2, D2, R1, R2, P1, P2 (stereo_calib's intrinsics.yml and extrinsics.yml); the pair is rectified on the GPU first, every
output lies on the rectified grid, the depth uses the calibration P1 / P2 define, and the pixels outside the left view's
validity mask have no disparity (NaN), depth or vertex (mc-cnn_b200/rectify.py).  Training (-a train_tr / train_all) is not part of this tool.  See mc-cnn_b200/evaluate.py for
what each action computes and where it deliberately differs from main.lua.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PRESET_OPTIONS = {"L1": int, "tau1": float, "cbca_i1": int, "cbca_i2": int, "pi1": float, "pi2": float, "sgm_q1": float,
                  "sgm_q2": float, "alpha1": float, "tau_so": float, "sgm_i": int, "blur_sigma": float, "blur_t": float}
ACTIONS = ("test_te", "test_all", "submit", "time", "predict")


def _flag(v):
    """main.lua's boolean options: `-tiny` alone, or `-tiny true|false|1|0`"""
    return str(v).lower() not in ("false", "0", "")


def parser():
    ap = argparse.ArgumentParser(prog="run_main.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    ap.add_argument("arch", choices=("fast", "slow", "ad", "census"))
    ap.add_argument("-a", default="test_te", help="|".join(ACTIONS))
    ap.add_argument("-net_fname", default="")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    ap.add_argument("-tiny", nargs="?", const=True, default=False, type=_flag)
    ap.add_argument("-rect", default="imperfect")
    ap.add_argument("-color", default="gray")
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-out", default="out")
    ap.add_argument("-left", default="")
    ap.add_argument("-right", default="")
    ap.add_argument("-disp_max", type=int, default=None)
    ap.add_argument("-at", type=int, default=0)
    for name in ("debug", "use_cache", "make_cache"):
        ap.add_argument("-" + name, nargs="?", const=True, default=False, type=_flag)
    ap.add_argument("-sm_terminate", default="")
    ap.add_argument("-sm_skip", default="")
    ap.add_argument("-confidence", nargs="?", const=True, default=False, type=_flag)
    ap.add_argument("-calib", default="")
    ap.add_argument("-rectify", action="append", default=[])
    ap.add_argument("-ply", nargs="?", const=True, default=False, type=_flag)
    ap.add_argument("-max_depth", type=float, default=None)
    ap.add_argument("-density", type=float, default=None)
    for name, typ in PRESET_OPTIONS.items():
        ap.add_argument("-" + name, type=typ, default=None)
    return ap


def parse_args(argv=None):
    """-> (namespace, preset overrides dict).  Refuses what the actions do not implement before any GPU work."""
    from mccnn_b200 import evaluate

    args = parser().parse_args(argv)
    if args.a in ("train_tr", "train_all"):
        raise SystemExit("run_main.py: -a %s (training) is not supported; use a trained net with -net_fname" % args.a)
    if args.a not in ACTIONS:
        raise SystemExit("run_main.py: unknown action -a %s (%s)" % (args.a, ", ".join(ACTIONS)))
    if args.gpu < 1:
        raise SystemExit("run_main.py: -gpu is 1-based")
    if args.confidence and args.a != "predict":
        raise SystemExit("run_main.py: -confidence writes conf.bin next to -a predict's outputs; -a %s writes none" % args.a)
    if args.calib and args.a != "predict":
        raise SystemExit("run_main.py: -calib writes depth.bin next to -a predict's outputs; -a %s writes none" % args.a)
    if args.rectify and args.a != "predict":
        raise SystemExit("run_main.py: -rectify rectifies -a predict's raw pair; -a %s reads no raw pair" % args.a)
    if args.rectify and args.calib:
        raise SystemExit("run_main.py: -rectify defines the rectified pair's calibration; give -rectify or -calib, not both")
    if len(args.rectify) > 2:
        raise SystemExit("run_main.py: -rectify takes one or two files (e.g. intrinsics.yml and extrinsics.yml)")
    for f in args.rectify:
        if not os.path.isfile(f):
            raise SystemExit("run_main.py: -rectify %s is not a file" % f)
    if (args.ply or args.max_depth is not None or args.density is not None) and not (args.calib or args.rectify):
        raise SystemExit("run_main.py: -ply, -max_depth and -density apply to the depth outputs, which need -calib or -rectify")
    if args.max_depth is not None and not args.max_depth > 0:
        raise SystemExit("run_main.py: -max_depth must be > 0")
    if args.density is not None:
        if not args.confidence:
            raise SystemExit("run_main.py: -density keeps the most confident pixels; it needs -confidence")
        if not 0 < args.density <= 1:
            raise SystemExit("run_main.py: -density must be in (0, 1]")
    evaluate.check_options(args.dataset, at=args.at, color=args.color, debug=args.debug, use_cache=args.use_cache,
                           make_cache=args.make_cache)
    overrides = {k: getattr(args, k) for k in PRESET_OPTIONS if getattr(args, k) is not None}
    stage = {k: getattr(args, k) for k in ("sm_terminate", "sm_skip") if getattr(args, k)}
    if stage:                                              # main.lua's step names; make_params maps them to codes
        evaluate.check_stage_options(args.dataset, args.arch, **dict(overrides, **stage))
        overrides.update(stage)
    args.device = args.gpu - 1
    return args, overrides


def main(argv=None):
    args, overrides = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import dataio, evaluate, frontend, predict_kitti

    if args.a == "predict":
        if not (args.left and args.right and args.disp_max):
            raise SystemExit("run_main.py: -a predict needs -left, -right and -disp_max")
        depth_opts = {}
        if args.calib:
            depth_opts = dict(calib=dataio.read_calib(args.calib, args.dataset), ply=args.ply, max_depth=args.max_depth,
                              density=args.density)
        if args.rectify:
            H, W = predict_kitti.scan([(args.left, args.right, None)])[0]
            depth_opts = dict(rectify=dataio.read_rectification(args.rectify, "opencv", size=(W, H)), ply=args.ply,
                              max_depth=args.max_depth, density=args.density)
        frontend.predict(args.left, args.right, dataset=args.dataset, arch=args.arch, disp_max=args.disp_max,
                         out_dir=".", device=args.device, net_fname=args.net_fname or None, confidence=args.confidence,
                         **depth_opts, **overrides)
        return 0
    ev = evaluate.Evaluator(args.dataset, args.arch, net_fname=args.net_fname or None, device=args.device, **overrides)
    try:
        if args.a == "time":
            ev.time(tiny=args.tiny)
        elif args.a == "submit":
            ev.submit(data_root=args.data_root, out=args.out, rect=args.rect, color=args.color)
        else:
            ev.test(args.a, data_root=args.data_root, rect=args.rect, color=args.color)
    finally:
        ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
