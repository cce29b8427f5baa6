"""main.lua -debug for the test actions: what run_main.py prints for -a test_te / test_all, and for every example main.lua's
three images -- the ground truth and the prediction in the jet colour map, and the left image with good pixels tinted green
and bad ones red.

    python tools/debug_images.py kitti fast -a test_te -net_fname net/net_kitti_fast_-a_train_all.t7 -out tmp
    python tools/debug_images.py mb census -a test_te -data_root /data

Files: <dataset>_<id>_gt.png, <dataset>_<arch>_<id>_pred.png and <dataset>_<arch>_<id>_err.png under -out (default tmp,
where main.lua writes them).  The images are made after each example's timed region, so the runtime column is the one
run_main.py prints.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ACTIONS = ("test_te", "test_all")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="debug_images.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    ap.add_argument("arch", choices=("fast", "slow", "ad", "census"))
    ap.add_argument("-a", default="test_te", help="|".join(ACTIONS))
    ap.add_argument("-net_fname", default="")
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-out", default="tmp")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    args = ap.parse_args(argv)
    if args.a not in ACTIONS:
        raise SystemExit("debug_images.py: -a %s: main.lua writes -debug images for %s only" % (args.a, " and ".join(ACTIONS)))
    if args.gpu < 1:
        raise SystemExit("debug_images.py: -gpu is 1-based")
    if args.arch in ("fast", "slow") and not args.net_fname:
        raise SystemExit("debug_images.py: arch '%s' needs -net_fname" % args.arch)
    if args.dataset == "mb" and args.a == "test_all":
        raise SystemExit("debug_images.py: test_all not supported on Middlebury.")           # main.lua:1136
    args.device = args.gpu - 1
    return args


def main(argv=None):
    args = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import evaluate

    ev = evaluate.Evaluator(args.dataset, args.arch, net_fname=args.net_fname or None, device=args.device)
    try:
        ev.test(args.a, data_root=args.data_root, debug_dir=args.out)
    finally:
        ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
