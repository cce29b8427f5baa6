"""Score the margin confidence of a trained network's maps by the sparsification curve (an addition beyond the reference;
mc-cnn_b200/confidence.py, DESIGN §19).

    python tools/sparsification.py kitti fast -a test_te -net_fname net/net_kitti_fast_-a_train_all.t7 -data_root /data
    python tools/sparsification.py mb census -a test_te -rect imperfect -err_at 2

One line ``id<TAB>err<TAB>auc<TAB>auc_opt`` per example of main.lua's test_te / test_all list, numbers as Lua prints them
(%.14g), then ``mean`` and the three means.  err is run_main.py's per-example error (the curve's last point); auc the area
under the curve of the bad-pixel share against the share of ground-truth pixels kept, most confident first; auc_opt the same
for the ideal ordering.  -err_at defaults to main.lua's (3 for KITTI, 1 for Middlebury); -L1 ... -blur_t and -sm_terminate /
-sm_skip override the stereo method as in run_main.py.  Middlebury has no test_all, as in main.lua.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from run_main import PRESET_OPTIONS  # noqa: E402


def parser():
    ap = argparse.ArgumentParser(prog="sparsification.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    ap.add_argument("arch", choices=("fast", "slow", "ad", "census"))
    ap.add_argument("-a", default="test_te", choices=("test_te", "test_all"))
    ap.add_argument("-net_fname", default="")
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-rect", default="imperfect")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    ap.add_argument("-err_at", type=float, default=None)
    ap.add_argument("-sm_terminate", default="")
    ap.add_argument("-sm_skip", default="")
    for name, typ in PRESET_OPTIONS.items():
        ap.add_argument("-" + name, type=typ, default=None)
    return ap


def parse_args(argv=None):
    """-> (namespace, preset overrides).  Refuses what cannot run before any GPU work."""
    from mccnn_b200 import evaluate

    args = parser().parse_args(argv)
    if args.dataset == "mb" and args.a == "test_all":
        raise SystemExit("sparsification.py: test_all not supported on Middlebury (main.lua:1136)")
    if args.gpu < 1:
        raise SystemExit("sparsification.py: -gpu is 1-based")
    if args.err_at is not None and not args.err_at >= 0:
        raise SystemExit("sparsification.py: -err_at must be >= 0")
    overrides = {k: getattr(args, k) for k in PRESET_OPTIONS if getattr(args, k) is not None}
    stage = {k: getattr(args, k) for k in ("sm_terminate", "sm_skip") if getattr(args, k)}
    if stage:
        evaluate.check_stage_options(args.dataset, args.arch, **dict(overrides, **stage))
        overrides.update(stage)
    args.device = args.gpu - 1
    return args, overrides


def main(argv=None):
    args, overrides = parse_args(argv)
    from mccnn_b200 import evaluate

    ev = evaluate.Evaluator(args.dataset, args.arch, net_fname=args.net_fname or None, device=args.device, **overrides)
    try:
        return ev.sparsification(args.a, data_root=args.data_root, rect=args.rect, err_at=args.err_at)
    finally:
        ev.close()


if __name__ == "__main__":
    main()
    sys.exit(0)
