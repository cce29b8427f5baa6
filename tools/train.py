"""main.lua's training actions for the fast architecture on KITTI: ``-a train_tr`` and ``-a train_all``.

    python tools/train.py kitti fast -a train_tr -data_root /data             # 14 epochs, then test_te with the new net
    python tools/train.py kitti2015 fast -a train_all -data_root /data -out out   # 14 epochs on nnz_tr + nnz_te, then submit

Option names and defaults are main.lua's (-gpu is 1-based as there): the network and training options (-l1 -fm -ks -lr -bs
-mom -true1 -false1 -false2 -m -pow), the augmentation options (-hflip ... -d_contrast) and the stereo method's overrides of
run_main.py (-L1 ... -blur_t) for the evaluation that follows.  The net goes to <data_root>/net/net_<cmd_str>.t7, named from
main.lua's arguments.  Everything the trainer does not implement is refused before any GPU work; see mc-cnn_b200/train.py.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from run_main import PRESET_OPTIONS, _flag  # noqa: E402

TOOL_ONLY = ("-data_root", "-out")


def parser():
    from mccnn_b200 import train

    ap = argparse.ArgumentParser(prog="train.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    ap.add_argument("arch", choices=("fast", "slow", "ad", "census"))
    ap.add_argument("-a", default="train_tr")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    ap.add_argument("-seed", type=int, default=42)
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-out", default="out")
    ap.add_argument("-subset", type=float, default=1)
    ap.add_argument("-debug", nargs="?", const=True, default=False, type=_flag)
    for name, v in dict(train.AUGMENT, **train.NET).items():
        ap.add_argument("-" + name, type=type(v), default=None)
    for name, typ in PRESET_OPTIONS.items():
        ap.add_argument("-" + name, type=typ, default=None)
    return ap


def main_args(argv):
    """main.lua's arguments after dataset and arch, without this tool's own options (for cmd_str)"""
    out, skip = [], False
    for a in argv[2:]:
        if skip:
            skip = False
        elif a in TOOL_ONLY:
            skip = True
        elif not a.startswith(TOOL_ONLY):
            out.append(a)
    return out


def parse_args(argv=None):
    """-> (namespace, training options, stereo overrides).  Refuses what the trainer does not implement."""
    from mccnn_b200 import train

    argv = list(sys.argv[1:] if argv is None else argv)
    args = parser().parse_args(argv)
    if args.a not in ("train_tr", "train_all"):
        raise SystemExit("train.py: -a %s is not a training action (train_tr, train_all); see run_main.py" % args.a)
    if args.gpu < 1:
        raise SystemExit("train.py: -gpu is 1-based")
    if args.subset < 1:
        raise SystemExit("train.py: -subset %s is not supported (the whole training set is used)" % args.subset)
    if args.debug:
        raise SystemExit("train.py: -debug (a net file per epoch) is not supported")
    given = {k: getattr(args, k) for k in dict(train.AUGMENT, **train.NET) if getattr(args, k) is not None}
    try:
        o = train.options(args.dataset, args.arch, **given)
    except ValueError as e:
        raise SystemExit("train.py: %s" % e)
    stereo = {k: getattr(args, k) for k in PRESET_OPTIONS if getattr(args, k) is not None}
    args.device = args.gpu - 1
    args.argv = argv
    return args, o, stereo


def main(argv=None):
    args, o, stereo = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import train

    fname = train.net_path(args.data_root, args.dataset, main_args(args.argv))
    if os.path.exists(fname):
        raise SystemExit("train.py: %s already exists; remove it first" % fname)
    print(" ".join(args.argv) + " ", flush=True)                                  # main.lua:6-9
    train.train(args.dataset, args.a, o, args=main_args(args.argv), data_root=args.data_root, seed=args.seed,
                device=args.device, out=args.out, stereo=stereo, log=lambda s: print(s, flush=True))
    return 0


if __name__ == "__main__":
    sys.exit(main())
