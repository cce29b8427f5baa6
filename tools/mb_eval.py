"""Score the MiddEval3 training scenes with the SDK's evaldisp metrics and the website's error quantiles, on the GPU.

    python tools/mb_eval.py predict fast -net_fname net/net_mb_fast_-a_train_all.t7 -data_root /data [-res F|H] [-out O] \\
        [-gpu 1]
    python tools/mb_eval.py predict census -data_root /data                  # -arch: fast, slow, census or ad
    python tools/mb_eval.py score O -data_root /data [-res F|H] [-alg MC-CNN-fst] [-gpu 1]

`predict` runs the net over the 15 ``MiddEval3/trainingH`` pairs of the raw tree (no preprocessed data.mb.* set needed) at
main.lua's mb preset and scores each map; with -out it also writes ``O/trainingH/<scene>/disp0<method>.pfm`` and
``time<method>.txt`` as ``-a submit`` does.  `score` scores such a directory (-alg picks ``disp0<ALG>.pfm`` when a scene
holds several).  Both print one tab-separated line per scene: its name, then for nonocc and then all: bad0.5, bad1, bad2,
bad4, invalid, avgerr, rms, A50, A90, A95, A99, coverage; then the line of means.  Rates are fractions.  The ground truth
is read from ``<data_root>/data.mb/unzip/MiddEval3/trainingF`` (-res F, the default, as the website scores) or
``trainingH`` (-res H): disp0GT.pfm and mask0nocc.png, from the SDK's MiddEval3-GT0-F.zip / -GT0-H.zip.  -gpu is 1-based
as in main.lua.  See mc-cnn_b200/mb_eval.py.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="mb_eval.py", description=__doc__.splitlines()[0])
    sub = ap.add_subparsers(dest="action", required=True)
    p = sub.add_parser("predict", help="run a net over the training pairs and score each map")
    p.add_argument("arch", choices=("fast", "slow", "census", "ad"))
    p.add_argument("-net_fname", default="")
    p.add_argument("-data_root", default=".")
    p.add_argument("-res", choices=("F", "H"), default="F")
    p.add_argument("-out", default=None, help="also write the maps here, in -a submit's layout")
    p.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    p.add_argument("-density", type=float, default=None,
                   help="keep this share of each map's pixels, the most confident ones, +inf elsewhere; in (0, 1]")
    s = sub.add_parser("score", help="score the maps of a directory in -a submit's layout")
    s.add_argument("out")
    s.add_argument("-data_root", default=".")
    s.add_argument("-res", choices=("F", "H"), default="F")
    s.add_argument("-alg", default=None, help="score disp0<ALG>.pfm")
    s.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def parse_args(argv=None):
    """Refuses what cannot run before any file or GPU is touched."""
    args = parser().parse_args(argv)
    if args.gpu < 1:
        raise SystemExit("mb_eval.py: -gpu is 1-based")
    if args.action == "predict":
        if args.arch in ("fast", "slow") and not args.net_fname:
            raise SystemExit("mb_eval.py: arch '%s' needs -net_fname" % args.arch)
        if args.density is not None and not 0 < args.density <= 1:
            raise SystemExit("mb_eval.py: -density must be in (0, 1]")
    elif not os.path.isdir(args.out):
        raise SystemExit("mb_eval.py: %s is not a directory" % args.out)
    return args


def main(argv=None):
    args = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import mb_eval

    if args.action == "predict":
        mb_eval.evaluate_training(args.arch, args.net_fname or None, data_root=args.data_root, res=args.res, out=args.out,
                                  device=args.gpu - 1, density=args.density)
    else:
        mb_eval.score_dir(args.out, data_root=args.data_root, res=args.res, alg=args.alg, device=args.gpu - 1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
