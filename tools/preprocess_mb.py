"""preprocess_mb.py: the raw Middlebury sets, unpacked, into main.lua's data.mb.<rect>_<color> layout.

    python tools/preprocess_mb.py imperfect gray -data_root /data     # /data/data.mb/unzip -> /data/data.mb.imperfect_gray
    python tools/preprocess_mb.py perfect rgb -gpu 2

Expects ``<data_root>/data.mb/unzip/vision.middlebury.edu/stereo/data/scenes{2014,2006,2005,2003,2001}/...`` and
``<data_root>/data.mb/unzip/MiddEval3/{trainingH,testH}`` as the archives unpack, and writes x_<i>_<j>, dispnoc<i>, meta,
nnz_tr, nnz_te, te (.bin + .dim + .type) and fname_submit.txt to ``<data_root>/data.mb.<rect>_<color>/``.  -gpu is 1-based,
as in main.lua; the per-pixel work runs there.  Prints what the script prints.  Refuses to overwrite existing outputs.  See
mc-cnn_b200/preprocess.py for what is computed and where it deliberately differs from the script.
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="preprocess_mb.py", description=__doc__.splitlines()[0])
    ap.add_argument("rect", choices=("perfect", "imperfect"))
    ap.add_argument("color", choices=("gray", "rgb"))
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def main(argv=None):
    args = parser().parse_args(argv)
    if args.gpu < 1:
        raise SystemExit("preprocess_mb.py: -gpu is 1-based")
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import preprocess

    t0 = time.perf_counter()
    preprocess.preprocess_mb(args.data_root, args.rect, args.color, device=args.gpu - 1, log=print)
    sys.stderr.write("preprocess_mb.py: %.2f s\n" % (time.perf_counter() - t0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
