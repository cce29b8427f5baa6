"""samples/bin2png.lua: left.png, right.png and disp.png from the left.bin, right.bin and disp.bin that -a predict writes.

    python tools/bin2png.py [DIR] [-disp_max 70] [-height 370] [-width 1226]

The defaults are the script's constants.  Each file's size must be what -disp_max, -height and -width make it (D*H*W*4
bytes, H*W*4 for disp.bin); otherwise nothing runs.  The images are drawn on the first GPU (mc-cnn_b200/render.py).
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    """-> namespace; refuses missing or mis-sized files before any GPU work"""
    ap = argparse.ArgumentParser(prog="bin2png.py", description=__doc__.splitlines()[0])
    ap.add_argument("dir", nargs="?", default=".")
    ap.add_argument("-disp_max", type=int, default=70)
    ap.add_argument("-height", type=int, default=370)
    ap.add_argument("-width", type=int, default=1226)
    args = ap.parse_args(argv)
    from mccnn_b200 import render

    try:
        render.check_bins(args.dir, args.disp_max, args.height, args.width)
    except ValueError as e:
        raise SystemExit("bin2png.py: %s" % e)
    return args


def main(argv=None):
    args = parse_args(argv)
    from mccnn_b200 import render

    render.bin2png(args.dir, disp_max=args.disp_max, height=args.height, width=args.width)
    return 0


if __name__ == "__main__":
    sys.exit(main())
