"""Write rectified PNGs of raw stereo pairs, rectified on the GPU (an addition beyond the reference; DESIGN §22).

    python tools/rectify.py -left L.png -right R.png -rectify intrinsics.yml [-rectify extrinsics.yml] -out O
    python tools/rectify.py -drive /data/raw/2011_09_26/2011_09_26_drive_0001_extract -out O [-every k]

One pair (-left / -right with OpenCV FileStorage YAML files, the keys of run_main.py -rectify) writes O/left.png,
O/right.png and O/mask.png; an unrectified KITTI raw drive (its calibration from the date directory's
calib_cam_to_cam.txt) writes O/<drive>/image_00/data/%010d.png, image_01/data/%010d.png and mask/%010d.png per frame.  The
mask is 255 where the left view is valid and 0 elsewhere.  A non-empty output directory is refused.  -gpu is 1-based.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    """Refuses what cannot run before any GPU work."""
    ap = argparse.ArgumentParser(prog="rectify.py", description=__doc__.splitlines()[0])
    ap.add_argument("-left", default="")
    ap.add_argument("-right", default="")
    ap.add_argument("-rectify", action="append", default=[], help="an OpenCV FileStorage YAML file; repeatable")
    ap.add_argument("-drive", default="", help="an unrectified KITTI raw drive <date>/<date>_drive_<nnnn>_extract")
    ap.add_argument("-every", type=int, default=1)
    ap.add_argument("-out", required=True)
    ap.add_argument("-gpu", type=int, default=1)
    args = ap.parse_args(argv)
    pair = bool(args.left or args.right or args.rectify)
    if pair == bool(args.drive):
        raise SystemExit("rectify.py: give -left, -right and -rectify, or -drive")
    if pair:
        if not (args.left and args.right and args.rectify):
            raise SystemExit("rectify.py: a pair needs -left, -right and -rectify")
        for f in [args.left, args.right] + args.rectify:
            if not os.path.isfile(f):
                raise SystemExit("rectify.py: %s is not a file" % f)
    else:
        if not os.path.isdir(args.drive):
            raise SystemExit("rectify.py: %s is not a directory" % args.drive)
        if not os.path.basename(os.path.normpath(args.drive)).endswith("_extract"):
            raise SystemExit("rectify.py: %s is not an unrectified (_extract) drive" % args.drive)
    if args.every < 1:
        raise SystemExit("rectify.py: -every must be at least 1")
    if args.gpu < 1:
        raise SystemExit("rectify.py: -gpu is 1-based")
    if os.path.isdir(args.out) and os.listdir(args.out):
        raise SystemExit("rectify.py: output directory %s is not empty" % args.out)
    return args


def _save(t, path):
    from PIL import Image

    os.makedirs(os.path.dirname(path), exist_ok=True)
    a = t.cpu().numpy()
    Image.fromarray(a, "L" if a.ndim == 2 else "RGB").save(path, format="PNG")


def main(argv=None):
    args = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import dataio, frontend, predict_kitti, predict_raw
    from mccnn_b200.rectify import rectify

    dev = args.gpu - 1
    if args.drive:
        frames = predict_raw.drive_frames([args.drive], args.every)
        files = predict_raw.pair_files(frames)
        rects = predict_raw.read_rects(frames, predict_kitti.scan(files))       # every refusal before any GPU work
        for fr, (left, right, _), rect in zip(frames, files, rects):
            l2, r2, valid = rectify(frontend.load_bytes(left), frontend.load_bytes(right), rect, dev)
            base = os.path.join(args.out, predict_raw.drive_name(args.drive))
            name = "%010d.png" % fr.index
            _save(l2, os.path.join(base, "image_00", "data", name))
            _save(r2, os.path.join(base, "image_01", "data", name))
            _save(valid * 255, os.path.join(base, "mask", name))
        return 0
    H, W = predict_kitti.scan([(args.left, args.right, None)])[0]
    rect = dataio.read_rectification(args.rectify, "opencv", size=(W, H))
    l2, r2, valid = rectify(frontend.load_bytes(args.left), frontend.load_bytes(args.right), rect, dev)
    _save(l2, os.path.join(args.out, "left.png"))
    _save(r2, os.path.join(args.out, "right.png"))
    _save(valid * 255, os.path.join(args.out, "mask.png"))
    return 0


if __name__ == "__main__":
    sys.exit(main())
