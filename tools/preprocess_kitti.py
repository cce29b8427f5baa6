"""preprocess_kitti.lua: the raw KITTI 2012 / 2015 archives, unpacked, into main.lua's data layout.

    python tools/preprocess_kitti.py both -data_root /data      # /data/data.kitti/unzip -> /data/data.kitti/*.bin, same for 2015
    python tools/preprocess_kitti.py kitti2015 -gpu 2

Expects ``<data_root>/data.kitti/unzip/{training,testing}/...`` and ``<data_root>/data.kitti2015/unzip/...`` as the archives
unpack and writes x0, x1, dispnoc, metadata, tr, te, nnz_tr and nnz_te (.bin + .dim + .type) next to ``unzip/``.  -gpu is
1-based, as in main.lua; the training-sample lists are computed there.  Prints what the script prints.  Refuses to overwrite
existing outputs.  See mc-cnn_b200/preprocess.py for what is computed and where it deliberately differs from the script.
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DATASETS = {"kitti": ("kitti",), "kitti2015": ("kitti2015",), "both": ("kitti", "kitti2015")}


def parser():
    ap = argparse.ArgumentParser(prog="preprocess_kitti.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=tuple(DATASETS))
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def main(argv=None):
    args = parser().parse_args(argv)
    if args.gpu < 1:
        raise SystemExit("preprocess_kitti.py: -gpu is 1-based")
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import preprocess

    for dataset in DATASETS[args.dataset]:                      # refuse before any work
        preprocess.check_outputs_absent(preprocess.output_dir(args.data_root, dataset))
    t0 = time.perf_counter()
    for dataset in DATASETS[args.dataset]:
        preprocess.preprocess_kitti(args.data_root, dataset, device=args.gpu - 1, log=print)
    sys.stderr.write("preprocess_kitti.py: %.2f s\n" % (time.perf_counter() - t0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
