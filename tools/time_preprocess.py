"""Time preprocess_kitti's GPU stage and the whole tool.

    python tools/time_preprocess.py [--maps 194] [--tree-images 41] [--out DIR]

1. The sample lists (mccnn_kitti_nnz_count + _fill, the cleaning included) for a stack of --maps seeded 350 x 1242 maps in
   readPNG16's domain, with their left images on the device: host clock around the call, which ends by copying the two
   lists to the host (so after a device synchronise); the first call is a warm-up, the median of five is reported.
2. tools/preprocess_kitti.py kitti on a synthetic raw tree of --tree-images training images (375 x 1242) plus 2 testing
   images: wall time of the process.
Prints one line per number with the card's name and power limit.
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:                                   # noqa: BLE001 -- the card's name is informative only
        import torch

        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=194)
    ap.add_argument("--tree-images", type=int, default=41)
    args = ap.parse_args(argv)

    import numpy as np
    import torch

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import preprocess, synth
    from oracle import make_preprocess_golden as mpg

    rng = np.random.default_rng(0)
    y = mpg.png16(rng, (args.maps, 1, 350, 1242), dmax=200)
    x0 = rng.standard_normal(y.shape).astype(np.float32)
    is_te = np.zeros(args.maps, bool)
    is_te[rng.permutation(args.maps)[:40]] = True
    disp, x0d = torch.from_numpy(y).cuda(), torch.from_numpy(x0).cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    free0 = torch.cuda.mem_get_info()[0]
    ts, rows = [], None
    for _ in range(6):
        t0 = time.perf_counter()
        tr, te = preprocess.kitti_nnz(disp, x0d, is_te)
        tr, te = tr.cpu(), te.cpu()
        ts.append(time.perf_counter() - t0)
        rows = (len(tr), len(te))
    med = sorted(ts[1:])[len(ts[1:]) // 2]
    print("card: %s" % card())
    print("gpu stage (count + fill + D2H of the lists), %d maps 350x1242: median %.2f ms (min %.2f, max %.2f); rows tr %d, "
          "te %d" % (args.maps, med * 1e3, min(ts[1:]) * 1e3, max(ts[1:]) * 1e3, rows[0], rows[1]))
    print("torch peak allocated during the stage (maps, images and lists; the library's scratch is 12 bytes per row on "
          "top): %.1f MB; device free memory before: %.0f MB" % (torch.cuda.max_memory_allocated() / 2 ** 20, free0 / 2 ** 20))
    del disp, x0d

    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        synth.write_kitti_raw(root, "kitti", n_tr=args.tree_images, n_te=2, H=375, seed=1)
        t_synth = time.perf_counter() - t0
        t0 = time.perf_counter()
        subprocess.check_call([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), "preprocess_kitti.py"),
                               "kitti", "-data_root", root], stdout=subprocess.DEVNULL)
        t_tool = time.perf_counter() - t0
    print("tools/preprocess_kitti.py kitti on a synthetic tree of %d + 2 images 375x1242: %.2f s wall (writing the tree "
          "took %.2f s)" % (args.tree_images, t_tool, t_synth))
    return 0


if __name__ == "__main__":
    sys.exit(main())
