"""Time preprocess_mb's GPU stage on a full-size 2014 scene and the whole tool on the synthetic tree.

    python tools/time_preprocess_mb.py [--views 28] [--height 1988] [--width 2880]

1. One full-size 2014 scene on the device: --views seeded RGB views of height x width (28 = im0, im1, im1E, im1L and
   4 lights x 3 exposures x 2 cameras) halved (mccnn_mb_half_image), standardised (mccnn_mb_views,
   grey), and its three full-size maps halved, masked and listed (mccnn_mb_half_disp, _mask, _nnz_count / _fill).  Host
   clock around the stage, which ends by copying the views, dispnoc and the rows to the host; the first run is a warm-up,
   the median of five is reported, with torch's peak allocation.
2. tools/preprocess_mb.py imperfect gray on synth.write_mb_raw's tree: wall time of the process.
Prints one line per number with the card's name and power limit, read in the same run.
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
    ap.add_argument("--views", type=int, default=28)
    ap.add_argument("--height", type=int, default=1988)
    ap.add_argument("--width", type=int, default=2880)
    args = ap.parse_args(argv)

    import numpy as np
    import torch

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import preprocess, synth

    H, W = args.height, args.width
    rng = np.random.default_rng(0)
    v = synth.natural_image(rng, H // 4, W // 4)
    base = np.repeat(np.repeat(np.clip(np.rint(128 + 50 * v), 0, 255).astype(np.uint8), 4, 0), 4, 1)
    views = np.stack([np.stack([base + np.uint8(k + c) for c in range(3)], 2) for k in range(args.views)])
    d0 = np.repeat(np.repeat(rng.uniform(0, 200, (H // 16, W // 16)), 16, 0), 16, 1).astype(np.float32)
    d0[rng.random(d0.shape) < 0.1] = np.inf
    maps = np.stack([d0, synth._mb_right_map(rng, d0), rng.uniform(-0.7, 0.7, d0.shape).astype(np.float32)])

    def stage():
        x = torch.from_numpy(views).cuda()
        half = preprocess.mb_half_image(x)
        out = preprocess.mb_views(half, 1).cpu()
        m = preprocess.mb_half_disp(torch.from_numpy(maps).cuda())
        mask = preprocess.mb_mask(m[0], m[1], m[2])
        dispnoc, rows = preprocess.mb_nnz(m[0], mask, 1)
        return out, dispnoc.cpu(), rows.cpu()

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ts, n_rows = [], 0
    for _ in range(6):
        t0 = time.perf_counter()
        _, _, rows = stage()
        ts.append(time.perf_counter() - t0)
        n_rows = len(rows)
    t = sorted(ts[1:])
    print("card: %s" % card())
    print("gpu stage of one 2014 scene (%d views %dx%d halved and standardised, 3 maps halved, mask, lists; with the H2D "
          "of the bytes and the D2H of the results): median %.1f ms (min %.1f, max %.1f); rows %d"
          % (args.views, H, W, t[len(t) // 2] * 1e3, t[0] * 1e3, t[-1] * 1e3, n_rows))
    print("torch peak allocated during the stage: %.0f MB (the library's scratch comes on top: the fp32 row pass of the "
          "halving, %.0f MB here)" % (torch.cuda.max_memory_allocated() / 2 ** 20,
                                       args.views * H * (W // 2) * 3 * 4 / 2 ** 20))

    with tempfile.TemporaryDirectory() as root:
        synth.write_mb_raw(root)
        t0 = time.perf_counter()
        subprocess.check_call([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), "preprocess_mb.py"),
                               "imperfect", "gray", "-data_root", root], stdout=subprocess.DEVNULL)
        print("tools/preprocess_mb.py imperfect gray on synth.write_mb_raw's tree (49 images): %.2f s wall"
              % (time.perf_counter() - t0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
