"""Time the rectification of raw stereo pairs (mc-cnn_b200/rectify.py, DESIGN §22) on the GPU.

    python tools/time_rectify.py [--frames 8] [--arch census] [--disp_max 228] [--rounds 200] [--json out.json]

Reported: the median time of one mccnn_rectify_pair call (CUDA events around the call, the buffers allocated once) for a
1392 x 512 raw pair rectified to 1242 x 375, grey and RGB, with KITTI-like cameras; and the frames per second of
predict_raw -disp over a seeded synthetic unrectified drive of that size (synth.write_kitti_extract_drive) against a
_sync drive of the same rectified scenes, each timed over the whole drive after one warm-up pass.  The card's name and
power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, predict_raw, rectify, synth  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_confidence import card, timed  # noqa: E402

H, W, HRAW, WRAW = 375, 1242, 512, 1392


def kernel_ms(rect, nch, rounds, dev):
    """median ms of one mccnn_rectify_pair call on a random nch-channel raw pair"""
    rng = np.random.default_rng(0)
    shape = (HRAW, WRAW) if nch == 1 else (HRAW, WRAW, 3)
    l, r = (torch.from_numpy(rng.integers(0, 256, shape).astype(np.uint8)).to(dev) for _ in range(2))
    tail = () if nch == 1 else (3,)
    ol, orr = (torch.empty((H, W) + tail, dtype=torch.uint8, device=dev) for _ in range(2))
    valid = torch.empty((H, W), dtype=torch.uint8, device=dev)
    pl, pr = rectify.params(rect.left), rectify.params(rect.right)
    lib, s = adcensus.lib(), adcensus._stream(valid)

    def call():
        adcensus._check(lib.mccnn_rectify_pair(l.data_ptr(), r.data_ptr(), nch, HRAW, WRAW, pl.ctypes.data, pr.ctypes.data,
                                               H, W, ol.data_ptr(), orr.data_ptr(), valid.data_ptr(), s),
                        "mccnn_rectify_pair")

    for _ in range(10):
        call()
    torch.cuda.synchronize()
    return statistics.median(timed(call) for _ in range(rounds))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--arch", default="census", choices=("census", "ad"))
    ap.add_argument("--disp_max", type=int, default=228)
    ap.add_argument("--rounds", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    name, power = card()
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        ext, _, sync = synth.write_kitti_extract_drive(tmp, n=a.frames, H=H, W=W, Hraw=HRAW, Wraw=WRAW, seed=0, sync=True)
        rect = dataio.read_rectification(os.path.dirname(ext), "kitti_raw")
        out = {"card": name, "power_limit": power, "raw": [HRAW, WRAW], "rect": [H, W], "arch": a.arch,
               "disp_max": a.disp_max, "frames": a.frames}
        out["rectify_grey_ms"] = kernel_ms(rect, 1, a.rounds, dev)
        out["rectify_rgb_ms"] = kernel_ms(rect, 3, a.rounds, dev)

        def loop(drive, tag):
            t0 = time.perf_counter()
            predict_raw.predict_raw("kitti", a.arch, [drive], out=os.path.join(tmp, tag), disp=True, disp_max=a.disp_max,
                                    device=0, verbose=False)
            return time.perf_counter() - t0

        loop(sync, "warm_sync")
        loop(ext, "warm_extract")
        t_sync, t_ext = loop(sync, "sync"), loop(ext, "extract")
    out["sync_fps"], out["extract_fps"] = a.frames / t_sync, a.frames / t_ext
    print("card: %s, power limit %s" % (name, power))
    print("mccnn_rectify_pair %dx%d -> %dx%d: grey %.4f ms, RGB %.4f ms per pair (median of %d)"
          % (HRAW, WRAW, H, W, out["rectify_grey_ms"], out["rectify_rgb_ms"], a.rounds))
    print("predict_raw -disp %s D %d, %d frames: _sync %.2f frames/s, _extract %.2f frames/s"
          % (a.arch, a.disp_max, a.frames, out["sync_fps"], out["extract_fps"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
