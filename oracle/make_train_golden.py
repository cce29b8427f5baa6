"""Write tests/golden/train/warp.npz: OpenCV's own cubic warps of make_patch (main.lua:607-619) -- TEST INFRASTRUCTURE.

    python oracle/make_train_golden.py          # needs cv2 (4.x); the reference called OpenCV 2.4's C API (unpinned)

Each case is ``cv2.warpAffine(src, M, (ws, ws), flags=INTER_CUBIC, borderMode=BORDER_CONSTANT, borderValue=0)`` of one float32
source with a float32 matrix built by make_patch's mul32 chain: patches inside the image, partly and wholly outside it,
rotation, shear, horizontal and vertical flips, fractional columns and ws = 9 and 11.
"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import train as ot  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "train", "warp.npz")


def cases(rng, H, W):
    out = []
    for k in range(400):
        ws = 9 if k % 4 else 11
        kind = k % 5
        if kind == 0:                                        # inside
            dim3, dim4 = rng.uniform(8, H - 8), rng.uniform(8, W - 8)
        elif kind == 1:                                      # across an edge
            dim3, dim4 = rng.choice([rng.uniform(-4, 4), rng.uniform(H - 4, H + 4)]), rng.uniform(-4, W + 4)
        elif kind == 2:                                      # wholly outside
            dim3, dim4 = rng.uniform(-30, -12), rng.uniform(W + 12, W + 30)
        else:                                                # anywhere, fractional columns
            dim3, dim4 = rng.uniform(-6, H + 6), rng.integers(0, W) + rng.uniform(0, 1)
        s = rng.uniform(0.8, 1)
        scale = [s * rng.uniform(0.9, 1) * (-1 if k % 7 == 0 else 1), s * (-1 if k % 11 == 0 else 1)]
        phi = rng.uniform(-7, 7) * math.pi / 180
        trans = [rng.uniform(-1, 1) * (k % 3 == 0), rng.uniform(-1, 1) * (k % 3 == 1)]
        m = ot.patch_matrix(ws, dim3, dim4 - rng.uniform(0, 60) * (k % 2), scale, phi, trans, rng.uniform(-0.3, 0.3))
        out.append((ws, m))
    return out


def main():
    import cv2

    rng = np.random.default_rng(20151212)
    H, W = 48, 96
    src = rng.standard_normal((H, W)).astype(np.float32)
    cs = cases(rng, H, W)
    ws = np.array([c[0] for c in cs], np.int32)
    m = np.stack([c[1] for c in cs])
    out = np.zeros((len(cs), 11, 11), np.float32)
    for i, (w, mi) in enumerate(cs):
        out[i, :w, :w] = cv2.warpAffine(src, mi.reshape(2, 3), (w, w), flags=cv2.INTER_CUBIC,
                                        borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, src=src, ws=ws, m=m, out=out, cv2_version=np.array(cv2.__version__))
    print("%s: %d cases (OpenCV %s)" % (OUT, len(cs), cv2.__version__))


if __name__ == "__main__":
    main()
