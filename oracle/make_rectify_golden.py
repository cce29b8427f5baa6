"""Build tests/golden/rectify.npz and the OpenCV FileStorage fixtures tests/golden/rectify_intrinsics.yml /
rectify_extrinsics.yml from OpenCV itself (cv2, CPU only) -- TEST INFRASTRUCTURE, run where cv2 imports:

    python oracle/make_rectify_golden.py

Three cameras (DESIGN §22), each with K, D, R, P, size and rect_size:
* ``kitti``: KITTI-like, 1392 x 512 raw, 1242 x 375 rectified, 5 coefficients (k1 about -0.37), a small R_rect;
* ``rational``: 8 coefficients (OpenCV's rational model), 640 x 480 both;
* ``alpha1``: 4 coefficients, 160 x 120, P from cv2.stereoRectify with alpha = 1, so part of the rectified grid falls
  outside the raw image.
For each, ``<cam>_mapx`` / ``<cam>_mapy`` are cv2.initUndistortRectifyMap's float coordinates at every STEP-th row and
column of the rectified grid (``<cam>_rows`` / ``<cam>_cols``).  For ``alpha1`` also ``alpha1_tex``, a seeded
high-contrast random texture of the raw size, and ``alpha1_remap``, cv2.remap of it with the full maps, INTER_LINEAR and
BORDER_REPLICATE.  The YAML pair is stereo_calib's layout (M1 D1 M2 D2 / R T R1 R2 P1 P2 Q) of the ``alpha1`` rig.
"""
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(_HERE), "tests", "golden")
STEP = 8


def _rot(rx, ry, rz):
    import cv2

    return cv2.Rodrigues(np.array([rx, ry, rz], np.float64))[0]


def cameras():
    import cv2

    out = {}
    K = np.array([[959.791, 0, 696.0217], [0, 956.9251, 224.1806], [0, 0, 1]])
    D = np.array([-0.3691481, 0.1968681, 0.001353473, 0.0005677587, -0.06770705])
    P = np.array([[721.5377, 0, 609.5593, 0], [0, 721.5377, 172.854, 0], [0, 0, 1, 0]])
    out["kitti"] = (K, D, _rot(0.0017, -0.0099, 0.0043), P, (1392, 512), (1242, 375))
    K = np.array([[512.0, 0, 321.3], [0, 508.5, 238.7], [0, 0, 1]])
    D = np.array([0.11, -0.05, 0.0012, -0.0007, 0.012, 0.13, -0.04, 0.016])
    P = np.array([[480.0, 0, 318.0, 0], [0, 480.0, 241.0, 0], [0, 0, 1, 0]])
    out["rational"] = (K, D, _rot(0.004, 0.012, -0.006), P, (640, 480), (640, 480))
    K1 = np.array([[150.0, 0, 81.0], [0, 149.0, 58.5], [0, 0, 1]])
    K2 = np.array([[151.5, 0, 78.5], [0, 150.0, 61.0], [0, 0, 1]])
    D1 = np.array([-0.21, 0.06, 0.0015, -0.001])
    D2 = np.array([-0.19, 0.05, -0.001, 0.0012])
    Rs, T = _rot(0.01, -0.03, 0.008), np.array([-0.12, 0.002, 0.001])
    size = (160, 120)
    R1, R2, P1, P2, Q, _, _ = cv2.stereoRectify(K1, D1, K2, D2, size, Rs, T, alpha=1.0)
    out["alpha1"] = (K1, D1, R1, P1, size, size)
    return out, dict(M1=K1, D1=D1, M2=K2, D2=D2, R=Rs, T=T, R1=R1, R2=R2, P1=P1, P2=P2, Q=Q)


def main():
    import cv2

    cams, rig = cameras()
    arrays = {}
    for name, (K, D, R, P, size, rect_size) in cams.items():
        mx, my = cv2.initUndistortRectifyMap(K, D, R, P, rect_size, cv2.CV_32FC1)
        rows, cols = np.arange(0, rect_size[1], STEP), np.arange(0, rect_size[0], STEP)
        arrays.update({name + "_K": K.reshape(-1), name + "_D": D, name + "_R": R.reshape(-1), name + "_P": P.reshape(-1),
                       name + "_size": np.array(size), name + "_rect_size": np.array(rect_size), name + "_rows": rows,
                       name + "_cols": cols, name + "_mapx": mx[np.ix_(rows, cols)], name + "_mapy": my[np.ix_(rows, cols)]})
        if name == "alpha1":
            rng = np.random.default_rng(0)
            tex = np.kron(rng.integers(0, 256, (size[1] // 2, size[0] // 2)), np.ones((2, 2), np.int64)).astype(np.uint8)
            arrays["alpha1_tex"] = tex
            arrays["alpha1_remap"] = cv2.remap(tex, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE)
    np.savez_compressed(os.path.join(GOLDEN, "rectify.npz"), **arrays)
    for fname, keys in (("rectify_intrinsics.yml", ("M1", "D1", "M2", "D2")),
                        ("rectify_extrinsics.yml", ("R", "T", "R1", "R2", "P1", "P2", "Q"))):
        fs = cv2.FileStorage(os.path.join(GOLDEN, fname), cv2.FILE_STORAGE_WRITE)
        for k in keys:
            fs.write(k, rig[k] if rig[k].ndim == 2 else rig[k].reshape(1, -1))
        fs.release()


if __name__ == "__main__":
    main()
