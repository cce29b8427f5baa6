"""numpy restatement of DESIGN §21's projection rule (mccnn_velo_depth_map): a LiDAR scan into a sparse depth map.

Each point, in float32 with every operation rounded once: x' = ((P00 x + P01 y) + P02 z) + P03, likewise y' (row 1) and z'
(row 2); kept when min_depth < z' < inf; pixel u = rint(x' / z') - 1, v = rint(y' / z') - 1 (ties to even), kept inside
the image; each pixel the smallest z' of its points, 0 where none."""
import numpy as np


def project(pts, P):
    """(z', u, v, kept) of every point; u, v as float32 before the image test"""
    pts = np.asarray(pts, np.float32).reshape(-1, 4)
    P = np.asarray(P, np.float64).reshape(3, 4).astype(np.float32)
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    with np.errstate(all="ignore"):
        r = [((P[i, 0] * x + P[i, 1] * y) + P[i, 2] * z) + P[i, 3] for i in range(3)]
        zc = r[2]
        u = np.rint(r[0] / zc) - np.float32(1)
        v = np.rint(r[1] / zc) - np.float32(1)
    return zc, u, v


def velo_depth_map(pts, P, H, W, min_depth):
    """the (H, W) float32 map: a scatter-min of the kept points, in index order"""
    zc, u, v = project(pts, P)
    with np.errstate(invalid="ignore"):
        keep = (zc > np.float32(min_depth)) & (zc < np.inf) & (u >= 0) & (u < W) & (v >= 0) & (v < H)
    out = np.full(H * W, np.inf, np.float32)
    idx = v[keep].astype(np.int64) * W + u[keep].astype(np.int64)
    np.minimum.at(out, idx, zc[keep])
    out[np.isinf(out)] = 0
    return out.reshape(H, W)


def brute_force(pts, P, H, W, min_depth):
    """the same map pixel by pixel: the minimum over the points that land on it"""
    zc, u, v = project(pts, P)
    out = np.zeros((H, W), np.float32)
    for y in range(H):
        for x in range(W):
            with np.errstate(invalid="ignore"):
                m = (u == x) & (v == y) & (zc > np.float32(min_depth)) & (zc < np.inf)
            if m.any():
                out[y, x] = zc[m].min()
    return out
