"""numpy restatement of frame-to-model tracking (mc-cnn_b200/track.py, csrc/track.cu), for tests/test_track.py and
tests/test_gpu_track.py.  Written from DESIGN §25:

* levels: level l keeps the pixels (2^l x, 2^l y), ceil(H / 2^l) x ceil(W / 2^l);
* vertices: the source's from its disparity by depth_oracle's fp32 rule (max_depth included), the model's from its fp32
  depth (NaN = none) with X and Y of the same rule, promoted to float64;
* normals: n = (V(x+1, y) - V) x (V(x, y+1) - V), normalised, negated when n . V > 0, float64 with one rounding per
  operation, invalid when a vertex is missing or |n| is not finite and > 0;
* a step: q = R p + t, n' = R n; q_z > 0; u = floor((((q_x / q_z) f + cx) 2^-l) + 0.5), likewise v; the model's vertex m
  and normal n_m there; d = q - m, kept when d . d <= delta^2 and n' . n_m >= cos theta; r = n_m . d, J = (q x n_m, n_m);
  28 terms per pixel (J_a J_b for a <= b row by row, J_a r, r^2), +0.0 for a skipped pixel;
* the sum: chunks of 1024 pixels in row-major order, zero-padded, each reduced by stride halving (a[i] += a[i + s], s =
  512 .. 1); the chunk sums zero-padded to a power of two and reduced the same way.

The host side (solve, update, the level loop, the prediction) is the package's own track.run_icp and track.predict."""
import importlib.util
import math
import os

import numpy as np


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(os.path.dirname(os.path.abspath(__file__)), name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


depth_oracle = _load("depth_oracle")
tsdf_oracle = _load("tsdf_oracle")

LEVELS = 3
CHUNK = 1024


def level_shape(H, W, l):
    return -(-H // (1 << l)), -(-W // (1 << l))


def normals(V):
    """(3, h, w) float64 normals of (3, h, w) vertices, NaN where invalid"""
    _, h, w = V.shape
    N = np.full(V.shape, np.nan)
    if h < 2 or w < 2:
        return N
    p = V[:, :-1, :-1]
    a = V[:, :-1, 1:] - p
    b = V[:, 1:, :-1] - p
    c = np.stack([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])
    with np.errstate(invalid="ignore", over="ignore"):
        ln = np.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2])
        ok = (ln > 0) & (ln <= np.finfo(np.float64).max)
        n = c / np.where(ok, ln, 1.0)
        dot = (n[0] * p[0] + n[1] * p[1]) + n[2] * p[2]
    n = np.where(dot > 0, -n, n)
    N[:, :-1, :-1] = np.where(ok, n, np.nan)
    return N


def pyramid(Z, X, Y):
    """[(V, N) per level] of full-resolution fp32 maps, NaN Z = no vertex"""
    out = []
    for l in range(LEVELS):
        s = 1 << l
        z = Z[::s, ::s]
        ok = ~np.isnan(z)
        V = np.stack([np.where(ok, X[::s, ::s], np.nan), np.where(ok, Y[::s, ::s], np.nan), np.where(ok, z, np.nan)]).astype(np.float64)
        out.append((V, normals(V)))
    return out


def source_pyramid(disp, cal, max_depth=None):
    return pyramid(*depth_oracle.depth32(disp, cal, max_depth))


def model_pyramid(Z, cal):
    Z = np.asarray(Z, np.float32)
    H, W = Z.shape
    f, cx, cy = np.float32(cal.f), np.float32(cal.cx), np.float32(cal.cy)
    x = np.arange(W, dtype=np.float32)[None, :]
    y = np.arange(H, dtype=np.float32)[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        X = ((x - cx) * Z) / f
        Y = ((y - cy) * Z) / f
    return pyramid(Z, X.astype(np.float32), Y.astype(np.float32))


def terms(src, mod, cal, level, pose12, delta, cos_t):
    """((n, 28) float64 terms of the level's pixels in row-major order, (n,) inlier mask)"""
    V, N = src[level]
    Vm, Nm = mod[level]
    _, hl, wl = V.shape
    p, ns = V.reshape(3, -1), N.reshape(3, -1)
    P = np.asarray(pose12, np.float64).reshape(3, 4)
    q = [((P[a, 0] * p[0] + P[a, 1] * p[1]) + P[a, 2] * p[2]) + P[a, 3] for a in range(3)]
    nr = [(P[a, 0] * ns[0] + P[a, 1] * ns[1]) + P[a, 2] * ns[2] for a in range(3)]
    f, cx, cy = (float(np.float32(v)) for v in (cal.f, cal.cx, cal.cy))
    scale = math.ldexp(1.0, -level)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ok = ~np.isnan(ns[0]) & (q[2] > 0)
        u = np.floor((((q[0] / q[2]) * f + cx) * scale) + 0.5)
        v = np.floor((((q[1] / q[2]) * f + cy) * scale) + 0.5)
        ok &= (u >= 0) & (u < wl) & (v >= 0) & (v < hl)
    j = np.where(ok, v, 0).astype(np.int64) * wl + np.where(ok, u, 0).astype(np.int64)
    m, nm = Vm.reshape(3, -1)[:, j], Nm.reshape(3, -1)[:, j]
    ok &= ~np.isnan(nm[0])
    d = [q[a] - m[a] for a in range(3)]
    with np.errstate(invalid="ignore", over="ignore"):
        dd = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
        c = (nr[0] * nm[0] + nr[1] * nm[1]) + nr[2] * nm[2]
        ok &= (dd <= delta * delta) & (c >= cos_t)
        J = [q[1] * nm[2] - q[2] * nm[1], q[2] * nm[0] - q[0] * nm[2], q[0] * nm[1] - q[1] * nm[0], nm[0], nm[1], nm[2],
             (nm[0] * d[0] + nm[1] * d[1]) + nm[2] * d[2]]
    J = [np.where(ok, x, 0.0) for x in J]
    cols = [J[a] * J[b] for a in range(6) for b in range(a, 6)] + [J[a] * J[6] for a in range(6)] + [J[6] * J[6]]
    return np.stack(cols, 1), ok


def halve(a):
    """stride halving over axis 1 (a power of two long) down to one element"""
    while a.shape[1] > 1:
        h = a.shape[1] // 2
        a = a[:, :h] + a[:, h:]
    return a[:, 0]


def tree_sum(t):
    """the 28 sums of (n, 28) terms in the fixed tree"""
    n = len(t)
    nch = max(1, -(-n // CHUNK))
    a = np.zeros((nch * CHUNK, t.shape[1]))
    a[:n] = t
    chunk = halve(a.reshape(nch, CHUNK, -1))
    P = 1
    while P < nch:
        P *= 2
    b = np.zeros((P, t.shape[1]))
    b[:nch] = chunk
    return halve(b[None])[0]


def step(src, mod, cal, level, pose12, delta, cos_t):
    """(28 sums, inliers, 0 photometric inliers, the level's source vertices), as mccnn_track_step without gates"""
    t, ok = terms(src, mod, cal, level, pose12, delta, cos_t)
    return tree_sum(t), int(ok.sum()), 0, int((~np.isnan(src[level][0][2])).sum())


def track(track_mod, disp, cal, Z, W_prev, W_pred, max_depth=None, **params):
    """track_mod.Tracker.track's (pose, inliers, lost) from the numpy pyramids"""
    src, mod = source_pyramid(disp, cal, max_depth), model_pyramid(Z, cal)
    Wp, Wq = track_mod.as4(W_prev), track_mod.as4(W_pred)
    fn = lambda level, p12, delta, cos_t: step(src, mod, cal, level, p12, delta, cos_t)
    T, inliers, lost = track_mod.run_icp(fn, track_mod.rigid_inv(Wp) @ Wq, **params)
    return (Wq if lost else Wp @ T), inliers, lost


def track_drive(track_mod, disps, imgs, cal, voxel, trunc=None, mode="track", oxts=None, max_depth=None, **params):
    """fuse_drive's loop with poses 'track' or 'refine' over one drive's maps: (poses, lost frame indices, the Field)"""
    field = tsdf_oracle.Field(voxel, trunc)
    poses, lost = [], []
    H, W = np.asarray(disps[0]).shape
    for k, (d, img) in enumerate(zip(disps, imgs)):
        if k == 0:
            pose = np.eye(4)
        else:
            Z = field.render(cal, poses[-1], H, W, 1, max_depth)
            pose, _, is_lost = track(track_mod, d, cal, Z, poses[-1], track_mod.predict(mode, poses, oxts), max_depth, **params)
            if is_lost:
                lost.append(k)
                poses.append(pose)
                continue
        field.add(d, cal, img, pose, max_depth)
        poses.append(pose)
    return poses, lost, field
