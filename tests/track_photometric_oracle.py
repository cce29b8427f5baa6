"""numpy restatement of joint photometric and point-to-plane tracking (mc-cnn_b200/track.py, csrc/track.cu), for
tests/test_track_photometric.py and tests/test_gpu_track_photometric.py.  Written from DESIGN §26:

* intensity: a (H, W) uint8 image as fp32, or ((R + G) + B) / 3 in fp32 of a (H, W, 3) one; level l + 1 is a centred
  [1/4 1/2 1/4] blur of level l sampled at even pixels, rows first (h = (L(2x-1) / 4 + L(2x) / 2) + L(2x+1) / 4, indices
  clamped), then columns the same way, in fp32; levels ceil(H / 2^l) x ceil(W / 2^l);
* gradients of the reference, float64 from the fp32 values: g_x = 0.5 (L(x+1, y) - L(x-1, y)) for 1 <= x <= w - 2,
  likewise g_y, NaN elsewhere;
* a pixel's photometric term: a source vertex p, q = R p + t, q_z > 0; the nearest model pixel (§25's step 3) holds a
  model vertex m with |q - m|^2 <= delta^2; x_l = ((q_x / q_z) f + cx) 2^-l (likewise y_l), x0 = floor(x_l), fx = x_l - x0,
  1 <= x0, x0 + 1 <= w_l - 2 (likewise y); I_r, g_x, g_y sampled bilinearly (along x, then y, each a + f (b - a));
  r = I_r - I_s; kept when g_x^2 + g_y^2 >= g_min^2 and |r| <= rho; with s = f 2^-l, a = g_x s / q_z, b = g_y s / q_z,
  c = -(a q_x + b q_y) / q_z, G = (a, b, c), J = (q x G, G); float64, one rounding per operation, in this order;
* the sums: §25's 28 terms per pixel and its tree (track_oracle.tree_sum), geometric then photometric.

The host side (the joint solve, the level loop) is the package's own track.run_icp and track.solve_joint."""
import importlib.util
import math
import os

import numpy as np


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(os.path.dirname(os.path.abspath(__file__)), name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


track_oracle = _load("track_oracle")
tsdf_oracle = track_oracle.tsdf_oracle
LEVELS = track_oracle.LEVELS


def intensity(img):
    """fp32 (H, W) intensity of a (H, W) or (H, W, 3) uint8 image"""
    a = np.asarray(img)
    if a.ndim == 2:
        return a.astype(np.float32)
    c = a.astype(np.float32)
    return ((c[..., 0] + c[..., 1]) + c[..., 2]) / np.float32(3.0)


def down(L):
    """the next level of fp32 level L: the [1/4 1/2 1/4] blur at even pixels, rows first, then columns"""
    h, w = L.shape
    q, half = np.float32(0.25), np.float32(0.5)
    x = 2 * np.arange(-(-w // 2))
    R = (q * L[:, np.clip(x - 1, 0, w - 1)] + half * L[:, x]) + q * L[:, np.clip(x + 1, 0, w - 1)]
    y = 2 * np.arange(-(-h // 2))
    return (q * R[np.clip(y - 1, 0, h - 1)] + half * R[y]) + q * R[np.clip(y + 1, 0, h - 1)]


def gradients(L):
    """(g_x, g_y) float64 of fp32 level L, NaN where undefined"""
    d = L.astype(np.float64)
    gx, gy = np.full(d.shape, np.nan), np.full(d.shape, np.nan)
    gx[:, 1:-1] = 0.5 * (d[:, 2:] - d[:, :-2])
    gy[1:-1, :] = 0.5 * (d[2:, :] - d[:-2, :])
    return gx, gy


def pyramid(img):
    """[(I fp32, g_x, g_y) per level] of an image"""
    out, L = [], intensity(img)
    for l in range(LEVELS):
        if l:
            L = down(L)
        out.append((L,) + gradients(L))
    return out


def _bilinear(P, x0, y0, fx, fy):
    P = P.astype(np.float64)
    h, w = P.shape
    x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)      # only kept pixels' values are used
    x0, y0 = np.minimum(x0, w - 1), np.minimum(y0, h - 1)
    a, b = P[y0, x0], P[y0, x1]
    c, d = P[y1, x0], P[y1, x1]
    top = a + fx * (b - a)
    bot = c + fx * (d - c)
    return top + fy * (bot - top)


def photometric_jacobian(src, mod, isrc, iref, cal, level, pose12, delta, g_min, rho):
    """([J_0 .. J_5, r], each (n,) float64 over the level's pixels in row-major order, 0 where skipped; (n,) inlier mask);
    src and mod are track_oracle pyramids, isrc and iref :func:`pyramid`s"""
    V = src[level][0]
    Vm = mod[level][0]
    _, hl, wl = V.shape
    p = V.reshape(3, -1)
    P = np.asarray(pose12, np.float64).reshape(3, 4)
    q = [((P[a, 0] * p[0] + P[a, 1] * p[1]) + P[a, 2] * p[2]) + P[a, 3] for a in range(3)]
    f, cx, cy = (float(np.float32(v)) for v in (cal.f, cal.cx, cal.cy))
    scale = math.ldexp(1.0, -level)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ok = ~np.isnan(p[0]) & (q[2] > 0)
        xs = ((q[0] / q[2]) * f + cx) * scale
        ys = ((q[1] / q[2]) * f + cy) * scale
        u, v = np.floor(xs + 0.5), np.floor(ys + 0.5)
        ok &= (u >= 0) & (u < wl) & (v >= 0) & (v < hl)
    j = np.where(ok, v, 0).astype(np.int64) * wl + np.where(ok, u, 0).astype(np.int64)
    m = Vm.reshape(3, -1)[:, j]
    ok &= ~np.isnan(m[0])
    d = [q[a] - m[a] for a in range(3)]
    with np.errstate(invalid="ignore", over="ignore"):
        ok &= ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) <= delta * delta
        x0, y0 = np.floor(xs), np.floor(ys)
        ok &= (x0 >= 1) & (x0 + 1 <= wl - 2) & (y0 >= 1) & (y0 + 1 <= hl - 2)
        fx, fy = xs - x0, ys - y0
    xi, yi = np.where(ok, x0, 1).astype(np.int64), np.where(ok, y0, 1).astype(np.int64)
    Ir, gxr, gyr = iref[level]
    Is = isrc[level][0].reshape(-1).astype(np.float64)
    s = f * scale
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        I = _bilinear(Ir, xi, yi, fx, fy)
        gx = _bilinear(gxr, xi, yi, fx, fy)
        gy = _bilinear(gyr, xi, yi, fx, fy)
        r = I - Is
        ok &= ((gx * gx + gy * gy) >= g_min * g_min) & (np.abs(r) <= rho)
        a = (gx * s) / q[2]
        b = (gy * s) / q[2]
        c = -(a * q[0] + b * q[1]) / q[2]
        J = [q[1] * c - q[2] * b, q[2] * a - q[0] * c, q[0] * b - q[1] * a, a, b, c, r]
    return [np.where(ok, x, 0.0) for x in J], ok


def photometric_terms(src, mod, isrc, iref, cal, level, pose12, delta, g_min, rho):
    """((n, 28) float64 photometric terms of the level's pixels in row-major order, (n,) inlier mask)"""
    J, ok = photometric_jacobian(src, mod, isrc, iref, cal, level, pose12, delta, g_min, rho)
    cols = [J[a] * J[b] for a in range(6) for b in range(a, 6)] + [J[a] * J[6] for a in range(6)] + [J[6] * J[6]]
    return np.stack(cols, 1), ok


def step(src, mod, isrc, iref, cal, level, pose12, delta, cos_t, g_min, rho):
    """(56 sums: geometric then photometric, geometric inliers, photometric inliers, the level's source vertices), as
    mccnn_track_step with gates {g_min, rho}"""
    tg, okg = track_oracle.terms(src, mod, cal, level, pose12, delta, cos_t)
    tp, okp = photometric_terms(src, mod, isrc, iref, cal, level, pose12, delta, g_min, rho)
    sums = np.concatenate([track_oracle.tree_sum(tg), track_oracle.tree_sum(tp)])
    return sums, int(okg.sum()), int(okp.sum()), int((~np.isnan(src[level][0][2])).sum())


def track(track_mod, disp, cal, Z, W_prev, W_pred, left, ref_left, photometric, rho=30.0, grad_min=2.0, max_depth=None,
          **params):
    """track_mod.Tracker(photometric=...).track's (pose, inliers, lost) from the numpy pyramids"""
    src, mod = track_oracle.source_pyramid(disp, cal, max_depth), track_oracle.model_pyramid(Z, cal)
    isrc, iref = pyramid(left), pyramid(ref_left)
    Wp, Wq = track_mod.as4(W_prev), track_mod.as4(W_pred)
    fn = lambda level, p12, delta, cos_t: step(src, mod, isrc, iref, cal, level, p12, delta, cos_t, grad_min, rho)
    T, inliers, lost = track_mod.run_icp(fn, track_mod.rigid_inv(Wp) @ Wq, photometric=photometric, **params)
    return (Wq if lost else Wp @ T), inliers, lost


def track_drive(track_mod, disps, imgs, cal, voxel, trunc=None, mode="track", oxts=None, max_depth=None, photometric=0.0,
                rho=30.0, grad_min=2.0):
    """fuse_drive's tracked loop with the photometric term over one drive's maps: (poses, lost frame indices, the Field);
    the reference image is the previous frame's, lost or not"""
    if not photometric:
        return track_oracle.track_drive(track_mod, disps, imgs, cal, voxel, trunc, mode, oxts, max_depth)
    field = tsdf_oracle.Field(voxel, trunc)
    poses, lost = [], []
    H, W = np.asarray(disps[0]).shape
    for k, (d, img) in enumerate(zip(disps, imgs)):
        if k == 0:
            pose = np.eye(4)
        else:
            Z = field.render(cal, poses[-1], H, W, 1, max_depth)
            pose, _, is_lost = track(track_mod, d, cal, Z, poses[-1], track_mod.predict(mode, poses, oxts), img, imgs[k - 1],
                                     photometric, rho, grad_min, max_depth)
            if is_lost:
                lost.append(k)
                poses.append(pose)
                continue
        field.add(d, cal, img, pose, max_depth)
        poses.append(pose)
    return poses, lost, field
