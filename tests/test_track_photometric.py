"""CPU: the photometric term of tracking (DESIGN §26) -- the numpy restatement (tests/track_photometric_oracle.py) against
a loop of one operation at a time, its Jacobian against finite differences, the joint solve, the street scene's
degeneracy that the term removes, the synthetic drive's defaults, and every refusal before any GPU work."""
import hashlib
import importlib.util
import math
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, fusion, synth, track

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


po = _load("track_photometric_oracle", "tests", "track_photometric_oracle.py")
to = po.track_oracle
fuse_tool = _load("fuse_raw_tool_track_photometric", "tools", "fuse_raw.py")


def _f32(v):
    return float(np.float32(v))


def _brute_pyramid(img):
    """the intensity pyramid and gradients, one Python-float operation at a time (fp32 rounding by np.float32)"""
    a = np.asarray(img)
    H, W = a.shape[:2]
    L = [[_f32(a[y, x]) if a.ndim == 2 else
          _f32(_f32(_f32(_f32(a[y, x, 0]) + _f32(a[y, x, 1])) + _f32(a[y, x, 2])) / 3.0) for x in range(W)] for y in range(H)]
    out = []
    for l in range(3):
        if l:
            h, w = len(L), len(L[0])
            h2, w2 = -(-h // 2), -(-w // 2)
            blur = lambda v0, v1, v2: _f32(_f32(_f32(0.25 * v0) + _f32(0.5 * v1)) + _f32(0.25 * v2))
            R = [[blur(L[y][max(2 * x - 1, 0)], L[y][2 * x], L[y][min(2 * x + 1, w - 1)]) for x in range(w2)] for y in range(h)]
            L = [[blur(R[max(2 * y - 1, 0)][x], R[2 * y][x], R[min(2 * y + 1, h - 1)][x]) for x in range(w2)] for y in range(h2)]
        h, w = len(L), len(L[0])
        gx = [[0.5 * (L[y][x + 1] - L[y][x - 1]) if 1 <= x <= w - 2 else math.nan for x in range(w)] for y in range(h)]
        gy = [[0.5 * (L[y + 1][x] - L[y - 1][x]) if 1 <= y <= h - 2 else math.nan for x in range(w)] for y in range(h)]
        out.append((np.array(L, np.float32), np.array(gx), np.array(gy)))
    return out


def same_bits(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, what
    assert np.array_equal(np.isnan(a), np.isnan(b)), "%s: NaN patterns differ" % what
    assert np.array_equal(a.view(np.uint64)[~np.isnan(a)], b.view(np.uint64)[~np.isnan(b)]), "%s: values differ" % what


@pytest.mark.parametrize("H,W,nch", [(7, 5, 1), (13, 22, 3), (9, 31, 1), (2, 3, 3)])
def test_pyramid_is_a_brute_force_loop(H, W, nch):
    rng = np.random.default_rng(H * W + nch)
    img = rng.integers(0, 256, (H, W) if nch == 1 else (H, W, 3), dtype=np.uint8)
    got, want = po.pyramid(img), _brute_pyramid(img)
    for l in range(3):
        assert got[l][0].shape == to.level_shape(H, W, l)
        for k in range(3):
            same_bits(got[l][k], want[l][k], "level %d plane %d" % (l, k))


def test_grey_rgb_repeats_the_byte():
    rng = np.random.default_rng(1)
    g = rng.integers(0, 256, (6, 9), dtype=np.uint8)
    assert np.array_equal(po.intensity(np.stack([g] * 3, -1)), g.astype(np.float32))


def _plane_frame(H, W, k=2, planes=synth.POSED_PLANES):
    cal = dataio.Calib(float(W), W / 2 - 0.25, H / 2 + 0.5, synth.POSED_B, 0.0, None, None)
    P = synth.posed_camera_poses(k + 1)[k]
    Z, _, grey = synth.posed_render(P, H, W, cal.f, cal.cx, cal.cy, planes=planes)
    disp = (np.float32(cal.f * cal.baseline) / Z).astype(np.float32)
    Zm = Z.astype(np.float32)
    Zm[~np.isfinite(Zm)] = np.nan
    return cal, disp, Zm, np.clip(np.rint(grey), 0, 255).astype(np.uint8)


def test_terms_are_a_brute_force_loop():
    """every pixel's photometric Jacobian and residual, recomputed with Python floats one operation at a time"""
    rng = np.random.default_rng(2)
    H, W = 37, 71
    cal, disp, Zm, img = _plane_frame(H, W)
    disp = disp * (1 + 0.02 * rng.standard_normal(disp.shape)).astype(np.float32)
    disp[rng.random(disp.shape) < 0.1] = np.nan
    Zm[rng.random(Zm.shape) < 0.1] = np.nan
    ref = np.clip(img.astype(np.int64) + rng.integers(-20, 21, img.shape), 0, 255).astype(np.uint8)
    src, mod = to.source_pyramid(disp, cal, 30.0), to.model_pyramid(Zm, cal)
    isrc, iref = po.pyramid(img), po.pyramid(ref)
    T = np.eye(4)
    T[:3, :3] = track.rodrigues([0.004, -0.01, 0.006])
    T[:3, 3] = [0.03, -0.02, 0.05]
    p12 = T[:3].reshape(12)
    f, cx, cy = (_f32(v) for v in (cal.f, cal.cx, cal.cy))
    g_min, rho = 2.0, 15.0
    for level in range(3):
        delta = 0.3 * (level + 1)
        J, ok = po.photometric_jacobian(src, mod, isrc, iref, cal, level, p12, delta, g_min, rho)
        V, Vm = src[level][0], mod[level][0]
        Ir, gxr, gyr = iref[level]
        Is = isrc[level][0]
        _, hl, wl = V.shape
        s = f * 2.0 ** -level
        kept = 0
        for i in range(hl * wl):
            y, x = divmod(i, wl)
            want = [0.0] * 7
            p = [float(V[a, y, x]) for a in range(3)]
            q = [((p12[4 * a] * p[0] + p12[4 * a + 1] * p[1]) + p12[4 * a + 2] * p[2]) + p12[4 * a + 3] for a in range(3)]
            good = not math.isnan(p[0]) and q[2] > 0
            if good:
                xs = (((q[0] / q[2]) * f + cx) * 2.0 ** -level)
                ys = (((q[1] / q[2]) * f + cy) * 2.0 ** -level)
                u, v = math.floor(xs + 0.5), math.floor(ys + 0.5)
                good = 0 <= u < wl and 0 <= v < hl and not math.isnan(Vm[0, v, u])
            if good:
                d = [q[a] - float(Vm[a, v, u]) for a in range(3)]
                x0, y0 = math.floor(xs), math.floor(ys)
                good = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] <= delta * delta and 1 <= x0 and x0 + 1 <= wl - 2 and \
                    1 <= y0 and y0 + 1 <= hl - 2
            if good:
                fx, fy = xs - x0, ys - y0

                def bil(P):
                    a, b, c, e = (float(P[y0 + dy, x0 + dx]) for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)))
                    top, bot = a + fx * (b - a), c + fx * (e - c)
                    return top + fy * (bot - top)

                r = bil(Ir) - float(Is[y, x])
                gx, gy = bil(gxr), bil(gyr)
                good = gx * gx + gy * gy >= g_min * g_min and abs(r) <= rho
            if good:
                a, b = (gx * s) / q[2], (gy * s) / q[2]
                c = -(a * q[0] + b * q[1]) / q[2]
                want = [q[1] * c - q[2] * b, q[2] * a - q[0] * c, q[0] * b - q[1] * a, a, b, c, r]
                kept += 1
            got = [float(J[k][i]) for k in range(7)]
            assert np.array_equal(np.array(got).view(np.uint64), np.array(want).view(np.uint64)), "level %d pixel %d" % (level, i)
            assert bool(ok[i]) == good
        assert kept > 20, "level %d keeps %d pixels" % (level, kept)
    t, _ = po.photometric_terms(src, mod, isrc, iref, cal, 0, p12, 0.3, g_min, rho)
    J, _ = po.photometric_jacobian(src, mod, isrc, iref, cal, 0, p12, 0.3, g_min, rho)
    assert np.array_equal(t[:, 27], J[6] * J[6]) and np.array_equal(t[:, 1], J[0] * J[1])


def test_jacobian_is_the_derivative_of_the_residual():
    """J against central differences of r(xi) on a linear intensity ramp (which bilinear sampling reproduces exactly):
    r + J xi is the residual after [Rodrigues(omega) | tau] T"""
    H, W = 40, 60
    cal = dataio.Calib(50.0, 29.75, 20.5, 0.5, 0.0, None, None)
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    Z = (6.0 + 0.03 * x - 0.02 * y).astype(np.float32)
    src = mod = to.model_pyramid(Z, cal)
    ramp = (0.25 * x + 0.5 * y + 3.0).astype(np.float32)
    iref = [(ramp,) + po.gradients(ramp)] * 3
    isrc = [(np.full((H, W), 7.0, np.float32),) * 3] * 3
    T = np.eye(4)
    T[:3, :3] = track.rodrigues([0.01, -0.02, 0.015])
    T[:3, 3] = [0.05, 0.03, -0.1]
    args = (0, 1e9, 0.0, 1e9)                        # level, delta, g_min, rho: nothing gated
    J, ok = po.photometric_jacobian(src, mod, isrc, iref, cal, args[0], T[:3].reshape(12), *args[1:])
    h = 1e-6
    fd = np.zeros((6, H * W))
    oks = ok.copy()
    for k in range(6):
        e = np.zeros(6)
        e[k] = h
        rp, okp = po.photometric_jacobian(src, mod, isrc, iref, cal, args[0], track.update(T, e)[:3].reshape(12), *args[1:])
        rm, okm = po.photometric_jacobian(src, mod, isrc, iref, cal, args[0], track.update(T, -e)[:3].reshape(12), *args[1:])
        fd[k] = (rp[6] - rm[6]) / (2 * h)
        oks &= okp & okm
    assert oks.sum() > 1000
    Jm = np.stack(J[:6])[:, oks]
    err = np.abs(Jm - fd[:, oks]).max(1) / np.abs(Jm).max(1)
    assert (err < 1e-6).all(), err


def test_solve_joint():
    rng = np.random.default_rng(3)
    M = rng.standard_normal((50, 7))
    sums = np.array([M[:, a] @ M[:, b] for a in range(6) for b in range(a, 6)] + [M[:, a] @ M[:, 6] for a in range(6)]
                    + [M[:, 6] @ M[:, 6]])
    sp = sums[::-1].copy()
    assert np.array_equal(track.solve_joint(sums, sp, 50, 7, 0.0), track.solve(sums, 57))
    assert np.array_equal(track.solve_joint(sums, sums, 50, 0, 0.0), track.solve(sums, 50))
    assert np.array_equal(track.solve_joint(sums, sums, 40, 10, 0.25), track.solve(sums + 0.25 * sums, 50))
    assert track.solve_joint(np.zeros(28), sums, 3, 2, 1e-4) is None          # count = 5 < 6


def test_run_icp_default_is_geometric():
    """photometric 0 (the default) runs the geometric step and its solve; a joint step's geometric inliers decide lost"""
    cal, disp, Zm, img = _plane_frame(48, 160)
    src, mod = to.source_pyramid(disp, cal), to.model_pyramid(Zm, cal)
    geo = lambda level, p12, delta, cos_t: to.step(src, mod, cal, level, p12, delta, cos_t)
    T0 = np.eye(4)
    T0[:3, 3] = [0.02, -0.01, 0.03]
    a = track.run_icp(geo, T0)
    isrc = iref = po.pyramid(img)
    joint = lambda level, p12, delta, cos_t: po.step(src, mod, isrc, iref, cal, level, p12, delta, cos_t, 2.0, 30.0)
    b = track.run_icp(joint, T0, photometric=0.01)
    assert a[1] == b[1] or abs(a[1] - b[1]) < 0.05 * a[1]
    assert not a[2] and not b[2]
    assert np.abs(a[0][:3, 3]).max() < 1e-3 and np.abs(b[0][:3, 3]).max() < 1e-3


def _street_A(lam):
    """the level-0 A of the street seen from frame 1, aligned to frame 0 at the true relative pose"""
    H, W = 96, 160
    cal = dataio.Calib(float(W), W / 2 - 0.25, H / 2 + 0.5, synth.POSED_B, 0.0, None, None)
    poses = synth.posed_camera_poses(2, 0.5)
    frames = []
    for P in poses:
        Z, _, grey = synth.posed_render(P, H, W, cal.f, cal.cx, cal.cy, planes=synth.STREET_PLANES)
        frames.append((Z, np.clip(np.rint(grey), 0, 255).astype(np.uint8)))
    disp = (np.float32(cal.f * cal.baseline) / frames[1][0]).astype(np.float32)
    Zm = frames[0][0].astype(np.float32)
    Zm[~np.isfinite(Zm)] = np.nan
    src, mod = to.source_pyramid(disp, cal, 40.0), to.model_pyramid(Zm, cal)
    isrc, iref = po.pyramid(frames[1][1]), po.pyramid(frames[0][1])
    T = track.rigid_inv(poses[0]) @ poses[1]
    s, ng, nph, _ = po.step(src, mod, isrc, iref, cal, 0, T[:3].reshape(12), 0.25, math.cos(math.radians(30)), 2.0, 30.0)
    assert ng > 1000 and nph > 1000
    sums = s[:28] + lam * lam * s[28:]
    A = np.empty((6, 6))
    k = 0
    for a in range(6):
        for b in range(a, 6):
            A[a, b] = A[b, a] = sums[k]
            k += 1
    return A


def test_street_is_degenerate_along_the_street_without_the_term():
    """the street's normals all lie across it: the geometric A's weakest direction is the translation along it (z), held
    only by the normals' rounding noise (an eigenvalue ratio below 1e-5); the photometric term stiffens that direction
    more than a thousandfold"""
    Ag, Aj = _street_A(0.0), _street_A(0.01)
    ev, vec = np.linalg.eigh(Ag)
    assert abs(vec[5, 0]) > 0.99, vec[:, 0]
    ratio_g = ev[0] / ev[-1]
    evj = np.linalg.eigvalsh(Aj)
    ratio_j = evj[0] / evj[-1]
    ez = np.zeros(6)
    ez[5] = 1.0
    print("street: geometric ratio %.3g, z stiffness %.3g; joint ratio %.3g, z stiffness %.3g"
          % (ratio_g, ez @ Ag @ ez, ratio_j, ez @ Aj @ ez))
    assert ratio_g < 1e-5
    assert ratio_j > 100 * ratio_g
    assert ez @ Aj @ ez > 1e3 * (ez @ Ag @ ez)


# sha256 of the default drive's files and returned arrays (n 3, 24 x 64, with scans), as written before plane sets and
# per-frame steps existed
DEFAULT_DRIVE_SHA256 = "c350bef74313d31ad88845e8da281f6b7cdf2a12871d9cf085e095d05d3173cf"


def _drive_digest(root, out):
    h = hashlib.sha256()
    for d, _, files in sorted(os.walk(root)):
        for f in sorted(files):
            p = os.path.join(d, f)
            h.update(os.path.relpath(p, root).encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    for a in out[1] + out[2] + out[3]:
        h.update(a.tobytes())
    return h.hexdigest()


def test_posed_drive_defaults_and_street(tmp_path):
    a = str(tmp_path / "a")
    assert _drive_digest(a, synth.write_kitti_posed_drive(a, n=3, H=24, W=64, velodyne=True)) == DEFAULT_DRIVE_SHA256
    b = str(tmp_path / "b")
    out = synth.write_kitti_posed_drive(b, n=3, H=24, W=64, velodyne=True, planes=synth.POSED_PLANES, step=(0.4, 0.4))
    assert _drive_digest(b, out) == DEFAULT_DRIVE_SHA256
    steps = (0.4, 0.55, 0.45, 0.6, 0.5)
    _, _, pids, poses = synth.write_kitti_posed_drive(str(tmp_path / "c"), n=5, H=24, W=64, planes=synth.STREET_PLANES,
                                                      step=steps)
    for k in range(4):
        assert abs(np.linalg.norm(poses[k + 1][:3, 3] - poses[k][:3, 3]) - steps[k]) < 1e-12
    assert set(np.unique(pids[0])) <= {-1, 0, 1, 2}
    with pytest.raises(ValueError, match="5 frames need at least 4 steps"):
        synth.posed_camera_poses(5, (0.4, 0.5))


def _base(drive, out):
    return ["kitti", "census", "-drive", drive, "-out", out, "-voxel", "0.1"]


def test_refusals(tmp_path, monkeypatch):
    """each before any GPU work (or CUDA handle), with its own message"""
    for kw in (dict(photometric=-0.01), dict(photometric=math.nan), dict(rho=-1.0), dict(rho=math.inf), dict(grad_min=-2.0),
               dict(grad_min=math.nan)):
        name = next(iter(kw))
        with pytest.raises(ValueError, match="%s must be a finite number >= 0" % name):
            track.Tracker(8, 8, **kw)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=2, H=16, W=48)
    out = str(tmp_path / "out")
    b = _base(drive, out) + ["-mesh"]
    with pytest.raises(SystemExit, match="-photometric weighs a term of the tracking; it needs -poses track or refine"):
        fuse_tool.main(b + ["-photometric", "0.01"])
    with pytest.raises(SystemExit, match="-photometric weighs a term"):
        fuse_tool.main(b + ["-poses", "oxts", "-photometric", "0"])
    for flag, v in (("-photometric", "-0.01"), ("-photometric", "nan"), ("-photometric", "inf"), ("-rho", "-1"),
                    ("-rho", "inf"), ("-grad_min", "-0.5"), ("-grad_min", "nan")):
        extra = [] if flag == "-photometric" else ["-photometric", "0.01"]
        with pytest.raises(SystemExit, match="%s must be a finite number >= 0" % flag):
            fuse_tool.main(b + ["-poses", "track"] + extra + [flag, v])
    with pytest.raises(ValueError, match="photometric weighs a term of the tracking: it needs poses"):
        fusion.fuse_drive("kitti", "census", [drive], out=out, mesh=True, photometric=0.01)
    with pytest.raises(ValueError, match="rho must be a finite number >= 0"):
        fusion.fuse_drive("kitti", "census", [drive], out=out, mesh=True, poses="track", photometric=0.01, rho=-1.0)
    assert not os.path.exists(out)
