"""numpy restatement of the truncated signed distance field (mc-cnn_b200/fusion.py's TSDF, csrc/tsdf.cu), for
tests/test_tsdf.py and tests/test_gpu_tsdf.py.  Written from DESIGN §24:

* grid: voxel index i = floor(w / v) (float64), brick index floor(i / 8), the brick's key §23's key of its index, kept when
  every axis lies in [-2^20, 2^20); voxel centre c = (i + 0.5) v in float64; local voxel order (z, y, x);
* allocation: K = ceil(mu / (4 v)), s = fp32(mu / K); each valid pixel's ray points at z = Z + fp32(j) s (fp32), j = -K .. K,
  z > 0, X and Y of depth_oracle's fp32 rule at z, the world point of fusion_oracle's float64 rule;
* integration: every voxel of every brick; q = R^T (c - t) in float64; the pixel (floor((q_x / q_z) f + cx + 0.5), likewise
  y) in the image with a depth Z and q_z > 0; eta = Z - q_z; eta >= -mu: S += min(eta, mu) / mu, n += 1; |eta| < mu: the
  colour bytes added, nc += 1;
* mesh: marching tetrahedra on the Kuhn split of each cube of voxel centres (tet_triangles), vertices ordered by (brick,
  local voxel, edge direction x y z xy xz yz xyz), faces by (brick, local voxel, tetrahedron, triangle);
* render: samples at camera depth fp32(k v), k >= 1, trilinear over 8 observed voxel centres; the first k with samples
  k - 1 and k valid and phi_{k-1} >= 0 > phi_k gives Z = fp32(z_{k-1} + (v phi_{k-1}) / (phi_{k-1} - phi_k))."""
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

HALF = 1 << 20
VOX = 512
# edge directions as corner bits (x 1, y 2, z 4), in vertex order, and the direction index of corner bits
DIR_BITS = (1, 2, 4, 3, 5, 6, 7)
DIR_OF = {b: d for d, b in enumerate(DIR_BITS)}
# the Kuhn tetrahedra {0, e_p1, e_p1 + e_p2, 7} over the axis permutations in lexicographic order, and their parity
PERMS = ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))
TETS = tuple((0, 1 << p[0], (1 << p[0]) | (1 << p[1]), 7) for p in PERMS)
TET_ODD = (False, True, True, False, False, True)
# even reorderings of a tetrahedron's corners bringing the lone corner, or the two negative corners, first
ORD1 = ((0, 1, 2, 3), (1, 0, 3, 2), (2, 3, 0, 1), (3, 2, 1, 0))
ORD2 = {(0, 1): (0, 1, 2, 3), (0, 2): (0, 2, 3, 1), (0, 3): (0, 3, 1, 2), (1, 2): (1, 2, 0, 3), (1, 3): (1, 3, 2, 0),
        (2, 3): (2, 3, 0, 1)}


def K_of(voxel, trunc):
    return int(math.ceil(float(trunc) / (4.0 * float(voxel))))


def tet_triangles(neg, odd=False):
    """the triangles of a tetrahedron whose corners 0..3 have negative flags `neg`: each a tuple of 3 edges (p, q) of
    corner indices, oriented toward positive phi for a positively oriented tetrahedron (reversed when `odd`)"""
    neg = [bool(x) for x in neg]
    k = sum(neg)
    if k in (0, 4):
        tris = []
    elif k == 2:
        a, b, c, d = ORD2[tuple(i for i in range(4) if neg[i])]
        tris = [((a, c), (a, d), (b, d)), ((a, c), (b, d), (b, c))]
    else:
        lone = neg.index(True) if k == 1 else neg.index(False)
        o = ORD1[lone]
        tri = ((o[0], o[1]), (o[0], o[2]), (o[0], o[3]))
        tris = [tri if k == 1 else (tri[0], tri[2], tri[1])]
    return [(t[0], t[2], t[1]) for t in tris] if odd else tris


def brick_index(keys):
    k = np.asarray(keys, np.uint64)
    m = np.uint64((1 << 21) - 1)
    return np.stack([((k >> np.uint64(s)) & m).astype(np.int64) - HALF for s in (42, 21, 0)], 1)


def brick_keys(b):
    """(keys uint64, kept mask) of brick indices b (n, 3) float64 or int64"""
    b = np.asarray(b)
    with np.errstate(invalid="ignore"):
        keep = np.all((b >= -HALF) & (b < HALF), axis=1)
    i = b[keep].astype(np.int64) + HALF
    keys = (i[:, 0].astype(np.uint64) << np.uint64(42)) | (i[:, 1].astype(np.uint64) << np.uint64(21)) | i[:, 2].astype(np.uint64)
    return keys, keep


def to_world(X, Y, Z, pose):
    P = np.asarray(pose, np.float64).reshape(-1)[:12].reshape(3, 4)
    p = [np.asarray(a, np.float64) for a in (X, Y, Z)]
    return np.stack([((P[k, 0] * p[0] + P[k, 1] * p[1]) + P[k, 2] * p[2]) + P[k, 3] for k in range(3)], -1)


def lateral(u, c0, z, f):
    return ((np.asarray(u, np.float32) - np.float32(c0)) * z) / np.float32(f)


def alloc_keys(disp, cal, pose, voxel, trunc, max_depth=None):
    """(the unique brick keys a frame allocates, its valid pixels, its points outside the key range)"""
    Z = depth_oracle.depth32(disp, cal, max_depth)[0]
    ok = ~np.isnan(Z)
    ys, xs = np.nonzero(ok)
    z0 = Z[ok]
    K = K_of(voxel, trunc)
    s = np.float32(trunc / K)
    keys, outside = [], 0
    for j in range(-K, K + 1):
        z = (z0 + np.float32(j) * s).astype(np.float32)
        m = z > 0
        w = to_world(lateral(xs[m], cal.cx, z[m], cal.f), lateral(ys[m], cal.cy, z[m], cal.f), z[m], pose)
        with np.errstate(invalid="ignore", over="ignore"):
            b = np.floor(np.floor(w / np.float64(voxel)) * 0.125)
        k, keep = brick_keys(b)
        outside += int((~keep).sum())
        keys.append(k)
    return np.unique(np.concatenate(keys)).astype(np.uint64), int(ok.sum()), outside


def _rgb3(rgb):
    rgb = np.asarray(rgb, np.uint8)
    return np.repeat(rgb[:, :, None], 3, axis=2) if rgb.ndim == 2 else rgb


LOCAL = np.stack([np.arange(VOX) & 7, (np.arange(VOX) >> 3) & 7, np.arange(VOX) >> 6], 1)   # (512, 3): x, y, z


def centres(keys, voxel, offset=(0, 0, 0)):
    """(n, 512, 3) float64 voxel centres (of the voxels `offset` away)"""
    i = 8 * brick_index(keys)[:, None, :] + LOCAL[None] + np.asarray(offset, np.int64)
    return (i.astype(np.float64) + 0.5) * np.float64(voxel)


class Field:
    """the field of the rule, in ascending key order: keys (b,), S (b, 512) float64, n, nc (b, 512) int32, col (b, 512, 3)"""

    def __init__(self, voxel, trunc=None):
        self.voxel = float(voxel)
        self.trunc = 4.0 * self.voxel if trunc is None else float(trunc)
        self.keys = np.zeros(0, np.uint64)
        self.S = np.zeros((0, VOX))
        self.n = np.zeros((0, VOX), np.int32)
        self.nc = np.zeros((0, VOX), np.int32)
        self.col = np.zeros((0, VOX, 3), np.int32)
        self.pixels = self.outside = 0

    def allocate(self, fk):
        keys = np.union1d(self.keys, fk).astype(np.uint64)
        pos = np.searchsorted(keys, self.keys)
        S, n, nc, col = np.zeros((len(keys), VOX)), np.zeros((len(keys), VOX), np.int32), np.zeros((len(keys), VOX), np.int32), \
            np.zeros((len(keys), VOX, 3), np.int32)
        S[pos], n[pos], nc[pos], col[pos] = self.S, self.n, self.nc, self.col
        self.keys, self.S, self.n, self.nc, self.col = keys, S, n, nc, col

    def add(self, disp, cal, rgb, pose, max_depth=None):
        fk, pix, out = alloc_keys(disp, cal, pose, self.voxel, self.trunc, max_depth)
        self.pixels += pix
        self.outside += out
        self.allocate(fk)
        self.integrate(disp, cal, rgb, pose, max_depth)

    def integrate(self, disp, cal, rgb, pose, max_depth=None):
        if not len(self.keys):
            return
        H, W = np.asarray(disp).shape
        c = centres(self.keys, self.voxel).reshape(-1, 3)
        P = np.asarray(pose, np.float64).reshape(-1)[:12].reshape(3, 4)
        d = c - P[:, 3]
        q = [(P[0, a] * d[:, 0] + P[1, a] * d[:, 1]) + P[2, a] * d[:, 2] for a in range(3)]
        f, cx, cy = (float(np.float32(x)) for x in (cal.f, cal.cx, cal.cy))
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            u = np.floor(((q[0] / q[2]) * f + cx) + 0.5)
            v = np.floor(((q[1] / q[2]) * f + cy) + 0.5)
            ok = (q[2] > 0) & (u >= 0) & (u < W) & (v >= 0) & (v < H)
        p = np.where(ok, v, 0).astype(np.int64) * W + np.where(ok, u, 0).astype(np.int64)
        Z = depth_oracle.depth32(disp, cal, max_depth)[0].reshape(-1)[p]
        ok &= ~np.isnan(Z)
        mu = self.trunc
        eta = Z.astype(np.float64) - q[2]
        with np.errstate(invalid="ignore"):
            upd = ok & (eta >= -mu)
            col = upd & (np.abs(eta) < mu)
        S, n, nc, cs = self.S.reshape(-1), self.n.reshape(-1), self.nc.reshape(-1), self.col.reshape(-1, 3)
        S[upd] = S[upd] + np.minimum(eta[upd], mu) / mu
        n[upd] += 1
        nc[col] += 1
        cs[col] += _rgb3(rgb).reshape(-1, 3)[p[col]].astype(np.int32)

    # ---- reading the field ----

    def _observed(self, min_frames):
        obs = self.n >= min_frames
        with np.errstate(divide="ignore", invalid="ignore"):
            phi = np.where(obs, self.S / np.maximum(self.n, 1), 0.0)
        return obs, phi

    def _neighbours(self):
        """(b, 8) table index of the brick at b + corner bits o, -1 when absent"""
        b = brick_index(self.keys)
        out = np.full((len(b), 8), -1, np.int64)
        for o in range(8):
            nb = b + np.array([o & 1, (o >> 1) & 1, (o >> 2) & 1])
            with np.errstate(invalid="ignore"):
                inr = np.all((nb >= -HALF) & (nb < HALF), axis=1)
            k, _ = brick_keys(np.where(inr[:, None], nb, 0))
            at = np.minimum(np.searchsorted(self.keys, k), len(self.keys) - 1)
            out[:, o] = np.where(inr & (self.keys[at] == k), at, -1)
        return out

    def _corners(self, min_frames):
        """(brick (b, 512, 8), local (512, 8), observed (b, 512, 8), phi (b, 512, 8)) of each voxel's cube corners"""
        obs, phi = self._observed(min_frames)
        nbr = self._neighbours()
        o = np.arange(8)
        g = LOCAL[:, None, :] + np.stack([o & 1, (o >> 1) & 1, (o >> 2) & 1], 1)[None]        # (512, 8, 3)
        which = (g[..., 0] >> 3) | ((g[..., 1] >> 3) << 1) | ((g[..., 2] >> 3) << 2)
        local = ((g[..., 2] & 7) << 6) | ((g[..., 1] & 7) << 3) | (g[..., 0] & 7)
        cb = nbr[:, which]                                                                  # (b, 512, 8)
        safe = np.maximum(cb, 0)
        ob = (cb >= 0) & obs[safe, local[None]]
        ph = np.where(ob, phi[safe, local[None]], 0.0)
        return cb, local, ob, ph

    def mesh(self, min_frames=1):
        """(xyz (V, 3) float32, rgb (V, 3) uint8, faces (F, 3) int32)"""
        nb = len(self.keys)
        if not nb:
            return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8), np.zeros((0, 3), np.int32)
        cb, local, ob, ph = self._corners(min_frames)
        neg = ph < 0
        # vertices: (brick, voxel, direction) in C order
        em = np.stack([ob[..., 0] & ob[..., o] & (neg[..., 0] != neg[..., o]) for o in DIR_BITS], -1)    # (b, 512, 7)
        vid = np.full(em.shape, -1, np.int64)
        vid[em] = np.arange(int(em.sum()))
        bi, li, di = np.nonzero(em)
        o = np.array(DIR_BITS)[di]
        pa, pb = ph[bi, li, 0], ph[bi, li, o]
        t = pa / (pa - pb)
        ca = centres(self.keys, self.voxel)[bi, li]
        ob3 = np.stack([o & 1, (o >> 1) & 1, (o >> 2) & 1], 1)
        cbb = ((8 * brick_index(self.keys)[bi] + LOCAL[li] + ob3).astype(np.float64) + 0.5) * self.voxel
        xyz = (ca + t[:, None] * (cbb - ca)).astype(np.float32)
        sa, la = cb[bi, li, 0], local[li, 0]
        sb, lb = cb[bi, li, o], local[li, o]
        near = t < 0.5
        s1, l1 = np.where(near, sa, sb), np.where(near, la, lb)
        s2, l2 = np.where(near, sb, sa), np.where(near, lb, la)
        use2 = self.nc[s1, l1] == 0
        s1, l1 = np.where(use2, s2, s1), np.where(use2, l2, l1)
        nc = self.nc[s1, l1].astype(np.int64)
        C = self.col[s1, l1].astype(np.int64)
        rgb = np.where(nc[:, None] > 0, (C + nc[:, None] // 2) // np.maximum(nc, 1)[:, None], 0).astype(np.uint8)
        # faces: (brick, voxel, tetrahedron, triangle) in C order
        slots = np.full((nb, VOX, 6, 2, 3), -1, np.int64)
        for ti, tet in enumerate(TETS):
            allobs = ob[..., tet[0]] & ob[..., tet[1]] & ob[..., tet[2]] & ob[..., tet[3]]
            code = sum(neg[..., tet[k]].astype(np.int64) << k for k in range(4))
            for case in range(1, 15):
                sel = allobs & (code == case)
                if not sel.any():
                    continue
                bs, ls = np.nonzero(sel)
                for r, tri in enumerate(tet_triangles([(case >> k) & 1 for k in range(4)], TET_ODD[ti])):
                    for y, (p, q) in enumerate(tri):
                        lo, hi = sorted((tet[p], tet[q]), key=lambda c: bin(c).count("1"))
                        slots[bs, ls, ti, r, y] = vid[cb[bs, ls, lo], local[ls, lo], DIR_OF[hi ^ lo]]
        faces = slots.reshape(-1, 3)
        faces = faces[faces[:, 0] >= 0].astype(np.int32)
        return xyz, rgb, faces

    def mesh_ply(self, min_frames=1):
        """the bytes of depth.write_mesh_ply's file of the mesh"""
        xyz, rgb, faces = self.mesh(min_frames)
        return mesh_ply_bytes(xyz, rgb, faces)

    def _far(self, pose):
        b = brick_index(self.keys)
        lo, hi = b.min(0) * 8 * self.voxel, (b.max(0) + 1) * 8 * self.voxel
        P = np.asarray(pose, np.float64).reshape(-1)[:12].reshape(3, 4)
        row = np.linalg.inv(P[:, :3])[2]
        z = max(float(row @ (np.array([hi[x] if o >> x & 1 else lo[x] for x in range(3)]) - P[:, 3])) for o in range(8))
        return z + 1e-6 * abs(z) + 2 * self.voxel

    def sample(self, w, min_frames=1):
        """(valid, phi) of world points w (n, 3) by trilinear interpolation over the 8 surrounding voxel centres"""
        obs, phi = self._observed(min_frames)
        v = np.float64(self.voxel)
        with np.errstate(invalid="ignore", over="ignore"):
            gg = w / v - 0.5
            g = np.floor(gg)
            fr = gg - g
            ok = np.all((g >= -8.0 * HALF) & (g < 8.0 * HALF - 1), axis=1)
        i0 = np.where(ok[:, None], g, 0).astype(np.int64)
        ph = np.zeros((len(w), 8))
        for o in range(8):
            vi = i0 + np.array([o & 1, (o >> 1) & 1, (o >> 2) & 1])
            k, inr = brick_keys(vi >> 3)
            kk = np.zeros(len(w), np.uint64)
            kk[inr] = k
            at = np.minimum(np.searchsorted(self.keys, kk), max(len(self.keys) - 1, 0))
            found = inr & (self.keys[at] == kk) if len(self.keys) else np.zeros(len(w), bool)
            l = ((vi[:, 2] & 7) << 6) | ((vi[:, 1] & 7) << 3) | (vi[:, 0] & 7)
            ok &= found & obs[at, l] if len(self.keys) else found
            ph[:, o] = np.where(ok, phi[at, l], 0.0) if len(self.keys) else 0.0
        c4 = [ph[:, 2 * k] + fr[:, 0] * (ph[:, 2 * k + 1] - ph[:, 2 * k]) for k in range(4)]
        c2 = [c4[2 * k] + fr[:, 1] * (c4[2 * k + 1] - c4[2 * k]) for k in range(2)]
        return ok, c2[0] + fr[:, 2] * (c2[1] - c2[0])

    def render(self, cal, pose, H, W, min_frames=1, max_depth=None):
        """(H, W) float32 depth, NaN where the ray meets no zero crossing"""
        out = np.full(H * W, np.nan, np.float32)
        if not len(self.keys):
            return out.reshape(H, W)
        zfar = min(math.inf if max_depth is None else float(np.float32(max_depth)), self._far(pose))
        kmax = int(math.ceil(zfar / self.voxel)) + 1
        cap = np.float32(np.inf if max_depth is None else max_depth)
        ys, xs = np.divmod(np.arange(H * W), W)
        live = np.ones(H * W, bool)
        prev = np.zeros(H * W, bool)
        phi_prev = np.zeros(H * W)
        z_prev = np.float32(0)
        for k in range(1, kmax + 1):
            z = np.float32(k * self.voxel)
            if not z <= cap:
                break
            idx = np.nonzero(live)[0]
            if not len(idx):
                break
            zz = np.full(len(idx), z, np.float32)
            w = to_world(lateral(xs[idx], cal.cx, zz, cal.f), lateral(ys[idx], cal.cy, zz, cal.f), zz, pose)
            ok, phi = self.sample(w, min_frames)
            hit = ok & prev[idx] & (phi_prev[idx] >= 0) & (phi < 0)
            h = idx[hit]
            pp = phi_prev[h]
            out[h] = (np.float64(z_prev) + (self.voxel * pp) / (pp - phi[hit])).astype(np.float32)
            live[h] = False
            prev[idx], phi_prev[idx] = ok, np.where(ok, phi, 0.0)
            z_prev = z
        return out.reshape(H, W)


def sampled_bricks(keys, frames, tables, voxel, trunc=None, max_depth=None):
    """the Field of the sorted bricks `keys` alone, each voxel integrated by the per-voxel rule over `frames` [(disp, cal,
    rgb, pose)] while its brick is in the table: `tables` holds the sorted keys of the table after each frame's allocation.
    These are the values those bricks hold in the whole field of the frames, at the cost of the sample."""
    keys = np.asarray(keys, np.uint64)
    f = Field(voxel, trunc)
    f.allocate(keys)
    for (disp, cal, rgb, pose), table in zip(frames, tables):
        have = np.isin(keys, table)
        g = Field(voxel, trunc)
        g.keys, g.S, g.n, g.nc, g.col = keys[have], f.S[have], f.n[have], f.nc[have], f.col[have]
        g.integrate(disp, cal, rgb, pose, max_depth)
        f.S[have], f.n[have], f.nc[have], f.col[have] = g.S, g.n, g.nc, g.col
    return f


MESH_HEADER = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
               "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\n"
               "property list uchar int vertex_indices\nend_header\n")


def mesh_ply_bytes(xyz, rgb, faces):
    rec = np.zeros(len(xyz), np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))
    rec["xyz"], rec["rgb"] = xyz, rgb
    fr = np.zeros(len(faces), np.dtype([("n", "u1"), ("v", "<i4", 3)]))
    fr["n"], fr["v"] = 3, faces
    return (MESH_HEADER % (len(xyz), len(faces))).encode("ascii") + rec.tobytes() + fr.tobytes()
