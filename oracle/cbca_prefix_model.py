"""Numerical model of an O(1)-per-pixel CBCA (prefix sums along x, then along y) -- TEST INFRASTRUCTURE
ONLY; a design study for a tolerance-mode kernel, no product code uses it.

cbca (adcensus.cu:343-377) sums vol[d] over a cross-shaped support: rows yy in (yy_s, yy_t), and in every
row the run xx in (xx_s(yy), xx_t(yy)).  The run of row yy depends on (d, yy, x) only, NOT on which output
row y uses it, so with
    S(d, yy, x) = sum of vol[d, yy, xx_s+1 .. xx_t-1]   = P(yy, xx_t) - P(yy, xx_s + 1)      (P: prefix along x)
    C(d, yy, x) = number of taps of that run
the output is a difference of prefix sums of S along y:
    out(d, y, x) = (T(yy_t, x) - T(yy_s + 1, x)) / (N(yy_t, x) - N(yy_s + 1, x))             (T, N: prefix of S, C along y)
i.e. a constant amount of work per pixel instead of one addition per tap -- but a different summation
order, so it is only within rounding of the reference (the north star allows 1e-4 relative for float
aggregation; index outputs stay bit-exact only as far as no arg-min is decided by that rounding).
`tile` limits the length of every prefix (a kernel works on tiles with a halo), which bounds the
cancellation error; `dtype` is the precision the prefixes are held in.

`emulate_ws` restates the kernel that ships in the default mode, cbca_ws_kernel (csrc/cbca_tma.cu), index for index in
float32 numpy, with switches for the mistakes the GPU tests must be able to see.
"""
import numpy as np


def cbca_prefix(x0c, x1c, vol, direction, dtype=np.float32, tile=(32, 128)):
    x0c, x1c, vol = (np.asarray(a, np.float32) for a in (x0c, x1c, vol))
    D, H, W = vol.shape
    out = vol.copy()                                                       # x' outside the image: plain copy (:353-354)
    ys, xs = np.mgrid[0:H, 0:W]
    for d in range(D):
        sh = d * direction
        xp = xs + sh
        valid = (xp >= 0) & (xp < W)
        xpc = np.clip(xp, 0, W - 1)
        # per (yy, x): the run of row yy (:362-363) and the vertical range of output (y, x) (:359-360)
        xx_s = np.maximum(x0c[0], x1c[0][ys, xpc] - sh).astype(np.int64)
        xx_t = np.minimum(x0c[1], x1c[1][ys, xpc] - sh).astype(np.int64)
        yy_s = np.maximum(x0c[2], x1c[2][ys, xpc]).astype(np.int64)
        yy_t = np.minimum(x0c[3], x1c[3][ys, xpc]).astype(np.int64)
        v = np.where(np.isnan(vol[d]), np.float32(0), vol[d])
        ty, tx = tile
        res = np.full((H, W), np.nan, np.float32)
        for y0 in range(0, H, ty):
            for x0 in range(0, W, tx):
                y1, x1 = min(y0 + ty, H), min(x0 + tx, W)
                # halo: everything the outputs of this tile can reach
                ya, yb = max(0, int(yy_s[y0:y1, x0:x1].min()) + 1), min(H, int(yy_t[y0:y1, x0:x1].max()))
                if yb <= ya:
                    ya, yb = y0, y1
                xa = max(0, int(xx_s[ya:yb, x0:x1].min()) + 1)
                xb = min(W, int(xx_t[ya:yb, x0:x1].max()))
                if xb <= xa:
                    xa, xb = x0, x1
                P = np.zeros((yb - ya, xb - xa + 1), dtype)
                P[:, 1:] = np.cumsum(v[ya:yb, xa:xb].astype(dtype), axis=1, dtype=dtype)
                rows = np.arange(ya, yb)[:, None] - ya
                lo = np.clip(xx_s[ya:yb, x0:x1] + 1, xa, xb) - xa
                hi = np.clip(xx_t[ya:yb, x0:x1], xa, xb) - xa
                hi = np.maximum(hi, lo)
                S = (P[rows, hi] - P[rows, lo]).astype(dtype)               # row sums of the runs, every row of the halo
                C = (hi - lo).astype(np.int64)
                T = np.zeros((yb - ya + 1, x1 - x0), dtype)
                T[1:] = np.cumsum(S, axis=0, dtype=dtype)
                N = np.zeros((yb - ya + 1, x1 - x0), np.int64)
                N[1:] = np.cumsum(C, axis=0)
                cols = np.arange(x1 - x0)[None, :]
                a = np.clip(yy_s[y0:y1, x0:x1] + 1, ya, yb) - ya
                b = np.clip(yy_t[y0:y1, x0:x1], ya, yb) - ya
                b = np.maximum(b, a)
                num = (T[b, cols] - T[a, cols]).astype(np.float32)
                den = (N[b, cols] - N[a, cols]).astype(np.float32)
                with np.errstate(invalid="ignore", divide="ignore"):
                    res[y0:y1, x0:x1] = num / den
        out[d] = np.where(valid, res, vol[d])
    return out


# cbca_ws_kernel's constants (cbca_tma.cu)
WS_TX, WS_TY, WS_HO, WS_TWP, WS_RING, WS_DCH, EPL = 128, 64, 32, 144, 16, 20, 9
f32 = np.float32


def pack_hv(xc):
    """cbca_tma.cu pack_arms_hv_kernel: H word 4L | 4(R - 1) << 16, V word U << 8 | D << 24 (lengths clipped)"""
    H, W = xc.shape[1:]
    ys, xs = np.mgrid[0:H, 0:W]
    l = np.clip(xs - xc[0].astype(np.int64), 0, 255)
    r = np.clip(xc[1].astype(np.int64) - xs, 1, 255)
    u = np.clip(ys - xc[2].astype(np.int64), 0, 255)
    d = np.clip(xc[3].astype(np.int64) - ys, 0, 255)
    return (4 * l) | ((4 * (r - 1)) << 16), (u << 8) | (d << 24)


def _minu2(a, b):
    return np.minimum(a & 0xffff, b & 0xffff) | (np.minimum(a >> 16, b >> 16) << 16)


def _row_prefix(row):
    """one tile row as a prefix warp scans it: 16 lanes x 9 consecutive columns, sequential in a lane, a 4-step
    Hillis-Steele scan of the lane totals, base = inclusive total - own last value"""
    v = row.reshape(16, EPL).copy()
    for i in range(1, EPL):
        v[:, i] = v[:, i] + v[:, i - 1]
    incl = v[:, EPL - 1].copy()
    for o in (1, 2, 4, 8):
        up = np.concatenate([np.zeros(o, f32), incl[:-o]])
        incl = np.where(np.arange(16) >= o, incl + up, incl).astype(f32)
    base = (incl - v[:, EPL - 1]).astype(f32)
    return (v + base[:, None]).astype(f32).reshape(-1)


def emulate_ws(x0c, x1c, vol, direction, R, centre=True, scrub_rule=True, run_end=0, swap_ud=False):
    """cbca_ws_kernel<R> (cbca_tma.cu) restated index for index in numpy float32: equal D chunks of <= 20 and the nproc
    copy of planes whose tile lies in the invalid triangle; per plane the TMA box from (x0 - HX, y0 - HALO) at the 144-float
    pitch, zero outside the image; the tile's mid pixel subtracted (centring) and NaN counted as 0 where the box reaches
    the invalid triangle (scrub); row prefixes as the prefix warps scan them (9 columns per lane, 16 lanes); each walker
    thread's running (T, N) sums in a 16-row ring, an output = ring(y + Dn - 1) - ring(y - U), T / N with one Newton step,
    plus the centre value.  The reciprocal is exact here (the kernel's rcp.approx is within an ulp before the Newton step).
    Mutations: centre=False drops the centring, scrub_rule=False the scrub, run_end=1 reads each run one column too far
    right, swap_ud=True exchanges the up and down arm lengths."""
    D, H, W = vol.shape
    HALO = R + 1
    HX = (HALO + 3) & ~3
    TH = WS_TY + 2 * R + 1
    NWALK = 2 * R + WS_HO
    h0, v0 = pack_hv(x0c)
    h1, v1 = pack_hv(x1c)
    out = np.full_like(vol, f32(-12345.0))
    dch = -(-D // -(-D // WS_DCH))
    c = np.arange(WS_TX)

    def at(a, yy, xx):                             # 0 outside the image (staged windows, registers)
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        return np.where(ok, a[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0)

    for d0 in range(0, D, dch):
        dn = min(dch, D - d0)
        for y0 in range(0, H, WS_TY):
            for x0 in range(0, W, WS_TX):
                nproc = 0
                while nproc < dn and not ((x0 + WS_TX - 1 - (d0 + nproc) < 0) if direction < 0 else (x0 + d0 + nproc >= W)):
                    nproc += 1
                x = x0 + c
                for dd in range(dn):
                    d = d0 + dd
                    if dd >= nproc:                 # plane entirely inside the invalid triangle: plain copy
                        out[d, y0:y0 + WS_TY, x0:x0 + WS_TX] = vol[d, y0:y0 + WS_TY, x0:x0 + WS_TX]
                        continue
                    # the TMA box: (x0 - HX, y0 - HALO), TH rows of WS_TWP floats, zero outside the (W, H, D) view
                    yy = y0 - HALO + np.arange(TH)[:, None]
                    xx = x0 - HX + np.arange(WS_TWP)[None, :]
                    ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
                    P = np.where(ok, vol[d][np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], f32(0)).astype(f32)
                    m = P[HALO + WS_TY // 2, HX + WS_TX // 2]
                    mu = m if (centre and abs(m) <= 3.0e38) else f32(0)
                    scrub = (x0 - HX - d < 0) if direction < 0 else (x0 - HX + WS_TWP + d > W)
                    P = (P - mu).astype(f32)
                    if scrub and scrub_rule:
                        P = np.where(P == P, P, f32(0)).astype(f32)
                    P = np.stack([_row_prefix(r) for r in P])
                    sh = d * direction
                    xs = x + sh
                    valid_col = (x < W) & (xs >= 0) & (xs < W)
                    for h in range(2):
                        yb = y0 + WS_HO * h
                        nv = np.where(x < W, max(0, min(WS_HO, H - yb)), 0)
                        nst = np.where(valid_col, nv, 0)
                        ring = np.zeros((WS_RING, 2, WS_TX), f32)
                        run = np.zeros((2, WS_TX), f32)
                        for rr in range(1, NWALK + 1):
                            iy = yb - HALO + rr                       # image row of relative row rr
                            hw = _minu2(at(h0, iy, x), at(h1, iy, xs))
                            L4, R4 = hw & 0xffff, hw >> 16
                            prow = P[WS_HO * h + rr]
                            ph = prow[c + HX + (R4 >> 2) + run_end]
                            pl = prow[c + HX - (L4 >> 2)]
                            S = (ph - pl).astype(f32)
                            nf = ((L4 + R4) // 4).astype(f32)
                            run = np.stack([run[0] + S, run[1] + nf]).astype(f32)
                            ring[rr % WS_RING] = run
                            if rr >= 2 * R + 1:
                                k = rr - 2 * R - 1
                                vw = _minu2(at(v0, yb + k, x), at(v1, yb + k, xs))
                                U, Dn = (vw & 0xffff) >> 8, vw >> 24
                                if swap_ud:
                                    U, Dn = Dn, U
                                rk = HALO + k
                                a = ring[(rk - 1 + Dn) % WS_RING, :, c]
                                b = ring[(rk - U) % WS_RING, :, c]
                                T, N = (a[:, 0] - b[:, 0]).astype(f32), (a[:, 1] - b[:, 1]).astype(f32)
                                with np.errstate(divide="ignore", invalid="ignore"):
                                    rc = (f32(1) / N).astype(f32)
                                    q = (T * rc).astype(f32)
                                    e = (T.astype(np.float64) - q.astype(np.float64) * N).astype(f32)
                                    q = f32(q + (e.astype(np.float64) * rc).astype(f32))
                                    q = (q + mu).astype(f32)
                                st = k < nst
                                y = yb + k
                                if y < H:
                                    out[d, y, x[st]] = q[st]
                        cp = ~valid_col & (x < W)
                        if cp.any():
                            out[d, yb:yb + WS_HO, x[cp]] = vol[d, yb:yb + WS_HO, x[cp]]
    return out
