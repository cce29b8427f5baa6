"""numpy restatement of DESIGN §22's rectification rule (mccnn_rectify_pair), operation for operation in float32.

Output pixel (u, v): X = (iR00 u + iR01 v) + iR02 (Y, Z likewise); x = X / Z, y = Y / Z; r2 = x x + y y;
rad = (1 + r2 (k1 + r2 (k2 + r2 k3))) / (1 + r2 (k4 + r2 (k5 + r2 k6))); xd = x rad + (2 p1 x y + p2 (r2 + 2 x x));
yd = y rad + (p1 (r2 + 2 y y) + 2 p2 x y); sx = fx xd + cx, sy = fy yd + cy.  Bilinear sampling with the taps clamped
into the raw image, v = (1 - b) ((1 - a) I00 + a I01) + b ((1 - a) I10 + a I11), the byte rint(v).  Valid: -0.5 <= sx <
W - 0.5 and -0.5 <= sy < H - 0.5; Z <= 0 or a non-finite coordinate: invalid, bytes 0."""
import numpy as np

f32 = np.float32


def source_map(params, Ho, Wo):
    """(sx, sy, front) float32 (Ho, Wo) of one camera's MCCNN_RECTIFY_NPARAM parameters; front is Z > 0 (sx, sy are NaN
    where it is not)"""
    p = np.asarray(params, np.float32)
    iR, (fx, fy, cx, cy), (k1, k2, p1, p2, k3, k4, k5, k6) = p[:9], p[9:13], p[13:21]
    v, u = np.meshgrid(np.arange(Ho, dtype=np.float32), np.arange(Wo, dtype=np.float32), indexing="ij")
    one, two = f32(1), f32(2)
    with np.errstate(all="ignore"):
        X = (iR[0] * u + iR[1] * v) + iR[2]
        Y = (iR[3] * u + iR[4] * v) + iR[5]
        Z = (iR[6] * u + iR[7] * v) + iR[8]
        front = Z > 0
        x, y = X / Z, Y / Z
        r2 = x * x + y * y
        rad = (one + r2 * (k1 + r2 * (k2 + r2 * k3))) / (one + r2 * (k4 + r2 * (k5 + r2 * k6)))
        xd = x * rad + (two * p1 * x * y + p2 * (r2 + two * x * x))
        yd = y * rad + (p1 * (r2 + two * y * y) + two * p2 * x * y)
        sx, sy = fx * xd + cx, fy * yd + cy
    nan = f32(np.nan)
    return np.where(front, sx, nan).astype(np.float32), np.where(front, sy, nan).astype(np.float32), front


def sample(img, sx, sy):
    """(bytes (Ho, Wo[, 3]) uint8, valid (Ho, Wo) bool) of the raw image `img` ((H, W) or (H, W, 3) uint8) at (sx, sy)"""
    img = np.asarray(img, np.uint8)
    H, W = img.shape[:2]
    ok = np.isfinite(sx) & np.isfinite(sy)
    with np.errstate(all="ignore"):
        fx0, fy0 = np.floor(np.where(ok, sx, 0)).astype(np.float32), np.floor(np.where(ok, sy, 0)).astype(np.float32)
        a, b = (np.where(ok, sx, 0) - fx0).astype(np.float32), (np.where(ok, sy, 0) - fy0).astype(np.float32)
    a1, b1 = f32(1) - a, f32(1) - b
    x0 = np.clip(fx0, 0, W - 1).astype(np.int64)
    x1 = np.clip(fx0 + f32(1), 0, W - 1).astype(np.int64)
    y0 = np.clip(fy0, 0, H - 1).astype(np.int64)
    y1 = np.clip(fy0 + f32(1), 0, H - 1).astype(np.int64)
    I = img.astype(np.float32)
    if I.ndim == 3:
        a, b, a1, b1 = a[..., None], b[..., None], a1[..., None], b1[..., None]
    top = a1 * I[y0, x0] + a * I[y0, x1]
    bot = a1 * I[y1, x0] + a * I[y1, x1]
    out = np.rint(b1 * top + b * bot).astype(np.uint8)
    out[~ok] = 0
    with np.errstate(invalid="ignore"):
        valid = ok & (sx >= f32(-0.5)) & (sx < f32(W) - f32(0.5)) & (sy >= f32(-0.5)) & (sy < f32(H) - f32(0.5))
    return out, valid


def rectify(img, params, Ho, Wo):
    """(bytes, valid) of one view"""
    sx, sy, _ = source_map(params, Ho, Wo)
    return sample(img, sx, sy)
