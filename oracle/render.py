"""numpy restatement of the result images -- TEST INFRASTRUCTURE.

The four operations of csrc/render.cu with the reference's operation order and precision, one numpy operation per
reference tensor operation:

* ``volume_grey``: samples/bin2png.lua:17-24 on a (D, H, W) volume;
* ``map_grey``: bin2png.lua:27-28 on a disparity map;
* ``grey2jet``: adcensus.grey2jet (adcensus.cu:2001-2053) of the map as main.lua:1242 / 1260 hand it over, with the
  ground truth's blue-channel mask of main.lua:1261;
* ``error_image``: main.lua:1243-1252, the left image tinted green (good) and red (bad) in fp32.

Every result is quantised as Torch7's image.save writes a float image (``quantise``).
"""
import numpy as np

BIG = np.float32(1e38)           # fromfile's NaN replacement (bin2png.lua:13-14), as a float32 store


class RangeError(ValueError):
    """grey2jet's assert(0) (adcensus.cu:2045-2046): a value that is NaN or outside [-0.1, 4.1] after the x4"""


def quantise(x):
    """image.save of a float image: image.saturate's clamp to [0, 1], times 255 in double, truncated to uint8 by the byte
    conversion (NaN survives the clamp and converts to 0 on x86)"""
    v = np.asarray(x).astype(np.float64)
    v = np.where(v < 0, 0.0, np.where(v > 1, 1.0, v))
    v = np.where(np.isnan(v), 0.0, v)
    return np.trunc(v * 255.0).astype(np.uint8)


def fromfile_nan(x):
    """x[x:ne(x)] = 1e38"""
    x = np.asarray(x, dtype=np.float32)
    return np.where(np.isnan(x), BIG, x)


def volume_grey(vol):
    """_, i = vol:min(2) (first index on ties, 1-based); i:float():div(D); quantised (H, W) bytes"""
    vol = fromfile_nan(vol)
    D = vol.shape[0]
    idx = np.argmin(vol, axis=0)                 # the first of equal minima, as TH's strict < scan
    return quantise((idx + 1).astype(np.float32) / np.float32(D))


def map_grey(x, d):
    """disp:div(d) in fp32; quantised (H, W) bytes"""
    return quantise(fromfile_nan(x) / np.float32(d))


def jet_colours(grey):
    """adcensus.grey2jet's colours of a float64 grey image: (3, ...) float64 planes R, G, B; RangeError where the reference
    asserts"""
    val = np.asarray(grey, dtype=np.float64) * 4
    r, g, b = np.zeros_like(val), np.zeros_like(val), np.zeros_like(val)
    bands = [(-0.1 <= val) & (val < 0.5), (0.5 <= val) & (val < 1.5), (1.5 <= val) & (val < 2.5),
             (2.5 <= val) & (val < 3.5), (3.5 <= val) & (val <= 4.1)]
    if not np.logical_or.reduce(bands).all():
        bad = val[~np.logical_or.reduce(bands)]
        raise RangeError("grey2jet: %d value(s) outside [-0.1, 4.1] after the x4, e.g. %r" % (bad.size, bad.flat[0]))
    m = bands[0]
    b[m] = 0.5 + val[m]
    m = bands[1]
    g[m], b[m] = val[m] - 0.5, 1
    m = bands[2]
    r[m], g[m], b[m] = val[m] - 1.5, 1, 1 - (val[m] - 1.5)
    m = bands[3]
    r[m], g[m] = 1, 1 - (val[m] - 2.5)
    m = bands[4]
    r[m] = 1 - (val[m] - 3.5)
    return np.stack([r, g, b])


def jet_grey(x, disp_max):
    """x:double():add(1):div(disp_max), the grey image main.lua hands to grey2jet"""
    return (np.asarray(x, dtype=np.float32).astype(np.float64) + 1) / float(disp_max)


def grey2jet(x, disp_max, mask_blue=False):
    """main.lua:1241-1242 (prediction) or 1259-1261 (ground truth, mask_blue: blue times (x != 0)): (H, W, 3) bytes"""
    x = np.asarray(x, dtype=np.float32)
    rgb = jet_colours(jet_grey(x, disp_max))
    if mask_blue:
        rgb[2] = rgb[2] * (x != 0).astype(np.float64)
    return np.moveaxis(quantise(rgb), 0, -1)


def error_image(x0, pred, gt, err_at):
    """main.lua:1243-1252 in fp32: (H, W, 3) bytes.  cutorch's div(255) is a multiplication by f32(1 / 255)."""
    f = np.float32
    x0, pred, gt = (np.asarray(a, dtype=np.float32) for a in (x0, pred, gt))
    grey = ((x0 * f(50)) + f(150)) * (f(1) / f(255))
    diff = np.abs(gt - pred)
    mask = (gt != 0).astype(np.float32)
    bad = (diff > f(err_at)).astype(np.float32) * mask
    good = (diff <= f(err_at)).astype(np.float32) * mask
    r = (grey + f(0.5) * bad) + f(-0.5) * good
    g = (grey + f(-0.5) * bad) + f(0.5) * good
    b = (grey + f(-0.5) * bad) + f(-0.5) * good
    return np.stack([quantise(r), quantise(g), quantise(b)], axis=-1)
