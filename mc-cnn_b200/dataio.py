"""Data formats on either side of the hot path: what `preprocess_*.py/.lua`
write and `main.lua` reads back, the error metric of `-a test_te`, and the submission writers.

* ``fromfile`` / ``tofile``: the ``<name>`` + ``<name>.dim`` + ``<name>.type`` triple
  (main.lua:353-380, preprocess_mb.py:99-106);
* ``read_png16`` / ``write_png16``: KITTI disparity maps, uint16 = disparity * 256, 0 = invalid
  (adcensus.cu:1670-1706);
* ``write_pfm`` / ``read_pfm``: Middlebury disparity maps (adcensus.cu:1708-1722; the reader is
  preprocess_mb.py:13-57 without the down-sampling);
* ``bad_pixel_rate``: share of ground-truth pixels whose error exceeds ``err_at`` (3 px KITTI,
  1 px Middlebury; main.lua:400, 453, 1228-1236);
* ``kitti_submission_image``: the prediction pasted into the bottom rows of the full-size frame
  (main.lua:1203-1205).

Plain numpy / PIL host code: nothing here touches the GPU.
"""
import os

import numpy as np

_TYPES = {"float32": np.float32, "int32": np.int32, "int64": np.int64}
ERR_AT = {"kitti": 3.0, "kitti2015": 3.0, "mb": 1.0}


def fromfile(fname):
    """main.lua:353-380: dims from ``fname.dim`` (one per line), dtype from ``fname.type``, raw
    little-endian data from ``fname``.  A ``.dim`` holding the single line ``0`` is an empty tensor."""
    with open(fname + ".dim") as f:
        dim = [int(float(line)) for line in f.read().split()]
    if len(dim) == 1 and dim[0] == 0:
        return np.empty((0,), np.float64)                       # torch.Tensor()
    with open(fname + ".type") as f:
        t = f.read().strip()
    if t not in _TYPES:
        raise ValueError("%s: unsupported type %r (float32, int32, int64)" % (fname, t))
    x = np.fromfile(fname, dtype=np.dtype(_TYPES[t]).newbyteorder("<"))
    n = int(np.prod(dim))
    if x.size != n:
        raise ValueError("%s: %d elements on disk, .dim says %s" % (fname, x.size, dim))
    return x.reshape(dim).astype(_TYPES[t], copy=False)


def tofile(fname, x):
    """preprocess_mb.py:99-106 / preprocess_kitti.lua:118-144: the inverse of :func:`fromfile`"""
    if x is None:
        open(fname + ".dim", "w").write("0\n")
        return
    x = np.ascontiguousarray(x)
    if str(x.dtype) not in _TYPES:
        raise ValueError("unsupported dtype %s" % x.dtype)
    x.astype(x.dtype.newbyteorder("<"), copy=False).tofile(fname)
    open(fname + ".type", "w").write(str(x.dtype))
    open(fname + ".dim", "w").write("\n".join(map(str, x.shape)))


def read_png16_raw(fname):
    """the stored uint16 (H,W) values of a 16-bit grey PNG (disparity * 256, 0 = invalid)"""
    from PIL import Image

    with Image.open(fname) as im:
        if im.mode not in ("I;16", "I;16B", "I"):
            raise ValueError("%s: 16-bit grey PNG expected, got mode %s" % (fname, im.mode))
        return np.asarray(im).astype(np.uint16)


def read_png16(fname):
    """adcensus.cu:1670-1686: 16-bit grey PNG -> float32 (H,W), 0 stays 0 (invalid), else value / 256"""
    v = read_png16_raw(fname)
    return np.where(v == 0, np.float32(0.0), v.astype(np.float32) / np.float32(256.0)).astype(np.float32)


def write_png16(img, fname):
    """adcensus.cu:1688-1706: pixel = (uint16)(val < 1e-5 ? 0 : val * 256), the product in fp32,
    truncated towards zero (values past the uint16 range are clamped instead of wrapping)"""
    from PIL import Image

    img = np.asarray(img, dtype=np.float32)
    assert img.ndim == 2
    v = np.where(img < np.float32(1e-5), np.float32(0.0), img * np.float32(256.0))
    v = np.clip(np.trunc(v), 0, 65535).astype(np.uint16)
    Image.fromarray(v).save(fname, format="PNG")  # uint16 -> mode I;16


def write_pfm(img, fname):
    """adcensus.cu:1708-1722: ``Pf``, width height, scale -0.003922 (little endian), then the rows
    exactly as given (main.lua:1215 passes the vertically flipped map, PFM rows run bottom-up)"""
    img = np.ascontiguousarray(img, dtype="<f4")
    assert img.ndim == 2
    with open(fname, "wb") as f:
        f.write(("Pf\n%d %d\n-0.003922\n" % (img.shape[1], img.shape[0])).encode("ascii"))
        img.tofile(f)


def read_pfm(fname):
    """single-channel PFM -> float32 (H,W) in FILE row order (flip it to get top-down rows)"""
    with open(fname, "rb") as f:
        if f.readline().strip() != b"Pf":
            raise ValueError("%s: not a single-channel PFM" % fname)
        w, h = (int(t) for t in f.readline().split())
        scale = float(f.readline().strip())
        data = np.fromfile(f, dtype="<f4" if scale < 0 else ">f4", count=w * h)
    if data.size != w * h:
        raise ValueError("%s: truncated" % fname)
    return data.reshape(h, w).astype(np.float32)


def bad_pixel_rate(pred, actual, err_at):
    """main.lua:1228-1236: mask = actual != 0; err = #(|actual - pred| > err_at and mask) / #mask"""
    pred = np.asarray(pred, dtype=np.float32)
    actual = np.asarray(actual, dtype=np.float32)
    assert pred.shape == actual.shape
    mask = actual != 0
    n = int(mask.sum())
    if n == 0:
        return float("nan")                                      # 0 / 0 in the reference as well
    bad = (np.abs(actual - pred) > np.float32(err_at)) & mask
    return float(bad.sum()) / n


def kitti_submission_image(pred, img_height, img_width):
    """main.lua:1203-1205: a zero (img_height, img_width) frame whose LAST pred.shape[0] rows are the
    prediction (the networks see the bottom `height` rows of a KITTI frame)"""
    pred = np.asarray(pred, dtype=np.float32)
    h, w = pred.shape
    assert h <= img_height and w == img_width
    out = np.zeros((img_height, img_width), np.float32)
    out[img_height - h:] = pred
    return out


def write_kitti_submission(pred, img_height, img_width, out_dir, idx, dataset="kitti"):
    """main.lua:1203-1212: ``out/%06d_10.png`` (kitti) or ``out/disp_0/%06d_10.png`` (kitti2015)"""
    path = out_dir if dataset == "kitti" else os.path.join(out_dir, "disp_0")
    os.makedirs(path, exist_ok=True)
    fname = os.path.join(path, "%06d_10.png" % idx)
    write_png16(kitti_submission_image(pred, img_height, img_width), fname)
    return fname
