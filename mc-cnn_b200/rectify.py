"""Rectify a calibrated raw stereo pair on the GPU (an addition beyond the reference; DESIGN §22).

    rect = dataio.read_rectification("/data/raw/2011_09_26", "kitti_raw")      # or ("intrinsics.yml", "extrinsics.yml"),
    left2, right2, valid = rectify(left, right, rect, device=0)                 #    "opencv", size=(W, H)

`left` / `right` are the decoded raw views as frontend.load_bytes returns them, (H, W) grey or (H, W, 3) R, G, B uint8,
host or device, of the cameras' raw size.  The results are CUDA uint8: the two rectified views (H', W'[, 3]) and the left
view's validity mask (H', W'), 1 valid and 0 not, on the grid of ``rect.calib``.

The rule (mccnn_rectify_pair, OpenCV's initUndistortRectifyMap model): with iR = inv(P[:, :3] R) computed in float64 and
rounded once to fp32, each output pixel (u, v) maps, in fp32 with every operation rounded once and in this order, to
X = (iR00 u + iR01 v) + iR02 (Y, Z likewise); x = X / Z, y = Y / Z; r2 = x x + y y;
rad = (1 + r2 (k1 + r2 (k2 + r2 k3))) / (1 + r2 (k4 + r2 (k5 + r2 k6))); xd = x rad + (2 p1 x y + p2 (r2 + 2 x x));
yd = y rad + (p1 (r2 + 2 y y) + 2 p2 x y); sx = fx xd + cx, sy = fy yd + cy.  The raw view is sampled bilinearly at
(sx, sy) with the taps clamped into the image, v = (1 - b) ((1 - a) I00 + a I01) + b ((1 - a) I10 + a I11) with a, b the
fractional parts, and the byte is rint(v).  A pixel is valid when -0.5 <= sx < W - 0.5 and -0.5 <= sy < H - 0.5; where
Z <= 0 or a coordinate is not finite it is invalid and its bytes are 0.
"""
import numpy as np

NPARAM = 21                              # MCCNN_RECTIFY_NPARAM


def params(cam):
    """the MCCNN_RECTIFY_NPARAM float32 parameters of one :data:`dataio.CameraRect`: iR = inv(P[:, :3] R) (float64, rounded
    once), fx, fy, cx, cy of K, k1 k2 p1 p2 k3 k4 k5 k6 (missing ones 0)"""
    P = np.asarray(cam.P, np.float64).reshape(3, 4)
    iR = np.linalg.inv(P[:, :3] @ np.asarray(cam.R, np.float64).reshape(3, 3))
    K = cam.K
    k = list(cam.D) + [0.0] * (8 - len(cam.D))
    return np.concatenate([iR.reshape(-1), [K[0], K[4], K[2], K[5]], k]).astype(np.float32)


def _view(v, name, dev):
    import torch

    t = v if isinstance(v, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(v))
    if t.dtype != torch.uint8 or not (t.dim() == 2 or (t.dim() == 3 and t.size(2) == 3)):
        raise ValueError("%s view: (H, W) or (H, W, 3) uint8 expected, got %s %s" % (name, t.dtype, tuple(t.shape)))
    return t.to(dev).contiguous()


def rectify(left, right, rect, device=0):
    """(left', right', valid): the raw views `left` / `right` rectified by `rect` (a :class:`dataio.StereoRect`) on CUDA
    device `device` (mccnn_rectify_pair, one launch); refuses views that differ in shape or are not of the cameras' size
    before any launch."""
    import torch

    from .adcensus import _check, _stream, lib

    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    shapes = [tuple(np.shape(v)) for v in (left, right)]
    if shapes[0] != shapes[1]:
        raise ValueError("the two views must have the same size and channels, got %s and %s" % tuple(shapes))
    H, W = shapes[0][:2]
    rect.check_size(H, W, "rectify")
    Wo, Ho = rect.left.rect_size
    pl, pr = params(rect.left), params(rect.right)
    with torch.cuda.device(dev):
        views = [_view(v, n, dev) for v, n in ((left, "left"), (right, "right"))]
        tail = tuple(views[0].shape[2:])
        outs = [torch.empty((Ho, Wo) + tail, dtype=torch.uint8, device=dev) for _ in range(2)]
        valid = torch.empty((Ho, Wo), dtype=torch.uint8, device=dev)
        _check(lib().mccnn_rectify_pair(views[0].data_ptr(), views[1].data_ptr(), 1 if not tail else 3, H, W,
                                        pl.ctypes.data, pr.ctypes.data, Ho, Wo, outs[0].data_ptr(), outs[1].data_ptr(),
                                        valid.data_ptr(), _stream(valid)), "mccnn_rectify_pair")
    return outs[0], outs[1], valid
