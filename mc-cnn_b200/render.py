"""The images a user looks at a result with: samples/bin2png.lua's grey PNGs of ``left.bin``, ``right.bin`` and ``disp.bin``,
and main.lua -debug's three PNGs per validation example (main.lua:1240-1265).

    render.bin2png("out")                                    # out/left.png, out/right.png, out/disp.png
    python tools/bin2png.py out -disp_max 70

Every pixel is computed on the GPU by csrc/render.cu (include/adcensus_b200.h, ``mccnn_render_*``), in the precision of the
reference's tensors, and quantised as Torch7's image.save writes a float image: clamp to [0, 1], times 255 in double,
truncated.  The host only writes the bytes with PIL: mode ``L`` for grey, ``RGB`` for colour.
"""
import os

import numpy as np
import torch

from .adcensus import AdcensusError, _check, _stream, _t, lib

BIN2PNG = ("left", "right", "disp")          # bin2png.lua's files, in the order it writes them


def _bytes(shape, device):
    return torch.empty(shape, dtype=torch.uint8, device=device)


def volume_file_grey(path, D, H, W, device=0):
    """bin2png.lua:17-24 on the (1, D, H, W) float32 file `path`: (H, W) uint8 CUDA tensor.  The file is streamed through the
    GPU in row chunks; it is never held whole on the host or the device."""
    dev = torch.device("cuda", device)
    out = _bytes((H, W), dev)
    with torch.cuda.device(dev):
        _check(lib().mccnn_render_volume_file(os.fsencode(path), int(D), int(H), int(W), out.data_ptr(), _stream(out)),
               "render_volume_file(%s)" % path)
    return out


def map_grey(x, d):
    """bin2png.lua:27-28, ``disp:div(d)`` of a (.., H, W) CUDA float map: (H, W) uint8 CUDA tensor"""
    p = _t(x, 1, "map_grey")
    H, W = x.size(-2), x.size(-1)
    out = _bytes((H, W), x.device)
    with torch.cuda.device(x.device):
        _check(lib().mccnn_render_map(p, H, W, int(d), out.data_ptr(), _stream(x)), "render_map")
    return out


def grey2jet(x, disp_max, mask_blue=False):
    """adcensus.grey2jet of ``x:double():add(1):div(disp_max)`` (main.lua:1242 / 1260) for a (.., H, W) CUDA float map:
    (H, W, 3) uint8 CUDA tensor.  mask_blue: blue times (x != 0), the ground-truth image of main.lua:1261.  A value the
    reference asserts on (NaN, or outside [-0.1, 4.1] after the x4) raises AdcensusError."""
    p = _t(x, 1, "grey2jet")
    H, W = x.size(-2), x.size(-1)
    out = _bytes((H, W, 3), x.device)
    with torch.cuda.device(x.device):
        rc = lib().mccnn_render_jet(p, H, W, int(disp_max), 1 if mask_blue else 0, out.data_ptr(), _stream(x))
    if rc == -3:                                                          # ADCENSUS_ERANGE
        raise AdcensusError("grey2jet: a disparity outside the colour map (NaN, or (x + 1) / %d * 4 outside [-0.1, 4.1])"
                            % disp_max)
    _check(rc, "grey2jet")
    return out


def error_image(x0, pred, gt, err_at):
    """main.lua:1243-1252: the left image x0 in grey, good pixels tinted green and bad ones red; (H, W, 3) uint8 CUDA tensor.
    x0, pred and gt are CUDA float maps of one shape."""
    n = "error_image"
    a, b, c = _t(x0, 1, n), _t(pred, 2, n), _t(gt, 3, n)
    H, W = pred.size(-2), pred.size(-1)
    for narg, t in ((1, x0), (3, gt)):
        if t.numel() != H * W or t.device != pred.device:
            raise AdcensusError("bad argument #%d to '%s' (a %dx%d map on %s expected)" % (narg, n, H, W, pred.device))
    out = _bytes((H, W, 3), pred.device)
    with torch.cuda.device(pred.device):
        _check(lib().mccnn_render_error(a, b, c, H, W, float(err_at), out.data_ptr(), _stream(pred)), n)
    return out


def save_png(path, img):
    """an (H, W) byte image as an 8-bit grey PNG (mode L), an (H, W, 3) one as RGB"""
    from PIL import Image

    a = np.ascontiguousarray(img.cpu().numpy() if isinstance(img, torch.Tensor) else img, dtype=np.uint8)
    if a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] != 3):
        raise ValueError("save_png: (H, W) or (H, W, 3) bytes expected, got %s" % (a.shape,))
    Image.fromarray(a, "L" if a.ndim == 2 else "RGB").save(path, format="PNG")


def check_bins(dir, disp_max, height, width):
    """the three files bin2png.lua reads, each of the size it views it as: {name: path}; ValueError otherwise"""
    if disp_max < 1 or height < 1 or width < 1:
        raise ValueError("bin2png: disp_max, height and width must be positive (got %d, %d, %d)" % (disp_max, height, width))
    paths = {}
    for name in BIN2PNG:
        p = os.path.join(dir, name + ".bin")
        want = (1 if name == "disp" else disp_max) * height * width * 4
        if not os.path.isfile(p):
            raise ValueError("bin2png: %s not found" % p)
        got = os.path.getsize(p)
        if got != want:
            shape = "1x%dx%d" % (height, width) if name == "disp" else "%dx%dx%d" % (disp_max, height, width)
            raise ValueError("bin2png: %s holds %d bytes, a %s float32 %s needs %d (check -disp_max, -height, -width)"
                             % (p, got, shape, "map" if name == "disp" else "volume", want))
        paths[name] = p
    return paths


def bin2png(dir=".", disp_max=70, height=370, width=1226, device=0):
    """samples/bin2png.lua in `dir` (its constants d, h, w are the defaults): left.png and right.png, the arg-min over
    disparities of left.bin / right.bin over disp_max, and disp.png, disp.bin over disp_max.  Prints the script's
    "Writing ..." lines; returns the paths written.  Every file's size is checked before any GPU work."""
    paths = check_bins(dir, disp_max, height, width)
    dev = torch.device("cuda", device)
    written = []
    for name in BIN2PNG:
        out = os.path.join(dir, name + ".png")
        print("Writing %s.png" % name, flush=True)
        if name == "disp":
            with torch.cuda.device(dev):
                m = torch.from_numpy(np.fromfile(paths[name], dtype="<f4").reshape(height, width)).to(dev)
            img = map_grey(m, disp_max)
        else:
            img = volume_file_grey(paths[name], disp_max, height, width, device=device)
        save_png(out, img)
        written.append(out)
    return written


def debug_names(dataset, arch, id_):
    """main.lua:1263-1265's file names for one example: (gt, pred, err)"""
    return ("%s_%s_gt.png" % (dataset, id_), "%s_%s_%s_pred.png" % (dataset, arch, id_),
            "%s_%s_%s_err.png" % (dataset, arch, id_))


def debug_images(x0, pred, gt, disp_max, err_at):
    """main.lua:1240-1261 for one example: (gt, pred, err) images, each (H, W, 3) uint8 on the device; x0 the left image,
    pred and gt the maps, all CUDA float (H, W)"""
    return grey2jet(gt, disp_max, mask_blue=True), grey2jet(pred, disp_max), error_image(x0, pred, gt, err_at)


def write_debug_images(debug_dir, dataset, arch, id_, x0, pred, gt, disp_max, err_at, device=0):
    """the three PNGs of main.lua -debug for one example under `debug_dir`, drawn on `device` from the (H, W) float maps
    x0, pred and gt (numpy or torch): their paths"""
    dev = torch.device("cuda", device) if isinstance(device, int) else device
    maps = [torch.as_tensor(np.asarray(a, dtype=np.float32) if not isinstance(a, torch.Tensor) else a)
            .to(dev, torch.float32).contiguous() for a in (x0, pred, gt)]
    os.makedirs(debug_dir, exist_ok=True)
    paths = [os.path.join(debug_dir, n) for n in debug_names(dataset, arch, id_)]
    with torch.cuda.device(dev):
        for p, img in zip(paths, debug_images(*maps, disp_max, err_at)):
            save_png(p, img)
    return paths
