"""Image front end of ``main.lua ... -a predict`` (main.lua:1084-1104): load the two views, grey
conversion, standardisation, ``stereo_predict`` on the GPU, and the raw ``.bin`` outputs.

With arch ``ad`` or ``census`` (main.lua:932-942) no trained network is needed, so two PNG files
are enough to run the whole hot path end to end; with arch ``fast`` the caller supplies the
(2,C,H,W) tower output.

Parity notes: ``image.load`` / ``image.rgb2y`` / ``mean`` / ``std`` are Torch7's
``image`` and ``TH`` (version unpinned, not under /root/reference).  This module restates their
documented arithmetic -- byte values as floats, Y = 0.299 R + 0.587 G + 0.114 B accumulated in
fp32 in that order, mean and the unbiased (n-1) standard deviation accumulated in double, the
scalar applied in fp32 -- **parity unpinned** for the last bit of the double accumulations; every
stage after the (2,1,H,W) batch is the bit-exact path of :mod:`pipeline`.

Which stereo method a (dataset, arch, network) runs -- preset, fix_border's width, network stages -- is decided by
:class:`StereoMethod` for every prediction path.
"""
import os

import numpy as np

from . import confidence as confidence_
from . import dataio, depth, pipeline


def load_bytes(path):
    """The decoded 8-bit image of ``image.load(path, nil, 'byte')``: (H, W) uint8 for grey files, (H, W, 3) interleaved R, G, B
    for colour (an alpha channel is dropped); a 16-bit file keeps its high byte."""
    from PIL import Image

    with Image.open(path) as im:
        if im.mode in ("I;16", "I;16B", "I"):            # 16-bit grey: 'byte' loading keeps the high byte
            a = np.asarray(im, dtype=np.uint32) >> 8
            if a.size and a.max() > 255:
                raise ValueError("%s: more than 16 bits per pixel" % path)
            return a.astype(np.uint8)
        if im.mode in ("L", "1", "P", "LA"):
            return np.array(im.convert("L"), dtype=np.uint8)
        return np.array(im.convert("RGB"), dtype=np.uint8)


def load_image(path):
    """``image.load(path, nil, 'byte'):float()``: (C,H,W) float32 with the byte values 0..255
    (C = 1 for grey files, 3 for colour; an alpha channel is dropped)."""
    a = load_bytes(path)
    a = a[None] if a.ndim == 2 else a.transpose(2, 0, 1)
    return np.ascontiguousarray(a.astype(np.float32))


def rgb2y(x):
    """``image.rgb2y``: (3,H,W) -> (1,H,W), Y = 0 + 0.299 R, += 0.587 G, += 0.114 B in fp32."""
    x = np.asarray(x, dtype=np.float32)
    assert x.ndim == 3 and x.shape[0] == 3
    y = np.float32(0.299) * x[0]
    y = y + np.float32(0.587) * x[1]
    y = y + np.float32(0.114) * x[2]
    return y[None].astype(np.float32)


def standardise(x):
    """``x:add(-x:mean()):div(x:std())`` (main.lua:1094-1095): double accumulation, unbiased std taken
    AFTER the mean was subtracted, scalars applied in fp32."""
    x = np.asarray(x, dtype=np.float32)
    n = x.size
    assert n > 1
    m = float(x.astype(np.float64).sum() / n)
    x = x + np.float32(-m)
    m2 = x.astype(np.float64).sum() / n
    var = float(((x.astype(np.float64) - m2) ** 2).sum() / (n - 1))
    assert var > 0, "constant image"
    return (x / np.float32(np.sqrt(var))).astype(np.float32)


def make_batch(left, right):
    """main.lua:1085-1100: two image files (or (C,H,W) / (H,W) arrays) -> x_batch (2,1,H,W) float32."""
    out = []
    for v in (left, right):
        a = load_image(v) if isinstance(v, (str, os.PathLike)) else np.asarray(v, dtype=np.float32)
        if a.ndim == 2:
            a = a[None]
        if a.shape[0] == 3:
            a = rgb2y(a)                                                        # :1088-1092
        assert a.shape[0] == 1, "grey or RGB images expected"
        out.append(standardise(a))                                              # :1094-1095
    assert out[0].shape == out[1].shape, "the two views must have the same size"
    return np.ascontiguousarray(np.stack(out))                                  # :1097-1100


def make_batch_cuda(left, right, device=0):
    """:func:`make_batch` on the GPU (csrc/frontend.cu, mccnn_frontend_batch), bit-identical to it: `left` / `right` the decoded
    views as :func:`load_bytes` returns them, (H, W) or (H, W, 3) uint8 numpy arrays or torch tensors (host or device), both
    grey or both colour.  Only the bytes are copied to `device` (a torch.device or index); returns x_batch (2,1,H,W) CUDA
    float32.  Waits for the two views' statistics and refuses a constant view, as :func:`standardise` does."""
    import torch

    from .adcensus import _check, _stream, lib

    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    views = [v if isinstance(v, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(v)) for v in (left, right)]
    for name, v in zip(("left", "right"), views):
        if v.dtype != torch.uint8 or not (v.dim() == 2 or (v.dim() == 3 and v.size(2) == 3)):
            raise ValueError("%s view: (H, W) or (H, W, 3) uint8 expected, got %s %s" % (name, v.dtype, tuple(v.shape)))
    if views[0].shape != views[1].shape:
        raise ValueError("the two views must have the same size and channels, got %s and %s"
                         % (tuple(views[0].shape), tuple(views[1].shape)))
    H, W = views[0].shape[:2]
    nch = 1 if views[0].dim() == 2 else 3
    with torch.cuda.device(dev):
        views = [v.to(dev).contiguous() for v in views]
        x_batch = torch.empty((2, 1, H, W), dtype=torch.float32, device=dev)
        stats = torch.empty((2, 3), dtype=torch.float64, device=dev)
        _check(lib().mccnn_frontend_batch(views[0].data_ptr(), views[1].data_ptr(), nch, H, W, x_batch.data_ptr(),
                                          stats.data_ptr(), _stream(x_batch)), "mccnn_frontend_batch")
        var = stats[:, 2].cpu()
    for name, v in zip(("left", "right"), var.tolist()):
        if not v > 0:
            raise ValueError("%s view: constant image (standardise needs a non-zero variance)" % name)
    return x_batch


def write_bin(path, t):
    """``torch.DiskFile(path,'w'):binary():writeFloat(t:float():storage())``: raw little-endian fp32"""
    np.ascontiguousarray(t, dtype="<f4").tofile(path)


def load_net(net_fname, arch):
    """``torch.load(opt.net_fname, 'ascii')`` (main.lua:893-901) on the host: the :class:`t7.Net` of `net_fname`, which must
    hold a network of architecture `arch` ('fast' or 'slow')."""
    from . import t7

    net = t7.load_net(net_fname)
    if net.arch != arch:
        raise ValueError("%s holds a '%s' network, arch '%s' was asked for" % (net_fname, net.arch, arch))
    return net


def net_border(net):
    """fix_border's width for a network (main.lua:382-391, 923): (window - 1) / 2 = the sum of (kW - 1) / 2 over the
    tower's convolutions (4 for the published 4-layer 3x3 KITTI towers, 5 for Middlebury's 5 layers)."""
    return sum((w.shape[3] - 1) // 2 for w, _ in net.tower)


class StereoMethod:
    """The stereo method of ``main.lua <dataset> <arch> -net_fname N``, decided in one place for every prediction path.

    The constructor does no GPU work: it checks the arch, loads the network of arch 'fast' / 'slow' from `net_fname` and
    checks its arch (main.lua:893-901), and sets ``opt``, the preset of (dataset, arch) with `overrides` and fix_border's
    width from the network (main.lua:382-391, 923; the preset's without a network; an explicit `border` wins).
    :meth:`stages` then builds the network's GPU stages once, and :meth:`close` releases them."""

    def __init__(self, dataset, arch, net_fname=None, **overrides):
        pipeline.check_arch(arch)
        self.dataset, self.arch = dataset, arch
        self.net = load_net(net_fname, arch) if net_fname and arch in ("fast", "slow") else None
        if self.net is not None:
            overrides.setdefault("border", net_border(self.net))
        self.overrides = overrides
        self.opt = self.params()
        self.tower = self.head = None

    @property
    def needs_net(self):
        """arch 'fast' / 'slow' without a network: the tower's input to the stereo method has to come from elsewhere"""
        return self.arch in ("fast", "slow") and self.net is None

    def params(self, **overrides):
        """``opt`` with more `overrides`"""
        return pipeline.make_params(self.dataset, self.arch, **dict(self.overrides, **overrides))

    def stages(self, device):
        """(FeatureTower, ScorerHead or None) of the network on `device` (a torch.device or index), built on the first call --
        net_te, and for 'slow' net_te2 (main.lua:894-900); (None, None) for 'ad' / 'census'."""
        if self.needs_net:
            raise ValueError("arch '%s' needs -net_fname" % self.arch)
        if self.net is not None and self.tower is None:
            import torch

            from .feature_tower import FeatureTower
            from .scorer_head import ScorerHead

            dev = torch.device("cuda", device) if isinstance(device, int) else device
            with torch.cuda.device(dev):
                self.tower = FeatureTower(self.net.tower, arch=self.arch, device=dev.index)
                self.head = ScorerHead(self.net.head, device=dev.index) if self.arch == "slow" else None
        return self.tower, self.head

    def close(self):
        """release the stages :meth:`stages` built"""
        for st in (self.tower, self.head):
            if st is not None:
                st.close()
        self.tower = self.head = None


def predict(left, right, dataset="kitti", arch="census", disp_max=70, features=None, out_dir=None, device=0,
            net_fname=None, confidence=False, calib=None, ply=False, max_depth=None, density=None, rectify=None,
            **overrides):
    """``main.lua <dataset> <arch> -a predict -net_fname N -left L -right R -disp_max D`` from the image files on:
    returns disp (H,W) float32 (numpy).  With `out_dir`, writes right.bin and left.bin ((1,D,H,W), in
    that order, main.lua:1042-1047) and disp.bin ((1,1,H,W), :1103) there.  arch 'fast' / 'slow' take the trained
    network from `net_fname` (the reference's ascii .t7, main.lua:893-901, read by :mod:`t7`) and run it on the GPU
    (feature tower, and for 'slow' the scorer head); arch 'fast' alternatively accepts `features` (2,C,H,W), the
    unit-norm tower output; 'ad' / 'census' need neither.  With `confidence` (an addition beyond the reference), also writes
    conf.bin, the margin confidence of the left volume (mc-cnn_b200/confidence.py), and for presets with the LR check lr.bin,
    main.lua:1056's outlier map, both (1,1,H,W) float32, each announced by a ``Writing`` line in main.lua's format.

    With `calib`, a :data:`dataio.Calib` of the pair (an addition beyond the reference, DESIGN §20), also writes depth.bin,
    the metric depth of disp ((1,1,H,W) float32, NaN = no depth, Z > `max_depth` dropped), and with `ply` points.ply, the
    point cloud coloured from the left image's bytes.  `density` (with `confidence`) keeps in both only the pixels
    confidence.sparsify keeps.

    With `rectify`, a :class:`dataio.StereoRect` of the raw cameras (DESIGN §22), the views are first rectified on the GPU
    (rectify.rectify) and the unchanged path runs on the rectified bytes: every output lies on the rectified grid, `calib`
    is rectify.calib (passing both is refused), the point cloud is coloured from the rectified left bytes, and the pixels
    outside the left view's validity mask have no disparity (NaN in disp.bin and in every map made from it), so no depth and
    no vertex either."""
    import torch

    if rectify is not None:
        if calib is not None:
            raise ValueError("rectify defines the calibration of the rectified pair: pass rectify or calib, not both")
        calib = rectify.calib
    if (ply or max_depth is not None or density is not None) and calib is None:
        raise ValueError("ply, max_depth and density apply to the depth outputs, which need calib")
    if density is not None and not confidence:
        raise ValueError("density ranks pixels by their confidence: it needs confidence")
    colour = None
    if rectify is not None:
        left, right = (load_bytes(v) if isinstance(v, (str, os.PathLike)) else np.asarray(v) for v in (left, right))
        rectify.check_size(left.shape[0], left.shape[1], "rectify")
    elif calib is not None:
        colour = load_bytes(left) if isinstance(left, (str, os.PathLike)) else np.asarray(left)
        dataio.check_calib_size(calib, colour.shape[0], colour.shape[1], "calib")
    method = StereoMethod(dataset, arch, None if features is not None else net_fname, **overrides)   # before any GPU work
    if method.needs_net and features is None:
        raise ValueError("arch '%s' needs -net_fname (or, for 'fast', the tower output in `features`)" % arch)
    if method.needs_net and arch == "slow":
        raise ValueError("arch 'slow' needs -net_fname: the scorer head's weights come with the tower's")

    dev = torch.device("cuda", device)
    valid = None
    if rectify is not None:
        from .rectify import rectify as rectify_pair

        left, right, valid = rectify_pair(left, right, rectify, dev)
        colour = left
        x_batch = make_batch_cuda(left, right, dev)
    else:
        x_batch = torch.from_numpy(make_batch(left, right)).to(dev)
    try:
        with torch.cuda.device(dev):
            tower, head = (None, None) if method.needs_net else method.stages(dev)
            feats = None
            if tower is not None:
                feats = tower.forward(x_batch)                                  # main.lua:944 / :957
            elif arch == "fast":
                feats = torch.as_tensor(features, dtype=torch.float32).to(dev).contiguous()
            H, W = x_batch.shape[2:]
            conf = torch.empty((H, W), device=dev) if confidence else None
            lr = torch.empty((H, W), device=dev) if confidence and method.opt.lr_check else None
            disp, volL, volR = pipeline.stereo_predict(x_batch, feats, method.opt, int(disp_max), want_vols=True, arch=arch,
                                                       head=head, conf=conf, lr=lr)
            if valid is not None:                                               # before density and depth
                disp = disp.masked_fill(valid.reshape(disp.shape) == 0, float("nan"))
            Z = pts = None
            if calib is not None:
                dmap = disp.reshape(H, W) if density is None else confidence_.sparsify(disp.reshape(H, W), conf, density)
                Z = depth.depth(dmap, calib, max_depth)
                if ply:
                    pts = depth.point_cloud(dmap, calib, colour, max_depth=max_depth)
        disp_h = disp.cpu().numpy()
    finally:
        method.close()
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
        write_bin(os.path.join(out_dir, "right.bin"), volR.cpu().numpy())       # direction 1 comes first
        write_bin(os.path.join(out_dir, "left.bin"), volL.cpu().numpy())
        write_bin(os.path.join(out_dir, "disp.bin"), disp_h)
        for name, t in (("conf", conf), ("lr", lr)):
            if t is not None:
                print("Writing %s.bin, 1 x 1 x %d x %d" % (name, H, W), flush=True)
                write_bin(os.path.join(out_dir, name + ".bin"), t.cpu().numpy())
        if Z is not None:
            print("Writing depth.bin, 1 x 1 x %d x %d" % (H, W), flush=True)
            write_bin(os.path.join(out_dir, "depth.bin"), Z.cpu().numpy())
        if pts is not None:
            print("Writing points.ply, %d points" % pts.n, flush=True)
            depth.write_ply(os.path.join(out_dir, "points.ply"), pts)
    return disp_h[0, 0]
