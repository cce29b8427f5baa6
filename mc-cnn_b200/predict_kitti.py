"""predict_kitti.lua in one process: a trained network over every full-size raw KITTI pair.

    res = predict_kitti("test", "kitti", net_fname="net/net_kitti_fast_-a_train_all.t7", data_root="/data")
    # prints "i<TAB>err" per training pair (0-based), then the mean 3-pixel error; res.errors, res.mean
    files = predict_kitti("submit", "kitti2015", net_fname=N, data_root="/data", out="out")   # out/disp_0/%06d_10.png

The script runs ``main.lua kitti fast -a predict -disp_max 228`` once per pair, reloading the network each time.  Here the
network and the stereo method are built once (:class:`evaluate.Evaluator`: for arch 'fast' one pipeline created at the
largest (H, W, disp_max) of the set, then run at each pair's own size; 'slow', 'census' and 'ad' through the operator
chain; fix_border's width from the net), and each pair goes

    PNG decode (host, a background thread working one pair ahead) -> the bytes to the GPU -> frontend.make_batch_cuda ->
    Evaluator.stereo_predict -> (test) the bad / valid pixel counts on the device, one pair of numbers read back
                                (submit) the map read back and written by dataio.write_kitti_submission

Files are those of preprocess_kitti.lua (:mod:`preprocess`'s LAYOUT and input_files): 2012 grey image_0 / image_1 with
disp_noc, 2015 RGB image_2 / image_3 (through rgb2y) with disp_noc_0; ``test`` reads ``training/``, ``submit``
``testing/``.  Images keep their own sizes (nothing is cropped).  Each error is dataio.bad_pixel_rate(disp,
read_png16(disp_noc), 3) over the whole image, and the mean is accumulated in pair order as the script's err_sum.

Under torch.distributed (one process per GPU, e.g. torchrun) the pairs are shared round-robin (batch.run_sharded); each
rank returns only its counts, or the indices of the files it wrote, and rank 0 prints in pair order what one process
prints.

Deliberate deviations from predict_kitti.lua: KITTI 2015 and archs other than 'fast' are accepted; missing files, views of
different sizes and a ground truth of another size are refused before any GPU work; ``submit`` refuses a non-empty output
directory (as Evaluator.submit does) and also writes 2015 maps, under ``out/disp_0/``.

An addition beyond the reference: ``submit`` with `density` p in (0, 1] writes sparse maps, the ceil(p H W) pixels of
largest margin confidence and 0 (the PNG16 invalid value) elsewhere (:func:`confidence.sparsify`).

Another addition: with `depth`, either action also writes each pair's metric depth as ``out/depth_0/%06d_10.png`` (KITTI's
depth format, dataio.write_depth_png16: round(Z * 256), 0 = none), and with `ply` its coloured point cloud as
``out/points_0/%06d_10.ply`` (:mod:`depth`), both from the map submit writes (the sparse one under `density`).  The
calibration is read from beside the images: ``calib/%06d.txt`` (2012, in the data archive) or ``calib_cam_to_cam/%06d.txt``
(2015, from the calibration archive data_scene_flow_calib.zip unpacked into the same ``unzip/`` directory).
"""
import concurrent.futures
import os
from collections import namedtuple

import numpy as np

from . import batch, confidence, dataio, evaluate, frontend, preprocess, rectify
from . import depth as depth_

ACTIONS = ("test", "submit")
DISP_MAX = 228                          # predict_kitti.lua:37
ERR_AT = 3.0                            # :67

TestResult = namedtuple("TestResult", "errors mean")


def pair_files(data_root, dataset, action):
    """[(left, right, disp_noc or None)] of the training pairs (test) or the testing pairs (submit), in index order"""
    sub = "training" if action == "test" else "testing"
    return [f[2:] for f in preprocess.input_files(data_root, dataset) if f[0] == sub]


def _header(path):
    from PIL import Image

    with Image.open(path) as im:
        return im.size[::-1], im.mode in ("L", "1", "P", "LA", "I;16", "I;16B", "I")


def scan(files):
    """(H, W) of every pair from the PNG headers.  Refuses views of different sizes, a grey view paired with a colour one,
    and a ground truth whose size is not the images'."""
    shapes = []
    for left, right, gt in files:
        (shape, grey), (shape_r, grey_r) = _header(left), _header(right)
        if shape != shape_r:
            raise ValueError("%s is %dx%d, %s is %dx%d" % (left, shape[0], shape[1], right, shape_r[0], shape_r[1]))
        if grey != grey_r:
            raise ValueError("%s and %s: one view is grey, the other colour" % (left, right))
        if gt is not None and _header(gt)[0] != shape:
            raise ValueError("%s is %dx%d, the images are %dx%d" % (gt, *_header(gt)[0], *shape))
        if shape[0] * shape[1] >= 1 << 24:      # the counts travel between ranks as float32
            raise ValueError("%s: %dx%d pixels, more than this tool counts" % (left, shape[0], shape[1]))
        shapes.append(shape)
    return shapes


def decode(pair):
    """(left bytes, right bytes, ground truth uint16 or None) of one pair"""
    left, right, gt = pair
    return frontend.load_bytes(left), frontend.load_bytes(right), dataio.read_png16_raw(gt) if gt is not None else None


class Prefetch:
    """decode() of the pairs in `order`: get(i) returns pair i, and first starts decoding the pair after it in a background
    thread, so that the next pair's PNGs are decoded while this one runs on the GPU.  enabled=False decodes in get()."""

    def __init__(self, files, order, enabled=True):
        self.files, self.order = files, list(order)
        self.pos = {i: k for k, i in enumerate(self.order)}
        self.pool = concurrent.futures.ThreadPoolExecutor(max_workers=1) if enabled else None
        self.pending = {}

    def _start(self, i):
        if i not in self.pending:
            self.pending[i] = self.pool.submit(decode, self.files[i])

    def get(self, i):
        if self.pool is None:
            return decode(self.files[i])
        self._start(i)
        k = self.pos[i] + 1
        if k < len(self.order):
            self._start(self.order[k])
        return self.pending.pop(i).result()

    def close(self):
        if self.pool is not None:
            for f in self.pending.values():
                f.cancel()
            self.pool.shutdown(wait=True)


class PairRunner:
    """The stereo method of (dataset, arch, net) over a list of pairs, shared by every tool that predicts a sequence of
    image files: one :class:`evaluate.Evaluator` prepared at the largest (H, W, disp_max) of `shapes`, and this rank's
    pairs (``batch.shard_indices`` of `rank`, `world`) decoded one ahead in a background thread (:class:`Prefetch`).
    :meth:`predict` gives one pair's device map; :meth:`close` releases both.

    `rects` (DESIGN §22), one :class:`dataio.StereoRect` or None per pair: a pair that has one is decoded on the host as
    usual, rectified on the device (rectify.rectify) before make_batch_cuda, and its map is NaN outside the left view's
    validity mask; `shapes` are then the rectified shapes the pipeline runs at."""

    def __init__(self, files, shapes, dataset, arch, net_fname, disp_max, device, rank, world, prefetch=True, rects=None,
                 **overrides):
        self.ev = evaluate.Evaluator(dataset, arch, net_fname=net_fname, device=device, **overrides)
        self.dev = self.ev.dev
        self.disp_max = int(disp_max)
        self.pre = Prefetch(files, batch.shard_indices(len(files), rank, world), enabled=prefetch)
        self.shapes = [(H, W, self.disp_max) for H, W in shapes]
        self.rects = rects

    def prepare(self):
        self.ev.prepare(self.shapes)

    def predict(self, i, conf=False):
        """(left bytes, right bytes, ground truth or None, the (H, W) device map, its margin confidence or None) of pair i"""
        import torch

        left, right, gt = self.pre.get(i)
        rect = self.rects[i] if self.rects is not None else None
        if rect is not None:
            left, right, valid = rectify.rectify(left, right, rect, self.dev)
        x_batch = frontend.make_batch_cuda(left, right, self.dev)
        c = None
        if conf:
            c = torch.empty(x_batch.shape[2:], device=self.dev)
            pred = self.ev.stereo_predict(x_batch, self.disp_max, conf=c)
        else:
            pred = self.ev.stereo_predict(x_batch, self.disp_max)
        if rect is not None:
            pred = pred.masked_fill(valid == 0, float("nan"))
        return left, right, gt, pred, c

    def close(self):
        self.pre.close()
        self.ev.close()


CALIB_DIR = {"kitti": "calib", "kitti2015": "calib_cam_to_cam"}


def calib_file(left, dataset):
    """the calibration file of the pair whose left image is `left` (``<sub>/image_*/%06d_10.png``)"""
    sub = os.path.dirname(os.path.dirname(left))
    return os.path.join(sub, CALIB_DIR[dataset], os.path.basename(left)[:6] + ".txt")


def read_calibs(files, shapes, dataset):
    """the :data:`dataio.Calib` of every pair, refused (naming the file) when missing, malformed or of another size"""
    out = []
    for (left, _, _), (H, W) in zip(files, shapes):
        path = calib_file(left, dataset)
        if not os.path.isfile(path):
            raise FileNotFoundError("missing calibration file %s" % path)
        cal = dataio.read_calib(path, dataset)
        dataio.check_calib_size(cal, H, W, path)
        out.append(cal)
    return out


def depth_files(out, i):
    """(depth PNG, point cloud) of pair i"""
    return (os.path.join(out, "depth_0", "%06d_10.png" % i), os.path.join(out, "points_0", "%06d_10.ply" % i))


def write_depth(pred, left, cal, out, i, ply):
    """pair i's depth PNG, and with `ply` its point cloud, from the device map `pred`"""
    fz, fp = depth_files(out, i)
    os.makedirs(os.path.dirname(fz), exist_ok=True)
    dataio.write_depth_png16(depth_.depth(pred, cal).cpu().numpy(), fz)
    if ply:
        os.makedirs(os.path.dirname(fp), exist_ok=True)
        depth_.write_ply(fp, depth_.point_cloud(pred, cal, left))


def error_counts(disp, gt16, err_at=ERR_AT):
    """(bad, valid) pixel counts of one device map against its PNG16 ground truth (mccnn_kitti_error_count): disp (H, W) CUDA
    float32, gt16 (H, W) uint16 values (numpy, or an int16 / uint16 torch tensor).  Returns a (2,) int64 CUDA tensor."""
    import torch

    from .adcensus import _check, _stream, _t, lib

    name = "mccnn_kitti_error_count"
    p = _t(disp, 1, name)
    if disp.dim() != 2:
        raise ValueError("%s: disp must be (H, W), got %s" % (name, tuple(disp.shape)))
    if isinstance(gt16, np.ndarray):
        gt16 = torch.from_numpy(np.ascontiguousarray(gt16, dtype=np.uint16).view(np.int16))
    if tuple(gt16.shape) != tuple(disp.shape) or gt16.element_size() != 2:
        raise ValueError("%s: ground truth (H, W) 16-bit %s expected, got %s %s"
                         % (name, tuple(disp.shape), gt16.dtype, tuple(gt16.shape)))
    H, W = disp.shape
    with torch.cuda.device(disp.device):
        g = gt16.to(disp.device).contiguous()
        counts = torch.empty(2, dtype=torch.int64, device=disp.device)
        _check(lib().mccnn_kitti_error_count(p, g.data_ptr(), H, W, err_at, counts.data_ptr(), _stream(disp)), name)
    return counts


def error_rate(bad, valid):
    """bad / valid as predict_kitti.lua computes it (0 / 0 is NaN there as well)"""
    return float(bad) / valid if valid else float("nan")


def report(action, n, compute, rank=None, world=None, submission_file=None, verbose=True):
    """batch.run_sharded(n, compute): compute(i) gives pair i's (bad, valid) counts (test) or its index once written
    (submit).  On rank 0 prints predict_kitti.lua's lines in pair order and returns the TestResult / the list of written
    files (``submission_file(i)``); other ranks return None."""
    import torch.distributed as dist

    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    res = batch.run_sharded(n, compute, rank, world)
    if rank != 0:
        return None
    if action == "submit":
        files = []
        for i, r in enumerate(res):
            assert int(r.reshape(-1)[0]) == i, "pair %d came back as %s" % (i, r)
            files.append(submission_file(i))
            if verbose:
                print(i, flush=True)                                            # :77
        return files
    errors, err_sum = [], 0.0
    for i, r in enumerate(res):
        bad, valid = (int(v) for v in r.reshape(-1).tolist())
        errors.append(error_rate(bad, valid))
        err_sum = err_sum + errors[-1]                                           # :69, in pair order
        if verbose:
            print("%d\t%s" % (i, evaluate.lua_num(errors[-1])), flush=True)      # :70
    mean = err_sum / n if n else float("nan")
    if verbose:
        print(evaluate.lua_num(mean), flush=True)                                # :85
    return TestResult(errors, mean)


def check_out(out):
    """submit's output directory: refused when it holds anything but ``.empty``"""
    if os.path.isdir(out) and any(f != ".empty" for f in os.listdir(out)):
        raise ValueError("submit: output directory %s is not empty" % out)


def predict_kitti(action, dataset, net_fname=None, arch="fast", data_root=".", out="out", disp_max=DISP_MAX, device=0,
                  prefetch=True, verbose=True, density=None, depth=False, ply=False, **overrides):
    """predict_kitti.lua's `test` or `submit` on the raw `dataset` ('kitti' or 'kitti2015') under `data_root` on CUDA device
    `device`; `overrides` change the stereo method's preset as in Evaluator.  Returns, on rank 0, the TestResult (errors per
    training pair, mean) or the list of written files; None on other ranks.  `prefetch` False decodes each pair in turn.
    `depth` / `ply` also write the depth maps / point clouds (module docstring)."""
    import torch
    import torch.distributed as dist

    if action not in ACTIONS:
        raise ValueError("action must be 'test' or 'submit', got %r" % (action,))
    if dataset not in preprocess.LAYOUT:
        raise ValueError("dataset must be 'kitti' or 'kitti2015', got %r" % (dataset,))
    if int(disp_max) < 1:
        raise ValueError("disp_max must be at least 1, got %r" % (disp_max,))
    if density is not None:
        if action != "submit":
            raise ValueError("density applies to the maps submit writes; %s writes none" % action)
        confidence.check_density(density)
    if ply and not depth:
        raise ValueError("ply writes the point clouds of the depth maps: it needs depth")
    files = pair_files(data_root, dataset, action)
    shapes = scan(files)
    calibs = read_calibs(files, shapes, dataset) if depth else None
    distributed = dist.is_initialized() and dist.get_world_size() > 1
    if action == "submit" or depth:
        check_out(out)
        if distributed:
            dist.barrier()                      # every rank has looked at `out` before any rank writes to it
    rank = dist.get_rank() if distributed else 0
    world = dist.get_world_size() if distributed else 1
    run = PairRunner(files, shapes, dataset, arch, net_fname, disp_max, device, rank, world, prefetch, **overrides)
    submission_file = lambda i: os.path.join(out if dataset == "kitti" else os.path.join(out, "disp_0"), "%06d_10.png" % i)

    def compute(i):
        left, _, gt, pred, conf = run.predict(i, conf=density is not None)
        if action == "test":
            if depth:
                with torch.cuda.device(run.dev):
                    write_depth(pred, left, calibs[i], out, i, ply)
            return error_counts(pred, gt).cpu()
        if density is not None:
            with torch.cuda.device(run.dev):
                pred = confidence.sparsify(pred, conf, density, 0.0)
        if depth:
            with torch.cuda.device(run.dev):
                write_depth(pred, left, calibs[i], out, i, ply)
        H, W = shapes[i]
        f = dataio.write_kitti_submission(pred.cpu().numpy(), H, W, out, i, dataset)
        assert f == submission_file(i)
        return torch.tensor([i])

    try:
        run.prepare()
        return report(action, len(files), compute, rank, world, submission_file, verbose)
    finally:
        run.close()
