"""The KITTI 2012 / 2015 devkits' stereo metrics on the training pairs, on the GPU.

    res = evaluate_training("kitti", "net/net_kitti_fast_-a_train_all.t7", "fast", data_root="/data")
    # prints one tab-separated line of rates per training pair (0-based), then the devkit's table; res.pairs, res.total
    res = evaluate_training("kitti2015", N, "fast", data_root="/data", out="out")     # also out/disp_0/%06d_10.png
    res = score_dir("kitti2015", "out", data_root="/data")                            # the same table from those files

main.lua and predict_kitti.lua print one number per pair, the share of non-occluded pixels more than 3 px off, taken on the
float map.  The KITTI servers score what they receive instead, the PNG16 map, after filling its invalid pixels by the
devkit's background interpolation:

* KITTI 2012: Out-Noc / Out-All at 2, 3, 4 and 5 px, Avg-Noc / Avg-All (mean absolute error in px) and the density;
* KITTI 2015: D1 (bad when the error is > 3 px and > 5 % of the true disparity) for background, foreground and all pixels,
  against the non-occluded ('noc') and the full ('all') ground truth, and the density.

The definitions are oracle/kitti_devkit.py's docstring (DESIGN.md §17); parity with the devkit binaries is not pinned.  Per
pair, :func:`devkit_counts` runs mccnn_kitti_devkit_counts (csrc/kitti_eval.cu): the map quantised as
dataio.write_png16 stores it, interpolated, and scored into integer counts and float64 error sums on the device.  Rates are
quotients of counts; totals over a set are pixel-weighted (the counts and sums added over the pairs, then divided).  Every
number is printed with evaluate.lua_num and is a fraction (the Avg columns are in px).

:func:`evaluate_training` runs predict_kitti.py test's loop (the same Evaluator, front end and PNG prefetch) and scores each
map; :func:`score_dir` scores PNG16 maps already written in submission layout (``D/%06d_10.png`` for 2012,
``D/disp_0/%06d_10.png`` for 2015).  Under torch.distributed the pairs are shared round-robin (batch.run_sharded) and rank 0
prints in pair order.  Missing ground-truth files (disp_occ / disp_occ_0, and obj_map for 2015), files of the wrong kind and
size mismatches are refused before any GPU work.
"""
import os
from collections import OrderedDict, namedtuple

import numpy as np

from . import batch, confidence, dataio, evaluate, frontend, predict_kitti, preprocess

DATASETS = ("kitti", "kitti2015")
GT_OCC = {"kitti": "disp_occ", "kitti2015": "disp_occ_0"}
OBJ_MAP = "obj_map"                     # KITTI 2015 only

# the count layout of mccnn_kitti_devkit_counts (include/adcensus_b200.h): counts[r, k], r 0 = noc, 1 = all
GT, DENSE, OUT2, OUT3, OUT4, OUT5, D1_BG, D1_FG, GT_BG, GT_FG = range(10)
NCOUNT = 10
REGIONS = ("noc", "all")
THRESHOLDS = (2, 3, 4, 5)
OUT = dict(zip(THRESHOLDS, (OUT2, OUT3, OUT4, OUT5)))

Counts = namedtuple("Counts", "counts sums")           # (2, NCOUNT) int64 and (2,) float64 CUDA tensors
Scores = namedtuple("Scores", "pairs total counts sums")  # per-pair rate dicts, the set's rates, its summed counts and sums


def _u16(x, dev, name, what):
    """a (H, W) 16-bit device tensor of the stored values x (numpy uint16, or an int16 / uint16 tensor)"""
    import torch

    if isinstance(x, np.ndarray):
        if x.dtype != np.uint16:
            raise ValueError("%s: %s must be uint16, got %s" % (name, what, x.dtype))
        x = torch.from_numpy(np.ascontiguousarray(x).view(np.int16))
    if not isinstance(x, torch.Tensor) or x.element_size() != 2 or x.is_floating_point():
        raise ValueError("%s: %s must be 16-bit integer values" % (name, what))
    return x.to(dev).contiguous()


def devkit_counts(disp_or_png16, gt_noc16, gt_occ16, obj_map=None, ipol=None, device=None):
    """The devkit's counts of one estimate: `disp_or_png16` a (H, W) CUDA float32 map (quantised as write_png16 stores it)
    or the stored uint16 values (numpy, or an int16 / uint16 tensor); gt_noc16 / gt_occ16 the ground truths' stored values;
    obj_map (H, W) 8-bit or None (all background).  `ipol`, a (H, W) CUDA float32 tensor, receives the interpolated
    estimate.  Runs on the float map's device, else on `device` (default: the current one), asynchronously on its current
    stream.  Returns Counts(counts (2, NCOUNT) int64, sums (2,) float64), CUDA tensors."""
    import torch

    from .adcensus import _check, _stream, lib

    name = "mccnn_kitti_devkit_counts"
    is_float = isinstance(disp_or_png16, torch.Tensor) and disp_or_png16.is_floating_point()
    if is_float:
        if not disp_or_png16.is_cuda or disp_or_png16.dtype != torch.float32:
            raise ValueError("%s: a float map must be a CUDA float32 tensor" % name)
        dev = disp_or_png16.device
    else:
        dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
    shape = tuple(disp_or_png16.shape)
    if len(shape) != 2:
        raise ValueError("%s: the estimate must be (H, W), got %s" % (name, shape))
    H, W = shape
    with torch.cuda.device(dev):
        disp = disp_or_png16.contiguous() if is_float else None
        disp16 = None if is_float else _u16(disp_or_png16, dev, name, "the estimate")
        noc, occ = _u16(gt_noc16, dev, name, "gt_noc16"), _u16(gt_occ16, dev, name, "gt_occ16")
        obj = None
        if obj_map is not None:
            obj = torch.as_tensor(np.ascontiguousarray(obj_map) if isinstance(obj_map, np.ndarray) else obj_map)
            if obj.dtype != torch.uint8:
                raise ValueError("%s: obj_map must be 8-bit, got %s" % (name, obj.dtype))
            obj = obj.to(dev).contiguous()
        for what, t in (("gt_noc16", noc), ("gt_occ16", occ), ("obj_map", obj), ("ipol", ipol)):
            if t is not None and tuple(t.shape) != shape:
                raise ValueError("%s: %s is %s, the estimate %s" % (name, what, tuple(t.shape), shape))
        if ipol is not None and (not ipol.is_cuda or ipol.device != dev or ipol.dtype != torch.float32
                                 or not ipol.is_contiguous()):
            raise ValueError("%s: ipol must be a contiguous float32 tensor on %s" % (name, dev))
        counts = torch.empty((2, NCOUNT), dtype=torch.int64, device=dev)
        sums = torch.empty(2, dtype=torch.float64, device=dev)
        ptr = lambda t: None if t is None else t.data_ptr()
        stream = _stream(disp if is_float else noc)
        _check(lib().mccnn_kitti_devkit_counts(ptr(disp), ptr(disp16), noc.data_ptr(), occ.data_ptr(), ptr(obj), H, W,
                                               ptr(ipol), counts.data_ptr(), sums.data_ptr(), stream), name)
    return Counts(counts, sums)


# ---- rates and the printed table ----------------------------------------------------------------------------------------


def columns(dataset):
    """the names of the per-pair line's rates, in order"""
    if dataset == "kitti":
        return (["out_noc_%d" % t for t in THRESHOLDS] + ["out_all_%d" % t for t in THRESHOLDS]
                + ["avg_noc", "avg_all", "density"])
    return ["d1_%s_%s" % (part, r) for r in REGIONS for part in ("bg", "fg", "all")] + ["density"]


def rates(counts, sums, dataset):
    """OrderedDict {column: rate} of host counts (2, NCOUNT) and sums (2,); 0 / 0 is NaN.  Density is taken against the
    full ('all') ground truth."""
    c = np.asarray(counts, dtype=np.int64).reshape(2, NCOUNT)
    s = np.asarray(sums, dtype=np.float64).reshape(2)
    q = predict_kitti.error_rate
    out = OrderedDict()
    if dataset == "kitti":
        for r, reg in enumerate(REGIONS):
            for t in THRESHOLDS:
                out["out_%s_%d" % (reg, t)] = q(c[r, OUT[t]], c[r, GT])
        for r, reg in enumerate(REGIONS):
            out["avg_%s" % reg] = float(s[r]) / int(c[r, GT]) if c[r, GT] else float("nan")
    else:
        for r, reg in enumerate(REGIONS):
            out["d1_bg_%s" % reg] = q(c[r, D1_BG], c[r, GT_BG])
            out["d1_fg_%s" % reg] = q(c[r, D1_FG], c[r, GT_FG])
            out["d1_all_%s" % reg] = q(c[r, D1_BG] + c[r, D1_FG], c[r, GT])
    out["density"] = q(c[1, DENSE], c[1, GT])
    return out


def pair_line(i, r):
    return "\t".join([str(i)] + [evaluate.lua_num(v) for v in r.values()])


def table(r, dataset):
    """the devkit's summary table of the rates r, as lines"""
    n = evaluate.lua_num
    if dataset == "kitti":
        lines = ["Error\tOut-Noc\tOut-All\tAvg-Noc\tAvg-All"]
        for t in THRESHOLDS:
            lines.append("%d px\t%s\t%s\t%s\t%s" % (t, n(r["out_noc_%d" % t]), n(r["out_all_%d" % t]), n(r["avg_noc"]),
                                                    n(r["avg_all"])))
    else:
        lines = ["Error\tD1-bg\tD1-fg\tD1-all"]
        for reg in REGIONS:
            lines.append("%s\t%s\t%s\t%s" % (reg, n(r["d1_bg_%s" % reg]), n(r["d1_fg_%s" % reg]), n(r["d1_all_%s" % reg])))
    lines.append("Density\t%s" % n(r["density"]))
    return lines


# run_sharded gathers float32: the counts are exact there (each < 2^24, checked with the sizes), the float64 sums travel
# as four 16-bit words each
def _pack(c):
    import torch

    counts = c.counts.cpu().numpy().reshape(-1)
    words = np.ascontiguousarray(c.sums.cpu().numpy(), dtype="<f8").view("<u2")
    return torch.from_numpy(np.concatenate([counts, words]).astype(np.float32))


def _unpack(t):
    v = t.reshape(-1).cpu().numpy()
    counts = v[:2 * NCOUNT].astype(np.int64).reshape(2, NCOUNT)
    sums = v[2 * NCOUNT:].astype("<u2").view("<f8").astype(np.float64)
    return counts, sums


def report(dataset, n, compute, rank=None, world=None, verbose=True):
    """batch.run_sharded(n, compute), compute(i) giving _pack(devkit_counts(...)) of pair i.  On rank 0 prints the per-pair
    lines in pair order and the table of the totals, and returns the Scores; other ranks return None."""
    import torch.distributed as dist

    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    res = batch.run_sharded(n, compute, rank, world)
    if rank != 0:
        return None
    pairs = []
    total_c, total_s = np.zeros((2, NCOUNT), np.int64), np.zeros(2, np.float64)
    for i, t in enumerate(res):
        c, s = _unpack(t)
        total_c += c
        total_s = total_s + s                               # in pair order
        pairs.append(rates(c, s, dataset))
        if verbose:
            print(pair_line(i, pairs[-1]), flush=True)
    total = rates(total_c, total_s, dataset)
    if verbose:
        print("\n".join(table(total, dataset)), flush=True)
    return Scores(pairs, total, total_c, total_s)


# ---- files ----------------------------------------------------------------------------------------------------------------

_PNG16 = ("I;16", "I;16B", "I")


def _png(path):
    """(H, W), mode of a PNG's header"""
    from PIL import Image

    with Image.open(path) as im:
        return im.size[::-1], im.mode


def _check_dataset(dataset):
    if dataset not in DATASETS:
        raise ValueError("dataset must be 'kitti' or 'kitti2015', got %r" % (dataset,))


def training_files(data_root, dataset):
    """[(left, right, disp_noc, disp_occ, obj_map or None)] of the raw training pairs in index order; refuses a missing
    file"""
    _check_dataset(dataset)
    sub = os.path.join(data_root, preprocess.LAYOUT[dataset]["path"], "unzip", "training")
    out = []
    for left, right, noc in predict_kitti.pair_files(data_root, dataset, "test"):
        name = os.path.basename(noc)
        occ = os.path.join(sub, GT_OCC[dataset], name)
        obj = os.path.join(sub, OBJ_MAP, name) if dataset == "kitti2015" else None
        for p in (occ, obj):
            if p is not None and not os.path.exists(p):
                raise FileNotFoundError("missing input file %s" % p)
        out.append((left, right, noc, occ, obj))
    return out


def check_maps(files, shapes):
    """Refuses a ground truth or estimate that is not a 16-bit grey PNG, an obj_map that is not 8-bit and any of them whose
    size is not the pair's.  files[i]: (estimate or None, disp_noc, disp_occ, obj_map or None); shapes[i]: (H, W)."""
    for f, shape in zip(files, shapes):
        if shape[0] * shape[1] >= 1 << 24:          # the counts travel between ranks as float32
            raise ValueError("%s: %dx%d pixels, more than this tool counts" % (f[1], shape[0], shape[1]))
        for k, p in enumerate(f):
            if p is None:
                continue
            size, mode = _png(p)
            if k < 3 and mode not in _PNG16:
                raise ValueError("%s: 16-bit grey PNG expected, got mode %s" % (p, mode))
            if k == 3 and mode not in ("L", "P"):
                raise ValueError("%s: 8-bit PNG expected, got mode %s" % (p, mode))
            if size != tuple(shape):
                raise ValueError("%s is %dx%d, the pair is %dx%d" % (p, size[0], size[1], shape[0], shape[1]))


def _read_obj(path):
    from PIL import Image

    with Image.open(path) as im:
        return np.array(im, dtype=np.uint8)


def _decode_maps(f):
    """the ground truth predict_kitti.decode does not read: disp_occ's values and the obj_map (or None)"""
    occ, obj = f
    return dataio.read_png16_raw(occ), None if obj is None else _read_obj(obj)


def _decode_score(f):
    est, noc, occ, obj = f
    return (dataio.read_png16_raw(est), dataio.read_png16_raw(noc), dataio.read_png16_raw(occ),
            None if obj is None else _read_obj(obj))


class _Prefetch(predict_kitti.Prefetch):
    """predict_kitti.Prefetch with another decoder"""

    def __init__(self, files, order, decode, enabled=True):
        super().__init__(files, order, enabled)
        self.decode = decode

    def _start(self, i):
        if i not in self.pending:
            self.pending[i] = self.pool.submit(self.decode, self.files[i])

    def get(self, i):
        return self.decode(self.files[i]) if self.pool is None else super().get(i)


def submission_file(out, dataset, i):
    """dataio.write_kitti_submission's file of pair i"""
    return os.path.join(out if dataset == "kitti" else os.path.join(out, "disp_0"), "%06d_10.png" % i)


def _world():
    import torch.distributed as dist

    distributed = dist.is_initialized() and dist.get_world_size() > 1
    return (dist.get_rank(), dist.get_world_size()) if distributed else (0, 1)


# ---- the two entry points -------------------------------------------------------------------------------------------------


def evaluate_training(dataset, net_fname, arch="fast", data_root=".", disp_max=predict_kitti.DISP_MAX, out=None, device=0,
                      prefetch=True, verbose=True, density=None, **overrides):
    """The net over every raw training pair of `dataset` under `data_root` (predict_kitti.py test's loop, on CUDA device
    `device`; `overrides` change the stereo method's preset as in Evaluator), each map scored by devkit_counts.  With `out`,
    each map is also written in submission layout (refused when `out` is not empty), so that score_dir(dataset, out, ...)
    gives the same numbers.  With `density` in (0, 1] (an addition beyond the reference), each map is first made sparse,
    keeping the ceil(density H W) pixels of largest margin confidence (:func:`confidence.sparsify`, 0 elsewhere): what is
    scored and written is the sparse map, whose dropped pixels the devkit fills by its background interpolation.  Returns
    the Scores on rank 0, None on other ranks."""
    import torch
    import torch.distributed as dist

    _check_dataset(dataset)
    if int(disp_max) < 1:
        raise ValueError("disp_max must be at least 1, got %r" % (disp_max,))
    if density is not None:
        confidence.check_density(density)
    files = training_files(data_root, dataset)
    shapes = predict_kitti.scan([f[:3] for f in files])
    check_maps([(None,) + f[2:] for f in files], shapes)
    rank, world = _world()
    if out is not None:
        predict_kitti.check_out(out)
        if world > 1:
            dist.barrier()                      # every rank has looked at `out` before any rank writes to it
    ev = evaluate.Evaluator(dataset, arch, net_fname=net_fname, device=device, **overrides)
    # two decoding threads one pair ahead: predict_kitti's (the views and disp_noc) and one for disp_occ and obj_map, so
    # that the extra maps do not lengthen the host's share of a pair
    order = batch.shard_indices(len(files), rank, world)
    pre = predict_kitti.Prefetch([f[:3] for f in files], order, enabled=prefetch)
    pre_maps = _Prefetch([f[3:] for f in files], order, _decode_maps, enabled=prefetch)
    disp_max = int(disp_max)

    def compute(i):
        left, right, noc = pre.get(i)
        occ, obj = pre_maps.get(i)
        x_batch = frontend.make_batch_cuda(left, right, ev.dev)
        if density is None:
            pred = ev.stereo_predict(x_batch, disp_max)
        else:
            conf = torch.empty(x_batch.shape[2:], device=ev.dev)
            pred = ev.stereo_predict(x_batch, disp_max, conf=conf)
            with torch.cuda.device(ev.dev):
                pred = confidence.sparsify(pred, conf, density, 0.0)
        c = devkit_counts(pred, noc, occ, obj)
        if out is not None:
            H, W = shapes[i]
            f = dataio.write_kitti_submission(pred.cpu().numpy(), H, W, out, i, dataset)
            assert f == submission_file(out, dataset, i)
        return _pack(c)

    try:
        ev.prepare([(H, W, disp_max) for H, W in shapes])
        return report(dataset, len(files), compute, rank, world, verbose)
    finally:
        pre.close()
        pre_maps.close()
        ev.close()


def score_dir(dataset, pred_dir, data_root=".", device=0, prefetch=True, verbose=True):
    """Scores the PNG16 maps in submission layout under `pred_dir` (``%06d_10.png``, under ``disp_0/`` for kitti2015)
    against the raw training ground truth of `dataset` under `data_root`, on CUDA device `device`.  Every training pair
    needs its map.  Returns the Scores on rank 0, None on other ranks."""
    import torch

    _check_dataset(dataset)
    files = []
    for i, (_, _, noc, occ, obj) in enumerate(training_files(data_root, dataset)):
        est = submission_file(pred_dir, dataset, i)
        if not os.path.exists(est):
            raise FileNotFoundError("missing estimate %s" % est)
        files.append((est, noc, occ, obj))
    shapes = [_png(f[1])[0] for f in files]
    check_maps(files, shapes)
    rank, world = _world()
    pre = _Prefetch(files, batch.shard_indices(len(files), rank, world), _decode_score, enabled=prefetch)

    def compute(i):
        with torch.cuda.device(device):
            return _pack(devkit_counts(*pre.get(i), device=device))

    try:
        return report(dataset, len(files), compute, rank, world, verbose)
    finally:
        pre.close()
