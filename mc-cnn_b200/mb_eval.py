"""The MiddEval3 SDK's evaldisp metrics and the website's error quantiles on the 15 training scenes, on the GPU.

    res = evaluate_training("fast", "net/net_mb_fast_-a_train_all.t7", data_root="/data")
    # prints one tab-separated line per scene, then the line of means; res.scenes, res.rows, res.mean
    res = evaluate_training("slow", N, data_root="/data", out="out")    # also out/trainingH/<scene>/disp0MC-CNN-acrt.pfm
    res = score_dir("out", data_root="/data")                          # the same lines from those files

main.lua's test_te reports bad 1.0 on ten half-size 2014 scenes; the Middlebury table reports, per scene and for the
non-occluded ('nonocc') and all pixels, bad 0.5 / 1 / 2 / 4 (invalid pixels counted as bad), the invalid share, avgerr,
rms and the A50 / A90 / A95 / A99 error quantiles, on the MiddEval3 training images.  The definitions are
oracle/mb_evaldisp.py's docstring (DESIGN.md §18); parity with the SDK binary and the website is not pinned.

:func:`evaldisp` runs mccnn_mb_evaldisp (csrc/mb_eval.cu) on one map: integer counts, float64 error sums and the exact
quantiles, on the device.  :func:`metrics` turns them into the reported values.  Every number is printed with
evaluate.lua_num; rates are fractions, avgerr, rms and the quantiles are in pixels of the ground truth's resolution.  The
line of means is the plain mean of each column over the scenes (the website's per-scene weights are not applied).

The ground truth is read from ``<data_root>/data.mb/unzip/MiddEval3/training{F,H}/<scene>/{disp0GT.pfm, mask0nocc.png}``,
where the SDK's MiddEval3-GT0-F.zip / -GT0-H.zip unpack, and ndisp from ``trainingH/<scene>/calib.txt``.  res 'F' (the
website's resolution) compares the half-size map at scale 2, res 'H' at scale 1.  Missing files, PFMs that are not
single-channel, masks that are not 8-bit grey, size ratios other than 1, 2 or 4 and ambiguous maps are refused before any
GPU work.
"""
import os
import re
from collections import OrderedDict, namedtuple

import numpy as np

from . import confidence, dataio, evaluate, preprocess

REGIONS = ("nonocc", "all")
# the count layout of mccnn_mb_evaldisp (include/adcensus_b200.h): counts[r, k], r 0 = nonocc, 1 = all
N, VALID, BAD05, BAD1, BAD2, BAD4, INVALID = range(7)
NCOUNT = 7
THRESHOLDS = (0.5, 1, 2, 4)
BAD = dict(zip(THRESHOLDS, (BAD05, BAD1, BAD2, BAD4)))
PERCENT = (50, 90, 95, 99)
NAMES = ["bad%g" % t for t in THRESHOLDS] + ["invalid", "avgerr", "rms"] + ["A%d" % p for p in PERCENT] + ["coverage"]
RES = {"F": "trainingF", "H": "trainingH"}
GT_FILE, MASK_FILE = "disp0GT.pfm", "mask0nocc.png"

Eval = namedtuple("Eval", "counts sums quantiles")          # (2, NCOUNT) int64, (2, 2) float64, (2, 4) float32
Scores = namedtuple("Scores", "scenes rows mean evals")     # names, per-scene OrderedDicts, their means, host Evals

_SCRATCH = None


def scratch_bytes():
    """MCCNN_MB_EVAL_SCRATCH_BYTES, read from include/adcensus_b200.h"""
    global _SCRATCH
    if _SCRATCH is None:
        from .adcensus import HEADER_PATH

        with open(HEADER_PATH) as f:
            _SCRATCH = int(re.search(r"#define\s+MCCNN_MB_EVAL_SCRATCH_BYTES\s+(\d+)", f.read()).group(1))
    return _SCRATCH


def evaldisp(disp, gt, mask, maxdisp, scratch=None):
    """The SDK's counts of one map: disp (h, w), gt (Hg, Wg) top-down CUDA float32 tensors on one device (+inf = unknown),
    mask (Hg, Wg) CUDA uint8 or None (every pixel non-occluded), maxdisp the scene's ndisp.  `scratch`, a CUDA uint8 tensor
    of scratch_bytes(), is allocated when None.  Asynchronous on the current stream of the map's device.  Returns Eval of
    CUDA tensors: counts (2, NCOUNT) int64, sums (2, 2) float64 (sum(err), sum(err^2)), quantiles (2, 4) float32."""
    import torch

    from .adcensus import _check, _stream, lib

    name = "mccnn_mb_evaldisp"
    for what, t, dtype in (("disp", disp, torch.float32), ("gt", gt, torch.float32), ("mask", mask, torch.uint8)):
        if t is None and what == "mask":
            continue
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or t.dim() != 2:
            raise ValueError("%s: %s must be a (H, W) CUDA %s tensor" % (name, what, dtype))
        if t.device != disp.device:
            raise ValueError("%s: %s is on %s, disp on %s" % (name, what, t.device, disp.device))
    if mask is not None and mask.shape != gt.shape:
        raise ValueError("%s: the mask is %s, the ground truth %s" % (name, tuple(mask.shape), tuple(gt.shape)))
    dev = disp.device
    with torch.cuda.device(dev):
        disp, gt = disp.contiguous(), gt.contiguous()
        mask = None if mask is None else mask.contiguous()
        if scratch is None:
            scratch = torch.empty(scratch_bytes(), dtype=torch.uint8, device=dev)
        elif (scratch.device != dev or scratch.dtype != torch.uint8 or scratch.numel() < scratch_bytes()
              or not scratch.is_contiguous() or scratch.data_ptr() % 8):
            raise ValueError("%s: scratch must be %d contiguous bytes on %s, 8-byte aligned" % (name, scratch_bytes(), dev))
        counts = torch.empty((2, NCOUNT), dtype=torch.int64, device=dev)
        sums = torch.empty((2, 2), dtype=torch.float64, device=dev)
        quantiles = torch.empty((2, len(PERCENT)), dtype=torch.float32, device=dev)
        (h, w), (Hg, Wg) = disp.shape, gt.shape
        _check(lib().mccnn_mb_evaldisp(disp.data_ptr(), h, w, gt.data_ptr(), Hg, Wg,
                                       None if mask is None else mask.data_ptr(), int(maxdisp), counts.data_ptr(),
                                       sums.data_ptr(), quantiles.data_ptr(), scratch.data_ptr(), _stream(disp)), name)
    return Eval(counts, sums, quantiles)


# ---- the reported values and the printed lines -------------------------------------------------------------------------


def columns():
    """the names of a scene line's values, in order"""
    return ["%s_%s" % (r, n) for r in REGIONS for n in NAMES]


def metrics(counts, sums, quantiles, gt_pixels):
    """OrderedDict {column: value} of host counts (2, NCOUNT), sums (2, 2) and quantiles (2, 4) of a ground truth of
    `gt_pixels` pixels; 0 / 0 is NaN"""
    c = np.asarray(counts, dtype=np.int64).reshape(2, NCOUNT)
    s = np.asarray(sums, dtype=np.float64).reshape(2, 2)
    a = np.asarray(quantiles, dtype=np.float32).reshape(2, len(PERCENT))
    q = lambda x, y: float(x) / float(y) if y else float("nan")
    out = OrderedDict()
    for r, reg in enumerate(REGIONS):
        n, inv = int(c[r, N]), int(c[r, INVALID])
        for t in THRESHOLDS:
            out["%s_bad%g" % (reg, t)] = q(c[r, BAD[t]] + inv, n)
        out["%s_invalid" % reg] = q(inv, n)
        out["%s_avgerr" % reg] = q(s[r, 0], n - inv)
        out["%s_rms" % reg] = float(np.sqrt(q(s[r, 1], n - inv)))
        for j, p in enumerate(PERCENT):
            out["%s_A%d" % (reg, p)] = float(a[r, j])
        out["%s_coverage" % reg] = q(n, gt_pixels)
    return out


def mean_row(rows):
    """the plain mean of each column over the scenes (NaN when a scene's value is NaN)"""
    return OrderedDict((k, float(np.mean([r[k] for r in rows])) if rows else float("nan")) for k in columns())


def line(name, row):
    return "\t".join([name] + [evaluate.lua_num(v) for v in row.values()])


# ---- files ----------------------------------------------------------------------------------------------------------------


def _check_res(res):
    if res not in RES:
        raise ValueError("res must be 'F' or 'H', got %r" % (res,))


def training_scenes(data_root):
    """the MiddEval3 training scenes, the directories of ``trainingH``, in name order"""
    base = os.path.join(data_root, preprocess.MB_EVAL, "trainingH")
    return [d for d in preprocess._listdir(base) if os.path.isdir(os.path.join(base, d))]


def scene_dir(data_root, scene, sub="trainingH"):
    return os.path.join(data_root, preprocess.MB_EVAL, sub, scene)


def gt_files(data_root, scene, res="F"):
    """(disp0GT.pfm, mask0nocc.png) of the scene at resolution `res`"""
    _check_res(res)
    d = scene_dir(data_root, scene, RES[res])
    return os.path.join(d, GT_FILE), os.path.join(d, MASK_FILE)


def find_map(out, scene, alg=None):
    """``out/trainingH/<scene>/disp0<alg>.pfm``; without `alg` the scene's only disp0*.pfm"""
    d = os.path.join(out, "trainingH", scene)
    if alg is not None:
        p = os.path.join(d, "disp0%s.pfm" % alg)
        if not os.path.isfile(p):
            raise FileNotFoundError("missing map %s" % p)
        return p
    found = sorted(f for f in os.listdir(d) if f.startswith("disp0") and f.endswith(".pfm")) if os.path.isdir(d) else []
    if not found:
        raise FileNotFoundError("missing map %s" % os.path.join(d, "disp0<ALG>.pfm"))
    if len(found) > 1:
        raise ValueError("%s holds %s: name the method with -alg" % (d, ", ".join(found)))
    return os.path.join(d, found[0])


def check_scene(size, gt, mask):
    """Refuses a ground truth that is missing or not a single-channel PFM, a mask that is missing, not 8-bit grey or not the
    ground truth's size, and a ground truth that is not 1, 2 or 4 times the map's `size` (h, w).  Returns (Hg, Wg)."""
    Hg, Wg = preprocess._pfm_size(gt)
    ms = preprocess._grey_size(mask)
    if ms != (Hg, Wg):
        raise ValueError("%s is %dx%d, the ground truth %dx%d" % (mask, ms[0], ms[1], Hg, Wg))
    h, w = size
    scale = Wg // w
    if scale not in (1, 2, 4) or Wg != scale * w or Hg != scale * h:
        raise ValueError("%s is %dx%d, the map %dx%d: the ratio must be 1, 2 or 4" % (gt, Hg, Wg, h, w))
    if Hg * Wg >= 1 << 31:
        raise ValueError("%s: %dx%d pixels, more than this tool counts" % (gt, Hg, Wg))
    return Hg, Wg


def _read_topdown(path):
    """a PFM's map with top-down rows (PFMs store the bottom row first)"""
    return np.ascontiguousarray(np.flipud(dataio.read_pfm(path)))


def _score(disp, gt_path, mask_path, ndisp, dev):
    """metrics and host Eval of one map (a CUDA tensor) against its ground-truth files"""
    import torch

    gt = torch.from_numpy(_read_topdown(gt_path)).to(dev)
    mask = torch.from_numpy(preprocess._read_grey(mask_path)).to(dev)
    e = evaldisp(disp, gt, mask, ndisp)
    host = Eval(*(t.cpu().numpy() for t in e))
    return metrics(*host, gt.numel()), host


class _Report:
    """collects the scene lines, printing each as it comes, then the line of means"""

    def __init__(self, verbose):
        self.verbose, self.scenes, self.rows, self.evals = verbose, [], [], []

    def add(self, scene, row, ev):
        self.scenes.append(scene)
        self.rows.append(row)
        self.evals.append(ev)
        if self.verbose:
            print(line(scene, row), flush=True)

    def done(self):
        mean = mean_row(self.rows)
        if self.verbose:
            print(line("mean", mean), flush=True)
        return Scores(self.scenes, self.rows, mean, self.evals)


# ---- the two entry points -------------------------------------------------------------------------------------------------


def score_dir(out, data_root=".", res="F", alg=None, device=0, verbose=True):
    """Scores the maps ``out/trainingH/<scene>/disp0<alg>.pfm`` (Evaluator.submit's layout; without `alg` each scene's only
    disp0*.pfm) of every MiddEval3 training scene under `data_root` against the ground truth at resolution `res`, on CUDA
    device `device`.  Prints one line per scene and the line of means; returns the Scores."""
    import torch

    _check_res(res)
    todo = []
    for s in training_scenes(data_root):
        ndisp = preprocess._ndisp(os.path.join(scene_dir(data_root, s), "calib.txt"))
        p = find_map(out, s, alg)
        gt, mask = gt_files(data_root, s, res)
        check_scene(preprocess._pfm_size(p), gt, mask)
        todo.append((s, p, gt, mask, ndisp))
    dev = torch.device("cuda", device)
    rep = _Report(verbose)
    with torch.cuda.device(dev):
        for s, p, gt, mask, ndisp in todo:
            rep.add(s, *_score(torch.from_numpy(_read_topdown(p)).to(dev), gt, mask, ndisp, dev))
    return rep.done()


def evaluate_training(arch, net_fname=None, data_root=".", res="F", out=None, device=0, verbose=True, density=None,
                      **overrides):
    """The net over the 15 MiddEval3 ``trainingH`` pairs, read from the raw files (grey views through the GPU read_im of
    preprocess_mb, disp_max = the scene's ndisp), each map predicted by evaluate.Evaluator at the mb preset of `arch`
    (`overrides` as in Evaluator) on CUDA device `device` and scored at resolution `res`.  With `out` (refused when not
    empty), each map and its runtime are also written as Evaluator.submit writes them, ``out/trainingH/<scene>/
    disp0<method>.pfm`` (rows bottom-up) and ``time<method>.txt``, so that score_dir(out, ...) prints the same lines.
    Prints one line per scene and the line of means; returns the Scores.  With `density` in (0, 1] (an addition beyond the
    reference), each map keeps the ceil(density H W) pixels of largest margin confidence and holds +inf, the SDK's invalid
    value, elsewhere (:func:`confidence.sparsify`, after the timed region); that map is scored and written."""
    import torch

    _check_res(res)
    if density is not None:
        confidence.check_density(density)
    todo = []
    for s in training_scenes(data_root):
        d = scene_dir(data_root, s)
        views = [os.path.join(d, "im0.png"), os.path.join(d, "im1.png")]
        size = preprocess._same_size(s, [(p, preprocess._image_size(p)) for p in views])
        ndisp = preprocess._ndisp(os.path.join(d, "calib.txt"))
        gt, mask = gt_files(data_root, s, res)
        check_scene(size, gt, mask)
        todo.append((s, views, size, ndisp, gt, mask))
    if out is not None and os.path.isdir(out) and any(f != ".empty" for f in os.listdir(out)):
        raise ValueError("output directory %s is not empty" % out)
    ev = evaluate.Evaluator("mb", arch, net_fname=net_fname, device=device, **overrides)
    rep = _Report(verbose)
    try:
        ev.prepare([size + (ndisp,) for _, _, size, ndisp, _, _ in todo])
        with torch.cuda.device(ev.dev):
            for s, views, size, ndisp, gt, mask in todo:
                x = preprocess._mb_views(dict(groups=[(views, (2,))], half=False), "gray", ev.dev)[0]
                conf = None if density is None else torch.empty(size, device=ev.dev)
                pred, runtime = ev.timed(torch.from_numpy(np.ascontiguousarray(x)).to(ev.dev), ndisp, conf=conf)
                if conf is not None:
                    pred = confidence.sparsify(pred, conf, density, float("inf"))
                rep.add(s, *_score(pred, gt, mask, ndisp, ev.dev))
                if out is not None:
                    base = os.path.join(out, "trainingH", s)
                    os.makedirs(base, exist_ok=True)
                    dataio.write_pfm(np.flipud(pred.cpu().numpy()), os.path.join(base, "disp0%s.pfm" % ev.method_name))
                    with open(os.path.join(base, "time%s.txt" % ev.method_name), "w") as f:
                        f.write(evaluate.lua_num(runtime))
    finally:
        ev.close()
    return rep.done()
