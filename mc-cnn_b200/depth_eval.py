"""Depth metrics of the stereo method on the KITTI 2012 / 2015 and MiddEval3 training pairs, on the GPU (an addition beyond
the reference; DESIGN §20).

    res = evaluate_training("kitti", "net/net_kitti_fast_-a_train_all.t7", data_root="/data")
    # prints one tab-separated line per pair (index or scene, then the metrics), then the line of means; res.names, res.rows
    res = score_dir("kitti", "out", data_root="/data", source="depth")    # out/depth_0/%06d_10.png
    res = score_dir("mb", "out", data_root="/data")                         # out/trainingH/<scene>/disp0*.pfm

The metrics are :func:`depth.metrics`'s: abs_rel, sq_rel, rmse, rmse_log (metres), a1, a2, a3, n and coverage.  KITTI scores
each map against disp_noc and disp_occ (the ``noc_`` and ``occ_`` columns) with min_depth 1e-3 m and max_depth 80 m, under
the calibration beside the images (predict_kitti.calib_file); MiddEval3 scores the half-size ``trainingH`` maps against
``trainingH/<scene>/disp0GT.pfm`` (the ``all_`` columns; +inf = unknown) with min_depth 1e-3 m and no cap, under the
scene's calib.txt.  The line of means is the plain mean of each column over the pairs, in pair order.

``score_dir`` reads what the other tools write: KITTI disparity maps in submission layout (predict_kitti submit,
kitti_eval -out) or depth maps (predict_kitti -depth; source 'depth'), MiddEval3 disparity PFMs (mb_eval -out).  A PNG map
is quantised to 1/256 px or 1/256 m, so its numbers differ from `evaluate_training`'s by that rounding.

Under torch.distributed the pairs are shared round-robin (batch.run_sharded) and rank 0 prints what one process prints.
"""
import os
from collections import namedtuple

import numpy as np

from . import batch, dataio, depth, evaluate, frontend, kitti_eval, mb_eval, predict_kitti, preprocess

DATASETS = ("kitti", "kitti2015", "mb")
Scores = namedtuple("Scores", "names rows mean")    # pair names, per-pair value lists (columns()), their means


def regions(dataset):
    return ("all",) if dataset == "mb" else ("noc", "occ")


def columns(dataset):
    """the names of a pair line's values, in order"""
    return ["%s_%s" % (r, m) for r in regions(dataset) for m in depth.METRICS]


def max_depth_of(dataset):
    return None if dataset == "mb" else depth.KITTI_MAX_DEPTH


def line(name, values):
    return "\t".join([str(name)] + [evaluate.lua_num(v) for v in values])


def _check_dataset(dataset):
    if dataset not in DATASETS:
        raise ValueError("dataset must be one of %s, got %r" % (", ".join(DATASETS), dataset))


def _read_gt(path):
    """a ground-truth disparity map as float32 (H, W): PNG16 (0 = none) or a top-down PFM (+inf = none)"""
    return mb_eval._read_topdown(path) if path.endswith(".pfm") else dataio.read_png16(path)


def training_pairs(data_root, dataset):
    """[(name, left, right, calib, [ground-truth file per region])] of the training pairs, in order; refuses missing files,
    malformed calibrations and sizes that disagree, before any GPU work"""
    _check_dataset(dataset)
    if dataset != "mb":
        files = kitti_eval.training_files(data_root, dataset)
        shapes = predict_kitti.scan([f[:3] for f in files])
        kitti_eval.check_maps([(None,) + f[2:] for f in files], shapes)
        calibs = predict_kitti.read_calibs([f[:3] for f in files], shapes, dataset)
        return [(i, f[0], f[1], c, [f[2], f[3]]) for i, (f, c) in enumerate(zip(files, calibs))]
    out = []
    for s in mb_eval.training_scenes(data_root):
        d = mb_eval.scene_dir(data_root, s)
        views = [os.path.join(d, "im0.png"), os.path.join(d, "im1.png")]
        h, w = preprocess._same_size(s, [(p, preprocess._image_size(p)) for p in views])
        cal_path = os.path.join(d, "calib.txt")
        cal = dataio.read_calib(cal_path, "mb")
        dataio.check_calib_size(cal, h, w, cal_path)
        gt = mb_eval.gt_files(data_root, s, "H")[0]
        if preprocess._pfm_size(gt) != (h, w):
            raise ValueError("%s is %dx%d, the images %dx%d" % (gt, *preprocess._pfm_size(gt), h, w))
        out.append((s, views[0], views[1], cal, [gt]))
    return out


def _pack(rows):
    """the float64 values of a pair as float32 words (what batch.run_sharded carries exactly)"""
    import torch

    return torch.from_numpy(np.ascontiguousarray(np.asarray(rows, dtype="<f8")).view("<u2").astype(np.float32))


def _unpack(t):
    return [float(v) for v in t.reshape(-1).cpu().numpy().astype("<u2").view("<f8")]


def _score(pred, gts, cal, dataset, is_depth=False):
    """the pair's values, columns() order, of the device map `pred` against the ground-truth files `gts`"""
    import torch

    out = []
    for g in gts:
        gt = torch.from_numpy(_read_gt(g)).to(pred.device)
        out += list(depth.metrics(pred, gt, cal, depth.MIN_DEPTH, max_depth_of(dataset), is_depth=is_depth))
    return out


def report(dataset, names, compute, rank=None, world=None, verbose=True, ncol=None):
    """batch.run_sharded over the pairs; rank 0 prints one line per pair and the line of means and returns the Scores"""
    import torch.distributed as dist

    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    res = batch.run_sharded(len(names), lambda i: _pack(compute(i)), rank, world)
    if rank != 0:
        return None
    rows = []
    for name, t in zip(names, res):
        rows.append(_unpack(t))
        if verbose:
            print(line(name, rows[-1]), flush=True)
    ncol = len(columns(dataset)) if ncol is None else ncol
    mean = [sum(r[k] for r in rows) / len(rows) if rows else float("nan") for k in range(ncol)]
    if verbose:
        print(line("mean", mean), flush=True)
    return Scores(list(names), rows, mean)


def _world():
    import torch.distributed as dist

    distributed = dist.is_initialized() and dist.get_world_size() > 1
    return (dist.get_rank(), dist.get_world_size()) if distributed else (0, 1)


def evaluate_training(dataset, net_fname=None, arch="fast", data_root=".", disp_max=predict_kitti.DISP_MAX, device=0,
                      verbose=True, **overrides):
    """The net over every training pair of `dataset` (KITTI: predict_kitti test's loop at `disp_max`; MiddEval3: the
    trainingH grey views at each scene's ndisp, as mb_eval), each map scored by :func:`depth.metrics` on CUDA device
    `device`.  Prints one line per pair and the line of means; returns the Scores on rank 0, None on other ranks."""
    import torch

    pairs = training_pairs(data_root, dataset)
    if int(disp_max) < 1:
        raise ValueError("disp_max must be at least 1, got %r" % (disp_max,))
    rank, world = _world()
    ev = evaluate.Evaluator(dataset, arch, net_fname=net_fname, device=device, **overrides)
    ndisp = {}
    if dataset == "mb":
        for name, left, _, _, _ in pairs:
            ndisp[name] = preprocess._ndisp(os.path.join(os.path.dirname(left), "calib.txt"))

    def compute(i):
        name, left, right, cal, gts = pairs[i]
        with torch.cuda.device(ev.dev):
            if dataset == "mb":
                x = preprocess._mb_views(dict(groups=[([left, right], (2,))], half=False), "gray", ev.dev)[0]
                pred = ev.stereo_predict(torch.from_numpy(np.ascontiguousarray(x)).to(ev.dev), ndisp[name])
            else:
                x_batch = frontend.make_batch_cuda(frontend.load_bytes(left), frontend.load_bytes(right), ev.dev)
                pred = ev.stereo_predict(x_batch, int(disp_max))
            return _score(pred, gts, cal, dataset)

    try:
        sizes = [tuple(preprocess._image_size(p[1])) for p in pairs]
        ev.prepare([s + (ndisp[p[0]] if dataset == "mb" else int(disp_max),) for s, p in zip(sizes, pairs)])
        return report(dataset, [p[0] for p in pairs], compute, rank, world, verbose)
    finally:
        ev.close()


def map_file(out, dataset, i, name, source):
    """the written map of pair i (scene `name`) under `out`"""
    if dataset == "mb":
        if source != "disp":
            raise ValueError("MiddEval3 maps are scored from disparity PFMs only")
        return mb_eval.find_map(out, name)
    if source == "depth":
        return predict_kitti.depth_files(out, i)[0]
    return kitti_eval.submission_file(out, dataset, i)


def score_dir(dataset, pred_dir, data_root=".", source="disp", device=0, verbose=True):
    """Scores the maps written under `pred_dir` (module docstring; `source` 'disp' or 'depth') against the training ground
    truth of `dataset` under `data_root`, on CUDA device `device`.  Every training pair needs its map.  Returns the Scores
    on rank 0, None on other ranks."""
    import torch

    if source not in ("disp", "depth"):
        raise ValueError("source must be 'disp' or 'depth', got %r" % (source,))
    pairs = training_pairs(data_root, dataset)
    files = []
    for i, (name, left, _, _, _) in enumerate(pairs):
        f = map_file(pred_dir, dataset, i, name, source)
        if not os.path.isfile(f):
            raise FileNotFoundError("missing map %s" % f)
        files.append(f)
    rank, world = _world()

    def compute(i):
        _, _, _, cal, gts = pairs[i]
        f = files[i]
        if f.endswith(".pfm"):
            m = mb_eval._read_topdown(f)
        else:
            m = dataio.read_depth_png16(f) if source == "depth" else dataio.read_png16(f)
        with torch.cuda.device(device):
            pred = torch.from_numpy(m).to(torch.device("cuda", device))
            return _score(pred, gts, cal, dataset, is_depth=source == "depth")

    return report(dataset, [p[0] for p in pairs], compute, rank, world, verbose)


# ---- KITTI raw drives against the projected Velodyne scans (DESIGN §21) ------------------------------------------------------

RAW_COLUMNS = ["lidar_%s" % m for m in depth.METRICS]
# the published crop rectangles, fractions of (H, H, W, W): rows [top, bottom), columns [left, right) (Garg et al. 2016;
# Eigen et al. 2014)
CROPS = {"garg": (0.40810811, 0.99189189, 0.03594771, 0.96405229), "eigen": (0.3324324, 0.91351351, 0.0359477, 0.96405229)}


def crop_box(crop, H, W):
    """(top, bottom, left, right) of crop 'garg' / 'eigen' at H x W: each fraction times the size in float64, truncated"""
    if crop not in CROPS:
        raise ValueError("crop must be garg, eigen or none, got %r" % (crop,))
    a, b, c, d = CROPS[crop]
    return int(a * H), int(b * H), int(c * W), int(d * W)


def lidar_gt(scan, cal, H, W, device, min_depth=depth.MIN_DEPTH, crop="none"):
    """the ground-truth disparity of a frame: its scan (host (N, 4) float32) projected into an H x W depth map
    (depth.velo_depth), 0 outside the crop rectangle, turned into the disparity fB / Z (NaN where no point) that
    depth.metrics takes"""
    import torch

    Z = depth.velo_depth(torch.from_numpy(scan).to(device), cal, H, W, min_depth)
    if crop != "none":
        t, b, l, r = crop_box(crop, H, W)
        for rows, cols in ((slice(0, t), slice(None)), (slice(b, None), slice(None)), (slice(None), slice(0, l)),
                           (slice(None), slice(r, None))):
            Z[rows, cols] = 0.0
    return depth.disparity_of_depth(Z, cal)


def _check_raw(min_depth, max_depth, crop):
    if not (0 < min_depth <= max_depth):
        raise ValueError("need 0 < min_depth <= max_depth, got %r, %r" % (min_depth, max_depth))
    if crop != "none":
        crop_box(crop, 1, 1)


def _raw_inputs(frames):
    """(pair files, shapes, calibrations) of the frames, refused before any GPU work as predict_raw refuses them"""
    from . import predict_raw

    predict_raw.check_synced(sorted({fr.drive for fr in frames}))
    files = predict_raw.pair_files(frames)
    shapes = predict_kitti.scan(files)
    return files, shapes, predict_raw.read_calibs(frames, shapes)


def evaluate_raw(dataset, arch, frames, net_fname=None, disp_max=predict_kitti.DISP_MAX, min_depth=depth.MIN_DEPTH,
                 max_depth=depth.KITTI_MAX_DEPTH, crop="none", device=0, prefetch=True, verbose=True, **overrides):
    """The net over each raw frame of `frames` (predict_raw.Frame list; predict_raw.drive_frames(..., velodyne=True) or
    read_list), each map scored against the frame's projected scan (:func:`lidar_gt`) by depth.metrics with `min_depth` and
    `max_depth`.  Prints one line per frame (predict_raw.frame_name, then the RAW_COLUMNS values) and the line of means;
    returns the Scores on rank 0, None on other ranks."""
    from . import predict_raw

    _check_raw(min_depth, max_depth, crop)
    files, shapes, cals = _raw_inputs(frames)
    rank, world = _world()
    run = predict_kitti.PairRunner(files, shapes, dataset, arch, net_fname, disp_max, device, rank, world, prefetch,
                                   **overrides)

    def compute(i):
        import torch

        fr = frames[i]
        cal = cals[predict_raw.date_dir(fr.drive)]
        _, _, _, pred, _ = run.predict(i)
        with torch.cuda.device(run.dev):
            gt = lidar_gt(dataio.read_velodyne(dataio.raw_file(fr.drive, dataio.RAW_SCAN, fr.index)), cal, *shapes[i],
                          run.dev, min_depth, crop)
            return list(depth.metrics(pred, gt, cal, min_depth, max_depth))

    try:
        run.prepare()
        return report("raw", [predict_raw.frame_name(f) for f in frames], compute, rank, world, verbose, len(RAW_COLUMNS))
    finally:
        run.close()


def score_raw(frames, pred_dir, source="disp", min_depth=depth.MIN_DEPTH, max_depth=depth.KITTI_MAX_DEPTH, crop="none",
              device=0, verbose=True):
    """Scores the maps predict_raw wrote under `pred_dir` (``<drive>/disp/%010d.png``, or with `source` 'depth'
    ``<drive>/depth/%010d.png``) for `frames` against their projected scans, as :func:`evaluate_raw` does.  Every frame
    needs its map."""
    import torch

    from . import predict_raw

    if source not in ("disp", "depth"):
        raise ValueError("source must be 'disp' or 'depth', got %r" % (source,))
    _check_raw(min_depth, max_depth, crop)
    maps = [predict_raw.out_file(pred_dir, fr, source) for fr in frames]
    for f in maps:
        if not os.path.isfile(f):
            raise FileNotFoundError("missing map %s" % f)
    _, shapes, cals = _raw_inputs(frames)
    rank, world = _world()
    dev = torch.device("cuda", device)

    def compute(i):
        fr = frames[i]
        m = dataio.read_depth_png16(maps[i]) if source == "depth" else dataio.read_png16(maps[i])
        if m.shape != tuple(shapes[i]):
            raise ValueError("%s is %dx%d, the images %dx%d" % (maps[i], *m.shape, *shapes[i]))
        cal = cals[predict_raw.date_dir(fr.drive)]
        with torch.cuda.device(dev):
            gt = lidar_gt(dataio.read_velodyne(dataio.raw_file(fr.drive, dataio.RAW_SCAN, fr.index)), cal, *shapes[i], dev,
                          min_depth, crop)
            return list(depth.metrics(torch.from_numpy(m).to(dev), gt, cal, min_depth, max_depth, is_depth=source == "depth"))

    return report("raw", [predict_raw.frame_name(f) for f in frames], compute, rank, world, verbose, len(RAW_COLUMNS))
