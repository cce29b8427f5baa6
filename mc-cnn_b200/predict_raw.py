"""The stereo method over whole KITTI raw drives in one process (an addition beyond the reference; DESIGN §21).

    names = predict_raw("kitti", "fast", ["/data/raw/2011_09_26/2011_09_26_drive_0002_sync"], net_fname=N, out="O",
                        disp=True, depth=True, ply=True)
    # O/2011_09_26_drive_0002_sync/disp/%010d.png, depth/%010d.png, points/%010d.ply; prints "<date>/<drive> <frame>" per frame

A drive is ``<date>/<date>_drive_<nnnn>_sync`` as KITTI's raw archives unpack: the grey rectified pair
``image_00/data/%010d.png`` / ``image_01/data/%010d.png`` per frame, ``velodyne_points/data/%010d.bin`` scans, and the
calibration in the date directory (dataio.read_calib(date, 'kitti_raw')).  `dataset` 'kitti' or 'kitti2015' picks the
stereo method's presets.  Every frame runs through :class:`predict_kitti.PairRunner`, the loop predict_kitti uses: one
pipeline at the largest shape, the next pair's PNGs decoded while the GPU works.  Under torch.distributed (torchrun, one
process per GPU) the frames of all drives, in drive then frame order, go round-robin over the ranks; each rank writes its
own frames' files and rank 0 prints every frame's line in order.

A drive whose name ends in ``_extract`` (KITTI's unsynced+unrectified archives, the same image layout) is read as
unrectified (DESIGN §22): each frame is rectified on the GPU by dataio.read_rectification(date, 'kitti_raw') to S_rect_00
before the unchanged stereo method, its outputs lie on the rectified grid with the calibration that rectification defines,
and the pixels outside the left view's validity mask have no disparity, depth or vertex (0 in the disparity PNG).  Its
raw images must be of size S_00 / S_01.

Outputs under ``out/<drive>/``: ``disp/%010d.png`` (KITTI's PNG16, dataio.write_png16), ``depth/%010d.png``
(dataio.write_depth_png16 of depth.depth), ``points/%010d.ply`` (depth.point_cloud coloured by the left image) and
``conf/%010d.bin`` (the margin confidence, (1, 1, H, W) float32 in main.lua's .bin layout).  `density` p keeps, in the
disparity, depth and cloud, the ceil(p H W) pixels of largest margin confidence (confidence.sparsify).  A drive whose
output directory is not empty is refused before any GPU work.
"""
import os
from collections import namedtuple

from . import batch, confidence as confidence_, dataio, frontend, predict_kitti
from . import depth as depth_

DATASETS = ("kitti", "kitti2015")
Frame = namedtuple("Frame", "drive index")          # drive: the drive directory; index: the frame number


def drive_name(drive):
    return os.path.basename(os.path.normpath(drive))


def date_dir(drive):
    return os.path.dirname(os.path.normpath(drive))


def frame_name(fr):
    """``<date>/<drive> <frame>``, the line of a split file"""
    return "%s/%s %010d" % (os.path.basename(date_dir(fr.drive)), drive_name(fr.drive), fr.index)


def drive_frames(drives, every=1, velodyne=False):
    """the :data:`Frame` list of `drives`, in drive order then ascending frame order, every `every`-th frame of each drive
    (dataio.raw_frames: a frame missing on one side is refused)"""
    if int(every) < 1:
        raise ValueError("every must be at least 1, got %r" % (every,))
    names = [drive_name(d) for d in drives]
    if len(set(names)) != len(names):
        raise ValueError("a drive is named twice: %s" % ", ".join(names))
    return [Frame(d, i) for d in drives for i in dataio.raw_frames(d, velodyne)[::int(every)]]


def read_list(path, data_root):
    """the :data:`Frame` list of a split file: lines ``<date>/<drive> <frame>`` under `data_root`, in file order; refuses a
    malformed line and a frame whose images or scan are missing"""
    out = []
    with open(path) as f:
        for k, line in enumerate(f, 1):
            if not line.strip():
                continue
            parts = line.split()
            if len(parts) != 2 or not parts[1].isdigit() or parts[0].count("/") != 1:
                raise ValueError("%s:%d: '<date>/<drive> <frame>' expected, got %r" % (path, k, line.rstrip("\n")))
            fr = Frame(os.path.join(data_root, parts[0]), int(parts[1]))
            check_synced([fr.drive])
            for what in (dataio.RAW_LEFT, dataio.RAW_RIGHT, dataio.RAW_SCAN):
                p = dataio.raw_file(fr.drive, what, fr.index)
                if not os.path.isfile(p):
                    raise FileNotFoundError("%s:%d: missing %s" % (path, k, p))
            out.append(fr)
    if not out:
        raise ValueError("%s: no frames" % path)
    return out


def pair_files(frames):
    """[(left, right, None)] of the frames, as predict_kitti.Prefetch decodes them"""
    return [(dataio.raw_file(fr.drive, dataio.RAW_LEFT, fr.index), dataio.raw_file(fr.drive, dataio.RAW_RIGHT, fr.index), None)
            for fr in frames]


def is_extract(drive):
    """whether `drive` is an unrectified KITTI raw drive (its name ends in ``_extract``)"""
    return drive_name(drive).endswith(dataio.RAW_EXTRACT)


def check_synced(drives):
    """refuses unrectified (``_extract``) drives where a drive is scored against its Velodyne scans"""
    for d in drives:
        if is_extract(d):
            raise ValueError("%s is an unrectified (_extract) drive: its scans are text files, not synchronised with the "
                             "cameras, so it cannot be scored against them; use the drive's _sync version" % d)


def read_rects(frames, shapes):
    """[dataio.StereoRect of its date, or None] per frame: the rectification of every frame of an ``_extract`` drive, each
    date's refused when it is missing or malformed or its raw size is not the frame's"""
    rects, out = {}, []
    for fr, (H, W) in zip(frames, shapes):
        if not is_extract(fr.drive):
            out.append(None)
            continue
        d = date_dir(fr.drive)
        if d not in rects:
            rects[d] = dataio.read_rectification(d, "kitti_raw")
        rects[d].check_size(H, W, os.path.join(d, dataio.RAW_CAM))
        out.append(rects[d])
    return out


def read_calibs(frames, shapes):
    """{date directory: RawCalib} of the frames' dates, each refused when it is missing, malformed or not of the size of one
    of its frames"""
    cals = {}
    for fr, (H, W) in zip(frames, shapes):
        d = date_dir(fr.drive)
        if d not in cals:
            cals[d] = dataio.read_calib(d, "kitti_raw")
        dataio.check_calib_size(cals[d], H, W, os.path.join(d, dataio.RAW_CAM))
    return cals


def out_file(out, fr, kind):
    """the output file of frame `fr`: kind 'disp', 'depth', 'points' or 'conf'"""
    ext = {"disp": ".png", "depth": ".png", "points": ".ply", "conf": ".bin"}[kind]
    return os.path.join(out, drive_name(fr.drive), kind, "%010d%s" % (fr.index, ext))


def check_out(out, drives):
    """refuses a drive whose output directory holds anything"""
    for d in drives:
        o = os.path.join(out, drive_name(d))
        if os.path.isdir(o) and os.listdir(o):
            raise ValueError("output directory %s is not empty" % o)


def _world():
    import torch.distributed as dist

    distributed = dist.is_initialized() and dist.get_world_size() > 1
    return (dist.get_rank(), dist.get_world_size()) if distributed else (0, 1)


def predict_raw(dataset, arch, drives, net_fname=None, out="out", disp=False, depth=False, ply=False, confidence=False,
                density=None, every=1, disp_max=predict_kitti.DISP_MAX, device=0, prefetch=True, verbose=True,
                **overrides):
    """The net over every `every`-th frame of each drive directory in `drives` on CUDA device `device`, writing what the
    flags ask for under `out` (module docstring).  Returns, on rank 0, the frame names in order (and prints them); None on
    other ranks."""
    import torch
    import torch.distributed as dist

    if dataset not in DATASETS:
        raise ValueError("dataset must be 'kitti' or 'kitti2015', got %r" % (dataset,))
    if int(disp_max) < 1:
        raise ValueError("disp_max must be at least 1, got %r" % (disp_max,))
    if not (disp or depth or ply or confidence):
        raise ValueError("nothing to write: ask for disp, depth, ply or confidence")
    if density is not None:
        if not confidence:
            raise ValueError("density ranks pixels by their confidence: it needs confidence")
        confidence_.check_density(density)
    if not drives:
        raise ValueError("no drive given")
    frames = drive_frames(drives, every)
    files = pair_files(frames)
    shapes = predict_kitti.scan(files)
    rects = read_rects(frames, shapes)
    synced = [k for k, r in enumerate(rects) if r is None]
    cals = read_calibs([frames[k] for k in synced], [shapes[k] for k in synced])
    shapes = [s if r is None else r.left.rect_size[::-1] for s, r in zip(shapes, rects)]
    check_out(out, drives)
    rank, world = _world()
    if world > 1:
        dist.barrier()                          # every rank has looked at `out` before any rank writes to it
    run = predict_kitti.PairRunner(files, shapes, dataset, arch, net_fname, disp_max, device, rank, world, prefetch,
                                   rects=rects if any(rects) else None, **overrides)

    def path(fr, kind):
        p = out_file(out, fr, kind)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        return p

    def compute(i):
        fr = frames[i]
        left, _, _, pred, conf = run.predict(i, conf=confidence)
        with torch.cuda.device(run.dev):
            if confidence:
                frontend.write_bin(path(fr, "conf"), conf.reshape(1, 1, *conf.shape).cpu().numpy())
            if density is not None:
                pred = confidence_.sparsify(pred, conf, density, 0.0)
            cal = cals[date_dir(fr.drive)] if rects[i] is None else rects[i].calib
            if depth:
                dataio.write_depth_png16(depth_.depth(pred, cal).cpu().numpy(), path(fr, "depth"))
            if ply:
                depth_.write_ply(path(fr, "points"), depth_.point_cloud(pred, cal, left))
            if disp:
                if rects[i] is not None:                        # no disparity outside the mask: 0 in KITTI's PNG16
                    pred = pred.nan_to_num(nan=0.0, posinf=float("inf"), neginf=float("-inf"))
                dataio.write_png16(pred.cpu().numpy(), path(fr, "disp"))
        return torch.tensor([i])

    try:
        run.prepare()
        res = batch.run_sharded(len(frames), compute, rank, world)
    finally:
        run.close()
    if rank != 0:
        return None
    names = []
    for i, r in enumerate(res):
        assert int(r.reshape(-1)[0]) == i, "frame %d came back as %s" % (i, r)
        names.append(frame_name(frames[i]))
        if verbose:
            print(names[-1], flush=True)
    return names
