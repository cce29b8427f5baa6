"""predict_kitti.lua: a trained net over every full-size raw KITTI pair, in one process per GPU.

    python tools/predict_kitti.py test   kitti     -net_fname net/net_kitti_fast_-a_train_all.t7 -data_root /data
    python tools/predict_kitti.py submit kitti2015 -net_fname N -data_root /data -out out [-arch fast|slow|census|ad] \\
        [-disp_max 228] [-gpu 1]
    torchrun --nproc-per-node 8 tools/predict_kitti.py test kitti -net_fname N -data_root /data

`test` prints ``i<TAB>err`` for every training pair (0-based), then the mean 3-pixel error; `submit` writes
``out/%06d_10.png`` (kitti) or ``out/disp_0/%06d_10.png`` (kitti2015) for every testing pair and prints its index.  The raw
archives are read from ``<data_root>/data.kitti/unzip`` or ``data.kitti2015/unzip``, as preprocess_kitti.py reads them.
-gpu is 1-based as in main.lua.  Under torchrun each process takes the GPU of its LOCAL_RANK and the pairs are shared
round-robin; the output is the one a single process prints.  `submit -density p` (an addition beyond the reference) keeps
the ceil(p H W) pixels of largest margin confidence in each map and writes 0, the invalid value, elsewhere.  `-depth`
(also an addition) writes each pair's metric depth as ``out/depth_0/%06d_10.png`` (KITTI's depth format), and with `-ply`
its coloured point cloud as ``out/points_0/%06d_10.ply``, from the calibration files beside the images.  See
mc-cnn_b200/predict_kitti.py.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="predict_kitti.py", description=__doc__.splitlines()[0])
    ap.add_argument("action", choices=("test", "submit"))
    ap.add_argument("dataset", choices=("kitti", "kitti2015"))
    ap.add_argument("-net_fname", default="")
    ap.add_argument("-arch", choices=("fast", "slow", "census", "ad"), default="fast")
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-out", default="out")
    ap.add_argument("-disp_max", type=int, default=228)
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    ap.add_argument("-density", type=float, default=None, help="submit: keep this share of each map's pixels, in (0, 1]")
    ap.add_argument("-depth", action="store_true", help="also write out/depth_0/%%06d_10.png, the metric depth")
    ap.add_argument("-ply", action="store_true", help="with -depth: also write out/points_0/%%06d_10.ply")
    return ap


def parse_args(argv=None):
    """Refuses what cannot run before any file or GPU is touched."""
    args = parser().parse_args(argv)
    if args.arch in ("fast", "slow") and not args.net_fname:
        raise SystemExit("predict_kitti.py: arch '%s' needs -net_fname" % args.arch)
    if args.disp_max < 1:
        raise SystemExit("predict_kitti.py: -disp_max must be at least 1")
    if args.gpu < 1:
        raise SystemExit("predict_kitti.py: -gpu is 1-based")
    if args.density is not None:
        if args.action != "submit":
            raise SystemExit("predict_kitti.py: -density applies to the maps submit writes; test writes none")
        if not 0 < args.density <= 1:
            raise SystemExit("predict_kitti.py: -density must be in (0, 1]")
    if args.ply and not args.depth:
        raise SystemExit("predict_kitti.py: -ply writes the point clouds of the depth maps; it needs -depth")
    return args


def main(argv=None):
    args = parse_args(argv)
    import torch.distributed as dist

    import mccnn_b200  # noqa: F401
    from mccnn_b200.predict_kitti import predict_kitti

    world = int(os.environ.get("WORLD_SIZE", "1"))
    device = args.gpu - 1
    if world > 1:
        # only two counts (or one index) per pair cross between processes: gloo on the host is enough
        dist.init_process_group("gloo")
        device = int(os.environ.get("LOCAL_RANK", "0"))
    try:
        predict_kitti(args.action, args.dataset, net_fname=args.net_fname or None, arch=args.arch, data_root=args.data_root,
                      out=args.out, disp_max=args.disp_max, device=device, density=args.density, depth=args.depth,
                      ply=args.ply)
    finally:
        if world > 1:
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
