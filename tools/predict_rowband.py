"""main.lua's ``-a predict`` for one pair, its rows split over the GPUs of a torchrun job (mccnn_b200.rowband.predict_pair).

    torchrun --nproc-per-node N tools/predict_rowband.py kitti slow -left L.png -right R.png -disp_max 228 -net_fname N
    python tools/predict_rowband.py mb census -left L.png -right R.png -disp_max 140 -out out     # one process: one GPU

Option names are tools/run_main.py's; -L1 ... -blur_t override the preset.  Writes right.bin, left.bin ((1, D, H, W)) and
disp.bin ((1, 1, H, W)) into -out (default: the working directory, as main.lua's predict does): the bytes
``run_main.py -a predict`` writes for the same options.  What run_main.py -a predict refuses is refused here too, and so are
-sm_terminate / -sm_skip (the row-band chain runs the full stereo method), all before any GPU work.  Under torchrun rank r
uses GPU LOCAL_RANK; one process uses -gpu.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(1, os.path.dirname(os.path.abspath(__file__)))
import run_main  # noqa: E402


def parse_args(argv=None):
    """-> (namespace, preset overrides); raises SystemExit on what the row-band predict does not run"""
    argv = list(sys.argv[1:] if argv is None else argv)
    args, overrides = run_main.parse_args(["-a", "predict", "-out", "."] + argv)
    if args.a != "predict":
        raise SystemExit("predict_rowband.py: only -a predict (got -a %s)" % args.a)
    if not (args.left and args.right and args.disp_max):
        raise SystemExit("predict_rowband.py: -left, -right and -disp_max are needed")
    for k in ("sm_terminate", "sm_skip"):
        if k in overrides:
            raise SystemExit("predict_rowband.py: -%s is not supported: the row bands run the full chain (use run_main.py)" % k)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import frontend

    try:
        method = frontend.StereoMethod(args.dataset, args.arch, args.net_fname or None, **overrides)
    except ValueError as e:
        raise SystemExit("predict_rowband.py: %s" % e)
    if method.needs_net:
        raise SystemExit("predict_rowband.py: arch '%s' needs -net_fname" % args.arch)
    return args, overrides


def main(argv=None):
    args, overrides = parse_args(argv)
    import torch
    import torch.distributed as dist

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import rowband

    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ["LOCAL_RANK"]) if "LOCAL_RANK" in os.environ else args.device
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    try:
        rowband.predict_pair(args.left, args.right, dataset=args.dataset, arch=args.arch, disp_max=args.disp_max,
                             net_fname=args.net_fname or None, comm=rowband.Comm(), device=dev, out_dir=args.out, **overrides)
    finally:
        if world > 1:
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
