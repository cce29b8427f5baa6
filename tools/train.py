"""main.lua's training actions for the fast architecture on KITTI: ``-a train_tr`` and ``-a train_all``.

    python tools/train.py kitti fast -a train_tr -data_root /data             # 14 epochs, then test_te with the new net
    python tools/train.py kitti2015 fast -a train_all -data_root /data -out out   # 14 epochs on nnz_tr + nnz_te, then submit

Option names and defaults are main.lua's (-gpu is 1-based as there): the network and training options (-l1 -fm -ks -lr -bs
-mom -true1 -false1 -false2 -m -pow), the augmentation options (-hflip ... -d_contrast) and the stereo method's overrides of
run_main.py (-L1 ... -blur_t) for the evaluation that follows.  The net goes to <data_root>/net/net_<cmd_str>.t7, named from
main.lua's arguments.  Everything the trainer does not implement is refused before any GPU work; see mc-cnn_b200/train.py.
The slow architecture is trained by tools/train_slow.py, and both architectures on Middlebury by tools/train_mb.py; both
share this parser.

Checkpoints (none of these three is part of the net's name):

    -checkpoint_steps K   write the training state every K steps of an epoch (K a positive multiple of 256, the chunk
                          size) and at the end of every epoch, to <data_root>/net/net_<cmd_str>.state.npz
    -stop_after S         at the first chunk boundary after S seconds of training, write the state and exit with 75
    -resume               continue from this command line's checkpoint if there is one, otherwise start fresh

    while python tools/train.py kitti fast -a train_tr -data_root /data -resume -stop_after 3000; [ $? -eq 75 ]; do :; done

A resumed run prints the remaining epoch lines and writes the net an uninterrupted run would, bit for bit; the checkpoint is
deleted once the net file is written.  A checkpoint of other options or another training set is refused.

Several GPUs (both architectures, KITTI or Middlebury): one process per GPU under torchrun, each on the GPU of its
LOCAL_RANK (so -gpu is refused there), NCCL between them.  The epoch lines, the net file and the checkpoints are those of
one GPU, bit for bit, and a checkpoint written by one rank count resumes on another.  The rank count must be a power of
two and at most 2 bs; rank 0 prints, writes and runs test_te / submit.

    torchrun --nproc-per-node 8 tools/train.py kitti fast -a train_tr -data_root /data
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from run_main import PRESET_OPTIONS, _flag  # noqa: E402

TOOL_ONLY = ("-data_root", "-out", "-checkpoint_steps", "-stop_after")     # options with a value
TOOL_FLAGS = ("-resume",)


def _names(mb):
    """the training options a tool accepts: KITTI's, plus main.lua's mb-only -ds -d_exp -d_light for the Middlebury tool"""
    from mccnn_b200 import train

    return {**train.AUGMENT, **train.NET, **train.NET_SLOW, **(train.MB_DRAWS if mb else {})}


def parser(prog="train.py", description=__doc__.splitlines()[0], mb=False):
    ap = argparse.ArgumentParser(prog=prog, description=description)
    ap.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    ap.add_argument("arch", choices=("fast", "slow", "ad", "census"))
    ap.add_argument("-a", default="train_tr")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    ap.add_argument("-seed", type=int, default=42)
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-out", default="out")
    ap.add_argument("-subset", type=float, default=1)
    ap.add_argument("-debug", nargs="?", const=True, default=False, type=_flag)
    ap.add_argument("-checkpoint_steps", type=int, default=None)
    ap.add_argument("-stop_after", type=float, default=None)
    ap.add_argument("-resume", action="store_true")
    if mb:
        ap.add_argument("-rect", choices=("perfect", "imperfect"), default="imperfect")
        ap.add_argument("-color", default="gray")
    for name, v in _names(mb).items():
        ap.add_argument("-" + name, type=type(v), default=None)
    for name, typ in PRESET_OPTIONS.items():
        ap.add_argument("-" + name, type=typ, default=None)
    return ap


def main_args(argv):
    """main.lua's arguments after dataset and arch, without this tool's own options (for cmd_str)"""
    out, skip = [], False
    for a in argv[2:]:
        if skip:
            skip = False
        elif a in TOOL_ONLY:
            skip = True
        elif a not in TOOL_FLAGS and not a.startswith(TOOL_ONLY):
            out.append(a)
    return out


# the KITTI tools and the architecture each trains; the other one is named in the refusal.  train_mb.py trains both
# architectures on Middlebury (arch None below).
TOOLS = {"fast": "train.py", "slow": "train_slow.py"}
MB_TOOL = "train_mb.py"


def parse_args(argv=None, arch="fast"):
    """-> (namespace, training options, stereo overrides).  Refuses what the trainer does not implement, and every arch
    but `arch` (arch None: the Middlebury tool, fast or slow on dataset mb only)."""
    from mccnn_b200 import train

    mb = arch is None
    prog = MB_TOOL if mb else TOOLS[arch]
    argv = list(sys.argv[1:] if argv is None else argv)
    args = parser(prog, mb=mb).parse_args(argv)
    if mb:
        if args.dataset != "mb":
            raise SystemExit("%s: dataset %s: this tool trains on Middlebury (mb); use train.py or train_slow.py"
                             % (prog, args.dataset))
        if args.arch not in TOOLS:
            raise SystemExit("%s: arch %s: only the fast and slow architectures can be trained" % (prog, args.arch))
        if args.color != "gray":
            raise SystemExit("%s: -color %s is not supported: three-plane images need a 3-plane first layer in the "
                             "trainer, the feature tower and the evaluation; only -color gray is" % (prog, args.color))
    elif args.arch != arch:
        other = [TOOLS[a] for a in TOOLS if a == args.arch]
        raise SystemExit("%s: arch %s: only the %s architecture can be trained by this tool%s"
                         % (prog, args.arch, arch, "; use %s" % other[0] if other else ""))
    elif args.dataset == "mb":
        raise SystemExit("%s: dataset mb: Middlebury training is done by %s" % (prog, MB_TOOL))
    if args.a not in ("train_tr", "train_all"):
        raise SystemExit("%s: -a %s is not a training action (train_tr, train_all); see run_main.py" % (prog, args.a))
    if args.gpu < 1:
        raise SystemExit("%s: -gpu is 1-based" % prog)
    if args.subset < 1:
        raise SystemExit("%s: -subset %s is not supported (the whole training set is used)" % (prog, args.subset))
    if args.debug:
        raise SystemExit("%s: -debug (a net file per epoch) is not supported" % prog)
    try:
        train.check_checkpoint_options(args.checkpoint_steps, args.stop_after)
    except ValueError as e:
        raise SystemExit("%s: %s" % (prog, e))
    given = {k: getattr(args, k) for k in _names(mb) if getattr(args, k) is not None}
    try:
        o = train.options(args.dataset, args.arch, **given)
    except ValueError as e:
        raise SystemExit("%s: %s" % (prog, e))
    stereo = {k: getattr(args, k) for k in PRESET_OPTIONS if getattr(args, k) is not None}
    args.device = args.gpu - 1
    args.argv = argv
    return args, o, stereo


def main(argv=None, arch="fast"):
    args, o, stereo = parse_args(argv, arch)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import train

    prog = MB_TOOL if arch is None else TOOLS[arch]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    try:
        train.check_world(world, o)
    except ValueError as e:
        raise SystemExit("%s: torchrun with %s" % (prog, e))
    if world > 1 and any(a == "-gpu" or a.startswith("-gpu=") for a in args.argv):
        raise SystemExit("%s: -gpu under torchrun: each process trains on the GPU of its LOCAL_RANK, and the net records "
                         "rank 0's GPU 1; leave -gpu out" % prog)
    fname = train.net_path(args.data_root, args.dataset, main_args(args.argv), args.arch)
    if os.path.exists(fname):
        raise SystemExit("%s: %s already exists; remove it first" % (prog, fname))
    rect = {"rect": args.rect} if arch is None else {}
    if arch is None:                                                              # refuse a bad set before printing
        try:
            train.MbTrainSet(args.data_root, args.rect, args.a)
        except (OSError, ValueError) as e:
            raise SystemExit("%s: %s" % (prog, e))
    if rank == 0:
        print(" ".join(args.argv) + " ", flush=True)                              # main.lua:6-9
    ckpt = dict(checkpoint_steps=args.checkpoint_steps, stop_after=args.stop_after, resume=args.resume)
    device, comm = args.device, None
    if world > 1:
        import torch
        import torch.distributed as dist

        from mccnn_b200 import rowband

        device = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(device)
        dist.init_process_group("nccl", device_id=torch.device("cuda", device))
        comm = rowband.Comm()
    try:
        train.train(args.dataset, args.a, o, args=main_args(args.argv), data_root=args.data_root, seed=args.seed,
                    device=device, out=args.out, stereo=stereo, log=lambda s: print(s, flush=True), comm=comm, **rect,
                    **ckpt)
    except (MemoryError, train.CheckpointError) as e:                            # the mb planes do not fit, a bad checkpoint
        raise SystemExit("%s: %s" % (prog, e))
    except train.Stopped as e:
        if rank == 0:
            print("%s: %s" % (prog, e), file=sys.stderr, flush=True)
        return train.EX_TEMPFAIL
    finally:
        if comm is not None:
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
