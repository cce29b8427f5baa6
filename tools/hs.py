"""hs.py's parameter search for action test_te on the GPU: one process scores every candidate (mc-cnn_b200/search.py).

    python tools/hs.py random kitti slow test_te net/net_kitti_slow_-a_train_tr.t7 -log hs.log -n 100
    python tools/hs.py hillclimb_fast kitti fast test_te net/net_kitti_fast_-a_train_tr.t7 -log hs.log
    python tools/hs.py random mb census test_te - -log hs.log -rect imperfect -color gray

Positional arguments are hs.py's: METHOD (random, hillclimb_slow, hillclimb_fast, hillclimb_dim), DATASET, ARCH, ACTION and
NET_FNAME ('-' for ad / census, which need no net).  Every evaluation appends hs.py's line (``score dataset arch test_te
-name value ... -use_cache | -net_fname N``) to -log with one write and prints it; the hillclimb methods re-read the log before
every proposal, so several processes (one per GPU, -gpu is 1-based) can share one log.  -n stops after that many
evaluations (default 0: run until interrupted, as hs.py does); points hs.py's valid() rejects are not evaluated and not
counted.

Deliberate differences from hs.py: one -log file instead of the hs.sh.* files of the working directory; -n; a candidate
whose prediction contains NaN is reported on stderr, not logged, and the search goes on (main.lua would assert, ending
hs.py); the 'slow' volumes are cached in pinned host memory for the life of the process instead of cache/*.t7 files; only
test_te is supported.
"""
import argparse
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="hs.py", description=__doc__.splitlines()[0])
    ap.add_argument("method", choices=("random", "hillclimb_slow", "hillclimb_fast", "hillclimb_dim"))
    ap.add_argument("dataset", choices=("mb", "kitti", "kitti2015"))
    ap.add_argument("arch", choices=("fast", "slow", "ad", "census"))
    ap.add_argument("action", choices=("test_te", "train_tr", "da"))
    ap.add_argument("net_fname", help="the trained net (.t7); '-' for ad / census")
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    ap.add_argument("-rect", default="imperfect")
    ap.add_argument("-color", default="gray")
    ap.add_argument("-log", default="hs.log", help="results file, appended to (default hs.log)")
    ap.add_argument("-n", type=int, default=0, help="number of evaluations (0: until interrupted)")
    ap.add_argument("-seed", type=int, default=None, help="seed of the proposals (default: unseeded)")
    return ap


def read_results(path, dataset, arch, params):
    from mccnn_b200 import search

    if not os.path.exists(path):
        return []
    with open(path) as f:
        return search.parse_log(f, dataset, arch, params)


def parse_args(argv=None):
    """-> namespace.  Refuses, before any GPU work, what the search cannot do."""
    from mccnn_b200 import evaluate, search

    args = parser().parse_args(argv)
    if args.action != "test_te":
        raise SystemExit("hs.py: action %s (training) is not supported; only test_te is" % args.action)
    if args.gpu < 1:
        raise SystemExit("hs.py: -gpu is 1-based")
    if args.n < 0:
        raise SystemExit("hs.py: -n must be >= 0")
    try:
        evaluate.check_options(args.dataset, color=args.color)
    except ValueError as e:
        raise SystemExit("hs.py: %s" % e)
    if args.arch in ("fast", "slow"):
        if args.net_fname in ("", "-"):
            raise SystemExit("hs.py: arch %s needs a net file" % args.arch)
        if not os.path.exists(args.net_fname):
            raise SystemExit("hs.py: net file %s does not exist" % args.net_fname)
    args.params = search.grid(args.dataset, args.arch)
    if args.method.startswith("hillclimb"):
        try:
            results = read_results(args.log, args.dataset, args.arch, args.params)
        except search.SearchError as e:
            raise SystemExit("hs.py: %s: %s" % (args.log, e))
        if not results:
            raise SystemExit("hs.py: %s has no line for %s %s test_te to climb from; start with the random method"
                             % (args.log, args.dataset, args.arch))
    args.device = args.gpu - 1
    return args


def append_line(path, line):
    """one write per line (O_APPEND), so that processes sharing the log do not interleave inside a line"""
    fd = os.open(path, os.O_WRONLY | os.O_APPEND | os.O_CREAT, 0o644)
    try:
        os.write(fd, (line + "\n").encode())
    finally:
        os.close(fd)


def main(argv=None, searcher=None):
    """`searcher`: an already built search.Searcher for these arguments (the tests pass one in)"""
    args = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import search

    rng = random.Random(args.seed)
    own = searcher is None
    if own:
        searcher = search.Searcher(args.dataset, args.arch, net_fname=None if args.net_fname == "-" else args.net_fname,
                                   data_root=args.data_root, rect=args.rect, color=args.color, device=args.device)
    done = 0
    try:
        while args.n == 0 or done < args.n:
            results = None
            if args.method.startswith("hillclimb"):
                try:
                    results = read_results(args.log, args.dataset, args.arch, args.params)
                except search.SearchError as e:
                    raise SystemExit("hs.py: %s: %s" % (args.log, e))
            x = search.propose(args.method, args.params, rng, results)
            ps = search.point(args.params, x)
            if not search.valid(dict(ps)):
                continue
            done += 1
            try:
                score, _ = searcher.score(dict(ps))
            except search.NaNPrediction as e:
                sys.stderr.write("hs.py: skipped %s: %s\n" % (search.format_params(ps), e))
                sys.stderr.flush()
                continue
            line = search.format_line(score, args.dataset, args.arch, ps, args.net_fname)
            append_line(args.log, line)
            print(line, flush=True)
    except KeyboardInterrupt:
        pass
    finally:
        if own:
            searcher.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
