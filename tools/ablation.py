"""The stereo method's ablation on the test_te examples in one process: the validation error of the full chain, of the chain
with each step left out (main.lua's -sm_skip) and of the chain stopped after each step (-sm_terminate).

    python tools/ablation.py kitti fast net/net_kitti_fast_-a_train_tr.t7 -data_root /data
    python tools/ablation.py mb census - -rect imperfect

Positional arguments: DATASET (kitti, kitti2015, mb), ARCH (fast, slow, ad, census) and NET_FNAME ('-' for ad / census).
Prints one ``variant<TAB>score`` line per variant, in chain order: ``full``, ``-sm_skip <step>`` ..., ``-sm_terminate <step>``
....  A score is what ``run_main.py DATASET ARCH -a test_te`` with that option prints as its last line, as a float
(float('%.14g' % mean)).  Steps that do no work in the preset are left out, since their variants repeat another one's
result (run_main.py refuses them): the LR-check steps (skip occlusion, terminate occlusion and mismatch) on mb, and the
CBCA steps where the preset has no CBCA iterations (skip cbca and terminate cbca1 / cbca2 in the fast presets).

Every variant runs through one search.Searcher: the images stay on the device, one pipeline is re-targeted per variant and,
for arch slow, the scorer head's volumes are computed once for all variants.  A variant whose prediction contains NaN (where
main.lua:1224 asserts) is reported on stderr and printed with the score ``nan``; the ablation goes on.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parser():
    ap = argparse.ArgumentParser(prog="ablation.py", description=__doc__.splitlines()[0])
    ap.add_argument("dataset", choices=("kitti", "kitti2015", "mb"))
    ap.add_argument("arch", choices=("fast", "slow", "ad", "census"))
    ap.add_argument("net_fname", help="the trained net (.t7); '-' for ad / census")
    ap.add_argument("-data_root", default=".")
    ap.add_argument("-rect", default="imperfect")
    ap.add_argument("-gpu", type=int, default=1, help="1-based GPU number, as in main.lua")
    return ap


def parse_args(argv=None):
    """-> namespace.  Refuses, before any GPU work, what the ablation cannot run."""
    args = parser().parse_args(argv)
    if args.gpu < 1:
        raise SystemExit("ablation.py: -gpu is 1-based")
    if args.arch in ("fast", "slow"):
        if args.net_fname in ("", "-"):
            raise SystemExit("ablation.py: arch %s needs a net file" % args.arch)
        if not os.path.exists(args.net_fname):
            raise SystemExit("ablation.py: net file %s does not exist" % args.net_fname)
    args.device = args.gpu - 1
    return args


def main(argv=None, searcher=None):
    """`searcher`: an already built search.Searcher for these arguments (the tests pass one in).  Returns [(label, score)]."""
    args = parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import evaluate, search

    own = searcher is None
    if own:
        searcher = search.Searcher(args.dataset, args.arch, net_fname=None if args.net_fname == "-" else args.net_fname,
                                   data_root=args.data_root, rect=args.rect, device=args.device)
    out = []
    try:
        for label, overrides in search.ablation_variants(searcher.opt):
            try:
                score, _ = searcher.score(overrides)
            except search.NaNPrediction as e:
                sys.stderr.write("ablation.py: %s: %s\n" % (label, e))
                sys.stderr.flush()
                score = float("nan")
            out.append((label, score))
            print("%s\t%s" % (label, evaluate.lua_num(score)), flush=True)
    finally:
        if own:
            searcher.close()
    return out


if __name__ == "__main__":
    main()
    sys.exit(0)
