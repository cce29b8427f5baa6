"""Wall time of the stereo-method ablation (tools/ablation.py) against the same variants run one Evaluator at a time, on a
synthetic KITTI-size validation set.

    python tools/time_ablation.py [-n_te 8] [-archs fast,slow] [-out time_ablation.json]

Workload: tools/time_search.py's set and random nets (350 x 1242, D = 228).  Per arch:

* ablation_s: tools/ablation.py's main() in this process, Searcher construction included (for 'slow' that is the one pass
  of the scorer head over every image);
* evaluators_s: for every variant, Evaluator(...) construction + test('test_te') -- what running ``run_main.py -a test_te
  -sm_skip X`` per variant costs minus process start-up;
* scores_match: every ablation score equals float('%.14g' % the Evaluator's mean).

Prints one JSON object with the card's name and power limit, read in the same run.  Needs a GPU.
"""
import argparse
import contextlib
import importlib.util
import io
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def time_arch(arch, root, net):
    import torch

    from mccnn_b200 import evaluate, pipeline, search

    ab = _tool("ablation")
    torch.cuda.synchronize()
    t = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        res = ab.main(["kitti", arch, net or "-", "-data_root", root])
    torch.cuda.synchronize()
    out = {"variants": len(res), "ablation_s": time.perf_counter() - t}
    torch.cuda.empty_cache()
    t = time.perf_counter()
    variants =search.ablation_variants(pipeline.make_params("kitti", arch))
    match = [l for l, _ in variants] == [l for l, _ in res]
    for (label, ov), (_, score) in zip(variants, res):
        ev = evaluate.Evaluator("kitti", arch, net_fname=net, **ov)
        try:
            want = float("%.14g" % ev.test("test_te", data_root=root, verbose=False).mean)
        except ValueError:                                   # NaN prediction
            want = float("nan")
        finally:
            ev.close()
        match = match and (score == want or (score != score and want != want))
    torch.cuda.synchronize()
    out.update(evaluators_s=time.perf_counter() - t, scores_match=match, scores=dict((l, s) for l, s in res))
    out["speedup"] = out["evaluators_s"] / out["ablation_s"]
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(prog="time_ablation.py", description=__doc__.splitlines()[0])
    ap.add_argument("-n_te", type=int, default=8)
    ap.add_argument("-archs", default="fast,slow")
    ap.add_argument("-seed", type=int, default=0)
    ap.add_argument("-out", default="")
    a = ap.parse_args(argv)
    import torch

    import mccnn_b200  # noqa: F401

    if not torch.cuda.is_available():
        raise SystemExit("time_ablation.py: no GPU")
    ts = _tool("time_search")
    out = {"workload": {"H": ts.H, "W": ts.W, "D": ts.D, "n_te": a.n_te}, "card": ts.card()}
    with tempfile.TemporaryDirectory() as tmp:
        nets = ts.write_world(tmp, a.n_te, a.seed)
        for arch in [s for s in a.archs.split(",") if s]:
            out[arch] = time_arch(arch, tmp, nets.get(arch))
            print(json.dumps({arch: out[arch]}), flush=True)
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
