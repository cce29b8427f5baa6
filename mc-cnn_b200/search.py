"""hs.py's parameter search with action ``test_te`` (hs.py:53-153 grids, :155-211 the loop): choose the stereo method's
parameters for a network by scoring candidate parameter sets on the validation images.

    s = Searcher("kitti", "slow", net_fname="net/net_kitti_slow_-a_train_tr.t7")
    score, errs = s.score({"L1": 5, "cbca_i1": 2, ...})    # == float("%.14g" % Evaluator(..., **p).test("test_te").mean)

hs.py starts one ``main.lua ... -a test_te`` process per candidate, which reloads the data and the net and recomputes every
image's matching cost.  The parameters only act after the cost volume, so here one process holds what does not change:

* the images and ground truths on the device, one :class:`pipeline.StereoPipeline` at the largest (H, W, D) of the examples,
  re-targeted per candidate with ``set_params``;
* arch 'slow': the scorer head's volumes (+ fix_border) of every example, computed once into pinned host memory (left volume
  only without the LR check) and staged into two device slots on a copy stream, the copy of example i + 1 overlapping the
  chain of example i (``run_volumes``);
* arch 'fast': the tower runs per candidate on the device-resident images, then ``run_shape`` (its output would take 8.9 GB
  of device memory at KITTI size for 40 images, so it is not kept);
* arch 'ad' / 'census': the volumes are recomputed per example into one reusable device buffer, then ``run_volumes``.

The CBCA mode is the one :class:`evaluate.Evaluator` runs for the arch, so that the scores are the same numbers: the default
mode for 'fast' (``run_shape``), the exact mode for 'slow', 'ad' and 'census' (the operator chain, bit-identical to the
reference).  Bad pixels are counted on the device (main.lua:1230-1236 in float32) with one host read per candidate.

A candidate may also set main.lua's ``sm_skip`` / ``sm_terminate`` (``s.score({"sm_skip": "sgm"})``): the same cached volumes
and the same pipeline then score a stereo-method ablation (:func:`ablation_variants`, tools/ablation.py).

The log lines are hs.py's (``score dataset arch test_te -name value ... -use_cache`` / ``-net_fname N``), so hs.sh.* output
and ours can be mixed.
"""
import os
import random

import numpy as np
import torch

from . import adcensus, dataio, evaluate, frontend, pipeline

METHODS = ("random", "hillclimb_slow", "hillclimb_fast", "hillclimb_dim")
ARCHS = pipeline.ARCHS
DATASETS = ("kitti", "kitti2015", "mb")

# hs.py:53-91 -- the same grid for kitti / kitti2015 x slow, ad and census; Python literals kept (int vs float), the log
# prints them as hs.py does
KITTI_TE = [
    ("L1", [0, 1, 2, 3, 4, 5, 6]),
    ("cbca_i1", [0, 2, 4, 6, 8]),
    ("cbca_i2", [0, 2, 4, 6, 8]),
    ("tau1", [0.01, 0.02, 0.03, 0.05, 0.08, 0.13, 0.22, 0.36, 0.6, 1.0]),
    ("pi1", [0.25, 0.33, 0.44, 0.57, 0.76, 1.0, 1.32, 1.74, 2.3, 3.03, 4.0]),
    ("pi2", [8.0, 10.56, 13.93, 18.38, 24.25, 32.0, 42.22, 55.72, 73.52, 97.01, 128.0]),
    ("sgm_q1", [3, 3.5, 4, 4.5, 5]),
    ("sgm_q2", [2, 2.5, 3, 3.5, 4, 4.5]),
    ("alpha1", [1.0, 1.25, 1.5, 1.75, 2.0, 2.25, 2.5, 2.75]),
    ("tau_so", [0.01, 0.02, 0.03, 0.05, 0.08, 0.13, 0.22, 0.36, 0.6, 1.0]),
    ("blur_sigma", [1.0, 1.29, 1.67, 2.15, 2.78, 3.59, 4.64, 5.99, 7.74, 10.0]),
    ("blur_t", [1, 2, 3, 4, 5, 6, 7]),
]
# hs.py:93-107 -- kitti / kitti2015 x fast
KITTI_FAST = [
    ("pi1", [0.25, 0.33, 0.44, 0.57, 0.76, 1.0, 1.32, 1.74, 2.3, 3.03, 4.0]),
    ("pi2", [8.0, 10.56, 13.93, 18.38, 24.25, 32.0, 42.22, 55.72, 73.52, 97.01, 128.0]),
    ("sgm_q1", [3, 3.5, 4, 4.5, 5]),
    ("sgm_q2", [2, 2.5, 3, 3.5, 4, 4.5]),
    ("alpha1", [1.0, 1.25, 1.5, 1.75, 2.0, 2.25, 2.5, 2.75]),
    ("tau_so", [0.01, 0.02, 0.03, 0.05, 0.08, 0.13, 0.22, 0.36, 0.6, 1.0]),
    ("blur_sigma", [1.0, 1.29, 1.67, 2.15, 2.78, 3.59, 4.64, 5.99, 7.74, 10.0]),
    ("blur_t", [1, 2, 3, 4, 5, 6, 7]),
]
# hs.py:135-153 -- mb x any arch (L1, cbca_i1, cbca_i2 and tau1 are commented out there)
MB_TE = [
    ("pi1", [0.2, 0.3, 0.4, 0.6, 0.8, 1.0, 1.3, 1.7, 2.3, 3.0, 4.0]),
    ("pi2", [2.0, 2.6, 3.5, 4.6, 6.1, 8.0, 10.6, 13.9, 18.4, 24.3, 32.0]),
    ("sgm_q1", [3, 3.5, 4, 4.5, 5]),
    ("sgm_q2", [2, 2.5, 3, 3.5, 4, 4.5]),
    ("alpha1", [1.0, 1.25, 1.5, 1.75, 2.0, 2.25, 2.5, 2.75]),
    ("tau_so", [0.01, 0.02, 0.03, 0.05, 0.08, 0.13, 0.22, 0.36, 0.6, 1.0]),
    ("blur_sigma", [1.0, 1.29, 1.67, 2.15, 2.78, 3.59, 4.64, 5.99, 7.74, 10.0]),
    ("blur_t", [1, 2, 3, 4, 5]),
]


class SearchError(ValueError):
    """A log or an argument the search cannot use."""


class NaNPrediction(ValueError):
    """A parameter set whose prediction contains NaN on an example (main.lua:1224 asserts there)."""

    def __init__(self, example_id):
        super().__init__("example %s: the prediction contains NaN" % (example_id,))
        self.example_id = example_id


def grid(dataset, arch):
    """hs.py:53-153: the test_te grid of (dataset, arch) as [(name, values)]"""
    if dataset not in DATASETS or arch not in ARCHS:
        raise SearchError("no test_te grid for dataset %r, arch %r" % (dataset, arch))
    if dataset == "mb":
        return MB_TE
    return KITTI_FAST if arch == "fast" else KITTI_TE


def valid(ps):
    """hs.py's valid(): pi1 must not exceed pi2"""
    return not ps["pi1"] > ps["pi2"]


def point(params, x):
    """hs.py:198: grid indices -> [(name, value)]"""
    return [(params[i][0], params[i][1][x[i]]) for i in range(len(params))]


def format_params(ps):
    """hs.py:203: '-name value ...' with Python's str() of each literal"""
    return " ".join("-{} {}".format(*p) for p in ps)


def format_line(score, dataset, arch, ps, net_fname="-"):
    """hs.py:203-211: the line hs.py prints for one evaluation (without the newline)"""
    ps_str = format_params(ps)
    if arch == "slow":
        ps_str += " -use_cache"
    else:
        ps_str += " -net_fname {}".format(net_fname)
    return " ".join(str(v) for v in (score, dataset, arch, "test_te", ps_str))


def parse_log(lines, dataset, arch, params):
    """hs.py:159-168: the (score, ps_str) of every line for (dataset, arch, test_te).  Lines that do not split into five fields
    or whose score is not a number are skipped (hs.py's ValueError); a matching line whose parameter names are not the grid's,
    in order, is refused."""
    out = []
    for line in lines:
        try:
            score, dataset_, arch_, action_, ps_str = line.strip().split(" ", 4)
            score = float(score)
        except ValueError:
            continue
        if dataset_ == dataset and arch_ == arch and action_ == "test_te":
            recover(params, ps_str)
            out.append((score, ps_str))
    return out


def recover(params, ps_str):
    """hs.py:171-178: grid indices of a logged point, each value mapped to the nearest grid value (ties: the lower index);
    tokens after the grid's (-use_cache, -net_fname N) are ignored"""
    tok = ps_str.split()
    x = []
    for i, (name, vals) in enumerate(params):
        if 2 * i + 1 >= len(tok) or tok[2 * i] != "-" + name:
            raise SearchError("log line %r: parameter %d is not -%s (the %s grid is %s)"
                              % (ps_str, i + 1, name, "test_te", " ".join(n for n, _ in params)))
        try:
            val = float(tok[2 * i + 1])
        except ValueError:
            raise SearchError("log line %r: -%s %r is not a number" % (ps_str, name, tok[2 * i + 1]))
        x.append(min([(abs(val - v), j) for j, v in enumerate(vals)])[1])
    return x


def propose(method, params, rng, results=None):
    """hs.py:156-195: the next grid indices.  random: uniform; hillclimb_*: from the minimum of `results` ((score, ps_str) of
    the matching log lines), move to neighbours -- every coordinate by -1 / 0 / +1 (fast), one random coordinate (slow), or
    one random coordinate to any value (dim).  `rng` is a random.Random."""
    if method == "random":
        return [rng.randint(0, len(vals) - 1) for _, vals in params]
    if method not in METHODS:
        raise SearchError("method must be one of %s, got %r" % (", ".join(METHODS), method))
    if not results:
        raise SearchError("%s: the log has no line for this dataset, arch and action to climb from" % method)
    _, ps_str = min(results)
    x = recover(params, ps_str)
    if method == "hillclimb_dim":
        i = rng.randrange(len(params))
        x[i] = rng.randrange(len(params[i][1]))
    else:
        ps = range(len(params)) if method == "hillclimb_fast" else [rng.randint(0, len(params) - 1)]
        for i in ps:
            ns = [x[i]]
            if x[i] - 1 >= 0:
                ns.append(x[i] - 1)
            if x[i] + 1 < len(params[i][1]):
                ns.append(x[i] + 1)
            x[i] = rng.choice(ns)
    return x


def ablation_variants(opt):
    """The stereo-method ablation for the parameters `opt` (a pipeline.Params) as [(label, overrides)]: the full chain, each
    ``-sm_skip`` step, then each ``-sm_terminate`` step (main.lua:953-1082), in the order the chain runs them.  Steps that
    do no work with these parameters (pipeline.idle_steps: the LR-check steps on mb, CBCA in the fast presets, ...) are
    left out, since their variants repeat another one's result."""
    idle = pipeline.idle_steps(opt)
    out = [("full", {})]
    for option, names in (("sm_skip", SKIP_STEPS), ("sm_terminate", TERMINATE_STEPS)):
        out += [("-%s %s" % (option, n), {option: n}) for n in names if n not in idle]
    return out


# main.lua's step names in chain order (main.lua:988-1077); the same names as pipeline.SM_SKIP / SM_TERMINATE
SKIP_STEPS = ("cbca", "sgm", "occlusion", "subpixel_enchancement", "median", "bilateral")
TERMINATE_STEPS = ("cnn", "cbca1", "sgm", "cbca2", "occlusion", "mismatch", "subpixel_enchancement", "median")


class Searcher:
    """Scores parameter sets of one (dataset, arch, net) on the test_te examples; see the module docstring."""

    def __init__(self, dataset, arch, net_fname=None, data_root=".", rect="imperfect", color="gray", device=0):
        evaluate.check_options(dataset, color=color)
        self.dataset, self.arch = dataset, arch
        self.params = grid(dataset, arch)
        self.method = frontend.StereoMethod(dataset, arch, net_fname)
        if self.method.needs_net:
            raise SearchError("arch '%s' needs a net file" % arch)
        self.opt = self.method.opt
        self.dev = torch.device("cuda", device)
        self.err_at = dataio.ERR_AT[dataset]
        self.data = evaluate.load_data(dataset, data_root, rect, color)
        self.examples = self.data.examples("test_te")
        self.head_calls = 0
        self.cache_fill_seconds = 0.0
        self.sp = None
        with torch.cuda.device(self.dev):
            self.x, self.gt, self.shapes, self.ids = [], [], [], []
            for ex in self.examples:
                x, disp_max, id_, _, img_width = self.data.example(ex)
                self.x.append(torch.from_numpy(x).to(self.dev))
                self.gt.append(torch.from_numpy(self.data.ground_truth(ex, img_width)).to(self.dev))
                self.shapes.append((x.shape[2], x.shape[3], disp_max))
                self.ids.append(id_)
            self.tower, self.head = self.method.stages(self.dev)
            H, W, D = (max(s[k] for s in self.shapes) for k in range(3))
            self.sp = pipeline.StereoPipeline(self.tower.fm if self.tower else 1, D, H, W, self.opt, device=self.dev.index,
                                              cbca_mode=None if arch == "fast" else "exact")
            self.copy_stream = torch.cuda.Stream(self.dev)
            nv = 2 if self.opt.lr_check else 1
            if arch == "slow":
                self._fill_cache(nv)
                self.slots = [torch.empty(nv * D * H * W, device=self.dev) for _ in range(2)]
                self.ev_in = [torch.cuda.Event() for _ in range(2)]
                self.ev_free = [torch.cuda.Event() for _ in range(2)]
            elif arch in ("ad", "census"):
                self.vols = torch.empty(nv * D * H * W, device=self.dev)

    def close(self):
        if self.sp is not None:
            self.sp.close()
        self.method.close()
        self.sp = self.tower = self.head = None

    def _views(self, buf, i):
        """(volL, volR or None) as (1, D, H, W) views of the first elements of `buf` at example i's shape"""
        H, W, D = self.shapes[i]
        n = D * H * W
        vl = buf[:n].view(1, D, H, W)
        vr = buf[n:2 * n].view(1, D, H, W) if self.opt.lr_check else None
        return vl, vr

    def head_volumes(self, i):
        """arch 'slow', example i: the scorer head's volumes + fix_border (main.lua:956-981), as pipeline.stereo_predict
        makes them: (volL, volR or None), (1, D, H, W) device tensors"""
        self.head_calls += 1
        x = self.x[i]
        D = self.shapes[i][2]
        feats = self.tower.forward(x)
        vl, vr = self.head.volumes(feats[0].contiguous(), feats[1].contiguous(), D, want_right=bool(self.opt.lr_check))
        adcensus.fix_border(vl, self.opt.border, -1)                                            # :981
        if vr is not None:
            adcensus.fix_border(vr, self.opt.border, 1)
        return vl, vr

    def _fill_cache(self, nv):
        """every example's head volumes into pinned host memory, allocated up front"""
        import time

        sizes = [nv * D * H * W for H, W, D in self.shapes]
        total = 4 * sum(sizes)
        try:
            self.cache = [torch.empty(n, dtype=torch.float32, pin_memory=True) for n in sizes]
        except RuntimeError as e:
            self.cache = None
            raise MemoryError("arch 'slow': the cost-volume cache needs %d bytes of pinned host memory (%d examples), which "
                              "could not be allocated: %s" % (total, len(sizes), str(e).splitlines()[0])) from None
        self.cache_bytes = total
        torch.cuda.synchronize(self.dev)
        t0 = time.perf_counter()
        for i in range(len(self.examples)):
            vl, vr = self.head_volumes(i)
            n = vl.numel()
            self.cache[i][:n].copy_(vl.reshape(-1))
            if vr is not None:
                self.cache[i][n:].copy_(vr.reshape(-1))
        torch.cuda.synchronize(self.dev)
        self.cache_fill_seconds = time.perf_counter() - t0

    def _stage(self, i):
        """H2D of example i's cached volumes into slot i % 2 on the copy stream, once the slot's previous example is done"""
        k = i % 2
        n = self.cache[i].numel()
        with torch.cuda.stream(self.copy_stream):
            if i >= 2:
                self.copy_stream.wait_event(self.ev_free[k])
            self.slots[k][:n].copy_(self.cache[i], non_blocking=True)
            self.ev_in[k].record(self.copy_stream)

    def predict(self, i):
        """the disparity map of example i with the current parameters, (H, W) on the device, ordered on the current stream.
        arch 'slow' expects example i to have been staged (_stage)."""
        x = self.x[i]
        D = self.shapes[i][2]
        if self.arch == "fast":
            feats = self.tower.forward(x)
            return self.sp.run_shape(feats[0], feats[1], x[0, 0], x[1, 0], disp_max=D)
        if self.arch == "slow":
            k = i % 2
            torch.cuda.current_stream(self.dev).wait_event(self.ev_in[k])
            vl, vr = self._views(self.slots[k], i)
            disp = self.sp.run_volumes(vl, vr, x[0, 0], x[1, 0], disp_max=D)
            self.ev_free[k].record(torch.cuda.current_stream(self.dev))
            return disp
        vl, vr = self._views(self.vols, i)
        adcensus.fill_nan(vl)                                                                    # :933 / :939
        cost = adcensus.ad if self.arch == "ad" else adcensus.census
        cost(x[0:1], x[1:2], vl, -1)                                                             # :934 / :940
        if vr is not None:
            adcensus.fill_nan(vr)
            cost(x[1:2], x[0:1], vr, 1)                                                          # :935 / :941
        return self.sp.run_volumes(vl, vr, x[0, 0], x[1, 0], disp_max=D)

    def options(self, overrides):
        """the Params of a candidate: the preset with the net's border, then `overrides` ({name: value})"""
        unknown = set(overrides) - set(n for n, _ in pipeline.Params._fields_)
        if unknown:
            raise SearchError("unknown parameter(s) %s" % ", ".join(sorted(unknown)))
        return self.method.params(**overrides)

    def score(self, overrides):
        """(score, [err per example]) of one parameter set: err = bad / valid pixels (main.lua:1224-1236), score =
        float('%.14g' % mean), what hs.py reads from main.lua's last line.  Raises NaNPrediction for a prediction with NaN."""
        opt = self.options(dict(overrides))
        n = len(self.examples)
        with torch.cuda.device(self.dev):
            self.sp.set_params(opt)
            self.opt = opt
            counts = torch.zeros((n, 3), dtype=torch.int64, device=self.dev)      # bad, valid, NaN
            if self.arch == "slow" and n:
                self._stage(0)
            for i in range(n):
                if self.arch == "slow" and i + 1 < n:
                    self._stage(i + 1)
                pred = self.predict(i)
                gt = self.gt[i]
                mask = gt != 0                                                                   # :1230
                counts[i, 0] = ((torch.abs(gt - pred) > self.err_at) & mask).sum()                # :1231-1234
                counts[i, 1] = mask.sum()
                counts[i, 2] = torch.isnan(pred).sum()
            c = counts.cpu().numpy()
        for i in range(n):
            if c[i, 2]:
                raise NaNPrediction(self.ids[i])
        errs = [float(b) / v if v else float("nan") for b, v in c[:, :2].tolist()]
        mean = sum(errs) / len(errs) if errs else float("nan")
        return float("%.14g" % mean), errs
