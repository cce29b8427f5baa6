"""The evaluation actions of main.lua for a trained network: ``-a test_te``, ``-a test_all``, ``-a submit`` and ``-a time``
(main.lua:393-491 loading, 1107-1138 example lists, 1140-1170 time, 1172-1293 the loop, the metric and the writers).

    ev = Evaluator("kitti", "fast", net_fname="net/net_kitti_fast_-a_train_all.t7")
    res = ev.test("test_te", data_root=".")        # res.examples: [(example, id, runtime, err)], res.mean
    ev.submit(data_root=".", out="out")            # PNG16 / PFM + time files, then out/submission.zip
    ev.time()                                      # best-of-N runtime of stereo_predict

Each action prints what main.lua prints (``runtime\\terr`` per example, the mean; the minimum for ``time``), numbers as Lua's
tostring writes them (%.14g), and returns the values as well.

Stage routing per image (the timed region is exactly main.lua's ``stereo_predict(x_batch, id)``):

* arch 'fast': feature tower -> :meth:`pipeline.StereoPipeline.run_shape` on one pipeline created at the largest (H, W, D)
  of the examples, before the loop;
* arch 'slow': feature tower -> scorer head -> :func:`pipeline.stereo_predict`;
* arch 'ad' / 'census': :func:`pipeline.stereo_predict`.

Deliberate deviations from main.lua:

* ``submit`` refuses a non-empty output directory instead of running ``rm -rf out/*``;
* n_te is ``len(x0) - len(dispnoc)`` instead of the constant 195 / 200 (preprocess_kitti.lua writes dispnoc for the
  training rows only, so on real data the two agree), and KITTI's H and W come from x0's shape;
* ``-at 1`` (the combined 2012 + 2015 loader, used for training), ``-color rgb``, ``-debug`` and ``-use_cache`` /
  ``-make_cache`` are refused (none changes the default result); -debug's images come from ``test(..., debug_dir=...)``
  (tools/debug_images.py) instead;
* ``-sm_terminate`` / ``-sm_skip`` (``Evaluator(..., sm_skip="sgm")``) accept only the step names main.lua tests
  (:data:`pipeline.SM_TERMINATE`, :data:`pipeline.SM_SKIP`); main.lua ignores any other name and runs the full chain.
  :func:`check_options` does not see the architecture and refuses both; :func:`check_stage_options`, which the command
  line uses, also refuses a step that does no work in the stereo method at hand (``-sm_terminate cbca1`` for kitti
  fast, which has no CBCA), whose result main.lua would print under the wrong variant's name;
* a Middlebury set smaller than 30 images submits all of them.

As in main.lua, the first example's runtime includes one-time initialisation; there is no hidden warm-up.
"""
import os
import time
import zipfile
from collections import namedtuple

import numpy as np
import torch

from . import dataio, frontend, pipeline, synth

ACTIONS = ("test_te", "test_all", "submit", "time")
TIME_SHAPES = {"tiny": (240, 320, 32), "kitti": (350, 1242, 228), "mb": (1000, 1500, 200)}   # main.lua:1141-1150
KITTI_DISP_MAX = 228                                                                          # main.lua:397

TestResult = namedtuple("TestResult", "examples mean")            # examples: [(example, id, runtime, err)]
SubmitResult = namedtuple("SubmitResult", "examples files zip")   # examples: [(example, id, runtime)]
TimeResult = namedtuple("TimeResult", "runtime_min runtimes")


def lua_num(x):
    """Lua 5.1's tostring of a number (LUAI_NUMFFORMAT "%.14g")"""
    return "%.14g" % x


def check_options(dataset, at=0, color="gray", debug=False, use_cache=False, make_cache=False, sm_terminate="",
                  sm_skip=""):
    """Refuse the main.lua options this module does not implement, with the reason."""
    if dataset not in ("kitti", "kitti2015", "mb"):
        raise ValueError("dataset must be 'kitti', 'kitti2015' or 'mb', got %r" % (dataset,))
    if at:
        raise ValueError("-at 1 (the combined KITTI 2012 + 2015 loader of main.lua:403-426) is not supported: it only "
                         "matters for training")
    if color != "gray":
        raise ValueError("-color %s is not supported: only grey Middlebury sets (-color gray) are" % color)
    if debug:
        raise ValueError("-debug is not supported: write its images with tools/debug_images.py (Evaluator.test(debug_dir=...)); "
                         "its other effect, saving the net after every training epoch (main.lua:877), is not implemented")
    for name, v in (("-use_cache", use_cache), ("-make_cache", make_cache)):
        if v:
            raise ValueError("%s is not supported" % name)
    # which steps exist depends on the architecture and its parameters, which this check does not see
    for name, v in (("-sm_terminate", sm_terminate), ("-sm_skip", sm_skip)):
        if v:
            raise ValueError("%s is checked with the stereo method it applies to: use check_stage_options(dataset, arch, "
                             "...)" % name)


def check_stage_options(dataset, arch, sm_terminate="", sm_skip="", **overrides):
    """Refuse a -sm_terminate / -sm_skip value that is not one of main.lua's step names, or that names a step doing no work
    in the stereo method of (dataset, arch) with `overrides` (pipeline.idle_steps): main.lua would run it and print the
    result of another variant under this one's name -- a wrong row in an ablation table."""
    opt = pipeline.make_params(dataset, arch, sm_terminate=sm_terminate, sm_skip=sm_skip, **overrides)
    idle = pipeline.idle_steps(opt)
    for option, name in (("sm_terminate", sm_terminate), ("sm_skip", sm_skip)):
        if name in idle:
            raise ValueError("-%s %s: that step does no work in the %s %s stereo method (cbca_i1 %d, cbca_i2 %d, sgm_i %d, "
                             "LR check %s), so the result would be another variant's"
                             % (option, name, dataset, arch, opt.cbca_i1, opt.cbca_i2, opt.sgm_i,
                                "on" if opt.lr_check else "off"))
    return opt


def _fromfile(path):
    for p in (path, path + ".dim"):
        if not os.path.exists(p):
            raise FileNotFoundError("missing data file %s" % p)
    return dataio.fromfile(path)


class KittiData:
    """main.lua:427-445: data.kitti/ or data.kitti2015/ under `data_root`."""

    def __init__(self, dataset, data_root="."):
        self.dataset = dataset
        d = os.path.join(data_root, "data.kitti" if dataset == "kitti" else "data.kitti2015")
        self.X0 = _fromfile(os.path.join(d, "x0.bin"))
        self.X1 = _fromfile(os.path.join(d, "x1.bin"))
        self.dispnoc = _fromfile(os.path.join(d, "dispnoc.bin"))
        self.metadata = _fromfile(os.path.join(d, "metadata.bin"))
        self.tr = _fromfile(os.path.join(d, "tr.bin")).astype(np.int64).reshape(-1)
        self.te = _fromfile(os.path.join(d, "te.bin")).astype(np.int64).reshape(-1)
        self.n_te = len(self.X0) - len(self.dispnoc)
        self.height, self.width = self.X0.shape[2], self.X0.shape[3]

    def examples(self, action):
        """main.lua:1107-1138 as 0-based row indices (the files hold 1-based ones)"""
        if action == "test_te":
            rows = self.te
        elif action == "test_all":
            rows = np.concatenate([self.tr, self.te])
        elif action == "submit":
            return list(range(len(self.X0) - self.n_te, len(self.X0)))
        else:
            raise ValueError("no example list for action %r" % (action,))
        return [int(i) - 1 for i in rows]

    def example(self, i):
        """main.lua:1177-1182: (x_batch (2,1,H,img_width), disp_max, id, img_height, img_width)"""
        img_height, img_width, id_ = (int(v) for v in self.metadata[i])
        x = np.ascontiguousarray(np.stack([self.X0[i, :, :, :img_width], self.X1[i, :, :, :img_width]]))
        return x, KITTI_DISP_MAX, id_, img_height, img_width

    def ground_truth(self, i, img_width):
        """main.lua:1226: the first img_width columns of dispnoc[i]"""
        if i >= len(self.dispnoc):
            raise ValueError("example %d has no ground truth (dispnoc holds %d rows)" % (i + 1, len(self.dispnoc)))
        return np.ascontiguousarray(self.dispnoc[i, 0, :, :img_width])

    def shape_of(self, i):
        return self.height, int(self.metadata[i, 1]), KITTI_DISP_MAX


class MiddleburyData:
    """main.lua:447-491: data.mb.<rect>_<color>/ under `data_root`; only light 1 of every image (the one the test and
    submit actions read)."""

    def __init__(self, data_root=".", rect="imperfect", color="gray"):
        self.dataset = "mb"
        d = os.path.join(data_root, "data.mb.%s_%s" % (rect, color))
        self.te = _fromfile(os.path.join(d, "te.bin")).astype(np.int64).reshape(-1)
        self.metadata = _fromfile(os.path.join(d, "meta.bin"))
        fs = os.path.join(d, "fname_submit.txt")
        if not os.path.exists(fs):
            raise FileNotFoundError("missing data file %s" % fs)
        with open(fs) as f:
            self.fname_submit = f.read().splitlines()
        self.X, self.dispnoc = [], {}
        for n in range(1, len(self.metadata) + 1):
            self.X.append(_fromfile(os.path.join(d, "x_%d_1.bin" % n)))
            g = os.path.join(d, "dispnoc%d.bin" % n)
            if os.path.exists(g):
                self.dispnoc[n - 1] = g

    def examples(self, action):
        """main.lua:1114-1131 as (0-based image index, 1-based right view)"""
        if action == "test_te":
            return [(int(i) - 1, 2) for i in self.te] + [(4, 3), (4, 4)]
        if action == "test_all":
            raise ValueError("test_all not supported on Middlebury.")                          # main.lua:1136
        if action == "submit":
            return [(i, 2) for i in range(max(0, len(self.X) - 30), len(self.X))]
        raise ValueError("no example list for action %r" % (action,))

    def example(self, ex):
        """main.lua:1184-1188: (x_batch (2,1,H,W), disp_max, id, H, W)"""
        i, right = ex
        disp_max = self.shape_of(ex)[2]
        views = self.X[i]
        if right > views.shape[0]:
            raise ValueError("Middlebury example %d_%d: image %d has %d views" % (i + 1, right, i + 1, views.shape[0]))
        x = np.ascontiguousarray(np.stack([views[0], views[right - 1]]))
        return x, disp_max, "%d_%d" % (i + 1, right), x.shape[2], x.shape[3]

    def ground_truth(self, ex, img_width=None):
        i = ex[0]
        if i not in self.dispnoc:
            raise ValueError("Middlebury image %d has no dispnoc%d.bin" % (i + 1, i + 1))
        g = dataio.fromfile(self.dispnoc[i])
        return g.reshape(g.shape[-2], g.shape[-1])

    def shape_of(self, ex):
        i, right = ex
        H, W, disp_max = (int(v) for v in self.metadata[i])
        if disp_max < 1:
            raise ValueError("Middlebury example %d_%d: disp_max %d (meta.bin) is not a disparity range" % (i + 1, right, disp_max))
        return H, W, disp_max


def load_data(dataset, data_root=".", rect="imperfect", color="gray"):
    check_options(dataset, color=color)
    if dataset == "mb":
        return MiddleburyData(data_root, rect, color)
    return KittiData(dataset, data_root)


class Evaluator:
    """The network and stereo method of one (dataset, arch), built once (:class:`frontend.StereoMethod`): tower and head on
    `device`, the parameters of main.lua's presets with `overrides`, fix_border's width from the network."""

    def __init__(self, dataset, arch, net_fname=None, device=0, **overrides):
        check_options(dataset)
        self.dataset, self.arch = dataset, arch
        self.method = frontend.StereoMethod(dataset, arch, net_fname, **overrides)
        self.opt = self.method.opt
        self.dev = torch.device("cuda", device)
        self.tower, self.head = self.method.stages(self.dev)
        self.sp = None

    @property
    def method_name(self):
        return "MC-CNN-" + ("fst" if self.arch == "fast" else "acrt")                          # main.lua:1217

    def prepare(self, shapes):
        """arch 'fast': one pipeline for every (H, W, D) in `shapes`, created at the largest of each"""
        if self.arch != "fast":
            return
        H, W, D = (max(s[k] for s in shapes) for k in range(3))
        if self.sp is not None:
            if H <= self.sp.H and W <= self.sp.W and D <= self.sp.D:
                return
            self.sp.close()
        self.sp = pipeline.StereoPipeline(self.tower.fm, D, H, W, self.opt, device=self.dev.index)

    def close(self):
        """release the pipeline, the feature tower and the scorer head"""
        if self.sp is not None:
            self.sp.close()
            self.sp = None
        self.method.close()

    def stereo_predict(self, x_batch, disp_max, conf=None, lr=None):
        """main.lua:929-1082 for one (2,1,H,W) device batch: (H, W) device disparity map.  `conf` / `lr`: (H, W) device
        tensors that receive the margin confidence and the LR check's outlier map (mc-cnn_b200/confidence.py)."""
        with torch.cuda.device(self.dev):
            if self.arch == "fast":
                feats = self.tower.forward(x_batch)
                return self.sp.run_shape(feats[0], feats[1], x_batch[0, 0], x_batch[1, 0], disp_max=disp_max, conf=conf,
                                         lr=lr)
            feats = self.tower.forward(x_batch) if self.arch == "slow" else None
            return pipeline.stereo_predict(x_batch, feats, self.opt, disp_max, arch=self.arch, head=self.head, conf=conf,
                                           lr=lr)[0, 0]

    def timed(self, x_batch, disp_max, conf=None):
        """main.lua:1195-1200: (pred, runtime in seconds) with the device synchronised before and after"""
        torch.cuda.synchronize(self.dev)
        t0 = time.perf_counter()
        pred = self.stereo_predict(x_batch, disp_max) if conf is None else self.stereo_predict(x_batch, disp_max, conf=conf)
        torch.cuda.synchronize(self.dev)
        return pred, time.perf_counter() - t0

    def _loop(self, data, examples):
        self.prepare([data.shape_of(ex) for ex in examples])
        for ex in examples:
            x, disp_max, id_, img_height, img_width = data.example(ex)
            x_batch = torch.from_numpy(x).to(self.dev)
            pred, runtime = self.timed(x_batch, disp_max)
            yield ex, id_, runtime, pred.cpu().numpy(), img_height, img_width

    def test(self, action="test_te", data_root=".", data=None, rect="imperfect", color="gray", verbose=True, debug_dir=None):
        """``-a test_te`` / ``-a test_all``: per example ``runtime\\terr`` and the mean bad-pixel rate (main.lua:1224-1238, 1292).
        With `debug_dir`, each example's images of main.lua -debug are written there after its timed region
        (main.lua:1240-1265, :func:`render.write_debug_images`)."""
        if action not in ("test_te", "test_all"):
            raise ValueError("test() runs test_te or test_all, not %r" % (action,))
        data = data or load_data(self.dataset, data_root, rect, color)
        err_at = dataio.ERR_AT[self.dataset]
        out = []
        for ex, id_, runtime, pred, _, img_width in self._loop(data, data.examples(action)):
            if np.isnan(pred).any():                                                            # main.lua:1224
                raise ValueError("example %s: the prediction contains NaN" % (id_,))
            gt = data.ground_truth(ex, img_width)
            err = dataio.bad_pixel_rate(pred, gt, err_at)
            out.append((ex, id_, runtime, err))
            if verbose:
                print("%s\t%s" % (lua_num(runtime), lua_num(err)), flush=True)
            if debug_dir is not None:
                from . import render

                x, disp_max = data.example(ex)[:2]
                render.write_debug_images(debug_dir, self.dataset, self.arch, id_, x[0, 0], pred, gt, disp_max, err_at,
                                          device=self.dev)
        mean = sum(e[3] for e in out) / len(out) if out else float("nan")
        if verbose:
            print(lua_num(mean), flush=True)
        return TestResult(out, mean)

    def sparsification(self, action="test_te", data_root=".", data=None, rect="imperfect", color="gray", err_at=None,
                       verbose=True):
        """The sparsification curve of each example's map under its margin confidence (an addition beyond the reference,
        mc-cnn_b200/confidence.py): per example ``id\terr\tauc\tauc_opt`` (err = test()'s, e_20 of the curve), then
        ``mean`` and the three means.  `err_at` defaults to main.lua's for the dataset.  Returns [(id, Sparsification)]."""
        from . import confidence

        if action not in ("test_te", "test_all"):
            raise ValueError("sparsification() runs test_te or test_all, not %r" % (action,))
        data = data or load_data(self.dataset, data_root, rect, color)
        err_at = dataio.ERR_AT[self.dataset] if err_at is None else err_at
        examples = data.examples(action)
        self.prepare([data.shape_of(ex) for ex in examples])
        out = []
        for ex in examples:
            x, disp_max, id_, _, img_width = data.example(ex)
            x_batch = torch.from_numpy(x).to(self.dev)
            conf = torch.empty(x.shape[2:], device=self.dev)
            pred = self.stereo_predict(x_batch, disp_max, conf=conf)
            if torch.isnan(pred).any():                                                         # main.lua:1224
                raise ValueError("example %s: the prediction contains NaN" % (id_,))
            gt = torch.from_numpy(np.ascontiguousarray(data.ground_truth(ex, img_width), np.float32)).to(self.dev)
            with torch.cuda.device(self.dev):
                res = confidence.sparsification(pred.contiguous(), conf, gt.contiguous(), err_at)
            out.append((id_, res))
            if verbose:
                print("\t".join([str(id_)] + [lua_num(v) for v in (res.curve[-1], res.auc, res.auc_opt)]), flush=True)
        if verbose:
            means = [(sum(f(r) for _, r in out) / len(out)) if out else float("nan")
                     for f in (lambda r: r.curve[-1], lambda r: r.auc, lambda r: r.auc_opt)]
            print("\t".join(["mean"] + [lua_num(v) for v in means]), flush=True)
        return out

    def submit(self, data_root=".", out="out", data=None, rect="imperfect", color="gray"):
        """``-a submit`` (main.lua:1107-1120, 1202-1222, 1288-1290): KITTI PNG16 maps (kitti2015 under disp_0/), Middlebury
        disp0<method>.pfm (rows bottom-up) + time<method>.txt per image, then ``out/submission.zip`` (without ``.empty``)"""
        if os.path.isdir(out) and any(f != ".empty" for f in os.listdir(out)):
            raise ValueError("submit: output directory %s is not empty" % out)
        os.makedirs(out, exist_ok=True)
        data = data or load_data(self.dataset, data_root, rect, color)
        done, files = [], []
        for ex, id_, runtime, pred, img_height, img_width in self._loop(data, data.examples("submit")):
            if self.dataset in ("kitti", "kitti2015"):
                files.append(dataio.write_kitti_submission(pred, img_height, img_width, out, id_, self.dataset))
            else:
                base = os.path.join(out, data.fname_submit[ex[0] - (len(data.X) - len(data.fname_submit))])
                os.makedirs(base, exist_ok=True)
                files.append(os.path.join(base, "disp0%s.pfm" % self.method_name))
                dataio.write_pfm(np.flipud(pred), files[-1])
                files.append(os.path.join(base, "time%s.txt" % self.method_name))
                with open(files[-1], "w") as f:
                    f.write(lua_num(runtime))
            done.append((ex, id_, runtime))
        return SubmitResult(done, files, write_zip(out))

    def time(self, tiny=False, seed=0, n=None, verbose=True):
        """``-a time`` (main.lua:1140-1170): the minimum over N = 30 ('fast') or 3 runs of stereo_predict on one seeded pair at
        240x320 D 32 (-tiny), 350x1242 D 228 (kitti) or 1000x1500 D 200 (mb)"""
        key = "tiny" if tiny else self.dataset
        if key not in TIME_SHAPES:
            raise ValueError("-a time has no input size for %s (main.lua:1141-1150: -tiny, kitti or mb)" % self.dataset)
        H, W, D = TIME_SHAPES[key]
        rng = np.random.default_rng(seed)
        x = np.stack([synth._standardise(synth.natural_image(rng, H, W))[None] for _ in range(2)])
        x_batch = torch.from_numpy(np.ascontiguousarray(x)).to(self.dev)
        self.prepare([(H, W, D)])
        n = n or (30 if self.arch == "fast" else 3)                                             # main.lua:1152
        runtimes = [self.timed(x_batch, D)[1] for _ in range(n)]
        if verbose:
            print(lua_num(min(runtimes)), flush=True)
        return TimeResult(min(runtimes), runtimes)


def write_zip(out):
    """``cd out; zip -r submission.zip . -x .empty``: every directory and file under `out` with paths relative to it"""
    path = os.path.join(out, "submission.zip")
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for d, dirs, fs in os.walk(out):
            dirs.sort()
            rel = os.path.relpath(d, out)
            if rel != ".":
                z.write(d, rel + "/")
            for f in sorted(fs):
                p = os.path.join(d, f)
                if f == ".empty" or os.path.abspath(p) == os.path.abspath(path):
                    continue
                z.write(p, os.path.relpath(p, out))
    return path
