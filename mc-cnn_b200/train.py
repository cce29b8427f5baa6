"""main.lua's ``-a train_tr`` / ``-a train_all`` (main.lua:602-890) for the fast and slow architectures on KITTI 2012 / 2015
and Middlebury.

    opt = options("kitti", lr=0.002)                                   # main.lua's presets (:34-49, :206-262) + overrides
    fname = train("kitti", "train_tr", opt, data_root=".", seed=42)   # 14 epochs, net/net_<cmd_str>.t7, then test_te
    opt = options("kitti", "slow")                                     # arch 'slow' (:70-114): l2, nh2; no -m / -pow
    fname = train("kitti", "train_all", opt, args=["-a", "train_all"])  # ... then submit

Per step (bs / 2 samples of four ws x ws patches, ws = 1 + 2 l1): the host draws the augmentation parameters and builds each
patch's float 2x3 matrix as make_patch does (:607-619); the GPU (csrc/train.cu) warps the patches out of the device-resident
X0 / X1 (OpenCV's cubic warpAffine, restated bit for bit), runs net_tr forward and backward with Margin2 and applies the
momentum update, as one CUDA graph.  The host builds the next chunk of steps while the GPU runs the current one, and reads
the per-step losses once per epoch.

Random numbers: one Torch7 stream, ``torch.manualSeed(seed)`` (:340) -- MT19937 after init_genrand(seed), which numpy's
``MT19937._legacy_seeding`` reproduces -- consumed as main.lua consumes it: ``torch.randperm(#nnz)`` once (:657), each
convolution's reset() (weight then bias, U(-1/sqrt(9 cin), +1/sqrt(9 cin)) in double, stored as float), then per sample the
torch.uniform calls of :791-818 in order, each r / 2^32 * (b - a) + a in double (the flip draws only with -hflip / -vflip 1).
Torch7 is not available to compare against, so parity with Torch7 itself is **unpinned**, as in :mod:`preprocess`; the stream
is pinned against ``preprocess.MT19937`` and the line-by-line restatement in oracle/train.py.

Arch 'slow' (net_tr of main.lua:663-677, BCECriterion2): the stream is consumed as randperm, net_tr's constructors (each
convolution's reset(), then each nn.Linear's: weight (out, in) in order, then bias, U(-1/sqrt(in), +1/sqrt(in))), then
net_te's l1 convolutions constructed anew -- their reset() draws are thrown away when the weights are tied (:697-724), but
they advance the stream; SpatialConvolution1_fw draws nothing -- then the per-sample draws as for 'fast'.  This order is
read from the sources; parity with Torch7 is unpinned, and it is pinned against oracle/train_slow.py.

Dataset mb (main.lua:455-491, 828-841): the training images are every light group ``x_<i>_<j>.bin``, j >= 2, of the
images the nnz rows name, one device pair per (image, light, exposure) in a table the sampler reads (:class:`MbTrainSet`,
``mccnn_trainer_create``).  After the uniforms of :791-818 each sample draws light, exp, the d_exp test, exp_ only
when that test passes, then the d_light test, so a sample takes a variable number of words: ``mccnn_mb_sample_starts``
finds the boundaries in a buffer of raw words, numpy gathers the columns (:func:`draw_params_mb`), and the words drawn past
the last sample of a chunk go back to the stream, so chunked building gives the records building everything at once gives.
``torch.random()`` is taken to be one 32-bit output, like each uniform; pinned against oracle/train_mb.py, not Torch7.
Only grey sets (``-color gray``) are trained.

Deliberate deviations from main.lua:

* only archs 'fast' and 'slow' and datasets kitti / kitti2015 / mb; ``-at 1``, ``-subset`` < 1, ``-debug`` and (mb)
  ``-color rgb`` are refused;
* the net file goes to ``<data_root>/net/`` and an existing file is refused; the file name is built from main.lua's options
  only (``-data_root`` and ``-out`` are not part of it);
* Margin2's loss is the hinge terms summed in order, then divided by bs / 2 (Torch7's ``mean`` reduces in another order),
  BCECriterion2's ``sum`` is taken in row order, and the convolutions and Linear layers accumulate in another order than
  cuDNN / cuBLAS: all are fp32.
"""
import ctypes
import math
import os
import time

import numpy as np

from . import dataio, evaluate

EPOCHS = 14                                  # main.lua:779
LR_DROP_EPOCH = 12                           # :783-785
CHUNK = 256                                  # steps per host -> device copy of the warp parameters
TWO32 = 1.0 / 4294967296.0

# main.lua:34-49 (KITTI augmentation) and :206-262 (arch 'fast', kitti / kitti2015: the same training options)
AUGMENT = dict(hflip=0, vflip=0, rotate=7.0, hscale=0.9, scale=1.0, trans=0.0, hshear=0.1, brightness=0.7, contrast=1.3,
               d_vtrans=0.0, d_rotate=0.0, d_hscale=1.0, d_hshear=0.0, d_brightness=0.3, d_contrast=1.0)
NET = dict(at=0, m=0.2, pow=1, l1=4, fm=64, ks=3, lr=0.002, bs=128, mom=0.9, true1=1.0, false1=4.0, false2=10.0)
# main.lua:70-84 (arch 'slow', kitti / kitti2015)
NET_SLOW = dict(at=0, l1=4, fm=112, ks=3, l2=4, nh2=384, lr=0.003, bs=128, mom=0.9, true1=1.0, false1=4.0, false2=10.0)
PRESETS = {"fast": NET, "slow": NET_SLOW}
# main.lua:50-66 (Middlebury augmentation), :263-280 (arch 'fast', mb) and :115-131 (arch 'slow', mb); -ds is stored and,
# as in main.lua, has no effect
AUGMENT_MB = dict(hflip=0, vflip=0, rotate=28.0, hscale=0.8, scale=0.8, trans=0.0, hshear=0.1, brightness=1.3, contrast=1.1,
                  d_vtrans=1.0, d_rotate=3.0, d_hscale=0.9, d_hshear=0.3, d_brightness=0.7, d_contrast=1.1)
MB_DRAWS = dict(ds=2001, d_exp=0.2, d_light=0.2)
NET_MB = dict(m=0.2, pow=1, **MB_DRAWS, l1=5, fm=64, ks=3, lr=0.002, bs=128, mom=0.9, true1=0.5, false1=1.5, false2=6.0)
NET_SLOW_MB = dict(**MB_DRAWS, l1=5, fm=112, ks=3, l2=3, nh2=384, lr=0.003, bs=128, mom=0.9, true1=0.5, false1=1.5,
                   false2=18.0)
PRESETS_MB = {"fast": NET_MB, "slow": NET_SLOW_MB}
WARP_DTYPE = np.dtype([("m", "<f4", (6,)), ("contrast", "<f4"), ("brightness", "<f4"), ("image", "<i4"), ("view", "<i4")])
PAIR_DTYPE = np.dtype([("x0", "<u8"), ("x1", "<u8"), ("H", "<i4"), ("W", "<i4")])      # mccnn_train_pair
TRAIN_PARAMS, TRAIN_MOMENTA, TRAIN_GRADS, TRAIN_PATCHES, TRAIN_TOWER, TRAIN_NORM, TRAIN_NORMALIZED, TRAIN_JOIN, \
    TRAIN_JOIN_GRAD, TRAIN_HINGE, TRAIN_NORM_GRAD_OUT, TRAIN_DZ, TRAIN_LOSS = range(13)
TRAIN_ROWS, TRAIN_FC, TRAIN_SIGMOID, TRAIN_BCE_GRAD, TRAIN_ROWS_GRAD = range(13, 18)      # arch 'slow' only
SHARD_TOWER_OUT, SHARD_WGRAD_PART = range(2)                                               # a shard's gathered buffers
WGRAD_THREADS = 256                          # csrc/train.cu's WG_NT: thread t of wgrad_kernel sums patches t, t + 256, ...


def check_world(world, o):
    """refuse a data-parallel run of `world` ranks that cannot give the one-GPU bits, before any GPU work"""
    if world == 1:
        return
    if world < 1 or world & (world - 1):
        raise ValueError("%s ranks: data-parallel training needs a power of two ranks, so that each rank's patches are "
                         "whole residue classes of the %d-thread weight-gradient tree" % (world, WGRAD_THREADS))
    if world > min(WGRAD_THREADS, 2 * o["bs"]):
        raise ValueError("%d ranks: more ranks than the %d patches of a batch of -bs %d (at most %d ranks)"
                         % (world, 2 * o["bs"], o["bs"], min(WGRAD_THREADS, 2 * o["bs"])))


def shard_size(N, rank, world):
    """the patches n = rank, rank + world, ... of a batch of N: an arch 'fast' rank's share"""
    return (N - rank + world - 1) // world


def slow_shard_plan(o, rank, world):
    """an arch 'slow' rank's share (mccnn_trainer_slow_shard_plan) -> (b0, b1, e, [(z0, z1, nsplit)] per tower layer): it
    owns the patches [b0, b1) and the weight-gradient splits [z0, z1) of each layer, and runs the tower on [b0, e)"""
    from .adcensus import _check, lib

    plan = np.zeros(3 + 3 * o["l1"], np.int64)
    _check(lib().mccnn_trainer_slow_shard_plan(o["l1"], o["fm"], o["bs"], rank, world,
                                               plan.ctypes.data_as(ctypes.c_void_p)), "mccnn_trainer_slow_shard_plan")
    return int(plan[0]), int(plan[1]), int(plan[2]), [tuple(int(v) for v in plan[3 + 3 * k:6 + 3 * k])
                                                      for k in range(o["l1"])]


def shard_patches(o, rank, world):
    """the patches of each batch a rank samples, as (first, stride, count): 'fast' rank, world, shard_size; 'slow' the
    patches [b0, e) of its plan"""
    if arch_of(o) == "slow":
        b0, _, e, _ = slow_shard_plan(o, rank, world)
        return b0, 1, e - b0
    return rank, world, shard_size(2 * o["bs"], rank, world)


def shard_warps(warps, o, rank, world):
    """rank's records of a chunk of whole-batch records (nsteps N,) -> (nsteps count,) of :func:`shard_patches`"""
    first, stride, count = shard_patches(o, rank, world)
    w = np.asarray(warps).reshape(-1, 2 * o["bs"])
    return np.ascontiguousarray(w[:, first:first + stride * (count - 1) + 1:stride]).reshape(-1)


def options(dataset, arch="fast", **overrides):
    """main.lua's training options for (dataset, arch) with `overrides`; refuses what this module does not train"""
    if dataset not in ("kitti", "kitti2015", "mb"):
        raise ValueError("dataset must be 'kitti', 'kitti2015' or 'mb', got %r" % (dataset,))
    if arch not in PRESETS:
        raise ValueError("arch %s: only the fast and slow architectures can be trained" % arch)
    o = dict(AUGMENT_MB, **PRESETS_MB[arch]) if dataset == "mb" else dict(AUGMENT, **PRESETS[arch])
    for k, v in overrides.items():
        if k not in o:
            raise ValueError("-%s is not a training option of arch %s" % (k, arch))
        o[k] = type(o[k])(v)
    check(o)
    return o


def arch_of(o):
    return "slow" if "l2" in o else "fast"


def check(o):
    """main.lua's asserts (:797, :810) and the limits of csrc/train.cu and the inference feature tower / scorer head"""
    if o.get("at"):
        raise ValueError("-at 1 (the combined KITTI 2012 + 2015 training set) is not supported")
    if o["ks"] != 3:
        raise ValueError("-ks %d: only 3x3 kernels are supported" % o["ks"])
    if not 1 <= o["l1"] <= 8:
        raise ValueError("-l1 %d: 1 to 8 layers are supported" % o["l1"])
    if o["fm"] < 16 or o["fm"] > 128 or o["fm"] % 16:
        raise ValueError("-fm %d: the feature tower runs 16 to 128 planes in steps of 16" % o["fm"])
    if o["bs"] < 2 or o["bs"] % 2:
        raise ValueError("-bs %d: the batch size must be even and at least 2" % o["bs"])
    if "pow" in o and o["pow"] not in (1, 2):
        raise ValueError("-pow %d: Margin2 takes pow 1 or 2" % o["pow"])
    if "l2" in o and not 1 <= o["l2"] <= 4:
        raise ValueError("-l2 %d: the scorer head runs 1 to 4 hidden layers" % o["l2"])
    if "nh2" in o and o["nh2"] not in (128, 256, 384):
        raise ValueError("-nh2 %d: the scorer head runs 128, 256 or 384 units" % o["nh2"])
    if not (o["hscale"] <= 1 and o["scale"] <= 1):
        raise ValueError("-hscale and -scale must be <= 1 (main.lua:797)")
    if not (o["contrast"] >= 1 and o["d_contrast"] >= 1):
        raise ValueError("-contrast and -d_contrast must be >= 1 (main.lua:810)")


def steps_per_epoch(n, bs):
    """the iterations of ``for t = 1, n - bs/2, bs/2`` (main.lua:789)"""
    h = bs // 2
    return max(0, (n - h - 1) // h + 1) if n - h >= 1 else 0


def lr_at(lr, epoch):
    """opt.lr during `epoch` (1-based): divided by 10 from epoch 12 on (main.lua:783-785)"""
    return lr / 10 if epoch >= LR_DROP_EPOCH else lr


def cmd_str(dataset, args, arch="fast"):
    """save_net's name stem (main.lua:344-347): dataset_arch then '_' + each further argument"""
    return "_".join([dataset, arch] + list(args))


def net_lines(o):
    """print_net(net_tr) (main.lua:542-564, 751); for 'slow' the other modules as the nn of that era prints them (unpinned)"""
    if arch_of(o) == "slow":
        out = []
        for i in range(o["l1"]):
            out += ["conv(in=%d, out=%d, k=%d)" % (1 if i == 0 else o["fm"], o["fm"], o["ks"]), "cudnn.ReLU"]
        out.append("nn.Reshape(%dx%d)" % (o["bs"], 2 * o["fm"]))
        for i in range(o["l2"]):
            out += ["nn.Linear(%d -> %d)" % (2 * o["fm"] if i == 0 else o["nh2"], o["nh2"]), "cudnn.ReLU"]
        return out + ["nn.Linear(%d -> 1)" % o["nh2"], "cudnn.Sigmoid"]
    out = []
    for i in range(o["l1"]):
        out.append("conv(in=%d, out=%d, k=%d)" % (1 if i == 0 else o["fm"], o["fm"], o["ks"]))
        if i < o["l1"] - 1:
            out.append("cudnn.ReLU")
    return out + ["nn.Normalize2", "nn.StereoJoin1"]


def epoch_line(epoch, err, lr, seconds):
    """``print(epoch, err_tr / err_tr_cnt, opt.lr, sys.clock() - time)`` (main.lua:880)"""
    return "\t".join(evaluate.lua_num(v) for v in (epoch, err, lr, seconds))


class Stream:
    """Torch7's generator after ``torch.manualSeed(seed)``: numpy's MT19937 with init_genrand seeding."""

    def __init__(self, seed):
        self.bg = np.random.MT19937()
        self.bg._legacy_seeding(seed)
        self.carry = np.zeros(0, np.uint32)      # words drawn ahead and handed back (see unread)

    def raw(self, n):
        if not len(self.carry):
            return self.bg.random_raw(n).astype(np.uint32)
        head, self.carry = self.carry[:n], self.carry[n:]
        return np.concatenate([head, self.bg.random_raw(n - len(head)).astype(np.uint32)])

    def unread(self, words):
        """hand back words that were drawn but not used: the next raw() returns them first"""
        self.carry = np.concatenate([np.asarray(words, np.uint32), self.carry])

    def uniform(self, n, a, b):
        return self.raw(n) * TWO32 * (b - a) + a

    def state(self):
        """-> (MT19937 key (624,) uint32, pos, carry): everything the next raw() depends on"""
        s = self.bg.state["state"]
        return np.asarray(s["key"], np.uint32).copy(), int(s["pos"]), self.carry.copy()

    def restore(self, key, pos, carry):
        self.bg.state = {"bit_generator": "MT19937", "state": {"key": np.asarray(key, np.uint32), "pos": int(pos)}}
        self.carry = np.asarray(carry, np.uint32).copy()


def randperm(stream, n):
    """``torch.randperm(n)`` as 1-based int64 (THTensor_(randperm): n - 1 swaps, one draw each)"""
    from .adcensus import _check, lib

    perm = np.arange(n, dtype=np.int64)
    step = 1 << 22
    for i0 in range(0, max(n - 1, 0), step):
        k = min(step, n - 1 - i0)
        d = np.ascontiguousarray(stream.raw(k))
        _check(lib().mccnn_randperm_swaps(perm.ctypes.data_as(ctypes.c_void_p), n, i0, d.ctypes.data_as(ctypes.c_void_p), k),
               "randperm")
    return perm + 1


def init_weights(stream, l1, fm, n_in=1, ks=3):
    """each convolution's reset() in order -> [(W (fm, cin, ks, ks), b (fm,))] float32"""
    out = []
    for i in range(l1):
        cin = n_in if i == 0 else fm
        stdv = 1 / math.sqrt(ks * ks * cin)
        w = stream.uniform(fm * cin * ks * ks, -stdv, stdv).astype(np.float32).reshape(fm, cin, ks, ks)
        b = stream.uniform(fm, -stdv, stdv).astype(np.float32)
        out.append((w, b))
    return out


def init_linear(stream, n_in, n_out):
    """nn.Linear(n_in, n_out):reset(): weight (out, in) then bias, U(-1/sqrt(in), +1/sqrt(in)) -> (W, b) float32"""
    stdv = 1 / math.sqrt(n_in)
    w = stream.uniform(n_out * n_in, -stdv, stdv).astype(np.float32).reshape(n_out, n_in)
    return w, stream.uniform(n_out, -stdv, stdv).astype(np.float32)


def init_slow(stream, o):
    """arch 'slow': net_tr's constructors, then net_te's convolutions, whose draws are thrown away (main.lua:663-695)
    -> (tower, head)"""
    tower = init_weights(stream, o["l1"], o["fm"])
    head = [init_linear(stream, 2 * o["fm"] if i == 0 else o["nh2"], o["nh2"]) for i in range(o["l2"])]
    head.append(init_linear(stream, o["nh2"], 1))
    init_weights(stream, o["l1"], o["fm"])
    return tower, head


def init_net(stream, o):
    """the reset() draws of either arch -> (tower, head); head None for 'fast'"""
    return init_slow(stream, o) if arch_of(o) == "slow" else (init_weights(stream, o["l1"], o["fm"]), None)


def uniform_columns(o):
    """the torch.uniform calls of main.lua:791-818 for one sample, in order"""
    return ["d_pos", "d_neg", "neg", "s", "hscale"] + (["hflip"] if o["hflip"] == 1 else []) + \
        (["vflip"] if o["vflip"] == 1 else []) + ["hshear", "trans0", "trans1", "phi", "brightness", "contrast",
                                                  "d_hscale", "d_hshear", "d_vtrans", "d_rotate", "d_brightness",
                                                  "d_contrast"]


def draw_params(stream, o, n):
    """the torch.uniform calls of main.lua:791-818 for n samples -> dict of float64 arrays (n,) (scale, trans pairs as
    two arrays)"""
    cols = uniform_columns(o)
    return params_from_words(stream.raw(n * len(cols)).reshape(n, len(cols)), o)


def params_from_words(words, o):
    """main.lua:791-818 from each sample's uniform words (n, len(uniform_columns(o))) uint32 -> dict as draw_params"""
    cols = uniform_columns(o)
    r = words.astype(np.float64) * TWO32
    c = {k: r[:, j] for j, k in enumerate(cols)}
    u = lambda k, a, b: c[k] * (b - a) + a
    p = {}
    p["d_pos"] = u("d_pos", -o["true1"], o["true1"])
    d_neg = u("d_neg", o["false1"], o["false2"])
    p["d_neg"] = np.where(c["neg"] < 0.5, -d_neg, d_neg)
    s = u("s", o["scale"], 1)
    sc0, sc1 = s * u("hscale", o["hscale"], 1), s
    if o["hflip"] == 1:
        sc0 = np.where(c["hflip"] < 0.5, -sc0, sc0)
    if o["vflip"] == 1:
        sc1 = np.where(c["vflip"] < 0.5, -sc1, sc1)
    p["scale"] = (sc0, sc1)
    p["hshear"] = u("hshear", -o["hshear"], o["hshear"])
    p["trans"] = (u("trans0", -o["trans"], o["trans"]), u("trans1", -o["trans"], o["trans"]))
    p["phi"] = u("phi", -o["rotate"] * math.pi / 180, o["rotate"] * math.pi / 180)
    p["brightness"] = u("brightness", -o["brightness"], o["brightness"])
    p["contrast"] = u("contrast", 1 / o["contrast"], o["contrast"])
    p["scale_"] = (p["scale"][0] * u("d_hscale", o["d_hscale"], 1), p["scale"][1])
    p["hshear_"] = p["hshear"] + u("d_hshear", -o["d_hshear"], o["d_hshear"])
    p["trans_"] = (p["trans"][0], p["trans"][1] + u("d_vtrans", -o["d_vtrans"], o["d_vtrans"]))
    p["phi_"] = p["phi"] + u("d_rotate", -o["d_rotate"] * math.pi / 180, o["d_rotate"] * math.pi / 180)
    p["brightness_"] = p["brightness"] + u("d_brightness", -o["d_brightness"], o["d_brightness"])
    p["contrast_"] = p["contrast"] * u("d_contrast", 1 / o["d_contrast"], o["d_contrast"])
    return p


def mb_sample_starts(raw, base, d_exp, cap):
    """mccnn_mb_sample_starts: (first word of each of the first <= cap whole samples, words they take)"""
    from .adcensus import _check, lib

    raw = np.ascontiguousarray(raw, np.uint32)
    starts = np.zeros(cap, np.int64)
    count, used = ctypes.c_longlong(), ctypes.c_longlong()
    _check(lib().mccnn_mb_sample_starts(raw.ctypes.data_as(ctypes.c_void_p), len(raw), base, d_exp,
                                        starts.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(count), ctypes.byref(used)),
           "mccnn_mb_sample_starts")
    return starts[:count.value], used.value


def draw_params_mb(stream, o, n_light, n_exp):
    """main.lua:791-841 for dataset mb, for len(n_light) samples whose images have n_light light groups j >= 2 and n_exp
    exposures in each -> (draw_params' dict, light, exp, light_, exp_ as int64 arrays, 1-based as in main.lua).

    A sample takes base + 4 or base + 5 words (exp_ is drawn only when the d_exp test passes), so the boundaries are found
    by a walk over the raw words (mccnn_mb_sample_starts); the words drawn past the last sample go back to `stream`.
    torch.random() is taken to be one 32-bit word, as for the uniforms."""
    n_light, n_exp = np.asarray(n_light, np.int64), np.asarray(n_exp, np.int64)
    n = len(n_light)
    base = len(uniform_columns(o))
    raw = stream.raw(n * (base + 5))                                              # enough for n samples
    starts, used = mb_sample_starts(raw, base, o["d_exp"], n)
    assert len(starts) == n
    stream.unread(raw[used:])
    p = params_from_words(raw[starts[:, None] + np.arange(base)], o)
    w = lambda k: raw[starts + base + k].astype(np.int64)
    light = w(0) % n_light + 2                                                    # :829
    exp = w(1) % n_exp + 1                                                        # :830
    t_exp = w(2) * TWO32 < o["d_exp"]                                             # :833
    exp_ = np.where(t_exp, w(3) % n_exp + 1, exp)                                 # :834
    t_light = raw[starts + base + 3 + t_exp].astype(np.float64) * TWO32 < o["d_light"]   # :836
    light_ = np.where(t_light, np.maximum(2, light - 1), light)                   # :837
    return p, light, exp, light_, exp_


def _mul32(a, b):
    """main.lua:603-605 on arrays"""
    return [a[0] * b[0] + a[1] * b[3], a[0] * b[1] + a[1] * b[4], a[0] * b[2] + a[1] * b[5] + a[2],
            a[3] * b[0] + a[4] * b[3], a[3] * b[1] + a[4] * b[4], a[3] * b[2] + a[4] * b[5] + a[5]]


def patch_matrices(ws, dim3, dim4, scale, phi, trans, hshear):
    """make_patch's matrix (main.lua:608-616) for arrays of patches -> (n, 6) float32"""
    m = [1, 0, -dim4, 0, 1, -dim3]
    m = _mul32([1, 0, trans[0], 0, 1, trans[1]], m)
    m = _mul32([scale[0], 0, 0, 0, scale[1], 0], m)
    c = np.array([math.cos(v) for v in phi])
    s = np.array([math.sin(v) for v in phi])
    m = _mul32([c, s, 0, -s, c, 0], m)
    m = _mul32([1, hshear, 0, 0, 1, 0], m)
    m = _mul32([1, 0, (ws - 1) / 2, 0, 1, (ws - 1) / 2], m)
    n = len(dim3)
    return np.stack([np.broadcast_to(np.asarray(v, np.float64), (n,)) for v in m], 1).astype(np.float32)


def make_warps(p, rows, ws, pairs=None):
    """main.lua:820-846: the (4 n,) mccnn_warp records of n samples from their parameters `p` and nnz rows (n, 4)
    (image 1-based, dim3, dim4, d).  The patches read image - 1 of X0 / X1, or with `pairs` = (left, right) (n,) pair
    indices (Middlebury) pair left's x0 and pair right's x1."""
    rows = np.asarray(rows, np.float32).astype(np.float64)
    n = len(rows)
    img, dim3, dim4, d = rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3]
    a = (p["scale"], p["phi"], p["trans"], p["hshear"])
    b = (p["scale_"], p["phi_"], p["trans_"], p["hshear_"])
    out = np.zeros((n, 4), WARP_DTYPE)
    out["m"][:, 0] = out["m"][:, 2] = patch_matrices(ws, dim3, dim4, *a)
    out["m"][:, 1] = patch_matrices(ws, dim3, dim4 - d + p["d_pos"], *b)
    out["m"][:, 3] = patch_matrices(ws, dim3, dim4 - d + p["d_neg"], *b)
    for j, (c, br) in enumerate([(p["contrast"], p["brightness"]), (p["contrast_"], p["brightness_"])] * 2):
        out["contrast"][:, j] = c.astype(np.float32)
        out["brightness"][:, j] = br.astype(np.float32)
    if pairs is None:
        out["image"] = (img.astype(np.int64) - 1)[:, None]
    else:
        out["image"] = np.stack([pairs[0], pairs[1], pairs[0], pairs[1]], 1)
    out["view"] = np.array([0, 1, 0, 1], np.int32)[None]
    return out.reshape(-1)


def sample_patches(X0, X1, warps, ws):
    """the sampler alone on the pairs (X0[i, 0], X1[i, 0]): X0 / X1 (n_img, 1, H, W) CUDA float32, warps a WARP_DTYPE
    array -> (len(warps), ws, ws) CUDA float32"""
    from .adcensus import _t

    name = "sample_patches"
    _t(X0, 1, name)
    _t(X1, 2, name)
    if X0.shape != X1.shape or X0.dim() != 4 or X0.shape[1] != 1:
        raise ValueError("%s: X0 and X1 must both be (n, 1, H, W)" % name)
    return sample_patches_pairs([(X0[i, 0], X1[i, 0]) for i in range(len(X0))], warps, ws)


def pair_table(planes):
    """[(x0, x1)] CUDA float32 (H, W) contiguous planes -> PAIR_DTYPE array (the planes must outlive every use)"""
    import torch

    t = np.zeros(len(planes), PAIR_DTYPE)
    for i, (a, b) in enumerate(planes):
        if a.shape != b.shape or a.dim() != 2 or not (a.is_contiguous() and b.is_contiguous()) or \
                a.dtype != torch.float32 or b.dtype != torch.float32 or not (a.is_cuda and b.is_cuda):
            raise ValueError("pair %d: x0 and x1 must be contiguous CUDA float32 (H, W) planes of one shape" % i)
        t[i] = (a.data_ptr(), b.data_ptr(), a.shape[0], a.shape[1])
    return t


def sample_patches_pairs(planes, warps, ws):
    """the sampler alone on a table of pairs (mccnn_train_sample_pairs): planes [(x0, x1)] CUDA float32 (H, W) planes,
    sizes free per pair, warps a WARP_DTYPE array whose image is a pair index -> (len(warps), ws, ws) CUDA float32"""
    import torch

    from .adcensus import _check, _stream, lib

    dev = planes[0][0].device
    table = torch.from_numpy(pair_table(planes).view(np.uint8)).to(dev)
    w = torch.from_numpy(np.ascontiguousarray(warps, WARP_DTYPE).view(np.uint8)).to(dev)
    out = torch.empty((len(warps), ws, ws), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _check(lib().mccnn_train_sample_pairs(table.data_ptr(), len(planes), w.data_ptr(), len(warps), ws, out.data_ptr(),
                                              _stream(out)), "sample_patches_pairs")
    return out


class TrainerConfig(ctypes.Structure):
    """mccnn_trainer_config"""

    _fields_ = [
        ("slow", ctypes.c_int),
        ("l1", ctypes.c_int),
        ("fm", ctypes.c_int),
        ("bs", ctypes.c_int),
        ("mom", ctypes.c_float),
        ("margin", ctypes.c_float),
        ("pow", ctypes.c_int),
        ("l2", ctypes.c_int),
        ("nh2", ctypes.c_int),
        ("chunk", ctypes.c_int),
        ("loss_cap", ctypes.c_int),
        ("rank", ctypes.c_int),
        ("world", ctypes.c_int),
    ]


class Trainer:
    """csrc/train.cu's trainer: net_tr + Margin2 ('fast') or + BCECriterion2 ('slow', when `o` has l2) and the momentum
    update on `device`, sampling from the pairs (X0[i, 0], X1[i, 0]) of X0 / X1 (n_img, 1, H, W) CUDA, or with `planes` =
    [(x0, x1)] CUDA (H, W) planes from that table of stereo pairs (a warp's image is a pair index).

    With `world` > 1, rank `rank` of a data-parallel run whose ranks exchange through `comm` (a rowband.Comm: send / recv
    / exchange / barrier): every rank is given the same records, runs the tower on its share of each batch
    (:func:`shard_warps`) and ends each step with the parameters, momenta and loss of the one-GPU trainer, bit for bit
    (csrc/train.cu's mccnn_trainer_create with world > 1)."""

    def __init__(self, o, X0=None, X1=None, chunk=CHUNK, loss_cap=1, device=None, planes=None, rank=0, world=1,
                 comm=None):
        import torch

        from .adcensus import _check, _stream, _t, lib

        check_world(world, o)
        if world > 1 and (comm is None or not 0 <= rank < world):
            raise ValueError("Trainer: rank %s of %d ranks needs a communicator" % (rank, world))
        self.rank, self.world, self.comm = rank, world, comm
        self.o, self.chunk = o, chunk
        src = X0 if planes is None else planes[0][0]
        self.dev = src.device if device is None else torch.device("cuda", device)
        self.arch = arch_of(o)
        self.l1, self.fm, self.bs = o["l1"], o["fm"], o["bs"]
        self.l2, self.nh2 = o.get("l2"), o.get("nh2")
        self.ws = 1 + 2 * self.l1
        self.N = 2 * self.bs
        self._keep = (X0, X1, planes)
        self._h = ctypes.c_void_p()
        if planes is None:
            _t(X0, 1, "Trainer")
            _t(X1, 2, "Trainer")
            planes = [(X0[i, 0], X1[i, 0]) for i in range(len(X0))]
        t = pair_table(planes)
        slow = self.arch == "slow"
        cfg = TrainerConfig(slow=slow, l1=self.l1, fm=self.fm, bs=self.bs, mom=o["mom"], margin=0 if slow else o["m"],
                            pow=1 if slow else o["pow"], l2=self.l2 or 0, nh2=self.nh2 or 0, chunk=chunk,
                            loss_cap=loss_cap, rank=rank, world=world)
        with torch.cuda.device(self.dev):
            self.stream = torch.cuda.current_stream(self.dev)
            _check(lib().mccnn_trainer_create(ctypes.byref(self._h), ctypes.byref(cfg), t.ctypes.data_as(ctypes.c_void_p),
                                              len(t), self.dev.index, _stream(src)), "mccnn_trainer_create")
            if world > 1:
                self.n_warps = shard_patches(o, rank, world)[2]
                self._gathered = [self._shard_slots(w) for w in (SHARD_TOWER_OUT, SHARD_WGRAD_PART)]
        self.launches_per_step = lib().mccnn_trainer_launches_per_step(self._h)

    def _shard_slots(self, what):
        """a shard's gathered buffer as views of the trainer's memory: [piece][rank] -> CUDA tensor (that rank's slot)"""
        import torch

        from .adcensus import _check, lib

        ptr, count = ctypes.c_void_p(), ctypes.c_longlong()
        _check(lib().mccnn_trainer_shard_buffer(self._h, what, ctypes.byref(ptr), ctypes.byref(count)),
               "mccnn_trainer_shard_buffer")
        view = type("DeviceArray", (), {"__cuda_array_interface__": dict(shape=(count.value,), typestr="<f4",
                                                                          data=(ptr.value, False), version=2)})()
        buf = torch.as_tensor(view, device=self.dev)
        out = []
        for piece in range(lib().mccnn_trainer_shard_pieces(self._h, what)):
            slots = []
            for r in range(self.world):
                off, n = ctypes.c_longlong(), ctypes.c_longlong()
                _check(lib().mccnn_trainer_shard_slot(self._h, what, piece, r, ctypes.byref(off), ctypes.byref(n)),
                       "mccnn_trainer_shard_slot")
                slots.append(buf[off.value:off.value + n.value])
            out.append(slots)
        return out

    def _all_gather(self, pieces):
        """every rank's slot of each piece from that rank, on the trainer's stream (empty slots are not sent)"""
        import torch

        with torch.cuda.stream(self.stream):
            for slots in pieces:
                mine = slots[self.rank]
                others = [p for p in range(self.world) if p != self.rank]
                self.comm.exchange({p: mine for p in others if mine.numel()},
                                   {p: slots[p] for p in others if slots[p].numel()})

    def close(self):
        from .adcensus import lib

        if getattr(self, "_h", None):
            lib().mccnn_trainer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def size(self, what):
        from .adcensus import lib

        return lib().mccnn_trainer_size(self._h, what)

    def get(self, what):
        """a copy of one of the trainer's buffers (TRAIN_*) as a CUDA float32 tensor"""
        import torch

        from .adcensus import _check, lib

        out = torch.empty(self.size(what), dtype=torch.float32, device=self.dev)
        _check(lib().mccnn_trainer_get(self._h, what, out.data_ptr(), self.stream.cuda_stream), "mccnn_trainer_get")
        return out

    def set(self, what, src):
        import torch

        from .adcensus import _check, lib

        t = torch.as_tensor(src, dtype=torch.float32).reshape(-1).to(self.dev).contiguous()
        if t.numel() != self.size(what):
            raise ValueError("Trainer.set: %d values for a buffer of %d" % (t.numel(), self.size(what)))
        _check(lib().mccnn_trainer_set(self._h, what, t.data_ptr(), self.stream.cuda_stream), "mccnn_trainer_set")
        self.stream.synchronize()

    def set_layers(self, layers, head=None):
        self.set(TRAIN_PARAMS, flatten(list(layers) + list(head or [])))

    def layers(self, what=TRAIN_PARAMS):
        """the tower's (W, b) of the parameters, momenta or gradients"""
        return unflatten(self.get(what).cpu().numpy(), self.l1, self.fm)

    def net(self, what=TRAIN_PARAMS):
        """(tower, head) of the parameters, momenta or gradients; head None for 'fast'"""
        v = self.get(what).cpu().numpy()
        tower = unflatten(v, self.l1, self.fm)
        return tower, (unflatten_head(v, self.l1, self.fm, self.l2, self.nh2) if self.arch == "slow" else None)

    def run(self, warps, lr):
        """len(warps) / N steps (<= chunk) from a WARP_DTYPE array (pinned host or CUDA uint8 tensor, or numpy).  A shard
        takes the whole batch's records as numpy, or its own share (:func:`shard_warps`) as a tensor."""
        import torch

        from .adcensus import _check, lib

        if isinstance(warps, np.ndarray):
            if self.world > 1:
                warps = shard_warps(warps, self.o, self.rank, self.world)
            warps = torch.from_numpy(np.ascontiguousarray(warps, WARP_DTYPE).view(np.uint8)).to(self.dev)
        if self.world == 1:
            nsteps = warps.numel() // (WARP_DTYPE.itemsize * self.N)
            _check(lib().mccnn_trainer_run(self._h, warps.data_ptr(), nsteps, lr, self.stream.cuda_stream),
                   "mccnn_trainer_run")
            return warps
        nsteps = warps.numel() // (WARP_DTYPE.itemsize * self.n_warps)
        _check(lib().mccnn_trainer_shard_begin(self._h, warps.data_ptr(), nsteps, lr, self.stream.cuda_stream),
               "mccnn_trainer_shard_begin")
        for _ in range(nsteps):
            for seg in range(3):
                _check(lib().mccnn_trainer_shard_segment(self._h, seg, self.stream.cuda_stream),
                       "mccnn_trainer_shard_segment")
                if seg < 2:
                    self._all_gather(self._gathered[seg])
        return warps

    def step_patches(self, patches, lr):
        import torch

        from .adcensus import _check, lib

        t = torch.as_tensor(patches, dtype=torch.float32).to(self.dev).contiguous()
        if t.numel() != self.N * self.ws * self.ws:
            raise ValueError("step_patches: (%d, 1, %d, %d) patches expected" % (self.N, self.ws, self.ws))
        _check(lib().mccnn_trainer_step_patches(self._h, t.data_ptr(), lr, self.stream.cuda_stream),
               "mccnn_trainer_step_patches")
        self._last = t

    def reset_losses(self):
        from .adcensus import _check, lib

        _check(lib().mccnn_trainer_reset_losses(self._h, self.stream.cuda_stream), "mccnn_trainer_reset_losses")

    def run_chunk(self, warps, lr):
        """run() from a WARP_DTYPE numpy array through two pinned host buffers, alternating; the host waits only before
        it refills a buffer, for the chunk that last read it"""
        import torch

        if self.world > 1:
            warps = shard_warps(warps, self.o, self.rank, self.world)
        if not hasattr(self, "_pinned"):
            rec = WARP_DTYPE.itemsize * (self.N if self.world == 1 else self.n_warps)
            self._pinned = [torch.empty(self.chunk * rec, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
            self._events, self._next = [None, None], 0
        b, nbytes = self._next, warps.nbytes
        if self._events[b] is not None:
            self._events[b].synchronize()
        self._pinned[b][:nbytes].numpy()[:] = warps.view(np.uint8)
        self.run(self._pinned[b][:nbytes], lr)
        self._events[b] = torch.cuda.Event()
        self._events[b].record(self.stream)
        self._next = 1 - b

    def losses(self, n):
        """the first n per-step losses since reset_losses(), float32"""
        return self.get(TRAIN_LOSS)[:n].cpu().numpy()

    def state(self):
        """-> (parameters, momenta) float32, read after the stream has drained"""
        self.stream.synchronize()
        return tuple(self.get(w).cpu().numpy() for w in (TRAIN_PARAMS, TRAIN_MOMENTA))

    def load_state(self, params, momenta):
        self.set(TRAIN_PARAMS, params)
        self.set(TRAIN_MOMENTA, momenta)


def flatten(layers):
    return np.concatenate([np.concatenate([np.asarray(w, np.float32).reshape(-1), np.asarray(b, np.float32).reshape(-1)])
                           for w, b in layers])


def unflatten(v, l1, fm):
    out, o = [], 0
    for i in range(l1):
        cin = 1 if i == 0 else fm
        w = v[o:o + fm * cin * 9].reshape(fm, cin, 3, 3)
        o += fm * cin * 9
        out.append((w.copy(), v[o:o + fm].copy()))
        o += fm
    return out


def unflatten_head(v, l1, fm, l2, nh2):
    """the Linear layers' (W (out, in), b (out,)) after the tower's parameters"""
    o = sum(fm * (1 if i == 0 else fm) * 9 + fm for i in range(l1))
    out = []
    for j in range(l2 + 1):
        n_in, n_out = 2 * fm if j == 0 else nh2, nh2 if j < l2 else 1
        w = v[o:o + n_out * n_in].reshape(n_out, n_in)
        o += n_out * n_in
        out.append((w.copy(), v[o:o + n_out].copy()))
        o += n_out
    return out


def load_nnz(data, action, data_root):
    d = os.path.join(data_root, "data.kitti" if data.dataset == "kitti" else "data.kitti2015")
    nnz = evaluate._fromfile(os.path.join(d, "nnz_tr.bin"))
    if action == "train_all":                                                    # main.lua:650-654
        nnz = np.concatenate([nnz, evaluate._fromfile(os.path.join(d, "nnz_te.bin"))])
    nnz = np.ascontiguousarray(nnz, np.float32).reshape(-1, 4)
    if len(nnz) and not (nnz[:, 0].min() >= 1 and nnz[:, 0].max() <= len(data.X0)):
        raise ValueError("%s: nnz rows name images outside 1 .. %d" % (d, len(data.X0)))
    return nnz


def _dims(path):
    """the dimensions in `path`.dim, after checking that the data, .dim and .type files exist"""
    for p in (path, path + ".dim", path + ".type"):
        if not os.path.exists(p):
            raise FileNotFoundError("missing data file %s" % p)
    with open(path + ".dim") as f:
        return [int(float(v)) for v in f.read().split()]


class MbTrainSet:
    """The training images of data.mb.<rect>_gray/ (main.lua:455-491): the nnz rows of `action` (nnz_tr, plus nnz_te for
    train_all) and, for every image they name, its light groups x_<i>_<j>.bin, j >= 2, each (n_exp, 2, 1, H, W).

    Everything is checked on the host from the .dim files, before any GPU work: a missing file, a row naming an image
    with no light group j >= 2 (main.lua:829 would take % 0), and an image whose light groups hold unequal exposure
    counts (:834-840 index light_ with an exposure drawn for light).  :meth:`upload` then refuses a set whose planes do
    not fit in the device's free memory, and copies each group file to the device once.  Pair (image, light, exp) is
    index ``first[image] + (light - 2) n_exp[image] + exp - 1``: x0 = group[exp - 1, 0], x1 = group[exp - 1, 1]."""

    def __init__(self, data_root=".", rect="imperfect", action="train_tr"):
        self.dir = d = os.path.join(data_root, "data.mb.%s_gray" % rect)
        nnz = evaluate._fromfile(os.path.join(d, "nnz_tr.bin"))
        if action == "train_all":                                                # main.lua:650-654
            nnz = np.concatenate([nnz, evaluate._fromfile(os.path.join(d, "nnz_te.bin"))])
        self.nnz = np.ascontiguousarray(nnz, np.float32).reshape(-1, 4)
        n_img = len(evaluate._fromfile(os.path.join(d, "meta.bin")))
        imgs = np.unique(self.nnz[:, 0]).astype(np.int64)
        if len(imgs) and not (imgs[0] >= 1 and imgs[-1] <= n_img):
            raise ValueError("%s: nnz rows name images outside 1 .. %d" % (d, n_img))
        self.groups = []                                                         # (image, light, path, dims)
        self.nbytes = 0
        counts = {}
        for i in imgs:
            exps = []
            j = 2
            while os.path.exists(os.path.join(d, "x_%d_%d.bin.dim" % (i, j))):
                p = os.path.join(d, "x_%d_%d.bin" % (i, j))
                dims = _dims(p)
                if len(dims) != 5 or dims[0] < 1 or dims[1] != 2 or dims[2] != 1 or min(dims[3:]) < 1:
                    raise ValueError("%s: a light group must be (n_exp, 2, 1, H, W), the .dim says %s" % (p, dims))
                self.groups.append((int(i), j, p, dims))
                self.nbytes += 4 * int(np.prod(dims))
                exps.append(dims[0])
                j += 1
            if not exps:
                raise ValueError("%s: nnz rows name image %d, which has no light group x_%d_2.bin (main.lua:829 would "
                                 "take %% 0)" % (d, i, i))
            if len(set(exps)) != 1:
                raise ValueError("%s: image %d's light groups hold unequal exposure counts %s (main.lua:834-840 index "
                                 "light_ with an exposure drawn for light)" % (d, i, exps))
            counts[int(i)] = (len(exps), exps[0])
        self._index(n_img, counts)

    @classmethod
    def from_counts(cls, nnz, counts):
        """the draws and pair indices of a set whose planes are built elsewhere (tools/time_train.py): counts
        {image: (light groups, exposures)}, pairs in the same order as :meth:`upload`'s"""
        self = cls.__new__(cls)
        self.dir, self.nnz, self.groups, self.nbytes = None, np.ascontiguousarray(nnz, np.float32).reshape(-1, 4), [], 0
        self._index(max(counts), counts)
        return self

    def _index(self, n_img, counts):
        self.n_light = np.zeros(n_img + 1, np.int64)                            # by 1-based image
        self.n_exp = np.zeros(n_img + 1, np.int64)
        self.first = np.full(n_img + 1, -1, np.int64)
        n_pairs = 0
        for i in sorted(counts):
            self.n_light[i], self.n_exp[i] = counts[i]
            self.first[i] = n_pairs
            n_pairs += counts[i][0] * counts[i][1]
        self.n_pairs = n_pairs

    def pair_index(self, img, light, exp):
        """(image, light, exp), 1-based as in main.lua (arrays or scalars) -> the 0-based pair index"""
        img = np.asarray(img, np.int64)
        return self.first[img] + (np.asarray(light) - 2) * self.n_exp[img] + np.asarray(exp) - 1

    def check_fits(self, free):
        if self.nbytes > free:
            raise MemoryError("%s: the training planes need %d bytes on the device, %d are free" % (self.dir, self.nbytes,
                                                                                                      free))

    def upload(self, device):
        """-> [(x0, x1)] CUDA (H, W) planes in pair order, views of one device tensor per group file"""
        import torch

        dev = torch.device("cuda", device)
        self.check_fits(torch.cuda.mem_get_info(dev)[0])
        planes = []
        for _, _, p, dims in self.groups:
            g = torch.from_numpy(np.ascontiguousarray(dataio.fromfile(p), np.float32).reshape(dims)).to(dev)
            planes += [(g[e, 0, 0], g[e, 1, 0]) for e in range(dims[0])]
        return planes

    def warps(self, stream, o, rows, ws):
        """main.lua:791-846 for the samples of nnz `rows` -> WARP_DTYPE records naming pairs"""
        img = rows[:, 0].astype(np.int64)
        p, light, exp, light_, exp_ = draw_params_mb(stream, o, self.n_light[img], self.n_exp[img])
        return make_warps(p, rows, ws, pairs=(self.pair_index(img, light, exp), self.pair_index(img, light_, exp_)))


def net_path(data_root, dataset, args, arch="fast"):
    return os.path.join(data_root, "net", "net_%s.t7" % cmd_str(dataset, args, arch))


# Checkpoints (-checkpoint_steps / -stop_after / -resume): <net file without .t7>.state.npz holds the position, the
# parameters and momenta, the epoch's losses so far and the random stream, with a fingerprint of the run it belongs to.
CHECKPOINT_FORMAT = 1
EX_TEMPFAIL = 75                     # the exit status of a run stopped by -stop_after: "try again"


class CheckpointError(ValueError):
    """a checkpoint that cannot be resumed, or checkpoint options that cannot be honoured"""


class Stopped(Exception):
    """-stop_after ran out: the state is in `path`, to continue at (`epoch`, `step`)"""

    def __init__(self, path, epoch, step):
        super().__init__("stopped: checkpoint %s at epoch %d, step %d" % (path, epoch, step))
        self.path, self.epoch, self.step = path, epoch, step


def checkpoint_path(data_root, dataset, args, arch="fast"):
    return net_path(data_root, dataset, args, arch)[:-len(".t7")] + ".state.npz"


def check_checkpoint_options(checkpoint_steps=None, stop_after=None):
    if checkpoint_steps is not None and (checkpoint_steps < 1 or checkpoint_steps % CHUNK):
        raise CheckpointError("-checkpoint_steps %s: must be a positive multiple of the chunk size %d (checkpoints are "
                              "taken at chunk boundaries)" % (checkpoint_steps, CHUNK))
    if stop_after is not None and not stop_after > 0:
        raise CheckpointError("-stop_after %s: must be a positive number of seconds" % (stop_after,))


def fingerprint(dataset, action, o, seed, cmd, nnz, shapes, rect=None):
    """what a checkpoint must match to be resumed: the run's options and the training set's nnz rows (a SHA-256 of their
    bytes) and file shapes `shapes` [(name, shape)].  The pixels are not hashed."""
    import hashlib

    nnz = np.ascontiguousarray(nnz, np.float32)
    return dict(dataset=dataset, arch=arch_of(o), action=action, o=dict(o), seed=int(seed), rect=rect, cmd_str=cmd,
                nnz_rows=len(nnz), nnz_sha256=hashlib.sha256(nnz.tobytes()).hexdigest(),
                shapes=[[name, [int(v) for v in shape]] for name, shape in shapes])


def _library_version():
    from . import adcensus

    return adcensus.version()


def save_checkpoint(path, fp, epoch, step, lr, elapsed, params, momenta, losses, stream):
    """write the state to a temporary name, fsync it, then replace `path`: a stop during the write keeps the old file"""
    import json

    key, pos, carry = stream.state()
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        np.savez(f, format=np.int64(CHECKPOINT_FORMAT), version=np.array(_library_version()),
                 fingerprint=np.array(json.dumps(fp, sort_keys=True)), epoch=np.int64(epoch), step=np.int64(step),
                 lr=np.float64(lr), elapsed=np.float64(elapsed), params=np.asarray(params, np.float32),
                 momenta=np.asarray(momenta, np.float32), losses=np.asarray(losses, np.float32), mt_key=key,
                 mt_pos=np.int64(pos), carry=carry)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)
    try:                                                                         # make the rename itself durable
        dfd = os.open(os.path.dirname(os.path.abspath(path)), os.O_RDONLY)
        try:
            os.fsync(dfd)
        finally:
            os.close(dfd)
    except OSError:
        pass


def load_checkpoint(path, fp):
    """-> dict of the saved state; refuses a file that is truncated, of another format or of another run (naming the
    field of the fingerprint that differs)"""
    import json

    try:
        with np.load(path, allow_pickle=False) as z:
            st = {k: z[k] for k in z.files}
    except Exception as e:  # noqa: BLE001 -- a truncated zip fails in several ways
        raise CheckpointError("%s: not a readable checkpoint (truncated?): %s" % (path, e))
    want = ("format", "version", "fingerprint", "epoch", "step", "lr", "elapsed", "params", "momenta", "losses",
            "mt_key", "mt_pos", "carry")
    if "format" not in st or int(st["format"]) != CHECKPOINT_FORMAT:
        raise CheckpointError("%s: checkpoint format %s, this library reads format %d"
                              % (path, st["format"] if "format" in st else "missing", CHECKPOINT_FORMAT))
    missing = [k for k in want if k not in st]
    if missing:
        raise CheckpointError("%s: checkpoint lacks %s (truncated?)" % (path, ", ".join(missing)))
    got, fp = json.loads(str(st["fingerprint"])), json.loads(json.dumps(fp, sort_keys=True))
    for k in sorted(set(got) | set(fp)):
        if k == "o":
            for name in sorted(set(got.get(k, {})) | set(fp[k])):
                if got.get(k, {}).get(name) != fp[k].get(name):
                    raise CheckpointError("%s: belongs to another run: option -%s is %s there, %s here"
                                          % (path, name, got.get(k, {}).get(name), fp[k].get(name)))
        elif got.get(k) != fp.get(k):
            raise CheckpointError("%s: belongs to another run: %s is %s there, %s here" % (path, k, got.get(k), fp.get(k)))
    out = {k: st[k] for k in ("params", "momenta", "losses", "mt_key", "carry")}
    out.update(epoch=int(st["epoch"]), step=int(st["step"]), lr=float(st["lr"]), elapsed=float(st["elapsed"]),
               mt_pos=int(st["mt_pos"]), version=str(st["version"]))
    return out


class Checkpoints:
    """Where and when :func:`fit` writes the state: `steps` (within an epoch, a multiple of CHUNK, or None) and at every
    epoch's end if `steps` is set; `stop_after` seconds of this process's training (or None), after which it writes the
    state and raises :class:`Stopped` at the next chunk boundary.  `clock` is the clock of `stop_after`."""

    def __init__(self, path, fp, steps=None, stop_after=None, clock=time.monotonic):
        check_checkpoint_options(steps, stop_after)
        self.path, self.fp, self.steps, self.stop_after, self.clock = path, fp, steps, stop_after, clock
        self.t_begin = None

    def start(self):
        self.t_begin = self.clock()

    def stop_due(self):
        return self.stop_after is not None and self.clock() - self.t_begin >= self.stop_after

    def due(self, step):
        return self.steps is not None and step % self.steps == 0

    def save(self, tr, stream, epoch, step, lr, elapsed, losses):
        params, momenta = tr.state()
        save_checkpoint(self.path, self.fp, epoch, step, lr, elapsed, params, momenta, losses, stream)


def _agree(comm, flag, device):
    """rank 0's `flag` on every rank of `comm` (a stop is decided by rank 0's clock alone)"""
    import torch

    if comm is None or comm.world == 1:
        return flag
    t = torch.tensor([int(flag)], dtype=torch.int32, device=device)
    comm.exchange({p: t for p in range(1, comm.world)} if comm.rank == 0 else {}, {} if comm.rank == 0 else {0: t})
    return bool(t.item())


def fit(tr, nnz, perm, build, o, stream, epochs=EPOCHS, log=print, ckpt=None, start=None, comm=None):
    """main.lua:779-881: the epochs of chunks from (start["epoch"], start["step"]) (or from the beginning), driving `tr`
    (a :class:`Trainer`) with the records `build`(n steps, nnz rows) makes from `stream`; `log` receives the epoch lines.
    With `ckpt` (:class:`Checkpoints`) the state is written at chunk boundaries and at the end of each epoch.  With `comm`
    (a data-parallel run: every rank calls fit with the same arguments) only rank 0 logs and writes the state, and rank 0's
    clock decides a stop for every rank."""
    if comm is not None and comm.rank != 0:
        log = lambda line: None                                                 # noqa: E731
    writer = comm is None or comm.rank == 0
    agree = (lambda flag: flag) if comm is None else (lambda flag: _agree(comm, flag, tr.dev))
    h = o["bs"] // 2
    nsteps = steps_per_epoch(len(nnz), o["bs"])
    epoch0, step0 = (start["epoch"], start["step"]) if start else (1, 0)
    t0 = time.time() - (start["elapsed"] if start else 0.0)
    if ckpt:
        ckpt.start()
    for epoch in range(epoch0, epochs + 1):
        lr = lr_at(o["lr"], epoch)
        tr.reset_losses()
        first = step0 if epoch == epoch0 else 0
        done = np.asarray(start["losses"], np.float32) if start and epoch == epoch0 else np.zeros(0, np.float32)
        for s0 in range(first, nsteps, CHUNK):
            n = min(CHUNK, nsteps - s0)
            rows = nnz[perm[s0 * h:(s0 + n) * h] - 1]                          # perm[t + i - 1], :820
            tr.run_chunk(build(n, rows), lr)
            s1 = s0 + n
            if ckpt and s1 < nsteps:
                stop = agree(ckpt.stop_due())
                if (stop or ckpt.due(s1)) and writer:
                    ckpt.save(tr, stream, epoch, s1, lr, time.time() - t0, np.concatenate([done, tr.losses(s1 - first)]))
                if stop:
                    raise Stopped(ckpt.path, epoch, s1)
        losses = np.concatenate([done, tr.losses(nsteps - first)]).astype(np.float64)
        ok = (losses >= 0) & (losses < 100)                                      # :861-866
        for v in losses[~ok]:
            log("WARNING! err=%f" % v)
        err = np.cumsum(losses[ok])[-1] / ok.sum() if ok.any() else float("nan")
        log(epoch_line(epoch, err, lr, time.time() - t0))
        if ckpt:
            stop = epoch < epochs and agree(ckpt.stop_due())
            if (stop or ckpt.steps is not None) and writer:
                ckpt.save(tr, stream, epoch + 1, 0, lr_at(o["lr"], epoch + 1), time.time() - t0, np.zeros(0, np.float32))
            if stop:
                raise Stopped(ckpt.path, epoch + 1, 0)


def train(dataset, action, o, args=(), data_root=".", seed=42, device=0, out="out", stereo=None, log=print, epochs=EPOCHS,
          rect="imperfect", checkpoint_steps=None, stop_after=None, resume=False, comm=None):
    """main.lua:602-890 for arch 'fast' or 'slow' (as `o` was made): returns the saved net's file name.  `args` are main.lua's arguments after
    dataset and arch (for the file name), `stereo` the stereo method's overrides for the evaluation that follows;
    `log` receives the printed lines.  For dataset mb the set is data.mb.<rect>_gray (see :class:`MbTrainSet`).

    Checkpoints (:func:`checkpoint_path`, next to the net): `checkpoint_steps` K writes the state every K steps of an
    epoch and at each epoch's end; `stop_after` S writes it at the first chunk boundary after S seconds and raises
    :class:`Stopped`; `resume` continues from the checkpoint if there is one.  A resumed run gives the bits of an
    uninterrupted one; the checkpoint is deleted once the net file is written.

    With `comm` (a rowband.Comm of world > 1 ranks, each calling train with the same arguments and its own `device`) the
    batches are shared out as :class:`Trainer` says and the run gives the one-GPU bits; only rank 0 prints, writes the
    checkpoints and the net and runs the evaluation.  The checkpoint does not record the number of ranks: a state written
    by R ranks resumes on any other count."""
    import torch

    from . import t7

    if action not in ("train_tr", "train_all"):
        raise ValueError("action must be train_tr or train_all, got %r" % (action,))
    check(o)
    check_checkpoint_options(checkpoint_steps, stop_after)
    rank, world = (comm.rank, comm.world) if comm is not None else (0, 1)
    check_world(world, o)
    if world == 1:
        comm = None
    arch = arch_of(o)
    fname = net_path(data_root, dataset, args, arch)
    if os.path.exists(fname):
        raise FileExistsError("%s already exists; remove it first" % fname)
    if action == "train_all" and os.path.isdir(out) and any(f != ".empty" for f in os.listdir(out)):
        raise ValueError("submit: output directory %s is not empty" % out)
    data = evaluate.load_data(dataset, data_root, rect)
    mb = MbTrainSet(data_root, rect, action) if dataset == "mb" else None
    nnz = mb.nnz if mb else load_nnz(data, action, data_root)
    ckpt = start = None
    if checkpoint_steps is not None or stop_after is not None or resume:
        shapes = [(os.path.basename(p), dims) for _, _, p, dims in mb.groups] if mb else \
            [("x0.bin", data.X0.shape), ("x1.bin", data.X1.shape)]
        fp = fingerprint(dataset, action, o, seed, cmd_str(dataset, args, arch), nnz, shapes, rect if mb else None)
        ckpt = Checkpoints(checkpoint_path(data_root, dataset, args, arch), fp, checkpoint_steps, stop_after)
        if resume and os.path.exists(ckpt.path):
            start = load_checkpoint(ckpt.path, fp)
        os.makedirs(os.path.dirname(ckpt.path), exist_ok=True)
    planes = mb.upload(device) if mb else None
    stream = Stream(seed)                                                        # main.lua:340
    perm = randperm(stream, len(nnz))                                            # :657
    tower, head = init_net(stream, o)                                            # :663-736
    if start:                                                                    # the initial weights are replaced
        stream.restore(start["mt_key"], start["mt_pos"], start["carry"])
    if rank != 0:
        log = lambda line: None                                                 # noqa: E731
    for line in net_lines(o):
        log(line)
    h = o["bs"] // 2
    nsteps = steps_per_epoch(len(nnz), o["bs"])
    dev = torch.device("cuda", device)
    with torch.cuda.device(dev):
        if mb:
            tr = Trainer(o, chunk=CHUNK, loss_cap=max(nsteps, 1), device=device, planes=planes, rank=rank, world=world,
                         comm=comm)
            build = lambda n, rows: mb.warps(stream, o, rows, tr.ws)                                      # :791-846
        else:
            X0 = torch.from_numpy(np.ascontiguousarray(data.X0, np.float32)).to(dev)
            X1 = torch.from_numpy(np.ascontiguousarray(data.X1, np.float32)).to(dev)
            tr = Trainer(o, X0, X1, chunk=CHUNK, loss_cap=max(nsteps, 1), device=device, rank=rank, world=world, comm=comm)
            build = lambda n, rows: make_warps(draw_params(stream, o, n * h), rows, tr.ws)
        try:
            if start:
                tr.load_state(start["params"], start["momenta"])
            else:
                tr.set_layers(tower, head)
            fit(tr, nnz, perm, build, o, stream, epochs=epochs, log=log, ckpt=ckpt, start=start, comm=comm)
            tower, head = tr.net()
        finally:
            tr.close()
    if mb:                                                                       # the training planes are not needed now
        del planes, tr
        torch.cuda.empty_cache()
    if rank != 0:                                                                # rank 0 writes and evaluates the net
        return fname
    os.makedirs(os.path.dirname(fname), exist_ok=True)
    extra = dict(rect=rect, color="gray") if mb else {}
    t7.save_net(fname, tower, head, opt=dict(o, a=action, seed=seed, gpu=device + 1, **extra))   # :883, save_net(0)
    if ckpt and os.path.exists(ckpt.path):                                       # the net file holds the result now
        os.remove(ckpt.path)
    ev = evaluate.Evaluator(dataset, arch, net_fname=fname, device=device, **(stereo or {}))
    try:
        if action == "train_tr":                                                 # :884-888
            ev.test("test_te", data_root=data_root, data=data)
        else:
            ev.submit(data_root=data_root, out=out, data=data)
    finally:
        ev.close()
    return fname
