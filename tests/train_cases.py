"""The training kernels' shapes, restated from csrc/train.cu, and the cases of tests/test_gpu_train_edges.py.

A trainer's launches are fixed when it is created: ``create()`` lays out the parameter vector and the activation buffers,
sizes the fast tower's shared memory and, for arch 'slow', splits each tower weight gradient over k; ``enqueue_step`` and
``enqueue_slow`` then launch one fixed sequence per step.  Each function below restates one of those rules, next to a
comment naming the lines it restates.  tests/test_train_cases.py checks, without a GPU, that the cases reach every tile
and loop edge these rules produce and that their inputs have teeth; the GPU test runs each case against float64 autograd.
"""
from collections import namedtuple

import numpy as np

BM = BN = 64                     # gemm_kernel's tile (train.cu: BM, BN, BK, GT)
BK = 16
WG_NT = 256                      # wgrad_kernel's threads: each loops over patches n = t, t + 256, ...
SMEM_OPTIN = 232448              # an H100's opt-in shared memory per block
BAR = 1e-4                       # the GPU test's bar: 1e-4 of each compared tensor's max |value|


def div_up(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------ the restatement

Layout = namedtuple("Layout", "l1 fm ws N woff boff aoff sides nparam")


def layout(l1, fm, bs, l2=0, nh2=0, slow=False):
    """create(): L.ws = 1 + 2 l1, L.N = 2 bs; per layer k, W (fm, cin, 3, 3) at woff[k], b (fm) at boff[k], the (N, fm,
    s_k, s_k) activations at aoff[k], s_k = ws - 2 (k + 1); for 'slow' the Linear layers' W (out, in) and b (out) follow
    (fwoff / fboff, not kept here).  -> Layout, nparam the length of the parameter vector"""
    ws, N = 1 + 2 * l1, 2 * bs
    off = aoff = 0
    woff, boff, aoffs, sides = [], [], [], []
    for k in range(l1):
        cin, s = (fm if k else 1), ws - 2 * (k + 1)
        woff.append(off)
        off += fm * cin * 9
        boff.append(off)
        off += fm
        aoffs.append(aoff)
        aoff += N * fm * s * s
        sides.append(s)
    if slow:
        for j in range(l2 + 1):
            n_in, n_out = (nh2 if j else 2 * fm), (nh2 if j < l2 else 1)
            off += n_out * n_in + n_out
    return Layout(l1, fm, ws, N, woff, boff, aoffs, sides, off)


def fast_smem(l1, fm):
    """create(): bufsz = max(ws^2, fm (ws - 2k)^2 for 1 <= k < l1) floats, smem = 2 bufsz floats (tower_fwd_kernel and
    tower_bwd_kernel each hold two layers)"""
    ws = 1 + 2 * l1
    bufsz = ws * ws
    for k in range(1, l1):
        bufsz = max(bufsz, fm * (ws - 2 * k) ** 2)
    return 2 * bufsz * 4


def split_k(l1, fm, bs):
    """create(), arch 'slow': layer k's ConvWgrad has K = N s_k^2; about 256 blocks of at least 256 k each:
    tiles = div_up(fm, BM) div_up(9 cin + 1, BN), want = max(1, min(div_up(256, tiles), div_up(K, 256))),
    kchunk = div_up(div_up(K, want), BK) BK, nsplit = div_up(K, kchunk) -> [(K, kchunk, nsplit)] per layer"""
    L = layout(l1, fm, bs)
    out = []
    for k in range(l1):
        cin, s = (fm if k else 1), L.sides[k]
        K = L.N * s * s
        tiles = div_up(fm, BM) * div_up(cin * 9 + 1, BN)
        want = max(1, min(div_up(256, tiles), div_up(K, 256)))
        kchunk = div_up(div_up(K, want), BK) * BK
        out.append((K, kchunk, div_up(K, kchunk)))
    return out


# one gemm_kernel launch: the functor, the tower layer (k) or Linear (j) it serves, its M x N x K, kchunk and nsplit; the
# grid is (div_up(N, BN), div_up(M, BM), nsplit) (launch_gemm)
Gemm = namedtuple("Gemm", "op layer M N K kchunk nsplit")


def slow_gemms(l1, fm, l2, nh2, bs):
    """enqueue_slow()'s launch_gemm calls in order: ConvFwd per layer (M fm, N patches x so^2, K 9 cin); FcFwd per Linear
    (M bs, N nh2, K in); then from the last Linear down, FcBwdData (M bs, N in, K nh2) and FcWgrad (M nh2, N in + 1,
    K bs); ConvBwdData for k = l1 - 1 .. 1 (M fm, N patches x si^2, K 9 fm); ConvWgrad per layer (M fm, N 9 cin + 1,
    K patches x so^2, split over k)"""
    L = layout(l1, fm, bs)
    out = []
    for k in range(l1):
        cin = fm if k else 1
        out.append(Gemm("ConvFwd", k, fm, L.N * L.sides[k] ** 2, 9 * cin, 9 * cin, 1))
    for j in range(l2):
        n_in = nh2 if j else 2 * fm
        out.append(Gemm("FcFwd", j, bs, nh2, n_in, n_in, 1))
    for j in range(l2 - 1, -1, -1):
        n_in = nh2 if j else 2 * fm
        out.append(Gemm("FcBwdData", j, bs, n_in, nh2, nh2, 1))
        out.append(Gemm("FcWgrad", j, nh2, n_in + 1, bs, bs, 1))
    for k in range(l1 - 1, 0, -1):
        si = L.sides[k] + 2
        out.append(Gemm("ConvBwdData", k, fm, L.N * si * si, 9 * fm, 9 * fm, 1))
    for k, (K, kchunk, nsplit) in enumerate(split_k(l1, fm, bs)):
        cin = fm if k else 1
        out.append(Gemm("ConvWgrad", k, fm, 9 * cin + 1, K, kchunk, nsplit))
    return out


def launches_per_step(slow, l1, l2=0):
    """mccnn_trainer_launches_per_step: 'slow' 3 + 3 l1 + 3 l2 (the sampler, l1 + 2 l2 + (l1 - 1) + l1 GEMMs,
    slow_head_kernel, wgrad_reduce_kernel, update_kernel); 'fast' 5 + l1 (the sampler, tower_fwd, head, tower_bwd, one
    wgrad_kernel per layer, update)"""
    return 3 + 3 * l1 + 3 * l2 if slow else 5 + l1


# ------------------------------------------------------------------------------------------------------------ the cases

FastCase = namedtuple("FastCase", "name l1 fm bs pow margin")
SlowCase = namedtuple("SlowCase", "name l1 fm l2 nh2 bs")


def _presets():
    from mccnn_b200 import train

    out = []
    for ds in ("kitti", "mb"):
        f, s = train.options(ds, "fast"), train.options(ds, "slow")
        out.append(FastCase(ds, f["l1"], f["fm"], f["bs"], f["pow"], f["m"]))
        out.append(SlowCase(ds, s["l1"], s["fm"], s["l2"], s["nh2"], s["bs"]))
    return out


_P = _presets()
FAST_CASES = [c for c in _P if isinstance(c, FastCase)] + [
    FastCase("ws3", 1, 16, 2, 1, 0.2),               # no tower_bwd layer, one sample, 64 head threads
    FastCase("ws17", 8, 128, 130, 2, 0.2),           # the largest smem; N = 260 > 256 with a remainder; 512 head threads
    FastCase("bs256", 2, 48, 256, 1, 0.5),           # N = 512: two patches per wgrad thread, no remainder
    FastCase("fm96", 3, 96, 24, 2, 0.3),             # fm % 64 = 32
]
SLOW_CASES = [c for c in _P if isinstance(c, SlowCase)] + [
    SlowCase("ws3", 1, 16, 1, 128, 2),               # bs = 2, nsplit 1 everywhere
    SlowCase("ws17", 8, 128, 2, 256, 66),            # the bias-only last ConvWgrad tile; bs % 64 = 2
    SlowCase("fm48", 3, 48, 4, 256, 126),
    SlowCase("fm80", 2, 80, 3, 128, 40),             # ConvWgrad N = 721, FcWgrad N = 161: N % 64 = 17 and 33
    SlowCase("fm96", 6, 96, 2, 384, 20),             # fm % 64 = 32
]


def case_id(c):
    if isinstance(c, FastCase):
        return "fast_%s_l1%d_fm%d_bs%d_pow%d" % (c.name, c.l1, c.fm, c.bs, c.pow)
    return "slow_%s_l1%d_fm%d_l2%d_nh2%d_bs%d" % (c.name, c.l1, c.fm, c.l2, c.nh2, c.bs)


def options(c):
    """train.options for a case (the kitti augmentation; the net options of the case)"""
    from mccnn_b200 import train

    if isinstance(c, FastCase):
        return train.options("kitti", "fast", l1=c.l1, fm=c.fm, bs=c.bs, pow=c.pow, m=c.margin)
    return train.options("kitti", "slow", l1=c.l1, fm=c.fm, l2=c.l2, nh2=c.nh2, bs=c.bs)


# ------------------------------------------------------------------------------------------------------------ the inputs

F_MIN = 1e-3                     # no sample's hinge argument f = neg - pos + m is closer to 0 than this
RELU_TIE = 1e-6                  # nor an active patch's pre-activation, relative to its layer's max |z| in that patch


def tower64(x, layers, device=None):
    """the fast tower in float64: x (n, 1, ws, ws) -> (normalized outputs (n, fm), each patch's nearest ReLU tie: the
    least min |z_k| / max |z_k| over the patch's own pre-activations of each layer k with a ReLU, inf at l1 = 1)"""
    import torch

    h = torch.as_tensor(np.asarray(x), dtype=torch.float64, device=device)
    tie = torch.full((len(h),), np.inf, dtype=torch.float64, device=device)
    for i, (w, b) in enumerate(layers):
        h = torch.nn.functional.conv2d(h, torch.as_tensor(np.asarray(w, np.float64), device=device),
                                       torch.as_tensor(np.asarray(b, np.float64), device=device))
        if i < len(layers) - 1:
            a = h.abs().reshape(len(h), -1)
            tie = torch.minimum(tie, a.min(1).values / a.max(1).values.clamp_min(1e-300))
            h = torch.relu(h)
    h = h.reshape(len(h), -1)
    return (h / ((h * h).sum(1, keepdim=True) + 1e-5).sqrt()).cpu().numpy(), tie.cpu().numpy()


def _draw(rng, k, ws, scale=1.0):
    """k patches of standard normal values times a per-patch scale, log-uniform in [1, 64], times `scale`"""
    s = 2 ** rng.uniform(0, 6, (k, 1, 1, 1)) * scale
    return (rng.standard_normal((k, 1, ws, ws)) * s).astype(np.float32)


def fast_patches(c, layers, seed, device=None):
    """(2 bs, 1, ws, ws) float32 patches for a fast case: sample i is patches 4i .. 4i + 3 (left, positive, left, negative).

    * Every third sample but the last has its positive patch a copy of its left patch, so its pos is near 1 and, once the
      negative patch's features are far enough from the left ones, its hinge is made inactive (f < 0): with 4 or more
      samples that is at least a quarter of them.
    * The last sample is made active, so that the patches past wgrad_kernel's first 256 (the last sample's, when
      N % 256 = 4) carry a gradient; a batch of one sample is that sample alone.
    * No sample's |f| is below F_MIN under `layers` in float64, and no active sample has a pre-activation within
      RELU_TIE of 0, relative to that layer's max |z| in the same patch: otherwise fp32 and float64 may take different
      branches of Margin2 or of a ReLU.
    * Each patch has its own scale, log-uniform in [1, 64]: a deep tower's features of unit-scale patches all point about
      the same way (join > 0.998 at l1 = 8), so the hinge gradients of a sample's four patches nearly cancel and the last
      layer's gradients are sums that cancel to a few thousandths of their terms.  Only the weights, not the biases, tell
      inputs of different scales apart.

    A sample that misses any of these is drawn again (an inactive one: a new negative patch, of a larger scale each
    round)."""
    rng = np.random.default_rng(seed)
    ws, n = 1 + 2 * c.l1, c.bs // 2
    left, pos, neg = (_draw(rng, n, ws) for _ in range(3))
    copy = (np.arange(n) % 3 == 0) & (np.arange(n) < n - 1)
    last = np.arange(n) == n - 1
    pos[copy] = left[copy]
    redo = np.ones(n, bool)
    for r in range(1, 61):
        idx = np.flatnonzero(redo)
        (fl, tl), (fp, tp), (fn, tn) = (tower64(v[idx], layers, device) for v in (left, pos, neg))
        f = (fl * fn).sum(1) - (fl * fp).sum(1) + c.margin
        bad = (np.abs(f) < F_MIN) | (copy[idx] & (f >= 0)) | (last[idx] & (f <= 0)) | \
            ((f > 0) & (np.minimum(np.minimum(tl, tp), tn) < RELU_TIE))
        redo[:] = False
        redo[idx[bad]] = True
        if not redo.any():
            break
        inactive, active = redo & copy, redo & ~copy
        neg[inactive] = _draw(rng, int(inactive.sum()), ws, 2 ** (r / 2))
        for v in (left, pos, neg):
            v[active] = _draw(rng, int(active.sum()), ws)
    assert not redo.any(), "no patches met the inputs' conditions"
    return np.stack([left, pos, left, neg], 1).reshape(4 * n, 1, ws, ws)


def slow_patches(c, seed):
    rng = np.random.default_rng(seed)
    ws = 1 + 2 * c.l1
    return rng.standard_normal((2 * c.bs, 1, ws, ws)).astype(np.float32)


def init_layers(c, seed):
    """the reset() draws of the case's net -> (tower, head); head None for 'fast'"""
    from mccnn_b200 import train

    return train.init_net(train.Stream(seed), options(c))
