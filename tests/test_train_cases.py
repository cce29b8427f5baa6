"""CPU: the cases of tests/test_gpu_train_edges.py reach every tile and loop edge of the training kernels, and their inputs
have teeth.  The edges come from tests/train_cases.py's restatement of csrc/train.cu's create() and enqueue_slow(); the
teeth are computed in float64, in the style of test_kernel_mistakes.py: each mistake a training kernel could carry is made
in a hand-written float64 restatement of the step's backward pass (checked first against autograd), and on every case where
it applies it moves a quantity the GPU test compares by more than ten times that test's bar.  Nothing runs on a GPU."""
import importlib.util
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("train_cases", os.path.join(ROOT, "tests", "train_cases.py"))
tc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(tc)

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import train  # noqa: E402
from oracle import train as ot  # noqa: E402
from oracle import train_slow as ots  # noqa: E402

# ------------------------------------------------------------------------------------------------------------ the rules

@pytest.mark.parametrize("c", tc.FAST_CASES + tc.SLOW_CASES, ids=tc.case_id)
def test_layout_is_the_parameter_vector(c):
    """the restated offsets are those train.py's flatten / unflatten use, and the options pass train.check"""
    o = tc.options(c)
    slow = isinstance(c, tc.SlowCase)
    L = tc.layout(c.l1, c.fm, c.bs, *((c.l2, c.nh2, True) if slow else ()))
    tower, head = tc.init_layers(c, 0)
    v = train.flatten(list(tower) + list(head or []))
    assert L.nparam == len(v) and L.ws == 1 + 2 * c.l1 and L.N == 2 * c.bs
    for k, (w, b) in enumerate(tower):
        assert np.array_equal(v[L.woff[k]:L.woff[k] + w.size], w.reshape(-1))
        assert np.array_equal(v[L.boff[k]:L.boff[k] + b.size], b)
    assert L.aoff[-1] + L.N * c.fm == sum(L.N * c.fm * s * s for s in L.sides) and L.sides[-1] == 1
    assert o["l1"] == c.l1 and o["fm"] == c.fm and o["bs"] == c.bs


def test_split_and_launch_rules():
    for c in tc.SLOW_CASES:
        for K, kchunk, nsplit in tc.split_k(c.l1, c.fm, c.bs):
            assert kchunk % tc.BK == 0 and (nsplit - 1) * kchunk < K <= nsplit * kchunk
        gemms = tc.slow_gemms(c.l1, c.fm, c.l2, c.nh2, c.bs)
        # the GEMMs plus the sampler, slow_head_kernel, wgrad_reduce_kernel and update_kernel
        assert len(gemms) + 4 == tc.launches_per_step(True, c.l1, c.l2)
    assert tc.launches_per_step(False, 4) == 9 and tc.launches_per_step(True, 4, 4) == 27    # DESIGN.md §12, §13
    assert tc.fast_smem(4, 64) == 2 * 64 * 49 * 4                                              # 25 KB at the presets


def test_presets_are_verbatim():
    for ds in ("kitti", "mb"):
        f, s = train.options(ds, "fast"), train.options(ds, "slow")
        assert tc.FastCase(ds, f["l1"], f["fm"], f["bs"], f["pow"], f["m"]) in tc.FAST_CASES
        assert tc.SlowCase(ds, s["l1"], s["fm"], s["l2"], s["nh2"], s["bs"]) in tc.SLOW_CASES
    assert {(c.l1, c.fm) for c in tc.FAST_CASES if c.name == "mb"} == {(5, 64)}
    assert {(c.l1, c.l2) for c in tc.SLOW_CASES if c.name == "mb"} == {(5, 3)}


# ------------------------------------------------------------------------------------------------------------- coverage

def test_fast_cases_reach_every_edge():
    cs = tc.FAST_CASES
    assert {c.fm % 64 for c in cs} == {0, 16, 32, 48}
    assert 2 in {c.bs for c in cs} and {0, 2} <= {c.bs % 64 for c in cs}
    Ns = [2 * c.bs for c in cs]
    assert any(N < tc.WG_NT for N in Ns) and tc.WG_NT in Ns and any(N > tc.WG_NT and N % tc.WG_NT for N in Ns)
    assert any(N > tc.WG_NT and N % tc.WG_NT == 0 for N in Ns)                  # more than one full loop
    assert {1, 8} <= {c.l1 for c in cs} and {c.pow for c in cs} == {1, 2}
    assert {4 * 16, 4 * 128} <= {4 * c.fm for c in cs}                          # head_kernel's fewest and most threads
    # the largest shared memory train.check admits (l1 8, fm 128) is a case, and fits an H100's opt-in limit
    admitted = max(tc.fast_smem(l1, fm) for l1 in range(1, 9) for fm in range(16, 129, 16))
    assert admitted == tc.fast_smem(8, 128) == 230400 <= tc.SMEM_OPTIN
    assert max(tc.fast_smem(c.l1, c.fm) for c in cs) == admitted


def test_slow_cases_reach_every_edge():
    cs = tc.SLOW_CASES
    assert {c.fm % 64 for c in cs} == {0, 16, 32, 48}
    assert 2 in {c.bs for c in cs} and {0, 2} <= {c.bs % 64 for c in cs}
    assert {1, 8} <= {c.l1 for c in cs}
    assert {c.l2 for c in cs} == {1, 2, 3, 4} and {c.nh2 for c in cs} == {128, 256, 384}
    assert any(c.l2 >= 2 for c in cs)                                           # an nh2 x nh2 Linear
    g = [x for c in cs for x in tc.slow_gemms(c.l1, c.fm, c.l2, c.nh2, c.bs)]
    conv_wgrad = [x for x in g if x.op == "ConvWgrad"]
    assert any(x.N % tc.BN == 1 and x.N > 1 for x in conv_wgrad)               # a last tile holding only the bias column
    assert {x.N % tc.BN for x in g if x.op == "FcWgrad"} == {1, 33}
    assert {x.M % tc.BM for x in g if x.op == "ConvFwd"} == {0, 16, 32, 48}     # M remainders, fm % 64
    assert {0, 2} <= {x.M % tc.BM for x in g if x.op == "FcFwd"}                 # bs % 64
    assert all(x.K == 9 < tc.BK for x in g if x.op == "ConvFwd" and x.layer == 0)
    assert any(x.nsplit == 1 for x in conv_wgrad)
    assert any(x.nsplit > 1 and x.K % x.kchunk for x in conv_wgrad)             # a partial last chunk
    assert any(x.nsplit > 1 and x.K % x.kchunk == 0 for x in conv_wgrad)


# ----------------------------------------------------------------------------------------------------------- the inputs

@pytest.mark.parametrize("c", tc.FAST_CASES, ids=tc.case_id)
def test_fast_inputs_take_both_hinge_branches(c):
    tower, _ = tc.init_layers(c, 1)
    x = tc.fast_patches(c, tower, 2)
    _, _, it = ot.step64(x.astype(np.float64), tower, c.margin, c.pow, inter=True)
    f = it["join"][1::2] - it["join"][0::2] + c.margin
    assert np.abs(f).min() >= tc.F_MIN
    assert f[-1] > 0
    if len(f) >= 4:
        assert (f < 0).sum() >= len(f) / 4 and (f > 0).any()


# ------------------------------------------------------------------------------------------------------------ the teeth

def ratio(got, want):
    """|got - want| in units of the GPU test's bar, 1e-4 of max |want|"""
    return float(np.abs(got - want).max()) / (tc.BAR * max(float(np.abs(want).max()), 1e-30))


def t64(a):
    return torch.as_tensor(np.asarray(a, np.float64))


def conv_input_grad(dz, w, flip=True):
    """dLoss / d(layer input) of a valid 3x3 convolution; flip=False reads the kernel unflipped"""
    w = t64(w)
    return torch.nn.functional.conv_transpose2d(t64(dz), w if flip else w.flip(-1, -2)).numpy()


def wgrad(inp, dz):
    w = torch.nn.grad.conv2d_weight(t64(inp), (dz.shape[1], inp.shape[1], 3, 3), t64(dz)).numpy()
    return w, dz.sum((0, 2, 3))


def acts(it, relu_last):
    """each layer's stored activations, as the trainer keeps them (ReLU after every layer but, for 'fast', the last)"""
    z = it["z"]
    return [np.maximum(a, 0) if k < len(z) - 1 or relu_last else a for k, a in enumerate(z)]


def tower_mistakes(c, tower, it, grads, relu_last):
    """-> {mistake: [ratio per place it applies]} for the mistakes in the tower's backward pass"""
    L = tc.layout(c.l1, c.fm, c.bs)
    a = acts(it, relu_last)
    flat = np.concatenate([v.reshape(-1) for v in a])
    out = {"bias column dropped": [], "ConvBwdData unflipped": [], "ReLU mask of layer k": []}
    for k in range(c.l1):
        out["bias column dropped"].append(ratio(np.zeros_like(grads[k][1]), grads[k][1]))
        if k == 0:
            continue
        right = conv_input_grad(it["dz"][k], tower[k][0]) * (it["z"][k - 1] > 0)
        assert ratio(right, it["dz"][k - 1]) < 1e-6                        # the restatement is the backward pass
        wrong = conv_input_grad(it["dz"][k], tower[k][0], flip=False) * (it["z"][k - 1] > 0)
        out["ConvBwdData unflipped"].append(ratio(wrong, it["dz"][k - 1]))
        n = a[k - 1].size                                                   # act + aoff[k] read as layer k - 1's
        mask = np.zeros(n, bool)
        src = flat[L.aoff[k]:L.aoff[k] + n] > 0
        mask[:len(src)] = src
        wrong = conv_input_grad(it["dz"][k], tower[k][0]) * mask.reshape(a[k - 1].shape)
        out["ReLU mask of layer k"].append(ratio(wrong, it["dz"][k - 1]))
    return out


def fast_head64(F, c, swap=False, hinge_all=False, no_exclusion=False):
    """head_kernel in float64 with a mistake switched on: F (N, fm) the last layer's output -> (hinge, dz)"""
    nq = (F * F).sum(1, keepdims=True) + 1e-5
    nout = F / np.sqrt(nq)
    join = (nout[0::2] * nout[1::2]).sum(1)
    pos, neg = join[0::2], join[1::2]
    f = (pos - neg if swap else neg - pos) + c.margin
    act = (f > 0) | hinge_all
    h = np.maximum(f, 0) if c.pow == 1 else 0.5 * np.maximum(f, 0) ** 2
    g1 = act * (1.0 if c.pow == 1 else f)
    gj = np.stack([-g1, g1], 1).reshape(-1) / len(f)
    if swap:
        gj = -gj
    partner = nout.reshape(-1, 2, F.shape[1])[:, ::-1].reshape(F.shape)
    go = partner * np.repeat(gj, 2)[:, None]
    s = (F * go).sum(1, keepdims=True)
    if not no_exclusion:
        s = s - F * go
    return h, (nq - F * F) / nq ** 1.5 * go - s * F / nq ** 1.5


@pytest.mark.parametrize("c", tc.FAST_CASES, ids=tc.case_id)
def test_fast_mistakes_exceed_ten_bars(c):
    tower, _ = tc.init_layers(c, 1)
    x = tc.fast_patches(c, tower, 2).astype(np.float64)
    _, grads, it = ot.step64(x, tower, c.margin, c.pow, inter=True)
    F = it["z"][-1].reshape(2 * c.bs, c.fm)
    h, dz = fast_head64(F, c)
    assert ratio(h, it["hinge"]) < 1e-6 and ratio(dz, it["dz"][-1].reshape(F.shape)) < 1e-6
    m = tower_mistakes(c, tower, it, grads, False)
    m["pos / neg swapped"] = [ratio(fast_head64(F, c, swap=True)[0], it["hinge"])]
    if (it["join"][1::2] - it["join"][0::2] + c.margin < 0).any():
        m["hinge gradient on inactive samples"] = [ratio(fast_head64(F, c, hinge_all=True)[1], dz)]
    m["Normalize backward without d != c"] = [ratio(fast_head64(F, c, no_exclusion=True)[1], dz)]
    if 2 * c.bs > tc.WG_NT:                                                 # wgrad_kernel without patch N - 1
        inp = [x] + acts(it, False)[:-1]
        m["last patch dropped from wgrad"] = [max(ratio(gw - p[0], gw), ratio(gb - p[1], gb))
                                             for (gw, gb), i, d in zip(grads, inp, it["dz"])
                                             for p in [wgrad(i[-1:], d[-1:])]]
    for name, r in m.items():
        assert max(r, default=np.inf) > 10, (name, r)
    assert all(v > 10 for v in m["bias column dropped"] + m["ConvBwdData unflipped"])


def slow_head_chain(it, head, j_wrong):
    """FcBwdData from Linear l2 - 1 down to rows_grad, with Linear j_wrong's weight read transposed -> (rows_grad,
    [dLoss/d Linear j's output])"""
    l2 = len(head) - 1
    dfc = {l2 - 1: it["fc_grad"][l2 - 1]}
    for j in range(l2 - 1, 0, -1):
        w = head[j][0].astype(np.float64)
        dfc[j - 1] = (dfc[j] @ (w.T if j == j_wrong else w)) * (it["fc"][j - 1] > 0)
    return dfc[0] @ head[0][0].astype(np.float64), dfc


@pytest.mark.parametrize("c", tc.SLOW_CASES, ids=tc.case_id)
def test_slow_mistakes_exceed_ten_bars(c):
    tower, head = tc.init_layers(c, 1)
    x = tc.slow_patches(c, 2).astype(np.float64)
    _, gt, gh, _, it = ots.step64_slow(x, tower, head, inter=True)
    m = tower_mistakes(c, tower, it, gt, True)
    m["bias column dropped"] += [ratio(np.zeros_like(gb), gb) for _, gb in gh[:-1]]    # FcWgrad's
    rows_grad, _ = slow_head_chain(it, head, -1)
    assert ratio(rows_grad, it["rows_grad"]) < 1e-6
    if c.l2 >= 2:
        m["FcBwdData transposed"] = []
        for j in range(1, c.l2):
            wrong, dfc = slow_head_chain(it, head, j)
            xj = it["rows"] if j == 1 else np.maximum(it["fc"][j - 2], 0)
            m["FcBwdData transposed"].append(max(ratio(wrong, it["rows_grad"]), ratio(dfc[j - 1].T @ xj, gh[j - 1][0])))
    inp = [x] + acts(it, True)[:-1]
    chunks = []
    for (K, kchunk, nsplit), (gw, gb), i, d in zip(tc.split_k(c.l1, c.fm, c.bs), gt, inp, it["dz"]):
        if nsplit > 1:                                                      # the last k = (n, y, x) chunk dropped
            keep = (np.arange(K) >= (nsplit - 1) * kchunk).reshape(d.shape[0], 1, *d.shape[2:])
            pw, pb = wgrad(i, d * keep)
            chunks.append(max(ratio(gw - pw, gw), ratio(gb - pb, gb)))
    if chunks:
        m["last split-k chunk dropped"] = chunks
    for name, r in m.items():
        assert max(r, default=np.inf) > 10, (name, r)
    assert all(v > 10 for v in m["bias column dropped"] + m["ConvBwdData unflipped"])
