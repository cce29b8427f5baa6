"""GPU: every training kernel at its tile and loop edges against float64 autograd, at the cases of tests/train_cases.py
(the four kitti / mb presets among them).  Per case, at the initial weights and again after a few run() steps: the loss,
every gradient and every intermediate the trainer exposes, each layer's tensor on its own, within 1e-4 of that tensor's
max |value|, and the momentum update bit for bit.  Also: run() reads step i's warps on step i, the fast tower the trainer
trains is the FeatureTower that tests with it, and the sampler at ws 3 and 17."""
import importlib.util
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import train  # noqa: E402
from oracle import train as ot  # noqa: E402
from oracle import train_slow as ots  # noqa: E402

_spec = importlib.util.spec_from_file_location("train_cases", os.path.join(ROOT, "tests", "train_cases.py"))
tc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(tc)

DEV = torch.device("cuda", 0)
H, W = 40, 90                    # the images the sampler reads during run()
LR = 0.003


def _trainer(c, rng, chunk=4, loss_cap=16):
    X0, X1 = (torch.from_numpy(rng.standard_normal((2, 1, H, W)).astype(np.float32)).to(DEV) for _ in range(2))
    return train.Trainer(tc.options(c), X0, X1, chunk=chunk, loss_cap=loss_cap, device=0), X0, X1


def _warps(rng, o, n, ws, stream):
    rows = np.stack([rng.integers(1, 3, n), rng.integers(0, H, n), rng.integers(0, W, n), rng.uniform(0, 60, n)],
                    1).astype(np.float32)
    return train.make_warps(train.draw_params(stream, o, n), rows, ws)


class Errors:
    """each compared tensor against float64, within BAR of its max |value|; keeps the largest relative error per kind"""

    def __init__(self, case):
        self.case, self.worst = case, {}

    def __call__(self, kind, name, got, want):
        want = np.asarray(want, np.float64)
        got = np.asarray(got, np.float64).reshape(want.shape)
        err = float(np.abs(got - want).max()) / max(float(np.abs(want).max()), 1e-30)
        self.worst[kind] = max(self.worst.get(kind, 0.0), err)
        assert err <= tc.BAR, "%s %s: %.3g of its max |value| (bar %g)" % (self.case, name, err, tc.BAR)

    def report(self):
        print("\n%s: largest relative error %s" % (self.case, ", ".join("%s %.2g" % kv for kv in sorted(self.worst.items()))))


def _layers_of(tr, v):
    """a (N, fm, s, s) per layer view of the trainer's TRAIN_TOWER or TRAIN_DZ"""
    L = tc.layout(tr.l1, tr.fm, tr.bs)
    return [v[L.aoff[k]:L.aoff[k] + L.N * tr.fm * s * s] for k, s in enumerate(L.sides)]


def _check_fast(c, tr, x, tower, err):
    loss64, grads, it = ot.step64(x.astype(np.float64), tower, c.margin, c.pow, inter=True, device=DEV)
    loss = float(tr.get(train.TRAIN_LOSS)[0])
    assert abs(loss - loss64) <= tc.BAR * max(abs(loss64), 1e-3), (loss, loss64)
    err.worst["loss"] = max(err.worst.get("loss", 0.0), abs(loss - loss64) / max(abs(loss64), 1e-3))
    for k, ((gw, gb), (ww, wb)) in enumerate(zip(tr.layers(train.TRAIN_GRADS), grads)):
        err("weight gradient", "layer %d dW" % k, gw, ww)
        err("bias gradient", "layer %d db" % k, gb, wb)
    act = _layers_of(tr, tr.get(train.TRAIN_TOWER).cpu().numpy())
    dz = _layers_of(tr, tr.get(train.TRAIN_DZ).cpu().numpy())
    for k in range(c.l1):
        z = it["z"][k]
        err("activation", "layer %d activation" % k, act[k], z if k == c.l1 - 1 else np.maximum(z, 0))
        err("dLoss/dz", "layer %d dLoss/dz" % k, dz[k], it["dz"][k])
    err("norm", "norm", tr.get(train.TRAIN_NORM).cpu().numpy(), it["norm"])
    err("normalized", "normalized", tr.get(train.TRAIN_NORMALIZED).cpu().numpy(), it["normalized"])
    err("join", "join", tr.get(train.TRAIN_JOIN).cpu().numpy(), it["join"])
    err("hinge", "hinge", tr.get(train.TRAIN_HINGE).cpu().numpy(), it["hinge"])


def _check_slow(c, tr, x, tower, head, err):
    loss64, gt, gh, _, it = ots.step64_slow(x.astype(np.float64), tower, head, inter=True, device=DEV)
    loss = float(tr.get(train.TRAIN_LOSS)[0])
    assert abs(loss - loss64) <= tc.BAR * max(abs(loss64), 1e-3), (loss, loss64)
    err.worst["loss"] = max(err.worst.get("loss", 0.0), abs(loss - loss64) / max(abs(loss64), 1e-3))
    got_t, got_h = tr.net(train.TRAIN_GRADS)
    for k, ((gw, gb), (ww, wb)) in enumerate(zip(got_t, gt)):
        err("weight gradient", "layer %d dW" % k, gw, ww)
        err("bias gradient", "layer %d db" % k, gb, wb)
    for j, ((gw, gb), (ww, wb)) in enumerate(zip(got_h, gh)):
        err("Linear weight gradient", "Linear %d dW" % j, gw, ww)
        err("Linear bias gradient", "Linear %d db" % j, gb, wb)
    act = _layers_of(tr, tr.get(train.TRAIN_TOWER).cpu().numpy())
    dz = _layers_of(tr, tr.get(train.TRAIN_DZ).cpu().numpy())
    for k in range(c.l1):
        err("activation", "layer %d activation" % k, act[k], np.maximum(it["z"][k], 0))
        err("dLoss/dz", "layer %d dLoss/dz" % k, dz[k], it["dz"][k])
    err("rows", "rows", tr.get(train.TRAIN_ROWS).cpu().numpy(), it["rows"])
    err("rows gradient", "rows gradient", tr.get(train.TRAIN_ROWS_GRAD).cpu().numpy(), it["rows_grad"])
    fc = tr.get(train.TRAIN_FC).cpu().numpy()
    n = c.bs * c.nh2
    for j in range(c.l2):
        err("Linear output", "Linear %d output" % j, fc[j * n:(j + 1) * n], np.maximum(it["fc"][j], 0))
    err("Linear output", "last Linear output", fc[c.l2 * n:], it["fc"][c.l2].reshape(-1))
    err("sigmoid", "sigmoid", tr.get(train.TRAIN_SIGMOID).cpu().numpy(), it["sigmoid"])


@pytest.mark.parametrize("c", tc.FAST_CASES + tc.SLOW_CASES, ids=tc.case_id)
def test_step_matches_float64_at_every_edge(c):
    slow = isinstance(c, tc.SlowCase)
    o = tc.options(c)
    rng = np.random.default_rng(c.l1 * 1000 + c.fm + c.bs)
    tr, _, _ = _trainer(c, rng)
    assert tr.launches_per_step == tc.launches_per_step(slow, c.l1, c.l2 if slow else 0)
    assert tr.size(train.TRAIN_PARAMS) == tc.layout(c.l1, c.fm, c.bs, *((c.l2, c.nh2, True) if slow else ())).nparam
    tr.set_layers(*tc.init_layers(c, 1))
    s = train.Stream(3)
    err = Errors(tc.case_id(c))
    for point in range(2):
        if point:                                                                # three sampler steps along a run
            tr.run(_warps(rng, o, 3 * c.bs // 2, tr.ws, s), LR)
            torch.cuda.synchronize()
        tower, head = tr.net()
        x = tc.slow_patches(c, 10 + point) if slow else tc.fast_patches(c, tower, 10 + point, device=DEV)
        p0, v0 = (tr.get(w).cpu().numpy() for w in (train.TRAIN_PARAMS, train.TRAIN_MOMENTA))
        tr.reset_losses()
        tr.step_patches(x, LR)
        torch.cuda.synchronize()
        if slow:
            _check_slow(c, tr, x, tower, head, err)
        else:
            _check_fast(c, tr, x, tower, err)
        p1, v1 = ot.update32(p0, v0, tr.get(train.TRAIN_GRADS).cpu().numpy(), o["mom"], LR)
        assert np.array_equal(tr.get(train.TRAIN_MOMENTA).cpu().numpy().view(np.int32), v1.view(np.int32)), point
        assert np.array_equal(tr.get(train.TRAIN_PARAMS).cpu().numpy().view(np.int32), p1.view(np.int32)), point
    err.report()
    tr.close()


def _case(name, arch="fast"):
    return next(c for c in (tc.FAST_CASES if arch == "fast" else tc.SLOW_CASES) if c.name == name)


@pytest.mark.parametrize("arch", ["fast", "slow"])
def test_run_reads_each_steps_warps(arch):
    """run() over k distinct steps' warps gives the bits of k x (sample_patches of step i's warps -> step_patches)"""
    c = _case("bs256") if arch == "fast" else _case("fm48", "slow")
    assert arch == "slow" or 2 * c.bs > tc.WG_NT
    o = tc.options(c)
    rng = np.random.default_rng(21)
    a, X0, X1 = _trainer(c, rng)
    b = train.Trainer(o, X0, X1, chunk=4, loss_cap=16, device=0)
    layers = tc.init_layers(c, 1)
    for tr in (a, b):
        tr.set_layers(*layers)
    k, N = 3, a.N
    w = _warps(rng, o, k * c.bs // 2, a.ws, train.Stream(4))
    a.run(w, LR)
    patches = []
    for i in range(k):
        patches.append(train.sample_patches(X0, X1, w[i * N:(i + 1) * N], a.ws))
        b.step_patches(patches[-1], LR)
    torch.cuda.synchronize()
    assert not torch.equal(patches[0], patches[1]) and not torch.equal(patches[1], patches[2])
    assert torch.equal(a.get(train.TRAIN_PATCHES), patches[-1].reshape(-1))
    for what in (train.TRAIN_PARAMS, train.TRAIN_MOMENTA, train.TRAIN_LOSS):
        x, y = a.get(what).cpu().numpy(), b.get(what).cpu().numpy()
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), what
    assert len(set(a.get(train.TRAIN_LOSS)[:k].tolist())) == k
    a.close()
    b.close()


@pytest.mark.parametrize("name", ["kitti", "ws17"])
def test_fast_train_and_test_are_tied(name):
    """the trainer's normalized tower output is FeatureTower(arch='fast')'s, at the centre of each patch"""
    from mccnn_b200 import feature_tower

    c = _case(name)
    o = tc.options(c)
    rng = np.random.default_rng(22)
    tr, _, _ = _trainer(c, rng)
    tr.set_layers(*tc.init_layers(c, 1))
    tr.run(_warps(rng, o, 3 * c.bs // 2, tr.ws, train.Stream(5)), LR)            # away from the init
    tower = tr.layers()
    x = tc.fast_patches(c, tower, 23, device=DEV)
    tr.step_patches(x, LR)
    torch.cuda.synchronize()
    got = tr.get(train.TRAIN_NORMALIZED).reshape(tr.N, c.fm)
    tr.close()
    ft = feature_tower.FeatureTower(tower, arch="fast", device=0)
    want = ft.forward(torch.from_numpy(x).to(DEV))[:, :, c.l1, c.l1]             # the centre: no padding reached
    torch.cuda.synchronize()
    ft.close()
    e = float((got - want).abs().max())
    print("\n%s: trainer vs FeatureTower, largest difference %.2g" % (name, e))
    assert e <= 1e-4, e


@pytest.mark.parametrize("ws", [3, 17])
def test_sampler_bit_exact_small_and_large_patches(ws):
    rng = np.random.default_rng(ws)
    Hs, Ws = 60, 130
    X0, X1 = (rng.standard_normal((2, 1, Hs, Ws)).astype(np.float32) for _ in range(2))
    o = train.options("kitti", hflip=1, vflip=1, trans=2.0, d_vtrans=1.0, d_rotate=3.0, d_hshear=0.2, rotate=20.0)
    n = 96
    rows = np.stack([rng.integers(1, 3, n), rng.uniform(-ws, Hs + ws, n), rng.uniform(-ws, Ws + ws, n),
                     rng.uniform(0, 40, n)], 1).astype(np.float32)
    w = train.make_warps(train.draw_params(train.Stream(ws), o, n), rows, ws)          # 384 patches
    w["m"][:16, 2] += np.float32(Ws + 2.0)                                            # wholly outside
    w["m"][16:32, 5] -= np.float32(Hs + 8.0)
    got = train.sample_patches(torch.from_numpy(X0).to(DEV), torch.from_numpy(X1).to(DEV), w, ws).cpu().numpy()
    for i, r in enumerate(w):
        src = (X1 if r["view"] else X0)[r["image"], 0]
        want = (ot.warp_affine(src, r["m"], ws) * r["contrast"] + r["brightness"]).astype(np.float32)
        assert np.array_equal(got[i].view(np.int32), want.view(np.int32)), i
