"""GPU: the label cleaning kernels and the training-sample lists of csrc/preprocess.cu, and preprocess_kitti end to end.

Every kernel output must equal, bit for bit, the reference's own kernels (oracle/_ref/libadcensus_ref.so through the shim,
where it has been built) and the stored fixtures of tests/golden/preprocess; the fused clean + compaction must give nnz_tr /
nnz_te equal row for row to remove_nonvisible -> remove_occluded -> remove_white -> make_dataset2 run through the shim.
End to end, tools/preprocess_kitti.py on a full-size synthetic raw tree must write what the CPU restatement computes, and
main.lua's test_te must run on the result."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, evaluate, preprocess, synth  # noqa: E402
from oracle import make_preprocess_golden as mpg  # noqa: E402
from oracle import preprocess as opp  # noqa: E402
from oracle import refdriver  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "preprocess")


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ours(y, x0, is_te):
    """the same outputs as mpg.reference_outputs, from this library"""
    res = {}
    for name, ops in (("nonvisible", ("nv",)), ("occluded", ("occ",)), ("nonvisible_occluded", ("nv", "occ")),
                      ("white", ("w",))):
        t = cu(y)
        for op in ops:
            if op == "nv":
                adcensus.remove_nonvisible(t)
            elif op == "occ":
                adcensus.remove_occluded(t)
            else:
                adcensus.remove_white(cu(x0), t)
        res[name] = t.cpu().numpy()
    disp = cu(y)
    nnz_tr, nnz_te = preprocess.kitti_nnz(disp, cu(x0), is_te.astype(bool))
    res["nnz_tr"], res["nnz_te"] = nnz_tr.cpu().numpy(), nnz_te.cpu().numpy()
    assert np.array_equal(disp.cpu().numpy(), y), "kitti_nnz modified its input"
    return res


def assert_same(got, want, what):
    for k in want:
        assert got[k].shape == want[k].shape, "%s %s: shape %s, want %s" % (what, k, got[k].shape, want[k].shape)
        bad = np.argwhere(got[k] != want[k])
        assert not len(bad), "%s %s: %d entries differ, first at %s (%r, want %r)" % (
            what, k, len(bad), bad[0], got[k][tuple(bad[0])], want[k][tuple(bad[0])])


@pytest.fixture(scope="module")
def shim():
    if not os.path.exists(refdriver.REF_LIB):
        pytest.skip("oracle/_ref/libadcensus_ref.so has not been built (needs the reference tree)")
    return refdriver.ShimLibrary(refdriver.REF_LIB)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "*.npz"))), ids=os.path.basename)
def test_kernels_equal_the_reference_fixtures(path):
    g = np.load(path)
    want = {k: g[k] for k in ("nonvisible", "occluded", "nonvisible_occluded", "white", "nnz_tr", "nnz_te")}
    assert_same(ours(g["y"], g["x0"], g["is_te"]), want, os.path.basename(path))


def stack(seed, n, H, W, dmax=200):
    rng = np.random.default_rng(seed)
    y = mpg.png16(rng, (n, 1, H, W), dmax=dmax)
    y[:, :, ::7] = np.floor(y[:, :, ::7] * 4) / 4                 # quarter steps: exact ties
    y[0, 0, 1] = 0                                                # a row with no valid pixel
    x0 = rng.standard_normal(y.shape).astype(np.float32)
    x0[rng.random(y.shape) < 0.01] = 255
    is_te = (rng.random(n) < 0.3).astype(np.int32)
    is_te[0] = 1
    if n > 1:
        is_te[-1] = 0
    return y, x0, is_te


@pytest.mark.parametrize("n,H,W", [(1, 350, 1242), (45, 350, 1242), (3, 350, 1241), (2, 17, 333), (4, 9, 1),
                                   (1, 5, 4099)])
def test_kernels_and_lists_equal_the_live_reference(shim, n, H, W):
    y, x0, is_te = stack(n * 1000 + W, n, H, W)
    want = mpg.reference_outputs(shim, y, x0, is_te)
    got = ours(y, x0, is_te)
    assert_same(got, want, "%dx%dx%d" % (n, H, W))
    if n * H * W <= 2 * 350 * 1242:                             # and the CPU restatement agrees with both
        cpu = dict(nonvisible=opp.remove_nonvisible(y), occluded=opp.remove_occluded(y), white=opp.remove_white(x0, y))
        assert_same(got, cpu, "cpu %dx%dx%d" % (n, H, W))
    if n == 45:
        assert len(got["nnz_tr"]) > 10 ** 6 and len(got["nnz_te"]) > 10 ** 5


def test_side_stream_and_second_call_agree():
    y, x0, is_te = stack(5, 6, 64, 300)
    want = ours(y, x0, is_te)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = ours(y, x0, is_te)
    assert_same(got, want, "side stream")


def test_bad_arguments():
    t = torch.zeros((1, 1, 4, 40000), device="cuda")
    with pytest.raises(adcensus.AdcensusError, match="size limit"):
        adcensus.remove_occluded(t)
    with pytest.raises(adcensus.AdcensusError, match="size limit"):
        preprocess.kitti_nnz(t, t, [False])
    with pytest.raises(adcensus.AdcensusError, match="te flags"):
        preprocess.kitti_nnz(t[..., :8].contiguous(), t[..., :8].contiguous(), [False, True])
    with pytest.raises(adcensus.AdcensusError, match="elements"):
        adcensus.remove_white(torch.zeros(3, device="cuda"), torch.zeros(4, device="cuda"))


@pytest.fixture(scope="module")
def e2e_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti_raw"))
    synth.write_kitti_raw(root, "kitti", n_tr=41, n_te=2, H=375, widths=(1242, 1241, 1224), seed=21)
    synth.write_kitti_raw(root, "kitti2015", n_tr=41, n_te=2, H=376, widths=(1242, 1238), seed=22)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "preprocess_kitti.py"), "both", "-data_root", root,
                        "-gpu", "1"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr
    return root, r.stdout


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015"])
def test_tool_end_to_end_equals_the_cpu_restatement_and_feeds_test_te(e2e_root, dataset, capsys):
    root, out = e2e_root
    lines = out.split("\n")
    year = "dataset %d" % preprocess.LAYOUT[dataset]["year"]
    k = lines.index(year)
    assert lines[k + 1:k + 44] == [str(i) for i in range(1, 44)]
    want = opp.preprocess_kitti(root, dataset)
    d = preprocess.output_dir(root, dataset)
    for f in preprocess.OUTPUTS:
        got = dataio.fromfile(os.path.join(d, f))
        w = want[f[:-4]]
        assert got.dtype == w.dtype and got.shape == w.shape, f
        assert np.array_equal(got, w), "%s %s differs from the CPU restatement" % (dataset, f)
    assert want["x0"].shape == (43, 1, 350, 1242) and len(want["nnz_tr"]) > 10 ** 5 and len(want["nnz_te"]) > 10 ** 6
    # dispnoc keeps the maps as read: the cleaning removed entries from the lists, not from the file
    n_valid = int((want["dispnoc"] > 0.5).sum())
    assert n_valid > len(want["nnz_tr"]) + len(want["nnz_te"])
    capsys.readouterr()
    ev = evaluate.Evaluator(dataset, "census")
    try:
        res = ev.test("test_te", data_root=root)
    finally:
        ev.close()
    assert [e[0] + 1 for e in res.examples] == want["te"].tolist()
    assert all(np.isfinite(e[3]) and 0 <= e[3] <= 1 for e in res.examples) and 0 < res.mean < 1
