"""CPU: preprocess_kitti.lua's restatement (mccnn_b200/preprocess.py, oracle/preprocess.py) -- the cleaning rules against the
reference's own outputs, the suffix-min rule against the reference's loop, the Torch7 split, the host side of the script and
its refusals.  The GPU half (the kernels and the sample lists) is tests/test_gpu_preprocess.py."""
import glob
import importlib.util
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, preprocess, synth
from oracle import preprocess as opp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "preprocess")
SMALL = dict(height=30, width=64)


def _tool():
    spec = importlib.util.spec_from_file_location("preprocess_kitti_tool", os.path.join(ROOT, "tools", "preprocess_kitti.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def golden_cases():
    return sorted(glob.glob(os.path.join(GOLDEN, "*.npz")))


def test_fixtures_present():
    assert {os.path.basename(p) for p in golden_cases()} == {"ties_w77.npz", "random_5x6x131.npz", "wide_2x3x1242.npz"}


@pytest.mark.parametrize("path", golden_cases(), ids=os.path.basename)
def test_cpu_restatement_equals_the_reference_fixtures(path):
    g = np.load(path)
    y, x0, is_te = g["y"], g["x0"], g["is_te"]
    assert np.array_equal(opp.remove_nonvisible(y), g["nonvisible"])
    assert np.array_equal(opp.remove_occluded(y), g["occluded"])
    assert np.array_equal(opp.remove_occluded(opp.remove_nonvisible(y)), g["nonvisible_occluded"])
    assert np.array_equal(opp.remove_white(x0, y), g["white"])
    te = np.nonzero(is_te)[0] + 1
    nnz_tr, nnz_te = opp.nnz_lists(y, x0, te)
    assert np.array_equal(nnz_tr, g["nnz_tr"]) and np.array_equal(nnz_te, g["nnz_te"])


def test_fixtures_exercise_every_rule():
    """ties that must not occlude, rows with no valid pixel, 1242 columns, white pixels, both lists non-empty somewhere"""
    g = np.load(os.path.join(GOLDEN, "ties_w77.npz"))
    assert g["nonvisible_occluded"][0, 0, 0, 10] == 3.0 and g["nonvisible_occluded"][0, 0, 0, 20] == 2.5   # ties kept
    assert g["nonvisible_occluded"][0, 0, 0, 30] == 0                                                       # occluded
    assert not g["y"][0, 0, 1].any()
    w = np.load(os.path.join(GOLDEN, "wide_2x3x1242.npz"))
    assert w["y"].shape[-1] == 1242 and len(w["nnz_tr"]) and len(w["nnz_te"])
    r = np.load(os.path.join(GOLDEN, "random_5x6x131.npz"))
    assert (r["white"] != r["y"]).any() and (r["occluded"] != r["y"]).any()


def suffix_min_rule(y):
    """the rule of csrc/preprocess.cu: occluded iff min over j > x of (j - y_j) < x - y_x"""
    y = np.asarray(y, np.float32)
    a = np.arange(y.shape[-1], dtype=np.float32) - y
    suf = np.minimum.accumulate(a[..., ::-1], axis=-1)[..., ::-1]
    after = np.concatenate([suf[..., 1:], np.full(y.shape[:-1] + (1,), np.inf, np.float32)], axis=-1)
    return np.where(after < a, np.float32(0), y)


def png16_maps(rng, shape, dmax):
    v = np.floor(rng.uniform(0, dmax * 256, size=shape)) / 256
    runs = np.repeat(rng.integers(0, int(dmax) * 4, size=shape[:-1] + (shape[-1] // 5 + 1,)) / 4, 5, axis=-1)
    v = np.where(rng.random(shape) < 0.6, runs[..., :shape[-1]], v)           # quarter steps: many exact ties
    v[rng.random(shape) < 0.15] = 0
    return v.astype(np.float32)


@pytest.mark.parametrize("seed", range(6))
def test_suffix_min_rule_equals_the_reference_loop(seed):
    rng = np.random.default_rng(seed)
    W = int(rng.integers(2, 400))
    y = png16_maps(rng, (3, 20, W), dmax=float(rng.choice([4, 40, 255.99])))
    for m in (y, opp.remove_nonvisible(y)):
        assert np.array_equal(suffix_min_rule(m), opp.remove_occluded(m))


def test_reference_loop_is_order_independent():
    """the reference's threads zero pixels while others read them: any order of in-place, one-pixel-at-a-time decisions gives
    the decisions made on the values before the call"""
    rng = np.random.default_rng(7)
    for _ in range(20):
        y = png16_maps(rng, (40,), dmax=12)
        want = opp.remove_occluded(y)
        for _ in range(5):
            v = y.copy()
            for x in rng.permutation(len(v)):
                for i in range(1, len(v) - x):
                    if np.float32(i) - v[x + i] < -v[x]:
                        v[x] = 0
                        break
            assert np.array_equal(v, want)


def test_mt19937_matches_std_mt19937(tmp_path):
    cxx = shutil.which("c++") or shutil.which("g++") or shutil.which("clang++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    src = tmp_path / "mt.cpp"
    src.write_text(r"""
#include <cstdio>
#include <random>
#include <vector>
int main() {
  std::mt19937 g(42);
  for (int i = 0; i < 1500; i++) std::printf("%u\n", (unsigned)g());
  for (long n : {194L, 200L}) {          // THTensor_(randperm) after torch.manualSeed(42), + 1
    std::mt19937 r(42);
    std::vector<long> p(n);
    for (long i = 0; i < n; i++) p[i] = i;
    for (long i = 0; i < n - 1; i++) { long z = (long)(r() % (unsigned long)(n - i)); std::swap(p[i], p[i + z]); }
    for (long i = 0; i < n; i++) std::printf("%ld\n", p[i] + 1);
  }
}
""")
    exe = tmp_path / "mt"
    subprocess.check_call([cxx, "-O1", "-o", str(exe), str(src)])
    vals = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    g = preprocess.MT19937(42)
    assert [g.random() for _ in range(1500)] == vals[:1500]
    assert preprocess.randperm(194).tolist() == vals[1500:1694]
    assert preprocess.randperm(200).tolist() == vals[1694:]


def test_split_is_deterministic_and_matches_the_stored_split():
    stored = json.load(open(os.path.join(GOLDEN, "split.json")))
    for n in (194, 200):
        tr, te = preprocess.split(n)
        assert tr.dtype == te.dtype == np.int64 and len(te) == 40 and len(tr) == n - 40
        assert sorted(np.concatenate([te, tr]).tolist()) == list(range(1, n + 1))
        assert tr.tolist() == stored[str(n)]["tr"] and te.tolist() == stored[str(n)]["te"]
        t2, e2 = preprocess.split(n)
        assert np.array_equal(tr, t2) and np.array_equal(te, e2)
    with pytest.raises(ValueError, match="at least one more"):
        preprocess.split(40)


@pytest.fixture(scope="module")
def raw_trees(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("raw"))
    synth.write_kitti_raw(root, "kitti", n_tr=41, n_te=2, H=36, widths=(64, 57, 61), seed=3, D=16)
    synth.write_kitti_raw(root, "kitti2015", n_tr=42, n_te=3, H=33, widths=(60, 64), seed=4, D=16)
    return root


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015"])
def test_host_side_equals_the_cpu_restatement(raw_trees, dataset, tmp_path):
    want = opp.preprocess_kitti(raw_trees, dataset, **SMALL)
    host = preprocess.load_host(raw_trees, dataset, **SMALL)
    for k in ("x0", "x1", "dispnoc", "metadata"):
        assert host[k].dtype == want[k].dtype and np.array_equal(host[k], want[k]), k
    n_tr, n_te = (41, 2) if dataset == "kitti" else (42, 3)
    assert (host["n_tr"], host["n_te"]) == (n_tr, n_te)
    assert host["metadata"][:, 0].tolist() == [36 if dataset == "kitti" else 33] * (n_tr + n_te)
    assert host["metadata"][:, 2].tolist() == list(range(n_tr)) + list(range(n_te))
    w = host["metadata"][0, 1]
    assert not host["x0"][0, :, :, w:].any() and host["x0"][0, :, :, :w].std() > 0.5
    tr, te = preprocess.split(n_tr)
    assert np.array_equal(tr, want["tr"]) and np.array_equal(te, want["te"])
    # the sample lists of the restatement come from the maps as read: uncleaned dispnoc, rows of valid entries only
    assert len(want["nnz_tr"]) and len(want["nnz_te"]) and (want["nnz_tr"][:, 3] > 0.5).all()
    assert set(np.unique(want["nnz_te"][:, 0]).astype(int)) <= set(te.tolist())
    # the writer: .bin + .dim + .type per output, read back by main.lua's loader
    d = str(tmp_path / "out")
    preprocess.write_outputs(d, want)
    for f in preprocess.OUTPUTS:
        back = dataio.fromfile(os.path.join(d, f))
        assert back.dtype == want[f[:-4]].dtype and np.array_equal(back, want[f[:-4]]), f
    assert open(os.path.join(d, "metadata.bin.type")).read() == "int32"
    assert open(os.path.join(d, "te.bin.type")).read() == "int64"
    assert open(os.path.join(d, "x0.bin.dim")).read().split() == [str(n_tr + n_te), "1", "30", "64"]


def test_refuses_existing_outputs(raw_trees, tmp_path):
    root = str(tmp_path)
    shutil.copytree(os.path.join(raw_trees, "data.kitti"), os.path.join(root, "data.kitti"))
    open(os.path.join(root, "data.kitti", "te.bin.dim"), "w").write("40\n")
    with pytest.raises(FileExistsError, match="te.bin.dim"):
        preprocess.preprocess_kitti(root, "kitti", **SMALL)
    assert sorted(os.listdir(os.path.join(root, "data.kitti"))) == ["te.bin.dim", "unzip"]
    with pytest.raises(FileExistsError, match="te.bin.dim"):
        _tool().main(["both", "-data_root", root])            # the tool refuses before any work as well


def test_refuses_short_images_few_training_images_and_missing_maps(raw_trees, tmp_path):
    with pytest.raises(ValueError, match="fewer than the 40 the crop keeps"):
        preprocess.preprocess_kitti(raw_trees, "kitti", height=40, width=64)
    with pytest.raises(ValueError, match="columns, more than the 60"):
        preprocess.preprocess_kitti(raw_trees, "kitti", height=30, width=60)
    root = str(tmp_path)
    d = os.path.join(root, "data.kitti", "unzip")
    shutil.copytree(os.path.join(raw_trees, "data.kitti", "unzip"), d)
    os.remove(os.path.join(d, "training", "disp_noc", "000007_10.png"))
    with pytest.raises(FileNotFoundError, match="disp_noc/000007_10.png"):
        preprocess.preprocess_kitti(root, "kitti", **SMALL)
    shutil.copy(os.path.join(raw_trees, "data.kitti", "unzip", "training", "disp_noc", "000007_10.png"),
                os.path.join(d, "training", "disp_noc"))
    for sub in ("image_0", "image_1", "disp_noc"):
        os.remove(os.path.join(d, "training", sub, "000040_10.png"))
    with pytest.raises(ValueError, match="40 training images"):
        preprocess.preprocess_kitti(root, "kitti", **SMALL)
    assert sorted(os.listdir(os.path.join(root, "data.kitti"))) == ["unzip"]


def test_tool_arguments():
    tool = _tool()
    a = tool.parser().parse_args(["both", "-data_root", "/d", "-gpu", "2"])
    assert (a.dataset, a.data_root, a.gpu) == ("both", "/d", 2)
    with pytest.raises(SystemExit):
        tool.parser().parse_args(["mb"])
    with pytest.raises(SystemExit, match="1-based"):
        tool.main(["kitti", "-gpu", "0"])
