"""CPU: preprocess_mb.py's restatement (mccnn_b200/preprocess.py, oracle/preprocess_mb.py) -- the oracle against the
script's own read_im / load_pfm outputs, numpy's pairwise summation, the discovery of a raw tree in the script's order, and
every refusal (with nothing written).  The GPU half is tests/test_gpu_preprocess_mb.py."""
import os
import shutil

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import preprocess, synth
from oracle import preprocess_mb as opm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "preprocess_mb")


def _golden(name):
    return np.load(os.path.join(GOLDEN, name))


def test_oracle_read_im_equals_the_scripts_fixtures(tmp_path):
    g = _golden("read_im.npz")
    names = sorted({k.split("/")[0] for k in g.files})
    assert {"rgb_png_61x97", "rgb_ppm_13x11", "grey_pgm_43x17", "grey_png_16x16", "rgb_png_2x3"} == set(names)
    for name in names:
        p = tmp_path / (name + "." + name.split("_")[1])
        p.write_bytes(g[name + "/file"].tobytes())
        rgb = opm.imread_rgb(str(p))
        for color in ("gray", "rgb"):
            want = g[name + "/" + color]
            got = opm.read_im(rgb, color)
            assert got.dtype == want.dtype and np.array_equal(got, want), (name, color)


def test_grey_of_grey_is_not_the_identity():
    v = np.arange(256, dtype=np.uint8)
    grey = opm.cv_grey(np.repeat(v[:, None], 3, 1))
    assert int((grey != v.astype(np.float32)).sum()) == 29
    g = _golden("read_im.npz")
    x = g["grey_png_16x16/gray"]                   # every byte value: the script's output carries the same 29 deviations
    assert np.array_equal(opm.read_im(np.repeat(np.arange(256, dtype=np.uint8).reshape(16, 16, 1), 3, 2), "gray"), x)


def test_oracle_pfm_reading_and_halving_equal_the_scripts_fixtures(tmp_path):
    g = _golden("pfm.npz")
    for name in ("special_10x14", "random_36x50"):
        p = tmp_path / (name + ".pfm")
        p.write_bytes(g[name + "/file"].tobytes())
        assert np.array_equal(opm.read_pfm(str(p)), g[name + "/load"], equal_nan=True)
        assert np.array_equal(opm.half_disp(g[name + "/load"]), g[name + "/half"], equal_nan=True)
        h = tmp_path / (name + ".pfm.H.pfm")
        h.write_bytes(g[name + "/half_file"].tobytes())
        assert np.array_equal(opm.read_pfm(str(h)), g[name + "/half_cached"], equal_nan=True)
        assert np.array_equal(g[name + "/half_cached"], g[name + "/half"], equal_nan=True)
    s = g["special_10x14/half"]
    assert np.isnan(s).any() and np.isinf(s).any() and (s == np.float32(7.25) / 2).any()


@pytest.mark.parametrize("n", list(range(1, 201)) + [8191, 8192, 8193])
def test_pairwise_sum_equals_numpy(n):
    rng = np.random.default_rng(n)
    a = rng.uniform(0, 255, n).astype(np.float32)
    assert opm.pairwise_sum(a) == a.sum()
    m, s = opm.mean_std(a)
    assert m == a.mean() and s == a.std()


@pytest.mark.parametrize("shape", [(1000, 1500), (1000, 1500, 3), (997, 1483)], ids=str)
def test_pairwise_sum_equals_numpy_at_full_frame(shape):
    rng = np.random.default_rng(1)
    b = rng.integers(0, 256, shape).astype(np.float32)
    x = b.transpose(2, 0, 1) if b.ndim == 3 else b[None]       # read_im's rgb layout: a transposed view
    m, s = opm.mean_std(b.ravel())
    assert m == x.mean() and s == x.std()


# ---- the host side --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("mb_raw"))
    synth.write_mb_raw(root, seed=3)
    return root


@pytest.fixture
def copy(tree, tmp_path):
    root = str(tmp_path / "root")
    shutil.copytree(tree, root)
    return root


def test_discovery_follows_the_script(tree):
    sc = preprocess.mb_scenes(tree, "imperfect")
    logs = [s["log"] for s in sc]
    assert logs[:11] == ["Scene%02d" % k for k in range(11)]
    assert logs[11:19] == ["Aloe", "Baby1", "Art", "conesH", "teddyH", "map", "sawtooth", "tsukuba"]   # Books: no disp1.png
    assert logs[19:34] == ["trainingH/" + n for n in sorted(synth.MB_SUBMIT_NAMES)]
    assert logs[34:] == ["testH/" + n for n in sorted(n + "T" for n in synth.MB_SUBMIT_NAMES)]
    assert [s["submit"] for s in sc[-30:]] == logs[-30:] and all(s["submit"] is None for s in sc[:-30])
    # exposures: counts cycle through 2, 3, 5, 6, 7, 8 with the other camera one more on every third scene
    want = {2: (2, 2), 3: (3, 2), 5: (3, 2), 6: (3, 2), 7: (3, 2), 8: (3, 2)}
    for k in range(11):
        groups = sc[k]["groups"]
        assert groups[0][1] == (4,) and len(groups) == 1 + 1 + k % 3
        assert all(g[1] == want[(2, 3, 5, 6, 7, 8)[k % 6]] for g in groups[1:])
    files = sc[0]["groups"][1][0]                                # exposures 0, 1 of Scene00 (2 and 3 present)
    assert [os.path.basename(f) for f in files] == ["im0e0.png", "im1e0.png", "im0e1.png", "im1e1.png"]
    assert [os.path.basename(f) for f in sc[1]["groups"][1][0]][::2] == ["im0e0.png", "im0e1.png", "im0e2.png"]
    assert sc[4]["groups"][1][0][0].endswith("L1/im0e1.png")     # 7 exposures -> 1, 3, 5
    assert [s["ndisp"] for s in sc[:11]] == [24] * 11
    assert [s["ndisp"] for s in sc[11:16]] == ["ceil"] * 5 and [s["ndisp"] for s in sc[16:19]] == [-1] * 3
    assert [s["ndisp"] for s in sc[19:]] == [24] * 30
    assert sc[0]["size"] == (40, 96)
    perf = preprocess.mb_scenes(tree, "perfect")
    assert perf[0]["groups"][1][0][0].split(os.sep)[-4] == "Scene00-perfect"
    assert perf[0]["groups"][0][0][0].split(os.sep)[-2] == "Scene00-imperfect"


def test_exposure_table(tree):
    sc = preprocess.mb_scenes(tree, "imperfect")
    for k, first in ((0, 0), (1, 0), (2, 0), (3, 0), (4, 1), (5, 1)):          # min over the cameras: 2, 2, 5, 6, 7, 8
        assert os.path.basename(sc[k]["groups"][1][0][0]) == "im0e%d.png" % first
    assert preprocess.MB_EXPOSURES == {8: (1, 3, 5), 7: (1, 3, 5), 6: (0, 2, 4), 5: (0, 2, 4), 3: (0, 1, 2), 2: (0, 1)}


def test_ndisp_is_floor_division_and_junk_names_are_ignored(copy):
    base = os.path.join(copy, preprocess.MB_DATA, "scenes2014", "datasets", "Scene03-imperfect")
    with open(os.path.join(base, "calib.txt"), "w") as f:
        f.write("ndisp=49\n")
    open(os.path.join(base, "ambient", "L1", "notes.txt"), "w").close()
    sc = preprocess.mb_scenes(copy, "imperfect")
    assert sc[3]["ndisp"] == 24


def test_empty_groups_write_the_data_file_too(tmp_path):
    preprocess._tofile_mb(str(tmp_path / "x_12_1.bin"), None)
    assert open(tmp_path / "x_12_1.bin.dim").read() == "0\n" and os.path.getsize(tmp_path / "x_12_1.bin") == 0


def test_oracle_runs_the_whole_script(tree):
    o = opm.preprocess_mb(tree, "imperfect", "gray")
    assert len(o["X"]) == 49 and o["meta"].shape == (49, 3) and o["meta"].dtype == np.int32
    assert [x is None for x in o["X"][11]] == [True, False, False, False]
    assert o["X"][0][0].shape == (4, 1, 40, 96) and o["X"][0][1].shape == (2, 2, 1, 40, 96)
    assert set(np.unique(o["nnz_te"][:, 0]).tolist()) == set(range(1, 11))
    assert set(np.unique(o["nnz_tr"][:, 0]).tolist()) == set(range(11, 20))
    tr = o["nnz_tr"]
    assert ((tr[:, 0] == 17) & (tr[:, 3] == 0)).any()                    # 2001 map: 0 is a real disparity
    assert o["te"].dtype == np.int64 and o["te"].tolist() == list(range(1, 11))
    assert o["meta"][11:16, 2].min() > 0 and (o["meta"][16:19, 2] == -1).all()


def _refused(root, exc, match, rect="imperfect"):
    with pytest.raises(exc, match=match):
        preprocess.preprocess_mb(root, rect, "gray")
    assert not os.path.exists(preprocess.mb_output_dir(root, rect, "gray")), "something was written"


def test_refuses_fewer_than_ten_2014_scenes(copy):
    base = os.path.join(copy, preprocess.MB_DATA, "scenes2014", "datasets")
    for k in (4, 7):
        shutil.rmtree(os.path.join(base, "Scene%02d-imperfect" % k))
    _refused(copy, ValueError, "9 2014 scenes")


def test_refuses_an_exposure_count_outside_the_table(copy):
    l1 = os.path.join(copy, preprocess.MB_DATA, "scenes2014", "datasets", "Scene02-imperfect", "ambient", "L1")
    for f in os.listdir(l1):
        if f.startswith("im") and f[4] in "4" and f.endswith(".png"):
            os.remove(os.path.join(l1, f))                              # 5 exposures -> 4
    _refused(copy, ValueError, "4 exposures")


def test_refuses_16_bit_images(copy):
    from PIL import Image

    p = os.path.join(copy, "data.mb", "unzip", "MiddEval3", "testH", "PianoT", "im1.png")
    Image.fromarray(np.zeros((40, 96), np.uint16)).save(p)
    _refused(copy, ValueError, "8-bit images expected")


def test_refuses_colour_disparity_images(copy):
    from PIL import Image

    p = os.path.join(copy, preprocess.MB_DATA, "scenes2003", "teddyH", "disp6.pgm")
    Image.fromarray(np.zeros((40, 96, 3), np.uint8)).save(p.replace(".pgm", ".ppm"))
    os.replace(p.replace(".pgm", ".ppm"), p)
    _refused(copy, ValueError, "grey map expected")


def test_refuses_colour_pfm(copy):
    p = os.path.join(copy, preprocess.MB_DATA, "scenes2014", "datasets", "Scene06-imperfect", "disp0y.pfm")
    with open(p, "wb") as f:
        f.write(b"PF\n96 80\n-1.0\n" + np.zeros(80 * 96 * 3, "<f4").tobytes())
    _refused(copy, ValueError, "single-channel PFM")


def test_refuses_odd_full_size_views(copy):
    from PIL import Image

    p = os.path.join(copy, preprocess.MB_DATA, "scenes2014", "datasets", "Scene07-imperfect", "im1E.png")
    Image.fromarray(np.zeros((80, 191, 3), np.uint8)).save(p)
    _refused(copy, ValueError, "halving needs even sizes")


def test_refuses_missing_files_and_mismatched_sizes(copy):
    base = os.path.join(copy, preprocess.MB_DATA, "scenes2006", "HalfSize", "Aloe")
    os.remove(os.path.join(base, "Illum2", "Exp1", "view5.png"))
    _refused(copy, FileNotFoundError, "view5.png")


def test_refuses_mismatched_map_size(copy):
    from PIL import Image

    p = os.path.join(copy, preprocess.MB_DATA, "scenes2001", "data", "tsukuba", "nonocc.png")
    Image.fromarray(np.zeros((40, 94), np.uint8)).save(p)
    _refused(copy, ValueError, "nonocc.png is 40x94")


def test_refuses_existing_outputs(copy):
    d = preprocess.mb_output_dir(copy, "imperfect", "gray")
    os.makedirs(d)
    open(os.path.join(d, "meta.bin.dim"), "w").close()
    with pytest.raises(FileExistsError, match="meta.bin.dim"):
        preprocess.preprocess_mb(copy, "imperfect", "gray")
    assert os.listdir(d) == ["meta.bin.dim"]


def test_refuses_bad_options(copy):
    with pytest.raises(ValueError, match="color"):
        preprocess.preprocess_mb(copy, "imperfect", "grey")
    _refused(copy, ValueError, "rect", rect="both")


def test_tool_parses_the_scripts_arguments():
    import importlib.util

    spec = importlib.util.spec_from_file_location("preprocess_mb_tool", os.path.join(ROOT, "tools", "preprocess_mb.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    a = mod.parser().parse_args(["perfect", "rgb", "-data_root", "/d", "-gpu", "2"])
    assert (a.rect, a.color, a.data_root, a.gpu) == ("perfect", "rgb", "/d", 2)
    with pytest.raises(SystemExit):
        mod.parser().parse_args(["imperfect", "grey"])
