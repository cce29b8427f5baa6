"""GPU: the result images of csrc/render.cu byte for byte against the numpy restatement (oracle/render.py) and the reference's
grey2jet fixture, then end to end: -a predict's bins through bin2png, and Evaluator.test(debug_dir=...) on synthetic KITTI and
Middlebury sets."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, evaluate, frontend, pipeline, render, synth  # noqa: E402
from oracle import render as orr  # noqa: E402

SIZES = [(1, 1), (370, 1226), (1000, 1500)]


def _specials(rng, a, frac=0.01):
    """NaN, +-inf, f32(1e38) (NaN's stand-in in bin2png) and 2e38 sprinkled over a float32 array"""
    flat = a.reshape(-1)
    for v in (np.nan, np.inf, -np.inf, 1e38, 2e38):
        flat[rng.random(flat.size) < frac] = v
    return a


def _volume(rng, D, H, W):
    vol = rng.integers(0, 6, (D, H, W)).astype(np.float32)               # small integers: many ties
    _specials(rng, vol, 0.02)
    vol[:, rng.random((H, W)) < 0.05] = np.nan                            # all-NaN columns
    return vol


@pytest.mark.parametrize("D,H,W", [(1, 1, 1), (70, 1, 1), (400, 1, 1), (1, 1000, 1500), (70, 370, 1226),
                                   (228, 370, 1226), (400, 64, 1500), (70, 1000, 1500)])
def test_volume_file_grey_equals_oracle(tmp_path, D, H, W):
    rng = np.random.default_rng(D * 7 + H)
    vol = _volume(rng, D, H, W)
    path = str(tmp_path / "left.bin")
    vol.astype("<f4").tofile(path)
    got = render.volume_file_grey(path, D, H, W).cpu().numpy()
    assert np.array_equal(got, orr.volume_grey(vol))       # 70x370x1226 and larger span several 64 MiB chunks


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("d", [1, 70, 228, 400])
def test_map_grey_equals_oracle(H, W, d):
    rng = np.random.default_rng(H + d)
    x = _specials(rng, rng.uniform(-5, d * 1.2, (H, W)).astype(np.float32))
    got = render.map_grey(torch.from_numpy(x).cuda(), d).cpu().numpy()
    assert np.array_equal(got, orr.map_grey(x, d))


def _jet_map(rng, H, W, dm):
    lo, hi = -1 - 0.025 * dm, 1.025 * dm - 1                              # (x + 1) / dm * 4 in [-0.1, 4.1]
    x = rng.uniform(lo, hi, (H, W)).astype(np.float32)
    x = np.clip(x, np.nextafter(np.float32(lo), np.float32(0)), np.nextafter(np.float32(hi), np.float32(0)))
    k = min(x.size, dm)
    x.reshape(-1)[:k] = np.arange(k, dtype=np.float32)                    # the integer disparities
    x.reshape(-1)[rng.random(x.size) < 0.05] = 0                          # no ground truth (blue masked)
    return x


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("dm", [1, 70, 228])
@pytest.mark.parametrize("mask_blue", [False, True])
def test_grey2jet_equals_oracle(H, W, dm, mask_blue):
    x = _jet_map(np.random.default_rng(H * dm), H, W, dm)
    got = render.grey2jet(torch.from_numpy(x).cuda(), dm, mask_blue=mask_blue).cpu().numpy()
    assert np.array_equal(got, orr.grey2jet(x, dm, mask_blue=mask_blue))


@pytest.mark.parametrize("dm", [70, 228])
def test_grey2jet_equals_reference_fixture(golden_dir, dm):
    z = np.load(os.path.join(golden_dir, "render.npz"))
    grey = (np.arange(dm) + 1) / dm                                       # main.lua's grey of disparity d = 0 .. dm - 1
    idx = np.array([np.flatnonzero(z["grey"] == g)[0] for g in grey])
    want = np.moveaxis(orr.quantise(z["rgb"][:, idx]), 0, -1)[None]
    got = render.grey2jet(torch.arange(dm, dtype=torch.float32, device="cuda")[None], dm).cpu().numpy()
    assert np.array_equal(got, want)


@pytest.mark.parametrize("bad", [float("nan"), -1 - 0.026 * 70, 1.026 * 70 - 1, float("inf")])
def test_grey2jet_refuses_nan_and_out_of_range(bad):
    x = torch.zeros((37, 53), device="cuda")
    x[20, 30] = bad
    with pytest.raises(adcensus.AdcensusError, match="outside the colour map"):
        render.grey2jet(x, 70)
    torch.cuda.synchronize()
    render.grey2jet(torch.zeros((37, 53), device="cuda"), 70)            # the device is still usable


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("err_at", [3.0, 1.0])
def test_error_image_equals_oracle(H, W, err_at):
    rng = np.random.default_rng(H + int(err_at))
    x0 = rng.standard_normal((H, W)).astype(np.float32) * np.float32(1.5)
    gt = rng.uniform(0, 60, (H, W)).astype(np.float32)
    gt[rng.random((H, W)) < 0.3] = 0
    step = rng.choice(np.array([-err_at - 0.5, -err_at, -0.3, 0, err_at, err_at + 0.25, 7], np.float32), (H, W))
    pred = (gt + step).astype(np.float32)                                 # |gt - pred| on both sides of err_at, and on it
    t = lambda a: torch.from_numpy(a).cuda()
    got = render.error_image(t(x0), t(pred), t(gt), err_at).cpu().numpy()
    assert np.array_equal(got, orr.error_image(x0, pred, gt, err_at))


def _png(path):
    from PIL import Image

    with Image.open(path) as im:
        return im.mode, np.asarray(im).copy()


def test_bin2png_on_predict_output(tmp_path, capsys):
    from PIL import Image

    H, W, shift = 48, 130, 7
    base = synth.natural_image(np.random.default_rng(4), H, W + shift)
    u8 = np.clip((base - base.min()) / (base.max() - base.min()) * 255.0, 0, 255).astype(np.uint8)
    lp, rp = str(tmp_path / "l.png"), str(tmp_path / "r.png")
    Image.fromarray(np.ascontiguousarray(u8[:, shift:])).save(lp)
    Image.fromarray(np.ascontiguousarray(u8[:, :W])).save(rp)
    out = str(tmp_path / "out")
    frontend.predict(lp, rp, "kitti", "census", disp_max=70, out_dir=out)
    capsys.readouterr()
    render.bin2png(out, disp_max=70, height=H, width=W)
    assert capsys.readouterr().out.splitlines() == ["Writing left.png", "Writing right.png", "Writing disp.png"]
    for name in ("left", "right"):
        vol = np.fromfile(os.path.join(out, name + ".bin"), "<f4").reshape(70, H, W)
        mode, a = _png(os.path.join(out, name + ".png"))
        assert mode == "L" and np.array_equal(a, orr.volume_grey(vol)), name
    mode, a = _png(os.path.join(out, "disp.png"))
    disp = np.fromfile(os.path.join(out, "disp.bin"), "<f4").reshape(H, W)
    assert mode == "L" and np.array_equal(a, orr.map_grey(disp, 70))


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("render_eval"))
    synth.write_kitti_set(root, "kitti", n_tr=3, n_te=2, H=32, width=150, widths=(150, 131), seed=21)
    synth.write_mb_set(root, n=6, shapes=((32, 96, 24), (40, 110, 40)), seed=22)
    return root


@pytest.mark.parametrize("dataset", ["kitti", "mb"])
def test_debug_images_equal_oracle_and_leave_the_errors_alone(sets, tmp_path, dataset, capsys):
    ev = evaluate.Evaluator(dataset, "census")
    plain = ev.test("test_te", data_root=sets)
    plain_out = capsys.readouterr().out.splitlines()
    dbg = str(tmp_path / "tmp")
    res = ev.test("test_te", data_root=sets, debug_dir=dbg)
    dbg_out = capsys.readouterr().out.splitlines()
    ev.close()
    assert [e[3] for e in res.examples] == [e[3] for e in plain.examples] and res.mean == plain.mean
    col = lambda lines: [l.split("\t")[1] for l in lines[:-1]] + lines[-1:]
    assert col(dbg_out) == col(plain_out)
    data = evaluate.load_data(dataset, sets)
    opt = pipeline.make_params(dataset, "census")
    err_at = {"kitti": 3.0, "mb": 1.0}[dataset]
    names = set()
    for ex, id_, _, _ in res.examples:
        x, disp_max, _, _, img_width = data.example(ex)
        pred = pipeline.stereo_predict(torch.from_numpy(x).cuda(), None, opt, disp_max, arch="census")[0, 0].cpu().numpy()
        gt = data.ground_truth(ex, img_width)
        want = (orr.grey2jet(gt, disp_max, mask_blue=True), orr.grey2jet(pred, disp_max),
                orr.error_image(x[0, 0], pred, gt, err_at))
        files = render.debug_names(dataset, "census", id_)
        assert files[0] == "%s_%s_gt.png" % (dataset, id_)
        for f, w in zip(files, want):
            mode, a = _png(os.path.join(dbg, f))
            assert mode == "RGB" and np.array_equal(a, w), (id_, f)
        names.update(files)
    assert set(os.listdir(dbg)) == names and len(names) == 3 * len(res.examples)
