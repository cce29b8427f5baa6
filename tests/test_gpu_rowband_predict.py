"""GPU: one pair predicted by row bands from the images (rowband.band_source / predict_pair, tools/predict_rowband.py).

* On one device, rank by rank: each rank's band volumes (feature tower on the band's rows, scorer head on the band, census /
  AD on the band's rows, then fix_border) equal the corresponding rows of the whole image's volumes bit for bit, for
  N = 2, 3, 5 ranks, every architecture, at 350 x 1242 and at a small size with odd W and H divisible by none of the N.
  This pins that the wgmma tower and scorer head compute each pixel independently of the frame's height.
* A one-process run of tools/predict_rowband.py writes the files frontend.predict writes, byte for byte, for every arch.
* On two GPUs (skipped below two): torchrun runs of the tool for 'slow' and 'census' write the same files as
  frontend.predict on one GPU.
Random networks of the published KITTI shapes (fast: 4 x 64; slow: 4 x 112, head 4 x 384), written with t7.save_net."""
import filecmp
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import frontend, pipeline, rowband, synth, t7  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARCHS = ("fast", "slow", "census", "ad")


def _net(path, arch, seed=3):
    rng = np.random.default_rng(seed)
    if arch == "fast":
        t7.save_net(path, oft.make_weights(rng, l1=4, fm=64))
    else:
        t7.save_net(path, oft.make_weights(rng, l1=4, fm=112), osh.make_weights(rng, 112, 384, 4), {"fm": 112})
    return path


def _images(tmp_path, H, W, shift=7, seed=22):
    from PIL import Image

    base = synth.natural_image(np.random.default_rng(seed), H, W + shift)
    u8 = np.clip((base - base.min()) / (base.max() - base.min()) * 255.0, 0, 255).astype(np.uint8)
    lp, rp = str(tmp_path / "left.png"), str(tmp_path / "right.png")
    Image.fromarray(np.ascontiguousarray(u8[:, shift:])).save(lp)
    Image.fromarray(np.ascontiguousarray(u8[:, :W])).save(rp)
    return lp, rp


def _same(a, b):
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("H,W,D", [(350, 1242, 228), (47, 131, 20)])
def test_band_volumes_equal_rows_of_the_whole_image(tmp_path, arch, H, W, D):
    dev = torch.device("cuda", 0)
    lp, rp = _images(tmp_path, H, W)
    xb = torch.from_numpy(frontend.make_batch(lp, rp)).to(dev)
    method = frontend.StereoMethod("kitti", arch, _net(str(tmp_path / "net.t7"), arch) if arch in ("fast", "slow") else None)
    tower, head = method.stages(dev)
    feats = tower.forward(xb) if tower is not None else None
    opt = pipeline.make_params("kitti", arch)
    # the volumes as main.lua holds them at :986: the chain stopped right after the matching cost
    _, wantL, wantR = pipeline.stereo_predict(xb, feats, pipeline.make_params("kitti", arch, sm_terminate="cnn"), D,
                                              want_vols=True, arch=arch, head=head)
    wantL, wantR = wantL[0], wantR[0]
    del feats
    volumes, extends = rowband.band_source(rowband.CudaOps(dev), xb, D, opt, arch, tower, head)
    assert extends == (arch != "slow")
    for N in (2, 3, 5):
        covered = 0
        for r in range(N):
            ya, yb = rowband.source_rows(H, N, r, opt, extends)
            vl, vr = volumes(ya, yb, (1, -1))
            assert _same(vl, wantL[:, ya:yb]), "%s N %d rank %d: left volume rows [%d, %d)" % (arch, N, r, ya, yb)
            assert _same(vr, wantR[:, ya:yb]), "%s N %d rank %d: right volume rows [%d, %d)" % (arch, N, r, ya, yb)
            covered += yb - ya
            del vl, vr
        if not extends:
            assert covered == H
    torch.cuda.synchronize()
    method.close()


def _frontend_files(tmp_path, lp, rp, arch, D, net):
    out = str(tmp_path / "frontend")
    frontend.predict(lp, rp, "kitti", arch, disp_max=D, out_dir=out, net_fname=net)
    torch.cuda.synchronize()
    return out


def _tool_argv(arch, lp, rp, D, net, out):
    argv = ["tools/predict_rowband.py", "kitti", arch, "-left", lp, "-right", rp, "-disp_max", str(D), "-out", out]
    return argv + (["-net_fname", net] if net else [])


def _assert_same_files(a, b):
    for name in ("right.bin", "left.bin", "disp.bin"):
        assert filecmp.cmp(os.path.join(a, name), os.path.join(b, name), shallow=False), name


@pytest.mark.parametrize("arch", ARCHS)
def test_tool_one_process_writes_frontend_predict_files(tmp_path, arch):
    H, W, D = 61, 203, 24
    lp, rp = _images(tmp_path, H, W)
    net = _net(str(tmp_path / "net.t7"), arch) if arch in ("fast", "slow") else None
    want = _frontend_files(tmp_path, lp, rp, arch, D, net)
    out = str(tmp_path / "rowband")
    r = subprocess.run([sys.executable] + _tool_argv(arch, lp, rp, D, net, out), cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    _assert_same_files(out, want)
    assert os.path.getsize(os.path.join(out, "left.bin")) == D * H * W * 4


@pytest.mark.parametrize("arch,port", [("slow", 29571), ("census", 29572)])
def test_tool_two_gpus_writes_frontend_predict_files(tmp_path, arch, port):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    H, W, D = 97, 230, 40
    lp, rp = _images(tmp_path, H, W)
    net = _net(str(tmp_path / "net.t7"), arch) if arch == "slow" else None
    want = _frontend_files(tmp_path, lp, rp, arch, D, net)
    out = str(tmp_path / "rowband")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port)] + _tool_argv(arch, lp, rp, D, net, out)
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    _assert_same_files(out, want)
