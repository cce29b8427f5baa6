"""`main.lua <dataset> <arch> -a predict -net_fname N -left L -right R -disp_max D` from files on (frontend.predict): the
network comes from an ascii .t7 (mccnn_b200/t7.py), runs through the wgmma feature tower (+ scorer head for 'slow') and
the adcensus chain.  Against the same stages driven directly with the layers the file was written from: the text format is
exact for fp32, so everything must match bit for bit -- and the stages themselves are held to the oracle by
test_gpu_feature_tower / test_gpu_scorer_head / test_gpu_parity."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import feature_tower, frontend, pipeline, scorer_head, synth, t7  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402


@pytest.mark.parametrize("arch", ["fast", "slow"])
def test_predict_from_net_file(tmp_path, arch):
    from PIL import Image

    H, W, D, shift, fm, nh2 = 36, 140, 16, 6, 16, 128
    rng = np.random.default_rng(5)
    base = synth.natural_image(np.random.default_rng(22), H, W + shift)
    u8 = np.clip((base - base.min()) / (base.max() - base.min()) * 255.0, 0, 255).astype(np.uint8)
    lp, rp = str(tmp_path / "l.png"), str(tmp_path / "r.png")
    Image.fromarray(np.ascontiguousarray(u8[:, :W])).save(lp)
    Image.fromarray(np.ascontiguousarray(u8[:, shift:])).save(rp)
    layers = oft.make_weights(rng, l1=3, fm=fm)
    head_layers = osh.make_weights(rng, fm, nh2, 2) if arch == "slow" else None
    net = str(tmp_path / "net.t7")
    t7.save_net(net, layers, head_layers, {"fm": fm})
    out = tmp_path / "out"
    disp = frontend.predict(lp, rp, "kitti", arch, disp_max=D, out_dir=str(out), net_fname=net)

    xb = torch.from_numpy(frontend.make_batch(lp, rp)).to("cuda:0")
    tower = feature_tower.FeatureTower(layers, arch=arch)
    head = scorer_head.ScorerHead(head_layers) if arch == "slow" else None
    opt = pipeline.make_params("kitti", arch, border=3)                # fix_border's width of the 3-layer net
    want, wl, wr = pipeline.stereo_predict(xb, tower.forward(xb), opt, D, want_vols=True, arch=arch, head=head)
    torch.cuda.synchronize()
    assert disp.shape == (H, W) and np.isfinite(disp).all()
    assert np.array_equal(disp, want.cpu().numpy()[0, 0]), "disparity map differs from the directly driven stages"
    for name, ref in (("right.bin", wr), ("left.bin", wl), ("disp.bin", want)):
        data = np.fromfile(str(out / name), "<f4")
        assert np.array_equal(data, ref.cpu().numpy().ravel(), equal_nan=True), name
    tower.close()
    if head is not None:
        head.close()


def test_arch_mismatch_and_missing_net_are_refused(tmp_path):
    rng = np.random.default_rng(0)
    img = synth.natural_image(rng, 20, 60).astype(np.float32)
    net = str(tmp_path / "fast.t7")
    t7.save_net(net, oft.make_weights(rng, l1=2, fm=16))
    with pytest.raises(ValueError, match="'fast' network"):
        frontend.predict(img, img, "kitti", "slow", disp_max=8, net_fname=net)
    with pytest.raises(ValueError, match="net_fname"):
        frontend.predict(img, img, "kitti", "fast", disp_max=8)
