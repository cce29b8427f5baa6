"""GPU: the feature tower and the scorer head run on the device that holds their weights, whatever the current device is,
and refuse input on another device (or on the CPU) on the host, before any call into the library."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, feature_tower, pipeline, scorer_head, synth  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402


def _nets(seed=3, fm=16, nh2=128):
    rng = np.random.default_rng(seed)
    return oft.make_weights(rng, l1=3, fm=fm), osh.make_weights(rng, fm, nh2, 2)


def _no_library_calls(monkeypatch):
    """after this, any call into the CUDA library fails the test"""
    def lib():
        raise AssertionError("the library was called")
    monkeypatch.setattr(adcensus, "lib", lib)


def test_refuses_input_on_the_cpu(monkeypatch):
    tl, hl = _nets()
    tower = feature_tower.FeatureTower(tl, arch="slow", device=0)
    head = scorer_head.ScorerHead(hl, device=0)
    x = torch.zeros((2, 1, 4, 70))
    f = torch.zeros((16, 4, 70))
    fd = f.to("cuda:0")
    with monkeypatch.context() as m:
        _no_library_calls(m)
        with pytest.raises(adcensus.AdcensusError):
            tower.forward(x)
        with pytest.raises(adcensus.AdcensusError):
            head.volumes(f, f, 8)
        with pytest.raises(adcensus.AdcensusError):
            head.volumes(fd, f, 8)                                  # features on two devices
        with pytest.raises(adcensus.AdcensusError):
            head.volumes(f, fd, 8)
    tower.close()
    head.close()


def _need2():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")


def test_refuses_input_on_another_gpu(monkeypatch):
    _need2()
    tl, hl = _nets()
    tower = feature_tower.FeatureTower(tl, arch="slow", device=1)
    head = scorer_head.ScorerHead(hl, device=1)
    f0, f1 = torch.zeros((16, 4, 70), device="cuda:0"), torch.zeros((16, 4, 70), device="cuda:1")
    with monkeypatch.context() as m:
        _no_library_calls(m)
        with pytest.raises(adcensus.AdcensusError):
            tower.forward(torch.zeros((2, 1, 4, 70), device="cuda:0"))
        for a, b in ((f0, f0), (f0, f1), (f1, f0)):
            with pytest.raises(adcensus.AdcensusError):
                head.volumes(a, b, 8)
    tower.close()
    head.close()


def test_slow_arch_on_the_second_gpu_equals_the_first():
    """tower, head and the operator chain on cuda:1 while the current device is 0: the same bits as on cuda:0"""
    _need2()
    H, W, D = 40, 150, 24
    p = synth.make_pair(H, W, 4, D, seed=9)
    x = torch.from_numpy(np.stack([p["imgL"], p["imgR"]])[:, None].astype(np.float32))
    opt = pipeline.make_params("kitti", "slow")
    tl, hl = _nets()
    torch.cuda.set_device(0)
    out = []
    for dev in (0, 1):
        tower = feature_tower.FeatureTower(tl, arch="slow", device=dev)
        head = scorer_head.ScorerHead(hl, device=dev)
        xb = x.to("cuda:%d" % dev)
        feats = tower.forward(xb)
        disp, vl, vr = pipeline.stereo_predict(xb, feats, opt, D, want_vols=True, arch="slow", head=head)
        torch.cuda.synchronize(dev)
        assert torch.cuda.current_device() == 0
        out.append([t.contiguous().cpu() for t in (feats, vl, vr, disp)])
        tower.close()
        head.close()
    for a, b, what in zip(out[0], out[1], ("features", "left volume", "right volume", "disparity map")):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what + " differs between cuda:0 and cuda:1"
