"""CPU, world_size 2 and 3 over gloo: one pair predicted by row bands from the standardised images for every architecture
(rowband.band_predict): each rank computes the cost volumes of its own rows only -- the feature tower on the band's rows,
the scorer head ('slow') on the band itself with the first CBCA block's halo rows exchanged, census / AD on the band's rows
-- then the band chain.  The CPU oracle stands in for the CUDA operators and the two networks.  The disparity map, both
volumes and the files rowband.write_outputs writes must equal the single-process oracle chain bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_rowband_gloo import OracleOps, _free_port  # noqa: E402


class ImageOracleOps(OracleOps):
    """OracleOps with the image-based matching costs (main.lua:932-942)"""

    def ad(self, x0, x1, D, direction):
        return torch.from_numpy(self.o.ad(self._n(x0)[0], self._n(x1)[0], D, direction))

    def census(self, x0, x1, D, direction):
        return torch.from_numpy(self.o.census(self._n(x0), self._n(x1), D, direction))


class OracleTower:
    """FeatureTower's interface on oracle/feature_tower.py (float64 accumulation)"""

    def __init__(self, layers, arch):
        self.layers, self.arch, self.l1 = layers, arch, len(layers)

    def forward(self, x):
        from oracle import tower_head_cases as thc

        return torch.from_numpy(thc.tower_want(x.numpy(), self.layers, self.arch))


class CountingHead:
    """ScorerHead's interface on oracle/scorer_head.py; records the rows and directions of every call"""

    def __init__(self, layers):
        self.layers, self.calls = layers, []

    def volumes(self, fL, fR, D, want_left=True, want_right=True):
        from oracle import scorer_head as osh

        self.calls.append((fL.shape[1], bool(want_left), bool(want_right)))
        out = []
        for want, direction in ((want_left, -1), (want_right, 1)):
            out.append(torch.from_numpy(osh.head_volume(fL.numpy(), fR.numpy(), D, self.layers, direction))[None]
                       if want else None)
        return out[0], out[1]


# name -> ((dataset, arch), overrides, H, W, D, world, want_vols)
CASES = {
    "kitti_fast": (("kitti", "fast"), dict(cbca_i1=2, L1=4, cbca_i2=1), 37, 52, 12, 2, True),
    "mb_fast": (("mb", "fast"), {}, 41, 48, 9, 3, True),
    "kitti_slow": (("kitti", "slow"), dict(cbca_i2=2), 37, 52, 12, 3, True),
    # L1 14: halo 13, two first-block iterations need 26 rows, the bands hold 13 -> one exchange per iteration
    "mb_slow": (("mb", "slow"), dict(cbca_i2=2), 41, 48, 9, 3, True),
    "mb_slow_disp_only": (("mb", "slow"), dict(cbca_i2=2), 41, 48, 9, 2, False),
    "kitti_census": (("kitti", "census"), {}, 37, 52, 12, 2, True),
    "mb_census": (("mb", "census"), dict(cbca_i2=2), 41, 48, 9, 3, True),
    "kitti_ad": (("kitti", "ad"), {}, 37, 52, 12, 3, True),
    "mb_ad": (("mb", "ad"), {}, 41, 48, 9, 2, True),
}


def _problem(case):
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import frontend, pipeline, synth
    from oracle import feature_tower as oft
    from oracle import scorer_head as osh

    (dataset, arch), over, H, W, D, world, want_vols = CASES[case]
    opt = pipeline.make_params(dataset, arch, **over)
    rng = np.random.default_rng(H * W + D)
    img = synth.natural_image(rng, H, W + 5)
    x_batch = frontend.make_batch(img[:, 5:], img[:, :W])
    l1 = 4 if dataset == "kitti" else 5
    tower = oft.make_weights(rng, l1=l1, fm=8) if arch in ("fast", "slow") else None
    head = osh.make_weights(rng, fm=8, nh2=16, l2=2) if arch == "slow" else None
    return opt, x_batch, D, arch, tower, head, world, want_vols


def _want(case):
    """the single-process oracle chain on the whole image: disp (H, W), volL, volR (D, H, W)"""
    from oracle import oracle as orc
    from oracle import scorer_head as osh
    from oracle import tower_head_cases as thc

    opt, x_batch, D, arch, tower, head, _, _ = _problem(case)
    imgL, imgR = x_batch[0, 0], x_batch[1, 0]
    params = orc.Params(**opt.as_dict())
    if arch in ("ad", "census"):
        return orc.stereo_predict_chain(imgL, imgR, D, params, arch=arch, want_vols=True)
    f = thc.tower_want(x_batch, tower, arch)
    if arch == "fast":
        return orc.stereo_predict_chain(imgL, imgR, D, params, arch="fast", featL=f[0], featR=f[1], want_vols=True)
    vl = osh.head_volume(f[0], f[1], D, head, -1)
    vr = osh.head_volume(f[0], f[1], D, head, 1)
    return orc.stereo_predict_chain(imgL, imgR, D, params, arch="volumes", want_vols=True, volL=vl, volR=vr)


def _worker(rank, world, port, case, outdir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from mccnn_b200 import rowband
    from oracle import oracle as orc

    opt, x_batch, D, arch, tower, head, _, want_vols = _problem(case)
    head_op = CountingHead(head) if head is not None else None
    tower_op = OracleTower(tower, arch) if tower is not None else None
    comm = rowband.Comm()
    out = rowband.band_predict(ImageOracleOps(orc), torch.from_numpy(x_batch), D, opt, arch, tower_op, head_op, comm,
                               want_vols=want_vols)
    disp = out[0] if want_vols else out
    np.save(os.path.join(outdir, "disp_rank%d.npy" % rank), disp.numpy())
    if want_vols:
        np.save(os.path.join(outdir, "volL_rank%d.npy" % rank), out[1].numpy())
        np.save(os.path.join(outdir, "volR_rank%d.npy" % rank), out[2].numpy())
        rowband.write_outputs(os.path.join(outdir, "files"), disp, out[1], out[2], comm)
    if head_op is not None:
        np.save(os.path.join(outdir, "head_calls_rank%d.npy" % rank), np.array(head_op.calls, dtype=np.int64))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("case", sorted(CASES))
def test_band_predict_matches_single_process(tmp_path, case):
    sys.path.insert(0, ROOT)
    from mccnn_b200 import rowband
    from oracle import oracle as orc

    orc.lib()                                   # built here once, not by the ranks at the same time
    opt, x_batch, D, arch, _, _, world, want_vols = _problem(case)
    H, W = x_batch.shape[2:]
    mp.spawn(_worker, args=(world, _free_port(), case, str(tmp_path)), nprocs=world, join=True)
    want, wL, wR = _want(case)
    same = lambda a, b: a.shape == b.shape and np.array_equal(a, b, equal_nan=True)
    for r in range(world):
        got = np.load(os.path.join(str(tmp_path), "disp_rank%d.npy" % r))
        assert same(got, want), "rank %d of %d: disparity map differs from the single-process chain" % (r, world)
        y0, y1 = rowband.split(H, world, r)
        if want_vols:
            assert same(np.load(os.path.join(str(tmp_path), "volL_rank%d.npy" % r)), wL[:, y0:y1]), "rank %d: left volume" % r
            assert same(np.load(os.path.join(str(tmp_path), "volR_rank%d.npy" % r)), wR[:, y0:y1]), "rank %d: right volume" % r
        if arch == "slow":
            # the head scores this rank's band and nothing else, in one call; the right volume only when it is consumed
            calls = np.load(os.path.join(str(tmp_path), "head_calls_rank%d.npy" % r)).tolist()
            right = bool(want_vols or opt.lr_check)
            assert calls == [[y1 - y0, 1, int(right)]], "rank %d scored %s, its band is rows [%d, %d)" % (r, calls, y0, y1)
    if want_vols:
        files = os.path.join(str(tmp_path), "files")
        for name, ref in (("right.bin", wR), ("left.bin", wL), ("disp.bin", want)):
            data = np.fromfile(os.path.join(files, name), "<f4")
            assert np.array_equal(data, ref.astype("<f4").ravel(), equal_nan=True), name


def test_mb_slow_case_falls_back_to_one_exchange_per_iteration():
    """the split of "mb_slow": the first CBCA block's 2 x halo rows exceed a band, the bands are at least one halo tall"""
    sys.path.insert(0, ROOT)
    from mccnn_b200 import rowband

    opt, x_batch, _, _, _, _, world, _ = _problem("mb_slow")
    H = x_batch.shape[2]
    halo = rowband.cbca_halo(opt)[1]
    band_min = min(b - a for a, b in (rowband.split(H, world, p) for p in range(world)))
    assert halo <= band_min < opt.cbca_i1 * halo


def test_source_rows():
    sys.path.insert(0, ROOT)
    from mccnn_b200 import pipeline, rowband

    opt = pipeline.make_params("kitti", "census")           # L1 0 -> arm 2, halo 1; cbca_i1 4 -> 4 rows
    assert rowband.source_rows(100, 4, 0, opt, True) == (0, 29)
    assert rowband.source_rows(100, 4, 1, opt, True) == (21, 54)
    assert rowband.source_rows(100, 4, 3, opt, True) == (71, 100)
    assert rowband.source_rows(100, 4, 1, opt, False) == (25, 50)


def test_band_predict_refuses_stage_options_and_unknown_arch():
    sys.path.insert(0, ROOT)
    from mccnn_b200 import pipeline, rowband
    from oracle import oracle as orc

    xb = torch.zeros((2, 1, 8, 8))
    with pytest.raises(ValueError, match="sm_skip"):
        rowband.band_predict(ImageOracleOps(orc), xb, 4, pipeline.make_params("kitti", "census", sm_skip="sgm"), "census")
    with pytest.raises(ValueError, match="arch"):
        rowband.band_predict(ImageOracleOps(orc), xb, 4, pipeline.make_params("kitti", "census"), "cnn")
    with pytest.raises(ValueError, match="tower"):
        rowband.band_predict(ImageOracleOps(orc), xb, 4, pipeline.make_params("kitti", "slow"), "slow")


@pytest.mark.parametrize("argv,msg", [
    (["kitti", "census", "-left", "l.png", "-right", "r.png", "-disp_max", "8", "-sm_skip", "sgm"], "sm_skip"),
    (["kitti", "census", "-left", "l.png", "-right", "r.png", "-disp_max", "8", "-sm_terminate", "cbca1"], "sm_terminate"),
    (["kitti", "census", "-left", "l.png", "-disp_max", "8"], "-right"),
    (["kitti", "fast", "-left", "l.png", "-right", "r.png", "-disp_max", "8"], "net_fname"),
    (["kitti", "census", "-a", "test_te", "-left", "l.png", "-right", "r.png", "-disp_max", "8"], "-a predict"),
    (["mb", "census", "-left", "l.png", "-right", "r.png", "-disp_max", "8", "-color", "rgb"], "color"),
])
def test_tool_refuses_before_any_gpu_work(argv, msg):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import predict_rowband

    with pytest.raises((SystemExit, ValueError), match=msg):
        predict_rowband.parse_args(argv)


def test_tool_refuses_a_net_of_the_other_arch(tmp_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import predict_rowband
    from mccnn_b200 import frontend, t7
    from oracle import feature_tower as oft

    net = str(tmp_path / "fast.t7")
    t7.save_net(net, oft.make_weights(np.random.default_rng(0), l1=2, fm=16))
    with pytest.raises(SystemExit, match="'fast' network"):
        predict_rowband.parse_args(["kitti", "slow", "-left", "l", "-right", "r", "-disp_max", "8", "-net_fname", net])
    args, over = predict_rowband.parse_args(["kitti", "fast", "-left", "l", "-right", "r", "-disp_max", "8", "-net_fname", net])
    assert over == {} and args.out == "."
    assert frontend.StereoMethod(args.dataset, args.arch, args.net_fname, **over).opt.border == 2      # the net's, not 4


def test_predict_pair_refuses_before_any_gpu_work(tmp_path):
    sys.path.insert(0, ROOT)
    from mccnn_b200 import rowband, t7
    from oracle import feature_tower as oft

    img = np.random.default_rng(1).random((20, 30)).astype(np.float32)
    net = str(tmp_path / "fast.t7")
    t7.save_net(net, oft.make_weights(np.random.default_rng(0), l1=2, fm=16))
    with pytest.raises(ValueError, match="net_fname"):
        rowband.predict_pair(img, img, "kitti", "fast", disp_max=8)
    with pytest.raises(ValueError, match="'fast' network"):
        rowband.predict_pair(img, img, "kitti", "slow", disp_max=8, net_fname=net)
    with pytest.raises(ValueError, match="sm_terminate"):
        rowband.predict_pair(img, img, "kitti", "census", disp_max=8, sm_terminate="sgm")
    with pytest.raises(ValueError, match="arch"):
        rowband.predict_pair(img, img, "kitti", "cnn", disp_max=8)
