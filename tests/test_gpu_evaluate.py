"""GPU: main.lua's -a test_te / test_all / submit / time (mccnn_b200/evaluate.py) on synthetic KITTI and Middlebury sets with
random networks written to .t7 files.  Every per-example error, the mean and every submission file must equal what the
operator chain (pipeline.stereo_predict), driven directly with the layers the net file was written from and the net's
fix_border width, gives on the same inputs -- also for arch 'fast', whose evaluation runs one StereoPipeline at many shapes."""
import os
import zipfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, evaluate, feature_tower, pipeline, scorer_head, synth, t7  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402

NET_BORDER = 3    # both nets have three 3x3 layers; the presets say 4 (kitti) and 5 (mb)


@pytest.fixture(scope="module")
def world(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("eval"))
    synth.write_kitti_set(root, "kitti", n_tr=4, n_te=2, H=32, width=300, widths=(300, 263, 281), seed=11)
    synth.write_mb_set(root, n=6, shapes=((32, 96, 24), (40, 110, 40)), seed=12)
    rng = np.random.default_rng(13)
    layers = {"fast": (oft.make_weights(rng, l1=3, fm=64), None),
              "slow": (oft.make_weights(rng, l1=3, fm=16), osh.make_weights(rng, 16, 128, 2))}
    nets = {}
    for arch, (tower, head) in layers.items():
        nets[arch] = os.path.join(root, "net_%s.t7" % arch)
        t7.save_net(nets[arch], tower, head)
    return dict(root=root, layers=layers, nets=nets)


def _reference_maps(world, dataset, arch, examples):
    """pipeline.stereo_predict on each example, stages built directly from the layers"""
    data = evaluate.load_data(dataset, world["root"])
    tower = head = None
    if arch in ("fast", "slow"):
        tl, hl = world["layers"][arch]
        tower = feature_tower.FeatureTower(tl, arch=arch)
        head = scorer_head.ScorerHead(hl) if hl is not None else None
        opt = pipeline.make_params(dataset, arch, border=NET_BORDER)
    else:
        opt = pipeline.make_params(dataset, arch)
    maps = []
    for ex in examples:
        x, disp_max, _, _, img_width = data.example(ex)
        xb = torch.from_numpy(x).cuda()
        feats = tower.forward(xb) if tower is not None else None
        d = pipeline.stereo_predict(xb, feats, opt, disp_max, arch=arch, head=head)
        has_gt = ex[0] in data.dispnoc if dataset == "mb" else ex < len(data.dispnoc)
        maps.append((d.cpu().numpy()[0, 0], data.ground_truth(ex, img_width) if has_gt else None))
    return data, maps


def _evaluator(world, dataset, arch):
    return evaluate.Evaluator(dataset, arch, net_fname=world["nets"].get(arch) if arch in ("fast", "slow") else None)


@pytest.mark.parametrize("arch", ["fast", "slow", "census"])
@pytest.mark.parametrize("dataset,action", [("kitti", "test_te"), ("kitti", "test_all"), ("mb", "test_te")])
def test_test_actions_equal_the_operator_chain(world, dataset, action, arch, capsys):
    ev = _evaluator(world, dataset, arch)
    if arch in ("fast", "slow"):
        assert ev.opt.border == NET_BORDER
    res = ev.test(action, data_root=world["root"])
    data, maps = _reference_maps(world, dataset, arch, [e[0] for e in res.examples])
    assert [e[0] for e in res.examples] == data.examples(action)
    errs = []
    for (ex, id_, runtime, err), (pred, gt) in zip(res.examples, maps):
        want = dataio.bad_pixel_rate(pred, gt, dataio.ERR_AT[dataset])
        assert err == want, "%s %s %s example %s: err %r, operator chain %r" % (dataset, arch, action, id_, err, want)
        assert runtime > 0
        errs.append(want)
    assert res.mean == sum(errs) / len(errs)
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == len(errs) + 1 and lines[-1] == "%.14g" % res.mean
    assert lines[0].split("\t")[1] == "%.14g" % errs[0]
    if action == "test_all" and arch == "fast":        # several widths, one odd: one pipeline at the largest shape served all
        assert len({m[0].shape[1] for m in maps}) > 1 and any(m[0].shape[1] % 2 for m in maps)
        assert (ev.sp.H, ev.sp.W, ev.sp.D) == (32, max(m[0].shape[1] for m in maps), 228)
    ev.close()


@pytest.mark.parametrize("dataset,arch", [("kitti", "fast"), ("mb", "slow"), ("mb", "fast")])
def test_submit_files_equal_the_writers_on_the_operator_chain(world, tmp_path, dataset, arch):
    ev = _evaluator(world, dataset, arch)
    out = tmp_path / "out"
    out.mkdir()
    (out / ".empty").write_bytes(b"")
    res = ev.submit(data_root=world["root"], out=str(out))
    ev.close()
    data, maps = _reference_maps(world, dataset, arch, [e[0] for e in res.examples])
    assert [e[0] for e in res.examples] == data.examples("submit")
    want_dir = tmp_path / "want"
    want_dir.mkdir()
    names = set()
    for (ex, id_, runtime), (pred, _) in zip(res.examples, maps):
        if dataset == "kitti":
            img_height, img_width = int(data.metadata[ex, 0]), int(data.metadata[ex, 1])
            rel = os.path.relpath(dataio.write_kitti_submission(pred, img_height, img_width, str(want_dir), id_, dataset),
                                  str(want_dir))
            names.add(rel)
        else:
            sub = data.fname_submit[ex[0] - (len(data.X) - len(data.fname_submit))]
            os.makedirs(want_dir / sub, exist_ok=True)
            rel = os.path.join(sub, "disp0%s.pfm" % ev.method_name)
            dataio.write_pfm(np.flipud(pred), str(want_dir / rel))
            names.add(rel)
            t = open(out / sub / ("time%s.txt" % ev.method_name)).read()
            assert t == "%.14g" % runtime and float(t) > 0
            names.add(os.path.join(sub, "time%s.txt" % ev.method_name))
            for parts in (sub.split("/")[:1], sub.split("/")):
                names.add("/".join(parts) + "/")
        assert (out / rel).read_bytes() == (want_dir / rel).read_bytes(), id_
    with zipfile.ZipFile(res.zip) as z:
        assert set(z.namelist()) == names


@pytest.mark.parametrize("arch,n", [("fast", 30), ("slow", 3), ("census", 3)])
def test_time_tiny(world, arch, n, capsys):
    ev = _evaluator(world, "kitti", arch)
    res = ev.time(tiny=True)
    ev.close()
    assert len(res.runtimes) == n and np.isfinite(res.runtime_min) and res.runtime_min > 0
    assert res.runtime_min == min(res.runtimes)
    assert capsys.readouterr().out.strip() == "%.14g" % res.runtime_min
