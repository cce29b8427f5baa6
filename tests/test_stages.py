"""CPU: main.lua's -sm_terminate / -sm_skip (main.lua:953-1082) -- the step names and their codes, the refusals of
make_params, evaluate.check_stage_options, tools/run_main.py, tools/ablation.py and the row-band driver, the stage plan, and the
oracle chain of every variant against a hand composition of the per-operator oracle functions.  The GPU side is
tests/test_gpu_stages.py."""
import importlib.util
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import evaluate, pipeline, rowband, search, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


sc = _load("stage_chain", "tests", "stage_chain.py")

# The steps in chain order, and which of them each variant runs (with the LR check; without it, occlusion and mismatch never
# run).  Written out from the table of main.lua:988-1079, independently of pipeline.stages and of stage_chain.
ORDER = ("cbca1", "sgm", "cbca2", "occlusion", "mismatch", "subpixel", "median", "bilateral")
SKIPPED = {"cbca": {"cbca1", "cbca2"}, "sgm": {"sgm"}, "occlusion": {"occlusion", "mismatch"},
           "subpixel_enchancement": {"subpixel"}, "median": {"median"}, "bilateral": {"bilateral"}}
LAST = {"cnn": None, "cbca1": "cbca1", "sgm": "sgm", "cbca2": "cbca2", "occlusion": "occlusion", "mismatch": "mismatch",
        "subpixel_enchancement": "subpixel", "median": "median"}


def expected_steps(terminate, skip, lr_check):
    steps = set(ORDER)
    if skip:
        steps -= SKIPPED[skip]
    if terminate and not (terminate in ("occlusion", "mismatch") and not lr_check):
        last = LAST[terminate]
        steps &= set(ORDER[:ORDER.index(last) + 1]) if last else set()
    if not lr_check:
        steps -= {"occlusion", "mismatch"}
    return steps


def hand_chain(orc, imgL, imgR, volL, volR, D, opt, steps):
    """the per-operator oracle functions composed for one set of steps (main.lua:986-1079)"""
    x0c, x1c = orc.cross(imgL, opt.L1, opt.tau1), orc.cross(imgR, opt.L1, opt.tau1)
    vols, disp = {}, {}
    for direction, vol in ((1, volR), (-1, volL)):
        if "cbca1" in steps:
            for _ in range(opt.cbca_i1):
                vol = orc.cbca(x0c, x1c, vol, direction)
        if "sgm" in steps:
            for _ in range(opt.sgm_i):
                vol = orc.transpose_hwd_to_dhw_div4(orc.sgm2(imgL, imgR, orc.transpose_dhw_to_hwd(vol), opt.pi1, opt.pi2,
                                                             opt.tau_so, opt.alpha1, opt.sgm_q1, opt.sgm_q2, direction))
        if "cbca2" in steps:
            for _ in range(opt.cbca_i2):
                vol = orc.cbca(x0c, x1c, vol, direction)
        vols[direction], disp[direction] = vol, orc.spatial_argmin(vol) - 1
    d = disp[-1]
    if "occlusion" in steps or "mismatch" in steps:
        outlier = orc.outlier_detection(disp[-1], disp[1], D)
        if "occlusion" in steps:
            d = orc.interpolate_occlusion(d, outlier)
        if "mismatch" in steps:
            d = orc.interpolate_mismatch(d, outlier)
    if "subpixel" in steps:
        d = orc.subpixel_enchancement(d, vols[-1], D)
    if "median" in steps:
        d = orc.median2d(d, 5)
    if "bilateral" in steps:
        d = orc.mean2d(d, orc.gaussian(opt.blur_sigma), opt.blur_t)
    return d, vols[-1], vols[1]


def test_names_map_to_codes():
    assert pipeline.Params._fields_[-2:] == [("sm_terminate", pipeline.ctypes.c_int), ("sm_skip", pipeline.ctypes.c_int)]
    p = pipeline.make_params("kitti", "fast")
    assert (p.sm_terminate, p.sm_skip) == (0, 0)
    codes = {"cnn": 1, "cbca1": 2, "sgm": 3, "cbca2": 4, "occlusion": 5, "mismatch": 6, "subpixel_enchancement": 7, "median": 8}
    for name, code in codes.items():
        assert pipeline.make_params("kitti", "fast", sm_terminate=name).sm_terminate == code
    skips = {"sgm": 3, "occlusion": 5, "subpixel_enchancement": 7, "median": 8, "bilateral": 9, "cbca": 10}
    for name, code in skips.items():
        assert pipeline.make_params("mb", "census", sm_skip=name).sm_skip == code
    assert set(pipeline.SM_TERMINATE) == {""} | set(sc.TERMINATE) and set(pipeline.SM_SKIP) == {""} | set(sc.SKIP)
    assert pipeline.make_params("kitti", "fast", sm_terminate="", sm_skip="").as_dict() == p.as_dict()


@pytest.mark.parametrize("option,name", [("sm_terminate", "bilateral"), ("sm_terminate", "cbca"), ("sm_skip", "cnn"),
                                         ("sm_skip", "cbca1"), ("sm_skip", "mismatch"), ("sm_skip", "subpixel"),
                                         ("sm_terminate", "SGM"), ("sm_skip", 3), ("sm_terminate", None)])
def test_unknown_names_are_refused(option, name):
    valid = " ".join(sc.TERMINATE if option == "sm_terminate" else sc.SKIP)
    with pytest.raises(ValueError, match="-%s .*valid: %s" % (option, valid)):
        pipeline.make_params("kitti", "fast", **{option: name})
    with pytest.raises(ValueError, match="-%s .*valid: %s" % (option, valid)):
        evaluate.check_stage_options("kitti", "census", **{option: name})


def test_check_stage_options_accepts_every_step_that_does_work():
    for t in sc.TERMINATE:
        evaluate.check_stage_options("kitti", "census", sm_terminate=t)        # CBCA 4 + 8, SGM, LR check
        evaluate.check_stage_options("kitti2015", "slow", sm_terminate=t, cbca_i2=1)
    for s in sc.SKIP:
        evaluate.check_stage_options("kitti", "accurate_cbca4", sm_skip=s)
    opt = evaluate.check_stage_options("kitti2015", "ad", sm_terminate="sgm", sm_skip="cbca")
    assert (opt.sm_terminate, opt.sm_skip, opt.cbca_i2) == (3, 10, 4)          # the kitti ad preset
    # check_options does not see the arch: it refuses both and points to check_stage_options
    for option in ("sm_terminate", "sm_skip"):
        with pytest.raises(ValueError, match="-%s is checked .* check_stage_options" % option):
            evaluate.check_options("kitti", **{option: "sgm"})


@pytest.mark.parametrize("dataset,arch,option,name,over", [
    ("kitti", "fast", "sm_terminate", "cbca1", {}),                # the fast presets have no CBCA
    ("kitti2015", "fast", "sm_terminate", "cbca2", {}),
    ("kitti", "fast", "sm_skip", "cbca", {}),
    ("kitti", "slow", "sm_terminate", "cbca2", {}),                # cbca_i2 = 0
    ("kitti", "ad", "sm_terminate", "cbca1", {}),                  # cbca_i1 = 0
    ("mb", "census", "sm_skip", "occlusion", {}),                  # no LR check
    ("mb", "slow", "sm_terminate", "occlusion", {}),
    ("mb", "fast", "sm_terminate", "mismatch", {}),
    ("kitti", "census", "sm_skip", "sgm", dict(sgm_i=0)),
    ("kitti", "census", "sm_terminate", "cbca1", dict(cbca_i1=0)),
])
def test_steps_that_do_no_work_are_refused(dataset, arch, option, name, over):
    with pytest.raises(ValueError, match="-%s %s: that step does no work in the %s %s" % (option, name, dataset, arch)):
        evaluate.check_stage_options(dataset, arch, **dict(over, **{option: name}))
    # the same variant is still a valid pipeline parameter set: it equals another variant (test_mb_no_op_variants...)
    pipeline.make_params(dataset, arch, **dict(over, **{option: name}))


def test_idle_steps_follow_the_parameters():
    assert pipeline.idle_steps(pipeline.make_params("kitti", "fast")) == {"cbca", "cbca1", "cbca2"}
    assert pipeline.idle_steps(pipeline.make_params("mb", "fast")) == {"cbca", "cbca1", "cbca2", "occlusion", "mismatch"}
    assert pipeline.idle_steps(pipeline.make_params("kitti", "accurate_cbca4")) == set()
    assert pipeline.idle_steps(pipeline.make_params("kitti", "fast", cbca_i2=1, sgm_i=0)) == {"cbca1", "sgm"}
    evaluate.check_stage_options("kitti", "fast", sm_terminate="cbca1", cbca_i1=2)       # an override brings the step back


@pytest.mark.parametrize("lr_check", [0, 1])
@pytest.mark.parametrize("variant", sc.VARIANTS, ids=sc.variant_id)
def test_stage_plan_follows_the_table(variant, lr_check):
    t, s = variant
    opt = pipeline.make_params("kitti", "accurate_cbca4", lr_check=lr_check, sm_terminate=t, sm_skip=s)
    st = pipeline.stages(opt)
    assert {k for k, v in st.items() if v} == expected_steps(t, s, lr_check)


CHAIN_CASES = [  # (dataset, arch, overrides): arch fast and census, KITTI and Middlebury presets
    ("kitti", "fast", {}),
    ("kitti", "accurate_cbca4", {}),
    ("mb", "fast", {}),
    ("kitti", "census", dict(cbca_i1=2, cbca_i2=2)),
    ("mb", "census", dict(cbca_i1=2, cbca_i2=2)),
]
H, W, C, D = 11, 29, 8, 7


def _inputs(orc, dataset, arch, over):
    opt = pipeline.make_params(dataset, arch, **over)
    p = synth.make_pair(H, W, C, D, seed=5)
    if arch == "census":
        volL, volR = orc.census(p["imgL"], p["imgR"], D, -1), orc.census(p["imgR"], p["imgL"], D, 1)
    else:
        volL, volR = orc.stereo_join(p["featL"], p["featR"], D)
        orc.fix_border(volL, opt.border, -1)
        orc.fix_border(volR, opt.border, 1)
    return opt, p, volL, volR


@pytest.mark.parametrize("dataset,arch,over", CHAIN_CASES, ids=lambda v: v if isinstance(v, str) else "")
def test_oracle_chain_equals_hand_composition(oracle, dataset, arch, over):
    opt, p, volL, volR = _inputs(oracle, dataset, arch, over)
    kind = "census" if arch == "census" else "fast"
    full = oracle.stereo_predict_chain(p["imgL"], p["imgR"], D, sc.full_chain_params(oracle, opt), arch=kind,
                                       featL=p["featL"], featR=p["featR"])
    for t, s in sc.VARIANTS:
        got, gL, gR = sc.oracle_chain(oracle, p["imgL"], p["imgR"], D, opt, t, s, arch=kind, featL=p["featL"],
                                      featR=p["featR"], want_vols=True)
        want, wL, wR = hand_chain(oracle, p["imgL"], p["imgR"], volL, volR, D, opt, expected_steps(t, s, opt.lr_check))
        what = "%s %s %s" % (dataset, arch, sc.variant_id((t, s)))
        for g, w, n in ((got, want, "disp"), (gL, wL, "left volume"), (gR, wR, "right volume")):
            assert np.array_equal(g, w, equal_nan=True), "%s: %s differs from the hand composition" % (what, n)
        if not (t or s):
            assert np.array_equal(got, full, equal_nan=True), "%s: differs from oracle.stereo_predict_chain" % what


@pytest.mark.parametrize("arch", ["fast", "census"])
def test_mb_no_op_variants_equal_the_full_chain(oracle, arch):
    opt, p, _, _ = _inputs(oracle, "mb", arch, dict(cbca_i1=2, cbca_i2=2) if arch == "census" else {})
    run = lambda t, s: sc.oracle_chain(oracle, p["imgL"], p["imgR"], D, opt, t, s, arch=arch, featL=p["featL"], featR=p["featR"])
    full = run("", "")
    for t, s in (("", "occlusion"), ("occlusion", ""), ("mismatch", "")):
        assert np.array_equal(run(t, s), full, equal_nan=True), (t, s)
    lr_only = {"occlusion", "mismatch"}
    assert lr_only <= pipeline.idle_steps(opt)
    if arch == "census":                             # CBCA and SGM do work: only the LR-check variants are left out
        assert [v for _, v in search.ablation_variants(opt)] == (
            [{}] + [{"sm_skip": s} for s in sc.SKIP if s not in lr_only]
            + [{"sm_terminate": t} for t in sc.TERMINATE if t not in lr_only])


@pytest.mark.parametrize("dataset,arch,over", CHAIN_CASES, ids=lambda v: v if isinstance(v, str) else "")
def test_terminate_cnn_is_the_raw_volume_argmin(oracle, dataset, arch, over):
    opt, p, volL, _ = _inputs(oracle, dataset, arch, over)
    got = sc.oracle_chain(oracle, p["imgL"], p["imgR"], D, opt, "cnn", "", arch="census" if arch == "census" else "fast",
                          featL=p["featL"], featR=p["featR"])
    assert np.array_equal(got, oracle.spatial_argmin(volL) - 1)
    if arch != "census":
        assert np.isnan(volL).any()                 # NaN at invalid positions, skipped by the argmin


def test_full_chain_params_refuses_a_variant(oracle):
    with pytest.raises(AssertionError, match="full chain only"):
        sc.full_chain_params(oracle, pipeline.make_params("kitti", "fast", sm_skip="sgm"))


def test_rowband_refuses_stage_options_before_any_work():
    for over in (dict(sm_skip="median"), dict(sm_terminate="cnn")):
        opt = pipeline.make_params("mb", "fast", **over)
        with pytest.raises(ValueError, match="row-band .* -%s is not supported" % next(iter(over))):
            rowband.stereo_predict_rowband(None, None, None, None, None, 8, opt)


def test_ablation_variants():
    v = search.ablation_variants(pipeline.make_params("kitti", "accurate_cbca4"))
    assert v[0] == ("full", {}) and len(v) == 15
    assert [l for l, _ in v[1:7]] == ["-sm_skip " + s for s in sc.SKIP]
    assert [l for l, _ in v[7:]] == ["-sm_terminate " + t for t in sc.TERMINATE]
    for _, ov in v:                                  # every variant is a valid candidate of the search
        pipeline.make_params("kitti", "fast", **ov)
    # steps that do no work are left out, as run_main.py refuses them
    for dataset, arch in (("kitti", "fast"), ("kitti2015", "slow"), ("mb", "census"), ("mb", "fast"), ("kitti", "ad")):
        opt = pipeline.make_params(dataset, arch)
        labels = [l for l, _ in search.ablation_variants(opt)]
        idle = pipeline.idle_steps(opt)
        assert labels == ["full"] + ["-sm_skip " + s for s in sc.SKIP if s not in idle] + [
            "-sm_terminate " + t for t in sc.TERMINATE if t not in idle]
        for l, ov in search.ablation_variants(opt)[1:]:
            evaluate.check_stage_options(dataset, arch, **ov)
    assert len(search.ablation_variants(pipeline.make_params("kitti", "fast"))) == 12
    assert len(search.ablation_variants(pipeline.make_params("mb", "census"))) == 12
    assert len(search.ablation_variants(pipeline.make_params("mb", "fast"))) == 9


def test_ablation_cli_refusals():
    ab = _load("ablation", "tools", "ablation.py")
    args = ab.parse_args(["mb", "census", "-", "-rect", "perfect", "-gpu", "2"])
    assert (args.dataset, args.arch, args.rect, args.device) == ("mb", "census", "perfect", 1)
    for bad, msg in ((["kitti", "fast", "-"], "needs a net file"), (["kitti", "slow", "/no/such.t7"], "does not exist"),
                     (["kitti", "ad", "-", "-gpu", "0"], "1-based")):
        with pytest.raises(SystemExit, match=msg):
            ab.parse_args(bad)


def _run_main():
    return _load("run_main", "tools", "run_main.py")


def test_run_main_parses_the_stage_options():
    rm = _run_main()
    args, ov = rm.parse_args(["kitti", "fast", "-a", "test_te", "-net_fname", "n.t7", "-sm_skip", "sgm"])
    assert ov == {"sm_skip": "sgm"}
    args, ov = rm.parse_args(["mb", "census", "-a", "predict", "-left", "l", "-right", "r", "-disp_max", "9",
                              "-sm_terminate", "cbca1", "-pi1", "2"])
    assert ov == {"sm_terminate": "cbca1", "pi1": 2.0}
    args, ov = rm.parse_args(["kitti", "census", "-sm_terminate", "", "-sm_skip", ""])
    assert ov == {}
    args, ov = rm.parse_args(["kitti", "fast", "-sm_terminate", "cbca1", "-cbca_i1", "2"])
    assert ov == {"sm_terminate": "cbca1", "cbca_i1": 2}
    for bad, msg in ((["kitti", "fast", "-sm_terminate", "bilateral"], "-sm_terminate 'bilateral' is not a step"),
                     (["kitti", "fast", "-sm_skip", "cnn"], "-sm_skip 'cnn' is not a step"),
                     (["kitti", "fast", "-sm_terminate", "cbca1"], "-sm_terminate cbca1: that step does no work"),
                     (["mb", "census", "-a", "predict", "-sm_skip", "occlusion"], "-sm_skip occlusion: that step"),
                     (["kitti", "census", "-sm_skip", "sgm", "-sgm_i", "0"], "-sm_skip sgm: that step")):
        with pytest.raises(ValueError, match=msg):
            rm.parse_args(bad)


def test_run_main_still_refuses_the_other_options():
    rm = _run_main()
    for bad, msg in ((["kitti", "slow", "-at", "1"], "-at 1"), (["mb", "fast", "-color", "rgb"], "-color rgb"),
                     (["kitti", "fast", "-debug"], "-debug"), (["kitti", "fast", "-use_cache"], "-use_cache"),
                     (["kitti", "fast", "-make_cache", "1"], "-make_cache")):
        with pytest.raises(ValueError, match=msg):
            rm.parse_args(bad)
