"""Sampled background features (UseSampleFeature: 1, the OMD configuration) on the GPU against the serial restatement in
tests/sample_reference.py: the sampler and the option-II filter bit for bit, the whole tracker against the oracle pipeline, seeds, batches
that mix the two options, the create-time refusals and the host shim."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests.sample_reference import SAMPLE_N, SampleOracleTracker, filter_static_sampled, sample_keypoints
from tests.test_tracker_batch_gpu import GET_NAMES, _assert_maps_same, _assert_same
from tests.test_tracker_gpu import _compare
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_frame, make_sequence_frame

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
OMD_K = np.array([618.3587036132812, 618.5924072265625, 328.9866333007812, 237.7507629394531], np.float32)
# example/omd.yaml; the synthetic depth is disparity * 256 for bf = 387.5744, so DepthMapFactor stays 256.  A 6 / 2 window fires the
# windowed BA at f_id 5 and 9.
OMD = dict(width=640, height=480, fx=float(OMD_K[0]), fy=float(OMD_K[1]), cx=float(OMD_K[2]), cy=float(OMD_K[3]), depth_factor=256.0, th_depth_bg=40.0,
           th_depth_obj=25.0, max_track_bg=1200, max_track_obj=800, sf_mg_thres=0.02, sf_ds_thres=0.99, n_features=3000, is_kitti=0, dataset=1,
           window_size=6, overlap_size=2)


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@pytest.mark.parametrize("h,w", [(480, 640), (375, 1242)])
def test_sampler_equals_reference(ctx, h, w):
    """seeds 0 and 2^32 - 1 plus f_id: the frame seed wraps to 0, which cv::RNG maps to 0xffffffff"""
    seeds = [0, 1, 2, 2 ** 32 - 1, (2 ** 32 - 1 + 1) % 2 ** 32, (2 ** 32 - 1 + 2) % 2 ** 32, 123456789]
    kx, ky, ms = capi.sample_keys(ctx, seeds, w, h)
    assert kx.shape == (len(seeds), SAMPLE_N) and ms > 0
    for i, s in enumerate(seeds):
        rx, ry = sample_keypoints(h, w, s)
        assert np.array_equal(kx[i], rx) and np.array_equal(ky[i], ry), f"seed {s}"


def test_sampler_refuses_small_images(ctx):
    with pytest.raises(capi.VdoError):
        capi.sample_keys(ctx, [1], 19, 480)
    with pytest.raises(capi.VdoError):
        capi.sample_keys(ctx, [1], 640, 19)


def _hostile_frame(w, h, seed):
    """a textured frame where many samples are refused: labelled blocks, zero flow in a band, invalid or far depth, and flow that carries
    targets past every edge (negative targets, which the option-I bounds would let through)"""
    rng = np.random.default_rng(seed)
    gray = make_frame(seed=seed, width=w, height=h, n_obj=0)["gray"]
    mask = np.zeros((h, w), np.int32)
    mask[h // 4:h // 2, w // 5:w // 2] = 3
    mask[2 * h // 3:, 3 * w // 4:] = 7
    disp = rng.uniform(8.0, 60.0, (h, w)).astype(np.float32) * 256.0
    disp[rng.random((h, w)) < 0.05] = -1.0                                # depth 0 after preparation
    disp[:, : w // 10] = 100.0                                            # about 1000 m: beyond ThDepthBG
    flow = rng.normal(0.0, 3.0, (h, w, 2)).astype(np.float32)
    flow[h // 2: h // 2 + h // 8] = 0.0
    flow[:, w // 10: w // 5, 0] = -float(w)                               # targets left of the image
    flow[: h // 8, :, 1] = -float(h) / 4                                  # targets above the image
    flow[:, 9 * w // 10:, 0] = float(w) / 8                               # targets right of the image
    return gray, disp, flow, mask


@pytest.mark.parametrize("w,h,seed", [(640, 480, 0), (1242, 375, 2 ** 32 - 1)])
def test_frame_build_equals_reference(ctx, w, h, seed):
    """a tracker's first frame keeps exactly the option-II keys of the reference, with their correspondences, flows and depths"""
    gray, disp, flow, mask = _hostile_frame(w, h, 5 + w)
    kw = dict(OMD, width=w, height=h, cx=w * 0.5, cy=h * 0.5)
    tr = capi.Tracker(ctx, use_sample_feature=1, sample_seed=seed, **kw)
    orc = SampleOracleTracker(use_sample_feature=1, sample_seed=seed, width=w, height=h, K4=(kw["fx"], kw["fy"], kw["cx"], kw["cy"]), depth_factor=256.0,
                              n_features=3000, is_kitti=False)
    orc.track(gray, disp, flow, mask, [])
    tr.track(gray, disp.copy(), flow, mask.copy(), [])
    C = orc.cur
    kx, ky = sample_keypoints(h, w, seed)
    keep, cx, cy, fu, fv, dep = filter_static_sampled(kx, ky, mask, orc.depth, flow, 40.0)
    assert 0 < len(keep) < SAMPLE_N // 2, "the frame refuses most samples"
    assert np.array_equal(C.statKeysTmp, np.stack([kx[keep], ky[keep]], 1))
    assert len(tr.get("mvKeys")) > 0
    assert np.array_equal(tr.get("mvStatKeysTmp").reshape(-1, 2), C.statKeysTmp)
    assert np.array_equal(tr.get("mvCorres").reshape(-1, 2), C.corres)
    assert np.array_equal(tr.get("mvFlowNext").reshape(-1, 2), C.flowNext)
    assert np.array_equal(tr.get("mvStatDepthTmp"), C.statDepthTmp)
    # the option-I bounds would keep samples whose target lies left of or above the image
    tx, ty = kx + flow[ky.astype(int), kx.astype(int), 0], ky + flow[ky.astype(int), kx.astype(int), 1]
    assert ((tx <= 0) | (ty <= 0)).sum() > 100


def _omd_frame(t, seed):
    return make_sequence_frame(t, seed=seed, width=640, height=480, K=OMD_K)


def test_tracker_equals_oracle_pipeline(ctx):
    seed, n = 17, 11
    tr = capi.Tracker(ctx, use_sample_feature=1, sample_seed=seed, **OMD)
    orc = SampleOracleTracker(use_sample_feature=1, sample_seed=seed, width=640, height=480, K4=OMD_K, depth_factor=256.0, sf_mg_thres=0.02,
                              sf_ds_thres=0.99, n_features=3000, is_kitti=False, window_size=6, overlap_size=2)
    for t in range(n):
        f = _omd_frame(t, 3)
        T_ref = orc.track(f["gray"], f["depth_raw"], f["flow"], f["mask"], f["obj_ids"])
        d, m = f["depth_raw"].copy(), f["mask"].copy()
        T = tr.track(f["gray"], d, f["flow"], m, f["obj_ids"], writeback=True)
        assert np.abs(T - T_ref).max() <= 1e-4, f"frame {t}: Tcw"
        assert np.array_equal(m, orc.mask) and np.array_equal(d, orc.depth), f"frame {t}: write-back"
        _compare(tr, orc, t)
    assert len(orc.local_ba) >= 2 and int(tr.get("local_ba")[0]) == len(orc.local_ba)
    for name, ref in (("vmCameraPose", orc.map["cameraPose"]),):
        got = tr.map_get(name).reshape(-1, 4, 4)
        assert np.abs(got - np.asarray(ref)).max() <= 1e-4, name


def test_seeds(ctx):
    """the same seed twice gives the same run; another seed other static keys"""
    runs = []
    for seed in (5, 5, 6):
        tr = capi.Tracker(ctx, use_sample_feature=1, sample_seed=seed, **OMD)
        keys = []
        for t in range(3):
            f = _omd_frame(t, 1)
            tr.track(f["gray"], f["depth_raw"].copy(), f["flow"], f["mask"].copy(), f["obj_ids"])
            keys.append({name: tr.get(name).copy() for name in GET_NAMES})
        runs.append(keys)
    for a, b in zip(runs[0], runs[1]):
        for name in GET_NAMES:
            assert np.array_equal(a[name], b[name]), name
    assert not np.array_equal(runs[0][0]["mvStatKeysTmp"], runs[2][0]["mvStatKeysTmp"])


def test_batch_mixing_options_equals_separate_calls(ctx):
    """B = 4: sampling on (two seeds, one of them wrapping), off, and on with other thresholds; tracker 3 joins at step 2"""
    cfg = [dict(use_sample_feature=1, sample_seed=11), dict(use_sample_feature=0), dict(use_sample_feature=1, sample_seed=2 ** 32 - 2),
           dict(use_sample_feature=1, sample_seed=11, th_depth_bg=30.0)]
    tb = [capi.Tracker(ctx, **dict(OMD, **c)) for c in cfg]
    ts = [capi.Tracker(ctx, **dict(OMD, **c)) for c in cfg]
    pos = [0] * 4
    for step in range(8):
        members = [i for i in range(4) if not (i == 3 and step < 2)]
        fr = {i: _omd_frame(pos[i], i) for i in members}
        dev = {i: [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (fr[i]["gray"], fr[i]["depth_raw"], fr[i]["flow"], fr[i]["mask"])]
               for i in members}
        Tb = capi.track_tensors_batch([tb[i] for i in members], [dev[i][0] for i in members], [dev[i][1] for i in members], [dev[i][2] for i in members],
                                      [dev[i][3] for i in members], [fr[i]["obj_ids"] for i in members])
        for k, i in enumerate(members):
            g, d, fl, m = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (fr[i]["gray"], fr[i]["depth_raw"], fr[i]["flow"], fr[i]["mask"])]
            Ts = ts[i].track_tensors(g, d, fl, m, fr[i]["obj_ids"])
            assert np.array_equal(Tb[k], Ts), f"step {step} tracker {i}: Tcw"
            _assert_same(tb[i], ts[i], f"step {step} tracker {i}")
            assert torch.equal(dev[i][1], d) and torch.equal(dev[i][3], m), f"step {step} tracker {i}: write-back"
            pos[i] += 1
    for i in range(4):
        _assert_maps_same(tb[i], ts[i], f"tracker {i}")
    assert int(tb[0].get("local_ba")[0]) >= 1


def test_create_refusals(ctx):
    for kw in (dict(use_sample_feature=2), dict(use_sample_feature=-1), dict(use_sample_feature=1, width=0, height=0)):
        p = capi.TrackerParams()
        ctx.L.vdo_tracker_params_default(capi.C.byref(p))
        for k, v in dict(OMD, **kw).items():
            setattr(p, k, v)
        h = capi.C.c_void_p()
        assert ctx.L.vdo_tracker_create(ctx.h, capi.C.byref(p), capi.C.byref(h)) == ERR_ARG, kw
        assert not h.value, f"{kw}: nothing is handed out"
    capi.Tracker(ctx, width=0, height=0)                                  # a map-only handle without sampling is still accepted


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = os.path.join(ROOT, "tests", "shim_stub")
YAML = """%YAML:1.0
Camera.fx: 618.3587036132812
Camera.fy: 618.5924072265625
Camera.cx: 328.9866333007812
Camera.cy: 237.7507629394531
Camera.k1: 0.0
Camera.width: 640
Camera.height: 480
Camera.fps: 30.0
Camera.bf: 387.5744
Camera.RGB: 1
ChooseData: 1
DepthMapFactor: 256.0
ThDepthBG: 40.0
ThDepthOBJ: 25.0
MaxTrackPointBG: 1200
MaxTrackPointOBJ: 800
SFMgThres: 0.02
SFDsThres: 0.99
WINDOW_SIZE: 20
OVERLAP_SIZE: 4
UseSampleFeature: 1
SampleSeed: 4000000000
ORBextractor.nFeatures: 3000
ORBextractor.scaleFactor: 1.2
ORBextractor.nLevels: 8
ORBextractor.iniThFAST: 20
ORBextractor.minThFAST: 7
"""


def test_shim_runs_sampled_features_repeatably(tmp_path):
    subprocess.check_call(["make", "-C", SHIM, "shim_main"], stdout=subprocess.DEVNULL)
    n, w, h = 4, 640, 480
    outs = []
    for run in ("a", "b"):
        d = tmp_path / run
        d.mkdir()
        (d / "s.yaml").write_text(YAML)
        for t in range(n):
            f = _omd_frame(t, 2)
            b = str(d / f"f{t}")
            np.repeat(f["gray"][..., None], 3, -1).astype(np.uint8).tofile(b + ".rgb")
            f["depth_raw"].astype(np.float32).tofile(b + ".depth"); f["flow"].astype(np.float32).tofile(b + ".flow"); f["mask"].astype(np.int32).tofile(b + ".mask")
            np.array([len(f["obj_ids"])], np.int32).tofile(b + ".ngt"); np.array(f["obj_ids"], np.int32).tofile(b + ".gt")
        r = subprocess.run([os.path.join(SHIM, "shim_main"), str(d / "s.yaml"), str(d), str(n), str(w), str(h)], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        assert "SampleSeed: 4000000000" in r.stdout
        outs.append(d)
    files = sorted(p.name for p in outs[0].iterdir() if p.name.startswith("out_") or p.name.endswith("_out"))
    assert any(nm.startswith("out_") for nm in files)
    for nm in files:
        assert (outs[0] / nm).read_bytes() == (outs[1] / nm).read_bytes(), nm
    tr = SampleOracleTracker(use_sample_feature=1, sample_seed=4000000000, width=w, height=h, K4=OMD_K, depth_factor=256.0, sf_mg_thres=0.02,
                             sf_ds_thres=0.99, n_features=3000, is_kitti=False)
    poses = [np.array(l.split()[2:], np.float32).reshape(4, 4) for l in r.stdout.splitlines() if l.startswith("POSE")]
    for t in range(n):
        f = _omd_frame(t, 2)
        T = tr.track(f["gray"], f["depth_raw"], f["flow"], f["mask"], f["obj_ids"])
        assert np.abs(poses[t] - T).max() <= 1e-4, f"frame {t}"
