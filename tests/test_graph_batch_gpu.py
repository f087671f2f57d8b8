"""vdo_graph_optimize_batch on the GPU: every graph of a batch ends where its own vdo_graph_optimize takes it, and a tracker batch whose
windowed optimisations fire on the same call (solved by one vdo_graph_optimize_batch) ends where separate trackers end.

The single-graph solver sums chi2 and the tile accumulators with fp64 atomics across CTAs, so two solves of one graph may differ in the
last bits: separate and batched solves are compared to 1e-10 (estimates) and rtol 1e-12 (chi2 history), not bit for bit."""
import numpy as np
import pytest
import torch

from oracle import pyoracle as po
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_batch_graph, make_sequence_frame, PARTIAL_BATCH

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
KW = dict(max_iterations=100, gain_threshold=1e-3)      # the windowed optimiser's cap and gain threshold


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def _window_graphs():
    """8 sliding windows (20 frames, 300-3000 static points), a 6-camera graph, and one window whose pointxyz edges are listed backwards
    (vertex numbers decrease along a landmark's edge list: no band, so the dense path forms the static term point by point)"""
    gs = [make_batch_graph(n_frames=20, n_objects=0, n_static=n, n_dynamic=0, seed=s, consts=PARTIAL_BATCH)
          for s, n in zip(range(30, 38), (300, 3000, 800, 1500, 2200, 450, 2600, 1000))]
    gs.append(make_batch_graph(n_frames=6, n_objects=0, n_static=500, n_dynamic=0, seed=40, consts=PARTIAL_BATCH))
    g = make_batch_graph(n_frames=20, n_objects=0, n_static=1200, n_dynamic=0, seed=41, consts=PARTIAL_BATCH)
    rev = dict(g)
    for k in ("obs_cp", "obs_z", "obs_w", "obs_delta"):
        rev[k] = np.ascontiguousarray(g[k][::-1])
    gs.append(rev)
    return gs


def _pose_err(a, b):
    return np.abs(a - b).max(axis=1)


def _check_against(r, est, r0, est0, atol, rtol=1e-12):
    assert r["iterations"] == r0["iterations"] and r["trials"] == r0["trials"]
    np.testing.assert_allclose(r["chi2"], r0["chi2"], rtol=rtol)
    assert np.abs(est[0] - est0[0]).max() <= atol and np.abs(est[1] - est0[1]).max() <= atol


def test_dense_batch_matches_separate_and_oracle(ctx):
    gs = _window_graphs()
    sep = []
    for g in gs:
        G = capi.BatchGraph(ctx, g)
        assert G.solver_info()["dense"] == 1
        sep.append((G.optimize(**KW), G.vertices()))
    Gs = [capi.BatchGraph(ctx, g) for g in gs]
    assert Gs[-1].solver_info()["band_width"] == 0 and Gs[0].solver_info()["band_width"] > 0
    rs = capi.optimize_batch(Gs, **KW)
    for i, (g, G, r, (r0, est0)) in enumerate(zip(gs, Gs, rs, sep)):
        est = G.vertices()
        _check_against(r, est, r0, est0, 1e-10)
        assert r["pcg_iterations"] == 0
        ro = po.ba_optimize(g, max_iters=KW["max_iterations"], gain_threshold=KW["gain_threshold"])
        assert r["iterations"] == ro["iters"], f"graph {i}"
        assert max(_pose_err(est[0], ro["se3"])) <= 1e-8 and np.abs(est[1] - ro["pt"]).max() <= 1e-8, f"graph {i}"
    # every step of all the dense graphs is one set of launches
    singles = [r0["kernel_launches"] for r0, _ in sep]
    assert rs[0]["kernel_launches"] <= 2 * max(singles) and rs[0]["kernel_launches"] < sum(singles)


def test_mixed_dense_and_pcg_batch(ctx):
    gs = _window_graphs()[:3]
    gs.insert(1, make_batch_graph(n_frames=12, n_objects=1, n_static=400, n_dynamic=80, seed=3))    # dynamic objects: PCG path
    sep = []
    for g in gs:
        G = capi.BatchGraph(ctx, g)
        sep.append((G.optimize(**KW), G.vertices()))
    Gs = [capi.BatchGraph(ctx, g) for g in gs]
    assert [G.solver_info()["dense"] for G in Gs] == [1, 0, 1, 1]
    rs = capi.optimize_batch(Gs, **KW)
    for i, (G, r, (r0, est0)) in enumerate(zip(Gs, rs, sep)):
        if i == 1:
            # the PCG graph: its atomics-level differences pass through every PCG iteration of 34 LM iterations, so two separate
            # solves of it already differ by about 1e-11 in chi2
            _check_against(r, G.vertices(), r0, est0, 1e-8, rtol=1e-9)
        else:
            _check_against(r, G.vertices(), r0, est0, 1e-10)
    assert rs[1]["pcg_iterations"] > 0


# ---- tracker batch: four sequences with one window setting (their windows fire on the same calls) and one with another ----
SEQS = [dict(seed=s, window_size=6, overlap_size=2) for s in range(4)] + [dict(seed=4, window_size=8, overlap_size=3)]
N_FRAMES = 14
GET_NAMES = ("Tcw", "mVelocity", "mvKeys", "mvStatKeys", "mvStatDepth", "mvCorres", "mvObjKeys", "mvObjDepth", "vObjLabel", "nModLabel",
             "vObjMod", "max_id", "f_id", "local_ba")
MAP_NAMES = ("vmCameraPose", "vmCameraPose_RF", "vmRigidMotion", "vmRigidMotion_RF", "vmRigidCentre", "n_per_frame", "vp3DPointSta",
             "vp3DPointDyn", "vnRMLabel", "n_frames")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_tracker_batch_windows_equal_separate_trackers(ctx):
    frames = [[make_sequence_frame(t, seed=s["seed"]) for t in range(N_FRAMES)] for s in SEQS]
    mk = lambda s: capi.Tracker(ctx, window_size=s["window_size"], overlap_size=s["overlap_size"])   # noqa: E731
    tb, ts = [mk(s) for s in SEQS], [mk(s) for s in SEQS]
    B = len(SEQS)
    for t in range(N_FRAMES):
        fr = [frames[i][t] for i in range(B)]
        ins_b = [[_dev(f[k]) for k in ("gray", "depth_raw", "flow", "mask")] for f in fr]
        ins_s = [[_dev(f[k]) for k in ("gray", "depth_raw", "flow", "mask")] for f in fr]
        Tb = capi.track_tensors_batch(tb, *[[x[k] for x in ins_b] for k in range(4)], [f["obj_ids"] for f in fr])
        for i in range(B):
            Ts = ts[i].track_tensors(*ins_s[i], fr[i]["obj_ids"])
            assert np.array_equal(Tb[i], Ts), f"frame {t} sequence {i}: Tcw"
            for name in GET_NAMES:
                np.testing.assert_array_equal(tb[i].get(name), ts[i].get(name), err_msg=f"frame {t} sequence {i}: {name}")
    for i in range(B):
        for name in MAP_NAMES:
            np.testing.assert_array_equal(tb[i].map_get(name), ts[i].map_get(name), err_msg=f"sequence {i}: {name}")
    runs = [int(tb[i].get("local_ba")[0]) for i in range(B)]
    assert runs == [3, 3, 3, 3, 2]                       # windows at f_id 5, 9, 13 (6/2) and 7, 12 (8/3)
    assert all(tb[i].get("stage_ms")[8] > 0 for i in range(B))
