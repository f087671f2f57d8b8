"""Full-batch optimisation of several graphs / trackers in one call: vdo_graph_optimize_batch with PCG-path graphs (their trial steps as one
set of launches, one read-back per PCG chunk for all of them) and vdo_tracker_batch_optimize_batch.

Every graph of a batch must end where its own vdo_graph_optimize takes it: the same LM iterations, trials and PCG iterations.  The
solver sums the tile accumulators and chi2 with fp64 atomics across CTAs, so two solves of one PCG graph already differ in the last bits
(test_graph_batch_gpu.py); estimates and chi2 histories are compared at the tolerance that spread allows, not bit for bit.  The tracker
maps are float32 and are compared to 1e-5."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_batch_graph, make_sequence_frame, iso_inv, iso_mul, iso_R, iso_t, PARTIAL_BATCH

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import ba_shapes  # noqa: E402
import make_map_graph_golden as mg  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
KW = dict(max_iterations=60, gain_threshold=1e-4)


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def _pcg_graphs():
    """PCG-path graphs of different sizes and convergence: synthetic sequences with objects, and the tiled PCG shapes of ba_shapes"""
    gs = [make_batch_graph(n_frames=f, n_objects=o, n_static=s, n_dynamic=dy, seed=seed)
          for f, o, s, dy, seed in ((12, 1, 400, 80, 3), (20, 2, 1500, 300, 7), (8, 1, 150, 40, 11), (30, 3, 3000, 600, 5))]
    gs.append(make_batch_graph(n_frames=10, n_objects=1, n_static=200, n_dynamic=60, seed=12, odo_sigma_t=0.5, odo_sigma_r=0.2))
    for name in ("chains_short", "precond_paths"):
        gs.append(ba_shapes.SHAPES[name]()[0])
    return gs


def _separate(ctx, gs, **kw):
    out = []
    for g in gs:
        G = capi.BatchGraph(ctx, g)
        out.append((G.optimize(**kw), G.vertices()))
    return out


def _check(r, est, r0, est0, what):
    for k in ("iterations", "trials"):
        assert r[k] == r0[k], f"{what}: {k} {r[k]} != {r0[k]}"
    # a graph that needs thousands of PCG iterations can cross its convergence test one iteration earlier or later on atomics-level
    # differences, in two separate solves as well as in a batch
    assert abs(r["pcg_iterations"] - r0["pcg_iterations"]) <= r0["pcg_iterations"] // 1000, f"{what}: pcg_iterations {r['pcg_iterations']} != {r0['pcg_iterations']}"
    np.testing.assert_allclose(r["chi2"], r0["chi2"], rtol=1e-9, err_msg=what)
    assert np.abs(est[0] - est0[0]).max() <= 1e-8 and np.abs(est[1] - est0[1]).max() <= 1e-8, what


@pytest.fixture(scope="module")
def pcg_ref(ctx):
    gs = _pcg_graphs()
    ref = _separate(ctx, gs, **KW)
    for g in gs:
        info = capi.BatchGraph(ctx, g).solver_info()
        assert info["tiled"] == 1 and info["dense"] == 0
    assert len({r0["pcg_iterations"] for r0, _ in ref}) >= 4 and len({r0["iterations"] for r0, _ in ref}) >= 3
    return gs, ref


@pytest.mark.parametrize("pick", [(0, 1), (2, 4, 5), (0, 1, 2, 3, 4, 5, 6, 1)])
def test_pcg_batch_equals_separate(ctx, pcg_ref, pick):
    gs, ref = pcg_ref
    Gs = [capi.BatchGraph(ctx, gs[i]) for i in pick]
    rs = capi.optimize_batch(Gs, **KW)
    for i, G, r in zip(pick, Gs, rs):
        _check(r, G.vertices(), ref[i][0], ref[i][1], f"graph {i}")
    singles = [ref[i][0]["kernel_launches"] for i in pick]
    assert rs[0]["kernel_launches"] < sum(singles)


def test_mixed_dense_and_pcg_batch(ctx, pcg_ref):
    gs, ref = pcg_ref
    dense = [make_batch_graph(n_frames=20, n_objects=0, n_static=n, n_dynamic=0, seed=s, consts=PARTIAL_BATCH) for s, n in ((30, 300), (31, 900))]
    ref_d = _separate(ctx, dense, **KW)
    order = [("d", 0), ("p", 1), ("d", 1), ("p", 3), ("p", 0)]
    Gs = [capi.BatchGraph(ctx, dense[i] if k == "d" else gs[i]) for k, i in order]
    assert [G.solver_info()["dense"] for G in Gs] == [1, 0, 1, 0, 0]
    rs = capi.optimize_batch(Gs, **KW)
    for (k, i), G, r in zip(order, Gs, rs):
        r0, est0 = ref_d[i] if k == "d" else ref[i]
        _check(r, G.vertices(), r0, est0, f"{k}{i}")


def test_config4_golden_inside_a_batch(ctx):
    import ast
    d = np.load(os.path.join(HERE, "golden", "ba_config4.npz"))
    g = make_batch_graph(**ast.literal_eval(str(d["cfg"])))
    other = make_batch_graph(n_frames=20, n_objects=2, n_static=1500, n_dynamic=300, seed=7)
    Gs = [capi.BatchGraph(ctx, g), capi.BatchGraph(ctx, other)]
    assert Gs[0].solver_info()["dense"] == 0
    r = capi.optimize_batch(Gs, max_iterations=300, gain_threshold=1e-4)[0]
    se3, pt = Gs[0].vertices()
    assert r["iterations"] == int(d["iters"]) == 35
    np.testing.assert_allclose(r["chi2"][:36], d["chi2"], rtol=1e-6)
    dd = iso_mul(iso_inv(se3), d["se3"])
    assert np.abs(iso_t(dd)).max() <= 1e-5 and np.abs(iso_R(dd) - np.eye(3)).max() <= 1e-5


# ---- tracker level ----
MAP_NAMES = ("vmCameraPose", "vmCameraPose_RF", "vmRigidMotion", "vmRigidMotion_RF", "vp3DPointSta", "vp3DPointDyn")
STAT_KEYS = ("iterations", "trials", "pcg_iterations")


def _maps(t):
    return {k: t.map_get(k) for k in MAP_NAMES}


def _same_maps(a, b, what):
    for k in MAP_NAMES:
        assert a[k].shape == b[k].shape, f"{what}: {k}"
        np.testing.assert_allclose(a[k], b[k], rtol=0, atol=1e-5, err_msg=f"{what}: {k}")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(scope="module")
def tracked(ctx):
    """two identical sets of three config-3-style trackers (seeds 0..2, 10 / 13 / 16 frames, windows of 6 with overlap 2), both fed
    through track_tensors_batch"""
    lens = (10, 13, 16)
    frames = [[make_sequence_frame(t, seed=s) for t in range(n)] for s, n in enumerate(lens)]
    sets = [[capi.Tracker(ctx, n_features=3000, window_size=6, overlap_size=2) for _ in lens] for _ in range(2)]
    for t in range(max(lens)):
        live = [i for i, n in enumerate(lens) if t < n]
        for trs in sets:
            fr = [frames[i][t] for i in live]
            ins = [[_dev(f[k]) for k in ("gray", "depth_raw", "flow", "mask")] for f in fr]
            capi.track_tensors_batch([trs[i] for i in live], *[[x[k] for x in ins] for k in range(4)], [f["obj_ids"] for f in fr])
    for a, b in zip(*sets):
        _same_maps(_maps(a), _maps(b), "twins after tracking")
    return sets


@pytest.mark.parametrize("mode", [1, 0])
def test_tracker_batch_equals_one_by_one(ctx, tracked, mode):
    batched, twins = tracked
    rs = capi.batch_optimize_trackers(batched, mode)
    r1 = [t.batch_optimize(mode) for t in twins]
    for i, (a, b, r, r0) in enumerate(zip(batched, twins, rs, r1)):
        _same_maps(_maps(a), _maps(b), f"mode {mode} tracker {i}")
        for k in STAT_KEYS:
            assert r[k] == r0[k], f"mode {mode} tracker {i}: {k}"
        assert r["sizes"] == r0["sizes"]
    if mode == 1:
        assert all(r["pcg_iterations"] > 0 for r in rs)


def _pushed(ctx, z):
    tr = capi.Tracker(ctx, width=0, height=0, window_size=int(z["window"]), overlap_size=4)
    for f in mg.unflat_frames(z):
        tr.map_push(**f)
    return tr


@pytest.mark.parametrize("mode", [1, 0])
def test_map_only_trackers(ctx, mode):
    """the pushed golden maps; a map whose full-batch graph the solver refuses (duplicate associations give a landmark two successors)
    is refused the same way inside the batch, and the batch then changes no map"""
    zs = [np.load(os.path.join(HERE, "golden", name)) for name, _, _ in mg.MAPS]
    a = [_pushed(ctx, z) for z in zs]
    b = [_pushed(ctx, z) for z in zs]
    kw = dict(max_iterations=50, gain_threshold=1e-4)
    r1, ok = [], []
    for t in b:
        try:
            r1.append(t.batch_optimize(mode, **kw)); ok.append(True)
        except capi.VdoError:
            r1.append(None); ok.append(False)
    if not all(ok):
        before = [_maps(t) for t in a]
        with pytest.raises(capi.VdoError, match=r"\(-3\)"):
            capi.batch_optimize_trackers(a, mode, **kw)
        for t, m in zip(a, before):
            for k in MAP_NAMES:
                assert np.array_equal(t.map_get(k), m[k])
    keep = [i for i in range(len(a)) if ok[i]]
    assert mode == 1 or len(keep) == len(a)
    if not keep:
        return
    rs = capi.batch_optimize_trackers([a[i] for i in keep], mode, **kw)
    for i, r in zip(keep, rs):
        _same_maps(_maps(a[i]), _maps(b[i]), f"pushed map {i}, mode {mode}")
        for k in STAT_KEYS:
            assert r[k] == r1[i][k]


def test_refusals_change_no_tracker(ctx):
    zs = [np.load(os.path.join(HERE, "golden", name)) for name, _, _ in mg.MAPS]
    ts = [_pushed(ctx, z) for z in zs]
    short = capi.Tracker(ctx, width=0, height=0, window_size=8, overlap_size=4)
    short.map_push(**mg.unflat_frames(zs[0])[0])                  # one frame: too short for either mode
    win = capi.Tracker(ctx, width=0, height=0, window_size=30, overlap_size=4)
    for f in mg.unflat_frames(zs[0]):
        win.map_push(**f)                                          # 8 frames: enough for mode 1, too short for a 30-frame window
    ctx2 = capi.Context(0)
    other = _pushed(ctx2, zs[0])
    everyone = ts + [short, win, other]
    before = [_maps(t) for t in everyone]
    L = ctx.L
    o = capi.LMOptions()
    L.vdo_lm_options_default(C.byref(o))

    def call(handles, mode=1, n=None, opt=None):
        arr = (C.c_void_p * max(len(handles), 1))(*handles)
        return L.vdo_tracker_batch_optimize_batch(arr, C.c_int(len(handles) if n is None else n), C.c_int(mode), opt, None, None)

    h = [t.h_.value for t in ts]
    assert call([h[0], h[1], h[0]]) == -2                          # repeated tracker
    assert b"repeats" in L.vdo_tracker_last_error(ts[0].h_)
    assert call([h[0], None, h[1]]) == -2                          # NULL entry
    assert call([h[0], h[1]], n=0) == -2                           # n < 1
    assert L.vdo_tracker_batch_optimize_batch(None, C.c_int(2), C.c_int(1), None, None, None) == -2
    assert call([h[0], h[1]], mode=2) == -2                        # no such mode
    assert call([h[0], other.h_.value]) == -2                      # another context
    assert call([h[0], short.h_.value, h[1]]) == -4                # VDO_ERR_STATE: map too short
    assert call([h[0], win.h_.value], mode=0, opt=C.byref(o)) == -4
    with pytest.raises(capi.VdoError):
        capi.batch_optimize_trackers([], 1)
    with pytest.raises(capi.VdoError):
        capi.batch_optimize_trackers([ts[0], ts[0]], 1)
    for t, m in zip(everyone, before):
        _same_maps(_maps(t), m, "after the refusals")
        for k in MAP_NAMES:
            assert np.array_equal(t.map_get(k), m[k])
    # the trackers still optimise normally afterwards
    rs = capi.batch_optimize_trackers([ts[0], ts[1]], 0)
    assert all(r["iterations"] >= 1 for r in rs)
