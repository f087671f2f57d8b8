"""The device Map -> factor graph builder (map_graph.cu): tracklet tables kept per frame, graph assembly for the windowed and the full
batch, bit for bit against what the host builder it replaced produced (tests/golden/map_graph_*.npz, tests/golden/make_map_graph_golden.py)."""
import os
import sys

import numpy as np
import pytest
import torch

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_sequence_frame

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_map_graph_golden as mg  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def _golden(name):
    return np.load(os.path.join(HERE, "golden", name))


def _check_tables(tr, asso, labels, n_feat, what):
    """the tracker's tables of both kinds against vdo_tracklets_build on the full history"""
    for kind in (0, 1):
        tab = tr.tracklets(kind)
        rows = asso[kind]
        ref, oid = capi.tracklets_build(rows, labels if kind == 1 else None) if rows else ([], [])
        n_trk = len(tab["len"])
        assert n_trk == len(ref), f"{what} kind {kind}: tracklet count"
        off = np.concatenate([[0], np.cumsum(n_feat[kind])])
        got = [[(int(tab["head_frame"][t]), int(tab["head_feat"][t]))] + [None] * (int(tab["len"][t]) - 1) for t in range(n_trk)]
        for f in range(1, len(n_feat[kind])):
            for j in range(n_feat[kind][f]):
                t = int(tab["trk"][off[f] + j])
                if t == -1:
                    continue
                p = int(tab["pos"][off[f] + j])
                assert got[t][p] is None, f"{what} kind {kind}: two entries at one position"
                got[t][p] = (f, j)
        assert got == [list(r) for r in ref], f"{what} kind {kind}: tracklets"
        if kind == 1:
            assert tab["obj_lab"].tolist() == list(oid), f"{what}: ObjLab"
        for t in range(n_trk):                       # the entry before each one
            for p in range(1, len(got[t])):
                f, j = got[t][p]
                assert (int(tab["prev_frame"][off[f] + j]), int(tab["prev_feat"][off[f] + j])) == got[t][p - 1], f"{what} kind {kind}: prev"


def _push_golden(ctx, z, upto=None):
    frames = mg.unflat_frames(z)
    tr = capi.Tracker(ctx, width=0, height=0, window_size=int(z["window"]), overlap_size=4)
    for f in frames[:upto]:
        tr.map_push(**f)
    return tr, frames


@pytest.mark.parametrize("name", [m[0] for m in mg.MAPS])
def test_tables_of_pushed_maps(ctx, name):
    z = _golden(name)
    frames = mg.unflat_frames(z)
    tr = capi.Tracker(ctx, width=0, height=0, window_size=int(z["window"]), overlap_size=4)
    asso, labels, n_feat = ([], []), [], ([], [])
    dup_set = dup_unset = 0
    for i, f in enumerate(frames):
        tr.map_push(**f)
        n_feat[0].append(len(f["feat_sta"])); n_feat[1].append(len(f["feat_dyn"]))
        if i > 0:
            for kind, key in ((0, "asso_sta"), (1, "asso_dyn")):
                a = f[key]
                asso[kind].append(a)
                v, c = np.unique(a[a != -1], return_counts=True)
                if i > 1:
                    prev_has = asso[kind][-2] != -1
                    dup_set += int(np.sum(prev_has[v[c > 1]])); dup_unset += int(np.sum(~prev_has[v[c > 1]]))
            labels.append(f["feat_label"])
        _check_tables(tr, asso, labels, n_feat, f"{name} frame {i}")
    assert dup_set > 0 and dup_unset > 0, "the map holds duplicate associations on both kinds of previous feature"
    assert any((f["asso_sta"] == -1).any() for f in frames[1:])


@pytest.mark.parametrize("name", [m[0] for m in mg.MAPS])
@pytest.mark.parametrize("mode", [0, 1])
def test_graph_bit_identical_to_host_builder(ctx, name, mode):
    z = _golden(name)
    tr, frames = _push_golden(ctx, z)
    g = tr.graph_export(mode)
    for k in mg.GRAPH_KEYS:
        ref = z[f"m{mode}_{k}"]
        assert g[k].dtype == ref.dtype and g[k].shape == ref.shape, (k, g[k].shape, ref.shape)
        assert np.array_equal(g[k], ref), f"{name} mode {mode}: {k}"
    n, w = len(frames), int(z["window"])
    if mode == 0:
        assert (len(g["prior_v"]) == 1) == (n == w)
        if n > w:                                           # chains whose head lies before the window are left out
            assert len(g["obs_w"]) < sum(len(f["feat_sta"]) for f in frames[n - w:])
    else:
        assert len(g["ter_pph"]) > 0 and len(g["se3e_w"]) > n - 1            # ternary and smoothing edges present


def test_bad_association_refuses_graphs(ctx):
    z = _golden("map_graph_window.npz")
    frames = mg.unflat_frames(z)
    tr = capi.Tracker(ctx, width=0, height=0, window_size=4, overlap_size=2)
    for i, f in enumerate(frames[:5]):
        if i == 3:
            f = dict(f, asso_sta=f["asso_sta"].copy())
            f["asso_sta"][0] = len(frames[2]["feat_sta"])          # one past the previous frame's features
        tr.map_push(**f)
    with pytest.raises(capi.VdoError, match=r"-2"):
        tr.graph_export(0)


def test_tables_of_tracked_sequence(ctx):
    """after every frame of a tracked sequence the tables equal vdo_tracklets_build on the map's whole history"""
    tr = capi.Tracker(ctx, window_size=6, overlap_size=2)
    asso, labels, n_feat = ([], []), [], ([], [])
    for t in range(9):
        f = make_sequence_frame(t, seed=4)
        tr.track(f["gray"], f["depth_raw"].copy(), f["flow"], f["mask"].copy(), f["obj_ids"])
        n_feat[0].append(len(tr.get("mvStatKeysTmp")) // 2); n_feat[1].append(len(tr.get("mvObjKeys")) // 2)
        if t > 0:
            asso[0].append(tr.get("nStaInlierID")); asso[1].append(tr.get("nDynInlierID")); labels.append(tr.get("vObjLabel"))
        _check_tables(tr, asso, labels, n_feat, f"frame {t}")
    assert int(tr.get("local_ba")[0]) >= 1


def _record(trs, Ts):
    return mg.tracker_record([{"tracker": tr, "Tcw": T} for tr, T in zip(trs, Ts)])


def test_whole_tracker_batch_and_golden(ctx):
    """config-3 sequences over 40 frames (windows at f_id 19 and 35): separate and batched trackers (B = 4, staggered starts) agree bit for
    bit, and the first sequence reproduces the record of the host builder"""
    from bench import sequence_frames
    n, B = mg.TRACKER_FRAMES, 4
    gz = _golden("map_graph_tracker.npz")
    seqs = [sequence_frames(n, seed) for seed in range(B)]
    held = [[tuple(torch.from_numpy(f[k]).to(DEV) for k in ("gray", "depth_raw", "flow", "mask")) + (f["obj_ids"],) for f in s] for s in seqs]
    del seqs
    sep = [capi.Tracker(ctx, n_features=3000) for _ in range(B)]
    bat = [capi.Tracker(ctx, n_features=3000) for _ in range(B)]
    Ts, Tb = [[] for _ in range(B)], [[] for _ in range(B)]
    for step in range(n + B - 1):
        members = [i for i in range(B) if 0 <= step - i < n]                 # tracker i starts at step i
        for i in members:
            h = held[i][step - i]
            Ts[i].append(sep[i].track_tensors(*h[:4], h[4], writeback=False))
        T = capi.track_tensors_batch([bat[i] for i in members], *[[held[i][step - i][k] for i in members] for k in range(5)], writeback=False)
        for q, i in enumerate(members):
            Tb[i].append(T[q])
    rs, rb = _record(sep, [np.stack(x) for x in Ts]), _record(bat, [np.stack(x) for x in Tb])
    for k in rs:
        assert np.array_equal(rs[k], rb[k]), f"separate vs batched: {k}"
    assert rs["t0_local_ba"].tolist()[0] == 2
    for k in gz.files:
        if k.startswith("t0_"):
            assert np.array_equal(rs[k], gz[k]), f"against the host builder's record: {k}"


def test_graph_assembly_launches_once_per_call(ctx):
    """torch.profiler on a window step of 8 trackers: each graph-assembly kernel runs once for the whole call"""
    from torch.profiler import ProfilerActivity, profile
    B = 8
    frames = [make_sequence_frame(t, seed=1) for t in range(20)]
    held = [tuple(torch.from_numpy(f[k]).to(DEV) for k in ("gray", "depth_raw", "flow", "mask")) for f in frames]
    trs = [capi.Tracker(ctx) for _ in range(B)]
    for t in range(20):
        step = lambda: capi.track_tensors_batch(trs, *[[held[t][k]] * B for k in range(4)], [frames[t]["obj_ids"]] * B, writeback=False)
        if t < 19:
            step()
            continue
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
    assert all(int(tr.get("local_ba")[0]) == 1 for tr in trs)
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    for k in ("k_mark_heads", "k_decide", "k_write", "k_tracklets_push"):
        assert sum(k in nm for nm in names) == 1, (k, [nm for nm in names if k in nm])
