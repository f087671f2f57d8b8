"""Freezes the Map -> factor graph builder's output (vdo_tracker_graph_export, both modes) on seeded maps, and a whole config-3 tracker run,
into tests/golden/map_graph_*.npz.  tests/test_map_graph_gpu.py requires the current builder to give these arrays bit for bit.

The maps are pushed through vdo_tracker_map_push and are built to hold what the builder must get right: duplicate associations (two features
of a frame naming the same feature of the previous frame, whether or not that one already belongs to a tracklet), -1 associations, tracklets
that start before the window, a map whose length equals the window (the prior), and objects that appear, vanish and come back (smoothing edges
and the object-motion look-up of every dynamic observation).

Needs a CUDA device.  Re-run only when the builder's output is deliberately changed:
    python tests/golden/make_map_graph_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

HERE = os.path.dirname(os.path.abspath(__file__))
GRAPH_KEYS = ("se3", "pt", "prior_v", "prior_Z", "prior_w", "se3e_ij", "se3e_Z", "se3e_w", "se3e_delta", "obs_cp", "obs_z", "obs_w", "obs_delta",
              "ter_pph", "ter_w", "ter_delta")
# (name, frames, window); every map is exported in both modes
MAPS = (("map_graph_window.npz", 8, 8), ("map_graph_long.npz", 23, 8))
TRACKER_FRAMES = 40
OBJECTS = (1, 2, 3, 5)


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _pose(rng, scale):
    T = np.eye(4)
    T[:3, :3] = _rot(rng) if scale else np.eye(3)
    T[:3, 3] = rng.normal(size=3) * max(scale, 1e-3)
    return T.astype(np.float32)


def _assoc(rng, n, n_prev, prev_has):
    """associations of n features into the n_prev of the previous frame: -1 for about 15 %, and duplicates on purpose, some on a previous
    feature that already has a tracklet (prev_has), some on one that does not"""
    a = rng.integers(0, max(n_prev, 1), n).astype(np.int32) if n_prev else np.full(n, -1, np.int32)
    a[rng.random(n) < 0.15] = -1
    if n_prev and n >= 4:
        on = np.flatnonzero(prev_has[:n_prev]) if prev_has is not None else np.zeros(0, int)
        off = np.flatnonzero(~prev_has[:n_prev]) if prev_has is not None else np.arange(n_prev)
        for pool in (on, off):
            if len(pool):
                j = rng.choice(n, 2, replace=False)
                a[j] = int(rng.choice(pool))
    return a


def seeded_map(seed, n_frames):
    """frames of a map as the keyword arguments of Tracker.map_push"""
    rng = np.random.default_rng(seed)
    frames = []
    n_sta_prev = n_dyn_prev = 0
    has_sta = has_dyn = None
    for i in range(n_frames):
        n_sta, n_dyn = int(rng.integers(30, 60)), int(rng.integers(20, 45))
        present = [o for k, o in enumerate(OBJECTS) if (i // (2 + k)) % 3 != 1]       # object k vanishes for 2 + k frames out of every 3 (2 + k)
        f = dict(feat_sta=rng.uniform([0, 0], [1242, 375], (n_sta, 2)), dep_sta=rng.uniform(1, 40, n_sta), p3d_sta=rng.normal(size=(n_sta, 3)) * 10,
                 feat_dyn=rng.uniform([0, 0], [1242, 375], (n_dyn, 2)), dep_dyn=rng.uniform(1, 25, n_dyn), p3d_dyn=rng.normal(size=(n_dyn, 3)) * 10,
                 camera_pose=_pose(rng, 1.0))
        if i > 0:
            f["asso_sta"] = _assoc(rng, n_sta, n_sta_prev, has_sta)
            f["asso_dyn"] = _assoc(rng, n_dyn, n_dyn_prev, has_dyn)
            lab = rng.choice(np.array(OBJECTS + (-1, 4), np.int32), n_dyn)                 # 4 never has a motion; -1 = no object
            f["feat_label"] = lab
            f["rigid_motion"] = np.stack([_pose(rng, 0.5)] + [_pose(rng, 0.2) for _ in present])
            f["rm_label"] = np.array([0] + present, np.int32)
            has_sta, has_dyn = f["asso_sta"] != -1, f["asso_dyn"] != -1
        n_sta_prev, n_dyn_prev = n_sta, n_dyn
        frames.append(f)
    return frames


def push_map(ctx, frames, window):
    from vdo_slam_b200 import capi
    tr = capi.Tracker(ctx, width=0, height=0, window_size=window, overlap_size=4)
    for f in frames:
        tr.map_push(**f)
    return tr


def flat_frames(frames):
    """the pushed frames as flat arrays (the golden file keeps the map itself, so the test does not depend on this generator's RNG)"""
    out = {}
    for k in ("feat_sta", "dep_sta", "p3d_sta", "feat_dyn", "dep_dyn", "p3d_dyn", "camera_pose", "asso_sta", "asso_dyn", "feat_label", "rigid_motion", "rm_label"):
        rows = [np.asarray(f[k]) for f in frames if k in f]
        dt = np.int32 if k in ("asso_sta", "asso_dyn", "feat_label", "rm_label") else np.float32
        out["in_" + k] = np.concatenate([r.reshape(len(r), -1) if r.ndim > 1 else r.reshape(-1, 1) for r in rows]).astype(dt)
        out["in_n_" + k] = np.array([len(r) for r in rows], np.int32)
    return out


def unflat_frames(z):
    """inverse of flat_frames on a loaded golden file"""
    n_frames = len(z["in_n_feat_sta"])
    frames = [dict() for _ in range(n_frames)]
    for k in ("feat_sta", "dep_sta", "p3d_sta", "feat_dyn", "dep_dyn", "p3d_dyn", "camera_pose", "asso_sta", "asso_dyn", "feat_label", "rigid_motion", "rm_label"):
        cnt = z["in_n_" + k]
        first = n_frames - len(cnt)
        off = np.concatenate([[0], np.cumsum(cnt)])
        for j in range(len(cnt)):
            a = z["in_" + k][off[j]:off[j + 1]]
            frames[first + j][k] = a.reshape(-1) if a.shape[1] == 1 else a
    for f in frames:
        f["camera_pose"] = f["camera_pose"].reshape(4, 4)
        if "rigid_motion" in f:
            f["rigid_motion"] = f["rigid_motion"].reshape(-1, 4, 4)
    return frames


def tracker_record(trs):
    """what the whole-tracker test compares: poses, the map's camera poses and motions, static points (digest) and the windowed-BA counters"""
    out = {}
    for i, tr in enumerate(trs):
        out[f"t{i}_Tcw"] = tr["Tcw"]
        t = tr["tracker"]
        out[f"t{i}_vmCameraPose"] = t.map_get("vmCameraPose")
        out[f"t{i}_vmRigidMotion"] = t.map_get("vmRigidMotion")
        out[f"t{i}_vp3DPointSta_sha256"] = np.array(hashlib.sha256(t.map_get("vp3DPointSta").tobytes()).hexdigest())
        out[f"t{i}_local_ba"] = t.get("local_ba")
    return out


def run_tracker(ctx, frames_of_seed, n_frames):
    import torch
    from vdo_slam_b200 import capi
    dev = torch.device("cuda", 0)
    tr = capi.Tracker(ctx, n_features=3000)
    Ts = []
    for f in frames_of_seed[:n_frames]:
        h = [torch.from_numpy(f[k]).to(dev) for k in ("gray", "depth_raw", "flow", "mask")]
        Ts.append(tr.track_tensors(*h, f["obj_ids"], writeback=False))
    return {"tracker": tr, "Tcw": np.stack(Ts)}


def main():
    from bench import sequence_frames
    from vdo_slam_b200 import capi
    ctx = capi.Context(0)
    for k, (name, n, window) in enumerate(MAPS):
        frames = seeded_map(100 + k, n)
        tr = push_map(ctx, frames, window)
        out = flat_frames(frames)
        out["window"] = np.int32(window)
        for mode in (0, 1):
            g = tr.graph_export(mode)
            for key in GRAPH_KEYS:
                out[f"m{mode}_{key}"] = g[key]
        np.savez_compressed(os.path.join(HERE, name), **out)
        print(name, {m: len(out[f"m{m}_obs_w"]) for m in (0, 1)}, "observations;", len(out["m1_ter_w"]), "ternary;", len(out["m0_prior_w"]), "prior")
    seq = sequence_frames(TRACKER_FRAMES, 0)
    rec = tracker_record([run_tracker(ctx, seq, TRACKER_FRAMES)])
    np.savez_compressed(os.path.join(HERE, "map_graph_tracker.npz"), frames=np.int32(TRACKER_FRAMES), seed=np.int32(0), **rec)
    print("map_graph_tracker.npz local_ba", rec["t0_local_ba"].tolist())


if __name__ == "__main__":
    main()
