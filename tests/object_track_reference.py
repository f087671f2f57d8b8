"""Host route of the object step with scene flow and object tracking that vdo_obj_track_batch_dev (capi.ObjectMotion.track) runs on the
device: the resident frame's vdo_frame_sample_objects on the last frame, the current-frame look-up at each flow target in numpy,
capi.scene_flow (GetSceneFlowObj), capi.dyn_obj_tracking (DynObjTracking) on the samples of the object slots, then for the dynamic objects
capi.init_model_batch with the motion model looked up by ID, the min_inliers gate, capi.pose_opt_flow2 (mode 1) and H = Tcw_cur^-1 X.
Its result, given the same inputs, must equal the device call's bit for bit."""
import numpy as np

from tests.object_motion_reference import EYE, inv4, mul4, unproject_world, velocity
from vdo_slam_b200 import capi

f32 = np.float32


def majority(v):
    """tracking_ops.cu majority_label: the most frequent value, ties to the smaller"""
    u, c = np.unique(np.asarray(v), return_counts=True)
    return int(u[np.argmax(c)]) if len(u) else 0


def reset_state(M):
    """the previous-result arrays of one pair at the start of a sequence"""
    return dict(label=np.full(M, -1, np.int32), id=np.full(M, -1, np.int32), stat=np.zeros(M, np.int32), H=np.tile(EYE, (M, 1, 1)),
                max_id=np.int32(1))


def host_track(ctx, depth, flow, mask, depth_cur, mask_cur, K, M, Tcw_last=None, Tcw_cur=None, prev=None, step=4, th_depth_obj=25.0,
               sf_mg_thres=0.12, sf_ds_thres=0.3, shrink=(25, 50), iters=500, thr=0.4, conf=0.98, min_inliers=50, quirk=1):
    """One pair.  depth, flow, mask: the last frame; depth_cur, mask_cur: the current frame (masks within int32); K (4,); M: object slots;
    Tcw_last, Tcw_cur: None or 4x4; prev: None or one pair's row of the previous result (label, id, stat, H, max_id).
    Returns dict of numpy arrays in the layout of one pair of ObjectMotion.track's result (samples: n_samples rows)."""
    h, w = depth.shape
    Tl = EYE if Tcw_last is None else np.asarray(Tcw_last, f32)
    Tc = EYE if Tcw_cur is None else np.asarray(Tcw_cur, f32)
    Kf = np.asarray(K, f32)
    fr = capi.Frame(ctx, w, h)
    fr.upload(depth=depth, flow=flow, mask=mask)
    s = fr.sample_objects(th_depth_obj, step)
    fr.close()
    n = len(s["x"])
    # the current look-up (Tracking.cc:288-305)
    u, v = s["cx"].astype(np.int64), s["cy"].astype(np.int64)
    inb = (u < w - 1) & (u > 0) & (v < h - 1) & (v > 0)
    uu, vv = np.where(inb, u, 0), np.where(inb, v, 0)
    d = np.where(inb, depth_cur[vv, uu], f32(0))
    ok = inb & (d < f32(th_depth_obj)) & (d > 0)
    dc = np.where(ok, d, f32(0.1)).astype(f32)
    lc = np.where(ok, mask_cur[vv, uu], 0).astype(np.int32)
    flow3d, _, valid = capi.scene_flow(ctx, s["x"].astype(f32), s["y"].astype(f32), s["depth"], Tl, s["cx"], s["cy"], dc, Tc, Kf, s["label"], lc)
    labels = sorted(set(lc[valid].tolist()))
    slots = labels[:M]
    r = dict(n_samples=n, pair_status=capi.OM_PAIR_OBJECT_CAP if len(labels) > M else 0,
             sample_x=s["x"], sample_y=s["y"], sample_label=s["label"], sample_depth=s["depth"], sample_cx=s["cx"], sample_cy=s["cy"],
             sample_flow=np.stack([s["fx"], s["fy"]], 1), sample_slot=np.full(n, -1, np.int32), sample_flags=np.zeros(n, np.uint8),
             sample_flow_ref=np.stack([s["fx"], s["fy"]], 1).astype(np.float64), label_cur=lc, depth_cur=dc, flow3d=flow3d,
             obj_label=np.where(valid, -2, -1).astype(np.int32),
             label=np.full(M, -1, np.int32), H=np.tile(EYE, (M, 1, 1)), X=np.tile(EYE, (M, 1, 1)), T_init=np.tile(EYE, (M, 1, 1)),
             centre=np.zeros((M, 3), f32), velocity=np.zeros((M, 3), f32), info=np.zeros((M, 8), np.int32), stats=np.zeros((M, 8)),
             status=np.zeros(M, np.int32), id=np.full(M, -1, np.int32), cls=np.zeros(M, np.int32), vote=np.zeros(M, np.int32),
             stat=np.zeros(M, np.int32), max_id=np.int32(1 if prev is None else prev["max_id"]))
    r["info"][:, 6] = -1
    r["stats"][:, 0] = -1
    ids = []
    for j, L in enumerate(slots):
        idx = np.nonzero(valid & (lc == L))[0]
        ids.append(idx)
        r["sample_slot"][idx] = j
        r["label"][j] = L
        obj = unproject_world(s["x"][idx].astype(f32), s["y"][idx].astype(f32), s["depth"][idx], Kf, Tl)
        for c in range(3):
            r["centre"][j, c] = np.add.accumulate(obj[:, c], dtype=f32)[-1] * f32(1.0 / len(idx))
    # DynObjTracking on the slots' samples (a sample of a label past the slots is never classified)
    sel = np.concatenate(ids) if ids else np.zeros(0, np.int64)
    sel.sort()
    pv = reset_state(M) if prev is None else prev
    ol, objs, mod_label, sem_pos, max_id = capi.dyn_obj_tracking(
        ctx, lc[sel], np.zeros(len(sel), np.int32), np.stack([s["cx"][sel], s["cy"][sel]], 1), dc[sel], flow3d[sel], s["label"][sel],
        pv["label"], np.asarray(pv["stat"], np.uint8), pv["id"], h, w, shrink[0], shrink[1], sf_mg_thres, sf_ds_thres, th_depth_obj,
        1 if prev is None else 2, int(pv["max_id"]))
    r["max_id"] = np.int32(max_id)
    r["obj_label"][sel] = ol
    for j, idx in enumerate(ids):
        L = slots[j]
        if L in sem_pos:
            r["cls"][j] = capi.OT_DYNAMIC
        elif (ol[np.searchsorted(sel, idx)] == 0).all():
            r["cls"][j] = capi.OT_STATIC
        else:                                  # boundary or far: the boundary fraction decides, in float
            cx, cy = s["cx"][idx], s["cy"][idx]
            out = (cy < f32(shrink[0])) | (cy > f32(h - shrink[0])) | (cx < f32(shrink[1])) | (cx > f32(w - shrink[1]))
            r["cls"][j] = capi.OT_BOUNDARY if f32(out.sum()) / f32(len(idx)) > f32(0.5) else capi.OT_FAR
    # the dynamic objects: the motion model by ID, RANSAC, the gate, the LM
    probs, dyn = [], []
    for k, L in enumerate(sem_pos):
        j = slots.index(L)
        idx = ids[j]
        r["id"][j] = mod_label[k]
        r["vote"][j] = majority(s["label"][idx])
        T_mm = None
        hit = np.nonzero(np.asarray(pv["id"]) == mod_label[k])[0]
        if prev is not None and len(hit):
            T_mm = mul4(Tc, pv["H"][hit[0]])
        obj = unproject_world(s["x"][idx].astype(f32), s["y"][idx].astype(f32), s["depth"][idx], Kf, Tl)
        probs.append(dict(obj=obj, img=np.stack([s["cx"][idx], s["cy"][idx]], 1), T_mm=T_mm))
        dyn.append(j)
    im = capi.init_model_batch(ctx, probs, Kf, iters, thr, conf) if probs else []
    lm_jobs = []
    for j, q in zip(dyn, im):
        idx = ids[j]
        sub = idx[q["sub"]]
        r["T_init"][j] = q["T"]
        r["info"][j] = [len(idx), q["n_ransac"], q["n_mm"], int(q["used_mm"]), len(sub), q["iters_run"], q["best_it"], q["n_valid"]]
        r["sample_flags"][sub] = 1
        r["obj_label"][np.setdiff1d(idx, sub)] = -1                     # Tracking.cc:1841-1845
        lm = len(sub) >= min_inliers
        st = capi.OM_NO_MODEL if q["best_it"] < 0 else 0
        r["status"][j] = st | (0 if lm else capi.OM_FEW_INLIERS) | (capi.OM_USED_MM if q["used_mm"] else 0)
        r["stat"][j] = int(lm)
        if lm:
            lm_jobs.append((j, sub, dict(pts=np.stack([s["x"][sub], s["y"][sub]], 1).astype(f32), depth=s["depth"][sub],
                                         flow=np.stack([s["fx"][sub], s["fy"][sub]], 1), K=Kf, Tcw_last=Tl, T_init=q["T"])))
    if lm_jobs:
        res = capi.pose_opt_flow2(ctx, [pb for _, _, pb in lm_jobs], quirk=quirk, modes=[1] * len(lm_jobs))
        Ti = inv4(Tc)
        for (j, sub, _), o in zip(lm_jobs, res):
            r["X"][j] = o["T"]
            r["stats"][j] = o["stats"]
            r["H"][j] = mul4(Ti, o["T"])
            r["velocity"][j] = velocity(r["H"][j], r["centre"][j])
            r["sample_flags"][sub] |= np.where(o["inlier"], 2, 0).astype(np.uint8)
            r["sample_flow_ref"][sub] = o["flow"]
            r["obj_label"][sub[~np.asarray(o["inlier"], bool)]] = -1
    return r
