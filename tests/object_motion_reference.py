"""Host route of the object step that vdo_obj_motion_batch_dev (capi.ObjectMotion) runs on the device: the resident frame's
vdo_frame_sample_objects, grouping by label and back-projection in numpy in the tracker's float rounding, capi.init_model_batch with the
constant-motion model, the min_inliers gate, capi.pose_opt_flow2 (mode 1) and H = Tcw_cur^-1 X.  Its result, given the same inputs, must
equal the device call's bit for bit."""
import numpy as np

from vdo_slam_b200 import capi

f32 = np.float32
EYE = np.eye(4, dtype=f32)


def mul4(A, B):
    """cv::Mat A * B of two 4x4 CV_32F as tracker.cpp rounds it: a0*b0 + a1*b1 + a2*b2 + a3*b3 in float, left to right"""
    A, B = np.asarray(A, f32).reshape(4, 4), np.asarray(B, f32).reshape(4, 4)
    C = np.zeros((4, 4), f32)
    for i in range(4):
        s = A[i, 0] * B[0]
        for k in range(1, 4):
            s = s + A[i, k] * B[k]
        C[i] = s
    return C


def inv4(T):
    """Converter::toInvMatrix as tracker.cpp rounds it: R^T, and -R^T t accumulated in double"""
    T = np.asarray(T, f32).reshape(4, 4)
    I = EYE.copy()
    I[:3, :3] = T[:3, :3].T
    for i in range(3):
        s = 0.0
        for k in range(3):
            s += float(T[k, i]) * float(T[k, 3])
        I[i, 3] = f32(-s)
    return I


def unproject_world(u, v, z, K, Tcw):
    """Frame::UnprojectStereoObject as tracker.cpp's unproject_world rounds it (float back-projection, double products in a fixed order)"""
    Kf = np.asarray(K, f32)
    invfx, invfy = f32(1) / Kf[0], f32(1) / Kf[1]
    u, v, z = np.asarray(u, f32), np.asarray(v, f32), np.asarray(z, f32)
    x = (u - Kf[2]) * z * invfx
    y = (v - Kf[3]) * z * invfy
    T = np.asarray(Tcw, f32).reshape(16).astype(np.float64)
    cols = []
    for r in range(3):
        twl = np.float64(f32(-(T[r] * T[3] + T[4 + r] * T[7] + T[8 + r] * T[11])))
        cols.append((T[r] * x.astype(np.float64) + T[4 + r] * y.astype(np.float64) + T[8 + r] * z.astype(np.float64) + twl).astype(f32))
    return np.stack(cols, 1) if len(u) else np.zeros((0, 3), f32)


def velocity(H, c):
    """Tracking.cc:958: t_H - (I - R_H) c, the 3x3 difference and the float gemm rounded as cv::Mat rounds them"""
    H = np.asarray(H, f32)
    M = np.eye(3, dtype=f32) - H[:3, :3]
    c = np.asarray(c, f32)
    s = M[:, 0] * c[0]
    s = s + M[:, 1] * c[1]
    s = s + M[:, 2] * c[2]
    return H[:3, 3] - s


def host_route(ctx, depth, flow, mask, K, M, Tcw_last=None, Tcw_cur=None, prev_label=None, prev_H=None, step=4, th_depth_obj=25.0, iters=500,
               thr=0.4, conf=0.98, min_inliers=50, quirk=1):
    """One pair.  depth (H, W) f32 metric, flow (H, W, 2) f32, mask (H, W) int labels (within int32), K (4,); M: object slots;
    Tcw_last, Tcw_cur: None or 4x4; prev_label (M,), prev_H (M, 4, 4): the previous result, or None.
    Returns dict of numpy arrays in the layout of one pair of ObjectMotion.estimate's result (samples: n_samples rows)."""
    h, w = depth.shape
    Tl = EYE if Tcw_last is None else np.asarray(Tcw_last, f32)
    Tc = EYE if Tcw_cur is None else np.asarray(Tcw_cur, f32)
    fr = capi.Frame(ctx, w, h)
    fr.upload(depth=depth, flow=flow, mask=mask)
    s = fr.sample_objects(th_depth_obj, step)
    fr.close()
    n = len(s["x"])
    labels = sorted(set(s["label"].tolist()))
    slots = labels[:M]
    r = dict(n_samples=n, pair_status=capi.OM_PAIR_OBJECT_CAP if len(labels) > M else 0,
             sample_x=s["x"], sample_y=s["y"], sample_label=s["label"], sample_depth=s["depth"], sample_cx=s["cx"], sample_cy=s["cy"],
             sample_flow=np.stack([s["fx"], s["fy"]], 1), sample_slot=np.full(n, -1, np.int32), sample_flags=np.zeros(n, np.uint8),
             sample_flow_ref=np.stack([s["fx"], s["fy"]], 1).astype(np.float64),
             label=np.full(M, -1, np.int32), H=np.tile(EYE, (M, 1, 1)), X=np.tile(EYE, (M, 1, 1)), T_init=np.tile(EYE, (M, 1, 1)),
             centre=np.zeros((M, 3), f32), velocity=np.zeros((M, 3), f32), info=np.zeros((M, 8), np.int32), stats=np.zeros((M, 8)),
             status=np.zeros(M, np.int32))
    r["info"][:, 6] = -1
    r["stats"][:, 0] = -1
    probs, ids = [], []
    for j, L in enumerate(slots):
        idx = np.nonzero(s["label"] == L)[0]
        ids.append(idx)
        r["sample_slot"][idx] = j
        r["label"][j] = L
        obj = unproject_world(s["x"][idx].astype(f32), s["y"][idx].astype(f32), s["depth"][idx], K, Tl)
        for c in range(3):                     # the float sum in point order, times (float)(1.0 / n)
            r["centre"][j, c] = np.add.accumulate(obj[:, c], dtype=f32)[-1] * f32(1.0 / len(idx))
        T_mm = None
        if prev_label is not None and L != -1:
            hit = np.nonzero(np.asarray(prev_label) == L)[0]
            if len(hit):
                T_mm = mul4(Tc, prev_H[hit[0]])
        probs.append(dict(obj=obj, img=np.stack([s["cx"][idx], s["cy"][idx]], 1), T_mm=T_mm))
    im = capi.init_model_batch(ctx, probs, np.asarray(K, f32), iters, thr, conf) if probs else []
    lm_jobs = []
    for j, (idx, q) in enumerate(zip(ids, im)):
        sub = idx[q["sub"]]
        r["T_init"][j] = q["T"]
        r["info"][j] = [len(idx), q["n_ransac"], q["n_mm"], int(q["used_mm"]), len(sub), q["iters_run"], q["best_it"], q["n_valid"]]
        r["sample_flags"][sub] = 1
        lm = len(sub) >= min_inliers
        st = (capi.OM_FEW_POINTS if len(idx) < 4 else 0) | (capi.OM_NO_MODEL if len(idx) >= 4 and q["best_it"] < 0 else 0)
        r["status"][j] = st | (0 if lm else capi.OM_FEW_INLIERS) | (capi.OM_USED_MM if q["used_mm"] else 0)
        if lm:
            lm_jobs.append((j, sub, dict(pts=np.stack([s["x"][sub], s["y"][sub]], 1).astype(f32), depth=s["depth"][sub],
                                         flow=np.stack([s["fx"][sub], s["fy"][sub]], 1), K=np.asarray(K, f32), Tcw_last=Tl, T_init=q["T"])))
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
    return r
