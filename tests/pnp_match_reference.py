"""Host restatement of the correspondence gather of vdo_pnp_match_batch_dev (include/vdo_b200.h), in the float32 rounding the device
uses: the arrays it returns, given to capi.init_model_batch, must give the device call's result bit for bit."""
import numpy as np


def gather(qx, qy, q_count, tx, ty, t_count, idx, dist, depth, K, Tcw=None, ratio=None, max_depth=None):
    """One pair.  qx, qy: the query frame's (cap_q,) keypoints; tx, ty: the train frame's; idx, dist: (cap_q, k) orb_match rows of the
    pair; depth: (H, W) metric depth of the query frame; K: fx, fy, cx, cy of the query frame; Tcw: None or its 4x4 pose.
    Returns (sel: query indices of the correspondences in ascending order, obj (n, 3) f32, img (n, 2) f32)."""
    cap_q, cap_t = len(qx), len(tx)
    nq = int(q_count) if 0 <= q_count <= cap_q else 0
    nt = int(t_count) if 0 <= t_count <= cap_t else 0
    f32 = np.float32
    u, v = np.asarray(qx[:nq], f32), np.asarray(qy[:nq], f32)
    j = np.asarray(idx[:nq, 0], np.int64)
    ok = (j >= 0) & (j < nt)
    if ratio is not None and ratio > 0:
        ok &= (idx[:nq, 1] >= 0) & (dist[:nq, 0].astype(f32) < f32(ratio) * dist[:nq, 1].astype(f32))
    H, W = depth.shape
    with np.errstate(invalid="ignore"):
        inside = (u > f32(-1)) & (u < f32(W)) & (v > f32(-1)) & (v < f32(H))
    ui = np.where(inside, np.trunc(np.where(inside, u, 0)), 0).astype(np.int64)
    vi = np.where(inside, np.trunc(np.where(inside, v, 0)), 0).astype(np.int64)
    z = np.where(inside, depth[vi, ui], f32(0)).astype(f32)
    with np.errstate(invalid="ignore"):
        ok &= inside & ((z > 0) & (z <= f32(max_depth)) if max_depth is not None and max_depth > 0 else z > 0)
    sel = np.nonzero(ok)[0]
    Kf = np.asarray(K, f32)
    invfx, invfy = f32(1) / Kf[0], f32(1) / Kf[1]
    zs, us, vs = z[sel], u[sel], v[sel]
    x = (us - Kf[2]) * zs * invfx
    y = (vs - Kf[3]) * zs * invfy
    if Tcw is None:
        obj = np.stack([x, y, zs], 1).astype(f32)
    else:
        T = np.asarray(Tcw, f32).reshape(16).astype(np.float64)       # tracker.cpp unproject_world: Twc = Tcw^-1, double products, float results
        cols = []
        for r in range(3):
            twl = np.float64(f32(-(T[r] * T[3] + T[4 + r] * T[7] + T[8 + r] * T[11])))
            cols.append((T[r] * x.astype(np.float64) + T[4 + r] * y.astype(np.float64) + T[8 + r] * zs.astype(np.float64) + twl).astype(f32))
        obj = np.stack(cols, 1)
    jj = j[sel]
    img = np.stack([np.asarray(tx, f32)[jj], np.asarray(ty, f32)[jj]], 1) if len(sel) else np.zeros((0, 2), f32)
    return sel, obj, img
