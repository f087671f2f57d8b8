"""ctypes front-end of oracle/liboracle.so (TEST INFRASTRUCTURE ONLY; see oracle/__init__.py)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h"))]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def _p(a, ty):
    return a.ctypes.data_as(C.POINTER(ty))


def _graph_args(g, se3, pt):
    d, i = C.c_double, C.c_int
    return [len(se3), _p(se3, d), len(pt), _p(pt, d),
            len(g["prior_v"]), _p(g["prior_v"], i), _p(g["prior_Z"], d), _p(g["prior_w"], d),
            len(g["se3e_ij"]), _p(g["se3e_ij"], i), _p(g["se3e_Z"], d), _p(g["se3e_w"], d), _p(g["se3e_delta"], d),
            len(g["obs_cp"]), _p(g["obs_cp"], i), _p(g["obs_z"], d), _p(g["obs_w"], d), _p(g["obs_delta"], d),
            len(g["ter_pph"]), _p(g["ter_pph"], i), _p(g["ter_w"], d), _p(g["ter_delta"], d)]


def ba_optimize(g, max_iters=300, gain_threshold=1e-4, verbose=False):
    """Runs the oracle LM on graph dict `g` (vdo_slam_b200.synth.make_batch_graph layout).
    Returns dict(se3, pt, iters, chi2 (len iters+1), stats)."""
    L = lib()
    se3 = g["se3"].copy()
    pt = g["pt"].copy()
    hist = np.zeros(max_iters + 1)
    stats = np.zeros(8)
    L.vdo_oracle_ba_optimize.restype = C.c_int
    n = L.vdo_oracle_ba_optimize(*_graph_args(g, se3, pt), C.c_int(max_iters), C.c_double(gain_threshold),
                                 C.c_int(int(verbose)), _p(hist, C.c_double), _p(stats, C.c_double))
    return dict(se3=se3, pt=pt, iters=n, chi2=hist[: n + 1].copy(),
                stats=dict(lam=stats[0], trials=int(stats[1]), lnz=int(stats[2]), t_linear=stats[3], t_total=stats[4]))


def se3_frame_order(g):
    """Elimination positions of the se3 vertices for the blocked solver: by frame (camera k, then the motion vertices k -> k+1),
    which makes the reduced matrix banded.  The frame of a motion vertex is the camera that observes p1 of one of its ternary
    edges; a motion vertex without ternary edges inherits the frame of its smoothness neighbour (or goes last)."""
    C = len(g["se3"])
    n_cam = int(g.get("n_cam", 0)) or int(g["obs_cp"][:, 0].max()) + 1
    key = np.full(C, np.inf)
    key[:n_cam] = np.arange(n_cam)
    if len(g["ter_pph"]):
        cam_of_pt = np.full(len(g["pt"]), -1, np.int64)
        cam_of_pt[g["obs_cp"][:, 1]] = g["obs_cp"][:, 0]
        key[g["ter_pph"][:, 2]] = cam_of_pt[g["ter_pph"][:, 0]] + 0.5
    for _ in range(4):
        bad = ~np.isfinite(key)
        if not bad.any():
            break
        for i, j in g["se3e_ij"]:
            if bad[i] and not bad[j]:
                key[i] = key[j] - 1
            elif bad[j] and not bad[i]:
                key[j] = key[i] + 1
    order = np.argsort(key, kind="stable")
    pos = np.empty(C, np.int32)
    pos[order] = np.arange(C, dtype=np.int32)
    return pos


def ba_optimize_blocked(g, max_iters=300, gain_threshold=1e-4, verbose=False, se3_pos="frame", nthreads=0, time_budget_s=0.0):
    """Same LM as ba_optimize with the blocked direct solver of oracle/ba_block.h (points eliminated per tracklet, tiled band
    Cholesky of the reduced matrix, OpenMP).  se3_pos: "frame" (se3_frame_order), None (identity) or an int array."""
    L = lib()
    se3 = g["se3"].copy()
    pt = g["pt"].copy()
    hist = np.zeros(max_iters + 1)
    lam = np.zeros(max_iters + 1)
    t_hist = np.zeros(max_iters + 1)
    stats = np.zeros(8)
    if isinstance(se3_pos, str):
        se3_pos = se3_frame_order(g)
    pos_arg = _p(np.ascontiguousarray(se3_pos, np.int32), C.c_int) if se3_pos is not None else None
    L.vdo_oracle_ba_optimize_blocked.restype = C.c_int
    n = L.vdo_oracle_ba_optimize_blocked(*_graph_args(g, se3, pt), C.c_int(max_iters), C.c_double(gain_threshold), C.c_int(int(verbose)),
                                         _p(hist, C.c_double), _p(stats, C.c_double), pos_arg, C.c_int(int(nthreads)),
                                         _p(lam, C.c_double), C.c_double(float(time_budget_s)), _p(t_hist, C.c_double))
    return dict(se3=se3, pt=pt, iters=n, chi2=hist[: n + 1].copy(), lam=lam[:n].copy(), t_iter=t_hist[:n].copy(),
                stats=dict(lam=stats[0], trials=int(stats[1]), band_doubles=int(stats[2]), t_linear=stats[3], t_total=stats[4],
                           t_setup=stats[5], t_schur=stats[6], t_chol=stats[7]))


def ba_dense_system(g):
    L = lib()
    se3 = g["se3"].copy()
    pt = g["pt"].copy()
    n = 3 * len(pt) + 6 * len(se3)
    H = np.zeros((n, n))
    b = np.zeros(n)
    chi = C.c_double(0)
    L.vdo_oracle_ba_dense_system(*_graph_args(g, se3, pt), _p(H, C.c_double), _p(b, C.c_double), C.byref(chi))
    return H, b, chi.value


def ba_sparse_system(g):
    """H (symmetric scipy.sparse CSC matrix), b and the robust chi2 of graph `g` at its estimates, in the scalar order of
    ba_dense_system (3 per point, then 6 per se3 vertex); the oracle's own sparse storage, so any shape it can factor fits."""
    import scipy.sparse as sp
    L = lib()
    se3 = np.ascontiguousarray(g["se3"], np.float64).copy()
    pt = np.ascontiguousarray(g["pt"], np.float64).copy()
    n = 3 * len(pt) + 6 * len(se3)
    L.vdo_oracle_ba_sparse_system.restype = C.c_int64
    args = _graph_args(g, se3, pt)
    nnz = L.vdo_oracle_ba_sparse_system(*args, C.c_int64(0), None, None, None, None, None)
    Ap = np.zeros(n + 1, np.int64)
    Ai = np.zeros(max(nnz, 1), np.int32)
    Ax = np.zeros(max(nnz, 1))
    b = np.zeros(n)
    chi = C.c_double(0)
    L.vdo_oracle_ba_sparse_system(*args, C.c_int64(nnz), _p(Ap, C.c_int64), _p(Ai, C.c_int), _p(Ax, C.c_double), _p(b, C.c_double), C.byref(chi))
    U = sp.csc_matrix((Ax[:nnz], Ai[:nnz], Ap), shape=(n, n))
    H = (U + sp.triu(U, 1).T).tocsc()
    return H, b, chi.value


def edge_eval(kind, a, b, c):
    L = lib()
    a, b, c = (np.ascontiguousarray(x, np.float64) for x in (a, b, c))
    err = np.zeros(6)
    Ja, Jb, Jc = np.zeros(36), np.zeros(36), np.zeros(36)
    L.vdo_oracle_edge_eval(C.c_int(kind), *(_p(x, C.c_double) for x in (a, b, c, err, Ja, Jb, Jc)))
    return err, Ja, Jb, Jc


def iso_oplus(T, upd):
    T = np.ascontiguousarray(T, np.float64).copy()
    upd = np.ascontiguousarray(upd, np.float64)
    lib().vdo_oracle_iso_oplus(_p(T, C.c_double), _p(upd, C.c_double))
    return T


def flow2(p, mode=1, quirk=1, trace=False):
    """Oracle for Optimizer::PoseOptimizationFlow2 (mode=1) / Flow2Cam (mode=0) on a make_flow_problem dict.  trace=True adds
    `trace`, the LM trace in the layout of the GPU entry (vdo_slam_b200.capi.parse_flow2_trace)."""
    L = lib()
    n = len(p["depth"])
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    pts, depth, flow, K, Tl, Ti = f32(p["pts"]), f32(p["depth"]), f32(p["flow"]), f32(p["K"]), f32(p["Tcw_last"]), f32(p["T_init"])
    T_out = np.zeros((4, 4), np.float32); flow_out = np.zeros((n, 2)); inl = np.zeros(n, np.uint8); stats = np.zeros(16)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    args = [C.c_int(mode), C.c_int(quirk), C.c_int(n), fp(pts), fp(depth), fp(flow), fp(K), fp(Tl), fp(Ti),
            fp(T_out), _p(flow_out, C.c_double), inl.ctypes.data_as(C.POINTER(C.c_uint8)), _p(stats, C.c_double)]
    if trace:
        from vdo_slam_b200.capi import FLOW2_TRACE_DOUBLES, parse_flow2_trace
        tr = np.zeros(FLOW2_TRACE_DOUBLES)
        L.vdo_oracle_flow2_trace.restype = C.c_int
        it = L.vdo_oracle_flow2_trace(*args, _p(tr, C.c_double))
    else:
        L.vdo_oracle_flow2.restype = C.c_int
        it = L.vdo_oracle_flow2(*args)
    out = dict(T=T_out, flow=flow_out, inlier=inl.astype(bool), iters=it, trials=int(stats[1]), chi2=stats[2], lam=stats[3],
               n_inliers=int(stats[4]), q=stats[5:9].copy(), t=stats[9:12].copy())
    if trace:
        out["trace"] = parse_flow2_trace(tr)
    return out


def pnp_ransac(obj, img, K4, max_iters=500, thr=0.4, conf=0.98):
    """oracle/pnp_ransac.c.  obj (n,3) f32 world points, img (n,2) f32 pixels, K4 = (fx, fy, cx, cy).
    Returns dict(Rt (12,) [R row-major | t], inliers (ascending), stats, Rt_hyp) or None when RANSAC fails."""
    L = lib()
    obj = np.ascontiguousarray(obj, np.float32); img = np.ascontiguousarray(img, np.float32)
    K = np.ascontiguousarray(K4, np.float64)
    n = len(obj)
    Rt, Rh = np.zeros(12), np.zeros(12)
    inl = np.zeros(max(n, 1), np.int32); stats = np.zeros(3, np.int32)
    L.vdo_oracle_pnp_ransac.restype = C.c_int
    m = L.vdo_oracle_pnp_ransac(C.c_int(n), _p(obj, C.c_float), _p(img, C.c_float), _p(K, C.c_double), C.c_int(max_iters), C.c_double(thr),
                                C.c_double(conf), _p(Rt, C.c_double), _p(inl, C.c_int), _p(stats, C.c_int), _p(Rh, C.c_double))
    if m <= 0:
        return None
    return dict(Rt=Rt, inliers=inl[:m].copy(), stats=stats.tolist(), Rt_hyp=Rh)


def ransac_samples(n, iters=500):
    L = lib()
    idx = np.zeros((iters, 4), np.int32)
    L.vdo_oracle_ransac_samples(C.c_int(n), C.c_int(iters), _p(idx, C.c_int))
    return idx


def p3p4(P, uv, K4):
    L = lib()
    P = np.ascontiguousarray(P, np.float64); uv = np.ascontiguousarray(uv, np.float64); K = np.ascontiguousarray(K4, np.float64)
    Rt = np.zeros(12)
    L.vdo_oracle_p3p4.restype = C.c_int
    ok = L.vdo_oracle_p3p4(_p(P, C.c_double), _p(uv, C.c_double), _p(K, C.c_double), _p(Rt, C.c_double))
    return Rt if ok else None
