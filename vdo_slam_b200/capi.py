"""ctypes binding of libvdo_b200.so (C ABI in include/vdo_b200.h).

The library is built in-tree by `__graft_entry__.build()` (nvcc, sm_90a).  There is no CPU fallback: if the
shared object is missing or no CUDA device is usable, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvdo_b200.so")


class LMOptions(C.Structure):
    _fields_ = [("max_iterations", C.c_int), ("gain_threshold", C.c_double), ("max_trials", C.c_int),
                ("pcg_rel_tol", C.c_double), ("pcg_max_iterations", C.c_int), ("verbose", C.c_int),
                ("force_all_iterations", C.c_int), ("pcg_loose_tol", C.c_double), ("pcg_switch_gain", C.c_double)]


class LMStats(C.Structure):
    _fields_ = [("iterations", C.c_int), ("trials", C.c_int), ("pcg_iterations", C.c_int),
                ("initial_chi2", C.c_double), ("final_chi2", C.c_double), ("final_lambda", C.c_double),
                ("ms_linearize", C.c_double), ("ms_solve", C.c_double), ("ms_total", C.c_double),
                ("kernel_launches", C.c_int)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class VdoError(RuntimeError):
    pass


_libs = {}


def load(path: str | None = None) -> C.CDLL:
    path = path or LIB_PATH
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise VdoError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
                       "There is no CPU fallback.")
    L = C.CDLL(path)
    L.vdo_last_error.restype = C.c_char_p
    L.vdo_ctx_stream.restype = C.c_uint64
    # the structs below are mirrored by hand: refuse a library whose layout differs (it would write past the ctypes buffers)
    for name, cls in (("vdo_lm_options", LMOptions), ("vdo_lm_stats", LMStats), ("vdo_tracker_params", globals().get("TrackerParams")),
                      ("vdo_dev_plane", globals().get("DevPlane")), ("vdo_orb_batch_out", globals().get("OrbBatchOut")),
                      ("vdo_orb_desc_set", globals().get("OrbDescSet")), ("vdo_orb_match_opts", globals().get("OrbMatchOpts")),
                      ("vdo_orb_match_out", globals().get("OrbMatchOut")), ("vdo_pnp_match_opts", globals().get("PnpMatchOpts")),
                      ("vdo_pnp_out", globals().get("PnpOut")), ("vdo_pose_refine_opts", globals().get("PoseRefineOpts")),
                      ("vdo_pose_refine_out", globals().get("PoseRefineOut")), ("vdo_obj_motion_opts", globals().get("ObjMotionOpts")),
                      ("vdo_obj_motion_out", globals().get("ObjMotionOut")),
                      ("vdo_obj_track_opts", globals().get("ObjTrackOpts")), ("vdo_obj_track_out", globals().get("ObjTrackOut")),
                      ("vdo_obj_mask_out", globals().get("ObjMaskOut")), ("vdo_obj_feat_set", globals().get("ObjFeatSet")),
                      ("vdo_stat_feat_set", globals().get("StatFeatSet")), ("vdo_stat_opts", globals().get("StatOpts")),
                      ("vdo_cam_track_opts", globals().get("CamTrackOpts")), ("vdo_cam_track_out", globals().get("CamTrackOut"))):
        if cls is not None and hasattr(L, "vdo_abi_struct_size"):
            n = L.vdo_abi_struct_size(name.encode())
            if n != C.sizeof(cls):
                raise VdoError(f"{path}: sizeof({name}) is {n} in the library but {C.sizeof(cls)} in capi.py -- rebuild the library or update the binding")
    _libs[path] = L
    return L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class Context:
    """vdo_ctx: one per System (device + stream)."""

    def __init__(self, device: int = 0, lib_path: str | None = None):
        self.L = load(lib_path)
        self.device = device
        self.h = C.c_void_p()
        rc = self.L.vdo_ctx_create(C.c_int(device), C.byref(self.h))
        if rc != 0:
            raise VdoError(f"vdo_ctx_create(device={device}) failed with {rc}: no usable CUDA device (no CPU fallback)")

    def check(self, rc: int, what: str):
        if rc != 0:
            raise VdoError(f"{what} failed with {rc}: {self.L.vdo_last_error(self.h).decode()}")

    @property
    def stream(self) -> int:
        return int(self.L.vdo_ctx_stream(self.h))

    rank, world = 0, 1

    def init_comm(self, rank: int, world: int, dist=None):
        """Multi-GPU: create the NCCL communicator of this context (id from rank 0, broadcast through torch.distributed)."""
        self.rank, self.world = rank, world
        if world <= 1:
            return
        import torch
        dist = dist or torch.distributed
        buf = C.create_string_buffer(128)
        if rank == 0:
            self.check(self.L.vdo_nccl_unique_id(buf), "vdo_nccl_unique_id")
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
        t = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone().to(dev)
        dist.broadcast(t, src=0)
        idb = bytes(t.cpu().numpy().tobytes())
        self.check(self.L.vdo_ctx_init_comm(self.h, C.c_int(rank), C.c_int(world), C.c_char_p(idb)), "vdo_ctx_init_comm")

    def set_collective_emul(self, rank: int, world: int, dist):
        """TEST ONLY (tests/emul/libvdo_emul.so): all-reduce of the emulated backend through torch.distributed (gloo)."""
        import torch
        self.rank, self.world = rank, world
        CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.c_size_t, C.c_int, C.c_void_p)

        def _cb(ptr, n, op, user):
            a = np.ctypeslib.as_array(ptr, shape=(n,))
            t = torch.from_numpy(a)
            dist.all_reduce(t, op=dist.ReduceOp.SUM if op == 0 else dist.ReduceOp.MAX)

        self._cb = CB(_cb)
        self.check(self.L.vdo_emul_set_collective(self.h, C.c_int(rank), C.c_int(world), self._cb, None), "vdo_emul_set_collective")

    def close(self):
        if self.h:
            self.L.vdo_ctx_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def g2o_read(ctx: "Context", path: str) -> dict:
    """Parse a .g2o file (the reference's optimizer.save() dumps) into the dict layout of synth.make_batch_graph plus the file
    ids (se3_id / pt_id / fixed_id) and the information matrices as written (prior_info / se3e_info: n x 21, obs_info /
    ter_info: n x 6, upper triangles)."""
    L = ctx.L
    h = C.c_void_p()
    rc = L.vdo_g2o_read(path.encode(), C.byref(h))
    if rc != 0:
        L.vdo_g2o_error.restype = C.c_char_p
        msg = L.vdo_g2o_error(h).decode() if h else "cannot open"
        if h:
            L.vdo_g2o_free(h)
        raise VdoError(f"vdo_g2o_read({path}) failed ({rc}): {msg}")
    try:
        cnt = (C.c_int64 * 8)()
        ctx.check(L.vdo_g2o_counts(h, cnt), "vdo_g2o_counts")
        n_se3, n_pt, n_pr, n_se, n_ob, n_te, n_fix, n_off = list(cnt)

        def geti(name, shape):
            a = np.zeros(shape, np.int32)
            ctx.check(L.vdo_g2o_get_i32(h, name.encode(), _ip(a), C.c_int64(a.size)), name)
            return a

        def getf(name, shape):
            a = np.zeros(shape, np.float64)
            ctx.check(L.vdo_g2o_get_f64(h, name.encode(), _dp(a), C.c_int64(a.size)), name)
            return a
        g = {"se3": getf("se3", (n_se3, 12)), "pt": getf("pt", (n_pt, 3)), "se3_id": geti("se3_id", (n_se3,)), "pt_id": geti("pt_id", (n_pt,)),
             "fixed_id": geti("fixed_id", (n_fix,)), "prior_v": geti("prior_v", (n_pr,)), "prior_Z": getf("prior_Z", (n_pr, 12)),
             "prior_info": getf("prior_info", (n_pr, 21)), "se3e_ij": geti("se3e_ij", (n_se, 2)), "se3e_Z": getf("se3e_Z", (n_se, 12)),
             "se3e_info": getf("se3e_info", (n_se, 21)), "obs_cp": geti("obs_cp", (n_ob, 2)), "obs_z": getf("obs_z", (n_ob, 3)),
             "obs_info": getf("obs_info", (n_ob, 6)), "ter_pph": geti("ter_pph", (n_te, 3)), "ter_meas": getf("ter_meas", (n_te, 3)),
             "ter_info": getf("ter_info", (n_te, 6)), "offset": getf("offset", (n_off, 13))}
        g["prior_w"] = g["prior_info"][:, 0].copy(); g["se3e_w"] = g["se3e_info"][:, 0].copy()
        g["obs_w"] = g["obs_info"][:, 0].copy(); g["ter_w"] = g["ter_info"][:, 0].copy()
        return g
    finally:
        L.vdo_g2o_free(h)


def g2o_write(ctx: "Context", path: str, g: dict, precision: int = 0):
    """Write a graph in the make_batch_graph layout as a .g2o file (ids from g['se3_id'] / g['pt_id'] when present)."""
    se3, pt = _f64(g["se3"]), _f64(g["pt"])
    sid = _i32(g["se3_id"]) if "se3_id" in g else None
    pid = _i32(g["pt_id"]) if "pt_id" in g else None
    fix = _i32(g.get("fixed_id", np.zeros(0, np.int32)))
    pv, pZ, pw = _i32(g["prior_v"]), _f64(g["prior_Z"]), _f64(g["prior_w"])
    ij, sZ, sw = _i32(g["se3e_ij"]), _f64(g["se3e_Z"]), _f64(g["se3e_w"])
    cp, oz, ow = _i32(g["obs_cp"]), _f64(g["obs_z"]), _f64(g["obs_w"])
    pph, tw = _i32(g["ter_pph"]), _f64(g["ter_w"])
    ctx.check(ctx.L.vdo_g2o_write(path.encode(), len(se3), _dp(se3), _ip(sid) if sid is not None else None, len(pt), _dp(pt),
                                  _ip(pid) if pid is not None else None, len(fix), _ip(fix), len(pv), _ip(pv), _dp(pZ), _dp(pw), len(sw), _ip(ij), _dp(sZ), _dp(sw),
                                  len(ow), _ip(cp), _dp(oz), _dp(ow), len(tw), _ip(pph), _dp(tw), int(precision)), "vdo_g2o_write")


def _lm_options(ctx, max_iterations, gain_threshold, pcg_rel_tol, pcg_max_iterations, verbose, force_all_iterations,
                pcg_loose_tol, pcg_switch_gain) -> LMOptions:
    o = LMOptions()
    ctx.L.vdo_lm_options_default(C.byref(o))
    o.max_iterations, o.gain_threshold = int(max_iterations), float(gain_threshold)
    o.pcg_max_iterations = int(pcg_max_iterations)
    if pcg_rel_tol is not None:
        o.pcg_rel_tol = float(pcg_rel_tol)
    if pcg_loose_tol is not None:
        o.pcg_loose_tol = float(pcg_loose_tol)
    if pcg_switch_gain is not None:
        o.pcg_switch_gain = float(pcg_switch_gain)
    o.verbose, o.force_all_iterations = int(verbose), int(force_all_iterations)
    return o


def optimize_batch(graphs, max_iterations=300, gain_threshold=1e-4, pcg_rel_tol=None, pcg_max_iterations=2000,
                   verbose=False, force_all_iterations=False, pcg_loose_tol=None, pcg_switch_gain=None):
    """vdo_graph_optimize_batch: optimise several finalized BatchGraphs of one Context in one call.  Each graph ends where its own
    BatchGraph.optimize(...) with the same keywords takes it; returns one dict per graph with the keys of BatchGraph.optimize
    (ms_* and kernel_launches describe the whole call)."""
    graphs = list(graphs)
    if not graphs:
        raise VdoError("optimize_batch: no graphs")
    ctx = graphs[0].ctx
    o = _lm_options(ctx, max_iterations, gain_threshold, pcg_rel_tol, pcg_max_iterations, verbose, force_all_iterations,
                    pcg_loose_tol, pcg_switch_gain)
    n = len(graphs)
    hs = (C.c_void_p * n)(*[g.h.value if g is not None else None for g in graphs])
    st = (LMStats * n)()
    hist = [np.zeros(max_iterations + 1) for _ in range(n)]
    hp = (C.POINTER(C.c_double) * n)(*[_dp(h) for h in hist])
    ctx.check(ctx.L.vdo_graph_optimize_batch(hs, C.c_int(n), C.byref(o), st, hp), "vdo_graph_optimize_batch")
    out = []
    for i in range(n):
        d = st[i].asdict()
        d["chi2"] = hist[i][: st[i].iterations + 1].copy()
        out.append(d)
    return out


def debug_trial(graphs, lambdas, reortho=None, pcg_rel_tol=1e-12, pcg_max_iterations=4000):
    """TEST HOOK (vdo_graph_debug_trial): one LM trial of each BatchGraph at damping lambdas[k] (re-orthogonalising graph k's rotations
    after the update when reortho[k]), sharing launches as optimize_batch does; the estimates are restored afterwards.  Returns one dict
    per graph: xp (n_se3, 6), xl (n_pt, 3), se3 (n_se3, 12), pt (n_pt, 3) (the updated estimates), chi2 (robust chi2 at them),
    scale (sum x (lambda x + b)), pcg_iterations, ok."""
    graphs = list(graphs)
    if not graphs:
        raise VdoError("debug_trial: no graphs")
    ctx, n = graphs[0].ctx, len(graphs)
    lam = _f64(lambdas).reshape(-1)
    rt = _i32(np.zeros(n) if reortho is None else np.asarray(reortho, bool)).reshape(-1)
    if len(lam) != n or len(rt) != n:
        raise VdoError(f"debug_trial: {n} graphs, {len(lam)} lambdas, {len(rt)} reortho flags")
    outs = [dict(xp=np.zeros((g.n_se3, 6)), xl=np.zeros((g.n_pt, 3)), se3=np.zeros((g.n_se3, 12)), pt=np.zeros((g.n_pt, 3))) for g in graphs]
    arrs = {k: (C.POINTER(C.c_double) * n)(*[_dp(o[k]) for o in outs]) for k in ("xp", "xl", "se3", "pt")}
    chi2, scale = np.zeros(n), np.zeros(n)
    it, ok = np.zeros(n, np.int32), np.zeros(n, np.int32)
    hs = (C.c_void_p * n)(*[g.h.value for g in graphs])
    ctx.check(ctx.L.vdo_graph_debug_trial(hs, C.c_int(n), _dp(lam), _ip(rt), C.c_double(pcg_rel_tol), C.c_int(int(pcg_max_iterations)),
                                          arrs["xp"], arrs["xl"], arrs["se3"], arrs["pt"], _dp(chi2), _dp(scale), _ip(it), _ip(ok)),
              "vdo_graph_debug_trial")
    for k, o in enumerate(outs):
        o.update(chi2=float(chi2[k]), scale=float(scale[k]), pcg_iterations=int(it[k]), ok=bool(ok[k]))
    return outs


class BatchGraph:
    """vdo_graph: the factor graph of Optimizer::FullBatchOptimization / PartialBatchOptimization."""

    @classmethod
    def from_g2o(cls, ctx: "Context", path: str, delta_se3: float, delta_pointxyz: float, delta_motion: float):
        """Load a .g2o file straight into a finalised graph (vdo_g2o_read + vdo_graph_from_g2o)."""
        L = ctx.L
        f = C.c_void_p()
        rc = L.vdo_g2o_read(path.encode(), C.byref(f))
        if rc != 0:
            if f:
                L.vdo_g2o_free(f)
            raise VdoError(f"vdo_g2o_read({path}) failed ({rc})")
        try:
            cnt = (C.c_int64 * 8)()
            ctx.check(L.vdo_g2o_counts(f, cnt), "vdo_g2o_counts")
            self = cls.__new__(cls)
            self.ctx, self.h = ctx, C.c_void_p()
            self.n_se3, self.n_pt = int(cnt[0]), int(cnt[1])
            ctx.check(L.vdo_graph_from_g2o(ctx.h, f, C.c_double(delta_se3), C.c_double(delta_pointxyz), C.c_double(delta_motion), C.byref(self.h)), "vdo_graph_from_g2o")
            return self
        finally:
            L.vdo_g2o_free(f)

    def __init__(self, ctx: Context, g: dict):
        """g: dict in the layout of vdo_slam_b200.synth.make_batch_graph."""
        self.ctx, L = ctx, ctx.L
        self.h = C.c_void_p()
        ctx.check(L.vdo_graph_create(ctx.h, C.byref(self.h)), "vdo_graph_create")
        se3, pt = _f64(g["se3"]), _f64(g["pt"])
        self.n_se3, self.n_pt = len(se3), len(pt)
        ctx.check(L.vdo_graph_set_vertices(self.h, len(se3), _dp(se3), len(pt), _dp(pt)), "vdo_graph_set_vertices")
        if len(g["prior_v"]):
            v, Z, w = _i32(g["prior_v"]), _f64(g["prior_Z"]), _f64(g["prior_w"])
            ctx.check(L.vdo_graph_add_edges_se3_prior(self.h, len(v), _ip(v), _dp(Z), _dp(w)), "add_edges_se3_prior")
        if len(g["se3e_ij"]):
            ij, Z, w, dl = _i32(g["se3e_ij"]), _f64(g["se3e_Z"]), _f64(g["se3e_w"]), _f64(g["se3e_delta"])
            ctx.check(L.vdo_graph_add_edges_se3(self.h, len(w), _ip(ij), _dp(Z), _dp(w), _dp(dl)), "add_edges_se3")
        if len(g["obs_cp"]):
            cp, z, w, dl = _i32(g["obs_cp"]), _f64(g["obs_z"]), _f64(g["obs_w"]), _f64(g["obs_delta"])
            ctx.check(L.vdo_graph_add_edges_se3_pointxyz(self.h, len(w), _ip(cp), _dp(z), _dp(w), _dp(dl)), "add_edges_se3_pointxyz")
        if len(g["ter_pph"]):
            pph, w, dl = _i32(g["ter_pph"]), _f64(g["ter_w"]), _f64(g["ter_delta"])
            ctx.check(L.vdo_graph_add_edges_landmark_motion(self.h, len(w), _ip(pph), _dp(w), _dp(dl)), "add_edges_landmark_motion")
        ctx.check(L.vdo_graph_finalize(self.h), "vdo_graph_finalize")

    def optimize(self, max_iterations=300, gain_threshold=1e-4, pcg_rel_tol=None, pcg_max_iterations=2000,
                 verbose=False, force_all_iterations=False, pcg_loose_tol=None, pcg_switch_gain=None):
        o = _lm_options(self.ctx, max_iterations, gain_threshold, pcg_rel_tol, pcg_max_iterations, verbose, force_all_iterations,
                        pcg_loose_tol, pcg_switch_gain)
        st = LMStats()
        hist = np.zeros(max_iterations + 1)
        self.ctx.check(self.ctx.L.vdo_graph_optimize(self.h, C.byref(o), C.byref(st), _dp(hist)), "vdo_graph_optimize")
        d = st.asdict()
        d["chi2"] = hist[: st.iterations + 1].copy()
        return d

    def vertices(self):
        se3 = np.zeros((self.n_se3, 12))
        pt = np.zeros((self.n_pt, 3))
        self.ctx.check(self.ctx.L.vdo_graph_get_vertices(self.h, _dp(se3), _dp(pt)), "vdo_graph_get_vertices")
        return se3, pt

    def vertices_gathered(self, dist):
        """Sharded graphs: every rank gets all landmark estimates (each rank holds only its own after optimize())."""
        import torch
        se3 = np.zeros((self.n_se3, 12))
        pt = np.full((self.n_pt, 3), np.nan)
        self.ctx.check(self.ctx.L.vdo_graph_get_vertices(self.h, _dp(se3), _dp(pt)), "vdo_graph_get_vertices")
        own = ~np.isnan(pt[:, 0])
        t = torch.from_numpy(np.where(own[:, None], pt, 0.0).copy())
        c = torch.from_numpy(own.astype(np.float64))
        if dist.get_backend() == "nccl":
            t, c = t.cuda(), c.cuda()
        dist.all_reduce(t); dist.all_reduce(c)
        assert bool((c.cpu() == 1).all()), "every landmark must be owned by exactly one rank"
        return se3, t.cpu().numpy()

    def reset(self):
        self.ctx.check(self.ctx.L.vdo_graph_reset_vertices(self.h), "vdo_graph_reset_vertices")

    def info(self):
        out = (C.c_int64 * 8)()
        self.ctx.check(self.ctx.L.vdo_graph_info(self.h, out), "vdo_graph_info")
        return dict(zip(["n_se3", "n_pt", "n_pointxyz_edges", "n_motion_edges", "n_se3_edges", "n_prior", "n_tracklets", "device_bytes"], list(out)))

    def solver_info(self):
        out = (C.c_int64 * 8)()
        self.ctx.check(self.ctx.L.vdo_graph_solver_info(self.h, out), "vdo_graph_solver_info")
        return dict(zip(["tiled", "n_tiles", "n_static_tiles", "band_width", "band_rows", "dense", "path_sharded", "n_paths"], list(out)))

    def time_kernel(self, name: str, reps: int = 20) -> float:
        ms = C.c_float(0)
        self.ctx.check(self.ctx.L.vdo_graph_time_kernel(self.h, name.encode(), C.c_int(reps), C.byref(ms)), f"vdo_graph_time_kernel({name})")
        return float(ms.value)

    def debug_linearize(self):
        Hpp = np.zeros((self.n_se3, 6, 6)); bp = np.zeros((self.n_se3, 6)); Hll = np.zeros(self.n_pt); bl = np.zeros((self.n_pt, 3))
        chi = C.c_double(0)
        self.ctx.check(self.ctx.L.vdo_graph_debug_linearize(self.h, _dp(Hpp), _dp(bp), _dp(Hll), _dp(bl), C.byref(chi)), "debug_linearize")
        return Hpp, bp, Hll, bl, chi.value

    def debug_apply(self, lam: float, op: str, x=None):
        """One operator of the reduced system at the current estimates (vdo_graph_debug_apply): op "S" / "Minv" / "rhs" take and
        return (n_se3, 6) arrays; "backsub" takes x_p (n_se3, 6) and returns x_l (n_pt, 3)."""
        out = np.zeros((self.n_pt, 3) if op == "backsub" else (self.n_se3, 6))
        xin = _f64(x).reshape(self.n_se3, 6) if x is not None else None
        self.ctx.check(self.ctx.L.vdo_graph_debug_apply(self.h, C.c_double(lam), op.encode(), _dp(xin) if xin is not None else None, _dp(out)),
                       f"debug_apply({op})")
        return out

    def debug_solve(self, lam: float, pcg_rel_tol: float = 1e-6, pcg_max_iterations: int = 2000):
        """One linear solve (H + lam I) x = b at the current estimates, as an LM trial runs it (vdo_graph_debug_solve), without the update.
        Returns dict(xp (n_se3, 6), xl (n_pt, 3), r (n_se3, 6) PCG recurrence residual, pcg_iterations)."""
        xp, r = np.zeros((self.n_se3, 6)), np.zeros((self.n_se3, 6))
        xl = np.zeros((self.n_pt, 3))
        it = C.c_int(0)
        self.ctx.check(self.ctx.L.vdo_graph_debug_solve(self.h, C.c_double(lam), C.c_double(pcg_rel_tol), C.c_int(int(pcg_max_iterations)),
                                                        _dp(xp), _dp(xl), _dp(r), C.byref(it)), "debug_solve")
        return dict(xp=xp, xl=xl, r=r, pcg_iterations=int(it.value))

    def debug_trial(self, lam: float, reortho: bool = False, pcg_rel_tol: float = 1e-12, pcg_max_iterations: int = 4000):
        """One LM trial of this graph alone (module-level debug_trial with n = 1)."""
        return debug_trial([self], [lam], [reortho], pcg_rel_tol, pcg_max_iterations)[0]

    def close(self):
        if self.h:
            self.ctx.L.vdo_graph_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# layout of one problem's LM trace (VDO_FLOW2_TRACE_* in include/vdo_b200.h)
FLOW2_TRACE_DOUBLES, FLOW2_TRACE_REC, FLOW2_TRACE_RECLEN = 96 + 16 * 2000, 96, 16
FLOW2_STOP = {1: "few_points", 2: "trials", 3: "rho_zero", 4: "no_progress", 5: "chi2_rose", 6: "max_iters"}


def parse_flow2_trace(t):
    """One problem's trace (FLOW2_TRACE_DOUBLES doubles) as dict(Hpp, bp, S, g, x, stop, rec); rec is (trials, 14):
    iteration, lambda, ok2, trial chi2, chi2 before the trial, scale, rho, accepted, the pose increment (6)."""
    nrec = int(t[91])
    rec = t[FLOW2_TRACE_REC:FLOW2_TRACE_REC + FLOW2_TRACE_RECLEN * nrec].reshape(nrec, FLOW2_TRACE_RECLEN)[:, :14].copy()
    return dict(Hpp=t[0:36].reshape(6, 6).copy(), bp=t[36:42].copy(), S=t[42:78].reshape(6, 6).copy(), g=t[78:84].copy(),
                x=t[84:90].copy(), stop=FLOW2_STOP.get(int(t[90]), int(t[90])), rec=rec)


def pose_opt_flow2(ctx: Context, problems, quirk: int = 1, modes=None, trace: bool = False):
    """Optimizer::PoseOptimizationFlow2 / Flow2Cam for a list of problems (dicts shaped like synth.make_flow_problem), in one
    call.  Returns a list of dict(T, flow, inlier, iters, trials, chi2, lam, n_inliers, stats); with trace=True each dict also
    has `trace` (parse_flow2_trace) from vdo_pose_opt_flow2_trace."""
    L = ctx.L
    nprob = len(problems)
    modes = np.asarray(modes if modes is not None else [1] * nprob, np.int32)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    off = np.zeros(nprob + 1, np.int32)
    off[1:] = np.cumsum([len(p["depth"]) for p in problems])
    cat = lambda k, shape: f32(np.concatenate([np.asarray(p[k], np.float32).reshape(shape) for p in problems], 0)) if off[-1] else np.zeros((0,) + shape[1:], np.float32)
    pts, depth, flow = cat("pts", (-1, 2)), cat("depth", (-1,)), cat("flow", (-1, 2))
    K = f32(np.stack([p["K"] for p in problems])); Tl = f32(np.stack([p["Tcw_last"] for p in problems])); Ti = f32(np.stack([p["T_init"] for p in problems]))
    T_out = np.zeros((nprob, 4, 4), np.float32); flow_out = np.zeros((int(off[-1]), 2)); inl = np.zeros(int(off[-1]), np.uint8); stats = np.zeros((nprob, 8))
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    args = [ctx.h, C.c_int(quirk), C.c_int(nprob), _ip(modes), _ip(off), fp(pts), fp(depth), fp(flow), fp(K), fp(Tl), fp(Ti),
            fp(T_out), _dp(flow_out), inl.ctypes.data_as(C.POINTER(C.c_uint8)), _dp(stats)]
    if trace:
        tr = np.zeros((nprob, FLOW2_TRACE_DOUBLES))
        ctx.check(L.vdo_pose_opt_flow2_trace(*args, _dp(tr)), "vdo_pose_opt_flow2_trace")
    else:
        ctx.check(L.vdo_pose_opt_flow2_batch(*args), "vdo_pose_opt_flow2_batch")
    out = []
    for i in range(nprob):
        a, b = off[i], off[i + 1]
        out.append(dict(T=T_out[i], flow=flow_out[a:b], inlier=inl[a:b].astype(bool), iters=int(stats[i, 0]), trials=int(stats[i, 1]),
                        chi2=stats[i, 2], lam=stats[i, 3], n_inliers=int(stats[i, 4]), stats=stats[i].copy()))
        if trace:
            out[-1]["trace"] = parse_flow2_trace(tr[i])
    return out


def pose_opt_flow2_time(ctx: Context, nprob: int, quirk: int = 1, reps: int = 20) -> float:
    ms = C.c_float(0)
    ctx.check(ctx.L.vdo_pose_opt_flow2_time(ctx.h, C.c_int(quirk), C.c_int(nprob), C.c_int(reps), C.byref(ms)), "vdo_pose_opt_flow2_time")
    return float(ms.value)


class DevPlane(C.Structure):
    """vdo_dev_plane: a width x height plane in device memory at element strides."""
    _fields_ = [("data_dev", C.c_void_p), ("dtype", C.c_int), ("channels", C.c_int), ("stride_y", C.c_int64), ("stride_x", C.c_int64),
                ("stride_c", C.c_int64), ("rgb", C.c_int)]


VDO_DT_U8, VDO_DT_F32, VDO_DT_I32, VDO_DT_I64 = 1, 2, 3, 4


def _dev_plane(ctx: Context, kind: str, t, w: int, h: int, rgb: bool = True) -> DevPlane:
    """torch CUDA tensor -> DevPlane, any strides.  Layouts: image (H,W), (H,W,C) or (C,H,W) u8 with C in {3, 4}; depth (H,W) f32;
    flow (H,W,2) or (2,H,W) f32; mask (H,W) int32 or int64.  ValueError on a wrong type, device, dtype or shape."""
    import torch
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{kind}: expected a torch tensor, got {type(t).__name__}")
    if t.device.type != "cuda" or t.device.index != ctx.device:
        raise ValueError(f"{kind}: tensor is on {t.device}, the context runs on cuda:{ctx.device}")
    shp, s = tuple(t.shape), t.stride()
    want = {"image": (torch.uint8,), "depth": (torch.float32,), "flow": (torch.float32,), "mask": (torch.int32, torch.int64)}[kind]
    if t.dtype not in want:
        raise ValueError(f"{kind}: dtype {t.dtype}, expected {' or '.join(str(d) for d in want)}")
    sc, ch = 0, 1
    if t.dim() == 2 and kind in ("image", "depth", "mask"):
        (H, W), (sy, sx) = shp, s
    elif t.dim() == 3 and kind == "image" and shp[2] in (3, 4):          # H and W are >= 64, so HWC and CHW cannot be confused
        (H, W, ch), (sy, sx, sc) = shp, s
    elif t.dim() == 3 and kind == "image" and shp[0] in (3, 4):
        (ch, H, W), (sc, sy, sx) = shp, s
    elif t.dim() == 3 and kind == "flow" and shp[2] == 2:
        (H, W, ch), (sy, sx, sc) = shp, s
    elif t.dim() == 3 and kind == "flow" and shp[0] == 2:
        (ch, H, W), (sc, sy, sx) = shp, s
    else:
        raise ValueError(f"{kind}: shape {shp} is not an accepted layout")
    if (H, W) != (h, w):
        raise ValueError(f"{kind}: {W}x{H} but the frame is {w}x{h}")
    dt = {torch.uint8: VDO_DT_U8, torch.float32: VDO_DT_F32, torch.int32: VDO_DT_I32, torch.int64: VDO_DT_I64}[t.dtype]
    return DevPlane(t.data_ptr(), dt, ch, sy, sx, sc, int(bool(rgb)))


def _torch_stream(ctx: Context) -> int:
    """the cudaStream_t of torch's current stream on the context's device"""
    import torch
    return int(torch.cuda.current_stream(torch.device("cuda", ctx.device)).cuda_stream)


def _dev_planes(ctx: Context, w: int, h: int, rgb: bool, **planes):
    """(DevPlane or None per name in order, caller stream handle): the stream is torch's current stream on the context's device"""
    out = [None if t is None else _dev_plane(ctx, k, t, w, h, rgb) for k, t in planes.items()]
    return out, _torch_stream(ctx)


class Frame:
    """vdo_frame: one RGB-D frame resident on the device (gray u8, depth f32, flow f32x2, mask i32)."""

    def __init__(self, ctx: Context, width: int, height: int):
        self.ctx, self.w, self.h = ctx, width, height
        self.h_ = C.c_void_p()
        ctx.check(ctx.L.vdo_frame_create(ctx.h, C.c_int(width), C.c_int(height), C.byref(self.h_)), "vdo_frame_create")

    def upload(self, gray=None, depth=None, flow=None, mask=None):
        self._keep = [None if a is None else np.ascontiguousarray(a, dt) for a, dt in ((gray, np.uint8), (depth, np.float32), (flow, np.float32), (mask, np.int32))]
        ptr = lambda a, ty: None if a is None else a.ctypes.data_as(C.POINTER(ty))
        g, d, f, m = self._keep
        self.ctx.check(self.ctx.L.vdo_frame_upload(self.h_, ptr(g, C.c_ubyte), ptr(d, C.c_float), ptr(f, C.c_float), ptr(m, C.c_int)), "vdo_frame_upload")

    def upload_tensors(self, image=None, depth=None, flow=None, mask=None, rgb=True):
        """vdo_frame_upload_dev from torch CUDA tensors (layouts: see _dev_plane; a colour image is converted to gray on the device,
        in RGB(A) order when rgb else BGR(A)).  Ordered after the work queued on torch's current stream; None keeps what is resident."""
        planes, stream = _dev_planes(self.ctx, self.w, self.h, rgb, image=image, depth=depth, flow=flow, mask=mask)
        ref = lambda p: None if p is None else C.byref(p)
        self.ctx.check(self.ctx.L.vdo_frame_upload_dev(self.h_, *[ref(p) for p in planes], C.c_uint64(stream)), "vdo_frame_upload_dev")

    def orb_describe(self, n):
        """vdo_orb_describe: descriptors (n x 32 u8) of the keypoints of the last orb_extract()."""
        out = np.zeros((max(n, 1), 32), np.uint8)
        self.ctx.check(self.ctx.L.vdo_orb_describe(self.h_, C.c_int(n), out.ctypes.data_as(C.POINTER(C.c_ubyte))), "vdo_orb_describe")
        return out[:n]

    def debug_blur(self, level, shape):
        out = np.zeros(shape, np.uint8)
        self.ctx.check(self.ctx.L.vdo_frame_debug_blur(self.h_, C.c_int(level), out.ctypes.data_as(C.POINTER(C.c_ubyte))), "vdo_frame_debug_blur")
        return out

    def depth_prep(self, bf, factor):
        out = np.zeros((self.h, self.w), np.float32)
        self.ctx.check(self.ctx.L.vdo_frame_depth_prep(self.h_, C.c_float(bf), C.c_float(factor), out.ctypes.data_as(C.POINTER(C.c_float))), "vdo_frame_depth_prep")
        return out

    def orb_extract(self, nfeatures=2500, scale=1.2, nlevels=8, ini_th=20, min_th=7, max_out=20000):
        f32 = lambda n: np.zeros(n, np.float32); i32 = lambda n: np.zeros(n, np.int32)
        x, y, resp, ang = f32(max_out), f32(max_out), f32(max_out), f32(max_out)
        octv, size, ncand = i32(max_out), i32(max_out), i32(nlevels)
        n = C.c_int(0)
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float)); ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))
        self.ctx.check(self.ctx.L.vdo_orb_extract(self.h_, C.c_int(nfeatures), C.c_float(scale), C.c_int(nlevels), C.c_int(ini_th), C.c_int(min_th), C.c_int(max_out),
                                                  fp(x), fp(y), ip(octv), fp(resp), fp(ang), ip(size), C.byref(n), ip(ncand)), "vdo_orb_extract")
        k = n.value
        return dict(x=x[:k], y=y[:k], octave=octv[:k], response=resp[:k], angle=ang[:k], size=size[:k], n_candidates=ncand.tolist())

    def filter_static(self, kx, ky, th_depth):
        n = len(kx)
        kx, ky = np.ascontiguousarray(kx, np.float32), np.ascontiguousarray(ky, np.float32)
        idx = np.zeros(n, np.int32); out = [np.zeros(n, np.float32) for _ in range(5)]
        m = C.c_int(0)
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        self.ctx.check(self.ctx.L.vdo_frame_filter_static(self.h_, C.c_int(n), fp(kx), fp(ky), C.c_float(th_depth), idx.ctypes.data_as(C.POINTER(C.c_int)),
                                                          *[fp(a) for a in out], C.byref(m)), "vdo_frame_filter_static")
        k = m.value
        return (idx[:k],) + tuple(a[:k] for a in out)

    def sample_objects(self, th_depth_obj, step=4, max_out=None):
        max_out = max_out or ((self.w + step - 1) // step) * ((self.h + step - 1) // step)
        x, y, lab = (np.zeros(max_out, np.int32) for _ in range(3))
        cx, cy, fx, fy, dep = (np.zeros(max_out, np.float32) for _ in range(5))
        n = C.c_int(0)
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float)); ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))
        self.ctx.check(self.ctx.L.vdo_frame_sample_objects(self.h_, C.c_float(th_depth_obj), C.c_int(step), C.c_int(max_out), ip(x), ip(y), fp(cx), fp(cy), fp(fx), fp(fy),
                                                           fp(dep), ip(lab), C.byref(n)), "vdo_frame_sample_objects")
        k = n.value
        return dict(x=x[:k], y=y[:k], cx=cx[:k], cy=cy[:k], fx=fx[:k], fy=fy[:k], depth=dep[:k], label=lab[:k])

    def debug_level(self, level: int):
        w, h = C.c_int(0), C.c_int(0)
        self.ctx.check(self.ctx.L.vdo_frame_debug_level(self.h_, C.c_int(level), None, None, C.byref(w), C.byref(h)), "vdo_frame_debug_level")
        img = np.zeros((h.value, w.value), np.uint8); sc = np.zeros((h.value, w.value), np.uint8)
        up = lambda a: a.ctypes.data_as(C.POINTER(C.c_ubyte))
        self.ctx.check(self.ctx.L.vdo_frame_debug_level(self.h_, C.c_int(level), up(img), up(sc), None, None), "vdo_frame_debug_level")
        return img, sc

    def orb_time(self, reps=20):
        ms = C.c_float(0)
        self.ctx.check(self.ctx.L.vdo_orb_time(self.h_, C.c_int(reps), C.byref(ms)), "vdo_orb_time")
        return float(ms.value)

    def close(self):
        if self.h_:
            self.ctx.L.vdo_frame_destroy(self.h_)
            self.h_ = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def scene_flow(ctx: Context, u_prev, v_prev, z_prev, Tcw_prev, u_cur, v_cur, z_cur, Tcw_cur, K, lab_prev, lab_cur):
    n = len(u_prev)
    f32 = lambda a: np.ascontiguousarray(a, np.float32); i32 = lambda a: np.ascontiguousarray(a, np.int32)
    arrs = [f32(a) for a in (u_prev, v_prev, z_prev)] + [f32(Tcw_prev)] + [f32(a) for a in (u_cur, v_cur, z_cur)] + [f32(Tcw_cur), f32(K)]
    lp, lc = i32(lab_prev), i32(lab_cur)
    flow3d = np.zeros((n, 3), np.float32); Xp = np.zeros((n, 3), np.float32); valid = np.zeros(n, np.uint8)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    ctx.check(ctx.L.vdo_scene_flow(ctx.h, C.c_int(n), *[fp(a) for a in arrs], lp.ctypes.data_as(C.POINTER(C.c_int)), lc.ctypes.data_as(C.POINTER(C.c_int)),
                                   fp(flow3d), fp(Xp), valid.ctypes.data_as(C.POINTER(C.c_uint8))), "vdo_scene_flow")
    return flow3d, Xp, valid.astype(bool)


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def tracklets_build(assoc_rows, label_rows=None, lib_path: str | None = None):
    """vdo_tracklets_build (host-only): Tracking::GetStaticTrack / GetDynamicTrackNew.  Returns (tracklets, obj_ids)."""
    L = load(lib_path)
    rb = np.zeros(len(assoc_rows) + 1, np.int32)
    rb[1:] = np.cumsum([len(r) for r in assoc_rows])
    flat = _i32(np.concatenate([np.asarray(r, np.int32) for r in assoc_rows])) if len(assoc_rows) and rb[-1] else np.zeros(0, np.int32)
    lab = None
    if label_rows is not None:
        lab = _i32(np.concatenate([np.asarray(r, np.int32) for r in label_rows])) if rb[-1] else np.zeros(0, np.int32)
    max_t = int(np.count_nonzero(flat != -1)) + 1
    max_e = 2 * max_t
    tb, tf, tk, oid = np.zeros(max_t + 1, np.int32), np.zeros(max_e, np.int32), np.zeros(max_e, np.int32), np.zeros(max_t, np.int32)
    nt = C.c_int(0)
    rc = L.vdo_tracklets_build(C.c_int(len(assoc_rows)), _ip(rb), _ip(flat), None if lab is None else _ip(lab), C.c_int(max_t), C.c_int(max_e),
                               C.byref(nt), _ip(tb), _ip(tf), _ip(tk), _ip(oid))
    if rc != 0:
        raise VdoError(f"vdo_tracklets_build failed ({rc})")
    n = nt.value
    trk = [list(zip(tf[tb[t]:tb[t + 1]].tolist(), tk[tb[t]:tb[t + 1]].tolist())) for t in range(n)]
    return trk, (oid[:n].tolist() if label_rows is not None else [])


def update_mask(cur: "Frame", last: "Frame", sem_label_last, corres):
    """vdo_update_mask: Tracking::UpdateMask on two resident frames.  Returns (updated mask, recovered labels)."""
    ctx = cur.ctx
    sl = _i32(sem_label_last)
    n = len(sl)
    corres = np.asarray(corres, np.float32).reshape(-1, 2)
    cx, cy = np.ascontiguousarray(corres[:, 0]), np.ascontiguousarray(corres[:, 1])
    out = np.zeros((cur.h, cur.w), np.int32)
    wl = np.zeros(max(1, len(set(sl.tolist()))), np.int32)
    nw = C.c_int(0)
    ctx.check(ctx.L.vdo_update_mask(cur.h_, last.h_, C.c_int(n), _ip(sl), _fp(cx), _fp(cy), _ip(out), C.byref(nw), _ip(wl)), "vdo_update_mask")
    return out, wl[:nw.value].tolist()


def dyn_obj_tracking(ctx: Context, sem_label, obj_label, keys, depth, flow3d, sem_label_last, last_sem_position, last_obj_stat, last_mod_label,
                     rows, cols, shrink_row, shrink_col, sf_mg_thres, sf_ds_thres, th_depth_obj, f_id, max_id, max_objects=256):
    """vdo_dyn_obj_tracking: Tracking::DynObjTracking.  Returns (obj_label', objects, mod_label, sem_position, max_id')."""
    sl, ol, sll = _i32(sem_label), _i32(obj_label).copy(), _i32(sem_label_last)
    n = len(sl)
    keys = np.asarray(keys, np.float32).reshape(-1, 2)
    kx, ky = np.ascontiguousarray(keys[:, 0]), np.ascontiguousarray(keys[:, 1])
    dp, f3 = np.ascontiguousarray(depth, np.float32), np.ascontiguousarray(flow3d, np.float32)
    lsp, lml = _i32(last_sem_position), _i32(last_mod_label)
    los = np.ascontiguousarray(last_obj_stat, np.uint8)
    mid, no = C.c_int(max_id), C.c_int(0)
    ob, oi = np.zeros(max_objects + 1, np.int32), np.zeros(max(n, 1), np.int32)
    ml, sp = np.zeros(max_objects, np.int32), np.zeros(max_objects, np.int32)
    ctx.check(ctx.L.vdo_dyn_obj_tracking(ctx.h, C.c_int(n), _ip(sl), _ip(ol), _fp(kx), _fp(ky), _fp(dp), _fp(f3), _ip(sll), C.c_int(len(lsp)), _ip(lsp),
                                         los.ctypes.data_as(C.POINTER(C.c_ubyte)), _ip(lml), C.c_int(rows), C.c_int(cols), C.c_int(shrink_row), C.c_int(shrink_col),
                                         C.c_float(sf_mg_thres), C.c_float(sf_ds_thres), C.c_float(th_depth_obj), C.c_int(f_id), C.byref(mid), C.c_int(max_objects),
                                         C.byref(no), _ip(ob), _ip(oi), _ip(ml), _ip(sp)), "vdo_dyn_obj_tracking")
    k = no.value
    objs = [oi[ob[t]:ob[t + 1]].tolist() for t in range(k)]
    return ol, objs, ml[:k].tolist(), sp[:k].tolist(), mid.value


def init_model_batch(ctx: Context, problems, K4, iters=500, thr=0.4, conf=0.98):
    """vdo_init_model_batch: GetInitModelCam/Obj for a batch.  problems: list of dict(obj (n,3), img (n,2), T_mm (4,4) or None).
    Returns list of dict(T, sub (local indices), n_ransac, n_mm, used_mm, iters_run, best_it, n_valid, Rt, Rt_hyp)."""
    npb = len(problems)
    off = np.zeros(npb + 1, np.int32)
    off[1:] = np.cumsum([len(p["obj"]) for p in problems])
    tot = int(off[-1])
    obj = np.ascontiguousarray(np.concatenate([np.asarray(p["obj"], np.float32).reshape(-1, 3) for p in problems]) if tot else np.zeros((0, 3), np.float32))
    img = np.ascontiguousarray(np.concatenate([np.asarray(p["img"], np.float32).reshape(-1, 2) for p in problems]) if tot else np.zeros((0, 2), np.float32))
    Tmm = np.zeros((npb, 16), np.float32); has = np.zeros(npb, np.uint8)
    for i, p in enumerate(problems):
        if p.get("T_mm") is not None:
            Tmm[i] = np.asarray(p["T_mm"], np.float32).reshape(16); has[i] = 1
    K = np.ascontiguousarray(K4, np.float32)
    T = np.zeros((npb, 16), np.float32); nsub = np.zeros(npb, np.int32); sub = np.zeros(max(tot, 1), np.int32)
    info = np.zeros((npb, 8), np.int32); Rt = np.zeros((npb, 12)); Rh = np.zeros((npb, 12))
    ctx.check(ctx.L.vdo_init_model_batch(ctx.h, C.c_int(npb), _ip(off), _fp(obj), _fp(img), _fp(K), C.c_int(iters), C.c_double(thr), C.c_double(conf),
                                         _fp(Tmm), has.ctypes.data_as(C.POINTER(C.c_ubyte)), _fp(T), _ip(nsub), _ip(sub), _ip(info), _dp(Rt), _dp(Rh)), "vdo_init_model_batch")
    out = []
    for i in range(npb):
        out.append(dict(T=T[i].reshape(4, 4).copy(), sub=sub[off[i]:off[i] + nsub[i]].copy(), n_ransac=int(info[i, 0]), n_mm=int(info[i, 1]), used_mm=bool(info[i, 2]),
                        iters_run=int(info[i, 4]), best_it=int(info[i, 5]), n_valid=int(info[i, 6]), Rt=Rt[i].copy(), Rt_hyp=Rh[i].copy()))
    return out


def renew_frame_info(cur: "Frame", tm_sta, stat_keys, samp_keys, max_num_sta, obj_inliers, obj_stat, sem_position, mod_label, obj_keys, obj_label,
                     tmp_keys, tmp_depth, tmp_sem, tmp_flow, tmp_corres, max_num_obj, K4, Twc):
    """vdo_renew_frame_info: Tracking::RenewFrameInfo on a resident frame.  Returns (static dict, object dict)."""
    ctx = cur.ctx
    f2 = lambda a: np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, 2))
    tm = _i32(tm_sta); sk = f2(stat_keys); sp = f2(samp_keys); ok = f2(obj_keys); ol = _i32(obj_label)
    n_obj = len(obj_inliers)
    ib = np.zeros(n_obj + 1, np.int32); ib[1:] = np.cumsum([len(x) for x in obj_inliers])
    ii = _i32(np.concatenate([np.asarray(x, np.int32) for x in obj_inliers])) if n_obj and ib[-1] else np.zeros(0, np.int32)
    st = np.ascontiguousarray(obj_stat, np.uint8); sem = _i32(sem_position); ml = _i32(mod_label)
    tk = f2(tmp_keys); td = np.ascontiguousarray(tmp_depth, np.float32); ts = _i32(tmp_sem); tf = f2(tmp_flow); tc = f2(tmp_corres)
    K = np.ascontiguousarray(K4, np.float32); T = np.ascontiguousarray(Twc, np.float32).reshape(16)
    cap_s = len(tm) + len(sp) + 8; cap_o = int(ib[-1]) + (n_obj + 1) * len(tk) + 8
    z2 = lambda n: np.zeros((n, 2), np.float32)
    s_keys, s_cor, s_flow, s_id, s_dep, s_3d = z2(cap_s), z2(cap_s), z2(cap_s), np.zeros(cap_s, np.int32), np.zeros(cap_s, np.float32), np.zeros((cap_s, 3), np.float32)
    o_keys, o_dep, o_cor, o_flow = z2(cap_o), np.zeros(cap_o, np.float32), z2(cap_o), z2(cap_o)
    o_sem, o_id, o_lab, o_3d = np.zeros(cap_o, np.int32), np.zeros(cap_o, np.int32), np.zeros(cap_o, np.int32), np.zeros((cap_o, 3), np.float32)
    ns, no = C.c_int(0), C.c_int(0)
    ub = lambda a: a.ctypes.data_as(C.POINTER(C.c_ubyte))
    ctx.check(ctx.L.vdo_renew_frame_info(cur.h_, C.c_int(len(tm)), _ip(tm), C.c_int(len(sk)), _fp(sk), C.c_int(len(sp)), _fp(sp), C.c_int(max_num_sta),
                                         C.c_int(n_obj), _ip(ib), _ip(ii), ub(st), _ip(sem), _ip(ml), C.c_int(len(ok)), _fp(ok), _ip(ol), C.c_int(len(tk)),
                                         _fp(tk), _fp(td), _ip(ts), _fp(tf), _fp(tc), C.c_int(max_num_obj), _fp(K), _fp(T),
                                         C.c_int(cap_s), C.byref(ns), _fp(s_keys), _fp(s_cor), _fp(s_flow), _ip(s_id), _fp(s_dep), _fp(s_3d),
                                         C.c_int(cap_o), C.byref(no), _fp(o_keys), _fp(o_dep), _fp(o_cor), _fp(o_flow), _ip(o_sem), _ip(o_id), _ip(o_lab), _fp(o_3d)),
              "vdo_renew_frame_info")
    a, b = ns.value, no.value
    return (dict(keys=s_keys[:a], corres=s_cor[:a], flow=s_flow[:a], inlier_id=s_id[:a], depth=s_dep[:a], p3d=s_3d[:a]),
            dict(keys=o_keys[:b], depth=o_dep[:b], corres=o_cor[:b], flow=o_flow[:b], sem=o_sem[:b], inlier_id=o_id[:b], label=o_lab[:b], p3d=o_3d[:b]))


SAMPLE_KEYS = 3000   # VDO_SAMPLE_KEYS


def sample_keys(ctx: Context, seeds, width: int, height: int):
    """vdo_sample_keys: Frame::SampleKeyPoints of a width x height image from cv::RNG(seed), one frame per seed, in one launch.
    Returns kx, ky (len(seeds) x SAMPLE_KEYS f32) and the launch's device time in ms (CUDA events)."""
    s = np.ascontiguousarray(np.asarray(seeds, np.int64) & 0xffffffff, np.uint32)
    kx, ky = np.zeros((len(s), SAMPLE_KEYS), np.float32), np.zeros((len(s), SAMPLE_KEYS), np.float32)
    ms = C.c_float(0)
    ctx.check(ctx.L.vdo_sample_keys(ctx.h, C.c_int(len(s)), C.c_int(width), C.c_int(height), s.ctypes.data_as(C.POINTER(C.c_uint)), _fp(kx), _fp(ky),
                                    C.byref(ms)), "vdo_sample_keys")
    return kx, ky, float(ms.value)


class TrackerParams(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("depth_factor", C.c_float), ("th_depth_bg", C.c_float), ("th_depth_obj", C.c_float), ("max_track_bg", C.c_int), ("max_track_obj", C.c_int),
                ("sf_mg_thres", C.c_float), ("sf_ds_thres", C.c_float), ("n_features", C.c_int), ("scale_factor", C.c_float), ("n_levels", C.c_int),
                ("ini_th_fast", C.c_int), ("min_th_fast", C.c_int), ("is_kitti", C.c_int), ("quirk", C.c_int), ("window_size", C.c_int),
                ("overlap_size", C.c_int), ("local_batch", C.c_int), ("dataset", C.c_int), ("use_sample_feature", C.c_int),
                ("sample_seed", C.c_uint)]


class Tracker:
    """vdo_tracker: System::TrackRGBD -> Tracking::GrabImageRGBD -> Tracking::Track on the device stages."""
    _INT = {"nStaInlierID", "vSemObjLabel", "vObjLabel", "nDynInlierID", "nModLabel", "nSemPosition", "bObjStat", "TemperalMatch_subset", "max_id", "f_id", "local_ba"}

    def __init__(self, ctx: Context, **overrides):
        self.ctx = ctx
        self.params = TrackerParams()
        ctx.L.vdo_tracker_params_default(C.byref(self.params))
        for k, v in overrides.items():
            setattr(self.params, k, v)
        self.h_ = C.c_void_p()
        ctx.check(ctx.L.vdo_tracker_create(ctx.h, C.byref(self.params), C.byref(self.h_)), "vdo_tracker_create")
        ctx.L.vdo_tracker_last_error.restype = C.c_char_p

    def track(self, gray, depth, flow, mask, gt_ids, writeback=True):
        """depth (f32 h x w) and mask (i32 h x w) must be C-contiguous arrays; with writeback they are mutated like the reference's cv::Mat."""
        assert depth.dtype == np.float32 and depth.flags.c_contiguous and mask.dtype == np.int32 and mask.flags.c_contiguous
        g = np.ascontiguousarray(gray, np.uint8); f = np.ascontiguousarray(flow, np.float32)
        ids = _i32(gt_ids)
        T = np.zeros((4, 4), np.float32)
        h, w = g.shape
        assert depth.shape == (h, w) and mask.shape == (h, w) and f.shape == (h, w, 2)
        rc = self.ctx.L.vdo_tracker_track(self.h_, C.c_int(w), C.c_int(h), g.ctypes.data_as(C.POINTER(C.c_ubyte)), _fp(depth), _fp(f), _ip(mask), C.c_int(len(ids)),
                                          _ip(ids), C.c_int(int(writeback)), _fp(T))
        if rc != 0:
            raise VdoError(f"vdo_tracker_track failed ({rc}): {self.ctx.L.vdo_tracker_last_error(self.h_).decode()}")
        return T

    def track_tensors(self, image, depth, flow, mask, gt_ids, writeback=True, rgb=True):
        """vdo_tracker_track_dev on torch CUDA tensors in any strides (layouts: see _dev_plane), ordered after the work queued on torch's
        current stream.  With writeback, depth and mask are updated in place like track() does to its arrays.  Returns Tcw."""
        w, h = self.params.width, self.params.height
        planes, stream = _dev_planes(self.ctx, w, h, rgb, image=image, depth=depth, flow=flow, mask=mask)
        ids = _i32(gt_ids)
        T = np.zeros((4, 4), np.float32)
        rc = self.ctx.L.vdo_tracker_track_dev(self.h_, C.c_int(w), C.c_int(h), *[C.byref(p) for p in planes], C.c_int(len(ids)), _ip(ids),
                                              C.c_int(int(writeback)), C.c_uint64(stream), _fp(T))
        if rc != 0:
            raise VdoError(f"vdo_tracker_track_dev failed ({rc}): {self.ctx.L.vdo_tracker_last_error(self.h_).decode()}")
        return T

    def get(self, name: str):
        n = C.c_int(0)
        self.ctx.check(self.ctx.L.vdo_tracker_get(self.h_, name.encode(), None, C.c_int(0), C.byref(n)), "vdo_tracker_get")
        out = np.zeros(max(n.value, 1), np.int32 if name in self._INT else np.float32)
        self.ctx.check(self.ctx.L.vdo_tracker_get(self.h_, name.encode(), out.ctypes.data_as(C.c_void_p), C.c_int(len(out)), C.byref(n)), "vdo_tracker_get")
        return out[:n.value]

    _GI = {"prior_v", "se3e_ij", "obs_cp", "ter_pph"}

    def graph_export(self, mode: int):
        """arrays the Map->graph builder hands to vdo_graph_* (mode 0 partial window, 1 full batch), in make_batch_graph layout"""
        g = {}
        shapes = dict(se3=(-1, 12), pt=(-1, 3), prior_Z=(-1, 12), se3e_Z=(-1, 12), obs_z=(-1, 3), se3e_ij=(-1, 2), obs_cp=(-1, 2), ter_pph=(-1, 3))
        for name in ("se3", "pt", "prior_v", "prior_Z", "prior_w", "se3e_ij", "se3e_Z", "se3e_w", "se3e_delta", "obs_cp", "obs_z", "obs_w", "obs_delta", "ter_pph",
                     "ter_w", "ter_delta"):
            n = C.c_int(0)
            self.ctx.check(self.ctx.L.vdo_tracker_graph_export(self.h_, C.c_int(mode), name.encode(), None, C.c_int(0), C.byref(n)), "vdo_tracker_graph_export")
            out = np.zeros(max(n.value, 1), np.int32 if name in self._GI else np.float64)
            self.ctx.check(self.ctx.L.vdo_tracker_graph_export(self.h_, C.c_int(mode), name.encode(), out.ctypes.data_as(C.c_void_p), C.c_int(len(out)), C.byref(n)),
                           "vdo_tracker_graph_export")
            g[name] = out[:n.value].reshape(shapes.get(name, -1))
        return g

    def batch_optimize(self, mode: int, **opt):
        o = LMOptions(); self.ctx.L.vdo_lm_options_default(C.byref(o))
        st = LMStats(); info = np.zeros(6, np.int32)
        po = None
        if opt:
            for k, v in opt.items():
                setattr(o, k, v)
            po = C.byref(o)
        rc = self.ctx.L.vdo_tracker_batch_optimize(self.h_, C.c_int(mode), po, C.byref(st), _ip(info))
        if rc != 0:
            raise VdoError(f"vdo_tracker_batch_optimize failed ({rc}): {self.ctx.L.vdo_tracker_last_error(self.h_).decode()}")
        r = st.asdict(); r["sizes"] = dict(zip(["n_se3", "n_pt", "n_prior", "n_se3_edges", "n_obs", "n_ternary"], info.tolist()))
        return r

    def map_push(self, feat_sta, dep_sta, p3d_sta, feat_dyn, dep_dyn, p3d_dyn, camera_pose, asso_sta=None, asso_dyn=None, feat_label=None,
                 rigid_motion=None, rm_label=None):
        """vdo_tracker_map_push: one frame of an externally built map (frame 0 without associations and motions).  feat (n, 2), p3d (n, 3),
        camera_pose 4x4 Twc, rigid_motion (m, 4, 4) with entry 0 the camera, rm_label (m,)."""
        f32 = lambda a, w: np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, w) if w else np.asarray(a, np.float32).reshape(-1))
        fs, ds, ps, fd, dd, pd = f32(feat_sta, 2), f32(dep_sta, 0), f32(p3d_sta, 3), f32(feat_dyn, 2), f32(dep_dyn, 0), f32(p3d_dyn, 3)
        P = f32(camera_pose, 16)
        keep = [_i32(a) if a is not None else None for a in (asso_sta, asso_dyn, feat_label, rm_label)]
        M = None if rigid_motion is None else f32(rigid_motion, 16)
        n_mot = 0 if M is None else len(M)
        rc = self.ctx.L.vdo_tracker_map_push(self.h_, C.c_int(len(fs)), _fp(fs), _fp(ds), _fp(ps), None if keep[0] is None else _ip(keep[0]), C.c_int(len(fd)),
                                             _fp(fd), _fp(dd), _fp(pd), None if keep[1] is None else _ip(keep[1]), None if keep[2] is None else _ip(keep[2]),
                                             _fp(P), C.c_int(n_mot), None if M is None else _fp(M), None if keep[3] is None else _ip(keep[3]))
        if rc != 0:
            raise VdoError(f"vdo_tracker_map_push failed ({rc}): {self.ctx.L.vdo_tracker_last_error(self.h_).decode()}")

    def tracklets(self, kind: int) -> dict:
        """vdo_tracker_tracklets_get: the tracklet tables the graph builder reads (kind 0 static, 1 dynamic)"""
        out = {}
        for name in ("trk", "pos", "prev_frame", "prev_feat", "len", "head_frame", "head_feat", "obj_lab"):
            n = C.c_int(0)
            self.ctx.check(self.ctx.L.vdo_tracker_tracklets_get(self.h_, C.c_int(kind), name.encode(), None, C.c_int(0), C.byref(n)), "vdo_tracker_tracklets_get")
            a = np.zeros(max(n.value, 1), np.int32)
            self.ctx.check(self.ctx.L.vdo_tracker_tracklets_get(self.h_, C.c_int(kind), name.encode(), _ip(a), C.c_int(len(a)), C.byref(n)), "vdo_tracker_tracklets_get")
            out[name] = a[:n.value]
        return out

    def map_get(self, name: str):
        n = C.c_int(0)
        self.ctx.check(self.ctx.L.vdo_tracker_map_get(self.h_, name.encode(), None, C.c_int(0), C.byref(n)), "vdo_tracker_map_get")
        out = np.zeros(max(n.value, 1), np.int32 if name in ("vnRMLabel", "n_frames", "n_per_frame") else np.float32)
        self.ctx.check(self.ctx.L.vdo_tracker_map_get(self.h_, name.encode(), out.ctypes.data_as(C.c_void_p), C.c_int(len(out)), C.byref(n)), "vdo_tracker_map_get")
        return out[:n.value]

    def close(self):
        if getattr(self, "h_", None):
            self.ctx.L.vdo_tracker_destroy(self.h_)
            self.h_ = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- per-frame input files of the reference's driver (vdo_io_*, host-only; SURVEY 8(f) N3) ----
def io_read_png(ctx: "Context", path: str) -> np.ndarray:
    """cv::imread(path, UNCHANGED): uint8 / uint16, HxW or HxWxC in BGR[A] order."""
    w, h, ch, bd = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    ctx.check(ctx.L.vdo_io_png_info(path.encode(), C.byref(w), C.byref(h), C.byref(ch), C.byref(bd)), f"vdo_io_png_info({path})")
    a = np.zeros((h.value, w.value, ch.value), np.uint8 if bd.value == 8 else np.uint16)
    ctx.check(ctx.L.vdo_io_read_png(path.encode(), a.ctypes.data_as(C.c_void_p), C.c_size_t(a.nbytes)), f"vdo_io_read_png({path})")
    return a[:, :, 0] if ch.value == 1 else a


def io_read_png_gray_f32(ctx: "Context", path: str, w: int, h: int) -> np.ndarray:
    a = np.zeros((h, w), np.float32)
    ctx.check(ctx.L.vdo_io_read_png_gray_f32(path.encode(), a.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(w), C.c_int(h)), f"vdo_io_read_png_gray_f32({path})")
    return a


def io_read_flo(ctx: "Context", path: str) -> np.ndarray:
    w, h = C.c_int(), C.c_int()
    ctx.check(ctx.L.vdo_io_flo_info(path.encode(), C.byref(w), C.byref(h)), f"vdo_io_flo_info({path})")
    a = np.zeros((h.value, w.value, 2), np.float32)
    ctx.check(ctx.L.vdo_io_read_flo(path.encode(), a.ctypes.data_as(C.POINTER(C.c_float)), C.c_size_t(a.size)), f"vdo_io_read_flo({path})")
    return a


def io_read_mask_txt(ctx: "Context", path: str, w: int, h: int) -> np.ndarray:
    a = np.zeros((h, w), np.int32)
    ctx.check(ctx.L.vdo_io_read_mask_txt(path.encode(), _ip(a), C.c_int(w), C.c_int(h)), f"vdo_io_read_mask_txt({path})")
    return a


# ---- result files / metrics (vdo_results_*, vdo_metric_error; host-only; SURVEY 8(f) N4) ----
def _flatten_frames(per_frame):
    """list (frames) of lists (entries) of arrays -> (counts i32, stacked f32 array)"""
    cnt = np.array([len(f) for f in per_frame], np.int32)
    flat = [np.asarray(m, np.float32) for f in per_frame for m in f]
    return cnt, (np.stack(flat) if flat else np.zeros((0, 4, 4), np.float32))


def results_write_poses(ctx: "Context", path: str, poses, start_frame: int = 0):
    P = np.ascontiguousarray(np.asarray(poses, np.float32).reshape(-1, 16))
    ctx.check(ctx.L.vdo_results_write_poses(path.encode(), C.c_int(start_frame), C.c_int(len(P)), _fp(P)), "vdo_results_write_poses")


def results_write_object_motions(ctx: "Context", path: str, motions, labels, pose_pre=None, start_frame: int = 0):
    cnt, H = _flatten_frames(motions)
    H = np.ascontiguousarray(H.reshape(-1, 16))
    lab = np.ascontiguousarray(np.concatenate([np.asarray(l, np.int32) for l in labels]) if len(labels) else np.zeros(0, np.int32))
    L = None
    if pose_pre is not None:
        L = np.ascontiguousarray(_flatten_frames(pose_pre)[1].reshape(-1, 16))
    ctx.check(ctx.L.vdo_results_write_object_motions(path.encode(), C.c_int(start_frame), C.c_int(len(cnt)), _ip(cnt), _ip(lab), _fp(H),
                                                     _fp(L) if L is not None else None), "vdo_results_write_object_motions")


def results_write_object_centres(ctx: "Context", path: str, centres, labels, start_frame: int = 0):
    cnt = np.array([len(f) for f in centres], np.int32)
    Cn = np.ascontiguousarray(np.concatenate([np.asarray(f, np.float32).reshape(-1, 3) for f in centres]) if len(centres) else np.zeros((0, 3), np.float32))
    lab = np.ascontiguousarray(np.concatenate([np.asarray(l, np.int32) for l in labels]) if len(labels) else np.zeros(0, np.int32))
    ctx.check(ctx.L.vdo_results_write_object_centres(path.encode(), C.c_int(start_frame), C.c_int(len(cnt)), _ip(cnt), _ip(lab), _fp(Cn)), "vdo_results_write_object_centres")


def metric_error(ctx: "Context", cam, cam_gt, motions, pose_pre, motions_gt, labels, obj_stat, max_id: int) -> dict:
    Cm = np.ascontiguousarray(np.asarray(cam, np.float32).reshape(-1, 16)); Cg = np.ascontiguousarray(np.asarray(cam_gt, np.float32).reshape(-1, 16))
    cnt, H = _flatten_frames(motions)
    H = np.ascontiguousarray(H.reshape(-1, 16)); L = np.ascontiguousarray(_flatten_frames(pose_pre)[1].reshape(-1, 16)); G = np.ascontiguousarray(_flatten_frames(motions_gt)[1].reshape(-1, 16))
    lab = np.ascontiguousarray(np.concatenate([np.asarray(l, np.int32) for l in labels]))
    st = np.ascontiguousarray(np.concatenate([np.asarray(s, np.uint8) for s in obj_stat]))
    out = np.zeros(4, np.float32); n = max(max_id - 1, 0)
    et, er, ec = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.int32)
    ctx.check(ctx.L.vdo_metric_error(C.c_int(len(Cm)), _fp(Cm), _fp(Cg), C.c_int(len(cnt)), _ip(cnt), _ip(lab), st.ctypes.data_as(C.POINTER(C.c_ubyte)), _fp(H), _fp(L), _fp(G),
                                     C.c_int(max_id), _fp(out), _fp(et), _fp(er), _ip(ec)), "vdo_metric_error")
    return {"cam_t": float(out[0]), "cam_r": float(out[1]), "obj_t": float(out[2]), "obj_r": float(out[3]), "each_t": et, "each_r": er, "each_count": ec}


def batch_optimize_trackers(trackers, mode: int, **opt):
    """vdo_tracker_batch_optimize_batch: Tracker.batch_optimize(mode, **opt) of several trackers of one context in one call (one graph
    build, one optimize_batch of all their graphs, one write-back per map).  Tracker i ends where trackers[i].batch_optimize(mode, **opt)
    takes it.  Returns one dict per tracker with the keys of Tracker.batch_optimize (ms_* and kernel_launches describe the whole call)."""
    trackers = list(trackers)
    if not trackers:
        raise VdoError("batch_optimize_trackers: no trackers")
    ctx = trackers[0].ctx
    n = len(trackers)
    o = LMOptions(); ctx.L.vdo_lm_options_default(C.byref(o))
    po = None
    if opt:
        for k, v in opt.items():
            setattr(o, k, v)
        po = C.byref(o)
    st = (LMStats * n)()
    info = np.zeros((n, 6), np.int32)
    hs = (C.c_void_p * n)(*[t.h_.value if t is not None and t.h_ else None for t in trackers])
    rc = ctx.L.vdo_tracker_batch_optimize_batch(hs, C.c_int(n), C.c_int(mode), po, st, _ip(info))
    if rc != 0:
        who = trackers[0].h_ if trackers[0] is not None else None
        msg = ctx.L.vdo_tracker_last_error(who).decode() if who else ""
        raise VdoError(f"vdo_tracker_batch_optimize_batch failed ({rc}): {msg}")
    out = []
    for i in range(n):
        r = st[i].asdict()
        r["sizes"] = dict(zip(["n_se3", "n_pt", "n_prior", "n_se3_edges", "n_obs", "n_ternary"], info[i].tolist()))
        out.append(r)
    return out


def _track_list(name, entry, own_size, trackers, images, depths, flows, masks, gt_ids, writeback, rgb):
    """the body of track_tensors_batch / track_tensors_mixed (name), calling the C function entry; own_size: each tracker's planes are
    checked against its own width and height, else against trackers[0]'s"""
    trackers = list(trackers)
    B = len(trackers)
    if B == 0:
        raise ValueError(f"{name}: no trackers")
    ins = {}
    for kind, v in (("image", images), ("depth", depths), ("flow", flows), ("mask", masks)):
        items = list(v.unbind(0)) if hasattr(v, "unbind") else list(v)
        if len(items) != B:
            raise ValueError(f"{kind}: {len(items)} planes for {B} trackers")
        ins[kind] = items
    gt = [_i32(g) for g in gt_ids]
    if len(gt) != B:
        raise ValueError(f"gt_ids: {len(gt)} id lists for {B} trackers")
    ctx = trackers[0].ctx
    arrays = {k: (DevPlane * B)() for k in ins}
    stream = 0
    for i in range(B):
        p = trackers[i if own_size else 0].params
        try:
            planes, stream = _dev_planes(ctx, p.width, p.height, rgb, **{k: ins[k][i] for k in ("image", "depth", "flow", "mask")})
        except ValueError as e:
            raise ValueError(f"trackers[{i}]: {e}") if own_size else e
        for k, pl in zip(("image", "depth", "flow", "mask"), planes):
            arrays[k][i] = pl
    begin = np.zeros(B + 1, np.int32)
    begin[1:] = np.cumsum([len(g) for g in gt])
    ids = np.concatenate(gt).astype(np.int32) if begin[-1] else np.zeros(1, np.int32)
    handles = (C.c_void_p * B)(*[t.h_.value for t in trackers])
    T = np.zeros((B, 4, 4), np.float32)
    rc = getattr(ctx.L, entry)(handles, C.c_int(B), arrays["image"], arrays["depth"], arrays["flow"], arrays["mask"], _ip(begin), _ip(ids),
                               C.c_int(int(writeback)), C.c_uint64(stream), _fp(T))
    if rc != 0:
        raise VdoError(f"{entry} failed ({rc}): {ctx.L.vdo_tracker_last_error(trackers[0].h_).decode()}")
    return T


def track_tensors_batch(trackers, images, depths, flows, masks, gt_ids, writeback=True, rgb=True):
    """vdo_tracker_track_batch_dev: advance B trackers by one frame each, every batched stage as one set of launches.  Tracker i gets
    exactly what trackers[i].track_tensors(images[i], ...) gives it.  Each input is a list of B tensors or a tensor with a leading batch
    dimension; every element is passed as a view (layouts: see _dev_plane), nothing is copied.  gt_ids: B sequences of ids.  The trackers
    must share a context, the image size and the ORB settings.  Returns Tcw as a (B, 4, 4) array."""
    return _track_list("track_tensors_batch", "vdo_tracker_track_batch_dev", False, trackers, images, depths, flows, masks, gt_ids, writeback, rgb)


def track_tensors_mixed(trackers, images, depths, flows, masks, gt_ids, writeback=True, rgb=True):
    """vdo_tracker_track_mixed_dev: track_tensors_batch for trackers that may also differ in image size and ORB settings (KITTI and OMD
    sequences, the cameras of one vehicle) -- still one set of launches per batched stage.  images, depths, flows, masks: lists of B
    tensors (or tensors with a leading batch dimension when the sizes agree), each checked against its own tracker's width and height;
    a wrong shape, dtype or device raises ValueError before the C call.  Returns Tcw as a (B, 4, 4) array."""
    return _track_list("track_tensors_mixed", "vdo_tracker_track_mixed_dev", True, trackers, images, depths, flows, masks, gt_ids, writeback, rgb)


class _Estimator:
    """A device-chain handle (vdo_<_NAME>_create / _destroy / _info): h_, close(), and info() as a dict of the first len(_INFO)
    values of the info entry."""
    _NAME: str
    _INFO: tuple

    def __init__(self, ctx: Context, *args):
        self.ctx = ctx
        self.h_ = C.c_void_p()
        entry = f"vdo_{self._NAME}_create"
        ctx.check(getattr(ctx.L, entry)(ctx.h, *args, C.byref(self.h_)), entry)

    def info(self) -> dict:
        out = (C.c_int64 * 4)()
        entry = f"vdo_{self._NAME}_info"
        self.ctx.check(getattr(self.ctx.L, entry)(self.h_, out), entry)
        return dict(zip(self._INFO, list(out)))

    def close(self):
        if getattr(self, "h_", None):
            getattr(self.ctx.L, f"vdo_{self._NAME}_destroy")(self.h_)
            self.h_ = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# An entry's device outputs are declared once, as name -> (torch dtype name, trailing shape) with one row per pair; a str in the trailing
# shape names a size of the call (a capacity, k).  The C struct of their pointers has the fields <name>_dev in table order.
def _out_shapes(table: dict, P: int, **sizes) -> dict:
    """name -> (torch dtype, shape) of the outputs of P pairs"""
    import torch
    return {k: (getattr(torch, dt), (P,) + tuple(sizes[d] if isinstance(d, str) else d for d in tail)) for k, (dt, tail) in table.items()}


def _empty_outputs(ctx: Context, shapes: dict) -> dict:
    import torch
    dev = torch.device("cuda", ctx.device)
    return {k: torch.empty(shp, dtype=dt, device=dev) for k, (dt, shp) in shapes.items()}


def _out_ptrs(ctx: Context, out: dict, shapes: dict, table: dict) -> list:
    """the device pointers of out in table order (None for a name not in shapes), each tensor checked against shapes"""
    for k, (dt, shp) in shapes.items():
        _cuda_tensor(ctx, f"out[{k!r}]", out.get(k), dt, shp)
    return [out[k].data_ptr() if k in shapes else None for k in table]


class OrbBatchOut(C.Structure):
    """vdo_orb_batch_out: device pointers of the outputs of vdo_orb_extract_batch_dev"""
    _fields_ = [(k, C.c_void_p) for k in ("x_dev", "y_dev", "octave_dev", "response_dev", "angle_dev", "size_dev", "desc_dev", "count_dev",
                                          "n_candidates_dev", "status_dev")]


ORB_STATUS_NODE_BOUND, ORB_STATUS_INPUT, ORB_STATUS_ROUNDS = 1, 2, 4


class OrbExtractor(_Estimator):
    """vdo_orb_extractor: ORBextractor::operator() for batches of device images, entirely on the GPU.

    One extractor serves up to max_batch frames of width x height with fixed ORB settings (the ORBextractor.* keys; defaults as
    Frame.orb_extract).  extract() enqueues the whole path on torch's current stream and never synchronises; frame i of the result equals
    Frame.upload + orb_extract + orb_describe on the same gray image, bit for bit."""

    _NAME, _INFO = "orb_extractor", ("capacity", "device_bytes", "n_levels", "max_batch")
    _PER_KP = (("x", "float32"), ("y", "float32"), ("octave", "int32"), ("response", "float32"), ("angle", "float32"), ("size", "int32"))

    def __init__(self, ctx: Context, width: int, height: int, max_batch: int, n_features: int = 2500, scale_factor: float = 1.2,
                 n_levels: int = 8, ini_th_fast: int = 20, min_th_fast: int = 7):
        self.w, self.h, self.max_batch, self.n_levels = int(width), int(height), int(max_batch), int(n_levels)
        super().__init__(ctx, C.c_int(width), C.c_int(height), C.c_int(max_batch), C.c_int(n_features), C.c_float(scale_factor),
                         C.c_int(n_levels), C.c_int(ini_th_fast), C.c_int(min_th_fast))
        self.capacity = self.info()["capacity"]

    def empty_outputs(self, batch: int, describe: bool = True) -> dict:
        """output tensors for `batch` frames (pass as extract(..., out=)): per keypoint (batch, capacity), descriptors (batch, capacity, 32)
        u8, count / status (batch,) and n_candidates (batch, n_levels) int32"""
        import torch
        dev = torch.device("cuda", self.ctx.device)
        out = {k: torch.empty((batch, self.capacity), dtype=getattr(torch, dt), device=dev) for k, dt in self._PER_KP}
        if describe:
            out["descriptors"] = torch.empty((batch, self.capacity, 32), dtype=torch.uint8, device=dev)
        out["count"] = torch.empty(batch, dtype=torch.int32, device=dev)
        out["n_candidates"] = torch.empty((batch, self.n_levels), dtype=torch.int32, device=dev)
        out["status"] = torch.empty(batch, dtype=torch.int32, device=dev)
        return out

    def _check_out(self, out: dict, n: int, describe: bool):
        import torch
        want = {k: (getattr(torch, dt), (self.capacity,)) for k, dt in self._PER_KP}
        want.update(count=(torch.int32, ()), n_candidates=(torch.int32, (self.n_levels,)), status=(torch.int32, ()))
        if describe:
            want["descriptors"] = (torch.uint8, (self.capacity, 32))
        for k, (dt, tail) in want.items():
            t = out.get(k)
            if not isinstance(t, torch.Tensor):
                raise ValueError(f"out[{k!r}]: missing (see empty_outputs)")
            if t.device.type != "cuda" or t.device.index != self.ctx.device or t.dtype != dt or not t.is_contiguous() \
                    or t.dim() != 1 + len(tail) or tuple(t.shape[1:]) != tail or t.shape[0] < n:
                raise ValueError(f"out[{k!r}]: {t.dtype} {tuple(t.shape)} on {t.device}, expected a contiguous {dt} ({n}+, "
                                 f"{', '.join(map(str, tail))}) tensor on cuda:{self.ctx.device}")

    def extract(self, images, describe: bool = True, out: dict | None = None, rgb: bool = True) -> dict:
        """images: a (B,H,W), (B,H,W,C) or (B,C,H,W) u8 CUDA tensor or a list of (H,W) / (H,W,C) / (C,H,W) ones, any strides; C in {3, 4} is
        converted to gray on the device (RGB(A) order when rgb, else BGR(A)).  Returns CUDA tensors: x, y, octave, response, angle, size
        (B, capacity), descriptors (B, capacity, 32) when describe, count (B,), n_candidates (B, n_levels), status (B,); frame i's keypoints
        are the first count[i] entries of its row.  out: tensors from empty_outputs() with at least B rows, written in place (the call then
        allocates nothing and can be captured in a CUDA graph).  Enqueued on torch's current stream; nothing is synchronised."""
        import torch
        if isinstance(images, torch.Tensor):
            if images.dim() not in (3, 4):
                raise ValueError(f"images: shape {tuple(images.shape)}; expected (B,H,W), (B,H,W,C) or (B,C,H,W), or a list of frames")
            items = list(images.unbind(0))
        else:
            items = list(images)
        n = len(items)
        if n < 1 or n > self.max_batch:
            raise ValueError(f"images: {n} frames, the extractor takes 1 .. {self.max_batch}")
        planes = (DevPlane * n)()
        for i, t in enumerate(items):
            planes[i] = _dev_plane(self.ctx, "image", t, self.w, self.h, rgb)
        if out is None:
            out = self.empty_outputs(n, describe)
        self._check_out(out, n, describe)
        o = OrbBatchOut(*[out[k].data_ptr() if (k in out and (k != "descriptors" or describe)) else None
                          for k in ("x", "y", "octave", "response", "angle", "size", "descriptors", "count", "n_candidates", "status")])
        self.ctx.check(self.ctx.L.vdo_orb_extract_batch_dev(self.h_, C.c_int(n), planes, C.byref(o), C.c_uint64(_torch_stream(self.ctx))),
                       "vdo_orb_extract_batch_dev")
        keys = [k for k, _ in self._PER_KP] + (["descriptors"] if describe else []) + ["count", "n_candidates", "status"]
        return {k: out[k][:n] for k in keys}


def orb_debug_octree(ctx: Context, keys, minX: int, maxX: int, minY: int, maxY: int, N: int):
    """TEST HOOK (vdo_orb_debug_octree): the device octree alone.  keys: (n, 3) x, y (relative to minX, minY), response.  Returns (kept keys
    as an (m, 3) float32 array in list order, status bits)."""
    k = np.ascontiguousarray(np.asarray(keys, np.float32).reshape(-1, 3))
    n = len(k)
    x, y, r = (np.ascontiguousarray(k[:, j]) for j in range(3))
    ox, oy, orr = (np.zeros(max(n, 1), np.float32) for _ in range(3))
    m, st = C.c_int(0), C.c_int(0)
    ctx.check(ctx.L.vdo_orb_debug_octree(ctx.h, C.c_int(n), _fp(x), _fp(y), _fp(r), C.c_int(minX), C.c_int(maxX), C.c_int(minY), C.c_int(maxY), C.c_int(N),
                                         _fp(ox), _fp(oy), _fp(orr), C.byref(m), C.byref(st)), "vdo_orb_debug_octree")
    return np.stack([ox[:m.value], oy[:m.value], orr[:m.value]], 1), st.value


class OrbDescSet(C.Structure):
    """vdo_orb_desc_set: device pointers of one descriptor set (the layout OrbExtractor.extract writes)"""
    _fields_ = [("desc_dev", C.c_void_p), ("x_dev", C.c_void_p), ("y_dev", C.c_void_p), ("count_dev", C.c_void_p),
                ("n_frames", C.c_int32), ("cap", C.c_int32)]


class OrbMatchOpts(C.Structure):
    _fields_ = [("k", C.c_int32), ("cross_check", C.c_int32), ("radius", C.c_float)]


_MATCH_OUT = {"idx": ("int32", ("query_cap", "k")), "dist": ("int32", ("query_cap", "k")), "rev_idx": ("int32", ("train_cap",)), "status": ("int32", ())}


class OrbMatchOut(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _MATCH_OUT]


ORB_MATCH_STATUS_QUERY_COUNT, ORB_MATCH_STATUS_TRAIN_COUNT = 1, 2


def _cuda_tensor(ctx: Context, what: str, t, dtype, shape: tuple):
    """ValueError unless t is a contiguous CUDA tensor on the context's device with this dtype and shape (None: any extent)"""
    import torch
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{what}: expected a torch tensor, got {type(t).__name__}")
    if t.device.type != "cuda" or t.device.index != ctx.device or t.dtype != dtype or not t.is_contiguous() or t.dim() != len(shape) \
            or any(s is not None and s != n for s, n in zip(shape, t.shape)):
        want = ", ".join("*" if s is None else str(s) for s in shape)
        raise ValueError(f"{what}: {t.dtype} {tuple(t.shape)} on {t.device}, expected a contiguous {dtype} ({want}) tensor on cuda:{ctx.device}")
    return t


def _desc_set(ctx: Context, what: str, s: dict, positions: bool) -> OrbDescSet:
    import torch
    d = _cuda_tensor(ctx, f"{what}['descriptors']", s.get("descriptors"), torch.uint8, (None, None, 32))
    F, cap = int(d.shape[0]), int(d.shape[1])
    cnt = _cuda_tensor(ctx, f"{what}['count']", s.get("count"), torch.int32, (F,))
    x = y = None
    if positions:
        x = _cuda_tensor(ctx, f"{what}['x']", s.get("x"), torch.float32, (F, cap))
        y = _cuda_tensor(ctx, f"{what}['y']", s.get("y"), torch.float32, (F, cap))
    return OrbDescSet(d.data_ptr(), x.data_ptr() if x is not None else None, y.data_ptr() if y is not None else None, cnt.data_ptr(), F, cap)


def _match_shapes(P: int, query_cap: int, train_cap: int, k: int, cross_check: bool) -> dict:
    sh = _out_shapes(_MATCH_OUT, P, query_cap=query_cap, train_cap=train_cap, k=k)
    if not cross_check:
        del sh["rev_idx"]
    return sh


def orb_match_empty_outputs(ctx: Context, n_pairs: int, query_cap: int, train_cap: int, k: int = 2, cross_check: bool = False) -> dict:
    """output tensors of orb_match for n_pairs pairs (pass as orb_match(..., out=)): idx, dist (n_pairs, query_cap, k), status (n_pairs,)
    int32, and rev_idx (n_pairs, train_cap) int32 when cross_check"""
    out = _empty_outputs(ctx, _match_shapes(n_pairs, query_cap, train_cap, k, cross_check))
    return {kk: out[kk] for kk in ("idx", "dist", "status", "rev_idx") if kk in out}   # rev_idx last


def orb_match(ctx: Context, query: dict, train: dict, pairs, k: int = 2, radius: float | None = None, pred=None, cross_check: bool = False,
              out: dict | None = None) -> dict:
    """vdo_orb_match_batch_dev: cv2.BFMatcher(NORM_HAMMING).knnMatch of descriptor sets held on the GPU, for up to 64 pairs per call.

    query, train: OrbExtractor.extract() results (or dicts with the same 'descriptors' (F, cap, 32) u8, 'count' (F,) int32 and, for a
    train set searched in a window, 'x' / 'y' (F, cap) float32 CUDA tensors); they may be the same dict.  pairs: P (query frame, train
    frame) index pairs.  For query keypoint i < count[q] of pair p, idx[p, i] / dist[p, i] hold the k in {1, 2} nearest train keypoints
    j < count[t] by Hamming distance, in increasing distance with ties to the lower j, and -1 where a query has fewer than k candidates;
    slots past count[q] are left as they were.
      radius, pred: search window: train j is a candidate only if |x_t[j] - pred[p, i, 0]| <= radius and |y_t[j] - pred[p, i, 1]| <= radius
        (pred: (P, query cap, 2) float32, e.g. the query position plus the flow at it).
      cross_check (k = 1): keep i -> j only if i is j's best query (ties to the lower i); rev_idx (P, train cap) then holds each train
        keypoint's best query.
    Lowe's ratio test on a k = 2 result: good = dist[..., 0] < ratio * dist[..., 1].
    Returns CUDA tensors idx, dist (P, query cap, k), rev_idx when cross_check, and status (P,): ORB_MATCH_STATUS_* bits for a count outside
    0 .. cap.  out: tensors from orb_match_empty_outputs() with P rows, written in place (the call then allocates nothing and can be
    captured in a CUDA graph).  Enqueued on torch's current stream; nothing is synchronised.  ValueError on a wrong dtype, shape or device."""
    import torch
    win = radius is not None and radius > 0
    if k not in (1, 2):
        raise ValueError(f"k = {k}; expected 1 or 2")
    if cross_check and k != 1:
        raise ValueError("cross_check needs k = 1")
    pr = np.ascontiguousarray(np.asarray(pairs, dtype=np.int64).reshape(-1, 2)).astype(np.int32)
    P = len(pr)
    if P < 1 or P > 64:
        raise ValueError(f"pairs: {P} pairs, a call takes 1 .. 64")
    qs = _desc_set(ctx, "query", query, False)
    ts = _desc_set(ctx, "train", train, win)
    pred_ptr = None
    if win:
        if pred is None:
            raise ValueError("radius needs pred (P, query cap, 2)")
        pred_ptr = _cuda_tensor(ctx, "pred", pred, torch.float32, (P, qs.cap, 2)).data_ptr()
    shapes = _match_shapes(P, qs.cap, ts.cap, k, cross_check)
    if out is None:
        out = _empty_outputs(ctx, shapes)
    o = OrbMatchOut(*_out_ptrs(ctx, out, shapes, _MATCH_OUT))
    opts = OrbMatchOpts(k, int(cross_check), float(radius) if win else 0.0)
    ctx.check(ctx.L.vdo_orb_match_batch_dev(ctx.h, C.c_int(P), pr.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(qs), C.byref(ts),
                                            C.c_void_p(pred_ptr), C.byref(opts), C.byref(o), C.c_uint64(_torch_stream(ctx))), "vdo_orb_match_batch_dev")
    return {kk: out[kk] for kk in shapes}


class PnpMatchOpts(C.Structure):
    _fields_ = [("k", C.c_int32), ("ratio", C.c_float), ("max_depth", C.c_float), ("iters", C.c_int32), ("thr", C.c_double), ("conf", C.c_double)]


_PNP_OUT = {"T": ("float32", (4, 4)), "Rt": ("float64", (12,)), "inlier": ("uint8", ("query_cap",)), "n_corr": ("int32", ()),
            "n_inlier": ("int32", ()), "info": ("int32", (4,))}


class PnpOut(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _PNP_OUT]


class PoseRefineOpts(C.Structure):
    _fields_ = [("k", C.c_int32), ("ratio", C.c_float), ("max_depth", C.c_float), ("quirk", C.c_int32)]


_REFINE_OUT = {"T": ("float32", (4, 4)), "flow": ("float64", ("query_cap", 2)), "inlier": ("uint8", ("query_cap",)), "n_points": ("int32", ()),
               "stats": ("float64", (8,)), "status": ("int32", ())}


class PoseRefineOut(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _REFINE_OUT]


PNP_STATUS_QUERY_COUNT, PNP_STATUS_TRAIN_COUNT, PNP_STATUS_FEW_POINTS, PNP_STATUS_NO_MODEL = 1, 2, 4, 8


def _per_pair(what: str, a, P: int, shape: tuple) -> np.ndarray:
    """host float32 array of one value (shape) for all pairs, or one per pair (P, *shape) -> (P, *shape) C-contiguous"""
    v = np.asarray(a, dtype=np.float32)
    if v.shape == shape:
        v = np.broadcast_to(v, (P,) + shape)
    if v.shape != (P,) + shape:
        raise ValueError(f"{what}: shape {v.shape}; expected {shape} or {(P,) + shape}")
    return np.ascontiguousarray(v)


def _corr_inputs(ctx: Context, who: str, max_pairs: int, cap: int, query: dict, train: dict, pairs, matches: dict, depths, ratio, max_depth):
    """the inputs of the correspondence rule shared by PnpSolver.solve and PoseRefiner.refine, checked: (pairs (P, 2) int32, query and train
    OrbDescSet, idx, dist, k, P DevPlanes, their (P, 2) int32 sizes).  ValueError on a wrong shape, dtype, device or value."""
    import torch
    pr = np.ascontiguousarray(np.asarray(pairs, dtype=np.int64).reshape(-1, 2)).astype(np.int32)
    P = len(pr)
    if P < 1 or P > min(64, max_pairs):
        raise ValueError(f"pairs: {P} pairs, the {who} takes 1 .. {min(64, max_pairs)}")
    sets = []
    for what, s in (("query", query), ("train", train)):
        x = _cuda_tensor(ctx, f"{what}['x']", s.get("x"), torch.float32, (None, None))
        F, c = int(x.shape[0]), int(x.shape[1])
        y = _cuda_tensor(ctx, f"{what}['y']", s.get("y"), torch.float32, (F, c))
        cnt = _cuda_tensor(ctx, f"{what}['count']", s.get("count"), torch.int32, (F,))
        sets.append(OrbDescSet(None, x.data_ptr(), y.data_ptr(), cnt.data_ptr(), F, c))
    qs, ts = sets
    if qs.cap > cap:
        raise ValueError(f"query: capacity {qs.cap} exceeds the {who}'s cap {cap}")
    if ((pr[:, 0] < 0) | (pr[:, 0] >= qs.n_frames) | (pr[:, 1] < 0) | (pr[:, 1] >= ts.n_frames)).any():
        raise ValueError(f"pairs: a frame index outside the sets' {qs.n_frames} x {ts.n_frames} frames")
    idx = matches.get("idx") if isinstance(matches, dict) else None
    if not isinstance(idx, torch.Tensor) or idx.dim() != 3 or idx.shape[2] not in (1, 2):
        raise ValueError("matches['idx']: expected the (P, query cap, k) int32 tensor of orb_match, k in {1, 2}")
    k = int(idx.shape[2])
    _cuda_tensor(ctx, "matches['idx']", idx, torch.int32, (P, qs.cap, k))
    dist = _cuda_tensor(ctx, "matches['dist']", matches.get("dist"), torch.int32, (P, qs.cap, k))
    if ratio is not None and (np.isnan(ratio) or (ratio > 0 and k != 2)):
        raise ValueError(f"ratio = {ratio}: the ratio test needs k = 2 matches and a number")
    if max_depth is not None and np.isnan(max_depth):
        raise ValueError("max_depth is NaN")
    depths = list(depths.unbind(0)) if isinstance(depths, torch.Tensor) else list(depths)
    if len(depths) != P:
        raise ValueError(f"depths: {len(depths)} planes for {P} pairs")
    planes, wh = (DevPlane * P)(), np.zeros((P, 2), np.int32)
    for p, d in enumerate(depths):
        if not isinstance(d, torch.Tensor) or d.dim() != 2:
            raise ValueError(f"depths[{p}]: expected an (H, W) float32 CUDA tensor")
        planes[p] = _dev_plane(ctx, "depth", d, int(d.shape[1]), int(d.shape[0]))
        wh[p] = (d.shape[1], d.shape[0])
    return pr, qs, ts, idx, dist, k, planes, wh


class PnpSolver(_Estimator):
    """vdo_pnp_solver: cv::solvePnPRansac(AP3P) on the ORB matches of up to max_pairs frame pairs, entirely on the GPU.

    The step after OrbExtractor.extract and orb_match: each pair's matched query keypoints are back-projected through the query frame's
    depth and the train frame's pose is estimated from them, as init_model_batch (no motion model) estimates it from the same arrays,
    bit for bit.  cap: the largest query keypoint capacity a call may use (OrbExtractor.capacity); max_iters: the most RANSAC iterations."""

    _NAME, _INFO = "pnp_solver", ("max_pairs", "cap", "max_iters", "device_bytes")

    def __init__(self, ctx: Context, max_pairs: int, cap: int, max_iters: int = 500):
        self.max_pairs, self.cap, self.max_iters = int(max_pairs), int(cap), int(max_iters)
        super().__init__(ctx, C.c_int(max_pairs), C.c_int(cap), C.c_int(max_iters))

    def empty_outputs(self, P: int, query_cap: int | None = None) -> dict:
        """output tensors for P pairs (pass as solve(..., out=)): T (P, 4, 4) f32, Rt (P, 12) f64 (R row-major, then t), inlier (P, query_cap) u8 (query_cap
        defaults to the solver's cap), n_corr, n_inlier (P,) and info (P, 4) int32"""
        return _empty_outputs(self.ctx, _out_shapes(_PNP_OUT, P, query_cap=self.cap if query_cap is None else int(query_cap)))

    def solve(self, query: dict, train: dict, pairs, matches: dict, depths, K, K_train=None, Tcw_query=None, ratio: float | None = None,
              max_depth: float | None = None, iters: int = 500, thr: float = 0.4, conf: float = 0.98, out: dict | None = None) -> dict:
        """vdo_pnp_match_batch_dev.  query, train: OrbExtractor.extract() results ('x', 'y' (F, cap) f32, 'count' (F,) int32; descriptors
        are not read); pairs: P (query frame, train frame); matches: the orb_match result of the same pairs ('idx', 'dist' (P, query cap,
        k) int32, k in {1, 2}); depths: P (H, W) float32 CUDA tensors, any strides, the metric depth of each pair's query frame.
        K (fx, fy, cx, cy) of the query frames and K_train (None: K) of the train frames: (4,) or (P, 4).  Tcw_query: None, (4, 4) or
        (P, 4, 4), the query frames' poses; with it the points are in the world frame and T is the train frame's Tcw.
        ratio: Lowe's test dist0 < ratio * dist1 (k = 2); max_depth: keep 0 < z <= max_depth (None: z > 0).
        Correspondence i of pair p is query keypoint i < count[q] with a valid match j = idx[p, i, 0] < count[t] that passes both tests;
        the 3-D point is the back-projection of (x_q[i], y_q[i]) at depth[(int)y, (int)x], the observation (x_t[j], y_t[j]).
        Returns CUDA tensors T (P, 4, 4), Rt (P, 12) (the refitted R row-major, then t; [I | 0] without a model), inlier (P, query cap) u8 (slots past count[q] untouched), n_corr, n_inlier (P,),
        info (P, 4): iterations run, winning iteration, valid minimal solves, PNP_STATUS_* bits.  out: tensors from empty_outputs(),
        written in place (the call then allocates nothing and can be captured in a CUDA graph).  Enqueued on torch's current stream;
        nothing is synchronised.  ValueError on a wrong shape, dtype or device."""
        pr, qs, ts, idx, dist, k, planes, wh = _corr_inputs(self.ctx, "solver", self.max_pairs, self.cap, query, train, pairs, matches, depths, ratio, max_depth)
        P = len(pr)
        if not 1 <= int(iters) <= self.max_iters:
            raise ValueError(f"iters = {iters} outside 1 .. {self.max_iters}")
        if not thr > 0 or not 0 < conf < 1:
            raise ValueError(f"thr = {thr}, conf = {conf}; expected thr > 0 and 0 < conf < 1")
        Kq = _per_pair("K", K, P, (4,))
        Kt = None if K_train is None else _per_pair("K_train", K_train, P, (4,))
        Tq = None if Tcw_query is None else _per_pair("Tcw_query", Tcw_query, P, (4, 4))
        shapes = _out_shapes(_PNP_OUT, P, query_cap=qs.cap)
        if out is None:
            out = _empty_outputs(self.ctx, shapes)
        o = PnpOut(*_out_ptrs(self.ctx, out, shapes, _PNP_OUT))
        opts = PnpMatchOpts(k, float(ratio) if ratio is not None else 0.0, float(max_depth) if max_depth is not None else 0.0, int(iters), float(thr), float(conf))
        self.ctx.check(self.ctx.L.vdo_pnp_match_batch_dev(self.h_, C.c_int(P), pr.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(qs), C.byref(ts),
                                                          C.c_void_p(idx.data_ptr()), C.c_void_p(dist.data_ptr()), planes, wh.ctypes.data_as(C.POINTER(C.c_int32)),
                                                          _fp(Kq), None if Kt is None else _fp(Kt), None if Tq is None else _fp(Tq), C.byref(opts), C.byref(o),
                                                          C.c_uint64(_torch_stream(self.ctx))), "vdo_pnp_match_batch_dev")
        return {kk: out[kk] for kk in shapes}


class PoseRefiner(_Estimator):
    """vdo_pose_refiner: Optimizer::PoseOptimizationFlow2Cam (the joint flow / pose LM of pose_opt_flow2, mode 0) on the ORB matches of up
    to max_pairs frame pairs, entirely on the GPU.

    The step after PnpSolver.solve, as the reference tracker takes it: each pair's correspondences (the rule of PnpSolver.solve, restricted
    by a mask such as its inlier flags) are refined from an initial pose held on the device, as pose_opt_flow2 refines the same arrays,
    bit for bit.  cap: the largest query keypoint capacity a call may use (OrbExtractor.capacity)."""

    _NAME, _INFO = "pose_refiner", ("max_pairs", "cap", "device_bytes")

    def __init__(self, ctx: Context, max_pairs: int, cap: int):
        self.max_pairs, self.cap = int(max_pairs), int(cap)
        super().__init__(ctx, C.c_int(max_pairs), C.c_int(cap))

    def empty_outputs(self, P: int, query_cap: int | None = None) -> dict:
        """output tensors for P pairs (pass as refine(..., out=)): T (P, 4, 4) f32, flow (P, query_cap, 2) f64, inlier (P, query_cap) u8
        (query_cap defaults to the refiner's cap), n_points (P,) int32, stats (P, 8) f64 and status (P,) int32"""
        return _empty_outputs(self.ctx, _out_shapes(_REFINE_OUT, P, query_cap=self.cap if query_cap is None else int(query_cap)))

    def refine(self, query: dict, train: dict, pairs, matches: dict, depths, K, T_init, mask=None, Tcw_query=None, ratio: float | None = None,
               max_depth: float | None = None, quirk: int = 1, out: dict | None = None) -> dict:
        """vdo_pose_refine_batch_dev.  query, train, pairs, matches, depths, K, Tcw_query, ratio, max_depth: as PnpSolver.solve (one K per
        pair: the flow model projects with a single camera).  T_init: (P, 4, 4) float32 CUDA tensor, the initial pose of each pair (e.g.
        PnpSolver.solve's T); mask: None or (P, query cap) uint8 CUDA tensor, a correspondence enters only where it is non-zero (e.g.
        PnpSolver.solve's inlier).  quirk: 0 or 1, as pose_opt_flow2.
        Point i of pair p is (x_q[i], y_q[i]) at its depth, with the flow estimate (x_t[j] - x_q[i], y_t[j] - y_q[i]), j = idx[p, i, 0].
        Returns CUDA tensors T (P, 4, 4) (with Tcw_query the train frame's Tcw, else the query -> train pose; identity with fewer than 3
        points), flow (P, query cap, 2) f64 (the refined flow of the points that entered; other slots untouched), inlier (P, query cap) u8
        (1: entered and chi2 <= 0.04; 0 for the other i < count[q]; slots past count[q] untouched), n_points (P,), stats (P, 8) (as
        pose_opt_flow2; [0] = -1 with fewer than 3 points) and status (P,) (PNP_STATUS_QUERY_COUNT / _TRAIN_COUNT bits).  out: tensors
        from empty_outputs(), written in place (the call then allocates nothing and can be captured in a CUDA graph).  Enqueued on torch's
        current stream; nothing is synchronised.  ValueError on a wrong shape, dtype, device or value."""
        import torch
        pr, qs, ts, idx, dist, k, planes, wh = _corr_inputs(self.ctx, "refiner", self.max_pairs, self.cap, query, train, pairs, matches, depths, ratio, max_depth)
        P = len(pr)
        if quirk not in (0, 1):
            raise ValueError(f"quirk = {quirk}; expected 0 or 1")
        Ti = _cuda_tensor(self.ctx, "T_init", T_init, torch.float32, (P, 4, 4))
        mk = None if mask is None else _cuda_tensor(self.ctx, "mask", mask, torch.uint8, (P, qs.cap))
        Kq = _per_pair("K", K, P, (4,))
        Tq = None if Tcw_query is None else _per_pair("Tcw_query", Tcw_query, P, (4, 4))
        shapes = _out_shapes(_REFINE_OUT, P, query_cap=qs.cap)
        if out is None:
            out = _empty_outputs(self.ctx, shapes)
        o = PoseRefineOut(*_out_ptrs(self.ctx, out, shapes, _REFINE_OUT))
        opts = PoseRefineOpts(k, float(ratio) if ratio is not None else 0.0, float(max_depth) if max_depth is not None else 0.0, int(quirk))
        self.ctx.check(self.ctx.L.vdo_pose_refine_batch_dev(self.h_, C.c_int(P), pr.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(qs), C.byref(ts),
                                                            C.c_void_p(idx.data_ptr()), C.c_void_p(dist.data_ptr()), planes, wh.ctypes.data_as(C.POINTER(C.c_int32)),
                                                            _fp(Kq), None if Tq is None else _fp(Tq), C.c_void_p(Ti.data_ptr()),
                                                            C.c_void_p(None if mk is None else mk.data_ptr()), C.byref(opts), C.byref(o),
                                                            C.c_uint64(_torch_stream(self.ctx))), "vdo_pose_refine_batch_dev")
        return {kk: out[kk] for kk in shapes}


class ObjMotionOpts(C.Structure):
    _fields_ = [("step", C.c_int32), ("th_depth_obj", C.c_float), ("iters", C.c_int32), ("min_inliers", C.c_int32), ("thr", C.c_double),
                ("conf", C.c_double), ("quirk", C.c_int32), ("pad", C.c_int32)]


# per object slot (P, M, ...), per sample (P, cap, ...), per pair (P,)
_OM_OUT = {"label": ("int32", ("M",)), "H": ("float32", ("M", 4, 4)), "X": ("float32", ("M", 4, 4)), "T_init": ("float32", ("M", 4, 4)),
           "centre": ("float32", ("M", 3)), "velocity": ("float32", ("M", 3)), "info": ("int32", ("M", 8)), "stats": ("float64", ("M", 8)),
           "status": ("int32", ("M",)),
           "sample_x": ("int32", ("cap",)), "sample_y": ("int32", ("cap",)), "sample_label": ("int32", ("cap",)), "sample_slot": ("int32", ("cap",)),
           "sample_depth": ("float32", ("cap",)), "sample_cx": ("float32", ("cap",)), "sample_cy": ("float32", ("cap",)),
           "sample_flow": ("float32", ("cap", 2)), "sample_flow_ref": ("float64", ("cap", 2)), "sample_flags": ("uint8", ("cap",)),
           "n_samples": ("int32", ()), "pair_status": ("int32", ())}


class ObjMotionOut(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _OM_OUT]


class ObjTrackOpts(C.Structure):
    _fields_ = [("step", C.c_int32), ("th_depth_obj", C.c_float), ("iters", C.c_int32), ("min_inliers", C.c_int32), ("thr", C.c_double),
                ("conf", C.c_double), ("quirk", C.c_int32), ("sf_mg_thres", C.c_float), ("sf_ds_thres", C.c_float), ("shrink_row", C.c_int32),
                ("shrink_col", C.c_int32), ("pad", C.c_int32)]


# track(): the outputs of estimate() and these, per object slot (P, M), per sample (P, cap, ...), per pair (P,)
_OT_OUT = dict(_OM_OUT, **{"id": ("int32", ("M",)), "cls": ("int32", ("M",)), "vote": ("int32", ("M",)), "stat": ("int32", ("M",)),
                           "label_cur": ("int32", ("cap",)), "depth_cur": ("float32", ("cap",)), "flow3d": ("float32", ("cap", 3)),
                           "obj_label": ("int32", ("cap",)), "max_id": ("int32", ())})


class ObjTrackOut(C.Structure):
    _fields_ = [("motion", ObjMotionOut)] + [(k + "_dev", C.c_void_p) for k in _OT_OUT if k not in _OM_OUT]


# update_mask(): per object slot (P, M), per pair (P,)
_OU_OUT = {"label": ("int32", ("M",)), "n_vote": ("int32", ("M",)), "vote": ("int32", ("M",)), "recovered": ("int32", ("M",)),
           "n_samples": ("int32", ()), "pair_status": ("int32", ())}


class ObjMaskOut(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _OU_OUT]


# renew(): the carried feature set, per row (P, cap, ...), per pair (P,)
_OS_SET = {"x": ("int32", ("cap",)), "y": ("int32", ("cap",)), "label": ("int32", ("cap",)), "depth": ("float32", ("cap",)),
           "cx": ("float32", ("cap",)), "cy": ("float32", ("cap",)), "flow": ("float32", ("cap", 2)), "inlier_id": ("int32", ("cap",)),
           "obj_label": ("int32", ("cap",)), "point": ("float32", ("cap", 3)), "count": ("int32", ()), "status": ("int32", ())}


class ObjFeatSet(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _OS_SET]


OM_FEW_POINTS, OM_NO_MODEL, OM_FEW_INLIERS, OM_USED_MM = 1, 2, 4, 8
OT_EMPTY, OT_DYNAMIC, OT_STATIC, OT_BOUNDARY, OT_FAR = 0, 1, 2, 3, 4
OM_PAIR_OBJECT_CAP, OM_PAIR_LABEL_RANGE, OM_PAIR_FEATURE_CAP, OM_PAIR_SET_COUNT = 1, 2, 4, 8
VDO_ERR_ARG = -2
OM_MAX_ITERS = 500   # VDO_OBJ_MOTION_MAX_ITERS


class ObjectMotion(_Estimator):
    """vdo_obj_motion: the object step of the reference tracker (sampling, GetInitModelObj, PoseOptimizationFlow2, H = Tcw_cur^-1 X) for
    up to max_pairs frame pairs with up to max_objects objects each, entirely on the GPU.

    The step after PoseRefiner.refine: each pair's last frame (metric depth, flow to the current frame, instance mask) is sampled, every
    mask label is an object, and its rigid motion is estimated as the host route (Frame.sample_objects, init_model_batch with the
    constant-motion model, pose_opt_flow2 mode 1) estimates it from the same arrays, bit for bit.  cap: the most samples of a pair,
    at least ceil(W / step) * ceil(H / step) of every frame a call may use."""

    _NAME, _INFO = "obj_motion", ("max_pairs", "max_objects", "cap", "device_bytes")

    def __init__(self, ctx: Context, max_pairs: int, max_objects: int, cap: int):
        self.max_pairs, self.max_objects, self.cap = int(max_pairs), int(max_objects), int(cap)
        super().__init__(ctx, C.c_int(max_pairs), C.c_int(max_objects), C.c_int(cap))

    def _shapes(self, P: int, table: dict = _OM_OUT) -> dict:
        return _out_shapes(table, P, M=self.max_objects, cap=self.cap)

    def empty_outputs(self, P: int, track: bool = False, update_mask: bool = False, renew: bool = False) -> dict:
        """output tensors for P pairs (pass as estimate(..., out=), with track=True as track(..., out=), with update_mask=True as
        update_mask(..., out=), with renew=True as renew(..., out=)); see those calls for their meaning"""
        return _empty_outputs(self.ctx, self._shapes(P, _OS_SET if renew else _OU_OUT if update_mask else _OT_OUT if track else _OM_OUT))

    def _set(self, samples, P: int):
        """the checked ObjFeatSet of a renew() result for P pairs, or None"""
        if samples is None:
            return None
        if not isinstance(samples, dict):
            raise ValueError("samples: expected the dict of a previous renew()")
        return ObjFeatSet(*_out_ptrs(self.ctx, samples, self._shapes(P, _OS_SET), _OS_SET))


    def _planes(self, depths, flows, masks, step, th_depth_obj, iters, thr, conf, min_inliers, quirk):
        """the checked last-frame planes and options of estimate() and track(): (depth, flow, mask DevPlane arrays, (P, 2) sizes)"""
        import torch
        planes = []
        for what, kind, ts in (("depths", "depth", depths), ("flows", "flow", flows), ("masks", "mask", masks)):
            ts = list(ts.unbind(0)) if isinstance(ts, torch.Tensor) else list(ts)
            planes.append(ts)
        P = len(planes[0])
        if P < 1 or P > self.max_pairs:
            raise ValueError(f"depths: {P} pairs, the estimator takes 1 .. {self.max_pairs}")
        if len(planes[1]) != P or len(planes[2]) != P:
            raise ValueError(f"depths, flows, masks: {P}, {len(planes[1])}, {len(planes[2])} planes; expected one of each per pair")
        if int(step) < 1:
            raise ValueError(f"step = {step}; expected >= 1")
        if np.isnan(th_depth_obj):
            raise ValueError("th_depth_obj is NaN")
        if not 1 <= int(iters) <= OM_MAX_ITERS or not thr > 0 or not 0 < conf < 1:
            raise ValueError(f"iters = {iters}, thr = {thr}, conf = {conf}; expected 1 .. {OM_MAX_ITERS}, > 0 and inside (0, 1)")
        if int(min_inliers) < 0 or quirk not in (0, 1):
            raise ValueError(f"min_inliers = {min_inliers}, quirk = {quirk}; expected >= 0 and 0 or 1")
        dp, fp, mp, wh = (DevPlane * P)(), (DevPlane * P)(), (DevPlane * P)(), np.zeros((P, 2), np.int32)
        for p in range(P):
            d = planes[0][p]
            if not isinstance(d, torch.Tensor) or d.dim() != 2:
                raise ValueError(f"depths[{p}]: expected an (H, W) float32 CUDA tensor")
            h, w = int(d.shape[0]), int(d.shape[1])
            n = ((w + step - 1) // step) * ((h + step - 1) // step)
            if n > self.cap:
                raise ValueError(f"pair {p}: {w}x{h} at step {step} has {n} sample positions, above the estimator's cap {self.cap}")
            dp[p] = _dev_plane(self.ctx, "depth", d, w, h)
            fp[p] = _dev_plane(self.ctx, "flow", planes[1][p], w, h)
            mp[p] = _dev_plane(self.ctx, "mask", planes[2][p], w, h)
            wh[p] = (w, h)
        return dp, fp, mp, wh

    def estimate(self, depths, flows, masks, K, Tcw_last=None, Tcw_cur=None, prev: dict | None = None, step: int = 4, th_depth_obj: float = 25.0,
                 iters: int = 500, thr: float = 0.4, conf: float = 0.98, min_inliers: int = 50, quirk: int = 1, out: dict | None = None) -> dict:
        """vdo_obj_motion_batch_dev.  depths, flows, masks: P CUDA tensors each (or stacked tensors), the LAST frame of each pair at any
        strides: metric depth (H, W) float32, flow to the current frame (H, W, 2) or (2, H, W) float32, instance mask (H, W) int32 or int64
        (0 = background, every other label an object).  K: (4,) or (P, 4) fx, fy, cx, cy.  Tcw_last, Tcw_cur: None (identity) or (P, 4, 4)
        float32 CUDA tensors, e.g. PoseRefiner.refine's T for the current frame; with identity poses H is the motion in the last camera's
        frame.  prev: None or the previous call's result (its 'label' and 'H' give the constant-motion models).  step, th_depth_obj (the
        reference's ThDepthObj), iters, thr, conf, min_inliers, quirk: as in the reference's settings (iters <= 500).
        Returns CUDA tensors.  Per object slot (P, max_objects): label (-1: empty slot; the slots hold the distinct labels in ascending
        order), H (vObjMod), X (the LM result), T_init (the initial model), centre (3), velocity (3, t_H - (I - R_H) c, metres per frame),
        info (8: samples, n_ransac, n_mm, used_mm, n_sub, iterations run, winning iteration, valid minimal solves), stats (8, as
        pose_opt_flow2), status (OM_* bits).  Per sample (P, cap; entries past n_samples untouched): sample_x, sample_y, sample_label,
        sample_slot (-1: not estimated), sample_depth, sample_cx, sample_cy, sample_flow (2), sample_flow_ref (2, f64), sample_flags (1: in
        the chosen initial set, 2: LM inlier).  Per pair (P,): n_samples, pair_status (OM_PAIR_* bits).  out: tensors from
        empty_outputs(), written in place (the call then allocates nothing and can be captured in a CUDA graph).  Enqueued on torch's
        current stream; nothing is synchronised.  ValueError on a wrong shape, dtype, device or value."""
        import torch
        dp, fp, mp, wh = self._planes(depths, flows, masks, step, th_depth_obj, iters, thr, conf, min_inliers, quirk)
        P = len(wh)
        Kp = _per_pair("K", K, P, (4,))
        M = self.max_objects
        Tl = None if Tcw_last is None else _cuda_tensor(self.ctx, "Tcw_last", Tcw_last, torch.float32, (P, 4, 4))
        Tc = None if Tcw_cur is None else _cuda_tensor(self.ctx, "Tcw_cur", Tcw_cur, torch.float32, (P, 4, 4))
        pl = pH = None
        if prev is not None:
            if not isinstance(prev, dict):
                raise ValueError("prev: expected the dict of a previous estimate()")
            pl = _cuda_tensor(self.ctx, "prev['label']", prev.get("label"), torch.int32, (P, M))
            pH = _cuda_tensor(self.ctx, "prev['H']", prev.get("H"), torch.float32, (P, M, 4, 4))
        shapes = self._shapes(P)
        if out is None:
            out = _empty_outputs(self.ctx, shapes)
        o = ObjMotionOut(*_out_ptrs(self.ctx, out, shapes, _OM_OUT))
        opts = ObjMotionOpts(int(step), float(th_depth_obj), int(iters), int(min_inliers), float(thr), float(conf), int(quirk), 0)
        ptr = lambda t: C.c_void_p(None if t is None else t.data_ptr())
        self.ctx.check(self.ctx.L.vdo_obj_motion_batch_dev(self.h_, C.c_int(P), dp, fp, mp, wh.ctypes.data_as(C.POINTER(C.c_int32)), _fp(Kp),
                                                           ptr(Tl), ptr(Tc), ptr(pl), ptr(pH), C.byref(opts), C.byref(o),
                                                           C.c_uint64(_torch_stream(self.ctx))),
                       "vdo_obj_motion_batch_dev")
        return {k: out[k] for k in shapes}

    def track(self, depths, flows, masks, depths_cur, masks_cur, K, Tcw_last=None, Tcw_cur=None, prev: dict | None = None, step: int = 4,
              th_depth_obj: float = 25.0, sf_mg_thres: float = 0.12, sf_ds_thres: float = 0.3, shrink=(25, 50), iters: int = 500, thr: float = 0.4,
              conf: float = 0.98, min_inliers: int = 50, quirk: int = 1, samples: dict | None = None, out: dict | None = None) -> dict:
        """vdo_obj_track_batch_dev: the reference's object step with its scene flow and object tracking (GetSceneFlowObj, DynObjTracking)
        ahead of the motion estimate.  depths, flows, masks, K, Tcw_last, Tcw_cur, step, th_depth_obj, iters, thr, conf, min_inliers, quirk: as
        estimate(); depths_cur, masks_cur: P CUDA tensors each (or stacked), the CURRENT frame's metric depth (H, W) float32 and instance mask
        (H, W) int32 or int64 at any strides, of the last frame's size.  The current mask's labels need not match the last one's: objects are
        identified by the IDs this call hands out.  sf_mg_thres, sf_ds_thres: SFMgThres and SFDsThres; shrink: the border band (rows,
        columns), (25, 50) for KITTI and (0, 0) otherwise.  prev: None (the start of a sequence) or the previous track() result, whose label,
        id, stat, H and max_id carry the object table; to restart one pair of a batch, write the reset state into its row (label -1, id -1,
        stat 0, H identity, max_id 1).
        Returns CUDA tensors: estimate()'s, where a slot's label is its CURRENT label (the slots hold the distinct current labels of the valid
        samples in ascending order) and only dynamic slots are estimated, plus per slot (P, max_objects): id (-1 unless dynamic), cls (OT_*),
        vote (the voted last label of a dynamic slot, else 0), stat (1: dynamic and passed the min_inliers gate); per sample (P, cap):
        label_cur, depth_cur (the look-up at the flow target; 0 and 0.1 when it fails), flow3d (3, the world-frame scene flow, 0 for an
        invalid sample), obj_label (-2 never classified, -1 invalid / boundary / far / outside the chosen set / LM outlier, 0 static, the ID
        otherwise); per pair: max_id.  samples: None (every pair samples its last frame) or the renew() result of the previous pair of each
        sequence (vdo_obj_track_set_batch_dev): a pair whose count is >= 0 takes its samples from that set, in row order, as the reference
        does after its first pair; count -1 samples the last frame.  The set must not be the out= of the renew() this result feeds.
        out: tensors from empty_outputs(P, track=True), written in place (the call then allocates nothing and can be captured in a CUDA
        graph).  Enqueued on torch's current stream; nothing is synchronised.  ValueError on a wrong shape, dtype, device or value."""
        import torch
        dp, fp, mp, wh = self._planes(depths, flows, masks, step, th_depth_obj, iters, thr, conf, min_inliers, quirk)
        P = len(wh)
        dc, mc = (DevPlane * P)(), (DevPlane * P)()
        for what, kind, ts, arr in (("depths_cur", "depth", depths_cur, dc), ("masks_cur", "mask", masks_cur, mc)):
            ts = list(ts.unbind(0)) if isinstance(ts, torch.Tensor) else list(ts)
            if len(ts) != P:
                raise ValueError(f"{what}: {len(ts)} planes for {P} pairs")
            for p in range(P):
                arr[p] = _dev_plane(self.ctx, kind, ts[p], int(wh[p, 0]), int(wh[p, 1]))
        if np.isnan(sf_mg_thres) or np.isnan(sf_ds_thres):
            raise ValueError(f"sf_mg_thres = {sf_mg_thres}, sf_ds_thres = {sf_ds_thres}; expected numbers")
        sr, sc = (int(v) for v in shrink)
        if sr < 0 or sc < 0:
            raise ValueError(f"shrink = {shrink}; expected (rows, columns) >= 0")
        Kp = _per_pair("K", K, P, (4,))
        M = self.max_objects
        Tl = None if Tcw_last is None else _cuda_tensor(self.ctx, "Tcw_last", Tcw_last, torch.float32, (P, 4, 4))
        Tc = None if Tcw_cur is None else _cuda_tensor(self.ctx, "Tcw_cur", Tcw_cur, torch.float32, (P, 4, 4))
        pv = [None] * 5
        if prev is not None:
            if not isinstance(prev, dict) or "id" not in prev or "max_id" not in prev:
                raise ValueError("prev: expected the dict of a previous track()")
            pv = [_cuda_tensor(self.ctx, f"prev[{k!r}]", prev.get(k), dt, shp) for k, dt, shp in
                  (("label", torch.int32, (P, M)), ("id", torch.int32, (P, M)), ("stat", torch.int32, (P, M)), ("H", torch.float32, (P, M, 4, 4)),
                   ("max_id", torch.int32, (P,)))]
        shapes = self._shapes(P, _OT_OUT)
        if out is None:
            out = _empty_outputs(self.ctx, shapes)
        ptrs = _out_ptrs(self.ctx, out, shapes, _OT_OUT)
        o = ObjTrackOut(ObjMotionOut(*ptrs[:len(_OM_OUT)]), *ptrs[len(_OM_OUT):])
        opts = ObjTrackOpts(int(step), float(th_depth_obj), int(iters), int(min_inliers), float(thr), float(conf), int(quirk), float(sf_mg_thres),
                            float(sf_ds_thres), sr, sc, 0)
        ptr = lambda t: C.c_void_p(None if t is None else t.data_ptr())
        S = self._set(samples, P)
        args = (self.h_, C.c_int(P), dp, fp, mp, dc, mc, wh.ctypes.data_as(C.POINTER(C.c_int32)), _fp(Kp), ptr(Tl), ptr(Tc), *[ptr(t) for t in pv])
        tail = (C.byref(opts), C.byref(o), C.c_uint64(_torch_stream(self.ctx)))
        if S is None:
            self.ctx.check(self.ctx.L.vdo_obj_track_batch_dev(*args, *tail), "vdo_obj_track_batch_dev")
        else:
            self.ctx.check(self.ctx.L.vdo_obj_track_set_batch_dev(*args, C.byref(S), *tail), "vdo_obj_track_set_batch_dev")
        return {k: out[k] for k in shapes}

    def update_mask(self, depths, flows, masks, masks_cur, step: int = 4, th_depth_obj: float = 25.0, samples: dict | None = None,
                    out: dict | None = None) -> dict:
        """vdo_obj_update_mask_batch_dev: the reference's UpdateMask, which recovers in the current mask the objects the segmentation missed.
        depths, flows, masks, step, th_depth_obj: the LAST frames and sampling as estimate() and track(); masks_cur: P CUDA tensors (or one
        stacked tensor), the CURRENT frame's instance mask (H, W) int32 or int64 at any strides, updated IN PLACE.
        Per slot (the distinct sample labels ascending, the first max_objects), in order: the samples whose flow target (int)cx, (int)cy lies
        strictly inside the image vote with the current label there, as updated by the earlier slots; with at least 100 voters and a majority
        (ties: the smaller label) of 0, every last-frame pixel of the slot's label is pushed along its flow (truncated) into the current mask
        (the higher slot wins a pixel two slots push onto).  Only pixels that receive a recovered label are written.  Call it on a pair before
        track() on the same pair; the updated mask is the next pair's mask.  A recovered region carries the last frame's label, so labels
        should be stable across frames (or at least not reused for another object).  samples: None (the voters are the last frame's samples)
        or the renew() result of the previous pair of each sequence (vdo_obj_update_mask_set_batch_dev): a pair whose count is >= 0 votes
        with the set's (label, cx, cy), the reference's vSemObjLabel and mvObjCorres; count -1 samples the last frame.
        The pairs of one call are independent: no masks_cur may share memory with any plane of the call, so consecutive frames of a sequence
        go in consecutive calls, not as pairs (t, t + 1) of one call.
        Returns CUDA tensors per slot (P, max_objects): label (the LAST-frame label, -1 empty), n_vote (voters), vote (the majority current
        label, 0 with fewer than 100 voters or OM_PAIR_LABEL_RANGE), recovered (1: pushed into the mask); per pair (P,): n_samples,
        pair_status (OM_PAIR_OBJECT_CAP; OM_PAIR_LABEL_RANGE for an i64 label outside int32 in the last mask at a sample or in the current
        mask at a voter's target: the pair then recovers nothing).  out: tensors from empty_outputs(P, update_mask=True), written in place
        (the call then allocates nothing and can be captured in a CUDA graph).  Enqueued on torch's current stream; nothing is synchronised.
        ValueError on a wrong shape, dtype, device or value, on a masks_cur whose pixels are not distinct elements and on overlapping planes,
        before anything is written."""
        import torch
        dp, fp, mp, wh = self._planes(depths, flows, masks, step, th_depth_obj, OM_MAX_ITERS, 0.4, 0.98, 0, 1)
        P = len(wh)
        ts = list(masks_cur.unbind(0)) if isinstance(masks_cur, torch.Tensor) else list(masks_cur)
        if len(ts) != P:
            raise ValueError(f"masks_cur: {len(ts)} planes for {P} pairs")
        mc = (DevPlane * P)()
        for p in range(P):
            mc[p] = _dev_plane(self.ctx, "mask", ts[p], int(wh[p, 0]), int(wh[p, 1]))
        shapes = self._shapes(P, _OU_OUT)
        if out is None:
            out = _empty_outputs(self.ctx, shapes)
        o = ObjMaskOut(*_out_ptrs(self.ctx, out, shapes, _OU_OUT))
        S = self._set(samples, P)
        args = (self.h_, C.c_int(P), dp, fp, mp, mc, wh.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int32(int(step)), C.c_float(float(th_depth_obj)))
        tail = (C.byref(o), C.c_uint64(_torch_stream(self.ctx)))
        if S is None:
            fn, rc = "vdo_obj_update_mask_batch_dev", self.ctx.L.vdo_obj_update_mask_batch_dev(*args, *tail)
        else:
            fn, rc = "vdo_obj_update_mask_set_batch_dev", self.ctx.L.vdo_obj_update_mask_set_batch_dev(*args, C.byref(S), *tail)
        if rc == VDO_ERR_ARG:               # the layout and overlap checks of mask_cur live in the library; its message names the pair
            raise ValueError(self.ctx.L.vdo_last_error(self.ctx.h).decode())
        self.ctx.check(rc, fn)
        return {k: out[k] for k in shapes}

    def renew(self, track_result: dict, depths_cur, flows_cur, masks_cur, K, Tcw_cur=None, step: int = 4, th_depth_obj: float = 25.0,
              max_track_obj: int = 800, out: dict | None = None) -> dict:
        """vdo_obj_renew_batch_dev: the object half of the reference's RenewFrameInfo, the current frame's object features carried into the
        next pair.  track_result: the track() result of the same P pairs; depths_cur, flows_cur, masks_cur: P CUDA tensors each (or stacked),
        the CURRENT frame's metric depth (H, W) float32, its flow to the NEXT frame (H, W, 2) or (2, H, W) float32 and its mask (as
        update_mask() left it) int32 or int64, at any strides; K: (4,) or (P, 4); Tcw_cur: None (identity) or (P, 4, 4) float32 CUDA tensor.
        step, th_depth_obj: the raster sampling of the current frame; max_track_obj: MaxTrackPointOBJ, >= 0.
        Rows, in order: the LM inliers of each stat slot carried along their refined flow (kept on the current mask, at 0 < depth < 25, with
        the flow target inside); each stat slot topped up to max_track_obj rows from the raster samples of its current label (passes of
        stride 15, skipping pixels a carried key sits on); all raster samples of every label that is no stat slot's, ascending.
        Returns CUDA tensors per row (P, cap): x, y (integer pixel), label, depth, cx, cy, flow (2), inlier_id (the row of the same point in
        track_result's samples, -1 for a new point), obj_label (the object ID, -2 for a new label), point (3, the world point); per pair:
        count (rows; -1 with OM_PAIR_LABEL_RANGE) and status (OM_PAIR_FEATURE_CAP when rows past cap were dropped, OM_PAIR_LABEL_RANGE).
        Pass it as samples= to the next pair's update_mask() and track().  out: tensors from empty_outputs(P, renew=True), written in place
        (the call then allocates nothing and can be captured in a CUDA graph).  Enqueued on torch's current stream; nothing is synchronised.
        ValueError on a wrong shape, dtype, device or value."""
        import torch
        dp, fp, mp, wh = self._planes(depths_cur, flows_cur, masks_cur, step, th_depth_obj, OM_MAX_ITERS, 0.4, 0.98, 0, 1)
        P = len(wh)
        if int(max_track_obj) < 0:
            raise ValueError(f"max_track_obj = {max_track_obj}; expected >= 0")
        if not isinstance(track_result, dict):
            raise ValueError("track_result: expected the dict of a track() of the same pairs")
        tshapes = self._shapes(P, _OT_OUT)
        used = {k: tshapes[k] for k in ("label", "sample_x", "sample_y", "sample_slot", "sample_flags", "sample_flow_ref", "n_samples", "id", "stat",
                                        "obj_label")}
        ptrs = _out_ptrs(self.ctx, track_result, used, _OT_OUT)
        t = ObjTrackOut(ObjMotionOut(*ptrs[:len(_OM_OUT)]), *ptrs[len(_OM_OUT):])
        Kp = _per_pair("K", K, P, (4,))
        Tc = None if Tcw_cur is None else _cuda_tensor(self.ctx, "Tcw_cur", Tcw_cur, torch.float32, (P, 4, 4))
        shapes = self._shapes(P, _OS_SET)
        if out is None:
            out = _empty_outputs(self.ctx, shapes)
        S = ObjFeatSet(*_out_ptrs(self.ctx, out, shapes, _OS_SET))
        self.ctx.check(self.ctx.L.vdo_obj_renew_batch_dev(self.h_, C.c_int(P), C.byref(t), dp, fp, mp, wh.ctypes.data_as(C.POINTER(C.c_int32)), _fp(Kp),
                                                          C.c_void_p(None if Tc is None else Tc.data_ptr()), C.c_int32(int(step)),
                                                          C.c_float(float(th_depth_obj)), C.c_int32(int(max_track_obj)), C.byref(S),
                                                          C.c_uint64(_torch_stream(self.ctx))), "vdo_obj_renew_batch_dev")
        return {k: out[k] for k in shapes}


# the carried background set, per row (P, cap, ...) and per pair (P, ...); a fresh set has count -1
_SS_SET = {"x": ("float32", ("cap",)), "y": ("float32", ("cap",)), "depth": ("float32", ("cap",)), "cx": ("float32", ("cap",)),
           "cy": ("float32", ("cap",)), "flow": ("float32", ("cap", 2)), "inlier_id": ("int32", ("cap",)), "point": ("float32", ("cap", 3)),
           "count": ("int32", ()), "status": ("int32", ()), "Tcw": ("float32", (4, 4)), "velocity": ("float32", (4, 4)), "has_velocity": ("int32", ())}


class StatFeatSet(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _SS_SET]


class StatOpts(C.Structure):
    _fields_ = [("th_depth_bg", C.c_float), ("max_track_bg", C.c_int32), ("use_sample_feature", C.c_int32), ("pad", C.c_int32)]


class CamTrackOpts(C.Structure):
    _fields_ = [("iters", C.c_int32), ("quirk", C.c_int32), ("thr", C.c_double), ("conf", C.c_double)]


# track(): per pair (P, ...), per row (P, cap, ...)
_CT_OUT = {"T": ("float32", (4, 4)), "T_init": ("float32", (4, 4)), "velocity": ("float32", (4, 4)), "info": ("int32", (8,)), "stats": ("float64", (8,)),
           "status": ("int32", ()), "flags": ("uint8", ("cap",)), "key": ("float32", ("cap", 2)), "flow_ref": ("float64", ("cap", 2))}


class CamTrackOut(C.Structure):
    _fields_ = [(k + "_dev", C.c_void_p) for k in _CT_OUT]


CAM_FEW_POINTS, CAM_NO_MODEL, CAM_USED_MM, CAM_SET_COUNT, CAM_KEY_COUNT = 1, 2, 4, 8, 16
CAM_MAX_ITERS = 500   # VDO_CAM_MOTION_MAX_ITERS


def _key_set(ctx: Context, what: str, keys: dict) -> OrbDescSet:
    """the x, y (F, cap) float32 and count (F,) int32 CUDA tensors of an OrbExtractor.extract() or sample_keys_dev() result"""
    import torch
    if not isinstance(keys, dict):
        raise ValueError(f"{what}: expected the dict of OrbExtractor.extract() or sample_keys_dev()")
    x = _cuda_tensor(ctx, f"{what}['x']", keys.get("x"), torch.float32, (None, None))
    F, cap = int(x.shape[0]), int(x.shape[1])
    y = _cuda_tensor(ctx, f"{what}['y']", keys.get("y"), torch.float32, (F, cap))
    cnt = _cuda_tensor(ctx, f"{what}['count']", keys.get("count"), torch.int32, (F,))
    return OrbDescSet(None, x.data_ptr(), y.data_ptr(), cnt.data_ptr(), F, cap)


class CameraMotion(_Estimator):
    """vdo_cam_motion: the camera step of the reference tracker (GetInitModelCam against the constant-velocity model, then
    PoseOptimizationFlow2Cam) on the last frame's background features carried along the flow, and the static half of RenewFrameInfo that
    carries them into the next frame, for up to max_pairs frame pairs, entirely on the GPU.

    Per frame: build(S) (fills the pairs whose set count is -1), cam = track(S), then S' = renew(S, cam).  The set holds the frame's pose and
    the velocity, so a sequence carries one object from pair to pair; writing -1 into a pair's count restarts it.  ObjectMotion's calls take
    S['Tcw'] as Tcw_last and cam['T'] as Tcw_cur.  cap: the most rows of a pair's set, at least the key sets' capacity and max_track_bg + 1."""

    _NAME, _INFO = "cam_motion", ("max_pairs", "cap", "max_iters", "device_bytes")

    def __init__(self, ctx: Context, max_pairs: int, cap: int):
        self.max_pairs, self.cap = int(max_pairs), int(cap)
        super().__init__(ctx, C.c_int(max_pairs), C.c_int(cap))

    def _shapes(self, P: int, table: dict) -> dict:
        return _out_shapes(table, P, cap=self.cap)

    def empty_outputs(self, P: int, set: bool = True) -> dict:
        """with set=True a fresh background set for P pairs (count -1: build() fills it), else the output tensors of track(..., out=)"""
        out = _empty_outputs(self.ctx, self._shapes(P, _SS_SET if set else _CT_OUT))
        if set:
            out["count"].fill_(-1)
        return out

    def _set(self, what: str, s, P: int) -> StatFeatSet:
        if not isinstance(s, dict):
            raise ValueError(f"{what}: expected a background set (empty_outputs(P) or a renew() result)")
        return StatFeatSet(*_out_ptrs(self.ctx, s, self._shapes(P, _SS_SET), _SS_SET))

    def _frames(self, keys, depths, flows, masks, K, orb_count, th_depth_bg, max_track_bg, use_sample_feature):
        """the checked key set, planes, sizes, K, gate and options of build() and renew()"""
        import torch
        planes = []
        for ts in (depths, flows, masks):
            planes.append(list(ts.unbind(0)) if isinstance(ts, torch.Tensor) else list(ts))
        P = len(planes[0])
        if P < 1 or P > self.max_pairs:
            raise ValueError(f"depths: {P} pairs, the estimator takes 1 .. {self.max_pairs}")
        if len(planes[1]) != P or len(planes[2]) != P:
            raise ValueError(f"depths, flows, masks: {P}, {len(planes[1])}, {len(planes[2])} planes; expected one of each per pair")
        ks = _key_set(self.ctx, "keys", keys)
        if ks.n_frames < P or ks.cap > self.cap:
            raise ValueError(f"keys: {ks.n_frames} frames of capacity {ks.cap}; expected at least {P} frames and a capacity up to the cap {self.cap}")
        if np.isnan(th_depth_bg) or use_sample_feature not in (0, 1):
            raise ValueError(f"th_depth_bg = {th_depth_bg}, use_sample_feature = {use_sample_feature}; expected a number and 0 or 1")
        if not 0 <= int(max_track_bg) < self.cap:
            raise ValueError(f"max_track_bg = {max_track_bg}; expected 0 .. cap - 1 = {self.cap - 1}")
        gate = None
        if use_sample_feature:
            gate = _cuda_tensor(self.ctx, "orb_count", orb_count, torch.int32, (None,))
            if gate.shape[0] < P:
                raise ValueError(f"orb_count: {gate.shape[0]} counts for {P} pairs")
        dp, fp, mp, wh = (DevPlane * P)(), (DevPlane * P)(), (DevPlane * P)(), np.zeros((P, 2), np.int32)
        for p in range(P):
            d = planes[0][p]
            if not isinstance(d, torch.Tensor) or d.dim() != 2:
                raise ValueError(f"depths[{p}]: expected an (H, W) float32 CUDA tensor")
            h, w = int(d.shape[0]), int(d.shape[1])
            dp[p] = _dev_plane(self.ctx, "depth", d, w, h)
            fp[p] = _dev_plane(self.ctx, "flow", planes[1][p], w, h)
            mp[p] = _dev_plane(self.ctx, "mask", planes[2][p], w, h)
            wh[p] = (w, h)
        Kp = _per_pair("K", K, P, (4,))
        opts = StatOpts(float(th_depth_bg), int(max_track_bg), int(use_sample_feature), 0)
        return P, ks, dp, fp, mp, wh, Kp, gate, opts

    def build(self, keys: dict, depths, flows, masks, K, set: dict, th_depth_bg: float = 40.0, use_sample_feature: int = 0, orb_count=None) -> dict:
        """vdo_stat_build_batch_dev: Frame::Frame's static set of the LAST frame of every pair whose set count is -1, in place; the other
        pairs are left as they are.  keys: the last frames' key set (frame p for pair p): OrbExtractor.extract()'s ORB keypoints for option I,
        sample_keys_dev()'s keys for option II (use_sample_feature=1, with orb_count the frames' ORB counts: a frame without ORB keypoints
        gets an empty set).  depths, flows, masks: P CUDA tensors each (or stacked), metric depth (H, W) float32, flow to the current frame
        (H, W, 2) or (2, H, W) float32, mask (H, W) int32 or int64, at any strides.  K: (4,) or (P, 4).  Rows: the keys on the background
        (mask 0) with 0 < depth <= th_depth_bg, non-zero flow and the flow target inside the image; inlier_id -1, point the camera-frame
        back-projection; per pair Tcw = I and no velocity.  Returns set.  ValueError on a wrong shape, dtype, device or value."""
        P, ks, dp, fp, mp, wh, Kp, gate, opts = self._frames(keys, depths, flows, masks, K, orb_count, th_depth_bg, 0, use_sample_feature)
        S = self._set("set", set, P)
        self.ctx.check(self.ctx.L.vdo_stat_build_batch_dev(self.h_, C.c_int(P), C.byref(ks), dp, fp, mp, wh.ctypes.data_as(C.POINTER(C.c_int32)), _fp(Kp),
                                                           C.c_void_p(None if gate is None else gate.data_ptr()), C.byref(opts), C.byref(S),
                                                           C.c_uint64(_torch_stream(self.ctx))), "vdo_stat_build_batch_dev")
        return set

    def track(self, set: dict, K, iters: int = 500, thr: float = 0.4, conf: float = 0.98, quirk: int = 1, out: dict | None = None) -> dict:
        """vdo_cam_track_batch_dev: the reference's camera step from the sets alone.  set: the P pairs' background sets (build() or renew());
        K: (4,) or (P, 4).  Each row's world point (its key and depth through the set's Tcw) is observed at its corres; GetInitModelCam
        (AP3P RANSAC, iters, thr, conf) is chosen against the constant-velocity model velocity * Tcw (Tcw on the first pair), and a chosen
        set of at least 3 rows is refined by PoseOptimizationFlow2Cam (quirk).
        Returns CUDA tensors per pair: T (4, 4, the current mTcw), T_init, velocity (T * Tcw^-1), info (8: rows, n_ransac, n_mm, used_mm,
        n_sub, iterations run, winning iteration, valid minimal solves), stats (8, as pose_opt_flow2; [0] = -1 without the LM), status
        (CAM_* bits); per row (P, cap; rows past count untouched): flags (1 chosen, 2 LM inlier, 4 still in TemperalMatch_subset), key (2,
        the current frame's mvStatKeys), flow_ref (2, f64).  out: tensors from empty_outputs(P, set=False), written in place (the call then
        allocates nothing and can be captured in a CUDA graph).  Enqueued on torch's current stream; nothing is synchronised."""
        P = int(set["count"].shape[0]) if isinstance(set, dict) and "count" in set else 0
        if P < 1 or P > self.max_pairs:
            raise ValueError(f"set: {P} pairs, the estimator takes 1 .. {self.max_pairs}")
        if not 1 <= int(iters) <= CAM_MAX_ITERS or not thr > 0 or not 0 < conf < 1 or quirk not in (0, 1):
            raise ValueError(f"iters = {iters}, thr = {thr}, conf = {conf}, quirk = {quirk}; expected 1 .. {CAM_MAX_ITERS}, > 0, inside (0, 1) and 0 or 1")
        S = self._set("set", set, P)
        Kp = _per_pair("K", K, P, (4,))
        shapes = self._shapes(P, _CT_OUT)
        if out is None:
            out = _empty_outputs(self.ctx, shapes)
        o = CamTrackOut(*_out_ptrs(self.ctx, out, shapes, _CT_OUT))
        opts = CamTrackOpts(int(iters), int(quirk), float(thr), float(conf))
        self.ctx.check(self.ctx.L.vdo_cam_track_batch_dev(self.h_, C.c_int(P), C.byref(S), _fp(Kp), C.byref(opts), C.byref(o),
                                                          C.c_uint64(_torch_stream(self.ctx))), "vdo_cam_track_batch_dev")
        return {k: out[k] for k in shapes}

    def renew(self, last: dict, cam: dict, keys: dict, depths_cur, flows_cur, masks_cur, K, max_track_bg: int = 1200, th_depth_bg: float = 40.0,
              use_sample_feature: int = 0, orb_count=None, out: dict | None = None) -> dict:
        """vdo_stat_renew_batch_dev: the static half of the reference's RenewFrameInfo, the current frame's background set.  last, cam: the
        set track() read and its result; keys: the CURRENT frames' key set (ORB keypoints for option I, sample_keys_dev()'s raw keys for
        option II with orb_count); depths_cur, flows_cur, masks_cur: the CURRENT frames' metric depth, flow to the NEXT frame and mask as
        update_mask() left it.  Rows: the rows still in TemperalMatch_subset whose current key passes the reference's test (mask 0,
        0 < depth <= 40, non-zero flow, key and target strictly inside), in row order, at most max_track_bg + 1 of them (inlier_id: the row);
        then, while fewer than max_track_bg are held, the key list (option II: the keys passing build()'s rule) in passes of stride 20, a key
        closer than 1 px to a carried one skipped (inlier_id -1).  Points are in the world frame; per pair Tcw = cam['T'], velocity =
        cam['velocity'].  out: a set from empty_outputs(P) other than last, written in place (the call then allocates nothing and can be
        captured in a CUDA graph).  Enqueued on torch's current stream; nothing is synchronised.  ValueError on a wrong shape, dtype, device
        or value."""
        P, ks, dp, fp, mp, wh, Kp, gate, opts = self._frames(keys, depths_cur, flows_cur, masks_cur, K, orb_count, th_depth_bg, max_track_bg,
                                                             use_sample_feature)
        L = self._set("last", last, P)
        if not isinstance(cam, dict):
            raise ValueError("cam: expected the dict of a track() of the same pairs")
        cshapes = self._shapes(P, _CT_OUT)
        used = {k: cshapes[k] for k in ("T", "velocity", "status", "flags", "key")}
        co = CamTrackOut(*_out_ptrs(self.ctx, cam, used, _CT_OUT))
        if out is None:
            out = self.empty_outputs(P)
        S = self._set("out", out, P)
        self.ctx.check(self.ctx.L.vdo_stat_renew_batch_dev(self.h_, C.c_int(P), C.byref(L), C.byref(co), C.byref(ks), dp, fp, mp,
                                                           wh.ctypes.data_as(C.POINTER(C.c_int32)), _fp(Kp),
                                                           C.c_void_p(None if gate is None else gate.data_ptr()), C.byref(opts), C.byref(S),
                                                           C.c_uint64(_torch_stream(self.ctx))), "vdo_stat_renew_batch_dev")
        return out


def sample_keys_dev(ctx: Context, seeds_dev, width: int, height: int, out: dict | None = None) -> dict:
    """vdo_sample_keys_dev: sample_keys on the device.  seeds_dev: (F,) int32 CUDA tensor (read as uint32), frame i's cv::RNG seed, e.g.
    sample_seed + f_id.  Returns CUDA tensors x, y (F, SAMPLE_KEYS) float32 and count (F,) int32 (all SAMPLE_KEYS), the layout
    CameraMotion.build / renew take as keys.  out: tensors of those shapes, written in place (the call then allocates nothing and can be
    captured in a CUDA graph; a replay reads the seeds as they are then).  Enqueued on torch's current stream."""
    import torch
    s = _cuda_tensor(ctx, "seeds_dev", seeds_dev, torch.int32, (None,))
    F = int(s.shape[0])
    shapes = {"x": (torch.float32, (F, SAMPLE_KEYS)), "y": (torch.float32, (F, SAMPLE_KEYS)), "count": (torch.int32, (F,))}
    if out is None:
        out = _empty_outputs(ctx, shapes)
    for k, (dt, shp) in shapes.items():
        _cuda_tensor(ctx, f"out[{k!r}]", out.get(k), dt, shp)
    ctx.check(ctx.L.vdo_sample_keys_dev(ctx.h, C.c_int(F), C.c_void_p(s.data_ptr()), C.c_int(width), C.c_int(height), C.c_void_p(out["x"].data_ptr()),
                                        C.c_void_p(out["y"].data_ptr()), C.c_void_p(out["count"].data_ptr()), C.c_uint64(_torch_stream(ctx))),
              "vdo_sample_keys_dev")
    return {k: out[k] for k in shapes}
