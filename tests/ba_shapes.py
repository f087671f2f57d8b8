"""Small batch graphs, each built to put one boundary of the batch solver's kernels under test.

Every graph has non-identity camera rotations and object motions of 10-20 degrees (so the rotated-frame chain algebra, the world-frame
vertex sums and the moving of torques between origins all matter), estimates perturbed off the ground truth, and Huber deltas set per
(information, delta) class so that the edges of one class fall on both sides of the quadratic / linear switch.

SHAPES maps a name to a function returning (graph dict in the synth.make_batch_graph layout, expectations).  Expectations are checked
against BatchGraph.solver_info() of the default layout ("dense" only where the backend has a dense path); REFUSED holds graphs that
vdo_graph_finalize must refuse with VDO_ERR_UNSUPPORTED.  Kernel limits the shapes aim at (vdo_slam_b200/csrc/ba_types.h): VDO_TILE_L = 256 landmarks and
VDO_TILE_E = 768 pointxyz edges per tile, 255 vertices per tile, vertex runs cut at VDO_SEG2 = 15 and VDO_SEG = 64, paths of the
preconditioner up to VDO_PCR_SHORT = 32 vertices on one CTA, bands up to 32 vertices wide, 6C <= 168 on the dense path, 256 edge classes.
"""
from __future__ import annotations

import numpy as np

from oracle import pyoracle as po
from vdo_slam_b200.synth import _rot, iso, iso_R, iso_t, iso_inv, iso_mul, iso_apply

VDO_ERR_UNSUPPORTED = -3


def _rand_rot(rng, lo=10.0, hi=20.0):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    return _rot(ax, np.deg2rad(rng.uniform(lo, hi)) * rng.choice([-1.0, 1.0]))


class Scene:
    """Ground truth first (cameras along a line, each turned 10-20 degrees; object motions turning 10-20 degrees about a pivot near the
    points they move), then graph() perturbs the estimates and adds measurement noise."""

    def __init__(self, n_cam, seed, odometry=True):
        self.rng = np.random.default_rng(seed)
        self.se3 = [iso(_rand_rot(self.rng), np.array([0.8 * k, 0.3 * np.sin(k), 0.1 * k])) for k in range(n_cam)]
        self.n_cam = n_cam
        self.se3e = [(k, k + 1) for k in range(n_cam - 1)] if odometry else []
        self.pts, self.obs, self.ter = [], [], []

    def cam_point(self, c):
        """A world point 4-12 m in front of camera c."""
        T = self.se3[c]
        return iso_apply(T, np.array([self.rng.uniform(-3, 3), self.rng.uniform(-2, 2), self.rng.uniform(4, 12)]))

    def motion(self, pivot):
        R = _rand_rot(self.rng)
        v = self.rng.normal(scale=0.3, size=3)
        self.se3.append(iso(R, pivot - R @ pivot + v))
        return len(self.se3) - 1

    def motion_path(self, n, pivot, smooth=True):
        ids = [self.motion(pivot) for _ in range(n)]
        if smooth:
            self.se3e += [(ids[k], ids[k + 1]) for k in range(n - 1)]
        return ids

    def static(self, cams, p=None):
        p = self.cam_point(cams[0]) if p is None else p
        self.pts.append(p)
        k = len(self.pts) - 1
        self.obs += [(c, k) for c in cams]
        return k

    def chain(self, cams_per, motions):
        """Landmarks p_0 .. p_{L-1} of one dynamic point, p_{k+1} = H_{motions[k]} p_k, landmark k seen by cams_per[k]."""
        first = next((c[0] for c in cams_per if len(c)), 0)
        p = self.cam_point(first)
        ids = []
        for k, cams in enumerate(cams_per):
            ids.append(self.static(cams, p))
            if k + 1 < len(cams_per):
                H = self.se3[motions[k]]
                p = iso_R(H) @ p + iso_t(H)
                self.ter.append((ids[-1], len(self.pts), motions[k]))
        return ids

    def graph(self, obs_classes=4, ter_classes=4, se3_classes=2, obs_order=None):
        rng = self.rng
        se3_gt = np.array(self.se3)
        pt_gt = np.array(self.pts).reshape(-1, 3)
        C, P = len(se3_gt), len(pt_gt)
        se3 = np.array([iso_mul(T, iso(_rand_rot(rng, 0.5, 1.5), rng.normal(scale=0.02, size=3))) for T in se3_gt])
        pt = pt_gt + rng.normal(scale=0.03, size=pt_gt.shape)
        cp = np.array(self.obs, np.int32).reshape(-1, 2)
        if obs_order is not None:
            cp = cp[obs_order]
        z = iso_apply(iso_inv(se3_gt[cp[:, 0]]), pt_gt[cp[:, 1]]) + rng.normal(scale=0.01, size=(len(cp), 3))
        e_obs = iso_apply(iso_inv(se3[cp[:, 0]]), pt[cp[:, 1]]) - z
        pph = np.array(self.ter, np.int32).reshape(-1, 3)
        e_ter = pt[pph[:, 0]] - iso_apply(iso_inv(se3[pph[:, 2]]), pt[pph[:, 1]]) if len(pph) else np.zeros((0, 3))
        ij = np.array(self.se3e, np.int32).reshape(-1, 2)
        Z = np.array([iso_mul(iso_mul(iso_inv(se3_gt[i]), se3_gt[j]), iso(_rot(np.array([0, 0, 1.0]), rng.normal(scale=0.01)), rng.normal(scale=0.01, size=3)))
                      for i, j in ij]).reshape(-1, 12)
        e_se3 = np.array([po.edge_eval(1, Z[k], se3[i], se3[j])[0] for k, (i, j) in enumerate(ij)]).reshape(-1, 6)

        def classes(err, n_cls, w0):
            """(w, delta) per edge: class = edge index mod n_cls; delta between the robust norms of the class's edges."""
            n = len(err)
            cls = np.arange(n) % max(n_cls, 1)
            w = w0 * (1.0 + 0.01 * cls)
            r = np.sqrt(w * (err ** 2).sum(1))
            d = np.zeros(n)
            for c in range(max(n_cls, 1)):
                m = cls == c
                if m.any():
                    d[m] = np.median(r[m]) * (0.7 if c % 2 else 1.3)
            return w, d
        ow, od = classes(e_obs, obs_classes, 16.0)
        tw, td = classes(e_ter, ter_classes, 10.0)
        sw, sd = classes(e_se3, se3_classes, 100.0)
        g = dict(se3=se3, pt=pt, prior_v=np.zeros(1, np.int32), prior_Z=se3_gt[:1].copy(), prior_w=np.array([1e4]),
                 se3e_ij=ij, se3e_Z=Z, se3e_w=sw, se3e_delta=sd, obs_cp=cp, obs_z=z, obs_w=ow, obs_delta=od,
                 ter_pph=pph, ter_w=tw, ter_delta=td)
        for k, v in list(g.items()):
            g[k] = np.ascontiguousarray(v, dtype=np.int32 if v.dtype.kind == "i" else np.float64)
        return g


def _cams(s, k, n):
    """n consecutive cameras starting at k (wrapping)."""
    return [(k + i) % s.n_cam for i in range(n)]


def chains(lengths, n_cam=24, obs_per=2, seed=1, lone=0):
    """One chain per length (its own path of motion vertices), plus `lone` dynamic points without a landmark-motion edge."""
    s = Scene(n_cam, seed)
    for i, L in enumerate(lengths):
        piv = s.cam_point(i % n_cam)
        mot = s.motion_path(L - 1, piv)
        s.chain([_cams(s, (i + k) % n_cam, obs_per) for k in range(L)], mot)
    for i in range(lone):
        s.static(_cams(s, i, 1))
    return s.graph()


def static_tile_fill(seed=2):
    """192 points x 4 edges fill one static tile to exactly 768 edges; a 193rd point with one edge makes 769."""
    s = Scene(16, seed)
    for k in range(192):
        s.static(_cams(s, k % 13, 4))
    s.static([15])
    return s.graph()


def static_odd(seed=3):
    """Edge counts per landmark 1..5 (a total that is not a multiple of 16), a landmark with no observation, cameras with no landmark."""
    s = Scene(16, seed)
    for k in range(37):
        s.static(_cams(s, k % 8, 1 + k % 5))
    s.pts.append(s.cam_point(3))                       # no observation at all
    return s.graph()


def static_255_cams(seed=4):
    """Point k seen by cameras k and k+1: the first static tile meets exactly 255 cameras (the 8-bit slot limit)."""
    s = Scene(300, seed)
    for k in range(299):
        s.static([k, k + 1])
    return s.graph()


def vertex_runs(sizes, seed=5):
    """For each n in sizes: n landmarks of one tile seen by one camera (runs cut at 15 and 64 entries), each also by a second camera."""
    s = Scene(2 * len(sizes) + 2, seed)
    for i, n in enumerate(sizes):
        for k in range(n):
            s.static([2 * i, 2 * i + 1])
    return s.graph()


def motion_runs(sizes, seed=6):
    """For each n in sizes: n chains of two landmarks whose landmark-motion edges share one motion vertex."""
    s = Scene(10, seed)
    for i, n in enumerate(sizes):
        h = s.motion(s.cam_point(i))
        for k in range(n):
            s.chain([[i], [i + 1]], [h])
    return s.graph()


def precond_paths(seed=7):
    """Paths of the se3-se3 edge graph with 1, 2, 32, 33, 64, 65 and 300 vertices (the camera path), a branching and a cyclic component."""
    s = Scene(300, seed)
    for k in range(0, 298, 2):
        s.static([k, k + 1, k + 2])
    for i, n in enumerate((1, 2, 32, 33, 64, 65)):
        mot = s.motion_path(n, s.cam_point(i))
        s.chain([[(i * 7 + k) % 300] for k in range(n + 1)], mot)
    star = s.motion_path(4, s.cam_point(50), smooth=False)
    s.se3e += [(star[0], star[1]), (star[0], star[2]), (star[0], star[3])]
    ring = s.motion_path(4, s.cam_point(60))
    s.se3e.append((ring[3], ring[0]))
    for grp in (star, ring):
        for h in grp:
            s.chain([[50], [51]], [h])
    return s.graph()


def band(width, n_cam=40, seed=8, decreasing=False):
    """Static points over consecutive cameras, the widest spanning `width` camera numbers (in decreasing order if `decreasing`)."""
    s = Scene(n_cam, seed)
    for k in range(n_cam - width + 1):
        s.static(list(range(k, k + width)) if width <= 3 else [k, k + width // 2, k + width - 1])
        s.static([k + (k * 5) % width])
    g = s.graph()
    if decreasing:
        s2 = Scene(n_cam, seed)
        s2.se3, s2.se3e, s2.pts, s2.obs = s.se3, s.se3e, s.pts, s.obs
        g = s2.graph(obs_order=np.arange(len(s.obs))[::-1])
    return g


def dense(n_cam, seed=9):
    """Static-only graph of n_cam cameras: 6C = 162, 168 (the dense path's capacity) or 174 (PCG)."""
    s = Scene(n_cam, seed)
    for k in range(4 * n_cam):
        s.static(_cams(s, k % (n_cam - 3), 3))
    return s.graph()


def edge_classes(n_obs_cls, n_ter_cls, seed=10):
    """n distinct (information, Huber delta) pairs on the pointxyz and on the landmark-motion edges."""
    s = Scene(20, seed)
    piv = s.cam_point(0)
    for i in range(6):
        mot = s.motion_path(50, piv)
        s.chain([_cams(s, (i + k) % 20, 1) for k in range(51)], mot)
    for k in range(40):
        s.static(_cams(s, k % 18, 2))
    return s.graph(obs_classes=n_obs_cls, ter_classes=n_ter_cls)


def permuted(seed=11):
    """A mixed graph handed over with its se3 and point ids randomly permuted."""
    g = chains([2, 17, 40], n_cam=16, seed=seed, lone=3)
    s = Scene(1, seed)
    rng = s.rng
    C, P = len(g["se3"]), len(g["pt"])
    ps, pp = rng.permutation(C), rng.permutation(P)
    h = dict(g)
    h["se3"] = np.empty_like(g["se3"]); h["se3"][ps] = g["se3"]
    h["pt"] = np.empty_like(g["pt"]); h["pt"][pp] = g["pt"]
    h["prior_v"] = ps[g["prior_v"]].astype(np.int32)
    h["se3e_ij"] = ps[g["se3e_ij"]].astype(np.int32)
    h["obs_cp"] = np.stack([ps[g["obs_cp"][:, 0]], pp[g["obs_cp"][:, 1]]], -1).astype(np.int32)
    h["ter_pph"] = np.stack([pp[g["ter_pph"][:, 0]], pp[g["ter_pph"][:, 1]], ps[g["ter_pph"][:, 2]]], -1).astype(np.int32)
    return {k: np.ascontiguousarray(v) for k, v in h.items()}


def push_off_orthonormal(g, seed, eps=1e-7):
    """g with every input rotation pushed ~eps off orthonormal (R + eps N), so that the re-orthogonalisation of the update moves it by
    ~eps (it moves an orthonormal rotation by ~1e-16, which no test can tell from not re-orthogonalising)."""
    g = dict(g, se3=g["se3"].copy())
    g["se3"][:, :9] += eps * np.random.default_rng(seed).standard_normal((len(g["se3"]), 9))
    return g


def off_orthonormal(seed=12, eps=1e-7):
    """A small mixed graph with its rotations off orthonormal (push_off_orthonormal).  Not in SHAPES: the operator tests keep
    their graphs."""
    return push_off_orthonormal(chains([2, 5, 9], n_cam=8, seed=seed, lone=2), seed, eps)


def long_track_graph():
    """One dynamic point tracked over 258 frames (more landmarks than a tile holds), 40 static points, identity rotations: the graph
    falls back to the chunked layout."""
    rng = np.random.default_rng(5)
    F = 258
    I9 = np.eye(3).reshape(-1)

    def iso(t):
        return np.concatenate([I9, np.asarray(t, float)])
    cams = np.array([iso([0.05 * f, 0, 0]) for f in range(F)])
    H_true = iso([0.1, 0.0, 0.02])                                           # constant object motion per frame (world frame)
    mots = np.array([H_true for _ in range(F - 1)])
    dyn = np.array([[2.0, 0.5, 12.0] + f * H_true[9:] for f in range(F)])     # one dynamic point, one copy per frame
    stat = rng.uniform([-5, -2, 8], [20, 2, 30], (40, 3))
    se3 = np.concatenate([cams, mots]); pt = np.concatenate([stat, dyn])
    cp, z = [], []
    for f in range(F):
        for j in range(len(stat)):
            if (j + f) % 4 == 0:
                cp.append((f, j)); z.append(stat[j] - cams[f, 9:] + rng.normal(0, 0.01, 3))
        cp.append((f, len(stat) + f)); z.append(dyn[f] - cams[f, 9:] + rng.normal(0, 0.01, 3))
    ij = [(f, f + 1) for f in range(F - 1)] + [(F + k, F + k + 1) for k in range(F - 2)]
    Z = [iso([0.05, 0, 0])] * (F - 1) + [iso([0, 0, 0])] * (F - 2)
    w = [100.0] * (F - 1) + [50.0] * (F - 2)
    ter = [(len(stat) + f, len(stat) + f + 1, F + f) for f in range(F - 1)]
    return {"se3": se3 + np.concatenate([np.zeros((len(se3), 9)), rng.normal(0, 0.01, (len(se3), 3))], 1), "pt": pt + rng.normal(0, 0.03, pt.shape),
            "prior_v": np.array([0], np.int32), "prior_Z": cams[:1].copy(), "prior_w": np.array([1e4]),
            "se3e_ij": np.array(ij, np.int32), "se3e_Z": np.array(Z), "se3e_w": np.array(w), "se3e_delta": np.full(len(w), 0.1),
            "obs_cp": np.array(cp, np.int32), "obs_z": np.array(z), "obs_w": np.full(len(cp), 16.0), "obs_delta": np.full(len(cp), 0.05),
            "ter_pph": np.array(ter, np.int32), "ter_w": np.full(len(ter), 20.0), "ter_delta": np.full(len(ter), 0.05)}


SHAPES = {
    # chain length in a tile: warp scan (1, 2, 31, 32, 33), 8-warp carry (64, 255), a full tile (256)
    "chains_short": lambda: (chains([2, 31, 32, 33], lone=1), {"tiled": 1}),
    "chain_64": lambda: (chains([64, 5]), {"tiled": 1}),
    "chain_255": lambda: (chains([255], n_cam=40, obs_per=3), {"tiled": 1}),
    # 256 landmarks and 768 edges in one chain tile, 255 motion vertices (the most a chain tile can meet)
    "chain_256": lambda: (chains([256], n_cam=40, obs_per=3), {"tiled": 1}),
    "chain_257": lambda: (chains([257], n_cam=40, obs_per=2), {"tiled": 0}),
    "static_tile_fill": lambda: (static_tile_fill(), {"tiled": 1, "n_tiles": 2}),
    "static_odd": lambda: (static_odd(), {"tiled": 1}),
    "static_255_cams": lambda: (static_255_cams(), {"tiled": 1, "n_tiles": 2}),
    "vertex_runs": lambda: (vertex_runs([15, 16, 30, 64, 65]), {"tiled": 1, "n_tiles": 1}),
    "vertex_run_100": lambda: (vertex_runs([100]), {"tiled": 1, "n_tiles": 1}),
    "motion_runs": lambda: (motion_runs([15, 16, 30, 64]), {"tiled": 1}),
    "precond_paths": lambda: (precond_paths(), {"tiled": 1}),
    "band_1": lambda: (band(1), {"band_width": 1}),
    "band_8": lambda: (band(8), {"band_width": 8}),
    "band_9": lambda: (band(9), {"band_width": 9}),
    "band_32": lambda: (band(32), {"band_width": 32}),
    "band_33": lambda: (band(33), {"band_width": 0}),
    "band_decreasing": lambda: (band(5, decreasing=True), {"band_width": 0}),
    "dense_162": lambda: (dense(27), {"dense": 1}),
    "dense_168": lambda: (dense(28), {"dense": 1}),
    "dense_174": lambda: (dense(29), {"dense": 0}),
    "classes_256": lambda: (edge_classes(256, 256), {"tiled": 1}),
    "permuted": lambda: (permuted(), {}),
}
# finalize must refuse these
REFUSED = {
    "classes_257_obs": lambda: edge_classes(257, 4),
    "classes_257_ter": lambda: edge_classes(4, 257),
}
