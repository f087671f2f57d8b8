"""Float64 reference of the reduced-camera system the batch solver works on, built from the oracle's H and b.

Scalar order is the oracle's: 3 per point, then 6 per se3 vertex.  lambda is added to every diagonal entry of H (g2o's setLambda).
  S(lambda)   = H_pp + lambda I - sum_t H_pt (H_tt + lambda I)^-1 H_tp      (t: a static point, or a whole chain of landmarks)
  rhs(lambda) = b_p - H_pl (H_ll + lambda I)^-1 b_l
  backsub     = (H_ll + lambda I)^-1 (b_l - H_lp x_p)
  M(lambda)   = the preconditioner: H_pp + lambda I restricted to its 6x6 diagonal blocks and to the blocks of the se3-se3 edges of every
                connected component of the se3-se3 edge graph that is a simple path (branching or cyclic components keep their diagonal
                blocks only), minus, per vertex, the landmark term of each of its edges on its own (see M()).  That is the diagonal block
                of S(lambda) when a vertex meets every tracklet through at most one edge.
  scale       = sum x (lambda x + b) over x = (x_l, x_p), b at the estimates the reference was built on (g2o's computeScale)
Each tracklet block is inverted on its own (a chain has at most a few hundred landmarks), so S is exact to rounding.  Every operator
also returns the magnitude of the sum it forms (the same expression with absolute values), which scales the tolerances of the tests.
robust_chi2 and reorthogonalize are the LM update's other two references: the robust chi2 at any estimates, and g2o's
approximateNearestOrthogonalMatrix.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import pyoracle as po


def _components(n, edges):
    parent = np.arange(n)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in edges:
        ra, rb = find(int(a)), find(int(b))
        if ra != rb:
            parent[ra] = rb
    return np.array([find(i) for i in range(n)], np.int64)


def robust_chi2(g, se3, pt):
    """Robust chi2 of graph g with its estimates replaced by se3 (n_se3, 12) and pt (n_pt, 3)."""
    return po.ba_sparse_system(dict(g, se3=np.ascontiguousarray(se3, np.float64), pt=np.ascontiguousarray(pt, np.float64)))[2]


def reorthogonalize(R):
    """R - R (R^T R - I) / 2 of (..., 3, 3) rotations (isometry3d_mappings.h approximateNearestOrthogonalMatrix)."""
    R = np.asarray(R, np.float64)
    return R - 0.5 * R @ (np.swapaxes(R, -1, -2) @ R - np.eye(3))


def tracklets(g):
    """Landmark sets of the tracklets: chains linked by the landmark-motion edges, every other landmark alone."""
    P = len(g["pt"])
    comp = _components(P, g["ter_pph"][:, :2]) if len(g["ter_pph"]) else np.arange(P)
    order = np.argsort(comp, kind="stable")
    cuts = np.flatnonzero(np.diff(comp[order])) + 1
    return np.split(order, cuts)


def path_edges(g):
    """Indices of the se3-se3 edges that lie on a component of the se3-se3 edge graph that is a simple path."""
    C = len(g["se3"])
    ij = np.asarray(g["se3e_ij"], np.int64).reshape(-1, 2)
    if len(ij) == 0:
        return np.zeros(0, np.int64)
    comp = _components(C, ij)
    deg = np.bincount(ij.ravel(), minlength=C)
    n_v = np.bincount(comp, minlength=C)
    n_e = np.bincount(comp[ij[:, 0]], minlength=C)
    bad = np.zeros(C, bool)
    bad[comp[deg > 2]] = True
    is_path = (~bad) & (n_e == n_v - 1)
    return np.flatnonzero(is_path[comp[ij[:, 0]]])


class Reference:
    def __init__(self, g):
        H, b, self.chi2 = po.ba_sparse_system(g)
        self.P, self.C = len(g["pt"]), len(g["se3"])
        n3 = 3 * self.P
        H = H.tocsr()
        self.Hll = H[:n3, :n3].tocsr()
        self.Hlp = H[:n3, n3:].tocsr()
        self.Hpp = H[n3:, n3:].toarray()
        self.bl, self.bp = b[:n3].copy(), b[n3:].copy()
        self.max_diag = float(np.abs(H.diagonal()).max()) if H.shape[0] else 0.0
        self.tracklets = tracklets(g)
        self.path_edges = path_edges(g)
        self.ij = np.asarray(g["se3e_ij"], np.int64).reshape(-1, 2)
        cp = np.asarray(g["obs_cp"], np.int64).reshape(-1, 2)
        pph = np.asarray(g["ter_pph"], np.int64).reshape(-1, 3)
        assert len(np.unique(cp, axis=0)) == len(cp), "the preconditioner reference assumes one edge per (camera, point) pair"
        self._edge_sets = [(cp[:, 1:2], cp[:, 0]), (pph[:, :2], pph[:, 2])]
        self._cache = {}

    def lambdas(self):
        """The LM's initial damping (1e-5 max |H_jj|) and one 1e4 times larger."""
        lam = 1e-5 * self.max_diag
        return [lam, 1e4 * lam]

    def _linv(self, lam):
        """(H_ll + lam I)^-1, block diagonal by tracklet, as a sparse matrix."""
        if lam in self._cache:
            return self._cache[lam]
        rows, cols, vals = [], [], []
        single = np.array([t[0] for t in self.tracklets if len(t) == 1], np.int64)
        if len(single):
            B = np.zeros((len(single), 3, 3))
            for i in range(3):
                for j in range(3):
                    B[:, i, j] = np.asarray(self.Hll[3 * single + i, 3 * single + j]).ravel()
            B += lam * np.eye(3)
            Bi = np.linalg.inv(B)
            ii, jj = np.meshgrid(np.arange(3), np.arange(3), indexing="ij")
            rows.append((3 * single[:, None, None] + ii).ravel()); cols.append((3 * single[:, None, None] + jj).ravel()); vals.append(Bi.ravel())
        for t in self.tracklets:
            if len(t) == 1:
                continue
            idx = (3 * np.sort(t)[:, None] + np.arange(3)).ravel()
            A = self.Hll[idx][:, idx].toarray() + lam * np.eye(len(idx))
            Ai = np.linalg.solve(A, np.eye(len(idx)))
            Ai = 0.5 * (Ai + Ai.T)
            r, c = np.meshgrid(idx, idx, indexing="ij")
            rows.append(r.ravel()); cols.append(c.ravel()); vals.append(Ai.ravel())
        n3 = 3 * self.P
        if rows:
            Li = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n3, n3))
        else:
            Li = sp.csr_matrix((n3, n3))
        self._cache[lam] = Li
        return Li

    def S(self, lam):
        """Dense S(lam) and the dense magnitude |H_pp + lam I| + |H_pl| |(H_ll + lam I)^-1| |H_lp|."""
        key = ("S", lam)
        if key not in self._cache:
            Li = self._linv(lam)
            A = self.Hpp + lam * np.eye(6 * self.C)
            T = (self.Hlp.T @ (Li @ self.Hlp)).toarray()
            Habs = abs(self.Hlp)
            Tabs = (Habs.T @ (abs(Li) @ Habs)).toarray()
            self._cache[key] = (A - T, np.abs(A) + Tabs)
        return self._cache[key]

    def rhs(self, lam):
        Li = self._linv(lam)
        y = Li @ self.bl
        return self.bp - self.Hlp.T @ y, np.abs(self.bp) + abs(self.Hlp).T @ (abs(Li) @ np.abs(self.bl))

    def backsub(self, lam, xp):
        Li = self._linv(lam)
        xp = np.asarray(xp).ravel()
        return Li @ (self.bl - self.Hlp @ xp), abs(Li) @ (np.abs(self.bl) + abs(self.Hlp) @ np.abs(xp))

    def scale(self, lam, xp, xl):
        """sum x (lam x + b) over the step (xp: 6 per se3 vertex, xl: 3 per point) and its magnitude sum |x| (lam |x| + |b|)."""
        x = np.concatenate([np.asarray(xl).ravel(), np.asarray(xp).ravel()])
        b = np.concatenate([self.bl, self.bp])
        return float(x @ (lam * x + b)), float(np.abs(x) @ (lam * np.abs(x) + np.abs(b)))

    def M(self, lam):
        """Dense preconditioner matrix M(lam)."""
        key = ("M", lam)
        if key not in self._cache:
            Li = self._linv(lam).tocsr()
            M = np.zeros((6 * self.C, 6 * self.C))
            for v in range(self.C):
                M[6 * v:6 * v + 6, 6 * v:6 * v + 6] = self.Hpp[6 * v:6 * v + 6, 6 * v:6 * v + 6] + lam * np.eye(6)
            # landmark term, edge by edge: H_vL (H_LL + lam I)^-1 H_Lv over the landmarks L of one edge (one point, or the two points of a
            # landmark-motion edge).  It equals the diagonal block of H_pl (H_ll + lam I)^-1 H_lp whenever a vertex meets every tracklet
            # through at most one edge, as in the graphs the reference's optimisers build (one copy of a dynamic point per frame).
            for lm, v in self._edge_sets:
                if len(v) == 0:
                    continue
                idx = (3 * lm[:, :, None] + np.arange(3)).reshape(len(lm), -1)          # (E, 3 or 6) scalar rows
                cols = 6 * v[:, None] + np.arange(6)
                B = np.asarray(self.Hlp[np.repeat(idx, 6, 1).ravel(), np.tile(cols, (1, idx.shape[1])).ravel()]).reshape(len(v), idx.shape[1], 6)
                Lb = np.asarray(Li[np.repeat(idx, idx.shape[1], 1).ravel(), np.tile(idx, (1, idx.shape[1])).ravel()]).reshape(len(v), idx.shape[1], idx.shape[1])
                T = np.einsum("eia,eij,ejb->eab", B, Lb, B)
                np.add.at(M.reshape(self.C, 6, self.C, 6), (v, slice(None), v, slice(None)), -T)
            for e in self.path_edges:
                i, j = self.ij[e]
                M[6 * i:6 * i + 6, 6 * j:6 * j + 6] = self.Hpp[6 * i:6 * i + 6, 6 * j:6 * j + 6]
                M[6 * j:6 * j + 6, 6 * i:6 * i + 6] = self.Hpp[6 * j:6 * j + 6, 6 * i:6 * i + 6]
            self._cache[key] = M
        return self._cache[key]
