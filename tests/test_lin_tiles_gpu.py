"""The linearisation tile kernel at the edges of its staging and of its vertex side, against the float64 reference (tests/ba_reference.py):
H_pp, b_p, H_ll, b_l and chi2 of debug_linearize, and the chi2-only form through the chi2 of one trial's updated estimates.  On the same
graphs in a batch, the preconditioner and back-substitution tiles, which also stage by the launch's capacities.

  * run descriptors (osegs2 / tsegs2) beyond the counts a tile stages in shared memory, for static and chain tiles;
  * a chain tile meeting 255 motion vertices (the 8-bit slot limit) and 200 cameras;
  * vertex runs of exactly 1, 15 and 16 entries (VDO_SEG2 = 15), for cameras and for motion vertices;
  * a batch whose graphs have small and large tile capacities, in both orders: the launch's shared memory is sized for the largest
    graph, each graph carves it by its own capacities.  The preconditioner is checked through the step of one chunk of 8 PCG iterations,
    which depends on it (dropping its landmark term moves that step by 2e-4 to 0.1 of its magnitude on these graphs):
      x_p after 8 iterations   |x_p - pcg8_ref|        <= 1e-10 max |pcg8_ref|
      x_l of that step         |x_l - backsub_ref(x_p)| <= 1e-11 max(its magnitude)
"""
from __future__ import annotations

import numpy as np
import pytest

from vdo_slam_b200 import capi
from tests.ba_reference import Reference
from tests.ba_shapes import Scene, _cams, chains, motion_runs, vertex_runs
from tests.test_ba_operators import backend  # noqa: F401
from tests.test_ba_trial import TOL_BATCH, TOL_XL, check, check_linearisation, check_trial

TOL_PCG8 = 1e-10


def static_many_runs(seed=21):
    """One static tile of 240 landmarks x 3 edges meeting 240 cameras: 240 camera runs, more than a static tile stages (192)."""
    s = Scene(240, seed)
    for k in range(240):
        s.static(_cams(s, k, 3))
    return s.graph()


def chain_many_runs(seed=22):
    """One chain of 256 landmarks, landmark k seen by camera k mod 200: a chain tile meeting 200 cameras and 255 motion vertices, with
    200 camera runs and 255 motion runs (more than the 96 of each a chain tile stages)."""
    return chains([256], n_cam=200, obs_per=1, seed=seed)


GRAPHS = {
    "static_many_runs": static_many_runs,
    "chain_many_runs": chain_many_runs,
    "static_runs_1_15_16": lambda: vertex_runs([1, 15, 16], seed=23),
    "motion_runs_1_15_16": lambda: motion_runs([1, 15, 16], seed=24),
}
_g, _ref = {}, {}


def graph(name):
    if name not in _g:
        _g[name] = GRAPHS[name]()
        _ref[name] = Reference(_g[name])
    return _g[name], _ref[name]


@pytest.mark.parametrize("name", list(GRAPHS))
def test_linearisation_and_chi2_match_float64_reference(backend, name):
    be, ctx = backend
    g, ref = graph(name)
    G = capi.BatchGraph(ctx, g)
    check_linearisation(be, G, ref, name)
    lam = ref.lambdas()[0]
    check_trial(be, g, ref, lam, False, G.debug_trial(lam), name)


@pytest.mark.parametrize("order", ["small_first", "large_first"])
def test_batch_of_small_and_large_tiles_matches_lone_graphs(backend, order):
    """A small chain graph and a small static graph beside the two graphs with the largest capacities (capE, capV, capH) above."""
    be, ctx = backend
    names = ["motion_runs_1_15_16", "static_runs_1_15_16", "chain_many_runs", "static_many_runs"]
    if order == "large_first":
        names = names[::-1]
    items = [graph(n) for n in names]
    Gs = [capi.BatchGraph(ctx, g) for g, _ in items]
    lams = [ref.lambdas()[0] for _, ref in items]
    outs = capi.debug_trial(Gs, lams)
    for name, (g, ref), G, lam, out in zip(names, items, Gs, lams, outs):
        where = f"{name} in a batch ({order})"
        check_trial(be, g, ref, lam, False, out, where)
        lone = G.debug_trial(lam)
        for f in ("xp", "xl", "se3", "pt"):
            check(be, "batch vs lone", np.abs(out[f] - lone[f]).max(), max(np.abs(lone[f]).max(), 1.0), TOL_BATCH, f"{where}: {f}")
        check(be, "batch vs lone", out["chi2"] - lone["chi2"], lone["chi2"], TOL_BATCH, f"{where}: chi2")
        check_linearisation(be, G, ref, where)


def pcg_reference(ref, lam, n):
    """x_p after n iterations of the preconditioned CG from x = 0, in float64 with the reference's S and M."""
    S, _ = ref.S(lam)
    M = ref.M(lam)
    b, _ = ref.rhs(lam)
    x, r = np.zeros_like(b), b.copy()
    z = np.linalg.solve(M, r)
    p, rz = z.copy(), r @ z
    for _ in range(n):
        Sp = S @ p
        a = rz / (p @ Sp)
        x += a * p
        r -= a * Sp
        z = np.linalg.solve(M, r)
        rz_new = r @ z
        p = z + (rz_new / rz) * p
        rz = rz_new
    return x


@pytest.mark.parametrize("order", ["small_first", "large_first"])
def test_batch_preconditioner_and_back_substitution_match_float64_reference(backend, order):
    """The graphs of the batch test above, one chunk of PCG iterations each (no graph converges at a relative tolerance of 1e-30).  A graph
    that the dense path solves has no preconditioner: its back-substitution is checked alone."""
    be, ctx = backend
    names = ["motion_runs_1_15_16", "static_runs_1_15_16", "chain_many_runs", "static_many_runs"]
    if order == "large_first":
        names = names[::-1]
    items = [graph(n) for n in names]
    Gs = [capi.BatchGraph(ctx, g) for g, _ in items]
    lams = [ref.lambdas()[0] for _, ref in items]
    outs = capi.debug_trial(Gs, lams, pcg_rel_tol=1e-30, pcg_max_iterations=8)
    for name, (g, ref), G, lam, out in zip(names, items, Gs, lams, outs):
        where = f"{name} in a batch ({order}), lambda={lam:.3g}"
        dense = G.solver_info()["dense"]
        assert out["ok"] and out["pcg_iterations"] == (0 if dense else 8), f"{where}: ok={out['ok']} after {out['pcg_iterations']} PCG iterations"
        xp, xl = out["xp"].ravel(), out["xl"].ravel()
        if not dense:
            x_ref = pcg_reference(ref, lam, 8)
            check(be, "x_p after 8 PCG iterations", np.abs(xp - x_ref).max(), np.abs(x_ref).max(), TOL_PCG8, where)
        xl_ref, xl_mag = ref.backsub(lam, xp)
        check(be, "step x_l", np.abs(xl - xl_ref).max(), xl_mag.max(), TOL_XL, where)
