"""The linearisation tile kernel at the edges of its staging and of its vertex side, against the float64 reference (tests/ba_reference.py):
H_pp, b_p, H_ll, b_l and chi2 of debug_linearize, and the chi2-only form through the chi2 of one trial's updated estimates.

  * run descriptors (osegs2 / tsegs2) beyond the counts a tile stages in shared memory, for static and chain tiles;
  * a chain tile meeting 255 motion vertices (the 8-bit slot limit) and 200 cameras;
  * vertex runs of exactly 1, 15 and 16 entries (VDO_SEG2 = 15), for cameras and for motion vertices;
  * a batch whose graphs have small and large tile capacities, in both orders: the launch's shared memory is sized for the largest
    graph, each graph carves it by its own capacities.
"""
from __future__ import annotations

import numpy as np
import pytest

from vdo_slam_b200 import capi
from tests.ba_reference import Reference
from tests.ba_shapes import Scene, _cams, chains, motion_runs, vertex_runs
from tests.test_ba_operators import backend  # noqa: F401
from tests.test_ba_trial import TOL_BATCH, check, check_linearisation, check_trial


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
