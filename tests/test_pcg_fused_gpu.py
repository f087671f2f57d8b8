"""The fused PCG iteration of the tiled layout on one GPU (DESIGN 5b): p update with the H_pp product, the landmark-side product (band or
static tiles, forked with the chain tiles), the finalize with the partials of p.Ap, and the PCR step (long-path clusters with the
short-path CTAs beside them), whose last CTA sets the scalars.

The PCG updates its residual by recurrence, r_{k+1} = r_k - alpha_k A p_k, with every A p_k formed inside the fused launches.  After a solve
that recurrence residual must equal rhs - S x computed by the separate operator kernels (debug_apply "S"): a wrong or stale Ap, p or vw in
any iteration, the first one included, would set the two apart.  This is checked at a graph that uses the band, at the same graph without
it (VDO_BA_BAND=0, static products by the matrix-free tile kernel) and with its edges listed backwards (no band either), for one chunk of
8 iterations and for a solve to a tight tolerance.  A batch of two PCG-path graphs of different sizes runs the same steps as one set of
launches per step and must end where each graph's own solve ends.  Graphs are closed inside each test, before the module's context."""
import numpy as np
import pytest

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_batch_graph

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def _graph(reverse=False, **kw):
    g = make_batch_graph(**(dict(n_frames=40, n_objects=2, n_static=6000, n_dynamic=1500, seed=11) | kw))
    if reverse:
        g = dict(g)
        for k in ("obs_cp", "obs_z", "obs_w", "obs_delta"):
            g[k] = np.ascontiguousarray(g[k][::-1])
    return g


@pytest.mark.parametrize("layout", ["band", "no_band", "reversed"])
@pytest.mark.parametrize("max_iters", [8, 2000])
def test_fused_recurrence_matches_operator(ctx, monkeypatch, layout, max_iters):
    if layout == "no_band":
        monkeypatch.setenv("VDO_BA_BAND", "0")
    G = capi.BatchGraph(ctx, _graph(reverse=layout == "reversed"))
    try:
        info = G.solver_info()
        assert info["tiled"] == 1 and info["dense"] == 0 and info["path_sharded"] == 0
        assert (info["band_width"] > 0) == (layout == "band")
        lam = 1e-2
        s = G.debug_solve(lam, pcg_rel_tol=1e-12, pcg_max_iterations=max_iters)
        rhs = G.debug_apply(lam, "rhs")
        true_r = rhs - G.debug_apply(lam, "S", s["xp"])
    finally:
        G.close()
    assert 0 < s["pcg_iterations"] <= max_iters
    scale = np.abs(rhs).max()
    assert np.abs(s["r"] - true_r).max() <= 1e-9 * scale
    if max_iters == 8:
        assert np.abs(true_r).max() < scale                 # the solve moved: the first direction was formed
    else:
        assert np.abs(true_r).max() <= 1e-5 * scale


def test_batch_of_two_pcg_graphs_matches_separate_solves(ctx):
    gs = [_graph(), _graph(n_frames=28, n_static=4000, n_dynamic=900, seed=12)]
    kw = dict(max_iterations=30, gain_threshold=1e-4)
    sep = []
    for g in gs:
        G = capi.BatchGraph(ctx, g)
        assert G.solver_info()["dense"] == 0
        sep.append((G.optimize(**kw), G.vertices()))
        G.close()
    Gs = [capi.BatchGraph(ctx, g) for g in gs]
    rs = capi.optimize_batch(Gs, **kw)
    ests = [G.vertices() for G in Gs]
    for G in Gs:
        G.close()
    for est, r, (r0, est0) in zip(ests, rs, sep):
        assert r["pcg_iterations"] > 0
        # fp64 atomics of the tile sums differ between any two solves; their effect passes through every PCG iteration
        assert r["iterations"] == r0["iterations"] and r["trials"] == r0["trials"]
        np.testing.assert_allclose(r["chi2"], r0["chi2"], rtol=1e-9)
        assert np.abs(est[0] - est0[0]).max() <= 1e-8 and np.abs(est[1] - est0[1]).max() <= 1e-8
