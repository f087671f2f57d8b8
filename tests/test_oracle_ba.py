"""Self-checks of the batch-LM oracle (oracle/ba_lm.c).  The reference ships no golden vectors, so the
restatement is checked through properties: analytic Jacobians vs finite differences (where g2o's own
Jacobians are exact derivatives), linear-solve residuals, monotone LM descent, termination rules."""
import numpy as np
import pytest

from oracle import pyoracle as po
from vdo_slam_b200.synth import make_batch_graph, iso, _rot, graph_sizes


def _rand_iso(rng, scale_t=2.0, ang=0.7):
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    return iso(_rot(ax, rng.uniform(-ang, ang)), rng.normal(scale=scale_t, size=3))


def _fd(fun, x0, apply, dim, eps=1e-6):
    J = np.zeros((len(fun(x0)), dim))
    for k in range(dim):
        d = np.zeros(dim); d[k] = eps
        J[:, k] = (fun(apply(x0, d)) - fun(apply(x0, -d))) / (2 * eps)
    return J


def test_edge_se3_jacobians_match_finite_differences():
    rng = np.random.default_rng(0)
    for _ in range(20):
        Z, Xi, Xj = _rand_iso(rng), _rand_iso(rng), _rand_iso(rng)
        e, Ji, Jj, _ = po.edge_eval(1, Z, Xi, Xj)
        Ji, Jj = Ji.reshape(6, 6), Jj.reshape(6, 6)
        fi = _fd(lambda X: po.edge_eval(1, Z, X, Xj)[0], Xi, po.iso_oplus, 6)
        fj = _fd(lambda X: po.edge_eval(1, Z, Xi, X)[0], Xj, po.iso_oplus, 6)
        np.testing.assert_allclose(Ji, fi, atol=2e-6)
        np.testing.assert_allclose(Jj, fj, atol=2e-6)


def test_edge_prior_jacobian_matches_finite_differences():
    rng = np.random.default_rng(1)
    for _ in range(10):
        Z, X = _rand_iso(rng), _rand_iso(rng)
        e, J, _, _ = po.edge_eval(0, Z, X, X)
        f = _fd(lambda T: po.edge_eval(0, Z, T, T)[0], X, po.iso_oplus, 6)
        np.testing.assert_allclose(J.reshape(6, 6), f, atol=2e-6)


def test_edge_obs_jacobians():
    rng = np.random.default_rng(2)
    for _ in range(10):
        X, p, z = _rand_iso(rng), rng.normal(size=3) * 5, rng.normal(size=3)
        e, Jc, Jp, _ = po.edge_eval(2, X, p, z)
        Jc, Jp = Jc[:18].reshape(3, 6), Jp[:9].reshape(3, 3)
        fc = _fd(lambda T: po.edge_eval(2, T, p, z)[0][:3], X, po.iso_oplus, 6)
        fp = _fd(lambda q: po.edge_eval(2, X, q, z)[0][:3], p, lambda q, d: q + d, 3)
        np.testing.assert_allclose(Jc, fc, atol=2e-6)
        np.testing.assert_allclose(Jp, fp, atol=2e-6)


def test_edge_ternary_jacobians_point_parts_exact_and_motion_part_is_g2o_approximation():
    rng = np.random.default_rng(3)
    p1, p2, H = rng.normal(size=3), rng.normal(size=3) * 3, _rand_iso(rng)
    e, J1, J2, Jh = po.edge_eval(3, p1, p2, H)
    f1 = _fd(lambda q: po.edge_eval(3, q, p2, H)[0][:3], p1, lambda q, d: q + d, 3)
    f2 = _fd(lambda q: po.edge_eval(3, p1, q, H)[0][:3], p2, lambda q, d: q + d, 3)
    fh = _fd(lambda T: po.edge_eval(3, p1, p2, T)[0][:3], H, po.iso_oplus, 6)
    np.testing.assert_allclose(J1[:9].reshape(3, 3), f1, atol=1e-6)
    np.testing.assert_allclose(J2[:9].reshape(3, 3), f2, atol=1e-6)
    Jh = Jh[:18].reshape(3, 6)
    np.testing.assert_allclose(Jh[:, :3], fh[:, :3], atol=1e-6)
    # the reference's rotational block is half the true derivative (types_dyn_slam3d.cpp:71-76 has no factor 2)
    np.testing.assert_allclose(2 * Jh[:, 3:], fh[:, 3:], atol=1e-5)


def test_dense_system_is_symmetric_psd_and_gradient_matches():
    g = make_batch_graph(n_frames=6, n_objects=1, n_static=40, n_dynamic=10, seed=7)
    H, b, chi = po.ba_dense_system(g)
    assert np.allclose(H, H.T)
    w = np.linalg.eigvalsh(H)
    assert w.min() > -1e-9 * w.max()
    assert chi > 0 and np.isfinite(b).all()


def test_lm_descends_and_terminates():
    g = make_batch_graph(n_frames=12, n_objects=1, n_static=300, n_dynamic=60, seed=3)
    r = po.ba_optimize(g, max_iters=100, gain_threshold=1e-4)
    chi = r["chi2"]
    assert r["iters"] >= 2 and r["iters"] <= 100
    assert (np.diff(chi) <= 1e-12).all()
    assert chi[-1] < chi[0]
    # fixed iteration budget path (terminate action disabled)
    r2 = po.ba_optimize(g, max_iters=5, gain_threshold=0.0)
    assert r2["iters"] == 5
    np.testing.assert_allclose(r2["chi2"], chi[:6], rtol=0, atol=0)


def test_generator_shapes():
    g = make_batch_graph(n_frames=10, n_objects=2, n_static=100, n_dynamic=30, seed=11)
    s = graph_sizes(g)
    assert s["E_p"] == len(g["obs_z"]) and s["P"] == len(g["pt_gt"])
    assert g["obs_cp"][:, 0].max() < 10 and g["obs_cp"][:, 1].max() < s["P"]
    if s["E_t"]:
        assert (g["ter_pph"][:, 1] == g["ter_pph"][:, 0] + 1).all()
        assert g["ter_pph"][:, 2].min() >= 10 and g["ter_pph"][:, 2].max() < s["C"]


# ---- the blocked direct solver (oracle/ba_block.h) is the same Cholesky solve as the scalar one (oracle/ba_lm.c) ----
@pytest.mark.parametrize("cfg", [dict(n_frames=30, n_objects=2, n_static=1500, n_dynamic=300, seed=1),
                                 dict(n_frames=16, n_objects=3, n_static=300, n_dynamic=500, seed=5),
                                 dict(n_frames=20, n_objects=0, n_static=800, n_dynamic=0, seed=2)])
def test_blocked_solver_equals_the_scalar_sparse_cholesky(cfg):
    g = make_batch_graph(**cfg)
    a = po.ba_optimize(g)
    for pos, nt in (("frame", 1), ("frame", 3), (None, 2)):
        b = po.ba_optimize_blocked(g, se3_pos=pos, nthreads=nt)
        assert a["iters"] == b["iters"]
        np.testing.assert_allclose(a["chi2"], b["chi2"], rtol=1e-8)
        assert np.abs(a["se3"] - b["se3"]).max() < 1e-7 and np.abs(a["pt"] - b["pt"]).max() < 1e-7


def test_blocked_solver_is_deterministic_across_thread_counts():
    g = make_batch_graph(n_frames=25, n_objects=2, n_static=900, n_dynamic=250, seed=11)
    a = po.ba_optimize_blocked(g, nthreads=1)
    b = po.ba_optimize_blocked(g, nthreads=5)
    assert a["iters"] == b["iters"] and np.array_equal(a["se3"], b["se3"]) and np.array_equal(a["pt"], b["pt"])


def test_first_lm_step_of_both_solvers_agrees_tightly():
    # one LM iteration = one linear solve: the two factorisations must agree to solver precision
    g = make_batch_graph(n_frames=40, n_objects=2, n_static=2500, n_dynamic=600, seed=3)
    a = po.ba_optimize(g, max_iters=1, gain_threshold=0.0)
    b = po.ba_optimize_blocked(g, max_iters=1, gain_threshold=0.0)
    assert np.abs(a["se3"] - b["se3"]).max() < 1e-11 and np.abs(a["pt"] - b["pt"]).max() < 1e-10


def test_sparse_system_export_matches_dense_export():
    g = make_batch_graph(n_frames=6, n_objects=2, n_static=40, n_dynamic=20, seed=3)
    H, b, chi = po.ba_dense_system(g)
    Hs, bs, chis = po.ba_sparse_system(g)
    assert Hs.shape == H.shape
    assert np.array_equal(Hs.toarray(), H)
    assert np.array_equal(bs, b) and chis == chi
