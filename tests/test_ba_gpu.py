"""GPU parity tests of the batch factor-graph path (through the C ABI of libvdo_b200.so) against the CPU oracle.
Tolerances: north_star asks pose / motion / point agreement <= 1e-4.  The only approximation on the GPU path is the PCG solve of the
reduced system (default relative tolerance 1e-6, the oracle factorises directly): the default is held to 1e-5 here, and a 1e-10 solve
to 1e-7, so that regressions show up early."""
import numpy as np
import pytest

from oracle import pyoracle as po
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_batch_graph, PARTIAL_BATCH, iso_inv, iso_mul, iso_t, iso_R
from tests.ba_shapes import long_track_graph

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def _pose_err(a, b):
    d = iso_mul(iso_inv(a), b)
    return float(np.abs(iso_t(d)).max()), float(np.abs(iso_R(d) - np.eye(3)).max())


def test_linearisation_matches_oracle_blocks(ctx):
    g = make_batch_graph(n_frames=8, n_objects=2, n_static=120, n_dynamic=40, seed=7)
    G = capi.BatchGraph(ctx, g)
    Hpp, bp, Hll, bl, chi = G.debug_linearize()
    H, b, chi_o = po.ba_dense_system(g)
    P, C = len(g["pt"]), len(g["se3"])
    assert abs(chi - chi_o) <= 1e-12 * chi_o
    Ho = H[3 * P:, 3 * P:]
    scale = np.abs(Hpp).max()
    for v in range(C):
        np.testing.assert_allclose(Hpp[v], Ho[6 * v:6 * v + 6, 6 * v:6 * v + 6], rtol=0, atol=1e-12 * scale)
    # odometry errors are pure rounding noise here (initial poses = chained odometry), times information 1e3
    np.testing.assert_allclose(bp, b[3 * P:].reshape(C, 6), rtol=0, atol=1e-9 * np.abs(bp).max())
    np.testing.assert_allclose(Hll, np.array([H[3 * k, 3 * k] for k in range(P)]), rtol=1e-12)
    np.testing.assert_allclose(bl, b[:3 * P].reshape(P, 3), rtol=0, atol=1e-11 * np.abs(bl).max())


@pytest.mark.parametrize("seed,frames,objs,ns,nd", [(1, 30, 2, 1500, 300), (2, 20, 0, 800, 0), (5, 16, 3, 300, 500)])
def test_full_batch_lm_matches_oracle(ctx, seed, frames, objs, ns, nd):
    g = make_batch_graph(n_frames=frames, n_objects=objs, n_static=ns, n_dynamic=nd, seed=seed)
    G = capi.BatchGraph(ctx, g)
    r = G.optimize(max_iterations=300, gain_threshold=1e-4)
    ro = po.ba_optimize(g, max_iters=300, gain_threshold=1e-4)
    assert r["iterations"] == ro["iters"]
    n = r["iterations"] + 1
    np.testing.assert_allclose(r["chi2"][:n], ro["chi2"][:n], rtol=1e-6)
    se3, pt = G.vertices()
    et, er = _pose_err(se3, ro["se3"])
    assert et <= 1e-5 and er <= 1e-5           # north_star tolerance: 1e-4
    assert np.abs(pt - ro["pt"]).max() <= 1e-5
    G.reset()
    r = G.optimize(max_iterations=300, gain_threshold=1e-4, pcg_rel_tol=1e-10)      # tight linear solves: the LM runs coincide
    assert r["iterations"] == ro["iters"]
    np.testing.assert_allclose(r["chi2"][:n], ro["chi2"][:n], rtol=1e-8)
    se3, pt = G.vertices()
    et, er = _pose_err(se3, ro["se3"])
    assert et <= 1e-7 and er <= 1e-7 and np.abs(pt - ro["pt"]).max() <= 1e-7


def test_partial_batch_constants_static_only(ctx):
    # the sliding-window optimiser: 20 frames, camera poses + static points only (src/Optimizer.cc:190-213)
    g = make_batch_graph(n_frames=20, n_objects=0, n_static=2000, n_dynamic=0, seed=9, consts=PARTIAL_BATCH)
    G = capi.BatchGraph(ctx, g)
    r = G.optimize(max_iterations=100, gain_threshold=1e-3)
    ro = po.ba_optimize(g, max_iters=100, gain_threshold=1e-3)
    assert r["iterations"] == ro["iters"]
    se3, pt = G.vertices()
    assert max(_pose_err(se3, ro["se3"])) <= 1e-5 and np.abs(pt - ro["pt"]).max() <= 1e-5


def test_dense_reduced_system_path_matches_oracle_and_pcg(ctx, monkeypatch):
    """NS1: small static-only graphs (the 20-camera sliding window) form S explicitly and factor it on the fp64 tensor cores (mma.sync m8n8k4)
    instead of running the matrix-free PCG: a direct solve, so the LM run coincides with the oracle's to rounding; the PCG path agrees."""
    g = make_batch_graph(n_frames=20, n_objects=0, n_static=2500, n_dynamic=0, seed=13, consts=PARTIAL_BATCH)
    ro = po.ba_optimize(g, max_iters=100, gain_threshold=1e-3)
    G = capi.BatchGraph(ctx, g)                                   # qualifies: tiled, static only, 6C = 120 <= 168
    r = G.optimize(max_iterations=100, gain_threshold=1e-3)
    assert r["iterations"] == ro["iters"] and r["pcg_iterations"] == 0        # no PCG ran
    n = r["iterations"] + 1
    np.testing.assert_allclose(r["chi2"][:n], ro["chi2"][:n], rtol=1e-9)
    se3, pt = G.vertices()
    assert max(_pose_err(se3, ro["se3"])) <= 1e-8 and np.abs(pt - ro["pt"]).max() <= 1e-8
    monkeypatch.setenv("VDO_BA_DENSE", "0")
    G2 = capi.BatchGraph(ctx, g)
    r2 = G2.optimize(max_iterations=100, gain_threshold=1e-3, pcg_rel_tol=1e-10)
    assert r2["iterations"] == ro["iters"] and r2["pcg_iterations"] > 0
    se3b, ptb = G2.vertices()
    assert max(_pose_err(se3, se3b)) <= 1e-7 and np.abs(pt - ptb).max() <= 1e-7


def test_banded_static_block_matches_matrix_free_product(ctx, monkeypatch):
    """Graphs whose static landmarks list their observing vertices in increasing order within 32 consecutive vertex numbers (tracks over
    consecutive frames) form the static block of the reduced matrix explicitly (10 moments per vertex pair, re-formed per trial) and multiply
    by it inside the PCG; any other graph keeps the matrix-free tile kernel.  Both give the oracle's solve."""
    g = make_batch_graph(n_frames=40, n_objects=2, n_static=3000, n_dynamic=400, seed=21)
    ro = po.ba_optimize(g, max_iters=300, gain_threshold=1e-4)
    G = capi.BatchGraph(ctx, g)
    si = G.solver_info()
    assert si["tiled"] == 1 and 0 < si["band_width"] <= 32 and si["band_rows"] >= 40
    r = G.optimize(max_iterations=300, gain_threshold=1e-4, pcg_rel_tol=1e-10)
    a, b = G.vertices()
    assert r["iterations"] == ro["iters"] and max(_pose_err(a, ro["se3"])) <= 1e-7 and np.abs(b - ro["pt"]).max() <= 1e-7
    # the same edges listed backwards: vertex numbers decrease along a landmark's edge list -> no band, same answer
    g2 = dict(g)
    for k in ("obs_cp", "obs_z", "obs_w", "obs_delta"):
        g2[k] = np.ascontiguousarray(g[k][::-1])
    G2 = capi.BatchGraph(ctx, g2)
    assert G2.solver_info()["band_width"] == 0
    r2 = G2.optimize(max_iterations=300, gain_threshold=1e-4, pcg_rel_tol=1e-10)
    c, d = G2.vertices()
    assert r2["iterations"] == ro["iters"] and max(_pose_err(a, c)) <= 1e-7 and np.abs(b - d).max() <= 1e-7
    monkeypatch.setenv("VDO_BA_BAND", "0")
    G3 = capi.BatchGraph(ctx, g)
    assert G3.solver_info()["band_width"] == 0
    r3 = G3.optimize(max_iterations=300, gain_threshold=1e-4, pcg_rel_tol=1e-10)
    e, f = G3.vertices()
    assert r3["iterations"] == ro["iters"] and max(_pose_err(a, e)) <= 1e-7 and np.abs(b - f).max() <= 1e-7


def test_reset_and_repeat_is_reproducible_to_rounding(ctx):
    g = make_batch_graph(n_frames=15, n_objects=1, n_static=500, n_dynamic=100, seed=4)
    G = capi.BatchGraph(ctx, g)
    r1 = G.optimize(max_iterations=10, gain_threshold=0.0)
    a, b = G.vertices()
    G.reset()
    r2 = G.optimize(max_iterations=10, gain_threshold=0.0)
    c, d = G.vertices()
    assert r1["iterations"] == r2["iterations"] == 10
    assert np.abs(a - c).max() <= 1e-9 and np.abs(b - d).max() <= 1e-9   # fp64 atomics reorder sums


def test_large_graph_properties(ctx):
    # config-4-shaped graph at 1/4 scale: too slow for the oracle's full run, so check size-independent properties:
    # monotone robust chi2, agreement of the first LM iterations with the oracle, finite estimates
    g = make_batch_graph(n_frames=100, n_objects=3, n_static=10000, n_dynamic=2500, seed=4)
    G = capi.BatchGraph(ctx, g)
    r = G.optimize(max_iterations=12, gain_threshold=0.0)
    chi = r["chi2"]
    assert (np.diff(chi) <= 0).all() and chi[-1] < chi[0]
    ro = po.ba_optimize(g, max_iters=3, gain_threshold=0.0)
    np.testing.assert_allclose(chi[:4], ro["chi2"][:4], rtol=1e-6)
    se3, pt = G.vertices()
    assert np.isfinite(se3).all() and np.isfinite(pt).all()


def test_tracklet_too_large_for_a_tile_falls_back_to_the_chunked_layout(ctx):
    """A dynamic point tracked over more frames than a tile holds landmarks (VDO_TILE_L = 256) runs the chunked kernels (k_lin_static,
    k_lin_tracklets, k_vertex_sym, k_schur_static, k_schur_chains8, k_schur_vertex) in a full LM run that matches the oracle."""
    g = long_track_graph()
    G = capi.BatchGraph(ctx, g)
    assert G.solver_info()["tiled"] == 0
    r = G.optimize(max_iterations=2, gain_threshold=0)
    ro = po.ba_optimize(g, max_iters=2, gain_threshold=0)
    assert r["iterations"] == ro["iters"]
    assert np.abs(G.vertices()[0] - ro["se3"]).max() < 1e-5 and np.abs(G.vertices()[1] - ro["pt"]).max() < 1e-5


def test_rejects_branching_landmark_motion_graph(ctx):
    g = make_batch_graph(n_frames=6, n_objects=1, n_static=20, n_dynamic=10, seed=1)
    g = dict(g)
    t = g["ter_pph"].copy()
    t[1, 0] = t[0, 0]                      # two successors for one landmark
    g["ter_pph"] = t
    with pytest.raises(capi.VdoError):
        capi.BatchGraph(ctx, g)


def test_two_gpu_sharded_solve_matches_oracle(tmp_path):
    import os, socket, subprocess, sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "r0.npz")
    procs = [subprocess.Popen([sys.executable, os.path.join(root, "tests", "_dist_worker_gpu.py"), str(r), "2", str(port), out]) for r in range(2)]
    for p in procs:
        assert p.wait(timeout=600) == 0
    d = np.load(out)
    g = make_batch_graph(n_frames=30, n_objects=2, n_static=1500, n_dynamic=300, seed=1)
    ro = po.ba_optimize(g)
    assert int(d["iters"]) == ro["iters"]
    assert np.abs(d["se3"] - ro["se3"]).max() < 1e-5 and np.abs(d["pt"] - ro["pt"]).max() < 1e-5
    # BASELINE config 4 sharded over 2 ranks against the oracle's frozen full solve
    gold = np.load(os.path.join(root, "tests", "golden", "ba_config4.npz"))
    assert int(d["c4_iters"]) == int(gold["iters"])
    np.testing.assert_allclose(d["c4_chi2"][: int(gold["iters"]) + 1], gold["chi2"], rtol=1e-6)
    assert max(_pose_err(d["c4_se3"], gold["se3"])) <= 1e-5 and np.abs(d["c4_pt"][gold["pt_idx"]] - gold["pt"]).max() <= 1e-5
