"""CPU-only tests of the product's host logic (graph ingestion, tracklet / chain ordering, LM + Schur + PCG driver,
C ABI) by linking the real driver against the serial kernel emulation in tests/emul (no CUDA involved), plus the
"library loads and exports every declared symbol" check for the CUDA build."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_batch_graph
from tests.ba_shapes import long_track_graph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tests", "emul", "libvdo_emul.so")


@pytest.fixture(scope="module")
def ectx():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emul"), "libvdo_emul.so"], stdout=subprocess.DEVNULL)
    return capi.Context(0, lib_path=EMUL)


def test_driver_matches_oracle_on_dynamic_graph(ectx):
    g = make_batch_graph(n_frames=14, n_objects=2, n_static=300, n_dynamic=120, seed=1)
    G = capi.BatchGraph(ectx, g)
    r = G.optimize()
    ro = po.ba_optimize(g)
    assert r["iterations"] == ro["iters"]
    se3, pt = G.vertices()
    assert np.abs(se3 - ro["se3"]).max() < 1e-5 and np.abs(pt - ro["pt"]).max() < 1e-5      # default PCG tolerance 1e-6; north_star: 1e-4
    assert r["pcg_iterations"] < 60 * r["trials"]      # the chain preconditioner keeps PCG short


def test_vertex_numbering_is_invisible_to_the_caller(ectx):
    g = make_batch_graph(n_frames=8, n_objects=1, n_static=60, n_dynamic=20, seed=2)
    rng = np.random.default_rng(0)
    C, P = len(g["se3"]), len(g["pt"])
    ps, pp = rng.permutation(C), rng.permutation(P)          # new index of old vertex
    h = dict(g)
    h["se3"] = np.empty_like(g["se3"]); h["se3"][ps] = g["se3"]
    h["pt"] = np.empty_like(g["pt"]); h["pt"][pp] = g["pt"]
    h["prior_v"] = ps[g["prior_v"]].astype(np.int32)
    h["se3e_ij"] = ps[g["se3e_ij"]].astype(np.int32)
    h["obs_cp"] = np.stack([ps[g["obs_cp"][:, 0]], pp[g["obs_cp"][:, 1]]], -1).astype(np.int32)
    h["ter_pph"] = np.stack([pp[g["ter_pph"][:, 0]], pp[g["ter_pph"][:, 1]], ps[g["ter_pph"][:, 2]]], -1).astype(np.int32)
    Ga, Gb = capi.BatchGraph(ectx, g), capi.BatchGraph(ectx, h)
    ra, rb = Ga.optimize(max_iterations=6, gain_threshold=0), Gb.optimize(max_iterations=6, gain_threshold=0)
    sa, pa = Ga.vertices(); sb, pb = Gb.vertices()
    np.testing.assert_allclose(sb[ps], sa, atol=1e-9)
    np.testing.assert_allclose(pb[pp], pa, atol=1e-9)


def test_error_paths(ectx):
    g = make_batch_graph(n_frames=5, n_objects=1, n_static=10, n_dynamic=6, seed=1)
    bad = dict(g); bad["obs_cp"] = g["obs_cp"].copy(); bad["obs_cp"][0, 1] = 10 ** 6
    with pytest.raises(capi.VdoError):
        capi.BatchGraph(ectx, bad)
    cyc = dict(g); t = g["ter_pph"].copy(); t[0, 1] = t[0, 0]; cyc["ter_pph"] = t
    with pytest.raises(capi.VdoError):
        capi.BatchGraph(ectx, cyc)


def test_empty_and_degenerate_graphs(ectx):
    g = make_batch_graph(n_frames=3, n_objects=0, n_static=5, n_dynamic=0, seed=1)
    G = capi.BatchGraph(ectx, g)
    r = G.optimize(max_iterations=3, gain_threshold=0)
    assert r["iterations"] >= 1 and np.isfinite(r["final_chi2"])
    # cameras only (pose graph): no landmarks at all
    h = dict(g); h["pt"] = np.zeros((0, 3)); h["obs_cp"] = np.zeros((0, 2), np.int32)
    for k in ("obs_z",): h[k] = np.zeros((0, 3))
    for k in ("obs_w", "obs_delta"): h[k] = np.zeros(0)
    G2 = capi.BatchGraph(ectx, h)
    r2 = G2.optimize(max_iterations=5, gain_threshold=0)
    ro = po.ba_optimize(h, max_iters=5, gain_threshold=0)
    assert np.abs(G2.vertices()[0] - ro["se3"]).max() < 1e-8


def test_cuda_library_exports_every_declared_symbol():
    from vdo_slam_b200 import build
    so = build.build()
    hdr = open(os.path.join(ROOT, "include", "vdo_b200.h")).read()
    names = sorted(set(re.findall(r"\b(vdo_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 15
    L = ctypes.CDLL(so)            # loads without a GPU; no compute call is made here
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/vdo_b200.h but not exported"


def test_product_refuses_to_run_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(capi.VdoError):
        capi.Context(0)


def test_tiled_and_chunked_layouts_agree(ectx, monkeypatch):
    """The default tiled layout (tiles of whole tracklets, vertex-sorted segments, world-frame sums) and the chunked
    vertex-major layout run the same LM: identical iteration / PCG counts, estimates equal to rounding."""
    g = make_batch_graph(n_frames=30, n_objects=2, n_static=1500, n_dynamic=400, seed=11)
    res = {}
    for lay in ("tiled", "chunked"):
        monkeypatch.setenv("VDO_BA_LAYOUT", lay)
        G = capi.BatchGraph(ectx, g)
        lin = G.debug_linearize()
        r = G.optimize(max_iterations=8, gain_threshold=0)
        res[lay] = (r, G.vertices(), lin)
    (ra, va, la), (rb, vb, lb) = res["tiled"], res["chunked"]
    assert ra["iterations"] == rb["iterations"] and ra["trials"] == rb["trials"] and ra["pcg_iterations"] == rb["pcg_iterations"]
    np.testing.assert_allclose(va[0], vb[0], atol=1e-10); np.testing.assert_allclose(va[1], vb[1], atol=1e-10)
    for x, y in zip(la, lb):       # H_pp blocks, b_p, H_ll, b_l, chi2 of the first linearisation
        x, y = np.asarray(x), np.asarray(y)
        assert np.abs(x - y).max() <= 1e-9 * max(1.0, np.abs(y).max())


def test_tracklet_too_large_for_a_tile_falls_back_to_the_chunked_layout(ectx):
    """A dynamic point tracked over more frames than a tile holds landmarks (VDO_TILE_L = 256) cannot be tiled: the graph
    is solved on the chunked layout instead of being rejected or truncated."""
    g = long_track_graph()
    G = capi.BatchGraph(ectx, g)
    r = G.optimize(max_iterations=2, gain_threshold=0)
    ro = po.ba_optimize(g, max_iters=2, gain_threshold=0)              # (the oracle's sparse Cholesky is the slow side here)
    assert r["iterations"] == ro["iters"]
    assert np.abs(G.vertices()[0] - ro["se3"]).max() < 1e-5 and np.abs(G.vertices()[1] - ro["pt"]).max() < 1e-5


@pytest.mark.parametrize("seed,frames,objs,ns,nd", [(21, 6, 1, 40, 10), (22, 45, 4, 900, 600), (23, 12, 0, 700, 0), (24, 25, 3, 5, 300), (25, 3, 1, 2000, 30)])
def test_tiled_layout_first_linearisation_and_schur_products_match_chunked(ectx, monkeypatch, seed, frames, objs, ns, nd):
    """Shape sweep (few / many tracklets per tile, static-only, dynamic-heavy, more edges than one tile holds): the first
    linearisation (H_pp, b_p, H_ll, b_l, chi2) and three LM iterations agree between the two layouts."""
    g = make_batch_graph(n_frames=frames, n_objects=objs, n_static=ns, n_dynamic=nd, seed=seed)
    out = {}
    for lay in ("tiled", "chunked"):
        monkeypatch.setenv("VDO_BA_LAYOUT", lay)
        G = capi.BatchGraph(ectx, g)
        lin = [np.asarray(x) for x in G.debug_linearize()]
        r = G.optimize(max_iterations=3, gain_threshold=0)
        out[lay] = (lin, r, G.vertices())
    for x, y in zip(out["tiled"][0], out["chunked"][0]):
        assert np.abs(x - y).max() <= 1e-9 * max(1.0, np.abs(y).max())
    assert out["tiled"][1]["iterations"] == out["chunked"][1]["iterations"]
    np.testing.assert_allclose(out["tiled"][2][0], out["chunked"][2][0], atol=1e-9)
    np.testing.assert_allclose(out["tiled"][2][1], out["chunked"][2][1], atol=1e-9)


def test_ingest_is_independent_of_the_host_thread_count(ectx, monkeypatch):
    """Graph ingestion is threaded (stable bucket partition of the edge list, per-tile sorts); the device layout -- and with it
    every sum order -- must not depend on the number of workers."""
    g = make_batch_graph(n_frames=25, n_objects=2, n_static=1200, n_dynamic=300, seed=9)
    res = []
    for nthreads in ("1", "5", "16"):
        monkeypatch.setenv("VDO_HOST_THREADS", nthreads)
        G = capi.BatchGraph(ectx, g)
        lin = [np.asarray(x) for x in G.debug_linearize()]
        G.optimize(max_iterations=3, gain_threshold=0)
        res.append((lin, G.vertices()))
    for lin, v in res[1:]:
        for x, y in zip(lin, res[0][0]):
            assert np.array_equal(x, y)
        assert np.array_equal(v[0], res[0][1][0]) and np.array_equal(v[1], res[0][1][1])


def test_banded_static_block_decision_and_result(ectx, monkeypatch):
    """Driver logic of the explicit banded static block (DESIGN.md 5d) on the emulated backend, which restates the band formation and the band
    product serially: it is chosen exactly when every static landmark lists its observing vertices in increasing order inside a window of 32
    vertex numbers, and the LM run is the same with and without it (and equal to the oracle's)."""
    g = make_batch_graph(n_frames=24, n_objects=2, n_static=500, n_dynamic=120, seed=11)
    ro = po.ba_optimize(g)
    G = capi.BatchGraph(ectx, g)
    si = G.solver_info()
    assert si["tiled"] == 1 and 0 < si["band_width"] <= 32 and si["band_rows"] >= 24 and si["dense"] == 0
    r = G.optimize(pcg_rel_tol=1e-10)
    a, b = G.vertices()
    assert r["iterations"] == ro["iters"] and np.abs(a - ro["se3"]).max() < 1e-7 and np.abs(b - ro["pt"]).max() < 1e-7
    # edge list reversed: a landmark's vertices now DEcrease along its edge list -> refused, matrix-free product, same answer
    h = dict(g)
    for k in ("obs_cp", "obs_z", "obs_w", "obs_delta"):
        h[k] = np.ascontiguousarray(g[k][::-1])
    H = capi.BatchGraph(ectx, h)
    assert H.solver_info()["band_width"] == 0
    r2 = H.optimize(pcg_rel_tol=1e-10)
    c, d = H.vertices()
    assert r2["iterations"] == ro["iters"] and np.abs(a - c).max() < 1e-7 and np.abs(b - d).max() < 1e-7
    # a landmark seen by two cameras 40 frames apart: wider than the widest band
    w = make_batch_graph(n_frames=48, n_objects=0, n_static=200, n_dynamic=0, seed=12)
    w = dict(w)
    cp = w["obs_cp"].copy()
    first = np.flatnonzero(cp[:, 1] == cp[0, 1])
    cp[first[0], 0] = 0; cp[first[-1], 0] = 45                  # (vertex numbers of the camera path follow the frame order)
    w["obs_cp"] = cp
    assert capi.BatchGraph(ectx, w).solver_info()["band_width"] == 0
    monkeypatch.setenv("VDO_BA_BAND", "0")
    assert capi.BatchGraph(ectx, g).solver_info()["band_width"] == 0


def test_two_contexts_ingest_concurrently(ectx):
    """The ingest's worker pool is process-wide and its sections are serialised: two host threads building graphs on two contexts at the
    same time (ctypes releases the GIL) must get the layouts and results of the serial runs."""
    import threading
    g = make_batch_graph(n_frames=30, n_objects=2, n_static=4000, n_dynamic=600, seed=5)
    ref = capi.BatchGraph(ectx, g)
    r0 = ref.optimize(max_iterations=3, gain_threshold=0)
    a0, b0 = ref.vertices()
    ctxs = [capi.Context(0, lib_path=EMUL) for _ in range(2)]
    out = [None, None]

    def work(i):
        for _ in range(3):
            G = capi.BatchGraph(ctxs[i], g)
            r = G.optimize(max_iterations=3, gain_threshold=0)
            out[i] = (r["chi2"].copy(), *G.vertices())
            G.close()

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in th: t.start()
    for t in th: t.join()
    for i in range(2):
        assert out[i] is not None
        np.testing.assert_array_equal(out[i][0], r0["chi2"])
        np.testing.assert_array_equal(out[i][1], a0); np.testing.assert_array_equal(out[i][2], b0)
