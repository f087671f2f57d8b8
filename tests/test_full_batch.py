"""vdo_graph_optimize_batch with several PCG-path graphs on the serial kernel emulation (tests/emul): the batched PCG trials (preconditioner,
rhs, init and chunks of 8 iterations for every graph still iterating, one read-back per chunk) must give every graph exactly what its own
vdo_graph_optimize gives.  The emulation is serial, so the results are compared bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_batch_graph, PARTIAL_BATCH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ba_shapes  # noqa: E402

EMUL = os.path.join(ROOT, "tests", "emul", "libvdo_emul.so")
PER_GRAPH = ("iterations", "trials", "pcg_iterations", "initial_chi2", "final_chi2", "final_lambda")


@pytest.fixture(scope="module")
def ectx():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emul"), "libvdo_emul.so"], stdout=subprocess.DEVNULL)
    return capi.Context(0, lib_path=EMUL)


def _pcg_graphs():
    return [
        make_batch_graph(n_frames=10, n_objects=2, n_static=150, n_dynamic=60, seed=5),
        make_batch_graph(n_frames=14, n_objects=1, n_static=300, n_dynamic=120, seed=1),
        make_batch_graph(n_frames=8, n_objects=1, n_static=80, n_dynamic=30, seed=11, odo_sigma_t=0.5, odo_sigma_r=0.2),
        ba_shapes.SHAPES["chains_short"]()[0],
    ]


def _run(ctx, gs, batched, **kw):
    Gs = [capi.BatchGraph(ctx, g) for g in gs]
    rs = capi.optimize_batch(Gs, **kw) if batched else [G.optimize(**kw) for G in Gs]
    return rs, [G.vertices() for G in Gs], Gs


def _same(ra, rb, ea, eb, what):
    for k in PER_GRAPH:
        assert ra[k] == rb[k], f"{what}: {k}"
    assert np.array_equal(ra["chi2"], rb["chi2"]), what
    assert np.array_equal(ea[0], eb[0]) and np.array_equal(ea[1], eb[1]), what


@pytest.mark.parametrize("kw", [dict(max_iterations=30, gain_threshold=1e-4),
                                dict(max_iterations=6, gain_threshold=1e-4, pcg_max_iterations=20),   # PCG stopped by its cap, mid-chunk
                                dict(max_iterations=5, gain_threshold=1e-4, force_all_iterations=True, pcg_rel_tol=1e-9)])
def test_pcg_batch_equals_separate_bit_for_bit(ectx, kw):
    gs = _pcg_graphs()
    r0, e0, Gs = _run(ectx, gs, False, **kw)
    assert all(G.solver_info()["tiled"] == 1 and G.solver_info()["dense"] == 0 for G in Gs)
    if "pcg_max_iterations" not in kw:
        assert len({r["pcg_iterations"] for r in r0}) >= 3, "the graphs should need different numbers of PCG iterations"
    r1, e1, _ = _run(ectx, gs, True, **kw)
    for i in range(len(gs)):
        _same(r1[i], r0[i], e1[i], e0[i], f"graph {i}")


def test_pcg_batch_with_dense_and_chunked_graphs(ectx, monkeypatch):
    """two PCG graphs batched, next to two dense graphs (batched among themselves) and a chunked-layout graph (run on its own)"""
    gs = _pcg_graphs()[:2]
    dense = [make_batch_graph(n_frames=20, n_objects=0, n_static=n, n_dynamic=0, seed=s, consts=PARTIAL_BATCH) for s, n in ((3, 300), (4, 200))]
    kw = dict(max_iterations=25, gain_threshold=1e-4)
    chunk_g = make_batch_graph(n_frames=9, n_objects=1, n_static=120, n_dynamic=40, seed=21)
    monkeypatch.setenv("VDO_BA_LAYOUT", "chunked")
    Gc = capi.BatchGraph(ectx, chunk_g)
    rc0 = capi.BatchGraph(ectx, chunk_g).optimize(**kw)
    monkeypatch.delenv("VDO_BA_LAYOUT")
    assert Gc.solver_info()["tiled"] == 0
    ref = [_run(ectx, [g], False, **kw) for g in (gs[0], dense[0], gs[1], dense[1])]
    Gs = [capi.BatchGraph(ectx, g) for g in (gs[0], dense[0], gs[1], dense[1])] + [Gc]
    rs = capi.optimize_batch(Gs, **kw)
    for i in range(4):
        _same(rs[i], ref[i][0][0], Gs[i].vertices(), ref[i][1][0], f"graph {i}")
    for k in PER_GRAPH:
        assert rs[4][k] == rc0[k]
