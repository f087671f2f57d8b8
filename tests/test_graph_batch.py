"""vdo_graph_optimize_batch on the serial kernel emulation (tests/emul): the round-based LM driver must give every graph exactly
what its own vdo_graph_optimize gives, whatever the other graphs in the batch do.  The emulation is serial, so the results are
compared bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_batch_graph, PARTIAL_BATCH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tests", "emul", "libvdo_emul.so")
# every field of vdo_lm_stats that describes one graph (ms_* and kernel_launches describe the whole call)
PER_GRAPH = ("iterations", "trials", "pcg_iterations", "initial_chi2", "final_chi2", "final_lambda")


@pytest.fixture(scope="module")
def ectx():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emul"), "libvdo_emul.so"], stdout=subprocess.DEVNULL)
    return capi.Context(0, lib_path=EMUL)


def _graphs():
    return [
        make_batch_graph(n_frames=20, n_objects=0, n_static=400, n_dynamic=0, seed=3, consts=PARTIAL_BATCH),
        make_batch_graph(n_frames=10, n_objects=2, n_static=150, n_dynamic=60, seed=5),
        make_batch_graph(n_frames=6, n_objects=0, n_static=40, n_dynamic=0, seed=8),
        make_batch_graph(n_frames=14, n_objects=1, n_static=300, n_dynamic=120, seed=1),
        # large odometry noise: the first trials overshoot and are rejected
        make_batch_graph(n_frames=8, n_objects=1, n_static=80, n_dynamic=30, seed=11, odo_sigma_t=0.5, odo_sigma_r=0.2),
    ]


def _same(ra, rb):
    for k in PER_GRAPH:
        assert ra[k] == rb[k] or (np.isnan(ra[k]) and np.isnan(rb[k])), k
    assert np.array_equal(ra["chi2"], rb["chi2"])


def _separate(ctx, gs, **kw):
    out = []
    for g in gs:
        G = capi.BatchGraph(ctx, g)
        out.append((G.optimize(**kw), G.vertices()))
    return out


@pytest.mark.parametrize("kw", [dict(max_iterations=40, gain_threshold=1e-4), dict(max_iterations=7, gain_threshold=1e-4, force_all_iterations=True)])
def test_batch_equals_separate_bit_for_bit(ectx, kw):
    gs = _graphs()
    ref = _separate(ectx, gs, **kw)
    Gs = [capi.BatchGraph(ectx, g) for g in gs]
    rs = capi.optimize_batch(Gs, **kw)
    assert len(rs) == len(gs)
    for (r0, (se3_0, pt_0)), r, G in zip(ref, rs, Gs):
        _same(r0, r)
        se3, pt = G.vertices()
        assert np.array_equal(se3, se3_0) and np.array_equal(pt, pt_0)
    # every entry reports the whole call
    assert len({r["kernel_launches"] for r in rs}) == 1 and len({r["ms_total"] for r in rs}) == 1
    assert rs[0]["kernel_launches"] >= max(r0["kernel_launches"] for r0, _ in ref)
    if not kw.get("force_all_iterations"):
        assert len({r0["iterations"] for r0, _ in ref}) >= 3, "the graphs should stop at different iterations"
        assert any(r0["trials"] > r0["iterations"] for r0, _ in ref), "at least one graph should reject a trial"
    else:
        assert all(r0["iterations"] == 7 for r0, _ in ref)


def test_order_and_batch_of_one(ectx):
    gs = _graphs()[:4]
    kw = dict(max_iterations=30, gain_threshold=1e-4)
    Gs = [capi.BatchGraph(ectx, g) for g in gs]
    rs = capi.optimize_batch(Gs, **kw)
    est = [G.vertices() for G in Gs]
    perm = [2, 0, 3, 1]
    Hs = [capi.BatchGraph(ectx, gs[i]) for i in perm]
    rp = capi.optimize_batch(Hs, **kw)
    for j, i in enumerate(perm):
        _same(rs[i], rp[j])
        se3, pt = Hs[j].vertices()
        assert np.array_equal(se3, est[i][0]) and np.array_equal(pt, est[i][1])
    # n = 1 is optimize()
    A, B = capi.BatchGraph(ectx, gs[1]), capi.BatchGraph(ectx, gs[1])
    ra, (rb,) = A.optimize(**kw), capi.optimize_batch([B], **kw)
    _same(ra, rb)
    assert ra["kernel_launches"] == rb["kernel_launches"]
    assert all(np.array_equal(x, y) for x, y in zip(A.vertices(), B.vertices()))


def test_refusals_change_nothing(ectx):
    L = ectx.L
    gs = _graphs()[:2]
    Gs = [capi.BatchGraph(ectx, g) for g in gs]
    before = [G.vertices() for G in Gs]
    raw = C.c_void_p()                                   # created but never finalized
    ectx.check(L.vdo_graph_create(ectx.h, C.byref(raw)), "vdo_graph_create")
    try:
        o = capi.LMOptions()
        L.vdo_lm_options_default(C.byref(o))

        def call(handles, n=None):
            arr = (C.c_void_p * max(len(handles), 1))(*handles)
            return L.vdo_graph_optimize_batch(arr, C.c_int(len(handles) if n is None else n), C.byref(o), None, None)

        h0, h1 = Gs[0].h.value, Gs[1].h.value
        assert call([h0, h1, h0]) == -2                  # VDO_ERR_ARG: repeated graph
        assert b"repeats" in L.vdo_last_error(ectx.h)
        assert call([h0, None, h1]) == -2                # NULL entry
        assert call([h0, h1], n=0) == -2                 # n < 1
        assert L.vdo_graph_optimize_batch(None, C.c_int(2), C.byref(o), None, None) == -2
        assert call([h0, raw.value, h1]) == -4           # VDO_ERR_STATE: not finalized
        with pytest.raises(capi.VdoError):
            capi.optimize_batch([Gs[0], Gs[0]])
        with pytest.raises(capi.VdoError):
            capi.optimize_batch([])
    finally:
        L.vdo_graph_destroy(raw)
    for G, (se3, pt) in zip(Gs, before):
        a, b = G.vertices()
        assert np.array_equal(a, se3) and np.array_equal(b, pt)
    # the graphs still optimise normally afterwards
    rs = capi.optimize_batch(Gs, max_iterations=5)
    assert all(r["iterations"] >= 1 for r in rs)
