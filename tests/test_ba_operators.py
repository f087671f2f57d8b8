"""Operator-level tests of the batch solver against a float64 reference (tests/ba_reference.py) on graphs built to reach the kernels'
boundaries (tests/ba_shapes.py): the reduced-matrix product S p, the preconditioner z = M^-1 r, the right-hand side, the back-substitution
and one whole linear solve, each through the test hooks vdo_graph_debug_apply / vdo_graph_debug_solve, at the LM's initial damping and at
one 1e4 times larger, under every layout switch that applies to the shape.

The same tests run on the serial emulation of the kernels (tests/emul, without a GPU) and on the CUDA backend (marked gpu).

Tolerances are relative to the magnitude of the sum each operator forms (the same expression in absolute values):
  S p                 |S p - S_ref p|                       <= 1e-11 * max(|H_pp + lam I| |p| + |H_pl| |(H_ll + lam I)^-1| |H_lp| |p|)
  M^-1 r              |M_ref z - r|                         <= 1e-10 * max(|M_ref| |z|)                 (backward error)
  rhs, back-subst.    |y - y_ref|                           <= 1e-11 * max(magnitude of y_ref's sum)
  solve (PCG)         |(rhs_ref - S_ref x_p) - r_recurrence| <= 1e-10 * max(|S_ref| |x_p| + |rhs_ref|)
  solve (dense)       |rhs_ref - S_ref x_p|                 <= 1e-9 * max(|S_ref| |x_p| + |rhs_ref|)
"""
import os
import subprocess
import zlib

import numpy as np
import pytest

from vdo_slam_b200 import capi
from tests.ba_reference import Reference
from tests.ba_shapes import SHAPES, REFUSED

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tests", "emul", "libvdo_emul.so")

TOL_S, TOL_MINV, TOL_RHS, TOL_BACKSUB, TOL_PCG_RES, TOL_DENSE = 1e-11, 1e-10, 1e-11, 1e-11, 1e-10, 1e-9
LAYOUTS = {"default": {}, "no_band": {"VDO_BA_BAND": "0"}, "chunked": {"VDO_BA_LAYOUT": "chunked"}, "no_dense": {"VDO_BA_DENSE": "0"}}
BACKENDS = ["emul", pytest.param("cuda", marks=pytest.mark.gpu)]

_ctx, _graphs, _refs, _info = {}, {}, {}, {}


@pytest.fixture(scope="module", params=BACKENDS)
def backend(request):
    if request.param not in _ctx:
        if request.param == "emul":
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emul"), "libvdo_emul.so"], stdout=subprocess.DEVNULL)
            _ctx["emul"] = capi.Context(0, lib_path=EMUL)
        else:
            _ctx["cuda"] = capi.Context(0)
    return request.param, _ctx[request.param]


def shape(name):
    if name not in _graphs:
        _graphs[name] = SHAPES[name]()
    return _graphs[name]


def reference(name):
    if name not in _refs:
        _refs[name] = Reference(shape(name)[0])
    return _refs[name]


def build(ctx, g, monkeypatch, layout):
    for k, v in LAYOUTS[layout].items():
        monkeypatch.setenv(k, v)
    G = capi.BatchGraph(ctx, g)
    for k in LAYOUTS[layout]:
        monkeypatch.delenv(k)
    return G


def default_info(be, ctx, name, monkeypatch):
    if (be, name) not in _info:
        _info[(be, name)] = build(ctx, shape(name)[0], monkeypatch, "default").solver_info()
    return _info[(be, name)]


def rel(err, mag):
    return float(np.abs(err).max() / max(np.abs(mag).max(), 1e-300))


def skip_unless_layout_applies(info, layout):
    """A layout switch is tested only on shapes whose default layout it changes."""
    if layout == "no_band" and info["band_width"] == 0:
        pytest.skip("the default layout has no band")
    if layout == "no_dense" and info["dense"] == 0:
        pytest.skip("the default layout has no dense path")
    if layout == "chunked" and info["tiled"] == 0:
        pytest.skip("the default layout is already chunked")


@pytest.mark.parametrize("name", list(SHAPES))
def test_shape_reaches_its_boundary(backend, name, monkeypatch):
    """Each shape lands on the solver path it was built for (tile counts, chunked fallback, band width, dense path)."""
    be, ctx = backend
    info = default_info(be, ctx, name, monkeypatch)
    for k, v in shape(name)[1].items():
        if k == "dense" and be == "emul":
            continue                      # the emulation has no dense path
        assert info[k] == v, f"{name}: solver_info()[{k!r}] = {info[k]}, expected {v} ({info})"


@pytest.mark.parametrize("name", list(REFUSED))
def test_more_than_256_edge_classes_are_refused(backend, name):
    be, ctx = backend
    with pytest.raises(capi.VdoError, match="failed with -3"):
        capi.BatchGraph(ctx, REFUSED[name]())


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("name", list(SHAPES))
def test_operators_match_float64_reference(backend, name, layout, monkeypatch):
    be, ctx = backend
    skip_unless_layout_applies(default_info(be, ctx, name, monkeypatch), layout)
    g = shape(name)[0]
    ref = reference(name)
    G = build(ctx, g, monkeypatch, layout)
    si = G.solver_info()
    rng = np.random.default_rng(zlib.crc32(f"{name}/{layout}".encode()))
    C = ref.C
    for lam in ref.lambdas():
        S, Sabs = ref.S(lam)
        M = ref.M(lam)
        for _ in range(3):
            p = rng.standard_normal(6 * C)
            y = G.debug_apply(lam, "S", p).ravel()
            e = rel(y - S @ p, Sabs @ np.abs(p))
            assert e <= TOL_S, f"S p on {name}/{layout}, lambda={lam:.3g}: relative error {e:.3g}"
        r = rng.standard_normal(6 * C)
        z = G.debug_apply(lam, "Minv", r).ravel()
        e = rel(M @ z - r, np.abs(M) @ np.abs(z))
        assert e <= TOL_MINV, f"M^-1 r on {name}/{layout}, lambda={lam:.3g}: backward error {e:.3g}"
        b_ref, b_mag = ref.rhs(lam)
        e = rel(G.debug_apply(lam, "rhs").ravel() - b_ref, b_mag)
        assert e <= TOL_RHS, f"rhs on {name}/{layout}, lambda={lam:.3g}: relative error {e:.3g}"
        xp = rng.standard_normal(6 * C)
        xl_ref, xl_mag = ref.backsub(lam, xp)
        e = rel(G.debug_apply(lam, "backsub", xp).ravel() - xl_ref, xl_mag)
        assert e <= TOL_BACKSUB, f"back-substitution on {name}/{layout}, lambda={lam:.3g}: relative error {e:.3g}"
        # one whole solve as an LM trial runs it (the captured PCG iteration, or the dense Cholesky)
        sol = G.debug_solve(lam, pcg_rel_tol=1e-12, pcg_max_iterations=4000)
        x = sol["xp"].ravel()
        r_true = b_ref - S @ x
        mag = Sabs @ np.abs(x) + np.abs(b_ref)
        if si["dense"]:
            e = rel(r_true, mag)
            assert sol["pcg_iterations"] == 0 and e <= TOL_DENSE, f"dense solve on {name}/{layout}, lambda={lam:.3g}: backward error {e:.3g}"
        else:
            e = rel(r_true - sol["r"].ravel(), mag)
            assert e <= TOL_PCG_RES, f"PCG on {name}/{layout}, lambda={lam:.3g}: true vs recurrence residual {e:.3g} after {sol['pcg_iterations']} iterations"
            assert sol["pcg_iterations"] < 4000
        xl_ref, xl_mag = ref.backsub(lam, x)
        e = rel(sol["xl"].ravel() - xl_ref, xl_mag)
        assert e <= TOL_BACKSUB, f"x_l of the solve on {name}/{layout}, lambda={lam:.3g}: relative error {e:.3g}"


def test_products_at_a_repeated_lambda_after_relinearising(backend):
    """Regression: every linearisation used to zero all device scalars, including the damping the S p kernels read, while the CUDA
    backend re-sends the damping only when it changes -- a second solve (or product) at the previous lambda then multiplied by
    H_pp + 0 I.  Each hook call re-linearises, so the same product twice must agree with the reference both times."""
    be, ctx = backend
    ref = reference("static_odd")
    G = capi.BatchGraph(ctx, shape("static_odd")[0])
    lam = ref.lambdas()[1]
    S, Sabs = ref.S(lam)
    p = np.random.default_rng(3).standard_normal(6 * ref.C)
    for _ in range(2):
        e = rel(G.debug_apply(lam, "S", p).ravel() - S @ p, Sabs @ np.abs(p))
        assert e <= TOL_S, f"S p at a repeated lambda: relative error {e:.3g}"


def test_hooks_leave_the_lm_run_unchanged(backend, monkeypatch):
    """optimize() after the hooks gives the run it gives without them: bit for bit on the emulation; on the GPU to the 1e-9 by which two
    runs differ anyway (fp64 atomics sum in varying order)."""
    be, ctx = backend
    g = shape("chains_short")[0]
    runs = []
    for hooks in (False, True):
        G = capi.BatchGraph(ctx, g)
        if hooks:
            lam = reference("chains_short").lambdas()[1]
            x = np.ones(6 * G.n_se3)
            for op in ("S", "Minv", "rhs", "backsub"):
                G.debug_apply(lam, op, x)
            G.debug_solve(lam, 1e-12)
            G.debug_trial(lam, reortho=True)
        r = G.optimize(max_iterations=10, gain_threshold=0.0)
        runs.append((r, *G.vertices()))
    (ra, sa, pa), (rb, sb, pb) = runs
    assert ra["iterations"] == rb["iterations"] and ra["trials"] == rb["trials"]
    if be == "emul":
        assert ra["pcg_iterations"] == rb["pcg_iterations"]
        assert np.array_equal(ra["chi2"], rb["chi2"]) and np.array_equal(sa, sb) and np.array_equal(pa, pb)
    else:
        np.testing.assert_allclose(ra["chi2"], rb["chi2"], rtol=1e-9)
        assert np.abs(sa - sb).max() <= 1e-9 and np.abs(pa - pb).max() <= 1e-9
