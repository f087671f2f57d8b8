"""Tests of the batch solver's linearisation and of whole LM trials against a float64 reference (tests/ba_reference.py), on the boundary
graphs of tests/ba_shapes.py under every layout switch that applies, for a lone graph and for batches that share launches.

A trial runs through the test hook vdo_graph_debug_trial (capi.debug_trial): linearisation, solve, back-substitution, update and the
robust chi2 of the updated estimates, exactly as optimize_batch takes one trial, then the estimates are restored.  Each stage is checked
against the reference built at the estimates the trial starts from:
  H_pp diagonal blocks  |H_ij - ref|          <= 1e-12 sqrt(H_ii H_jj)     (Cauchy-Schwarz: H = J^T W J with positive Huber weights)
  b (se3 and points)    |b_i - ref|           <= 1e-12 sqrt(H_ii chi2)
  H_ll diagonal         |hll_k - H[3k,3k]|    <= 1e-12 H[3k,3k]            (exactly 0 for a landmark without edges)
  chi2 (linearisation)  |chi2 - ref|          <= 1e-12 chi2
  step x_p              |rhs_ref - S_ref x_p| <= 1e-9 max(|S_ref| |x_p| + |rhs_ref|)   (the true residual; both solvers)
  step x_l              |x_l - backsub_ref(x_p)| <= 1e-11 max(its magnitude)
  update                points bit for bit pt + x_l; se3 within 1e-14 (1 + |t|) of iso_oplus(T, x_p), re-orthogonalised when asked
  chi2 (trial)          |chi2 - ref|          <= 1e-12 ref, the reference evaluated at the trial's own updated estimates
  scale                 |sum x (lam x + b) - ref| <= 1e-12 sum |x| (lam |x| + |b|)
Batches give every graph its own damping and re-orthogonalise every other graph; each graph must meet the bounds above and agree with
its lone trial to 1e-9 (the GPU sums with fp64 atomics in varying order).  Five-iteration LM runs at pcg_rel_tol 1e-12 follow the oracle's
LM: equal iteration and trial counts, chi2 history at rtol 1e-9, estimates within 1e-9.

The same tests run on the serial emulation of the kernels (tests/emul, without a GPU; about 1.5 minutes of CPU time, most of it in the
emulated LM runs on the long chains) and on the CUDA backend (marked gpu; under a minute on an H100).  Run with -s to see the worst
error of each check and where it occurred.
"""
import numpy as np
import pytest

from oracle import pyoracle as po
from vdo_slam_b200 import capi
from tests.ba_reference import Reference, robust_chi2, reorthogonalize
from tests.ba_shapes import (SHAPES, band, chains, dense, motion_runs, off_orthonormal, push_off_orthonormal, static_odd, static_tile_fill,
                             vertex_runs)
from tests.test_ba_operators import LAYOUTS, backend, build, default_info, reference, shape, skip_unless_layout_applies  # noqa: F401

TOL_LIN, TOL_STEP, TOL_XL, TOL_SE3, TOL_CHI2, TOL_SCALE, TOL_BATCH, TOL_LM = 1e-12, 1e-9, 1e-11, 1e-14, 1e-12, 1e-12, 1e-9, 1e-9
LM = dict(max_iterations=5, gain_threshold=0.0, pcg_rel_tol=1e-12, pcg_max_iterations=4000)

WORST = {}          # (backend, check) -> (worst error over the run in units of the check's magnitude, where)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for (be, what), (e, where) in sorted(WORST.items()):
        print(f"[test_ba_trial] {be:5s} {what:24s} worst {e:.3g}  ({where})")


def check(be, what, err, mag, tol, where):
    """max |err| / mag over the entries (mag > 0) must be <= tol; where mag == 0 the error must be exactly 0."""
    err = np.abs(np.asarray(err, np.float64))
    mag = np.broadcast_to(np.abs(np.asarray(mag, np.float64)), err.shape).ravel()
    err = err.ravel()
    zero = mag == 0
    assert not err[zero].any(), f"{what} on {where}: {int((err[zero] != 0).sum())} entries differ where the reference is exactly 0"
    e = float((err[~zero] / mag[~zero]).max()) if (~zero).any() else 0.0
    if e >= WORST.get((be, what), (0.0, ""))[0]:
        WORST[(be, what)] = (e, where)
    assert e <= tol, f"{what} on {where}: error {e:.3g} of its magnitude (bound {tol:g})"
    return e


def check_linearisation(be, G, ref, where):
    Hpp, bp, Hll, bl, chi2 = G.debug_linearize()
    C = ref.C
    blocks = ref.Hpp.reshape(C, 6, C, 6)[np.arange(C), :, np.arange(C), :]
    dp = np.diagonal(ref.Hpp).reshape(C, 6)
    dl = ref.Hll.diagonal()
    check(be, "H_pp blocks", Hpp - blocks, np.sqrt(dp[:, :, None] * dp[:, None, :]), TOL_LIN, where)
    check(be, "b_p", bp.ravel() - ref.bp, np.sqrt(dp.ravel() * ref.chi2), TOL_LIN, where)
    check(be, "b_l", bl.ravel() - ref.bl, np.sqrt(dl * ref.chi2), TOL_LIN, where)
    check(be, "hll", Hll - dl[0::3], dl[0::3], TOL_LIN, where)
    check(be, "chi2 (linearisation)", chi2 - ref.chi2, ref.chi2, TOL_LIN, where)


def oplus_reference(g, xp, rt):
    T = np.array([po.iso_oplus(g["se3"][v], xp[v]) for v in range(len(xp))]).reshape(-1, 12)
    if rt:
        T[:, :9] = reorthogonalize(T[:, :9].reshape(-1, 3, 3)).reshape(-1, 9)
    return T


def check_update(be, g, rt, out, where):
    """The trial's estimates are the oplus of its own step onto the estimates it started from."""
    assert np.array_equal(out["pt"], g["pt"] + out["xl"]), f"points of the update on {where} are not pt + x_l bit for bit"
    T = oplus_reference(g, out["xp"], rt)
    check(be, "se3 update", out["se3"] - T, 1.0 + np.linalg.norm(T[:, 9:], axis=1)[:, None], TOL_SE3, where)


def check_trial(be, g, ref, lam, rt, out, where):
    """Every stage of one trial of graph g (estimates as given to the graph) at damping lam against the reference."""
    where = f"{where}, lambda={lam:.3g}{', reortho' if rt else ''}"
    assert out["ok"], f"the solve broke down on {where}"
    xp, xl = out["xp"].ravel(), out["xl"].ravel()
    S, Sabs = ref.S(lam)
    b_ref, _ = ref.rhs(lam)
    check(be, "step x_p (true residual)", np.abs(b_ref - S @ xp).max(), (Sabs @ np.abs(xp) + np.abs(b_ref)).max(), TOL_STEP, where)
    xl_ref, xl_mag = ref.backsub(lam, xp)
    check(be, "step x_l", np.abs(xl - xl_ref).max(), xl_mag.max(), TOL_XL, where)
    check_update(be, g, rt, out, where)
    chi_ref = robust_chi2(g, out["se3"], out["pt"])
    check(be, "chi2 (trial)", out["chi2"] - chi_ref, chi_ref, TOL_CHI2, where)
    s_ref, s_mag = ref.scale(lam, xp, xl)
    check(be, "scale", out["scale"] - s_ref, s_mag, TOL_SCALE, where)


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("name", list(SHAPES))
def test_linearisation_matches_float64_reference(backend, name, layout, monkeypatch):
    be, ctx = backend
    skip_unless_layout_applies(default_info(be, ctx, name, monkeypatch), layout)
    G = build(ctx, shape(name)[0], monkeypatch, layout)
    check_linearisation(be, G, reference(name), f"{name}/{layout}")


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("name", list(SHAPES))
def test_trial_matches_float64_reference(backend, name, layout, monkeypatch):
    be, ctx = backend
    skip_unless_layout_applies(default_info(be, ctx, name, monkeypatch), layout)
    g = shape(name)[0]
    ref = reference(name)
    G = build(ctx, g, monkeypatch, layout)
    for lam in ref.lambdas():
        out = G.debug_trial(lam)
        check_trial(be, g, ref, lam, False, out, f"{name}/{layout}")
        se3, pt = G.vertices()
        assert np.array_equal(se3, g["se3"]) and np.array_equal(pt, g["pt"]), "debug_trial did not restore the estimates"


def test_trial_reorthogonalises_the_rotations(backend):
    """Rotations ~1e-7 off orthonormal: with the flag the update ends at R - R (R^T R - I) / 2 of the oplus result; without it the
    result stays ~1e-7 away from that, so the check sees the re-orthogonalisation.  Only the update is compared: the kernels'
    linearisation follows the oracle's for orthonormal rotations only (on this graph their steps differ by ~1e-6 relative)."""
    be, ctx = backend
    g = off_orthonormal()
    G = capi.BatchGraph(ctx, g)
    lam = Reference(g).lambdas()[0]
    on = G.debug_trial(lam, reortho=True)
    check_update(be, g, True, on, "off_orthonormal, reortho")
    off = G.debug_trial(lam, reortho=False)
    check_update(be, g, False, off, "off_orthonormal")
    assert np.abs(off["se3"] - oplus_reference(g, off["xp"], True)).max() > 1e-9, "the re-orthogonalisation is not visible on this graph"


def _small(k, n):
    """Graph k of a batch of n: the small builders in turn, each with its own seed (no two graphs alike).  Every third graph, and the last
    two, get rotations off orthonormal (push_off_orthonormal): dense-path (static_odd) and PCG-path (motion_runs) graphs throughout the
    tables, with and without the re-orthogonalisation, and in the 65- and 130-graph batches on both sides of a 64-graph parameter chunk
    boundary of the launch tables (the dense graphs come first there).  The label names the graph: equal labels, equal graphs."""
    seed = 1000 + k
    g = [lambda: chains([2, 5], n_cam=8, seed=seed), lambda: static_odd(seed), lambda: vertex_runs([15, 16], seed),
         lambda: motion_runs([3, 4], seed), lambda: band(4, n_cam=32, seed=seed), lambda: dense(8, seed)][k % 6]()
    if k % 3 == 1 or k >= n - 2:
        return f"small/{k}/off", push_off_orthonormal(g, seed), "default", True
    return f"small/{k}", g, "default", False


def _batch(kind):
    """(label, graph, layout, rotations off orthonormal) of each graph of a batch composition."""
    if kind == "all_shapes":
        return [(n, shape(n)[0], "default", False) for n in SHAPES]
    if kind == "static_between_chains":
        # static-only graphs first, between and last among chain-only graphs: the tables of the chain tiles hold empty ranges at both ends
        # and in the middle (and those of the static tiles around the chain graphs).  no_dense keeps the static graphs on the PCG tables.
        st = [(f"static_tile_fill/{s}", static_tile_fill(s), "no_dense", False) for s in (2, 13, 14)]
        ch = [(n, shape(n)[0], "default", False) for n in ("chain_256", "motion_runs")]
        return [st[0], ch[0], st[1], ch[1], st[2]]
    if kind == "dense_and_paths":
        return [(n, shape(n)[0], "default", False) for n in ("dense_162", "dense_168", "precond_paths")]
    n = int(kind[1:])
    return [_small(k, n) for k in range(n)]


_refs_by_label = {}       # the graphs of _batch that are not in SHAPES (the same label is the same graph)


@pytest.mark.parametrize("kind", ["all_shapes", "static_between_chains", "dense_and_paths", "n64", "n65", "n130"])
def test_batched_trials_match_reference_and_lone_trials(backend, kind, monkeypatch):
    """One call for a whole batch (the CUDA backend shares launches through its launch tables, past 64 graphs in several parameter
    chunks); every graph at its own damping, re-orthogonalising every other graph.  Graphs with rotations off orthonormal show whether
    their own flag was applied; their steps do not follow the oracle's (see the lone test above), so only their update is compared."""
    be, ctx = backend
    items = _batch(kind)
    Gs = [build(ctx, g, monkeypatch, layout) for _, g, layout, _ in items]
    refs = []
    for label, g, _, _ in items:
        if label in SHAPES:
            refs.append(reference(label))
        else:
            if label not in _refs_by_label:
                _refs_by_label[label] = Reference(g)
            refs.append(_refs_by_label[label])
    lams = [refs[k].lambdas()[k % 2] * (1 + k / 64) for k in range(len(items))]
    rts = [k % 2 == 1 for k in range(len(items))]
    outs = capi.debug_trial(Gs, lams, rts)
    for k, ((label, g, layout, off), G, ref, out) in enumerate(zip(items, Gs, refs, outs)):
        where = f"graph {k} ({label}/{layout}) of {kind}"
        if off:
            check_update(be, g, rts[k], out, f"{where}{', reortho' if rts[k] else ''}")
            assert np.abs(out["se3"] - oplus_reference(g, out["xp"], not rts[k])).max() > 1e-9, \
                f"{where}: the update is as close to the {'plain' if rts[k] else 're-orthogonalised'} oplus as to its own"
        else:
            check_trial(be, g, ref, lams[k], rts[k], out, where)
        lone = G.debug_trial(lams[k], rts[k])
        for f in ("xp", "xl", "se3", "pt"):
            check(be, "batch vs lone", np.abs(out[f] - lone[f]).max(), max(np.abs(lone[f]).max(), 1.0), TOL_BATCH, f"{where}: {f}")
        check(be, "batch vs lone", out["chi2"] - lone["chi2"], lone["chi2"], TOL_BATCH, f"{where}: chi2")
        check(be, "batch vs lone", out["scale"] - lone["scale"], max(abs(lone["scale"]), 1e-300), TOL_BATCH, f"{where}: scale")


def test_debug_trial_refuses_what_optimize_batch_refuses(backend):
    be, ctx = backend
    g = shape("chains_short")[0]
    G, H = capi.BatchGraph(ctx, g), capi.BatchGraph(ctx, g)
    with pytest.raises(capi.VdoError, match="repeats graph"):
        capi.debug_trial([G, H, G], [1.0, 1.0, 1.0])
    with pytest.raises(capi.VdoError, match="negative or NaN"):
        capi.debug_trial([G, H], [1.0, -1.0])
    with pytest.raises(capi.VdoError, match="negative or NaN"):
        G.debug_trial(float("nan"))
    other = capi.Context(0, lib_path=ctx.L._name)
    X = capi.BatchGraph(other, g)
    with pytest.raises(capi.VdoError, match="another context"):
        capi.debug_trial([G, X], [1.0, 1.0])
    se3, pt = G.vertices()
    assert np.array_equal(se3, g["se3"]) and np.array_equal(pt, g["pt"])


_oracle_lm = {}


def oracle_lm(name):
    if name not in _oracle_lm:
        _oracle_lm[name] = po.ba_optimize(shape(name)[0], max_iters=LM["max_iterations"], gain_threshold=0.0)
    return _oracle_lm[name]


def check_lm(name, r, se3, pt):
    o = oracle_lm(name)
    assert r["iterations"] == o["iters"] and r["trials"] == o["stats"]["trials"], \
        f"{name}: {r['iterations']} iterations / {r['trials']} trials, the oracle {o['iters']} / {o['stats']['trials']}"
    np.testing.assert_allclose(r["chi2"], o["chi2"], rtol=TOL_LM, err_msg=f"{name}: chi2 history")
    assert np.abs(se3 - o["se3"]).max() <= TOL_LM and np.abs(pt - o["pt"]).max() <= TOL_LM, \
        f"{name}: estimates differ from the oracle's by {max(np.abs(se3 - o['se3']).max(), np.abs(pt - o['pt']).max()):.3g}"


@pytest.mark.parametrize("name", list(SHAPES))
def test_lm_run_matches_oracle(backend, name):
    be, ctx = backend
    G = capi.BatchGraph(ctx, shape(name)[0])
    r = G.optimize(**LM)
    check_lm(name, r, *G.vertices())


def test_lm_batch_of_all_shapes_matches_oracle(backend):
    be, ctx = backend
    Gs = [capi.BatchGraph(ctx, shape(n)[0]) for n in SHAPES]
    rs = capi.optimize_batch(Gs, **LM)
    for n, G, r in zip(SHAPES, Gs, rs):
        check_lm(n, r, *G.vertices())
