"""The per-frame flow / pose LM (vdo_pose_opt_flow2*) at its kernels' boundaries, against a long-double numpy reference of its first
step (tests/flow_reference.py) and, trial by trial, against the CPU oracle (oracle/flow_lm.c) through the LM trace of
vdo_pose_opt_flow2_trace.

Sizes: n < 3 (nothing optimised), fewer points than the cluster's 8 CTAs (3, 7), empty or short CTAs (8, 9, 17), the first n at which
a cluster thread takes a second point (2049), the largest problem whose points fit the cluster's shared memory (11376) and the first
that does not (11377), and single-CTA problems (16385, 40000).  The single-CTA kernel is also run on small problems (3, 511, 512,
513, 2049) in a process of its own with VDO_FLOW_SINGLE_CTA=1.  Every size runs in both modes and both arithmetic modes (quirk),
each on a problem variant: a KITTI-like Tcw_last tens of metres from the origin, a 640x480 K, no outliers, 60 % outliers (most points
in the Huber branch), a large initial error (5 deg, 0.5 m).

Tolerances.  Operators, relative to the magnitude of each sum (the same sum over absolute values): H_pp, b_p, S, g <= 1e-12.  The
first step's backward error on the full damped system (quirk 0) or on S (quirk 1) <= 1e-10.  Trace against the oracle: the
accept / reject and ok2 sequences and the stop reason are identical, trial chi2 within rtol 1e-8, lambda within rtol 1e-6, then the
end state: T <= 1e-6, flow <= 1e-7, inliers exact, iterations and trials equal.  One exception: from the first trial at which the
oracle's |chi2 before - trial chi2| <= 1e-10 chi2 before + noise(chi2 before), summation order alone can flip a decision, so the
sequences are compared up to that trial and only the end-state tolerances are required after it.  noise(chi2) = 2 sqrt(0.1 n chi2) de
+ 0.1 n de^2 is what rounding the residuals (pixel differences of ~1e3 px, de = 1e-11 px, 50 ulps) does to a chi2; it is also added to
the trial chi2 tolerance.  It matters only near chi2 = 0: a problem that fits exactly (n = 3, quirk 0) goes down to chi2 ~ 1e-26, where
the trial chi2 values are rounding noise; at chi2 ~ 1e3 with n = 40000 it is 4e-11 of chi2.

A problem's result does not depend on the batch it runs in: a batch with problems on both kernels, run in two orders, equals each
problem run alone, bit for bit.  Malformed batches are refused before any device work.
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle import pyoracle as po
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_flow_problem, _rot
from tests.flow_reference import FlowStep

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SIZES = [2, 3, 7, 8, 9, 17, 2047, 2048, 2049, 11376, 11377, 16385, 40000]
SINGLE_CTA_SIZES = [3, 511, 512, 513, 2049]
MODES_QUIRKS = [(0, 0), (0, 1), (1, 0), (1, 1)]
VARIANTS = ("plain", "tcw_last", "vga_k", "no_outliers", "outliers_60", "large_init")
TOL_OP, TOL_BACKWARD, TOL_SCALE = 1e-12, 1e-10, 1e-10
TOL_CHI2, TOL_LAM, TOL_T, TOL_FLOW = 1e-8, 1e-6, 1e-6, 1e-7
TIE, RES_ROUNDING = 1e-10, 1e-11


def chi2_noise(chi2, n):
    """What rounding each of n residuals by RES_ROUNDING px does to a robust chi2 (weight 0.1) of that size."""
    return 2 * np.sqrt(0.1 * n * np.abs(chi2)) * RES_ROUNDING + 0.1 * n * RES_ROUNDING ** 2


def _kitti_like_tcw():
    """World -> last camera of a car 50 m from the origin, heading 35 deg off the world z axis, camera 1.65 m above the road."""
    Twc = np.eye(4)
    Twc[:3, :3] = _rot(np.array([0.0, 1.0, 0.0]), np.deg2rad(35.0))
    Twc[:3, 3] = (28.0, -1.65, 41.0)
    return np.linalg.inv(Twc).astype(np.float32)


TCW_KITTI = _kitti_like_tcw()
VGA_K = np.array([525.0, 525.0, 319.5, 239.5], np.float32)


def make_case(n, variant, seed):
    kw = {}
    if variant == "tcw_last":
        kw["Tcw_last"] = TCW_KITTI
    elif variant == "vga_k":
        kw.update(K=VGA_K, width=640, height=480)
    elif variant == "no_outliers":
        kw["outlier_frac"] = 0.0
    elif variant == "outliers_60":
        kw["outlier_frac"] = 0.6
    p = make_flow_problem(n=n, seed=seed, **kw)
    if variant == "large_init":          # 5 deg about a fixed axis and 0.5 m, in the last camera's frame
        ax = np.array([0.3, -0.8, 0.5]); ax /= np.linalg.norm(ax)
        dT = np.eye(4); dT[:3, :3] = _rot(ax, np.deg2rad(5.0)); dT[:3, 3] = 0.5 * np.array([0.6, 0.0, 0.8])
        Tl = p["Tcw_last"].astype(np.float64)
        p["T_init"] = (p["T_true"] @ np.linalg.inv(Tl) @ dT @ Tl).astype(np.float32)
    return p


_cache = {}


def _cached(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def boundary_problem(n, mode, quirk):
    i = SIZES.index(n)
    return _cached(("p", n, mode, quirk), lambda: make_case(n, VARIANTS[(i + 2 * mode + quirk) % 6], 1000 * (i + 1) + 2 * mode + quirk))


def single_cta_problem(n, mode, quirk):
    i = SINGLE_CTA_SIZES.index(n)
    return _cached(("s", n, mode, quirk), lambda: make_case(n, VARIANTS[(i + 2 * mode + quirk + 3) % 6], 50000 + 1000 * i + 2 * mode + quirk))


def oracle(kind, n, mode, quirk):
    p = boundary_problem(n, mode, quirk) if kind == "p" else single_cta_problem(n, mode, quirk)
    return _cached(("o", kind, n, mode, quirk), lambda: po.flow2(p, mode=mode, quirk=quirk, trace=True))


def rel(got, ref, mag):
    err = np.abs(np.asarray(got, np.longdouble) - ref)
    r = np.where(mag > 0, err / np.where(mag > 0, mag, 1), np.where(err > 0, np.inf, 0))
    return float(r.max())


def check_operators(tr, ref):
    """H_pp, b_p, S, g and the first step of one trace against the reference; returns the deviations."""
    dev = dict(Hpp=rel(tr["Hpp"], ref.Hpp, ref.Hpp_mag), bp=rel(tr["bp"], ref.bp, ref.bp_mag),
               S=rel(tr["S"], ref.S, ref.S_mag), g=rel(tr["g"], ref.g, ref.g_mag))
    rec0 = tr["rec"][0]
    dev["lam0"] = abs(rec0[1] - float(ref.lam)) / float(ref.lam)
    for k in ("Hpp", "bp", "S", "g", "lam0"):
        assert dev[k] <= TOL_OP, f"{k}: {dev[k]:.3e} > {TOL_OP}"
    if rec0[2]:
        dev["backward"] = ref.backward_error(tr["x"])
        assert dev["backward"] <= TOL_BACKWARD, f"backward error of the first step {dev['backward']:.3e} > {TOL_BACKWARD}"
        s, mag = ref.scale(tr["x"])
        dev["scale"] = abs(rec0[5] - s) / mag
        assert dev["scale"] <= TOL_SCALE, f"scale of the first trial {dev['scale']:.3e} > {TOL_SCALE}"
    else:                                # the solve failed: the matrix it reads is not positive definite
        Ssym = np.tril(ref.S) + np.tril(ref.S, -1).T
        with pytest.raises(np.linalg.LinAlgError):
            np.linalg.cholesky(Ssym.astype(np.float64))
    return dev


def compare_with_oracle(g, o, label):
    """Trace and end state of a GPU run against the oracle (see the module docstring); returns the deviations."""
    G, O = g["trace"]["rec"], o["trace"]["rec"]
    n = len(g["flow"])
    ties = np.nonzero(np.abs(O[:, 4] - O[:, 3]) <= TIE * np.abs(O[:, 4]) + chi2_noise(O[:, 4], n))[0]
    k = int(ties[0]) if len(ties) else len(O)
    assert len(G) >= k, f"{label}: the GPU ran {len(G)} trials, the oracle {len(O)} with no near tie before trial {k}"
    for col, name in ((0, "iteration"), (2, "ok2"), (7, "accepted")):
        bad = np.nonzero(G[:k, col] != O[:k, col])[0]
        assert not len(bad), f"{label}: {name} differs first at trial {bad[0]} (gpu {G[bad[0], col]}, oracle {O[bad[0], col]})"
    dev = dict(trials_compared=k, tie=int(ties[0]) if len(ties) else None)
    # deviation in units of the tolerance rtol |chi2| + noise(chi2), reported as the rtol it amounts to
    dev["chi2_trial"] = float((np.abs(G[:k, 3] - O[:k, 3]) / (np.abs(O[:k, 3]) + chi2_noise(O[:k, 3], n) / TOL_CHI2)).max()) if k else 0.0
    dev["lam"] = float((np.abs(G[:k, 1] - O[:k, 1]) / np.abs(O[:k, 1])).max()) if k else 0.0
    assert dev["chi2_trial"] <= TOL_CHI2, f"{label}: trial chi2 {dev['chi2_trial']:.3e} > {TOL_CHI2}"
    assert dev["lam"] <= TOL_LAM, f"{label}: lambda {dev['lam']:.3e} > {TOL_LAM}"
    if not len(ties):
        assert len(G) == len(O) and g["trace"]["stop"] == o["trace"]["stop"], \
            f"{label}: gpu {len(G)} trials, stop {g['trace']['stop']}; oracle {len(O)} trials, stop {o['trace']['stop']}"
        assert g["iters"] == o["iters"] and g["trials"] == o["trials"]
        assert abs(g["chi2"] - o["chi2"]) <= TOL_CHI2 * o["chi2"]
    dev["T"] = float(np.abs(g["T"] - o["T"]).max())
    dev["flow"] = float(np.abs(g["flow"] - o["flow"]).max())
    assert dev["T"] <= TOL_T, f"{label}: max |dT| {dev['T']:.3e} > {TOL_T}"
    assert dev["flow"] <= TOL_FLOW, f"{label}: max |dflow| {dev['flow']:.3e} > {TOL_FLOW}"
    assert np.array_equal(g["inlier"], o["inlier"]), f"{label}: {(g['inlier'] != o['inlier']).sum()} inlier flags differ"
    return dev


def check_few_points(g, o, p):
    assert g["iters"] == -1 and o["iters"] == -1
    assert np.array_equal(g["T"], np.eye(4, dtype=np.float32))
    assert np.array_equal(g["flow"], p["flow"].astype(np.float64)) and not g["inlier"].any()
    assert g["trace"]["stop"] == o["trace"]["stop"] == "few_points" and len(g["trace"]["rec"]) == 0


def report(label, dev):
    print(f"[flow-lm] {label} " + " ".join(f"{k}={v:.2e}" if isinstance(v, float) else f"{k}={v}" for k, v in dev.items()))


# ---- without a GPU: the oracle against the reference ----

@pytest.mark.parametrize("mode,quirk", MODES_QUIRKS)
@pytest.mark.parametrize("n", SIZES)
def test_oracle_first_step_matches_reference(n, mode, quirk):
    o = oracle("p", n, mode, quirk)
    if n < 3:
        assert o["iters"] == -1 and o["trace"]["stop"] == "few_points"
        return
    report(f"oracle n={n} mode={mode} quirk={quirk}", check_operators(o["trace"], FlowStep(boundary_problem(n, mode, quirk), mode, quirk)))


@pytest.mark.parametrize("n", [3, 17, 2049])
def test_reference_full_solve_agrees_with_its_elimination(n):
    """The reference's two routes to the first step agree: one sparse solve of the full quirk-0 system, and its own S, g."""
    ref = FlowStep(boundary_problem(n, 0, 0), 0, 0)
    x_full = ref.solve_full()
    x_schur = np.linalg.solve(ref.S.astype(np.float64), ref.g.astype(np.float64))
    assert ref.backward_error(x_full) <= TOL_BACKWARD and ref.backward_error(x_schur) <= TOL_BACKWARD
    assert np.abs(x_full - x_schur).max() <= 1e-8 * np.abs(x_full).max()


# ---- on the GPU ----

@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,quirk", MODES_QUIRKS)
@pytest.mark.parametrize("n", SIZES)
def test_gpu_first_step_and_trace(ctx, n, mode, quirk):
    p = boundary_problem(n, mode, quirk)
    g = capi.pose_opt_flow2(ctx, [p], quirk=quirk, modes=[mode], trace=True)[0]
    o = oracle("p", n, mode, quirk)
    if n < 3:
        check_few_points(g, o, p)
        return
    label = f"gpu n={n} mode={mode} quirk={quirk}"
    dev = check_operators(g["trace"], FlowStep(p, mode, quirk))
    dev.update(compare_with_oracle(g, o, label))
    report(label, dev)


@pytest.fixture(scope="module")
def single_cta_runs():
    cases = [(n, m, q) for n in SINGLE_CTA_SIZES for m, q in MODES_QUIRKS]
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "single_cta.npz")
        env = dict(os.environ, VDO_FLOW_SINGLE_CTA="1")
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_flow_single_cta_worker.py"), out] + [f"{n}:{m}:{q}" for n, m, q in cases],
                           env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        z = np.load(out)
        return {k: z[k] for k in z.files}


@pytest.mark.gpu
@pytest.mark.parametrize("mode,quirk", MODES_QUIRKS)
@pytest.mark.parametrize("n", SINGLE_CTA_SIZES)
def test_gpu_single_cta_kernel(single_cta_runs, n, mode, quirk):
    z, key = single_cta_runs, f"{n}_{mode}_{quirk}_"
    st = z[key + "stats"]
    rec = z[key + "trace_rec"].reshape(-1, 14)
    tr = {k: z[key + "trace_" + k] for k in ("Hpp", "bp", "S", "g", "x")}
    tr.update(rec=rec, stop=str(z[key + "trace_stop"]))
    g = dict(T=z[key + "T"], flow=z[key + "flow"], inlier=z[key + "inlier"], iters=int(st[0]), trials=int(st[1]), chi2=st[2], trace=tr)
    p = single_cta_problem(n, mode, quirk)
    label = f"single-CTA n={n} mode={mode} quirk={quirk}"
    dev = check_operators(tr, FlowStep(p, mode, quirk))
    dev.update(compare_with_oracle(g, oracle("s", n, mode, quirk), label))
    report(label, dev)


BATCH_SIZES = [0, 1, 2, 3, 9, 17, 150, 900, 2049, 3000, 5000, 11376, 11377, 12000, 16385, 700, 64, 8, 2, 40, 2500, 20000, 400, 1200]


@pytest.mark.gpu
@pytest.mark.parametrize("quirk", [1, 0])
def test_gpu_result_does_not_depend_on_the_batch(ctx, quirk):
    """Problems on both kernels, n of 0, 1 and 2, mixed modes, K and Tcw_last: each problem's T, flow, inliers and stats are the same
    bit for bit in two orders of one batch and alone."""
    probs = [make_case(n, VARIANTS[i % 6], 9000 + i) for i, n in enumerate(BATCH_SIZES)]
    modes = [(i // 3) % 2 for i in range(len(probs))]
    alone = [capi.pose_opt_flow2(ctx, [p], quirk=quirk, modes=[m])[0] for p, m in zip(probs, modes)]
    rng = np.random.default_rng(77)
    bad = []
    for order in (rng.permutation(len(probs)), rng.permutation(len(probs))):
        got = capi.pose_opt_flow2(ctx, [probs[j] for j in order], quirk=quirk, modes=[modes[j] for j in order])
        for g, j in zip(got, order):
            a = alone[j]
            diff = [k for k in ("T", "flow", "inlier", "stats") if not np.array_equal(g[k], a[k])]
            if diff:
                bad.append(f"n={BATCH_SIZES[j]}: {diff} (iterations batch {g['iters']} alone {a['iters']}, "
                           f"max |dT| {np.abs(g['T'] - a['T']).max():.2e})")
    assert not bad, f"{len(bad)} results depend on the batch: " + "; ".join(bad)


# ---- refusals (ctypes, before any device work) ----

def _call(ctx, mode, off, pts, depth, flow, K, Tl, Ti, T_out, flow_out, inl, stats):
    ptr = lambda a, ty: None if a is None else a.ctypes.data_as(C.POINTER(ty))
    f, d = C.c_float, C.c_double
    return ctx.L.vdo_pose_opt_flow2_batch(ctx.h, C.c_int(1), C.c_int(len(mode)), ptr(mode, C.c_int), ptr(off, C.c_int), ptr(pts, f),
                                          ptr(depth, f), ptr(flow, f), ptr(K, f), ptr(Tl, f), ptr(Ti, f), ptr(T_out, f), ptr(flow_out, d),
                                          ptr(inl, C.c_uint8), ptr(stats, d))


@pytest.mark.gpu
def test_gpu_malformed_batches_are_refused(ctx):
    probs = [make_flow_problem(n=n, seed=s) for n, s in ((40, 1), (60, 2), (30, 3))]
    tot = 130
    a = dict(mode=np.array([1, 0, 1], np.int32), off=np.array([0, 40, 100, tot], np.int32),
             pts=np.concatenate([p["pts"] for p in probs]), depth=np.concatenate([p["depth"] for p in probs]),
             flow=np.concatenate([p["flow"] for p in probs]), K=np.stack([p["K"] for p in probs]),
             Tl=np.stack([p["Tcw_last"] for p in probs]), Ti=np.stack([p["T_init"] for p in probs]))
    outs = lambda: dict(T_out=np.full((3, 4, 4), 7, np.float32), flow_out=np.full((tot, 2), -3.0), inl=np.full(tot, 9, np.uint8),
                        stats=np.full((3, 8), 5.0))
    cases = {
        "offset[0] != 0": dict(off=np.array([1, 40, 100, tot], np.int32)),
        "decreasing offset": dict(off=np.array([0, 100, 40, tot], np.int32)),
        "offset past the end, then back": dict(off=np.array([0, 40, 1 << 30, tot], np.int32)),
        "mode 2": dict(mode=np.array([1, 2, 1], np.int32)),
        "mode -1": dict(mode=np.array([-1, 0, 1], np.int32)),
        "NULL pts": dict(pts=None), "NULL depth": dict(depth=None), "NULL flow": dict(flow=None),
    }
    for what, change in cases.items():
        args, o = dict(a, **change), outs()
        rc = _call(ctx, **args, **o)
        assert rc == -2, f"{what}: returned {rc}, expected VDO_ERR_ARG"
        ref = outs()
        assert all(np.array_equal(o[k], ref[k]) for k in o), f"{what}: an output was written"
    o = outs()
    assert _call(ctx, **a, **o) == 0 and o["stats"][0, 0] > 0          # the context still works
    # no points at all: NULL point arrays are fine, every problem returns identity without optimising
    o = dict(T_out=np.zeros((3, 4, 4), np.float32), flow_out=None, inl=None, stats=np.zeros((3, 8)))
    assert _call(ctx, a["mode"], np.zeros(4, np.int32), None, None, None, a["K"], a["Tl"], a["Ti"], **o) == 0
    assert np.array_equal(o["T_out"], np.broadcast_to(np.eye(4, dtype=np.float32), (3, 4, 4))) and (o["stats"][:, 0] == -1).all()
