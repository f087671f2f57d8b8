"""The device ORB path (OrbExtractor / vdo_orb_extract_batch_dev and Frame.orb_extract / orb_describe) against the oracle across image
sizes, ORB settings and image content, including pyramid levels too small for a cell and levels of 1 to 7 px.

Tolerances as in test_orb_batch_gpu.py: candidate counts per level and keypoint x, y, octave, response and size exactly, angles within
1e-3 degrees, descriptors within max(4, bits / 50000) differing bits; pyramid, FAST score maps and blurred levels bit for bit against cv2
on every level.  Each case states the regime it is for (level sizes, cells per level, initial octree nodes, capacities), computed with
the oracle's formulas and asserted, and prints it with -s.  Also: the create-time refusals, and a mixed tracker batch with a geometry
whose small levels have no cells."""
import ctypes as C
import math

import cv2
import numpy as np
import pytest
import torch

from oracle import image_ops as io
from tests.test_image_oracle import _fast_score
from vdo_slam_b200 import capi

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG, ERR_UNSUPPORTED = -2, -3
FIELDS = ("x", "y", "octave", "response", "angle", "size")
DEFAULT = dict(n_features=2500, scale_factor=1.2, n_levels=8, ini_th_fast=20, min_th_fast=7)
OCT_MAX_CAP = 8192


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


# ------------------------------------------------------------------------------------------------ content (seeded, any size >= 64 x 64)
def noise(seed, w, h):
    """smoothed Gaussian noise, contrast-stretched to 0 .. 255"""
    rng = np.random.default_rng(seed)
    a = cv2.GaussianBlur(rng.normal(0, 1, (h, w)).astype(np.float32), (0, 0), 1.5)
    lo, hi = np.percentile(a, (1, 99))
    return np.clip((a - lo) / (hi - lo) * 255, 0, 255).round().astype(np.uint8)


def checker(seed, w, h):
    """a checkerboard of period 2 or 4 px whose squares take one of four grey levels per colour: dense strict 3x3 maxima, equal scores
    side by side, and deep octrees"""
    rng = np.random.default_rng(seed)
    s = 1 + seed % 2
    y, x = np.mgrid[0:h, 0:w]
    i, j = y // s, x // s
    base = np.where((i + j) % 2 == 0, 50, 190)
    step = rng.integers(0, 4, (h // s + 1, w // s + 1)) * 15
    return (base + step[i, j]).astype(np.uint8)


def weak_corners(seed, w, h):
    """a flat image with a few isolated pixels 12 grey levels up (score 11, strict maxima): no corner reaches iniThFAST = 20, so every
    cell falls back to minThFAST"""
    rng = np.random.default_rng(seed)
    img = np.full((h, w), 100, np.uint8)
    n = max(4, w * h // 4000)
    img[rng.integers(20, h - 20, n), rng.integers(20, w - 20, n)] = 112
    return img


def saturated(seed, w, h):
    """0 / 255 only: smoothed noise thresholded at its median"""
    a = noise(seed, w, h)
    return np.where(a > np.median(a), 255, 0).astype(np.uint8)


def ramp(seed, w, h):
    y, x = np.mgrid[0:h, 0:w]
    return ((x * (1 + seed % 3) + 2 * y) * 255 // (w * (1 + seed % 3) + 2 * h)).astype(np.uint8)


CONTENT = dict(noise=noise, checker=checker, weak=weak_corners, saturated=saturated, ramp=ramp)


# ------------------------------------------------------------------------------------------------ the regime of a case, by the oracle's formulas
def regime(w, h, s):
    """per level: size, cells, initial octree nodes (0 without cells) and octree capacity max(N + 2, 4 nIni) (0 without cells)"""
    prm = io.OrbParams(s["n_features"], s["scale_factor"], s["n_levels"], s["ini_th_fast"], s["min_th_fast"])
    out = []
    for l in range(s["n_levels"]):
        lw = w if l == 0 else io.cvround(float(np.float32(w) * prm.inv_scale[l]))
        lh = h if l == 0 else io.cvround(float(np.float32(h) * prm.inv_scale[l]))
        cells, (minX, maxX, minY, maxY) = io.level_cells(lw, lh) if min(lw, lh) > 0 else ([], (0, 0, 0, 0))
        nini = int(math.floor(float(np.float32(maxX - minX) / np.float32(maxY - minY)) + 0.5)) if cells else 0
        out.append(dict(w=lw, h=lh, cells=len(cells), nini=nini, N=prm.per_level[l], cap=max(prm.per_level[l] + 2, 4 * nini) if cells else 0))
    return out


def _print_regime(name, R, ncand=None, angle_err=None):
    print(f"\n[{name}] sizes {[(r['w'], r['h']) for r in R]} cells {[r['cells'] for r in R]} nIni {[r['nini'] for r in R]} "
          f"caps {[r['cap'] for r in R]}" + (f" candidates {ncand}" if ncand is not None else "") +
          (f" worst angle error {angle_err:.2e} deg" if angle_err is not None else ""))


# ------------------------------------------------------------------------------------------------ comparisons
def _oracle(gray, s):
    r = io.orb_extract(gray, io.OrbParams(s["n_features"], s["scale_factor"], s["n_levels"], s["ini_th_fast"], s["min_th_fast"]))
    r["descriptors"] = io.orb_describe(r)
    return r


def _row(res, i):
    n = int(res["count"][i])
    d = {k: res[k][i, :n].cpu().numpy() for k in FIELDS}
    d["descriptors"] = res["descriptors"][i, :n].cpu().numpy()
    d["n_candidates"] = res["n_candidates"][i].cpu().tolist()
    d["status"] = int(res["status"][i])
    return d


def _assert_matches_oracle(got, ref, what):
    """returns the worst angle error"""
    assert got["n_candidates"] == ref["n_candidates"], f"{what}: candidates per level {got['n_candidates']} vs {ref['n_candidates']}"
    assert len(got["x"]) == len(ref["x"]), f"{what}: {len(got['x'])} keypoints vs {len(ref['x'])}"
    for k in ("x", "y", "octave", "response", "size"):
        assert np.array_equal(np.asarray(got[k]), ref[k]), f"{what}: {k}"
    err = float(np.abs(got["angle"] - ref["angle"]).max()) if len(got["x"]) else 0.0
    assert err <= 1e-3, f"{what}: angle off by {err}"
    nbits = int(np.unpackbits(got["descriptors"] ^ ref["descriptors"]).sum())
    assert got["descriptors"].shape == ref["descriptors"].shape and nbits <= max(4, got["descriptors"].size * 8 // 50000), f"{what}: {nbits} bits"
    return err


def _score_ref(img):
    """cv::cornerScore<16> clipped at 0 on the level; a level under 7 px has no pixel whose ring fits, all 0"""
    h, w = img.shape
    return np.zeros((h, w), np.int32) if h < 7 or w < 7 else np.minimum(_fast_score(img), 255)


def _frame_path(ctx, gray, s, ref, what):
    """Frame.upload + orb_extract + orb_describe on the same image: the oracle's keypoints and descriptors, and pyramid, score map and
    blur of every level bit for bit against cv2"""
    h, w = gray.shape
    F = capi.Frame(ctx, w, h)
    F.upload(gray=gray)
    g = F.orb_extract(s["n_features"], s["scale_factor"], s["n_levels"], s["ini_th_fast"], s["min_th_fast"], max_out=max(len(ref["x"]), 1))
    n = len(g["x"])
    g["descriptors"] = F.orb_describe(n)
    err = _assert_matches_oracle(g, ref, f"{what} (Frame path)")
    for lv, img in enumerate(ref["levels"]):
        dimg, dsc = F.debug_level(lv)
        assert dimg.shape == img.shape and np.array_equal(dimg, img), f"{what}: pyramid level {lv} {img.shape}"
        assert np.array_equal(dsc.astype(np.int32), _score_ref(img)), f"{what}: score level {lv} {img.shape}"
        if n:                                          # the levels are blurred by a describe call with keypoints
            assert np.array_equal(F.debug_blur(lv, img.shape), io.blur_level(img)), f"{what}: blur level {lv} {img.shape}"
    F.close()
    return g, err


def _run_case(ctx, name, w, h, s, contents):
    """one extractor batch of len(contents) frames and the Frame path on the first; returns the regime and the oracle results"""
    R = regime(w, h, s)
    grays = [CONTENT[c](seed, w, h) for seed, c in enumerate(contents)]
    refs = [_oracle(g, s) for g in grays]
    ex = capi.OrbExtractor(ctx, w, h, len(grays), **s)
    assert ex.capacity == sum(r["cap"] for r in R), f"{name}: capacity"
    res = ex.extract(torch.from_numpy(np.stack(grays)).to(DEV))
    torch.cuda.synchronize()
    worst = 0.0
    for i, (c, ref) in enumerate(zip(contents, refs)):
        got = _row(res, i)
        assert got["status"] == 0 and len(got["x"]) <= ex.capacity, f"{name} {c}"
        worst = max(worst, _assert_matches_oracle(got, ref, f"{name} frame {i} ({c})"))
    fp, err = _frame_path(ctx, grays[0], s, refs[0], f"{name} ({contents[0]})")
    row0 = _row(res, 0)
    for k in FIELDS + ("descriptors",):
        assert np.array_equal(fp[k], row0[k]), f"{name}: Frame path and extractor differ in {k}"
    _print_regime(name, R, [r["n_candidates"] for r in refs], max(worst, err))
    return R, refs


# ------------------------------------------------------------------------------------------------ 1. geometries
def _with_cells(R):
    return [r["cells"] > 0 for r in R]


def _levels_with_cells(k, n=8):
    return [l < k for l in range(n)]


# (name, w, h, settings, contents, regime check)
GEOMETRIES = [
    ("64x64", 64, 64, DEFAULT, ("noise", "checker", "weak"), lambda R: _with_cells(R) == _levels_with_cells(1)),
    ("65x97", 65, 97, DEFAULT, ("noise", "saturated", "ramp"), lambda R: _with_cells(R) == _levels_with_cells(1) and R[0]["cells"] == 2),
    ("97x65", 97, 65, DEFAULT, ("noise", "saturated", "noise"), lambda R: _with_cells(R) == _levels_with_cells(1) and R[0]["nini"] == 2),
    # frames shorter than 221 px lose a level's cells at 8 levels of 1.2: 375x220 has none on level 7, 375x221 has cells on every level
    ("375x220", 375, 220, DEFAULT, ("noise", "checker", "noise"), lambda R: _with_cells(R) == _levels_with_cells(7) and R[7]["h"] == 61),
    ("375x221", 375, 221, DEFAULT, ("noise", "weak", "noise"), lambda R: all(_with_cells(R)) and R[7]["h"] == 62),
    ("1241x374", 1241, 374, DEFAULT, ("noise", "saturated", "noise"), lambda R: all(_with_cells(R))),
    ("1243x376", 1243, 376, DEFAULT, ("noise", "ramp", "noise"), lambda R: all(_with_cells(R))),
    ("1242x375_content", 1242, 375, DEFAULT, ("checker", "weak", "saturated"), lambda R: all(_with_cells(R))),
    ("1920x1080", 1920, 1080, DEFAULT, ("noise", "noise", "noise"), lambda R: all(_with_cells(R)) and R[0]["cells"] > 2000),
    # wide strips: over 100 initial nodes on level 0; with 500 features the capacity of that level is 4 nIni, not N + 2
    ("4096x64", 4096, 64, DEFAULT, ("noise", "checker", "weak"), lambda R: _with_cells(R) == _levels_with_cells(1) and R[0]["nini"] > 100),
    ("4096x64_nf500", 4096, 64, dict(DEFAULT, n_features=500), ("noise", "checker", "noise"),
     lambda R: R[0]["nini"] > 100 and R[0]["cap"] == 4 * R[0]["nini"] > R[0]["N"] + 2),
    ("4096x96", 4096, 96, DEFAULT, ("noise", "saturated", "noise"), lambda R: _with_cells(R) == _levels_with_cells(3) and R[0]["nini"] == 64),
    ("4096x96_nf500", 4096, 96, dict(DEFAULT, n_features=500), ("noise", "noise", "noise"),
     lambda R: all(r["cap"] == 4 * r["nini"] > r["N"] + 2 for r in R[:3])),
    ("480x640", 480, 640, DEFAULT, ("noise", "noise", "noise"), lambda R: all(_with_cells(R)) and all(r["nini"] == 1 for r in R)),
    # (w - 32) / (h - 32) exactly 0.5, 1.5 and 2.5 on level 0: nIni rounds half away from zero on the host and on the device
    ("132x232_half", 132, 232, dict(DEFAULT, n_levels=1), ("noise", "noise", "noise"), lambda R: R[0]["nini"] == 1),
    ("332x232_1.5", 332, 232, DEFAULT, ("noise", "noise", "noise"), lambda R: R[0]["nini"] == 2),
    ("282x132_2.5", 282, 132, DEFAULT, ("noise", "noise", "noise"), lambda R: R[0]["nini"] == 3 and _with_cells(R) == _levels_with_cells(5)),
]


@pytest.mark.parametrize("case", GEOMETRIES, ids=[c[0] for c in GEOMETRIES])
def test_geometry_matches_oracle(ctx, case):
    name, w, h, s, contents, check = case
    R = regime(w, h, s)
    assert check(R), f"{name} is no longer the regime it is meant to test: {R}"
    if name.endswith(("_half", "_1.5", "_2.5")):
        r = np.float32(w - 32) / np.float32(h - 32)
        assert r * 2 == math.floor(r * 2) and r != math.floor(r), f"{name}: (w - 32) / (h - 32) = {r} is not k + 1/2"
    _run_case(ctx, name, w, h, s, contents)


# ------------------------------------------------------------------------------------------------ 2. settings
def _first_refused_nfeatures(w, h, s):
    """the smallest n_features whose largest level capacity exceeds OCT_MAX_CAP (the capacity grows with n_features)"""
    cap = lambda nf: max(r["cap"] for r in regime(w, h, dict(s, n_features=nf)))
    lo, hi = 1, 1
    while cap(hi) <= OCT_MAX_CAP:
        lo, hi = hi, 2 * hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if cap(mid) <= OCT_MAX_CAP else (lo, mid)
    return hi


SETTINGS = [
    ("levels1", 1242, 375, dict(DEFAULT, n_levels=1), lambda R: len(R) == 1),
    ("levels2", 1242, 375, dict(DEFAULT, n_levels=2), lambda R: len(R) == 2),
    ("levels12", 1242, 375, dict(DEFAULT, n_levels=12), lambda R: _with_cells(R) == _levels_with_cells(10, 12)),
    ("scale1.01", 640, 480, dict(DEFAULT, scale_factor=1.01, n_levels=12), lambda R: R[11]["w"] == 574),
    ("scale1.5", 640, 480, dict(DEFAULT, scale_factor=1.5, n_levels=12), lambda R: min(R[11]["w"], R[11]["h"]) < 7),
    # 64x64 at 2.0 with 7 levels: 64, 32, 16, 8, 4, 2 and 1 px
    ("scale2.0_64x64", 64, 64, dict(DEFAULT, scale_factor=2.0, n_levels=7), lambda R: [r["w"] for r in R] == [64, 32, 16, 8, 4, 2, 1]),
    ("scale2.0_97x65", 97, 65, dict(DEFAULT, scale_factor=2.0, n_levels=7), lambda R: [(r["w"], r["h"]) for r in R][-1] == (2, 1)),
    ("nfeatures1", 1242, 375, dict(DEFAULT, n_features=1), lambda R: R[0]["N"] == 0 and R[-1]["N"] == 1),
    ("nfeatures7", 1242, 375, dict(DEFAULT, n_features=7), lambda R: sum(r["N"] for r in R[:-1]) == 8 and R[-1]["N"] == 0),   # the last level's quota clamps at 0
    ("nfeatures20000", 640, 480, dict(DEFAULT, n_features=20000), lambda R: R[0]["cap"] > 4000),
    ("nfeatures_at_cap", 640, 480, None, lambda R: max(r["cap"] for r in R) == OCT_MAX_CAP),
    ("ini_eq_min", 1242, 375, dict(DEFAULT, ini_th_fast=12, min_th_fast=12), lambda R: True),
    ("min1", 1242, 375, dict(DEFAULT, ini_th_fast=20, min_th_fast=1), lambda R: True),
]


def _settings_contents(name):
    if name in ("ini_eq_min", "min1", "scale2.0_64x64"):
        return ("noise", "weak", "checker")
    if name in ("nfeatures20000", "nfeatures_at_cap"):            # one dense frame: the oracle's octree over 20 000+ nodes is slow
        return ("noise", "weak", "ramp")
    return ("noise", "noise", "saturated")


@pytest.mark.parametrize("case", SETTINGS, ids=[c[0] for c in SETTINGS])
def test_settings_match_oracle(ctx, case):
    name, w, h, s, check = case
    if s is None:                                      # the largest n_features whose level capacities stay within OCT_MAX_CAP
        s = dict(DEFAULT, n_features=_first_refused_nfeatures(w, h, DEFAULT) - 1)
    R = regime(w, h, s)
    assert check(R), f"{name} is no longer the regime it is meant to test: {R}"
    _run_case(ctx, name, w, h, s, _settings_contents(name))


# ------------------------------------------------------------------------------------------------ 3. create-time refusals
def _refusals():
    nf = _first_refused_nfeatures(640, 480, DEFAULT)
    return [
        ("375x1242 (nIni = 0 on level 0)", 375, 1242, DEFAULT, ERR_UNSUPPORTED, "no initial octree node", True),
        ("220x375 (nIni = 0 on level 4, which has cells)", 220, 375, DEFAULT, ERR_UNSUPPORTED, "level 4", True),
        ("64x64 at 2.0 with 8 levels (level 7 is 0 px)", 64, 64, dict(DEFAULT, scale_factor=2.0, n_levels=8), ERR_ARG, "level 7", True),
        # the node bound is the device's: the oracle's octree has no such limit
        (f"640x480 with {nf} features (capacity over {OCT_MAX_CAP})", 640, 480, dict(DEFAULT, n_features=nf), ERR_UNSUPPORTED, "octree nodes", False),
    ]


def test_create_time_refusals(ctx):
    """the extractor and the Frame path refuse these geometries when they are set up, with the call and the reason in the error, before
    any device work: a refused Frame.orb_extract keeps the frame's previous extraction.  The oracle refuses (or cannot size) the first
    three too"""
    cases = _refusals()
    R = regime(375, 1242, DEFAULT)
    assert R[0]["cells"] > 0 and R[0]["nini"] == 0
    R = regime(220, 375, DEFAULT)
    assert R[0]["nini"] == 1 and R[4]["cells"] > 0 and R[4]["nini"] == 0
    R = regime(64, 64, cases[2][3])
    assert (R[6]["w"], R[7]["w"]) == (1, 0)
    R = regime(640, 480, cases[3][3])
    assert max(r["cap"] for r in R) == OCT_MAX_CAP + 1
    L = ctx.L
    for what, w, h, s, rc, reason, oracle_refuses in cases:
        _print_regime(what, regime(w, h, s))
        if oracle_refuses:
            with pytest.raises((ValueError, cv2.error)):
                io.orb_extract(noise(0, w, h), io.OrbParams(s["n_features"], s["scale_factor"], s["n_levels"], s["ini_th_fast"], s["min_th_fast"]))
        h_ = C.c_void_p(None)
        got = L.vdo_orb_extractor_create(ctx.h, C.c_int(w), C.c_int(h), C.c_int(3), C.c_int(s["n_features"]), C.c_float(s["scale_factor"]),
                                         C.c_int(s["n_levels"]), C.c_int(s["ini_th_fast"]), C.c_int(s["min_th_fast"]), C.byref(h_))
        err = L.vdo_last_error(ctx.h).decode()
        assert got == rc and h_.value is None, what
        assert err.startswith("vdo_orb_extractor_create: ") and reason in err, f"{what}: {err}"
        # the Frame path: a frame that has extracted with valid settings (one level, where level 0 has an initial node) keeps that
        # extraction when the next settings are refused; a frame that never extracted still has nothing to show
        F = capi.Frame(ctx, w, h)
        g = noise(1, w, h)
        F.upload(gray=g)
        baseline = regime(w, h, dict(DEFAULT, n_levels=1))[0]["nini"] >= 1
        if baseline:
            F.orb_extract(nlevels=1)
            before = F.debug_level(0)
        with pytest.raises(capi.VdoError, match=f"vdo_orb_extract failed with {rc}: vdo_orb_extract: .*{reason}"):
            F.orb_extract(s["n_features"], s["scale_factor"], s["n_levels"], s["ini_th_fast"], s["min_th_fast"])
        if baseline:
            after = F.debug_level(0)
            assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1]) and np.array_equal(after[0], g), what
        else:
            with pytest.raises(capi.VdoError):
                F.debug_level(0)
        F.close()
    # tracker creation refuses the zero-size level (an argument out of range); the extractor's limits are reported when tracking
    with pytest.raises(capi.VdoError, match="vdo_tracker_create: ORB settings: level 7 of 64x64"):
        capi.Tracker(ctx, width=64, height=64, scale_factor=2.0, n_levels=8)
    capi.Tracker(ctx, width=64, height=64, scale_factor=2.0, n_levels=7)


# ------------------------------------------------------------------------------------------------ 4. a mixed tracker batch with cell-less levels
def test_mixed_batch_with_levels_without_cells(ctx):
    """one track_tensors_mixed call over a 1242x375 and a 200x96 sequence: the launch grids are sized by the larger geometry, and every
    level of the 200x96 one from level 3 on has no cells.  Each tracker must equal tracking it alone, step by step."""
    from tests.test_tracker_mixed_gpu import _alone, _assert_same, _frames, _inputs, _mixed, _tracker
    R = regime(200, 96, DEFAULT)
    assert _with_cells(R) == _levels_with_cells(3), R
    _print_regime("mixed 200x96", R)
    seqs = (dict(seed=0, w=1242, h=375, K=None, start=0, params=dict(window_size=6, overlap_size=2)),
            dict(seed=5, w=200, h=96, K=(180.0, 180.0, 99.5, 47.5), start=0, params=dict(n_features=700, window_size=6, overlap_size=2)))
    steps = 4
    frames = [_frames(s, steps) for s in seqs]
    tm = [_tracker(ctx, s) for s in seqs]
    ts = [_tracker(ctx, s) for s in seqs]
    for t in range(steps):
        ins_m = [_inputs(frames[i][t], t, i) for i in range(2)]
        ins_s = [_inputs(frames[i][t], t, i) for i in range(2)]
        Tm = _mixed(tm, ins_m, [frames[i][t]["obj_ids"] for i in range(2)])
        for i in range(2):
            what = f"step {t} sequence {i} ({seqs[i]['w']}x{seqs[i]['h']})"
            Ts = _alone(ts[i], ins_s[i], frames[i][t]["obj_ids"])
            assert np.array_equal(Tm[i], Ts), f"{what}: Tcw"
            _assert_same(tm[i], ts[i], what)
            assert torch.equal(ins_m[i][1], ins_s[i][1]) and torch.equal(ins_m[i][3], ins_s[i][3]), f"{what}: write-back"
    for i in range(2):
        assert len(tm[i].get("mvKeys")) > 0, f"sequence {i}: keypoints"
