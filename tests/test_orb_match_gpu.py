"""ORB descriptor matching on the device (capi.orb_match / vdo_orb_match_batch_dev) against the numpy restatement of
cv2.BFMatcher(NORM_HAMMING) (tests/orb_match_reference.py) and cv2 itself: knnMatch k = 1 and 2, with and without a search window, and
crossCheck, exactly.  Inputs: OrbExtractor descriptors of consecutive synth.make_sequence_frame frames (1242 x 375, 3 000 features; the
window is predicted from the synthetic flow) and planted sets with repeated descriptors, so equal distances occur.  Also: batch and split
independence at 64 pairs, capture in a CUDA graph, the refusals, and counts outside 0 .. cap found on the device."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import orb_match_reference as R
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_sequence_frame

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
DEV = torch.device("cuda", 0)
ERR_ARG = -2
W, H = 1242, 375
UNSET = -7          # fill of the output tensors: slots the call must not write keep it
MODES = [(1, "plain"), (2, "plain"), (1, "window"), (2, "window"), (1, "cross"), (1, "cross-window")]


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@pytest.fixture(scope="module")
def seq(ctx):
    """descriptors of frames 0..3 of sequence 0 (host copies too) and each frame's flow to the next"""
    frames = [make_sequence_frame(t, seed=0, width=W, height=H) for t in range(4)]
    ex = capi.OrbExtractor(ctx, W, H, 4, n_features=3000)
    gray = torch.from_numpy(np.stack([f["gray"] for f in frames])).to(DEV)
    r = ex.extract(gray)
    s = {k: r[k].clone() for k in ("descriptors", "x", "y", "count")}
    torch.cuda.synchronize()
    assert (r["status"] == 0).all() and (s["count"] > 1000).all()
    return s, [f["flow"] for f in frames]


def planted(seed: int, F: int = 4, cap: int = 520, counts=(520, 0, 1, 383)):
    """a descriptor set on a 1000 x 600 field whose rows often repeat across and within frames"""
    rng = np.random.default_rng(seed)
    d = rng.integers(0, 256, (F, cap, 32), dtype=np.uint8)
    pool = d[0, :60].copy()
    for f in range(F):
        sel = rng.integers(0, cap, cap // 2)
        d[f, sel] = pool[rng.integers(0, len(pool), len(sel))]
    xy = rng.uniform(0, [1000, 600], (F, cap, 2)).astype(np.float32)
    return {"descriptors": torch.from_numpy(d).to(DEV), "x": torch.from_numpy(np.ascontiguousarray(xy[..., 0])).to(DEV),
            "y": torch.from_numpy(np.ascontiguousarray(xy[..., 1])).to(DEV), "count": torch.tensor(counts, dtype=torch.int32, device=DEV)}


def host(s):
    return {k: s[k].cpu().numpy() for k in ("descriptors", "x", "y", "count")}


def pred_of(qs, pairs, flows=None):
    """(P, cap, 2) predicted positions: the query position, moved by the flow to the next frame when the pair is (t, t + 1)"""
    cap = qs["x"].shape[1]
    out = np.zeros((len(pairs), cap, 2), np.float32)
    for p, (q, t) in enumerate(pairs):
        x, y = qs["x"][q], qs["y"][q]
        out[p, :, 0], out[p, :, 1] = x, y
        if flows is not None and t == q + 1:
            xi = np.clip(np.nan_to_num(x), 0, W - 1).astype(np.int64)     # rows past the count hold whatever the buffer held
            yi = np.clip(np.nan_to_num(y), 0, H - 1).astype(np.int64)
            out[p, :, 0] = x + flows[q][yi, xi, 0].astype(np.float32)
            out[p, :, 1] = y + flows[q][yi, xi, 1].astype(np.float32)
    return out


def mode_args(mode):
    return dict(radius=15.0 if "window" in mode else None, cross_check="cross" in mode)


def filled_out(ctx, P, qcap, tcap, k, cross):
    o = capi.orb_match_empty_outputs(ctx, P, qcap, tcap, k, cross)
    for t in o.values():
        t.fill_(UNSET)
    return o


def check_pair(res, p, qh, th, q, t, k, mode, pred, with_cv2=True):
    """pair p of a result against the reference (and cv2): rows < count[q] exactly, rows past it untouched"""
    nq, nt = int(qh["count"][q]), int(th["count"][t])
    cand = None
    if "window" in mode:
        cand = R.window_mask(th["x"][t, :nt], th["y"][t, :nt], pred[p, :nq], 15.0)
    ri, rd, rr = R.match(qh["descriptors"][q, :nq], th["descriptors"][t, :nt], k, cand, "cross" in mode)
    gi, gd = res["idx"][p].cpu().numpy(), res["dist"][p].cpu().numpy()
    np.testing.assert_array_equal(gi[:nq], ri, err_msg=f"pair {p} ({q}, {t}) {mode} k={k}: idx")
    np.testing.assert_array_equal(gd[:nq], rd, err_msg=f"pair {p} ({q}, {t}) {mode} k={k}: dist")
    assert (gi[nq:] == UNSET).all() and (gd[nq:] == UNSET).all(), "slots past the query count were written"
    if "rev_idx" in res:
        gr = res["rev_idx"][p].cpu().numpy()
        np.testing.assert_array_equal(gr[:nt], rr, err_msg=f"pair {p}: rev_idx")
        assert (gr[nt:] == UNSET).all()
    assert int(res["status"][p]) == 0
    if with_cv2 and not ("cross" in mode and "window" in mode):
        ci, cd = R.cv2_knn(cv2, qh["descriptors"][q, :nq], th["descriptors"][t, :nt], k, cand, "cross" in mode)
        np.testing.assert_array_equal(gi[:nq], ci)
        np.testing.assert_array_equal(gd[:nq], cd)
    return ri


@pytest.mark.parametrize("k,mode", MODES)
def test_extracted_frames_equal_reference(ctx, seq, k, mode):
    s, flows = seq
    sh = host(s)
    pairs = [(0, 1), (1, 2), (2, 3), (3, 0), (2, 2)]     # consecutive frames, an unrelated pair, a set against itself
    pred = pred_of(sh, pairs, flows)
    a = mode_args(mode)
    out = filled_out(ctx, len(pairs), s["x"].shape[1], s["x"].shape[1], k, a["cross_check"])
    res = capi.orb_match(ctx, s, s, pairs, k=k, pred=torch.from_numpy(pred).to(DEV), out=out, **a)
    torch.cuda.synchronize()
    for p, (q, t) in enumerate(pairs):
        ri = check_pair(res, p, sh, sh, q, t, k, mode, pred)
        if (q, t) == (0, 1) and mode == "window":
            assert (ri[:, 0] >= 0).mean() > 0.5, "the flow-predicted window should find most features"
        if (q, t) == (2, 2) and mode == "plain":
            assert (ri[:, 0] == np.arange(len(ri))).mean() > 0.9   # every row finds itself unless an earlier row is equal


@pytest.mark.parametrize("k,mode", MODES)
def test_planted_ties_and_empty_frames(ctx, k, mode):
    qs, ts = planted(11), planted(12, counts=(520, 1, 0, 400))
    ts["descriptors"][:, ::3] = qs["descriptors"][0, 100:100 + 174]   # train rows equal to query rows: ties at distance 0
    qh, th = host(qs), host(ts)
    pairs = [(0, 0), (0, 1), (0, 2), (1, 0), (2, 3), (3, 3), (3, 0)]
    pred = pred_of(qh, pairs)
    a = mode_args(mode)
    out = filled_out(ctx, len(pairs), 520, 520, k, a["cross_check"])
    res = capi.orb_match(ctx, qs, ts, pairs, k=k, pred=torch.from_numpy(pred).to(DEV), out=out, **a)
    torch.cuda.synchronize()
    for p, (q, t) in enumerate(pairs):
        check_pair(res, p, qh, th, q, t, k, mode, pred)
    if "window" in mode:
        assert (res["idx"][0, :, 0] == -1).any(), "the window should leave some queries without a candidate"
    else:
        assert (res["dist"][0, :, 0] == 0).sum() > 100


@pytest.mark.parametrize("k,mode", [(2, "plain"), (2, "window"), (1, "cross"), (1, "cross-window")])
def test_batch_of_64_equals_each_pair_alone(ctx, seq, k, mode):
    s, flows = seq
    cap = s["x"].shape[1]
    # eight frames: the four extracted ones and the same with other counts
    big = {key: torch.cat([s[key], s[key]]) for key in ("descriptors", "x", "y")}
    c = s["count"].cpu().tolist()
    big["count"] = torch.tensor(c + [c[0] // 2, 7, 0, c[3] - 101], dtype=torch.int32, device=DEV)
    rng = np.random.default_rng(5)
    pairs = [tuple(int(v) for v in rng.integers(0, 8, 2)) for _ in range(64)]
    pairs[:3] = [(0, 1), (4, 5), (6, 2)]
    bh = host(big)
    pred = pred_of(bh, pairs)
    pred_t = torch.from_numpy(pred).to(DEV)
    a = mode_args(mode)
    res = capi.orb_match(ctx, big, big, pairs, k=k, pred=pred_t, out=filled_out(ctx, 64, cap, cap, k, a["cross_check"]), **a)
    torch.cuda.synchronize()
    for p in range(64):
        one = capi.orb_match(ctx, big, big, [pairs[p]], k=k, pred=pred_t[p:p + 1].contiguous(), out=filled_out(ctx, 1, cap, cap, k, a["cross_check"]), **a)
        for key in one:
            assert torch.equal(one[key][0], res[key][p]), f"pair {p} {pairs[p]}: {key} differs alone and in the batch"
    for p in (0, 1, 2, 10):
        check_pair(res, p, bh, bh, *pairs[p], k, mode, pred, with_cv2=False)


def test_cuda_graph_replay_equals_eager(ctx, seq):
    s, flows = seq
    cap = s["x"].shape[1]
    qs = {key: s[key][:2].clone() for key in s}
    ts = {key: s[key][2:].clone() for key in s}
    pairs = [(0, 0), (1, 1), (0, 1)]
    pred = torch.from_numpy(pred_of(host(qs), pairs)).to(DEV)
    out = capi.orb_match_empty_outputs(ctx, 3, cap, cap, 1, True)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):      # warm-up outside the capture
        capi.orb_match(ctx, qs, ts, pairs, k=1, radius=15.0, pred=pred, cross_check=True, out=out)
    torch.cuda.current_stream(DEV).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        capi.orb_match(ctx, qs, ts, pairs, k=1, radius=15.0, pred=pred, cross_check=True, out=out)
    # new descriptors in the captured input tensors: frames swapped, one count lowered
    for key in s:
        qs[key].copy_(s[key][2:]); ts[key].copy_(s[key][:2])
    qs["count"][1] -= 300
    pred.copy_(torch.from_numpy(pred_of(host(qs), pairs)).to(DEV))
    for t in out.values():
        t.fill_(UNSET)
    g.replay()
    eager = capi.orb_match(ctx, qs, ts, pairs, k=1, radius=15.0, pred=pred, cross_check=True, out=filled_out(ctx, 3, cap, cap, 1, True))
    torch.cuda.synchronize()
    for key in eager:
        assert torch.equal(out[key], eager[key]), key


def test_count_outside_range_sets_status(ctx, seq):
    s, _ = seq
    cap = s["x"].shape[1]
    bad = {key: s[key].clone() for key in s}
    bad["count"][1] = cap + 1
    bad["count"][2] = -1
    sh = host(s)
    pairs = [(1, 0), (0, 2), (0, 3), (2, 1)]
    out = filled_out(ctx, 4, cap, cap, 1, True)
    res = capi.orb_match(ctx, bad, bad, pairs, k=1, cross_check=True, out=out)
    torch.cuda.synchronize()
    Q, T = capi.ORB_MATCH_STATUS_QUERY_COUNT, capi.ORB_MATCH_STATUS_TRAIN_COUNT
    assert res["status"].tolist() == [Q, T, 0, Q | T]
    assert (res["idx"][0] == UNSET).all() and (res["dist"][0] == UNSET).all()     # query rows not written
    n0 = int(sh["count"][0])
    assert (res["idx"][1, :n0] == -1).all() and (res["dist"][1, :n0] == -1).all()  # train taken as empty
    assert (res["idx"][1, n0:] == UNSET).all() and (res["rev_idx"][1] == UNSET).all()
    assert (res["idx"][3] == UNSET).all() and (res["rev_idx"][3] == UNSET).all()
    np.testing.assert_array_equal(res["idx"][2, :n0, 0].cpu().numpy(), R.match(sh["descriptors"][0, :n0], sh["descriptors"][3, :int(sh["count"][3])], 1,
                                                                                 cross_check=True)[0][:, 0])


def test_python_refusals(ctx, seq):
    s, _ = seq
    cap = s["x"].shape[1]
    with pytest.raises(ValueError):
        capi.orb_match(ctx, {**s, "descriptors": s["descriptors"].to(torch.int32)}, s, [(0, 1)])
    with pytest.raises(ValueError):
        capi.orb_match(ctx, {**s, "count": s["count"].cpu()}, s, [(0, 1)])
    with pytest.raises(ValueError):
        capi.orb_match(ctx, s, s, [(0, 1)], radius=10.0, pred=torch.zeros((1, cap, 3), device=DEV))
    with pytest.raises(ValueError):
        capi.orb_match(ctx, s, s, [(0, 1)], radius=10.0)
    with pytest.raises(ValueError):
        capi.orb_match(ctx, s, s, [(0, 1)], k=2, cross_check=True)
    with pytest.raises(ValueError):
        capi.orb_match(ctx, s, s, [(0, 1)] * 65)
    with pytest.raises(ValueError):
        capi.orb_match(ctx, s, s, [(0, 1)], out=capi.orb_match_empty_outputs(ctx, 1, cap, cap, 1))


def test_c_refusals_write_nothing(ctx, seq):
    s, _ = seq
    cap = s["x"].shape[1]
    L = ctx.L
    pairs_np = np.array([[0, 1], [1, 2]], np.int32)
    pred = torch.zeros((2, cap, 2), device=DEV)
    out = filled_out(ctx, 2, cap, cap, 1, True)
    host_buf = np.zeros(cap * 32 * 4, np.uint8)

    def call(P=2, pairs=pairs_np.ctypes.data, k=1, cross=1, radius=10.0, pred_p=pred.data_ptr(), q=None, t=None, o=None, opts=True):
        qs = capi.OrbDescSet(s["descriptors"].data_ptr(), s["x"].data_ptr(), s["y"].data_ptr(), s["count"].data_ptr(), 4, cap)
        ts = capi.OrbDescSet(s["descriptors"].data_ptr(), s["x"].data_ptr(), s["y"].data_ptr(), s["count"].data_ptr(), 4, cap)
        oo = capi.OrbMatchOut(out["idx"].data_ptr(), out["dist"].data_ptr(), out["rev_idx"].data_ptr(), out["status"].data_ptr())
        for st, ch in ((qs, q), (ts, t), (oo, o)):
            for key, v in (ch or {}).items():
                setattr(st, key, v)
        op = capi.OrbMatchOpts(k, cross, radius)
        return L.vdo_orb_match_batch_dev(ctx.h, C.c_int(P), C.c_void_p(pairs), C.byref(qs), C.byref(ts), C.c_void_p(pred_p),
                                         C.byref(op) if opts else None, C.byref(oo), C.c_uint64(0))

    bad_pairs = np.array([[0, 4], [1, 2]], np.int32)
    neg_pairs = np.array([[-1, 0], [1, 2]], np.int32)
    d = s["descriptors"].data_ptr()
    cases = {
        "P = 0": dict(P=0), "P = 65": dict(P=65), "pairs NULL": dict(pairs=None),
        "train frame out of range": dict(pairs=bad_pairs.ctypes.data), "query frame negative": dict(pairs=neg_pairs.ctypes.data),
        "k = 0": dict(k=0, cross=0), "k = 3": dict(k=3, cross=0), "cross_check with k = 2": dict(k=2),
        "cross_check without rev_idx": dict(o={"rev_idx_dev": None}), "NaN radius": dict(radius=float("nan")),
        "window without train x": dict(t={"x_dev": None}), "window without train y": dict(t={"y_dev": None}), "window without pred": dict(pred_p=None),
        "opts NULL": dict(opts=False), "cap 0": dict(q={"cap": 0}), "cap 2^23": dict(t={"cap": 1 << 23}), "no frames": dict(q={"n_frames": 0}),
        "desc NULL": dict(q={"desc_dev": None}), "count NULL": dict(t={"count_dev": None}), "idx NULL": dict(o={"idx_dev": None}),
        "dist NULL": dict(o={"dist_dev": None}), "status NULL": dict(o={"status_dev": None}),
        "desc in host memory": dict(q={"desc_dev": host_buf.ctypes.data}), "desc misaligned": dict(t={"desc_dev": d + 4}),
        "count misaligned": dict(q={"count_dev": s["count"].data_ptr() + 2}), "idx misaligned": dict(o={"idx_dev": out["idx"].data_ptr() + 1}),
        "pred misaligned": dict(pred_p=pred.data_ptr() + 2), "rev_idx in host memory": dict(o={"rev_idx_dev": host_buf.ctypes.data}),
    }
    for name, kw in cases.items():
        assert call(**kw) == ERR_ARG, name
        assert L.vdo_last_error(ctx.h).decode().startswith("vdo_orb_match_batch_dev"), name
    torch.cuda.synchronize()
    for key, t in out.items():
        assert (t == UNSET).all(), f"a refused call wrote {key}"
    assert (host_buf == 0).all()
    assert call() == 0          # the unmodified call is accepted
    torch.cuda.synchronize()
    assert (out["status"] == 0).all()
