"""Brute-force restatement of cv2.BFMatcher(NORM_HAMMING) as vdo_orb_match_batch_dev defines it (include/vdo_b200.h), for the tests.

match(desc_q, desc_t, k, cand=None, cross_check=False): desc_q (nq, 32) and desc_t (nt, 32) u8, cand (nq, nt) bool or None (every pair).
Returns idx, dist (nq, k) int32 -- the k candidates of smallest Hamming distance per query, in increasing distance, equal distances to the
lower train index, -1 where missing -- and rev (nt,) int32, each train keypoint's best candidate query (ties to the lower query index, -1:
none).  With cross_check (k = 1) a match i -> j is kept only if rev[j] == i.
window_mask(tx, ty, pred, radius): the candidate predicate of a search window, |x_t - px| <= r and |y_t - py| <= r in float32."""
from __future__ import annotations

import numpy as np


def hamming(desc_q: np.ndarray, desc_t: np.ndarray) -> np.ndarray:
    """(nq, nt) int32 Hamming distances of 256-bit descriptors"""
    a = np.ascontiguousarray(desc_q, np.uint8).reshape(-1, 32).view(np.uint64)
    b = np.ascontiguousarray(desc_t, np.uint8).reshape(-1, 32).view(np.uint64)
    out = np.zeros((len(a), len(b)), np.int32)
    for s in range(0, len(a), 256):
        out[s:s + 256] = np.bitwise_count(a[s:s + 256, None, :] ^ b[None, :, :]).sum(-1, dtype=np.int32)
    return out


def window_mask(tx, ty, pred, radius) -> np.ndarray:
    tx, ty = np.asarray(tx, np.float32), np.asarray(ty, np.float32)
    px, py = np.asarray(pred, np.float32)[:, 0], np.asarray(pred, np.float32)[:, 1]
    r = np.float32(radius)
    return (np.abs(tx[None, :] - px[:, None]) <= r) & (np.abs(ty[None, :] - py[:, None]) <= r)


def match(desc_q, desc_t, k: int, cand=None, cross_check: bool = False):
    assert k in (1, 2) and not (cross_check and k != 1)
    nq, nt = len(desc_q), len(desc_t)
    idx = np.full((nq, k), -1, np.int32)
    dist = np.full((nq, k), -1, np.int32)
    rev = np.full(nt, -1, np.int32)
    if nq == 0 or nt == 0:
        return idx, dist, rev
    d = hamming(desc_q, desc_t).astype(np.int64)
    ok = np.ones((nq, nt), bool) if cand is None else np.asarray(cand, bool)
    none = np.iinfo(np.int64).max
    # keys ordered by distance, then index: the smallest keys are the matches
    kf = np.where(ok, d * (nt + 1) + np.arange(nt)[None, :], none)
    best = np.sort(np.partition(kf, min(k, nt) - 1, axis=1)[:, :k], axis=1) if nt > k else np.sort(kf, axis=1)[:, :k]
    for s in range(best.shape[1]):
        have = best[:, s] != none
        idx[have, s] = best[have, s] % (nt + 1)
        dist[have, s] = best[have, s] // (nt + 1)
    kr = np.where(ok, d * (nq + 1) + np.arange(nq)[:, None], none).min(axis=0)
    have = kr != none
    rev[have] = kr[have] % (nq + 1)
    if cross_check:
        j = idx[:, 0]
        lost = (j >= 0) & (rev[np.maximum(j, 0)] != np.arange(nq))
        idx[lost, 0] = -1
        dist[lost, 0] = -1
    return idx, dist, rev


def cv2_knn(cv2, desc_q, desc_t, k: int, cand=None, cross_check: bool = False):
    """the same arrays from cv2.BFMatcher: knnMatch(k, mask=cand) or, with cross_check, BFMatcher(crossCheck=True).match"""
    nq = len(desc_q)
    idx = np.full((nq, k), -1, np.int32)
    dist = np.full((nq, k), -1, np.int32)
    q = np.ascontiguousarray(desc_q, np.uint8)
    t = np.ascontiguousarray(desc_t, np.uint8)
    if cross_check:
        if len(t) == 0:   # cv2 asserts on an empty train set here; no query has a match
            return idx, dist
        for m in cv2.BFMatcher(cv2.NORM_HAMMING, crossCheck=True).match(q, t):
            idx[m.queryIdx, 0], dist[m.queryIdx, 0] = m.trainIdx, int(m.distance)
        return idx, dist
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    res = bf.knnMatch(q, t, k=k) if cand is None else bf.knnMatch(q, t, k=k, mask=np.ascontiguousarray(cand, np.uint8))
    for row in res:
        for s, m in enumerate(row):
            idx[m.queryIdx, s], dist[m.queryIdx, s] = m.trainIdx, int(m.distance)
    return idx, dist
