"""The numpy restatement of ORB descriptor matching (tests/orb_match_reference.py) pinned to cv2.BFMatcher(NORM_HAMMING): knnMatch with
k = 1 and 2, knnMatch with a search-window mask, and crossCheck=True match, on random descriptors with planted duplicates so that equal
distances occur, at counts 0, 1 and the full set."""
import numpy as np
import pytest

from tests import orb_match_reference as R

cv2 = pytest.importorskip("cv2")
CAP = 400


def planted_set(seed: int, n: int = CAP):
    """n descriptors in which many rows repeat (exact ties) or differ from another row in one bit (ties between neighbours), and
    positions on a 200 x 100 field"""
    rng = np.random.default_rng(seed)
    d = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    src = rng.integers(0, n, n // 3)
    d[rng.integers(0, n, n // 3)] = d[src]
    flip = rng.integers(0, n, n // 6)
    d[flip, rng.integers(0, 32, len(flip))] ^= np.uint8(1) << rng.integers(0, 8, len(flip)).astype(np.uint8)
    xy = rng.uniform(0, [200, 100], (n, 2)).astype(np.float32)
    return d, xy


@pytest.fixture(scope="module")
def sets():
    q, qxy = planted_set(1)
    t, txy = planted_set(2)
    # the train set shares rows with the query set, so queries have several equally near train keypoints
    rng = np.random.default_rng(3)
    t[::5] = q[rng.integers(0, CAP, len(t[::5]))]
    t[1::5] = t[::5]
    return q, qxy, t, txy


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("nq,nt", [(CAP, CAP), (0, CAP), (CAP, 0), (1, CAP), (CAP, 1), (1, 1), (0, 0)])
def test_knn_equals_cv2(sets, k, nq, nt):
    q, _, t, _ = sets
    idx, dist, _ = R.match(q[:nq], t[:nt], k)
    ci, cd = R.cv2_knn(cv2, q[:nq], t[:nt], k)
    np.testing.assert_array_equal(idx, ci)
    np.testing.assert_array_equal(dist, cd)
    if nq == CAP and nt == CAP:
        assert (dist[:, 0] == dist[:, -1]).sum() > 10, "the planted sets must produce equal distances"


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("radius", [4.0, 15.0])
def test_window_equals_cv2_mask(sets, k, radius):
    q, qxy, t, txy = sets
    pred = qxy + np.float32(0.5)
    M = R.window_mask(txy[:, 0], txy[:, 1], pred, radius)
    idx, dist, _ = R.match(q, t, k, M)
    ci, cd = R.cv2_knn(cv2, q, t, k, M)
    np.testing.assert_array_equal(idx, ci)
    np.testing.assert_array_equal(dist, cd)
    if radius == 4.0:
        assert (idx[:, 0] < 0).any() and (idx[:, 1 if k == 2 else 0] >= 0).any(), "some queries must have no candidate, others k"


@pytest.mark.parametrize("nq,nt", [(CAP, CAP), (1, CAP), (CAP, 1), (0, CAP), (CAP, 0)])
def test_cross_check_equals_cv2(sets, nq, nt):
    q, _, t, _ = sets
    idx, dist, rev = R.match(q[:nq], t[:nt], 1, None, cross_check=True)
    ci, cd = R.cv2_knn(cv2, q[:nq], t[:nt], 1, cross_check=True)
    np.testing.assert_array_equal(idx, ci)
    np.testing.assert_array_equal(dist, cd)


def test_cross_check_self(sets):
    q = sets[0]
    idx, dist, rev = R.match(q, q, 1, None, cross_check=True)
    ci, cd = R.cv2_knn(cv2, q, q, 1, cross_check=True)
    np.testing.assert_array_equal(idx, ci)
    np.testing.assert_array_equal(dist, cd)


def test_reverse_best_query(sets):
    """rev[j] is the lowest query index at the smallest distance to j among j's candidates"""
    q, qxy, t, txy = sets
    M = R.window_mask(txy[:, 0], txy[:, 1], qxy, 10.0)
    _, _, rev = R.match(q, t, 1, M)
    D = np.where(M, R.hamming(q, t), 10 ** 6)
    for j in range(len(t)):
        if not M[:, j].any():
            assert rev[j] == -1
        else:
            assert rev[j] == int(np.flatnonzero(D[:, j] == D[:, j].min())[0])
