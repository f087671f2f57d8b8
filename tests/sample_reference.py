"""Serial restatement of the sampled background features (UseSampleFeature: 1) for the tests: cv::RNG, Frame::SampleKeyPoints
(src/Frame.cc:672-740), the option-II static filter (src/Frame.cc:130-168, 181-194) and the renewal source (src/Tracking.cc:2718-2721), with
the oracle pipeline extended to run the OMD configuration.  The generator is pinned to cv2 in tests/test_sample_features.py."""
import numpy as np

from oracle.tracking_pipeline import OracleTracker

RNG_A = 4164903690
RNG_M = RNG_A * 2 ** 32 - 1
SAMPLE_N, SAMPLE_DIV = 3000, 20


class CvRNG:
    """cv::RNG: state = (uint64)(unsigned)state * 4164903690u + (state >> 32); RNG(0) starts from 0xffffffff."""

    def __init__(self, seed: int):
        seed &= 0xffffffff
        self.state = seed if seed else 0xffffffff

    def next(self) -> int:
        self.state = (self.state & 0xffffffff) * RNG_A + (self.state >> 32)
        return self.state & 0xffffffff

    def uniform(self, a: int, b: int) -> int:
        return a if a == b else a + self.next() % (b - a)


def rng_jump(state: int, k: int) -> int:
    """the state k steps after `state` (< 2^32, nonzero): the LCG form A^k * state mod (A * 2^32 - 1)"""
    return pow(RNG_A, k, RNG_M) * state % RNG_M


def sample_keypoints(rows: int, cols: int, seed: int):
    """Frame::SampleKeyPoints with cv::RNG(seed): x, y (f32, integer values) cell by cell (i*20 + j), in draw order inside a cell"""
    rng = CvRNG(seed)
    xs, ys = cols // SAMPLE_DIV, rows // SAMPLE_DIV
    grid = [[] for _ in range(SAMPLE_DIV * SAMPLE_DIV)]
    n = 0
    while n < SAMPLE_N:
        for i in range(SAMPLE_DIV):
            for j in range(SAMPLE_DIV):
                x = rng.uniform(i * xs, (i + 1) * xs)
                y = rng.uniform(j * ys, (j + 1) * ys)
                if x >= cols or y >= rows or x <= 0 or y <= 0:
                    continue
                grid[i * SAMPLE_DIV + j].append((x, y))
                n += 1
                if n >= SAMPLE_N:
                    break
            if n >= SAMPLE_N:
                break
    k = np.array([p for cell in grid for p in cell], np.float32)
    return k[:, 0].copy(), k[:, 1].copy()


def filter_static_sampled(kx, ky, mask, depth, flow, th_depth):
    """Frame.cc:130-168 + 181-194 (option II): the target is bounded on both sides, the key itself is not tested"""
    h, w = mask.shape
    keep, cx, cy, fu, fv, dep = [], [], [], [], [], []
    for i in range(len(kx)):
        x, y = int(kx[i]), int(ky[i])
        if mask[y, x] != 0:
            continue
        d = depth[y, x]
        if d > np.float32(th_depth) or d <= 0:
            continue
        fx, fy = flow[y, x, 0], flow[y, x, 1]
        if fx != 0 and fy != 0:
            tx, ty = np.float32(kx[i] + fx), np.float32(ky[i] + fy)
            if tx < w and ty < h and tx > 0 and ty > 0:
                keep.append(i); cx.append(tx); cy.append(ty); fu.append(fx); fv.append(fy)
                dep.append(d if d > 0 else np.float32(-1))
    return (np.asarray(keep, np.int32), np.asarray(cx, np.float32), np.asarray(cy, np.float32), np.asarray(fu, np.float32),
            np.asarray(fv, np.float32), np.asarray(dep, np.float32))


class SampleOracleTracker(OracleTracker):
    """OracleTracker with UseSampleFeature: frame f_id samples from cv::RNG((uint32)(sample_seed + f_id))"""

    def __init__(self, use_sample_feature=1, sample_seed=0, **kw):
        super().__init__(**kw)
        self.sample, self.seed = use_sample_feature, sample_seed

    def _build_frame(self, gray, depth, flow, mask):
        F = super()._build_frame(gray, depth, flow, mask)
        if not self.sample or len(F.keys) == 0:                  # Frame.cc:95-98: no ORB keypoints, no static keys either
            return F
        kx, ky = sample_keypoints(self.h, self.w, (self.seed + self.f_id) & 0xffffffff)
        keep, cx, cy, fu, fv, dep = filter_static_sampled(kx, ky, mask, depth, flow, self.th_bg)
        F.statKeysTmp = np.stack([kx[keep], ky[keep]], 1).astype(np.float32).reshape(-1, 2)
        F.corres = np.stack([cx, cy], 1).astype(np.float32).reshape(-1, 2)
        F.flowNext = np.stack([fu, fv], 1).astype(np.float32).reshape(-1, 2)
        F.statDepthTmp = dep
        return F

    def _track(self, C, L, depth, flow, mask):
        if not self.sample:
            return super()._track(C, L, depth, flow, mask)
        keys, C.keys = C.keys, C.statKeysTmp                      # RenewFrameInfo tops up from mvStatKeysTmp (Tracking.cc:2718-2721)
        try:
            super()._track(C, L, depth, flow, mask)
        finally:
            C.keys = keys
