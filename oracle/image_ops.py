"""oracle/image_ops.py -- TEST INFRASTRUCTURE ONLY: CPU restatement of the image side of the per-frame path.

What the reference owns is restated in numpy / plain Python, line by line; what OpenCV owns is delegated to the cv2
installed in this image (4.13 headless -- the reference pins 3.4.0, Dockerfile:40-63; the drift is stated, not hidden),
which therefore acts as the pin for FAST, resize and fastAtan2:

  depth pre-processing      src/Tracking.cc:180-204
  ORBextractor              src/ORBextractor.cc:399-459 (ctor), :1112-1137 (ComputePyramid), :754-842
                            (ComputeKeyPointsOctTree), :470-526 (DivideNode), :528-752 (DistributeOctTree),
                            :66-93 (IC_Angle), :1035-1110 (operator())
  Frame static filter       src/Frame.cc:100-129, :181-194
  Frame object sampling     src/Frame.cc:200-228
  back-projection           src/Frame.cc:484-555 (cv::Mat float gemm: double accumulation, float result)
  scene flow                src/Tracking.cc:1278-1364

One deliberate deviation: DistributeOctTree sorts (size, node pointer) pairs, i.e. breaks ties between equally sized
nodes by heap address (ORBextractor.cc:673) -- not reproducible by anyone.  Here ties are broken by node creation order
(later-created node first, which is what an increasing bump allocator would give); the CUDA path uses the same rule.
"""
from __future__ import annotations

import math

import cv2
import numpy as np

PATCH_SIZE, HALF_PATCH_SIZE, EDGE_THRESHOLD = 31, 15, 19


# ------------------------------------------------------------------------------------------------- depth
def depth_prep(d: np.ndarray, bf: float, factor: float) -> np.ndarray:
    d = d.astype(np.float32)
    with np.errstate(divide="ignore"):
        out = np.float32(bf) / (d / np.float32(factor))
    return np.where(d < 0, np.float32(0), out).astype(np.float32)


# ------------------------------------------------------------------------------------------------- ORB
class OrbParams:
    def __init__(self, nfeatures=2500, scale=1.2, nlevels=8, ini_th=20, min_th=7):
        self.nfeatures, self.nlevels, self.ini_th, self.min_th = nfeatures, nlevels, ini_th, min_th
        sf = np.float32(scale)
        self.scale_factor = [np.float32(1.0)]
        for _ in range(1, nlevels):
            self.scale_factor.append(np.float32(self.scale_factor[-1] * sf))
        self.inv_scale = [np.float32(1.0) / s for s in self.scale_factor]
        factor = np.float32(1.0) / sf
        nd = np.float32(nfeatures) * (np.float32(1) - factor) / (np.float32(1) - np.float32(math.pow(float(factor), float(nlevels))))
        self.per_level, tot = [], 0
        for _ in range(nlevels - 1):
            self.per_level.append(int(cvround(float(nd)))); tot += self.per_level[-1]
            nd = np.float32(nd * factor)
        self.per_level.append(max(nfeatures - tot, 0))
        # umax of the circular patch
        vmax = int(math.floor(HALF_PATCH_SIZE * math.sqrt(2.0) / 2 + 1))
        vmin = int(math.ceil(HALF_PATCH_SIZE * math.sqrt(2.0) / 2))
        hp2 = HALF_PATCH_SIZE * HALF_PATCH_SIZE
        umax = [0] * (HALF_PATCH_SIZE + 1)
        for v in range(vmax + 1):
            umax[v] = cvround(math.sqrt(hp2 - v * v))
        v0 = 0
        for v in range(HALF_PATCH_SIZE, vmin - 1, -1):
            while umax[v0] == umax[v0 + 1]:
                v0 += 1
            umax[v] = v0
            v0 += 1
        self.umax = umax


def cvround(x: float) -> int:
    """cvRound: round half to even (lrint)."""
    return int(np.rint(x))


def compute_pyramid(gray: np.ndarray, prm: OrbParams):
    levels = [gray.copy()]
    h, w = gray.shape
    for lv in range(1, prm.nlevels):
        s = prm.inv_scale[lv]
        sz = (cvround(float(np.float32(w) * s)), cvround(float(np.float32(h) * s)))
        levels.append(cv2.resize(levels[lv - 1], sz, interpolation=cv2.INTER_LINEAR))
    return levels


def level_cells(w: int, h: int):
    """Cell grid of ComputeKeyPointsOctTree for a level of size w x h: list of (iniX, iniY, maxX, maxY, offX, offY) in the
    reference's loop order, plus the borders.

    A level narrower or shorter than 62 px has nCols = 0 or nRows = 0, and the reference then divides by zero
    (ORBextractor.cc:773-776): its result is undefined there.  This returns no cells for such a level, which is the product's
    rule (OrbGeometry::build in frame_kernels.cu), not the reference's: the level yields no candidates and no keypoints, and its
    quota is not handed to other levels."""
    minB = EDGE_THRESHOLD - 3
    maxBX, maxBY = w - EDGE_THRESHOLD + 3, h - EDGE_THRESHOLD + 3
    width, height = np.float32(maxBX - minB), np.float32(maxBY - minB)
    nCols, nRows = int(width / np.float32(30)), int(height / np.float32(30))
    if nCols < 1 or nRows < 1:
        return [], (minB, maxBX, minB, maxBY)
    wCell, hCell = int(math.ceil(float(width / np.float32(nCols)))), int(math.ceil(float(height / np.float32(nRows))))
    cells = []
    for i in range(nRows):
        iniY = minB + i * hCell
        maxY = iniY + hCell + 6
        if iniY >= maxBY - 3:
            continue
        maxY = min(maxY, maxBY)
        for j in range(nCols):
            iniX = minB + j * wCell
            maxX = iniX + wCell + 6
            if iniX >= maxBX - 6:
                continue
            maxX = min(maxX, maxBX)
            cells.append((iniX, iniY, maxX, maxY, j * wCell, i * hCell))
    return cells, (minB, maxBX, minB, maxBY)


def fast_candidates(img: np.ndarray, prm: OrbParams):
    """(x, y, response) in level coordinates relative to minBorder, in the reference's push_back order."""
    h, w = img.shape
    cells, _ = level_cells(w, h)
    det_hi = cv2.FastFeatureDetector_create(prm.ini_th, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
    det_lo = cv2.FastFeatureDetector_create(prm.min_th, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
    out = []
    for (x0, y0, x1, y1, ox, oy) in cells:
        roi = np.ascontiguousarray(img[y0:y1, x0:x1])
        kps = det_hi.detect(roi)
        if not kps:
            kps = det_lo.detect(roi)
        for k in kps:
            out.append((np.float32(k.pt[0] + ox), np.float32(k.pt[1] + oy), np.float32(k.response)))
    return out


class _Node:
    __slots__ = ("UL", "UR", "BL", "BR", "keys", "no_more", "alive", "seq")

    def __init__(self):
        self.keys, self.no_more, self.alive, self.seq = [], False, True, 0


def _divide(n: _Node):
    halfX = int(math.ceil(float(np.float32(n.UR[0] - n.UL[0]) / np.float32(2))))
    halfY = int(math.ceil(float(np.float32(n.BR[1] - n.UL[1]) / np.float32(2))))
    c = [_Node() for _ in range(4)]
    c[0].UL = n.UL; c[0].UR = (n.UL[0] + halfX, n.UL[1]); c[0].BL = (n.UL[0], n.UL[1] + halfY); c[0].BR = (n.UL[0] + halfX, n.UL[1] + halfY)
    c[1].UL = c[0].UR; c[1].UR = n.UR; c[1].BL = c[0].BR; c[1].BR = (n.UR[0], n.UL[1] + halfY)
    c[2].UL = c[0].BL; c[2].UR = c[0].BR; c[2].BL = n.BL; c[2].BR = (c[0].BR[0], n.BL[1])
    c[3].UL = c[2].UR; c[3].UR = c[1].BR; c[3].BL = c[2].BR; c[3].BR = n.BR
    for kp in n.keys:
        if kp[0] < c[0].UR[0]:
            (c[0] if kp[1] < c[0].BR[1] else c[2]).keys.append(kp)
        elif kp[1] < c[0].BR[1]:
            c[1].keys.append(kp)
        else:
            c[3].keys.append(kp)
    for k in c:
        if len(k.keys) == 1:
            k.no_more = True
    return c


def distribute_octtree(keys, minX, maxX, minY, maxY, N):
    """keys: list of (x, y, response) float32.  Returns the retained keys in the reference's output order (list order).

    Raises ValueError when the border box gives no initial node (nIni < 1: (maxX - minX) / (maxY - minY) < 0.5, an image more than
    about twice as tall as wide), whatever the keys: the reference indexes an empty node vector there (ORBextractor.cc:558), and the
    device extractor refuses such a geometry at creation."""
    nIni = int(math.floor(float(np.float32(maxX - minX) / np.float32(maxY - minY)) + 0.5))   # C round(): half away from zero
    if nIni < 1:
        raise ValueError(f"DistributeOctTree: nIni = {nIni} initial nodes for the border box x [{minX}, {maxX}) y [{minY}, {maxY})")
    if not keys:
        return []
    hX = np.float32(maxX - minX) / np.float32(nIni)
    nodes = []          # python list emulating std::list: index 0 = front; push_front = insert(0)
    ini = []
    for i in range(nIni):
        n = _Node()
        n.UL = (int(hX * np.float32(i)), 0); n.UR = (int(hX * np.float32(i + 1)), 0)
        n.BL = (n.UL[0], maxY - minY); n.BR = (n.UR[0], maxY - minY)
        nodes.append(n); ini.append(n)
    for kp in keys:
        ini[int(kp[0] / hX)].keys.append(kp)
    nodes = [n for n in nodes if n.keys]
    for n in nodes:
        if len(n.keys) == 1:
            n.no_more = True
    seq = [0]

    def push_children(n, lst, expand):
        for c in _divide(n):
            if c.keys:
                seq[0] += 1; c.seq = seq[0]
                lst.insert(0, c)
                if len(c.keys) > 1:
                    expand.append(c)

    finish = False
    while not finish:
        prev = len(nodes)
        expand = []
        i = 0
        # iterate the list front to back; children are pushed to the FRONT, i.e. never revisited in this pass
        cur = list(nodes)
        for n in cur:
            if n.no_more:
                continue
            push_children(n, nodes, expand)
            nodes.remove(n)
        if len(nodes) >= N or len(nodes) == prev:
            finish = True
        elif len(nodes) + len(expand) * 3 > N:
            while not finish:
                prev = len(nodes)
                prev_expand = expand
                expand = []
                # sort ascending by (size, pointer) and walk from the back: largest first; ties -> latest created first
                prev_expand.sort(key=lambda c: (len(c.keys), c.seq))
                for n in reversed(prev_expand):
                    push_children(n, nodes, expand)
                    nodes.remove(n)
                    if len(nodes) >= N:
                        break
                if len(nodes) >= N or len(nodes) == prev:
                    finish = True
    out = []
    for n in nodes:
        best = n.keys[0]
        for k in n.keys[1:]:
            if k[2] > best[2]:
                best = k
        out.append(best)
    return out


def ic_angle(img: np.ndarray, x: float, y: float, umax) -> float:
    cx, cy = cvround(x), cvround(y)
    m01 = m10 = 0
    row = img[cy].astype(np.int64)
    for u in range(-HALF_PATCH_SIZE, HALF_PATCH_SIZE + 1):
        m10 += u * int(row[cx + u])
    for v in range(1, HALF_PATCH_SIZE + 1):
        d = umax[v]
        rp, rm = img[cy + v].astype(np.int64), img[cy - v].astype(np.int64)
        us = np.arange(-d, d + 1)
        vp, vm = rp[cx + us], rm[cx + us]
        m01 += v * int((vp - vm).sum())
        m10 += int((us * (vp + vm)).sum())
    return float(cv2.fastAtan2(float(np.float32(m01)), float(np.float32(m10))))


def orb_extract(gray: np.ndarray, prm: OrbParams, with_angle=True):
    """ORBextractor::operator(): returns dict(x, y (float32, level-0 coordinates), octave, response, angle, size) in output order,
    plus per-level candidate counts."""
    levels = compute_pyramid(gray, prm)
    xs, ys, octv, resp, ang, size, ncand, lxs, lys = [], [], [], [], [], [], [], [], []
    for lv, img in enumerate(levels):
        h, w = img.shape
        cells, (minX, maxX, minY, maxY) = level_cells(w, h)
        cand = fast_candidates(img, prm)
        ncand.append(len(cand))
        kept = distribute_octtree(cand, minX, maxX, minY, maxY, prm.per_level[lv]) if cells else []     # a level without cells keeps nothing
        sps = int(np.float32(PATCH_SIZE) * prm.scale_factor[lv])
        for (x, y, r) in kept:
            lx, ly = np.float32(x + np.float32(minX)), np.float32(y + np.float32(minY))
            a = ic_angle(img, float(lx), float(ly), prm.umax) if with_angle else -1.0
            if lv != 0:
                fx, fy = np.float32(lx * prm.scale_factor[lv]), np.float32(ly * prm.scale_factor[lv])
            else:
                fx, fy = lx, ly
            xs.append(fx); ys.append(fy); octv.append(lv); resp.append(r); ang.append(a); size.append(sps); lxs.append(lx); lys.append(ly)
    return dict(x=np.asarray(xs, np.float32), y=np.asarray(ys, np.float32), octave=np.asarray(octv, np.int32),
                response=np.asarray(resp, np.float32), angle=np.asarray(ang, np.float32), size=np.asarray(size, np.int32),
                n_candidates=ncand, levels=levels, level_x=np.asarray(lxs, np.float32), level_y=np.asarray(lys, np.float32))


# ------------------------------------------------------------------------------------------------- descriptors (A6)
def orb_pattern():
    """The 256 point pairs of ORB's learned sampling pattern (src/ORBextractor.cc:139-397; OpenCV's bit_pattern_31_), read from the
    data file the CUDA kernel includes (vdo_slam_b200/csrc/orb_pattern.inc).  Pinned below against cv2.ORB, which carries the same table."""
    import os
    import re
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vdo_slam_b200", "csrc", "orb_pattern.inc")
    txt = "".join(l for l in open(path) if not l.lstrip().startswith("//"))
    v = np.array([int(t) for t in re.findall(r"-?\d+", txt)], np.int32)
    assert len(v) == 1024
    return v.reshape(512, 2)


def blur_level(img: np.ndarray) -> np.ndarray:
    """GaussianBlur(workingMat, Size(7, 7), 2, 2, BORDER_REFLECT_101) (src/ORBextractor.cc:1083-1084): OpenCV's own (cv2 4.13; 3.4.0 filtered
    in float -- version drift stated)."""
    return cv2.GaussianBlur(img, (7, 7), 2, None, 2, cv2.BORDER_REFLECT_101)


def blur_level_fixed_point(img: np.ndarray) -> np.ndarray:
    """The arithmetic cv2 4.13 uses for that call on CV_8U, restated (what k_blur7_batch implements): Q8.8 kernel {18, 34, 48, 56, 48, 34, 18},
    horizontal pass in Q8.8, vertical in Q16.16, (v + 2^15) >> 16."""
    k = np.array([18, 34, 48, 56, 48, 34, 18], np.int64)
    p = cv2.copyMakeBorder(img, 3, 3, 3, 3, cv2.BORDER_REFLECT_101).astype(np.int64)
    H, W = img.shape
    h = sum(k[i] * p[:, i:i + W] for i in range(7))
    v = sum(k[i] * h[i:i + H, :] for i in range(7))
    return ((v + (1 << 15)) >> 16).astype(np.uint8)


def orb_descriptor(blurred: np.ndarray, x: float, y: float, angle_deg: float, pattern=None) -> np.ndarray:
    """computeOrbDescriptor (src/ORBextractor.cc:97-136) on a blurred level image; (x, y) in level coordinates.  float arithmetic as written
    there (products and sums in float, cvRound = round-half-even)."""
    pat = orb_pattern() if pattern is None else pattern
    f32 = np.float32
    ang = f32(f32(angle_deg) * f32(np.pi / f32(180.0)))
    a, b = f32(np.cos(np.float64(ang))), f32(np.sin(np.float64(ang)))
    cy, cx = cvround(float(y)), cvround(float(x))
    px, py = pat[:, 0].astype(f32), pat[:, 1].astype(f32)
    iy = np.rint(px * b + py * a).astype(np.int64)
    ix = np.rint(px * a - py * b).astype(np.int64)
    vals = blurred[cy + iy, cx + ix].astype(np.int32).reshape(256, 2)
    bits = (vals[:, 0] < vals[:, 1]).astype(np.uint8).reshape(32, 8)
    return (bits << np.arange(8, dtype=np.uint8)).sum(1).astype(np.uint8)


def orb_describe(res: dict) -> np.ndarray:
    """Descriptors (n x 32 u8) of an orb_extract() result: per level blur + rotated pair tests (src/ORBextractor.cc:1075-1091)."""
    pat = orb_pattern()
    blurred = [blur_level(im) for im in res["levels"]]
    out = np.zeros((len(res["x"]), 32), np.uint8)
    for i in range(len(out)):
        out[i] = orb_descriptor(blurred[int(res["octave"][i])], res["level_x"][i], res["level_y"][i], res["angle"][i], pat)
    return out


# ------------------------------------------------------------------------------------------------- Frame sampling
def filter_static(kx, ky, mask, depth, flow, th_depth):
    """Frame.cc:100-129 + 181-194.  Returns indices of kept keypoints (order preserved), correspondences, flows, depths."""
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
            if np.float32(kx[i] + fx) < w and np.float32(ky[i] + fy) < h and kx[i] < w and ky[i] < h:
                keep.append(i); cx.append(np.float32(kx[i] + fx)); cy.append(np.float32(ky[i] + fy)); fu.append(fx); fv.append(fy)
                dd = depth[int(ky[i]), int(kx[i])]
                dep.append(dd if dd > 0 else np.float32(-1))
    return (np.asarray(keep, np.int32), np.asarray(cx, np.float32), np.asarray(cy, np.float32), np.asarray(fu, np.float32),
            np.asarray(fv, np.float32), np.asarray(dep, np.float32))


def sample_objects(mask, depth, flow, th_depth_obj, step=4):
    """Frame.cc:200-228: raster scan with stride 4; returns x, y (int), corres x,y, flow, depth, label in push_back order."""
    h, w = mask.shape
    ys, xs = np.mgrid[0:h:step, 0:w:step]
    ys, xs = ys.ravel(), xs.ravel()
    m, d = mask[ys, xs], depth[ys, xs]
    fx, fy = flow[ys, xs, 0], flow[ys, xs, 1]
    tx, ty = (xs.astype(np.float32) + fx).astype(np.float32), (ys.astype(np.float32) + fy).astype(np.float32)
    ok = (m != 0) & (d < np.float32(th_depth_obj)) & (d > 0) & (tx < w) & (tx > 0) & (ty < h) & (ty > 0)
    return dict(x=xs[ok].astype(np.int32), y=ys[ok].astype(np.int32), cx=tx[ok], cy=ty[ok], fx=fx[ok], fy=fy[ok], depth=d[ok],
                label=m[ok].astype(np.int32))


# ------------------------------------------------------------------------------------------------- back-projection
def unproject_world(u, v, z, K, Tcw):
    """Frame::UnprojectStereoStat/Object: float arithmetic, Rwl*x+twl as a cv::Mat float gemm (double accumulation)."""
    fx, fy, cx, cy = [np.float32(k) for k in K]
    invfx, invfy = np.float32(1.0) / fx, np.float32(1.0) / fy
    u, v, z = np.asarray(u, np.float32), np.asarray(v, np.float32), np.asarray(z, np.float32)
    x = ((u - cx) * z * invfx).astype(np.float32)
    y = ((v - cy) * z * invfy).astype(np.float32)
    T = np.asarray(Tcw, np.float32)
    Rwl = T[:3, :3].T.astype(np.float64)
    twl = (-(Rwl @ T[:3, 3].astype(np.float64))).astype(np.float32)
    X = np.stack([x, y, z], -1).astype(np.float64)
    return (X @ Rwl.T + twl.astype(np.float64)).astype(np.float32)


def scene_flow(u_prev, v_prev, z_prev, Tcw_prev, u_cur, v_cur, z_cur, Tcw_cur, K, lab_prev, lab_cur):
    """Tracking::GetSceneFlowObj: flow3d = X_w(cur) - X_w(prev) in float; invalid (label <= 0 in either frame) -> label -1."""
    Xp = unproject_world(u_prev, v_prev, z_prev, K, Tcw_prev)
    Xc = unproject_world(u_cur, v_cur, z_cur, K, Tcw_cur)
    valid = (np.asarray(lab_cur) > 0) & (np.asarray(lab_prev) > 0)
    f = (Xc - Xp).astype(np.float32)
    f[~valid] = 0
    return f, valid
