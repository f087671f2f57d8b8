// frame_kernels.cu -- image side of the per-frame path on sm_90a: depth pre-processing, ORB keypoints (pyramid, FAST score,
// per-cell FAST + NMS with threshold fallback, octree distribution, intensity-centroid angle), flow-guided static filter,
// semi-dense object sampling, back-projection and scene flow.  The ORB path has one implementation, the extractor (vdo_orb_extractor): it
// runs everything, octree included (k_octree), on the device for up to 64 frames per call, and vdo_orb_extract / vdo_orb_describe and the
// tracker's frame build run on it.
//
// Reference semantics (restated on the CPU in oracle/image_ops.py, with cv2 as the pin for the OpenCV-owned arithmetic):
//   depth pre-processing        src/Tracking.cc:180-204
//   ORBextractor                src/ORBextractor.cc:399-459, 754-842, 470-752, 66-93, 1035-1137
//   cv::resize (u8 INTER_LINEAR), cv::FAST (9/16, NMS), cv::fastAtan2: OpenCV (un-vendored); formulas verified bit-exact
//                               against cv2 4.13 in tests/test_image_oracle.py
//   Frame static filter         src/Frame.cc:100-129, 181-194
//   Frame object sampling       src/Frame.cc:200-228
//   back-projection, scene flow src/Frame.cc:484-555, src/Tracking.cc:1278-1364
//
// A KITTI frame is 1242x375 (0.47 Mpx, ~9 MB of inputs): every kernel here is launch-/latency-bound, not HBM-bound; the
// point of the GPU path is to keep the frame resident next to the LM kernels, not bandwidth.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"
#include "frame_batch.h"
#include "frame_px.cuh"

namespace {


constexpr int EDGE_THRESHOLD = 19, PATCH_SIZE = 31, HALF_PATCH = 15, MAX_LEVELS = 12, CELL_CAP = 512;

// ------------------------------------------------------------------------------------------------ depth
// Batched kernels take a per-launch table with one entry per sequence (blockIdx.z / blockIdx.y / blockIdx.x, or a segment search for
// point lists); each entry carries its own image geometry, the grid is sized for the largest entry and threads past an entry's extent
// return.  The per-element arithmetic is the single-frame one.
struct DepthSeq { float* d; float bf, factor; int n; };   // n: pixels of this frame
__global__ void k_depth_prep(const DepthSeq* __restrict__ tab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const DepthSeq q = tab[blockIdx.y];
  if (i >= q.n) return;
  float* __restrict__ d = q.d;
  const float bf = q.bf, factor = q.factor;
  const float v = d[i];
  d[i] = (v < 0.f) ? 0.f : (bf > 0.f ? __fdiv_rn(bf, __fdiv_rn(v, factor)) : v);   // mbf/(d/mDepthMapFactor), IEEE divisions (d == 0 -> +inf); bf <= 0: clamp only
}

// ------------------------------------------------------------------------------------------------ device ingest / write-back
// Caller planes (vdo_dev_plane) at element strides <-> the resident row-major buffers.  One thread per pixel with threads along x,
// so each plane is read at one fixed element stride across a warp (1 for CHW / planar views, the channel count for HWC).
// one gray pixel of an image plane: a 1-channel plane is copied; colour is cvtColor [RGB|BGR][A]2GRAY in 8-bit fixed point
// (System.cc shim, src/Tracking.cc:209-222)
__device__ __forceinline__ unsigned char gray_px(const PlaneArg& img, int x, int y) {
  const unsigned char* s = (const unsigned char*)img.p + (y * img.sy + x * img.sx);
  if (img.ch == 1) return s[0];
  const int c0 = s[0], G = s[img.sc], c2 = s[2 * img.sc];
  const int R = img.rgb ? c0 : c2, B = img.rgb ? c2 : c0;
  return (unsigned char)((R * 4899 + G * 9617 + B * 1868 + (1 << 13)) >> 14);
}
struct IngestSeq { PlaneArg img, dep, flo, msk; unsigned char* gray; float* depth; float2* flow; int* mask; int* bad_label; int w, h; };
__global__ void __launch_bounds__(256) k_ingest_frame(const IngestSeq* __restrict__ tab) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const IngestSeq& q = tab[blockIdx.z];
  const int w = q.w, h = q.h;
  if (x >= w || y >= h) return;
  const PlaneArg img = q.img, dep = q.dep, flo = q.flo, msk = q.msk;
  unsigned char* __restrict__ gray = q.gray; float* __restrict__ depth = q.depth; float2* __restrict__ flow = q.flow; int* __restrict__ mask = q.mask;
  const size_t p = (size_t)y * w + x;
  if (img.p) gray[p] = gray_px(img, x, y);
  if (dep.p) depth[p] = plane_depth(dep, x, y);
  if (flo.p) flow[p] = plane_flow(flo, x, y);
  if (msk.p) mask[p] = plane_label(msk, x, y, q.bad_label);   // the host refuses a frame with a bad label
}
// the prepared depth and (when given) the mask back into the caller's planes: the device form of the reference mutating the caller's
// cv::Mat (src/Tracking.cc:180-204, :3062)
__global__ void __launch_bounds__(256) k_writeback_frame(const float* __restrict__ depth, const int* __restrict__ mask, int w, int h, PlaneArg dep, PlaneArg msk) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const size_t p = (size_t)y * w + x;
  if (dep.p) ((float*)dep.p)[y * dep.sy + x * dep.sx] = depth[p];
  if (msk.p) {
    const long long o = y * msk.sy + x * msk.sx;
    if (msk.dtype == VDO_DT_I64) ((long long*)msk.p)[o] = mask[p];
    else ((int*)msk.p)[o] = mask[p];
  }
}

// ------------------------------------------------------------------------------------------------ pyramid
// OpenCV u8 INTER_LINEAR: 11-bit fixed-point coefficients, horizontal pass in int, vertical pass with >>4, >>16, +2, >>2.
__device__ __forceinline__ void lin_coeff(int dpos, int sn, double scale, int& s0, int& s1, int& a0, int& a1) {
  float f = (float)((dpos + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (s < 0) { s = 0; f = 0.f; }
  if (s >= sn - 1) { s = sn - 1; f = 0.f; }
  s0 = s; s1 = min(s + 1, sn - 1);
  a0 = __float2int_rn((1.f - f) * 2048.f);
  a1 = __float2int_rn(f * 2048.f);
}
// one pyramid level of one sequence: input plane (sw x sh), output plane (dw x dh); a level the sequence does not have is 0 x 0
struct PairSeq { const unsigned char* src; unsigned char* dst; int sw, sh, dw, dh; };
__global__ void k_resize_u8(const PairSeq* __restrict__ tab) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const PairSeq& q = tab[blockIdx.z];
  const int sw = q.sw, sh = q.sh, dw = q.dw, dh = q.dh;
  if (x >= dw || y >= dh) return;
  const unsigned char* __restrict__ src = q.src; unsigned char* __restrict__ dst = q.dst;
  int x0, x1, ax0, ax1, y0, y1, ay0, ay1;
  lin_coeff(x, sw, (double)sw / dw, x0, x1, ax0, ax1);
  lin_coeff(y, sh, (double)sh / dh, y0, y1, ay0, ay1);
  const int h0 = src[(size_t)y0 * sw + x0] * ax0 + src[(size_t)y0 * sw + x1] * ax1;
  const int h1 = src[(size_t)y1 * sw + x0] * ax0 + src[(size_t)y1 * sw + x1] * ax1;
  int v = (((ay0 * (h0 >> 4)) >> 16) + ((ay1 * (h1 >> 4)) >> 16) + 2) >> 2;
  dst[(size_t)y * dw + x] = (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// ------------------------------------------------------------------------------------------------ FAST score
// score(p) = max over the 16 arcs of 9 contiguous circle pixels of min(|I_p - I_k| signed consistently) - 1
// (== cv::cornerScore<16>); a pixel is a FAST-9/16 corner at threshold t iff score >= t.
__global__ void k_fast_score(const PairSeq* __restrict__ tab) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const PairSeq& q = tab[blockIdx.z];
  const int w = q.dw, h = q.dh;
  if (x >= w || y >= h) return;
  const unsigned char* __restrict__ img = q.src; unsigned char* __restrict__ score = q.dst;
  int out = 0;
  if (x >= 3 && y >= 3 && x < w - 3 && y < h - 3) {
    const unsigned char* p = img + (size_t)y * w + x;
    const int v = p[0];
    // Bresenham circle of radius 3, clockwise from (0,+3); signed differences centre - neighbour
    int d[16];
    d[0] = v - p[3 * w];      d[1] = v - p[3 * w + 1];  d[2] = v - p[2 * w + 2];  d[3] = v - p[w + 3];
    d[4] = v - p[3];          d[5] = v - p[-w + 3];     d[6] = v - p[-2 * w + 2]; d[7] = v - p[-3 * w + 1];
    d[8] = v - p[-3 * w];     d[9] = v - p[-3 * w - 1]; d[10] = v - p[-2 * w - 2]; d[11] = v - p[-w - 3];
    d[12] = v - p[-3];        d[13] = v - p[w - 3];     d[14] = v - p[2 * w - 2]; d[15] = v - p[3 * w - 1];
    // cornerScore = (largest t such that 9 contiguous circle pixels are all > v + t or all < v - t), found by bisection on t with
    // 16-bit circle masks.  (A first version used min/max chains; ptxas for sm_100a fused those into VIMNMX3 and the result came
    // out wrong although the PTX was correct, so this kernel avoids integer min/max.)
    auto is_corner = [&](int t) -> bool {
      unsigned br = 0, dk = 0;
#pragma unroll
      for (int k = 0; k < 16; ++k) { br |= (unsigned)(d[k] > t) << k; dk |= (unsigned)(d[k] < -t) << k; }
      auto nine = [](unsigned m) -> bool {
        m |= m << 16;                                   // unroll the circle
        unsigned a = m & (m >> 1);                      // 2 contiguous
        a &= a >> 2;                                    // 4
        a &= a >> 4;                                    // 8
        a &= m >> 8;                                    // 9
        return (a & 0xffffu) != 0u;
      };
      return nine(br) || nine(dk);
    };
    int lo = -1, hi = 255;                              // invariant: corner at lo (t = -1 is always true), not a corner at hi
#pragma unroll 1
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (is_corner(mid)) lo = mid; else hi = mid;
    }
    out = lo < 0 ? 0 : lo;
  }
  score[(size_t)y * w + x] = (unsigned char)out;
}

// ------------------------------------------------------------------------------------------------ per-cell FAST + NMS
struct Cell {   // ROI [x0,x1) x [y0,y1) in level coordinates; keypoint offset (j*wCell, i*hCell); the score map (row stride w) it reads;
                // the FAST thresholds of its frame (iniThFAST, minThFAST)
  int x0, y0, x1, y1, offx, offy, w, thr_hi, thr_lo;
  const unsigned char* score;
};
struct KpOut { float x, y, resp; };

// One CTA per cell.  Detection region = ROI minus a 3-px frame (cv::FAST on the ROI); NMS neighbours outside it count as 0;
// first threshold thr_hi, and if the cell stays empty thr_lo.  Output row-major, like cv::FAST.
// One launch serves every level of every sequence: each cell names its own score map and thresholds.
__global__ void __launch_bounds__(256) k_fast_cells(const Cell* __restrict__ cells, KpOut* __restrict__ out, int* __restrict__ count) {
  __shared__ unsigned char s[64 * 64];     // cell <= 60 px on a side (width / floor(width / 30) < 60) plus the zero halo
  __shared__ int wsum[8];
  __shared__ int total;
  const Cell c = cells[blockIdx.x];
  const unsigned char* __restrict__ score = c.score; const int w = c.w;
  const int rx0 = c.x0 + 3, ry0 = c.y0 + 3, rw = c.x1 - c.x0 - 6, rh = c.y1 - c.y0 - 6;   // detection region
  const int pw = rw + 2, ph = rh + 2;                                                          // with a zero halo
  for (int i = threadIdx.x; i < pw * ph; i += blockDim.x) {
    const int lx = i % pw - 1, ly = i / pw - 1;
    s[i] = (lx >= 0 && ly >= 0 && lx < rw && ly < rh) ? score[(size_t)(ry0 + ly) * w + rx0 + lx] : 0;
  }
  __syncthreads();
  const int npx = rw * rh;
  const int per = (npx + blockDim.x - 1) / blockDim.x;        // contiguous row-major range per thread keeps the output ordered
  const int b = threadIdx.x * per, e = min(b + per, npx);
  for (int pass = 0; pass < 2; ++pass) {
    const int thr = pass == 0 ? c.thr_hi : c.thr_lo;
    int cnt = 0;
    for (int i = b; i < e; ++i) {
      const int lx = i % rw, ly = i / rw;
      const int v = s[(ly + 1) * pw + lx + 1];
      if (v < thr) continue;
      bool ismax = true;
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
          if (dx == 0 && dy == 0) continue;
          int nb = s[(ly + 1 + dy) * pw + lx + 1 + dx];
          if (nb < thr) nb = 0;
          ismax = ismax && (v > nb);
        }
      cnt += ismax;
    }
    // exclusive scan of cnt over the CTA (warp shuffles + one smem hop)
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) wsum[wid] = incl;
    __syncthreads();
    if (threadIdx.x == 0) { int acc = 0; for (int k = 0; k < 8; ++k) { const int t = wsum[k]; wsum[k] = acc; acc += t; } total = acc; }
    __syncthreads();
    int pos = wsum[wid] + incl - cnt;
    const int tot = total;
    if (tot > 0) {
      KpOut* o = out + (size_t)blockIdx.x * CELL_CAP;
      for (int i = b; i < e; ++i) {
        const int lx = i % rw, ly = i / rw;
        const int v = s[(ly + 1) * pw + lx + 1];
        if (v < thr) continue;
        bool ismax = true;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
          for (int dx = -1; dx <= 1; ++dx) {
            if (dx == 0 && dy == 0) continue;
            int nb = s[(ly + 1 + dy) * pw + lx + 1 + dx];
            if (nb < thr) nb = 0;
            ismax = ismax && (v > nb);
          }
        if (ismax) {
          if (pos < CELL_CAP) { o[pos].x = (float)(lx + 3 + c.offx); o[pos].y = (float)(ly + 3 + c.offy); o[pos].resp = (float)v; }
          ++pos;
        }
      }
      if (threadIdx.x == 0) count[blockIdx.x] = min(tot, CELL_CAP);
      return;                      // uniform: every thread sees the same `total`
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) count[blockIdx.x] = 0;
}

// ------------------------------------------------------------------------------------------------ IC_Angle
struct UmaxArg { int v[16]; };
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {   // cv::fastAtan2 (scalar path), no FMA contraction
  const float s = (float)(180.0 / 3.14159265358979323846);
  const float p1 = 0.9997878412794807f * s, p3 = -0.3258083974640975f * s, p5 = 0.1555786518463281f * s, p7 = -0.04432655554792128f * s;
  const float ax = fabsf(x), ay = fabsf(y), eps = 2.2204460492503131e-16f;
  float a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, eps)); c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, eps)); c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}
struct KpLvl { float x, y; int level; };
struct LevelDesc { const unsigned char* img; int w, h; };
struct LevelsArg { LevelDesc L[MAX_LEVELS]; };
// IC_Angle of keypoint k on its level image L, by one warp: lanes stride over the rows v = 0..15 of the circular patch.  Every lane must
// call it (warp reduction); the angle is valid on lane 0.
__device__ __forceinline__ float ic_angle_warp(const LevelDesc& L, const KpLvl& k, const UmaxArg& umax, int lane) {
  const int cx = __float2int_rn(k.x), cy = __float2int_rn(k.y);
  int m01 = 0, m10 = 0;
  if (lane <= HALF_PATCH) {
    const int v = lane;
    if (v == 0) {
      const unsigned char* r = L.img + (size_t)cy * L.w + cx;
      for (int u = -HALF_PATCH; u <= HALF_PATCH; ++u) m10 += u * (int)r[u];
    } else {
      const int d = umax.v[v];
      const unsigned char* rp = L.img + (size_t)(cy + v) * L.w + cx;
      const unsigned char* rm = L.img + (size_t)(cy - v) * L.w + cx;
      int vs = 0;
      for (int u = -d; u <= d; ++u) { const int a = rp[u], b = rm[u]; vs += a - b; m10 += u * (a + b); }
      m01 = v * vs;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { m01 += __shfl_down_sync(0xffffffffu, m01, o); m10 += __shfl_down_sync(0xffffffffu, m10, o); }
  return fast_atan2_deg((float)m01, (float)m10);
}

// ------------------------------------------------------------------------------------------------ sampling (ordered compaction)
struct ObjSample { int x, y; float cx, cy, fx, fy, depth; int label; };
struct SampleSeq { const int* mask; const float* depth; const float* flow; float th; ObjSample* out; int* n_out; int w, h, cap; };
// Frame.cc:200-228: stride-`step` raster scan, one CTA per sequence so that the output keeps the raster (push_back) order
__global__ void __launch_bounds__(1024) k_sample_objects(const SampleSeq* __restrict__ tab, int step) {
  __shared__ int wsum[33];
  const SampleSeq& q = tab[blockIdx.x];
  const int* __restrict__ mask = q.mask; const float* __restrict__ depth = q.depth; const float* __restrict__ flow = q.flow;
  ObjSample* __restrict__ out = q.out; const float th = q.th;
  const int w = q.w, h = q.h, cap = q.cap;
  const int nx = (w + step - 1) / step, ny = (h + step - 1) / step, n = nx * ny;
  int base = 0;
  for (int start = 0; start < n; start += blockDim.x) {
    const int i = start + threadIdx.x;
    int ok = 0, x = 0, y = 0, m = 0; float d = 0, fx = 0, fy = 0, tx = 0, ty = 0;
    if (i < n) {
      x = (i % nx) * step; y = (i / nx) * step;
      const size_t p = (size_t)y * w + x;
      m = mask[p]; d = depth[p];
      ok = object_sample(x, y, m, d, th, w, h, [&](float& a, float& b) { a = flow[2 * p]; b = flow[2 * p + 1]; }, fx, fy, tx, ty);
    }
    int tot;
    const int pos = base + cta_excl_scan(ok, wsum, tot);
    if (ok && pos < cap) out[pos] = ObjSample{x, y, tx, ty, fx, fy, d, m};
    base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *q.n_out = min(base, cap);
}
struct StatOut { int idx; float cx, cy, fu, fv, depth; };
struct StaticSeq { const float* kx; const float* ky; int n; float th; int sampled; const int* mask; const float* depth; const float* flow; StatOut* out; int* n_out;
                  int w, h; };
// Frame.cc:100-129 + 181-194: keep keys on static background with valid depth and non-zero flow staying in the image (frame_px.cuh's
// static_key); one CTA per sequence.
__global__ void __launch_bounds__(1024) k_filter_static(const StaticSeq* __restrict__ tab) {
  __shared__ int wsum[33];
  const StaticSeq& q = tab[blockIdx.x];
  const int w = q.w, h = q.h;
  const float* __restrict__ kx = q.kx; const float* __restrict__ ky = q.ky; const int* __restrict__ mask = q.mask;
  const float* __restrict__ depth = q.depth; const float* __restrict__ flow = q.flow; StatOut* __restrict__ out = q.out;
  const int n = q.n; const float th = q.th; const bool sampled = q.sampled != 0;
  int base = 0;
  for (int start = 0; start < n; start += blockDim.x) {
    const int i = start + threadIdx.x;
    int ok = 0; float fx = 0, fy = 0, px = 0, py = 0, dd = -1.f;
    if (i < n) {
      px = kx[i]; py = ky[i];
      float d;
      ok = static_key(px, py, th, sampled, w, h, [=](int x, int y) { return mask[(size_t)y * w + x] == 0; },
                      [=](int x, int y) { return depth[(size_t)y * w + x]; },
                      [=](int x, int y, float& u, float& v) { const size_t p = (size_t)y * w + x; u = flow[2 * p]; v = flow[2 * p + 1]; }, d, fx, fy);
      if (ok) dd = d > 0.f ? d : -1.f;
    }
    int tot;
    const int pos = base + cta_excl_scan(ok, wsum, tot);
    if (ok) out[pos] = StatOut{i, __fadd_rn(px, fx), __fadd_rn(py, fy), fx, fy, dd};
    base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *q.n_out = base;
}

// Frame::SampleKeyPoints (src/Frame.cc:672-740): rounds over the 20 x 20 grid (x cell i outer, y cell j inner), each visit drawing
// x = rng.uniform(i*xs, (i+1)*xs) then y = rng.uniform(j*ys, (j+1)*ys) and rejecting x <= 0 || y <= 0, until SAMPLE_N keys are accepted;
// returned cell by cell (i*20 + j ascending), in draw order inside a cell.
//
// cv::RNG is the multiply-with-carry step state' = (uint32)state * A + (state >> 32), uniform(a, b) = a + (uint32)state' % (b - a),
// RNG(0) starting from 0xffffffff.  For a state below 2^32 its k-th successor is the LCG value A^k * state mod M with M = A*2^32 - 1
// (A*2^32 = 1 mod M, so A * (hi*2^32 + lo) = hi + A*lo), and it never reaches M (the orbit of a nonzero residue avoids 0), so each
// thread jumps straight to its own draws.  Every round accepts at least the 361 cells with i, j >= 1, so SAMPLE_ROUNDS rounds always
// reach SAMPLE_N keys.
constexpr int SAMPLE_N = VDO_SAMPLE_KEYS, SAMPLE_DIV = 20, SAMPLE_CELLS = SAMPLE_DIV * SAMPLE_DIV, SAMPLE_ROUNDS = 9, SAMPLE_THREADS = 416;
static_assert(SAMPLE_ROUNDS * (SAMPLE_DIV - 1) * (SAMPLE_DIV - 1) >= SAMPLE_N, "too few rounds for SAMPLE_N keys");
static_assert(SAMPLE_THREADS >= SAMPLE_CELLS && SAMPLE_THREADS % 32 == 0, "one thread per cell");
constexpr unsigned long long RNG_A = 4164903690ull, RNG_M = RNG_A * 4294967296ull - 1ull;
// x * y mod M for x, y < M: the 128-bit product P = q * (A*2^32) + r * 2^32 + p0 with (q, r) = divmod(P >> 32, A) is q + r*2^32 + p0 mod M
__device__ __forceinline__ unsigned long long rng_mulmod(unsigned long long x, unsigned long long y) {
  const unsigned long long lo = x * y, hi = __umul64hi(x, y);
  unsigned long long cur = hi;                                  // (P >> 96) < A: the long division by A starts at the second 32-bit digit
  const unsigned long long q1 = cur / RNG_A;
  cur = ((cur % RNG_A) << 32) | (lo >> 32);
  const unsigned long long q0 = cur / RNG_A;
  unsigned long long q = (q1 << 32) + q0, r = ((cur % RNG_A) << 32) | (lo & 0xffffffffull);   // both <= M
  if (q >= RNG_M) q -= RNG_M;
  if (r >= RNG_M) r -= RNG_M;
  return r >= RNG_M - q ? r - (RNG_M - q) : r + q;
}
__device__ __forceinline__ unsigned long long rng_pow(unsigned long long e) {   // A^e mod M
  unsigned long long r = 1, b = RNG_A;
  for (; e; e >>= 1) { if (e & 1) r = rng_mulmod(r, b); b = rng_mulmod(b, b); }
  return r;
}
__device__ __forceinline__ unsigned rng_next(unsigned long long& s) { s = (s & 0xffffffffull) * RNG_A + (s >> 32); return (unsigned)s; }
struct SampleKeysSeq { unsigned seed; float* kx; float* ky; int w, h; };   // w x h: the frame's size (cols, rows)
// one CTA per frame, thread c owns grid cell c: its visit in round r is visit r*400 + c, drawing the values of states 2*visit + 1 and + 2
__device__ __forceinline__ void sample_keys_cta(const SampleKeysSeq q) {
  __shared__ int wsum[33];
  const int c = threadIdx.x, ci = c / SAMPLE_DIV, cj = c % SAMPLE_DIV;
  const int xs = q.w / SAMPLE_DIV, ys = q.h / SAMPLE_DIV;
  int kx[SAMPLE_ROUNDS], ky[SAMPLE_ROUNDS], keep = 0;
  if (c < SAMPLE_CELLS) {
    const unsigned long long jump = rng_pow(2 * SAMPLE_CELLS - 2);
    unsigned long long s = rng_mulmod(rng_pow(2 * (unsigned long long)c), q.seed ? q.seed : 0xffffffffull);
#pragma unroll
    for (int r = 0; r < SAMPLE_ROUNDS; ++r) {
      kx[r] = ci * xs + (int)(rng_next(s) % (unsigned)xs);
      ky[r] = cj * ys + (int)(rng_next(s) % (unsigned)ys);
      if (kx[r] > 0 && ky[r] > 0) keep |= 1 << r;              // x < cols and y < rows hold by construction
      s = rng_mulmod(s, jump);
    }
  }
  // the reference stops at the SAMPLE_N-th acceptance in visit order (round-major, cell-minor)
  int base = 0;
#pragma unroll
  for (int r = 0; r < SAMPLE_ROUNDS; ++r) {
    int tot;
    const int pos = base + cta_excl_scan((keep >> r) & 1, wsum, tot);
    if (pos >= SAMPLE_N) keep &= ~(1 << r);
    base += tot;
  }
  int tot;
  int o = cta_excl_scan(__popc(keep), wsum, tot);               // cell-major output: exclusive scan of the per-cell counts
#pragma unroll
  for (int r = 0; r < SAMPLE_ROUNDS; ++r)
    if ((keep >> r) & 1) { q.kx[o] = (float)kx[r]; q.ky[o] = (float)ky[r]; ++o; }
}
__global__ void __launch_bounds__(SAMPLE_THREADS) k_sample_keys(const SampleKeysSeq* __restrict__ tab) { sample_keys_cta(tab[blockIdx.x]); }
// vdo_sample_keys_dev: frame i's seed from the device, its keys at row i of x / y (VDO_SAMPLE_KEYS per row), its count VDO_SAMPLE_KEYS
__global__ void __launch_bounds__(SAMPLE_THREADS) k_sample_keys_dev(const unsigned* __restrict__ seeds, float* __restrict__ x, float* __restrict__ y,
                                                                    int* __restrict__ count, int w, int h) {
  const size_t row = (size_t)blockIdx.x * SAMPLE_N;
  sample_keys_cta(SampleKeysSeq{seeds[blockIdx.x], x + row, y + row, w, h});
  if (threadIdx.x == 0) count[blockIdx.x] = SAMPLE_N;
}

// Dense packing of the per-cell candidate lists (cell-major, row-major inside a cell = the candidate order DistributeOctTree sees):
// k_cell_offsets: exclusive scan of the cell counts by one CTA; k_cell_gather: one CTA per cell copies its entries.
__global__ void __launch_bounds__(1024) k_cell_offsets(const int* __restrict__ count, int n, int* __restrict__ offset) {
  __shared__ int s[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < n ? count[i] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
      __syncthreads();
      s[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < n) offset[i] = carry + s[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += s[1023];
    __syncthreads();
  }
  if (threadIdx.x == 0) offset[n] = carry;
}
__global__ void k_cell_gather(const KpOut* __restrict__ cell_out, const int* __restrict__ count, const int* __restrict__ offset, KpOut* __restrict__ dense) {
  const int c = blockIdx.x, n = count[c], o = offset[c];
  for (int k = threadIdx.x; k < n; k += blockDim.x) dense[o + k] = cell_out[(size_t)c * CELL_CAP + k];
}

// ------------------------------------------------------------------------------------------------ back-projection / scene flow
struct Pose32 { float R[9], t[3]; };   // Tcw rows
// X_w = Rwl * x3Dc + twl as a cv::Mat float gemm: products accumulated in double, one rounding to float (twl itself is float)
__device__ __forceinline__ void unproject_world(float u, float v, float z, const float* K, const Pose32& T, float* X) {
  const float invfx = __fdiv_rn(1.f, K[0]), invfy = __fdiv_rn(1.f, K[1]);
  const float x = __fmul_rn(__fmul_rn(__fsub_rn(u, K[2]), z), invfx), y = __fmul_rn(__fmul_rn(__fsub_rn(v, K[3]), z), invfy);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double twl = (double)(float)(-((double)T.R[r] * (double)T.t[0] + (double)T.R[3 + r] * (double)T.t[1] + (double)T.R[6 + r] * (double)T.t[2]));
    X[r] = (float)((double)T.R[r] * (double)x + (double)T.R[3 + r] * (double)y + (double)T.R[6 + r] * (double)z + twl);
  }
}
struct FlowSeg { Pose32 Tp, Tc; float K[4]; int begin; };   // points [begin, next begin) of the launch are this sequence's
__global__ void k_scene_flow(int n, const FlowSeg* __restrict__ seg, int nseg, const float* __restrict__ up, const float* __restrict__ vp,
                             const float* __restrict__ zp, const float* __restrict__ uc, const float* __restrict__ vc, const float* __restrict__ zc,
                             const int* __restrict__ labp, const int* __restrict__ labc, float* __restrict__ flow3d, float* __restrict__ Xp_out,
                             unsigned char* __restrict__ valid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int s = 0;
  while (s + 1 < nseg && seg[s + 1].begin <= i) ++s;
  const Pose32 Tp = seg[s].Tp, Tc = seg[s].Tc;
  const float Kf[4] = {seg[s].K[0], seg[s].K[1], seg[s].K[2], seg[s].K[3]};
  float Xp[3], Xc[3];
  unproject_world(up[i], vp[i], zp[i], Kf, Tp, Xp);
  unproject_world(uc[i], vc[i], zc[i], Kf, Tc, Xc);
  const bool ok = labc[i] > 0 && labp[i] > 0;
  valid[i] = ok;
#pragma unroll
  for (int r = 0; r < 3; ++r) { flow3d[3 * i + r] = ok ? __fsub_rn(Xc[r], Xp[r]) : 0.f; if (Xp_out) Xp_out[3 * i + r] = Xp[r]; }
}

// vdo_obj_track_batch_dev's current look-up and scene flow, one thread per sample of pair blockIdx.y.  It lives here, next to k_scene_flow, so
// that unproject_world is compiled with this file's flags (--fmad=true: the double sums may contract to DFMA) and rounds as k_scene_flow does.
struct TrackFlowPair { PlaneArg dep, msk; int w, h; float K[4]; };
struct TrackFlowArg { const float *Tl, *Tc; int cap; float th; TrackFlowPair pr[VDO_OBJ_MOTION_MAX_PAIRS]; };
__device__ __forceinline__ Pose32 pose32_of(const float* T) {   // Tcw row-major, NULL: identity
  Pose32 P;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) P.R[3 * r + c] = T ? T[4 * r + c] : (r == c ? 1.f : 0.f);
    P.t[r] = T ? T[4 * r + 3] : 0.f;
  }
  return P;
}
__global__ void __launch_bounds__(256) k_ot_flow(const __grid_constant__ TrackFlowArg a, vdo_obj_track_out o, int* __restrict__ pstat, int* __restrict__ glab) {
  const int p = blockIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= o.motion.n_samples_dev[p]) return;
  const TrackFlowPair& q = a.pr[p];
  const size_t i = (size_t)p * a.cap + k;
  const float cx = o.motion.sample_cx_dev[i], cy = o.motion.sample_cy_dev[i];
  const int u = (int)cx, v = (int)cy;            // Tracking.cc:288-305 (tracker.cpp's look-up)
  float dc = 0.1f;
  int lc = 0;
  if (u < q.w - 1 && u > 0 && v < q.h - 1 && v > 0) {
    const float d = plane_depth(q.dep, u, v);
    if (d < a.th && d > 0.f) {
      int bad = 0;
      dc = d; lc = plane_label(q.msk, u, v, &bad);
      if (bad) atomicOr(pstat + p, VDO_OM_PAIR_LABEL_RANGE);
    }
  }
  const float Kf[4] = {q.K[0], q.K[1], q.K[2], q.K[3]};
  float Xp[3], Xc[3];
  unproject_world((float)o.motion.sample_x_dev[i], (float)o.motion.sample_y_dev[i], o.motion.sample_depth_dev[i], Kf, pose32_of(a.Tl ? a.Tl + 16 * p : nullptr), Xp);
  unproject_world(cx, cy, dc, Kf, pose32_of(a.Tc ? a.Tc + 16 * p : nullptr), Xc);
  const bool ok = lc > 0 && o.motion.sample_label_dev[i] > 0;
#pragma unroll
  for (int r = 0; r < 3; ++r) o.flow3d_dev[3 * i + r] = ok ? __fsub_rn(Xc[r], Xp[r]) : 0.f;
  o.label_cur_dev[i] = lc; o.depth_cur_dev[i] = dc;
  glab[i] = ok ? lc : 0;                          // the grouping label: 0 leaves the sample out of every object
}

// ------------------------------------------------------------------------------------------------ host side
struct OrbSetup {
  int nfeatures = 0, nlevels = 0, ini_th = 0, min_th = 0;
  float scale_factor[MAX_LEVELS], inv_scale[MAX_LEVELS];
  int per_level[MAX_LEVELS];
  int umax[16];
  void init(int nf, float sf, int nl, int ini, int mn) {
    nfeatures = nf; nlevels = nl; ini_th = ini; min_th = mn;
    scale_factor[0] = 1.f;
    for (int i = 1; i < nl; ++i) scale_factor[i] = scale_factor[i - 1] * sf;
    for (int i = 0; i < nl; ++i) inv_scale[i] = 1.f / scale_factor[i];
    float factor = 1.f / sf;
    float nd = nf * (1 - factor) / (1 - (float)std::pow((double)factor, (double)nl));
    int sum = 0;
    for (int l = 0; l < nl - 1; ++l) { per_level[l] = (int)std::lrint(nd); sum += per_level[l]; nd *= factor; }
    per_level[nl - 1] = std::max(nf - sum, 0);
    int vmax = (int)std::floor(HALF_PATCH * std::sqrt(2.f) / 2 + 1), vmin = (int)std::ceil(HALF_PATCH * std::sqrt(2.f) / 2);
    const double hp2 = HALF_PATCH * HALF_PATCH;
    for (int v = 0; v <= vmax; ++v) umax[v] = (int)std::lrint(std::sqrt(hp2 - v * v));
    for (int v = HALF_PATCH, v0 = 0; v >= vmin; --v) { while (umax[v0] == umax[v0 + 1]) ++v0; umax[v] = v0; ++v0; }
  }
};

}  // namespace

// ================================================================================================ C ABI

// ------------------------------------------------------------------------------------------------ descriptors (A6)
// GaussianBlur(level, Size(7,7), 2, 2, BORDER_REFLECT_101) as OpenCV computes it for CV_8U (fixed point, bit-exact against cv2 4.13):
// Q8.8 kernel {18, 34, 48, 56, 48, 34, 18} / 256, horizontal pass kept in Q8.8, vertical pass in Q16.16, (v + 2^15) >> 16.
// (src/ORBextractor.cc:1083-1084.  OpenCV 3.4.0, which the reference's Dockerfile builds, still filtered in float: version drift.)
// cv::borderInterpolate(BORDER_REFLECT_101): reflect until inside, so that levels of 1 to 3 px (where a 3-px reach crosses the image more
// than once) read what OpenCV reads; a 1-px line is constant
__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}
__device__ __forceinline__ unsigned char blur7_px(const unsigned char* __restrict__ src, int w, int h, int x, int y) {
  const int kq[7] = {18, 34, 48, 56, 48, 34, 18};
  int xs[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) xs[i] = reflect101(x + i - 3, w);
  unsigned int v = 0;
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    const unsigned char* row = src + (size_t)reflect101(y + j - 3, h) * w;
    unsigned int hsum = 0;
#pragma unroll
    for (int i = 0; i < 7; ++i) hsum += (unsigned int)kq[i] * row[xs[i]];
    v += (unsigned int)kq[j] * hsum;
  }
  return (unsigned char)((v + (1u << 15)) >> 16);
}
// computeOrbDescriptor (src/ORBextractor.cc:97-136): one warp per keypoint, one descriptor byte (8 pair tests) per lane.
__constant__ signed char c_orb_pattern[1024] = {
#include "orb_pattern.inc"
};
struct BlurLevels { const unsigned char* img[MAX_LEVELS]; int w[MAX_LEVELS], h[MAX_LEVELS]; };
// descriptor byte `lane` (pair tests 8 lane .. 8 lane + 7) of keypoint kp at angle ang_deg on its blurred level img (row stride w)
__device__ __forceinline__ unsigned char orb_desc_byte(const unsigned char* __restrict__ img, int w, const KpLvl& kp, float ang_deg, int lane) {
  const float factorPI = (float)(3.14159265358979323846 / 180.f);
  const float angle = __fmul_rn(ang_deg, factorPI);
  const float a = (float)cos((double)angle), b = (float)sin((double)angle);
  const unsigned char* center = img + (size_t)__float2int_rn(kp.y) * w + __float2int_rn(kp.x);
  int val = 0;
#pragma unroll
  for (int bit = 0; bit < 8; ++bit) {
    const signed char* pt = c_orb_pattern + 4 * (8 * lane + bit);
    int t[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const float px = (float)pt[2 * q], py = (float)pt[2 * q + 1];
      const int iy = __float2int_rn(__fadd_rn(__fmul_rn(px, b), __fmul_rn(py, a)));
      const int ix = __float2int_rn(__fsub_rn(__fmul_rn(px, a), __fmul_rn(py, b)));
      t[q] = center[iy * w + ix];
    }
    val |= (t[0] < t[1]) << bit;
  }
  return (unsigned char)val;
}

namespace vdo {
bool OrbKey::operator<(const OrbKey& o) const {
  return std::tie(w, h, nfeatures, scale_factor, nlevels, ini_th, min_th) < std::tie(o.w, o.h, o.nfeatures, o.scale_factor, o.nlevels, o.ini_th, o.min_th);
}
bool OrbKey::operator==(const OrbKey& o) const { return !(*this < o) && !(o < *this); }
int orb_create(vdo_ctx* ctx, const std::vector<OrbKey>& keys, const std::vector<int>& slots, int max_batch, vdo_orb_extractor** out);
void orb_extractor_info(const vdo_orb_extractor* ex, int* cap, int* nlevels);
// An extractor with device outputs (vdo_orb_batch_out) for max_batch frames.  The outputs of a call of n frames are packed in the order
// x, y, count, status (the tracker's read-back), octave, response, angle, size, n_candidates (vdo_orb_extract's), descriptors.  Frame i's
// keypoints start at i * cap, cap being the largest keypoint capacity of the extractor's geometries.
struct OrbJob {
  vdo_orb_extractor* ex = nullptr;
  std::vector<OrbKey> keys; std::vector<int> slots;             // the extractor's geometries and the frames each holds
  int max_batch = 0, cap = 0, nlevels = 0; bool desc = false;
  char* buf = nullptr;
  bool same(const OrbKey& k) const { return ex && keys.size() == 1 && keys[0] == k; }
  void release() { vdo_orb_extractor_destroy(ex); cudaFree(buf); ex = nullptr; buf = nullptr; max_batch = 0; keys.clear(); slots.clear(); }
  // VDO_ERR_ARG / VDO_ERR_UNSUPPORTED for the settings vdo_orb_extractor_create refuses
  int create(vdo_ctx* ctx, const std::vector<OrbKey>& k, const std::vector<int>& s, int batch, bool with_desc) {
    release();
    if (int rc = orb_create(ctx, k, s, batch, &ex)) return rc;
    orb_extractor_info(ex, &cap, &nlevels);
    keys = k; slots = s; desc = with_desc;
    if (cudaMalloc(&buf, keys_bytes(batch) + (desc ? (size_t)batch * cap * 32 : 0)) != cudaSuccess) { cudaGetLastError(); release(); return VDO_ERR_CUDA; }
    max_batch = batch;
    return VDO_OK;
  }
  size_t head_bytes(int n) const { return sizeof(int) * ((size_t)2 * n * cap + 2 * n); }
  size_t keys_bytes(int n) const { return sizeof(int) * ((size_t)6 * n * cap + 2 * n + (size_t)n * nlevels); }
  // the layout of a call of n frames at `base` (buf, or a host copy of it)
  vdo_orb_batch_out outs(int n, void* base) const {
    const size_t m = (size_t)n * cap;
    vdo_orb_batch_out o;
    o.x_dev = (float*)base; o.y_dev = o.x_dev + m; o.count_dev = (int32_t*)(o.y_dev + m); o.status_dev = o.count_dev + n;
    o.octave_dev = o.status_dev + n; o.response_dev = (float*)(o.octave_dev + m); o.angle_dev = o.response_dev + m; o.size_dev = (int32_t*)(o.angle_dev + m);
    o.n_candidates_dev = o.size_dev + m;
    o.desc_dev = desc ? (uint8_t*)(o.n_candidates_dev + (size_t)n * nlevels) : nullptr;
    return o;
  }
};
}  // namespace vdo

struct vdo_frame {
  vdo_ctx* ctx; cudaStream_t st;
  int w, h;
  unsigned char* gray = nullptr; float* depth = nullptr; float* flow = nullptr; int* mask = nullptr;
  vdo::OrbJob orb;                                                 // vdo_orb_extract's extractor (max_batch 1), made on first use
  int orb_count = -1;                                              // keypoints of the last vdo_orb_extract that returned angles, else -1
  bool orb_blurred = false;                                        // vdo_orb_describe has blurred the extractor's levels
  int dev = -1;                                                    // device of the resident buffers (= the context's)
  cudaEvent_t ev_in = nullptr;                                     // device ingest: caller-stream event
};

namespace {
// Per-stream workspace of the batched stages: per-launch tables, ingest flags and the outputs of the point-list kernels.  Every stage
// synchronises the context stream before its caller reads the results, and the next stage's table upload is ordered after the kernels
// that read the previous one, so one stage's buffers are free for the next.
struct BatchWs {
  char* tab = nullptr; size_t tab_cap = 0;
  int* flags = nullptr; int flags_cap = 0;
  char* out = nullptr; size_t out_cap = 0;
  int* counts = nullptr; int counts_cap = 0;
};
std::mutex g_ws_mu;
std::map<cudaStream_t, BatchWs> g_ws;
BatchWs& ws_of(cudaStream_t st) { std::lock_guard<std::mutex> lk(g_ws_mu); return g_ws[st]; }
// the extractors of the tracker's frame build, one per (stream, set of distinct image sizes with ORB settings), under g_ws_mu
// (vdo::orb_job_for)
std::map<std::pair<cudaStream_t, std::vector<vdo::OrbKey>>, vdo::OrbJob> g_orb;

template <class T> int grow_dev(T*& p, size_t& cap, size_t need) {
  if (need <= cap) return VDO_OK;
  cudaFree(p); p = nullptr; cap = 0;
  VDO_CUDA(cudaMalloc(&p, sizeof(T) * need * 2));
  cap = need * 2;
  return VDO_OK;
}
template <class T> int grow_dev(T*& p, int& cap, size_t need) { size_t c = (size_t)cap; const int rc = grow_dev(p, c, need); cap = (int)c; return rc; }

// host image of one upload of per-launch tables: entries added at 16-byte aligned offsets, one H2D copy, device pointers by offset
struct Tabs {
  std::vector<char> h;
  template <class T> size_t add(const T* v, size_t n) {
    const size_t o = (h.size() + 15) & ~(size_t)15;
    h.resize(o + sizeof(T) * n);
    if (n) std::memcpy(h.data() + o, v, sizeof(T) * n);
    return o;
  }
  template <class T> size_t add(const std::vector<T>& v) { return add(v.data(), v.size()); }
  int upload(BatchWs& W, cudaStream_t st) {
    if (int rc = grow_dev(W.tab, W.tab_cap, h.size() + 16)) return rc;
    VDO_CUDA(cudaMemcpyAsync(W.tab, h.data(), h.size(), cudaMemcpyHostToDevice, st));
    return VDO_OK;
  }
  template <class T> static const T* at(const BatchWs& W, size_t o) { return (const T*)(W.tab + o); }
};
}  // namespace

extern "C" int vdo_frame_create(vdo_ctx* ctx, int width, int height, vdo_frame** out) {
  if (!ctx || !out || width < 64 || height < 64) return VDO_ERR_ARG;
  vdo_frame* f = new vdo_frame;
  f->ctx = ctx; f->st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx); f->w = width; f->h = height;
  const size_t n = (size_t)width * height;
  VDO_CUDA(cudaMalloc(&f->gray, n)); VDO_CUDA(cudaMalloc(&f->depth, n * 4)); VDO_CUDA(cudaMalloc(&f->flow, n * 8)); VDO_CUDA(cudaMalloc(&f->mask, n * 4));
  VDO_CUDA(cudaEventCreateWithFlags(&f->ev_in, cudaEventDisableTiming));
  cudaPointerAttributes a;
  VDO_CUDA(cudaPointerGetAttributes(&a, f->gray));
  f->dev = a.device;
  *out = f;
  return VDO_OK;
}
extern "C" void vdo_frame_destroy(vdo_frame* f) {
  if (!f) return;
  cudaFree(f->gray); cudaFree(f->depth); cudaFree(f->flow); cudaFree(f->mask);
  if (f->ev_in) cudaEventDestroy(f->ev_in);
  f->orb.release();
  delete f;
}
// D2H of the resident mask (the tracker writes it back into the caller's buffer only when UpdateMask changed it)
extern "C" int vdo_frame_read_mask(vdo_frame* f, int* mask_out) {
  if (!f || !mask_out) return VDO_ERR_ARG;
  VDO_CUDA(cudaMemcpyAsync(mask_out, f->mask, sizeof(int) * (size_t)f->w * f->h, cudaMemcpyDeviceToHost, f->st));
  VDO_CUDA(cudaStreamSynchronize(f->st));
  return VDO_OK;
}
// internal: device pointers of a resident frame for the other translation units (tracking_ops.cu)
extern "C" int vdo_frame_device_ptrs(vdo_frame* f, unsigned char** gray, float** depth, float** flow, int** mask, int* w, int* h, void** stream) {
  if (!f) return VDO_ERR_ARG;
  if (gray) *gray = f->gray; if (depth) *depth = f->depth; if (flow) *flow = f->flow; if (mask) *mask = f->mask;
  if (w) *w = f->w; if (h) *h = f->h; if (stream) *stream = (void*)f->st;
  return VDO_OK;
}
// any of the four pointers may be NULL (keep what is resident)
extern "C" int vdo_frame_upload(vdo_frame* f, const unsigned char* gray, const float* depth, const float* flow, const int* mask) {
  if (!f) return VDO_ERR_ARG;
  const size_t n = (size_t)f->w * f->h;
  if (gray) VDO_CUDA(cudaMemcpyAsync(f->gray, gray, n, cudaMemcpyHostToDevice, f->st));
  if (depth) VDO_CUDA(cudaMemcpyAsync(f->depth, depth, n * 4, cudaMemcpyHostToDevice, f->st));
  if (flow) VDO_CUDA(cudaMemcpyAsync(f->flow, flow, n * 8, cudaMemcpyHostToDevice, f->st));
  if (mask) VDO_CUDA(cudaMemcpyAsync(f->mask, mask, n * 4, cudaMemcpyHostToDevice, f->st));
  return VDO_OK;
}

// ---- device ingest (vdo_dev_plane).  Shared by vdo_frame_upload_dev and the tracker, which needs its three steps apart:
// check + enqueue, then (after depth prep) the wait that reports the label-range flags, and the write-back once UpdateMask has run.
namespace vdo {
int check_dev_ptr(const void* p, int dev, const std::string& who, std::string& err) {
  cudaPointerAttributes a;
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) cudaGetLastError();
  if (e != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != dev) {
    err = who + " is not device memory of device " + std::to_string(dev) +
          (e != cudaSuccess ? std::string(" (") + cudaGetErrorString(e) + ")"
                            : " (memory type " + std::to_string((int)a.type) + " on device " + std::to_string(a.device) + ")");
    return VDO_ERR_ARG;
  }
  return VDO_OK;
}

// planes: image, depth, flow, mask (any may be NULL); target[k]: plane k will also be written back
int frame_check_planes(const vdo_frame* f, const vdo_dev_plane* const planes[4], const bool target[4], std::string& err) {
  static const char* kName[4] = {"image", "depth", "flow", "mask"};
  for (int k = 0; k < 4; ++k) {
    const vdo_dev_plane* pl = planes[k];
    if (!pl) continue;
    const std::string who = std::string(kName[k]) + " plane: ";
    const int dt = pl->dtype, ch = pl->channels;
    const bool shape_ok = k == 0 ? (dt == VDO_DT_U8 && (ch == 1 || ch == 3 || ch == 4))
                        : k == 1 ? (dt == VDO_DT_F32 && ch == 1)
                        : k == 2 ? (dt == VDO_DT_F32 && ch == 2)
                                 : ((dt == VDO_DT_I32 || dt == VDO_DT_I64) && ch == 1);
    if (!shape_ok) {
      static const char* kWant[4] = {"u8 with 1, 3 or 4 channels", "f32 with 1 channel", "f32 with 2 channels", "i32 or i64 with 1 channel"};
      err = who + "dtype " + std::to_string(dt) + " with " + std::to_string(ch) + " channels; expected " + kWant[k];
      return VDO_ERR_ARG;
    }
    const size_t es = dt == VDO_DT_U8 ? 1 : dt == VDO_DT_I64 ? 8 : 4;
    if (!pl->data_dev || (uintptr_t)pl->data_dev % es) { err = who + "data_dev is NULL or not aligned to its element size"; return VDO_ERR_ARG; }
    if (target && target[k] && (pl->stride_x == 0 || pl->stride_y == 0)) { err = who + "a write-back target needs non-zero stride_x and stride_y"; return VDO_ERR_ARG; }
    if (int rc = check_dev_ptr(pl->data_dev, f->dev, who + "data_dev", err)) return rc;
  }
  return VDO_OK;
}
// one k_ingest_frame launch over the n frames, on the context stream after everything queued so far on the caller's stream; planes
// already checked
int frames_ingest_dev(vdo_frame* const* fs, int n, const vdo_dev_plane* const* planes, uint64_t stream) {
  vdo_frame* f0 = fs[0];
  BatchWs& W = ws_of(f0->st);
  VDO_CUDA(cudaEventRecord(f0->ev_in, (cudaStream_t)(uintptr_t)stream));
  VDO_CUDA(cudaStreamWaitEvent(f0->st, f0->ev_in, 0));
  if (int rc = grow_dev(W.flags, W.flags_cap, (size_t)n)) return rc;
  VDO_CUDA(cudaMemsetAsync(W.flags, 0, sizeof(int) * n, f0->st));
  std::vector<IngestSeq> q(n);
  for (int i = 0; i < n; ++i) {
    vdo_frame* f = fs[i];
    const vdo_dev_plane* const* pl = planes + 4 * i;
    q[i] = IngestSeq{plane_arg(pl[0]), plane_arg(pl[1]), plane_arg(pl[2]), plane_arg(pl[3]), f->gray, f->depth, (float2*)f->flow, f->mask, W.flags + i, f->w, f->h};
  }
  Tabs T;
  const size_t o = T.add(q);
  if (int rc = T.upload(W, f0->st)) return rc;
  int mw = 0, mh = 0;
  for (int i = 0; i < n; ++i) { mw = std::max(mw, fs[i]->w); mh = std::max(mh, fs[i]->h); }
  dim3 b(32, 8), g((mw + 31) / 32, (mh + 7) / 8, n);
  k_ingest_frame<<<g, b, 0, f0->st>>>(Tabs::at<IngestSeq>(W, o));
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
int frames_ingest_wait(vdo_frame* const* fs, int n, int* bad, std::string& err) {
  BatchWs& W = ws_of(fs[0]->st);
  std::vector<int> h(n, 0);
  VDO_CUDA(cudaMemcpyAsync(h.data(), W.flags, sizeof(int) * n, cudaMemcpyDeviceToHost, fs[0]->st));
  VDO_CUDA(cudaStreamSynchronize(fs[0]->st));
  for (int i = 0; i < n; ++i)
    if (h[i]) { if (bad) *bad = i; err = "mask plane: an i64 label lies outside the int32 range"; return VDO_ERR_ARG; }
  return VDO_OK;
}
// resident depth (and mask, when given) -> the caller's planes, enqueued on the context stream; planes already checked as targets
int frame_writeback_dev(vdo_frame* f, const vdo_dev_plane* depth, const vdo_dev_plane* mask) {
  if (!depth && !mask) return VDO_OK;
  dim3 b(32, 8), g((f->w + 31) / 32, (f->h + 7) / 8);
  k_writeback_frame<<<g, b, 0, f->st>>>(f->depth, f->mask, f->w, f->h, plane_arg(depth), plane_arg(mask));
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
int frames_depth_prep(vdo_frame* const* fs, int n, const float* bf, const float* factor) {
  vdo_frame* f0 = fs[0];
  BatchWs& W = ws_of(f0->st);
  std::vector<DepthSeq> q(n);
  int npx = 0;
  for (int i = 0; i < n; ++i) { q[i] = DepthSeq{fs[i]->depth, bf[i], factor[i], fs[i]->w * fs[i]->h}; npx = std::max(npx, q[i].n); }
  Tabs T;
  const size_t o = T.add(q);
  if (int rc = T.upload(W, f0->st)) return rc;
  k_depth_prep<<<dim3((npx + 255) / 256, n), 256, 0, f0->st>>>(Tabs::at<DepthSeq>(W, o));
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}

// the static filter of n frames: one k_sample_keys launch over the sampling frames (one CTA per frame) when there are any, one
// k_filter_static launch (one CTA per frame), one read-back of the counts, one of the kept keys and the samples
int filter_static_batch(vdo_frame* const* fs, int n, const float* const* kx, const float* const* ky, const int* nk, const float* th, const long long* seed,
                        StaticKeys* out) {
  vdo_frame* f0 = fs[0];
  const cudaStream_t st = f0->st;
  BatchWs& W = ws_of(st);
  std::vector<size_t> beg(n + 1, 0);
  for (int i = 0; i < n; ++i) beg[i + 1] = beg[i] + (size_t)(seed && seed[i] >= 0 ? SAMPLE_N : nk[i]);
  const size_t tot = beg[n];
  for (int i = 0; i < n; ++i) {
    StaticKeys& o = out[i];
    o.idx.clear(); o.cx.clear(); o.cy.clear(); o.fu.clear(); o.fv.clear(); o.depth.clear(); o.kx.clear(); o.ky.clear();
  }
  if (tot == 0) return VDO_OK;
  if (int rc = grow_dev(W.out, W.out_cap, (sizeof(float) * 2 + sizeof(StatOut)) * tot + 64)) return rc;
  if (int rc = grow_dev(W.counts, W.counts_cap, (size_t)n)) return rc;
  float* d_k = (float*)W.out; StatOut* d_out = (StatOut*)(d_k + 2 * tot);
  std::vector<float> hk(2 * tot);
  std::vector<StaticSeq> q(n);
  std::vector<SampleKeysSeq> sq;
  for (int i = 0; i < n; ++i) {
    const bool samp = seed && seed[i] >= 0;
    if (samp) sq.push_back(SampleKeysSeq{(unsigned)seed[i], d_k + beg[i], d_k + tot + beg[i], fs[i]->w, fs[i]->h});
    else if (nk[i]) { std::memcpy(&hk[beg[i]], kx[i], sizeof(float) * nk[i]); std::memcpy(&hk[tot + beg[i]], ky[i], sizeof(float) * nk[i]); }
    q[i] = StaticSeq{d_k + beg[i], d_k + tot + beg[i], (int)(beg[i + 1] - beg[i]), th[i], samp ? 1 : 0, fs[i]->mask, fs[i]->depth, fs[i]->flow, d_out + beg[i],
                     W.counts + i, fs[i]->w, fs[i]->h};
  }
  if (sq.size() < (size_t)n) VDO_CUDA(cudaMemcpyAsync(d_k, hk.data(), sizeof(float) * 2 * tot, cudaMemcpyHostToDevice, st));
  Tabs T;
  const size_t o = T.add(q), os = T.add(sq);
  if (int rc = T.upload(W, st)) return rc;
  if (!sq.empty()) {
    k_sample_keys<<<(unsigned)sq.size(), SAMPLE_THREADS, 0, st>>>(Tabs::at<SampleKeysSeq>(W, os));
    VDO_CUDA(cudaGetLastError());
  }
  k_filter_static<<<n, 1024, 0, st>>>(Tabs::at<StaticSeq>(W, o));
  VDO_CUDA(cudaGetLastError());
  std::vector<int> m(n);
  VDO_CUDA(cudaMemcpyAsync(m.data(), W.counts, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  std::vector<StatOut> h(tot);
  bool any = false;
  for (int i = 0; i < n; ++i) {
    if (m[i]) { any = true; VDO_CUDA(cudaMemcpyAsync(&h[beg[i]], d_out + beg[i], sizeof(StatOut) * m[i], cudaMemcpyDeviceToHost, st)); }
    if (seed && seed[i] >= 0) {
      any = true;
      out[i].kx.resize(SAMPLE_N); out[i].ky.resize(SAMPLE_N);
      VDO_CUDA(cudaMemcpyAsync(out[i].kx.data(), d_k + beg[i], sizeof(float) * SAMPLE_N, cudaMemcpyDeviceToHost, st));
      VDO_CUDA(cudaMemcpyAsync(out[i].ky.data(), d_k + tot + beg[i], sizeof(float) * SAMPLE_N, cudaMemcpyDeviceToHost, st));
    }
  }
  if (any) VDO_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    StaticKeys& o = out[i];
    const StatOut* r = &h[beg[i]];
    o.idx.resize(m[i]); o.cx.resize(m[i]); o.cy.resize(m[i]); o.fu.resize(m[i]); o.fv.resize(m[i]); o.depth.resize(m[i]);
    for (int k = 0; k < m[i]; ++k) { o.idx[k] = r[k].idx; o.cx[k] = r[k].cx; o.cy[k] = r[k].cy; o.fu[k] = r[k].fu; o.fv[k] = r[k].fv; o.depth[k] = r[k].depth; }
  }
  return VDO_OK;
}

// object samples of n frames: one k_sample_objects launch (one CTA per frame), one read-back of the counts, one of the samples
int sample_objects_batch(vdo_frame* const* fs, int n, const float* th, int step, const int* cap, ObjSamples* out) {
  vdo_frame* f0 = fs[0];
  const cudaStream_t st = f0->st;
  BatchWs& W = ws_of(st);
  std::vector<size_t> beg(n + 1, 0);
  for (int i = 0; i < n; ++i) beg[i + 1] = beg[i] + (size_t)cap[i];
  if (int rc = grow_dev(W.out, W.out_cap, sizeof(ObjSample) * beg[n] + 64)) return rc;
  if (int rc = grow_dev(W.counts, W.counts_cap, (size_t)n)) return rc;
  ObjSample* d_out = (ObjSample*)W.out;
  std::vector<SampleSeq> q(n);
  for (int i = 0; i < n; ++i) q[i] = SampleSeq{fs[i]->mask, fs[i]->depth, fs[i]->flow, th[i], d_out + beg[i], W.counts + i, fs[i]->w, fs[i]->h, cap[i]};
  Tabs T;
  const size_t o = T.add(q);
  if (int rc = T.upload(W, st)) return rc;
  k_sample_objects<<<n, 1024, 0, st>>>(Tabs::at<SampleSeq>(W, o), step);
  VDO_CUDA(cudaGetLastError());
  std::vector<int> m(n);
  VDO_CUDA(cudaMemcpyAsync(m.data(), W.counts, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  std::vector<std::vector<ObjSample>> h(n);
  bool any = false;
  for (int i = 0; i < n; ++i) {
    h[i].resize(m[i]);
    if (m[i]) { any = true; VDO_CUDA(cudaMemcpyAsync(h[i].data(), d_out + beg[i], sizeof(ObjSample) * m[i], cudaMemcpyDeviceToHost, st)); }
  }
  if (any) VDO_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    ObjSamples& s = out[i];
    const int k = m[i];
    s.x.resize(k); s.y.resize(k); s.label.resize(k); s.cx.resize(k); s.cy.resize(k); s.fx.resize(k); s.fy.resize(k); s.depth.resize(k);
    for (int j = 0; j < k; ++j) {
      const ObjSample& r = h[i][j];
      s.x[j] = r.x; s.y[j] = r.y; s.cx[j] = r.cx; s.cy[j] = r.cy; s.fx[j] = r.fx; s.fy[j] = r.fy; s.depth[j] = r.depth; s.label[j] = r.label;
    }
  }
  return VDO_OK;
}

void obj_track_flow_launch(int P, const vdo_dev_plane* depth_cur, const vdo_dev_plane* mask_cur, const int32_t* wh, const float* K, const float* Tcw_last,
                           const float* Tcw_cur, int cap, int max_n, float th_depth_obj, const vdo_obj_track_out& out, int* pstat, int* glab, uint64_t stream) {
  TrackFlowArg a;
  std::memset(&a, 0, sizeof a);
  a.Tl = Tcw_last; a.Tc = Tcw_cur; a.cap = cap; a.th = th_depth_obj;
  for (int p = 0; p < P; ++p) {
    TrackFlowPair& q = a.pr[p];
    q.dep = plane_arg(&depth_cur[p]); q.msk = plane_arg(&mask_cur[p]); q.w = wh[2 * p]; q.h = wh[2 * p + 1];
    for (int c = 0; c < 4; ++c) q.K[c] = K[4 * p + c];
  }
  k_ot_flow<<<dim3((std::max(max_n, 1) + 255) / 256, P), 256, 0, (cudaStream_t)(uintptr_t)stream>>>(a, out, pstat, glab);
}

// scene flow of nseg point segments, one launch; the context stream is synchronised before it returns
int scene_flow_batch(vdo_ctx* ctx, int nseg, const int* begin, const float* Tcw_prev, const float* Tcw_cur, const float* K, const float* u_prev,
                     const float* v_prev, const float* z_prev, const float* u_cur, const float* v_cur, const float* z_cur, const int* label_prev,
                     const int* label_cur, float* flow3d, float* Xw_prev, unsigned char* valid) {
  const int n = begin[nseg];
  if (n == 0) return VDO_OK;
  cudaStream_t st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx);
  BatchWs& W = ws_of(st);
  const size_t fl = (size_t)n;
  if (int rc = grow_dev(W.out, W.out_cap, fl * 4 * (6 + 2 + 3 + 3) + fl + 64)) return rc;
  float* d = (float*)W.out;
  float *up = d, *vp = up + fl, *zp = vp + fl, *uc = zp + fl, *vc = uc + fl, *zc = vc + fl;
  int *lp = (int*)(zc + fl), *lc = lp + fl;
  float *df = (float*)(lc + fl), *dx = df + 3 * fl;
  unsigned char* dv = (unsigned char*)(dx + 3 * fl);
  const float* hs[6] = {u_prev, v_prev, z_prev, u_cur, v_cur, z_cur};
  for (int k = 0; k < 6; ++k) VDO_CUDA(cudaMemcpyAsync(d + k * fl, hs[k], fl * 4, cudaMemcpyHostToDevice, st));
  VDO_CUDA(cudaMemcpyAsync(lp, label_prev, fl * 4, cudaMemcpyHostToDevice, st));
  VDO_CUDA(cudaMemcpyAsync(lc, label_cur, fl * 4, cudaMemcpyHostToDevice, st));
  std::vector<FlowSeg> seg(nseg);
  for (int s = 0; s < nseg; ++s) {
    FlowSeg& q = seg[s];
    const float* Tp = Tcw_prev + 16 * s; const float* Tc = Tcw_cur + 16 * s;
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) { q.Tp.R[3 * r + c] = Tp[4 * r + c]; q.Tc.R[3 * r + c] = Tc[4 * r + c]; } q.Tp.t[r] = Tp[4 * r + 3]; q.Tc.t[r] = Tc[4 * r + 3]; }
    for (int k = 0; k < 4; ++k) q.K[k] = K[4 * s + k];
    q.begin = begin[s];
  }
  Tabs T;
  const size_t o = T.add(seg);
  if (int rc = T.upload(W, st)) return rc;
  k_scene_flow<<<(n + 255) / 256, 256, 0, st>>>(n, Tabs::at<FlowSeg>(W, o), nseg, up, vp, zp, uc, vc, zc, lp, lc, df, dx, dv);
  VDO_CUDA(cudaGetLastError());
  VDO_CUDA(cudaMemcpyAsync(flow3d, df, fl * 12, cudaMemcpyDeviceToHost, st));
  if (Xw_prev) VDO_CUDA(cudaMemcpyAsync(Xw_prev, dx, fl * 12, cudaMemcpyDeviceToHost, st));
  if (valid) VDO_CUDA(cudaMemcpyAsync(valid, dv, fl, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  return VDO_OK;
}
}  // namespace vdo

extern "C" int vdo_frame_upload_dev(vdo_frame* f, const vdo_dev_plane* image, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
                                    uint64_t stream) {
  if (!f) return VDO_ERR_ARG;
  const vdo_dev_plane* planes[4] = {image, depth, flow, mask};
  if (!image && !depth && !flow && !mask) return VDO_OK;
  std::string err;
  int rc = vdo::frame_check_planes(f, planes, nullptr, err);
  if (rc == VDO_OK) rc = vdo::frames_ingest_dev(&f, 1, planes, stream);
  if (rc == VDO_OK) rc = vdo::frames_ingest_wait(&f, 1, nullptr, err);
  if (rc != VDO_OK && !err.empty()) vdo::ctx_set_error(f->ctx, "vdo_frame_upload_dev: " + err);
  return rc;
}
extern "C" int vdo_frame_depth_prep(vdo_frame* f, float bf, float factor, float* depth_out) {
  if (!f) return VDO_ERR_ARG;
  if (int rc = vdo::frames_depth_prep(&f, 1, &bf, &factor)) return rc;
  if (depth_out) { VDO_CUDA(cudaMemcpyAsync(depth_out, f->depth, (size_t)f->w * f->h * 4, cudaMemcpyDeviceToHost, f->st)); VDO_CUDA(cudaStreamSynchronize(f->st)); }
  return VDO_OK;
}

extern "C" int vdo_frame_sample_objects(vdo_frame* f, float th_depth_obj, int step, int max_out, int* x, int* y, float* cx, float* cy,
                                        float* fx, float* fy, float* depth, int* label, int* n_out) {
  if (!f || step < 1 || max_out < 0 || !n_out) return VDO_ERR_ARG;
  vdo::ObjSamples s;
  if (int rc = vdo::sample_objects_batch(&f, 1, &th_depth_obj, step, &max_out, &s)) return rc;
  const int n = (int)s.x.size();
  for (int i = 0; i < n; ++i) { x[i] = s.x[i]; y[i] = s.y[i]; cx[i] = s.cx[i]; cy[i] = s.cy[i]; fx[i] = s.fx[i]; fy[i] = s.fy[i]; depth[i] = s.depth[i]; label[i] = s.label[i]; }
  *n_out = n;
  return VDO_OK;
}

extern "C" int vdo_frame_filter_static(vdo_frame* f, int n, const float* kx, const float* ky, float th_depth, int* keep_idx, float* cx, float* cy,
                                       float* fu, float* fv, float* depth, int* n_out) {
  if (!f || n < 0 || !n_out) return VDO_ERR_ARG;
  if (n == 0) { *n_out = 0; return VDO_OK; }
  vdo::StaticKeys s;
  if (int rc = vdo::filter_static_batch(&f, 1, &kx, &ky, &n, &th_depth, nullptr, &s)) return rc;
  const int m = (int)s.idx.size();
  for (int i = 0; i < m; ++i) { keep_idx[i] = s.idx[i]; cx[i] = s.cx[i]; cy[i] = s.cy[i]; fu[i] = s.fu[i]; fv[i] = s.fv[i]; depth[i] = s.depth[i]; }
  *n_out = m;
  return VDO_OK;
}

extern "C" int vdo_sample_keys(vdo_ctx* ctx, int n, int width, int height, const unsigned* seeds, float* kx, float* ky, float* kernel_ms) {
  if (!ctx || n < 1 || width < 20 || height < 20 || !seeds || !kx || !ky) return VDO_ERR_ARG;
  const cudaStream_t st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx);
  BatchWs& W = ws_of(st);
  const size_t tot = (size_t)SAMPLE_N * n;
  if (int rc = grow_dev(W.out, W.out_cap, sizeof(float) * 2 * tot + 64)) return rc;
  float* d = (float*)W.out;
  std::vector<SampleKeysSeq> sq(n);
  for (int i = 0; i < n; ++i) sq[i] = SampleKeysSeq{seeds[i], d + (size_t)SAMPLE_N * i, d + tot + (size_t)SAMPLE_N * i, width, height};
  Tabs T;
  const size_t o = T.add(sq);
  if (int rc = T.upload(W, st)) return rc;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  if (kernel_ms) { VDO_CUDA(cudaEventCreate(&ev[0])); VDO_CUDA(cudaEventCreate(&ev[1])); VDO_CUDA(cudaEventRecord(ev[0], st)); }
  k_sample_keys<<<n, SAMPLE_THREADS, 0, st>>>(Tabs::at<SampleKeysSeq>(W, o));
  VDO_CUDA(cudaGetLastError());
  if (kernel_ms) VDO_CUDA(cudaEventRecord(ev[1], st));
  VDO_CUDA(cudaMemcpyAsync(kx, d, sizeof(float) * tot, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaMemcpyAsync(ky, d + tot, sizeof(float) * tot, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  if (kernel_ms) {
    VDO_CUDA(cudaEventElapsedTime(kernel_ms, ev[0], ev[1]));
    cudaEventDestroy(ev[0]); cudaEventDestroy(ev[1]);
  }
  return VDO_OK;
}

extern "C" int vdo_sample_keys_dev(vdo_ctx* ctx, int n, const uint32_t* seeds_dev, int width, int height, float* x_dev, float* y_dev, int32_t* count_dev,
                                   uint64_t stream) {
  if (!ctx) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(ctx, "vdo_sample_keys_dev: " + s); return VDO_ERR_ARG; };
  if (n < 1 || n > 65535) return refuse("n = " + std::to_string(n) + " outside 1 .. 65535");
  if (width < 20 || height < 20) return refuse(std::to_string(width) + " x " + std::to_string(height) + "; expected a width and height >= 20");
  int dev = 0, n_sm = 0;
  vdo::ctx_device(ctx, &dev, &n_sm);
  const std::string why = vdo::check_ptrs({{seeds_dev, 4, "seeds_dev"}, {x_dev, 4, "x_dev"}, {y_dev, 4, "y_dev"}, {count_dev, 4, "count_dev"}}, dev);
  if (!why.empty()) return refuse(why);
  k_sample_keys_dev<<<n, SAMPLE_THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>(seeds_dev, x_dev, y_dev, count_dev, width, height);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}

extern "C" int vdo_scene_flow(vdo_ctx* ctx, int n, const float* u_prev, const float* v_prev, const float* z_prev, const float* Tcw_prev,
                              const float* u_cur, const float* v_cur, const float* z_cur, const float* Tcw_cur, const float* K,
                              const int* label_prev, const int* label_cur, float* flow3d, float* Xw_prev, unsigned char* valid) {
  if (!ctx || n < 0) return VDO_ERR_ARG;
  if (n == 0) return VDO_OK;
  const int begin[2] = {0, n};
  return vdo::scene_flow_batch(ctx, 1, begin, Tcw_prev, Tcw_cur, K, u_prev, v_prev, z_prev, u_cur, v_cur, z_cur, label_prev, label_cur, flow3d, Xw_prev, valid);
}

// ================================================================================================ batched ORB extractor
// vdo_orb_extract_batch_dev: the ORB path of up to max_batch device images per call, on the caller's stream, with every buffer and launch
// table made at creation.  The kernels above run through per-launch tables (pyramid, score and blur planes with their sizes, the
// cell lists of every frame, the octree's (frame, level) entries); the octree (DistributeOctTree) runs on the device, and the per-call
// image pointers travel by value.  The same extractor serves the tracker's frame build with several geometries (image size + ORB settings):
// each frame of a call names its geometry, and the tables of each layout of geometries are built on its first use and kept.
namespace {
constexpr int ORB_MAX_BATCH = 64, OCT_MAX_CAP = 8192, OCT_MAX_ROUNDS = 1024;

// ---- DistributeOctTree (src/ORBextractor.cc:528-752) on the device, one CTA per (frame, level), bit-identical to the reference
// (restated in oracle/image_ops.py).
// The node list lives in list order in a global array.  Each key (a candidate, by its index into the level's dense candidate list) carries
// the list slot of the node that holds it, so a node's keys are the candidates naming it, in candidate order -- the order the reference's
// key vectors keep, since every split is a stable partition.  One round:
//   - every node with > 1 key is expandable; a key histogram gives each expandable node its four child counts;
//   - the processing order is list order (full round) or, in the sorted phase, (size, creation sequence) descending -- the reference walks
//     its ascending sort from the back; ties go to the later-created node -- cut where the list reaches N: expansion r runs iff
//     S + sum_{r' < r} (children(r') - 1) < N, the reference's "break once lNodes.size() >= N" after each expansion;
//   - children are pushed to the front and their parents erased in place, so the new list is the children in reverse creation order
//     (creation order = processing order, children 0..3 of each) followed by the nodes that were not expanded, in their old order;
//   - the reference's termination tests, on the new list size and the number of expandable nodes in it.
// Output: the node list front to back, each node's key of largest response (first in candidate order among equal responses).
//
// Node bound.  Let nIni be the number of initial nodes and N the level's quota.  The first full round expands at most nIni nodes into at
// most 4 nIni.  Every later full round starts only when size + 3 * expandable <= N, and expands exactly the expandable nodes, each adding
// at most 3: the list stays <= N.  A sorted-phase expansion runs only while the list is < N and adds at most 3: <= N + 2.  So the list
// never holds more than cap = max(N + 2, 4 nIni) nodes, and the level's output (one key per node) fits cap slots.  The kernel checks the
// bound anyway: a list that would exceed cap sets VDO_ORB_STATUS_NODE_BOUND and the frame reports no keypoints, never a truncated list.
struct OctNode { int x0, y0, x1, y1, cnt, seq; };          // rectangle [x0, x1) x [y0, y1) relative to (minX, minY); keys; creation sequence
// one (frame, level) of a call: cells [c0, c1) and slots [off, off + cap) of the call, frame fr
struct OctLevel { int minX, maxX, minY, maxY, N, cap, c0, c1, off, fr; };
struct OctArgs {
  const OctLevel* lv;                                      // per (frame, level), frame-major
  const int* cell_off; const KpOut* dense;                 // k_cell_offsets / k_cell_gather of all frames of the call
  int* knode;                                              // per candidate: list slot of its node (indexed like dense)
  OctNode* nodes; int* ints; unsigned long long* best;     // per slot: 2 nodes, 11 ints, one best key
  KpOut* kept; int* kept_cnt; int* status;                 // per slot: a kept key; per (frame, level) count; per frame
};

__device__ __forceinline__ void oct_mid(const OctNode& n, int& mx, int& my) {   // DivideNode: halfX = ceil((URx - ULx) / 2.f)
  mx = n.x0 + (int)ceilf(__fdiv_rn((float)(n.x1 - n.x0), 2.f));
  my = n.y0 + (int)ceilf(__fdiv_rn((float)(n.y1 - n.y0), 2.f));
}
__device__ __forceinline__ int oct_quad(const OctNode& n, float kx, float ky) {
  int mx, my; oct_mid(n, mx, my);
  return kx < (float)mx ? (ky < (float)my ? 0 : 2) : (ky < (float)my ? 1 : 3);
}
__device__ __forceinline__ OctNode oct_child(const OctNode& n, int q, int cnt, int seq) {
  int mx, my; oct_mid(n, mx, my);
  return OctNode{(q & 1) ? mx : n.x0, (q & 2) ? my : n.y0, (q & 1) ? n.x1 : mx, (q & 2) ? n.y1 : my, cnt, seq};
}
__device__ __forceinline__ int oct_nchild(const int* c) { return (c[0] > 0) + (c[1] > 0) + (c[2] > 0) + (c[3] > 0); }

__global__ void __launch_bounds__(1024) k_octree(const OctArgs a, int* __restrict__ n_cand_out) {
  extern __shared__ unsigned long long s_key[];            // sorted-phase keys: a power of two >= the largest level capacity
  __shared__ int wsum[33];
  const int slot = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const OctLevel L = a.lv[slot];
  const int fr = L.fr;
  const int k0 = a.cell_off[L.c0], nk = a.cell_off[L.c1] - k0;
  if (tid == 0 && n_cand_out) n_cand_out[slot] = nk;
  int* kcnt = a.kept_cnt + slot;
  if (nk == 0) { if (tid == 0) *kcnt = 0; return; }
  const KpOut* __restrict__ key = a.dense + k0;
  int* __restrict__ knode = a.knode + k0;
  const size_t fb = (size_t)L.off;
  OctNode* NA = a.nodes + 2 * fb;
  OctNode* NB = NA + L.cap;
  int* cc = a.ints + 11 * fb;                              // 4 per node: child key counts
  int* cslot = cc + 4 * L.cap;                             // 4 per node: list slot of each child
  int* sslot = cslot + 4 * L.cap;                          // new slot of a node that is not expanded
  int* cbeg = sslot + L.cap;                               // creation index of an expanded node's first child, -1: not expanded
  int* order = cbeg + L.cap;                               // processing order
  unsigned long long* best = a.best + fb;
  auto fail = [&](int bit) { if (tid == 0) { atomicOr(a.status + fr, bit); *kcnt = 0; } };

  // ---- initial nodes: nIni columns of width hX; empty ones are erased
  const int W = L.maxX - L.minX, H = L.maxY - L.minY;
  const int nIni = (int)roundf(__fdiv_rn((float)W, (float)H));
  if (nIni < 1 || nIni > L.cap || nk >= (1 << 24)) { fail(VDO_ORB_STATUS_INPUT); return; }   // node sizes enter the sort key in 24 bits
  const float hX = __fdiv_rn((float)W, (float)nIni);
  for (int i = tid; i < nIni; i += nt) cc[i] = 0;
  __syncthreads();
  int bad = 0;
  for (int k = tid; k < nk; k += nt) {
    const int j = (int)__fdiv_rn(key[k].x, hX);
    if (j < 0 || j >= nIni) bad = 1;
    else { knode[k] = j; atomicAdd(&cc[j], 1); }
  }
  if (__syncthreads_or(bad)) { fail(VDO_ORB_STATUS_INPUT); return; }
  int S = 0;
  for (int base = 0; base < nIni; base += nt) {
    const int i = base + tid, c = i < nIni ? cc[i] : 0;
    int tot;
    const int pos = S + cta_excl_scan(c > 0, wsum, tot);
    if (c > 0) { NA[pos] = OctNode{(int)__fmul_rn(hX, (float)i), 0, (int)__fmul_rn(hX, (float)(i + 1)), H, c, 0}; sslot[i] = pos; }
    S += tot;
  }
  __syncthreads();
  for (int k = tid; k < nk; k += nt) knode[k] = sslot[knode[k]];

  bool sorted = false;
  int seq0 = 0;
  for (int round = 0;; ++round) {
    if (round == OCT_MAX_ROUNDS || seq0 + 4 * S >= (1 << 26)) { fail(VDO_ORB_STATUS_ROUNDS); return; }
    for (int i = tid; i < S; i += nt) { cc[4 * i] = cc[4 * i + 1] = cc[4 * i + 2] = cc[4 * i + 3] = 0; cbeg[i] = -1; }
    __syncthreads();
    for (int k = tid; k < nk; k += nt) {                   // child histogram of the expandable nodes
      const int j = knode[k];
      const OctNode n = NA[j];
      if (n.cnt > 1) atomicAdd(&cc[4 * j + oct_quad(n, key[k].x, key[k].y)], 1);
    }
    __syncthreads();
    int P = 0;                                             // expansions this round, in processing order
    if (!sorted) {
      for (int base = 0; base < S; base += nt) {
        const int i = base + tid;
        const bool e = i < S && NA[i].cnt > 1;
        int tot;
        const int pos = P + cta_excl_scan(e, wsum, tot);
        if (e) order[pos] = i;
        P += tot;
      }
    } else {
      int E = 0;                                           // key = size | creation sequence | slot (seq < 2^26, slot < 2^14)
      for (int base = 0; base < S; base += nt) {
        const int i = base + tid;
        const bool e = i < S && NA[i].cnt > 1;
        int tot;
        const int pos = E + cta_excl_scan(e, wsum, tot);
        if (e) s_key[pos] = ((unsigned long long)NA[i].cnt << 40) | ((unsigned long long)NA[i].seq << 14) | (unsigned long long)i;
        E += tot;
      }
      int P2 = 1;
      while (P2 < E) P2 <<= 1;
      for (int i = E + tid; i < P2; i += nt) s_key[i] = 0ull;
      __syncthreads();
      for (int kk = 2; kk <= P2; kk <<= 1)                 // bitonic sort, descending
        for (int j = kk >> 1; j > 0; j >>= 1) {
          for (int i = tid; i < P2; i += nt) {
            const int l = i ^ j;
            if (l > i) {
              const unsigned long long x = s_key[i], y = s_key[l];
              if ((i & kk) == 0 ? x < y : x > y) { s_key[i] = y; s_key[l] = x; }
            }
          }
          __syncthreads();
        }
      int grown = 0;                                       // list growth of the expansions before this chunk
      for (int base = 0; base < E; base += nt) {
        const int r = base + tid;
        const int j = r < E ? (int)(s_key[r] & 0x3fffull) : 0;
        const int d = r < E ? oct_nchild(cc + 4 * j) - 1 : 0;
        int tot;
        const int before = grown + cta_excl_scan(d, wsum, tot);
        const bool run = r < E && S + before < L.N;
        if (run) order[r] = j;
        P += __syncthreads_count(run);
        grown += tot;
      }
    }
    __syncthreads();
    int C = 0;                                             // children created this round
    for (int base = 0; base < P; base += nt) {
      const int p = base + tid;
      const int j = p < P ? order[p] : 0, c = p < P ? oct_nchild(cc + 4 * j) : 0;
      int tot;
      const int pos = C + cta_excl_scan(c, wsum, tot);
      if (p < P) cbeg[j] = pos;
      C += tot;
    }
    __syncthreads();
    int S2 = C;                                            // new list: C children, then the nodes that stay
    for (int base = 0; base < S; base += nt) {
      const int i = base + tid;
      const bool s = i < S && cbeg[i] < 0;
      int tot;
      const int pos = S2 + cta_excl_scan(s, wsum, tot);
      if (s) { sslot[i] = pos; if (pos < L.cap) NB[pos] = NA[i]; }
      S2 += tot;
    }
    if (S2 > L.cap) { fail(VDO_ORB_STATUS_NODE_BOUND); return; }
    for (int p = tid; p < P; p += nt) {
      const int j = order[p];
      const OctNode n = NA[j];
      int c = cbeg[j];
      for (int q = 0; q < 4; ++q) {
        const int m = cc[4 * j + q];
        if (m == 0) continue;
        const int s = C - 1 - c;                           // pushed to the front: reverse creation order
        NB[s] = oct_child(n, q, m, seq0 + c + 1);
        cslot[4 * j + q] = s;
        ++c;
      }
    }
    __syncthreads();
    for (int k = tid; k < nk; k += nt) {                   // keys follow their node
      const int j = knode[k];
      knode[k] = cbeg[j] >= 0 ? cslot[4 * j + oct_quad(NA[j], key[k].x, key[k].y)] : sslot[j];
    }
    seq0 += C;
    const int prev = S;
    S = S2;
    OctNode* t = NA; NA = NB; NB = t;
    int E2 = 0;                                            // expandable nodes of the new list (the reference's nToExpand)
    for (int base = 0; base < S; base += nt) { const int i = base + tid; E2 += __syncthreads_count(i < S && NA[i].cnt > 1); }
    if (S >= L.N || S == prev) break;
    if (!sorted && S + 3 * E2 > L.N) sorted = true;
  }
  // ---- each node keeps its key of largest response; equal responses: the first in candidate order
  for (int i = tid; i < S; i += nt) best[i] = 0ull;
  __syncthreads();
  for (int k = tid; k < nk; k += nt) {
    unsigned int u = __float_as_uint(__fadd_rn(key[k].resp, 0.f));      // -0 -> +0; then an order-preserving map of the float to u32
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    atomicMax(best + knode[k], ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned int)k));
  }
  __syncthreads();
  KpOut* kept = a.kept + fb;
  for (int i = tid; i < S; i += nt) kept[i] = key[0xffffffffu - (unsigned int)(best[i] & 0xffffffffull)];
  if (tid == 0) *kcnt = S;
}

// ---- gray ingest of the call's images (pointers by value), level-major output, angles, blur and descriptors of a batch
struct IngestImages { PlaneArg img[ORB_MAX_BATCH]; };
PlaneArg gray_plane(const vdo_frame* f) { return PlaneArg{f->gray, f->w, 1, 0, VDO_DT_U8, 1, 0}; }   // a frame's resident gray image
// lv0: the level-0 entries of the pyramid table (dst: the frame's level-0 plane, dw x dh its size)
__global__ void __launch_bounds__(256) k_ingest_gray(const IngestImages a, const PairSeq* __restrict__ lv0) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const PairSeq& q = lv0[blockIdx.z];
  const int w = q.dw, h = q.dh;
  if (x >= w || y >= h) return;
  q.dst[(size_t)y * w + x] = gray_px(a.img[blockIdx.z], x, y);
}
// per frame: its levels, the first of its (frame, level) entries, and per level the border, scale, size and slot offset
struct OrbLevelsOut { float minX[MAX_LEVELS], minY[MAX_LEVELS], scale[MAX_LEVELS]; int size[MAX_LEVELS], off[MAX_LEVELS]; int nlev, lv0; };
struct OrbOut { float* x; float* y; int* oct; float* resp; float* ang; int* size; unsigned char* desc; int* count; int* status; };
// one CTA per frame: the kept keys of every level, level-major, in level-0 coordinates (src/ORBextractor.cc:1098-1108); a frame whose octree
// failed reports no keypoints
__global__ void __launch_bounds__(256) k_orb_scatter(const KpOut* __restrict__ kept, const int* __restrict__ kept_cnt, const int* __restrict__ status,
                                                     int cap, const OrbLevelsOut* __restrict__ lvs, KpLvl* __restrict__ kps, int* __restrict__ kp_count, OrbOut o) {
  __shared__ int beg[MAX_LEVELS + 1];
  const int fr = blockIdx.x, st = status[fr];
  const OrbLevelsOut& lv = lvs[fr];
  const int nlev = lv.nlev;
  if (threadIdx.x == 0) {
    beg[0] = 0;
    for (int l = 0; l < nlev; ++l) beg[l + 1] = beg[l] + (st ? 0 : kept_cnt[lv.lv0 + l]);
  }
  __syncthreads();
  for (int l = 0; l < nlev; ++l)
    for (int j = threadIdx.x; j < beg[l + 1] - beg[l]; j += blockDim.x) {
      const KpOut k = kept[(size_t)fr * cap + lv.off[l] + j];
      const float lx = __fadd_rn(k.x, lv.minX[l]), ly = __fadd_rn(k.y, lv.minY[l]);
      const size_t p = (size_t)fr * cap + beg[l] + j;
      kps[p] = KpLvl{lx, ly, l};
      o.x[p] = l ? __fmul_rn(lx, lv.scale[l]) : lx;
      o.y[p] = l ? __fmul_rn(ly, lv.scale[l]) : ly;
      o.oct[p] = l; o.resp[p] = k.resp; o.size[p] = lv.size[l];
    }
  if (threadIdx.x == 0) { kp_count[fr] = o.count[fr] = beg[nlev]; o.status[fr] = st; }
}
// one warp per keypoint slot; frame = slot / cap, slots past the frame's count return
__global__ void k_ic_angle_batch(const KpLvl* __restrict__ kps, const int* __restrict__ kp_count, int n_slots, int cap, const LevelsArg* __restrict__ levels,
                                 UmaxArg umax, float* __restrict__ angle) {
  const int gid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gid >= n_slots) return;
  const int fr = gid / cap;
  if (gid - fr * cap >= kp_count[fr]) return;
  const KpLvl k = kps[gid];
  const float a = ic_angle_warp(levels[fr].L[k.level], k, umax, lane);
  if (lane == 0) angle[gid] = a;
}
__global__ void k_blur7_batch(const PairSeq* __restrict__ tab) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const PairSeq& q = tab[blockIdx.z];
  const int w = q.dw, h = q.dh;
  if (x >= w || y >= h) return;
  q.dst[(size_t)y * w + x] = blur7_px(q.src, w, h, x, y);
}
__global__ void k_orb_descriptors_batch(const KpLvl* __restrict__ kps, const float* __restrict__ ang, const int* __restrict__ kp_count, int n_slots,
                                        int cap, const BlurLevels* __restrict__ levels, unsigned char* __restrict__ desc) {
  const int gid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gid >= n_slots) return;
  const int fr = gid / cap;
  if (gid - fr * cap >= kp_count[fr]) return;
  const KpLvl kp = kps[gid];
  desc[(size_t)gid * 32 + lane] = orb_desc_byte(levels[fr].img[kp.level], levels[fr].w[kp.level], kp, ang[gid], lane);
}

// level geometry of ComputeKeyPointsOctTree (src/ORBextractor.cc:754-842) for a w x h image: level sizes, borders, the cell grid of every
// level (cells_begin[l] .. cells_begin[l + 1]) and the initial octree node count per level; VDO_ERR_UNSUPPORTED for cells over 62 px
struct OrbGeometry {
  int lw[MAX_LEVELS], lh[MAX_LEVELS], bord[MAX_LEVELS][4], nini[MAX_LEVELS];
  std::vector<Cell> grid; std::vector<int> cell_begin, cell_level;
  int build(int w, int h, const OrbSetup& P) {
    cell_begin.assign(P.nlevels + 1, 0);
    for (int l = 0; l < P.nlevels; ++l) {
      lw[l] = l ? (int)std::lrint((float)w * P.inv_scale[l]) : w;
      lh[l] = l ? (int)std::lrint((float)h * P.inv_scale[l]) : h;
      const int minB = EDGE_THRESHOLD - 3, maxBX = lw[l] - EDGE_THRESHOLD + 3, maxBY = lh[l] - EDGE_THRESHOLD + 3;
      bord[l][0] = minB; bord[l][1] = maxBX; bord[l][2] = minB; bord[l][3] = maxBY;
      nini[l] = 0;
      const float width = (float)(maxBX - minB), height = (float)(maxBY - minB);
      const int nCols = (int)(width / 30.f), nRows = (int)(height / 30.f);
      if (nCols < 1 || nRows < 1) { cell_begin[l + 1] = (int)grid.size(); continue; }
      const int wCell = (int)std::ceil(width / nCols), hCell = (int)std::ceil(height / nRows);
      if (wCell + 2 > 64 || hCell + 2 > 64) return VDO_ERR_UNSUPPORTED;
      nini[l] = (int)std::round(static_cast<float>(maxBX - minB) / (maxBY - minB));
      for (int i = 0; i < nRows; ++i) {
        const int iniY = minB + i * hCell; int maxY = iniY + hCell + 6;
        if (iniY >= maxBY - 3) continue;
        if (maxY > maxBY) maxY = maxBY;
        for (int j = 0; j < nCols; ++j) {
          const int iniX = minB + j * wCell; int maxX = iniX + wCell + 6;
          if (iniX >= maxBX - 6) continue;
          if (maxX > maxBX) maxX = maxBX;
          grid.push_back(Cell{iniX, iniY, maxX, maxY, j * wCell, i * hCell, lw[l], P.ini_th, P.min_th, nullptr});
          cell_level.push_back(l);
        }
      }
      cell_begin[l + 1] = (int)grid.size();
    }
    return VDO_OK;
  }
};
// octree capacity of a level: max(N + 2, 4 nIni) (see k_octree); 0 for a level without cells
int oct_cap(int N, int nini) { return nini > 0 ? std::max(N + 2, 4 * nini) : 0; }
int oct_smem(int max_cap) { int p = 1; while (p < max_cap) p <<= 1; return (int)sizeof(unsigned long long) * p; }

// One geometry of an extractor (an image size with its ORB settings): the level geometry, the octree levels and output table of one frame,
// and the planes of `slots` frames.
struct OrbGeo {
  OrbSetup P; OrbGeometry G;
  int w = 0, h = 0, slots = 0, cap = 0, max_cap = 1;
  std::vector<OctLevel> lv;                                    // per level: cells and slots relative to the frame's own
  OrbLevelsOut lvo{};                                          // lv0 relative to the frame's first (frame, level) entry
  unsigned char *pyr[MAX_LEVELS] = {nullptr}, *score[MAX_LEVELS] = {nullptr}, *blur[MAX_LEVELS] = {nullptr};   // `slots` planes per level
  int ncell() const { return (int)G.grid.size(); }
  size_t plane(int l) const { return (size_t)G.lw[l] * G.lh[l]; }
  // what vdo_orb_extractor_create refuses, with the reason in why: VDO_ERR_ARG for out-of-range arguments and for a pyramid level under
  // 1 px in either direction (cv::resize asserts on an empty size), VDO_ERR_UNSUPPORTED for cells over 62 px, a level capacity over
  // OCT_MAX_CAP or a level with cells and no initial octree node
  int init(const vdo::OrbKey& k, std::string& why) {
    if (k.w < 64 || k.h < 64 || k.nfeatures < 1 || !(k.scale_factor > 1.f) || k.nlevels < 1 || k.nlevels > MAX_LEVELS) {
      why = "image " + std::to_string(k.w) + "x" + std::to_string(k.h) + ", nfeatures " + std::to_string(k.nfeatures) + ", scale factor " +
            std::to_string(k.scale_factor) + ", nlevels " + std::to_string(k.nlevels) +
            ": expected an image of at least 64x64, nfeatures >= 1, a scale factor above 1 and 1 .. 12 levels";
      return VDO_ERR_ARG;
    }
    w = k.w; h = k.h;
    P.init(k.nfeatures, k.scale_factor, k.nlevels, k.ini_th, k.min_th);
    if (int rc = G.build(w, h, P)) { why = "a cell over 62 px"; return rc; }
    const std::string geom = std::to_string(w) + "x" + std::to_string(h) + " at scale factor " + std::to_string(k.scale_factor);
    for (int l = 1; l < k.nlevels; ++l)
      if (G.lw[l] < 1 || G.lh[l] < 1) {
        why = "level " + std::to_string(l) + " of " + geom + " is " + std::to_string(G.lw[l]) + "x" + std::to_string(G.lh[l]) + " px; every level needs at least 1x1";
        return VDO_ERR_ARG;
      }
    lv.resize(k.nlevels);
    for (int l = 0; l < k.nlevels; ++l) {
      const int c = oct_cap(P.per_level[l], G.nini[l]);
      if (c > OCT_MAX_CAP) {
        why = "level " + std::to_string(l) + " of " + geom + " needs " + std::to_string(c) + " octree nodes for its " + std::to_string(P.per_level[l]) +
              " features; the limit is " + std::to_string(OCT_MAX_CAP);
        return VDO_ERR_UNSUPPORTED;
      }
      if (G.cell_begin[l + 1] > G.cell_begin[l] && G.nini[l] < 1) {
        why = "level " + std::to_string(l) + " of " + geom + " has no initial octree node (nIni = 0: the image is more than about twice as tall as wide)";
        return VDO_ERR_UNSUPPORTED;
      }
      lv[l] = OctLevel{G.bord[l][0], G.bord[l][1], G.bord[l][2], G.bord[l][3], P.per_level[l], c, G.cell_begin[l], G.cell_begin[l + 1], cap, 0};
      lvo.minX[l] = (float)G.bord[l][0]; lvo.minY[l] = (float)G.bord[l][2]; lvo.scale[l] = P.scale_factor[l];
      lvo.size[l] = (int)(PATCH_SIZE * P.scale_factor[l]); lvo.off[l] = cap;
      cap += c; max_cap = std::max(max_cap, c);
    }
    lvo.nlev = k.nlevels; lvo.lv0 = 0;
    return VDO_OK;
  }
};
// The launch tables of one frame layout: the geometry of each batch position, a frame taking the next slot of its geometry.  A call of
// n frames runs on the tables of any layout whose first n positions are its frames' geometries.
struct OrbTabs {
  std::vector<int> geo;                                        // per position
  int nlev = 0;                                                // the most levels of any position
  std::vector<int> gw, gh;                                     // per level: the largest level size among the positions (the grid)
  std::vector<int> cell_begin, oct_begin;                      // per position: its first cell / (frame, level) entry; one more at the end
  PairSeq *rs = nullptr, *sc = nullptr, *bl = nullptr;         // [level][position]
  Cell* cells = nullptr; OctLevel* oct = nullptr;              // concatenated over the positions
  LevelsArg* ang = nullptr; BlurLevels* desc = nullptr; OrbLevelsOut* lvo = nullptr;   // per position
};
}  // namespace

struct vdo_orb_extractor : vdo::WorkSpace {
  vdo_ctx* ctx = nullptr;
  int dev = -1, max_batch = 0, cap = 0, nlev = 0, smem = 0;    // cap: the largest geometry capacity (the per-frame output stride)
  std::vector<OrbGeo> geo;
  std::vector<OrbTabs> tabs;
  KpOut *cell_out = nullptr, *dense = nullptr; int *cell_cnt = nullptr, *cell_off = nullptr;
  OctArgs oct{};
  KpLvl* kps = nullptr; int* kp_count = nullptr;
  UmaxArg umax{};
  template <class T> int upload(T*& p, const std::vector<T>& v) {
    VDO_CUDA(alloc(p, v.size()));
    VDO_CUDA(cudaMemcpy(p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
    return VDO_OK;
  }
  // the tables of a layout starting with geo[0 .. n), built on first use; VDO_ERR_ARG if a geometry has too few slots
  int tables_for(const int* g, int n, const OrbTabs** out) {
    for (const OrbTabs& T : tabs)
      if ((int)T.geo.size() >= n && std::equal(g, g + n, T.geo.begin())) { *out = &T; return VDO_OK; }
    OrbTabs T;
    T.geo.assign(g, g + n);
    std::vector<int> used(geo.size(), 0), slot(n);
    for (int i = 0; i < n; ++i) {
      slot[i] = used[g[i]]++;
      if (slot[i] >= geo[g[i]].slots) return VDO_ERR_ARG;
      T.nlev = std::max(T.nlev, geo[g[i]].P.nlevels);
    }
    const int L = T.nlev;
    T.gw.assign(L, 0); T.gh.assign(L, 0); T.cell_begin.assign(n + 1, 0); T.oct_begin.assign(n + 1, 0);
    std::vector<PairSeq> rs((size_t)L * n, PairSeq{nullptr, nullptr, 0, 0, 0, 0}), sc = rs, bl = rs;
    std::vector<Cell> cells; std::vector<OctLevel> oc;
    std::vector<LevelsArg> la(n); std::vector<BlurLevels> bla(n); std::vector<OrbLevelsOut> lo(n);
    for (int i = 0; i < n; ++i) {
      const OrbGeo& q = geo[g[i]]; const OrbGeometry& G = q.G; const int s = slot[i];
      std::memset(&la[i], 0, sizeof la[i]); std::memset(&bla[i], 0, sizeof bla[i]);
      for (int l = 0; l < q.P.nlevels; ++l) {
        const size_t np = q.plane(l);
        T.gw[l] = std::max(T.gw[l], G.lw[l]); T.gh[l] = std::max(T.gh[l], G.lh[l]);
        rs[(size_t)l * n + i] = l ? PairSeq{q.pyr[l - 1] + q.plane(l - 1) * s, q.pyr[l] + np * s, G.lw[l - 1], G.lh[l - 1], G.lw[l], G.lh[l]}
                                  : PairSeq{nullptr, q.pyr[0] + np * s, 0, 0, G.lw[0], G.lh[0]};
        sc[(size_t)l * n + i] = PairSeq{q.pyr[l] + np * s, q.score[l] + np * s, G.lw[l], G.lh[l], G.lw[l], G.lh[l]};
        bl[(size_t)l * n + i] = PairSeq{q.pyr[l] + np * s, q.blur[l] + np * s, G.lw[l], G.lh[l], G.lw[l], G.lh[l]};
        la[i].L[l] = LevelDesc{q.pyr[l] + np * s, G.lw[l], G.lh[l]};
        bla[i].img[l] = q.blur[l] + np * s; bla[i].w[l] = G.lw[l]; bla[i].h[l] = G.lh[l];
        OctLevel o = q.lv[l];
        o.c0 += T.cell_begin[i]; o.c1 += T.cell_begin[i]; o.off += i * cap; o.fr = i;
        oc.push_back(o);
      }
      for (int c = 0; c < q.ncell(); ++c) {
        Cell x = G.grid[c];
        x.score = q.score[G.cell_level[c]] + q.plane(G.cell_level[c]) * s;
        cells.push_back(x);
      }
      lo[i] = q.lvo; lo[i].lv0 = T.oct_begin[i];
      T.cell_begin[i + 1] = (int)cells.size(); T.oct_begin[i + 1] = (int)oc.size();
    }
    if (int rc = upload(T.rs, rs)) return rc;
    if (int rc = upload(T.sc, sc)) return rc;
    if (int rc = upload(T.bl, bl)) return rc;
    if (int rc = upload(T.cells, cells)) return rc;
    if (int rc = upload(T.oct, oc)) return rc;
    if (int rc = upload(T.ang, la)) return rc;
    if (int rc = upload(T.desc, bla)) return rc;
    if (int rc = upload(T.lvo, lo)) return rc;
    tabs.push_back(std::move(T));
    *out = &tabs.back();
    return VDO_OK;
  }
};

namespace vdo {
// An extractor of max_batch frames over the geometries keys, slots[g] frames of keys[g] per call; the refusals of vdo_orb_extractor_create
int orb_create(vdo_ctx* ctx, const std::vector<OrbKey>& keys, const std::vector<int>& slots, int max_batch, vdo_orb_extractor** out) {
  if (!ctx || !out || keys.empty() || keys.size() != slots.size() || max_batch < 1 || max_batch > ORB_MAX_BATCH) return VDO_ERR_ARG;
  *out = nullptr;
  std::unique_ptr<vdo_orb_extractor> ex(new vdo_orb_extractor);
  ex->ctx = ctx; ex->max_batch = max_batch;
  ex->geo.resize(keys.size());
  int max_cap = 1;
  size_t ncell = 0;
  for (size_t g = 0; g < keys.size(); ++g) {
    OrbGeo& q = ex->geo[g];
    std::string why;
    if (int rc = q.init(keys[g], why)) return rc;
    q.slots = std::min(slots[g], max_batch);
    ex->cap = std::max(ex->cap, q.cap); ex->nlev = std::max(ex->nlev, q.P.nlevels); max_cap = std::max(max_cap, q.max_cap);
    ncell += (size_t)q.slots * q.ncell();
    for (int l = 0; l < q.P.nlevels; ++l) {
      const size_t np = q.plane(l);
      VDO_CUDA(ex->alloc(q.pyr[l], np * q.slots)); VDO_CUDA(ex->alloc(q.score[l], np * q.slots)); VDO_CUDA(ex->alloc(q.blur[l], np * q.slots));
    }
  }
  for (int i = 0; i < 16; ++i) ex->umax.v[i] = ex->geo[0].P.umax[i];   // a function of HALF_PATCH alone
  ex->smem = oct_smem(max_cap);
  VDO_CUDA(cudaFuncSetAttribute(k_octree, cudaFuncAttributeMaxDynamicSharedMemorySize, oct_smem(OCT_MAX_CAP)));
  // candidates (a call holds at most `slots` frames of each geometry), octree work space, outputs of the octree and of the scatter
  const int B = max_batch, C = ex->cap;
  const size_t ncand = ncell * CELL_CAP;
  VDO_CUDA(ex->alloc(ex->cell_out, ncand)); VDO_CUDA(ex->alloc(ex->dense, ncand)); VDO_CUDA(ex->alloc(ex->cell_cnt, ncell)); VDO_CUDA(ex->alloc(ex->cell_off, ncell + 1));
  OctArgs& o = ex->oct;
  o.cell_off = ex->cell_off; o.dense = ex->dense;
  VDO_CUDA(ex->alloc(o.knode, ncand)); VDO_CUDA(ex->alloc(o.nodes, (size_t)2 * B * C)); VDO_CUDA(ex->alloc(o.ints, (size_t)11 * B * C));
  VDO_CUDA(ex->alloc(o.best, (size_t)B * C)); VDO_CUDA(ex->alloc(o.kept, (size_t)B * C)); VDO_CUDA(ex->alloc(o.kept_cnt, (size_t)B * ex->nlev)); VDO_CUDA(ex->alloc(o.status, (size_t)B));
  VDO_CUDA(ex->alloc(ex->kps, (size_t)B * C)); VDO_CUDA(ex->alloc(ex->kp_count, (size_t)B));
  cudaPointerAttributes a;
  VDO_CUDA(cudaPointerGetAttributes(&a, ex->dense));
  ex->dev = a.device;
  *out = ex.release();
  return VDO_OK;
}
void orb_extractor_info(const vdo_orb_extractor* ex, int* cap, int* nlevels) { *cap = ex->cap; *nlevels = ex->nlev; }
int orb_key_check(const OrbKey& k, std::string& why) { OrbGeo q; return q.init(k, why); }
}  // namespace vdo

extern "C" int vdo_orb_extractor_create(vdo_ctx* ctx, int width, int height, int max_batch, int nfeatures, float scale_factor, int nlevels, int ini_th,
                                        int min_th, vdo_orb_extractor** out) {
  if (!ctx || !out) return VDO_ERR_ARG;
  const vdo::OrbKey key{width, height, nfeatures, scale_factor, nlevels, ini_th, min_th};
  std::string why;
  if (int rc = vdo::orb_key_check(key, why)) { vdo::ctx_set_error(ctx, "vdo_orb_extractor_create: " + why); return rc; }
  vdo_orb_extractor* ex = nullptr;
  if (int rc = vdo::orb_create(ctx, {key}, {max_batch}, max_batch, &ex)) return rc;
  const std::vector<int> layout(max_batch, 0);                 // every launch table made at creation
  const OrbTabs* T = nullptr;
  if (int rc = ex->tables_for(layout.data(), max_batch, &T)) { delete ex; return rc; }
  *out = ex;
  return VDO_OK;
}
extern "C" void vdo_orb_extractor_destroy(vdo_orb_extractor* ex) { delete ex; }
extern "C" int vdo_orb_extractor_info(const vdo_orb_extractor* ex, int64_t out[4]) {
  if (!ex || !out) return VDO_ERR_ARG;
  out[0] = ex->cap; out[1] = (int64_t)ex->bytes; out[2] = ex->nlev; out[3] = ex->max_batch;
  return VDO_OK;
}

namespace vdo {
// pyramid and FAST score maps of frames 0 .. n-1 of the layout T (level 0 ingested): per level one launch over the frames that have it
static void orb_pyramid(const OrbTabs& T, int n, cudaStream_t st) {
  const dim3 b(32, 8);
  const size_t stride = T.geo.size();
  for (int l = 0; l < T.nlev; ++l) {
    const dim3 g((T.gw[l] + 31) / 32, (T.gh[l] + 7) / 8, n);
    if (l > 0) k_resize_u8<<<g, b, 0, st>>>(T.rs + (size_t)l * stride);
    k_fast_score<<<g, b, 0, st>>>(T.sc + (size_t)l * stride);
  }
}
// the keypoint part of vdo_orb_extract_batch_dev on checked arguments, all on stream st: ingest, pyramid, FAST, cells, octree, level-major
// output, angles.  Frame i has geometry geo[i].  The extractor keeps the keypoints (level coordinates) for orb_run_describe.
static int orb_run_keys(vdo_orb_extractor* ex, const int* geo, int n, const IngestImages& im, const vdo_orb_batch_out& out, cudaStream_t st,
                        const OrbTabs** tabs = nullptr) {
  const OrbTabs* T = nullptr;
  if (int rc = ex->tables_for(geo, n, &T)) return rc;
  if (tabs) *tabs = T;
  const int ntot = T->cell_begin[n];
  VDO_CUDA(cudaMemsetAsync(ex->oct.status, 0, sizeof(int) * n, st));
  k_ingest_gray<<<dim3((T->gw[0] + 31) / 32, (T->gh[0] + 7) / 8, n), dim3(32, 8), 0, st>>>(im, T->rs);
  orb_pyramid(*T, n, st);
  k_fast_cells<<<ntot, 256, 0, st>>>(T->cells, ex->cell_out, ex->cell_cnt);
  k_cell_offsets<<<1, 1024, 0, st>>>(ex->cell_cnt, ntot, ex->cell_off);
  k_cell_gather<<<ntot, 64, 0, st>>>(ex->cell_out, ex->cell_cnt, ex->cell_off, ex->dense);
  OctArgs a = ex->oct;
  a.lv = T->oct;
  k_octree<<<T->oct_begin[n], 1024, ex->smem, st>>>(a, out.n_candidates_dev);
  const OrbOut o{out.x_dev, out.y_dev, out.octave_dev, out.response_dev, out.angle_dev, out.size_dev, out.desc_dev, out.count_dev, out.status_dev};
  k_orb_scatter<<<n, 256, 0, st>>>(ex->oct.kept, ex->oct.kept_cnt, ex->oct.status, ex->cap, T->lvo, ex->kps, ex->kp_count, o);
  const int slots = n * ex->cap;
  k_ic_angle_batch<<<(int)(((size_t)slots * 32 + 255) / 256), 256, 0, st>>>(ex->kps, ex->kp_count, slots, ex->cap, T->ang, ex->umax, out.angle_dev);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
// the describe part: the 7x7 blur of every level, then the descriptors of the keypoints and angles (out.angle_dev) of the last orb_run_keys,
// which ran on the layout T
static int orb_run_describe(const vdo_orb_extractor* ex, const OrbTabs& T, int n, const vdo_orb_batch_out& out, cudaStream_t st) {
  const size_t stride = T.geo.size();
  for (int l = 0; l < T.nlev; ++l)
    k_blur7_batch<<<dim3((T.gw[l] + 31) / 32, (T.gh[l] + 7) / 8, n), dim3(32, 8), 0, st>>>(T.bl + (size_t)l * stride);
  const int slots = n * ex->cap;
  k_orb_descriptors_batch<<<(int)(((size_t)slots * 32 + 255) / 256), 256, 0, st>>>(ex->kps, out.angle_dev, ex->kp_count, slots, ex->cap, T.desc, out.desc_dev);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
}  // namespace vdo

extern "C" int vdo_orb_extract_batch_dev(vdo_orb_extractor* ex, int n, const vdo_dev_plane* images, const vdo_orb_batch_out* out, uint64_t stream) {
  if (!ex) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& m) { vdo::ctx_set_error(ex->ctx, "vdo_orb_extract_batch_dev: " + m); return VDO_ERR_ARG; };
  if (n < 1 || n > ex->max_batch) return refuse("n = " + std::to_string(n) + " outside 1 .. max_batch = " + std::to_string(ex->max_batch));
  if (!images || !out) return refuse("images or out is NULL");
  IngestImages im;
  std::memset(&im, 0, sizeof im);
  for (int i = 0; i < n; ++i) {
    const vdo_dev_plane& pl = images[i];
    const std::string who = "image " + std::to_string(i);
    if (pl.dtype != VDO_DT_U8 || !(pl.channels == 1 || pl.channels == 3 || pl.channels == 4))
      return refuse(who + ": dtype " + std::to_string(pl.dtype) + " with " + std::to_string(pl.channels) + " channels; expected u8 with 1, 3 or 4 channels");
    if (std::string why = vdo::check_ptrs({{pl.data_dev, 1, who + ": data_dev"}}, ex->dev); !why.empty()) return refuse(why);
    im.img[i] = plane_arg(&pl);
  }
  const vdo::DevPtrs outs = {
      {out->x_dev, 4, "x_dev"}, {out->y_dev, 4, "y_dev"}, {out->octave_dev, 4, "octave_dev"}, {out->response_dev, 4, "response_dev"},
      {out->angle_dev, 4, "angle_dev"}, {out->size_dev, 4, "size_dev"}, {out->count_dev, 4, "count_dev"},
      {out->n_candidates_dev, 4, "n_candidates_dev"}, {out->status_dev, 4, "status_dev"}, {out->desc_dev, 1, "desc_dev", out->desc_dev != nullptr}};
  if (std::string why = vdo::check_ptrs(outs, ex->dev); !why.empty()) return refuse(why);
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const std::vector<int> geo(n, 0);
  const OrbTabs* T = nullptr;
  if (int rc = vdo::orb_run_keys(ex, geo.data(), n, im, *out, st, &T)) return rc;
  return out->desc_dev ? vdo::orb_run_describe(ex, *T, n, *out, st) : VDO_OK;
}

// ---- the single-frame entries, on slot 0 of the frame's own extractor, and the tracker's frame build, on the cached extractors
extern "C" int vdo_orb_extract(vdo_frame* f, int nfeatures, float scale_factor, int nlevels, int ini_th, int min_th, int max_out,
                               float* x, float* y, int* octave, float* response, float* angle, int* size, int* n_out, int* n_candidates) {
  if (!f || nlevels < 1 || nlevels > MAX_LEVELS || !x || !y || !n_out) return VDO_ERR_ARG;
  vdo::OrbJob& J = f->orb;
  f->orb_count = -1;
  const vdo::OrbKey key{f->w, f->h, nfeatures, scale_factor, nlevels, ini_th, min_th};
  if (!J.same(key)) {
    std::string why;                                           // refused before the frame's current extractor is released
    if (int rc = vdo::orb_key_check(key, why)) { vdo::ctx_set_error(f->ctx, "vdo_orb_extract: " + why); return rc; }
    f->orb_blurred = false;
    if (int rc = J.create(f->ctx, {key}, {1}, 1, true)) return rc;
  }
  IngestImages im;
  std::memset(&im, 0, sizeof im);
  im.img[0] = gray_plane(f);
  const int geo0 = 0;
  if (int rc = vdo::orb_run_keys(J.ex, &geo0, 1, im, J.outs(1, J.buf), f->st)) return rc;
  std::vector<char> h(J.keys_bytes(1));
  VDO_CUDA(cudaMemcpyAsync(h.data(), J.buf, h.size(), cudaMemcpyDeviceToHost, f->st));
  VDO_CUDA(cudaStreamSynchronize(f->st));
  const vdo_orb_batch_out o = J.outs(1, h.data());
  if (*o.status_dev) { vdo::ctx_set_error(f->ctx, "vdo_orb_extract: device octree status " + std::to_string(*o.status_dev)); return VDO_ERR_UNSUPPORTED; }
  if (n_candidates) std::memcpy(n_candidates, o.n_candidates_dev, sizeof(int) * nlevels);
  *n_out = std::min(*o.count_dev, max_out);
  for (int i = 0; i < *n_out; ++i) {
    x[i] = o.x_dev[i]; y[i] = o.y_dev[i];
    if (octave) octave[i] = o.octave_dev[i];
    if (response) response[i] = o.response_dev[i];
    if (angle) angle[i] = o.angle_dev[i];
    if (size) size[i] = o.size_dev[i];
  }
  f->orb_count = angle ? *o.count_dev : -1;
  return VDO_OK;
}

// Descriptors of the keypoints of the last vdo_orb_extract call (which must have asked for angles): 7x7 sigma-2 blur of every level, then
// the 256 rotated pair tests.  desc_out: n x 32 bytes, in the order vdo_orb_extract returned the keypoints.
extern "C" int vdo_orb_describe(vdo_frame* f, int n, unsigned char* desc_out) {
  if (!f || !f->orb.ex || n < 0 || (n && !desc_out)) return VDO_ERR_ARG;
  if (f->orb_count < 0 || n > f->orb_count) return VDO_ERR_STATE;
  if (n == 0) return VDO_OK;
  const vdo_orb_batch_out o = f->orb.outs(1, f->orb.buf);
  if (int rc = vdo::orb_run_describe(f->orb.ex, f->orb.ex->tabs[0], 1, o, f->st)) return rc;
  f->orb_blurred = true;
  VDO_CUDA(cudaMemcpyAsync(desc_out, o.desc_dev, (size_t)n * 32, cudaMemcpyDeviceToHost, f->st));
  VDO_CUDA(cudaStreamSynchronize(f->st));
  return VDO_OK;
}
// test hook: the blurred level of the last vdo_orb_describe call
extern "C" int vdo_frame_debug_blur(vdo_frame* f, int level, unsigned char* img_out) {
  if (!f || !f->orb_blurred || level < 0 || level >= f->orb.nlevels || !img_out) return VDO_ERR_ARG;
  const OrbGeo& q = f->orb.ex->geo[0];
  VDO_CUDA(cudaMemcpyAsync(img_out, q.blur[level], q.plane(level), cudaMemcpyDeviceToHost, f->st));
  VDO_CUDA(cudaStreamSynchronize(f->st));
  return VDO_OK;
}
// test hook: download pyramid level `level` (and its FAST score map) computed by the last vdo_orb_extract; sizes via w_out/h_out
extern "C" int vdo_frame_debug_level(vdo_frame* f, int level, unsigned char* img_out, unsigned char* score_out, int* w_out, int* h_out) {
  if (!f || !f->orb.ex || level < 0 || level >= f->orb.nlevels) return VDO_ERR_ARG;
  const OrbGeo& q = f->orb.ex->geo[0];
  if (w_out) *w_out = q.G.lw[level];
  if (h_out) *h_out = q.G.lh[level];
  const size_t n = q.plane(level);
  if (img_out) VDO_CUDA(cudaMemcpyAsync(img_out, q.pyr[level], n, cudaMemcpyDeviceToHost, f->st));
  if (score_out) VDO_CUDA(cudaMemcpyAsync(score_out, q.score[level], n, cudaMemcpyDeviceToHost, f->st));
  VDO_CUDA(cudaStreamSynchronize(f->st));
  return VDO_OK;
}
// device-resident timing of the ORB front end (pyramid + score) for bench/profiles: returns avg ms over reps
extern "C" int vdo_orb_time(vdo_frame* f, int reps, float* ms_avg) {
  if (!f || !f->orb.ex || reps <= 0 || !ms_avg) return VDO_ERR_ARG;
  const OrbTabs& T = f->orb.ex->tabs[0];
  cudaEvent_t e0, e1; VDO_CUDA(cudaEventCreate(&e0)); VDO_CUDA(cudaEventCreate(&e1));
  vdo::orb_pyramid(T, 1, f->st);
  VDO_CUDA(cudaEventRecord(e0, f->st));
  for (int i = 0; i < reps; ++i) vdo::orb_pyramid(T, 1, f->st);
  VDO_CUDA(cudaEventRecord(e1, f->st));
  VDO_CUDA(cudaEventSynchronize(e1));
  float ms = 0; VDO_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  *ms_avg = ms / reps;
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return VDO_OK;
}

namespace vdo {
int orb_job_for(vdo_frame* const* fs, const OrbKey* keys, int n, OrbJob** out, int* geo, int* bad) {
  std::vector<OrbKey> ks(keys, keys + n);                      // the distinct geometries in key order
  std::sort(ks.begin(), ks.end());
  ks.erase(std::unique(ks.begin(), ks.end()), ks.end());
  const int batch = std::min(n, ORB_MAX_BATCH);
  std::vector<int> slots(ks.size(), 0);                        // the most frames of each geometry in one 64-frame chunk
  for (int c0 = 0; c0 < n; c0 += ORB_MAX_BATCH) {
    std::vector<int> cnt(ks.size(), 0);
    for (int i = c0; i < std::min(n, c0 + ORB_MAX_BATCH); ++i) {
      geo[i] = (int)(std::lower_bound(ks.begin(), ks.end(), keys[i]) - ks.begin());
      slots[geo[i]] = std::max(slots[geo[i]], ++cnt[geo[i]]);
    }
  }
  std::lock_guard<std::mutex> lk(g_ws_mu);
  const auto key = std::make_pair(fs[0]->st, ks);
  auto it = g_orb.find(key);
  if (it != g_orb.end()) {
    const OrbJob& J = it->second;
    bool fits = J.max_batch >= batch;
    for (size_t g = 0; g < ks.size() && fits; ++g) fits = J.slots[g] >= slots[g];
    if (fits) { *out = &it->second; return VDO_OK; }
  } else {
    for (const OrbKey& k : ks) {                               // checked as vdo_orb_extractor_create checks them, before any allocation
      OrbGeo q;
      std::string why;
      if (int rc = q.init(k, why)) {
        for (int i = 0; i < n; ++i) if (keys[i] == k) { *bad = i; break; }
        return rc;
      }
    }
    it = g_orb.emplace(key, OrbJob{}).first;
  }
  OrbJob& J = it->second;                                      // grown to what this call needs and what it held
  for (size_t g = 0; g < J.slots.size(); ++g) slots[g] = std::max(slots[g], J.slots[g]);
  if (int rc = J.create(fs[0]->ctx, ks, slots, std::max(batch, J.max_batch), false)) { g_orb.erase(it); *bad = 0; return rc; }
  *out = &J;
  return VDO_OK;
}
int orb_xy_batch(const OrbJob& J, vdo_frame* const* fs, const int* geo, int n, OrbXY* out) {
  const cudaStream_t st = fs[0]->st;
  const int B = ORB_MAX_BATCH;
  const size_t stride = J.head_bytes(std::min(B, n));     // one chunk's x, y, count and status on the host
  std::vector<char> h(stride * ((n + B - 1) / B));
  for (int c0 = 0; c0 < n; c0 += B) {
    const int m = std::min(B, n - c0);
    IngestImages im;
    std::memset(&im, 0, sizeof im);
    for (int i = 0; i < m; ++i) im.img[i] = gray_plane(fs[c0 + i]);
    if (int rc = orb_run_keys(J.ex, geo + c0, m, im, J.outs(m, J.buf), st)) return rc;
    VDO_CUDA(cudaMemcpyAsync(h.data() + stride * (c0 / B), J.buf, J.head_bytes(m), cudaMemcpyDeviceToHost, st));
  }
  VDO_CUDA(cudaStreamSynchronize(st));
  for (int c0 = 0; c0 < n; c0 += B) {
    const int m = std::min(B, n - c0);
    const vdo_orb_batch_out o = J.outs(m, h.data() + stride * (c0 / B));
    for (int i = 0; i < m; ++i) {
      if (o.status_dev[i]) return VDO_ERR_UNSUPPORTED;   // an octree bound breach: never expected (see k_octree)
      const float* x = o.x_dev + (size_t)i * J.cap; const float* y = o.y_dev + (size_t)i * J.cap;
      out[c0 + i].x.assign(x, x + o.count_dev[i]); out[c0 + i].y.assign(y, y + o.count_dev[i]);
    }
  }
  return VDO_OK;
}
}  // namespace vdo

extern "C" int vdo_orb_debug_octree(vdo_ctx* ctx, int n, const float* kx, const float* ky, const float* kr, int minX, int maxX, int minY, int maxY, int N,
                                    float* out_x, float* out_y, float* out_r, int* n_out, int* status) {
  if (!ctx || n < 0 || (n && (!kx || !ky || !kr || !out_x || !out_y || !out_r)) || !n_out || !status || N < 0 || maxY <= minY) return VDO_ERR_ARG;
  const int nini = (int)std::round(static_cast<float>(maxX - minX) / (maxY - minY));
  const int cap = std::max(oct_cap(N, nini), std::max(N + 2, 4));
  if (cap > OCT_MAX_CAP) return VDO_ERR_UNSUPPORTED;
  const cudaStream_t st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx);
  std::vector<KpOut> h(n);
  for (int i = 0; i < n; ++i) h[i] = KpOut{kx[i], ky[i], kr[i]};
  const OctLevel lv{minX, maxX, minY, maxY, N, cap, 0, 1, 0, 0};
  const int off[2] = {0, n};
  char* d = nullptr;
  const size_t nk = (size_t)std::max(n, 1);
  const size_t o_lv = 0, o_off = 64, o_dense = 128, o_knode = o_dense + sizeof(KpOut) * nk, o_nodes = (o_knode + 4 * nk + 63) & ~(size_t)63,
               o_ints = o_nodes + sizeof(OctNode) * 2 * cap, o_best = (o_ints + 4 * 11 * (size_t)cap + 63) & ~(size_t)63, o_kept = o_best + 8 * (size_t)cap,
               o_cnt = (o_kept + sizeof(KpOut) * cap + 63) & ~(size_t)63, o_st = o_cnt + 64, total = o_st + 64;
  VDO_CUDA(cudaMalloc(&d, total));
  auto run = [&]() -> int {
    VDO_CUDA(cudaMemsetAsync(d, 0, total, st));
    VDO_CUDA(cudaMemcpyAsync(d + o_lv, &lv, sizeof lv, cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(d + o_off, off, sizeof off, cudaMemcpyHostToDevice, st));
    if (n) VDO_CUDA(cudaMemcpyAsync(d + o_dense, h.data(), sizeof(KpOut) * n, cudaMemcpyHostToDevice, st));
    OctArgs a{(const OctLevel*)(d + o_lv), (const int*)(d + o_off), (const KpOut*)(d + o_dense), (int*)(d + o_knode),
              (OctNode*)(d + o_nodes), (int*)(d + o_ints), (unsigned long long*)(d + o_best), (KpOut*)(d + o_kept), (int*)(d + o_cnt), (int*)(d + o_st)};
    VDO_CUDA(cudaFuncSetAttribute(k_octree, cudaFuncAttributeMaxDynamicSharedMemorySize, oct_smem(OCT_MAX_CAP)));
    k_octree<<<1, 1024, oct_smem(cap), st>>>(a, nullptr);
    VDO_CUDA(cudaGetLastError());
    int cnt = 0;
    VDO_CUDA(cudaMemcpyAsync(&cnt, d + o_cnt, sizeof cnt, cudaMemcpyDeviceToHost, st));
    VDO_CUDA(cudaMemcpyAsync(status, d + o_st, sizeof(int), cudaMemcpyDeviceToHost, st));
    VDO_CUDA(cudaStreamSynchronize(st));
    std::vector<KpOut> k(cnt);
    if (cnt) {
      VDO_CUDA(cudaMemcpyAsync(k.data(), d + o_kept, sizeof(KpOut) * cnt, cudaMemcpyDeviceToHost, st));
      VDO_CUDA(cudaStreamSynchronize(st));
    }
    for (int i = 0; i < cnt; ++i) { out_x[i] = k[i].x; out_y[i] = k[i].y; out_r[i] = k[i].resp; }
    *n_out = cnt;
    return VDO_OK;
  };
  const int rc = run();
  cudaFree(d);
  return rc;
}
