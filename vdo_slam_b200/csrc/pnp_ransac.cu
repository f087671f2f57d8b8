// pnp_ransac.cu -- initial-model stage of the per-frame path (SURVEY.md 8 row A10 / N1): batched P3P + RANSAC on the
// device, constant-motion-model inlier test, choice of the initial model.
//
// Replaces: Tracking::GetInitModelCam / GetInitModelObj (src/Tracking.cc:1614-1715, 1717-1849) and the OpenCV 3.4
// cv::solvePnPRansac(..., 500, 0.4, 0.98, inliers, SOLVEPNP_AP3P) call inside them.
//
// Layout of one call (camera, or all objects of a frame as a batch):
//   k_pnp_hyp    one thread per (problem, RANSAC iteration): 4 sampled points -> P3P (Grunert quartic, Ferrari + bisection
//                on the resolvent, + - * / sqrt only) -> one model chosen by the 4th point
//   k_pnp_score  one CTA per (problem, iteration): inlier count of that model over the problem's points
//   k_pnp_finish one CTA per problem: replay of the sequential RANSAC bookkeeping over the 500 counts (strictly-better
//                replacement, adaptive iteration cap), ordered compaction of the winner's inliers, 8 Gauss-Newton refit steps
//                (fixed-order sums), constant-motion-model inliers in the reference's float arithmetic, choice of the model.
// The sample table is produced on the host by the same cv::RNG recurrence OpenCV uses (sequential by nature, 2000 draws).
//
// vdo_pnp_match_batch_dev runs the same three kernels on correspondences that exist only on the device (ORB matches of P frame pairs):
//   k_pnp_gather   one CTA per pair: ordered compaction of the valid matches into the pair's segment, back-projection through the query
//                  depth, local -> query index map, the pair's PnpProb
//   k_pnp_samples  one thread per pair: the sample table of make_samples for the pair's device count
//   k_pnp_hyp / k_pnp_score / k_pnp_finish   unchanged
//   k_pnp_scatter  one CTA per pair: PnpOut -> the caller's arrays, inlier flags per query keypoint
// This file is compiled with --fmad=false: with no contraction every operation rounds like the C oracle
// (oracle/pnp_ransac.c), so hypotheses, counts and inlier sets are bit-identical; only log/pow in the iteration-cap formula
// go through libm (their result is rounded to an integer).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/vdo_b200.h"
#include "dev_solvers.cuh"
#include "dev_entry.h"
#include "frame_batch.h"
#include "pnp_corr.cuh"

namespace {
constexpr int FIN_THREADS = 256;

using vdo::PnpProb;
using vdo::PnpOut;

__device__ __forceinline__ double poly4(const double* c, double x) { return (((c[0] * x + c[1]) * x + c[2]) * x + c[3]) * x + c[4]; }
__device__ __forceinline__ double dpoly4(const double* c, double x) { return ((4 * c[0] * x + 3 * c[1]) * x + 2 * c[2]) * x + c[3]; }

__device__ __forceinline__ int solve_quartic(const double* c, double* roots) {
  if (fabs(c[0]) < 1e-300) return 0;
  const double b = c[1] / c[0], cc = c[2] / c[0], d = c[3] / c[0], e = c[4] / c[0];
  const double b2 = b * b;
  const double p = cc - 3.0 * b2 / 8.0;
  const double q = d - b * cc / 2.0 + b2 * b / 8.0;
  const double r = e - b * d / 4.0 + b2 * cc / 16.0 - 3.0 * b2 * b2 / 256.0;
  double y[4]; int n = 0;
  const double k1 = p, k2 = p * p / 4.0 - r, k3 = -q * q / 8.0;
  double hi = 1.0 + fmax(fabs(k1), fmax(fabs(k2), fabs(k3))), lo = 0.0;
  for (int it = 0; it < 80; ++it) {
    const double m = 0.5 * (lo + hi);
    const double f = ((m + k1) * m + k2) * m + k3;
    if (f > 0) hi = m; else lo = m;
  }
  double m = 0.5 * (lo + hi);
  for (int it = 0; it < 3; ++it) {
    const double f = ((m + k1) * m + k2) * m + k3, df = (3.0 * m + 2.0 * k1) * m + k2;
    if (df != 0.0) { const double mn = m - f / df; if (mn > 0.0) m = mn; }
  }
  if (m > 1e-14 * (1.0 + fabs(p))) {
    const double s = sqrt(2.0 * m), h = p / 2.0 + m, g = q / (2.0 * s);
    double disc = s * s - 4.0 * (h + g);
    if (disc >= 0) { const double sq = sqrt(disc); y[n++] = 0.5 * (s + sq); y[n++] = 0.5 * (s - sq); }
    disc = s * s - 4.0 * (h - g);
    if (disc >= 0) { const double sq = sqrt(disc); y[n++] = 0.5 * (-s + sq); y[n++] = 0.5 * (-s - sq); }
  } else {
    const double disc = p * p - 4.0 * r;
    if (disc >= 0) {
      const double sq = sqrt(disc), z1 = 0.5 * (-p + sq), z2 = 0.5 * (-p - sq);
      if (z1 >= 0) { const double t = sqrt(z1); y[n++] = t; y[n++] = -t; }
      if (z2 >= 0) { const double t = sqrt(z2); y[n++] = t; y[n++] = -t; }
    }
  }
  for (int i = 0; i < n; ++i) {
    double x = y[i] - b / 4.0;
    for (int it = 0; it < 2; ++it) { const double df = dpoly4(c, x); if (df != 0.0) x = x - poly4(c, x) / df; }
    roots[i] = x;
  }
  return n;
}

struct V3 { double x, y, z; };
__device__ __forceinline__ V3 cross3(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ double dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ bool unit3(V3& a) { const double n = sqrt(dot3(a, a)); if (!(n > 1e-300)) return false; a.x = a.x / n; a.y = a.y / n; a.z = a.z / n; return true; }
struct Fr { V3 e1, e2, e3; bool ok; };
__device__ __forceinline__ Fr frame3(V3 A, V3 B, V3 C) {
  Fr f; f.ok = false;
  V3 ab{B.x - A.x, B.y - A.y, B.z - A.z}, ac{C.x - A.x, C.y - A.y, C.z - A.z};
  f.e1 = ab;
  if (!unit3(f.e1)) return f;
  f.e3 = cross3(f.e1, ac);
  if (!unit3(f.e3)) return f;
  f.e2 = cross3(f.e3, f.e1);
  f.ok = true;
  return f;
}
__device__ __forceinline__ double sqd(V3 a, V3 b) { return (a.x - b.x) * (a.x - b.x) + (a.y - b.y) * (a.y - b.y) + (a.z - b.z) * (a.z - b.z); }

// values are kept in named scalars / small structs (pointers to thread-local arrays across calls are avoided in this code base)
__device__ __forceinline__ bool p3p4(const V3* P, const double* uv, const double* K, double* Rt) {
  V3 f[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    f[k] = {(uv[2 * k] - K[2]) / K[0], (uv[2 * k + 1] - K[3]) / K[1], 1.0};
    if (!unit3(f[k])) return false;
  }
  const double d12 = sqd(P[1], P[2]), d02 = sqd(P[0], P[2]), d01 = sqd(P[0], P[1]);
  if (!(d02 > 1e-300) || !(d01 > 1e-300) || !(d12 > 1e-300)) return false;
  const double c12 = dot3(f[1], f[2]), c02 = dot3(f[0], f[2]), c01 = dot3(f[0], f[1]);
  const double K1 = (d12 - d01) / d02, K2 = d01 / d02;
  const double n2 = K1 - 1.0, n1 = -2.0 * K1 * c02, n0 = K1 + 1.0, e1 = -2.0 * c12, e0 = 2.0 * c01;
  const double q2 = -K2, q1 = 2.0 * K2 * c02, q0 = 1.0 - K2;
  double c[5];
  const double nd3 = n2 * e1, nd2 = n2 * e0 + n1 * e1, nd1 = n1 * e0 + n0 * e1, nd0 = n0 * e0;
  const double dd2 = e1 * e1, dd1 = 2.0 * e1 * e0, dd0 = e0 * e0;
  c[0] = n2 * n2 + dd2 * q2;
  c[1] = 2.0 * n2 * n1 - 2.0 * c01 * nd3 + (dd2 * q1 + dd1 * q2);
  c[2] = (2.0 * n2 * n0 + n1 * n1) - 2.0 * c01 * nd2 + (dd2 * q0 + dd1 * q1 + dd0 * q2);
  c[3] = 2.0 * n1 * n0 - 2.0 * c01 * nd1 + (dd1 * q0 + dd0 * q1);
  c[4] = n0 * n0 - 2.0 * c01 * nd0 + dd0 * q0;
  double roots[4];
  const int nr = solve_quartic(c, roots);
  const Fr E = frame3(P[0], P[1], P[2]);
  if (!E.ok) return false;
  double best = 1e300; bool found = false;
  for (int i = 0; i < nr; ++i) {
    const double v = roots[i];
    if (!(v > 0)) continue;
    const double D = e1 * v + e0;
    if (fabs(D) < 1e-12) continue;
    const double u = ((n2 * v + n1) * v + n0) / D;
    if (!(u > 0)) continue;
    const double den = 1.0 + v * v - 2.0 * v * c02;
    if (!(den > 0)) continue;
    const double s0 = sqrt(d02 / den), s1 = u * s0, s2 = v * s0;
    const V3 X0{s0 * f[0].x, s0 * f[0].y, s0 * f[0].z}, X1{s1 * f[1].x, s1 * f[1].y, s1 * f[1].z}, X2{s2 * f[2].x, s2 * f[2].y, s2 * f[2].z};
    const Fr G = frame3(X0, X1, X2);
    if (!G.ok) continue;
    double R[9], t[3];
    const double g1[3] = {G.e1.x, G.e1.y, G.e1.z}, g2[3] = {G.e2.x, G.e2.y, G.e2.z}, g3[3] = {G.e3.x, G.e3.y, G.e3.z};
    const double a1[3] = {E.e1.x, E.e1.y, E.e1.z}, a2[3] = {E.e2.x, E.e2.y, E.e2.z}, a3[3] = {E.e3.x, E.e3.y, E.e3.z};
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) R[3 * a + b] = g1[a] * a1[b] + g2[a] * a2[b] + g3[a] * a3[b];
    const double x0[3] = {X0.x, X0.y, X0.z};
#pragma unroll
    for (int a = 0; a < 3; ++a) t[a] = x0[a] - (R[3 * a] * P[0].x + R[3 * a + 1] * P[0].y + R[3 * a + 2] * P[0].z);
    const V3 P3 = P[3];
    const double xc = R[0] * P3.x + R[1] * P3.y + R[2] * P3.z + t[0], yc = R[3] * P3.x + R[4] * P3.y + R[5] * P3.z + t[1],
                 zc = R[6] * P3.x + R[7] * P3.y + R[8] * P3.z + t[2];
    if (!(zc > 0)) continue;
    const double du = K[0] * xc / zc + K[2] - uv[6], dv = K[1] * yc / zc + K[3] - uv[7];
    const double err = du * du + dv * dv;
    if (err < best) {
      best = err; found = true;
#pragma unroll
      for (int a = 0; a < 9; ++a) Rt[a] = R[a];
      Rt[9] = t[0]; Rt[10] = t[1]; Rt[11] = t[2];
    }
  }
  return found;
}

__device__ __forceinline__ bool is_inlier(const double* Rt, const float* o, const float* m, const double* K, float thr2) {
  const double X = o[0], Y = o[1], Z = o[2];
  const double xc = Rt[0] * X + Rt[1] * Y + Rt[2] * Z + Rt[9], yc = Rt[3] * X + Rt[4] * Y + Rt[5] * Z + Rt[10], zc = Rt[6] * X + Rt[7] * Y + Rt[8] * Z + Rt[11];
  const double iz = zc != 0.0 ? 1.0 / zc : 1.0;
  const float pu = (float)(K[0] * (xc * iz) + K[2]), pv = (float)(K[1] * (yc * iz) + K[3]);
  const float du = m[0] - pu, dv = m[1] - pv;
  const float err = du * du + dv * dv;
  return err <= thr2;
}

__global__ void k_pnp_hyp(const PnpProb* __restrict__ prob, const float* __restrict__ obj, const float* __restrict__ img, const int* __restrict__ samples,
                          int iters, double* __restrict__ models, int* __restrict__ counts) {
  const int it = blockIdx.x * blockDim.x + threadIdx.x, p = blockIdx.y;
  if (it >= iters) return;
  const PnpProb pr = prob[p];
  const size_t h = (size_t)p * iters + it;
  if (pr.n < 4) { counts[h] = -1; return; }
  V3 P[4]; double uv[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = pr.off + samples[4 * h + k];
    P[k] = {(double)obj[3 * i], (double)obj[3 * i + 1], (double)obj[3 * i + 2]};
    uv[2 * k] = img[2 * i]; uv[2 * k + 1] = img[2 * i + 1];
  }
  double M[12];
  const bool ok = p3p4(P, uv, pr.K, M);
  counts[h] = ok ? 0 : -1;
  if (ok) for (int a = 0; a < 12; ++a) models[12 * h + a] = M[a];
}

__global__ void __launch_bounds__(128) k_pnp_score(const PnpProb* __restrict__ prob, const float* __restrict__ obj, const float* __restrict__ img, int iters, float thr2,
                                                   const double* __restrict__ models, int* __restrict__ counts) {
  const int it = blockIdx.x, p = blockIdx.y;
  const size_t h = (size_t)p * iters + it;
  if (counts[h] < 0) return;
  __shared__ double M[12]; __shared__ double K[4]; __shared__ int cnt; __shared__ int off, n;
  if (threadIdx.x < 12) M[threadIdx.x] = models[12 * h + threadIdx.x];
  if (threadIdx.x == 0) { cnt = 0; off = prob[p].off; n = prob[p].n; }
  if (threadIdx.x < 4) K[threadIdx.x] = prob[p].K[threadIdx.x];
  __syncthreads();
  int c = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) c += is_inlier(M, obj + 3 * (size_t)(off + i), img + 2 * (size_t)(off + i), K, thr2) ? 1 : 0;
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&cnt, c);
  __syncthreads();
  if (threadIdx.x == 0) counts[h] = cnt;
}

__device__ __forceinline__ int update_num_iters(double p, double ep, int model_points, int max_iters) {
  p = fmin(fmax(p, 0.), 1.); ep = fmin(fmax(ep, 0.), 1.);
  double num = fmax(1. - p, 2.2250738585072014e-308), denom = 1. - pow(1. - ep, (double)model_points);
  if (denom < 2.2250738585072014e-308) return 0;
  num = log(num); denom = log(denom);
  return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : __double2int_rn(num / denom);
}

struct PredRansac {
  const double* Rt; const float* obj; const float* img; const double* K; float thr2;
  __device__ __forceinline__ bool operator()(int i) const { return is_inlier(Rt, obj + 3 * (size_t)i, img + 2 * (size_t)i, K, thr2); }
};
// Tracking.cc:1676-1691: x3D_c = R x + t as a float gemm (double accumulation, one rounding), then float projection
struct PredMm {
  const float* T; const float* Kf; const float* obj; const float* img; double thr;
  __device__ __forceinline__ bool operator()(int i) const {
    const float* o = obj + 3 * (size_t)i; const float* m = img + 2 * (size_t)i;
    const float xc = (float)((double)T[0] * o[0] + (double)T[1] * o[1] + (double)T[2] * o[2] + (double)T[3]);
    const float yc = (float)((double)T[4] * o[0] + (double)T[5] * o[1] + (double)T[6] * o[2] + (double)T[7]);
    const float zc = (float)((double)T[8] * o[0] + (double)T[9] * o[1] + (double)T[10] * o[2] + (double)T[11]);
    const float invz = (float)(1.0 / (double)zc);
    const float u = Kf[0] * xc * invz + Kf[2], v = Kf[1] * yc * invz + Kf[3];
    const float u_ = m[0] - u, v_ = m[1] - v;
    const float rpe = sqrtf(u_ * u_ + v_ * v_);
    return (double)rpe < thr;
  }
};

__global__ void __launch_bounds__(FIN_THREADS) k_pnp_finish(const PnpProb* __restrict__ prob, const float* __restrict__ obj_all, const float* __restrict__ img_all,
                                                            int iters, double thr, double conf, const double* __restrict__ models, const int* __restrict__ counts,
                                                            PnpOut* __restrict__ out, int* __restrict__ ransac_idx, int* __restrict__ mm_idx, int* __restrict__ sub_idx) {
  const int p = blockIdx.x, tid = threadIdx.x;
  __shared__ PnpProb pr;
  __shared__ double Rt[12];
  __shared__ int s_scan[FIN_THREADS];
  __shared__ double s_red[FIN_THREADS];
  __shared__ double s_sum[27];
  __shared__ int s_best, s_run, s_valid, s_ok, s_base;
  if (tid == 0) pr = prob[p];
  __syncthreads();
  const float* obj = obj_all + 3 * (size_t)pr.off; const float* img = img_all + 2 * (size_t)pr.off;
  int* r_idx = ransac_idx + pr.off; int* m_idx = mm_idx + pr.off; int* s_idx = sub_idx + pr.off;
  const float thr2 = (float)(thr * thr);
  if (tid == 0) {                      // replay of RANSACPointSetRegistrator::run over the precomputed counts
    int niters = iters, best = 0, best_it = -1, nvalid = 0, it = 0;
    if (pr.n >= 4)
      for (; it < niters; ++it) {
        const int c = counts[(size_t)p * iters + it];
        if (c < 0) continue;
        ++nvalid;
        if (c > (best > 3 ? best : 3)) { best = c; best_it = it; niters = update_num_iters(conf, (double)(pr.n - c) / pr.n, 4, niters); }
      }
    s_best = best_it; s_run = it; s_valid = nvalid;
  }
  __syncthreads();
  int n_ransac = 0;
  if (s_best >= 0) {
    if (tid < 12) Rt[tid] = models[12 * ((size_t)p * iters + s_best) + tid];
    __syncthreads();
    if (tid < 12) out[p].Rt_hyp[tid] = Rt[tid];
    const PredRansac ia{Rt, obj, img, pr.K, thr2};
    n_ransac = compact_ordered<FIN_THREADS>(pr.n, ia, r_idx, s_scan, &s_base);
    // ---- Gauss-Newton refit, 8 steps, lane-strided partial sums folded 128..1 ----
    for (int step = 0; step < 8; ++step) {
      double acc[27];
#pragma unroll
      for (int k = 0; k < 27; ++k) acc[k] = 0.0;
      for (int q = tid; q < n_ransac; q += FIN_THREADS) {
        const float* o = obj + 3 * (size_t)r_idx[q]; const float* m = img + 2 * (size_t)r_idx[q];
        const double X = o[0], Y = o[1], Z = o[2];
        const double xc = Rt[0] * X + Rt[1] * Y + Rt[2] * Z + Rt[9], yc = Rt[3] * X + Rt[4] * Y + Rt[5] * Z + Rt[10], zc = Rt[6] * X + Rt[7] * Y + Rt[8] * Z + Rt[11];
        const double iz = 1.0 / zc;
        const double ru = pr.K[0] * xc * iz + pr.K[2] - (double)m[0], rv = pr.K[1] * yc * iz + pr.K[3] - (double)m[1];
        const double a0 = pr.K[0] * iz, a2 = -pr.K[0] * xc * iz * iz, b1 = pr.K[1] * iz, b2 = -pr.K[1] * yc * iz * iz;
        double Ju[6], Jv[6];
        Ju[0] = 2.0 * (a2 * yc);             Ju[1] = 2.0 * (a0 * zc - a2 * xc); Ju[2] = 2.0 * (-a0 * yc);
        Jv[0] = 2.0 * (-b1 * zc + b2 * yc);  Jv[1] = 2.0 * (-b2 * xc);          Jv[2] = 2.0 * (b1 * xc);
        Ju[3] = a0; Ju[4] = 0.0; Ju[5] = a2; Jv[3] = 0.0; Jv[4] = b1; Jv[5] = b2;
        int k = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
          for (int b = a; b < 6; ++b) { acc[k] = acc[k] + (Ju[a] * Ju[b] + Jv[a] * Jv[b]); ++k; }
#pragma unroll
        for (int a = 0; a < 6; ++a) acc[21 + a] = acc[21 + a] + (Ju[a] * ru + Jv[a] * rv);
      }
#pragma unroll 1
      for (int k = 0; k < 27; ++k) {
        s_red[tid] = acc[k];
        __syncthreads();
        for (int s = FIN_THREADS / 2; s >= 1; s >>= 1) {
          if (tid < s) s_red[tid] = s_red[tid] + s_red[tid + s];
          __syncthreads();
        }
        if (tid == 0) s_sum[k] = s_red[0];
        __syncthreads();
      }
      if (tid == 0) {
        double H[36], g[6], x[6];
        int k = 0;
        for (int a = 0; a < 6; ++a)
          for (int b = a; b < 6; ++b) { H[6 * a + b] = s_sum[k]; H[6 * b + a] = s_sum[k]; ++k; }
        for (int a = 0; a < 6; ++a) g[a] = -s_sum[21 + a];
        bool ok = true;
        for (int j = 0; j < 6 && ok; ++j) {
          double s = H[7 * j];
          for (int kk = 0; kk < j; ++kk) s = s - H[6 * j + kk] * H[6 * j + kk];
          if (!(s > 0)) { ok = false; break; }
          const double l = sqrt(s); H[7 * j] = l;
          for (int i = j + 1; i < 6; ++i) {
            double v = H[6 * i + j];
            for (int kk = 0; kk < j; ++kk) v = v - H[6 * i + kk] * H[6 * j + kk];
            H[6 * i + j] = v / l;
          }
        }
        if (ok) {
          double y[6];
          for (int i = 0; i < 6; ++i) { double v = g[i]; for (int kk = 0; kk < i; ++kk) v = v - H[6 * i + kk] * y[kk]; y[i] = v / H[7 * i]; }
          for (int i = 5; i >= 0; --i) { double v = y[i]; for (int kk = i + 1; kk < 6; ++kk) v = v - H[6 * kk + i] * x[kk]; x[i] = v / H[7 * i]; }
          const double w0 = x[0], w1 = x[1], w2 = x[2], nn = w0 * w0 + w1 * w1 + w2 * w2, sc = 2.0 / (1.0 + nn);
          const double C[9] = {1.0 + sc * (-(w1 * w1 + w2 * w2)), sc * (-w2 + w0 * w1), sc * (w1 + w0 * w2),
                               sc * (w2 + w0 * w1), 1.0 + sc * (-(w0 * w0 + w2 * w2)), sc * (-w0 + w1 * w2),
                               sc * (-w1 + w0 * w2), sc * (w0 + w1 * w2), 1.0 + sc * (-(w0 * w0 + w1 * w1))};
          double Rn[12];
          for (int a = 0; a < 3; ++a) {
            for (int b = 0; b < 3; ++b) Rn[3 * a + b] = C[3 * a] * Rt[b] + C[3 * a + 1] * Rt[3 + b] + C[3 * a + 2] * Rt[6 + b];
            Rn[9 + a] = C[3 * a] * Rt[9] + C[3 * a + 1] * Rt[10] + C[3 * a + 2] * Rt[11] + x[3 + a];
          }
          for (int a = 0; a < 12; ++a) Rt[a] = Rn[a];
        }
        s_ok = ok ? 1 : 0;
      }
      __syncthreads();
      if (!s_ok) break;
    }
    if (tid < 12) out[p].Rt[tid] = Rt[tid];
  }
  __syncthreads();
  // ---- constant-motion model ----
  int n_mm = 0;
  if (pr.has_mm) {
    const PredMm ma{pr.mm, pr.Kf, obj, img, thr};
    n_mm = compact_ordered<FIN_THREADS>(pr.n, ma, m_idx, s_scan, &s_base);
  }
  // ---- choice (Tracking.cc:1694-1712 / 1807-1839): RANSAC wins only with strictly more inliers; objects without a previous motion use RANSAC ----
  const bool use_mm = pr.has_mm && !(n_ransac > n_mm);
  const int n_sub = use_mm ? n_mm : n_ransac;
  for (int q = tid; q < n_sub; q += FIN_THREADS) s_idx[q] = use_mm ? m_idx[q] : r_idx[q];
  if (tid == 0) {
    PnpOut& o = out[p];
    o.n_ransac = n_ransac; o.n_mm = n_mm; o.used_mm = use_mm ? 1 : 0; o.n_sub = n_sub; o.iters_run = s_run; o.best_it = s_best; o.n_valid = s_valid;
    float T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    if (use_mm) { for (int a = 0; a < 12; ++a) T[a] = pr.mm[a]; }
    else if (s_best >= 0) {
      for (int a = 0; a < 3; ++a) { for (int b = 0; b < 3; ++b) T[4 * a + b] = (float)Rt[3 * a + b]; T[4 * a + 3] = (float)Rt[9 + a]; }
    }
    for (int a = 0; a < 16; ++a) o.T[a] = T[a];
  }
}

struct PnpArena {
  size_t cap_pts = 0, cap_prob = 0, cap_hyp = 0;
  float *obj = 0, *img = 0;
  int *r_idx = 0, *m_idx = 0, *s_idx = 0, *samples = 0, *counts = 0;
  double* models = 0;
  PnpProb *prob = 0, *h_prob = 0;
  PnpOut *out = 0, *h_out = 0;
  int* h_samples = 0;
  std::map<int, std::vector<int>> sample_cache;      // n -> iters*4 indices (the draw sequence depends on n only)
  int cache_iters = 0;
  int launches = 0;
};
std::mutex g_mu;
std::map<uint64_t, PnpArena> g_arenas;

struct CvRng { uint64_t s; __host__ __device__ unsigned next() { s = (uint64_t)(unsigned)s * 4164903690U + (unsigned)(s >> 32); return (unsigned)s; } };
void make_samples(int n, int iters, int* idx) {
  CvRng r{(uint64_t)-1};
  for (int it = 0; it < iters; ++it)
    for (int i = 0; i < 4; ++i)
      for (;;) {
        const int v = (int)(r.next() % (unsigned)n); int j;
        idx[4 * it + i] = v;
        for (j = 0; j < i; ++j) if (idx[4 * it + j] == v) break;
        if (j == i) break;
      }
}

// ---- vdo_pnp_match_batch_dev: correspondences gathered from ORB matches, sample table drawn on the device ----
// one CTA per pair: ordered compaction of the correspondences into the pair's segment (local -> query index map in lmap), then the
// back-projection (Frame::UnprojectStereoStat in float; with Tcw, the world point as tracker.cpp's unproject_world rounds it) and the
// train keypoint of each, and the pair's PnpProb
__global__ void __launch_bounds__(FIN_THREADS) k_pnp_gather(const __grid_constant__ PnpGatherArg a,PnpProb* __restrict__ prob, float* __restrict__ obj, float* __restrict__ img,
                                                            int* __restrict__ lmap, int* __restrict__ nq_out, int* __restrict__ status) {
  const int p = blockIdx.x, tid = threadIdx.x;
  __shared__ int s_scan[FIN_THREADS];
  __shared__ int s_base;
  const PnpPairArg& pa = a.pr[p];
  const int cq = a.qcount[pa.q], ct = a.tcount[pa.t];
  const int nq = valid_count(cq, a.qcap), nt = valid_count(ct, a.tcap);
  const size_t off = (size_t)p * a.seg;
  const PredCorr pc{&a, &pa, a.qx + (size_t)pa.q * a.qcap, a.qy + (size_t)pa.q * a.qcap, a.idx + (size_t)p * a.qcap * a.k, a.dist + (size_t)p * a.qcap * a.k, nt};
  const int n = compact_ordered<FIN_THREADS>(nq, pc, lmap + off, s_scan, &s_base);
  const float* tx = a.tx + (size_t)pa.t * a.tcap; const float* ty = a.ty + (size_t)pa.t * a.tcap;
  const float invfx = 1.0f / pa.Kq[0], invfy = 1.0f / pa.Kq[1];
  for (int r = tid; r < n; r += FIN_THREADS) {
    const int i = lmap[off + r], j = pc.idx[(size_t)i * a.k];
    float z;
    pc.depth_at(i, &z);
    const float u = pc.qx[i], v = pc.qy[i];
    const float x = (u - pa.Kq[2]) * z * invfx, y = (v - pa.Kq[3]) * z * invfy;
    float* o = obj + 3 * (off + r);
    if (pa.has_T) {
      const float* T = pa.T;
      for (int c = 0; c < 3; ++c) {
        const double twl = (double)(float)(-((double)T[c] * (double)T[3] + (double)T[4 + c] * (double)T[7] + (double)T[8 + c] * (double)T[11]));
        o[c] = (float)((double)T[c] * (double)x + (double)T[4 + c] * (double)y + (double)T[8 + c] * (double)z + twl);
      }
    } else { o[0] = x; o[1] = y; o[2] = z; }
    img[2 * (off + r)] = tx[j]; img[2 * (off + r) + 1] = ty[j];
  }
  if (tid == 0) {
    PnpProb pb;
    pb.off = (int)off; pb.n = n;
    for (int c = 0; c < 4; ++c) { pb.K[c] = (double)pa.Kt[c]; pb.Kf[c] = pa.Kt[c]; }
    for (int c = 0; c < 12; ++c) pb.mm[c] = 0.f;
    pb.has_mm = 0; pb.pad = 0;
    prob[p] = pb;
    nq_out[p] = nq;
    status[p] = (cq == nq ? 0 : VDO_PNP_STATUS_QUERY_COUNT) | (ct == nt ? 0 : VDO_PNP_STATUS_TRAIN_COUNT);
  }
}

// the sample table of make_samples for each pair's device count: the draws of cv::RNG(-1) are one sequential recurrence, so one thread
// draws a pair's whole table (a pair with n < 4 gets none: k_pnp_hyp does not read it)
__global__ void k_pnp_samples(const PnpProb* __restrict__ prob, int P, int iters, int* __restrict__ samples) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int n = prob[p].n;
  if (n < 4) return;
  int4* dst = reinterpret_cast<int4*>(samples) + (size_t)p * iters;
  CvRng r{(uint64_t)-1};
  for (int it = 0; it < iters; ++it) {
    int s[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      for (;;) {
        const int v = (int)(r.next() % (unsigned)n);
        bool dup = false;
#pragma unroll
        for (int j = 0; j < i; ++j) dup = dup || s[j] == v;
        s[i] = v;
        if (!dup) break;
      }
    dst[it] = make_int4(s[0], s[1], s[2], s[3]);
  }
}

// k_pnp_finish's PnpOut -> the caller's outputs; the inlier flags of the query keypoints through the local -> query map
__global__ void __launch_bounds__(FIN_THREADS) k_pnp_scatter(const PnpProb* __restrict__ prob, const PnpOut* __restrict__ res, const int* __restrict__ ransac_idx,
                                                             const int* __restrict__ lmap, const int* __restrict__ nq_in, const int* __restrict__ status, int qcap,
                                                             vdo_pnp_out o) {
  const int p = blockIdx.x, tid = threadIdx.x;
  const PnpProb& pr = prob[p];
  const PnpOut& r = res[p];
  const bool model = pr.n >= 4 && r.best_it >= 0;
  const int n_in = model ? r.n_ransac : 0;
  uint8_t* row = o.inlier_dev + (size_t)p * qcap;
  for (int i = tid; i < nq_in[p]; i += FIN_THREADS) row[i] = 0;
  __syncthreads();
  for (int k = tid; k < n_in; k += FIN_THREADS) row[lmap[pr.off + ransac_idx[pr.off + k]]] = 1;
  if (tid < 16) o.T_dev[16 * p + tid] = r.T[tid];
  if (o.Rt_dev && tid < 12) o.Rt_dev[12 * p + tid] = model ? r.Rt[tid] : (tid == 0 || tid == 4 || tid == 8 ? 1.0 : 0.0);
  if (tid == 0) {
    o.n_corr_dev[p] = pr.n;
    o.n_inlier_dev[p] = n_in;
    int* info = o.info_dev + 4 * p;
    info[0] = r.iters_run; info[1] = r.best_it; info[2] = r.n_valid;
    info[3] = status[p] | (pr.n < 4 ? VDO_PNP_STATUS_FEW_POINTS : 0) | (pr.n >= 4 && r.best_it < 0 ? VDO_PNP_STATUS_NO_MODEL : 0);
  }
}
}  // namespace

// T_mm: nprob x 16 (4x4 row-major float) constant-motion models, has_mm: nprob flags (NULL = none).  K4 = fx, fy, cx, cy.
// Outputs per problem: T_init (16 floats), n_sub + sub_idx (local ascending indices of the chosen inlier set, written at the
// problem's offset), info (nprob x 8 ints: n_ransac, n_mm, used_mm, n_sub, iterations run, winning iteration, valid hypotheses, 0),
// Rt_refit / Rt_hyp (nprob x 12 doubles, may be NULL; test hooks).
extern "C" int vdo_init_model_batch(vdo_ctx* ctx, int nprob, const int* offsets, const float* obj3d, const float* img2d, const float* K4, int iters,
                                    double thr, double conf, const float* T_mm, const unsigned char* has_mm, float* T_init, int* n_sub, int* sub_idx,
                                    int* info, double* Rt_refit, double* Rt_hyp) {
  return vdo::init_model_batch(ctx, nprob, offsets, obj3d, img2d, K4, 0, iters, thr, conf, T_mm, has_mm, T_init, n_sub, sub_idx, info, Rt_refit, Rt_hyp);
}
// the same with intrinsics K4 + k_stride * p for problem p: the tracker batches the problems of several sequences, each with its own K
int vdo::init_model_batch(vdo_ctx* ctx, int nprob, const int* offsets, const float* obj3d, const float* img2d, const float* K4, int k_stride, int iters,
                          double thr, double conf, const float* T_mm, const unsigned char* has_mm, float* T_init, int* n_sub, int* sub_idx, int* info,
                          double* Rt_refit, double* Rt_hyp) {
  if (!ctx || nprob <= 0 || !offsets || !K4 || iters <= 0 || iters > 4096) return VDO_ERR_ARG;
  cudaStream_t st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx);
  std::lock_guard<std::mutex> lk(g_mu);
  PnpArena& A = g_arenas[(uint64_t)(uintptr_t)st];
  const size_t total = (size_t)offsets[nprob];
  if (total > A.cap_pts) {
    const size_t cap = total * 2 + 1024;
    cudaFree(A.obj); cudaFree(A.img); cudaFree(A.r_idx); cudaFree(A.m_idx); cudaFree(A.s_idx);
    VDO_CUDA(cudaMalloc(&A.obj, cap * 12)); VDO_CUDA(cudaMalloc(&A.img, cap * 8)); VDO_CUDA(cudaMalloc(&A.r_idx, cap * 4)); VDO_CUDA(cudaMalloc(&A.m_idx, cap * 4)); VDO_CUDA(cudaMalloc(&A.s_idx, cap * 4));
    A.cap_pts = cap;
  }
  const size_t nh = (size_t)nprob * iters;
  if ((size_t)nprob > A.cap_prob || nh > A.cap_hyp) {
    const size_t cp = (size_t)nprob * 2 + 8, ch = cp * iters;
    cudaFree(A.prob); cudaFree(A.out); cudaFree(A.samples); cudaFree(A.counts); cudaFree(A.models);
    cudaFreeHost(A.h_prob); cudaFreeHost(A.h_out); cudaFreeHost(A.h_samples);
    VDO_CUDA(cudaMalloc(&A.prob, cp * sizeof(PnpProb))); VDO_CUDA(cudaMalloc(&A.out, cp * sizeof(PnpOut)));
    VDO_CUDA(cudaMalloc(&A.samples, ch * 16)); VDO_CUDA(cudaMalloc(&A.counts, ch * 4)); VDO_CUDA(cudaMalloc(&A.models, ch * 96));
    VDO_CUDA(cudaMallocHost(&A.h_prob, cp * sizeof(PnpProb))); VDO_CUDA(cudaMallocHost(&A.h_out, cp * sizeof(PnpOut))); VDO_CUDA(cudaMallocHost(&A.h_samples, ch * 16));
    A.cap_prob = cp; A.cap_hyp = ch;
  }
  if (A.cache_iters != iters) { A.sample_cache.clear(); A.cache_iters = iters; }
  for (int p = 0; p < nprob; ++p) {
    PnpProb& q = A.h_prob[p];
    q.off = offsets[p]; q.n = offsets[p + 1] - offsets[p];
    const float* Kp = K4 + (size_t)k_stride * p;
    for (int k = 0; k < 4; ++k) { q.K[k] = (double)Kp[k]; q.Kf[k] = Kp[k]; }
    q.has_mm = (T_mm && (!has_mm || has_mm[p])) ? 1 : 0; q.pad = 0;
    if (q.has_mm) std::memcpy(q.mm, T_mm + 16 * p, 48); else std::memset(q.mm, 0, 48);
    int* dst = A.h_samples + (size_t)p * iters * 4;
    if (q.n >= 4) {
      auto itc = A.sample_cache.find(q.n);
      if (itc == A.sample_cache.end()) {
        if (A.sample_cache.size() > 4096) A.sample_cache.clear();
        std::vector<int> v((size_t)iters * 4);
        make_samples(q.n, iters, v.data());
        itc = A.sample_cache.emplace(q.n, std::move(v)).first;
      }
      std::memcpy(dst, itc->second.data(), (size_t)iters * 16);
    } else std::memset(dst, 0, (size_t)iters * 16);
  }
  VDO_CUDA(cudaMemcpyAsync(A.prob, A.h_prob, nprob * sizeof(PnpProb), cudaMemcpyHostToDevice, st));
  VDO_CUDA(cudaMemcpyAsync(A.samples, A.h_samples, nh * 16, cudaMemcpyHostToDevice, st));
  if (total) {
    VDO_CUDA(cudaMemcpyAsync(A.obj, obj3d, total * 12, cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(A.img, img2d, total * 8, cudaMemcpyHostToDevice, st));
  }
  vdo::pnp_ransac_launch(A.prob, nprob, A.obj, A.img, A.samples, iters, thr, conf, A.models, A.counts, A.out, A.r_idx, A.m_idx, A.s_idx, st);
  A.launches += 3;
  VDO_CUDA(cudaGetLastError());
  VDO_CUDA(cudaMemcpyAsync(A.h_out, A.out, nprob * sizeof(PnpOut), cudaMemcpyDeviceToHost, st));
  if (total && sub_idx) VDO_CUDA(cudaMemcpyAsync(sub_idx, A.s_idx, total * 4, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  for (int p = 0; p < nprob; ++p) {
    const PnpOut& o = A.h_out[p];
    if (T_init) std::memcpy(T_init + 16 * p, o.T, 64);
    if (n_sub) n_sub[p] = o.n_sub;
    if (info) { int* d = info + 8 * p; d[0] = o.n_ransac; d[1] = o.n_mm; d[2] = o.used_mm; d[3] = o.n_sub; d[4] = o.iters_run; d[5] = o.best_it; d[6] = o.n_valid; d[7] = 0; }
    if (Rt_refit) std::memcpy(Rt_refit + 12 * p, o.Rt, 96);
    if (Rt_hyp) std::memcpy(Rt_hyp + 12 * p, o.Rt_hyp, 96);
  }
  return VDO_OK;
}

// ---- launchers for problems resident on the device (dev_solvers.cuh) ----
void vdo::pnp_samples_launch(const PnpProb* prob, int nprob, int iters, int* samples, cudaStream_t st) {
  k_pnp_samples<<<(nprob + PNP_MAX_PAIRS - 1) / PNP_MAX_PAIRS, PNP_MAX_PAIRS, 0, st>>>(prob, nprob, iters, samples);
}
void vdo::pnp_ransac_launch(const PnpProb* prob, int nprob, const float* obj, const float* img, const int* samples, int iters, double thr, double conf,
                            double* models, int* counts, PnpOut* out, int* r_idx, int* m_idx, int* s_idx, cudaStream_t st) {
  k_pnp_hyp<<<dim3((iters + 63) / 64, nprob), 64, 0, st>>>(prob, obj, img, samples, iters, models, counts);
  k_pnp_score<<<dim3(iters, nprob), 128, 0, st>>>(prob, obj, img, iters, (float)(thr * thr), models, counts);
  k_pnp_finish<<<nprob, FIN_THREADS, 0, st>>>(prob, obj, img, iters, thr, conf, models, counts, out, r_idx, m_idx, s_idx);
}

extern "C" int vdo_init_model_launches(vdo_ctx* ctx) {
  if (!ctx) return 0;
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_arenas.find((uint64_t)(uintptr_t)vdo_ctx_stream(ctx));
  return it == g_arenas.end() ? 0 : it->second.launches;
}

// ---- vdo_pnp_solver: the work space of vdo_pnp_match_batch_dev, all allocated at creation ----
struct vdo_pnp_solver : vdo::WorkSpace {
  vdo_ctx* ctx = nullptr;
  int dev = 0, max_pairs = 0, cap = 0, max_iters = 0;
  float *obj = nullptr, *img = nullptr;                                          // max_pairs x cap segments
  int *lmap = nullptr, *r_idx = nullptr, *m_idx = nullptr, *s_idx = nullptr;
  int *samples = nullptr, *counts = nullptr;                                     // max_pairs x max_iters (x 4)
  double* models = nullptr;
  PnpProb* prob = nullptr;
  PnpOut* res = nullptr;
  int *nq = nullptr, *status = nullptr;                                          // max_pairs
};

extern "C" int vdo_pnp_solver_create(vdo_ctx* ctx, int max_pairs, int cap, int max_iters, vdo_pnp_solver** out) {
  if (!ctx || !out) return VDO_ERR_ARG;
  *out = nullptr;
  if (max_pairs < 1 || max_pairs > PNP_MAX_PAIRS || cap < 1 || max_iters < 1 || max_iters > 4096) {
    vdo::ctx_set_error(ctx, "vdo_pnp_solver_create: max_pairs = " + std::to_string(max_pairs) + ", cap = " + std::to_string(cap) + ", max_iters = " +
                                std::to_string(max_iters) + "; expected 1 .. 64, >= 1, 1 .. 4096");
    return VDO_ERR_ARG;
  }
  vdo_pnp_solver* s = new vdo_pnp_solver;
  s->ctx = ctx; s->max_pairs = max_pairs; s->cap = cap; s->max_iters = max_iters;
  int n_sm = 0;
  vdo::ctx_device(ctx, &s->dev, &n_sm);
  const size_t pts = (size_t)max_pairs * cap, hyp = (size_t)max_pairs * max_iters;
  return vdo::create_done(ctx, "vdo_pnp_solver_create", s,
                          {s->alloc(s->obj, 3 * pts), s->alloc(s->img, 2 * pts), s->alloc(s->lmap, pts), s->alloc(s->r_idx, pts), s->alloc(s->m_idx, pts),
                           s->alloc(s->s_idx, pts), s->alloc(s->samples, 4 * hyp), s->alloc(s->counts, hyp), s->alloc(s->models, 12 * hyp),
                           s->alloc(s->prob, (size_t)max_pairs), s->alloc(s->res, (size_t)max_pairs), s->alloc(s->nq, (size_t)max_pairs),
                           s->alloc(s->status, (size_t)max_pairs)},
                          out);
}
extern "C" void vdo_pnp_solver_destroy(vdo_pnp_solver* s) { delete s; }
extern "C" int vdo_pnp_solver_info(const vdo_pnp_solver* s, int64_t out[4]) {
  if (!s || !out) return VDO_ERR_ARG;
  out[0] = s->max_pairs; out[1] = s->cap; out[2] = s->max_iters; out[3] = (int64_t)s->bytes;
  return VDO_OK;
}

extern "C" int vdo_pnp_match_batch_dev(vdo_pnp_solver* s, int P, const int32_t* pairs, const vdo_orb_desc_set* query, const vdo_orb_desc_set* train,
                                       const int32_t* idx_dev, const int32_t* dist_dev, const vdo_dev_plane* depth, const int32_t* depth_wh,
                                       const float* K_query, const float* K_train, const float* Tcw_query, const vdo_pnp_match_opts* opts,
                                       const vdo_pnp_out* out, uint64_t stream) {
  if (!s) return VDO_ERR_ARG;
  auto check_iters = [&]() -> std::string {
    const int it = opts->iters;
    return it < 1 || it > s->max_iters ? "iters = " + std::to_string(it) + " outside 1 .. " + std::to_string(s->max_iters) : "";
  };
  auto check_rest = [&](vdo::DevPtrs& ptrs) -> std::string {
    const vdo_pnp_match_opts& o = *opts;
    if (!(o.thr > 0.0)) return "thr = " + std::to_string(o.thr) + "; expected > 0";
    if (!(o.conf > 0.0 && o.conf < 1.0)) return "conf = " + std::to_string(o.conf) + "; expected inside (0, 1)";
    ptrs = {{out->T_dev, 4, "out.T_dev"}, {out->inlier_dev, 1, "out.inlier_dev"}, {out->n_corr_dev, 4, "out.n_corr_dev"},
            {out->n_inlier_dev, 4, "out.n_inlier_dev"}, {out->info_dev, 4, "out.info_dev"}, {out->Rt_dev, 8, "out.Rt_dev", out->Rt_dev != nullptr}};
    return "";
  };
  PnpGatherArg ga;
  if (std::string why = corr_check("solver", s->max_pairs, s->cap, s->dev, P, pairs, query, train, idx_dev, dist_dev, depth, depth_wh, "K_query", K_query,
                                   K_train, Tcw_query, opts, out, check_iters, check_rest, ga);
      !why.empty()) {
    vdo::ctx_set_error(s->ctx, "vdo_pnp_match_batch_dev: " + why);
    return VDO_ERR_ARG;
  }
  const vdo_pnp_match_opts& o = *opts;
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  k_pnp_gather<<<P, FIN_THREADS, 0, st>>>(ga, s->prob, s->obj, s->img, s->lmap, s->nq, s->status);
  vdo::pnp_samples_launch(s->prob, P, o.iters, s->samples, st);
  vdo::pnp_ransac_launch(s->prob, P, s->obj, s->img, s->samples, o.iters, o.thr, o.conf, s->models, s->counts, s->res, s->r_idx, s->m_idx, s->s_idx, st);
  k_pnp_scatter<<<P, FIN_THREADS, 0, st>>>(s->prob, s->res, s->r_idx, s->lmap, s->nq, s->status, query->cap, *out);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
