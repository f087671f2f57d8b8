// flow_lm.cu -- per-frame joint optical-flow / SE(3) refinement on sm_90a: the whole Levenberg-Marquardt solve of
// Optimizer::PoseOptimizationFlow2 (object motion) / PoseOptimizationFlow2Cam (camera pose) runs inside one kernel,
// a cluster of CTAs or one CTA per optimisation problem (all objects of a frame are batched into at most two launches),
// with no host round trips: this path is latency-bound (config 2: 2 000 points, ~0.2 MB per iteration), not bandwidth-bound.
//
// Reference semantics (see also oracle/flow_lm.c, which restates the same lines on the CPU):
//   graph                src/Optimizer.cc:2755-2972 (Flow2), :2333-2542 (Flow2Cam)
//   edges / vertices     g2o/types/types_six_dof_expmap.h:67-85,414-476 ; .cpp:772-775,805-845 ; types_sba.h:78-95
//   SE3Quat::exp, *      g2o/types/se3quat.h:58-60,105-122,228-262,286-291
//   LM + outer loop      g2o/core/optimization_algorithm_levenberg.cpp:61-164 ; sparse_optimizer.cpp:354-427
//   Schur + dense LDLT   g2o/core/block_solver.hpp:352-486 ; g2o/solvers/linear_solver_dense.h:65-113
//   quirk mode           SURVEY.md section 7.2 H1 (2-D flow vertices inside BlockSolver_6_3's 3x3 landmark blocks)
#include <cuda_runtime.h>
#include <cooperative_groups.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"
#include "dev_solvers.cuh"
#include "pnp_corr.cuh"

namespace {

constexpr int FL_THREADS = 512;
constexpr int FL_NV = 44;            // widest reduction: 36 (Schur matrix) + 6 (rhs) + 2 spare

using vdo::FlowProb;
using vdo::FlowDev;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

__device__ void quat_to_rot(const double* q, double* R) {
  double tx = 2 * q[0], ty = 2 * q[1], tz = 2 * q[2];
  double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3];
  double txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
  double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
__device__ void rot_to_quat(const double* R, double* q) {   // Eigen::Quaternion(Matrix3)
  double t = R[0] + R[4] + R[8];
  if (t > 0.0) {
    t = sqrt(t + 1.0); q[3] = 0.5 * t; t = 0.5 / t;
    q[0] = (R[7] - R[5]) * t; q[1] = (R[2] - R[6]) * t; q[2] = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[4 * i]) i = 2;
    int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    double qq[4];
    qq[i] = 0.5 * t; t = 0.5 / t;
    qq[3] = (R[3 * k + j] - R[3 * j + k]) * t; qq[j] = (R[3 * j + i] + R[3 * i + j]) * t; qq[k] = (R[3 * k + i] + R[3 * i + k]) * t;
    q[0] = qq[0]; q[1] = qq[1]; q[2] = qq[2]; q[3] = qq[3];
  }
}
__device__ void quat_normalize_pos(double* q) {   // SE3Quat::normalizeRotation
  if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
__device__ void m3mul(const double* a, const double* b, double* c) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) c[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}
// T <- exp(u) * T   (state: q[4] = {x,y,z,w}, t[3])
__device__ void se3_oplus(double* q, double* t, const double* u) {
  const double om[3] = {u[0], u[1], u[2]}, up[3] = {u[3], u[4], u[5]};
  const double th = sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
  const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
  double O2[9], R[9], V[9];
  m3mul(O, O, O2);
  if (th < 0.00001) {
    for (int i = 0; i < 9; ++i) R[i] = O[i] + O2[i];
    R[0] += 1; R[4] += 1; R[8] += 1;
    for (int i = 0; i < 9; ++i) V[i] = R[i];
  } else {
    const double a = sin(th) / th, b = (1 - cos(th)) / (th * th), c = (th - sin(th)) / pow(th, 3.0);
    for (int i = 0; i < 9; ++i) { R[i] = a * O[i] + b * O2[i]; V[i] = b * O[i] + c * O2[i]; }
    R[0] += 1; R[4] += 1; R[8] += 1; V[0] += 1; V[4] += 1; V[8] += 1;
  }
  double qi[4], ti[3];
  rot_to_quat(R, qi);
  for (int i = 0; i < 3; ++i) ti[i] = V[3 * i] * up[0] + V[3 * i + 1] * up[1] + V[3 * i + 2] * up[2];
  quat_normalize_pos(qi);
  double Ri[9], rt[3], qn[4];
  quat_to_rot(qi, Ri);
  for (int i = 0; i < 3; ++i) rt[i] = Ri[3 * i] * t[0] + Ri[3 * i + 1] * t[1] + Ri[3 * i + 2] * t[2];
  qn[3] = qi[3] * q[3] - qi[0] * q[0] - qi[1] * q[1] - qi[2] * q[2];
  qn[0] = qi[3] * q[0] + qi[0] * q[3] + qi[1] * q[2] - qi[2] * q[1];
  qn[1] = qi[3] * q[1] + qi[1] * q[3] + qi[2] * q[0] - qi[0] * q[2];
  qn[2] = qi[3] * q[2] + qi[2] * q[3] + qi[0] * q[1] - qi[1] * q[0];
  for (int i = 0; i < 3; ++i) t[i] = ti[i] + rt[i];
  for (int i = 0; i < 4; ++i) q[i] = qn[i];
  quat_normalize_pos(q);
}
// Cholesky solve of the symmetric matrix given by the LOWER triangle of S (what Eigen's LDLT reads).
// L (36) and y (6) are caller-provided work arrays (shared memory).
__device__ bool solve6_lower(const double* S, const double* g, double* x, double* L, double* y) {
  for (int i = 0; i < 36; ++i) L[i] = 0;
  for (int j = 0; j < 6; ++j) {
    double d = S[7 * j];
    for (int k = 0; k < j; ++k) d -= L[6 * j + k] * L[6 * j + k];
    if (!(d > 0)) return false;
    d = sqrt(d);
    L[7 * j] = d;
    for (int i = j + 1; i < 6; ++i) {
      double s = S[6 * i + j];
      for (int k = 0; k < j; ++k) s -= L[6 * i + k] * L[6 * j + k];
      L[6 * i + j] = s / d;
    }
  }
  for (int i = 0; i < 6; ++i) { double s = g[i]; for (int k = 0; k < i; ++k) s -= L[6 * i + k] * y[k]; y[i] = s / L[7 * i]; }
  for (int i = 5; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < 6; ++k) s -= L[6 * k + i] * x[k]; x[i] = s / L[7 * i]; }
  return true;
}
__device__ __forceinline__ void huber_f(double e2, double delta, double dsqr, double& rho, double& w) {
  if (e2 <= dsqr) { rho = e2; w = 1.0; }
  else { const double s = sqrt(e2); rho = 2 * s * delta - dsqr; w = delta / s; }
}

struct FlowShared {
  double q[4], t[3], R[9];
  double qbk[4], tbk[3];
  double xp[6], Hpp[36], bp[6];
  double Sm[36], g[6], x[6], L[36], y[6];
  double lambda, ni, current, temp, rho, chi2_check, last_trial_chi;
  int nbad, qmax, ok, ok2, accept, iters, trials, stop_trials;
  int stop;                           // VDO_FLOW2_STOP_* once ok drops to 0
  int refresh;                        // the next iteration must recompute the errors and chi2 first (see end_iteration)
};

// trace writes of thread 0 (tr: this problem's trace, or NULL)
__device__ void trace_copy(double* dst, const double* src, int k) { for (int i = 0; i < k; ++i) dst[i] = src[i]; }
__device__ void trace_trial(double* tr, const FlowShared& S, int it, double lambda, double temp, double cur0, double scale) {
  if (S.trials >= VDO_FLOW2_TRACE_MAXREC) return;
  double* r = tr + VDO_FLOW2_TRACE_REC + (size_t)VDO_FLOW2_TRACE_RECLEN * S.trials;
  r[0] = it; r[1] = lambda; r[2] = S.ok2; r[3] = temp; r[4] = cur0; r[5] = scale; r[6] = S.rho; r[7] = S.accept;
  trace_copy(r + 8, S.xp, 6);
}
// end of an LM iteration (sparse_optimizer.cpp:354-427): decides whether the next one runs
__device__ void end_iteration(FlowShared& S, int it, double ini) {
  S.iters++;
  if (S.qmax == 10 || S.rho == 0) { S.ok = 0; S.stop = S.qmax == 10 ? VDO_FLOW2_STOP_TRIALS : VDO_FLOW2_STOP_RHO_ZERO; }
  else { if ((ini - S.current) * 1e3 < ini) S.nbad++; else S.nbad = 0; if (S.nbad >= 3) { S.ok = 0; S.stop = VDO_FLOW2_STOP_NO_PROGRESS; } }
  if (S.chi2_check < S.last_trial_chi && it > 0) { if (S.ok) S.stop = VDO_FLOW2_STOP_CHI2_ROSE; S.ok = 0; }
  S.chi2_check = S.last_trial_chi;
  // g2o recomputes the errors and chi2 at the start of every iteration (optimization_algorithm_levenberg.cpp:75-82).  After an
  // accepted trial the errors are that state's and its chi2 is the trial's (current differs from it only when a failed solve was
  // accepted with current = DBL_MAX); after a rejected one the errors are the rejected state's, so the kernel recomputes them.
  if (S.accept) S.current = S.last_trial_chi;
  else S.refresh = 1;
}
__device__ void trace_end(double* tr, const FlowShared& S) {
  tr[VDO_FLOW2_TRACE_STOP] = S.ok ? VDO_FLOW2_STOP_MAX_ITERS : S.stop;
  tr[VDO_FLOW2_TRACE_NREC] = S.trials < VDO_FLOW2_TRACE_MAXREC ? S.trials : VDO_FLOW2_TRACE_MAXREC;
}

// -------------------------------------------------------------------------------------------------------------------------
// One LM body, two launch shapes.  A problem runs on CL CTAs of THREADS threads: a thread-block CLUSTER of FC_CL CTAs of FC_THREADS
// (k_flow2_lm_cl) or one CTA of FL_THREADS (k_flow2_lm).  CTA r owns the points [r * per, min(n, (r + 1) * per)), per = ceil(n / CL),
// one point per thread per pass.  Their state (FL_FIELDS doubles per point: world point, flow and its backup, error, the camera-frame
// point of the linearisation -- the 2x6 Jacobian is recomputed from it --, weight, H, b, delta) is structure-of-arrays: in the
// cluster's shared memory, or in the global scratch for the single CTA, whose problems do not fit there.  Sums over all points are
// formed per CTA (shuffles + one smem hop), published in the CTA's shared memory and, after ONE cluster barrier, read by every CTA
// through distributed shared memory and added in CTA order -- every CTA obtains bit-identical totals, so the scalar part of the
// iteration (6x6 Cholesky, exp-map update, lambda logic) is simply executed by thread 0 of every CTA on its own copy of the state: no
// broadcast, no second barrier.  The two shapes differ only in where the points live and in that last step of the sums; the number
// of threads sets the order of the sums, so a problem's result depends on its shape alone.
constexpr int FC_CL = 8, FC_THREADS = 256, FL_FIELDS = 18;
enum { C_XW = 0, C_F = 3, C_FBK = 5, C_ERR = 7, C_XL = 9, C_W = 12, C_H = 13, C_BL = 14, C_DL = 16 };

template <int WARPS>
struct FlowRed {
  double wred[WARPS * FL_NV];           // per-warp partials
  double part[2][FL_NV + 1];            // this CTA's partial sums (+ max), double-buffered across reductions (cluster shape)
  double tot[FL_NV + 1];                // totals over the problem
};
// NV sums (+ one max, HAS_MAX) over all threads of the problem's CL CTAs; afterwards R.tot[0..NV) (and R.tot[NV]) hold the totals in
// every CTA.  With one CTA its partial sums are the totals.
template <int NV, bool HAS_MAX, int CL, int WARPS>
__device__ __forceinline__ void lm_reduce(double* acc, double mx, FlowRed<WARPS>& R, int& phase) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    double v = warp_sum(acc[i]);
    if (lane == 0) R.wred[w * FL_NV + i] = v;
  }
  if (HAS_MAX) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
    if (lane == 0) R.wred[w * FL_NV + NV] = mx;
  }
  __syncthreads();
  double* mine = CL > 1 ? R.part[phase & 1] : R.tot;
  if (threadIdx.x < NV) {
    double s = 0;
    for (int k = 0; k < WARPS; ++k) s += R.wred[k * FL_NV + threadIdx.x];
    mine[threadIdx.x] = s;
  } else if (HAS_MAX && threadIdx.x == NV) {
    double m = 0;
    for (int k = 0; k < WARPS; ++k) m = fmax(m, R.wred[k * FL_NV + NV]);
    mine[NV] = m;
  }
  if constexpr (CL > 1) {
    cooperative_groups::cluster_group cl = cooperative_groups::this_cluster();
    cl.sync();
    if (threadIdx.x < NV) {
      double s = 0;
      for (int r = 0; r < CL; ++r) s += cl.map_shared_rank(mine, r)[threadIdx.x];
      R.tot[threadIdx.x] = s;
    } else if (HAS_MAX && threadIdx.x == NV) {
      double m = 0;
      for (int r = 0; r < CL; ++r) m = fmax(m, cl.map_shared_rank(mine, r)[NV]);
      R.tot[NV] = m;
    }
    ++phase;
  }
  __syncthreads();
}

// the problem's LM solve on CL CTAs of THREADS threads; pt: this CTA's points' state, field f of local point j at pt[f * ld + j]
template <int CL, int THREADS>
__device__ __forceinline__ void flow2_lm(const FlowDev& d, double* pt, int ld) {
  __shared__ FlowRed<THREADS / 32> R;
  __shared__ FlowShared S;
  const int crank = CL > 1 ? (int)cooperative_groups::this_cluster().block_rank() : 0, tid = threadIdx.x;
  const FlowProb P = d.prob[blockIdx.x / CL];
  const int n = P.n, out = P.out;
  double* const tr = (d.trace && crank == 0) ? d.trace + (size_t)out * VDO_FLOW2_TRACE_DOUBLES : nullptr;
  const float* pts = d.pts + 2 * (size_t)P.offset;
  const float* dep = d.depth + P.offset;
  const float* flo = d.flow + 2 * (size_t)P.offset;
  const double fx = P.K[0], fy = P.K[1], cx = P.K[2], cy = P.K[3];
  const double w_rep = 0.1, w_prior = P.mode ? 0.5 : 0.3;
  const double delta = (double)(float)sqrt((double)0.04f);
  const double dsqr = (double)(float)(delta * delta);
  const int max_iters = P.mode ? 200 : 100;
  // this CTA's points: [i0, i1)
  const int per = (n + CL - 1) / CL, i0 = min(n, crank * per), i1 = min(n, i0 + per), nloc = i1 - i0;
  int phase = 0;
#define PT(f, j) pt[(size_t)(f) * ld + (j)]
  if (n < 3) {   // reference: returns identity / 0 without optimising (Optimizer.cc:2449-2450, 2872-2873)
    if (crank == 0) {
      if (tid < 16) d.T_out[16 * out + tid] = (tid % 5 == 0) ? 1.f : 0.f;
      if (tid < 8) d.stats[8 * out + tid] = tid == 0 ? -1 : 0;
      if (tid == 0 && tr) { tr[VDO_FLOW2_TRACE_STOP] = VDO_FLOW2_STOP_FEW_POINTS; tr[VDO_FLOW2_TRACE_NREC] = 0; }
      for (int i = tid; i < n; i += THREADS) { d.inlier[P.offset + i] = 0; d.flow_out[2 * (size_t)(P.offset + i)] = flo[2 * i]; d.flow_out[2 * (size_t)(P.offset + i) + 1] = flo[2 * i + 1]; }
    }
    return;
  }
  // ---- setup: Twl in float (double accumulation, float result -- cv::Mat expression semantics), Xw per point ----
  if (tid == 0) {
    const float* M = P.T_init;
    double R0[9] = {M[0], M[1], M[2], M[4], M[5], M[6], M[8], M[9], M[10]};
    rot_to_quat(R0, S.q);
    S.t[0] = M[3]; S.t[1] = M[7]; S.t[2] = M[11];
    quat_normalize_pos(S.q);
    quat_to_rot(S.q, S.R);
    S.lambda = -1; S.ni = 2; S.nbad = 0; S.ok = 1; S.iters = 0; S.trials = 0; S.chi2_check = 0; S.last_trial_chi = 0; S.stop = 0; S.refresh = 0;
    for (int i = 0; i < 6; ++i) S.xp[i] = 0;
  }
  {
    double Rwl[9], twl[3];
    for (int r = 0; r < 3; ++r) {
      double s = 0;
      for (int c = 0; c < 3; ++c) { Rwl[3 * r + c] = P.Tcw_last[4 * c + r]; s += (double)P.Tcw_last[4 * c + r] * (double)P.Tcw_last[4 * c + 3]; }
      twl[r] = (double)(float)(-s);
    }
    for (int j = tid; j < nloc; j += THREADS) {
      const int i = i0 + j;
      const double ox = pts[2 * i], oy = pts[2 * i + 1], z = dep[i];
      const double X[3] = {(ox - cx) * z / fx, (oy - cy) * z / fy, z};
      for (int r = 0; r < 3; ++r) PT(C_XW + r, j) = Rwl[3 * r] * X[0] + Rwl[3 * r + 1] * X[1] + Rwl[3 * r + 2] * X[2] + twl[r];
      PT(C_F, j) = flo[2 * i]; PT(C_F + 1, j) = flo[2 * i + 1];
      PT(C_DL, j) = 0; PT(C_DL + 1, j) = 0;
    }
  }
  __syncthreads();

  // robust chi2 at the current (T, f); writes err[]; also carries the trial's scale sum.  Totals: R.tot[0] = chi2, R.tot[1] = scale
  // (computeActiveErrors + activeRobustChi2)
  auto chi_pass = [&](double extra) {
    double acc[2] = {0.0, extra};
    for (int j = tid; j < nloc; j += THREADS) {
      const int i = i0 + j;
      const double xw = PT(C_XW, j), yw = PT(C_XW + 1, j), zw = PT(C_XW + 2, j);
      const double x = S.R[0] * xw + S.R[1] * yw + S.R[2] * zw + S.t[0];
      const double y = S.R[3] * xw + S.R[4] * yw + S.R[5] * zw + S.t[1];
      const double z = S.R[6] * xw + S.R[7] * yw + S.R[8] * zw + S.t[2];
      const double f0 = PT(C_F, j), f1 = PT(C_F + 1, j);
      const double ex = (double)pts[2 * i] + f0 - (x / z * fx + cx);
      const double ey = (double)pts[2 * i + 1] + f1 - (y / z * fy + cy);
      PT(C_ERR, j) = ex; PT(C_ERR + 1, j) = ey;
      double rho, hw;
      huber_f(w_rep * (ex * ex + ey * ey), delta, dsqr, rho, hw);
      const double px = f0 - (double)flo[2 * i], py = f1 - (double)flo[2 * i + 1];
      acc[0] += rho + w_prior * (px * px + py * py);
    }
    lm_reduce<2, false, CL>(acc, 0.0, R, phase);
  };
  auto jac = [&](int j, double* J) {      // 2x6 Jacobian of the linearisation point (types_six_dof_expmap.cpp:813-845)
    const double x = PT(C_XL, j), y = PT(C_XL + 1, j), z = PT(C_XL + 2, j), z2 = z * z;
    J[0] = x * y / z2 * fx; J[1] = -(1 + (x * x / z2)) * fx; J[2] = y / z * fx; J[3] = -1. / z * fx; J[4] = 0; J[5] = x / z2 * fx;
    J[6] = (1 + y * y / z2) * fy; J[7] = -x * y / z2 * fy; J[8] = -x / z * fy; J[9] = 0; J[10] = -1. / z * fy; J[11] = y / z2 * fy;
  };

  chi_pass(0.0);
  if (tid == 0) S.current = R.tot[0];
  __syncthreads();

  for (int it = 0; it < max_iters; ++it) {
    if (!S.ok) break;
    const double ini = S.current;
    // ---- buildSystem: J, w, h, bl per point; Hpp (21) + bp (6) + max h ----
    {
      double acc[27];
#pragma unroll
      for (int i = 0; i < 27; ++i) acc[i] = 0.0;
      double maxh = 0.0;
      for (int j = tid; j < nloc; j += THREADS) {
        const int i = i0 + j;
        const double xw = PT(C_XW, j), yw = PT(C_XW + 1, j), zw = PT(C_XW + 2, j);
        PT(C_XL, j) = S.R[0] * xw + S.R[1] * yw + S.R[2] * zw + S.t[0];
        PT(C_XL + 1, j) = S.R[3] * xw + S.R[4] * yw + S.R[5] * zw + S.t[1];
        PT(C_XL + 2, j) = S.R[6] * xw + S.R[7] * yw + S.R[8] * zw + S.t[2];
        double J[12]; jac(j, J);
        const double ex = PT(C_ERR, j), ey = PT(C_ERR + 1, j);
        double rho, hw;
        huber_f(w_rep * (ex * ex + ey * ey), delta, dsqr, rho, hw);
        const double w = w_rep * hw, h = w + w_prior;
        PT(C_W, j) = w; PT(C_H, j) = h;
        PT(C_BL, j) = -(w * ex + w_prior * (PT(C_F, j) - (double)flo[2 * i]));
        PT(C_BL + 1, j) = -(w * ey + w_prior * (PT(C_F + 1, j) - (double)flo[2 * i + 1]));
        int q = 0;
#pragma unroll
        for (int r = 0; r < 6; ++r) {
          acc[21 + r] -= w * (J[r] * ex + J[6 + r] * ey);
#pragma unroll
          for (int c = r; c < 6; ++c) acc[q++] += w * (J[r] * J[c] + J[6 + r] * J[6 + c]);
        }
        maxh = fmax(maxh, h);
      }
      lm_reduce<27, true, CL>(acc, maxh, R, phase);
      if (tid == 0) {
        int q = 0;
        for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) { S.Hpp[6 * a + b] = R.tot[q]; S.Hpp[6 * b + a] = R.tot[q]; ++q; }
        for (int a = 0; a < 6; ++a) S.bp[a] = R.tot[21 + a];
        if (it == 0) {
          double md = R.tot[27];
          for (int a = 0; a < 6; ++a) md = fmax(md, fabs(S.Hpp[7 * a]));
          S.lambda = 1e-5 * md; S.ni = 2; S.nbad = 0;
          if (tr) { trace_copy(tr + VDO_FLOW2_TRACE_HPP, S.Hpp, 36); trace_copy(tr + VDO_FLOW2_TRACE_BP, S.bp, 6); }
        }
        S.qmax = 0; S.stop_trials = 0;
      }
      __syncthreads();
    }
    // ---- lambda trials ----
    while (true) {
      const double lambda = S.lambda;
      // push + Schur complement accumulation
      double acc[42];
#pragma unroll
      for (int i = 0; i < 42; ++i) acc[i] = 0.0;
      for (int j = tid; j < nloc; j += THREADS) {
        PT(C_FBK, j) = PT(C_F, j); PT(C_FBK + 1, j) = PT(C_F + 1, j);
        const double w = PT(C_W, j), h = PT(C_H, j), pp = h + lambda;
        double J[12]; jac(j, J);
        double B0[6], B1[6];
#pragma unroll
        for (int r = 0; r < 6; ++r) { B0[r] = w * J[r]; B1[r] = w * J[6 + r]; }
        const double bl0 = PT(C_BL, j), bl1 = PT(C_BL + 1, j);
        if (!d.quirk) {
          const double ip = 1.0 / pp;
          const double d0 = bl0 * ip, d1 = bl1 * ip;
#pragma unroll
          for (int r = 0; r < 6; ++r) {
            acc[36 + r] += B0[r] * d0 + B1[r] * d1;
#pragma unroll
            for (int c = 0; c < 6; ++c) acc[6 * r + c] += (B0[r] * B0[c] + B1[r] * B1[c]) * ip;
          }
        } else {
          const double a = 1.0 / pp, b = -h / (pp * lambda), c2 = 1.0 / lambda;
          const double d0 = a * bl0 + b * bl1, d1 = c2 * bl1;
#pragma unroll
          for (int r = 0; r < 6; ++r) {
            acc[36 + r] += B0[r] * d0 + B1[r] * d1;
#pragma unroll
            for (int c = 0; c < 6; ++c) acc[6 * r + c] += a * B0[r] * B0[c] + b * B0[r] * B1[c] + c2 * B1[r] * B1[c];
          }
        }
      }
      lm_reduce<42, false, CL>(acc, 0.0, R, phase);
      if (tid == 0) {
        for (int k = 0; k < 36; ++k) S.Sm[k] = S.Hpp[k] - R.tot[k];
        for (int k = 0; k < 6; ++k) { S.Sm[7 * k] += lambda; S.g[k] = S.bp[k] - R.tot[36 + k]; }
        for (int k = 0; k < 4; ++k) S.qbk[k] = S.q[k];
        for (int k = 0; k < 3; ++k) S.tbk[k] = S.t[k];
        S.ok2 = solve6_lower(S.Sm, S.g, S.x, S.L, S.y) ? 1 : 0;
        if (S.ok2) for (int k = 0; k < 6; ++k) S.xp[k] = S.x[k];      // a failed solve leaves the previous x in place
        if (tr && S.trials == 0) { trace_copy(tr + VDO_FLOW2_TRACE_S, S.Sm, 36); trace_copy(tr + VDO_FLOW2_TRACE_G, S.g, 6); trace_copy(tr + VDO_FLOW2_TRACE_X, S.xp, 6); }
        se3_oplus(S.q, S.t, S.xp);
        quat_to_rot(S.q, S.R);
      }
      __syncthreads();
      // back substitution + update of the flows + computeScale
      double scale = 0.0;
      {
        const int ok2 = S.ok2;
        for (int j = tid; j < nloc; j += THREADS) {
          const int i = i0 + j;
          const double bl0 = PT(C_BL, j), bl1 = PT(C_BL + 1, j);
          if (ok2) {
            const double w = PT(C_W, j), h = PT(C_H, j), pp = h + lambda;
            double J[12]; jac(j, J);
            double cu = bl0, cv = bl1;
#pragma unroll
            for (int r = 0; r < 6; ++r) { cu -= w * J[r] * S.xp[r]; cv -= w * J[6 + r] * S.xp[r]; }
            if (!d.quirk) { PT(C_DL, j) = cu / pp; PT(C_DL + 1, j) = cv / pp; }
            else { PT(C_DL, j) = cu / pp - h * cv / (pp * lambda) + (i >= 1 ? cu / lambda : 0.0); PT(C_DL + 1, j) = cv / lambda; }
          }
          const double d0 = PT(C_DL, j), d1 = PT(C_DL + 1, j);
          PT(C_F, j) += d0; PT(C_F + 1, j) += d1;
          scale += d0 * (lambda * d0 + bl0) + d1 * (lambda * d1 + bl1);
        }
      }
      chi_pass(scale);
      if (tid == 0) {
        const double temp = R.tot[0];
        double sc_all = R.tot[1];
        for (int r = 0; r < 6; ++r) sc_all += S.xp[r] * (lambda * S.xp[r] + S.bp[r]);
        S.last_trial_chi = temp;
        const double cur0 = S.current;
        double tchi = S.ok2 ? temp : 1.7976931348623157e308;
        double rho = (S.current - tchi) / (sc_all + 1e-3);
        S.rho = rho;
        if (rho > 0 && isfinite(tchi)) {
          double alpha = 1. - pow(2 * rho - 1, 3.0);
          alpha = fmin(alpha, 2. / 3.);
          S.lambda *= fmax(1. / 3., alpha); S.ni = 2; S.current = tchi; S.accept = 1;
        } else {
          S.lambda *= S.ni; S.ni *= 2; S.accept = 0;
          for (int k = 0; k < 4; ++k) S.q[k] = S.qbk[k];
          for (int k = 0; k < 3; ++k) S.t[k] = S.tbk[k];
          quat_to_rot(S.q, S.R);
        }
        if (d.debug && crank == 0) printf("[flow2 dbg] it %d trial %d lambda %.6g ok2 %d temp %.9g current %.9g scale %.6g rho %.6g xp %.3g %.3g %.3g %.3g %.3g %.3g\n", it, S.qmax, lambda, S.ok2, temp, S.current, sc_all, rho, S.xp[0], S.xp[1], S.xp[2], S.xp[3], S.xp[4], S.xp[5]);
        if (tr) trace_trial(tr, S, it, lambda, temp, cur0, sc_all);
        S.qmax++; S.trials++;
        S.stop_trials = !(rho < 0 && S.qmax < 10);
      }
      __syncthreads();
      if (!S.accept)
        for (int j = tid; j < nloc; j += THREADS) { PT(C_F, j) = PT(C_FBK, j); PT(C_F + 1, j) = PT(C_FBK + 1, j); }
      __syncthreads();
      if (S.stop_trials) break;
    }
    if (tid == 0) end_iteration(S, it, ini);
    __syncthreads();
    if (S.refresh && S.ok) {
      chi_pass(0.0);
      if (tid == 0) { S.current = R.tot[0]; S.refresh = 0; }
      __syncthreads();
    }
  }
  // ---- classification (on _error as left by the last trial), outputs ----
  double nin[1] = {0};
  for (int j = tid; j < nloc; j += THREADS) {
    const int i = i0 + j;
    const float c = (float)(w_rep * (PT(C_ERR, j) * PT(C_ERR, j) + PT(C_ERR + 1, j) * PT(C_ERR + 1, j)));
    const unsigned char in = !(c > 0.04f);
    d.inlier[P.offset + i] = in; nin[0] += in;
    d.flow_out[2 * (size_t)(P.offset + i)] = PT(C_F, j); d.flow_out[2 * (size_t)(P.offset + i) + 1] = PT(C_F + 1, j);
  }
  lm_reduce<1, false, CL>(nin, 0.0, R, phase);
  if (tid == 0 && crank == 0) {
    float* To = d.T_out + 16 * out;
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) To[4 * r + c] = (float)S.R[3 * r + c]; To[4 * r + 3] = (float)S.t[r]; }
    To[12] = To[13] = To[14] = 0.f; To[15] = 1.f;
    double* st = d.stats + 8 * out;
    st[0] = S.iters; st[1] = S.trials; st[2] = S.current; st[3] = S.lambda; st[4] = R.tot[0];
    st[5] = 0; st[6] = 0; st[7] = 0;
    if (tr) trace_end(tr, S);
  }
  if constexpr (CL > 1) cooperative_groups::this_cluster().sync();   // no CTA may leave while another still reads its partial sums
#undef PT
}

__global__ void __cluster_dims__(FC_CL, 1, 1) __launch_bounds__(FC_THREADS) k_flow2_lm_cl(FlowDev d, int npc) {
  extern __shared__ __align__(16) double pt_sm[];        // FL_FIELDS x npc, field-major
  flow2_lm<FC_CL, FC_THREADS>(d, pt_sm, npc);
}
__global__ void __launch_bounds__(FL_THREADS) k_flow2_lm(FlowDev d) {
  const FlowProb& P = d.prob[blockIdx.x];               // FL_FIELDS x n, field-major, in the problem's share of the scratch
  flow2_lm<1, FL_THREADS>(d, d.scratch + (size_t)P.offset * FL_FIELDS, P.n);
}

// ---- host side: a persistent device arena per context stream ----
// Each problem runs on the kernel its own size selects, so its result does not depend on the other problems of its batch:
// n <= FC_MAX_N on the cluster kernel (its points fit the shared memory of FC_CL CTAs), the rest on the single-CTA kernel.
constexpr size_t FC_SMEM_MAX = 200 * 1024;
constexpr int FC_MAX_N = VDO_FLOW2_CLUSTER_MAX_N;
static_assert((size_t)FL_FIELDS * ((FC_MAX_N + FC_CL - 1) / FC_CL) * sizeof(double) <= FC_SMEM_MAX &&
              (size_t)FL_FIELDS * ((FC_MAX_N + FC_CL) / FC_CL) * sizeof(double) > FC_SMEM_MAX,
              "VDO_FLOW2_CLUSTER_MAX_N must be the largest problem whose points fit the cluster's shared memory");

struct FlowArena {
  size_t cap_pts = 0, cap_prob = 0, cap_trace = 0;
  float *pts = 0, *depth = 0, *flow = 0, *T_out = 0;
  double *scratch = 0, *flow_out = 0, *stats = 0, *trace = 0;
  unsigned char* inlier = 0;
  FlowProb* prob = 0;         // the cluster kernel's problems first, then the single-CTA kernel's
  FlowProb* h_prob = 0;       // pinned
  float* h_T = 0; double* h_stats = 0;
  int launches = 0;
  int last_nprob = 0, last_ncl = 0, last_npc = 0;   // the split of the last batch (replayed by vdo_pose_opt_flow2_time)
};
std::mutex g_mu;
std::map<uint64_t, FlowArena> g_arenas;

static bool force_single_cta() {
  static const bool v = std::getenv("VDO_FLOW_SINGLE_CTA") != nullptr;   // read once per process
  return v;
}
// ncl problems (d.prob[0, ncl)) on the cluster kernel with npc points per CTA, then nsingle (d.prob[ncl, ncl + nsingle)) on k_flow2_lm
static void flow_launch(const FlowDev& d, int ncl, int npc, int nsingle, cudaStream_t st) {
  if (ncl > 0) {
    static bool opted = false;
    if (!opted) { cudaFuncSetAttribute(k_flow2_lm_cl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FC_SMEM_MAX); opted = true; }
    k_flow2_lm_cl<<<ncl * FC_CL, FC_THREADS, (size_t)FL_FIELDS * npc * sizeof(double), st>>>(d, npc);
  }
  if (nsingle > 0) {
    FlowDev ds = d;
    ds.prob = d.prob + ncl;
    k_flow2_lm<<<nsingle, FL_THREADS, 0, st>>>(ds);
  }
}

// ---- vdo_pose_refine_batch_dev: the problems are gathered from ORB matches on the device ----
constexpr int RG_THREADS = 256;

// the correspondences of vdo_pnp_match_batch_dev that the caller's mask keeps (mask: the pair's row, or NULL)
struct PredRefine {
  PredCorr c; const uint8_t* mask;
  __device__ __forceinline__ bool operator()(int i) const { return (!mask || mask[i]) && c(i); }
};

// one CTA per pair: ordered compaction of the problem's points into the pair's segment (offset p * seg, local -> query index map in
// lmap), their pixel, depth and flow estimate, and the pair's FlowProb (K and Tcw_last from the by-value argument, T_init from the device)
__global__ void __launch_bounds__(RG_THREADS) k_refine_gather(const __grid_constant__ PnpGatherArg a, const uint8_t* __restrict__ mask,
                                                              const float* __restrict__ T_init, FlowProb* __restrict__ prob, float* __restrict__ pts,
                                                              float* __restrict__ depth, float* __restrict__ flow, int* __restrict__ lmap,
                                                              int* __restrict__ nq_out, int* __restrict__ status) {
  const int p = blockIdx.x, tid = threadIdx.x;
  __shared__ int s_scan[RG_THREADS];
  __shared__ int s_base;
  const PnpPairArg& pa = a.pr[p];
  const int cq = a.qcount[pa.q], ct = a.tcount[pa.t];
  const int nq = valid_count(cq, a.qcap), nt = valid_count(ct, a.tcap);
  const size_t off = (size_t)p * a.seg;
  const PredRefine pc{{&a, &pa, a.qx + (size_t)pa.q * a.qcap, a.qy + (size_t)pa.q * a.qcap, a.idx + (size_t)p * a.qcap * a.k,
                       a.dist + (size_t)p * a.qcap * a.k, nt},
                      mask ? mask + (size_t)p * a.qcap : nullptr};
  const int n = compact_ordered<RG_THREADS>(nq, pc, lmap + off, s_scan, &s_base);
  const float* tx = a.tx + (size_t)pa.t * a.tcap; const float* ty = a.ty + (size_t)pa.t * a.tcap;
  for (int r = tid; r < n; r += RG_THREADS) {
    const int i = lmap[off + r], j = pc.c.idx[(size_t)i * a.k];
    float z;
    pc.c.depth_at(i, &z);
    const float u = pc.c.qx[i], v = pc.c.qy[i];
    pts[2 * (off + r)] = u; pts[2 * (off + r) + 1] = v;
    depth[off + r] = z;
    flow[2 * (off + r)] = tx[j] - u; flow[2 * (off + r) + 1] = ty[j] - v;
  }
  if (tid == 0) {
    FlowProb pb;
    pb.mode = 0; pb.n = n; pb.offset = (int)off; pb.out = p;
    for (int c = 0; c < 4; ++c) pb.K[c] = pa.Kq[c];
    for (int c = 0; c < 16; ++c) pb.Tcw_last[c] = c < 12 && pa.has_T ? pa.T[c] : (c % 5 == 0 ? 1.f : 0.f);
    for (int c = 0; c < 16; ++c) pb.T_init[c] = T_init[16 * p + c];
    prob[p] = pb;
    nq_out[p] = nq;
    status[p] = (cq == nq ? 0 : VDO_PNP_STATUS_QUERY_COUNT) | (ct == nt ? 0 : VDO_PNP_STATUS_TRAIN_COUNT);
  }
}

// The host does not know n, so both shapes are launched over all P problems and each returns at once for a problem of the other shape
// (the rule of vdo_pose_opt_flow2_batch: n <= FC_MAX_N on the cluster).  All CTAs of a cluster read the same n and leave together.
// npc only strides the shared-memory fields: a problem's CTA still owns ceil(n / FC_CL) points, so its sums are those of k_flow2_lm_cl.
__global__ void __cluster_dims__(FC_CL, 1, 1) __launch_bounds__(FC_THREADS) k_refine_lm_cl(FlowDev d, int npc) {
  extern __shared__ __align__(16) double pt_sm[];        // FL_FIELDS x npc, field-major
  if (d.prob[blockIdx.x / FC_CL].n > FC_MAX_N) return;
  flow2_lm<FC_CL, FC_THREADS>(d, pt_sm, npc);
}
__global__ void __launch_bounds__(FL_THREADS) k_refine_lm(FlowDev d) {
  const FlowProb& P = d.prob[blockIdx.x];
  if (P.n <= FC_MAX_N) return;
  flow2_lm<1, FL_THREADS>(d, d.scratch + (size_t)P.offset * FL_FIELDS, P.n);
}

// one CTA per pair: the problem's flows and inlier flags -> the query keypoints' slots (the flags of i < count[q] zeroed first)
__global__ void __launch_bounds__(RG_THREADS) k_refine_scatter(const FlowProb* __restrict__ prob, const int* __restrict__ lmap, const double* __restrict__ flow_res,
                                                               const unsigned char* __restrict__ inl_res, const int* __restrict__ nq_in,
                                                               const int* __restrict__ status, int qcap, vdo_pose_refine_out o) {
  const int p = blockIdx.x, tid = threadIdx.x;
  const int n = prob[p].n;
  const size_t off = (size_t)prob[p].offset;
  uint8_t* row = o.inlier_dev + (size_t)p * qcap;
  double* frow = o.flow_dev + 2 * (size_t)p * qcap;
  for (int i = tid; i < nq_in[p]; i += RG_THREADS) row[i] = 0;
  __syncthreads();
  for (int r = tid; r < n; r += RG_THREADS) {
    const int i = lmap[off + r];
    row[i] = inl_res[off + r];
    frow[2 * i] = flow_res[2 * (off + r)]; frow[2 * i + 1] = flow_res[2 * (off + r) + 1];
  }
  if (tid == 0) { o.n_points_dev[p] = n; o.status_dev[p] = status[p]; }
}

}  // namespace

extern "C" int vdo_pose_opt_flow2_trace(vdo_ctx* ctx, int quirk, int nprob, const int* mode, const int* offset, const float* pts,
                                        const float* depth, const float* flow, const float* K, const float* Tcw_last, const float* T_init,
                                        float* T_out, double* flow_out, unsigned char* inlier, double* stats, double* trace) {
  if (!ctx) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& m) { vdo::ctx_set_error(ctx, "vdo_pose_opt_flow2_batch: " + m); return VDO_ERR_ARG; };
  if (nprob <= 0 || !mode || !offset) return refuse("nprob < 1 or a NULL mode / offset array");
  if (!K || !Tcw_last || !T_init || !T_out) return refuse("a NULL per-problem array (K, Tcw_last, T_init, T_out)");
  if (offset[0] != 0) return refuse("offset[0] is " + std::to_string(offset[0]) + ", not 0");
  for (int p = 0; p < nprob; ++p) {
    if (offset[p + 1] < offset[p]) return refuse("offset[" + std::to_string(p + 1) + "] < offset[" + std::to_string(p) + "]");
    if (mode[p] != 0 && mode[p] != 1) return refuse("mode[" + std::to_string(p) + "] is " + std::to_string(mode[p]) + ", not 0 or 1");
  }
  const size_t total = (size_t)offset[nprob];
  if (total > 0 && (!pts || !depth || !flow || !flow_out || !inlier)) return refuse("a NULL point array (pts, depth, flow, flow_out, inlier)");
  cudaStream_t st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx);
  std::lock_guard<std::mutex> lk(g_mu);
  FlowArena& A = g_arenas[(uint64_t)(uintptr_t)st];
  if (total > A.cap_pts) {
    size_t cap = total * 2 + 1024;
    cudaFree(A.pts); cudaFree(A.depth); cudaFree(A.flow); cudaFree(A.scratch); cudaFree(A.flow_out); cudaFree(A.inlier);
    VDO_CUDA(cudaMalloc(&A.pts, cap * 8)); VDO_CUDA(cudaMalloc(&A.depth, cap * 4)); VDO_CUDA(cudaMalloc(&A.flow, cap * 8));
    VDO_CUDA(cudaMalloc(&A.scratch, cap * FL_FIELDS * 8)); VDO_CUDA(cudaMalloc(&A.flow_out, cap * 16)); VDO_CUDA(cudaMalloc(&A.inlier, cap));
    A.cap_pts = cap;
  }
  if ((size_t)nprob > A.cap_prob) {
    size_t cap = (size_t)nprob * 2 + 8;
    cudaFree(A.prob); cudaFree(A.T_out); cudaFree(A.stats); cudaFreeHost(A.h_prob); cudaFreeHost(A.h_T); cudaFreeHost(A.h_stats);
    VDO_CUDA(cudaMalloc(&A.prob, cap * sizeof(FlowProb))); VDO_CUDA(cudaMalloc(&A.T_out, cap * 64)); VDO_CUDA(cudaMalloc(&A.stats, cap * 64));
    VDO_CUDA(cudaMallocHost(&A.h_prob, cap * sizeof(FlowProb))); VDO_CUDA(cudaMallocHost(&A.h_T, cap * 64)); VDO_CUDA(cudaMallocHost(&A.h_stats, cap * 64));
    A.cap_prob = cap;
  }
  const size_t trace_doubles = (size_t)nprob * VDO_FLOW2_TRACE_DOUBLES;
  if (trace && trace_doubles > A.cap_trace) {
    cudaFree(A.trace);
    A.trace = 0; A.cap_trace = 0;
    VDO_CUDA(cudaMalloc(&A.trace, trace_doubles * 8));
    A.cap_trace = trace_doubles;
  }
  // the cluster kernel's problems first, then the single-CTA kernel's, each in batch order
  const bool single_only = force_single_cta();
  int ncl = 0, max_cl = 0;
  for (int pass = 0; pass < 2; ++pass)
    for (int p = 0, k = pass ? ncl : 0; p < nprob; ++p) {
      const int n = offset[p + 1] - offset[p];
      const bool cl = !single_only && n <= FC_MAX_N;
      if (cl != (pass == 0)) continue;
      FlowProb& q = A.h_prob[k++];
      q.mode = mode[p]; q.n = n; q.offset = offset[p]; q.out = p;
      std::memcpy(q.K, K + 4 * p, 16); std::memcpy(q.Tcw_last, Tcw_last + 16 * p, 64); std::memcpy(q.T_init, T_init + 16 * p, 64);
      if (pass == 0) { ++ncl; max_cl = std::max(max_cl, n); }
    }
  const int npc = std::max(1, (max_cl + FC_CL - 1) / FC_CL);
  VDO_CUDA(cudaMemcpyAsync(A.prob, A.h_prob, nprob * sizeof(FlowProb), cudaMemcpyHostToDevice, st));
  if (total) {
    VDO_CUDA(cudaMemcpyAsync(A.pts, pts, total * 8, cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(A.depth, depth, total * 4, cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(A.flow, flow, total * 8, cudaMemcpyHostToDevice, st));
  }
  if (trace) VDO_CUDA(cudaMemsetAsync(A.trace, 0, trace_doubles * 8, st));
  FlowDev d{A.prob, A.pts, A.depth, A.flow, A.scratch, A.T_out, A.flow_out, A.inlier, A.stats, quirk & 1, (quirk >> 1) & 1, trace ? A.trace : nullptr};
  A.last_nprob = nprob; A.last_ncl = ncl; A.last_npc = npc;
  flow_launch(d, ncl, npc, nprob - ncl, st);
  A.launches++;
  VDO_CUDA(cudaGetLastError());
  VDO_CUDA(cudaMemcpyAsync(A.h_T, A.T_out, (size_t)nprob * 64, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaMemcpyAsync(A.h_stats, A.stats, (size_t)nprob * 64, cudaMemcpyDeviceToHost, st));
  if (total) {
    VDO_CUDA(cudaMemcpyAsync(flow_out, A.flow_out, total * 16, cudaMemcpyDeviceToHost, st));
    VDO_CUDA(cudaMemcpyAsync(inlier, A.inlier, total, cudaMemcpyDeviceToHost, st));
  }
  if (trace) VDO_CUDA(cudaMemcpyAsync(trace, A.trace, trace_doubles * 8, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  std::memcpy(T_out, A.h_T, (size_t)nprob * 64);
  if (stats) std::memcpy(stats, A.h_stats, (size_t)nprob * 64);
  return VDO_OK;
}

extern "C" int vdo_pose_opt_flow2_batch(vdo_ctx* ctx, int quirk, int nprob, const int* mode, const int* offset, const float* pts,
                                        const float* depth, const float* flow, const float* K, const float* Tcw_last, const float* T_init,
                                        float* T_out, double* flow_out, unsigned char* inlier, double* stats) {
  return vdo_pose_opt_flow2_trace(ctx, quirk, nprob, mode, offset, pts, depth, flow, K, Tcw_last, T_init, T_out, flow_out, inlier, stats, nullptr);
}

extern "C" int vdo_pose_opt_flow2(vdo_ctx* ctx, int mode, int quirk, int n, const float* pts, const float* depth, const float* flow,
                                  const float* K, const float* Tcw_last, const float* T_init, float* T_out, double* flow_out,
                                  unsigned char* inlier, double* stats) {
  int off[2] = {0, n};
  return vdo_pose_opt_flow2_batch(ctx, quirk, 1, &mode, off, pts, depth, flow, K, Tcw_last, T_init, T_out, flow_out, inlier, stats);
}

// device-resident timing hook for bench.py: re-runs the last batch `reps` times without host copies, with that batch's kernel split
extern "C" int vdo_pose_opt_flow2_time(vdo_ctx* ctx, int quirk, int nprob, int reps, float* ms_avg) {
  if (!ctx || nprob <= 0 || reps <= 0 || !ms_avg) return VDO_ERR_ARG;
  cudaStream_t st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx);
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_arenas.find((uint64_t)(uintptr_t)st);
  if (it == g_arenas.end() || nprob != it->second.last_nprob) return VDO_ERR_STATE;
  FlowArena& A = it->second;
  FlowDev d{A.prob, A.pts, A.depth, A.flow, A.scratch, A.T_out, A.flow_out, A.inlier, A.stats, quirk & 1, (quirk >> 1) & 1, nullptr};
  cudaEvent_t e0, e1;
  VDO_CUDA(cudaEventCreate(&e0)); VDO_CUDA(cudaEventCreate(&e1));
  flow_launch(d, A.last_ncl, A.last_npc, nprob - A.last_ncl, st);
  VDO_CUDA(cudaEventRecord(e0, st));
  for (int i = 0; i < reps; ++i) flow_launch(d, A.last_ncl, A.last_npc, nprob - A.last_ncl, st);
  VDO_CUDA(cudaEventRecord(e1, st));
  VDO_CUDA(cudaEventSynchronize(e1));
  float ms = 0; VDO_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  *ms_avg = ms / reps;
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return VDO_OK;
}

// ---- launchers for problems resident on the device (dev_solvers.cuh) ----
int vdo::flow_lm_fields() { return FL_FIELDS; }
cudaError_t vdo::flow_lm_prepare() { return cudaFuncSetAttribute(k_refine_lm_cl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FC_SMEM_MAX); }
void vdo::flow_lm_launch(const FlowDev& d, int nprob, int max_n, cudaStream_t st) {
  const int npc = (std::min(max_n, FC_MAX_N) + FC_CL - 1) / FC_CL;
  k_refine_lm_cl<<<nprob * FC_CL, FC_THREADS, (size_t)FL_FIELDS * npc * sizeof(double), st>>>(d, npc);
  if (max_n > FC_MAX_N) k_refine_lm<<<nprob, FL_THREADS, 0, st>>>(d);
}

// ---- vdo_pose_refiner: the work space of vdo_pose_refine_batch_dev, all allocated at creation ----
struct vdo_pose_refiner : vdo::WorkSpace {
  vdo_ctx* ctx = nullptr;
  int dev = 0, max_pairs = 0, cap = 0;
  FlowProb* prob = nullptr;                                            // max_pairs
  float *pts = nullptr, *depth = nullptr, *flow = nullptr;             // max_pairs x cap segments
  int* lmap = nullptr;
  double *flow_out = nullptr, *scratch = nullptr;                      // scratch: max_pairs x cap x FL_FIELDS, only when cap > FC_MAX_N
  unsigned char* inlier = nullptr;
  int *nq = nullptr, *status = nullptr;                                // max_pairs
};

extern "C" int vdo_pose_refiner_create(vdo_ctx* ctx, int max_pairs, int cap, vdo_pose_refiner** out) {
  if (!ctx || !out) return VDO_ERR_ARG;
  *out = nullptr;
  if (max_pairs < 1 || max_pairs > PNP_MAX_PAIRS || cap < 1 || (int64_t)max_pairs * cap > INT_MAX) {
    vdo::ctx_set_error(ctx, "vdo_pose_refiner_create: max_pairs = " + std::to_string(max_pairs) + ", cap = " + std::to_string(cap) +
                                "; expected 1 .. 64 and >= 1, with max_pairs x cap below 2^31");
    return VDO_ERR_ARG;
  }
  vdo_pose_refiner* r = new vdo_pose_refiner;
  r->ctx = ctx; r->max_pairs = max_pairs; r->cap = cap;
  int n_sm = 0;
  vdo::ctx_device(ctx, &r->dev, &n_sm);
  const size_t pts = (size_t)max_pairs * cap;
  return vdo::create_done(ctx, "vdo_pose_refiner_create", r,
                          {r->alloc(r->prob, (size_t)max_pairs), r->alloc(r->pts, 2 * pts), r->alloc(r->depth, pts), r->alloc(r->flow, 2 * pts),
                           r->alloc(r->lmap, pts), r->alloc(r->flow_out, 2 * pts), r->alloc(r->inlier, pts), r->alloc(r->nq, (size_t)max_pairs),
                           r->alloc(r->status, (size_t)max_pairs), cap > FC_MAX_N ? r->alloc(r->scratch, pts * FL_FIELDS) : cudaSuccess,
                           vdo::flow_lm_prepare()},
                          out);
}
extern "C" void vdo_pose_refiner_destroy(vdo_pose_refiner* r) { delete r; }
extern "C" int vdo_pose_refiner_info(const vdo_pose_refiner* r, int64_t out[4]) {
  if (!r || !out) return VDO_ERR_ARG;
  out[0] = r->max_pairs; out[1] = r->cap; out[2] = (int64_t)r->bytes; out[3] = 0;
  return VDO_OK;
}

extern "C" int vdo_pose_refine_batch_dev(vdo_pose_refiner* r, int P, const int32_t* pairs, const vdo_orb_desc_set* query, const vdo_orb_desc_set* train,
                                         const int32_t* idx_dev, const int32_t* dist_dev, const vdo_dev_plane* depth, const int32_t* depth_wh,
                                         const float* K, const float* Tcw_query, const float* T_init_dev, const uint8_t* mask_dev,
                                         const vdo_pose_refine_opts* opts, const vdo_pose_refine_out* out, uint64_t stream) {
  if (!r) return VDO_ERR_ARG;
  auto check_rest = [&](vdo::DevPtrs& ptrs) -> std::string {
    if (opts->quirk != 0 && opts->quirk != 1) return "quirk = " + std::to_string(opts->quirk) + "; expected 0 or 1";
    ptrs = {{T_init_dev, 4, "T_init_dev"}, {out->T_dev, 4, "out.T_dev"}, {out->flow_dev, 8, "out.flow_dev"}, {out->inlier_dev, 1, "out.inlier_dev"},
            {out->n_points_dev, 4, "out.n_points_dev"}, {out->stats_dev, 8, "out.stats_dev"}, {out->status_dev, 4, "out.status_dev"},
            {mask_dev, 1, "mask_dev", mask_dev != nullptr}};
    return "";
  };
  PnpGatherArg ga;
  if (std::string why = corr_check("refiner", r->max_pairs, r->cap, r->dev, P, pairs, query, train, idx_dev, dist_dev, depth, depth_wh, "K", K, nullptr,
                                   Tcw_query, opts, out, [] { return std::string(); }, check_rest, ga);
      !why.empty()) {
    vdo::ctx_set_error(r->ctx, "vdo_pose_refine_batch_dev: " + why);
    return VDO_ERR_ARG;
  }
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  // T_out and stats are the caller's outputs (problem p writes row p); flows and flags go through the pair's segment to the scatter
  const FlowDev d{r->prob, r->pts, r->depth, r->flow, r->scratch, out->T_dev, r->flow_out, r->inlier, out->stats_dev, opts->quirk, 0, nullptr};
  k_refine_gather<<<P, RG_THREADS, 0, st>>>(ga, mask_dev, T_init_dev, r->prob, r->pts, r->depth, r->flow, r->lmap, r->nq, r->status);
  vdo::flow_lm_launch(d, P, query->cap, st);
  k_refine_scatter<<<P, RG_THREADS, 0, st>>>(r->prob, r->lmap, r->flow_out, r->inlier, r->nq, r->status, query->cap, *out);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
