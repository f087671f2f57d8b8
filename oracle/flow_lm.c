/*
 * oracle/flow_lm.c -- TEST INFRASTRUCTURE ONLY (CPU oracle + timed CPU baseline; never on the product path).
 *
 * CPU restatement of the reference's per-frame joint flow / SE(3) refinement:
 *   Optimizer::PoseOptimizationFlow2     src/Optimizer.cc:2755-2972   (object motion; prior 0.5*I, optimize(200))
 *   Optimizer::PoseOptimizationFlow2Cam  src/Optimizer.cc:2333-2542   (camera pose;  prior 0.3*I, optimize(100))
 *   EdgeSE3ProjectFlow2 / EdgeFlowPrior  g2o/types/types_six_dof_expmap.h:414-476, .cpp:772-775, 805-845
 *   VertexSE3Expmap / SE3Quat::exp       g2o/types/types_six_dof_expmap.h:67-85, se3quat.h:58-60, 105-122, 228-301
 *   Converter::toSE3Quat / toCvMat       src/Converter.cc:25-41
 *   LM / outer loop                      g2o/core/optimization_algorithm_levenberg.cpp:61-164, sparse_optimizer.cpp:354-427
 *   Schur solve + dense LDLT             g2o/core/block_solver.hpp:352-486, g2o/solvers/linear_solver_dense.h:65-113
 *
 * Two arithmetic modes (SURVEY.md section 7.2, H1):
 *   quirk = 1  REF_QUIRK: the 2-D flow vertices live in BlockSolver_6_3's 3x3 landmark blocks.  In a Release build the
 *              2x2 Hessian [h 0; 0 h] is mapped onto the first four doubles of the zeroed 3x3 block, lambda is added to the
 *              3x3 diagonal, the 3x3 inverse and 3-vector strides are used => D^-1 = [[1/p, -h/(p lam), 0],[0,1/lam,0],[0,0,1/lam]]
 *              (p = h + lam), a non-symmetric Schur update of which LDLT reads the lower triangle, and a spill of
 *              c_u(i+1)/lam into the u-increment of landmark i+1.  This is derived from reading the source only -- the
 *              reference binary cannot be built here -- and is flagged as such everywhere.
 *   quirk = 0  CLEAN: the intended 2x2 arithmetic, D^-1 = 1/(h + lam) * I2.
 *
 * Parity status: UNPINNED (no reference tests / golden vectors exist; OpenCV's float gemm used for Twl and Eigen's LDLT
 * pivoting are outside the tree and restated from their documented behaviour).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "se3_math.h"
#include "../include/vdo_b200.h"   /* VDO_FLOW2_TRACE_* / VDO_FLOW2_STOP_*: the trace layout the GPU entry writes */

typedef struct { double q[4]; double t[3]; } se3q;   /* q = {x,y,z,w} */

static void se3q_normalize(se3q *T) {               /* SE3Quat::normalizeRotation */
  if (T->q[3] < 0) { T->q[0] = -T->q[0]; T->q[1] = -T->q[1]; T->q[2] = -T->q[2]; T->q[3] = -T->q[3]; }
  quat_normalize(T->q);
}
static void se3q_from_f32(const float *M, se3q *T) { /* Converter::toSE3Quat: SE3Quat(R, t) */
  double R[9] = {M[0], M[1], M[2], M[4], M[5], M[6], M[8], M[9], M[10]};
  quat_from_m3(R, T->q);
  T->t[0] = M[3]; T->t[1] = M[7]; T->t[2] = M[11];
  se3q_normalize(T);
}
static void quat_mul(const double *a, const double *b, double *o) { /* Eigen quaternion product, {x,y,z,w} */
  double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
/* SE3Quat::exp(update) * estimate  (VertexSE3Expmap::oplusImpl) */
static void se3q_oplus(se3q *T, const double *u) {
  double om[3] = {u[0], u[1], u[2]}, up[3] = {u[3], u[4], u[5]};
  double th = sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
  double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0}, O2[9], R[9], V[9];
  m3_mul(O, O, O2);
  if (th < 0.00001) {
    for (int i = 0; i < 9; ++i) R[i] = O[i] + O2[i];
    R[0] += 1; R[4] += 1; R[8] += 1;
    memcpy(V, R, sizeof R);
  } else {
    double a = sin(th) / th, b = (1 - cos(th)) / (th * th), c = (th - sin(th)) / pow(th, 3);
    for (int i = 0; i < 9; ++i) { R[i] = a * O[i] + b * O2[i]; V[i] = b * O[i] + c * O2[i]; }
    R[0] += 1; R[4] += 1; R[8] += 1; V[0] += 1; V[4] += 1; V[8] += 1;
  }
  se3q inc;
  quat_from_m3(R, inc.q);
  m3_vec(V, up, inc.t);
  se3q_normalize(&inc);
  /* operator*: t = t_inc + r_inc * t_est ; r = r_inc * r_est ; normalize */
  double Ri[9], rt[3], qn[4];
  quat_to_m3(inc.q, Ri);
  m3_vec(Ri, T->t, rt);
  quat_mul(inc.q, T->q, qn);
  T->t[0] = inc.t[0] + rt[0]; T->t[1] = inc.t[1] + rt[1]; T->t[2] = inc.t[2] + rt[2];
  memcpy(T->q, qn, sizeof qn);
  se3q_normalize(T);
}

typedef struct {
  int n, quirk;
  double fx, fy, cx, cy, w_rep, w_prior, delta;
  const double *Xw, *obs, *fhat;     /* n x 3, n x 2, n x 2 */
  double *f;                          /* n x 2 current flows */
  se3q T;
  double *err;                        /* n x 2: _error of the reprojection edges as left by the last computeActiveErrors */
} flow_t;

static void huber_f(double e2, double delta, double *rho, double *w) {
  double dsqr = (double)(float)(delta * delta);
  if (e2 <= dsqr) { *rho = e2; *w = 1.0; }
  else { double s = sqrt(e2); *rho = 2 * s * delta - dsqr; *w = delta / s; }
}
/* computeActiveErrors + activeRobustChi2 */
static double flow_chi2(flow_t *g) {
  double R[9], chi = 0;
  quat_to_m3(g->T.q, R);
  for (int i = 0; i < g->n; ++i) {
    double X[3];
    m3_vec(R, g->Xw + 3 * i, X);
    X[0] += g->T.t[0]; X[1] += g->T.t[1]; X[2] += g->T.t[2];
    double ex = g->obs[2 * i] + g->f[2 * i] - (X[0] / X[2] * g->fx + g->cx);
    double ey = g->obs[2 * i + 1] + g->f[2 * i + 1] - (X[1] / X[2] * g->fy + g->cy);
    g->err[2 * i] = ex; g->err[2 * i + 1] = ey;
    double rho, w;
    huber_f(g->w_rep * (ex * ex + ey * ey), g->delta, &rho, &w);
    chi += rho;
    double px = g->f[2 * i] - g->fhat[2 * i], py = g->f[2 * i + 1] - g->fhat[2 * i + 1];
    chi += g->w_prior * (px * px + py * py);
  }
  return chi;
}

/* LDLT-equivalent solve of the symmetric matrix given by the LOWER triangle of S (6x6 row-major). Returns 0 if not positive. */
static int solve6_lower(const double *S, const double *g, double *x) {
  double L[36] = {0}, y[6];
  for (int j = 0; j < 6; ++j) {
    double d = S[7 * j];
    for (int k = 0; k < j; ++k) d -= L[6 * j + k] * L[6 * j + k];
    if (!(d > 0)) return 0;
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
  return 1;
}

/*
 * mode: 0 = camera (Flow2Cam: prior information 0.3, optimize(100)), 1 = object (Flow2: 0.5, optimize(200)).
 * pts n x 2 (last-frame pixels), depth n, flow n x 2 (measured flow), K = {fx,fy,cx,cy}, Tcw_last / T_init 4x4 row-major f32.
 * Outputs: T_out 4x4 f32, flow_out n x 2 (refined flow of every point), inlier n (1 = chi2 <= 0.04 at the state g2o's
 * _error arrays were left in), stats = {iterations, trials, final chi2, final lambda, n_inliers}.
 * Returns the number of LM iterations, or -1 when n < 3 (the reference then returns identity / 0 without optimising).
 * trace (VDO_FLOW2_TRACE_DOUBLES, or NULL): the LM trace in the layout of vdo_pose_opt_flow2_trace (include/vdo_b200.h).
 */
static int flow2_run(int mode, int quirk, int n, const float *pts, const float *depth, const float *flow, const float *K,
                     const float *Tcw_last, const float *T_init, float *T_out, double *flow_out, uint8_t *inlier, double *stats,
                     double *trace) {
  if (trace) memset(trace, 0, sizeof(double) * VDO_FLOW2_TRACE_DOUBLES);
  if (n < 3) {
    if (trace) trace[VDO_FLOW2_TRACE_STOP] = VDO_FLOW2_STOP_FEW_POINTS;
    return -1;
  }
  flow_t G; memset(&G, 0, sizeof G);
  flow_t *g = &G;
  g->n = n; g->quirk = quirk;
  g->fx = K[0]; g->fy = K[1]; g->cx = K[2]; g->cy = K[3];
  g->w_rep = 0.1; g->w_prior = mode ? 0.5 : 0.3;
  { float rp = 0.04f; float dm = (float)sqrt((double)rp); g->delta = dm; }
  const int max_iters = mode ? 200 : 100;
  /* Twl = inverse of the last frame's Tcw, formed in float like the cv::Mat expressions (double accumulation, float result) */
  double Rwl[9], twl[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) Rwl[3 * r + c] = Tcw_last[4 * c + r];
    double s = 0;
    for (int j = 0; j < 3; ++j) s += (double)Tcw_last[4 * j + r] * (double)Tcw_last[4 * j + 3];
    twl[r] = (double)(float)(-s);
  }
  double *Xw = (double *)malloc(sizeof(double) * 3 * n), *obs = (double *)malloc(sizeof(double) * 2 * n);
  double *fhat = (double *)malloc(sizeof(double) * 2 * n), *f = (double *)malloc(sizeof(double) * 2 * n);
  double *fbk = (double *)malloc(sizeof(double) * 2 * n), *err = (double *)malloc(sizeof(double) * 2 * n);
  double *hl = (double *)malloc(sizeof(double) * n), *bl = (double *)malloc(sizeof(double) * 2 * n), *J = (double *)malloc(sizeof(double) * 12 * n);
  double *wl = (double *)malloc(sizeof(double) * n), *dl = (double *)malloc(sizeof(double) * 2 * n);
  for (int i = 0; i < n; ++i) {
    double ox = pts[2 * i], oy = pts[2 * i + 1], d = depth[i];
    double Xc[3] = {(ox - g->cx) * d / g->fx, (oy - g->cy) * d / g->fy, d}, X[3];
    m3_vec(Rwl, Xc, X);
    Xw[3 * i] = X[0] + twl[0]; Xw[3 * i + 1] = X[1] + twl[1]; Xw[3 * i + 2] = X[2] + twl[2];
    obs[2 * i] = ox; obs[2 * i + 1] = oy;
    fhat[2 * i] = flow[2 * i]; fhat[2 * i + 1] = flow[2 * i + 1];
    f[2 * i] = fhat[2 * i]; f[2 * i + 1] = fhat[2 * i + 1];
  }
  g->Xw = Xw; g->obs = obs; g->fhat = fhat; g->f = f; g->err = err;
  se3q_from_f32(T_init, &g->T);

  double lambda = -1, ni = 2; int nbad = 0, trials = 0, iters = 0, ok = 1, stop = 0;
  double xp[6] = {0, 0, 0, 0, 0, 0};
  memset(dl, 0, sizeof(double) * 2 * n);
  double chi2_check = 0, last_trial_chi = 0;
  for (int it = 0; it < max_iters && ok; ++it) {
    double current = flow_chi2(g), temp = current, ini = current;
    /* buildSystem */
    double Hpp[36] = {0}, bp[6] = {0}, R[9], maxd = 0;
    quat_to_m3(g->T.q, R);
    for (int i = 0; i < n; ++i) {
      double X[3];
      m3_vec(R, Xw + 3 * i, X);
      double x = X[0] + g->T.t[0], y = X[1] + g->T.t[1], z = X[2] + g->T.t[2], z2 = z * z;
      double *Ji = J + 12 * i;
      Ji[0] = x * y / z2 * g->fx; Ji[1] = -(1 + (x * x / z2)) * g->fx; Ji[2] = y / z * g->fx; Ji[3] = -1. / z * g->fx; Ji[4] = 0; Ji[5] = x / z2 * g->fx;
      Ji[6] = (1 + y * y / z2) * g->fy; Ji[7] = -x * y / z2 * g->fy; Ji[8] = -x / z * g->fy; Ji[9] = 0; Ji[10] = -1. / z * g->fy; Ji[11] = y / z2 * g->fy;
      double ex = err[2 * i], ey = err[2 * i + 1], rho, hw;
      huber_f(g->w_rep * (ex * ex + ey * ey), g->delta, &rho, &hw);
      double w = g->w_rep * hw;
      wl[i] = w;
      hl[i] = w + g->w_prior;
      bl[2 * i] = -(w * ex + g->w_prior * (f[2 * i] - fhat[2 * i]));
      bl[2 * i + 1] = -(w * ey + g->w_prior * (f[2 * i + 1] - fhat[2 * i + 1]));
      for (int r = 0; r < 6; ++r) {
        bp[r] -= w * (Ji[r] * ex + Ji[6 + r] * ey);
        for (int c = 0; c < 6; ++c) Hpp[6 * r + c] += w * (Ji[r] * Ji[c] + Ji[6 + r] * Ji[6 + c]);
      }
      if (hl[i] > maxd) maxd = hl[i];
    }
    if (it == 0) {
      for (int r = 0; r < 6; ++r) if (fabs(Hpp[7 * r]) > maxd) maxd = fabs(Hpp[7 * r]);
      lambda = 1e-5 * maxd; ni = 2; nbad = 0;
      if (trace) { memcpy(trace + VDO_FLOW2_TRACE_HPP, Hpp, sizeof Hpp); memcpy(trace + VDO_FLOW2_TRACE_BP, bp, sizeof bp); }
    }
    double rho = 0; int qmax = 0;
    se3q Tbk;
    do {
      Tbk = g->T; memcpy(fbk, f, sizeof(double) * 2 * n);                 /* push */
      double S[36], gs[6];
      memcpy(S, Hpp, sizeof S); memcpy(gs, bp, sizeof gs);
      for (int r = 0; r < 6; ++r) S[7 * r] += lambda;
      for (int i = 0; i < n; ++i) {
        const double *Ji = J + 12 * i; double w = wl[i], h = hl[i], p = h + lambda;
        double B0[6], B1[6];
        for (int r = 0; r < 6; ++r) { B0[r] = w * Ji[r]; B1[r] = w * Ji[6 + r]; }
        if (!quirk) {
          double ip = 1.0 / p;
          for (int r = 0; r < 6; ++r) {
            gs[r] -= (B0[r] * bl[2 * i] + B1[r] * bl[2 * i + 1]) * ip;
            for (int c = 0; c < 6; ++c) S[6 * r + c] -= (B0[r] * B0[c] + B1[r] * B1[c]) * ip;
          }
        } else {
          double a = 1.0 / p, b = -h / (p * lambda), c2 = 1.0 / lambda;
          double d0 = a * bl[2 * i] + b * bl[2 * i + 1], d1 = c2 * bl[2 * i + 1];
          for (int r = 0; r < 6; ++r) {
            gs[r] -= B0[r] * d0 + B1[r] * d1;
            for (int c = 0; c < 6; ++c) S[6 * r + c] -= a * B0[r] * B0[c] + b * B0[r] * B1[c] + c2 * B1[r] * B1[c];
          }
        }
      }
      double xnew[6];
      int ok2 = solve6_lower(S, gs, xnew);
      double scale = 0;
      if (ok2) memcpy(xp, xnew, sizeof xnew);
      if (trace && trials == 0) {
        memcpy(trace + VDO_FLOW2_TRACE_S, S, sizeof S); memcpy(trace + VDO_FLOW2_TRACE_G, gs, sizeof gs); memcpy(trace + VDO_FLOW2_TRACE_X, xp, sizeof xp);
      }
      if (ok2) {            /* a failed LDLT leaves the solver's x untouched (linear_solver_dense.h:107-112): the old x is applied */
        for (int i = 0; i < n; ++i) {
          const double *Ji = J + 12 * i; double w = wl[i], h = hl[i], p = h + lambda;
          double cu = bl[2 * i], cv = bl[2 * i + 1];
          for (int r = 0; r < 6; ++r) { cu -= w * Ji[r] * xp[r]; cv -= w * Ji[6 + r] * xp[r]; }
          if (!quirk) { dl[2 * i] = cu / p; dl[2 * i + 1] = cv / p; }
          else { dl[2 * i] = cu / p - h * cv / (p * lambda) + (i >= 1 ? cu / lambda : 0.0); dl[2 * i + 1] = cv / lambda; }
        }
      }
      {
        se3q_oplus(&g->T, xp);
        for (int i = 0; i < 2 * n; ++i) { f[i] += dl[i]; scale += dl[i] * (lambda * dl[i] + bl[i]); }
        for (int r = 0; r < 6; ++r) scale += xp[r] * (lambda * xp[r] + bp[r]);
      }
      temp = flow_chi2(g);
      last_trial_chi = temp;
      if (!ok2) temp = DBL_MAX;
      rho = (current - temp) / (scale + 1e-3);
      const double lambda_trial = lambda, current_before = current;
      int accepted = 0;
      if (rho > 0 && isfinite(temp)) {
        double alpha = 1. - pow(2 * rho - 1, 3);
        if (alpha > 2. / 3.) alpha = 2. / 3.;
        lambda *= (alpha < 1. / 3. ? 1. / 3. : alpha); ni = 2; current = temp; accepted = 1;
      } else {
        lambda *= ni; ni *= 2;
        g->T = Tbk; memcpy(f, fbk, sizeof(double) * 2 * n);                /* pop: estimates only, err[] keeps the trial's values */
      }
      if (trace && trials < VDO_FLOW2_TRACE_MAXREC) {
        double *r = trace + VDO_FLOW2_TRACE_REC + (size_t)VDO_FLOW2_TRACE_RECLEN * trials;
        r[0] = it; r[1] = lambda_trial; r[2] = ok2; r[3] = last_trial_chi; r[4] = current_before; r[5] = scale; r[6] = rho; r[7] = accepted;
        memcpy(r + 8, xp, sizeof xp);
      }
      ++qmax; ++trials;
    } while (rho < 0 && qmax < 10);
    ++iters;
    if (qmax == 10 || rho == 0) { ok = 0; stop = qmax == 10 ? VDO_FLOW2_STOP_TRIALS : VDO_FLOW2_STOP_RHO_ZERO; }
    else { if ((ini - current) * 1e3 < ini) nbad++; else nbad = 0; if (nbad >= 3) { ok = 0; stop = VDO_FLOW2_STOP_NO_PROGRESS; } }
    if (chi2_check < last_trial_chi && it > 0) { if (ok) stop = VDO_FLOW2_STOP_CHI2_ROSE; ok = 0; }   /* sparse_optimizer.cpp:393-396, on the stale _error values */
    chi2_check = last_trial_chi;
  }
  if (trace) {
    trace[VDO_FLOW2_TRACE_STOP] = ok ? VDO_FLOW2_STOP_MAX_ITERS : stop;
    trace[VDO_FLOW2_TRACE_NREC] = trials < VDO_FLOW2_TRACE_MAXREC ? trials : VDO_FLOW2_TRACE_MAXREC;
  }
  /* classification on e->chi2() = 0.1 |_error|^2 compared in float with 0.04f (Optimizer.cc:2899-2930) */
  int n_in = 0;
  for (int i = 0; i < n; ++i) {
    float c = (float)(g->w_rep * (err[2 * i] * err[2 * i] + err[2 * i + 1] * err[2 * i + 1]));
    inlier[i] = !(c > 0.04f);
    n_in += inlier[i];
    flow_out[2 * i] = f[2 * i]; flow_out[2 * i + 1] = f[2 * i + 1];
  }
  double R[9];
  quat_to_m3(g->T.q, R);
  for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) T_out[4 * r + c] = (float)R[3 * r + c]; T_out[4 * r + 3] = (float)g->T.t[r]; }
  T_out[12] = T_out[13] = T_out[14] = 0; T_out[15] = 1;
  if (stats) { stats[0] = iters; stats[1] = trials; stats[2] = flow_chi2(g); stats[3] = lambda; stats[4] = n_in;
               stats[5] = g->T.q[0]; stats[6] = g->T.q[1]; stats[7] = g->T.q[2]; stats[8] = g->T.q[3]; stats[9] = g->T.t[0]; stats[10] = g->T.t[1]; stats[11] = g->T.t[2]; }
  free(Xw); free(obs); free(fhat); free(f); free(fbk); free(err); free(hl); free(bl); free(J); free(wl); free(dl);
  return iters;
}

int vdo_oracle_flow2(int mode, int quirk, int n, const float *pts, const float *depth, const float *flow, const float *K,
                     const float *Tcw_last, const float *T_init, float *T_out, double *flow_out, uint8_t *inlier, double *stats) {
  return flow2_run(mode, quirk, n, pts, depth, flow, K, Tcw_last, T_init, T_out, flow_out, inlier, stats, NULL);
}
int vdo_oracle_flow2_trace(int mode, int quirk, int n, const float *pts, const float *depth, const float *flow, const float *K,
                           const float *Tcw_last, const float *T_init, float *T_out, double *flow_out, uint8_t *inlier, double *stats,
                           double *trace) {
  return flow2_run(mode, quirk, n, pts, depth, flow, K, Tcw_last, T_init, T_out, flow_out, inlier, stats, trace);
}
