/* oracle/pnp_ransac.c -- CPU restatement of the initial-model stage (TEST INFRASTRUCTURE ONLY; never linked into the product).
 *
 * Reference call sites: Tracking::GetInitModelCam / GetInitModelObj (src/Tracking.cc:1614-1715, 1717-1849):
 *   cv::solvePnPRansac(pre_3d, cur_2d, K, dist=0, rvec, tvec, false, 500, 0.4, 0.98, inliers, SOLVEPNP_AP3P), then the
 *   constant-motion model's inlier count at the same 0.4 px threshold decides which initial model is used.
 *
 * The RANSAC engine and the minimal solver live in OpenCV 3.4.0 (Dockerfile:40-63), which is NOT part of the reference tree:
 * parity is UNPINNED for that part.  What is restated here is the published structure of that engine:
 *   - cv::RNG (multiply-with-carry, A = 4164903690) seeded with (uint64)-1, uniform(0,n) = next() % n,
 *   - per iteration 4 distinct indices drawn with per-slot rejection, 3 points -> P3P, 4th point picks the solution,
 *   - inlier = squared float reprojection error <= (float)(thr*thr),
 *   - best model replaced when strictly more inliers; iteration cap updated by RANSACUpdateNumIters(conf, outlier ratio, 4),
 *   - inlier indices ascending; final model refitted on the inliers (OpenCV refits with EPnP; here: 8 Gauss-Newton steps on
 *     the reprojection error -- documented deviation, the refit only seeds the LM of A9).
 * The minimal solver is a plain Grunert-type P3P (quartic in the depth ratio, solved by Ferrari with a bisection on the
 * resolvent), written with + - * / sqrt only, so that the CUDA kernel (compiled --fmad=false) produces bit-identical
 * hypotheses; this file must be compiled with -ffp-contract=off.
 * It is cross-checked against cv2.solvePnPRansac (4.13) in tests/test_pnp_ransac.py (pose and inlier-set agreement, not
 * bit parity). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint64_t s; } cvrng;
static unsigned rng_next(cvrng* r) { r->s = (uint64_t)(unsigned)r->s * 4164903690U + (unsigned)(r->s >> 32); return (unsigned)r->s; }

/* sample table: iters x 4 indices, exactly the draws RANSACPointSetRegistrator::getSubset would make */
void vdo_oracle_ransac_samples(int n, int iters, int* idx) {
  cvrng r = {(uint64_t)-1};
  for (int it = 0; it < iters; ++it)
    for (int i = 0; i < 4; ++i) {
      for (;;) {
        int v = (int)(rng_next(&r) % (unsigned)n), j;
        idx[4 * it + i] = v;
        for (j = 0; j < i; ++j) if (idx[4 * it + j] == v) break;
        if (j == i) break;
      }
    }
}

static double poly4(const double* c, double x) { return (((c[0] * x + c[1]) * x + c[2]) * x + c[3]) * x + c[4]; }
static double dpoly4(const double* c, double x) { return ((4 * c[0] * x + 3 * c[1]) * x + 2 * c[2]) * x + c[3]; }

/* real roots of c0 x^4 + ... + c4 (Ferrari; resolvent root by bisection; two Newton polish steps) */
static int solve_quartic(const double* c, double* roots) {
  if (fabs(c[0]) < 1e-300) return 0;
  const double b = c[1] / c[0], cc = c[2] / c[0], d = c[3] / c[0], e = c[4] / c[0];
  const double b2 = b * b;
  const double p = cc - 3.0 * b2 / 8.0;
  const double q = d - b * cc / 2.0 + b2 * b / 8.0;
  const double r = e - b * d / 4.0 + b2 * cc / 16.0 - 3.0 * b2 * b2 / 256.0;
  double y[4]; int n = 0;
  const double k1 = p, k2 = p * p / 4.0 - r, k3 = -q * q / 8.0;      /* m^3 + k1 m^2 + k2 m + k3 = 0, f(0) <= 0 */
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
    double disc = s * s - 4.0 * (h + g);                            /* y^2 - s y + (h + g) = 0 */
    if (disc >= 0) { const double sq = sqrt(disc); y[n++] = 0.5 * (s + sq); y[n++] = 0.5 * (s - sq); }
    disc = s * s - 4.0 * (h - g);                                   /* y^2 + s y + (h - g) = 0 */
    if (disc >= 0) { const double sq = sqrt(disc); y[n++] = 0.5 * (-s + sq); y[n++] = 0.5 * (-s - sq); }
  } else {                                                          /* biquadratic */
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

static void cross3(const double* a, const double* b, double* o) { o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0]; }
static double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static int unit3(double* a) { const double n = sqrt(dot3(a, a)); if (!(n > 1e-300)) return 0; a[0] = a[0] / n; a[1] = a[1] / n; a[2] = a[2] / n; return 1; }
static int frame3(const double* A, const double* B, const double* C, double* E) {   /* E = [e1 e2 e3] as rows */
  double ab[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]}, ac[3] = {C[0] - A[0], C[1] - A[1], C[2] - A[2]};
  memcpy(E, ab, sizeof ab);
  if (!unit3(E)) return 0;
  cross3(E, ac, E + 6);
  if (!unit3(E + 6)) return 0;
  cross3(E + 6, E, E + 3);
  return 1;
}

/* P3P on points 0..2, solution chosen by the 4th; P world (4x3), uv pixel (4x2); Rt = R row-major (9) + t (3).  Returns 1 if a model exists */
static int p3p4(const double* P, const double* uv, const double* K, double* Rt) {
  double f[3][3];
  for (int k = 0; k < 3; ++k) {
    f[k][0] = (uv[2 * k] - K[2]) / K[0]; f[k][1] = (uv[2 * k + 1] - K[3]) / K[1]; f[k][2] = 1.0;
    if (!unit3(f[k])) return 0;
  }
  double d[3];
  #define SQD(i, j) ((P[3*i]-P[3*j])*(P[3*i]-P[3*j]) + (P[3*i+1]-P[3*j+1])*(P[3*i+1]-P[3*j+1]) + (P[3*i+2]-P[3*j+2])*(P[3*i+2]-P[3*j+2]))
  const double d12 = SQD(1, 2), d02 = SQD(0, 2), d01 = SQD(0, 1);
  #undef SQD
  if (!(d02 > 1e-300) || !(d01 > 1e-300) || !(d12 > 1e-300)) return 0;
  const double c12 = dot3(f[1], f[2]), c02 = dot3(f[0], f[2]), c01 = dot3(f[0], f[1]);
  const double K1 = (d12 - d01) / d02, K2 = d01 / d02;
  const double n2 = K1 - 1.0, n1 = -2.0 * K1 * c02, n0 = K1 + 1.0, e1 = -2.0 * c12, e0 = 2.0 * c01;
  const double q2 = -K2, q1 = 2.0 * K2 * c02, q0 = 1.0 - K2;
  double c[5];
  /* N^2 - 2 c01 N D + D^2 Q */
  const double nd3 = n2 * e1, nd2 = n2 * e0 + n1 * e1, nd1 = n1 * e0 + n0 * e1, nd0 = n0 * e0;
  const double dd2 = e1 * e1, dd1 = 2.0 * e1 * e0, dd0 = e0 * e0;
  c[0] = n2 * n2 + dd2 * q2;
  c[1] = 2.0 * n2 * n1 - 2.0 * c01 * nd3 + (dd2 * q1 + dd1 * q2);
  c[2] = (2.0 * n2 * n0 + n1 * n1) - 2.0 * c01 * nd2 + (dd2 * q0 + dd1 * q1 + dd0 * q2);
  c[3] = 2.0 * n1 * n0 - 2.0 * c01 * nd1 + (dd1 * q0 + dd0 * q1);
  c[4] = n0 * n0 - 2.0 * c01 * nd0 + dd0 * q0;
  double roots[4];
  const int nr = solve_quartic(c, roots);
  double E[9];
  if (!frame3(P, P + 3, P + 6, E)) return 0;
  double best = 1e300; int found = 0;
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
    double X[9] = {s0 * f[0][0], s0 * f[0][1], s0 * f[0][2], s1 * f[1][0], s1 * f[1][1], s1 * f[1][2], s2 * f[2][0], s2 * f[2][1], s2 * f[2][2]};
    double G[9];
    if (!frame3(X, X + 3, X + 6, G)) continue;
    double R[9], t[3];
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) R[3 * a + b] = G[a] * E[b] + G[3 + a] * E[3 + b] + G[6 + a] * E[6 + b];
    for (int a = 0; a < 3; ++a) t[a] = X[a] - (R[3 * a] * P[0] + R[3 * a + 1] * P[1] + R[3 * a + 2] * P[2]);
    const double* P3 = P + 9;
    const double xc = R[0] * P3[0] + R[1] * P3[1] + R[2] * P3[2] + t[0], yc = R[3] * P3[0] + R[4] * P3[1] + R[5] * P3[2] + t[1],
                 zc = R[6] * P3[0] + R[7] * P3[1] + R[8] * P3[2] + t[2];
    if (!(zc > 0)) continue;
    const double du = K[0] * xc / zc + K[2] - uv[6], dv = K[1] * yc / zc + K[3] - uv[7];
    const double err = du * du + dv * dv;
    if (err < best) { best = err; found = 1; memcpy(Rt, R, sizeof R); memcpy(Rt + 9, t, sizeof t); }
  }
  (void)d;
  return found;
}

static int is_inlier(const double* Rt, const float* obj, const float* img, const double* K, float thr2) {
  const double X = obj[0], Y = obj[1], Z = obj[2];
  const double xc = Rt[0] * X + Rt[1] * Y + Rt[2] * Z + Rt[9], yc = Rt[3] * X + Rt[4] * Y + Rt[5] * Z + Rt[10], zc = Rt[6] * X + Rt[7] * Y + Rt[8] * Z + Rt[11];
  const double iz = zc != 0.0 ? 1.0 / zc : 1.0;
  const float pu = (float)(K[0] * (xc * iz) + K[2]), pv = (float)(K[1] * (yc * iz) + K[3]);
  const float du = img[0] - pu, dv = img[1] - pv;
  const float err = du * du + dv * dv;
  return err <= thr2;
}

static int update_num_iters(double p, double ep, int model_points, int max_iters) {     /* cv::RANSACUpdateNumIters */
  p = fmax(p, 0.); p = fmin(p, 1.); ep = fmax(ep, 0.); ep = fmin(ep, 1.);
  double num = fmax(1. - p, 2.2250738585072014e-308), denom = 1. - pow(1. - ep, model_points);
  if (denom < 2.2250738585072014e-308) return 0;
  num = log(num); denom = log(denom);
  return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)lrint(num / denom);
}

static int chol6_solve(double* H, const double* b, double* x) {      /* H (36, row-major, overwritten) x = b */
  for (int j = 0; j < 6; ++j) {
    double s = H[7 * j];
    for (int k = 0; k < j; ++k) s = s - H[6 * j + k] * H[6 * j + k];
    if (!(s > 0)) return 0;
    const double l = sqrt(s); H[7 * j] = l;
    for (int i = j + 1; i < 6; ++i) {
      double v = H[6 * i + j];
      for (int k = 0; k < j; ++k) v = v - H[6 * i + k] * H[6 * j + k];
      H[6 * i + j] = v / l;
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) { double v = b[i]; for (int k = 0; k < i; ++k) v = v - H[6 * i + k] * y[k]; y[i] = v / H[7 * i]; }
  for (int i = 5; i >= 0; --i) { double v = y[i]; for (int k = i + 1; k < 6; ++k) v = v - H[6 * k + i] * x[k]; x[i] = v / H[7 * i]; }
  return 1;
}

#define GN_LANES 256
/* 8 Gauss-Newton steps on the pixel reprojection error over the listed inliers; update T <- Cayley(w) * T.
 * Summation order: lane l accumulates inliers l, l+256, ... ascending; lanes are then folded 128, 64, ..., 1 (the CUDA kernel's order) */
static void gn_refit(double* Rt, int ninl, const int* inl, const float* obj, const float* img, const double* K) {
  double (*acc)[27] = malloc(sizeof(double[27]) * GN_LANES);
  for (int it = 0; it < 8; ++it) {
    memset(acc, 0, sizeof(double[27]) * GN_LANES);
    for (int l = 0; l < GN_LANES; ++l)
      for (int q = l; q < ninl; q += GN_LANES) {
        const float* o = obj + 3 * inl[q]; const float* m = img + 2 * inl[q];
        const double X = o[0], Y = o[1], Z = o[2];
        const double xc = Rt[0] * X + Rt[1] * Y + Rt[2] * Z + Rt[9], yc = Rt[3] * X + Rt[4] * Y + Rt[5] * Z + Rt[10], zc = Rt[6] * X + Rt[7] * Y + Rt[8] * Z + Rt[11];
        const double iz = 1.0 / zc;
        const double ru = K[0] * xc * iz + K[2] - (double)m[0], rv = K[1] * yc * iz + K[3] - (double)m[1];
        /* d(proj)/d(Xc) and dXc/d[w, v] = [-[Xc]x*2 | I] for the Cayley update (dR = 2[w]x to first order) */
        const double a0 = K[0] * iz, a2 = -K[0] * xc * iz * iz, b1 = K[1] * iz, b2 = -K[1] * yc * iz * iz;
        double Ju[6], Jv[6];
        /* -2[Xc]x columns: d/dw0 = 2*(0, -zc... ) -> dXc = 2 w x Xc */
        Ju[0] = 2.0 * (a2 * yc);              Ju[1] = 2.0 * (a0 * zc - a2 * xc);  Ju[2] = 2.0 * (-a0 * yc);
        Jv[0] = 2.0 * (-b1 * zc + b2 * yc);   Jv[1] = 2.0 * (-b2 * xc);           Jv[2] = 2.0 * (b1 * xc);
        Ju[3] = a0; Ju[4] = 0.0; Ju[5] = a2;  Jv[3] = 0.0; Jv[4] = b1; Jv[5] = b2;
        int k = 0;
        for (int a = 0; a < 6; ++a)
          for (int b = a; b < 6; ++b) { acc[l][k] = acc[l][k] + (Ju[a] * Ju[b] + Jv[a] * Jv[b]); ++k; }
        for (int a = 0; a < 6; ++a) acc[l][21 + a] = acc[l][21 + a] + (Ju[a] * ru + Jv[a] * rv);
      }
    for (int s = GN_LANES / 2; s >= 1; s >>= 1)
      for (int l = 0; l < s; ++l)
        for (int k = 0; k < 27; ++k) acc[l][k] = acc[l][k] + acc[l + s][k];
    double H[36], g[6], x[6];
    int k = 0;
    for (int a = 0; a < 6; ++a)
      for (int b = a; b < 6; ++b) { H[6 * a + b] = acc[0][k]; H[6 * b + a] = acc[0][k]; ++k; }
    for (int a = 0; a < 6; ++a) g[a] = -acc[0][21 + a];
    if (!chol6_solve(H, g, x)) break;
    const double w0 = x[0], w1 = x[1], w2 = x[2], n2 = w0 * w0 + w1 * w1 + w2 * w2, sc = 2.0 / (1.0 + n2);
    /* C = I + sc ([w]x + [w]x^2) */
    double C[9] = {1.0 + sc * (-(w1 * w1 + w2 * w2)), sc * (-w2 + w0 * w1), sc * (w1 + w0 * w2),
                   sc * (w2 + w0 * w1), 1.0 + sc * (-(w0 * w0 + w2 * w2)), sc * (-w0 + w1 * w2),
                   sc * (-w1 + w0 * w2), sc * (w0 + w1 * w2), 1.0 + sc * (-(w0 * w0 + w1 * w1))};
    double Rn[12];
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) Rn[3 * a + b] = C[3 * a] * Rt[b] + C[3 * a + 1] * Rt[3 + b] + C[3 * a + 2] * Rt[6 + b];
      Rn[9 + a] = C[3 * a] * Rt[9] + C[3 * a + 1] * Rt[10] + C[3 * a + 2] * Rt[11] + x[3 + a];
    }
    memcpy(Rt, Rn, sizeof Rn);
  }
  free(acc);
}

/* stats: [0] iterations executed, [1] index of the winning hypothesis, [2] #valid hypotheses among those executed.
 * Returns the number of inliers (0 = failure; Rt untouched).  inl receives ascending inlier indices. */
int vdo_oracle_pnp_ransac(int n, const float* obj, const float* img, const double* K, int max_iters, double thr, double conf,
                          double* Rt, int* inl, int* stats, double* Rt_best_hyp) {
  if (stats) stats[0] = stats[1] = stats[2] = 0;
  if (n < 4) return 0;
  int* samples = malloc(sizeof(int) * 4 * (size_t)max_iters);
  vdo_oracle_ransac_samples(n, max_iters, samples);
  const float thr2 = (float)(thr * thr);
  int niters = max_iters, best = 0, best_it = -1, nvalid = 0, it;
  double best_Rt[12];
  for (it = 0; it < niters; ++it) {
    double P[12], uv[8], M[12];
    for (int k = 0; k < 4; ++k) {
      const int i = samples[4 * it + k];
      P[3 * k] = obj[3 * i]; P[3 * k + 1] = obj[3 * i + 1]; P[3 * k + 2] = obj[3 * i + 2];
      uv[2 * k] = img[2 * i]; uv[2 * k + 1] = img[2 * i + 1];
    }
    if (!p3p4(P, uv, K, M)) continue;
    ++nvalid;
    int good = 0;
    for (int i = 0; i < n; ++i) good += is_inlier(M, obj + 3 * i, img + 2 * i, K, thr2);
    if (good > (best > 3 ? best : 3)) {
      best = good; best_it = it; memcpy(best_Rt, M, sizeof M);
      niters = update_num_iters(conf, (double)(n - good) / n, 4, niters);
    }
  }
  free(samples);
  if (stats) { stats[0] = it; stats[1] = best_it; stats[2] = nvalid; }
  if (best_it < 0) return 0;
  int m = 0;
  for (int i = 0; i < n; ++i) if (is_inlier(best_Rt, obj + 3 * i, img + 2 * i, K, thr2)) inl[m++] = i;
  if (Rt_best_hyp) memcpy(Rt_best_hyp, best_Rt, sizeof best_Rt);
  memcpy(Rt, best_Rt, sizeof best_Rt);
  gn_refit(Rt, m, inl, obj, img, K);
  return m;
}

/* debug / unit-test entry: one minimal solve */
int vdo_oracle_p3p4(const double* P, const double* uv, const double* K, double* Rt) { return p3p4(P, uv, K, Rt); }
