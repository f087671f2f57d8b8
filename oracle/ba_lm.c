/*
 * oracle/ba_lm.c -- TEST INFRASTRUCTURE ONLY (CPU oracle + timed CPU baseline; never on the product path).
 *
 * CPU restatement of the reference's batch factor-graph optimisation:
 *   graph semantics   src/Optimizer.cc:1232-2175 (FullBatchOptimization), :42-1230 (PartialBatchOptimization)
 *   LM                g2o/core/optimization_algorithm_levenberg.cpp:61-189
 *   outer loop        g2o/core/sparse_optimizer.cpp:354-427  (incl. the "chi2 went up -> stop" patch :393-396)
 *   terminate action  g2o/core/sparse_optimizer_terminate_action.cpp:49-85
 *   quadratic forms   g2o/core/base_{unary,binary,multi}_edge.hpp
 *   system build      g2o/core/block_solver.hpp:501-604 (no Schur: nothing is marginalised in the batch optimisers)
 *   linear solve      g2o/solvers/linear_solver_csparse.h:108-144 -> sparse Cholesky of the FULL system
 *                     (numeric phase as in g2o/solvers/csparse_extension.cpp:69-124, i.e. Davis' up-looking
 *                     Cholesky; CSparse itself is an un-vendored dependency -- the distro's libsuitesparse,
 *                     Dockerfile:69 -- whose published algorithm (T. Davis, "Direct Methods for Sparse Linear
 *                     Systems", ch. 4) is restated here.  Ordering: the reference uses block-AMD
 *                     (linear_solver_csparse.h:248-346); this file uses "points first, then 6-dof vertices",
 *                     the classic bundle-adjustment fill-reducing order.  The ordering changes rounding only.)
 *
 * Parity status: UNPINNED.  The reference has no tests, fixtures or golden vectors (SURVEY.md section 4) and cannot be
 * built in this container (Eigen3 / OpenCV / CSparse absent), so this restatement is checked only against
 * itself (finite-difference Jacobians, linear-solve residuals) -- see tests/test_oracle_ba.py.
 *
 * Restrictions (match the reference's usage): information matrices are scalar * Identity; the camera offset
 * parameter is Identity; ternary-edge measurement is zero; no fixed vertices.
 */
#include <stdio.h>
#include <stdlib.h>
#include <stdint.h>
#include <float.h>
#include "ba_edges.h"

typedef struct {
  int n_se3, n_pt;
  double *se3, *pt;                 /* states (in/out) */
  int n_prior; const int *prior_v; const double *prior_Z, *prior_w;
  int n_se3e; const int *se3e_ij; const double *se3e_Z, *se3e_w, *se3e_delta;
  int n_obs; const int *obs_cp; const double *obs_z, *obs_w, *obs_delta;
  int n_ter; const int *ter_pph; const double *ter_w, *ter_delta;
  /* linear system */
  int n;                            /* scalar dimension 3P + 6C */
  int64_t nnzA; int64_t *Ap; int *Ai; double *Ax;   /* upper triangular CSC of H (permuted order) */
  int64_t npair; int64_t *pair_key; int *pair_off;  /* unique off-diagonal block pairs (col-major key) and row offset inside the column */
  int *diag_off;                    /* per block: row offset of the diagonal block inside its columns */
  /* per-edge pair indices */
  int64_t *obs_pair, *ter_pair /*3 per*/, *se3e_pair;
  double *b, *x;
  /* cholesky */
  int *parent; int64_t *Lp; int *Li; double *Lx; int64_t lnz;
  int *cwork; double *xwork; int64_t *colfill;
  long oplus_calls;
} ba_t;

#include <time.h>
static double now_s(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + 1e-9 * ts.tv_nsec; }

static inline int blk_dim(const ba_t *g, int blk) { return blk < g->n_pt ? 3 : 6; }
static inline int blk_col(const ba_t *g, int blk) { return blk < g->n_pt ? 3 * blk : 3 * g->n_pt + 6 * (blk - g->n_pt); }

static int cmp_i64(const void *a, const void *b) {
  int64_t x = *(const int64_t *)a, y = *(const int64_t *)b;
  return (x > y) - (x < y);
}
static inline int64_t mk_key(const ba_t *g, int a, int b) { /* a<b block ids; column-major */
  int64_t N = (int64_t)g->n_pt + g->n_se3;
  return (int64_t)b * N + a;
}
static int64_t find_pair(const ba_t *g, int a, int b) {
  if (a > b) { int t = a; a = b; b = t; }
  int64_t key = mk_key(g, a, b), lo = 0, hi = g->npair - 1;
  while (lo <= hi) {
    int64_t mid = (lo + hi) >> 1;
    if (g->pair_key[mid] < key) lo = mid + 1; else if (g->pair_key[mid] > key) hi = mid - 1; else return mid;
  }
  return -1;
}

/* ---- structure (the analogue of BlockSolver::buildStructure, block_solver.hpp:142-295) ---- */
static int build_structure(ba_t *g) {
  const int P = g->n_pt, C = g->n_se3;
  const int64_t NB = (int64_t)P + C;
  int64_t cap = (int64_t)g->n_obs + 3 * (int64_t)g->n_ter + g->n_se3e, m = 0;
  int64_t *keys = (int64_t *)malloc(sizeof(int64_t) * (cap > 0 ? cap : 1));
  for (int e = 0; e < g->n_obs; ++e) keys[m++] = mk_key(g, g->obs_cp[2 * e + 1], P + g->obs_cp[2 * e]);
  for (int e = 0; e < g->n_ter; ++e) {
    int p1 = g->ter_pph[3 * e], p2 = g->ter_pph[3 * e + 1], h = P + g->ter_pph[3 * e + 2];
    keys[m++] = p1 < p2 ? mk_key(g, p1, p2) : mk_key(g, p2, p1);
    keys[m++] = mk_key(g, p1, h);
    keys[m++] = mk_key(g, p2, h);
  }
  for (int e = 0; e < g->n_se3e; ++e) {
    int i = P + g->se3e_ij[2 * e], j = P + g->se3e_ij[2 * e + 1];
    keys[m++] = i < j ? mk_key(g, i, j) : mk_key(g, j, i);
  }
  qsort(keys, (size_t)m, sizeof(int64_t), cmp_i64);
  int64_t u = 0;
  for (int64_t i = 0; i < m; ++i) if (i == 0 || keys[i] != keys[i - 1]) keys[u++] = keys[i];
  g->npair = u; g->pair_key = keys;
  g->pair_off = (int *)malloc(sizeof(int) * (u > 0 ? u : 1));
  g->diag_off = (int *)malloc(sizeof(int) * NB);
  g->n = 3 * P + 6 * C;
  g->Ap = (int64_t *)malloc(sizeof(int64_t) * ((size_t)g->n + 1));
  /* pass 1: per column-block height */
  int64_t nnz = 0, k = 0;
  for (int64_t b = 0; b < NB; ++b) {
    int rows = 0;
    while (k < u && keys[k] / NB == b) { g->pair_off[k] = rows; rows += blk_dim(g, (int)(keys[k] % NB)); ++k; }
    g->diag_off[b] = rows;
    int db = blk_dim(g, (int)b), c0 = blk_col(g, (int)b);
    for (int c = 0; c < db; ++c) { g->Ap[c0 + c] = nnz; nnz += rows + c + 1; }
  }
  g->Ap[g->n] = nnz; g->nnzA = nnz;
  g->Ai = (int *)malloc(sizeof(int) * (size_t)nnz);
  g->Ax = (double *)malloc(sizeof(double) * (size_t)nnz);
  k = 0;
  for (int64_t b = 0; b < NB; ++b) {
    int64_t k0 = k;
    while (k < u && keys[k] / NB == b) ++k;
    int db = blk_dim(g, (int)b), c0 = blk_col(g, (int)b);
    for (int c = 0; c < db; ++c) {
      int64_t p = g->Ap[c0 + c];
      for (int64_t q = k0; q < k; ++q) {
        int a = (int)(keys[q] % NB), da = blk_dim(g, a), r0 = blk_col(g, a);
        for (int r = 0; r < da; ++r) g->Ai[p++] = r0 + r;
      }
      for (int r = 0; r <= c; ++r) g->Ai[p++] = c0 + r;
    }
  }
  g->obs_pair = (int64_t *)malloc(sizeof(int64_t) * (g->n_obs > 0 ? g->n_obs : 1));
  g->ter_pair = (int64_t *)malloc(sizeof(int64_t) * (g->n_ter > 0 ? 3 * (size_t)g->n_ter : 1));
  g->se3e_pair = (int64_t *)malloc(sizeof(int64_t) * (g->n_se3e > 0 ? g->n_se3e : 1));
  for (int e = 0; e < g->n_obs; ++e) g->obs_pair[e] = find_pair(g, g->obs_cp[2 * e + 1], P + g->obs_cp[2 * e]);
  for (int e = 0; e < g->n_ter; ++e) {
    int p1 = g->ter_pph[3 * e], p2 = g->ter_pph[3 * e + 1], h = P + g->ter_pph[3 * e + 2];
    g->ter_pair[3 * e] = find_pair(g, p1, p2);
    g->ter_pair[3 * e + 1] = find_pair(g, p1, h);
    g->ter_pair[3 * e + 2] = find_pair(g, p2, h);
  }
  for (int e = 0; e < g->n_se3e; ++e) g->se3e_pair[e] = find_pair(g, P + g->se3e_ij[2 * e], P + g->se3e_ij[2 * e + 1]);
  g->b = (double *)calloc((size_t)g->n, sizeof(double));
  g->x = (double *)calloc((size_t)g->n, sizeof(double));
  return 0;
}

/* add J_a^T * W * J_b (W scalar) into the stored block; a,b are block ids, Ja is (dim x da), Jb is (dim x db) row-major */
static void add_offdiag(ba_t *g, int64_t pair, int a, int b, const double *Ja, const double *Jb, int dim, double w) {
  const double *JA = Ja, *JB = Jb;
  if (a > b) { int t = a; a = b; b = t; JA = Jb; JB = Ja; }
  int da = blk_dim(g, a), db = blk_dim(g, b), c0 = blk_col(g, b), off = g->pair_off[pair];
  for (int c = 0; c < db; ++c) {
    double *col = g->Ax + g->Ap[c0 + c] + off;
    for (int r = 0; r < da; ++r) {
      double s = 0;
      for (int k = 0; k < dim; ++k) s += JA[k * da + r] * JB[k * db + c];
      col[r] += w * s;
    }
  }
}
static void add_diag(ba_t *g, int blk, const double *J, int dim, double w, const double *err) {
  int d = blk_dim(g, blk), c0 = blk_col(g, blk), off = g->diag_off[blk];
  for (int c = 0; c < d; ++c) {
    double *col = g->Ax + g->Ap[c0 + c] + off;
    for (int r = 0; r <= c; ++r) {
      double s = 0;
      for (int k = 0; k < dim; ++k) s += J[k * d + r] * J[k * d + c];
      col[r] += w * s;
    }
    double s = 0;
    for (int k = 0; k < dim; ++k) s += J[k * d + c] * err[k];
    g->b[c0 + c] -= w * s;        /* b += J^T * (-rho' Omega e) */
  }
}

/* ---- errors / robust chi2 (SparseOptimizer::computeActiveErrors + activeRobustChi2, sparse_optimizer.cpp:61-114) ---- */
static double robust_chi2(const ba_t *g) {
  double chi = 0, e[6], rho[3];
  for (int k = 0; k < g->n_prior; ++k) {
    edge_prior_error(g->prior_Z + 12 * k, g->se3 + 12 * g->prior_v[k], e);
    double c = 0; for (int i = 0; i < 6; ++i) c += e[i] * e[i];
    chi += g->prior_w[k] * c;
  }
  for (int k = 0; k < g->n_se3e; ++k) {
    edge_se3_error(g->se3e_Z + 12 * k, g->se3 + 12 * g->se3e_ij[2 * k], g->se3 + 12 * g->se3e_ij[2 * k + 1], e);
    double c = 0; for (int i = 0; i < 6; ++i) c += e[i] * e[i];
    c *= g->se3e_w[k];
    if (g->se3e_delta[k] > 0) { huber(c, g->se3e_delta[k], rho); chi += rho[0]; } else chi += c;
  }
  for (int k = 0; k < g->n_obs; ++k) {
    edge_obs_error(g->se3 + 12 * g->obs_cp[2 * k], g->pt + 3 * g->obs_cp[2 * k + 1], g->obs_z + 3 * k, e);
    double c = g->obs_w[k] * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
    if (g->obs_delta[k] > 0) { huber(c, g->obs_delta[k], rho); chi += rho[0]; } else chi += c;
  }
  for (int k = 0; k < g->n_ter; ++k) {
    edge_ter_error(g->pt + 3 * g->ter_pph[3 * k], g->pt + 3 * g->ter_pph[3 * k + 1], g->se3 + 12 * g->ter_pph[3 * k + 2], e);
    double c = g->ter_w[k] * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
    if (g->ter_delta[k] > 0) { huber(c, g->ter_delta[k], rho); chi += rho[0]; } else chi += c;
  }
  return chi;
}

/* ---- buildSystem (block_solver.hpp:501-560): linearizeOplus + constructQuadraticForm for every edge ---- */
static void build_system(ba_t *g) {
  const int P = g->n_pt;
  memset(g->Ax, 0, sizeof(double) * (size_t)g->nnzA);
  memset(g->b, 0, sizeof(double) * (size_t)g->n);
  double e[6], rho[3], Ji[36], Jj[36];
  for (int k = 0; k < g->n_prior; ++k) {         /* BaseUnaryEdge, no kernel (Optimizer.cc:1364-1373) */
    int v = g->prior_v[k];
    edge_prior_error(g->prior_Z + 12 * k, g->se3 + 12 * v, e);
    edge_prior_jac(g->prior_Z + 12 * k, g->se3 + 12 * v, Ji);
    add_diag(g, P + v, Ji, 6, g->prior_w[k], e);
  }
  for (int k = 0; k < g->n_se3e; ++k) {          /* BaseBinaryEdge<6> */
    int i = g->se3e_ij[2 * k], j = g->se3e_ij[2 * k + 1];
    const double *Z = g->se3e_Z + 12 * k;
    edge_se3_error(Z, g->se3 + 12 * i, g->se3 + 12 * j, e);
    edge_se3_jac(Z, g->se3 + 12 * i, g->se3 + 12 * j, Ji, Jj);
    double w = g->se3e_w[k];
    if (g->se3e_delta[k] > 0) {
      double c = 0; for (int q = 0; q < 6; ++q) c += e[q] * e[q];
      huber(w * c, g->se3e_delta[k], rho); w *= rho[1];
    }
    add_diag(g, P + i, Ji, 6, w, e);
    add_diag(g, P + j, Jj, 6, w, e);
    add_offdiag(g, g->se3e_pair[k], P + i, P + j, Ji, Jj, 6, w);
  }
  for (int k = 0; k < g->n_obs; ++k) {           /* BaseBinaryEdge<3> */
    int c = g->obs_cp[2 * k], p = g->obs_cp[2 * k + 1];
    edge_obs_error(g->se3 + 12 * c, g->pt + 3 * p, g->obs_z + 3 * k, e);
    edge_obs_jac(g->se3 + 12 * c, g->pt + 3 * p, Ji, Jj);
    double w = g->obs_w[k];
    if (g->obs_delta[k] > 0) { huber(w * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), g->obs_delta[k], rho); w *= rho[1]; }
    add_diag(g, P + c, Ji, 3, w, e);
    add_diag(g, p, Jj, 3, w, e);
    add_offdiag(g, g->obs_pair[k], P + c, p, Ji, Jj, 3, w);
  }
  for (int k = 0; k < g->n_ter; ++k) {           /* BaseMultiEdge<3> (base_multi_edge.hpp:35-48,170-222) */
    int p1 = g->ter_pph[3 * k], p2 = g->ter_pph[3 * k + 1], h = g->ter_pph[3 * k + 2];
    double J1[9], J2[9], Jh[18];
    edge_ter_error(g->pt + 3 * p1, g->pt + 3 * p2, g->se3 + 12 * h, e);
    edge_ter_jac(g->pt + 3 * p2, g->se3 + 12 * h, J1, J2, Jh);
    double w = g->ter_w[k];
    if (g->ter_delta[k] > 0) { huber(w * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), g->ter_delta[k], rho); w *= rho[1]; }
    add_diag(g, p1, J1, 3, w, e);
    add_diag(g, p2, J2, 3, w, e);
    add_diag(g, P + h, Jh, 3, w, e);
    add_offdiag(g, g->ter_pair[3 * k], p1, p2, J1, J2, 3, w);
    add_offdiag(g, g->ter_pair[3 * k + 1], p1, P + h, J1, Jh, 3, w);
    add_offdiag(g, g->ter_pair[3 * k + 2], p2, P + h, J2, Jh, 3, w);
  }
}

/* ---- sparse Cholesky (symbolic: elimination tree + column counts; numeric: up-looking) ---- */
static int64_t row_pattern(const ba_t *g, int k, int *stack, int *mark) {
  /* nonzero pattern of row k of L = nodes reached from the entries of A(:,k) up the elimination tree */
  int64_t top = g->n;
  mark[k] = k;
  for (int64_t p = g->Ap[k]; p < g->Ap[k + 1]; ++p) {
    int i = g->Ai[p];
    if (i >= k) continue;
    int len = 0;
    while (mark[i] != k) { stack[len++] = i; mark[i] = k; i = g->parent[i]; }
    while (len > 0) stack[--top] = stack[--len];
  }
  return top;
}
static int chol_symbolic(ba_t *g) {
  const int n = g->n;
  g->parent = (int *)malloc(sizeof(int) * n);
  int *anc = (int *)malloc(sizeof(int) * n);
  for (int k = 0; k < n; ++k) {
    g->parent[k] = -1; anc[k] = -1;
    for (int64_t p = g->Ap[k]; p < g->Ap[k + 1]; ++p) {
      int i = g->Ai[p];
      while (i != -1 && i < k) {
        int nx = anc[i];
        anc[i] = k;
        if (nx == -1) g->parent[i] = k;
        i = nx;
      }
    }
  }
  free(anc);
  int *mark = (int *)malloc(sizeof(int) * n), *stack = (int *)malloc(sizeof(int) * n);
  int64_t *cnt = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
  for (int k = 0; k < n; ++k) mark[k] = -1;
  for (int k = 0; k < n; ++k) {
    int64_t top = row_pattern(g, k, stack, mark);
    for (int64_t t = top; t < n; ++t) cnt[stack[t]]++;
    cnt[k]++;
  }
  g->Lp = (int64_t *)malloc(sizeof(int64_t) * ((size_t)n + 1));
  int64_t s = 0;
  for (int k = 0; k < n; ++k) { g->Lp[k] = s; s += cnt[k]; }
  g->Lp[n] = s; g->lnz = s;
  free(cnt);
  g->Li = (int *)malloc(sizeof(int) * (size_t)s);
  g->Lx = (double *)malloc(sizeof(double) * (size_t)s);
  g->cwork = mark; g->xwork = (double *)calloc((size_t)n, sizeof(double));
  g->colfill = (int64_t *)malloc(sizeof(int64_t) * n);
  free(stack);
  return 0;
}
/* factor (A + lambda I) and solve; returns 0 if not positive definite */
static int chol_solve(ba_t *g, double lambda) {
  const int n = g->n;
  int *mark = g->cwork, *stack = (int *)malloc(sizeof(int) * n);
  double *w = g->xwork;
  for (int k = 0; k < n; ++k) { mark[k] = -1; g->colfill[k] = g->Lp[k]; w[k] = 0; }
  int ok = 1;
  for (int k = 0; k < n && ok; ++k) {
    int64_t top = row_pattern(g, k, stack, mark);
    double d = 0;
    for (int64_t p = g->Ap[k]; p < g->Ap[k + 1]; ++p) {
      int i = g->Ai[p];
      if (i < k) w[i] = g->Ax[p]; else if (i == k) d = g->Ax[p] + lambda;
    }
    for (int64_t t = top; t < n; ++t) {
      int i = stack[t];
      double lki = w[i] / g->Lx[g->Lp[i]];
      w[i] = 0;
      for (int64_t p = g->Lp[i] + 1; p < g->colfill[i]; ++p) w[g->Li[p]] -= g->Lx[p] * lki;
      d -= lki * lki;
      int64_t q = g->colfill[i]++;
      g->Li[q] = k; g->Lx[q] = lki;
    }
    if (d <= 0) { ok = 0; break; }
    int64_t q = g->colfill[k]++;
    g->Li[q] = k; g->Lx[q] = sqrt(d);
  }
  free(stack);
  if (!ok) return 0;
  double *x = g->x;
  memcpy(x, g->b, sizeof(double) * n);
  for (int j = 0; j < n; ++j) {               /* L y = b */
    x[j] /= g->Lx[g->Lp[j]];
    for (int64_t p = g->Lp[j] + 1; p < g->Lp[j + 1]; ++p) x[g->Li[p]] -= g->Lx[p] * x[j];
  }
  for (int j = n - 1; j >= 0; --j) {          /* L^T x = y */
    for (int64_t p = g->Lp[j] + 1; p < g->Lp[j + 1]; ++p) x[j] -= g->Lx[p] * x[g->Li[p]];
    x[j] /= g->Lx[g->Lp[j]];
  }
  return 1;
}

/* ---- update (SparseOptimizer::update, sparse_optimizer.cpp:430-443; VertexSE3::oplusImpl; VertexPointXYZ += ) ---- */
static void apply_update(ba_t *g) {
  const int P = g->n_pt, C = g->n_se3;
  for (int p = 0; p < 3 * P; ++p) g->pt[p] += g->x[p];
  g->oplus_calls++;
  int ortho = 0;
  if (g->oplus_calls > 1000) { g->oplus_calls = 0; ortho = 1; }   /* vertex_se3.h:110-113 */
  for (int v = 0; v < C; ++v) {
    iso_oplus(g->se3 + 12 * v, g->x + 3 * P + 6 * v);
    if (ortho) m3_approx_orthogonalize(g->se3 + 12 * v);
  }
}

static void ba_free(ba_t *g) {
  free(g->Ap); free(g->Ai); free(g->Ax); free(g->pair_key); free(g->pair_off); free(g->diag_off);
  free(g->obs_pair); free(g->ter_pair); free(g->se3e_pair); free(g->b); free(g->x);
  free(g->parent); free(g->Lp); free(g->Li); free(g->Lx); free(g->cwork); free(g->xwork); free(g->colfill);
}

/*
 * Runs SparseOptimizer::optimize(max_iters) with OptimizationAlgorithmLevenberg and a
 * SparseOptimizerTerminateAction(gain_threshold) (gain_threshold <= 0 disables the action), verbose=true
 * semantics (errors are recomputed at the current estimate after each iteration, Optimizer.cc:1769).
 * chi2_hist[0] = initial robust chi2, chi2_hist[i+1] = robust chi2 after iteration i.
 * stats[0]=final lambda, stats[1]=total LM trials, stats[2]=nnz(L), stats[3]=seconds in linear solves,
 * stats[4]=seconds total.
 * Returns the number of iterations performed (like optimize()), or -1 on structural failure.
 */
#include "ba_block.h"

static int ba_optimize_impl(int n_se3, double *se3, int n_pt, double *pt,
                           int n_prior, const int *prior_v, const double *prior_Z, const double *prior_w,
                           int n_se3e, const int *se3e_ij, const double *se3e_Z, const double *se3e_w, const double *se3e_delta,
                           int n_obs, const int *obs_cp, const double *obs_z, const double *obs_w, const double *obs_delta,
                           int n_ter, const int *ter_pph, const double *ter_w, const double *ter_delta,
                           int max_iters, double gain_threshold, int verbose, double *chi2_hist, double *stats,
                           int solver, const int *se3_pos, int nthreads, double *lam_hist, double time_budget_s, double *t_hist) {
  ba_t G; memset(&G, 0, sizeof G);
  ba_t *g = &G;
  blk_t BK; blk_t *B = &BK;
  g->n_se3 = n_se3; g->se3 = se3; g->n_pt = n_pt; g->pt = pt;
  g->n_prior = n_prior; g->prior_v = prior_v; g->prior_Z = prior_Z; g->prior_w = prior_w;
  g->n_se3e = n_se3e; g->se3e_ij = se3e_ij; g->se3e_Z = se3e_Z; g->se3e_w = se3e_w; g->se3e_delta = se3e_delta;
  g->n_obs = n_obs; g->obs_cp = obs_cp; g->obs_z = obs_z; g->obs_w = obs_w; g->obs_delta = obs_delta;
  g->n_ter = n_ter; g->ter_pph = ter_pph; g->ter_w = ter_w; g->ter_delta = ter_delta;
  double t_start = now_s(), t_lin = 0, t_setup = 0;
  if (solver == 0) {
    build_structure(g);
    chol_symbolic(g);
  } else {                                  /* blocked solver (ba_block.h): same system, same solution */
    g->n = 3 * n_pt + 6 * n_se3;
    g->b = (double *)calloc((size_t)g->n + 1, sizeof(double));
    g->x = (double *)calloc((size_t)g->n + 1, sizeof(double));
    blk_structure(g, B, se3_pos, nthreads);
  }
  t_setup = now_s() - t_start;
  const int P = n_pt, C = n_se3, n = g->n;
  double *bk_se3 = (double *)malloc(sizeof(double) * 12 * (size_t)(C > 0 ? C : 1));
  double *bk_pt = (double *)malloc(sizeof(double) * 3 * (size_t)(P > 0 ? P : 1));

  double lambda = -1, ni = 2; int nbad = 0; long trials = 0;
  int iters_done = 0, stop_flag = 0, ok = 1;
  double chi2_check = 0, last_chi_action = 0;
  if (chi2_hist) chi2_hist[0] = robust_chi2(g);
  for (int it = 0; it < max_iters && !stop_flag && ok; ++it) {
    /* ---- OptimizationAlgorithmLevenberg::solve ---- */
    double current = robust_chi2(g), temp = current, ini = current;
    double md = 0;
    if (solver == 0) {
      build_system(g);
      if (it == 0) for (int j = 0; j < n; ++j) { double d = fabs(g->Ax[g->Ap[j + 1] - 1]); if (d > md) md = d; }
    } else md = blk_build_system(g, B);
    if (it == 0) { lambda = 1e-5 * md; ni = 2; nbad = 0; }   /* computeLambdaInit: tau * max |H_jj| */
    double rho = 0; int qmax = 0, result_ok = 1;
    do {
      memcpy(bk_se3, g->se3, sizeof(double) * 12 * C); memcpy(bk_pt, g->pt, sizeof(double) * 3 * P);   /* push */
      double t0 = now_s();
      int ok2 = solver == 0 ? chol_solve(g, lambda) : blk_solve(g, B, lambda);
      t_lin += now_s() - t0;
      if (!ok2) memcpy(g->x, g->b, sizeof(double) * n);  /* linear_solver_csparse.h:124-126: x was pre-loaded with b and the failed factorisation leaves it there */
      apply_update(g);
      temp = robust_chi2(g);
      if (!ok2) temp = DBL_MAX;
      rho = current - temp;
      double scale = 0;
      for (int j = 0; j < n; ++j) scale += g->x[j] * (lambda * g->x[j] + g->b[j]);
      scale += 1e-3;
      rho /= scale;
      if (rho > 0 && isfinite(temp)) {
        double alpha = 1. - pow(2 * rho - 1, 3);
        if (alpha > 2. / 3.) alpha = 2. / 3.;
        double sf = alpha < 1. / 3. ? 1. / 3. : alpha;
        lambda *= sf; ni = 2; current = temp;         /* discardTop */
      } else {
        lambda *= ni; ni *= 2;
        memcpy(g->se3, bk_se3, sizeof(double) * 12 * C); memcpy(g->pt, bk_pt, sizeof(double) * 3 * P);  /* pop */
      }
      ++qmax; ++trials;
    } while (rho < 0 && qmax < 10 && !stop_flag);
    if (qmax == 10 || rho == 0) result_ok = 0;       /* Terminate */
    else {
      if ((ini - current) * 1e3 < ini) nbad++; else nbad = 0;
      if (nbad >= 3) result_ok = 0;
    }
    ok = result_ok;
    /* ---- back in SparseOptimizer::optimize ---- */
    double chi_now = robust_chi2(g);                 /* verbose: errors are at the current (restored) estimate */
    if (chi2_check < chi_now && it > 0) ok = 0;
    chi2_check = chi_now;
    if (chi2_hist) chi2_hist[it + 1] = chi_now;
    if (lam_hist) lam_hist[it] = lambda;
    if (t_hist) t_hist[it] = now_s() - t_start;
    if (verbose) fprintf(stderr, "[oracle] iteration= %d\t chi2= %.9g\t lambda= %.6g\t levenbergIter= %d\t t= %.1fs\n", it, chi_now, lambda, qmax, now_s() - t_start);
    ++iters_done;
    if (time_budget_s > 0 && now_s() - t_start > time_budget_s) break;    /* bench only: bounded sample of the solve */
    if (gain_threshold > 0) {                        /* postIteration: SparseOptimizerTerminateAction */
      if (it == 0) last_chi_action = chi_now;
      else {
        double gain = (last_chi_action - chi_now) / chi_now;
        last_chi_action = chi_now;
        if (gain >= 0 && gain < gain_threshold) stop_flag = 1;
      }
    }
  }
  if (stats) {
    stats[0] = lambda; stats[1] = (double)trials; stats[2] = (double)g->lnz; stats[3] = t_lin; stats[4] = now_s() - t_start; stats[5] = t_setup;
    if (solver != 0) { stats[2] = (double)B->toff[B->T] * BLK_NB * BLK_NB; stats[6] = B->t_schur; stats[7] = B->t_chol; }
  }
  free(bk_se3); free(bk_pt);
  if (solver == 0) ba_free(g); else { free(g->b); free(g->x); blk_free(B); }
  return iters_done;
}

int vdo_oracle_ba_optimize(int n_se3, double *se3, int n_pt, double *pt,
                           int n_prior, const int *prior_v, const double *prior_Z, const double *prior_w,
                           int n_se3e, const int *se3e_ij, const double *se3e_Z, const double *se3e_w, const double *se3e_delta,
                           int n_obs, const int *obs_cp, const double *obs_z, const double *obs_w, const double *obs_delta,
                           int n_ter, const int *ter_pph, const double *ter_w, const double *ter_delta,
                           int max_iters, double gain_threshold, int verbose, double *chi2_hist, double *stats) {
  return ba_optimize_impl(n_se3, se3, n_pt, pt, n_prior, prior_v, prior_Z, prior_w, n_se3e, se3e_ij, se3e_Z, se3e_w, se3e_delta,
                          n_obs, obs_cp, obs_z, obs_w, obs_delta, n_ter, ter_pph, ter_w, ter_delta,
                          max_iters, gain_threshold, verbose, chi2_hist, stats, 0, NULL, 1, NULL, 0.0, NULL);
}

/* Same LM, blocked linear solver (ba_block.h).  se3_pos[v] = position of se3 vertex v in the elimination order (NULL: identity);
 * nthreads <= 0: all;  lam_hist[i] = lambda after iteration i;  time_budget_s > 0 stops after the iteration that crosses it
 * (bench.py's bounded CPU sample); t_hist[i] = seconds since the call started when iteration i ended; stats[5..7] = setup / Schur /
 * band-Cholesky seconds. */
int vdo_oracle_ba_optimize_blocked(int n_se3, double *se3, int n_pt, double *pt,
                           int n_prior, const int *prior_v, const double *prior_Z, const double *prior_w,
                           int n_se3e, const int *se3e_ij, const double *se3e_Z, const double *se3e_w, const double *se3e_delta,
                           int n_obs, const int *obs_cp, const double *obs_z, const double *obs_w, const double *obs_delta,
                           int n_ter, const int *ter_pph, const double *ter_w, const double *ter_delta,
                           int max_iters, double gain_threshold, int verbose, double *chi2_hist, double *stats,
                           const int *se3_pos, int nthreads, double *lam_hist, double time_budget_s, double *t_hist) {
  return ba_optimize_impl(n_se3, se3, n_pt, pt, n_prior, prior_v, prior_Z, prior_w, n_se3e, se3e_ij, se3e_Z, se3e_w, se3e_delta,
                          n_obs, obs_cp, obs_z, obs_w, obs_delta, n_ter, ter_pph, ter_w, ter_delta,
                          max_iters, gain_threshold, verbose, chi2_hist, stats, 1, se3_pos, nthreads, lam_hist, time_budget_s, t_hist);
}

/* ---- small debugging / test entry points ---- */

/* dense H (n x n, symmetric, row-major) and b in the oracle's scalar order (points first, then se3), n = 3P+6C */
int vdo_oracle_ba_dense_system(int n_se3, double *se3, int n_pt, double *pt,
                               int n_prior, const int *prior_v, const double *prior_Z, const double *prior_w,
                               int n_se3e, const int *se3e_ij, const double *se3e_Z, const double *se3e_w, const double *se3e_delta,
                               int n_obs, const int *obs_cp, const double *obs_z, const double *obs_w, const double *obs_delta,
                               int n_ter, const int *ter_pph, const double *ter_w, const double *ter_delta,
                               double *H, double *b, double *chi2) {
  ba_t G; memset(&G, 0, sizeof G);
  ba_t *g = &G;
  g->n_se3 = n_se3; g->se3 = se3; g->n_pt = n_pt; g->pt = pt;
  g->n_prior = n_prior; g->prior_v = prior_v; g->prior_Z = prior_Z; g->prior_w = prior_w;
  g->n_se3e = n_se3e; g->se3e_ij = se3e_ij; g->se3e_Z = se3e_Z; g->se3e_w = se3e_w; g->se3e_delta = se3e_delta;
  g->n_obs = n_obs; g->obs_cp = obs_cp; g->obs_z = obs_z; g->obs_w = obs_w; g->obs_delta = obs_delta;
  g->n_ter = n_ter; g->ter_pph = ter_pph; g->ter_w = ter_w; g->ter_delta = ter_delta;
  build_structure(g);
  build_system(g);
  int n = g->n;
  memset(H, 0, sizeof(double) * (size_t)n * n);
  for (int j = 0; j < n; ++j)
    for (int64_t p = g->Ap[j]; p < g->Ap[j + 1]; ++p) { H[(size_t)g->Ai[p] * n + j] = g->Ax[p]; H[(size_t)j * n + g->Ai[p]] = g->Ax[p]; }
  memcpy(b, g->b, sizeof(double) * n);
  if (chi2) *chi2 = robust_chi2(g);
  /* solve once with lambda=0-ish check is done in python */
  free(g->Ap); free(g->Ai); free(g->Ax); free(g->pair_key); free(g->pair_off); free(g->diag_off);
  free(g->obs_pair); free(g->ter_pair); free(g->se3e_pair); free(g->b); free(g->x);
  return n;
}

/* the same H as a CSC upper triangle (column pointers Ap[n+1], row indices Ai[nnz], values Ax[nnz]; rows of a column are not sorted),
 * b (n) and the robust chi2, in the same scalar order.  Returns nnz; the arrays are written only when cap >= nnz, so a caller may
 * first ask for the size with cap = 0 (and NULL arrays). */
int64_t vdo_oracle_ba_sparse_system(int n_se3, double *se3, int n_pt, double *pt,
                                    int n_prior, const int *prior_v, const double *prior_Z, const double *prior_w,
                                    int n_se3e, const int *se3e_ij, const double *se3e_Z, const double *se3e_w, const double *se3e_delta,
                                    int n_obs, const int *obs_cp, const double *obs_z, const double *obs_w, const double *obs_delta,
                                    int n_ter, const int *ter_pph, const double *ter_w, const double *ter_delta,
                                    int64_t cap, int64_t *Ap, int *Ai, double *Ax, double *b, double *chi2) {
  ba_t G; memset(&G, 0, sizeof G);
  ba_t *g = &G;
  g->n_se3 = n_se3; g->se3 = se3; g->n_pt = n_pt; g->pt = pt;
  g->n_prior = n_prior; g->prior_v = prior_v; g->prior_Z = prior_Z; g->prior_w = prior_w;
  g->n_se3e = n_se3e; g->se3e_ij = se3e_ij; g->se3e_Z = se3e_Z; g->se3e_w = se3e_w; g->se3e_delta = se3e_delta;
  g->n_obs = n_obs; g->obs_cp = obs_cp; g->obs_z = obs_z; g->obs_w = obs_w; g->obs_delta = obs_delta;
  g->n_ter = n_ter; g->ter_pph = ter_pph; g->ter_w = ter_w; g->ter_delta = ter_delta;
  build_structure(g);
  const int64_t nnz = g->nnzA;
  if (cap >= nnz) {
    build_system(g);
    memcpy(Ap, g->Ap, sizeof(int64_t) * ((size_t)g->n + 1));
    memcpy(Ai, g->Ai, sizeof(int) * (size_t)nnz);
    memcpy(Ax, g->Ax, sizeof(double) * (size_t)nnz);
    memcpy(b, g->b, sizeof(double) * (size_t)g->n);
    if (chi2) *chi2 = robust_chi2(g);
  }
  free(g->Ap); free(g->Ai); free(g->Ax); free(g->pair_key); free(g->pair_off); free(g->diag_off);
  free(g->obs_pair); free(g->ter_pair); free(g->se3e_pair); free(g->b); free(g->x);
  return nnz;
}

/* raw edge functions for finite-difference tests: kind 0=prior 1=se3 2=obs 3=ternary */
void vdo_oracle_edge_eval(int kind, const double *a, const double *b, const double *c, double *err, double *Ja, double *Jb, double *Jc) {
  switch (kind) {
    case 0: edge_prior_error(a, b, err); edge_prior_jac(a, b, Ja); break;              /* a=Z b=X */
    case 1: edge_se3_error(a, b, c, err); edge_se3_jac(a, b, c, Ja, Jb); break;        /* a=Z b=Xi c=Xj */
    case 2: edge_obs_error(a, b, c, err); edge_obs_jac(a, b, Ja, Jb); break;           /* a=Xc b=p c=z */
    case 3: edge_ter_error(a, b, c, err); edge_ter_jac(b, c, Ja, Jb, Jc); break;       /* a=p1 b=p2 c=H */
  }
}
void vdo_oracle_iso_oplus(double *T, const double *upd) { iso_oplus(T, upd); }
void vdo_oracle_iso_from_Rt_via_quat(const double *R, const double *t, double *T) { iso_from_Rt_via_quat(R, t, T); }
