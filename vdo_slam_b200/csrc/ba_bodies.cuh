// ba_bodies.cuh -- per-thread work items of the batch-LM kernels (one tracklet / one edge / one vertex).
// VDO_HD: the CUDA kernels in ba_kernels.cu wrap these with the parallel reductions; tests/emul runs them serially.
#pragma once
#include "ba_math.cuh"
#include "ba_types.h"

namespace vdo {

// ---------------------------------------------------------------------------------------------------------------
// Landmark side of the linearisation, one tracklet per call.  Returns the robust chi2 of the tracklet's
// EdgeSE3PointXYZ and LandmarkMotionTernaryEdge factors.  With write: robustified weights, H_ll diagonal (scalar
// per landmark: J_p^T J_p = R R^T = I for scalar information) and b_l.
// ---------------------------------------------------------------------------------------------------------------
VDO_HD double body_lin_tracklet(const BaDev& d, int t, bool write) {
  const int kb = d.tk_begin[t], ke = d.tk_begin[t + 1];
  double chi = 0.0, carry_d = 0.0, carry_b[3] = {0, 0, 0};
  double p[3] = {d.pt[3 * kb], d.pt[3 * kb + 1], d.pt[3 * kb + 2]};
  for (int k = kb; k < ke; ++k) {
    double dsum = carry_d, b[3] = {carry_b[0], carry_b[1], carry_b[2]};
    carry_d = 0; carry_b[0] = carry_b[1] = carry_b[2] = 0;
    const int eb = d.lm_obs_begin[k], ee = d.lm_obs_begin[k + 1];
    for (int e = eb; e < ee; ++e) {
      Iso T; iso_load(d.se3 + 12 * (size_t)d.lm_cam[e], T);
      double Zc[3]; iso_inv_apply(T, p, Zc);
      const double* z = d.lm_z + 3 * (size_t)e;
      double err[3] = {Zc[0] - z[0], Zc[1] - z[1], Zc[2] - z[2]};
      const int cls = d.lm_cls[e];
      const double w = d.obs_cls_w[cls];
      double rho, hw; huber(w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]), d.obs_cls_d[cls], rho, hw);
      chi += rho;
      if (write) {
        const double om = w * hw;
        d.lm_omega[e] = om;
        dsum += om;
        double Re[3]; rot_apply(T.R, err, Re);
        b[0] -= om * Re[0]; b[1] -= om * Re[1]; b[2] -= om * Re[2];
      }
    }
    const int h = d.tk_h[k];
    double pn[3] = {0, 0, 0};
    if (h >= 0) {
      pn[0] = d.pt[3 * (k + 1)]; pn[1] = d.pt[3 * (k + 1) + 1]; pn[2] = d.pt[3 * (k + 1) + 2];
      Iso H; iso_load(d.se3 + 12 * (size_t)h, H);
      double q[3]; iso_inv_apply(H, pn, q);
      double err[3] = {p[0] - q[0], p[1] - q[1], p[2] - q[2]};
      const int cls = d.tk_cls[k];
      const double w = d.ter_cls_w[cls];
      double rho, hw; huber(w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]), d.ter_cls_d[cls], rho, hw);
      chi += rho;
      if (write) {
        const double om = w * hw;
        d.tk_omega[k] = om;
        dsum += om;
        b[0] -= om * err[0]; b[1] -= om * err[1]; b[2] -= om * err[2];
        double Re[3]; rot_apply(H.R, err, Re);
        carry_d = om; carry_b[0] = om * Re[0]; carry_b[1] = om * Re[1]; carry_b[2] = om * Re[2];
      }
    } else if (write) {
      d.tk_omega[k] = 0.0;
    }
    if (write) {
      d.hll[k] = dsum;
      d.bl[3 * k] = b[0]; d.bl[3 * k + 1] = b[1]; d.bl[3 * k + 2] = b[2];
    }
    if (h >= 0) { p[0] = pn[0]; p[1] = pn[1]; p[2] = pn[2]; }
    else if (k + 1 < ke) { p[0] = d.pt[3 * (k + 1)]; p[1] = d.pt[3 * (k + 1) + 1]; p[2] = d.pt[3 * (k + 1) + 2]; }
  }
  return chi;
}

// ---- static landmarks (no ternary edges): one landmark per call, edge loop unrolled 2x/4x for memory-level parallelism ----
VDO_HD double body_lin_static(const BaDev& d, int k, bool write) {
  const double p[3] = {d.pt[3 * (size_t)k], d.pt[3 * (size_t)k + 1], d.pt[3 * (size_t)k + 2]};
  const int eb = d.lm_obs_begin[k], ee = d.lm_obs_begin[k + 1];
  double chi = 0.0, dsum = 0.0, b[3] = {0, 0, 0};
  for (int e0 = eb; e0 < ee; e0 += 2) {
    const bool two = e0 + 1 < ee;
    const int e1 = two ? e0 + 1 : e0;
    Iso T0, T1;
    iso_load(d.se3 + 12 * (size_t)d.lm_cam[e0], T0);
    iso_load(d.se3 + 12 * (size_t)d.lm_cam[e1], T1);
    const double* z0 = d.lm_z + 3 * (size_t)e0; const double* z1 = d.lm_z + 3 * (size_t)e1;
    const int c0 = d.lm_cls[e0], c1 = d.lm_cls[e1];
    double Z0[3], Z1[3];
    iso_inv_apply(T0, p, Z0); iso_inv_apply(T1, p, Z1);
    const double r0[3] = {Z0[0] - z0[0], Z0[1] - z0[1], Z0[2] - z0[2]};
    const double r1[3] = {Z1[0] - z1[0], Z1[1] - z1[1], Z1[2] - z1[2]};
    const double w0 = d.obs_cls_w[c0], w1 = d.obs_cls_w[c1];
    double rho0, h0, rho1, h1;
    huber(w0 * (r0[0] * r0[0] + r0[1] * r0[1] + r0[2] * r0[2]), d.obs_cls_d[c0], rho0, h0);
    huber(w1 * (r1[0] * r1[0] + r1[1] * r1[1] + r1[2] * r1[2]), d.obs_cls_d[c1], rho1, h1);
    chi += rho0;
    if (two) chi += rho1;
    if (write) {
      const double o0 = w0 * h0, o1 = two ? w1 * h1 : 0.0;
      d.lm_omega[e0] = o0;
      if (two) d.lm_omega[e1] = o1;
      double R0[3], R1[3];
      rot_apply(T0.R, r0, R0); rot_apply(T1.R, r1, R1);
      dsum += o0 + o1;
      b[0] -= o0 * R0[0] + o1 * R1[0]; b[1] -= o0 * R0[1] + o1 * R1[1]; b[2] -= o0 * R0[2] + o1 * R1[2];
    }
  }
  if (write) {
    d.tk_omega[k] = 0.0;
    d.hll[k] = dsum;
    d.bl[3 * (size_t)k] = b[0]; d.bl[3 * (size_t)k + 1] = b[1]; d.bl[3 * (size_t)k + 2] = b[2];
  }
  return chi;
}
VDO_HD void body_factor_static(const BaDev& d, int k, double lambda) {
  const double s = d.hll[k] + lambda;
  d.pt_s[k] = s; d.pt_g[k] = 1.0 / s; d.tk_gamma[k] = 0.0;
}
// mode 0: out = bl / s ; mode 1: out = (Hlp v) / s ; mode 2: out = (bl - Hlp v) / s   (v enters through d.vw)
VDO_HD void body_schur_static(const BaDev& d, int k, int mode, double* __restrict__ out) {
  double u[3] = {0, 0, 0};
  if (mode != 0) {
    const double p[3] = {d.pt[3 * (size_t)k], d.pt[3 * (size_t)k + 1], d.pt[3 * (size_t)k + 2]};
    const int eb = d.lm_obs_begin[k], ee = d.lm_obs_begin[k + 1];
    for (int e0 = eb; e0 < ee; e0 += 4) {
      int c[4]; double om[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool in = e0 + j < ee;
        c[j] = d.lm_cam[in ? e0 + j : e0];
        om[j] = in ? d.lm_omega[e0 + j] : 0.0;
      }
      double w[4][6];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double* ww = d.vw + 6 * (size_t)c[j];
#pragma unroll
        for (int i = 0; i < 6; ++i) w[j][i] = ww[i];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        double pxb[3]; cross3(p, &w[j][3], pxb);
        u[0] += om[j] * (w[j][0] + 2 * pxb[0]); u[1] += om[j] * (w[j][1] + 2 * pxb[1]); u[2] += om[j] * (w[j][2] + 2 * pxb[2]);
      }
    }
  }
  double y[3];
  if (mode == 0) { y[0] = d.bl[3 * (size_t)k]; y[1] = d.bl[3 * (size_t)k + 1]; y[2] = d.bl[3 * (size_t)k + 2]; }
  else if (mode == 1) { y[0] = u[0]; y[1] = u[1]; y[2] = u[2]; }
  else { y[0] = d.bl[3 * (size_t)k] - u[0]; y[1] = d.bl[3 * (size_t)k + 1] - u[1]; y[2] = d.bl[3 * (size_t)k + 2] - u[2]; }
  const double is = 1.0 / d.pt_s[k];
  out[3 * (size_t)k] = y[0] * is; out[3 * (size_t)k + 1] = y[1] * is; out[3 * (size_t)k + 2] = y[2] * is;
}

// Schur pivots of the tracklet's (H_ll + lambda I): with scalar diagonal blocks d_k I and off-diagonal blocks
// -omega_k R_k^T, the block recursion S_{k+1} = d_{k+1} I - omega_k^2 R_k S_k^-1 R_k^T stays a scalar times I, i.e.
// H_ll = Q (T (x) I3) Q^T with T the scalar tridiagonal (d_k, -omega_k) and Q block-diagonal orthogonal.
// Also emits the scalars of H_ll^-1 the preconditioner needs: g_k = (T^-1)_kk and, per ternary edge (k,k+1),
// gamma_k = g_k + g_{k+1} - 2 (T^-1)_{k,k+1}  (from the 2x2 system left after eliminating both sides).
VDO_HD void body_factor_tracklet(const BaDev& d, int t, double lambda) {
  const int kb = d.tk_begin[t], ke = d.tk_begin[t + 1];
  double s_prev = 1.0, om_prev = 0.0;
  for (int k = kb; k < ke; ++k) {
    double s = d.hll[k] + lambda - om_prev * om_prev / s_prev;
    d.pt_s[k] = s;
    s_prev = s; om_prev = d.tk_omega[k];
  }
  double t_next = 1.0;
  for (int k = ke - 1; k >= kb; --k) {
    const double dk = d.hll[k] + lambda, sk = d.pt_s[k];
    double tk = dk;
    if (k < ke - 1) {
      const double om = d.tk_omega[k];
      tk -= om * om / t_next;
      const double det = sk * t_next - om * om;
      d.tk_gamma[k] = (t_next + sk - 2.0 * om) / det;
    } else {
      d.tk_gamma[k] = 0.0;
    }
    d.pt_g[k] = 1.0 / (sk + tk - dk);
    t_next = tk;
  }
}

// World-frame image of an se3 increment v = [vt, vr] of vertex c, so that the EdgeSE3PointXYZ product needs no pose:
//   H_lp,e v_c = omega R_c J_c v_c = omega R_c(-vt + 2 Zc x vr) = omega (gamma + 2 p x beta),
//   beta = R_c vr,  gamma = -R_c vt - 2 t_c x beta          (R (a x b) = (R a) x (R b), R Zc = p - t_c)
VDO_HD void body_vertex_transform(const BaDev& d, int c, const double* __restrict__ v, double* __restrict__ vw) {
  const double* T = d.se3 + 12 * (size_t)c;
  double al[3], be[3], tb[3];
  rot_apply(T, v + 6 * (size_t)c, al);
  rot_apply(T, v + 6 * (size_t)c + 3, be);
  cross3(T + 9, be, tb);
  double* o = vw + 6 * (size_t)c;
  o[0] = -al[0] - 2 * tb[0]; o[1] = -al[1] - 2 * tb[1]; o[2] = -al[2] - 2 * tb[2];
  o[3] = be[0]; o[4] = be[1]; o[5] = be[2];
  if (d.vh) {   // tiled layout: image seen by the ternary edges, R_H (J_H v) = gamma' - p2 x beta with gamma' = R vt + t x beta
    double* oh = d.vh + 6 * (size_t)c;
    oh[0] = al[0] + tb[0]; oh[1] = al[1] + tb[1]; oh[2] = al[2] + tb[2]; oh[3] = be[0]; oh[4] = be[1]; oh[5] = be[2];
  }
}

// mode 0: out = Hll^-1 bl ; mode 1: out = Hll^-1 (Hlp v) ; mode 2: out = Hll^-1 (bl - Hlp v)
VDO_HD void body_schur_tracklet(const BaDev& d, int t, int mode, const double* __restrict__ v, double* __restrict__ out) {
  const int kb = d.tk_begin[t], ke = d.tk_begin[t + 1];
  double carry_u[3] = {0, 0, 0};
  double y_prev[3] = {0, 0, 0}, f_prev = 0.0, Rprev[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  double p[3] = {d.pt[3 * kb], d.pt[3 * kb + 1], d.pt[3 * kb + 2]};
  for (int k = kb; k < ke; ++k) {
    double u[3] = {carry_u[0], carry_u[1], carry_u[2]};
    carry_u[0] = carry_u[1] = carry_u[2] = 0;
    const int h = d.tk_h[k];
    double Rh[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double pn[3] = {0, 0, 0};
    if (mode != 0) {
      const int eb = d.lm_obs_begin[k], ee = d.lm_obs_begin[k + 1];
      for (int e = eb; e < ee; ++e) {
        const double* w = d.vw + 6 * (size_t)d.lm_cam[e];
        double pxb[3]; cross3(p, w + 3, pxb);
        const double om = d.lm_omega[e];
        u[0] += om * (w[0] + 2 * pxb[0]); u[1] += om * (w[1] + 2 * pxb[1]); u[2] += om * (w[2] + 2 * pxb[2]);
      }
    }
    if (h >= 0) {
      Iso H; iso_load(d.se3 + 12 * (size_t)h, H);
#pragma unroll
      for (int i = 0; i < 9; ++i) Rh[i] = H.R[i];
      pn[0] = d.pt[3 * (k + 1)]; pn[1] = d.pt[3 * (k + 1) + 1]; pn[2] = d.pt[3 * (k + 1) + 2];
      if (mode != 0) {
        double q[3]; iso_inv_apply(H, pn, q);
        double a[3]; ter_Jh_mul(q, v + 6 * (size_t)h, a);
        const double om = d.tk_omega[k];
        u[0] += om * a[0]; u[1] += om * a[1]; u[2] += om * a[2];
        double Ra[3]; rot_apply(H.R, a, Ra);
        carry_u[0] = -om * Ra[0]; carry_u[1] = -om * Ra[1]; carry_u[2] = -om * Ra[2];
      }
    }
    double y[3];
    if (mode == 0) { y[0] = d.bl[3 * k]; y[1] = d.bl[3 * k + 1]; y[2] = d.bl[3 * k + 2]; }
    else if (mode == 1) { y[0] = u[0]; y[1] = u[1]; y[2] = u[2]; }
    else { y[0] = d.bl[3 * k] - u[0]; y[1] = d.bl[3 * k + 1] - u[1]; y[2] = d.bl[3 * k + 2] - u[2]; }
    if (k > kb) {   // y_k += (omega_{k-1}/s_{k-1}) R_{k-1} y_{k-1}
      double Ry[3]; rot_apply(Rprev, y_prev, Ry);
      y[0] += f_prev * Ry[0]; y[1] += f_prev * Ry[1]; y[2] += f_prev * Ry[2];
    }
    if (ke - kb == 1) {   // static point: no chain, z = y / s
      const double is = 1.0 / d.pt_s[k];
      out[3 * k] = y[0] * is; out[3 * k + 1] = y[1] * is; out[3 * k + 2] = y[2] * is;
      return;
    }
    out[3 * k] = y[0]; out[3 * k + 1] = y[1]; out[3 * k + 2] = y[2];
    y_prev[0] = y[0]; y_prev[1] = y[1]; y_prev[2] = y[2];
    f_prev = d.tk_omega[k] / d.pt_s[k];
#pragma unroll
    for (int i = 0; i < 9; ++i) Rprev[i] = Rh[i];
    if (h >= 0) { p[0] = pn[0]; p[1] = pn[1]; p[2] = pn[2]; }
    else if (k + 1 < ke) { p[0] = d.pt[3 * (k + 1)]; p[1] = d.pt[3 * (k + 1) + 1]; p[2] = d.pt[3 * (k + 1) + 2]; }
  }
  // back substitution: z_k = (y_k + omega_k R_k^T z_{k+1}) / s_k
  double zn[3] = {0, 0, 0};
  for (int k = ke - 1; k >= kb; --k) {
    double y[3] = {out[3 * k], out[3 * k + 1], out[3 * k + 2]};
    if (k < ke - 1) {
      const int h = d.tk_h[k];
      if (h >= 0) {
        const double* R = d.se3 + 12 * (size_t)h;
        double Rt[3]; rot_t_apply(R, zn, Rt);
        const double om = d.tk_omega[k];
        y[0] += om * Rt[0]; y[1] += om * Rt[1]; y[2] += om * Rt[2];
      }
    }
    const double is = 1.0 / d.pt_s[k];
    zn[0] = y[0] * is; zn[1] = y[1] * is; zn[2] = y[2] * is;
    out[3 * k] = zn[0]; out[3 * k + 1] = zn[1]; out[3 * k + 2] = zn[2];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// se3-vertex side, one edge per call; the caller reduces A21/g6 (or acc6) over the chunk and adds to the vertex.
// ---------------------------------------------------------------------------------------------------------------
VDO_HD void body_lin_vertex_obs(const BaDev& d, const Iso& T, int e, double* A21, double* g6) {
  const double* p = d.pt + 3 * (size_t)d.vm_pt[e];
  double Zc[3]; iso_inv_apply(T, p, Zc);
  const double* z = d.vm_z + 3 * (size_t)e;
  double err[3] = {Zc[0] - z[0], Zc[1] - z[1], Zc[2] - z[2]};
  const int cls = d.vm_cls[e];
  const double w = d.obs_cls_w[cls];
  double rho, hw; huber(w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]), d.obs_cls_d[cls], rho, hw);
  const double om = w * hw;
  d.vm_omega[e] = om;
  obs_accumulate_pose(Zc, err, om, A21, g6);
}
VDO_HD void body_schur_vertex_obs(const BaDev& d, const Iso& T, int e, double* acc6) {
  const int k = d.vm_pt[e];
  const double* p = d.pt + 3 * (size_t)k;
  double Zc[3]; iso_inv_apply(T, p, Zc);
  double a[3]; rot_t_apply(T.R, d.zl + 3 * (size_t)k, a);
  double o[6]; obs_JcT_mul(Zc, a, o);
  const double om = d.vm_omega[e];
#pragma unroll
  for (int i = 0; i < 6; ++i) acc6[i] += om * o[i];
}
VDO_HD void body_lin_vertex_ter(const BaDev& d, const Iso& H, int e, double* A21, double* g6) {
  const int k = d.hm_p1[e];
  const double* p1 = d.pt + 3 * (size_t)k;
  double q[3]; iso_inv_apply(H, p1 + 3, q);
  double err[3] = {p1[0] - q[0], p1[1] - q[1], p1[2] - q[2]};
  const int cls = d.hm_cls[e];
  const double w = d.ter_cls_w[cls];
  double rho, hw; huber(w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]), d.ter_cls_d[cls], rho, hw);
  const double om = w * hw;
  d.hm_omega[e] = om;
  ter_accumulate_pose(q, err, om, A21, g6);
}
VDO_HD void body_schur_vertex_ter(const BaDev& d, const Iso& H, int e, double* acc6) {
  const int k = d.hm_p1[e];
  double q[3]; iso_inv_apply(H, d.pt + 3 * (size_t)(k + 1), q);
  double Rz[3]; rot_t_apply(H.R, d.zl + 3 * (size_t)(k + 1), Rz);
  const double* z1 = d.zl + 3 * (size_t)k;
  double a[3] = {z1[0] - Rz[0], z1[1] - Rz[1], z1[2] - Rz[2]};
  double o[6]; ter_JhT_mul(q, a, o);
  const double om = d.hm_omega[e];
#pragma unroll
  for (int i = 0; i < 6; ++i) acc6[i] += om * o[i];
}

// EdgeSE3 / EdgeSE3Prior, one edge per call.  Outputs: chi (robust), and with jac: Hi,Hj (36, J^T W J), Hoff (36,
// J_i^T W J_j), gi,gj (6, -J^T W e).  Returns false for a prior edge (j < 0: Hj/Hoff/gj untouched).
VDO_HD bool body_se3_edge(const BaDev& d, int e, bool jac, double& chi, double* Hi, double* Hj, double* Hoff, double* gi, double* gj) {
  const int i = d.se_i[e], j = d.se_j[e];
  Iso Z, Xi; iso_load(d.se_Z + 12 * (size_t)e, Z); iso_load(d.se3 + 12 * (size_t)i, Xi);
  double err[6], Ji[36], Jj[36];
  double w = d.se_w[e];
  if (j < 0) {
    edge_prior_eval(Z, Xi, err, Ji, jac);
    double e2 = 0; for (int k = 0; k < 6; ++k) e2 += err[k] * err[k];
    chi = w * e2;
  } else {
    Iso Xj; iso_load(d.se3 + 12 * (size_t)j, Xj);
    edge_se3_eval(Z, Xi, Xj, err, Ji, Jj, jac);
    double e2 = 0; for (int k = 0; k < 6; ++k) e2 += err[k] * err[k];
    double rho, hw; huber(w * e2, d.se_delta[e], rho, hw);
    chi = rho; w *= hw;
  }
  if (!jac) return j >= 0;
  for (int r = 0; r < 6; ++r) {
    double g = 0;
    for (int k = 0; k < 6; ++k) g += Ji[6 * k + r] * err[k];
    gi[r] = -w * g;
    for (int c = 0; c < 6; ++c) {
      double s = 0;
      for (int k = 0; k < 6; ++k) s += Ji[6 * k + r] * Ji[6 * k + c];
      Hi[6 * r + c] = w * s;
    }
  }
  if (j >= 0) {
    for (int r = 0; r < 6; ++r) {
      double g = 0;
      for (int k = 0; k < 6; ++k) g += Jj[6 * k + r] * err[k];
      gj[r] = -w * g;
      for (int c = 0; c < 6; ++c) {
        double s = 0, o = 0;
        for (int k = 0; k < 6; ++k) { s += Jj[6 * k + r] * Jj[6 * k + c]; o += Ji[6 * k + r] * Jj[6 * k + c]; }
        Hj[6 * r + c] = w * s;
        Hoff[6 * r + c] = w * o;
      }
    }
  }
  return j >= 0;
}

// out_v = (Hpp_vv + lambda I) x_v + sum over se3-se3 neighbours
VDO_HD void body_hpp_mul(const BaDev& d, int v, double lambda, const double* __restrict__ x, double* __restrict__ out) {
  const double* H = d.Hpp + 36 * (size_t)v;
  const double* xv = x + 6 * (size_t)v;
  double o[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    double s = lambda * xv[r];
#pragma unroll
    for (int c = 0; c < 6; ++c) s += H[6 * r + c] * xv[c];
    o[r] = s;
  }
  for (int n = d.nbr_begin[v]; n < d.nbr_begin[v + 1]; ++n) {
    const double* B = d.se_Hoff + 36 * (size_t)d.nbr_edge[n];
    const double* xo = x + 6 * (size_t)d.nbr_other[n];
    if (d.nbr_tr[n]) {
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = 0; c < 6; ++c) o[r] += B[6 * c + r] * xo[c];
    } else {
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = 0; c < 6; ++c) o[r] += B[6 * r + c] * xo[c];
    }
  }
#pragma unroll
  for (int r = 0; r < 6; ++r) out[6 * (size_t)v + r] = d.own ? o[r] : 0.0;   // sharded graphs: rank 0 contributes H_pp p, every rank its landmark terms
  body_vertex_transform(d, v, x, d.vw);
}

// Preconditioner pieces: diagonal block of Hpl Hll^-1 Hlp seen from the se3 vertex, per edge.
VDO_HD void body_precond_vertex_obs(const BaDev& d, const Iso& T, int e, double* A21) {
  const int k = d.vm_pt[e];
  double Zc[3]; iso_inv_apply(T, d.pt + 3 * (size_t)k, Zc);
  const double om = d.vm_omega[e];
  const double zero[3] = {0, 0, 0};
  double g[6] = {0, 0, 0, 0, 0, 0};
  obs_accumulate_pose(Zc, zero, om * om * d.pt_g[k], A21, g);
}
VDO_HD void body_precond_vertex_ter(const BaDev& d, const Iso& H, int e, double* A21) {
  const int k = d.hm_p1[e];
  double q[3]; iso_inv_apply(H, d.pt + 3 * (size_t)(k + 1), q);
  const double om = d.hm_omega[e];
  const double zero[3] = {0, 0, 0};
  double g[6] = {0, 0, 0, 0, 0, 0};
  ter_accumulate_pose(q, zero, om * om * d.tk_gamma[k], A21, g);
}
// ---- parallel cyclic reduction along a path [pb, pe) of the block-tridiagonal preconditioner (the serial emulation's restatement of
// the factorisation; the CUDA kernels reduce the same M by block cyclic reduction) ----
// level data: D[v] (6x6 SPD), L[v] = M(v, v - s) (zero when v - s < pb).  M(v, v + s) = L[v + s]^T.
VDO_HD void mat6_mul(const double* A, const double* B, double* C) {        // C = A B
  for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) { double s = 0; for (int k = 0; k < 6; ++k) s += A[6 * r + k] * B[6 * k + c]; C[6 * r + c] = s; }
}
VDO_HD void mat6_mul_nt(const double* A, const double* B, double* C) {     // C = A B^T
  for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) { double s = 0; for (int k = 0; k < 6; ++k) s += A[6 * r + k] * B[6 * c + k]; C[6 * r + c] = s; }
}
VDO_HD void mat6_mul_tn(const double* A, const double* B, double* C) {     // C = A^T B
  for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) { double s = 0; for (int k = 0; k < 6; ++k) s += A[6 * k + r] * B[6 * k + c]; C[6 * r + c] = s; }
}
// level-0 setup for vertex v: D = assembled diagonal block (in Minv), L = M(v, v-1) from the se3-se3 edge block
VDO_HD void body_pcr_setup(const BaDev& d, int v, double* D, double* L) {
  const double* S = d.Minv + 36 * (size_t)v;
  for (int i = 0; i < 36; ++i) D[36 * (size_t)v + i] = S[i];
  const int e = d.pcr_edge[v];
  double* Lv = L + 36 * (size_t)v;
  if (e < 0) { for (int i = 0; i < 36; ++i) Lv[i] = 0; return; }
  const double* B = d.se_Hoff + 36 * (size_t)e;
  if (d.pcr_tr[v]) { for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) Lv[6 * r + c] = B[6 * c + r]; }
  else { for (int i = 0; i < 36; ++i) Lv[i] = B[i]; }
}
VDO_HD void body_pcr_invert(const BaDev& d, int v, const double* D, double* Dinv, double lambda, int* bad) {
  double M[36];
  for (int i = 0; i < 36; ++i) M[i] = D[36 * (size_t)v + i];
  if (!spd6_inverse(M)) {
    for (int i = 0; i < 36; ++i) M[i] = 0;
    for (int i = 0; i < 6; ++i) M[7 * i] = 1.0 / (fabs(D[36 * (size_t)v + 7 * i]) + lambda);
    *bad = 1;
  }
  for (int i = 0; i < 36; ++i) Dinv[36 * (size_t)v + i] = M[i];
}
// One reduction step with stride s, split into two passes of (vertex, row, col) work items so that a whole cluster
// can share a chain:  pass 1  A_v = -L_v Dinv_{v-s},  G_v = -L_{v+s}^T Dinv_{v+s}   (zero outside the chain)
//                     pass 2  D'_v = D_v + A_v L_v^T + G_v L_{v+s},  L'_v = A_v L_{v-s}
VDO_HD void body_pcr_AG(int v, int r, int c, int pb, int pe, int s, const double* L, const double* Dinv, double* A, double* G) {
  double a = 0.0, g = 0.0;
  if (v - s >= pb) {
    const double* Lv = L + 36 * (size_t)v + 6 * r; const double* Di = Dinv + 36 * (size_t)(v - s) + c;
    a = -(Lv[0] * Di[0] + Lv[1] * Di[6] + Lv[2] * Di[12] + Lv[3] * Di[18] + Lv[4] * Di[24] + Lv[5] * Di[30]);
  }
  if (v + s < pe) {
    const double* Lp = L + 36 * (size_t)(v + s) + r; const double* Di = Dinv + 36 * (size_t)(v + s) + c;
    g = -(Lp[0] * Di[0] + Lp[6] * Di[6] + Lp[12] * Di[12] + Lp[18] * Di[18] + Lp[24] * Di[24] + Lp[30] * Di[30]);
  }
  A[36 * (size_t)v + 6 * r + c] = a; G[36 * (size_t)v + 6 * r + c] = g;
}
VDO_HD void body_pcr_DL(int v, int r, int c, int pb, int pe, int s, const double* D, const double* L, const double* A, const double* G,
                        double* Dn, double* Ln) {
  double dd = D[36 * (size_t)v + 6 * r + c], ll = 0.0;
  if (v - s >= pb) {
    const double* a = A + 36 * (size_t)v + 6 * r; const double* Lv = L + 36 * (size_t)v + 6 * c;
    dd += a[0] * Lv[0] + a[1] * Lv[1] + a[2] * Lv[2] + a[3] * Lv[3] + a[4] * Lv[4] + a[5] * Lv[5];
    if (v - 2 * s >= pb) {
      const double* Lm = L + 36 * (size_t)(v - s) + c;
      ll = a[0] * Lm[0] + a[1] * Lm[6] + a[2] * Lm[12] + a[3] * Lm[18] + a[4] * Lm[24] + a[5] * Lm[30];
    }
  }
  if (v + s < pe) {
    const double* g = G + 36 * (size_t)v + 6 * r; const double* Lp = L + 36 * (size_t)(v + s) + c;
    dd += g[0] * Lp[0] + g[1] * Lp[6] + g[2] * Lp[12] + g[3] * Lp[18] + g[4] * Lp[24] + g[5] * Lp[30];
  }
  Dn[36 * (size_t)v + 6 * r + c] = dd; Ln[36 * (size_t)v + 6 * r + c] = ll;
}
// solve phase, one level: bn_v = b_v + A_v b_{v-s} + G_v b_{v+s}
VDO_HD void body_pcr_apply(int v, int pb, int pe, int s, const double* A, const double* G, const double* b, double* bn) {
  double o[6];
  for (int i = 0; i < 6; ++i) o[i] = b[6 * (size_t)v + i];
  if (v - s >= pb) {
    const double* a = A + 36 * (size_t)v; const double* x = b + 6 * (size_t)(v - s);
    for (int r = 0; r < 6; ++r) { double t = 0; for (int c = 0; c < 6; ++c) t += a[6 * r + c] * x[c]; o[r] += t; }
  }
  if (v + s < pe) {
    const double* g = G + 36 * (size_t)v; const double* x = b + 6 * (size_t)(v + s);
    for (int r = 0; r < 6; ++r) { double t = 0; for (int c = 0; c < 6; ++c) t += g[6 * r + c] * x[c]; o[r] += t; }
  }
  for (int i = 0; i < 6; ++i) bn[6 * (size_t)v + i] = o[i];
}
VDO_HD int pcr_num_levels(int m) { int l = 0; while ((1 << l) < m) ++l; return l; }
VDO_HD void mul6(const double* M, const double* x, double* o) {
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    double s = 0;
#pragma unroll
    for (int c = 0; c < 6; ++c) s += M[6 * r + c] * x[c];
    o[r] = s;
  }
}

// vertex update; returns this vertex's part of computeScale() = sum_j x_j (lambda x_j + b_j)
VDO_HD double body_update_se3(const BaDev& d, int v, double lambda, bool reortho) {
  Iso T; iso_load(d.se3 + 12 * (size_t)v, T);
  const double* x = d.xp + 6 * (size_t)v;
  const double* b = d.bp + 6 * (size_t)v;
  iso_oplus(T, x);
  if (reortho) rot_reorthogonalize(T.R);
  iso_store(d.se3 + 12 * (size_t)v, T);
  double s = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i) s += x[i] * (lambda * x[i] + b[i]);
  return d.own ? s : 0.0;
}
VDO_HD double body_update_pt(const BaDev& d, int k, double lambda) {
  double s = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double x = d.xl[3 * (size_t)k + i];
    d.pt[3 * (size_t)k + i] += x;
    s += x * (lambda * x + d.bl[3 * (size_t)k + i]);
  }
  return s;
}

}  // namespace vdo
