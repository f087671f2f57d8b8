// ba_tiles.cuh -- per-item bodies of the TILED batch-LM kernels (ba_types.h: Tile / Seg).
//
// One tile = a run of whole tracklets (<= VDO_TILE_L landmarks, <= VDO_TILE_E EdgeSE3PointXYZ) owned by one CTA.  A tile
// kernel is a fixed sequence of phases separated by CTA barriers; each phase is a loop over independent items (edges,
// landmarks, tracklets, or lanes of a vertex-sorted segment).  The phase bodies below are VDO_HD so that the CUDA kernels
// (ba_kernels.cu, threads strided over the items, fp64 atomics) and the serial emulation of the
// CPU-only host-logic tests (tests/emul, plain loops) run the same arithmetic on the same tile data structures.
//
// Everything the se3-vertex side needs is accumulated in the WORLD frame, so that no per-edge pose transform of the sums
// is needed and a tile touches each edge once:
//   EdgeSE3PointXYZ (g2o/types/edge_se3_pointxyz.cpp:99-140): with w = p - t_c, Zc = R_c^T w, e_w = R_c err = w - R_c z,
//       J_c = [-I | 2[Zc]x] = R_c^T [-I | 2[w]x] blockdiag(R_c, R_c)   =>   J_c^T J_c = B^T N^T N B,   J_c^T err = B^T N^T e_w
//   LandmarkMotionTernaryEdge (g2o/types/types_dyn_slam3d.cpp:53-85; the reference's Jacobian, without the factor 2):
//       with w' = p2 - t_H, q = R_H^T w', e' = R_H err:   J_H = [I | -[q]x] = R_H^T [I | -[w']x] blockdiag(R_H, R_H)
// The 16 sums  S0 = sum om, S1 = sum om w, S2 = sum om w w^T (6), G0 = sum om e, G1 = sum om w x e  per vertex are turned into
// the 6x6 block / 6-vector in the vertex' local frame by one small per-vertex kernel (tile_finalize_*).
#pragma once
#include "ba_math.cuh"
#include "ba_types.h"

namespace vdo {

// Tile-local views.  "view" members alias a contiguous range of a global array, element 0 = the tile's first landmark /
// edge / segment: in the CUDA kernels they point at shared-memory copies brought in by bulk async copies (TMA) at kernel
// start, in the emulation straight at the global arrays.  "stash" members are per-tile scratch written by the phases.
struct TileSm {
  // views
  double* P = 0;       // pt            3 / landmark
  double* S = 0;       // pt_s (Schur) or pt_g (preconditioner)   1 / landmark
  double* GAM = 0;     // tk_gamma      1 / landmark (preconditioner, chains)
  double* QS = 0;      // pt_Q          9 / landmark (chains)
  int* HH = 0;         // tk_h          motion vertex of edge (k, k+1) or -1
  uint8_t* TCLS = 0;   // tk_cls
  int* LB = 0;         // lm_obs_begin  nl + 1 entries, global edge indices
  int* CAM = 0;        // lm_cam        1 / edge
  uint8_t* LML = 0;    // lm_lml        1 / edge
  uint16_t* PERM = 0;  // ob_perm       1 / edge
  uint16_t* TPERM = 0; // tr_perm       1 / landmark
  const Seg* OSEG = 0; const Seg* TSEG = 0;   // the tile's segments
  double* OST = 0; double* TST = 0;           // translation of each segment's vertex (3 / segment), or null
  // views in the Schur / preconditioner kernels, stashes in the linearisation
  double* OM = 0;      // lm_omega      1 / edge
  double* OMT = 0;     // tk_omega      1 / landmark
  // stashes
  double* EW = 0;      // 3 / edge      lin: e_w ; schur (static): the edge's term of Hlp v
  double* Z = 0;       // 3 / landmark  schur: world-frame z (chains: g-hat first)
  double* Y = 0;       // 3 / landmark  chains: y-hat / z-hat
  double* IS = 0;      // 1 / landmark  1 / pivot
  double* TC = 0;      // 4 / landmark  lin chains: (omega, omega e') handed to landmark k+1
  double* E2 = 0;      // 3 / landmark  lin chains: e' of edge (k, k+1)
};
// emulation / reference wiring of the views straight onto the global arrays
inline void tile_views_global(const BaDev& d, const Tile& tl, bool precond, TileSm& sm) {
  sm.P = d.pt + 3 * (size_t)tl.k0; sm.S = (precond ? d.pt_g : d.pt_s) + tl.k0; sm.GAM = d.tk_gamma + tl.k0;
  sm.QS = d.pt_Q ? d.pt_Q + 9 * ((ptrdiff_t)tl.k0 - d.Tstat) : nullptr;
  sm.HH = d.tk_h + tl.k0; sm.TCLS = d.tk_cls + tl.k0; sm.LB = d.lm_obs_begin + tl.k0;
  sm.CAM = d.lm_cam + tl.e0; sm.LML = d.lm_lml + tl.e0; sm.PERM = d.ob_perm + tl.e0; sm.TPERM = d.tr_perm + tl.k0;
  sm.OSEG = d.osegs + tl.os0; sm.TSEG = d.tsegs + tl.ts0; sm.OST = nullptr; sm.TST = nullptr;
  sm.OM = d.lm_omega + tl.e0; sm.OMT = d.tk_omega + tl.k0;
}

// sums [4 PART, 4 PART + 4) of the 16 (the CUDA kernel gives each part its own thread; a holds the part's four sums)
template <int PART>
VDO_HD void acc16_add_part(double* a, double om, const double* w, const double* e) {
  const double ox = om * w[0], oy = om * w[1], oz = om * w[2];
  if (PART == 0) { a[0] += om; a[1] += ox; a[2] += oy; a[3] += oz; }
  else if (PART == 1) { a[0] += ox * w[0]; a[1] += ox * w[1]; a[2] += ox * w[2]; a[3] += oy * w[1]; }
  else if (PART == 2) { a[0] += oy * w[2]; a[1] += oz * w[2]; a[2] += om * e[0]; a[3] += om * e[1]; }
  else { a[0] += om * e[2]; a[1] += oy * e[2] - oz * e[1]; a[2] += oz * e[0] - ox * e[2]; a[3] += ox * e[1] - oy * e[0]; }
}
VDO_HD void acc16_add(double* a, double om, const double* w, const double* e) {
  acc16_add_part<0>(a, om, w, e); acc16_add_part<1>(a + 4, om, w, e); acc16_add_part<2>(a + 8, om, w, e); acc16_add_part<3>(a + 12, om, w, e);
}
VDO_HD void acc10_add(double* a, double om, const double* w) {
  a[0] += om;
  const double ox = om * w[0], oy = om * w[1], oz = om * w[2];
  a[1] += ox; a[2] += oy; a[3] += oz;
  a[4] += ox * w[0]; a[5] += ox * w[1]; a[6] += ox * w[2]; a[7] += oy * w[1]; a[8] += oy * w[2]; a[9] += oz * w[2];
}

// ---------------------------------------------------------------------------------------------------------------
// linearisation
// ---------------------------------------------------------------------------------------------------------------
// one EdgeSE3PointXYZ (tile-local index i) seen from camera pose T: robust chi2; with WRITE the robustified weight (global + stash) and e_w
template <bool WRITE>
VDO_HD double tile_lin_edge_at(const BaDev& d, const Tile& tl, int i, int lml, const double* T, TileSm& sm) {
  const size_t e = (size_t)tl.e0 + i;
  const double* z = d.lm_z + 3 * e;
  const double w[3] = {sm.P[3 * lml] - T[9], sm.P[3 * lml + 1] - T[10], sm.P[3 * lml + 2] - T[11]};
  double Rz[3]; rot_apply(T, z, Rz);
  const double ew[3] = {w[0] - Rz[0], w[1] - Rz[1], w[2] - Rz[2]};
  const int cls = d.lm_cls[e];
  const double wi = d.obs_cls_w[cls];
  double rho, hw; huber(wi * (ew[0] * ew[0] + ew[1] * ew[1] + ew[2] * ew[2]), d.obs_cls_d[cls], rho, hw);
  if (WRITE) {
    const double om = wi * hw;
    d.lm_omega[e] = om;
    sm.OM[i] = om; sm.EW[3 * i] = ew[0]; sm.EW[3 * i + 1] = ew[1]; sm.EW[3 * i + 2] = ew[2];
  }
  return rho;
}
template <bool WRITE>
VDO_HD double tile_lin_edge(const BaDev& d, const Tile& tl, int i, int lml, TileSm& sm) { return tile_lin_edge_at<WRITE>(d, tl, i, lml, d.se3 + 12 * (size_t)sm.CAM[i], sm); }
// landmark sums of the pointxyz edges of landmark j (tile-local): hll part and b_l part
VDO_HD void tile_lin_landmark_obs(const BaDev& d, const Tile& tl, int j, const TileSm& sm, double& dsum, double* b) {
  const int ib = sm.LB[j] - tl.e0, ie = sm.LB[j + 1] - tl.e0;
  for (int i = ib; i < ie; ++i) {
    const double om = sm.OM[i];
    dsum += om;
    b[0] -= om * sm.EW[3 * i]; b[1] -= om * sm.EW[3 * i + 1]; b[2] -= om * sm.EW[3 * i + 2];
  }
}
// ternary edge (k, k+1) of landmark j (chains) with motion pose H (nullptr: no such edge): chi2; with WRITE omega -> tk_omega, stash for
// landmark k+1 and for the scatter; adds the edge's contribution to landmark k's own sums
template <bool WRITE>
VDO_HD double tile_lin_ternary_at(const BaDev& d, const Tile& tl, int j, const double* H, TileSm& sm, double& dsum, double* b) {
  const int k = tl.k0 + j;
  if (!H) {
    if (WRITE) { d.tk_omega[k] = 0.0; sm.TC[4 * j] = sm.TC[4 * j + 1] = sm.TC[4 * j + 2] = sm.TC[4 * j + 3] = 0.0; sm.OMT[j] = 0.0; }
    return 0.0;
  }
  const double w[3] = {sm.P[3 * j + 3] - H[9], sm.P[3 * j + 4] - H[10], sm.P[3 * j + 5] - H[11]};
  double q[3]; rot_t_apply(H, w, q);
  const double err[3] = {sm.P[3 * j] - q[0], sm.P[3 * j + 1] - q[1], sm.P[3 * j + 2] - q[2]};
  const int cls = sm.TCLS[j];
  const double wi = d.ter_cls_w[cls];
  double rho, hw; huber(wi * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]), d.ter_cls_d[cls], rho, hw);
  if (WRITE) {
    const double om = wi * hw;
    d.tk_omega[k] = om;
    dsum += om;
    b[0] -= om * err[0]; b[1] -= om * err[1]; b[2] -= om * err[2];
    double Re[3]; rot_apply(H, err, Re);
    sm.TC[4 * j] = om; sm.TC[4 * j + 1] = om * Re[0]; sm.TC[4 * j + 2] = om * Re[1]; sm.TC[4 * j + 3] = om * Re[2];
    sm.E2[3 * j] = Re[0]; sm.E2[3 * j + 1] = Re[1]; sm.E2[3 * j + 2] = Re[2];
    sm.OMT[j] = om;
  }
  return rho;
}
template <bool WRITE>
VDO_HD double tile_lin_ternary(const BaDev& d, const Tile& tl, int j, TileSm& sm, double& dsum, double* b) {
  const int h = sm.HH[j];
  return tile_lin_ternary_at<WRITE>(d, tl, j, h >= 0 ? d.se3 + 12 * (size_t)h : nullptr, sm, dsum, b);
}
// one step of the chain rotations: Q := Q R^T (row r of the product needs only row r of Q)
VDO_HD void chain_Q_step(double* Q, const double* R) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double q0 = Q[3 * r], q1 = Q[3 * r + 1], q2 = Q[3 * r + 2];
#pragma unroll
    for (int c = 0; c < 3; ++c) Q[3 * r + c] = q0 * R[3 * c] + q1 * R[3 * c + 1] + q2 * R[3 * c + 2];
  }
}
// Q_k along one tracklet (tile-local tracklet jt): Q_kb = I, Q_{k+1} = Q_k R_k^T
VDO_HD void tile_chain_Q(const BaDev& d, const Tile& tl, int jt) {
  const int kb = d.tk_begin[tl.t0 + jt], ke = d.tk_begin[tl.t0 + jt + 1];
  double Q[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int k = kb; k < ke; ++k) {
    double* o = d.pt_Q + 9 * (size_t)(k - d.Tstat);
#pragma unroll
    for (int i = 0; i < 9; ++i) o[i] = Q[i];
    const int h = d.tk_h[k];
    if (h >= 0 && k + 1 < ke) chain_Q_step(Q, d.se3 + 12 * (size_t)h);
  }
}
// one lane of a pointxyz segment: world-frame sums for vertex sg.v   (linearisation: 16 sums)
VDO_HD void tile_lin_oseg_item(const BaDev& d, const Tile& tl, const Seg& sg, int l, const TileSm& sm, const double* t, double* acc) {
  const int i = sm.PERM[sg.begin - tl.e0 + l];
  const int j = sm.LML[i];
  const double w[3] = {sm.P[3 * j] - t[0], sm.P[3 * j + 1] - t[1], sm.P[3 * j + 2] - t[2]};
  acc16_add(acc, sm.OM[i], w, sm.EW + 3 * i);
}
VDO_HD void tile_lin_tseg_item(const BaDev& d, const Tile& tl, const Seg& sg, int l, const TileSm& sm, const double* t, double* acc) {
  const int j = sm.TPERM[sg.begin - tl.k0 + l];
  const double w[3] = {sm.P[3 * j + 3] - t[0], sm.P[3 * j + 4] - t[1], sm.P[3 * j + 5] - t[2]};
  acc16_add(acc, sm.OMT[j], w, sm.E2 + 3 * j);
}
// preconditioner: diagonal blocks of Hpl Hll^-1 Hlp seen from the vertex (10 sums, weight omega^2 * (Hll^-1 scalar))
VDO_HD void tile_pre_oseg_item(const BaDev& d, const Tile& tl, const Seg& sg, int l, const TileSm& sm, const double* t, double* acc) {
  const int i = sm.PERM[sg.begin - tl.e0 + l];
  const int j = sm.LML[i];
  const double om = sm.OM[i];
  const double w[3] = {sm.P[3 * j] - t[0], sm.P[3 * j + 1] - t[1], sm.P[3 * j + 2] - t[2]};
  acc10_add(acc, om * om * sm.S[j], w);            // S views pt_g here
}
VDO_HD void tile_pre_tseg_item(const BaDev& d, const Tile& tl, const Seg& sg, int l, const TileSm& sm, const double* t, double* acc) {
  const int j = sm.TPERM[sg.begin - tl.k0 + l];
  const double om = sm.OMT[j];
  const double w[3] = {sm.P[3 * j + 3] - t[0], sm.P[3 * j + 4] - t[1], sm.P[3 * j + 5] - t[2]};
  acc10_add(acc, om * om * sm.GAM[j], w);
}

// per-vertex conversion of the world-frame sums into the vertex' local frame.
//   kind 0 (pointxyz): M = [[S0 I, -2[S1]x],[.., 4(tr(S2) I - S2)]], g = [G0 ; 2 G1]
//   kind 1 (ternary) : M = [[S0 I,  -[S1]x],[..,   tr(S2) I - S2 ]], g = -[G0 ; G1]
// H36 += sgn * B^T M B (full row-major 6x6), g6 += B^T g   (B = blockdiag(R, R), so blocks are R^T X R)
VDO_HD void tile_acc_to_local(const double* a, int kind, const double* R, double sgn, double* H36, double* g6) {
  const double c1 = kind == 0 ? 2.0 : 1.0, c2 = kind == 0 ? 4.0 : 1.0;
  const double tr = a[4] + a[7] + a[9];
  // world-frame blocks
  const double TR[9] = {0, c1 * a[3], -c1 * a[2], -c1 * a[3], 0, c1 * a[1], c1 * a[2], -c1 * a[1], 0};      // -c1 [S1]x
  const double BR[9] = {c2 * (tr - a[4]), -c2 * a[5], -c2 * a[6], -c2 * a[5], c2 * (tr - a[7]), -c2 * a[8], -c2 * a[6], -c2 * a[8], c2 * (tr - a[9])};
  double X[9], Y[9];
  // R^T X R for X = TR, BR   (R^T I R = I for the top-left block)
  auto rtxr = [&](const double* Xw, double* out) {
    double Tm[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) Tm[3 * r + c] = Xw[3 * r] * R[c] + Xw[3 * r + 1] * R[3 + c] + Xw[3 * r + 2] * R[6 + c];       // X R
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) out[3 * r + c] = R[r] * Tm[c] + R[3 + r] * Tm[3 + c] + R[6 + r] * Tm[6 + c];                 // R^T (X R)
  };
  rtxr(TR, X); rtxr(BR, Y);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    H36[6 * r + r] += sgn * a[0];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      H36[6 * r + 3 + c] += sgn * X[3 * r + c];
      H36[6 * (3 + c) + r] += sgn * X[3 * r + c];
      H36[6 * (3 + r) + 3 + c] += sgn * Y[3 * r + c];
    }
  }
  if (g6) {
    const double s = kind == 0 ? 1.0 : -1.0;
    const double g0[3] = {s * a[10], s * a[11], s * a[12]}, g1[3] = {s * c1 * a[13], s * c1 * a[14], s * c1 * a[15]};
    double o0[3], o1[3];
    rot_t_apply(R, g0, o0); rot_t_apply(R, g1, o1);
    g6[0] += o0[0]; g6[1] += o0[1]; g6[2] += o0[2]; g6[3] += o1[0]; g6[4] += o1[1]; g6[5] += o1[2];
  }
}
// per vertex, after the tile kernels of one linearisation: Hpp += , bp += ; clears the accumulators
VDO_HD void tile_finalize_lin(const BaDev& d, int v) {
  const double* R = d.se3 + 12 * (size_t)v;
  double* ao = d.accO + 16 * (size_t)v; double* at = d.accT + 16 * (size_t)v;
  double H[36], g[6];
#pragma unroll
  for (int i = 0; i < 36; ++i) H[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) g[i] = 0.0;
  tile_acc_to_local(ao, 0, R, 1.0, H, g);
  if (at[0] != 0.0) tile_acc_to_local(at, 1, R, 1.0, H, g);
#pragma unroll
  for (int i = 0; i < 36; ++i) d.Hpp[36 * (size_t)v + i] += H[i];
#pragma unroll
  for (int i = 0; i < 6; ++i) d.bp[6 * (size_t)v + i] += g[i];
#pragma unroll
  for (int i = 0; i < 16; ++i) { ao[i] = 0.0; at[i] = 0.0; }
}
VDO_HD void tile_finalize_precond(const BaDev& d, int v) {
  const double* R = d.se3 + 12 * (size_t)v;
  double* ao = d.accO + 16 * (size_t)v; double* at = d.accT + 16 * (size_t)v;
  double H[36];
#pragma unroll
  for (int i = 0; i < 36; ++i) H[i] = 0.0;
  tile_acc_to_local(ao, 0, R, -1.0, H, nullptr);
  if (at[0] != 0.0) tile_acc_to_local(at, 1, R, -1.0, H, nullptr);
#pragma unroll
  for (int i = 0; i < 36; ++i) d.Minv[36 * (size_t)v + i] += H[i];
#pragma unroll
  for (int i = 0; i < 10; ++i) { ao[i] = 0.0; at[i] = 0.0; }
}
// out_v += sign * B^T acc6_v ; clears acc6_v
VDO_HD void tile_finalize_schur(const BaDev& d, int v, double sign, double* __restrict__ out) {
  const double* R = d.se3 + 12 * (size_t)v;
  double* a = d.acc6 + 6 * (size_t)v;
  double o0[3], o1[3];
  rot_t_apply(R, a, o0); rot_t_apply(R, a + 3, o1);
  double* o = out + 6 * (size_t)v;
  o[0] += sign * o0[0]; o[1] += sign * o0[1]; o[2] += sign * o0[2]; o[3] += sign * o1[0]; o[4] += sign * o1[1]; o[5] += sign * o1[2];
#pragma unroll
  for (int i = 0; i < 6; ++i) a[i] = 0.0;
}
// (the per-vertex world-frame images vw / vh of the vector a Schur product multiplies are written by body_vertex_transform,
//  ba_bodies.cuh:  pointxyz  Hlp,e v = omega (gamma + 2 p x beta), vw = [-R vt - 2 t x beta, beta = R vr];
//                  ternary   R_H (J_H v) = gamma' - p2 x beta,    vh = [ R vt +   t x beta, beta])

// ---------------------------------------------------------------------------------------------------------------
// Schur products.  mode 0: z = Hll^-1 bl ; mode 1: z = Hll^-1 (Hlp v) ; mode 2: xl = Hll^-1 (bl - Hlp v) (written to d.xl).
// Modes 0 and 1 do not write z: the tile scatters Hpl z into acc6 straight from shared memory.
// ---------------------------------------------------------------------------------------------------------------
// static tiles, per edge (mode != 0): the edge's term of Hlp v
template <int MODE>
VDO_HD void tile_schur_edge(const BaDev& d, const Tile& tl, int i, TileSm& sm) {
  if (MODE != 0) {
    const int lml = sm.LML[i];
    const double om = sm.OM[i];
    const double* w = d.vw + 6 * (size_t)sm.CAM[i];
    double pxb[3]; cross3(sm.P + 3 * lml, w + 3, pxb);
    sm.EW[3 * i] = om * (w[0] + 2 * pxb[0]); sm.EW[3 * i + 1] = om * (w[1] + 2 * pxb[1]); sm.EW[3 * i + 2] = om * (w[2] + 2 * pxb[2]);
  }
}
template <int MODE>
VDO_HD void tile_schur_static_landmark(const BaDev& d, const Tile& tl, int j, TileSm& sm) {
  const int k = tl.k0 + j;
  double u[3] = {0, 0, 0};
  if (MODE != 0) {
    const int ib = sm.LB[j] - tl.e0, ie = sm.LB[j + 1] - tl.e0;
    for (int i = ib; i < ie; ++i) { u[0] += sm.EW[3 * i]; u[1] += sm.EW[3 * i + 1]; u[2] += sm.EW[3 * i + 2]; }
  }
  double y[3];
  if (MODE == 1) { y[0] = u[0]; y[1] = u[1]; y[2] = u[2]; }
  else {
    const double* b = d.bl + 3 * (size_t)k;
    y[0] = b[0] - u[0]; y[1] = b[1] - u[1]; y[2] = b[2] - u[2];
  }
  const double is = 1.0 / sm.S[j];
  if (MODE == 2) { double* o = d.xl + 3 * (size_t)k; o[0] = y[0] * is; o[1] = y[1] * is; o[2] = y[2] * is; }
  else { sm.Z[3 * j] = y[0] * is; sm.Z[3 * j + 1] = y[1] * is; sm.Z[3 * j + 2] = y[2] * is; }
}
// one lane of a pointxyz segment: acc6 += -omega [z ; 2 w x z]
VDO_HD void tile_schur_oseg_item(const BaDev& d, const Tile& tl, const Seg& sg, int l, const TileSm& sm, const double* t, double* acc) {
  const int i = sm.PERM[sg.begin - tl.e0 + l];
  const int j = sm.LML[i];
  const double om = sm.OM[i];
  const double* z = sm.Z + 3 * j;
  const double w[3] = {sm.P[3 * j] - t[0], sm.P[3 * j + 1] - t[1], sm.P[3 * j + 2] - t[2]};
  double c[3]; cross3(w, z, c);
  acc[0] -= om * z[0]; acc[1] -= om * z[1]; acc[2] -= om * z[2];
  acc[3] -= 2 * om * c[0]; acc[4] -= 2 * om * c[1]; acc[5] -= 2 * om * c[2];
}
// chains, phase 1 per landmark: 1 / pivot; u-hat without the outgoing ternary term; g-hat of the incoming edge into sm.Z
template <int MODE>
VDO_HD void tile_schur_chain_u(const BaDev& d, const Tile& tl, int j, TileSm& sm) {
  const double* p = sm.P + 3 * j;
  const double* Q = sm.QS + 9 * j;
  sm.IS[j] = 1.0 / sm.S[j];
  double uh[3] = {0, 0, 0}, gh[3] = {0, 0, 0};
  if (MODE != 0) {
    double u[3] = {0, 0, 0};
    const int ib = sm.LB[j] - tl.e0, ie = sm.LB[j + 1] - tl.e0;
    for (int i = ib; i < ie; ++i) {
      const double om = sm.OM[i];
      const double* w = d.vw + 6 * (size_t)sm.CAM[i];
      double pxb[3]; cross3(p, w + 3, pxb);
      u[0] += om * (w[0] + 2 * pxb[0]); u[1] += om * (w[1] + 2 * pxb[1]); u[2] += om * (w[2] + 2 * pxb[2]);
    }
    rot_apply(Q, u, uh);
    const int hp = j > 0 ? sm.HH[j - 1] : -1;
    if (hp >= 0) {
      const double* w = d.vh + 6 * (size_t)hp;
      double pxb[3]; cross3(p, w + 3, pxb);
      const double g[3] = {w[0] - pxb[0], w[1] - pxb[1], w[2] - pxb[2]};
      rot_apply(Q, g, gh);
      const double om = sm.OMT[j - 1];
      uh[0] -= om * gh[0]; uh[1] -= om * gh[1]; uh[2] -= om * gh[2];
    }
  }
  sm.Z[3 * j] = gh[0]; sm.Z[3 * j + 1] = gh[1]; sm.Z[3 * j + 2] = gh[2];
  sm.Y[3 * j] = uh[0]; sm.Y[3 * j + 1] = uh[1]; sm.Y[3 * j + 2] = uh[2];
}
// chains, phase 2 per landmark: add the outgoing ternary term, form y-hat
template <int MODE>
VDO_HD void tile_schur_chain_y(const BaDev& d, const Tile& tl, int j, TileSm& sm) {
  const int k = tl.k0 + j;
  double uh[3] = {sm.Y[3 * j], sm.Y[3 * j + 1], sm.Y[3 * j + 2]};
  if (MODE != 0 && sm.HH[j] >= 0) {
    const double om = sm.OMT[j];
    uh[0] += om * sm.Z[3 * j + 3]; uh[1] += om * sm.Z[3 * j + 4]; uh[2] += om * sm.Z[3 * j + 5];
  }
  if (MODE != 1) {
    double bh[3]; rot_apply(sm.QS + 9 * j, d.bl + 3 * (size_t)k, bh);
    if (MODE == 0) { uh[0] = bh[0]; uh[1] = bh[1]; uh[2] = bh[2]; }
    else { uh[0] = bh[0] - uh[0]; uh[1] = bh[1] - uh[1]; uh[2] = bh[2] - uh[2]; }
  }
  sm.Y[3 * j] = uh[0]; sm.Y[3 * j + 1] = uh[1]; sm.Y[3 * j + 2] = uh[2];
}
// chains, phase 3 per tracklet: scalar forward / backward substitution in the rotated frame (three right-hand sides)
VDO_HD void tile_schur_chain_walk(const BaDev& d, const Tile& tl, int jt, TileSm& sm) {
  const int jb = d.tk_begin[tl.t0 + jt] - tl.k0, je = d.tk_begin[tl.t0 + jt + 1] - tl.k0;
  // forward: y_j = y_j + f_{j-1} y_{j-1}, f = omega / pivot.  The operands of step j + 1 are fetched before step j's FMAs so
  // that the recurrence costs one dependent FMA per step, not a shared-memory round trip.
  double y0 = sm.Y[3 * jb], y1 = sm.Y[3 * jb + 1], y2 = sm.Y[3 * jb + 2];
  double f = sm.OMT[jb] * sm.IS[jb];
  double n0 = 0, n1 = 0, n2 = 0;
  if (jb + 1 < je) { n0 = sm.Y[3 * jb + 3]; n1 = sm.Y[3 * jb + 4]; n2 = sm.Y[3 * jb + 5]; }
  for (int j = jb + 1; j < je; ++j) {
    const double c0 = n0, c1 = n1, c2 = n2, cf = f;
    f = sm.OMT[j] * sm.IS[j];
    if (j + 1 < je) { n0 = sm.Y[3 * j + 3]; n1 = sm.Y[3 * j + 4]; n2 = sm.Y[3 * j + 5]; }
    y0 = c0 + cf * y0; y1 = c1 + cf * y1; y2 = c2 + cf * y2;
    sm.Y[3 * j] = y0; sm.Y[3 * j + 1] = y1; sm.Y[3 * j + 2] = y2;
  }
  // backward: z_j = y_j / s_j + (omega_j / s_j) z_{j+1}
  double z0 = 0, z1 = 0, z2 = 0;
  double is = sm.IS[je - 1];
  double a0 = y0 * is, a1 = y1 * is, a2 = y2 * is, c = 0.0;   // last landmark: no successor (omega = 0)
  for (int j = je - 1; j >= jb; --j) {
    const double b0 = a0, b1 = a1, b2 = a2, bc = c;
    if (j > jb) {
      is = sm.IS[j - 1];
      a0 = sm.Y[3 * j - 3] * is; a1 = sm.Y[3 * j - 2] * is; a2 = sm.Y[3 * j - 1] * is; c = sm.OMT[j - 1] * is;
    }
    z0 = b0 + bc * z0; z1 = b1 + bc * z1; z2 = b2 + bc * z2;
    sm.Y[3 * j] = z0; sm.Y[3 * j + 1] = z1; sm.Y[3 * j + 2] = z2;
  }
}
// chains, phase 4 per landmark: back to the world frame
template <int MODE>
VDO_HD void tile_schur_chain_z(const BaDev& d, const Tile& tl, int j, TileSm& sm) {
  double z[3]; rot_t_apply(sm.QS + 9 * j, sm.Y + 3 * j, z);
  if (MODE == 2) { double* o = d.xl + 3 * (size_t)(tl.k0 + j); o[0] = z[0]; o[1] = z[1]; o[2] = z[2]; }
  else { sm.Z[3 * j] = z[0]; sm.Z[3 * j + 1] = z[1]; sm.Z[3 * j + 2] = z[2]; }
}
// one lane of a ternary segment: a' = R_H z_k - z_{k+1} = Q_{k+1}^T (zh_k - zh_{k+1});  acc6 += omega [a' ; w' x a']
VDO_HD void tile_schur_tseg_item(const BaDev& d, const Tile& tl, const Seg& sg, int l, const TileSm& sm, const double* t, double* acc) {
  const int j = sm.TPERM[sg.begin - tl.k0 + l];
  const double dz[3] = {sm.Y[3 * j] - sm.Y[3 * j + 3], sm.Y[3 * j + 1] - sm.Y[3 * j + 4], sm.Y[3 * j + 2] - sm.Y[3 * j + 5]};
  double a[3]; rot_t_apply(sm.QS + 9 * (j + 1), dz, a);
  const double w[3] = {sm.P[3 * j + 3] - t[0], sm.P[3 * j + 4] - t[1], sm.P[3 * j + 5] - t[2]};
  double c[3]; cross3(w, a, c);
  const double om = sm.OMT[j];
  acc[0] += om * a[0]; acc[1] += om * a[1]; acc[2] += om * a[2];
  acc[3] += om * c[0]; acc[4] += om * c[1]; acc[5] += om * c[2];
}

}  // namespace vdo
