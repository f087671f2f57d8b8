// cam_motion.cu -- the background half of Tracking::Track for P frame pairs on the device, from a carried background set
// (vdo_stat_feat_set): Frame::Frame's static set of a sequence's first frame (Frame.cc:100-194 and Initialization, Tracking.cc:1219-1227), the
// camera step (:672-713: GetInitModelCam :1614-1715 against the constant-velocity model, PoseOptimizationFlow2Cam, mVelocity) and the static
// half of RenewFrameInfo (:2663-2814).
//
// Launch of vdo_stat_build_batch_dev:
//   k_sb_build     one CTA per pair (a pair whose count is not -1 returns at once): the ordered compaction of the keys that pass
//                  frame_px.cuh's static_key
// Launches of vdo_cam_track_batch_dev:
//   k_ct_gather    one CTA per pair: the rows' world points and observations, the motion model, one PnpProb
//   k_pnp_samples / k_pnp_hyp / k_pnp_score / k_pnp_finish   pnp_ransac.cu's kernels, unchanged (dev_solvers.cuh launchers)
//   k_ct_lm_prep   one CTA per pair: a chosen set of at least 3 rows as the pair's FlowProb (mode 0)
//   k_refine_lm_cl / k_refine_lm   flow_lm.cu's kernels, unchanged
//   k_ct_finish    one CTA per pair: T, velocity, info and status; flags, current keys and refined flows per row
// Launch of vdo_stat_renew_batch_dev:
//   k_sr_select    one CTA per pair: the carried rows (a flag pass and an ordered compaction), then the top-up: the reference visits its list
//                  in passes of stride 20, so a candidate's rank is the number of kept candidates in earlier passes plus those before it in
//                  its own pass, counted per residue of the list index
// This file is compiled with --fmad=false: the back-projections, the 4x4 products and inverses (pose4.cuh) and the key updates then round
// as the tracker's host code rounds them.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"
#include "dev_solvers.cuh"
#include "frame_px.cuh"
#include "pose4.cuh"

namespace {
using vdo::FlowDev;
using vdo::FlowProb;
using vdo::PnpOut;
using vdo::PnpProb;

constexpr int CM_MAX_PAIRS = VDO_CAM_MOTION_MAX_PAIRS, CM_THREADS = 256, SR_THREADS = 1024, SR_STAGE = 2048, SR_PASSES = 20;

struct StatPair { PlaneArg dep, flo, msk; int w, h; float K[4]; };
struct StatArg {                // a call's host parameters, passed by value so that a captured call replays with them
  const float *kx, *ky;         // the key set: frame p at p * kcap
  const int *kcount, *gate;     // gate: option II's ORB counts, or NULL
  int kcap, C, max_bg, sampled;
  float th;
  StatPair pr[CM_MAX_PAIRS];
};

// a set row: key, depth, corres key + flow, flow, inlier id and point
__device__ __forceinline__ void put_row(const vdo_stat_feat_set& s, size_t i, float kx, float ky, float d, float fx, float fy, int id, const float* X) {
  s.x_dev[i] = kx; s.y_dev[i] = ky; s.depth_dev[i] = d; s.cx_dev[i] = __fadd_rn(kx, fx); s.cy_dev[i] = __fadd_rn(ky, fy);
  s.flow_dev[2 * i] = fx; s.flow_dev[2 * i + 1] = fy; s.inlier_id_dev[i] = id;
  for (int c = 0; c < 3; ++c) s.point_dev[3 * i + c] = X[c];
}
__device__ __forceinline__ int key_count(const StatArg& a, int p, int* status) {
  const int n = a.kcount[p];
  if (n < 0 || n > a.kcap) { *status |= VDO_CAM_KEY_COUNT; return 0; }
  return a.sampled && a.gate[p] <= 0 ? 0 : n;           // Frame.cc:97-98: a frame without ORB keypoints gets no static keys
}
// the build's rule (static_key on the pair's planes, th_depth_bg, the option's bounds) for a key whose pixel lies in the image
__device__ __forceinline__ bool build_key(const StatPair& q, float th, bool sampled, float px, float py, float& d, float& fx, float& fy) {
  const int x = (int)px, y = (int)py;
  if (!(x >= 0 && x < q.w && y >= 0 && y < q.h)) return false;
  return static_key(px, py, th, sampled, q.w, q.h, [&](int u, int v) { return plane_unlabelled(q.msk, u, v); }, [&](int u, int v) { return plane_depth(q.dep, u, v); },
                    [&](int u, int v, float& a, float& b) { const float2 f = plane_flow(q.flo, u, v); a = f.x; b = f.y; }, d, fx, fy);
}
// RenewFrameInfo's test of a carried row or a top-up candidate (:2680-2704, :2750-2777): 0 < (int)x < W, 0 < (int)y < H, then the option-II
// rule at the hard-coded depth bound 40
__device__ __forceinline__ bool renew_key(const StatPair& q, float px, float py, float& d, float& fx, float& fy) {
  const int x = (int)px, y = (int)py;
  if (x >= q.w || y >= q.h || x <= 0 || y <= 0) return false;
  return build_key(q, 40.f, true, px, py, d, fx, fy);
}

// ---- vdo_stat_build_batch_dev ----
__global__ void __launch_bounds__(SR_THREADS) k_sb_build(const __grid_constant__ StatArg a, vdo_stat_feat_set s) {
  __shared__ int wsum[33];
  const int p = blockIdx.x, tid = threadIdx.x;
  if (s.count_dev[p] != -1) return;                     // the same for the whole CTA
  const StatPair& q = a.pr[p];
  int status = 0;
  const int n = key_count(a, p, &status);
  const size_t koff = (size_t)p * a.kcap, off = (size_t)p * a.C;
  const float invfx = 1.0f / q.K[0], invfy = 1.0f / q.K[1];
  int base = 0;
  for (int start = 0; start < n; start += SR_THREADS) {
    const int j = start + tid;
    float px = 0.f, py = 0.f, d = 0.f, fx = 0.f, fy = 0.f;
    int ok = 0;
    if (j < n) { px = a.kx[koff + j]; py = a.ky[koff + j]; ok = build_key(q, a.th, a.sampled, px, py, d, fx, fy); }
    int tot;
    const int pos = base + cta_excl_scan(ok, wsum, tot);
    if (ok) {                                           // Optimizer::Get3DinCamera (tracker.cpp get3d_camera)
      const float X[3] = {(px - q.K[2]) * d * invfx, (py - q.K[3]) * d * invfy, d};
      put_row(s, off + pos, px, py, d > 0.f ? d : -1.f, fx, fy, -1, X);
    }
    base += tot;
    __syncthreads();
  }
  if (tid < 16) { s.Tcw_dev[16 * p + tid] = tid % 5 == 0 ? 1.f : 0.f; s.velocity_dev[16 * p + tid] = tid % 5 == 0 ? 1.f : 0.f; }
  if (tid == 0) { s.count_dev[p] = base; s.status_dev[p] = status; s.has_velocity_dev[p] = 0; }
}

// ---- vdo_cam_track_batch_dev ----
struct CamArg { int C; float K[CM_MAX_PAIRS][4]; };
__device__ __forceinline__ int set_rows(const vdo_stat_feat_set& s, int p, int C) { const int c = s.count_dev[p]; return c >= 0 && c <= C ? c : 0; }

// one CTA per pair: the rows' world points (UnprojectStereoStat through the set's Tcw) and observations (cx, cy), and the pair's problem
__global__ void __launch_bounds__(CM_THREADS) k_ct_gather(const __grid_constant__ CamArg a, vdo_stat_feat_set s, float* __restrict__ obj,
                                                          float* __restrict__ img, PnpProb* __restrict__ prob) {
  __shared__ float s_T[16];
  const int p = blockIdx.x, tid = threadIdx.x, n = set_rows(s, p, a.C);
  const size_t off = (size_t)p * a.C;
  if (tid < 16) s_T[tid] = s.Tcw_dev[16 * p + tid];
  __syncthreads();
  for (int k = tid; k < n; k += CM_THREADS) {
    const size_t i = off + k;
    unproject_world(s.x_dev[i], s.y_dev[i], s.depth_dev[i], a.K[p], s_T, obj + 3 * i);
    img[2 * i] = s.cx_dev[i]; img[2 * i + 1] = s.cy_dev[i];
  }
  if (tid == 0) {
    PnpProb pb;
    pb.off = (int)off; pb.n = n;
    for (int c = 0; c < 4; ++c) { pb.K[c] = (double)a.K[p][c]; pb.Kf[c] = a.K[p][c]; }
    float mm[16];                                       // the constant-velocity model (:1636-1640); the first pair's is Tcw itself
    if (s.has_velocity_dev[p]) mul4(s.velocity_dev + 16 * p, s_T, mm);
    else for (int c = 0; c < 16; ++c) mm[c] = s_T[c];
    for (int c = 0; c < 12; ++c) pb.mm[c] = mm[c];
    pb.has_mm = 1; pb.pad = 0;
    prob[p] = pb;
  }
}

__device__ __forceinline__ bool runs_lm(const PnpOut& r) { return r.n_sub >= 3; }   // tracker.cpp:299

// one CTA per pair: the chosen set's (x, y), depth and flow as the pair's LM problem from T_init (none below 3 rows)
__global__ void __launch_bounds__(CM_THREADS) k_ct_lm_prep(const __grid_constant__ CamArg a, vdo_stat_feat_set s, const PnpProb* __restrict__ prob,
                                                           const PnpOut* __restrict__ res, const int* __restrict__ s_idx, float* __restrict__ pts,
                                                           float* __restrict__ depth, float* __restrict__ flow, FlowProb* __restrict__ fprob) {
  const int p = blockIdx.x, tid = threadIdx.x;
  const PnpProb pr = prob[p];
  const PnpOut& r = res[p];
  const int n = runs_lm(r) ? r.n_sub : 0;
  for (int k = tid; k < n; k += CM_THREADS) {
    const size_t g = (size_t)pr.off + k, i = (size_t)pr.off + s_idx[g];
    pts[2 * g] = s.x_dev[i]; pts[2 * g + 1] = s.y_dev[i];
    depth[g] = s.depth_dev[i];
    flow[2 * g] = s.flow_dev[2 * i]; flow[2 * g + 1] = s.flow_dev[2 * i + 1];
  }
  if (tid == 0) {
    FlowProb fp;
    fp.mode = 0; fp.n = n; fp.offset = pr.off; fp.out = p;
    for (int c = 0; c < 4; ++c) fp.K[c] = a.K[p][c];
    for (int c = 0; c < 16; ++c) { fp.Tcw_last[c] = s.Tcw_dev[16 * p + c]; fp.T_init[c] = r.T[c]; }
    fprob[p] = fp;
  }
}

// one CTA per pair: per row the flags, the current key and the refined flow; per pair T, T_init, velocity, info and status
__global__ void __launch_bounds__(CM_THREADS) k_ct_finish(const __grid_constant__ CamArg a, vdo_stat_feat_set s, vdo_cam_track_out o,
                                                          const PnpProb* __restrict__ prob, const PnpOut* __restrict__ res, const int* __restrict__ s_idx,
                                                          const float* __restrict__ X, const double* __restrict__ flow_res, const unsigned char* __restrict__ inl) {
  const int p = blockIdx.x, tid = threadIdx.x;
  const PnpProb pr = prob[p];
  const PnpOut& r = res[p];
  const bool lm = runs_lm(r);
  for (int k = tid; k < pr.n; k += CM_THREADS) {
    const size_t i = (size_t)pr.off + k;
    o.flags_dev[i] = 0;
    o.key_dev[2 * i] = s.cx_dev[i]; o.key_dev[2 * i + 1] = s.cy_dev[i];            // mCurrentFrame.mvStatKeys = mLastFrame.mvCorres
    o.flow_ref_dev[2 * i] = (double)s.flow_dev[2 * i]; o.flow_ref_dev[2 * i + 1] = (double)s.flow_dev[2 * i + 1];
  }
  __syncthreads();
  for (int k = tid; k < r.n_sub; k += CM_THREADS) {
    const size_t g = (size_t)pr.off + k, i = (size_t)pr.off + s_idx[g];
    const bool in = lm && inl[g];
    o.flags_dev[i] = 1 | (in ? 2 : 0) | (!lm || in ? 4 : 0);
    if (lm) { o.flow_ref_dev[2 * i] = flow_res[2 * g]; o.flow_ref_dev[2 * i + 1] = flow_res[2 * g + 1]; }
    if (in) { o.key_dev[2 * i] = (float)((double)s.x_dev[i] + flow_res[2 * g]); o.key_dev[2 * i + 1] = (float)((double)s.y_dev[i] + flow_res[2 * g + 1]); }
  }
  if (tid == 0) {
    float T[16], Tl[16], Ti[16], V[16];
    for (int c = 0; c < 16; ++c) { T[c] = lm ? X[16 * p + c] : r.T[c]; Tl[c] = s.Tcw_dev[16 * p + c]; }
    inv4(Tl, Ti);
    mul4(T, Ti, V);                                     // mVelocity = mTcw * LastTwc (:700-706)
    for (int c = 0; c < 16; ++c) { o.T_dev[16 * p + c] = T[c]; o.T_init_dev[16 * p + c] = r.T[c]; o.velocity_dev[16 * p + c] = V[c]; }
    int* info = o.info_dev + 8 * p;
    info[0] = pr.n; info[1] = r.n_ransac; info[2] = r.n_mm; info[3] = r.used_mm; info[4] = r.n_sub; info[5] = r.iters_run; info[6] = r.best_it;
    info[7] = r.n_valid;
    const int c = s.count_dev[p];
    o.status_dev[p] = (pr.n < 4 ? VDO_CAM_FEW_POINTS : 0) | (pr.n >= 4 && r.best_it < 0 ? VDO_CAM_NO_MODEL : 0) | (r.used_mm ? VDO_CAM_USED_MM : 0) |
                      (c < 0 || c > a.C ? VDO_CAM_SET_COUNT : 0);
  }
}

// ---- vdo_stat_renew_batch_dev: one CTA per pair ----
__global__ void __launch_bounds__(SR_THREADS) k_sr_select(const __grid_constant__ StatArg a, vdo_stat_feat_set last, vdo_cam_track_out cam,
                                                          vdo_stat_feat_set s) {
  __shared__ int wsum[33];
  __shared__ float s_key[2 * SR_STAGE];
  __shared__ int s_w[SR_THREADS / 32][SR_PASSES], s_cnt[SR_PASSES], s_run[SR_PASSES], s_ctot[SR_PASSES];
  __shared__ float s_Twc[16];
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, C = a.C;
  const StatPair& q = a.pr[p];
  const size_t off = (size_t)p * C, koff = (size_t)p * a.kcap;
  const int lc = last.count_dev[p];
  int status = lc < -1 || lc > C || (cam.status_dev[p] & VDO_CAM_SET_COUNT) ? VDO_CAM_SET_COUNT : 0;
  const int n = status ? 0 : max(lc, 0);
  if (tid == 0) inv4(cam.T_dev + 16 * p, s_Twc);        // Converter::toInvMatrix(mTcw)
  if (tid < SR_PASSES) { s_cnt[tid] = 0; s_run[tid] = 0; }
  for (int k = tid; k < SR_THREADS / 32 * SR_PASSES; k += SR_THREADS) s_w[k / SR_PASSES][k % SR_PASSES] = 0;
  __syncthreads();
  // Optimizer::Get3DinWorld (tracking_ops.cu get3d_world's rounding)
  const float invfx = 1.0f / q.K[0], invfy = 1.0f / q.K[1];
  const auto put = [&](int pos, float kx, float ky, float d, float fx, float fy, int id) {
    const float x = (kx - q.K[2]) * d * invfx, y = (ky - q.K[3]) * d * invfy;
    float X[3];
    for (int c = 0; c < 3; ++c)
      X[c] = (float)((double)s_Twc[4 * c] * (double)x + (double)s_Twc[4 * c + 1] * (double)y + (double)s_Twc[4 * c + 2] * (double)d + (double)s_Twc[4 * c + 3]);
    put_row(s, off + pos, kx, ky, d, fx, fy, id, X);
  };
  // 1. the carried rows: the first max_bg + 1 rows of the subset that pass, in row order
  int base = 0;
  for (int start = 0; start < n && base <= a.max_bg; start += SR_THREADS) {
    const int i = start + tid;
    float kx = 0.f, ky = 0.f, d = 0.f, fx = 0.f, fy = 0.f;
    int ok = 0;
    if (i < n && (cam.flags_dev[off + i] & 4)) { kx = cam.key_dev[2 * (off + i)]; ky = cam.key_dev[2 * (off + i) + 1]; ok = renew_key(q, kx, ky, d, fx, fy); }
    int tot;
    const int pos = base + cta_excl_scan(ok, wsum, tot);
    if (ok && pos <= a.max_bg) put(pos, kx, ky, d, fx, fy, i);
    base += tot;
    __syncthreads();
  }
  const int ns = min(base, a.max_bg + 1), need = ns < a.max_bg ? a.max_bg - ns : 0;
  // 2. the top-up: two passes over the list, the first counting the kept candidates per residue, the second placing them by rank
  int added = 0;
  const int nk = need ? key_count(a, p, &status) : 0;
  for (int phase = 0; phase < 2 && nk; ++phase) {
    int fbase = 0;
    for (int start = 0; start < nk; start += SR_THREADS) {
      const int j = start + tid;
      float kx = 0.f, ky = 0.f, d = 0.f, fx = 0.f, fy = 0.f;
      int listed = 0;
      if (j < nk) {
        kx = a.kx[koff + j]; ky = a.ky[koff + j];
        listed = !a.sampled || build_key(q, a.th, true, kx, ky, d, fx, fy);     // option II: the frame build's keys
      }
      int tot;
      const int f = fbase + cta_excl_scan(listed, wsum, tot);
      fbase += tot;
      bool cand = listed && renew_key(q, kx, ky, d, fx, fy);
      bool near = false;
      for (int s0 = 0; s0 < ns; s0 += SR_STAGE) {                                 // the carried keys, staged
        const int m = min(SR_STAGE, ns - s0);
        __syncthreads();
        for (int k = tid; k < m; k += SR_THREADS) { s_key[2 * k] = s.x_dev[off + s0 + k]; s_key[2 * k + 1] = s.y_dev[off + s0 + k]; }
        __syncthreads();
        if (cand && !near) near = near_any(kx, ky, s_key, m);
      }
      cand = cand && !near;
      const int r = f % SR_PASSES;
      if (phase == 0) {
        if (cand) atomicAdd(&s_cnt[r], 1);
        continue;
      }
      // the rank of f in visit order: the kept candidates of earlier passes, of this pass in earlier chunks, warps and lanes
      const unsigned same = __match_any_sync(0xffffffffu, cand ? r : -1);
      const int wr = __popc(same & ((1u << lane) - 1u));
      if (cand && wr == 0) s_w[wid][r] = __popc(same);
      __syncthreads();
      if (tid < SR_PASSES) {
        int acc = 0;
        for (int w = 0; w < SR_THREADS / 32; ++w) { const int c = s_w[w][tid]; s_w[w][tid] = acc; acc += c; }
        s_ctot[tid] = acc;
      }
      __syncthreads();
      if (cand) {
        const int rank = s_cnt[r] + s_run[r] + s_w[wid][r] + wr;
        if (rank < need) put(ns + rank, kx, ky, d, fx, fy, -1);
      }
      __syncthreads();
      if (tid < SR_PASSES) s_run[tid] += s_ctot[tid];
      for (int k = tid; k < SR_THREADS / 32 * SR_PASSES; k += SR_THREADS) s_w[k / SR_PASSES][k % SR_PASSES] = 0;
      __syncthreads();
    }
    __syncthreads();
    if (phase == 0 && tid == 0) {                       // counts -> the first rank of each pass
      int acc = 0;
      for (int r = 0; r < SR_PASSES; ++r) { const int c = s_cnt[r]; s_cnt[r] = acc; acc += c; }
      s_ctot[0] = acc;
    }
    __syncthreads();
    if (phase == 0) added = min(need, s_ctot[0]);
    __syncthreads();
  }
  if (tid < 16) { s.Tcw_dev[16 * p + tid] = cam.T_dev[16 * p + tid]; s.velocity_dev[16 * p + tid] = cam.velocity_dev[16 * p + tid]; }
  if (tid == 0) { s.count_dev[p] = ns + added; s.status_dev[p] = status; s.has_velocity_dev[p] = 1; }
}

}  // namespace

// ---- vdo_cam_motion: the work space of vdo_cam_track_batch_dev, all allocated at creation ----
struct vdo_cam_motion : vdo::WorkSpace {
  vdo_ctx* ctx = nullptr;
  int dev = 0, max_pairs = 0, cap = 0;
  float *obj = nullptr, *img = nullptr;                                 // world points, observations
  int *r_idx = nullptr, *m_idx = nullptr, *s_idx = nullptr;
  int *samples = nullptr, *counts = nullptr;                            // pairs x VDO_CAM_MOTION_MAX_ITERS (x 4)
  double* models = nullptr;
  PnpProb* prob = nullptr;
  PnpOut* res = nullptr;
  FlowProb* fprob = nullptr;
  float *pts = nullptr, *depth = nullptr, *flow = nullptr, *X = nullptr;   // LM inputs at the pairs' offsets; X: the LM's poses
  double *flow_res = nullptr, *scratch = nullptr;                       // scratch: only when cap > the cluster limit
  unsigned char* inl = nullptr;
};

extern "C" int vdo_cam_motion_create(vdo_ctx* ctx, int max_pairs, int cap, vdo_cam_motion** out) {
  if (!ctx || !out) return VDO_ERR_ARG;
  *out = nullptr;
  if (max_pairs < 1 || max_pairs > CM_MAX_PAIRS || cap < 1 || (int64_t)max_pairs * cap > INT_MAX) {
    vdo::ctx_set_error(ctx, "vdo_cam_motion_create: max_pairs = " + std::to_string(max_pairs) + ", cap = " + std::to_string(cap) +
                                "; expected 1 .. 64 and >= 1, with max_pairs x cap below 2^31");
    return VDO_ERR_ARG;
  }
  vdo_cam_motion* m = new vdo_cam_motion;
  m->ctx = ctx; m->max_pairs = max_pairs; m->cap = cap;
  int n_sm = 0;
  vdo::ctx_device(ctx, &m->dev, &n_sm);
  const size_t pts = (size_t)max_pairs * cap, P = (size_t)max_pairs, hyp = P * VDO_CAM_MOTION_MAX_ITERS;
  return vdo::create_done(ctx, "vdo_cam_motion_create", m,
                          {m->alloc(m->obj, 3 * pts), m->alloc(m->img, 2 * pts), m->alloc(m->r_idx, pts), m->alloc(m->m_idx, pts), m->alloc(m->s_idx, pts),
                           m->alloc(m->samples, 4 * hyp), m->alloc(m->counts, hyp), m->alloc(m->models, 12 * hyp), m->alloc(m->prob, P),
                           m->alloc(m->res, P), m->alloc(m->fprob, P), m->alloc(m->pts, 2 * pts), m->alloc(m->depth, pts), m->alloc(m->flow, 2 * pts),
                           m->alloc(m->X, 16 * P), m->alloc(m->flow_res, 2 * pts), m->alloc(m->inl, pts),
                           cap > VDO_FLOW2_CLUSTER_MAX_N ? m->alloc(m->scratch, pts * vdo::flow_lm_fields()) : cudaSuccess, vdo::flow_lm_prepare()},
                          out);
}
extern "C" void vdo_cam_motion_destroy(vdo_cam_motion* m) { delete m; }
extern "C" int vdo_cam_motion_info(const vdo_cam_motion* m, int64_t out[4]) {
  if (!m || !out) return VDO_ERR_ARG;
  out[0] = m->max_pairs; out[1] = m->cap; out[2] = VDO_CAM_MOTION_MAX_ITERS; out[3] = (int64_t)m->bytes;
  return VDO_OK;
}

namespace {
// the set's fields, checked into ptrs (rows: the per-row columns; pair: count, status, Tcw, velocity, has_velocity)
void set_ptrs(const vdo_stat_feat_set& s, const std::string& who, bool rows, vdo::DevPtrs& ptrs) {
  if (rows)
    ptrs.insert(ptrs.end(), {{s.x_dev, 4, who + ".x_dev"}, {s.y_dev, 4, who + ".y_dev"}, {s.depth_dev, 4, who + ".depth_dev"}, {s.cx_dev, 4, who + ".cx_dev"},
                             {s.cy_dev, 4, who + ".cy_dev"}, {s.flow_dev, 4, who + ".flow_dev"}, {s.inlier_id_dev, 4, who + ".inlier_id_dev"},
                             {s.point_dev, 4, who + ".point_dev"}});
  ptrs.insert(ptrs.end(), {{s.count_dev, 4, who + ".count_dev"}, {s.status_dev, 4, who + ".status_dev"}, {s.Tcw_dev, 4, who + ".Tcw_dev"},
                           {s.velocity_dev, 4, who + ".velocity_dev"}, {s.has_velocity_dev, 4, who + ".has_velocity_dev"}});
}

// the checks build and renew share, in order: "" or the refusal; fills a (keys, planes, K, options) and ptrs
std::string stat_check(const vdo_cam_motion* m, int P, const vdo_orb_desc_set* keys, const vdo_dev_plane* depth, const vdo_dev_plane* flow,
                       const vdo_dev_plane* mask, const int32_t* wh, const float* K, const int32_t* gate_count_dev, const vdo_stat_opts* opts, StatArg& a,
                       vdo::DevPtrs& ptrs) {
  if (P < 1 || P > m->max_pairs) return "P = " + std::to_string(P) + " outside 1 .. " + std::to_string(m->max_pairs);
  if (!keys || !depth || !flow || !mask || !wh || !K || !opts) return "keys, depth, flow, mask, wh, K or opts is NULL";
  if (keys->n_frames < P) return "keys.n_frames = " + std::to_string(keys->n_frames) + " below P = " + std::to_string(P);
  if (keys->cap < 1 || keys->cap > m->cap) return "keys.cap = " + std::to_string(keys->cap) + " outside 1 .. the estimator's cap " + std::to_string(m->cap);
  const vdo_stat_opts& o = *opts;
  if (std::isnan(o.th_depth_bg)) return "th_depth_bg is NaN";
  if (o.use_sample_feature != 0 && o.use_sample_feature != 1) return "use_sample_feature = " + std::to_string(o.use_sample_feature) + "; expected 0 or 1";
  if (o.use_sample_feature && !gate_count_dev) return "gate_count_dev is NULL with use_sample_feature = 1";
  std::memset(&a, 0, sizeof a);
  for (int p = 0; p < P; ++p) {
    const std::string who = "pair " + std::to_string(p) + ": ";
    const int w = wh[2 * p], h = wh[2 * p + 1];
    if (w < 1 || h < 1) return who + std::to_string(w) + " x " + std::to_string(h) + "; expected a width and height >= 1";
    const vdo_dev_plane* pl[3] = {&depth[p], &flow[p], &mask[p]};
    static const char* kName[3] = {"depth", "flow", "mask"};
    static const char* kWant[3] = {"f32 with 1 channel", "f32 with 2 channels", "i32 or i64 with 1 channel"};
    for (int k = 0; k < 3; ++k) {
      const int dt = pl[k]->dtype, ch = pl[k]->channels;
      const bool ok = k == 0 ? dt == VDO_DT_F32 && ch == 1 : k == 1 ? dt == VDO_DT_F32 && ch == 2 : (dt == VDO_DT_I32 || dt == VDO_DT_I64) && ch == 1;
      if (!ok) return who + kName[k] + " plane: dtype " + std::to_string(dt) + " with " + std::to_string(ch) + " channels; expected " + kWant[k];
      ptrs.push_back({pl[k]->data_dev, size_t(dt == VDO_DT_I64 ? 8 : 4), who + kName[k] + " plane data_dev"});
    }
    StatPair& q = a.pr[p];
    q.dep = plane_arg(&depth[p]); q.flo = plane_arg(&flow[p]); q.msk = plane_arg(&mask[p]); q.w = w; q.h = h;
    for (int c = 0; c < 4; ++c) q.K[c] = K[4 * p + c];
  }
  ptrs.insert(ptrs.end(), {{keys->x_dev, 4, "keys.x_dev"}, {keys->y_dev, 4, "keys.y_dev"}, {keys->count_dev, 4, "keys.count_dev"},
                           {gate_count_dev, 4, "gate_count_dev", o.use_sample_feature != 0}});
  a.kx = keys->x_dev; a.ky = keys->y_dev; a.kcount = keys->count_dev; a.gate = gate_count_dev; a.kcap = keys->cap;
  a.C = m->cap; a.max_bg = o.max_track_bg; a.sampled = o.use_sample_feature; a.th = o.th_depth_bg;
  return "";
}
}  // namespace

extern "C" int vdo_stat_build_batch_dev(vdo_cam_motion* m, int P, const vdo_orb_desc_set* keys, const vdo_dev_plane* depth, const vdo_dev_plane* flow,
                                        const vdo_dev_plane* mask, const int32_t* wh, const float* K, const int32_t* gate_count_dev,
                                        const vdo_stat_opts* opts, const vdo_stat_feat_set* set, uint64_t stream) {
  if (!m) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(m->ctx, "vdo_stat_build_batch_dev: " + s); return VDO_ERR_ARG; };
  StatArg a;
  vdo::DevPtrs ptrs;
  if (std::string why = stat_check(m, P, keys, depth, flow, mask, wh, K, gate_count_dev, opts, a, ptrs); !why.empty()) return refuse(why);
  if (!set) return refuse("set is NULL");
  set_ptrs(*set, "set", true, ptrs);
  if (std::string why = vdo::check_ptrs(ptrs, m->dev); !why.empty()) return refuse(why);
  k_sb_build<<<P, SR_THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>(a, *set);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}

extern "C" int vdo_cam_track_batch_dev(vdo_cam_motion* m, int P, const vdo_stat_feat_set* set, const float* K, const vdo_cam_track_opts* opts,
                                       const vdo_cam_track_out* out, uint64_t stream) {
  if (!m) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(m->ctx, "vdo_cam_track_batch_dev: " + s); return VDO_ERR_ARG; };
  if (P < 1 || P > m->max_pairs) return refuse("P = " + std::to_string(P) + " outside 1 .. " + std::to_string(m->max_pairs));
  if (!set || !K || !opts || !out) return refuse("set, K, opts or out is NULL");
  const vdo_cam_track_opts& o = *opts;
  if (o.iters < 1 || o.iters > VDO_CAM_MOTION_MAX_ITERS) return refuse("iters = " + std::to_string(o.iters) + " outside 1 .. " + std::to_string(VDO_CAM_MOTION_MAX_ITERS));
  if (!(o.thr > 0.0)) return refuse("thr = " + std::to_string(o.thr) + "; expected > 0");
  if (!(o.conf > 0.0 && o.conf < 1.0)) return refuse("conf = " + std::to_string(o.conf) + "; expected inside (0, 1)");
  if (o.quirk != 0 && o.quirk != 1) return refuse("quirk = " + std::to_string(o.quirk) + "; expected 0 or 1");
  vdo::DevPtrs ptrs;
  set_ptrs(*set, "set", true, ptrs);
  const vdo_cam_track_out& u = *out;
  ptrs.insert(ptrs.end(), {{u.T_dev, 4, "out.T_dev"}, {u.T_init_dev, 4, "out.T_init_dev"}, {u.velocity_dev, 4, "out.velocity_dev"},
                           {u.info_dev, 4, "out.info_dev"}, {u.stats_dev, 8, "out.stats_dev"}, {u.status_dev, 4, "out.status_dev"},
                           {u.flags_dev, 1, "out.flags_dev"}, {u.key_dev, 4, "out.key_dev"}, {u.flow_ref_dev, 8, "out.flow_ref_dev"}});
  if (std::string why = vdo::check_ptrs(ptrs, m->dev); !why.empty()) return refuse(why);
  CamArg a;
  std::memset(&a, 0, sizeof a);
  a.C = m->cap;
  for (int p = 0; p < P; ++p)
    for (int c = 0; c < 4; ++c) a.K[p][c] = K[4 * p + c];
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  k_ct_gather<<<P, CM_THREADS, 0, st>>>(a, *set, m->obj, m->img, m->prob);
  vdo::pnp_samples_launch(m->prob, P, o.iters, m->samples, st);
  vdo::pnp_ransac_launch(m->prob, P, m->obj, m->img, m->samples, o.iters, o.thr, o.conf, m->models, m->counts, m->res, m->r_idx, m->m_idx, m->s_idx, st);
  k_ct_lm_prep<<<P, CM_THREADS, 0, st>>>(a, *set, m->prob, m->res, m->s_idx, m->pts, m->depth, m->flow, m->fprob);
  const FlowDev d{m->fprob, m->pts, m->depth, m->flow, m->scratch, m->X, m->flow_res, m->inl, u.stats_dev, o.quirk, 0, nullptr};
  vdo::flow_lm_launch(d, P, m->cap, st);
  k_ct_finish<<<P, CM_THREADS, 0, st>>>(a, *set, u, m->prob, m->res, m->s_idx, m->X, m->flow_res, m->inl);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}

extern "C" int vdo_stat_renew_batch_dev(vdo_cam_motion* m, int P, const vdo_stat_feat_set* last, const vdo_cam_track_out* cam, const vdo_orb_desc_set* keys,
                                        const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask, const int32_t* wh, const float* K,
                                        const int32_t* gate_count_dev, const vdo_stat_opts* opts, const vdo_stat_feat_set* set_out, uint64_t stream) {
  if (!m) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(m->ctx, "vdo_stat_renew_batch_dev: " + s); return VDO_ERR_ARG; };
  StatArg a;
  vdo::DevPtrs ptrs;
  if (std::string why = stat_check(m, P, keys, depth, flow, mask, wh, K, gate_count_dev, opts, a, ptrs); !why.empty()) return refuse(why);
  if (!last || !cam || !set_out) return refuse("last, cam or set_out is NULL");
  if (opts->max_track_bg < 0 || (int64_t)opts->max_track_bg + 1 > m->cap)
    return refuse("max_track_bg = " + std::to_string(opts->max_track_bg) + "; expected 0 .. cap - 1 = " + std::to_string(m->cap - 1));
  ptrs.push_back({last->count_dev, 4, "last.count_dev"});
  const vdo_cam_track_out& c = *cam;
  ptrs.insert(ptrs.end(), {{c.T_dev, 4, "cam.T_dev"}, {c.velocity_dev, 4, "cam.velocity_dev"}, {c.status_dev, 4, "cam.status_dev"},
                           {c.flags_dev, 1, "cam.flags_dev"}, {c.key_dev, 4, "cam.key_dev"}});
  set_ptrs(*set_out, "set_out", true, ptrs);
  if (std::string why = vdo::check_ptrs(ptrs, m->dev); !why.empty()) return refuse(why);
  k_sr_select<<<P, SR_THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>(a, *last, c, *set_out);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
