// obj_motion.cu -- the object step of Tracking::Track (src/Tracking.cc:760-1003, bJoint = true) for P frame pairs on the device, from the
// caller's planes: semi-dense sampling of each pair's last frame, grouping by instance label, the initial model of GetInitModelObj
// (:1717-1849) with the constant-motion-model choice, the min_inliers gate, PoseOptimizationFlow2 (Optimizer.cc:2755-2972, mode 1) and
// H = Tcw_cur^-1 X (:933) with the object centre (:856-866) and velocity (:958).
//
// Launches of vdo_obj_motion_batch_dev (problems = P x max_objects object slots, sized on the host; an empty slot's CTAs return at once):
//   k_om_sample      one CTA per pair: the stride-`step` raster of the pair's planes through the sampling rule of frame_px.cuh, in raster
//                    order, into the pair's sample segment (offset p * cap)
//   k_om_group       one CTA per pair: the distinct labels (ascending, the first max_objects), a stable counting sort of the samples by
//                    slot, the world points and observations, the centres, the motion models and one PnpProb per slot
//   k_pnp_samples / k_pnp_hyp / k_pnp_score / k_pnp_finish   pnp_ransac.cu's kernels, unchanged (dev_solvers.cuh launchers)
//   k_om_lm_prep     one CTA per slot: the min_inliers gate, the chosen set compacted into the slot's FlowProb (mode 1)
//   k_refine_lm_cl / k_refine_lm   flow_lm.cu's kernels, unchanged (the single-CTA one only when an object may exceed the cluster's limit)
//   k_om_finish      one CTA per slot: H, velocity, counters and status; the chosen set's flags and refined flows per sample
// Launches of vdo_obj_track_batch_dev (GetSceneFlowObj and DynObjTracking, Tracking.cc:1278-1612, ahead of the same object step):
//   k_om_sample      as above
//   k_ot_flow        (frame_kernels.cu, built with k_scene_flow's flags) one thread per sample: the current look-up and the scene flow
//   k_ot_group       one CTA per pair: k_om_group's sort by current label, the vote, the classification (dyn_obj.cuh), the IDs, and one
//                    PnpProb per slot (empty unless dynamic; the motion model by ID)
//   the RANSAC kernels, k_om_lm_prep, the LM and k_om_finish as above
//   k_ot_finish      one CTA per pair: stat per slot, vObjLabel per sample
// This file is compiled with --fmad=false: the 4x4 products, the inverse, the back-projection (pose4.cuh), the centre and the velocity then
// round as the tracker's host helpers (tracker.cpp mul4 / inv4 / unproject_world, cv::Mat float arithmetic) round them.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"
#include "dev_solvers.cuh"
#include "dyn_obj.cuh"
#include "frame_batch.h"
#include "frame_px.cuh"
#include "pnp_corr.cuh"
#include "pose4.cuh"

namespace {
using vdo::FlowDev;
using vdo::FlowProb;
using vdo::PnpOut;
using vdo::PnpProb;

constexpr int OM_MAX_PAIRS = VDO_OBJ_MOTION_MAX_PAIRS, OM_MAX_OBJ = VDO_OBJ_MOTION_MAX_OBJECTS;
constexpr int OM_SAMPLE_THREADS = 1024, OM_THREADS = 256;

struct ObjPair { PlaneArg dep, flo, msk; int w, h; float K[4]; };
struct ObjArg {                 // the call's host parameters, passed by value so that a captured call replays with them
  const float *Tl, *Tc;         // device P x 16, or NULL (identity)
  const int* prev_label;        // device P x M, or NULL (no motion models)
  const float* prev_H;          // device P x M x 16
  int step, cap, M, min_inliers;
  float th;
  ObjPair pr[OM_MAX_PAIRS];
};
struct TrackArg {               // vdo_obj_track_batch_dev's further parameters (prev_label and prev_H travel in ObjArg)
  const int *prev_id, *prev_stat, *prev_max_id;   // device P x M, P x M, P; all NULL: the reset state
  float sf_mg, sf_ds;
  int shrink_row, shrink_col;
};

// ---- 1. samples ----
// pair p's raster samples (one CTA of OM_SAMPLE_THREADS)
__device__ __forceinline__ void om_raster(const ObjArg& a, const vdo_obj_motion_out& o, int* __restrict__ pstat, int p) {
  __shared__ int wsum[33];
  __shared__ int s_bad;
  const ObjPair& q = a.pr[p];
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  const int w = q.w, h = q.h, step = a.step;
  const int nx = (w + step - 1) / step, ny = (h + step - 1) / step, n = nx * ny;
  const size_t off = (size_t)p * a.cap;
  int base = 0;
  for (int start = 0; start < n; start += OM_SAMPLE_THREADS) {
    const int i = start + threadIdx.x;
    int ok = 0, x = 0, y = 0, m = 0; float d = 0, fx = 0, fy = 0, tx = 0, ty = 0;
    if (i < n) {
      x = (i % nx) * step; y = (i / nx) * step;
      m = plane_label(q.msk, x, y, &s_bad); d = plane_depth(q.dep, x, y);
      ok = object_sample(x, y, m, d, a.th, w, h, [&](float& u, float& v) { const float2 f = plane_flow(q.flo, x, y); u = f.x; v = f.y; }, fx, fy, tx, ty);
    }
    int tot;
    const size_t k = off + base + cta_excl_scan(ok, wsum, tot);   // the host refused a cap below n: no sample is dropped
    if (ok) {
      o.sample_x_dev[k] = x; o.sample_y_dev[k] = y; o.sample_label_dev[k] = m; o.sample_depth_dev[k] = d;
      o.sample_cx_dev[k] = tx; o.sample_cy_dev[k] = ty; o.sample_flow_dev[2 * k] = fx; o.sample_flow_dev[2 * k + 1] = fy;
    }
    base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) { o.n_samples_dev[p] = base; pstat[p] = s_bad ? VDO_OM_PAIR_LABEL_RANGE : 0; }
}
__global__ void __launch_bounds__(OM_SAMPLE_THREADS) k_om_sample(const __grid_constant__ ObjArg a, vdo_obj_motion_out o, int* __restrict__ pstat) {
  om_raster(a, o, pstat, blockIdx.x);
}

// the carried feature set of the *_set entries (vdo_obj_feat_set, the fields they read)
struct SetArg { const int *x, *y, *label, *count; const float *depth, *cx, *cy, *flow; };
// k_om_sample for the *_set entries: a pair with a carried set (count 0 .. cap) copies its rows, a pair with count -1 samples its raster
__global__ void __launch_bounds__(OM_SAMPLE_THREADS) k_os_sample(const __grid_constant__ ObjArg a, const __grid_constant__ SetArg s, vdo_obj_motion_out o,
                                                                 int* __restrict__ pstat) {
  const int p = blockIdx.x, cnt = s.count[p];
  if (cnt == -1) { om_raster(a, o, pstat, p); return; }
  const bool ok = cnt >= 0 && cnt <= a.cap;
  const int n = ok ? cnt : 0;
  const size_t off = (size_t)p * a.cap;
  for (int k = threadIdx.x; k < n; k += OM_SAMPLE_THREADS) {
    const size_t i = off + k;
    o.sample_x_dev[i] = s.x[i]; o.sample_y_dev[i] = s.y[i]; o.sample_label_dev[i] = s.label[i]; o.sample_depth_dev[i] = s.depth[i];
    o.sample_cx_dev[i] = s.cx[i]; o.sample_cy_dev[i] = s.cy[i]; o.sample_flow_dev[2 * i] = s.flow[2 * i]; o.sample_flow_dev[2 * i + 1] = s.flow[2 * i + 1];
  }
  if (threadIdx.x == 0) { o.n_samples_dev[p] = n; pstat[p] = ok ? 0 : VDO_OM_PAIR_SET_COUNT; }
}

// ---- 2. objects ----
__device__ __forceinline__ long long block_min(long long v, long long* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  long long m = s_red[0];
  for (int k = 1; k < OM_THREADS / 32; ++k) m = min(m, s_red[k]);
  __syncthreads();
  return m;
}

// One CTA per pair (k_om_group, k_ot_group): the grouping of the pair's n samples by lab (0: in no object).  Labels: repeated minimum above
// the last label found, at most M + 1 times (the (M + 1)-th only flags the cap).  The stable counting sort gives each thread a contiguous run
// of samples, so slot s's points keep the raster order: count per (slot, thread), scan per slot over threads, place.  Returns the number of
// labels found (at most M + 1); slot s holds ord[off + s_beg[s] .. off + s_beg[s + 1]).
__device__ __forceinline__ int group_sort(const int* __restrict__ lab, int n, int M, bool skip, size_t off, const vdo_obj_motion_out& o, int* __restrict__ ord,
                                          int (*s_cnt)[OM_THREADS], int* s_lab, int* s_beg, int* s_tot, long long* s_red) {
  const int tid = threadIdx.x;
  int nl = 0;
  if (!skip)
    for (; nl <= M; ++nl) {
      const long long prev = nl ? s_lab[nl - 1] : LLONG_MIN;
      long long mn = LLONG_MAX;
      for (int i = tid; i < n; i += OM_THREADS) { const long long v = lab[i]; if (v != 0 && v > prev && v < mn) mn = v; }
      mn = block_min(mn, s_red);
      if (mn == LLONG_MAX) break;
      if (tid == 0) s_lab[nl] = (int)mn;
      __syncthreads();
    }
  const int nobj = min(nl, M);
  // count: slot of each sample (binary search of the sorted labels), per (slot, thread)
  const int per = (n + OM_THREADS - 1) / OM_THREADS, i0 = min(n, tid * per), i1 = min(n, i0 + per);
  for (int s = 0; s < nobj; ++s) s_cnt[s][tid] = 0;
  for (int i = i0; i < i1; ++i) {
    const int v = lab[i];
    int lo = 0, hi = nobj;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_lab[mid] < v) lo = mid + 1; else hi = mid; }
    const int s = lo < nobj && s_lab[lo] == v ? lo : -1;
    o.sample_slot_dev[off + i] = s;
    o.sample_flags_dev[off + i] = 0;
    o.sample_flow_ref_dev[2 * (off + i)] = o.sample_flow_dev[2 * (off + i)];
    o.sample_flow_ref_dev[2 * (off + i) + 1] = o.sample_flow_dev[2 * (off + i) + 1];
    if (s >= 0) ++s_cnt[s][tid];
  }
  __syncthreads();
  if (tid < nobj) {
    int acc = 0;
    for (int t = 0; t < OM_THREADS; ++t) { const int c = s_cnt[tid][t]; s_cnt[tid][t] = acc; acc += c; }
    s_tot[tid] = acc;
  }
  __syncthreads();
  if (tid == 0) { int b = 0; for (int s = 0; s < nobj; ++s) { s_beg[s] = b; b += s_tot[s]; } s_beg[nobj] = b; }
  __syncthreads();
  for (int i = i0; i < i1; ++i) {
    const int s = o.sample_slot_dev[off + i];
    if (s >= 0) ord[off + s_beg[s] + s_cnt[s][tid]++] = i;
  }
  __syncthreads();
  return nl;
}

// the world points and observations of the nobj slots in slot order, then the centres: one thread per (slot, coordinate), the float sum in
// point order
__device__ __forceinline__ void group_points(const ObjPair& q, int M, int nobj, size_t off, size_t row, const vdo_obj_motion_out& o, const int* __restrict__ ord,
                                             float* __restrict__ obj, float* __restrict__ img, const int* s_beg, const float* s_Tl) {
  const int tid = threadIdx.x;
  for (int k = tid; k < s_beg[nobj]; k += OM_THREADS) {
    const int i = ord[off + k];
    unproject_world((float)o.sample_x_dev[off + i], (float)o.sample_y_dev[off + i], o.sample_depth_dev[off + i], q.K, s_Tl, obj + 3 * (off + k));
    img[2 * (off + k)] = o.sample_cx_dev[off + i]; img[2 * (off + k) + 1] = o.sample_cy_dev[off + i];
  }
  __syncthreads();
  if (tid < 3 * M) {                      // ObjCentre3D_pre + x3D_p in float, then cv::Mat / size() (convertTo with alpha = 1/n)
    const int s = tid / 3, r = tid % 3;
    float c = 0.f;
    if (s < nobj) {
      for (int k = s_beg[s]; k < s_beg[s + 1]; ++k) c = c + obj[3 * (off + k) + r];
      c = c * (float)(1.0 / (double)(s_beg[s + 1] - s_beg[s]));
    }
    o.centre_dev[3 * (row + s) + r] = c;
  }
}

// the RANSAC problem of a slot holding the n points from sorted position beg, without a motion model
__device__ __forceinline__ PnpProb slot_problem(const ObjPair& q, size_t off, int beg, int n) {
  PnpProb pb;
  pb.off = (int)(off + beg); pb.n = n;
  for (int c = 0; c < 4; ++c) { pb.K[c] = (double)q.K[c]; pb.Kf[c] = q.K[c]; }
  for (int c = 0; c < 12; ++c) pb.mm[c] = 0.f;
  pb.has_mm = 0; pb.pad = 0;
  return pb;
}

// One CTA per pair: the pair's samples grouped by their (last-frame) label, the world points, centres, motion models (by label) and problems.
__global__ void __launch_bounds__(OM_THREADS) k_om_group(const __grid_constant__ ObjArg a, vdo_obj_motion_out o, const int* __restrict__ pstat,
                                                         int* __restrict__ ord, float* __restrict__ obj, float* __restrict__ img, PnpProb* __restrict__ prob) {
  __shared__ int s_cnt[OM_MAX_OBJ][OM_THREADS];
  __shared__ int s_lab[OM_MAX_OBJ + 1], s_beg[OM_MAX_OBJ + 1], s_tot[OM_MAX_OBJ];
  __shared__ long long s_red[OM_THREADS / 32];
  __shared__ float s_Tl[16], s_Tc[16];
  const int p = blockIdx.x, tid = threadIdx.x, M = a.M;
  const ObjPair& q = a.pr[p];
  const size_t off = (size_t)p * a.cap;
  const int n = o.n_samples_dev[p];
  if (tid < 16) { s_Tl[tid] = a.Tl ? a.Tl[16 * p + tid] : (tid % 5 == 0 ? 1.f : 0.f); s_Tc[tid] = a.Tc ? a.Tc[16 * p + tid] : (tid % 5 == 0 ? 1.f : 0.f); }
  const int nl = group_sort(o.sample_label_dev + off, n, M, pstat[p] & VDO_OM_PAIR_LABEL_RANGE, off, o, ord, s_cnt, s_lab, s_beg, s_tot, s_red);
  const int nobj = min(nl, M);
  const size_t row = (size_t)p * M;
  group_points(q, M, nobj, off, row, o, ord, obj, img, s_beg, s_Tl);
  if (tid < M) {
    const int s = tid;
    PnpProb pb = slot_problem(q, off, s < nobj ? s_beg[s] : 0, s < nobj ? s_beg[s + 1] - s_beg[s] : 0);
    if (s < nobj && a.prev_label) {       // the PreObjID lookup: the first previous slot with the label
      const int L = s_lab[s];
      for (int j = 0; j < M; ++j)
        if (L != -1 && a.prev_label[row + j] == L) {
          float mm[16];
          mul4(s_Tc, a.prev_H + 16 * (row + j), mm);
          for (int c = 0; c < 12; ++c) pb.mm[c] = mm[c];
          pb.has_mm = 1;
          break;
        }
    }
    prob[row + s] = pb;
    o.label_dev[row + s] = s < nobj ? s_lab[s] : -1;
  }
  if (tid == 0) o.pair_status_dev[p] = pstat[p] | (nl > M ? VDO_OM_PAIR_OBJECT_CAP : 0);
}

// the majority of lab over the slot's samples ord[b .. e) by one warp: ascending labels by repeated minimum, the first with the largest count
// (tracking_ops.cu majority_label's tie rule)
__device__ __forceinline__ int warp_majority(const int* __restrict__ lab, const int* __restrict__ ord, int b, int e) {
  const int lane = threadIdx.x & 31;
  int best = 0, best_n = -1;
  for (long long prev = LLONG_MIN;;) {
    long long mn = LLONG_MAX;
    for (int k = b + lane; k < e; k += 32) { const long long v = lab[ord[k]]; if (v > prev && v < mn) mn = v; }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, s));
    if (mn == LLONG_MAX) break;
    int c = 0;
    for (int k = b + lane; k < e; k += 32) c += lab[ord[k]] == mn;
    c = __reduce_add_sync(0xffffffffu, c);
    if (c > best_n) { best_n = c; best = (int)mn; }
    prev = mn;
  }
  return best;
}

// One CTA per pair: DynObjTracking on the pair's valid samples (glab, the current label), then the world points, centres and problems of the
// dynamic slots (the others get empty problems), with the motion model looked up by ID.
__global__ void __launch_bounds__(OM_THREADS) k_ot_group(const __grid_constant__ ObjArg a, const __grid_constant__ TrackArg t, vdo_obj_track_out ot,
                                                         const int* __restrict__ pstat, const int* __restrict__ glab, int* __restrict__ ord,
                                                         float* __restrict__ obj, float* __restrict__ img, PnpProb* __restrict__ prob) {
  __shared__ int s_cnt[OM_MAX_OBJ][OM_THREADS];
  __shared__ int s_lab[OM_MAX_OBJ + 1], s_beg[OM_MAX_OBJ + 1], s_tot[OM_MAX_OBJ];
  __shared__ long long s_red[OM_THREADS / 32];
  __shared__ float s_Tl[16], s_Tc[16];
  __shared__ int s_cls[OM_MAX_OBJ], s_vote[OM_MAX_OBJ], s_id[OM_MAX_OBJ];
  const vdo_obj_motion_out& o = ot.motion;
  const int p = blockIdx.x, tid = threadIdx.x, M = a.M;
  const ObjPair& q = a.pr[p];
  const size_t off = (size_t)p * a.cap, row = (size_t)p * M;
  const int n = o.n_samples_dev[p];
  if (tid < 16) { s_Tl[tid] = a.Tl ? a.Tl[16 * p + tid] : (tid % 5 == 0 ? 1.f : 0.f); s_Tc[tid] = a.Tc ? a.Tc[16 * p + tid] : (tid % 5 == 0 ? 1.f : 0.f); }
  const int nl = group_sort(glab + off, n, M, pstat[p] & VDO_OM_PAIR_LABEL_RANGE, off, o, ord, s_cnt, s_lab, s_beg, s_tot, s_red);
  const int nobj = min(nl, M);
  // the vote of every slot, one warp per slot (only a dynamic slot's is used)
  for (int s = tid >> 5; s < nobj; s += OM_THREADS / 32) {
    const int v = warp_majority(o.sample_label_dev + off, ord + off, s_beg[s], s_beg[s + 1]);
    if ((tid & 31) == 0) s_vote[s] = v;
  }
  // the classification, one thread per slot walking its points in order (the sums of vdo_dyn_obj_tracking)
  if (tid < nobj) {
    ObjStat st{0.f, 0.f, 0.f, s_beg[tid + 1] - s_beg[tid]};
    for (int k = s_beg[tid]; k < s_beg[tid + 1]; ++k) {
      obj_stat_add(st, o.sample_cx_dev + off, o.sample_cy_dev + off, ot.depth_cur_dev + off, ot.flow3d_dev + 3 * off, ord[off + k], q.h, q.w, t.shrink_row,
                   t.shrink_col, t.sf_mg);
    }
    s_cls[tid] = obj_class(st, t.sf_ds, a.th);
  }
  __syncthreads();
  // the IDs in ascending label order (:1548-1599)
  if (tid == 0) {
    int max_id = t.prev_max_id ? t.prev_max_id[p] : 1;
    for (int s = 0; s < nobj; ++s) {
      int id = -1;
      if (s_cls[s] == OBJ_DYNAMIC) {
        if (max_id != 1 && t.prev_max_id)
          for (int j = 0; j < M; ++j)
            if (a.prev_label[row + j] == s_vote[s] && t.prev_stat[row + j]) { id = t.prev_id[row + j]; break; }
        if (id == -1) id = max_id++;
      }
      s_id[s] = id;
    }
    ot.max_id_dev[p] = max_id;
  }
  __syncthreads();
  group_points(q, M, nobj, off, row, o, ord, obj, img, s_beg, s_Tl);
  if (tid < M) {
    const int s = tid;
    const bool dyn = s < nobj && s_cls[s] == OBJ_DYNAMIC;
    PnpProb pb = slot_problem(q, off, s < nobj ? s_beg[s] : 0, dyn ? s_beg[s + 1] - s_beg[s] : 0);
    if (dyn && t.prev_max_id)             // the motion model by ID (tracker.cpp:407-409): the first previous slot with the ID, stat not required
      for (int j = 0; j < M; ++j)
        if (t.prev_id[row + j] == s_id[s]) {
          float mm[16];
          mul4(s_Tc, a.prev_H + 16 * (row + j), mm);
          for (int c = 0; c < 12; ++c) pb.mm[c] = mm[c];
          pb.has_mm = 1;
          break;
        }
    prob[row + s] = pb;
    o.label_dev[row + s] = s < nobj ? s_lab[s] : -1;
    ot.id_dev[row + s] = s < nobj ? s_id[s] : -1;
    ot.cls_dev[row + s] = s < nobj ? s_cls[s] : VDO_OT_EMPTY;
    ot.vote_dev[row + s] = dyn ? s_vote[s] : 0;
  }
  if (tid == 0) o.pair_status_dev[p] = pstat[p] | (nl > M ? VDO_OM_PAIR_OBJECT_CAP : 0);
}

// ---- 4. the gate and the LM problems ----
__device__ __forceinline__ bool runs_lm(const PnpProb& pr, const PnpOut& r, int min_inliers) { return pr.n > 0 && r.n_sub >= min_inliers; }

// one CTA per slot: the chosen set (local indices s_idx at the slot's off) -> the LM's points (the samples' pixel, depth and flow)
__global__ void __launch_bounds__(OM_THREADS) k_om_lm_prep(const __grid_constant__ ObjArg a, vdo_obj_motion_out o, const PnpProb* __restrict__ prob,
                                                           const PnpOut* __restrict__ res, const int* __restrict__ s_idx, const int* __restrict__ ord,
                                                           float* __restrict__ pts, float* __restrict__ depth, float* __restrict__ flow, FlowProb* __restrict__ fprob) {
  const int j = blockIdx.x, p = j / a.M, tid = threadIdx.x;
  const PnpProb pr = prob[j];
  const PnpOut& r = res[j];
  const int n = runs_lm(pr, r, a.min_inliers) ? r.n_sub : 0;
  const size_t off = (size_t)p * a.cap;
  for (int k = tid; k < n; k += OM_THREADS) {
    const size_t g = (size_t)pr.off + k, i = off + ord[pr.off + s_idx[g]];
    pts[2 * g] = (float)o.sample_x_dev[i]; pts[2 * g + 1] = (float)o.sample_y_dev[i];
    depth[g] = o.sample_depth_dev[i];
    flow[2 * g] = o.sample_flow_dev[2 * i]; flow[2 * g + 1] = o.sample_flow_dev[2 * i + 1];
  }
  if (tid == 0) {
    FlowProb fp;
    fp.mode = 1; fp.n = n; fp.offset = pr.off; fp.out = j;
    for (int c = 0; c < 4; ++c) fp.K[c] = a.pr[p].K[c];
    load_pose(a.Tl, p, fp.Tcw_last);
    for (int c = 0; c < 16; ++c) fp.T_init[c] = r.T[c];
    fprob[j] = fp;
  }
}

// ---- 6. per slot outputs and the per-sample scatter of the chosen set ----
__global__ void __launch_bounds__(OM_THREADS) k_om_finish(const __grid_constant__ ObjArg a, vdo_obj_motion_out o, const PnpProb* __restrict__ prob,
                                                          const PnpOut* __restrict__ res, const int* __restrict__ s_idx, const int* __restrict__ ord,
                                                          const double* __restrict__ flow_res, const unsigned char* __restrict__ inl) {
  const int j = blockIdx.x, p = j / a.M, tid = threadIdx.x;
  const PnpProb pr = prob[j];
  const PnpOut& r = res[j];
  const bool lm = runs_lm(pr, r, a.min_inliers);
  const size_t off = (size_t)p * a.cap;
  for (int k = tid; k < r.n_sub; k += OM_THREADS) {
    const size_t g = (size_t)pr.off + k, i = off + ord[pr.off + s_idx[g]];
    o.sample_flags_dev[i] = 1 | (lm && inl[g] ? 2 : 0);
    if (lm) { o.sample_flow_ref_dev[2 * i] = flow_res[2 * g]; o.sample_flow_ref_dev[2 * i + 1] = flow_res[2 * g + 1]; }
  }
  if (tid == 0) {
    float H[16];
    for (int c = 0; c < 16; ++c) H[c] = c % 5 == 0 ? 1.f : 0.f;
    if (lm) {
      float Tc[16], Ti[16];
      load_pose(a.Tc, p, Tc);
      inv4(Tc, Ti);
      mul4(Ti, o.X_dev + 16 * (size_t)j, H);
    }
    for (int c = 0; c < 16; ++c) { o.H_dev[16 * (size_t)j + c] = H[c]; o.T_init_dev[16 * (size_t)j + c] = r.T[c]; }
    // sp_est_v = H.t - (I - H.R) * c: the 3x3 difference, then the float gemm with the centre, then the difference
    const float* cen = o.centre_dev + 3 * (size_t)j;
    for (int i = 0; i < 3; ++i) {
      float s = ((i == 0 ? 1.f : 0.f) - H[4 * i]) * cen[0];
      s = s + ((i == 1 ? 1.f : 0.f) - H[4 * i + 1]) * cen[1];
      s = s + ((i == 2 ? 1.f : 0.f) - H[4 * i + 2]) * cen[2];
      o.velocity_dev[3 * (size_t)j + i] = H[4 * i + 3] - s;
    }
    int* info = o.info_dev + 8 * (size_t)j;
    info[0] = pr.n; info[1] = r.n_ransac; info[2] = r.n_mm; info[3] = r.used_mm; info[4] = r.n_sub; info[5] = r.iters_run; info[6] = r.best_it;
    info[7] = r.n_valid;
    o.status_dev[j] = pr.n == 0 ? 0
                                : (pr.n < 4 ? VDO_OM_FEW_POINTS : 0) | (pr.n >= 4 && r.best_it < 0 ? VDO_OM_NO_MODEL : 0) |
                                      (lm ? 0 : VDO_OM_FEW_INLIERS) | (r.used_mm ? VDO_OM_USED_MM : 0);
  }
}

// ---- 7. vdo_obj_track_batch_dev: stat per slot and vObjLabel per sample, one CTA per pair ----
__global__ void __launch_bounds__(OM_THREADS) k_ot_finish(const __grid_constant__ ObjArg a, vdo_obj_track_out ot, const int* __restrict__ glab) {
  const vdo_obj_motion_out& o = ot.motion;
  const int p = blockIdx.x, tid = threadIdx.x;
  const size_t off = (size_t)p * a.cap, row = (size_t)p * a.M;
  // a dynamic slot has >= 150 points, so it ran the LM exactly when VDO_OM_FEW_INLIERS is clear
  auto passed = [&](int s) { return ot.cls_dev[row + s] == OBJ_DYNAMIC && !(o.status_dev[row + s] & VDO_OM_FEW_INLIERS); };
  for (int s = tid; s < a.M; s += OM_THREADS) ot.stat_dev[row + s] = passed(s);
  const int n = o.n_samples_dev[p];
  for (int k = tid; k < n; k += OM_THREADS) {
    const size_t i = off + k;
    const int s = o.sample_slot_dev[i];
    int lab = -2;                                                       // valid, but its label got no slot
    if (!glab[i]) lab = -1;                                             // GetSceneFlowObj: a label <= 0
    else if (s >= 0) {
      const int cls = ot.cls_dev[row + s];
      if (cls == OBJ_STATIC) lab = 0;
      else if (cls != OBJ_DYNAMIC) lab = -1;
      else {
        const int f = o.sample_flags_dev[i];
        const bool lm = !(o.status_dev[row + s] & VDO_OM_FEW_INLIERS);
        lab = !(f & 1) || (lm && !(f & 2)) ? -1 : ot.id_dev[row + s];  // outside the chosen set (:1841-1845), an LM outlier
      }
    }
    ot.obj_label_dev[i] = lab;
  }
}

// ---- 8. vdo_obj_update_mask_batch_dev: UpdateMask (Tracking.cc:2997-3068) on the caller's current masks ----
// The call runs no RANSAC and no LM, so the samples and its tables live in work space those leave idle (MaskArg, set up on the host).
// Pair p's tables: a hash of the in-image sample targets (key: the pixel index y * W + x, UM_EMPTY when free), each with a word whose bit s
// says that slot s's last-frame mask is pushed onto that pixel, and UM_TAB ints: the slot boundaries in the sorted order, then:
enum { UM_NOBJ = OM_MAX_OBJ + 1, UM_CAND, UM_REC, UM_HP, UM_TAB };   // slots; slots with >= 100 voters; recovered slots; hash size
constexpr unsigned long long UM_EMPTY = ~0ull;
constexpr int UM_MIN_VOTES = 100;

struct MaskArg {
  PlaneArg cur[OM_MAX_PAIRS];     // mask_cur of each pair (i32 or i64), written in place
  unsigned long long* key;        // pair p's hash at key + p * hs
  unsigned* word;                 // its words, at word + p * hs
  int* tab;                       // pair p's table at tab + p * tab_stride
  int* vlab;                      // P x cap: the current labels of a slot's voters, at the slot's sorted positions
  int hs, tab_stride;
  vdo_obj_mask_out o;
};

__device__ __forceinline__ unsigned um_hash(unsigned long long k, int hp) { return (unsigned)(((k * 0x9E3779B97F4A7C15ull) >> 32) % (unsigned)hp); }
// linear probing; a table always has a free entry (it holds at most one key per sample, hp > n), so both loops end
__device__ __forceinline__ void um_insert(unsigned long long* key, int hp, unsigned long long k) {
  for (unsigned h = um_hash(k, hp);; h = h + 1 == (unsigned)hp ? 0 : h + 1) {
    const unsigned long long old = atomicCAS(key + h, UM_EMPTY, k);
    if (old == UM_EMPTY || old == k) return;
  }
}
__device__ __forceinline__ int um_find(const unsigned long long* key, int hp, unsigned long long k) {
  for (unsigned h = um_hash(k, hp);; h = h + 1 == (unsigned)hp ? 0 : h + 1) {
    const unsigned long long v = key[h];
    if (v == k) return (int)h;
    if (v == UM_EMPTY) return -1;
  }
}
// the current mask's element at pixel (x, y)
__device__ __forceinline__ long long cur_label(const PlaneArg& c, int x, int y) {
  const long long o = y * c.sy + x * c.sx;
  return c.dtype == VDO_DT_I64 ? ((const long long*)c.p)[o] : (long long)((const int*)c.p)[o];
}
// UpdateMask's image test of a flow target (truncated to int): strictly inside
__device__ __forceinline__ bool um_inside(int x, int y, int w, int h) { return x < w && x > 0 && y < h && y > 0; }

// One CTA per pair: k_om_group's sort of the samples by (last-frame) label into slots, the voter counts (in-image targets; they do not depend
// on the mask) and, when some slot has >= 100 voters, every slotted sample's in-image target in the pair's hash.
__global__ void __launch_bounds__(OM_THREADS) k_um_group(const __grid_constant__ ObjArg a, const __grid_constant__ MaskArg u, vdo_obj_motion_out o,
                                                         const int* __restrict__ pstat, int* __restrict__ ord) {
  __shared__ int s_cnt[OM_MAX_OBJ][OM_THREADS];
  __shared__ int s_lab[OM_MAX_OBJ + 1], s_beg[OM_MAX_OBJ + 1], s_tot[OM_MAX_OBJ];
  __shared__ long long s_red[OM_THREADS / 32];
  __shared__ int s_vote[OM_MAX_OBJ];
  const int p = blockIdx.x, tid = threadIdx.x, M = a.M;
  const ObjPair& q = a.pr[p];
  const size_t off = (size_t)p * a.cap, row = (size_t)p * M;
  const int n = o.n_samples_dev[p];
  if (tid < OM_MAX_OBJ) s_vote[tid] = 0;
  const int nl = group_sort(o.sample_label_dev + off, n, M, pstat[p] & VDO_OM_PAIR_LABEL_RANGE, off, o, ord, s_cnt, s_lab, s_beg, s_tot, s_red);
  const int nobj = min(nl, M), ns = s_beg[nobj];
  for (int s = 0; s < nobj; ++s) {
    int c = 0;
    for (int k = s_beg[s] + tid; k < s_beg[s + 1]; k += OM_THREADS) {
      const int i = ord[off + k];
      c += um_inside((int)o.sample_cx_dev[off + i], (int)o.sample_cy_dev[off + i], q.w, q.h);
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((tid & 31) == 0 && c) atomicAdd(&s_vote[s], c);
  }
  __syncthreads();
  unsigned cand = 0;
  for (int s = 0; s < nobj; ++s) cand |= s_vote[s] >= UM_MIN_VOTES ? 1u << s : 0u;
  // at most ns <= n <= cap keys: 2 ns + 1 entries, or hs = 3 cap / 2 > cap (a candidate has >= 100 samples, so cap >= 100) keep one free
  const int hp = cand ? min(u.hs, 2 * ns + 1) : 0;
  unsigned long long* key = u.key + (size_t)p * u.hs;
  if (cand) {
    for (int k = tid; k < hp; k += OM_THREADS) { key[k] = UM_EMPTY; u.word[(size_t)p * u.hs + k] = 0u; }
    __syncthreads();
    for (int k = tid; k < ns; k += OM_THREADS) {
      const int i = ord[off + k], x = (int)o.sample_cx_dev[off + i], y = (int)o.sample_cy_dev[off + i];
      if (um_inside(x, y, q.w, q.h)) um_insert(key, hp, (unsigned long long)y * q.w + x);
    }
  }
  int* tab = u.tab + (size_t)p * u.tab_stride;
  if (tid <= nobj) tab[tid] = s_beg[tid];
  if (tid < M) {
    u.o.label_dev[row + tid] = tid < nobj ? s_lab[tid] : -1;
    u.o.n_vote_dev[row + tid] = tid < nobj ? s_vote[tid] : 0;
  }
  if (tid == 0) {
    tab[UM_NOBJ] = nobj; tab[UM_CAND] = (int)cand; tab[UM_REC] = 0; tab[UM_HP] = hp;
    u.o.pair_status_dev[p] = pstat[p] | (nl > M ? VDO_OM_PAIR_OBJECT_CAP : 0);
  }
}

// the slot of last-frame pixel (x, y): its label among the nobj sorted slot labels, or -1
__device__ __forceinline__ int um_slot(const ObjPair& q, int x, int y, const int* s_lab, int nobj) {
  int bad;
  const int v = plane_label(q.msk, x, y, &bad);                 // an i64 label wraps as the host route's int32 mask does
  int lo = 0, hi = nobj;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_lab[mid] < v) lo = mid + 1; else hi = mid; }
  return lo < nobj && s_lab[lo] == v ? lo : -1;
}

// Pixel passes over each pair's last frame (grid: pixels of the largest frame x P; one thread per pixel).  Pixel (k, j) of slot s goes to
// (k + (int)fx, j + (int)fy).  PASS 0: for a candidate slot whose target is a sample target, set bit s of that target's word.  PASS 1: for
// a recovered slot, claim the target (the type's minimum).  PASS 2: for a recovered slot, atomicMax the slot's label into the target: the
// highest recovered slot that pushes onto a pixel wins, as the reference's last write does.
template <int PASS>
__global__ void __launch_bounds__(OM_THREADS) k_um_pixels(const __grid_constant__ ObjArg a, const __grid_constant__ MaskArg u) {
  __shared__ int s_lab[OM_MAX_OBJ];
  const int p = blockIdx.y;
  const int* tab = u.tab + (size_t)p * u.tab_stride;
  const unsigned sel = (unsigned)tab[PASS == 0 ? UM_CAND : UM_REC];
  if (!sel) return;                                               // the same for the whole CTA
  const int nobj = tab[UM_NOBJ];
  if (threadIdx.x < nobj) s_lab[threadIdx.x] = u.o.label_dev[(size_t)p * a.M + threadIdx.x];
  __syncthreads();
  const ObjPair& q = a.pr[p];
  const long long pix = (long long)blockIdx.x * OM_THREADS + threadIdx.x;
  if (pix >= (long long)q.w * q.h) return;
  const int k = (int)(pix % q.w), j = (int)(pix / q.w);
  const int s = um_slot(q, k, j, s_lab, nobj);
  if (s < 0 || !(sel >> s & 1u)) return;
  const float2 f = plane_flow(q.flo, k, j);
  const int x = k + (int)f.x, y = j + (int)f.y;
  if (!um_inside(x, y, q.w, q.h)) return;
  if (PASS == 0) {
    const int e = um_find(u.key + (size_t)p * u.hs, tab[UM_HP], (unsigned long long)y * q.w + x);
    if (e >= 0) atomicOr(u.word + (size_t)p * u.hs + e, 1u << s);
    return;
  }
  const PlaneArg& c = u.cur[p];
  const long long o = y * c.sy + x * c.sx;
  if (c.dtype == VDO_DT_I64) {
    long long* t = (long long*)c.p + o;
    if (PASS == 1) *t = LLONG_MIN; else atomicMax(t, (long long)s_lab[s]);
  } else {
    int* t = (int*)c.p + o;
    if (PASS == 1) *t = INT_MIN; else atomicMax(t, s_lab[s]);
  }
}

__device__ __forceinline__ int block_sum(int v, int* s_red) {
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = 0;
  for (int k = 0; k < OM_THREADS / 32; ++k) t += s_red[k];
  __syncthreads();
  return t;
}

// One CTA per pair, the slots in ascending label order with the recovered set R.  Voter q of slot i reads the label of the highest slot in
// word(q) & R & (slots below i) -- the last of the earlier recoveries that wrote q -- or else the caller's mask at q, which nothing has written
// yet.  That is the mask the reference's loop reads at slot i.  An i64 current label outside int32 at any voter's target sets
// VDO_OM_PAIR_LABEL_RANGE and the pair recovers nothing.
__global__ void __launch_bounds__(OM_THREADS) k_um_vote(const __grid_constant__ ObjArg a, const __grid_constant__ MaskArg u, vdo_obj_motion_out o,
                                                        const int* __restrict__ ord) {
  __shared__ int wsum[33], s_beg[OM_MAX_OBJ + 1], s_lab[OM_MAX_OBJ], s_red[OM_THREADS / 32];
  __shared__ long long s_redl[OM_THREADS / 32];
  __shared__ int s_bad;
  const int p = blockIdx.x, tid = threadIdx.x;
  const ObjPair& q = a.pr[p];
  const PlaneArg& c = u.cur[p];
  const size_t off = (size_t)p * a.cap, row = (size_t)p * a.M;
  int* tab = u.tab + (size_t)p * u.tab_stride;
  const int nobj = tab[UM_NOBJ], hp = tab[UM_HP];
  const unsigned cand = (unsigned)tab[UM_CAND];
  const unsigned long long* key = u.key + (size_t)p * u.hs;
  const unsigned* word = u.word + (size_t)p * u.hs;
  if (tid <= nobj) s_beg[tid] = tab[tid];
  if (tid < nobj) s_lab[tid] = u.o.label_dev[row + tid];
  if (tid == 0) s_bad = 0;
  __syncthreads();
  if (c.dtype == VDO_DT_I64)
    for (int k = tid; k < s_beg[nobj]; k += OM_THREADS) {
      const int i = ord[off + k], x = (int)o.sample_cx_dev[off + i], y = (int)o.sample_cy_dev[off + i];
      if (um_inside(x, y, q.w, q.h)) { const long long v = cur_label(c, x, y); if (v < INT_MIN || v > INT_MAX) s_bad = 1; }
    }
  __syncthreads();
  const bool bad = s_bad;
  unsigned R = 0;
  for (int s = 0; s < nobj; ++s) {
    int vote = 0;
    if (!bad && (cand >> s & 1u)) {
      const unsigned below = R & ((1u << s) - 1u);
      int nv = 0;                                                 // compact the voters' current labels to vlab[off + s_beg[s] ..)
      for (int k0 = s_beg[s]; k0 < s_beg[s + 1]; k0 += OM_THREADS) {
        const int k = k0 + tid;
        int x = 0, y = 0, ok = 0;
        if (k < s_beg[s + 1]) {
          const int i = ord[off + k];
          x = (int)o.sample_cx_dev[off + i]; y = (int)o.sample_cy_dev[off + i];
          ok = um_inside(x, y, q.w, q.h);
        }
        int tot;
        const int pos = cta_excl_scan(ok, wsum, tot);
        if (ok) {
          const unsigned w = below ? word[um_find(key, hp, (unsigned long long)y * q.w + x)] & below : 0u;
          u.vlab[off + s_beg[s] + nv + pos] = w ? s_lab[31 - __clz(w)] : (int)cur_label(c, x, y);
        }
        nv += tot;
      }
      __syncthreads();
      // the majority: labels ascending by repeated minimum, the first with the largest count (majority_label's tie rule)
      const int* vl = u.vlab + off + s_beg[s];
      int best_n = -1;
      for (long long prev = LLONG_MIN;;) {
        long long mn = LLONG_MAX;
        for (int k = tid; k < nv; k += OM_THREADS) { const long long v = vl[k]; if (v > prev && v < mn) mn = v; }
        mn = block_min(mn, s_redl);
        if (mn == LLONG_MAX) break;
        int cnt = 0;
        for (int k = tid; k < nv; k += OM_THREADS) cnt += vl[k] == mn;
        cnt = block_sum(cnt, s_red);
        if (cnt > best_n) { best_n = cnt; vote = (int)mn; }
        prev = mn;
      }
      if (vote == 0) R |= 1u << s;
    }
    if (tid == 0) { u.o.vote_dev[row + s] = vote; u.o.recovered_dev[row + s] = R >> s & 1u; }
  }
  for (int s = nobj + tid; s < a.M; s += OM_THREADS) { u.o.vote_dev[row + s] = 0; u.o.recovered_dev[row + s] = 0; }
  if (tid == 0) {
    tab[UM_REC] = (int)R;
    if (bad) u.o.pair_status_dev[p] |= VDO_OM_PAIR_LABEL_RANGE;
  }
}

// ---- 9. vdo_obj_renew_batch_dev: the object half of RenewFrameInfo (Tracking.cc:2817-2991), one CTA per pair ----
// The reference walks its candidates one by one, but each accept / reject depends only on the candidate and on the keys of step 1, so
// every step is a split: a key per candidate (its bucket, or -1), the per-bucket ranks in visit order, and a placement.
struct RenewArg {
  vdo_obj_track_out t;            // the track call's result (read)
  vdo_obj_motion_out r;           // the current frame's raster samples (work space; k_om_sample's columns)
  vdo_obj_feat_set s;             // the renewed set (written)
  int* used;                      // P x cap: 1 at a raster position a key of step 1 sits on
  int max_obj;                    // MaxTrackPointOBJ
};

// The stable split of a sequence of n elements into K <= OM_MAX_OBJ buckets, one contiguous run of the sequence per thread.  key(v): the
// bucket of element v or -1; bucket b keeps its first quota(b) elements and lies after the kept elements of the buckets below it.
// emit(v, b, pos) for every kept element.  Returns the kept total.  All threads call it.
template <class Key, class Quota, class Emit>
__device__ __forceinline__ int rn_split(int n, int K, const Key& key, const Quota& quota, const Emit& emit, int (*s_cnt)[OM_THREADS], int* s_base) {
  const int tid = threadIdx.x, per = (n + OM_THREADS - 1) / OM_THREADS, i0 = min(n, tid * per), i1 = min(n, i0 + per);
  for (int b = 0; b < K; ++b) s_cnt[b][tid] = 0;
  for (int v = i0; v < i1; ++v) { const int b = key(v); if (b >= 0) ++s_cnt[b][tid]; }
  __syncthreads();
  if (tid < K) {
    int acc = 0;
    for (int t = 0; t < OM_THREADS; ++t) { const int c = s_cnt[tid][t]; s_cnt[tid][t] = acc; acc += c; }
    s_base[OM_MAX_OBJ + 1 + tid] = acc;
  }
  __syncthreads();
  if (tid == 0) { int b0 = 0; for (int b = 0; b < K; ++b) { s_base[b] = b0; b0 += min(s_base[OM_MAX_OBJ + 1 + b], quota(b)); } s_base[OM_MAX_OBJ] = b0; }
  __syncthreads();
  for (int v = i0; v < i1; ++v) {
    const int b = key(v);
    if (b >= 0) { const int r = s_cnt[b][tid]++; if (r < quota(b)) emit(v, b, s_base[b] + r); }
  }
  const int tot = s_base[OM_MAX_OBJ];
  __syncthreads();
  return tot;
}

// step 1's test of a carried LM inlier at last pixel (x0, y0) with refined flow (ux, uy) (:2841-2866): its key (x, y) and, when it is kept,
// the current label, depth and flow there
__device__ __forceinline__ bool rn_carried(const ObjPair& q, int x0, int y0, double ux, double uy, int& x, int& y, int& m, float& d, float2& f, int* bad) {
  x = (int)(float)((double)x0 + ux); y = (int)(float)((double)y0 + uy);       // mvObjKeys as the tracker updates it, then (int)
  if (x >= q.w || y >= q.h || x <= 0 || y <= 0) return false;
  m = plane_label(q.msk, x, y, bad); d = plane_depth(q.dep, x, y);
  if (!(m != 0 && d < 25.f && d > 0.f)) return false;                       // the depth bound is hard-coded in the reference
  f = plane_flow(q.flo, x, y);
  const float cx = __fadd_rn((float)x, f.x), cy = __fadd_rn((float)y, f.y);
  return cx < (float)q.w && cy < (float)q.h && cx > 0.f && cy > 0.f;
}
// position v of the visit order of the top-up (passes start = 0 .. 14, stride 15) over n samples -> the sample index
__device__ __forceinline__ int rn_visit(int v, int n) {
  const int q = n / 15, big = (n % 15) * (q + 1);                           // the first n % 15 passes visit q + 1 samples, the others q
  return v < big ? v / (q + 1) + 15 * (v % (q + 1)) : n % 15 + (v - big) / q + 15 * ((v - big) % q);
}
// index of v among the k ascending values of tab, or -1
__device__ __forceinline__ int rn_find(const int* tab, int k, long long v) {
  int lo = 0, hi = k;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (tab[mid] < v) lo = mid + 1; else hi = mid; }
  return lo < k && tab[lo] == v ? lo : -1;
}

__global__ void __launch_bounds__(OM_THREADS) k_rn_select(const __grid_constant__ ObjArg a, const __grid_constant__ RenewArg u, const int* __restrict__ pstat) {
  __shared__ int s_cnt[OM_MAX_OBJ][OM_THREADS];
  __shared__ int s_base[2 * OM_MAX_OBJ + 1];
  __shared__ int s_stat[OM_MAX_OBJ], s_id[OM_MAX_OBJ], s_fea[OM_MAX_OBJ];
  __shared__ int s_known[OM_MAX_OBJ], s_blab[OM_MAX_OBJ], s_bslot[OM_MAX_OBJ];   // stat slots' labels; a split's bucket labels and slots
  __shared__ int s_nknown, s_nb, s_bad;
  __shared__ long long s_red[OM_THREADS / 32];
  __shared__ float s_Twc[16];
  const int p = blockIdx.x, tid = threadIdx.x, M = a.M, C = a.cap, step = a.step;
  const ObjPair& q = a.pr[p];
  const vdo_obj_motion_out& o = u.t.motion;
  const vdo_obj_motion_out& r = u.r;
  const vdo_obj_feat_set& s = u.s;
  const size_t off = (size_t)p * C, row = (size_t)p * M;
  const int n1 = o.n_samples_dev[p], nr = r.n_samples_dev[p], nx = (q.w + step - 1) / step, npos = nx * ((q.h + step - 1) / step);
  if (tid < M) { s_stat[tid] = u.t.stat_dev[row + tid]; s_id[tid] = u.t.id_dev[row + tid]; }
  if (tid == 0) {
    float Tc[16];
    load_pose(a.Tc, p, Tc);
    inv4(Tc, s_Twc);                                                        // Converter::toInvMatrix(Tcw_cur)
    s_bad = 0;
  }
  for (int k = tid; k < npos; k += OM_THREADS) u.used[off + k] = 0;
  __syncthreads();
  if (tid == 0) {
    int nk = 0;
    for (int j = 0; j < M; ++j) if (s_stat[j]) s_known[nk++] = o.label_dev[row + j];   // slots hold ascending labels
    s_nknown = nk;
  }
  // one row of the set; rows past C are dropped.  point: Optimizer::Get3DinWorld (tracking_ops.cu get3d_world's rounding)
  auto put = [&](int pos, int x, int y, int m, float d, float cx, float cy, float fx, float fy, int inl, int lab) {
    if (pos >= C) return;
    const size_t i = off + pos;
    s.x_dev[i] = x; s.y_dev[i] = y; s.label_dev[i] = m; s.depth_dev[i] = d; s.cx_dev[i] = cx; s.cy_dev[i] = cy;
    s.flow_dev[2 * i] = fx; s.flow_dev[2 * i + 1] = fy; s.inlier_id_dev[i] = inl; s.obj_label_dev[i] = lab;
    const float invfx = 1.0f / q.K[0], invfy = 1.0f / q.K[1];
    const float X = ((float)x - q.K[2]) * d * invfx, Y = ((float)y - q.K[3]) * d * invfy;
    for (int c = 0; c < 3; ++c)
      s.point_dev[3 * i + c] = (float)((double)s_Twc[4 * c] * (double)X + (double)s_Twc[4 * c + 1] * (double)Y + (double)s_Twc[4 * c + 2] * (double)d +
                                       (double)s_Twc[4 * c + 3]);
  };
  const auto all = [](int) { return INT_MAX; };
  // 1. the LM inliers of the stat slots, slot by slot, in row order
  const auto key1 = [&](int k) {
    const size_t i = off + k;
    const int sl = o.sample_slot_dev[i];
    if (sl < 0 || !s_stat[sl] || !(o.sample_flags_dev[i] & 2)) return -1;
    int x, y, m; float d; float2 f;
    return rn_carried(q, o.sample_x_dev[i], o.sample_y_dev[i], o.sample_flow_ref_dev[2 * i], o.sample_flow_ref_dev[2 * i + 1], x, y, m, d, f, &s_bad) ? sl : -1;
  };
  const auto emit1 = [&](int k, int, int pos) {
    const size_t i = off + k;
    int x, y, m; float d; float2 f;
    rn_carried(q, o.sample_x_dev[i], o.sample_y_dev[i], o.sample_flow_ref_dev[2 * i], o.sample_flow_ref_dev[2 * i + 1], x, y, m, d, f, &s_bad);
    put(pos, x, y, m, d, __fadd_rn((float)x, f.x), __fadd_rn((float)y, f.y), f.x, f.y, k, u.t.obj_label_dev[i]);
    if (x % step == 0 && y % step == 0) u.used[off + (y / step) * nx + x / step] = 1;   // the only keys a raster sample can sit on
  };
  const int c1 = rn_split(n1, M, key1, all, emit1, s_cnt, s_base);
  // 2. the top-up of each stat slot short of max_obj rows: its label's raster samples in the stride-15 passes, not on a key of 1
  if (tid < M) s_fea[tid] = s_base[OM_MAX_OBJ + 1 + tid];
  __syncthreads();
  if (tid == 0) {
    int nb = 0;
    for (int j = 0; j < M; ++j)
      if (s_stat[j] && s_fea[j] < u.max_obj) { s_blab[nb] = o.label_dev[row + j]; s_bslot[nb++] = j; }
    s_nb = nb;
  }
  __syncthreads();
  const auto key2 = [&](int v) {
    const int j = rn_visit(v, nr);
    const size_t i = off + j;
    const int b = rn_find(s_blab, s_nb, r.sample_label_dev[i]);
    return b >= 0 && !u.used[off + (r.sample_y_dev[i] / step) * nx + r.sample_x_dev[i] / step] ? b : -1;
  };
  const auto quota2 = [&](int b) { return u.max_obj - s_fea[s_bslot[b]]; };
  const auto emit2 = [&](int v, int b, int pos) {
    const size_t i = off + rn_visit(v, nr);
    put(c1 + pos, r.sample_x_dev[i], r.sample_y_dev[i], r.sample_label_dev[i], r.sample_depth_dev[i], r.sample_cx_dev[i], r.sample_cy_dev[i],
        r.sample_flow_dev[2 * i], r.sample_flow_dev[2 * i + 1], -1, s_id[s_bslot[b]]);
  };
  int tot = c1 + rn_split(nr, s_nb, key2, quota2, emit2, s_cnt, s_base);
  // 3. the labels that are no stat slot's, ascending, OM_MAX_OBJ at a time: all their raster samples in raster order
  const int nknown = s_nknown;
  for (long long prev = LLONG_MIN;;) {
    int nb = 0;
    for (; nb < OM_MAX_OBJ; ++nb) {
      long long mn = LLONG_MAX;
      for (int j = tid; j < nr; j += OM_THREADS) {
        const long long v = r.sample_label_dev[off + j];
        if (v > prev && v < mn && rn_find(s_known, nknown, v) < 0) mn = v;
      }
      mn = block_min(mn, s_red);
      if (mn == LLONG_MAX) break;
      if (tid == 0) s_blab[nb] = (int)mn;
      prev = mn;
    }
    __syncthreads();
    if (nb == 0) break;
    const auto key3 = [&](int j) { return rn_find(s_blab, nb, r.sample_label_dev[off + j]); };
    const auto emit3 = [&](int j, int, int pos) {
      const size_t i = off + j;
      put(tot + pos, r.sample_x_dev[i], r.sample_y_dev[i], r.sample_label_dev[i], r.sample_depth_dev[i], r.sample_cx_dev[i], r.sample_cy_dev[i],
          r.sample_flow_dev[2 * i], r.sample_flow_dev[2 * i + 1], -1, -2);
    };
    tot += rn_split(nr, nb, key3, all, emit3, s_cnt, s_base);
    if (nb < OM_MAX_OBJ) break;
  }
  if (tid == 0) {
    const bool bad = s_bad || (pstat[p] & VDO_OM_PAIR_LABEL_RANGE);
    s.count_dev[p] = bad ? -1 : min(tot, C);
    s.status_dev[p] = bad ? VDO_OM_PAIR_LABEL_RANGE : tot > C ? VDO_OM_PAIR_FEATURE_CAP : 0;
  }
}

}  // namespace

// ---- vdo_obj_motion: the work space of vdo_obj_motion_batch_dev, all allocated at creation ----
struct vdo_obj_motion : vdo::WorkSpace {
  vdo_ctx* ctx = nullptr;
  int dev = 0, max_pairs = 0, max_objects = 0, cap = 0;
  int* pstat = nullptr;                                                 // max_pairs
  int* ord = nullptr;                                                   // max_pairs x cap: sample index of each object point
  int* glab = nullptr;                                                  // max_pairs x cap: vdo_obj_track_batch_dev's grouping label
  float *obj = nullptr, *img = nullptr;                                 // world points, observations
  int *r_idx = nullptr, *m_idx = nullptr, *s_idx = nullptr;
  int *samples = nullptr, *counts = nullptr;                            // slots x VDO_OBJ_MOTION_MAX_ITERS (x 4)
  double* models = nullptr;
  PnpProb* prob = nullptr;                                              // slots
  PnpOut* res = nullptr;
  FlowProb* fprob = nullptr;
  float *pts = nullptr, *depth = nullptr, *flow = nullptr;              // LM inputs at the slots' offsets
  double *flow_res = nullptr, *scratch = nullptr;                       // scratch: max_pairs x cap x FL_FIELDS, only when cap > the cluster limit
  unsigned char* inl = nullptr;
};

extern "C" int vdo_obj_motion_create(vdo_ctx* ctx, int max_pairs, int max_objects, int cap, vdo_obj_motion** out) {
  if (!ctx || !out) return VDO_ERR_ARG;
  *out = nullptr;
  if (max_pairs < 1 || max_pairs > OM_MAX_PAIRS || max_objects < 1 || max_objects > OM_MAX_OBJ || cap < 1 || (int64_t)max_pairs * cap > INT_MAX) {
    vdo::ctx_set_error(ctx, "vdo_obj_motion_create: max_pairs = " + std::to_string(max_pairs) + ", max_objects = " + std::to_string(max_objects) +
                                ", cap = " + std::to_string(cap) + "; expected 1 .. 64, 1 .. 32 and >= 1, with max_pairs x cap below 2^31");
    return VDO_ERR_ARG;
  }
  vdo_obj_motion* m = new vdo_obj_motion;
  m->ctx = ctx; m->max_pairs = max_pairs; m->max_objects = max_objects; m->cap = cap;
  int n_sm = 0;
  vdo::ctx_device(ctx, &m->dev, &n_sm);
  const size_t pts = (size_t)max_pairs * cap, slots = (size_t)max_pairs * max_objects, hyp = slots * VDO_OBJ_MOTION_MAX_ITERS;
  return vdo::create_done(ctx, "vdo_obj_motion_create", m,
                          {m->alloc(m->pstat, (size_t)max_pairs), m->alloc(m->ord, pts), m->alloc(m->obj, 3 * pts), m->alloc(m->img, 2 * pts),
                           m->alloc(m->r_idx, pts), m->alloc(m->m_idx, pts), m->alloc(m->s_idx, pts), m->alloc(m->samples, 4 * hyp),
                           m->alloc(m->counts, hyp), m->alloc(m->models, 12 * hyp), m->alloc(m->prob, slots), m->alloc(m->res, slots),
                           m->alloc(m->fprob, slots), m->alloc(m->pts, 2 * pts), m->alloc(m->depth, pts), m->alloc(m->flow, 2 * pts),
                           m->alloc(m->flow_res, 2 * pts), m->alloc(m->inl, pts), m->alloc(m->glab, pts),
                           cap > VDO_FLOW2_CLUSTER_MAX_N ? m->alloc(m->scratch, pts * vdo::flow_lm_fields()) : cudaSuccess, vdo::flow_lm_prepare()},
                          out);
}
extern "C" void vdo_obj_motion_destroy(vdo_obj_motion* m) { delete m; }
extern "C" int vdo_obj_motion_info(const vdo_obj_motion* m, int64_t out[4]) {
  if (!m || !out) return VDO_ERR_ARG;
  out[0] = m->max_pairs; out[1] = m->max_objects; out[2] = m->cap; out[3] = (int64_t)m->bytes;
  return VDO_OK;
}

namespace {
// the option checks of both entries, in order: "" or the refusal
std::string om_check_opts(const vdo_obj_motion_opts& o) {
  if (o.step < 1) return "step = " + std::to_string(o.step) + "; expected >= 1";
  if (std::isnan(o.th_depth_obj)) return "th_depth_obj is NaN";
  if (o.iters < 1 || o.iters > VDO_OBJ_MOTION_MAX_ITERS) return "iters = " + std::to_string(o.iters) + " outside 1 .. " + std::to_string(VDO_OBJ_MOTION_MAX_ITERS);
  if (!(o.thr > 0.0)) return "thr = " + std::to_string(o.thr) + "; expected > 0";
  if (!(o.conf > 0.0 && o.conf < 1.0)) return "conf = " + std::to_string(o.conf) + "; expected inside (0, 1)";
  if (o.min_inliers < 0) return "min_inliers = " + std::to_string(o.min_inliers) + "; expected >= 0";
  if (o.quirk != 0 && o.quirk != 1) return "quirk = " + std::to_string(o.quirk) + "; expected 0 or 1";
  return "";
}

// the checks of pair p's size and last planes: "" or the refusal; fills a.pr[p], max_n and the planes' entries of ptrs
std::string om_check_pair(const vdo_obj_motion* m, int p, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask, const int32_t* wh,
                          const float* K, int step, ObjArg& a, int& max_n, vdo::DevPtrs& ptrs) {
  const std::string who = "pair " + std::to_string(p) + ": ";
  const int w = wh[2 * p], h = wh[2 * p + 1];
  if (w < 1 || h < 1) return who + std::to_string(w) + " x " + std::to_string(h) + "; expected a width and height >= 1";
  const int64_t n = (int64_t)((w + step - 1) / step) * ((h + step - 1) / step);
  if (n > m->cap) return who + std::to_string(n) + " sample positions exceed the estimator's cap " + std::to_string(m->cap);
  max_n = std::max(max_n, (int)n);
  const vdo_dev_plane* pl[3] = {&depth[p], &flow[p], &mask[p]};
  static const char* kName[3] = {"depth", "flow", "mask"};
  for (int k = 0; k < 3; ++k) {
    const int dt = pl[k]->dtype, ch = pl[k]->channels;
    const bool ok = k == 0 ? dt == VDO_DT_F32 && ch == 1 : k == 1 ? dt == VDO_DT_F32 && ch == 2 : (dt == VDO_DT_I32 || dt == VDO_DT_I64) && ch == 1;
    static const char* kWant[3] = {"f32 with 1 channel", "f32 with 2 channels", "i32 or i64 with 1 channel"};
    if (!ok) return who + kName[k] + " plane: dtype " + std::to_string(dt) + " with " + std::to_string(ch) + " channels; expected " + kWant[k];
    ptrs.push_back({pl[k]->data_dev, size_t(dt == VDO_DT_I64 ? 8 : 4), who + kName[k] + " plane data_dev"});
  }
  ObjPair& q = a.pr[p];
  q.dep = plane_arg(&depth[p]); q.flo = plane_arg(&flow[p]); q.msk = plane_arg(&mask[p]); q.w = w; q.h = h;
  for (int c = 0; c < 4; ++c) q.K[c] = K[4 * p + c];
  return "";
}

void om_out_ptrs(const vdo_obj_motion_out& u, vdo::DevPtrs& ptrs) {
  ptrs.insert(ptrs.end(), {{u.label_dev, 4, "out.label_dev"}, {u.H_dev, 4, "out.H_dev"}, {u.X_dev, 4, "out.X_dev"}, {u.T_init_dev, 4, "out.T_init_dev"},
                           {u.centre_dev, 4, "out.centre_dev"}, {u.velocity_dev, 4, "out.velocity_dev"}, {u.info_dev, 4, "out.info_dev"},
                           {u.stats_dev, 8, "out.stats_dev"}, {u.status_dev, 4, "out.status_dev"}, {u.sample_x_dev, 4, "out.sample_x_dev"},
                           {u.sample_y_dev, 4, "out.sample_y_dev"}, {u.sample_label_dev, 4, "out.sample_label_dev"},
                           {u.sample_slot_dev, 4, "out.sample_slot_dev"}, {u.sample_depth_dev, 4, "out.sample_depth_dev"},
                           {u.sample_cx_dev, 4, "out.sample_cx_dev"}, {u.sample_cy_dev, 4, "out.sample_cy_dev"},
                           {u.sample_flow_dev, 4, "out.sample_flow_dev"}, {u.sample_flow_ref_dev, 8, "out.sample_flow_ref_dev"},
                           {u.sample_flags_dev, 1, "out.sample_flags_dev"}, {u.n_samples_dev, 4, "out.n_samples_dev"},
                           {u.pair_status_dev, 4, "out.pair_status_dev"}});
}

// the launches after the grouping, shared by both entries: RANSAC, the gate, the LM and the per-slot outputs
void om_solve(vdo_obj_motion* m, const ObjArg& a, const vdo_obj_motion_out& u, const vdo_obj_motion_opts& o, int nprob, int max_n, cudaStream_t st) {
  vdo::pnp_samples_launch(m->prob, nprob, o.iters, m->samples, st);
  vdo::pnp_ransac_launch(m->prob, nprob, m->obj, m->img, m->samples, o.iters, o.thr, o.conf, m->models, m->counts, m->res, m->r_idx, m->m_idx, m->s_idx, st);
  k_om_lm_prep<<<nprob, OM_THREADS, 0, st>>>(a, u, m->prob, m->res, m->s_idx, m->ord, m->pts, m->depth, m->flow, m->fprob);
  const FlowDev d{m->fprob, m->pts, m->depth, m->flow, m->scratch, u.X_dev, m->flow_res, m->inl, u.stats_dev, o.quirk, 0, nullptr};
  vdo::flow_lm_launch(d, nprob, max_n, st);
  k_om_finish<<<nprob, OM_THREADS, 0, st>>>(a, u, m->prob, m->res, m->s_idx, m->ord, m->flow_res, m->inl);
}
}  // namespace

extern "C" int vdo_obj_motion_batch_dev(vdo_obj_motion* m, int P, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
                                        const int32_t* wh, const float* K, const float* Tcw_last_dev, const float* Tcw_cur_dev,
                                        const int32_t* prev_label_dev, const float* prev_H_dev, const vdo_obj_motion_opts* opts,
                                        const vdo_obj_motion_out* out, uint64_t stream) {
  if (!m) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(m->ctx, "vdo_obj_motion_batch_dev: " + s); return VDO_ERR_ARG; };
  if (P < 1 || P > m->max_pairs) return refuse("P = " + std::to_string(P) + " outside 1 .. " + std::to_string(m->max_pairs));
  if (!depth || !flow || !mask || !wh || !K || !opts || !out) return refuse("depth, flow, mask, wh, K, opts or out is NULL");
  const vdo_obj_motion_opts& o = *opts;
  if (std::string why = om_check_opts(o); !why.empty()) return refuse(why);
  if (!prev_label_dev != !prev_H_dev) return refuse("prev_label_dev and prev_H_dev must both be given or both be NULL");
  ObjArg a;
  std::memset(&a, 0, sizeof a);
  int max_n = 0;
  vdo::DevPtrs ptrs;
  for (int p = 0; p < P; ++p)
    if (std::string why = om_check_pair(m, p, depth, flow, mask, wh, K, o.step, a, max_n, ptrs); !why.empty()) return refuse(why);
  const vdo_obj_motion_out& u = *out;
  ptrs.insert(ptrs.end(), {{Tcw_last_dev, 4, "Tcw_last_dev", Tcw_last_dev != nullptr}, {Tcw_cur_dev, 4, "Tcw_cur_dev", Tcw_cur_dev != nullptr},
                           {prev_label_dev, 4, "prev_label_dev", prev_label_dev != nullptr}, {prev_H_dev, 4, "prev_H_dev", prev_H_dev != nullptr}});
  om_out_ptrs(u, ptrs);
  if (std::string why = vdo::check_ptrs(ptrs, m->dev); !why.empty()) return refuse(why);
  a.Tl = Tcw_last_dev; a.Tc = Tcw_cur_dev; a.prev_label = prev_label_dev; a.prev_H = prev_H_dev;
  a.step = o.step; a.cap = m->cap; a.M = m->max_objects; a.min_inliers = o.min_inliers; a.th = o.th_depth_obj;
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  k_om_sample<<<P, OM_SAMPLE_THREADS, 0, st>>>(a, u, m->pstat);
  k_om_group<<<P, OM_THREADS, 0, st>>>(a, u, m->pstat, m->ord, m->obj, m->img, m->prob);
  om_solve(m, a, u, o, P * m->max_objects, max_n, st);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}

namespace {
// the set fields the *_set entries read, checked into ptrs; an empty SetArg without a set
SetArg set_arg(const vdo_obj_feat_set* s, vdo::DevPtrs& ptrs) {
  if (!s) return SetArg{};
  ptrs.insert(ptrs.end(), {{s->x_dev, 4, "last.x_dev"}, {s->y_dev, 4, "last.y_dev"}, {s->label_dev, 4, "last.label_dev"}, {s->depth_dev, 4, "last.depth_dev"},
                           {s->cx_dev, 4, "last.cx_dev"}, {s->cy_dev, 4, "last.cy_dev"}, {s->flow_dev, 4, "last.flow_dev"}, {s->count_dev, 4, "last.count_dev"}});
  return SetArg{s->x_dev, s->y_dev, s->label_dev, s->count_dev, s->depth_dev, s->cx_dev, s->cy_dev, s->flow_dev};
}

// vdo_obj_track_batch_dev (last NULL) and vdo_obj_track_set_batch_dev
int obj_track(const char* fn, bool with_set, vdo_obj_motion* m, int P, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
              const vdo_dev_plane* depth_cur, const vdo_dev_plane* mask_cur, const int32_t* wh, const float* K, const float* Tcw_last_dev,
              const float* Tcw_cur_dev, const int32_t* prev_label_dev, const int32_t* prev_id_dev, const int32_t* prev_stat_dev, const float* prev_H_dev,
              const int32_t* prev_max_id_dev, const vdo_obj_feat_set* last, const vdo_obj_track_opts* opts, const vdo_obj_track_out* out, uint64_t stream) {
  if (!m) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(m->ctx, std::string(fn) + ": " + s); return VDO_ERR_ARG; };
  if (P < 1 || P > m->max_pairs) return refuse("P = " + std::to_string(P) + " outside 1 .. " + std::to_string(m->max_pairs));
  if (!depth || !flow || !mask || !depth_cur || !mask_cur || !wh || !K || !opts || !out)
    return refuse("depth, flow, mask, depth_cur, mask_cur, wh, K, opts or out is NULL");
  if (with_set && !last) return refuse("last is NULL");
  const vdo_obj_track_opts& to = *opts;
  const vdo_obj_motion_opts o{to.step, to.th_depth_obj, to.iters, to.min_inliers, to.thr, to.conf, to.quirk, 0};
  if (std::string why = om_check_opts(o); !why.empty()) return refuse(why);
  if (std::isnan(to.sf_mg_thres) || std::isnan(to.sf_ds_thres)) return refuse("sf_mg_thres or sf_ds_thres is NaN");
  if (to.shrink_row < 0 || to.shrink_col < 0)
    return refuse("shrink_row = " + std::to_string(to.shrink_row) + ", shrink_col = " + std::to_string(to.shrink_col) + "; expected >= 0");
  const int n_prev = !!prev_label_dev + !!prev_id_dev + !!prev_stat_dev + !!prev_H_dev + !!prev_max_id_dev;
  if (n_prev != 0 && n_prev != 5) return refuse("prev_label_dev, prev_id_dev, prev_stat_dev, prev_H_dev and prev_max_id_dev must all be given or all be NULL");
  ObjArg a;
  std::memset(&a, 0, sizeof a);
  int max_n = 0;
  vdo::DevPtrs ptrs;
  for (int p = 0; p < P; ++p) {
    if (std::string why = om_check_pair(m, p, depth, flow, mask, wh, K, o.step, a, max_n, ptrs); !why.empty()) return refuse(why);
    const std::string who = "pair " + std::to_string(p) + ": ";
    if (depth_cur[p].dtype != VDO_DT_F32 || depth_cur[p].channels != 1) return refuse(who + "depth_cur plane: expected f32 with 1 channel");
    if ((mask_cur[p].dtype != VDO_DT_I32 && mask_cur[p].dtype != VDO_DT_I64) || mask_cur[p].channels != 1)
      return refuse(who + "mask_cur plane: expected i32 or i64 with 1 channel");
    ptrs.push_back({depth_cur[p].data_dev, 4, who + "depth_cur plane data_dev"});
    ptrs.push_back({mask_cur[p].data_dev, size_t(mask_cur[p].dtype == VDO_DT_I64 ? 8 : 4), who + "mask_cur plane data_dev"});
  }
  const vdo_obj_track_out& u = *out;
  ptrs.insert(ptrs.end(), {{Tcw_last_dev, 4, "Tcw_last_dev", Tcw_last_dev != nullptr}, {Tcw_cur_dev, 4, "Tcw_cur_dev", Tcw_cur_dev != nullptr},
                           {prev_label_dev, 4, "prev_label_dev", n_prev > 0}, {prev_id_dev, 4, "prev_id_dev", n_prev > 0},
                           {prev_stat_dev, 4, "prev_stat_dev", n_prev > 0}, {prev_H_dev, 4, "prev_H_dev", n_prev > 0},
                           {prev_max_id_dev, 4, "prev_max_id_dev", n_prev > 0}});
  om_out_ptrs(u.motion, ptrs);
  ptrs.insert(ptrs.end(), {{u.id_dev, 4, "out.id_dev"}, {u.cls_dev, 4, "out.cls_dev"}, {u.vote_dev, 4, "out.vote_dev"}, {u.stat_dev, 4, "out.stat_dev"},
                           {u.label_cur_dev, 4, "out.label_cur_dev"}, {u.depth_cur_dev, 4, "out.depth_cur_dev"}, {u.flow3d_dev, 4, "out.flow3d_dev"},
                           {u.obj_label_dev, 4, "out.obj_label_dev"}, {u.max_id_dev, 4, "out.max_id_dev"}});
  const SetArg sa = set_arg(with_set ? last : nullptr, ptrs);
  if (std::string why = vdo::check_ptrs(ptrs, m->dev); !why.empty()) return refuse(why);
  a.Tl = Tcw_last_dev; a.Tc = Tcw_cur_dev; a.prev_label = prev_label_dev; a.prev_H = prev_H_dev;
  a.step = o.step; a.cap = m->cap; a.M = m->max_objects; a.min_inliers = o.min_inliers; a.th = o.th_depth_obj;
  const TrackArg t{prev_id_dev, prev_stat_dev, prev_max_id_dev, to.sf_mg_thres, to.sf_ds_thres, to.shrink_row, to.shrink_col};
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  if (with_set) {
    k_os_sample<<<P, OM_SAMPLE_THREADS, 0, st>>>(a, sa, u.motion, m->pstat);
    max_n = m->cap;                                                     // a carried set may hold up to cap samples
  } else {
    k_om_sample<<<P, OM_SAMPLE_THREADS, 0, st>>>(a, u.motion, m->pstat);
  }
  vdo::obj_track_flow_launch(P, depth_cur, mask_cur, wh, K, Tcw_last_dev, Tcw_cur_dev, m->cap, max_n, o.th_depth_obj, u, m->pstat, m->glab, stream);
  k_ot_group<<<P, OM_THREADS, 0, st>>>(a, t, u, m->pstat, m->glab, m->ord, m->obj, m->img, m->prob);
  om_solve(m, a, u.motion, o, P * m->max_objects, max_n, st);
  k_ot_finish<<<P, OM_THREADS, 0, st>>>(a, u, m->glab);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
}  // namespace

extern "C" int vdo_obj_track_batch_dev(vdo_obj_motion* m, int P, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
                                       const vdo_dev_plane* depth_cur, const vdo_dev_plane* mask_cur, const int32_t* wh, const float* K,
                                       const float* Tcw_last_dev, const float* Tcw_cur_dev, const int32_t* prev_label_dev, const int32_t* prev_id_dev,
                                       const int32_t* prev_stat_dev, const float* prev_H_dev, const int32_t* prev_max_id_dev,
                                       const vdo_obj_track_opts* opts, const vdo_obj_track_out* out, uint64_t stream) {
  return obj_track("vdo_obj_track_batch_dev", false, m, P, depth, flow, mask, depth_cur, mask_cur, wh, K, Tcw_last_dev, Tcw_cur_dev, prev_label_dev,
                   prev_id_dev, prev_stat_dev, prev_H_dev, prev_max_id_dev, nullptr, opts, out, stream);
}
extern "C" int vdo_obj_track_set_batch_dev(vdo_obj_motion* m, int P, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
                                           const vdo_dev_plane* depth_cur, const vdo_dev_plane* mask_cur, const int32_t* wh, const float* K,
                                           const float* Tcw_last_dev, const float* Tcw_cur_dev, const int32_t* prev_label_dev, const int32_t* prev_id_dev,
                                           const int32_t* prev_stat_dev, const float* prev_H_dev, const int32_t* prev_max_id_dev,
                                           const vdo_obj_feat_set* last, const vdo_obj_track_opts* opts, const vdo_obj_track_out* out, uint64_t stream) {
  return obj_track("vdo_obj_track_set_batch_dev", true, m, P, depth, flow, mask, depth_cur, mask_cur, wh, K, Tcw_last_dev, Tcw_cur_dev, prev_label_dev,
                   prev_id_dev, prev_stat_dev, prev_H_dev, prev_max_id_dev, last, opts, out, stream);
}

namespace {
// the byte range [lo, hi) a plane's w x h pixels (and channels) can touch
struct ByteRange { __int128 lo, hi; };
ByteRange plane_bytes(const vdo_dev_plane& pl, int w, int h) {
  const __int128 e = pl.dtype == VDO_DT_I64 ? 8 : pl.dtype == VDO_DT_U8 ? 1 : 4;
  __int128 lo = 0, hi = 0;
  const __int128 ext[3] = {(__int128)(w - 1) * pl.stride_x, (__int128)(h - 1) * pl.stride_y, (__int128)(pl.channels - 1) * pl.stride_c};
  for (const __int128 v : ext) { lo += v < 0 ? v : 0; hi += v > 0 ? v : 0; }
  const __int128 base = (__int128)(uintptr_t)pl.data_dev;
  return {base + lo * e, base + (hi + 1) * e};
}
// w x h pixels at element strides (sy, sx) are distinct elements when one axis steps at least 1 and the other at least its whole extent
bool distinct_pixels(const vdo_dev_plane& pl, int w, int h) {
  const unsigned long long ax = pl.stride_x < 0 ? 0ull - (unsigned long long)pl.stride_x : (unsigned long long)pl.stride_x;
  const unsigned long long ay = pl.stride_y < 0 ? 0ull - (unsigned long long)pl.stride_y : (unsigned long long)pl.stride_y;
  return (ax >= 1 && ay / (unsigned long long)w >= ax) || (ay >= 1 && ax / (unsigned long long)h >= ay);
}

// vdo_obj_update_mask_batch_dev (last NULL) and vdo_obj_update_mask_set_batch_dev
int obj_update_mask(const char* fn, bool with_set, vdo_obj_motion* m, int P, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
                    const vdo_dev_plane* mask_cur, const int32_t* wh, int32_t step, float th_depth_obj, const vdo_obj_feat_set* last,
                    const vdo_obj_mask_out* out, uint64_t stream) {
  if (!m) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(m->ctx, std::string(fn) + ": " + s); return VDO_ERR_ARG; };
  if (P < 1 || P > m->max_pairs) return refuse("P = " + std::to_string(P) + " outside 1 .. " + std::to_string(m->max_pairs));
  if (!depth || !flow || !mask || !mask_cur || !wh || !out) return refuse("depth, flow, mask, mask_cur, wh or out is NULL");
  if (with_set && !last) return refuse("last is NULL");
  const vdo_obj_motion_opts o{step, th_depth_obj, 1, 0, 1.0, 0.5, 0, 0};     // only step and th_depth_obj are used
  if (std::string why = om_check_opts(o); !why.empty()) return refuse(why);
  static const float kNoK[4 * OM_MAX_PAIRS] = {};                             // the samples need no intrinsics
  ObjArg a;
  std::memset(&a, 0, sizeof a);
  MaskArg u;
  std::memset(&u, 0, sizeof u);
  int max_n = 0;
  int64_t max_px = 0;
  vdo::DevPtrs ptrs;
  for (int p = 0; p < P; ++p) {
    if (std::string why = om_check_pair(m, p, depth, flow, mask, wh, kNoK, step, a, max_n, ptrs); !why.empty()) return refuse(why);
    const std::string who = "pair " + std::to_string(p) + ": ";
    const vdo_dev_plane& c = mask_cur[p];
    if ((c.dtype != VDO_DT_I32 && c.dtype != VDO_DT_I64) || c.channels != 1) return refuse(who + "mask_cur plane: expected i32 or i64 with 1 channel");
    if (!distinct_pixels(c, wh[2 * p], wh[2 * p + 1]))
      return refuse(who + "mask_cur plane: strides (" + std::to_string(c.stride_y) + ", " + std::to_string(c.stride_x) + ") do not map its " +
                    std::to_string(wh[2 * p]) + " x " + std::to_string(wh[2 * p + 1]) + " pixels to distinct elements");
    ptrs.push_back({c.data_dev, size_t(c.dtype == VDO_DT_I64 ? 8 : 4), who + "mask_cur plane data_dev"});
    u.cur[p] = plane_arg(&c);
    max_px = std::max(max_px, (int64_t)wh[2 * p] * wh[2 * p + 1]);
  }
  // mask_cur is written: it may share no byte with any plane of the call (pairs are independent; consecutive frames go in consecutive calls)
  for (int p = 0; p < P; ++p) {
    const ByteRange c = plane_bytes(mask_cur[p], wh[2 * p], wh[2 * p + 1]);
    for (int r = 0; r < P; ++r) {
      const vdo_dev_plane* pl[4] = {&depth[r], &flow[r], &mask[r], &mask_cur[r]};
      static const char* kName[4] = {"depth", "flow", "mask", "mask_cur"};
      for (int k = 0; k < 4; ++k) {
        if (k == 3 && r == p) continue;
        const ByteRange b = plane_bytes(*pl[k], wh[2 * r], wh[2 * r + 1]);
        if (c.lo < b.hi && b.lo < c.hi)
          return refuse("pair " + std::to_string(p) + ": mask_cur plane overlaps the " + kName[k] + " plane of pair " + std::to_string(r));
      }
    }
  }
  const vdo_obj_mask_out& uo = *out;
  ptrs.insert(ptrs.end(), {{uo.label_dev, 4, "out.label_dev"}, {uo.n_vote_dev, 4, "out.n_vote_dev"}, {uo.vote_dev, 4, "out.vote_dev"},
                           {uo.recovered_dev, 4, "out.recovered_dev"}, {uo.n_samples_dev, 4, "out.n_samples_dev"},
                           {uo.pair_status_dev, 4, "out.pair_status_dev"}});
  const SetArg sa = set_arg(with_set ? last : nullptr, ptrs);
  if (std::string why = vdo::check_ptrs(ptrs, m->dev); !why.empty()) return refuse(why);
  a.step = step; a.cap = m->cap; a.M = m->max_objects; a.th = th_depth_obj;
  // the idle work space of the RANSAC and the LM: the samples (k_om_sample's and group_sort's per-sample arrays), the hashes in obj (as 64-bit
  // keys) and img (words), the tables in the RANSAC counters, the voters' labels in glab
  const size_t pts = (size_t)m->max_pairs * m->cap;
  vdo_obj_motion_out so;
  std::memset(&so, 0, sizeof so);
  so.sample_x_dev = m->r_idx; so.sample_y_dev = m->m_idx; so.sample_label_dev = m->s_idx; so.sample_depth_dev = m->depth;
  so.sample_cx_dev = m->pts; so.sample_cy_dev = m->pts + pts; so.sample_flow_dev = m->flow; so.sample_slot_dev = m->glab;
  so.sample_flow_ref_dev = m->flow_res; so.sample_flags_dev = m->inl; so.n_samples_dev = uo.n_samples_dev;
  u.key = (unsigned long long*)m->obj; u.word = (unsigned*)m->img; u.hs = (int)(3 * (size_t)m->cap / 2);
  u.tab = m->counts; u.tab_stride = m->max_objects * VDO_OBJ_MOTION_MAX_ITERS;
  u.vlab = m->glab;
  u.o = uo;
  static_assert(UM_TAB <= VDO_OBJ_MOTION_MAX_ITERS, "a pair's table fits in its RANSAC counters");
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const dim3 px((unsigned)((max_px + OM_THREADS - 1) / OM_THREADS), (unsigned)P);
  if (with_set) k_os_sample<<<P, OM_SAMPLE_THREADS, 0, st>>>(a, sa, so, m->pstat);
  else k_om_sample<<<P, OM_SAMPLE_THREADS, 0, st>>>(a, so, m->pstat);
  k_um_group<<<P, OM_THREADS, 0, st>>>(a, u, so, m->pstat, m->ord);
  k_um_pixels<0><<<px, OM_THREADS, 0, st>>>(a, u);
  k_um_vote<<<P, OM_THREADS, 0, st>>>(a, u, so, m->ord);
  k_um_pixels<1><<<px, OM_THREADS, 0, st>>>(a, u);
  k_um_pixels<2><<<px, OM_THREADS, 0, st>>>(a, u);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
}  // namespace

extern "C" int vdo_obj_update_mask_batch_dev(vdo_obj_motion* m, int P, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
                                             const vdo_dev_plane* mask_cur, const int32_t* wh, int32_t step, float th_depth_obj,
                                             const vdo_obj_mask_out* out, uint64_t stream) {
  return obj_update_mask("vdo_obj_update_mask_batch_dev", false, m, P, depth, flow, mask, mask_cur, wh, step, th_depth_obj, nullptr, out, stream);
}
extern "C" int vdo_obj_update_mask_set_batch_dev(vdo_obj_motion* m, int P, const vdo_dev_plane* depth, const vdo_dev_plane* flow, const vdo_dev_plane* mask,
                                                 const vdo_dev_plane* mask_cur, const int32_t* wh, int32_t step, float th_depth_obj,
                                                 const vdo_obj_feat_set* last, const vdo_obj_mask_out* out, uint64_t stream) {
  return obj_update_mask("vdo_obj_update_mask_set_batch_dev", true, m, P, depth, flow, mask, mask_cur, wh, step, th_depth_obj, last, out, stream);
}

extern "C" int vdo_obj_renew_batch_dev(vdo_obj_motion* m, int P, const vdo_obj_track_out* track_out, const vdo_dev_plane* depth_cur,
                                       const vdo_dev_plane* flow_cur, const vdo_dev_plane* mask_cur, const int32_t* wh, const float* K,
                                       const float* Tcw_cur_dev, int32_t step, float th_depth_obj, int32_t max_track_obj,
                                       const vdo_obj_feat_set* set_out, uint64_t stream) {
  if (!m) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& s) { vdo::ctx_set_error(m->ctx, "vdo_obj_renew_batch_dev: " + s); return VDO_ERR_ARG; };
  if (P < 1 || P > m->max_pairs) return refuse("P = " + std::to_string(P) + " outside 1 .. " + std::to_string(m->max_pairs));
  if (!track_out || !depth_cur || !flow_cur || !mask_cur || !wh || !K || !set_out)
    return refuse("track_out, depth_cur, flow_cur, mask_cur, wh, K or set_out is NULL");
  const vdo_obj_motion_opts o{step, th_depth_obj, 1, 0, 1.0, 0.5, 0, 0};     // only step and th_depth_obj are used
  if (std::string why = om_check_opts(o); !why.empty()) return refuse(why);
  if (max_track_obj < 0) return refuse("max_track_obj = " + std::to_string(max_track_obj) + "; expected >= 0");
  ObjArg a;
  std::memset(&a, 0, sizeof a);
  int max_n = 0;
  vdo::DevPtrs ptrs;
  for (int p = 0; p < P; ++p)
    if (std::string why = om_check_pair(m, p, depth_cur, flow_cur, mask_cur, wh, K, step, a, max_n, ptrs); !why.empty()) return refuse(why);
  const vdo_obj_track_out& t = *track_out;
  const vdo_obj_motion_out& tm = t.motion;
  const vdo_obj_feat_set& s = *set_out;
  ptrs.insert(ptrs.end(), {{Tcw_cur_dev, 4, "Tcw_cur_dev", Tcw_cur_dev != nullptr}, {tm.label_dev, 4, "track_out.motion.label_dev"},
                           {tm.sample_x_dev, 4, "track_out.motion.sample_x_dev"}, {tm.sample_y_dev, 4, "track_out.motion.sample_y_dev"},
                           {tm.sample_slot_dev, 4, "track_out.motion.sample_slot_dev"}, {tm.sample_flags_dev, 1, "track_out.motion.sample_flags_dev"},
                           {tm.sample_flow_ref_dev, 8, "track_out.motion.sample_flow_ref_dev"}, {tm.n_samples_dev, 4, "track_out.motion.n_samples_dev"},
                           {t.id_dev, 4, "track_out.id_dev"}, {t.stat_dev, 4, "track_out.stat_dev"}, {t.obj_label_dev, 4, "track_out.obj_label_dev"},
                           {s.x_dev, 4, "set_out.x_dev"}, {s.y_dev, 4, "set_out.y_dev"}, {s.label_dev, 4, "set_out.label_dev"},
                           {s.depth_dev, 4, "set_out.depth_dev"}, {s.cx_dev, 4, "set_out.cx_dev"}, {s.cy_dev, 4, "set_out.cy_dev"},
                           {s.flow_dev, 4, "set_out.flow_dev"}, {s.inlier_id_dev, 4, "set_out.inlier_id_dev"}, {s.obj_label_dev, 4, "set_out.obj_label_dev"},
                           {s.point_dev, 4, "set_out.point_dev"}, {s.count_dev, 4, "set_out.count_dev"}, {s.status_dev, 4, "set_out.status_dev"}});
  if (std::string why = vdo::check_ptrs(ptrs, m->dev); !why.empty()) return refuse(why);
  a.Tc = Tcw_cur_dev; a.step = step; a.cap = m->cap; a.M = m->max_objects; a.th = th_depth_obj;
  // the idle work space of the RANSAC and the LM: the current raster samples as vdo_obj_update_mask_batch_dev keeps them, their count in
  // the RANSAC counters, the raster positions taken by carried keys in glab
  const size_t pts = (size_t)m->max_pairs * m->cap;
  RenewArg u;
  std::memset(&u, 0, sizeof u);
  u.t = t; u.s = s; u.used = m->glab; u.max_obj = max_track_obj;
  vdo_obj_motion_out& r = u.r;
  r.sample_x_dev = m->r_idx; r.sample_y_dev = m->m_idx; r.sample_label_dev = m->s_idx; r.sample_depth_dev = m->depth;
  r.sample_cx_dev = m->pts; r.sample_cy_dev = m->pts + pts; r.sample_flow_dev = m->flow; r.n_samples_dev = m->counts;
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  k_om_sample<<<P, OM_SAMPLE_THREADS, 0, st>>>(a, r, m->pstat);
  k_rn_select<<<P, OM_THREADS, 0, st>>>(a, u, m->pstat);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
