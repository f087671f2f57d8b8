// pnp_corr.cuh -- the correspondence rule of the device calls on ORB matches of P frame pairs (include/vdo_b200.h, vdo_pnp_match_batch_dev),
// shared by vdo_pnp_match_batch_dev (pnp_ransac.cu) and vdo_pose_refine_batch_dev (flow_lm.cu): the per-pair host parameters carried by
// value in one kernel argument, the predicate that decides whether query keypoint i is a correspondence, and the ordered compaction that
// gathers the correspondences of a pair in ascending i inside one CTA; on the host, the argument checks both calls share.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"

namespace {

constexpr int PNP_MAX_PAIRS = 64;
struct PnpPairArg {                 // one pair's host parameters, passed by value so that a captured call replays with them
  const float* depth; long long sy, sx; int w, h;
  int q, t, has_T, pad;
  float Kq[4], Kt[4], T[12];        // T: rows 0..2 of the query frame's Tcw
};
struct PnpGatherArg {
  const float *qx, *qy, *tx, *ty;
  const int *qcount, *tcount, *idx, *dist;
  int qcap, tcap, k, seg;           // seg: the solver's per-pair segment (offset p * seg)
  float ratio, max_depth;
  PnpPairArg pr[PNP_MAX_PAIRS];
};

__device__ __forceinline__ int valid_count(int c, int cap) { return c >= 0 && c <= cap ? c : 0; }

// is query keypoint i of the pair a correspondence (include/vdo_b200.h); z: the depth it reads
struct PredCorr {
  const PnpGatherArg* a; const PnpPairArg* pa; const float *qx, *qy; const int *idx, *dist; int nt;
  __device__ __forceinline__ bool depth_at(int i, float* z) const {
    const float u = qx[i], v = qy[i];
    if (!(u > -1.f && u < (float)pa->w && v > -1.f && v < (float)pa->h)) return false;   // (int) truncates toward zero
    *z = pa->depth[(long long)(int)v * pa->sy + (long long)(int)u * pa->sx];
    return true;
  }
  __device__ __forceinline__ bool operator()(int i) const {
    const int j = idx[(size_t)i * a->k];
    if (!(j >= 0 && j < nt)) return false;
    if (a->ratio > 0.f && !(idx[(size_t)i * a->k + 1] >= 0 && (float)dist[(size_t)i * a->k] < a->ratio * (float)dist[(size_t)i * a->k + 1])) return false;
    float z;
    if (!depth_at(i, &z)) return false;
    return a->max_depth > 0.f ? (z > 0.f && z <= a->max_depth) : z > 0.f;
  }
};

// ordered compaction of flagged indices of [0,n) into out (ascending) by a CTA of THREADS threads; returns the count.  All threads of
// the CTA call it.
template <int THREADS, class Pred>
__device__ __forceinline__ int compact_ordered(int n, const Pred& pred, int* out, int* s_scan, int* s_base) {
  if (threadIdx.x == 0) *s_base = 0;
  __syncthreads();
  for (int start = 0; start < n; start += THREADS) {
    const int i = start + threadIdx.x;
    const int f = (i < n && pred(i)) ? 1 : 0;
    s_scan[threadIdx.x] = f;
    __syncthreads();
    for (int o = 1; o < THREADS; o <<= 1) {
      const int v = threadIdx.x >= o ? s_scan[threadIdx.x - o] : 0;
      __syncthreads();
      s_scan[threadIdx.x] += v;
      __syncthreads();
    }
    if (f) out[*s_base + s_scan[threadIdx.x] - 1] = i;
    __syncthreads();
    if (threadIdx.x == THREADS - 1) *s_base += s_scan[threadIdx.x];
    __syncthreads();
  }
  return *s_base;
}

// ---- host side: the argument checks both calls share ----
// The checks of a call on a solver or refiner (holder) with max_pairs, cap and device dev, in this order: P; the NULL arguments (k_name: the
// call's name for K_query); the sets' sizes; query.cap against the holder's cap; own_first(); k, ratio and max_depth of opts;
// own_then(extra); the pairs and depth planes (depth_wh: their sizes); the device arrays of the rule, then extra.  own_first / own_then:
// the caller's checks of its other options ("" or a reason); own_then also appends the caller's device arrays (its outputs) to extra.
// "" with ga complete (K_train NULL = K_query, Tcw_query NULL = none), or why the call is refused.
template <class Opts, class First, class Then>
std::string corr_check(const char* holder, int max_pairs, int cap, int dev, int P, const int32_t* pairs, const vdo_orb_desc_set* query,
                       const vdo_orb_desc_set* train, const int32_t* idx_dev, const int32_t* dist_dev, const vdo_dev_plane* depth, const int32_t* depth_wh,
                       const char* k_name, const float* K_query, const float* K_train, const float* Tcw_query, const Opts* opts, const void* out,
                       const First& own_first, const Then& own_then, PnpGatherArg& ga) {
  const int max_p = std::min(PNP_MAX_PAIRS, max_pairs);
  if (P < 1 || P > max_p) return "P = " + std::to_string(P) + " outside 1 .. " + std::to_string(max_p);
  if (!pairs || !query || !train || !depth || !depth_wh || !K_query || !opts || !out)
    return std::string("pairs, query, train, depth, depth_wh, ") + k_name + ", opts or out is NULL";
  for (const auto& q : {std::make_pair("query", query), std::make_pair("train", train)})
    if (q.second->n_frames < 1 || q.second->cap < 1)
      return std::string(q.first) + ": n_frames = " + std::to_string(q.second->n_frames) + ", cap = " + std::to_string(q.second->cap) + "; expected >= 1";
  if (query->cap > cap) return "query.cap = " + std::to_string(query->cap) + " exceeds the " + holder + "'s cap " + std::to_string(cap);
  if (std::string why = own_first(); !why.empty()) return why;
  const Opts& o = *opts;
  if (o.k != 1 && o.k != 2) return "k = " + std::to_string(o.k) + "; expected 1 or 2";
  if (std::isnan(o.ratio) || std::isnan(o.max_depth)) return "ratio or max_depth is NaN";
  if (o.ratio > 0.f && o.k != 2) return "the ratio test needs k = 2";
  vdo::DevPtrs extra;
  if (std::string why = own_then(extra); !why.empty()) return why;
  std::memset(&ga, 0, sizeof ga);
  for (int p = 0; p < P; ++p) {
    PnpPairArg& pa = ga.pr[p];
    pa.q = pairs[2 * p]; pa.t = pairs[2 * p + 1];
    if (pa.q < 0 || pa.q >= query->n_frames || pa.t < 0 || pa.t >= train->n_frames)
      return "pair " + std::to_string(p) + " = (" + std::to_string(pa.q) + ", " + std::to_string(pa.t) + ") outside the sets' " +
             std::to_string(query->n_frames) + " x " + std::to_string(train->n_frames) + " frames";
    const vdo_dev_plane& pl = depth[p];
    const std::string who = "depth plane " + std::to_string(p);
    if (pl.dtype != VDO_DT_F32 || pl.channels != 1)
      return who + ": dtype " + std::to_string(pl.dtype) + " with " + std::to_string(pl.channels) + " channels; expected f32 with 1 channel";
    if (depth_wh[2 * p] < 1 || depth_wh[2 * p + 1] < 1)
      return who + ": " + std::to_string(depth_wh[2 * p]) + " x " + std::to_string(depth_wh[2 * p + 1]) + "; expected a width and height >= 1";
    pa.depth = (const float*)pl.data_dev; pa.sy = pl.stride_y; pa.sx = pl.stride_x; pa.w = depth_wh[2 * p]; pa.h = depth_wh[2 * p + 1];
    const float* Kt = K_train ? K_train : K_query;
    for (int c = 0; c < 4; ++c) { pa.Kq[c] = K_query[4 * p + c]; pa.Kt[c] = Kt[4 * p + c]; }
    pa.has_T = Tcw_query ? 1 : 0;
    if (Tcw_query) std::memcpy(pa.T, Tcw_query + 16 * p, 48);
  }
  // every device pointer the call reads or writes: NULL, misaligned or not on the holder's device is refused
  vdo::DevPtrs ptrs = {{query->x_dev, 4, "query.x_dev"}, {query->y_dev, 4, "query.y_dev"}, {query->count_dev, 4, "query.count_dev"},
                       {train->x_dev, 4, "train.x_dev"}, {train->y_dev, 4, "train.y_dev"}, {train->count_dev, 4, "train.count_dev"},
                       {idx_dev, 4, "idx_dev"}, {dist_dev, 4, "dist_dev"}};
  for (int p = 0; p < P; ++p) ptrs.push_back({depth[p].data_dev, 4, "depth plane " + std::to_string(p) + ": data_dev"});
  ptrs.insert(ptrs.end(), extra.begin(), extra.end());
  if (std::string why = vdo::check_ptrs(ptrs, dev); !why.empty()) return why;
  ga.qx = query->x_dev; ga.qy = query->y_dev; ga.tx = train->x_dev; ga.ty = train->y_dev;
  ga.qcount = query->count_dev; ga.tcount = train->count_dev; ga.idx = idx_dev; ga.dist = dist_dev;
  ga.qcap = query->cap; ga.tcap = train->cap; ga.k = o.k; ga.seg = cap;
  ga.ratio = o.ratio > 0.f ? o.ratio : 0.f; ga.max_depth = o.max_depth > 0.f ? o.max_depth : 0.f;
  return "";
}

}  // namespace
