// orb_match.cu -- vdo_orb_match_batch_dev: brute-force Hamming k-nearest neighbours (k <= 2) of ORB descriptors, optionally inside a
// search window and cross-checked, for up to 64 (query frame, train frame) pairs per call (semantics: include/vdo_b200.h).
//
// A candidate is kept as one 32-bit key (distance << 23) | index: distance <= 256 takes 9 bits, index < cap < 2^23 the rest.  The smaller
// key is the smaller distance, and on equal distances the lower index, which is cv2.BFMatcher's order.  The output arrays hold these
// keys while the scans run, so the call needs no work space:
//   k_match_init    per pair: status bits; every output slot of a valid keypoint := NONE (0xffffffff)
//   k_match_scan    a CTA holds QT "own" descriptors in registers, one per thread, and streams the "other" side's descriptors of its split
//                   of the index range through shared memory in increasing index, keeping its best k keys with strict-less updates.
//                   It then merges them into the pair's slots with atomicMin: slot 0 keeps the smallest key inserted, and each insert
//                   pushes whichever of (its key, the key slot 0 held) slot 0 does not keep into slot 1, so slot 1 ends as the second
//                   smallest key of all.  The best k of the union of the splits' best k is the best k overall, so the result does not
//                   depend on the split.  Forward (own = query, other = train) into idx; reverse (own = train, other = query, k = 1)
//                   into rev_idx.
//   k_match_finish  keys -> (idx, dist), -1 for NONE; with cross-check, i -> j survives only when rev_idx[j] names i
//   k_match_finish_rev  rev_idx keys -> query index
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"


namespace {
constexpr int MATCH_MAX_PAIRS = 64;
constexpr int QT = 128;              // own keypoints per CTA, one per thread
constexpr int TC = 128;              // other-side descriptors per shared-memory chunk
constexpr int IDX_BITS = 23;
constexpr unsigned IDX_MASK = (1u << IDX_BITS) - 1u;
constexpr unsigned NONE = 0xffffffffu;

struct SetArg { const uint4* desc; const float* x; const float* y; const int* count; int cap; };
struct PairArg { int q[MATCH_MAX_PAIRS], t[MATCH_MAX_PAIRS]; };   // by value, as IngestImages

// keypoints of frame f; a count outside 0 .. cap is taken as 0 (k_match_init reports it)
__device__ __forceinline__ int set_count(const SetArg& s, int f) {
  const int c = s.count[f];
  return c >= 0 && c <= s.cap ? c : 0;
}

template <int K>
__device__ __forceinline__ void insert_key(unsigned* slot, unsigned key) {
  const unsigned old = atomicMin(slot, key);
  if (K == 2) atomicMin(slot + 1, max(key, old));
}

__global__ void __launch_bounds__(256) k_match_init(const SetArg Q, const SetArg T, const PairArg pr, int K, unsigned* __restrict__ idx,
                                                    unsigned* __restrict__ rev, int* __restrict__ status) {
  const int p = blockIdx.y, fq = pr.q[p], ft = pr.t[p];
  const int nq = set_count(Q, fq), nt = set_count(T, ft);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int cq = Q.count[fq], ct = T.count[ft];
    status[p] = (cq < 0 || cq > Q.cap ? VDO_ORB_MATCH_STATUS_QUERY_COUNT : 0) | (ct < 0 || ct > T.cap ? VDO_ORB_MATCH_STATUS_TRAIN_COUNT : 0);
  }
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nq * K; i += stride) idx[(size_t)p * Q.cap * K + i] = NONE;
  if (rev)
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += stride) rev[(size_t)p * T.cap + j] = NONE;
}

// REV = false: own = query keypoints of pair blockIdx.z (position: pred), other = train keypoints (position: x, y), slots = idx.
// REV = true:  own = train keypoints, other = query keypoints, slots = rev_idx (K = 1).  The window predicate is |x_t - px| <= r and
// |y_t - py| <= r either way (float subtraction is exactly antisymmetric).  blockIdx.y: the split [y * span, (y + 1) * span) of the
// other side's indices.
template <int K, bool REV, bool WIN>
__global__ void __launch_bounds__(QT) k_match_scan(const SetArg Q, const SetArg T, const PairArg pr, const float* __restrict__ pred, float radius,
                                                   int span, unsigned* __restrict__ slots) {
  __shared__ uint4 sd[TC][2];
  __shared__ float2 sp[WIN ? TC : 1];
  const int p = blockIdx.z, fq = pr.q[p], ft = pr.t[p];
  const int nq = set_count(Q, fq), nt = set_count(T, ft);
  const int na = REV ? nt : nq, nb = REV ? nq : nt;
  const int i0 = blockIdx.x * QT, i = i0 + threadIdx.x;
  const int j0 = blockIdx.y * span, j1 = min(j0 + span, nb);
  if (i0 >= na || j0 >= j1) return;
  const bool act = i < na;
  const uint4* qd = Q.desc + (size_t)fq * Q.cap * 2;   // rows of the pair's frames
  const uint4* td = T.desc + (size_t)ft * T.cap * 2;
  const float* pq = pred + (size_t)p * Q.cap * 2;
  const float* tx = T.x + (size_t)ft * T.cap;
  const float* ty = T.y + (size_t)ft * T.cap;
  const uint4* bd = REV ? qd : td;
  uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
  float ox = 0.f, oy = 0.f;
  if (act) {
    const uint4* d = (REV ? td : qd) + 2 * i;
    q0 = d[0]; q1 = d[1];
    if (WIN) {
      if (REV) { ox = tx[i]; oy = ty[i]; }
      else { ox = pq[2 * i]; oy = pq[2 * i + 1]; }
    }
  }
  unsigned k1 = NONE, k2 = NONE;
  for (int c0 = j0; c0 < j1; c0 += TC) {
    const int nc = min(TC, j1 - c0);
    __syncthreads();
    for (int t = threadIdx.x; t < nc; t += QT) {
      const int j = c0 + t;
      sd[t][0] = bd[2 * j]; sd[t][1] = bd[2 * j + 1];
      if (WIN) sp[t] = REV ? make_float2(pq[2 * j], pq[2 * j + 1]) : make_float2(tx[j], ty[j]);
    }
    __syncthreads();
    if (!act) continue;
#pragma unroll 4
    for (int t = 0; t < nc; ++t) {
      if (WIN && !(fabsf(sp[t].x - ox) <= radius && fabsf(sp[t].y - oy) <= radius)) continue;
      const uint4 a = sd[t][0], b = sd[t][1];
      const unsigned dist = __popc(a.x ^ q0.x) + __popc(a.y ^ q0.y) + __popc(a.z ^ q0.z) + __popc(a.w ^ q0.w) +
                            __popc(b.x ^ q1.x) + __popc(b.y ^ q1.y) + __popc(b.z ^ q1.z) + __popc(b.w ^ q1.w);
      const unsigned key = (dist << IDX_BITS) | (unsigned)(c0 + t);
      // indices increase, so strict-less keeps the earlier index on equal distances
      if (key < k1) { if (K == 2) k2 = k1; k1 = key; }
      else if (K == 2 && key < k2) k2 = key;
    }
  }
  if (!act || k1 == NONE) return;
  unsigned* slot = slots + ((size_t)p * (REV ? T.cap : Q.cap) + i) * K;
  insert_key<K>(slot, k1);
  if (K == 2 && k2 != NONE) insert_key<K>(slot, k2);
}

template <int K>
__global__ void __launch_bounds__(256) k_match_finish(const SetArg Q, const SetArg T, const PairArg pr, int* __restrict__ idx, int* __restrict__ dist,
                                                      const unsigned* __restrict__ rev) {
  const int p = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= set_count(Q, pr.q[p])) return;
  const size_t o = ((size_t)p * Q.cap + i) * K;
  for (int s = 0; s < K; ++s) {
    const unsigned key = (unsigned)idx[o + s];
    int j = key == NONE ? -1 : (int)(key & IDX_MASK), d = key == NONE ? -1 : (int)(key >> IDX_BITS);
    // rev_idx still holds keys here; a matched j has i as a candidate, so its key is not NONE
    if (rev && j >= 0 && (rev[(size_t)p * T.cap + j] & IDX_MASK) != (unsigned)i) j = d = -1;
    idx[o + s] = j; dist[o + s] = d;
  }
}

__global__ void __launch_bounds__(256) k_match_finish_rev(const SetArg T, const PairArg pr, unsigned* __restrict__ rev) {
  const int p = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= set_count(T, pr.t[p])) return;
  unsigned& r = rev[(size_t)p * T.cap + j];
  r = r == NONE ? NONE : (r & IDX_MASK);
}

// grid of a scan: own tiles x splits x pairs, splits of whole TC chunks, enough CTAs for about 8 per SM
dim3 scan_grid(int P, int own_cap, int other_cap, int n_sm, int* span) {
  const int tiles = (own_cap + QT - 1) / QT, chunks = (other_cap + TC - 1) / TC;
  const int want = std::max(1, std::min(chunks, (8 * n_sm + P * tiles - 1) / (P * tiles)));
  *span = (chunks + want - 1) / want * TC;
  return dim3(tiles, (other_cap + *span - 1) / *span, P);
}

template <bool REV, bool WIN>
void launch_scan(int K, dim3 g, cudaStream_t st, const SetArg& Q, const SetArg& T, const PairArg& pr, const float* pred, float r, int span, unsigned* slots) {
  if (K == 2) k_match_scan<2, REV, WIN><<<g, QT, 0, st>>>(Q, T, pr, pred, r, span, slots);
  else k_match_scan<1, REV, WIN><<<g, QT, 0, st>>>(Q, T, pr, pred, r, span, slots);
}
}  // namespace

extern "C" int vdo_orb_match_batch_dev(vdo_ctx* ctx, int P, const int32_t* pairs, const vdo_orb_desc_set* query, const vdo_orb_desc_set* train,
                                       const float* pred_dev, const vdo_orb_match_opts* opts, const vdo_orb_match_out* out, uint64_t stream) {
  if (!ctx) return VDO_ERR_ARG;
  auto refuse = [&](const std::string& m) { vdo::ctx_set_error(ctx, "vdo_orb_match_batch_dev: " + m); return VDO_ERR_ARG; };
  if (P < 1 || P > MATCH_MAX_PAIRS) return refuse("P = " + std::to_string(P) + " outside 1 .. " + std::to_string(MATCH_MAX_PAIRS));
  if (!pairs || !query || !train || !opts || !out) return refuse("pairs, query, train, opts or out is NULL");
  const int K = opts->k;
  if (K != 1 && K != 2) return refuse("k = " + std::to_string(K) + "; expected 1 or 2");
  if (opts->cross_check != 0 && opts->cross_check != 1) return refuse("cross_check = " + std::to_string(opts->cross_check) + "; expected 0 or 1");
  const bool cross = opts->cross_check == 1;
  if (cross && K != 1) return refuse("cross_check needs k = 1");
  if (cross && !out->rev_idx_dev) return refuse("cross_check needs rev_idx_dev");
  if (std::isnan(opts->radius)) return refuse("radius is NaN");
  const bool win = opts->radius > 0.f;
  for (const auto& s : {std::make_pair("query", query), std::make_pair("train", train)})
    if (s.second->n_frames < 1 || s.second->cap < 1 || (unsigned)s.second->cap > IDX_MASK)
      return refuse(std::string(s.first) + ": n_frames = " + std::to_string(s.second->n_frames) + ", cap = " + std::to_string(s.second->cap) +
                    "; expected n_frames >= 1 and 1 <= cap < 2^23");
  PairArg pr;
  for (int p = 0; p < P; ++p) {
    pr.q[p] = pairs[2 * p]; pr.t[p] = pairs[2 * p + 1];
    if (pr.q[p] < 0 || pr.q[p] >= query->n_frames || pr.t[p] < 0 || pr.t[p] >= train->n_frames)
      return refuse("pair " + std::to_string(p) + " = (" + std::to_string(pr.q[p]) + ", " + std::to_string(pr.t[p]) + ") outside the sets' " +
                    std::to_string(query->n_frames) + " x " + std::to_string(train->n_frames) + " frames");
  }
  for (int p = P; p < MATCH_MAX_PAIRS; ++p) pr.q[p] = pr.t[p] = 0;
  int dev = 0, n_sm = 0;
  vdo::ctx_device(ctx, &dev, &n_sm);
  // every pointer the call reads or writes: NULL, misaligned or not on the context's device is refused
  const vdo::DevPtrs ptrs = {
      {query->desc_dev, 16, "query.desc_dev"}, {query->count_dev, 4, "query.count_dev"},
      {train->desc_dev, 16, "train.desc_dev"}, {train->count_dev, 4, "train.count_dev"},
      {train->x_dev, 4, "train.x_dev (a window reads it)", win}, {train->y_dev, 4, "train.y_dev (a window reads it)", win},
      {pred_dev, 4, "pred_dev (a window reads it)", win},
      {out->idx_dev, 4, "out.idx_dev"}, {out->dist_dev, 4, "out.dist_dev"}, {out->status_dev, 4, "out.status_dev"},
      {out->rev_idx_dev, 4, "out.rev_idx_dev", out->rev_idx_dev != nullptr}};
  if (std::string why = vdo::check_ptrs(ptrs, dev); !why.empty()) return refuse(why);
  const SetArg Q{(const uint4*)query->desc_dev, query->x_dev, query->y_dev, query->count_dev, query->cap};
  const SetArg T{(const uint4*)train->desc_dev, train->x_dev, train->y_dev, train->count_dev, train->cap};
  const cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  unsigned* idx = (unsigned*)out->idx_dev;
  unsigned* rev = (unsigned*)out->rev_idx_dev;
  const float r = opts->radius;
  const int init_blocks = (std::max(query->cap * K, train->cap) + 255) / 256;
  k_match_init<<<dim3(init_blocks, P), 256, 0, st>>>(Q, T, pr, K, idx, rev, out->status_dev);
  int span = 0;
  dim3 g = scan_grid(P, query->cap, train->cap, n_sm, &span);
  if (win) launch_scan<false, true>(K, g, st, Q, T, pr, pred_dev, r, span, idx);
  else launch_scan<false, false>(K, g, st, Q, T, pr, pred_dev, r, span, idx);
  if (rev) {
    g = scan_grid(P, train->cap, query->cap, n_sm, &span);
    if (win) launch_scan<true, true>(1, g, st, Q, T, pr, pred_dev, r, span, rev);
    else launch_scan<true, false>(1, g, st, Q, T, pr, pred_dev, r, span, rev);
  }
  const unsigned* cc = cross ? rev : nullptr;
  if (K == 2) k_match_finish<2><<<dim3((query->cap + 255) / 256, P), 256, 0, st>>>(Q, T, pr, out->idx_dev, out->dist_dev, cc);
  else k_match_finish<1><<<dim3((query->cap + 255) / 256, P), 256, 0, st>>>(Q, T, pr, out->idx_dev, out->dist_dev, cc);
  if (rev) k_match_finish_rev<<<dim3((train->cap + 255) / 256, P), 256, 0, st>>>(T, pr, rev);
  VDO_CUDA(cudaGetLastError());
  return VDO_OK;
}
