// tracking_ops.cu -- bookkeeping stages of Tracking that sit between the kernels: tracklet chaining (A16), mask propagation
// (A15) and dynamic-object classification / ID assignment (A13).  These are integer, order-dependent procedures over a few
// thousand to a few hundred thousand elements: the image-sized work (mask gather / forward warp) and the per-object
// reductions run on the device next to the resident frame, the decisions (which are sequential by definition in the
// reference: IDs are handed out in label order) run on the host side of the call.
//
// Reference semantics (restated in oracle/tracking_ops.py):
//   Tracking::GetStaticTrack / GetDynamicTrackNew   src/Tracking.cc:2201-2307, 2309-2421
//   Tracking::UpdateMask                            src/Tracking.cc:2997-3110
//   Tracking::DynObjTracking                        src/Tracking.cc:1366-1612  (ground-truth bookkeeping :1531-1544 excluded)
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"
#include "frame_px.cuh"
#include "dyn_obj.cuh"
#include "frame_batch.h"

namespace {

// Per-stream scratch arena: every entry point of this file is synchronous on the context stream, so the scratch of one call can be
// recycled by the next.  Chunks are only added during a call; at the start of the next call several chunks are merged into one.
// (cudaMalloc / cudaFree per call cost tens of microseconds each and cudaFree synchronises the device.)
struct Arena {
  struct Chunk { char* p; size_t cap, off; };
  std::vector<Chunk> chunks;
  void reset() {
    if (chunks.size() > 1) {
      size_t tot = 0;
      for (auto& c : chunks) { tot += c.cap; cudaFree(c.p); }
      chunks.clear();
      char* p = nullptr;
      if (cudaMalloc(&p, tot) == cudaSuccess) chunks.push_back({p, tot, 0});
    }
    for (auto& c : chunks) c.off = 0;
  }
  void* alloc(size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (bytes == 0) bytes = 256;
    for (auto& c : chunks) if (c.off + bytes <= c.cap) { void* r = c.p + c.off; c.off += bytes; return r; }
    const size_t cap = std::max(bytes, (size_t)1 << 20);
    char* p = nullptr;
    if (cudaMalloc(&p, cap) != cudaSuccess) return nullptr;
    chunks.push_back({p, cap, bytes});
    return p;
  }
};
std::mutex g_arena_mu;
std::map<cudaStream_t, Arena> g_arena;
Arena& arena_begin(cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_arena_mu);
  Arena& a = g_arena[st];
  a.reset();
  return a;
}
struct DevBuf {
  void* p = nullptr;
  cudaError_t alloc(Arena& a, size_t bytes) { p = a.alloc(bytes); return p ? cudaSuccess : cudaErrorMemoryAllocation; }
  template <class T> T* as() { return (T*)p; }
};

// label of the current mask at the (truncated) flow target of every last-frame object point; -1 = outside (u>0, v>0 strict)
__global__ void k_gather_mask(const int* __restrict__ mask, int w, int h, const float* __restrict__ cx, const float* __restrict__ cy, int n, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int u = (int)cx[i], v = (int)cy[i];
  out[i] = (u < w && u > 0 && v < h && v > 0) ? mask[(size_t)v * w + u] : -1;
}
// forward-warp one object of the last mask into the current mask by the (int-truncated) last flow
__global__ void k_mask_warp(const int* __restrict__ mask_last, const float* __restrict__ flow_last, int w, int h, int label, int* __restrict__ mask_cur) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (k >= w) return;
  const size_t p = (size_t)j * w + k;
  if (mask_last[p] != label) return;
  const int fx = (int)flow_last[2 * p], fy = (int)flow_last[2 * p + 1];
  const int x = k + fx, y = j + fy;
  if (x < w && x > 0 && y < h && y > 0) mask_cur[(size_t)y * w + x] = label;   // every colliding write stores the same value
}

// one thread per object walks its points in index order: float sums round exactly like the reference's loops
__global__ void k_obj_stats(const int* __restrict__ obj_begin, const int* __restrict__ obj_idx, int n_obj, const float* __restrict__ kx,
                            const float* __restrict__ ky, const float* __restrict__ depth, const float* __restrict__ flow3d, int rows, int cols,
                            int shr_row, int shr_col, float sf_thres, ObjStat* __restrict__ out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_obj) return;
  ObjStat s{0.f, 0.f, 0.f, obj_begin[o + 1] - obj_begin[o]};
  for (int q = obj_begin[o]; q < obj_begin[o + 1]; ++q) {
    obj_stat_add(s, kx, ky, depth, flow3d, obj_idx[q], rows, cols, shr_row, shr_col, sf_thres);
  }
  out[o] = s;
}

// majority label with the reference's ordering: std::map (ascending label) then sort by count descending; ties keep the
// smaller label first (what std::sort's insertion-sort path does for the <= 16 distinct labels seen in practice)
int majority_label(const std::vector<int>& v) {
  std::map<int, int> dups;
  for (int k : v) ++dups[k];
  int best = 0, cnt = -1;
  for (auto& kv : dups) if (kv.second > cnt) { cnt = kv.second; best = kv.first; }
  return best;
}
}  // namespace

// frame internals needed here (defined in frame_kernels.cu)
extern "C" int vdo_frame_device_ptrs(vdo_frame* f, unsigned char** gray, float** depth, float** flow, int** mask, int* w, int* h, void** stream);

// ------------------------------------------------------------------------------------------------ A16
extern "C" int vdo_tracklets_build(int n_rows, const int* row_begin, const int* assoc, const int* labels, int max_tracklets, int max_entries,
                                   int* n_trk, int* trk_begin, int* trk_frame, int* trk_feat, int* obj_id) {
  if (n_rows < 0 || !row_begin || !n_trk || !trk_begin) return VDO_ERR_ARG;
  std::vector<std::vector<std::pair<int, int>>> T;
  std::vector<int> oid, pre, cur;
  for (int i = 0; i < n_rows; ++i) {
    const int n = row_begin[i + 1] - row_begin[i];
    cur.assign(n, -1);
    for (int j = 0; j < n; ++j) {
      const int a = assoc[row_begin[i] + j];
      if (a == -1) continue;
      if (i > 0 && a >= 0 && a < (int)pre.size() && pre[a] != -1) { T[pre[a]].push_back({i + 1, j}); cur[j] = pre[a]; }
      else {
        if (i > 0 && (a < 0 || a >= (int)pre.size())) return VDO_ERR_ARG;
        T.push_back({{i, a}, {i + 1, j}});
        if (labels) oid.push_back(labels[row_begin[i] + j]);
        cur[j] = (int)T.size() - 1;
      }
    }
    pre.swap(cur);
  }
  size_t tot = 0;
  for (auto& t : T) tot += t.size();
  *n_trk = (int)T.size();
  if ((int)T.size() > max_tracklets || (long)tot > (long)max_entries) return VDO_ERR_ARG;
  int off = 0;
  for (size_t t = 0; t < T.size(); ++t) {
    trk_begin[t] = off;
    for (auto& pr : T[t]) { trk_frame[off] = pr.first; trk_feat[off] = pr.second; ++off; }
    if (labels && obj_id) obj_id[t] = oid[t];
  }
  trk_begin[T.size()] = off;
  return VDO_OK;
}

// ------------------------------------------------------------------------------------------------ A15
// cur / last: resident frames (masks + last flow).  sem_label_last, corres_x/y: last frame's vSemObjLabel and mvObjCorres (n points).
// mask_out (may be NULL) receives the updated current mask so the caller's cv::Mat is mutated like in the reference.
extern "C" int vdo_update_mask(vdo_frame* cur, vdo_frame* last, int n, const int* sem_label_last, const float* corres_x, const float* corres_y,
                               int* mask_out, int* n_warped, int* warped_labels) {
  if (!cur || !last || n < 0) return VDO_ERR_ARG;
  int *mcur, *mlast, w, h, w2, h2; float *fl_last; void* stv;
  if (vdo_frame_device_ptrs(cur, nullptr, nullptr, nullptr, &mcur, &w, &h, &stv)) return VDO_ERR_ARG;
  if (vdo_frame_device_ptrs(last, nullptr, nullptr, &fl_last, &mlast, &w2, &h2, nullptr)) return VDO_ERR_ARG;
  if (w != w2 || h != h2) return VDO_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stv;
  if (n_warped) *n_warped = 0;
  std::vector<int> uni(sem_label_last, sem_label_last + n);
  std::sort(uni.begin(), uni.end());
  uni.erase(std::unique(uni.begin(), uni.end()), uni.end());
  float *d_cx = nullptr, *d_cy = nullptr; int* d_lab = nullptr;
  Arena& A = arena_begin(st);
  if (n > 0) {
    DevBuf b1, b2, b3;
    VDO_CUDA(b1.alloc(A, sizeof(float) * n)); VDO_CUDA(b2.alloc(A, sizeof(float) * n)); VDO_CUDA(b3.alloc(A, sizeof(int) * n));
    d_cx = b1.as<float>(); d_cy = b2.as<float>(); d_lab = b3.as<int>();
    VDO_CUDA(cudaMemcpyAsync(d_cx, corres_x, sizeof(float) * n, cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(d_cy, corres_y, sizeof(float) * n, cudaMemcpyHostToDevice, st));
  }
  std::vector<int> lab(n);
  bool stale = true;
  for (size_t oi = 0; oi < uni.size(); ++oi) {
    if (stale && n > 0) {          // (re)gather: an earlier object's warp may have changed the labels this object votes on
      k_gather_mask<<<(n + 255) / 256, 256, 0, st>>>(mcur, w, h, d_cx, d_cy, n, d_lab);
      VDO_CUDA(cudaMemcpyAsync(lab.data(), d_lab, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
      VDO_CUDA(cudaStreamSynchronize(st));
      stale = false;
    }
    std::vector<int> tmp;
    for (int i = 0; i < n; ++i) if (sem_label_last[i] == uni[oi] && lab[i] != -1) tmp.push_back(lab[i]);
    if (tmp.size() < 100) continue;
    if (majority_label(tmp) != 0) continue;
    dim3 b(256), g((w + 255) / 256, h);
    k_mask_warp<<<g, b, 0, st>>>(mlast, fl_last, w, h, uni[oi], mcur);
    if (warped_labels && n_warped) warped_labels[*n_warped] = uni[oi];
    if (n_warped) ++*n_warped;
    stale = true;
  }
  if (mask_out) VDO_CUDA(cudaMemcpyAsync(mask_out, mcur, sizeof(int) * (size_t)w * h, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  return VDO_OK;
}

// ------------------------------------------------------------------------------------------------ A13
// Inputs are the current frame's object points (n): semantic label, tracking label (in/out), pixel, depth, scene flow (n x 3),
// the same points' semantic labels in the last frame, and the last frame's object table (nSemPosition, bObjStat, nModLabel).
// Outputs: obj_label (in place), the kept objects as CSR (obj_begin / obj_idx, indices into the point arrays) with their
// tracking ids (mod_label) and semantic labels (sem_position), and max_id (in/out).
extern "C" int vdo_dyn_obj_tracking(vdo_ctx* ctx, int n, const int* sem_label, int* obj_label, const float* kx, const float* ky, const float* depth,
                                    const float* flow3d, const int* sem_label_last, int n_last_obj, const int* last_sem_position,
                                    const unsigned char* last_obj_stat, const int* last_mod_label, int rows, int cols, int shrink_row, int shrink_col,
                                    float sf_mg_thres, float sf_ds_thres, float th_depth_obj, int f_id, int* max_id, int max_objects,
                                    int* n_objects, int* obj_begin, int* obj_idx, int* mod_label, int* sem_position) {
  if (!ctx || n < 0 || !max_id || !n_objects) return VDO_ERR_ARG;
  cudaStream_t st = (cudaStream_t)(uintptr_t)vdo_ctx_stream(ctx);
  *n_objects = 0;
  std::vector<int> uni(sem_label, sem_label + n);
  std::sort(uni.begin(), uni.end());
  uni.erase(std::unique(uni.begin(), uni.end()), uni.end());
  std::vector<std::vector<int>> posi(uni.size());
  for (int i = 0; i < n; ++i) {
    if (obj_label[i] == -1) continue;
    const int j = (int)(std::lower_bound(uni.begin(), uni.end(), sem_label[i]) - uni.begin());
    posi[j].push_back(i);
  }
  // ---- per-object statistics on the device (one sequential thread per object, reference rounding) ----
  std::vector<int> ob(1, 0), oidx;
  for (auto& p : posi) { oidx.insert(oidx.end(), p.begin(), p.end()); ob.push_back((int)oidx.size()); }
  const int no = (int)posi.size();
  std::vector<ObjStat> stats(no);
  if (no > 0 && !oidx.empty()) {
    Arena& A = arena_begin(st);
    DevBuf c1, c2, c3, c4, c5, c6, c7;
    VDO_CUDA(c1.alloc(A, sizeof(int) * (no + 1))); VDO_CUDA(c2.alloc(A, sizeof(int) * oidx.size()));
    VDO_CUDA(c3.alloc(A, sizeof(float) * n)); VDO_CUDA(c4.alloc(A, sizeof(float) * n)); VDO_CUDA(c5.alloc(A, sizeof(float) * n)); VDO_CUDA(c6.alloc(A, sizeof(float) * 3 * n));
    VDO_CUDA(c7.alloc(A, sizeof(ObjStat) * no));
    int *d_ob = c1.as<int>(), *d_oi = c2.as<int>(); float *d_kx = c3.as<float>(), *d_ky = c4.as<float>(), *d_dp = c5.as<float>(), *d_f3 = c6.as<float>();
    ObjStat* d_st = c7.as<ObjStat>();
    VDO_CUDA(cudaMemcpyAsync(d_ob, ob.data(), sizeof(int) * (no + 1), cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(d_oi, oidx.data(), sizeof(int) * oidx.size(), cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(d_kx, kx, sizeof(float) * n, cudaMemcpyHostToDevice, st)); VDO_CUDA(cudaMemcpyAsync(d_ky, ky, sizeof(float) * n, cudaMemcpyHostToDevice, st));
    VDO_CUDA(cudaMemcpyAsync(d_dp, depth, sizeof(float) * n, cudaMemcpyHostToDevice, st)); VDO_CUDA(cudaMemcpyAsync(d_f3, flow3d, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, st));
    k_obj_stats<<<(no + 31) / 32, 32, 0, st>>>(d_ob, d_oi, no, d_kx, d_ky, d_dp, d_f3, rows, cols, shrink_row, shrink_col, sf_mg_thres, d_st);
    VDO_CUDA(cudaMemcpyAsync(stats.data(), d_st, sizeof(ObjStat) * no, cudaMemcpyDeviceToHost, st));
    VDO_CUDA(cudaStreamSynchronize(st));
  }
  // ---- decisions, in label order like the reference ----
  std::vector<std::vector<int>> obj_new; std::vector<int> sem_new;
  for (int i = 0; i < no; ++i) {
    if (posi[i].empty()) continue;                            // (the reference would divide 0/0 here: NaN > 0.5 is false -> kept, then dropped for size < 150)
    const int cls = obj_class(stats[i], sf_ds_thres, th_depth_obj);
    if (cls != OBJ_DYNAMIC) { for (int k : posi[i]) obj_label[k] = cls == OBJ_STATIC ? 0 : -1; continue; }
    obj_new.push_back(posi[i]); sem_new.push_back(uni[i]);
  }
  if (f_id == 1) *max_id = 1;
  if ((int)obj_new.size() > max_objects) return VDO_ERR_ARG;
  int off = 0;
  for (size_t i = 0; i < obj_new.size(); ++i) {
    std::vector<int> lb;
    for (int k : obj_new[i]) lb.push_back(sem_label_last[k]);
    const int new_lab = majority_label(lb);
    int id = -1;
    if (*max_id == 1) { id = *max_id; *max_id += 1; }
    else {
      for (int k = 0; k < n_last_obj; ++k)
        if (last_sem_position[k] == new_lab && last_obj_stat[k]) { id = last_mod_label[k]; break; }
      if (id == -1) { id = *max_id; *max_id += 1; }
    }
    for (int k : obj_new[i]) obj_label[k] = id;
    mod_label[i] = id; sem_position[i] = sem_new[i];
    obj_begin[i] = off;
    for (int k : obj_new[i]) obj_idx[off++] = k;
  }
  obj_begin[obj_new.size()] = off;
  *n_objects = (int)obj_new.size();
  return VDO_OK;
}

// ------------------------------------------------------------------------------------------------ A14
// Tracking::RenewFrameInfo (src/Tracking.cc:2660-2995).  The reference walks candidates sequentially, but every accept / reject
// test depends only on the candidate, the current images and a SNAPSHOT of the inlier set taken before the top-up starts
// (mvKeysTmpCheck / mvObjKeysTmpCheck), so the tests run as two kernel launches (inliers of static + objects; then top-up
// candidates against the snapshots) and only the ordered "take until the quota is met" selection stays on the host.
namespace {
struct RenewCand { float fx, fy, depth; int flag, x, y, sem; };
// static inlier / ORB candidate test (:2680-2704, :2750-2777): pixel truncated, mask == 0, 0 < depth <= 40, both flow components non-zero,
// float key + flow strictly inside the image
__device__ __forceinline__ void test_static(float kx, float ky, const int* mask, const float* depth, const float* flow, int w, int h, RenewCand& c) {
  c.flag = 0; c.fx = c.fy = c.depth = 0.f; c.sem = 0;
  const int x = (int)kx, y = (int)ky;
  c.x = x; c.y = y;
  if (x >= w || y >= h || x <= 0 || y <= 0) return;
  const size_t p = (size_t)y * w + x;
  if (mask[p] != 0) return;
  const float d = depth[p];
  if (d > 40.f || d <= 0.f) return;
  const float fx = flow[2 * p], fy = flow[2 * p + 1];
  if (fx != 0.f && fy != 0.f) {
    const float cx = __fadd_rn(kx, fx), cy = __fadd_rn(ky, fy);
    if (cx < (float)w && cy < (float)h && cx > 0.f && cy > 0.f) { c.flag = 1; c.fx = fx; c.fy = fy; c.depth = d; }
  }
}
__global__ void k_renew_inliers(int n_tm, const int* __restrict__ tm, const float* __restrict__ stat_keys, int n_oinl, const int* __restrict__ oinl,
                                const float* __restrict__ obj_keys, const int* __restrict__ mask, const float* __restrict__ depth,
                                const float* __restrict__ flow, int w, int h, RenewCand* __restrict__ sta, RenewCand* __restrict__ obj) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_tm) {
    RenewCand c; c.flag = 0; c.fx = c.fy = c.depth = 0.f; c.x = c.y = c.sem = 0;
    const int t = tm[i];
    if (t != -1) test_static(stat_keys[2 * t], stat_keys[2 * t + 1], mask, depth, flow, w, h, c);
    sta[i] = c;
  } else if (i < n_tm + n_oinl) {
    // object inlier (:2841-2866): integer pixel, mask != 0, 0 < depth < 25, integer pixel + flow strictly inside
    const int q = i - n_tm, idx = oinl[q];
    RenewCand c; c.flag = 0; c.fx = c.fy = c.depth = 0.f; c.sem = 0;
    const int x = (int)obj_keys[2 * idx], y = (int)obj_keys[2 * idx + 1];
    c.x = x; c.y = y;
    if (!(x >= w || y >= h || x <= 0 || y <= 0)) {
      const size_t p = (size_t)y * w + x;
      const float d = depth[p];
      if (mask[p] != 0 && d < 25.f && d > 0.f) {
        const float fx = flow[2 * p], fy = flow[2 * p + 1];
        const float cx = __fadd_rn((float)x, fx), cy = __fadd_rn((float)y, fy);
        if (cx < (float)w && cy < (float)h && cx > 0.f && cy > 0.f) { c.flag = 1; c.fx = fx; c.fy = fy; c.depth = d; c.sem = mask[p]; }
      }
    }
    obj[q] = c;
  }
}
// the "already used" test of the top-up loops is frame_px.cuh's near_any
__global__ void k_renew_candidates(int n_samp, const float* __restrict__ samp, int n_snap_s, const float* __restrict__ snap_s, int n_tmp,
                                   const float* __restrict__ tmp_keys, int n_snap_o, const float* __restrict__ snap_o, const int* __restrict__ mask,
                                   const float* __restrict__ depth, const float* __restrict__ flow, int w, int h, RenewCand* __restrict__ sta,
                                   unsigned char* __restrict__ tmp_used) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_samp) {
    RenewCand c; c.flag = 0; c.fx = c.fy = c.depth = 0.f; c.x = c.y = c.sem = 0;
    const float kx = samp[2 * i], ky = samp[2 * i + 1];
    if (!near_any(kx, ky, snap_s, n_snap_s)) test_static(kx, ky, mask, depth, flow, w, h, c);
    sta[i] = c;
  } else if (i < n_samp + n_tmp) {
    const int j = i - n_samp;
    tmp_used[j] = near_any(tmp_keys[2 * j], tmp_keys[2 * j + 1], snap_o, n_snap_o) ? 1 : 0;
  }
}
// Optimizer::Get3DinWorld (src/Optimizer.cc:2974-2993): float back-projection, then Rwc*x + twc as a float gemm
inline void get3d_world(float u, float v, float z, const float* K4, const float* Twc, float* X) {
  const float invfx = 1.0f / K4[0], invfy = 1.0f / K4[1];
  const float x = (u - K4[2]) * z * invfx, y = (v - K4[3]) * z * invfy;
  for (int r = 0; r < 3; ++r)
    X[r] = (float)((double)Twc[4 * r] * (double)x + (double)Twc[4 * r + 1] * (double)y + (double)Twc[4 * r + 2] * (double)z + (double)Twc[4 * r + 3]);
}
}  // namespace

extern "C" int vdo_renew_frame_info(vdo_frame* cur, int n_tm, const int* tm_sta, int n_stat, const float* stat_keys, int n_samp, const float* samp_keys,
                                    int max_num_sta, int n_obj, const int* inl_begin, const int* inl_idx, const unsigned char* obj_stat,
                                    const int* sem_position, const int* mod_label, int n_objkeys, const float* obj_keys, const int* obj_label, int n_tmp,
                                    const float* tmp_keys, const float* tmp_depth, const int* tmp_sem, const float* tmp_flow, const float* tmp_corres,
                                    int max_num_obj, const float* K4, const float* Twc, int cap_sta, int* n_sta_out, float* sta_keys, float* sta_corres,
                                    float* sta_flow, int* sta_inlier_id, float* sta_depth, float* sta_3d, int cap_obj, int* n_obj_out, float* o_keys,
                                    float* o_depth, float* o_corres, float* o_flow, int* o_sem, int* o_inlier_id, int* o_label, float* o_3d) {
  if (!cur || n_tm < 0 || n_stat < 0 || n_samp < 0 || n_obj < 0 || n_tmp < 0 || !K4 || !Twc || !n_sta_out || !n_obj_out) return VDO_ERR_ARG;
  int *mask, w, h; float *depth, *flow; void* stv;
  if (vdo_frame_device_ptrs(cur, nullptr, &depth, &flow, &mask, &w, &h, &stv)) return VDO_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stv;
  for (int i = 0; i < n_tm; ++i) if (tm_sta[i] < -1 || tm_sta[i] >= n_stat) return VDO_ERR_ARG;
  // object inlier entries of the objects that are still alive (:2833-2838)
  std::vector<int> oinl; std::vector<int> oinl_begin(n_obj + 1, 0);
  for (int i = 0; i < n_obj; ++i) {
    oinl_begin[i] = (int)oinl.size();
    if (obj_stat[i]) for (int q = inl_begin[i]; q < inl_begin[i + 1]; ++q) { if (inl_idx[q] < 0 || inl_idx[q] >= n_objkeys) return VDO_ERR_ARG; oinl.push_back(inl_idx[q]); }
  }
  oinl_begin[n_obj] = (int)oinl.size();
  const int n_oinl = (int)oinl.size();
  Arena& A = arena_begin(st);
  DevBuf b_tm, b_sk, b_oi, b_ok, b_cs, b_co, b_samp, b_tmp, b_snap_s, b_snap_o, b_cc, b_used;
  VDO_CUDA(b_tm.alloc(A, sizeof(int) * n_tm)); VDO_CUDA(b_sk.alloc(A, sizeof(float) * 2 * n_stat)); VDO_CUDA(b_oi.alloc(A, sizeof(int) * n_oinl)); VDO_CUDA(b_ok.alloc(A, sizeof(float) * 2 * n_objkeys));
  VDO_CUDA(b_cs.alloc(A, sizeof(RenewCand) * n_tm)); VDO_CUDA(b_co.alloc(A, sizeof(RenewCand) * n_oinl));
  VDO_CUDA(b_samp.alloc(A, sizeof(float) * 2 * n_samp)); VDO_CUDA(b_tmp.alloc(A, sizeof(float) * 2 * n_tmp));
  if (n_tm) VDO_CUDA(cudaMemcpyAsync(b_tm.p, tm_sta, sizeof(int) * n_tm, cudaMemcpyHostToDevice, st));
  if (n_stat) VDO_CUDA(cudaMemcpyAsync(b_sk.p, stat_keys, sizeof(float) * 2 * n_stat, cudaMemcpyHostToDevice, st));
  if (n_oinl) VDO_CUDA(cudaMemcpyAsync(b_oi.p, oinl.data(), sizeof(int) * n_oinl, cudaMemcpyHostToDevice, st));
  if (n_objkeys) VDO_CUDA(cudaMemcpyAsync(b_ok.p, obj_keys, sizeof(float) * 2 * n_objkeys, cudaMemcpyHostToDevice, st));
  if (n_samp) VDO_CUDA(cudaMemcpyAsync(b_samp.p, samp_keys, sizeof(float) * 2 * n_samp, cudaMemcpyHostToDevice, st));
  if (n_tmp) VDO_CUDA(cudaMemcpyAsync(b_tmp.p, tmp_keys, sizeof(float) * 2 * n_tmp, cudaMemcpyHostToDevice, st));
  std::vector<RenewCand> cs(n_tm), co(n_oinl);
  if (n_tm + n_oinl > 0) {
    k_renew_inliers<<<(n_tm + n_oinl + 127) / 128, 128, 0, st>>>(n_tm, b_tm.as<int>(), b_sk.as<float>(), n_oinl, b_oi.as<int>(), b_ok.as<float>(), mask, depth, flow, w, h,
                                                                  b_cs.as<RenewCand>(), b_co.as<RenewCand>());
    if (n_tm) VDO_CUDA(cudaMemcpyAsync(cs.data(), b_cs.p, sizeof(RenewCand) * n_tm, cudaMemcpyDeviceToHost, st));
    if (n_oinl) VDO_CUDA(cudaMemcpyAsync(co.data(), b_co.p, sizeof(RenewCand) * n_oinl, cudaMemcpyDeviceToHost, st));
  }
  VDO_CUDA(cudaStreamSynchronize(st));
  // ---- static (1): inliers in TM order; the size test comes after the push and uses '>' (:2706-2707) ----
  int ns = 0; bool overflow = false;
  auto push_sta = [&](float kx, float ky, const RenewCand& c, int id) {
    if (ns >= cap_sta) { overflow = true; return; }
    sta_keys[2 * ns] = kx; sta_keys[2 * ns + 1] = ky; sta_corres[2 * ns] = kx + c.fx; sta_corres[2 * ns + 1] = ky + c.fy;
    sta_flow[2 * ns] = c.fx; sta_flow[2 * ns + 1] = c.fy; sta_inlier_id[ns] = id; sta_depth[ns] = c.depth;
    get3d_world(kx, ky, c.depth, K4, Twc, sta_3d + 3 * ns);
    ++ns;
  };
  for (int i = 0; i < n_tm; ++i) {
    if (tm_sta[i] == -1) continue;
    if (cs[i].flag) push_sta(stat_keys[2 * tm_sta[i]], stat_keys[2 * tm_sta[i] + 1], cs[i], tm_sta[i]);
    if (ns > max_num_sta) break;
  }
  const int n_snap_s = ns;
  // ---- objects (1): inliers of each live object in order (:2839-2869) ----
  int no = 0;
  std::vector<int> fea_count(n_obj, -1);
  auto push_obj = [&](float kx, float ky, float d, float cx, float cy, float fx, float fy, int sem, int inl, int lab) {
    if (no >= cap_obj) { overflow = true; return; }
    o_keys[2 * no] = kx; o_keys[2 * no + 1] = ky; o_depth[no] = d; o_corres[2 * no] = cx; o_corres[2 * no + 1] = cy; o_flow[2 * no] = fx; o_flow[2 * no + 1] = fy;
    o_sem[no] = sem; o_inlier_id[no] = inl; o_label[no] = lab;
    get3d_world(kx, ky, d, K4, Twc, o_3d + 3 * no);
    ++no;
  };
  for (int i = 0; i < n_obj; ++i) {
    if (!obj_stat[i]) continue;
    int count = 0;
    for (int q = oinl_begin[i]; q < oinl_begin[i + 1]; ++q) {
      const RenewCand& c = co[q];
      if (!c.flag) continue;
      push_obj((float)c.x, (float)c.y, c.depth, (float)c.x + c.fx, (float)c.y + c.fy, c.fx, c.fy, c.sem, oinl[q], obj_label[oinl[q]]);
      ++count;
    }
    fea_count[i] = count;
  }
  const int n_snap_o = no;
  // ---- (2) top-up candidates against the two snapshots ----
  std::vector<RenewCand> cc(n_samp); std::vector<unsigned char> used(n_tmp, 0);
  const bool need_sta = ns < max_num_sta && n_samp > 0;
  bool need_obj = false;
  for (int i = 0; i < n_obj; ++i) if (obj_stat[i] && fea_count[i] < max_num_obj) need_obj = true;
  need_obj = need_obj && n_tmp > 0;
  if (need_sta || need_obj) {
    VDO_CUDA(b_snap_s.alloc(A, sizeof(float) * 2 * n_snap_s)); VDO_CUDA(b_snap_o.alloc(A, sizeof(float) * 2 * n_snap_o));
    VDO_CUDA(b_cc.alloc(A, sizeof(RenewCand) * n_samp)); VDO_CUDA(b_used.alloc(A, n_tmp));
    if (n_snap_s) VDO_CUDA(cudaMemcpyAsync(b_snap_s.p, sta_keys, sizeof(float) * 2 * n_snap_s, cudaMemcpyHostToDevice, st));
    if (n_snap_o) VDO_CUDA(cudaMemcpyAsync(b_snap_o.p, o_keys, sizeof(float) * 2 * n_snap_o, cudaMemcpyHostToDevice, st));
    const int ns_k = need_sta ? n_samp : 0, nt_k = need_obj ? n_tmp : 0;
    k_renew_candidates<<<(ns_k + nt_k + 127) / 128, 128, 0, st>>>(ns_k, b_samp.as<float>(), n_snap_s, b_snap_s.as<float>(), nt_k, b_tmp.as<float>(), n_snap_o,
                                                                  b_snap_o.as<float>(), mask, depth, flow, w, h, b_cc.as<RenewCand>(), b_used.as<unsigned char>());
    if (ns_k) VDO_CUDA(cudaMemcpyAsync(cc.data(), b_cc.p, sizeof(RenewCand) * n_samp, cudaMemcpyDeviceToHost, st));
    if (nt_k) VDO_CUDA(cudaMemcpyAsync(used.data(), b_used.p, n_tmp, cudaMemcpyDeviceToHost, st));
    VDO_CUDA(cudaStreamSynchronize(st));
  }
  {   // static top-up: passes start_id = 0..19 with stride 20 (:2719-2790)
    int tot = ns, start_id = 0; const int step = 20;
    while (tot < max_num_sta) {
      if (start_id == step) break;
      for (int i = start_id; i < n_samp; i += step) {
        if (cc[i].flag) { push_sta(samp_keys[2 * i], samp_keys[2 * i + 1], cc[i], -1); ++tot; }
        if (tot >= max_num_sta) break;
      }
      ++start_id;
    }
  }
  // object top-up: per live object, stride-15 passes over this frame's fresh samples with the same semantic label (:2873-2927)
  for (int i = 0; i < n_obj; ++i) {
    if (!obj_stat[i]) continue;
    const int sem = sem_position[i];
    int tot = fea_count[i], start_id = 0; const int step = 15;
    while (tot < max_num_obj) {
      if (start_id == step) break;
      for (int j = start_id; j < n_tmp; j += step) {
        if (tmp_sem[j] != sem) continue;
        if (used[j]) continue;
        push_obj(tmp_keys[2 * j], tmp_keys[2 * j + 1], tmp_depth[j], tmp_corres[2 * j], tmp_corres[2 * j + 1], tmp_flow[2 * j], tmp_flow[2 * j + 1], tmp_sem[j], -1, mod_label[i]);
        ++tot;
        if (tot >= max_num_obj) break;
      }
      ++start_id;
    }
  }
  // (3) objects that appear for the first time (or failed this frame): all their samples, label -2 (:2929-2972)
  {
    std::vector<int> uni(tmp_sem, tmp_sem + n_tmp);
    std::sort(uni.begin(), uni.end());
    uni.erase(std::unique(uni.begin(), uni.end()), uni.end());
    std::vector<char> known(uni.size(), 0);
    for (int i = 0; i < n_obj; ++i)
      for (size_t j = 0; j < uni.size(); ++j)
        if (uni[j] == sem_position[i] && obj_stat[i]) { known[j] = 1; break; }
    for (size_t i = 0; i < uni.size(); ++i) {
      if (known[i]) continue;
      for (int j = 0; j < n_tmp; ++j)
        if (uni[i] == tmp_sem[j])
          push_obj(tmp_keys[2 * j], tmp_keys[2 * j + 1], tmp_depth[j], tmp_corres[2 * j], tmp_corres[2 * j + 1], tmp_flow[2 * j], tmp_flow[2 * j + 1], tmp_sem[j], -1, -2);
    }
  }
  *n_sta_out = ns; *n_obj_out = no;
  return overflow ? VDO_ERR_ARG : VDO_OK;
}

// ------------------------------------------------------------------------------------------------ point look-ups
namespace {
struct GatherSeg { const float* depth; const int* mask; int begin, w, h; };   // keys [begin, next begin) of the launch read this w x h frame
__global__ void k_gather_points(int n, const GatherSeg* __restrict__ seg, int nseg, const float* __restrict__ keys, float* __restrict__ d_out,
                                int* __restrict__ m_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int s = 0;
  while (s + 1 < nseg && seg[s + 1].begin <= i) ++s;
  const float* __restrict__ depth = seg[s].depth; const int* __restrict__ mask = seg[s].mask;
  const int w = seg[s].w, h = seg[s].h;
  const int u = (int)keys[2 * i], v = (int)keys[2 * i + 1];
  const bool in = u >= 0 && u < w && v >= 0 && v < h;
  d_out[i] = in ? depth[(size_t)v * w + u] : 0.f;
  m_out[i] = in ? mask[(size_t)v * w + u] : 0;
}
}  // namespace
namespace vdo {
// segments [begin[s], begin[s + 1]) of keys (x, y interleaved) looked up in frame fs[s], one launch; the frames may differ in size
int gather_batch(vdo_frame* const* fs, int nseg, const int* begin, const float* keys, float* depth_out, int* mask_out) {
  const int n = begin[nseg];
  if (n == 0) return VDO_OK;
  void* stv;
  if (vdo_frame_device_ptrs(fs[0], nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, &stv)) return VDO_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stv;
  std::vector<GatherSeg> seg(nseg);
  for (int s = 0; s < nseg; ++s) {
    float* depth; int* mask; int w, h;
    if (vdo_frame_device_ptrs(fs[s], nullptr, &depth, nullptr, &mask, &w, &h, nullptr)) return VDO_ERR_ARG;
    seg[s] = GatherSeg{depth, mask, begin[s], w, h};
  }
  Arena& A = arena_begin(st);
  DevBuf bk, bd, bm, bs;
  VDO_CUDA(bk.alloc(A, sizeof(float) * 2 * n)); VDO_CUDA(bd.alloc(A, sizeof(float) * n)); VDO_CUDA(bm.alloc(A, sizeof(int) * n)); VDO_CUDA(bs.alloc(A, sizeof(GatherSeg) * nseg));
  VDO_CUDA(cudaMemcpyAsync(bk.p, keys, sizeof(float) * 2 * n, cudaMemcpyHostToDevice, st));
  VDO_CUDA(cudaMemcpyAsync(bs.p, seg.data(), sizeof(GatherSeg) * nseg, cudaMemcpyHostToDevice, st));
  k_gather_points<<<(n + 255) / 256, 256, 0, st>>>(n, bs.as<GatherSeg>(), nseg, bk.as<float>(), bd.as<float>(), bm.as<int>());
  VDO_CUDA(cudaGetLastError());
  VDO_CUDA(cudaMemcpyAsync(depth_out, bd.p, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaMemcpyAsync(mask_out, bm.p, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  return VDO_OK;
}
}  // namespace vdo
// depth and mask label at the truncated pixel of each key (x, y interleaved); 0 / 0 outside the image.
// Used for the "update current frame from last" look-ups of Tracking::GrabImageRGBD (src/Tracking.cc:262-312).
extern "C" int vdo_frame_gather(vdo_frame* f, int n, const float* keys, float* depth_out, int* mask_out) {
  if (!f || n < 0 || (n && (!keys || !depth_out || !mask_out))) return VDO_ERR_ARG;
  const int begin[2] = {0, n};
  return vdo::gather_batch(&f, 1, begin, keys, depth_out, mask_out);
}
