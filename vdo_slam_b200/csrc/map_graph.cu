// map_graph.cu -- the tracker's map -> factor graph construction on the device (SURVEY.md 8f N2).
//
// Tracklet tables.  Every frame that enters a tracker's map extends two tables (static and dynamic features) with that frame's
// associations, by the rule of vdo_tracklets_build (tracking_ops.cu, Tracking::GetStaticTrack / GetDynamicTrackNew): a feature whose
// association a names a previous-frame feature that belongs to a tracklet is appended to that tracklet; every other feature with
// a != -1 opens a new tracklet whose first entry is (previous frame, a).  New tracklets are numbered in feature order; two features of
// one frame that name the same tracklet are appended in feature order.  Per feature the tables keep its tracklet (-1: none, so the
// feature can only head tracklets), its position in it and the entry before it; per tracklet its length, head, last entry and, for
// dynamic tracklets, the label of the feature that opened it (ObjLab).  A frame costs one upload of its associations and one launch,
// whatever the length of the history.
//
// Graph assembly.  From the tables and the features of the frames a graph covers, the observations, points and ternary edges of
// Optimizer::PartialBatchOptimization (mode 0: the last window_size frames, static only) and FullBatchOptimization (mode 1: every
// frame) come out in the order of the host construction they replace (tracker.cpp keeps the pose vertices and SE3 edges, which
// are a handful per frame): per frame, the static observations in feature order, then the dynamic ones; a static point per tracklet
// head, a dynamic point per dynamic observation.  Which observations enter is decided per feature:
//   static  head (no tracklet of its own): it heads a tracklet of length >= 3;  else: its tracklet has length >= 3 and its head lies
//           in the graph's frames (an earlier head has no vertex, PartialBatchOptimization skips the whole chain);
//   dynamic head: as static;  else: its tracklet has length >= 3 and the frame has a motion vertex for the tracklet's ObjLab.
// A static observation uses its tracklet head's point; a kept dynamic observation whose previous entry was kept adds a ternary edge.
// Point, observation and ternary numbers come from one exclusive scan over the features of every graph of the call, so all trackers
// of a call share one upload, four launches and one read-back.
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"
#include "frame_batch.h"


namespace vdo {

namespace {
template <class T> struct DevVec {            // grow-only device array that keeps its contents
  T* p = nullptr; size_t cap = 0;
  cudaError_t reserve(size_t n, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    const size_t nc = std::max(n, std::max<size_t>(2 * cap, 4096));
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, nc * sizeof(T));
    if (e != cudaSuccess) return e;
    if (cap) {
      if ((e = cudaMemcpyAsync(q, p, cap * sizeof(T), cudaMemcpyDeviceToDevice, st)) != cudaSuccess) { cudaFree(q); return e; }
      if ((e = cudaStreamSynchronize(st)) != cudaSuccess) { cudaFree(q); return e; }
      cudaFree(p);
    }
    p = q; cap = nc;
    return cudaSuccess;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct HostStage {                            // grow-only pinned staging buffer
  char* p = nullptr; size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    const size_t nc = std::max(n, 2 * cap + (1 << 16));
    cudaError_t e = cudaMallocHost(&p, nc);
    if (e == cudaSuccess) cap = nc;
    return e;
  }
};
// upload and read-back buffers of the calls on one stream (every call ends in a synchronise of its stream, so the next can reuse them)
struct Scratch { DevVec<char> dev; HostStage up, back; };
std::mutex g_scratch_mu;
std::map<cudaStream_t, Scratch> g_scratch;
Scratch& scratch_of(cudaStream_t st) { std::lock_guard<std::mutex> lk(g_scratch_mu); return g_scratch[st]; }
template <class T> size_t put(std::vector<char>& b, const T* v, size_t n) {   // 16-byte aligned append; returns the byte offset
  const size_t off = (b.size() + 15) & ~(size_t)15;
  b.resize(off + n * sizeof(T));
  if (n) std::memcpy(b.data() + off, v, n * sizeof(T));
  return off;
}
}  // namespace

struct TrackletKind {
  DevVec<int> trk, pos, pf, pj;               // per feature (frames concatenated)
  DevVec<int> len, hf, hj, tf, tj, lab;       // per tracklet
  std::vector<long long> feat_off{0};         // per frame: first feature of the frame; back() = features so far
  std::vector<int> ntrk_after;                // per frame: tracklets once the frame's associations are in
  std::vector<int> prev_asso;                 // the last frame's associations (decides which features open tracklets)
  int n_trk = 0;
};
struct Tracklets {
  TrackletKind k[2];                          // 0 static, 1 dynamic
  bool bad = false;                           // an association outside the previous frame's features
  void release() { for (auto& t : k) { t.trk.release(); t.pos.release(); t.pf.release(); t.pj.release(); t.len.release(); t.hf.release(); t.hj.release(); t.tf.release(); t.tj.release(); t.lab.release(); } }
};
Tracklets* tracklets_create() { return new Tracklets; }
void tracklets_destroy(Tracklets* t) { if (t) { t->release(); delete t; } }
bool tracklets_bad(const Tracklets* t) { return t->bad; }
int tracklets_frames(const Tracklets* t) { return (int)t->k[0].feat_off.size() - 1; }

namespace {
struct PushJob {                              // one frame's associations into one kind of one tracker
  int *trk, *pos, *pf, *pj, *len, *hf, *hj, *tf, *tj, *lab;
  const int* asso; const int* label;          // device (inside the upload); label NULL for static
  long long off_prev, off;                    // first feature of the previous / this frame
  int n, f, trk0;
};

// one warp per job walks the frame's features in chunks of 32; a chunk's appends to one tracklet are ranked with __match_any_sync
__global__ void k_tracklets_push(const PushJob* __restrict__ jobs) {
  const PushJob J = jobs[blockIdx.x];
  const int lane = threadIdx.x;
  const unsigned lt = (1u << lane) - 1u;
  int next_new = J.trk0;
  for (int base = 0; base < J.n; base += 32) {
    const int j = base + lane;
    const int a = j < J.n ? J.asso[j] : -1;
    int t = -1;
    if (a != -1 && J.f >= 2) t = J.trk[J.off_prev + a];
    const bool fresh = a != -1 && t == -1, app = a != -1 && t != -1;
    const unsigned fm = __ballot_sync(0xffffffffu, fresh);
    int pos = 0, pf = -1, pj = -1;
    if (fresh) {
      t = next_new + __popc(fm & lt);
      J.len[t] = 2; J.hf[t] = J.f - 1; J.hj[t] = a; J.tf[t] = J.f; J.tj[t] = j;
      if (J.lab) J.lab[t] = J.label[j];
      pos = 1; pf = J.f - 1; pj = a;
    }
    next_new += __popc(fm);
    const unsigned grp = __match_any_sync(0xffffffffu, app ? t : -1);
    int L = 0;
    if (app) {
      L = J.len[t];
      const unsigned before = grp & lt;
      pos = L + __popc(before);
      if (before) { pf = J.f; pj = base + 31 - __clz(before); }
      else { pf = J.tf[t]; pj = J.tj[t]; }
    }
    __syncwarp();
    if (app && (grp >> lane) == 1u) { J.len[t] = L + __popc(grp); J.tf[t] = J.f; J.tj[t] = j; }   // the group's last lane
    if (j < J.n) { J.trk[J.off + j] = t; J.pos[J.off + j] = pos; J.pf[J.off + j] = pf; J.pj[J.off + j] = pj; }
    __syncwarp();
  }
}
}  // namespace

int tracklets_push(void* stream, Tracklets* const* T, int n, const TrackletFrame* fr) {
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<char> up;
  std::vector<PushJob> jobs;
  std::vector<size_t> asso_off, lab_off;
  for (int i = 0; i < n; ++i) {
    Tracklets& R = *T[i];
    for (int kd = 0; kd < 2; ++kd) {
      TrackletKind& K = R.k[kd];
      const int nf = kd ? fr[i].n_dyn : fr[i].n_sta;
      const int* asso = kd ? fr[i].asso_dyn : fr[i].asso_sta;
      const int f = (int)K.feat_off.size() - 1;            // index of the frame being added
      const long long off = K.feat_off.back();
      K.feat_off.push_back(off + nf);
      if (f == 0 || R.bad) { K.ntrk_after.push_back(K.n_trk); K.prev_asso.assign(nf, -1); continue; }
      const long long off_prev = K.feat_off[f - 1];
      const int n_prev = (int)(off - off_prev);
      int fresh = 0;
      for (int j = 0; j < nf; ++j) {
        const int a = asso[j];
        if (a == -1) continue;
        if (a < 0 || a >= n_prev) { R.bad = true; break; }
        if (f == 1 || K.prev_asso[a] == -1) ++fresh;
      }
      if (R.bad) { K.ntrk_after.push_back(K.n_trk); continue; }
      cudaError_t e = cudaSuccess;
      for (DevVec<int>* v : {&K.trk, &K.pos, &K.pf, &K.pj}) if (e == cudaSuccess) e = v->reserve((size_t)off + nf + 1, st);
      for (DevVec<int>* v : {&K.len, &K.hf, &K.hj, &K.tf, &K.tj, &K.lab}) if (e == cudaSuccess) e = v->reserve((size_t)K.n_trk + fresh + 1, st);
      VDO_CUDA(e);
      PushJob J{K.trk.p, K.pos.p, K.pf.p, K.pj.p, K.len.p, K.hf.p, K.hj.p, K.tf.p, K.tj.p, kd ? K.lab.p : nullptr, nullptr, nullptr, off_prev, off, nf, f, K.n_trk};
      jobs.push_back(J);
      asso_off.push_back(put(up, asso, nf));
      lab_off.push_back(kd ? put(up, fr[i].label_dyn, nf) : 0);
      K.n_trk += fresh;
      K.ntrk_after.push_back(K.n_trk);
      K.prev_asso.assign(asso, asso + nf);
    }
  }
  if (jobs.empty()) return VDO_OK;
  const size_t jobs_off = put(up, jobs.data(), jobs.size());
  Scratch& sc = scratch_of(st);
  HostStage& stage = sc.up;
  DevVec<char>& dev = sc.dev;
  VDO_CUDA(stage.reserve(up.size()));
  std::memcpy(stage.p, up.data(), up.size());
  VDO_CUDA(dev.reserve(up.size(), st));
  for (size_t q = 0; q < jobs.size(); ++q) {
    PushJob* J = (PushJob*)(stage.p + jobs_off) + q;
    J->asso = (const int*)(dev.p + asso_off[q]);
    J->label = J->lab ? (const int*)(dev.p + lab_off[q]) : nullptr;
  }
  VDO_CUDA(cudaMemcpyAsync(dev.p, stage.p, up.size(), cudaMemcpyHostToDevice, st));
  k_tracklets_push<<<(int)jobs.size(), 32, 0, st>>>((const PushJob*)(dev.p + jobs_off));
  VDO_CUDA(cudaGetLastError());
  VDO_CUDA(cudaStreamSynchronize(st));
  return VDO_OK;
}

int tracklets_read(void* stream, const Tracklets* T, int kind, TrackletDump* out) {
  cudaStream_t st = (cudaStream_t)stream;
  const TrackletKind& K = T->k[kind];
  const size_t nf = (size_t)K.feat_off.back(), nt = (size_t)K.n_trk;
  out->feat_off.assign(K.feat_off.begin(), K.feat_off.end());
  std::vector<int>* fv[4] = {&out->trk, &out->pos, &out->pf, &out->pj};
  const DevVec<int>* fd[4] = {&K.trk, &K.pos, &K.pf, &K.pj};
  std::vector<int>* tv[4] = {&out->len, &out->hf, &out->hj, &out->lab};
  const DevVec<int>* td[4] = {&K.len, &K.hf, &K.hj, &K.lab};
  // frame 0 has no associations: its features are never appended, and the tables only cover features the kernel wrote
  const size_t first = K.feat_off.size() > 1 ? (size_t)K.feat_off[1] : nf;
  for (int q = 0; q < 4; ++q) {
    fv[q]->assign(nf, q == 1 ? 0 : -1);
    if (nf > first) VDO_CUDA(cudaMemcpyAsync(fv[q]->data() + first, fd[q]->p + first, (nf - first) * sizeof(int), cudaMemcpyDeviceToHost, st));
    tv[q]->assign(nt, 0);
    if (nt && (kind == 1 || q < 3)) VDO_CUDA(cudaMemcpyAsync(tv[q]->data(), td[q]->p, nt * sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  VDO_CUDA(cudaStreamSynchronize(st));
  return VDO_OK;
}

// ------------------------------------------------------------------------------------------------ graph assembly
namespace {
struct FrameRow {                             // one frame of one graph
  int slot;                                   // first slot of the frame (slots: static features, then dynamic, frame after frame)
  int n_sta, n_dyn, cam, mot_begin, mot_n, f;
  long long sta_off, dyn_off;                 // first feature of the frame in the tracklet tables
};
struct GraphJob {
  const int *s_trk, *s_len, *s_hf, *s_hj, *s_pf, *s_pj;
  const int *d_trk, *d_len, *d_hf, *d_hj, *d_pf, *d_pj, *d_lab;
  const FrameRow* rows; const float* feat;    // 6 floats per slot: u, v, depth, X, Y, Z
  const int* mot;                             // (label, vertex) pairs of the frames' object motions
  int n_rows, start, slot0, n_slots, s_t0, s_nt, d_t0, d_nt;
  float invfx, invfy, cx, cy;
  // outputs (device; layout sized by n_slots)
  int* totals; double* pt; int* obs_cp; double* obs_z; int* ter; int* mak;
};
struct Cnt { int pt, obs, ter, pad; };
struct CntSum { __device__ Cnt operator()(const Cnt& a, const Cnt& b) const { return Cnt{a.pt + b.pt, a.obs + b.obs, a.ter + b.ter, 0}; } };

__device__ int row_of(const GraphJob& G, int s) {          // frame row holding slot s (s relative to the graph)
  int lo = 0, hi = G.n_rows - 1;
  while (lo < hi) { const int m = (lo + hi + 1) >> 1; if (G.rows[m].slot <= s) lo = m; else hi = m - 1; }
  return lo;
}
__device__ int row_of_frame(const GraphJob& G, int f) { return f - G.start; }
__device__ int objv_of(const GraphJob& G, const FrameRow& r, int label) {
  for (int k = 0; k < r.mot_n; ++k) if (G.mot[2 * (r.mot_begin + k)] == label) return G.mot[2 * (r.mot_begin + k) + 1];
  return -1;
}

// heads of tracklets of length >= 3 whose head lies in the graph
__global__ void k_mark_heads(const GraphJob* __restrict__ jobs, int* __restrict__ head) {
  const GraphJob& G = jobs[blockIdx.y];
  for (int kd = 0; kd < 2; ++kd) {
    const int t0 = kd ? G.d_t0 : G.s_t0, nt = kd ? G.d_nt : G.s_nt;
    const int *len = kd ? G.d_len : G.s_len, *hf = kd ? G.d_hf : G.s_hf, *hj = kd ? G.d_hj : G.s_hj;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nt; q += gridDim.x * blockDim.x) {
      const int t = t0 + q;
      if (len[t] < 3) continue;
      const FrameRow& r = G.rows[row_of_frame(G, hf[t])];
      head[G.slot0 + r.slot + (kd ? r.n_sta : 0) + hj[t]] = 1;
    }
  }
}

struct Decision { bool kept, new_pt; int trk, row, kd, j; };
__device__ Decision decide(const GraphJob& G, const int* head, int s) {
  Decision d{false, false, -1, row_of(G, s), 0, 0};
  const FrameRow& r = G.rows[d.row];
  d.j = s - r.slot;
  if (d.j >= r.n_sta) { d.kd = 1; d.j -= r.n_sta; }
  if (!d.kd) {
    d.trk = r.f == 0 ? -1 : G.s_trk[r.sta_off + d.j];
    d.kept = d.trk == -1 ? head[G.slot0 + s] != 0 : (G.s_len[d.trk] >= 3 && G.s_hf[d.trk] >= G.start);
    d.new_pt = d.kept && d.trk == -1;
  } else {
    d.trk = r.f == 0 ? -1 : G.d_trk[r.dyn_off + d.j];
    d.kept = d.trk == -1 ? head[G.slot0 + s] != 0 : (G.d_len[d.trk] >= 3 && objv_of(G, r, G.d_lab[d.trk]) != -1);
    d.new_pt = d.kept;
  }
  return d;
}
// the slot of the entry before a kept dynamic observation, or -1 when that entry has no point
__device__ int prev_dyn_slot(const GraphJob& G, const int* head, const Decision& d) {
  const FrameRow& r = G.rows[d.row];
  const long long q = r.dyn_off + d.j;
  const int pf = G.d_pf[q], pj = G.d_pj[q];
  const FrameRow& rp = G.rows[row_of_frame(G, pf)];
  const int sp = rp.slot + rp.n_sta + pj;
  const int ptrk = rp.f == 0 ? -1 : G.d_trk[rp.dyn_off + pj];
  const bool kept = ptrk == -1 ? head[G.slot0 + sp] != 0 : (G.d_len[ptrk] >= 3 && objv_of(G, rp, G.d_lab[ptrk]) != -1);
  return kept ? sp : -1;
}

__global__ void k_decide(const GraphJob* __restrict__ jobs, const int* __restrict__ head, Cnt* __restrict__ cnt) {
  const GraphJob& G = jobs[blockIdx.y];
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < G.n_slots; s += gridDim.x * blockDim.x) {
    const Decision d = decide(G, head, s);
    Cnt c{d.new_pt ? 1 : 0, d.kept ? 1 : 0, 0, 0};
    if (d.kd && d.kept && d.trk != -1) c.ter = prev_dyn_slot(G, head, d) != -1 ? 1 : 0;
    cnt[G.slot0 + s] = c;
  }
}

// Optimizer::Get3DinCamera in float, rounded step by step like the host
__device__ void get3d(const GraphJob& G, const float* f, double* z) {
  const float u = f[0], v = f[1], dep = f[2];
  z[0] = (double)__fmul_rn(__fmul_rn(__fsub_rn(u, G.cx), dep), G.invfx);
  z[1] = (double)__fmul_rn(__fmul_rn(__fsub_rn(v, G.cy), dep), G.invfy);
  z[2] = (double)dep;
}

__global__ void k_write(const GraphJob* __restrict__ jobs, const int* __restrict__ head, const Cnt* __restrict__ scan) {
  const GraphJob& G = jobs[blockIdx.y];
  const Cnt b = scan[G.slot0];
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= G.n_slots; s += gridDim.x * blockDim.x) {
    const Cnt c = scan[G.slot0 + s];
    if (s == G.n_slots) { G.totals[0] = c.pt - b.pt; G.totals[1] = c.obs - b.obs; G.totals[2] = c.ter - b.ter; continue; }
    const Decision d = decide(G, head, s);
    if (!d.kept) { G.mak[s] = -1; continue; }
    const FrameRow& r = G.rows[d.row];
    const float* f = G.feat + 6 * (size_t)s;
    int p;
    if (d.new_pt) {
      p = c.pt - b.pt;
      for (int k = 0; k < 3; ++k) G.pt[3 * (size_t)p + k] = (double)f[3 + k];
    } else {                                                   // static: the point of the tracklet's head
      const FrameRow& rh = G.rows[row_of_frame(G, G.s_hf[d.trk])];
      p = scan[G.slot0 + rh.slot + G.s_hj[d.trk]].pt - b.pt;
    }
    const int o = c.obs - b.obs;
    G.obs_cp[2 * o] = r.cam; G.obs_cp[2 * o + 1] = p;
    get3d(G, f, &G.obs_z[3 * (size_t)o]);
    G.mak[s] = p;
    if (d.kd && d.trk != -1) {
      const int sp = prev_dyn_slot(G, head, d);
      if (sp != -1) {
        const int e = c.ter - b.ter;
        G.ter[3 * e] = scan[G.slot0 + sp].pt - b.pt; G.ter[3 * e + 1] = p; G.ter[3 * e + 2] = objv_of(G, r, G.d_lab[d.trk]);
      }
    }
  }
}
}  // namespace

int graphs_assemble(void* stream, int n, const GraphInput* in, GraphOutput* out) {
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<char> up;
  std::vector<GraphJob> jobs(n);
  std::vector<size_t> rows_off(n), feat_off(n), mot_off(n);
  int total = 0;
  size_t out_bytes = 0;
  std::vector<size_t> o_tot(n), o_pt(n), o_cz(n), o_cp(n), o_ter(n), o_mak(n);
  auto grow = [&](size_t bytes) { const size_t off = (out_bytes + 15) & ~(size_t)15; out_bytes = off + bytes; return off; };
  for (int i = 0; i < n; ++i) {
    const GraphInput& g = in[i];
    const Tracklets& R = *g.tables;
    GraphJob& J = jobs[i];
    const TrackletKind &S = R.k[0], &D = R.k[1];
    J = GraphJob{S.trk.p, S.len.p, S.hf.p, S.hj.p, S.pf.p, S.pj.p, D.trk.p, D.len.p, D.hf.p, D.hj.p, D.pf.p, D.pj.p, D.lab.p, nullptr, nullptr, nullptr,
                 (int)g.rows.size(), g.start, total, g.n_slots, S.ntrk_after[g.start], S.n_trk - S.ntrk_after[g.start],
                 g.dynamic ? D.ntrk_after[g.start] : 0, g.dynamic ? D.n_trk - D.ntrk_after[g.start] : 0, g.invfx, g.invfy, g.cx, g.cy,
                 nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    std::vector<FrameRow> rows(g.rows.size());
    for (size_t q = 0; q < g.rows.size(); ++q) {
      const GraphRow& a = g.rows[q];
      rows[q] = FrameRow{a.slot, a.n_sta, a.n_dyn, a.cam, a.mot_begin, a.mot_n, g.start + (int)q, S.feat_off[g.start + q], D.feat_off[g.start + q]};
    }
    rows_off[i] = put(up, rows.data(), rows.size());
    feat_off[i] = put(up, g.feat.data(), g.feat.size());
    mot_off[i] = put(up, g.mot.data(), g.mot.size());
    total += g.n_slots;
    const size_t ns = (size_t)g.n_slots + 1;
    o_tot[i] = grow(4 * sizeof(int)); o_pt[i] = grow(3 * ns * sizeof(double)); o_cz[i] = grow(3 * ns * sizeof(double));
    o_cp[i] = grow(2 * ns * sizeof(int)); o_ter[i] = grow(3 * ns * sizeof(int)); o_mak[i] = grow(ns * sizeof(int));
  }
  const size_t jobs_off = put(up, jobs.data(), jobs.size());
  // device scratch: upload | head flags | counts | scan | cub temp | outputs
  size_t cub_bytes = 0;
  cub::DeviceScan::ExclusiveScan((void*)nullptr, cub_bytes, (const Cnt*)nullptr, (Cnt*)nullptr, CntSum(), Cnt{0, 0, 0, 0}, total + 1, st);
  const size_t a_up = 0, a_head = (up.size() + 255) & ~(size_t)255, a_cnt = a_head + (((size_t)total + 1) * sizeof(int) + 255) / 256 * 256;
  const size_t a_scan = a_cnt + ((size_t)total + 1) * sizeof(Cnt), a_cub = (a_scan + ((size_t)total + 1) * sizeof(Cnt) + 255) & ~(size_t)255;
  const size_t a_out = (a_cub + cub_bytes + 255) & ~(size_t)255, bytes = a_out + out_bytes;
  Scratch& sc = scratch_of(st);
  DevVec<char>& dev = sc.dev;
  HostStage &stage = sc.up, &back = sc.back;
  VDO_CUDA(dev.reserve(bytes, st));
  VDO_CUDA(stage.reserve(up.size()));
  VDO_CUDA(back.reserve(out_bytes));
  char* base = dev.p;
  for (int i = 0; i < n; ++i) {
    GraphJob& J = jobs[i];
    J.rows = (const FrameRow*)(base + a_up + rows_off[i]); J.feat = (const float*)(base + a_up + feat_off[i]); J.mot = (const int*)(base + a_up + mot_off[i]);
    char* o = base + a_out;
    J.totals = (int*)(o + o_tot[i]); J.pt = (double*)(o + o_pt[i]); J.obs_z = (double*)(o + o_cz[i]); J.obs_cp = (int*)(o + o_cp[i]);
    J.ter = (int*)(o + o_ter[i]); J.mak = (int*)(o + o_mak[i]);
  }
  std::memcpy(up.data() + jobs_off, jobs.data(), jobs.size() * sizeof(GraphJob));
  std::memcpy(stage.p, up.data(), up.size());
  int max_slots = 1;
  for (int i = 0; i < n; ++i) max_slots = std::max(max_slots, in[i].n_slots + 1);
  const GraphJob* dj = (const GraphJob*)(base + a_up + jobs_off);
  int* head = (int*)(base + a_head);
  Cnt* cnt = (Cnt*)(base + a_cnt);
  Cnt* scan = (Cnt*)(base + a_scan);
  VDO_CUDA(cudaMemcpyAsync(base, stage.p, up.size(), cudaMemcpyHostToDevice, st));
  VDO_CUDA(cudaMemsetAsync(head, 0, ((size_t)total + 1) * sizeof(int), st));
  VDO_CUDA(cudaMemsetAsync(cnt + total, 0, sizeof(Cnt), st));
  const dim3 blk(256), grd((unsigned)std::min((max_slots + 255) / 256, 1024), (unsigned)n);
  k_mark_heads<<<grd, blk, 0, st>>>(dj, head);
  k_decide<<<grd, blk, 0, st>>>(dj, head, cnt);
  VDO_CUDA(cub::DeviceScan::ExclusiveScan(base + a_cub, cub_bytes, cnt, scan, CntSum(), Cnt{0, 0, 0, 0}, total + 1, st));
  k_write<<<grd, blk, 0, st>>>(dj, head, scan);
  VDO_CUDA(cudaGetLastError());
  VDO_CUDA(cudaMemcpyAsync(back.p, base + a_out, out_bytes, cudaMemcpyDeviceToHost, st));
  VDO_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    const char* o = back.p;
    const int* tot = (const int*)(o + o_tot[i]);
    GraphOutput& R = out[i];
    R.pt.assign((const double*)(o + o_pt[i]), (const double*)(o + o_pt[i]) + 3 * (size_t)tot[0]);
    R.obs_cp.assign((const int*)(o + o_cp[i]), (const int*)(o + o_cp[i]) + 2 * (size_t)tot[1]);
    R.obs_z.assign((const double*)(o + o_cz[i]), (const double*)(o + o_cz[i]) + 3 * (size_t)tot[1]);
    R.ter_pph.assign((const int*)(o + o_ter[i]), (const int*)(o + o_ter[i]) + 3 * (size_t)tot[2]);
    R.mak.assign((const int*)(o + o_mak[i]), (const int*)(o + o_mak[i]) + in[i].n_slots);
  }
  return VDO_OK;
}

}  // namespace vdo
