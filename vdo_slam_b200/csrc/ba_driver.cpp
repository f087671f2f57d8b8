// ba_driver.cpp -- see ba_driver.h.  Pure host C++: no CUDA calls here, everything device-side goes through BaBackend.
#include "ba_driver.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <numeric>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <unistd.h>

namespace vdo {

namespace {
// Host-side worker threads of finalize() (graph ingestion is memory-latency-bound scatter work; the reference's own
// graph construction is single-threaded, src/Optimizer.cc:1232-1930).  VDO_HOST_THREADS overrides the default.
int host_threads() {
  const char* e = std::getenv("VDO_HOST_THREADS");
  const int v = e ? std::atoi(e) : (int)std::min(32u, std::max(1u, std::thread::hardware_concurrency()));
  return std::max(1, std::min(v, 64));
}
// Worker pool of the host-side ingest: the ~30 parallel sections of one finalize() would otherwise create and join their threads each time
// (15 threads x 30 sections: milliseconds of pure thread start-up per graph).  Sections are serialised (one pool per process); a section
// started from inside a worker runs inline.
class HostPool {
 public:
  ~HostPool() {
    { std::lock_guard<std::mutex> lk(m_); stop_ = true; ++gen_; }
    cv_work_.notify_all();
    for (auto& t : th_) t.join();
  }
  void run(int nthreads, const std::function<void(int, int)>& fn) {
    if (nthreads <= 1 || inside_) { for (int t = 0; t < nthreads; ++t) fn(t, nthreads); return; }
    std::lock_guard<std::mutex> section(run_);
    {
      std::lock_guard<std::mutex> lk(m_);
      if (pid_ != getpid()) {          // forked child: the parent's workers do not exist here (their std::thread objects are abandoned, not joined)
        new std::vector<std::thread>(std::move(th_));
        th_.clear(); pid_ = getpid();
      }
      while ((int)th_.size() < nthreads - 1) { const int id = (int)th_.size() + 1; th_.emplace_back([this, id] { worker(id); }); }
      fn_ = &fn; n_ = nthreads; pending_ = nthreads - 1; ++gen_;
    }
    cv_work_.notify_all();
    inside_ = true; fn(0, nthreads); inside_ = false;
    std::unique_lock<std::mutex> lk(m_);
    cv_done_.wait(lk, [this] { return pending_ == 0; });
    fn_ = nullptr;
  }
 private:
  void worker(int id) {
    inside_ = true;
    unsigned long seen = 0;
    for (;;) {
      const std::function<void(int, int)>* fn = nullptr; int n = 0;
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_work_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
        if (id < n_) { fn = fn_; n = n_; }
      }
      if (!fn) continue;
      (*fn)(id, n);
      std::lock_guard<std::mutex> lk(m_);
      if (--pending_ == 0) cv_done_.notify_one();
    }
  }
  std::vector<std::thread> th_;
  std::mutex m_, run_;
  std::condition_variable cv_work_, cv_done_;
  const std::function<void(int, int)>* fn_ = nullptr;
  int n_ = 0, pending_ = 0;
  unsigned long gen_ = 0;
  bool stop_ = false;
  pid_t pid_ = getpid();
  static thread_local bool inside_;
};
thread_local bool HostPool::inside_ = false;
HostPool& host_pool() { static HostPool* p = new HostPool; return *p; }     // leaked on purpose: no joins during static destruction
template <typename F> void parallel_for(int nthreads, F fn) {   // fn(thread index, thread count)
  if (nthreads <= 1) { fn(0, 1); return; }
  const std::function<void(int, int)> f = fn;
  host_pool().run(nthreads, f);
}
struct Phase {
  BaBackend* be; float* acc; bool on;
  Phase(BaBackend* b, float* a, bool o) : be(b), acc(a), on(o) { if (on) be->timer_start(3); }
  ~Phase() { if (on) *acc += be->timer_stop_ms(3); }
};
}  // namespace

void BaGraph::copy_bytes(void* dst, const void* src, size_t bytes) {
  if (bytes < ((size_t)4 << 20)) { std::memcpy(dst, src, bytes); return; }
  parallel_for(std::min(host_threads(), 16), [&](int t, int n) {
    const size_t a = (bytes * t / n) & ~(size_t)63, b = t + 1 == n ? bytes : ((bytes * (t + 1) / n) & ~(size_t)63);
    std::memcpy((char*)dst + a, (const char*)src + a, b - a);
  });
}
void BaGraph::fill_bytes(void* dst, int byte, size_t bytes) {
  if (bytes < ((size_t)8 << 20)) { std::memset(dst, byte, bytes); return; }
  parallel_for(std::min(host_threads(), 8), [&](int t, int n) {
    const size_t a = (bytes * t / n) & ~(size_t)63, b = t + 1 == n ? bytes : ((bytes * (t + 1) / n) & ~(size_t)63);
    std::memset((char*)dst + a, byte, b - a);
  });
}

BaGraph::~BaGraph() {
  if (finalized_) be_->release(d_);
  drop_stage();
  for (void* p : owned_) be_->free_(p);
}

int BaGraph::set_vertices(int n_se3, const double* se3, int n_pt, const double* pt) {
  if (finalized_) return fail(VDO_ERR_STATE, "set_vertices after finalize");
  if (n_se3 < 0 || n_pt < 0 || (n_se3 && !se3) || (n_pt && !pt)) return fail(VDO_ERR_ARG, "set_vertices: bad arguments");
  n_se3_ = n_se3; n_pt_ = n_pt;
  h_se3_ = HostBuf<double>(); h_pt_ = HostBuf<double>();
  append(h_se3_, se3, 12 * (size_t)n_se3);
  append(h_pt_, pt, 3 * (size_t)n_pt);
  return VDO_OK;
}
int BaGraph::add_prior(int n, const int* v, const double* Z, const double* w) {
  if (finalized_) return fail(VDO_ERR_STATE, "add after finalize");
  for (int i = 0; i < n; ++i) if (v[i] < 0 || v[i] >= n_se3_) return fail(VDO_ERR_ARG, "prior edge: vertex out of range");
  pr_v_.insert(pr_v_.end(), v, v + n); pr_Z_.insert(pr_Z_.end(), Z, Z + 12 * (size_t)n); pr_w_.insert(pr_w_.end(), w, w + n);
  return VDO_OK;
}
int BaGraph::add_se3(int n, const int* ij, const double* Z, const double* w, const double* delta) {
  if (finalized_) return fail(VDO_ERR_STATE, "add after finalize");
  for (int i = 0; i < 2 * n; ++i) if (ij[i] < 0 || ij[i] >= n_se3_) return fail(VDO_ERR_ARG, "se3 edge: vertex out of range");
  for (int i = 0; i < n; ++i) if (ij[2 * i] == ij[2 * i + 1]) return fail(VDO_ERR_ARG, "se3 edge: self loop");
  se_ij_.insert(se_ij_.end(), ij, ij + 2 * (size_t)n); se_Z_.insert(se_Z_.end(), Z, Z + 12 * (size_t)n);
  se_w_.insert(se_w_.end(), w, w + n); se_d_.insert(se_d_.end(), delta, delta + n);
  return VDO_OK;
}
int BaGraph::add_obs(int n, const int* cp, const double* z, const double* w, const double* delta) {
  if (finalized_) return fail(VDO_ERR_STATE, "add after finalize");
  for (int i = 0; i < n; ++i)
    if (cp[2 * i] < 0 || cp[2 * i] >= n_se3_ || cp[2 * i + 1] < 0 || cp[2 * i + 1] >= n_pt_) return fail(VDO_ERR_ARG, "pointxyz edge: vertex out of range");
  append(ob_cp_, cp, 2 * (size_t)n); append(ob_z_, z, 3 * (size_t)n);
  append(ob_w_, w, (size_t)n); append(ob_d_, delta, (size_t)n);
  return VDO_OK;
}
int BaGraph::add_ter(int n, const int* pph, const double* w, const double* delta) {
  if (finalized_) return fail(VDO_ERR_STATE, "add after finalize");
  for (int i = 0; i < n; ++i)
    if (pph[3 * i] < 0 || pph[3 * i] >= n_pt_ || pph[3 * i + 1] < 0 || pph[3 * i + 1] >= n_pt_ || pph[3 * i + 2] < 0 || pph[3 * i + 2] >= n_se3_)
      return fail(VDO_ERR_ARG, "landmark-motion edge: vertex out of range");
  append(te_pph_, pph, 3 * (size_t)n); append(te_w_, w, (size_t)n); append(te_d_, delta, (size_t)n);
  return VDO_OK;
}

namespace {
// [a, b): part t of an even split of [0, n) over nt host threads
std::pair<int, int> thread_range(int n, int t, int nt) { return {(int)((int64_t)n * t / nt), (int)((int64_t)n * (t + 1) / nt)}; }
// Path-forcing switches for comparing two solver paths on one graph: VDO_BA_LAYOUT=chunked, VDO_BA_DENSE=0, VDO_BA_BAND=0.
struct Switches { bool chunked, dense, band; };
Switches read_switches() {
  auto is = [](const char* name, const char* v) { const char* e = std::getenv(name); return e && std::string(e) == v; };
  return Switches{is("VDO_BA_LAYOUT", "chunked"), !is("VDO_BA_DENSE", "0"), !is("VDO_BA_BAND", "0")}; }
struct ClassTable {
  std::map<std::pair<double, double>, int> ids;
  std::vector<double> w, d;
  int get(double ww, double dd) {
    auto key = std::make_pair(ww, dd > 0 ? dd : 0.0);
    auto it = ids.find(key);
    if (it != ids.end()) return it->second;
    int id = (int)w.size();
    ids[key] = id; w.push_back(ww); d.push_back(key.second);
    return id;
  }
};
// Stable counting sort of items [0, n) by se3 vertex (vertex_of(i) < 0: no vertex): put(i, slot) for every item in order, and the
// chunks of at most VDO_CHUNK slots of one vertex
template <typename V, typename F> void vertex_major(int C, int n, V vertex_of, F put, std::vector<Chunk>& chunks) {
  std::vector<int> begin(C + 1, 0);
  for (int i = 0; i < n; ++i) if (vertex_of(i) >= 0) begin[vertex_of(i) + 1]++;
  for (int v = 0; v < C; ++v) begin[v + 1] += begin[v];
  std::vector<int> fill(begin.begin(), begin.end() - 1);
  for (int i = 0; i < n; ++i) if (vertex_of(i) >= 0) put(i, fill[vertex_of(i)]++);
  for (int v = 0; v < C; ++v)
    for (int b = begin[v]; b < begin[v + 1]; b += VDO_CHUNK) chunks.push_back(Chunk{v, b, std::min(b + VDO_CHUNK, begin[v + 1]), 0});
}
// stable counting sort of ids by key_of_id[id], in parallel: chunk t of the list counts its keys, the (key, chunk) prefix gives every chunk
// its output cursor per key, every chunk scatters its ids in order -- the result of a stable sort does not depend on the thread count
void counting_sort(std::vector<int>& ids, const HostBuf<int>& key_of_id, int nkeys, int NT) {
  const int n = (int)ids.size();
  if (n == 0) return;
  const int W = (n < 65536 || (size_t)nkeys * NT > 4 * (size_t)n) ? 1 : NT;
  std::vector<int> keys(n), out(n), hist((size_t)W * nkeys, 0);
  parallel_for(W, [&](int t, int w) {
    const auto [a, b] = thread_range(n, t, w);
    int* h = &hist[(size_t)t * nkeys];
    for (int i = a; i < b; ++i) { const int k = key_of_id[ids[i]]; keys[i] = k; h[k]++; }
  });
  { int run = 0; for (int k = 0; k < nkeys; ++k) for (int t = 0; t < W; ++t) { int& h = hist[(size_t)t * nkeys + k]; const int c = h; h = run; run += c; } }
  parallel_for(W, [&](int t, int w) {
    const auto [a, b] = thread_range(n, t, w);
    int* h = &hist[(size_t)t * nkeys];
    for (int i = a; i < b; ++i) out[h[keys[i]]++] = ids[i];
  });
  ids.swap(out);
}
// se3 vertices: renumber so that every path of the se3-se3 edge graph (camera odometry chain, per-object motion-smoothness chains) is
// a contiguous, ordered index range; other vertices become singleton paths.  Returns path_begin.
std::vector<int> se3_path_order(int C, const std::vector<int>& se_ij, std::vector<int>& new_of_old) {
  const int Es = (int)se_ij.size() / 2;
  std::vector<int> path_begin, deg(C, 0), nb0(C, -1), nb1(C, -1), comp(C);
  std::iota(comp.begin(), comp.end(), 0);
  auto find = [&](int x) { while (comp[x] != x) { comp[x] = comp[comp[x]]; x = comp[x]; } return x; };
  std::vector<char> bad_comp(C, 0);
  for (int e = 0; e < Es; ++e) {
    int a = se_ij[2 * e], b = se_ij[2 * e + 1];
    int ra = find(a), rb = find(b);
    if (ra == rb) bad_comp[ra] = 1;            // cycle or duplicate edge
    else { comp[ra] = rb; if (bad_comp[ra]) bad_comp[rb] = 1; }
    if (deg[a] == 0) nb0[a] = b; else if (deg[a] == 1) nb1[a] = b;
    if (deg[b] == 0) nb0[b] = a; else if (deg[b] == 1) nb1[b] = a;
    deg[a]++; deg[b]++;
  }
  for (int v = 0; v < C; ++v) if (deg[v] > 2) bad_comp[find(v)] = 1;
  new_of_old.assign(C, -1);
  int cnt = 0;
  for (int v = 0; v < C; ++v) {
    if (new_of_old[v] != -1) continue;
    const bool is_path = !bad_comp[find(v)];
    if (!is_path || deg[v] == 0) { path_begin.push_back(cnt); new_of_old[v] = cnt++; continue; }
    if (deg[v] == 2) continue;                 // interior vertex: reached from its path's smaller endpoint
    path_begin.push_back(cnt);
    int prev = -1, cur = v;
    while (cur != -1) {
      new_of_old[cur] = cnt++;
      int nx = (nb0[cur] != prev) ? nb0[cur] : nb1[cur];
      if (deg[cur] == 1 && prev != -1) nx = -1;
      prev = cur; cur = nx;
    }
  }
  for (int v = 0; v < C; ++v) if (new_of_old[v] == -1) { path_begin.push_back(cnt); new_of_old[v] = cnt++; }  // safety
  path_begin.push_back(cnt);
  return path_begin;
}
// Tiles of whole tracklets: at most VDO_TILE_L landmarks and VDO_TILE_E pointxyz edges each.  False when a tracklet does not fit in a
// tile; the graph then takes the chunked vertex-major layout.
// Greedy packing inside FIXED segments of the tracklet order (their number depends on the graph only, so the layout is the same for any
// thread count); a tile never spans two segments, hence the segments pack in parallel.  A tile also meets at most 255 distinct cameras
// (edges address them by an 8-bit slot): cam_tile[c] = serial of the tile that saw camera c last.
bool pack_tiles(const std::vector<int>& tk_begin, int Tstat, const HostBuf<int>& lm_begin, const HostBuf<int>& lm_cam, int C, int NT,
                std::vector<Tile>& tiles, int& n_stat) {
  const int T = (int)tk_begin.size() - 1, nseg_st = std::max(1, std::min(48, Tstat / 8192)), nseg_ch = std::max(1, std::min(16, (T - Tstat) / 2048));
  struct SegOut { std::vector<Tile> tiles; int bad = 0; };
  std::vector<SegOut> segs((size_t)nseg_st + nseg_ch);
  auto pack = [&](int t_lo, int t_hi, SegOut& out) {
    if (t_lo >= t_hi) return;
    Tile cur{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<int> cam_tile(C, -1), fresh;
    int tile_serial = 0, ncam_cur = 0;
    auto close = [&](int t) {
      if (cur.t1 > cur.t0) out.tiles.push_back(cur);
      cur.t0 = cur.t1 = t; cur.k0 = cur.k1 = tk_begin[t]; cur.e0 = cur.e1 = lm_begin[tk_begin[t]];
      ++tile_serial; ncam_cur = 0;
    };
    close(t_lo);
    for (int t = t_lo; t < t_hi; ++t) {
      const int nl = tk_begin[t + 1] - tk_begin[t], ea = lm_begin[tk_begin[t]], eb = lm_begin[tk_begin[t + 1]], ne = eb - ea;
      if (nl > VDO_TILE_L || ne > VDO_TILE_E) { out.bad = 1; return; }
      auto count_fresh = [&]() { fresh.clear(); for (int e = ea; e < eb; ++e) if (cam_tile[lm_cam[e]] != tile_serial) { cam_tile[lm_cam[e]] = tile_serial; fresh.push_back(lm_cam[e]); } };
      count_fresh();
      if ((cur.k1 - cur.k0) + nl > VDO_TILE_L || (cur.e1 - cur.e0) + ne > VDO_TILE_E || ncam_cur + (int)fresh.size() > 255) { close(t); count_fresh(); }
      if ((int)fresh.size() > 255) { out.bad = 1; return; }                 // one tracklet seen by more than 255 cameras
      ncam_cur += (int)fresh.size();
      cur.t1 = t + 1; cur.k1 = tk_begin[t + 1]; cur.e1 = eb;
    }
    if (cur.t1 > cur.t0) out.tiles.push_back(cur);
  };
  const int nseg = nseg_st + nseg_ch;
  parallel_for(std::min(NT, nseg), [&](int w, int n) {
    for (int sg = w; sg < nseg; sg += n) {
      const bool st = sg < nseg_st;
      const auto [a, b] = st ? thread_range(Tstat, sg, nseg_st) : thread_range(T - Tstat, sg - nseg_st, nseg_ch);
      pack(st ? a : Tstat + a, st ? b : Tstat + b, segs[sg]);
    }
  });
  for (int sg = 0; sg < nseg; ++sg) {
    if (segs[sg].bad) { tiles.clear(); return false; }
    if (sg == nseg_st) n_stat = (int)tiles.size();
    tiles.insert(tiles.end(), segs[sg].tiles.begin(), segs[sg].tiles.end());
  }
  return true;
}
// Vertex-sorted runs of a range of tiles: pointxyz (os) and ternary (ts) runs cut at VDO_SEG entries, the same runs cut at VDO_SEG2
// entries (os2 / ts2), and the tiles' vertex lists.  A Tile holds its ranges in these lists.
struct TileRuns {
  std::vector<Seg> os, ts, os2, ts2; std::vector<int> verts;
  // appends w, the runs of tiles t[0, n): their ranges, counted in w, are rebased to this one
  void append(const TileRuns& w, Tile* t, int n) {
    auto cat = [&](auto& dst, const auto& src, int Tile::*lo, int Tile::*hi) {
      const int base = (int)dst.size();
      for (int i = 0; i < n; ++i) { t[i].*lo += base; if (hi) t[i].*hi += base; }
      dst.insert(dst.end(), src.begin(), src.end());
    };
    cat(os, w.os, &Tile::os0, &Tile::os1); cat(ts, w.ts, &Tile::ts0, &Tile::ts1);
    cat(os2, w.os2, &Tile::qo0, &Tile::qo1); cat(ts2, w.ts2, &Tile::qt0, &Tile::qt1);
    cat(verts, w.verts, &Tile::vs0, nullptr);
  }
};
// the sorted entries perm[base, base + n), cut into runs of at most cap entries of one key
void cut_runs(const std::vector<int>& keys, const HostBuf<uint16_t>& perm, int base, int n, int cap, std::vector<Seg>& out) {
  for (int a = 0; a < n;) {
    const int v = keys[perm[base + a]];
    int b = a;
    while (b < n && b - a < cap && keys[perm[base + b]] == v) ++b;
    out.push_back(Seg{v, base + a, b - a, 0});
    a = b;
  }
}
}  // namespace
// Landmarks of this rank in tracklet order (begin: T + 1 landmark ranges), static landmarks (tracklets [0, Tstat)) first; the landmark
// renumbering is new_of_old_.  The pointxyz edges of bucket b (consecutive old landmark ids) are eidx[bucket[b], bucket[b + 1]), in the
// caller's order; n_obs: pointxyz edges per old landmark id.
struct BaGraph::Tracklets { std::vector<int> begin; HostBuf<int> old_of_new; int Tstat = 0, T = 0, P = 0; std::vector<int64_t> bucket; HostBuf<int> eidx, n_obs; };
struct BaGraph::EdgeClasses { ClassTable table; HostBuf<uint8_t> of_edge; };
struct BaGraph::LmStream { HostBuf<int> begin, cam; HostBuf<double> z; HostBuf<uint8_t> cls; int E = 0; };   // pointxyz edges in landmark order
// per landmark k: motion vertex (-1: none) and class of the ternary edge (k, k+1)
struct BaGraph::Ternary { HostBuf<int> h; HostBuf<uint8_t> cls; ClassTable table; int E = 0; };
struct BaGraph::TileLayout { bool tiled = false; std::vector<Tile> tiles; int n_stat = 0; TileRuns runs;
                             HostBuf<uint16_t> ob_perm, tr_perm; HostBuf<uint8_t> lm_lml, lm_cslot, tk_hslot; HostBuf<uint32_t> ob_ps; };
struct BaGraph::Chunked { std::vector<int> vm_pt; std::vector<double> vm_z; std::vector<uint8_t> vm_cls; std::vector<Chunk> obs_chunks;
                          std::vector<int> hm_p1; std::vector<uint8_t> hm_cls; std::vector<Chunk> ter_chunks; };
struct BaGraph::Se3Edges { std::vector<int> i, j; std::vector<double> Z, w, d; std::vector<int> nbr_begin, nbr_edge, nbr_other;
                           std::vector<uint8_t> nbr_tr; std::vector<int> path_of, pcr_edge; std::vector<uint8_t> pcr_tr; int max_len = 1; };
struct BaGraph::Solvers { bool dense = false; int band_W = 0, band_v0 = 0, band_n = 0; };   // band_W 0: no band
// Tracklets: chains of landmarks linked by ternary edges.
int BaGraph::order_tracklets(int NT, const Lap& lap, Tracklets& tk) {
  const int C = n_se3_, P = n_pt_, Eo = (int)ob_w_.size(), Et = (int)te_w_.size(), rank = be_->rank, world = be_->world;
  HostBuf<int> next = stage_fill<int>(P, 0xFF), prev = stage_fill<int>(P, 0xFF), ter_of = stage_fill<int>(P, 0xFF);
  for (int e = 0; e < Et; ++e) {
    int p1 = te_pph_[3 * e], p2 = te_pph_[3 * e + 1];
    if (p1 == p2 || next[p1] != -1 || prev[p2] != -1)
      return fail(VDO_ERR_UNSUPPORTED, "landmark-motion edges must form simple chains (one predecessor / successor per landmark)");
    next[p1] = p2; prev[p2] = p1; ter_of[p1] = e;
  }
  lap("  chain links");
  new_of_old_.assign(P, -1);
  tk.old_of_new = stage<int>(P);
  // Tracklet order.  Static landmarks (tracklets of one vertex) first, then the chains: the two groups run different
  // kernels.  Inside each group tracklets are ordered by the first se3 vertex that observes them (chains: by the motion
  // vertex of their first ternary edge, then by the first observing camera), so that the landmarks of one tile meet only
  // a few se3 vertices and the per-tile vertex-sorted segments stay long.  Counting sorts: O(P + C).
  // Multi-GPU: tracklets are dealt round-robin to the ranks (each group separately, in this order); a rank keeps only its
  // own landmarks and their edges, the se3 state is replicated.
  // Edge partition: the pointxyz edges are split, in the caller's order, into NB buckets of consecutive (old) landmark ids --
  // a stable parallel counting sort by bucket (chunk t of the edge list counts, then writes its edge indices behind the
  // chunks before it).  Everything per-landmark below (first camera, edge count, the scatter into landmark order) is then
  // done by the worker that owns the bucket, reading only its own edges: O(E) work in total and the same result for any
  // thread count.
  const int NB = NT, P0 = std::max(P, 1);
  auto bucket_of = [NB, P0](int p) { return (int)((int64_t)p * NB / P0); };
  std::vector<int64_t> tb((size_t)NT * NB + 1, 0);
  parallel_for(NT, [&](int t, int n) {
    const auto [a, b] = thread_range(Eo, t, n);
    int64_t* c = &tb[(size_t)t * NB];
    for (int e = a; e < b; ++e) c[bucket_of(ob_cp_[2 * e + 1])]++;
  });
  std::vector<int64_t> off((size_t)NB * NT + 1, 0);      // off[b * NT + t]: first slot of chunk t inside bucket b
  { int64_t run = 0; for (int b = 0; b < NB; ++b) for (int t = 0; t < NT; ++t) { off[(size_t)b * NT + t] = run; run += tb[(size_t)t * NB + b]; } off[(size_t)NB * NT] = run; }
  tk.eidx = stage<int>(Eo);
  parallel_for(NT, [&](int t, int n) {
    const auto [a, b] = thread_range(Eo, t, n);
    std::vector<int64_t> cur(NB);
    for (int k = 0; k < NB; ++k) cur[k] = off[(size_t)k * NT + t];
    for (int e = a; e < b; ++e) tk.eidx[cur[bucket_of(ob_cp_[2 * e + 1])]++] = e;
  });
  for (int b = 0; b <= NB; ++b) tk.bucket.push_back(off[(size_t)b * NT]);
  HostBuf<int> first_cam = stage<int>(P); tk.n_obs = stage_fill<int>(P, 0);
  parallel_for(NB, [&](int b, int) {
    const int lo = (int)(((int64_t)b * P + NB - 1) / NB), hi = (int)(((int64_t)(b + 1) * P + NB - 1) / NB);   // landmarks p with bucket_of(p) == b
    for (int p = lo; p < hi && p < P; ++p) first_cam[p] = C;
    for (int64_t q = tk.bucket[b]; q < tk.bucket[b + 1]; ++q) {
      const int e = tk.eidx[q], p = ob_cp_[2 * e + 1], c = new_se3_of_old_[ob_cp_[2 * e]];
      if (c < first_cam[p]) first_cam[p] = c;
      tk.n_obs[p]++;
    }
  });
  lap("  first_cam scan");
  std::vector<int> stat_ids, chain_heads;
  {   // heads of tracklets, in landmark order (parallel count, then fill)
    std::vector<size_t> ns(NT + 1, 0), nc(NT + 1, 0);
    parallel_for(NT, [&](int t, int n) {
      const auto [a, b] = thread_range(P, t, n);
      size_t s0 = 0, c0 = 0;
      for (int p = a; p < b; ++p) if (prev[p] == -1) { if (next[p] == -1) ++s0; else ++c0; }
      ns[t + 1] = s0; nc[t + 1] = c0;
    });
    for (int t = 0; t < NT; ++t) { ns[t + 1] += ns[t]; nc[t + 1] += nc[t]; }
    stat_ids.resize(ns[NT]); chain_heads.resize(nc[NT]);
    parallel_for(NT, [&](int t, int n) {
      const auto [a, b] = thread_range(P, t, n);
      size_t s0 = ns[t], c0 = nc[t];
      for (int p = a; p < b; ++p) if (prev[p] == -1) { if (next[p] == -1) stat_ids[s0++] = p; else chain_heads[c0++] = p; }
    });
  }
  lap("  collect heads");
  {   // static landmarks: by first observing camera, inside one camera by DESCENDING edge count -- the lanes of a warp that loops over
      // its landmarks' edges then run the same trip counts (geometric track lengths: a warp of mixed landmarks idles ~55 % of its lanes)
    int mx = 0;
    for (int p : stat_ids) mx = std::max(mx, tk.n_obs[p]);
    HostBuf<int> neg = stage<int>(P);
    parallel_for(NT, [&](int t, int n) {
      const auto [a, b] = thread_range((int)stat_ids.size(), t, n);
      for (int i = a; i < b; ++i) neg[stat_ids[i]] = mx - tk.n_obs[stat_ids[i]];
    });
    counting_sort(stat_ids, neg, mx + 1, NT);
  }
  counting_sort(stat_ids, first_cam, C + 1, NT);
  {
    HostBuf<int> first_h = stage_fill<int>(P, 0);
    for (int p : chain_heads) first_h[p] = new_se3_of_old_[te_pph_[3 * ter_of[p] + 2]];
    counting_sort(chain_heads, first_cam, C + 1, NT);
    counting_sort(chain_heads, first_h, C + 1, NT);
  }
  lap("  counting sorts");
  // chain lengths (parallel walks); every landmark must be a static point or lie on a chain that starts at a head
  const int n_heads = (int)chain_heads.size();
  std::vector<int> chain_len(n_heads);
  std::vector<int64_t> seen_part(NT, 0);
  parallel_for(NT, [&](int t, int n) {
    const auto [a, b] = thread_range(n_heads, t, n);
    int64_t sum = 0;
    for (int i = a; i < b; ++i) { int len = 0; for (int q = chain_heads[i]; q != -1; q = next[q]) ++len; chain_len[i] = len; sum += len; }
    seen_part[t] = sum;
  });
  int64_t n_seen = (int64_t)stat_ids.size();
  for (int64_t v : seen_part) n_seen += v;
  if (n_seen != P) return fail(VDO_ERR_UNSUPPORTED, "landmark-motion edges contain a cycle");
  // deal the tracklets to the ranks (round-robin in sorted order) and number the kept landmarks
  std::vector<int> stat_keep, head_keep, head_len;
  if (world == 1) { stat_keep.swap(stat_ids); head_keep.swap(chain_heads); head_len.swap(chain_len); }
  else {
    for (size_t i = rank; i < stat_ids.size(); i += world) stat_keep.push_back(stat_ids[i]);
    for (size_t i = rank; i < chain_heads.size(); i += world) { head_keep.push_back(chain_heads[i]); head_len.push_back(chain_len[i]); }
  }
  const int Tstat = (int)stat_keep.size(), Tch = (int)head_keep.size();
  tk.begin.resize((size_t)Tstat + Tch + 1);
  { int run = Tstat; for (int i = 0; i < Tch; ++i) { tk.begin[Tstat + i] = run; run += head_len[i]; } tk.begin[Tstat + Tch] = run; tk.P = run; }
  parallel_for(NT, [&](int t, int n) {
    const auto [a, b] = thread_range(Tstat, t, n);
    for (int i = a; i < b; ++i) { tk.begin[i] = i; new_of_old_[stat_keep[i]] = i; tk.old_of_new[i] = stat_keep[i]; }
    const auto [c, d2] = thread_range(Tch, t, n);
    for (int i = c; i < d2; ++i) { int k = tk.begin[Tstat + i]; for (int q = head_keep[i]; q != -1; q = next[q]) { new_of_old_[q] = k; tk.old_of_new[k++] = q; } }
  });
  tk.Tstat = Tstat; tk.T = Tstat + Tch;
  return VDO_OK;
}
// (information, Huber delta) class of every edge of one family; at most 256 classes
int BaGraph::edge_classes(const HostBuf<double>& w, const HostBuf<double>& d, int NT, const char* family, EdgeClasses& out) {
  const int n = (int)w.size();
  out.of_edge = stage<uint8_t>(n);
  // fast path: every edge carries the first edge's (information, delta) pair (checked in parallel)
  std::vector<char> uniform(NT, 1);
  if (n > 0) {
    const double w0 = w[0], d0 = d[0];
    parallel_for(NT, [&](int t, int nt) {
      const auto [a, b] = thread_range(n, t, nt);
      char u = 1;
      for (int e = a; e < b; ++e) if (w[e] != w0 || d[e] != d0) { u = 0; break; }
      uniform[t] = u;
    });
  }
  bool all_uniform = n > 0;
  for (char u : uniform) all_uniform = all_uniform && u;
  if (all_uniform) { const int c0 = out.table.get(w[0], d[0]); fill_bytes(out.of_edge.p, c0, (size_t)n); return VDO_OK; }
  double lw = 0, ld = 0; int lc = -1;
  for (int e = 0; e < n; ++e) {                  // sequential with a last-value cache: consecutive edges almost always share their class
    if (lc < 0 || w[e] != lw || d[e] != ld) {
      lc = out.table.get(w[e], d[e]); lw = w[e]; ld = d[e];
      if (lc > 255) return fail(VDO_ERR_UNSUPPORTED, std::string("more than 256 distinct (information, Huber delta) pairs on ") + family + " edges");
    }
    out.of_edge[e] = (uint8_t)lc;
  }
  return VDO_OK;
}
// Landmark-major pointxyz stream: edges per landmark in the new order (gathered from the per-old-landmark counts), prefix sum, then the
// scatter: the worker that owns a bucket walks its edges in the caller's order and appends each to its landmark's slot range, so the
// order of a landmark's edges is the caller's order whatever the thread count.
BaGraph::LmStream BaGraph::landmark_stream(const Tracklets& tk, const HostBuf<uint8_t>& ecls, int NT, const Lap& lap) {
  const int P = tk.P, NB = (int)tk.bucket.size() - 1;
  LmStream lm;
  lm.begin = stage<int>((size_t)P + 1); lm.begin[0] = 0;
  parallel_for(NT, [&](int t, int n) {
    const auto [a, b] = thread_range(P, t, n);
    for (int k = a; k < b; ++k) lm.begin[k + 1] = tk.n_obs[tk.old_of_new[k]];
  });
  lap("  count");
  for (int k = 0; k < P; ++k) lm.begin[k + 1] += lm.begin[k];
  const int Eo = lm.E = lm.begin[P];
  lm.cam = stage<int>(Eo); lm.z = stage<double>(3 * (size_t)Eo); lm.cls = stage<uint8_t>(Eo);
  HostBuf<int> written = tk.n_obs;        // reused: edges of the (old) landmark written so far
  fill_bytes(written.p, 0, sizeof(int) * (size_t)n_pt_);
  lap("  prefix + alloc");
  parallel_for(NB, [&](int b, int) {
    for (int64_t q = tk.bucket[b]; q < tk.bucket[b + 1]; ++q) {
      const int e = tk.eidx[q], p = ob_cp_[2 * e + 1], k = new_of_old_[p];
      if (k < 0) continue;                                       // landmark owned by another rank
      const int pos = lm.begin[k] + written[p]++;
      lm.cam[pos] = new_se3_of_old_[ob_cp_[2 * e]];
      lm.z[3 * (size_t)pos] = ob_z_[3 * (size_t)e]; lm.z[3 * (size_t)pos + 1] = ob_z_[3 * (size_t)e + 1]; lm.z[3 * (size_t)pos + 2] = ob_z_[3 * (size_t)e + 2];
      lm.cls[pos] = ecls[e];
    }
  });
  return lm;
}
// Ternary edges per landmark (as p1)
int BaGraph::ternary_edges(const Tracklets& tk, int NT, Ternary& ter) {
  const int P = tk.P, Et_all = (int)te_w_.size();
  ter.h = stage_fill<int>(P, 0xFF); ter.cls = stage_fill<uint8_t>(P, 0);
  EdgeClasses tc;
  if (int rc = edge_classes(te_w_, te_d_, NT, "landmark-motion", tc)) return rc;
  ter.table = std::move(tc.table);
  parallel_for(NT, [&](int t, int n) {                     // every landmark is p1 of at most one edge: the writes are disjoint
    const auto [a, b] = thread_range(Et_all, t, n);
    for (int e = a; e < b; ++e)
      if (const int k = new_of_old_[te_pph_[3 * e]]; k >= 0) { ter.h[k] = new_se3_of_old_[te_pph_[3 * e + 2]]; ter.cls[k] = tc.of_edge[e]; }
  });
  ter.E = tk.P - tk.T;                                     // a chain of L landmarks has L - 1 ternary edges, a static landmark none
  return VDO_OK;
}
// Vertex-major streams of the chunked layout, built by walking the landmark-major ones so that each vertex's edges stay landmark-sorted
BaGraph::Chunked BaGraph::chunked_streams(const LmStream& lm, const Ternary& ter, int C, int P) {
  Chunked ch;
  ch.vm_pt.resize(lm.E); ch.vm_z.resize(3 * (size_t)lm.E); ch.vm_cls.resize(lm.E);
  int k = 0;
  vertex_major(C, lm.E, [&](int pos) { return lm.cam[pos]; }, [&](int pos, int q) {
    while (lm.begin[k + 1] <= pos) ++k;
    ch.vm_pt[q] = k; ch.vm_cls[q] = lm.cls[pos];
    for (int i = 0; i < 3; ++i) ch.vm_z[3 * (size_t)q + i] = lm.z[3 * (size_t)pos + i];
  }, ch.obs_chunks);
  ch.hm_p1.resize(ter.E); ch.hm_cls.resize(ter.E);
  vertex_major(C, P, [&](int k) { return ter.h[k]; }, [&](int k, int q) { ch.hm_p1[q] = k; ch.hm_cls[q] = ter.cls[k]; }, ch.ter_chunks);
  return ch;
}
// Per tile: the tile-local landmark of every pointxyz edge, the vertex-sorted order of its pointxyz and ternary edges cut into runs of one
// vertex, and its vertex list, with each edge's 8-bit slot in that list.
int BaGraph::tile_runs(const LmStream& lm, const Ternary& ter, int P, int NT, TileLayout& tl) {
  const int Eo = lm.E;
  tl.ob_perm = stage<uint16_t>(Eo); tl.tr_perm = stage_fill<uint16_t>(P, 0); tl.lm_lml = stage<uint8_t>(Eo); tl.ob_ps = stage<uint32_t>(Eo);
  tl.lm_cslot = stage<uint8_t>(Eo); tl.tk_hslot = stage_fill<uint8_t>(P, 0xFF);
  // tiles are independent: each worker handles a contiguous range of tiles into its own runs, which are then concatenated in tile order
  const int ntl = (int)tl.tiles.size();
  const int NW = std::max(1, std::min(NT, ntl / 64 + 1));
  std::vector<TileRuns> w_runs(NW);
  std::vector<char> w_bad(NW, 0);
  parallel_for(NW, [&](int wt, int wn) {
    std::vector<int> keys(std::max(VDO_TILE_E, VDO_TILE_L)), idx(keys.size()), bucket;
    TileRuns& r = w_runs[wt];
    // stable sort of idx[0..n) by keys[idx] into perm[base, base + n) (counting sort over the key range when it is small), cut into runs
    // of at most VDO_SEG and VDO_SEG2 entries (Schur kernels: one thread per (run, component)); the distinct keys in sorted order are
    // appended to the tile's vertex list and slot[base + idx] is the position of idx's key there.  Returns the number of distinct keys.
    auto sort_and_cut = [&](int n, int base, HostBuf<uint16_t>& perm, std::vector<Seg>& segs, std::vector<Seg>& segs2, HostBuf<uint8_t>& slot) {
      if (n == 0) return 0;
      int lo = keys[idx[0]], hi = lo;
      for (int a = 1; a < n; ++a) { lo = std::min(lo, keys[idx[a]]); hi = std::max(hi, keys[idx[a]]); }
      const int range = hi - lo + 1;
      if (range <= 8 * n + 64) {
        bucket.assign(range + 1, 0);
        for (int a = 0; a < n; ++a) bucket[keys[idx[a]] - lo + 1]++;
        for (int a = 0; a < range; ++a) bucket[a + 1] += bucket[a];
        for (int a = 0; a < n; ++a) perm[base + bucket[keys[idx[a]] - lo]++] = (uint16_t)idx[a];
      } else {
        std::stable_sort(idx.begin(), idx.begin() + n, [&](int x, int y) { return keys[x] < keys[y]; });
        for (int a = 0; a < n; ++a) perm[base + a] = (uint16_t)idx[a];
      }
      cut_runs(keys, perm, base, n, VDO_SEG, segs);
      cut_runs(keys, perm, base, n, VDO_SEG2, segs2);
      int nv = 0;
      for (int q = 0; q < n; ++q) {
        const int i = perm[base + q];
        if (q == 0 || keys[i] != keys[perm[base + q - 1]]) { r.verts.push_back(keys[i]); ++nv; }
        slot[base + i] = (uint8_t)(nv - 1);
      }
      return nv;
    };
    const auto [ta, tb] = thread_range(ntl, wt, wn);
    for (int ti = ta; ti < tb; ++ti) {
      Tile& t = tl.tiles[ti];
      for (int k = t.k0; k < t.k1; ++k) for (int e = lm.begin[k]; e < lm.begin[k + 1]; ++e) tl.lm_lml[e] = (uint8_t)(k - t.k0);
      const int ne = t.e1 - t.e0;
      for (int i = 0; i < ne; ++i) { keys[i] = lm.cam[t.e0 + i]; idx[i] = i; }
      // the tile's vertex list: the cameras of its sorted pointxyz runs, then the motion vertices of its sorted ternary runs
      t.os0 = (int)r.os.size(); t.qo0 = (int)r.os2.size(); t.vs0 = (int)r.verts.size();
      const int ncam = sort_and_cut(ne, t.e0, tl.ob_perm, r.os, r.os2, tl.lm_cslot);
      t.os1 = (int)r.os.size(); t.qo1 = (int)r.os2.size();
      // sorted order: permutation and tile-local landmark in one word
      for (int q = 0; q < ne; ++q) { const int i = tl.ob_perm[t.e0 + q]; tl.ob_ps[t.e0 + q] = (uint32_t)i | ((uint32_t)tl.lm_lml[t.e0 + i] << 16); }
      int nt = 0;
      for (int k = t.k0; k < t.k1; ++k) if (ter.h[k] >= 0) { keys[k - t.k0] = ter.h[k]; idx[nt++] = k - t.k0; }
      t.ts0 = (int)r.ts.size(); t.qt0 = (int)r.ts2.size();
      const int nmot = sort_and_cut(nt, t.k0, tl.tr_perm, r.ts, r.ts2, tl.tk_hslot);
      t.ts1 = (int)r.ts.size(); t.qt1 = (int)r.ts2.size();
      if (ncam > 255 || nmot > 255) w_bad[wt] = 1;
      t.nv = ncam | (nmot << 16);
    }
  });
  for (int wt = 0; wt < NW; ++wt) {
    const auto [ta, tb] = thread_range(ntl, wt, NW);
    tl.runs.append(w_runs[wt], tl.tiles.data() + ta, tb - ta);
    if (w_bad[wt]) return fail(VDO_ERR_UNSUPPORTED, "a tile meets more than 255 motion vertices");
  }
  return VDO_OK;
}
// se3-se3 edges (priors first, j = -1), H_pp adjacency and the chain-preconditioner wiring
BaGraph::Se3Edges BaGraph::se3_edges(const std::vector<int>& path_begin) const {
  const int C = n_se3_, Ep = (int)pr_w_.size(), Es = (int)se_w_.size(), Ese = Ep + Es;
  auto S3 = [&](int old_id) { return new_se3_of_old_[old_id]; };
  Se3Edges se;
  se.i.resize(Ese); se.j.resize(Ese); se.Z.resize(12 * (size_t)Ese); se.w.resize(Ese); se.d.resize(Ese);
  for (int e = 0; e < Ep; ++e) { se.i[e] = S3(pr_v_[e]); se.j[e] = -1; se.w[e] = pr_w_[e]; se.d[e] = 0; std::memcpy(&se.Z[12 * (size_t)e], &pr_Z_[12 * (size_t)e], 96); }
  for (int e = 0; e < Es; ++e) {
    int q = Ep + e;
    se.i[q] = S3(se_ij_[2 * e]); se.j[q] = S3(se_ij_[2 * e + 1]); se.w[q] = se_w_[e]; se.d[q] = se_d_[e] > 0 ? se_d_[e] : 0;
    std::memcpy(&se.Z[12 * (size_t)q], &se_Z_[12 * (size_t)e], 96);
  }
  se.nbr_begin.assign(C + 1, 0);
  for (int e = Ep; e < Ese; ++e) { se.nbr_begin[se.i[e] + 1]++; se.nbr_begin[se.j[e] + 1]++; }
  for (int v = 0; v < C; ++v) se.nbr_begin[v + 1] += se.nbr_begin[v];
  std::vector<int> nfill(se.nbr_begin.begin(), se.nbr_begin.end() - 1);
  se.nbr_edge.resize(2 * (size_t)Es); se.nbr_other.resize(2 * (size_t)Es); se.nbr_tr.resize(2 * (size_t)Es);
  for (int e = Ep; e < Ese; ++e) {
    int a = nfill[se.i[e]]++; se.nbr_edge[a] = e; se.nbr_other[a] = se.j[e]; se.nbr_tr[a] = 0;
    int b = nfill[se.j[e]]++; se.nbr_edge[b] = e; se.nbr_other[b] = se.i[e]; se.nbr_tr[b] = 1;
  }
  // chain-preconditioner wiring: edge between internal vertices v-1 and v of the same path
  const int n_paths = (int)path_begin.size() - 1;
  se.path_of.resize(C); se.pcr_edge.assign(C, -1); se.pcr_tr.assign(C, 0);
  for (int pth = 0; pth < n_paths; ++pth) {
    for (int v = path_begin[pth]; v < path_begin[pth + 1]; ++v) se.path_of[v] = pth;
    se.max_len = std::max(se.max_len, path_begin[pth + 1] - path_begin[pth]);
  }
  for (int e = Ep; e < Ese; ++e) {
    int a = se.i[e], b = se.j[e];
    if (se.path_of[a] != se.path_of[b]) continue;       // (only inside non-path components, which were split into singletons)
    if (b == a + 1) { se.pcr_edge[b] = e; se.pcr_tr[b] = 1; }        // M(b, a) = H_ab^T
    else if (a == b + 1) { se.pcr_edge[a] = e; se.pcr_tr[a] = 0; }   // M(a, b) = H_ab
  }
  return se;
}
// estimates in path order (se3) and in this rank's landmark order (pt)
void BaGraph::states(const Tracklets& tk, int NT, HostBuf<double>& se3, HostBuf<double>& pt) {
  const int C = n_se3_, P = tk.P;
  se3 = stage<double>(12 * (size_t)C);
  for (int o = 0; o < C; ++o) std::memcpy(&se3[12 * (size_t)new_se3_of_old_[o]], &h_se3_[12 * (size_t)o], 96);
  pt = stage<double>(3 * (size_t)P);
  parallel_for(NT, [&](int t, int n) {
    const auto [a, b] = thread_range(P, t, n);
    for (int k = a; k < b; ++k) for (int i = 0; i < 3; ++i) pt[3 * (size_t)k + i] = h_pt_[3 * (size_t)tk.old_of_new[k] + i];
  });
}
// The dense path takes small static-only graphs on one rank.  The explicit static block of the reduced matrix (banded in the se3
// numbering) is possible when every static landmark lists its observing vertices in strictly increasing order within a window of
// band_max_width() consecutive vertex numbers (tracks over consecutive frames); otherwise the matrix-free static tile kernel stays in the PCG.
BaGraph::Solvers BaGraph::choose_solvers(bool allow_dense, bool allow_band, bool tiled, const Tracklets& tk, const LmStream& lm, int NT) const {
  const int C = n_se3_, Tstat = tk.Tstat, Wmax = be_->band_max_width();
  Solvers s;
  s.dense = allow_dense && tiled && be_->world == 1 && Tstat == tk.T && 6 * C <= be_->dense_capacity();
  if (!tiled || Tstat == 0 || Wmax <= 0) return s;
  std::vector<int> w_W(NT, 0), w_v0(NT, C), w_v1(NT, -1), w_bad(NT, 0);
  parallel_for(NT, [&](int t, int n) {
    const auto [a, b] = thread_range(Tstat, t, n);
    int W = 0, v0 = C, v1 = -1, bad = 0;
    for (int k = a; k < b && !bad; ++k) {
      const int e0 = lm.begin[k], e1 = lm.begin[k + 1];
      if (e1 <= e0) continue;
      for (int e = e0 + 1; e < e1; ++e) if (lm.cam[e] <= lm.cam[e - 1]) { bad = 1; break; }
      W = std::max(W, lm.cam[e1 - 1] - lm.cam[e0] + 1); v0 = std::min(v0, lm.cam[e0]); v1 = std::max(v1, lm.cam[e1 - 1]);
    }
    w_W[t] = W; w_v0[t] = v0; w_v1[t] = v1; w_bad[t] = bad;
  });
  int W = 0, v0 = C, v1 = -1, bad = 0;
  for (int t = 0; t < NT; ++t) { W = std::max(W, w_W[t]); v0 = std::min(v0, w_v0[t]); v1 = std::max(v1, w_v1[t]); bad |= w_bad[t]; }
  if (allow_band && !bad && v1 >= v0 && W <= Wmax && (size_t)(v1 - v0 + 1) * W * 80 <= ((size_t)512 << 20)) {
    s.band_W = W; s.band_v0 = v0; s.band_n = v1 - v0 + 1;
  }
  return s;
}
void BaGraph::upload_layout(const std::vector<int>& path_begin, const Tracklets& tk, const LmStream& lm, const EdgeClasses& oc, const Ternary& ter,
                            const TileLayout& tl, const Chunked& ch, const Se3Edges& se, const HostBuf<double>& se3, const HostBuf<double>& pt,
                            const Solvers& sv) {
  const int C = n_se3_, P = tk.P, Eo = lm.E, Ese = (int)se.i.size(), n_paths = (int)path_begin.size() - 1, rank = be_->rank, world = be_->world;
  BaDev& d = d_;
  d.C = C; d.P = P; d.T = tk.T; d.Tstat = tk.Tstat; d.own = (rank == 0) ? 1 : 0;
  P_all_ = n_pt_; d.Eobs = Eo; d.Eter = ter.E; d.Ese = Ese;
  d.n_obs_chunks = (int)ch.obs_chunks.size(); d.n_ter_chunks = (int)ch.ter_chunks.size(); d.n_nbr = (int)se.nbr_edge.size();
  d.se3 = upload(se3); d.pt = upload(pt);
  d.se3_init = dalloc<double>(12 * (size_t)C); d.pt_init = dalloc<double>(3 * (size_t)P);
  be_->d2d(d.se3_init, d.se3, 96 * (size_t)C); be_->d2d(d.pt_init, d.pt, 24 * (size_t)P);
  d.se3_bk = dalloc<double>(12 * (size_t)C); d.pt_bk = dalloc<double>(3 * (size_t)P);
  d.tk_begin = upload(tk.begin);
  d.lm_obs_begin = upload(lm.begin); d.lm_cam = upload(lm.cam); d.lm_z = upload(lm.z); d.lm_cls = upload(lm.cls); d.lm_omega = dalloc<double>(Eo);
  d.tk_h = upload(ter.h); d.tk_cls = upload(ter.cls); d.tk_omega = dalloc<double>(P);
  d.tiled = tl.tiled ? 1 : 0;
  if (!tl.tiled) {
    d.vm_pt = upload(ch.vm_pt); d.vm_z = upload(ch.vm_z); d.vm_cls = upload(ch.vm_cls); d.vm_omega = dalloc<double>(Eo); d.obs_chunks = upload(ch.obs_chunks);
    d.hm_p1 = upload(ch.hm_p1); d.hm_cls = upload(ch.hm_cls); d.hm_omega = dalloc<double>(ter.E); d.ter_chunks = upload(ch.ter_chunks);
  } else {
    const std::vector<Tile>& tiles = tl.tiles;
    d.n_tiles = (int)tiles.size(); d.n_tiles_stat = tl.n_stat; d.n_osegs = (int)tl.runs.os.size(); d.n_tsegs = (int)tl.runs.ts.size();
    d.capE_st = d.capE_ch = 16; d.capV_st = d.capV_ch = d.capH_ch = 1;
    for (int ti = 0; ti < d.n_tiles; ++ti) {
      const bool st = ti < tl.n_stat;
      int& cap = st ? d.capE_st : d.capE_ch;
      cap = std::max(cap, (tiles[ti].e1 - tiles[ti].e0 + 15) & ~15);
      int& cv = st ? d.capV_st : d.capV_ch;
      cv = std::max(cv, tiles[ti].nv & 0xFFFF);
      if (!st) d.capH_ch = std::max(d.capH_ch, tiles[ti].nv >> 16);
    }
    d.tiles = upload(tiles); d.osegs = upload(tl.runs.os); d.tsegs = upload(tl.runs.ts); d.osegs2 = upload(tl.runs.os2); d.tsegs2 = upload(tl.runs.ts2);
    d.ob_perm = upload(tl.ob_perm); d.tr_perm = upload(tl.tr_perm); d.lm_lml = upload(tl.lm_lml); d.ob_ps = upload(tl.ob_ps);
    d.tile_verts = upload(tl.runs.verts); d.lm_cslot = upload(tl.lm_cslot); d.tk_hslot = upload(tl.tk_hslot);
    d.pt_Q = dalloc<double>(9 * (size_t)std::max(P - tk.Tstat, 1));
    d.accO = dalloc<double>(16 * (size_t)C); d.accT = dalloc<double>(16 * (size_t)C); d.acc6 = dalloc<double>(12 * (size_t)C);
    d.vh = dalloc<double>(6 * (size_t)C);
  }
  d.se_i = upload(se.i); d.se_j = upload(se.j); d.se_Z = upload(se.Z); d.se_w = upload(se.w); d.se_delta = upload(se.d); d.se_Hoff = dalloc<double>(36 * (size_t)Ese);
  d.nbr_begin = upload(se.nbr_begin); d.nbr_edge = upload(se.nbr_edge); d.nbr_other = upload(se.nbr_other); d.nbr_tr = upload(se.nbr_tr);
  d.Hpp = dalloc<double>(42 * (size_t)C); d.bp = d.Hpp + 36 * (size_t)C; d.hll = dalloc<double>(P); d.bl = dalloc<double>(3 * (size_t)P);
  d.pt_s = dalloc<double>(P); d.Minv = dalloc<double>(36 * (size_t)C);
  d.pt_g = dalloc<double>(P); d.tk_gamma = dalloc<double>(P);
  d.n_paths = n_paths;
  d.path_begin = upload(path_begin); d.path_of = upload(se.path_of); d.pcr_edge = upload(se.pcr_edge); d.pcr_tr = upload(se.pcr_tr);
  size_t nDL = 0, nAG = 0, nb = 0;
  be_->precond_blocks(C, se.max_len, nDL, nAG, nb);
  d.pcr_D = dalloc<double>(36 * nDL); d.pcr_L = dalloc<double>(36 * nDL); d.pcr_Dinv = dalloc<double>(36 * (size_t)C);
  d.pcr_A = dalloc<double>(36 * nAG); d.pcr_G = dalloc<double>(36 * nAG);
  d.pcr_b = dalloc<double>(6 * nb);
  d.xp = dalloc<double>(6 * (size_t)C); d.r = dalloc<double>(6 * (size_t)C); d.z = dalloc<double>(6 * (size_t)C);
  d.p = dalloc<double>(6 * (size_t)C); d.Ap = dalloc<double>(6 * (size_t)C); d.rhs = dalloc<double>(6 * (size_t)C);
  d.p2 = dalloc<double>(6 * (size_t)C); d.ticket = dalloc<unsigned int>(4);
  if (sv.dense) d.Sdense = dalloc<double>((size_t)36 * C * C + 6 * (size_t)C + 8);
  if (sv.band_W) {
    d.band_W = sv.band_W; d.band_v0 = sv.band_v0; d.band_n = sv.band_n;
    d.band = dalloc<double>((size_t)d.band_n * d.band_W * 10);
  }
  d.zl = tl.tiled ? nullptr : dalloc<double>(3 * (size_t)P); d.xl = dalloc<double>(3 * (size_t)P); d.vw = dalloc<double>(6 * (size_t)C);
  auto upload256 = [&](std::vector<double> v) { v.resize(256, 0.0); return upload(v); };
  d.obs_cls_w = upload256(oc.table.w); d.obs_cls_d = upload256(oc.table.d); d.ter_cls_w = upload256(ter.table.w); d.ter_cls_d = upload256(ter.table.d);
  d.scal = dalloc<double>(SC_N);
  d.n_part_pap = tl.tiled ? std::max(1, (C + 127) / 128) : 148;    // tiled: one partial of p.Ap per CTA of the finalize kernel (128 vertices each)
  d.n_part_rz = std::max(1, n_paths) * 8;
  d.part_pap = dalloc<double>(d.n_part_pap); d.part_rz = dalloc<double>(d.n_part_rz);
  const bool sharded = be_->shard_paths(d);          // collective; on success d.z / d.part_rz point into the exchange buffer
  std::vector<int> own, shorts;
  for (int pth = 0; pth < n_paths; ++pth) {
    if (sharded && pth % world != rank) continue;
    if (path_begin[pth + 1] - path_begin[pth] > VDO_PCR_SHORT) own.push_back(pth); else shorts.push_back(pth);
  }
  d.n_own_long = (int)own.size();
  own.insert(own.end(), shorts.begin(), shorts.end());
  d.n_own_paths = (int)own.size();
  d.own_paths = upload(own);
  be_->sync();
}
int BaGraph::finalize() {
  if (finalized_) return fail(VDO_ERR_STATE, "finalize called twice");
  const Switches sw = read_switches();
  const bool prof = std::getenv("VDO_PROFILE") != nullptr;
  auto tp0 = std::chrono::steady_clock::now();
  const Lap lap = [&](const char* what) {
    if (!prof) return;
    auto t = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[vdo_b200] finalize: %-28s %.1f ms\n", what, std::chrono::duration<double, std::milli>(t - tp0).count());
    tp0 = t;
  };
  const int C = n_se3_, NT = host_threads();
  int rc;
  const std::vector<int> path_begin = se3_path_order(C, se_ij_, new_se3_of_old_);
  lap("se3 paths");
  Tracklets tk; if ((rc = order_tracklets(NT, lap, tk))) return rc;
  lap("tracklet order");
  EdgeClasses oc; if ((rc = edge_classes(ob_w_, ob_d_, NT, "pointxyz", oc))) return rc;
  lap("  edge classes");
  const LmStream lm = landmark_stream(tk, oc.of_edge, NT, lap);
  lap("landmark-major stream");
  TileLayout tl;
  tl.tiled = !sw.chunked && pack_tiles(tk.begin, tk.Tstat, lm.begin, lm.cam, C, NT, tl.tiles, tl.n_stat);
  Ternary ter; if ((rc = ternary_edges(tk, NT, ter))) return rc;
  const Chunked ch = tl.tiled ? Chunked() : chunked_streams(lm, ter, C, tk.P);
  lap("ternary / chunked streams");
  if (tl.tiled && (rc = tile_runs(lm, ter, tk.P, NT, tl))) return rc;
  lap("tile segments");
  const Se3Edges se = se3_edges(path_begin);
  HostBuf<double> se3, pt; states(tk, NT, se3, pt);
  lap("se3 edges, states");
  upload_layout(path_begin, tk, lm, oc, ter, tl, ch, se, se3, pt, choose_solvers(sw.dense, sw.band, tl.tiled, tk, lm, NT));
  lap("alloc + upload");
  // host staging is no longer needed (keep the landmark map for read-back)
  ob_z_ = HostBuf<double>(); ob_w_ = HostBuf<double>(); ob_d_ = HostBuf<double>(); ob_cp_ = HostBuf<int>();
  te_pph_ = HostBuf<int>(); te_w_ = HostBuf<double>(); te_d_ = HostBuf<double>();
  std::vector<double>().swap(se_Z_); std::vector<double>().swap(pr_Z_);
  h_se3_ = HostBuf<double>(); h_pt_ = HostBuf<double>();
  n_prior_ = (int)pr_w_.size();
  drop_stage();                 // every upload above has completed (sync): the staging arena can be rewound
  finalized_ = true;
  return VDO_OK;
}

int BaGraph::get_vertices(double* se3, double* pt) {
  if (!finalized_) return fail(VDO_ERR_STATE, "get_vertices before finalize");
  if (se3) {
    std::vector<double> tmp(12 * (size_t)d_.C);
    be_->d2h(tmp.data(), d_.se3, 96 * (size_t)d_.C);
    for (int o = 0; o < d_.C; ++o) std::memcpy(se3 + 12 * (size_t)o, &tmp[12 * (size_t)new_se3_of_old_[o]], 96);
  }
  if (pt) {
    HostBuf<double> tmp = stage<double>(3 * (size_t)d_.P);
    be_->d2h(tmp.data(), d_.pt, 24 * (size_t)d_.P);
    const int Pa = P_all_;
    parallel_for(std::min(host_threads(), 8), [&](int t, int n) {     // landmarks owned by other ranks are left untouched in the caller's buffer
      const auto [a, b] = thread_range(Pa, t, n);
      for (int o = a; o < b; ++o) {
        const int k = new_of_old_[o];
        if (k < 0) continue;
        pt[3 * (size_t)o] = tmp[3 * (size_t)k]; pt[3 * (size_t)o + 1] = tmp[3 * (size_t)k + 1]; pt[3 * (size_t)o + 2] = tmp[3 * (size_t)k + 2];
      }
    });
    drop_stage();
  }
  return VDO_OK;
}
int BaGraph::reset_vertices() {
  if (!finalized_) return fail(VDO_ERR_STATE, "reset_vertices before finalize");
  be_->d2d(d_.se3, d_.se3_init, 96 * (size_t)d_.C);
  be_->d2d(d_.pt, d_.pt_init, 24 * (size_t)d_.P);
  oplus_calls_ = 0;
  return VDO_OK;
}
int BaGraph::info(int64_t out[8]) const {
  out[0] = d_.C; out[1] = d_.P; out[2] = d_.Eobs; out[3] = d_.Eter; out[4] = d_.Ese; out[5] = n_prior_; out[6] = d_.T; out[7] = (int64_t)bytes_;
  return VDO_OK;
}

int BaGraph::solver_info(int64_t out[8]) const {
  out[0] = d_.tiled; out[1] = d_.n_tiles; out[2] = d_.n_tiles_stat; out[3] = d_.band ? d_.band_W : 0; out[4] = d_.band ? d_.band_n : 0;
  out[5] = d_.Sdense ? 1 : 0; out[6] = d_.xg_paths; out[7] = d_.n_paths;
  return VDO_OK;
}

// ---- buildSystem (g2o/core/block_solver.hpp:501-560) ----
void BaGraph::zero_system() {
  be_->zero(d_.Hpp, 336 * (size_t)d_.C);          // H_pp diagonal blocks and b_p are one buffer (one all-reduce)
  // SC_LAMBDA / SC_TOL2 stay: they hold the PCG parameters the backend last wrote, and it writes them again only when they change
  // (a solve at the lambda of the previous solve would otherwise multiply by H_pp + 0 I)
  be_->zero(d_.scal, sizeof(double) * SC_LAMBDA);
}

struct BaGraph::Round {
  std::vector<int> flag, rt;
  std::vector<double> lam, tol2;
  explicit Round(int n) : flag(n, 0), rt(n, 0), lam(n, 0.0), tol2(n, 0.0) {}
  void set(BaBackend* be) const { be->batch_set(flag.data(), lam.data(), rt.data(), tol2.data()); }
};

void BaGraph::lin_round(BaGraph* const* gs, int n, Round& r) {
  BaBackend* be = gs[0]->be_;
  for (int k = 0; k < n; ++k) if (r.flag[k] & BaBackend::BATCH_LIN) gs[k]->zero_system();
  r.set(be);
  be->lin_tracklets_batch(BaBackend::BATCH_LIN, true);
  be->lin_vertex_batch(BaBackend::BATCH_LIN);
  be->lin_se3_edges_batch(BaBackend::BATCH_LIN, true);
  for (int k = 0; k < n; ++k) {
    if (!(r.flag[k] & BaBackend::BATCH_LIN)) continue;
    be->allreduce_sum(gs[k]->d_.Hpp, 42 * (size_t)gs[k]->d_.C);
    be->allreduce_sum(gs[k]->d_.scal + SC_CHI2, 1);
  }
  be->max_diagonal_batch(BaBackend::BATCH_MAXDIAG);
  for (int k = 0; k < n; ++k) if (r.flag[k] & BaBackend::BATCH_MAXDIAG) be->allreduce_max(gs[k]->d_.scal + SC_MAXDIAG, 1);
}

// computeActiveErrors + activeRobustChi2 into scal[SC_CHI2]; len 2 also sums scal[SC_SCALE] across ranks (adjacent)
void BaGraph::chi2_step(BaGraph* const* gs, int n, const Round& r, int len) {
  BaBackend* be = gs[0]->be_;
  for (int k = 0; k < n; ++k) if (r.flag[k] & BaBackend::BATCH_TRIAL) be->zero(gs[k]->d_.scal + SC_CHI2, sizeof(double));
  be->lin_tracklets_batch(BaBackend::BATCH_TRIAL, false);
  be->lin_se3_edges_batch(BaBackend::BATCH_TRIAL, false);
  for (int k = 0; k < n; ++k) if (r.flag[k] & BaBackend::BATCH_TRIAL) be->allreduce_sum(gs[k]->d_.scal + SC_CHI2, len);
}

// One LM trial of every graph whose flags hold BATCH_TRIAL, solved by the dense path (BATCH_DENSE) or landmark elimination + PCG on the
// reduced se3 system (BATCH_PCG), in stages up to `last`: push; set-up (H_ll + lambda I pivots, the dense solve or the preconditioner
// M(lambda) and band of S(lambda), rhs, PCG init); the PCG in chunks of 8 iterations with one read-back per chunk of the scalars of every
// graph still iterating, each graph leaving the chunks where its own solve stops; back-substitution; update and chi2 of the new estimate.
// pcg_iters[k] / ok[k]: PCG iterations of graph k and whether its solve succeeded.  prof_ms: VDO_PROFILE phase timers, or NULL.
void BaGraph::trial_round(BaGraph* const* gs, int n, Round& r, int pcg_max_iterations, Stage last, float* prof_ms, int* pcg_iters, int* ok) {
  using B = BaBackend;
  BaBackend* be = gs[0]->be_;
  const bool prof = prof_ms != nullptr;
  float unused[5];
  float* ms = prof ? prof_ms : unused;
  for (int k = 0; k < n; ++k) if (r.flag[k] & B::BATCH_TRIAL) { gs[k]->push(); pcg_iters[k] = 0; ok[k] = 1; }
  r.set(be);
  {
    Phase ph(be, &ms[0], prof);
    be->factor_landmarks_batch(B::BATCH_TRIAL);
    be->dense_solve_batch(B::BATCH_DENSE);          // status in scal[SC_DENSE], read back with the trial's scalars
    be->precondition_batch(B::BATCH_PCG);
  }
  {
    Phase ph(be, &ms[1], prof);
    be->schur_rhs_batch(B::BATCH_PCG);
    for (int k = 0; k < n; ++k) if (r.flag[k] & B::BATCH_PCG) be->allreduce_sum(gs[k]->d_.rhs, 6 * (size_t)gs[k]->d_.C);
    be->pcg_init_batch(B::BATCH_PCG);
  }
  if (last == SETUP) return;
  {
    Phase ph(be, &ms[2], prof);
    const int chunk = 8;
    std::vector<int> run;
    for (int k = 0; k < n; ++k) if (r.flag[k] & B::BATCH_PCG) run.push_back(k);
    std::vector<const double*> src;
    std::vector<double> sc;
    for (int it = 0; !run.empty() && it < pcg_max_iterations; it += chunk) {
      be->pcg_iterate_batch(B::BATCH_PCG, chunk);
      src.clear();
      for (int k : run) src.push_back(gs[k]->d_.scal);
      sc.resize(run.size() * SC_N);
      be->read_scalars(src.data(), (int)run.size(), SC_N, sc.data());
      size_t m = 0;
      for (size_t j = 0; j < run.size(); ++j) {
        const int k = run[j];
        const double* c = &sc[j * SC_N];
        if (c[SC_DONE] == 0.0 && it + chunk < pcg_max_iterations) { run[m++] = k; continue; }
        BaDev& d = gs[k]->d_;
        pcg_iters[k] = (int)c[SC_ITERS];
        if (c[SC_DONE] >= 2.0 || !std::isfinite(c[SC_RZ])) ok[k] = 0;   // breakdown (p.Ap <= 0 or NaN), or 3: a peer never answered
        if (d.xg_paths) be->allreduce_sum(d.xp, 6 * (size_t)d.C);      // path-sharded preconditioner: every rank updated x on its own paths only
        r.flag[k] &= ~B::BATCH_PCG;
      }
      const bool changed = m < run.size();
      run.resize(m);
      if (changed && !run.empty()) r.set(be);
    }
  }
  {
    Phase ph(be, &ms[3], prof);
    be->back_substitute_batch(B::BATCH_TRIAL);      // xl = Hll^-1 (bl - Hlp xp)
  }
  if (last == BACKSUB) return;
  Phase ph(be, &ms[4], prof);
  for (int k = 0; k < n; ++k) if (r.flag[k] & B::BATCH_TRIAL) be->zero(gs[k]->d_.scal + SC_SCALE, sizeof(double));
  be->apply_update_batch(B::BATCH_TRIAL);
  chi2_step(gs, n, r, 2);
}

bool BaGraph::lone(Stage last, double lambda, int solver, double tol2, int pcg_max_iterations, int* pcg_iters) {
  BaGraph* self = this;
  BaDev* d = &d_;
  Round r(1);
  int it = 0, ok = 1;
  be_->batch_begin(&d, 1);
  r.flag[0] = BaBackend::BATCH_LIN;
  lin_round(&self, 1, r);
  if (last != LINEARIZE) {
    r.flag[0] = BaBackend::BATCH_TRIAL | solver; r.lam[0] = lambda; r.tol2[0] = tol2;
    trial_round(&self, 1, r, pcg_max_iterations, last, nullptr, &it, &ok);
  }
  be_->batch_end();
  if (pcg_iters) *pcg_iters = it;
  return ok != 0;
}

// LM state of one graph inside optimize_batch (g2o/core/optimization_algorithm_levenberg.cpp:61-164 per graph)
struct BaGraph::LmState {
  BaGraph* g = nullptr; double* hist = nullptr;
  double lambda = -1, ni = 2; int nbad = 0, trials = 0, pcg_total = 0, iters_done = 0, it = 0;
  bool stop_flag = false, ok = true, done = false;
  double chi2_check = 0, last_chi_action = 0, chi_cur = 0, chi_init = 0, gain_prev = 1.0;
  bool in_iter = false, trial_ok = true;     // inside the trials of LM iteration `it`; the last trial's solve succeeded
  double ini = 0, current = 0; int qmax = 0; double rho = 0;
};

int BaGraph::optimize(const vdo_lm_options& o_in, vdo_lm_stats* stats, double* hist) {
  BaGraph* self = this;
  return optimize_batch(&self, 1, o_in, stats, &hist);
}

void BaGraph::push() {
  be_->d2d(d_.se3_bk, d_.se3, 96 * (size_t)d_.C);
  be_->d2d(d_.pt_bk, d_.pt, 24 * (size_t)d_.P);
}
void BaGraph::pop() {
  be_->d2d(d_.se3, d_.se3_bk, 96 * (size_t)d_.C);
  be_->d2d(d_.pt, d_.pt_bk, 24 * (size_t)d_.P);
}
bool BaGraph::next_oplus_reorthogonalizes() {
  ++oplus_calls_;
  if (oplus_calls_ <= 1000) return false;
  oplus_calls_ = 0;                                 // vertex_se3.h:110-113
  return true;
}

// Rounds: the graphs that start an LM iteration are linearised (and, at iteration 0, give their max diagonal: one read-back for all);
// then every graph inside an iteration takes its next trial, one read-back brings every graph's scalars, and each graph takes its
// accept / reject and stop decisions exactly as a lone optimize() does.  A graph's device work and decisions do not depend on the others.
int BaGraph::optimize_batch(BaGraph* const* gs, int n, const vdo_lm_options& o_in, vdo_lm_stats* stats, double* const* hists) {
  for (int k = 0; k < n; ++k) if (!gs[k]->finalized_) return gs[k]->fail(VDO_ERR_STATE, "optimize before finalize");
  vdo_lm_options opt = o_in;
  if (opt.max_trials <= 0) opt.max_trials = 10;
  if (opt.pcg_rel_tol <= 0) opt.pcg_rel_tol = 1e-6;
  if (opt.pcg_max_iterations <= 0) opt.pcg_max_iterations = 2000;
  BaBackend* be = gs[0]->be_;
  const int launches0 = be->launches();
  const bool prof = std::getenv("VDO_PROFILE") != nullptr;
  float prof_ms[5] = {0, 0, 0, 0, 0};
  std::vector<LmState> S(n);
  std::vector<const double*> src(n);
  std::vector<double> sc((size_t)n * SC_N);
  std::vector<int> act, pcg_iters(n, 0), trial_ok(n, 1);
  act.reserve(n);
  std::vector<BaDev*> ds(n);
  Round r(n);
  be->timer_start(0);
  for (int k = 0; k < n; ++k) {
    S[k].g = gs[k]; S[k].hist = hists ? hists[k] : nullptr;
    ds[k] = &gs[k]->d_;
    r.flag[k] = BaBackend::BATCH_TRIAL;
    src[k] = gs[k]->d_.scal + SC_CHI2;
  }
  be->batch_begin(ds.data(), n);
  r.set(be);
  chi2_step(gs, n, r, 1);
  float ms_lin = 0, ms_solve = 0;
  be->read_scalars(src.data(), n, 1, sc.data());
  for (int k = 0; k < n; ++k) {
    S[k].chi_cur = S[k].chi_init = sc[k];
    if (S[k].hist) S[k].hist[0] = sc[k];
  }
  // Forcing schedule of the inexact solves: while the previous LM iteration still gained more than pcg_switch_gain (relative chi2
  // decrease), the reduced system is solved to pcg_loose_tol only; near convergence to pcg_rel_tol.  Disabled unless both are set.
  const double loose_tol = opt.pcg_loose_tol, switch_gain = opt.pcg_switch_gain;
  bool solve_timer = false;
  for (;;) {
    // graphs that start an LM iteration: linearise, and at iteration 0 read the largest diagonal entry for the initial lambda
    act.clear();
    for (int k = 0; k < n; ++k) {
      LmState& s = S[k];
      if (s.done || s.in_iter) continue;
      if (s.it < opt.max_iterations && ((!s.stop_flag && s.ok) || opt.force_all_iterations)) act.push_back(k); else s.done = true;
    }
    if (!act.empty()) {
      be->timer_start(1);
      int n0 = 0;
      std::fill(r.flag.begin(), r.flag.end(), 0);
      for (int k : act) {
        LmState& s = S[k]; BaGraph* g = s.g;
        g->cur_pcg_tol_ = (loose_tol > opt.pcg_rel_tol && switch_gain > 0 && s.gain_prev > switch_gain) ? loose_tol : opt.pcg_rel_tol;
        s.ini = s.current = s.chi_cur;
        r.flag[k] = BaBackend::BATCH_LIN | (s.it == 0 ? BaBackend::BATCH_MAXDIAG : 0);
        if (s.it == 0) src[n0++] = g->d_.scal + SC_MAXDIAG;
        s.in_iter = true; s.qmax = 0; s.rho = 0;
      }
      lin_round(gs, n, r);
      if (n0) {
        be->read_scalars(src.data(), n0, 1, sc.data());
        int i = 0;
        for (int k : act) if (S[k].it == 0) { S[k].lambda = 1e-5 * sc[i++]; S[k].ni = 2; S[k].nbad = 0; }
      }
      ms_lin += be->timer_stop_ms(1);
    }
    act.clear();
    for (int k = 0; k < n; ++k) if (S[k].in_iter) act.push_back(k);
    if (act.empty()) break;
    // one trial of every graph inside an LM iteration
    if (!solve_timer) { be->timer_start(2); solve_timer = true; }
    std::fill(r.flag.begin(), r.flag.end(), 0);
    for (size_t i = 0; i < act.size(); ++i) {
      const int k = act[i];
      BaGraph* g = S[k].g;
      r.flag[k] = BaBackend::BATCH_TRIAL | (g->d_.Sdense ? BaBackend::BATCH_DENSE : BaBackend::BATCH_PCG);
      r.lam[k] = S[k].lambda; r.rt[k] = g->next_oplus_reorthogonalizes() ? 1 : 0;
      const double tol_now = g->cur_pcg_tol_ > 0 ? g->cur_pcg_tol_ : opt.pcg_rel_tol;
      r.tol2[k] = tol_now * tol_now;
      src[i] = g->d_.scal;
    }
    trial_round(gs, n, r, opt.pcg_max_iterations, UPDATE, prof ? prof_ms : nullptr, pcg_iters.data(), trial_ok.data());
    for (int k : act) { S[k].pcg_total += pcg_iters[k]; S[k].trial_ok = trial_ok[k] != 0; }
    be->read_scalars(src.data(), (int)act.size(), SC_N, sc.data());
    bool iteration_ended = false;
    for (size_t i = 0; i < act.size(); ++i) {
      LmState& s = S[act[i]]; BaGraph* g = s.g; BaDev& d = g->d_;
      const double* c = &sc[i * SC_N];
      double temp = c[SC_CHI2];
      if (!s.trial_ok || (d.Sdense && c[SC_DENSE] != 0.0)) temp = DBL_MAX;
      s.rho = s.current - temp;
      const double scale = c[SC_SCALE] + 1e-3;
      s.rho /= scale;
      if (s.rho > 0 && std::isfinite(temp)) {
        double alpha = 1. - std::pow(2 * s.rho - 1, 3);
        alpha = std::min(alpha, 2. / 3.);
        const double sf = std::max(1. / 3., alpha);
        s.lambda *= sf; s.ni = 2; s.current = temp;
      } else {
        s.lambda *= s.ni; s.ni *= 2;
        g->pop();
      }
      ++s.qmax; ++s.trials;
      if (s.rho < 0 && s.qmax < opt.max_trials && !s.stop_flag) continue;
      // the LM iteration of this graph is over
      s.in_iter = false; iteration_ended = true;
      g->last_lambda_ = s.lambda;
      bool result_ok = true;
      if (s.qmax == opt.max_trials || s.rho == 0) result_ok = false;
      else {
        if ((s.ini - s.current) * 1e3 < s.ini) s.nbad++; else s.nbad = 0;
        if (s.nbad >= 3) result_ok = false;
      }
      s.ok = result_ok;
      const double chi_now = s.current;     // errors at the (restored) estimate == last accepted chi2
      s.gain_prev = chi_now > 0 ? (s.ini - chi_now) / chi_now : 0.0;
      if (s.chi2_check < chi_now && s.it > 0) s.ok = false;
      s.chi2_check = chi_now;
      s.chi_cur = chi_now;
      if (s.hist) s.hist[s.it + 1] = chi_now;
      if (opt.verbose) std::fprintf(stderr, "[vdo_b200] iteration= %d\t chi2= %.9g\t lambda= %.6g\t levenbergIter= %d\t pcg= %d\n", s.it, chi_now, s.lambda, s.qmax, s.pcg_total);
      ++s.iters_done;
      if (opt.gain_threshold > 0) {
        if (s.it == 0) s.last_chi_action = chi_now;
        else {
          const double gain = (s.last_chi_action - chi_now) / chi_now;
          s.last_chi_action = chi_now;
          if (gain >= 0 && gain < opt.gain_threshold) s.stop_flag = true;
        }
      }
      ++s.it;
    }
    if (iteration_ended) { ms_solve += be->timer_stop_ms(2); solve_timer = false; }
  }
  be->batch_end();
  const float ms_total = be->timer_stop_ms(0);
  const int launches = be->launches() - launches0;
  if (prof) {
    int iters = 0, trials = 0, pcg = 0;
    for (const LmState& s : S) { iters += s.iters_done; trials += s.trials; pcg += s.pcg_total; }
    std::fprintf(stderr, "[vdo_b200] phases (ms, synchronising timers): factor+precond %.2f | rhs+init %.2f | pcg %.2f | backsubst %.2f | update+chi2 %.2f | linearize %.2f | total %.2f (iters %d trials %d pcg %d)\n", prof_ms[0], prof_ms[1], prof_ms[2], prof_ms[3], prof_ms[4], ms_lin, ms_total, iters, trials, pcg);
  }
  for (int k = 0; k < n; ++k) {
    const LmState& s = S[k];
    if (stats) {
      vdo_lm_stats& st = stats[k];
      st.iterations = s.iters_done; st.trials = s.trials; st.pcg_iterations = s.pcg_total;
      st.initial_chi2 = s.chi_init; st.final_chi2 = s.chi_cur; st.final_lambda = s.lambda;
      st.ms_linearize = ms_lin; st.ms_solve = ms_solve; st.ms_total = ms_total;
      st.kernel_launches = launches;
    }
  }
  return VDO_OK;
}

int BaGraph::time_kernel(const char* name, int reps, float* ms_avg) {
  if (!finalized_) return fail(VDO_ERR_STATE, "time_kernel before finalize");
  if (!name || reps <= 0 || !ms_avg) return fail(VDO_ERR_ARG, "time_kernel: bad arguments");
  BaDev& d = d_;
  const std::string n(name);
  const double lam = last_lambda_;
  auto run = [&]() -> bool {
    if (n == "lin_tracklets") be_->lin_tracklets(d, true);
    else if (n == "chi2_tracklets") be_->lin_tracklets(d, false);
    else if (n == "lin_vertex_obs") be_->lin_vertex_obs(d);
    else if (n == "lin_vertex_ter") be_->lin_vertex_ter(d);
    else if (n == "lin_se3_edges") be_->lin_se3_edges(d, true);
    else if (n == "linearize") lone(LINEARIZE, 0.0, 0, 0.0, 0, nullptr);
    else if (n == "factor_landmarks") be_->factor_landmarks(d, lam);
    else if (n == "precond") { be_->precond_begin(d, lam); be_->precond_vertex_obs(d); be_->precond_vertex_ter(d); be_->precond_factor(d, lam); }
    else if (n == "band_form") be_->band_form(d);
    else if (n == "precond_tiles") { be_->precond_begin(d, lam); be_->precond_vertex_obs(d); be_->precond_vertex_ter(d); }
    else if (n == "pcr_factor") be_->precond_factor(d, lam);
    else if (n == "schur_landmarks") be_->schur_landmarks(d, 1, d.p);
    else if (n == "schur_static") be_->schur_landmarks_part(d, 1, d.p, 0);
    else if (n == "schur_static_mf") { double* b = d.band; d.band = nullptr; be_->schur_landmarks_part(d, 1, d.p, 0); d.band = b; }   // the matrix-free tile kernel even when the band is on
    else if (n == "schur_chains") be_->schur_landmarks_part(d, 1, d.p, 1);
    else if (n == "lin_static") be_->lin_tracklets_part(d, true, 0);
    else if (n == "lin_chains") be_->lin_tracklets_part(d, true, 1);
    else if (n == "pcg_step_a") { be_->pcg_dot_pAp(d); be_->pcg_step(d, 0.0); }
    else if (n == "schur_vertex_obs") be_->schur_vertex_obs(d, -1.0, d.Ap);
    else if (n == "schur_vertex_ter") be_->schur_vertex_ter(d, -1.0, d.Ap);
    else if (n == "hpp_mul") be_->hpp_mul(d, lam, d.p, d.Ap);
    else if (n == "pcg_dot") be_->pcg_dot_pAp(d);
    else if (n == "pcg_step") be_->pcg_step(d, 0.0);
    else if (n == "pcg_iterate8") be_->pcg_iterate(d, lam, 0.0, 8);
    else return false;
    return true;
  };
  // a valid, never-converging PCG state: linearise + factor at the last lambda, rhs, init
  if (d.tiled) {   // a previous timing of a tile kernel alone leaves its vertex-side sums behind: start clean
    be_->zero(d.accO, 128 * (size_t)d.C); be_->zero(d.accT, 128 * (size_t)d.C); be_->zero(d.acc6, 48 * (size_t)d.C);
  }
  lone(SETUP, lam, BaBackend::BATCH_PCG, 0.0, 0, nullptr);
  if (!run()) return fail(VDO_ERR_ARG, "time_kernel: unknown kernel name");
  be_->sync();
  be_->timer_start(3);
  for (int i = 0; i < reps; ++i) run();
  *ms_avg = be_->timer_stop_ms(3) / reps;
  return VDO_OK;
}

int BaGraph::debug_linearize(double* Hpp, double* bp, double* Hll, double* bl, double* chi2) {
  if (!finalized_) return fail(VDO_ERR_STATE, "debug_linearize before finalize");
  lone(LINEARIZE, 0.0, 0, 0.0, 0, nullptr);
  {
    std::vector<double> tH(36 * (size_t)d_.C), tg(6 * (size_t)d_.C);
    be_->d2h(tH.data(), d_.Hpp, 288 * (size_t)d_.C);
    be_->d2h(tg.data(), d_.bp, 48 * (size_t)d_.C);
    for (int o = 0; o < d_.C; ++o) {
      int v = new_se3_of_old_[o];
      if (Hpp) std::memcpy(Hpp + 36 * (size_t)o, &tH[36 * (size_t)v], 288);
      if (bp) std::memcpy(bp + 6 * (size_t)o, &tg[6 * (size_t)v], 48);
    }
  }
  std::vector<double> th(d_.P), tb(3 * (size_t)d_.P);
  be_->d2h(th.data(), d_.hll, 8 * (size_t)d_.P);
  be_->d2h(tb.data(), d_.bl, 24 * (size_t)d_.P);
  for (int o = 0; o < P_all_; ++o) {
    int k = new_of_old_[o];
    if (k < 0) continue;
    if (Hll) Hll[o] = th[k];
    if (bl) for (int i = 0; i < 3; ++i) bl[3 * (size_t)o + i] = tb[3 * (size_t)k + i];
  }
  if (chi2) be_->d2h(chi2, d_.scal + SC_CHI2, sizeof(double));
  return VDO_OK;
}

// The operator hooks below run the same rounds and backend primitives as an LM trial, on the buffers a trial uses (p, Ap, rhs, r, z, xp,
// xl, the backup of the estimates), which every trial rewrites before it reads them: an optimize() after them starts from the same state
// as one without them.  debug_apply sets up the PCG path, also for a graph that the dense path solves.
int BaGraph::debug_apply(double lambda, const char* op, const double* in, double* out) {
  if (!finalized_) return fail(VDO_ERR_STATE, "debug_apply before finalize");
  if (be_->world > 1) return fail(VDO_ERR_STATE, "debug_apply: sharded graphs are not supported");
  const std::string o(op ? op : "");
  const int kind = o == "S" ? 0 : o == "Minv" ? 1 : o == "rhs" ? 2 : o == "backsub" ? 3 : -1;
  if (kind < 0 || !out || (kind != 2 && !in) || !(lambda >= 0)) return fail(VDO_ERR_ARG, "debug_apply: bad arguments");
  BaDev& d = d_;
  const int C = d.C;
  std::vector<double> v(6 * (size_t)C);
  auto upload6 = [&](double* dst) {           // caller's se3 numbering -> path order
    for (int c = 0; c < C; ++c) std::memcpy(&v[6 * (size_t)new_se3_of_old_[c]], in + 6 * (size_t)c, 48);
    if (C) be_->h2d(dst, v.data(), 48 * (size_t)C);
  };
  auto download6 = [&](const double* src) {
    if (C) be_->d2h(v.data(), src, 48 * (size_t)C);
    for (int c = 0; c < C; ++c) std::memcpy(out + 6 * (size_t)c, &v[6 * (size_t)new_se3_of_old_[c]], 48);
  };
  lone(SETUP, lambda, BaBackend::BATCH_PCG, 0.0, 0, nullptr);     // ... which leaves the rhs in d.rhs
  if (kind == 0) {
    upload6(d.p);
    be_->zero(d.scal + SC_DONE, sizeof(double));      // the S*p kernels stand still once a PCG has converged
    be_->hpp_mul(d, lambda, d.p, d.Ap);
    be_->schur_landmarks(d, 1, d.p);
    be_->schur_vertex_obs(d, -1.0, d.Ap);
    be_->schur_vertex_ter(d, -1.0, d.Ap);
    download6(d.Ap);
  } else if (kind == 1) {
    upload6(d.rhs);
    be_->pcg_init(d);
    download6(d.z);
  } else if (kind == 2) {
    download6(d.rhs);
  } else {
    upload6(d.xp);
    be_->vertex_transform(d, d.xp);
    be_->schur_landmarks(d, 2, d.xp);
    std::vector<double> xl(3 * (size_t)d.P);
    if (d.P) be_->d2h(xl.data(), d.xl, 24 * (size_t)d.P);
    for (int p = 0; p < P_all_; ++p) std::memcpy(out + 3 * (size_t)p, &xl[3 * (size_t)new_of_old_[p]], 24);
  }
  return VDO_OK;
}

int BaGraph::debug_solve(double lambda, double pcg_rel_tol, int pcg_max_iterations, double* xp, double* xl, double* r_rec, int* pcg_iters) {
  if (!finalized_) return fail(VDO_ERR_STATE, "debug_solve before finalize");
  if (be_->world > 1) return fail(VDO_ERR_STATE, "debug_solve: sharded graphs are not supported");
  if (!(lambda >= 0)) return fail(VDO_ERR_ARG, "debug_solve: bad lambda");
  BaDev& d = d_;
  const double tol = pcg_rel_tol > 0 ? pcg_rel_tol : 1e-6;
  int it = 0;
  bool ok = lone(BACKSUB, lambda, d.Sdense ? BaBackend::BATCH_DENSE : BaBackend::BATCH_PCG, tol * tol, pcg_max_iterations > 0 ? pcg_max_iterations : 2000, &it);
  if (d.Sdense) { double st; be_->d2h(&st, d.scal + SC_DENSE, sizeof(double)); ok = st == 0.0; }
  read_se3_vec(d.xp, xp);
  read_se3_vec(d.Sdense ? nullptr : d.r, r_rec);
  read_pt_vec(d.xl, xl);
  if (pcg_iters) *pcg_iters = it;
  return ok ? VDO_OK : fail(VDO_ERR_UNSUPPORTED, "debug_solve: the linear solve broke down (reduced matrix not positive definite)");
}

void BaGraph::read_se3_vec(const double* src, double* dst) {
  if (!dst) return;
  const int C = d_.C;
  std::vector<double> v(6 * (size_t)C, 0.0);
  if (src && C) be_->d2h(v.data(), src, 48 * (size_t)C);
  for (int c = 0; c < C; ++c) std::memcpy(dst + 6 * (size_t)c, &v[6 * (size_t)new_se3_of_old_[c]], 48);
}
void BaGraph::read_pt_vec(const double* src, double* dst) {
  if (!dst) return;
  std::vector<double> t(3 * (size_t)d_.P);
  if (d_.P) be_->d2h(t.data(), src, 24 * (size_t)d_.P);
  for (int p = 0; p < P_all_; ++p) {
    const int k = new_of_old_[p];
    if (k >= 0) std::memcpy(dst + 3 * (size_t)p, &t[3 * (size_t)k], 24);     // landmarks of other ranks: left untouched
  }
}

// One LM trial per graph exactly as optimize_batch takes it: batch_begin over all n graphs (so two or more dense-path graphs, or two or
// more PCG-path graphs of the tiled layout, share every launch), the linearisation, then the trial up to the update and the robust chi2
// of the new estimates.  The re-orthogonalisation is the caller's flag, so oplus_calls_ does not move; the pop at the end restores every
// graph's estimates, and the buffers the trial wrote are rewritten by any later trial before they are read.
int BaGraph::debug_trial(BaGraph* const* gs, int n, const double* lambda, const int* reortho, double pcg_rel_tol, int pcg_max_iterations,
                         double* const* xp, double* const* xl, double* const* se3, double* const* pt, double* chi2, double* scale,
                         int* pcg_iters, int* ok) {
  using B = BaBackend;
  BaBackend* be = gs[0]->be_;
  const double tol = pcg_rel_tol > 0 ? pcg_rel_tol : 1e-6;
  std::vector<BaDev*> ds(n);
  std::vector<int> it(n, 0), good(n, 1);
  Round r(n);
  for (int k = 0; k < n; ++k) { ds[k] = &gs[k]->d_; r.flag[k] = B::BATCH_LIN; }
  be->batch_begin(ds.data(), n);
  lin_round(gs, n, r);
  for (int k = 0; k < n; ++k) {
    r.flag[k] = B::BATCH_TRIAL | (gs[k]->d_.Sdense ? B::BATCH_DENSE : B::BATCH_PCG);
    r.lam[k] = lambda[k]; r.rt[k] = reortho && reortho[k] ? 1 : 0; r.tol2[k] = tol * tol;
  }
  trial_round(gs, n, r, pcg_max_iterations > 0 ? pcg_max_iterations : 2000, UPDATE, nullptr, it.data(), good.data());
  be->batch_end();
  for (int k = 0; k < n; ++k) {
    BaGraph* g = gs[k];
    const BaDev& d = g->d_;
    double sc[SC_N];
    be->d2h(sc, d.scal, sizeof sc);
    if (chi2) chi2[k] = sc[SC_CHI2];
    if (scale) scale[k] = sc[SC_SCALE];
    if (pcg_iters) pcg_iters[k] = it[k];
    if (ok) ok[k] = good[k] && !(d.Sdense && sc[SC_DENSE] != 0.0);
    if (xp) g->read_se3_vec(d.xp, xp[k]);
    if (xl) g->read_pt_vec(d.xl, xl[k]);
    g->get_vertices(se3 ? se3[k] : nullptr, pt ? pt[k] : nullptr);
    g->pop();
  }
  return VDO_OK;
}

}  // namespace vdo
