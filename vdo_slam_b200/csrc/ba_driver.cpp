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
void make_chunks(const std::vector<int>& begin, std::vector<Chunk>& out) {
  for (int v = 0; v + 1 < (int)begin.size(); ++v)
    for (int b = begin[v]; b < begin[v + 1]; b += VDO_CHUNK) out.push_back(Chunk{v, b, std::min(b + VDO_CHUNK, begin[v + 1]), 0});
}
}  // namespace

int BaGraph::finalize() {
  if (finalized_) return fail(VDO_ERR_STATE, "finalize called twice");
  const bool prof_fin = std::getenv("VDO_PROFILE") != nullptr;
  auto tp0 = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!prof_fin) return;
    auto t = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[vdo_b200] finalize: %-28s %.1f ms\n", what, std::chrono::duration<double, std::milli>(t - tp0).count());
    tp0 = t;
  };
  const int C = n_se3_; int P = n_pt_;
  const int Eo_all = (int)ob_w_.size(), Et_all = (int)te_w_.size(), Es = (int)se_w_.size(), Ep = (int)pr_w_.size();
  // ---- se3 vertices: renumber so that every path of the se3-se3 edge graph (camera odometry chain, per-object
  //      motion-smoothness chains) is a contiguous, ordered index range; other vertices become singleton paths ----
  std::vector<int> path_begin;
  {
    std::vector<int> deg(C, 0), nb0(C, -1), nb1(C, -1), comp(C);
    std::iota(comp.begin(), comp.end(), 0);
    auto find = [&](int x) { while (comp[x] != x) { comp[x] = comp[comp[x]]; x = comp[x]; } return x; };
    std::vector<char> bad_comp(C, 0);
    for (int e = 0; e < Es; ++e) {
      int a = se_ij_[2 * e], b = se_ij_[2 * e + 1];
      int ra = find(a), rb = find(b);
      if (ra == rb) bad_comp[ra] = 1;            // cycle or duplicate edge
      else { comp[ra] = rb; if (bad_comp[ra]) bad_comp[rb] = 1; }
      if (deg[a] == 0) nb0[a] = b; else if (deg[a] == 1) nb1[a] = b;
      if (deg[b] == 0) nb0[b] = a; else if (deg[b] == 1) nb1[b] = a;
      deg[a]++; deg[b]++;
    }
    for (int v = 0; v < C; ++v) if (deg[v] > 2) bad_comp[find(v)] = 1;
    for (int v = 0; v < C; ++v) if (bad_comp[v] && comp[v] == v) { /* propagated below through find() */ }
    new_se3_of_old_.assign(C, -1);
    int cnt = 0;
    for (int v = 0; v < C; ++v) {
      if (new_se3_of_old_[v] != -1) continue;
      const bool is_path = !bad_comp[find(v)];
      if (!is_path || deg[v] == 0) { path_begin.push_back(cnt); new_se3_of_old_[v] = cnt++; continue; }
      if (deg[v] == 2) continue;                 // interior vertex: reached from its path's smaller endpoint
      path_begin.push_back(cnt);
      int prev = -1, cur = v;
      while (cur != -1) {
        new_se3_of_old_[cur] = cnt++;
        int nx = (nb0[cur] != prev) ? nb0[cur] : nb1[cur];
        if (deg[cur] == 1 && prev != -1) nx = -1;
        prev = cur; cur = nx;
      }
    }
    for (int v = 0; v < C; ++v) if (new_se3_of_old_[v] == -1) { path_begin.push_back(cnt); new_se3_of_old_[v] = cnt++; }  // safety
    path_begin.push_back(cnt);
  }
  auto S3 = [&](int old_id) { return new_se3_of_old_[old_id]; };
  lap("se3 paths");
  // ---- tracklets: chains of landmarks linked by ternary edges ----
  HostBuf<int> next = stage_fill<int>(P, 0xFF), prev = stage_fill<int>(P, 0xFF), ter_of = stage_fill<int>(P, 0xFF);
  for (int e = 0; e < Et_all; ++e) {
    int p1 = te_pph_[3 * e], p2 = te_pph_[3 * e + 1];
    if (p1 == p2 || next[p1] != -1 || prev[p2] != -1)
      return fail(VDO_ERR_UNSUPPORTED, "landmark-motion edges must form simple chains (one predecessor / successor per landmark)");
    next[p1] = p2; prev[p2] = p1; ter_of[p1] = e;
  }
  lap("  chain links");
  new_of_old_.assign(P, -1);
  HostBuf<int> old_of_new = stage<int>(P);
  std::vector<int> tk_begin;
  int cnt = 0;
  // Tracklet order.  Static landmarks (tracklets of one vertex) first, then the chains: the two groups run different
  // kernels.  Inside each group tracklets are ordered by the first se3 vertex that observes them (chains: by the motion
  // vertex of their first ternary edge, then by the first observing camera), so that the landmarks of one tile meet only
  // a few se3 vertices and the per-tile vertex-sorted segments stay long.  Counting sorts: O(P + C).
  // Multi-GPU: tracklets are dealt round-robin to the ranks (each group separately, in this order); a rank keeps only its
  // own landmarks and their edges, the se3 state is replicated.
  const int rank = be_->rank, world = be_->world;
  // Edge partition: the pointxyz edges are split, in the caller's order, into NB buckets of consecutive (old) landmark ids --
  // a stable parallel counting sort by bucket (chunk t of the edge list counts, then writes its edge indices behind the
  // chunks before it).  Everything per-landmark below (first camera, edge count, the scatter into landmark order) is then
  // done by the worker that owns the bucket, reading only its own edges: O(E) work in total and the same result for any
  // thread count.
  const int NT = host_threads(), NB = NT, P0 = std::max(P, 1);
  auto bucket_of = [NB, P0](int p) { return (int)((int64_t)p * NB / P0); };
  std::vector<int64_t> tb((size_t)NT * NB + 1, 0);
  parallel_for(NT, [&](int t, int n) {
    const int a = (int)((int64_t)Eo_all * t / n), b = (int)((int64_t)Eo_all * (t + 1) / n);
    int64_t* c = &tb[(size_t)t * NB];
    for (int e = a; e < b; ++e) c[bucket_of(ob_cp_[2 * e + 1])]++;
  });
  std::vector<int64_t> off((size_t)NB * NT + 1, 0);      // off[b * NT + t]: first slot of chunk t inside bucket b
  { int64_t run = 0; for (int b = 0; b < NB; ++b) for (int t = 0; t < NT; ++t) { off[(size_t)b * NT + t] = run; run += tb[(size_t)t * NB + b]; } off[(size_t)NB * NT] = run; }
  HostBuf<int> eidx = stage<int>(Eo_all);
  parallel_for(NT, [&](int t, int n) {
    const int a = (int)((int64_t)Eo_all * t / n), b = (int)((int64_t)Eo_all * (t + 1) / n);
    std::vector<int64_t> cur(NB);
    for (int k = 0; k < NB; ++k) cur[k] = off[(size_t)k * NT + t];
    for (int e = a; e < b; ++e) eidx[cur[bucket_of(ob_cp_[2 * e + 1])]++] = e;
  });
  HostBuf<int> first_cam = stage<int>(P), cnt_old = stage_fill<int>(P, 0);
  parallel_for(NB, [&](int b, int) {
    const int lo = (int)(((int64_t)b * P + NB - 1) / NB), hi = (int)(((int64_t)(b + 1) * P + NB - 1) / NB);   // landmarks p with bucket_of(p) == b
    for (int p = lo; p < hi && p < P; ++p) first_cam[p] = C;
    for (int64_t q = off[(size_t)b * NT]; q < off[(size_t)(b + 1) * NT]; ++q) {
      const int e = eidx[q], p = ob_cp_[2 * e + 1], c = S3(ob_cp_[2 * e]);
      if (c < first_cam[p]) first_cam[p] = c;
      cnt_old[p]++;
    }
  });
  lap("  first_cam scan");
  // stable counting sort of ids by key_of_id[id], in parallel: chunk t of the list counts its keys, the (key, chunk) prefix gives every chunk
  // its output cursor per key, every chunk scatters its ids in order -- the result of a stable sort does not depend on the thread count
  auto counting_sort = [&](std::vector<int>& ids, const HostBuf<int>& key_of_id, int nkeys) {
    const size_t n = ids.size();
    if (n == 0) return;
    const int W = (n < 65536 || (size_t)nkeys * NT > 4 * n) ? 1 : NT;
    std::vector<int> keys(n), out(n);
    std::vector<int> hist((size_t)W * nkeys, 0);
    parallel_for(W, [&](int t, int w) {
      const size_t a = n * t / w, b = n * (t + 1) / w;
      int* h = &hist[(size_t)t * nkeys];
      for (size_t i = a; i < b; ++i) { const int k = key_of_id[ids[i]]; keys[i] = k; h[k]++; }
    });
    { int run = 0; for (int k = 0; k < nkeys; ++k) for (int t = 0; t < W; ++t) { int& h = hist[(size_t)t * nkeys + k]; const int c = h; h = run; run += c; } }
    parallel_for(W, [&](int t, int w) {
      const size_t a = n * t / w, b = n * (t + 1) / w;
      int* h = &hist[(size_t)t * nkeys];
      for (size_t i = a; i < b; ++i) out[h[keys[i]]++] = ids[i];
    });
    ids.swap(out);
  };
  std::vector<int> stat_ids, chain_heads;
  {   // heads of tracklets, in landmark order (parallel count, then fill)
    std::vector<size_t> ns(NT + 1, 0), nc(NT + 1, 0);
    parallel_for(NT, [&](int t, int n) {
      const int a = (int)((int64_t)P * t / n), b = (int)((int64_t)P * (t + 1) / n);
      size_t s0 = 0, c0 = 0;
      for (int p = a; p < b; ++p) if (prev[p] == -1) { if (next[p] == -1) ++s0; else ++c0; }
      ns[t + 1] = s0; nc[t + 1] = c0;
    });
    for (int t = 0; t < NT; ++t) { ns[t + 1] += ns[t]; nc[t + 1] += nc[t]; }
    stat_ids.resize(ns[NT]); chain_heads.resize(nc[NT]);
    parallel_for(NT, [&](int t, int n) {
      const int a = (int)((int64_t)P * t / n), b = (int)((int64_t)P * (t + 1) / n);
      size_t s0 = ns[t], c0 = nc[t];
      for (int p = a; p < b; ++p) if (prev[p] == -1) { if (next[p] == -1) stat_ids[s0++] = p; else chain_heads[c0++] = p; }
    });
  }
  lap("  collect heads");
  {   // static landmarks: by first observing camera, inside one camera by DESCENDING edge count -- the lanes of a warp that loops over
      // its landmarks' edges then run the same trip counts (geometric track lengths: a warp of mixed landmarks idles ~55 % of its lanes)
    int mx = 0;
    for (int p : stat_ids) mx = std::max(mx, cnt_old[p]);
    HostBuf<int> neg = stage<int>(P);
    parallel_for(NT, [&](int t, int n) {
      const size_t a = stat_ids.size() * t / n, b = stat_ids.size() * (t + 1) / n;
      for (size_t i = a; i < b; ++i) neg[stat_ids[i]] = mx - cnt_old[stat_ids[i]];
    });
    counting_sort(stat_ids, neg, mx + 1);
  }
  counting_sort(stat_ids, first_cam, C + 1);
  {
    HostBuf<int> first_h = stage_fill<int>(P, 0);
    for (int p : chain_heads) first_h[p] = S3(te_pph_[3 * ter_of[p] + 2]);
    counting_sort(chain_heads, first_cam, C + 1);
    counting_sort(chain_heads, first_h, C + 1);
  }
  lap("  counting sorts");
  // chain lengths (parallel walks); every landmark must be a static point or lie on a chain that starts at a head
  const int n_heads = (int)chain_heads.size();
  std::vector<int> chain_len(n_heads);
  std::vector<int64_t> seen_part(NT, 0);
  parallel_for(NT, [&](int t, int n) {
    const int a = (int)((int64_t)n_heads * t / n), b = (int)((int64_t)n_heads * (t + 1) / n);
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
  tk_begin.resize((size_t)Tstat + Tch + 1);
  { int run = Tstat; for (int i = 0; i < Tch; ++i) { tk_begin[Tstat + i] = run; run += head_len[i]; } tk_begin[Tstat + Tch] = run; cnt = run; }
  parallel_for(NT, [&](int t, int n) {
    const int a = (int)((int64_t)Tstat * t / n), b = (int)((int64_t)Tstat * (t + 1) / n);
    for (int i = a; i < b; ++i) { tk_begin[i] = i; new_of_old_[stat_keep[i]] = i; old_of_new[i] = stat_keep[i]; }
    const int c = (int)((int64_t)Tch * t / n), d2 = (int)((int64_t)Tch * (t + 1) / n);
    for (int i = c; i < d2; ++i) { int k = tk_begin[Tstat + i]; for (int q = head_keep[i]; q != -1; q = next[q]) { new_of_old_[q] = k; old_of_new[k++] = q; } }
  });
  const int P_all = P;
  P = cnt;                      // from here on P = landmarks owned by this rank
  const int T = (int)tk_begin.size() - 1;

  lap("tracklet order");
  ClassTable oc, tc;
  // ---- landmark-major pointxyz stream ----
  // Edge classes first (sequential; consecutive edges almost always share their (information, delta) pair), then the scatter
  // into landmark order by worker threads that each own a contiguous landmark range and scan the edge list in order, so the
  // order of a landmark's edges is the caller's order whatever the thread count.
  HostBuf<uint8_t> ecls = stage<uint8_t>(Eo_all);
  {
    // fast path: every edge carries the first edge's (information, delta) pair (checked in parallel)
    std::vector<char> uniform(NT, 1);
    if (Eo_all > 0) {
      const double w0 = ob_w_[0], d0 = ob_d_[0];
      parallel_for(NT, [&](int t, int n) {
        const int a = (int)((int64_t)Eo_all * t / n), b = (int)((int64_t)Eo_all * (t + 1) / n);
        char u = 1;
        for (int e = a; e < b; ++e) if (ob_w_[e] != w0 || ob_d_[e] != d0) { u = 0; break; }
        uniform[t] = u;
      });
    }
    bool all_uniform = Eo_all > 0;
    for (char u : uniform) all_uniform = all_uniform && u;
    if (all_uniform) { const int c0 = oc.get(ob_w_[0], ob_d_[0]); fill_bytes(ecls.p, c0, (size_t)Eo_all); }
    else {
      double lw = 0, ld = 0; int lc = -1;
      for (int e = 0; e < Eo_all; ++e) {
        if (lc < 0 || ob_w_[e] != lw || ob_d_[e] != ld) {
          lc = oc.get(ob_w_[e], ob_d_[e]); lw = ob_w_[e]; ld = ob_d_[e];
          if (lc > 255) return fail(VDO_ERR_UNSUPPORTED, "more than 256 distinct (information, Huber delta) pairs on pointxyz edges");
        }
        ecls[e] = (uint8_t)lc;
      }
    }
  }
  lap("  edge classes");
  // edges per landmark in the new order (gathered from the per-old-landmark counts), prefix sum, then the scatter: the worker
  // that owns a bucket walks its edges in the caller's order and appends each to its landmark's slot range
  HostBuf<int> lm_begin = stage<int>((size_t)P + 1);
  lm_begin[0] = 0;
  parallel_for(NT, [&](int t, int n) {
    const int a = (int)((int64_t)P * t / n), b = (int)((int64_t)P * (t + 1) / n);
    for (int k = a; k < b; ++k) lm_begin[k + 1] = cnt_old[old_of_new[k]];
  });
  lap("  count");
  for (int k = 0; k < P; ++k) lm_begin[k + 1] += lm_begin[k];
  const int Eo = lm_begin[P];
  HostBuf<int> lm_cam = stage<int>(Eo);
  HostBuf<double> lm_z = stage<double>(3 * (size_t)Eo);
  HostBuf<uint8_t> lm_cls = stage<uint8_t>(Eo);
  fill_bytes(cnt_old.p, 0, sizeof(int) * (size_t)P_all);        // reused: edges of the (old) landmark written so far
  lap("  prefix + alloc");
  parallel_for(NB, [&](int b, int) {
    for (int64_t q = off[(size_t)b * NT]; q < off[(size_t)(b + 1) * NT]; ++q) {
      const int e = eidx[q], p = ob_cp_[2 * e + 1], k = new_of_old_[p];
      if (k < 0) continue;                                       // landmark owned by another rank
      const int pos = lm_begin[k] + cnt_old[p]++;
      lm_cam[pos] = new_se3_of_old_[ob_cp_[2 * e]];
      lm_z[3 * (size_t)pos] = ob_z_[3 * (size_t)e]; lm_z[3 * (size_t)pos + 1] = ob_z_[3 * (size_t)e + 1]; lm_z[3 * (size_t)pos + 2] = ob_z_[3 * (size_t)e + 2];
      lm_cls[pos] = ecls[e];
    }
  });
  lap("landmark-major stream");
  // ---- layout choice: tiles of whole tracklets (default) or, when a tracklet is too large for a tile (more than
  //      VDO_TILE_L landmarks or VDO_TILE_E pointxyz edges) or VDO_BA_LAYOUT=chunked is set, the chunked vertex-major layout ----
  std::vector<Tile> tiles;
  int n_tiles_stat = 0;
  bool tiled = true;
  {
    const char* env = std::getenv("VDO_BA_LAYOUT");
    if (env && std::string(env) == "chunked") tiled = false;
    // Greedy packing of whole tracklets into tiles, inside FIXED segments of the tracklet order (their number depends on the graph only, so
    // the layout is the same for any thread count); a tile never spans two segments, hence the segments pack in parallel.  A tile also meets
    // at most 255 distinct cameras (edges address them by an 8-bit slot): cam_tile[c] = serial of the tile that saw camera c last.
    const int nseg_st = std::max(1, std::min(48, Tstat / 8192)), nseg_ch = std::max(1, std::min(16, (T - Tstat) / 2048));
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
    if (tiled) {
      const int nseg = nseg_st + nseg_ch;
      parallel_for(std::min(NT, nseg), [&](int w, int n) {
        for (int sg = w; sg < nseg; sg += n) {
          if (sg < nseg_st) pack((int)((int64_t)Tstat * sg / nseg_st), (int)((int64_t)Tstat * (sg + 1) / nseg_st), segs[sg]);
          else { const int c = sg - nseg_st, Tc = T - Tstat; pack(Tstat + (int)((int64_t)Tc * c / nseg_ch), Tstat + (int)((int64_t)Tc * (c + 1) / nseg_ch), segs[sg]); }
        }
      });
      for (int sg = 0; sg < nseg && tiled; ++sg) {
        if (segs[sg].bad) tiled = false;
        if (sg == nseg_st) n_tiles_stat = (int)tiles.size();
        tiles.insert(tiles.end(), segs[sg].tiles.begin(), segs[sg].tiles.end());
      }
      if (!tiled) tiles.clear();
    }
  }
  std::vector<int> vm_begin(C + 1, 0), vm_pt;
  std::vector<double> vm_z;
  std::vector<uint8_t> vm_cls;
  std::vector<Chunk> obs_chunks;
  if (!tiled) {
  // ---- vertex-major pointxyz stream: walk the landmark-major stream so each vertex's edges stay landmark-sorted ----
  for (int pos = 0; pos < Eo; ++pos) vm_begin[lm_cam[pos] + 1]++;
  for (int v = 0; v < C; ++v) vm_begin[v + 1] += vm_begin[v];
  std::vector<int> vfill(vm_begin.begin(), vm_begin.end() - 1);
  vm_pt.resize(Eo); vm_z.resize(3 * (size_t)Eo); vm_cls.resize(Eo);
  {
    int k = 0;
    for (int pos = 0; pos < Eo; ++pos) {
      while (lm_begin[k + 1] <= pos) ++k;
      int q = vfill[lm_cam[pos]]++;
      vm_pt[q] = k; vm_cls[q] = lm_cls[pos];
      for (int i = 0; i < 3; ++i) vm_z[3 * (size_t)q + i] = lm_z[3 * (size_t)pos + i];
    }
  }
  make_chunks(vm_begin, obs_chunks);
  }
  // ---- ternary edges: per landmark (as p1) and motion-vertex-major ----
  HostBuf<int> tk_h = stage_fill<int>(P, 0xFF);
  HostBuf<uint8_t> tk_cls = stage_fill<uint8_t>(P, 0);
  std::vector<int> hm_begin(C + 1, 0);
  int Et = 0;
  {
    HostBuf<uint8_t> tcls = stage<uint8_t>(Et_all);
    double lw = 0, ld = 0; int lc = -1;
    for (int e = 0; e < Et_all; ++e) {                       // classes: sequential with a last-value cache (one map look-up per change)
      if (lc < 0 || te_w_[e] != lw || te_d_[e] != ld) {
        lc = tc.get(te_w_[e], te_d_[e]); lw = te_w_[e]; ld = te_d_[e];
        if (lc > 255) return fail(VDO_ERR_UNSUPPORTED, "more than 256 distinct (information, Huber delta) pairs on landmark-motion edges");
      }
      tcls[e] = (uint8_t)lc;
    }
    std::vector<int> et_part(NT, 0);
    parallel_for(NT, [&](int t, int n) {                     // every landmark is p1 of at most one edge: the writes are disjoint
      const int a = (int)((int64_t)Et_all * t / n), b = (int)((int64_t)Et_all * (t + 1) / n);
      int cnt_t = 0;
      for (int e = a; e < b; ++e) {
        const int k = new_of_old_[te_pph_[3 * e]];
        if (k < 0) continue;
        ++cnt_t;
        tk_h[k] = S3(te_pph_[3 * e + 2]); tk_cls[k] = tcls[e];
      }
      et_part[t] = cnt_t;
    });
    for (int c : et_part) Et += c;
    if (!tiled) for (int k = 0; k < P; ++k) if (tk_h[k] >= 0) hm_begin[tk_h[k] + 1]++;
  }
  std::vector<int> hm_p1;
  std::vector<uint8_t> hm_cls;
  std::vector<Chunk> ter_chunks;
  if (!tiled) {
    for (int v = 0; v < C; ++v) hm_begin[v + 1] += hm_begin[v];
    std::vector<int> hfill(hm_begin.begin(), hm_begin.end() - 1);
    hm_p1.resize(Et); hm_cls.resize(Et);
    for (int k = 0; k < P; ++k) {   // landmark order keeps each motion vertex's edges landmark-sorted
      if (tk_h[k] < 0) continue;
      int q = hfill[tk_h[k]]++;
      hm_p1[q] = k; hm_cls[q] = tk_cls[k];
    }
    make_chunks(hm_begin, ter_chunks);
  }
  lap("ternary / chunked streams");
  // ---- tiles: tile-local landmark of every edge, vertex-sorted order of the tile's edges, segments of one vertex ----
  HostBuf<uint16_t> ob_perm, tr_perm;
  HostBuf<uint8_t> lm_lml, lm_cslot, tk_hslot;
  HostBuf<uint32_t> ob_ps;
  std::vector<int> tile_verts;
  std::vector<Seg> osegs, tsegs, osegs2, tsegs2;
  if (tiled) {
    ob_perm = stage<uint16_t>(Eo); tr_perm = stage_fill<uint16_t>(P, 0); lm_lml = stage<uint8_t>(Eo); ob_ps = stage<uint32_t>(Eo);
    lm_cslot = stage<uint8_t>(Eo); tk_hslot = stage_fill<uint8_t>(P, 0xFF);
    // tiles are independent: each worker handles a contiguous range of tiles into its own segment lists, which are then
    // concatenated in tile order (segment indices of a tile are rebased by the lists that precede it)
    const int ntl = (int)tiles.size();
    const int NW = std::max(1, std::min(NT, ntl / 64 + 1));
    std::vector<std::vector<Seg>> w_os(NW), w_ts(NW), w_os2(NW), w_ts2(NW);
    std::vector<std::vector<int>> w_tv(NW);
    std::vector<char> w_bad(NW, 0);
    parallel_for(NW, [&](int wt, int wn) {
      std::vector<int> keys(std::max(VDO_TILE_E, VDO_TILE_L)), idx(keys.size()), bucket;
      std::vector<Seg>& los = w_os[wt]; std::vector<Seg>& lts = w_ts[wt];
      std::vector<Seg>& los2 = w_os2[wt]; std::vector<Seg>& lts2 = w_ts2[wt];
      std::vector<int>& ltv = w_tv[wt];
      // stable sort of idx[0..n) by keys[idx] (counting sort over the key range when it is small), then cut into segments
      auto sort_and_cut = [&](int n, int base, HostBuf<uint16_t>& perm, std::vector<Seg>& segs, std::vector<Seg>& segs2) {
        if (n == 0) return;
        int lo = keys[idx[0]], hi = lo;
        for (int a = 1; a < n; ++a) { lo = std::min(lo, keys[idx[a]]); hi = std::max(hi, keys[idx[a]]); }
        const int range = hi - lo + 1;
        if (range <= 8 * n + 64) {
          bucket.assign(range + 1, 0);
          for (int a = 0; a < n; ++a) bucket[keys[idx[a]] - lo + 1]++;
          for (int r = 0; r < range; ++r) bucket[r + 1] += bucket[r];
          for (int a = 0; a < n; ++a) perm[base + bucket[keys[idx[a]] - lo]++] = (uint16_t)idx[a];
        } else {
          std::stable_sort(idx.begin(), idx.begin() + n, [&](int x, int y) { return keys[x] < keys[y]; });
          for (int a = 0; a < n; ++a) perm[base + a] = (uint16_t)idx[a];
        }
        for (int a = 0; a < n;) {
          const int v = keys[perm[base + a]];
          int b = a;
          while (b < n && b - a < VDO_SEG && keys[perm[base + b]] == v) ++b;
          segs.push_back(Seg{v, base + a, b - a, 0});
          a = b;
        }
        for (int a = 0; a < n;) {                 // the same runs cut at VDO_SEG2 entries (Schur kernels: one thread per (run, component))
          const int v = keys[perm[base + a]];
          int b = a;
          while (b < n && b - a < VDO_SEG2 && keys[perm[base + b]] == v) ++b;
          segs2.push_back(Seg{v, base + a, b - a, 0});
          a = b;
        }
      };
      const int ta = (int)((int64_t)ntl * wt / wn), tb = (int)((int64_t)ntl * (wt + 1) / wn);
      for (int ti = ta; ti < tb; ++ti) {
        Tile& tl = tiles[ti];
        for (int k = tl.k0; k < tl.k1; ++k) for (int e = lm_begin[k]; e < lm_begin[k + 1]; ++e) lm_lml[e] = (uint8_t)(k - tl.k0);
        const int ne = tl.e1 - tl.e0;
        for (int i = 0; i < ne; ++i) { keys[i] = lm_cam[tl.e0 + i]; idx[i] = i; }
        tl.os0 = (int)los.size(); tl.qo0 = (int)los2.size();
        sort_and_cut(ne, tl.e0, ob_perm, los, los2);
        tl.os1 = (int)los.size(); tl.qo1 = (int)los2.size();
        // sorted order: permutation and tile-local landmark in one word; the tile's camera list = the vertices of its sorted runs
        tl.vs0 = (int)ltv.size();
        int ncam = 0, nmot = 0;
        for (int q = 0; q < ne; ++q) {
          const int i = ob_perm[tl.e0 + q];
          ob_ps[tl.e0 + q] = (uint32_t)i | ((uint32_t)lm_lml[tl.e0 + i] << 16);
          const int cam = lm_cam[tl.e0 + i];
          if (q == 0 || cam != lm_cam[tl.e0 + ob_perm[tl.e0 + q - 1]]) { ltv.push_back(cam); ++ncam; }
          lm_cslot[tl.e0 + i] = (uint8_t)(ncam - 1);
        }
        int nt = 0;
        for (int k = tl.k0; k < tl.k1; ++k) if (tk_h[k] >= 0) { keys[k - tl.k0] = tk_h[k]; idx[nt++] = k - tl.k0; }
        tl.ts0 = (int)lts.size(); tl.qt0 = (int)lts2.size();
        sort_and_cut(nt, tl.k0, tr_perm, lts, lts2);
        tl.ts1 = (int)lts.size(); tl.qt1 = (int)lts2.size();
        for (int q = 0; q < nt; ++q) {
          const int j = tr_perm[tl.k0 + q], h = tk_h[tl.k0 + j];
          if (q == 0 || h != tk_h[tl.k0 + tr_perm[tl.k0 + q - 1]]) { ltv.push_back(h); ++nmot; }
          tk_hslot[tl.k0 + j] = (uint8_t)(nmot - 1);
        }
        if (ncam > 255 || nmot > 255) w_bad[wt] = 1;
        tl.nv = ncam | (nmot << 16);
      }
    });
    for (int wt = 0; wt < NW; ++wt) {
      const int ta = (int)((int64_t)ntl * wt / NW), tb = (int)((int64_t)ntl * (wt + 1) / NW);
      const int ob = (int)osegs.size(), tb0 = (int)tsegs.size(), ob2 = (int)osegs2.size(), tb2 = (int)tsegs2.size();
      for (int ti = ta; ti < tb; ++ti) {
        tiles[ti].os0 += ob; tiles[ti].os1 += ob; tiles[ti].ts0 += tb0; tiles[ti].ts1 += tb0;
        tiles[ti].qo0 += ob2; tiles[ti].qo1 += ob2; tiles[ti].qt0 += tb2; tiles[ti].qt1 += tb2;
      }
      osegs.insert(osegs.end(), w_os[wt].begin(), w_os[wt].end());
      tsegs.insert(tsegs.end(), w_ts[wt].begin(), w_ts[wt].end());
      osegs2.insert(osegs2.end(), w_os2[wt].begin(), w_os2[wt].end());
      tsegs2.insert(tsegs2.end(), w_ts2[wt].begin(), w_ts2[wt].end());
      const int vb0 = (int)tile_verts.size();
      for (int ti = ta; ti < tb; ++ti) tiles[ti].vs0 += vb0;
      tile_verts.insert(tile_verts.end(), w_tv[wt].begin(), w_tv[wt].end());
      if (w_bad[wt]) return fail(VDO_ERR_UNSUPPORTED, "a tile meets more than 255 motion vertices");
    }
  }
  lap("tile segments");
  // ---- se3-se3 edges (priors first, j = -1) and H_pp adjacency ----
  const int Ese = Ep + Es;
  std::vector<int> se_i(Ese), se_j(Ese);
  std::vector<double> se_Z(12 * (size_t)Ese), se_w(Ese), se_d(Ese);
  for (int e = 0; e < Ep; ++e) { se_i[e] = S3(pr_v_[e]); se_j[e] = -1; se_w[e] = pr_w_[e]; se_d[e] = 0; std::memcpy(&se_Z[12 * (size_t)e], &pr_Z_[12 * (size_t)e], 96); }
  for (int e = 0; e < Es; ++e) {
    int q = Ep + e;
    se_i[q] = S3(se_ij_[2 * e]); se_j[q] = S3(se_ij_[2 * e + 1]); se_w[q] = se_w_[e]; se_d[q] = se_d_[e] > 0 ? se_d_[e] : 0;
    std::memcpy(&se_Z[12 * (size_t)q], &se_Z_[12 * (size_t)e], 96);
  }
  std::vector<int> nbr_begin(C + 1, 0);
  for (int e = Ep; e < Ese; ++e) { nbr_begin[se_i[e] + 1]++; nbr_begin[se_j[e] + 1]++; }
  for (int v = 0; v < C; ++v) nbr_begin[v + 1] += nbr_begin[v];
  std::vector<int> nfill(nbr_begin.begin(), nbr_begin.end() - 1), nbr_edge(2 * (size_t)Es), nbr_other(2 * (size_t)Es);
  std::vector<uint8_t> nbr_tr(2 * (size_t)Es);
  for (int e = Ep; e < Ese; ++e) {
    int a = nfill[se_i[e]]++; nbr_edge[a] = e; nbr_other[a] = se_j[e]; nbr_tr[a] = 0;
    int b = nfill[se_j[e]]++; nbr_edge[b] = e; nbr_other[b] = se_i[e]; nbr_tr[b] = 1;
  }
  // ---- chain-preconditioner wiring: edge between internal vertices v-1 and v of the same path ----
  const int n_paths = (int)path_begin.size() - 1;
  std::vector<int> path_of(C), pcr_edge(C, -1);
  std::vector<uint8_t> pcr_tr(C, 0);
  int max_len = 1;
  for (int pth = 0; pth < n_paths; ++pth) {
    for (int v = path_begin[pth]; v < path_begin[pth + 1]; ++v) path_of[v] = pth;
    max_len = std::max(max_len, path_begin[pth + 1] - path_begin[pth]);
  }
  for (int e = Ep; e < Ese; ++e) {
    int a = se_i[e], b = se_j[e];
    if (path_of[a] != path_of[b]) continue;       // (only inside non-path components, which were split into singletons)
    if (b == a + 1) { pcr_edge[b] = e; pcr_tr[b] = 1; }        // M(b, a) = H_ab^T
    else if (a == b + 1) { pcr_edge[a] = e; pcr_tr[a] = 0; }   // M(a, b) = H_ab
  }
  int pcr_levels = 0; while ((1 << pcr_levels) < max_len) ++pcr_levels;
  HostBuf<double> se3_int = stage<double>(12 * (size_t)C);
  for (int o = 0; o < C; ++o) std::memcpy(&se3_int[12 * (size_t)S3(o)], &h_se3_[12 * (size_t)o], 96);
  // ---- states in internal landmark order ----
  HostBuf<double> pt_int = stage<double>(3 * (size_t)P);
  parallel_for(NT, [&](int t, int n) {
    const int a = (int)((int64_t)P * t / n), b = (int)((int64_t)P * (t + 1) / n);
    for (int k = a; k < b; ++k) for (int i = 0; i < 3; ++i) pt_int[3 * (size_t)k + i] = h_pt_[3 * (size_t)old_of_new[k] + i];
  });

  lap("se3 edges, states");
  // ---- upload ----
  BaDev& d = d_;
  d.C = C; d.P = P; d.T = T; d.Tstat = Tstat; d.own = (rank == 0) ? 1 : 0;
  P_all_ = P_all; d.Eobs = Eo; d.Eter = Et; d.Ese = Ese;
  d.n_obs_chunks = (int)obs_chunks.size(); d.n_ter_chunks = (int)ter_chunks.size(); d.n_nbr = (int)nbr_edge.size();
  d.se3 = upload(se3_int); d.pt = upload(pt_int);
  d.se3_init = dalloc<double>(12 * (size_t)C); d.pt_init = dalloc<double>(3 * (size_t)P);
  be_->d2d(d.se3_init, d.se3, 96 * (size_t)C); be_->d2d(d.pt_init, d.pt, 24 * (size_t)P);
  d.se3_bk = dalloc<double>(12 * (size_t)C); d.pt_bk = dalloc<double>(3 * (size_t)P);
  d.tk_begin = upload(tk_begin);
  d.lm_obs_begin = upload(lm_begin); d.lm_cam = upload(lm_cam); d.lm_z = upload(lm_z); d.lm_cls = upload(lm_cls); d.lm_omega = dalloc<double>(Eo);
  d.tk_h = upload(tk_h); d.tk_cls = upload(tk_cls); d.tk_omega = dalloc<double>(P);
  d.tiled = tiled ? 1 : 0;
  if (!tiled) {
    d.vm_pt = upload(vm_pt); d.vm_z = upload(vm_z); d.vm_cls = upload(vm_cls); d.vm_omega = dalloc<double>(Eo); d.obs_chunks = upload(obs_chunks);
    d.hm_p1 = upload(hm_p1); d.hm_cls = upload(hm_cls); d.hm_omega = dalloc<double>(Et); d.ter_chunks = upload(ter_chunks);
  } else {
    d.n_tiles = (int)tiles.size(); d.n_tiles_stat = n_tiles_stat; d.n_osegs = (int)osegs.size(); d.n_tsegs = (int)tsegs.size();
    d.capE_st = d.capE_ch = 16; d.capV_st = d.capV_ch = d.capH_ch = 1;
    for (int ti = 0; ti < d.n_tiles; ++ti) {
      const bool st = ti < n_tiles_stat;
      int& cap = st ? d.capE_st : d.capE_ch;
      cap = std::max(cap, (tiles[ti].e1 - tiles[ti].e0 + 15) & ~15);
      int& cv = st ? d.capV_st : d.capV_ch;
      cv = std::max(cv, tiles[ti].nv & 0xFFFF);
      if (!st) d.capH_ch = std::max(d.capH_ch, tiles[ti].nv >> 16);
    }
    d.tiles = upload(tiles); d.osegs = upload(osegs); d.tsegs = upload(tsegs); d.osegs2 = upload(osegs2); d.tsegs2 = upload(tsegs2);
    d.ob_perm = upload(ob_perm); d.tr_perm = upload(tr_perm); d.lm_lml = upload(lm_lml); d.ob_ps = upload(ob_ps);
    d.tile_verts = upload(tile_verts); d.lm_cslot = upload(lm_cslot); d.tk_hslot = upload(tk_hslot);
    d.pt_Q = dalloc<double>(9 * (size_t)std::max(P - Tstat, 1));
    d.accO = dalloc<double>(16 * (size_t)C); d.accT = dalloc<double>(16 * (size_t)C); d.acc6 = dalloc<double>(12 * (size_t)C);
    d.vh = dalloc<double>(6 * (size_t)C);
  }
  d.se_i = upload(se_i); d.se_j = upload(se_j); d.se_Z = upload(se_Z); d.se_w = upload(se_w); d.se_delta = upload(se_d); d.se_Hoff = dalloc<double>(36 * (size_t)Ese);
  d.nbr_begin = upload(nbr_begin); d.nbr_edge = upload(nbr_edge); d.nbr_other = upload(nbr_other); d.nbr_tr = upload(nbr_tr);
  d.Hpp = dalloc<double>(42 * (size_t)C); d.bp = d.Hpp + 36 * (size_t)C; d.hll = dalloc<double>(P); d.bl = dalloc<double>(3 * (size_t)P);
  d.pt_s = dalloc<double>(P); d.Minv = dalloc<double>(36 * (size_t)C);
  d.pt_g = dalloc<double>(P); d.tk_gamma = dalloc<double>(P);
  d.n_paths = n_paths; d.pcr_levels = pcr_levels;
  d.path_begin = upload(path_begin); d.path_of = upload(path_of); d.pcr_edge = upload(pcr_edge); d.pcr_tr = upload(pcr_tr);
  d.pcr_D = dalloc<double>(72 * (size_t)C); d.pcr_L = dalloc<double>(72 * (size_t)C); d.pcr_Dinv = dalloc<double>(36 * (size_t)C);
  d.pcr_A = dalloc<double>(36 * (size_t)C * std::max(pcr_levels, 1)); d.pcr_G = dalloc<double>(36 * (size_t)C * std::max(pcr_levels, 1));
  d.pcr_b = dalloc<double>(12 * (size_t)C);
  d.xp = dalloc<double>(6 * (size_t)C); d.r = dalloc<double>(6 * (size_t)C); d.z = dalloc<double>(6 * (size_t)C);
  d.p = dalloc<double>(6 * (size_t)C); d.Ap = dalloc<double>(6 * (size_t)C); d.rhs = dalloc<double>(6 * (size_t)C);
  d.p2 = dalloc<double>(6 * (size_t)C); d.ticket = dalloc<unsigned int>(4);
  {
    const char* env = std::getenv("VDO_BA_DENSE");   // "0": never; default: whenever the graph qualifies
    const bool want = !(env && std::string(env) == "0");
    if (want && tiled && world == 1 && Tstat == T && 6 * C <= be_->dense_capacity()) d.Sdense = dalloc<double>((size_t)36 * C * C + 6 * (size_t)C + 8);
  }
  if (tiled && Tstat > 0 && be_->band_max_width() > 0) {
    // Explicit static block of the reduced matrix (banded in the se3 numbering): possible when every static landmark lists its
    // observing vertices in strictly increasing order within a window of band_max_width() consecutive vertex numbers (tracks over
    // consecutive frames).  Otherwise the matrix-free static tile kernel stays in the PCG.
    const char* env = std::getenv("VDO_BA_BAND");      // "0": never
    const int Wmax = be_->band_max_width();
    std::vector<int> w_W(NT, 0), w_v0(NT, C), w_v1(NT, -1), w_bad(NT, 0);
    parallel_for(NT, [&](int t, int n) {
      const int a = (int)((int64_t)Tstat * t / n), b = (int)((int64_t)Tstat * (t + 1) / n);
      int W = 0, v0 = C, v1 = -1, bad = 0;
      for (int k = a; k < b && !bad; ++k) {
        const int e0 = lm_begin[k], e1 = lm_begin[k + 1];
        if (e1 <= e0) continue;
        for (int e = e0 + 1; e < e1; ++e) if (lm_cam[e] <= lm_cam[e - 1]) { bad = 1; break; }
        W = std::max(W, lm_cam[e1 - 1] - lm_cam[e0] + 1); v0 = std::min(v0, lm_cam[e0]); v1 = std::max(v1, lm_cam[e1 - 1]);
      }
      w_W[t] = W; w_v0[t] = v0; w_v1[t] = v1; w_bad[t] = bad;
    });
    int W = 0, v0 = C, v1 = -1, bad = 0;
    for (int t = 0; t < NT; ++t) { W = std::max(W, w_W[t]); v0 = std::min(v0, w_v0[t]); v1 = std::max(v1, w_v1[t]); bad |= w_bad[t]; }
    if (!(env && std::string(env) == "0") && !bad && v1 >= v0 && W <= Wmax && (size_t)(v1 - v0 + 1) * W * 80 <= ((size_t)512 << 20)) {
      d.band_W = W; d.band_v0 = v0; d.band_n = v1 - v0 + 1;
      d.band = dalloc<double>((size_t)d.band_n * W * 10);
    }
  }
  d.zl = tiled ? nullptr : dalloc<double>(3 * (size_t)P); d.xl = dalloc<double>(3 * (size_t)P); d.vw = dalloc<double>(6 * (size_t)C);
  oc.w.resize(256, 0.0); oc.d.resize(256, 0.0); tc.w.resize(256, 0.0); tc.d.resize(256, 0.0);
  d.obs_cls_w = upload(oc.w); d.obs_cls_d = upload(oc.d); d.ter_cls_w = upload(tc.w); d.ter_cls_d = upload(tc.d);
  d.scal = dalloc<double>(SC_N);
  d.n_part_pap = tiled ? std::max(1, (C + 127) / 128) : 148;    // tiled: one partial of p.Ap per CTA of the finalize kernel (128 vertices each)
  d.n_part_rz = std::max(1, n_paths) * 8;
  d.part_pap = dalloc<double>(d.n_part_pap); d.part_rz = dalloc<double>(d.n_part_rz);
  {
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
  }
  be_->sync();
  lap("alloc + upload");
  // host staging is no longer needed (keep the landmark map for read-back)
  ob_z_ = HostBuf<double>(); ob_w_ = HostBuf<double>(); ob_d_ = HostBuf<double>(); ob_cp_ = HostBuf<int>();
  te_pph_ = HostBuf<int>(); te_w_ = HostBuf<double>(); te_d_ = HostBuf<double>();
  std::vector<double>().swap(se_Z_); std::vector<double>().swap(pr_Z_);
  h_se3_ = HostBuf<double>(); h_pt_ = HostBuf<double>();
  n_prior_ = Ep;
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
      const int a = (int)((int64_t)Pa * t / n), b = (int)((int64_t)Pa * (t + 1) / n);
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
  double loose_tol = opt.pcg_loose_tol, switch_gain = opt.pcg_switch_gain;
  if (const char* e = std::getenv("VDO_PCG_LOOSE")) loose_tol = std::atof(e);
  if (const char* e = std::getenv("VDO_PCG_SWITCH")) switch_gain = std::atof(e);
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
