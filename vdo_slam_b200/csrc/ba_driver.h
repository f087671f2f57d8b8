// ba_driver.h -- host side of the batch factor-graph optimiser: graph ingestion (the analogue of
// g2o::SparseOptimizer::initializeOptimization + BlockSolver::buildStructure) and the Levenberg-Marquardt loop
// (g2o/core/optimization_algorithm_levenberg.cpp:61-164, sparse_optimizer.cpp:354-427) driving backend kernels.
#pragma once
#include <functional>
#include <string>
#include <vector>
#include "ba_types.h"
#include "../../include/vdo_b200.h"

namespace vdo {

// array in the backend's staging arena: plain memory, NOT zero-initialised, valid until the graph releases the arena
template <typename T> struct HostBuf {
  T* p = nullptr; size_t n = 0;
  T& operator[](size_t i) { return p[i]; }
  const T& operator[](size_t i) const { return p[i]; }
  T* data() { return p; }
  const T* data() const { return p; }
  size_t size() const { return n; }
  bool empty() const { return n == 0; }
  T* begin() { return p; }
  T* end() { return p + n; }
};

class BaGraph {
 public:
  explicit BaGraph(BaBackend* be) : be_(be) {}
  ~BaGraph();
  int set_vertices(int n_se3, const double* se3, int n_pt, const double* pt);
  int add_prior(int n, const int* v, const double* Z, const double* w);
  int add_se3(int n, const int* ij, const double* Z, const double* w, const double* delta);
  int add_obs(int n, const int* cp, const double* z, const double* w, const double* delta);
  int add_ter(int n, const int* pph, const double* w, const double* delta);
  int finalize();
  int optimize(const vdo_lm_options& opt, vdo_lm_stats* stats, double* chi2_history);
  // n finalized graphs of one backend in LM rounds: every graph makes the decisions optimize() makes alone; the device work of a
  // round is enqueued for all graphs before the one read-back of their scalars.  stats / chi2_history: n entries or NULL.
  static int optimize_batch(BaGraph* const* graphs, int n, const vdo_lm_options& opt, vdo_lm_stats* stats, double* const* chi2_history);
  bool finalized() const { return finalized_; }
  BaBackend* backend() const { return be_; }
  int get_vertices(double* se3, double* pt);
  int reset_vertices();
  int info(int64_t out[8]) const;
  int solver_info(int64_t out[8]) const;
  int debug_linearize(double* Hpp, double* bp, double* Hll, double* bl, double* chi2);
  int debug_apply(double lambda, const char* op, const double* in, double* out);
  int debug_solve(double lambda, double pcg_rel_tol, int pcg_max_iterations, double* xp, double* xl, double* r_rec, int* pcg_iters);
  // n finalized graphs of one backend (distinct, world 1, lambda[k] >= 0: the caller checks): one LM trial each as optimize_batch runs
  // it, then the pop.  Outputs per graph k (every array may be NULL, and so may any xp[k] / xl[k] / se3[k] / pt[k]).
  static int debug_trial(BaGraph* const* gs, int n, const double* lambda, const int* reortho, double pcg_rel_tol, int pcg_max_iterations,
                         double* const* xp, double* const* xl, double* const* se3, double* const* pt, double* chi2, double* scale,
                         int* pcg_iters, int* ok);
  int time_kernel(const char* name, int reps, float* ms_avg);
  const std::string& error() const { return err_; }

 private:
  template <typename T> T* dalloc(size_t n) { bytes_ += n * sizeof(T); T* p = (T*)be_->alloc(n * sizeof(T) + 16); owned_.push_back(p); return p; }   // +16: the tile kernels' bulk copies round ranges up to 16 B
  template <typename T> HostBuf<T> stage(size_t n) { hold_stage(); HostBuf<T> b; b.n = n; b.p = (T*)be_->staging().take(n * sizeof(T) + 16); return b; }
  template <typename T> HostBuf<T> stage_fill(size_t n, int byte) { HostBuf<T> b = stage<T>(n); fill_bytes(b.p, byte, n * sizeof(T)); return b; }
  template <typename T> void append(HostBuf<T>& b, const T* src, size_t n) {
    HostBuf<T> nb = stage<T>(b.n + n);
    if (b.n) copy_bytes(nb.p, b.p, b.n * sizeof(T));
    copy_bytes(nb.p + b.n, src, n * sizeof(T));
    b = nb;
  }
  template <typename T> T* upload(const HostBuf<T>& v) { T* p = dalloc<T>(v.size()); if (!v.empty()) be_->h2d_async(p, v.data(), v.size() * sizeof(T)); return p; }
  void hold_stage() { if (!holds_stage_) { be_->staging().acquire(); holds_stage_ = true; } }
  void drop_stage() { if (holds_stage_) { be_->staging().release(); holds_stage_ = false; } }
  static void copy_bytes(void* dst, const void* src, size_t bytes);   // threaded for large blocks
  static void fill_bytes(void* dst, int byte, size_t bytes);
  bool holds_stage_ = false;
  template <typename T> T* upload(const std::vector<T>& v) { T* p = dalloc<T>(v.size()); if (!v.empty()) be_->h2d(p, v.data(), v.size() * sizeof(T)); return p; }
  void zero_system();               // H_pp, b_p and the per-linearisation scalars
  void push();                      // estimates -> backup
  void pop();                       // backup -> estimates
  void read_se3_vec(const double* src, double* dst);   // device, 6 per vertex in path order -> caller's numbering; src NULL: zeros
  void read_pt_vec(const double* src, double* dst);    // device, 3 per own landmark in tracklet order -> caller's numbering
  bool next_oplus_reorthogonalizes();   // counts an oplus; true when this one re-orthogonalises the rotations
  struct LmState;
  // The rounds of the LM loop over the graphs gs[0..n) of one backend, between its batch_begin and batch_end.  Round: per graph its step
  // flags (BaBackend::BATCH_*), the lambda, re-orthogonalisation and squared PCG tolerance of its trial.
  struct Round;
  enum Stage { LINEARIZE, SETUP, BACKSUB, UPDATE };
  static void lin_round(BaGraph* const* gs, int n, Round& r);     // buildSystem; the largest diagonal entry for BATCH_MAXDIAG
  static void chi2_step(BaGraph* const* gs, int n, const Round& r, int len);   // robust chi2 of the BATCH_TRIAL graphs
  static void trial_round(BaGraph* const* gs, int n, Round& r, int pcg_max_iterations, Stage last, float* prof_ms, int* pcg_iters, int* ok);
  // this graph alone: linearisation, then its trial up to `last` (solver: BATCH_DENSE or BATCH_PCG); false if the solve broke down
  bool lone(Stage last, double lambda, int solver, double tol2, int pcg_max_iterations, int* pcg_iters);
  int fail(int code, const std::string& m) { err_ = m; return code; }
  // Stages of finalize(), in the order it runs them; what each produces is a struct defined in ba_driver.cpp.  lap: VDO_PROFILE timer.
  using Lap = std::function<void(const char*)>;
  struct Tracklets; struct EdgeClasses; struct LmStream; struct Ternary; struct TileLayout; struct Chunked; struct Se3Edges; struct Solvers;
  int order_tracklets(int NT, const Lap& lap, Tracklets& tk);
  int edge_classes(const HostBuf<double>& w, const HostBuf<double>& d, int NT, const char* family, EdgeClasses& out);
  LmStream landmark_stream(const Tracklets& tk, const HostBuf<uint8_t>& ecls, int NT, const Lap& lap);
  int ternary_edges(const Tracklets& tk, int NT, Ternary& ter);
  static Chunked chunked_streams(const LmStream& lm, const Ternary& ter, int C, int P);
  int tile_runs(const LmStream& lm, const Ternary& ter, int P, int NT, TileLayout& tl);
  Se3Edges se3_edges(const std::vector<int>& path_begin) const;
  void states(const Tracklets& tk, int NT, HostBuf<double>& se3, HostBuf<double>& pt);
  Solvers choose_solvers(bool allow_dense, bool allow_band, bool tiled, const Tracklets& tk, const LmStream& lm, int NT) const;
  void upload_layout(const std::vector<int>& path_begin, const Tracklets& tk, const LmStream& lm, const EdgeClasses& oc, const Ternary& ter,
                     const TileLayout& tl, const Chunked& ch, const Se3Edges& se, const HostBuf<double>& se3, const HostBuf<double>& pt,
                     const Solvers& sv);

  BaBackend* be_;
  BaDev d_;
  std::vector<void*> owned_;
  size_t bytes_ = 0;
  bool finalized_ = false;
  std::string err_;
  long oplus_calls_ = 0;
  double last_lambda_ = 1.0;
  double cur_pcg_tol_ = 0.0;        // tolerance of the current LM iteration's solves (forcing schedule), 0 = opt.pcg_rel_tol
  // host staging (until finalize)
  int n_se3_ = 0, n_pt_ = 0, P_all_ = 0;
  HostBuf<double> h_se3_, h_pt_;
  std::vector<int> pr_v_; std::vector<double> pr_Z_, pr_w_;
  std::vector<int> se_ij_; std::vector<double> se_Z_, se_w_, se_d_;
  HostBuf<int> ob_cp_; HostBuf<double> ob_z_, ob_w_, ob_d_;
  HostBuf<int> te_pph_; HostBuf<double> te_w_, te_d_;
  int n_prior_ = 0;
  std::vector<int> new_of_old_;     // landmark renumbering
  std::vector<int> new_se3_of_old_; // se3 renumbering (path order)
};

}  // namespace vdo
