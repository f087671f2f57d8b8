// vdo_capi.cpp -- extern "C" boundary of libvdo_b200.so (declarations and reference citations: include/vdo_b200.h).
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "../../include/vdo_b200.h"
#include "ba_driver.h"

struct vdo_ctx {
  vdo::BaBackend* be = nullptr;
  std::string err;
};
struct vdo_graph {
  vdo_ctx* ctx;
  vdo::BaGraph* g;
};

namespace vdo {
BaBackend* ctx_backend(vdo_ctx* c) { return c ? c->be : nullptr; }
void ctx_set_error(vdo_ctx* c, const std::string& msg) { if (c) c->err = msg; }   // for calls that only hold a frame (frame_kernels.cu)
}

extern "C" {

int vdo_ctx_create(int device, vdo_ctx** out) {
  if (!out) return VDO_ERR_ARG;
  *out = nullptr;
  vdo_ctx* c = new (std::nothrow) vdo_ctx;
  if (!c) return VDO_ERR_ARG;
  char msg[512] = {0};
  c->be = vdo::make_backend(device, msg, sizeof msg);
  if (!c->be) {
    // no CPU fallback: the caller gets an error, and the message through a static buffer
    static thread_local std::string last;
    last = msg;
    delete c;
    std::fprintf(stderr, "[vdo_b200] vdo_ctx_create failed: %s\n", last.c_str());
    return VDO_ERR_CUDA;
  }
  *out = c;
  return VDO_OK;
}
void vdo_ctx_destroy(vdo_ctx* ctx) {
  if (!ctx) return;
  delete ctx->be;
  delete ctx;
}
const char* vdo_last_error(const vdo_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
uint64_t vdo_ctx_stream(const vdo_ctx* ctx) { return ctx ? (uint64_t)(uintptr_t)ctx->be->stream() : 0; }

int vdo_graph_create(vdo_ctx* ctx, vdo_graph** out) {
  if (!ctx || !out) return VDO_ERR_ARG;
  vdo_graph* g = new vdo_graph{ctx, new vdo::BaGraph(ctx->be)};
  *out = g;
  return VDO_OK;
}
void vdo_graph_destroy(vdo_graph* g) {
  if (!g) return;
  delete g->g;
  delete g;
}
#define VDO_FWD(call)                    \
  if (!g) return VDO_ERR_ARG;            \
  int rc_ = g->g->call;                  \
  if (rc_ != VDO_OK) g->ctx->err = g->g->error(); \
  return rc_;

int vdo_graph_set_vertices(vdo_graph* g, int n_se3, const double* se3, int n_pt, const double* pt) { VDO_FWD(set_vertices(n_se3, se3, n_pt, pt)) }
int vdo_graph_add_edges_se3_prior(vdo_graph* g, int n, const int* v, const double* Z, const double* w) { VDO_FWD(add_prior(n, v, Z, w)) }
int vdo_graph_add_edges_se3(vdo_graph* g, int n, const int* ij, const double* Z, const double* w, const double* delta) { VDO_FWD(add_se3(n, ij, Z, w, delta)) }
int vdo_graph_add_edges_se3_pointxyz(vdo_graph* g, int n, const int* cp, const double* z, const double* w, const double* delta) { VDO_FWD(add_obs(n, cp, z, w, delta)) }
int vdo_graph_add_edges_landmark_motion(vdo_graph* g, int n, const int* pph, const double* w, const double* delta) { VDO_FWD(add_ter(n, pph, w, delta)) }
int vdo_graph_finalize(vdo_graph* g) { VDO_FWD(finalize()) }

int vdo_abi_struct_size(const char* name) {
  if (!name) return -1;
  const std::string s(name);
  if (s == "vdo_lm_options") return (int)sizeof(vdo_lm_options);
  if (s == "vdo_lm_stats") return (int)sizeof(vdo_lm_stats);
  if (s == "vdo_tracker_params") return (int)sizeof(vdo_tracker_params);
  if (s == "vdo_dev_plane") return (int)sizeof(vdo_dev_plane);
  if (s == "vdo_orb_batch_out") return (int)sizeof(vdo_orb_batch_out);
  if (s == "vdo_orb_desc_set") return (int)sizeof(vdo_orb_desc_set);
  if (s == "vdo_orb_match_opts") return (int)sizeof(vdo_orb_match_opts);
  if (s == "vdo_orb_match_out") return (int)sizeof(vdo_orb_match_out);
  if (s == "vdo_pnp_match_opts") return (int)sizeof(vdo_pnp_match_opts);
  if (s == "vdo_pnp_out") return (int)sizeof(vdo_pnp_out);
  if (s == "vdo_pose_refine_opts") return (int)sizeof(vdo_pose_refine_opts);
  if (s == "vdo_pose_refine_out") return (int)sizeof(vdo_pose_refine_out);
  if (s == "vdo_obj_motion_opts") return (int)sizeof(vdo_obj_motion_opts);
  if (s == "vdo_obj_motion_out") return (int)sizeof(vdo_obj_motion_out);
  if (s == "vdo_obj_track_opts") return (int)sizeof(vdo_obj_track_opts);
  if (s == "vdo_obj_track_out") return (int)sizeof(vdo_obj_track_out);
  if (s == "vdo_obj_mask_out") return (int)sizeof(vdo_obj_mask_out);
  if (s == "vdo_obj_feat_set") return (int)sizeof(vdo_obj_feat_set);
  if (s == "vdo_stat_feat_set") return (int)sizeof(vdo_stat_feat_set);
  if (s == "vdo_stat_opts") return (int)sizeof(vdo_stat_opts);
  if (s == "vdo_cam_track_opts") return (int)sizeof(vdo_cam_track_opts);
  if (s == "vdo_cam_track_out") return (int)sizeof(vdo_cam_track_out);
  return -1;
}

void vdo_lm_options_default(vdo_lm_options* o) {
  if (!o) return;
  std::memset(o, 0, sizeof *o);
  o->max_iterations = 300; o->gain_threshold = 1e-4; o->max_trials = 10;
  o->pcg_rel_tol = 1e-6; o->pcg_max_iterations = 2000; o->verbose = 0; o->force_all_iterations = 0; o->pcg_loose_tol = 0.0; o->pcg_switch_gain = 0.0;
}
int vdo_graph_optimize(vdo_graph* g, const vdo_lm_options* opt, vdo_lm_stats* stats, double* chi2_history) {
  vdo_lm_options o;
  if (opt) o = *opt; else vdo_lm_options_default(&o);
  VDO_FWD(optimize(o, stats, chi2_history))
}
}  // extern "C"
namespace {
// the graphs of a batch call: n >= 1 distinct, non-NULL, finalized graphs of one context on one GPU
int batch_graphs(vdo_graph* const* graphs, int n, const char* what, std::vector<vdo::BaGraph*>& gs) {
  if (!graphs || n < 1 || !graphs[0]) return VDO_ERR_ARG;
  vdo_ctx* ctx = graphs[0]->ctx;
  const std::string w(what);
  gs.resize(n);
  for (int i = 0; i < n; ++i) {
    if (!graphs[i]) { ctx->err = w + ": graph " + std::to_string(i) + " is NULL"; return VDO_ERR_ARG; }
    if (graphs[i]->ctx != ctx) { ctx->err = w + ": graph " + std::to_string(i) + " belongs to another context"; return VDO_ERR_ARG; }
    for (int j = 0; j < i; ++j)
      if (graphs[j] == graphs[i]) { ctx->err = w + ": graph " + std::to_string(i) + " repeats graph " + std::to_string(j); return VDO_ERR_ARG; }
    gs[i] = graphs[i]->g;
  }
  for (int i = 0; i < n; ++i)
    if (!gs[i]->finalized()) { ctx->err = w + ": graph " + std::to_string(i) + " is not finalized"; return VDO_ERR_STATE; }
  if (ctx->be->world > 1) { ctx->err = w + ": sharded graphs (world > 1) are not supported"; return VDO_ERR_UNSUPPORTED; }
  return VDO_OK;
}
}  // namespace
extern "C" {

int vdo_graph_optimize_batch(vdo_graph* const* graphs, int n, const vdo_lm_options* opt, vdo_lm_stats* stats, double* const* chi2_history) {
  std::vector<vdo::BaGraph*> gs;
  if (const int rc = batch_graphs(graphs, n, "vdo_graph_optimize_batch", gs)) return rc;
  vdo_ctx* ctx = graphs[0]->ctx;
  vdo_lm_options o;
  if (opt) o = *opt; else vdo_lm_options_default(&o);
  const int rc = vdo::BaGraph::optimize_batch(gs.data(), n, o, stats, chi2_history);
  if (rc != VDO_OK) for (int i = 0; i < n; ++i) if (!gs[i]->error().empty()) { ctx->err = gs[i]->error(); break; }
  return rc;
}
int vdo_graph_get_vertices(const vdo_graph* g, double* se3, double* pt) { VDO_FWD(get_vertices(se3, pt)) }
int vdo_graph_reset_vertices(vdo_graph* g) { VDO_FWD(reset_vertices()) }
int vdo_graph_info(const vdo_graph* g, int64_t out[8]) { VDO_FWD(info(out)) }
int vdo_graph_solver_info(const vdo_graph* g, int64_t out[8]) { VDO_FWD(solver_info(out)) }
int vdo_graph_debug_linearize(vdo_graph* g, double* Hpp, double* bp, double* Hll, double* bl, double* chi2) { VDO_FWD(debug_linearize(Hpp, bp, Hll, bl, chi2)) }
int vdo_graph_debug_apply(vdo_graph* g, double lambda, const char* op, const double* in, double* out) { VDO_FWD(debug_apply(lambda, op, in, out)) }
int vdo_graph_debug_solve(vdo_graph* g, double lambda, double pcg_rel_tol, int pcg_max_iterations, double* xp, double* xl, double* r_rec, int* pcg_iters) {
  VDO_FWD(debug_solve(lambda, pcg_rel_tol, pcg_max_iterations, xp, xl, r_rec, pcg_iters))
}
int vdo_graph_debug_trial(vdo_graph* const* graphs, int n, const double* lambda, const int* reortho, double pcg_rel_tol, int pcg_max_iterations,
                          double* const* xp, double* const* xl, double* const* se3, double* const* pt, double* chi2, double* scale,
                          int* pcg_iters, int* ok) {
  std::vector<vdo::BaGraph*> gs;
  if (const int rc = batch_graphs(graphs, n, "vdo_graph_debug_trial", gs)) return rc;
  vdo_ctx* ctx = graphs[0]->ctx;
  if (!lambda) { ctx->err = "vdo_graph_debug_trial: lambda is NULL"; return VDO_ERR_ARG; }
  for (int i = 0; i < n; ++i)
    if (!(lambda[i] >= 0)) { ctx->err = "vdo_graph_debug_trial: lambda of graph " + std::to_string(i) + " is negative or NaN"; return VDO_ERR_ARG; }
  return vdo::BaGraph::debug_trial(gs.data(), n, lambda, reortho, pcg_rel_tol, pcg_max_iterations, xp, xl, se3, pt, chi2, scale, pcg_iters, ok);
}

int vdo_graph_time_kernel(vdo_graph* g, const char* name, int reps, float* ms_avg) { VDO_FWD(time_kernel(name, reps, ms_avg)) }

}  // extern "C"
