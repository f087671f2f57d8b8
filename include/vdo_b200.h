/*
 * vdo_b200.h -- C ABI of the H100-native (sm_90a) VDO-SLAM hot path (libvdo_b200.so).
 *
 * The reference (halajun/VDO_SLAM) has no FFI layer: its hot path is plain C++ inside libObjSLAM.so.
 * Each entry point below names the reference interface it replaces (paths relative to the reference root;
 * g2o/ = dependencies/g2o/g2o/).  Host wrappers with the reference's own C++ signatures
 * (VDO_SLAM::Optimizer, ORBextractor, ...) sit above this ABI; see INTEGRATION.md.
 *
 * Conventions
 *   - plain pointers + sizes, caller-allocated outputs, int status return (0 = VDO_OK, <0 = error;
 *     vdo_last_error() gives the text).  No exceptions cross the boundary, nothing calls exit().
 *   - every pointer is a HOST pointer unless the parameter name ends in _dev.
 *   - an SE(3) value ("iso") is 12 doubles: rotation row-major (9) then translation (3) -- the memory
 *     image of g2o's Isometry3 estimate (g2o/types/vertex_se3.h:50) without Eigen's column-major packing.
 *   - there is NO CPU fallback: every compute entry point fails with VDO_ERR_CUDA when no sm_90 device
 *     is usable.
 */
#ifndef VDO_B200_H
#define VDO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VDO_OK 0
#define VDO_ERR_CUDA (-1)        /* CUDA runtime / no device */
#define VDO_ERR_ARG (-2)         /* bad argument */
#define VDO_ERR_UNSUPPORTED (-3) /* graph shape outside what the reference's optimisers build */
#define VDO_ERR_STATE (-4)       /* call order violated */
#define VDO_ERR_NCCL (-5)

typedef struct vdo_ctx vdo_ctx;     /* one per VDO_SLAM::System (src/System.cc:22-48): device, stream, arenas */
typedef struct vdo_graph vdo_graph; /* one per g2o::SparseOptimizer instance of the batch optimisers */

int vdo_ctx_create(int device, vdo_ctx **out);
void vdo_ctx_destroy(vdo_ctx *ctx);
const char *vdo_last_error(const vdo_ctx *ctx);
/* cudaStream_t of the context as an integer handle (so torch / callers can order work against it) */
uint64_t vdo_ctx_stream(const vdo_ctx *ctx);

/* Multi-GPU (one process per GPU).  The batch graph shards by tracklet: after vdo_ctx_init_comm, vdo_graph_finalize keeps
 * the tracklets of this rank only (round-robin), the se3 state is replicated, and partial se3-side sums are all-reduced
 * over NCCL (H_pp/b_p once per linearisation, the 6C-vector S*p once per PCG iteration, chi2/scale once per LM trial).
 * rank 0 calls vdo_nccl_unique_id and ships the 128 bytes to the other ranks (e.g. torch.distributed broadcast). */
int vdo_nccl_unique_id(char *out128);
int vdo_ctx_init_comm(vdo_ctx *ctx, int rank, int world, const char *id128);

/* ------------------------------------------------------------------------------------------------
 * Batch factor-graph optimisation.  Replaces the g2o::SparseOptimizer + OptimizationAlgorithmLevenberg +
 * BlockSolverX + LinearSolverCSparse stack as driven by Optimizer::FullBatchOptimization
 * (src/Optimizer.cc:1232-2175) and Optimizer::PartialBatchOptimization (src/Optimizer.cc:42-1230).
 * ------------------------------------------------------------------------------------------------ */

/* new g2o::SparseOptimizer (src/Optimizer.cc:1312-1323, :172-183) */
int vdo_graph_create(vdo_ctx *ctx, vdo_graph **out);
void vdo_graph_destroy(vdo_graph *g);

/* optimizer.addVertex(VertexSE3 / VertexPointXYZ) with setEstimate (src/Optimizer.cc:1359-1363, 1412-1416,
 * 1571-1582).  se3: n_se3 x 12 iso (camera poses and object motions share one index space), pt: n_pt x 3. */
int vdo_graph_set_vertices(vdo_graph *g, int n_se3, const double *se3, int n_pt, const double *pt);

/* EdgeSE3Prior, identity offset parameter, information = w * I6, no kernel (src/Optimizer.cc:1364-1373;
 * g2o/types/edge_se3_prior.cpp:89-102).  v: n se3 indices, Z: n x 12 iso, w: n */
int vdo_graph_add_edges_se3_prior(vdo_graph *g, int n, const int *v, const double *Z, const double *w);

/* EdgeSE3 (odometry and motion-smoothness edges; src/Optimizer.cc:1383-1399, 1596-1623;
 * g2o/types/edge_se3.cpp:77-104).  ij: n x 2 se3 indices, Z: n x 12, information = w * I6,
 * Huber delta (<= 0: no robust kernel). */
int vdo_graph_add_edges_se3(vdo_graph *g, int n, const int *ij, const double *Z, const double *w, const double *delta);

/* EdgeSE3PointXYZ, identity offset (src/Optimizer.cc:1421-1435; g2o/types/edge_se3_pointxyz.cpp:99-140).
 * cp: n x 2 (se3 index, point index), z: n x 3 measured point in the camera frame, information = w * I3 */
int vdo_graph_add_edges_se3_pointxyz(vdo_graph *g, int n, const int *cp, const double *z, const double *w, const double *delta);

/* LandmarkMotionTernaryEdge, measurement 0 (src/Optimizer.cc:1724-1741; g2o/types/types_dyn_slam3d.cpp:53-85).
 * pph: n x 3 (point p1, point p2, motion se3 index), information = w * I3 */
int vdo_graph_add_edges_landmark_motion(vdo_graph *g, int n, const int *pph, const double *w, const double *delta);

/* optimizer.initializeOptimization() + BlockSolver::buildStructure (src/Optimizer.cc:1768;
 * g2o/core/block_solver.hpp:142-295): orders landmarks by tracklet, builds the edge streams, uploads to HBM. */
int vdo_graph_finalize(vdo_graph *g);

typedef struct vdo_lm_options {
  int max_iterations;       /* optimizer.optimize(N): 300 full batch, 100 partial (src/Optimizer.cc:1935, :807) */
  double gain_threshold;    /* SparseOptimizerTerminateAction::setGainThreshold; <= 0: action not installed */
  int max_trials;           /* maxTrialsAfterFailure, g2o default 10 */
  double pcg_rel_tol;       /* reduced-camera PCG: stop when sqrt(r.M^-1 r) <= tol * initial.  Default 1e-6: on BASELINE config 5 the LM run then
                               has the oracle's iteration count and ends within 9e-7 (poses) / 1.2e-6 m (points) of its direct-solve result (the
                               required agreement is 1e-4) */
  int pcg_max_iterations;   /* default 2000 */
  int verbose;              /* per-iteration line on stderr, like optimizer.setVerbose(true) */
  int force_all_iterations; /* benchmarking: ignore every stop rule and run exactly max_iterations */
  double pcg_loose_tol;     /* forcing schedule of the inexact linear solves: while the previous LM iteration reduced chi2 by more than */
  double pcg_switch_gain;   /* pcg_switch_gain (relative), solve to pcg_loose_tol instead of pcg_rel_tol.  0 / 0: off (default) */
} vdo_lm_options;

typedef struct vdo_lm_stats {
  int iterations;           /* return value of SparseOptimizer::optimize */
  int trials;               /* total LM trials (linear solves) */
  int pcg_iterations;       /* total PCG iterations over all solves */
  double initial_chi2, final_chi2, final_lambda;
  double ms_linearize, ms_solve, ms_total; /* CUDA-event times on the context stream */
  int kernel_launches;      /* kernels launched by this optimize() call */
} vdo_lm_stats;

/* Converter (src/Converter.cc:25-41, 151-166) and the cv::Mat 4x4 product as the reference's float / double rounding rules (host-only):
 * toSE3Quat (rotation -> Eigen quaternion, w >= 0, normalised; q = x y z w), toCvMat (quaternion -> rotation, rounded to float),
 * toInvMatrix ([R^T | -R^T t], the translation accumulated in double and rounded once), A * B of two 4x4 CV_32F (float accumulation). */
int vdo_convert_to_se3quat(const float *T16, double *q4, double *t3);
int vdo_convert_to_cvmat(const double *q4, const double *t3, float *T16);
int vdo_convert_inv_matrix(const float *T16, float *out16);
int vdo_convert_mul4(const float *A16, const float *B16, float *out16);

/* sizeof() of a public struct as this library was built ("vdo_lm_options", "vdo_lm_stats", "vdo_tracker_params", "vdo_dev_plane",
 * "vdo_orb_batch_out", "vdo_orb_desc_set", "vdo_orb_match_opts", "vdo_orb_match_out", "vdo_pnp_match_opts", "vdo_pnp_out",
 * "vdo_pose_refine_opts", "vdo_pose_refine_out", "vdo_obj_motion_opts", "vdo_obj_motion_out", "vdo_obj_track_opts",
 * "vdo_obj_track_out", "vdo_obj_mask_out"; -1: unknown name): FFI
 * bindings that mirror the structs by hand (ctypes, cgo, JNI) check it at load time -- a binding that lags a struct extension would
 * otherwise have the library write past its buffer. */
int vdo_abi_struct_size(const char *name);

void vdo_lm_options_default(vdo_lm_options *o);

/* optimizer.optimize(max_iterations) (g2o/core/sparse_optimizer.cpp:354-427 with
 * OptimizationAlgorithmLevenberg::solve, g2o/core/optimization_algorithm_levenberg.cpp:61-164).
 * chi2_history (may be NULL): max_iterations+1 doubles, [0] = initial robust chi2. */
int vdo_graph_optimize(vdo_graph *g, const vdo_lm_options *opt, vdo_lm_stats *stats, double *chi2_history);

/* n finalized graphs of one context, optimised together.  Graph i ends exactly where vdo_graph_optimize(graphs[i], opt, ...) takes it:
 * the same LM decisions (lambda schedule, accepted / rejected trials, stop rules) on the same arithmetic per graph.  Graphs on the dense
 * reduced-system path (vdo_graph_solver_info out[5] == 1) share every device step: one set of launches and one host synchronise per step
 * for all of them.  So do the PCG-path graphs of the tiled layout (out[0] == 1, out[5] == 0) when there are at least two: their
 * linearisation, preconditioner, right-hand side, PCG iterations (chunks of 8 for every graph not yet converged, one read-back of all
 * their scalars per chunk), back-substitution and update run as one set of launches per step.  A graph alone of its kind, and graphs of
 * the chunked layout, run their steps one graph at a time inside the same rounds.  stats / chi2_history: n entries each (either
 * may be NULL, and any chi2_history[i] may be NULL); ms_* and kernel_launches of every entry describe the whole call.
 * VDO_ERR_ARG: n < 1, a NULL or repeated graph, graphs on different contexts.  VDO_ERR_STATE: a graph not finalized.
 * VDO_ERR_UNSUPPORTED: a sharded context (world > 1).  Every refusal happens before any device work and changes no graph. */
int vdo_graph_optimize_batch(vdo_graph *const *graphs, int n, const vdo_lm_options *opt, vdo_lm_stats *stats, double *const *chi2_history);

/* vertex->getEstimateData() (src/Optimizer.cc:2094-2172) */
int vdo_graph_get_vertices(const vdo_graph *g, double *se3, double *pt);
/* restore the estimates given to vdo_graph_set_vertices (device-to-device; used to repeat a solve) */
int vdo_graph_reset_vertices(vdo_graph *g);

/* sizes after finalize: out[0]=n_se3 out[1]=n_pt out[2]=n_pointxyz_edges out[3]=n_motion_edges out[4]=n_se3_edges
 * out[5]=n_prior out[6]=n_tracklets out[7]=device bytes held */
int vdo_graph_info(const vdo_graph *g, int64_t out[8]);
/* which solver paths the finalized graph uses: out[0]=tiled layout (0/1) out[1]=tiles out[2]=static tiles out[3]=width of the explicit
 * banded static block of the reduced matrix (0: matrix-free static product) out[4]=rows of that band out[5]=dense reduced-matrix path (0/1)
 * out[6]=preconditioner sharded by se3 path over the ranks (0/1) out[7]=se3 paths */
int vdo_graph_solver_info(const vdo_graph *g, int64_t out[8]);

/* Test hooks: one linearisation at the current estimates, returned in the caller's vertex numbering.
 * Hpp_diag: n_se3 x 36 (row-major 6x6 diagonal blocks), bp: n_se3 x 6, Hll_diag: n_pt (scalar: the 3x3
 * diagonal blocks are that scalar times I3 for scalar information), bl: n_pt x 3, chi2: robust chi2. */
int vdo_graph_debug_linearize(vdo_graph *g, double *Hpp_diag, double *bp, double *Hll_diag, double *bl, double *chi2);
/* Test hook: linearises at the current estimates, factors the landmark blocks and builds the preconditioner for lambda (added to every
 * diagonal entry of H), then applies one operator of the reduced system.  Vectors are in the caller's vertex numbering and the local
 * tangent coordinates of the update (6 per se3 vertex, 3 per point).  op:
 *   "S"       out = S(lambda) in, S = H_pp + lambda I - H_pl (H_ll + lambda I)^-1 H_lp, by the product the PCG iterates with
 *   "Minv"    out = M(lambda)^-1 in, the PCG preconditioner (block-tridiagonal along the paths of the se3-se3 edge graph)
 *   "rhs"     out = b_p - H_pl (H_ll + lambda I)^-1 b_l (in is ignored and may be NULL)
 *   "backsub" in = x_p (n_se3 x 6), out = x_l = (H_ll + lambda I)^-1 (b_l - H_lp x_p) (n_pt x 3)
 * The estimates are not changed.  Sharded graphs (world > 1) are refused with VDO_ERR_STATE. */
int vdo_graph_debug_apply(vdo_graph *g, double lambda, const char *op, const double *in, double *out);
/* Test hook: one linearisation and one linear solve (H + lambda I) x = b as an LM trial runs it (dense reduced matrix or PCG, including
 * the captured PCG iteration), without applying the update.  xp: n_se3 x 6, xl: n_pt x 3, r_rec: n_se3 x 6 recurrence residual of the
 * PCG (zeros on the dense path), pcg_iters: PCG iterations (0 on the dense path).  Any output may be NULL.  pcg_rel_tol <= 0 and
 * pcg_max_iterations <= 0 select the defaults of vdo_lm_options_default.  Returns VDO_ERR_UNSUPPORTED when the solve broke down. */
int vdo_graph_debug_solve(vdo_graph *g, double lambda, double pcg_rel_tol, int pcg_max_iterations, double *xp, double *xl, double *r_rec,
                          int *pcg_iters);
/* Test hook: one LM trial of each of n graphs of one context, as vdo_graph_optimize_batch runs it -- the graphs share launches exactly as
 * they do there (n = 1: the lone graph's launches) -- at the damping lambda[k] >= 0 of graph k, with the rotations re-orthogonalised after
 * the update when reortho[k] != 0 (reortho NULL: never).  The trial linearises at the current estimates, solves (dense reduced matrix or
 * PCG to pcg_rel_tol), back-substitutes, updates and evaluates the robust chi2 at the new estimates; then every graph's estimates are
 * restored, so a later vdo_graph_optimize runs as if this call had not been made.  Outputs of graph k, in the caller's vertex numbering:
 * xp[k]: n_se3 x 6 and xl[k]: n_pt x 3, the step; se3[k]: n_se3 x 12 and pt[k]: n_pt x 3, the updated estimates; chi2[k]: robust chi2
 * at them; scale[k]: sum x (lambda x + b) over the step; pcg_iters[k]: PCG iterations (0 on the dense path); ok[k]: 0 when the solve
 * broke down.  Every output array, and any entry of xp / xl / se3 / pt, may be NULL.  pcg_rel_tol <= 0 and pcg_max_iterations <= 0
 * select the defaults of vdo_lm_options_default.  Refuses what vdo_graph_optimize_batch refuses, and a lambda < 0 or NaN (VDO_ERR_ARG). */
int vdo_graph_debug_trial(vdo_graph *const *graphs, int n, const double *lambda, const int *reortho, double pcg_rel_tol, int pcg_max_iterations,
                          double *const *xp, double *const *xl, double *const *se3, double *const *pt, double *chi2, double *scale,
                          int *pcg_iters, int *ok);

/* ------------------------------------------------------------------------------------------------
 * .g2o files: the on-disk format of the graphs the reference dumps around every batch optimisation
 * (optimizer.save(...), src/Optimizer.cc:806,808,1934,1936 -> g2o/core/optimizable_graph.cpp:589-622, element syntax in
 * g2o/types/{vertex_se3,vertex_pointxyz,edge_se3,edge_se3_prior,edge_se3_pointxyz,types_dyn_slam3d,parameter_se3_offset}.cpp,
 * tags in g2o/types/types_slam3d.cpp:37-57).  Host-only.  Edge arrays use compact vertex indices (position of the vertex in
 * the file), the *_id arrays keep the file ids; information matrices are returned as written (upper triangle: 21 / 6
 * values).  Robust kernels are not part of the format, so vdo_graph_from_g2o takes the Huber deltas as arguments. */
typedef struct vdo_g2o vdo_g2o;
int vdo_g2o_read(const char *path, vdo_g2o **out);   /* on a parse error *out still carries the message (vdo_g2o_error) */
void vdo_g2o_free(vdo_g2o *g);
const char *vdo_g2o_error(const vdo_g2o *g);
/* out: n_se3, n_pt, n_prior, n_se3_edges, n_pointxyz_edges, n_motion_edges, n_fixed, n_offset_params */
int vdo_g2o_counts(const vdo_g2o *g, int64_t out[8]);
/* int arrays: se3_id pt_id fixed_id prior_v se3e_ij obs_cp ter_pph ; double arrays: se3 pt prior_Z prior_info se3e_Z
 * se3e_info obs_z obs_info ter_meas ter_info offset */
int vdo_g2o_get_i32(const vdo_g2o *g, const char *name, int *dst, int64_t cap);
int vdo_g2o_get_f64(const vdo_g2o *g, const char *name, double *dst, int64_t cap);
/* parsed file -> finalised graph; VDO_ERR_UNSUPPORTED unless every information matrix is w*I, motion measurements are
 * zero and the sensor offset is the identity, i.e. the family src/Optimizer.cc constructs */
int vdo_graph_from_g2o(vdo_ctx *ctx, const vdo_g2o *file, double delta_se3, double delta_pointxyz, double delta_motion, vdo_graph **out);
/* arrays in the layout of vdo_graph_add_* -> file; ids NULL: se3 vertex i -> i, point j -> n_se3 + j; precision <= 0: 17 digits */
int vdo_g2o_write(const char *path, int n_se3, const double *se3, const int *se3_id, int n_pt, const double *pt, const int *pt_id, int n_fixed,
                  const int *fixed_id, int n_prior, const int *prior_v, const double *prior_Z, const double *prior_w, int n_se3e, const int *se3e_ij,
                  const double *se3e_Z, const double *se3e_w, int n_obs, const int *obs_cp, const double *obs_z, const double *obs_w, int n_ter,
                  const int *ter_pph, const double *ter_w, int precision);

/* ------------------------------------------------------------------------------------------------
 * Per-frame input files of the reference's driver (example/vdo_slam.cc:98-141): PNG image / 16-bit disparity
 * (cv::imread UNCHANGED, :105-110), Middlebury .flo (cv::optflow::readOpticalFlow, :117), text label mask (LoadMask,
 * :253-450).  Host-only decoders; colour pixels in OpenCV order (BGR / BGRA), 16-bit samples host-endian. */
int vdo_io_png_info(const char *path, int *w, int *h, int *channels, int *bit_depth);
int vdo_io_read_png(const char *path, void *dst, size_t dst_bytes);            /* h x w x channels, uint8 or uint16 */
int vdo_io_read_png_gray_f32(const char *path, float *dst, int w, int h);      /* == imD.convertTo(imD_f, CV_32F) */
int vdo_io_flo_info(const char *path, int *w, int *h);
int vdo_io_read_flo(const char *path, float *dst, size_t dst_floats);          /* h x w x 2 (u, v) = CV_32FC2 */
int vdo_io_read_mask_txt(const char *path, int32_t *dst, int w, int h);        /* CV_32SC1, zeros where the file has zeros */

/* ------------------------------------------------------------------------------------------------
 * Result files and error metrics (the step after the path): System::SaveResults (src/System.cc:66-244) and
 * Tracking::GetMetricError (src/Tracking.cc:3243-3386), in the reference's float arithmetic and text format
 * (fixed, 9 decimals).  Per-frame entry lists are flattened: n_per_frame[i] entries for frame i (entry 0 = the camera,
 * skipped by both functions like the reference's `for j = 1`), labels / matrices of all frames back to back.  Host-only. */
int vdo_results_write_poses(const char *path, int start_frame, int n, const float *T16);   /* initial_/refined_stereo_new.txt, cam_pose_gt_stereo.txt */
/* obj_mot_stereo[_rf]_new.txt: body-frame motion toInvMatrix(pose_pre) * H * pose_pre ; pose_pre16 == NULL: as stored (obj_mot_gt.txt) */
int vdo_results_write_object_motions(const char *path, int start_frame, int n_frames, const int *n_per_frame, const int *labels, const float *H16,
                                     const float *pose_pre16);
int vdo_results_write_object_centres(const char *path, int start_frame, int n_frames, const int *n_per_frame, const int *labels, const float *centre3);
/* out4 = {camera t, camera R [deg], objects t, objects R [deg]} (means); each_obj_* have max_id - 1 entries (may be NULL) */
int vdo_metric_error(int n_cam, const float *cam16, const float *cam_gt16, int n_frames, const int *n_per_frame, const int *labels,
                     const unsigned char *obj_stat, const float *H16, const float *pose_pre16, const float *H_gt16, int max_id, float out4[4],
                     float *each_obj_t, float *each_obj_r, int *each_obj_count);

/* ------------------------------------------------------------------------------------------------
 * Per-frame joint optical-flow / SE(3) refinement.  Replaces Optimizer::PoseOptimizationFlow2 (object motion,
 * src/Optimizer.cc:2755-2972: prior information 0.5*I2, optimize(200)) and Optimizer::PoseOptimizationFlow2Cam (camera
 * pose, src/Optimizer.cc:2333-2542: prior 0.3*I2, optimize(100)), i.e. the g2o graph of one VertexSE3Expmap + n
 * VertexSBAFlow with EdgeSE3ProjectFlow2 (information 0.1*I2, Huber sqrt(0.04)) and EdgeFlowPrior edges, solved by
 * OptimizationAlgorithmLevenberg over BlockSolver_6_3 + LinearSolverDense.  The whole LM solve runs in one kernel.
 *
 *   mode       0 = camera (Flow2Cam), 1 = object (Flow2)
 *   quirk      1 = reproduce the arithmetic of 2-D flow vertices inside BlockSolver_6_3's 3x3 blocks (SURVEY.md H1;
 *              derived from source reading, the reference binary cannot be built here), 0 = intended 2x2 arithmetic
 *   pts        n x 2 f32  pixel of each point in the LAST frame   (pLastFrame->mvObjKeys / mvStatKeys[...].pt)
 *   depth      n     f32  its depth                               (mvObjDepth / mvStatDepth)
 *   flow       n x 2 f32  measured optical flow                   (mvObjFlowNext / mvFlowNext)
 *   K          4     f32  fx, fy, cx, cy                          (Frame::fx ...)
 *   Tcw_last   4x4   f32  row-major, pLastFrame->mTcw             (Twl is formed from it as the reference does, in float)
 *   T_init     4x4   f32  row-major, pCurFrame->mInitModel / mTcw
 * outputs
 *   T_out      4x4   f32  Converter::toCvMat(vSE3->estimate())
 *   flow_out   n x 2 f64  refined flow of every point (the caller adds it to the last-frame pixel for inliers)
 *   inlier     n     u8   1 if chi2 <= 0.04 (vIsOutlier[i] == false)
 *   stats      8     f64  [0] LM iterations (-1: n < 3, nothing optimised, T_out = identity) [1] trials [2] robust chi2
 *                         [3] lambda [4] inlier count
 * The batch form runs nprob independent problems (all objects of a frame): offset has nprob+1 entries into the concatenated
 * pts / depth / flow / flow_out / inlier arrays; K, Tcw_last, T_init, T_out, stats are per problem.  Each problem runs on the
 * kernel its own size selects (n <= VDO_FLOW2_CLUSTER_MAX_N: a cluster with the points in shared memory, else one CTA), at most
 * two launches per call, so a problem's outputs do not depend on which other problems share its batch, bit for bit.
 * VDO_ERR_ARG before any device work: nprob < 1, offset[0] != 0 or a decreasing offset, a mode outside {0, 1}, a NULL
 * per-problem array, or NULL point arrays when the total point count is above 0. */
#define VDO_FLOW2_CLUSTER_MAX_N 11376   /* 8 CTAs x 1422 points x 18 doubles = 204 768 of the 204 800 bytes of opted-in smem */
int vdo_pose_opt_flow2(vdo_ctx *ctx, int mode, int quirk, int n, const float *pts, const float *depth, const float *flow,
                       const float *K, const float *Tcw_last, const float *T_init, float *T_out, double *flow_out,
                       unsigned char *inlier, double *stats);
int vdo_pose_opt_flow2_batch(vdo_ctx *ctx, int quirk, int nprob, const int *mode, const int *offset, const float *pts,
                             const float *depth, const float *flow, const float *K, const float *Tcw_last,
                             const float *T_init, float *T_out, double *flow_out, unsigned char *inlier, double *stats);
/* The batch call with an LM trace (a test hook): trace holds nprob x VDO_FLOW2_TRACE_DOUBLES doubles, zeroed and then written by
 * thread 0 of the problem's first CTA.  Layout of one problem's trace (offsets in doubles):
 *   HPP   36  H_pp of the first linearisation (row-major)        BP  6  b_p of the first linearisation
 *   S     36  Schur matrix of the first trial, lambda on its diagonal, every entry as formed (the solve reads the lower triangle)
 *   G      6  its right-hand side                                 X   6  the pose increment applied by the first trial
 *   STOP      why the LM stopped (VDO_FLOW2_STOP_*)               NREC   number of trial records
 *   REC       NREC records of VDO_FLOW2_TRACE_RECLEN doubles, one per lambda trial:
 *             [0] iteration [1] lambda of the trial [2] ok2 (1: the 6x6 solve succeeded) [3] trial chi2 [4] chi2 before the trial
 *             [5] scale (predicted decrease) [6] rho [7] accepted [8..14) the pose increment applied
 * vdo_pose_opt_flow2_batch is this call with trace = NULL; the kernels then do no trace work. */
#define VDO_FLOW2_TRACE_HPP 0
#define VDO_FLOW2_TRACE_BP 36
#define VDO_FLOW2_TRACE_S 42
#define VDO_FLOW2_TRACE_G 78
#define VDO_FLOW2_TRACE_X 84
#define VDO_FLOW2_TRACE_STOP 90
#define VDO_FLOW2_TRACE_NREC 91
#define VDO_FLOW2_TRACE_REC 96
#define VDO_FLOW2_TRACE_RECLEN 16
#define VDO_FLOW2_TRACE_MAXREC 2000     /* 200 iterations x 10 trials */
#define VDO_FLOW2_TRACE_DOUBLES (VDO_FLOW2_TRACE_REC + VDO_FLOW2_TRACE_RECLEN * VDO_FLOW2_TRACE_MAXREC)
#define VDO_FLOW2_STOP_FEW_POINTS 1     /* n < 3: nothing optimised */
#define VDO_FLOW2_STOP_TRIALS 2         /* ten trials of one iteration failed */
#define VDO_FLOW2_STOP_RHO_ZERO 3       /* rho == 0 */
#define VDO_FLOW2_STOP_NO_PROGRESS 4    /* three iterations in a row gained less than 1e-3 of chi2 */
#define VDO_FLOW2_STOP_CHI2_ROSE 5      /* the last trial's chi2 exceeded the previous iteration's */
#define VDO_FLOW2_STOP_MAX_ITERS 6      /* the iteration cap (100 camera, 200 object) */
int vdo_pose_opt_flow2_trace(vdo_ctx *ctx, int quirk, int nprob, const int *mode, const int *offset, const float *pts,
                             const float *depth, const float *flow, const float *K, const float *Tcw_last,
                             const float *T_init, float *T_out, double *flow_out, unsigned char *inlier, double *stats,
                             double *trace);
/* measurement: re-run the last uploaded batch `reps` times on the device (no host copies, the same kernel split as that call),
 * average ms per call; nprob must be that batch's size (VDO_ERR_STATE otherwise) */
int vdo_pose_opt_flow2_time(vdo_ctx *ctx, int quirk, int nprob, int reps, float *ms_avg);

/* ------------------------------------------------------------------------------------------------
 * Image side of the per-frame path.  A vdo_frame keeps one frame's images resident in HBM: gray (u8), depth (f32),
 * optical flow (f32 x2, interleaved like CV_32FC2) and semantic mask (i32), all row-major width x height with no padding.
 * ------------------------------------------------------------------------------------------------ */
typedef struct vdo_frame vdo_frame;
int vdo_frame_create(vdo_ctx *ctx, int width, int height, vdo_frame **out);
void vdo_frame_destroy(vdo_frame *f);
/* H2D of the images TrackRGBD receives (include/System.h:49-51); any pointer may be NULL to keep what is resident */
int vdo_frame_upload(vdo_frame *f, const unsigned char *gray, const float *depth, const float *flow, const int *mask);

/* A width x height plane in DEVICE memory, e.g. a torch CUDA tensor or a view of one.  Element (y, x, c) sits at
 * data_dev + y*stride_y + x*stride_x + c*stride_c elements of the dtype, so crops, HWC, CHW and other permuted views
 * need no copy.  Strides may take any value for inputs (0 broadcasts); write-back targets refuse a zero stride_x or
 * stride_y, because every pixel would land on the same element.  data_dev must be aligned to the element size. */
#define VDO_DT_U8 1
#define VDO_DT_F32 2
#define VDO_DT_I32 3
#define VDO_DT_I64 4
typedef struct vdo_dev_plane {
  const void *data_dev;                 /* device memory of the context's device */
  int dtype, channels;                  /* VDO_DT_*, 1 | 2 | 3 | 4 */
  int64_t stride_y, stride_x, stride_c; /* element strides */
  int rgb;                              /* 3/4-channel images: 1 = RGB(A) order (Camera.RGB: 1), 0 = BGR(A) */
} vdo_dev_plane;
/* Device form of vdo_frame_upload: one kernel reads the given planes at their strides into the resident buffers.
 *   image  u8, 1 channel (copied) or 3 / 4 channels (cvtColor RGB[A]/BGR[A]2GRAY in the 8-bit fixed point of OpenCV 3.4, which
 *          the reference builds, (R*4899 + G*9617 + B*1868 + 2^13) >> 14, alpha ignored; src/Tracking.cc:209-222; the System shim's
 *          host conversion is the same formula; cv2 4.x uses 15-bit coefficients, at most one grey level away); depth f32, 1 channel;
 *          flow f32, 2 channels (u, v) -- (H,W,2) and planar (2,H,W) alike; mask i32 or i64, 1 channel.
 *   Any plane may be NULL (keep what is resident).  Another dtype / channel count, a pointer that is not device memory of
 *   the context's device (host, pinned host, managed or another GPU's memory) or a misaligned pointer: VDO_ERR_ARG, before any
 *   device work.  An i64 label outside the int32 range is found on the device and the call returns VDO_ERR_ARG: the labels are
 *   never silently truncated, and the frame's resident planes must then be uploaded again before use.
 *   stream: the caller's cudaStream_t (0 = legacy default stream).  The context stream is non-blocking, so the call records
 *   an event on `stream` and makes the context stream wait on it: inputs produced by work queued earlier on `stream` are seen
 *   without a host synchronise.  The call synchronises the context stream once before it returns; after that the inputs
 *   may be freed or overwritten. */
int vdo_frame_upload_dev(vdo_frame *f, const vdo_dev_plane *image, const vdo_dev_plane *depth, const vdo_dev_plane *flow,
                         const vdo_dev_plane *mask, uint64_t stream);
/* Tracking::GrabImageRGBD depth pre-processing (src/Tracking.cc:180-204): d < 0 -> 0, else bf / (d / factor), in place on the
 * resident depth; depth_out (may be NULL) receives the result so the caller's cv::Mat can be mutated like the reference does */
/* bf <= 0: clamp negatives to 0 only (the reference's VirtualKITTI branch) */
int vdo_frame_depth_prep(vdo_frame *f, float bf, float factor, float *depth_out);
/* ORBextractor::operator() (include/ORBextractor.h:47-49, src/ORBextractor.cc:1035-1110) on the resident gray image:
 * pyramid (cv::resize INTER_LINEAR chain), FAST-9/16 per 30-px cell with threshold fallback, octree distribution, IC_Angle.
 * Outputs are in the reference's keypoint order (level-major); max_out bounds the arrays; n_candidates (nlevels, may be NULL)
 * receives the per-level FAST candidate counts.  Descriptors are not produced (dead code in the reference, ORBextractor.cc:1091).
 * Runs on an extractor (vdo_orb_extractor, max_batch 1) that the frame creates on first use and again whenever the settings change, so it refuses
 * what vdo_orb_extractor_create refuses, with the same codes; the frame holds that extractor's device memory until it is destroyed. */
int vdo_orb_extract(vdo_frame *f, int nfeatures, float scale_factor, int nlevels, int ini_th, int min_th, int max_out, float *x,
                    float *y, int *octave, float *response, float *angle, int *size, int *n_out, int *n_candidates);
/* Frame::Frame static candidates (src/Frame.cc:100-129, 181-194): keep ORB keypoints with mask == 0, 0 < depth <= th_depth,
 * non-zero flow whose target stays inside the image.  keep_idx = indices into the input, in order. */
int vdo_frame_filter_static(vdo_frame *f, int n, const float *kx, const float *ky, float th_depth, int *keep_idx, float *cx,
                            float *cy, float *fu, float *fv, float *depth, int *n_out);
/* Frame::SampleKeyPoints (src/Frame.cc:672-740), the background keys of UseSampleFeature: 1: VDO_SAMPLE_KEYS random keys over a 20 x 20
 * grid of the width x height image, drawn from cv::RNG(seeds[i]) exactly as OpenCV's generator draws them, in the reference's order
 * (grid cell by cell, draw order inside a cell).  n frames in one launch; kx / ky: n x VDO_SAMPLE_KEYS f32 each (integer values).
 * width and height must be at least 20 (VDO_ERR_ARG).  kernel_ms (may be NULL): the launch's device time from CUDA events. */
#define VDO_SAMPLE_KEYS 3000
int vdo_sample_keys(vdo_ctx *ctx, int n, int width, int height, const unsigned *seeds, float *kx, float *ky, float *kernel_ms);
/* Frame::Frame semi-dense object sampling (src/Frame.cc:200-228): raster scan with the given stride, mask != 0,
 * 0 < depth < th_depth_obj, flow target inside the image; outputs in raster (push_back) order */
int vdo_frame_sample_objects(vdo_frame *f, float th_depth_obj, int step, int max_out, int *x, int *y, float *cx, float *cy,
                             float *fx, float *fy, float *depth, int *label, int *n_out);
/* Tracking::GetSceneFlowObj with Frame::UnprojectStereoObject (src/Tracking.cc:1278-1364, src/Frame.cc:521-555):
 * flow3d[i] = X_w(cur, i) - X_w(prev, i) in float; valid[i] = both labels > 0 (otherwise the reference sets vObjLabel = -1).
 * Tcw_* are 4x4 row-major f32 (Frame::mTcw); Xw_prev (n x 3, may be NULL) returns the previous-frame world points. */
int vdo_scene_flow(vdo_ctx *ctx, int n, const float *u_prev, const float *v_prev, const float *z_prev, const float *Tcw_prev,
                   const float *u_cur, const float *v_cur, const float *z_cur, const float *Tcw_cur, const float *K,
                   const int *label_prev, const int *label_cur, float *flow3d, float *Xw_prev, unsigned char *valid);
/* 7x7 sigma-2 Gaussian blur of every pyramid level + rotated-BRIEF descriptors (src/ORBextractor.cc:1083-1084, 97-136, pattern :139-397) of the
 * keypoints of the last vdo_orb_extract call (which must have returned angles).  The reference allocates the descriptor matrix and never fills
 * it (the computeDescriptors call is commented out, :1091); this is that call.  desc_out: n x 32 bytes in vdo_orb_extract's keypoint order. */
int vdo_orb_describe(vdo_frame *f, int n, unsigned char *desc_out);
int vdo_frame_debug_blur(vdo_frame *f, int level, unsigned char *img_out);   /* test hook: blurred level of the last vdo_orb_describe */
/* test hook: pyramid level and FAST score map (u8, cv::cornerScore clipped at 0) of the last vdo_orb_extract call */
int vdo_frame_debug_level(vdo_frame *f, int level, unsigned char *img_out, unsigned char *score_out, int *w_out, int *h_out);
/* measurement: device time of the ORB front end (pyramid + FAST score maps) on the resident image */
int vdo_orb_time(vdo_frame *f, int reps, float *ms_avg);

/* ---- batched ORB extraction from device images (ORBextractor::operator(), include/ORBextractor.h:36-110) -----------------------
 * An extractor holds everything one call needs for up to max_batch frames of one size and one set of ORB settings: pyramids, score
 * maps, cell lists, octree work space and the launch tables, all allocated at creation.  A call then runs entirely on the caller's
 * stream: ingest (gray copy, or the colour conversion of vdo_frame_upload_dev) -> pyramid -> FAST scores -> per-cell FAST + NMS ->
 * dense candidate lists -> DistributeOctTree on the device (one CTA per frame and level) -> level-major output -> IC_Angle ->
 * optionally the 7x7 blur and the rotated-BRIEF descriptors.  It does not synchronise the host, allocate, or copy from host memory, so
 * it may be captured in a CUDA graph.  vdo_orb_extract, vdo_orb_describe and the tracker's frame build run on extractors too, so per
 * frame the results equal theirs on the same gray image, bit for bit, in the same order.
 *
 * Keypoint capacity per frame = sum over levels of max(N_l + 2, 4 nIni_l), N_l the level's feature quota and nIni_l the number of
 * initial octree nodes (round((maxX - minX) / (maxY - minY)) of the level's border box): the octree never holds more nodes than that
 * (see k_octree in frame_kernels.cu), and every kept keypoint is one node.  A level under 62 px in either direction has no cells: it
 * contributes no candidates and no keypoints, and its quota is not given to other levels (the reference divides by zero there).
 * VDO_ERR_ARG at creation for an image under 64x64, nfeatures < 1, scale_factor <= 1, nlevels outside 1 .. 12, or a pyramid level
 * under 1 px in either direction (cv::resize asserts on it); VDO_ERR_UNSUPPORTED when a level's capacity exceeds 8192, its cells
 * exceed 62 px, or a level with cells has nIni_l < 1 (an image more than about twice as tall as wide).  Either way the reason is in
 * vdo_last_error, prefixed with the refusing call.  max_batch: 1 .. 64. */
typedef struct vdo_orb_extractor vdo_orb_extractor;
int vdo_orb_extractor_create(vdo_ctx *ctx, int width, int height, int max_batch, int nfeatures, float scale_factor, int nlevels, int ini_th,
                             int min_th, vdo_orb_extractor **out);
void vdo_orb_extractor_destroy(vdo_orb_extractor *ex);
/* out[0] = keypoint capacity per frame, out[1] = device bytes held, out[2] = nlevels, out[3] = max_batch */
int vdo_orb_extractor_info(const vdo_orb_extractor *ex, int64_t out[4]);
/* Caller-allocated DEVICE outputs of vdo_orb_extract_batch_dev for n frames; cap = the capacity of vdo_orb_extractor_info.  Frame i's
 * keypoints are entries [i*cap, i*cap + count_dev[i]) of the per-keypoint arrays, in vdo_orb_extract's order (level-major, level-0
 * coordinates); entries past the count are left as they were. */
typedef struct vdo_orb_batch_out {
  float *x_dev, *y_dev;            /* n x cap */
  int32_t *octave_dev;             /* n x cap */
  float *response_dev, *angle_dev; /* n x cap (angle in degrees) */
  int32_t *size_dev;               /* n x cap */
  uint8_t *desc_dev;               /* n x cap x 32, or NULL: no blur and no descriptors */
  int32_t *count_dev;              /* n: keypoints of the frame */
  int32_t *n_candidates_dev;       /* n x nlevels: FAST candidates per level (vdo_orb_extract's n_candidates) */
  int32_t *status_dev;             /* n: 0, or VDO_ORB_STATUS_* bits; a frame with a non-zero status reports count 0 */
} vdo_orb_batch_out;
#define VDO_ORB_STATUS_NODE_BOUND 1 /* a level's octree exceeded its node bound (never expected: the bound is proven, and checked) */
#define VDO_ORB_STATUS_INPUT 2      /* a candidate outside the level's initial nodes (only reachable through vdo_orb_debug_octree) */
#define VDO_ORB_STATUS_ROUNDS 4     /* a level's octree did not finish within its round limit (never expected) */
/* images: n planes (vdo_dev_plane, u8 with 1, 3 or 4 channels, width x height of the extractor, any strides).  VDO_ERR_ARG before
 * any device work for n < 1 or n > max_batch, a plane of another dtype or channel count, or any image or output pointer that is not
 * device memory of the context's device or not aligned to its element size.  stream: the caller's cudaStream_t (0 = legacy default);
 * every launch goes there, and the inputs must stay valid until the work queued on it has run. */
int vdo_orb_extract_batch_dev(vdo_orb_extractor *ex, int n, const vdo_dev_plane *images, const vdo_orb_batch_out *out, uint64_t stream);
/* test hook: the device octree alone on n host candidates (x, y relative to (minX, minY), response), DistributeOctTree(keys, minX, maxX,
 * minY, maxY, N) (src/ORBextractor.cc:528-752).  Writes the kept keys in list order (at most n; *n_out of them) and the status bits;
 * synchronises the context stream. */
int vdo_orb_debug_octree(vdo_ctx *ctx, int n, const float *kx, const float *ky, const float *kr, int minX, int maxX, int minY, int maxY, int N,
                         float *out_x, float *out_y, float *out_r, int *n_out, int *status);

/* ---- ORB descriptor matching on the device (cv2.BFMatcher(NORM_HAMMING) restated) -----------------------------------------------
 * A call matches P pairs (query frame, train frame) of two descriptor sets in the layout vdo_orb_batch_out writes.  For each query
 * keypoint i < count[q] the output holds the k in {1, 2} train keypoints j < count[t] with the smallest Hamming distance between the
 * 256-bit descriptors, in increasing distance, equal distances to the lower j: knnMatch(desc_q[:nq], desc_t[:nt], k) entry for entry.
 *   window (radius > 0): train j is a candidate of query i only if |x_t[j] - px[i]| <= radius and |y_t[j] - py[i]| <= radius in float32,
 *     (px, py) = pred_dev[p][i], a predicted level-0 position in the train frame: knnMatch(..., mask=M) with M that predicate.
 *   cross_check (k = 1 only): keep i -> j only if i is j's best query under the same candidate predicate, ties to the lower i; without a
 *     window this is BFMatcher(NORM_HAMMING, crossCheck=True).match.
 *   A query with fewer than k candidates gets index -1 and distance -1 in the missing places.  Query slots at or past count[q] (and
 *   rev_idx slots at or past count[t]) are left as they were.
 * The result does not depend on P, on the other pairs of the call, or on how the work is split over the GPU. */
typedef struct vdo_orb_desc_set {
  const uint8_t *desc_dev;  /* F x cap x 32 (16-byte aligned) */
  const float *x_dev;       /* F x cap level-0 positions; read only with a window (train set), may be NULL otherwise */
  const float *y_dev;
  const int32_t *count_dev; /* F: keypoints per frame; a value outside 0 .. cap sets a status bit (see below) */
  int32_t n_frames, cap;    /* F >= 1; 1 <= cap < 2^23 */
} vdo_orb_desc_set;
typedef struct vdo_orb_match_opts {
  int32_t k;           /* 1 or 2 */
  int32_t cross_check; /* 0 or 1 (k = 1 only; needs rev_idx_dev) */
  float radius;        /* search window half-size in level-0 pixels; <= 0: no window */
} vdo_orb_match_opts;
typedef struct vdo_orb_match_out {
  int32_t *idx_dev, *dist_dev; /* P x query.cap x k: train index and Hamming distance, -1 where missing */
  int32_t *rev_idx_dev;        /* P x train.cap: each train keypoint's best query (-1: none), or NULL; required with cross_check */
  int32_t *status_dev;         /* P: 0, or VDO_ORB_MATCH_STATUS_* bits */
} vdo_orb_match_out;
#define VDO_ORB_MATCH_STATUS_QUERY_COUNT 1 /* count[q] outside 0 .. cap: the pair's query rows are not written */
#define VDO_ORB_MATCH_STATUS_TRAIN_COUNT 2 /* count[t] outside 0 .. cap: taken as 0 (every query gets -1; rev_idx not written) */
/* pairs: host array of P (query frame, train frame) index pairs, 1 <= P <= 64.  query and train may be the same set.  pred_dev: P x
 * query.cap x 2 f32 (px, py), required with a window and ignored without.  VDO_ERR_ARG before any device work for: P outside 1 .. 64, a
 * frame index out of range, k not 1 or 2, cross_check with k = 2 or without rev_idx_dev, a NaN radius, a window without train x/y or
 * pred_dev, and any pointer that is NULL where required, not device memory of the context's device, or not aligned to its element size.
 * stream: the caller's cudaStream_t (0 = legacy default); the call enqueues 3 to 5 kernels there and does not allocate, copy from host
 * memory or synchronise, so it may be captured in a CUDA graph. */
int vdo_orb_match_batch_dev(vdo_ctx *ctx, int P, const int32_t *pairs, const vdo_orb_desc_set *query, const vdo_orb_desc_set *train,
                            const float *pred_dev, const vdo_orb_match_opts *opts, const vdo_orb_match_out *out, uint64_t stream);

/* ---- initial model (SURVEY.md 8 row A10 / next-row N1) ------------------------------------------------------------------
 * vdo_init_model_batch  <- Tracking::GetInitModelCam / GetInitModelObj (src/Tracking.cc:1614-1715, 1717-1849), including the
 *   cv::solvePnPRansac(pre_3d, cur_2d, K, 0, rvec, tvec, false, iters=500, thr=0.4, conf=0.98, inliers, SOLVEPNP_AP3P) call
 *   (OpenCV 3.4; engine restated in oracle/pnp_ransac.c).  One problem per camera / object: points offsets[p]..offsets[p+1] of
 *   obj3d (pre_3d, n x 3 f32, world) and img2d (cur_2d, n x 2 f32).  K4 = fx, fy, cx, cy (Frame::fx.. / mK).  T_mm (nprob x 16,
 *   4x4 row-major f32) is the constant-motion model (mVelocity*mLastFrame.mTcw, or mTcw*vObjMod[PreObjID]); has_mm[p] = 0 for an
 *   object with no previous motion (PreObjID == -1).  Outputs: T_init (nprob x 16: `output`), n_sub[p] and sub_idx (the chosen
 *   inlier subset as ascending LOCAL indices, stored from offsets[p]); info (nprob x 8 ints: inliers.rows, MM_inlier.size(),
 *   motion model used, n_sub, RANSAC iterations run, winning iteration, valid minimal solves, 0); Rt_refit / Rt_hyp
 *   (nprob x 12 f64 [R row-major | t], may be NULL): refitted model and winning hypothesis (test hooks). */
int vdo_init_model_batch(vdo_ctx *ctx, int nprob, const int *offsets, const float *obj3d, const float *img2d, const float *K4, int iters,
                         double thr, double conf, const float *T_mm, const unsigned char *has_mm, float *T_init, int *n_sub, int *sub_idx,
                         int *info, double *Rt_refit, double *Rt_hyp);
/* kernels launched so far by vdo_init_model_batch on this context (bench accounting) */
int vdo_init_model_launches(vdo_ctx *ctx);

/* ---- pose of matched ORB frame pairs on the device (cv::solvePnPRansac(AP3P) on descriptor matches) ---------------------------
 * The step after vdo_orb_extract_batch_dev and vdo_orb_match_batch_dev: for each of P (query frame, train frame) pairs the query
 * keypoints are back-projected through the query frame's depth, and the engine of vdo_init_model_batch (no motion model) estimates the
 * train camera's pose from those 3-D points and the matched train keypoints.  A solver holds all work space, allocated at creation.
 *
 * Correspondences of pair p = (q, t): query keypoint i < count[q], in ascending i, when all of these hold
 *   - j = idx[p][i][0] satisfies 0 <= j < count[t];
 *   - ratio > 0 (k = 2 only): idx[p][i][1] >= 0 and (float)dist[p][i][0] < ratio * (float)dist[p][i][1];
 *   - z = depth at row (int)y_q[i], column (int)x_q[i] (truncation; a pixel outside the plane fails) satisfies 0 < z <= max_depth
 *     (max_depth <= 0: z > 0).
 * Its 3-D point is Frame::UnprojectStereoStat's (src/Frame.cc:484-519) in float, x = (u - cx) z (1/fx), y = (v - cy) z (1/fy), with
 * (u, v) = (x_q[i], y_q[i]) and K_query; with Tcw_query it is then moved into the world frame as Tracking does (Twc = Tcw^-1, the
 * products accumulated in double and rounded to float once).  Its observation is (x_t[j], y_t[j]) and the camera is K_train.
 * The result equals vdo_init_model_batch with no motion model on exactly those arrays, bit for bit: T, Rt, the inlier set, the
 * iterations run, the winning iteration and the valid-solve count.  With Tcw_query the query frame's pose, T is the train frame's Tcw
 * (the RANSAC branch of Tracking::GetInitModelCam, src/Tracking.cc:1614-1715).
 * The per-pair work (gather, the RANSAC sample table drawn on the device from cv::RNG(-1) as OpenCV draws it, hypotheses, scores,
 * bookkeeping and refit) runs in six launches on the caller's stream; the call does not synchronise the host, allocate, or read pageable
 * host memory after its argument checks, so it may be captured in a CUDA graph.  A replay uses the host parameters of the captured call
 * (pairs, K, Tcw, options, pointers) and the device inputs' contents at replay time.  One solver runs one call at a time: calls on one
 * solver must be ordered (one stream, or synchronised between streams). */
typedef struct vdo_pnp_solver vdo_pnp_solver;
/* max_pairs 1 .. 64, cap >= 1 (query keypoint capacity per frame, the largest query.cap a call may use), max_iters 1 .. 4096 */
int vdo_pnp_solver_create(vdo_ctx *ctx, int max_pairs, int cap, int max_iters, vdo_pnp_solver **out);
void vdo_pnp_solver_destroy(vdo_pnp_solver *s);
/* out: max_pairs, cap, max_iters, device bytes held */
int vdo_pnp_solver_info(const vdo_pnp_solver *s, int64_t out[4]);

typedef struct vdo_pnp_match_opts {
  int32_t k;          /* columns of the orb_match result idx / dist hold (1 or 2); column 0 is the correspondence */
  float ratio;        /* > 0 (k = 2 only): Lowe's ratio test as above; <= 0: off */
  float max_depth;    /* > 0: keep 0 < z <= max_depth (ThDepthBG-style); <= 0: z > 0 only */
  int32_t iters;      /* RANSAC iterations, 1 .. max_iters (the reference: 500) */
  double thr, conf;   /* reprojection threshold in px (> 0) and confidence in (0, 1) (the reference: 0.4, 0.98) */
} vdo_pnp_match_opts;

typedef struct vdo_pnp_out {   /* caller-allocated DEVICE outputs for P pairs */
  float *T_dev;                /* P x 16: 4x4 row-major, the refitted model rounded to float as vdo_init_model_batch returns it; identity if none */
  double *Rt_dev;              /* P x 12 f64 refitted [R row-major | t] ([I | 0] if none), or NULL */
  uint8_t *inlier_dev;         /* P x query.cap: 1 where query keypoint i < count[q] is in the RANSAC inlier set, else 0; slots at or past
                                  count[q] (all slots with QUERY_COUNT) are left as they were */
  int32_t *n_corr_dev;         /* P: correspondences */
  int32_t *n_inlier_dev;       /* P: RANSAC inliers (0 if no model) */
  int32_t *info_dev;           /* P x 4: iterations run, winning iteration (-1: none), valid minimal solves, VDO_PNP_STATUS_* bits */
} vdo_pnp_out;
#define VDO_PNP_STATUS_QUERY_COUNT 1 /* count[q] outside 0 .. query.cap: no correspondences, the inlier row is not written */
#define VDO_PNP_STATUS_TRAIN_COUNT 2 /* count[t] outside 0 .. train.cap: taken as 0, so no correspondences */
#define VDO_PNP_STATUS_FEW_POINTS 4  /* fewer than 4 correspondences: T identity, n_inlier 0 */
#define VDO_PNP_STATUS_NO_MODEL 8    /* no hypothesis had more than 3 inliers: T identity, n_inlier 0 */

/* pairs: host P x 2 (query frame, train frame), as for vdo_orb_match_batch_dev.  query / train: the descriptor sets of that call;
 * x_dev, y_dev and count_dev are read, desc_dev is not.  idx_dev / dist_dev: vdo_orb_match_batch_dev's P x query.cap x k outputs for the
 * same pairs.  depth: P planes (f32, 1 channel, any strides), the metric depth of each pair's query frame, depth_wh (host P x 2) its
 * width and height.  K_query: host P x 4 (fx, fy, cx, cy) of the query frames; K_train: host P x 4, NULL = K_query.  Tcw_query: host
 * P x 16 (4x4 row-major f32), NULL = identity.  stream: the caller's cudaStream_t (0 = legacy default).
 * VDO_ERR_ARG before any device work for: P outside 1 .. min(64, max_pairs); a frame index out of range; query.cap > cap of the solver;
 * n_frames or cap < 1 in a set; iters outside 1 .. max_iters; k not 1 or 2, or ratio > 0 with k = 1; thr NaN or <= 0, conf outside
 * (0, 1); a NaN ratio or max_depth; a depth plane that is not f32 with one channel, or a width or height < 1; and any required pointer
 * (all but K_train, Tcw_query and Rt_dev) that is NULL, not device memory of the context's device where it is a device pointer, or not
 * aligned to its element size. */
int vdo_pnp_match_batch_dev(vdo_pnp_solver *s, int P, const int32_t *pairs, const vdo_orb_desc_set *query, const vdo_orb_desc_set *train,
                            const int32_t *idx_dev, const int32_t *dist_dev, const vdo_dev_plane *depth, const int32_t *depth_wh,
                            const float *K_query, const float *K_train, const float *Tcw_query, const vdo_pnp_match_opts *opts,
                            const vdo_pnp_out *out, uint64_t stream);

/* ---- refined pose of matched ORB frame pairs on the device (Optimizer::PoseOptimizationFlow2Cam on descriptor matches) ----------
 * The step after vdo_pnp_match_batch_dev, as Tracking::Track takes it with the shipped settings (src/Tracking.cc:687-699): the joint
 * flow / SE(3) Levenberg-Marquardt of vdo_pose_opt_flow2 (mode 0, camera) on the correspondences of each of P (query, train) pairs,
 * started from a pose the caller holds on the device.  A refiner holds all work space, allocated at creation.
 *
 * Problem of pair p = (q, t): query keypoint i enters when it is a correspondence under the rule of vdo_pnp_match_batch_dev (k, ratio,
 * max_depth) and mask_dev[p][i] != 0 (no mask: every correspondence), in ascending i.  Its point is (x_q[i], y_q[i]), its depth the z the
 * rule read, its flow estimate (x_t[j] - x_q[i], y_t[j] - y_q[i]) in float with j = idx[p][i][0].  The problem uses K[p] for projection
 * and back-projection (the flow model has one camera), Tcw_last = Tcw_query[p] (identity if NULL) and T_init = T_init_dev[p].  With
 * vdo_pnp_match_batch_dev's T and inlier flags as T_init_dev and mask_dev this is PoseOptimizationFlow2Cam(cur, last, TemperalMatch_subset)
 * after the RANSAC branch of Tracking::GetInitModelCam: with Tcw_query, T is the train frame's Tcw; without it, the query -> train pose.
 * T_init_dev may hold any initial pose (a constant-velocity model, say); choosing between models is the caller's.
 * The result equals vdo_pose_opt_flow2_batch(ctx, quirk, ...) on the same arrays gathered on the host, bit for bit (T, stats, flow,
 * inlier): each problem runs on the kernel shape its own n selects (n <= VDO_FLOW2_CLUSTER_MAX_N: a cluster, else one CTA), chosen on the
 * device, so it does not depend on which other pairs share the call.  (The VDO_FLOW_SINGLE_CTA test switch of the host entry does not
 * apply here.)  At most four launches on the caller's stream (gather, cluster LM, single-CTA LM when query.cap > VDO_FLOW2_CLUSTER_MAX_N,
 * scatter); the call does not synchronise the host, allocate, or read pageable host memory after its argument checks, so it may be
 * captured in a CUDA graph, and a replay uses the captured call's host parameters.  Calls on one refiner must be ordered. */
typedef struct vdo_pose_refiner vdo_pose_refiner;
/* max_pairs 1 .. 64, cap >= 1 (the largest query.cap a call may use; max_pairs x cap below 2^31).  A cap above
 * VDO_FLOW2_CLUSTER_MAX_N also allocates the single-CTA kernel's scratch, max_pairs x cap x 144 bytes. */
int vdo_pose_refiner_create(vdo_ctx *ctx, int max_pairs, int cap, vdo_pose_refiner **out);
void vdo_pose_refiner_destroy(vdo_pose_refiner *r);
/* out: max_pairs, cap, device bytes held, 0 */
int vdo_pose_refiner_info(const vdo_pose_refiner *r, int64_t out[4]);

typedef struct vdo_pose_refine_opts {
  int32_t k; float ratio; float max_depth;   /* the correspondence rule, as in vdo_pnp_match_opts */
  int32_t quirk;                             /* 0 or 1, as vdo_pose_opt_flow2 (the tracker's default is 1) */
} vdo_pose_refine_opts;

typedef struct vdo_pose_refine_out {         /* caller-allocated DEVICE outputs for P pairs */
  float *T_dev;          /* P x 16: the refined pose, vdo_pose_opt_flow2's T_out (identity when n < 3) */
  double *flow_dev;      /* P x query.cap x 2: the refined flow of every query keypoint that entered the problem; other slots untouched */
  uint8_t *inlier_dev;   /* P x query.cap: 1 = entered and chi2 <= 0.04; 0 for every other i < count[q]; slots >= count[q] untouched */
  int32_t *n_points_dev; /* P: points in the pair's problem */
  double *stats_dev;     /* P x 8: vdo_pose_opt_flow2's stats ([0] = -1 when n < 3) */
  int32_t *status_dev;   /* P: VDO_PNP_STATUS_QUERY_COUNT / _TRAIN_COUNT bits, as vdo_pnp_match_batch_dev sets them */
} vdo_pose_refine_out;

/* Arguments as vdo_pnp_match_batch_dev's, with K (host P x 4) for K_query and no K_train.  T_init_dev: device P x 16 (4x4 row-major
 * f32); mask_dev: device P x query.cap u8, or NULL.
 * VDO_ERR_ARG before any device work, writing nothing, for: every refusal of vdo_pnp_match_batch_dev that applies (P, frame indices,
 * query.cap above the refiner's cap, set sizes, k, ratio, max_depth, depth planes, NULL, misaligned or foreign pointers); quirk not 0
 * or 1; a NULL T_init_dev; T_init_dev or a non-NULL mask_dev that is not device memory of the context's device or not aligned to its
 * element size. */
int vdo_pose_refine_batch_dev(vdo_pose_refiner *r, int P, const int32_t *pairs, const vdo_orb_desc_set *query,
                              const vdo_orb_desc_set *train, const int32_t *idx_dev, const int32_t *dist_dev,
                              const vdo_dev_plane *depth, const int32_t *depth_wh, const float *K, const float *Tcw_query,
                              const float *T_init_dev, const uint8_t *mask_dev, const vdo_pose_refine_opts *opts,
                              const vdo_pose_refine_out *out, uint64_t stream);

/* ---- rigid motions of segmented objects between frame pairs on the device (Tracking::Track's object step, bJoint = true) ----------
 * Tracking::Track lines 760-1003 without the ground-truth presence gate, for each of P (last, current) frame pairs: the last frame is
 * sampled semi-densely (Frame.cc:200-228), every object of its instance mask gets the initial model of GetInitModelObj
 * (Tracking.cc:1717-1849: solvePnPRansac(AP3P) on the object's world points and flow-propagated pixels, then the choice against the
 * constant-motion model), objects with at least min_inliers inliers are refined by PoseOptimizationFlow2 (Optimizer.cc:2755-2972,
 * vdo_pose_opt_flow2 mode 1) and their motion H = Tcw_cur^-1 X (Tracking.cc:933) is reported with the object centre (:856-866).
 * The caller's mask labels are the object identities; samples are fresh every pair.  An estimator holds all work space, allocated at
 * creation.
 *
 * Samples of pair p: the stride-`step` raster of the last frame (x = 0, step, ...; y likewise), in raster order, where mask != 0,
 * 0 < depth < th_depth_obj and the flow target (cx, cy) = (x + fx, y + fy) (float) lies strictly inside the image (the rule of
 * vdo_frame_sample_objects).  Object slots: the distinct non-zero labels among the samples in ascending order, the first max_objects of
 * them (more: the largest are dropped and VDO_OM_PAIR_OBJECT_CAP is set).  Object s holds its samples in raster order; point k's world
 * point is Frame::UnprojectStereoObject of (x, y, depth) with K[p] and Tcw_last[p] (rounded as the tracker rounds it), its observation
 * (cx, cy).  Centre: the float sum of the world points in order times (float)(1.0 / n).  Motion model: for slot s with label L, the
 * first j with prev_label[p][j] == L (a prev_label of -1 is an empty slot and never matches) gives T_mm = Tcw_cur[p] * prev_H[p][j]
 * (cv::Mat float gemm rounding); passing the previous call's label_dev and H_dev reproduces the reference's sequence.  RANSAC as
 * vdo_init_model_batch(iters, thr, conf); with n_sub >= min_inliers, the LM (mode 1, quirk) from T_init on the chosen set with the
 * samples' (x, y), depth and flow, Tcw_last[p] and K[p], giving X; H = Tcw_cur^-1 X (Converter::toInvMatrix, float gemm); velocity
 * t_H - (I - R_H) c in float (Tracking.cc:958, metres per frame).  With identity poses H is the motion in the last camera's frame.
 * Equal, bit for bit, to vdo_frame_sample_objects + host grouping + vdo_init_model_batch + vdo_pose_opt_flow2_batch on the same inputs.
 *
 * At most ten launches on `stream`; the call does not synchronise the host, allocate, or read pageable host memory after its argument
 * checks, so it may be captured in a CUDA graph, and a replay uses the captured call's host parameters (K, planes, options).  Calls on
 * one estimator must be ordered. */
typedef struct vdo_obj_motion vdo_obj_motion;
#define VDO_OBJ_MOTION_MAX_PAIRS 64
#define VDO_OBJ_MOTION_MAX_OBJECTS 32
#define VDO_OBJ_MOTION_MAX_ITERS 500
/* max_pairs 1 .. 64, max_objects 1 .. 32 (object slots per pair), cap >= 1 (samples per pair; max_pairs x cap below 2^31).  A cap above
 * VDO_FLOW2_CLUSTER_MAX_N also allocates the single-CTA LM scratch, max_pairs x cap x 144 bytes. */
int vdo_obj_motion_create(vdo_ctx *ctx, int max_pairs, int max_objects, int cap, vdo_obj_motion **out);
void vdo_obj_motion_destroy(vdo_obj_motion *m);
/* out: max_pairs, max_objects, cap, device bytes held */
int vdo_obj_motion_info(const vdo_obj_motion *m, int64_t out[4]);

typedef struct vdo_obj_motion_opts {
  int32_t step;           /* sampling stride (the reference: 4) */
  float th_depth_obj;     /* ThDepthObj: samples need depth < th_depth_obj */
  int32_t iters;          /* RANSAC iterations, 1 .. VDO_OBJ_MOTION_MAX_ITERS (500) */
  int32_t min_inliers;    /* the initialisation gate, >= 0 (50) */
  double thr, conf;       /* RANSAC reprojection threshold > 0 (0.4) and confidence in (0, 1) (0.98) */
  int32_t quirk;          /* 0 or 1, as vdo_pose_opt_flow2 (1) */
  int32_t pad;
} vdo_obj_motion_opts;

typedef struct vdo_obj_motion_out {   /* caller-allocated DEVICE outputs; M = the estimator's max_objects, C = its cap */
  /* per object slot, P x M: */
  int32_t *label_dev;     /* the slot's label, -1 for an empty slot */
  float *H_dev;           /* x 16: vObjMod, Tcw_cur^-1 X; identity without the LM and for an empty slot */
  float *X_dev;           /* x 16: the LM result Obj_X_tmp; identity without the LM */
  float *T_init_dev;      /* x 16: mInitModel, vdo_init_model_batch's T_init (identity for an empty slot) */
  float *centre_dev;      /* x 3: ObjCentre3D_pre in the world frame (0 for an empty slot) */
  float *velocity_dev;    /* x 3: t_H - (I - R_H) c (0 without the LM) */
  int32_t *info_dev;      /* x 8: samples n, then vdo_init_model_batch's n_ransac, n_mm, used_mm, n_sub, iterations run, winning
                             iteration, valid minimal solves (for an empty slot: 0, with winning iteration -1) */
  double *stats_dev;      /* x 8: vdo_pose_opt_flow2's stats; [0] = -1 without the LM */
  int32_t *status_dev;    /* VDO_OM_* bits */
  /* per sample, P x C (entries past n_samples untouched): */
  int32_t *sample_x_dev, *sample_y_dev, *sample_label_dev;
  int32_t *sample_slot_dev;      /* the sample's object slot, -1 for a dropped label or a pair with VDO_OM_PAIR_LABEL_RANGE */
  float *sample_depth_dev, *sample_cx_dev, *sample_cy_dev;
  float *sample_flow_dev;        /* x 2: the input flow at the sample */
  double *sample_flow_ref_dev;   /* x 2: the LM's refined flow for a sample in an LM problem, the input flow otherwise */
  uint8_t *sample_flags_dev;     /* 1: in the chosen initial inlier set, 2: LM inlier (chi2 <= 0.04) */
  /* per pair, P: */
  int32_t *n_samples_dev;
  int32_t *pair_status_dev;      /* VDO_OM_PAIR_* bits */
} vdo_obj_motion_out;
#define VDO_OM_FEW_POINTS 1      /* fewer than 4 samples: no RANSAC */
#define VDO_OM_NO_MODEL 2        /* 4 or more samples, no hypothesis with more than 3 inliers */
#define VDO_OM_FEW_INLIERS 4     /* n_sub < min_inliers: no LM, H = X = identity as the reference sets them */
#define VDO_OM_USED_MM 8         /* the constant-motion model was chosen */
#define VDO_OM_PAIR_OBJECT_CAP 1 /* the pair has more than max_objects labels: the largest are dropped */
#define VDO_OM_PAIR_LABEL_RANGE 2 /* an i64 mask label outside the int32 range: the pair's objects are not estimated */

/* depth, flow, mask, wh: P each, the LAST frame of the pair: metric depth f32 (1 channel), its flow to the current frame f32 (2 channels,
 * HWC or CHW), its instance mask i32 or i64, at any strides (vdo_dev_plane); wh: host P x 2 (width, height).  K: host P x 4 (fx, fy, cx,
 * cy).  Tcw_last_dev, Tcw_cur_dev: device P x 16 (4x4 row-major f32) or NULL (identity).  prev_label_dev (device P x M int32) and
 * prev_H_dev (device P x M x 16 f32): both NULL (no motion models) or both given.
 * VDO_ERR_ARG before any device work, writing nothing, for: P outside 1 .. max_pairs; a NULL depth, flow, mask, wh, K, opts or out; a
 * plane of another dtype or channel count, NULL, misaligned or not device memory of the context's device; a width or height < 1; step
 * < 1; ceil(w / step) x ceil(h / step) above the estimator's cap for any pair; th_depth_obj NaN; iters outside 1 .. 500; thr <= 0; conf
 * outside (0, 1); min_inliers < 0; quirk not 0 or 1; only one of prev_label_dev / prev_H_dev; any given device pointer (inputs and every
 * output) NULL, misaligned or foreign. */
int vdo_obj_motion_batch_dev(vdo_obj_motion *m, int P, const vdo_dev_plane *depth, const vdo_dev_plane *flow, const vdo_dev_plane *mask,
                             const int32_t *wh, const float *K, const float *Tcw_last_dev, const float *Tcw_cur_dev,
                             const int32_t *prev_label_dev, const float *prev_H_dev, const vdo_obj_motion_opts *opts,
                             const vdo_obj_motion_out *out, uint64_t stream);

/* ---- tracked objects between frame pairs on the device (GetSceneFlowObj + DynObjTracking ahead of the object step) -----------------
 * vdo_obj_track_batch_dev runs the reference's object step in its order on a vdo_obj_motion estimator: the last frame is sampled as
 * vdo_obj_motion_batch_dev samples it; each sample looks up the current frame at its flow target (Tracking.cc:288-305): u = (int)cx,
 * v = (int)cy, and when 0 < u < W-1, 0 < v < H-1 and 0 < depth_cur(v, u) < th_depth_obj the current depth and label are depth_cur(v, u)
 * and mask_cur(v, u), otherwise 0.1 and 0.  Scene flow (GetSceneFlowObj, :1278-1364): flow3d = X_w(cx, cy, depth_cur, Tcw_cur) -
 * X_w(x, y, depth, Tcw_last) (Frame::UnprojectStereoObject), equal to vdo_scene_flow bit for bit; a sample whose current or last label is
 * <= 0 gets object label -1 and flow3d 0.  DynObjTracking (:1366-1612): the other (valid) samples are grouped by CURRENT label, ascending,
 * each group in raster order; object slots are the first max_objects labels (more: VDO_OM_PAIR_OBJECT_CAP, their samples are not
 * classified).  Per slot, in this order: boundary when more than 0.5 of its points (cx, cy) lie outside the band shrink_row <= y <=
 * H - shrink_row, shrink_col <= x <= W - shrink_col; static when the fraction of points with |(flow3d.x, flow3d.z)| < sf_mg_thres is above
 * sf_ds_thres (those samples get object label 0); far when the mean current depth (float sum in point order) is above th_depth_obj or the
 * slot has fewer than 150 points; dynamic otherwise (the float rounding of vdo_dyn_obj_tracking).  IDs, for the dynamic slots in ascending
 * label order: vote = the majority last label of the slot's samples (ties: the smaller label); if max_id == 1 a fresh ID (max_id++),
 * otherwise the id of the first previous slot with label == vote and stat, else max_id++.  Two slots may get the same ID, as in the
 * reference.  Then, for the dynamic slots only, the object step of vdo_obj_motion_batch_dev (GetInitModelObj, the min_inliers gate,
 * PoseOptimizationFlow2 mode 1, H, centre, velocity) with the motion model Tcw_cur * prev_H[j] of the first previous slot j whose id equals
 * the slot's ID (stat not required, tracker.cpp:407-409).  stat (bObjStat) is 1 for a dynamic slot that passed the gate (:885-897).
 * Per-sample object label (vObjLabel): -2 never classified, -1 invalid, boundary or far, 0 static, the ID otherwise, then -1 outside the
 * chosen RANSAC set (:1841-1845) and for LM outliers.
 * UpdateMask is vdo_obj_update_mask_batch_dev: call it on the same pair first (the current mask as given is what the reference uses
 * whenever UpdateMask recovers nothing).  This call samples the last frame afresh; vdo_obj_track_set_batch_dev takes the samples from
 * the feature set vdo_obj_renew_batch_dev carried over from the previous pair (RenewFrameInfo), as the reference does after its first
 * pair.  Not done here: the ground-truth gate.
 *
 * State: the previous call's label, id, stat and H (per slot) and max_id (per pair) are passed as prev_*; all NULL is the reset state
 * (every slot empty, max_id = 1, what the reference does at f_id == 1).  A pair whose sequence starts anew in a batch is reset by writing
 * that state into its row of the prev arrays: label -1, id -1, stat 0, H identity, max_id 1.
 * Launches on `stream`: k_om_sample, k_ot_flow, k_ot_group, the RANSAC kernels, k_om_lm_prep, the LM, k_om_finish, k_ot_finish; no
 * allocation, host synchronise or pageable host read after the checks, so the call may be captured in a CUDA graph. */
typedef struct vdo_obj_track_opts {
  int32_t step;           /* as vdo_obj_motion_opts */
  float th_depth_obj;
  int32_t iters;
  int32_t min_inliers;
  double thr, conf;
  int32_t quirk;
  float sf_mg_thres;      /* SFMgThres: a point is static when |(sf.x, sf.z)| < sf_mg_thres (0.12) */
  float sf_ds_thres;      /* SFDsThres: an object is static when more than this fraction of its points are (0.3) */
  int32_t shrink_row, shrink_col;   /* border band (25, 50 for KITTI; 0 otherwise), >= 0 */
  int32_t pad;
} vdo_obj_track_opts;

typedef struct vdo_obj_track_out {    /* caller-allocated DEVICE outputs; M = the estimator's max_objects, C = its cap */
  vdo_obj_motion_out motion;  /* as vdo_obj_motion_batch_dev; label_dev is the slot's CURRENT label, sample_label_dev the last label */
  /* per object slot, P x M: */
  int32_t *id_dev;        /* the object ID of a dynamic slot, -1 otherwise */
  int32_t *cls_dev;       /* VDO_OT_* */
  int32_t *vote_dev;      /* the voted last label of a dynamic slot, 0 otherwise */
  int32_t *stat_dev;      /* 1: dynamic and passed the gate */
  /* per sample, P x C (entries past n_samples untouched): */
  int32_t *label_cur_dev; /* the current label at the flow target (0 when the look-up fails) */
  float *depth_cur_dev;   /* the current depth at the flow target (0.1 when the look-up fails) */
  float *flow3d_dev;      /* x 3: the world-frame scene flow (0 for an invalid sample) */
  int32_t *obj_label_dev; /* vObjLabel */
  /* per pair, P: */
  int32_t *max_id_dev;
} vdo_obj_track_out;
#define VDO_OT_EMPTY 0
#define VDO_OT_DYNAMIC 1
#define VDO_OT_STATIC 2
#define VDO_OT_BOUNDARY 3
#define VDO_OT_FAR 4

/* depth, flow, mask: the last frames as vdo_obj_motion_batch_dev; depth_cur, mask_cur: P each, the current frame's metric depth (f32) and
 * instance mask (i32 or i64) at any strides, read at the pair's wh like the last planes.  prev_label_dev, prev_id_dev, prev_stat_dev (device
 * P x M int32), prev_H_dev (P x M x 16 f32) and prev_max_id_dev (P int32): all NULL or all given.
 * VDO_ERR_ARG before any device work, writing nothing, for: every refusal of vdo_obj_motion_batch_dev; a NULL depth_cur or mask_cur; a
 * current plane of another dtype or channel count; sf_mg_thres or sf_ds_thres NaN; a negative shrink;
 * prev partly given; any given device pointer (inputs and every output) NULL, misaligned or foreign. */
int vdo_obj_track_batch_dev(vdo_obj_motion *m, int P, const vdo_dev_plane *depth, const vdo_dev_plane *flow, const vdo_dev_plane *mask,
                            const vdo_dev_plane *depth_cur, const vdo_dev_plane *mask_cur, const int32_t *wh, const float *K,
                            const float *Tcw_last_dev, const float *Tcw_cur_dev, const int32_t *prev_label_dev, const int32_t *prev_id_dev,
                            const int32_t *prev_stat_dev, const float *prev_H_dev, const int32_t *prev_max_id_dev,
                            const vdo_obj_track_opts *opts, const vdo_obj_track_out *out, uint64_t stream);

/* ---- objects the segmentation missed, recovered in the current masks on the device (Tracking::UpdateMask) ---------------------------
 * vdo_obj_update_mask_batch_dev runs UpdateMask (Tracking.cc:2997-3068) for P independent (last, current) pairs on a vdo_obj_motion
 * estimator, writing the caller's current masks in place.  Samples: exactly those of vdo_obj_motion_batch_dev / vdo_obj_track_batch_dev
 * with the same step and th_depth_obj (they stand for the last frame's vSemObjLabel and mvObjCorres), so update_mask then track on the
 * same planes is the reference's order for a pair.  Slots: the distinct sample labels ascending (UniLab), the first max_objects of them
 * (more: VDO_OM_PAIR_OBJECT_CAP, the others are neither voted nor recovered).  Slot by slot in ascending order: the samples whose target
 * u = (int)cx, v = (int)cy satisfies 0 < u < W, 0 < v < H read mask_cur(v, u) as updated by the earlier slots' recoveries; with fewer than
 * 100 such voters the slot is skipped; otherwise when the majority label (ties: the smaller label) is 0 the slot is recovered: every
 * last-frame pixel (k, j) with mask == label goes to x = k + (int)fx, y = j + (int)fy and, when 0 < x < W and 0 < y < H, mask_cur(y, x)
 * becomes the label.  Where several recovered slots push onto one pixel the highest slot wins (it writes last in the reference).  Only
 * pixels that get a recovered label are written.  An i64 last label outside int32 at a sample (as vdo_obj_motion_batch_dev) or an i64
 * current label outside int32 at a voter's target sets VDO_OM_PAIR_LABEL_RANGE: that pair recovers nothing and its mask_cur is untouched.
 * Equal, bit for bit, to vdo_frame_sample_objects + vdo_update_mask on resident frames with the same planes whenever the pair has at most
 * max_objects labels and no current label of -1 at a voter's target (vdo_update_mask's gather uses -1 as its outside marker and drops
 * such a voter; the reference counts it, and so does this call).
 * Pairs of one call are independent: no mask_cur may share a byte with any plane of the call.  Consecutive frames of one sequence go in
 * consecutive calls, the updated mask_cur of one call being the next call's mask.
 * Launches on `stream` (six): k_om_sample, k_um_group (the slots, voter counts and the sample-target hash), k_um_pixels<0> (which
 * slots push onto each sample target), k_um_vote (the sequential vote), k_um_pixels<1> and k_um_pixels<2> (claim, then atomicMax the
 * recovered labels); no allocation, host synchronise or pageable host read after the checks, so the call may be captured in a CUDA graph.
 * The work space is the estimator's: the call uses what the RANSAC and the LM leave idle. */
typedef struct vdo_obj_mask_out {     /* caller-allocated DEVICE outputs; M = the estimator's max_objects */
  /* per object slot, P x M: */
  int32_t *label_dev;     /* the slot's LAST-frame label, -1 for an empty slot */
  int32_t *n_vote_dev;    /* the slot's samples whose target is inside the image (LabTmp.size()) */
  int32_t *vote_dev;      /* the majority current label the slot saw (after the earlier slots' recoveries); 0 when n_vote < 100 or the
                             pair has VDO_OM_PAIR_LABEL_RANGE */
  int32_t *recovered_dev; /* 1: the slot's last mask was pushed into mask_cur */
  /* per pair, P: */
  int32_t *n_samples_dev;
  int32_t *pair_status_dev;  /* VDO_OM_PAIR_OBJECT_CAP, VDO_OM_PAIR_LABEL_RANGE */
} vdo_obj_mask_out;

/* depth, flow, mask, wh, step, th_depth_obj: the last frames and sampling as vdo_obj_motion_batch_dev; mask_cur: P, the current frame's
 * instance mask i32 or i64 (1 channel) at any strides, read and written in place.
 * VDO_ERR_ARG before any device work, writing nothing, for: every refusal of vdo_obj_motion_batch_dev that applies (P, a NULL array,
 * plane types, sizes, the cap, step < 1, th_depth_obj NaN, NULL, misaligned or foreign device pointers); a NULL mask_cur or one of
 * another dtype or channel count; a mask_cur whose pixels are not distinct elements (neither |stride_x| >= 1 and |stride_y| >=
 * W |stride_x| nor |stride_y| >= 1 and |stride_x| >= H |stride_y|); a mask_cur whose byte range overlaps any other plane of the call,
 * another pair's mask_cur included. */
int vdo_obj_update_mask_batch_dev(vdo_obj_motion *m, int P, const vdo_dev_plane *depth, const vdo_dev_plane *flow, const vdo_dev_plane *mask,
                                  const vdo_dev_plane *mask_cur, const int32_t *wh, int32_t step, float th_depth_obj,
                                  const vdo_obj_mask_out *out, uint64_t stream);

/* ---- object features carried across frame pairs on the device (the object half of Tracking::RenewFrameInfo) ---------------------------
 * The reference does not sample a frame afresh once it is tracked: its object features (mvObjKeys, vSemObjLabel, mvObjCorres, ...) are the
 * previous frame's LM inliers carried along the refined flow, topped up from the frame's raster samples, plus every sample of a label that
 * is new in this frame (Tracking.cc:2817-2991).  vdo_obj_renew_batch_dev builds that set for P pairs from a vdo_obj_track_batch_dev /
 * vdo_obj_track_set_batch_dev result; vdo_obj_track_set_batch_dev and vdo_obj_update_mask_set_batch_dev read it where the other entries
 * sample the last frame.  A pair's set rows also carry nDynInlierID, the row of the same point in the previous set, from which tracklets
 * are built.  Per frame, with S the set of the previous step (none at the start):
 *   update_mask_set(last planes, S, mask_cur) -> track_set(last planes, current planes, S, prev) -> S' = renew(track result, current planes)
 * A pair with count == -1 has no carried set: the two calls then sample its last frame as vdo_obj_track_batch_dev does (Initialization,
 * Tracking.cc:1215-1276); writing -1 into a pair's count restarts its sequence, as the reset row of prev does.
 *
 * Renewal of pair p (vdo_obj_renew_batch_dev), in the reference's order:
 *   1. for each slot with stat, in slot order, its LM inliers (sample flag 2) in ascending sample row: key x = (int)(float)((double)
 *      sample_x + sample_flow_ref.x), y likewise (mvObjKeys as the tracker updates it); kept when 0 < x < W, 0 < y < H, mask_cur != 0,
 *      0 < depth_cur < 25 (hard-coded, :2849) and (float)x + flow_cur.x, (float)y + flow_cur.y lie strictly inside the image.  Row: the
 *      key, depth_cur, label mask_cur, flow flow_cur, corres (float)x + fx, obj_label the sample's obj_label, inlier_id the sample row.
 *   2. each stat slot with fewer than max_track_obj rows from 1 is topped up from the current frame's raster samples (the sampling of
 *      vdo_obj_motion_batch_dev with step and th_depth_obj on the current planes) whose label is the slot's current label, visited in
 *      passes start = 0 .. 14 of stride 15, skipping a sample on the pixel of any key of 1 (the reference's "closer than 1 px"; both are
 *      integer pixels); the first max_track_obj - (rows from 1) such samples, obj_label the slot's ID, inlier_id -1.
 *   3. every raster label that is not the current label of a stat slot, ascending: all its samples in raster order, obj_label -2,
 *      inlier_id -1.
 *   point = Optimizer::Get3DinWorld(key, depth, K, toInvMatrix(Tcw_cur)), rounded as the tracker rounds it.
 * Equal, bit for bit, to vdo_renew_frame_info (object part) on the same inputs.  More than C rows: the rows past C (in this order) are
 * dropped and VDO_OM_PAIR_FEATURE_CAP is set; the top-up quotas and the pixel test still count every row of step 1.  An i64 current label
 * outside int32 at a raster sample or a kept key sets VDO_OM_PAIR_LABEL_RANGE and the pair gets no set (count -1).
 * The selection runs as a flag pass, per-slot ranks in visit order and a compaction: two launches (k_om_sample on the current planes, then
 * k_rn_select, one CTA per pair), no allocation, host synchronise or pageable host read after the checks, so the call may be captured in
 * a CUDA graph.  The work space is the estimator's (what the RANSAC and the LM leave idle); it does not grow. */
typedef struct vdo_obj_feat_set {     /* caller-allocated DEVICE table; C = the estimator's cap */
  /* per row, P x C (rows past count untouched): */
  int32_t *x_dev, *y_dev;  /* integer pixel (mvObjKeys) */
  int32_t *label_dev;      /* vSemObjLabel */
  float *depth_dev;        /* mvObjDepth */
  float *cx_dev, *cy_dev;  /* mvObjCorres */
  float *flow_dev;         /* x 2: mvObjFlowNext */
  int32_t *inlier_id_dev;  /* nDynInlierID: the row of the same point in the previous set (or raster), -1 for a new point */
  int32_t *obj_label_dev;  /* vObjLabel: the object ID, -2 for a label new in this frame, or the carried sample's label */
  float *point_dev;        /* x 3: mvObj3DPoint, world frame */
  /* per pair, P: */
  int32_t *count_dev;      /* rows, or -1: no carried set (the last frame is sampled) */
  int32_t *status_dev;     /* VDO_OM_PAIR_FEATURE_CAP, VDO_OM_PAIR_LABEL_RANGE */
} vdo_obj_feat_set;
#define VDO_OM_PAIR_FEATURE_CAP 4 /* the renewed set had more than C rows: the last ones (in the order above) are dropped */
#define VDO_OM_PAIR_SET_COUNT 8   /* the set's count lies outside -1 .. C (track / update_mask with a set): the pair has no samples */

/* track_out: the vdo_obj_track_batch_dev / vdo_obj_track_set_batch_dev result of the same P pairs (read only: per slot label, id, stat;
 * per sample x, y, slot, flags, flow_ref, obj_label; n_samples).  depth_cur, flow_cur, mask_cur: P planes of the CURRENT frame (metric
 * depth f32, flow to the NEXT frame f32 with 2 channels, the mask as updated by UpdateMask, i32 or i64) at any strides, of size wh (host
 * P x 2); K: host P x 4; Tcw_cur_dev: device P x 16 or NULL (identity).  step, th_depth_obj: the raster sampling of step 2 and 3.
 * VDO_ERR_ARG before any device work, writing nothing, for: P outside 1 .. max_pairs; a NULL track_out, plane array, wh, K or set_out;
 * a plane of another dtype or channel count; a width or height < 1; step < 1; ceil(w / step) x ceil(h / step) above the cap; th_depth_obj
 * NaN; max_track_obj < 0; any device pointer (planes, Tcw_cur_dev if given, the track_out fields read and every set_out field) NULL,
 * misaligned or foreign. */
int vdo_obj_renew_batch_dev(vdo_obj_motion *m, int P, const vdo_obj_track_out *track_out, const vdo_dev_plane *depth_cur,
                            const vdo_dev_plane *flow_cur, const vdo_dev_plane *mask_cur, const int32_t *wh, const float *K,
                            const float *Tcw_cur_dev, int32_t step, float th_depth_obj, int32_t max_track_obj,
                            const vdo_obj_feat_set *set_out, uint64_t stream);

/* vdo_obj_track_batch_dev with the samples of each pair whose last->count_dev is 0 .. C taken from its set, in row order (x, y, label,
 * depth, cx, cy, flow); "raster order" in that call's rules then means row order.  A pair with count -1 samples its last frame as
 * vdo_obj_track_batch_dev does; any other count sets VDO_OM_PAIR_SET_COUNT and the pair has no samples.  The outputs are the same, so
 * vdo_obj_renew_batch_dev can read them.  Refusals: those of vdo_obj_track_batch_dev, plus a NULL last or a NULL, misaligned or foreign
 * pointer among the set's fields read (x, y, label, depth, cx, cy, flow, count).  The set may not be the one set_out of the renewal this
 * call feeds (it is read here and written there). */
int vdo_obj_track_set_batch_dev(vdo_obj_motion *m, int P, const vdo_dev_plane *depth, const vdo_dev_plane *flow, const vdo_dev_plane *mask,
                                const vdo_dev_plane *depth_cur, const vdo_dev_plane *mask_cur, const int32_t *wh, const float *K,
                                const float *Tcw_last_dev, const float *Tcw_cur_dev, const int32_t *prev_label_dev, const int32_t *prev_id_dev,
                                const int32_t *prev_stat_dev, const float *prev_H_dev, const int32_t *prev_max_id_dev,
                                const vdo_obj_feat_set *last, const vdo_obj_track_opts *opts, const vdo_obj_track_out *out, uint64_t stream);

/* vdo_obj_update_mask_batch_dev with the voters of each pair whose last->count_dev is 0 .. C taken from its set: the rows' (label, cx, cy),
 * the reference's mLastFrame.vSemObjLabel and mvObjCorres.  The recovered pixels are still pushed from the last mask along the last flow
 * (:2997-3068).  count -1: the last frame is sampled as vdo_obj_update_mask_batch_dev does; any other count: VDO_OM_PAIR_SET_COUNT, no
 * voters.  Refusals: those of vdo_obj_update_mask_batch_dev, plus a NULL last or a NULL, misaligned or foreign set field read. */
int vdo_obj_update_mask_set_batch_dev(vdo_obj_motion *m, int P, const vdo_dev_plane *depth, const vdo_dev_plane *flow, const vdo_dev_plane *mask,
                                      const vdo_dev_plane *mask_cur, const int32_t *wh, int32_t step, float th_depth_obj,
                                      const vdo_obj_feat_set *last, const vdo_obj_mask_out *out, uint64_t stream);

/* ---- the camera across frame pairs on the device (Tracking::Track's camera step and the static half of RenewFrameInfo) ----------------
 * The reference does not match descriptors to track the camera.  Its correspondences are the last frame's background features carried
 * along the flow (mCurrentFrame.mvStatKeys = mLastFrame.mvCorres, Tracking.cc:256); its pose is GetInitModelCam (AP3P RANSAC against the
 * constant-velocity model, :1614-1715) refined by PoseOptimizationFlow2Cam (:672-713); and RenewFrameInfo carries the inliers into the next
 * frame and tops them up (:2663-2814).  A vdo_cam_motion estimator runs that chain for up to 64 pairs per call from a carried background
 * set (vdo_stat_feat_set), which also holds the frame's pose and the velocity.  Per frame, with S the set of the previous step:
 *   build(last keys and planes, S)            fills the pairs whose count is -1 (a sequence start or restart) and leaves the others
 *   cam = cam_track(S)                        the current pose T; the object calls take S.Tcw as Tcw_last and cam.T as Tcw_cur
 *   S' = stat_renew(S, cam, current keys and planes)
 * Every entry refuses with VDO_ERR_ARG (the reason in vdo_last_error) before any device work, writing nothing; after its checks it does not
 * allocate, synchronise the host or read pageable host memory, so the whole step may be captured in one CUDA graph, and a replay uses the
 * captured call's host parameters (K, planes, options).  Calls on one estimator must be ordered. */
typedef struct vdo_cam_motion vdo_cam_motion;
#define VDO_CAM_MOTION_MAX_PAIRS 64
#define VDO_CAM_MOTION_MAX_ITERS 500
/* max_pairs 1 .. 64, cap >= 1 (rows of a pair's set; max_pairs x cap below 2^31).  A cap above VDO_FLOW2_CLUSTER_MAX_N also allocates the
 * single-CTA LM scratch, max_pairs x cap x 144 bytes. */
int vdo_cam_motion_create(vdo_ctx *ctx, int max_pairs, int cap, vdo_cam_motion **out);
void vdo_cam_motion_destroy(vdo_cam_motion *m);
/* out: max_pairs, cap, VDO_CAM_MOTION_MAX_ITERS, device bytes held */
int vdo_cam_motion_info(const vdo_cam_motion *m, int64_t out[4]);

typedef struct vdo_stat_feat_set {    /* caller-allocated DEVICE table, the reference's mLastFrame background state; C = the estimator's cap */
  /* per row, P x C (rows past count untouched): */
  float *x_dev, *y_dev;    /* mvStatKeysTmp (sub-pixel) */
  float *depth_dev;        /* mvStatDepthTmp */
  float *cx_dev, *cy_dev;  /* mvCorres */
  float *flow_dev;         /* x 2: mvFlowNext */
  int32_t *inlier_id_dev;  /* nStaInlierID: the row of the same point in the previous set, -1 for a new point */
  float *point_dev;        /* x 3: mvStat3DPointTmp (camera frame after a build, world frame after a renewal) */
  /* per pair, P: */
  int32_t *count_dev;      /* rows, or -1: no set yet (build fills it) */
  int32_t *status_dev;     /* VDO_CAM_* bits of the call that wrote the set */
  float *Tcw_dev;          /* x 16: the frame's mTcw */
  float *velocity_dev;     /* x 16: mVelocity */
  int32_t *has_velocity_dev; /* 0: the reference's empty mVelocity (the first pair's motion model is Tcw itself) */
} vdo_stat_feat_set;
#define VDO_CAM_FEW_POINTS 1  /* cam_track: fewer than 4 rows, no RANSAC */
#define VDO_CAM_NO_MODEL 2    /* cam_track: 4 or more rows, no hypothesis with more than 3 inliers */
#define VDO_CAM_USED_MM 4     /* cam_track: the constant-velocity model was chosen */
#define VDO_CAM_SET_COUNT 8   /* a set count outside its range (cam_track: 0 .. C; stat_renew: -1 .. C, or the cam output's bit): no rows */
#define VDO_CAM_KEY_COUNT 16  /* a key set count outside 0 .. its cap: taken as 0 */

typedef struct vdo_stat_opts {
  float th_depth_bg;           /* ThDepthBG of the build (40); the renewal's carried rows use the reference's hard-coded 40 */
  int32_t max_track_bg;        /* MaxTrackPointBG of the renewal, 0 .. cap - 1 (1200) */
  int32_t use_sample_feature;  /* 0: option I, keys are ORB keypoints; 1: option II, keys are sampled (vdo_sample_keys_dev) */
  int32_t pad;
} vdo_stat_opts;

/* Frame::Frame's static set (Frame.cc:100-194) of the pairs whose set count is -1; the other pairs are not touched, so the call can sit in
 * every step of a captured graph.  keys: the LAST frames' key set (frame p for pair p; x, y and count are read, desc is not): ORB keypoints
 * for option I, sampled keys for option II.  depth, flow, mask: P planes of the LAST frames (metric depth f32, flow to the current frame f32
 * with 2 channels HWC or CHW, mask i32 or i64) at any strides, of size wh (host P x 2); K: host P x 4.  gate_count_dev: option II only, device
 * P int32, the frames' ORB keypoint counts: a frame with none gets an empty set (Frame.cc:97-98); NULL with option I.
 * Rows, in key order: the keys with mask == 0, 0 < depth <= th_depth_bg, both flow components non-zero and the target (x + fx, y + fy)
 * inside the image -- option I by the far edges only (key and target < W, H), option II on both sides (frame_px.cuh static_key, the rule of
 * vdo_frame_filter_static); a key whose pixel lies outside the image is dropped.  Row: the key, depth, corres (x + fx, y + fy), flow,
 * inlier_id -1, point = Get3DinCamera (Initialization, Tracking.cc:1219-1227).  Pair: count, status (0 or VDO_CAM_KEY_COUNT), Tcw = I,
 * velocity = I, has_velocity = 0.  One launch (k_sb_build, one CTA per pair).
 * VDO_ERR_ARG for: P outside 1 .. max_pairs; a NULL keys, plane array, wh, K, opts or set; keys.n_frames < P or keys.cap outside 1 .. C
 * (the set cannot overflow); a plane of another dtype or channel count; a width or height < 1; th_depth_bg NaN; use_sample_feature not 0
 * or 1; gate_count_dev NULL with option II; any device pointer read or written NULL, misaligned or foreign. */
int vdo_stat_build_batch_dev(vdo_cam_motion *m, int P, const vdo_orb_desc_set *keys, const vdo_dev_plane *depth, const vdo_dev_plane *flow,
                             const vdo_dev_plane *mask, const int32_t *wh, const float *K, const int32_t *gate_count_dev,
                             const vdo_stat_opts *opts, const vdo_stat_feat_set *set, uint64_t stream);

typedef struct vdo_cam_track_opts {
  int32_t iters;          /* RANSAC iterations, 1 .. VDO_CAM_MOTION_MAX_ITERS (500) */
  int32_t quirk;          /* 0 or 1, as vdo_pose_opt_flow2 (1) */
  double thr, conf;       /* reprojection threshold > 0 (0.4) and confidence in (0, 1) (0.98) */
} vdo_cam_track_opts;

typedef struct vdo_cam_track_out {    /* caller-allocated DEVICE outputs; C = the estimator's cap */
  /* per pair, P: */
  float *T_dev;           /* x 16: the current mTcw */
  float *T_init_dev;      /* x 16: GetInitModelCam's model */
  float *velocity_dev;    /* x 16: mVelocity = T * Tcw^-1 */
  int32_t *info_dev;      /* x 8: rows n, n_ransac, n_mm, used_mm, n_sub, iterations run, winning iteration, valid minimal solves */
  double *stats_dev;      /* x 8: vdo_pose_opt_flow2's stats; [0] = -1 without the LM */
  int32_t *status_dev;    /* VDO_CAM_FEW_POINTS, _NO_MODEL, _USED_MM, _SET_COUNT */
  /* per row, P x C (rows past the set's count untouched): */
  uint8_t *flags_dev;     /* 1: in the chosen set, 2: LM inlier, 4: still in TemperalMatch_subset */
  float *key_dev;         /* x 2: the current frame's mvStatKeys */
  double *flow_ref_dev;   /* x 2: the LM's refined flow for a row in the LM problem, the set's flow otherwise */
} vdo_cam_track_out;

/* The camera step (Tracking.cc:672-713, tracker.cpp track_frames) from the sets alone.  Row i of pair p: the world point
 * UnprojectStereoStat(x, y, depth) through the set's Tcw (rounded as the tracker rounds it), observed at (cx, cy); the motion model is
 * velocity * Tcw (cv::Mat float gemm) when has_velocity, else Tcw.  GetInitModelCam as vdo_init_model_batch with that model; when the chosen
 * set has at least 3 rows, PoseOptimizationFlow2Cam (vdo_pose_opt_flow2 mode 0, quirk) on its (x, y), depth and flow from T_init, giving T
 * (else T = T_init).  An LM inlier's key is (float)((double)x + refined flow); every other row keeps (cx, cy).  Rows the LM rejects leave
 * TemperalMatch_subset.  velocity = T * toInvMatrix(Tcw).  Equal, bit for bit, to vdo_init_model_batch + vdo_pose_opt_flow2_batch on the
 * same rows.  Launches: k_ct_gather, the RANSAC kernels, k_ct_lm_prep, the LM, k_ct_finish.
 * VDO_ERR_ARG for: P outside 1 .. max_pairs; a NULL set, K, opts or out; iters outside 1 .. 500; thr <= 0; conf outside (0, 1); quirk not 0
 * or 1; any set field read or output NULL, misaligned or foreign. */
int vdo_cam_track_batch_dev(vdo_cam_motion *m, int P, const vdo_stat_feat_set *set, const float *K, const vdo_cam_track_opts *opts,
                            const vdo_cam_track_out *out, uint64_t stream);

/* The static half of RenewFrameInfo (Tracking.cc:2663-2814): the next set from the last set and the vdo_cam_track_batch_dev result of the
 * same pairs.  keys: the CURRENT frames' key set (frame p for pair p): ORB keypoints (mvKeys) for option I, the raw sampled keys for option
 * II.  depth, flow, mask: the CURRENT frames' metric depth, flow to the NEXT frame and mask as UpdateMask left it, of size wh (the
 * reference runs UpdateMask before it builds the frame, so its option-II list is filtered with the updated mask too).
 *   1. carried: the rows with flag 4 in row order, key = cam.key; kept when 0 < (int)x < W, 0 < (int)y < H, mask == 0, 0 < depth <= 40
 *      (hard-coded), both flow components non-zero and the target strictly inside; the size test comes after the push and uses '>', so up to
 *      max_track_bg + 1 rows are carried.  inlier_id: the row.
 *   2. top-up, while fewer than max_track_bg rows are held: the top-up list is the key set (option I), or the keys that pass the build's
 *      option-II rule with th_depth_bg (option II; none when gate_count_dev[p] is 0), visited in passes start = 0 .. 19 of stride 20 over the
 *      list; a candidate closer than 1 px to any carried key (float sqrt of float squares) is skipped, the others take the rule of 1; the
 *      first max_track_bg - carried of them, inlier_id -1.
 *   Row: key, depth, corres key + flow, flow, point = Get3DinWorld(key, depth, K, toInvMatrix(T)).  Pair: count, status, Tcw = cam.T,
 *   velocity = cam.velocity, has_velocity = 1.
 * Equal, bit for bit, to vdo_renew_frame_info's static part on the same inputs.  One launch (k_sr_select, one CTA per pair: flag passes,
 * ranks in visit order, a compaction).  The last set and set_out must be different tables.
 * VDO_ERR_ARG for: everything vdo_stat_build_batch_dev refuses that applies; a NULL last or cam; max_track_bg < 0 or max_track_bg + 1 > C;
 * any set field or cam field read NULL, misaligned or foreign. */
int vdo_stat_renew_batch_dev(vdo_cam_motion *m, int P, const vdo_stat_feat_set *last, const vdo_cam_track_out *cam, const vdo_orb_desc_set *keys,
                             const vdo_dev_plane *depth, const vdo_dev_plane *flow, const vdo_dev_plane *mask, const int32_t *wh, const float *K,
                             const int32_t *gate_count_dev, const vdo_stat_opts *opts, const vdo_stat_feat_set *set_out, uint64_t stream);

/* vdo_sample_keys on the device: frame i's VDO_SAMPLE_KEYS keys from cv::RNG(seeds_dev[i]) into row i of x_dev / y_dev (n x
 * VDO_SAMPLE_KEYS f32) and count_dev[i] = VDO_SAMPLE_KEYS, a layout a vdo_orb_desc_set of cap VDO_SAMPLE_KEYS can point at.  The seeds are
 * read on the device, so a replayed graph draws frame f_id's keys from cv::RNG(sample_seed + f_id) once the caller advances them.  One
 * launch on `stream`.  VDO_ERR_ARG for n outside 1 .. 65535, a width or height < 20, or a pointer NULL, misaligned or foreign. */
int vdo_sample_keys_dev(vdo_ctx *ctx, int n, const uint32_t *seeds_dev, int width, int height, float *x_dev, float *y_dev, int32_t *count_dev,
                        uint64_t stream);

/* ---- tracking bookkeeping (SURVEY.md 8 rows A13, A15, A16) -----------------------------------------------------------
 * vdo_tracklets_build  <- Tracking::GetStaticTrack / GetDynamicTrackNew (src/Tracking.cc:2201-2307, 2309-2421).
 *   Row i (0-based, i = frame pair id) holds row_begin[i+1]-row_begin[i] features of frame i+1; assoc[k] is the index of the
 *   same feature in frame i's row (Map::vnAssoSta / vnAssoDyn), -1 = no correspondence; labels (NULL for the static map) is
 *   Map::vnFeatLabel (the dynamic-object id of the feature).  Tracklets come out in the reference's creation order as CSR:
 *   entry e of tracklet t is (trk_frame[e], trk_feat[e]) = TrackLets[t][.] = (frame id, feature id); obj_id[t] = ObjLab[t].
 *   Host-only (no device work).  Returns VDO_ERR_ARG (with *n_trk set) when max_tracklets / max_entries are too small. */
int vdo_tracklets_build(int n_rows, const int *row_begin, const int *assoc, const int *labels, int max_tracklets, int max_entries,
                        int *n_trk, int *trk_begin, int *trk_frame, int *trk_feat, int *obj_id);
/* vdo_update_mask  <- Tracking::UpdateMask (src/Tracking.cc:2997-3110).  cur / last are resident frames (mask of both, flow of
 *   last).  sem_label_last / corres_x / corres_y are the last frame's vSemObjLabel and mvObjCorres (n object points).  The
 *   current mask is updated in place on the device; mask_out (h*w int, may be NULL) receives it (the caller's mSegMap);
 *   warped_labels (may be NULL, sized for the number of distinct labels) lists the objects whose mask was recovered. */
int vdo_update_mask(vdo_frame *cur, vdo_frame *last, int n, const int *sem_label_last, const float *corres_x, const float *corres_y,
                    int *mask_out, int *n_warped, int *warped_labels);
/* vdo_dyn_obj_tracking  <- Tracking::DynObjTracking (src/Tracking.cc:1366-1612; ground-truth bookkeeping :1531-1544 excluded).
 *   n object points of the current frame: sem_label (vSemObjLabel), obj_label (vObjLabel, in/out), kx/ky (mvObjKeys),
 *   depth (mvObjDepth), flow3d (vFlow_3d, n x 3), sem_label_last (mLastFrame.vSemObjLabel); the last frame's object table
 *   (nSemPosition, bObjStat, nModLabel); rows/cols of the image, shrink_row/col (25/50 for KITTI, 0 otherwise),
 *   sf_mg_thres / sf_ds_thres / th_depth_obj (fSFMgThres, fSFDsThres, mThDepthObj), f_id and max_id (in/out).
 *   Outputs: the kept objects as CSR over point indices (return value ObjIdNew), mod_label (nModLabel), sem_position
 *   (nSemPosition). */
int vdo_dyn_obj_tracking(vdo_ctx *ctx, int n, const int *sem_label, int *obj_label, const float *kx, const float *ky, const float *depth,
                         const float *flow3d, const int *sem_label_last, int n_last_obj, const int *last_sem_position,
                         const unsigned char *last_obj_stat, const int *last_mod_label, int rows, int cols, int shrink_row, int shrink_col,
                         float sf_mg_thres, float sf_ds_thres, float th_depth_obj, int f_id, int *max_id, int max_objects,
                         int *n_objects, int *obj_begin, int *obj_idx, int *mod_label, int *sem_position);

/* vdo_renew_frame_info  <- Tracking::RenewFrameInfo (src/Tracking.cc:2660-2995).  `cur` holds the current images (prepared depth,
 *   updated mask, flow).  Static part: tm_sta (TM_sta = TemperalMatch_subset after Flow2Cam, -1 = outlier) indexes stat_keys
 *   (mCurrentFrame.mvStatKeys, n_stat x 2); samp_keys (n_samp x 2) is mvKeys (ORB) or mvStatKeysTmp (nUseSampleFea == 1);
 *   max_num_sta = nMaxTrackPointBG.  Object part: inl_begin / inl_idx = vnObjInlierID (CSR over n_obj objects), obj_stat =
 *   bObjStat, sem_position = nSemPosition, mod_label = nModLabel, obj_keys / obj_label = mvObjKeys / vObjLabel (n_objkeys),
 *   tmp_* = this frame's fresh semi-dense samples (mvTmpObjKeys, mvTmpObjDepth, mvTmpSemObjLabel, mvTmpObjFlowNext, mvTmpObjCorres;
 *   n_tmp), max_num_obj = nMaxTrackPointOBJ.  K4 = fx, fy, cx, cy; Twc = Converter::toInvMatrix(mTcw), 4x4 row-major f32.
 *   Outputs (caller-allocated, capacities cap_sta / cap_obj): static mvStatKeysTmp, mvCorres, mvFlowNext, nStaInlierID,
 *   mvStatDepthTmp, mvStat3DPointTmp; objects mvObjKeys, mvObjDepth, mvObjCorres, mvObjFlowNext, vSemObjLabel, nDynInlierID,
 *   vObjLabel, mvObj3DPoint.  The depth limits 40 / 25 are hard-coded like in the reference (:2691, :2849). */
int vdo_renew_frame_info(vdo_frame *cur, int n_tm, const int *tm_sta, int n_stat, const float *stat_keys, int n_samp, const float *samp_keys,
                         int max_num_sta, int n_obj, const int *inl_begin, const int *inl_idx, const unsigned char *obj_stat,
                         const int *sem_position, const int *mod_label, int n_objkeys, const float *obj_keys, const int *obj_label, int n_tmp,
                         const float *tmp_keys, const float *tmp_depth, const int *tmp_sem, const float *tmp_flow, const float *tmp_corres,
                         int max_num_obj, const float *K4, const float *Twc, int cap_sta, int *n_sta_out, float *sta_keys, float *sta_corres,
                         float *sta_flow, int *sta_inlier_id, float *sta_depth, float *sta_3d, int cap_obj, int *n_obj_out, float *o_keys,
                         float *o_depth, float *o_corres, float *o_flow, int *o_sem, int *o_inlier_id, int *o_label, float *o_3d);

/* depth and mask label at the truncated pixel of each key (x, y interleaved, n x 2 f32); 0 / 0 outside the image.  The
 * "update current frame from last" look-ups of Tracking::GrabImageRGBD (src/Tracking.cc:262-312). */
int vdo_frame_gather(vdo_frame *f, int n, const float *keys, float *depth_out, int *mask_out);
int vdo_frame_read_mask(vdo_frame *f, int *mask_out);   /* D2H of the resident (possibly updated) semantic mask */

/* ------------------------------------------------------------------------------------------------
 * Whole per-frame path: System::TrackRGBD -> Tracking::GrabImageRGBD -> Tracking::Track (include/System.h:49-51,
 * src/Tracking.cc:164-648, 650-1212) sequenced over the stages above, with the per-frame state of `Frame` and the slice of `Map`
 * the batch optimisers read kept inside the tracker.  Settings mirror the YAML keys Tracking::Tracking reads
 * (src/Tracking.cc:57-162; defaults = example/kitti-0000-0013.yaml).
 * ------------------------------------------------------------------------------------------------ */
typedef struct vdo_tracker vdo_tracker;
typedef struct vdo_tracker_params {
  int width, height;                 /* Camera.width / Camera.height */
  float fx, fy, cx, cy;              /* Camera.fx .. */
  float bf, depth_factor;            /* Camera.bf, DepthMapFactor */
  float th_depth_bg, th_depth_obj;   /* ThDepthBG, ThDepthOBJ */
  int max_track_bg, max_track_obj;   /* MaxTrackPointBG, MaxTrackPointOBJ */
  float sf_mg_thres, sf_ds_thres;    /* SFMgThres, SFDsThres */
  int n_features; float scale_factor; int n_levels, ini_th_fast, min_th_fast;   /* ORBextractor.* */
  int is_kitti;                      /* mTestData == KITTI: boundary shrink 25 / 50 px (src/Tracking.cc:1405-1409) */
  int quirk;                         /* see vdo_pose_opt_flow2 */
  int window_size, overlap_size;     /* WINDOW_SIZE, OVERLAP_SIZE */
  int local_batch;                   /* bLocalBatch: run PartialBatchOptimization inside vdo_tracker_track on the reference's schedule
                                        ((f_id - OVERLAP + 1) % (WINDOW - OVERLAP) == 0 && f_id >= WINDOW - 1, src/Tracking.cc:1150-1160) */
  int dataset;                       /* ChooseData / mTestData (src/Tracking.cc:150-160): 1 OMD, 2 KITTI, 3 VirtualKITTI; 0 = KITTI when is_kitti else OMD.
                                        OMD and KITTI convert the raw disparity to depth (bf / (d / factor)); VirtualKITTI only clamps negatives
                                        to 0 (src/Tracking.cc:180-204) */
  int use_sample_feature;            /* UseSampleFeature: 0 static keys from the ORB keypoints (option I, src/Frame.cc:100-129); 1 from
                                        Frame::SampleKeyPoints (option II, :130-168, vdo_sample_keys), and RenewFrameInfo tops the static set up
                                        from them (src/Tracking.cc:2718-2721).  ORB still runs: a frame without keypoints gets no keys. */
  unsigned sample_seed;              /* with use_sample_feature: frame f_id draws from cv::RNG((uint32)(sample_seed + f_id)) -- the reference run
                                        whose time(NULL) read sample_seed + f_id at frame f_id */
} vdo_tracker_params;
void vdo_tracker_params_default(vdo_tracker_params *p);
/* VDO_ERR_ARG (reason in vdo_last_error) for ORB settings vdo_orb_extractor_create refuses with VDO_ERR_ARG, such as a pyramid level
 * under 1 px; its VDO_ERR_UNSUPPORTED limits are reported by the first tracking call (see vdo_tracker_track). */
int vdo_tracker_create(vdo_ctx *ctx, const vdo_tracker_params *params, vdo_tracker **out);
void vdo_tracker_destroy(vdo_tracker *t);
const char *vdo_tracker_last_error(const vdo_tracker *t);
/* One frame.  gray: h x w u8; depth: h x w f32 raw disparity*factor as example/vdo_slam.cc passes it -- when writeback != 0 it is
 * overwritten with metric depth like the reference does to the caller's cv::Mat (src/Tracking.cc:180-204); flow: h x w x 2 f32;
 * mask: h x w i32 -- when writeback != 0 it receives the propagated labels (UpdateMask, :3062).  gt_sem_ids: semantic ids that have a
 * ground-truth object pose in this frame (vObjPose_gt[i][1]); the reference only estimates motion for objects present in the
 * ground truth of both frames (:767-810).  Tcw_out: 4x4 row-major f32 = the returned mCurrentFrame.mTcw.
 * width / height: size of the four buffers; VDO_ERR_ARG unless they equal the tracker's (the buffers are read -- and with writeback
 * written -- as width x height arrays).  The frame build runs on a vdo_orb_extractor cached per context stream, size and ORB settings
 * (grown to the largest batch, at most 64 frames per call), so ORB settings vdo_orb_extractor_create refuses are refused here with its
 * code, before the tracker's state changes. */
int vdo_tracker_track(vdo_tracker *t, int width, int height, const unsigned char *gray, float *depth, const float *flow, int *mask, int n_gt,
                      const int *gt_sem_ids, int writeback, float *Tcw_out);
/* vdo_tracker_track on device-resident inputs (see vdo_dev_plane and vdo_frame_upload_dev for the accepted planes and the stream
 * rule); all four planes are required, and the image may be colour.  The result is bit for bit the one vdo_tracker_track gives for
 * the same gray / depth / flow / mask.  writeback != 0: the prepared depth is scattered into the depth plane and, when UpdateMask
 * changed it, the propagated mask into the mask plane (i32 or i64), on the device and at their strides; both must then have
 * non-zero stride_x and stride_y.  Everything that can be refused is checked before the tracker's state changes, including the
 * device-side label-range check: a refused frame leaves the tracker as it was, and the next call tracks as if it never came.
 * The call synchronises the context stream before it returns; then the write-back is visible to every stream. */
int vdo_tracker_track_dev(vdo_tracker *t, int width, int height, const vdo_dev_plane *image, const vdo_dev_plane *depth,
                          const vdo_dev_plane *flow, const vdo_dev_plane *mask, int n_gt, const int *gt_sem_ids, int writeback,
                          uint64_t stream, float *Tcw_out);
/* n trackers advanced by one frame each: tracker i gets exactly what vdo_tracker_track_dev(trackers[i], ...) gives it, bit for bit
 * (per-frame state, written-back depth and mask, the map, windowed optimisations, Tcw_out + 16 i), but each batched stage does the device
 * work of all n frames as one set of launches with one synchronise: ingest + depth prep, the frame build (the ORB extractor in chunks of
 * at most 64 frames, static filter, object samples), the key look-ups, the camera's initial model and flow LM, the scene flow, and the objects' initial
 * models and flow LM.  UpdateMask, DynObjTracking, RenewFrameInfo, the map push and the windowed optimisation run per tracker.
 * images / depths / flows / masks: n planes each, with the plane and stream rules of vdo_tracker_track_dev.  gt_begin: n + 1 offsets
 * from 0; the ground-truth semantic ids of tracker i are gt_ids[gt_begin[i] .. gt_begin[i + 1]).  Trackers may be at different points of
 * their sequences (one on its first frame, others mid-sequence) and may differ in intrinsics, bf, depth_factor, thresholds, dataset,
 * window settings, quirk, use_sample_feature and sample_seed.  They must be distinct, non-NULL, on one context, and share width, height and the ORB settings
 * (n_features, scale_factor, n_levels, ini_th_fast, min_th_fast): VDO_ERR_ARG otherwise, VDO_ERR_STATE for a map-only handle.  A refused
 * call -- including a device-side label-range refusal of any one frame -- leaves every tracker unchanged and writes nothing back;
 * vdo_tracker_last_error(trackers[0]) names the offending index.  stage_ms of each tracker accumulates the wall time of every batched
 * stage it took part in. */
int vdo_tracker_track_batch_dev(vdo_tracker *const *trackers, int n, const vdo_dev_plane *images, const vdo_dev_plane *depths,
                                const vdo_dev_plane *flows, const vdo_dev_plane *masks, const int *gt_begin, const int *gt_ids,
                                int writeback, uint64_t stream, float *Tcw_out);
/* vdo_tracker_track_batch_dev for trackers that may also differ in width, height and the ORB settings (KITTI and OMD sequences, the
 * cameras of one vehicle): the same arguments, checks, guarantees and launches, and each plane is checked against its own tracker's
 * size.  Every per-frame table carries its frame's geometry, so frames of different sizes and settings share each launch, and one
 * 64-frame extractor chunk may hold several geometries.  ORB settings that vdo_orb_extractor_create refuses for any one tracker refuse
 * the call (with its code; the error names the tracker) before any tracker changes.  On trackers of one geometry it is
 * vdo_tracker_track_batch_dev. */
int vdo_tracker_track_mixed_dev(vdo_tracker *const *trackers, int n, const vdo_dev_plane *images, const vdo_dev_plane *depths,
                                const vdo_dev_plane *flows, const vdo_dev_plane *masks, const int *gt_begin, const int *gt_ids,
                                int writeback, uint64_t stream, float *Tcw_out);
/* Named read-back of the frame state after the last call ('f' arrays are f32, the others i32; out may be NULL to query the size):
 * Tcw mVelocity mvKeys mvStatKeysTmp mvStatDepthTmp mvCorres mvFlowNext mvStat3DPointTmp nStaInlierID mvObjKeys mvObjDepth
 * mvObjCorres mvObjFlowNext mvObj3DPoint vSemObjLabel vObjLabel nDynInlierID vFlow_3d nModLabel nSemPosition bObjStat vObjMod
 * vObjCentre3D TemperalMatch_subset max_id f_id; stage_ms (9 x f32, accumulated host wall-clock per stage since creation: upload+depth, mask,
 * frame build (ORB + static filter + object samples), look-ups, initial camera model, camera LM, objects, renewal, windowed BA);
 * local_ba (2 x i32: windowed optimisations run, their LM iterations) */
int vdo_tracker_get(const vdo_tracker *t, const char *name, void *out, int cap_elems, int *n_elems);

/* Map -> factor graph -> optimise -> write back (SURVEY.md 8f N2): mode 0 = Optimizer::PartialBatchOptimization(pMap, K, WINDOW_SIZE)
 * (src/Optimizer.cc:42-1230) over the last window_size frames, mode 1 = Optimizer::FullBatchOptimization(pMap, K) (:1232-2175),
 * on the map the tracker accumulated (Tracking.cc:1016-1070).  opt may be NULL (the reference's optimize(100 | 300) and gain
 * thresholds 1e-3 | 1e-4).  info (may be NULL, 6 ints): vertices se3 / point, edges prior / se3 / point-observation / landmark-motion. */
int vdo_tracker_batch_optimize(vdo_tracker *t, int mode, const vdo_lm_options *opt, vdo_lm_stats *stats, int *info);
/* vdo_tracker_batch_optimize of n trackers in one call (e.g. FullBatchOptimization at the end of n sequences): one graph build over the
 * list, one vdo_graph_optimize_batch of all the graphs, and the write-back into each map.  Tracker i ends where
 * vdo_tracker_batch_optimize(ts[i], mode, opt, ...) takes it.  Map-only handles are accepted.  opt may be NULL (the mode's reference
 * options, as above); stats: n entries, info: n x 6 ints (either may be NULL).  VDO_ERR_ARG: n < 1, a NULL or repeated tracker, trackers
 * on different contexts, mode not 0 / 1.  VDO_ERR_STATE: a map too short for the mode.  Every refusal happens before any work and changes
 * no tracker; the message is on ts[0] (vdo_tracker_last_error). */
int vdo_tracker_batch_optimize_batch(vdo_tracker *const *ts, int n, int mode, const vdo_lm_options *opt, vdo_lm_stats *stats, int *info);
/* test hook: the arrays the builder passes to vdo_graph_* for a mode.  f64 names: se3 pt prior_Z prior_w se3e_Z se3e_w se3e_delta
 * obs_z obs_w obs_delta ter_w ter_delta; i32 names: prior_v se3e_ij obs_cp ter_pph.  out may be NULL to query the element count. */
int vdo_tracker_graph_export(vdo_tracker *t, int mode, const char *name, void *out, int cap_elems, int *n_elems);
/* map read-back (include/Map.h:34-84): vmCameraPose / vmCameraPose_RF (n_frames x 16 f32: the windowed BA refines the first, the full
 * batch the second, src/Optimizer.cc:1058-1101 / :2094-2133), vmRigidMotion / vmRigidMotion_RF (every frame's motions concatenated, 16 f32
 * each, entry 0 = camera motion), vmRigidCentre (3 f32 each, same order), vnRMLabel (i32, same order), n_per_frame (entries per frame,
 * i32), n_frames (i32) */
int vdo_tracker_map_get(const vdo_tracker *t, const char *name, void *out, int cap_elems, int *n_elems);
/* test hook: the tracklet tables the graph builder reads, kind 0 static / 1 dynamic, i32.  Per feature (frames concatenated, frame 0 included):
 * trk (tracklet, -1 none), pos (position in it), prev_frame / prev_feat (the entry before it); per tracklet: len, head_frame, head_feat,
 * obj_lab (dynamic only: the label of the feature that opened it).  out may be NULL to query the element count. */
int vdo_tracker_tracklets_get(vdo_tracker *t, int kind, const char *name, void *out, int cap_elems, int *n_elems);
/* Externally built maps -- the input of Optimizer::FullBatchOptimization(Map*, K) / PartialBatchOptimization(Map*, K, WINDOW_SIZE)
 * (include/Optimizer.h:29-30): create a handle with params.width == params.height == 0 (intrinsics, window_size and overlap_size are used),
 * push the Map frame by frame, run vdo_tracker_batch_optimize and read vmCameraPose[_RF] / vmRigidMotion[_RF] / vp3DPointSta / vp3DPointDyn
 * (xyz per feature, all frames concatenated) back with vdo_tracker_map_get.  Frame 0: n_mot = 0, asso / label arrays ignored. */
int vdo_tracker_map_push(vdo_tracker *t, int n_sta, const float *feat_sta, const float *dep_sta, const float *p3d_sta, const int *asso_sta, int n_dyn,
                         const float *feat_dyn, const float *dep_dyn, const float *p3d_dyn, const int *asso_dyn, const int *feat_label,
                         const float *camera_pose16, int n_mot, const float *rigid_motion16, const int *rm_label);

/* Measurement hook (bench.py roofline): runs one kernel (or kernel group) of the batch path `reps` times back to back
 * on the context stream between two CUDA events, after one untimed warm-up launch, and returns the average in ms.
 * The graph must have been optimised at least once (buffers hold a valid linearisation / factorisation).
 * names: "lin_tracklets" "chi2_tracklets" "lin_vertex_obs" "lin_vertex_ter" "lin_se3_edges" "linearize" (all four)
 *        "factor_landmarks" "precond" (assembly + PCR factorisation) "schur_landmarks" "schur_vertex_obs"
 *        "schur_vertex_ter" "hpp_mul" "pcg_dot" "pcg_step" "pcg_iterate8" (8 PCG iterations as launched in a solve)
 *        "schur_static" "schur_chains" "lin_static" "lin_chains" (the two halves of the landmark passes) "pcg_step_a" */
int vdo_graph_time_kernel(vdo_graph *g, const char *name, int reps, float *ms_avg);

#ifdef __cplusplus
}
#endif
#endif
