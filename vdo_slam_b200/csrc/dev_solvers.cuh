// dev_solvers.cuh -- the problem layouts of the two per-frame solvers and internal launchers that run them on problems already resident on
// the device, in the style of frame_batch.h: the RANSAC + initial-model kernels of pnp_ransac.cu (k_pnp_samples, k_pnp_hyp, k_pnp_score,
// k_pnp_finish) and the flow / pose LM kernels of flow_lm.cu (k_refine_lm_cl, k_refine_lm).  The kernels stay where they are; a caller in
// another file (obj_motion.cu) writes the problems and launches them through these functions.
#pragma once
#include <cuda_runtime.h>

namespace vdo {

// ---- pnp_ransac.cu: one RANSAC / initial-model problem ----
struct PnpProb {
  int off, n;          // the problem's points: obj / img [off, off + n)
  double K[4];
  float Kf[4];
  float mm[12];        // motion model, rows of [R|t]
  int has_mm;
  int pad;
};
struct PnpOut {         // per problem
  double Rt[12];        // refitted RANSAC model
  double Rt_hyp[12];    // winning hypothesis
  float T[16];          // chosen initial model, 4x4 row-major
  int n_ransac, n_mm, used_mm, n_sub, iters_run, best_it, n_valid, pad;
};
// the sample tables of nprob problems whose n is on the device (k_pnp_samples; samples: nprob x iters x 4)
void pnp_samples_launch(const PnpProb* prob, int nprob, int iters, int* samples, cudaStream_t st);
// hypotheses, scores and the initial model of nprob problems (k_pnp_hyp, k_pnp_score, k_pnp_finish); models: nprob x iters x 12,
// counts: nprob x iters; r_idx / m_idx / s_idx: the RANSAC, motion-model and chosen inlier sets, local indices at each problem's off
void pnp_ransac_launch(const PnpProb* prob, int nprob, const float* obj, const float* img, const int* samples, int iters, double thr, double conf,
                       double* models, int* counts, PnpOut* out, int* r_idx, int* m_idx, int* s_idx, cudaStream_t st);

// ---- flow_lm.cu: one joint flow / SE(3) LM problem ----
struct FlowProb {
  int mode, n, offset;
  int out;                           // the problem's index in the caller's batch (T_out, stats, trace)
  float K[4];
  float Tcw_last[16];
  float T_init[16];
};
struct FlowDev {
  const FlowProb* prob;
  const float *pts, *depth, *flow;   // inputs, concatenated over problems
  double* scratch;                   // per point FL_FIELDS doubles (single-CTA shape)
  float* T_out;                      // nprob x 16
  double* flow_out;                  // total x 2
  unsigned char* inlier;             // total
  double* stats;                     // nprob x 8
  int quirk;
  int debug;
  double* trace;                     // nprob x VDO_FLOW2_TRACE_DOUBLES, or NULL (no trace work)
};
// doubles of single-CTA scratch per point (d.scratch holds them for every point of a problem that may exceed VDO_FLOW2_CLUSTER_MAX_N)
int flow_lm_fields();
// allows the cluster kernel its shared memory; once per process before flow_lm_launch
cudaError_t flow_lm_prepare();
// the nprob problems of d.prob, whose n is on the device and at most max_n: the cluster kernel over all of them (points per CTA sized from
// min(max_n, VDO_FLOW2_CLUSTER_MAX_N)) and, when max_n > VDO_FLOW2_CLUSTER_MAX_N, the single-CTA kernel over all of them; each problem
// runs on the one its own n selects (k_refine_lm_cl / k_refine_lm)
void flow_lm_launch(const FlowDev& d, int nprob, int max_n, cudaStream_t st);

}  // namespace vdo
