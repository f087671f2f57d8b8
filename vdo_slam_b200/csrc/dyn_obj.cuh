// dyn_obj.cuh -- the per-object rule of Tracking::DynObjTracking (src/Tracking.cc:1372-1599), shared by vdo_dyn_obj_tracking (tracking_ops.cu,
// per-object sums on the device, decisions on the host) and vdo_obj_track_batch_dev (obj_motion.cu, all on the device), so that both classify
// with the same float rounding: the sums run in point order, one point at a time.
#pragma once
#include <cuda_runtime.h>

namespace {

struct ObjStat { float boundary, sf_count, depth_sum; int n; };

// point i (kx, ky, depth, flow3d (x 3)) added to s (:1414-1420, :1445-1452)
__device__ __forceinline__ void obj_stat_add(ObjStat& s, const float* __restrict__ kx, const float* __restrict__ ky, const float* __restrict__ depth,
                                             const float* __restrict__ flow3d, int i, int rows, int cols, int shr_row, int shr_col, float sf_thres) {
  const float u = kx[i], v = ky[i];
  if (v < (float)shr_row || v > (float)(rows - shr_row) || u < (float)shr_col || u > (float)(cols - shr_col)) s.boundary = __fadd_rn(s.boundary, 1.f);
  s.depth_sum = __fadd_rn(s.depth_sum, depth[i]);
  const float fx = flow3d[3 * i], fz = flow3d[3 * i + 2];
  const float nrm = sqrtf(__fadd_rn(__fmul_rn(fx, fx), __fmul_rn(fz, fz)));
  if (nrm < sf_thres) s.sf_count = __fadd_rn(s.sf_count, 1.f);
}

enum ObjClass { OBJ_DYNAMIC = 1, OBJ_STATIC = 2, OBJ_BOUNDARY = 3, OBJ_FAR = 4 };   // the VDO_OT_* codes
// the decision for an object of s.n > 0 points (:1421, :1490, :1497), in the reference's order
__host__ __device__ __forceinline__ int obj_class(const ObjStat& s, float sf_ds_thres, float th_depth_obj) {
  const float sz = (float)s.n;
  if (s.boundary / sz > 0.5f) return OBJ_BOUNDARY;
  if (s.sf_count / sz > sf_ds_thres) return OBJ_STATIC;
  if (s.depth_sum / sz > th_depth_obj || s.n < 150) return OBJ_FAR;
  return OBJ_DYNAMIC;
}

}  // namespace
