// frame_px.cuh -- per-pixel rules of the frame ingest and the object sampling, shared by the kernels that read caller planes or resident
// frames: the strided plane readers of vdo_frame_upload_dev (frame_kernels.cu, k_ingest_frame) and the semi-dense object sampling test of
// Frame.cc:200-228 (k_sample_objects on a resident frame, k_om_sample of vdo_obj_motion_batch_dev on caller planes, obj_motion.cu), the
// static key test of Frame.cc:100-194 (k_filter_static, and cam_motion.cu's build and renewal on caller planes) and RenewFrameInfo's 1 px
// test (tracking_ops.cu, cam_motion.cu), so that every caller of a rule keeps exactly the same keys.
#pragma once
#include <cuda_runtime.h>

#include <climits>

#include "../../include/vdo_b200.h"

namespace {

// a caller plane (vdo_dev_plane) at element strides; p == nullptr: plane not given
struct PlaneArg { const void* p; long long sy, sx, sc; int dtype, ch, rgb; };
inline PlaneArg plane_arg(const vdo_dev_plane* pl) {
  if (!pl) return PlaneArg{nullptr, 0, 0, 0, 0, 0, 0};
  return PlaneArg{pl->data_dev, (long long)pl->stride_y, (long long)pl->stride_x, (long long)pl->stride_c, pl->dtype, pl->channels, pl->rgb};
}

// depth (f32, 1 channel) at pixel (x, y)
__device__ __forceinline__ float plane_depth(const PlaneArg& d, int x, int y) { return ((const float*)d.p)[y * d.sy + x * d.sx]; }
// flow (f32, 2 channels, HWC or CHW) at pixel (x, y)
__device__ __forceinline__ float2 plane_flow(const PlaneArg& f, int x, int y) {
  const float* s = (const float*)f.p + (y * f.sy + x * f.sx);
  return make_float2(s[0], s[f.sc]);
}
// mask label (i32 or i64) at pixel (x, y); an i64 label outside the int32 range sets *bad (its truncated value is never used)
__device__ __forceinline__ int plane_label(const PlaneArg& m, int x, int y, int* bad) {
  const long long o = y * m.sy + x * m.sx;
  if (m.dtype == VDO_DT_I64) {
    const long long v = ((const long long*)m.p)[o];
    if (v < INT_MIN || v > INT_MAX) *bad = 1;
    return (int)v;
  }
  return ((const int*)m.p)[o];
}

// Frame.cc:200-228, one pixel (x, y) of a w x h frame with label m and depth d: an object sample when m != 0, 0 < d < th and the flow
// target (x + fx, y + fy) lies strictly inside the image.  flow() is read only for a pixel that passes the label and depth tests.
template <class Flow>
__device__ __forceinline__ bool object_sample(int x, int y, int m, float d, float th, int w, int h, const Flow& flow, float& fx, float& fy, float& tx,
                                              float& ty) {
  if (!(m != 0 && d < th && d > 0.f)) return false;
  flow(fx, fy);
  tx = __fadd_rn((float)x, fx); ty = __fadd_rn((float)y, fy);
  return tx < (float)w && tx > 0.f && ty < (float)h && ty > 0.f;
}

// is the mask (i32 or i64) 0 at pixel (x, y); an i64 label is compared whole
__device__ __forceinline__ bool plane_unlabelled(const PlaneArg& m, int x, int y) {
  const long long o = y * m.sy + x * m.sx;
  return m.dtype == VDO_DT_I64 ? ((const long long*)m.p)[o] == 0 : ((const int*)m.p)[o] == 0;
}

// Frame.cc:100-129 + 181-194, the static test of key (px, py) of a w x h frame, read at pixel ((int)px, (int)py): mask == 0, 0 < depth <= th,
// both flow components non-zero, and the target (px + fx, py + fy) inside the image -- ORB keypoints (option I, :100-129) bound the key and
// its target by the far edges only, sampled keys (option II, :130-168) bound the target on both sides and not the key.  unlabelled(x, y),
// depth(x, y) and flow(x, y, fx, fy) read the frame; d, fx, fy: what was read.
template <class Unlabelled, class Depth, class Flow>
__device__ __forceinline__ bool static_key(float px, float py, float th, bool sampled, int w, int h, const Unlabelled& unlabelled, const Depth& depth,
                                           const Flow& flow, float& d, float& fx, float& fy) {
  const int x = (int)px, y = (int)py;
  d = depth(x, y);
  bool ok = false;
  if (unlabelled(x, y) && !(d > th || d <= 0.f)) {
    flow(x, y, fx, fy);
    if (fx != 0.f && fy != 0.f) {
      const float tx = __fadd_rn(px, fx), ty = __fadd_rn(py, fy);
      ok = sampled ? (tx < (float)w && ty < (float)h && tx > 0.f && ty > 0.f) : (tx < (float)w && ty < (float)h && px < (float)w && py < (float)h);
    }
  }
  return ok;
}

// the "already used" test of RenewFrameInfo's top-up loops (Tracking.cc:2735-2748, :2893-2907): any of the n keys of snap (x, y interleaved)
// closer than 1 px, as the float sqrt of float squares
__device__ __forceinline__ bool near_any(float kx, float ky, const float* __restrict__ snap, int n) {
  for (int j = 0; j < n; ++j) {
    const float dx = __fsub_rn(snap[2 * j], kx), dy = __fsub_rn(snap[2 * j + 1], ky);
    if (sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) < 1.0f) return true;
  }
  return false;
}

// exclusive scan of one flag per thread over the CTA (blockDim.x a multiple of 32, at most 1024); total: the CTA's sum.  All threads call it.
__device__ __forceinline__ int cta_excl_scan(int flag, int* wsum /*33*/, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int incl = flag;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  __syncthreads();
  if (lane == 31) wsum[wid] = incl;
  __syncthreads();
  if (threadIdx.x == 0) { int acc = 0; for (int k = 0; k < nw; ++k) { const int t = wsum[k]; wsum[k] = acc; acc += t; } wsum[32] = acc; }
  __syncthreads();
  total = wsum[32];
  return wsum[wid] + incl - flag;
}

}  // namespace
