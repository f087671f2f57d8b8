// pose4.cuh -- the 4x4 pose algebra and back-projections of the device pair calls, with the rounding of the tracker's host helpers
// (tracker.cpp mul4 / inv4 / unproject_world / get3d_camera, tracking_ops.cu get3d_world: cv::Mat float arithmetic).  Shared by
// obj_motion.cu and cam_motion.cu; both are compiled with --fmad=false, so that nothing here is contracted into an FMA.
#pragma once
#include <cuda_runtime.h>

namespace {

// cv::Mat A * B of two 4x4 CV_32F: a0*b0 + a1*b1 + a2*b2 + a3*b3 in float, left to right
__device__ __forceinline__ void mul4(const float* A, const float* B, float* C) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float s = A[4 * i] * B[j];
      s = s + A[4 * i + 1] * B[4 + j];
      s = s + A[4 * i + 2] * B[8 + j];
      s = s + A[4 * i + 3] * B[12 + j];
      C[4 * i + j] = s;
    }
}
// Converter::toInvMatrix: [R^T | -R^T t], the translation accumulated in double
__device__ __forceinline__ void inv4(const float* T, float* I) {
  for (int k = 0; k < 16; ++k) I[k] = k % 5 == 0 ? 1.f : 0.f;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) I[4 * i + j] = T[4 * j + i];
    double s = 0;
    for (int k = 0; k < 3; ++k) s += (double)T[4 * k + i] * (double)T[4 * k + 3];
    I[4 * i + 3] = (float)(-s);
  }
}
// Frame::UnprojectStereoObject / UnprojectStereoStat: the world point of pixel (u, v) at depth z through Tcw
__device__ __forceinline__ void unproject_world(float u, float v, float z, const float* K, const float* Tcw, float* X) {
  const float invfx = 1.0f / K[0], invfy = 1.0f / K[1];
  const float x = (u - K[2]) * z * invfx, y = (v - K[3]) * z * invfy;
  for (int r = 0; r < 3; ++r) {
    const double twl = (double)(float)(-((double)Tcw[r] * (double)Tcw[3] + (double)Tcw[4 + r] * (double)Tcw[7] + (double)Tcw[8 + r] * (double)Tcw[11]));
    X[r] = (float)((double)Tcw[r] * (double)x + (double)Tcw[4 + r] * (double)y + (double)Tcw[8 + r] * (double)z + twl);
  }
}
__device__ __forceinline__ void load_pose(const float* T, int p, float* dst) {
  for (int k = 0; k < 16; ++k) dst[k] = T ? T[16 * p + k] : (k % 5 == 0 ? 1.f : 0.f);
}

}  // namespace
