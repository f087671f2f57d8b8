// dev_entry.h -- host-side pieces every C entry around the device kernels shares: the CUDA-error return, the context accessors, the device
// pointer checks of the device-resident calls, and the work space that an estimator handle allocates once at creation.  Host code only.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <initializer_list>
#include <string>
#include <vector>

#include "../../include/vdo_b200.h"

// a CUDA call that fails is printed and the enclosing entry returns VDO_ERR_CUDA
#define VDO_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::fprintf(stderr, "[vdo_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return VDO_ERR_CUDA; } } while (0)

namespace vdo {

// vdo_capi.cpp: the message vdo_last_error returns
void ctx_set_error(vdo_ctx* c, const std::string& msg);
// ba_kernels.cu: the context's device and its SM count
void ctx_device(vdo_ctx* c, int* dev, int* n_sm);
// frame_kernels.cu: VDO_ERR_ARG (with the reason in err) unless p is device memory of device `dev` (not host, pinned host, managed or
// another GPU's memory)
int check_dev_ptr(const void* p, int dev, const std::string& who, std::string& err);

// a device array a call reads or writes; used = false: the call does not read it this time, so it is not checked
struct DevPtr { const void* p; size_t align; std::string name; bool used = true; };
using DevPtrs = std::vector<DevPtr>;
// NULL, misaligned or not device memory of device dev: "" or why the call is refused
inline std::string check_ptrs(const DevPtrs& ptrs, int dev) {
  std::string err;
  for (const DevPtr& q : ptrs) {
    if (!q.used) continue;
    if (!q.p) return q.name + " is NULL";
    if ((uintptr_t)q.p % q.align) return q.name + " is not aligned to " + std::to_string(q.align) + " bytes";
    if (check_dev_ptr(q.p, dev, q.name, err)) return err;
  }
  return "";
}

// The device memory of an estimator handle: every allocation is counted in bytes and freed with the handle.
struct WorkSpace {
  std::vector<void*> allocs;
  size_t bytes = 0;
  WorkSpace() = default;
  WorkSpace(const WorkSpace&) = delete;
  WorkSpace& operator=(const WorkSpace&) = delete;
  ~WorkSpace() { for (void* p : allocs) cudaFree(p); }
  // max(n, 1) elements
  template <class T> cudaError_t alloc(T*& p, size_t n) {
    p = nullptr;
    const size_t b = sizeof(T) * std::max<size_t>(n, 1);
    const cudaError_t e = cudaMalloc(&p, b);
    if (e == cudaSuccess) { allocs.push_back(p); bytes += b; }
    return e;
  }
};

// the end of `entry` creating w: *out = w when every step (the allocations, flow_lm_prepare) succeeded; otherwise w is deleted and the
// first failure is the context's error, "<entry>: <CUDA error>", with VDO_ERR_CUDA
template <class W> int create_done(vdo_ctx* ctx, const char* entry, W* w, std::initializer_list<cudaError_t> steps, W** out) {
  for (cudaError_t e : steps)
    if (e != cudaSuccess) {
      cudaGetLastError();
      ctx_set_error(ctx, std::string(entry) + ": " + cudaGetErrorString(e));
      delete w;
      return VDO_ERR_CUDA;
    }
  *out = w;
  return VDO_OK;
}

}  // namespace vdo
