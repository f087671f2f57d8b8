// ba_kernels.cu -- sm_90a kernels of the batch factor-graph path and the CUDA implementation of BaBackend.
//
// All arithmetic is fp64 (g2o runs in double; SURVEY.md H4).  The path is HBM/L2-bound stream-gather-reduce work over
// edge streams, so the kernels are organised around coalesced / bulk-copied edge streams and shuffle reductions, not tensor
// cores.  Two layouts of the landmark / edge side share this backend (chosen per graph by BaGraph::finalize, d.tiled):
//   * tiled (default, ba_tile_kernels.cuh): one CTA per tile of whole tracklets, TMA-staged landmark blocks, landmark-side
//     sums in shared memory, se3-vertex-side sums in the world frame over vertex-sorted warp segments; edges stored once
//   * chunked (this file; graphs whose tracklets do not fit a tile): one thread per tracklet on the landmark-major stream
//     (k_lin_tracklets, k_schur_*), one CTA per <=512-edge chunk of a vertex's own copy of the edge stream (k_vertex_sym,
//     k_schur_vertex: 21+6 or 6 per-thread accumulators, warp-shuffle tree + one smem hop, <=42 atomics per chunk)
// Common to both: the reduced system is applied matrix-free inside a PCG whose preconditioner is block-tridiagonal along the
// se3-se3 edge chains and solved by block cyclic reduction (one thread-block cluster per chain); 8 PCG iterations are one
// CUDA-graph launch.  Kernel bodies live in ba_bodies.cuh / ba_tiles.cuh (shared with the serial emulation under tests/emul).
#include <cuda_runtime.h>
#include <cooperative_groups.h>

#include <cstdio>
#include <cstring>

#include <dlfcn.h>
#include <nccl.h>

#include <map>
#include <set>
#include <type_traits>
#include <utility>

#include "ba_bodies.cuh"

namespace cg = cooperative_groups;

namespace vdo {

constexpr int PCR_CL = 8;   // CTAs per thread-block cluster working on one LONG chain of the preconditioner (short chains: one CTA)

#define CK(x)                                                                                       \
  do {                                                                                              \
    cudaError_t e_ = (x);                                                                           \
    if (e_ != cudaSuccess) { std::fprintf(stderr, "[vdo_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); } \
  } while (0)

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
// block-wide sum; result valid in thread 0.  smem must hold >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* smem) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) smem[w] = v;
  __syncthreads();
  v = (threadIdx.x < nw) ? smem[threadIdx.x] : 0.0;
  if (w == 0) v = warp_sum(v);
  return v;
}

// deterministic sum of a[0..n) by one CTA (fixed per-thread strides, fixed tree): same inputs => same bits on every rank.
// All threads receive the result.  smem must hold >= 33 doubles.
__device__ __forceinline__ double det_sum(const double* __restrict__ a, int n, double* smem) {
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += a[i];
  v = block_sum(v, smem);
  if (threadIdx.x == 0) smem[32] = v;
  __syncthreads();
  return smem[32];
}

// ---- graph selectors: every step of the tiled and dense LM paths is one kernel template on S ----
// One: a lone graph, its BaDev by value and the scalars of its trial; the launch is the graph's own grid.
// Many: one step of several graphs (BaGraph::optimize_batch) in one launch.  Every graph keeps the grid of its lone launch: launch table
// t lists, per graph g, its first CTA first[t][g] (built once per call, the graphs do not change after finalize), and a CTA runs the body
// with that graph's BaDev and its local block index.  flags[g] (written by k_batch_params whenever the caller changes them) selects the
// graphs the step runs on; lambda[g] / reortho[g] / tol2[g] are the trial's.  Tables of the dense solve are empty for PCG-path graphs and
// those of the PCG empty for dense ones.  The cluster kernels' tables (BT_PCR_L, BT_PCG_L) hold whole clusters per graph, so every CTA of
// a cluster picks the same graph.
enum { BT_TILE_LIN, BT_TILE_LIN_CH, BT_FIN_LIN, BT_SE3, BT_MAXDIAG, BT_FACTOR, BT_BAND_FORM, BT_VTRANS, BT_BACKSUB, BT_BACKSUB_CH, BT_UPDATE,
       // dense path only
       BT_DINIT, BT_DSE3, BT_FROM_BAND, BT_SCHUR2, BT_FIN_SCHUR2, BT_DSCHUR, BT_CHOL,
       // PCG path only (tiled layout): preconditioner, rhs, init and the fused iteration
       BT_PRE_BEGIN, BT_PRE_ST, BT_PRE_CH, BT_PRE_FIN, BT_PCR_L, BT_PCR_S, BT_RHS_ST, BT_RHS_CH, BT_VERT, BT_PCG_L, BT_PCG_S, BT_PCG_FIN, BT_BAND_MUL,
       BT_S2_ST, BT_S2_CH, BT_PHPP, BT_FIN_DOT, BT_N };
struct BatchDev { const BaDev* ds; const int* first; const int* band_per; int* flags; double* lambda; int* reortho; double* tol2; int n; };
struct One {
  BaDev d; double lam; int rt, par, band_per;   // par: PCG parity (p_k in d.p when 0, in d.p2 when 1); band_per: tiles per CTA of k_band_form
  __device__ __forceinline__ const BaDev* pick(int& blk, int& g) const { blk = blockIdx.x; g = 0; return &d; }
  __device__ __forceinline__ double lambda(int) const { return lam; }
  __device__ __forceinline__ int reortho(int) const { return rt; }
  __device__ __forceinline__ int parity() const { return par; }
  __device__ __forceinline__ int tiles_per_cta(int) const { return band_per; }
  __device__ __forceinline__ int ctas(int) const { return (int)gridDim.x; }
};
struct Many {
  BatchDev B; const int* f; int bit, par;      // f: the launch table of the step (first + BT_* x (n + 1)); bit: the flag a graph must hold
  // the graph of this CTA and its local block index, or nullptr when the step does not run on that graph
  __device__ __forceinline__ const BaDev* pick(int& blk, int& g) const {
    const int b = blockIdx.x;
    int lo = 0, hi = B.n;                        // f[lo] <= b < f[hi]
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (f[mid] <= b) lo = mid; else hi = mid; }
    blk = b - f[lo]; g = lo;
    return (B.flags[lo] & bit) ? B.ds + lo : nullptr;
  }
  __device__ __forceinline__ double lambda(int g) const { return B.lambda[g]; }
  __device__ __forceinline__ int reortho(int g) const { return B.reortho[g]; }
  __device__ __forceinline__ int parity() const { return par; }
  __device__ __forceinline__ int tiles_per_cta(int g) const { return B.band_per[g]; }
  __device__ __forceinline__ int ctas(int g) const { return f[g + 1] - f[g]; }
};
#define VDO_PICK                                   \
  int blk_, g_;                                    \
  const BaDev* const dp_ = s.pick(blk_, g_);       \
  if (!dp_) return;                                \
  const BaDev& d = *dp_;
__host__ __device__ __forceinline__ unsigned int pcg_total_ctas(const BaDev& d) { return (unsigned int)(d.n_own_long * PCR_CL + (d.n_own_paths - d.n_own_long)); }

// ---------------------------------------------------------------------------------------------------------------
template <bool WRITE>
__global__ void __launch_bounds__(128) k_lin_tracklets(BaDev d) {
  __shared__ double red[32];
  const int t = d.Tstat + blockIdx.x * blockDim.x + threadIdx.x;
  double chi = 0.0;
  if (t < d.T) chi = body_lin_tracklet(d, t, WRITE);
  chi = block_sum(chi, red);
  if (threadIdx.x == 0 && chi != 0.0) atomicAdd(d.scal + SC_CHI2, chi);
}
template <bool WRITE>
__global__ void __launch_bounds__(256) k_lin_static(BaDev d) {
  __shared__ double red[32];
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  double chi = 0.0;
  if (k < d.Tstat) chi = body_lin_static(d, k, WRITE);
  chi = block_sum(chi, red);
  if (threadIdx.x == 0 && chi != 0.0) atomicAdd(d.scal + SC_CHI2, chi);
}

// reduce NV per-thread values over the CTA into smem out[NV]
template <int NV>
__device__ __forceinline__ void block_reduce_vec(double* acc, double* smem /*[nwarps*NV]*/) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    double v = warp_sum(acc[i]);
    if (lane == 0) smem[w * NV + i] = v;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = 0;
    for (int k = 0; k < nw; ++k) s += smem[k * NV + threadIdx.x];
    smem[threadIdx.x] = s;   // safe: thread i only reads column i of every row, and row 0 column i is its own
  }
  __syncthreads();
}

// MODE 0: linearise (Hpp += A, bp += g) ; MODE 1: preconditioner (Minv -= A) ;  OBS: pointxyz vs ternary stream
template <int MODE, bool OBS>
__global__ void __launch_bounds__(128) k_vertex_sym(BaDev d) {
  __shared__ double sm[4 * 27];
  const Chunk ch = OBS ? d.obs_chunks[blockIdx.x] : d.ter_chunks[blockIdx.x];
  Iso T; iso_load(d.se3 + 12 * (size_t)ch.v, T);
  double acc[27];
#pragma unroll
  for (int i = 0; i < 27; ++i) acc[i] = 0.0;
  for (int e = ch.begin + threadIdx.x; e < ch.end; e += blockDim.x) {
    if (MODE == 0) { if (OBS) body_lin_vertex_obs(d, T, e, acc, acc + 21); else body_lin_vertex_ter(d, T, e, acc, acc + 21); }
    else { if (OBS) body_precond_vertex_obs(d, T, e, acc); else body_precond_vertex_ter(d, T, e, acc); }
  }
  block_reduce_vec<27>(acc, sm);
  if (threadIdx.x < 36) {
    const int r = threadIdx.x / 6, c = threadIdx.x % 6;
    const double v = sm[r <= c ? sym6_idx(r, c) : sym6_idx(c, r)];
    if (MODE == 0) atomicAdd(d.Hpp + 36 * (size_t)ch.v + threadIdx.x, v);
    else atomicAdd(d.Minv + 36 * (size_t)ch.v + threadIdx.x, -v);
  } else if (MODE == 0 && threadIdx.x < 42) {
    atomicAdd(d.bp + 6 * (size_t)ch.v + (threadIdx.x - 36), sm[21 + threadIdx.x - 36]);
  }
}

template <bool OBS>
__global__ void __launch_bounds__(128) k_schur_vertex(BaDev d, double sign, double* __restrict__ out, int check_done) {
  __shared__ double sm[4 * 6];
  if (check_done && d.scal[SC_DONE] != 0.0) return;
  const Chunk ch = OBS ? d.obs_chunks[blockIdx.x] : d.ter_chunks[blockIdx.x];
  Iso T; iso_load(d.se3 + 12 * (size_t)ch.v, T);
  double acc[6] = {0, 0, 0, 0, 0, 0};
  for (int e = ch.begin + threadIdx.x; e < ch.end; e += blockDim.x) {
    if (OBS) body_schur_vertex_obs(d, T, e, acc); else body_schur_vertex_ter(d, T, e, acc);
  }
  block_reduce_vec<6>(acc, sm);
  if (threadIdx.x < 6) atomicAdd(out + 6 * (size_t)ch.v + threadIdx.x, sign * sm[threadIdx.x]);
}

template <bool WRITE>
__device__ __forceinline__ void k_lin_se3_edges_body(const BaDev& d, int bx) {
  __shared__ double red[32];
  const int e = bx * blockDim.x + threadIdx.x;
  double chi = 0.0;
  if (e < d.Ese) {
    double Hi[36], Hj[36], Ho[36], gi[6], gj[6];
    const bool binary = body_se3_edge(d, e, WRITE, chi, Hi, Hj, Ho, gi, gj);
    if (!d.own) chi = 0.0;      // sharded graphs: the se3-se3 edges are accumulated by rank 0 only (every rank keeps J_i^T W J_j)
    if (WRITE) {
      const int i = d.se_i[e];
      if (d.own) {
        for (int k = 0; k < 36; ++k) atomicAdd(d.Hpp + 36 * (size_t)i + k, Hi[k]);
        for (int k = 0; k < 6; ++k) atomicAdd(d.bp + 6 * (size_t)i + k, gi[k]);
      }
      if (binary) {
        const int j = d.se_j[e];
        for (int k = 0; k < 36; ++k) { if (d.own) atomicAdd(d.Hpp + 36 * (size_t)j + k, Hj[k]); d.se_Hoff[36 * (size_t)e + k] = Ho[k]; }
        if (d.own) for (int k = 0; k < 6; ++k) atomicAdd(d.bp + 6 * (size_t)j + k, gj[k]);
      }
    }
  }
  chi = block_sum(chi, red);
  if (threadIdx.x == 0 && chi != 0.0) atomicAdd(d.scal + SC_CHI2, chi);
}
template <class S, bool WRITE>
__global__ void __launch_bounds__(64) k_lin_se3_edges(S s) { VDO_PICK k_lin_se3_edges_body<WRITE>(d, blk_); }

__device__ __forceinline__ void k_max_diagonal_body(const BaDev& d, int bx, int gx) {
  __shared__ double red[32];
  const int n1 = d.C * 6, n = n1 + d.P;
  double m = 0.0;
  for (int i = bx * blockDim.x + threadIdx.x; i < n; i += gx * blockDim.x)
    m = fmax(m, i < n1 ? fabs(d.Hpp[36 * (size_t)(i / 6) + 7 * (i % 6)]) : fabs(d.hll[i - n1]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_down_sync(0xffffffffu, m, o));
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) m = fmax(m, red[k]);
    atomicMax(reinterpret_cast<unsigned long long*>(d.scal + SC_MAXDIAG), (unsigned long long)__double_as_longlong(m));  // m >= 0
  }
}
template <class S>
__global__ void __launch_bounds__(256) k_max_diagonal(S s) { VDO_PICK k_max_diagonal_body(d, blk_, s.ctas(g_)); }

__device__ __forceinline__ void k_factor_landmarks_body(const BaDev& d, double lambda, int bx) {
  const int t = bx * blockDim.x + threadIdx.x;
  if (t < d.Tstat) body_factor_static(d, t, lambda);
  else if (t < d.T) body_factor_tracklet(d, t, lambda);
}
template <class S>
__global__ void __launch_bounds__(128) k_factor_landmarks(S s) { VDO_PICK k_factor_landmarks_body(d, s.lambda(g_), blk_); }

// Chains (dynamic tracklets): 8 lanes cooperate on one tracklet.  Each lane owns one landmark of the current 8-landmark
// segment and does that landmark's gathers (pointxyz edges through the per-vertex world-frame vectors, its ternary edge through the
// motion pose) in parallel with its neighbours; only the 3-vector recursions y_k = u_k + f_{k-1} R_{k-1} y_{k-1} (forward) and
// z_k = (y_k + omega_k R_k^T z_{k+1}) / s_k (backward) walk the lanes, one shuffle of 3 doubles per step.
// mode 0: out = Hll^-1 bl ; mode 1: out = Hll^-1 (Hlp v) ; mode 2: out = Hll^-1 (bl - Hlp v)
template <int MODE>
__global__ void __launch_bounds__(128) k_schur_chains8(BaDev d, const double* __restrict__ v, double* __restrict__ out) {
  if (MODE == 1 && d.scal[SC_DONE] != 0.0) return;
  const int lane8 = threadIdx.x & 7;
  const int t = d.Tstat + ((blockIdx.x * blockDim.x + threadIdx.x) >> 3);
  const bool live = t < d.T;
  const int kb = live ? d.tk_begin[t] : 0, ke = live ? d.tk_begin[t + 1] : 0;
  const unsigned FULL = 0xffffffffu;
  double seg_w[3] = {0, 0, 0};       // f_{k-1} R_{k-1} y_{k-1} entering the segment
  double seg_c[3] = {0, 0, 0};       // ternary contribution of edge (k-1, k) to u_k entering the segment
  // ---------------- forward ----------------
  for (int base = kb; __any_sync(FULL, base < ke); base += 8) {
    const int k = base + lane8;
    const bool valid = k < ke;
    double u[3] = {0, 0, 0}, cn[3] = {0, 0, 0}, R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double f = 0.0;
    if (valid) {
      const int h = d.tk_h[k];
      const double om = d.tk_omega[k];
      f = om / d.pt_s[k];
      if (MODE != 0) {
        const double p[3] = {d.pt[3 * (size_t)k], d.pt[3 * (size_t)k + 1], d.pt[3 * (size_t)k + 2]};
        for (int e = d.lm_obs_begin[k]; e < d.lm_obs_begin[k + 1]; ++e) {
          const double* w = d.vw + 6 * (size_t)d.lm_cam[e];
          double pxb[3]; cross3(p, w + 3, pxb);
          const double oe = d.lm_omega[e];
          u[0] += oe * (w[0] + 2 * pxb[0]); u[1] += oe * (w[1] + 2 * pxb[1]); u[2] += oe * (w[2] + 2 * pxb[2]);
        }
      }
      if (h >= 0) {
        Iso H; iso_load(d.se3 + 12 * (size_t)h, H);
#pragma unroll
        for (int i = 0; i < 9; ++i) R[i] = H.R[i];
        if (MODE != 0) {
          const double pn[3] = {d.pt[3 * (size_t)(k + 1)], d.pt[3 * (size_t)(k + 1) + 1], d.pt[3 * (size_t)(k + 1) + 2]};
          double q[3]; iso_inv_apply(H, pn, q);
          double a[3]; ter_Jh_mul(q, v + 6 * (size_t)h, a);
          u[0] += om * a[0]; u[1] += om * a[1]; u[2] += om * a[2];
          double Ra[3]; rot_apply(H.R, a, Ra);
          cn[0] = -om * Ra[0]; cn[1] = -om * Ra[1]; cn[2] = -om * Ra[2];
        }
      }
    }
    // ternary contribution from the previous landmark's edge
    double cp[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) { cp[i] = __shfl_up_sync(FULL, cn[i], 1, 8); if (lane8 == 0) cp[i] = seg_c[i]; }
#pragma unroll
    for (int i = 0; i < 3; ++i) { u[i] += cp[i]; seg_c[i] = __shfl_sync(FULL, cn[i], 7, 8); }
    double y[3];
    if (valid) {
      if (MODE == 0) { y[0] = d.bl[3 * (size_t)k]; y[1] = d.bl[3 * (size_t)k + 1]; y[2] = d.bl[3 * (size_t)k + 2]; }
      else if (MODE == 1) { y[0] = u[0]; y[1] = u[1]; y[2] = u[2]; }
      else { y[0] = d.bl[3 * (size_t)k] - u[0]; y[1] = d.bl[3 * (size_t)k + 1] - u[1]; y[2] = d.bl[3 * (size_t)k + 2] - u[2]; }
    } else { y[0] = y[1] = y[2] = 0; }
    double wout[3] = {0, 0, 0};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      double win[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) win[i] = __shfl_up_sync(FULL, wout[i], 1, 8);
      if (lane8 == j) {
        if (j == 0) { win[0] = seg_w[0]; win[1] = seg_w[1]; win[2] = seg_w[2]; }
        y[0] += win[0]; y[1] += win[1]; y[2] += win[2];
        double Ry[3]; rot_apply(R, y, Ry);
        wout[0] = f * Ry[0]; wout[1] = f * Ry[1]; wout[2] = f * Ry[2];
      }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) seg_w[i] = __shfl_sync(FULL, wout[i], 7, 8);
    if (valid) { out[3 * (size_t)k] = y[0]; out[3 * (size_t)k + 1] = y[1]; out[3 * (size_t)k + 2] = y[2]; }
  }
  // ---------------- backward ----------------
  double seg_z[3] = {0, 0, 0};       // z of the first landmark of the following segment
  const int nseg = (ke - kb + 7) >> 3;
  int max_seg = nseg;
  { const int a = __shfl_xor_sync(FULL, max_seg, 8); if (a > max_seg) max_seg = a; }      // uniform trip count per warp (4 groups of 8 lanes)
  { const int a = __shfl_xor_sync(FULL, max_seg, 16); if (a > max_seg) max_seg = a; }
  for (int sgi = max_seg - 1; sgi >= 0; --sgi) {
    const int k = kb + 8 * sgi + lane8;
    const bool valid = sgi < nseg && k < ke;
    double y[3] = {0, 0, 0}, Rt[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, om = 0.0, is = 0.0;
    bool last = true;
    if (valid) {
      y[0] = out[3 * (size_t)k]; y[1] = out[3 * (size_t)k + 1]; y[2] = out[3 * (size_t)k + 2];
      is = 1.0 / d.pt_s[k];
      const int h = d.tk_h[k];
      if (h >= 0 && k + 1 < ke) {
        last = false; om = d.tk_omega[k];
        const double* Rp = d.se3 + 12 * (size_t)h;
#pragma unroll
        for (int i = 0; i < 9; ++i) Rt[i] = Rp[i];
      }
    }
    double z[3] = {0, 0, 0};
#pragma unroll
    for (int j = 7; j >= 0; --j) {
      double zn[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) zn[i] = __shfl_down_sync(FULL, z[i], 1, 8);
      if (lane8 == j && valid) {
        if (j == 7) { zn[0] = seg_z[0]; zn[1] = seg_z[1]; zn[2] = seg_z[2]; }
        if (!last) {
          double t3[3]; rot_t_apply(Rt, zn, t3);
          y[0] += om * t3[0]; y[1] += om * t3[1]; y[2] += om * t3[2];
        }
        z[0] = y[0] * is; z[1] = y[1] * is; z[2] = y[2] * is;
      }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) seg_z[i] = __shfl_sync(FULL, z[i], 0, 8);
    if (valid) { out[3 * (size_t)k] = z[0]; out[3 * (size_t)k + 1] = z[1]; out[3 * (size_t)k + 2] = z[2]; }
  }
}

template <int MODE>
__global__ void __launch_bounds__(256) k_schur_static(BaDev d, double* __restrict__ out) {
  if (MODE == 1 && d.scal[SC_DONE] != 0.0) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < d.Tstat) body_schur_static(d, k, MODE, out);
}

__device__ __forceinline__ void k_precond_begin_body(const BaDev& d, double lambda, int bx) {
  const int i = bx * blockDim.x + threadIdx.x;
  if (i < d.C * 36) { const int k = i % 36; d.Minv[i] = d.own ? d.Hpp[i] + ((k % 7) == 0 ? lambda : 0.0) : 0.0; }
}
template <class S>
__global__ void __launch_bounds__(128) k_precond_begin(S s) { VDO_PICK k_precond_begin_body(d, s.lambda(g_), blk_); }

__global__ void k_set_scalars(BaDev d, double lambda, double tol2) { d.scal[SC_LAMBDA] = lambda; d.scal[SC_TOL2] = tol2; }
__device__ __forceinline__ void k_vertex_transform_body(const BaDev& d, const double* __restrict__ x, int bx) {
  const int v = bx * blockDim.x + threadIdx.x;
  if (v < d.C) body_vertex_transform(d, v, x, d.vw);
}
// x: the vector to transform, nullptr for every graph's own xp
template <class S>
__global__ void __launch_bounds__(128) k_vertex_transform(S s, const double* __restrict__ x) { VDO_PICK k_vertex_transform_body(d, x ? x : d.xp, blk_); }
__global__ void __launch_bounds__(128) k_hpp_mul(BaDev d, const double* __restrict__ x, double* __restrict__ out) {
  if (d.scal[SC_DONE] != 0.0) return;
  const double lambda = d.scal[SC_LAMBDA];
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < d.C) body_hpp_mul(d, v, lambda, x, out);
}

// ---- block cyclic reduction: one thread-block CLUSTER (PCR_CL CTAs) per long path, cluster.sync() between the wide levels ----
// CL = CTAs per cluster: PCR_CL for long paths, 1 (plain CTA, the cluster barrier degenerates to a CTA barrier) for paths of at most
// PCR_SHORT vertices -- most paths are short (objects seen for a few frames, single motion vertices) and a cluster of 8 CTAs each would only
// multiply the number of waves the launch needs.  path0: position of the launch's first path in own_paths (long paths first).
//
// Level l (stride s = 2^l) of a path of n vertices (local index j = v - pb) works on the vertices with j % s == 0: those with j % 2s == s
// are eliminated, the others (j = 2s k, the level's survivors) absorb them.  Vertex 0 is eliminated alone after the last level.  Every
// eliminated vertex u has the survivor u - s on its left, which stores Dinv_u; survivors store their operators A_v, G_v once per level,
// level-major: slot 2 pb + off_l + k, off_l = sum of the survivor counts of the levels below l (a path holds fewer than 2n slots).
// A level whose work fits one CTA runs on the cluster's rank 0 alone, behind __syncthreads instead of a cluster barrier.
// CTAs per SM the preconditioner's cluster kernels are built for: 4 for a lone graph (64 registers: all of config 5's long-path clusters
// in one wave); 2 for the batched form, whose graph selection costs registers that 64 would spill
template <class S> constexpr int bcr_ctas_per_sm() { return std::is_same<S, One>::value ? 4 : 2; }
__device__ __forceinline__ int bcr_survivors(int n, int l) { return (n - 1 + (2 << l)) >> (l + 1); }    // j = 0, 2s, 4s, ... < n
__device__ __forceinline__ int bcr_eliminated(int n, int l) { return (n - 1 + (1 << l)) >> (l + 1); }  // j = s, 3s, 5s, ... < n

// In-place Gauss-Jordan inverse of an SPD 6x6 whose row i lives in lane i of an aligned 8-lane group (lanes 6, 7 of the group and groups
// without a block carry the identity; every lane of the warp executes the shuffles).  The pivots are those of the LDL^T factorisation:
// a non-positive (or non-finite) one reports "not SPD" exactly where the Cholesky of body_pcr_invert does.
__device__ __forceinline__ bool gj6_rows(double (&a)[6], int i) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const double piv = __shfl_sync(0xffffffffu, a[k], k, 8);
    if (!(piv > 0.0) || !(piv < 1e300)) ok = false;
    const double pinv = 1.0 / piv, f = a[k] * pinv;
#pragma unroll
    for (int c = 0; c < 6; ++c) {                            // pivot row k is fetched one element at a time (register pressure)
      const double rk = __shfl_sync(0xffffffffu, a[c], k, 8);
      if (i == k) a[c] = (c == k) ? pinv : rk * pinv;
      else a[c] = (c == k) ? -f : a[c] - f * rk;
    }
  }
  return ok;
}
// row i of the inverse of the block whose row i is src (identity rows when !act); a block that is not SPD gets the diagonal fallback
// 1 / (|D_ii| + lambda).  Returns false for such a block.
__device__ __forceinline__ bool inv6_rows(double (&a)[6], const double* src, bool act, int i, double lambda) {
  double dii = 1.0;
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    a[c] = act ? src[c] : (c == (i % 6) ? 1.0 : 0.0);
    if (c == i) dii = a[c];
  }
  const bool ok = gj6_rows(a, i);
  if (!ok) {
#pragma unroll
    for (int c = 0; c < 6; ++c) a[c] = (c == i) ? 1.0 / (fabs(dii) + lambda) : 0.0;
  }
  return ok || !act;
}
// Factorisation: an 8-lane group owns a survivor v of the level, lane i its row i of every block.  With L_v = M(v, v - s) of the level
// (level 0: the se3-se3 edge block; zero outside the path) and D the level's diagonal blocks (level 0: the assembled blocks in Minv):
//   Dinv_{v+-s} = D_{v+-s}^-1 (each eliminated block is inverted by both of its survivors, so a level needs one barrier),
//   A_v = -L_v Dinv_{v-s},  G_v = -L_{v+s}^T Dinv_{v+s},  D'_v = D_v + A_v L_v^T + G_v L_{v+s},  L'_v = A_v L_{v-s}.
// A level writes D and L of its survivors only and reads those of its eliminated vertices only, so both are updated in place.
template <int CL>
__device__ __forceinline__ void k_pcr_factor_body(const BaDev& d, double lambda, int path0, int bx) {
  cg::cluster_group cl = cg::this_cluster();
  const int path = d.own_paths[path0 + bx / CL];
  const int pb = d.path_begin[path], n = d.path_begin[path + 1] - pb;
  const int nl = pcr_num_levels(n), rank = (int)cl.block_rank(), i = threadIdx.x & 7;
  __shared__ double sblk[32 * 180];                          // per 8-lane group: L_v, D_{v-s}, L_{v-s}, L_{v+s}, D_{v+s}
  double* const blk = sblk + 180 * (threadIdx.x >> 3);
  int bad = 0;
  size_t off = 2 * (size_t)pb;
#pragma unroll 1
  for (int l = 0; l < nl; ++l) {
    const int s = 1 << l, cnt = bcr_survivors(n, l);
    const bool wide = cnt > 32;
    if (!wide && rank != 0) break;                           // the remaining levels run on rank 0
    const int g0 = (wide ? rank * (int)blockDim.x + (int)threadIdx.x : (int)threadIdx.x) >> 3, ng = wide ? CL * 32 : 32;
    const double* const Ds = l ? d.pcr_D : d.Minv;
#pragma unroll 1
    for (int k0 = 0; k0 < cnt; k0 += ng) {
      const int k = k0 + g0, j = 2 * s * k, v = pb + j;
      const bool has = k < cnt, hm = has && k > 0, hp = has && j + s < n, act = has && i < 6;
      __syncwarp();
      if (has) {
#pragma unroll 1
        for (int q = 0; q < 5; ++q) {                        // block q of the group: its source and whether it is stored transposed
          const int w = q == 0 ? v : q <= 2 ? v - s : v + s;
          const double* src = nullptr;
          bool tr = false;
          if (q <= 2 ? hm : hp) {
            if (q == 1 || q == 4) src = Ds + 36 * (size_t)w;
            else if (l) src = d.pcr_L + 36 * (size_t)w;
            else if (const int ed = d.pcr_edge[w]; ed >= 0) { src = d.se_Hoff + 36 * (size_t)ed; tr = d.pcr_tr[w] != 0; }
          }
#pragma unroll
          for (int t = 0; t < 5; ++t) {
            const int o = i + 8 * t;
            if (o < 36) blk[36 * q + o] = src ? src[tr ? 6 * (o % 6) + o / 6 : o] : 0.0;
          }
        }
      }
      __syncwarp();
      double a[6];
      inv6_rows(a, blk + 36 + 6 * i, act && hm, i, lambda);
      if (act) {
#pragma unroll
        for (int c = 0; c < 6; ++c) blk[36 + 6 * i + c] = a[c];
      }
      __syncwarp();
      const bool ok = inv6_rows(a, blk + 144 + 6 * i, act && hp, i, lambda);
      if (act && hp) {
        double* o = d.pcr_Dinv + 36 * (size_t)(v + s) + 6 * i;
#pragma unroll
        for (int c = 0; c < 6; ++c) { blk[144 + 6 * i + c] = a[c]; o[c] = a[c]; }
        if (!ok && i == 0) bad = 1;
      }
      __syncwarp();
      if (act) {
        const double *Lv = blk, *Dim = blk + 36, *Lm = blk + 72, *Lp = blk + 108, *Dip = blk + 144;
        double av[6] = {0, 0, 0, 0, 0, 0}, t[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) {
          const double lk = Lv[6 * i + kk];
#pragma unroll
          for (int c = 0; c < 6; ++c) av[c] -= lk * Dim[6 * kk + c];
        }
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) {
#pragma unroll
          for (int c = 0; c < 6; ++c) t[c] += av[kk] * Lm[6 * kk + c];
        }
        double* Ao = d.pcr_A + 36 * (off + k) + 6 * i; double* Lo = d.pcr_L + 36 * (size_t)v + 6 * i;
#pragma unroll
        for (int c = 0; c < 6; ++c) { Ao[c] = av[c]; Lo[c] = t[c]; t[c] = Ds[36 * (size_t)v + 6 * i + c]; }
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) {
#pragma unroll
          for (int c = 0; c < 6; ++c) t[c] += av[kk] * Lv[6 * c + kk];
        }
#pragma unroll
        for (int c = 0; c < 6; ++c) av[c] = 0.0;
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) {
          const double lp = Lp[6 * kk + i];
#pragma unroll
          for (int c = 0; c < 6; ++c) av[c] -= lp * Dip[6 * kk + c];
        }
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) {
#pragma unroll
          for (int c = 0; c < 6; ++c) t[c] += av[kk] * Lp[6 * kk + c];
        }
        double* Go = d.pcr_G + 36 * (off + k) + 6 * i; double* Do = d.pcr_D + 36 * (size_t)v + 6 * i;
#pragma unroll
        for (int c = 0; c < 6; ++c) { Go[c] = av[c]; Do[c] = t[c]; }
      }
    }
    if (wide) cl.sync(); else __syncthreads();
    off += cnt;
  }
  if (rank == 0 && threadIdx.x < 32) {                       // vertex 0, alone at the top
    double a[6];
    const bool act = threadIdx.x < 6;
    const bool ok = inv6_rows(a, (nl ? d.pcr_D : d.Minv) + 36 * (size_t)pb + 6 * i, act, i, lambda);
    if (act) {
#pragma unroll
      for (int c = 0; c < 6; ++c) d.pcr_Dinv[36 * (size_t)pb + 6 * i + c] = a[c];
      if (!ok && i == 0) bad = 1;
    }
  }
  if (bad) atomicAdd(d.scal + SC_BAD, 1.0);
}
template <class S, int CL>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(256, bcr_ctas_per_sm<S>()) k_pcr_factor(S s) { VDO_PICK k_pcr_factor_body<CL>(d, s.lambda(g_), CL > 1 ? 0 : d.n_own_long, blk_); }

__device__ __forceinline__ double dot6(const double* a, const double* x) { return a[0] * x[0] + a[1] * x[1] + a[2] * x[2] + a[3] * x[3] + a[4] * x[4] + a[5] * x[5]; }
// z = M^-1 r for the cluster's path (r final for the whole path on entry); returns this thread's share of r.z (of the z items it wrote).
//   forward, l = 0 .. nl-1:  b_v += A_v b_{v-s} + G_v b_{v+s} for the survivors (b = r before the first level; in place)
//   top:                     x_0 = Dinv_0 b_0
//   back, l = nl-1 .. 0:     x_u = Dinv_u b_u + G_{u-s}^T x_{u-s} + A_{u+s}^T x_{u+s} for the eliminated vertices (x in z)
// A level reads only vertices the other levels wrote, so one barrier separates two levels.  The levels with more than BCR_TOP survivors
// run on the whole cluster through pcr_b / z in global memory, behind cluster barriers; from the first level with at most BCR_TOP survivors
// (l0) up and back down to l0, rank 0 alone works on the vertices at multiples of 2^l0 in shared memory behind __syncthreads (the camera
// path of 1 000 vertices: 6 cluster barriers; paths of up to 2 BCR_TOP vertices: none).  The path's operators are first pulled into L2 (the
// PCG's tile kernels evict them between two applies), and what a thread's next item needs besides the vector entries of the level before
// (its operator rows; going back also Dinv_u b_u) is read before the barrier that precedes the level.
// z is complete for the path only after a barrier of the whole cluster: the caller provides it before reading z written by other threads.
constexpr int BCR_TOP = 84;
template <int CL>
__device__ __forceinline__ double pcr_solve_path(const BaDev& d, cg::cluster_group& cl, int pb, int pe, const double* r, double* z) {
  __shared__ double sb[12 * BCR_TOP], sx[12 * BCR_TOP];      // b and x of the vertices j = q 2^l0, q < 2 BCR_TOP
  const int n = pe - pb, nl = pcr_num_levels(n), rank = (int)cl.block_rank();
  const int tid = rank * blockDim.x + threadIdx.x, nth = CL * blockDim.x;
  double* const b = d.pcr_b;
  int l0 = 0, slots = 0;
  #pragma unroll 1
  for (int l = 0; l < nl; ++l) { const int c = bcr_survivors(n, l); if (c > BCR_TOP) l0 = l + 1; slots += c; }
  {
    const double *A = d.pcr_A + 72 * (size_t)pb, *G = d.pcr_G + 72 * (size_t)pb, *Di = d.pcr_Dinv + 36 * (size_t)pb;
    for (int o = 16 * tid; o < 36 * slots; o += 16 * nth) {
      asm volatile("prefetch.global.L2 [%0];" ::"l"(A + o));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(G + o));
    }
    for (int o = 16 * tid; o < 36 * n; o += 16 * nth) asm volatile("prefetch.global.L2 [%0];" ::"l"(Di + o));
  }
  double p0[6], p1[6], x0 = 0.0, rz = 0.0;
  size_t off = 2 * (size_t)pb;
  // forward row of survivor item w at level l (stride s): rows of A_v, G_v of its slot; `end` = this thread's item bound
  auto fetch_fwd = [&](int w, int end, int s) {
    const int k = w / 6, i = w - 6 * k;
    const bool on = w < end, ia = on && k > 0, ig = on && 2 * s * k + s < n;
    const double* a = d.pcr_A + 36 * (off + k) + 6 * i; const double* g = d.pcr_G + 36 * (off + k) + 6 * i;
#pragma unroll
    for (int c = 0; c < 6; ++c) { p0[c] = ia ? a[c] : 0.0; p1[c] = ig ? g[c] : 0.0; }
  };
  // back row of eliminated item w at level l: columns of G_{u-s}, A_{u+s} and Dinv_u b_u, b_u read from bu(j)
  auto fetch_back = [&](int w, int end, int s, auto bu) {
    const int m = w / 6, i = w - 6 * m, j = s + 2 * s * m;
    const bool on = w < end, ia = on && j + s < n;
    const double* g = d.pcr_G + 36 * (off + m) + i; const double* a = d.pcr_A + 36 * (off + m + 1) + i;
#pragma unroll
    for (int c = 0; c < 6; ++c) { p0[c] = on ? g[6 * c] : 0.0; p1[c] = ia ? a[6 * c] : 0.0; }
    x0 = on ? dot6(d.pcr_Dinv + 36 * ((size_t)pb + j) + 6 * i, bu(j)) : 0.0;
  };
  auto row6 = [](const double* p, const double* x) { return p[0] * x[0] + p[1] * x[1] + p[2] * x[2] + p[3] * x[3] + p[4] * x[4] + p[5] * x[5]; };
  #pragma unroll 1
  for (int l = 0; l < l0; ++l) {                             // wide forward levels
    const int s = 1 << l, end = 6 * bcr_survivors(n, l);
    const double* src = l ? b : r;
    int w = tid;
    fetch_fwd(w, end, s);
    if (l) cl.sync();
    for (; w < end; w += nth) {
      const int k = w / 6, i = w - 6 * k, j = 2 * s * k;
      const size_t v = pb + j;
      double o = src[6 * v + i];
      if (k > 0) o += row6(p0, src + 6 * (v - s));
      if (j + s < n) o += row6(p1, src + 6 * (v + s));
      b[6 * v + i] = o;
      fetch_fwd(w + nth, end, s);
    }
    off += end / 6;
  }
  if (l0) cl.sync();
  const int S0 = 1 << l0, nq = (n - 1 + S0) >> l0;
  if (rank == 0) {                                           // the top of the reduction, in shared memory
    const int bd = (int)blockDim.x;
    const double* src = l0 ? b : r;
    for (int w = threadIdx.x; w < 6 * nq; w += bd) { const int q = w / 6; sb[w] = src[6 * ((size_t)pb + (size_t)q * S0) + w - 6 * q]; }
    #pragma unroll 1
    for (int l = l0; l < nl; ++l) {
      const int s = 1 << l, h = s >> l0, end = 6 * bcr_survivors(n, l);
      int w = threadIdx.x;
      fetch_fwd(w, end, s);
      __syncthreads();
      for (; w < end; w += bd) {
        const int k = w / 6, i = w - 6 * k, q = 2 * h * k;
        double o = sb[6 * q + i];
        if (k > 0) o += row6(p0, sb + 6 * (q - h));
        if (2 * s * k + s < n) o += row6(p1, sb + 6 * (q + h));
        sb[6 * q + i] = o;
        fetch_fwd(w + bd, end, s);
      }
      off += end / 6;
    }
    __syncthreads();
    if (threadIdx.x < 6) sx[threadIdx.x] = dot6(d.pcr_Dinv + 36 * (size_t)pb + 6 * threadIdx.x, sb);
    auto sbu = [&](int j) { return sb + 6 * (j >> l0); };
    #pragma unroll 1
    for (int l = nl - 1; l >= l0; --l) {
      const int s = 1 << l, h = s >> l0, end = 6 * bcr_eliminated(n, l);
      off -= bcr_survivors(n, l);
      int w = threadIdx.x;
      fetch_back(w, end, s, sbu);
      __syncthreads();
      for (; w < end; w += bd) {
        const int m = w / 6, i = w - 6 * m, q = h + 2 * h * m;
        double x = x0 + row6(p0, sx + 6 * (q - h));
        if (s + 2 * s * m + s < n) x += row6(p1, sx + 6 * (q + h));
        sx[6 * q + i] = x;
        fetch_back(w + bd, end, s, sbu);
      }
    }
    __syncthreads();
    for (int w = threadIdx.x; w < 6 * nq; w += bd) {
      const int q = w / 6; const size_t e = 6 * ((size_t)pb + (size_t)q * S0) + w - 6 * q;
      z[e] = sx[w]; rz += sx[w] * r[e];
    }
  }                                                          // (rank 0 leaves off where the top began: at level l0)
  #pragma unroll 1
  for (int l = l0 - 1; l >= 0; --l) {                        // wide back levels
    const int s = 1 << l, end = 6 * bcr_eliminated(n, l);
    const double* src = l ? b : r;
    off -= bcr_survivors(n, l);
    int w = tid;
    fetch_back(w, end, s, [&](int j) { return src + 6 * ((size_t)pb + j); });
    cl.sync();
    for (; w < end; w += nth) {
      const int m = w / 6, i = w - 6 * m, j = s + 2 * s * m;
      const size_t u = pb + j;
      double x = x0 + row6(p0, z + 6 * (u - s));
      if (j + s < n) x += row6(p1, z + 6 * (u + s));
      z[6 * u + i] = x; rz += x * r[6 * u + i];
      fetch_back(w + nth, end, s, [&](int jj) { return src + 6 * ((size_t)pb + jj); });
    }
  }
  return rz;
}

// Path-sharded preconditioner: the CTAs of one path publish their part of z (already in this rank's d.z) and their partial of r.z to
// every other rank; the last CTA of the launch to finish fences and raises this rank's flag of the second exchange on every rank.
template <int CL>
__device__ __forceinline__ void xchg_publish_z(const BaDev& d, cg::cluster_group& cl, int path, int pb, int pe, double rz_part, int* is_last_sm, unsigned int total_ctas) {
  const int tid = cl.block_rank() * blockDim.x + threadIdx.x, nth = CL * blockDim.x;
  const int pidx = path * PCR_CL + (int)cl.block_rank();
  if (threadIdx.x == 0) d.part_rz[pidx] = rz_part;
  if (!d.xg_paths) return;
  cl.sync();                                           // every CTA of the cluster wrote its share of z
  for (int r = 0; r < d.xg_world; ++r) {
    if (r == d.xg_rank) continue;
    double* zr = d.xg_slots[r] + d.xg_off_z;
    for (int w = tid; w < 6 * (pe - pb); w += nth) { const size_t q = 6 * (size_t)pb + w; zr[q] = d.z[q]; }
    if (threadIdx.x == 0) (d.xg_slots[r] + d.xg_off_prz)[pidx] = rz_part;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned int t = atomicAdd(d.ticket + 2, 1u);
    *is_last_sm = (t == total_ctas - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!*is_last_sm || threadIdx.x != 0) return;
  __threadfence_system();
  d.ticket[2] = 0u;
  const unsigned long long epoch = d.xg_epoch[192] + 1ull;
  d.xg_epoch[192] = epoch;
  for (int r = 0; r < d.xg_world; ++r) { volatile unsigned long long* f = d.xg_flags[r] + 320 + d.xg_rank; *f = epoch; }
}
// thread 0 of a CTA: wait until every rank's z part of the current epoch has arrived.  Returns false after ~2 s (a peer died).
__device__ __forceinline__ bool xchg_wait_z(const BaDev& d) {
  const unsigned long long epoch = d.xg_epoch[192];
  volatile unsigned long long* f = d.xg_flags[d.xg_rank] + 320;
  const long long t0 = clock64();
  for (int r = 0; r < d.xg_world; ++r)
    while (f[r] < epoch) if (clock64() - t0 > 4000000000ll) return false;
  __threadfence_system();
  return true;
}

template <int CL>
__device__ __forceinline__ void k_pcg_init_body(const BaDev& d, int path0, unsigned int total_ctas, int bx) {
  __shared__ double red[32];
  __shared__ int is_last;
  cg::cluster_group cl = cg::this_cluster();
  const int path = d.own_paths[path0 + bx / CL];
  const int pb = d.path_begin[path], pe = d.path_begin[path + 1];
  const int tid = cl.block_rank() * blockDim.x + threadIdx.x, nth = CL * blockDim.x;
  for (int w = tid; w < 6 * (pe - pb); w += nth) { const size_t q = 6 * (size_t)pb + w; d.r[q] = d.rhs[q]; d.xp[q] = 0.0; }
  if (pe - pb > 1) cl.sync();
  double rz = pcr_solve_path<CL>(d, cl, pb, pe, d.r, d.z);
  cl.sync();                                                 // z of the path is complete (its items were written by several CTAs)
  for (int w = tid; w < 6 * (pe - pb); w += nth) { const size_t q = 6 * (size_t)pb + w; d.p[q] = d.z[q]; }
  rz = block_sum(rz, red);
  if (threadIdx.x == 0) red[0] = rz;
  __syncthreads();
  xchg_publish_z<CL>(d, cl, path, pb, pe, red[0], &is_last, total_ctas);
}
template <class S, int CL>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(256, bcr_ctas_per_sm<S>()) k_pcg_init(S s) { VDO_PICK k_pcg_init_body<CL>(d, CL > 1 ? 0 : d.n_own_long, pcg_total_ctas(d), blk_); }
__device__ __forceinline__ void k_pcg_init_fin_body(const BaDev& d) {
  __shared__ double red[33];
  __shared__ int okw;
  if (d.xg_paths) {
    if (threadIdx.x == 0) okw = xchg_wait_z(d) ? 1 : 0;
    __syncthreads();
    if (!okw) { if (threadIdx.x == 0) d.scal[SC_DONE] = 3.0; return; }
  }
  const double rz = det_sum(d.part_rz, d.n_paths * PCR_CL, red);
  if (threadIdx.x != 0) return;
  d.scal[SC_RZ] = rz; d.scal[SC_RZ0] = rz; d.scal[SC_RZ_NEW] = 0.0; d.scal[SC_PAP] = 0.0; d.scal[SC_ITERS] = 0.0; d.scal[SC_BETA] = 0.0;
  d.scal[SC_DONE] = (rz > 0.0) ? 0.0 : 1.0;
}
template <class S>
__global__ void __launch_bounds__(256) k_pcg_init_fin(S s) { VDO_PICK (void)blk_; k_pcg_init_fin_body(d); }
__global__ void __launch_bounds__(256) k_pcg_dot(BaDev d) {
  __shared__ double red[32];
  if (d.scal[SC_DONE] != 0.0) return;
  const int n = d.C * 6;
  double s = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) s += d.p[i] * d.Ap[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) d.part_pap[blockIdx.x] = s;
}
// x += alpha p ; r -= alpha Ap ; z = M^-1 r ; rz_new += r.z.  FUSED: p is passed explicitly (double-buffered) and the last CTA to
// finish does the work of k_pcg_step_b's beta and of k_pcg_scalars.
template <bool FUSED, int CL>
__device__ __forceinline__ void k_pcg_step_a_body(const BaDev& d, const double* __restrict__ p, int path0, unsigned int total_ctas, int bx) {
  __shared__ double red[33];
  __shared__ int is_last;
  if (d.scal[SC_DONE] != 0.0) return;
  cg::cluster_group cl = cg::this_cluster();
  const double pap = det_sum(d.part_pap, d.n_part_pap, red), rz = d.scal[SC_RZ];
  const double alpha = (pap > 0.0) ? rz / pap : 0.0;
  const int path = d.own_paths[path0 + bx / CL];
  const int pb = d.path_begin[path], pe = d.path_begin[path + 1];
  const int tid = cl.block_rank() * blockDim.x + threadIdx.x, nth = CL * blockDim.x;
  for (int w = tid; w < 6 * (pe - pb); w += nth) { const size_t q = 6 * (size_t)pb + w; d.xp[q] += alpha * p[q]; d.r[q] -= alpha * d.Ap[q]; }
  if (pe - pb > 1) cl.sync();
  double rzn = pcr_solve_path<CL>(d, cl, pb, pe, d.r, d.z);
  rzn = block_sum(rzn, red);
  if (threadIdx.x == 0) red[0] = rzn;
  __syncthreads();
  xchg_publish_z<CL>(d, cl, path, pb, pe, red[0], &is_last, total_ctas);     // part_rz (and, path-sharded, z / part_rz on the other ranks)
  if (!FUSED || d.xg_paths) return;                           // path-sharded: k_pcg_scalars_x does the scalars once every part has arrived
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int t = atomicAdd(d.ticket, 1u);
    is_last = (t == total_ctas - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const double rz_new = det_sum(d.part_rz, d.n_paths * PCR_CL, red);
  if (threadIdx.x != 0) return;
  *d.ticket = 0u;
  if (!(pap > 0.0) || !isfinite(pap) || !isfinite(rz_new)) { d.scal[SC_DONE] = 2.0; return; }
  d.scal[SC_BETA] = rz_new / rz; d.scal[SC_RZ] = rz_new; d.scal[SC_ITERS] += 1.0;
  if (rz_new <= d.scal[SC_TOL2] * d.scal[SC_RZ0]) d.scal[SC_DONE] = 1.0;
}
// p_{k+1} is d.p for parity 1 and d.p2 for parity 0 (the non-fused iteration keeps p in d.p: parity 1)
template <class S, bool FUSED, int CL>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(256, bcr_ctas_per_sm<S>()) k_pcg_step_a(S s) {
  VDO_PICK k_pcg_step_a_body<FUSED, CL>(d, s.parity() ? d.p : d.p2, CL > 1 ? 0 : d.n_own_long, pcg_total_ctas(d), blk_);
}
// ---- fused PCG iteration (single GPU): 4 dependent launches per iteration instead of 8 ----
//   k_pcg_p_hpp            p_{k+1} = z + beta p_k (out of place, recomputed for the path neighbours), Ap = (Hpp + lambda I) p, vw / vh
//   k_tile_schur2 x 2      Hpl Hll^-1 Hlp p (band or static tiles, and chain tiles, forked)
//   k_tile_finalize_ap_dot Ap -= B^T sums, partials of p.Ap
//   k_pcg_step_a<true>     alpha, x, r, z = M^-1 r (block cyclic reduction; long-path clusters and short-path CTAs forked), partials of r.z; the LAST CTA to
//                          finish sums them (fixed order) and sets beta, rz, the iteration count and the convergence flag
// Eight lanes per vertex, lane r < 6 forming row r of the products (16 vertices per 128-thread CTA): with one thread per vertex, config 5
// (C = 13 416) left 4 warps per SM and the kernel waited on its dependent loads.  Row r adds its terms in the order of the 6x6 loops.
__device__ __forceinline__ void k_pcg_p_hpp_body(const BaDev& d, const double* __restrict__ p_in, double* __restrict__ p_out, double* __restrict__ out, int bx) {
  if (d.scal[SC_DONE] != 0.0) return;
  const double lambda = d.scal[SC_LAMBDA], beta = d.scal[SC_BETA];
  const int v = bx * (blockDim.x >> 3) + (threadIdx.x >> 3), r = threadIdx.x & 7;
  if (v >= d.C) return;                                      // the vertex's eight lanes leave together
  double xv[6];
#pragma unroll
  for (int c = 0; c < 6; ++c) xv[c] = d.z[6 * (size_t)v + c] + beta * p_in[6 * (size_t)v + c];
  if (r < 6) {
    const double xr = d.z[6 * (size_t)v + r] + beta * p_in[6 * (size_t)v + r];   // = xv[r] (registers are not indexed by lane)
    p_out[6 * (size_t)v + r] = xr;
    const double* H = d.Hpp + 36 * (size_t)v + 6 * r;
    double o = lambda * xr;
#pragma unroll
    for (int c = 0; c < 6; ++c) o += H[c] * xv[c];
    for (int n = d.nbr_begin[v]; n < d.nbr_begin[v + 1]; ++n) {
      const double* B = d.se_Hoff + 36 * (size_t)d.nbr_edge[n];
      const size_t u = 6 * (size_t)d.nbr_other[n];
      double xo[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) xo[c] = d.z[u + c] + beta * p_in[u + c];
      if (d.nbr_tr[n]) {
#pragma unroll
        for (int c = 0; c < 6; ++c) o += B[6 * c + r] * xo[c];
      } else {
#pragma unroll
        for (int c = 0; c < 6; ++c) o += B[6 * r + c] * xo[c];
      }
    }
    out[6 * (size_t)v + r] = d.own ? o : 0.0;
  }
  __syncwarp(0xffu << (threadIdx.x & 24));                   // p_out of the vertex is written
  if (r == 0) body_vertex_transform(d, v, p_out, d.vw);
}
// parity 0 reads p and writes p2, parity 1 the other way round
template <class S>
__global__ void __launch_bounds__(128) k_pcg_p_hpp(S s) { VDO_PICK k_pcg_p_hpp_body(d, s.parity() ? d.p2 : d.p, s.parity() ? d.p : d.p2, d.Ap, blk_); }

// ---- sharded PCG iteration: all-reduce of the 6C-vector S*p through peer memory (NVLink), inside the captured graph ----
// Every rank holds, for each sender r, a slot of 6C doubles (double-buffered by the parity of an epoch counter).
//   k_xchg_scatter  per vertex: this rank's partial (Hpp p on rank 0) - B^T (tile sums), stored straight into slot[rank] of EVERY
//                   rank (remote stores); the last CTA to finish fences (system scope), bumps the epoch and stores it into
//                   flag[rank] of every rank
//   k_xchg_reduce   waits until all world flags carry the epoch, then sums the world slots IN RANK ORDER -- every rank adds the
//                   same numbers in the same order, so Ap (and with it every PCG scalar and the convergence flag) is bit-identical
//                   on all ranks -- and forms the CTA's share of p.Ap
// Nothing here is enqueued by the host per iteration: the kernels are ordinary graph nodes.
__global__ void __launch_bounds__(128) k_xchg_scatter(BaDev d, double sign, const double* __restrict__ own_part) {
  __shared__ int is_last;
  if (d.scal[SC_DONE] != 0.0) return;
  const unsigned long long epoch = *d.xg_epoch + 1ull;            // the epoch this vector belongs to (bumped below by the last CTA)
  const size_t n6 = 6 * (size_t)d.C;
  const size_t slot = ((epoch & 1ull) * (size_t)d.xg_world + (size_t)d.xg_rank) * n6;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < d.C) {
    const double* T = d.se3 + 12 * (size_t)v;
    double* a = d.acc6 + 12 * (size_t)v;
    const double F[3] = {a[0] + a[6], a[1] + a[7], a[2] + a[8]};
    const double G[3] = {2 * a[0] + a[6], 2 * a[1] + a[7], 2 * a[2] + a[8]};
    double txg[3]; cross3(T + 9, G, txg);
    const double M[3] = {a[3] + a[9] - txg[0], a[4] + a[10] - txg[1], a[5] + a[11] - txg[2]};
    double o0[3], o1[3];
    rot_t_apply(T, F, o0); rot_t_apply(T, M, o1);
    const double* op = own_part + 6 * (size_t)v;
    const double o[6] = {op[0] + sign * o0[0], op[1] + sign * o0[1], op[2] + sign * o0[2], op[3] + sign * o1[0], op[4] + sign * o1[1], op[5] + sign * o1[2]};
#pragma unroll
    for (int i = 0; i < 12; ++i) a[i] = 0.0;
    for (int r = 0; r < d.xg_world; ++r) {
      double* dst = d.xg_slots[r] + slot + 6 * (size_t)v;
#pragma unroll
      for (int i = 0; i < 6; ++i) dst[i] = o[i];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned int t = atomicAdd(d.ticket + 1, 1u);
    is_last = (t == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!is_last || threadIdx.x != 0) return;
  __threadfence_system();
  d.ticket[1] = 0u;
  *d.xg_epoch = epoch;
  for (int r = 0; r < d.xg_world; ++r) {
    volatile unsigned long long* f = d.xg_flags[r] + d.xg_rank;
    *f = epoch;
  }
}
__global__ void __launch_bounds__(128) k_xchg_reduce(BaDev d, double* __restrict__ out, const double* __restrict__ pdot) {
  __shared__ double red[32];
  __shared__ int failed;
  if (d.scal[SC_DONE] != 0.0) return;
  const unsigned long long epoch = *d.xg_epoch;
  if (threadIdx.x == 0) {
    failed = 0;
    volatile unsigned long long* f = d.xg_flags[d.xg_rank];
    const long long t0 = clock64();
    for (int r = 0; r < d.xg_world; ++r)
      while (f[r] < epoch) {
        if (clock64() - t0 > 4000000000ll) { failed = 1; break; }       // ~2 s: a peer died; do not hang the GPU
      }
    __threadfence_system();
  }
  __syncthreads();
  if (failed) { if (threadIdx.x == 0 && blockIdx.x == 0) d.scal[SC_DONE] = 3.0; return; }
  const size_t n6 = 6 * (size_t)d.C;
  const double* base = d.xg_slots[d.xg_rank] + (epoch & 1ull) * (size_t)d.xg_world * n6;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  double s = 0.0;
  if (v < d.C) {
    double o[6] = {0, 0, 0, 0, 0, 0};
    for (int r = 0; r < d.xg_world; ++r) {
      const volatile double* src = base + (size_t)r * n6 + 6 * (size_t)v;
#pragma unroll
      for (int i = 0; i < 6; ++i) o[i] += src[i];
    }
    const double* pv = pdot + 6 * (size_t)v;
#pragma unroll
    for (int i = 0; i < 6; ++i) { out[6 * (size_t)v + i] = o[i]; s += pv[i] * o[i]; }
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) d.part_pap[blockIdx.x] = s;
}

__global__ void __launch_bounds__(256) k_pcg_step_b(BaDev d) {
  __shared__ double red[33];
  if (d.scal[SC_DONE] != 0.0) return;
  const double beta = det_sum(d.part_rz, d.n_paths * PCR_CL, red) / d.scal[SC_RZ];
  const int n = d.C * 6;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) d.p[i] = d.z[i] + beta * d.p[i];
}
__global__ void __launch_bounds__(256) k_pcg_scalars(BaDev d) {
  __shared__ double red[33];
  if (d.scal[SC_DONE] != 0.0) return;
  const double tol2 = d.scal[SC_TOL2];
  const double pap = det_sum(d.part_pap, d.n_part_pap, red);
  const double rzn = det_sum(d.part_rz, d.n_paths * PCR_CL, red);
  if (threadIdx.x != 0) return;
  if (!(pap > 0.0) || !isfinite(pap) || !isfinite(rzn)) { d.scal[SC_DONE] = 2.0; return; }
  d.scal[SC_RZ] = rzn; d.scal[SC_RZ_NEW] = 0.0; d.scal[SC_PAP] = 0.0; d.scal[SC_ITERS] += 1.0;
  if (rzn <= tol2 * d.scal[SC_RZ0]) d.scal[SC_DONE] = 1.0;
}

// path-sharded preconditioner: waits for every rank's part of z / r.z, then the scalars of k_pcg_step_a<true>'s last CTA (identical on all ranks)
__global__ void __launch_bounds__(256) k_pcg_scalars_x(BaDev d) {
  __shared__ double red[33];
  __shared__ int okw;
  if (d.scal[SC_DONE] != 0.0) return;
  if (threadIdx.x == 0) okw = xchg_wait_z(d) ? 1 : 0;
  __syncthreads();
  if (!okw) { if (threadIdx.x == 0) d.scal[SC_DONE] = 3.0; return; }
  const double pap = det_sum(d.part_pap, d.n_part_pap, red);
  const double rz_new = det_sum(d.part_rz, d.n_paths * PCR_CL, red);
  if (threadIdx.x != 0) return;
  const double rz = d.scal[SC_RZ];
  if (!(pap > 0.0) || !isfinite(pap) || !isfinite(rz_new)) { d.scal[SC_DONE] = 2.0; return; }
  d.scal[SC_BETA] = rz_new / rz; d.scal[SC_RZ] = rz_new; d.scal[SC_ITERS] += 1.0;
  if (rz_new <= d.scal[SC_TOL2] * d.scal[SC_RZ0]) d.scal[SC_DONE] = 1.0;
}

// ---- dense reduced system for small static-only graphs (NS1) ----
// S (n x n, n = 6C, row-major, lower triangle used) = Hpp + lambda I (+ se3-se3 off-diagonal blocks) - sum_j (1 / s_j) H_pl,j H_pl,j^T, rhs = bp - sum_j H_pl,j b_l,j / s_j
// with H_pl for an EdgeSE3PointXYZ = om J_c^T J_p, J_c = [-I | 2 [Zc]x], J_p = R_c^T (edge_se3_pointxyz.cpp:99-140).
__device__ __forceinline__ void k_dense_init_body(const BaDev& d, double lambda, int n, int bx) {
  const int i = bx * blockDim.x + threadIdx.x;
  double* S = d.Sdense; double* rhs = S + (size_t)n * n;
  if (i < n * n) {
    const int r = i / n, c = i % n, vr = r / 6, vc = c / 6;
    double v = 0.0;
    if (vr == vc) { v = d.Hpp[36 * (size_t)vr + 6 * (r % 6) + (c % 6)]; if (r == c) v += lambda; }
    S[i] = v;
  }
  if (i < n) rhs[i] = d.bp[i];
  if (i == 0) rhs[n] = 0.0;                       // status word: != 0 after the factorisation means "not positive definite"
}
template <class S>
__global__ void __launch_bounds__(128) k_dense_init(S s) { VDO_PICK k_dense_init_body(d, s.lambda(g_), 6 * d.C, blk_); }
__device__ __forceinline__ void k_dense_se3_edges_body(const BaDev& d, int n, int bx) {
  const int e = bx * blockDim.x + threadIdx.x;
  if (e >= d.Ese || d.se_j[e] < 0) return;
  const int i = d.se_i[e], j = d.se_j[e];
  const double* H = d.se_Hoff + 36 * (size_t)e;    // J_i^T W J_j: rows i, columns j
  double* S = d.Sdense;
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) {
      if (i > j) atomicAdd(S + (size_t)(6 * i + r) * n + 6 * j + c, H[6 * r + c]);
      else atomicAdd(S + (size_t)(6 * j + c) * n + 6 * i + r, H[6 * r + c]);
    }
}
template <class S>
__global__ void __launch_bounds__(64) k_dense_se3_edges(S s) { VDO_PICK k_dense_se3_edges_body(d, 6 * d.C, blk_); }
__device__ __forceinline__ void k_dense_schur_body(const BaDev& d, int n, int bx) {
  const int k = bx * blockDim.x + threadIdx.x;
  if (k >= d.P) return;
  const int eb = d.lm_obs_begin[k], ee = d.lm_obs_begin[k + 1];
  if (ee <= eb) return;
  const double is = 1.0 / d.pt_s[k];
  const double p[3] = {d.pt[3 * (size_t)k], d.pt[3 * (size_t)k + 1], d.pt[3 * (size_t)k + 2]};
  const double bls[3] = {d.bl[3 * (size_t)k] * is, d.bl[3 * (size_t)k + 1] * is, d.bl[3 * (size_t)k + 2] * is};
  double* S = d.Sdense; double* rhs = S + (size_t)n * n;
  // M_c = om J_c^T R_c^T (6 x 3): rows 0-2 = -om R^T, rows 3-5 = om (2 [Zc]x)^T R^T
  auto make_M = [&](int e, double* M) -> int {
    const int c = d.lm_cam[e];
    const double* T = d.se3 + 12 * (size_t)c;
    const double w[3] = {p[0] - T[9], p[1] - T[10], p[2] - T[11]};
    double Zc[3]; rot_t_apply(T, w, Zc);
    const double om = d.lm_omega[e];
    // 2 [Zc]x = [[0, -2z, 2y], [2z, 0, -2x], [-2y, 2x, 0]];  J_c^T rows 3-5 = (2 [Zc]x)^T
    const double A[9] = {0, 2 * Zc[2], -2 * Zc[1], -2 * Zc[2], 0, 2 * Zc[0], 2 * Zc[1], -2 * Zc[0], 0};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        M[3 * r + q] = -om * T[3 * q + r];                                                  // -om R^T
        M[9 + 3 * r + q] = om * (A[3 * r] * T[3 * q] + A[3 * r + 1] * T[3 * q + 1] + A[3 * r + 2] * T[3 * q + 2]);   // om A R^T
      }
    return c;
  };
  for (int e1 = eb; e1 < ee; ++e1) {
    double M1[18]; const int c1 = make_M(e1, M1);
#pragma unroll
    for (int r = 0; r < 6; ++r) atomicAdd(rhs + 6 * c1 + r, -(M1[3 * r] * bls[0] + M1[3 * r + 1] * bls[1] + M1[3 * r + 2] * bls[2]));
    for (int e2 = eb; e2 < ee; ++e2) {
      double M2[18]; const int c2 = make_M(e2, M2);
      if (c2 > c1) continue;                                                                  // lower triangle (blocks with c1 >= c2)
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          atomicAdd(S + (size_t)(6 * c1 + r) * n + 6 * c2 + q, -is * (M1[3 * r] * M2[3 * q] + M1[3 * r + 1] * M2[3 * q + 1] + M1[3 * r + 2] * M2[3 * q + 2]));
        }
    }
  }
}
template <class S>
__global__ void __launch_bounds__(128) k_dense_schur(S s) { VDO_PICK k_dense_schur_body(d, 6 * d.C, blk_); }
// S += the static Schur term from the band (see k_band_form / k_band_mul): block (row vertex b = a + k, column vertex a) = Y_b Kc X_a with
//   X_a = [[-R, -2 [t]x R], [0, R]]  (local increment -> the world-frame vector vw of body_vertex_transform),
//   Kc  = [[M0 I, 2 [M1]x], [2 [M1]x, 4 (M2 - tr(M2) I)]]  (the band product, sign folded in),
//   Y_b = [[R^T, 0], [-2 R^T [t]x, R^T]]  (k_tile_finalize_schur2: torque moved to the vertex origin, rotated into the vertex frame).
// One thread per (a, k); every block is written by exactly one thread (no atomics -- the thread-per-landmark k_dense_schur issued
// ~600 fp64 atomics per landmark onto the 20 x 20 blocks and was dominated by their contention).
__device__ __forceinline__ void k_dense_from_band_body(const BaDev& d, int n, int bx) {
  const int idx = bx * blockDim.x + threadIdx.x;
  const int W = d.band_W;
  if (idx >= d.band_n * W) return;
  const int a = idx / W, k = idx - a * W, b = a + k;
  if (b >= d.band_n) return;
  const double* m = d.band + (size_t)idx * 10;
  if (m[0] == 0.0) return;
  const int va = d.band_v0 + a, vb = d.band_v0 + b;
  const double* Ta = d.se3 + 12 * (size_t)va; const double* Tb = d.se3 + 12 * (size_t)vb;
  auto skew = [](const double* t, double* K) { K[0] = 0; K[1] = -t[2]; K[2] = t[1]; K[3] = t[2]; K[4] = 0; K[5] = -t[0]; K[6] = -t[1]; K[7] = t[0]; K[8] = 0; };
  double X[36], Kc[36], Z[36];
  {   // X_a
    double tx[9]; skew(Ta + 9, tx);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        const double txr = tx[3 * r] * Ta[c] + tx[3 * r + 1] * Ta[3 + c] + tx[3 * r + 2] * Ta[6 + c];     // ([t]x R)[r][c]
        X[6 * r + c] = -Ta[3 * r + c]; X[6 * r + 3 + c] = -2.0 * txr;
        X[6 * (r + 3) + c] = 0.0; X[6 * (r + 3) + 3 + c] = Ta[3 * r + c];
      }
  }
  {   // Kc
    const double m1[3] = {m[1], m[2], m[3]};
    double m1x[9]; skew(m1, m1x);
    const double M2[9] = {m[4], m[5], m[6], m[5], m[7], m[8], m[6], m[8], m[9]};
    const double tr = m[4] + m[7] + m[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        Kc[6 * r + c] = (r == c) ? m[0] : 0.0; Kc[6 * r + 3 + c] = 2.0 * m1x[3 * r + c];
        Kc[6 * (r + 3) + c] = 2.0 * m1x[3 * r + c]; Kc[6 * (r + 3) + 3 + c] = 4.0 * (M2[3 * r + c] - (r == c ? tr : 0.0));
      }
  }
  mat6_mul(Kc, X, Z);
  double Y[36];
  {   // Y_b
    double tx[9]; skew(Tb + 9, tx);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        const double rtx = Tb[r] * tx[c] + Tb[3 + r] * tx[3 + c] + Tb[6 + r] * tx[6 + c];                   // (R^T [t]x)[r][c]
        Y[6 * r + c] = Tb[3 * c + r]; Y[6 * r + 3 + c] = 0.0;
        Y[6 * (r + 3) + c] = -2.0 * rtx; Y[6 * (r + 3) + 3 + c] = Tb[3 * c + r];
      }
  }
  double B[36];
  mat6_mul(Y, Z, B);
  double* S = d.Sdense;
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) S[(size_t)(6 * vb + r) * n + 6 * va + c] += B[6 * r + c];
}
template <class S>
__global__ void __launch_bounds__(128) k_dense_from_band(S s) { VDO_PICK k_dense_from_band_body(d, 6 * d.C, blk_); }
// One CTA: blocked right-looking Cholesky of the lower triangle of S in shared memory (8-column panels; the trailing update
// A[i][j] -= L[i][k] L[j][k]^T over 8x8 tiles is two mma.sync.m8n8k4.f64 per tile), then the two triangular solves.  n <= DENSE_MAX.
constexpr int DENSE_MAX = 168;
__device__ __forceinline__ void dmma_m8n8k4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void k_dense_chol_body(const BaDev& d, int n, int bx) {
  extern __shared__ double sA[];                    // npad x ld, row-major; ld = npad + 1 (bank spread)
  const int npad = (n + 7) & ~7, ld = npad + 1;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  double* S = d.Sdense; double* rhs = S + (size_t)n * n;
  __shared__ int bad;
  if (tid == 0) bad = 0;
  for (int i = tid; i < npad * npad; i += blockDim.x) {
    const int r = i / npad, c = i % npad;
    double v = 0.0;
    if (r < n && c < n) v = (c <= r) ? S[(size_t)r * n + c] : S[(size_t)c * n + r];   // mirror the lower triangle (block (c1 == c2) parts were written in full)
    else if (r == c) v = 1.0;                                                        // padding: identity
    sA[r * ld + c] = v;
  }
  __syncthreads();
  const int nb = npad / 8;
  for (int kb = 0; kb < nb; ++kb) {
    const int k0 = 8 * kb;
    if (warp == 0) {                                // 8 x 8 diagonal block, unblocked (lanes = rows)
      for (int j = 0; j < 8; ++j) {
        double djj = sA[(k0 + j) * ld + k0 + j];
        if (!(djj > 0.0)) { if (lane == 0) bad = 1; djj = 1.0; }
        const double l = sqrt(djj);
        __syncwarp();
        if (lane == j) sA[(k0 + j) * ld + k0 + j] = l;
        if (lane > j && lane < 8) sA[(k0 + lane) * ld + k0 + j] /= l;
        __syncwarp();
        if (lane > j && lane < 8) {
          const double lij = sA[(k0 + lane) * ld + k0 + j];
          for (int c = j + 1; c <= lane; ++c) sA[(k0 + lane) * ld + k0 + c] -= lij * sA[(k0 + c) * ld + k0 + j];
        }
        __syncwarp();
      }
    }
    __syncthreads();
    // panel: rows below the diagonal block solve x L_kk^T = a (one thread per row)
    for (int r = k0 + 8 + tid; r < npad; r += blockDim.x) {
      double x[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        double s = sA[r * ld + k0 + j];
#pragma unroll
        for (int c = 0; c < j; ++c) s -= x[c] * sA[(k0 + j) * ld + k0 + c];
        x[j] = s / sA[(k0 + j) * ld + k0 + j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) sA[r * ld + k0 + j] = x[j];
    }
    __syncthreads();
    // trailing update on the fp64 tensor cores: tile (ib, jb), ib >= jb > kb:  A_ij -= L_ik L_jk^T
    const int nt = nb - kb - 1, ntiles = nt * (nt + 1) / 2;
    for (int t = warp; t < ntiles; t += nw) {
      int a = 0, rem = t;
      while (rem >= nt - a) { rem -= nt - a; ++a; }
      const int jb = kb + 1 + a, ib = jb + rem;
      const int g = lane >> 2, q = lane & 3;        // fragment coordinates: A row g / col q (+4), B row q (+4) / col g, C row g / cols 2q, 2q + 1
      double c0 = 0.0, c1 = 0.0;
      dmma_m8n8k4(c0, c1, sA[(8 * ib + g) * ld + k0 + q], sA[(8 * jb + g) * ld + k0 + q]);
      dmma_m8n8k4(c0, c1, sA[(8 * ib + g) * ld + k0 + 4 + q], sA[(8 * jb + g) * ld + k0 + 4 + q]);
      sA[(8 * ib + g) * ld + 8 * jb + 2 * q] -= c0;
      sA[(8 * ib + g) * ld + 8 * jb + 2 * q + 1] -= c1;
    }
    __syncthreads();
  }
  // L y = rhs, L^T x = y (warp 0; n is small)
  __shared__ double y[DENSE_MAX];
  for (int i = tid; i < npad; i += blockDim.x) y[i] = i < n ? rhs[i] : 0.0;
  __syncthreads();
  if (warp == 0) {
    for (int i = 0; i < n; ++i) {
      double s = 0.0;
      for (int c = lane; c < i; c += 32) s += sA[i * ld + c] * y[c];
      s = warp_sum(s);
      if (lane == 0) y[i] = (y[i] - s) / sA[i * ld + i];
      __syncwarp();
    }
    for (int i = n - 1; i >= 0; --i) {
      double s = 0.0;
      for (int c = i + 1 + lane; c < n; c += 32) s += sA[c * ld + i] * y[c];
      s = warp_sum(s);
      if (lane == 0) y[i] = (y[i] - s) / sA[i * ld + i];
      __syncwarp();
    }
  }
  __syncthreads();
  for (int i = tid; i < n; i += blockDim.x) d.xp[i] = y[i];
  if (tid == 0) rhs[n] = bad ? 1.0 : 0.0;
}
template <class S>
__global__ void __launch_bounds__(256) k_dense_chol(S s) { VDO_PICK k_dense_chol_body(d, 6 * d.C, blk_); }

__device__ __forceinline__ void k_apply_update_body(const BaDev& d, double lambda, int reortho, int bx) {
  __shared__ double red[32];
  const int i = bx * blockDim.x + threadIdx.x;
  double s = 0.0;
  if (i < d.C) s = body_update_se3(d, i, lambda, reortho != 0);
  else if (i < d.C + d.P) s = body_update_pt(d, i - d.C, lambda);
  s = block_sum(s, red);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(d.scal + SC_SCALE, s);
}
template <class S>
__global__ void __launch_bounds__(128) k_apply_update(S s) { VDO_PICK k_apply_update_body(d, s.lambda(g_), s.reortho(g_), blk_); }

}  // namespace vdo
#include "ba_tile_kernels.cuh"
namespace vdo {

constexpr int BATCH_PARAMS_MAX = 64;
struct BatchParams { int n0, n; int flags[BATCH_PARAMS_MAX], reortho[BATCH_PARAMS_MAX]; double lambda[BATCH_PARAMS_MAX], tol2[BATCH_PARAMS_MAX]; };
__global__ void k_batch_params(BatchDev B, BatchParams p) {
  const int i = threadIdx.x;
  if (i < p.n) { B.flags[p.n0 + i] = p.flags[i]; B.lambda[p.n0 + i] = p.lambda[i]; B.reortho[p.n0 + i] = p.reortho[i]; B.tol2[p.n0 + i] = p.tol2[i]; }
}
// the PCG init of a batch stores every graph's lambda and tolerance where the iteration kernels read them (the lone graph: set_scalars)
__global__ void k_batch_scalars(BatchDev B, int bit) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < B.n && (B.flags[g] & bit)) { B.ds[g].scal[SC_LAMBDA] = B.lambda[g]; B.ds[g].scal[SC_TOL2] = B.tol2[g]; }
}
#undef VDO_PICK

// ---------------------------------------------------------------------------------------------------------------
// NCCL is resolved at run time (dlopen) so that the library links without it and picks up the copy torch already loaded
struct NcclApi {
  void* h = nullptr;
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclAllReduce) AllReduce = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  bool load() {
    if (h) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (h) break; }
    if (!h) return false;
    GetUniqueId = (decltype(GetUniqueId))dlsym(h, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(h, "ncclCommInitRank");
    CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
    AllReduce = (decltype(AllReduce))dlsym(h, "ncclAllReduce");
    AllGather = (decltype(AllGather))dlsym(h, "ncclAllGather");
    GetErrorString = (decltype(GetErrorString))dlsym(h, "ncclGetErrorString");
    return GetUniqueId && CommInitRank && CommDestroy && AllReduce;
  }
};
static NcclApi g_nccl;

// the scalar blocks of up to GATHER_MAX graphs, copied into one contiguous buffer for a single read-back
constexpr int GATHER_MAX = 64;
struct GatherSrc { const double* src[GATHER_MAX]; int n, len; };
__global__ void __launch_bounds__(256) k_gather_scalars(GatherSrc g, double* out) {
  for (int i = threadIdx.x; i < g.n * g.len; i += blockDim.x) out[i] = g.src[i / g.len][i % g.len];
}

struct CudaBackend : BaBackend {
  int dev = 0;
  int n_sm = 132;                        // SMs of the device (grid sizes of the grid-stride kernels)
  ncclComm_t comm = nullptr;
  void allreduce_sum(double* b, size_t n) override {
    if (world <= 1 || n == 0) return;
    ncclResult_t r = g_nccl.AllReduce(b, b, n, ncclDouble, ncclSum, comm, st);
    if (r != ncclSuccess) std::fprintf(stderr, "[vdo_b200] ncclAllReduce failed: %s\n", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    ++n_coll;
  }
  void allreduce_max(double* b, size_t n) override {
    if (world <= 1 || n == 0) return;
    ncclResult_t r = g_nccl.AllReduce(b, b, n, ncclDouble, ncclMax, comm, st);
    if (r != ncclSuccess) std::fprintf(stderr, "[vdo_b200] ncclAllReduce failed: %s\n", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    ++n_coll;
  }
  int n_coll = 0;
  // ---- peer-memory exchange of the sharded PCG iteration: one buffer per rank (flags + 2 x world slots of 6C doubles), mapped into every
  //      other rank through CUDA IPC (handles all-gathered over NCCL once per buffer size) ----
  struct Xchg {
    char* local = nullptr; size_t bytes = 0, off_z = 0, off_prz = 0; int C = 0, n_paths = 0; bool ok = false, tried = false;
    std::vector<char*> peer;                 // peer[r]: this process' mapping of rank r's buffer (peer[rank] == local)
    double** d_slots = nullptr; unsigned long long** d_flags = nullptr; unsigned long long* d_epoch = nullptr;
  } xg;
  static constexpr size_t XG_HDR = 4096;     // flags (world x u64) + epoch live in the first page of the buffer
  void xchg_release() {
    drop_graphs();                           // captured PCG graphs carry the buffer's addresses
    for (size_t r = 0; r < xg.peer.size(); ++r) if ((int)r != rank && xg.peer[r]) cudaIpcCloseMemHandle(xg.peer[r]);
    xg.peer.clear();
    if (xg.local) cudaFree(xg.local);
    if (xg.d_slots) cudaFree(xg.d_slots);
    if (xg.d_flags) cudaFree(xg.d_flags);
    xg = Xchg();
  }
  // collective: every rank calls it with the same C.  Returns false (and the caller falls back to NCCL all-reduces) when peer mapping is unavailable.
  bool xchg_setup(int C, int n_paths) {
    if (xg.ok && xg.C >= C && xg.n_paths >= n_paths) return true;
    if (xg.tried && !xg.ok) return false;
    if (std::getenv("VDO_NO_PEER_EXCHANGE")) { xg.tried = true; return false; }
    CK(cudaStreamSynchronize(st));
    xchg_release();
    xg.tried = true; xg.C = C; xg.n_paths = n_paths;
    // header | 2 x world slots of 6C | z (6C) | part_rz (n_paths x PCR_CL)
    xg.off_z = 2 * (size_t)world * 6 * (size_t)C; xg.off_prz = xg.off_z + 6 * (size_t)C;
    xg.bytes = XG_HDR + sizeof(double) * (xg.off_prz + (size_t)n_paths * PCR_CL + 2);
    bool good = g_nccl.AllGather != nullptr;
    if (good && cudaMalloc(&xg.local, xg.bytes) != cudaSuccess) { cudaGetLastError(); xg.local = nullptr; good = false; }
    if (good) CK(cudaMemsetAsync(xg.local, 0, xg.bytes, st));
    cudaIpcMemHandle_t mine; std::memset(&mine, 0, sizeof mine);
    if (good && cudaIpcGetMemHandle(&mine, xg.local) != cudaSuccess) { cudaGetLastError(); good = false; }
    // all-gather {ok flag, handle} -- also the agreement on whether every rank got this far
    struct Rec { int ok; int pad; cudaIpcMemHandle_t h; };
    Rec rec; rec.ok = good ? 1 : 0; rec.pad = 0; rec.h = mine;
    char* d_all = nullptr; CK(cudaMalloc(&d_all, sizeof(Rec) * (size_t)world));
    CK(cudaMemcpyAsync(d_all + sizeof(Rec) * (size_t)rank, &rec, sizeof(Rec), cudaMemcpyHostToDevice, st));
    if (g_nccl.AllGather) {
      ncclResult_t r = g_nccl.AllGather(d_all + sizeof(Rec) * (size_t)rank, d_all, sizeof(Rec), ncclChar, comm, st);
      if (r != ncclSuccess) good = false;
    }
    std::vector<Rec> all(world);
    CK(cudaMemcpyAsync(all.data(), d_all, sizeof(Rec) * (size_t)world, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    cudaFree(d_all);
    for (int r = 0; r < world; ++r) if (!all[r].ok) good = false;
    if (good) {
      xg.peer.assign(world, nullptr);
      for (int r = 0; r < world && good; ++r) {
        if (r == rank) { xg.peer[r] = xg.local; continue; }
        void* ptr = nullptr;
        if (cudaIpcOpenMemHandle(&ptr, all[r].h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); good = false; }
        xg.peer[r] = (char*)ptr;
      }
    }
    // agree on the outcome (a rank that failed to map a peer must take every rank down to the NCCL path)
    double flag = good ? 0.0 : 1.0, *d_flag = nullptr;
    CK(cudaMalloc(&d_flag, sizeof(double)));
    CK(cudaMemcpyAsync(d_flag, &flag, sizeof(double), cudaMemcpyHostToDevice, st));
    allreduce_sum(d_flag, 1);
    CK(cudaMemcpyAsync(&flag, d_flag, sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    cudaFree(d_flag);
    if (flag != 0.0) { xchg_release(); xg.tried = true; std::fprintf(stderr, "[vdo_b200] rank %d: peer-memory exchange unavailable, using NCCL all-reduces per PCG iteration\n", rank); return false; }
    std::vector<double*> hs(world); std::vector<unsigned long long*> hf(world);
    for (int r = 0; r < world; ++r) { hf[r] = (unsigned long long*)xg.peer[r]; hs[r] = (double*)(xg.peer[r] + XG_HDR); }
    CK(cudaMalloc(&xg.d_slots, sizeof(double*) * (size_t)world)); CK(cudaMalloc(&xg.d_flags, sizeof(unsigned long long*) * (size_t)world));
    CK(cudaMemcpyAsync(xg.d_slots, hs.data(), sizeof(double*) * (size_t)world, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(xg.d_flags, hf.data(), sizeof(unsigned long long*) * (size_t)world, cudaMemcpyHostToDevice, st));
    xg.d_epoch = (unsigned long long*)(xg.local + 8 * 256);       // behind the flags (world <= 256)
    CK(cudaStreamSynchronize(st));
    xg.ok = true;
    return true;
  }
  cudaStream_t st = nullptr, st2 = nullptr;   // st2: second branch inside the captured PCG graph
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  int n_launch = 0;
  cudaEvent_t ev0[4], ev1[4];
  ~CudaBackend() override {
    for (int i = 0; i < 4; ++i) { cudaEventDestroy(ev0[i]); cudaEventDestroy(ev1[i]); }
    if (gather_buf) free_(gather_buf);
    for (auto& kv : pool) cudaFree(kv.second);
    arena.destroy();
    xchg_release();
    if (comm) g_nccl.CommDestroy(comm);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (st2) cudaStreamDestroy(st2);
    if (st) cudaStreamDestroy(st);
  }
  // pinned staging arena (graph ingestion builds its upload streams in it) and a caching device allocator: graphs of the
  // same shape are created again and again by the callers (one per window / per solve), so freed blocks are kept and
  // handed back by exact size instead of going through cudaFree / cudaMalloc (both synchronise the device)
  struct PinnedArena : HostArena {
    char* raw_alloc(size_t b) override { void* p = nullptr; if (cudaHostAlloc(&p, b, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); p = std::malloc(b); pageable.insert(p); } return (char*)p; }
    void raw_free(char* p) override { if (pageable.count(p)) { pageable.erase(p); std::free(p); } else cudaFreeHost(p); }
    std::set<void*> pageable;
  } arena;
  HostArena& staging() override { return arena; }
  std::multimap<size_t, void*> pool;      // free device blocks by size
  std::map<void*, size_t> live;           // size of every block handed out
  size_t pool_bytes = 0;
  static constexpr size_t POOL_MAX = (size_t)24 << 30;
  // size classes: 1/16 steps of the enclosing power of two (<= 12.5 % slack), powers of two up to 4 KB -- callers such as the per-window
  // optimiser build graphs whose array sizes differ by a few elements from run to run; with exact sizes every buffer missed the cache
  // (~100 cudaMalloc per graph, with occasional long stalls when the driver grew its heap)
  static size_t size_class(size_t b) {
    size_t p2 = 256;
    while (p2 < b) p2 <<= 1;
    if (p2 <= 4096) return p2;
    const size_t step = p2 >> 4;
    return (b + step - 1) / step * step;
  }
  void* alloc(size_t b) override {
    b = b ? b : 8;
    const size_t cls = size_class(b);
    void* p = nullptr;
    auto it = pool.find(cls);
    if (it != pool.end()) { p = it->second; pool_bytes -= cls; pool.erase(it); }
    else CK(cudaMalloc(&p, cls));
    live[p] = cls;
    CK(cudaMemsetAsync(p, 0, b, st));
    return p;
  }
  void free_(void* p) override {
    auto it = live.find(p);
    if (it == live.end()) { cudaFree(p); return; }
    const size_t b = it->second;
    live.erase(it);
    if (pool_bytes + b <= POOL_MAX) { pool.emplace(b, p); pool_bytes += b; }   // all users are ordered on st: no synchronisation needed
    else cudaFree(p);
  }
  void h2d_async(void* d, const void* s, size_t b) override { CK(cudaMemcpyAsync(d, s, b, cudaMemcpyHostToDevice, st)); }
  void h2d(void* d, const void* s, size_t b) override { CK(cudaMemcpyAsync(d, s, b, cudaMemcpyHostToDevice, st)); CK(cudaStreamSynchronize(st)); }
  void d2h(void* d, const void* s, size_t b) override { CK(cudaMemcpyAsync(d, s, b, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st)); }
  void d2d(void* d, const void* s, size_t b) override { CK(cudaMemcpyAsync(d, s, b, cudaMemcpyDeviceToDevice, st)); }
  // several graphs' scalars: one gather kernel into gather_buf, one copy back, one synchronise
  double* gather_buf = nullptr; size_t gather_cap = 0;
  void read_scalars(const double* const* src, int n, int len, double* out) override {
    if (n == 1) { d2h(out, src[0], sizeof(double) * (size_t)len); return; }
    const size_t total = (size_t)n * len;
    if (total > gather_cap) {
      if (gather_buf) free_(gather_buf);
      gather_cap = std::max(total, (size_t)1024);
      gather_buf = (double*)alloc(sizeof(double) * gather_cap);
    }
    for (int k0 = 0; k0 < n; k0 += GATHER_MAX) {
      GatherSrc g;
      g.n = std::min(GATHER_MAX, n - k0); g.len = len;
      for (int k = 0; k < g.n; ++k) g.src[k] = src[k0 + k];
      k_gather_scalars<<<1, 256, 0, st>>>(g, gather_buf + (size_t)k0 * len); ++n_launch;
    }
    d2h(out, gather_buf, sizeof(double) * total);
  }
  void zero(void* d, size_t b) override { CK(cudaMemsetAsync(d, 0, b, st)); }
  void sync() override { CK(cudaStreamSynchronize(st)); }
  int launches() const override { return n_launch; }
  void* stream() const override { return (void*)st; }
  void timer_start(int s) override { CK(cudaEventRecord(ev0[s], st)); }
  float timer_stop_ms(int s) override { float ms = 0; CK(cudaEventRecord(ev1[s], st)); CK(cudaEventSynchronize(ev1[s])); CK(cudaEventElapsedTime(&ms, ev0[s], ev1[s])); return ms; }

  static int nblk(int n, int b) { return n > 0 ? (n + b - 1) / b : 0; }
#define LAUNCH(kern, grid, block, ...)                         \
  do {                                                         \
    if ((grid) > 0) { kern<<<(grid), (block), 0, st>>>(__VA_ARGS__); ++n_launch; } \
  } while (0)

  // ---- launch shape of every step (BT_*) of the tiled and dense paths: one definition for a lone graph and for a batch's tables ----
  int band_per(const BaDev& d) const { return max(1, (d.n_tiles_stat + n_sm * 3 - 1) / (n_sm * 3)); }   // 3 CTAs per SM, each a run of consecutive tiles
  int grid(const BaDev& d, int t) const {
    const int ns = d.n_tiles_stat, nc = d.n_tiles - d.n_tiles_stat;
    switch (t) {
      case BT_TILE_LIN: case BT_BACKSUB: case BT_PRE_ST: case BT_RHS_ST: return ns;
      case BT_TILE_LIN_CH: case BT_BACKSUB_CH: case BT_PRE_CH: case BT_RHS_CH: case BT_S2_CH: return nc;
      case BT_FIN_LIN: case BT_VTRANS: case BT_PRE_FIN: case BT_VERT: return nblk(d.C, 128);
      case BT_SE3: case BT_DSE3: return nblk(d.Ese, 64);
      case BT_MAXDIAG: return min(nblk(d.C * 6 + d.P, 256), n_sm * 8);
      case BT_FACTOR: return nblk(d.T, 128);
      case BT_BAND_FORM: return d.band && ns > 0 ? nblk(ns, band_per(d)) : 0;
      case BT_UPDATE: return nblk(d.C + d.P, 128);
      case BT_DINIT: return nblk(36 * d.C * d.C, 128);
      case BT_FROM_BAND: return d.band ? nblk(d.band_n * d.band_W, 128) : 0;
      case BT_SCHUR2: return d.band ? ns : 0;                        // right-hand side of the dense path through the band ...
      case BT_FIN_SCHUR2: return d.band ? nblk(d.C, 128) : 0;
      case BT_DSCHUR: return d.band ? 0 : nblk(d.P, 128);            // ... or the per-landmark Schur kernel
      case BT_CHOL: case BT_PCG_FIN: return 1;
      case BT_PRE_BEGIN: return nblk(d.C * 36, 128);
      case BT_PCR_L: case BT_PCG_L: return d.n_own_long * PCR_CL;    // long paths (clusters of PCR_CL CTAs) first in own_paths,
      case BT_PCR_S: case BT_PCG_S: return d.n_own_paths - d.n_own_long;   // then the short ones (one CTA each)
      case BT_BAND_MUL: return d.band && ns > 0 ? nblk(d.band_n, 8) : 0;   // S*p of the static tiles: the band ...
      case BT_S2_ST: return d.band ? 0 : ns;                         // ... or the matrix-free tile kernel
      case BT_PHPP: return nblk(d.C, 16);                           // 8 lanes per vertex
      case BT_FIN_DOT: return nblk(d.C, 128);                        // 8 lanes per vertex, 128 vertices per partial of p.Ap
    }
    return 0;
  }
  static int threads(int t) {
    switch (t) {
      case BT_TILE_LIN: case BT_TILE_LIN_CH: case BT_BAND_FORM: case BT_BACKSUB: case BT_BACKSUB_CH: case BT_SCHUR2: case BT_PRE_ST: case BT_PRE_CH:
      case BT_RHS_ST: case BT_RHS_CH: case BT_S2_ST: case BT_S2_CH: return VDO_TILE_L;
      case BT_SE3: case BT_DSE3: return 64;
      case BT_MAXDIAG: case BT_CHOL: case BT_PCR_L: case BT_PCR_S: case BT_PCG_L: case BT_PCG_S: case BT_PCG_FIN: case BT_BAND_MUL: return 256;
      case BT_FIN_DOT: return 1024;
    }
    return 128;
  }
  // dynamic shared memory (a batch's launch takes the largest of its graphs)
  static size_t smem(const BaDev& d, int t) {
    switch (t) {
      case BT_TILE_LIN: return smem_lin(false, d.capE_st, d.capV_st, 0);
      case BT_TILE_LIN_CH: return smem_lin(true, d.capE_ch, d.capV_ch, d.capH_ch);
      case BT_PRE_ST: return smem_pre(false, d.capE_st);
      case BT_PRE_CH: return smem_pre(true, d.capE_ch);
      case BT_SCHUR2: case BT_RHS_ST: case BT_S2_ST: case BT_BACKSUB: return smem_sch2(false, d.capE_st, d.capV_st, 1);
      case BT_RHS_CH: case BT_S2_CH: case BT_BACKSUB_CH: return smem_sch2(true, d.capE_ch, d.capV_ch, d.capH_ch);
      case BT_BAND_FORM: return smem_band(d.capE_st);
      case BT_CHOL: { const size_t npad = (6 * (size_t)d.C + 7) & ~(size_t)7; return sizeof(double) * npad * (npad + 1); }
    }
    return 0;
  }
  // the kernels whose dynamic shared memory can pass 48 KB, sized for the largest tile and dense system
  template <class S> static void optin() {
    BaDev m;
    m.capE_st = m.capE_ch = VDO_TILE_E; m.capV_st = m.capV_ch = m.capH_ch = 255; m.C = DENSE_MAX / 6;
    auto set = [&](const void* f, int t) { if (smem(m, t) > 48 * 1024) CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem(m, t))); };
    set((const void*)k_tile_lin<S, false, true>, BT_TILE_LIN); set((const void*)k_tile_lin<S, false, false>, BT_TILE_LIN);
    set((const void*)k_tile_lin<S, true, true>, BT_TILE_LIN_CH); set((const void*)k_tile_lin<S, true, false>, BT_TILE_LIN_CH);
    set((const void*)k_tile_precond<S, false>, BT_PRE_ST); set((const void*)k_tile_precond<S, true>, BT_PRE_CH);
    set((const void*)k_tile_schur2<S, false, 0>, BT_RHS_ST); set((const void*)k_tile_schur2<S, false, 1>, BT_S2_ST);
    set((const void*)k_tile_schur2<S, true, 0>, BT_RHS_CH); set((const void*)k_tile_schur2<S, true, 1>, BT_S2_CH);
    set((const void*)k_tile_schur2<S, false, 2>, BT_BACKSUB); set((const void*)k_tile_schur2<S, true, 2>, BT_BACKSUB_CH);
    set((const void*)k_band_form<S>, BT_BAND_FORM);
    set((const void*)k_dense_chol<S>, BT_CHOL);
  }

  // ---- selectors: a lone graph, or the graphs of the launch tables whose flags hold `bit` ----
  One one(const BaDev& d, double lambda = 0.0, int reortho = 0, int parity = 0) const { return One{d, lambda, reortho, parity, band_per(d)}; }
  // the tables launch a step when one of their graphs takes part in the round (the PCG steps: when one of them is still iterating);
  // otherwise the selector is empty and launches nothing
  Many many(int bit) const {
    Many s{bdev, nullptr, bit, 0};
    bool live = false;
    for (int f : tflags) live |= (f & (bit == BATCH_PCG ? BATCH_PCG : ~0)) != 0;
    if (!live) s.B.n = 0;
    return s;
  }
  static void set_parity(One& s, int par) { s.par = par; }
  static void set_parity(Many& s, int par) { s.par = par; }
  int ctas(const One& s, int t) const { return grid(s.d, t); }
  int ctas(const Many& s, int t) const { return s.B.n ? bfirst[(size_t)t * (s.B.n + 1) + s.B.n] : 0; }
  size_t smem_of(const One& s, int t) const { return smem(s.d, t); }
  size_t smem_of(const Many&, int t) const { return bsmem[t]; }
  static One with_table(One s, int) { return s; }
  static Many with_table(Many s, int t) { s.f = s.B.first + (size_t)t * (s.B.n + 1); return s; }
  template <class F> void each(const One& s, F f) { f(s.d); }
  template <class F> void each(const Many& s, F f) { for (size_t i = 0; i < tab.size(); ++i) if (tflags[i] & s.bit) f(*bds_[tab[i]]); }
  // one launch of step t; a grid of 0 skips it
  template <class S, class... P, class... A> void run(void (*k)(S, P...), const S& s, int t, cudaStream_t stream, A... a) {
    const int n = ctas(s, t);
    if (n > 0) { k<<<n, threads(t), smem_of(s, t), stream>>>(with_table(s, t), a...); ++n_launch; }
  }

  // ---- the steps, written once for both selectors ----
  template <class S> void lin_tiles(const S& s, bool write, int part) {   // part: 0 static tiles, 1 chain tiles, -1 both
    if (part != 1) run(write ? k_tile_lin<S, false, true> : k_tile_lin<S, false, false>, s, BT_TILE_LIN, st);
    if (part != 0) run(write ? k_tile_lin<S, true, true> : k_tile_lin<S, true, false>, s, BT_TILE_LIN_CH, st);
  }
  template <class S> void max_diag(const S& s) {
    each(s, [&](const BaDev& d) { zero(d.scal + SC_MAXDIAG, sizeof(double)); });
    run(k_max_diagonal<S>, s, BT_MAXDIAG, st);
  }
  template <class S> void band_form_(const S& s) {
    each(s, [&](const BaDev& d) { if (d.band && d.n_tiles_stat > 0) zero(d.band, sizeof(double) * 10 * (size_t)d.band_n * d.band_W); });
    run(k_band_form<S>, s, BT_BAND_FORM, st);
  }
  // dense reduced system + tensor-core Cholesky (small static-only graphs)
  template <class S> void dense_solve_(const S& s) {
    run(k_dense_init<S>, s, BT_DINIT, st);
    run(k_dense_se3_edges<S>, s, BT_DSE3, st);
    // with a band: static Schur term from the band moments (one writer per block), right-hand side through the mode-0 tile kernel + finalize
    band_form_(s);
    run(k_dense_from_band<S>, s, BT_FROM_BAND, st);
    run(k_tile_schur2<S, false, 0>, s, BT_SCHUR2, st);
    run(k_tile_finalize_schur2<S, FIN_DENSE_RHS>, s, BT_FIN_SCHUR2, st);
    run(k_dense_schur<S>, s, BT_DSCHUR, st);
    run(k_dense_chol<S>, s, BT_CHOL, st);
    each(s, [&](const BaDev& d) { d2d(d.scal + SC_DENSE, d.Sdense + 36 * (size_t)d.C * d.C + 6 * (size_t)d.C, sizeof(double)); });
  }
  template <class S> void precond_tiles(const S& s) {
    run(k_tile_precond<S, false>, s, BT_PRE_ST, st);
    run(k_tile_precond<S, true>, s, BT_PRE_CH, st);
    run(k_tile_finalize_precond<S>, s, BT_PRE_FIN, st);
  }
  template <class S> void pcr_factor(const S& s) {
    run(k_pcr_factor<S, PCR_CL>, s, BT_PCR_L, st);
    run(k_pcr_factor<S, 1>, s, BT_PCR_S, st);
  }
  template <class S> void rhs_tiles(const S& s) {
    run(k_tile_schur2<S, false, 0>, s, BT_RHS_ST, st);
    run(k_tile_schur2<S, true, 0>, s, BT_RHS_CH, st);
  }
  // S*p on the landmark side: static tiles on st, chain tiles on chain_stream
  template <class S> void schur_product(const S& s, int part, cudaStream_t chain_stream) {
    if (part != 1) { run(k_band_mul<S>, s, BT_BAND_MUL, st); run(k_tile_schur2<S, false, 1>, s, BT_S2_ST, st); }
    if (part != 0) run(k_tile_schur2<S, true, 1>, s, BT_S2_CH, chain_stream);
  }
  template <class S> void backsub_tiles(const S& s) {
    run(k_tile_schur2<S, false, 2>, s, BT_BACKSUB, st);
    run(k_tile_schur2<S, true, 2>, s, BT_BACKSUB_CH, st);
  }
  // the long paths' clusters and the short paths' CTAs solve disjoint paths: the short ones run on st2 beside the clusters (the last CTA of
  // either launch to finish sums the partials of r.z, in path order)
  template <bool FUSED, class S> void step_a(const S& s) {
    bool fork = ctas(s, BT_PCG_L) > 0 && ctas(s, BT_PCG_S) > 0;
    if constexpr (std::is_same<S, One>::value) fork &= !s.d.xg_paths;   // the path-sharded exchange keeps its launch order
    if (fork) { CK(cudaEventRecord(ev_fork, st)); CK(cudaStreamWaitEvent(st2, ev_fork, 0)); }
    run(k_pcg_step_a<S, FUSED, PCR_CL>, s, BT_PCG_L, st);
    run(k_pcg_step_a<S, FUSED, 1>, s, BT_PCG_S, fork ? st2 : st);
    if (fork) { CK(cudaEventRecord(ev_join, st2)); CK(cudaStreamWaitEvent(st, ev_join, 0)); }
  }
  template <class S> void pcg_init_(const S& s) {
    each(s, [&](const BaDev& d) {
      zero(d.scal + SC_PAP, 6 * sizeof(double));   // PAP, RZ, RZ_NEW, RZ0, DONE, ITERS
      if (d.xg_paths) zero(d.xp, 48 * (size_t)d.C);   // path-sharded: a rank touches x on its own paths only; the rest must read 0 in the final sum
    });
    if constexpr (std::is_same<S, Many>::value) {
      if (s.B.n) { k_batch_scalars<<<nblk(s.B.n, 128), 128, 0, st>>>(s.B, s.bit); ++n_launch; }
      each(s, [&](const BaDev& d) { set_cache.erase(d.scal); });   // set_scalars must write these graphs' scalars again
    }
    run(k_pcg_init<S, PCR_CL>, s, BT_PCG_L, st);
    run(k_pcg_init<S, 1>, s, BT_PCG_S, st);
    run(k_pcg_init_fin<S>, s, BT_PCG_FIN, st);
  }
  // one fused PCG iteration (tiled layout): p update + H_pp product, static products forked with the chain tiles, finalize with the partials
  // of p.Ap, PCR step and scalars.  parity b & 1 of iteration b: p_k in d.p, p_{k+1} in d.p2 for even b.
  template <class S> void pcg_fused(S s, int b, bool peer) {
    set_parity(s, b & 1);
    run(k_pcg_p_hpp<S>, s, BT_PHPP, st);
    // fork: static products on st, chain tiles on st2 (independent landmark sets; both add into acc6 with atomics)
    CK(cudaEventRecord(ev_fork, st)); CK(cudaStreamWaitEvent(st2, ev_fork, 0));
    schur_product(s, -1, st2);
    CK(cudaEventRecord(ev_join, st2)); CK(cudaStreamWaitEvent(st, ev_join, 0));
    if constexpr (std::is_same<S, One>::value) {
      const BaDev& d = s.d;
      const double* p_out = (b & 1) ? d.p : d.p2;
      if (peer) {
        LAUNCH(k_xchg_scatter, nblk(d.C, 128), 128, d, -1.0, (const double*)d.Ap);      // partial S*p into slot[rank] of every rank
        LAUNCH(k_xchg_reduce, nblk(d.C, 128), 128, d, d.Ap, p_out);                     // sum of the slots in rank order, partials of p.Ap
      }
    }
    if (!peer) run(k_tile_finalize_ap_dot<S>, s, BT_FIN_DOT, st);                        // Ap -= B^T sums, and the partials of p.Ap
    step_a<true>(s);
    if constexpr (std::is_same<S, One>::value) { if (s.d.xg_paths) LAUNCH(k_pcg_scalars_x, 1, 256, s.d); }
  }
  // the launches of body() captured as one CUDA graph; *launches: how many kernels one replay runs
  template <class F> cudaGraphExec_t capture(F body, int* launches) {
    cudaGraph_t g = nullptr; cudaGraphExec_t ge = nullptr;
    const int before = n_launch;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    body();
    CK(cudaStreamEndCapture(st, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    cudaGraphDestroy(g);
    *launches = n_launch - before;
    n_launch = before;
    return ge;
  }

  // ---- lone graph ----
  void lin_tracklets(BaDev& d, bool write) override {
    if (d.tiled) { lin_tiles(one(d), write, -1); return; }
    if (write) { LAUNCH(k_lin_static<true>, nblk(d.Tstat, 256), 256, d); LAUNCH(k_lin_tracklets<true>, nblk(d.T - d.Tstat, 128), 128, d); }
    else { LAUNCH(k_lin_static<false>, nblk(d.Tstat, 256), 256, d); LAUNCH(k_lin_tracklets<false>, nblk(d.T - d.Tstat, 128), 128, d); }
  }
  // tiled layout: the tile kernels of lin_tracklets(write) have already formed the vertex-side sums in the world frame;
  // lin_vertex_obs turns them into H_pp / b_p, lin_vertex_ter has nothing left to do (same split for precond_* and schur_vertex_*)
  void lin_vertex_obs(BaDev& d) override {
    if (d.tiled) { run(k_tile_finalize_lin<One>, one(d), BT_FIN_LIN, st); return; }
    auto k = k_vertex_sym<0, true>; LAUNCH(k, d.n_obs_chunks, 128, d);
  }
  void lin_vertex_ter(BaDev& d) override { if (d.tiled) return; auto k = k_vertex_sym<0, false>; LAUNCH(k, d.n_ter_chunks, 128, d); }
  void lin_se3_edges(BaDev& d, bool write) override { run(write ? k_lin_se3_edges<One, true> : k_lin_se3_edges<One, false>, one(d), BT_SE3, st); }
  void max_diagonal(BaDev& d) override { max_diag(one(d)); }
  int band_max_width() const override { return 32; }
  void band_form(BaDev& d) override { band_form_(one(d)); }
  void factor_landmarks(BaDev& d, double lambda) override { run(k_factor_landmarks<One>, one(d, lambda), BT_FACTOR, st); }
  void precond_begin(BaDev& d, double lambda) override { run(k_precond_begin<One>, one(d, lambda), BT_PRE_BEGIN, st); }
  void precond_vertex_obs(BaDev& d) override {
    if (d.tiled) { precond_tiles(one(d)); return; }
    auto k = k_vertex_sym<1, true>; LAUNCH(k, d.n_obs_chunks, 128, d);
  }
  void precond_vertex_ter(BaDev& d) override { if (d.tiled) return; auto k = k_vertex_sym<1, false>; LAUNCH(k, d.n_ter_chunks, 128, d); }
  void precond_factor(BaDev& d, double lambda) override { pcr_factor(one(d, lambda)); }
  // block cyclic reduction: D, L and b updated in place, operators stored once per survivor and level (fewer than 2n slots per path)
  void precond_blocks(int C, int, size_t& nDL, size_t& nAG, size_t& nb) const override { nDL = (size_t)C; nAG = 2 * (size_t)C; nb = (size_t)C; }
  void schur_landmarks(BaDev& d, int mode, const double* v) override {
    if (d.tiled) {
      if (mode == 0) rhs_tiles(one(d)); else if (mode == 1) schur_product(one(d), -1, st); else backsub_tiles(one(d));
      return;
    }
    const int g = nblk((d.T - d.Tstat) * 8, 128), gs = nblk(d.Tstat, 256);
    if (mode == 0) { LAUNCH(k_schur_static<0>, gs, 256, d, d.zl); LAUNCH(k_schur_chains8<0>, g, 128, d, v, d.zl); }
    else if (mode == 1) { LAUNCH(k_schur_static<1>, gs, 256, d, d.zl); LAUNCH(k_schur_chains8<1>, g, 128, d, v, d.zl); }
    else { LAUNCH(k_schur_static<2>, gs, 256, d, d.xl); LAUNCH(k_schur_chains8<2>, g, 128, d, v, d.xl); }
  }
  void schur_landmarks_part(BaDev& d, int mode, const double* v, int part) override {
    if (d.tiled) { schur_product(one(d), part, st); return; }
    const int g = nblk((d.T - d.Tstat) * 8, 128), gs = nblk(d.Tstat, 256);
    if (part == 0) LAUNCH(k_schur_static<1>, gs, 256, d, d.zl); else LAUNCH(k_schur_chains8<1>, g, 128, d, v, d.zl);
    (void)mode;
  }
  void lin_tracklets_part(BaDev& d, bool write, int part) override {
    if (d.tiled) { lin_tiles(one(d), true, part); return; }
    (void)write;
    if (part == 0) LAUNCH(k_lin_static<true>, nblk(d.Tstat, 256), 256, d); else LAUNCH(k_lin_tracklets<true>, nblk(d.T - d.Tstat, 128), 128, d);
  }
  // tiled layout: the solver's two outputs of the vertex pass, d.rhs or d.Ap, both with sign -1
  void schur_vertex_obs(BaDev& d, double sign, double* out) override {
    if (d.tiled) { run(out == d.Ap ? k_tile_finalize_schur2<One, FIN_AP> : k_tile_finalize_schur2<One, FIN_RHS>, one(d), BT_VERT, st); return; }
    LAUNCH(k_schur_vertex<true>, d.n_obs_chunks, 128, d, sign, out, out == d.Ap ? 1 : 0);
  }
  void schur_vertex_ter(BaDev& d, double sign, double* out) override {
    if (d.tiled) return;
    LAUNCH(k_schur_vertex<false>, d.n_ter_chunks, 128, d, sign, out, out == d.Ap ? 1 : 0);
  }
  // lambda and tol2 of a lone graph's PCG kernels, as last written to its device scalars (per graph: the per-graph forms of a batch call
  // interleave the chunks of several graphs); -1 until written
  std::map<const double*, std::pair<double, double>> set_cache;
  std::pair<double, double>& cached(const BaDev& d) { return set_cache.try_emplace(d.scal, -1.0, -1.0).first->second; }
  void set_scalars(BaDev& d, double lambda, double tol2) {
    std::pair<double, double>& c = cached(d);
    if (lambda != c.first || tol2 != c.second) { LAUNCH(k_set_scalars, 1, 1, d, lambda, tol2); c = {lambda, tol2}; }
  }
  void vertex_transform(BaDev& d, const double* v) override { run(k_vertex_transform<One>, one(d), BT_VTRANS, st, v); }
  void hpp_mul(BaDev& d, double lambda, const double* x, double* out) override { const double t2 = cached(d).second; set_scalars(d, lambda, t2 < 0 ? 0.0 : t2); LAUNCH(k_hpp_mul, nblk(d.C, 128), 128, d, x, out); }
  void pcg_init(BaDev& d) override { pcg_init_(one(d)); }
  void pcg_dot_pAp(BaDev& d) override { LAUNCH(k_pcg_dot, d.n_part_pap, 256, d); }   // one CTA per slot of part_pap
  void pcg_step(BaDev& d, double tol2) override {
    set_scalars(d, cached(d).first, tol2);
    step_a<false>(one(d, 0.0, 0, 1));
    LAUNCH(k_pcg_step_b, min(nblk(d.C * 6, 256), n_sm), 256, d);
    LAUNCH(k_pcg_scalars, 1, 256, d);
  }
  // n PCG iterations as ONE CUDA-graph launch (captured once per factor graph and batch size; lambda / tolerance travel
  // through device scalars so the captured kernel arguments never change)
  std::map<std::pair<const void*, int>, cudaGraphExec_t> graphs;
  void pcg_iterate(BaDev& d, double lambda, double tol2, int n) override {
    // sharded: the same captured graph with the all-reduce of S*p done by two kernels over peer memory (k_xchg_scatter / k_xchg_reduce);
    // without peer mapping (or with the chunked layout) plain launches + one NCCL all-reduce per iteration
    bool peer = false;
    if (world > 1) {
      peer = d.tiled && d.xg_paths && xg.ok;            // decided (collectively) at finalize: shard_paths
      if (!peer) { BaBackend::pcg_iterate(d, lambda, tol2, n); return; }
    }
    set_scalars(d, lambda, tol2);
    auto key = std::make_pair((const void*)d.scal, n);
    auto it = graphs.find(key);
    if (it == graphs.end()) {
      cudaGraphExec_t ge = capture([&] {
        const int gch = nblk((d.T - d.Tstat) * 8, 128), gst = nblk(d.Tstat, 256);
        for (int b = 0; b < n; ++b) {
          if (d.tiled) { pcg_fused(one(d), b, peer); continue; }   // n is even: the search direction ends in d.p again
          LAUNCH(k_hpp_mul, nblk(d.C, 128), 128, d, (const double*)d.p, d.Ap);
          // fork: static landmarks on st, chains on st2 (independent landmark sets; the chain kernel is latency-bound)
          CK(cudaEventRecord(ev_fork, st)); CK(cudaStreamWaitEvent(st2, ev_fork, 0));
          LAUNCH(k_schur_static<1>, gst, 256, d, d.zl);
          if (gch > 0) { k_schur_chains8<1><<<gch, 128, 0, st2>>>(d, (const double*)d.p, d.zl); ++n_launch; }
          CK(cudaEventRecord(ev_join, st2)); CK(cudaStreamWaitEvent(st, ev_join, 0));
          // fork: the two vertex-major passes add into Ap with atomics and are independent of each other
          CK(cudaEventRecord(ev_fork, st)); CK(cudaStreamWaitEvent(st2, ev_fork, 0));
          schur_vertex_obs(d, -1.0, d.Ap);
          if (d.n_ter_chunks > 0) { k_schur_vertex<false><<<d.n_ter_chunks, 128, 0, st2>>>(d, -1.0, d.Ap, 1); ++n_launch; }
          CK(cudaEventRecord(ev_join, st2)); CK(cudaStreamWaitEvent(st, ev_join, 0));
          LAUNCH(k_pcg_dot, d.n_part_pap, 256, d);
          step_a<false>(one(d, 0.0, 0, 1));
          LAUNCH(k_pcg_step_b, min(nblk(d.C * 6, 256), n_sm), 256, d);
          LAUNCH(k_pcg_scalars, 1, 256, d);
        }
      }, &per_batch[key]);
      it = graphs.emplace(key, ge).first;
    }
    CK(cudaGraphLaunch(it->second, st));
    n_launch += per_batch[key];
  }
  std::map<std::pair<const void*, int>, int> per_batch;
  // sharded graphs with the tiled layout: map the exchange buffer, move z / part_rz into it and shard the preconditioner by path
  bool shard_paths(BaDev& d) override {
    if (world <= 1 || !d.tiled || d.n_paths < world) return false;      // (every rank must own at least one path: it raises a flag per solve)
    if (!xchg_setup(d.C, d.n_paths)) return false;
    d.xg_rank = rank; d.xg_world = world; d.xg_slots = xg.d_slots; d.xg_flags = xg.d_flags; d.xg_epoch = xg.d_epoch;
    d.xg_paths = 1; d.xg_off_z = xg.off_z; d.xg_off_prz = xg.off_prz;
    d.z = (double*)(xg.local + XG_HDR) + xg.off_z;
    d.part_rz = (double*)(xg.local + XG_HDR) + xg.off_prz;
    return true;
  }
  void drop_graphs() {
    for (auto& kv : graphs) cudaGraphExecDestroy(kv.second);
    graphs.clear(); per_batch.clear();
  }
  void release(BaDev& d) override {
    for (auto it = graphs.begin(); it != graphs.end();) {
      if (it->first.first == (const void*)d.scal) { cudaGraphExecDestroy(it->second); per_batch.erase(it->first); it = graphs.erase(it); } else ++it;
    }
    set_cache.erase(d.scal);
  }
  int dense_capacity() const override { return DENSE_MAX; }
  void dense_solve(BaDev& d, double lambda) override { dense_solve_(one(d, lambda)); }
  void apply_update(BaDev& d, double lambda, bool reortho) override { run(k_apply_update<One>, one(d, lambda, reortho ? 1 : 0), BT_UPDATE, st); }

  // ---- batch: the dense-path graphs of a call, when there are two or more, and likewise its PCG-path graphs of the tiled layout on one
  //      GPU, take each step as one launch per kernel through launch tables built once per call.  Every other graph runs the per-graph
  //      forms of the base class, which are its lone launches. ----
  BatchDev bdev{};
  std::vector<int> tab;                    // the graphs in the tables (positions in the call), in table order
  std::vector<int> tflags;                 // ... their step flags (the base class sees 0 for them)
  std::vector<int> wflags, wrt; std::vector<double> wlam, wtol2;   // ... their flags and parameters as last written to the device
  std::vector<int> bfirst;                 // BT_N x (n + 1): first CTA of every graph in each launch table
  size_t bsmem[BT_N] = {};                 // dynamic shared memory of each table's launch
  void* bbuf = nullptr;
  static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }
  cudaGraphExec_t bpcg = nullptr; int bpcg_n = 0, bpcg_launches = 0;   // the captured PCG chunk of the call (pcg_iterate_batch)
  void batch_begin(BaDev* const* all, int n_all) override {
    BaBackend::batch_begin(all, n_all);
    tab.clear();
    for (int pass = 0; pass < 2; ++pass) {
      std::vector<int> ks;
      for (int k = 0; k < n_all; ++k) {
        const BaDev& d = *all[k];
        if (pass == 0 ? d.Sdense != nullptr : (!d.Sdense && d.tiled && !d.xg_paths && world == 1)) ks.push_back(k);
      }
      if (ks.size() >= 2) tab.insert(tab.end(), ks.begin(), ks.end());
    }
    const int n = (int)tab.size();
    tflags.assign(n, 0); wflags.assign(n, 0); wrt.assign(n, 0); wlam.assign(n, 0.0); wtol2.assign(n, 0.0);
    if (!n) return;
    bfirst.assign((size_t)BT_N * (n + 1), 0);
    std::vector<int> per(n, 1);
    for (int t = 0; t < BT_N; ++t) bsmem[t] = 0;
    for (int k = 0; k < n; ++k) {
      const BaDev& d = *all[tab[k]];
      const bool dn = d.Sdense != nullptr;
      per[k] = band_per(d);
      for (int t = 0; t < BT_N; ++t) {
        const int g = (t >= BT_PRE_BEGIN ? dn : (t >= BT_DINIT && !dn)) ? 0 : grid(d, t);
        bfirst[(size_t)t * (n + 1) + k + 1] = bfirst[(size_t)t * (n + 1) + k] + g;
        if (g > 0) bsmem[t] = std::max(bsmem[t], smem(d, t));
      }
    }
    const size_t o_first = align16(sizeof(BaDev) * (size_t)n), o_per = o_first + align16(sizeof(int) * bfirst.size()), o_flags = o_per + align16(sizeof(int) * n),
                 o_rt = o_flags + align16(sizeof(int) * n), o_lam = o_rt + align16(sizeof(int) * n), o_tol = o_lam + align16(sizeof(double) * (size_t)n),
                 total = o_tol + sizeof(double) * (size_t)n;
    std::vector<char> h(o_flags, 0);
    for (int k = 0; k < n; ++k) std::memcpy(h.data() + sizeof(BaDev) * (size_t)k, all[tab[k]], sizeof(BaDev));
    std::memcpy(h.data() + o_first, bfirst.data(), sizeof(int) * bfirst.size());
    std::memcpy(h.data() + o_per, per.data(), sizeof(int) * n);
    bbuf = alloc(total);
    h2d(bbuf, h.data(), h.size());
    char* b = (char*)bbuf;
    bdev = BatchDev{(const BaDev*)b, (const int*)(b + o_first), (const int*)(b + o_per), (int*)(b + o_flags), (double*)(b + o_lam), (int*)(b + o_rt), (double*)(b + o_tol), n};
  }
  void batch_end() override {
    if (bpcg) { CK(cudaGraphExecDestroy(bpcg)); bpcg = nullptr; }
    if (bbuf) free_(bbuf);
    bbuf = nullptr; bdev = BatchDev{}; tab.clear(); tflags.clear();
    BaBackend::batch_end();
  }
  void batch_set(const int* flags, const double* lambda, const int* reortho, const double* tol2) override {
    BaBackend::batch_set(flags, lambda, reortho, tol2);
    const int n = (int)tab.size();
    bool on = false, pcg = false;
    for (int i = 0; i < n; ++i) { tflags[i] = bflags_[tab[i]]; bflags_[tab[i]] = 0; on |= tflags[i] != 0; pcg |= (tflags[i] & BATCH_PCG) != 0; }
    // the device copy is rewritten when a graph of the tables takes part in the round and its flags or parameters changed.  A graph that
    // leaves the PCG after the tables' last PCG graph needs no write: the steps up to the next round test BATCH_TRIAL only.
    const int mask = pcg ? ~0 : ~BATCH_PCG;
    bool stale = false;
    for (int i = 0; i < n; ++i) {
      const int k = tab[i];
      stale |= ((tflags[i] ^ wflags[i]) & mask) != 0 || lambda[k] != wlam[i] || reortho[k] != wrt[i] || tol2[k] != wtol2[i];
    }
    if (!on || !stale) return;
    for (int k0 = 0; k0 < n; k0 += BATCH_PARAMS_MAX) {
      BatchParams p;
      p.n0 = k0; p.n = std::min(BATCH_PARAMS_MAX, n - k0);
      for (int i = 0; i < p.n; ++i) {
        const int j = k0 + i, k = tab[j];
        p.flags[i] = wflags[j] = tflags[j]; p.lambda[i] = wlam[j] = lambda[k]; p.reortho[i] = wrt[j] = reortho[k]; p.tol2[i] = wtol2[j] = tol2[k];
      }
      k_batch_params<<<1, BATCH_PARAMS_MAX, 0, st>>>(bdev, p); ++n_launch;
    }
  }
  // each step: the tables' graphs in one launch per kernel, then the other graphs through the base class
  void lin_tracklets_batch(int bit, bool write) override { lin_tiles(many(bit), write, -1); BaBackend::lin_tracklets_batch(bit, write); }
  void lin_vertex_batch(int bit) override { run(k_tile_finalize_lin<Many>, many(bit), BT_FIN_LIN, st); BaBackend::lin_vertex_batch(bit); }
  void lin_se3_edges_batch(int bit, bool write) override {
    run(write ? k_lin_se3_edges<Many, true> : k_lin_se3_edges<Many, false>, many(bit), BT_SE3, st);
    BaBackend::lin_se3_edges_batch(bit, write);
  }
  void max_diagonal_batch(int bit) override { max_diag(many(bit)); BaBackend::max_diagonal_batch(bit); }
  void factor_landmarks_batch(int bit) override { run(k_factor_landmarks<Many>, many(bit), BT_FACTOR, st); BaBackend::factor_landmarks_batch(bit); }
  void dense_solve_batch(int bit) override { dense_solve_(many(bit)); BaBackend::dense_solve_batch(bit); }
  void back_substitute_batch(int bit) override {
    run(k_vertex_transform<Many>, many(bit), BT_VTRANS, st, (const double*)nullptr);
    backsub_tiles(many(bit));
    BaBackend::back_substitute_batch(bit);
  }
  void apply_update_batch(int bit) override { run(k_apply_update<Many>, many(bit), BT_UPDATE, st); BaBackend::apply_update_batch(bit); }
  void precondition_batch(int bit) override {
    const Many s = many(bit);
    each(s, [&](const BaDev& d) { zero(d.scal + SC_BAD, sizeof(double)); });
    run(k_precond_begin<Many>, s, BT_PRE_BEGIN, st);
    precond_tiles(s);
    pcr_factor(s);
    band_form_(s);
    BaBackend::precondition_batch(bit);
  }
  void schur_rhs_batch(int bit) override {
    const Many s = many(bit);
    rhs_tiles(s);
    each(s, [&](const BaDev& d) { d2d(d.rhs, d.bp, 48 * (size_t)d.C); });
    run(k_tile_finalize_schur2<Many, FIN_RHS>, s, BT_VERT, st);
    BaBackend::schur_rhs_batch(bit);
  }
  void pcg_init_batch(int bit) override { pcg_init_(many(bit)); BaBackend::pcg_init_batch(bit); }
  // the tables' n fused iterations, captured as one CUDA graph per call: the tables and buffers do not change until batch_end, and the
  // flags, lambda and tolerance are read on the device
  void pcg_iterate_batch(int bit, int n) override {
    if (many(bit).B.n) {
      if (bpcg && bpcg_n != n) { CK(cudaGraphExecDestroy(bpcg)); bpcg = nullptr; }
      if (!bpcg) {
        bpcg = capture([&] { for (int b = 0; b < n; ++b) pcg_fused(many(bit), b, false); }, &bpcg_launches);
        bpcg_n = n;
      }
      CK(cudaGraphLaunch(bpcg, st));
      n_launch += bpcg_launches;
    }
    BaBackend::pcg_iterate_batch(bit, n);
  }
};

BaBackend* make_backend(int device, char* err, size_t errlen) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) { std::snprintf(err, errlen, "no CUDA device (%s); libvdo_b200 has no CPU path", cudaGetErrorString(e)); return nullptr; }
  if (device < 0 || device >= n) { std::snprintf(err, errlen, "device %d out of range (%d visible)", device, n); return nullptr; }
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) { std::snprintf(err, errlen, "cudaGetDeviceProperties: %s", cudaGetErrorString(e)); return nullptr; }
  if (prop.major != 9 || prop.minor != 0) { std::snprintf(err, errlen, "device %d is sm_%d%d; this build carries sm_90a code only", device, prop.major, prop.minor); return nullptr; }
  if ((e = cudaSetDevice(device)) != cudaSuccess) { std::snprintf(err, errlen, "cudaSetDevice: %s", cudaGetErrorString(e)); return nullptr; }
  CudaBackend::optin<One>();
  CudaBackend::optin<Many>();
  CudaBackend* b = new CudaBackend;
  b->dev = device;
  b->n_sm = prop.multiProcessorCount;
  if ((e = cudaStreamCreateWithFlags(&b->st, cudaStreamNonBlocking)) != cudaSuccess) { std::snprintf(err, errlen, "cudaStreamCreate: %s", cudaGetErrorString(e)); delete b; return nullptr; }
  for (int i = 0; i < 4; ++i) { cudaEventCreate(&b->ev0[i]); cudaEventCreate(&b->ev1[i]); }
  cudaStreamCreateWithFlags(&b->st2, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&b->ev_fork, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&b->ev_join, cudaEventDisableTiming);
  return b;
}

}  // namespace vdo

// ---- multi-GPU bootstrap (C ABI, declared in include/vdo_b200.h) ----
struct vdo_ctx;
namespace vdo {
BaBackend* ctx_backend(vdo_ctx* c);
// device ordinal and SM count of a context (orb_match.cu)
void ctx_device(vdo_ctx* c, int* dev, int* n_sm) {
  const CudaBackend* be = static_cast<const CudaBackend*>(ctx_backend(c));
  *dev = be->dev; *n_sm = be->n_sm;
}
}  // namespace vdo
extern "C" int vdo_nccl_unique_id(char* out128) {
  if (!out128) return -2;
  if (!vdo::g_nccl.load()) return -5;
  ncclUniqueId id;
  if (vdo::g_nccl.GetUniqueId(&id) != ncclSuccess) return -5;
  std::memcpy(out128, &id, sizeof id);
  return 0;
}
extern "C" int vdo_ctx_init_comm(vdo_ctx* ctx, int rank, int world, const char* id128) {
  vdo::CudaBackend* be = static_cast<vdo::CudaBackend*>(vdo::ctx_backend(ctx));
  if (!be || !id128 || world < 1 || rank < 0 || rank >= world) return -2;
  if (world == 1) { be->rank = 0; be->world = 1; return 0; }
  if (!vdo::g_nccl.load()) return -5;
  ncclUniqueId id;
  std::memcpy(&id, id128, sizeof id);
  cudaSetDevice(be->dev);
  ncclResult_t r = vdo::g_nccl.CommInitRank(&be->comm, world, id, rank);
  if (r != ncclSuccess) { std::fprintf(stderr, "[vdo_b200] ncclCommInitRank failed: %s\n", vdo::g_nccl.GetErrorString ? vdo::g_nccl.GetErrorString(r) : "?"); return -5; }
  be->rank = rank; be->world = world;
  return 0;
}
