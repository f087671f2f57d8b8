// ba_tile_kernels.cuh -- sm_90a kernels of the tiled batch-LM layout (included by ba_kernels.cu; bodies in ba_tiles.cuh).
//
// One CTA (VDO_TILE_L = 256 threads) per tile.  Every contiguous range of a global array the tile needs (landmark block,
// pivots, edge weights / cameras / tile-local landmark ids, the vertex-sorted permutation, the segment descriptors, Q_k) is
// brought into shared memory by ONE elected thread with 1-D bulk async copies (cp.async.bulk.shared::cluster.global, the
// TMA engine) completing on an mbarrier, so that all of the tile's HBM traffic is in flight at once and the phases below
// run out of shared memory; only the per-vertex gathers (poses / world-frame vectors, L2-resident) and the edge
// measurements of the linearisation are ordinary loads.  Phases:
//   k_tile_lin     per edge: residual, Huber weight (written once to HBM), e_w stash -> per landmark: H_ll / b_l ->
//                  per (run, part) of the vertex-sorted runs: 4 of the 16 world-frame sums, one atomic per (vertex, sum) -> chains: Q_k
//   k_tile_precond per (run, half): 10 sums of the diagonal blocks of Hpl Hll^-1 Hlp
//   k_tile_schur2  per landmark: bl (mode 0), Hlp v (mode 1) or bl - Hlp v (mode 2) -> Hll^-1 (chains: scalar tridiagonal in the
//                  Q-rotated frame, CTA-wide scans) -> modes 0 / 1: per (run, component): Hpl z, one atomic each; mode 2: xl.
// Bytes per launch (algorithmic, every array touched once): see bench.py kernel_bytes and DESIGN.md section 5.
#pragma once
#include "ba_tiles.cuh"

namespace vdo {

constexpr int TILE_OSEG2_CAP_ST = 192, TILE_OSEG2_CAP_CH = 96, TILE_TSEG2_CAP = 96;   // runs of VDO_SEG2 entries (osegs2 / tsegs2) staged per tile

// ---- mbarrier + 1-D bulk copy (PTX ISA: mbarrier.*, cp.async.bulk) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, 0x989680;\n"   /* suspend-time hint: waiters sleep instead of spinning */
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}

// Carves the CTA's dynamic shared memory.  view(): a staged copy of g[first, first + count) -- the copy starts at the
// enclosing 16-byte boundary and is rounded up to 16 bytes (bulk copies need both; every device array is allocated with 16
// spare bytes at its end), the returned pointer addresses element `first`.  Only the elected thread issues copies.
struct TileStager {
  char* cur; uint64_t* bar; bool issue; uint32_t tx = 0;
  __device__ TileStager(void* base, uint64_t* b, bool is) : cur((char*)base), bar(b), issue(is) {}
  template <typename T> __device__ __forceinline__ T* view(const T* g, size_t first, int count, int cap) {
    const uintptr_t a = (uintptr_t)(g + first);
    const uint32_t delta = (uint32_t)(a & 15), bytes = (delta + (uint32_t)count * (uint32_t)sizeof(T) + 15u) & ~15u;
    char* dst = cur;
    cur += view_bytes<T>(cap);
    if (issue && count > 0) { bulk_g2s(dst, (const void*)(a - delta), bytes, bar); tx += bytes; }
    return (T*)(dst + delta);
  }
  template <typename T> __device__ __forceinline__ T* stash(int cap) { T* p = (T*)cur; cur += (cap * sizeof(T) + 15) & ~(size_t)15; return p; }
  template <typename T> __host__ __device__ static constexpr size_t view_bytes(int cap) { return ((cap * sizeof(T) + 15) & ~(size_t)15) + 16; }
  __device__ __forceinline__ void commit() { if (issue) mbar_arrive_expect_tx(bar, tx); }
};
template <typename T> constexpr size_t vb(int cap) { return TileStager::view_bytes<T>(cap); }
constexpr size_t sb(size_t n) { return (n + 15) & ~(size_t)15; }

// Linearisation.  Phases: per edge (static tiles) or per landmark (chain tiles: its pointxyz edges, then its ternary edge): residual,
// Huber weight (written once to HBM), e_w stash -> per landmark: H_ll / b_l -> vertex side -> (chains) Q_k.
//  * the poses (R, t) of the tile's cameras and motion vertices are gathered into shared memory by warps 1..7 while warp 0 stages the
//    tile; edges address them by their 8-bit slot (lm_cslot / tk_hslot) instead of gathering 96 bytes each from global memory.
//  * the vertex side is one thread per (run, part) of the vertex-sorted runs of <= VDO_SEG2 entries (osegs2 / tsegs2): a thread adds
//    its four of the 16 world-frame sums (acc16_add_part) over its run from shared memory into a shared partial; then one thread per
//    (vertex, part) adds the partials of the vertex' runs in run order and issues one fp64 atomic per sum.  Passes of <= 64 runs end
//    at a vertex boundary (a vertex has at most 52 runs in a tile), so a tile adds to each of its vertices once: the sums do not depend
//    on the order the atomics land in whenever a vertex meets at most two tiles (two terms added to zero commute exactly), as in the
//    small windowed graphs of the tracker, whose results must not depend on whether its graphs are solved alone or in a batch.
//  * chains: one thread per tracklet walks Q_{k+1} = Q_k R_k^T out of the shared pose copy into shared memory; the CTA then writes
//    pt_Q with coalesced stores.
//  * per-edge and per-vertex arrays are sized by the launch's capacities (capE / capV / capH: largest tile of the launch).
inline size_t smem_lin(bool chains, int capE, int capV, int capH) {   // must mirror the carve order inside k_tile_lin_body
  size_t stash = sb((size_t)capE * 8) + sb(3 * (size_t)capE * 8);
  if (chains) {
    stash += sb(VDO_TILE_L * 8) + sb(4 * VDO_TILE_L * 8) + sb(3 * VDO_TILE_L * 8);
    if (stash < sb(9 * VDO_TILE_L * 8)) stash = sb(9 * VDO_TILE_L * 8);     // Q_k reuses the stashes once the vertex side is done
  }
  size_t b = sb(12 * (size_t)(capV + (chains ? capH : 0)) * 8) + sb(4 * VDO_TILE_L * 8) + vb<double>(3 * VDO_TILE_L) + vb<int>(VDO_TILE_L + 1) + vb<uint8_t>(capE) +
             vb<uint32_t>(capE) + vb<Seg>(chains ? TILE_OSEG2_CAP_CH : TILE_OSEG2_CAP_ST);
  if (!chains) b += vb<uint8_t>(capE);
  else b += vb<int>(VDO_TILE_L + 1) + vb<uint8_t>(VDO_TILE_L) + vb<uint8_t>(VDO_TILE_L) + vb<uint16_t>(VDO_TILE_L) + vb<Seg>(TILE_TSEG2_CAP);
  return b + stash;
}

// Vertex side over the runs seg[0, n) of a tile: run(s, PART, a) adds run s's four sums of part PART to a.  Passes of <= VDO_TILE_L / 4
// runs ending at a vertex boundary; sPart: 4 * VDO_TILE_L doubles of shared memory; dst(v): the vertex' 16 accumulators.
template <typename R, typename D>
__device__ __forceinline__ void lin_vertex_side(const Seg* seg, int n, double* sPart, int tid, R run, D dst) {
  constexpr int RUNS = VDO_TILE_L / 4;
  const int part = tid & 3;
  for (int r0 = 0; r0 < n;) {
    int r1 = min(r0 + RUNS, n);
    while (r1 < n && seg[r1].v == seg[r1 - 1].v) --r1;
    const int s = r0 + (tid >> 2);
    double a[4] = {0, 0, 0, 0};
    if (s < r1) {
      switch (part) {
        case 0: run(s, std::integral_constant<int, 0>(), a); break;
        case 1: run(s, std::integral_constant<int, 1>(), a); break;
        case 2: run(s, std::integral_constant<int, 2>(), a); break;
        default: run(s, std::integral_constant<int, 3>(), a); break;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) sPart[4 * tid + i] = a[i];
    }
    __syncthreads();
    if (s < r1 && (s == r0 || seg[s - 1].v != seg[s].v)) {
      const int v = seg[s].v;
      for (int e = s + 1; e < r1 && seg[e].v == v; ++e) {
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] += sPart[4 * (4 * (e - r0) + part) + i];
      }
      double* o = dst(v) + 4 * part;
#pragma unroll
      for (int i = 0; i < 4; ++i) if (a[i] != 0.0) atomicAdd(o + i, a[i]);
    }
    __syncthreads();
    r0 = r1;
  }
}

template <bool CHAINS, bool WRITE>
__device__ __forceinline__ void k_tile_lin_body(const BaDev& d, int tile0, int capE, int capV, int capH, int bx) {
  extern __shared__ __align__(16) unsigned char tile_sh[];
  __shared__ double red[32];
  __shared__ __align__(8) uint64_t bar;
  __shared__ uint32_t tab[12];                              // shared-memory offsets of the staged views (computed by warp 0 only)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Tile tl = d.tiles[tile0 + bx];
  const int nl = tl.k1 - tl.k0, ne = tl.e1 - tl.e0, ncam = tl.nv & 0xFFFF, nmot = tl.nv >> 16;
  const int n_os = WRITE ? tl.qo1 - tl.qo0 : 0, n_ts = (CHAINS && WRITE) ? tl.qt1 - tl.qt0 : 0;
  constexpr int OCAP = CHAINS ? TILE_OSEG2_CAP_CH : TILE_OSEG2_CAP_ST;
  double* sT = (double*)tile_sh;                            // 12 per slot: the tile's cameras, then its motion vertices; then the
                                                            // vertex side's partial sums (4 per thread)
  if (warp == 0) {
    if (lane == 0) mbar_init(&bar, 1);
    __syncwarp();
    TileStager sg(tile_sh + sb(12 * (size_t)(capV + (CHAINS ? capH : 0)) * 8) + sb(4 * VDO_TILE_L * 8), &bar, lane == 0);
    auto off = [&](const void* ptr) { return (uint32_t)((const unsigned char*)ptr - tile_sh); };
    uint32_t o[12];
    o[0] = off(sg.view<double>(d.pt, 3 * (size_t)tl.k0, 3 * nl, 3 * VDO_TILE_L));
    o[1] = off(sg.view<int>(d.lm_obs_begin, (size_t)tl.k0, (CHAINS || WRITE) ? nl + 1 : 0, VDO_TILE_L + 1));
    o[2] = off(sg.view<uint8_t>(d.lm_cslot, (size_t)tl.e0, ne, capE));
    o[3] = off(sg.view<uint32_t>(d.ob_ps, (size_t)tl.e0, WRITE ? ne : 0, capE));
    o[4] = off(sg.view<Seg>(d.osegs2, (size_t)tl.qo0, n_os <= OCAP ? n_os : 0, OCAP));
    if (!CHAINS) {
      o[5] = off(sg.view<uint8_t>(d.lm_lml, (size_t)tl.e0, ne, capE));
    } else {
      o[6] = off(sg.view<int>(d.tk_begin, (size_t)tl.t0, WRITE ? tl.t1 - tl.t0 + 1 : 0, VDO_TILE_L + 1));
      o[7] = off(sg.view<uint8_t>(d.tk_hslot, (size_t)tl.k0, nl, VDO_TILE_L));
      o[8] = off(sg.view<uint8_t>(d.tk_cls, (size_t)tl.k0, nl, VDO_TILE_L));
      o[9] = off(sg.view<uint16_t>(d.tr_perm, (size_t)tl.k0, WRITE ? nl : 0, VDO_TILE_L));
      o[10] = off(sg.view<Seg>(d.tsegs2, (size_t)tl.qt0, n_ts <= TILE_TSEG2_CAP ? n_ts : 0, TILE_TSEG2_CAP));
    }
    o[11] = off(sg.stash<double>(1));                       // the stashes start here (sizes: smem_lin)
    sg.commit();
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < 12; ++i) tab[i] = o[i];
    }
    mbar_wait(&bar, 0);
  } else {
    for (int i = tid - 32; i < 12 * (ncam + nmot); i += VDO_TILE_L - 32) { const int s = i / 12; sT[i] = d.se3[12 * (size_t)d.tile_verts[tl.vs0 + s] + (i - 12 * s)]; }
  }
  __syncthreads();
  TileSm sm;
  sm.P = (double*)(tile_sh + tab[0]);
  sm.LB = (int*)(tile_sh + tab[1]);
  const uint8_t* sCS = (const uint8_t*)(tile_sh + tab[2]);
  const uint32_t* sPS = (const uint32_t*)(tile_sh + tab[3]);
  const Seg* oseg = n_os <= OCAP ? (const Seg*)(tile_sh + tab[4]) : d.osegs2 + tl.qo0;
  double* stash = (double*)(tile_sh + tab[11]);
  sm.OM = stash; sm.EW = stash + capE;
  const uint8_t* sHS = nullptr; const int* sTB = nullptr; const uint16_t* sTPERM = nullptr; const Seg* tseg = nullptr;
  if (!CHAINS) {
    sm.LML = (uint8_t*)(tile_sh + tab[5]);
  } else {
    sTB = (const int*)(tile_sh + tab[6]); sHS = (const uint8_t*)(tile_sh + tab[7]); sm.TCLS = (uint8_t*)(tile_sh + tab[8]);
    sTPERM = (const uint16_t*)(tile_sh + tab[9]);
    tseg = n_ts <= TILE_TSEG2_CAP ? (const Seg*)(tile_sh + tab[10]) : d.tsegs2 + tl.qt0;
    sm.OMT = stash + 4 * capE; sm.TC = sm.OMT + VDO_TILE_L; sm.E2 = sm.TC + 4 * VDO_TILE_L;
  }
  const double* sH = sT + 12 * ncam;                        // motion vertices
  double chi = 0.0;
  if (!CHAINS) {
    for (int i = tid; i < ne; i += VDO_TILE_L) chi += tile_lin_edge_at<WRITE>(d, tl, i, sm.LML[i], sT + 12 * sCS[i], sm);
    if (WRITE) {
      __syncthreads();
      if (tid < nl) {
        double dsum = 0.0, b[3] = {0, 0, 0};
        tile_lin_landmark_obs(d, tl, tid, sm, dsum, b);
        const size_t k = (size_t)tl.k0 + tid;
        d.tk_omega[k] = 0.0; d.hll[k] = dsum; d.bl[3 * k] = b[0]; d.bl[3 * k + 1] = b[1]; d.bl[3 * k + 2] = b[2];
      }
    }
  } else {
    double dsum = 0.0, b[3] = {0, 0, 0};
    if (tid < nl) {
      const int ib = sm.LB[tid] - tl.e0, ie = sm.LB[tid + 1] - tl.e0;
      for (int i = ib; i < ie; ++i) chi += tile_lin_edge_at<WRITE>(d, tl, i, tid, sT + 12 * sCS[i], sm);
      if (WRITE) tile_lin_landmark_obs(d, tl, tid, sm, dsum, b);
      const int hs = sHS[tid];
      chi += tile_lin_ternary_at<WRITE>(d, tl, tid, hs != 255 ? sH + 12 * hs : nullptr, sm, dsum, b);
    }
    if (WRITE) {
      __syncthreads();
      if (tid < nl) {
        if (tid > 0) { dsum += sm.TC[4 * tid - 4]; b[0] += sm.TC[4 * tid - 3]; b[1] += sm.TC[4 * tid - 2]; b[2] += sm.TC[4 * tid - 1]; }
        const size_t k = (size_t)tl.k0 + tid;
        d.hll[k] = dsum; d.bl[3 * k] = b[0]; d.bl[3 * k + 1] = b[1]; d.bl[3 * k + 2] = b[2];
      }
    }
  }
  if (WRITE) {
    // ---- vertex side: one thread per (run, part), one atomic per (vertex, sum) ----
    double* sPart = (double*)(tile_sh + sb(12 * (size_t)(capV + (CHAINS ? capH : 0)) * 8));
    lin_vertex_side(oseg, n_os, sPart, tid,
        [&](int s, auto part, double (&a)[4]) {
          const Seg sgm = oseg[s];
          const int q0 = sgm.begin - tl.e0;
          const double* tv = sT + 12 * sCS[sPS[q0] & 0xFFFFu] + 9;
          const double t[3] = {tv[0], tv[1], tv[2]};
          for (int q = q0; q < q0 + sgm.n; ++q) {
            const uint32_t ps = sPS[q];
            const int i = ps & 0xFFFFu, j = ps >> 16;
            const double w[3] = {sm.P[3 * j] - t[0], sm.P[3 * j + 1] - t[1], sm.P[3 * j + 2] - t[2]};
            acc16_add_part<decltype(part)::value>(a, sm.OM[i], w, sm.EW + 3 * i);
          }
        },
        [&](int v) { return d.accO + 16 * (size_t)v; });
    if (CHAINS) {
      lin_vertex_side(tseg, n_ts, sPart, tid,
          [&](int s, auto part, double (&a)[4]) {
            const Seg sgm = tseg[s];
            const int q0 = sgm.begin - tl.k0;
            const double* tv = sH + 12 * sHS[sTPERM[q0]] + 9;
            const double t[3] = {tv[0], tv[1], tv[2]};
            for (int q = q0; q < q0 + sgm.n; ++q) {
              const int j = sTPERM[q];
              const double w[3] = {sm.P[3 * j + 3] - t[0], sm.P[3 * j + 4] - t[1], sm.P[3 * j + 5] - t[2]};
              acc16_add_part<decltype(part)::value>(a, sm.OMT[j], w, sm.E2 + 3 * j);
            }
          },
          [&](int v) { return d.accT + 16 * (size_t)v; });
      // ---- Q_k: the products of tile_chain_Q, out of the shared pose copy, into the stashes (read by every thread above: barrier) ----
      __syncthreads();
      double* sQ = stash;
      if (tid < tl.t1 - tl.t0) {
        const int jb = sTB[tid] - tl.k0, je = sTB[tid + 1] - tl.k0;
        double Q[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        for (int j = jb; j < je; ++j) {
#pragma unroll
          for (int i = 0; i < 9; ++i) sQ[9 * j + i] = Q[i];
          const int hs = sHS[j];
          if (hs != 255 && j + 1 < je) chain_Q_step(Q, sH + 12 * hs);
        }
      }
      __syncthreads();
      double* gQ = d.pt_Q + 9 * (size_t)(tl.k0 - d.Tstat);
      for (int i = tid; i < 9 * nl; i += VDO_TILE_L) gQ[i] = sQ[i];
    }
  }
  chi = block_sum(chi, red);
  if (tid == 0 && chi != 0.0) atomicAdd(d.scal + SC_CHI2, chi);
}
template <class S, bool CHAINS, bool WRITE>
__global__ void __launch_bounds__(VDO_TILE_L, 4) k_tile_lin(S s) {
  VDO_PICK
  if (CHAINS) k_tile_lin_body<true, WRITE>(d, d.n_tiles_stat, d.capE_ch, d.capV_ch, d.capH_ch, blk_);
  else k_tile_lin_body<false, WRITE>(d, 0, d.capE_st, d.capV_st, 0, blk_);
}

// Preconditioner sums: per vertex S0 = sum c, S1 = sum c w, S2 = sum c w w^T (acc10_add) with c = om^2 g and w = p - t_v, g the
// landmark's block of H_ll^-1 (pointxyz edges: pt_g; ternary edges: tk_gamma).  The vertex side runs as in k_tile_schur2: one thread
// per (run, half) of the vertex-sorted runs of <= VDO_SEG2 entries (osegs2 / tsegs2), a thread summing its five components over its
// run from shared memory and issuing five fp64 atomics.  The warp-per-segment scheme of seg_loop left most lanes idle on the short
// runs of the chain tiles and spent 16 shuffles per segment on a 10-sum transpose reduction.
template <int H>
__device__ __forceinline__ void precond_run_add(double (&a)[5], double c, const double* w) {
  const double ox = c * w[0], oy = c * w[1], oz = c * w[2];
  if (H == 0) { a[0] += c; a[1] += ox; a[2] += oy; a[3] += oz; a[4] += ox * w[0]; }
  else { a[0] += ox * w[1]; a[1] += ox * w[2]; a[2] += oy * w[1]; a[3] += oy * w[2]; a[4] += oz * w[2]; }
}
__device__ __forceinline__ void precond_run_flush(const double (&a)[5], double* dst) {
#pragma unroll
  for (int i = 0; i < 5; ++i) if (a[i] != 0.0) atomicAdd(dst + i, a[i]);
}
// The per-edge arrays are sized by the launch's capE (largest tile of the launch) and carved last, so that the other views keep
// fixed offsets.
inline size_t smem_pre(bool chains, int capE) {      // must mirror the carve order inside k_tile_precond_body
  size_t b = vb<double>(3 * VDO_TILE_L) + vb<double>(VDO_TILE_L) + vb<Seg>(chains ? TILE_OSEG2_CAP_CH : TILE_OSEG2_CAP_ST);
  if (chains) b += vb<double>(VDO_TILE_L) + vb<double>(VDO_TILE_L) + vb<uint16_t>(VDO_TILE_L) + vb<Seg>(TILE_TSEG2_CAP);
  return b + vb<double>(capE) + vb<uint32_t>(capE);
}
template <bool CHAINS>
__device__ __forceinline__ void k_tile_precond_body(const BaDev& d, int tile0, int capE, int bx) {
  extern __shared__ __align__(16) unsigned char tile_sh[];
  __shared__ __align__(8) uint64_t bar;
  const int tid = threadIdx.x;
  const Tile tl = d.tiles[tile0 + bx];
  const int nl = tl.k1 - tl.k0, ne = tl.e1 - tl.e0;
  if (tid == 0) mbar_init(&bar, 1);
  __syncthreads();
  TileStager sg(tile_sh, &bar, tid == 0);
  const double* sP = sg.view<double>(d.pt, 3 * (size_t)tl.k0, 3 * nl, 3 * VDO_TILE_L);
  const double* sG = sg.view<double>(d.pt_g, (size_t)tl.k0, nl, VDO_TILE_L);
  constexpr int OCAP = CHAINS ? TILE_OSEG2_CAP_CH : TILE_OSEG2_CAP_ST;
  const int n_os = tl.qo1 - tl.qo0, n_ts = tl.qt1 - tl.qt0;
  const Seg* so = sg.view<Seg>(d.osegs2, (size_t)tl.qo0, n_os <= OCAP ? n_os : 0, OCAP);
  const Seg* oseg = n_os <= OCAP ? so : d.osegs2 + tl.qo0;
  const double *sGAM = nullptr, *sOMT = nullptr;
  const uint16_t* sTPERM = nullptr;
  const Seg* tseg = nullptr;
  if (CHAINS) {
    sGAM = sg.view<double>(d.tk_gamma, (size_t)tl.k0, nl, VDO_TILE_L);
    sOMT = sg.view<double>(d.tk_omega, (size_t)tl.k0, nl, VDO_TILE_L);
    sTPERM = sg.view<uint16_t>(d.tr_perm, (size_t)tl.k0, nl, VDO_TILE_L);
    const Seg* st = sg.view<Seg>(d.tsegs2, (size_t)tl.qt0, n_ts <= TILE_TSEG2_CAP ? n_ts : 0, TILE_TSEG2_CAP);
    tseg = n_ts <= TILE_TSEG2_CAP ? st : d.tsegs2 + tl.qt0;
  }
  const double* sOM = sg.view<double>(d.lm_omega, (size_t)tl.e0, ne, capE);
  const uint32_t* sPS = sg.view<uint32_t>(d.ob_ps, (size_t)tl.e0, ne, capE);
  sg.commit();
  mbar_wait(&bar, 0);
  for (int item = tid; item < 2 * n_os; item += VDO_TILE_L) {
    const Seg sgm = oseg[item >> 1];
    const double* T = d.se3 + 12 * (size_t)sgm.v;
    const double t[3] = {T[9], T[10], T[11]};
    const int q0 = sgm.begin - tl.e0;
    auto run = [&](auto h) {
      double a[5] = {0, 0, 0, 0, 0};
      for (int q = q0; q < q0 + sgm.n; ++q) {
        const uint32_t ps = sPS[q];
        const int i = ps & 0xFFFFu, j = ps >> 16;
        const double om = sOM[i];
        const double w[3] = {sP[3 * j] - t[0], sP[3 * j + 1] - t[1], sP[3 * j + 2] - t[2]};
        precond_run_add<decltype(h)::value>(a, om * om * sG[j], w);
      }
      precond_run_flush(a, d.accO + 16 * (size_t)sgm.v + 5 * decltype(h)::value);
    };
    if (item & 1) run(std::integral_constant<int, 1>()); else run(std::integral_constant<int, 0>());
  }
  if (CHAINS) {
    for (int item = tid; item < 2 * n_ts; item += VDO_TILE_L) {
      const Seg sgm = tseg[item >> 1];
      const double* T = d.se3 + 12 * (size_t)sgm.v;
      const double t[3] = {T[9], T[10], T[11]};
      const int q0 = sgm.begin - tl.k0;
      auto run = [&](auto h) {
        double a[5] = {0, 0, 0, 0, 0};
        for (int q = q0; q < q0 + sgm.n; ++q) {
          const int j = sTPERM[q];
          const double om = sOMT[j];
          const double w[3] = {sP[3 * j + 3] - t[0], sP[3 * j + 4] - t[1], sP[3 * j + 5] - t[2]};
          precond_run_add<decltype(h)::value>(a, om * om * sGAM[j], w);
        }
        precond_run_flush(a, d.accT + 16 * (size_t)sgm.v + 5 * decltype(h)::value);
      };
      if (item & 1) run(std::integral_constant<int, 1>()); else run(std::integral_constant<int, 0>());
    }
  }
}
template <class S, bool CHAINS>
__global__ void __launch_bounds__(VDO_TILE_L) k_tile_precond(S s) {
  VDO_PICK
  if (CHAINS) k_tile_precond_body<true>(d, d.n_tiles_stat, d.capE_ch, blk_);
  else k_tile_precond_body<false>(d, 0, d.capE_st, blk_);
}

// -------------------------------------------------------------------------------------------------------------------------
// Schur tiles: mode 0 the rhs of the PCG, mode 1 its S*p, mode 2 the back-substitution xl = Hll^-1 (bl - Hlp v), which has no vertex
// side.  The emulation runs the per-item bodies of ba_tiles.cuh (tile_schur_*); this kernel differs from them as follows:
//  * per-edge work is 6 FMAs in both directions.  Forward: u_j = sum_e om_e (gamma_c + 2 p_j x beta_c) =
//    (sum om gamma) + 2 p_j x (sum om beta): one 6-vector FMA per edge, one cross product per LANDMARK.  Backward: the edge's
//    force / torque on its vertex, -om [z_j ; 2 (p_j - t_c) x z_j], is summed as om [z_j ; p_j x z_j] (again a per-landmark
//    6-vector, kept in shared memory) -- i.e. the torque is taken about the WORLD origin and moved to the vertex origin by the
//    per-vertex finalize kernel (torque_v = torque_0 - t_v x force).
//  * the per-vertex vectors vw / vh of the (few dozen) se3 vertices a tile meets are gathered into shared memory while the
//    bulk copies are in flight; edges address them by an 8-bit slot (lm_cslot / tk_hslot, 1 B instead of a 4 B vertex index),
//    so the landmark loop has no global gather on its critical path.
//  * the vertex side is ONE THREAD PER (RUN, COMPONENT): the tile's edges in vertex-sorted order are cut into runs of one
//    vertex and at most VDO_SEG2 = 15 entries (osegs2 / tsegs2; odd, so that threads walking consecutive full runs hit distinct banks); a thread adds its component over its run from shared memory
//    and issues one fp64 atomic.  No shuffles, no selects, no idle lanes on short runs (chain tiles average 8 entries per
//    vertex: a warp per 64-entry segment ran them at 12 % lane utilisation).
//  * chains: the two scalar recurrences of the tracklet solve (forward y_j = c_j + f_{j-1} y_{j-1}, backward
//    z_j = y_j / s_j + g_j z_{j+1}; the coefficients vanish at tracklet boundaries, so no segment bookkeeping) are CTA-wide
//    scans: Kogge-Stone over the 32 lanes of a warp with shuffles, then a carry across the 8 warps through shared memory --
//    instead of one thread per tracklet walking it (<= 53 of 256 threads busy, the rest waiting at the barrier).
//  * mode 2 forms bl - Hlp v with the products of mode 1 (the ternary term enters with its sign flipped through g^), runs the same
//    scans and writes xl; it stages no run lists and has no vertex phase.
//  * only warp 0 polls the mbarrier; the other warps sleep in the CTA barrier.
//  * per-edge / per-vertex arrays are staged with the launch's own capacities (largest tile of the launch, known at ingest):
//    chain tiles (one pointxyz edge per landmark) fit 4 CTAs per SM.
// acc6 layout (12 / vertex): [F_o, M_o, F_t, M_t]  pointxyz force / world-origin torque, ternary force / torque.
inline size_t smem_sch2(bool chains, int capE, int capV, int capH) {      // must mirror the carve order inside k_tile_schur2
  size_t b = sb(6 * (size_t)capV * 8) + (chains ? sb(6 * (size_t)capH * 8) : 0) +
             vb<double>(3 * VDO_TILE_L) + vb<double>(VDO_TILE_L) + vb<int>(VDO_TILE_L + 1) + vb<double>(capE) + vb<uint8_t>(capE) + vb<uint32_t>(capE) +
             vb<Seg>(chains ? TILE_OSEG2_CAP_CH : TILE_OSEG2_CAP_ST) + sb(6 * VDO_TILE_L * 8);
  if (chains) b += vb<double>(9 * VDO_TILE_L) + vb<double>(VDO_TILE_L) + vb<uint8_t>(VDO_TILE_L) + vb<uint16_t>(VDO_TILE_L) + vb<Seg>(TILE_TSEG2_CAP) + sb(64 * 8);
  return b;
}

template <bool CHAINS, int MODE>
__device__ __forceinline__ void k_tile_schur2_body(const BaDev& d, int tile0, int capE, int capV, int capH, int bx) {
  extern __shared__ __align__(16) unsigned char tile_sh[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ uint32_t tab[16];                              // shared-memory offsets of the staged views (computed by warp 0 only)
  if (MODE == 1 && d.scal[SC_DONE] != 0.0) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Tile tl = d.tiles[tile0 + bx];
  const int nl = tl.k1 - tl.k0, ne = tl.e1 - tl.e0, ncam = tl.nv & 0xFFFF, nmot = tl.nv >> 16;
  double* sVW = (double*)tile_sh;                           // vw of the tile's cameras, vh of its motion vertices: fixed places, filled by warps 1..7
  double* sVH = sVW + 6 * capV;
  unsigned char* carve0 = tile_sh + sb(6 * (size_t)capV * 8) + (CHAINS ? sb(6 * (size_t)capH * 8) : 0);
  if (warp == 0) {
    // staging: warp 0 alone carves the views, issues the bulk copies (lane 0) and waits for them; the other warps meanwhile gather
    // the per-vertex vectors and then sleep in the CTA barrier
    if (lane == 0) mbar_init(&bar, 1);
    __syncwarp();
    TileStager sg(carve0, &bar, lane == 0);
    auto off = [&](const void* ptr) { return (uint32_t)((const unsigned char*)ptr - tile_sh); };
    uint32_t o[16];
    o[0] = off(sg.view<double>(d.pt, 3 * (size_t)tl.k0, 3 * nl, 3 * VDO_TILE_L));
    o[1] = off(sg.view<double>(d.pt_s, (size_t)tl.k0, nl, VDO_TILE_L));
    o[2] = off(sg.view<int>(d.lm_obs_begin, (size_t)tl.k0, nl + 1, VDO_TILE_L + 1));
    o[3] = off(sg.view<double>(d.lm_omega, (size_t)tl.e0, ne, capE));
    o[4] = off(sg.view<uint8_t>(d.lm_cslot, (size_t)tl.e0, MODE != 0 ? ne : 0, capE));
    o[5] = off(sg.view<uint32_t>(d.ob_ps, (size_t)tl.e0, MODE != 2 ? ne : 0, capE));
    {
      const int cap = CHAINS ? TILE_OSEG2_CAP_CH : TILE_OSEG2_CAP_ST, n = tl.qo1 - tl.qo0;
      o[6] = off(sg.view<Seg>(d.osegs2, (size_t)tl.qo0, MODE != 2 && n <= cap ? n : 0, cap));
    }
    o[7] = off(sg.stash<double>(6 * VDO_TILE_L));
    if (CHAINS) {
      o[8] = off(sg.view<double>(d.pt_Q, 9 * (size_t)(tl.k0 - d.Tstat), 9 * nl, 9 * VDO_TILE_L));
      o[9] = off(sg.view<double>(d.tk_omega, (size_t)tl.k0, nl, VDO_TILE_L));
      o[10] = off(sg.view<uint8_t>(d.tk_hslot, (size_t)tl.k0, nl, VDO_TILE_L));
      o[11] = off(sg.view<uint16_t>(d.tr_perm, (size_t)tl.k0, MODE != 2 ? nl : 0, VDO_TILE_L));
      const int n = tl.qt1 - tl.qt0;
      o[12] = off(sg.view<Seg>(d.tsegs2, (size_t)tl.qt0, MODE != 2 && n <= TILE_TSEG2_CAP ? n : 0, TILE_TSEG2_CAP));
      o[13] = off(sg.stash<double>(64));
    }
    sg.commit();
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < (CHAINS ? 14 : 8); ++i) tab[i] = o[i];
    }
    mbar_wait(&bar, 0);
  } else if (MODE != 0) {
    for (int i = tid - 32; i < 6 * ncam; i += VDO_TILE_L - 32) { const int s = i / 6; sVW[i] = d.vw[6 * (size_t)d.tile_verts[tl.vs0 + s] + (i - 6 * s)]; }
    if (CHAINS) for (int i = tid - 32; i < 6 * nmot; i += VDO_TILE_L - 32) { const int s = i / 6; sVH[i] = d.vh[6 * (size_t)d.tile_verts[tl.vs0 + ncam + s] + (i - 6 * s)]; }
  }
  __syncthreads();
  double* sP = (double*)(tile_sh + tab[0]);
  double* sS = (double*)(tile_sh + tab[1]);
  const int* sLB = (const int*)(tile_sh + tab[2]);
  const double* sOM = (const double*)(tile_sh + tab[3]);
  const uint8_t* sCS = (const uint8_t*)(tile_sh + tab[4]);
  const uint32_t* sPS = (const uint32_t*)(tile_sh + tab[5]);
  const int n_os = tl.qo1 - tl.qo0;
  const Seg* oseg = n_os <= (CHAINS ? TILE_OSEG2_CAP_CH : TILE_OSEG2_CAP_ST) ? (const Seg*)(tile_sh + tab[6]) : d.osegs2 + tl.qo0;
  double* sZM = (double*)(tile_sh + tab[7]);                // per landmark [z ; p x z] at the end; chains: first half g^, second half z^ until then
  double *sQ = nullptr, *sAM = nullptr, *sOMT = nullptr, *sZ = sZM, *sY = sZM + 3 * VDO_TILE_L, *sWS = nullptr;
  const uint8_t* sHS = nullptr; const uint16_t* sTPERM = nullptr; const Seg* tseg = nullptr;
  const int n_ts = tl.qt1 - tl.qt0;
  if (CHAINS) {
    sQ = (double*)(tile_sh + tab[8]); sAM = (double*)(((uintptr_t)sQ + 15) & ~(uintptr_t)15);   // Q_k's space holds the ternary sums at the end (16-byte aligned)
    sOMT = (double*)(tile_sh + tab[9]); sHS = (const uint8_t*)(tile_sh + tab[10]); sTPERM = (const uint16_t*)(tile_sh + tab[11]);
    tseg = n_ts <= TILE_TSEG2_CAP ? (const Seg*)(tile_sh + tab[12]) : d.tsegs2 + tl.qt0;
    sWS = (double*)(tile_sh + tab[13]);
  }
  // ---- landmark phase ----
  double p[3] = {0, 0, 0}, u[3] = {0, 0, 0};
  if (tid < nl) {
    p[0] = sP[3 * tid]; p[1] = sP[3 * tid + 1]; p[2] = sP[3 * tid + 2];
    if (MODE != 0) {
      double a[6] = {0, 0, 0, 0, 0, 0};
      const int ib = sLB[tid] - tl.e0, ie = sLB[tid + 1] - tl.e0;
      for (int i = ib; i < ie; ++i) {
        const double om = sOM[i];
        const double2* w = reinterpret_cast<const double2*>(sVW + 6 * (int)sCS[i]);
        const double2 w0 = w[0], w1 = w[1], w2 = w[2];
        a[0] += om * w0.x; a[1] += om * w0.y; a[2] += om * w1.x; a[3] += om * w1.y; a[4] += om * w2.x; a[5] += om * w2.y;
      }
      double pxb[3]; cross3(sP + 3 * tid, a + 3, pxb);   // p from shared memory: static mode 2 would spill p across the loop
      u[0] = a[0] + 2 * pxb[0]; u[1] = a[1] + 2 * pxb[1]; u[2] = a[2] + 2 * pxb[2];
    }
    if (MODE != 1) {
      const double* b = d.bl + 3 * ((size_t)tl.k0 + tid);
      u[0] = b[0] - u[0]; u[1] = b[1] - u[1]; u[2] = b[2] - u[2];
    }
  }
  if (!CHAINS) {
    if (tid < nl) {
      const double is = 1.0 / sS[tid];
      const double z[3] = {u[0] * is, u[1] * is, u[2] * is};
      if (MODE == 2) {
        double* o = d.xl + 3 * ((size_t)tl.k0 + tid);
        o[0] = z[0]; o[1] = z[1]; o[2] = z[2];
      } else {
        double m[3]; cross3(p, z, m);
        double2* o = reinterpret_cast<double2*>(sZM + 6 * tid);
        o[0] = make_double2(z[0], z[1]); o[1] = make_double2(z[2], m[0]); o[2] = make_double2(m[1], m[2]);
      }
    }
  } else {
    // chains: H_ll of a tracklet is (scalar tridiagonal) (x) I3 in the frame x^_k = Q_k x_k (see ba_tiles.cuh)
    const bool live = tid < nl;
    const bool has_out = live && sHS[tid] != 255;
    double uh[3] = {0, 0, 0}, is = 0.0, omt = 0.0;
    if (live) {
      const double* Q = sQ + 9 * tid;
      is = 1.0 / sS[tid]; omt = sOMT[tid];
      rot_apply(Q, u, uh);                               // mode 0: b^ = Q b_l; mode 2: Q (b_l - u)
      if (MODE != 0) {
        double gh[3] = {0, 0, 0};
        const int hp = tid > 0 ? (int)sHS[tid - 1] : 255;
        if (hp != 255) {                                 // incoming ternary edge (k-1, k)
          const double* w = sVH + 6 * hp;
          double pxb[3]; cross3(p, w + 3, pxb);
          const double sgn = MODE == 1 ? 1.0 : -1.0;     // mode 2: -Hlp v
          const double g[3] = {sgn * (w[0] - pxb[0]), sgn * (w[1] - pxb[1]), sgn * (w[2] - pxb[2])};
          rot_apply(Q, g, gh);
          const double om = sOMT[tid - 1];
          uh[0] -= om * gh[0]; uh[1] -= om * gh[1]; uh[2] -= om * gh[2];
        }
        sZ[3 * tid] = gh[0]; sZ[3 * tid + 1] = gh[1]; sZ[3 * tid + 2] = gh[2];
      }
      sS[tid] = omt * is;                                // f_j = om_j / s_j, read by landmark j + 1
    }
    __syncthreads();
    if (MODE != 0 && has_out) {                          // outgoing ternary edge (k, k+1)
      uh[0] += omt * sZ[3 * tid + 3]; uh[1] += omt * sZ[3 * tid + 4]; uh[2] += omt * sZ[3 * tid + 5];
    }
    // forward: y_j = u^_j + f_{j-1} y_{j-1}   (f = 0 across tracklet boundaries)
    double a = (live && tid > 0) ? sS[tid - 1] : 0.0;
    double b0 = uh[0], b1 = uh[1], b2 = uh[2];
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const double ap = __shfl_up_sync(0xffffffffu, a, dd), p0 = __shfl_up_sync(0xffffffffu, b0, dd), p1 = __shfl_up_sync(0xffffffffu, b1, dd), p2 = __shfl_up_sync(0xffffffffu, b2, dd);
      if (lane >= dd) { b0 += a * p0; b1 += a * p1; b2 += a * p2; a *= ap; }
    }
    if (lane == 31) { sWS[4 * warp] = a; sWS[4 * warp + 1] = b0; sWS[4 * warp + 2] = b1; sWS[4 * warp + 3] = b2; }
    __syncthreads();
    {
      double c0 = 0, c1 = 0, c2 = 0;
      for (int w2 = 0; w2 < warp; ++w2) { const double a2 = sWS[4 * w2]; c0 = sWS[4 * w2 + 1] + a2 * c0; c1 = sWS[4 * w2 + 2] + a2 * c1; c2 = sWS[4 * w2 + 3] + a2 * c2; }
      b0 += a * c0; b1 += a * c1; b2 += a * c2;          // y_j
    }
    // backward: z_j = y_j / s_j + (om_j / s_j) z_{j+1}
    double g = live ? omt * is : 0.0;
    double e0 = b0 * is, e1 = b1 * is, e2 = b2 * is;
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const double gp = __shfl_down_sync(0xffffffffu, g, dd), p0 = __shfl_down_sync(0xffffffffu, e0, dd), p1 = __shfl_down_sync(0xffffffffu, e1, dd), p2 = __shfl_down_sync(0xffffffffu, e2, dd);
      if (lane + dd < 32) { e0 += g * p0; e1 += g * p1; e2 += g * p2; g *= gp; }
    }
    if (lane == 0) { sWS[32 + 4 * warp] = g; sWS[32 + 4 * warp + 1] = e0; sWS[32 + 4 * warp + 2] = e1; sWS[32 + 4 * warp + 3] = e2; }
    __syncthreads();
    {
      double c0 = 0, c1 = 0, c2 = 0;
      for (int w2 = VDO_TILE_L / 32 - 1; w2 > warp; --w2) { const double g2 = sWS[32 + 4 * w2]; c0 = sWS[32 + 4 * w2 + 1] + g2 * c0; c1 = sWS[32 + 4 * w2 + 2] + g2 * c1; c2 = sWS[32 + 4 * w2 + 3] + g2 * c2; }
      e0 += g * c0; e1 += g * c1; e2 += g * c2;          // z^_j
    }
    if (MODE == 2) {
      if (live) { const double zh[3] = {e0, e1, e2}; rot_t_apply(sQ + 9 * tid, zh, d.xl + 3 * ((size_t)tl.k0 + tid)); }
      return;
    }
    if (live) { sY[3 * tid] = e0; sY[3 * tid + 1] = e1; sY[3 * tid + 2] = e2; }
    __syncthreads();
    double zm[6] = {0, 0, 0, 0, 0, 0}, am[6] = {0, 0, 0, 0, 0, 0};
    if (live) {
      const double zh[3] = {e0, e1, e2};
      rot_t_apply(sQ + 9 * tid, zh, zm);
      cross3(p, zm, zm + 3);
      if (has_out) {                                       // ternary edge (k, k+1): a' = Q_{k+1}^T (z^_k - z^_{k+1}); om [a' ; p_{k+1} x a']
        const double dz[3] = {e0 - sY[3 * tid + 3], e1 - sY[3 * tid + 4], e2 - sY[3 * tid + 5]};
        double av[3]; rot_t_apply(sQ + 9 * (tid + 1), dz, av);
        double cv[3]; cross3(sP + 3 * tid + 3, av, cv);
        am[0] = omt * av[0]; am[1] = omt * av[1]; am[2] = omt * av[2]; am[3] = omt * cv[0]; am[4] = omt * cv[1]; am[5] = omt * cv[2];
      }
    }
    __syncthreads();                                       // every thread has read Q / z^: their space is reused
    if (live) {
      double2* o = reinterpret_cast<double2*>(sZM + 6 * tid); double2* o2 = reinterpret_cast<double2*>(sAM + 6 * tid);
      o[0] = make_double2(zm[0], zm[1]); o[1] = make_double2(zm[2], zm[3]); o[2] = make_double2(zm[4], zm[5]);
      o2[0] = make_double2(am[0], am[1]); o2[1] = make_double2(am[2], am[3]); o2[2] = make_double2(am[4], am[5]);
    }
  }
  if (MODE == 2) return;
  __syncthreads();
  // ---- vertex phase: one thread per (run, component pair) ----
  for (int item = tid; item < 3 * n_os; item += VDO_TILE_L) {
    const int s = item / 3, c2 = item - 3 * s;
    const Seg sgm = oseg[s];
    const int q0 = sgm.begin - tl.e0;
    double ax = 0.0, ay = 0.0;
#pragma unroll 4
    for (int q = q0; q < q0 + sgm.n; ++q) {
      const uint32_t ps = sPS[q];
      const double om = sOM[ps & 0xFFFFu];
      const double2 zz = *reinterpret_cast<const double2*>(sZM + 6 * (int)(ps >> 16) + 2 * c2);
      ax += om * zz.x; ay += om * zz.y;
    }
    // components (2 c2, 2 c2 + 1) of [F_o ; M_o] = -[sum om z ; 2 sum om p x z]
    double* dst = d.acc6 + 12 * (size_t)sgm.v + 2 * c2;
    const double fx = c2 == 0 ? -1.0 : (c2 == 1 ? -1.0 : -2.0), fy = c2 == 0 ? -1.0 : -2.0;
    if (ax != 0.0) atomicAdd(dst, fx * ax);
    if (ay != 0.0) atomicAdd(dst + 1, fy * ay);
  }
  if (CHAINS) {
    for (int item = tid; item < 3 * n_ts; item += VDO_TILE_L) {
      const int s = item / 3, c2 = item - 3 * s;
      const Seg sgm = tseg[s];
      const int q0 = sgm.begin - tl.k0;
      double ax = 0.0, ay = 0.0;
#pragma unroll 4
      for (int q = q0; q < q0 + sgm.n; ++q) { const double2 zz = *reinterpret_cast<const double2*>(sAM + 6 * (int)sTPERM[q] + 2 * c2); ax += zz.x; ay += zz.y; }
      double* dst = d.acc6 + 12 * (size_t)sgm.v + 6 + 2 * c2;
      if (ax != 0.0) atomicAdd(dst, ax);
      if (ay != 0.0) atomicAdd(dst + 1, ay);
    }
  }
}
template <class S, bool CHAINS, int MODE>
__global__ void __launch_bounds__(VDO_TILE_L, CHAINS ? 4 : 5) k_tile_schur2(S s) {
  VDO_PICK
  if (CHAINS) k_tile_schur2_body<true, MODE>(d, d.n_tiles_stat, d.capE_ch, d.capV_ch, d.capH_ch, blk_);
  else k_tile_schur2_body<false, MODE>(d, 0, d.capE_st, d.capV_st, 1, blk_);
}

// -------------------------------------------------------------------------------------------------------------------------
// Banded static block of the reduced matrix.  band[(a - band_v0) * W + k] holds the 10 moments  sum_l g [1, p_l, p_l p_l^T],
// g = om_la om_l(a+k) / s_l, over the static landmarks seen by both vertex a and vertex a + k (k = 0: om_la^2 / s_l): everything S_static
// needs (the Jacobians are [I ; p x] up to the per-vertex frame change the finalize kernel applies).  It is re-formed for every LM trial
// (s_l = sum om + lambda) and turns the PCG's static product from a 79 MB pass over the edges into a 2.4 MB banded multiply (k_band_mul).
//
// Formation: CTAs own runs of consecutive static tiles (tiles are ordered by first vertex, so a run meets a window of ~40 vertices).  Per tile,
// a WARP takes a vertex c of the tile and walks c's edges in the tile's vertex-sorted order, four edges per step: lane = (edge of the step, offset
// k < 8).  A landmark's edges are sorted by vertex, so the partner edge of edge i for offset k is at most k places further.  All lanes of a warp
// run the same trip count (a first version with one thread per (vertex, k) ran at the longest edge list of the 32 vertices in its warp).
// The few pairs with offset >= 8 (tracks longer than 8 frames) are done by a thread per landmark.  Sums go to a shared-memory window of the
// CTA (vertex x offset x 10 moments) and from there to the band with atomics when the run ends: 10 atomics per (vertex, k) and RUN of tiles.
constexpr int BAND_SPAN = 36, BAND_KS = 16;   // window: vertices x offsets kept in shared memory (the rest goes straight to global atomics)
inline size_t smem_band(int capE) {
  return sb(3 * VDO_TILE_L * 8) + sb(VDO_TILE_L * 8) + sb((VDO_TILE_L + 1) * 4) + sb((size_t)capE * 8) + 2 * sb((size_t)capE) + 2 * sb((size_t)capE * 4) + 3 * sb(256 * 4) +
         sb((size_t)BAND_SPAN * BAND_KS * 10 * 8);
}
__device__ __forceinline__ void k_band_form_body(const BaDev& d, int tiles_per_cta, int capE, int bx) {
  extern __shared__ __align__(16) unsigned char tile_sh[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned char* c0 = tile_sh;
  auto carve = [&](size_t bytes) { unsigned char* p = c0; c0 += sb(bytes); return p; };
  double* sP = (double*)carve(3 * VDO_TILE_L * 8);
  double* sIS = (double*)carve(VDO_TILE_L * 8);
  int* sLB = (int*)carve((VDO_TILE_L + 1) * 4);
  double* sOM = (double*)carve((size_t)capE * 8);
  uint8_t* sCS = (uint8_t*)carve((size_t)capE);
  uint32_t* sPS = (uint32_t*)carve((size_t)capE * 4);
  int* sCAM = (int*)carve((size_t)capE * 4);                  // per edge (landmark-major): its vertex number
  uint8_t* sREM = (uint8_t*)carve((size_t)capE);              // ... and how many edges of the same landmark follow it
  int* sTV = (int*)carve(256 * 4);
  int* sQ0 = (int*)carve(256 * 4);
  int* sQ1 = (int*)carve(256 * 4);
  double* sACC = (double*)carve((size_t)BAND_SPAN * BAND_KS * 10 * 8);
  __shared__ int sML[2];                                       // longest track of the current tile (double buffered: reset one tile ahead)
  if (tid < 2) sML[tid] = 0;
  const int t_begin = bx * tiles_per_cta, t_end = min(t_begin + tiles_per_cta, d.n_tiles_stat);
  if (t_begin >= t_end) return;
  for (int i = tid; i < BAND_SPAN * BAND_KS * 10; i += VDO_TILE_L) sACC[i] = 0.0;
  const int W = d.band_W;
  const int vbase = d.tile_verts[d.tiles[t_begin].vs0];
  auto moments = [&](double g, int l, double (&acc)[10]) {
    const double px = sP[3 * l], py = sP[3 * l + 1], pz = sP[3 * l + 2];
    const double gx = g * px, gy = g * py, gz = g * pz;
    acc[0] += g; acc[1] += gx; acc[2] += gy; acc[3] += gz;
    acc[4] += gx * px; acc[5] += gx * py; acc[6] += gx * pz; acc[7] += gy * py; acc[8] += gy * pz; acc[9] += gz * pz;
  };
  for (int t = t_begin; t < t_end; ++t) {
    const Tile tl = d.tiles[t];
    const int nl = tl.k1 - tl.k0, ne = tl.e1 - tl.e0, ncam = tl.nv & 0xFFFF, n_os = tl.qo1 - tl.qo0;
    __syncthreads();                                           // the previous tile is done with the staged arrays
    if (tid < nl) {
      const size_t k = (size_t)tl.k0 + tid;
      sP[3 * tid] = d.pt[3 * k]; sP[3 * tid + 1] = d.pt[3 * k + 1]; sP[3 * tid + 2] = d.pt[3 * k + 2];
      sIS[tid] = 1.0 / d.pt_s[k];
    }
    for (int i = tid; i <= nl; i += VDO_TILE_L) sLB[i] = d.lm_obs_begin[tl.k0 + i] - tl.e0;
    for (int e = tid; e < ne; e += VDO_TILE_L) { sOM[e] = d.lm_omega[tl.e0 + e]; sCS[e] = d.lm_cslot[tl.e0 + e]; sPS[e] = d.ob_ps[tl.e0 + e]; }
    if (tid < ncam) sTV[tid] = d.tile_verts[tl.vs0 + tid];
    __syncthreads();
    for (int s = tid; s < n_os; s += VDO_TILE_L) {
      const Seg g = d.osegs2[tl.qo0 + s];
      const int q0 = g.begin - tl.e0, slot = sCS[sPS[q0] & 0xFFFFu];
      if (s == 0 || d.osegs2[tl.qo0 + s - 1].v != g.v) sQ0[slot] = q0;
      if (s == n_os - 1 || d.osegs2[tl.qo0 + s + 1].v != g.v) sQ1[slot] = q0 + g.n;
    }
    if (tid < nl && sLB[tid + 1] > sLB[tid]) atomicMax(&sML[t & 1], sTV[sCS[sLB[tid + 1] - 1]] - sTV[sCS[sLB[tid]]] + 1);
    for (int e = tid; e < ne; e += VDO_TILE_L) { sCAM[e] = sTV[sCS[e]]; sREM[e] = (uint8_t)min(255, sLB[(int)d.lm_lml[tl.e0 + e] + 1] - 1 - e); }
    if (tid == 0) sML[(t + 1) & 1] = 0;
    __syncthreads();
    const int vlast = sTV[ncam - 1];
    // Each warp takes an equal share [qa, qb) of the tile's edges in vertex-sorted order (a vertex's edges are contiguous there) and walks it
    // vertex by vertex, 4 edges per step: lane = (sub-edge, offset within a sweep of 8 offsets); sweeps beyond the first only when the tile has
    // tracks that long.  A vertex whose edges straddle two shares is summed by both warps: the window is updated with shared-memory atomics.
    const int sub = lane >> 3, maxlen = sML[t & 1];
    const int qa = (int)((long long)ne * warp / (VDO_TILE_L / 32)), qb = (int)((long long)ne * (warp + 1) / (VDO_TILE_L / 32));
    int c = 0;
    if (qa < qb) { int lo = 0, hi = ncam - 1; while (lo < hi) { const int mid = (lo + hi) >> 1; if (sQ1[mid] > qa) hi = mid; else lo = mid + 1; } c = lo; }
    for (int q0 = qa; q0 < qb; ++c) {
      const int q1 = min(sQ1[c], qb), vc = sTV[c];
      const int kmax = min(min(W, maxlen), vlast - vc + 1);      // offsets that can have a pair at all
      for (int k0 = 0; k0 < kmax; k0 += 8) {
        const int k = k0 + (lane & 7), target = vc + k;
        double acc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        if (k < kmax)
          for (int q = q0 + sub; q < q1; q += 4) {
            const uint32_t ps = sPS[q];
            const int i = (int)(ps & 0xFFFFu), l = (int)(ps >> 16);
            int j = i + min(k, (int)sREM[i]);                        // a landmark's edges are sorted by vertex: the partner is at most k places on
            int cj = sCAM[j];
            while (cj > target) cj = sCAM[--j];                     // (stops at j == i at the latest: vertex vc <= target)
            if (cj != target) continue;
            moments(sOM[i] * sOM[j] * sIS[l], l, acc);
          }
        __syncwarp();
#pragma unroll
        for (int m = 0; m < 10; ++m) { acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], 8); acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], 16); }
        if (lane < 8 && acc[0] != 0.0) {
          const int r = vc - vbase;
          const bool win = r >= 0 && r < BAND_SPAN && k < BAND_KS;
          if (win && q0 == sQ0[c] && q1 == sQ1[c]) {               // the whole vertex is this warp's: plain update
            double* dst = sACC + ((size_t)r * BAND_KS + k) * 10;
#pragma unroll
            for (int m = 0; m < 10; ++m) dst[m] += acc[m];
          } else if (win) {
            double* dst = sACC + ((size_t)r * BAND_KS + k) * 10;
#pragma unroll
            for (int m = 0; m < 10; ++m) atomicAdd(dst + m, acc[m]);
          } else {
            double* dst = d.band + ((size_t)(vc - d.band_v0) * W + k) * 10;
#pragma unroll
            for (int m = 0; m < 10; ++m) atomicAdd(dst + m, acc[m]);
          }
        }
      }
      q0 = q1;
    }
  }
  __syncthreads();
  for (int e = tid; e < BAND_SPAN * BAND_KS; e += VDO_TILE_L) {
    const int r = e / BAND_KS, k = e - r * BAND_KS;
    const double* src = sACC + (size_t)e * 10;
    if (src[0] == 0.0 || k >= W) continue;
    double* dst = d.band + ((size_t)(vbase + r - d.band_v0) * W + k) * 10;
#pragma unroll
    for (int m = 0; m < 10; ++m) atomicAdd(dst + m, src[m]);
  }
}
template <class S>
__global__ void __launch_bounds__(VDO_TILE_L, 3) k_band_form(S s) { VDO_PICK k_band_form_body(d, s.tiles_per_cta(g_), d.capE_st, blk_); }

// S_static * p from the band (replaces k_tile_schur2<static, 1> inside the PCG): one warp per row a, lanes over the offsets -(W-1) .. W-1.
// With vw_b = [gamma_b ; beta_b] and the moments (M0, M1, M2) of the pair (a, b):
//   F_o[a] -= M0 gamma_b + 2 M1 x beta_b,      M_o[a] -= 2 (M1 x gamma_b + 2 (M2 - tr(M2) I) beta_b)
// (the sums the static tile kernel leaves in acc6: p x (p x beta) = (p p^T - |p|^2 I) beta).  The band is 2.4 MB for 1000 cameras and W = 30:
// L2-resident, against 79 MB of edge data per product for the matrix-free kernel.
__device__ __forceinline__ void k_band_mul_body(const BaDev& d, int bx) {
  if (d.scal[SC_DONE] != 0.0) return;
  const int a = bx * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (a >= d.band_n) return;
  const int W = d.band_W;
  double F[3] = {0, 0, 0}, M[3] = {0, 0, 0};
  for (int o = lane; o < 2 * W - 1; o += 32) {
    const int kk = o - (W - 1), b = a + kk;
    if (b < 0 || b >= d.band_n) continue;
    const double* m = d.band + (kk >= 0 ? ((size_t)a * W + kk) : ((size_t)b * W - kk)) * 10;
    const double m0 = m[0];
    if (m0 == 0.0) continue;
    const double* w = d.vw + 6 * (size_t)(d.band_v0 + b);
    const double g[3] = {w[0], w[1], w[2]}, be[3] = {w[3], w[4], w[5]};
    const double m1[3] = {m[1], m[2], m[3]};
    double c1[3], c2[3];
    cross3(m1, be, c1); cross3(m1, g, c2);
    const double tr = m[4] + m[7] + m[9];
    const double q0 = m[4] * be[0] + m[5] * be[1] + m[6] * be[2] - tr * be[0];
    const double q1 = m[5] * be[0] + m[7] * be[1] + m[8] * be[2] - tr * be[1];
    const double q2 = m[6] * be[0] + m[8] * be[1] + m[9] * be[2] - tr * be[2];
    F[0] -= m0 * g[0] + 2 * c1[0]; F[1] -= m0 * g[1] + 2 * c1[1]; F[2] -= m0 * g[2] + 2 * c1[2];
    M[0] -= 2 * (c2[0] + 2 * q0); M[1] -= 2 * (c2[1] + 2 * q1); M[2] -= 2 * (c2[2] + 2 * q2);
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
    for (int i = 0; i < 3; ++i) { F[i] += __shfl_down_sync(0xffffffffu, F[i], s); M[i] += __shfl_down_sync(0xffffffffu, M[i], s); }
  }
  if (lane == 0) {
    double* dst = d.acc6 + 12 * (size_t)(d.band_v0 + a);
    atomicAdd(dst, F[0]); atomicAdd(dst + 1, F[1]); atomicAdd(dst + 2, F[2]); atomicAdd(dst + 3, M[0]); atomicAdd(dst + 4, M[1]); atomicAdd(dst + 5, M[2]);
  }
}
template <class S>
__global__ void __launch_bounds__(256) k_band_mul(S s) { VDO_PICK k_band_mul_body(d, blk_); }

// per vertex: out_v += sign * B^T [F ; M - t x (2 F_o + F_t)] (torque moved to the vertex origin); clears the sums.
__device__ __forceinline__ void k_tile_finalize_schur2_body(const BaDev& d, double sign, double* __restrict__ out, int check_done, int bx) {
  if (check_done && d.scal[SC_DONE] != 0.0) return;
  const int v = bx * blockDim.x + threadIdx.x;
  if (v < d.C) {
    const double* T = d.se3 + 12 * (size_t)v;
    double* a = d.acc6 + 12 * (size_t)v;
    const double F[3] = {a[0] + a[6], a[1] + a[7], a[2] + a[8]};
    const double G[3] = {2 * a[0] + a[6], 2 * a[1] + a[7], 2 * a[2] + a[8]};
    double txg[3]; cross3(T + 9, G, txg);
    const double M[3] = {a[3] + a[9] - txg[0], a[4] + a[10] - txg[1], a[5] + a[11] - txg[2]};
    double o0[3], o1[3];
    rot_t_apply(T, F, o0); rot_t_apply(T, M, o1);
    double* o = out + 6 * (size_t)v;
    o[0] += sign * o0[0]; o[1] += sign * o0[1]; o[2] += sign * o0[2]; o[3] += sign * o1[0]; o[4] += sign * o1[1]; o[5] += sign * o1[2];
#pragma unroll
    for (int i = 0; i < 12; ++i) a[i] = 0.0;
  }
}
// OUT: where the product goes -- the dense path's right-hand side, the PCG's rhs, or its Ap (stops once converged)
enum { FIN_DENSE_RHS, FIN_RHS, FIN_AP };
template <class S, int OUT>
__global__ void __launch_bounds__(128) k_tile_finalize_schur2(S s) {
  VDO_PICK
  if (OUT == FIN_DENSE_RHS) k_tile_finalize_schur2_body(d, -1.0, d.Sdense + 36 * (size_t)d.C * d.C, 0, blk_);
  else if (OUT == FIN_RHS) k_tile_finalize_schur2_body(d, -1.0, d.rhs, 0, blk_);
  else k_tile_finalize_schur2_body(d, -1.0, d.Ap, 1, blk_);
}
// The fused PCG iteration's finalize: Ap -= B^T sums and the partial of p.Ap against p = p_{k+1} of each 128 vertices (part_pap[bx]).
// Eight lanes per vertex (lane r < 6 forms row r; 1024 threads for the 128 vertices of a partial): with one thread per vertex, config 5
// (C = 13 416) left 4 warps per SM.  Every value is formed as in k_tile_finalize_schur2_body (a lane evaluates the row of rot_t_apply it
// owns), and each partial adds its 128 vertex terms in the order of block_sum over a 128-thread CTA: the same bits.
__device__ __forceinline__ void k_tile_finalize_ap_dot_body(const BaDev& d, const double* __restrict__ pdot, int bx) {
  __shared__ double sv[128], red[4];
  if (d.scal[SC_DONE] != 0.0) return;
  const int t = threadIdx.x >> 3, r = threadIdx.x & 7, v = bx * 128 + t;
  const unsigned int grp = 0xffu << (threadIdx.x & 24);
  double sdot = 0.0;
  if (v < d.C) {
    const double* T = d.se3 + 12 * (size_t)v;
    double* a = d.acc6 + 12 * (size_t)v;
    const double F[3] = {a[0] + a[6], a[1] + a[7], a[2] + a[8]};
    const double G[3] = {2 * a[0] + a[6], 2 * a[1] + a[7], 2 * a[2] + a[8]};
    double txg[3]; cross3(T + 9, G, txg);
    const double M[3] = {a[3] + a[9] - txg[0], a[4] + a[10] - txg[1], a[5] + a[11] - txg[2]};
    __syncwarp(grp);                                           // the vertex's lanes have read its sums
    double o = 0.0;
    if (r < 6) {
      const int k = r < 3 ? r : r - 3;
      const double w0 = r < 3 ? F[0] : M[0], w1 = r < 3 ? F[1] : M[1], w2 = r < 3 ? F[2] : M[2];
      const double q = T[k] * w0 + T[3 + k] * w1 + T[6 + k] * w2;   // row k of rot_t_apply(T, F or M)
      double* out = d.Ap + 6 * (size_t)v + r;
      o = *out + -1.0 * q;
      *out = o;
      a[r] = 0.0; a[r + 6] = 0.0;
    }
    double ov[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) ov[i] = __shfl_sync(grp, o, (threadIdx.x & 31 & ~7) + i);
    if (r == 0) {
      const double* pv = pdot + 6 * (size_t)v;
      sdot = pv[0] * ov[0] + pv[1] * ov[1] + pv[2] * ov[2] + pv[3] * ov[3] + pv[4] * ov[4] + pv[5] * ov[5];
    }
  }
  if (r == 0) sv[t] = sdot;
  __syncthreads();
  // block_sum of a 128-thread CTA over sv
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double x = 0.0;
  if (threadIdx.x < 128) {
    x = warp_sum(sv[threadIdx.x]);
    if (lane == 0) red[w] = x;
  }
  __syncthreads();
  if (w == 0) {
    x = lane < 4 ? red[lane] : 0.0;
    x = warp_sum(x);
    if (lane == 0) d.part_pap[bx] = x;
  }
}
template <class S>
__global__ void __launch_bounds__(1024) k_tile_finalize_ap_dot(S s) { VDO_PICK k_tile_finalize_ap_dot_body(d, s.parity() ? d.p : d.p2, blk_); }

__device__ __forceinline__ void k_tile_finalize_lin_body(const BaDev& d, int bx) {
  const int v = bx * blockDim.x + threadIdx.x;
  if (v < d.C) tile_finalize_lin(d, v);
}
template <class S>
__global__ void __launch_bounds__(128) k_tile_finalize_lin(S s) { VDO_PICK k_tile_finalize_lin_body(d, blk_); }
__device__ __forceinline__ void k_tile_finalize_precond_body(const BaDev& d, int bx) {
  const int v = bx * blockDim.x + threadIdx.x;
  if (v < d.C) tile_finalize_precond(d, v);
}
template <class S>
__global__ void __launch_bounds__(128) k_tile_finalize_precond(S s) { VDO_PICK k_tile_finalize_precond_body(d, blk_); }

}  // namespace vdo
