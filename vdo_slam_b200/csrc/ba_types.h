// ba_types.h -- HBM data layout of one batch factor graph and the backend interface the LM driver runs on.
//
// Layout (all fp64 unless noted).  "Landmark" = VertexPointXYZ.  Landmarks are renumbered so that each tracklet
// (a static point, or the chain p_0 - p_1 - ... of per-frame copies of one dynamic point tied by
// LandmarkMotionTernaryEdges) is contiguous and in chain order; that makes H_ll block-tridiagonal per tracklet.
//
//   se3[C*12]            vertex estimates (camera poses + object motions), AoS iso
//   pt[P*3]              landmark estimates, tracklet order
//   tk_begin[T+1]        landmark range of tracklet t
//   landmark-major EdgeSE3PointXYZ stream (sorted by landmark): lm_obs_begin[P+1], lm_cam[E], lm_z[E*3], lm_cls[E] (u8),
//                        lm_omega[E] (robustified weight, rewritten by every linearisation)
//   per landmark k:      tk_h[k]  = motion vertex of the ternary edge (k, k+1), or -1;  tk_cls[k]; tk_omega[k]
//   (chunked layout only) vertex-major EdgeSE3PointXYZ stream (sorted by se3 vertex): vm_pt[E], vm_z[E*3], vm_cls[E], vm_omega[E],
//                        cut into chunks {vertex, begin, end} of at most VDO_CHUNK edges
//   (chunked layout only) vertex-major ternary stream (sorted by motion vertex): hm_p1[Et] (landmark index of p1; p2 = p1 + 1), hm_cls, hm_omega,
//                        chunks likewise
//   se3-se3 edges (prior: j = -1): se_i, se_j, se_Z[*12], se_w, se_delta, se_Hoff[*36] (J_i^T W J_j, written by linearise)
//   adjacency for H_pp * v: nbr_begin[C+1], nbr_edge[], nbr_other[], nbr_tr[] (1: use block transposed)
//   system: Hpp[C*36] (diagonal blocks, full row-major), bp[C*6], hll[P] (H_ll diagonal blocks are hll*I3), bl[P*3],
//           pt_s[P] (Schur pivots of the per-tracklet tridiagonal for the current lambda), pt_g[P], tk_gamma[P]
//           (diagonal / coupling scalars of Hll^-1 for the preconditioner), Minv[C*36]
//   edge classes: (information weight, Huber delta) pairs; at most 256 distinct pairs per edge family
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define VDO_CHUNK 512
// Tiled layout (default): the landmark side is cut into tiles of whole tracklets, at most VDO_TILE_L landmarks and
// VDO_TILE_E EdgeSE3PointXYZ per tile.  One CTA owns one tile: landmark blocks are staged in shared memory, the
// landmark-side sums are formed there, and the se3-vertex-side sums are formed by walking the tile's edges in
// vertex-sorted order (ob_perm / tr_perm) in warp-sized segments of one vertex each -- one reduction + a handful of
// atomics per segment.  Edges are therefore stored ONCE (landmark-major); the vertex-major copies of the chunked
// layout do not exist in this mode.
#define VDO_TILE_L 256
#define VDO_TILE_E 768
#define VDO_PCR_SHORT 32    // paths up to this many vertices: one CTA (one (vertex, row) item per thread); longer: a cluster of PCR_CL CTAs
#define VDO_SEG 64
#define VDO_SEG2 15   // Schur kernels: runs of one vertex cut at 15 entries (odd: threads walking consecutive full runs hit distinct shared-memory banks), one thread per (run, component pair)

namespace vdo {

struct Chunk { int v, begin, end, pad; };
// tile: landmarks [k0,k1), EdgeSE3PointXYZ [e0,e1) (landmark-major), tracklets [t0,t1), vertex-sorted segments of the
// pointxyz edges [os0,os1) and of the ternary edges [ts0,ts1)
// [qo0,qo1) / [qt0,qt1): the same vertex-sorted runs cut at VDO_SEG2 entries (osegs2 / tsegs2)
// [vs0, vs0 + ncam + nmot): the tile's own list of se3 vertices in tile_verts -- the cameras its pointxyz edges meet first, then the
// motion vertices of its ternary edges; edges carry the 8-bit position in that list (lm_cslot / tk_hslot)
struct Tile { int k0, k1, e0, e1, t0, t1, os0, os1, ts0, ts1, qo0, qo1, qt0, qt1, vs0, nv; };   // nv = ncam | nmot << 16
// segment: <= VDO_SEG consecutive entries of ob_perm (or tr_perm) starting at `begin`, all on se3 vertex v (one warp, two entries per lane)
struct Seg { int v, begin, n, pad; };

struct BaDev {
  int own = 1;     // 1 on the rank that accumulates the se3-se3 edges / se3 parts of scalar sums (rank 0), 0 elsewhere
  int Tstat = 0;   // tracklets [0, Tstat) are static landmarks (tracklet t == landmark t); [Tstat, T) are chains
  int C = 0, P = 0, T = 0, Eobs = 0, Eter = 0, Ese = 0, n_obs_chunks = 0, n_ter_chunks = 0, n_nbr = 0;
  double *se3 = 0, *pt = 0, *se3_bk = 0, *pt_bk = 0, *se3_init = 0, *pt_init = 0;
  int* tk_begin = 0;
  int* lm_obs_begin = 0; int* lm_cam = 0; double* lm_z = 0; uint8_t* lm_cls = 0; double* lm_omega = 0;
  int* tk_h = 0; uint8_t* tk_cls = 0; double* tk_omega = 0;
  int* vm_pt = 0; double* vm_z = 0; uint8_t* vm_cls = 0; double* vm_omega = 0; Chunk* obs_chunks = 0;
  int* hm_p1 = 0; uint8_t* hm_cls = 0; double* hm_omega = 0; Chunk* ter_chunks = 0;
  int *se_i = 0, *se_j = 0; double *se_Z = 0, *se_w = 0, *se_delta = 0, *se_Hoff = 0;
  int *nbr_begin = 0, *nbr_edge = 0, *nbr_other = 0; uint8_t* nbr_tr = 0;
  double *Hpp = 0, *bp = 0, *hll = 0, *bl = 0, *pt_s = 0, *Minv = 0;
  double *pt_g = 0, *tk_gamma = 0;
  // chain preconditioner (block-tridiagonal along the paths of the se3-se3 edge graph, factored by cyclic reduction; sizes of the
  // pcr_* arrays: BaBackend::precond_blocks)
  int n_paths = 0;
  int* path_begin = 0;            // n_paths+1 ; se3 vertices are renumbered so that each path is a contiguous index range
  int* path_of = 0;               // C : path id of each vertex
  int* pcr_edge = 0; uint8_t* pcr_tr = 0;   // C : se3-se3 edge linking vertex v-1 and v (or -1), and whether M(v, v-1) = Hoff^T
  double *pcr_D = 0, *pcr_L = 0, *pcr_Dinv = 0;   // level matrices D and L of the reduction, C*36 inverses Dinv
  double *pcr_A = 0, *pcr_G = 0;  // elimination operators
  double *pcr_b = 0;              // scratch vector(s) of the solve   // per landmark: diagonal scalar of Hll^-1; per ternary edge: g_k + g_k+1 - 2 g_k,k+1
  double *xp = 0, *r = 0, *z = 0, *p = 0, *Ap = 0, *rhs = 0; // 6C each
  // banded static block of the reduced matrix (see k_band_mul): for rows [band_v0, band_v0 + band_n) of se3 vertices and offsets 0..band_W-1,
  // the 10 moments sum_l (om_la om_lb / s_l) [1, p_l, p_l p_l^T] over the static landmarks seen by both; re-formed per trial (s_l holds lambda)
  double* band = 0; int band_W = 0, band_v0 = 0, band_n = 0;
  double* Sdense = 0;       // (6C)^2 + 6C + 8: dense reduced matrix, right-hand side and status of the dense path (only allocated for small static-only graphs)
  double* p2 = 0;           // 6C: second buffer of the search direction (the fused PCG kernels write p_{k+1} = z + beta p_k out of place)
  unsigned int* ticket = 0; // "last CTA done" counters of the fused PCG step ([0]) and of the peer exchange ([1])
  // ---- multi-GPU exchange of the sharded PCG iteration (CUDA backend, peer memory over NVLink; see k_xchg_scatter / k_xchg_reduce) ----
  int xg_rank = 0, xg_world = 1;
  double** xg_slots = 0;             // device array [world]: base of every rank's slot buffer (2 parities x world senders x 6C doubles)
  unsigned long long** xg_flags = 0; // device array [world]: every rank's flag array (world entries: epoch of the last vector received from each sender)
  unsigned long long* xg_epoch = 0;  // local epoch counter (second exchange: flags at +320, epoch at +192 entries)
  // Path sharding of the preconditioner (only with the peer exchange): rank r factors and solves the paths p with p % world == r, stores
  // its part of z = M^-1 r and its partial sums of r.z straight into every rank's copy (d.z / d.part_rz then live in the exchange buffer)
  int xg_paths = 0;
  size_t xg_off_z = 0, xg_off_prz = 0;   // offsets (doubles, from a rank's slot base) of its z vector and its part_rz array
  int* own_paths = 0; int n_own_paths = 0;   // the paths this rank factors / solves (all of them unless xg_paths), the LONG ones first
  int n_own_long = 0;                        // ... of which this many have more than VDO_PCR_SHORT vertices (solved by a cluster of CTAs; the rest by one CTA each)
  double *zl = 0, *xl = 0;                                    // 3P each
  double *vw = 0;   // 6C: per-vertex world-frame image [gamma, beta] of the vector the landmark pass multiplies (see body_vertex_transform)
  double *obs_cls_w = 0, *obs_cls_d = 0, *ter_cls_w = 0, *ter_cls_d = 0;  // 256 each
  // ---- tiled layout ----
  int tiled = 0, n_tiles_stat = 0, n_tiles = 0, n_osegs = 0, n_tsegs = 0;
  int capE_st = 16, capE_ch = 16;   // largest pointxyz-edge count of a static / chain tile, rounded up to 16 (shared-memory capacity of the launches)
  Tile* tiles = 0; Seg* osegs = 0; Seg* tsegs = 0; Seg* osegs2 = 0; Seg* tsegs2 = 0;
  uint32_t* ob_ps = 0;     // Eobs: per position q of the camera-sorted order: ob_perm[q] | lm_lml[e0 + ob_perm[q]] << 16 (one load instead of two)
  int* tile_verts = 0;     // per tile [vs0, vs0 + ncam + nmot): se3 vertices the tile meets (cameras, then motion vertices)
  uint8_t* lm_cslot = 0;   // Eobs: position of the edge's camera in its tile's vertex list
  uint8_t* tk_hslot = 0;   // P: position (counted from the tile's first motion vertex) of the motion vertex of ternary edge (k, k+1); 255 = no edge
  int capV_st = 1, capV_ch = 1, capH_ch = 1;   // largest camera / motion-vertex list of a static / chain tile
  uint16_t* ob_perm = 0;   // Eobs: position in the tile's camera-sorted order -> tile-local edge index (e - e0)
  uint16_t* tr_perm = 0;   // P: position (k0 + i) in the tile's motion-vertex-sorted order -> tile-local landmark index of p1
  uint8_t* lm_lml = 0;     // Eobs: tile-local landmark index of each pointxyz edge
  double* pt_Q = 0;        // 9 per chain landmark (index k - Tstat): Q_k = (R_{k-1} ... R_{kb})^T, rotates landmark k into the
                           // frame in which its tracklet's H_ll is (scalar tridiagonal) (x) I3
  double *accO = 0, *accT = 0;   // 16 per se3 vertex: world-frame sums of the pointxyz / ternary edges (see tile_acc16)
  double* acc6 = 0;        // 12 per se3 vertex: world-frame Hpl*z sums of one Schur product.  CUDA backend: [F_o, M_o, F_t, M_t] = force and
                           // torque ABOUT THE WORLD ORIGIN of the pointxyz / ternary edges (k_tile_schur2; the finalize kernel moves the
                           // torque to the vertex origin).  Emulation: the first 6 hold [force, torque about the vertex origin].
  double* vh = 0;          // 6C: per-vertex world-frame image of v as seen by ternary edges (vw is the pointxyz one)
  double* scal = 0;  // device scalars, see SC_* below
  double *part_pap = 0, *part_rz = 0;   // per-CTA partial sums of p.Ap (<= 148) and r.z (n_paths * 8): summed in a FIXED order so that
                                        // every rank of a sharded solve computes bit-identical PCG scalars (and convergence flags)
  int n_part_pap = 0, n_part_rz = 0;
};

// SC_DENSE: copy of the dense path's status word of the last solve (!= 0: the reduced matrix was not positive definite), read back
// with the other scalars of a trial
enum { SC_CHI2 = 0, SC_SCALE = 1, SC_MAXDIAG = 2, SC_PAP = 3, SC_RZ = 4, SC_RZ_NEW = 5, SC_RZ0 = 6, SC_DONE = 7, SC_ITERS = 8, SC_BAD = 9,
       SC_LAMBDA = 10, SC_TOL2 = 11, SC_BETA = 12, SC_DENSE = 13, SC_N = 16 };

// Grow-only host staging arena (pinned memory in the CUDA backend): graph ingestion builds every stream it uploads directly
// in it, so host->device copies run at PCIe speed without a bounce buffer and repeated graphs pay no page faults.  Memory
// is handed out until the last user releases the arena; then it is rewound (and coalesced into one block).
struct HostArena {
  struct Block { char* p; size_t cap, used; };
  std::vector<Block> blocks;
  int users = 0;
  virtual ~HostArena() {}
  virtual char* raw_alloc(size_t bytes) = 0;
  virtual void raw_free(char* p) = 0;
  void* take(size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    for (Block& b : blocks) if (b.cap - b.used >= bytes) { void* r = b.p + b.used; b.used += bytes; return r; }
    const size_t cap = bytes > ((size_t)64 << 20) ? bytes : ((size_t)64 << 20);
    if (std::getenv("VDO_ARENA_TRACE")) std::fprintf(stderr, "[vdo_b200] staging arena: new block of %zu MB for a request of %zu bytes (%zu blocks, users %d)\n", cap >> 20, bytes, blocks.size(), users);
    Block nb{raw_alloc(cap), cap, bytes};
    blocks.push_back(nb);
    return nb.p;
  }
  void acquire() { ++users; }
  void release() {
    if (--users > 0) return;
    users = 0;
    if (blocks.size() > 1) {
      size_t total = 0;
      for (Block& b : blocks) { total += b.cap; raw_free(b.p); }
      blocks.clear();
      blocks.push_back(Block{raw_alloc(total), total, 0});
    }
    for (Block& b : blocks) b.used = 0;
  }
  void destroy() { for (Block& b : blocks) raw_free(b.p); blocks.clear(); }
};

// The backend: memory + one function per kernel.  Implemented for CUDA in ba_kernels.cu (the product) and, for the
// CPU-only host-logic tests, as serial loops over the same per-thread bodies in tests/emul/ba_backend_emul.cpp.
struct BaBackend {
  virtual ~BaBackend() {}
  // multi-GPU: landmark-sharded graphs sum their partial se3-side quantities across ranks (NCCL in the CUDA backend)
  int rank = 0, world = 1;
  virtual void allreduce_sum(double* buf, size_t n) { (void)buf; (void)n; }
  virtual void allreduce_max(double* buf, size_t n) { (void)buf; (void)n; }
  virtual void* alloc(size_t bytes) = 0;            // zero-initialised
  virtual void free_(void* p) = 0;
  virtual void h2d(void* dst, const void* src, size_t bytes) = 0;
  virtual void h2d_async(void* dst, const void* src, size_t bytes) { h2d(dst, src, bytes); }   // src in staging memory; ordered on the stream
  virtual HostArena& staging() = 0;
  virtual void d2h(void* dst, const void* src, size_t bytes) = 0;   // synchronises the stream first
  // out[k * len + i] = src[k][i] for k < n, i < len: the scalars of several graphs with ONE synchronise.  n == 1 is a plain d2h.
  virtual void read_scalars(const double* const* src, int n, int len, double* out) {
    for (int k = 0; k < n; ++k) d2h(out + (size_t)k * len, src[k], sizeof(double) * (size_t)len);
  }
  virtual void d2d(void* dst, const void* src, size_t bytes) = 0;
  virtual void zero(void* dst, size_t bytes) = 0;
  virtual void sync() = 0;
  virtual int launches() const = 0;
  virtual void* stream() const = 0;
  virtual void timer_start(int slot) = 0;
  virtual float timer_stop_ms(int slot) = 0;        // synchronises

  // --- linearisation (buildSystem) ---
  // landmark side: robust chi2 of all EdgeSE3PointXYZ + ternary edges into scal[SC_CHI2]; if write: lm_omega, tk_omega, hll, bl
  virtual void lin_tracklets(BaDev& d, bool write) = 0;
  // se3 side of EdgeSE3PointXYZ / ternary edges: Hpp += , bp += , vm_omega / hm_omega
  virtual void lin_vertex_obs(BaDev& d) = 0;
  virtual void lin_vertex_ter(BaDev& d) = 0;
  // EdgeSE3 + EdgeSE3Prior: chi2 into scal[SC_CHI2]; if write: Hpp, bp, se_Hoff
  virtual void lin_se3_edges(BaDev& d, bool write) = 0;
  // scal[SC_MAXDIAG] = max |diagonal of H|
  virtual void max_diagonal(BaDev& d) = 0;
  // --- per-trial factorisation ---
  virtual void factor_landmarks(BaDev& d, double lambda) = 0;   // pt_s
  // Preconditioner M = Hpp(se3-se3 edges, incl. off-diagonal blocks) + lambda I + blockdiag(Hpp_landmark - Hpl Hll^-1 Hlp), the landmark
  // term summed edge by edge (exact when a vertex meets every tracklet through at most one edge; DESIGN.md section 2):
  //   precond_begin: Minv = Hpp_vv + lambda I ; precond_vertex_*: Minv -= diagonal blocks of Hpl Hll^-1 Hlp ;
  //   precond_factor: cyclic-reduction factorisation of the block-tridiagonal M along each path (pcr_*);
  //   scal[SC_BAD] counts blocks that were not SPD.
  // precond_blocks: blocks of 36 doubles of pcr_D and of pcr_L (nDL) and of pcr_A and of pcr_G (nAG), and 6-vectors of pcr_b (nb), for C
  // vertices on paths of at most max_len vertices.  The default is the layout of the per-level parallel cyclic reduction of the body_pcr_*
  // bodies: D, L and b double buffered, the operators of every vertex at every level.
  virtual void precond_blocks(int C, int max_len, size_t& nDL, size_t& nAG, size_t& nb) const {
    int nl = 1;
    while ((1 << nl) < max_len) ++nl;
    nDL = 2 * (size_t)C; nAG = (size_t)C * nl; nb = 2 * (size_t)C;
  }
  virtual void precond_begin(BaDev& d, double lambda) = 0;
  virtual void precond_vertex_obs(BaDev& d) = 0;
  virtual void precond_vertex_ter(BaDev& d) = 0;
  virtual void precond_factor(BaDev& d, double lambda) = 0;
  // --- Schur products ---
  // mode 0: zl = Hll^-1 bl ; mode 1: zl = Hll^-1 (Hlp v) ; mode 2: xl = Hll^-1 (bl - Hlp v).  Modes 1/2 read v through d.vw
  // (vertex_transform / hpp_mul must have run on v) and, for ternary edges, v itself.
  virtual void schur_landmarks(BaDev& d, int mode, const double* v) = 0;
  // measurement only: part 0 = static landmarks, part 1 = chains
  virtual void schur_landmarks_part(BaDev& d, int mode, const double* v, int part) { (void)part; schur_landmarks(d, mode, v); }
  virtual void lin_tracklets_part(BaDev& d, bool write, int part) { (void)part; lin_tracklets(d, write); }
  // out[vertex] += sign * sum_edges Hpl_e * zl[landmark(e)]
  virtual void schur_vertex_obs(BaDev& d, double sign, double* out) = 0;
  virtual void schur_vertex_ter(BaDev& d, double sign, double* out) = 0;
  // vw = world-frame image of v (needed by schur_landmarks modes 1 and 2)
  virtual void vertex_transform(BaDev& d, const double* v) = 0;
  // out = (Hpp + lambda I) v  (diagonal blocks and se3-se3 off-diagonal blocks); also performs vertex_transform(v)
  virtual void hpp_mul(BaDev& d, double lambda, const double* v, double* out) = 0;
  // --- PCG vector steps (device-side scalars; no host sync) ---
  virtual void pcg_init(BaDev& d) = 0;     // r = rhs (x = 0), z = Minv r, p = z, rz = r.z, rz0 = rz, done = 0, iters = 0
  virtual void pcg_dot_pAp(BaDev& d) = 0;  // scal[SC_PAP] = p.Ap
  virtual void pcg_step(BaDev& d, double tol2) = 0;  // alpha, x, r, z, rz_new, beta, p; done=1 if rz_new <= tol2 * rz0, done=2 on breakdown
  // n PCG iterations (S*p, p.Ap, x/r/z update, beta, p update) without host involvement.  The default composes the
  // primitives above; the CUDA backend replays a captured CUDA graph.
  virtual void pcg_iterate(BaDev& d, double lambda, double tol2, int n) {
    for (int b = 0; b < n; ++b) {
      hpp_mul(d, lambda, d.p, d.Ap);
      schur_landmarks(d, 1, d.p);
      schur_vertex_obs(d, -1.0, d.Ap);
      schur_vertex_ter(d, -1.0, d.Ap);
      allreduce_sum(d.Ap, 6 * (size_t)d.C);
      pcg_dot_pAp(d);
      pcg_step(d, tol2);
    }
  }
  virtual void release(BaDev& d) { (void)d; }   // drop anything cached for this graph (called before its buffers are freed)
  // Dense reduced system (small static-only graphs, e.g. the 20-camera sliding window): S = Hpp + lambda I - Hpl Hll^-1 Hlp formed explicitly
  // (6C x 6C) and solved by a Cholesky factorisation whose trailing updates run on the fp64 tensor cores (mma.sync m8n8k4) -- the
  // BlockSolver Schur path of g2o/core/block_solver.hpp:352-486 instead of the matrix-free PCG.  dense_capacity(): largest 6C (0: unsupported);
  // dense_solve(): enqueues xp = S^-1 (bp - Hpl Hll^-1 bl) after factor_landmarks(lambda) and copies the status word (!= 0: S is not
  // positive definite) to scal[SC_DENSE] on the device: the caller reads it back with its other scalars.
  virtual int dense_capacity() const { return 0; }
  // widest supported band of the explicit static block (0: the backend has no band path); band_form(): fill d.band after factor_landmarks
  virtual int band_max_width() const { return 0; }
  virtual void band_form(BaDev& d) { (void)d; }
  virtual void dense_solve(BaDev& d, double lambda) { (void)d; (void)lambda; }
  // multi-GPU: may turn on path sharding of the preconditioner for this graph (collective; called once from finalize after d is complete).
  // Returns the list of paths this rank owns (default: every path).
  virtual bool shard_paths(BaDev& d) { (void)d; return false; }
  // --- update / acceptance ---
  virtual void apply_update(BaDev& d, double lambda, bool reorthogonalize) = 0;  // oplus; scal[SC_SCALE] = sum x (lambda x + b)

  // --- the steps of the LM rounds (BaGraph's linearisation and trial rounds), over the graphs of a call ---
  // batch_begin: every graph of the call, fixed until batch_end.  batch_set: per graph its step flags (BATCH_*), the lambda /
  // reorthogonalisation of its trial and the squared relative tolerance of its PCG.  Each *_batch step runs the single-graph step on the
  // graphs whose flags hold `bit`, with the single graph's partition and sums; the memsets and copies around the steps stay with the caller
  // (except inside the PCG-path forms, which replace whole blocks of a trial).  The defaults call the single-graph forms one graph after
  // another; the backend chooses which graphs share launches (the CUDA backend: launch tables for two or more graphs of a kind).
  // BATCH_TRIAL: every graph with a trial in this round; BATCH_DENSE: ... that is solved by the dense path; BATCH_PCG: ... whose PCG is
  // still iterating (cleared by the caller once the graph has converged or used its iterations).
  enum { BATCH_LIN = 1, BATCH_MAXDIAG = 2, BATCH_TRIAL = 4, BATCH_DENSE = 8, BATCH_PCG = 16 };
  virtual void batch_begin(BaDev* const* ds, int n) {
    bds_.assign(ds, ds + n); bflags_.assign(n, 0); blam_.assign(n, 0.0); brt_.assign(n, 0); btol2_.assign(n, 0.0);
  }
  virtual void batch_end() { bds_.clear(); }
  virtual void batch_set(const int* flags, const double* lambda, const int* reortho, const double* tol2) {
    for (size_t k = 0; k < bds_.size(); ++k) { bflags_[k] = flags[k]; blam_[k] = lambda[k]; brt_[k] = reortho[k]; btol2_[k] = tol2[k]; }
  }
  virtual void lin_tracklets_batch(int bit, bool write) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) lin_tracklets(*bds_[k], write); }
  virtual void lin_vertex_batch(int bit) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) { lin_vertex_obs(*bds_[k]); lin_vertex_ter(*bds_[k]); } }
  virtual void lin_se3_edges_batch(int bit, bool write) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) lin_se3_edges(*bds_[k], write); }
  virtual void max_diagonal_batch(int bit) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) max_diagonal(*bds_[k]); }
  virtual void factor_landmarks_batch(int bit) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) factor_landmarks(*bds_[k], blam_[k]); }
  virtual void dense_solve_batch(int bit) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) dense_solve(*bds_[k], blam_[k]); }
  virtual void back_substitute_batch(int bit) {   // vertex_transform(xp) + schur_landmarks(mode 2, xp)
    for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) { vertex_transform(*bds_[k], bds_[k]->xp); schur_landmarks(*bds_[k], 2, bds_[k]->xp); }
  }
  virtual void apply_update_batch(int bit) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) apply_update(*bds_[k], blam_[k], brt_[k] != 0); }
  // PCG-path trial, after factor_landmarks_batch:
  //   precondition_batch: SC_BAD = 0, precond_begin / _vertex_*, the all-reduce of Minv (sharded graphs), precond_factor, band_form
  //   schur_rhs_batch:    rhs = bp - Hpl Hll^-1 bl (each rank's part)
  //   pcg_init_batch:     pcg_init, with scal[SC_LAMBDA] / scal[SC_TOL2] = the trial's lambda and tol2
  //   pcg_iterate_batch:  n PCG iterations (pcg_iterate)
  virtual void precondition_batch(int bit) {
    for (size_t k = 0; k < bds_.size(); ++k) {
      if (!(bflags_[k] & bit)) continue;
      BaDev& d = *bds_[k];
      zero(d.scal + SC_BAD, sizeof(double));
      precond_begin(d, blam_[k]); precond_vertex_obs(d); precond_vertex_ter(d);
      allreduce_sum(d.Minv, 36 * (size_t)d.C);
      precond_factor(d, blam_[k]);
      if (d.band) band_form(d);
    }
  }
  virtual void schur_rhs_batch(int bit) {
    for (size_t k = 0; k < bds_.size(); ++k) {
      if (!(bflags_[k] & bit)) continue;
      BaDev& d = *bds_[k];
      schur_landmarks(d, 0, nullptr);
      if (d.own) d2d(d.rhs, d.bp, 48 * (size_t)d.C); else zero(d.rhs, 48 * (size_t)d.C);
      schur_vertex_obs(d, -1.0, d.rhs); schur_vertex_ter(d, -1.0, d.rhs);
    }
  }
  virtual void pcg_init_batch(int bit) { for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) pcg_init(*bds_[k]); }
  virtual void pcg_iterate_batch(int bit, int n) {
    for (size_t k = 0; k < bds_.size(); ++k) if (bflags_[k] & bit) pcg_iterate(*bds_[k], blam_[k], btol2_[k], n);
  }
 protected:
  std::vector<BaDev*> bds_;
  std::vector<int> bflags_, brt_;
  std::vector<double> blam_, btol2_;
};

// Product: CUDA implementation (ba_kernels.cu); returns nullptr and fills *err when no usable sm_90 device exists.
BaBackend* make_backend(int device, char* err, size_t errlen);

}  // namespace vdo
