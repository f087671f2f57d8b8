// g2o_io.cpp -- reader / writer of the reference's on-disk factor-graph format (SURVEY.md section 8(f) N2).
//
// The reference dumps every batch graph it optimises with g2o's text serialisation (src/Optimizer.cc:806,808,1934,1936 ->
// OptimizableGraph::save, g2o/core/optimizable_graph.cpp:589-622).  One element per line, "TAG fields...":
//   PARAMS_SE3OFFSET id  tx ty tz qx qy qz qw                         (parameter_se3_offset.cpp:48-64)
//   VERTEX_SE3:QUAT  id  tx ty tz qx qy qz qw                         (vertex_se3.cpp:49-64, toVectorQT)
//   VERTEX_TRACKXYZ  id  x y z                                        (vertex_pointxyz.cpp:39-53)
//   FIX id                                                            (optimizable_graph.cpp:835-837)
//   EDGE_SE3:QUAT      i j     tx ty tz qx qy qz qw  + 21 upper-triangle information entries   (edge_se3.cpp:43-75)
//   EDGE_SE3_PRIOR     i   pid tx ty tz qx qy qz qw  + 21                                      (edge_se3_prior.cpp:55-86)
//   EDGE_SE3_TRACKXYZ  c p pid x y z                 + 6                                       (edge_se3_pointxyz.cpp:63-96)
//   EDGE_SE3_MOTION    p1 p2 h x y z                 + 6                                       (types_dyn_slam3d.cpp:28-51)
// with the tags of g2o/types/types_slam3d.cpp:37-57; vertices are written in id order, edges in insertion order.  Robust
// kernels are NOT part of the format (g2o never serialises them), so the Huber deltas are arguments of the loader.
// Host code only: nothing here touches the device.  Numbers are written with 17 significant digits by default (loss-free
// round trip); precision 6 reproduces the reference's own files (default ostream precision).
#include <sys/stat.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/vdo_b200.h"
#include "ba_math.cuh"

struct vdo_g2o {
  // vertices in file order; compact indices (position in these arrays) are what the edge arrays use
  std::vector<int> se3_id, pt_id;
  std::vector<double> se3, pt;                 // 12 / 3 per vertex (iso layout of include/vdo_b200.h)
  std::vector<int> fixed_id;
  std::vector<int> prior_v; std::vector<double> prior_Z, prior_info;      // 12, 21 per edge
  std::vector<int> se3e_ij; std::vector<double> se3e_Z, se3e_info;       // 2, 12, 21
  std::vector<int> obs_cp; std::vector<double> obs_z, obs_info;          // 2, 3, 6
  std::vector<int> ter_pph; std::vector<double> ter_meas, ter_info;      // 3, 3, 6
  std::vector<double> offset;                  // PARAMS_SE3OFFSET entries: id, iso (13 per entry)
  std::string err;
};

namespace {
void qt_to_iso(const double* v7, double* iso, bool normalize) {
  double q[4] = {v7[3], v7[4], v7[5], v7[6]};
  if (normalize) {
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    if (n > 0) for (double& x : q) x /= n;
  }
  vdo::rot_from_quat(q, iso);
  iso[9] = v7[0]; iso[10] = v7[1]; iso[11] = v7[2];
}
void iso_to_qt(const double* iso, double* v7) {      // internal::toVectorQT: [t, q.x q.y q.z q.w]
  double q[4];
  vdo::quat_from_rot(iso, q);
  v7[0] = iso[9]; v7[1] = iso[10]; v7[2] = iso[11]; v7[3] = q[0]; v7[4] = q[1]; v7[5] = q[2]; v7[6] = q[3];
}
bool read_doubles(char*& p, int n, double* out) {
  for (int i = 0; i < n; ++i) {
    char* e = nullptr;
    out[i] = std::strtod(p, &e);
    if (e == p) return false;
    p = e;
  }
  return true;
}
bool read_ints(char*& p, int n, int* out) {
  for (int i = 0; i < n; ++i) {
    char* e = nullptr;
    long v = std::strtol(p, &e, 10);
    if (e == p) return false;
    out[i] = (int)v; p = e;
  }
  return true;
}
}  // namespace

extern "C" {

int vdo_g2o_read(const char* path, vdo_g2o** out) {
  if (!path || !out) return VDO_ERR_ARG;
  *out = nullptr;
  FILE* f = std::fopen(path, "rb");
  if (!f) return VDO_ERR_ARG;
  // only a regular file: some file systems open a directory and report its size as 0, which would read as an empty graph
  struct stat st;
  if (fstat(fileno(f), &st) != 0 || !S_ISREG(st.st_mode)) { std::fclose(f); return VDO_ERR_ARG; }
  std::fseek(f, 0, SEEK_END);
  const long sz = std::ftell(f);
  std::fseek(f, 0, SEEK_SET);
  if (sz < 0 || (unsigned long)sz > ((unsigned long)1 << 33)) { std::fclose(f); return VDO_ERR_ARG; }   // directory / pipe / absurd size
  std::vector<char> buf;
  try { buf.resize((size_t)sz + 1); } catch (...) { std::fclose(f); return VDO_ERR_ARG; }
  const size_t got = std::fread(buf.data(), 1, (size_t)sz, f);
  std::fclose(f);
  if (got != (size_t)sz) return VDO_ERR_ARG;                         // short read
  buf[got] = 0;
  vdo_g2o* g = new vdo_g2o;
  std::map<int, int> se3_of, pt_of;             // file id -> compact index
  struct Pending { int kind; int ids[3]; double v[28]; };
  std::vector<Pending> edges;                   // resolved after all vertices are known (g2o requires vertices first, we do not)
  char* line = buf.data();
  int lineno = 0;
  auto bad = [&](const char* what) { g->err = std::string(path) + ":" + std::to_string(lineno) + ": " + what; };
  while (*line) {
    char* nl = std::strchr(line, '\n');
    if (nl) *nl = 0;
    ++lineno;
    char* p = line;
    while (*p == ' ' || *p == '\t' || *p == '\r') ++p;
    char* tag = p;
    while (*p && *p != ' ' && *p != '\t' && *p != '\r') ++p;
    const std::string t(tag, p);
    bool ok = true;
    if (t.empty() || t[0] == '#') {
    } else if (t == "VERTEX_SE3:QUAT") {
      int id; double v[7], iso[12];
      ok = read_ints(p, 1, &id) && read_doubles(p, 7, v);
      if (ok) { qt_to_iso(v, iso, false); se3_of[id] = (int)g->se3_id.size(); g->se3_id.push_back(id); g->se3.insert(g->se3.end(), iso, iso + 12); }
    } else if (t == "VERTEX_TRACKXYZ") {
      int id; double v[3];
      ok = read_ints(p, 1, &id) && read_doubles(p, 3, v);
      if (ok) { pt_of[id] = (int)g->pt_id.size(); g->pt_id.push_back(id); g->pt.insert(g->pt.end(), v, v + 3); }
    } else if (t == "FIX") {
      int id; ok = read_ints(p, 1, &id);
      if (ok) g->fixed_id.push_back(id);
    } else if (t == "PARAMS_SE3OFFSET") {
      int id; double v[7], iso[12];
      ok = read_ints(p, 1, &id) && read_doubles(p, 7, v);
      if (ok) { qt_to_iso(v, iso, true); g->offset.push_back(id); g->offset.insert(g->offset.end(), iso, iso + 12); }
    } else if (t == "EDGE_SE3:QUAT") {
      Pending e; e.kind = 0;
      ok = read_ints(p, 2, e.ids) && read_doubles(p, 28, e.v);
      if (ok) edges.push_back(e);
    } else if (t == "EDGE_SE3_PRIOR") {
      Pending e; e.kind = 1; int pid;
      ok = read_ints(p, 1, e.ids) && read_ints(p, 1, &pid) && read_doubles(p, 28, e.v);
      if (ok) edges.push_back(e);
    } else if (t == "EDGE_SE3_TRACKXYZ") {
      Pending e; e.kind = 2; int pid;
      ok = read_ints(p, 2, e.ids) && read_ints(p, 1, &pid) && read_doubles(p, 9, e.v);
      if (ok) edges.push_back(e);
    } else if (t == "EDGE_SE3_MOTION") {
      Pending e; e.kind = 3;
      ok = read_ints(p, 3, e.ids) && read_doubles(p, 9, e.v);
      if (ok) edges.push_back(e);
    } else {
      bad(("unsupported tag " + t).c_str()); *out = g; return VDO_ERR_UNSUPPORTED;
    }
    if (!ok) { bad("malformed line"); *out = g; return VDO_ERR_ARG; }
    if (!nl) break;
    line = nl + 1;
  }
  auto look = [&](const std::map<int, int>& m, int id, int& idx) { auto it = m.find(id); if (it == m.end()) return false; idx = it->second; return true; };
  for (const Pending& e : edges) {
    double iso[12];
    int a, b, c;
    bool ok = true;
    if (e.kind == 0) {
      ok = look(se3_of, e.ids[0], a) && look(se3_of, e.ids[1], b);
      if (ok) { qt_to_iso(e.v, iso, true); g->se3e_ij.push_back(a); g->se3e_ij.push_back(b); g->se3e_Z.insert(g->se3e_Z.end(), iso, iso + 12); g->se3e_info.insert(g->se3e_info.end(), e.v + 7, e.v + 28); }
    } else if (e.kind == 1) {
      ok = look(se3_of, e.ids[0], a);
      if (ok) { qt_to_iso(e.v, iso, false); g->prior_v.push_back(a); g->prior_Z.insert(g->prior_Z.end(), iso, iso + 12); g->prior_info.insert(g->prior_info.end(), e.v + 7, e.v + 28); }
    } else if (e.kind == 2) {
      ok = look(se3_of, e.ids[0], a) && look(pt_of, e.ids[1], b);
      if (ok) { g->obs_cp.push_back(a); g->obs_cp.push_back(b); g->obs_z.insert(g->obs_z.end(), e.v, e.v + 3); g->obs_info.insert(g->obs_info.end(), e.v + 3, e.v + 9); }
    } else {
      ok = look(pt_of, e.ids[0], a) && look(pt_of, e.ids[1], b) && look(se3_of, e.ids[2], c);
      if (ok) { g->ter_pph.push_back(a); g->ter_pph.push_back(b); g->ter_pph.push_back(c); g->ter_meas.insert(g->ter_meas.end(), e.v, e.v + 3); g->ter_info.insert(g->ter_info.end(), e.v + 3, e.v + 9); }
    }
    if (!ok) { g->err = std::string(path) + ": edge refers to a vertex that is not in the file"; *out = g; return VDO_ERR_ARG; }
  }
  *out = g;
  return VDO_OK;
}

void vdo_g2o_free(vdo_g2o* g) { delete g; }
const char* vdo_g2o_error(const vdo_g2o* g) { return g ? g->err.c_str() : "null"; }

int vdo_g2o_counts(const vdo_g2o* g, int64_t out[8]) {
  if (!g || !out) return VDO_ERR_ARG;
  out[0] = (int64_t)g->se3_id.size(); out[1] = (int64_t)g->pt_id.size(); out[2] = (int64_t)g->prior_v.size(); out[3] = (int64_t)g->se3e_ij.size() / 2;
  out[4] = (int64_t)g->obs_cp.size() / 2; out[5] = (int64_t)g->ter_pph.size() / 3; out[6] = (int64_t)g->fixed_id.size(); out[7] = (int64_t)g->offset.size() / 13;
  return VDO_OK;
}
// copies one array out; name: se3_id pt_id fixed_id prior_v se3e_ij obs_cp ter_pph (int) | se3 pt prior_Z prior_info se3e_Z se3e_info obs_z
// obs_info ter_meas ter_info offset (double).  `cap` = capacity of dst in elements.
int vdo_g2o_get_i32(const vdo_g2o* g, const char* name, int* dst, int64_t cap) {
  if (!g || !name || !dst) return VDO_ERR_ARG;
  const std::string n(name);
  const std::vector<int>* v = n == "se3_id" ? &g->se3_id : n == "pt_id" ? &g->pt_id : n == "fixed_id" ? &g->fixed_id : n == "prior_v" ? &g->prior_v
                            : n == "se3e_ij" ? &g->se3e_ij : n == "obs_cp" ? &g->obs_cp : n == "ter_pph" ? &g->ter_pph : nullptr;
  if (!v || (int64_t)v->size() > cap) return VDO_ERR_ARG;
  if (!v->empty()) std::memcpy(dst, v->data(), v->size() * sizeof(int));
  return VDO_OK;
}
int vdo_g2o_get_f64(const vdo_g2o* g, const char* name, double* dst, int64_t cap) {
  if (!g || !name || !dst) return VDO_ERR_ARG;
  const std::string n(name);
  const std::vector<double>* v = n == "se3" ? &g->se3 : n == "pt" ? &g->pt : n == "prior_Z" ? &g->prior_Z : n == "prior_info" ? &g->prior_info
                               : n == "se3e_Z" ? &g->se3e_Z : n == "se3e_info" ? &g->se3e_info : n == "obs_z" ? &g->obs_z : n == "obs_info" ? &g->obs_info
                               : n == "ter_meas" ? &g->ter_meas : n == "ter_info" ? &g->ter_info : n == "offset" ? &g->offset : nullptr;
  if (!v || (int64_t)v->size() > cap) return VDO_ERR_ARG;
  if (!v->empty()) std::memcpy(dst, v->data(), v->size() * sizeof(double));
  return VDO_OK;
}

// Builds a vdo_graph from a parsed file.  The batch solver covers exactly the family the reference constructs: scalar
// information w * I on every edge, zero landmark-motion measurement, identity sensor offset -- anything else is
// VDO_ERR_UNSUPPORTED (never approximated).  delta_*: Huber deltas of the three robustified edge families (<= 0: none), as
// src/Optimizer.cc sets them on the edges it creates (deltaHuberCamMot / deltaHuber3D / deltaHuberObjMot = 1e-4, :1352; :213).
int vdo_graph_from_g2o(vdo_ctx* ctx, const vdo_g2o* f, double delta_se3, double delta_pointxyz, double delta_motion, vdo_graph** out) {
  if (!ctx || !f || !out) return VDO_ERR_ARG;
  *out = nullptr;
  auto scalar21 = [](const double* u, double& w) {      // upper triangle of a 6x6: w on the diagonal, 0 elsewhere
    w = u[0];
    int k = 0;
    for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j, ++k) if (std::fabs(u[k] - (i == j ? w : 0.0)) > 1e-12 * std::fabs(w)) return false;
    return true;
  };
  auto scalar6 = [](const double* u, double& w) {
    w = u[0];
    int k = 0;
    for (int i = 0; i < 3; ++i) for (int j = i; j < 3; ++j, ++k) if (std::fabs(u[k] - (i == j ? w : 0.0)) > 1e-12 * std::fabs(w)) return false;
    return true;
  };
  for (size_t o = 0; o < f->offset.size(); o += 13) {
    const double* T = &f->offset[o + 1];
    const double I[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
    for (int i = 0; i < 12; ++i) if (std::fabs(T[i] - I[i]) > 1e-12) return VDO_ERR_UNSUPPORTED;
  }
  const int np = (int)f->prior_v.size(), ns = (int)f->se3e_ij.size() / 2, no = (int)f->obs_cp.size() / 2, nt = (int)f->ter_pph.size() / 3;
  std::vector<double> wp(np), ws(ns), wo(no), wt(nt), ds(ns, delta_se3), dob(no, delta_pointxyz), dt(nt, delta_motion);
  for (int e = 0; e < np; ++e) if (!scalar21(&f->prior_info[21 * (size_t)e], wp[e])) return VDO_ERR_UNSUPPORTED;
  for (int e = 0; e < ns; ++e) if (!scalar21(&f->se3e_info[21 * (size_t)e], ws[e])) return VDO_ERR_UNSUPPORTED;
  for (int e = 0; e < no; ++e) if (!scalar6(&f->obs_info[6 * (size_t)e], wo[e])) return VDO_ERR_UNSUPPORTED;
  for (int e = 0; e < nt; ++e) {
    if (!scalar6(&f->ter_info[6 * (size_t)e], wt[e])) return VDO_ERR_UNSUPPORTED;
    for (int i = 0; i < 3; ++i) if (f->ter_meas[3 * (size_t)e + i] != 0.0) return VDO_ERR_UNSUPPORTED;
  }
  vdo_graph* g = nullptr;
  int rc = vdo_graph_create(ctx, &g);
  if (rc != VDO_OK) return rc;
  rc = vdo_graph_set_vertices(g, (int)f->se3_id.size(), f->se3.data(), (int)f->pt_id.size(), f->pt.data());
  if (rc == VDO_OK && np) rc = vdo_graph_add_edges_se3_prior(g, np, f->prior_v.data(), f->prior_Z.data(), wp.data());
  if (rc == VDO_OK && ns) rc = vdo_graph_add_edges_se3(g, ns, f->se3e_ij.data(), f->se3e_Z.data(), ws.data(), ds.data());
  if (rc == VDO_OK && no) rc = vdo_graph_add_edges_se3_pointxyz(g, no, f->obs_cp.data(), f->obs_z.data(), wo.data(), dob.data());
  if (rc == VDO_OK && nt) rc = vdo_graph_add_edges_landmark_motion(g, nt, f->ter_pph.data(), wt.data(), dt.data());
  if (rc == VDO_OK) rc = vdo_graph_finalize(g);
  if (rc != VDO_OK) { vdo_graph_destroy(g); return rc; }
  *out = g;
  return VDO_OK;
}

// Writes a graph in the arrays' layout of vdo_graph_add_* (scalar information per edge).  se3_id / pt_id: file ids of the
// vertices (NULL: se3 vertex i gets id i, point j gets id n_se3 + j).  Vertices are written in id order like
// OptimizableGraph::save, edges in the order prior, se3, pointxyz, motion.  precision: significant digits (<= 0: 17).
int vdo_g2o_write(const char* path, int n_se3, const double* se3, const int* se3_id, int n_pt, const double* pt, const int* pt_id, int n_fixed,
                  const int* fixed_id, int n_prior, const int* prior_v, const double* prior_Z, const double* prior_w, int n_se3e, const int* se3e_ij,
                  const double* se3e_Z, const double* se3e_w, int n_obs, const int* obs_cp, const double* obs_z, const double* obs_w, int n_ter,
                  const int* ter_pph, const double* ter_w, int precision) {
  if (!path) return VDO_ERR_ARG;
  FILE* f = std::fopen(path, "wb");
  if (!f) return VDO_ERR_ARG;
  const int prec = precision > 0 ? precision : 17;
  auto num = [&](double v) { std::fprintf(f, "%.*g ", prec, v); };
  auto sid = [&](int i) { return se3_id ? se3_id[i] : i; };
  auto pid = [&](int j) { return pt_id ? pt_id[j] : n_se3 + j; };
  std::fprintf(f, "PARAMS_SE3OFFSET 0 0 0 0 0 0 0 1 \n");
  std::map<int, std::pair<int, int>> order;      // file id -> (kind, compact index)
  for (int i = 0; i < n_se3; ++i) order[sid(i)] = {0, i};
  for (int j = 0; j < n_pt; ++j) order[pid(j)] = {1, j};
  std::map<int, bool> fixed;
  for (int i = 0; i < n_fixed; ++i) fixed[fixed_id[i]] = true;
  for (const auto& kv : order) {
    if (kv.second.first == 0) {
      double v[7]; iso_to_qt(se3 + 12 * (size_t)kv.second.second, v);
      std::fprintf(f, "VERTEX_SE3:QUAT %d ", kv.first);
      for (double x : v) num(x);
    } else {
      std::fprintf(f, "VERTEX_TRACKXYZ %d ", kv.first);
      for (int i = 0; i < 3; ++i) num(pt[3 * (size_t)kv.second.second + i]);
    }
    std::fprintf(f, "\n");
    if (fixed.count(kv.first)) std::fprintf(f, "FIX %d\n", kv.first);
  }
  auto info = [&](int dim, double w) { for (int i = 0; i < dim; ++i) for (int j = i; j < dim; ++j) num(i == j ? w : 0.0); };
  for (int e = 0; e < n_prior; ++e) {
    double v[7]; iso_to_qt(prior_Z + 12 * (size_t)e, v);
    std::fprintf(f, "EDGE_SE3_PRIOR %d 0 ", sid(prior_v[e]));
    for (double x : v) num(x);
    info(6, prior_w[e]); std::fprintf(f, "\n");
  }
  for (int e = 0; e < n_se3e; ++e) {
    double v[7]; iso_to_qt(se3e_Z + 12 * (size_t)e, v);
    std::fprintf(f, "EDGE_SE3:QUAT %d %d ", sid(se3e_ij[2 * e]), sid(se3e_ij[2 * e + 1]));
    for (double x : v) num(x);
    info(6, se3e_w[e]); std::fprintf(f, "\n");
  }
  for (int e = 0; e < n_obs; ++e) {
    std::fprintf(f, "EDGE_SE3_TRACKXYZ %d %d 0 ", sid(obs_cp[2 * e]), pid(obs_cp[2 * e + 1]));
    for (int i = 0; i < 3; ++i) num(obs_z[3 * (size_t)e + i]);
    info(3, obs_w[e]); std::fprintf(f, "\n");
  }
  for (int e = 0; e < n_ter; ++e) {
    std::fprintf(f, "EDGE_SE3_MOTION %d %d %d 0 0 0 ", pid(ter_pph[3 * e]), pid(ter_pph[3 * e + 1]), sid(ter_pph[3 * e + 2]));
    info(3, ter_w[e]); std::fprintf(f, "\n");
  }
  const bool ok = std::ferror(f) == 0;
  std::fclose(f);
  return ok ? VDO_OK : VDO_ERR_ARG;
}

}  // extern "C"
