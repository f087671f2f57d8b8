// tracker.cpp -- host side of the per-frame path: the sequencing of Tracking::GrabImageRGBD + Tracking::Track
// (src/Tracking.cc:164-648, 650-1212) over the device stages of this library.  It owns two resident frames (current / last),
// the per-frame vectors the reference keeps in `Frame` (include/Frame.h:110-196) and the slice of `Map` (include/Map.h:34-84)
// the batch optimisers read.  Everything numerical happens in the stages it calls (depth prep, ORB front end, static filter,
// object sampling, mask propagation, initial model, joint flow/pose LM, scene flow, object classification, renewal); the code
// here is control flow, index bookkeeping and 4x4 float algebra with cv::Mat rounding (float gemm = double accumulation,
// one rounding).  Ground-truth error metrics, drawing and file output of the reference are not part of the hot path.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/vdo_b200.h"
#include "dev_entry.h"
#include "frame_batch.h"

namespace {
using M4 = std::array<float, 16>;
M4 eye4() { M4 m{}; m[0] = m[5] = m[10] = m[15] = 1.f; return m; }
// cv::Mat A * B of two 4x4 CV_32F (e.g. `mCurrentFrame.mTcw * Converter::toInvMatrix(mLastFrame.mTcw)`, src/Tracking.cc:700-706):
// OpenCV's gemm takes its small-matrix branch (no flags, inner dimension <= 4) and evaluates a0*b0 + a1*b1 + a2*b2 + a3*b3 in
// FLOAT, left to right.  Pinned bit for bit against cv2.gemm (tests/test_results_io.py for the same formula in results_io.cpp;
// the oracle pipeline calls cv2.gemm itself, so the tracker parity tests pin this one).
M4 mul4(const M4& A, const M4& B) {
  M4 C{};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float s = A[4 * i] * B[j];
      s = s + A[4 * i + 1] * B[4 + j];
      s = s + A[4 * i + 2] * B[8 + j];
      s = s + A[4 * i + 3] * B[12 + j];
      C[4 * i + j] = s;
    }
  return C;
}
// Converter::toInvMatrix (src/Converter.cc:151-166): [R^T | -R^T t]
M4 inv4(const M4& T) {
  M4 I = eye4();
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) I[4 * i + j] = T[4 * j + i];
    double s = 0;
    for (int k = 0; k < 3; ++k) s += (double)T[4 * k + i] * (double)T[4 * k + 3];
    I[4 * i + 3] = (float)(-s);
  }
  return I;
}

struct FrameState {
  vdo_frame* img = nullptr;
  M4 Tcw = eye4();
  std::vector<float> keys;                                              // mvKeys (x, y)
  std::vector<float> statKeysTmp, corres, flowNext, statDepthTmp, stat3DTmp;   // mvStatKeysTmp, mvCorres, mvFlowNext, mvStatDepthTmp, mvStat3DPointTmp
  std::vector<float> statKeys, statDepth;                               // mvStatKeys, mvStatDepth
  std::vector<int> staInlierID;                                         // nStaInlierID
  std::vector<float> objKeys, objCorres, objFlowNext, objDepth, obj3D;  // mvObjKeys, mvObjCorres, mvObjFlowNext, mvObjDepth, mvObj3DPoint
  std::vector<int> semObjLabel, objLabel, dynInlierID;                  // vSemObjLabel, vObjLabel, nDynInlierID
  std::vector<float> flow3d;                                            // vFlow_3d
  std::vector<int> nModLabel, nSemPosition, semPosiGt;                  // nModLabel, nSemPosition, nSemPosi_gt
  std::vector<unsigned char> bObjStat;
  std::vector<M4> vObjMod;
  std::vector<float> vObjCentre3D;                                      // 3 per object (src/Tracking.cc:856-866)
  std::vector<std::vector<int>> vnObjID, vnObjInlierID;
  void clear_dynamic() {
    keys.clear(); statKeysTmp.clear(); corres.clear(); flowNext.clear(); statDepthTmp.clear(); stat3DTmp.clear(); statKeys.clear(); statDepth.clear();
    staInlierID.clear(); objKeys.clear(); objCorres.clear(); objFlowNext.clear(); objDepth.clear(); obj3D.clear(); semObjLabel.clear(); objLabel.clear();
    dynInlierID.clear(); flow3d.clear(); nModLabel.clear(); nSemPosition.clear(); semPosiGt.clear(); bObjStat.clear(); vObjMod.clear(); vObjCentre3D.clear(); vnObjID.clear();
    vnObjInlierID.clear();
  }
};

struct MapSlice {        // what Tracking::Track pushes per frame (src/Tracking.cc:1016-1070)
  std::vector<std::vector<float>> featSta, depSta, p3dSta, featDyn, depDyn, p3dDyn;
  std::vector<std::vector<int>> assoSta, assoDyn, featLabel, rmLabel, smLabel;
  std::vector<M4> cameraPose, cameraPose_RF;              // vmCameraPose (updated by the windowed BA) / vmCameraPose_RF (by the full batch)
  std::vector<std::vector<M4>> rigidMotion, rigidMotion_RF;
  std::vector<std::vector<float>> rigidCentre;            // vmRigidCentre: 3 floats per entry (entry 0 = camera = 0)
};
}  // namespace

struct vdo_tracker {
  vdo_ctx* ctx = nullptr;
  vdo_tracker_params p{};
  FrameState fr[2];
  int cur = 0;                 // index of the current frame; last = 1 - cur
  bool first = true;
  int f_id = 0, max_id = 1;
  bool has_velocity = false;
  M4 velocity = eye4();
  std::vector<float> tmpObjKeys, tmpObjDepth, tmpObjFlowNext, tmpObjCorres; std::vector<int> tmpSemObjLabel;   // mvTmp*
  std::vector<int> temperalMatch, temperalMatchSubset;
  MapSlice map;
  vdo::Tracklets* tracklets = nullptr;   // device tracklet tables of the map (map_graph.cu), extended with every frame pushed
  std::string err;
  double stage_ms[9] = {0};
  int frames = 0, local_ba_runs = 0, local_ba_iters = 0;
  // scratch
  std::vector<float> s_f[12]; std::vector<int> s_i[8]; std::vector<unsigned char> s_b[2]; std::vector<double> s_d[2];
};

namespace {
struct StageTimer {
  double* acc; std::chrono::steady_clock::time_point t0;
  explicit StageTimer(double* a) : acc(a), t0(std::chrono::steady_clock::now()) {}
  ~StageTimer() { *acc += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};
#define TK(call) do { int rc_ = (call); if (rc_ != VDO_OK) { t->err = std::string(#call) + " failed"; return rc_; } } while (0)
// The per-frame path runs in phases over a list of trackers (vdo_tracker_track / _dev are the list of one): a batched stage does the
// device work of every tracker of the list with one set of launches and one synchronise, and each tracker accumulates its wall time.
using Span = std::vector<vdo_tracker*>;
#define TB(call) do { int rc_ = (call); if (rc_ != VDO_OK) { for (vdo_tracker* t_ : ts) t_->err = std::string(#call) + " failed"; return rc_; } } while (0)
struct BatchTimer {
  const Span& ts; int k; std::chrono::steady_clock::time_point t0;
  BatchTimer(const Span& s, int stage) : ts(s), k(stage), t0(std::chrono::steady_clock::now()) {}
  ~BatchTimer() {
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    for (vdo_tracker* t : ts) t->stage_ms[k] += ms;
  }
};
FrameState& cur_of(vdo_tracker* t) { return t->fr[t->cur]; }
FrameState& last_of(vdo_tracker* t) { return t->fr[1 - t->cur]; }

void get3d_camera(float u, float v, float z, const vdo_tracker_params& p, float* X) {      // Optimizer::Get3DinCamera (src/Optimizer.cc:2995-3013)
  const float invfx = 1.0f / p.fx, invfy = 1.0f / p.fy;
  X[0] = (u - p.cx) * z * invfx; X[1] = (v - p.cy) * z * invfy; X[2] = z;
}
// Frame::UnprojectStereoStat / UnprojectStereoObject (src/Frame.cc:484-555): world point of a last-frame key
void unproject_world(float u, float v, float z, const vdo_tracker_params& p, const M4& Tcw, float* X) {
  const float invfx = 1.0f / p.fx, invfy = 1.0f / p.fy;
  const float x = (u - p.cx) * z * invfx, y = (v - p.cy) * z * invfy;
  for (int r = 0; r < 3; ++r) {
    const double twl = (double)(float)(-((double)Tcw[r] * (double)Tcw[3] + (double)Tcw[4 + r] * (double)Tcw[7] + (double)Tcw[8 + r] * (double)Tcw[11]));
    X[r] = (float)((double)Tcw[r] * (double)x + (double)Tcw[4 + r] * (double)y + (double)Tcw[8 + r] * (double)z + twl);
  }
}

// Frame::Frame (src/Frame.cc:61-260) of the current frame of every tracker: ORB keypoints, static candidates, semi-dense object samples.
// Each tracker keeps its own image size and ORB settings; geo[i]: tracker i's geometry on the extractor orb.
int build_frames(const Span& ts, const vdo::OrbJob& orb, const int* geo) {
  const int n = (int)ts.size();
  std::vector<vdo_frame*> fs(n);
  for (int i = 0; i < n; ++i) fs[i] = cur_of(ts[i]).img;
  std::vector<vdo::OrbXY> K(n);
  TB(vdo::orb_xy_batch(orb, fs.data(), geo, n, K.data()));
  std::vector<int> with, nk;                                              // Frame.cc:83-84: a frame without keypoints gets nothing else
  std::vector<vdo_frame*> fw; std::vector<const float*> kx, ky; std::vector<float> th_bg, th_obj;
  std::vector<long long> seed;                                            // option II: cv::RNG((uint32)(sample_seed + f_id)); -1: option I
  for (int i = 0; i < n; ++i) {
    FrameState& F = cur_of(ts[i]);
    const int max_kp = ts[i]->p.n_features * 2 + 4096;
    const int m = std::min((int)K[i].x.size(), max_kp);
    F.keys.resize(2 * (size_t)m);
    for (int k = 0; k < m; ++k) { F.keys[2 * k] = K[i].x[k]; F.keys[2 * k + 1] = K[i].y[k]; }
    if (m == 0) continue;
    with.push_back(i); nk.push_back(m); fw.push_back(fs[i]); kx.push_back(K[i].x.data()); ky.push_back(K[i].y.data());
    th_bg.push_back(ts[i]->p.th_depth_bg); th_obj.push_back(ts[i]->p.th_depth_obj);
    const vdo_tracker_params& p = ts[i]->p;
    seed.push_back(p.use_sample_feature ? (long long)(uint32_t)(p.sample_seed + (uint32_t)ts[i]->f_id) : -1);
  }
  const int nw = (int)with.size();
  if (nw == 0) return VDO_OK;
  std::vector<vdo::StaticKeys> S(nw);
  TB(vdo::filter_static_batch(fw.data(), nw, kx.data(), ky.data(), nk.data(), th_bg.data(), seed.data(), S.data()));
  const int step = 4;
  std::vector<int> cap(nw);                                               // every grid point of the frame
  for (int j = 0; j < nw; ++j) { const vdo_tracker_params& p = ts[with[j]]->p; cap[j] = ((p.width + step - 1) / step) * ((p.height + step - 1) / step); }
  std::vector<vdo::ObjSamples> O(nw);
  TB(vdo::sample_objects_batch(fw.data(), nw, th_obj.data(), step, cap.data(), O.data()));
  for (int j = 0; j < nw; ++j) {
    FrameState& F = cur_of(ts[with[j]]);
    const vdo::StaticKeys& st = S[j]; const vdo::ObjSamples& o = O[j];
    const std::vector<float>& sx = st.kx.empty() ? K[with[j]].x : st.kx; const std::vector<float>& sy = st.kx.empty() ? K[with[j]].y : st.ky;
    const int m = (int)st.idx.size();
    F.statKeysTmp.resize(2 * (size_t)m); F.corres.resize(2 * (size_t)m); F.flowNext.resize(2 * (size_t)m); F.statDepthTmp.resize(m);
    for (int i = 0; i < m; ++i) {
      F.statKeysTmp[2 * i] = sx[st.idx[i]]; F.statKeysTmp[2 * i + 1] = sy[st.idx[i]];
      F.corres[2 * i] = st.cx[i]; F.corres[2 * i + 1] = st.cy[i]; F.flowNext[2 * i] = st.fu[i]; F.flowNext[2 * i + 1] = st.fv[i];
      F.statDepthTmp[i] = st.depth[i] > 0 ? st.depth[i] : -1.f;
    }
    const int q = (int)o.x.size();
    F.objKeys.resize(2 * (size_t)q); F.objCorres.resize(2 * (size_t)q); F.objFlowNext.resize(2 * (size_t)q); F.objDepth.resize(q); F.semObjLabel.resize(q);
    for (int i = 0; i < q; ++i) {
      F.objKeys[2 * i] = (float)o.x[i]; F.objKeys[2 * i + 1] = (float)o.y[i]; F.objCorres[2 * i] = o.cx[i]; F.objCorres[2 * i + 1] = o.cy[i];
      F.objFlowNext[2 * i] = o.fx[i]; F.objFlowNext[2 * i + 1] = o.fy[i]; F.objDepth[i] = o.depth[i]; F.semObjLabel[i] = o.label[i];
    }
  }
  return VDO_OK;
}

// Optimizer::PoseOptimizationFlow2Cam / Flow2 host wrapper for a batch of problems, each indexing the LAST frame's arrays of its tracker.
// One vdo_pose_opt_flow2_batch launch per distinct quirk among the trackers (one in practice); problems are independent.
struct FlowJob { vdo_tracker* t; int mode; const std::vector<int>* idx; M4 T_init; };
int run_flow(const Span& ts, bool objects, const std::vector<FlowJob>& jobs, std::vector<M4>& T_out, std::vector<double>& flow_out,
             std::vector<unsigned char>& inlier, std::vector<int>& offs) {
  const int np = (int)jobs.size();
  offs.assign(np + 1, 0);
  for (int j = 0; j < np; ++j) offs[j + 1] = offs[j] + (int)jobs[j].idx->size();
  const int tot = offs[np];
  std::vector<float> pts(2 * (size_t)tot + 2), dep((size_t)tot + 1), flo(2 * (size_t)tot + 2);
  std::vector<int> mode(np); std::vector<float> Kc(4 * (size_t)np), Tl(16 * (size_t)np), Ti(16 * (size_t)np), To(16 * (size_t)np);
  for (int j = 0; j < np; ++j) {
    const vdo_tracker_params& p = jobs[j].t->p;
    const FrameState& L = last_of(jobs[j].t);
    const std::vector<float>& K = objects ? L.objKeys : L.statKeys; const std::vector<float>& D = objects ? L.objDepth : L.statDepth;
    const std::vector<float>& F = objects ? L.objFlowNext : L.flowNext;
    mode[j] = jobs[j].mode;
    const float k4[4] = {p.fx, p.fy, p.cx, p.cy};
    std::memcpy(&Kc[4 * j], k4, 16); std::memcpy(&Tl[16 * j], L.Tcw.data(), 64); std::memcpy(&Ti[16 * j], jobs[j].T_init.data(), 64);
    int q = offs[j];
    for (int id : *jobs[j].idx) { pts[2 * q] = K[2 * id]; pts[2 * q + 1] = K[2 * id + 1]; dep[q] = D[id]; flo[2 * q] = F[2 * id]; flo[2 * q + 1] = F[2 * id + 1]; ++q; }
  }
  flow_out.assign(2 * (size_t)tot + 2, 0.0); inlier.assign((size_t)tot + 1, 0);
  std::vector<double> stats(8 * (size_t)np, 0.0);
  std::vector<char> done(np, 0);
  for (int j0 = 0; j0 < np; ++j0) {
    if (done[j0]) continue;
    const int quirk = jobs[j0].t->p.quirk;
    std::vector<int> g;                                                   // the problems of this quirk, in job order
    for (int j = j0; j < np; ++j) if (!done[j] && jobs[j].t->p.quirk == quirk) { g.push_back(j); done[j] = 1; }
    if ((int)g.size() == np) {
      TB(vdo_pose_opt_flow2_batch(ts[0]->ctx, quirk, np, mode.data(), offs.data(), pts.data(), dep.data(), flo.data(), Kc.data(), Tl.data(), Ti.data(),
                                  To.data(), flow_out.data(), inlier.data(), stats.data()));
      break;
    }
    const int ng = (int)g.size();
    std::vector<int> gm(ng), go(ng + 1, 0);
    std::vector<float> gp, gd, gf, gK(4 * (size_t)ng), gTl(16 * (size_t)ng), gTi(16 * (size_t)ng), gTo(16 * (size_t)ng);
    for (int a = 0; a < ng; ++a) {
      const int j = g[a];
      gm[a] = mode[j]; go[a + 1] = go[a] + (offs[j + 1] - offs[j]);
      gp.insert(gp.end(), pts.begin() + 2 * (size_t)offs[j], pts.begin() + 2 * (size_t)offs[j + 1]);
      gd.insert(gd.end(), dep.begin() + offs[j], dep.begin() + offs[j + 1]);
      gf.insert(gf.end(), flo.begin() + 2 * (size_t)offs[j], flo.begin() + 2 * (size_t)offs[j + 1]);
      std::memcpy(&gK[4 * a], &Kc[4 * j], 16); std::memcpy(&gTl[16 * a], &Tl[16 * j], 64); std::memcpy(&gTi[16 * a], &Ti[16 * j], 64);
    }
    const int gt = go[ng];
    gp.resize(2 * (size_t)gt + 2); gd.resize((size_t)gt + 1); gf.resize(2 * (size_t)gt + 2);
    std::vector<double> gfo(2 * (size_t)gt + 2, 0.0), gst(8 * (size_t)ng, 0.0); std::vector<unsigned char> ginl((size_t)gt + 1, 0);
    TB(vdo_pose_opt_flow2_batch(ts[0]->ctx, quirk, ng, gm.data(), go.data(), gp.data(), gd.data(), gf.data(), gK.data(), gTl.data(), gTi.data(), gTo.data(),
                                gfo.data(), ginl.data(), gst.data()));
    for (int a = 0; a < ng; ++a) {
      const int j = g[a];
      std::memcpy(&To[16 * j], &gTo[16 * a], 64);
      for (int q = 0; q < offs[j + 1] - offs[j]; ++q) {
        flow_out[2 * (size_t)(offs[j] + q)] = gfo[2 * (size_t)(go[a] + q)]; flow_out[2 * (size_t)(offs[j] + q) + 1] = gfo[2 * (size_t)(go[a] + q) + 1];
        inlier[offs[j] + q] = ginl[go[a] + q];
      }
    }
  }
  T_out.resize(np);
  for (int j = 0; j < np; ++j) std::memcpy(T_out[j].data(), &To[16 * j], 64);
  return VDO_OK;
}

// Tracking::Track after the first frame (src/Tracking.cc:650-1003) for every tracker of the list: camera, scene flow, objects, renewal
int track_frames(const Span& ts) {
  const int n = (int)ts.size();
  // ---------------- camera (Tracking.cc:672-711) ----------------
  {   // GetInitModelCam (:1614-1715): one RANSAC problem per tracker
    BatchTimer timer(ts, 4);
    std::vector<int> offs(n + 1, 0);
    for (int i = 0; i < n; ++i) offs[i + 1] = offs[i] + (int)cur_of(ts[i]).statKeys.size() / 2;
    const int tot = offs[n];
    std::vector<float> obj3(3 * (size_t)tot + 3), img2(2 * (size_t)tot + 2), K4(4 * (size_t)n), Tmm(16 * (size_t)n), T0(16 * (size_t)n);
    std::vector<unsigned char> has(n, 1);
    std::vector<int> nsub(n), sub(tot + 1);
    for (int i = 0; i < n; ++i) {
      vdo_tracker* t = ts[i]; const vdo_tracker_params& p = t->p;
      FrameState& C = cur_of(t); const FrameState& L = last_of(t);
      const int Ns = offs[i + 1] - offs[i];
      t->temperalMatch.resize(Ns);
      for (int k = 0; k < Ns; ++k) t->temperalMatch[k] = k;
      for (int k = 0; k < Ns; ++k) {
        const int q = offs[i] + k;
        img2[2 * q] = C.statKeys[2 * k]; img2[2 * q + 1] = C.statKeys[2 * k + 1];
        unproject_world(L.statKeys[2 * k], L.statKeys[2 * k + 1], L.statDepth[k], p, L.Tcw, &obj3[3 * q]);
      }
      const M4 mm = t->has_velocity ? mul4(t->velocity, L.Tcw) : L.Tcw;
      std::memcpy(&Tmm[16 * i], mm.data(), 64);
      const float k4[4] = {p.fx, p.fy, p.cx, p.cy};
      std::memcpy(&K4[4 * i], k4, 16);
    }
    TB(vdo::init_model_batch(ts[0]->ctx, n, offs.data(), obj3.data(), img2.data(), K4.data(), 4, 500, 0.4, 0.98, Tmm.data(), has.data(), T0.data(), nsub.data(),
                             sub.data(), nullptr, nullptr, nullptr));
    for (int i = 0; i < n; ++i) {
      vdo_tracker* t = ts[i];
      t->temperalMatchSubset.assign(sub.begin() + offs[i], sub.begin() + offs[i] + nsub[i]);   // MatchId[i] == i
      std::memcpy(cur_of(t).Tcw.data(), &T0[16 * i], 64);
    }
  }
  {   // PoseOptimizationFlow2Cam (src/Optimizer.cc:2333-2542): one problem per tracker with at least 3 matches
    BatchTimer timer(ts, 5);
    std::vector<FlowJob> jobs;
    for (vdo_tracker* t : ts)
      if ((int)t->temperalMatchSubset.size() >= 3) jobs.push_back({t, 0, &t->temperalMatchSubset, cur_of(t).Tcw});
    if (!jobs.empty()) {
      std::vector<M4> To; std::vector<double> fo; std::vector<unsigned char> inl; std::vector<int> fo_offs;
      TB(run_flow(ts, false, jobs, To, fo, inl, fo_offs));
      for (size_t j = 0; j < jobs.size(); ++j) {
        vdo_tracker* t = jobs[j].t;
        FrameState& C = cur_of(t); const FrameState& L = last_of(t);
        C.Tcw = To[j];
        for (size_t i = 0; i < t->temperalMatchSubset.size(); ++i) {
          const int id = t->temperalMatchSubset[i]; const size_t g = (size_t)fo_offs[j] + i;
          if (inl[g]) {
            C.statKeys[2 * id] = (float)((double)L.statKeys[2 * id] + fo[2 * g]);
            C.statKeys[2 * id + 1] = (float)((double)L.statKeys[2 * id + 1] + fo[2 * g + 1]);
          } else t->temperalMatchSubset[i] = -1;
        }
      }
    }
  }
  for (vdo_tracker* t : ts) { t->velocity = mul4(cur_of(t).Tcw, inv4(last_of(t).Tcw)); t->has_velocity = true; }   // :700-706
  // ---------------- objects (:735-1003) ----------------
  {   // GetSceneFlowObj (:1278-1364): one launch over the object points of every tracker
    BatchTimer timer(ts, 6);
    std::vector<int> begin(n + 1, 0);
    for (int i = 0; i < n; ++i) { cur_of(ts[i]).flow3d.assign(cur_of(ts[i]).objKeys.size() / 2 * 3, 0.f); begin[i + 1] = begin[i] + (int)cur_of(ts[i]).objKeys.size() / 2; }
    const int tot = begin[n];
    if (tot > 0) {
      std::vector<float> up(tot), vp(tot), zp(tot), uc(tot), vc(tot), zc(tot), Tp(16 * (size_t)n), Tc(16 * (size_t)n), K4(4 * (size_t)n), f3(3 * (size_t)tot);
      std::vector<int> lp(tot), lc(tot); std::vector<unsigned char> valid(tot);
      for (int i = 0; i < n; ++i) {
        const vdo_tracker_params& p = ts[i]->p; const FrameState& C = cur_of(ts[i]); const FrameState& L = last_of(ts[i]);
        for (int k = 0, q = begin[i]; q < begin[i + 1]; ++k, ++q) {
          up[q] = L.objKeys[2 * k]; vp[q] = L.objKeys[2 * k + 1]; zp[q] = L.objDepth[k]; lp[q] = L.semObjLabel[k];
          uc[q] = C.objKeys[2 * k]; vc[q] = C.objKeys[2 * k + 1]; zc[q] = C.objDepth[k]; lc[q] = C.semObjLabel[k];
        }
        std::memcpy(&Tp[16 * i], L.Tcw.data(), 64); std::memcpy(&Tc[16 * i], C.Tcw.data(), 64);
        const float k4[4] = {p.fx, p.fy, p.cx, p.cy};
        std::memcpy(&K4[4 * i], k4, 16);
      }
      TB(vdo::scene_flow_batch(ts[0]->ctx, n, begin.data(), Tp.data(), Tc.data(), K4.data(), up.data(), vp.data(), zp.data(), uc.data(), vc.data(), zc.data(),
                               lp.data(), lc.data(), f3.data(), nullptr, valid.data()));
      for (int i = 0; i < n; ++i) {
        FrameState& C = cur_of(ts[i]);
        std::copy(f3.begin() + 3 * (size_t)begin[i], f3.begin() + 3 * (size_t)begin[i + 1], C.flow3d.begin());
        for (int k = 0, q = begin[i]; q < begin[i + 1]; ++k, ++q) if (!valid[q]) C.objLabel[k] = -1;
      }
    }
  }
  // DynObjTracking (:1366-1612), per tracker
  std::vector<std::vector<std::vector<int>>> objIdNew(n);
  std::vector<std::vector<int>> live(n);
  for (int ti = 0; ti < n; ++ti) {
    vdo_tracker* t = ts[ti]; const vdo_tracker_params& p = t->p;
    FrameState& C = cur_of(t); const FrameState& L = last_of(t);
    StageTimer stage_timer_6(&t->stage_ms[6]);
    const int No = (int)C.objKeys.size() / 2;
    std::vector<int> ob(257), oi(No + 1), ml(256), sp(256);
    int nobj = 0;
    {
      std::vector<float> kx(No + 1), ky(No + 1);
      for (int i = 0; i < No; ++i) { kx[i] = C.objKeys[2 * i]; ky[i] = C.objKeys[2 * i + 1]; }
      TK(vdo_dyn_obj_tracking(t->ctx, No, C.semObjLabel.data(), C.objLabel.data(), kx.data(), ky.data(), C.objDepth.data(), C.flow3d.data(), L.semObjLabel.data(),
                              (int)L.nSemPosition.size(), L.nSemPosition.data(), L.bObjStat.data(), L.nModLabel.data(), p.height, p.width, p.is_kitti ? 25 : 0,
                              p.is_kitti ? 50 : 0, p.sf_mg_thres, p.sf_ds_thres, p.th_depth_obj, t->f_id, &t->max_id, 256, &nobj, ob.data(), oi.data(), ml.data(),
                              sp.data()));
    }
    C.nModLabel.assign(ml.begin(), ml.begin() + nobj); C.nSemPosition.assign(sp.begin(), sp.begin() + nobj);
    C.bObjStat.assign(nobj, 1); C.vObjMod.assign(nobj, eye4()); C.vnObjID.assign(nobj, {}); C.vnObjInlierID.assign(nobj, {});
    C.vObjCentre3D.assign(3 * (size_t)nobj, 0.f);
    objIdNew[ti].resize(nobj);
    for (int i = 0; i < nobj; ++i) objIdNew[ti][i].assign(oi.begin() + ob[i], oi.begin() + ob[i + 1]);
    // ground-truth presence gate (:767-810)
    for (int i = 0; i < nobj; ++i) {
      const int sem = C.nSemPosition[i];
      const bool g1 = std::find(L.semPosiGt.begin(), L.semPosiGt.end(), sem) != L.semPosiGt.end();
      const bool g2 = std::find(C.semPosiGt.begin(), C.semPosiGt.end(), sem) != C.semPosiGt.end();
      if (!g1 || !g2) { C.bObjStat[i] = 0; C.vnObjInlierID[i] = objIdNew[ti][i]; continue; }
      C.vnObjID[i] = objIdNew[ti][i];
      live[ti].push_back(i);
    }
  }
  // per live object of every tracker: initial model (:1717-1849), joint flow / motion LM (src/Optimizer.cc:2755-2972).  The objects are
  // independent of each other (disjoint point sets), so the two device stages run as one batch each.
  {
    BatchTimer timer(ts, 6);
    struct Prob { int ti, obj; };
    std::vector<Prob> probs;
    for (int ti = 0; ti < n; ++ti) for (int i : live[ti]) probs.push_back({ti, i});
    if (!probs.empty()) {
      const int np = (int)probs.size();
      std::vector<int> offs(np + 1, 0);
      for (int j = 0; j < np; ++j) offs[j + 1] = offs[j] + (int)objIdNew[probs[j].ti][probs[j].obj].size();
      const int tot = offs[np];
      std::vector<float> obj3(3 * (size_t)tot + 3), img2(2 * (size_t)tot + 2), Tmm(16 * (size_t)np), Tin(16 * (size_t)np), K4(4 * (size_t)np);
      std::vector<unsigned char> has(np, 0);
      std::vector<int> nsub(np), sub(tot + 1);
      for (int j = 0; j < np; ++j) {
        vdo_tracker* t = ts[probs[j].ti]; const vdo_tracker_params& p = t->p; const int i = probs[j].obj;
        FrameState& C = cur_of(t); const FrameState& L = last_of(t);
        int q = offs[j];
        float cs[3] = {0.f, 0.f, 0.f};
        for (int id : objIdNew[probs[j].ti][i]) {
          img2[2 * q] = C.objKeys[2 * id]; img2[2 * q + 1] = C.objKeys[2 * id + 1];
          unproject_world(L.objKeys[2 * id], L.objKeys[2 * id + 1], L.objDepth[id], p, L.Tcw, &obj3[3 * q]);
          for (int r = 0; r < 3; ++r) cs[r] = cs[r] + obj3[3 * q + r];                       // ObjCentre3D_pre + x3D_p, float
          ++q;
        }
        const float inv_n = (float)(1.0 / (double)objIdNew[probs[j].ti][i].size());        // cv::Mat / size(): convertTo with alpha = 1/n, float
        for (int r = 0; r < 3; ++r) C.vObjCentre3D[3 * (size_t)i + r] = cs[r] * inv_n;
        int pre = -1;
        for (size_t k = 0; k < L.nModLabel.size(); ++k) if (L.nModLabel[k] == C.nModLabel[i]) { pre = (int)k; break; }
        if (pre != -1) { has[j] = 1; const M4 mm = mul4(C.Tcw, L.vObjMod[pre]); std::memcpy(&Tmm[16 * j], mm.data(), 64); }
        const float k4[4] = {p.fx, p.fy, p.cx, p.cy};
        std::memcpy(&K4[4 * j], k4, 16);
      }
      TB(vdo::init_model_batch(ts[0]->ctx, np, offs.data(), obj3.data(), img2.data(), K4.data(), 4, 500, 0.4, 0.98, Tmm.data(), has.data(), Tin.data(), nsub.data(),
                               sub.data(), nullptr, nullptr, nullptr));
      std::vector<std::vector<int>> idIn(np);
      std::vector<FlowJob> jobs; std::vector<int> jobProb;
      for (int j = 0; j < np; ++j) {
        vdo_tracker* t = ts[probs[j].ti]; const int i = probs[j].obj;
        FrameState& C = cur_of(t);
        const std::vector<int>& ids = objIdNew[probs[j].ti][i];
        std::vector<char> kept(ids.size(), 0);
        idIn[j].resize(nsub[j]);
        for (int q = 0; q < nsub[j]; ++q) { const int loc = sub[offs[j] + q]; idIn[j][q] = ids[loc]; kept[loc] = 1; }
        for (size_t q = 0; q < ids.size(); ++q) if (!kept[q]) C.objLabel[ids[q]] = -1;       // :1841-1845
        if ((int)idIn[j].size() < 50) { C.bObjStat[i] = 0; C.vnObjInlierID[i] = idIn[j]; continue; }   // :885-897
        M4 Ti; std::memcpy(Ti.data(), &Tin[16 * j], 64);
        jobs.push_back({t, 1, &idIn[j], Ti}); jobProb.push_back(j);
      }
      if (!jobs.empty()) {
        std::vector<M4> To; std::vector<double> fo; std::vector<unsigned char> inl; std::vector<int> fo_offs;
        TB(run_flow(ts, true, jobs, To, fo, inl, fo_offs));
        for (size_t j = 0; j < jobs.size(); ++j) {
          vdo_tracker* t = jobs[j].t; const int i = probs[jobProb[j]].obj; const std::vector<int>& ids = *jobs[j].idx;
          FrameState& C = cur_of(t); const FrameState& L = last_of(t);
          std::vector<int> inlierID;
          for (size_t q = 0; q < ids.size(); ++q) {
            const int id = ids[q]; const size_t g = (size_t)fo_offs[j] + q;
            if (inl[g]) {
              C.objKeys[2 * id] = (float)((double)L.objKeys[2 * id] + fo[2 * g]);
              C.objKeys[2 * id + 1] = (float)((double)L.objKeys[2 * id + 1] + fo[2 * g + 1]);
              inlierID.push_back(id);
            } else C.objLabel[id] = -1;
          }
          C.vObjMod[i] = mul4(inv4(C.Tcw), To[j]);                               // :907
          C.vnObjInlierID[i] = inlierID;
        }
      }
    }
  }
  // ---------------- RenewFrameInfo (:2660-2995), per tracker ----------------
  for (vdo_tracker* t : ts) {
    const vdo_tracker_params& p = t->p;
    const float K4[4] = {p.fx, p.fy, p.cx, p.cy};
    FrameState& C = cur_of(t);
    StageTimer stage_timer_7(&t->stage_ms[7]);
    const int nobj = (int)C.nModLabel.size(), Ns = (int)C.statKeys.size() / 2, No = (int)C.objKeys.size() / 2;
    const M4 Twc = inv4(C.Tcw);
    std::vector<int> ib(nobj + 1, 0), ii;
    for (int i = 0; i < nobj; ++i) { ii.insert(ii.end(), C.vnObjInlierID[i].begin(), C.vnObjInlierID[i].end()); ib[i + 1] = (int)ii.size(); }
    // the top-up source (src/Tracking.cc:2718-2721): the frame's option-II keys when sampling, else mvKeys.  statKeysTmp still holds the
    // frame build's keys here; the renewal below replaces it.
    const std::vector<float>& samp = p.use_sample_feature ? C.statKeysTmp : C.keys;
    const int nTm = (int)t->temperalMatchSubset.size(), nSamp = (int)samp.size() / 2, nTmp = (int)t->tmpSemObjLabel.size();
    const int capS = nTm + nSamp + 8, capO = (int)ii.size() + (nobj + 1) * nTmp + 8;
    std::vector<float> sk(2 * (size_t)capS), sc(2 * (size_t)capS), sf(2 * (size_t)capS), sd(capS), s3(3 * (size_t)capS);
    std::vector<int> sid(capS);
    std::vector<float> okk(2 * (size_t)capO), od(capO), oc(2 * (size_t)capO), of(2 * (size_t)capO), o3(3 * (size_t)capO);
    std::vector<int> osem(capO), oid(capO), olab(capO);
    int ns = 0, no = 0;
    TK(vdo_renew_frame_info(C.img, nTm, t->temperalMatchSubset.data(), Ns, C.statKeys.data(), nSamp, samp.data(), p.max_track_bg, nobj, ib.data(), ii.data(),
                            C.bObjStat.data(), C.nSemPosition.data(), C.nModLabel.data(), No, C.objKeys.data(), C.objLabel.data(), nTmp, t->tmpObjKeys.data(),
                            t->tmpObjDepth.data(), t->tmpSemObjLabel.data(), t->tmpObjFlowNext.data(), t->tmpObjCorres.data(), p.max_track_obj, K4, Twc.data(), capS, &ns,
                            sk.data(), sc.data(), sf.data(), sid.data(), sd.data(), s3.data(), capO, &no, okk.data(), od.data(), oc.data(), of.data(), osem.data(),
                            oid.data(), olab.data(), o3.data()));
    C.statKeysTmp.assign(sk.begin(), sk.begin() + 2 * (size_t)ns); C.corres.assign(sc.begin(), sc.begin() + 2 * (size_t)ns);
    C.flowNext.assign(sf.begin(), sf.begin() + 2 * (size_t)ns); C.statDepthTmp.assign(sd.begin(), sd.begin() + ns);
    C.stat3DTmp.assign(s3.begin(), s3.begin() + 3 * (size_t)ns); C.staInlierID.assign(sid.begin(), sid.begin() + ns);
    C.objKeys.assign(okk.begin(), okk.begin() + 2 * (size_t)no); C.objDepth.assign(od.begin(), od.begin() + no);
    C.objCorres.assign(oc.begin(), oc.begin() + 2 * (size_t)no); C.objFlowNext.assign(of.begin(), of.begin() + 2 * (size_t)no);
    C.obj3D.assign(o3.begin(), o3.begin() + 3 * (size_t)no); C.semObjLabel.assign(osem.begin(), osem.begin() + no);
    C.dynInlierID.assign(oid.begin(), oid.begin() + no); C.objLabel.assign(olab.begin(), olab.begin() + no);
  }
  return VDO_OK;
}

// the newest map frame of every tracker of the list into its tracklet tables: one upload and one launch
int push_tracklets(const Span& ts) {
  std::vector<vdo::Tracklets*> T;
  std::vector<vdo::TrackletFrame> fr;
  for (vdo_tracker* t : ts) {
    const MapSlice& m = t->map;
    const bool first = m.featSta.size() == 1;
    T.push_back(t->tracklets);
    fr.push_back({(int)m.featSta.back().size() / 2, (int)m.featDyn.back().size() / 2, first ? nullptr : m.assoSta.back().data(),
                  first ? nullptr : m.assoDyn.back().data(), first ? nullptr : m.featLabel.back().data()});
  }
  TB(vdo::tracklets_push((void*)(uintptr_t)vdo_ctx_stream(ts[0]->ctx), T.data(), (int)T.size(), fr.data()));
  return VDO_OK;
}

void push_map(vdo_tracker* t, const FrameState& C, bool first) {          // Tracking.cc:1235-1246 (first frame), :1016-1070
  MapSlice& m = t->map;
  m.featSta.push_back(C.statKeysTmp); m.depSta.push_back(C.statDepthTmp); m.p3dSta.push_back(C.stat3DTmp);
  m.featDyn.push_back(C.objKeys); m.depDyn.push_back(C.objDepth); m.p3dDyn.push_back(C.obj3D);
  m.cameraPose.push_back(first ? eye4() : inv4(C.Tcw));
  m.cameraPose_RF.push_back(m.cameraPose.back());
  if (first) return;
  m.assoSta.push_back(C.staInlierID); m.assoDyn.push_back(C.dynInlierID); m.featLabel.push_back(C.objLabel);
  std::vector<M4> mot{inv4(t->velocity)}; std::vector<int> rl{0}, sl{0};
  std::vector<float> cen{0.f, 0.f, 0.f};
  for (size_t i = 0; i < C.vObjMod.size(); ++i) {
    if (!C.bObjStat[i]) continue;
    mot.push_back(C.vObjMod[i]); rl.push_back(C.nModLabel[i]); sl.push_back(C.nSemPosition[i]);
    for (int r = 0; r < 3; ++r) cen.push_back(C.vObjCentre3D[3 * i + r]);
  }
  m.rigidMotion.push_back(mot); m.rigidMotion_RF.push_back(mot); m.rmLabel.push_back(rl); m.smLabel.push_back(sl); m.rigidCentre.push_back(cen);
}

}  // namespace

extern "C" void vdo_tracker_params_default(vdo_tracker_params* p) {       // example/kitti-0000-0013.yaml
  if (!p) return;
  std::memset(p, 0, sizeof *p);
  p->width = 1242; p->height = 375; p->fx = 721.5377f; p->fy = 721.5377f; p->cx = 609.5593f; p->cy = 172.8540f; p->bf = 387.5744f; p->depth_factor = 256.f;
  p->th_depth_bg = 40.f; p->th_depth_obj = 25.f; p->max_track_bg = 1200; p->max_track_obj = 800; p->sf_mg_thres = 0.12f; p->sf_ds_thres = 0.3f;
  p->n_features = 2500; p->scale_factor = 1.2f; p->n_levels = 8; p->ini_th_fast = 20; p->min_th_fast = 7; p->is_kitti = 1; p->quirk = 1;
  p->window_size = 20; p->overlap_size = 4; p->local_batch = 1;
}

extern "C" int vdo_tracker_create(vdo_ctx* ctx, const vdo_tracker_params* params, vdo_tracker** out) {
  // width == height == 0: a MAP-ONLY handle (no frame buffers): frames are pushed with vdo_tracker_map_push and optimised with
  // vdo_tracker_batch_optimize -- the form Optimizer::FullBatchOptimization(Map*, K) / PartialBatchOptimization take their input in
  const bool map_only = params && params->width == 0 && params->height == 0;
  if (!ctx || !params || !out || (!map_only && (params->width < 64 || params->height < 64))) return VDO_ERR_ARG;
  // UseSampleFeature is 0 or 1; the sampling grid's steps width / 20 and height / 20 must not be 0
  if (params->use_sample_feature != 0 && params->use_sample_feature != 1) return VDO_ERR_ARG;
  if (params->use_sample_feature && (params->width < 20 || params->height < 20)) return VDO_ERR_ARG;
  // ORB settings out of range (VDO_ERR_ARG of vdo_orb_extractor_create: level counts, scale factors, a pyramid level under 1 px) are
  // refused here; the extractor's limits (VDO_ERR_UNSUPPORTED) are reported by the first tracking call, before any state changes
  if (!map_only) {
    std::string why;
    const vdo::OrbKey key{params->width, params->height, params->n_features, params->scale_factor, params->n_levels, params->ini_th_fast, params->min_th_fast};
    if (vdo::orb_key_check(key, why) == VDO_ERR_ARG) { vdo::ctx_set_error(ctx, "vdo_tracker_create: ORB settings: " + why); return VDO_ERR_ARG; }
  }
  vdo_tracker* t = new vdo_tracker;
  t->ctx = ctx; t->p = *params;
  t->tracklets = vdo::tracklets_create();
  for (int i = 0; i < 2 && !map_only; ++i)
    if (vdo_frame_create(ctx, params->width, params->height, &t->fr[i].img) != VDO_OK) { vdo_tracker_destroy(t); return VDO_ERR_CUDA; }
  *out = t;
  return VDO_OK;
}
// One frame of an externally built Map (include/Map.h:34-84; what Tracking::Track pushes per frame, src/Tracking.cc:1016-1105).  Frame 0
// carries no associations / motions (n_mot == 0).  Arrays: feat (x, y) pairs, p3d xyz triples, asso / label one int per feature,
// camera_pose16 = vmCameraPose[i] (Twc, row-major), rigid_motion16 = vmRigidMotion[i - 1] (n_mot matrices, entry 0 = camera), rm_label likewise.
extern "C" int vdo_tracker_map_push(vdo_tracker* t, int n_sta, const float* feat_sta, const float* dep_sta, const float* p3d_sta, const int* asso_sta, int n_dyn,
                                    const float* feat_dyn, const float* dep_dyn, const float* p3d_dyn, const int* asso_dyn, const int* feat_label,
                                    const float* camera_pose16, int n_mot, const float* rigid_motion16, const int* rm_label) {
  if (!t || n_sta < 0 || n_dyn < 0 || n_mot < 0 || !camera_pose16) return VDO_ERR_ARG;
  if ((n_sta && (!feat_sta || !dep_sta || !p3d_sta)) || (n_dyn && (!feat_dyn || !dep_dyn || !p3d_dyn)) || (n_mot && (!rigid_motion16 || !rm_label))) return VDO_ERR_ARG;
  MapSlice& m = t->map;
  const bool first = m.featSta.empty();
  if (first != (n_mot == 0)) { t->err = "vdo_tracker_map_push: frame 0 has no motions, every later frame has at least the camera motion"; return VDO_ERR_ARG; }
  if (!first && ((n_sta && !asso_sta) || (n_dyn && (!asso_dyn || !feat_label)))) return VDO_ERR_ARG;
  m.featSta.emplace_back(feat_sta, feat_sta + 2 * (size_t)n_sta); m.depSta.emplace_back(dep_sta, dep_sta + n_sta); m.p3dSta.emplace_back(p3d_sta, p3d_sta + 3 * (size_t)n_sta);
  m.featDyn.emplace_back(feat_dyn, feat_dyn + 2 * (size_t)n_dyn); m.depDyn.emplace_back(dep_dyn, dep_dyn + n_dyn); m.p3dDyn.emplace_back(p3d_dyn, p3d_dyn + 3 * (size_t)n_dyn);
  M4 P; std::memcpy(P.data(), camera_pose16, 64);
  m.cameraPose.push_back(P); m.cameraPose_RF.push_back(P);
  if (!first) {
    m.assoSta.emplace_back(asso_sta, asso_sta + n_sta); m.assoDyn.emplace_back(asso_dyn, asso_dyn + n_dyn); m.featLabel.emplace_back(feat_label, feat_label + n_dyn);
    std::vector<M4> mot(n_mot);
    for (int j = 0; j < n_mot; ++j) std::memcpy(mot[j].data(), rigid_motion16 + 16 * (size_t)j, 64);
    m.rigidMotion.push_back(mot); m.rigidMotion_RF.push_back(mot);
    m.rmLabel.emplace_back(rm_label, rm_label + n_mot); m.smLabel.emplace_back(rm_label, rm_label + n_mot);
    m.rigidCentre.emplace_back(3 * (size_t)n_mot, 0.f);
  }
  return push_tracklets(Span{t});
}
extern "C" void vdo_tracker_destroy(vdo_tracker* t) {
  if (!t) return;
  for (int i = 0; i < 2; ++i) if (t->fr[i].img) vdo_frame_destroy(t->fr[i].img);
  vdo::tracklets_destroy(t->tracklets);
  delete t;
}
extern "C" const char* vdo_tracker_last_error(const vdo_tracker* t) { return t ? t->err.c_str() : "null tracker"; }

namespace {
// The caller's images: host buffers (vdo_tracker_track) or device planes image / depth / flow / mask (vdo_tracker_track_dev / _batch_dev)
struct FrameInput {
  const unsigned char* gray = nullptr; float* depth = nullptr; const float* flow = nullptr; int* mask = nullptr;
  const vdo_dev_plane* planes[4] = {nullptr, nullptr, nullptr, nullptr}; uint64_t stream = 0;
  bool dev = false;
};

std::vector<vdo_frame*> img_frames(const Span& ts) {   // a resident frame of every tracker (its stream and size are the tracker's)
  std::vector<vdo_frame*> f;
  for (vdo_tracker* t : ts) f.push_back(t->fr[0].img);
  return f;
}

// Tracking::GrabImageRGBD up to the new Frame (src/Tracking.cc:164-204, :2997-3110) for every tracker of the list: the caller's images
// into the frame that becomes current, depth pre-processing, UpdateMask, and the write-back into the caller's buffers.  Upload and depth
// preparation run on the buffer about to become current (after a tracked frame: the frame before last, which nothing reads any more)
// before any tracker swaps current / last, so a list refused there -- by the device-side label-range check of any one frame -- leaves
// every tracker unchanged.  So does a list whose frame-build extractor (*orb, looked up first) refuses the ORB settings of any one tracker
// or fails to allocate.  geo: per tracker, its geometry (image size and ORB settings) on *orb.
// Host buffers come one tracker at a time; device planes are ingested with one launch for the list.
int grab_frames(const Span& ts, const FrameInput* in, int writeback, const char* fn, vdo::OrbJob** orb, std::vector<int>& geo) {
  const int n = (int)ts.size();
  std::vector<vdo::OrbKey> keys(n);
  for (int i = 0; i < n; ++i) {
    const vdo_tracker_params& p = ts[i]->p;
    keys[i] = vdo::OrbKey{p.width, p.height, p.n_features, p.scale_factor, p.n_levels, p.ini_th_fast, p.min_th_fast};
  }
  geo.assign(n, 0);
  int bad = 0;
  if (int rc = vdo::orb_job_for(img_frames(ts).data(), keys.data(), n, orb, geo.data(), &bad)) {
    ts[0]->err = std::string(fn) + ": " + (n > 1 ? "trackers[" + std::to_string(bad) + "]: " : std::string()) +
                 "the ORB extractor refuses these ORB settings or could not be allocated (vdo_orb_extractor_create: " + std::to_string(rc) + ")";
    return rc;
  }
  std::vector<vdo_frame*> img(n);
  for (int i = 0; i < n; ++i) img[i] = ts[i]->fr[ts[i]->first ? ts[i]->cur : 1 - ts[i]->cur].img;
  {
    BatchTimer timer(ts, 0);
    std::vector<float> bf(n), factor(n);
    for (int i = 0; i < n; ++i) {
      const vdo_tracker_params& p = ts[i]->p;
      const int dataset = p.dataset ? p.dataset : (p.is_kitti ? 2 : 1);
      bf[i] = dataset == 3 ? 0.f : p.bf; factor[i] = p.depth_factor;
    }
    if (in[0].dev) {
      std::vector<const vdo_dev_plane*> planes(4 * (size_t)n);
      for (int i = 0; i < n; ++i) for (int k = 0; k < 4; ++k) planes[4 * i + k] = in[i].planes[k];
      TB(vdo::frames_ingest_dev(img.data(), n, planes.data(), in[0].stream));
      TB(vdo::frames_depth_prep(img.data(), n, bf.data(), factor.data()));                  // :180-204 (written back below)
      std::string e; int bad = 0;
      if (int rc = vdo::frames_ingest_wait(img.data(), n, &bad, e)) {
        ts[0]->err = std::string(fn) + ": " + (e.empty() ? std::string("CUDA error") : (n > 1 ? "trackers[" + std::to_string(bad) + "]: " : std::string()) + e);
        return rc;
      }
    } else {
      for (int i = 0; i < n; ++i) {
        vdo_tracker* t = ts[i];
        TK(vdo_frame_upload(img[i], in[i].gray, in[i].depth, in[i].flow, in[i].mask));
        TK(vdo_frame_depth_prep(img[i], bf[i], factor[i], writeback ? in[i].depth : nullptr));   // :180-204, in place on the caller's Mat
      }
    }
  }
  for (int i = 0; i < n; ++i) {
    vdo_tracker* t = ts[i];
    if (!t->first) t->cur = 1 - t->cur;
    FrameState& C = cur_of(t); FrameState& L = last_of(t);
    C.clear_dynamic(); C.img = img[i]; C.Tcw = eye4();
    if (t->first) t->f_id = 0;
    StageTimer stage_timer_1(&t->stage_ms[1]);
    int nw = 0;
    if (!t->first) {                                                                            // UpdateMask (:2997-3110)
      const int m = (int)L.semObjLabel.size();
      std::vector<float> cx(m + 1), cy(m + 1);
      for (int k = 0; k < m; ++k) { cx[k] = L.objCorres[2 * k]; cy[k] = L.objCorres[2 * k + 1]; }
      TK(vdo_update_mask(C.img, L.img, m, L.semObjLabel.data(), cx.data(), cy.data(), nullptr, &nw, nullptr));
    }
    // the caller's mask already holds the labels unless an object was warped into it (:3062)
    if (writeback && in[i].dev) TK(vdo::frame_writeback_dev(C.img, in[i].planes[1], nw > 0 ? in[i].planes[3] : nullptr));   // synchronised by the frame build
    else if (writeback && nw > 0) TK(vdo_frame_read_mask(C.img, in[i].mask));
  }
  return VDO_OK;
}

int windowed_optimize(const Span& due);   // below, next to the map -> graph construction

// the rest of GrabImageRGBD and Tracking::Track on the frames grab_frames made current (src/Tracking.cc:205-648, 650-1212).
// gt_begin / gt_ids: the ground-truth semantic ids of tracker i are gt_ids[gt_begin[i] .. gt_begin[i + 1]); Tcw_out: 16 floats per tracker.
int track_grabbed(const Span& ts, const vdo::OrbJob& orb, const int* geo, const int* gt_begin, const int* gt_ids, float* Tcw_out) {
  const int n = (int)ts.size();
  {
    BatchTimer timer(ts, 2);
    if (int rc = build_frames(ts, orb, geo)) return rc;
  }
  Span rest;                                                                                    // trackers past their first frame
  for (vdo_tracker* t : ts) if (!t->first) rest.push_back(t);
  if (!rest.empty()) {                                                                          // :254-312, both look-ups of every tracker in one launch
    BatchTimer timer(rest, 3);
    const Span& ts = rest;
    const int m = (int)rest.size();
    std::vector<vdo_frame*> segf(2 * (size_t)m);
    std::vector<int> begin(2 * (size_t)m + 1, 0);
    for (int j = 0; j < m; ++j) {
      vdo_tracker* t = rest[j];
      FrameState& C = cur_of(t); const FrameState& L = last_of(t);
      C.statKeys = L.corres;
      t->tmpObjKeys = C.objKeys; t->tmpObjDepth = C.objDepth; t->tmpSemObjLabel = C.semObjLabel; t->tmpObjFlowNext = C.objFlowNext; t->tmpObjCorres = C.objCorres;
      C.objKeys = L.objCorres;
      segf[2 * j] = segf[2 * j + 1] = C.img;
      begin[2 * j + 1] = begin[2 * j] + (int)C.statKeys.size() / 2;
      begin[2 * j + 2] = begin[2 * j + 1] + (int)C.objKeys.size() / 2;
    }
    const int tot = begin[2 * m];
    std::vector<float> keys(2 * (size_t)tot + 2), d((size_t)tot + 1); std::vector<int> mk((size_t)tot + 1);
    for (int j = 0; j < m; ++j) {
      const FrameState& C = cur_of(rest[j]);
      std::copy(C.statKeys.begin(), C.statKeys.end(), keys.begin() + 2 * (size_t)begin[2 * j]);
      std::copy(C.objKeys.begin(), C.objKeys.end(), keys.begin() + 2 * (size_t)begin[2 * j + 1]);
    }
    TB(vdo::gather_batch(segf.data(), 2 * m, begin.data(), keys.data(), d.data(), mk.data()));
    for (int j = 0; j < m; ++j) {
      const vdo_tracker_params& p = rest[j]->p;
      FrameState& C = cur_of(rest[j]);
      const int Ns = (int)C.statKeys.size() / 2;
      C.statDepth.resize(Ns);
      for (int i = 0; i < Ns; ++i) {
        const int u = (int)C.statKeys[2 * i], v = (int)C.statKeys[2 * i + 1];
        const bool in = u < p.width - 1 && u > 0 && v < p.height - 1 && v > 0;
        const float di = d[begin[2 * j] + i];
        C.statDepth[i] = (in && di > 0) ? di : -1.f;
      }
      const int No = (int)C.objKeys.size() / 2;
      C.objDepth.assign(No, 0.1f); C.semObjLabel.assign(No, 0);
      for (int i = 0; i < No; ++i) {
        const int u = (int)C.objKeys[2 * i], v = (int)C.objKeys[2 * i + 1];
        const float od = d[begin[2 * j + 1] + i]; const int om = mk[begin[2 * j + 1] + i];
        if (u < p.width - 1 && u > 0 && v < p.height - 1 && v > 0 && od < p.th_depth_obj && od > 0) { C.objDepth[i] = od; C.semObjLabel[i] = om; }
      }
    }
  }
  for (int i = 0; i < n; ++i) {
    FrameState& C = cur_of(ts[i]);
    C.semPosiGt.assign(gt_ids + gt_begin[i], gt_ids + gt_begin[i + 1]);
    C.objLabel.assign(C.objKeys.size() / 2, -2);                                                // :345
  }
  for (vdo_tracker* t : ts) {
    if (!t->first) continue;
    const vdo_tracker_params& p = t->p;                                                         // Initialization (:1215-1276)
    FrameState& C = cur_of(t);
    const int ns = (int)C.statKeysTmp.size() / 2, no = (int)C.objKeys.size() / 2;
    C.stat3DTmp.resize(3 * (size_t)ns); C.obj3D.resize(3 * (size_t)no);
    for (int i = 0; i < ns; ++i) get3d_camera(C.statKeysTmp[2 * i], C.statKeysTmp[2 * i + 1], C.statDepthTmp[i], p, &C.stat3DTmp[3 * i]);
    for (int i = 0; i < no; ++i) get3d_camera(C.objKeys[2 * i], C.objKeys[2 * i + 1], C.objDepth[i], p, &C.obj3D[3 * i]);
    C.Tcw = eye4();
    push_map(t, C, true);
  }
  if (!rest.empty()) {
    if (int rc = track_frames(rest)) return rc;
    for (vdo_tracker* t : rest) push_map(t, cur_of(t), false);
  }
  if (int rc = push_tracklets(ts)) return rc;
  Span due;                                                                                     // windowed optimisations of this call
  for (int i = 0; i < n; ++i) {
    vdo_tracker* t = ts[i]; const vdo_tracker_params& p = t->p;
    FrameState& C = cur_of(t);
    t->first = false;
    // mLastFrame = Frame(mCurrentFrame) with the "new added" overrides (:1006-1014): the next call reads this frame through L
    C.statKeys = C.statKeysTmp; C.statDepth = C.statDepthTmp;
    // windowed optimisation on the reference's schedule (src/Tracking.cc:1150-1160)
    if (p.local_batch && p.window_size > p.overlap_size && p.overlap_size >= 0 && (t->f_id - p.overlap_size + 1) % (p.window_size - p.overlap_size) == 0 &&
        t->f_id >= p.window_size - 1)
      due.push_back(t);
    t->f_id += 1; t->frames += 1;
    if (Tcw_out) std::memcpy(Tcw_out + 16 * (size_t)i, C.Tcw.data(), 64);
  }
  if (!due.empty()) {
    BatchTimer timer(due, 8);
    if (int rc = windowed_optimize(due)) return rc;
  }
  return VDO_OK;
}

int check_size(vdo_tracker* t, const char* fn, int width, int height) {
  const vdo_tracker_params& p = t->p;
  if (!t->fr[0].img) { t->err = std::string(fn) + " on a map-only handle"; return VDO_ERR_STATE; }
  if (width != p.width || height != p.height) {
    t->err = std::string(fn) + ": buffers are " + std::to_string(width) + "x" + std::to_string(height) + " but the tracker was created for " + std::to_string(p.width) +
             "x" + std::to_string(p.height);
    return VDO_ERR_ARG;
  }
  return VDO_OK;
}
}  // namespace

// System::TrackRGBD / Tracking::GrabImageRGBD (include/System.h:49-51, src/Tracking.cc:164-648)
extern "C" int vdo_tracker_track(vdo_tracker* t, int width, int height, const unsigned char* gray, float* depth, const float* flow, int* mask, int n_gt,
                                 const int* gt_sem_ids, int writeback, float* Tcw_out) {
  if (!t || !gray || !depth || !flow || !mask || n_gt < 0) return VDO_ERR_ARG;
  if (int rc = check_size(t, "vdo_tracker_track", width, height)) return rc;
  FrameInput in;
  in.gray = gray; in.depth = depth; in.flow = flow; in.mask = mask;
  const Span ts{t};
  const int gt_begin[2] = {0, n_gt};
  vdo::OrbJob* orb = nullptr; std::vector<int> geo;
  if (int rc = grab_frames(ts, &in, writeback, "vdo_tracker_track", &orb, geo)) return rc;
  return track_grabbed(ts, *orb, geo.data(), gt_begin, gt_sem_ids, Tcw_out);
}

// the same on device-resident planes (include/vdo_b200.h: vdo_dev_plane, vdo_frame_upload_dev)
extern "C" int vdo_tracker_track_dev(vdo_tracker* t, int width, int height, const vdo_dev_plane* image, const vdo_dev_plane* depth, const vdo_dev_plane* flow,
                                     const vdo_dev_plane* mask, int n_gt, const int* gt_sem_ids, int writeback, uint64_t stream, float* Tcw_out) {
  if (!t || n_gt < 0 || (n_gt > 0 && !gt_sem_ids)) return VDO_ERR_ARG;
  if (!image || !depth || !flow || !mask) { t->err = "vdo_tracker_track_dev: all four planes are required"; return VDO_ERR_ARG; }
  if (int rc = check_size(t, "vdo_tracker_track_dev", width, height)) return rc;
  FrameInput in;
  in.planes[0] = image; in.planes[1] = depth; in.planes[2] = flow; in.planes[3] = mask; in.stream = stream; in.dev = true;
  const bool target[4] = {false, writeback != 0, false, writeback != 0};
  std::string e;
  if (int rc = vdo::frame_check_planes(t->fr[0].img, in.planes, target, e)) { t->err = "vdo_tracker_track_dev: " + e; return rc; }
  const Span ts{t};
  const int gt_begin[2] = {0, n_gt};
  vdo::OrbJob* orb = nullptr; std::vector<int> geo;
  if (int rc = grab_frames(ts, &in, writeback, "vdo_tracker_track_dev", &orb, geo)) return rc;
  return track_grabbed(ts, *orb, geo.data(), gt_begin, gt_sem_ids, Tcw_out);
}

namespace {
// n trackers advanced by one frame each, every batched stage as one set of launches: the body of vdo_tracker_track_batch_dev and
// vdo_tracker_track_mixed_dev.  same_geometry: refuse trackers that differ from trackers[0] in image size or ORB settings.
int track_list(const char* fn, bool same_geometry, vdo_tracker* const* trackers, int n, const vdo_dev_plane* images, const vdo_dev_plane* depths,
               const vdo_dev_plane* flows, const vdo_dev_plane* masks, const int* gt_begin, const int* gt_ids, int writeback, uint64_t stream, float* Tcw_out) {
  if (!trackers || n < 1 || !trackers[0]) return VDO_ERR_ARG;
  vdo_tracker* t0 = trackers[0];
  auto fail = [&](int rc, const std::string& m) { t0->err = std::string(fn) + ": " + m; return rc; };
  if (!images || !depths || !flows || !masks) return fail(VDO_ERR_ARG, "all four plane arrays are required");
  if (!gt_begin || gt_begin[0] != 0) return fail(VDO_ERR_ARG, "gt_begin must hold n + 1 offsets starting at 0");
  for (int i = 0; i < n; ++i)
    if (gt_begin[i + 1] < gt_begin[i]) return fail(VDO_ERR_ARG, "gt_begin[" + std::to_string(i + 1) + "] is smaller than gt_begin[" + std::to_string(i) + "]");
  if (gt_begin[n] > 0 && !gt_ids) return fail(VDO_ERR_ARG, "gt_ids is NULL but gt_begin[n] > 0");
  const vdo_tracker_params& p0 = t0->p;
  for (int i = 0; i < n; ++i) {
    vdo_tracker* t = trackers[i];
    const std::string who = "trackers[" + std::to_string(i) + "]";
    if (!t) return fail(VDO_ERR_ARG, who + " is NULL");
    for (int j = 0; j < i; ++j) if (trackers[j] == t) return fail(VDO_ERR_ARG, who + " repeats trackers[" + std::to_string(j) + "]");
    if (!t->fr[0].img) return fail(VDO_ERR_STATE, who + " is a map-only handle");
    if (t->ctx != t0->ctx) return fail(VDO_ERR_ARG, who + " is on another context than trackers[0]");
    const vdo_tracker_params& p = t->p;
    if (same_geometry && (p.width != p0.width || p.height != p0.height || p.n_features != p0.n_features || p.scale_factor != p0.scale_factor ||
                          p.n_levels != p0.n_levels || p.ini_th_fast != p0.ini_th_fast || p.min_th_fast != p0.min_th_fast))
      return fail(VDO_ERR_ARG, who + " differs from trackers[0] in width, height or ORB settings (vdo_tracker_track_mixed_dev takes such trackers)");
  }
  std::vector<FrameInput> in(n);
  const bool target[4] = {false, writeback != 0, false, writeback != 0};
  for (int i = 0; i < n; ++i) {
    in[i].planes[0] = images + i; in[i].planes[1] = depths + i; in[i].planes[2] = flows + i; in[i].planes[3] = masks + i; in[i].stream = stream; in[i].dev = true;
    std::string e;
    if (int rc = vdo::frame_check_planes(trackers[i]->fr[0].img, in[i].planes, target, e)) return fail(rc, "trackers[" + std::to_string(i) + "]: " + e);
  }
  const Span ts(trackers, trackers + n);
  vdo::OrbJob* orb = nullptr; std::vector<int> geo;
  if (int rc = grab_frames(ts, in.data(), writeback, fn, &orb, geo)) return rc;
  return track_grabbed(ts, *orb, geo.data(), gt_begin, gt_ids, Tcw_out);
}
}  // namespace

// n trackers of one image size and ORB settings advanced by one frame each (include/vdo_b200.h)
extern "C" int vdo_tracker_track_batch_dev(vdo_tracker* const* trackers, int n, const vdo_dev_plane* images, const vdo_dev_plane* depths,
                                           const vdo_dev_plane* flows, const vdo_dev_plane* masks, const int* gt_begin, const int* gt_ids, int writeback,
                                           uint64_t stream, float* Tcw_out) {
  return track_list("vdo_tracker_track_batch_dev", true, trackers, n, images, depths, flows, masks, gt_begin, gt_ids, writeback, stream, Tcw_out);
}
// the same for trackers of any image sizes and ORB settings (include/vdo_b200.h)
extern "C" int vdo_tracker_track_mixed_dev(vdo_tracker* const* trackers, int n, const vdo_dev_plane* images, const vdo_dev_plane* depths,
                                           const vdo_dev_plane* flows, const vdo_dev_plane* masks, const int* gt_begin, const int* gt_ids, int writeback,
                                           uint64_t stream, float* Tcw_out) {
  return track_list("vdo_tracker_track_mixed_dev", false, trackers, n, images, depths, flows, masks, gt_begin, gt_ids, writeback, stream, Tcw_out);
}

// Named read-back of the state after the last vdo_tracker_track call (parity tests, host shim).  kind: 'f' float, 'i' int.
// Names: Tcw, mvKeys, mvStatKeys(Tmp), mvStatDepth(Tmp), mvCorres, mvFlowNext, mvStat3DPointTmp, nStaInlierID, mvObjKeys, mvObjDepth, mvObjCorres,
// mvObjFlowNext, mvObj3DPoint, vSemObjLabel, vObjLabel, nDynInlierID, vFlow_3d, nModLabel, nSemPosition, bObjStat, vObjMod, TemperalMatch_subset,
// max_id, f_id, mVelocity
extern "C" int vdo_tracker_get(const vdo_tracker* t, const char* name, void* out, int cap_elems, int* n_elems) {
  if (!t || !name || !n_elems) return VDO_ERR_ARG;
  const FrameState& C = t->fr[t->cur];
  const std::string s(name);
  auto put_f = [&](const float* p, size_t n) { *n_elems = (int)n; if (out && (int)n <= cap_elems && n) std::memcpy(out, p, n * 4); return (out && (int)n > cap_elems) ? VDO_ERR_ARG : VDO_OK; };
  auto put_i = [&](const int* p, size_t n) { *n_elems = (int)n; if (out && (int)n <= cap_elems && n) std::memcpy(out, p, n * 4); return (out && (int)n > cap_elems) ? VDO_ERR_ARG : VDO_OK; };
  if (s == "Tcw") return put_f(C.Tcw.data(), 16);
  if (s == "mVelocity") return put_f(t->velocity.data(), 16);
  if (s == "mvKeys") return put_f(C.keys.data(), C.keys.size());
  if (s == "mvStatKeys" || s == "mvStatKeysTmp") return put_f(C.statKeysTmp.data(), C.statKeysTmp.size());
  if (s == "mvStatDepth" || s == "mvStatDepthTmp") return put_f(C.statDepthTmp.data(), C.statDepthTmp.size());
  if (s == "mvCorres") return put_f(C.corres.data(), C.corres.size());
  if (s == "mvFlowNext") return put_f(C.flowNext.data(), C.flowNext.size());
  if (s == "mvStat3DPointTmp") return put_f(C.stat3DTmp.data(), C.stat3DTmp.size());
  if (s == "nStaInlierID") return put_i(C.staInlierID.data(), C.staInlierID.size());
  if (s == "mvObjKeys") return put_f(C.objKeys.data(), C.objKeys.size());
  if (s == "mvObjDepth") return put_f(C.objDepth.data(), C.objDepth.size());
  if (s == "mvObjCorres") return put_f(C.objCorres.data(), C.objCorres.size());
  if (s == "mvObjFlowNext") return put_f(C.objFlowNext.data(), C.objFlowNext.size());
  if (s == "mvObj3DPoint") return put_f(C.obj3D.data(), C.obj3D.size());
  if (s == "vSemObjLabel") return put_i(C.semObjLabel.data(), C.semObjLabel.size());
  if (s == "vObjLabel") return put_i(C.objLabel.data(), C.objLabel.size());
  if (s == "nDynInlierID") return put_i(C.dynInlierID.data(), C.dynInlierID.size());
  if (s == "vFlow_3d") return put_f(C.flow3d.data(), C.flow3d.size());
  if (s == "nModLabel") return put_i(C.nModLabel.data(), C.nModLabel.size());
  if (s == "nSemPosition") return put_i(C.nSemPosition.data(), C.nSemPosition.size());
  if (s == "TemperalMatch_subset") return put_i(t->temperalMatchSubset.data(), t->temperalMatchSubset.size());
  if (s == "bObjStat") { std::vector<int> v(C.bObjStat.begin(), C.bObjStat.end()); return put_i(v.data(), v.size()); }
  if (s == "vObjCentre3D") return put_f(C.vObjCentre3D.data(), C.vObjCentre3D.size());
  if (s == "vObjMod") { std::vector<float> v; for (auto& m : C.vObjMod) v.insert(v.end(), m.begin(), m.end()); return put_f(v.data(), v.size()); }
  if (s == "max_id") return put_i(&t->max_id, 1);
  if (s == "f_id") return put_i(&t->f_id, 1);
  if (s == "stage_ms") { float v[9]; for (int i = 0; i < 9; ++i) v[i] = (float)t->stage_ms[i]; return put_f(v, 9); }
  if (s == "local_ba") { const int v[2] = {t->local_ba_runs, t->local_ba_iters}; return put_i(v, 2); }
  return VDO_ERR_ARG;
}

// ------------------------------------------------------------------------------------------------ Map -> factor graph (SURVEY.md 8f N2)
// Graph construction of Optimizer::FullBatchOptimization (src/Optimizer.cc:1232-1767) and Optimizer::PartialBatchOptimization
// (:42-805) from the tracker's map, emitted as the arrays of the vdo_graph_* calls; refined camera poses, object motions and
// points are written back like :2094-2172 / :983-1050.  Where the reference would dereference a null vertex (a track whose
// previous position never received a vertex) the edge is skipped.
#include "ba_math.cuh"

namespace {
struct GraphArrays {
  std::vector<double> se3, pt, prior_Z, prior_w, se3e_Z, se3e_w, se3e_delta, obs_z, obs_w, obs_delta, ter_w, ter_delta;
  std::vector<int> prior_v, se3e_ij, obs_cp, ter_pph;
  std::vector<int> cam_vid;                       // per frame: se3 index of the camera vertex (-1 outside the window)
  std::vector<std::vector<int>> mot_vid;          // per frame pair: se3 index of each rigid-motion vertex (entry 0 unused)
  std::vector<std::vector<int>> makS, makD;       // per frame, per feature: point index (-1 = not in the graph)
  int max_iters = 300; double gain = 1e-4;
};
struct BatchConsts { float sigma2_cam, sigma2_3d_sta, sigma2_obj_smo, sigma2_obj, sigma2_3d_dyn; double prior_w; bool static_only; int max_iters; double gain; };
const BatchConsts kFull{0.001f, 80.f, 0.001f, 100.f, 80.f, 100000.0, false, 300, 1e-4};                 // src/Optimizer.cc:1330-1335
const BatchConsts kPartial{0.0001f, 16.f, 0.1f, 20.f, 16.f, 1.0 / 0.0000001, true, 100, 1e-3};          // :190-195, :230

// Converter::toSE3Quat (src/Converter.cc:25-35) + SE3Quat -> Isometry3d (se3quat.h): rotation re-normalised through the quaternion
void to_iso(const M4& T, double* out) {
  double R[9], q[4];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R[3 * i + j] = (double)T[4 * i + j];
  vdo::quat_from_rot(R, q);
  if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int k = 0; k < 4; ++k) q[k] /= n;
  vdo::rot_from_quat(q, out);
  out[9] = (double)T[3]; out[10] = (double)T[7]; out[11] = (double)T[11];
}
// getEstimateData -> Quaterniond -> rotation matrix -> Converter::toCvSE3 (src/Optimizer.cc:2094-2110)
M4 from_iso(const double* T) {
  double q[4], R[9];
  vdo::quat_from_rot(T, q);
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int k = 0; k < 4; ++k) q[k] /= n;
  vdo::rot_from_quat(q, R);
  M4 m = eye4();
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) m[4 * i + j] = (float)R[3 * i + j]; m[4 * i + 3] = (float)T[9 + i]; }
  return m;
}

// The graphs of one mode for every tracker of the list.  The pose vertices, the prior and the SE3 edges (a few per frame) are laid out here
// as in the reference; the points, observations and ternary edges come from the device builder (map_graph.cu), which reads each
// tracker's tracklet tables and the features of the graph's frames: one upload, one set of launches and one read-back for the list.
int build_graphs(const Span& ts, bool full, std::vector<GraphArrays>& Gs) {
  const BatchConsts& c = full ? kFull : kPartial;
  const int n = (int)ts.size();
  const double huber = (double)0.0001f;
  const double ident[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
  Gs.assign(n, GraphArrays());
  std::vector<vdo::GraphInput> in(n);
  for (int q = 0; q < n; ++q) {
    vdo_tracker* t = ts[q];
    const MapSlice& m = t->map;
    const int N = (int)m.featSta.size(), window = t->p.window_size;
    if (N < 2 || (!full && (window < 2 || N < window))) { t->err = "the map is too short for this optimisation"; return VDO_ERR_STATE; }
    if (vdo::tracklets_bad(t->tracklets)) { t->err = "an association of the map names a feature its previous frame does not have"; return VDO_ERR_ARG; }
    GraphArrays& G = Gs[q];
    G.makS.resize(N); G.makD.resize(N); G.cam_vid.assign(N, -1); G.mot_vid.resize(N - 1);
    for (int i = 0; i < N; ++i) {
      G.makS[i].assign(m.featSta[i].size() / 2, -1); G.makD[i].assign(m.featDyn[i].size() / 2, -1);
      if (i < N - 1) G.mot_vid[i].assign(m.rmLabel[i].size(), -1);
    }
    G.max_iters = c.max_iters; G.gain = c.gain;
    vdo::GraphInput& g = in[q];
    const int start = full ? 0 : N - window;
    g.tables = t->tracklets; g.start = start; g.dynamic = !c.static_only;
    g.invfx = 1.0f / t->p.fx; g.invfy = 1.0f / t->p.fy; g.cx = t->p.cx; g.cy = t->p.cy;       // Optimizer::Get3DinCamera
    int slot = 0, pre = -1;
    for (int i = start; i < N; ++i) {
      const int cur = (int)G.se3.size() / 12;
      double iso[12]; to_iso(m.cameraPose[i], iso);
      G.se3.insert(G.se3.end(), iso, iso + 12); G.cam_vid[i] = cur;
      if (cur == 0 && (full || N == window)) { G.prior_v.push_back(cur); G.prior_Z.insert(G.prior_Z.end(), iso, iso + 12); G.prior_w.push_back(c.prior_w); }
      if (i != start) {
        double z[12]; to_iso(m.rigidMotion[i - 1][0], z);
        G.se3e_ij.push_back(pre); G.se3e_ij.push_back(cur); G.se3e_Z.insert(G.se3e_Z.end(), z, z + 12);
        G.se3e_w.push_back(1.0 / (double)c.sigma2_cam); G.se3e_delta.push_back(huber);
      }
      vdo::GraphRow r{slot, (int)m.featSta[i].size() / 2, g.dynamic ? (int)m.featDyn[i].size() / 2 : 0, cur, (int)g.mot.size() / 2, 0};
      if (g.dynamic && i > 0) {                                         // object motion vertices and their smoothing edges (:1551-1600)
        for (size_t j = 1; j < m.rigidMotion[i - 1].size(); ++j) {
          const int v = (int)G.se3.size() / 12;
          G.se3.insert(G.se3.end(), ident, ident + 12);
          if (i > 2) {
            int trace = -1;
            for (size_t k = 0; k < m.rmLabel[i - 2].size(); ++k) if (m.rmLabel[i - 2][k] == m.rmLabel[i - 1][j]) { trace = (int)k; break; }
            if (trace != -1 && G.mot_vid[i - 2][trace] != -1) {
              G.se3e_ij.push_back(G.mot_vid[i - 2][trace]); G.se3e_ij.push_back(v); G.se3e_Z.insert(G.se3e_Z.end(), ident, ident + 12);
              G.se3e_w.push_back(1.0 / (double)c.sigma2_obj_smo); G.se3e_delta.push_back(huber);
            }
          }
          G.mot_vid[i - 1][j] = v;
          g.mot.push_back(m.rmLabel[i - 1][j]); g.mot.push_back(v); ++r.mot_n;
        }
      }
      g.rows.push_back(r);
      for (int kd = 0; kd < 2; ++kd) {                                  // the frame's slots: static features, then dynamic ones
        const int nf = kd ? r.n_dyn : r.n_sta;
        const float *key = (kd ? m.featDyn : m.featSta)[i].data(), *dep = (kd ? m.depDyn : m.depSta)[i].data(), *X = (kd ? m.p3dDyn : m.p3dSta)[i].data();
        for (int j = 0; j < nf; ++j) {
          const float v6[6] = {key[2 * j], key[2 * j + 1], dep[j], X[3 * j], X[3 * j + 1], X[3 * j + 2]};
          g.feat.insert(g.feat.end(), v6, v6 + 6);
        }
      }
      slot += r.n_sta + r.n_dyn;
      pre = cur;
    }
    g.n_slots = slot;
  }
  std::vector<vdo::GraphOutput> out(n);
  TB(vdo::graphs_assemble((void*)(uintptr_t)vdo_ctx_stream(ts[0]->ctx), n, in.data(), out.data()));
  for (int q = 0; q < n; ++q) {
    GraphArrays& G = Gs[q]; vdo::GraphOutput& o = out[q]; const vdo::GraphInput& g = in[q];
    G.pt.swap(o.pt); G.obs_cp.swap(o.obs_cp); G.obs_z.swap(o.obs_z); G.ter_pph.swap(o.ter_pph);
    // static and dynamic observations carry the same weight in both modes (sigma2_3d_sta == sigma2_3d_dyn)
    G.obs_w.assign(G.obs_cp.size() / 2, 1.0 / (double)c.sigma2_3d_sta); G.obs_delta.assign(G.obs_cp.size() / 2, huber);
    G.ter_w.assign(G.ter_pph.size() / 3, 1.0 / (double)c.sigma2_obj); G.ter_delta.assign(G.ter_pph.size() / 3, huber);
    for (size_t r = 0; r < g.rows.size(); ++r) {
      const int i = g.start + (int)r; const vdo::GraphRow& row = g.rows[r];
      std::copy(o.mak.begin() + row.slot, o.mak.begin() + row.slot + row.n_sta, G.makS[i].begin());
      std::copy(o.mak.begin() + row.slot + row.n_sta, o.mak.begin() + row.slot + row.n_sta + row.n_dyn, G.makD[i].begin());
    }
  }
  return VDO_OK;
}
}  // namespace

namespace {
// the factor graph of a PartialBatchOptimization (mode 0) / FullBatchOptimization (mode 1) of the tracker's map, built by build_graphs:
// ingested and finalized.  info (may be NULL): n_se3, n_pt, n_prior, n_se3_edges, n_obs, n_ternary.
int make_map_graph(vdo_tracker* t, const GraphArrays& G, vdo_graph** out, int* info) {
  *out = nullptr;
  const int ns = (int)G.se3.size() / 12, np = (int)G.pt.size() / 3;
  if (info) { info[0] = ns; info[1] = np; info[2] = (int)G.prior_v.size(); info[3] = (int)G.se3e_w.size(); info[4] = (int)G.obs_w.size(); info[5] = (int)G.ter_w.size(); }
  vdo_graph* g = nullptr;
  TK(vdo_graph_create(t->ctx, &g));
  int rc = vdo_graph_set_vertices(g, ns, G.se3.data(), np, G.pt.data());
  if (rc == VDO_OK && !G.prior_v.empty()) rc = vdo_graph_add_edges_se3_prior(g, (int)G.prior_v.size(), G.prior_v.data(), G.prior_Z.data(), G.prior_w.data());
  if (rc == VDO_OK && !G.se3e_w.empty()) rc = vdo_graph_add_edges_se3(g, (int)G.se3e_w.size(), G.se3e_ij.data(), G.se3e_Z.data(), G.se3e_w.data(), G.se3e_delta.data());
  if (rc == VDO_OK && !G.obs_w.empty()) rc = vdo_graph_add_edges_se3_pointxyz(g, (int)G.obs_w.size(), G.obs_cp.data(), G.obs_z.data(), G.obs_w.data(), G.obs_delta.data());
  if (rc == VDO_OK && !G.ter_w.empty()) rc = vdo_graph_add_edges_landmark_motion(g, (int)G.ter_w.size(), G.ter_pph.data(), G.ter_w.data(), G.ter_delta.data());
  if (rc == VDO_OK) rc = vdo_graph_finalize(g);
  if (rc != VDO_OK) { t->err = std::string("batch optimisation failed: ") + vdo_last_error(t->ctx); vdo_graph_destroy(g); return rc; }
  *out = g;
  return VDO_OK;
}
// the reference's iteration cap and gain threshold of the mode
vdo_lm_options map_graph_options(const GraphArrays& G) {
  vdo_lm_options o;
  vdo_lm_options_default(&o); o.max_iterations = G.max_iters; o.gain_threshold = G.gain;
  return o;
}
// refined camera poses, motions and points of an optimised map graph back into the map
int write_back_map_graph(vdo_tracker* t, int mode, const GraphArrays& G, vdo_graph* g) {
  const int ns = (int)G.se3.size() / 12, np = (int)G.pt.size() / 3;
  std::vector<double> se3(12 * (size_t)ns + 12), pt(3 * (size_t)np + 3);
  if (int rc = vdo_graph_get_vertices(g, se3.data(), pt.data())) { t->err = std::string("batch optimisation failed: ") + vdo_last_error(t->ctx); return rc; }
  MapSlice& m = t->map;
  const int N = (int)m.featSta.size();
  // PartialBatchOptimization writes vmCameraPose / vmRigidMotion (src/Optimizer.cc:1058-1101); FullBatchOptimization writes
  // vmCameraPose_RF[i + 1] / vmRigidMotion_RF and leaves the initial estimates alone (:2094-2133); both update the points
  std::vector<M4>& camOut = mode == 1 ? m.cameraPose_RF : m.cameraPose;
  std::vector<std::vector<M4>>& motOut = mode == 1 ? m.rigidMotion_RF : m.rigidMotion;
  for (int i = 0; i < N; ++i) {
    if (G.cam_vid[i] != -1 && (mode == 0 || i > 0)) camOut[i] = from_iso(&se3[12 * (size_t)G.cam_vid[i]]);
    for (size_t j = 0; j < G.makS[i].size(); ++j) if (G.makS[i][j] != -1) for (int k = 0; k < 3; ++k) m.p3dSta[i][3 * j + k] = (float)pt[3 * (size_t)G.makS[i][j] + k];
    for (size_t j = 0; j < G.makD[i].size(); ++j) if (G.makD[i][j] != -1) for (int k = 0; k < 3; ++k) m.p3dDyn[i][3 * j + k] = (float)pt[3 * (size_t)G.makD[i][j] + k];
  }
  for (int i = 0; i + 1 < N; ++i) {
    if (mode == 0) { if (G.cam_vid[i] != -1 && G.cam_vid[i + 1] != -1) m.rigidMotion[i][0] = mul4(inv4(m.cameraPose[i]), m.cameraPose[i + 1]); }   // :1001
    for (size_t j = 1; j < G.mot_vid[i].size(); ++j) if (G.mot_vid[i][j] != -1) motOut[i][j] = from_iso(&se3[12 * (size_t)G.mot_vid[i][j]]);
  }
  return VDO_OK;
}

// The windowed optimisations (PartialBatchOptimization) of every tracker in `due`, solved together by one vdo_graph_optimize_batch.
// Each tracker ends where its own windowed optimisation takes it; a failure leaves the error on the tracker it belongs to.
int windowed_optimize(const Span& due) {
  const int n = (int)due.size();
  std::vector<GraphArrays> G;
  std::vector<vdo_graph*> gs(n, nullptr);
  auto destroy = [&]() { for (vdo_graph* g : gs) vdo_graph_destroy(g); };
  if (int rc = build_graphs(due, false, G)) return rc;
  for (int i = 0; i < n; ++i)
    if (int rc = make_map_graph(due[i], G[i], &gs[i], nullptr)) { destroy(); return rc; }
  const vdo_lm_options o = map_graph_options(G[0]);      // mode 0: the same options for every tracker
  std::vector<vdo_lm_stats> st(n);
  if (int rc = vdo_graph_optimize_batch(gs.data(), n, &o, st.data(), nullptr)) {
    for (vdo_tracker* t : due) t->err = std::string("batch optimisation failed: ") + vdo_last_error(t->ctx);
    destroy();
    return rc;
  }
  for (int i = 0; i < n; ++i) {
    vdo_tracker* t = due[i];
    if (int rc = write_back_map_graph(t, 0, G[i], gs[i])) { destroy(); return rc; }
    t->local_ba_runs += 1; t->local_ba_iters += st[i].iterations;
  }
  destroy();
  return VDO_OK;
}
}  // namespace

// mode 0 = PartialBatchOptimization over the last window_size frames, 1 = FullBatchOptimization.  Builds the graph from the map,
// runs vdo_graph_optimize (opt may be NULL: the reference's iteration cap and gain threshold) and writes the refined camera poses,
// motions and points back into the map.  info (may be NULL): n_se3, n_pt, n_prior, n_se3_edges, n_obs, n_ternary.
extern "C" int vdo_tracker_batch_optimize(vdo_tracker* t, int mode, const vdo_lm_options* opt, vdo_lm_stats* stats, int* info) {
  if (!t || (mode != 0 && mode != 1)) return VDO_ERR_ARG;
  std::vector<GraphArrays> Gs;
  const bool prof = std::getenv("VDO_PROFILE") != nullptr;
  const auto tp0 = std::chrono::steady_clock::now();
  auto lap_ms = [&](const std::chrono::steady_clock::time_point& a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); };
  vdo_graph* g = nullptr;
  if (int rc = build_graphs(Span{t}, mode == 1, Gs)) return rc;
  const GraphArrays& G = Gs[0];
  const double ms_build = lap_ms(tp0);
  TK(make_map_graph(t, G, &g, info));
  const double ms_ingest = lap_ms(tp0);
  const vdo_lm_options o = opt ? *opt : map_graph_options(G);
  vdo_lm_stats st_local;
  int rc = vdo_graph_optimize(g, &o, stats ? stats : &st_local, nullptr);
  if (rc != VDO_OK) t->err = std::string("batch optimisation failed: ") + vdo_last_error(t->ctx);
  const double ms_opt = lap_ms(tp0) - ms_ingest;
  if (rc == VDO_OK) rc = write_back_map_graph(t, mode, G, g);
  vdo_graph_destroy(g);
  if (prof) std::fprintf(stderr, "[vdo_b200] batch_optimize mode %d: %d se3, %d points, %d obs | build %.2f ms | ingest + finalize %.2f | optimise %.2f (%d LM it) | read-back+free %.2f\n", mode,
                         (int)G.se3.size() / 12, (int)G.pt.size() / 3, (int)G.obs_w.size(), ms_build, ms_ingest - ms_build, ms_opt, (stats ? stats : &st_local)->iterations, lap_ms(tp0) - ms_ingest - ms_opt);
  return rc;
}

// vdo_tracker_batch_optimize of n trackers in one call: one graph build over the list, ingest + finalize per tracker, one
// vdo_graph_optimize_batch, write-back per tracker.  Tracker i ends where vdo_tracker_batch_optimize(ts[i], mode, opt, ...) takes it.
// The whole list is checked before anything runs; a refused call changes no tracker.  stats: n entries, info: n x 6 ints (may be NULL).
extern "C" int vdo_tracker_batch_optimize_batch(vdo_tracker* const* ts, int n, int mode, const vdo_lm_options* opt, vdo_lm_stats* stats, int* info) {
  if (!ts || n < 1 || !ts[0]) return VDO_ERR_ARG;
  for (int i = 0; i < n; ++i) {
    vdo_tracker* t = ts[i];
    if (!t) { ts[0]->err = "vdo_tracker_batch_optimize_batch: tracker " + std::to_string(i) + " is NULL"; return VDO_ERR_ARG; }
    for (int j = 0; j < i; ++j)
      if (ts[j] == t) { ts[0]->err = "vdo_tracker_batch_optimize_batch: tracker " + std::to_string(i) + " repeats tracker " + std::to_string(j); return VDO_ERR_ARG; }
    if (t->ctx != ts[0]->ctx) { ts[0]->err = "vdo_tracker_batch_optimize_batch: tracker " + std::to_string(i) + " belongs to another context"; return VDO_ERR_ARG; }
  }
  if (mode != 0 && mode != 1) { ts[0]->err = "vdo_tracker_batch_optimize_batch: mode must be 0 or 1"; return VDO_ERR_ARG; }
  for (int i = 0; i < n; ++i) {
    const int N = (int)ts[i]->map.featSta.size(), window = ts[i]->p.window_size;
    if (N < 2 || (mode == 0 && (window < 2 || N < window))) {
      ts[i]->err = "the map is too short for this optimisation";
      if (i) ts[0]->err = "vdo_tracker_batch_optimize_batch: the map of tracker " + std::to_string(i) + " is too short for this optimisation";
      return VDO_ERR_STATE;
    }
  }
  const bool prof = std::getenv("VDO_PROFILE") != nullptr;
  const auto tp0 = std::chrono::steady_clock::now();
  auto lap_ms = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tp0).count(); };
  const Span list(ts, ts + n);
  std::vector<GraphArrays> G;
  if (int rc = build_graphs(list, mode == 1, G)) return rc;
  const double ms_build = lap_ms();
  std::vector<vdo_graph*> gs(n, nullptr);
  auto destroy = [&]() { for (vdo_graph* g : gs) vdo_graph_destroy(g); };
  for (int i = 0; i < n; ++i)
    if (int rc = make_map_graph(ts[i], G[i], &gs[i], info ? info + 6 * (size_t)i : nullptr)) { destroy(); return rc; }
  const double ms_ingest = lap_ms();
  const vdo_lm_options o = opt ? *opt : map_graph_options(G[0]);      // the mode's options are the same for every tracker
  std::vector<vdo_lm_stats> st_local(stats ? 0 : n);
  if (int rc = vdo_graph_optimize_batch(gs.data(), n, &o, stats ? stats : st_local.data(), nullptr)) {
    for (int i = 0; i < n; ++i) ts[i]->err = std::string("batch optimisation failed: ") + vdo_last_error(ts[i]->ctx);
    destroy();
    return rc;
  }
  const double ms_opt = lap_ms() - ms_ingest;
  for (int i = 0; i < n; ++i)
    if (int rc = write_back_map_graph(ts[i], mode, G[i], gs[i])) { destroy(); return rc; }
  destroy();
  if (prof) std::fprintf(stderr, "[vdo_b200] batch_optimize_batch mode %d, %d trackers | build %.2f ms | ingest + finalize %.2f | optimise %.2f | read-back+free %.2f\n", mode, n,
                         ms_build, ms_ingest - ms_build, ms_opt, lap_ms() - ms_ingest - ms_opt);
  return VDO_OK;
}

// graph arrays of the last build for a mode (parity tests): name in {se3, pt, prior_Z, prior_w, se3e_Z, se3e_w, se3e_delta, obs_z, obs_w, obs_delta, ter_w,
// ter_delta} (f64) or {prior_v, se3e_ij, obs_cp, ter_pph} (i32; out is then an int buffer)
extern "C" int vdo_tracker_graph_export(vdo_tracker* t, int mode, const char* name, void* out, int cap_elems, int* n_elems) {
  if (!t || !name || !n_elems) return VDO_ERR_ARG;
  std::vector<GraphArrays> Gs;
  if (int rc = build_graphs(Span{t}, mode == 1, Gs)) return rc;
  const GraphArrays& G = Gs[0];
  const std::string s(name);
  const std::vector<double>* d = nullptr; const std::vector<int>* iv = nullptr;
  if (s == "se3") d = &G.se3; else if (s == "pt") d = &G.pt; else if (s == "prior_Z") d = &G.prior_Z; else if (s == "prior_w") d = &G.prior_w;
  else if (s == "se3e_Z") d = &G.se3e_Z; else if (s == "se3e_w") d = &G.se3e_w; else if (s == "se3e_delta") d = &G.se3e_delta; else if (s == "obs_z") d = &G.obs_z;
  else if (s == "obs_w") d = &G.obs_w; else if (s == "obs_delta") d = &G.obs_delta; else if (s == "ter_w") d = &G.ter_w; else if (s == "ter_delta") d = &G.ter_delta;
  else if (s == "prior_v") iv = &G.prior_v; else if (s == "se3e_ij") iv = &G.se3e_ij; else if (s == "obs_cp") iv = &G.obs_cp; else if (s == "ter_pph") iv = &G.ter_pph;
  else return VDO_ERR_ARG;
  const size_t n = d ? d->size() : iv->size();
  *n_elems = (int)n;
  if (!out) return VDO_OK;
  if ((int)n > cap_elems) return VDO_ERR_ARG;
  if (n) std::memcpy(out, d ? (const void*)d->data() : (const void*)iv->data(), n * (d ? 8 : 4));
  return VDO_OK;
}

extern "C" int vdo_tracker_tracklets_get(vdo_tracker* t, int kind, const char* name, void* out, int cap_elems, int* n_elems) {
  if (!t || !name || !n_elems || (kind != 0 && kind != 1)) return VDO_ERR_ARG;
  vdo::TrackletDump d;
  if (int rc = vdo::tracklets_read((void*)(uintptr_t)vdo_ctx_stream(t->ctx), t->tracklets, kind, &d)) { t->err = "vdo_tracker_tracklets_get: CUDA error"; return rc; }
  const std::string s(name);
  const std::vector<int>* v = s == "trk" ? &d.trk : s == "pos" ? &d.pos : s == "prev_frame" ? &d.pf : s == "prev_feat" ? &d.pj : s == "len" ? &d.len
                             : s == "head_frame" ? &d.hf : s == "head_feat" ? &d.hj : s == "obj_lab" ? &d.lab : nullptr;
  if (!v) return VDO_ERR_ARG;
  *n_elems = (int)v->size();
  if (!out) return VDO_OK;
  if ((int)v->size() > cap_elems) return VDO_ERR_ARG;
  if (!v->empty()) std::memcpy(out, v->data(), v->size() * 4);
  return VDO_OK;
}

// map read-back: "vmCameraPose" / "vmCameraPose_RF" (N x 16 f32), "vmRigidMotion" / "vmRigidMotion_RF" (all frames concatenated, 16 f32 each),
// "vmRigidCentre" (3 f32 each, same order), "vnRMLabel" (i32, same order), "n_per_frame" (entries per frame, i32), "n_frames"
extern "C" int vdo_tracker_map_get(const vdo_tracker* t, const char* name, void* out, int cap_elems, int* n_elems) {
  if (!t || !name || !n_elems) return VDO_ERR_ARG;
  const std::string s(name);
  std::vector<float> f; std::vector<int> iv; bool is_f = true;
  if (s == "vmCameraPose") for (auto& T : t->map.cameraPose) f.insert(f.end(), T.begin(), T.end());
  else if (s == "vmCameraPose_RF") for (auto& T : t->map.cameraPose_RF) f.insert(f.end(), T.begin(), T.end());
  else if (s == "vmRigidMotion") { for (auto& fr : t->map.rigidMotion) for (auto& T : fr) f.insert(f.end(), T.begin(), T.end()); }
  else if (s == "vmRigidMotion_RF") { for (auto& fr : t->map.rigidMotion_RF) for (auto& T : fr) f.insert(f.end(), T.begin(), T.end()); }
  else if (s == "vmRigidCentre") { for (auto& fr : t->map.rigidCentre) f.insert(f.end(), fr.begin(), fr.end()); }
  else if (s == "n_per_frame") { is_f = false; for (auto& fr : t->map.rmLabel) iv.push_back((int)fr.size()); }
  else if (s == "vp3DPointSta") { for (auto& fr : t->map.p3dSta) f.insert(f.end(), fr.begin(), fr.end()); }      // all frames concatenated, xyz per feature
  else if (s == "vp3DPointDyn") { for (auto& fr : t->map.p3dDyn) f.insert(f.end(), fr.begin(), fr.end()); }
  else if (s == "vnRMLabel") { is_f = false; for (auto& fr : t->map.rmLabel) iv.insert(iv.end(), fr.begin(), fr.end()); }
  else if (s == "n_frames") { is_f = false; iv.push_back((int)t->map.featSta.size()); }
  else return VDO_ERR_ARG;
  const size_t n = is_f ? f.size() : iv.size();
  *n_elems = (int)n;
  if (!out) return VDO_OK;
  if ((int)n > cap_elems) return VDO_ERR_ARG;
  if (n) std::memcpy(out, is_f ? (const void*)f.data() : (const void*)iv.data(), n * 4);
  return VDO_OK;
}
