// frame_batch.h -- internal batched stages of the per-frame path.  Each entry serves n frames (or point segments), each of its own size,
// with one launch per kernel and one synchronise of the context stream per read-back; the per-element arithmetic is the single-frame
// one, and the public single-frame entries of include/vdo_b200.h are these with n = 1.  All frames of one call share a context.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/vdo_b200.h"

namespace vdo {
// keypoints (x, y) of one frame in level-0 coordinates, in the order vdo_orb_extract returns them
struct OrbXY { std::vector<float> x, y; };
struct OrbJob;   // an extractor with its device outputs
// an image size with one set of ORB settings
struct OrbKey {
  int w, h, nfeatures; float scale_factor; int nlevels, ini_th, min_th;
  bool operator<(const OrbKey& o) const;
  bool operator==(const OrbKey& o) const;
};
// vdo_frame_filter_static / vdo_frame_sample_objects outputs of one frame; kx / ky: the VDO_SAMPLE_KEYS sampled keys of a sampling frame
// (idx indexes them), empty otherwise
struct StaticKeys { std::vector<int> idx; std::vector<float> cx, cy, fu, fv, depth, kx, ky; };
struct ObjSamples { std::vector<int> x, y, label; std::vector<float> cx, cy, fx, fy, depth; };

// frame_kernels.cu
// what vdo_orb_extractor_create refuses in the settings k (VDO_ERR_ARG or VDO_ERR_UNSUPPORTED, the reason in why); VDO_OK otherwise
int orb_key_check(const OrbKey& k, std::string& why);
int frame_check_planes(const vdo_frame* f, const vdo_dev_plane* const planes[4], const bool target[4], std::string& err);
// planes: 4 per frame (image, depth, flow, mask; any may be NULL); enqueued after the work queued so far on `stream`
int frames_ingest_dev(vdo_frame* const* fs, int n, const vdo_dev_plane* const* planes, uint64_t stream);
// synchronises the context stream; VDO_ERR_ARG with *bad = the first frame whose last ingest met an i64 label outside the int32 range
int frames_ingest_wait(vdo_frame* const* fs, int n, int* bad, std::string& err);
int frames_depth_prep(vdo_frame* const* fs, int n, const float* bf, const float* factor);
int frame_writeback_dev(vdo_frame* f, const vdo_dev_plane* depth, const vdo_dev_plane* mask);
// the cached extractor on fs[0]'s stream for n frames whose sizes and ORB settings are keys[i]: one geometry per distinct key, grown to run
// every 64-frame chunk of the n frames in one call; geo[i]: frame i's geometry.  Settings vdo_orb_extractor_create refuses are refused with
// its code before anything is allocated, *bad naming the first frame with them.
int orb_job_for(vdo_frame* const* fs, const OrbKey* keys, int n, OrbJob** out, int* geo, int* bad);
// ORB keypoints of the resident gray images of n frames on J (frame i of geometry geo[i]), in chunks of 64 frames, with one synchronise
int orb_xy_batch(const OrbJob& J, vdo_frame* const* fs, const int* geo, int n, OrbXY* out);
// kx / ky / nk: the keypoints of frame i (option I); th: ThDepthBG per frame.  seed: NULL, or per frame -1 for option I and otherwise the
// uint32 seed of the cv::RNG whose Frame::SampleKeyPoints draws are filtered instead (option II; kx / ky / nk of that frame unused)
int filter_static_batch(vdo_frame* const* fs, int n, const float* const* kx, const float* const* ky, const int* nk, const float* th, const long long* seed,
                        StaticKeys* out);
// cap: per frame, the most samples kept
int sample_objects_batch(vdo_frame* const* fs, int n, const float* th, int step, const int* cap, ObjSamples* out);
// vdo_obj_track_batch_dev's k_ot_flow on `stream` (arguments checked by the caller): the current look-up and the scene flow of the samples in
// out.motion (pair p's at offset p * cap, max_n the most sample positions of a pair); glab: the grouping label (the current label of a valid
// sample, else 0); an i64 current label outside the int32 range sets VDO_OM_PAIR_LABEL_RANGE in pstat
void obj_track_flow_launch(int P, const vdo_dev_plane* depth_cur, const vdo_dev_plane* mask_cur, const int32_t* wh, const float* K, const float* Tcw_last,
                           const float* Tcw_cur, int cap, int max_n, float th_depth_obj, const vdo_obj_track_out& out, int* pstat, int* glab, uint64_t stream);
// point segments [begin[s], begin[s + 1]) with their own poses (16 floats each) and K (4 floats each); arrays concatenated over segments
int scene_flow_batch(vdo_ctx* ctx, int nseg, const int* begin, const float* Tcw_prev, const float* Tcw_cur, const float* K, const float* u_prev,
                     const float* v_prev, const float* z_prev, const float* u_cur, const float* v_cur, const float* z_cur, const int* label_prev,
                     const int* label_cur, float* flow3d, float* Xw_prev, unsigned char* valid);

// tracking_ops.cu: depth and mask label at the truncated pixel of each key of segment s, read from frame fs[s]
int gather_batch(vdo_frame* const* fs, int nseg, const int* begin, const float* keys, float* depth_out, int* mask_out);

// pnp_ransac.cu: vdo_init_model_batch with intrinsics K4 + k_stride * p for problem p (k_stride 0: one K for all, 4: nprob x 4)
int init_model_batch(vdo_ctx* ctx, int nprob, const int* offsets, const float* obj3d, const float* img2d, const float* K4, int k_stride, int iters,
                     double thr, double conf, const float* T_mm, const unsigned char* has_mm, float* T_init, int* n_sub, int* sub_idx, int* info,
                     double* Rt_refit, double* Rt_hyp);

// map_graph.cu: the tracklet tables of one tracker's map, kept on the device and extended frame by frame
struct Tracklets;
Tracklets* tracklets_create();
void tracklets_destroy(Tracklets* t);
bool tracklets_bad(const Tracklets* t);           // an association named a feature the previous frame does not have
int tracklets_frames(const Tracklets* t);
// the frame entering the map of tracker i (associations and labels NULL for its first frame)
struct TrackletFrame { int n_sta, n_dyn; const int *asso_sta, *asso_dyn, *label_dyn; };
// the frames of n trackers, one upload and one launch; synchronises `stream`
int tracklets_push(void* stream, Tracklets* const* t, int n, const TrackletFrame* fr);
// the tables of one kind (0 static, 1 dynamic) as host arrays: per feature (frames concatenated, feat_off per frame) its tracklet, position and
// previous entry (frame, feature); per tracklet its length, head (frame, feature) and ObjLab
struct TrackletDump { std::vector<long long> feat_off; std::vector<int> trk, pos, pf, pj, len, hf, hj, lab; };
int tracklets_read(void* stream, const Tracklets* t, int kind, TrackletDump* out);
// one graph of a graphs_assemble call: frames start .. start + rows.size() - 1 of the map; per frame its first slot, static and dynamic
// feature counts (n_dyn = 0: static only), camera vertex and object motions (label, vertex) pairs mot[2 * mot_begin ..); feat: 6 floats
// per slot (u, v, depth, point x, y, z)
struct GraphRow { int slot, n_sta, n_dyn, cam, mot_begin, mot_n; };
struct GraphInput {
  const Tracklets* tables; int start, n_slots; bool dynamic; float invfx, invfy, cx, cy;
  std::vector<GraphRow> rows; std::vector<float> feat; std::vector<int> mot;
};
// points, observations (camera vertex, point; z), ternary edges (point, point, motion vertex) and the point of every slot (-1: none)
struct GraphOutput { std::vector<double> pt, obs_z; std::vector<int> obs_cp, ter_pph, mak; };
int graphs_assemble(void* stream, int n, const GraphInput* in, GraphOutput* out);
}  // namespace vdo
