// lm_pose.h -- internal interface between the detector (linemod_b200.cu) and the on-device pose stage (lm_icp.cu).
//
// The pose stage refines the NMS survivors of k_post_nms where they lie: per-template render crops registered once
// (lm_set_template_renders), then per frame k_pose_cloud (box test, back-projection, centroids, voxel keys), a CUB
// segmented radix sort of the voxel keys, k_pose_voxel (voxel means) and the ICP kernels of lm_icp_process_batch
// (k_icp_normals + k_icp_point_to_plane, or k_icp_point_to_point alone), all on the detector's stream.  The host composes result = T * init_base after the copy.
// The pose NMS (k_pose_nms, one CTA behind k_icp_point_to_plane) composes the poses on the device instead, runs the
// greedy translation NMS of linemod_ros/detect.py over them and compacts the kept ones into one output block.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "linemod_b200.h"

struct lm_pose_stage;

lm_pose_stage* pose_stage_create();
void pose_stage_destroy(lm_pose_stage* s);
// The bank changed: every registered render is dropped.
void pose_stage_clear(lm_pose_stage* s);
// Templates [first, first + n) of a bank of G templates (class_begin[n_classes + 1]).
int pose_stage_register(lm_pose_stage* s, const int32_t* class_begin, int n_classes, int64_t first, int64_t n,
                        const uint16_t* const* depths, int rows, int cols, const float* K, const float* R, const float* t);
// Every template of the selection has a render.
bool pose_stage_covers(const lm_pose_stage* s, const int32_t* sel, int64_t n_sel);

// A frame's pose stage is one chunk of survivors, a batch's one chunk per 1024 survivors.  Slot j of a chunk takes
// survivor rank + j * world, so the launches are sized for ceil(survivors / world) slots; unshared, rank 0 and world 1.
// Shared over the ranks of the peer exchange (lm_peer_share_pose), survivor i (pick order of k_post_nms, the same on
// every rank) is thus refined by rank i % world.  The ICP kernel's SHARE instantiation stores each survivor's result into
// the pose area of every rank's exchange buffer and raises this rank's pose flag there; k_pose_collect waits for the
// world flags in this rank's buffer and gathers the results in survivor order into the chunk's outputs, so the host and
// the pose NMS read what the unshared stage leaves.  The pose area: [2 slots][1024 survivors] entries of 160 bytes,
// then [2][LM_MAX_PEERS] int32 pose flags and an int32 ticket (pose_share_area_bytes in all).  Each pose exchange -- a
// shared frame, or one chunk of a shared batch -- has its own number on the detector's pose counter.
struct PoseShare {
  uint8_t* base[LM_MAX_PEERS];      // every rank's exchange buffer (peer mappings; this rank's own at [rank])
  uint64_t area_offset;             // byte offset of the pose area in every buffer
  int world, rank;
  int32_t seq;                      // the (first) pose exchange's number: slot = seq & 1; a batch's chunk c is seq + c
  unsigned long long timeout_ns;    // the collector gives up on a peer after this long
  int* abort_flag;                  // the device's abort flag of the exchange: raised on a timeout, honoured at once
};
size_t pose_share_area_bytes();

// What a frame's and a batch's pose stage share.
struct PoseOptions {
  int srows, scols;           // scene depth size
  int use_scene_cloud, max_iterations;
  int estimation;             // LM_ICP_POINT_TO_PLANE (k_icp_normals + k_icp_point_to_plane) or LM_ICP_POINT_TO_POINT
  cudaStream_t stream;
  const PoseShare* share;     // null: this rank refines every survivor
};
struct PoseEnqueue {
  PoseOptions o;
  const lm_match* d_surv;     // survivors in pick order (k_post_nms output)
  const int32_t* d_counts;    // [0] = survivors written
  const uint16_t* d_scene;    // scene depth, srows x scols u16 mm
  float sK[9];
  int bound;                  // survivors the launches are sized for (top_k, or every survivor k_post_nms may write)
};
int pose_stage_enqueue(lm_pose_stage* s, const PoseEnqueue& e, int64_t* launches);
// After pose_stage_finish / pose_stage_finish_nms of a frame with n survivors: what lm_pose_stats returns (survivors,
// hypotheses this rank refined, launches of the stage, 1 if shared).
void pose_stage_stats(const lm_pose_stage* s, int64_t n, int64_t* out4);
// After the stream has been synchronised: surv[n] are the survivors (host copy).  Outputs as lm_icp_process_batch.
int pose_stage_finish(lm_pose_stage* s, cudaStream_t st, const lm_match* surv, int64_t n, double* R_out, double* t_out,
                      float* residual);

// Pose NMS behind pose_stage_enqueue on the same stream: d_surv / d_counts as given to it.  Also enqueues the copy of
// the output block's header and first entries.
int pose_stage_enqueue_nms(lm_pose_stage* s, const lm_match* d_surv, const int32_t* d_counts, double thr, cudaStream_t st,
                           int64_t* launches);
// After the stream has been synchronised: the kept poses in keep order (outputs as lm_complete_detect).
int pose_stage_finish_nms(lm_pose_stage* s, cudaStream_t st, lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap,
                          int64_t* n_out, int64_t* n_survivors, int64_t* n_posed);

// A batch of frames through one pose stage (lm_detect_batch, lm_peer_detect_batch).  pose_batch_reserve returns room for
// n_frames scene depths of frame_pixels each (frame f at d_scene + f * frame_pixels) and max_surv survivors, which the
// caller fills on the stream: frame f's survivors at [first[f], first[f + 1]).  It also uploads the renders and grows
// every buffer pose_batch_run needs for max_surv survivors, so that the batch allocates no device memory once its frames run.
int pose_batch_reserve(lm_pose_stage* s, cudaStream_t st, int n_frames, int64_t frame_pixels, int64_t max_surv, uint16_t** d_scene,
                       lm_match** d_surv);
// Chunks of the pose stage of a batch with S survivors (each of at most 1024 slots).
int pose_batch_chunks(int64_t S);
struct PoseBatch {
  PoseOptions o;              // shared: chunk c is pose exchange o.share->seq + c
  int n_frames;
  const int64_t* first;       // [n_frames + 1] survivor offsets (host)
  const lm_match* surv;       // host copy of the survivors (pose_nms == 0 only)
  const float* sK;            // [n_frames][9]
  int pose_nms;               // 1: the pose NMS per frame (one CTA each), 0: the host composes the poses
  double thr;
};
// The pose stage over every survivor of the batch in chunks of at most 1024 survivors, then (pose_nms) one pose NMS
// launch for all frames; waits.  posed[f] / kept[f]: frame f's survivors with a pose, and its entries (kept poses, or
// every survivor without the pose NMS).  stats4 (may be null): what lm_pose_stats returns for the batch.
int pose_batch_run(lm_pose_stage* s, const PoseBatch& b, int64_t* launches, int64_t* posed, int64_t* kept, int64_t* stats4);
// Frame f's kept[f] entries after pose_batch_run, outputs as lm_complete_detect (pose_nms) or lm_complete_pose.
void pose_batch_frame(const lm_pose_stage* s, const PoseBatch& b, int f, lm_match* out, double* R_out, double* t_out, float* residual);
