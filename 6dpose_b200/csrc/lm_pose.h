// lm_pose.h -- internal interface between the detector (linemod_b200.cu) and the on-device pose stage (lm_icp.cu).
//
// The pose stage refines the NMS survivors of k_post_nms where they lie: per-template render crops registered once
// (lm_set_template_renders), then per run k_pose_cloud (box test, back-projection, centroids, voxel keys), a CUB
// segmented radix sort of the voxel keys, k_pose_voxel (voxel means) and the ICP kernels of lm_icp_process_batch
// (k_icp_normals + k_icp_point_to_plane, or k_icp_point_to_point alone), or the particle swarm k_pose_pso in their
// place (LM_POSE_PSO), all on the detector's stream.  A run is a batch
// of frames, and a single frame is a one-frame run of the same stage: the same chunks, outputs, readbacks and finish.
// The host composes result = T * init_base after the copy.  The pose NMS (k_pose_nms, one CTA per frame behind the ICP
// kernel) composes the poses on the device instead, runs the greedy translation NMS of linemod_ros/detect.py over them
// and compacts the kept ones into one output block.  A track run (lm_track, lm_track_batch) is a run whose clouds
// k_track_cloud builds from each object's transformation and the window its model projects to in its own frame, in
// place of k_pose_cloud; with view following on (lm_set_track_views), k_track_views re-chooses each object's template
// and T ahead of it.
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

// A run is one chunk per 1024 survivors, a frame's one chunk.  Slot j of a chunk takes
// survivor rank + j * world, so the launches are sized for ceil(survivors / world) slots; unshared, rank 0 and world 1.
// Shared over the ranks of the peer exchange (lm_peer_share_pose), survivor i (pick order of k_post_nms, the same on
// every rank) is thus refined by rank i % world.  The ICP kernel's SHARE instantiation stores each survivor's result into
// the pose area of every rank's exchange buffer and raises this rank's pose flag there (a verifying stage: the unshared ICP kernel, then k_pose_verify<true>, which
// verifies each survivor on the rank that holds its cloud and stores result and verification); k_pose_collect waits for the
// world flags in this rank's buffer and gathers the results in survivor order into the chunk's outputs, so the host and
// the pose NMS read what the unshared stage leaves.  The pose area: [2 slots][1024 survivors] entries of 192 bytes,
// then [2][LM_MAX_PEERS] int32 pose flags and an int32 ticket, then [2][1024] window records of 40 bytes that only track
// chunks use (pose_share_area_bytes in all).  Each pose exchange -- a shared frame, or one chunk of a shared batch or
// track run -- has its own number on the detector's pose counter.
struct PoseShare {
  uint8_t* base[LM_MAX_PEERS];      // every rank's exchange buffer (peer mappings; this rank's own at [rank])
  uint64_t area_offset;             // byte offset of the pose area in every buffer
  int world, rank;
  int32_t seq;                      // the (first) pose exchange's number: slot = seq & 1; a batch's chunk c is seq + c
  unsigned long long timeout_ns;    // the collector gives up on a peer after this long
  int* abort_flag;                  // the device's abort flag of the exchange: raised on a timeout, honoured at once
};
size_t pose_share_area_bytes();

// Pose verification (lm_set_pose_verify): on adds k_pose_verify behind each chunk's ICP kernel (shared: on the rank that
// refined the survivor, before its result is published); rank_by and min_score steer the pose NMS.
struct PoseVerifyOptions {
  int on, rank_by;
  double inlier_mm, min_score;
};

// The particle swarm of LM_POSE_PSO (lm_set_pose_search, include/linemod_b200.h): P, I, the bounds in metres and
// radians, the cost clamp in mm and the seed of the generator.
struct PoseSearch {
  int particles, iterations;
  double dt, dr, clamp_mm;
  unsigned long long seed;
};
// The defaults (64 particles, 40 iterations, 40 mm, 30 degrees, 20 mm, seed 0).
PoseSearch pose_search_default();
// LM_E_INVALID (with the message) unless the arguments of lm_set_pose_search lie within its limits; else *out.
int pose_search_make(int particles, int iterations, double dt_mm, double dr_deg, double clamp_mm, uint64_t seed, PoseSearch* out);

// What every chunk of a run shares.
struct PoseOptions {
  int srows, scols;           // scene depth size
  int use_scene_cloud, max_iterations;
  int estimation;             // LM_ICP_POINT_TO_PLANE (k_icp_normals + k_icp_point_to_plane), LM_ICP_POINT_TO_POINT or
                              // LM_POSE_PSO (k_pose_pso; no target cloud is built)
  cudaStream_t stream;
  const PoseShare* share;     // null: this rank refines every survivor (LM_POSE_PSO: always)
  PoseVerifyOptions verify;  // zero: off
  PoseSearch search;          // LM_POSE_PSO only
  int views;                  // track runs: view following on (lm_set_track_views), k_track_views ahead of each chunk
  double view_tau;            // its threshold 1 + 2 cos(turn_deg)
};

// One run of the pose stage: a batch of frames (lm_detect_batch, lm_peer_detect_batch), or a frame as a one-frame run
// whose survivor count lives on the device.  Chunk c takes survivors [1024 c, 1024 (c + 1)); with a share it is pose
// exchange share->seq + c.  The stage records the run it last enqueued (share and survivor offsets copied).
struct PoseRun {
  PoseOptions o;
  int n_frames;
  const int64_t* first;       // batch: [n_frames + 1] survivor offsets (host), frame f's at [first[f], first[f + 1]); frame: null
  const int32_t* d_counts;    // frame: [0] = survivors written (device)
  int bound;                  // most survivors of a frame (top_k, or every survivor k_post_nms may write); a frame's launches
                              // are sized for it
  const lm_match* d_surv;     // survivors in pick order (device)
  const uint16_t* d_scene;    // scene depth, srows x scols u16 mm; frame f's at + f * srows * scols
  const float* sK;            // [n_frames][9]
  int pose_nms;               // 1: pose_stage_enqueue_nms follows, so the ICP outputs are not read back
};

// Three calls, in this order, for a frame and a batch alike.
// The run's chunks on o.stream, each with its status block, then the copies the host will need: the status blocks and
// (pose_nms 0) the ICP outputs -- a batch's all, a frame's first window.  Grows the buffers for the run (and synchronises
// then); a batch's were grown by pose_batch_reserve.
int pose_stage_enqueue(lm_pose_stage* s, const PoseRun& run, int64_t* launches);
// Pose NMS behind pose_stage_enqueue on the same stream: one k_pose_nms launch, one CTA per frame.  Also enqueues the copy
// of the frames' heads and their kept poses (a batch's all, a frame's first window).
int pose_stage_enqueue_nms(lm_pose_stage* s, double thr, int64_t* launches);
// After the caller has synchronised the stream: the run's status, then frame f's entries -- its kept poses (pose NMS), or
// every survivor with its pose (outputs as lm_complete_pose) -- after those of frames 0..f-1 in out / R_out + 9k /
// t_out + 3k / residual[k] (out may be null).  surv: the host copy of the survivors (pose_nms 0 only); n: a frame's
// survivor count as read back.  counts[4f .. 4f + 2] = entries, survivors, survivors with a pose; *n_out = entries in all,
// LM_E_CAPACITY beyond cap (both written once the status is clean).  stats4 (may be null): what lm_pose_stats returns.
// Copies and waits again only for a frame's entries beyond its first window.
int pose_stage_finish(lm_pose_stage* s, const lm_match* surv, int64_t n, lm_match* out, double* R_out, double* t_out, float* residual,
                      int64_t cap, int64_t* n_out, int64_t* counts, int64_t* stats4);

// The run last finished.  The stage keeps one record of it, which three getters read:
//   pose_stage_verify (lm_pose_verify, lm_icp_verify): its entries' verification, in entry order.
//   pose_stage_transforms (lm_pose_transforms): its entries' transformations, T_out + 16k, NaN for an entry without a pose.
//   pose_stage_track_templates (lm_track_templates): its entries' templates within their class.
// What each returns, by what last happened on the stage:
//   - a frame or batch without the pose NMS (pose_stage_finish): verify, every survivor's when the run verified, else
//     LM_E_STATE; transforms, every survivor's (NaN where the reference returns early); templates, LM_E_STATE.
//   - a frame or batch with the pose NMS: the same for the kept poses, frame after frame in keep order.  k_pose_nms
//     stores each kept pose's survivor on the device; transforms copies the survivors' ICP outputs on the run's stream.
//   - a track run (pose_stage_track, 0 objects included): verify as above; transforms, every object's (NaN for an entry
//     not TRACKED); templates, every object's (see pose_stage_track_templates).
//   - an lm_icp call, on the ICP handle's own stage (n hypotheses; none: n = 0): verify, when lm_icp_set_verify is on,
//     every hypothesis's (score -1 and zero counts where it returns early), else LM_E_STATE.  Nothing reads its other
//     entries.
//   - a run whose finish failed: LM_E_STATE from all three.  A finish resets the record before it checks the run's
//     status blocks, so every failure past that point (a cloud overflow, a peer that did not publish, a survivor
//     without a render, LM_E_CAPACITY for too small outputs, a CUDA error) leaves it empty.  pose_stage_finish's check of
//     the survivor count against the launch comes before the reset, and a call that fails before it reaches the stage
//     leaves the record as it was.
//   - a run enqueued (pose_stage_enqueue, pose_batch_reserve) and not yet finished: verify still returns the last
//     finished run's verification; transforms and templates return LM_E_STATE.
// LM_E_CAPACITY (with *n) beyond cap.
int pose_stage_verify(const lm_pose_stage* s, float* score, int32_t* counts6, int64_t cap, int64_t* n);

// Slot `slot`'s item `what` of the last chunk enqueued (lm_debug_pose_clouds), after the caller has synchronised the
// stream.  Launches nothing.
int pose_stage_clouds(const lm_pose_stage* s, int slot, int what, void* out, int64_t cap);

// Tracking (lm_track, include/linemod_b200.h): object i of a track run starts from T at template g of the bank, whose
// render is registered.
struct TrackObject {
  int64_t g;
  double T[16];
};
// The scenes of a track run on o.stream: n_frames rows x cols u16 mm frames in the stage's batch scene slots (frame f
// at *d_scene + f * rows * cols; grown, never shrunk, and shared with pose_batch_reserve).  host: n_frames contiguous
// host images, copied at once; else the caller's device planes planes[f] (pitch bytes between rows, LM_DEPTH_U16_MM or
// LM_DEPTH_F32 with scale), converted as lm_bind_images_device converts them, one launch per frame.
int pose_track_scene(lm_pose_stage* s, cudaStream_t st, int n_frames, const uint16_t* host, const void* const* planes, int64_t pitch,
                     int format, float scale, int rows, int cols, const uint16_t** d_scene, int64_t* launches);
// One track run against the scenes of pose_track_scene, o.estimation an ICP: frame f's objects are obj[first[f],
// first[f + 1]) (at most 1024 per frame), its intrinsics sK + 9f; one chunk per 1024 objects, frames straddling chunk
// boundaries.  Then the outputs of lm_track in object order (an entry without the status TRACKED leaves its T, R, t
// untouched and gets residual -1).  Returns once they are on the host; the run is then the stage's last finished run
// (pose_stage_verify, pose_stage_transforms).  lm_track is the one-frame run.  With o.share (lm_peer_track_batch),
// chunk c is pose exchange o.share->seq + c: object i of a chunk is tracked by rank i % world, and its entry and window
// record travel to every rank as a shared batch chunk's entries do.  Allocates nothing once its first chunk is enqueued.
// stats4 (may be null): what lm_pose_stats returns, written once the run succeeded.
int pose_stage_track(lm_pose_stage* s, const PoseOptions& o, int n_frames, const uint16_t* d_scene, const float* sK, const TrackObject* obj,
                     const int64_t* first, int margin, int64_t* launches, double* T_out, double* R_out, double* t_out, float* residual,
                     int32_t* status, int32_t* box, int64_t* stats4);
// LM_E_INVALID unless turn_deg lies in [0, 180) (on only); else *tau = 1 + 2 cos(turn_deg) (libm cos), 0 when off.
int track_view_tau(int on, double turn_deg, double* tau);
// The template of every entry of the run last finished (lm_track_templates), within its class, in entry order: the one
// view following chose for a TRACKED entry, the start's for any other.  When it answers: pose_stage_verify.
int pose_stage_track_templates(const lm_pose_stage* s, int32_t* template_id, int64_t cap, int64_t* n);
// The transformation of every entry of the run last finished (lm_pose_transforms).  When it answers: pose_stage_verify.
int pose_stage_transforms(const lm_pose_stage* s, double* T_out, int64_t cap, int64_t* n);

// A batch's scene and survivor slots: room for n_frames scene depths of frame_pixels each (frame f at d_scene + f *
// frame_pixels) and max_surv survivors, which the caller fills on the stream.  It also uploads the renders and grows
// every buffer the run needs for max_surv survivors, so that the batch allocates no device memory once its frames run.
int pose_batch_reserve(lm_pose_stage* s, cudaStream_t st, int n_frames, int64_t frame_pixels, int64_t max_surv, bool verify,
                       uint16_t** d_scene, lm_match** d_surv);
// Chunks of a run with S survivors.
int pose_batch_chunks(int64_t S);

// An lm_icp call (lm_icp_process_batch, lm_icp_process_batch_device) is a run of the ICP handle's own stage: the same
// chunks (run_chunk, pose_chunk in lm_icp.cu) into the stage's run outputs, the same status check and the stage's
// verification (lm_icp_verify reads it as pose_stage_verify), but from renders it is handed per call instead of
// registered ones.  Its table has one entry per hypothesis, written on the device: k_icp_render_box reduces every
// render's non-zero extent, the host reads the extents back once (n x 16 bytes, one synchronise of the handle's stream),
// then k_icp_render_crop writes each entry (model_box's box, the anchor, K) and its crop.  The read-back sizes what the
// host cannot know before: the crop pool (n x the largest crop a posed hypothesis has) and the clouds' slot stride of the
// chunk buffers (that largest crop).  Sizing for whole renders instead (n x mrows x mcols) would cost a full-frame render
// ~2 x 300 000 points of cloud slots per hypothesis, far more device memory than any crop needs.  Survivor i of the
// call is hypothesis i: class 0, template i, at (x_i, y_i).

// Checks of a caller's device plane and stream (linemod_b200.cu), none of which touches the device: LM_E_INVALID unless
// p is device or managed memory of `device`, rows are at least `row` bytes apart and p and pitch are multiples of elem;
// unless stream is a CUDA stream of `device`.
int check_device_plane(int device, const char* what, const void* p, int64_t pitch, int64_t row, int elem);
int check_device_stream(int device, cudaStream_t stream);

// Checks shared by the detector, the ICP handle and the standalone entry points, LM_E_INVALID with the message unless a
// device plane `what` has a known depth format (and a float one a finite scale > 0), an estimation is known, an inlier
// distance is finite and >= 0.  open_device makes `device` current (LM_E_CUDA without a device, LM_E_INVALID out of range).
int check_depth_format(const char* what, int format, float scale);
int check_estimation(int estimation);
int check_inlier_mm(double inlier_mm);
int open_device(int device);
