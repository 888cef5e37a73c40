/* linemod_b200.h -- C-ABI of the H100-native LINEMOD match + ICP pose-refinement path.
 *
 * This is the drop-in boundary: the entry points below are what a binding of the reference's
 * `linemodLevelup_pybind` module (reference: linemodLevelup/pybind11.cpp:7-35) binds instead of the
 * C++ classes `linemodLevelup::Detector` (linemodLevelup/linemodLevelup.h:264-375) and `poseRefine`
 * (linemodLevelup.h:8-19).  Plain pointers and sizes only; no torch / OpenCV types.  All calls are
 * blocking; one in-flight call per handle.  Every function returns 0 on success or a negative
 * LM_E_* code, with a human-readable message available from lm_last_error() (thread-local).
 * There is NO CPU fallback: without a CUDA device lm_create() fails.
 *
 * Citations "LL.cpp:n" = linemodLevelup/linemodLevelup.cpp of meiqua/6DPose @ 619be57.
 */
#ifndef LINEMOD_B200_H
#define LINEMOD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LM_OK 0
#define LM_E_INVALID (-1) /* bad argument / a CV_Assert of the reference would fire */
#define LM_E_CUDA (-2)    /* CUDA runtime error */
#define LM_E_STATE (-3)   /* call order (no bank / no frame uploaded) */
#define LM_E_CAPACITY (-4)

#define LM_MAX_LEVELS 4
#define LM_MAX_MODALITIES 2

typedef struct lm_detector lm_detector; /* replaces linemodLevelup::Detector, LL.h:264 */

/* One detection.  Replaces linemodLevelup::Match (LL.h:225-258); class_index indexes the class list
 * given to lm_load_bank (the host shim maps it back to the class_id string). */
typedef struct lm_match {
  int32_t x, y;
  float similarity;
  int32_t class_index;
  int32_t template_id;
} lm_match;

/* Pre-finish record of a candidate that survived refinement (LL.cpp:1855-1938), produced by the GPU
 * stages.  `work` indexes the matched-template sequence of this call (global across shards); `seq` is
 * the candidate's index in its shard's pre-sort order (template order, then ascending coarse cell;
 * LL.cpp:1797-1939).  Records are appended unordered; sorting by (work, seq) restores the reference's
 * pre-sort order.  16 bytes: the all-gather payload. */
typedef struct lm_record {
  int16_t x, y;
  float similarity;
  int32_t work;
  int32_t seq;
} lm_record;

/* A result block in device memory = this header followed by `capacity` lm_record slots. */
typedef struct lm_result_header {
  int32_t count;             /* records kept (may exceed capacity: only `capacity` were stored) */
  int32_t coarse_candidates; /* candidates that passed the coarse threshold (LL.cpp:1836-1852) */
  int32_t capacity;
  int32_t shard;
} lm_result_header;

const char* lm_last_error(void);

/* Detector(num_features, T) / Detector(T) / Detector(): LL.cpp:1663-1692.  `T` has n_levels entries
 * (sampling step per pyramid level).  `device` is the CUDA ordinal; -1 creates a host-only handle that
 * can hold a bank, compute selections / shard ranges and run lm_finish (the merge step of a multi-GPU
 * match) but refuses every GPU stage with LM_E_STATE. */
int lm_create(int device, int n_levels, const int* T, lm_detector** out);
void lm_destroy(lm_detector* d);

/* Replace the template bank (class_templates, LL.h:361-362).  Flattened:
 *   class_begin[n_classes+1]  global template ranges per class, in the caller's class order
 *   tmeta[G][n_slots][4]      {width, height, feat_begin, feat_count}; n_slots = n_levels*2, slot =
 *                             level*2 + modality (LL.cpp:1964)
 *   feats[n_feats][3]         {x, y, label} (struct Feature, LL.h:23-34)
 * Fails with LM_E_INVALID on label outside [0,8), negative coordinates, > 8191 features in a
 * template (CV_Assert LL.cpp:1291), more than 4096 classes or more than 2^20 templates in a class (the
 * box NMS's canonical key, lm_enqueue_post). */
int lm_load_bank(lm_detector* d, int n_classes, const int32_t* class_begin, int n_slots, const int32_t* tmeta,
                 const int32_t* feats, int64_t n_feats);

/* Select which templates a call matches, in order: the concatenation of the given classes' template
 * ranges (Detector::match's class_ids loop, LL.cpp:1753-1769), then the slice [shard_index/shard_count)
 * of that sequence (contiguous, balanced by features x positions) -- the multi-GPU template shard.
 * n_classes_sel < 0 selects all classes in bank order. */
int lm_select(lm_detector* d, const int32_t* class_sel, int n_classes_sel, int shard_index, int shard_count);
/* Same with the shard layout chosen: LM_SHARD_CONTIGUOUS (lm_select's: one block of the sequence per shard) or
 * LM_SHARD_INTERLEAVED (shard r takes elements r, r + N, r + 2N, ...: neighbouring templates -- views and in-plane
 * variants that pass or fail together -- are dealt round the ranks, which evens out the candidate load).  Records
 * carry the global index in the selected sequence either way, so lm_finish is unchanged. */
#define LM_SHARD_CONTIGUOUS 0
#define LM_SHARD_INTERLEAVED 1
int lm_select_layout(lm_detector* d, const int32_t* class_sel, int n_classes_sel, int shard_index, int shard_count, int layout);
/* Index of this shard's first element inside the selected sequence and the shard's length (contiguous layout: the
 * shard is [begin, begin + count); interleaved: begin + k * shard_count, k < count). */
int lm_shard_range(lm_detector* d, int64_t* begin, int64_t* count);

/* Frame upload: quantized one-hot label images (output of QuantizedPyramid::quantize, LL.cpp:583-587,
 * 882-886) for every (level, modality), host pointers, index level*2+modality; rows/cols per level.
 * Fails where the reference asserts: rows%T, cols%T (LL.cpp:1217-1218), rows*cols%16 (LL.cpp:1136). */
int lm_upload_quantized(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols);

/* Same, but the label images already live in device memory (borrowed: they must stay valid and
 * unchanged until the stages enqueued on them have completed).  No copy is made. */
int lm_bind_quantized_device(lm_detector* d, const uint8_t* const* d_quantized, const int* rows, const int* cols);

/* Frame upload from the RAW images, quantization front-end on the GPU: rgb u8 rows x cols x 3, depth u16
 * rows x cols (mm), optional masks u8 rows x cols (255 = valid, NULL = none) -- the arguments of
 * Detector::match (LL.cpp:1702-1719).  Produces the same label images as the reference's
 * ColorGradientPyramid / DepthNormalPyramid (LL.cpp:350-505, 557-587, 729-886; parameters of
 * Detector(num_features, T): weak threshold 10, distance 2000 mm, difference 50 mm). */
int lm_upload_images(lm_detector* d, const uint8_t* rgb, const uint16_t* depth, int rows, int cols,
                     const uint8_t* mask_color, const uint8_t* mask_depth);

/* lm_upload_images for a frame already in device memory (a GPU decoder's output, a depth network's, a camera rig's
 * device buffers): one launch of k_fe_ingest copies it into the front-end's buffers, then the same front-end runs.
 *   Layout     rgb u8 rows x cols x 3, depth and the masks one element per pixel; pixels packed within a row, rows
 *              rgb_pitch / depth_pitch / mask_pitch BYTES apart (a crop view of a larger image is fine).  Every pointer
 *              is device or managed memory of the handle's device.  mask_color / mask_depth NULL: none (255 = valid).
 *   Depth      LM_DEPTH_U16_MM: u16 mm, copied as is.  LM_DEPTH_F32: float32 d, stored as v = d * depth_scale rounded
 *              once in float32, truncated to u16 for 0 <= v < 65536 -- for every such value bit for bit the reference
 *              driver's host conversion (depth *= depth_scale; depth.astype(np.uint16), linemod_and_levelup_test.py:
 *              315-317), i.e. (d_f32 * np.float32(depth_scale)).astype(np.uint16).  Deviation: NaN, negative, infinite
 *              and >= 65536 products, where numpy's cast is platform-defined, are 0 (no depth).
 *   Ordering   no host synchronise.  The call records an event on `stream` (a cudaStream_t; NULL = the legacy default
 *              stream) and the handle's stream waits on it, so what the producer enqueued on `stream` before the call
 *              has completed before the ingest reads the frame; after the ingest the handle records a second event and
 *              `stream` waits on it, so the caller's next write to the frame is ordered after the read.  The borrow
 *              ends when the ingest has run, not at lm_complete*.
 * A bound frame is a frame with depth exactly like an uploaded one: lm_enqueue (depth gate included), lm_enqueue_post,
 * lm_enqueue_pose and lm_enqueue_pose_nms take it unchanged, and lm_bind_images_device + lm_run + lm_fetch_records +
 * lm_finish is lm_match_images.  Beyond first use at a frame size (buffers, the normal table) nothing from the bind to
 * lm_enqueue_pose_nms synchronises the host after lm_prepare.
 * LM_E_INVALID, before any device work, for a null rgb or depth; a stream of another device; a pointer that is not device
 * or managed memory of the handle's device; a pitch shorter than a row; a depth pointer or pitch not aligned to its element size; an unknown
 * depth_format; a non-finite or non-positive depth_scale with LM_DEPTH_F32; and lm_upload_images' frame-size rules. */
#define LM_DEPTH_U16_MM 0
#define LM_DEPTH_F32 1
int lm_bind_images_device(lm_detector* d, const uint8_t* rgb, int64_t rgb_pitch, const void* depth, int64_t depth_pitch,
                          int depth_format, float depth_scale, int rows, int cols, const uint8_t* mask_color,
                          const uint8_t* mask_depth, int64_t mask_pitch, void* stream);

/* GPU stages on the uploaded frame: spread/response/linearize (LL.cpp:1094-1243), coarse similarity
 * scan + threshold (LL.cpp:1284-1354, 1836-1852), local 16x16 refinement up the pyramid
 * (LL.cpp:1366-1428, 1855-1938).  Leaves the ordered candidate records in device memory. */
int lm_run(lm_detector* d, float threshold);
/* lm_run split in two for pipelining: lm_enqueue issues every stage on the detector's stream and
 * returns without synchronising; lm_complete waits.  Every completion (lm_complete, lm_complete_post,
 * lm_complete_pose, lm_complete_detect, each frame of a batch) settles an overflow the same way: when the
 * frame passed more coarse candidates than the candidate list holds, or kept more records than the result
 * block holds, both grow and the frame is replayed from the refinement on, with every later stage enqueued
 * for it (box NMS, pose stage, pose NMS), in up to three passes.  A caller's result block
 * (lm_set_result_buffer) does not grow: LM_E_CAPACITY when the records outgrow it.  Neither grows with a
 * connected peer exchange: LM_E_CAPACITY. */
int lm_enqueue(lm_detector* d, float threshold);
int lm_complete(lm_detector* d);
/* Everything lm_enqueue does lazily on a new bank / selection / frame size (feature addresses for the frame size,
 * shard work lists, run buffers, the depth gate's tables), done now, with lm_enqueue's checks: the first lm_enqueue
 * afterwards only launches.  Needs a frame uploaded or bound (for its size).  SPMD callers use it so that no rank's
 * first frame lags the others'. */
int lm_prepare(lm_detector* d);
/* The bit-sliced coarse scan's plan for one shard, as lm_prepare builds it (host only, no device needed).  words[i] =
 * position words of item i (ceil(P / 32) clamped to 1..nwords; P = template_positions at the lowest level).
 *   table[n_entries][2]  (item, round) for each of the n_full full tasks (32 consecutive words of one item), items in
 *                        order; then (item, word) per lane of the remainder tasks: the n_rem remainder words of all
 *                        items end to end, 32 per task, the last task padded with copies of the last word.  table ==
 *                        null: only the counts and shape; cap < n_entries: LM_E_CAPACITY (counts still written)
 *   shape[4]             tasks, warps per team, warps per CTA, CTAs of the launch on sm_count SMs with plane_bytes of
 *                        bit-planes; CTA b takes tasks b, b + CTAs, b + 2 CTAs, ... */
int lm_coarse_tasks(const int32_t* words, int64_t n_items, int sm_count, int64_t plane_bytes, int32_t* table, int64_t cap,
                    int64_t* n_entries, int64_t* n_full, int64_t* n_rem, int32_t* shape);
/* The bit-sliced coarse scan's feature descriptors, as lm_prepare builds them (host only, no device needed), for a bank
 * in lm_load_bank's layout (feats[n][3] = x, y, label; tmeta[G][S][4] = width, height, first feature, count) at the
 * lowest level: slots slot_low .. slot_low + M - 1, sampling step T, level size rows x cols.  One word per feature:
 *   bits 0-4 bit shift inside the window's first word, bit 5 label 0, bit 6 label 7, bits 7-31 word offset of the
 *   window in the bit-plane buffer ((m * 8 + label) * lbw + word inside the label block, lbw = words per label block).
 * Features outside the level and padding hold *zero (a window that reads zeros).  A template's features, modalities in
 * order, lie end to end from info[g][0] (info[g][1] of them), padded to a multiple of 32.  fits[g] = 0: the word offsets
 * do not fit in 25 bits; the template has no descriptors and goes to the byte-wise coarse scan.  desc == null: only
 * n_desc, info, fits and zero; cap < n_desc: LM_E_CAPACITY. */
int lm_coarse_descriptors(const int32_t* feats, const int32_t* tmeta, int G, int S, int M, int slot_low, int T, int rows,
                          int cols, uint32_t* desc, int64_t cap, int64_t* n_desc, int32_t* info, uint8_t* fits,
                          uint32_t* zero);

/* Result block of the stages: by default an internal device buffer that grows on demand.  A caller
 * that wants the block in its own device memory (e.g. the send buffer of an NCCL all-gather) sets it
 * here; capacity is in records, the block is sizeof(lm_result_header) + capacity*sizeof(lm_record)
 * bytes.  d_block = NULL returns to the internal buffer. */
int lm_set_result_buffer(lm_detector* d, void* d_block, int64_t capacity_records);
int lm_device_result(lm_detector* d, void** d_block, int64_t* capacity_records);

/* Multi-GPU exchange fused into the refinement kernels (one process per GPU, template shards from
 * lm_select; the reference has no counterpart: its template loop is serial, LL.cpp:1797).  Every rank
 * owns an exchange buffer of 2 frame slots x `world` result blocks; once connected, the exact refinement
 * kernel (k_refine_bits / k_refine) stores every kept record into the block [slot][rank] of EVERY rank's buffer with peer stores over NVLink (local
 * stores for itself), its last CTA publishes the block header and a frame sequence flag, and a collector
 * kernel on the same stream waits for all `world` flags and packs the blocks into this handle's result
 * block.  lm_complete / lm_fetch_records / lm_device_result then see the kept records of ALL shards: no
 * separate collective, no host round trip between refinement and exchange.  All ranks must enqueue the
 * same frames in the same order (SPMD); capacity_records is per rank and per frame.  A collector that waits
 * longer than LINEMOD_B200_PEER_TIMEOUT_MS (default 1000) for a peer fails the frame (LM_E_STATE from
 * lm_complete) and raises a per-device abort flag every later collector honours at once; lm_peer_export
 * clears it.
 *   lm_peer_export        allocate the buffer, return its CUDA IPC handle (LM_PEER_HANDLE_BYTES bytes)
 *   lm_peer_connect       handles[world][LM_PEER_HANDLE_BYTES] of all ranks (own entry ignored)
 *   lm_peer_connect_local same, for handles living in ONE process: bases[world] from lm_peer_base
 *   lm_peer_disconnect    back to the single-GPU result block (callers barrier first) */
#define LM_PEER_HANDLE_BYTES 64
#define LM_MAX_PEERS 16
int lm_peer_export(lm_detector* d, int world, int64_t capacity_records, uint8_t* handle_out);
int lm_peer_base(lm_detector* d, void** base);
int lm_peer_connect(lm_detector* d, int rank, int world, const uint8_t* handles);
int lm_peer_connect_local(lm_detector* d, int rank, int world, void* const* bases);
int lm_peer_disconnect(lm_detector* d);

/* The pose stage shared over the ranks of the connected exchange (off by default).  lm_enqueue_pose of a frame then
 * refines only this rank's share of the box-NMS survivors: survivor i (pick order of the box NMS, the same on every
 * rank) is refined by rank i % world, so rank r's launches are sized for ceil(bound / world) slots and slot j takes
 * survivor r + j * world (bound = top_k, or 1024 for every survivor).  The survivor count is read on the device: no host
 * synchronisation.  The ICP kernel stores each result into the pose area of every rank's exchange buffer over NVLink and
 * its last CTA raises this rank's pose flag there; a collector kernel behind it waits for all `world` flags and gathers
 * the results in survivor order.  lm_complete_pose and lm_complete_detect then return on EVERY rank exactly what the
 * unshared stage returns, bit for bit (R, t, residual, -1 and untouched R / t on the early return of LL.cpp:52-55, NaN
 * patterns, the pose NMS's keep order and counts): each survivor's ICP is one deterministic job wherever it runs.  A
 * shared frame's pose stage is 6 launches (5 unshared), whatever the survivor count; 5 (4) with LM_ICP_POINT_TO_POINT.
 *   lm_peer_share_pose  on != 0 turns sharing on.  LM_E_STATE on a handle without a connected exchange.  A promise the
 *                       caller makes for every rank: every rank of the exchange sets the same value before its next
 *                       frame, and while it is on every rank runs the pose stage of every frame (a rank that runs the
 *                       match alone leaves its peers waiting).  Likewise every rank sets the same lm_set_pose_estimation
 *                       before its next frame: a shared frame's survivors are refined with the estimation of the rank
 *                       that owns them.  lm_peer_disconnect turns it off.  Ranks that are
 *                       handles of ONE process on ONE device: a pose stage that uploads renders or grows its buffers
 *                       (the first frame, a larger top_k) frees device memory, which waits for the whole device -- a
 *                       peer's pose collector included -- so run such a frame unshared first.
 * A peer whose poses do not arrive within LINEMOD_B200_PEER_TIMEOUT_MS fails the frame with LM_E_STATE (the message names
 * the pose exchange) and raises the device's abort flag of the exchange, as the record collector does.
 * Each pose exchange -- a shared frame, or one chunk of a shared lm_peer_detect_batch or lm_peer_track_batch -- takes
 * the next number of the handle's pose counter (reset by lm_peer_export), and consecutive exchanges alternate between
 * the two slots of the pose area.  lm_detect_batch and the track calls still refuse a connected exchange;
 * lm_peer_detect_batch and lm_peer_track_batch are their connected forms. */
int lm_peer_share_pose(lm_detector* d, int on);

/* Copy the kept records of the last completed run to the host, sorted by (work, seq). */
int lm_fetch_records(lm_detector* d, lm_record* out, int64_t cap, int64_t* n_out);

/* Host finisher: order records by (work, seq), map work -> (class_index, template_id) for the current
 * selection (work indices are global in the selected sequence), then the reference's
 * std::sort + std::unique (LL.cpp:1772-1774).  `records` may be the concatenation of all shards'
 * records in any order. */
int lm_finish(lm_detector* d, const lm_record* records, int64_t n, lm_match* out, int64_t cap, int64_t* n_out);

/* Post-match stage on the device (SURVEY.md 8f-3).  The reference's callers turn the match list into boxes
 * (x, y, x+width, y+height, similarity), run a greedy NMS at IoU 0.5 and refine the first three survivors
 * with poseRefine (linemod_and_levelup_test.py:34-61, 325-367; linemod_ros/detect.py:41-81, 94-134).  Here
 * the NMS runs on the device behind the refinement kernel, on the kept records where they lie (all shards'
 * records with a connected peer exchange), and only the top_k survivors are copied to the host.
 *   lm_set_boxes      wh[n_templates][2]: box size per template in bank order (the drivers take it from their
 *                     template-info files); NULL / never called = Template::width/height of level 0 (LL.h:36-45)
 *   lm_enqueue_post   after lm_enqueue, same stream; top_k <= 0 = every survivor (at most 1024)
 *   lm_complete_post  waits; out[n_out] in pick order (best first); n_records = kept records the NMS saw.  A frame
 *                     that overflowed is grown and replayed first (lm_complete)
 *   lm_match_top      lm_upload_quantized + lm_enqueue + lm_enqueue_post + lm_complete_post
 * The survivors are those of the drivers' pipeline, nms() on the finished match list (after std::sort + std::unique,
 * LL.cpp:1772-1774), restated without the unstable sorts: the kept records are put in the canonical order --
 * similarity descending, then template_id, class, y, x ascending (equal similarities, which the reference leaves to an
 * unstable sort, taken in that order) -- and each record equal to its predecessor there in (x, y, similarity, class)
 * is dropped, as std::unique drops it (Match::operator== ignores template_id).  Then the greedy NMS in that order,
 * IoU as in the reference's nms(): float64, "+1" pixel convention, suppressed when ovr > threshold.  A threshold
 * >= 1 suppresses nothing: the survivors are every record the canonical dedupe keeps, in pick order; there the
 * reference's own list also keeps duplicates that its sort's tie permutation did not make adjacent.  Banks of more
 * than 4096 classes or 2^20 templates per class are refused by lm_load_bank (the canonical key's widths). */
int lm_set_boxes(lm_detector* d, const int32_t* wh, int64_t n_templates);
int lm_enqueue_post(lm_detector* d, double iou_threshold, int top_k);
int lm_complete_post(lm_detector* d, lm_match* out, int64_t cap, int64_t* n_out, int64_t* n_records);
int lm_match_top(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols, float threshold,
                 double iou_threshold, int top_k, lm_match* out, int64_t cap, int64_t* n_out, int64_t* n_records);

/* Pose stage on the device: poseRefine::process for every NMS survivor, behind lm_enqueue_post on the same stream.
 * The drivers refine each survivor against render(model, K, R, t) of the matched template's info entry
 * (linemod_and_levelup_test.py:351-367; linemod_ros/detect.py:113-130) -- a constant of the template, registered once.
 * Registration keeps what poseRefine derives from the full render: the 9x9-dilated box of its non-zero pixels
 * (LL.cpp:43-50), the render cropped to that box and the anchor depth render[rows/2][cols/2]; only those, and K, go to
 * the device.  Per frame the device builds the clouds (scan-compacted in row-major order), the centroids and the
 * voxel down-sampling (CUB segmented radix sort + voxel means) and runs the ICP kernels; only the survivors and their
 * poses come back.  Clouds, initial guesses, R, t and residual are bit-identical to lm_icp_process_batch on the same
 * survivors and renders, NaN patterns included (lm_debug_pose_clouds shows the clouds); both fail with LM_E_INVALID where
 * a cloud spans more than 2^21 voxels of 2.5 mm along an axis (a tiny, zero or non-finite K).
 *   lm_set_template_renders  templates [first, first+n) of the bank (bank order, as lm_set_boxes); depths[i] is
 *                            rows x cols u16 mm, K + 9i / R + 9i row-major f32, t + 3i f32 mm.  May be called in
 *                            several ranges.  LM_E_INVALID for a render without a non-zero pixel or a range outside
 *                            the bank.  Loading another bank drops the renders.
 *   lm_enqueue_pose          after lm_enqueue_post, same stream, no host synchronisation.  The scene depth is that of
 *                            the frame lm_upload_images uploaded; sceneK is 9 f32.  LM_E_STATE without renders for
 *                            every selected template, for a frame from lm_upload_quantized / lm_bind_quantized_device
 *                            (no depth), or without lm_enqueue_post.  Buffers are sized for top_k survivors (every
 *                            survivor: 1024) times the largest registered crop.  The first call after a registration
 *                            or with a larger top_k uploads the crops / grows the buffers and synchronises the stream:
 *                            with a connected peer exchange, every rank enqueues its match before any rank enqueues
 *                            the post and pose stages.
 *   lm_complete_pose         waits.  out[n_out] are the survivors in pick order (as lm_complete_post); R_out + 9i,
 *                            t_out + 3i, residual[i] are lm_icp_process_batch's outputs for survivor i (residual -1 and
 *                            R/t untouched on the early return of LL.cpp:52-55).  A frame that overflowed is grown and
 *                            replayed first, pose stage included (lm_complete). */
int lm_set_template_renders(lm_detector* d, int64_t first, int64_t n, const uint16_t* const* depths, int rows, int cols,
                            const float* K, const float* R, const float* t);
int lm_enqueue_pose(lm_detector* d, const float* sceneK, int max_iterations, int use_scene_cloud);
int lm_complete_pose(lm_detector* d, lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap,
                     int64_t* n_out, int64_t* n_records);

/* The ICP's estimation step: the two branches of poseRefine::process behind USE_OPEN3D_P2PL (LL.cpp:122-135).  Both run
 * the same RegistrationICP loop (1 cm radius, the convergence test, max_iterations); only the update of each pass differs.
 *   POINT_TO_PLANE  TransformationEstimationPointToPlane against EstimateNormals' normals of the target (KNN 30): one
 *                   normals launch and one ICP launch
 *   POINT_TO_POINT  TransformationEstimationPointToPoint without scaling: Eigen's umeyama over the correspondences, a
 *                   closed-form rigid fit; no normals, so one launch.  It may need more passes to converge.
 * lm_set_pose_estimation sets it for the detector's next lm_enqueue_pose, lm_detect_batch and lm_peer_detect_batch; a frame
 * keeps the estimation it was enqueued with (the pose stage rerun after a result-block retry included).  No device work.
 * A frame's pose stage is then 4 launches (5 shared), a batch chunk likewise.  With a connected peer exchange, setting the
 * same value on every rank is the caller's promise, as with lm_peer_share_pose.  LM_POSE_PSO (below) replaces the ICP
 * with a particle swarm.  LM_E_INVALID for any other value. */
#define LM_ICP_POINT_TO_PLANE 0 /* TransformationEstimationPointToPlane, the reference's active branch (default) */
#define LM_ICP_POINT_TO_POINT 1 /* TransformationEstimationPointToPoint, LL.cpp:131-135 */
#define LM_POSE_PSO 3           /* particle swarm against the scene depth (below); 2 is not assigned and stays refused */
int lm_set_pose_estimation(lm_detector* d, int estimation);

/* LM_POSE_PSO: a third estimation, correspondence-free.  It replaces the ICP kernel of the pose stage with k_pose_pso
 * (one CTA per slot, persistent over the slots); the clouds before it and everything after it (the composition
 * T * init_base, verification, the pose NMS, the readbacks, the chunks) are unchanged.  k_icp_normals does not run, so a
 * frame's pose stage is 4 launches, as with point-to-point.  The item the reference's author left open
 * (linemodLevelup/notes.md: "PSO ... Correspondence-free pose estimation for 3D objects from noisy depth data").
 * Every operation below is correctly rounded (no FMA), in the order written, so tests/pose_pso_model.py restates it bit for
 * bit in numpy float64.  "a + b" etc. are double operations unless marked.
 *   Points   p_j, j < n: the down-sampled source cloud the ICP would register (metres, double, its order).  n = 0: T = S,
 *            fitness = rmse = 0.
 *   Start    S = the ICP's initial guess, identity rotation and translation s (the centroid difference).  A slot without
 *            a pose stays without one (residual -1, the early return of LL.cpp:52-55).  c_r = (sum_j (p_jr + s_r)) / n,
 *            summed from 0.0 in index order: the centroid under S.
 *   Particle x = (w0, w1, w2, t0, t1, t2), |w_k| <= dr (rad), |t_k| <= dt (m).  Its pose T(x) = Trans(c + t) Rot(w)
 *            Trans(-c) S, as [R | u]:
 *              y = (w0*w0 + w1*w1) + w2*w2.  y == 0: R = I.  Else A = sin(sqrt y)/sqrt y and B = (1 - cos(sqrt y))/y by
 *              their Taylor series to y^10 in Horner form (acc = a_10; acc = a_k + y*acc for k = 9..0; coefficients
 *              (-1)^k/(2k+1)! and (-1)^k/(2k+2)! as the nearest doubles; dr <= 45 degrees keeps them exact to rounding),
 *              K = [w]x, K2_rc = w_r*w_c (r != c), K2_rr = w_r*w_r - y, R_rc = (I_rc + A*K_rc) + B*K2_rc (Rodrigues).
 *              a_r = s_r - c_r;  u_r = (s_r + ((((R_r0*a_0) + R_r1*a_1) + R_r2*a_2) - a_r)) + t_r.
 *            x = 0 gives R = I and u = s.
 *   Cost     per point: q = T(x) p and its pixel exactly as pose verification's steps 3-4 (one shared device routine).
 *            Outside the frame or missing depth: e = clamp; else e = min(|d|, clamp), d in mm.  cost_j = (int32)floor(e *
 *            1000) (micrometres), the particle's cost sum_j cost_j in int64: exact in any order.  Lower is better.
 *   Swarm    P particles, I iterations.  Particle 0 starts at x = 0, particle i >= 1 at x_k = (2 D_k) * r - D_k with
 *            D = (dr, dr, dr, dt, dt, dt) and r = draw (i, iteration 0, k); velocities start at 0.  The best is the start
 *            (cost(S), evaluated as particle 0 of iteration 0).  Iteration k = 0 .. I-1: for k > 0 every particle moves,
 *              v = ((w*v + (c1*r1)*(p - x)) + (c2*r2)*(g - x)), r1 = draw (i, k, coordinate), r2 = draw (i, k, 6 +
 *              coordinate), w = 0.7298, c1 = c2 = 1.49618 (Clerc); v clamped to [-D, D]; x = x + v; where x leaves
 *              [-D, D] it is clamped to it and that coordinate of v set to 0;
 *            then every particle is evaluated; a particle's best p takes x when its cost is strictly lower (the first
 *            evaluation always); then the global best g takes the best personal best, the lowest index on ties, when its
 *            cost is strictly lower.  I = 0 evaluates the start alone.
 *   Draws    draw (i, k, q) of job J: splitmix64 seeded with `seed`, its output number ((J * 1024 + k) * 1024 + i) * 16 + q
 *            (0-based): z = seed + (number + 1) * 0x9E3779B97F4A7C15; z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9; z = (z ^ z >>
 *            27) * 0x94D049BB133111EB; z ^= z >> 31 (all mod 2^64), r = (z >> 11) * 2^-53 in [0, 1).  J is the
 *            survivor's index in its frame's pick order (lm_icp: the hypothesis index), so a batch frame, a single frame
 *            and a sharded unshared batch draw the same numbers for the same survivor.
 *   Output   the IcpOut of the slot: T = S while the start stays the best, else T(g); fitness = cost(g) / n / 1000 (mm per
 *            point, lower is better, so the pose NMS's -residual keeps its meaning); rmse = cost(S) / n / 1000 (what the
 *            search gained); iterations = I.  So cost(result) <= cost(S), and P = 1 or I = 0 returns S bit for bit.
 * The objective sees the surface the template's render sees, moved by T(x), as verification does: faces the new pose would
 * show are not checked.  use_scene_cloud has no effect: no target cloud is built.  The pose stage shared over the ranks
 * (lm_peer_share_pose) does not run it: lm_enqueue_pose and lm_peer_detect_batch return LM_E_STATE there.
 *   lm_set_pose_search      P (1..256), I (0..1000), dt_mm (0..10000), dr_deg (0..45), clamp_mm (0..1e6), all finite,
 *                           and the seed, for the detector's next pose stage; a frame keeps the settings it was
 *                           enqueued with, as the estimation.  LM_E_INVALID outside those limits.  No device work.
 *                           Defaults: 64, 40, 40 mm, 30 degrees, 20 mm, seed 0.
 *   lm_icp_set_pose_search  the same for the next lm_icp_process_batch / _device.
 *   lm_pose_search_points   the kernel on caller arrays: pts [n][3] f64 (m, 1 <= n < 2^31), start_t [3] f64 (s), scene
 *                           rows x cols u16 mm, sK [9] f32, the search settings and the job number J (0 <= J < 2^40).
 *                           T_out [16] f64 the result.  record (cap bytes, 8-byte words; may be null with cap 0): the
 *                           swarm record of LM_ICP_CAPTURE_SEARCH.
 * Swarm record (8 * (6 + I + 19 P) bytes): int64 cost(S), int64 cost(result), int64 index of the best particle (-1: the
 * start), f64 c[3], int64 global-best cost after each iteration [I], then the final f64 positions [P][6], velocities
 * [P][6] and personal bests [P][6], and int64 personal-best costs [P] (before any evaluation: INT64_MAX). */
int lm_set_pose_search(lm_detector* d, int particles, int iterations, double dt_mm, double dr_deg, double clamp_mm,
                       uint64_t seed);
int lm_pose_search_points(int device, const double* pts, int64_t n, const double* start_t, const uint16_t* scene, int rows,
                          int cols, const float* sK, int particles, int iterations, double dt_mm, double dr_deg,
                          double clamp_mm, uint64_t seed, int64_t job, double* T_out, void* record, int64_t cap);

/* Pose NMS on the device: the end of linemod_ros/detect.py's frame (:91-141), which refines every box-NMS survivor and
 * then drops duplicate objects in pose space with nms_norms(ts, -residual, 40.0) (:41-50, :130-131).  One CTA behind the
 * pose stage on the detector's stream; only the kept objects come back.
 *   1. Candidates: the survivors with a pose.  A survivor that took the early return of LL.cpp:52-55 takes no part and
 *      is not returned (deviation: detect.py would reuse the previous call's pose of its one global poseRefine, or
 *      raise on the first call; it also allocates ts one-dimensional, so ts[i,:] raises as written: its evident intent,
 *      3-vectors in mm, is followed).
 *   2. Score s_i = -(double)residual_i, residual the float fitness getResidual() returns: the script's sign is kept, so
 *      the LOWEST fitness ranks first.
 *   3. Order: s descending; equal scores (-0.0 == +0.0) in box-NMS pick order (the reference leaves them to an
 *      unstable argsort()[::-1]); NaN scores (lm_nms_translations only: fitness is finite) before every number, among
 *      themselves by ascending index.
 *   4. Greedy pass: keep the first remaining pose, drop every remaining j with !(d_ij > thr), d_ij =
 *      sqrt((dx*dx + dy*dy) + dz*dz) in float64, each operation correctly rounded, no FMA -- np.linalg.norm of a
 *      3-vector.  So a distance equal to thr suppresses, a NaN distance suppresses, and a kept pose with a NaN
 *      translation (zero anchor depth) suppresses every pose after it.
 *   5. Output: the kept poses in keep order; lm_match, R (9 f64) and t (3 f64, mm) bit-identical to what
 *      lm_complete_pose returns for that survivor, residual (f32).
 * The poses are composed on the device (T * init_base, then t * 1000) with the host's operations in its order, from the
 * R and t registered with each template's render.  Pose NMS spans classes, as detect.py's does.
 *   lm_enqueue_pose_nms  after lm_enqueue_pose, same stream, no host synchronisation; one launch whatever the survivor
 *                        count.  LM_E_STATE without a pending lm_enqueue_pose (or when already enqueued for it),
 *                        LM_E_INVALID for a NaN or negative threshold (+inf is accepted: every finite distance lies
 *                        within it, so only the best candidate is kept; 0 drops exact duplicates only).  The frame must then
 *                        complete through lm_complete_detect: lm_complete_pose returns LM_E_STATE.  With a connected peer
 *                        exchange, every rank enqueues its match before any rank enqueues the post, pose and pose NMS
 *                        stages.
 *   lm_complete_detect   waits; out[n_out], R_out + 9k, t_out + 3k, residual[k] are the kept poses; n_survivors =
 *                        box-NMS survivors, n_posed = those with a pose, n_records as lm_complete_post.  A frame that
 *                        overflowed is grown and replayed first, pose stage and pose NMS included (lm_complete).
 *   lm_nms_translations  steps 3-5 on caller arrays (t [n][3] f64, score [n] f64), with the same device routine, for the
 *                        poses of lm_icp_process_batch: keep[n_keep] are indices in keep order.  n <= 1024, else
 *                        LM_E_CAPACITY; threshold as above. */
int lm_enqueue_pose_nms(lm_detector* d, double translation_threshold_mm);
int lm_complete_detect(lm_detector* d, lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap,
                       int64_t* n_out, int64_t* n_survivors, int64_t* n_posed, int64_t* n_records);
int lm_nms_translations(int device, int64_t n, const double* t, const double* score, double thr, int32_t* keep,
                        int64_t* n_keep);

/* Pose verification on the device (default off): a depth-consistency score per refined pose, from the scene depth.
 * For survivor / hypothesis i with a pose (no early return of LL.cpp:52-55):
 *   1. Points: the model cloud the pose stage builds before voxel down-sampling -- every crop pixel with render depth > 0,
 *      back-projected with the template's K as the cloud building does (metres, double, row-major crop order).
 *      n_model is their count.
 *   2. Pose: T, the ICP's final 4x4 transformation (row-major double, lm_icp_capture's RESULT), which maps that cloud
 *      into the scene camera; used as is, whatever the estimation and use_scene_cloud.
 *   3. Transform and project: q_r = ((T[r][0] p_x + T[r][1] p_y) + T[r][2] p_z) + T[r][3], every operation correctly
 *      rounded, no FMA.  !(q_z > 0): outside.  Else u = (double)fx * (q_x / q_z) + (double)cx, v likewise with fy, cy,
 *      each operation rounded; column c = floor(u + 0.5), row r = floor(v + 0.5).  u or v not finite, or (c, r) off
 *      the frame: outside.
 *   4. Compare: z_s = scene depth at (r, c) (u16 mm), z_q = q_z * 1000 (mm).  z_s == 0: missing.  Else d = (double)z_s -
 *      z_q: |d| <= delta inlier, d < -delta occluded (something lies in front of the model), d > delta violation (the
 *      scene lies behind the model's surface, which would hide it).
 *   5. Outputs: six int32 counts n_model, outside, missing, inlier, occluded, violation (the last five sum to n_model),
 *      and score = inlier / (inlier + occluded + violation) as float (__fdiv_rn), 0 when that sum is 0.  A survivor
 *      without a pose: score -1 and zero counts (as its residual -1).  A NaN pose (zero anchor depth) puts every point
 *      outside: score 0.
 *   6. delta: inlier_mm, finite and >= 0; 10 mm (the ICP's correspondence radius) is the usual choice.
 * This is the surface the template's render sees, moved by T -- not a render at the refined pose: points the render hid
 * stay hidden, and faces the refined pose would newly show are not checked.  A score says how well the scene agrees
 * with that surface; it does not by itself tell a true object from a false one.
 * With verification on, the pose NMS can use it:
 *   rank_by  LM_VERIFY_RANK_FITNESS: today's score -(double)residual (the default); LM_VERIFY_RANK_SCORE: the
 *            verification score, descending.  Either way equal keys keep box-NMS pick order.
 *   min_score  a posed survivor whose score is below it is no pose-NMS candidate: it is neither kept nor suppresses
 *            others, as one without a pose.  -INFINITY: no minimum.
 * Without the pose NMS every survivor comes back with its score; nothing is dropped.
 *   lm_set_pose_verify   for the detector's next lm_enqueue_pose, lm_detect_batch and lm_peer_detect_batch; a frame keeps
 *                        the setting it was enqueued with (the replay after a result-block retry included).  No device
 *                        work.  With a connected peer exchange every rank sets the same value.  LM_E_INVALID for a NaN
 *                        or negative inlier_mm, an unknown rank_by, a NaN min_score, and for LM_VERIFY_RANK_SCORE or a
 *                        min_score other than -INFINITY with on == 0.  Each chunk of a pose stage takes one more launch
 *                        (k_pose_verify behind the ICP kernel).  A pose stage shared over the ranks (lm_peer_share_pose)
 *                        verifies each survivor on the rank that refined it, and its result travels with the pose: every
 *                        rank returns what the unshared stage returns.  The device buffers for the results are allocated
 *                        by the first run that verifies.
 *   lm_pose_verify       score[k], counts6 + 6k of entry k of the last completed frame or batch (lm_complete_pose /
 *                        lm_complete_detect / lm_detect_batch), in the order of its entries; *n their number.
 *                        LM_E_STATE when that run did not verify, LM_E_CAPACITY (with *n) when cap is smaller.
 *   lm_pose_verify_points  steps 3-5 on caller arrays with the same device routine: pts [n][3] f64 (m), T [16] f64,
 *                        scene rows x cols u16 mm, sK [9] f32. */
#define LM_VERIFY_RANK_FITNESS 0
#define LM_VERIFY_RANK_SCORE 1
int lm_set_pose_verify(lm_detector* d, int on, double inlier_mm, int rank_by, double min_score);
int lm_pose_verify(lm_detector* d, float* score, int32_t* counts6, int64_t cap, int64_t* n);
int lm_pose_verify_points(int device, const double* pts, int64_t n, const double* T, const uint16_t* scene, int rows, int cols,
                          const float* sK, double inlier_mm, int32_t* counts6, float* score);

/* Tracking on the device: detect once, then refine each object's last pose against the next frame's depth, with no match,
 * box NMS or pose NMS.  A new capability, not a port: the reference's live loop (linemod_ros/detect.py:167-168) runs the
 * whole detection on every frame.  A tracked object is (class index, template id within the class, T):
 *   T        the ICP's 4x4 transformation, row-major f64, which maps the template's render cloud (metres, the template's
 *            camera) into the scene camera: the T of LM_ICP_CAPTURE_RESULT and of verification's step 2, and what
 *            lm_pose_transforms returns for the entries of lm_complete_pose, lm_complete_detect, the batch calls and
 *            lm_track.  A caller holding only a pose (R, t mm) as lm_complete_pose returns it converts it with the
 *            template's registered R_b, t_b (init_base, LL.cpp:34-38: b = (t_b.x, t_b.y, (float)(t_b.z / 1000.0f)), each
 *            widened to double), every operation correctly rounded, no FMA, in this order:
 *              T_R[r][c] = ((R[r][0] * R_b[c][0]) + R[r][1] * R_b[c][1]) + R[r][2] * R_b[c][2]      (R R_b^T)
 *              T_t[r]    = t[r] / 1000 - (((T_R[r][0] * b_0) + T_R[r][1] * b_1) + T_R[r][2] * b_2)
 *            with row 3 = (0, 0, 0, 1).  T * init_base then gives (R, t) back up to rounding; bit for bit only for a T
 *            that came from the device.
 * Each object of a call is one slot of one pose-stage chunk (n <= 1024):
 *   0. View following (lm_set_track_views, off by default): the object may first switch to the template of its class
 *      whose training view lies closest to its current orientation, with T re-expressed for it; every later step then
 *      uses that template.  Off, the object keeps its template.
 *   1. Model cloud: exactly the pose stage's source cloud for that template -- its registered crop back-projected
 *      (LM_POSE_CAPTURE_RAW_MODEL) and voxel down-sampled -- bit-identical to what a detected survivor of the template gets.
 *   2. Window: every raw model point projected under T with verification's step 3, operation for operation; the
 *      min / max column and row of the points that land in the frame in front of the camera are the projected box
 *      (x, y, w, h), unclipped by the margin.  The window is that box grown by margin_px on each side and clipped to the
 *      frame.  No point in the frame: LM_TRACK_OUTSIDE.  A window of more than 4 A pixels, A the largest registered crop:
 *      LM_TRACK_WINDOW (the scene slot holds 4 A points, so an object may roughly double its image size between frames).
 *   3. Scene cloud: every window pixel with depth > 0, row-major, back-projected with sceneK as the pose stage
 *      back-projects scene pixels, and voxel down-sampled as the scene cloud is.  No such pixel: LM_TRACK_NO_DEPTH.
 *      Tracking always registers against the scene (the reference's model-against-itself target would leave T where it
 *      started), so use_scene_cloud plays no part.
 *   4. Refinement: the ICP of lm_set_pose_estimation (k_icp_normals + k_icp_point_to_plane, or k_icp_point_to_point)
 *      from IcpJob::init = T, with max_iterations.
 *   5. Outputs, entry i for object i: status[i] (LM_TRACK_*); box + 4i the projected box (zeros when OUTSIDE); for
 *      TRACKED: T_out + 16i the new T, R_out + 9i / t_out + 3i (mm) composed exactly as lm_complete_pose composes them,
 *      residual[i] the fitness.  Any other status: residual -1, and T, R and t left untouched.
 *   6. Verification: with lm_set_pose_verify on, k_pose_verify scores every tracked pose, and lm_pose_verify returns the
 *      scores in entry order (-1 for an entry not tracked).  Nothing is dropped; lm_nms_translations is the caller's.
 * Refusals, before any device work: LM_E_INVALID for a null argument, n < 0 or n > 1024, an empty image, max_iterations
 * < 0, margin_px < 0, an unknown depth format or a bad depth_scale, a class or template out of range, a non-finite entry
 * of T; LM_E_STATE for LM_POSE_PSO (its kernel starts from an identity rotation), a connected peer exchange (use
 * lm_peer_track_batch there), or an object
 * whose template has no registered render (and on a host-only handle); LM_E_CAPACITY as the pose stage's buffers.
 * A call runs on the detector's stream and returns once the outputs are on the host; it abandons a frame whose pose stage
 * is pending.  lm_debug_pose_clouds then describes its chunk: slot i is object i, POSED is 1 for TRACKED, INIT is T,
 * and LM_POSE_CAPTURE_WINDOW gives the window and status.  Launches: 5 (point-to-plane) or 4, plus 1 when verifying, plus
 * 1 with view following (per chunk, in every track call), plus 1 for lm_track_device's conversion.
 *   lm_track          depth: rows x cols u16 mm on the host, copied.
 *   lm_track_device   depth: a pitched device plane, LM_DEPTH_U16_MM or LM_DEPTH_F32 with depth_scale, converted as
 *                     lm_bind_images_device converts it and ordered as it orders the frame: an event on `stream` gates the
 *                     read, and `stream` waits on a second event once the conversion is done.
 *   lm_pose_transforms  T_out + 16k: the T of entry k of the pose run last finished (lm_complete_pose, lm_complete_detect
 *                     (its kept poses), the batch calls, lm_track), in entry order; NaN for an entry without a pose;
 *                     *n their number.  The pose NMS records each kept pose's survivor on the device; the T of
 *                     that survivor's ICP output is copied here, only when asked.  LM_E_STATE once another run has started or when the last one
 *                     failed; LM_E_CAPACITY (with *n) when cap is smaller. */
#define LM_TRACK_TRACKED 0
#define LM_TRACK_OUTSIDE 1
#define LM_TRACK_WINDOW 2
#define LM_TRACK_NO_DEPTH 3
typedef struct lm_track_object {
  int32_t class_index, template_id;
  double T[16];
} lm_track_object;
int lm_track(lm_detector* d, const uint16_t* depth, int rows, int cols, const float* sceneK, const lm_track_object* objects, int n,
             int max_iterations, int margin_px, double* T_out, double* R_out, double* t_out, float* residual, int32_t* status,
             int32_t* box);
int lm_track_device(lm_detector* d, const void* depth, int64_t depth_pitch, int depth_format, float depth_scale, int rows, int cols,
                    const float* sceneK, const lm_track_object* objects, int n, int max_iterations, int margin_px, double* T_out,
                    double* R_out, double* t_out, float* residual, int32_t* status, int32_t* box, void* stream);
int lm_pose_transforms(lm_detector* d, double* T_out, int64_t cap, int64_t* n);

/* View following for the track calls.  A tracked object's model cloud is the surface its template's render saw from one
 * viewpoint; once the object has turned far from that view, the scene shows faces the cloud lacks and the ICP drifts.
 * With view following on, k_track_views (one CTA per object, one launch per chunk, ahead of k_track_cloud) re-chooses
 * each object's template among the registered renders of its class from its rotation alone, and rewrites the object's
 * template and T on the device, so the window, both clouds, IcpJob::init, verification and LM_POSE_CAPTURE_* all see the
 * chosen template.  The rule, in double, every operation correctly rounded in the order written and no FMA; R_b, t_b
 * are the registered f32 values widened; the object has template k of class c and T (4x4, row-major):
 *   1. tau = 1.0 + 2.0 * cos(turn_deg * 0.017453292519943295) (libm cos, on the host).
 *   2. Ro[r][c] = ((T[r][0] * Rk[0][c]) + T[r][1] * Rk[1][c]) + T[r][2] * Rk[2][c], Rk = R_b of template k.
 *   3. s_j = trace(Ro^T R_j) for every template j of class c with a registered render (k included), summed from 0.0 as
 *      s = s + Ro[r][c] * R_j[r][c], r outer, c inner.  A NaN s_j is no candidate.
 *   4. !(s_k < tau): keep k (the object is within turn_deg of its template's view).  Otherwise j* = arg-max s_j, the
 *      lowest j on ties; switch only when j* != k and s_j* > s_k.  Kept: T stays the input's bits.
 *   5. Switching: P_j = [R_j | b_j], b_j[r] = t_bj[r] / 1000.0 (metres on every axis, since the render cloud is metric;
 *      unlike init_base, which converts t.z only), and
 *        Q_R[r][c] = ((Rk[r][0] * Rj[c][0]) + Rk[r][1] * Rj[c][1]) + Rk[r][2] * Rj[c][2]            (Rk Rj^T)
 *        Q_t[r]    = b_k[r] - (((Q_R[r][0] * b_j[0]) + Q_R[r][1] * b_j[1]) + Q_R[r][2] * b_j[2])
 *        T'[r][c]  = ((T[r][0] * Q_R[0][c]) + T[r][1] * Q_R[1][c]) + T[r][2] * Q_R[2][c]
 *        T'[r][3]  = (((T[r][0] * Q_t[0]) + T[r][1] * Q_t[1]) + T[r][2] * Q_t[2]) + T[r][3],   row 3 = (0, 0, 0, 1)
 *      so the physical object stays where T put it.
 * A call with view following on therefore returns, bit for bit, what the same call with it off returns for the objects
 * (class, j*, T') -- status, box, T, R, t, residual, lm_pose_transforms and lm_pose_verify -- and its R_out / t_out are
 * composed with the chosen template's render pose.  Shared over the ranks, every rank re-chooses every object of each
 * chunk, so the exchange's layout is unchanged.
 *   lm_set_track_views  for the detector's next lm_track, lm_track_device, lm_track_batch, lm_track_batch_device,
 *                       lm_peer_track_batch and lm_peer_track_batch_device.  on 0 ignores turn_deg.  LM_E_INVALID when
 *                       on and turn_deg is NaN, negative or >= 180.  No device work (a host-only handle takes it);
 *                       loading another bank keeps it.
 *   lm_track_templates  template_id[k]: the template within its class of entry k of the track run last finished, in
 *                       entry order -- the chosen one for a TRACKED entry, the start's for any other (whose T, R and t
 *                       stay untouched).  With view following off, every entry's start template.  *n their number.
 *                       LM_E_STATE when the run last finished was no track run or failed; LM_E_CAPACITY (with *n) when
 *                       cap is smaller.
 *   lm_track_views_points  k_track_views on caller arrays: one object at template k (T [16] f64) of one class of n
 *                       templates, R_b [n][9] and t_b [n][3] f32, all with a render; *chosen = the template it keeps or
 *                       switches to, T_out [16] its T.  LM_E_INVALID for a null argument, n < 1, k outside [0, n), a
 *                       non-finite T or a turn_deg lm_set_track_views refuses. */
int lm_set_track_views(lm_detector* d, int on, double turn_deg);
int lm_track_templates(lm_detector* d, int32_t* template_id, int64_t cap, int64_t* n);
int lm_track_views_points(int device, int64_t n, const float* R_b, const float* t_b, int64_t k, const double* T, double turn_deg,
                          int64_t* chosen, double* T_out);

/* Tracking a batch of depth frames in one call: several cameras, or several independent sequences at one time step (a
 * sequence's next frame starts from this one's results, so a batch never spans time).  Every frame's objects are slots
 * of one pose-stage run, so a few objects per frame no longer leave most of the GPU idle.
 *   Frames     frame f's depth is depth + f * rows * cols (lm_track_batch: host, one size for all frames, copied to the
 *              device in one copy) or the device plane depth[f] (lm_track_batch_device: a common pitch, format and
 *              scale, converted and ordered on `stream` as lm_track_device orders its plane); its intrinsics are
 *              sceneK + 9f.
 *   Objects    frame f's objects are the next n_objects[f] entries of `objects`, in frame order; n_objects[f] lies in
 *              [0, 1024], lm_track's bound, and a frame without objects may come anywhere.  The outputs (status, box + 4k,
 *              T_out + 16k, R_out + 9k, t_out + 3k, residual[k]) take the same entry order.
 *   Bit for bit  frame f's entries are what lm_track (or lm_track_device) returns for that frame and its objects alone:
 *              status, box, T, R, t and residual, NaN patterns included; lm_pose_transforms and, with verification on,
 *              lm_pose_verify then return every entry of the batch in entry order.  This holds because everything a slot
 *              computes -- its window, both clouds, its voxel sort segment, its ICP job and its verification -- depends
 *              only on its object and its own frame's depth and K, and the window cap 4 A only on the registered renders.
 *   Chunks     the run is cut into chunks of 1024 slots; a frame may straddle a chunk boundary.  Launches per chunk are a
 *              track chunk's (5 point-to-plane or 4, plus 1 when verifying, plus 1 with view following), plus one conversion per frame for
 *              lm_track_batch_device.  lm_debug_pose_clouds then describes the last chunk (slot i is entry 1024 c + i of
 *              chunk c).
 * Refusals, before any device work, are lm_track's with its codes and messages, plus the frame (and the object's index
 * within its frame) where one applies: LM_E_INVALID for a null argument, n_frames < 1, n_objects[f] outside [0, 1024],
 * an empty image, max_iterations < 0, margin_px < 0, a bad class, template or non-finite T, and (device) an unknown
 * depth format, a bad depth_scale, a plane of any frame that fails lm_bind_images_device's checks (named depth[f]) or a
 * stream of another device; LM_E_STATE for an object without a registered render, LM_POSE_PSO, a connected peer exchange
 * and a host-only handle.  Like lm_track, a call abandons a frame whose pose stage is pending and returns once the
 * outputs are on the host.
 * Device memory kept by the handle: n_frames depth slots of rows * cols * 2 bytes, shared with lm_detect_batch's, and
 * for each of the batch's objects a pose-stage output slot (ICP output, posed flag, frame index, window record and
 * object, with pinned host copies of the first two); the cloud buffers stay those of one 1024-object chunk. */
int lm_track_batch(lm_detector* d, int n_frames, const uint16_t* depth, int rows, int cols, const float* sceneK,
                   const lm_track_object* objects, const int32_t* n_objects, int max_iterations, int margin_px,
                   double* T_out, double* R_out, double* t_out, float* residual, int32_t* status, int32_t* box);
int lm_track_batch_device(lm_detector* d, int n_frames, const void* const* depth, int64_t depth_pitch, int depth_format,
                          float depth_scale, int rows, int cols, const float* sceneK, const lm_track_object* objects,
                          const int32_t* n_objects, int max_iterations, int margin_px, double* T_out, double* R_out,
                          double* t_out, float* residual, int32_t* status, int32_t* box, void* stream);

/* lm_track_batch and lm_track_batch_device over the ranks of a connected peer exchange, with the same arguments and
 * outputs.  Every rank returns what one unconnected handle holding the same renders returns from lm_track_batch on the
 * same frames and objects, bit for bit: status, box, T, R, t and residual, NaN patterns included; lm_pose_transforms and,
 * with verification on, lm_pose_verify then return the same entries.  Calling it is the caller's promise that every rank
 * calls it with the same frames, objects, estimation and verification settings, in the same order as its other pose
 * exchanges (shared frames, lm_peer_detect_batch).
 *   Pose       sharing off: every rank tracks every object itself, and the exchange is not touched (5 launches per chunk
 *              point-to-plane, 4 point-to-point).  Sharing on (lm_peer_share_pose): the run is cut into chunks of 1024
 *              objects as lm_track_batch cuts it; within a chunk of C objects, object i is tracked by rank i % world in
 *              ceil(C / world) slots.  The owner builds its window and clouds, refines it and (verification on) verifies
 *              it, then stores its ICP output, posed flag, overflow flag, verification and window record (window,
 *              projected box, status) into the pose area of every rank; a collector gathers them in object order, as for
 *              a shared batch chunk (6 launches per chunk point-to-plane, 5 point-to-point; a rank without an object in
 *              the chunk still publishes).  Each chunk is one pose exchange and takes the next number of the pose
 *              counter, so shared frames, lm_peer_detect_batch and lm_peer_track_batch interleave in any order.  Add 1
 *              launch per chunk when verifying, 1 per chunk with view following (every rank re-chooses every object
 *              of the chunk), and one conversion per frame for lm_peer_track_batch_device.  A run
 *              without objects launches nothing and exchanges nothing.
 * Refusals, before any device work: LM_E_STATE without a connected exchange, for LM_POSE_PSO and on a host-only handle;
 * otherwise every refusal of lm_track_batch / lm_track_batch_device with its code and "frame f: object k" message.
 * lm_track, lm_track_device, lm_track_batch and lm_track_batch_device still refuse a connected exchange.  A peer whose
 * poses do not arrive in time fails the call with LM_E_STATE (the message names the pose exchange).
 * No device memory is allocated or freed once the run's first chunk is enqueued: the scenes, the pose stage's outputs and
 * cloud buffers and the per-object records are grown before it.  Ranks that are handles of ONE process on ONE device call
 * from their own host threads, and each first runs the largest shape (frames, frame size, objects) it will run shared
 * with sharing off: that call grows the buffers while no collector spins, since a free waits for the whole device -- a
 * peer's collector included.  lm_pose_stats afterwards: the objects, the objects this rank tracked over all chunks, the
 * pose stage's launches (the conversions not counted) and 1 if shared. */
int lm_peer_track_batch(lm_detector* d, int n_frames, const uint16_t* depth, int rows, int cols, const float* sceneK,
                        const lm_track_object* objects, const int32_t* n_objects, int max_iterations, int margin_px,
                        double* T_out, double* R_out, double* t_out, float* residual, int32_t* status, int32_t* box);
int lm_peer_track_batch_device(lm_detector* d, int n_frames, const void* const* depth, int64_t depth_pitch, int depth_format,
                               float depth_scale, int rows, int cols, const float* sceneK, const lm_track_object* objects,
                               const int32_t* n_objects, int max_iterations, int margin_px, double* T_out, double* R_out,
                               double* t_out, float* residual, int32_t* status, int32_t* box, void* stream);

/* A batch of RGB-D frames in one call: each frame's match and box NMS, then one pose stage and (pose_nms) one pose NMS
 * for the survivors of every frame.  Frame f is rgb + f * rows * cols * 3 and depth + f * rows * cols (all frames one
 * size), masks[2f] / masks[2f + 1] its colour and depth masks (masks NULL: none), sceneK + 9f its intrinsics.  The other
 * arguments are those of lm_enqueue (threshold), lm_enqueue_post (iou_threshold, top_k), lm_enqueue_pose (max_iterations,
 * use_scene_cloud) and lm_enqueue_pose_nms (translation_threshold_mm).
 * Frame f's entries follow those of frames 0..f-1 in out / R_out + 9k / t_out + 3k / residual[k]; bit for bit they are
 * what the single-frame chain returns for that frame alone:
 *   pose_nms == 0  lm_upload_images, lm_enqueue, lm_enqueue_post, lm_enqueue_pose, lm_complete_pose: every survivor, in
 *                  pick order; residual -1 and R / t untouched on the early return of LL.cpp:52-55.
 *   pose_nms == 1  the same chain plus lm_enqueue_pose_nms, lm_complete_detect: the kept poses, in keep order.
 * frame_counts[4f .. 4f + 3] = entries, box-NMS survivors, survivors with a pose, kept records the box NMS saw.
 * *n_out = entries of the whole batch.  LM_E_CAPACITY (with *n_out the total needed) when cap is smaller (an
 * LM_E_CAPACITY that leaves *n_out unwritten comes from a frame's match, where growing cap does not help);
 * LM_E_INVALID for n_frames < 1 or a NaN / negative translation threshold with pose_nms; LM_E_STATE without renders
 * for every selected template, and with a connected peer exchange (use lm_peer_detect_batch there).
 * Each frame runs the single-frame match and box NMS and waits for them (a frame that overflows is grown and
 * replayed there, as lm_complete describes); its survivors and depth are copied aside on the stream.  The pose stage then runs once over all
 * S survivors in chunks of at most 1024 slots (the single-frame bound for top_k = 0, so its cloud buffers do not grow
 * with the batch): 5 launches per chunk (4 with LM_ICP_POINT_TO_POINT, lm_set_pose_estimation), plus 1 launch of the
 * pose NMS for every frame.  Before its first frame the call
 * uploads the renders and grows every buffer a batch of its shape (n_frames, rows x cols, top_k) may need.  Extra device
 * memory, kept by the handle for the next batch: n_frames depth slots (rows * cols * 2 bytes each, 614 KB at 640 x 480),
 * n_frames * (top_k, or 1024) survivor slots of 20 bytes, for each of those slots an ICP output, pose NMS entry, frame
 * index and posed flag (about 280 bytes, plus a pinned host copy of the first two), and the pose stage's cloud buffers
 * for min(n_frames * (top_k, or 1024), 1024) survivors. */
int lm_detect_batch(lm_detector* d, int n_frames, const uint8_t* rgb, const uint16_t* depth, int rows, int cols,
                    const uint8_t* const* masks, float threshold, const float* sceneK, double iou_threshold, int top_k,
                    int max_iterations, int use_scene_cloud, int pose_nms, double translation_threshold_mm,
                    lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap, int64_t* n_out,
                    int64_t* frame_counts);

/* lm_detect_batch over the ranks of a connected peer exchange, with the same arguments and outputs.  Every rank returns
 * what one unconnected handle over the whole bank returns from lm_detect_batch on the same frames, bit for bit: the
 * entries, R, t, residual (NaN patterns included) and all four frame_counts of every frame.  Calling it is the caller's
 * promise that every rank calls it with the same frames and arguments, in the same order as its other frames.
 *   Match      each frame's match runs the fused record exchange, as a connected single frame does, and its box NMS
 *              sees every shard's records, so every rank holds the same S survivors and the same chunks.
 *   Pose       sharing off: every rank refines every survivor (5 launches per chunk).  Sharing on (lm_peer_share_pose):
 *              within a chunk of C survivors, survivor i is refined by rank i % world in ceil(C / world) slots, and the
 *              results travel through the pose area as for a shared frame (6 launches per chunk; a rank without a
 *              survivor in the chunk still publishes).  Each chunk is one pose exchange.  Then 1 pose NMS launch.
 *              LM_ICP_POINT_TO_POINT takes one launch off each chunk (no normals).
 * LM_E_STATE without a connected exchange; the other argument and state errors are those of lm_detect_batch and come
 * before any device work.  LM_E_CAPACITY for too small outputs (*n_out = the total needed, > cap) comes on every rank
 * alike (the totals are the same), so a caller that grows cap and calls again does so on every rank.  LM_E_CAPACITY
 * with *n_out not written means a frame's records outgrew the exchange (a shard kept more than lm_peer_export's
 * capacity_records; the message names the peer exchange) or the result block, which does not grow while connected;
 * every rank sees it at the same frame, and calling again fails again: reconnect with a larger capacity.  A peer whose poses do not arrive in time fails the batch with LM_E_STATE
 * (the message names the pose exchange).  No device memory is allocated or freed once the first frame is enqueued.
 * Ranks that are handles of ONE process on ONE device call from their own host threads, and each first runs one
 * unconnected lm_detect_batch of the largest shape (n_frames, frame size, top_k) it will run connected: that one
 * uploads the renders and grows the buffers, which frees device memory, and a free waits for the whole device -- a
 * peer's collector included.  For the same reason, once connected, every rank calls lm_prepare (which grows the result
 * block to the exchange's size) before any rank enqueues a frame.  lm_pose_stats afterwards: S, the hypotheses this rank refined over all chunks, the pose
 * stage's launches (chunks x 6 shared, x 5 unshared, one fewer per chunk with LM_ICP_POINT_TO_POINT; the pose NMS not
 * counted) and 1 if shared. */
int lm_peer_detect_batch(lm_detector* d, int n_frames, const uint8_t* rgb, const uint16_t* depth, int rows, int cols,
                         const uint8_t* const* masks, float threshold, const float* sceneK, double iou_threshold, int top_k,
                         int max_iterations, int use_scene_cloud, int pose_nms, double translation_threshold_mm,
                         lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap, int64_t* n_out,
                         int64_t* frame_counts);

/* lm_detect_batch from frames already in device memory: frame f's upload is replaced by lm_bind_images_device of
 * (rgb[f], depth[f], masks ? masks[2f] : NULL, masks ? masks[2f + 1] : NULL) with the common pitches, depth format, scale
 * and stream -- n_frames device pointers per plane, held in host arrays.  From threshold on, the arguments, outputs,
 * frame_counts and errors are lm_detect_batch's; lm_bind_images_device's checks are made for every frame before any
 * device work.  Each frame's borrow ends with its ingest, ordered on `stream` as lm_bind_images_device orders it. */
int lm_detect_batch_device(lm_detector* d, int n_frames, const uint8_t* const* rgb, int64_t rgb_pitch, const void* const* depth,
                           int64_t depth_pitch, int depth_format, float depth_scale, int rows, int cols,
                           const uint8_t* const* masks, int64_t mask_pitch, void* stream, float threshold, const float* sceneK,
                           double iou_threshold, int top_k, int max_iterations, int use_scene_cloud, int pose_nms,
                           double translation_threshold_mm, lm_match* out, double* R_out, double* t_out, float* residual,
                           int64_t cap, int64_t* n_out, int64_t* frame_counts);

/* Convenience = lm_upload_quantized + lm_run + lm_fetch_records + lm_finish (single GPU):
 * Detector::match after quantization. */
int lm_match_quantized(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols,
                       float threshold, lm_match* out, int64_t cap, int64_t* n_out);

/* Detector::match proper (LL.cpp:1702-1777): raw images in, matches out. */
int lm_match_images(lm_detector* d, const uint8_t* rgb, const uint16_t* depth, int rows, int cols, const uint8_t* mask_color,
                    const uint8_t* mask_depth, float threshold, lm_match* out, int64_t cap, int64_t* n_out);

/* Depth gate of the coarse scan (off by default).  A bank rendered at several distances (the reference's allScales: 337
 * views at each of 600 ... 1800 mm) treats each scale as its own object, and small scales match random texture; the gate
 * keeps a template's coarse candidates only where the scene lies near the distance the template was trained at.
 * L = the lowest pyramid level, s = 2^(L-1) (levels - 1 halvings), T_L its step, Wd x Hd its coarse grid.  For candidate
 * position (cx, cy) of template t in the coarse scan, before its pass bit is counted:
 *   1. Cell summary, per frame: block (x, y) = full-resolution pixels [x*s*T_L, (x+1)*s*T_L) x [y*s*T_L, (y+1)*s*T_L) of
 *      the uploaded depth (u16 mm; masks do not affect it); lo(x, y) / hi(x, y) = min / max non-zero depth of the block.
 *      A block without a non-zero pixel is empty.
 *   2. Sample cell (sx, sy) = (cx + floor(floor(w_t / 2) / T_L), cy + floor(floor(h_t / 2) / T_L)), w_t x h_t =
 *      Template::width / height of t at level L, modality 0 (tmeta).
 *   3. Band zlo_t = ceil(z_t * (1 - tau)), zhi_t = floor(z_t * (1 + tau)), in float64, clamped to [0, 65535]; z_t = the
 *      template's training distance (mm), tau = the tolerance.
 *   4. The candidate passes iff sx >= Wd, or sy >= Hd, or the sample cell is empty, or t has no distance, or
 *      (lo <= zhi_t and hi >= zlo_t).  Every other candidate is removed before the candidate list, exactly as if its raw
 *      score were below the threshold; the match list is the reference's matchClass / sort / unique over the gated
 *      candidate set (so unique may keep a different template of a collapsed pair).
 * The gate adds one launch per frame (k_depth_cells, ahead of the coarse scan) and runs the gated variants of the coarse
 * kernels; with the gate off nothing of the frame changes.
 *   lm_set_template_depths  z_mm[i] = training distance of template first + i, bank order (as lm_set_boxes); NaN or <= 0:
 *                           never gated.  Loading another bank drops the distances.  LM_E_INVALID for a range outside the
 *                           bank.
 *   lm_set_depth_gate       on != 0 turns the gate on with `tolerance` (tau), for the next lm_enqueue (single frame or
 *                           batch); no device work, and a frame keeps the setting it was enqueued with (the rerun after a
 *                           result-block retry included).  LM_E_INVALID for tolerance < 0, >= 1 or NaN.  With the gate on,
 *                           lm_enqueue and lm_prepare fail with LM_E_STATE when no template of the bank has a distance, or when the
 *                           frame has no depth (lm_upload_quantized / lm_bind_quantized_device).  With a connected peer
 *                           exchange, every rank setting the same distances and gate before its next frame is the caller's
 *                           promise, as with lm_peer_share_pose: each rank gates its own shard on its own copy of the frame.
 *   lm_depth_gate_stats     of the last enqueued frame (single frame, or the last of a batch), which must have run gated
 *                           (else LM_E_STATE): [0] candidates of this handle's shard before the gate, [1] after it,
 *                           [2] empty cells, [3] work items of this handle's shard with a distance.  Synchronises the
 *                           stream. */
int lm_set_template_depths(lm_detector* d, int64_t first, int64_t n, const float* z_mm);
int lm_set_depth_gate(lm_detector* d, int on, double tolerance);
int lm_depth_gate_stats(lm_detector* d, int64_t* out4);

/* ---- introspection used by the parity tests and the benchmark ---- */
/* Quantized label image of (level, modality) of the uploaded frame: rows*cols bytes. */
int lm_debug_quantized(lm_detector* d, int level, int modality, uint8_t* out, int64_t cap);
/* Depth image (u16 mm, rows*cols) of the frame lm_upload_images uploaded or lm_bind_images_device bound. */
int lm_debug_depth(lm_detector* d, uint16_t* out, int64_t cap);
/* Linear memories of (level, modality) of the last lm_run: [8][T*T][(cols/T)*(rows/T)] bytes.  A level whose bytes that
 * run did not build (nothing read them) is built here first, from the frame still bound. */
int lm_debug_linear_memories(lm_detector* d, int level, int modality, uint8_t* out, int64_t cap);
/* Test getter: the lowest level's spread bit-planes of the last lm_run, [M][8][lbw] uint32 words (bit i of a label's
 * words: spread bit of linear-memory index i = grid * plane + position; the words behind the T*T*plane live bits are
 * zero).  *n_words (M*8*lbw; 0 when the level has none) is set before the capacity test (LM_E_CAPACITY when cap is
 * smaller; out may be null with cap 0).  Synchronises the stream. */
int lm_debug_bit_planes(lm_detector* d, uint32_t* out, int64_t cap, int64_t* n_words);
/* Development probe: the mean device time in microseconds of `reps` back-to-back launches of the K1 blocks of one level
 * (level -1: the whole launch), from the K1 plan the last frame recorded, rebuilding that frame's outputs in place.
 * Synchronises the stream.  LM_E_STATE before the first lm_run. */
int lm_debug_time_k1(lm_detector* d, int level, int reps, float* us);
/* Test getter: which kernels and launch shapes the last lm_run took, as the frame's plan recorded them when it was
 * enqueued (no launch; one small read of the filter's survivor counts).  LM_PLAN_ENTRIES int32 entries:
 * [0] linear memories by k_linear_memories_band (1) or k_linear_memories (0), [1] level built as H-planes only (-1:
 * none), [2] its positions per segment (pseg; 0: none), [3] the band kernel's shared memory (bytes), [4] rounds of
 * 32 x 32 position words at the lowest level, [5] its spread bit-planes are allocated (1/0), [6] templates on
 * k_coarse_packed, [7] templates on k_coarse_bytes, [8] k_coarse_packed stages the bit-planes in shared memory (1/0),
 * [9] its team split S, [10] bit-plane bytes, [11] its tasks ([8]..[11]: -1 without packed templates),
 * [12] the refinement filter is available for the frame size (1/0), [13] bit-sliced refinement (two levels, 1/0),
 * [14] templates of the shard the filter takes, [15] the frame ran depth-gated (1/0), then the work items (this
 * handle's shard only, also behind the peer exchange) of
 * [16] k_refine_filter_w, [17] k_refine_bits, [18] k_refine<true>, [19] k_refine<false> (-1: it did not run), [20] the
 * CTAs k_refine_bits runs with (the ones resident at once; -1: it did not run), [21] what K1 builds of the lowest level:
 * bit 0 its spread bit-planes, bit 1 its byte linear memories (built only when k_coarse_bytes has templates).
 * Describes the last completed frame only between lm_complete (or lm_run) and the next lm_enqueue, which records its own
 * frame's plan; the survivor counts are read from the device when the getter is called, so after a later lm_enqueue the
 * getter waits for that frame and reports its counts. */
#define LM_PLAN_ENTRIES 22
int lm_debug_plan(lm_detector* d, int32_t* out, int64_t cap);
/* Test getter: the coarse scan's outputs (k_coarse_packed / k_coarse_bytes) of the last completed frame, per work item of
 * this handle's shard in shard order.  dims3 = {n_work, nwords, plane} of the lowest level; `mask` receives
 * [n_work][nwords] pass words (bit j & 31 of word j >> 5: position j passed the coarse threshold, and the depth gate when
 * the frame ran gated), `raw` [n_work][plane] raw scores: the score at every position whose pass bit is set, 0 at every
 * other one (zeroed on the host; the device leaves stale values there).  Synchronises the stream and launches nothing.
 * dims3 is filled before the capacity test: LM_E_CAPACITY when mask_cap < n_work * nwords or raw_cap < n_work * plane
 * (mask and raw may be null with a capacity of 0, to ask for dims3).
 * LM_E_STATE on a handle with no completed frame (or a host-only one), or when the selection or the frame size has grown
 * since that frame.  Like lm_debug_plan it describes the last completed frame only between lm_complete (or lm_run) and
 * the next lm_enqueue, and while the bank, the selection and the frame size stay as they were; after a batch, its last
 * frame. */
int lm_debug_coarse(lm_detector* d, uint32_t* mask, int64_t mask_cap, uint16_t* raw, int64_t raw_cap, int32_t* dims3);
/* Test getter: the clouds the device pose stage built for the last chunk this handle enqueued (a frame is one chunk, a
 * batch one per 1024 survivors), copied from the stage's buffers to `out` (cap bytes).  Synchronises the stream and
 * launches nothing.  slot -1 with LM_POSE_CAPTURE_SLOTS: 4 int32 -- the chunk's slots, this rank's rank and world (0 and 1
 * unless the stage was shared, lm_peer_share_pose) and the run's index `first` of the chunk's first survivor: slot i
 * holds survivor first + rank + i * world (a batch's survivors in frame order).  Per slot:
 *   LM_POSE_CAPTURE_POSED      1 uint8: 1 when the survivor has a template whose box fits the frame (LL.cpp:52-55)
 *   LM_ICP_CAPTURE_COUNTS      2 int32: points of the down-sampled source and target clouds
 *   LM_ICP_CAPTURE_SOURCE      source cloud (the down-sampled model cloud), src x 3 f64
 *   LM_ICP_CAPTURE_TARGET      target cloud, tgt x 3 f64 (the source again unless use_scene_cloud)
 *   LM_ICP_CAPTURE_INIT        initial guess, 16 f64 row-major
 *   LM_POSE_CAPTURE_RAW_MODEL  the model cloud before down-sampling (what k_pose_verify reads), row-major pixel order
 *   LM_POSE_CAPTURE_RAW_SCENE  the scene cloud before down-sampling (empty without use_scene_cloud)
 *   LM_POSE_CAPTURE_WINDOW     5 int32, a track chunk only (lm_track; LM_E_STATE otherwise): the window x, y, w, h and
 *                              the status of the slot's object, for every slot
 * LM_E_STATE before any pose stage has run (and after a later one failed before it enqueued a chunk), and for every
 * item but POSED of a slot without a pose; LM_E_CAPACITY when cap is too small; LM_E_INVALID for a slot outside the chunk or an
 * item not listed.  Describes the last chunk only, until the next pose stage is enqueued. */
#define LM_POSE_CAPTURE_SLOTS 9
#define LM_POSE_CAPTURE_POSED 10
#define LM_POSE_CAPTURE_RAW_MODEL 11
#define LM_POSE_CAPTURE_RAW_SCENE 12
#define LM_POSE_CAPTURE_WINDOW 14
int lm_debug_pose_clouds(lm_detector* d, int slot, int what, void* out, int64_t cap);
/* Counters of the last lm_run: [0] templates scanned, [1] coarse candidates, [2] algorithmic bytes of
 * the coarse scan (sum over templates, modalities of features x positions; SURVEY 8d),
 * [3] algorithmic bytes of the refinement (features x 256 per refined candidate and level: the reference's work,
 * whichever kernel disposed of the candidate), [4] records kept after refinement, [5] bytes of the byte linear
 * memories the exact refinement kernel read (it stops early, exactly, on candidates that can no longer reach the
 * threshold), [6] the part of [3] that belongs to candidates the bit-sliced upper-bound filter dropped,
 * [7] bytes of H-planes that filter read.  [0],[2] describe this handle's shard.  `out8` has 8 entries. */
int lm_counters(lm_detector* d, int64_t* out8);
/* Per-stage device time in microseconds, from CUDA events recorded on the detector's stream around
 * each stage: [0] linear memories, [1] coarse scan, [2] candidate offsets, [3] refinement (= [5] + [6] + [7]),
 * [4] total, [5] candidate list + filter planes, [6] upper-bound filter, [7] exact refinement of the survivors (+ the
 * collector of the multi-GPU exchange).
 * lm_set_timing(d, slots) with slots > 0 enables it and keeps the last `slots` runs (0 disables);
 * lm_stage_times synchronises and returns the mean over the recorded runs.  `out8` has 8 entries. */
int lm_set_timing(lm_detector* d, int slots);
int lm_stage_times(lm_detector* d, float* out8);
/* The CUDA stream all work of this handle is issued on (cudaStream_t as void*). */
void* lm_stream(lm_detector* d);
/* Number of kernel launches issued by this handle since creation (the pose stage's CUB segmented sort counts as one;
 * a frame's pose stage is 5, whatever its survivor count; 6 when shared over the exchange; one fewer each with
 * LM_ICP_POINT_TO_POINT). */
int64_t lm_launch_count(lm_detector* d);
/* About the last pose stage this handle completed (lm_complete_pose / lm_complete_detect; lm_peer_detect_batch and
 * lm_peer_track_batch: see there; lm_detect_batch and lm_track_batch leave it as it was): [0] box-NMS survivors,
 * [1] hypotheses this rank refined (all survivors unshared; its share with lm_peer_share_pose, as counted by the ICP
 * kernel), [2] launches of the stage, [3] 1 if it was shared.  Zeros before the first.  `out4` has 4 entries. */
int lm_pose_stats(lm_detector* d, int64_t* out4);

/* ---- poseRefine (reference: linemodLevelup/linemodLevelup.h:8-19, linemodLevelup.cpp:27-155) ---- */
typedef struct lm_icp lm_icp; /* replaces class poseRefine's compute; the R/t/residual state lives in the caller */

int lm_icp_create(int device, lm_icp** out);
void lm_icp_destroy(lm_icp* h);

/* poseRefine::process.  sceneDepth / modelDepth: u16 millimetres, row-major; sceneK / modelK / R: 9 floats
 * row-major; t: 3 floats (mm); detectX/Y: the match position.  max_iterations: Open3D's
 * ICPConvergenceCriteria::max_iteration_ (the reference uses the default, 30).  Outputs: R_out 9
 * doubles row-major (getR), t_out 3 doubles in mm (getT), residual = ICP fitness (getResidual), or -1
 * with R_out/t_out untouched when the model box does not fit the scene at the match position
 * (early return, LL.cpp:52-55). */
int lm_icp_process(lm_icp* h, const uint16_t* scene_depth, int srows, int scols, const uint16_t* model_depth, int mrows,
                   int mcols, const float* sceneK, const float* modelK, const float* R, const float* t, int detectX,
                   int detectY, int max_iterations, double* R_out, double* t_out, float* residual);

/* The same for n hypotheses against one scene image (what the callers do for the top matches after NMS,
 * linemod_and_levelup_test.py:351-367): model_depths[i], modelK + 9i, R + 9i, t + 3i, detect_xy[2i..2i+1]; outputs
 * R_out + 9i, t_out + 3i, residual[i].  The scene and each distinct model_depths[i] (pointers may repeat) are copied to
 * the device once, then the call is lm_icp_process_batch_device's on those u16 planes; see there. */
int lm_icp_process_batch(lm_icp* h, int n_hyp, const uint16_t* scene_depth, int srows, int scols,
                         const uint16_t* const* model_depths, int mrows, int mcols, const float* sceneK, const float* modelK,
                         const float* R, const float* t, const int32_t* detect_xy, int max_iterations, double* R_out,
                         double* t_out, float* residual);

/* lm_icp_process_batch for a scene and renders already in device memory (a GPU decoder's depth, a depth network's, a GPU
 * renderer's output): the clouds are built on the device by the pose stage's kernels (k_pose_cloud, a segmented sort,
 * k_pose_voxel), fed by k_icp_scene, k_icp_render_box and k_icp_render_crop, then the ICP kernels run.
 *   Inputs     scene_depth srows x scols, rows scene_pitch BYTES apart; model_depths[i] mrows x mcols, rows
 *              model_pitches[i] bytes apart (pointers may repeat; crop views are fine).  Pixels packed within a row; every
 *              plane is device or managed memory of the handle's device.  scene_format / model_format: LM_DEPTH_U16_MM
 *              (u16 mm, as is) or LM_DEPTH_F32 (float32 d to u16 mm with scene_scale / model_scale, exactly as
 *              lm_bind_images_device converts it).  sceneK, modelK, R, t, detect_xy and the outputs are host arrays, as
 *              in lm_icp_process_batch.
 *   Semantics  R_out, t_out and residual are bit for bit lm_icp_process_batch's on the converted u16 images: the early
 *              return of LL.cpp:52-55 (residual -1, R_out / t_out untouched), all-zero renders, a zero anchor and the
 *              NaN patterns they give included.  The handle's estimation and use_scene_cloud apply.
 *   Ordering   as lm_bind_images_device: an event recorded on `stream` (a cudaStream_t; NULL = the legacy default stream)
 *              gates the reads, and `stream` waits on a second event behind the call's work.  The call returns once the
 *              outputs are on the host.
 * Both calls run on the handle's stream and synchronise it twice: once to read back the render boxes, which size the
 * crops (lm_pose.h), and once at the end.  Launches: 3 (k_icp_scene, k_icp_render_box, k_icp_render_crop) plus, per
 * chunk of 1024 hypotheses, the pose stage's 5 (LM_ICP_POINT_TO_PLANE) or 4 (LM_ICP_POINT_TO_POINT, LM_POSE_PSO), plus 1
 * per chunk when verifying; 2 when every hypothesis takes the early return; none for n_hyp 0.
 * LM_E_INVALID before any device work for a null argument, an empty image or max_iterations < 0; for
 * lm_icp_process_batch_device also for an unknown format, a non-finite or non-positive scale with LM_DEPTH_F32, a stream
 * of another device, a plane that is not device memory of the handle's device or whose pitch is shorter than a row or not
 * aligned to its elements.  LM_E_INVALID after the box read-back for a render whose box has 2^21 pixels or more
 * (lm_set_template_renders' limit), and after the chunks for a cloud that spans more than 2^21 voxels of 2.5 mm along an
 * axis (a tiny, zero or non-finite K); LM_E_CAPACITY when n_hyp (at most 1024 per chunk) renders' crops need 2^31 cloud
 * points or more.  With capture on (lm_icp_set_capture) the call also synchronises behind each chunk and copies out what
 * it built and kept; the outputs do not change.  lm_icp_last_stats and lm_icp_launch_count cover the call. */
int lm_icp_process_batch_device(lm_icp* h, int n_hyp, const void* scene_depth, int64_t scene_pitch, int scene_format,
                                float scene_scale, int srows, int scols, const void* const* model_depths,
                                const int64_t* model_pitches, int model_format, float model_scale, int mrows, int mcols,
                                const float* sceneK, const float* modelK, const float* R, const float* t,
                                const int32_t* detect_xy, int max_iterations, double* R_out, double* t_out, float* residual,
                                void* stream);

/* Of the last hypothesis with a pose: [0] points in the down-sampled cloud, [1] ICP iterations run, [2] inlier rmse (m);
 * [3] device time of the last call (us): from lm_icp_process_batch's copy of the planes, or lm_icp_process_batch_device's
 * gate on `stream`, to the end of its last chunk's kernels, the box read-back included, and k_pose_verify included when
 * the call verifies. */
int lm_icp_last_stats(lm_icp* h, double* out4);
/* NOT the reference's behaviour (default off): register the model cloud against the down-sampled SCENE
 * cloud, which is what LL.cpp:109 evidently meant to do (it down-samples the model cloud twice). */
int lm_icp_set_use_scene_cloud(lm_icp* h, int on);
/* LM_ICP_POINT_TO_PLANE (default: k_icp_normals + the ICP kernel), LM_ICP_POINT_TO_POINT (the ICP kernel alone) or
 * LM_POSE_PSO (k_pose_pso alone, with the settings of lm_icp_set_pose_search) for the next calls.  LM_E_INVALID for any
 * other value. */
int lm_icp_set_estimation(lm_icp* h, int estimation);
/* LM_POSE_PSO's settings for this handle (see lm_set_pose_search); hypothesis i of a call draws as job i. */
int lm_icp_set_pose_search(lm_icp* h, int particles, int iterations, double dt_mm, double dr_deg, double clamp_mm,
                           uint64_t seed);
int64_t lm_icp_launch_count(lm_icp* h);
/* Pose verification (see lm_set_pose_verify) for the next calls: one more launch per chunk of 1024 hypotheses.
 * lm_icp_verify: score[k], counts6 + 6k of hypothesis k of the last call, *n the hypotheses; LM_E_STATE when that call
 * did not verify.  LM_E_INVALID for a NaN or negative inlier_mm. */
int lm_icp_set_verify(lm_icp* h, int on, double inlier_mm);
int lm_icp_verify(lm_icp* h, float* score, int32_t* counts6, int64_t cap, int64_t* n);

/* ---- introspection of the ICP kernels, used by the stage-by-stage tests ---- */
/* While capture is on (default off), both calls keep, per hypothesis, what their kernels saw and kept in the last call;
 * a call that fails past its argument checks keeps nothing.  Turning capture on or off drops what was kept.  The
 * outputs do not depend on it. */
int lm_icp_set_capture(lm_icp* h, int on);
/* Copies item `what` of hypothesis `hyp` of the last call to `out` (cap bytes):
 *   COUNTS      2 int32: source and target points
 *   SOURCE      source cloud, src x 3 f64;  TARGET the target cloud, tgt x 3 f64
 *   NORMALS     target normals, tgt x 3 f64
 *   INIT        initial guess, 16 f64 row-major
 *   RESULT      19 f64: the final transformation (16, row-major), fitness, rmse, iterations
 *   KNN         tgt x 30 int32: the neighbours k_icp_normals kept (target indices, kept order, padded with -1)
 *   CORR_FIRST  src int32: the correspondence (target index, -1: none) of every source point on pass 0
 *   CORR_LAST   src int32: the same for the last pass the kernel ran (the pass whose fitness and rmse are returned)
 *   SEARCH      the swarm record of an LM_POSE_PSO call (lm_set_pose_search)
 * LM_E_STATE for a hypothesis that took the early return, and for an item the call's estimation did not compute:
 * NORMALS / KNN but with LM_ICP_POINT_TO_PLANE, CORR_* with LM_POSE_PSO, SEARCH but with LM_POSE_PSO.  LM_E_CAPACITY when
 * cap is too small, LM_E_INVALID for a hypothesis outside the last captured call. */
#define LM_ICP_CAPTURE_COUNTS 0
#define LM_ICP_CAPTURE_SOURCE 1
#define LM_ICP_CAPTURE_TARGET 2
#define LM_ICP_CAPTURE_NORMALS 3
#define LM_ICP_CAPTURE_INIT 4
#define LM_ICP_CAPTURE_RESULT 5
#define LM_ICP_CAPTURE_KNN 6
#define LM_ICP_CAPTURE_CORR_FIRST 7
#define LM_ICP_CAPTURE_CORR_LAST 8
#define LM_ICP_CAPTURE_SEARCH 13
int lm_icp_capture(lm_icp* h, int hyp, int what, void* out, int64_t cap);

#ifdef __cplusplus
}
#endif
#endif
