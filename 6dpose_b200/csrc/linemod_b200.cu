// linemod_b200.cu -- hand-written sm_90a kernels + C-ABI for the LINEMOD match hot path.
//
// Reference being replaced: linemodLevelup::Detector::match and everything below it
// (linemodLevelup/linemodLevelup.cpp of meiqua/6DPose @ 619be57, "LL.cpp"):
//   kernels (lm_kernels.cuh): k_linear_memories_band, k_coarse_packed / k_coarse_bytes, k_scan_counts, k_refine_prep,
//                             k_refine_filter_w, k_refine_bits / k_refine, k_peer_collect
//   lm_finish (host)   <- std::sort + std::unique                       LL.cpp:1772-1774
// Integer results (raw scores, x, y, template ids) are bit-exact; the float similarity is produced by
// the same two IEEE operations as the reference ((raw * 100.f) / (4 * n)).
//
// No tensor cores: bit-plane lookups / carry-save counters / small reductions.  No CPU fallback.

#include "linemod_b200.h"

#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <string>
#include <vector>

// --------------------------------------------------------------------------------------------
// error plumbing
// --------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return fail(LM_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

extern "C" const char* lm_last_error(void) { return g_err; }

// shared with lm_icp.cu
int lm_fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#include "lm_kernels.cuh"
#include "lm_frontend.cuh"
#include "lm_post.cuh"
#include "lm_pose.h"
#include "lm_buffer.h"

// Launch with programmatic stream serialization (see lm_pdl_wait in lm_kernels.cuh).
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}


// --------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------
#define LM_MAX_ROUNDS 5
#define LM_BITS_SMEM_LIMIT (200 * 1024)
#define LM_BAND_SMEM_LIMIT (160 * 1024)
#define LM_K2_SMEM_MAX (222 * 1024)  // dynamic shared memory of k_coarse_packed: bit-planes + the teams' partial counters
#define LM_CAND_DEFAULT (4ll << 20)  // candidate-list entries allocated up front (x 12 bytes)
#define LM_TEV 7  // timing events per frame: start, K1, K2, scan, prep, filter, end

struct LevelHost {
  int T = 0, rows = 0, cols = 0, Wd = 0, Hd = 0, plane = 0;
  DeviceArray<uint8_t> d_q[LM_MAX_MODALITIES];                   // owned upload buffers
  const uint8_t* q_src[LM_MAX_MODALITIES] = {nullptr, nullptr};  // what K1 reads (owned or caller's device memory)
  DeviceArray<uint8_t> d_lm;
  uint32_t mod_stride = 0;
  DeviceArray<uint32_t> d_bp;  // lowest level only: spread bit-planes [M][8][lbw]
  int lbw = 0, nwords = 0, rounds = 0;
};

// Words per label block of the lowest level's bit-planes: T*T*plane bits, then slack for the reads of lanes beyond the
// last word (a lane reads words idx and idx + 1 of a window, idx < 32 * rounds).  K1 never writes the slack, so a
// window that starts at the first slack word reads zeros in every lane (the coarse scan's zero descriptor).
static size_t bp_label_words(int T, int plane) {
  const size_t nwords = ((size_t)plane + 31) / 32, rounds = (nwords + 31) / 32;
  return (((size_t)T * T * plane + 31) / 32 + 32 * rounds + 4 + 3) & ~(size_t)3;
}

// K1 launch plan (plan_k1): block ranges per level (lowest level first), kernel variant and shared memory.
struct K1Plan {
  LinMemParams p;
  bool band = false;
  size_t smem = 0;
  int blocks = 0;
};

// Launch shape of k_coarse_packed (coarse_shape).
struct CoarseShape {
  bool smem;          // the bit-planes are staged in shared memory (k_coarse_packed<true>)
  int split, wpc, grid;
  size_t smem_bytes;  // dynamic shared memory: bit-planes + the teams' partial counters
};

// The kernel routes of the handle's frame, decided once by plan_frame: its stages launch from it, an overflow replay
// reruns its refinement from it, lm_debug_plan reports it.  Decisions only: what a replay may grow is resolved at launch.
struct FramePlan {
  K1Plan k1;                  // one K1 launch for every level: byte linear memories, H-planes, the lowest level's bit-planes
  int planes_level = -1;      // level K1 builds as H-planes only (-1: none)
  int stale = 0;              // levels (bit l) K1 leaves without byte linear memories (lm_debug_linear_memories builds them)
  bool gated = false;         // k_depth_cells, then the coarse kernels' gated instantiations
  bool packed = false;        // k_coarse_packed on the templates the bit-sliced scan takes, launched as `coarse`
  CoarseShape coarse = {};
  size_t plane_bytes = 0;     // the lowest level's bit-planes, which k_coarse_packed's shape follows
  bool bytes = false;         // k_coarse_bytes on the others
  bool scan_fused = false;    // k_coarse_packed scans the candidate counts itself: no k_scan_counts
  bool filter = false;        // k_refine_filter_w on the first refined level
  bool bits = false;          // k_refine_bits finishes the filter's survivors (two levels)
  bool bits_publish = false;  // ... and, as the frame's last appending kernel, publishes it to the peers
  bool refine = false;        // k_refine<filter>, byte-wise: the templates the filter does not take, or every candidate
  bool exchange = false;      // records go to this rank's block of the peer exchange, packed by k_peer_collect
};

// The stages enqueued for the handle's frame, each with the arguments a replay needs (complete_frame).  lm_enqueue sets
// the match's; every later lm_enqueue_* raises its stage's flag, and the completion that waits for a stage lowers it.
struct FrameChain {
  float threshold = 0.f; FramePlan plan;                    // lm_enqueue
  bool completed = false;  // lm_complete returned: the header, first records and counters are on the host (until a new
                           // frame, bank, selection, result block or exchange)
  bool post = false; double iou = 0.5; int top_k = 0;      // lm_enqueue_post
  bool pose = false; float sK[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  int max_iter = 30, use_scene = 0, estimation = LM_ICP_POINT_TO_PLANE;  // lm_enqueue_pose
  PoseVerifyOptions verify = {0, LM_VERIFY_RANK_FITNESS, 10.0, -INFINITY};
  PoseSearch search = pose_search_default();                // LM_POSE_PSO's settings
  bool pose_nms = false; double nms_thr = 40.0;             // lm_enqueue_pose_nms
};

struct lm_detector {
  int device = 0;
  // streams and events first: they outlive the buffers, which are freed in reverse order of declaration
  Stream stream;
  // host uploads: the upper-level label images travel on a second stream while the lowest level's linear
  // memories and the coarse scan already run (they only need the lowest level)
  Stream copy_stream;
  Event ev_fork, ev_upper;
  // lm_bind_images_device: the caller's stream up to the call -> the ingest -> the caller's stream after it
  Event ev_in, ev_out;
  std::vector<Event> tev;  // timing slots x LM_TEV events (ring)
  bool upper_pending = false;
  int L = 0, M = LM_MAX_MODALITIES;
  int T[LM_MAX_LEVELS] = {0};
  LevelHost lv[LM_MAX_LEVELS];
  bool have_frame = false;
  FrameChain chain;

  // bank (host)
  int n_classes = 0, S = 0, G = 0;
  std::vector<int32_t> class_begin, tmeta, feats;
  std::vector<uint8_t> feat_slot;  // slot (level*M+modality) of every feature
  // bank (device), prepared for the current frame size
  DeviceArray<TSlot> d_tslot;
  DeviceArray<uint32_t> d_fbase;
  DeviceArray<uint32_t> d_fxy;
  DeviceArray<uint32_t> d_fdesc;     // lowest-level features for k_coarse_packed, one word each (coarse_descriptors)
  DeviceArray<int2> d_k2info;        // [G]: first descriptor, lowest-level features
  std::vector<uint8_t> bits_ok;      // per template: the bit-sliced coarse kernel may take it
  std::vector<uint8_t> safe;         // per template: refinement never skips a feature (LL.cpp:1394)
  DeviceArray<uint8_t> d_safe;
  DeviceArray<uint16_t> d_galign;    // [G][S][16] feature counts per (address & 15) group
  // refinement filter (k_refine_filter_w) on the first refined level lr = L - 2: column-major H-planes + descriptors
  bool filter_ok = false;            // the current frame size / bank allow it
  // H-planes + zero tail, then the N-planes + zero tail at word rp_noff (N word = H word + rp_noff)
  DeviceArray<uint32_t> d_rp; int rp_nyb = 0; uint32_t rp_noff = 0;
  DeviceArray<uint32_t> d_rdesc;     // per feature of level lr, grouped per template, padded to multiples of 32
  int bits_grid = 0;                 // k_refine_bits CTAs: the resident ones (occupancy x SMs), 0 = not yet asked
  bool shard_all_eligible = false;   // every template of the shard is taken by the filter (no byte-wise refinement)
  DeviceArray<uint32_t> d_surv2;     // candidates of the templates the filter does not take
  DeviceArray<int2> d_rfeat;         // per template: first descriptor, count
  std::vector<int2> h_rfeat;
  DeviceArray<int4> d_finfo;         // per work item of the shard: first descriptor, count, width | height << 16,
                                     // flags | need << 8 (need: for the threshold of the call, see filter_thresholds)
  std::vector<int4> h_finfo;         // .w = flags only
  std::vector<int4> h_finfo_up;      // upload staging
  bool finfo_valid = false; float finfo_threshold = 0.f;
  DeviceArray<uint2> d_cand;         // ordered candidate list (k_refine_prep), cand_cap entries
  int64_t cand_need = 0;             // candidates of a frame that overflowed the list
  DeviceArray<uint32_t> d_surv;      // survivors of the filter [cand_cap]
  DeviceArray<int> d_queue;          // [0] next candidate, [1] survivors
  int prep_rows[LM_MAX_LEVELS] = {0}, prep_cols[LM_MAX_LEVELS] = {0};
  bool prepared = false;
  std::vector<TSlot> h_tslot;
  std::vector<uint8_t> feat_skip_low;

  // selection / shard
  std::vector<int32_t> sel;  // global template ids of the whole selected sequence
  int64_t shard_begin = 0, shard_count = 0;  // contiguous layout: [begin, begin + count) of sel
  int shard_index = 0, shard_n = 1;
  int shard_layout = LM_SHARD_CONTIGUOUS;
  int64_t work_base = 0, work_stride = 1;    // entry w of the shard is sel[work_base + w * work_stride]
  std::vector<int32_t> shard_sel;            // global template ids of this shard, in order
  DeviceArray<int32_t> d_work;
  int n_items_bits = 0;                                     // work items per coarse kernel
  DeviceArray<int32_t> d_items_bytes; int n_items_bytes = 0;
  DeviceArray<int2> d_k2task;                               // k_coarse_packed's task table of the shard (coarse_task_table)
  int k2_full = 0, k2_rem = 0, k2_tasks = 0;                // full tasks, remainder words, all tasks
  bool work_dirty = true;

  // per-run buffers
  DeviceArray<uint32_t> d_mask;      // [n_work][nwords] coarse pass bits
  DeviceArray<uint16_t> d_raw;       // [n_work][plane] coarse raw scores (passing cells)
  DeviceArray<int32_t> d_cnt, d_off;
  // result block (device): lm_result_header + capacity records (res_bytes); internal unless the caller set one
  lm_result_header* d_res = nullptr; int64_t res_cap = 0; bool res_external = false;
  DeviceArray<uint8_t> d_res_own;
  DeviceArray<unsigned long long> d_counters;
  PinnedArray<unsigned long long> h_counters;
  PinnedArray<uint8_t> h_res;        // staging: header + records
  int64_t h_valid = 0;               // records already copied to h_res

  std::vector<int> class_of;            // template -> class (lm_finish), rebuilt when the bank changes
  std::vector<int32_t> order_cnt;       // order_records scratch
  std::vector<lm_record> order_tmp, finish_rec;
  std::vector<uint8_t> finish_keys;

  // post-match stage (lm_post.cuh): greedy NMS on the device, top-k survivors to the host
  std::vector<int32_t> boxes;           // [G][2] caller's box sizes (empty: L0 template width/height)
  DeviceArray<PostInfo> d_post_info; bool post_dirty = true;
  DeviceArray<lm_match> d_post_out; PinnedArray<lm_match> h_post_out;  // LM_POST_MAX survivors
  DeviceArray<int32_t> d_post_counts; PinnedArray<int32_t> h_post_counts;
  DeviceArray<uint8_t> d_post_live;
  DeviceArray<PostKey> d_post_keys;  // k_post_nms's sort keys beyond LM_POST_SMEM_KEYS records

  // pose stage behind the NMS (lm_pose.h): per-template render crops, refinement of the survivors on the device
  lm_pose_stage* pose = nullptr;
  bool frame_depth = false;             // the frame came from lm_upload_images: fe_depth holds its depth
  int pose_estimation = LM_ICP_POINT_TO_PLANE;  // lm_set_pose_estimation: for the next pose stage
  PoseVerifyOptions pose_verify = {0, LM_VERIFY_RANK_FITNESS, 10.0, -INFINITY};  // lm_set_pose_verify: likewise
  PoseSearch pose_search = pose_search_default();  // lm_set_pose_search: likewise
  int track_views = 0; double track_view_tau = 0.0;  // lm_set_track_views: for the next track calls
  int64_t pose_stats[4] = {0, 0, 0, 0};  // lm_pose_stats of the last completed pose stage

  // multi-GPU exchange fused into k_refine (lm_peer_*)
  DeviceArray<uint8_t> px_buf;          // this rank's exchange buffer (IPC-exportable device memory)
  int64_t px_cap = 0;                   // records per block
  int px_world = 0, px_rank = -1;       // px_rank >= 0: connected
  bool px_ipc = false;                  // peer bases opened with cudaIpcOpenMemHandle
  uint8_t* px_base[LM_MAX_PEERS] = {nullptr};
  int32_t px_seq = 0;
  unsigned long long px_timeout_ns = 1000000000ull;  // collector gives up on a peer after 1 s (LINEMOD_B200_PEER_TIMEOUT_MS)
  bool px_share_pose = false;           // lm_peer_share_pose: the pose stage is divided over the ranks
  int32_t px_pose_seq = 0;              // pose exchanges so far: one per shared frame, one per chunk of a shared batch or track run
  DeviceArray<PeerExchange> d_px;       // device copy of the descriptor (static after connect)
  PeerExchange h_px;

  // GPU quantization front-end (lm_upload_images): per level colour image, unfiltered bins, gate, normals, masks
  struct FeLevel {
    int rows = 0, cols = 0;
    DeviceArray<uint8_t> src, qun, strong, normal;
    DeviceArray<uint8_t> mask[LM_MAX_MODALITIES];
  } fe[LM_MAX_LEVELS];
  DeviceArray<uint16_t> fe_depth; DeviceArray<uint8_t> fe_nraw;
  bool fe_lut = false;

  // depth gate of the coarse scan (lm_set_depth_gate)
  std::vector<float> tdepth;            // training distance per template of the bank (mm; NaN / <= 0: never gated)
  bool gate_on = false; double gate_tau = 0.0;
  bool gate_dirty = true;               // h_gate_item no longer fits the shard / distances / tolerance
  std::vector<uint2> h_gate_item;       // per work item of the shard: band and sample-cell offset (DepthGate::item)
  int64_t gate_with_z = 0;              // work items of the shard with a distance
  DeviceArray<uint2> d_gate_item;
  DeviceArray<uint32_t> d_cells;
  DeviceArray<unsigned> d_gate_before;

  bool timing = false;
  int64_t timing_runs = 0;
  int64_t launches = 0;
  int64_t alg_scan_bytes = 0;
  int sm_count = 132;

  ~lm_detector() { pose_stage_destroy(pose); }
};

// A result block: lm_result_header, then records.
static size_t res_bytes(int64_t records) { return sizeof(lm_result_header) + sizeof(lm_record) * (size_t)records; }
static int64_t res_records(size_t bytes) { return bytes ? (int64_t)((bytes - sizeof(lm_result_header)) / sizeof(lm_record)) : 0; }
static lm_result_header* hres(const lm_detector* d) { return reinterpret_cast<lm_result_header*>(d->h_res.get()); }
// The candidate lists are allocated together, d_surv2 last: its size is theirs.
static int64_t cand_cap(const lm_detector* d) { return (int64_t)d->d_surv2.size(); }

extern "C" int lm_create(int device, int n_levels, const int* T, lm_detector** out) {
  if (!out) return fail(LM_E_INVALID, "out is null");
  if (n_levels < 1 || n_levels > LM_MAX_LEVELS) return fail(LM_E_INVALID, "pyramid levels must be 1..%d", LM_MAX_LEVELS);
  for (int l = 0; l < n_levels; ++l)
    if (T[l] < 1 || T[l] > 16) return fail(LM_E_INVALID, "T[%d]=%d outside 1..16", l, T[l]);
  if (device == -1) {
    // host-only handle: bank / selection / shard ranges / lm_finish work, every GPU stage refuses to run
    lm_detector* d = new lm_detector();
    d->device = -1;
    d->L = n_levels;
    for (int l = 0; l < n_levels; ++l) d->T[l] = T[l];
    *out = d;
    return LM_OK;
  }
  const int rc = open_device(device);
  if (rc) return rc;
  std::unique_ptr<lm_detector> d(new lm_detector());
  d->device = device;
  d->L = n_levels;
  for (int l = 0; l < n_levels; ++l) d->T[l] = T[l];
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  d->sm_count = prop.multiProcessorCount;
  // function attributes are per DEVICE: every handle raises the dynamic shared-memory limits on its own device
  // (a process may hold handles on several GPUs, e.g. lm_peer_connect_local across devices)
  CU(cudaFuncSetAttribute(k_linear_memories_band, cudaFuncAttributeMaxDynamicSharedMemorySize, LM_BAND_SMEM_LIMIT));
  CU(cudaFuncSetAttribute(k_coarse_packed<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LM_K2_SMEM_MAX));
  CU(cudaFuncSetAttribute(k_coarse_packed<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  CU(cudaFuncSetAttribute(k_coarse_packed<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LM_K2_SMEM_MAX));
  CU(cudaFuncSetAttribute(k_coarse_packed<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  CU(cudaFuncSetAttribute(k_post_nms, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(PostKey) * LM_POST_SMEM_KEYS)));
  CU(d->stream.create(cudaStreamNonBlocking));
  CU(d->copy_stream.create(cudaStreamNonBlocking));
  CU(d->ev_fork.create(cudaEventDisableTiming));
  CU(d->ev_upper.create(cudaEventDisableTiming));
  CU(d->d_counters.assign(8));
  CU(cudaMemset(d->d_counters.get(), 0, 8 * sizeof(unsigned long long)));
  CU(d->h_counters.assign(8));
  memset(d->h_counters.get(), 0, 8 * sizeof(unsigned long long));
  CU(d->d_queue.assign(4));
  CU(cudaMemset(d->d_queue.get(), 0, 4 * sizeof(int)));
  *out = d.release();
  return LM_OK;
}

static void peer_release(lm_detector* d) {
  if (d->px_ipc)
    for (int r = 0; r < d->px_world; ++r)
      if (r != d->px_rank && d->px_base[r]) cudaIpcCloseMemHandle(d->px_base[r]);
  for (int r = 0; r < LM_MAX_PEERS; ++r) d->px_base[r] = nullptr;
  d->px_rank = -1;
  d->px_ipc = false;
  d->px_buf.reset();
  d->d_px.reset();
  d->px_world = 0;
  d->px_cap = 0;
  d->px_share_pose = false;
}

extern "C" void lm_destroy(lm_detector* d) {
  if (!d) return;
  if (d->device >= 0) {
    cudaSetDevice(d->device);
    if (d->stream.get()) cudaStreamSynchronize(d->stream.get());
    if (d->copy_stream.get()) cudaStreamSynchronize(d->copy_stream.get());
    peer_release(d);
  }
  delete d;
}

extern "C" void* lm_stream(lm_detector* d) { return d ? (void*)d->stream.get() : nullptr; }
extern "C" int64_t lm_launch_count(lm_detector* d) { return d ? d->launches : 0; }

extern "C" int lm_load_bank(lm_detector* d, int n_classes, const int32_t* class_begin, int n_slots, const int32_t* tmeta,
                            const int32_t* feats, int64_t n_feats) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (n_classes < 0 || !class_begin) return fail(LM_E_INVALID, "bad class table");
  if (n_slots != d->L * d->M)
    return fail(LM_E_INVALID, "template pyramids have %d templates, detector expects %d (levels x modalities)", n_slots,
                d->L * d->M);
  // the box NMS orders matches by a key of 12 bits of class and 20 of template_id (lm_post.cuh)
  if (n_classes > 4096) return fail(LM_E_INVALID, "bank of %d classes: at most 4096", n_classes);
  const int G = class_begin[n_classes];
  if (class_begin[0] != 0) return fail(LM_E_INVALID, "class_begin[0] must be 0");
  for (int c = 0; c < n_classes; ++c) {
    if (class_begin[c + 1] < class_begin[c]) return fail(LM_E_INVALID, "class_begin not monotone");
    if (class_begin[c + 1] - class_begin[c] > (1 << 20))
      return fail(LM_E_INVALID, "class %d has %d templates: at most 1048576", c, class_begin[c + 1] - class_begin[c]);
  }
  std::vector<uint8_t> slot_of((size_t)n_feats, 255);
  for (int g = 0; g < G; ++g)
    for (int s = 0; s < n_slots; ++s) {
      const int32_t* m4 = tmeta + ((size_t)g * n_slots + s) * 4;
      if (m4[2] < 0 || m4[3] < 0 || (int64_t)m4[2] + m4[3] > n_feats)
        return fail(LM_E_INVALID, "template %d slot %d: feature range out of bounds", g, s);
      if (m4[3] > 8191)  // CV_Assert(templ.features.size() <= 8191), LL.cpp:1291
        return fail(LM_E_INVALID, "template %d slot %d has %d features (> 8191)", g, s, m4[3]);
      if (m4[0] < 0 || m4[1] < 0 || m4[0] > 32767 || m4[1] > 32767)
        return fail(LM_E_INVALID, "template %d slot %d: width/height outside 0..32767", g, s);
      for (int i = 0; i < m4[3]; ++i) {
        const int32_t* f = feats + ((size_t)m4[2] + i) * 3;
        if (f[2] < 0 || f[2] > 7) return fail(LM_E_INVALID, "feature label %d outside [0,8)", f[2]);
        if (f[0] < 0 || f[1] < 0 || f[0] > 32767 || f[1] > 32767)
          return fail(LM_E_INVALID, "feature coordinate (%d,%d) outside 0..32767", f[0], f[1]);
        slot_of[(size_t)m4[2] + i] = (uint8_t)s;
      }
    }
  if (d->device >= 0) CU(cudaSetDevice(d->device));
  d->n_classes = n_classes;
  d->S = n_slots;
  d->G = G;
  d->class_begin.assign(class_begin, class_begin + n_classes + 1);
  d->tmeta.assign(tmeta, tmeta + (size_t)G * n_slots * 4);
  d->class_of.clear();
  d->boxes.clear();  // box sizes belong to the bank they were set for
  d->post_dirty = true;
  d->tdepth.clear();  // so do the training distances
  d->gate_dirty = true;
  if (d->pose) pose_stage_clear(d->pose);  // so do the template renders
  d->feats.assign(feats, feats + (size_t)n_feats * 3);
  d->feat_slot.swap(slot_of);
  d->d_tslot.reset(); d->d_fbase.reset(); d->d_fxy.reset(); d->d_fdesc.reset(); d->d_k2info.reset();
  if (d->device >= 0 && G > 0) CU(d->d_tslot.assign((size_t)G * n_slots));
  if (d->device >= 0 && n_feats > 0) {
    CU(d->d_fbase.assign((size_t)n_feats));
    CU(d->d_fxy.assign((size_t)n_feats));
  }
  d->prepared = false;
  d->chain.completed = false;
  // default selection: everything, one shard
  return lm_select(d, nullptr, -1, 0, 1);
}

// Which accumulator width the reference would use and whether it would assert (LL.cpp:1813-1824).
static int check_paths(const lm_detector* d, int g) {
  for (int l = 0; l < d->L; ++l) {
    int width = -1;
    for (int m = 0; m < d->M; ++m) {
      const int nf = d->tmeta[((size_t)g * d->S + l * d->M + m) * 4 + 3];
      if (width <= 0) width = nf < 64 ? 1 : (nf < 8192 ? 2 : width);
      if (width == 1 && nf > 63) return -1;  // CV_Assert(features.size() <= 63), LL.cpp:1457/1551
    }
  }
  return 0;
}

extern "C" int lm_select(lm_detector* d, const int32_t* class_sel, int n_classes_sel, int shard_index, int shard_count) {
  return lm_select_layout(d, class_sel, n_classes_sel, shard_index, shard_count, LM_SHARD_CONTIGUOUS);
}

extern "C" int lm_select_layout(lm_detector* d, const int32_t* class_sel, int n_classes_sel, int shard_index, int shard_count,
                                int layout) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (layout != LM_SHARD_CONTIGUOUS && layout != LM_SHARD_INTERLEAVED) return fail(LM_E_INVALID, "unknown shard layout %d", layout);
  if (shard_count < 1 || shard_index < 0 || shard_index >= shard_count) return fail(LM_E_INVALID, "bad shard %d/%d", shard_index, shard_count);
  std::vector<int32_t> sel;
  if (n_classes_sel < 0) {
    sel.resize(d->G);
    for (int g = 0; g < d->G; ++g) sel[g] = g;
  } else {
    for (int i = 0; i < n_classes_sel; ++i) {
      const int c = class_sel[i];
      if (c < 0 || c >= d->n_classes) return fail(LM_E_INVALID, "class index %d out of range", c);
      for (int g = d->class_begin[c]; g < d->class_begin[c + 1]; ++g) sel.push_back(g);
    }
  }
  for (int32_t g : sel)
    if (check_paths(d, g) != 0)
      return fail(LM_E_INVALID, "template %d: first modality has < 64 features but another has > 63 "
                                "(the reference asserts in similarity_64)", g);
  // contiguous shard, balanced by lowest-level feature count (the coarse scan's work per template)
  const int low = (d->L - 1) * d->M;
  std::vector<int64_t> cum(sel.size() + 1, 0);
  for (size_t i = 0; i < sel.size(); ++i) {
    int64_t c = 1;
    for (int m = 0; m < d->M; ++m) c += d->tmeta[((size_t)sel[i] * d->S + low + m) * 4 + 3];
    cum[i + 1] = cum[i] + c;
  }
  auto cut = [&](int k) -> int64_t {
    if (k <= 0) return 0;
    if (k >= shard_count) return (int64_t)sel.size();
    const int64_t target = cum.back() * k / shard_count;
    return (int64_t)(std::lower_bound(cum.begin(), cum.end(), target) - cum.begin());
  };
  d->shard_index = shard_index;
  d->shard_n = shard_count;
  d->shard_layout = layout;
  if (layout == LM_SHARD_INTERLEAVED) {
    // entry w of shard r is element r + w * N of the selected sequence: neighbouring templates (views / in-plane
    // variants of one another, which pass or fail together) are dealt round the ranks, so the candidate load per
    // rank evens out where contiguous blocks do not
    d->work_base = shard_index;
    d->work_stride = shard_count;
    d->shard_begin = shard_index;
    d->shard_count = ((int64_t)sel.size() - shard_index + shard_count - 1) / shard_count;
    if (d->shard_count < 0) d->shard_count = 0;
  } else {
    d->shard_begin = cut(shard_index);
    d->shard_count = cut(shard_index + 1) - d->shard_begin;
    d->work_base = d->shard_begin;
    d->work_stride = 1;
  }
  d->shard_sel.resize((size_t)d->shard_count);
  for (int64_t w = 0; w < d->shard_count; ++w) d->shard_sel[(size_t)w] = sel[(size_t)(d->work_base + w * d->work_stride)];
  d->sel.swap(sel);  // after the cuts: the lambda reads `sel`
  d->work_dirty = true;
  d->post_dirty = true;
  d->gate_dirty = true;
  d->chain.completed = false;
  return LM_OK;
}

extern "C" int lm_shard_range(lm_detector* d, int64_t* begin, int64_t* count) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (begin) *begin = d->shard_begin;
  if (count) *count = d->shard_count;
  return LM_OK;
}

// k_coarse_packed's feature descriptors: one word per lowest-level feature,
//   bits 0-4  bit shift of the window inside its first word (inner & 31),
//   bit 5     label 0: the lower neighbour label's plane is 7 planes up,
//   bit 6     label 7: the upper neighbour label's plane is 7 planes down,
//   bits 7-31 word offset of the window in the plane buffer: (m * 8 + label) * lbw + (inner >> 5),
// with inner = the feature's bit position inside its label block.  The neighbour labels' windows lie one plane below and
// above (lbw words), or 7 planes the other way at the two ends.  Features outside the level (LL.cpp:1330) and the padding
// get the zero descriptor: a window at the first slack word of label block 1, whose own and neighbours' windows read
// zeros (bp_label_words), so the kernel's loop has neither a skip branch nor a bounds check.  The features of a template
// (all modalities, in order) lie end to end from info.x, info.y of them, padded to a multiple of 32 so that one warp
// loads 32 of them with one aligned 128-byte load.  A template fits when every word offset does (25 bits); one that
// does not gets no descriptors and fits = 0.
#define LM_DESC_WORD_BITS 25
static uint32_t coarse_zero_descriptor(int T, int plane) {
  return (uint32_t)((bp_label_words(T, plane) + ((size_t)T * T * plane + 31) / 32) << 7);
}
static void coarse_descriptors(const int32_t* feats, const int32_t* tmeta, int G, int S, int M, int slot_low, int T, int rows,
                               int cols, std::vector<uint32_t>& desc, std::vector<int2>& info, std::vector<uint8_t>& fits) {
  const int Wd = cols / T, Hd = rows / T, plane = Wd * Hd;
  const uint64_t lbw = bp_label_words(T, plane);
  const uint32_t zero = coarse_zero_descriptor(T, plane);
  const bool zero_fits = lbw + ((uint64_t)T * T * plane + 31) / 32 < (1ull << LM_DESC_WORD_BITS);
  desc.clear();
  info.assign((size_t)G, make_int2(0, 0));
  fits.assign((size_t)G, 0);
  for (int g = 0; g < G; ++g) {
    const size_t first = desc.size();
    bool ok = zero_fits;
    int n = 0;
    for (int m = 0; m < M; ++m) {
      const int32_t* tm = &tmeta[((size_t)g * S + slot_low + m) * 4];
      for (int k = 0; k < tm[3]; ++k, ++n) {
        const int32_t* f = &feats[3 * ((size_t)tm[2] + k)];
        const int x = f[0], y = f[1], lab = f[2];
        if (x >= cols || y >= rows) {
          desc.push_back(zero);
          continue;
        }
        const uint64_t inner = (uint64_t)((y % T) * T + (x % T)) * plane + (uint64_t)(y / T) * Wd + (x / T);
        const uint64_t wh = (uint64_t)(m * 8 + lab) * lbw + (inner >> 5);
        ok = ok && wh < (1ull << LM_DESC_WORD_BITS);
        desc.push_back((uint32_t)(wh << 7) | ((lab == 7) ? 0x40u : 0u) | ((lab == 0) ? 0x20u : 0u) | (uint32_t)(inner & 31));
      }
    }
    if (!ok) {
      desc.resize(first);
      info[(size_t)g] = make_int2((int)first, 0);
      continue;
    }
    while ((desc.size() - first) % 32) desc.push_back(zero);
    info[(size_t)g] = make_int2((int)first, n);
    fits[(size_t)g] = 1;
  }
}

extern "C" int lm_coarse_descriptors(const int32_t* feats, const int32_t* tmeta, int G, int S, int M, int slot_low, int T,
                                     int rows, int cols, uint32_t* desc, int64_t cap, int64_t* n_desc, int32_t* info,
                                     uint8_t* fits, uint32_t* zero) {
  if (G < 0 || (G > 0 && (!feats || !tmeta)) || M < 1 || slot_low < 0 || slot_low + M > S || T < 1 ||
      rows < T || cols < T)
    return fail(LM_E_INVALID, "bad arguments");
  for (int64_t i = 0; i < (int64_t)G * M; ++i) {
    const int32_t* tm = &tmeta[((size_t)(i / M) * S + slot_low + i % M) * 4];
    if (tm[2] < 0 || tm[3] < 0) return fail(LM_E_INVALID, "template %lld: bad feature range", (long long)(i / M));
  }
  std::vector<uint32_t> d;
  std::vector<int2> k2;
  std::vector<uint8_t> ok;
  coarse_descriptors(feats, tmeta, G, S, M, slot_low, T, rows, cols, d, k2, ok);
  if (n_desc) *n_desc = (int64_t)d.size();
  if (zero) *zero = coarse_zero_descriptor(T, (cols / T) * (rows / T));
  for (int g = 0; g < G; ++g) {
    if (info) { info[2 * g] = k2[(size_t)g].x; info[2 * g + 1] = k2[(size_t)g].y; }
    if (fits) fits[g] = ok[(size_t)g];
  }
  if (desc) {
    if (cap < (int64_t)d.size()) return fail(LM_E_CAPACITY, "%lld descriptors, room for %lld", (long long)d.size(), (long long)cap);
    std::copy(d.begin(), d.end(), desc);
  }
  return LM_OK;
}

// Feature addresses depend on the frame size (Wd, Hd); recomputed when it changes.
static int prepare_bank(lm_detector* d) {
  bool same = d->prepared;
  for (int l = 0; l < d->L && same; ++l) same = d->prep_rows[l] == d->lv[l].rows && d->prep_cols[l] == d->lv[l].cols;
  if (same) return LM_OK;
  const size_t nf = d->feat_slot.size();
  std::vector<uint32_t> fbase(nf, 0), fxy(nf, 0);
  const int low_level = d->L - 1;
  for (size_t i = 0; i < nf; ++i) {
    const int s = d->feat_slot[i];
    if (s == 255) continue;  // feature not referenced by any template
    const int l = s / d->M, m = s % d->M;
    const LevelHost& lv = d->lv[l];
    const int x = d->feats[3 * i], y = d->feats[3 * i + 1], lab = d->feats[3 * i + 2];
    const int T = lv.T;
    const uint64_t a = (uint64_t)m * lv.mod_stride + (uint64_t)lab * T * T * lv.plane +
                       (uint64_t)((y % T) * T + (x % T)) * lv.plane + (uint64_t)(y / T) * lv.Wd + (x / T);
    fbase[i] = (uint32_t)a;
    uint32_t v = (uint32_t)x | ((uint32_t)y << 16);
    if (x >= lv.cols || y >= lv.rows) v |= LM_SKIP_BIT;  // LL.cpp:1330
    fxy[i] = v;
  }
  d->h_tslot.resize((size_t)d->G * d->S);
  for (int g = 0; g < d->G; ++g)
    for (int s = 0; s < d->S; ++s) {
      const int32_t* m4 = &d->tmeta[((size_t)g * d->S + s) * 4];
      const LevelHost& lv = d->lv[s / d->M];
      const int wf = (m4[0] - 1) / lv.T + 1, hf = (m4[1] - 1) / lv.T + 1;  // LL.cpp:1299-1300
      TSlot t;
      t.x = m4[2];
      t.y = m4[3];
      t.z = (lv.Hd - hf) * lv.Wd + (lv.Wd - wf) + 1;  // LL.cpp:1309
      t.w = (int)((uint32_t)m4[0] | ((uint32_t)m4[1] << 16));
      d->h_tslot[(size_t)g * d->S + s] = t;
    }
  // the bit-sliced coarse kernel counts in 8 bits and masks once: it takes templates with at most 255
  // lowest-level features in total and the same template_positions in every modality
  d->bits_ok.assign((size_t)d->G, 0);
  {
    const LevelHost& lv = d->lv[low_level];
    for (int g = 0; g < d->G && !lv.d_bp.empty(); ++g) {
      int total = 0;
      bool same = true;
      const TSlot& t0 = d->h_tslot[(size_t)g * d->S + low_level * d->M];
      for (int m = 0; m < d->M; ++m) {
        const TSlot& t = d->h_tslot[(size_t)g * d->S + low_level * d->M + m];
        total += t.y;
        same = same && t.z == t0.z;
      }
      d->bits_ok[g] = (total <= 255 && same) ? 1 : 0;
    }
  }
  // k_coarse_packed descriptors (coarse_descriptors); a template whose descriptors do not fit goes to k_coarse_bytes
  d->d_fdesc.reset();
  d->d_k2info.reset();
  {
    const LevelHost& lv = d->lv[low_level];
    if (!lv.d_bp.empty() && d->G > 0) {
      std::vector<uint32_t> desc;
      std::vector<int2> k2;
      std::vector<uint8_t> fits;
      coarse_descriptors(d->feats.data(), d->tmeta.data(), d->G, d->S, d->M, low_level * d->M, lv.T, lv.rows, lv.cols, desc,
                         k2, fits);
      for (int g = 0; g < d->G; ++g) d->bits_ok[g] &= fits[g];
      CU(upload(d->d_fdesc, desc, d->stream.get(), 1));
      CU(upload(d->d_k2info, k2, d->stream.get()));
      CU(cudaStreamSynchronize(d->stream.get()));
    }
  }
  // "safe" templates: at every refined level the clamp range is regular (max >= border) and every
  // feature lies inside the template box, so no feature can leave the image once a clamped patch
  // offset is applied (LL.cpp:1394 never skips) -- the refinement kernel then drops the per-feature test
  d->safe.assign((size_t)d->G, 0);
  for (int g = 0; g < d->G; ++g) {
    bool ok = true;
    for (int l = 0; l + 1 < d->L && ok; ++l) {
      const LevelHost& lv = d->lv[l];
      const int32_t* t0 = &d->tmeta[((size_t)g * d->S + l * d->M) * 4];
      const int border = 8 * lv.T;
      ok = lv.cols - t0[0] - border >= border && lv.rows - t0[1] - border >= border;
      for (int m = 0; m < d->M && ok; ++m) {
        const int32_t* tm = &d->tmeta[((size_t)g * d->S + l * d->M + m) * 4];
        for (int k = 0; k < tm[3] && ok; ++k) {
          const int32_t* f = &d->feats[3 * ((size_t)tm[2] + k)];
          ok = f[0] <= t0[0] && f[1] <= t0[1];
        }
      }
    }
    d->safe[g] = ok ? 1 : 0;
  }
  // refined levels: store each template's features grouped by (address & 15) -- sums do not depend
  // on the order, and the refinement kernel then knows the row alignment of a whole group at once
  std::vector<uint16_t> galign((size_t)d->G * d->S * 16, 0);
  for (int g = 0; g < d->G; ++g)
    for (int s = 0; s < d->S - d->M; ++s) {  // every slot above the lowest level
      const int32_t* tm = &d->tmeta[((size_t)g * d->S + s) * 4];
      const size_t b0 = (size_t)tm[2];
      const int n = tm[3];
      std::vector<int> order(n);
      for (int k = 0; k < n; ++k) order[k] = k;
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return (fbase[b0 + a] & 15u) < (fbase[b0 + b] & 15u); });
      std::vector<uint32_t> tb(n), tx(n);
      for (int k = 0; k < n; ++k) {
        tb[k] = fbase[b0 + order[k]];
        tx[k] = fxy[b0 + order[k]];
        ++galign[((size_t)g * d->S + s) * 16 + (tb[k] & 15u)];
      }
      for (int k = 0; k < n; ++k) { fbase[b0 + k] = tb[k]; fxy[b0 + k] = tx[k]; }
    }
  CU(upload(d->d_galign, galign, d->stream.get()));
  // refinement filter (k_refine_filter_w) on the first refined level: column-major H-planes [M*8*T*T][nyb][Wd] and one
  // descriptor per feature = plane word offset (incl. x / T) : 23 | y / T : 9.  Eligible templates ("safe", so that
  // the 16x16 patch of every feature is a true 2-D window of the level, and at most 511 features at that level) get
  // bit 1 of their flag byte; the others go to k_refine unfiltered.  The exact pass (k_refine_bits) also reads the
  // N-planes, same layout, behind the H-planes and their tail: a descriptor's N window is its H window + rp_noff words.
  d->filter_ok = false;
  std::vector<uint32_t> rdesc;
  std::vector<int2> rfeat((size_t)d->G, make_int2(0, 0));
  if (d->L >= 2) {
    const int lr = d->L - 2;
    const LevelHost& lv = d->lv[lr];
    const int T = lv.T, T2 = T * T;
    const int nyb = lv.Hd >= 16 ? ((lv.Hd - 16) >> 4) + 1 : 0;
    const size_t words = (size_t)d->M * 8 * T2 * nyb * lv.Wd;
    // all-zero tail behind the planes: where the padding descriptors (and nothing else) point
    const size_t tail = (size_t)(nyb + 1) * lv.Wd + 64;
    if (lv.Wd % 4 == 0 && lv.Wd >= 16 && lv.Hd >= 16 && lv.Hd <= 512 && words > 0 && words + tail <= (1u << 23)) {
      d->filter_ok = true;
      // a new layout gets new, zeroed planes: with M and T fixed, size and nyb fix Wd.  Equal sizes of two layouts do
      // not share: the old planes would lie where the new tails must read zeros
      if (2 * (words + tail) != d->d_rp.size() || nyb != d->rp_nyb) {
        CU(d->d_rp.assign(2 * (words + tail)));
        CU(cudaMemsetAsync(d->d_rp.get(), 0, 2 * (words + tail) * 4, d->stream.get()));  // halves no row block covers stay zero
      }
      d->rp_nyb = nyb;
      d->rp_noff = (uint32_t)(words + tail);
      for (int g = 0; g < d->G; ++g) {
        int nfl = 0;
        for (int m = 0; m < d->M; ++m) nfl += d->tmeta[((size_t)g * d->S + lr * d->M + m) * 4 + 3];
        if (!d->safe[g] || nfl < 1 || nfl > 511) continue;
        d->safe[g] |= 2;
        rfeat[(size_t)g] = make_int2((int)rdesc.size(), nfl);
        for (int m = 0; m < d->M; ++m) {
          const int32_t* tm = &d->tmeta[((size_t)g * d->S + lr * d->M + m) * 4];
          for (int k = 0; k < tm[3]; ++k) {
            const int32_t* f = &d->feats[3 * ((size_t)tm[2] + k)];
            const uint32_t pb = (uint32_t)((m * 8 + f[2]) * T2 + (f[1] % T) * T + (f[0] % T));
            rdesc.push_back((pb * (uint32_t)nyb * (uint32_t)lv.Wd + (uint32_t)(f[0] / T)) | ((uint32_t)(f[1] / T) << 23));
          }
        }
        while (rdesc.size() % 32) rdesc.push_back((uint32_t)words);  // padding: the zero tail (+ rp_noff: the N tail), row 0
      }
    }
  }
  d->h_rfeat = rfeat;
  d->d_rdesc.reset();
  d->d_rfeat.reset();
  if (d->filter_ok) {
    CU(upload(d->d_rdesc, rdesc, d->stream.get(), 1));
    CU(upload(d->d_rfeat, rfeat, d->stream.get(), 1));
  }
  CU(upload(d->d_safe, d->safe, d->stream.get()));
  if (nf) {
    CU(cudaMemcpyAsync(d->d_fbase.get(), fbase.data(), nf * 4, cudaMemcpyHostToDevice, d->stream.get()));
    CU(cudaMemcpyAsync(d->d_fxy.get(), fxy.data(), nf * 4, cudaMemcpyHostToDevice, d->stream.get()));
  }
  if (d->G) CU(cudaMemcpyAsync(d->d_tslot.get(), d->h_tslot.data(), sizeof(TSlot) * d->h_tslot.size(), cudaMemcpyHostToDevice, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));  // host vectors go out of scope
  d->feat_skip_low.assign(nf, 0);
  for (size_t i = 0; i < nf; ++i) d->feat_skip_low[i] = (fxy[i] & LM_SKIP_BIT) ? 1 : 0;
  for (int l = 0; l < d->L; ++l) { d->prep_rows[l] = d->lv[l].rows; d->prep_cols[l] = d->lv[l].cols; }
  d->prepared = true;
  d->work_dirty = true;
  d->post_dirty = true;
  return LM_OK;
}

// Task table of k_coarse_packed for one shard: the full rounds (32 consecutive words of one template) of every item in
// order as (work item, round), then the remainder words of every item laid end to end as (work item, word), 32 per task.
// The last remainder task is padded with copies of its last word (the kernel emits nothing for them).  items == null:
// item i is work item i.
static void coarse_task_table(const int32_t* items, const int32_t* words, int64_t n, std::vector<int2>& table,
                              int64_t& n_full, int64_t& n_rem) {
  table.clear();
  for (int64_t i = 0; i < n; ++i)
    for (int r = 0; r < words[i] >> 5; ++r) table.push_back(make_int2(items ? items[i] : (int)i, r));
  n_full = (int64_t)table.size();
  for (int64_t i = 0; i < n; ++i)
    for (int k = words[i] & ~31; k < words[i]; ++k) table.push_back(make_int2(items ? items[i] : (int)i, k));
  n_rem = (int64_t)table.size() - n_full;
  while ((table.size() - (size_t)n_full) % 32) table.push_back(table.back());
}

// Launch shape of k_coarse_packed for `tasks` tasks.  One task per warp (or per TEAM of S warps when the shard has fewer
// tasks than the GPU has warp slots: the team deals the task's features, so the kernel's latency follows the shard) and
// one round per CTA where the tasks fit: the CTA size follows the shard, so a small shard spreads over all SMs, and
// CTA b's share of the table (tasks b, b + grid, ...) never holds more tasks than the CTA has teams.
static CoarseShape coarse_shape(int64_t tasks, int sm_count, size_t plane_bytes) {
  CoarseShape c;
  c.smem = plane_bytes <= LM_BITS_SMEM_LIMIT;
  const long long slots = (long long)sm_count * (LM_PACK_THREADS / 32);
  const size_t part_room = LM_K2_SMEM_MAX - (c.smem ? plane_bytes : (size_t)LM_K2_SMEM_MAX - 64 * 1024);
  int S = 1;
  while (S < 8 && tasks * (S * 2) <= slots) {
    const int S2 = S * 2;
    long long w2 = (tasks * S2 + sm_count - 1) / sm_count;
    w2 = std::min<long long>(LM_PACK_THREADS / 32, std::max<long long>(std::max(4, S2), (w2 + S2 - 1) / S2 * S2));
    if ((size_t)(w2 / S2) * (S2 - 1) * 16 * 32 * 4 > part_room) break;
    S = S2;
  }
  c.split = S;
  const int unit = std::max(4, S);
  int wpc = (int)((tasks * S + sm_count - 1) / sm_count);
  c.wpc = std::min(LM_PACK_THREADS / 32, std::max(unit, (wpc + unit - 1) / unit * unit));
  c.grid = (int)std::max<long long>(1, std::min<long long>(sm_count, (tasks * S + c.wpc - 1) / c.wpc));
  c.smem_bytes = (c.smem ? plane_bytes : 0) + (size_t)(c.wpc / S) * (S - 1) * 16 * 32 * 4;
  return c;
}

extern "C" int lm_coarse_tasks(const int32_t* words, int64_t n_items, int sm_count, int64_t plane_bytes, int32_t* table,
                               int64_t cap, int64_t* n_entries, int64_t* n_full, int64_t* n_rem, int32_t* shape) {
  if (n_items < 0 || (n_items > 0 && !words) || sm_count < 1 || plane_bytes < 0) return fail(LM_E_INVALID, "bad arguments");
  for (int64_t i = 0; i < n_items; ++i)
    if (words[i] < 1) return fail(LM_E_INVALID, "item %lld has %d position words", (long long)i, words[i]);
  std::vector<int2> t;
  int64_t nf = 0, nr = 0;
  coarse_task_table(nullptr, words, n_items, t, nf, nr);
  if (n_entries) *n_entries = (int64_t)t.size();
  if (n_full) *n_full = nf;
  if (n_rem) *n_rem = nr;
  const int64_t tasks = nf + (nr + 31) / 32;
  if (shape) {
    const CoarseShape c = coarse_shape(tasks, sm_count, (size_t)plane_bytes);
    shape[0] = (int32_t)tasks;
    shape[1] = c.split;
    shape[2] = c.wpc;
    shape[3] = c.grid;
  }
  if (table) {
    if (cap < (int64_t)t.size()) return fail(LM_E_CAPACITY, "task table has %lld entries, room for %lld", (long long)t.size(), (long long)cap);
    for (size_t i = 0; i < t.size(); ++i) {
      table[2 * i] = t[i].x;
      table[2 * i + 1] = t[i].y;
    }
  }
  return LM_OK;
}

static int prepare_work(lm_detector* d) {
  if (!d->work_dirty) return LM_OK;
  const int64_t n = d->shard_count;
  CU(upload(d->d_work, d->shard_sel, d->stream.get()));
  if (n > 0) CU(cudaStreamSynchronize(d->stream.get()));
  {
    std::vector<int32_t> ib, iy;
    for (int64_t i = 0; i < n; ++i) (d->bits_ok[d->shard_sel[(size_t)i]] ? ib : iy).push_back((int32_t)i);
    d->n_items_bits = (int)ib.size();
    d->n_items_bytes = (int)iy.size();
    CU(upload(d->d_items_bytes, iy, d->stream.get()));
    // the bit-sliced coarse scan's tasks: position words per item for the current frame size
    d->d_k2task.reset();
    d->k2_full = d->k2_rem = d->k2_tasks = 0;
    std::vector<int2> tasks;
    if (!ib.empty()) {
      const LevelHost& low = d->lv[d->L - 1];
      std::vector<int32_t> words(ib.size());
      for (size_t i = 0; i < ib.size(); ++i) {
        const int g = d->shard_sel[(size_t)ib[i]];
        const int P = d->h_tslot[(size_t)g * d->S + (d->L - 1) * d->M].z;
        words[i] = std::min(std::max((P + 31) >> 5, 1), low.nwords);
      }
      int64_t nf = 0, nr = 0;
      coarse_task_table(ib.data(), words.data(), (int64_t)ib.size(), tasks, nf, nr);
      if (nf + (nr + 31) / 32 > INT32_MAX / 32) return fail(LM_E_CAPACITY, "%lld coarse-scan tasks", (long long)(nf + (nr + 31) / 32));
      d->k2_full = (int)nf;
      d->k2_rem = (int)nr;
      d->k2_tasks = (int)(nf + (nr + 31) / 32);
      CU(upload(d->d_k2task, tasks, d->stream.get()));
    }
    CU(cudaStreamSynchronize(d->stream.get()));
  }
  if ((size_t)n + 1 > d->d_off.size()) {  // d_off is allocated last: its size is the pair's
    d->d_cnt.reset(); d->d_off.reset();
    CU(d->d_cnt.assign((size_t)n + 1));
    CU(d->d_off.assign((size_t)n + 1));
  }
  d->d_finfo.reset();
  d->h_finfo.clear();
  if (d->filter_ok && n > 0) {
    const int lr = d->L - 2;
    d->h_finfo.resize((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
      const int g = d->shard_sel[(size_t)i];
      const int32_t* t0 = &d->tmeta[((size_t)g * d->S + lr * d->M) * 4];
      d->h_finfo[(size_t)i] = make_int4(d->h_rfeat[(size_t)g].x, d->h_rfeat[(size_t)g].y,
                                        (int)((uint32_t)t0[0] | ((uint32_t)t0[1] << 16)), (int)d->safe[(size_t)g]);
    }
    CU(d->d_finfo.assign((size_t)n));
    d->finfo_valid = false;  // the threshold-dependent part is filled in by lm_enqueue
    d->shard_all_eligible = true;
    for (const int4& f : d->h_finfo) d->shard_all_eligible = d->shard_all_eligible && (f.w & 2);
  }
  // per-template candidate counts are accumulated with atomics and re-zeroed by k_scan_counts
  CU(cudaMemsetAsync(d->d_cnt.get(), 0, sizeof(int32_t) * d->d_cnt.size(), d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  // algorithmic bytes of the coarse scan for this shard (SURVEY 8d): sum features x positions
  const int low = (d->L - 1) * d->M;
  int64_t bytes = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int g = d->shard_sel[(size_t)i];
    for (int m = 0; m < d->M; ++m) {
      const TSlot& t = d->h_tslot[(size_t)g * d->S + low + m];
      if (t.z <= 0) continue;
      int live = 0;
      for (int k = 0; k < t.y; ++k) live += d->feat_skip_low[(size_t)t.x + k] ? 0 : 1;
      bytes += (int64_t)live * t.z;
    }
  }
  d->alg_scan_bytes = bytes;
  d->work_dirty = false;
  return LM_OK;
}

// The depth gate's per-work-item table for the shard ({zlo | zhi << 16, ox | oy << 16}, see include/linemod_b200.h) and
// the cell-summary buffer for the frame size.  Only while the gate is on.
static int prepare_gate(lm_detector* d) {
  const LevelHost& low = d->lv[d->L - 1];
  CU(d->d_cells.reserve((size_t)low.plane));
  CU(d->d_gate_before.reserve(1));
  if (!d->gate_dirty) return LM_OK;
  const int64_t n = d->shard_count;
  const int TL = d->T[d->L - 1];
  d->h_gate_item.resize((size_t)n);
  d->gate_with_z = 0;
  for (int64_t w = 0; w < n; ++w) {
    const int g = d->shard_sel[(size_t)w];
    const int32_t* m4 = &d->tmeta[((size_t)g * d->S + (d->L - 1) * d->M) * 4];  // lowest level, modality 0
    const uint32_t ox = (uint32_t)((m4[0] / 2) / TL), oy = (uint32_t)((m4[1] / 2) / TL);
    const double z = (size_t)g < d->tdepth.size() ? (double)d->tdepth[(size_t)g] : NAN;
    uint32_t zlo = 0, zhi = 65535;  // no distance: every depth lies in the band
    if (z > 0.0) {
      const double lo = std::min(std::max(ceil(z * (1.0 - d->gate_tau)), 0.0), 65535.0);
      const double hi = std::min(std::max(floor(z * (1.0 + d->gate_tau)), 0.0), 65535.0);
      zlo = (uint32_t)lo;
      zhi = (uint32_t)hi;
      ++d->gate_with_z;
    }
    d->h_gate_item[(size_t)w] = make_uint2(zlo | (zhi << 16), ox | (oy << 16));
  }
  CU(d->d_gate_item.reserve((size_t)n));
  // on the stream, behind the frames already enqueued (they keep the table they were enqueued with); waited for, since
  // h_gate_item may change once this returns
  if (n > 0)
    CU(cudaMemcpyAsync(d->d_gate_item.get(), d->h_gate_item.data(), sizeof(uint2) * (size_t)n, cudaMemcpyHostToDevice, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  d->gate_dirty = false;
  return LM_OK;
}

// Smallest raw score that survives remove_if(similarity < threshold) (LL.cpp:1935-1937), host twin of lm_min_kept_raw:
// the same two IEEE single-precision operations ((raw * 100.f) / (4 * n)).
static int host_min_kept_raw(float threshold, int nfeat) {
  int lo = 0, hi = 4 * nfeat + 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    volatile float prod = (float)mid * 100.f;
    volatile float score = prod / (float)(4 * nfeat);
    if (!(score < threshold)) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// finfo[w].w = flags | need << 8 for this threshold: need = number of features whose label bit must be set at some cell
// of the patch for the candidate to be able to reach raw_keep (see k_refine_filter_w).
static int filter_thresholds(lm_detector* d, float threshold) {
  if (!d->filter_ok || d->d_finfo.empty() || d->h_finfo.empty()) return LM_OK;
  if (d->finfo_valid && memcmp(&threshold, &d->finfo_threshold, sizeof(float)) == 0) return LM_OK;
  d->h_finfo_up = d->h_finfo;
  int last_nf = -1, last_need = 0;
  for (int4& f : d->h_finfo_up) {
    if (!(f.w & 2)) continue;
    if (f.y != last_nf) {
      last_nf = f.y;
      const int over = host_min_kept_raw(threshold, f.y) - f.y;
      last_need = over > 0 ? (over + 2) / 3 : 0;
    }
    f.w |= last_need << 8;
  }
  CU(cudaMemcpyAsync(d->d_finfo.get(), d->h_finfo_up.data(), sizeof(int4) * d->h_finfo_up.size(), cudaMemcpyHostToDevice, d->stream.get()));
  d->finfo_valid = true;
  d->finfo_threshold = threshold;
  return LM_OK;
}

static int check_frame_dims(lm_detector* d, const int* rows, const int* cols) {
  for (int l = 0; l < d->L; ++l) {
    const int T = d->T[l];
    if (rows[l] <= 0 || cols[l] <= 0) return fail(LM_E_INVALID, "level %d: empty image", l);
    if (rows[l] % T || cols[l] % T)  // CV_Assert LL.cpp:1217-1218
      return fail(LM_E_INVALID, "level %d: %dx%d not a multiple of T=%d", l, cols[l], rows[l], T);
    if (((int64_t)rows[l] * cols[l]) % 16)  // CV_Assert LL.cpp:1136
      return fail(LM_E_INVALID, "level %d: rows*cols not a multiple of 16", l);
    if (rows[l] > 32767 || cols[l] > 32767) return fail(LM_E_INVALID, "level %d: image side > 32767", l);
  }
  const int l = d->L - 1;
  if ((int64_t)(rows[l] / d->T[l]) * (cols[l] / d->T[l]) > 65536)
    return fail(LM_E_INVALID, "lowest level has more than 65536 sampled positions");
  return LM_OK;
}

// (Re)allocate the per-level device buffers for a frame size.  A level of a new size is built aside and takes the
// place of the old one (freed first) once every allocation of it has succeeded.
static int size_levels(lm_detector* d, const int* rows, const int* cols, bool need_upload_buffers) {
  for (int l = 0; l < d->L; ++l) {
    if (d->lv[l].rows != rows[l] || d->lv[l].cols != cols[l] || d->lv[l].T != d->T[l]) {
      // the old level goes first: until the new one stands, there is no frame and nothing prepared for its size
      d->lv[l] = LevelHost();
      d->have_frame = false;
      d->prepared = false;
      LevelHost lv;
      lv.T = d->T[l]; lv.rows = rows[l]; lv.cols = cols[l];
      lv.Wd = cols[l] / lv.T; lv.Hd = rows[l] / lv.T; lv.plane = lv.Wd * lv.Hd;
      const size_t per_mod = (size_t)8 * lv.T * lv.T * lv.plane;
      // slack: the coarse scan reads up to one plane past a feature's base, the 16x16 patch up to 16 rows
      const size_t slack = (size_t)lv.plane + 16 * (size_t)lv.Wd + 256;
      if (per_mod * d->M + slack > 0xFFFFFFFFull) return fail(LM_E_INVALID, "level %d: linear memories exceed 4 GiB", l);
      lv.mod_stride = (uint32_t)per_mod;
      CU(lv.d_lm.assign(per_mod * d->M + slack));
      CU(cudaMemsetAsync(lv.d_lm.get(), 0, lv.d_lm.size(), d->stream.get()));
      lv.nwords = (lv.plane + 31) / 32;
      lv.rounds = (lv.nwords + 31) / 32;
      if (l == d->L - 1 && lv.rounds <= LM_MAX_ROUNDS) {
        lv.lbw = (int)bp_label_words(lv.T, lv.plane);
        const size_t words = (size_t)d->M * 8 * lv.lbw;
        CU(lv.d_bp.assign(words));
        CU(cudaMemsetAsync(lv.d_bp.get(), 0, words * 4, d->stream.get()));
      }
      d->lv[l] = std::move(lv);  // feature addresses depend on the frame size: prepare_bank recomputes them
    }
    if (need_upload_buffers)
      for (int m = 0; m < d->M; ++m) CU(d->lv[l].d_q[m].reserve((size_t)rows[l] * cols[l]));
  }
  return LM_OK;
}

static int upload_quantized(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols, bool sync);

extern "C" int lm_upload_quantized(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols) {
  return upload_quantized(d, quantized, rows, cols, true);
}

static int upload_quantized(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols, bool sync) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d || !quantized || !rows || !cols) return fail(LM_E_INVALID, "null argument");
  CU(cudaSetDevice(d->device));
  int rc = check_frame_dims(d, rows, cols);
  if (rc) return rc;
  rc = size_levels(d, rows, cols, true);
  if (rc) return rc;
  for (int i = 0; i < d->L * d->M; ++i)
    if (!quantized[i]) return fail(LM_E_INVALID, "quantized[%d] is null", i);
  // lowest level first, on the main stream: its linear memories and the coarse scan need nothing else.  The
  // larger upper levels follow on the copy stream (ordered behind everything already enqueued) and are joined
  // in front of the upper levels' linear memories (enqueue_match).
  const bool fork = d->L > 1;
  if (fork) {
    CU(cudaEventRecord(d->ev_fork.get(), d->stream.get()));
    CU(cudaStreamWaitEvent(d->copy_stream.get(), d->ev_fork.get(), 0));
  }
  for (int l = d->L - 1; l >= 0; --l) {
    LevelHost& lv = d->lv[l];
    cudaStream_t st = (fork && l < d->L - 1) ? d->copy_stream.get() : d->stream.get();
    for (int m = 0; m < d->M; ++m) {
      CU(cudaMemcpyAsync(lv.d_q[m].get(), quantized[l * d->M + m], (size_t)rows[l] * cols[l], cudaMemcpyHostToDevice, st));
      lv.q_src[m] = lv.d_q[m].get();
    }
  }
  if (fork) {
    CU(cudaEventRecord(d->ev_upper.get(), d->copy_stream.get()));
    d->upper_pending = true;
  }
  if (sync) {  // caller's buffers are only borrowed for the call
    CU(cudaStreamSynchronize(d->stream.get()));
    if (fork) CU(cudaStreamSynchronize(d->copy_stream.get()));
  }
  d->have_frame = true;
  d->frame_depth = false;
  d->chain.completed = false;
  return LM_OK;
}

extern "C" int lm_bind_quantized_device(lm_detector* d, const uint8_t* const* d_quantized, const int* rows, const int* cols) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d || !d_quantized || !rows || !cols) return fail(LM_E_INVALID, "null argument");
  CU(cudaSetDevice(d->device));
  int rc = check_frame_dims(d, rows, cols);
  if (rc) return rc;
  rc = size_levels(d, rows, cols, false);
  if (rc) return rc;
  for (int l = 0; l < d->L; ++l)
    for (int m = 0; m < d->M; ++m) {
      if (!d_quantized[l * d->M + m]) return fail(LM_E_INVALID, "d_quantized[%d] is null", l * d->M + m);
      d->lv[l].q_src[m] = d_quantized[l * d->M + m];
    }
  if (d->upper_pending) CU(cudaStreamWaitEvent(d->stream.get(), d->ev_upper.get(), 0));  // an earlier upload nobody consumed
  d->upper_pending = false;
  d->have_frame = true;
  d->frame_depth = false;
  d->chain.completed = false;
  return LM_OK;
}

// ---- GPU quantization front-end: Detector::match's modality processing (LL.cpp:1709-1741) -------------
// Pyramid sizes of a rows x cols frame, checked against the frame-size rules of every level.
static int fe_dims(lm_detector* d, int rows, int cols, int* lrows, int* lcols) {
  for (int l = 0; l < d->L; ++l) {
    lrows[l] = l ? lrows[l - 1] / 2 : rows;  // Size(src.cols / 2, src.rows / 2), LL.cpp:564, 866
    lcols[l] = l ? lcols[l - 1] / 2 : cols;
  }
  return check_frame_dims(d, lrows, lcols);
}

// The front-end's buffers for the frame size, and the label buffers of every level; joins an unconsumed upload.
static int fe_levels(lm_detector* d, const int* lrows, const int* lcols) {
  int rc = size_levels(d, lrows, lcols, true);
  if (rc) return rc;
  cudaStream_t st = d->stream.get();
  if (d->upper_pending) CU(cudaStreamWaitEvent(st, d->ev_upper.get(), 0));  // an earlier upload nobody consumed
  if (!d->fe_lut) {
    // NORMAL_LUT[.][vy][vx] of normal_lut.i: 45-degree sector (offset by half a sector) of atan2(vy-10, vx-10);
    // the rule reproduces all 8000 entries of the reference table (tests/test_frontend.py)
    uint8_t lut[400];
    for (int vy = 0; vy < 20; ++vy)
      for (int vx = 0; vx < 20; ++vx) {
        double a = atan2((double)(vy - 10), (double)(vx - 10)) * 180.0 / 3.14159265358979323846;
        a = fmod(a + 360.0, 360.0);
        lut[vy * 20 + vx] = (uint8_t)(1u << (((int)(fmod(a + 22.5, 360.0) / 45.0)) % 8));
      }
    CU(cudaMemcpyToSymbolAsync(c_normal_lut, lut, sizeof(lut), 0, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    d->fe_lut = true;
  }
  for (int l = 0; l < d->L; ++l) {
    if (d->fe[l].rows != lrows[l] || d->fe[l].cols != lcols[l]) {
      // built aside, recorded once every allocation succeeded (level 0 also sizes fe_depth / fe_nraw)
      d->fe[l] = lm_detector::FeLevel();
      d->have_frame = false;
      lm_detector::FeLevel f;
      const size_t n = (size_t)lrows[l] * lcols[l];
      CU(f.src.assign(n * 3)); CU(f.qun.assign(n)); CU(f.strong.assign(n)); CU(f.normal.assign(n));
      CU(f.mask[0].assign(n)); CU(f.mask[1].assign(n));
      if (l == 0) {
        d->fe_depth.reset(); d->fe_nraw.reset();
        CU(d->fe_depth.assign(n)); CU(d->fe_nraw.assign(n));
      }
      f.rows = lrows[l]; f.cols = lcols[l];
      d->fe[l] = std::move(f);
    }
  }
  return LM_OK;
}

// Label images of every level from the level-0 frame in fe[0].src / fe_depth / fe[0].mask[m] (masks[m]: given).
static int fe_quantize(lm_detector* d, const bool* masks) {
  cudaStream_t st = d->stream.get();
  auto grid2 = [](int w, int h) { return dim3((unsigned)((w + 31) / 32), (unsigned)((h + 7) / 8)); };
  for (int l = 0; l < d->L; ++l) {
    lm_detector::FeLevel& f = d->fe[l];
    LevelHost& lv = d->lv[l];
    if (l > 0) {
      lm_detector::FeLevel& up = d->fe[l - 1];
      CU(launch_pdl(k_fe_pyrdown, grid2(f.cols, f.rows), dim3(256), 0, st, (const uint8_t*)up.src.get(), up.rows, up.cols, f.src.get(), f.rows, f.cols));
      for (int m = 0; m < 2; ++m)
        if (masks[m])
          CU(launch_pdl(k_fe_decimate, grid2(f.cols, f.rows), dim3(256), 0, st, (const uint8_t*)up.mask[m].get(), up.cols, f.mask[m].get(), f.rows,
                        f.cols, (const uint8_t*)nullptr, (uint8_t*)nullptr));
      d->launches += 1 + (masks[0] ? 1 : 0) + (masks[1] ? 1 : 0);
    }
    // colour: weak threshold 10 -> gate on squared magnitude > 100 (ColorGradient(10, nf, 55), LL.cpp:1687)
    CU(launch_pdl(k_fe_gradient, grid2(f.cols, f.rows), dim3(FE_TW, FE_TH), 0, st, (const uint8_t*)f.src.get(), f.rows, f.cols, 100, f.qun.get(), f.strong.get()));
    CU(launch_pdl(k_fe_hysteresis, grid2(f.cols, f.rows), dim3(256), 0, st, (const uint8_t*)f.qun.get(), (const uint8_t*)f.strong.get(),
                  (const uint8_t*)(masks[0] ? f.mask[0].get() : nullptr), f.rows, f.cols, lv.d_q[0].get()));
    d->launches += 2;
    // depth: DepthNormal(2000, 50, nf, 2), LL.cpp:1688; upper levels decimate the LABELS (LL.cpp:865-868)
    if (l == 0) {
      CU(launch_pdl(k_fe_normals, grid2(f.cols, f.rows), dim3(256), 0, st, (const uint16_t*)d->fe_depth.get(), f.rows, f.cols, 2000, 50, d->fe_nraw.get()));
      CU(launch_pdl(k_fe_median, grid2(f.cols, f.rows), dim3(256), 0, st, (const uint8_t*)d->fe_nraw.get(),
                    (const uint8_t*)(masks[1] ? f.mask[1].get() : nullptr), f.rows, f.cols, f.normal.get(), lv.d_q[1].get()));
      d->launches += 2;
    } else {
      lm_detector::FeLevel& up = d->fe[l - 1];
      CU(launch_pdl(k_fe_decimate, grid2(f.cols, f.rows), dim3(256), 0, st, (const uint8_t*)up.normal.get(), up.cols, f.normal.get(), f.rows, f.cols,
                    (const uint8_t*)(masks[1] ? f.mask[1].get() : nullptr), lv.d_q[1].get()));
      d->launches += 1;
    }
    lv.q_src[0] = lv.d_q[0].get();
    lv.q_src[1] = lv.d_q[1].get();
  }
  return LM_OK;
}

// The frame state after lm_upload_images / lm_bind_images_device: a frame with depth, not yet matched.
static void fe_bound(lm_detector* d) {
  d->upper_pending = false;
  d->have_frame = true;
  d->frame_depth = true;
  d->chain.completed = false;
}

extern "C" int lm_upload_images(lm_detector* d, const uint8_t* rgb, const uint16_t* depth, int rows, int cols,
                                const uint8_t* mask_color, const uint8_t* mask_depth) {
  if (!d || !rgb || !depth) return fail(LM_E_INVALID, "null argument");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  CU(cudaSetDevice(d->device));
  int lrows[LM_MAX_LEVELS], lcols[LM_MAX_LEVELS];
  int rc = fe_dims(d, rows, cols, lrows, lcols);
  if (rc) return rc;
  rc = fe_levels(d, lrows, lcols);
  if (rc) return rc;
  cudaStream_t st = d->stream.get();
  const size_t n0 = (size_t)rows * cols;
  CU(cudaMemcpyAsync(d->fe[0].src.get(), rgb, n0 * 3, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d->fe_depth.get(), depth, n0 * 2, cudaMemcpyHostToDevice, st));
  const uint8_t* masks[2] = {mask_color, mask_depth};
  for (int m = 0; m < 2; ++m)
    if (masks[m]) CU(cudaMemcpyAsync(d->fe[0].mask[m].get(), masks[m], n0, cudaMemcpyHostToDevice, st));
  const bool given[2] = {masks[0] != nullptr, masks[1] != nullptr};
  rc = fe_quantize(d, given);
  if (rc) return rc;
  CU(cudaStreamSynchronize(st));  // the caller's images are only borrowed for the call
  CU(cudaGetLastError());
  fe_bound(d);
  return LM_OK;
}

// ---- frames already in device memory (lm_bind_images_device, lm_detect_batch_device) ------------------
struct DeviceFrame {
  const uint8_t* rgb; int64_t rgb_pitch;
  const void* depth; int64_t depth_pitch; int format; float scale;
  const uint8_t* mask[2]; int64_t mask_pitch;
};

// One plane of a device frame: present, on `device`, rows at least `row` bytes apart, element-aligned (lm_pose.h).
int check_device_plane(int device, const char* what, const void* p, int64_t pitch, int64_t row, int elem) {
  if (!p) return fail(LM_E_INVALID, "%s is null", what);
  if (pitch < row) return fail(LM_E_INVALID, "%s: row pitch %lld bytes is shorter than a row (%lld bytes)", what, (long long)pitch, (long long)row);
  if ((uintptr_t)p % elem || pitch % elem)
    return fail(LM_E_INVALID, "%s: pointer %p / pitch %lld not aligned to its %d-byte elements", what, p, (long long)pitch, elem);
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();  // clear the query's error: nothing was enqueued
    return fail(LM_E_INVALID, "%s: %p is not a CUDA pointer", what, p);
  }
  if ((a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != device)
    return fail(LM_E_INVALID, "%s: %p is not device or managed memory of device %d (%s, device %d)", what, p, device,
                a.type == cudaMemoryTypeHost ? "host memory" : a.type == cudaMemoryTypeUnregistered ? "unregistered host memory" : "device memory",
                a.device);
  return LM_OK;
}

// Every check of lm_bind_images_device, none of which touches the device.
// A caller's stream: a CUDA stream of `device` (lm_pose.h).
int check_device_stream(int device, cudaStream_t stream) {
  int sdev = -1;
  if (cudaStreamGetDevice(stream, &sdev) != cudaSuccess) {
    cudaGetLastError();  // clear the query's error: nothing was enqueued
    return fail(LM_E_INVALID, "stream %p is not a CUDA stream", (void*)stream);
  }
  if (sdev != device) return fail(LM_E_INVALID, "stream %p belongs to device %d, the handle to device %d", (void*)stream, sdev, device);
  return LM_OK;
}

// The argument checks the detector, the ICP handle and the standalone entry points share (lm_pose.h).
int check_depth_format(const char* what, int format, float scale) {
  if (format != LM_DEPTH_U16_MM && format != LM_DEPTH_F32)
    return fail(LM_E_INVALID, "%s: unknown depth format %d (LM_DEPTH_U16_MM %d, LM_DEPTH_F32 %d)", what, format, LM_DEPTH_U16_MM, LM_DEPTH_F32);
  if (format == LM_DEPTH_F32 && !(std::isfinite(scale) && scale > 0.f))
    return fail(LM_E_INVALID, "%s: scale %g: float depth needs a finite scale > 0", what, (double)scale);
  return LM_OK;
}

int check_estimation(int estimation) {
  if (estimation != LM_ICP_POINT_TO_PLANE && estimation != LM_ICP_POINT_TO_POINT && estimation != LM_POSE_PSO)
    return fail(LM_E_INVALID, "unknown ICP estimation %d (LM_ICP_POINT_TO_PLANE 0, LM_ICP_POINT_TO_POINT 1, LM_POSE_PSO 3)", estimation);
  return LM_OK;
}

int check_inlier_mm(double inlier_mm) {
  if (!(std::isfinite(inlier_mm) && inlier_mm >= 0.0)) return fail(LM_E_INVALID, "inlier distance %g mm: must be finite and >= 0", inlier_mm);
  return LM_OK;
}

int open_device(int device) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(LM_E_CUDA, "no CUDA device available (%s); this library has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(LM_E_INVALID, "device %d out of range (have %d)", device, ndev);
  CU(cudaSetDevice(device));
  return LM_OK;
}

static int check_device_frame(lm_detector* d, const DeviceFrame& f, int rows, int cols, cudaStream_t stream, int* lrows, int* lcols) {
  int rc = check_device_stream(d->device, stream);
  if (!rc) rc = check_depth_format("depth", f.format, f.scale);
  if (rc) return rc;
  rc = fe_dims(d, rows, cols, lrows, lcols);
  if (rc) return rc;
  const int esize = f.format == LM_DEPTH_F32 ? 4 : 2;
  rc = check_device_plane(d->device, "rgb", f.rgb, f.rgb_pitch, 3ll * cols, 1);
  if (!rc) rc = check_device_plane(d->device, "depth", f.depth, f.depth_pitch, (int64_t)esize * cols, esize);
  for (int m = 0; m < 2 && !rc; ++m)
    if (f.mask[m]) rc = check_device_plane(d->device, m ? "mask_depth" : "mask_color", f.mask[m], f.mask_pitch, cols, 1);
  return rc;
}

// The ingest of a checked device frame and the front-end behind it, ordered after the caller's stream and before its
// next work; no host synchronise (beyond lm_upload_images' first-use ones: buffers of a new size, the normal table).
static int bind_images_device(lm_detector* d, const DeviceFrame& f, int rows, int cols, const int* lrows, const int* lcols,
                              cudaStream_t caller) {
  int rc = fe_levels(d, lrows, lcols);
  if (rc) return rc;
  if (!d->ev_in.get()) CU(d->ev_in.create(cudaEventDisableTiming));
  if (!d->ev_out.get()) CU(d->ev_out.create(cudaEventDisableTiming));
  cudaStream_t st = d->stream.get();
  CU(cudaEventRecord(d->ev_in.get(), caller));
  CU(cudaStreamWaitEvent(st, d->ev_in.get(), 0));
  // a plain launch: it starts once the caller's work and everything before it on the stream have completed
  const dim3 grid((unsigned)((cols + FE_INGEST_PX - 1) / FE_INGEST_PX), (unsigned)rows);
  lm_detector::FeLevel& f0 = d->fe[0];
  k_fe_ingest<<<grid, FE_INGEST_PX, 0, st>>>(f.rgb, f.rgb_pitch, f.depth, f.depth_pitch, f.format == LM_DEPTH_F32 ? 1 : 0, f.scale,
                                             f.mask[0], f.mask[1], f.mask_pitch, cols, f0.src.get(), d->fe_depth.get(), f0.mask[0].get(), f0.mask[1].get());
  CU(cudaGetLastError());
  d->launches += 1;
  CU(cudaEventRecord(d->ev_out.get(), st));
  CU(cudaStreamWaitEvent(caller, d->ev_out.get(), 0));  // the borrow ends with the ingest
  const bool given[2] = {f.mask[0] != nullptr, f.mask[1] != nullptr};
  rc = fe_quantize(d, given);
  if (rc) return rc;
  fe_bound(d);
  return LM_OK;
}

extern "C" int lm_bind_images_device(lm_detector* d, const uint8_t* rgb, int64_t rgb_pitch, const void* depth, int64_t depth_pitch,
                                     int depth_format, float depth_scale, int rows, int cols, const uint8_t* mask_color,
                                     const uint8_t* mask_depth, int64_t mask_pitch, void* stream) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  CU(cudaSetDevice(d->device));
  const DeviceFrame f = {rgb, rgb_pitch, depth, depth_pitch, depth_format, depth_scale, {mask_color, mask_depth}, mask_pitch};
  int lrows[LM_MAX_LEVELS], lcols[LM_MAX_LEVELS];
  int rc = check_device_frame(d, f, rows, cols, (cudaStream_t)stream, lrows, lcols);
  if (rc) return rc;
  return bind_images_device(d, f, rows, cols, lrows, lcols, (cudaStream_t)stream);
}

extern "C" int lm_debug_depth(lm_detector* d, uint16_t* out, int64_t cap) {
  if (!d || !out) return fail(LM_E_INVALID, "null argument");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle");
  if (!d->have_frame || !d->frame_depth) return fail(LM_E_STATE, "no frame with depth uploaded or bound");
  const int64_t n = (int64_t)d->fe[0].rows * d->fe[0].cols;
  if (n > cap) return fail(LM_E_CAPACITY, "need %lld elements", (long long)n);
  CU(cudaSetDevice(d->device));
  CU(cudaMemcpyAsync(out, d->fe_depth.get(), (size_t)n * 2, cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  return LM_OK;
}

static LevelDev level_dev(const LevelHost& h) {
  LevelDev v;
  v.lm = h.d_lm.get(); v.T = h.T; v.rows = h.rows; v.cols = h.cols; v.Wd = h.Wd; v.Hd = h.Hd; v.plane = h.plane;
  v.off = h.T / 2 + (h.T % 2 - 1);
  v.mod_stride = h.mod_stride;
  return v;
}


// K1 launch plan.  planes_level >= 0: that level is built in planes mode (column-major H-planes only, no byte linear
// memories; see spread_planes_block).  low_bytes: the lowest level gets its byte linear memories too (only
// k_coarse_bytes and the debug getter read them); with_bit_planes: it gets its spread bit-planes (band kernel: CTAs of
// their own ahead of its byte CTAs, see spread_bits_block).
static void plan_k1(lm_detector* d, int planes_level, bool low_bytes, bool with_bit_planes, K1Plan& k) {
  LinMemParams& p = k.p;
  memset(&p, 0, sizeof(p));
  p.L = d->L; p.M = d->M; p.block_offset = 0;
  bool band = true;
  size_t smem = 0;
  for (int l = 0; l < d->L; ++l) {
    const LevelHost& lv = d->lv[l];
    band = band && (lv.cols % 4 == 0) && (lv.Wd % 4 == 0) && (lv.plane % 4 == 0);
    // the most segments (a divisor of Wd / 4, so that a segment keeps a multiple of 4 positions) that still
    // leave every thread of the CTA one 4-position group of one grid: equal, light CTAs on every level
    int nseg = 1;
    if (lv.Wd % 4 == 0)
      for (int j = 1; j <= 16 && j <= lv.Wd / 4; ++j)
        if ((lv.Wd / 4) % j == 0 && (lv.T * lv.T * (lv.Wd / 4)) / j >= 128) nseg = j;
    p.lv[l].nseg = nseg;
    const size_t wp = (size_t)((lv.Wd / nseg * lv.T + lv.T + 3 + 4) & ~3);
    size_t need = wp * (size_t)(2 * (2 * lv.T - 1) + lv.T);
    if (l == planes_level) {
      // positions per segment: T*T * pseg = one (grid, column) item per thread of the 128-thread CTA where possible
      int pseg = 4;
      for (int c : {32, 16, 8})
        if (lv.Wd % c == 0 && lv.T * lv.T * c <= 128) { pseg = c; break; }
      p.lv[l].pseg = pseg;
      const size_t wpp = (size_t)((pseg * lv.T + lv.T + 3 + 4) & ~3);
      need = wpp * (size_t)(2 * (16 * lv.T + lv.T - 1) + 16 * lv.T);
    }
    smem = std::max(smem, need);
  }
  band = band && smem <= LM_BAND_SMEM_LIMIT;
  int blocks = 0;
  // block index order = lowest level first: its CTAs are the heavy ones (T*T = 64 grids per position row), started last
  // they would be the tail of the launch; and a launch of the lowest level alone stays one block range (upper_pending)
  for (int l = d->L - 1; l >= 0; --l) {
    const LevelHost& lv = d->lv[l];
    LinMemLevel& q = p.lv[l];
    const bool low = l == d->L - 1;
    for (int m = 0; m < d->M; ++m) q.q[m] = lv.q_src[m];
    q.lm = low && !low_bytes ? nullptr : lv.d_lm.get();
    q.bp = low && with_bit_planes ? lv.d_bp.get() : nullptr;  // allocated for the lowest level only
    q.lbw = lv.lbw;
    q.T = lv.T; q.rows = lv.rows; q.cols = lv.cols; q.Wd = lv.Wd; q.Hd = lv.Hd; q.plane = lv.plane;
    q.mod_stride = lv.mod_stride;
    q.rp = nullptr; q.nyb = 0; q.bit_blocks = 0;
    const int n = lv.T * lv.T * lv.plane;
    if (!band) {
      blocks += q.lm || q.bp ? (n + 255) / 256 : 0;  // one thread per index builds both
    } else {
      if (q.bp) q.bit_blocks = ((n + 31) / 32 + LM_BP_CTA_WORDS - 1) / LM_BP_CTA_WORDS;
      blocks += q.bit_blocks;
      if (l == planes_level) {
        q.rp = d->d_rp.get(); q.nyb = d->rp_nyb;
        blocks += ((lv.Hd + 15) / 16) * (lv.Wd / q.pseg);
      } else if (q.lm) {
        blocks += lv.Hd * q.nseg;
      }
    }
    q.block_end = blocks;
  }
  k.band = band;
  k.smem = smem;
  k.blocks = blocks;
}

static int launch_k1(lm_detector* d, const K1Plan& k, int first_block, int n_blocks) {
  if (n_blocks <= 0) return LM_OK;
  LinMemParams p = k.p;
  p.block_offset = first_block;
  if (k.band) CU(launch_pdl(k_linear_memories_band, dim3((unsigned)n_blocks, (unsigned)d->M), dim3(128), k.smem, d->stream.get(), p));
  else CU(launch_pdl(k_linear_memories, dim3((unsigned)n_blocks, (unsigned)d->M), dim3(256), 0, d->stream.get(), p));
  ++d->launches;
  return LM_OK;
}

// The frame's routes (FramePlan), from the bank, shard, frame size, gate and exchange the prepare steps left.
static void plan_frame(lm_detector* d) {
  FramePlan& pl = d->chain.plan;
  pl.gated = d->gate_on;
  pl.exchange = d->px_rank >= 0;
  pl.filter = d->filter_ok && !d->d_rp.empty() && !d->d_finfo.empty();
  // two pyramid levels: the filtered level is the last one, its survivors are finished bit-sliced (k_refine_bits)
  pl.bits = pl.filter && d->L == 2;
  // byte-wise exact refinement: the templates the filter does not take, or every candidate without the bit-sliced pass
  pl.refine = !pl.bits || !d->shard_all_eligible;
  pl.bits_publish = pl.bits && !pl.refine;
  // K1 builds the filtered level as H-planes only when nothing reads its byte linear memories, and the lowest level's
  // bytes only for the byte-wise coarse scan (the refinement starts a level up)
  const int planes = pl.bits && !pl.refine ? d->L - 2 : -1;
  plan_k1(d, planes, d->n_items_bytes > 0, true, pl.k1);
  pl.planes_level = pl.k1.band ? planes : -1;  // only the band kernel has a planes mode
  pl.stale = 0;
  for (int l = 0; l < d->L; ++l)
    if (!pl.k1.p.lv[l].lm || pl.k1.p.lv[l].rp) pl.stale |= 1 << l;
  pl.packed = d->n_items_bits > 0;
  pl.bytes = d->n_items_bytes > 0;
  pl.scan_fused = pl.packed && !pl.bytes;
  pl.plane_bytes = ((size_t)d->M * 8 * d->lv[d->L - 1].lbw * 4 + 15) & ~(size_t)15;
  pl.coarse = pl.packed ? coarse_shape(d->k2_tasks, d->sm_count, pl.plane_bytes) : CoarseShape{};
}

// This rank's block of the current frame slot of the peer exchange.
static lm_result_header* exchange_block(const lm_detector* d) {
  return reinterpret_cast<lm_result_header*>(d->px_buf.get() + (size_t)(d->px_seq & 1) * d->h_px.slot_bytes +
                                             (size_t)d->h_px.rank * d->h_px.block_bytes);
}

// The block the frame's stages append records to, and its capacity.  Resolved at launch, never recorded: a replay may
// grow and move the result block.
struct AppendTarget { lm_result_header* hdr; int32_t capacity; };
static AppendTarget append_target(const lm_detector* d) {
  if (d->chain.plan.exchange) return {exchange_block(d), (int32_t)d->px_cap};
  return {d->d_res, (int32_t)d->res_cap};
}

// The frame's match up to its candidate offsets, as planned: K1, the depth gate's cell summary, the coarse scan and the
// scan of its counts, then K1's upper levels.  ev: the run's timing events (null: not timed).  No host synchronisation.
static int enqueue_match(lm_detector* d, const Event* ev) {
  const FramePlan& pl = d->chain.plan;
  const float threshold = d->chain.threshold;
  const int n_work = (int)d->shard_count;
  const LevelHost& low = d->lv[d->L - 1];
  cudaStream_t st = d->stream.get();
  if (pl.exchange) ++d->px_seq;  // the frame's number, and its slot of the exchange buffer
  if (ev) CU(cudaEventRecord(ev[0].get(), st));
  // K1: one launch for every level and modality.  Every live bit-plane word is stored whole each frame (the slack behind
  // them stays zero from allocation).  With a host upload in flight (upper levels still on the copy stream) the launch
  // is split: the lowest level now, the levels above it behind the coarse scan, once their images have landed.
  const K1Plan& k1 = pl.k1;
  const int k1_done = d->upper_pending ? k1.p.lv[d->L - 1].block_end : k1.blocks;
  int rc = launch_k1(d, k1, 0, k1_done);
  if (rc) return rc;
  if (ev) CU(cudaEventRecord(ev[1].get(), st));
  // depth gate: the frame's cell summary, ahead of K2
  DepthGate gate;  // read by the gated launches only
  if (pl.gated) {
    gate.cells = d->d_cells.get(); gate.item = d->d_gate_item.get(); gate.before = d->d_gate_before.get();
    gate.Wd = low.Wd; gate.Hd = low.Hd;
    const int B = low.T << (d->L - 1);  // s * T_L full-resolution pixels per cell side
    CU(launch_pdl(k_depth_cells, dim3((unsigned)((low.plane + 7) / 8)), dim3(256), 0, st, (const uint16_t*)d->fe_depth.get(),
                  d->fe[0].rows, d->fe[0].cols, B, low.Wd, low.Hd, d->d_cells.get(), d->d_gate_before.get()));
    ++d->launches;
  }
  const AppendTarget out = append_target(d);
  // K2
  if (pl.packed) {
    BitScanGateParams bp;
    bp.bp = low.d_bp.get(); bp.bp_words = (uint32_t)((size_t)d->M * 8 * low.lbw);
    bp.lbw = low.lbw; bp.plane = low.plane; bp.nwords = low.nwords;
    bp.tslot = d->d_tslot.get(); bp.fdesc = d->d_fdesc.get(); bp.k2info = d->d_k2info.get(); bp.work = d->d_work.get();
    bp.zero_desc = coarse_zero_descriptor(low.T, low.plane);
    bp.tasks = d->d_k2task.get(); bp.n_full = d->k2_full; bp.n_rem = d->k2_rem; bp.n_tasks = d->k2_tasks;
    bp.S = d->S; bp.M = d->M; bp.slot_low = (d->L - 1) * d->M;
    bp.threshold = threshold;
    bp.mask = d->d_mask.get(); bp.raw = d->d_raw.get(); bp.cnt = d->d_cnt.get();
    bp.off = pl.scan_fused ? d->d_off.get() : nullptr;
    bp.n_work = n_work;
    bp.hdr = out.hdr; bp.capacity = out.capacity;
    bp.shard = d->shard_index;
    bp.counters = d->d_counters.get();
    bp.queue = d->d_queue.get();
    bp.ticket = reinterpret_cast<int*>(d->d_counters.get() + 3);
    const CoarseShape& c = pl.coarse;
    bp.split = c.split;
    cudaError_t e = cudaSuccess;
    if (pl.gated) {
      bp.gate = gate;
      e = c.smem ? launch_pdl(k_coarse_packed<true, true>, dim3(c.grid), dim3(c.wpc * 32), c.smem_bytes, st, bp)
                 : launch_pdl(k_coarse_packed<false, true>, dim3(c.grid), dim3(c.wpc * 32), c.smem_bytes, st, bp);
    } else if (c.smem) {
      e = launch_pdl(k_coarse_packed<true, false>, dim3(c.grid), dim3(c.wpc * 32), c.smem_bytes, st, static_cast<const BitScanParams&>(bp));
    } else {
      e = launch_pdl(k_coarse_packed<false, false>, dim3(c.grid), dim3(c.wpc * 32), c.smem_bytes, st, static_cast<const BitScanParams&>(bp));
    }
    if (e != cudaSuccess) return fail(LM_E_CUDA, "k_coarse_packed launch failed: %s", cudaGetErrorString(e));
    ++d->launches;
  }
  if (pl.bytes) {
    ByteScanGateParams sp;
    sp.lv = level_dev(low);
    sp.tslot = d->d_tslot.get(); sp.fbase = d->d_fbase.get(); sp.fxy = d->d_fxy.get(); sp.work = d->d_work.get();
    sp.items = d->d_items_bytes.get();
    sp.S = d->S; sp.M = d->M; sp.slot_low = (d->L - 1) * d->M; sp.nwords = low.nwords;
    sp.threshold = threshold;
    sp.mask = d->d_mask.get(); sp.raw = d->d_raw.get(); sp.cnt = d->d_cnt.get();
    int bs = ((low.plane + 3) / 4 + 31) / 32 * 32;
    bs = std::max(32, std::min(bs, 1024));
    if (pl.gated) {
      sp.gate = gate;
      CU(launch_pdl(k_coarse_bytes<true>, dim3(d->n_items_bytes), dim3(bs), 0, st, sp));
    } else CU(launch_pdl(k_coarse_bytes<false>, dim3(d->n_items_bytes), dim3(bs), 0, st, static_cast<const ByteScanParams&>(sp)));
    ++d->launches;
  }
  if (ev) CU(cudaEventRecord(ev[2].get(), st));
  if (!pl.scan_fused) {
    CU(launch_pdl(k_scan_counts, dim3(1), dim3(1024), 0, st, d->d_cnt.get(), d->d_off.get(), n_work, out.hdr, (int)out.capacity,
                  d->shard_index, d->d_counters.get(), d->d_queue.get()));
    ++d->launches;
  }
  if (ev) CU(cudaEventRecord(ev[3].get(), st));
  if (k1_done < k1.blocks) {  // the upper levels' linear memories, behind their images
    CU(cudaStreamWaitEvent(st, d->ev_upper.get(), 0));
    rc = launch_k1(d, k1, k1_done, k1.blocks - k1_done);
    if (rc) return rc;
  }
  d->upper_pending = false;
  return LM_OK;
}

// The frame's refinement, as planned: candidate list, filter, exact passes, the exchange's collector.  An overflow replay
// runs it again (the coarse outputs are still in place) with ev null, so lm_stage_times covers a frame's first pass.
static int enqueue_refine(lm_detector* d, const Event* ev) {
  const FramePlan& pl = d->chain.plan;
  const float threshold = d->chain.threshold;
  const int n_work = (int)d->shard_count;
  const LevelHost& low = d->lv[d->L - 1];
  const int lr = d->L >= 2 ? d->L - 2 : 0;
  const LevelHost& lref = d->lv[lr];
  cudaStream_t st = d->stream.get();
  const AppendTarget out = append_target(d);
  {
    // ordered candidate list (+ the filter's H-planes of the first refined level)
    PrepParams pp;
    pp.off = d->d_off.get(); pp.mask = d->d_mask.get();
    pp.n_work = n_work; pp.nwords = low.nwords;
    pp.cand = d->d_cand.get(); pp.cand_cap = (int)cand_cap(d);
    pp.expand_blocks = std::max(1, std::min((n_work + 7) / 8, d->sm_count * 8));
    // H- and N-planes from the byte linear memories, or, after K1 in planes mode, N from K1's H-planes (eight labels a thread)
    pp.rp = pl.filter ? d->d_rp.get() : nullptr;
    pp.lm = (pl.stale >> lr) & 1 ? nullptr : lref.d_lm.get();
    pp.Wd = lref.Wd; pp.Hd = lref.Hd; pp.plane = lref.plane; pp.nyb = d->rp_nyb; pp.n_off = d->rp_noff;
    pp.t2 = lref.T * lref.T;
    pp.n_pb = d->M * 8 * pp.t2;
    const size_t plane_threads = (size_t)(pp.lm ? pp.n_pb : pp.n_pb / 8) * pp.nyb * (pp.Wd / 4);
    const int plane_blocks = pp.rp ? (int)((plane_threads + 255) / 256) : 0;
    CU(launch_pdl(k_refine_prep, dim3((unsigned)(pp.expand_blocks + plane_blocks)), dim3(256), 0, st, pp));
    ++d->launches;
  }
  if (ev) CU(cudaEventRecord(ev[4].get(), st));
  if (pl.filter) {
    FilterParams fp;
    fp.rp = d->d_rp.get(); fp.Wd = lref.Wd; fp.nyb = d->rp_nyb;
    fp.rdesc = d->d_rdesc.get(); fp.rfeat = d->d_rfeat.get(); fp.finfo = d->d_finfo.get(); fp.flags = d->d_safe.get();
    fp.tslot = d->d_tslot.get(); fp.work = d->d_work.get(); fp.S = d->S; fp.M = d->M; fp.L = d->L;
    fp.low = level_dev(low); fp.ref = level_dev(lref);
    fp.cand = d->d_cand.get(); fp.off = d->d_off.get(); fp.n_work = n_work; fp.cand_cap = (int)cand_cap(d);
    fp.threshold = threshold;
    fp.surv = d->d_surv.get(); fp.surv2 = pl.bits ? d->d_surv2.get() : nullptr; fp.queue = d->d_queue.get(); fp.counters = d->d_counters.get();
    CU(launch_pdl(k_refine_filter_w, dim3((unsigned)(d->sm_count * LM_FILTER_MIN_CTAS)), dim3(256), 0, st, fp));
    ++d->launches;
  }
  if (ev) CU(cudaEventRecord(ev[5].get(), st));
  if (pl.bits) {
    // exact refinement of the survivors, bit-sliced, from the same H-planes
    RefineBitsParams bq;
    bq.rp = d->d_rp.get(); bq.Wd = lref.Wd; bq.n_off = d->rp_noff;
    bq.rdesc = d->d_rdesc.get(); bq.finfo = d->d_finfo.get();
    bq.low = level_dev(low); bq.ref = level_dev(lref);
    bq.cand = d->d_cand.get(); bq.off = d->d_off.get(); bq.n_work = n_work; bq.cand_cap = (int)cand_cap(d);
    bq.surv = d->d_surv.get(); bq.queue = d->d_queue.get();
    bq.threshold = threshold;
    bq.work_begin = (int)d->work_base; bq.work_stride = (int)d->work_stride;
    bq.hdr = out.hdr; bq.capacity = out.capacity;
    bq.px = pl.exchange ? d->d_px.get() : nullptr; bq.px_seq = d->px_seq;
    bq.publish = pl.bits_publish ? 1 : 0;
    bq.counters = d->d_counters.get();
    if (d->bits_grid == 0) {  // one wave: the survivors are dealt over the CTAs that are resident at once
      int per_sm = 0;
      CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_refine_bits, 256, 0));
      d->bits_grid = std::max(1, per_sm) * d->sm_count;
    }
    CU(launch_pdl(k_refine_bits, dim3((unsigned)d->bits_grid), dim3(256), 0, st, bq));
    ++d->launches;
  }
  if (pl.refine) {
    // persistent grid: the candidate total is read on the device (no host round trip)
    RefineParams rp;
    for (int l = 0; l < d->L; ++l) rp.lv[l] = level_dev(d->lv[l]);
    rp.tslot = d->d_tslot.get(); rp.fbase = d->d_fbase.get(); rp.fxy = d->d_fxy.get(); rp.work = d->d_work.get();
    rp.off = d->d_off.get(); rp.cand = d->d_cand.get(); rp.cand_cap = (int)cand_cap(d); rp.raw = d->d_raw.get();
    rp.surv = pl.filter ? (pl.bits ? d->d_surv2.get() : d->d_surv.get()) : nullptr; rp.queue = d->d_queue.get();
    rp.surv_slot = pl.bits ? 2 : 1;
    rp.publish = 1;
    rp.n_work = n_work; rp.L = d->L; rp.S = d->S; rp.M = d->M;
    rp.work_begin = (int)d->work_base;
    rp.work_stride = (int)d->work_stride;
    rp.threshold = threshold;
    rp.hdr = out.hdr; rp.capacity = out.capacity;
    rp.px = pl.exchange ? d->d_px.get() : nullptr;
    rp.px_seq = d->px_seq;
    rp.counters = d->d_counters.get();
    rp.safe = d->d_safe.get(); rp.galign = d->d_galign.get();
    // 4 CTAs are resident per SM (64 registers x 256 threads); 16 per SM = four waves of equal shares, which
    // balances the very uneven per-candidate cost (row-wise early exit) better than one persistent wave
    // (measured: 4 -> 251 us, 8 -> 241, 12..32 -> 229)
    // behind the filter the work items are its few survivors: four warps share one (k_refine<true>)
    if (pl.filter) CU(launch_pdl(k_refine<true>, dim3(d->sm_count * 16), dim3(256), 0, st, rp));
    else CU(launch_pdl(k_refine<false>, dim3(d->sm_count * 16), dim3(256), 0, st, rp));
    ++d->launches;
  }
  if (pl.exchange) {
    // collector: waits for all ranks' frame flags, packs the blocks into the ordinary result block
    CU(launch_pdl(k_peer_collect, dim3(1), dim3(1024), 0, st, d->h_px, d->px_seq, (int32_t)d->px_cap, d->d_res, (int32_t)d->res_cap,
                  d->d_counters.get() + 2, d->px_timeout_ns));
    ++d->launches;
  }
  if (ev) CU(cudaEventRecord(ev[6].get(), st));
  return LM_OK;
}

// header + the first records in one copy; the common case needs no second round trip
#define LM_FIRST_FETCH 4096

static int enqueue_readback(lm_detector* d) {
  cudaStream_t st = d->stream.get();
  const int64_t first = std::min<int64_t>(d->res_cap, LM_FIRST_FETCH);
  CU(cudaMemcpyAsync(d->h_res.get(), d->d_res, sizeof(lm_result_header) + sizeof(lm_record) * (size_t)first,
                     cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(d->h_counters.get(), d->d_counters.get(), 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  d->h_valid = first;
  return LM_OK;
}

static int ensure_run_buffers(lm_detector* d) {
  const int64_t n_work = d->shard_count;
  const LevelHost& low = d->lv[d->L - 1];
  CU(d->d_mask.reserve((size_t)std::max<int64_t>(n_work, 1) * low.nwords));
  CU(d->d_raw.reserve((size_t)std::max<int64_t>(n_work, 1) * low.plane));
  // ordered candidate list + survivor list: worst case one entry per (template, cell); capped (a frame that overflows
  // the cap is redone from k_refine_prep with a larger list, like the result block)
  {
    const int64_t worst = std::max<int64_t>(n_work, 1) * low.plane;
    const int64_t want = std::min<int64_t>(worst, std::max<int64_t>(LM_CAND_DEFAULT, d->cand_need));
    if (want > cand_cap(d)) {
      d->d_cand.reset(); d->d_surv.reset(); d->d_surv2.reset();
      CU(d->d_cand.assign((size_t)want));
      CU(d->d_surv.assign((size_t)want));
      CU(d->d_surv2.assign((size_t)want));
    }
  }
  if (d->px_rank >= 0 && d->res_external) return fail(LM_E_STATE, "lm_set_result_buffer and a connected peer exchange exclude each other");
  if (d->px_rank >= 0) CU(d->d_res_own.reserve(res_bytes(d->px_cap * d->px_world)));
  if (!d->res_external) {
    if (d->d_res_own.empty()) CU(d->d_res_own.assign(res_bytes(1 << 16)));
    d->d_res = reinterpret_cast<lm_result_header*>(d->d_res_own.get());
    d->res_cap = res_records(d->d_res_own.size());
  }
  CU(d->h_res.reserve(res_bytes(d->res_cap)));
  return LM_OK;
}

static int enqueue_post(lm_detector* d, double iou_threshold, int top_k);
static int enqueue_pose(lm_detector* d);
static int enqueue_pose_nms(lm_detector* d);

// A frame kept more records than the result block holds, or passed more coarse candidates than the candidate list
// holds: grow what it outgrew and replay its chain from the refinement on (the coarse outputs are still in place), then
// every later stage the chain record holds.  A truncated candidate list makes the kept count a lower bound, so the
// block gets room for twice as many; if that is still too few, the next pass of complete_frame grows it again.
static int grow_and_replay(lm_detector* d, int64_t kept, int64_t cands) {
  const bool more_records = kept > d->res_cap;
  const bool more_cands = cands > cand_cap(d);
  if (more_records && d->res_external)
    return fail(LM_E_CAPACITY, "%lld records kept, caller's result buffer holds %lld", (long long)kept, (long long)d->res_cap);
  if (d->px_rank >= 0)
    return fail(LM_E_CAPACITY, "%lld records kept of %lld candidates: beyond the result block (%lld) or the candidate list (%lld) of a "
                "connected peer exchange", (long long)kept, (long long)cands, (long long)d->res_cap, (long long)cand_cap(d));
  if (more_cands) d->cand_need = cands;  // ensure_run_buffers reallocates the lists
  if (more_records || (more_cands && !d->res_external)) CU(d->d_res_own.reserve(res_bytes(kept * 2)));
  int rc = ensure_run_buffers(d);
  if (rc) return rc;
  // the header the coarse scan wrote, with the new capacity
  const lm_result_header hdr = {0, (int32_t)cands, (int32_t)d->res_cap, d->shard_index};
  CU(cudaMemcpy(d->d_res, &hdr, sizeof(hdr), cudaMemcpyHostToDevice));
  cudaStream_t st = d->stream.get();
  CU(cudaMemsetAsync(d->d_counters.get(), 0, 8 * sizeof(unsigned long long), st));  // [3] (the coarse scan's ticket) is 0 between launches
  CU(cudaMemsetAsync(d->d_queue.get(), 0, 4 * sizeof(int), st));
  CU(cudaMemsetAsync(&d->d_res->count, 0, sizeof(int32_t), st));
  const FrameChain& c = d->chain;
  rc = enqueue_refine(d, nullptr);
  if (!rc && c.post) rc = enqueue_post(d, c.iou, c.top_k);
  if (!rc && c.pose) rc = enqueue_pose(d);
  if (!rc && c.pose_nms) rc = enqueue_pose_nms(d);
  return rc;
}

#define LM_POST_FIRST 16      // survivors fetched with the box NMS's counts; the common top-k needs no second copy
#define LM_COMPLETE_PASSES 3  // grow-and-replay passes of one completion: two always suffice, the first may undercount

// Every completion ends here (lm_complete; with `post`, lm_complete_post / _pose / _detect and each batch frame): the
// readbacks of the awaited stage (the header, first records and counters; or the box NMS's counts, with `survivors` its
// first survivors, and the counters), one synchronise, the exchange's status, then the overflow test and at most
// LM_COMPLETE_PASSES grow-and-replay passes.  A replay also brings the grown frame's header back.
static int complete_frame(lm_detector* d, bool post, bool survivors) {
  cudaStream_t st = d->stream.get();
  for (int pass = 0;; ++pass) {
    if (!post || pass > 0) {
      int rc = enqueue_readback(d);
      if (rc) return rc;
    }
    if (post) {
      CU(cudaMemcpyAsync(d->h_post_counts.get(), d->d_post_counts.get(), sizeof(int32_t) * 4, cudaMemcpyDeviceToHost, st));
      if (survivors) CU(cudaMemcpyAsync(d->h_post_out.get(), d->d_post_out.get(), sizeof(lm_match) * LM_POST_FIRST, cudaMemcpyDeviceToHost, st));
      CU(cudaMemcpyAsync(d->h_counters.get(), d->d_counters.get(), 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    if (pass == 0 && d->px_rank >= 0) {
      if (d->h_counters[2] == 1)
        return fail(LM_E_STATE, "peer exchange: a rank did not publish frame %d within %llu ms (or an earlier frame already timed out "
                    "on this device); disconnect and reconnect the exchange", d->px_seq, d->px_timeout_ns / 1000000ull);
      if (d->h_counters[2] == 2)
        return fail(LM_E_CAPACITY, "peer exchange: a shard kept more than %lld records (capacity given to lm_peer_export)",
                    (long long)d->px_cap);
    }
    const int64_t kept = post ? d->h_post_counts[1] : hres(d)->count;
    int64_t cands = post ? d->h_post_counts[3] : hres(d)->coarse_candidates;
    if (!post && d->px_rank >= 0 && cands > cand_cap(d)) {
      // behind the exchange the header counts every rank's candidates; this rank's list holds only its own (off[n_work])
      int own = 0;
      CU(cudaMemcpyAsync(&own, d->d_off.get() + d->shard_count, sizeof(int), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      cands = own;
    }
    if (kept <= d->res_cap && cands <= cand_cap(d)) return LM_OK;
    if (pass == LM_COMPLETE_PASSES)
      return fail(LM_E_CAPACITY, "%lld records kept of %lld candidates after %d passes: the result block holds %lld, the candidate "
                  "list %lld", (long long)kept, (long long)cands, pass, (long long)d->res_cap, (long long)cand_cap(d));
    int rc = grow_and_replay(d, kept, cands);
    if (rc) return rc;
  }
}

// The lazy host steps of a run, in this order: feature addresses for the frame size, the shard's work lists, the run
// buffers, then the depth gate's tables (refused when the gate has nothing to gate by).  lm_prepare takes them ahead of
// the first frame, lm_enqueue before each one.
static int prepare_run(lm_detector* d) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (!d->have_frame) return fail(LM_E_STATE, "no frame uploaded (the frame size decides the feature addresses)");
  if (d->S == 0) return fail(LM_E_STATE, "no template bank loaded");
  CU(cudaSetDevice(d->device));
  int rc = prepare_bank(d);
  if (!rc) rc = prepare_work(d);
  if (!rc) rc = ensure_run_buffers(d);
  if (rc || !d->gate_on) return rc;
  if (std::none_of(d->tdepth.begin(), d->tdepth.end(), [](float z) { return z > 0.f; }))
    return fail(LM_E_STATE, "depth gate on, but no template of the bank has a training distance (lm_set_template_depths)");
  if (!d->frame_depth)
    return fail(LM_E_STATE, "depth gate on, but the frame has no depth image (lm_upload_quantized / lm_bind_quantized_device)");
  return prepare_gate(d);
}

extern "C" int lm_enqueue(lm_detector* d, float threshold) {
  int rc = prepare_run(d);
  if (rc) return rc;
  d->chain.threshold = threshold;
  rc = filter_thresholds(d, threshold);
  if (rc) return rc;
  plan_frame(d);
  // the run's timing events: the next slot of the ring (null: not timed)
  const Event* ev = d->timing ? d->tev.data() + LM_TEV * (size_t)(d->timing_runs++ % (int64_t)(d->tev.size() / LM_TEV)) : nullptr;
  rc = enqueue_match(d, ev);
  return rc ? rc : enqueue_refine(d, ev);
}

extern "C" int lm_prepare(lm_detector* d) { return prepare_run(d); }

extern "C" int lm_complete(lm_detector* d) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  CU(cudaSetDevice(d->device));
  int rc = complete_frame(d, false, false);
  if (rc) return rc;
  d->chain.completed = true;
  return LM_OK;
}

extern "C" int lm_run(lm_detector* d, float threshold) {
  int rc = lm_enqueue(d, threshold);
  if (rc) return rc;
  return lm_complete(d);
}

extern "C" int lm_set_result_buffer(lm_detector* d, void* d_block, int64_t capacity_records) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (d_block && capacity_records < 1) return fail(LM_E_INVALID, "capacity must be >= 1");
  if (capacity_records > 0x7FFFFFFF) return fail(LM_E_INVALID, "capacity too large");
  if (d_block && d->px_rank >= 0) return fail(LM_E_STATE, "lm_set_result_buffer and a connected peer exchange exclude each other");
  CU(cudaSetDevice(d->device));
  CU(cudaStreamSynchronize(d->stream.get()));
  d->res_external = d_block != nullptr;
  if (d->res_external) {
    d->d_res = (lm_result_header*)d_block;
    d->res_cap = capacity_records;
  }
  d->chain.completed = false;
  return LM_OK;
}

// The exchange buffer: the record blocks and their flags (PeerExchange), then the pose area of lm_peer_share_pose
// (lm_pose.h, PoseShare) at a 16-byte aligned offset.
static size_t peer_pose_offset(int world, int64_t cap) {
  const size_t records = 2 * (size_t)world * (sizeof(lm_result_header) + sizeof(lm_record) * (size_t)cap) +
                         sizeof(int32_t) * (2 * LM_MAX_PEERS + 4);
  return (records + 15) & ~(size_t)15;
}

static size_t peer_buffer_bytes(int world, int64_t cap) { return peer_pose_offset(world, cap) + pose_share_area_bytes(); }

extern "C" int lm_peer_export(lm_detector* d, int world, int64_t capacity_records, uint8_t* handle_out) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (world < 1 || world > LM_MAX_PEERS) return fail(LM_E_INVALID, "world %d outside 1..%d", world, LM_MAX_PEERS);
  if (capacity_records < 1 || capacity_records > (1 << 24)) return fail(LM_E_INVALID, "capacity outside 1..2^24");
  if (peer_buffer_bytes(world, capacity_records) > 0xF0000000ull) return fail(LM_E_INVALID, "exchange buffer too large");
  CU(cudaSetDevice(d->device));
  CU(cudaStreamSynchronize(d->stream.get()));
  peer_release(d);
  const size_t bytes = peer_buffer_bytes(world, capacity_records);
  CU(d->px_buf.assign(bytes));
  CU(cudaMemset(d->px_buf.get(), 0, bytes));
  CU(cudaDeviceSynchronize());
  d->px_world = world;
  d->px_cap = capacity_records;
  d->px_seq = 0;
  d->px_pose_seq = 0;
  {
    const int zero = 0;  // a fresh exchange starts with the device's abort flag down
    CU(cudaMemcpyToSymbol(g_px_abort, &zero, sizeof(int)));
    const char* ms = getenv("LINEMOD_B200_PEER_TIMEOUT_MS");
    const long long v = ms ? atoll(ms) : 1000;
    d->px_timeout_ns = (unsigned long long)(v < 1 ? 1 : (v > 600000 ? 600000 : v)) * 1000000ull;
  }
  if (handle_out) {
    static_assert(sizeof(cudaIpcMemHandle_t) <= LM_PEER_HANDLE_BYTES, "IPC handle size");
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, d->px_buf.get()));
    memset(handle_out, 0, LM_PEER_HANDLE_BYTES);
    memcpy(handle_out, &h, sizeof(h));
  }
  return LM_OK;
}

extern "C" int lm_peer_base(lm_detector* d, void** base) {
  if (!d || !base) return fail(LM_E_INVALID, "null argument");
  if (d->px_buf.empty()) return fail(LM_E_STATE, "lm_peer_export has not been called");
  *base = d->px_buf.get();
  return LM_OK;
}

static int peer_connect_common(lm_detector* d, int rank, int world) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (d->px_buf.empty()) return fail(LM_E_STATE, "lm_peer_export has not been called");
  if (world != d->px_world) return fail(LM_E_INVALID, "world %d differs from the exported one (%d)", world, d->px_world);
  if (rank < 0 || rank >= world) return fail(LM_E_INVALID, "rank %d outside 0..%d", rank, world - 1);
  if (d->px_rank >= 0) return fail(LM_E_STATE, "already connected");
  if (d->res_external) return fail(LM_E_STATE, "lm_set_result_buffer and the peer exchange exclude each other");
  return LM_OK;
}

static int peer_upload_descriptor(lm_detector* d) {
  PeerExchange px;
  memset(&px, 0, sizeof(px));
  for (int r = 0; r < d->px_world; ++r) px.base[r] = d->px_base[r];
  px.world = d->px_world; px.rank = d->px_rank;
  px.block_bytes = (uint32_t)(sizeof(lm_result_header) + sizeof(lm_record) * (size_t)d->px_cap);
  px.slot_bytes = px.block_bytes * (uint32_t)d->px_world;
  px.flags_offset = 2u * px.slot_bytes;
  d->h_px = px;
  CU(d->d_px.reserve(1));
  CU(cudaMemcpy(d->d_px.get(), &px, sizeof(px), cudaMemcpyHostToDevice));
  return LM_OK;
}

extern "C" int lm_peer_connect(lm_detector* d, int rank, int world, const uint8_t* handles) {
  int rc = peer_connect_common(d, rank, world);
  if (rc) return rc;
  if (!handles) return fail(LM_E_INVALID, "null handles");
  CU(cudaSetDevice(d->device));
  for (int r = 0; r < world; ++r) {
    if (r == rank) { d->px_base[r] = d->px_buf.get(); continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * LM_PEER_HANDLE_BYTES, sizeof(h));
    void* ptr = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      for (int q = 0; q < r; ++q)
        if (q != rank && d->px_base[q]) cudaIpcCloseMemHandle(d->px_base[q]);
      for (int q = 0; q < LM_MAX_PEERS; ++q) d->px_base[q] = nullptr;
      return fail(LM_E_CUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
    }
    d->px_base[r] = (uint8_t*)ptr;
  }
  d->px_ipc = true;
  d->px_rank = rank;
  d->chain.completed = false;
  return peer_upload_descriptor(d);
}

extern "C" int lm_peer_connect_local(lm_detector* d, int rank, int world, void* const* bases) {
  int rc = peer_connect_common(d, rank, world);
  if (rc) return rc;
  if (!bases) return fail(LM_E_INVALID, "null bases");
  CU(cudaSetDevice(d->device));
  for (int r = 0; r < world; ++r) {
    if (!bases[r]) return fail(LM_E_INVALID, "bases[%d] is null", r);
    cudaPointerAttributes at;
    CU(cudaPointerGetAttributes(&at, bases[r]));
    if (at.type != cudaMemoryTypeDevice) return fail(LM_E_INVALID, "bases[%d] is not device memory", r);
    if (at.device != d->device) {
      int can = 0;
      CU(cudaDeviceCanAccessPeer(&can, d->device, at.device));
      if (!can) return fail(LM_E_STATE, "device %d cannot access device %d", d->device, at.device);
      cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(LM_E_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
      (void)cudaGetLastError();
    }
    d->px_base[r] = (uint8_t*)bases[r];
  }
  d->px_base[rank] = d->px_buf.get();
  d->px_ipc = false;
  d->px_rank = rank;
  d->chain.completed = false;
  return peer_upload_descriptor(d);
}

extern "C" int lm_peer_share_pose(lm_detector* d, int on) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (d->px_rank < 0) return fail(LM_E_STATE, "lm_peer_share_pose needs a connected peer exchange");
  d->px_share_pose = on != 0;
  return LM_OK;
}

extern "C" int lm_peer_disconnect(lm_detector* d) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (d->device < 0) return LM_OK;
  CU(cudaSetDevice(d->device));
  CU(cudaStreamSynchronize(d->stream.get()));
  peer_release(d);
  d->chain.completed = false;
  return LM_OK;
}

extern "C" int lm_device_result(lm_detector* d, void** d_block, int64_t* capacity_records) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (!d->d_res) return fail(LM_E_STATE, "no result block yet (call lm_enqueue / lm_run first)");
  if (d_block) *d_block = d->d_res;
  if (capacity_records) *capacity_records = d->res_cap;
  return LM_OK;
}

static bool record_order(const lm_record& a, const lm_record& b) {
  if (a.work != b.work) return a.work < b.work;
  return a.seq < b.seq;
}

// (work, seq) order = the order in which the reference's loops produce the matches (LL.cpp:1797-1939).  The
// records arrive grouped by nothing (atomic append) but with few per template: one counting pass over `work`
// and an insertion sort by `seq` inside each template's run -- O(n + templates) instead of n log n compares.
static void order_records(lm_detector* d, lm_record* r, int64_t n) {
  if (n < 2 || std::is_sorted(r, r + n, record_order)) return;
  const int64_t n_sel = (int64_t)d->sel.size();
  bool in_range = n_sel > 0 && n_sel <= (1 << 22);
  for (int64_t i = 0; in_range && i < n; ++i) in_range = r[i].work >= 0 && r[i].work < n_sel;
  if (!in_range) {
    std::sort(r, r + n, record_order);
    return;
  }
  std::vector<int32_t>& cnt = d->order_cnt;
  cnt.assign((size_t)n_sel + 1, 0);
  for (int64_t i = 0; i < n; ++i) ++cnt[(size_t)r[i].work + 1];
  for (int64_t w = 0; w < n_sel; ++w) cnt[(size_t)w + 1] += cnt[(size_t)w];
  std::vector<lm_record>& tmp = d->order_tmp;
  tmp.resize((size_t)n);
  for (int64_t i = 0; i < n; ++i) {  // place, keeping each run sorted by seq
    const int32_t w = r[i].work;
    int32_t at = cnt[(size_t)w]++;
    tmp[(size_t)at] = r[i];
  }
  // cnt[w] is now the END of run w; runs are short: insertion sort by seq
  int32_t b = 0;
  for (int64_t w = 0; w < n_sel; ++w) {
    const int32_t e = cnt[(size_t)w];
    for (int32_t i = b + 1; i < e; ++i) {
      const lm_record x = tmp[(size_t)i];
      int32_t j = i - 1;
      while (j >= b && tmp[(size_t)j].seq > x.seq) { tmp[(size_t)j + 1] = tmp[(size_t)j]; --j; }
      tmp[(size_t)j + 1] = x;
    }
    b = e;
  }
  memcpy(r, tmp.data(), sizeof(lm_record) * (size_t)n);
}

extern "C" int lm_fetch_records(lm_detector* d, lm_record* out, int64_t cap, int64_t* n_out) {
  if (!d || !n_out) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.completed) return fail(LM_E_STATE, "lm_run has not been called");
  CU(cudaSetDevice(d->device));
  const int64_t n = hres(d)->count;
  *n_out = n;
  if (n > cap) return fail(LM_E_CAPACITY, "%lld records, capacity %lld", (long long)n, (long long)cap);
  lm_record* h = reinterpret_cast<lm_record*>(hres(d) + 1);
  if (n > d->h_valid) {  // the rest, beyond the first-fetch window
    CU(cudaMemcpyAsync(h + d->h_valid, reinterpret_cast<lm_record*>(d->d_res + 1) + d->h_valid,
                       sizeof(lm_record) * (size_t)(n - d->h_valid), cudaMemcpyDeviceToHost, d->stream.get()));
    CU(cudaStreamSynchronize(d->stream.get()));
    d->h_valid = n;
  }
  if (n > 0) {
    memcpy(out, h, sizeof(lm_record) * (size_t)n);
    order_records(d, out, n);  // the reference's pre-sort order
  }
  return LM_OK;
}

namespace {
struct HostMatch {  // LL.h:225-258 with class_index standing in for the class_id string
  int x, y;
  float similarity;
  int class_index, template_id;
  // operator< (similarity descending, then template_id ascending) lives in lm_finish's 64-bit sort keys
  bool operator==(const HostMatch& o) const {
    return x == o.x && y == o.y && similarity == o.similarity && class_index == o.class_index;
  }
};
}  // namespace

extern "C" int lm_finish(lm_detector* d, const lm_record* records, int64_t n, lm_match* out, int64_t cap, int64_t* n_out) {
  if (!d || !n_out || (n > 0 && !records)) return fail(LM_E_INVALID, "null argument");
  if ((int)d->class_of.size() != d->G) {
    d->class_of.resize((size_t)d->G);
    for (int c = 0; c < d->n_classes; ++c)
      for (int g = d->class_begin[c]; g < d->class_begin[c + 1]; ++g) d->class_of[(size_t)g] = c;
  }
  const std::vector<int>& class_of = d->class_of;
  // (work, seq) order = class order -> template_id -> coarse cell, the order in which the reference's loops insert
  // the matches (LL.cpp:1797-1939); callers that fetched the records through lm_fetch_records pass them sorted
  const lm_record* rec = records;
  if (!std::is_sorted(records, records + n, record_order)) {
    d->finish_rec.assign(records, records + n);
    order_records(d, d->finish_rec.data(), n);
    rec = d->finish_rec.data();
  }
  // std::sort(matches) with Match::operator< (similarity descending, then template_id ascending; LL.h:233-240,
  // LL.cpp:1772) on 16-byte keys: the comparator induces the same strict weak order on the same input sequence, so
  // libstdc++'s introsort takes the same decisions and leaves the same permutation (ties included) as it would on
  // the Match structs -- with one integer compare per step instead of a float and an int compare.
  struct SortKey {
    uint64_t key;  // ~order(similarity) : 32 | template_id : 32
    uint32_t idx;
    uint32_t pad;
    bool operator<(const SortKey& o) const { return key < o.key; }
  };
  static thread_local std::vector<HostMatch> v;  // scratch, reused between calls
  v.resize((size_t)n);
  std::vector<uint8_t>& keybuf = d->finish_keys;
  keybuf.resize(sizeof(SortKey) * (size_t)std::max<int64_t>(n, 1));
  SortKey* keys = reinterpret_cast<SortKey*>(keybuf.data());
  for (int64_t i = 0; i < n; ++i) {
    const lm_record& r = rec[i];
    if (r.work < 0 || (size_t)r.work >= d->sel.size())
      return fail(LM_E_INVALID, "record %lld: work index %d out of range", (long long)i, r.work);
    const int g = d->sel[r.work];
    const int c = class_of[g];
    const int tid = g - d->class_begin[c];
    v[(size_t)i] = HostMatch{r.x, r.y, r.similarity, c, tid};
    uint32_t b;
    memcpy(&b, &r.similarity, 4);
    if ((b << 1) == 0u) b = 0u;                                       // -0.0f == 0.0f for operator<
    const uint32_t ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);  // monotone in the float value
    keys[i].key = ((uint64_t)(~ord) << 32) | (uint32_t)tid;           // descending similarity, ascending template_id
    keys[i].idx = (uint32_t)i;
    keys[i].pad = 0;
  }
  std::sort(keys, keys + n);  // LL.cpp:1772
  // std::unique (LL.cpp:1773-1774): drop an element equal (x, y, similarity, class) to the last one KEPT
  int64_t m = 0;
  int64_t last = -1;
  for (int64_t i = 0; i < n; ++i) {
    const HostMatch& h = v[keys[i].idx];
    if (last >= 0 && v[(size_t)last] == h) continue;
    last = keys[i].idx;
    if (m < cap) {
      out[m].x = h.x; out[m].y = h.y; out[m].similarity = h.similarity;
      out[m].class_index = h.class_index; out[m].template_id = h.template_id;
    }
    ++m;
  }
  *n_out = m;
  if (m > cap) return fail(LM_E_CAPACITY, "%lld matches, capacity %lld", (long long)m, (long long)cap);
  return LM_OK;
}

// ---- post-match stage (SURVEY 8f-3) -------------------------------------------------------------
#define LM_POST_MAX 1024

extern "C" int lm_set_boxes(lm_detector* d, const int32_t* wh, int64_t n_templates) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (!wh) {
    d->boxes.clear();
  } else {
    if (n_templates != d->G) return fail(LM_E_INVALID, "%lld box sizes for a bank of %d templates", (long long)n_templates, d->G);
    for (int64_t i = 0; i < 2 * n_templates; ++i)
      if (wh[i] < 0 || wh[i] > 32767) return fail(LM_E_INVALID, "box size outside 0..32767");
    d->boxes.assign(wh, wh + 2 * n_templates);
  }
  d->post_dirty = true;
  return LM_OK;
}

static int prepare_post(lm_detector* d) {
  CU(d->d_post_out.reserve(LM_POST_MAX));
  CU(d->h_post_out.reserve(LM_POST_MAX));
  CU(d->d_post_counts.reserve(4));
  CU(d->h_post_counts.reserve(4));
  CU(d->d_post_live.reserve((size_t)d->res_cap));
  size_t keys = 1;
  while (keys < (size_t)d->res_cap) keys <<= 1;
  if (keys > LM_POST_SMEM_KEYS) CU(d->d_post_keys.reserve(keys));
  if (!d->post_dirty) return LM_OK;
  if (!d->boxes.empty() && (int64_t)d->boxes.size() != 2 * (int64_t)d->G) {
    d->boxes.clear();  // the bank changed under the caller's boxes
    return fail(LM_E_STATE, "box sizes were set for another bank: call lm_set_boxes again");
  }
  const int64_t n = (int64_t)d->sel.size();
  std::vector<int> class_of(d->G);
  for (int c = 0; c < d->n_classes; ++c)
    for (int g = d->class_begin[c]; g < d->class_begin[c + 1]; ++g) class_of[g] = c;
  std::vector<PostInfo> info((size_t)std::max<int64_t>(n, 1));
  for (int64_t i = 0; i < n; ++i) {
    const int g = d->sel[i];
    PostInfo& q = info[i];
    q.class_index = class_of[g];
    q.template_id = g - d->class_begin[class_of[g]];
    if (d->boxes.empty()) {  // Template::width / height of the first modality at level 0 (LL.h:36-45)
      q.width = d->tmeta[((size_t)g * d->S) * 4 + 0];
      q.height = d->tmeta[((size_t)g * d->S) * 4 + 1];
    } else {
      q.width = d->boxes[2 * (size_t)g];
      q.height = d->boxes[2 * (size_t)g + 1];
    }
  }
  CU(d->d_post_info.reserve(info.size()));
  CU(cudaMemcpyAsync(d->d_post_info.get(), info.data(), sizeof(PostInfo) * info.size(), cudaMemcpyHostToDevice, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  d->post_dirty = false;
  return LM_OK;
}

static int enqueue_post(lm_detector* d, double iou_threshold, int top_k) {
  int rc = prepare_post(d);
  if (rc) return rc;
  PostParams p;
  p.hdr = d->d_res; p.capacity = (int32_t)d->res_cap;
  p.info = d->d_post_info.get(); p.n_sel = (int32_t)d->sel.size();
  p.iou_threshold = iou_threshold; p.top_k = top_k;
  p.out = d->d_post_out.get(); p.out_capacity = LM_POST_MAX;
  p.out_counts = d->d_post_counts.get(); p.live = d->d_post_live.get(); p.keys = d->d_post_keys.get();
  CU(launch_pdl(k_post_nms, dim3(1), dim3(1024), sizeof(PostKey) * LM_POST_SMEM_KEYS, d->stream.get(), p));
  ++d->launches;
  return LM_OK;
}

extern "C" int lm_enqueue_post(lm_detector* d, double iou_threshold, int top_k) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (!d->d_res) return fail(LM_E_STATE, "no stages enqueued (call lm_enqueue first)");
  if (top_k > LM_POST_MAX) return fail(LM_E_INVALID, "top_k %d > %d", top_k, LM_POST_MAX);
  if (!(iou_threshold >= 0.0)) return fail(LM_E_INVALID, "IoU threshold must be >= 0");
  CU(cudaSetDevice(d->device));
  int rc = enqueue_post(d, iou_threshold, top_k);
  if (rc) return rc;
  d->chain.iou = iou_threshold;
  d->chain.top_k = top_k;
  d->chain.post = true;
  return LM_OK;
}

// The frame completed through its box NMS: n_out survivors (copied to out unless fetch is false, as for
// lm_complete_detect), n_records the kept records the NMS saw.
static int complete_post(lm_detector* d, lm_match* out, int64_t cap, int64_t* n_out, int64_t* n_records, bool fetch) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d || !n_out) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.post) return fail(LM_E_STATE, "lm_enqueue_post has not been called");
  CU(cudaSetDevice(d->device));
  int rc = complete_frame(d, true, fetch);
  d->chain.post = false;
  if (rc) return rc;
  const int64_t n = d->h_post_counts[0];
  if (n_records) *n_records = d->h_post_counts[1];
  *n_out = n;
  if (!fetch) return LM_OK;
  if (n > cap) return fail(LM_E_CAPACITY, "%lld survivors, capacity %lld", (long long)n, (long long)cap);
  if (n > LM_POST_FIRST) {
    cudaStream_t st = d->stream.get();
    CU(cudaMemcpyAsync(d->h_post_out.get() + LM_POST_FIRST, d->d_post_out.get() + LM_POST_FIRST, sizeof(lm_match) * (size_t)(n - LM_POST_FIRST),
                       cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
  }
  if (n > 0 && out) memcpy(out, d->h_post_out.get(), sizeof(lm_match) * (size_t)n);
  return LM_OK;
}

extern "C" int lm_complete_post(lm_detector* d, lm_match* out, int64_t cap, int64_t* n_out, int64_t* n_records) {
  return complete_post(d, out, cap, n_out, n_records, true);
}

extern "C" int lm_match_top(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols, float threshold,
                            double iou_threshold, int top_k, lm_match* out, int64_t cap, int64_t* n_out, int64_t* n_records) {
  int rc = upload_quantized(d, quantized, rows, cols, false);
  if (rc) return rc;
  rc = lm_enqueue(d, threshold);
  if (rc) return rc;
  rc = lm_enqueue_post(d, iou_threshold, top_k);
  if (rc) return rc;
  return lm_complete_post(d, out, cap, n_out, n_records);
}

// ---- pose stage behind the NMS (lm_pose.h, lm_icp.cu) ---------------------------------------------
extern "C" int lm_set_template_renders(lm_detector* d, int64_t first, int64_t n, const uint16_t* const* depths, int rows, int cols,
                                       const float* K, const float* R, const float* t) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (d->S == 0) return fail(LM_E_STATE, "no template bank loaded");
  if (!d->pose) d->pose = pose_stage_create();
  return pose_stage_register(d->pose, d->class_begin.data(), d->n_classes, first, n, depths, rows, cols, K, R, t);
}

// The connected exchange's pose area for the next pose exchange(s), numbered from seq.
static int pose_share_of(lm_detector* d, int32_t seq, PoseShare* sh) {
  memset(sh, 0, sizeof(*sh));
  for (int r = 0; r < d->px_world; ++r) sh->base[r] = d->px_base[r];
  sh->area_offset = peer_pose_offset(d->px_world, d->px_cap);
  sh->world = d->px_world; sh->rank = d->px_rank; sh->seq = seq;
  sh->timeout_ns = d->px_timeout_ns;
  void* abort_flag = nullptr;
  CU(cudaGetSymbolAddress(&abort_flag, g_px_abort));
  sh->abort_flag = (int*)abort_flag;
  return LM_OK;
}

static int enqueue_pose(lm_detector* d) {
  PoseShare sh;
  const bool share = d->px_rank >= 0 && d->px_share_pose;
  if (share) {
    if (d->px_seq < 1) return fail(LM_E_STATE, "pose exchange: no frame has been enqueued on the connected exchange");
    int rc = pose_share_of(d, ++d->px_pose_seq, &sh);
    if (rc) return rc;
  }
  const FrameChain& c = d->chain;
  PoseRun run;
  run.o = {d->fe[0].rows, d->fe[0].cols, c.use_scene, c.max_iter, c.estimation, d->stream.get(), share ? &sh : nullptr, c.verify, c.search};
  run.n_frames = 1; run.first = nullptr; run.d_counts = d->d_post_counts.get();
  run.bound = c.top_k > 0 ? std::min(c.top_k, LM_POST_MAX) : LM_POST_MAX;
  run.d_surv = d->d_post_out.get(); run.d_scene = d->fe_depth.get(); run.sK = c.sK;
  run.pose_nms = 0;  // lm_enqueue_pose_nms may follow
  return pose_stage_enqueue(d->pose, run, &d->launches);
}

extern "C" int lm_enqueue_pose(lm_detector* d, const float* sceneK, int max_iterations, int use_scene_cloud) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d || !sceneK) return fail(LM_E_INVALID, "null argument");
  if (max_iterations < 0) return fail(LM_E_INVALID, "max_iterations < 0");
  if (d->pose_estimation == LM_POSE_PSO && d->px_rank >= 0 && d->px_share_pose)
    return fail(LM_E_STATE, "the pose stage shared over the ranks does not run LM_POSE_PSO: turn lm_peer_share_pose off");
  FrameChain& c = d->chain;
  if (!c.post) return fail(LM_E_STATE, "lm_enqueue_post has not been called");
  if (!d->frame_depth) return fail(LM_E_STATE, "the frame has no depth image: upload it with lm_upload_images");
  if (!d->pose || !pose_stage_covers(d->pose, d->sel.data(), (int64_t)d->sel.size()))
    return fail(LM_E_STATE, "no template renders registered for every selected template of this bank (lm_set_template_renders)");
  CU(cudaSetDevice(d->device));
  memcpy(c.sK, sceneK, sizeof(c.sK));
  c.max_iter = max_iterations;
  c.use_scene = use_scene_cloud ? 1 : 0;
  c.estimation = d->pose_estimation;
  c.verify = d->pose_verify;
  c.search = d->pose_search;
  c.pose_nms = false;  // a new pose stage: any pose NMS enqueued before belongs to an abandoned frame
  int rc = enqueue_pose(d);
  if (rc) return rc;
  c.pose = true;
  return LM_OK;
}

extern "C" int lm_complete_pose(lm_detector* d, lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap,
                                int64_t* n_out, int64_t* n_records) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d || !n_out || (cap > 0 && (!R_out || !t_out || !residual))) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.pose) return fail(LM_E_STATE, "lm_enqueue_pose has not been called");
  if (d->chain.pose_nms) return fail(LM_E_STATE, "lm_enqueue_pose_nms is pending: complete the frame with lm_complete_detect");
  int rc = complete_post(d, out, cap, n_out, n_records, true);
  d->chain.pose = false;
  if (rc) return rc;
  int64_t n = 0, counts[4], stats[4];
  rc = pose_stage_finish(d->pose, d->h_post_out.get(), *n_out, out, R_out, t_out, residual, cap, &n, counts, stats);
  if (rc) return rc;
  memcpy(d->pose_stats, stats, sizeof(stats));
  return LM_OK;
}

static int enqueue_pose_nms(lm_detector* d) {
  return pose_stage_enqueue_nms(d->pose, d->chain.nms_thr, &d->launches);
}

extern "C" int lm_enqueue_pose_nms(lm_detector* d, double translation_threshold_mm) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (!(translation_threshold_mm >= 0.0)) return fail(LM_E_INVALID, "translation threshold must be >= 0 (NaN given or negative)");
  if (!d->chain.pose) return fail(LM_E_STATE, "lm_enqueue_pose has not been called");
  if (d->chain.pose_nms) return fail(LM_E_STATE, "lm_enqueue_pose_nms was already called for this frame");
  CU(cudaSetDevice(d->device));
  d->chain.nms_thr = translation_threshold_mm;
  int rc = enqueue_pose_nms(d);
  if (rc) return rc;
  d->chain.pose_nms = true;
  return LM_OK;
}

extern "C" int lm_complete_detect(lm_detector* d, lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap,
                                  int64_t* n_out, int64_t* n_survivors, int64_t* n_posed, int64_t* n_records) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d || !n_out || (cap > 0 && (!out || !R_out || !t_out || !residual))) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.pose_nms) return fail(LM_E_STATE, "lm_enqueue_pose_nms has not been called");
  int64_t n_surv = 0;
  int rc = complete_post(d, nullptr, 0, &n_surv, n_records, false);
  d->chain.pose = d->chain.pose_nms = false;
  if (rc) return rc;
  int64_t counts[4], stats[4];
  rc = pose_stage_finish(d->pose, nullptr, n_surv, out, R_out, t_out, residual, cap, n_out, counts, stats);
  if (rc && rc != LM_E_CAPACITY) return rc;  // a capacity error comes with the counts
  if (n_survivors) *n_survivors = counts[1];
  if (n_posed) *n_posed = counts[2];
  if (rc) return rc;
  memcpy(d->pose_stats, stats, sizeof(stats));
  return LM_OK;
}

extern "C" int lm_set_pose_estimation(lm_detector* d, int estimation) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  const int rc = check_estimation(estimation);
  if (rc) return rc;
  d->pose_estimation = estimation;
  return LM_OK;
}

extern "C" int lm_set_pose_search(lm_detector* d, int particles, int iterations, double dt_mm, double dr_deg, double clamp_mm,
                                  uint64_t seed) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  return pose_search_make(particles, iterations, dt_mm, dr_deg, clamp_mm, seed, &d->pose_search);
}

extern "C" int lm_set_pose_verify(lm_detector* d, int on, double inlier_mm, int rank_by, double min_score) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  const int rc = check_inlier_mm(inlier_mm);
  if (rc) return rc;
  if (rank_by != LM_VERIFY_RANK_FITNESS && rank_by != LM_VERIFY_RANK_SCORE)
    return fail(LM_E_INVALID, "unknown rank_by %d (LM_VERIFY_RANK_FITNESS 0, LM_VERIFY_RANK_SCORE 1)", rank_by);
  if (std::isnan(min_score)) return fail(LM_E_INVALID, "min_score is NaN (-INFINITY: no minimum)");
  if (!on && (rank_by != LM_VERIFY_RANK_FITNESS || min_score != -INFINITY))
    return fail(LM_E_INVALID, "rank_by score and min_score need pose verification on");
  d->pose_verify = {on ? 1 : 0, rank_by, inlier_mm, min_score};
  return LM_OK;
}

extern "C" int lm_pose_verify(lm_detector* d, float* score, int32_t* counts6, int64_t cap, int64_t* n) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (!d->pose) return fail(LM_E_STATE, "no pose stage has run");
  return pose_stage_verify(d->pose, score, counts6, cap, n);
}

extern "C" int lm_debug_pose_clouds(lm_detector* d, int slot, int what, void* out, int64_t cap) {
  if (!d || !out) return fail(LM_E_INVALID, "null argument");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle");
  if (!d->pose) return fail(LM_E_STATE, "no pose stage has run");
  CU(cudaSetDevice(d->device));
  CU(cudaStreamSynchronize(d->stream.get()));
  return pose_stage_clouds(d->pose, slot, what, out, cap);
}

// Object i of a track call (objects of its frame, or of lm_track) as the pose stage's TrackObject: LM_E_INVALID or
// LM_E_STATE with the message unless its class, template, T and render are good.
static int track_object(lm_detector* d, const lm_track_object& o, int i, TrackObject* out) {
  if (o.class_index < 0 || o.class_index >= d->n_classes)
    return fail(LM_E_INVALID, "object %d: class %d outside the bank's %d classes", i, o.class_index, d->n_classes);
  const int32_t nt = d->class_begin[o.class_index + 1] - d->class_begin[o.class_index];
  if (o.template_id < 0 || o.template_id >= nt)
    return fail(LM_E_INVALID, "object %d: template %d outside class %d's %d templates", i, o.template_id, o.class_index, nt);
  for (int k = 0; k < 16; ++k)
    if (!std::isfinite(o.T[k])) return fail(LM_E_INVALID, "object %d: T[%d] is not finite", i, k);
  out->g = d->class_begin[o.class_index] + o.template_id;
  memcpy(out->T, o.T, sizeof(o.T));
  const int32_t g = (int32_t)out->g;
  if (!d->pose || !pose_stage_covers(d->pose, &g, 1))
    return fail(LM_E_STATE, "object %d: no template render registered for class %d, template %d (lm_set_template_renders)", i,
                o.class_index, o.template_id);
  return LM_OK;
}

// lm_track, lm_track_device, lm_track_batch, lm_track_batch_device and (peers true: needs a connected exchange, which
// the others refuse) lm_peer_track_batch, lm_peer_track_batch_device: every refusal before any device work, then the
// scenes and one track run of the pose stage on the detector's stream, its chunks shared over the ranks with
// lm_peer_share_pose.  planes null: n_frames host images contiguous at depth; else frame f's device plane planes[f]
// (pitch, format, scale), ordered on `caller`.  Frame f has n_objects[f] objects, in frame order; batch false (lm_track,
// lm_track_device: one frame): the single call's messages.
static int track(lm_detector* d, bool peers, bool batch, int n_frames, const void* depth, const void* const* planes, int64_t pitch, int format,
                 float scale, cudaStream_t caller, int rows, int cols, const float* sceneK, const lm_track_object* objects,
                 const int32_t* n_objects, int max_iterations, int margin_px, double* T_out, double* R_out, double* t_out,
                 float* residual, int32_t* status, int32_t* box) {
  if (batch) {
    if (!d || !depth || !sceneK || !n_objects) return fail(LM_E_INVALID, "null argument");
    if (n_frames < 1) return fail(LM_E_INVALID, "n_frames %d < 1", n_frames);
    for (int f = 0; f < n_frames; ++f)
      if (n_objects[f] < 0 || n_objects[f] > LM_POST_MAX)
        return fail(LM_E_INVALID, "frame %d: %d objects, a track run takes 0 to %d per frame", f, n_objects[f], LM_POST_MAX);
  }
  std::vector<int64_t> first((size_t)n_frames + 1, 0);
  for (int f = 0; f < n_frames; ++f) first[(size_t)f + 1] = first[(size_t)f] + n_objects[f];
  const int64_t n = first[(size_t)n_frames];
  if (!d || !depth || !sceneK || n < 0 || (n > 0 && (!objects || !T_out || !R_out || !t_out || !residual || !status || !box)))
    return fail(LM_E_INVALID, batch ? "null argument" : "null argument or n < 0");
  if (n > LM_POST_MAX && !batch) return fail(LM_E_INVALID, "%d objects, a track run takes at most %d", (int)n, LM_POST_MAX);
  if (rows <= 0 || cols <= 0) return fail(LM_E_INVALID, "empty depth image %d x %d", rows, cols);
  if (max_iterations < 0) return fail(LM_E_INVALID, "max_iterations < 0");
  if (margin_px < 0) return fail(LM_E_INVALID, "margin_px %d < 0", margin_px);
  int rc = planes ? check_depth_format("depth", format, scale) : LM_OK;
  if (rc) return rc;
  if (d->pose_estimation == LM_POSE_PSO)
    return fail(LM_E_STATE, "tracking runs an ICP: LM_POSE_PSO starts from an identity rotation (lm_set_pose_estimation)");
  if (!peers && d->px_rank >= 0)
    return fail(LM_E_STATE, "tracking does not run with a connected peer exchange (every rank calls lm_peer_track_batch)");
  std::vector<TrackObject> obj((size_t)n);
  for (int f = 0; f < n_frames; ++f)
    for (int64_t k = first[(size_t)f]; k < first[(size_t)f + 1]; ++k) {
      rc = track_object(d, objects[k], (int)(k - first[(size_t)f]), &obj[(size_t)k]);
      if (rc && batch) return fail(rc, "frame %d: %s", f, std::string(g_err).c_str());
      if (rc) return rc;
    }
  if (peers && d->px_rank < 0) return fail(LM_E_STATE, "lm_peer_track_batch needs a connected peer exchange");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (planes) {
    rc = check_device_stream(d->device, caller);
    const int sz = format == LM_DEPTH_F32 ? 4 : 2;
    for (int f = 0; f < n_frames && !rc; ++f) {
      char what[40] = "depth";
      if (batch) snprintf(what, sizeof(what), "depth[%d]", f);
      rc = check_device_plane(d->device, what, planes[f], pitch, (int64_t)sz * cols, sz);
    }
    if (rc) return rc;
  }
  if (!d->pose) return fail(LM_E_STATE, "no template renders registered (lm_set_template_renders)");
  CU(cudaSetDevice(d->device));
  cudaStream_t st = d->stream.get();
  d->chain.pose = d->chain.pose_nms = false;  // the stage's buffers now hold the track run: a pending frame's pose stage is abandoned
  const uint16_t* scene = nullptr;
  if (planes) {  // the reads of the caller's planes start behind its stream's work, and its later work waits for the conversions
    if (!d->ev_in.get()) CU(d->ev_in.create(cudaEventDisableTiming));
    if (!d->ev_out.get()) CU(d->ev_out.create(cudaEventDisableTiming));
    CU(cudaEventRecord(d->ev_in.get(), caller));
    CU(cudaStreamWaitEvent(st, d->ev_in.get(), 0));
    rc = pose_track_scene(d->pose, st, n_frames, nullptr, planes, pitch, format, scale, rows, cols, &scene, &d->launches);
    CU(cudaEventRecord(d->ev_out.get(), st));
    CU(cudaStreamWaitEvent(caller, d->ev_out.get(), 0));
  } else {
    rc = pose_track_scene(d->pose, st, n_frames, static_cast<const uint16_t*>(depth), nullptr, 2 * (int64_t)cols, LM_DEPTH_U16_MM, 1.f,
                          rows, cols, &scene, &d->launches);
  }
  if (rc) return rc;
  PoseShare sh;
  const bool share = peers && d->px_share_pose;
  if (share) {  // one pose exchange per chunk, numbered on from the frames' and batches' ones
    rc = pose_share_of(d, d->px_pose_seq + 1, &sh);
    if (rc) return rc;
    d->px_pose_seq += pose_batch_chunks(first[(size_t)n_frames]);
  }
  PoseOptions o = {rows, cols, 1, max_iterations, d->pose_estimation, st, share ? &sh : nullptr, d->pose_verify, d->pose_search,
                   d->track_views, d->track_view_tau};
  return pose_stage_track(d->pose, o, n_frames, scene, sceneK, obj.data(), first.data(), margin_px, &d->launches, T_out, R_out, t_out,
                          residual, status, box, peers ? d->pose_stats : nullptr);
}

extern "C" int lm_track(lm_detector* d, const uint16_t* depth, int rows, int cols, const float* sceneK, const lm_track_object* objects,
                        int n, int max_iterations, int margin_px, double* T_out, double* R_out, double* t_out, float* residual,
                        int32_t* status, int32_t* box) {
  return track(d, false, false, 1, depth, nullptr, 0, LM_DEPTH_U16_MM, 1.f, nullptr, rows, cols, sceneK, objects, &n, max_iterations, margin_px,
               T_out, R_out, t_out, residual, status, box);
}

extern "C" int lm_track_device(lm_detector* d, const void* depth, int64_t depth_pitch, int depth_format, float depth_scale, int rows,
                               int cols, const float* sceneK, const lm_track_object* objects, int n, int max_iterations, int margin_px,
                               double* T_out, double* R_out, double* t_out, float* residual, int32_t* status, int32_t* box, void* stream) {
  return track(d, false, false, 1, depth, &depth, depth_pitch, depth_format, depth_scale, (cudaStream_t)stream, rows, cols, sceneK, objects, &n,
               max_iterations, margin_px, T_out, R_out, t_out, residual, status, box);
}

extern "C" int lm_track_batch(lm_detector* d, int n_frames, const uint16_t* depth, int rows, int cols, const float* sceneK,
                              const lm_track_object* objects, const int32_t* n_objects, int max_iterations, int margin_px, double* T_out,
                              double* R_out, double* t_out, float* residual, int32_t* status, int32_t* box) {
  return track(d, false, true, n_frames, depth, nullptr, 0, LM_DEPTH_U16_MM, 1.f, nullptr, rows, cols, sceneK, objects, n_objects, max_iterations,
               margin_px, T_out, R_out, t_out, residual, status, box);
}

extern "C" int lm_track_batch_device(lm_detector* d, int n_frames, const void* const* depth, int64_t depth_pitch, int depth_format,
                                     float depth_scale, int rows, int cols, const float* sceneK, const lm_track_object* objects,
                                     const int32_t* n_objects, int max_iterations, int margin_px, double* T_out, double* R_out,
                                     double* t_out, float* residual, int32_t* status, int32_t* box, void* stream) {
  return track(d, false, true, n_frames, depth, depth, depth_pitch, depth_format, depth_scale, (cudaStream_t)stream, rows, cols, sceneK, objects,
               n_objects, max_iterations, margin_px, T_out, R_out, t_out, residual, status, box);
}

extern "C" int lm_peer_track_batch(lm_detector* d, int n_frames, const uint16_t* depth, int rows, int cols, const float* sceneK,
                                   const lm_track_object* objects, const int32_t* n_objects, int max_iterations, int margin_px,
                                   double* T_out, double* R_out, double* t_out, float* residual, int32_t* status, int32_t* box) {
  return track(d, true, true, n_frames, depth, nullptr, 0, LM_DEPTH_U16_MM, 1.f, nullptr, rows, cols, sceneK, objects, n_objects,
               max_iterations, margin_px, T_out, R_out, t_out, residual, status, box);
}

extern "C" int lm_peer_track_batch_device(lm_detector* d, int n_frames, const void* const* depth, int64_t depth_pitch, int depth_format,
                                          float depth_scale, int rows, int cols, const float* sceneK, const lm_track_object* objects,
                                          const int32_t* n_objects, int max_iterations, int margin_px, double* T_out, double* R_out,
                                          double* t_out, float* residual, int32_t* status, int32_t* box, void* stream) {
  return track(d, true, true, n_frames, depth, depth, depth_pitch, depth_format, depth_scale, (cudaStream_t)stream, rows, cols, sceneK,
               objects, n_objects, max_iterations, margin_px, T_out, R_out, t_out, residual, status, box);
}

extern "C" int lm_set_track_views(lm_detector* d, int on, double turn_deg) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  double tau = 0.0;
  const int rc = track_view_tau(on, turn_deg, &tau);
  if (rc) return rc;
  d->track_views = on ? 1 : 0;
  d->track_view_tau = tau;
  return LM_OK;
}

extern "C" int lm_track_templates(lm_detector* d, int32_t* template_id, int64_t cap, int64_t* n) {
  if (!d || !n) return fail(LM_E_INVALID, "null argument");
  if (!d->pose) return fail(LM_E_STATE, "no pose stage has run");
  return pose_stage_track_templates(d->pose, template_id, cap, n);
}

extern "C" int lm_pose_transforms(lm_detector* d, double* T_out, int64_t cap, int64_t* n) {
  if (!d || !n) return fail(LM_E_INVALID, "null argument");
  if (!d->pose) return fail(LM_E_STATE, "no pose stage has run");
  if (d->device >= 0) CU(cudaSetDevice(d->device));
  return pose_stage_transforms(d->pose, T_out, cap, n);
}

extern "C" int lm_set_template_depths(lm_detector* d, int64_t first, int64_t n, const float* z_mm) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (first < 0 || n < 0 || first + n > d->G)
    return fail(LM_E_INVALID, "templates [%lld, %lld) outside the bank's %d", (long long)first, (long long)(first + n), d->G);
  if (n > 0 && !z_mm) return fail(LM_E_INVALID, "null distances");
  if (d->tdepth.size() != (size_t)d->G) d->tdepth.assign((size_t)d->G, NAN);
  for (int64_t i = 0; i < n; ++i) d->tdepth[(size_t)(first + i)] = z_mm[i];
  d->gate_dirty = true;
  return LM_OK;
}

extern "C" int lm_set_depth_gate(lm_detector* d, int on, double tolerance) {
  if (!d) return fail(LM_E_INVALID, "null detector");
  if (!(tolerance >= 0.0 && tolerance < 1.0)) return fail(LM_E_INVALID, "depth gate tolerance %g outside [0, 1)", tolerance);
  if (tolerance != d->gate_tau) d->gate_dirty = true;
  d->gate_on = on != 0;
  d->gate_tau = tolerance;
  return LM_OK;
}

extern "C" int lm_depth_gate_stats(lm_detector* d, int64_t* out4) {
  if (!d || !out4) return fail(LM_E_INVALID, "null argument");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle");
  if (!d->chain.plan.gated || !d->d_res) return fail(LM_E_STATE, "the last frame did not run with the depth gate");
  CU(cudaSetDevice(d->device));
  const LevelHost& low = d->lv[d->L - 1];
  std::vector<uint32_t> cells((size_t)low.plane);
  unsigned before = 0;
  lm_result_header hdr;
  CU(cudaMemcpyAsync(cells.data(), d->d_cells.get(), sizeof(uint32_t) * cells.size(), cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaMemcpyAsync(&before, d->d_gate_before.get(), sizeof(unsigned), cudaMemcpyDeviceToHost, d->stream.get()));
  // the header the coarse scan wrote, with its shard's candidate count (a result-block retry carries it to the grown block)
  const lm_result_header* scan = d->px_rank >= 0 ? exchange_block(d) : d->d_res;
  CU(cudaMemcpyAsync(&hdr, scan, sizeof(hdr), cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  int64_t empty = 0;
  for (uint32_t c : cells) empty += (c & 0xFFFFu) > (c >> 16);
  out4[0] = before;
  out4[1] = hdr.coarse_candidates;
  out4[2] = empty;
  out4[3] = d->gate_with_z;
  return LM_OK;
}

extern "C" int lm_pose_stats(lm_detector* d, int64_t* out4) {
  if (!d || !out4) return fail(LM_E_INVALID, "null argument");
  memcpy(out4, d->pose_stats, sizeof(d->pose_stats));
  return LM_OK;
}

// lm_detect_batch (peers false: refuses a connected exchange) and lm_peer_detect_batch (peers true: needs one).  With
// peers, each frame's match runs the fused record exchange; every rank then holds the same survivors, so the chunks of
// the pose stage -- shared or not -- are the same on every rank.
// lm_detect_batch_device's frames: frame f is device frame (rgb[f], depth[f], masks[2f], masks[2f + 1]), one pitch per plane.
struct DeviceFrames {
  const uint8_t* const* rgb; int64_t rgb_pitch;
  const void* const* depth; int64_t depth_pitch; int format; float scale;
  const uint8_t* const* masks; int64_t mask_pitch;
  cudaStream_t stream;
  DeviceFrame frame(int f) const {
    return {rgb[f], rgb_pitch, depth[f], depth_pitch, format, scale, {masks ? masks[2 * f] : nullptr, masks ? masks[2 * f + 1] : nullptr},
            mask_pitch};
  }
};

// dev NULL: host frames rgb / depth (lm_detect_batch, lm_peer_detect_batch); else dev's device frames, rgb / depth NULL.
static int detect_batch(lm_detector* d, bool peers, int n_frames, const uint8_t* rgb, const uint16_t* depth, const DeviceFrames* dev,
                        int rows, int cols, const uint8_t* const* masks, float threshold, const float* sceneK, double iou_threshold, int top_k,
                        int max_iterations, int use_scene_cloud, int pose_nms, double translation_threshold_mm, lm_match* out,
                        double* R_out, double* t_out, float* residual, int64_t cap, int64_t* n_out, int64_t* frame_counts) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d || (dev ? (!dev->rgb || !dev->depth) : (!rgb || !depth)) || !sceneK || !n_out || !frame_counts || (cap > 0 && (!out || !R_out || !t_out || !residual)))
    return fail(LM_E_INVALID, "null argument");
  if (n_frames < 1) return fail(LM_E_INVALID, "n_frames %d < 1", n_frames);
  if (rows <= 0 || cols <= 0) return fail(LM_E_INVALID, "empty frame size %d x %d", rows, cols);
  if (top_k > LM_POST_MAX) return fail(LM_E_INVALID, "top_k %d > %d", top_k, LM_POST_MAX);
  if (!(iou_threshold >= 0.0)) return fail(LM_E_INVALID, "IoU threshold must be >= 0");
  if (max_iterations < 0) return fail(LM_E_INVALID, "max_iterations < 0");
  if (pose_nms && !(translation_threshold_mm >= 0.0))
    return fail(LM_E_INVALID, "translation threshold must be >= 0 (NaN given or negative)");
  if (!peers && d->px_rank >= 0)
    return fail(LM_E_STATE, "lm_detect_batch does not run with a connected peer exchange (every rank calls lm_peer_detect_batch)");
  if (peers && d->px_rank < 0) return fail(LM_E_STATE, "lm_peer_detect_batch needs a connected peer exchange");
  if (peers && d->px_share_pose && d->pose_estimation == LM_POSE_PSO)
    return fail(LM_E_STATE, "the pose stage shared over the ranks does not run LM_POSE_PSO: turn lm_peer_share_pose off");
  if (!d->pose || !pose_stage_covers(d->pose, d->sel.data(), (int64_t)d->sel.size()))
    return fail(LM_E_STATE, "no template renders registered for every selected template of this bank (lm_set_template_renders)");
  CU(cudaSetDevice(d->device));
  int lrows[LM_MAX_LEVELS], lcols[LM_MAX_LEVELS];
  for (int f = 0; dev && f < n_frames; ++f) {
    int rc = check_device_frame(d, dev->frame(f), rows, cols, dev->stream, lrows, lcols);
    if (rc) return fail(rc, "frame %d: %s", f, std::string(g_err).c_str());
  }
  cudaStream_t st = d->stream.get();
  d->chain.pose = d->chain.pose_nms = false;  // a batch starts new frames: a pending single-frame pose stage is abandoned
  const int bound = top_k > 0 ? top_k : LM_POST_MAX;  // most survivors k_post_nms writes per frame
  const size_t n0 = (size_t)rows * cols;
  uint16_t* d_scene = nullptr;
  lm_match* d_surv = nullptr;
  int rc = pose_batch_reserve(d->pose, st, n_frames, (int64_t)n0, (int64_t)n_frames * bound, d->pose_verify.on != 0, &d_scene, &d_surv);
  if (rc) return rc;
  std::vector<int64_t> first((size_t)n_frames + 1, 0);
  std::vector<lm_match> surv(pose_nms ? 0 : (size_t)n_frames * bound);
  for (int f = 0; f < n_frames; ++f) {
    // the single-frame chain up to the box NMS, completed as a single frame is (complete_frame)
    rc = dev ? bind_images_device(d, dev->frame(f), rows, cols, lrows, lcols, dev->stream)
             : lm_upload_images(d, rgb + f * n0 * 3, depth + f * n0, rows, cols, masks ? masks[2 * f] : nullptr, masks ? masks[2 * f + 1] : nullptr);
    if (rc) return rc;
    rc = lm_enqueue(d, threshold);
    if (rc) return rc;
    rc = lm_enqueue_post(d, iou_threshold, top_k);
    if (rc) return rc;
    int64_t n = 0, n_rec = 0;
    rc = complete_post(d, pose_nms ? nullptr : surv.data() + first[f], bound, &n, &n_rec, !pose_nms);
    if (rc) return rc;
    // the next frame's post stage and upload overwrite both: copy them out first, on the stream
    if (n > 0) CU(cudaMemcpyAsync(d_surv + first[f], d->d_post_out.get(), sizeof(lm_match) * (size_t)n, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(d_scene + f * n0, d->fe_depth.get(), sizeof(uint16_t) * n0, cudaMemcpyDeviceToDevice, st));
    first[f + 1] = first[f] + n;
    frame_counts[4 * f + 1] = n;
    frame_counts[4 * f + 3] = n_rec;
  }
  PoseShare sh;
  const bool share = peers && d->px_share_pose;
  if (share) {  // one pose exchange per chunk, numbered on from the single frames' ones
    rc = pose_share_of(d, d->px_pose_seq + 1, &sh);
    if (rc) return rc;
    d->px_pose_seq += pose_batch_chunks(first[n_frames]);
  }
  PoseRun run;
  run.o = {rows, cols, use_scene_cloud ? 1 : 0, max_iterations, d->pose_estimation, st, share ? &sh : nullptr, d->pose_verify,
           d->pose_search};
  run.n_frames = n_frames; run.first = first.data(); run.d_counts = nullptr; run.bound = bound;
  run.d_surv = d_surv; run.d_scene = d_scene; run.sK = sceneK;
  run.pose_nms = pose_nms ? 1 : 0;
  rc = pose_stage_enqueue(d->pose, run, &d->launches);
  if (!rc && pose_nms) rc = pose_stage_enqueue_nms(d->pose, translation_threshold_mm, &d->launches);
  if (rc) return rc;
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  return pose_stage_finish(d->pose, surv.data(), 0, out, R_out, t_out, residual, cap, n_out, frame_counts, peers ? d->pose_stats : nullptr);
}

extern "C" int lm_detect_batch(lm_detector* d, int n_frames, const uint8_t* rgb, const uint16_t* depth, int rows, int cols,
                               const uint8_t* const* masks, float threshold, const float* sceneK, double iou_threshold, int top_k,
                               int max_iterations, int use_scene_cloud, int pose_nms, double translation_threshold_mm, lm_match* out,
                               double* R_out, double* t_out, float* residual, int64_t cap, int64_t* n_out, int64_t* frame_counts) {
  return detect_batch(d, false, n_frames, rgb, depth, nullptr, rows, cols, masks, threshold, sceneK, iou_threshold, top_k, max_iterations,
                      use_scene_cloud, pose_nms, translation_threshold_mm, out, R_out, t_out, residual, cap, n_out, frame_counts);
}

extern "C" int lm_peer_detect_batch(lm_detector* d, int n_frames, const uint8_t* rgb, const uint16_t* depth, int rows, int cols,
                                    const uint8_t* const* masks, float threshold, const float* sceneK, double iou_threshold, int top_k,
                                    int max_iterations, int use_scene_cloud, int pose_nms, double translation_threshold_mm,
                                    lm_match* out, double* R_out, double* t_out, float* residual, int64_t cap, int64_t* n_out,
                                    int64_t* frame_counts) {
  return detect_batch(d, true, n_frames, rgb, depth, nullptr, rows, cols, masks, threshold, sceneK, iou_threshold, top_k, max_iterations,
                      use_scene_cloud, pose_nms, translation_threshold_mm, out, R_out, t_out, residual, cap, n_out, frame_counts);
}

extern "C" int lm_detect_batch_device(lm_detector* d, int n_frames, const uint8_t* const* rgb, int64_t rgb_pitch, const void* const* depth,
                                      int64_t depth_pitch, int depth_format, float depth_scale, int rows, int cols,
                                      const uint8_t* const* masks, int64_t mask_pitch, void* stream, float threshold, const float* sceneK,
                                      double iou_threshold, int top_k, int max_iterations, int use_scene_cloud, int pose_nms,
                                      double translation_threshold_mm, lm_match* out, double* R_out, double* t_out, float* residual,
                                      int64_t cap, int64_t* n_out, int64_t* frame_counts) {
  const DeviceFrames dev = {rgb, rgb_pitch, depth, depth_pitch, depth_format, depth_scale, masks, mask_pitch, (cudaStream_t)stream};
  return detect_batch(d, false, n_frames, nullptr, nullptr, &dev, rows, cols, masks, threshold, sceneK, iou_threshold, top_k,
                      max_iterations, use_scene_cloud, pose_nms, translation_threshold_mm, out, R_out, t_out, residual, cap, n_out,
                      frame_counts);
}

// lm_run + lm_fetch_records + lm_finish of the frame just uploaded: the match list of lm_match_quantized / lm_match_images.
static int match_frame(lm_detector* d, float threshold, lm_match* out, int64_t cap, int64_t* n_out) {
  int rc = lm_run(d, threshold);
  if (rc) return rc;
  const int64_t n = hres(d)->count;
  std::vector<lm_record> rec((size_t)n);
  int64_t got = 0;
  rc = lm_fetch_records(d, rec.data(), n, &got);
  if (rc) return rc;
  return lm_finish(d, rec.data(), got, out, cap, n_out);
}

extern "C" int lm_match_quantized(lm_detector* d, const uint8_t* const* quantized, const int* rows, const int* cols,
                                  float threshold, lm_match* out, int64_t cap, int64_t* n_out) {
  int rc = upload_quantized(d, quantized, rows, cols, false);  // lm_run synchronises before this call returns
  return rc ? rc : match_frame(d, threshold, out, cap, n_out);
}

extern "C" int lm_match_images(lm_detector* d, const uint8_t* rgb, const uint16_t* depth, int rows, int cols, const uint8_t* mask_color,
                               const uint8_t* mask_depth, float threshold, lm_match* out, int64_t cap, int64_t* n_out) {
  int rc = lm_upload_images(d, rgb, depth, rows, cols, mask_color, mask_depth);
  return rc ? rc : match_frame(d, threshold, out, cap, n_out);
}

extern "C" int lm_debug_quantized(lm_detector* d, int level, int modality, uint8_t* out, int64_t cap) {
  if (!d || !out) return fail(LM_E_INVALID, "null argument");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle");
  if (!d->have_frame) return fail(LM_E_STATE, "no frame uploaded");
  if (level < 0 || level >= d->L || modality < 0 || modality >= d->M) return fail(LM_E_INVALID, "bad level/modality");
  const LevelHost& lv = d->lv[level];
  const int64_t n = (int64_t)lv.rows * lv.cols;
  if (n > cap) return fail(LM_E_CAPACITY, "need %lld bytes", (long long)n);
  CU(cudaSetDevice(d->device));
  CU(cudaMemcpyAsync(out, lv.q_src[modality], (size_t)n, cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  return LM_OK;
}

extern "C" int lm_debug_linear_memories(lm_detector* d, int level, int modality, uint8_t* out, int64_t cap) {
  if (!d || !out) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.completed) return fail(LM_E_STATE, "lm_run has not been called");
  if (level < 0 || level >= d->L || modality < 0 || modality >= d->M) return fail(LM_E_INVALID, "bad level/modality");
  const LevelHost& lv = d->lv[level];
  if ((int64_t)lv.mod_stride > cap) return fail(LM_E_CAPACITY, "need %u bytes", lv.mod_stride);
  CU(cudaSetDevice(d->device));
  if ((d->chain.plan.stale >> level) & 1) {
    // the last run did not build this level's bytes (H-planes only, or a lowest level nothing read them from): build them
    // now, from the frame that is still bound, without touching the bit-planes
    K1Plan k;
    plan_k1(d, -1, true, false, k);
    const int b0 = level == d->L - 1 ? 0 : k.p.lv[level + 1].block_end;
    int rc = launch_k1(d, k, b0, k.p.lv[level].block_end - b0);
    if (rc) return rc;
    d->chain.plan.stale &= ~(1 << level);
  }
  CU(cudaMemcpyAsync(out, lv.d_lm.get() + (size_t)modality * lv.mod_stride, lv.mod_stride, cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  return LM_OK;
}

// The lowest level's spread bit-planes as the last lm_run left them: [M][8][lbw] words (live words, then the slack the
// coarse scan's zero descriptor reads).
extern "C" int lm_debug_bit_planes(lm_detector* d, uint32_t* out, int64_t cap, int64_t* n_words) {
  if (!d || !n_words || (!out && cap > 0)) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.completed) return fail(LM_E_STATE, "lm_run has not been called");
  const LevelHost& low = d->lv[d->L - 1];
  *n_words = (int64_t)low.d_bp.size();
  if (*n_words > cap) return fail(LM_E_CAPACITY, "need %lld words", (long long)*n_words);
  if (*n_words == 0) return LM_OK;
  CU(cudaSetDevice(d->device));
  CU(cudaMemcpyAsync(out, low.d_bp.get(), sizeof(uint32_t) * (size_t)*n_words, cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  return LM_OK;
}

extern "C" int lm_debug_time_k1(lm_detector* d, int level, int reps, float* us) {
  if (!d || !us) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.completed) return fail(LM_E_STATE, "lm_run has not been called");
  if (level < -1 || level >= d->L || reps < 1) return fail(LM_E_INVALID, "bad level/reps");
  CU(cudaSetDevice(d->device));
  const K1Plan& k = d->chain.plan.k1;
  const int b0 = level < 0 || level == d->L - 1 ? 0 : k.p.lv[level + 1].block_end;
  const int b1 = level < 0 ? k.blocks : k.p.lv[level].block_end;
  Event e0, e1;
  CU(e0.create(cudaEventDefault));
  CU(e1.create(cudaEventDefault));
  CU(cudaEventRecord(e0.get(), d->stream.get()));
  for (int r = 0; r < reps; ++r) {
    int rc = launch_k1(d, k, b0, b1 - b0);
    if (rc) return rc;
  }
  CU(cudaEventRecord(e1.get(), d->stream.get()));
  CU(cudaEventSynchronize(e1.get()));
  float ms = 0.f;
  CU(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
  *us = ms * 1000.f / (float)reps;
  return LM_OK;
}

// The last frame's routes as its plan recorded them, beside the shard's and the frame size's figures the prepare steps
// left; only the survivor counts of the filter are read back from the device, behind whatever the stream holds (a frame
// enqueued since the last lm_complete would be waited for and reported: see the header).
extern "C" int lm_debug_plan(lm_detector* d, int32_t* out, int64_t cap) {
  if (!d || !out) return fail(LM_E_INVALID, "null argument");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle");
  if (!d->chain.completed) return fail(LM_E_STATE, "lm_run has not been called");
  if (cap < LM_PLAN_ENTRIES) return fail(LM_E_CAPACITY, "need %d entries", LM_PLAN_ENTRIES);
  CU(cudaSetDevice(d->device));
  int queue[4], listed = 0;
  CU(cudaMemcpyAsync(queue, d->d_queue.get(), sizeof(queue), cudaMemcpyDeviceToHost, d->stream.get()));
  // the shard's own list length (off[n_work]): behind the exchange the header counts every rank's candidates
  if (d->shard_count > 0 && (size_t)d->shard_count < d->d_off.size())
    CU(cudaMemcpyAsync(&listed, d->d_off.get() + d->shard_count, sizeof(int), cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  const FramePlan& pl = d->chain.plan;
  const LevelHost& low = d->lv[d->L - 1];
  for (int i = 0; i < LM_PLAN_ENTRIES; ++i) out[i] = -1;
  out[0] = pl.k1.band ? 1 : 0;
  out[1] = pl.planes_level;
  out[2] = pl.planes_level >= 0 ? pl.k1.p.lv[pl.planes_level].pseg : 0;
  out[3] = (int32_t)pl.k1.smem;
  out[4] = low.rounds;
  out[5] = !low.d_bp.empty() ? 1 : 0;
  out[6] = d->n_items_bits;
  out[7] = d->n_items_bytes;
  if (pl.packed) {
    out[8] = pl.coarse.smem ? 1 : 0;
    out[9] = pl.coarse.split;
    out[10] = (int32_t)pl.plane_bytes;
    out[11] = d->k2_tasks;
  }
  out[12] = d->filter_ok ? 1 : 0;
  out[13] = pl.bits ? 1 : 0;
  out[14] = (int32_t)std::count_if(d->h_finfo.begin(), d->h_finfo.end(), [](const int4& f) { return (f.w & 2) != 0; });
  out[15] = pl.gated ? 1 : 0;
  // work items of the refinement kernels that ran (-1: it did not run)
  const int total = (int)std::min<int64_t>(listed, cand_cap(d));  // what the refinement kernels take (k_refine_filter_w)
  if (pl.filter) out[16] = total;
  if (pl.bits) {
    out[17] = std::min(queue[1], total);
    out[20] = d->bits_grid;
  }
  if (pl.refine) {
    if (pl.filter) out[18] = std::min(queue[pl.bits ? 2 : 1], total);
    else out[19] = total;
  }
  const LinMemLevel& kl = pl.k1.p.lv[d->L - 1];
  out[21] = (kl.bp ? 1 : 0) | (kl.lm ? 2 : 0);
  return LM_OK;
}

// The coarse scan's outputs of the last lm_run, read back from the buffers k_refine_prep and k_refine read (no launch):
// the pass masks whole, the raw scores with every position whose pass bit is clear zeroed here (the device leaves stale
// values there).
extern "C" int lm_debug_coarse(lm_detector* d, uint32_t* mask, int64_t mask_cap, uint16_t* raw, int64_t raw_cap, int32_t* dims3) {
  if (!d || !dims3 || (!mask && mask_cap > 0) || (!raw && raw_cap > 0)) return fail(LM_E_INVALID, "null argument");
  if (d->device < 0) return fail(LM_E_STATE, "host-only handle");
  if (!d->chain.completed) return fail(LM_E_STATE, "lm_run has not been called");
  const LevelHost& low = d->lv[d->L - 1];
  const int64_t n_work = d->shard_count, nwords = low.nwords, plane = low.plane;
  if ((size_t)(n_work * nwords) > d->d_mask.size() || (size_t)(n_work * plane) > d->d_raw.size())
    return fail(LM_E_STATE, "the selection or the frame size changed since the last lm_run");
  dims3[0] = (int32_t)n_work; dims3[1] = (int32_t)nwords; dims3[2] = (int32_t)plane;
  if (n_work * nwords > mask_cap || n_work * plane > raw_cap)
    return fail(LM_E_CAPACITY, "need %lld mask words and %lld raw scores", (long long)(n_work * nwords), (long long)(n_work * plane));
  if (n_work == 0) return LM_OK;
  CU(cudaSetDevice(d->device));
  CU(cudaMemcpyAsync(mask, d->d_mask.get(), sizeof(uint32_t) * (size_t)(n_work * nwords), cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaMemcpyAsync(raw, d->d_raw.get(), sizeof(uint16_t) * (size_t)(n_work * plane), cudaMemcpyDeviceToHost, d->stream.get()));
  CU(cudaStreamSynchronize(d->stream.get()));
  for (int64_t w = 0; w < n_work; ++w)
    for (int64_t j = 0; j < plane; ++j)
      if (!((mask[w * nwords + (j >> 5)] >> (j & 31)) & 1u)) raw[w * plane + j] = 0;
  return LM_OK;
}

extern "C" int lm_counters(lm_detector* d, int64_t* out8) {
  if (!d || !out8) return fail(LM_E_INVALID, "null argument");
  if (!d->chain.completed) return fail(LM_E_STATE, "lm_run has not been called");
  out8[0] = d->shard_count;
  out8[1] = hres(d)->coarse_candidates;
  out8[2] = d->alg_scan_bytes;
  out8[3] = (int64_t)(d->h_counters[0] + d->h_counters[4]) * 256;  // the reference's refinement work, whoever disposed of it
  out8[4] = hres(d)->count;
  out8[5] = (int64_t)d->h_counters[1] * 16;
  out8[6] = (int64_t)d->h_counters[4] * 256;  // ... of which: candidates the filter dropped
  out8[7] = (int64_t)d->h_counters[5] * 4;    // plane bytes the filter and k_refine_bits read (one shared counter)
  return LM_OK;
}

extern "C" int lm_set_timing(lm_detector* d, int slots) {
  if (d && d->device < 0) return fail(LM_E_STATE, "host-only handle (device -1): GPU stages are unavailable");
  if (!d) return fail(LM_E_INVALID, "null detector");
  CU(cudaSetDevice(d->device));
  CU(cudaStreamSynchronize(d->stream.get()));
  // the old events go first; timing is on only once every new one exists
  d->tev.clear();
  d->timing_runs = 0;
  d->timing = false;
  std::vector<Event> tev((size_t)std::max(slots, 0) * LM_TEV);
  for (Event& e : tev) CU(e.create(cudaEventDefault));
  d->tev.swap(tev);
  d->timing = slots > 0;
  return LM_OK;
}

extern "C" int lm_stage_times(lm_detector* d, float* out8) {
  if (!d || !out8) return fail(LM_E_INVALID, "null argument");
  if (!d->timing || d->timing_runs == 0) return fail(LM_E_STATE, "timing not enabled / no run recorded");
  CU(cudaSetDevice(d->device));
  CU(cudaStreamSynchronize(d->stream.get()));
  const int64_t slots = (int64_t)d->tev.size() / LM_TEV;
  const int64_t n = std::min<int64_t>(slots, d->timing_runs);
  // events: 0 start | 1 linear memories | 2 coarse scan | 3 offsets (+ upper-level linear memories) | 4 candidate list +
  // filter planes | 5 filter | 6 exact refinement (+ collector)
  static const int from[8] = {0, 1, 2, 3, 0, 3, 4, 5}, to[8] = {1, 2, 3, 6, 6, 4, 5, 6};
  double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int64_t k = 0; k < n; ++k) {
    const Event* ev = d->tev.data() + LM_TEV * k;
    for (int i = 0; i < 8; ++i) {
      float ms;
      CU(cudaEventElapsedTime(&ms, ev[from[i]].get(), ev[to[i]].get()));
      acc[i] += ms * 1000.0;
    }
  }
  for (int i = 0; i < 8; ++i) out8[i] = (float)(acc[i] / (double)n);
  return LM_OK;
}
