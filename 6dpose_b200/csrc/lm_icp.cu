// lm_icp.cu -- poseRefine (point-to-plane ICP pose refinement) for sm_90a + its C-ABI.
//
// Reference being replaced: poseRefine::process, linemodLevelup/linemodLevelup.cpp:27-155 of
// meiqua/6DPose @ 619be57 ("LL.cpp"), and the Open3D calls it makes (Open3D is external and unpinned
// in the reference -- oracle/icp_oracle.py documents the restated semantics; PARITY UNPINNED).
//   k_pose_cloud, a CUB segmented sort, k_pose_voxel
//                         <- mask dilation + bounding box, cloud construction, voxel down-sampling
//                            (LL.cpp:34-109; PointCloud::VoxelDownSample)
//   k_icp_normals        <- PointCloud::EstimateNormals, KNN = 30 (LL.cpp:127)
//   k_icp_point_to_plane  <- RegistrationICP + TransformationEstimationPointToPlane (LL.cpp:128-130):
//                            nearest-neighbour correspondence search fused with the 6x6 J^T J / J^T r
//                            accumulation, the 6x6 solve and the convergence test; every iteration of
//                            one hypothesis runs inside one CTA, one launch for a batch of hypotheses
//   k_icp_point_to_point  <- RegistrationICP + TransformationEstimationPointToPoint (LL.cpp:131-135, the branch the
//                            reference takes without USE_OPEN3D_P2PL; lm_icp_set_estimation / lm_set_pose_estimation):
//                            the same loop with a closed-form rigid fit (Umeyama) per pass, and no normals
// All arithmetic is double, as in Open3D/Eigen.  The reference's quirks are kept: the ICP target is the
// down-sampled MODEL cloud (LL.cpp:109), only the z component of the initial translation is converted
// to metres (LL.cpp:37), `residual` carries the fitness (LL.cpp:148).
//
// The pose stage (lm_pose.h, end of this file) builds the clouds and initial guesses and feeds them to the ICP kernels;
// k_pose_nms may follow.  A frame, a batch chunk and their shared forms are all one chunk to pose_chunk and to the
// kernels, told apart by data only: the survivor count on the device, an optional frame table, and the slot rule
// survivor = rank + slot * world.  lm_icp_process_batch and lm_icp_process_batch_device feed the same chunks from renders
// and a scene (staged from the host, or in the caller's device memory): k_icp_scene, k_icp_render_box and
// k_icp_render_crop build the per-hypothesis table k_pose_cloud reads (end of this file).  With verification on
// (lm_set_pose_verify, lm_icp_set_verify) k_pose_verify follows the ICP kernel of an unshared chunk, and k_pose_nms<true>
// reads it.  A track chunk (lm_track) builds its clouds with k_track_cloud from given transformations instead of
// k_pose_cloud from match positions; the rest of the chunk is the same.

#include "linemod_b200.h"
#include "lm_pose.h"
#include "lm_buffer.h"
#include "lm_depth.cuh"

#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <limits>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <vector>

int lm_fail(int code, const char* fmt, ...);  // linemod_b200.cu

#define CUI(call)                                                                                      \
  do {                                                                                                 \
    cudaError_t e_ = (call);                                                                           \
    if (e_ != cudaSuccess)                                                                             \
      return lm_fail(LM_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

#define ICP_KNN 30
#define ICP_TILE 256
#define ICP_THREADS 512
#define ICP_NACC 30  // 21 (upper J^T J) + 6 (J^T r) + squared error + correspondences + 1 spare

struct IcpJob {  // one hypothesis
  int32_t src_first, src_count;  // source cloud: range in the concatenated point array
  int32_t tgt_first, tgt_count;  // target cloud (+ normals); the reference uses the source cloud again
  double init[16];               // row-major 4x4 initial guess
};

struct IcpOut {
  double T[16];  // row-major final transformation_
  double fitness, rmse;
  int32_t iterations, pad;
};

struct PoseVerify {  // one survivor / hypothesis (lm_set_pose_verify)
  int32_t counts[6];  // n_model, outside, missing, inlier, occluded, violation
  float score;        // -1: no pose
  int32_t pad;
};

// LM_POSE_PSO's limits, settings and kernel parameters (the kernel: k_pose_pso, behind pose verification below)
#define PSO_THREADS 256
#define PSO_CHUNK 2048       // source points held in shared memory at once; larger clouds are swept in chunks
#define PSO_MAX_PARTICLES 256
#define PSO_MAX_ITERATIONS 1000
#define PSO_MAX_JOB (1ll << 40)
#define PSO_PARTICLE_BYTES (30 * 8 + 2 * 8)  // T [12], x, v, p [6] each (f64); cost, best cost (int64)

PoseSearch pose_search_default() { return PoseSearch{64, 40, 0.040, 30.0 * 0.017453292519943295, 20.0, 0ull}; }

int pose_search_make(int particles, int iterations, double dt_mm, double dr_deg, double clamp_mm, uint64_t seed, PoseSearch* out) {
  if (particles < 1 || particles > PSO_MAX_PARTICLES)
    return lm_fail(LM_E_INVALID, "pose search: %d particles, must lie in [1, %d]", particles, PSO_MAX_PARTICLES);
  if (iterations < 0 || iterations > PSO_MAX_ITERATIONS)
    return lm_fail(LM_E_INVALID, "pose search: %d iterations, must lie in [0, %d]", iterations, PSO_MAX_ITERATIONS);
  if (!(std::isfinite(dt_mm) && dt_mm >= 0.0 && dt_mm <= 10000.0))
    return lm_fail(LM_E_INVALID, "pose search: translation bound %g mm, must be finite and in [0, 10000]", dt_mm);
  if (!(std::isfinite(dr_deg) && dr_deg >= 0.0 && dr_deg <= 45.0))
    return lm_fail(LM_E_INVALID, "pose search: rotation bound %g degrees, must be finite and in [0, 45]", dr_deg);
  if (!(std::isfinite(clamp_mm) && clamp_mm >= 0.0 && clamp_mm <= 1e6))
    return lm_fail(LM_E_INVALID, "pose search: cost clamp %g mm, must be finite and in [0, 1e6]", clamp_mm);
  *out = PoseSearch{particles, iterations, dt_mm / 1000.0, dr_deg * 0.017453292519943295, clamp_mm, (unsigned long long)seed};
  return LM_OK;
}

// Words of 8 bytes of one swarm record (LM_ICP_CAPTURE_SEARCH).
static int64_t pso_record_words(const PoseSearch& s) { return 6 + s.iterations + 19 * (int64_t)s.particles; }

struct PsoParams {
  const IcpJob* jobs;         // [n] the slots' source clouds (in pts) and start poses
  const double* pts;
  IcpOut* outs;
  int32_t n;
  const uint16_t* scene;      // as PoseParams: frame f's depth at scene + f * srows * scols
  int32_t srows, scols;
  float sK[9];
  const int32_t* frame_of;    // null: one frame, intrinsics sK; else per slot its frame, intrinsics sKs + 9 * frame
  const float* sKs;
  const int32_t* frame_first; // batch: frame f's first survivor in the run (job = first + slot - frame_first[frame])
  int64_t first;              // run index of slot 0's survivor
  const int64_t* job;         // per slot its job number (lm_pose_search_points); null: as above
  PoseSearch s;
  long long* record;          // null, or the slots' swarm records, record_words apart
  int64_t record_words;
};

static int launch_pso(const PsoParams& p, cudaStream_t st);

// --------------------------------------------------------------------------------------------
// normals: covariance of the 30 nearest neighbours, eigenvector of the smallest eigenvalue
// --------------------------------------------------------------------------------------------
__device__ void smallest_eigenvector_3x3(double a00, double a01, double a02, double a11, double a12, double a22, double* n) {
  // cyclic Jacobi on the symmetric 3x3 matrix, eigenvectors accumulated in v
  double a[3][3] = {{a00, a01, a02}, {a01, a11, a12}, {a02, a12, a22}};
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 24; ++sweep) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
    if (off < 1e-300) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq;
          a[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk;
          a[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = c * vkp - s * vkq;
          v[k][q] = s * vkp + c * vkq;
        }
      }
  }
  int m = 0;
  if (a[1][1] < a[m][m]) m = 1;
  if (a[2][2] < a[m][m]) m = 2;
  const double nx = v[0][m], ny = v[1][m], nz = v[2][m];
  const double len = sqrt(nx * nx + ny * ny + nz * nz);
  if (len > 0) { n[0] = nx / len; n[1] = ny / len; n[2] = nz / len; }
  else { n[0] = 0; n[1] = 0; n[2] = 1; }
}

// The clouds come out of k_pose_voxel sorted by voxel (x major), so index distance is spatial distance along
// x: tiles are visited outwards from the CTA's own points, and a side is abandoned once the x gap alone puts every
// remaining candidate beyond the current 30th neighbour of every thread (exact: a point of voxel column a has
// x in [lo_a, lo_a + ICP_VOXEL)).  The kept set is the 30 smallest (distance, index) pairs in that order --
// the same list a scan in index order with "first seen wins" produces -- so the normals do not depend on the
// visiting order.
#define ICP_VOXEL 0.0025

__device__ __forceinline__ void knn_scan_tile(const double (*s_t)[3], int t0, int m, double px, double py, double pz,
                                              double* bd, int* bi, int& have) {
  for (int k = 0; k < m; ++k) {
    const double dx = px - s_t[k][0], dy = py - s_t[k][1], dz = pz - s_t[k][2];
    const double d2 = dx * dx + dy * dy + dz * dz;
    const int idx = t0 + k;
    if (have < ICP_KNN || d2 < bd[have - 1] || (d2 == bd[have - 1] && idx < bi[have - 1])) {
      int pos = have < ICP_KNN ? have++ : ICP_KNN - 1;
      while (pos > 0 && (bd[pos - 1] > d2 || (bd[pos - 1] == d2 && bi[pos - 1] > idx))) {
        bd[pos] = bd[pos - 1];
        bi[pos] = bi[pos - 1];
        --pos;
      }
      bd[pos] = d2;
      bi[pos] = idx;
    }
  }
}

// knn_out (capture only, else null): ICP_KNN indices per target point, in kept order, padded with -1.
__global__ void __launch_bounds__(128) k_icp_normals(const IcpJob* __restrict__ jobs, const double* __restrict__ pts,
                                                     double* __restrict__ normals, int32_t* __restrict__ knn_out) {
  __shared__ double s_t[ICP_TILE][3];
  const IcpJob job = jobs[blockIdx.y];
  const int n = job.tgt_count;
  const double* __restrict__ P = pts + (size_t)job.tgt_first * 3;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < n;
  double px = 0, py = 0, pz = 0;
  if (live) { px = P[3 * i]; py = P[3 * i + 1]; pz = P[3 * i + 2]; }
  double bd[ICP_KNN];
  int bi[ICP_KNN];
  int have = 0;
  const int ntiles = (n + ICP_TILE - 1) / ICP_TILE;
  if (ntiles > 0) {
    const int center = min((int)((blockIdx.x * blockDim.x + blockDim.x / 2) / ICP_TILE), ntiles - 1);
    int lo = center - 1, hi = center + 1;
    bool more_lo = lo >= 0, more_hi = hi < ntiles;
    int tile = center;
    for (;;) {
      const int t0 = tile * ICP_TILE;
      __syncthreads();
      for (int k = threadIdx.x; k < ICP_TILE * 3; k += blockDim.x) {
        const int j = t0 + k / 3;
        (&s_t[0][0])[k] = j < n ? P[(size_t)3 * t0 + k] : 0.0;
      }
      __syncthreads();
      if (live) knn_scan_tile(s_t, t0, min(ICP_TILE, n - t0), px, py, pz, bd, bi, have);
      // next tile: alternate sides while they are worth visiting (block-uniform decisions)
      bool picked = false;
      for (int side = 0; side < 2 && !picked; ++side) {
        const bool up = ((tile >= center) == (side == 0)) ? false : true;  // prefer the side not just visited
        if (up && more_hi) {
          const double gap = P[(size_t)3 * hi * ICP_TILE] - ICP_VOXEL - px;  // every x beyond is > this
          const bool useless = !live || (have == ICP_KNN && gap > 0.0 && gap * gap > bd[ICP_KNN - 1]);
          if (__syncthreads_and(useless)) more_hi = false;
          else { tile = hi++; more_hi = hi < ntiles; picked = true; }
        } else if (!up && more_lo) {
          const int last = min((lo + 1) * ICP_TILE, n) - 1;
          const double gap = px - (P[(size_t)3 * last] + ICP_VOXEL);  // every x before is < that
          const bool useless = !live || (have == ICP_KNN && gap > 0.0 && gap * gap > bd[ICP_KNN - 1]);
          if (__syncthreads_and(useless)) more_lo = false;
          else { tile = lo--; more_lo = lo >= 0; picked = true; }
        }
      }
      if (!picked) break;
    }
  }
  if (!live) return;
  if (knn_out) {
    int32_t* ko = knn_out + ((size_t)job.tgt_first + i) * ICP_KNN;
    for (int k = 0; k < ICP_KNN; ++k) ko[k] = k < have ? bi[k] : -1;
  }
  double* out = normals + ((size_t)job.tgt_first + i) * 3;
  if (have < 3) { out[0] = 0; out[1] = 0; out[2] = 1; return; }
  // cumulants exactly as Open3D's ComputeNormal: E[x], E[x x^T], covariance = E[x x^T] - E[x] E[x]^T
  double c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int k = 0; k < have; ++k) {
    const double x = P[3 * bi[k]], y = P[3 * bi[k] + 1], z = P[3 * bi[k] + 2];
    c[0] += x; c[1] += y; c[2] += z;
    c[3] += x * x; c[4] += x * y; c[5] += x * z; c[6] += y * y; c[7] += y * z; c[8] += z * z;
  }
  for (int k = 0; k < 9; ++k) c[k] /= (double)have;
  smallest_eigenvector_3x3(c[3] - c[0] * c[0], c[4] - c[0] * c[1], c[5] - c[0] * c[2], c[6] - c[1] * c[1], c[7] - c[1] * c[2],
                           c[8] - c[2] * c[2], out);
}

// --------------------------------------------------------------------------------------------
// ICP: all iterations of one hypothesis inside one CTA
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// Solve the symmetric 6x6 system A x = b (Gaussian elimination with partial pivoting; Open3D uses
// Eigen's LDLT, same solution to rounding).  A singular system gives x = 0 (identity update).
__device__ void solve6(double A[6][6], double b[6], double x[6]) {
  bool singular = false;
  for (int k = 0; k < 6; ++k) {
    int m = k;
    for (int i = k + 1; i < 6; ++i)
      if (fabs(A[i][k]) > fabs(A[m][k])) m = i;
    if (!(fabs(A[m][k]) > 0.0)) { singular = true; break; }
    if (m != k) {
      for (int j = 0; j < 6; ++j) { const double t = A[k][j]; A[k][j] = A[m][j]; A[m][j] = t; }
      const double t = b[k]; b[k] = b[m]; b[m] = t;
    }
    for (int i = k + 1; i < 6; ++i) {
      const double f = A[i][k] / A[k][k];
      for (int j = k; j < 6; ++j) A[i][j] -= f * A[k][j];
      b[i] -= f * b[k];
    }
  }
  if (!singular)
    for (int i = 5; i >= 0; --i) {
      double s = b[i];
      for (int j = i + 1; j < 6; ++j) s -= A[i][j] * x[j];
      x[i] = s / A[i][i];
    }
  bool ok = !singular;
  for (int i = 0; i < 6 && ok; ++i) ok = isfinite(x[i]);
  if (!ok)
    for (int i = 0; i < 6; ++i) x[i] = 0.0;
}

// ---- the pose stage shared over the ranks of the peer exchange (lm_pose.h, PoseShare) ----
// Pose area of every rank's exchange buffer: [2 slots][POSE_SHARE_SLOTS] entries indexed by survivor, then
// [2][LM_MAX_PEERS] int32 pose flags (slot, publishing rank) and an int32 ticket, then [2 slots][POSE_SHARE_SLOTS]
// window records that only track chunks use.  One pose exchange (a shared frame, one chunk of a shared batch or of a
// shared track run) uses slot seq & 1, seq the exchange's number on the pose counter, which every rank
// advances once per exchange.  Two slots suffice: a rank stores the entries of exchange e only behind its collector of
// e - 1, which waited for every peer's flag of e - 1, and each peer raised that flag on its stream behind its own
// collector of e - 2, the last reader of the slot.
#define POSE_SHARE_SLOTS 1024  // == LM_POST_MAX, the most survivors k_post_nms writes
#define POSE_COLLECT_THREADS 256

struct PoseShareEntry {  // one survivor: all that pose_stage_finish and k_pose_nms read of it
  IcpOut out;
  int32_t posed;         // k_pose_cloud's verdict
  int32_t err;           // the owner's cloud-overflow flag (the stage's error is the OR over all ranks)
  PoseVerify ver;        // the owner's verification (k_pose_verify<true>); zero when the stage does not verify
};
static_assert(sizeof(PoseShareEntry) == 192 && sizeof(PoseShareEntry) % 16 == 0, "pose area entry layout");

#define POSE_SHARE_FLAGS ((size_t)2 * POSE_SHARE_SLOTS * sizeof(PoseShareEntry))  // byte offset of the flags in the area
// byte offset of a track chunk's window records, [2 slots][POSE_SHARE_SLOTS] TrackRec indexed by object, behind the ticket
#define POSE_SHARE_TRACK (POSE_SHARE_FLAGS + sizeof(int32_t) * (2 * LM_MAX_PEERS + 4))

struct TrackRec {  // one tracked object's window (x, y, w, h: clipped, with the margin), projected box (unclipped) and status
  int32_t window[4], box[4];
  int32_t status, pad;
};
static_assert(sizeof(TrackRec) % 8 == 0 && POSE_SHARE_TRACK % 8 == 0, "pose area track record layout");

size_t pose_share_area_bytes() { return POSE_SHARE_TRACK + (size_t)2 * POSE_SHARE_SLOTS * sizeof(TrackRec); }

struct PoseShareDev {
  uint8_t* area[LM_MAX_PEERS];  // every rank's pose area
  int32_t world, rank, seq;
  const int32_t* counts;        // [0] survivors written by k_post_nms (a batch or track chunk: the chunk's size)
  const uint8_t* posed;         // per slot of this rank (k_pose_cloud_share)
  int32_t* status;              // [0] cloud overflow (the OR over the ranks after k_pose_collect), [1] 1: a peer did not
                                // publish in time, [2] entries this rank published
  unsigned long long timeout_ns;
  int* abort_flag;
  TrackRec* rec;                // a track chunk's window records by object (k_track_cloud writes this rank's objects',
                                // k_pose_collect every object's); null for a survivor chunk
};

// Thread 0 of the CTA of slot blockIdx.x, after its last pass (the ICP kernel's SHARE instantiation, or k_pose_verify's
// behind the unshared ICP kernel when the stage verifies): the entry of its survivor (and a track chunk's window record)
// into the same place of every rank's pose area, then the ticket; the last CTA raises this rank's pose flag everywhere.
// The ticket counts CTAs in its low 16 bits and published entries above them.
__device__ __forceinline__ void pose_share_publish(const PoseShareDev& sh, const IcpOut& o, const PoseVerify& v) {
  const int i = sh.rank + (int)blockIdx.x * sh.world;  // survivor of this slot
  const bool mine = i < sh.counts[0];
  const int slot = sh.seq & 1;
  if (mine) {
    PoseShareEntry e;
    e.out = o;
    e.posed = sh.posed[blockIdx.x];
    e.err = sh.status[0];
    e.ver = v;
    const size_t at = ((size_t)slot * POSE_SHARE_SLOTS + i) * sizeof(PoseShareEntry);
    for (int q = 0; q < sh.world; ++q) *reinterpret_cast<PoseShareEntry*>(sh.area[q] + at) = e;
    if (sh.rec) {
      const TrackRec r = sh.rec[i];
      const size_t rat = POSE_SHARE_TRACK + ((size_t)slot * POSE_SHARE_SLOTS + i) * sizeof(TrackRec);
      for (int q = 0; q < sh.world; ++q) *reinterpret_cast<TrackRec*>(sh.area[q] + rat) = r;
    }
  }
  __threadfence_system();  // release: the entries before the ticket
  unsigned* ticket = reinterpret_cast<unsigned*>(sh.area[sh.rank] + POSE_SHARE_FLAGS) + 2 * LM_MAX_PEERS;
  const unsigned old = atomicAdd(ticket, 1u + (mine ? 1u << 16 : 0u));
  if ((old & 0xFFFFu) != gridDim.x - 1) return;
  *ticket = 0;
  sh.status[2] = (int32_t)(old >> 16) + (mine ? 1 : 0);
  __threadfence_system();
  for (int q = 0; q < sh.world; ++q)
    reinterpret_cast<volatile int32_t*>(sh.area[q] + POSE_SHARE_FLAGS)[slot * LM_MAX_PEERS + sh.rank] = sh.seq;
}

// ---- the estimation step of RegistrationICP: one class per TransformationEstimation ----
// Each keeps NACC sums per thread, of which [ERR] is the squared distance and [CNT] the number of the correspondences.
// add() takes one correspondence (p the transformed source point, v its target point, index bj); update() turns the
// block's totals into the 3x4 update matrix (thread 0).

// TransformationEstimationPointToPlane (LL.cpp:128-130): J^T J and J^T r of r = (p - q) . n_q, the 6x6 solve, and
// TransformVector6dToMatrix4d of the solution.
struct IcpPointToPlane {
  static constexpr int NACC = ICP_NACC, ERR = 27, CNT = 28;
  const double* __restrict__ Nm;  // target normals (k_icp_normals)
  __device__ __forceinline__ IcpPointToPlane(const IcpJob& job, const double*, const double* normals)
      : Nm(normals + (size_t)job.tgt_first * 3) {}
  __device__ __forceinline__ void add(double* acc, double px, double py, double pz, double vx, double vy, double vz, int bj,
                                      double best) const {
    const double nx = Nm[3 * bj], ny = Nm[3 * bj + 1], nz = Nm[3 * bj + 2];
    const double r = (px - vx) * nx + (py - vy) * ny + (pz - vz) * nz;
    const double J[6] = {py * nz - pz * ny, pz * nx - px * nz, px * ny - py * nx, nx, ny, nz};
    int q = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = a; b < 6; ++b) acc[q++] += J[a] * J[b];
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] += J[a] * r;
    acc[27] += best;
    acc[28] += 1.0;
  }
  __device__ __forceinline__ void update(const double* tot, double* U) const {
    double A[6][6], b[6], x[6] = {0, 0, 0, 0, 0, 0};
    int q = 0;
    for (int a = 0; a < 6; ++a)
      for (int c = a; c < 6; ++c) { A[a][c] = tot[q]; A[c][a] = tot[q]; ++q; }
    for (int a = 0; a < 6; ++a) b[a] = -tot[21 + a];
    solve6(A, b, x);
    // TransformVector6dToMatrix4d: Rz(x2) Ry(x1) Rx(x0), translation x3..5
    const double cx = cos(x[0]), sx = sin(x[0]), cy = cos(x[1]), sy = sin(x[1]), cz = cos(x[2]), sz = sin(x[2]);
    U[0] = cz * cy; U[1] = cz * sy * sx - sz * cx; U[2] = cz * sy * cx + sz * sx; U[3] = x[3];
    U[4] = sz * cy; U[5] = sz * sy * sx + cz * cx; U[6] = sz * sy * cx - cz * sx; U[7] = x[4];
    U[8] = -sy;     U[9] = cy * sx;                U[10] = cy * cx;               U[11] = x[5];
  }
};

// The rotation of Eigen's umeyama(src, dst, false) from sig = (1/n) sum (q - qbar)(p - pbar)^T: sig = U diag(d) V^T
// (one-sided Jacobi: plane rotations accumulated into V orthogonalise the columns of sig, d descending), then
// R = U S V^T with S = diag(1, 1, -1) when det U det V < 0.  U is completed to a right-handed orthonormal basis, which
// leaves R unchanged where sig has full rank (the sign of U's last column and S flip together) and makes it one of the
// optimal proper rotations where it has not (one pair: sig = 0 and R = I exactly; two or collinear pairs: rank 1).
__device__ void umeyama_rotation(const double sig[3][3], double R[3][3]) {
  double a[3][3], v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) a[r][c] = sig[r][c];
  for (int sweep = 0; sweep < 32; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double al = 0, be = 0, ga = 0;
        for (int k = 0; k < 3; ++k) { al += a[k][p] * a[k][p]; be += a[k][q] * a[k][q]; ga += a[k][p] * a[k][q]; }
        if (!(fabs(ga) > 1e-15 * sqrt(al) * sqrt(be))) continue;  // columns p, q orthogonal to rounding (or NaN)
        const double zeta = (be - al) / (2.0 * ga);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int k = 0; k < 3; ++k) {
          const double ap = a[k][p], aq = a[k][q];
          a[k][p] = c * ap - s * aq;
          a[k][q] = s * ap + c * aq;
          const double vp = v[k][p], vq = v[k][q];
          v[k][p] = c * vp - s * vq;
          v[k][q] = s * vp + c * vq;
        }
        rotated = true;
      }
    if (!rotated) break;
  }
  double d[3];
  for (int c = 0; c < 3; ++c) d[c] = sqrt(a[0][c] * a[0][c] + a[1][c] * a[1][c] + a[2][c] * a[2][c]);
  int o[3] = {0, 1, 2};  // columns by singular value, descending
  if (d[o[1]] > d[o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
  if (d[o[2]] > d[o[1]]) { const int t = o[1]; o[1] = o[2]; o[2] = t; }
  if (d[o[1]] > d[o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r][c] = r == c ? 1.0 : 0.0;
  const double d1 = d[o[0]];
  if (!(d1 > 0.0)) return;  // no spread (one pair), or a NaN
  double u[3][3];           // u[j]: column j of U
  for (int k = 0; k < 3; ++k) u[0][k] = a[k][o[0]] / d1;
  double w[3], dot = 0;
  for (int k = 0; k < 3; ++k) dot += a[k][o[1]] * u[0][k];
  for (int k = 0; k < 3; ++k) w[k] = a[k][o[1]] - dot * u[0][k];
  double nw = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (!(nw > 1e-13 * d1)) {  // rank 1: any unit vector orthogonal to u0, from the axis u0 is least aligned with
    int m = 0;
    if (fabs(u[0][1]) < fabs(u[0][m])) m = 1;
    if (fabs(u[0][2]) < fabs(u[0][m])) m = 2;
    for (int k = 0; k < 3; ++k) w[k] = (k == m ? 1.0 : 0.0) - u[0][m] * u[0][k];
    nw = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  }
  for (int k = 0; k < 3; ++k) u[1][k] = w[k] / nw;
  u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
  u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
  u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  double vc[3][3];  // vc[j]: column o[j] of V
  for (int j = 0; j < 3; ++j)
    for (int k = 0; k < 3; ++k) vc[j][k] = v[k][o[j]];
  const double det_v = vc[0][0] * (vc[1][1] * vc[2][2] - vc[1][2] * vc[2][1]) - vc[0][1] * (vc[1][0] * vc[2][2] - vc[1][2] * vc[2][0]) +
                       vc[0][2] * (vc[1][0] * vc[2][1] - vc[1][1] * vc[2][0]);
  const double s3 = det_v < 0 ? -1.0 : 1.0;  // det U = +1
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r][c] = u[0][r] * vc[0][c] + u[1][r] * vc[1][c] + s3 * u[2][r] * vc[2][c];
}

// TransformationEstimationPointToPoint with with_scaling = false (the reference's other branch, LL.cpp:131-135) [3p, from
// memory of Open3D 0.8/0.9 and Eigen 3.3; restated in tests/icp_p2p_oracle.py]: Eigen's umeyama over the correspondences,
// R as umeyama_rotation and t = qbar - R pbar; no correspondence gives the identity.
// The sums are taken relative to a reference point c near every pair (the target's middle point in x order, the same on
// every pass), so sig = S_qp / n - (S_q / n)(S_p / n)^T does not cancel the ~1 m depth of the clouds away.
struct IcpPointToPoint {
  static constexpr int NACC = 17, ERR = 15, CNT = 16;  // [0..2] sum p - c, [3..5] sum q - c, [6..14] sum (q - c)(p - c)^T
  double c0, c1, c2;
  __device__ __forceinline__ IcpPointToPoint(const IcpJob& job, const double* pts, const double*) : c0(0), c1(0), c2(0) {
    if (job.tgt_count > 0) {
      const double* Q = pts + ((size_t)job.tgt_first + job.tgt_count / 2) * 3;
      c0 = Q[0]; c1 = Q[1]; c2 = Q[2];
    }
  }
  __device__ __forceinline__ void add(double* acc, double px, double py, double pz, double vx, double vy, double vz, int,
                                      double best) const {
    const double p[3] = {px - c0, py - c1, pz - c2}, q[3] = {vx - c0, vy - c1, vz - c2};
#pragma unroll
    for (int i = 0; i < 3; ++i) { acc[i] += p[i]; acc[3 + i] += q[i]; }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) acc[6 + 3 * i + j] += q[i] * p[j];
    acc[15] += best;
    acc[16] += 1.0;
  }
  __device__ __forceinline__ void update(const double* tot, double* U) const {
    for (int k = 0; k < 12; ++k) U[k] = (k % 5 == 0) ? 1.0 : 0.0;
    const double n = tot[CNT];
    if (!(n > 0.0)) return;
    double mp[3], mq[3], sig[3][3], R[3][3];
    for (int k = 0; k < 3; ++k) { mp[k] = __ddiv_rn(tot[k], n); mq[k] = __ddiv_rn(tot[3 + k], n); }
    // no contraction: one pair must give sig = 0 exactly
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) sig[i][j] = __dsub_rn(__ddiv_rn(tot[6 + 3 * i + j], n), __dmul_rn(mq[i], mp[j]));
    umeyama_rotation(sig, R);
    const double pb[3] = {mp[0] + c0, mp[1] + c1, mp[2] + c2}, qb[3] = {mq[0] + c0, mq[1] + c1, mq[2] + c2};
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) U[4 * r + c] = R[r][c];
      U[4 * r + 3] = qb[r] - (R[r][0] * pb[0] + R[r][1] * pb[1] + R[r][2] * pb[2]);
    }
  }
};

// RegistrationICP (Open3D 0.8/0.9) for one job per CTA, all passes in the CTA: the radius search, fitness / rmse, the
// convergence test and T = update * T; the estimation step is Est's.
// corr_out (capture only, else null): 2 slots per source point, the correspondence (-1: none) of pass 0 and of the
// latest later pass.  SHARE: the result goes to the pose areas of the exchange (pose_share_publish) instead of outs; sh
// is unused otherwise.
template <bool SHARE, class Est>
__device__ __forceinline__ void icp_registration(const IcpJob* __restrict__ jobs, const double* __restrict__ pts,
                                                 const double* __restrict__ normals, IcpOut* __restrict__ outs, double max_d2,
                                                 int max_iter, double rel_fitness, double rel_rmse, int32_t* __restrict__ corr_out,
                                                 const PoseShareDev& sh) {
  __shared__ double s_t[ICP_TILE][3];
  __shared__ double s_red[ICP_THREADS / 32][Est::NACC];
  __shared__ double s_T[16];
  __shared__ int s_stop;
  const IcpJob job = jobs[blockIdx.x];
  const int n = job.src_count, nt = job.tgt_count;
  const double* __restrict__ P = pts + (size_t)job.src_first * 3;  // source cloud
  const double* __restrict__ Q = pts + (size_t)job.tgt_first * 3;  // target cloud (== source in the reference, LL.cpp:108-109)
  const Est est(job, pts, normals);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < 16) s_T[threadIdx.x] = job.init[threadIdx.x];
  if (threadIdx.x == 0) s_stop = 0;
  __syncthreads();

  double fit_prev = 0, rmse_prev = 0, fitness = 0, rmse = 0;
  int it = 0;
  for (int pass = 0;; ++pass) {
    const double r00 = s_T[0], r01 = s_T[1], r02 = s_T[2], tx = s_T[3];
    const double r10 = s_T[4], r11 = s_T[5], r12 = s_T[6], ty = s_T[7];
    const double r20 = s_T[8], r21 = s_T[9], r22 = s_T[10], tz = s_T[11];
    double acc[Est::NACC];
#pragma unroll
    for (int k = 0; k < Est::NACC; ++k) acc[k] = 0.0;

    for (int c0 = 0; c0 < n; c0 += ICP_THREADS) {
      const int i = c0 + threadIdx.x;
      const bool live = i < n;
      double px = 0, py = 0, pz = 0;
      if (live) {
        const double x = P[3 * i], y = P[3 * i + 1], z = P[3 * i + 2];
        px = r00 * x + r01 * y + r02 * z + tx;
        py = r10 * x + r11 * y + r12 * z + ty;
        pz = r20 * x + r21 * y + r22 * z + tz;
      }
      double best = max_d2;  // radius search, strict <
      int bj = -1;
      for (int t0 = 0; t0 < nt; t0 += ICP_TILE) {
        // The target cloud is sorted by voxel, x major (k_pose_voxel), so a tile covers the x range
        // [x(first) - voxel, x(last) + voxel]: a tile whose range is farther from EVERY source point of this pass than its
        // best squared distance so far cannot change any correspondence (strict <) and is skipped -- exact, and most
        // tiles go: the search radius is 1 cm, the cloud is ~10 cm wide
        {
          const int last = min(t0 + ICP_TILE, nt) - 1;
          const double tmin = Q[(size_t)3 * t0] - ICP_VOXEL, tmax = Q[(size_t)3 * last] + ICP_VOXEL;
          const double gap = !live ? 1e300 : (px < tmin ? tmin - px : (px > tmax ? px - tmax : 0.0));
          if (__syncthreads_and(!live || gap * gap >= best)) continue;
        }
        __syncthreads();
        for (int k = threadIdx.x; k < ICP_TILE * 3; k += blockDim.x) (&s_t[0][0])[k] = (t0 + k / 3) < nt ? Q[(size_t)3 * t0 + k] : 0.0;
        __syncthreads();
        if (live) {
          const int m = min(ICP_TILE, nt - t0);
#pragma unroll 4
          for (int k = 0; k < m; ++k) {
            const double dx = px - s_t[k][0], dy = py - s_t[k][1], dz = pz - s_t[k][2];
            const double d2 = dx * dx + dy * dy + dz * dz;
            if (d2 < best) { best = d2; bj = t0 + k; }
          }
        }
      }
      if (corr_out && live) corr_out[((size_t)job.src_first + i) * 2 + (pass > 0)] = bj;
      if (bj >= 0) {
        const double vx = Q[3 * bj], vy = Q[3 * bj + 1], vz = Q[3 * bj + 2];
        est.add(acc, px, py, pz, vx, vy, vz, bj, best);
      }
    }
    // block reduction of the sums
#pragma unroll
    for (int k = 0; k < Est::NACC; ++k) acc[k] = warp_sum(acc[k]);
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < Est::NACC; ++k) s_red[warp][k] = acc[k];
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot[Est::NACC];
      for (int k = 0; k < Est::NACC; ++k) {
        double s = 0;
        for (int w = 0; w < ICP_THREADS / 32; ++w) s += s_red[w][k];
        tot[k] = s;
      }
      const double ncorr = tot[Est::CNT];
      fitness = n > 0 ? ncorr / (double)n : 0.0;
      rmse = ncorr > 0 ? sqrt(tot[Est::ERR] / ncorr) : 0.0;
      bool stop = false;
      if (pass > 0 && fabs(fit_prev - fitness) < rel_fitness && fabs(rmse_prev - rmse) < rel_rmse) stop = true;
      if (pass >= max_iter) stop = true;
      if (!stop) {
        double U[12];
        est.update(tot, U);
        // T = update * T
        double Tn[12];
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 4; ++c)
            Tn[4 * r + c] = U[4 * r] * s_T[c] + U[4 * r + 1] * s_T[4 + c] + U[4 * r + 2] * s_T[8 + c] + (c == 3 ? U[4 * r + 3] : 0.0);
        for (int k = 0; k < 12; ++k) s_T[k] = Tn[k];
        fit_prev = fitness;
        rmse_prev = rmse;
        it = pass + 1;
      }
      s_stop = stop ? 1 : 0;
    }
    __syncthreads();
    if (s_stop) break;
  }
  if (threadIdx.x == 0) {
    IcpOut o;
    for (int k = 0; k < 16; ++k) o.T[k] = s_T[k];
    o.fitness = fitness; o.rmse = rmse; o.iterations = it; o.pad = 0;
    if (SHARE) pose_share_publish(sh, o, PoseVerify());
    else outs[blockIdx.x] = o;
  }
}

template <bool SHARE>
__global__ void __launch_bounds__(ICP_THREADS) k_icp_point_to_plane(const IcpJob* __restrict__ jobs, const double* __restrict__ pts,
                                                                    const double* __restrict__ normals, IcpOut* __restrict__ outs,
                                                                    double max_d2, int max_iter, double rel_fitness, double rel_rmse,
                                                                    int32_t* __restrict__ corr_out, PoseShareDev sh) {
  icp_registration<SHARE, IcpPointToPlane>(jobs, pts, normals, outs, max_d2, max_iter, rel_fitness, rel_rmse, corr_out, sh);
}

// No normals: k_icp_normals does not run before it (the reference's point-to-point branch calls no EstimateNormals).
template <bool SHARE>
__global__ void __launch_bounds__(ICP_THREADS) k_icp_point_to_point(const IcpJob* __restrict__ jobs, const double* __restrict__ pts,
                                                                    IcpOut* __restrict__ outs, double max_d2, int max_iter,
                                                                    double rel_fitness, double rel_rmse, int32_t* __restrict__ corr_out,
                                                                    PoseShareDev sh) {
  icp_registration<SHARE, IcpPointToPoint>(jobs, pts, nullptr, outs, max_d2, max_iter, rel_fitness, rel_rmse, corr_out, sh);
}

// The ICP kernel of estimation est over n jobs (point-to-plane reads the normals k_icp_normals left in nrm).
template <bool SHARE>
static void launch_icp(int est, unsigned n, cudaStream_t st, const IcpJob* jobs, const double* pts, const double* nrm, IcpOut* outs,
                       int max_iter, int32_t* corr_out, const PoseShareDev& sd) {
  if (est == LM_ICP_POINT_TO_POINT)
    k_icp_point_to_point<SHARE><<<n, ICP_THREADS, 0, st>>>(jobs, pts, outs, 0.01 * 0.01, max_iter, 1e-6, 1e-6, corr_out, sd);
  else
    k_icp_point_to_plane<SHARE><<<n, ICP_THREADS, 0, st>>>(jobs, pts, nrm, outs, 0.01 * 0.01, max_iter, 1e-6, 1e-6, corr_out, sd);
}

// One CTA behind the ICP kernel's SHARE instantiation on each rank's stream: waits (acquire) until every rank's pose flag of the
// frame has arrived in this rank's pose area, then copies the entries, in survivor order, into the stage's outs / posed.
// ver (a verifying stage, else null): the entries' verification, in the same order; a track chunk's window records go
// to sh.rec in object order.
__global__ void __launch_bounds__(POSE_COLLECT_THREADS) k_pose_collect(PoseShareDev sh, IcpOut* __restrict__ outs,
                                                                       uint8_t* __restrict__ posed, PoseVerify* __restrict__ ver) {
  __shared__ int s_late;
  const int tid = threadIdx.x;
  if (tid == 0) s_late = 0;
  __syncthreads();
  const int slot = sh.seq & 1;
  const uint8_t* mine = sh.area[sh.rank];
  if (tid < sh.world) {
    const volatile int32_t* flag = reinterpret_cast<const volatile int32_t*>(mine + POSE_SHARE_FLAGS) + slot * LM_MAX_PEERS + tid;
    const volatile int* abort_flag = sh.abort_flag;
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while ((int32_t)(*flag - sh.seq) < 0) {
      if (*abort_flag) { s_late = 1; break; }
      __nanosleep(200);
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > sh.timeout_ns) {  // a peer does not run the pose stage of this frame (or died)
        atomicExch(sh.abort_flag, 1);
        s_late = 1;
        break;
      }
    }
    __threadfence_system();  // acquire: the entries were fenced before the flag
  }
  __syncthreads();
  const int late = s_late;
  const int n = late ? 0 : min(sh.counts[0], POSE_SHARE_SLOTS);
  int err = 0;
  for (int i = tid; i < n; i += POSE_COLLECT_THREADS) {
    union {
      int4 v[sizeof(PoseShareEntry) / 16];
      PoseShareEntry e;
    } u;
    const int4* src = reinterpret_cast<const int4*>(mine + ((size_t)slot * POSE_SHARE_SLOTS + i) * sizeof(PoseShareEntry));
#pragma unroll
    for (int k = 0; k < (int)(sizeof(PoseShareEntry) / 16); ++k) u.v[k] = __ldcv(src + k);  // peers wrote them
    outs[i] = u.e.out;
    posed[i] = (uint8_t)u.e.posed;
    if (ver) ver[i] = u.e.ver;
    err |= u.e.err;
    if (sh.rec) {
      union {
        int2 v[sizeof(TrackRec) / 8];
        TrackRec r;
      } t;
      const int2* rsrc = reinterpret_cast<const int2*>(mine + POSE_SHARE_TRACK + ((size_t)slot * POSE_SHARE_SLOTS + i) * sizeof(TrackRec));
#pragma unroll
      for (int k = 0; k < (int)(sizeof(TrackRec) / 8); ++k) t.v[k] = __ldcv(rsrc + k);
      sh.rec[i] = t.r;
    }
  }
  err = __syncthreads_or(err);
  if (tid == 0) {
    sh.status[0] = err;
    sh.status[1] = late;
  }
}

// --------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------
struct IcpDevice;                    // the calls' buffers (end of this file)
static IcpDevice* icp_device_new();
static void icp_device_free(IcpDevice* d);

// lm_icp_set_capture: the kernels' intermediate results of a call, per point in the order of pts
struct IcpCapture {
  int estimation = LM_ICP_POINT_TO_PLANE;  // point-to-point computes no normals and no neighbour lists
  std::vector<IcpJob> jobs;
  std::vector<int> job_of;  // per hypothesis, -1: early return
  std::vector<IcpOut> outs;
  std::vector<double> pts, nrm;
  std::vector<int32_t> knn, corr;
  std::vector<long long> record;  // LM_POSE_PSO: the jobs' swarm records, record_words apart
  int64_t record_words = 0;
};

struct lm_icp {
  int device = 0;
  Stream stream;  // streams and events first: they outlive the buffers
  Event ev0, ev1;
  Event ev_in, ev_out;  // lm_icp_process_batch_device: the caller's stream -> the call -> the caller's stream
  int64_t launches = 0;
  bool use_scene_cloud = false;  // non-reference option: register against the scene cloud
  int estimation = LM_ICP_POINT_TO_PLANE;
  PoseSearch search = pose_search_default();  // lm_icp_set_pose_search (LM_POSE_PSO)
  int last_points = 0, last_iterations = 0;
  double last_rmse = 0;
  float last_kernel_us = 0;
  bool capture = false;
  IcpCapture cap;  // the last call's
  IcpDevice* dev = nullptr;  // its stage holds the verification of the last call's hypotheses (pose_stage_verify)
  bool verify = false;  // lm_icp_set_verify
  double verify_mm = 10.0;
};

extern "C" int lm_icp_create(int device, lm_icp** out) {
  if (!out) return lm_fail(LM_E_INVALID, "out is null");
  const int rc = open_device(device);
  if (rc) return rc;
  std::unique_ptr<lm_icp> h(new lm_icp());
  h->device = device;
  CUI(h->stream.create(cudaStreamNonBlocking));
  CUI(h->ev0.create(cudaEventDefault));
  CUI(h->ev1.create(cudaEventDefault));
  CUI(h->ev_in.create(cudaEventDisableTiming));
  CUI(h->ev_out.create(cudaEventDisableTiming));
  h->dev = icp_device_new();
  *out = h.release();
  return LM_OK;
}

extern "C" void lm_icp_destroy(lm_icp* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream.get());
  icp_device_free(h->dev);
  delete h;
}

namespace {

// init_base = [R | t] with only t.z converted to metres (LL.cpp:34-38)
void init_base(const float* R, const float* t, float* base) {
  for (int i = 0; i < 16; ++i) base[i] = 0.f;
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) base[4 * r + k] = R[3 * r + k];
    base[4 * r + 3] = t[r];
  }
  base[4 * 2 + 3] /= 1000.0f;
  base[15] = 1.f;
}

// result = transformation_ * init_base (LL.cpp:146); R_refined, t_refined * 1000 (LL.cpp:153-154)
void compose(const double* T, const float* base, double* R_out, double* t_out) {
  double res[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += T[4 * r + k] * (double)base[4 * k + c];
      res[4 * r + c] = s;
    }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) R_out[3 * r + c] = res[4 * r + c];
    t_out[r] = res[4 * r + 3] * 1000.0;
  }
}

// ICP output o against the render made with R, t, as lm_icp_process returns it: T * init_base and the fitness.
void render_pose(const IcpOut& o, const float* R, const float* t, double* R_out, double* t_out, float* residual) {
  float base[16];
  init_base(R, t, base);
  compose(o.T, base, R_out, t_out);
  *residual = (float)o.fitness;
}

}  // namespace

// dilate(modelDepth > 0, 9x9) + boundingRect (LL.cpp:43-50) from the extent [x0, x1] x [y0, y1] of the non-zero pixels
// (x1 < 0: none): that extent grown by 4, clipped to the image, as (x, y, w, h); no pixel gives the empty box
__host__ __device__ __forceinline__ void grow_box(int x0, int y0, int x1, int y1, int mrows, int mcols, int* box) {
  const int half = 4;
  box[0] = box[1] = box[2] = box[3] = 0;
  if (x1 >= 0) {
    box[0] = max(x0 - half, 0); box[1] = max(y0 - half, 0);
    box[2] = min(x1 + half, mcols - 1) - box[0] + 1;
    box[3] = min(y1 + half, mrows - 1) - box[1] + 1;
  }
}

namespace {

void model_box(const uint16_t* model, int mrows, int mcols, int* box) {
  int x0 = mcols, x1 = -1, y0 = mrows, y1 = -1;
  for (int r = 0; r < mrows; ++r)
    for (int q = 0; q < mcols; ++q)
      if (model[(size_t)r * mcols + q] > 0) { x0 = std::min(x0, q); x1 = std::max(x1, q); y0 = std::min(y0, r); y1 = std::max(y1, r); }
  grow_box(x0, y0, x1, y1, mrows, mcols, box);
}

}  // namespace

extern "C" int lm_icp_process(lm_icp* h, const uint16_t* scene_depth, int srows, int scols, const uint16_t* model_depth, int mrows,
                              int mcols, const float* sceneK, const float* modelK, const float* R, const float* t, int detectX,
                              int detectY, int max_iterations, double* R_out, double* t_out, float* residual) {
  const uint16_t* models[1] = {model_depth};
  const int32_t xy[2] = {detectX, detectY};
  return lm_icp_process_batch(h, 1, scene_depth, srows, scols, models, mrows, mcols, sceneK, modelK, R, t, xy, max_iterations, R_out,
                              t_out, residual);
}

// [0] points in the down-sampled cloud, [1] ICP iterations, [2] inlier rmse (m) -- of the LAST hypothesis with a pose --
// and [3] device time of the last call in microseconds (include/linemod_b200.h).
extern "C" int lm_icp_last_stats(lm_icp* h, double* out4) {
  if (!h || !out4) return lm_fail(LM_E_INVALID, "null argument");
  out4[0] = h->last_points; out4[1] = h->last_iterations; out4[2] = h->last_rmse; out4[3] = h->last_kernel_us;
  return LM_OK;
}

extern "C" int64_t lm_icp_launch_count(lm_icp* h) { return h ? h->launches : 0; }

extern "C" int lm_icp_set_use_scene_cloud(lm_icp* h, int on) {
  if (!h) return lm_fail(LM_E_INVALID, "null handle");
  h->use_scene_cloud = on != 0;
  return LM_OK;
}

extern "C" int lm_icp_set_estimation(lm_icp* h, int estimation) {
  if (!h) return lm_fail(LM_E_INVALID, "null handle");
  const int rc = check_estimation(estimation);
  if (rc) return rc;
  h->estimation = estimation;
  return LM_OK;
}

extern "C" int lm_icp_set_pose_search(lm_icp* h, int particles, int iterations, double dt_mm, double dr_deg, double clamp_mm, uint64_t seed) {
  if (!h) return lm_fail(LM_E_INVALID, "null handle");
  return pose_search_make(particles, iterations, dt_mm, dr_deg, clamp_mm, seed, &h->search);
}

extern "C" int lm_icp_set_verify(lm_icp* h, int on, double inlier_mm) {
  if (!h) return lm_fail(LM_E_INVALID, "null handle");
  const int rc = check_inlier_mm(inlier_mm);
  if (rc) return rc;
  h->verify = on != 0;
  h->verify_mm = inlier_mm;
  return LM_OK;
}

extern "C" int lm_icp_set_capture(lm_icp* h, int on) {
  if (!h) return lm_fail(LM_E_INVALID, "null handle");
  h->capture = on != 0;
  h->cap.job_of.clear();
  return LM_OK;
}

// --------------------------------------------------------------------------------------------
// pose stage on the device (lm_pose.h): clouds, initial guesses and the ICP for the NMS survivors or a call's hypotheses
// --------------------------------------------------------------------------------------------
// Exactness: every float / double operation of LL.cpp:34-109 is written with an _rn intrinsic (no FMA contraction),
// points are compacted with block scans in row-major order, the centroids are summed by one thread each in that order,
// and the voxel keys are sorted stably, so clouds and initial guesses are bit-identical to a sequential float64 build
// (tests/pose_cloud_model.py).
#define POSE_THREADS 512
#define POSE_KEY_BITS 21  // per voxel coordinate: 2^21 voxels of 2.5 mm = 5.2 km of cloud extent
#define POSE_FIRST_FETCH 16

struct PoseTpl {  // per template of the bank, registered once
  int32_t bx, by, bw, bh;  // dilated box of the render's non-zero pixels, clipped to the render
  int64_t crop;            // first pixel of the bw x bh crop in the crop pool
  float K[9];
  uint32_t anchor;         // render[rows / 2][cols / 2] (mm), usually outside the box
};

struct PoseParams {
  const lm_match* surv;
  const int32_t* counts;    // [0] survivors of the chunk
  const int32_t* class_begin;
  int32_t n_classes, n_tpl;
  const PoseTpl* tpl;
  const uint16_t* crops;
  const uint16_t* scene;
  int32_t srows, scols;
  float sK[9];
  int32_t A;          // points per cloud slot (largest crop)
  int32_t use_scene;
  double* raw;        // [2B][A][3] back-projected points: slot 2i model cloud, 2i + 1 scene cloud of survivor i
  double* cpts;       // [B][A][3] scene points that enter the scene centroid
  unsigned long long* keys;  // [2B][A] voxel keys (a, b, c) packed
  int32_t* vals;      // [2B][A] point index in the slot
  int32_t* seg_begin; // [2B]
  int32_t* seg_end;
  IcpJob* jobs;       // [B]
  int32_t* err;       // 1: a cloud spans more than 2^21 voxels along an axis
  uint8_t* posed;     // [B] 1: slot i's survivor has a template and its box fits the frame (no early return of LL.cpp:52-55)
  // null: every survivor is of one frame, depth scene and intrinsics sK.  Else survivor si belongs to frame
  // frame_of[si], whose depth is scene + frame * srows * scols and whose intrinsics are sKs + 9 * frame.
  const int32_t* frame_of;
  const float* sKs;
  int32_t rank, world;  // slot i takes survivor rank + i * world (lm_pose.h)
};

__device__ __forceinline__ double pose_backproject(int pix, float c, float f, double z) {
  return __dmul_rn((double)__fdiv_rn(__fsub_rn((float)pix, c), f), z);  // int - float -> float, / float, * double
}

__device__ __forceinline__ int pose_template(const PoseParams& p, const lm_match& m) {
  if (m.class_index < 0 || m.class_index >= p.n_classes) return -1;
  const int g = p.class_begin[m.class_index] + m.template_id;
  return (g >= 0 && g < p.n_tpl) ? g : -1;
}

// One CTA per survivor slot: slot i takes survivor si = p.rank + i * p.world, live iff si < p.counts[0] and the survivor
// has a template whose box fits the frame.  Slots that are not write empty jobs.
__global__ void __launch_bounds__(POSE_THREADS) k_pose_cloud(PoseParams p) {
  typedef cub::BlockScan<unsigned long long, POSE_THREADS> Scan;
  typedef cub::BlockReduce<double, POSE_THREADS> Reduce;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename Reduce::TempStorage reduce;
  } tmp;
  __shared__ double s_min[6], s_sum[6];
  const int i = blockIdx.x, tid = threadIdx.x;
  const size_t A = (size_t)p.A;
  const size_t sm = 2 * (size_t)i * A, ss = sm + A;  // first point of the model / scene slot
  IcpJob* job = p.jobs + i;
  lm_match m = {0, 0, 0.f, 0, 0};
  PoseTpl T;
  const int si = p.rank + i * p.world;  // survivor of this slot
  bool live = si < p.counts[0];
  const int frame = live && p.frame_of ? p.frame_of[si] : 0;
  const uint16_t* __restrict__ scene = p.scene + (size_t)frame * p.srows * p.scols;
  const float* __restrict__ fK = p.frame_of ? p.sKs + 9 * frame : nullptr;
  const float fx = fK ? fK[0] : p.sK[0], cx = fK ? fK[2] : p.sK[2], fy = fK ? fK[4] : p.sK[4], cy = fK ? fK[5] : p.sK[5];
  if (live) {
    m = p.surv[si];
    const int g = pose_template(p, m);
    live = g >= 0;
    if (live) {
      T = p.tpl[g];
      live = !(m.x + T.bw >= p.scols || m.y + T.bh >= p.srows);  // LL.cpp:52-55
    }
  }
  if (tid == 0) p.posed[i] = live ? 1 : 0;
  if (!live) {  // block-uniform
    if (tid == 0) {
      job->src_first = job->tgt_first = (int32_t)sm;
      job->src_count = job->tgt_count = 0;
      for (int k = 0; k < 16; ++k) job->init[k] = (k % 5 == 0) ? 1.0 : 0.0;
      p.seg_begin[2 * i] = p.seg_end[2 * i] = (int32_t)sm;
      p.seg_begin[2 * i + 1] = p.seg_end[2 * i + 1] = (int32_t)ss;
    }
    return;
  }
  const int bw = T.bw, npix = T.bw * T.bh, half = 4;
  const uint16_t* __restrict__ C = p.crops + T.crop;
  const double anchor = __ddiv_rn((double)T.anchor, 1000.0);
  double* __restrict__ M = p.raw + sm * 3;
  double* __restrict__ S = p.raw + ss * 3;
  double* __restrict__ Cs = p.cpts + (size_t)i * A * 3;
  const unsigned long long F = (1ull << POSE_KEY_BITS) - 1;
  // clouds (LL.cpp:57-99), row-major over the box: three compactions in one 64-bit scan (counts < 2^21 each)
  unsigned long long base = 0;
  for (int t0 = 0; t0 < npix; t0 += POSE_THREADS) {
    const int k = t0 + tid;
    bool fm = false, fs = false, fc = false;
    double mx = 0, my = 0, mz = 0, sx = 0, sy = 0, sz = 0;
    if (k < npix) {
      const int r = k / bw, q = k - r * bw;
      const uint16_t md = C[k];
      bool in = md > 0;
      // the dilated mask: every non-zero pixel lies inside the box, so the crop holds the whole 9 x 9 neighbourhood
      for (int dy = -half; dy <= half && !in; ++dy) {
        const int rr = r + dy;
        if (rr < 0 || rr >= T.bh) continue;
        for (int dx = -half; dx <= half; ++dx) {
          const int qq = q + dx;
          if (qq >= 0 && qq < bw && C[rr * bw + qq] > 0) { in = true; break; }
        }
      }
      if (in) {
        const int mr = r + T.by, mc = q + T.bx;
        int sr = r + m.y - half; if (sr < 0) sr = 0;
        int sc = q + m.x - half; if (sc < 0) sc = 0;
        if (md > 0) {
          fm = true;
          mz = __ddiv_rn((double)md, 1000.0);
          mx = pose_backproject(mc, T.K[2], T.K[0], mz);
          my = pose_backproject(mr, T.K[5], T.K[4], mz);
        }
        const uint16_t sd = scene[(size_t)sr * p.scols + sc];
        if (sd > 0) {
          sz = __ddiv_rn((double)sd, 1000.0);
          sx = pose_backproject(sc, cx, fx, sz);
          sy = pose_backproject(sr, cy, fy, sz);
          fs = p.use_scene != 0;
          fc = md > 0 && fabs(__dsub_rn(sz, anchor)) < 0.4;
        }
      }
    }
    const unsigned long long mine = (fm ? 1ull : 0ull) | (fs ? 1ull << POSE_KEY_BITS : 0ull) | (fc ? 1ull << (2 * POSE_KEY_BITS) : 0ull);
    unsigned long long excl, agg;
    Scan(tmp.scan).ExclusiveSum(mine, excl, agg);
    const unsigned long long at = base + excl;
    if (fm) { const size_t o = 3 * (at & F); M[o] = mx; M[o + 1] = my; M[o + 2] = mz; }
    if (fs) { const size_t o = 3 * ((at >> POSE_KEY_BITS) & F); S[o] = sx; S[o + 1] = sy; S[o + 2] = sz; }
    if (fc) { const size_t o = 3 * (at >> (2 * POSE_KEY_BITS)); Cs[o] = sx; Cs[o + 1] = sy; Cs[o + 2] = sz; }
    base += agg;
    __syncthreads();
  }
  const int nm = (int)(base & F), ns = (int)((base >> POSE_KEY_BITS) & F), nc = (int)(base >> (2 * POSE_KEY_BITS));
  // per-axis minima of both clouds (exact in any order)
  for (int c = 0; c < 6; ++c) {
    const double* P = c < 3 ? M : S;
    const int n = c < 3 ? nm : ns;
    double v = INFINITY;
    for (int j = tid; j < n; j += POSE_THREADS) v = fmin(v, P[3 * j + c % 3]);
    v = Reduce(tmp.reduce).Reduce(v, cub::Min());
    if (tid == 0) s_min[c] = v;
    __syncthreads();
  }
  if (tid < 6) {
    // centroids: one thread per sum, in the reference's sequential order (LL.cpp:71-104)
    const double* P = tid < 3 ? M : Cs;
    const int n = tid < 3 ? nm : nc;
    double s = 0.0;
    for (int j = 0; j < n; ++j) s = __dadd_rn(s, P[3 * j + tid % 3]);
    s_sum[tid] = s;
  } else if (tid >= 32) {
    // voxel keys floor((p - (min - v/2)) / v) of PointCloud::VoxelDownSample(0.0025), packed (a, b, c)
    for (int c2 = 0; c2 < 2; ++c2) {
      const double* P = c2 ? S : M;
      const int n = c2 ? ns : nm;
      const size_t slot = c2 ? ss : sm;
      double o[3];
      for (int c = 0; c < 3; ++c) o[c] = __dsub_rn(s_min[3 * c2 + c], 0.00125);
      for (int j = tid - 32; j < n; j += POSE_THREADS - 32) {
        unsigned long long key = 0;
        for (int c = 0; c < 3; ++c) {
          const double v = floor(__ddiv_rn(__dsub_rn(P[3 * j + c], o[c]), 0.0025));
          unsigned long long a = (unsigned long long)(long long)v;
          if (!(v >= 0.0 && v <= (double)F)) { atomicExch(p.err, 1); a = F; }
          key = (key << POSE_KEY_BITS) | a;
        }
        p.keys[slot + j] = key;
        p.vals[slot + j] = j;
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    for (int k = 0; k < 16; ++k) job->init[k] = (k % 5 == 0) ? 1.0 : 0.0;
    for (int c = 0; c < 3; ++c) {
      const double cm = __ddiv_rn(s_sum[c], (double)nm), cs = __ddiv_rn(s_sum[3 + c], (double)nc);  // 0/0 -> NaN as the reference
      job->init[4 * c + 3] = __dsub_rn(cs, cm);
    }
    job->src_first = job->tgt_first = (int32_t)sm;
    job->src_count = job->tgt_count = 0;  // k_pose_voxel sets the counts
    p.seg_begin[2 * i] = (int32_t)sm; p.seg_end[2 * i] = (int32_t)sm + nm;
    p.seg_begin[2 * i + 1] = (int32_t)ss; p.seg_end[2 * i + 1] = (int32_t)ss + ns;
  }
}

// One CTA per cloud slot: mean of every occupied voxel, summed in sorted voxel order (PointCloud::VoxelDownSample).
__global__ void __launch_bounds__(POSE_THREADS) k_pose_voxel(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals,
                                                             const int32_t* __restrict__ seg_begin, const int32_t* __restrict__ seg_end,
                                                             const double* __restrict__ raw, double* __restrict__ pts, IcpJob* jobs,
                                                             int use_scene) {
  typedef cub::BlockScan<int, POSE_THREADS> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const int s = blockIdx.x, tid = threadIdx.x;
  const int b = seg_begin[s], n = seg_end[s] - b;
  const unsigned long long* K = keys + b;
  const int32_t* V = vals + b;
  const double* P = raw + (size_t)b * 3;
  double* O = pts + (size_t)b * 3;
  int nv = 0;
  for (int t0 = 0; t0 < n; t0 += POSE_THREADS) {
    const int j = t0 + tid;
    const bool start = j < n && (j == 0 || K[j] != K[j - 1]);
    int excl, agg;
    Scan(tmp).ExclusiveSum(start ? 1 : 0, excl, agg);
    if (start) {
      double a0 = 0.0, a1 = 0.0, a2 = 0.0;
      int e = j;
      const unsigned long long key = K[j];
      for (; e < n && K[e] == key; ++e) {
        const double* q = P + 3 * (size_t)V[e];
        a0 = __dadd_rn(a0, q[0]); a1 = __dadd_rn(a1, q[1]); a2 = __dadd_rn(a2, q[2]);
      }
      const double c = (double)(e - j);
      double* o = O + 3 * (size_t)(nv + excl);
      o[0] = __ddiv_rn(a0, c); o[1] = __ddiv_rn(a1, c); o[2] = __ddiv_rn(a2, c);
    }
    nv += agg;
    __syncthreads();
  }
  if (tid == 0) {
    IcpJob* job = jobs + s / 2;
    if (s % 2 == 0) {
      job->src_first = b; job->src_count = nv;
      if (!use_scene) { job->tgt_first = b; job->tgt_count = nv; }  // the reference registers against the model cloud
    } else if (use_scene) {
      job->tgt_first = b; job->tgt_count = nv;
    }
  }
}

// --------------------------------------------------------------------------------------------
// pose verification (include/linemod_b200.h, lm_set_pose_verify): the raw model cloud moved by the ICP's T, projected
// into the scene depth
// --------------------------------------------------------------------------------------------
#define VERIFY_THREADS 256
enum { VERIFY_OUTSIDE, VERIFY_MISSING, VERIFY_INLIER, VERIFY_OCCLUDED, VERIFY_VIOLATION, VERIFY_CLASSES };

struct VerifyScene {
  const uint16_t* depth;  // rows x cols u16 mm
  int32_t rows, cols;
  float fx, fy, cx, cy;
};

// Steps 3-4 for one point p of the model cloud, T's first three rows in T[0..11]; every operation correctly rounded.
// *d receives z_s - z_q (mm) when the point is compared (inlier, occluded or violation).  k_pose_pso's cost uses the
// same routine with delta = +inf, where every compared point is an inlier.
__device__ __forceinline__ int verify_point(const double* T, double px, double py, double pz, const VerifyScene& sc, double delta,
                                            double* dz) {
  double q[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    q[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * r], px), __dmul_rn(T[4 * r + 1], py)), __dmul_rn(T[4 * r + 2], pz)), T[4 * r + 3]);
  if (!(q[2] > 0.0)) return VERIFY_OUTSIDE;
  const double u = __dadd_rn(__dmul_rn((double)sc.fx, __ddiv_rn(q[0], q[2])), (double)sc.cx);
  const double v = __dadd_rn(__dmul_rn((double)sc.fy, __ddiv_rn(q[1], q[2])), (double)sc.cy);
  if (!isfinite(u) || !isfinite(v)) return VERIFY_OUTSIDE;
  const double c = floor(__dadd_rn(u, 0.5)), r = floor(__dadd_rn(v, 0.5));
  if (!(c >= 0.0 && c < (double)sc.cols && r >= 0.0 && r < (double)sc.rows)) return VERIFY_OUTSIDE;
  const uint16_t zs = sc.depth[(size_t)r * sc.cols + (size_t)c];
  if (zs == 0) return VERIFY_MISSING;
  const double d = __dsub_rn((double)zs, __dmul_rn(q[2], 1000.0));
  *dz = d;
  if (fabs(d) <= delta) return VERIFY_INLIER;
  return d < 0.0 ? VERIFY_OCCLUDED : VERIFY_VIOLATION;
}

// The CTA's n points P classified and counted (step 5), returned on thread 0.  The counts are exact in any order.
__device__ PoseVerify verify_block(const double* __restrict__ P, int n, const double* T, const VerifyScene& sc, double delta) {
  __shared__ int s_cnt[VERIFY_CLASSES];
  if (threadIdx.x < VERIFY_CLASSES) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  int cnt[VERIFY_CLASSES] = {0, 0, 0, 0, 0};
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    double d;
    const int k = verify_point(T, P[3 * j], P[3 * j + 1], P[3 * j + 2], sc, delta, &d);
#pragma unroll
    for (int q = 0; q < VERIFY_CLASSES; ++q) cnt[q] += k == q;
  }
#pragma unroll
  for (int q = 0; q < VERIFY_CLASSES; ++q) {
    const int w = __reduce_add_sync(0xffffffffu, cnt[q]);
    if ((threadIdx.x & 31) == 0 && w) atomicAdd(&s_cnt[q], w);
  }
  __syncthreads();
  PoseVerify o;
  o.counts[0] = n;
  for (int q = 0; q < VERIFY_CLASSES; ++q) o.counts[1 + q] = s_cnt[q];
  const int den = s_cnt[VERIFY_INLIER] + s_cnt[VERIFY_OCCLUDED] + s_cnt[VERIFY_VIOLATION];
  o.score = den > 0 ? __fdiv_rn((float)s_cnt[VERIFY_INLIER], (float)den) : 0.f;
  o.pad = 0;
  return o;
}

// One CTA per chunk slot behind the unshared ICP kernel: slot i's raw model cloud (k_pose_cloud's model slot, segment
// 2i) moved by outs[i].T, against the scene of its survivor's frame.  A slot without a pose gets score -1 and zero
// counts.  Unshared, the result goes to out[i]; SHARE (a shared stage that verifies), slot i's ICP output and its
// verification go to the pose areas of the exchange (pose_share_publish), and out is unused.
template <bool SHARE>
__global__ void __launch_bounds__(VERIFY_THREADS) k_pose_verify(PoseParams p, const IcpOut* __restrict__ outs, double delta,
                                                                PoseVerify* __restrict__ out, PoseShareDev sh) {
  __shared__ double s_T[12];
  const int i = blockIdx.x;
  PoseVerify v;
  if (!p.posed[i]) {  // block-uniform
    for (int q = 0; q < 6; ++q) v.counts[q] = 0;
    v.score = -1.f;
    v.pad = 0;
  } else {
    const int frame = p.frame_of ? p.frame_of[p.rank + i * p.world] : 0;
    const float* fK = p.frame_of ? p.sKs + 9 * frame : nullptr;
    VerifyScene sc;
    sc.depth = p.scene + (size_t)frame * p.srows * p.scols;
    sc.rows = p.srows; sc.cols = p.scols;
    sc.fx = fK ? fK[0] : p.sK[0]; sc.cx = fK ? fK[2] : p.sK[2]; sc.fy = fK ? fK[4] : p.sK[4]; sc.cy = fK ? fK[5] : p.sK[5];
    if (threadIdx.x < 12) s_T[threadIdx.x] = outs[i].T[threadIdx.x];
    __syncthreads();
    const int b = p.seg_begin[2 * i];
    v = verify_block(p.raw + (size_t)b * 3, p.seg_end[2 * i] - b, s_T, sc, delta);
  }
  if (threadIdx.x == 0) {
    if (SHARE) pose_share_publish(sh, outs[i], v);
    else out[i] = v;
  }
}

// --------------------------------------------------------------------------------------------
// tracking (include/linemod_b200.h, lm_track): a chunk whose clouds come from a given transformation T instead of a
// match position -- the model cloud of the template, and the scene cloud of the window the model projects to under T
// --------------------------------------------------------------------------------------------
struct TrackParams {
  const TrackObject* obj;     // [counts[0]] template (bank index) and T
  const int32_t* counts;      // [0] objects of the chunk
  int32_t rank, world;        // slot j takes object rank + j * world (lm_pose.h)
  const PoseTpl* tpl;
  const uint16_t* crops;
  // object i's frame frame_of[i] (null: frame 0): its depth scene + frame * srows * scols, its intrinsics sKs + 9 * frame
  const uint16_t* scene;
  int32_t srows, scols;
  const int32_t* frame_of;
  const float* sKs;
  int32_t margin;
  int64_t cap;                // most window pixels (LM_TRACK_WINDOW beyond)
  int64_t stride, M;          // points per object: M model points, then cap scene points
  double* raw;                // slot j's model cloud at j * stride, its scene cloud at j * stride + M
  unsigned long long* keys;
  int32_t* vals;
  int32_t* seg_begin;         // [2n], as PoseParams
  int32_t* seg_end;
  IcpJob* jobs;
  int32_t* err;
  uint8_t* posed;             // per slot, 1: LM_TRACK_TRACKED
  TrackRec* rec;              // per object
};

// Voxel keys of the n points P (PointCloud::VoxelDownSample(0.0025) about the per-axis minima mn, as k_pose_cloud
// computes them) into keys / vals from slot on.
__device__ __forceinline__ void track_voxel_keys(const double* P, int n, const double* mn, size_t slot, unsigned long long* keys,
                                                 int32_t* vals, int32_t* err) {
  const unsigned long long F = (1ull << POSE_KEY_BITS) - 1;
  double o[3];
  for (int c = 0; c < 3; ++c) o[c] = __dsub_rn(mn[c], 0.00125);
  for (int j = threadIdx.x; j < n; j += POSE_THREADS) {
    unsigned long long key = 0;
    for (int c = 0; c < 3; ++c) {
      const double v = floor(__ddiv_rn(__dsub_rn(P[3 * j + c], o[c]), 0.0025));
      unsigned long long a = (unsigned long long)(long long)v;
      if (!(v >= 0.0 && v <= (double)F)) { atomicExch(err, 1); a = F; }
      key = (key << POSE_KEY_BITS) | a;
    }
    keys[slot + j] = key;
    vals[slot + j] = j;
  }
}

// verify_point's step 3 alone, operation for operation (verify_point itself is left as it is, so that k_pose_verify and
// k_pose_pso keep their code): true and the pixel (*c, *r) when the point lands in the frame in front of the camera.
__device__ __forceinline__ bool track_project(const double* T, double px, double py, double pz, const VerifyScene& sc, int* c, int* r) {
  double q[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    q[k] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * k], px), __dmul_rn(T[4 * k + 1], py)), __dmul_rn(T[4 * k + 2], pz)), T[4 * k + 3]);
  if (!(q[2] > 0.0)) return false;
  const double u = __dadd_rn(__dmul_rn((double)sc.fx, __ddiv_rn(q[0], q[2])), (double)sc.cx);
  const double v = __dadd_rn(__dmul_rn((double)sc.fy, __ddiv_rn(q[1], q[2])), (double)sc.cy);
  if (!isfinite(u) || !isfinite(v)) return false;
  const double fc = floor(__dadd_rn(u, 0.5)), fr = floor(__dadd_rn(v, 0.5));
  if (!(fc >= 0.0 && fc < (double)sc.cols && fr >= 0.0 && fr < (double)sc.rows)) return false;
  *c = (int)fc; *r = (int)fr;
  return true;
}

// One CTA per slot: slot j takes object rank + j * world, and a slot past the chunk's objects writes an empty job (the
// window record is the object's, the clouds, job and posed flag the slot's).  The model cloud is k_pose_cloud's (every crop pixel with render depth > 0, row-major); each of
// its points is projected under T (track_project) and the in-frame pixels' extent is reduced over the CTA.  The
// window's pixels with scene depth > 0 are back-projected in row-major order as k_pose_cloud back-projects the scene.
// Both clouds get their voxel keys; the job starts at T.  An object without the status TRACKED writes an empty job.
// Everything an object's CTA computes depends only on the object and its own frame's depth and intrinsics.
__global__ void __launch_bounds__(POSE_THREADS) k_track_cloud(TrackParams p) {
  typedef cub::BlockScan<int, POSE_THREADS> Scan;
  typedef cub::BlockReduce<double, POSE_THREADS> Reduce;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename Reduce::TempStorage reduce;
  } tmp;
  __shared__ double s_T[16], s_min[6];
  __shared__ int s_ext[4], s_win[4], s_status;
  const int j = blockIdx.x, tid = threadIdx.x;  // slot j
  const int i = p.rank + j * p.world;            // its object
  const size_t sm = (size_t)j * p.stride, ss = sm + p.M;
  IcpJob* job = p.jobs + j;
  if (i >= p.counts[0]) {  // block-uniform: a slot past the chunk's objects (shared) writes an empty job
    if (tid == 0) {
      p.posed[j] = 0;
      job->src_first = job->tgt_first = (int32_t)sm;
      job->src_count = job->tgt_count = 0;
      for (int k = 0; k < 16; ++k) job->init[k] = (k % 5 == 0) ? 1.0 : 0.0;
      p.seg_begin[2 * j] = p.seg_end[2 * j] = (int32_t)sm;
      p.seg_begin[2 * j + 1] = p.seg_end[2 * j + 1] = (int32_t)ss;
    }
    return;
  }
  const PoseTpl T = p.tpl[p.obj[i].g];
  __shared__ VerifyScene sc;  // the object's frame (shared: it stays out of the registers)
  double* __restrict__ Mp = p.raw + sm * 3;
  double* __restrict__ Sp = p.raw + ss * 3;
  if (tid < 16) s_T[tid] = p.obj[i].T[tid];
  if (tid == 0) {
    s_ext[0] = s_ext[1] = INT_MAX; s_ext[2] = s_ext[3] = -1;
    const int frame = p.frame_of ? p.frame_of[i] : 0;
    const float* fK = p.sKs + 9 * frame;
    sc.depth = p.scene + (size_t)frame * p.srows * p.scols;
    sc.rows = p.srows; sc.cols = p.scols;
    sc.fx = fK[0]; sc.cx = fK[2]; sc.fy = fK[4]; sc.cy = fK[5];
  }
  __syncthreads();
  const uint16_t* __restrict__ C = p.crops + T.crop;
  const int bw = T.bw, npix = T.bw * T.bh;
  int c0 = INT_MAX, r0 = INT_MAX, c1 = -1, r1 = -1;
  int base = 0;
  for (int t0 = 0; t0 < npix; t0 += POSE_THREADS) {
    const int k = t0 + tid;
    bool fm = false;
    double mx = 0, my = 0, mz = 0;
    if (k < npix && C[k] > 0) {
      const int r = k / bw, q = k - r * bw;
      fm = true;
      mz = __ddiv_rn((double)C[k], 1000.0);
      mx = pose_backproject(q + T.bx, T.K[2], T.K[0], mz);
      my = pose_backproject(r + T.by, T.K[5], T.K[4], mz);
      int pc, pr;
      if (track_project(s_T, mx, my, mz, sc, &pc, &pr)) {
        c0 = min(c0, pc); c1 = max(c1, pc);
        r0 = min(r0, pr); r1 = max(r1, pr);
      }
    }
    int excl, agg;
    Scan(tmp.scan).ExclusiveSum(fm ? 1 : 0, excl, agg);
    if (fm) { double* o = Mp + 3 * (size_t)(base + excl); o[0] = mx; o[1] = my; o[2] = mz; }
    base += agg;
    __syncthreads();
  }
  const int nm = base;
  c0 = __reduce_min_sync(0xffffffffu, c0); r0 = __reduce_min_sync(0xffffffffu, r0);
  c1 = __reduce_max_sync(0xffffffffu, c1); r1 = __reduce_max_sync(0xffffffffu, r1);
  if ((tid & 31) == 0) { atomicMin(&s_ext[0], c0); atomicMin(&s_ext[1], r0); atomicMax(&s_ext[2], c1); atomicMax(&s_ext[3], r1); }
  __syncthreads();
  if (tid == 0) {
    TrackRec& rc = p.rec[i];
    int st = LM_TRACK_TRACKED;
    for (int k = 0; k < 4; ++k) rc.window[k] = rc.box[k] = s_win[k] = 0;
    if (s_ext[2] < 0) {
      st = LM_TRACK_OUTSIDE;
    } else {
      const int64_t x0 = s_ext[0], y0 = s_ext[1], x1 = s_ext[2], y1 = s_ext[3], m = p.margin;
      rc.box[0] = (int)x0; rc.box[1] = (int)y0; rc.box[2] = (int)(x1 - x0 + 1); rc.box[3] = (int)(y1 - y0 + 1);
      const int64_t wx0 = max(x0 - m, (int64_t)0), wy0 = max(y0 - m, (int64_t)0);
      const int64_t wx1 = min(x1 + m, (int64_t)sc.cols - 1), wy1 = min(y1 + m, (int64_t)sc.rows - 1);
      s_win[0] = (int)wx0; s_win[1] = (int)wy0; s_win[2] = (int)(wx1 - wx0 + 1); s_win[3] = (int)(wy1 - wy0 + 1);
      for (int k = 0; k < 4; ++k) rc.window[k] = s_win[k];
      if ((int64_t)s_win[2] * s_win[3] > p.cap) st = LM_TRACK_WINDOW;
    }
    s_status = st;
  }
  __syncthreads();
  int ns = 0;
  if (s_status == LM_TRACK_TRACKED) {  // block-uniform
    const int wx = s_win[0], wy = s_win[1], ww = s_win[2], wpix = s_win[2] * s_win[3];
    base = 0;
    for (int t0 = 0; t0 < wpix; t0 += POSE_THREADS) {
      const int k = t0 + tid;
      bool fs = false;
      double sx = 0, sy = 0, sz = 0;
      if (k < wpix) {
        const int r = k / ww, q = k - r * ww;
        const int sr = wy + r, scol = wx + q;
        const uint16_t sd = sc.depth[(size_t)sr * sc.cols + scol];
        if (sd > 0) {
          fs = true;
          sz = __ddiv_rn((double)sd, 1000.0);
          sx = pose_backproject(scol, sc.cx, sc.fx, sz);
          sy = pose_backproject(sr, sc.cy, sc.fy, sz);
        }
      }
      int excl, agg;
      Scan(tmp.scan).ExclusiveSum(fs ? 1 : 0, excl, agg);
      if (fs) { double* o = Sp + 3 * (size_t)(base + excl); o[0] = sx; o[1] = sy; o[2] = sz; }
      base += agg;
      __syncthreads();
    }
    ns = base;
    if (ns == 0 && tid == 0) s_status = LM_TRACK_NO_DEPTH;
    __syncthreads();
  }
  if (s_status != LM_TRACK_TRACKED) {  // block-uniform
    if (tid == 0) {
      p.rec[i].status = s_status;
      p.posed[j] = 0;
      job->src_first = job->tgt_first = (int32_t)sm;
      job->src_count = job->tgt_count = 0;
      for (int k = 0; k < 16; ++k) job->init[k] = s_T[k];
      p.seg_begin[2 * j] = p.seg_end[2 * j] = (int32_t)sm;
      p.seg_begin[2 * j + 1] = p.seg_end[2 * j + 1] = (int32_t)ss;
    }
    return;
  }
  for (int c = 0; c < 6; ++c) {  // per-axis minima of both clouds (exact in any order)
    const double* P = c < 3 ? Mp : Sp;
    const int n = c < 3 ? nm : ns;
    double v = INFINITY;
    for (int j = tid; j < n; j += POSE_THREADS) v = fmin(v, P[3 * j + c % 3]);
    v = Reduce(tmp.reduce).Reduce(v, cub::Min());
    if (tid == 0) s_min[c] = v;
    __syncthreads();
  }
  track_voxel_keys(Mp, nm, s_min, sm, p.keys, p.vals, p.err);
  track_voxel_keys(Sp, ns, s_min + 3, ss, p.keys, p.vals, p.err);
  if (tid == 0) {
    p.rec[i].status = LM_TRACK_TRACKED;
    p.posed[j] = 1;
    for (int k = 0; k < 16; ++k) job->init[k] = s_T[k];
    job->src_first = job->tgt_first = (int32_t)sm;
    job->src_count = job->tgt_count = 0;  // k_pose_voxel sets the counts
    p.seg_begin[2 * j] = (int32_t)sm; p.seg_end[2 * j] = (int32_t)sm + nm;
    p.seg_begin[2 * j + 1] = (int32_t)ss; p.seg_end[2 * j + 1] = (int32_t)ss + ns;
  }
}

// --------------------------------------------------------------------------------------------
// LM_POSE_PSO (include/linemod_b200.h): a particle swarm over rotations about the cloud's centroid and translations,
// scored against the scene depth with pose verification's projection
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ double pso_draw(unsigned long long seed, long long job, int k, int i, int q) {
  const unsigned long long number = (((unsigned long long)job * 1024ull + (unsigned long long)k) * 1024ull + (unsigned long long)i) * 16ull +
                                    (unsigned long long)q;
  unsigned long long z = seed + (number + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return __dmul_rn((double)(z >> 11), 0x1.0p-53);
}

// T(x) = Trans(c + t) Rot(w) Trans(-c) S as [R | u] into T[0..11] (include/linemod_b200.h).
__device__ __forceinline__ void pso_pose(const double* x, const double* c, const double* s, double* T) {
  const double w0 = x[0], w1 = x[1], w2 = x[2];
  const double y = __dadd_rn(__dadd_rn(__dmul_rn(w0, w0), __dmul_rn(w1, w1)), __dmul_rn(w2, w2));
  double R[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
  if (y != 0.0) {
    const double SA[11] = {0x1.0000000000000p+0, -0x1.5555555555555p-3, 0x1.1111111111111p-7, -0x1.a01a01a01a01ap-13,
                           0x1.71de3a556c734p-19, -0x1.ae64567f544e4p-26, 0x1.6124613a86d09p-33, -0x1.ae7f3e733b81fp-41,
                           0x1.952c77030ad4ap-49, -0x1.2f49b46814157p-57, 0x1.71b8ef6dcf572p-66};
    const double SB[11] = {0x1.0000000000000p-1, -0x1.5555555555555p-5, 0x1.6c16c16c16c17p-10, -0x1.a01a01a01a01ap-16,
                           0x1.27e4fb7789f5cp-22, -0x1.1eed8eff8d898p-29, 0x1.93974a8c07c9dp-37, -0x1.ae7f3e733b81fp-45,
                           0x1.6827863b97d97p-53, -0x1.e542ba4020225p-62, 0x1.0ce396db7f853p-70};
    double A = SA[10], B = SB[10];
#pragma unroll
    for (int k = 9; k >= 0; --k) { A = __dadd_rn(SA[k], __dmul_rn(y, A)); B = __dadd_rn(SB[k], __dmul_rn(y, B)); }
    const double w[3] = {w0, w1, w2};
    const double K[9] = {0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const double k2 = r == q ? __dsub_rn(__dmul_rn(w[r], w[r]), y) : __dmul_rn(w[r], w[q]);
        R[3 * r + q] = __dadd_rn(__dadd_rn(r == q ? 1.0 : 0.0, __dmul_rn(A, K[3 * r + q])), __dmul_rn(B, k2));
      }
  }
  const double a[3] = {__dsub_rn(s[0], c[0]), __dsub_rn(s[1], c[1]), __dsub_rn(s[2], c[2])};
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double m = __dadd_rn(__dadd_rn(__dmul_rn(R[3 * r], a[0]), __dmul_rn(R[3 * r + 1], a[1])), __dmul_rn(R[3 * r + 2], a[2]));
    T[4 * r] = R[3 * r]; T[4 * r + 1] = R[3 * r + 1]; T[4 * r + 2] = R[3 * r + 2];
    T[4 * r + 3] = __dadd_rn(__dadd_rn(s[r], __dsub_rn(m, a[r])), x[3 + r]);
  }
}

__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// One CTA per slot, persistent over the slots (grid <= n).  Dynamic shared memory: the chunk of points [PSO_CHUNK][3],
// then per particle its pose, position, velocity and personal best, then its cost and best cost.  Warp w scores
// particles w, w + 8, ...: its lanes sweep the chunk's points and a warp reduction gives the particle's sum, which only
// that warp adds to.  The scene is read through L1 / L2.
__global__ void __launch_bounds__(PSO_THREADS) k_pose_pso(PsoParams p) {
  extern __shared__ __align__(16) double pso_smem[];
  __shared__ double s_c[3], s_g[6];
  __shared__ long long s_fs, s_fg;
  __shared__ int s_gi;
  const int P = p.s.particles, I = p.s.iterations, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* s_pts = pso_smem;                      // [PSO_CHUNK][3]
  double* s_T = s_pts + 3 * PSO_CHUNK;           // [P][12]
  double* s_x = s_T + 12 * P;                    // [P][6]
  double* s_v = s_x + 6 * P;
  double* s_p = s_v + 6 * P;
  long long* s_f = reinterpret_cast<long long*>(s_p + 6 * P);  // [P]
  long long* s_fp = s_f + P;                                   // [P]
  const int clamp_um = (int)floor(__dmul_rn(p.s.clamp_mm, 1000.0));
  for (int slot = blockIdx.x; slot < p.n; slot += gridDim.x) {
    const IcpJob job = p.jobs[slot];
    const int n = job.src_count;
    const double* __restrict__ P3 = p.pts + (size_t)job.src_first * 3;
    const double S[3] = {job.init[3], job.init[7], job.init[11]};
    if (n == 0) {  // no cloud (a slot without a pose): S, no search
      if (tid == 0) {
        IcpOut o;
        for (int k = 0; k < 16; ++k) o.T[k] = job.init[k];
        o.fitness = 0.0; o.rmse = 0.0; o.iterations = I; o.pad = 0;
        p.outs[slot] = o;
      }
      continue;  // block-uniform
    }
    const int frame = p.frame_of ? p.frame_of[slot] : 0;
    const long long J = p.job ? p.job[slot] : p.first + slot - (p.frame_first ? p.frame_first[frame] : 0);
    const float* fK = p.frame_of ? p.sKs + 9 * frame : p.sK;
    VerifyScene sc;
    sc.depth = p.scene + (size_t)frame * p.srows * p.scols;
    sc.rows = p.srows; sc.cols = p.scols;
    sc.fx = fK[0]; sc.cx = fK[2]; sc.fy = fK[4]; sc.cy = fK[5];
    __syncthreads();  // the previous slot's last reads of the shared arrays
    if (tid < 3) {  // the centroid under S, in index order
      double a = 0.0;
      const double st = tid == 0 ? S[0] : (tid == 1 ? S[1] : S[2]);
      for (int j = 0; j < n; ++j) a = __dadd_rn(a, __dadd_rn(P3[3 * j + tid], st));
      s_c[tid] = __ddiv_rn(a, (double)n);
    }
    const int nchunks = (n + PSO_CHUNK - 1) / PSO_CHUNK;
    auto load_chunk = [&](int c0) {
      const int m = min(PSO_CHUNK, n - c0);
      for (int k = tid; k < 3 * m; k += PSO_THREADS) s_pts[k] = P3[(size_t)3 * c0 + k];
    };
    if (nchunks == 1) load_chunk(0);
    const int np = I > 0 ? P : 1;  // I = 0: the start alone
    const int rounds = I > 0 ? I : 1;
    for (int k = 0; k < rounds; ++k) {
      // positions: the start (iteration 0), or the move
      for (int e = tid; e < 6 * np; e += PSO_THREADS) {
        const int i = e / 6, q = e - 6 * i;
        const double D = q < 3 ? p.s.dr : p.s.dt;
        double& x = s_x[e];
        double& v = s_v[e];
        if (k == 0) {
          v = 0.0;
          x = i == 0 ? 0.0 : __dsub_rn(__dmul_rn(__dmul_rn(2.0, D), pso_draw(p.s.seed, J, 0, i, q)), D);
          s_p[e] = x;
        } else {
          const double r1 = pso_draw(p.s.seed, J, k, i, q), r2 = pso_draw(p.s.seed, J, k, i, 6 + q);
          const double g = s_gi < 0 ? 0.0 : s_g[q];
          double nv = __dadd_rn(__dadd_rn(__dmul_rn(0.7298, v), __dmul_rn(__dmul_rn(1.49618, r1), __dsub_rn(s_p[e], x))),
                                __dmul_rn(__dmul_rn(1.49618, r2), __dsub_rn(g, x)));
          if (nv > D) nv = D;
          else if (nv < -D) nv = -D;
          double nx = __dadd_rn(x, nv);
          if (nx > D) { nx = D; nv = 0.0; }
          else if (nx < -D) { nx = -D; nv = 0.0; }
          x = nx;
          v = nv;
        }
      }
      __syncthreads();
      for (int i = tid; i < np; i += PSO_THREADS) {
        pso_pose(s_x + 6 * i, s_c, S, s_T + 12 * i);
        s_f[i] = 0;
        if (k == 0) s_fp[i] = 0x7FFFFFFFFFFFFFFFll;
      }
      __syncthreads();
      // the costs
      for (int ch = 0; ch < nchunks; ++ch) {
        const int c0 = ch * PSO_CHUNK, m = min(PSO_CHUNK, n - c0);
        if (nchunks > 1) {
          __syncthreads();
          load_chunk(c0);
          __syncthreads();
        }
        for (int i = warp; i < np; i += PSO_THREADS / 32) {
          double T[12];
#pragma unroll
          for (int q = 0; q < 12; ++q) T[q] = s_T[12 * i + q];
          long long sum = 0;
          for (int j = lane; j < m; j += 32) {
            double d = 0.0;
            const int cls = verify_point(T, s_pts[3 * j], s_pts[3 * j + 1], s_pts[3 * j + 2], sc, INFINITY, &d);
            sum += cls == VERIFY_INLIER ? (int)floor(__dmul_rn(fmin(fabs(d), p.s.clamp_mm), 1000.0)) : clamp_um;
          }
          sum = warp_sum_ll(sum);
          if (lane == 0) s_f[i] += sum;
        }
      }
      __syncthreads();
      if (k == 0 && tid == 0) { s_fs = s_f[0]; s_fg = s_f[0]; s_gi = -1; }
      if (I > 0) {
        for (int i = tid; i < P; i += PSO_THREADS)
          if (s_f[i] < s_fp[i]) {
            s_fp[i] = s_f[i];
            for (int q = 0; q < 6; ++q) s_p[6 * i + q] = s_x[6 * i + q];
          }
        __syncthreads();
        if (tid == 0) {
          for (int i = 0; i < P; ++i)
            if (s_fp[i] < s_fg) { s_fg = s_fp[i]; s_gi = i; }
          if (p.record) p.record[(size_t)slot * p.record_words + 6 + k] = s_fg;
        }
        __syncthreads();
        if (tid < 6 && s_gi >= 0) s_g[tid] = s_p[6 * s_gi + tid];
      }
      __syncthreads();
    }
    if (tid == 0) {
      IcpOut o;
      if (s_gi < 0) {
        for (int q = 0; q < 16; ++q) o.T[q] = job.init[q];
      } else {
        pso_pose(s_g, s_c, S, o.T);
        o.T[12] = 0.0; o.T[13] = 0.0; o.T[14] = 0.0; o.T[15] = 1.0;
      }
      o.fitness = __ddiv_rn(__ddiv_rn((double)s_fg, (double)n), 1000.0);
      o.rmse = __ddiv_rn(__ddiv_rn((double)s_fs, (double)n), 1000.0);
      o.iterations = I; o.pad = 0;
      p.outs[slot] = o;
    }
    if (p.record) {
      long long* r = p.record + (size_t)slot * p.record_words;
      if (tid == 0) {
        r[0] = s_fs; r[1] = s_fg; r[2] = s_gi;
        for (int q = 0; q < 3; ++q) r[3 + q] = __double_as_longlong(s_c[q]);
      }
      long long* sw = r + 6 + I;
      for (int e = tid; e < 6 * P; e += PSO_THREADS) {
        const bool set = e < 6 * np;
        sw[e] = __double_as_longlong(set ? s_x[e] : 0.0);
        sw[6 * P + e] = __double_as_longlong(set ? s_v[e] : 0.0);
        sw[12 * P + e] = __double_as_longlong(set ? s_p[e] : 0.0);
      }
      for (int i = tid; i < P; i += PSO_THREADS) sw[18 * P + i] = I > 0 ? s_fp[i] : 0x7FFFFFFFFFFFFFFFll;
    }
  }
}

static size_t pso_smem_bytes(int particles) { return sizeof(double) * 3 * PSO_CHUNK + (size_t)PSO_PARTICLE_BYTES * particles; }

// k_pose_pso over p.n slots on st: a grid of at most the CTAs resident at once.
// The CTAs of k_pose_pso resident at once on the current device with P particles: found once per (device, P), with the
// kernel's shared-memory limit raised on the device the first time.
static int pso_resident(int particles, int* out) {
  static std::mutex mu;
  static std::vector<std::vector<int>> resident;  // [device][P]: 0 until known
  int dev = 0;
  CUI(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if ((int)resident.size() <= dev) resident.resize((size_t)dev + 1);
  std::vector<int>& r = resident[(size_t)dev];
  if (r.empty()) {
    CUI(cudaFuncSetAttribute(k_pose_pso, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pso_smem_bytes(PSO_MAX_PARTICLES)));
    r.assign(PSO_MAX_PARTICLES + 1, 0);
  }
  if (!r[(size_t)particles]) {
    int sms = 0, per_sm = 0;
    CUI(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CUI(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pose_pso, PSO_THREADS, pso_smem_bytes(particles)));
    r[(size_t)particles] = std::max(1, sms * per_sm);
  }
  *out = r[(size_t)particles];
  return LM_OK;
}

static int launch_pso(const PsoParams& p, cudaStream_t st) {
  if (p.n <= 0) return LM_OK;
  const size_t smem = pso_smem_bytes(p.s.particles);
  int resident = 1;
  const int rc = pso_resident(p.s.particles, &resident);
  if (rc) return rc;
  const int grid = std::min(p.n, resident);
  k_pose_pso<<<grid, PSO_THREADS, smem, st>>>(p);
  CUI(cudaGetLastError());
  return LM_OK;
}

extern "C" int lm_pose_search_points(int device, const double* pts, int64_t n, const double* start_t, const uint16_t* scene, int rows,
                                     int cols, const float* sK, int particles, int iterations, double dt_mm, double dr_deg,
                                     double clamp_mm, uint64_t seed, int64_t job, double* T_out, void* record, int64_t cap) {
  if (!pts || !start_t || !scene || !sK || !T_out || (cap > 0 && !record)) return lm_fail(LM_E_INVALID, "null argument");
  if (n < 1 || n > 0x7FFFFFFFll) return lm_fail(LM_E_INVALID, "%lld points, must lie in [1, 2^31 - 1]", (long long)n);
  if (rows <= 0 || cols <= 0) return lm_fail(LM_E_INVALID, "empty scene %d x %d", rows, cols);
  if (job < 0 || job >= PSO_MAX_JOB) return lm_fail(LM_E_INVALID, "job %lld outside [0, 2^40)", (long long)job);
  PoseSearch s;
  int rc = pose_search_make(particles, iterations, dt_mm, dr_deg, clamp_mm, seed, &s);
  if (rc) return rc;
  const int64_t words = pso_record_words(s);
  if (cap > 0 && cap < 8 * words)
    return lm_fail(LM_E_CAPACITY, "the swarm record needs %lld bytes, cap is %lld", (long long)(8 * words), (long long)cap);
  rc = open_device(device);
  if (rc) return rc;
  // one allocation: pts [n][3], the job, its number, the output, the record, the scene
  IcpJob j;
  memset(&j, 0, sizeof(j));
  j.src_first = j.tgt_first = 0; j.src_count = j.tgt_count = (int32_t)n;
  for (int k = 0; k < 16; ++k) j.init[k] = (k % 5 == 0) ? 1.0 : 0.0;
  for (int r = 0; r < 3; ++r) j.init[4 * r + 3] = start_t[r];
  const int64_t jn = job;
  auto a16 = [](size_t b) { return (b + 15) & ~(size_t)15; };
  const size_t o_job = a16(sizeof(double) * 3 * (size_t)n), o_num = o_job + a16(sizeof(IcpJob)), o_out = o_num + 16;
  const size_t o_rec = o_out + a16(sizeof(IcpOut)), o_scene = o_rec + a16(8 * (size_t)words);
  DeviceArray<uint8_t> buf;
  CUI(buf.assign(o_scene + sizeof(uint16_t) * (size_t)rows * cols));
  uint8_t* b = buf.get();
  CUI(cudaMemcpy(b, pts, sizeof(double) * 3 * (size_t)n, cudaMemcpyHostToDevice));
  CUI(cudaMemcpy(b + o_job, &j, sizeof(j), cudaMemcpyHostToDevice));
  CUI(cudaMemcpy(b + o_num, &jn, sizeof(jn), cudaMemcpyHostToDevice));
  CUI(cudaMemcpy(b + o_scene, scene, sizeof(uint16_t) * (size_t)rows * cols, cudaMemcpyHostToDevice));
  PsoParams p;
  memset(&p, 0, sizeof(p));
  p.jobs = reinterpret_cast<const IcpJob*>(b + o_job); p.pts = reinterpret_cast<const double*>(b);
  p.outs = reinterpret_cast<IcpOut*>(b + o_out); p.n = 1;
  p.scene = reinterpret_cast<const uint16_t*>(b + o_scene); p.srows = rows; p.scols = cols;
  memcpy(p.sK, sK, sizeof(p.sK));
  p.job = reinterpret_cast<const int64_t*>(b + o_num);
  p.s = s;
  p.record = reinterpret_cast<long long*>(b + o_rec); p.record_words = words;
  rc = launch_pso(p, 0);
  if (rc) return rc;
  IcpOut o;
  CUI(cudaMemcpy(&o, b + o_out, sizeof(o), cudaMemcpyDeviceToHost));
  memcpy(T_out, o.T, sizeof(o.T));
  if (cap > 0) CUI(cudaMemcpy(record, b + o_rec, 8 * (size_t)words, cudaMemcpyDeviceToHost));
  return LM_OK;
}

// --------------------------------------------------------------------------------------------
// pose NMS (lm_pose.h): the greedy translation NMS of linemod_ros/detect.py:41-50, 130-131 behind the pose stage
// --------------------------------------------------------------------------------------------
// One CTA, one entry per thread (n <= NMS_THREADS).  Each round picks the best live entry with a block-wide arg-max
// (order-preserving 64-bit score key, lower index on ties), keeps it and drops every live entry j with
// !(d_ij > thr), d_ij = sqrt((dx*dx + dy*dy) + dz*dz) in float64 with every operation correctly rounded: what
// np.linalg.norm(ts[i] - ts[order[1:]], axis=1) computes for 3-vectors.  A NaN distance suppresses.
#define NMS_THREADS 1024  // == LM_POST_MAX, the most survivors k_post_nms writes

struct PoseRt {  // per template of the bank: the pose its render was made with (init_base, LL.cpp:34-38)
  float R[9], t[3];
};

struct PoseNmsHead {
  int32_t kept, survivors, posed, pad;
};

struct PoseNmsOut {  // one kept pose
  double R[9], t[3];  // as lm_complete_pose returns them (t in mm)
  lm_match m;
  float residual;
};

// Score order: descending, -0.0 == +0.0, NaN before every number (where argsort()[::-1] puts it).
__device__ __forceinline__ unsigned long long nms_score_key(double s) {
  if (s != s) return ~0ull;
  if (s == 0.0) return 1ull << 63;
  const unsigned long long b = (unsigned long long)__double_as_longlong(s);
  return (b >> 63) ? ~b : (b | (1ull << 63));
}

__device__ __forceinline__ void nms_argmax_warp(unsigned long long& k, int& i) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const unsigned long long ok = __shfl_down_sync(0xffffffffu, k, d);
    const int oi = __shfl_down_sync(0xffffffffu, i, d);
    if (oi >= 0 && (i < 0 || ok > k || (ok == k && oi < i))) { k = ok; i = oi; }
  }
}

// Thread i holds entry i: whether it takes part, its score key and its translation.  Returns the number kept on every
// thread; thread 0 writes the kept indices in keep order to keep[] (if not null), and a kept entry's thread gets its
// position in rank.
// blockDim.x == NMS_THREADS.
__device__ int nms_translations_block(bool cand, unsigned long long key, double tx, double ty, double tz, double thr,
                                      int32_t* keep, int& rank) {
  __shared__ unsigned long long s_key[NMS_THREADS / 32];
  __shared__ int s_idx[NMS_THREADS / 32];
  __shared__ int s_pick;
  __shared__ double s_t[3];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  bool live = cand;
  int kept = 0;
  rank = -1;
  for (;;) {
    unsigned long long bk = live ? key : 0ull;
    int bi = live ? tid : -1;
    nms_argmax_warp(bk, bi);
    if (lane == 0) { s_key[wid] = bk; s_idx[wid] = bi; }
    __syncthreads();
    if (wid == 0) {
      bk = s_key[lane]; bi = s_idx[lane];
      nms_argmax_warp(bk, bi);
      if (lane == 0) s_pick = bi;
    }
    __syncthreads();
    const int pick = s_pick;
    if (pick < 0) break;  // nothing live
    if (tid == pick) { s_t[0] = tx; s_t[1] = ty; s_t[2] = tz; live = false; rank = kept; }
    if (tid == 0 && keep) keep[kept] = pick;
    ++kept;
    __syncthreads();
    if (live) {
      const double dx = __dsub_rn(s_t[0], tx), dy = __dsub_rn(s_t[1], ty), dz = __dsub_rn(s_t[2], tz);
      const double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
      if (!(d > thr)) live = false;
    }
  }
  return kept;
}

// lm_nms_translations: the same pass on caller arrays, every entry a candidate.
__global__ void __launch_bounds__(NMS_THREADS) k_nms_translations(int n, const double* __restrict__ t, const double* __restrict__ score,
                                                                  double thr, int32_t* __restrict__ keep, int32_t* __restrict__ n_keep) {
  const int i = threadIdx.x;
  const bool cand = i < n;
  double tx = 0, ty = 0, tz = 0;
  unsigned long long key = 0;
  if (cand) { tx = t[3 * i]; ty = t[3 * i + 1]; tz = t[3 * i + 2]; key = nms_score_key(score[i]); }
  int rank;
  const int kept = nms_translations_block(cand, key, tx, ty, tz, thr, keep, rank);
  if (i == 0) *n_keep = kept;
}

// init_base entry (k, c) of the template's pose (init_base: only t.z in metres)
__device__ __forceinline__ float pose_base(const PoseRt& q, int k, int c) {
  if (k == 3) return c == 3 ? 1.f : 0.f;
  if (c < 3) return q.R[3 * k + c];
  return k == 2 ? __fdiv_rn(q.t[2], 1000.0f) : q.t[k];
}

// (transformation_ * init_base)[r][c], summed as compose() does (LL.cpp:146)
__device__ __forceinline__ double pose_compose(const double* T, const PoseRt& q, int r, int c) {
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) s = __dadd_rn(s, __dmul_rn(T[4 * r + k], (double)pose_base(q, k, c)));
  return s;
}

struct PoseNmsParams {
  const lm_match* surv;
  const int32_t* counts;    // [0] survivors written by k_post_nms (without frame_first)
  const uint8_t* posed;     // k_pose_cloud's verdict per survivor
  const IcpOut* outs;
  const PoseRt* rt;
  const int32_t* class_begin;
  double thr;
  PoseNmsHead* head;        // [frame]
  PoseNmsOut* out;          // kept poses in keep order, frame f's from out + frame_first[f]
  // null: one frame, survivors [0, counts[0]).  Else frame f's survivors are [frame_first[f], frame_first[f + 1]).
  const int32_t* frame_first;
  int32_t* src;             // per kept pose its survivor's index in the run (at out's index): its T is in outs
  // VERIFY only: per survivor its verification (k_pose_verify), per kept pose its copy (at out's index), and the
  // ranking and minimum score of lm_set_pose_verify
  const PoseVerify* ver;
  PoseVerify* vout;
  int32_t rank_by;
  double min_score;
};

// Behind the ICP kernel: candidates are the survivors with a pose, score -(double)residual.  One frame per CTA.
// Every kept pose's survivor goes to src.  VERIFY (behind k_pose_verify): a survivor scoring below min_score is no
// candidate, rank_by may put the score first, and every kept pose's verification goes to vout.
template <bool VERIFY>
__global__ void __launch_bounds__(NMS_THREADS) k_pose_nms(PoseNmsParams p) {
  const int i = threadIdx.x;
  const int first = p.frame_first ? p.frame_first[blockIdx.x] : 0;
  const int n = p.frame_first ? p.frame_first[blockIdx.x + 1] - first : min(p.counts[0], NMS_THREADS);
  const lm_match* __restrict__ surv = p.surv + first;
  const IcpOut* __restrict__ outs = p.outs + first;
  bool cand = false;
  double t[3] = {0, 0, 0};
  float res = 0.f;
  int g = 0;
  if (i < n && p.posed[first + i]) {
    const lm_match m = surv[i];
    g = p.class_begin[m.class_index] + m.template_id;  // k_pose_cloud found it: in range
    const PoseRt q = p.rt[g];
    for (int r = 0; r < 3; ++r) t[r] = __dmul_rn(pose_compose(outs[i].T, q, r, 3), 1000.0);
    res = __double2float_rn(outs[i].fitness);
    cand = true;
  }
  const int posed = __syncthreads_count(cand);
  unsigned long long key = nms_score_key(-(double)res);
  if (VERIFY && cand) {
    const float score = p.ver[first + i].score;
    if ((double)score < p.min_score) cand = false;
    if (p.rank_by == LM_VERIFY_RANK_SCORE) key = nms_score_key((double)score);
  }
  int rank;
  const int kept = nms_translations_block(cand, key, t[0], t[1], t[2], p.thr, nullptr, rank);
  if (VERIFY && rank >= 0) p.vout[first + rank] = p.ver[first + i];
  if (rank >= 0) {
    PoseNmsOut o;
    const PoseRt q = p.rt[g];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) o.R[3 * r + c] = pose_compose(outs[i].T, q, r, c);
    for (int r = 0; r < 3; ++r) o.t[r] = t[r];
    o.m = surv[i];
    o.residual = res;
    p.out[first + rank] = o;
    p.src[first + rank] = first + i;
  }
  if (i == 0) {
    PoseNmsHead h;
    h.kept = kept; h.survivors = p.frame_first ? n : p.counts[0]; h.posed = posed; h.pad = 0;
    p.head[blockIdx.x] = h;
  }
}

// --------------------------------------------------------------------------------------------
// view following (lm_set_track_views, include/linemod_b200.h): each tracked object re-chooses its template from its
// pose before k_track_cloud reads it
// --------------------------------------------------------------------------------------------
#define VIEW_THREADS 256

struct TrackViewParams {
  TrackObject* obj;           // [counts[0]]: template and T, overwritten with the chosen template and T'
  const int32_t* counts;      // [0] objects
  const PoseRt* rt;           // per template of the bank: R_b, t_b of its render
  const uint8_t* has;         // per template of the bank: 1 when its render is registered
  const int32_t* class_begin; // [n_classes + 1]
  int32_t n_classes;
  double tau;                 // 1 + 2 cos(turn_deg)
};

// ((a0 * b0) + a1 * b1) + a2 * b2, every operation correctly rounded
__device__ __forceinline__ double view_dot3(double a0, double b0, double a1, double b1, double a2, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

// trace(Ro^T R): s = s + Ro[r][c] * R[r][c] from 0.0, r outer, c inner
__device__ __forceinline__ double view_score(const double* Ro, const float* R) {
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < 9; ++k) s = __dadd_rn(s, __dmul_rn(Ro[k], (double)R[k]));
  return s;
}

// One CTA per object.  Its class is the one whose templates hold its template k; every thread scans a stride of the
// class's templates with a render, a block arg-max (nms_argmax_warp: lowest index on ties, a NaN score never a
// candidate) gives j*, and thread 0 decides and re-expresses T (include/linemod_b200.h, lm_set_track_views).
__global__ void __launch_bounds__(VIEW_THREADS) k_track_views(TrackViewParams p) {
  __shared__ double s_Ro[9];
  __shared__ int32_t s_range[2];
  __shared__ unsigned long long s_key[VIEW_THREADS / 32];
  __shared__ int s_idx[VIEW_THREADS / 32];
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (i >= p.counts[0]) return;  // block-uniform
  TrackObject* o = p.obj + i;
  const int64_t k = o->g;
  if (tid < 9) {
    const int r = tid / 3, c = tid - 3 * (tid / 3);
    const float* Rk = p.rt[k].R;
    s_Ro[tid] = view_dot3(o->T[4 * r], (double)Rk[c], o->T[4 * r + 1], (double)Rk[3 + c], o->T[4 * r + 2], (double)Rk[6 + c]);
  }
  if (tid == 0) {  // the last class beginning at or before k (an empty class shares its begin with the next)
    int lo = 0, hi = p.n_classes;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (p.class_begin[mid] <= k) lo = mid;
      else hi = mid;
    }
    s_range[0] = p.class_begin[lo]; s_range[1] = p.class_begin[lo + 1];
  }
  __syncthreads();
  double Ro[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) Ro[q] = s_Ro[q];
  unsigned long long bk = 0ull;
  int bi = -1;
  for (int j = s_range[0] + tid; j < s_range[1]; j += VIEW_THREADS) {
    if (!p.has[j]) continue;
    const double s = view_score(Ro, p.rt[j].R);
    if (s != s) continue;
    const unsigned long long key = nms_score_key(s);
    if (bi < 0 || key > bk) { bk = key; bi = j; }  // ascending j: the first of equal keys stays
  }
  nms_argmax_warp(bk, bi);
  if (lane == 0) { s_key[wid] = bk; s_idx[wid] = bi; }
  __syncthreads();
  if (wid != 0) return;
  bk = lane < VIEW_THREADS / 32 ? s_key[lane] : 0ull;
  bi = lane < VIEW_THREADS / 32 ? s_idx[lane] : -1;
  nms_argmax_warp(bk, bi);
  if (lane != 0) return;
  const double sk = view_score(Ro, p.rt[k].R);
  if (!(sk < p.tau) || bi < 0 || bi == k) return;
  const float* Rj = p.rt[bi].R;
  if (!(view_score(Ro, Rj) > sk)) return;
  const float* Rk = p.rt[k].R;
  double bk3[3], bj3[3], QR[9], Qt[3], T[16];
  for (int r = 0; r < 3; ++r) {
    bk3[r] = __ddiv_rn((double)p.rt[k].t[r], 1000.0);
    bj3[r] = __ddiv_rn((double)p.rt[bi].t[r], 1000.0);
  }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      QR[3 * r + c] = view_dot3(Rk[3 * r], Rj[3 * c], Rk[3 * r + 1], Rj[3 * c + 1], Rk[3 * r + 2], Rj[3 * c + 2]);
  for (int r = 0; r < 3; ++r) Qt[r] = __dsub_rn(bk3[r], view_dot3(QR[3 * r], bj3[0], QR[3 * r + 1], bj3[1], QR[3 * r + 2], bj3[2]));
  for (int q = 0; q < 16; ++q) T[q] = o->T[q];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) o->T[4 * r + c] = view_dot3(T[4 * r], QR[c], T[4 * r + 1], QR[3 + c], T[4 * r + 2], QR[6 + c]);
    o->T[4 * r + 3] = __dadd_rn(view_dot3(T[4 * r], Qt[0], T[4 * r + 1], Qt[1], T[4 * r + 2], Qt[2]), T[4 * r + 3]);
  }
  o->T[12] = o->T[13] = o->T[14] = 0.0; o->T[15] = 1.0;
  o->g = bi;
}

int track_view_tau(int on, double turn_deg, double* tau) {
  if (on && !(turn_deg >= 0.0 && turn_deg < 180.0))
    return lm_fail(LM_E_INVALID, "turn_deg must lie in [0, 180), got %g", turn_deg);
  *tau = on ? 1.0 + 2.0 * cos(turn_deg * 0.017453292519943295) : 0.0;
  return LM_OK;
}

struct TplHost {
  bool set = false;
  int box[4] = {0, 0, 0, 0};
  uint16_t anchor = 0;
  float K[9], R[9], t[3];
  std::vector<uint16_t> crop;
};

// What filled the finished-run record: a frame or batch without the pose NMS, one with it, a track run, an lm_icp call.
enum class PoseRunKind { none, poses, kept, track, icp };

// The run last finished: all that pose_stage_verify, pose_stage_transforms and pose_stage_track_templates read (lm_pose.h
// gives their rules).  Each finish resets it before anything can fail, and fills it once the run has succeeded.
struct PoseFinished {
  PoseRunKind kind = PoseRunKind::none;
  bool stale = false;             // a run has been prepared since: T, kept and tpl no longer answer; ver still does
  bool verified = false;          // the run verified: ver holds its entries' verification
  std::vector<PoseVerify> ver;
  std::vector<double> T;          // poses, track: [entry][16], NaN for an entry without a pose
  // kept: per frame, the index of its first kept pose in d_bksrc and d_bouts and its number of kept poses; the run's
  // survivors and stream
  std::vector<std::pair<int64_t, int64_t>> kept;
  int64_t survivors = 0;
  cudaStream_t stream = nullptr;
  std::vector<int32_t> tpl;       // track: per entry its template within its class

  void reset() {
    kind = PoseRunKind::none;
    stale = verified = false;
    ver.clear(); T.clear(); kept.clear(); tpl.clear();
    survivors = 0;
    stream = nullptr;
  }
  // A run of kind k succeeded; v (verify: its n entries') is the verification.
  void fill(PoseRunKind k, bool verify, const PoseVerify* v, int64_t n) {
    kind = k;
    stale = false;
    verified = verify;
    if (verify) ver.assign(v, v + n);
  }
  // n entries, none with a pose until compose() gives it one.
  void entries(int64_t n) { T.assign(16 * (size_t)n, std::numeric_limits<double>::quiet_NaN()); }
  // Entry i from ICP output o against the render made with R, t: its R, t and residual out (render_pose), its T here.
  void compose(int64_t i, const IcpOut& o, const float* R, const float* t, double* R_out, double* t_out, float* residual) {
    render_pose(o, R, t, R_out + 9 * i, t_out + 3 * i, residual + i);
    memcpy(T.data() + 16 * i, o.T, sizeof(o.T));
  }
};

struct lm_pose_stage {
  std::vector<TplHost> tpl;
  std::vector<int32_t> class_begin;
  bool dirty = false;          // the device copy of the registered renders is stale (a stage without any has none)
  int64_t area_max = 0;        // largest crop
  DeviceArray<PoseTpl> d_tpl; DeviceArray<uint16_t> d_crops; DeviceArray<int32_t> d_class_begin;
  DeviceArray<PoseRt> d_rt;    // per template: R, t of its render (k_pose_nms composes the poses)
  DeviceArray<uint8_t> d_has;  // per template: 1 when its render is registered (k_track_views)
  // per-chunk buffers for pose_slots() survivors of pose_area() points per crop (pose_buffers); d_posed: a shared
  // chunk's posed flags per slot, which k_pose_collect gathers into the run's
  DeviceArray<double> d_raw, d_cpts, d_pts, d_nrm;
  DeviceArray<unsigned long long> d_keys[2];
  DeviceArray<int32_t> d_vals[2];
  DeviceArray<int32_t> d_seg;
  DeviceArray<IcpJob> d_jobs;
  DeviceArray<uint8_t> d_sort_tmp;
  DeviceArray<uint8_t> d_posed;
  // A group of buffers that grows together is freed as a whole, then allocated in order: its last array is empty
  // unless every one was allocated, so its size stands for the group's.
  // a batch's scene slots and survivors, filled by the caller (pose_batch_reserve), and a track run's scenes
  DeviceArray<uint16_t> d_bscene;
  DeviceArray<lm_match> d_bsurv;
  // a run's outputs (pose_outputs), a frame's at offset 0: per survivor its frame, ICP output and posed flag, and per
  // kept pose of the pose NMS its survivor
  DeviceArray<int32_t> d_bframe;
  // only once a run verifies: per survivor its verification and per kept pose its copy, the host's copy of either
  // (h_bver last: survivors), and per chunk slot the ICP output a verifying shared stage publishes from
  DeviceArray<PoseVerify> d_bver, d_bvkept; PinnedArray<PoseVerify> h_bver;
  DeviceArray<IcpOut> d_souts;
  DeviceArray<IcpOut> d_bouts; DeviceArray<uint8_t> d_bposed; DeviceArray<int32_t> d_bksrc;
  PinnedArray<IcpOut> h_bouts;  // h_bouts last: survivors
  // per frame its first survivor and intrinsics, per chunk (at most one per frame) a status block (PoseChunk; [3] a
  // batch chunk's size)
  DeviceArray<int32_t> d_bfirst; DeviceArray<float> d_bsK;  // [frames + 1], [frames][9]
  DeviceArray<int32_t> d_bstat; PinnedArray<int32_t> h_bstat;  // h_bstat last: frames
  // the pose NMS block (nms_heads, nms_out)
  DeviceArray<uint8_t> d_bnms; PinnedArray<uint8_t> h_bnms;
  // the run last enqueued, its share and survivor offsets copied; its launches, and how many of its ICP outputs (or,
  // pose NMS enqueued, kept poses) are on their way to the host
  PoseRun run = {};
  PoseShare share = {};
  std::vector<int64_t> first;
  int64_t launches = 0, fetched = 0;
  PoseFinished done;
  // the last chunk pose_chunk enqueued (pose_stage_clouds): its slots, rank and world, its first survivor in the run and
  // its posed flags per slot.  valid false before the first chunk and from the next pose_prepare on, which may move the
  // buffers.
  struct {
    bool valid = false;
    int slots = 0, rank = 0, world = 1;
    int64_t first = 0;
    const uint8_t* posed = nullptr;
    bool track = false;  // a track chunk: d_trec holds its windows from `first` on
  } last;
  // tracking (pose_stage_track; its scenes are in d_bscene): the objects of the run and their windows
  DeviceArray<TrackObject> d_tobj;
  DeviceArray<TrackRec> d_trec; PinnedArray<TrackRec> h_trec;
};

// The per-chunk buffers: slots of 2 clouds of pose_area() points for each of pose_slots() survivors.  d_sort_tmp is
// allocated last, so both are 0 unless every buffer was allocated.
static int pose_slots(const lm_pose_stage* s) { return s->d_sort_tmp.empty() ? 0 : (int)s->d_jobs.size(); }
static int64_t pose_area(const lm_pose_stage* s) {
  return pose_slots(s) ? (int64_t)(s->d_cpts.size() / (3 * s->d_jobs.size())) : 0;
}

lm_pose_stage* pose_stage_create() { return new lm_pose_stage(); }

void pose_stage_destroy(lm_pose_stage* s) { delete s; }

void pose_stage_clear(lm_pose_stage* s) {
  s->tpl.clear();
  s->class_begin.clear();
  s->area_max = 0;
  s->dirty = true;
}

int pose_stage_register(lm_pose_stage* s, const int32_t* class_begin, int n_classes, int64_t first, int64_t n,
                        const uint16_t* const* depths, int rows, int cols, const float* K, const float* R, const float* t) {
  const int64_t G = class_begin[n_classes];
  if (!depths || !K || !R || !t) return lm_fail(LM_E_INVALID, "null argument");
  if (n < 1 || first < 0 || first + n > G)
    return lm_fail(LM_E_INVALID, "renders [%lld, %lld) outside the bank's %lld templates", (long long)first, (long long)(first + n), (long long)G);
  if (rows <= 0 || cols <= 0) return lm_fail(LM_E_INVALID, "empty render size %d x %d", rows, cols);
  std::vector<TplHost> add((size_t)n);
  for (int64_t i = 0; i < n; ++i) {
    const uint16_t* d = depths[i];
    if (!d) return lm_fail(LM_E_INVALID, "depths[%lld] is null", (long long)i);
    TplHost& h = add[(size_t)i];
    model_box(d, rows, cols, h.box);
    if (h.box[2] == 0) return lm_fail(LM_E_INVALID, "render of template %lld has no non-zero pixel", (long long)(first + i));
    if ((int64_t)h.box[2] * h.box[3] >= (1ll << POSE_KEY_BITS))
      return lm_fail(LM_E_INVALID, "render of template %lld: box of %d x %d pixels is too large", (long long)(first + i), h.box[2], h.box[3]);
    h.anchor = d[(size_t)(rows / 2) * cols + cols / 2];
    h.crop.resize((size_t)h.box[2] * h.box[3]);
    for (int r = 0; r < h.box[3]; ++r)
      memcpy(h.crop.data() + (size_t)r * h.box[2], d + (size_t)(r + h.box[1]) * cols + h.box[0], sizeof(uint16_t) * h.box[2]);
    memcpy(h.K, K + 9 * i, sizeof(h.K));
    memcpy(h.R, R + 9 * i, sizeof(h.R));
    memcpy(h.t, t + 3 * i, sizeof(h.t));
    h.set = true;
  }
  if ((int64_t)s->tpl.size() != G) s->tpl.assign((size_t)G, TplHost());
  s->class_begin.assign(class_begin, class_begin + n_classes + 1);
  for (int64_t i = 0; i < n; ++i) s->tpl[(size_t)(first + i)] = std::move(add[(size_t)i]);
  s->area_max = 0;
  for (const TplHost& h : s->tpl) s->area_max = std::max<int64_t>(s->area_max, (int64_t)h.crop.size());
  s->dirty = true;
  return LM_OK;
}

bool pose_stage_covers(const lm_pose_stage* s, const int32_t* sel, int64_t n_sel) {
  if (s->tpl.empty()) return false;
  for (int64_t k = 0; k < n_sel; ++k)
    if (sel[k] < 0 || sel[k] >= (int64_t)s->tpl.size() || !s->tpl[(size_t)sel[k]].set) return false;
  return true;
}

static int pose_upload(lm_pose_stage* s, cudaStream_t st) {
  std::vector<PoseTpl> tp(s->tpl.size());
  std::vector<PoseRt> rt(s->tpl.size());
  std::vector<uint8_t> has(s->tpl.size());
  int64_t pool = 0;
  for (size_t g = 0; g < s->tpl.size(); ++g) {
    const TplHost& h = s->tpl[g];
    PoseTpl& d = tp[g];
    d.bx = h.box[0]; d.by = h.box[1]; d.bw = h.box[2]; d.bh = h.box[3];
    d.crop = pool;
    d.anchor = h.anchor;
    for (int k = 0; k < 9; ++k) d.K[k] = h.set ? h.K[k] : 0.f;
    for (int k = 0; k < 9; ++k) rt[g].R[k] = h.set ? h.R[k] : 0.f;
    for (int k = 0; k < 3; ++k) rt[g].t[k] = h.set ? h.t[k] : 0.f;
    has[g] = h.set ? 1 : 0;
    pool += (int64_t)h.crop.size();
  }
  std::vector<uint16_t> crops((size_t)std::max<int64_t>(pool, 1));
  for (size_t g = 0; g < s->tpl.size(); ++g)
    if (!s->tpl[g].crop.empty()) memcpy(crops.data() + tp[g].crop, s->tpl[g].crop.data(), s->tpl[g].crop.size() * sizeof(uint16_t));
  CUI(cudaStreamSynchronize(st));  // an earlier frame may still read the old copy
  s->d_tpl.reset(); s->d_crops.reset(); s->d_class_begin.reset(); s->d_rt.reset(); s->d_has.reset();
  CUI(upload(s->d_tpl, tp, st));
  CUI(upload(s->d_rt, rt, st));
  CUI(upload(s->d_has, has, st));
  CUI(upload(s->d_crops, crops, st));
  CUI(upload(s->d_class_begin, s->class_begin, st));
  CUI(cudaStreamSynchronize(st));  // host vectors go out of scope
  s->dirty = false;
  return LM_OK;
}

static int pose_buffers(lm_pose_stage* s, cudaStream_t st, int bound, int64_t area) {
  if (bound <= pose_slots(s) && area <= pose_area(s)) return LM_OK;
  CUI(cudaStreamSynchronize(st));
  const int B = std::max(bound, pose_slots(s));
  const int64_t A = std::max(area, pose_area(s));
  const int64_t slots = 2 * (int64_t)B * A;  // points of every cloud slot
  if (slots > 0x7FFFFFFFll)
    return lm_fail(LM_E_CAPACITY, "pose stage: %d survivors x %lld-pixel crops exceed 2^31 points: lower top_k", B, (long long)A);
  s->d_raw.reset(); s->d_cpts.reset(); s->d_pts.reset(); s->d_nrm.reset();
  for (int k = 0; k < 2; ++k) { s->d_keys[k].reset(); s->d_vals[k].reset(); }
  s->d_seg.reset(); s->d_jobs.reset(); s->d_sort_tmp.reset(); s->d_posed.reset();
  CUI(s->d_raw.assign(3 * slots));
  CUI(s->d_pts.assign(3 * slots));
  CUI(s->d_nrm.assign(3 * slots));
  CUI(s->d_cpts.assign(3 * (slots / 2)));
  for (int k = 0; k < 2; ++k) {
    CUI(s->d_keys[k].assign(slots));
    CUI(s->d_vals[k].assign(slots));
  }
  CUI(s->d_seg.assign(4 * B));
  CUI(s->d_jobs.assign(B));
  CUI(s->d_posed.assign(B));
  cub::DoubleBuffer<unsigned long long> dk(s->d_keys[0].get(), s->d_keys[1].get());
  cub::DoubleBuffer<int32_t> dv(s->d_vals[0].get(), s->d_vals[1].get());
  size_t tmp_bytes = 0;
  CUI(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, tmp_bytes, dk, dv, (int)slots, 2 * B, s->d_seg.get(), s->d_seg.get() + 2 * B, 0,
                                               3 * POSE_KEY_BITS, st));
  CUI(s->d_sort_tmp.assign(std::max<size_t>(tmp_bytes, 16)));
  return LM_OK;
}

// The device side of one pose exchange: number seq, survivor count counts[0], this rank's per-slot posed flags, status
// as PoseShareDev.
static PoseShareDev share_dev(const PoseShare& sh, int32_t seq, const int32_t* counts, const uint8_t* posed, int32_t* status) {
  PoseShareDev sd;
  memset(&sd, 0, sizeof(sd));
  for (int r = 0; r < sh.world; ++r) sd.area[r] = sh.base[r] + sh.area_offset;
  sd.world = sh.world; sd.rank = sh.rank; sd.seq = seq;
  sd.counts = counts; sd.posed = posed; sd.status = status;
  sd.timeout_ns = sh.timeout_ns; sd.abort_flag = sh.abort_flag;
  return sd;
}

// One chunk of the pose stage (lm_pose.h): survivors surv[0, counts[0]), counts on the device, of one frame (frame_of
// null: depth scene, intrinsics sK) or of the frames frame_of gives.  The launches are sized for `slots` survivors.
// Their results go to outs / posed; status: [0] cloud overflow, shared [1] a peer's poses did not arrive, [2] entries
// this rank published.  seq: the chunk's pose exchange (shared).
// The renders a chunk's survivors use: survivor m takes entry class_begin[m.class_index] + m.template_id of tpl (n_tpl
// entries), whose crop lies in crops.
struct PoseTable {
  const PoseTpl* tpl;
  const uint16_t* crops;
  const int32_t* class_begin;
  int32_t n_classes, n_tpl;
};

struct PoseChunk {
  PoseTable table;
  const lm_match* surv;
  const int32_t* counts;
  int slots;
  int64_t first;    // the run's index of surv[0]
  const uint16_t* scene;
  const float* sK;
  IcpOut* outs;
  uint8_t* posed;
  PoseVerify* ver;  // o.verify.on: per survivor its verification
  int32_t* status;
  int32_t seq;
  // a batch's survivors' frames and the frames' intrinsics, and frame f's first survivor in the run (k_pose_pso's job
  // numbers); null: every survivor is of one frame
  const int32_t* frame_of = nullptr;
  const float* sKs = nullptr;
  const int32_t* frame_first = nullptr;
  // capture (unshared chunks; null: none): k_icp_normals' neighbour lists and the ICP kernel's correspondences, indexed
  // as the stage's points, and k_pose_pso's swarm records, record_words per slot
  int32_t* knn_out = nullptr;
  int32_t* corr_out = nullptr;
  long long* record = nullptr;
  int64_t record_words = 0;
  // a track chunk (lm_track; null: survivors): k_track_cloud builds the clouds from these objects instead of
  // k_pose_cloud; the stage's buffers, seg_begin / seg_end, jobs, err, posed, counts, rank, world, the scene and the
  // frame tables are filled in by pose_chunk.  Shared, its window records travel with the entries.
  const TrackParams* track = nullptr;
};

// k_pose_cloud, the segmented sort, k_pose_voxel, k_icp_normals (point-to-plane only) and the ICP kernel (or k_pose_pso,
// unshared only) over this rank's ceil(slots / world) slots, then (o.verify.on) k_pose_verify, then (shared) k_pose_collect.  A shared stage that
// verifies runs the ICP kernel's unshared instantiation into d_souts, and k_pose_verify<true> publishes.  Unshared, the cloud's posed flags and the ICP results
// go straight to the chunk's outputs; shared, to the stage's per-slot scratch, and k_pose_collect writes the outputs.
// Returns the chunk's launches (the sort counted once), or an error code (< 0).
static int pose_chunk(lm_pose_stage* s, const PoseOptions& o, const PoseChunk& c) {
  cudaStream_t st = o.stream;
  const PoseShare* sh = o.share;
  const int world = sh ? sh->world : 1;
  const int n = (c.slots + world - 1) / world;  // a rank without a survivor still publishes
  const int64_t A = pose_area(s);  // slot stride: the buffers' area, which may exceed the current largest crop
  PoseParams p;
  p.surv = c.surv; p.counts = c.counts;
  p.class_begin = c.table.class_begin; p.n_classes = c.table.n_classes; p.n_tpl = c.table.n_tpl;
  p.tpl = c.table.tpl; p.crops = c.table.crops;
  p.scene = c.scene; p.srows = o.srows; p.scols = o.scols;
  if (c.sK) memcpy(p.sK, c.sK, sizeof(p.sK));
  else memset(p.sK, 0, sizeof(p.sK));
  const bool pso = o.estimation == LM_POSE_PSO;
  p.A = (int32_t)A; p.use_scene = o.use_scene_cloud && !pso ? 1 : 0;  // the swarm registers against no target
  p.raw = s->d_raw.get(); p.cpts = s->d_cpts.get(); p.keys = s->d_keys[0].get(); p.vals = s->d_vals[0].get();
  p.seg_begin = s->d_seg.get(); p.seg_end = s->d_seg.get() + 2 * n;
  p.jobs = s->d_jobs.get(); p.err = c.status; p.posed = sh ? s->d_posed.get() : c.posed;
  p.frame_of = c.frame_of; p.sKs = c.sKs;
  p.rank = sh ? sh->rank : 0; p.world = world;
  int64_t items = 2 * n * A, tgt_max = A;  // points of the chunk's cloud slots, and of its largest target cloud
  if (c.track) {
    TrackParams q = *c.track;
    q.raw = p.raw; q.keys = p.keys; q.vals = p.vals; q.seg_begin = p.seg_begin; q.seg_end = p.seg_end;
    q.jobs = p.jobs; q.err = p.err; q.posed = p.posed;
    q.counts = c.counts; q.rank = p.rank; q.world = p.world;
    q.scene = c.scene; q.srows = o.srows; q.scols = o.scols; q.frame_of = c.frame_of; q.sKs = c.sKs;
    items = n * q.stride; tgt_max = q.cap;
    k_track_cloud<<<n, POSE_THREADS, 0, st>>>(q);
  } else {
    k_pose_cloud<<<n, POSE_THREADS, 0, st>>>(p);
  }
  // stable (radix) sort of each slot's keys: ties keep the point order, as std::stable_sort
  cub::DoubleBuffer<unsigned long long> dk(s->d_keys[0].get(), s->d_keys[1].get());
  cub::DoubleBuffer<int32_t> dv(s->d_vals[0].get(), s->d_vals[1].get());
  size_t tmp_bytes = s->d_sort_tmp.size();
  CUI(cub::DeviceSegmentedRadixSort::SortPairs(s->d_sort_tmp.get(), tmp_bytes, dk, dv, (int)items, 2 * n, p.seg_begin, p.seg_end, 0,
                                               3 * POSE_KEY_BITS, st));
  k_pose_voxel<<<2 * n, POSE_THREADS, 0, st>>>(dk.Current(), dv.Current(), p.seg_begin, p.seg_end, s->d_raw.get(), s->d_pts.get(), s->d_jobs.get(),
                                               p.use_scene);
  // the ICP kernels: empty jobs fall through
  const bool normals = o.estimation == LM_ICP_POINT_TO_PLANE;
  if (normals) {
    dim3 g((unsigned)((tgt_max + 127) / 128), (unsigned)n);
    k_icp_normals<<<g, 128, 0, st>>>(s->d_jobs.get(), s->d_pts.get(), s->d_nrm.get(), c.knn_out);
  }
  if (sh) {
    // the results travel to every rank; the collector gathers the chunk in survivor order
    PoseShareDev sd = share_dev(*sh, c.seq, c.counts, s->d_posed.get(), c.status);
    sd.rec = c.track ? c.track->rec : nullptr;  // a track chunk's window records travel with its entries
    if (o.verify.on) {  // the owner verifies (it holds the cloud), then publishes the pose and its verification
      launch_icp<false>(o.estimation, n, st, s->d_jobs.get(), s->d_pts.get(), s->d_nrm.get(), s->d_souts.get(), o.max_iterations, nullptr,
                        PoseShareDev());
      k_pose_verify<true><<<n, VERIFY_THREADS, 0, st>>>(p, s->d_souts.get(), o.verify.inlier_mm, nullptr, sd);
    } else {
      launch_icp<true>(o.estimation, n, st, s->d_jobs.get(), s->d_pts.get(), s->d_nrm.get(), nullptr, o.max_iterations, nullptr, sd);
    }
    k_pose_collect<<<1, POSE_COLLECT_THREADS, 0, st>>>(sd, c.outs, c.posed, o.verify.on ? c.ver : nullptr);
  } else {
    if (pso) {
      PsoParams q;
      memset(&q, 0, sizeof(q));
      q.jobs = s->d_jobs.get(); q.pts = s->d_pts.get(); q.outs = c.outs; q.n = n;
      q.scene = c.scene; q.srows = o.srows; q.scols = o.scols;
      memcpy(q.sK, p.sK, sizeof(q.sK));
      q.frame_of = c.frame_of; q.sKs = c.sKs; q.frame_first = c.frame_first; q.first = c.first;
      q.s = o.search;
      q.record = c.record; q.record_words = c.record_words;
      const int rc = launch_pso(q, st);
      if (rc) return rc;
    } else {
      launch_icp<false>(o.estimation, n, st, s->d_jobs.get(), s->d_pts.get(), s->d_nrm.get(), c.outs, o.max_iterations, c.corr_out,
                        PoseShareDev());
    }
    if (o.verify.on) k_pose_verify<false><<<n, VERIFY_THREADS, 0, st>>>(p, c.outs, o.verify.inlier_mm, c.ver, PoseShareDev());
  }
  CUI(cudaGetLastError());
  s->last.valid = true;
  s->last.slots = n; s->last.rank = p.rank; s->last.world = world;
  s->last.first = c.first;
  s->last.posed = p.posed;
  s->last.track = c.track != nullptr;
  return (sh ? 6 : 5) - (normals ? 0 : 1) + (o.verify.on ? 1 : 0);
}

int pose_stage_clouds(const lm_pose_stage* s, int slot, int what, void* out, int64_t cap) {
  if (!out) return lm_fail(LM_E_INVALID, "null argument");
  const auto& l = s->last;
  if (!l.valid) return lm_fail(LM_E_STATE, "no pose stage has run since the buffers last changed");
  int32_t head[4];
  uint8_t posed = 0;
  IcpJob j;
  int32_t seg[2] = {0, 0};
  const void* src = nullptr;
  int64_t bytes = 0;
  bool host = true;  // src is a host copy
  if (what == LM_POSE_CAPTURE_SLOTS) {
    if (slot != -1) return lm_fail(LM_E_INVALID, "LM_POSE_CAPTURE_SLOTS takes slot -1, not %d", slot);
    head[0] = l.slots; head[1] = l.rank; head[2] = l.world; head[3] = (int32_t)l.first;
    src = head; bytes = sizeof(head);
  } else {
    if (slot < 0 || slot >= l.slots) return lm_fail(LM_E_INVALID, "slot %d outside the %d of the last chunk", slot, l.slots);
    if (what != LM_POSE_CAPTURE_POSED && what != LM_ICP_CAPTURE_COUNTS && what != LM_ICP_CAPTURE_SOURCE &&
        what != LM_ICP_CAPTURE_TARGET && what != LM_ICP_CAPTURE_INIT && what != LM_POSE_CAPTURE_RAW_MODEL &&
        what != LM_POSE_CAPTURE_RAW_SCENE && what != LM_POSE_CAPTURE_WINDOW)
      return lm_fail(LM_E_INVALID, "unknown pose stage capture item %d", what);
    if (what == LM_POSE_CAPTURE_WINDOW && !l.track) return lm_fail(LM_E_STATE, "the last chunk was not a track chunk (lm_track): no window");
    CUI(cudaMemcpy(&posed, l.posed + slot, 1, cudaMemcpyDeviceToHost));
    if (what == LM_POSE_CAPTURE_WINDOW) {
      TrackRec rec;
      CUI(cudaMemcpy(&rec, s->d_trec.get() + l.first + l.rank + (int64_t)slot * l.world, sizeof(rec), cudaMemcpyDeviceToHost));
      const int32_t w5[5] = {rec.window[0], rec.window[1], rec.window[2], rec.window[3], rec.status};
      if (cap < (int64_t)sizeof(w5))
        return lm_fail(LM_E_CAPACITY, "pose stage capture item %d of slot %d needs %lld bytes, cap is %lld", what, slot, (long long)sizeof(w5),
                       (long long)cap);
      memcpy(out, w5, sizeof(w5));
      return LM_OK;
    }
    if (what == LM_POSE_CAPTURE_POSED) {
      src = &posed; bytes = 1;
    } else {
      if (!posed) return lm_fail(LM_E_STATE, "slot %d has no pose (no template, or its box leaves the frame): no cloud", slot);
      CUI(cudaMemcpy(&j, s->d_jobs.get() + slot, sizeof(j), cudaMemcpyDeviceToHost));
      const int k = 2 * slot + (what == LM_POSE_CAPTURE_RAW_SCENE ? 1 : 0);  // seg_end follows the chunk's 2 slots begins
      CUI(cudaMemcpy(&seg[0], s->d_seg.get() + k, sizeof(int32_t), cudaMemcpyDeviceToHost));
      CUI(cudaMemcpy(&seg[1], s->d_seg.get() + 2 * l.slots + k, sizeof(int32_t), cudaMemcpyDeviceToHost));
      switch (what) {
        case LM_ICP_CAPTURE_COUNTS:
          head[0] = j.src_count; head[1] = j.tgt_count;
          src = head; bytes = 2 * sizeof(int32_t);
          break;
        case LM_ICP_CAPTURE_SOURCE:
          src = s->d_pts.get() + (size_t)j.src_first * 3; bytes = (int64_t)j.src_count * 3 * sizeof(double); host = false;
          break;
        case LM_ICP_CAPTURE_TARGET:
          src = s->d_pts.get() + (size_t)j.tgt_first * 3; bytes = (int64_t)j.tgt_count * 3 * sizeof(double); host = false;
          break;
        case LM_ICP_CAPTURE_INIT:
          src = j.init; bytes = sizeof(j.init);
          break;
        default:  // RAW_MODEL, RAW_SCENE
          src = s->d_raw.get() + (size_t)seg[0] * 3; bytes = (int64_t)(seg[1] - seg[0]) * 3 * sizeof(double); host = false;
          break;
      }
    }
  }
  if (cap < bytes) return lm_fail(LM_E_CAPACITY, "pose stage capture item %d of slot %d needs %lld bytes, cap is %lld", what, slot,
                                  (long long)bytes, (long long)cap);
  if (bytes && host) memcpy(out, src, (size_t)bytes);
  if (bytes && !host) CUI(cudaMemcpy(out, src, (size_t)bytes, cudaMemcpyDeviceToHost));
  return LM_OK;
}

#define POSE_CHUNK 1024     // survivor slots per chunk: a frame's bound for top_k = 0
#define NMS_FIRST_FETCH 16

int pose_batch_chunks(int64_t S) { return (int)((S + POSE_CHUNK - 1) / POSE_CHUNK); }

// Chunk c of a run on the stage's registered renders and run outputs: survivors surv + c0 (c0 = c * POSE_CHUNK; counts
// as PoseChunk), launches for `slots` of them against the one frame scene / sK; its outputs, posed flags and verification
// from c0 on, status block c and pose exchange share->seq + c.
static PoseChunk run_chunk(lm_pose_stage* s, const PoseOptions& o, int c, const lm_match* surv, const int32_t* counts, int slots,
                           const uint16_t* scene, const float* sK) {
  const int64_t c0 = (int64_t)c * POSE_CHUNK;
  PoseChunk k;
  k.table = {s->d_tpl.get(), s->d_crops.get(), s->d_class_begin.get(), (int32_t)s->class_begin.size() - 1, (int32_t)s->tpl.size()};
  k.surv = surv ? surv + c0 : nullptr; k.counts = counts; k.slots = slots; k.first = c0;
  k.scene = scene; k.sK = sK;
  k.outs = s->d_bouts.get() + c0; k.posed = s->d_bposed.get() + c0; k.ver = o.verify.on ? s->d_bver.get() + c0 : nullptr;
  k.status = s->d_bstat.get() + 4 * c; k.seq = o.share ? o.share->seq + c : 0;
  return k;
}

// The pose NMS block of a run of n frames: the frames' heads, then the kept poses, frame f's from its first survivor.
// One copy thus brings back the heads and the first kept poses.
static PoseNmsHead* nms_heads(uint8_t* block) { return reinterpret_cast<PoseNmsHead*>(block); }
static PoseNmsOut* nms_out(uint8_t* block, int n) { return reinterpret_cast<PoseNmsOut*>(block + sizeof(PoseNmsHead) * n); }

// The outputs of a run of up to n_frames frames and S survivors.  Grow-only: an earlier run may still use them.
static int pose_outputs(lm_pose_stage* s, cudaStream_t st, int n_frames, int64_t S) {
  const size_t nms = sizeof(PoseNmsHead) * n_frames + sizeof(PoseNmsOut) * S;
  const bool frames = (size_t)4 * n_frames > s->h_bstat.size(), surv = (size_t)S > s->h_bouts.size(), block = nms > s->h_bnms.size();
  if (!frames && !surv && !block) return LM_OK;
  CUI(cudaStreamSynchronize(st));
  if (frames) {
    s->d_bfirst.reset(); s->d_bsK.reset(); s->d_bstat.reset(); s->h_bstat.reset();
    CUI(s->d_bfirst.assign(n_frames + 1));
    CUI(s->d_bsK.assign(9 * (size_t)n_frames));
    CUI(s->d_bstat.assign(4 * (size_t)n_frames));  // chunks <= frames: a frame has <= 1024 survivors
    CUI(s->h_bstat.assign(4 * (size_t)n_frames));
  }
  if (surv) {
    s->d_bframe.reset(); s->d_bouts.reset(); s->d_bposed.reset(); s->d_bksrc.reset(); s->h_bouts.reset();
    CUI(s->d_bframe.assign(S));
    CUI(s->d_bouts.assign(S));
    CUI(s->d_bposed.assign(S));
    CUI(s->d_bksrc.assign(S));
    CUI(s->h_bouts.assign(S));
  }
  if (block) {
    s->d_bnms.reset(); s->h_bnms.reset();
    CUI(s->d_bnms.assign(nms));
    CUI(s->h_bnms.assign(nms));
  }
  return LM_OK;
}

// The renders on the device and every buffer a run of n_frames frames and S survivors needs (verify: a verifying run's
// too).
static int pose_prepare(lm_pose_stage* s, cudaStream_t st, int n_frames, int64_t S, bool verify) {
  s->last.valid = false;
  s->done.stale = true;
  if (s->dirty) {
    int rc = pose_upload(s, st);
    if (rc) return rc;
  }
  S = std::max<int64_t>(S, 1);
  int rc = pose_outputs(s, st, n_frames, S);
  if (!rc) rc = pose_buffers(s, st, (int)std::min<int64_t>(S, POSE_CHUNK), s->area_max);
  if (rc || !verify) return rc;
  if ((size_t)S > s->h_bver.size()) {
    CUI(cudaStreamSynchronize(st));
    s->d_bver.reset(); s->d_bvkept.reset(); s->h_bver.reset();
    CUI(s->d_bver.assign(S));
    CUI(s->d_bvkept.assign(S));
    CUI(s->h_bver.assign(S));
  }
  if ((size_t)pose_slots(s) > s->d_souts.size()) {
    CUI(cudaStreamSynchronize(st));
    s->d_souts.reset();
    CUI(s->d_souts.assign(pose_slots(s)));
  }
  return LM_OK;
}

int pose_batch_reserve(lm_pose_stage* s, cudaStream_t st, int n_frames, int64_t frame_pixels, int64_t max_surv, bool verify,
                       uint16_t** d_scene, lm_match** d_surv) {
  const size_t pix = (size_t)n_frames * frame_pixels;
  if (pix > s->d_bscene.size() || (size_t)max_surv > s->d_bsurv.size()) {
    CUI(cudaStreamSynchronize(st));  // an earlier batch may still read them
    CUI(s->d_bscene.reserve(pix));
    CUI(s->d_bsurv.reserve((size_t)max_surv));
  }
  // and everything the run may need for max_surv survivors: once frames run, no device memory is freed (a free waits for
  // the whole device, a spinning peer collector of a shared batch included)
  int rc = pose_prepare(s, st, n_frames, max_surv, verify);
  if (rc) return rc;
  *d_scene = s->d_bscene.get();
  *d_surv = s->d_bsurv.get();
  return LM_OK;
}

// Entries of chunk c of a run of S entries.
static int chunk_size(int64_t S, int c) { return (int)std::min<int64_t>(S - (int64_t)c * POSE_CHUNK, POSE_CHUNK); }

// The tables a batch or track run's chunks read, on st: each entry's frame (entries of frame f: [first[f], first[f + 1])),
// each frame's intrinsics (sK + 9f), and each chunk's status block with its size in word 3.
static int run_tables(lm_pose_stage* s, cudaStream_t st, int nf, const int64_t* first, const float* sK) {
  const int64_t S = first[nf];
  const int nc = pose_batch_chunks(S);
  std::vector<int32_t> frame_of((size_t)S);
  for (int f = 0; f < nf; ++f)
    for (int64_t k = first[f]; k < first[f + 1]; ++k) frame_of[(size_t)k] = f;
  std::vector<int32_t> stat((size_t)4 * nc, 0);
  for (int c = 0; c < nc; ++c) stat[(size_t)4 * c + 3] = chunk_size(S, c);
  if (S) CUI(cudaMemcpyAsync(s->d_bframe.get(), frame_of.data(), sizeof(int32_t) * S, cudaMemcpyHostToDevice, st));
  CUI(cudaMemcpyAsync(s->d_bsK.get(), sK, sizeof(float) * 9 * nf, cudaMemcpyHostToDevice, st));
  if (nc) CUI(cudaMemcpyAsync(s->d_bstat.get(), stat.data(), sizeof(int32_t) * stat.size(), cudaMemcpyHostToDevice, st));
  return LM_OK;
}

int pose_stage_enqueue(lm_pose_stage* s, const PoseRun& run, int64_t* launches) {
  const PoseOptions& o = run.o;
  cudaStream_t st = o.stream;
  const PoseShare* sh = o.share;
  const bool batch = run.first != nullptr;
  const int nf = run.n_frames;
  const int64_t S = batch ? run.first[nf] : run.bound;  // survivors the outputs hold
  const int nc = batch ? pose_batch_chunks(S) : 1;
  if (sh && o.estimation == LM_POSE_PSO)
    return lm_fail(LM_E_STATE, "the pose stage shared over the ranks does not run LM_POSE_PSO: turn lm_peer_share_pose off");
  int rc = pose_prepare(s, st, nf, S, o.verify.on != 0);
  if (rc) return rc;
  if (batch) {
    rc = run_tables(s, st, nf, run.first, run.sK);
    if (rc) return rc;
    std::vector<int32_t> first32(run.first, run.first + nf + 1);  // each frame's first survivor (k_pose_nms, k_pose_pso)
    CUI(cudaMemcpyAsync(s->d_bfirst.get(), first32.data(), sizeof(int32_t) * (nf + 1), cudaMemcpyHostToDevice, st));
  } else {  // a frame's survivor count is the box NMS's
    CUI(cudaMemsetAsync(s->d_bstat.get(), 0, sizeof(int32_t) * 4, st));
  }
  int64_t stage_launches = 0;
  for (int c = 0; c < nc; ++c) {
    const int64_t c0 = (int64_t)c * POSE_CHUNK;
    PoseChunk k = run_chunk(s, o, c, run.d_surv, batch ? s->d_bstat.get() + 4 * c + 3 : run.d_counts,
                            batch ? chunk_size(S, c) : run.bound, run.d_scene, batch ? nullptr : run.sK);
    if (batch) { k.frame_of = s->d_bframe.get() + c0; k.sKs = s->d_bsK.get(); k.frame_first = s->d_bfirst.get(); }
    const int l = pose_chunk(s, o, k);
    if (l < 0) return l;
    stage_launches += l;
    *launches += l;
  }
  // the status blocks, and unless a pose NMS follows the ICP outputs: a batch's all, a frame's first window
  const int64_t fetch = run.pose_nms ? 0 : batch ? S : std::min(run.bound, POSE_FIRST_FETCH);
  if (fetch) CUI(cudaMemcpyAsync(s->h_bouts.get(), s->d_bouts.get(), sizeof(IcpOut) * fetch, cudaMemcpyDeviceToHost, st));
  if (fetch && o.verify.on) CUI(cudaMemcpyAsync(s->h_bver.get(), s->d_bver.get(), sizeof(PoseVerify) * fetch, cudaMemcpyDeviceToHost, st));
  if (nc) CUI(cudaMemcpyAsync(s->h_bstat.get(), s->d_bstat.get(), sizeof(int32_t) * 4 * nc, cudaMemcpyDeviceToHost, st));
  s->run = run;
  s->share = sh ? *sh : PoseShare();
  s->run.o.share = sh ? &s->share : nullptr;
  if (batch) s->first.assign(run.first, run.first + nf + 1);
  s->run.first = batch ? s->first.data() : nullptr;
  s->launches = stage_launches;
  s->fetched = fetch;
  return LM_OK;
}

int pose_stage_enqueue_nms(lm_pose_stage* s, double thr, int64_t* launches) {
  PoseRun& r = s->run;
  if (r.bound > NMS_THREADS) return lm_fail(LM_E_STATE, "pose stage launched for %d survivors, the pose NMS takes %d", r.bound, NMS_THREADS);
  const bool batch = r.first != nullptr;
  const int nf = r.n_frames;
  cudaStream_t st = r.o.stream;
  PoseNmsParams p;
  p.surv = r.d_surv; p.counts = batch ? nullptr : r.d_counts; p.posed = s->d_bposed.get(); p.outs = s->d_bouts.get();
  p.rt = s->d_rt.get(); p.class_begin = s->d_class_begin.get();
  p.thr = thr;
  p.head = nms_heads(s->d_bnms.get()); p.out = nms_out(s->d_bnms.get(), nf); p.src = s->d_bksrc.get();
  p.frame_first = batch ? s->d_bfirst.get() : nullptr;
  const PoseVerifyOptions& v = r.o.verify;
  p.ver = s->d_bver.get(); p.vout = s->d_bvkept.get(); p.rank_by = v.rank_by; p.min_score = v.min_score;
  if (v.on) k_pose_nms<true><<<nf, NMS_THREADS, 0, st>>>(p);
  else k_pose_nms<false><<<nf, NMS_THREADS, 0, st>>>(p);
  CUI(cudaGetLastError());
  ++*launches;
  // the heads and the kept poses (and their verification): a batch's all, a frame's first window
  r.pose_nms = 1;
  s->fetched = batch ? r.first[nf] : std::min(r.bound, NMS_FIRST_FETCH);
  CUI(cudaMemcpyAsync(s->h_bnms.get(), s->d_bnms.get(), sizeof(PoseNmsHead) * nf + sizeof(PoseNmsOut) * s->fetched, cudaMemcpyDeviceToHost, st));
  if (v.on) CUI(cudaMemcpyAsync(s->h_bver.get(), s->d_bvkept.get(), sizeof(PoseVerify) * s->fetched, cudaMemcpyDeviceToHost, st));
  return LM_OK;
}

// After the stream has been synchronised: the error of a run of n entries from its nb status blocks of 4 int32
// (PoseChunk), block c that of pose exchange sh->seq + c when shared (sh); a batch's message names the chunk.  Once they
// are clean, stats4 (may be null) gets what lm_pose_stats returns: n, the entries this rank published (unshared: n),
// the run's launches and 1 when shared.
static int pose_status(const int32_t* h, int nb, const PoseShare* sh, bool batch, int64_t n, int64_t launches, int64_t* stats4) {
  int32_t overflow = 0;
  int64_t published = 0;
  for (int c = 0; c < nb; ++c) {
    const int32_t* b = h + 4 * c;
    if (sh && b[1]) {
      if (batch)
        return lm_fail(LM_E_STATE, "pose exchange: a rank did not publish its poses of exchange %d (chunk %d of the batch) within %llu ms "
                       "(or an earlier collector on this device already gave up); every rank must run every batch while sharing is on",
                       sh->seq + c, c, sh->timeout_ns / 1000000ull);
      return lm_fail(LM_E_STATE, "pose exchange: a rank did not publish its poses of exchange %d within %llu ms (or an earlier collector "
                     "on this device already gave up); every rank must run the pose stage of every frame while sharing is on",
                     sh->seq + c, sh->timeout_ns / 1000000ull);
    }
    overflow |= b[0];
    if (sh) published += b[2];
  }
  if (overflow) return lm_fail(LM_E_INVALID, "pose stage: a cloud spans more than 2^%d voxels of 2.5 mm along an axis", POSE_KEY_BITS);
  if (stats4) {
    stats4[0] = n;
    stats4[1] = sh ? published : n;
    stats4[2] = launches;
    stats4[3] = sh ? 1 : 0;
  }
  return LM_OK;
}

// Survivor m's registered render, or null.
static const TplHost* survivor_render(const lm_pose_stage* s, const lm_match& m) {
  const int n_classes = (int)s->class_begin.size() - 1;
  const int64_t g = (m.class_index >= 0 && m.class_index < n_classes) ? (int64_t)s->class_begin[m.class_index] + m.template_id : -1;
  return (g >= 0 && g < (int64_t)s->tpl.size() && s->tpl[(size_t)g].set) ? &s->tpl[(size_t)g] : nullptr;
}

// LL.cpp:52-55: the reference returns early where the render's box, placed at the match, leaves the frame.
static bool survivor_fits(const TplHost& h, const lm_match& m, int srows, int scols) {
  return !(m.x + h.box[2] >= scols || m.y + h.box[3] >= srows);
}

// n kept poses e[] into the caller's arrays (out may be null).
static void copy_kept(const PoseNmsOut* e, int64_t n, lm_match* out, double* R_out, double* t_out, float* residual) {
  for (int64_t k = 0; k < n; ++k) {
    if (out) out[k] = e[k].m;
    memcpy(R_out + 9 * k, e[k].R, sizeof(e[k].R));
    memcpy(t_out + 3 * k, e[k].t, sizeof(e[k].t));
    residual[k] = e[k].residual;
  }
}

int pose_stage_finish(lm_pose_stage* s, const lm_match* surv, int64_t n, lm_match* out, double* R_out, double* t_out, float* residual,
                      int64_t cap, int64_t* n_out, int64_t* counts, int64_t* stats4) {
  const PoseRun& r = s->run;
  const PoseShare* sh = r.o.share;
  const bool batch = r.first != nullptr;
  const int nf = r.n_frames;
  const int64_t frame_first[2] = {0, n};
  const int64_t* first = batch ? r.first : frame_first;
  const int64_t S = first[nf];
  if (!batch && n > r.bound) return lm_fail(LM_E_STATE, "%lld survivors for a pose stage launched for %d", (long long)n, r.bound);
  const bool verify = r.o.verify.on != 0;
  PoseFinished& d = s->done;
  d.reset();
  int rc = pose_status(s->h_bstat.get(), batch ? pose_batch_chunks(S) : 1, sh, batch, S, s->launches, stats4);
  if (rc) return rc;
  const PoseNmsHead* heads = nms_heads(s->h_bnms.get());
  PoseNmsOut* entries = nms_out(s->h_bnms.get(), nf);
  int64_t total = 0, end = 0;  // entries, and the end of the host copy they need
  for (int f = 0; f < nf; ++f) {
    int64_t* fc = counts + 4 * f;
    if (r.pose_nms) {
      fc[0] = heads[f].kept; fc[1] = heads[f].survivors; fc[2] = heads[f].posed;
    } else {
      fc[0] = fc[1] = first[f + 1] - first[f];
      fc[2] = 0;
      for (int64_t i = first[f]; i < first[f + 1]; ++i) {
        const TplHost* h = survivor_render(s, surv[i]);
        if (!h && batch)
          return lm_fail(LM_E_STATE, "frame %d, survivor %lld: template without a registered render", f, (long long)(i - first[f]));
        if (!h) return lm_fail(LM_E_STATE, "survivor %lld: template without a registered render", (long long)i);
        if (survivor_fits(*h, surv[i], r.o.srows, r.o.scols)) ++fc[2];
      }
    }
    total += fc[0];
    end = std::max(end, first[f] + fc[0]);
  }
  *n_out = total;
  if (total > cap) {
    if (batch) return lm_fail(LM_E_CAPACITY, "%lld entries in the batch, capacity %lld", (long long)total, (long long)cap);
    return lm_fail(LM_E_CAPACITY, "%lld poses kept, capacity %lld", (long long)total, (long long)cap);
  }
  if (end > s->fetched) {  // a frame's entries beyond its first window
    cudaStream_t st = r.o.stream;
    if (verify)
      CUI(cudaMemcpyAsync(s->h_bver.get() + s->fetched, (r.pose_nms ? s->d_bvkept.get() : s->d_bver.get()) + s->fetched,
                          sizeof(PoseVerify) * (size_t)(end - s->fetched), cudaMemcpyDeviceToHost, st));
    if (r.pose_nms)
      CUI(cudaMemcpyAsync(entries + s->fetched, nms_out(s->d_bnms.get(), nf) + s->fetched, sizeof(PoseNmsOut) * (size_t)(end - s->fetched),
                          cudaMemcpyDeviceToHost, st));
    else
      CUI(cudaMemcpyAsync(s->h_bouts.get() + s->fetched, s->d_bouts.get() + s->fetched, sizeof(IcpOut) * (size_t)(end - s->fetched),
                          cudaMemcpyDeviceToHost, st));
    CUI(cudaStreamSynchronize(st));
  }
  if (r.pose_nms) {  // the kept poses' transformations stay on the device until pose_stage_transforms
    d.fill(PoseRunKind::kept, verify, s->h_bver.get(), 0);
    d.survivors = S;
    d.stream = r.o.stream;
    int64_t at = 0;
    for (int f = 0; f < nf; ++f) {
      copy_kept(entries + first[f], counts[4 * f], out ? out + at : nullptr, R_out + 9 * at, t_out + 3 * at, residual + at);
      if (verify) d.ver.insert(d.ver.end(), s->h_bver.get() + first[f], s->h_bver.get() + first[f] + counts[4 * f]);
      d.kept.emplace_back(first[f], counts[4 * f]);
      at += counts[4 * f];
    }
    return LM_OK;
  }
  d.fill(PoseRunKind::poses, verify, s->h_bver.get(), S);
  d.entries(S);
  for (int64_t i = 0; i < S; ++i) {  // every survivor, frame after frame; R / t untouched where the reference returns early
    if (out) out[i] = surv[i];
    const TplHost& h = *survivor_render(s, surv[i]);
    if (!survivor_fits(h, surv[i], r.o.srows, r.o.scols)) { residual[i] = -1.f; continue; }
    d.compose(i, s->h_bouts[i], h.R, h.t, R_out, t_out, residual);
  }
  return LM_OK;
}

// n verification results v[] into score[k] / counts6 + 6k (LM_E_CAPACITY beyond cap, *n written either way).
static int copy_verify(const PoseVerify* v, int64_t count, float* score, int32_t* counts6, int64_t cap, int64_t* n) {
  if (!n || (cap > 0 && (!score || !counts6))) return lm_fail(LM_E_INVALID, "null argument");
  *n = count;
  if (count > cap) return lm_fail(LM_E_CAPACITY, "%lld verified entries, capacity %lld", (long long)count, (long long)cap);
  for (int64_t k = 0; k < count; ++k) {
    score[k] = v[k].score;
    memcpy(counts6 + 6 * k, v[k].counts, sizeof(v[k].counts));
  }
  return LM_OK;
}

int pose_stage_verify(const lm_pose_stage* s, float* score, int32_t* counts6, int64_t cap, int64_t* n) {
  if (!s || !s->done.verified) return lm_fail(LM_E_STATE, "the last completed pose stage did not verify (lm_set_pose_verify, lm_icp_set_verify)");
  return copy_verify(s->done.ver.data(), (int64_t)s->done.ver.size(), score, counts6, cap, n);
}

extern "C" int lm_pose_verify_points(int device, const double* pts, int64_t n, const double* T, const uint16_t* scene, int rows,
                                     int cols, const float* sK, double inlier_mm, int32_t* counts6, float* score) {
  if (n < 0 || (n > 0 && !pts) || !T || !scene || !sK || !counts6 || !score) return lm_fail(LM_E_INVALID, "null argument or n < 0");
  if (rows <= 0 || cols <= 0) return lm_fail(LM_E_INVALID, "empty scene %d x %d", rows, cols);
  if (n > 0x7FFFFFFFll) return lm_fail(LM_E_CAPACITY, "%lld points, at most 2^31 - 1", (long long)n);
  int rc = check_inlier_mm(inlier_mm);
  if (!rc) rc = open_device(device);
  if (rc) return rc;
  // k_pose_verify over one slot: one allocation of pts [n][3], the pose (IcpOut), the segments (begin 0 at [0], end n at
  // [2]), the posed flag, the result and the scene [rows][cols]
  IcpOut o;
  memset(&o, 0, sizeof(o));
  memcpy(o.T, T, sizeof(o.T));
  const int32_t seg[4] = {0, 0, (int32_t)n, 0};
  const uint8_t posed = 1;
  const size_t o_out = sizeof(double) * 3 * (size_t)n, o_icp = o_out + sizeof(PoseVerify), o_seg = o_icp + sizeof(IcpOut);
  const size_t o_posed = o_seg + sizeof(seg), o_scene = o_posed + 16;
  DeviceArray<uint8_t> buf;
  CUI(buf.assign(o_scene + sizeof(uint16_t) * (size_t)rows * cols));
  uint8_t* b = buf.get();
  if (n > 0) CUI(cudaMemcpy(b, pts, o_out, cudaMemcpyHostToDevice));
  CUI(cudaMemcpy(b + o_icp, &o, sizeof(o), cudaMemcpyHostToDevice));
  CUI(cudaMemcpy(b + o_seg, seg, sizeof(seg), cudaMemcpyHostToDevice));
  CUI(cudaMemcpy(b + o_posed, &posed, 1, cudaMemcpyHostToDevice));
  CUI(cudaMemcpy(b + o_scene, scene, sizeof(uint16_t) * (size_t)rows * cols, cudaMemcpyHostToDevice));
  PoseParams p;
  memset(&p, 0, sizeof(p));
  p.scene = reinterpret_cast<const uint16_t*>(b + o_scene);
  p.srows = rows; p.scols = cols;
  memcpy(p.sK, sK, sizeof(p.sK));
  p.raw = reinterpret_cast<double*>(b);
  p.seg_begin = reinterpret_cast<int32_t*>(b + o_seg); p.seg_end = p.seg_begin + 2;
  p.posed = b + o_posed;
  p.rank = 0; p.world = 1;
  PoseVerify* d_out = reinterpret_cast<PoseVerify*>(b + o_out);
  k_pose_verify<false><<<1, VERIFY_THREADS>>>(p, reinterpret_cast<const IcpOut*>(b + o_icp), inlier_mm, d_out, PoseShareDev());
  CUI(cudaGetLastError());
  PoseVerify v;
  CUI(cudaMemcpy(&v, d_out, sizeof(v), cudaMemcpyDeviceToHost));
  memcpy(counts6, v.counts, sizeof(v.counts));
  *score = v.score;
  return LM_OK;
}

// View following on caller arrays (lm_track_views_points): k_track_views over one object of a one-class bank of n
// templates, every one with a render.
extern "C" int lm_track_views_points(int device, int64_t n, const float* R_b, const float* t_b, int64_t k, const double* T, double turn_deg,
                                     int64_t* chosen, double* T_out) {
  if (!R_b || !t_b || !T || !chosen || !T_out) return lm_fail(LM_E_INVALID, "null argument");
  if (n < 1 || n > 0x7FFFFFFFll) return lm_fail(LM_E_INVALID, "%lld templates, 1 to 2^31 - 1", (long long)n);
  if (k < 0 || k >= n) return lm_fail(LM_E_INVALID, "template %lld outside the %lld", (long long)k, (long long)n);
  for (int q = 0; q < 16; ++q)
    if (!std::isfinite(T[q])) return lm_fail(LM_E_INVALID, "T[%d] is not finite", q);
  double tau = 0.0;
  int rc = track_view_tau(1, turn_deg, &tau);
  if (!rc) rc = open_device(device);
  if (rc) return rc;
  std::vector<PoseRt> rt((size_t)n);
  for (int64_t j = 0; j < n; ++j) {
    memcpy(rt[(size_t)j].R, R_b + 9 * j, sizeof(rt[0].R));
    memcpy(rt[(size_t)j].t, t_b + 3 * j, sizeof(rt[0].t));
  }
  const std::vector<uint8_t> has((size_t)n, 1);
  const std::vector<int32_t> cb = {0, (int32_t)n, 1};  // class_begin, then the object count
  std::vector<TrackObject> obj(1);
  obj[0].g = k;
  memcpy(obj[0].T, T, sizeof(obj[0].T));
  DeviceArray<PoseRt> d_rt; DeviceArray<uint8_t> d_has; DeviceArray<int32_t> d_cb; DeviceArray<TrackObject> d_obj;
  CUI(upload(d_rt, rt, 0));
  CUI(upload(d_has, has, 0));
  CUI(upload(d_cb, cb, 0));
  CUI(upload(d_obj, obj, 0));
  TrackViewParams v;
  v.obj = d_obj.get(); v.counts = d_cb.get() + 2; v.rt = d_rt.get(); v.has = d_has.get(); v.class_begin = d_cb.get();
  v.n_classes = 1; v.tau = tau;
  k_track_views<<<1, VIEW_THREADS>>>(v);
  CUI(cudaGetLastError());
  CUI(cudaMemcpy(obj.data(), d_obj.get(), sizeof(TrackObject), cudaMemcpyDeviceToHost));
  *chosen = obj[0].g;
  memcpy(T_out, obj[0].T, sizeof(obj[0].T));
  return LM_OK;
}

// Steps 3-5 of the pose NMS on caller arrays (lm_nms_translations): the same device routine as k_pose_nms.
extern "C" int lm_nms_translations(int device, int64_t n, const double* t, const double* score, double thr, int32_t* keep,
                                   int64_t* n_keep) {
  if (!n_keep || n < 0 || (n > 0 && (!t || !score || !keep))) return lm_fail(LM_E_INVALID, "null argument or n < 0");
  if (!(thr >= 0.0)) return lm_fail(LM_E_INVALID, "translation threshold must be >= 0 (NaN given or negative)");
  if (n > NMS_THREADS) return lm_fail(LM_E_CAPACITY, "%lld translations, at most %d", (long long)n, NMS_THREADS);
  const int rc = open_device(device);
  if (rc) return rc;
  const size_t m = (size_t)std::max<int64_t>(n, 1);
  // one allocation: t [m][3], score [m], keep [m], n_keep
  DeviceArray<uint8_t> buf;
  CUI(buf.assign(sizeof(double) * 4 * m + sizeof(int32_t) * (m + 1)));
  double* d_t = reinterpret_cast<double*>(buf.get());
  double* d_s = d_t + 3 * m;
  int32_t* d_keep = reinterpret_cast<int32_t*>(d_s + m);
  int32_t* d_n = d_keep + m;
  if (n > 0) {
    CUI(cudaMemcpy(d_t, t, sizeof(double) * 3 * n, cudaMemcpyHostToDevice));
    CUI(cudaMemcpy(d_s, score, sizeof(double) * n, cudaMemcpyHostToDevice));
  }
  k_nms_translations<<<1, NMS_THREADS>>>((int)n, d_t, d_s, thr, d_keep, d_n);
  CUI(cudaGetLastError());
  int32_t got = 0;
  CUI(cudaMemcpy(&got, d_n, sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (got > 0) CUI(cudaMemcpy(keep, d_keep, sizeof(int32_t) * got, cudaMemcpyDeviceToHost));
  *n_keep = got;
  return LM_OK;
}

// --------------------------------------------------------------------------------------------
// lm_icp_process_batch_device: the pose stage's chunks fed from the caller's device planes (lm_pose.h)
// --------------------------------------------------------------------------------------------
#define ICP_DEV_PX 256       // threads of the scene and render kernels
#define RENDER_BOX_ROWS 16   // render rows per CTA of k_icp_render_box
#define RENDER_CROP_ROWS 8   // crop rows per CTA of k_icp_render_crop

struct RenderSrc {  // one render: the caller's plane, rows pitch bytes apart
  const uint8_t* p;
  int64_t pitch;
};

// The scene plane into the packed srows x scols u16 mm buffer k_pose_cloud reads.  CTA (bx, y): pixels
// [bx * ICP_DEV_PX, +ICP_DEV_PX) of row y.
__global__ void __launch_bounds__(ICP_DEV_PX) k_icp_scene(const uint8_t* __restrict__ src, int64_t pitch, int f32, float scale, int cols,
                                                         uint16_t* __restrict__ out) {
  const int y = blockIdx.y, x = blockIdx.x * ICP_DEV_PX + threadIdx.x;
  if (x < cols) out[(size_t)y * cols + x] = lm_depth_at(src + y * pitch, x, f32, scale);
}

// A caller's rows x cols depth plane (pitch bytes between rows, checked format and scale) into out on st.
static void launch_scene(const void* depth, int64_t pitch, int format, float scale, int rows, int cols, uint16_t* out, cudaStream_t st) {
  k_icp_scene<<<dim3((unsigned)((cols + ICP_DEV_PX - 1) / ICP_DEV_PX), (unsigned)rows), ICP_DEV_PX, 0, st>>>(
      static_cast<const uint8_t*>(depth), pitch, format == LM_DEPTH_F32 ? 1 : 0, scale, cols, out);
}

// The extent of render blockIdx.x's non-zero pixels (after conversion) over its rows [blockIdx.y * RENDER_BOX_ROWS,
// +RENDER_BOX_ROWS), merged into ext[4i ..]: min x, min y (unsigned, atomicMin), max x, max y (int, atomicMax), all bytes
// 0xFF before the launch (no pixel).  Exact in any order.
__global__ void __launch_bounds__(ICP_DEV_PX) k_icp_render_box(const RenderSrc* __restrict__ src, int f32, float scale, int mrows, int mcols,
                                                              uint32_t* __restrict__ ext) {
  const RenderSrc s = src[blockIdx.x];
  const int r0 = blockIdx.y * RENDER_BOX_ROWS, r1 = min(r0 + RENDER_BOX_ROWS, mrows);
  unsigned x0 = 0xFFFFFFFFu, y0 = 0xFFFFFFFFu;
  int x1 = -1, y1 = -1;
  for (int r = r0; r < r1; ++r) {
    const uint8_t* row = s.p + r * s.pitch;
    for (int q = threadIdx.x; q < mcols; q += ICP_DEV_PX)
      if (lm_depth_at(row, q, f32, scale) > 0) {
        x0 = min(x0, (unsigned)q); x1 = max(x1, q);
        y0 = min(y0, (unsigned)r); y1 = max(y1, r);
      }
  }
  x0 = __reduce_min_sync(0xffffffffu, x0); y0 = __reduce_min_sync(0xffffffffu, y0);
  x1 = __reduce_max_sync(0xffffffffu, x1); y1 = __reduce_max_sync(0xffffffffu, y1);
  if ((threadIdx.x & 31) == 0 && x1 >= 0) {
    uint32_t* e = ext + 4 * (size_t)blockIdx.x;
    atomicMin(e, x0); atomicMin(e + 1, y0);
    atomicMax(reinterpret_cast<int*>(e) + 2, x1); atomicMax(reinterpret_cast<int*>(e) + 3, y1);
  }
}

// Entry i = blockIdx.x of the call's table -- model_box's box grown from ext, the anchor render[mrows / 2][mcols / 2]
// and K -- and its crop rows [blockIdx.y * RENDER_CROP_ROWS, +RENDER_CROP_ROWS), packed at crops + i * stride.  A crop
// larger than stride is not written: the host sized stride for every hypothesis with a pose, so k_pose_cloud never reads it.
__global__ void __launch_bounds__(ICP_DEV_PX) k_icp_render_crop(const RenderSrc* __restrict__ src, int f32, float scale, int mrows, int mcols,
                                                               const uint32_t* __restrict__ ext, const float* __restrict__ K, int64_t stride,
                                                               PoseTpl* __restrict__ tpl, uint16_t* __restrict__ crops) {
  const int i = blockIdx.x;
  const RenderSrc s = src[i];
  const uint32_t* e = ext + 4 * (size_t)i;
  int box[4];
  grow_box((int)e[0], (int)e[1], (int)e[2], (int)e[3], mrows, mcols, box);
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    PoseTpl t;
    t.bx = box[0]; t.by = box[1]; t.bw = box[2]; t.bh = box[3];
    t.crop = (int64_t)i * stride;
    for (int k = 0; k < 9; ++k) t.K[k] = K[9 * i + k];
    t.anchor = lm_depth_at(s.p + (mrows / 2) * s.pitch, mcols / 2, f32, scale);
    tpl[i] = t;
  }
  const int bw = box[2], r1 = min((int)(blockIdx.y + 1) * RENDER_CROP_ROWS, box[3]);
  if ((int64_t)bw * box[3] > stride) return;
  uint16_t* __restrict__ C = crops + (size_t)i * stride;
  for (int r = blockIdx.y * RENDER_CROP_ROWS; r < r1; ++r) {
    const uint8_t* row = s.p + (box[1] + r) * s.pitch;
    for (int q = threadIdx.x; q < bw; q += ICP_DEV_PX) C[(size_t)r * bw + q] = lm_depth_at(row, box[0] + q, f32, scale);
  }
}

struct IcpDevice {
  lm_pose_stage stage;  // the chunks' buffers and run outputs, and the call's render table and crops in d_tpl / d_crops
  PinnedArray<uint16_t> h_planes; DeviceArray<uint16_t> planes;  // lm_icp_process_batch: the scene, then each distinct render
  DeviceArray<uint8_t> in;  // the call's inputs in one copy: renders, K, survivors, chunk sizes, class_begin
  DeviceArray<uint16_t> scene;
  DeviceArray<uint32_t> ext; PinnedArray<uint32_t> h_ext;  // [n][4] extents (k_icp_render_box)
  DeviceArray<int32_t> knn, corr; DeviceArray<long long> record;  // lm_icp_set_capture: the chunk's (PoseChunk)
};

static IcpDevice* icp_device_new() { return new IcpDevice(); }
static void icp_device_free(IcpDevice* d) { delete d; }

extern "C" int lm_icp_verify(lm_icp* h, float* score, int32_t* counts6, int64_t cap, int64_t* n) {
  if (!h) return lm_fail(LM_E_INVALID, "null handle");
  return pose_stage_verify(&h->dev->stage, score, counts6, cap, n);
}

extern "C" int lm_icp_capture(lm_icp* h, int hyp, int what, void* out, int64_t cap) {
  if (!h || !out) return lm_fail(LM_E_INVALID, "null argument");
  const auto& c = h->cap;
  if (hyp < 0 || hyp >= (int)c.job_of.size())
    return lm_fail(LM_E_INVALID, "hypothesis %d outside the %d of the last captured call", hyp, (int)c.job_of.size());
  if (c.job_of[hyp] < 0) return lm_fail(LM_E_STATE, "hypothesis %d took the early return: nothing was captured", hyp);
  const IcpJob& j = c.jobs[(size_t)c.job_of[hyp]];
  const IcpOut& o = c.outs[(size_t)c.job_of[hyp]];
  const void* src = nullptr;
  int64_t bytes = 0;
  std::vector<int32_t> tmp;
  double res[19];
  if (c.estimation == LM_POSE_PSO && (what == LM_ICP_CAPTURE_NORMALS || what == LM_ICP_CAPTURE_KNN || what == LM_ICP_CAPTURE_CORR_FIRST ||
                                       what == LM_ICP_CAPTURE_CORR_LAST))
    return lm_fail(LM_E_STATE, "capture item %d: the particle swarm computes no normals, neighbour lists or correspondences", what);
  if ((what == LM_ICP_CAPTURE_NORMALS || what == LM_ICP_CAPTURE_KNN) && c.estimation != LM_ICP_POINT_TO_PLANE)
    return lm_fail(LM_E_STATE, "capture item %d: the point-to-point estimation computes no normals or neighbour lists", what);
  if (what == LM_ICP_CAPTURE_SEARCH && c.estimation != LM_POSE_PSO)
    return lm_fail(LM_E_STATE, "capture item %d: only an LM_POSE_PSO call keeps swarm records", what);
  switch (what) {
    case LM_ICP_CAPTURE_COUNTS:
      tmp = {j.src_count, j.tgt_count};
      src = tmp.data(); bytes = 2 * sizeof(int32_t);
      break;
    case LM_ICP_CAPTURE_SOURCE:
      src = c.pts.data() + (size_t)j.src_first * 3; bytes = (int64_t)j.src_count * 3 * sizeof(double);
      break;
    case LM_ICP_CAPTURE_TARGET:
      src = c.pts.data() + (size_t)j.tgt_first * 3; bytes = (int64_t)j.tgt_count * 3 * sizeof(double);
      break;
    case LM_ICP_CAPTURE_NORMALS:
      src = c.nrm.data() + (size_t)j.tgt_first * 3; bytes = (int64_t)j.tgt_count * 3 * sizeof(double);
      break;
    case LM_ICP_CAPTURE_INIT:
      src = j.init; bytes = sizeof(j.init);
      break;
    case LM_ICP_CAPTURE_RESULT:
      memcpy(res, o.T, sizeof(o.T));
      res[16] = o.fitness; res[17] = o.rmse; res[18] = o.iterations;
      src = res; bytes = sizeof(res);
      break;
    case LM_ICP_CAPTURE_SEARCH:
      src = c.record.data() + (size_t)c.job_of[hyp] * c.record_words; bytes = c.record_words * (int64_t)sizeof(long long);
      break;
    case LM_ICP_CAPTURE_KNN:
      src = c.knn.data() + (size_t)j.tgt_first * ICP_KNN; bytes = (int64_t)j.tgt_count * ICP_KNN * sizeof(int32_t);
      break;
    case LM_ICP_CAPTURE_CORR_FIRST:
    case LM_ICP_CAPTURE_CORR_LAST: {
      // slot 1 holds the last pass after any update; without one, pass 0 was the last pass
      const int slot = (what == LM_ICP_CAPTURE_CORR_LAST && o.iterations > 0) ? 1 : 0;
      tmp.resize((size_t)j.src_count);
      for (int i = 0; i < j.src_count; ++i) tmp[(size_t)i] = c.corr[((size_t)j.src_first + i) * 2 + slot];
      src = tmp.data(); bytes = (int64_t)j.src_count * sizeof(int32_t);
      break;
    }
    default:
      return lm_fail(LM_E_INVALID, "unknown capture item %d", what);
  }
  if (cap < bytes) return lm_fail(LM_E_CAPACITY, "capture item %d of hypothesis %d needs %lld bytes, cap is %lld", what, hyp,
                                  (long long)bytes, (long long)cap);
  if (bytes) memcpy(out, src, (size_t)bytes);
  return LM_OK;
}

// The capture of the chunk of hypotheses [c0, c0 + n) behind it, before the next chunk reuses the buffers: each posed
// hypothesis's job, its clouds with their normals, neighbour lists and correspondences, and its swarm record, appended
// to cap in the stage's point order.
static int icp_capture_chunk(const IcpDevice& d, cudaStream_t st, int c0, int n, const uint8_t* posed, IcpCapture& cap) {
  const lm_pose_stage& s = d.stage;
  const bool pso = cap.estimation == LM_POSE_PSO, normals = cap.estimation == LM_ICP_POINT_TO_PLANE;
  const int64_t words = cap.record_words;
  CUI(cudaStreamSynchronize(st));
  std::vector<IcpJob> jobs((size_t)n);
  CUI(cudaMemcpy(jobs.data(), s.d_jobs.get(), sizeof(IcpJob) * jobs.size(), cudaMemcpyDeviceToHost));
  // points [first, first + count) of the stage's clouds, with their normals, neighbour lists and correspondences
  auto append = [&](int32_t first, int32_t count) {
    const size_t at = cap.pts.size() / 3, m = (size_t)count;
    cap.pts.resize(3 * (at + m));
    if (normals) { cap.nrm.resize(3 * (at + m)); cap.knn.resize(ICP_KNN * (at + m)); }
    if (!pso) cap.corr.resize(2 * (at + m));
    if (!m) return LM_OK;
    CUI(cudaMemcpy(cap.pts.data() + 3 * at, s.d_pts.get() + 3 * (size_t)first, sizeof(double) * 3 * m, cudaMemcpyDeviceToHost));
    if (normals) {
      CUI(cudaMemcpy(cap.nrm.data() + 3 * at, s.d_nrm.get() + 3 * (size_t)first, sizeof(double) * 3 * m, cudaMemcpyDeviceToHost));
      CUI(cudaMemcpy(cap.knn.data() + ICP_KNN * at, d.knn.get() + ICP_KNN * (size_t)first, sizeof(int32_t) * ICP_KNN * m,
                     cudaMemcpyDeviceToHost));
    }
    if (!pso) CUI(cudaMemcpy(cap.corr.data() + 2 * at, d.corr.get() + 2 * (size_t)first, sizeof(int32_t) * 2 * m, cudaMemcpyDeviceToHost));
    return LM_OK;
  };
  for (int i = 0; i < n; ++i) {
    if (!posed[i]) continue;
    IcpJob j = jobs[(size_t)i];
    const bool own_target = j.tgt_first != j.src_first;
    const int32_t src_at = (int32_t)(cap.pts.size() / 3);
    int rc = append(j.src_first, j.src_count);
    if (!rc && own_target) {
      const int32_t tgt_at = (int32_t)(cap.pts.size() / 3);
      rc = append(j.tgt_first, j.tgt_count);
      j.tgt_first = tgt_at;
    } else {
      j.tgt_first = src_at;
    }
    if (rc) return rc;
    j.src_first = src_at;
    if (pso) {
      cap.record.resize(cap.record.size() + (size_t)words);
      CUI(cudaMemcpy(cap.record.data() + cap.record.size() - words, d.record.get() + (size_t)i * words, sizeof(long long) * words,
                     cudaMemcpyDeviceToHost));
    }
    cap.job_of[(size_t)(c0 + i)] = (int)cap.jobs.size();
    cap.jobs.push_back(j);
  }
  return LM_OK;
}

static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// A call without hypotheses: no device work; it verified nothing (an empty verification) and captured nothing.
static int icp_no_hypotheses(lm_icp* h) {
  h->dev->stage.done.reset();
  h->dev->stage.done.fill(PoseRunKind::icp, h->verify, nullptr, 0);
  h->cap.job_of.clear();
  return LM_OK;
}

// lm_icp_process_batch and lm_icp_process_batch_device past their checks: n >= 1 hypotheses, the scene and renders[i] in
// device memory as lm_icp_process_batch_device takes them, on the handle's stream behind the caller's ev0.  A run of the
// handle's stage whose table holds the call's renders.  Returns once the outputs are on the host.
static int icp_batch(lm_icp* h, int n, const void* scene_depth, int64_t scene_pitch, int scene_format, float scene_scale, int srows,
                     int scols, const RenderSrc* renders, int model_format, float model_scale, int mrows, int mcols,
                     const float* sceneK, const float* modelK, const float* R, const float* t, const int32_t* detect_xy,
                     int max_iterations, double* R_out, double* t_out, float* residual) {
  IcpDevice& d = *h->dev;
  lm_pose_stage* s = &d.stage;
  s->done.reset();
  h->cap.job_of.clear();  // a call that fails keeps no capture
  cudaStream_t st = h->stream.get();
  IcpCapture cap;  // kept only when the call succeeds
  cap.estimation = h->estimation;
  cap.job_of.assign((size_t)n, -1);
  cap.record_words = pso_record_words(h->search);
  const int nc = pose_batch_chunks(n);
  // the inputs: survivor i is hypothesis i (class 0, template i) at detect_xy[i]; chunk c holds min(n - 1024 c, 1024)
  const size_t o_K = align16(sizeof(RenderSrc) * n), o_surv = align16(o_K + sizeof(float) * 9 * n);
  const size_t o_cnt = align16(o_surv + sizeof(lm_match) * n), o_cb = align16(o_cnt + sizeof(int32_t) * nc);
  std::vector<uint8_t> in(o_cb + 2 * sizeof(int32_t));
  lm_match* surv = reinterpret_cast<lm_match*>(in.data() + o_surv);
  int32_t* cnt = reinterpret_cast<int32_t*>(in.data() + o_cnt);
  memcpy(in.data(), renders, sizeof(RenderSrc) * n);
  for (int i = 0; i < n; ++i) surv[i] = {detect_xy[2 * i], detect_xy[2 * i + 1], 0.f, 0, i};
  memcpy(in.data() + o_K, modelK, sizeof(float) * 9 * n);
  for (int c = 0; c < nc; ++c) cnt[c] = std::min(n - c * POSE_CHUNK, POSE_CHUNK);
  const int32_t class_begin[2] = {0, n};
  memcpy(in.data() + o_cb, class_begin, sizeof(class_begin));
  // grow-only: a call of the same shape allocates nothing (the handle's stream is idle between calls)
  CUI(d.in.reserve(in.size()));
  CUI(d.scene.reserve((size_t)srows * scols));
  CUI(d.ext.reserve(4 * (size_t)n)); CUI(d.h_ext.reserve(4 * (size_t)n));
  CUI(s->d_tpl.reserve(n));
  const RenderSrc* d_src = reinterpret_cast<const RenderSrc*>(d.in.get());
  const float* d_K = reinterpret_cast<const float*>(d.in.get() + o_K);
  const int f32 = model_format == LM_DEPTH_F32 ? 1 : 0;
  CUI(cudaMemcpyAsync(d.in.get(), in.data(), in.size(), cudaMemcpyHostToDevice, st));
  CUI(cudaMemsetAsync(d.ext.get(), 0xFF, sizeof(uint32_t) * 4 * n, st));
  launch_scene(scene_depth, scene_pitch, scene_format, scene_scale, srows, scols, d.scene.get(), st);
  k_icp_render_box<<<dim3((unsigned)n, (unsigned)((mrows + RENDER_BOX_ROWS - 1) / RENDER_BOX_ROWS)), ICP_DEV_PX, 0, st>>>(
      d_src, f32, model_scale, mrows, mcols, d.ext.get());
  CUI(cudaGetLastError());
  h->launches += 2;
  // the one read-back: the boxes size the crops and the clouds' slots
  CUI(cudaMemcpyAsync(d.h_ext.get(), d.ext.get(), sizeof(uint32_t) * 4 * n, cudaMemcpyDeviceToHost, st));
  CUI(cudaStreamSynchronize(st));
  std::vector<uint8_t> posed((size_t)n);
  int64_t stride = 1;
  int max_bh = 1, last = -1;
  for (int i = 0; i < n; ++i) {
    const uint32_t* e = d.h_ext.get() + 4 * (size_t)i;
    int b[4];
    grow_box((int)e[0], (int)e[1], (int)e[2], (int)e[3], mrows, mcols, b);
    if ((int64_t)b[2] * b[3] >= (1ll << POSE_KEY_BITS))
      return lm_fail(LM_E_INVALID, "model_depths[%d]: box of %d x %d pixels is too large", i, b[2], b[3]);
    posed[(size_t)i] = !(detect_xy[2 * i] + b[2] >= scols || detect_xy[2 * i + 1] + b[3] >= srows);  // LL.cpp:52-55
    if (!posed[(size_t)i]) continue;
    stride = std::max<int64_t>(stride, (int64_t)b[2] * b[3]);
    max_bh = std::max(max_bh, b[3]);
    last = i;
  }
  if (last < 0) {  // every hypothesis takes the early return: no cloud to build, and every verification scores -1
    for (int i = 0; i < n; ++i) residual[i] = -1.f;
    std::vector<PoseVerify> none(h->verify ? (size_t)n : 0, PoseVerify());
    for (PoseVerify& v : none) v.score = -1.f;
    s->done.fill(PoseRunKind::icp, h->verify, none.data(), n);
    if (h->capture) h->cap = std::move(cap);
    return LM_OK;
  }
  // the run's buffers: clouds of the largest crop, and status blocks for the chunks and one more, whose first word
  // receives the source count of the last hypothesis with a pose
  s->area_max = stride;
  int rc = pose_prepare(s, st, nc + 1, n, h->verify);
  if (rc) return rc;
  CUI(s->d_crops.reserve((size_t)n * stride));
  if (h->capture) {  // the chunks' capture outputs, indexed as the stage's points and slots
    const size_t points = 2 * (size_t)pose_slots(s) * (size_t)pose_area(s);
    if (cap.estimation == LM_ICP_POINT_TO_PLANE) CUI(d.knn.reserve(points * ICP_KNN));
    if (cap.estimation != LM_POSE_PSO) CUI(d.corr.reserve(points * 2));
    else CUI(d.record.reserve((size_t)pose_slots(s) * cap.record_words));
  }
  k_icp_render_crop<<<dim3((unsigned)n, (unsigned)((max_bh + RENDER_CROP_ROWS - 1) / RENDER_CROP_ROWS)), ICP_DEV_PX, 0, st>>>(
      d_src, f32, model_scale, mrows, mcols, d.ext.get(), d_K, stride, s->d_tpl.get(), s->d_crops.get());
  CUI(cudaGetLastError());
  ++h->launches;
  CUI(cudaMemsetAsync(s->d_bstat.get(), 0, sizeof(int32_t) * 4 * nc, st));
  const PoseOptions o = {srows, scols, h->use_scene_cloud ? 1 : 0, max_iterations, h->estimation, st, nullptr,
                         {h->verify ? 1 : 0, LM_VERIFY_RANK_FITNESS, h->verify_mm, -INFINITY}, h->search};
  const PoseTable table = {s->d_tpl.get(), s->d_crops.get(), reinterpret_cast<const int32_t*>(d.in.get() + o_cb), 1, n};
  const lm_match* d_surv = reinterpret_cast<const lm_match*>(d.in.get() + o_surv);
  const int32_t* d_cnt = reinterpret_cast<const int32_t*>(d.in.get() + o_cnt);
  for (int c = 0; c < nc; ++c) {
    const int c0 = c * POSE_CHUNK;
    PoseChunk k = run_chunk(s, o, c, d_surv, d_cnt + c, cnt[c], d.scene.get(), sceneK);
    k.table = table;
    if (h->capture) {
      k.knn_out = d.knn.get(); k.corr_out = d.corr.get();
      k.record = d.record.get(); k.record_words = cap.record_words;
    }
    const int l = pose_chunk(s, o, k);
    if (l < 0) return l;
    h->launches += l;
    if (last >= c0 && last < c0 + cnt[c])  // the chunk's jobs are overwritten by the next chunk's
      CUI(cudaMemcpyAsync(s->h_bstat.get() + 4 * nc, &s->d_jobs.get()[last - c0].src_count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (h->capture) {
      rc = icp_capture_chunk(d, st, c0, cnt[c], posed.data() + c0, cap);
      if (rc) return rc;
    }
  }
  CUI(cudaEventRecord(h->ev1.get(), st));
  CUI(cudaMemcpyAsync(s->h_bouts.get(), s->d_bouts.get(), sizeof(IcpOut) * n, cudaMemcpyDeviceToHost, st));
  CUI(cudaMemcpyAsync(s->h_bstat.get(), s->d_bstat.get(), sizeof(int32_t) * 4 * nc, cudaMemcpyDeviceToHost, st));
  if (h->verify) CUI(cudaMemcpyAsync(s->h_bver.get(), s->d_bver.get(), sizeof(PoseVerify) * n, cudaMemcpyDeviceToHost, st));
  CUI(cudaStreamSynchronize(st));
  CUI(cudaGetLastError());
  float ms = 0;
  CUI(cudaEventElapsedTime(&ms, h->ev0.get(), h->ev1.get()));
  h->last_kernel_us = ms * 1000.f;
  rc = pose_status(s->h_bstat.get(), nc, nullptr, false, n, 0, nullptr);
  if (rc) return rc;
  s->done.fill(PoseRunKind::icp, h->verify, s->h_bver.get(), n);
  for (int i = 0; i < n; ++i) {
    if (posed[(size_t)i]) render_pose(s->h_bouts[(size_t)i], R + 9 * i, t + 3 * i, R_out + 9 * i, t_out + 3 * i, residual + i);
    else residual[i] = -1.f;
  }
  if (h->capture) {
    for (int i = 0; i < n; ++i)
      if (cap.job_of[(size_t)i] >= 0) cap.outs.push_back(s->h_bouts[(size_t)i]);
    h->cap = std::move(cap);
  }
  h->last_points = s->h_bstat[4 * (size_t)nc];
  h->last_iterations = s->h_bouts[(size_t)last].iterations;
  h->last_rmse = s->h_bouts[(size_t)last].rmse;
  return LM_OK;
}

// Batch of hypotheses against one scene depth image.  For hypothesis h: model_depths[h] (mrows x mcols
// u16), modelK + 9h, R + 9h, t + 3h, detect_xy[2h..2h+1].  Outputs R_out + 9h (row-major f64),
// t_out + 3h (mm), residual[h] (fitness; -1 on the early return of LL.cpp:52-55, outputs untouched).
extern "C" int lm_icp_process_batch(lm_icp* h, int n_hyp, const uint16_t* scene_depth, int srows, int scols,
                                    const uint16_t* const* model_depths, int mrows, int mcols, const float* sceneK,
                                    const float* modelK, const float* R, const float* t, const int32_t* detect_xy,
                                    int max_iterations, double* R_out, double* t_out, float* residual) {
  if (!h || n_hyp < 0 || !scene_depth || !model_depths || !sceneK || !modelK || !R || !t || !detect_xy || !R_out || !t_out || !residual)
    return lm_fail(LM_E_INVALID, "null argument");
  if (srows <= 0 || scols <= 0 || mrows <= 0 || mcols <= 0) return lm_fail(LM_E_INVALID, "empty image");
  if (max_iterations < 0) return lm_fail(LM_E_INVALID, "max_iterations < 0");
  for (int i = 0; i < n_hyp; ++i)
    if (!model_depths[i]) return lm_fail(LM_E_INVALID, "model_depths[%d] is null", i);
  if (n_hyp == 0) return icp_no_hypotheses(h);
  CUI(cudaSetDevice(h->device));
  // the scene, then each distinct render once (callers repeat one render for many hypotheses), staged and copied in one
  const size_t npix = (size_t)srows * scols, mpix = (size_t)mrows * mcols;
  std::unordered_map<const uint16_t*, size_t> plane_of;
  std::vector<size_t> at((size_t)n_hyp);
  for (int i = 0; i < n_hyp; ++i)
    at[(size_t)i] = plane_of.emplace(model_depths[i], npix + mpix * plane_of.size()).first->second;
  const size_t total = npix + mpix * plane_of.size();
  IcpDevice& d = *h->dev;
  CUI(d.h_planes.reserve(total));
  CUI(d.planes.reserve(total));
  memcpy(d.h_planes.get(), scene_depth, sizeof(uint16_t) * npix);
  for (const auto& p : plane_of) memcpy(d.h_planes.get() + p.second, p.first, sizeof(uint16_t) * mpix);
  std::vector<RenderSrc> src((size_t)n_hyp);
  for (int i = 0; i < n_hyp; ++i) src[(size_t)i] = {reinterpret_cast<const uint8_t*>(d.planes.get() + at[(size_t)i]), 2 * (int64_t)mcols};
  cudaStream_t st = h->stream.get();
  CUI(cudaEventRecord(h->ev0.get(), st));
  CUI(cudaMemcpyAsync(d.planes.get(), d.h_planes.get(), sizeof(uint16_t) * total, cudaMemcpyHostToDevice, st));
  return icp_batch(h, n_hyp, d.planes.get(), 2 * (int64_t)scols, LM_DEPTH_U16_MM, 1.f, srows, scols, src.data(), LM_DEPTH_U16_MM, 1.f,
                   mrows, mcols, sceneK, modelK, R, t, detect_xy, max_iterations, R_out, t_out, residual);
}

extern "C" int lm_icp_process_batch_device(lm_icp* h, int n_hyp, const void* scene_depth, int64_t scene_pitch, int scene_format,
                                           float scene_scale, int srows, int scols, const void* const* model_depths,
                                           const int64_t* model_pitches, int model_format, float model_scale, int mrows, int mcols,
                                           const float* sceneK, const float* modelK, const float* R, const float* t,
                                           const int32_t* detect_xy, int max_iterations, double* R_out, double* t_out, float* residual,
                                           void* stream) {
  if (!h || n_hyp < 0 || !scene_depth || !model_depths || !model_pitches || !sceneK || !modelK || !R || !t || !detect_xy || !R_out ||
      !t_out || !residual)
    return lm_fail(LM_E_INVALID, "null argument");
  if (srows <= 0 || scols <= 0 || mrows <= 0 || mcols <= 0) return lm_fail(LM_E_INVALID, "empty image");
  if (max_iterations < 0) return lm_fail(LM_E_INVALID, "max_iterations < 0");
  int rc = check_depth_format("scene_depth", scene_format, scene_scale);
  if (!rc) rc = check_depth_format("model_depths", model_format, model_scale);
  if (rc) return rc;
  cudaStream_t caller = (cudaStream_t)stream;
  rc = check_device_stream(h->device, caller);
  const int sz = scene_format == LM_DEPTH_F32 ? 4 : 2, mz = model_format == LM_DEPTH_F32 ? 4 : 2;
  if (!rc) rc = check_device_plane(h->device, "scene_depth", scene_depth, scene_pitch, (int64_t)sz * scols, sz);
  for (int i = 0; i < n_hyp && !rc; ++i) {
    char what[40];
    snprintf(what, sizeof(what), "model_depths[%d]", i);
    rc = check_device_plane(h->device, what, model_depths[i], model_pitches[i], (int64_t)mz * mcols, mz);
  }
  if (rc) return rc;
  if (n_hyp == 0) return icp_no_hypotheses(h);
  std::vector<RenderSrc> src((size_t)n_hyp);
  for (int i = 0; i < n_hyp; ++i) src[(size_t)i] = {static_cast<const uint8_t*>(model_depths[i]), model_pitches[i]};
  CUI(cudaSetDevice(h->device));
  // the reads of the caller's planes start behind its stream's work, and its later work waits for the call's
  cudaStream_t st = h->stream.get();
  CUI(cudaEventRecord(h->ev_in.get(), caller));
  CUI(cudaStreamWaitEvent(st, h->ev_in.get(), 0));
  CUI(cudaEventRecord(h->ev0.get(), st));
  rc = icp_batch(h, n_hyp, scene_depth, scene_pitch, scene_format, scene_scale, srows, scols, src.data(), model_format, model_scale,
                 mrows, mcols, sceneK, modelK, R, t, detect_xy, max_iterations, R_out, t_out, residual);
  CUI(cudaEventRecord(h->ev_out.get(), st));
  CUI(cudaStreamWaitEvent(caller, h->ev_out.get(), 0));
  return rc;
}

// --------------------------------------------------------------------------------------------
// tracking on the detector's pose stage (lm_track, lm_track_device, lm_track_batch, lm_track_batch_device) and the
// transformations of a finished run
// --------------------------------------------------------------------------------------------
int pose_track_scene(lm_pose_stage* s, cudaStream_t st, int n_frames, const uint16_t* host, const void* const* planes, int64_t pitch,
                     int format, float scale, int rows, int cols, const uint16_t** d_scene, int64_t* launches) {
  const size_t npix = (size_t)rows * cols;
  if ((size_t)n_frames * npix > s->d_bscene.size()) {
    CUI(cudaStreamSynchronize(st));  // an earlier run may still read it
    CUI(s->d_bscene.reserve((size_t)n_frames * npix));
  }
  if (host) {
    CUI(cudaMemcpyAsync(s->d_bscene.get(), host, sizeof(uint16_t) * n_frames * npix, cudaMemcpyHostToDevice, st));
  } else {
    for (int f = 0; f < n_frames; ++f) launch_scene(planes[f], pitch, format, scale, rows, cols, s->d_bscene.get() + f * npix, st);
    CUI(cudaGetLastError());
    *launches += n_frames;
  }
  *d_scene = s->d_bscene.get();
  return LM_OK;
}

int pose_stage_track(lm_pose_stage* s, const PoseOptions& o, int n_frames, const uint16_t* d_scene, const float* sK, const TrackObject* obj,
                     const int64_t* first, int margin, int64_t* launches, double* T_out, double* R_out, double* t_out, float* residual,
                     int32_t* status, int32_t* box, int64_t* stats4) {
  cudaStream_t st = o.stream;
  const PoseShare* sh = o.share;
  const bool verify = o.verify.on != 0;
  const int64_t n = first[n_frames];
  const int nc = pose_batch_chunks(n);
  PoseFinished& d = s->done;
  d.reset();
  // Every buffer of the run before its first chunk: once chunks run, no device memory is allocated or freed (a free
  // waits for the whole device, a spinning peer collector of a shared run included).  The cloud buffers come before
  // pose_prepare, which sizes the slot outputs a verifying shared chunk publishes from by them.
  // A chunk's slot: M model points (the largest crop), then a window of up to 4 M scene points.
  const int64_t M = s->area_max, W = 4 * M, stride = M + W, slots = std::min<int64_t>(n, POSE_CHUNK);
  int rc = n ? pose_buffers(s, st, (int)((slots * stride + 2 * M - 1) / (2 * M)), M) : LM_OK;
  if (!rc) rc = pose_prepare(s, st, n_frames, n, verify);
  if (rc) return rc;
  if (n == 0) {  // no chunk, so no status block to check
    d.fill(PoseRunKind::track, verify, nullptr, 0);
    return pose_status(s->h_bstat.get(), 0, sh, false, 0, 0, stats4);
  }
  if ((size_t)n > s->h_trec.size()) {
    CUI(cudaStreamSynchronize(st));
    s->d_tobj.reset(); s->d_trec.reset(); s->h_trec.reset();
    CUI(s->d_tobj.assign(n));
    CUI(s->d_trec.assign(n));
    CUI(s->h_trec.assign(n));
  }
  // the objects, and the tables that k_track_cloud, k_pose_verify and a shared chunk's publishers read
  CUI(cudaMemcpyAsync(s->d_tobj.get(), obj, sizeof(TrackObject) * n, cudaMemcpyHostToDevice, st));
  rc = run_tables(s, st, n_frames, first, sK);
  if (rc) return rc;
  int64_t stage_launches = 0;
  for (int c = 0; c < nc; ++c) {
    const int64_t c0 = (int64_t)c * POSE_CHUNK;
    const int m = chunk_size(n, c);
    if (o.views) {  // every rank re-chooses every object of the chunk, so all ranks hold the same objects
      TrackViewParams v;
      v.obj = s->d_tobj.get() + c0; v.counts = s->d_bstat.get() + 4 * c + 3;
      v.rt = s->d_rt.get(); v.has = s->d_has.get(); v.class_begin = s->d_class_begin.get();
      v.n_classes = (int32_t)s->class_begin.size() - 1; v.tau = o.view_tau;
      k_track_views<<<m, VIEW_THREADS, 0, st>>>(v);
      ++stage_launches;
      ++*launches;
    }
    TrackParams q;
    memset(&q, 0, sizeof(q));
    q.obj = s->d_tobj.get() + c0; q.tpl = s->d_tpl.get(); q.crops = s->d_crops.get();
    q.margin = margin; q.cap = W; q.stride = stride; q.M = M;
    q.rec = s->d_trec.get() + c0;
    PoseChunk k = run_chunk(s, o, c, nullptr, s->d_bstat.get() + 4 * c + 3, m, d_scene, nullptr);
    k.frame_of = s->d_bframe.get() + c0; k.sKs = s->d_bsK.get();
    k.track = &q;
    const int l = pose_chunk(s, o, k);
    if (l < 0) return l;
    stage_launches += l;
    *launches += l;
  }
  CUI(cudaMemcpyAsync(s->h_bouts.get(), s->d_bouts.get(), sizeof(IcpOut) * n, cudaMemcpyDeviceToHost, st));
  CUI(cudaMemcpyAsync(s->h_trec.get(), s->d_trec.get(), sizeof(TrackRec) * n, cudaMemcpyDeviceToHost, st));
  if (verify) CUI(cudaMemcpyAsync(s->h_bver.get(), s->d_bver.get(), sizeof(PoseVerify) * n, cudaMemcpyDeviceToHost, st));
  CUI(cudaMemcpyAsync(s->h_bstat.get(), s->d_bstat.get(), sizeof(int32_t) * 4 * nc, cudaMemcpyDeviceToHost, st));
  std::vector<TrackObject> chosen;  // view following: the objects as k_track_views left them
  if (o.views) {
    chosen.resize((size_t)n);
    CUI(cudaMemcpyAsync(chosen.data(), s->d_tobj.get(), sizeof(TrackObject) * n, cudaMemcpyDeviceToHost, st));
  }
  CUI(cudaStreamSynchronize(st));
  CUI(cudaGetLastError());
  rc = pose_status(s->h_bstat.get(), nc, sh, nc > 1, n, stage_launches, stats4);
  if (rc) return rc;
  d.fill(PoseRunKind::track, verify, s->h_bver.get(), n);
  d.entries(n);
  d.tpl.resize((size_t)n);
  for (int64_t i = 0; i < n; ++i) {
    const TrackRec& e = s->h_trec[(size_t)i];
    status[i] = e.status;
    memcpy(box + 4 * i, e.box, sizeof(e.box));
    // an entry not tracked keeps its start, template included
    const int64_t g = e.status == LM_TRACK_TRACKED && o.views ? chosen[(size_t)i].g : obj[i].g;
    const int64_t cls = std::upper_bound(s->class_begin.begin(), s->class_begin.end(), (int32_t)obj[i].g) - s->class_begin.begin() - 1;
    d.tpl[(size_t)i] = (int32_t)(g - s->class_begin[(size_t)cls]);
    if (e.status != LM_TRACK_TRACKED) { residual[i] = -1.f; continue; }
    const IcpOut& q = s->h_bouts[(size_t)i];
    const TplHost& h = s->tpl[(size_t)g];
    d.compose(i, q, h.R, h.t, R_out, t_out, residual);
    memcpy(T_out + 16 * i, q.T, sizeof(q.T));
  }
  return LM_OK;
}

int pose_stage_track_templates(const lm_pose_stage* s, int32_t* template_id, int64_t cap, int64_t* n) {
  if (!n || (cap > 0 && !template_id)) return lm_fail(LM_E_INVALID, "null argument");
  if (!s || s->done.kind != PoseRunKind::track || s->done.stale)
    return lm_fail(LM_E_STATE, "the pose run last finished was no track run (lm_track, lm_track_batch, lm_peer_track_batch), or it failed");
  const std::vector<int32_t>& tpl = s->done.tpl;
  *n = (int64_t)tpl.size();
  if (*n > cap) return lm_fail(LM_E_CAPACITY, "%lld entries, capacity %lld", (long long)*n, (long long)cap);
  if (*n) memcpy(template_id, tpl.data(), sizeof(int32_t) * (size_t)*n);
  return LM_OK;
}

int pose_stage_transforms(const lm_pose_stage* s, double* T_out, int64_t cap, int64_t* n) {
  if (!n || (cap > 0 && !T_out)) return lm_fail(LM_E_INVALID, "null argument");
  const PoseFinished& d = s->done;
  const bool poses = d.kind == PoseRunKind::poses || d.kind == PoseRunKind::kept || d.kind == PoseRunKind::track;
  if (!poses || d.stale) return lm_fail(LM_E_STATE, "no pose run has finished since the last one was enqueued (or it failed)");
  *n = (int64_t)d.T.size() / 16;
  for (const auto& k : d.kept) *n += k.second;
  if (*n > cap) return lm_fail(LM_E_CAPACITY, "%lld entries, capacity %lld", (long long)*n, (long long)cap);
  if (!d.T.empty()) memcpy(T_out, d.T.data(), sizeof(double) * d.T.size());
  if (d.kept.empty() || !*n) return LM_OK;
  // the pose NMS's kept poses: each names its survivor, whose ICP output holds its T.  Only a later run, which makes d
  // stale, writes d_bksrc and d_bouts again.
  std::vector<int32_t> src((size_t)d.survivors);
  std::vector<IcpOut> outs((size_t)d.survivors);
  CUI(cudaMemcpyAsync(src.data(), s->d_bksrc.get(), sizeof(int32_t) * src.size(), cudaMemcpyDeviceToHost, d.stream));
  CUI(cudaMemcpyAsync(outs.data(), s->d_bouts.get(), sizeof(IcpOut) * outs.size(), cudaMemcpyDeviceToHost, d.stream));
  CUI(cudaStreamSynchronize(d.stream));
  for (const auto& k : d.kept)
    for (int64_t j = 0; j < k.second; ++j, T_out += 16) memcpy(T_out, outs[(size_t)src[(size_t)(k.first + j)]].T, sizeof(double) * 16);
  return LM_OK;
}
