// Post-match stage on the device (SURVEY.md section 8f-3).
//
// The reference's callers never use the raw match list: linemod_and_levelup_test.py:325-345 builds boxes
// (x, y, x + width, y + height, similarity) and runs nms(dets, 0.5) (:34-61), then refines the first three
// survivors with poseRefine (:348-367); linemod_ros/detect.py:41-81, 94-134 does the same.  Here the greedy
// NMS runs on the device right behind k_refine, on the kept records where they lie, and only the top_k
// survivors cross PCIe.
//
// The drivers run nms() on the FINISHED match list, after std::sort + std::unique (LL.cpp:1772-1774), and
// Match::operator== (LL.h:243-246) ignores template_id: unique also drops a match of template B that follows one of
// template A at the same (x, y, similarity, class), although B's box may differ from A's.  So the kernel first sorts
// the kept records into the canonical order -- similarity descending, then template_id, class, y, x ascending: the
// reference's Match::operator< (LL.h:233-240), its ties (left to an unstable std::sort and an unstable numpy argsort,
// :41) resolved in that order -- and drops each record equal in (x, y, similarity, class) to its predecessor there.
// One bitonic sort of 16-byte keys in one CTA: in shared memory up to LM_POST_SMEM_KEYS records, beyond that in
// a global scratch of the next power of two above the result block's capacity.
//
// Then the greedy NMS walks that order: round r picks the first live record, emits it, and kills every later live
// record whose IoU with it exceeds the threshold -- exactly the reference's loop ("order = order[where(ovr <=
// thresh)]"), with the IoU in float64 and the "+1" pixel convention of :40, :51-54.
#pragma once
#include <limits.h>
#include <stdint.h>
#include "linemod_b200.h"

struct PostInfo {  // per entry of the selected template sequence
  int32_t class_index, template_id, width, height;
};

struct PostParams {
  const lm_result_header* hdr;  // result block: header + records (all shards' records in fused multi-GPU mode)
  int32_t capacity;
  const PostInfo* info;         // [n_sel], indexed by lm_record.work
  int32_t n_sel;
  double iou_threshold;
  int32_t top_k;                // <= 0: every survivor (bounded by out_capacity)
  lm_match* out;                // device: survivors in pick order
  int32_t out_capacity;
  int32_t* out_counts;          // [0] survivors written, [1] records seen, [2] survivors in total (if all were asked for), [3] coarse candidates
  uint8_t* live;                // [capacity] scratch
  struct PostKey* keys;         // [next power of two >= capacity] scratch, used beyond LM_POST_SMEM_KEYS records
};

__device__ __forceinline__ uint32_t lm_float_order(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);  // monotone in f
}

// Ascending = canonical order.  hi: ~similarity (order-preserving) : 32 | template_id : 20 | class : 12 (lm_load_bank
// refuses wider banks); lo: y : 16 | x : 16 | record slot : 32 (unique keys; padding is all ones and sorts last).
struct PostKey {
  unsigned long long hi, lo;
};

#define LM_POST_SMEM_KEYS 8192  // records sorted in shared memory (128 KB of keys)

__device__ __forceinline__ bool post_less(const PostKey& p, const PostKey& q) {
  return p.hi < q.hi || (p.hi == q.hi && p.lo < q.lo);
}

// equal in (x, y, similarity, class): what Match::operator== compares
__device__ __forceinline__ bool post_same_match(const PostKey& p, const PostKey& q) {
  return ((p.hi ^ q.hi) & 0xFFFFFFFF00000FFFull) == 0ull && ((p.lo ^ q.lo) >> 32) == 0ull;
}

__global__ void __launch_bounds__(1024) k_post_nms(PostParams p) {
  lm_pdl_wait();  // launched with programmatic stream serialization: the records / count of k_refine (k_peer_collect)
                  // are only visible after this returns
  extern __shared__ PostKey s_keys[];
  __shared__ int s_pick;
  const int tid = threadIdx.x;
  const int n = min(p.hdr->count, p.capacity);
  const lm_record* rec = reinterpret_cast<const lm_record*>(p.hdr + 1);
  int m = 1;
  while (m < n) m <<= 1;
  PostKey* keys = m <= LM_POST_SMEM_KEYS ? s_keys : p.keys;
  for (int i = tid; i < m; i += blockDim.x) {
    PostKey k;
    if (i < n) {
      const lm_record r = rec[i];
      const PostInfo inf = p.info[min(max(r.work, 0), p.n_sel - 1)];
      k.hi = ((unsigned long long)~lm_float_order(r.similarity) << 32) |
             ((unsigned long long)((uint32_t)inf.template_id & 0xFFFFFu) << 12) | (unsigned long long)((uint32_t)inf.class_index & 0xFFFu);
      k.lo = ((unsigned long long)(((uint32_t)(uint16_t)(r.y + 0x8000) << 16) | (uint32_t)(uint16_t)(r.x + 0x8000)) << 32) |
             (unsigned long long)(uint32_t)i;
    } else {
      k.hi = ~0ull; k.lo = ~0ull;
    }
    keys[i] = k;
  }
  __syncthreads();
  for (int k = 2; k <= m; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (m >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), l = i + j;
        const PostKey a = keys[i], b = keys[l];
        if (post_less(b, a) == ((i & k) == 0)) { keys[i] = b; keys[l] = a; }
      }
      __syncthreads();
    }
  // the canonical dedupe; live[] is indexed by position in the canonical order from here on
  for (int s = tid; s < n; s += blockDim.x) p.live[s] = (s == 0 || !post_same_match(keys[s - 1], keys[s])) ? 1 : 0;
  __syncthreads();
  const int want = p.top_k > 0 ? min(p.top_k, p.out_capacity) : p.out_capacity;
  int picked = 0, survivors = 0, cur = 0;
  for (;;) {
    // the first live position from cur on: everything before it was picked or suppressed
    int pick = INT_MAX;
    for (int base = cur; base < n && pick == INT_MAX; base += blockDim.x) {
      if (tid == 0) s_pick = INT_MAX;
      __syncthreads();
      if (base + tid < n && p.live[base + tid]) atomicMin(&s_pick, base + tid);
      __syncthreads();
      pick = s_pick;
      __syncthreads();
    }
    if (pick == INT_MAX) break;  // nothing live
    ++survivors;
    const lm_record pr = rec[(uint32_t)keys[pick].lo];
    const PostInfo pi = p.info[min(max(pr.work, 0), p.n_sel - 1)];
    if (picked < want) {
      if (tid == 0) {
        lm_match mt;
        mt.x = pr.x; mt.y = pr.y; mt.similarity = pr.similarity;
        mt.class_index = pi.class_index; mt.template_id = pi.template_id;
        p.out[picked] = mt;
      }
      ++picked;
    }
    if (p.top_k > 0 && picked >= want) break;
    // suppress: ovr = inter / (area_i + area_j - inter) > thresh, float64, +1 convention (:40, :51-56)
    const double x1 = pr.x, y1 = pr.y, x2 = (double)pr.x + pi.width, y2 = (double)pr.y + pi.height;
    const double area = (x2 - x1 + 1.0) * (y2 - y1 + 1.0);
    for (int s = pick + 1 + tid; s < n; s += blockDim.x) {
      if (!p.live[s]) continue;
      const lm_record r = rec[(uint32_t)keys[s].lo];
      const PostInfo inf = p.info[min(max(r.work, 0), p.n_sel - 1)];
      const double a1 = r.x, b1 = r.y, a2 = (double)r.x + inf.width, b2 = (double)r.y + inf.height;
      const double w = fmax(0.0, fmin(x2, a2) - fmax(x1, a1) + 1.0);
      const double h = fmax(0.0, fmin(y2, b2) - fmax(y1, b1) + 1.0);
      const double inter = w * h;
      const double ovr = inter / (area + (a2 - a1 + 1.0) * (b2 - b1 + 1.0) - inter);
      if (!(ovr <= p.iou_threshold)) p.live[s] = 0;
    }
    cur = pick + 1;
    __syncthreads();
  }
  if (tid == 0) {
    p.out_counts[0] = picked;
    p.out_counts[1] = p.hdr->count;
    p.out_counts[2] = p.top_k > 0 ? -1 : survivors;
    p.out_counts[3] = p.hdr->coarse_candidates;  // the host checks it against the candidate list's capacity
  }
}
