// lm_depth.cuh -- depth pixels of caller planes in device memory, as the library stores them: u16 millimetres.
//
// Shared by the front-end's ingest of a device frame (k_fe_ingest, lm_frontend.cuh) and the ICP's device inputs
// (k_icp_scene, k_icp_render_box, k_icp_render_crop in lm_icp.cu), so that a float depth plane converts one way everywhere.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

// Float depth to u16 mm as the reference's driver converts it on the host (depth *= depth_scale;
// depth.astype(np.uint16), linemod_and_levelup_test.py:315-317): one float32 product, truncated.  Products outside
// [0, 65536) -- NaN, negatives, infinities, >= 65536 -- are 0 (no depth), where numpy's cast is platform-defined.
__device__ __forceinline__ uint16_t lm_depth_mm(float d, float scale) {
  const float v = __fmul_rn(d, scale);
  return (v >= 0.f && v < 65536.f) ? (uint16_t)__float2uint_rz(v) : (uint16_t)0;
}

// Pixel x of a depth row: u16 mm as is, or float32 converted by lm_depth_mm.
__device__ __forceinline__ uint16_t lm_depth_at(const uint8_t* row, int x, int f32, float scale) {
  return f32 ? lm_depth_mm(((const float*)row)[x], scale) : ((const uint16_t*)row)[x];
}
