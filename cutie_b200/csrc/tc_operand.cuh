// Shared-memory operand layout of the TF32 wgmma affinity filter (sm_90a), written by the filter's in-kernel
// producers (affinity_tc.cu), which convert fp32 key rows on the fly.  (The bank's precomputed key image is FP16:
// tc_operand_f16.cuh.)
//
// A memory-token tile = 128 rows (tokens) x K = 136 tf32:
//   4 x [128 rows x 128 B] SWIZZLE_128B K-blocks  : [shr k_c^2 (c = 0..63) | shr k_c (c = 0..63)]
//   1 x [128 rows x  32 B] un-swizzled tail block  : [shr, BIG*invalid, shr, -eps P^2 | -2 eps P R, -eps R^2, 0, 0]
// with P = sqrt(shr |k|^2), R = sqrt(shr) rounded up a hair (the per-token TF32 error-bound factors).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cutie {

constexpr int TC_QT = 128;                 // queries per CTA (MMA M)
constexpr int TC_KTILE = 128;              // memory tokens per tile (MMA N)
constexpr int TC_BLK_BYTES = 128 * 128;    // one SW128 K-block: 128 rows x 128 B
constexpr int TC_TAIL_BYTES = 128 * 32;    // tail block: 128 rows x 8 tf32
constexpr int TC_OPER_BYTES = 4 * TC_BLK_BYTES + TC_TAIL_BYTES;   // 69632 bytes per 128-token tile
// Query operands are rounded to TF32 (RN, 2^-11) once per CTA; memory tokens are fed as raw fp32 and the tensor core
// ignores their low 13 mantissa bits (<= 2^-10), which saves ~600 conversion instructions per tile.  Product error
// <= 2^-11 + 2^-10 + 2^-21 = 1.466e-3; + fp32 accumulation over 136 terms + rounding of the bound's own operands.
constexpr float TC_TF32_EPS = 1.65e-3f;
constexpr float TC_BIG_E = 1e30f;

__device__ __forceinline__ float fsqrt_approx(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// byte offsets inside an operand buffer
__device__ __forceinline__ int off_main(int row, int elem) {     // elem in [0,128): 4 K-blocks of 32
  const int blk = elem >> 5, chunk = (elem & 31) >> 2, within = elem & 3;
  return blk * TC_BLK_BYTES + row * 128 + ((chunk ^ (row & 7)) << 4) + within * 4;
}
__device__ __forceinline__ int off_tail(int row, int elem) {     // elem in [0,8)
  return 4 * TC_BLK_BYTES + (elem >> 2) * 2048 + (row >> 3) * 128 + (row & 7) * 16 + (elem & 3) * 4;
}

// One token row handled by 16 consecutive lanes (lane c4 = lane & 15 owns channels 4*c4 .. 4*c4+3; all 32 lanes of
// the warp must call this).  `shr < 0` marks an invalid (out-of-range) row.  Writes the lane's two 16-byte chunks
// and, from lane c4 == 0, the row's tail; returns the error-bound factors through Pn / Rn.
__device__ __forceinline__ void store_key_row_operand(unsigned char* tile, int row, int c4, float4 v, float shr,
                                                      float& Pn, float& Rn) {
  const bool valid = shr >= 0.f;
  const float sh = valid ? shr : 0.f;
  const float4 ln = make_float4(sh * v.x, sh * v.y, sh * v.z, sh * v.w);
  float n2 = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w)));
  n2 += __shfl_xor_sync(0xffffffffu, n2, 1);
  n2 += __shfl_xor_sync(0xffffffffu, n2, 2);
  n2 += __shfl_xor_sync(0xffffffffu, n2, 4);
  n2 += __shfl_xor_sync(0xffffffffu, n2, 8);
  *reinterpret_cast<float4*>(tile + off_main(row, 4 * c4)) = make_float4(ln.x * v.x, ln.y * v.y, ln.z * v.z, ln.w * v.w);
  *reinterpret_cast<float4*>(tile + off_main(row, 64 + 4 * c4)) = ln;
  // per-row error-bound factors (rounded up a hair) and the tail block; all 16 lanes of the row hold the
  // same values, lane c4 == 0 stores them (small predicated body, no divergence region)
  Pn = fsqrt_approx(sh * n2) * 1.002f;
  Rn = fsqrt_approx(sh) * 1.002f;
  const float4 t0 = make_float4(sh, valid ? 0.f : TC_BIG_E, sh, -TC_TF32_EPS * Pn * Pn);
  const float4 t1 = make_float4(-2.f * TC_TF32_EPS * Pn * Rn, -TC_TF32_EPS * Rn * Rn, 0.f, 0.f);
  if (c4 == 0) {
    // tail: [shr, BIG if invalid, shr, -eps P^2 | -2 eps P R, -eps R^2, 0, 0]   x   [b2_hi, 1, b2_lo, 1 | v, v^2, 0, 0]
    *reinterpret_cast<float4*>(tile + off_tail(row, 0)) = t0;
    *reinterpret_cast<float4*>(tile + off_tail(row, 4)) = t1;
  }
}

}  // namespace cutie
