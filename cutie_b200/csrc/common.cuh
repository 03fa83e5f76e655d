// Shared helpers for the cutie_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/cutie_b200.h"

namespace cutie {

extern thread_local char g_last_error[512];

inline int fail(int code, const char* fmt, const char* fn) {
  snprintf(g_last_error, sizeof(g_last_error), fmt, fn);
  return code;
}

inline int set_cuda_error(const char* fn, cudaError_t e) {
  snprintf(g_last_error, sizeof(g_last_error), "%s: CUDA error: %s", fn, cudaGetErrorString(e));
  return -2;
}

#define CUTIE_REQUIRE(cond, what)                                                         \
  do {                                                                                    \
    if (!(cond)) return ::cutie::fail(-1, "%s: invalid argument: " what, __func__);       \
  } while (0)

#define CUTIE_CHECK_LAUNCH()                                                              \
  do {                                                                                    \
    cudaError_t e__ = cudaGetLastError();                                                 \
    if (e__ != cudaSuccess) return ::cutie::set_cuda_error(__func__, e__);                \
  } while (0)

constexpr int kMaxSeg = CUTIE_B200_MAX_SEGMENTS;

// A memory bank presented as up to 4 physically contiguous token-major runs.
struct KeySegments {
  const float* key[kMaxSeg];
  const float* shr[kMaxSeg];
  long long begin[kMaxSeg + 1];  // prefix sums of lengths: segment s covers [begin[s], begin[s+1])
  long long key_bs[kMaxSeg];
  long long shr_bs[kMaxSeg];
  int nseg;
};

// Objects per launch of the kernels that take per-object row pointers by value (readout gather, consolidation).
// Their C entry points accept any number of objects and launch once per group of at most kMaxObj.
constexpr int kMaxObj = 16;

struct RowSegments {
  const float* rows[kMaxSeg * kMaxObj];  // [segment][object]
  long long bs[kMaxSeg * kMaxObj];
  long long begin[kMaxSeg + 1];
  int nseg;
  int nobj;
};

// The prefix table of a bank passed as (num_segments, seg_len[]): begin[s] = seg_len[0] + ... + seg_len[s-1], and every
// entry from num_segments on holds the total, so seg_of() never steps past the last segment.  n_total (optional): the
// total the caller was promised.  Returns 0, or -1 with `fn` in cutie_b200_last_error() for a segment count outside
// 1..kMaxSeg, a negative length or lengths that do not sum to *n_total.
inline int segment_table(long long (&begin)[kMaxSeg + 1], int num_segments, const int64_t* seg_len,
                         const int64_t* n_total, const char* fn) {
  if (num_segments < 1 || num_segments > kMaxSeg) return fail(-1, "%s: invalid argument: 1..4 segments", fn);
  if (!seg_len) return fail(-1, "%s: invalid argument: null seg_len", fn);
  long long tot = 0;
  for (int s = 0; s < num_segments; ++s) {
    if (seg_len[s] < 0) return fail(-1, "%s: invalid argument: negative segment length", fn);
    begin[s] = tot;
    tot += seg_len[s];
  }
  for (int s = num_segments; s <= kMaxSeg; ++s) begin[s] = tot;
  if (n_total && tot != *n_total) return fail(-1, "%s: invalid argument: n_total != sum of segment lengths", fn);
  return 0;
}

__device__ __forceinline__ int seg_of(const long long* begin, int nseg, long long g) {
  int s = 0;
#pragma unroll
  for (int i = 1; i < kMaxSeg; ++i)
    if (i < nseg && g >= begin[i]) s = i;
  return s;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

inline int num_sms() {                     // of the CURRENT device (cached per ordinal)
  static int cache[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  if (cache[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cache[dev] = n > 0 ? n : 132;
  }
  return cache[dev];
}

// cudaFuncSetAttribute (opt-in dynamic shared memory) is per DEVICE: callers keep a `static bool done[64]` per call
// site and set the attribute the first time each device ordinal launches through it.
inline bool first_use_on_device(bool (&done)[64]) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return true;
  if (done[dev]) return false;
  done[dev] = true;
  return true;
}

}  // namespace cutie
