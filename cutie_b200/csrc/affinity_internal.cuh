// Internal (non-ABI) interfaces between affinity.cu (exact scan, orchestration of both filtered plans), affinity_tc.cu
// (TF32 wgmma candidate filter, level threshold hand-over, exact re-rank) and affinity_f16.cu (FP16 wgmma filter over the
// key operand image, threshold select).
#pragma once
#include "common.cuh"

namespace cutie {

// A "sample" of the bank: virtual indices i in [0, samp_count) map to tokens g = samp_begin + i * samp_stride
// of the concatenated segments.  stride 1 = the whole bank.  Levels use nested samples (strides 256, 16, 1).

struct TcFilterParams {
  KeySegments segs;
  const float* qk;
  const float* qe;
  long long Q;
  long long samp_begin, samp_stride, samp_count;
  int tiles_per_split, nsplit;
  const float* emax_in;    // [B][Q] upper bound of the k-th smallest exact energy of the previous level; null = +inf
  int* cand_idx;           // [B][Q][cap] token indices (per-query list, filled with atomics)
  float* cand_e;           // [B][Q][cap] their TF32 energies
  int* count;              // [B][Q] number of candidates (may exceed cap = overflow); zeroed by the caller
  float* dmax;             // [B][Q] largest error bound used (atomicMax on the bit pattern); zeroed by the caller
  int cap;
  float* dbg_energy;       // optional [B][Q][samp_count] tf32 energies (tests)
};

struct SelectParams {
  long long Q;
  const float* cand_e;
  const int* count;
  const float* dmax;
  int cap, top_k;
  float* emax_out;         // [B][Q]
};

struct RerankParams {
  KeySegments segs;
  const float* qk;
  const float* qe;
  long long Q, n_total;
  const int* cand_idx;
  const int* count;
  int cap, top_k, kpad;
  int* out_idx;
  float* out_w;
  float* out_sim;
  unsigned long long* usage_acc;
};

// Where the image tiles of a bank are: per segment the FP16 operand image of the arena it lives in
// (cutie_bank_key_image), addressed by physical 128-token tile.
struct ImageTiles {
  const unsigned char* img[kMaxSeg];
  long long bs[kMaxSeg];           // batch stride (bytes)
  long long tile0[kMaxSeg];        // first physical tile of the segment
  int lo0[kMaxSeg];                // row of the segment's first token inside that tile
  long long tcum[kMaxSeg + 1];     // prefix sums of the segments' tile counts
};

// FP16 filter over the key operand image (affinity_f16.cu): threshold sampling pass + candidate filter pass.
constexpr int F16_RESERVE = 16;            // candidate slots reserved per global atomic (per thread)
constexpr int F16_SLOTS = 8;               // running minima per sampling thread (threshold slots = splits x 2 x F16_SLOTS)
struct F16FilterParams {
  KeySegments segs;
  const float* qk;
  const float* qe;
  const float* key_mu;             // [B][64] centre the image was built with (null = 0): the operand uses qk - mu
  long long Q;
  // sample pass: tiles g = tile_phase + j * tile_stride of the image; output group_min [B][Q][groups_per_query]
  int tile_stride, tile_phase;
  float* group_min;
  int groups_per_query;
  // filter pass: thresholds in, per-query candidate lists out
  const float* emax_in;
  int* cand_idx;
  int* count;
  int cap;
  // CTA schedule (f16_schedule)
  int full_groups, splits_full, splits_half;
  ImageTiles tiles;
};
size_t f16_filter_smem_bytes();
int f16_schedule(F16FilterParams& p, long long B);
int launch_f16_filter(const F16FilterParams& p, long long B, int grid_x, bool sample, cudaStream_t st);
struct F16ThresholdParams {
  const float* group_min;      // [B][Q][groups] slot minima of the sample pass
  int groups, top_k, kpad;
  long long Q, n_total;
  float* emax_out;             // [B][Q]
  // optional seeds: [B][Q][kpad] token indices (first top_k entries; -1 = none), evaluated exactly against this query
  const int* seed_idx;
  KeySegments segs;
  const float* qk;
  const float* qe;
};
int launch_f16_threshold(const F16ThresholdParams& p, long long B, cudaStream_t st);

size_t tc_filter_smem_bytes();
int tc_split_count(long long B, long long Q, long long samp_count);
int launch_tc_filter(const TcFilterParams& p, long long B, cudaStream_t st);
int launch_level_select(const SelectParams& p, long long B, int kpad, cudaStream_t st);
int launch_rerank(const RerankParams& p, long long B, cudaStream_t st);

}  // namespace cutie
