// Tensor-core (wgmma) candidate filter + exact re-rank for the pixel-memory affinity (sm_90a).
//
// The exact scan (affinity.cu) spends 2 fp32 FFMA per (token, query, channel) on CUDA cores.  Here the dense
// contraction runs on the tensor cores in TF32 and is used only as a FILTER:
//
//   E[q,n] = -8 S[q,n] = shr_n * sum_c qe_c (k_c - qk_c)^2
//          = [qe | -2 qe qk | b2_hi 1 b2_lo] . [shr k^2 | shr k | shr BIG*invalid shr]      (K = 128 + 8)
//
//   A operand (M = 128 queries, resident for the CTA's lifetime) and B operand (N = 128 memory tokens per
//   tile, double buffered) are K-major, 4 x [128 rows x 128 B] SWIZZLE_128B blocks + one [128 x 32 B]
//   un-swizzled tail block; the epilogue warpgroups issue wgmma.m64n32k8 (tf32) for their 32-column groups and
//   re-deal the register fragments so that a thread owns one query row (frag_rows32).
//   Epilogue thread == query: the threshold is a register, candidates go to a per-query global list:
//   a token is a candidate iff  E_tf32 < Emax_q + delta,  where Emax_q is an upper bound of the k-th smallest
//   EXACT energy over a nested subset scanned by the previous level (k-th smallest TF32 energy there + the
//   largest error bound used there) and delta = eps * (P_tile + R_tile * sqrt(b2_q))^2 bounds the TF32 rounding
//   error (P_tile = max sqrt(shr |k|^2), R_tile = max sqrt(shr) over the tile).  A true top-k member therefore
//   always survives every level.  Survivors of the last level are re-ranked by the exact fp32 direct form
//   (affinity_rerank_kernel), so the final selection and weights are bit-identical to the exact scan's.
//
// Warp roles (384 threads): warps 0-3 one MMA + epilogue warpgroup; warps 4-7 / 8-11 two producer groups that
// alternate tiles (global fp32 rows -> scaled/squared/tf32-rounded swizzled smem; a group's next tile is in
// flight while the other group converts).
#include "topk_common.cuh"
#include "affinity_internal.cuh"
#include "tc_operand.cuh"
#include "tc_ptx.cuh"

namespace cutie {

constexpr int QT = TC_QT;               // queries per CTA (MMA M)
constexpr int KTILE = TC_KTILE;         // memory tokens per tile (MMA N)
constexpr int BLK_BYTES = TC_BLK_BYTES;
constexpr int OPER_BYTES = TC_OPER_BYTES;
constexpr int TC_THREADS = 384;         // warps 0-3 MMA + epilogue, warps 4-11 two producer groups
constexpr float TF32_EPS = TC_TF32_EPS;

// K-major un-swizzled descriptor of the [128 x 32 B] tail block: chunk-major, 16 row-groups of chunk 0 (128 B each),
// then chunk 1 at +2048 B.
__device__ __forceinline__ uint64_t desc_tail(uint32_t addr) { return desc_interleave(addr, 2048, 128); }
__device__ __forceinline__ unsigned low_mask32(int n) {      // bits [0, n) of a 32-bit word (any int)
  return n >= 32 ? 0xffffffffu : (n <= 0 ? 0u : ((1u << n) - 1u));
}
struct TcSmemTail {
  unsigned long long full[2], empty[2];
  float rowP[4][KTILE];     // [tile % 4][row] sqrt(shr)*|k|
  float rowR[4][KTILE];     // [tile % 4][row] sqrt(shr)
  float vq[QT];              // [query row] sqrt(b2)
};

template <bool DBG>
__global__ void __launch_bounds__(TC_THREADS, 1) affinity_tc_filter_kernel(const TcFilterParams p) {
  constexpr int EPI_WARPS = 4;
  constexpr int RESERVE = 32;     // candidate slots reserved per global atomic (per thread)
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* A = smem;                              // queries
  unsigned char* Bst = smem + OPER_BYTES;               // 2 stages of keys
  TcSmemTail& T = *reinterpret_cast<TcSmemTail*>(smem + 3 * OPER_BYTES);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, split = blockIdx.y;
  const long long q0 = (long long)blockIdx.x * QT;
  // Tiles are dealt to the key splits round-robin (split s takes tiles s, s + nsplit, ...): candidates cluster in
  // the part of the bank that resembles the current frame (recent memory frames), and contiguous ranges would
  // leave the CTAs owning that part with nearly all of the candidate work.
  // Tile g covers sample indices [128 g, 128 g + 128).
  const long long total_tiles = (p.samp_count + KTILE - 1) / KTILE;
  const long long tile_step = p.nsplit;
  const long long i_end = p.samp_count;
  const int ntiles = split < total_tiles ? (int)((total_tiles - split + tile_step - 1) / tile_step) : 0;
  auto tile_of = [&](int t) { return (long long)split + (long long)t * tile_step; };

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(&T.full[s]), 128);               // every thread of the producer group that converted the tile
      mbar_init(smem_u32(&T.empty[s]), 32 * EPI_WARPS);   // every MMA + epilogue thread is done with the tile
    }
    mbar_init_fence();
  }
  // ---- query operand: row = query, [qe | -2 qe qk] + tail [b2_hi, 1, b2_lo, 0...] ----
  if (tid < QT) {
    const long long q = q0 + tid;
    float b2 = 0.f;
    const bool qok = q < p.Q;
    const float* qe_p = p.qe + (long long)b * CKD * p.Q + (qok ? q : 0);
    const float* qk_p = p.qk + (long long)b * CKD * p.Q + (qok ? q : 0);
    // 16 channels at a time: all 32 loads of a batch are in flight together (the prologue is on every CTA's
    // critical path and the filter runs three launches per frame)
#pragma unroll 1
    for (int c0 = 0; c0 < CKD; c0 += 16) {
      float ev[16], kv[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        ev[i] = __ldg(qe_p + (long long)(c0 + i) * p.Q);
        kv[i] = __ldg(qk_p + (long long)(c0 + i) * p.Q);
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float e = qok ? ev[i] : 0.f, k = qok ? kv[i] : 0.f;
        b2 = fmaf(e * k, k, b2);
        *reinterpret_cast<float*>(A + off_main(tid, c0 + i)) = to_tf32(e);
        *reinterpret_cast<float*>(A + off_main(tid, 64 + c0 + i)) = to_tf32(-2.f * e * k);
      }
    }
    const float b2_hi = to_tf32(b2), b2_lo = to_tf32(b2 - b2_hi);
    const float vq_ = sqrtf(b2);
    float tl[8] = {b2_hi, 1.f, b2_lo, 1.f, to_tf32(vq_ * 1.0005f), to_tf32(vq_ * vq_ * 1.001f), 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) *reinterpret_cast<float*>(A + off_tail(tid, i)) = tl[i];
    T.vq[tid] = sqrtf(b2);
    fence_proxy_async();
  }
  __syncthreads();

  if (warp < EPI_WARPS) {
    // =========================== epilogue: thread == query ===========================
    const int row = frag_row(warp & 3, lane);                // the query row frag_rows32 gives this thread
    const long long q = q0 + row;
    const float vq = T.vq[row];
    // Emax: upper bound of the k-th smallest exact energy of the previous (nested) level; null => +inf
    const float emax = (q < p.Q) ? (p.emax_in ? p.emax_in[(long long)b * p.Q + q] : CUDART_INF_F) : -CUDART_INF_F;
    const uint32_t a_base = smem_u32(A);
    const long long bq = (long long)b * p.Q + (q < p.Q ? q : 0);
    int* my_idx = p.cand_idx + bq * p.cap;
    float* my_e = p.cand_e + bq * p.cap;
    const bool all_pass = (p.emax_in == nullptr);       // coarsest level: every token of the sample is kept
    int blk_base = 0, blk_used = RESERVE;
    if (all_pass && split == 0 && q < p.Q) p.count[bq] = (int)p.samp_count;
    for (int t = 0; t < ntiles; ++t) {
      const int a = t & 1;
      mbar_wait(smem_u32(&T.full[a]), (t >> 1) & 1);
      const uint32_t b_base = smem_u32(Bst + a * OPER_BYTES);
      const float thr = (q < p.Q) ? emax : -CUDART_INF_F;
      const long long ibase = tile_of(t) * KTILE;
      const int nvalid = (int)((i_end - ibase) < KTILE ? (i_end - ibase) : KTILE);      // valid rows [0, nvalid)
#pragma unroll 1
      for (int cg = 0; cg < 4; ++cg) {
        // D[128 queries x 32 tokens of group cg] as two M = 64 halves, K = 4 x 32 (swizzled blocks) + 8 (tail)
        float d0[16], d1[16];
        wg_fence_acc(d0);
        wg_fence_acc(d1);
        wg_fence();
        const uint32_t bcg = b_base + (uint32_t)(cg * 32 * 128);
#pragma unroll
        for (int blk = 0; blk < 4; ++blk)
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint64_t db = desc_sw128_kmajor(bcg + blk * BLK_BYTES + ks * 32);
            wgmma_tf32_n32(d0, desc_sw128_kmajor(a_base + blk * BLK_BYTES + ks * 32), db, blk | ks);
            wgmma_tf32_n32(d1, desc_sw128_kmajor(a_base + 64 * 128 + blk * BLK_BYTES + ks * 32), db, blk | ks);
          }
        const uint64_t dbt = desc_tail(b_base + 4 * BLK_BYTES + cg * 32 / 8 * 128);
        wgmma_tf32_n32(d0, desc_tail(a_base + 4 * BLK_BYTES), dbt, 1);
        wgmma_tf32_n32(d1, desc_tail(a_base + 4 * BLK_BYTES + 64 / 8 * 128), dbt, 1);
        wg_commit();
        wg_wait0();
        wg_fence_acc(d0);
        wg_fence_acc(d1);
        uint32_t r[32];
        frag_rows32<16, 0>(d0, d1, r);
        // r[j] = E_tf32 - eps (P_n + R_n v_q)^2 : a LOWER bound of the exact energy (invalid rows hold ~1e30)
        if (DBG) {
          if (q < p.Q)
            for (int j = 0; j < 32; ++j)
              if (cg * 32 + j < nvalid && ibase + cg * 32 + j < p.samp_count)
                p.dbg_energy[((long long)b * p.Q + q) * p.samp_count + ibase + cg * 32 + j] = __uint_as_float(r[j]);
        }
        // branch-free per-lane bitmask of passing columns (2 instructions per element) ...
        unsigned mask = 0u;
#pragma unroll
        for (int j = 0; j < 32; ++j) mask |= (__uint_as_float(r[j]) < thr) ? (1u << j) : 0u;
        mask &= low_mask32(nvalid - cg * 32);                    // columns of this group that hold real tokens
        // ... and a per-lane walk over the lane's own passing columns (iterations per group = the largest popcount
        // among the 32 queries, not the number of distinct passing columns).  The threshold hand-over also needs the value: it
        // is picked out of the 32 registers with a 5-level select tree on the column bits (31 SEL; no accumulator re-read,
        // no dynamic register indexing).
        unsigned m = mask;
        while (m) {
          const int j = __ffs(m) - 1;
          m &= m - 1;
          const int col = cg * 32 + j;
          uint32_t s16[16], s8[8], s4[4];
          const bool b4 = (j & 16) != 0, b3 = (j & 8) != 0, b2 = (j & 4) != 0, b1 = (j & 2) != 0, b0 = (j & 1) != 0;
#pragma unroll
          for (int i = 0; i < 16; ++i) s16[i] = b4 ? r[16 + i] : r[i];
#pragma unroll
          for (int i = 0; i < 8; ++i) s8[i] = b3 ? s16[8 + i] : s16[i];
#pragma unroll
          for (int i = 0; i < 4; ++i) s4[i] = b2 ? s8[4 + i] : s8[i];
          const uint32_t s2a = b1 ? s4[2] : s4[0], s2b = b1 ? s4[3] : s4[1];
          const float d = __uint_as_float(b0 ? s2b : s2a);
          const float s_ = T.rowP[t & 3][col] + T.rowR[t & 3][col] * vq;
          const float e_hi = d + 2.01f * TF32_EPS * s_ * s_;              // an UPPER bound of the exact energy
          int pos;
          if (all_pass) {
            pos = (int)(ibase + col);
          } else {
            // slots are reserved in blocks: one global atomic (latency ~1 us) per block of candidates of this
            // (query, CTA) instead of one per candidate; unused slots of the last block are voided at the end
            if (blk_used == RESERVE) { blk_base = atomicAdd(&p.count[bq], RESERVE); blk_used = 0; }
            pos = blk_base + blk_used++;
          }
          if (pos < p.cap) {
            my_idx[pos] = (int)(p.samp_begin + (ibase + col) * p.samp_stride);
            my_e[pos] = e_hi;
          }
        }
        __syncwarp();      // reconverge before the next aligned wgmma / the barrier arrive
      }
      mbar_arrive(smem_u32(&T.empty[a]));
    }
    if (!all_pass && blk_used < RESERVE)
      for (int u = blk_used; u < RESERVE; ++u)
        if (blk_base + u < p.cap) { my_idx[blk_base + u] = -1; my_e[blk_base + u] = CUDART_INF_F; }
  } else if (warp < 12) {
    // ============ producers: 16 lanes per token row (coalesced 256-B rows), next tile prefetched ============
    const int grp = (warp - 4) >> 2;     // producer group 0 handles even tiles (stage 0), group 1 odd tiles
    const int pt = (tid - 128) & 127;    // 0..127 within the group
    const int c4 = pt & 15;              // which 16-B chunk of the row this lane owns
    const int r0 = pt >> 4;              // rows r0 + 8*j, j = 0..15
    float4 kf[16];
    float shr[16];
    auto load_tile = [&](int t) {
      const long long i0 = tile_of(t) * KTILE;
      const long long g_first = p.samp_begin + i0 * p.samp_stride;
      const long long i_last = (i0 + KTILE <= i_end ? i0 + KTILE : i_end) - 1;
      const long long g_last = p.samp_begin + i_last * p.samp_stride;
      const int sg = seg_of(p.segs.begin, p.segs.nseg, g_first);
      if (i0 + KTILE <= i_end && sg == seg_of(p.segs.begin, p.segs.nseg, g_last)) {
        // whole tile inside one segment: one base pointer, constant row step
        const long long off0 = g_first - p.segs.begin[sg] + (long long)r0 * p.samp_stride;
        const float4* kp = reinterpret_cast<const float4*>(p.segs.key[sg] + (long long)b * p.segs.key_bs[sg] + off0 * CKD) + c4;
        const float* sp = p.segs.shr[sg] + (long long)b * p.segs.shr_bs[sg] + off0;
        const long long kstep = 8 * p.samp_stride * (CKD / 4), sstep = 8 * p.samp_stride;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          kf[j] = __ldg(kp + j * kstep);
          shr[j] = __ldg(sp + j * sstep);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const long long i = i0 + r0 + 8 * j;
          if (i < i_end) {
            const long long g = p.samp_begin + i * p.samp_stride;
            const int s2 = seg_of(p.segs.begin, p.segs.nseg, g);
            const long long off = g - p.segs.begin[s2];
            kf[j] = __ldg(reinterpret_cast<const float4*>(p.segs.key[s2] + (long long)b * p.segs.key_bs[s2] + off * CKD) + c4);
            shr[j] = __ldg(p.segs.shr[s2] + (long long)b * p.segs.shr_bs[s2] + off);
          } else {
            kf[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            shr[j] = -1.f;                 // marks an invalid row
          }
        }
      }
    };
    if (grp < ntiles) load_tile(grp);
    for (int t = grp; t < ntiles; t += 2) {
      const int s = t & 1;
      mbar_wait(smem_u32(&T.empty[s]), ((t >> 1) & 1) ^ 1);
      unsigned char* Bs = Bst + s * OPER_BYTES;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int row = r0 + 8 * j;
        float Pn, Rn;
        store_key_row_operand(Bs, row, c4, kf[j], shr[j], Pn, Rn);      // tc_operand.cuh
        if (c4 == 0) {
          T.rowP[t & 3][row] = Pn;
          T.rowR[t & 3][row] = Rn;
        }
      }
      fence_proxy_async();
      mbar_arrive(smem_u32(&T.full[s]));
      if (t + 2 < ntiles) load_tile(t + 2);       // in flight while the other group converts the next tile
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Threshold hand-over between filter levels: Emax_next[q] = (k-th smallest TF32 energy among this level's
// candidates) + (largest error bound the level used for q).  One warp per query; no key reads.
template <int NS>
__global__ void __launch_bounds__(256) affinity_level_select_kernel(const SelectParams p) {
  __shared__ float lv[8][KPAD_MAX];
  __shared__ int li[8][KPAD_MAX];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long bq = (long long)blockIdx.y * p.Q + (long long)blockIdx.x * 8 + warp;
  if ((long long)blockIdx.x * 8 + warp >= p.Q) return;
  const int n = p.count[bq];
  if (n > p.cap || n < p.top_k) {            // overflow (or impossible underflow): no usable bound
    if (lane == 0) p.emax_out[bq] = CUDART_INF_F;
    return;
  }
  for (int u = 0; u < NS; ++u) { lv[warp][lane + 32 * u] = -CUDART_INF_F; li[warp][lane + 32 * u] = INT_MAX; }
  __syncwarp();
  const float* ce = p.cand_e + bq * p.cap;
  for (int base = 0; base < n; base += 32) {
    const int j = base + lane;
    const float v = j < n ? -ce[j] : -CUDART_INF_F;       // rank by -E, descending
    const float kth = lv[warp][p.top_k - 1];
    unsigned bits = __ballot_sync(0xffffffffu, j < n && v > kth);
    while (bits) {
      const int src = __ffs(bits) - 1;
      bits &= bits - 1;
      const float cv = __shfl_sync(0xffffffffu, v, src);
      if (cv > lv[warp][p.top_k - 1]) list_insert<NS>(&lv[warp][0], &li[warp][0], lane, p.top_k, cv, base + src);
    }
  }
  if (lane == 0) {
    const float kth_e = -lv[warp][p.top_k - 1];
    const float bound = kth_e;                 // candidates carry upper bounds of their exact energies
    p.emax_out[bq] = bound + fabsf(bound) * 1e-6f + 1e-30f;
  }
}

// ------------------------------------------------------------------------------------------------
// Exact re-rank of the last level's candidates: one CTA (4 warps) per query.  Each warp evaluates chunks of 32
// candidates with the exact fp32 direct form and keeps a sorted top-k; warp 0 merges and finalises (softmax,
// usage).  A query whose candidate list overflowed is rescanned exhaustively (slow, correct, rare).
//
// Candidate key rows (256 B each) are fetched COALESCED -- a half-warp per row, 16 independent LDG.128 per lane in flight
// -- and staged in shared memory; each lane then evaluates its own candidate from shared memory with the same
// channel-sequential fp32 arithmetic as the exact scan (`exact_similarity_smem`), so results stay bit-identical.  (A lane
// reading its own row straight from global memory touches 32 different 128-byte lines per instruction: 512 L1 wavefronts
// per 32 candidates against 64 here, and the re-rank was bound by exactly that.)
constexpr int RR_LD = 68;                 // floats per staged row: 272 B, 16-byte aligned, conflict-free LDS.128 per quarter-warp

__device__ __forceinline__ float exact_similarity_smem(const float* __restrict__ krow, float shr, const float* __restrict__ a,
                                                       const float* __restrict__ b) {
  float acc = 0.f;
#pragma unroll
  for (int c4 = 0; c4 < CKD / 4; ++c4) {
    const float4 kf = *reinterpret_cast<const float4*>(krow + 4 * c4);
    float d;
    d = fmaf(a[4 * c4 + 0], kf.x, -b[4 * c4 + 0]); acc = fmaf(d, d, acc);
    d = fmaf(a[4 * c4 + 1], kf.y, -b[4 * c4 + 1]); acc = fmaf(d, d, acc);
    d = fmaf(a[4 * c4 + 2], kf.z, -b[4 * c4 + 2]); acc = fmaf(d, d, acc);
    d = fmaf(a[4 * c4 + 3], kf.w, -b[4 * c4 + 3]); acc = fmaf(d, d, acc);
  }
  return acc * (-shr * rsqrtf((float)CKD));
}

template <int NS>
__global__ void __launch_bounds__(128) affinity_rerank_kernel(const RerankParams p) {
  __shared__ float lv[4][KPAD_MAX];
  __shared__ int li[4][KPAD_MAX];
  __shared__ float qa[CKD], qb[CKD];
  __shared__ __align__(16) float rows[4][32][RR_LD];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y;
  const long long q = blockIdx.x;
  const long long bq = (long long)b * p.Q + q;
  for (int u = 0; u < NS; ++u) { lv[warp][lane + 32 * u] = -CUDART_INF_F; li[warp][lane + 32 * u] = INT_MAX; }
  if (tid < CKD) {
    const long long off = ((long long)b * CKD + tid) * p.Q + q;
    const float a = sqrtf(p.qe[off]);
    qa[tid] = a;
    qb[tid] = a * p.qk[off];
  }
  __syncthreads();
  int n = p.count[bq];
  const bool exhaustive = n > p.cap;
  if (exhaustive) n = (int)p.n_total;
  const int* cl = p.cand_idx + bq * p.cap;
  const int h = lane >> 4, c4 = lane & 15;
  for (int base = warp * 32; base < n; base += 128) {
    const int j = base + lane;
    int id = -1;
    if (j < n) id = exhaustive ? j : cl[j];
    const bool live = id >= 0;
    float shr = 0.f;
    const float* krow = nullptr;
    if (live) {
      const int sg = seg_of(p.segs.begin, p.segs.nseg, id);
      const long long off = (long long)id - p.segs.begin[sg];
      krow = p.segs.key[sg] + (long long)b * p.segs.key_bs[sg] + off * CKD;
      shr = __ldg(p.segs.shr[sg] + (long long)b * p.segs.shr_bs[sg] + off);
    }
    // cooperative, coalesced fetch: at step it the two half-warps fetch rows 2 it and 2 it + 1 (16 lanes x 16 B each)
    float4 piece[16];
#pragma unroll
    for (int it = 0; it < 16; ++it) {
      const unsigned long long rp = __shfl_sync(0xffffffffu, (unsigned long long)krow, 2 * it + h);
      piece[it] = rp ? __ldg(reinterpret_cast<const float4*>(rp) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int it = 0; it < 16; ++it) *reinterpret_cast<float4*>(&rows[warp][2 * it + h][4 * c4]) = piece[it];
    __syncwarp();
    const float sv = live ? exact_similarity_smem(&rows[warp][lane][0], shr, qa, qb) : -CUDART_INF_F;
    if (!live) id = INT_MAX;
    const float kth = lv[warp][p.top_k - 1];
    const int kthi = li[warp][p.top_k - 1];
    unsigned bits = __ballot_sync(0xffffffffu, live && (sv > kth || (sv == kth && id < kthi)));
    while (bits) {
      const int src = __ffs(bits) - 1;
      bits &= bits - 1;
      const float cs = __shfl_sync(0xffffffffu, sv, src);
      const int ci = __shfl_sync(0xffffffffu, id, src);
      const float k2 = lv[warp][p.top_k - 1];
      if (cs > k2 || (cs == k2 && ci < li[warp][p.top_k - 1]))
        list_insert<NS>(&lv[warp][0], &li[warp][0], lane, p.top_k, cs, ci);
    }
    __syncwarp();      // the staging rows are overwritten by the next chunk
  }
  __syncthreads();
  if (warp == 0) {
    for (int w = 1; w < 4; ++w) {
      for (int j = 0; j < p.top_k; ++j) {
        const float cs = lv[w][j];
        const int ci = li[w][j];
        if (ci == INT_MAX) break;
        const float k2 = lv[0][p.top_k - 1];
        if (!(cs > k2 || (cs == k2 && ci < li[0][p.top_k - 1]))) break;     // sorted: the rest lose too
        list_insert<NS>(&lv[0][0], &li[0][0], lane, p.top_k, cs, ci);
      }
    }
    const long long oo = bq * p.kpad;
    finalize_topk<NS>(&lv[0][0], &li[0][0], lane, p.top_k, p.kpad, p.out_idx + oo, p.out_w + oo,
                      p.out_sim ? p.out_sim + oo : nullptr,
                      p.usage_acc ? p.usage_acc + (long long)b * p.n_total : nullptr);
  }
}

size_t tc_filter_smem_bytes() { return (size_t)3 * OPER_BYTES + sizeof(TcSmemTail) + 64; }

int launch_tc_filter(const TcFilterParams& p, long long B, cudaStream_t st) {
  const size_t smem = tc_filter_smem_bytes();
  static bool attr_done[64] = {};
  if (first_use_on_device(attr_done)) {
    cudaFuncSetAttribute(affinity_tc_filter_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(affinity_tc_filter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  dim3 grid((unsigned)((p.Q + QT - 1) / QT), (unsigned)p.nsplit, (unsigned)B);
  if (p.dbg_energy)
    affinity_tc_filter_kernel<true><<<grid, TC_THREADS, smem, st>>>(p);
  else
    affinity_tc_filter_kernel<false><<<grid, TC_THREADS, smem, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("affinity_tc_filter_kernel", e);
  return 0;
}

int launch_level_select(const SelectParams& p, long long B, int kpad, cudaStream_t st) {
  dim3 grid((unsigned)((p.Q + 7) / 8), (unsigned)B);
  if (kpad == 32)
    affinity_level_select_kernel<1><<<grid, 256, 0, st>>>(p);
  else
    affinity_level_select_kernel<2><<<grid, 256, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("affinity_level_select_kernel", e);
  return 0;
}

int launch_rerank(const RerankParams& p, long long B, cudaStream_t st) {
  dim3 grid((unsigned)p.Q, (unsigned)B);
  if (p.kpad == 32)
    affinity_rerank_kernel<1><<<grid, 128, 0, st>>>(p);
  else
    affinity_rerank_kernel<2><<<grid, 128, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("affinity_rerank_kernel", e);
  return 0;
}

int tc_split_count(long long B, long long Q, long long samp_count) {
  const long long qtiles = (Q + QT - 1) / QT;
  const long long ntiles = (samp_count + KTILE - 1) / KTILE;
  long long s = num_sms() / (qtiles * B);
  if (s < 1) s = 1;
  if (s > ntiles) s = ntiles;
  if (s < 1) s = 1;
  return (int)s;
}

}  // namespace cutie
