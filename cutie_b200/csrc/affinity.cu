// Pixel-memory readout for sm_90a: similarity scan + exact streaming top-k, split merge + softmax, sparse value
// gather, usage commit; the plan (which passes run for a bank) and the host orchestration of both filtered plans --
// the TF32 levels of affinity_tc.cu and the FP16 image plan of affinity_f16.cu.  See include/cutie_b200.h for the
// contract and DESIGN.md for the roofline.
//
// Kernel 1  affinity_scan_kernel   grid (query tiles of 64, key splits, B), 256 threads, ~204 KB smem
//   Streams its split of the memory bank through a 2-stage cp.async pipeline of 128-token tiles
//   (token-major rows, 256 B each, padded to 272 B in smem so LDS.128 is conflict free), evaluates
//   S[n,q] = -shr[n]/sqrt(CK) * sum_c (a[q,c]*k[n,c] - b[q,c])^2 with a = sqrt(qe), b = a*qk
//   (2 FFMA per channel; cancellation free, unlike the reference's 3-term expansion), filters against
//   the per-query running k-th best, and pushes survivors into a CTA queue that the warps drain into
//   per-query sorted lists.  The [N,HW] similarity matrix never exists.
// Kernel 2  topk_merge_kernel      one warp per query: merges the per-split sorted lists, softmax over
//   the winners, optional fixed-point usage accumulation (deterministic).
// Kernel 3  readout_gather_kernel  one warp per query x object: gathers the k winning 1 KB value rows,
//   accumulates in registers, transposes through smem to the channel-major [B,K,CV,Q] output.
// Kernel 4  usage_commit_kernel    use_cnt += the fixed-point usage accumulators, life_cnt += 1.
#include <stdlib.h>

#include "topk_common.cuh"
#include "affinity_internal.cuh"

namespace cutie {
thread_local char g_last_error[512] = "";

constexpr int TQ = 64;     // queries per CTA
constexpr int TK = 128;    // memory tokens per tile
constexpr int NT = 256;    // threads per CTA
constexpr int LDT = 68;    // padded smem row stride (floats)
constexpr int QCAP = TQ * TK;

struct ScanParams {
  KeySegments segs;
  const float* qk;
  const float* qe;
  long long Q;
  long long n_total;
  long long samp_begin, samp_stride, samp_count;   // virtual index i -> token samp_begin + i*samp_stride
  int top_k;
  int kpad;
  int tiles_per_split;
  int nsplit;
  float* part_val;  // [B][nsplit][Q][kpad]
  int* part_idx;
};

struct ScanSmem {
  float ks[2][TK][LDT];
  float as_[TQ][LDT];
  float bs_[TQ][LDT];
  unsigned long long queue[QCAP];
  float lval[TQ][KPAD_MAX];
  int lidx[TQ][KPAD_MAX];
  float sh[2][TK];
  float tau[TQ];
  int qcount[2];
};

__device__ __forceinline__ void load_key_tile(ScanSmem& sm, int stage, const ScanParams& p, int b, long long i0,
                                              long long i_end, int tid) {
  const int c4 = tid & 15;
#pragma unroll
  for (int it = 0; it < TK / 16; ++it) {
    int r = (tid >> 4) + 16 * it;
    long long i = i0 + r;
    float* dst = &sm.ks[stage][r][4 * c4];
    if (i < i_end) {
      const long long g = p.samp_begin + i * p.samp_stride;
      int s = seg_of(p.segs.begin, p.segs.nseg, g);
      const float* src = p.segs.key[s] + (long long)b * p.segs.key_bs[s] + (g - p.segs.begin[s]) * CKD + 4 * c4;
      cp_async16(dst, src);
    } else {
      *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  if (tid < TK) {
    long long i = i0 + tid;
    if (i < i_end) {
      const long long g = p.samp_begin + i * p.samp_stride;
      int s = seg_of(p.segs.begin, p.segs.nseg, g);
      cp_async4(&sm.sh[stage][tid], p.segs.shr[s] + (long long)b * p.segs.shr_bs[s] + (g - p.segs.begin[s]));
    } else {
      sm.sh[stage][tid] = 0.f;
    }
  }
}

template <int NS>
__global__ void __launch_bounds__(NT, 1) affinity_scan_kernel(const ScanParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ScanSmem& sm = *reinterpret_cast<ScanSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, split = blockIdx.y;
  const long long q0 = (long long)blockIdx.x * TQ;
  const long long split_begin = (long long)split * p.tiles_per_split * TK;
  long long split_end = split_begin + (long long)p.tiles_per_split * TK;
  if (split_end > p.samp_count) split_end = p.samp_count;
  const int ntiles = split_end > split_begin ? (int)((split_end - split_begin + TK - 1) / TK) : 0;
  const float scale = rsqrtf((float)CKD);

  // ---- prologue: query operands a = sqrt(qe), b = a*qk, transposed to [q][c]; empty lists ----
  for (int i = tid; i < CKD * TQ; i += NT) {
    int c = i / TQ, q = i % TQ;
    float e = 0.f, k = 0.f;
    if (q0 + q < p.Q) {
      long long off = ((long long)b * CKD + c) * p.Q + q0 + q;
      e = p.qe[off];
      k = p.qk[off];
    }
    float a = sqrtf(e);
    sm.as_[q][c] = a;
    sm.bs_[q][c] = a * k;
  }
  for (int i = tid; i < TQ * KPAD_MAX; i += NT) {
    (&sm.lval[0][0])[i] = -CUDART_INF_F;
    (&sm.lidx[0][0])[i] = INT_MAX;
  }
  if (tid < TQ) sm.tau[tid] = -CUDART_INF_F;
  if (tid < 2) sm.qcount[tid] = 0;
  if (ntiles > 0) load_key_tile(sm, 0, p, b, split_begin, split_end, tid);
  cp_async_commit();

  const int tn = tid & 15, tq = tid >> 4;
  for (int t = 0; t < ntiles; ++t) {
    const int st = t & 1;
    cp_async_wait<0>();
    __syncthreads();
    if (t + 1 < ntiles) load_key_tile(sm, st ^ 1, p, b, split_begin + (long long)(t + 1) * TK, split_end, tid);
    cp_async_commit();

    // ---- 8 tokens x 4 queries per thread ----
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
    for (int c4 = 0; c4 < CKD / 4; ++c4) {
      float4 kf[8], af[4], bf[4];
#pragma unroll
      for (int i = 0; i < 8; ++i) kf[i] = *reinterpret_cast<const float4*>(&sm.ks[st][tn + 16 * i][4 * c4]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        af[j] = *reinterpret_cast<const float4*>(&sm.as_[tq + 16 * j][4 * c4]);
        bf[j] = *reinterpret_cast<const float4*>(&sm.bs_[tq + 16 * j][4 * c4]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float d;
          d = fmaf(af[j].x, kf[i].x, -bf[j].x); acc[i][j] = fmaf(d, d, acc[i][j]);
          d = fmaf(af[j].y, kf[i].y, -bf[j].y); acc[i][j] = fmaf(d, d, acc[i][j]);
          d = fmaf(af[j].z, kf[i].z, -bf[j].z); acc[i][j] = fmaf(d, d, acc[i][j]);
          d = fmaf(af[j].w, kf[i].w, -bf[j].w); acc[i][j] = fmaf(d, d, acc[i][j]);
        }
    }
    // ---- threshold filter -> CTA queue ----
    float tauq[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) tauq[j] = sm.tau[tq + 16 * j];
    const long long tile_g0 = split_begin + (long long)t * TK;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = tn + 16 * i;
      const float sscale = -sm.sh[st][r] * scale;
      const bool valid = tile_g0 + r < split_end;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float s = acc[i][j] * sscale;
        const bool pass = valid && (q0 + tq + 16 * j < p.Q) && (s > tauq[j]);
        const unsigned m = __ballot_sync(0xffffffffu, pass);
        if (m) {
          int base = 0;
          if (lane == 0) base = atomicAdd(&sm.qcount[st], __popc(m));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (pass) {
            const int slot = base + __popc(m & ((1u << lane) - 1u));
            const unsigned lo = ((unsigned)(tq + 16 * j) << 24) | (unsigned)(t * TK + r);
            sm.queue[slot] = ((unsigned long long)__float_as_uint(s) << 32) | lo;
          }
        }
      }
    }
    __syncthreads();
    // ---- drain: warp w owns queries q with q % 8 == w ----
    const int qn = sm.qcount[st];
    if (tid == 0) sm.qcount[st ^ 1] = 0;
    for (int base = 0; base < qn; base += 32) {
      const int e = base + lane;
      unsigned long long ent = 0ull;
      bool mine = false;
      if (e < qn) {
        ent = sm.queue[e];
        mine = (((unsigned)(ent >> 24) & 0xffu) & 7u) == (unsigned)warp;
      }
      unsigned bits = __ballot_sync(0xffffffffu, mine);
      while (bits) {
        const int src = __ffs(bits) - 1;
        bits &= bits - 1;
        const unsigned long long ce = __shfl_sync(0xffffffffu, ent, src);
        const float s = __uint_as_float((unsigned)(ce >> 32));
        const int ql = (int)((ce >> 24) & 0xffu);
        const int idx = (int)(p.samp_begin + (split_begin + (long long)(ce & 0xffffffu)) * p.samp_stride);
        const float kth = sm.lval[ql][p.top_k - 1];
        if (s > kth || (s == kth && idx < sm.lidx[ql][p.top_k - 1])) {
          float tau = list_insert<NS>(&sm.lval[ql][0], &sm.lidx[ql][0], lane, p.top_k, s, idx);
          if (lane == 0) sm.tau[ql] = tau;
          __syncwarp();
        }
      }
    }
  }
  __syncthreads();
  // ---- write this split's sorted lists ----
  const int kp = p.kpad;
  for (int i = tid; i < TQ * kp; i += NT) {
    int q = i / kp, j = i % kp;
    if (q0 + q < p.Q) {
      long long o = (((long long)b * p.nsplit + split) * p.Q + q0 + q) * kp + j;
      p.part_val[o] = sm.lval[q][j];
      p.part_idx[o] = sm.lidx[q][j];
    }
  }
}

struct MergeParams {
  const float* part_val;
  const int* part_idx;
  long long Q;
  long long n_total;
  int nsplit, top_k, kpad;
  int* out_idx;
  float* out_w;
  float* out_sim;
  unsigned long long* usage_acc;
};

template <int NS>
__global__ void __launch_bounds__(256) topk_merge_kernel(const MergeParams p) {
  __shared__ float lv[8][KPAD_MAX];
  __shared__ int li[8][KPAD_MAX];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const long long q = (long long)blockIdx.x * 8 + warp;
  if (q >= p.Q) return;
  const int kp = p.kpad;
  for (int u = 0; u < NS; ++u) { lv[warp][lane + 32 * u] = -CUDART_INF_F; li[warp][lane + 32 * u] = INT_MAX; }
  __syncwarp();
  // split 0 is already sorted: adopt it wholesale
  {
    const long long o = (((long long)b * p.nsplit) * p.Q + q) * kp;
    for (int u = 0; u < NS; ++u) {
      int slot = lane + 32 * u;
      if (slot < p.top_k) {
        const int ci = p.part_idx[o + slot];
        const bool dead = ci < 0 || ci == INT_MAX;          // -1 (public output format) or INT_MAX (scan lists)
        lv[warp][slot] = dead ? -CUDART_INF_F : p.part_val[o + slot];
        li[warp][slot] = dead ? INT_MAX : ci;
      }
    }
    __syncwarp();
  }
  for (int s = 1; s < p.nsplit; ++s) {
    const long long o = (((long long)b * p.nsplit + s) * p.Q + q) * kp;
    for (int j = 0; j < p.top_k; ++j) {
      const float cv = p.part_val[o + j];
      const int ci = p.part_idx[o + j];
      if (ci == INT_MAX || ci < 0) break;             // end of this split's list
      const float kth = lv[warp][p.top_k - 1];
      const int kthi = li[warp][p.top_k - 1];
      if (!(cv > kth || (cv == kth && ci < kthi))) break;   // sorted: the rest are worse too
      list_insert<NS>(&lv[warp][0], &li[warp][0], lane, p.top_k, cv, ci);
    }
  }
  const long long oo = ((long long)b * p.Q + q) * kp;
  finalize_topk<NS>(&lv[warp][0], &li[warp][0], lane, p.top_k, kp, p.out_idx + oo, p.out_w + oo,
                    p.out_sim ? p.out_sim + oo : nullptr,
                    p.usage_acc ? p.usage_acc + (long long)b * p.n_total : nullptr);
}

// ------------------------------------------------------------------------------------------------
struct GatherParams {
  const int* idx;
  const float* w;
  long long Q;
  int kpad;
  RowSegments segs;
  long long K, CV;
  float* out;
};

constexpr int GQ = 32;  // queries per CTA in the gather kernel

// CV == 256: each lane owns 8 channels (two float4) of the output row.
__global__ void __launch_bounds__(256) readout_gather_kernel(const GatherParams p) {
  __shared__ float tile[256][GQ + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int k = blockIdx.y, b = blockIdx.z;
  const long long q0 = (long long)blockIdx.x * GQ;
  const int ns = p.kpad / 32;
  for (int qi = warp; qi < GQ; qi += 8) {
    const long long q = q0 + qi;
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
    if (q < p.Q) {
      const long long o = ((long long)b * p.Q + q) * p.kpad;
      for (int u = 0; u < ns; ++u) {
        const int myi = p.idx[o + lane + 32 * u];
        const float myw = p.w[o + lane + 32 * u];
        unsigned livem = __ballot_sync(0xffffffffu, myi >= 0);   // holes allowed (sharded banks own a subset)
        while (livem) {
          // up to 4 winners per trip so several 1 KB row reads are in flight
          int js[4];
          int cnt = 0;
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            if (livem) { js[t] = __ffs(livem) - 1; livem &= livem - 1; ++cnt; } else { js[t] = -1; }
          }
          float4 v0[4], v1[4];
          float wj[4];
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            if (t < cnt) {
              const int id = __shfl_sync(0xffffffffu, myi, js[t]);
              wj[t] = __shfl_sync(0xffffffffu, myw, js[t]);
              const int s = seg_of(p.segs.begin, p.segs.nseg, id);
              const float* row = p.segs.rows[s * p.segs.nobj + k] + (long long)b * p.segs.bs[s * p.segs.nobj + k] +
                                 ((long long)id - p.segs.begin[s]) * 256;
              v0[t] = __ldg(reinterpret_cast<const float4*>(row) + lane);
              v1[t] = __ldg(reinterpret_cast<const float4*>(row) + 32 + lane);
            }
          }
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            if (t < cnt) {
              a0.x = fmaf(wj[t], v0[t].x, a0.x); a0.y = fmaf(wj[t], v0[t].y, a0.y);
              a0.z = fmaf(wj[t], v0[t].z, a0.z); a0.w = fmaf(wj[t], v0[t].w, a0.w);
              a1.x = fmaf(wj[t], v1[t].x, a1.x); a1.y = fmaf(wj[t], v1[t].y, a1.y);
              a1.z = fmaf(wj[t], v1[t].z, a1.z); a1.w = fmaf(wj[t], v1[t].w, a1.w);
            }
          }
        }
      }
    }
    const int c0 = 4 * lane;
    tile[c0 + 0][qi] = a0.x; tile[c0 + 1][qi] = a0.y; tile[c0 + 2][qi] = a0.z; tile[c0 + 3][qi] = a0.w;
    tile[128 + c0 + 0][qi] = a1.x; tile[128 + c0 + 1][qi] = a1.y; tile[128 + c0 + 2][qi] = a1.z; tile[128 + c0 + 3][qi] = a1.w;
  }
  __syncthreads();
  // channel-major store: out[b][k][c][q0 + lane]
  for (int c = warp; c < 256; c += 8) {
    const long long q = q0 + lane;
    if (q < p.Q) p.out[(((long long)b * p.K + k) * 256 + c) * p.Q + q] = tile[c][lane];
  }
}

__global__ void usage_commit_kernel(float* use, long long ubs, float* life, long long lbs,
                                    const unsigned long long* acc, long long abs_, long long off, long long n) {
  const int b = blockIdx.y;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double inc = (double)acc[(long long)b * abs_ + off + i] * (1.0 / (double)(1ull << CUTIE_B200_USAGE_FRAC_BITS));
    use[(long long)b * ubs + i] += (float)inc;
    life[(long long)b * lbs + i] += 1.f;
  }
}

static int pick_splits(long long B, long long Q, long long count) {
  const long long qtiles = (Q + TQ - 1) / TQ;
  const long long ntiles = (count + TK - 1) / TK;
  long long s = num_sms() / (qtiles * B);
  if (s < 1) s = 1;
  if (s > ntiles) s = ntiles;
  if (s < 1) s = 1;
  return (int)s;
}

// ---- plan: which passes run for a bank of n_total tokens ------------------------------------------------
// exact  (levels == 0): n_total < tc_min                 exact fp32 scan of everything (affinity_scan_kernel)
// filter (levels >= 1): nested strided samples, coarsest first (strides ... 256, 16, 1).  The coarsest sample has
//                       <= TC_CAP tokens so every one of them is a candidate; each level hands an upper bound of its
//                       k-th smallest energy to the next; the last level (stride 1) is re-ranked exactly.
struct Plan {
  int levels;             // 0 = exact scan only
  long long stride[8];    // coarsest first, last == 1
};
constexpr int TC_CAP = 4096;           // candidate slots per query (also the largest all-pass coarsest sample)
constexpr int TC_CAP_BIG = 16384;      // slots per query used for the candidate lists (overflow => exhaustive rescan of that query)

static long long g_tc_min_override = -1;
static long long g_image_level_launches = 0;     // calls served by the FP16 image plan (tests / diagnostics)

static long long tc_min_tokens() {
  if (g_tc_min_override >= 0) return g_tc_min_override;
  static long long v = -1;
  if (v < 0) {
    const char* e = getenv("CUTIE_B200_TC_MIN");
    v = e ? atoll(e) : 6144;
    const char* off = getenv("CUTIE_B200_NO_TC");
    if (off && off[0] == '1') v = (1ll << 40);
  }
  return v;
}

static Plan make_plan(long long n_total, int top_k) {
  Plan pl;
  pl.levels = 0;
  if (n_total < tc_min_tokens() || n_total < 2 * (long long)top_k) return pl;
  long long st[8];
  int n = 0;
  st[n++] = 1;
  while ((n_total + st[n - 1] - 1) / st[n - 1] > TC_CAP && n < 8) { st[n] = st[n - 1] * 16; ++n; }
  // the coarsest sample must still hold at least 2k tokens to give a meaningful bound
  while (n > 1 && (n_total + st[n - 1] - 1) / st[n - 1] < 2 * (long long)top_k) --n;
  if ((n_total + st[n - 1] - 1) / st[n - 1] > TC_CAP) return pl;      // cannot seed the thresholds: exact scan
  pl.levels = n;
  for (int i = 0; i < n; ++i) pl.stride[i] = st[n - 1 - i];
  return pl;
}

struct WsLayout {
  size_t part, cand_idx, cand_e, count, dmax, emax0, emax1;   // byte offsets
  size_t total;
};

// What every plan writes: cutie_affinity_topk's out_idx / out_w and its optional out_sim / usage_acc.
struct TopkOut {
  int* idx;
  float* w;
  float* sim;
  unsigned long long* usage_acc;
};

static size_t ws_take(size_t& off, size_t bytes) {
  const size_t o = off;
  off += (bytes + 255) / 256 * 256;
  return o;
}

// Workspace of the filtered plans from `off` on: per-query candidate lists, their counters, two threshold buffers.
static void filtered_ws_layout(WsLayout& w, size_t& off, long long B, long long Q) {
  w.cand_idx = ws_take(off, (size_t)B * Q * TC_CAP_BIG * 4);
  w.cand_e = ws_take(off, (size_t)B * Q * TC_CAP_BIG * 4);
  w.count = ws_take(off, (size_t)B * Q * 4);
  w.dmax = ws_take(off, (size_t)B * Q * 4);
  w.emax0 = ws_take(off, (size_t)B * Q * 4);
  w.emax1 = ws_take(off, (size_t)B * Q * 4);
}

static WsLayout ws_layout(long long B, long long Q, long long n_total, int top_k) {
  const int kpad = top_k <= 32 ? 32 : 64;
  WsLayout w;
  memset(&w, 0, sizeof(w));
  size_t off = 0;
  if (make_plan(n_total, top_k).levels == 0)
    w.part = ws_take(off, (size_t)B * pick_splits(B, Q, n_total) * Q * kpad * 8);
  else
    filtered_ws_layout(w, off, B, Q);
  w.total = off + 256;
  return w;
}

// Merge `nsplit` sorted lists per query into the top-k + softmax (topk_merge_kernel).
static int launch_merge(const float* part_val, const int* part_idx, long long B, long long Q, long long n_total,
                        int nsplit, int top_k, int kpad, const TopkOut& out, cudaStream_t st) {
  MergeParams mp;
  mp.part_val = part_val;
  mp.part_idx = part_idx;
  mp.Q = Q;
  mp.n_total = n_total;
  mp.nsplit = nsplit;
  mp.top_k = top_k;
  mp.kpad = kpad;
  mp.out_idx = out.idx;
  mp.out_w = out.w;
  mp.out_sim = out.sim;
  mp.usage_acc = out.usage_acc;
  dim3 mgrid((unsigned)((Q + 7) / 8), (unsigned)B);
  if (kpad == 32)
    topk_merge_kernel<1><<<mgrid, 256, 0, st>>>(mp);
  else
    topk_merge_kernel<2><<<mgrid, 256, 0, st>>>(mp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("topk_merge_kernel", e);
  return 0;
}

static int run_exact(const ScanParams& base, long long B, int nsplit, const TopkOut& out, cudaStream_t st) {
  ScanParams sp = base;
  const long long ntiles = (sp.samp_count + TK - 1) / TK;
  sp.nsplit = nsplit;
  sp.tiles_per_split = (int)((ntiles + nsplit - 1) / nsplit);
  if ((long long)sp.tiles_per_split * TK >= (1ll << 24)) return fail(-1, "%s: split too long", "run_exact");
  dim3 grid((unsigned)((sp.Q + TQ - 1) / TQ), (unsigned)nsplit, (unsigned)B);
  const size_t smem = sizeof(ScanSmem);
  static bool attr_done[64] = {};
  if (first_use_on_device(attr_done)) {
    cudaFuncSetAttribute(affinity_scan_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(affinity_scan_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  if (sp.kpad == 32)
    affinity_scan_kernel<1><<<grid, NT, smem, st>>>(sp);
  else
    affinity_scan_kernel<2><<<grid, NT, smem, st>>>(sp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("affinity_scan_kernel", e);
  return launch_merge(sp.part_val, sp.part_idx, B, sp.Q, sp.n_total, nsplit, sp.top_k, sp.kpad, out, st);
}

// Optional per-phase timing of the filtered plan (diagnostics: bench.py --phase-timing).  Events are recorded on
// the caller's stream, so they measure the kernels in situ; nothing synchronises until the times are read.
constexpr int PH_RING = 64, PH_MAX = 16;
static bool g_phase_on = false;
static cudaEvent_t g_phase_ev[PH_RING][PH_MAX];
static int g_phase_n[PH_RING];
static long long g_phase_calls = 0;
static bool g_phase_init = false;

static void phase_mark(int slot, cudaStream_t st) {
  if (!g_phase_on || slot < 0) return;
  if (g_phase_n[slot] < PH_MAX) cudaEventRecord(g_phase_ev[slot][g_phase_n[slot]++], st);
}
static int phase_begin(cudaStream_t st) {
  if (!g_phase_on) return -1;
  if (!g_phase_init) {
    for (int i = 0; i < PH_RING; ++i)
      for (int j = 0; j < PH_MAX; ++j) cudaEventCreate(&g_phase_ev[i][j]);
    g_phase_init = true;
  }
  const int slot = (int)(g_phase_calls++ % PH_RING);
  g_phase_n[slot] = 0;
  phase_mark(slot, st);
  return slot;
}

// Exact re-rank of the candidate lists a filtered plan left in the workspace (affinity_rerank_kernel).
static int rerank_candidates(const ScanParams& base, long long B, char* ws, const WsLayout& wl, const TopkOut& out,
                             cudaStream_t st) {
  RerankParams rp;
  memset(&rp, 0, sizeof(rp));
  rp.segs = base.segs;
  rp.qk = base.qk;
  rp.qe = base.qe;
  rp.Q = base.Q;
  rp.n_total = base.n_total;
  rp.cand_idx = (const int*)(ws + wl.cand_idx);
  rp.count = (const int*)(ws + wl.count);
  rp.cap = TC_CAP_BIG;
  rp.top_k = base.top_k;
  rp.kpad = base.kpad;
  rp.out_idx = out.idx;
  rp.out_w = out.w;
  rp.out_sim = out.sim;
  rp.usage_acc = out.usage_acc;
  return launch_rerank(rp, B, st);
}

// One filter level: zero the per-query counters, wgmma filter over the stride-`stride` sample.
static int run_filter_level(const ScanParams& base, long long B, long long stride, const float* emax_in, char* ws,
                            const WsLayout& wl, float* dbg_energy, cudaStream_t st) {
  TcFilterParams fp;
  memset(&fp, 0, sizeof(fp));
  fp.segs = base.segs;
  fp.qk = base.qk;
  fp.qe = base.qe;
  fp.Q = base.Q;
  fp.samp_begin = 0;
  fp.samp_stride = stride;
  fp.samp_count = (base.n_total + stride - 1) / stride;
  fp.nsplit = tc_split_count(B, base.Q, fp.samp_count);
  const long long ntiles = (fp.samp_count + 127) / 128;
  fp.tiles_per_split = (int)((ntiles + fp.nsplit - 1) / fp.nsplit);
  fp.emax_in = emax_in;
  fp.cand_idx = (int*)(ws + wl.cand_idx);
  fp.cand_e = (float*)(ws + wl.cand_e);
  fp.count = (int*)(ws + wl.count);
  fp.dmax = (float*)(ws + wl.dmax);
  fp.cap = TC_CAP_BIG;
  fp.dbg_energy = dbg_energy;
  cudaError_t e = cudaMemsetAsync(ws + wl.count, 0, (size_t)(wl.emax0 - wl.count), st);   // count + dmax
  if (e != cudaSuccess) return set_cuda_error("cudaMemsetAsync", e);
  return launch_tc_filter(fp, B, st);
}

// Where the image tiles of the bank `segs` are, from the caller's per-segment images (cutie_affinity_topk_img:
// seg_image_bstride in floats, seg_phys_begin = index of the segment's first token inside its arena).  Returns 1 when
// every non-empty segment has an image (the FP16 plan can run), 0 when one has none (the TF32 levels convert the keys
// on the fly), < 0 for an invalid argument, reported under the name `fn`.
static int image_tiles(ImageTiles& t, const KeySegments& segs, const void* const* seg_key_image,
                       const int64_t* seg_image_bstride, const int64_t* seg_phys_begin, const char* fn) {
  memset(&t, 0, sizeof(t));
  if (!seg_key_image) return 0;
  if (!seg_image_bstride || !seg_phys_begin)
    return fail(-1, "%s: invalid argument: image strides / physical offsets missing", fn);
  int on = 1;
  long long cum = 0;
  for (int s = 0; s < segs.nseg; ++s) {
    const long long n = segs.begin[s + 1] - segs.begin[s];
    if (n > 0 && !seg_key_image[s]) on = 0;
    if (seg_phys_begin[s] < 0) return fail(-1, "%s: invalid argument: negative physical offset", fn);
    if (((uintptr_t)seg_key_image[s] & 15) != 0)
      return fail(-1, "%s: invalid argument: key image must be 16-byte aligned", fn);
    t.img[s] = (const unsigned char*)seg_key_image[s];
    t.bs[s] = seg_image_bstride[s] * 4;
    t.tile0[s] = seg_phys_begin[s] / 128;
    t.lo0[s] = (int)(seg_phys_begin[s] % 128);
    t.tcum[s] = cum;
    cum += n > 0 ? (t.lo0[s] + n + 127) / 128 : 0;
  }
  for (int s = segs.nseg; s <= kMaxSeg; ++s) t.tcum[s] = cum;
  return on;
}

// FP16 plan over the key operand image: tile-sampled threshold pass -> k-th smallest slot minimum -> candidate filter
// over the whole image -> exact re-rank.  Two memsets + four launches per call, whatever the bank size.
// key_mu [B][64]: the key centre of the images (null = 0); seed_idx [B][Q][kpad]: threshold seeds (null = none).
static int run_filtered_f16(const ScanParams& base, long long B, const ImageTiles& tiles, const float* key_mu,
                            const int* seed_idx, char* ws, const WsLayout& wl, const TopkOut& out, cudaStream_t st) {
  F16FilterParams fp;
  memset(&fp, 0, sizeof(fp));
  fp.segs = base.segs;
  fp.qk = base.qk;
  fp.qe = base.qe;
  fp.key_mu = key_mu;
  fp.Q = base.Q;
  fp.tiles = tiles;
  const int grid_x = f16_schedule(fp, B);
  const int groups = (fp.full_groups > 0 ? fp.splits_full : fp.splits_half) * 2 * F16_SLOTS;    // threshold slots per query
  if (groups > TC_CAP_BIG) return fail(-1, "%s: too many key splits for the threshold workspace", "run_filtered_f16");
  // sample every `stride`-th tile: every split of a query group should still see >= 8 tiles (its 64 slots then hold
  // minima over >= 16 tokens each); small banks are sampled whole
  const long long max_splits = fp.full_groups > 0 ? fp.splits_full : fp.splits_half;
  long long stride = tiles.tcum[base.segs.nseg] / (8ll * max_splits);
  if (stride > 8) stride = 8;
  if (stride < 1) stride = 1;
  const int ph = phase_begin(st);
  float* group_min = (float*)(ws + wl.cand_e);
  float* emax = (float*)(ws + wl.emax0);
  cudaError_t e = cudaMemsetAsync(group_min, 0x7f, (size_t)B * base.Q * groups * 4, st);      // 0x7f7f7f7f = 3.4e38: "empty slot"
  if (e != cudaSuccess) return set_cuda_error("cudaMemsetAsync", e);
  fp.tile_stride = (int)stride;
  fp.tile_phase = 0;
  fp.group_min = group_min;
  fp.groups_per_query = groups;
  int rc = launch_f16_filter(fp, B, grid_x, true, st);
  if (rc) return rc;
  phase_mark(ph, st);
  F16ThresholdParams tp;
  memset(&tp, 0, sizeof(tp));
  tp.group_min = group_min;
  tp.groups = groups;
  tp.top_k = base.top_k;
  tp.kpad = base.kpad;
  tp.Q = base.Q;
  tp.n_total = base.n_total;
  tp.emax_out = emax;
  tp.seed_idx = seed_idx;
  tp.segs = base.segs;
  tp.qk = base.qk;
  tp.qe = base.qe;
  rc = launch_f16_threshold(tp, B, st);
  if (rc) return rc;
  phase_mark(ph, st);
  e = cudaMemsetAsync(ws + wl.count, 0, (size_t)B * base.Q * 4, st);
  if (e != cudaSuccess) return set_cuda_error("cudaMemsetAsync", e);
  fp.emax_in = emax;
  fp.cand_idx = (int*)(ws + wl.cand_idx);
  fp.count = (int*)(ws + wl.count);
  fp.cap = TC_CAP_BIG;
  rc = launch_f16_filter(fp, B, grid_x, false, st);
  if (rc) return rc;
  ++g_image_level_launches;
  phase_mark(ph, st);
  rc = rerank_candidates(base, B, ws, wl, out, st);
  phase_mark(ph, st);
  return rc;
}

// TF32 plan: the filter levels, coarsest first, each handing its thresholds to the next -> exact re-rank.
static int run_filtered(const ScanParams& base, long long B, const Plan& pl, char* ws, const WsLayout& wl,
                        const TopkOut& out, float* dbg_energy, cudaStream_t st) {
  float* emax[2] = {(float*)(ws + wl.emax0), (float*)(ws + wl.emax1)};
  const float* emax_in = nullptr;
  const int ph = phase_begin(st);
  for (int l = 0; l < pl.levels; ++l) {
    const bool last = (l == pl.levels - 1);
    int rc = run_filter_level(base, B, pl.stride[l], emax_in, ws, wl, last ? dbg_energy : nullptr, st);
    if (rc) return rc;
    phase_mark(ph, st);
    if (!last) {
      SelectParams sp;
      sp.Q = base.Q;
      sp.cand_e = (const float*)(ws + wl.cand_e);
      sp.count = (const int*)(ws + wl.count);
      sp.dmax = (const float*)(ws + wl.dmax);
      sp.cap = TC_CAP_BIG;
      sp.top_k = base.top_k;
      sp.emax_out = emax[l & 1];
      rc = launch_level_select(sp, B, base.kpad, st);
      if (rc) return rc;
      phase_mark(ph, st);
      emax_in = emax[l & 1];
    }
  }
  const int rc = rerank_candidates(base, B, ws, wl, out, st);
  phase_mark(ph, st);
  return rc;
}

}  // namespace cutie

using namespace cutie;

extern "C" int cutie_b200_abi_version(void) { return CUTIE_B200_ABI_VERSION; }
extern "C" const char* cutie_b200_last_error(void) { return g_last_error; }

extern "C" size_t cutie_affinity_workspace_bytes(int64_t B, int64_t Q, int64_t n_total, int top_k) {
  return ws_layout(B, Q, n_total, top_k).total;
}

// Banks with fewer tokens than this use the exact scan only (default 6144; env CUTIE_B200_TC_MIN /
// CUTIE_B200_NO_TC=1).  Negative restores the default.  Process-wide; meant for tests and tuning.
extern "C" void cutie_set_tc_min_tokens(int64_t n) { g_tc_min_override = n; }

// Per-phase device times (ms) of a filtered cutie_affinity_topk call: filter level, threshold select, ..., re-rank.
// cutie_debug_phase_timing(1) starts recording (a ring of the last 64 calls); cutie_debug_phase_times(calls_ago, ...)
// waits for that call's last event and returns the number of phases written.
extern "C" void cutie_debug_phase_timing(int enable) { g_phase_on = enable != 0; }
extern "C" int cutie_debug_phase_times(int64_t calls_ago, float* out_ms, int max_phases) {
  if (!g_phase_init || calls_ago < 0 || calls_ago >= PH_RING || calls_ago >= g_phase_calls || !out_ms) return 0;
  const int slot = (int)((g_phase_calls - 1 - calls_ago) % PH_RING);
  const int n = g_phase_n[slot];
  if (n < 2) return 0;
  if (cudaEventSynchronize(g_phase_ev[slot][n - 1]) != cudaSuccess) return 0;
  int k = 0;
  for (int i = 1; i < n && k < max_phases; ++i, ++k)
    if (cudaEventElapsedTime(&out_ms[k], g_phase_ev[slot][i - 1], g_phase_ev[slot][i]) != cudaSuccess) return k;
  return k;
}

// How many calls the FP16 image plan has served so far in this process (diagnostics / tests).
extern "C" int64_t cutie_debug_image_level_launches(void) { return g_image_level_launches; }

// Which plan cutie_affinity_topk will use: 0 = exact scan only, n >= 1 = n wgmma filter levels (see make_plan).
extern "C" int cutie_affinity_plan_levels(int64_t n_total, int top_k) { return make_plan(n_total, top_k).levels; }

// Diagnostics: byte offset of the per-query candidate counters [B][Q] int32 inside the workspace (-1: exact-scan plan).
extern "C" int64_t cutie_debug_ws_count_offset(int64_t B, int64_t Q, int64_t n_total, int top_k) {
  if (make_plan(n_total, top_k).levels == 0) return -1;
  return (int64_t)ws_layout(B, Q, n_total, top_k).count;
}

static int fill_scan_params(ScanParams& sp, int num_segments, const void* const* seg_key,
                            const void* const* seg_shrinkage, const int64_t* seg_len,
                            const int64_t* seg_key_bstride, const int64_t* seg_shr_bstride, const float* qk,
                            const float* qe, int64_t Q, int top_k, int kpad, int64_t n_total, const char* fn) {
  memset(&sp, 0, sizeof(sp));
  if (int rc = segment_table(sp.segs.begin, num_segments, seg_len, &n_total, fn)) return rc;
  for (int s = 0; s < num_segments; ++s) {
    sp.segs.key[s] = (const float*)seg_key[s];
    sp.segs.shr[s] = (const float*)seg_shrinkage[s];
    sp.segs.key_bs[s] = seg_key_bstride[s];
    sp.segs.shr_bs[s] = seg_shr_bstride[s];
  }
  sp.segs.nseg = num_segments;
  sp.qk = qk;
  sp.qe = qe;
  sp.Q = Q;
  sp.n_total = n_total;
  sp.top_k = top_k;
  sp.kpad = kpad;
  sp.samp_begin = 0;
  sp.samp_stride = 1;
  sp.samp_count = n_total;
  return 0;
}

extern "C" int cutie_affinity_topk_img(int num_segments, const void* const* seg_key,
                                       const void* const* seg_shrinkage, const int64_t* seg_len,
                                       const int64_t* seg_key_bstride, const int64_t* seg_shr_bstride,
                                       const void* const* seg_key_image, const int64_t* seg_image_bstride,
                                       const int64_t* seg_phys_begin, const float* key_mu, const int32_t* seed_idx,
                                       const float* qk, const float* qe, int64_t B,
                                       int64_t CK, int64_t Q, int top_k, int kpad, int32_t* out_idx, float* out_w,
                                       float* out_sim, unsigned long long* usage_acc, int64_t n_total,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  CUTIE_REQUIRE(CK == CKD, "CK must be 64");
  CUTIE_REQUIRE(kpad == 32 || kpad == 64, "kpad must be 32 or 64");
  CUTIE_REQUIRE(top_k >= 1 && top_k <= kpad, "1 <= top_k <= kpad");
  CUTIE_REQUIRE(B >= 1 && Q >= 1 && qk && qe && out_idx && out_w && workspace, "null/empty argument");
  CUTIE_REQUIRE(n_total >= top_k, "selected index k out of range (top_k > number of memory tokens)");
  CUTIE_REQUIRE(n_total < (1ll << 31), "bank too large for int32 indices");
  ScanParams sp;
  int rc = fill_scan_params(sp, num_segments, seg_key, seg_shrinkage, seg_len, seg_key_bstride, seg_shr_bstride, qk,
                            qe, Q, top_k, kpad, n_total, __func__);
  if (rc) return rc;
  const WsLayout wl = ws_layout(B, Q, n_total, top_k);
  CUTIE_REQUIRE(workspace_bytes >= wl.total, "workspace too small");
  char* ws = (char*)workspace;
  cudaStream_t st = (cudaStream_t)stream;
  const TopkOut out = {out_idx, out_w, out_sim, usage_acc};
  const Plan pl = make_plan(n_total, top_k);
  if (pl.levels == 0) {
    const int ns0 = pick_splits(B, Q, n_total);
    sp.part_val = (float*)(ws + wl.part);
    sp.part_idx = (int*)(ws + wl.part + (size_t)B * ns0 * Q * kpad * 4);
    return run_exact(sp, B, ns0, out, st);
  }
  ImageTiles tiles;
  const int with_images = image_tiles(tiles, sp.segs, seg_key_image, seg_image_bstride, seg_phys_begin, __func__);
  if (with_images < 0) return with_images;
  if (with_images) return run_filtered_f16(sp, B, tiles, key_mu, seed_idx, ws, wl, out, st);
  return run_filtered(sp, B, pl, ws, wl, out, nullptr, st);
}

extern "C" int cutie_affinity_topk(int num_segments, const void* const* seg_key, const void* const* seg_shrinkage,
                                   const int64_t* seg_len, const int64_t* seg_key_bstride,
                                   const int64_t* seg_shr_bstride, const float* qk, const float* qe, int64_t B,
                                   int64_t CK, int64_t Q, int top_k, int kpad, int32_t* out_idx, float* out_w,
                                   float* out_sim, unsigned long long* usage_acc, int64_t n_total, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  return cutie_affinity_topk_img(num_segments, seg_key, seg_shrinkage, seg_len, seg_key_bstride, seg_shr_bstride,
                                 nullptr, nullptr, nullptr, nullptr, nullptr, qk, qe, B, CK, Q, top_k, kpad, out_idx, out_w,
                                 out_sim,
                                 usage_acc, n_total, workspace, workspace_bytes, stream);
}

// Test hook: TF32 energies E[b,q,n] = -8 S of the wgmma filter for the whole bank (single level, no
// threshold; n_total <= 4096 so that every token fits the candidate list).  dbg_energy [B, Q, n_total] floats.
extern "C" int cutie_debug_tc_energy(int num_segments, const void* const* seg_key, const void* const* seg_shrinkage,
                                     const int64_t* seg_len, const int64_t* seg_key_bstride,
                                     const int64_t* seg_shr_bstride, const float* qk, const float* qe, int64_t B,
                                     int64_t Q, int64_t n_total, float* dbg_energy, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  CUTIE_REQUIRE(dbg_energy && workspace, "bad argument");
  CUTIE_REQUIRE(n_total <= TC_CAP, "debug hook handles at most 4096 tokens");
  ScanParams sp;
  int rc = fill_scan_params(sp, num_segments, seg_key, seg_shrinkage, seg_len, seg_key_bstride, seg_shr_bstride, qk,
                            qe, Q, 1, 32, n_total, __func__);
  if (rc) return rc;
  WsLayout wl;
  memset(&wl, 0, sizeof(wl));
  size_t off = 0;
  filtered_ws_layout(wl, off, B, Q);
  const size_t o_idx = ws_take(off, (size_t)B * Q * 32 * 4), o_w = ws_take(off, (size_t)B * Q * 32 * 4);   // unused outputs
  CUTIE_REQUIRE(workspace_bytes >= off, "workspace too small");
  Plan pl;
  pl.levels = 1;
  pl.stride[0] = 1;
  char* ws = (char*)workspace;
  const TopkOut out = {(int*)(ws + o_idx), (float*)(ws + o_w), nullptr, nullptr};
  return run_filtered(sp, B, pl, ws, wl, out, dbg_energy, (cudaStream_t)stream);
}

extern "C" int cutie_topk_merge(const float* part_val, const int32_t* part_idx, int64_t B, int64_t nparts, int64_t Q,
                                int top_k, int kpad, int32_t* out_idx, float* out_w, float* out_sim,
                                unsigned long long* usage_acc, int64_t n_total, void* stream) {
  CUTIE_REQUIRE(part_val && part_idx && out_idx && out_w, "null argument");
  CUTIE_REQUIRE(kpad == 32 || kpad == 64, "kpad must be 32 or 64");
  CUTIE_REQUIRE(top_k >= 1 && top_k <= kpad && nparts >= 1 && B >= 1 && Q >= 1, "bad sizes");
  const TopkOut out = {out_idx, out_w, out_sim, usage_acc};
  return launch_merge(part_val, part_idx, B, Q, n_total, (int)nparts, top_k, kpad, out, (cudaStream_t)stream);
}

extern "C" int cutie_readout_gather(const int32_t* idx, const float* w, int64_t B, int64_t Q, int kpad,
                                    int num_segments, const int64_t* seg_len, const void* const* seg_val,
                                    const int64_t* seg_val_bstride, int64_t K, int64_t CV, float* out, void* stream) {
  CUTIE_REQUIRE(CV == 256, "CV must be 256");
  CUTIE_REQUIRE(K >= 1, "at least one object");
  CUTIE_REQUIRE(kpad == 32 || kpad == 64, "kpad must be 32 or 64");
  CUTIE_REQUIRE(idx && w && out, "null argument");
  long long begin[kMaxSeg + 1];
  if (int rc = segment_table(begin, num_segments, seg_len, nullptr, __func__)) return rc;
  // The kernel's parameter block holds the row pointers of at most kMaxObj objects.  Each output plane out[b, k]
  // depends on object k alone, so larger calls launch once per group of kMaxObj objects with `out` offset by the
  // group; `K` stays the full count, the batch stride of `out`.
  for (long long k0 = 0; k0 < K; k0 += kMaxObj) {
    const int nk = (int)(K - k0 < kMaxObj ? K - k0 : kMaxObj);
    GatherParams gp;
    memset(&gp, 0, sizeof(gp));
    memcpy(gp.segs.begin, begin, sizeof(begin));
    for (int s = 0; s < num_segments; ++s)
      for (int k = 0; k < nk; ++k) {
        gp.segs.rows[s * nk + k] = (const float*)seg_val[s * K + k0 + k];
        gp.segs.bs[s * nk + k] = seg_val_bstride[s * K + k0 + k];
      }
    gp.segs.nseg = num_segments;
    gp.segs.nobj = nk;
    gp.idx = idx;
    gp.w = w;
    gp.Q = Q;
    gp.kpad = kpad;
    gp.K = K;
    gp.CV = CV;
    gp.out = out + k0 * CV * Q;
    dim3 grid((unsigned)((Q + GQ - 1) / GQ), (unsigned)nk, (unsigned)B);
    readout_gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(gp);
    CUTIE_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int cutie_usage_commit(float* use_cnt, int64_t use_bstride, float* life_cnt, int64_t life_bstride,
                                  const unsigned long long* usage_acc, int64_t acc_bstride, int64_t acc_offset,
                                  int64_t B, int64_t n, void* stream) {
  CUTIE_REQUIRE(use_cnt && life_cnt && usage_acc, "null argument");
  if (n <= 0) return 0;
  dim3 grid((unsigned)((n + 255) / 256), (unsigned)B);
  usage_commit_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(use_cnt, use_bstride, life_cnt, life_bstride, usage_acc,
                                                             acc_bstride, acc_offset, n);
  CUTIE_CHECK_LAUNCH();
  return 0;
}
