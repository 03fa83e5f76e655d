// Memory-bank maintenance kernels: layout transposes into/out of the token-major arena, row gathers,
// long-term potentiation (dense softmax readout), streaming object-summary sum.
#include <math_constants.h>

#include "common.cuh"
#include "tc_operand_f16.cuh"

namespace cutie {

// Operand image of the wgmma affinity filter for tokens [phys0, phys0 + n) of an arena: every 128-token physical
// tile is stored exactly as the FP16 filter wants it in shared memory (tc_operand_f16.cuh), so the filter fetches a
// tile with ONE 36 KB bulk copy instead of converting 128 fp32 rows per tile per query block.
// 16 lanes per token (coalesced 256-B key rows), 16 tokens per 256-thread CTA.
// `mu` ([B][64] or null): the bank's key centre.  The image holds k - mu (and the filter's query operand qk - mu): the
// energy sum_c qe (k - qk)^2 does not change, but the error bound eps shr (|k - mu| + v')^2 shrinks with |k - mu| --
// network-derived keys sit on a large common mean (|mu| = 9.0 of |k| = 9.7 with the bench weights: an 8.5x smaller band).
__global__ void __launch_bounds__(256) key_image_kernel(const float* __restrict__ key, long long key_bs,
                                                        const float* __restrict__ shr, long long shr_bs,
                                                        const float* __restrict__ mu, long long phys0, long long n,
                                                        unsigned char* __restrict__ img, long long img_bs_bytes) {
  const int b = blockIdx.y;
  const int c4 = threadIdx.x & 15;
  const long long i = (long long)blockIdx.x * 16 + (threadIdx.x >> 4);
  const bool live = i < n;
  const long long phys = phys0 + (live ? i : 0);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  float sh = 0.f;
  if (live) {
    v = __ldg(reinterpret_cast<const float4*>(key + (long long)b * key_bs + phys * 64) + c4);
    sh = __ldg(shr + (long long)b * shr_bs + phys);
    if (mu) {
      const float4 m = __ldg(reinterpret_cast<const float4*>(mu + (long long)b * 64) + c4);
      v = make_float4(v.x - m.x, v.y - m.y, v.z - m.z, v.w - m.w);
    }
  }
  unsigned char* tile = img + (long long)b * img_bs_bytes + (phys >> 7) * (long long)F16_OPER_BYTES;
  store_key_row_operand_f16(tile, (int)(phys & 127), c4, v, sh, live);   // dead rows: shuffles only, no stores
}

// out[b][c][r] = in[b][r][c]   in: [B, R, C] (row stride C), out: [B, C, R]
__global__ void transpose_kernel(const float* __restrict__ in, long long in_bs, float* __restrict__ out,
                                 long long out_bs, long long R, long long C) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const long long r0 = (long long)blockIdx.y * 32, c0 = (long long)blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    long long r = r0 + i, c = c0 + tx;
    tile[i][tx] = (r < R && c < C) ? in[(long long)b * in_bs + r * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    long long c = c0 + i, r = r0 + tx;
    if (c < C && r < R) out[(long long)b * out_bs + c * R + r] = tile[tx][i];
  }
}

struct GatherRows {
  const float* rows[kMaxSeg];
  long long bs[kMaxSeg];
  long long begin[kMaxSeg + 1];
  int nseg;
};

__global__ void gather_rows_kernel(const GatherRows g, const long long* __restrict__ index, float* __restrict__ dst,
                                   long long dst_bs, long long m, long long C) {
  const int b = blockIdx.y;
  const long long j = blockIdx.x;
  const long long id = index[(long long)b * m + j];
  const int s = seg_of(g.begin, g.nseg, id);
  const float* src = g.rows[s] + (long long)b * g.bs[s] + (id - g.begin[s]) * C;
  float* d = dst + (long long)b * dst_bs + j * C;
  for (long long c = threadIdx.x; c < C; c += blockDim.x) d[c] = src[c];
}

__global__ void accumulate_kernel(float* __restrict__ acc, const float* __restrict__ add, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) acc[i] += add[i];
}

// ---- long-term potentiation -------------------------------------------------------------------
constexpr int PT = 4;  // prototypes per CTA

struct ConsParams {
  KeySegments segs;
  RowSegments vals;
  const float* pk;
  long long pk_bs;
  const float* pe;
  long long pe_bs;
  long long P, n_total, K;  // K: objects of THIS launch (at most kMaxObj)
  float* out_val[kMaxObj];
  long long out_val_bs[kMaxObj];
  float* out_shr;
  long long out_shr_bs;
  float* ws;  // [B][P][n_total]
  float* out_max;   // optional [B][P]: the softmax's max over the candidates (the per-shard affinity maximum of the sharded path)
  float* out_sum;   // optional [B][P]: sum_n exp(S[n,p] - max)
  int readout_only; // phases 1-2 ran in an earlier launch of this call: ws holds exp(S - max); only the values are read out
};

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
  return r;
}

__global__ void __launch_bounds__(256) consolidate_kernel(const ConsParams p) {
  __shared__ float a_s[PT][64], b_s[PT][64];
  __shared__ float red[8];
  __shared__ float inv_sum[PT];
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const long long p0 = (long long)blockIdx.x * PT;
  float* ws = p.ws + ((long long)b * p.P + p0) * p.n_total;
  if (p.readout_only) {
    // A later object group: the first launch left exp(S - max) in ws.  The normaliser is summed again in the order and
    // with the reduction of phase 2, so 1/se -- and every object's value rows -- are bit-identical to that launch's.
    for (int pp = 0; pp < PT; ++pp) {
      if (p0 + pp >= p.P) break;
      float se = 0.f;
      for (long long n = tid; n < p.n_total; n += 256) se += ws[(long long)pp * p.n_total + n];
      se = block_reduce(se, red, false);
      if (tid == 0) inv_sum[pp] = 1.f / se;
    }
  } else {
    for (int i = tid; i < PT * 64; i += 256) {
      int pp = i / 64, c = i % 64;
      float e = 0.f, k = 0.f;
      if (p0 + pp < p.P) {
        e = p.pe[(long long)b * p.pe_bs + (p0 + pp) * 64 + c];
        k = p.pk[(long long)b * p.pk_bs + (p0 + pp) * 64 + c];
      }
      float a = sqrtf(e);
      a_s[pp][c] = a;
      b_s[pp][c] = a * k;
    }
    __syncthreads();
    // phase 1: similarities of every candidate token against this CTA's prototypes
    float lmax[PT];
#pragma unroll
    for (int pp = 0; pp < PT; ++pp) lmax[pp] = -CUDART_INF_F;
    for (long long n = tid; n < p.n_total; n += 256) {
      const int s = seg_of(p.segs.begin, p.segs.nseg, n);
      const float4* row = reinterpret_cast<const float4*>(p.segs.key[s] + (long long)b * p.segs.key_bs[s] +
                                                          (n - p.segs.begin[s]) * 64);
      const float shr = p.segs.shr[s][(long long)b * p.segs.shr_bs[s] + (n - p.segs.begin[s])];
      float acc[PT];
#pragma unroll
      for (int pp = 0; pp < PT; ++pp) acc[pp] = 0.f;
#pragma unroll 4
      for (int c4 = 0; c4 < 16; ++c4) {
        const float4 kf = __ldg(row + c4);
#pragma unroll
        for (int pp = 0; pp < PT; ++pp) {
          float d;
          d = fmaf(a_s[pp][4 * c4 + 0], kf.x, -b_s[pp][4 * c4 + 0]); acc[pp] = fmaf(d, d, acc[pp]);
          d = fmaf(a_s[pp][4 * c4 + 1], kf.y, -b_s[pp][4 * c4 + 1]); acc[pp] = fmaf(d, d, acc[pp]);
          d = fmaf(a_s[pp][4 * c4 + 2], kf.z, -b_s[pp][4 * c4 + 2]); acc[pp] = fmaf(d, d, acc[pp]);
          d = fmaf(a_s[pp][4 * c4 + 3], kf.w, -b_s[pp][4 * c4 + 3]); acc[pp] = fmaf(d, d, acc[pp]);
        }
      }
#pragma unroll
      for (int pp = 0; pp < PT; ++pp) {
        const float sv = -acc[pp] * shr * 0.125f;
        if (p0 + pp < p.P) ws[(long long)pp * p.n_total + n] = sv;
        lmax[pp] = fmaxf(lmax[pp], sv);
      }
    }
    // phase 2: softmax statistics + shrinkage readout
    for (int pp = 0; pp < PT; ++pp) {
      if (p0 + pp >= p.P) break;
      const float mx = block_reduce(lmax[pp], red, true);
      float se = 0.f, ss = 0.f;
      for (long long n = tid; n < p.n_total; n += 256) {
        const float e = expf(ws[(long long)pp * p.n_total + n] - mx);
        ws[(long long)pp * p.n_total + n] = e;
        const int s = seg_of(p.segs.begin, p.segs.nseg, n);
        se += e;
        ss += e * p.segs.shr[s][(long long)b * p.segs.shr_bs[s] + (n - p.segs.begin[s])];
      }
      se = block_reduce(se, red, false);
      ss = block_reduce(ss, red, false);
      if (tid == 0) {
        inv_sum[pp] = 1.f / se;
        p.out_shr[(long long)b * p.out_shr_bs + p0 + pp] = ss / se;
        if (p.out_max) {
          p.out_max[(long long)b * p.P + p0 + pp] = mx;
          p.out_sum[(long long)b * p.P + p0 + pp] = se;
        }
      }
    }
  }
  __syncthreads();
  // phase 3: value readout, thread == channel (CV == 256 == blockDim)
  for (int k = 0; k < (int)p.K; ++k) {
    float acc[PT];
#pragma unroll
    for (int pp = 0; pp < PT; ++pp) acc[pp] = 0.f;
    for (int s = 0; s < p.segs.nseg; ++s) {
      const float* vrow = p.vals.rows[s * p.vals.nobj + k] + (long long)b * p.vals.bs[s * p.vals.nobj + k];
      const long long nb = p.segs.begin[s], ne = p.segs.begin[s + 1];
#pragma unroll 4
      for (long long n = nb; n < ne; ++n) {
        const float v = vrow[(n - nb) * 256 + tid];
#pragma unroll
        for (int pp = 0; pp < PT; ++pp) acc[pp] = fmaf(ws[(long long)pp * p.n_total + n], v, acc[pp]);
      }
    }
#pragma unroll
    for (int pp = 0; pp < PT; ++pp)
      if (p0 + pp < p.P) p.out_val[k][(long long)b * p.out_val_bs[k] + (p0 + pp) * 256 + tid] = acc[pp] * inv_sum[pp];
  }
}

}  // namespace cutie

using namespace cutie;

static int launch_transpose(const float* in, int64_t in_bs, float* out, int64_t out_bs, int64_t B, int64_t R,
                            int64_t C, void* stream, const char* fn) {
  if (!in || !out || B < 1 || R < 0 || C < 0) return fail(-1, "%s: invalid argument", fn);
  if (R == 0 || C == 0) return 0;
  dim3 grid((unsigned)((C + 31) / 32), (unsigned)((R + 31) / 32), (unsigned)B);
  transpose_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(in, in_bs, out, out_bs, R, C);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(fn, e);
  return 0;
}

extern "C" int cutie_bank_append(const float* src, int64_t src_bstride, float* dst_rows, int64_t dst_bstride,
                                 int64_t B, int64_t C, int64_t n, void* stream) {
  // src [B, C, n] -> dst [B, n, C]
  return launch_transpose(src, src_bstride, dst_rows, dst_bstride, B, C, n, stream, __func__);
}

extern "C" int cutie_bank_key_image(const float* key_arena, int64_t key_bstride, const float* shr_arena,
                                    int64_t shr_bstride, int64_t B, int64_t phys_begin, int64_t n, float* image,
                                    int64_t image_bstride, int64_t image_tiles, const float* key_mu, void* stream) {
  CUTIE_REQUIRE(key_arena && shr_arena && image && B >= 1 && phys_begin >= 0 && n >= 0, "null/negative argument");
  CUTIE_REQUIRE((phys_begin + n + 127) / 128 <= image_tiles, "image too small for the token range");
  CUTIE_REQUIRE(((uintptr_t)image & 15) == 0 && ((uintptr_t)key_arena & 15) == 0, "16-byte alignment required");
  if (n == 0) return 0;
  dim3 grid((unsigned)((n + 15) / 16), (unsigned)B);
  CUTIE_REQUIRE(key_mu == nullptr || ((uintptr_t)key_mu & 15) == 0, "key_mu must be 16-byte aligned");
  key_image_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(key_arena, key_bstride, shr_arena, shr_bstride, key_mu,
                                                         phys_begin, n, reinterpret_cast<unsigned char*>(image),
                                                         image_bstride * 4);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_bank_export(const float* rows, int64_t rows_bstride, float* dst, int64_t dst_bstride, int64_t B,
                                 int64_t C, int64_t n, void* stream) {
  // rows [B, n, C] -> dst [B, C, n]
  return launch_transpose(rows, rows_bstride, dst, dst_bstride, B, n, C, stream, __func__);
}

extern "C" int cutie_bank_gather(int num_segments, const void* const* seg_rows, const int64_t* seg_len,
                                 const int64_t* seg_bstride, const int64_t* index, float* dst_rows,
                                 int64_t dst_bstride, int64_t B, int64_t m, int64_t C, void* stream) {
  CUTIE_REQUIRE(index && dst_rows && B >= 1 && C >= 1, "null/empty argument");
  GatherRows g;
  memset(&g, 0, sizeof(g));
  if (int rc = segment_table(g.begin, num_segments, seg_len, nullptr, __func__)) return rc;
  if (m <= 0) return 0;
  for (int s = 0; s < num_segments; ++s) {
    g.rows[s] = (const float*)seg_rows[s];
    g.bs[s] = seg_bstride[s];
  }
  g.nseg = num_segments;
  dim3 grid((unsigned)m, (unsigned)B);
  int threads = C >= 256 ? 256 : (C >= 64 ? 64 : 32);
  gather_rows_kernel<<<grid, threads, 0, (cudaStream_t)stream>>>(g, (const long long*)index, dst_rows, dst_bstride, m, C);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_consolidate_partial(int num_segments, const void* const* seg_key, const void* const* seg_shrinkage,
                                         const int64_t* seg_len, const int64_t* seg_key_bstride,
                                         const int64_t* seg_shr_bstride, const void* const* seg_val,
                                         const int64_t* seg_val_bstride, int64_t K, const float* proto_key,
                                         int64_t pk_bstride, const float* proto_sel, int64_t ps_bstride, int64_t B,
                                         int64_t P, int64_t CK, int64_t CV, void* const* out_val,
                                         const int64_t* out_val_bstride, float* out_shr, int64_t out_shr_bstride,
                                         float* out_max, float* out_sumexp, float* workspace, int64_t n_total,
                                         void* stream) {
  CUTIE_REQUIRE((out_max == nullptr) == (out_sumexp == nullptr), "out_max and out_sumexp come together");
  CUTIE_REQUIRE(CK == 64, "CK must be 64");
  CUTIE_REQUIRE(K >= 0, "negative object count");
  CUTIE_REQUIRE(K == 0 || CV == 256, "CV must be 256");
  CUTIE_REQUIRE(proto_key && proto_sel && out_shr && workspace && P >= 1 && B >= 1, "null/empty argument");
  CUTIE_REQUIRE(n_total >= 1, "no candidate tokens");
  ConsParams cp;
  memset(&cp, 0, sizeof(cp));
  if (int rc = segment_table(cp.segs.begin, num_segments, seg_len, &n_total, __func__)) return rc;
  memcpy(cp.vals.begin, cp.segs.begin, sizeof(cp.vals.begin));
  for (int s = 0; s < num_segments; ++s) {
    cp.segs.key[s] = (const float*)seg_key[s];
    cp.segs.shr[s] = (const float*)seg_shrinkage[s];
    cp.segs.key_bs[s] = seg_key_bstride[s];
    cp.segs.shr_bs[s] = seg_shr_bstride[s];
  }
  cp.segs.nseg = cp.vals.nseg = num_segments;
  cp.pk = proto_key;
  cp.pk_bs = pk_bstride;
  cp.pe = proto_sel;
  cp.pe_bs = ps_bstride;
  cp.P = P;
  cp.n_total = n_total;
  cp.out_shr = out_shr;
  cp.out_shr_bs = out_shr_bstride;
  cp.ws = workspace;
  cp.out_max = out_max;
  cp.out_sum = out_sumexp;
  dim3 grid((unsigned)((P + PT - 1) / PT), (unsigned)B);
  // One launch per group of at most kMaxObj objects.  The first computes the similarities and softmax statistics (the
  // bulk of the work: P x n_total x 64 FMAs) and reads out its objects; later groups reuse the exp(S - max) it left in the
  // workspace and only read out their values.
  for (long long k0 = 0; k0 == 0 || k0 < K; k0 += kMaxObj) {
    const int nk = (int)(K - k0 < kMaxObj ? K - k0 : kMaxObj);
    for (int s = 0; s < num_segments; ++s)
      for (int k = 0; k < nk; ++k) {
        cp.vals.rows[s * nk + k] = (const float*)seg_val[s * K + k0 + k];
        cp.vals.bs[s * nk + k] = seg_val_bstride[s * K + k0 + k];
      }
    cp.vals.nobj = nk;
    cp.K = nk;
    for (int k = 0; k < nk; ++k) {
      cp.out_val[k] = (float*)out_val[k0 + k];
      cp.out_val_bs[k] = out_val_bstride[k0 + k];
    }
    cp.readout_only = k0 > 0;
    consolidate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(cp);
    CUTIE_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int cutie_consolidate(int num_segments, const void* const* seg_key, const void* const* seg_shrinkage,
                                 const int64_t* seg_len, const int64_t* seg_key_bstride,
                                 const int64_t* seg_shr_bstride, const void* const* seg_val,
                                 const int64_t* seg_val_bstride, int64_t K, const float* proto_key, int64_t pk_bstride,
                                 const float* proto_sel, int64_t ps_bstride, int64_t B, int64_t P, int64_t CK,
                                 int64_t CV, void* const* out_val, const int64_t* out_val_bstride, float* out_shr,
                                 int64_t out_shr_bstride, float* workspace, int64_t n_total, void* stream) {
  return cutie_consolidate_partial(num_segments, seg_key, seg_shrinkage, seg_len, seg_key_bstride, seg_shr_bstride, seg_val,
                                   seg_val_bstride, K, proto_key, pk_bstride, proto_sel, ps_bstride, B, P, CK, CV, out_val,
                                   out_val_bstride, out_shr, out_shr_bstride, nullptr, nullptr, workspace, n_total, stream);
}

extern "C" int cutie_obj_summary_accumulate(float* acc, const float* add, int64_t n, void* stream) {
  CUTIE_REQUIRE(acc && add && n >= 0, "null argument");
  if (n == 0) return 0;
  accumulate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(acc, add, n);
  CUTIE_CHECK_LAUNCH();
  return 0;
}
