// Object-transformer kernels for sm_90a (fp32).  Shapes are the model's fixed ones: embed 256, 8 heads
// of 32, 16 object queries; the pixel axis (HW) and the number of objects are free.
// All pixel-side tensors are channel-major [B*K, 256, HW] (what the cuDNN convolutions around these
// kernels produce and consume), so lanes run along the contiguous pixel axis.
// This file: the query-side kernels (skinny linears, head folds, 16x16 self attention) and the aux-mask pass; the two
// cross attentions run on the tensor cores (qt_tc.cu).
#include <math_constants.h>

#include <algorithm>

#include "common.cuh"
#include "qt_combine.cuh"

namespace cutie {

constexpr int E_ = 256;   // embed dim
constexpr int H_ = 8;     // heads
constexpr int DH = 32;    // head dim
constexpr int NQ = 16;    // object queries

// ------------------------------------------------------------------------------------------------
// skinny fused linear: y[M,N] = epi( pro(x)[M,Kd] . W[N,Kd]^T )
struct LinearParams {
  const float* x;
  long long M, Kd, ldx;
  const float* W;
  long long ldw, N;
  const float* bias;
  const float* ln_w;
  const float* ln_b;
  const float* pe;
  int summary_norm, relu;
  const float* residual;
  long long residual_mod;
  float* xhat_out;
  float* y;
};

// CTA tile 16 rows x 16 cols, 256 threads (one output each).  The reduction axis goes through smem in chunks of
// 256 (the whole axis for embed 256 => one barrier).  Each warp owns 2 x-rows and 2 W-rows of the tile and issues
// ALL of their global loads (x, positional term, LayerNorm affine, W) before touching any of them, so the prologue
// costs one memory latency; LayerNorm statistics are reduced in registers (same summation order as a two-pass
// row reduction: lane-strided partial sums, then a butterfly).  The next chunk is prefetched into registers while
// the current one is multiplied (Kd = 2048 in the FFN's second linear).
constexpr int LIN_BM = 16, LIN_BN = 16, LIN_KC = 256, LIN_LD = LIN_KC + 4;   // +4: 16-B aligned rows, conflict-free LDS.128

// Activation loads.  The stand-alone kernels read their inputs through the read-only path; inside qt_chain_kernel the
// inputs of an op were written by OTHER CTAs earlier in the same launch: they are read with ld.global.cg (L2, coherent,
// ordered with the grid barrier), never through the non-coherent path.  Weights / biases / positional terms are
// read-only for the whole launch and keep __ldg in both forms.
template <bool CHAIN>
__device__ __forceinline__ float ld_act(const float* p) { return CHAIN ? __ldcg(p) : __ldg(p); }
template <bool CHAIN>
__device__ __forceinline__ float ld_act_plain(const float* p) { return CHAIN ? __ldcg(p) : *p; }
template <bool CHAIN>
__device__ __forceinline__ float4 ld_act4(const float4* p) { return CHAIN ? __ldcg(p) : *p; }

// one 16 x 16 output tile (bx = column tile, by = row tile); 256 threads
template <bool CHAIN>
__device__ __forceinline__ void qt_linear_tile(const LinearParams& p, const int bx, const int by, float (*xs)[LIN_LD],
                                               float (*wsm)[LIN_LD]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long m0 = (long long)by * LIN_BM, n0 = (long long)bx * LIN_BN;
  const int r_t = tid >> 4, cg = tid & 15;
  float acc = 0.f;
  float xv[2][8], wv[2][8];
  auto load_chunk = [&](long long k0) {
    const int kc = (int)((p.Kd - k0) < LIN_KC ? (p.Kd - k0) : LIN_KC);
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long m = m0 + warp + 8 * u, n = n0 + warp + 8 * u;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int kk = lane + 32 * i;
        xv[u][i] = (m < p.M && kk < kc) ? ld_act<CHAIN>(p.x + m * p.ldx + k0 + kk) : 0.f;
        wv[u][i] = (n < p.N && kk < kc) ? __ldg(p.W + n * p.ldw + k0 + kk) : 0.f;
      }
    }
  };
  load_chunk(0);
  for (long long k0 = 0; k0 < p.Kd; k0 += LIN_KC) {
    const int kc = (int)((p.Kd - k0) < LIN_KC ? (p.Kd - k0) : LIN_KC);
    // ---- prologue on this warp's two x rows (registers), then publish the tile ----
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int r = warp + 8 * u;
      const long long m = m0 + r;
      const bool live = m < p.M;
      float pev[8], lw[8], lb[8];
      float den = 1.f;
      if (live && p.summary_norm) den = ld_act<CHAIN>(p.x + m * p.ldx + p.Kd);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int kk = lane + 32 * i;
        pev[i] = (p.pe && live && kk < kc) ? ld_act<CHAIN>(p.pe + m * p.Kd + k0 + kk) : 0.f;
        lw[i] = p.ln_w ? __ldg(p.ln_w + kk) : 1.f;
        lb[i] = p.ln_w ? __ldg(p.ln_b + kk) : 0.f;
      }
      if (p.summary_norm) {
        den = 1.f / (den + 1e-4f);
#pragma unroll
        for (int i = 0; i < 8; ++i) xv[u][i] *= den;
      }
      if (p.ln_w) {                       // Kd == 256: the whole row is in this warp's registers
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) sum += xv[u][i];
        const float mean = warp_sum(sum) / (float)p.Kd;
        float var = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) { const float d = xv[u][i] - mean; var += d * d; }
        const float rstd = rsqrtf(warp_sum(var) / (float)p.Kd + 1e-5f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float v = (xv[u][i] - mean) * rstd * lw[i] + lb[i];
          if (p.xhat_out && bx == 0 && live) p.xhat_out[m * p.Kd + lane + 32 * i] = v;
          xv[u][i] = v;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        xs[r][lane + 32 * i] = xv[u][i] + pev[i];
        wsm[r][lane + 32 * i] = wv[u][i];
      }
    }
    __syncthreads();
    if (k0 + LIN_KC < p.Kd) load_chunk(k0 + LIN_KC);       // in flight during the multiply
    const float4* xr = reinterpret_cast<const float4*>(&xs[r_t][0]);
    const float4* wr = reinterpret_cast<const float4*>(&wsm[cg][0]);
#pragma unroll 8
    for (int k4 = 0; k4 < LIN_KC / 4; ++k4) {
      const float4 a = xr[k4], w = wr[k4];
      acc = fmaf(a.x, w.x, acc);
      acc = fmaf(a.y, w.y, acc);
      acc = fmaf(a.z, w.z, acc);
      acc = fmaf(a.w, w.w, acc);
    }
    if (k0 + LIN_KC < p.Kd) __syncthreads();
  }
  const long long m = m0 + r_t, n = n0 + cg;
  if (m < p.M && n < p.N) {
    float v = acc + (p.bias ? p.bias[n] : 0.f);
    if (p.relu) v = fmaxf(v, 0.f);
    if (p.residual) v += ld_act_plain<CHAIN>(p.residual + (p.residual_mod ? (m % p.residual_mod) : m) * p.N + n);
    p.y[m * p.N + n] = v;
  }
}
__global__ void __launch_bounds__(256) qt_linear_kernel(const LinearParams p) {
  __shared__ __align__(16) float xs[LIN_BM][LIN_LD];
  __shared__ __align__(16) float wsm[LIN_BN][LIN_LD];
  qt_linear_tile<false>(p, (int)blockIdx.x, (int)blockIdx.y, xs, wsm);
}

// ------------------------------------------------------------------------------------------------
// out[m,h,c] = scale * sum_d a[m,h*32+d] * Wx[h*32+d, c];  grid M, block 256 (thread == c)
template <bool CHAIN>
__device__ __forceinline__ void qt_head_fold_tile(const float* __restrict__ a, const float* __restrict__ W, long long ldw,
                                                  int transpose_w, float scale, const float* __restrict__ bias_vec,
                                                  float* __restrict__ out, float* __restrict__ dots, const long long m,
                                                  const int h, float* as) {
  const int c = threadIdx.x;
  if (c < DH) as[c] = ld_act_plain<CHAIN>(a + m * E_ + h * DH + c);
  __syncthreads();
  float acc = 0.f;
#pragma unroll 8
  for (int d = 0; d < DH; ++d) {
    const int r = h * DH + d;
    const float w = transpose_w ? W[(long long)c * ldw + r] : W[(long long)r * ldw + c];
    acc = fmaf(as[d], w, acc);
  }
  out[(m * H_ + h) * E_ + c] = acc * scale;
  if (dots && c < DH) {
    float v = warp_sum(as[c] * bias_vec[h * DH + c]);
    if (c == 0) dots[m * H_ + h] = v * scale;
  }
}
__global__ void __launch_bounds__(256) qt_head_fold_kernel(const float* __restrict__ a, const float* __restrict__ W,
                                                           long long ldw, int transpose_w, float scale,
                                                           const float* __restrict__ bias_vec, float* __restrict__ out,
                                                           float* __restrict__ dots) {
  __shared__ float as[DH];
  qt_head_fold_tile<false>(a, W, ldw, transpose_w, scale, bias_vec, out, dots, (long long)blockIdx.x, (int)blockIdx.y, as);
}

// ------------------------------------------------------------------------------------------------
// self attention core: grid = objects (M/16), block 256 = 8 warps = 8 heads
struct SelfAttnSmem {
  float ks[H_][NQ][DH], vs[H_][NQ][DH], ps[H_][NQ][NQ + 1];
};
template <bool CHAIN>
__device__ __forceinline__ void qt_self_attention_tile(const float* __restrict__ qk, const float* __restrict__ v,
                                                       float* __restrict__ out, const long long obj, SelfAttnSmem& S) {
  const int tid = threadIdx.x, lane = tid & 31, h = tid >> 5;
  const long long m0 = obj * NQ;
  for (int i = tid; i < NQ * E_; i += 256) {
    const int r = i / E_, c = i % E_;
    S.ks[c / DH][r][c % DH] = ld_act_plain<CHAIN>(qk + (m0 + r) * 2 * E_ + E_ + c);
    S.vs[c / DH][r][c % DH] = ld_act_plain<CHAIN>(v + (m0 + r) * E_ + c);
  }
  const float scale = rsqrtf((float)DH);
  const int i = lane & 15, jh = lane >> 4;
  float qreg[DH];
  {
    const float4* qrow = reinterpret_cast<const float4*>(qk + (m0 + i) * 2 * E_ + h * DH);
#pragma unroll
    for (int d4 = 0; d4 < DH / 4; ++d4) {
      const float4 t = ld_act4<CHAIN>(qrow + d4);
      qreg[4 * d4 + 0] = t.x; qreg[4 * d4 + 1] = t.y; qreg[4 * d4 + 2] = t.z; qreg[4 * d4 + 3] = t.w;
    }
  }
  __syncthreads();
  float s[8], mx = -CUDART_INF_F;
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
    const int j = jh * 8 + jj;
    float acc = 0.f;
#pragma unroll
    for (int d = 0; d < DH; ++d) acc = fmaf(qreg[d], S.ks[h][j][d], acc);
    s[jj] = acc * scale;
    mx = fmaxf(mx, s[jj]);
  }
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 16));
  float sum = 0.f;
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) { s[jj] = expf(s[jj] - mx); sum += s[jj]; }
  sum += __shfl_xor_sync(0xffffffffu, sum, 16);
  const float inv = 1.f / sum;
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) S.ps[h][i][jh * 8 + jj] = s[jj] * inv;
  __syncwarp();
  for (int r = 0; r < NQ; ++r) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < NQ; ++j) acc = fmaf(S.ps[h][r][j], S.vs[h][j][lane], acc);
    out[(m0 + r) * E_ + h * DH + lane] = acc;
  }
}
// self attention core: grid = objects (M/16), block 256 = 8 warps = 8 heads
__global__ void __launch_bounds__(256) qt_self_attention_kernel(const float* __restrict__ qk, const float* __restrict__ v,
                                                                float* __restrict__ out) {
  __shared__ SelfAttnSmem S;
  qt_self_attention_tile<false>(qk, v, out, (long long)blockIdx.x, S);
}

// ------------------------------------------------------------------------------------------------
// mask_pred + sigmoid + aggregate + foreground test.  grid (ceil(HW/32), B), block 256:
// lane == pixel, warp == group of 32 channels.
//
// Every kernel of this family forms its values through the device functions below, in the same order, so the logits and
// a pixel's foreground decision are the same bits whichever kernel ran: the fused forms (cutie_qt_aux_mask) or the split
// pair (cutie_qt_mask_logits, then cutie_qt_aux_fg over all objects' logits -- object sharding, where each rank computes
// the logits of its own objects and the foreground test needs everyone's).
constexpr int AUX_MAX_K = 32;
typedef float AuxPart[8][33];

// part[k][warp][lane] = the warp's 32-channel share of mask_pred's dot product for objects k0 .. k0 + nk - 1
__device__ __forceinline__ void aux_partials(const float* __restrict__ pixel, const float* wsm, long long b, long long K,
                                             long long k0, int nk, long long HW, long long px, int warp, int lane,
                                             AuxPart* part) {
  for (int k = 0; k < nk; ++k) {
    const float* base = pixel + ((b * K + k0 + k) * E_ + warp * 32) * HW;
    float acc = 0.f;
    if (px < HW) {
#pragma unroll 8
      for (int c = 0; c < 32; ++c) acc = fmaf(wsm[warp * 32 + c], fmaxf(base[(long long)c * HW + px], 0.f), acc);
    }
    part[k][warp][lane] = acc;
  }
}

__device__ __forceinline__ float aux_logit(const AuxPart* part, int k, int lane, float bias) {
  float v = bias;
#pragma unroll
  for (int g = 0; g < 8; ++g) v += part[k][g][lane];
  return v;
}

// the background probability prod(1 - p) folds in one object's logit
__device__ __forceinline__ float aux_fold_bg(float bgp, float v) {
  const float pr = 1.f / (1.f + expf(-v));
  return bgp * (1.f - pr);
}

// log-odds after clamping to [1e-7, 1-1e-7] (tensor_utils.py:50-52): of an object's logit, and of the background
__device__ __forceinline__ float aux_log_odds(float v) {
  const float pr = fminf(fmaxf(1.f / (1.f + expf(-v)), 1e-7f), 1.f - 1e-7f);
  return logf(pr / (1.f - pr));
}
__device__ __forceinline__ float aux_bg_log_odds(float bgp) {
  const float bc = fminf(fmaxf(bgp, 1e-7f), 1.f - 1e-7f);
  return logf(bc / (1.f - bc));
}

// one object's foreground flag of this warp's 32 pixels, and its count
__device__ __forceinline__ void aux_emit(bool live, bool f, uint8_t* fg, int* fg_count, int lane) {
  if (live) *fg = f ? 1 : 0;
  const unsigned m = __ballot_sync(0xffffffffu, f);
  if (lane == 0 && m) atomicAdd(fg_count, __popc(m));
}

__global__ void __launch_bounds__(256) qt_aux_mask_kernel(const float* __restrict__ pixel, const float* __restrict__ w,
                                                          const float* __restrict__ bias, long long K, long long HW,
                                                          float* __restrict__ logits, uint8_t* __restrict__ fg,
                                                          int* __restrict__ fg_count) {
  __shared__ AuxPart part[AUX_MAX_K];
  __shared__ float wsm[E_];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long b = blockIdx.y, px = (long long)blockIdx.x * 32 + lane;
  const bool live = px < HW;
  wsm[tid] = w[tid];
  __syncthreads();
  aux_partials(pixel, wsm, b, K, 0, (int)K, HW, px, warp, lane, part);
  __syncthreads();
  if (warp == 0) {
    float lg[AUX_MAX_K];
    float bgp = 1.f;
    for (int k = 0; k < K; ++k) {
      lg[k] = aux_logit(part, k, lane, bias[0]);
      bgp = aux_fold_bg(bgp, lg[k]);
    }
    float mx = aux_bg_log_odds(bgp);
    float lo[AUX_MAX_K];
    for (int k = 0; k < K; ++k) {
      lo[k] = aux_log_odds(lg[k]);
      mx = fmaxf(mx, lo[k]);
    }
    for (int k = 0; k < K; ++k) {
      if (live) logits[(b * K + k) * HW + px] = lg[k];
      aux_emit(live, live && lo[k] >= mx, fg + (b * K + k) * HW + px, &fg_count[b * K + k], lane);
    }
  }
}

// The same computation for K > AUX_MAX_K, where a pixel's K logits no longer fit in registers.  The objects go through
// the 8 warps in groups of AUX_MAX_K; warp 0 writes each group's logits to `logits` and folds them into prod(1 - p).
// Two more passes over k re-read the pixel's own logits: the log-odds maximum, then the foreground test.
__global__ void __launch_bounds__(256) qt_aux_mask_stream_kernel(const float* __restrict__ pixel,
                                                                 const float* __restrict__ w,
                                                                 const float* __restrict__ bias, long long K,
                                                                 long long HW, float* __restrict__ logits,
                                                                 uint8_t* __restrict__ fg, int* __restrict__ fg_count) {
  __shared__ AuxPart part[AUX_MAX_K];
  __shared__ float wsm[E_];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long b = blockIdx.y, px = (long long)blockIdx.x * 32 + lane;
  const bool live = px < HW;
  wsm[tid] = w[tid];
  __syncthreads();
  float bgp = 1.f;
  for (long long k0 = 0; k0 < K; k0 += AUX_MAX_K) {
    const int nk = (int)(K - k0 < AUX_MAX_K ? K - k0 : AUX_MAX_K);
    aux_partials(pixel, wsm, b, K, k0, nk, HW, px, warp, lane, part);
    __syncthreads();
    if (warp == 0) {
      for (int k = 0; k < nk; ++k) {
        const float v = aux_logit(part, k, lane, bias[0]);
        if (live) logits[(b * K + k0 + k) * HW + px] = v;
        bgp = aux_fold_bg(bgp, v);
      }
    }
    __syncthreads();   // part is refilled by the next group
  }
  if (warp != 0) return;
  float mx = aux_bg_log_odds(bgp);
  for (long long k = 0; k < K; ++k)
    if (live) mx = fmaxf(mx, aux_log_odds(logits[(b * K + k) * HW + px]));
  for (long long k = 0; k < K; ++k)
    aux_emit(live, live && aux_log_odds(logits[(b * K + k) * HW + px]) >= mx, fg + (b * K + k) * HW + px,
             &fg_count[b * K + k], lane);
}

// First half of the split form: the logits alone, [B, K, HW] for the K objects of `pixel`.
__global__ void __launch_bounds__(256) qt_mask_logits_kernel(const float* __restrict__ pixel, const float* __restrict__ w,
                                                             const float* __restrict__ bias, long long K, long long HW,
                                                             float* __restrict__ logits) {
  __shared__ AuxPart part[AUX_MAX_K];
  __shared__ float wsm[E_];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long b = blockIdx.y, px = (long long)blockIdx.x * 32 + lane;
  wsm[tid] = w[tid];
  __syncthreads();
  for (long long k0 = 0; k0 < K; k0 += AUX_MAX_K) {
    const int nk = (int)(K - k0 < AUX_MAX_K ? K - k0 : AUX_MAX_K);
    aux_partials(pixel, wsm, b, K, k0, nk, HW, px, warp, lane, part);
    __syncthreads();
    if (warp == 0 && px < HW)
      for (int k = 0; k < nk; ++k) logits[(b * K + k0 + k) * HW + px] = aux_logit(part, k, lane, bias[0]);
    __syncthreads();
  }
}

// Second half: the foreground test of the objects at positions pos[0 .. n) of all K objects' logits [B, K, HW].
// grid (ceil(HW/256), B), block 256, thread == pixel.  Up to AUX_MAX_K objects a pixel's logits and log-odds stay in
// registers (REG); above, the pixel's logits are re-read for each pass, as in qt_aux_mask_stream_kernel.
template <bool REG>
__global__ void __launch_bounds__(256) qt_aux_fg_kernel(const float* __restrict__ logits, const int* __restrict__ pos,
                                                        long long K, long long n, long long HW, uint8_t* __restrict__ fg,
                                                        int* __restrict__ fg_count) {
  const int lane = threadIdx.x & 31;
  const long long b = blockIdx.y, px = (long long)blockIdx.x * 256 + threadIdx.x;
  const bool live = px < HW;
  const float* lp = logits + b * K * HW + (live ? px : 0);
  float lo[REG ? AUX_MAX_K : 1];
  float bgp = 1.f;
  for (long long k = 0; k < K; ++k) bgp = aux_fold_bg(bgp, lp[k * HW]);
  float mx = aux_bg_log_odds(bgp);
  for (long long k = 0; k < K; ++k) {
    const float l = aux_log_odds(lp[k * HW]);
    if (REG) lo[k] = l;
    mx = fmaxf(mx, l);
  }
  for (long long j = 0; j < n; ++j) {
    const int k = pos[j];
    const float l = REG ? lo[k] : aux_log_odds(lp[(long long)k * HW]);
    aux_emit(live, live && l >= mx, fg + (b * n + j) * HW + px, &fg_count[b * n + j], lane);
  }
}

// ------------------------------------------------------------------------------------------------
// The query-side chain of a transformer block as ONE launch.  Between the two tensor-core cross attentions a block runs
// ~12 skinny ops on the [objects x 16, 256] query tile (combine, out-proj, LayerNorm + q/k/v projections, 16 x 16 self
// attention, FFN, head folds): as separate launches each is ~7 us of mostly launch + first-touch latency (29 + 9 + 3 + 3
// launches, ~330 us per frame at cfg 2).  Here a persistent grid walks an op list; ops of one PHASE are independent and
// their tiles are dealt round-robin to the CTAs, phases are separated by a grid barrier (one atomic + an acquire spin per
// CTA).  The op bodies are the stand-alone kernels' bodies (qt_linear_tile, ...): results are bit-identical to the separate
// launches.  Weights of later ops are prefetched into L2 while the first phase runs.
//
// Grid barrier: counter sync[0] counts arrivals of the whole launch (target = gridDim.x x barrier number); the last CTA to
// leave the kernel (sync[1]) zeroes both, so a launch always starts from zero -- also under CUDA-graph replay, where
// kernel arguments are frozen.  All CTAs are co-resident: the grid never exceeds the SM count and a CTA needs 47 KB of
// shared memory and 256 threads.  A spin gives up after ~1 s (a poisoned counter must not hang the GPU; sync[2] records it).
constexpr int CHAIN_MAX_TILES = 1024;      // pixel tiles of the combine op (64 pixels each)
struct ChainParams {
  cutie_qt_op op[CUTIE_QT_CHAIN_MAX_OPS];
  int nops;
  unsigned* sync;
  const void* pf_ptr[CUTIE_QT_CHAIN_MAX_PREFETCH];
  long long pf_bytes[CUTIE_QT_CHAIN_MAX_PREFETCH];
  int npf;
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void chain_grid_barrier(unsigned* sync, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(&sync[0], 1u);
    const long long t0 = clock64();
    while (ld_acquire_u32(&sync[0]) < target) {
      if (clock64() - t0 > (1ll << 31)) { atomicExch(&sync[2], 1u); break; }
    }
    __threadfence();
  }
  __syncthreads();
}

__device__ __forceinline__ long long chain_tiles(const cutie_qt_op& o) {
  switch (o.kind) {
    case CUTIE_QT_OP_LINEAR: return ((o.i[3] + LIN_BN - 1) / LIN_BN) * ((o.i[0] + LIN_BM - 1) / LIN_BM);
    case CUTIE_QT_OP_HEAD_FOLD: return o.i[0] * H_;
    case CUTIE_QT_OP_SELF_ATTENTION: return o.i[0] / NQ;
    default: return (long long)NQ * H_ * o.i[2];
  }
}

__global__ void __launch_bounds__(256) qt_chain_kernel(const __grid_constant__ ChainParams P) {
  __shared__ __align__(16) unsigned char raw[sizeof(SelfAttnSmem)];
  __shared__ float coef[CHAIN_MAX_TILES];
  __shared__ float zn[E_];
  static_assert(sizeof(SelfAttnSmem) >= 2 * LIN_BM * LIN_LD * sizeof(float), "the union is sized by the attention tile");
  float (*xs)[LIN_LD] = reinterpret_cast<float (*)[LIN_LD]>(raw);
  float (*wsm)[LIN_LD] = reinterpret_cast<float (*)[LIN_LD]>(raw + LIN_BM * LIN_LD * sizeof(float));
  // L2 prefetch of the weights the later phases will stream (128-byte lines dealt over the whole grid)
  for (int f = 0; f < P.npf; ++f) {
    const char* base = reinterpret_cast<const char*>(P.pf_ptr[f]);
    const long long lines = (P.pf_bytes[f] + 127) / 128;
    for (long long l = (long long)blockIdx.x * 256 + threadIdx.x; l < lines; l += (long long)gridDim.x * 256)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(base + l * 128));
  }
  unsigned barriers = 0;
  int phase = P.op[0].phase;
  for (int oi = 0; oi < P.nops; ++oi) {
    const cutie_qt_op& o = P.op[oi];
    if (o.phase != phase) {
      phase = o.phase;
      chain_grid_barrier(P.sync, gridDim.x * (++barriers));
    }
    const long long nt = chain_tiles(o);
    for (long long t = blockIdx.x; t < nt; t += gridDim.x) {
      if (o.kind == CUTIE_QT_OP_LINEAR) {
        LinearParams lp;
        lp.x = o.in[0]; lp.M = o.i[0]; lp.Kd = o.i[1]; lp.ldx = o.i[1] + ((o.i[4] & 1) ? 1 : 0);
        lp.W = o.in[1]; lp.ldw = o.i[2]; lp.N = o.i[3]; lp.bias = o.in[2]; lp.ln_w = o.in[3]; lp.ln_b = o.in[4];
        lp.pe = o.in[5]; lp.summary_norm = (int)(o.i[4] & 1); lp.relu = (int)((o.i[4] >> 1) & 1);
        lp.residual = o.in[6]; lp.residual_mod = o.i[5]; lp.xhat_out = o.out[1]; lp.y = o.out[0];
        const long long nbx = (o.i[3] + LIN_BN - 1) / LIN_BN;
        qt_linear_tile<true>(lp, (int)(t % nbx), (int)(t / nbx), xs, wsm);
      } else if (o.kind == CUTIE_QT_OP_HEAD_FOLD) {
        qt_head_fold_tile<true>(o.in[0], o.in[1], o.i[1], (int)o.i[2], o.f, o.in[2], o.out[0], o.out[1], t / H_, (int)(t % H_),
                                reinterpret_cast<float*>(raw));
      } else if (o.kind == CUTIE_QT_OP_SELF_ATTENTION) {
        qt_self_attention_tile<true>(o.in[0], o.in[1], o.out[0], t, *reinterpret_cast<SelfAttnSmem*>(raw));
      } else {
        const int i = (int)(t % NQ), h = (int)((t / NQ) % H_);
        qt_p2q_combine_tile<E_, H_, NQ>(o.in[0], (int)o.i[0], o.in[1], o.i[1], o.in[2], o.out[0], i, h, t / (NQ * H_), coef, zn);
      }
      __syncthreads();          // the tile's shared memory is reused by the next tile / op
    }
  }
  // leave the counters at zero for the next launch: the last CTA out resets them (every CTA has passed every barrier by then)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&P.sync[1], 1u) == gridDim.x - 1) {
      P.sync[0] = 0u;
      P.sync[1] = 0u;
      __threadfence();
    }
  }
}

}  // namespace cutie

using namespace cutie;

extern "C" int cutie_qt_linear(const float* x, int64_t M, int64_t Kd, const float* W, int64_t ldw, int64_t N,
                               const float* bias, const float* ln_w, const float* ln_b, const float* pe,
                               int summary_norm, int relu, const float* residual, int64_t residual_mod,
                               float* xhat_out, float* y, void* stream) {
  CUTIE_REQUIRE(x && W && y && M >= 1 && N >= 1 && Kd >= 1, "null/empty argument");
  CUTIE_REQUIRE((ln_w == nullptr) == (ln_b == nullptr), "ln_w and ln_b must be given together");
  CUTIE_REQUIRE(xhat_out == nullptr || ln_w != nullptr, "xhat_out needs LayerNorm");
  LinearParams p;
  p.x = x; p.M = M; p.Kd = Kd; p.ldx = Kd + (summary_norm ? 1 : 0);
  p.W = W; p.ldw = ldw; p.N = N; p.bias = bias; p.ln_w = ln_w; p.ln_b = ln_b; p.pe = pe;
  p.summary_norm = summary_norm; p.relu = relu; p.residual = residual; p.residual_mod = residual_mod;
  p.xhat_out = xhat_out; p.y = y;
  cudaStream_t st = (cudaStream_t)stream;
  CUTIE_REQUIRE(ln_w == nullptr || Kd == LIN_KC, "fused LayerNorm needs Kd == 256");
  qt_linear_kernel<<<dim3((unsigned)((N + LIN_BN - 1) / LIN_BN), (unsigned)((M + LIN_BM - 1) / LIN_BM)), 256, 0, st>>>(p);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_qt_head_fold(const float* a, int64_t M, int64_t E, int num_heads, const float* W, int64_t ldw,
                                  int transpose_w, float scale, const float* bias_vec, float* out, float* dots,
                                  void* stream) {
  CUTIE_REQUIRE(a && W && out && M >= 1, "null/empty argument");
  CUTIE_REQUIRE(E == E_ && num_heads == H_, "embed_dim must be 256 with 8 heads");
  CUTIE_REQUIRE((dots == nullptr) == (bias_vec == nullptr), "dots and bias_vec must be given together");
  qt_head_fold_kernel<<<dim3((unsigned)M, H_), 256, 0, (cudaStream_t)stream>>>(a, W, ldw, transpose_w, scale, bias_vec, out,
                                                                             dots);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_qt_self_attention(const float* qk, const float* v, int64_t M, int64_t E, int num_queries,
                                       int num_heads, float* out, void* stream) {
  CUTIE_REQUIRE(qk && v && out && M >= 1, "null/empty argument");
  CUTIE_REQUIRE(E == E_ && num_heads == H_ && num_queries == NQ && M % NQ == 0,
                "embed_dim 256, 8 heads, 16 queries");
  qt_self_attention_kernel<<<(unsigned)(M / NQ), 256, 0, (cudaStream_t)stream>>>(qk, v, out);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_qt_aux_mask(const float* pixel, const float* w, const float* b, int64_t B, int64_t K, int64_t E,
                                 int64_t HW, float* logits, uint8_t* fg, int32_t* fg_count, void* stream) {
  CUTIE_REQUIRE(pixel && w && b && logits && fg && fg_count, "null argument");
  CUTIE_REQUIRE(E == E_, "embed_dim must be 256");
  CUTIE_REQUIRE(K >= 1 && B >= 1 && HW >= 1, "empty argument");
  dim3 grid((unsigned)((HW + 31) / 32), (unsigned)B);
  if (K <= AUX_MAX_K)
    qt_aux_mask_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(pixel, w, b, K, HW, logits, fg, fg_count);
  else
    qt_aux_mask_stream_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(pixel, w, b, K, HW, logits, fg, fg_count);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_qt_mask_logits(const float* pixel, const float* w, const float* b, int64_t B, int64_t K, int64_t E,
                                    int64_t HW, float* logits, void* stream) {
  CUTIE_REQUIRE(pixel && w && b && logits, "null argument");
  CUTIE_REQUIRE(E == E_, "embed_dim must be 256");
  CUTIE_REQUIRE(K >= 1 && B >= 1 && HW >= 1, "empty argument");
  qt_mask_logits_kernel<<<dim3((unsigned)((HW + 31) / 32), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(pixel, w, b, K,
                                                                                                        HW, logits);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_qt_aux_fg(const float* logits, const int32_t* positions, int64_t B, int64_t K, int64_t n,
                               int64_t HW, uint8_t* fg, int32_t* fg_count, void* stream) {
  CUTIE_REQUIRE(logits && positions && fg && fg_count, "null argument");
  CUTIE_REQUIRE(K >= 1 && B >= 1 && HW >= 1 && n >= 1, "empty argument");
  CUTIE_REQUIRE(n <= K, "more positions than objects");
  dim3 grid((unsigned)((HW + 255) / 256), (unsigned)B);
  if (K <= AUX_MAX_K)
    qt_aux_fg_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(logits, positions, K, n, HW, fg, fg_count);
  else
    qt_aux_fg_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(logits, positions, K, n, HW, fg, fg_count);
  CUTIE_CHECK_LAUNCH();
  return 0;
}

extern "C" int cutie_qt_chain(const cutie_qt_op* ops, int nops, const void* const* prefetch_ptr,
                              const int64_t* prefetch_bytes, int nprefetch, uint32_t* sync_ws, void* stream) {
  CUTIE_REQUIRE(ops && nops >= 1 && nops <= CUTIE_QT_CHAIN_MAX_OPS, "1..16 ops");
  CUTIE_REQUIRE(nprefetch >= 0 && nprefetch <= CUTIE_QT_CHAIN_MAX_PREFETCH && (nprefetch == 0 || (prefetch_ptr && prefetch_bytes)),
                "0..16 prefetch ranges");
  CUTIE_REQUIRE(sync_ws != nullptr, "sync_ws: 4 zero-initialised uint32");
  ChainParams cp;
  memset(&cp, 0, sizeof(cp));
  long long max_tiles = 1;
  for (int i = 0; i < nops; ++i) {
    const cutie_qt_op& o = ops[i];
    CUTIE_REQUIRE(i == 0 || o.phase >= ops[i - 1].phase, "phases must not decrease");
    switch (o.kind) {
      case CUTIE_QT_OP_LINEAR:
        CUTIE_REQUIRE(o.in[0] && o.in[1] && o.out[0] && o.i[0] >= 1 && o.i[1] >= 1 && o.i[3] >= 1, "linear: null/empty argument");
        CUTIE_REQUIRE((o.in[3] == nullptr) == (o.in[4] == nullptr), "linear: ln_w and ln_b must be given together");
        CUTIE_REQUIRE(o.out[1] == nullptr || o.in[3] != nullptr, "linear: xhat_out needs LayerNorm");
        CUTIE_REQUIRE(o.in[3] == nullptr || o.i[1] == LIN_KC, "linear: fused LayerNorm needs Kd == 256");
        max_tiles = std::max(max_tiles, (long long)(((o.i[3] + LIN_BN - 1) / LIN_BN) * ((o.i[0] + LIN_BM - 1) / LIN_BM)));
        break;
      case CUTIE_QT_OP_HEAD_FOLD:
        CUTIE_REQUIRE(o.in[0] && o.in[1] && o.out[0] && o.i[0] >= 1, "head_fold: null/empty argument");
        CUTIE_REQUIRE((o.out[1] == nullptr) == (o.in[2] == nullptr), "head_fold: dots and bias_vec must be given together");
        max_tiles = std::max(max_tiles, (long long)o.i[0] * H_);
        break;
      case CUTIE_QT_OP_SELF_ATTENTION:
        CUTIE_REQUIRE(o.in[0] && o.in[1] && o.out[0] && o.i[0] >= NQ && o.i[0] % NQ == 0, "self_attention: M must be a multiple of 16");
        max_tiles = std::max(max_tiles, (long long)(o.i[0] / NQ));
        break;
      case CUTIE_QT_OP_P2Q_COMBINE:
        CUTIE_REQUIRE(o.in[0] && o.in[1] && o.in[2] && o.out[0] && o.i[2] >= 1, "p2q_combine: null/empty argument");
        CUTIE_REQUIRE(o.i[0] >= 1 && o.i[0] <= CHAIN_MAX_TILES, "p2q_combine: 1..1024 pixel tiles");
        max_tiles = std::max(max_tiles, (long long)NQ * H_ * o.i[2]);
        break;
      default:
        CUTIE_REQUIRE(false, "unknown op kind");
    }
    cp.op[i] = o;
  }
  cp.nops = nops;
  cp.sync = sync_ws;
  cp.npf = nprefetch;
  for (int i = 0; i < nprefetch; ++i) {
    cp.pf_ptr[i] = prefetch_ptr[i];
    cp.pf_bytes[i] = prefetch_bytes[i];
  }
  const long long sms = num_sms();
  const unsigned grid = (unsigned)std::min(sms, max_tiles);     // <= SM count: every CTA is resident (grid barrier)
  qt_chain_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(cp);
  CUTIE_CHECK_LAUNCH();
  return 0;
}
