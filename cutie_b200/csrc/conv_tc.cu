// 3x3 (zero-pad 1) and 1x1 convolutions, stride 1 or 2, as wgmma implicit GEMMs with fp32-class accuracy
// (3xTF32), sm_90a.
//
// SURVEY.md section 8(f): the PixelFFN / CAResBlock (transformer_layers.py:121-136, channel_attn.py:7-39), PixelFeatureFuser
// (big_modules.py:192-235), key projection (big_modules.py:66-87), MaskDecoder / SensoryUpdater (big_modules.py:238-306,
// modules.py:46-85) and ResNet trunk (utils/resnet.py) convolutions.  With the numerics the parity tests validate -- fp32,
// cuDNN TF32 off -- cuDNN runs them on the FP32 pipe; here they run on the tensor cores at fp32-class accuracy.
//
//   Y[n, co, y, x] = act( bias[co] + sum_{ci, dy, dx} W[co, ci, dy, dx] * pre(X)[n, ci, s y + dy - h, s x + dx - h]  (+ Z[n, co, y, x]) )
//
// GEMM view per CTA: D[co (M = 128), position (N <= 128)] += A_tap[co, ci] . B_tap[ci, position], K = 32 input channels
// per (chunk, tap) step, KS^2 taps x Cin / 32 chunks.
//
//   * A (weights) comes from a precomputed OPERAND IMAGE (cutie_conv_weight_image, built once per layer): for every
//     (128-channel output tile, 32-channel input chunk, tap) the [128 x 32] tf32 hi and lo planes in K-major
//     SWIZZLE_128B order, 32 KB, fetched through a 3-stage mbarrier ring.  Each MMA warpgroup reads only its own 64 rows
//     of a stage, so each refills its own half (a ring per warpgroup): one elected thread bulk-copies its hi and lo rows.
//   * B (activations), 3x3: the CTA's spatial tile is TH x TW output pixels; its input window with the 1-pixel halo is laid
//     out in shared memory ONCE per 32-channel chunk as rows of a local zero-padded grid -- row r = ly * (TW + 2) + lx + 1
//     holds the 32 channels of input pixel (ty0 + ly - 1, tx0 + lx - 1) as 128 bytes, K-major SWIZZLE_128B, hi and lo
//     planes.  Output position j = ty * (TW + 2) + lx reads, for tap (dy, dx), row j + dy * (TW + 2) + dx: EVERY TAP IS
//     THE SAME TILE READ THROUGH A DESCRIPTOR WHOSE START ADDRESS IS SHIFTED BY WHOLE ROWS -- no im2col copies, no
//     per-tap producer work.  (The hardware applies the 128-byte swizzle to absolute shared-memory address bits, so a
//     start shifted by r rows reads rows r.. of a tile that was written with the address-based pattern, with the
//     descriptor's base-offset field left 0.)  The two padding columns of every local row are computed and
//     discarded (TW / (TW + 2) efficiency); image borders are zero rows.
//     3x3 stride 2: the same trick over four PARITY PLANES of the input window (P[a][b](u, v) = in(2u + a, 2v + b)) stored
//     one after the other: tap (dy, dx) reads plane (dy != 1, dx != 1) at (u, v) = (oy - [dy == 0], ox - [dx == 0]) -- again
//     a constant row shift per tap.  The tile holds 4x the input per output, so N is ~32-48 positions per CTA.
//     1x1: a tile is 128 consecutive output pixels of the flattened image (stride 2: of the sub-sampled one), no halo; four
//     activation stages of 32 KB instead of two of 62 KB, each producer thread keeping two chunks of loads in flight.
//   * Layout-agnostic: X, Y and Z are addressed through (image, channel, pixel) strides -- dense NCHW (what the transformer
//     kernels emit) and channels-last (what the cuDNN trunks run in) both work without a re-layout; channels-last is the
//     natural one (a producer thread reads its 32 channels as 8 x 16 bytes, an epilogue warp stores 32 consecutive channels).
//   * 3xTF32: x = hi + lo with hi = tf32(x) RN, lo = tf32(x - hi); three MMAs per k-step (lo.hi + hi.lo + hi.hi), fp32
//     accumulation in registers (wgmma.m64n128k8 per warpgroup): relative error ~2^-21 per product.  The tensor core adds
//     each MMA's result to its accumulator with TRUNCATION, a bias that grows with the number of accumulations (one
//     accumulator over the whole K loop measured ~9x cuDNN's fp32 error at Cin = 256), so the MMAs of one (chunk, tap)
//     step go into a fresh accumulator that is then added to an fp32 total with round-to-nearest adds.
//   * Epilogue: straight from the accumulator fragments (element-wise); bias, optional residual, optional ReLU; ReLU on
//     the INPUT (the pre-activation blocks' conv(relu(x))) is applied by the producers for free.
//   * FP16 operands (template parameter F16; cutie_conv_tc_f16, what CUDA autocast asks of a convolution): the same kernel,
//     plan, tiles, epilogues and fp32 inputs / outputs, but the producers round pre(x) to fp16 (RN, one plane, no split),
//     the weight image holds one fp16 [128 x 32] plane per (chunk, tap) (8 KB), and a (chunk, tap) step is TWO
//     wgmma.m64n128k16.f32.f16.f16 per warpgroup instead of twelve tf32 ones.  A row of 32 channels is then 64 bytes, so
//     both operands use K-major SWIZZLE_64B (8-row atoms of 512 B, 16-byte chunk index XOR address bits 7-8).  The row-shift
//     argument above holds unchanged: the 64-byte swizzle is likewise applied to absolute address bits, every operand tile
//     base (activation stages, weight stages, the second warpgroup's half) is 512-byte aligned, so the producers' pattern
//     ((chunk ^ (row >> 1)) & 3 with row counted from the base) is the address-based one and a start shifted by r rows of
//     64 bytes reads rows r.. of it.  The fresh-accumulator-per-step promotion is kept (DESIGN.md section 3.7).
//
// Warp roles (384 threads = three warpgroups): warps 0-7 two MMA + epilogue warpgroups (output channels 0-63 / 64-127 of
// the tile; thread 0 of each also refills its weight ring), warps 8-11 activation producers (global fp32 -> hi/lo ->
// swizzled smem, next chunk's loads in flight during the current chunk's MMAs).  Three warpgroups put three warps on each
// SM sub-partition, so the per-thread register budget (168) holds both accumulators without spilling; a 17-warp block
// (5 warps on one sub-partition) capped it at 96 and spilled the promotion's total to local memory on every step.
#include "common.cuh"
#include "tc_ptx.cuh"

namespace cutie {

namespace {

constexpr int CV_M = 128;                         // output channels per CTA
constexpr int CV_KC = 32;                         // input channels per chunk
constexpr int CV_A_STAGES = 3;
constexpr int CV_THREADS = 384;
constexpr int CV_WARPS = CV_THREADS / 32;
constexpr int CV_PROD = 128;
constexpr int CV3_ROWS = 248;                     // 3x3: activation tile rows per stage (31 x 8: planes stay 1024-byte aligned)
constexpr int CV1_ROWS = 128;                     // 1x1
constexpr int CV_STAGING = 65 * 1024;             // the finished tile staged as fp32 [128][N | 1 <= 129] (66048 B), 1 KB aligned

// operand precision: 3xTF32 = hi | lo planes of 128-byte rows (32 tf32); FP16 = one plane of 64-byte rows (32 f16)
__host__ __device__ constexpr int cv_row_bytes(bool f16) { return f16 ? 64 : 128; }
__host__ __device__ constexpr int cv_planes(bool f16) { return f16 ? 1 : 2; }
__host__ __device__ constexpr int cv_a_bytes(bool f16) { return cv_planes(f16) * CV_M * cv_row_bytes(f16); }   // 32768 | 8192
// activation stages (3x3: 2 x 248 rows, 1x1: 4 x 128 rows); the epilogue's staging buffer aliases them, so at least that
__host__ __device__ constexpr int cv_x_bytes(int ks, bool f16) {
  const int operands = (ks == 3 ? 2 * CV3_ROWS : 4 * CV1_ROWS) * cv_planes(f16) * cv_row_bytes(f16);
  return operands > CV_STAGING ? operands : CV_STAGING;
}

struct ConvTail {
  unsigned long long a_full[2][CV_A_STAGES], a_empty[2][CV_A_STAGES], x_full[4], x_empty[4];   // a_*: per MMA warpgroup
  int last[2];
};
// 3xTF32: 126976 (3x3) | 131072 (1x1) activation bytes + 3 x 32 KB weight stages; FP16: 66560 + 3 x 8 KB
constexpr int cv_smem(int ks, bool f16) { return cv_x_bytes(ks, f16) + CV_A_STAGES * cv_a_bytes(f16) + (int)sizeof(ConvTail) + 64; }

struct ConvTcParams {
  const float* x;
  const unsigned char* wimg;   // [ceil(Cout / 128)][Cin / 32][taps][32768 (3xTF32) | 8192 (FP16)]
  const float* bias;           // [Cout] or null
  const float* z;              // residual, or null
  float* y;
  long long xs_n, xs_c, xs_p;  // element strides of X: image, channel, pixel (pixel index = row * Wi + column)
  long long ys_n, ys_c, ys_p;  // of Y
  long long zs_n, zs_c, zs_p;  // of Z
  int Cin, Cout, H, W;         // OUTPUT height / width
  int Hi, Wi, stride;          // input height / width; stride (1x1 only: 1 or 2)
  int TH, TW, tiles_x;         // 3x3: spatial tile and tiles per image row
  int pitch, xoff;             // 3x3: positions per local row (TW + 2 | TW + 1 at stride 2); column of output x = 0 (1 | 0)
  int plane_rows;              // 3x3 stride 2: rows of one parity plane of the activation tile
  int shift[9];                // 3x3: activation-tile row each tap's operand window starts at
  int N;                       // MMA N (multiple of 16, <= 128)
  int relu_in, relu_out, x_vec;
  int cl_vec;                  // channels-last Y (and Z) addressable as float4 along channels
  int q;                       // (tile, chunk) units per CTA (<= chunks per tile): CTA i owns units [i q, (i + 1) q)
  int T, tiles, cots;          // output tiles in all = NB * cots * tiles; spatial tiles per image; 128-channel tiles
  int maxslots;                // most shares a tile can have
  float* ws;                   // [T][maxslots][N][128] partial sums (position-major: coalesced both ways)
  int* counters;               // [T], zero on entry and on exit
};

struct ConvPart {              // one contiguous share of an output tile's input chunks
  int tile, cot, nb;           // spatial tile, 128-channel tile, image
  int ty0, tx0;                // 3x3: first output row / column of the tile
  long long pix0;              // 1x1: first flattened output pixel
  int c0, c1;                  // chunk range
  int slot, nslots;            // this share's index among the tile's contributors; their number
  long long tile_lin;          // (nb, cot, tile) linearised: workspace / counter index
};

template <int KS, bool F16>
__global__ void __launch_bounds__(CV_THREADS, 1) conv_tc_kernel(const ConvTcParams p) {
  constexpr int XROWS = KS == 3 ? CV3_ROWS : CV1_ROWS;
  constexpr int ROWB = cv_row_bytes(F16);                    // bytes per operand row (32 channels)
  constexpr int XPLANE = XROWS * ROWB;
  constexpr int XSTAGE = cv_planes(F16) * XPLANE;
  constexpr int XST = KS == 3 ? 2 : 4;                       // activation stages
  constexpr int A_BYTES = cv_a_bytes(F16);
  constexpr int TAPS = KS * KS;
  constexpr int RPT = KS == 3 ? 2 : 1;                       // tile rows per producer thread (3x3: r and r + 128)
  constexpr int DEPTH = KS == 3 ? 1 : 2;                     // chunks of global loads in flight per producer thread
  constexpr int A_HALF = 64 * ROWB;                          // one warpgroup's rows of one weight plane
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* Xs = smem;
  unsigned char* As = smem + cv_x_bytes(KS, F16);
  ConvTail& T = *reinterpret_cast<ConvTail*>(As + CV_A_STAGES * A_BYTES);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int TWp = p.pitch;                                   // positions per local row of the 3x3 tile
  const int C = p.Cin / CV_KC;                               // input chunks per output tile
  const long long HW = (long long)p.H * p.W;
  // ---- this CTA's share of the (output tile, input chunk) space: units [u0, u1), at most two tiles (host: q <= C) ----
  const long long U = (long long)p.T * C;
  const long long u0 = (long long)blockIdx.x * p.q, u1 = u0 + p.q < U ? u0 + p.q : U;
  auto make_part = [&](long long ua, long long ub) {
    ConvPart P;
    P.tile_lin = ua / C;
    P.c0 = (int)(ua - P.tile_lin * C);
    P.c1 = P.c0 + (int)(ub - ua);
    const long long first = (P.tile_lin * C) / p.q, last = (P.tile_lin * C + C - 1) / p.q;
    P.slot = (int)(blockIdx.x - first);
    P.nslots = (int)(last - first + 1);
    P.tile = (int)(P.tile_lin % p.tiles);
    const long long rest = P.tile_lin / p.tiles;
    P.cot = (int)(rest % p.cots);
    P.nb = (int)(rest / p.cots);
    P.ty0 = KS == 3 ? (P.tile / p.tiles_x) * p.TH : 0;
    P.tx0 = KS == 3 ? (P.tile % p.tiles_x) * p.TW : 0;
    P.pix0 = (long long)P.tile * p.N;
    return P;
  };
  const long long split_at = (u0 / C + 1) * C < u1 ? (u0 / C + 1) * C : u1;   // end of the first tile's share
  const int nparts = split_at < u1 ? 2 : 1;
  const ConvPart part0 = make_part(u0, split_at), part1 = make_part(nparts == 2 ? split_at : u0, u1);
  // a whole tile computed by this CTA alone goes straight from the accumulators to the output; shares meet in the workspace
  const bool direct = nparts == 1 && part0.nslots == 1;

  if (tid == 0) {
    for (int G = 0; G < 2; ++G)
      for (int s = 0; s < CV_A_STAGES; ++s) { mbar_init(smem_u32(&T.a_full[G][s]), 1); mbar_init(smem_u32(&T.a_empty[G][s]), 128); }
    for (int s = 0; s < XST; ++s) { mbar_init(smem_u32(&T.x_full[s]), CV_PROD); mbar_init(smem_u32(&T.x_empty[s]), 256); }
    T.last[0] = T.last[1] = 0;
    mbar_init_fence();
  }
  __syncthreads();
  // Dense-NCHW outputs: thread == channel would store 4 bytes per 128-byte line (8x write amplification in L2).  The
  // finished tile is staged in shared memory [channel][position] instead (the operand stages are free by then) and written
  // by the epilogue AND producer warps, a warp per (channel, tile row): 128-byte coalesced stores, residual read likewise.
  // Channels-last outputs are coalesced either way, but four epilogue warps with 32 accesses in flight each cannot keep
  // HBM busy on the wide, shallow layers (a bottleneck's closing 1x1 + residual ran at 0.5 TB/s): the same staging
  // ([position][channel]) lets all twelve warps move 16 bytes per lane, residual included.
  const bool staged_nchw = p.ys_p == 1 && (p.z == nullptr || p.zs_p == 1);
  const bool staged = staged_nchw || p.cl_vec;
  const int LD = p.N | 1;                                     // odd row pitch: conflict-free both ways
  auto store_staged_rows = [&](const ConvPart& P, int sw) {  // sw = warp, 0..CV_WARPS - 1
    const float* stage = reinterpret_cast<const float*>(smem);
    if (!staged_nchw) {                                      // channels-last: a warp per position, 4 channels per lane
      const int co4 = P.cot * CV_M + 4 * lane;
      if (co4 >= p.Cout) return;
      const float4 b4 = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + co4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      for (int j = sw; j < p.N; j += CV_WARPS) {
        long long pix;
        bool ok;
        if (KS == 3) {
          const int ty = j / TWp, lx = j - ty * TWp;
          const int gy = P.ty0 + ty, gx = P.tx0 + lx - p.xoff;
          ok = lx >= p.xoff && lx < p.TW + p.xoff && ty < p.TH && gy < p.H && gx < p.W;
          pix = (long long)gy * p.W + gx;
        } else {
          pix = P.pix0 + j;
          ok = pix < HW;
        }
        if (!ok) continue;
        float4 v = *reinterpret_cast<const float4*>(stage + j * CV_M + 4 * lane);
        v.x += b4.x; v.y += b4.y; v.z += b4.z; v.w += b4.w;
        if (p.z) {
          const float4 z4 = __ldg(reinterpret_cast<const float4*>(p.z + (long long)P.nb * p.zs_n + pix * p.zs_p + co4));
          v.x += z4.x; v.y += z4.y; v.z += z4.z; v.w += z4.w;
        }
        if (p.relu_out) v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
        *reinterpret_cast<float4*>(p.y + (long long)P.nb * p.ys_n + pix * p.ys_p + co4) = v;
      }
      return;
    }
    const int nseg = CV_M * (KS == 3 ? p.TH : 1);
    for (int seg = sw; seg < nseg; seg += CV_WARPS) {
      const int col = KS == 3 ? seg / p.TH : seg, ty = KS == 3 ? seg - col * p.TH : 0;
      const int co = P.cot * CV_M + col;
      if (co >= p.Cout) continue;
      long long pbase;
      int len, sbase;
      if (KS == 3) {
        const int gy = P.ty0 + ty;
        if (gy >= p.H) continue;
        pbase = (long long)gy * p.W + P.tx0;
        len = p.W - P.tx0 < p.TW ? p.W - P.tx0 : p.TW;
        sbase = col * LD + ty * TWp + p.xoff;
      } else {
        pbase = P.pix0;
        len = HW - P.pix0 < p.N ? (int)(HW - P.pix0) : p.N;
        sbase = col * LD;
      }
      const float b = p.bias ? __ldg(p.bias + co) : 0.f;
      float* yrow = p.y + (long long)P.nb * p.ys_n + (long long)co * p.ys_c + pbase;
      const float* zrow = p.z ? p.z + (long long)P.nb * p.zs_n + (long long)co * p.zs_c + pbase : nullptr;
      for (int i = lane; i < len; i += 32) {
        float val = stage[sbase + i] + b;
        if (zrow) val += __ldg(zrow + i);
        if (p.relu_out) val = fmaxf(val, 0.f);
        yrow[i] = val;
      }
    }
  };

  // Shared tiles: the CTA that arrived last adds the tile's shares IN SLOT ORDER -- all twelve warps, 16 bytes per lane
  // (four warps with scalar loads left this on the critical path at ~15 us per tile).  Channels-last outputs are finished
  // right here; dense-NCHW ones go through the staging buffer (transposed) and store_staged_rows.
  auto reduce_shares = [&](const ConvPart& P, int sw, bool to_stage) {
    const int co4 = P.cot * CV_M + 4 * lane;
    const float* wst = p.ws + (P.tile_lin * p.maxslots) * (long long)(p.N * CV_M) + 4 * lane;
    float* stage = reinterpret_cast<float*>(smem);
    const bool co_ok = co4 < p.Cout;
    const float4 b4 = (!to_stage && p.bias && co_ok) ? __ldg(reinterpret_cast<const float4*>(p.bias + co4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = sw; j < p.N; j += CV_WARPS) {
      long long pix = 0;
      bool ok = true;
      if (!to_stage) {
        if (KS == 3) {
          const int ty = j / TWp, lx = j - ty * TWp;
          const int gy = P.ty0 + ty, gx = P.tx0 + lx - p.xoff;
          ok = lx >= p.xoff && lx < p.TW + p.xoff && ty < p.TH && gy < p.H && gx < p.W;
          pix = (long long)gy * p.W + gx;
        } else {
          pix = P.pix0 + j;
          ok = pix < HW;
        }
        if (!ok || !co_ok) continue;
      }
      float4 v = __ldcg(reinterpret_cast<const float4*>(wst + (long long)j * CV_M));
      for (int k = 1; k < P.nslots; ++k) {
        const float4 t = __ldcg(reinterpret_cast<const float4*>(wst + ((long long)k * p.N + j) * CV_M));
        v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
      }
      if (to_stage) {
        stage[(4 * lane + 0) * LD + j] = v.x; stage[(4 * lane + 1) * LD + j] = v.y;
        stage[(4 * lane + 2) * LD + j] = v.z; stage[(4 * lane + 3) * LD + j] = v.w;
      } else {
        v.x += b4.x; v.y += b4.y; v.z += b4.z; v.w += b4.w;
        if (p.z) {
          const float4 z4 = __ldg(reinterpret_cast<const float4*>(p.z + (long long)P.nb * p.zs_n + pix * p.zs_p + co4));
          v.x += z4.x; v.y += z4.y; v.z += z4.z; v.w += z4.w;
        }
        if (p.relu_out) v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
        *reinterpret_cast<float4*>(p.y + (long long)P.nb * p.ys_n + pix * p.ys_p + co4) = v;
      }
    }
  };

  if (warp >= 8) {
    // ===== activation producers: thread == tile rows pt and pt + 128 (3x3) | row pt (1x1), all 32 channels of each =====
    const int pt = tid - 256;
    int xc = 0;                                              // chunks produced so far (stage ring position)
    for (int pi = 0; pi < nparts; ++pi) {
      const ConvPart& P = pi ? part1 : part0;
      const int chunks = P.c1 - P.c0;
      bool valid[RPT];
      const float* xb[RPT];
#pragma unroll
      for (int h = 0; h < RPT; ++h) {
        const int r = pt + CV_PROD * h;
        bool ok = false;
        long long poff = 0;
        if (KS == 3) {
          if (p.stride == 1) {
            const int rows_used = p.N + 2 * TWp + 2;
            if (r >= 1 && r < rows_used) {
              const int q = r - 1, ly = q / TWp, lx = q - ly * TWp;
              const int gy = P.ty0 + ly - 1, gx = P.tx0 + lx - 1;
              ok = ly < p.TH + 2 && gy >= 0 && gy < p.Hi && gx >= 0 && gx < p.Wi;
              poff = (long long)gy * p.Wi + gx;
            }
          } else {
            // stride 2: four parity planes P[a][b](u, v) = in(2u + a, 2v + b), each a local (TH + 1) x (TW + 1) grid whose
            // first row / column is u = ty0 - 1 / v = tx0 - 1; tap (dy, dx) reads plane (dy != 1, dx != 1) shifted by
            // (dy == 0, dx == 0)
            const int pl = r / p.plane_rows, q = r - pl * p.plane_rows;
            const int lu = q / TWp, lv = q - lu * TWp;
            const int gy = 2 * (P.ty0 - 1 + lu) + (pl >> 1), gx = 2 * (P.tx0 - 1 + lv) + (pl & 1);
            ok = pl < 4 && lu <= p.TH && gy >= 0 && gy < p.Hi && gx >= 0 && gx < p.Wi;
            poff = (long long)gy * p.Wi + gx;
          }
        } else {
          const long long op = P.pix0 + r;
          if (r < p.N && op < HW) {
            const int oy = (int)(op / p.W), ox = (int)(op - (long long)oy * p.W);
            ok = true;
            poff = (long long)(oy * p.stride) * p.Wi + ox * p.stride;
          }
        }
        valid[h] = ok;
        xb[h] = p.x + (long long)P.nb * p.xs_n + poff * p.xs_p + (long long)(P.c0 * CV_KC) * p.xs_c;
      }
      float v[DEPTH][RPT][CV_KC];
      auto load = [&](int c, float (&dst)[RPT][CV_KC]) {     // every row's loads of chunk c issued before any is used
#pragma unroll
        for (int h = 0; h < RPT; ++h) {
          if (p.x_vec) {                                       // channels-last: consecutive floats
#pragma unroll
            for (int k4 = 0; k4 < CV_KC / 4; ++k4) {
              const float4 f = valid[h] ? __ldg(reinterpret_cast<const float4*>(xb[h] + c * CV_KC + 4 * k4)) : make_float4(0.f, 0.f, 0.f, 0.f);
              dst[h][4 * k4] = f.x; dst[h][4 * k4 + 1] = f.y; dst[h][4 * k4 + 2] = f.z; dst[h][4 * k4 + 3] = f.w;
            }
          } else {
#pragma unroll
            for (int i = 0; i < CV_KC; ++i) dst[h][i] = valid[h] ? __ldg(xb[h] + (long long)(c * CV_KC + i) * p.xs_c) : 0.f;
          }
        }
      };
#pragma unroll
      for (int d = 0; d < DEPTH; ++d)
        if (d < chunks) load(d, v[d]);
#pragma unroll 1
      for (int cb = 0; cb < chunks; cb += DEPTH) {
#pragma unroll
        for (int d = 0; d < DEPTH; ++d) {
          const int c = cb + d;
          if (c < chunks) {
            const int s = xc % XST;
            mbar_wait(smem_u32(&T.x_empty[s]), ((xc / XST) & 1) ^ 1);
#pragma unroll
            for (int rh = 0; rh < RPT; ++rh) {
              const int r = pt + CV_PROD * rh;
              if (r >= XROWS) continue;
              const float* src = v[d][rh];
              if (F16) {
                unsigned char* row = Xs + s * XSTAGE + r * ROWB;
#pragma unroll
                for (int k8 = 0; k8 < CV_KC / 8; ++k8) {
                  float f[8];
#pragma unroll
                  for (int i = 0; i < 8; ++i) f[i] = p.relu_in ? fmaxf(src[8 * k8 + i], 0.f) : src[8 * k8 + i];
                  const int off = (k8 ^ ((r >> 1) & 3)) << 4;
                  *reinterpret_cast<uint4*>(row + off) =
                      make_uint4(f16x2_rn(f[0], f[1]), f16x2_rn(f[2], f[3]), f16x2_rn(f[4], f[5]), f16x2_rn(f[6], f[7]));
                }
              } else {
                unsigned char* hi = Xs + s * XSTAGE + r * 128;
                unsigned char* lo = hi + XPLANE;
#pragma unroll
                for (int k4 = 0; k4 < CV_KC / 4; ++k4) {
                  float4 f = make_float4(src[4 * k4], src[4 * k4 + 1], src[4 * k4 + 2], src[4 * k4 + 3]);
                  if (p.relu_in) f = make_float4(fmaxf(f.x, 0.f), fmaxf(f.y, 0.f), fmaxf(f.z, 0.f), fmaxf(f.w, 0.f));
                  const float4 h = make_float4(to_tf32(f.x), to_tf32(f.y), to_tf32(f.z), to_tf32(f.w));
                  const float4 l = make_float4(to_tf32(f.x - h.x), to_tf32(f.y - h.y), to_tf32(f.z - h.z), to_tf32(f.w - h.w));
                  const int off = (k4 ^ (r & 7)) << 4;
                  *reinterpret_cast<float4*>(hi + off) = h;
                  *reinterpret_cast<float4*>(lo + off) = l;
                }
              }
            }
            fence_proxy_async();
            mbar_arrive(smem_u32(&T.x_full[s]));
            ++xc;
            if (c + DEPTH < chunks) load(c + DEPTH, v[d]);
          }
        }
      }
    }
  } else {
    // ======================= MMA + epilogue: warpgroup G == output channels 64 G .. 64 G + 63 =======================
    const int G = warp >> 2, g = lane >> 2, t4 = lane & 3;
    const int cbase = 64 * G + 16 * (warp & 3) + g;          // fragment element 4 j + 2 h + e: channel cbase + 8 h,
    int i = 0, xc = 0;                                       // position 8 j + 2 t4 + e
    // The warpgroup's weight ring: rows 64 G .. 64 G + 63 of every plane of weight step j (both parts' steps in turn) go
    // to the same rows of stage j % CV_A_STAGES, copied by the warpgroup's thread 0 once its 128 threads have freed them.
    const int steps0 = (part0.c1 - part0.c0) * TAPS;
    const int nsteps = steps0 + (nparts == 2 ? (part1.c1 - part1.c0) * TAPS : 0);
    const bool issuer = (tid & 127) == 0;
    // first image step of each part, as scalars: the tap loop then reads no ConvPart (those live in local memory)
    const int wstep0 = (part0.cot * C + part0.c0) * TAPS, wstep1 = (part1.cot * C + part1.c0) * TAPS - steps0;
    auto issue_weights = [&](int j) {
      const unsigned char* src = p.wimg + (size_t)((j < steps0 ? wstep0 : wstep1) + j) * A_BYTES + G * A_HALF;
      const int s = j % CV_A_STAGES;
      const uint32_t dst = smem_u32(As + s * A_BYTES) + G * A_HALF, bar = smem_u32(&T.a_full[G][s]);
      mbar_arrive_expect_tx(bar, cv_planes(F16) * A_HALF);
#pragma unroll
      for (int pl = 0; pl < cv_planes(F16); ++pl) bulk_g2s(dst + pl * CV_M * ROWB, src + pl * CV_M * ROWB, A_HALF, bar);
    };
    if (issuer)
      for (int j = 0; j < CV_A_STAGES && j < nsteps; ++j) issue_weights(j);
    for (int pi = 0; pi < nparts; ++pi) {
      const ConvPart& P = pi ? part1 : part0;
      const int chunks = P.c1 - P.c0;
      float d[64], tot[64];
#pragma unroll
      for (int k = 0; k < 64; ++k) tot[k] = 0.f;
      wg_fence_acc(d);
      for (int c = 0; c < chunks; ++c, ++xc) {
        const int xs = xc % XST;
        mbar_wait(smem_u32(&T.x_full[xs]), (xc / XST) & 1);
        const uint32_t xb_hi = smem_u32(Xs + xs * XSTAGE), xb_lo = xb_hi + XPLANE;
#pragma unroll 1
        for (int t = 0; t < TAPS; ++t, ++i) {
          const int s = i % CV_A_STAGES;
          mbar_wait(smem_u32(&T.a_full[G][s]), (i / CV_A_STAGES) & 1);
          const uint32_t a_hi = smem_u32(As + s * A_BYTES) + G * 64 * ROWB, a_lo = a_hi + CV_M * 128;
          const uint32_t shift = KS == 3 ? (uint32_t)p.shift[t] * ROWB : 0u;
          wg_fence();
          if constexpr (F16) {
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)                     // k16 steps of 32 bytes
              wgmma_f16_n128(d, desc_sw64_kmajor(a_hi + ks * 32), desc_sw64_kmajor(xb_hi + shift + ks * 32), ks);
          } else {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
              const uint64_t da_hi = desc_sw128_kmajor(a_hi + ks * 32), da_lo = desc_sw128_kmajor(a_lo + ks * 32);
              const uint64_t db_hi = desc_sw128_kmajor(xb_hi + shift + ks * 32);
              const uint64_t db_lo = desc_sw128_kmajor(xb_lo + shift + ks * 32);
              wgmma_tf32_n128(d, da_lo, db_hi, ks != 0 ? 1 : 0);
              wgmma_tf32_n128(d, da_hi, db_lo, 1);
              wgmma_tf32_n128(d, da_hi, db_hi, 1);
            }
          }
          wg_commit();
          wg_wait0();
          wg_fence_acc(d);
          mbar_arrive(smem_u32(&T.a_empty[G][s]));
          if (issuer && i + CV_A_STAGES < nsteps) {
            mbar_wait(smem_u32(&T.a_empty[G][s]), (i / CV_A_STAGES) & 1);
            issue_weights(i + CV_A_STAGES);
          }
#pragma unroll
          for (int k = 0; k < 64; ++k) tot[k] += d[k];
        }
        mbar_arrive(smem_u32(&T.x_empty[xs]));
      }
      if (direct) {
        const bool to_stage = staged;
        // the staging buffer aliases the activation stages: both warpgroups' MMAs must be done with them
        if (to_stage) asm volatile("bar.sync 1, 256;" ::: "memory");
        float* stage = reinterpret_cast<float*>(smem);
#pragma unroll
        for (int k = 0; k < 64; ++k) {
          const int col = cbase + 8 * ((k >> 1) & 1), pos = 8 * (k >> 2) + 2 * t4 + (k & 1);
          if (pos >= p.N) continue;
          if (to_stage) {
            if (staged_nchw) stage[col * LD + pos] = tot[k];
            else stage[pos * CV_M + col] = tot[k];
            continue;
          }
          const int co = P.cot * CV_M + col;
          bool ok;
          long long pix;
          if (KS == 3) {
            const int ty = pos / TWp, lx = pos - ty * TWp;
            const int gy = P.ty0 + ty, gx = P.tx0 + lx - p.xoff;
            ok = lx >= p.xoff && lx < p.TW + p.xoff && ty < p.TH && gy < p.H && gx < p.W;
            pix = (long long)gy * p.W + gx;
          } else {
            pix = P.pix0 + pos;
            ok = pix < HW;
          }
          if (co < p.Cout && ok) {                         // the last channel tile may be padded (zero weight rows)
            float val = tot[k] + (p.bias ? __ldg(p.bias + co) : 0.f);
            if (p.z) val += __ldg(p.z + (long long)P.nb * p.zs_n + (long long)co * p.zs_c + pix * p.zs_p);
            if (p.relu_out) val = fmaxf(val, 0.f);
            p.y[(long long)P.nb * p.ys_n + (long long)co * p.ys_c + pix * p.ys_p] = val;
          }
        }
        if (tid == 0) T.last[0] = 1;
      } else {
        // ---- shares: partial tile -> workspace [tile][slot][position][channel] ----
        float* mine = p.ws + (P.tile_lin * p.maxslots + P.slot) * (long long)(p.N * CV_M);
#pragma unroll
        for (int k = 0; k < 64; ++k) {
          const int col = cbase + 8 * ((k >> 1) & 1), pos = 8 * (k >> 2) + 2 * t4 + (k & 1);
          if (pos < p.N) mine[pos * CV_M + col] = tot[k];
        }
      }
    }
    if (!direct) {
      __threadfence();
      asm volatile("bar.sync 1, 256;" ::: "memory");          // the two MMA warpgroups
      if (tid < nparts) {
        const ConvPart& P = tid ? part1 : part0;
        T.last[tid] = atomicAdd(p.counters + P.tile_lin, 1) == P.nslots - 1 ? 1 : 0;
      }
    }
  }
  // ================================== finish: all twelve warps ==================================
  for (int pi = 0; pi < nparts; ++pi) {
    const ConvPart& P = pi ? part1 : part0;
    asm volatile("bar.sync 2, 384;" ::: "memory");          // direct: the tile is staged; shares: who stores it is known
    const bool fin = T.last[pi] != 0;
    if (!direct && fin) {
      __threadfence();
      if (staged_nchw) {
        reduce_shares(P, warp, true);
      } else if (p.cl_vec) {
        reduce_shares(P, warp, false);
      } else if (warp < 4) {                               // odd layouts: thread == channel, element-wise
        const float* wst = p.ws + (P.tile_lin * p.maxslots) * (long long)(p.N * CV_M);
        const int co = P.cot * CV_M + tid;
        const float b = (p.bias && co < p.Cout) ? __ldg(p.bias + co) : 0.f;
        float* yb = p.y + (long long)P.nb * p.ys_n + (long long)co * p.ys_c;
        const float* zb = p.z ? p.z + (long long)P.nb * p.zs_n + (long long)co * p.zs_c : nullptr;
        for (int j = 0; j < p.N; ++j) {
          bool ok;
          long long pix;
          if (KS == 3) {
            const int ty = j / TWp, lx = j - ty * TWp;
            const int gy = P.ty0 + ty, gx = P.tx0 + lx - p.xoff;
            ok = lx >= p.xoff && lx < p.TW + p.xoff && ty < p.TH && gy < p.H && gx < p.W;
            pix = (long long)gy * p.W + gx;
          } else {
            pix = P.pix0 + j;
            ok = pix < HW;
          }
          if (!ok || co >= p.Cout) continue;
          float val = 0.f;
          for (int k = 0; k < P.nslots; ++k) val += __ldcg(wst + ((long long)k * p.N + j) * CV_M + tid);
          val += b;
          if (zb) val += __ldg(zb + pix * p.zs_p);
          if (p.relu_out) val = fmaxf(val, 0.f);
          yb[pix * p.ys_p] = val;
        }
      }
    }
    if (staged_nchw) {
      if (!direct) asm volatile("bar.sync 2, 384;" ::: "memory");   // shares added up in the staging buffer
      if (fin) store_staged_rows(P, warp);
    } else if (direct && p.cl_vec) {
      store_staged_rows(P, warp);
    }
    if (pi + 1 < nparts) asm volatile("bar.sync 2, 384;" ::: "memory");   // staging buffer free again
    if (!direct && fin && tid == 0) p.counters[P.tile_lin] = 0;           // ready for the next launch
  }
}

// weight operand image: one thread per (output channel, chunk, tap, 16-byte piece); weight [Cout, Cin, KS, KS]
__global__ void __launch_bounds__(256) conv_weight_image_kernel(const float* __restrict__ w, int Cout, int Cin, int taps,
                                                                unsigned char* __restrict__ img) {
  const int chunks = Cin / CV_KC;
  const long long total = (long long)((Cout + CV_M - 1) / CV_M * CV_M) * chunks * taps * 8;
  const long long f = (long long)blockIdx.x * 256 + threadIdx.x;
  if (f >= total) return;
  const int k4 = (int)(f & 7);
  long long g = f >> 3;
  const int row = (int)(g % CV_M); g /= CV_M;
  const int t = (int)(g % taps); g /= taps;
  const int c = (int)(g % chunks);
  const int cot = (int)(g / chunks);
  const int co = cot * CV_M + row;
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = co < Cout ? w[((long long)co * Cin + c * CV_KC + 4 * k4 + i) * taps + t] : 0.f;
  const float4 h = make_float4(to_tf32(v[0]), to_tf32(v[1]), to_tf32(v[2]), to_tf32(v[3]));
  const float4 l = make_float4(to_tf32(v[0] - h.x), to_tf32(v[1] - h.y), to_tf32(v[2] - h.z), to_tf32(v[3] - h.w));
  unsigned char* blk = img + (((size_t)cot * chunks + c) * taps + t) * cv_a_bytes(false);
  const int off = row * 128 + ((k4 ^ (row & 7)) << 4);
  *reinterpret_cast<float4*>(blk + off) = h;
  *reinterpret_cast<float4*>(blk + CV_M * 128 + off) = l;
}

// FP16 weight operand image: one fp16 [128 x 32] plane per (128-channel tile, chunk, tap), rows of 64 B in K-major
// SWIZZLE_64B order; one thread per (output channel, chunk, tap, 16-byte piece of 8 channels)
__global__ void __launch_bounds__(256) conv_weight_image_f16_kernel(const float* __restrict__ w, int Cout, int Cin, int taps,
                                                                    unsigned char* __restrict__ img) {
  const int chunks = Cin / CV_KC;
  const long long total = (long long)((Cout + CV_M - 1) / CV_M * CV_M) * chunks * taps * 4;
  const long long f = (long long)blockIdx.x * 256 + threadIdx.x;
  if (f >= total) return;
  const int k8 = (int)(f & 3);
  long long g = f >> 2;
  const int row = (int)(g % CV_M); g /= CV_M;
  const int t = (int)(g % taps); g /= taps;
  const int c = (int)(g % chunks);
  const int cot = (int)(g / chunks);
  const int co = cot * CV_M + row;
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = co < Cout ? w[((long long)co * Cin + c * CV_KC + 8 * k8 + i) * taps + t] : 0.f;
  unsigned char* blk = img + (((size_t)cot * chunks + c) * taps + t) * cv_a_bytes(true);
  *reinterpret_cast<uint4*>(blk + row * 64 + ((k8 ^ ((row >> 1) & 3)) << 4)) =
      make_uint4(f16x2_rn(v[0], v[1]), f16x2_rn(v[2], v[3]), f16x2_rn(v[4], v[5]), f16x2_rn(v[6], v[7]));
}

}  // namespace

}  // namespace cutie

using namespace cutie;

// argument checks of the entry points below that share a body: the message names the entry point (`fn`) like CUTIE_REQUIRE
#define CONV_REQUIRE(cond, what)                                                          \
  do {                                                                                    \
    if (!(cond)) return ::cutie::fail(-1, "%s: invalid argument: " what, fn);            \
  } while (0)

static int64_t conv_weight_image_bytes(int64_t Cout, int64_t Cin, int ksize, bool f16) {
  if (Cout < 1 || Cin < CV_KC || Cin % CV_KC || (ksize != 1 && ksize != 3)) return -1;
  return ((Cout + CV_M - 1) / CV_M) * (Cin / CV_KC) * ksize * ksize * (int64_t)cv_a_bytes(f16);
}

static int conv_weight_image(const char* fn, bool f16, const float* weight, int64_t Cout, int64_t Cin, int ksize, void* image,
                             void* stream) {
  CONV_REQUIRE(weight && image, "null argument");
  CONV_REQUIRE(ksize == 1 || ksize == 3, "1x1 or 3x3");
  CONV_REQUIRE(Cout >= 1 && Cin >= CV_KC && Cin % CV_KC == 0, "input channels must be a multiple of 32");
  const int taps = ksize * ksize;
  const long long pieces = (Cout + CV_M - 1) / CV_M * CV_M * (Cin / CV_KC) * taps;   // x 16-byte pieces per row
  if (f16)
    conv_weight_image_f16_kernel<<<(unsigned)((pieces * 4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        weight, (int)Cout, (int)Cin, taps, static_cast<unsigned char*>(image));
  else
    conv_weight_image_kernel<<<(unsigned)((pieces * 8 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        weight, (int)Cout, (int)Cin, taps, static_cast<unsigned char*>(image));
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : ::cutie::set_cuda_error(fn, e);
}

extern "C" int64_t cutie_conv_weight_image_bytes(int64_t Cout, int64_t Cin, int ksize) {
  return conv_weight_image_bytes(Cout, Cin, ksize, false);
}

extern "C" int cutie_conv_weight_image(const float* weight, int64_t Cout, int64_t Cin, int ksize, void* image, void* stream) {
  return conv_weight_image(__func__, false, weight, Cout, Cin, ksize, image, stream);
}

extern "C" int64_t cutie_conv_weight_image_f16_bytes(int64_t Cout, int64_t Cin, int ksize) {
  return conv_weight_image_bytes(Cout, Cin, ksize, true);
}

extern "C" int cutie_conv_weight_image_f16(const float* weight, int64_t Cout, int64_t Cin, int ksize, void* image, void* stream) {
  return conv_weight_image(__func__, true, weight, Cout, Cin, ksize, image, stream);
}

// 3x3 spatial tile: TW | tile width (full rows when they fit), TH rows, N = round16(TH * (TW + 2)) <= 128 and
// N + 2 (TW + 2) + 2 <= 248 rows; maximise useful pixels per MMA column over the whole image (edge tiles included)
// (stride 2: four parity planes of (TH + 1) x (TW + 1) rows each, N = round16(TH * (TW + 1)))
static int conv_plane_rows(int th, int tw, int n) { return (th + 1) * (tw + 1) + (n - th * (tw + 1)) + 1; }
static void conv_tile_shape(int H, int W, int stride, int* TH, int* TW, int* N) {
  double best = -1;
  const int pad = stride == 1 ? 2 : 1;
  for (int parts = 1; parts <= W; ++parts) {
    const int tw = (W + parts - 1) / parts;
    for (int th = 1; th <= H && th * (tw + pad) <= 128; ++th) {
      const int n = (th * (tw + pad) + 15) / 16 * 16;
      if (stride == 1 ? n + 2 * (tw + 2) + 2 > CV3_ROWS : 4 * conv_plane_rows(th, tw, n) > CV3_ROWS) continue;
      const long long tiles = (long long)((H + th - 1) / th) * ((W + tw - 1) / tw);
      const double eff = (double)H * W / ((double)tiles * n);
      // the most useful pixels per MMA column; among equals the larger N (fewer CTAs re-reading the weights)
      if (eff > best + 1e-9 || (eff > best - 1e-9 && n > *N)) { best = eff; *TH = th; *TW = tw; *N = n; }
    }
    if (tw <= 8) break;
  }
}

// Launch plan.  Work = (output tile, input chunk) units, T tiles x C chunks; CTA i owns units [i q, (i + 1) q) -- any q <= C
// is valid (a share then spans at most two tiles and a tile is shared by at most ceil(C / q) + 1 CTAs, which meet in the
// workspace).  Layers with at least as many output tiles as SMs run one whole tile per CTA (q = C); smaller layers split
// every tile uniformly over input-channel ranges.
struct ConvPlan { long long tiles, cots, T; int N, C, q, maxslots; long long ctas; int th, tw; };
static int conv_make_plan(int64_t NB, int64_t Cin, int64_t Cout, int64_t H_in, int64_t W_in, int ksize, int stride, int q_override,
                          ConvPlan* pl) {
  const int H = (int)((H_in - 1) / stride + 1), W = (int)((W_in - 1) / stride + 1);
  pl->th = pl->tw = 0; pl->N = 0;
  if (ksize == 3) {
    conv_tile_shape(H, W, stride, &pl->th, &pl->tw, &pl->N);
    if (pl->N < 16) return -1;
    pl->tiles = (long long)((W + pl->tw - 1) / pl->tw) * ((H + pl->th - 1) / pl->th);
  } else {
    const long long hw = (long long)H * W;
    pl->N = hw >= 128 ? 128 : (int)((hw + 15) / 16 * 16);
    pl->tiles = (hw + pl->N - 1) / pl->N;
  }
  pl->cots = (Cout + CV_M - 1) / CV_M;
  pl->T = pl->tiles * pl->cots * NB;
  pl->C = (int)(Cin / CV_KC);
  int q = pl->C;
  // Shares that stay inside one tile (q | C, i.e. a uniform split of every tile) cost one partial-tile round trip through
  // the workspace; shares that straddle two tiles pay it twice per CTA on the critical path and measured slower than not
  // sharing at all (scripts/conv_share_sweep.py: 256->256 3x3 x3 objects 65 us whole tiles, 101 us at q = 5), so the plan
  // only picks divisors of C: the largest split s with CTAs x s <= SMs and at least 2 chunks per CTA.
  for (int s = 2; s <= 8; ++s)
    if (pl->C % s == 0 && pl->T * s <= num_sms() && pl->C / s >= 2) q = pl->C / s;
  if (q_override > 0) q = q_override < pl->C ? q_override : pl->C;
  pl->q = q;
  pl->maxslots = (pl->C - 1) / q + 2;
  pl->ctas = (pl->T * pl->C + q - 1) / q;
  return 0;
}

extern "C" int cutie_conv_plan(int64_t NB, int64_t Cin, int64_t Cout, int64_t H_in, int64_t W_in, int ksize, int stride,
                               int units_per_cta, int64_t* out6) {
  CUTIE_REQUIRE(out6 && (ksize == 1 || ksize == 3) && (stride == 1 || stride == 2) && Cin >= CV_KC && Cin % CV_KC == 0 && NB >= 1 &&
                    Cout >= 1, "bad arguments");
  ConvPlan pl;
  CUTIE_REQUIRE(conv_make_plan(NB, Cin, Cout, H_in, W_in, ksize, stride, units_per_cta, &pl) == 0, "no tile shape for this geometry");
  out6[0] = pl.T; out6[1] = pl.N; out6[2] = pl.C; out6[3] = pl.q; out6[4] = pl.ctas;
  out6[5] = pl.q < pl.C ? pl.T * pl.maxslots * (long long)pl.N * CV_M : 0;          // workspace floats (0: none needed)
  return 0;
}

template <bool F16>
static int conv_tc_launch(const char* fn, const float* x, const int64_t* x_strides, const void* weight_image, const float* bias,
                          const float* residual, const int64_t* residual_strides, int64_t NB, int64_t Cin, int64_t Cout,
                          int64_t H_in, int64_t W_in, int ksize, int stride, int relu_in, int relu_out, float* y,
                          const int64_t* y_strides, int units_per_cta, float* workspace, int32_t* counters, void* stream) {
  CONV_REQUIRE(x && x_strides && weight_image && y && y_strides, "null argument");
  CONV_REQUIRE(residual == nullptr || residual_strides != nullptr, "residual needs strides");
  CONV_REQUIRE((ksize == 3 || ksize == 1) && (stride == 1 || stride == 2), "3x3 (zero pad 1) or 1x1, stride 1 or 2");
  CONV_REQUIRE(Cout >= 1 && Cin >= CV_KC && Cin % CV_KC == 0, "input channels must be a multiple of 32");
  CONV_REQUIRE(NB >= 1 && NB <= 65535 && H_in >= 1 && W_in >= 1 && H_in * W_in < (1ll << 30), "bad geometry");
  ConvPlan pl;
  CONV_REQUIRE(conv_make_plan(NB, Cin, Cout, H_in, W_in, ksize, stride, units_per_cta, &pl) == 0, "no tile shape for this geometry");
  CONV_REQUIRE(pl.q == pl.C || (workspace && counters), "shared tiles need the workspace and zeroed counters (cutie_conv_plan)");
  CONV_REQUIRE(pl.ctas <= 0x7fffffff, "too many tiles");
  ConvTcParams p;
  p.x = x; p.wimg = static_cast<const unsigned char*>(weight_image); p.bias = bias; p.z = residual; p.y = y;
  p.xs_n = x_strides[0]; p.xs_c = x_strides[1]; p.xs_p = x_strides[2];
  p.ys_n = y_strides[0]; p.ys_c = y_strides[1]; p.ys_p = y_strides[2];
  p.zs_n = residual ? residual_strides[0] : 0;
  p.zs_c = residual ? residual_strides[1] : 0;
  p.zs_p = residual ? residual_strides[2] : 0;
  p.Cin = (int)Cin; p.Cout = (int)Cout; p.Hi = (int)H_in; p.Wi = (int)W_in; p.stride = stride;
  p.H = (int)((H_in - 1) / stride + 1); p.W = (int)((W_in - 1) / stride + 1);
  p.relu_in = relu_in; p.relu_out = relu_out;
  // channels-last input: a producer thread reads its pixel's 32 channels as 8 x 16 bytes
  p.x_vec = (p.xs_c == 1 && p.xs_p % 4 == 0 && p.xs_n % 4 == 0 && reinterpret_cast<uintptr_t>(x) % 16 == 0) ? 1 : 0;
  auto vec4 = [](const void* ptr, long long sn, long long sc, long long sp) {
    return sc == 1 && sp % 4 == 0 && sn % 4 == 0 && reinterpret_cast<uintptr_t>(ptr) % 16 == 0;
  };
  p.cl_vec = (Cout % 4 == 0 && vec4(y, p.ys_n, p.ys_c, p.ys_p) && (bias == nullptr || reinterpret_cast<uintptr_t>(bias) % 16 == 0) &&
              (residual == nullptr || vec4(residual, p.zs_n, p.zs_c, p.zs_p))) ? 1 : 0;
  p.TH = pl.th; p.TW = pl.tw; p.N = pl.N; p.tiles_x = 1; p.pitch = 2; p.xoff = 0; p.plane_rows = 0;
  for (int t = 0; t < 9; ++t) p.shift[t] = 0;
  if (ksize == 3) {
    p.tiles_x = (p.W + p.TW - 1) / p.TW;
    if (stride == 1) {
      p.pitch = p.TW + 2; p.xoff = 1;
      for (int t = 0; t < 9; ++t) p.shift[t] = (t / 3) * p.pitch + (t % 3);
    } else {
      p.pitch = p.TW + 1; p.xoff = 0; p.plane_rows = conv_plane_rows(p.TH, p.TW, p.N);
      for (int t = 0; t < 9; ++t) {
        const int dy = t / 3, dx = t % 3;
        const int plane = (dy != 1 ? 2 : 0) + (dx != 1 ? 1 : 0);
        p.shift[t] = plane * p.plane_rows + (dy == 0 ? 0 : 1) * p.pitch + (dx == 0 ? 0 : 1);
      }
    }
  }
  p.q = pl.q; p.T = (int)pl.T; p.tiles = (int)pl.tiles; p.cots = (int)pl.cots; p.maxslots = pl.maxslots;
  p.ws = workspace; p.counters = counters;
  CONV_REQUIRE(pl.T <= 0x7fffffff, "too many tiles");
  static bool attr_done[64] = {};                            // (one per instantiation, i.e. per precision)
  if (first_use_on_device(attr_done)) {
    cudaFuncSetAttribute(conv_tc_kernel<3, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_smem(3, F16));
    cudaFuncSetAttribute(conv_tc_kernel<1, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_smem(1, F16));
  }
  if (ksize == 3)
    conv_tc_kernel<3, F16><<<(unsigned)pl.ctas, CV_THREADS, cv_smem(3, F16), (cudaStream_t)stream>>>(p);
  else
    conv_tc_kernel<1, F16><<<(unsigned)pl.ctas, CV_THREADS, cv_smem(1, F16), (cudaStream_t)stream>>>(p);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : ::cutie::set_cuda_error(fn, e);
}

extern "C" int cutie_conv_tc(const float* x, const int64_t* x_strides, const void* weight_image, const float* bias,
                             const float* residual, const int64_t* residual_strides, int64_t NB, int64_t Cin, int64_t Cout,
                             int64_t H_in, int64_t W_in, int ksize, int stride, int relu_in, int relu_out, float* y,
                             const int64_t* y_strides, int units_per_cta, float* workspace, int32_t* counters, void* stream) {
  return conv_tc_launch<false>(__func__, x, x_strides, weight_image, bias, residual, residual_strides, NB, Cin, Cout, H_in, W_in,
                               ksize, stride, relu_in, relu_out, y, y_strides, units_per_cta, workspace, counters, stream);
}

extern "C" int cutie_conv_tc_f16(const float* x, const int64_t* x_strides, const void* weight_image, const float* bias,
                                 const float* residual, const int64_t* residual_strides, int64_t NB, int64_t Cin, int64_t Cout,
                                 int64_t H_in, int64_t W_in, int ksize, int stride, int relu_in, int relu_out, float* y,
                                 const int64_t* y_strides, int units_per_cta, float* workspace, int32_t* counters, void* stream) {
  return conv_tc_launch<true>(__func__, x, x_strides, weight_image, bias, residual, residual_strides, NB, Cin, Cout, H_in, W_in,
                              ksize, stride, relu_in, relu_out, y, y_strides, units_per_cta, workspace, counters, stream);
}

extern "C" int cutie_debug_conv_tile_shape(int64_t H, int64_t W, int* out3) {
  int th = 0, tw = 0, n = 0;
  conv_tile_shape((int)H, (int)W, 1, &th, &tw, &n);
  out3[0] = th; out3[1] = tw; out3[2] = n;
  return 0;
}
