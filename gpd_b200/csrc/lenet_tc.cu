// lenet_tc.cu — LeNet conv1 / conv2 / ip1 (A14) on the sm_90a tensor cores (warpgroup wgmma.mma_async, accumulators in
// registers).
//
// Both convolutions are IM2COL-FREE implicit GEMMs. The activations of one image live in shared memory as
// "channel planes": plane p holds channels 8p..8p+7 of every pixel as one 16-byte group, pixels in row-major
// order. For output pixel m = y*W + x (W = input width) and filter tap (kh, kw) the 8 channels it needs are the
// 16-byte group  plane_p[m + kh*W + kw]  — so the A operand of the GEMM (rows = output pixels, K = taps x
// channels) is a Hankel matrix over that plane: row stride 16 B, K-chunk stride 16 B. This is exactly a K-major
// no-swizzle wgmma shared-memory descriptor with SBO = 128 B (8 rows x 16 B) and LBO = the byte distance between
// the two K-chunks of one instruction. No patch matrix is ever materialised; every wgmma reads the plane directly.
//
// Precision: the reference computes in float32 on raw 0..255 inputs (logits ~1e3), tolerance 1e-4 relative.
//   conv1: integer path (u8 x s8 -> s32): the uint8 image is the A operand as it is; each weight is a 24-bit integer times
//          a per-filter scale, split into three balanced int8 digits stacked along N (60 of the 64 B rows, see c1_col) so
//          ONE instruction stream reads A once; the int32 dot products are exact and the epilogue recombines the three
//          digits in float32 (see k_conv1_i8 below).
//   conv2: activations a and weights w are scaled by powers of two (exact) and split in two fp16 terms each;
//          D += w_hi a_hi + w_lo a_hi + w_hi a_lo  (error ~2^-22), with the filters as M and the pixels as N.
// Output pixels with x beyond the valid width are computed and discarded (7 % / 14 % of the rows / columns).
//
// conv1 computes a tile of 128 GEMM rows with two warpgroups (rows 0..63 | 64..127); conv2 is warp-specialised: a converter
// warpgroup feeds two consumer warpgroups that each own whole 224-column tiles and alternate on the tensor cores. The
// weights stay resident in shared memory (26.6 KB / 132 KB). The 2x2 max-pool + bias (+ReLU for the 12-channel net) is
// fused into the epilogue: conv1: registers -> x-pair max by shuffle -> small smem stage -> y-pair max -> global;
// conv2: x-pair max in registers -> y-pair max by shuffle -> small smem stage -> global.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int NF1 = 20, NF2 = 50, NH = 500;

// ---------------------------------------------------------------------------------------------------------
// conv1: image 60x60 P16 (16-byte pixels: C uint8 channels, zero padded) -> P1 [784 px][20] float32 (pixel-major), 2x2 max-pooled.
// Integer tensor-core path (wgmma .s32.u8.s8, int32 accumulators): the uint8 image IS the A operand — one pixel = one 16-byte
// K-chunk (C <= 16 channels, zero padded), so an instruction (K = 32) covers two filter taps.
// Weights: w = s_o * W, W a 24-bit signed integer (s_o = max|w_o| / 8.3e6 per filter), W = 65536 d0 + 256 d1 + d2 with
// balanced int8 digits; the three digit planes are B rows (accumulator columns) c1_col(o, digit), chosen so that the thread
// holding a row holds all three digits of its filters. The dot products are EXACT integers; the epilogue recombines them in
// float32 (error ~1e-7 relative, like float32 itself).
// tiles: 28 per image, tile t = output rows 2t, 2t+1 = GEMM rows m0 = 120 t .. +119 (of 128): 120 CONSECUTIVE pixels, so the
// 8-row core matrices of an A chunk are one contiguous range (SBO = 128 B).
// Two CTAs per SM (88 KB of shared memory each): while one waits for its next image (one bulk-async copy of the P16 image into
// its operand plane) or runs its epilogue, the other's instructions keep the tensor cores busy.
// ---------------------------------------------------------------------------------------------------------
constexpr int C1_W = 60, C1_NPIX = 3616, C1_PLANE = C1_NPIX * 16, C1_TILES = 28, C1_TILE_ROWS = 120;
constexpr int C1_N = 64, C1_BCHUNK = C1_N * 16;  // B rows: 3 digits x 20 filters (c1_col) + 4 zero rows
constexpr int C1_NCH = 25, C1_NMMA = 13;         // chunk c = kh*5 + kw (+1 zero-weight chunk)
constexpr int C1_NT = 256, C1_CTAS_PER_SM = 2;
constexpr int C1_IMG_BYTES = C1_W * C1_W * 16;  // one P16 image
constexpr int C1_B_BYTES = 2 * C1_NMMA * C1_BCHUNK;
constexpr int C1_STAGE_FLOATS = 28 * NF1;       // x-pooled upper output row of a tile
constexpr double C1_W_MAX = 127.0 * 65536 + 127.0 * 257;  // largest |W| of three balanced int8 digits (top digit <= 127)

// chunk c -> byte offset of row 0 inside the plane (monotonic in c)
__host__ __device__ constexpr uint32_t c1_off(int c) {
  return (uint32_t)((((c >= C1_NCH ? C1_NCH - 1 : c) / 5) * C1_W + (c >= C1_NCH ? C1_NCH - 1 : c) % 5) * 16);
}
// accumulator column (= B row) of digit tm of filter o: filter o = 4 f + q lives in the columns of lane quad q (8 j + 2 q + e),
// its digits in slots s = 3 f + tm (j = s / 2, e = s % 2) — thread slot s is accumulator value 4 (s / 2) + (s % 2) (+2: row + 8)
__host__ __device__ constexpr int c1_col(int o, int tm) {
  return 8 * ((3 * (o >> 2) + tm) >> 1) + 2 * (o & 3) + ((3 * (o >> 2) + tm) & 1);
}
__device__ __forceinline__ constexpr int c1_slot_reg(int s, int h) { return 4 * (s >> 1) + 2 * h + (s & 1); }

__global__ void __launch_bounds__(C1_NT, C1_CTAS_PER_SM) k_conv1_i8(const uint8_t *__restrict__ images /* P16 */, int n,
                                                                    const uint8_t *__restrict__ wblob,
                                                                    const C1Affine aff /* constant bank */, int relu,
                                                                    float *__restrict__ p1) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t pl_full;
  uint8_t *sB = smem;                                            // 26 chunks x 64 rows x 16 B (int8)
  uint8_t *sPl = sB + C1_B_BYTES;                                // 3616 px x 16 B (uint8)
  float *stage = reinterpret_cast<float *>(sPl + C1_PLANE);      // 2 x [28][20], alternating between tiles
  const int tid = threadIdx.x, wg_id = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;

  for (int i = tid; i < C1_B_BYTES / 16; i += C1_NT) reinterpret_cast<uint4 *>(sB)[i] = reinterpret_cast<const uint4 *>(wblob)[i];
  for (int i = C1_IMG_BYTES / 16 + tid; i < C1_PLANE / 16; i += C1_NT) reinterpret_cast<uint4 *>(sPl)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    wg::mbar_init(&pl_full, 1);  // the expect_tx arrival + the bulk copy's bytes
    wg::fence_mbar_init();
  }
  wg::fence_async_smem();  // weights and the zero tail (generic proxy) before the tensor-core reads (async proxy)
  __syncthreads();

  const uint32_t sB_u = wg::smem_u32(sB), sPl_u = wg::smem_u32(sPl) + (uint32_t)wg_id * 64 * 16;
  int it = 0;
  for (int im = blockIdx.x; im < n; im += gridDim.x, it++) {
    if (tid == 0) {
      wg::mbar_expect_tx(&pl_full, C1_IMG_BYTES);
      wg::bulk_g2s(sPl, images + (size_t)im * C1_IMG_BYTES, C1_IMG_BYTES, &pl_full);
    }
    wg::mbar_wait(&pl_full, it & 1);
    float *out = p1 + (size_t)im * 784 * NF1;
    for (int t = 0; t < C1_TILES; t++) {
      int32_t d[32];
      const uint32_t arow = sPl_u + (uint32_t)(t * C1_TILE_ROWS) * 16;
      wg::fence();
#pragma unroll
      for (int i = 0; i < C1_NMMA; i++) {
        const uint32_t a0 = c1_off(2 * i), a1 = c1_off(2 * i + 1);
        const uint32_t lbo = (2 * i + 1 >= C1_NCH) ? 16u : (a1 - a0);
        wg::mma_u8s8_n64(d, wg::desc(arow + a0, lbo, 128), wg::desc(sB_u + (uint32_t)(2 * i) * C1_BCHUNK, C1_BCHUNK, 128), i > 0);
      }
      wg::commit();
      wg::wait<0>();
      wg::reg_fence(d);
      // recombine the three digits of this thread's 5 filters (o = 4 f + q) for its two rows, then the x-pair max: rows r, r + 1
      // are lanes l, l ^ 4
      float v[2][5];
#pragma unroll
      for (int h = 0; h < 2; h++)
#pragma unroll
        for (int f = 0; f < 5; f++) {
          const float f0 = (float)d[c1_slot_reg(3 * f, h)], f1 = (float)d[c1_slot_reg(3 * f + 1, h)],
                      f2 = (float)d[c1_slot_reg(3 * f + 2, h)];
          v[h][f] = fmaf(f0, 65536.0f, fmaf(f1, 256.0f, f2));
          v[h][f] = fmaxf(v[h][f], __shfl_xor_sync(0xffffffffu, v[h][f], 4));
        }
      float *stg = stage + (t & 1) * C1_STAGE_FLOATS;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int r = wg_id * 64 + warp * 16 + (lane >> 2) + 8 * h, x = r >= C1_W ? r - C1_W : r;
        if (r < C1_W && (x & 1) == 0 && x < 56) {
#pragma unroll
          for (int f = 0; f < 5; f++) stg[(x >> 1) * NF1 + 4 * f + q] = v[h][f];
        }
      }
      __syncthreads();  // the upper row is staged; a stage buffer is rewritten two tiles later, after the next barrier
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int r = wg_id * 64 + warp * 16 + (lane >> 2) + 8 * h, x = r - C1_W;
        if (r >= C1_W && r < C1_TILE_ROWS && (x & 1) == 0 && x < 56) {
          float *o = out + (size_t)(t * 28 + (x >> 1)) * NF1;
#pragma unroll
          for (int f = 0; f < 5; f++) {
            const int ch = 4 * f + q;
            float m = fmaxf(v[h][f], stg[(x >> 1) * NF1 + ch]);
            m = fmaf(m, aff.scale[ch], aff.bias[ch]);
            if (relu) m = fmaxf(m, 0.0f);
            o[ch] = m;
          }
        }
      }
    }
    __syncthreads();  // every instruction of this image has read the plane before the next bulk copy overwrites it
  }
}

// ---------------------------------------------------------------------------------------------------------
// conv2: P1 [784 px][20] f32 -> ip1's fp16 hi/lo operand xc (k = c + 50 j, j = 12x12 pooled pixel), max-pooled.
// Transposed implicit GEMM: M = the 50 filters (padded to 64) = the weights as the A operand, N = 224 output pixels, K = taps x
// channels. Tile T (3 per image) = output rows 8T .. 8T+7 = GEMM columns n = y*28 + x over the TWELVE input rows 8T .. 8T+11
// (336 consecutive P1 pixels, 26.25 KB), held as six fp16 channel planes (hi p0..2, lo p0..2; plane 2 pairs two pixels, see
// c2_off) of 344 pixels. The 4 halo rows of a tile are converted twice. One CTA per SM, three warpgroups:
//   warpgroup 0, converter: loads a tile's float32 pixels from global memory (L2: a bulk prefetch pulls each tile in two
//     tiles ahead) straight into registers, converts them to the scaled fp16 hi/lo planes of a plane stage and arrives on
//     its `full` barrier.
//   warpgroups 1, 2, consumers: consumer c owns the tiles g = c, c + 2, ... of the CTA's sequence (and plane stage c) and
//     issues 33 x 3 m64n224k16 per tile. Named barriers order the two consumers' instruction batches (ping-pong), so the
//     tensor cores run one consumer's tile while the other runs its epilogue (x-pair max in registers, y-pair max by
//     shuffle -> own stage -> bias -> 16-byte stores of 8 consecutive k of xc).
// The three products w_hi a_hi, w_lo a_hi, w_hi a_lo land on the same output element at the same scale: ONE accumulator.
// An instruction reads 2 KB of weights + 7 KB of pixels per 112 tensor clocks (~82 B / clock of shared memory), and a
// tile's batch runs 11 088 tensor clocks, so the consumers hand the tensor cores over half as often per pixel as with
// 128-pixel tiles.
// ---------------------------------------------------------------------------------------------------------
constexpr int C2_W = 28, C2_NCH = 65, C2_NMMA = 33;
constexpr int C2_TILES = 3, C2_N = 8 * C2_W, C2_TILE_PIX = 12 * C2_W;  // 224 GEMM columns over 336 input pixels per tile
constexpr int C2_NPIX = C2_TILE_PIX + 8, C2_PLANE = C2_NPIX * 16;      // + an 8-pixel zero tail
constexpr int C2_ACHUNK = 2 * 64 * 16;                                  // one K-chunk of A: w_hi rows 0..63, w_lo rows 0..63
constexpr int C2_A_BYTES = 2 * C2_NMMA * C2_ACHUNK;                    // 66 chunks (the last one zero)
constexpr int C2_STAGE = 6 * C2_PLANE;                                  // one plane stage: hi p0..2, lo p0..2
constexpr int C2_STG_FLOATS = 4 * 12 * 50;                              // a tile's pooled outputs [py 0..3][px 0..11][50]
constexpr int C2_NT = 384;
// Shared memory: [A: 66 chunks x (hi, lo) x 64 rows x 16 B = 135 168 B][2 plane stages x 6 x 344 px x 16 B = 66 048 B]
// [2 pooled stages x 2 400 floats = 19 200 B] = 220 416 B dynamic. GEMM column n of chunk c reads pixel n + c2_off(c) / 16
// (+1 for the zero chunk 65, LBO 16), at most 223 + 4 * 28 + 4 + 1 = 340 of its plane: pixels 336..343 are the zero tail,
// written once, and only columns with x >= 24 (discarded) reach them, except as a right neighbour of plane 2 whose
// weights (tap kw = 5) are zero. The valid tap reads of a column stay in its own row, so nothing else crosses planes.
constexpr int C2_SMEM = C2_A_BYTES + 2 * C2_STAGE + 2 * C2_STG_FLOATS * 4;
static_assert(C2_SMEM + 64 * 4 + 4 * 8 <= 227 * 1024, "conv2: dynamic + static shared memory above the opt-in limit");
constexpr int IP_K = 7200, IP_KCH = IP_K / 8;  // ip1 reduction length, in 8-element chunks
// K-chunks (8 fp16 = 16 B per GEMM column): c < 50: plane p = c / 25 (channels 8p .. 8p+7), tap (kh, kw) = c % 25.
// c >= 50: plane 2 holds, per pixel, channels 16..19 of that pixel AND of its right neighbour, so one chunk covers the two
// taps (kh, 2j) and (kh, 2j+1) of the last four channels, j = (c - 50) % 3, kh = (c - 50) / 3 (the tap kw = 5 of j = 2 has
// zero weights): 65 chunks instead of 75 with a zero-padded third plane (-13 % tensor-core work).
__host__ __device__ constexpr uint32_t c2_off(int c) {
  const int cc = c >= C2_NCH ? C2_NCH - 1 : c;
  return cc < 50 ? (uint32_t)((cc / 25) * C2_PLANE + (((cc / 5) % 5) * C2_W + cc % 5) * 16)
                 : (uint32_t)(2 * C2_PLANE + (((cc - 50) / 3) * C2_W + 2 * ((cc - 50) % 3)) * 16);
}

__global__ void __launch_bounds__(C2_NT, 1) k_conv2_tc(const float *__restrict__ p1, int n, const uint8_t *__restrict__ wblob,
                                                       const float *__restrict__ bias, float a_scale, float out_scale, int relu,
                                                       __half *__restrict__ xc, float x_scale) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ float sbias[64];
  __shared__ uint64_t full[2], empty[2];
  uint8_t *sA = smem;                   // 66 chunks x (w_hi | w_lo) x 64 rows x 16 B
  uint8_t *sPl = sA + C2_A_BYTES;       // 2 plane stages
  float *stg = reinterpret_cast<float *>(sPl + 2 * C2_STAGE);  // the pooled stages of the two consumers
  const int tid = threadIdx.x, wg_id = tid >> 7, wt = tid & 127, warp = wt >> 5, lane = tid & 31, q = lane & 3;

  for (int i = tid; i < C2_A_BYTES / 16; i += C2_NT) reinterpret_cast<uint4 *>(sA)[i] = reinterpret_cast<const uint4 *>(wblob)[i];
  for (int i = tid; i < 2 * 6 * 8; i += C2_NT)
    reinterpret_cast<uint4 *>(sPl + (i >> 3) * C2_PLANE + (C2_TILE_PIX + (i & 7)) * 16)[0] = make_uint4(0, 0, 0, 0);
  if (tid < 64) sbias[tid] = tid < NF2 ? bias[tid] : 0.0f;
  if (tid == 0) {
    for (int s = 0; s < 2; s++) {
      wg::mbar_init(&full[s], 128);  // every converter thread, after its own proxy fence
      wg::mbar_init(&empty[s], 4);   // one arrival per consumer warp
    }
    wg::fence_mbar_init();
  }
  wg::fence_async_smem();  // weights and zero tails (generic proxy) before the tensor-core reads (async proxy)
  __syncthreads();

  // the CTA's tiles g = 0 .. G-1: image blockIdx.x + (g / 3) * gridDim.x, tile g % 3
  const int G = C2_TILES * ((n - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x);
  auto tile_src = [&](int g) {
    return p1 + ((size_t)blockIdx.x + (size_t)(g / C2_TILES) * gridDim.x) * 784 * NF1 + (size_t)(g % C2_TILES) * 8 * C2_W * NF1;
  };

  if (wg_id == 0) {
    // ===== converter
    wg::setmaxnreg_dec<40>();
    if (wt == 0)
      for (int g = 0; g < 2 && g < G; g++) wg::bulk_prefetch_l2(tile_src(g), C2_TILE_PIX * NF1 * 4);
    for (int g = 0; g < G; g++) {
      const int s = g & 1;
      const float *rs = tile_src(g);
      uint8_t *pl = sPl + s * C2_STAGE;
      if (wt == 0 && g + 2 < G) wg::bulk_prefetch_l2(tile_src(g + 2), C2_TILE_PIX * NF1 * 4);
      wg::mbar_wait(&empty[s], ((g >> 1) & 1) ^ 1);
      // (pixel, plane) items: 336 x 3; plane 2 takes channels 16..19 of the pixel and of its right neighbour
#pragma unroll 2
      for (int i = wt; i < C2_TILE_PIX * 3; i += 128) {
        const int lp = i / 3, p = i - lp * 3;
        const float *src = rs + lp * NF1 + p * 8;
        const float4 x0 = __ldg(reinterpret_cast<const float4 *>(src));
        float4 x1 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p < 2) x1 = __ldg(reinterpret_cast<const float4 *>(src + 4));
        else if (lp + 1 < C2_TILE_PIX) x1 = __ldg(reinterpret_cast<const float4 *>(src + NF1));
        const float x[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
        __half hi[8], lo[8];
#pragma unroll
        for (int e = 0; e < 8; e++) {
          float a = x[e] * a_scale;
          hi[e] = __float2half_rn(a);
          lo[e] = __float2half_rn(a - __half2float(hi[e]));
        }
        *reinterpret_cast<uint4 *>(pl + (size_t)p * C2_PLANE + (size_t)lp * 16) = *reinterpret_cast<uint4 *>(hi);
        *reinterpret_cast<uint4 *>(pl + (size_t)(3 + p) * C2_PLANE + (size_t)lp * 16) = *reinterpret_cast<uint4 *>(lo);
      }
      wg::fence_async_smem();  // this thread's plane writes -> the tensor-core reads
      wg::mbar_arrive(&full[s]);
    }
    return;
  }

  // ===== consumers
  wg::setmaxnreg_inc<232>();
  const int c = wg_id - 1;
  const uint32_t bpl = wg::smem_u32(sPl) + (uint32_t)c * C2_STAGE, sA_u = wg::smem_u32(sA);
  float *st = stg + c * C2_STG_FLOATS;
  for (int g = c; g < G; g += 2) {
    const int im = (int)blockIdx.x + (g / C2_TILES) * (int)gridDim.x, T = g % C2_TILES;
    // this consumer's batch goes after the other's previous one; the barrier also orders the previous epilogue's stage
    // reads (all 128 threads) before this tile's stage writes
    if (g > 0) wg::bar_sync(1 + c, 256);
    wg::mbar_wait(&full[c], (g >> 1) & 1);
    float d[C2_N / 2];
    wg::fence();
#pragma unroll
    for (int i = 0; i < C2_NMMA; i++) {  // w_hi a_hi + w_lo a_hi + w_hi a_lo
      const uint32_t a0 = c2_off(2 * i), a1 = c2_off(2 * i + 1);
      const uint32_t lbo = (2 * i + 1 >= C2_NCH) ? 16u : (a1 - a0);
      const uint64_t whi = wg::desc(sA_u + (uint32_t)(2 * i) * C2_ACHUNK, C2_ACHUNK, 128);
      const uint64_t wlo = wg::desc(sA_u + (uint32_t)(2 * i) * C2_ACHUNK + 64 * 16, C2_ACHUNK, 128);
      const uint64_t ahi = wg::desc(bpl + a0, lbo, 128), alo = wg::desc(bpl + 3 * C2_PLANE + a0, lbo, 128);
      wg::mma_f16_n224(d, whi, ahi, i > 0);
      wg::mma_f16_n224(d, wlo, ahi, true);
      wg::mma_f16_n224(d, whi, alo, true);
    }
    wg::commit();
    if (g + 1 < G) wg::bar_arrive(2 - c, 256);  // the other consumer may issue its next batch
    wg::wait<0>();
    wg::reg_fence(d);
    if (lane == 0) wg::mbar_arrive(&empty[c]);
    // value 4 j + 2 h + e of this thread: filter 16 warp + lane / 4 + 8 h, column 8 j + 2 q + e, so the x-pair
    // (e = 0, 1) is in the thread: column pair cp = 4 j + q = 14 y + x / 2. Its y-partner cp + 14 = 4 (j + 3) + q + 2
    // (q < 2) or 4 (j + 4) + q - 2 (q >= 2) is in lane l ^ 2, which sends the pair the receiver needs.
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int ch = 16 * warp + (lane >> 2) + 8 * h;
#pragma unroll
      for (int j = 0; j < C2_N / 8; j++) {
        const int j3 = j + 3 < C2_N / 8 ? j + 3 : C2_N / 8 - 1, j4 = j + 4 < C2_N / 8 ? j + 4 : C2_N / 8 - 1;
        const float mine = fmaxf(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
        const float send = q >= 2 ? fmaxf(d[4 * j3 + 2 * h], d[4 * j3 + 2 * h + 1]) : fmaxf(d[4 * j4 + 2 * h], d[4 * j4 + 2 * h + 1]);
        const float v = fmaxf(mine, __shfl_xor_sync(0xffffffffu, send, 2)) * out_scale;
        const int cp = 4 * j + q, y = cp / 14, px = cp - 14 * y;
        if ((y & 1) == 0 && px < 12 && ch < NF2) st[((y >> 1) * 12 + px) * NF2 + ch] = v;
      }
    }
    wg::bar_sync(3 + c, 128);
    // the tile's 4 x 12 x 50 = 2400 consecutive k (from 2400 T) are 300 whole 8-element chunks of ip1's A operand:
    // [tile im/128][hi|lo][k/8][row im%128][k%8] fp16, scaled by x_scale
    __half *xrow = xc + (size_t)(im >> 7) * 2 * IP_KCH * 128 * 8 + (size_t)(im & 127) * 8;
    for (int ci = wt; ci < C2_STG_FLOATS / 8; ci += 128) {
      __half hi[8], lo[8];
#pragma unroll
      for (int e = 0; e < 8; e++) {
        const int kk = 8 * ci + e;
        float m = st[kk] + sbias[kk % NF2];
        if (relu) m = fmaxf(m, 0.0f);
        const float a = m * x_scale;
        hi[e] = __float2half_rn(a);
        lo[e] = __float2half_rn(a - __half2float(hi[e]));
      }
      __half *dst = xrow + (size_t)(C2_STG_FLOATS / 8 * T + ci) * 128 * 8;
      *reinterpret_cast<uint4 *>(dst) = *reinterpret_cast<uint4 *>(hi);
      *reinterpret_cast<uint4 *>(dst + (size_t)IP_KCH * 128 * 8) = *reinterpret_cast<uint4 *>(lo);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// ip1: H3[n x 500] = relu(X[n x 7200] W[7200 x 500] + b) as a TMA-fed wgmma GEMM.
// CTA tile: 128 images x 128 outputs; X arrives as fp16 hi/lo in the canonical K-major layout written by conv2's
// epilogue, W as a host-prepared fp16 hi/lo blob — both are plain contiguous byte ranges per K-block, so the
// operand ring is filled by 1-D bulk copies (no tensor map needed).
// D[:, 0:128] += x_hi w_hi + x_lo w_hi ; D[:, 128:256] += x_hi w_lo ; summed and rescaled in the epilogue.
// warps 0-7: two consumer warpgroups (images 0..63 | 64..127 of the tile, 128 accumulators per thread), warp 8: producer.
// ---------------------------------------------------------------------------------------------------------
constexpr int IP_KB_CH = 6, IP_NKB = IP_KCH / IP_KB_CH, IP_STAGES = 4;     // 48-element K-blocks, 150 of them
constexpr int IP_A_BYTES = IP_KB_CH * 128 * 16, IP_B_BYTES = IP_KB_CH * 256 * 16;
constexpr int IP_STAGE_BYTES = 2 * IP_A_BYTES + IP_B_BYTES;                 // 49152
constexpr int IP_NT = 288;

__global__ void __launch_bounds__(IP_NT, 1) k_ip1_tc(const __half *__restrict__ xc, int n, const uint8_t *__restrict__ wblob,
                                                     const float *__restrict__ bias, float out_scale, float *__restrict__ h3) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t full[IP_STAGES], empty[IP_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ob = blockIdx.x, mt = blockIdx.y;
  if (tid == 0) {
    for (int s = 0; s < IP_STAGES; s++) {
      wg::mbar_init(&full[s], 1);
      wg::mbar_init(&empty[s], 8);  // one arrival per consumer warp
    }
    wg::fence_mbar_init();
  }
  __syncthreads();
  if (warp == 8) {
    // ===== producer: one elected lane streams the K-blocks through the ring
    if (wg::elect_one()) {
      const uint8_t *xa_hi = reinterpret_cast<const uint8_t *>(xc) + (size_t)mt * 2 * IP_KCH * 128 * 16;
      const uint8_t *xa_lo = xa_hi + (size_t)IP_KCH * 128 * 16;
      const uint8_t *wb = wblob + (size_t)ob * IP_NKB * IP_B_BYTES;
      for (int kb = 0; kb < IP_NKB; kb++) {
        const int s = kb % IP_STAGES;
        wg::mbar_wait(&empty[s], ((kb / IP_STAGES) & 1) ^ 1);
        uint8_t *st = smem + (size_t)s * IP_STAGE_BYTES;
        wg::mbar_expect_tx(&full[s], IP_STAGE_BYTES);
        wg::bulk_g2s(st, xa_hi + (size_t)kb * IP_A_BYTES, IP_A_BYTES, &full[s]);
        wg::bulk_g2s(st + IP_A_BYTES, xa_lo + (size_t)kb * IP_A_BYTES, IP_A_BYTES, &full[s]);
        wg::bulk_g2s(st + 2 * IP_A_BYTES, wb + (size_t)kb * IP_B_BYTES, IP_B_BYTES, &full[s]);
      }
    }
    __syncwarp();
    return;
  }
  // ===== consumers
  const int wg_id = warp >> 2, q = lane & 3;
  const uint32_t sm_u = wg::smem_u32(smem), a_row = (uint32_t)wg_id * 64 * 16;
  float d[128];
#pragma unroll
  for (int i = 0; i < 128; i++) d[i] = 0.0f;
  for (int kb = 0; kb < IP_NKB; kb++) {
    const int s = kb % IP_STAGES;
    wg::mbar_wait(&full[s], (kb / IP_STAGES) & 1);
    const uint32_t st = sm_u + (uint32_t)s * IP_STAGE_BYTES;
    wg::fence();
#pragma unroll
    for (int ks = 0; ks < IP_KB_CH / 2; ks++) {
      const uint64_t da_hi = wg::desc(st + a_row + (uint32_t)(2 * ks) * 128 * 16, 128 * 16, 128);
      const uint64_t da_lo = wg::desc(st + IP_A_BYTES + a_row + (uint32_t)(2 * ks) * 128 * 16, 128 * 16, 128);
      const uint64_t db = wg::desc(st + 2 * IP_A_BYTES + (uint32_t)(2 * ks) * 256 * 16, 256 * 16, 128);
      wg::mma_f16_n256(d, da_hi, db, (kb | ks) != 0);  // x_hi x [w_hi | w_lo]
      wg::mma_f16_n128(d, da_lo, db, true);            // x_lo x w_hi
    }
    wg::commit();
    wg::wait<1>();  // the instructions of K-block kb - 1 have read their stage: it may be refilled
    if (kb > 0 && lane == 0) wg::mbar_arrive(&empty[(kb - 1) % IP_STAGES]);
  }
  wg::wait<0>();
  wg::reg_fence(d);
  // columns c and 128 + c are values i and i + 64 of the same thread
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int im = mt * 128 + wg_id * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (im >= n) continue;
#pragma unroll
    for (int j = 0; j < 16; j++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int i = 4 * j + 2 * h + e, o = ob * 128 + 8 * j + 2 * q + e;
        if (o < NH) h3[(size_t)im * NH + o] = fmaxf((d[i] + d[i + 64]) * out_scale + __ldg(bias + o), 0.0f);
      }
  }
}

}  // namespace

static float pow2_scale(float maxabs, float target) {
  if (!(maxabs > 0.0f)) return 1.0f;
  const float q = target / maxabs;
  if (std::isinf(q)) return std::ldexp(1.0f, 127);  // maxabs below ~5e-38: the largest float32 power of two, not inf
  return std::exp2(std::floor(std::log2(q)));
}

// Build the tensor-core weight blobs from the reference's .bin layout (conv OIHW row-major).
int lenet_tc_upload(gpdb_ctx *ctx, const float *const w[8]) {
  const int C = ctx->prm.image_num_channels;
  LenetTc &t = ctx->tc;
  t.npl = 1;
  t.nch1 = C1_NCH;
  // conv1 blob: [chunk c = kh*5+kw (26, last zero)][row n = c1_col(o, digit) (64)][16 x int8: channel e], then 20 float scales
  std::vector<int8_t> b1((size_t)C1_B_BYTES + NF1 * sizeof(float), 0);
  {
    float *scales = reinterpret_cast<float *>(b1.data() + C1_B_BYTES);
    for (int o = 0; o < NF1; o++) {
      float mxo = 0.0f;
      for (size_t i = 0; i < (size_t)C * 25; i++) mxo = std::fmax(mxo, std::fabs(w[0][(size_t)o * C * 25 + i]));
      // Below max|w_o| ~ 1e-36 the scale is a float32 subnormal (or 0) with a few bits: rounded down, it would put
      // |W| past the largest value the digits hold, 127 * 65536 + 127 * 257 (the top digit clamped, that weight wrong by
      // up to ~7 %). Step it up to the next float until max|w_o| / s_o fits; a normal scale never moves.
      float so = mxo > 0.0f ? (float)((double)mxo / 8300000.0) : 1.0f;
      while ((double)mxo / (double)so > C1_W_MAX) so = std::nextafter(so, INFINITY);
      scales[o] = so;
      t.c1_aff.scale[o] = so;
      t.c1_aff.bias[o] = w[1][o];
      for (int ch = 0; ch < C && ch < 16; ch++)
        for (int kh = 0; kh < 5; kh++)
          for (int kw = 0; kw < 5; kw++) {
            const double wv = w[0][(((size_t)o * C + ch) * 5 + kh) * 5 + kw];
            long W = std::lround(wv / (double)scales[o]);
            int dg[3];
            for (int k = 2; k >= 1; k--) {  // balanced base-256 digits, least significant first
              long d = ((W + 128) % 256 + 256) % 256 - 128;
              dg[k] = (int)d;
              W = (W - d) / 256;
            }
            dg[0] = (int)std::max(-128L, std::min(127L, W));
            const int c = kh * 5 + kw;
            for (int tm = 0; tm < 3; tm++) b1[((size_t)c * C1_N + c1_col(o, tm)) * 16 + ch] = (int8_t)dg[tm];
          }
    }
  }
  // conv2 blob (the A operand): [chunk c (66, last zero)][w_hi | w_lo][filter row 0..63 (50 used)][8 x fp16], weights
  // scaled by 2^k
  float mx = 0.0f;
  for (size_t i = 0; i < (size_t)NF2 * NF1 * 25; i++) mx = std::fmax(mx, std::fabs(w[2][i]));
  t.w2_scale = pow2_scale(mx, 16.0f);
  // Activation scales of the fp16 hi/lo split. The hi term must stay below the fp16 maximum (65504) for ANY input image:
  // bound the activations from the weights (pool1 <= max_o sum_i |w1[o,i]| * 255 + |b1[o]|, propagated through conv2 for
  // pool2), so that scores can never silently become inf / NaN. The scale is the LARGEST power of two that keeps
  // scale * bound <= 60000, in both directions: a fixed scale would push the lo term of small activations (a model with
  // small conv1 weights) into fp16 subnormals, an absolute error of ~2^-25 / scale that no longer shrinks with the
  // activations. Scaling conv1's weights and all biases by 2^k then scales every logit by exactly 2^k.
  double a1_bound = 0.0;
  for (int o = 0; o < NF1; o++) {
    double sabs = 0.0;
    for (size_t i = 0; i < (size_t)C * 25; i++) sabs += std::fabs((double)w[0][(size_t)o * C * 25 + i]);
    a1_bound = std::max(a1_bound, sabs * 255.0 + std::fabs((double)w[1][o]));
  }
  double a2_bound = 0.0;
  for (int o = 0; o < NF2; o++) {
    double sabs = 0.0;
    for (size_t i = 0; i < (size_t)NF1 * 25; i++) sabs += std::fabs((double)w[2][(size_t)o * NF1 * 25 + i]);
    a2_bound = std::max(a2_bound, sabs * a1_bound + std::fabs((double)w[3][o]));
  }
  // The epilogue multiplies by 1 / (scale * w_scale): 2^j is also held to |j + log2 w_scale| <= 120, which keeps that
  // factor a normal float (weights whose bound would need more are ~2^100 away from any trained net).
  auto safe_scale = [](double bound, float w_scale) {
    const int we = std::ilogb(w_scale), lo = std::max(-126, -120 - we), hi = std::min(127, 120 - we);
    if (!(bound > 0.0)) return std::ldexp(1.0f, std::max(lo, std::min(hi, 0)));  // all-zero layer: any scale is exact
    int j = (int)std::floor(std::log2(60000.0 / bound));
    while (j > lo && std::ldexp(1.0, j) * bound > 60000.0) j--;  // log2 rounding, either way
    while (j < hi && std::ldexp(1.0, j + 1) * bound <= 60000.0) j++;
    return std::ldexp(1.0f, std::max(lo, std::min(hi, j)));
  };
  t.a2_scale = safe_scale(a1_bound, t.w2_scale);
  std::vector<__half> b2((size_t)C2_A_BYTES / 2, __float2half(0.0f));
  for (int c = 0; c < C2_NCH; c++) {
    for (int o = 0; o < NF2; o++)
      for (int e = 0; e < 8; e++) {
        int ch, kh, kw;
        if (c < 50) {
          ch = (c / 25) * 8 + e, kh = (c / 5) % 5, kw = c % 5;
        } else {  // channels 16..19 of two neighbouring taps (c2_off)
          ch = 16 + (e & 3), kh = (c - 50) / 3, kw = 2 * ((c - 50) % 3) + (e >> 2);
          if (kw >= 5) continue;
        }
        float wv = w[2][(((size_t)o * NF1 + ch) * 5 + kh) * 5 + kw] * t.w2_scale;
        __half hi = __float2half_rn(wv);
        __half lo = __float2half_rn(wv - __half2float(hi));
        b2[((size_t)(2 * c) * 64 + o) * 8 + e] = hi;
        b2[((size_t)(2 * c + 1) * 64 + o) * 8 + e] = lo;
      }
  }
  // ip1 blob: [o-block 4][K-block 150][chunk 6][row 256: 0..127 w_hi(o), 128..255 w_lo(o)][8 x fp16], W(o,k) = w[4][o + 500 k]
  mx = 0.0f;
  for (size_t i = 0; i < (size_t)NH * IP_K; i++) mx = std::fmax(mx, std::fabs(w[4][i]));
  t.w3_scale = pow2_scale(mx, 16.0f);
  t.x3_scale = safe_scale(a2_bound, t.w3_scale);
  std::vector<__half> b3((size_t)4 * IP_NKB * IP_KB_CH * 256 * 8, __float2half(0.0f));
  for (int ob = 0; ob < 4; ob++)
    for (int kc = 0; kc < IP_KCH; kc++) {
      const int kb = kc / IP_KB_CH, c = kc % IP_KB_CH;
      __half *dst = b3.data() + (((size_t)ob * IP_NKB + kb) * IP_KB_CH + c) * 256 * 8;
      for (int ol = 0; ol < 128; ol++) {
        const int o = ob * 128 + ol;
        if (o >= NH) continue;
        for (int e = 0; e < 8; e++) {
          float wv = w[4][(size_t)o + (size_t)NH * (kc * 8 + e)] * t.w3_scale;
          __half hi = __float2half_rn(wv);
          __half lo = __float2half_rn(wv - __half2float(hi));
          dst[(size_t)ol * 8 + e] = hi;
          dst[(size_t)(128 + ol) * 8 + e] = lo;
        }
      }
    }
  cudaFree(t.b1);
  cudaFree(t.b2);
  cudaFree(t.b3);
  t.b1 = t.b2 = t.b3 = nullptr;
  t.ready = false;
  if (cudaMalloc(&t.b1, b1.size()) != cudaSuccess || cudaMalloc(&t.b2, b2.size() * 2) != cudaSuccess ||
      cudaMemcpy(t.b1, b1.data(), b1.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(t.b2, b2.data(), b2.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMalloc(&t.b3, b3.size() * 2) != cudaSuccess ||
      cudaMemcpy(t.b3, b3.data(), b3.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "tensor-core weight upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    return GPDB_ERR_CUDA;
  }
  t.ready = ctx->prm.image_size == 60 && C <= 16;
  return GPDB_OK;
}

// conv1 + pool, conv2 + pool and ip1 + ReLU on wgmma; p1 [n][784][20] f32, xc = fp16 hi/lo ip1 operand, h3 [n][500]
int lenet_tc_forward(gpdb_ctx *ctx, const uint8_t *d_images, int n, float *p1, __half *xc, float *h3) {
  const LenetTc &t = ctx->tc;
  const int relu = ctx->prm.relu_after_conv;
  size_t sm1 = (size_t)C1_B_BYTES + C1_PLANE + 2 * C1_STAGE_FLOATS * sizeof(float);
  size_t sm2 = (size_t)C2_SMEM;
  size_t sm3 = (size_t)IP_STAGES * IP_STAGE_BYTES;
  CUDA_TRY(cudaFuncSetAttribute(k_conv1_i8, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
  CUDA_TRY(cudaFuncSetAttribute(k_conv2_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
  CUDA_TRY(cudaFuncSetAttribute(k_ip1_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm3));
  cudaEvent_t e1 = gpdb_st_begin(ctx);
  k_conv1_i8<<<std::min(n, C1_CTAS_PER_SM * ctx->sm_count), C1_NT, sm1, ctx->stream>>>(d_images, n, (const uint8_t *)t.b1, t.c1_aff, relu, p1);
  LAUNCH_CHECK();
  gpdb_st_end(ctx, 5, e1);
  cudaEvent_t e2 = gpdb_st_begin(ctx);
  k_conv2_tc<<<std::min(n, ctx->sm_count), C2_NT, sm2, ctx->stream>>>(p1, n, (const uint8_t *)t.b2, ctx->w.c2b, t.a2_scale,
                                                                       1.0f / (t.a2_scale * t.w2_scale), relu, xc, t.x3_scale);
  LAUNCH_CHECK();
  gpdb_st_end(ctx, 6, e2);
  cudaEvent_t e3 = gpdb_st_begin(ctx);
  dim3 g3(4, (n + 127) / 128);  // the four output blocks of an image tile run together and share its X through L2
  k_ip1_tc<<<g3, IP_NT, sm3, ctx->stream>>>(xc, n, (const uint8_t *)t.b3, ctx->w.i1b, 1.0f / (t.x3_scale * t.w3_scale), h3);
  LAUNCH_CHECK();
  gpdb_st_end(ctx, 7, e3);
  return GPDB_OK;
}

size_t lenet_tc_xc_bytes(int n) { return (size_t)((n + 127) / 128) * 2 * IP_KCH * 128 * 16; }

// p1 [n][784 px][20] -> [n][20][784]; xc [im/128][hi|lo][k/8][im%128][8] fp16 (scaled by x3_scale) -> (hi + lo) / x3_scale
// [n][7200] in float64: exactly the operand ip1 multiplies
int lenet_tc_read_layers(gpdb_ctx *ctx, int n, const float *p1, const __half *xc, const LenetLayers &out) {
  if (out.pool1) {
    std::vector<float> t((size_t)n * 784 * NF1);
    CUDA_TRY(cudaMemcpy(t.data(), p1, sizeof(float) * t.size(), cudaMemcpyDeviceToHost));
    for (size_t im = 0; im < (size_t)n; im++)
      for (int px = 0; px < 784; px++)
        for (int c = 0; c < NF1; c++) out.pool1[(im * NF1 + c) * 784 + px] = t[(im * 784 + px) * NF1 + c];
  }
  if (out.pool2) {
    std::vector<__half> t(lenet_tc_xc_bytes(n) / sizeof(__half));
    CUDA_TRY(cudaMemcpy(t.data(), xc, lenet_tc_xc_bytes(n), cudaMemcpyDeviceToHost));
    const double inv = 1.0 / (double)ctx->tc.x3_scale;  // a power of two: exact
    for (size_t im = 0; im < (size_t)n; im++)
      for (int k = 0; k < IP_K; k++) {
        const size_t hi = (((im >> 7) * 2 * IP_KCH + (size_t)(k >> 3)) * 128 + (im & 127)) * 8 + (k & 7);
        const size_t lo = hi + (size_t)IP_KCH * 128 * 8;
        out.pool2[im * IP_K + k] = ((double)__half2float(t[hi]) + (double)__half2float(t[lo])) * inv;
      }
  }
  return GPDB_OK;
}
