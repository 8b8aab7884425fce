// lenet_simt.cu — LeNet forward (A14) on CUDA cores in float32: the first, plainly-correct device
// path of net::Classifier::classifyImages (eigen_classifier.cpp:59-128, conv_layer.cpp:26-56,
// dense_layer.cpp:6-15). The wgmma implicit-GEMM path (lenet_tc.cu) is validated against this one.
//
//   conv1 (C->20, k5) + 2x2 max-pool : one image per CTA iteration, uint8 image staged CHW in shared
//          memory, weights [c][kh][kw][o] in shared memory, each thread owns a pooled pixel x 10 filters
//   conv2 (20->50, k5) + pool        : same shape of kernel, 100 KB of weights resident per CTA
//   ip1 (7200->500) + ReLU           : tiled SGEMM over the batch
//   ip2 (500->2), score = y1 - y0    : one warp per image
// Input: the images in the library's P16 layout (one 16-byte group per pixel: the cv::Mat HWC bytes of the pixel, zero
// padded — written by k_images, or converted from the caller's cv::Mat data by gpdb_classify), raw 0..255 values, no
// scaling (imageToArray, eigen_classifier.cpp:130-149).
#include <cuda_fp16.h>

#include <vector>

#include "common.cuh"

namespace {

constexpr int NF1 = 20, NF2 = 50, NH = 500;

// ---- conv1 + pool --------------------------------------------------------------------------------
// grid: persistent over images; block 224 threads; dyn smem: float w[C*25*20] | uint8 img[C*S*S]
__global__ void __launch_bounds__(224) k_conv1_pool(const uint8_t *__restrict__ images, int n, int S, int C,
                                                    const float *__restrict__ w_t /* [c][kh][kw][20] */,
                                                    const float *__restrict__ bias, int relu,
                                                    float *__restrict__ p1 /* [n][20][P][P] */) {
  extern __shared__ __align__(16) unsigned char dyn[];
  float *sw = reinterpret_cast<float *>(dyn);
  uint8_t *simg = reinterpret_cast<uint8_t *>(sw + C * 25 * NF1);
  const int O = S - 4, Pp = O / 2;
  for (int k = threadIdx.x; k < C * 25 * NF1; k += blockDim.x) sw[k] = w_t[k];
  for (int im = blockIdx.x; im < n; im += gridDim.x) {
    __syncthreads();
    const uint8_t *g = images + (size_t)im * S * S * 16;
    // P16 (16-byte pixels, channels 0..C-1) -> CHW bytes
    for (int k = threadIdx.x; k < S * S * C; k += blockDim.x) {
      int pix = k / C, c = k - pix * C;
      simg[c * S * S + pix] = g[pix * 16 + c];
    }
    __syncthreads();
    const int items = 2 * Pp * Pp;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
      const int ob = it / (Pp * Pp), pp = it - ob * Pp * Pp;
      const int py = pp / Pp, px = pp - py * Pp;
      float acc[4][10];
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int o = 0; o < 10; o++) acc[a][o] = 0.0f;
      for (int c = 0; c < C; c++) {
        float win[6][6];
        const uint8_t *ip = simg + c * S * S + (2 * py) * S + 2 * px;
#pragma unroll
        for (int r = 0; r < 6; r++)
#pragma unroll
          for (int q = 0; q < 6; q++) win[r][q] = (float)ip[r * S + q];
        const float *wp = sw + (c * 25) * NF1 + ob * 10;
#pragma unroll
        for (int kh = 0; kh < 5; kh++)
#pragma unroll
          for (int kw = 0; kw < 5; kw++) {
            float wv[10];
            const float2 *w2 = reinterpret_cast<const float2 *>(wp + (kh * 5 + kw) * NF1);
#pragma unroll
            for (int o = 0; o < 5; o++) {
              float2 t = w2[o];
              wv[2 * o] = t.x;
              wv[2 * o + 1] = t.y;
            }
#pragma unroll
            for (int o = 0; o < 10; o++) {
              acc[0][o] = fmaf(wv[o], win[kh][kw], acc[0][o]);
              acc[1][o] = fmaf(wv[o], win[kh][kw + 1], acc[1][o]);
              acc[2][o] = fmaf(wv[o], win[kh + 1][kw], acc[2][o]);
              acc[3][o] = fmaf(wv[o], win[kh + 1][kw + 1], acc[3][o]);
            }
          }
      }
#pragma unroll
      for (int o = 0; o < 10; o++) {
        float m = fmaxf(fmaxf(acc[0][o], acc[1][o]), fmaxf(acc[2][o], acc[3][o])) + bias[ob * 10 + o];
        if (relu) m = fmaxf(m, 0.0f);
        p1[(((size_t)im * NF1 + ob * 10 + o) * Pp + py) * Pp + px] = m;
      }
    }
  }
}

// ---- conv2 + pool --------------------------------------------------------------------------------
// block 240 threads; dyn smem: float w[20*25*50] | float in[20*P1*P1]
__global__ void __launch_bounds__(240) k_conv2_pool(const float *__restrict__ p1, int n, int P1,
                                                    const float *__restrict__ w_t /* [c][kh][kw][50] */,
                                                    const float *__restrict__ bias, int relu,
                                                    float *__restrict__ p2 /* [n][j][50], k = c + 50 j */) {
  extern __shared__ __align__(16) unsigned char dyn[];
  float *sw = reinterpret_cast<float *>(dyn);
  float *sin = sw + NF1 * 25 * NF2;
  const int O = P1 - 4, Pp = O / 2;
  for (int k = threadIdx.x; k < NF1 * 25 * NF2; k += blockDim.x) sw[k] = w_t[k];
  for (int im = blockIdx.x; im < n; im += gridDim.x) {
    __syncthreads();
    const float *g = p1 + (size_t)im * NF1 * P1 * P1;
    for (int k = threadIdx.x; k < NF1 * P1 * P1; k += blockDim.x) sin[k] = g[k];
    __syncthreads();
    const int items = 5 * Pp * Pp;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
      const int ob = it / (Pp * Pp), pp = it - ob * Pp * Pp;
      const int py = pp / Pp, px = pp - py * Pp;
      float acc[4][10];
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int o = 0; o < 10; o++) acc[a][o] = 0.0f;
      for (int c = 0; c < NF1; c++) {
        float win[6][6];
        const float *ip = sin + c * P1 * P1 + (2 * py) * P1 + 2 * px;
#pragma unroll
        for (int r = 0; r < 6; r++)
#pragma unroll
          for (int q = 0; q < 6; q += 2) {
            float2 t = *reinterpret_cast<const float2 *>(ip + r * P1 + q);
            win[r][q] = t.x;
            win[r][q + 1] = t.y;
          }
        const float *wp = sw + (c * 25) * NF2 + ob * 10;
#pragma unroll
        for (int kh = 0; kh < 5; kh++)
#pragma unroll
          for (int kw = 0; kw < 5; kw++) {
            float wv[10];
            const float2 *w2 = reinterpret_cast<const float2 *>(wp + (kh * 5 + kw) * NF2);
#pragma unroll
            for (int o = 0; o < 5; o++) {
              float2 t = w2[o];
              wv[2 * o] = t.x;
              wv[2 * o + 1] = t.y;
            }
#pragma unroll
            for (int o = 0; o < 10; o++) {
              acc[0][o] = fmaf(wv[o], win[kh][kw], acc[0][o]);
              acc[1][o] = fmaf(wv[o], win[kh][kw + 1], acc[1][o]);
              acc[2][o] = fmaf(wv[o], win[kh + 1][kw], acc[2][o]);
              acc[3][o] = fmaf(wv[o], win[kh + 1][kw + 1], acc[3][o]);
            }
          }
      }
      const int j = py * Pp + px;
#pragma unroll
      for (int o = 0; o < 10; o++) {
        float m = fmaxf(fmaxf(acc[0][o], acc[1][o]), fmaxf(acc[2][o], acc[3][o])) + bias[ob * 10 + o];
        if (relu) m = fmaxf(m, 0.0f);
        p2[(size_t)im * (NF2 * Pp * Pp) + (size_t)j * NF2 + ob * 10 + o] = m;
      }
    }
  }
}

// ---- ip1: H3[n x 500] = relu(X[n x K] W[K x 500] + b) ; tile 64 x 64, 256 threads, 4x4 per thread -----
__global__ void __launch_bounds__(256) k_ip1(const float *__restrict__ X, int n, int K, const float *__restrict__ W,
                                             const float *__restrict__ bias, float *__restrict__ H) {
  __shared__ float Xs[16][64 + 4];
  __shared__ float Ws[16][64 + 4];
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    {
      // X tile: 64 rows x 16 k  (thread: row = tid/4, kq = (tid%4)*4)
      int r = threadIdx.x >> 2, kq = (threadIdx.x & 3) * 4;
      float4 v = make_float4(0, 0, 0, 0);
      if (m0 + r < n) v = *reinterpret_cast<const float4 *>(X + (size_t)(m0 + r) * K + k0 + kq);
      Xs[kq][r] = v.x; Xs[kq + 1][r] = v.y; Xs[kq + 2][r] = v.z; Xs[kq + 3][r] = v.w;
      // W tile: 16 k x 64 cols (thread: k = tid/16, cq = (tid%16)*4)
      int kk = threadIdx.x >> 4, cq = (threadIdx.x & 15) * 4;
      float4 w = make_float4(0, 0, 0, 0);
      if (n0 + cq + 3 < NH) w = *reinterpret_cast<const float4 *>(W + (size_t)(k0 + kk) * NH + n0 + cq);
      else {
        float t[4] = {0, 0, 0, 0};
        for (int e = 0; e < 4; e++) if (n0 + cq + e < NH) t[e] = W[(size_t)(k0 + kk) * NH + n0 + cq + e];
        w = make_float4(t[0], t[1], t[2], t[3]);
      }
      *reinterpret_cast<float4 *>(&Ws[kk][cq]) = w;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; kk++) {
      float4 a = *reinterpret_cast<const float4 *>(&Xs[kk][ty * 4]);
      float4 b = *reinterpret_cast<const float4 *>(&Ws[kk][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    int r = m0 + ty * 4 + i;
    if (r >= n) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int c = n0 + tx * 4 + j;
      if (c < NH) H[(size_t)r * NH + c] = fmaxf(acc[i][j] + bias[c], 0.0f);
    }
  }
}

// ---- ip2 + score: one warp per image ----------------------------------------------------------------
__global__ void k_ip2(const float *__restrict__ H, int n, const float *__restrict__ W /* [k][2] */,
                      const float *__restrict__ bias, float *__restrict__ scores, float *__restrict__ logits) {
  int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n) return;
  float y0 = 0.0f, y1 = 0.0f;
  for (int k = lane; k < NH; k += 32) {
    float h = H[(size_t)i * NH + k];
    y0 = fmaf(W[2 * k], h, y0);
    y1 = fmaf(W[2 * k + 1], h, y1);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    y0 += __shfl_xor_sync(0xffffffffu, y0, o);
    y1 += __shfl_xor_sync(0xffffffffu, y1, o);
  }
  if (lane == 0) {
    y0 += bias[0];
    y1 += bias[1];
    scores[i] = y1 - y0;  // eigen_classifier.cpp:74
    if (logits) {
      logits[2 * (size_t)i] = y0;
      logits[2 * (size_t)i + 1] = y1;
    }
  }
}

}  // namespace

// Upload the reference's .bin layout (conv OIHW row-major, ip column-major (out,in)) and re-lay the conv
// filters as [c][kh][kw][o] for the kernels above. ip1/ip2 are used as stored: W(o,k) at o + OUT*k.
int lenet_upload(gpdb_ctx *ctx, const float *const w[8]) {
  const int C = ctx->prm.image_num_channels;
  LenetWeights &d = ctx->w;
  const size_t n1 = (size_t)NF1 * C * 25, n2 = (size_t)NF2 * NF1 * 25, n3 = (size_t)NH * 7200, n4 = 2 * NH;
  float *t1 = (float *)malloc(sizeof(float) * n1), *t2 = (float *)malloc(sizeof(float) * n2);
  for (int o = 0; o < NF1; o++)
    for (int c = 0; c < C; c++)
      for (int k = 0; k < 25; k++) t1[((size_t)c * 25 + k) * NF1 + o] = w[0][((size_t)o * C + c) * 25 + k];
  for (int o = 0; o < NF2; o++)
    for (int c = 0; c < NF1; c++)
      for (int k = 0; k < 25; k++) t2[((size_t)c * 25 + k) * NF2 + o] = w[2][((size_t)o * NF1 + c) * 25 + k];
  float **slots[8] = {&d.c1w, &d.c1b, &d.c2w, &d.c2b, &d.i1w, &d.i1b, &d.i2w, &d.i2b};
  const size_t sizes[8] = {n1, (size_t)NF1, n2, (size_t)NF2, n3, (size_t)NH, n4, 2};
  const float *src[8] = {t1, w[1], t2, w[3], w[4], w[5], w[6], w[7]};
  int rc = GPDB_OK;
  for (int i = 0; i < 8 && rc == GPDB_OK; i++) {
    cudaFree(*slots[i]);
    *slots[i] = nullptr;
    if (cudaMalloc(slots[i], sizeof(float) * sizes[i]) != cudaSuccess ||
        cudaMemcpy(*slots[i], src[i], sizeof(float) * sizes[i], cudaMemcpyHostToDevice) != cudaSuccess) {
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "weight upload failed: %s", cudaGetErrorString(cudaGetLastError()));
      rc = GPDB_ERR_CUDA;
    }
  }
  free(t1);
  free(t2);
  d.C = C;
  d.set = (rc == GPDB_OK);
  if (rc == GPDB_OK) rc = lenet_tc_upload(ctx, w);
  return rc;
}

// Copies the layer outputs of the forward pass that just ran (p2: the tensor-core xc operand or SIMT float32 [n][7200]).
static int read_layers(gpdb_ctx *ctx, int n, bool use_tc, const float *p1, const void *p2, const float *h3,
                       const LenetLayers &out) {
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (use_tc) {
    int rc = lenet_tc_read_layers(ctx, n, p1, reinterpret_cast<const __half *>(p2), out);
    if (rc != GPDB_OK) return rc;
  } else {
    const size_t np1 = (size_t)n * NF1 * 28 * 28, np2 = (size_t)n * 7200;
    if (out.pool1) CUDA_TRY(cudaMemcpy(out.pool1, p1, sizeof(float) * np1, cudaMemcpyDeviceToHost));
    if (out.pool2) {
      std::vector<float> t(np2);
      CUDA_TRY(cudaMemcpy(t.data(), p2, sizeof(float) * np2, cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < np2; i++) out.pool2[i] = t[i];
    }
  }
  if (out.ip1) CUDA_TRY(cudaMemcpy(out.ip1, h3, sizeof(float) * (size_t)n * NH, cudaMemcpyDeviceToHost));
  return GPDB_OK;
}

int lenet_simt_run(gpdb_ctx *ctx, const LenetWeights &w, const uint8_t *d_images, int n, float *p1, float *p2, float *h3,
                   float *d_scores, float *d_logits) {
  const int S = ctx->prm.image_size, C = ctx->prm.image_num_channels;
  const int P1 = (S - 4) / 2, P2 = (P1 - 4) / 2, K = NF2 * P2 * P2;
  const int relu = ctx->prm.relu_after_conv;
  size_t sm1 = sizeof(float) * C * 25 * NF1 + (size_t)C * S * S;
  size_t sm2 = sizeof(float) * (NF1 * 25 * NF2 + NF1 * P1 * P1);
  CUDA_TRY(cudaFuncSetAttribute(k_conv1_pool, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
  CUDA_TRY(cudaFuncSetAttribute(k_conv2_pool, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
  cudaEvent_t e1 = gpdb_st_begin(ctx);
  k_conv1_pool<<<std::min(n, ctx->sm_count * 2), 224, sm1, ctx->stream>>>(d_images, n, S, C, w.c1w, w.c1b, relu, p1);
  LAUNCH_CHECK();
  gpdb_st_end(ctx, 5, e1);
  cudaEvent_t e2 = gpdb_st_begin(ctx);
  k_conv2_pool<<<std::min(n, ctx->sm_count), 240, sm2, ctx->stream>>>(p1, n, P1, w.c2w, w.c2b, relu, p2);
  LAUNCH_CHECK();
  gpdb_st_end(ctx, 6, e2);
  cudaEvent_t e3 = gpdb_st_begin(ctx);
  dim3 g3((n + 63) / 64, (NH + 63) / 64);
  k_ip1<<<g3, 256, 0, ctx->stream>>>(p2, n, K, w.i1w, w.i1b, h3);
  LAUNCH_CHECK();
  k_ip2<<<(n * 32 + 255) / 256, 256, 0, ctx->stream>>>(h3, n, w.i2w, w.i2b, d_scores, d_logits);
  LAUNCH_CHECK();
  gpdb_st_end(ctx, 7, e3);
  return GPDB_OK;
}

int lenet_forward(gpdb_ctx *ctx, const uint8_t *d_images, int n, float *d_scores, float *d_logits,
                  const LenetLayers *layers) {
  if (n <= 0) return GPDB_OK;
  const int S = ctx->prm.image_size;
  const int P1 = (S - 4) / 2, P2 = (P1 - 4) / 2, K = NF2 * P2 * P2;
  if (S != 60) {  // 61..63 would also give ip1 7200 inputs, but the reference's network is built for 60 x 60
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "LeNet expects image_size 60 (ip1 input 7200), got %d (ip1 input %d)", S, K);
    return GPDB_ERR_INVALID;
  }
  const LenetWeights &w = ctx->w;
  const bool use_tc = ctx->tc.ready && ctx->prm.lenet_impl != 1;
  float *p1 = (float *)gpdb_scratch(ctx, SCR_WORK_A, sizeof(float) * (size_t)n * NF1 * P1 * P1);
  float *p2 = (float *)gpdb_scratch(ctx, SCR_WORK_B, use_tc ? lenet_tc_xc_bytes(n) : sizeof(float) * (size_t)n * K);
  float *h3 = (float *)gpdb_scratch(ctx, SCR_WORK_C, sizeof(float) * (size_t)n * NH);
  if (!p1 || !p2 || !h3) return GPDB_ERR_CUDA;
  if (use_tc) {
    int rc = lenet_tc_forward(ctx, d_images, n, p1, reinterpret_cast<__half *>(p2), h3);
    if (rc != GPDB_OK) return rc;
    cudaEvent_t e4 = gpdb_st_begin(ctx);
    k_ip2<<<(n * 32 + 255) / 256, 256, 0, ctx->stream>>>(h3, n, w.i2w, w.i2b, d_scores, d_logits);
    LAUNCH_CHECK();
    gpdb_st_end(ctx, 7, e4);
    return layers ? read_layers(ctx, n, true, p1, p2, h3, *layers) : GPDB_OK;
  }
  const int rc = lenet_simt_run(ctx, w, d_images, n, p1, p2, h3, d_scores, d_logits);
  if (rc != GPDB_OK) return rc;
  return layers ? read_layers(ctx, n, false, p1, p2, h3, *layers) : GPDB_OK;
}
