// train.cu — LeNet training on the CUDA cores in float32 (include/gpd_b200_train.h states every rule).
//
// A step of n images runs in chunks of at most GPDB_TRAIN_CHUNK images. Per chunk:
//   forward      geo_hwc_to_p16 + lenet_simt_run: the inference kernels themselves, with the trained weights re-laid
//   k_choice1/2  the pooling choice of every pooled value: the forward's FMA chains again, first maximum of fl(acc + b)
//   k_loss       per-image loss and d logits; k_loss_sum chains the losses in image order
//   k_gemm       ip2 / ip1 weight gradients (chained over the images) and d pool2; k_colsum the bias gradients
//   k_dh         d ip1 through ip2 and the ReLU
//   k_dconv2     d pool2 through the pool (and ReLU) into the dense d conv2
//   k_conv2_wgrad / k_conv1_wgrad  per-image weight and bias gradients over the pooled positions; k_colsum chains them
//   k_dpool1     d pool1 from d conv2 (one fixed order over filter, kh, kw)
// then one element-wise optimiser kernel over the eight parameter arrays. No atomics on floats anywhere: every sum has
// one order, so identical call sequences give identical weights. The entry points gpdb_train_begin,
// gpdb_train_step[_device], gpdb_debug_train_step and gpdb_train_weights, with their checks, follow the kernels.
#include <algorithm>
#include <cmath>

#include "../../include/gpd_b200_train.h"
#include "common.cuh"

namespace {

constexpr int NF1 = 20, NF2 = 50, NH = 500, S = 60, P1 = 28, O2 = 24, P2 = 12, K = 7200;
constexpr int NW2 = NF2 * NF1 * 25 + NF2;  // conv2 weights + biases: one gradient partial per image

}  // namespace

// The training state of a context: the eight parameter arrays (.bin layouts) at off[0..7], each of len[i] values and
// starting on a 16-byte boundary (k_ip1 reads ip1's weights as float4; every weight array holds a multiple of 4 values,
// so each bias still follows its weights directly); the same layout for the optimiser's buffers and the running
// gradient, and the conv filters re-laid for the forward kernels. The padding between arrays stays zero in the weights
// and the gradient and is never read.
struct TrainState {
  float *w, *m, *v, *g;  // weights; SGD momentum buffer / Adam first moment; Adam second moment; gradient of the step
  float *c1t, *c2t;      // conv filters as [c][kh][kw][o] (lenet_upload's layout), rebuilt before every forward
  float *loss;           // [0] the running loss sum of a step, [1] its mean
  size_t off[9], len[8];
  int C;
  gpdb_train_params p;
  long long t;  // optimiser steps taken since gpdb_train_begin
};

namespace {

// .bin conv filters -> [c][kh][kw][o] (dir 0), or back (dir 1)
__global__ void k_relayout(float *w1, float *w2, int C, float *t1, float *t2, int dir) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int n1 = NF1 * C * 25;
  if (e < n1) {
    const int o = e / (C * 25), c = (e / 25) % C, k = e % 25;
    float *a = w1 + e, *b = t1 + (c * 25 + k) * NF1 + o;
    if (dir) *a = *b; else *b = *a;
  } else if (e < n1 + NF2 * NF1 * 25) {
    const int f = e - n1, o = f / (NF1 * 25), c = (f / 25) % NF1, k = f % 25;
    float *a = w2 + f, *b = t2 + (c * 25 + k) * NF2 + o;
    if (dir) *a = *b; else *b = *a;
  }
}

// rule 2: the first maximum, in row-major window order, of fl(acc_a + b)
__device__ __forceinline__ uint8_t first_max(const float (&acc)[4], float b) {
  float best = acc[0] + b;
  int a = 0;
#pragma unroll
  for (int q = 1; q < 4; q++) {
    const float v = acc[q] + b;
    if (v > best) best = v, a = q;
  }
  return (uint8_t)a;
}

// conv1 pooling choices, one CTA per image: the image staged CHW in shared memory as k_conv1_pool does, each thread a
// pooled pixel of one filter, the four FMA chains in k_conv1_pool's order (c, kh, kw).
__global__ void __launch_bounds__(256) k_choice1(const uint8_t *__restrict__ hwc, int C, const float *__restrict__ w,
                                                 const float *__restrict__ b, uint8_t *__restrict__ ch /* [n][20][784] */) {
  extern __shared__ __align__(16) unsigned char dyn[];
  float *sw = reinterpret_cast<float *>(dyn);
  uint8_t *simg = reinterpret_cast<uint8_t *>(sw + NF1 * C * 25);
  const int im = blockIdx.x;
  for (int k = threadIdx.x; k < NF1 * C * 25; k += blockDim.x) sw[k] = w[k];
  const uint8_t *g = hwc + (size_t)im * S * S * C;
  for (int k = threadIdx.x; k < S * S * C; k += blockDim.x) {
    const int pix = k / C, c = k - pix * C;
    simg[c * S * S + pix] = g[k];
  }
  __syncthreads();
  for (int it = threadIdx.x; it < NF1 * P1 * P1; it += blockDim.x) {
    const int o = it / (P1 * P1), pp = it % (P1 * P1), py = pp / P1, px = pp % P1;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int c = 0; c < C; c++) {
      const uint8_t *ip = simg + c * S * S + (2 * py) * S + 2 * px;
      const float *wp = sw + (o * C + c) * 25;
#pragma unroll
      for (int kh = 0; kh < 5; kh++)
#pragma unroll
        for (int kw = 0; kw < 5; kw++) {
          const float wv = wp[kh * 5 + kw];
          acc[0] = fmaf(wv, (float)ip[kh * S + kw], acc[0]);
          acc[1] = fmaf(wv, (float)ip[kh * S + kw + 1], acc[1]);
          acc[2] = fmaf(wv, (float)ip[(kh + 1) * S + kw], acc[2]);
          acc[3] = fmaf(wv, (float)ip[(kh + 1) * S + kw + 1], acc[3]);
        }
    }
    ch[(size_t)im * NF1 * P1 * P1 + it] = first_max(acc, b[o]);
  }
}

// conv2 pooling choices, one CTA per image, pool1 and the .bin conv2 filters in shared memory; out in the k = c + 50 j
// order of pool2
__global__ void __launch_bounds__(256) k_choice2(const float *__restrict__ p1, const float *__restrict__ w,
                                                 const float *__restrict__ b, uint8_t *__restrict__ ch /* [n][7200] */) {
  extern __shared__ __align__(16) unsigned char dyn[];
  float *sw = reinterpret_cast<float *>(dyn);
  float *sin = sw + NF2 * NF1 * 25;
  const int im = blockIdx.x;
  for (int k = threadIdx.x; k < NF2 * NF1 * 25; k += blockDim.x) sw[k] = w[k];
  for (int k = threadIdx.x; k < NF1 * P1 * P1; k += blockDim.x) sin[k] = p1[(size_t)im * NF1 * P1 * P1 + k];
  __syncthreads();
  for (int it = threadIdx.x; it < K; it += blockDim.x) {
    const int o = it / (P2 * P2), j = it % (P2 * P2), py = j / P2, px = j % P2;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int c = 0; c < NF1; c++) {
      const float *ip = sin + c * P1 * P1 + (2 * py) * P1 + 2 * px;
      const float *wp = sw + (o * NF1 + c) * 25;
#pragma unroll
      for (int kh = 0; kh < 5; kh++)
#pragma unroll
        for (int kw = 0; kw < 5; kw++) {
          const float wv = wp[kh * 5 + kw];
          acc[0] = fmaf(wv, ip[kh * P1 + kw], acc[0]);
          acc[1] = fmaf(wv, ip[kh * P1 + kw + 1], acc[1]);
          acc[2] = fmaf(wv, ip[(kh + 1) * P1 + kw], acc[2]);
          acc[3] = fmaf(wv, ip[(kh + 1) * P1 + kw + 1], acc[3]);
        }
    }
    ch[(size_t)im * K + j * NF2 + o] = first_max(acc, b[o]);
  }
}

// rules 3 and 4, one thread per image; n_step is the whole step's image count
__global__ void k_loss(const float *__restrict__ logits, const int32_t *__restrict__ labels, int nb, float n_step,
                       float *__restrict__ loss, float *__restrict__ dz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb) return;
  const float z0 = logits[2 * i], z1 = logits[2 * i + 1];
  loss[i] = gpdb_train_loss(z0, z1, labels[i]);
  gpdb_train_dlogits(z0, z1, labels[i], n_step, dz + 2 * i);
}

// the step's loss: one chain over the images in order, continued from the previous chunk; the last chunk divides by n
__global__ void k_loss_sum(const float *__restrict__ loss, int nb, int first, int last, float n_step, float *acc,
                           float *out) {
  float s = first ? 0.0f : acc[0];
  for (int i = 0; i < nb; i++) s += loss[i];
  acc[0] = s;
  if (last) {
    acc[1] = s / n_step;
    if (out) *out = acc[1];
  }
}

// C[m][c] = (acc ? C[m][c] : 0) + sum_{r = 0..R-1} A(m, r) B(r, c), one FMA per term in r order, with A(m, r) =
// A[m am + r ar] and B(r, c) = B[r br + c bc]. Tiles of 64 x 64 outputs, 256 threads of 4 x 4, 16 r per stage.
__global__ void __launch_bounds__(256) k_gemm(const float *__restrict__ A, long am, long ar, const float *__restrict__ B,
                                              long br, long bc, float *__restrict__ Cm, int ldc, int M, int N, int R,
                                              int acc_in) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int m = m0 + ty * 4 + i, c = n0 + tx * 4 + j;
      acc[i][j] = (acc_in && m < M && c < N) ? Cm[(size_t)m * ldc + c] : 0.0f;
    }
  for (int r0 = 0; r0 < R; r0 += 16) {
    for (int e = threadIdx.x; e < 1024; e += 256) {
      int mm, rr;
      if (am == 1) mm = e & 63, rr = e >> 6; else rr = e & 15, mm = e >> 4;
      As[rr][mm] = (m0 + mm < M && r0 + rr < R) ? A[(size_t)(m0 + mm) * am + (size_t)(r0 + rr) * ar] : 0.0f;
      int cc;
      if (bc == 1) cc = e & 63, rr = e >> 6; else rr = e & 15, cc = e >> 4;
      Bs[rr][cc] = (n0 + cc < N && r0 + rr < R) ? B[(size_t)(r0 + rr) * br + (size_t)(n0 + cc) * bc] : 0.0f;
    }
    __syncthreads();
    const int rn = min(16, R - r0);
    for (int kk = 0; kk < rn; kk++) {
      const float4 a = *reinterpret_cast<const float4 *>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4 *>(&Bs[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int m = m0 + ty * 4 + i, c = n0 + tx * 4 + j;
      if (m < M && c < N) Cm[(size_t)m * ldc + c] = acc[i][j];
    }
}

// out[c] = (acc ? out[c] : 0) + X[0][c] + X[1][c] + ... + X[rows-1][c], in row order
__global__ void k_colsum(const float *__restrict__ X, int rows, int ld, int cols, float *__restrict__ out, int acc_in) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = acc_in ? out[c] : 0.0f;
  for (int r = 0; r < rows; r++) s += X[(size_t)r * ld + c];
  out[c] = s;
}

// d ip1 output through ip2 and ip1's ReLU
__global__ void k_dh(const float *__restrict__ h, const float *__restrict__ dz, const float *__restrict__ w2, int nb,
                     float *__restrict__ dh) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nb * NH) return;
  const int i = e / NH, k = e % NH;
  dh[e] = h[e] > 0.0f ? fmaf(w2[2 * k + 1], dz[2 * i + 1], w2[2 * k] * dz[2 * i]) : 0.0f;
}

// the gradient a pooled value passes to its chosen window position: all of it, or none under a ReLU that output 0
__device__ __forceinline__ float pooled_grad(float d, float pooled, int relu) { return (!relu || pooled > 0.0f) ? d : 0.0f; }

// d pool2 (k = c + 50 j) -> dense d conv2 [n][50][24][24]
__global__ void k_dconv2(const float *__restrict__ dx, const float *__restrict__ p2, const uint8_t *__restrict__ ch2,
                         int relu, int nb, float *__restrict__ dc2) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nb * NF2 * O2 * O2) return;
  const int i = e / (NF2 * O2 * O2), o = (e / (O2 * O2)) % NF2, Y = (e / O2) % O2, X = e % O2;
  const size_t k = (size_t)i * K + ((Y >> 1) * P2 + (X >> 1)) * NF2 + o;
  dc2[e] = ch2[k] == ((Y & 1) * 2 + (X & 1)) ? pooled_grad(dx[k], p2[k], relu) : 0.0f;
}

// conv2 weight and bias gradients of one image per CTA: partial[i][e], e in the .bin order (25 000 weights, 50 biases),
// each a chain over the 144 pooled positions in row-major order at their chosen windows
__global__ void __launch_bounds__(256) k_conv2_wgrad(const float *__restrict__ p1, const float *__restrict__ dx,
                                                     const float *__restrict__ p2, const uint8_t *__restrict__ ch2, int relu,
                                                     float *__restrict__ part) {
  extern __shared__ __align__(16) unsigned char dyn[];
  float *sp1 = reinterpret_cast<float *>(dyn);  // [20][28][28]
  float *sg = sp1 + NF1 * P1 * P1;              // [50][144]
  short *spos = reinterpret_cast<short *>(sg + K);
  const int im = blockIdx.x;
  for (int k = threadIdx.x; k < NF1 * P1 * P1; k += blockDim.x) sp1[k] = p1[(size_t)im * NF1 * P1 * P1 + k];
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int j = k / NF2, o = k % NF2, a = ch2[(size_t)im * K + k];
    sg[o * P2 * P2 + j] = pooled_grad(dx[(size_t)im * K + k], p2[(size_t)im * K + k], relu);
    spos[o * P2 * P2 + j] = (short)((2 * (j / P2) + (a >> 1)) * P1 + 2 * (j % P2) + (a & 1));
  }
  __syncthreads();
  for (int e = threadIdx.x; e < NW2; e += blockDim.x) {
    float acc = 0.0f;
    if (e < NF2 * NF1 * 25) {
      const int o = e / (NF1 * 25), c = (e / 25) % NF1, kh = (e % 25) / 5, kw = e % 5;
      const float *x = sp1 + c * P1 * P1 + kh * P1 + kw;
      const float *g = sg + o * P2 * P2;
      const short *q = spos + o * P2 * P2;
      for (int j = 0; j < P2 * P2; j++) acc = fmaf(g[j], x[q[j]], acc);
    } else {
      const float *g = sg + (e - NF2 * NF1 * 25) * P2 * P2;
      for (int j = 0; j < P2 * P2; j++) acc += g[j];
    }
    part[(size_t)im * NW2 + e] = acc;
  }
}

// d pool1 of one image per CTA: dp1[c][y][x] = sum over (o, kh, kw) in order of dc2[o][y-kh][x-kw] w2[o][c][kh][kw]
__global__ void __launch_bounds__(256) k_dpool1(const float *__restrict__ dc2, const float *__restrict__ w2,
                                                float *__restrict__ dp1) {
  extern __shared__ __align__(16) unsigned char dyn[];
  float *sd = reinterpret_cast<float *>(dyn);  // [50][24][24]
  const int im = blockIdx.x;
  for (int k = threadIdx.x; k < NF2 * O2 * O2; k += blockDim.x) sd[k] = dc2[(size_t)im * NF2 * O2 * O2 + k];
  __syncthreads();
  for (int e = threadIdx.x; e < NF1 * P1 * P1; e += blockDim.x) {
    const int c = e / (P1 * P1), y = (e / P1) % P1, x = e % P1;
    const int kh0 = max(0, y - (O2 - 1)), kh1 = min(4, y), kw0 = max(0, x - (O2 - 1)), kw1 = min(4, x);
    float acc = 0.0f;
    for (int o = 0; o < NF2; o++) {
      const float *wp = w2 + (o * NF1 + c) * 25;
      const float *d = sd + o * O2 * O2;
      for (int kh = kh0; kh <= kh1; kh++)
        for (int kw = kw0; kw <= kw1; kw++) acc = fmaf(d[(y - kh) * O2 + x - kw], __ldg(wp + kh * 5 + kw), acc);
    }
    dp1[(size_t)im * NF1 * P1 * P1 + e] = acc;
  }
}

// conv1 weight and bias gradients of one image per CTA: partial[i][e], e in the .bin order (500 C weights, 20 biases),
// each a chain over the 784 pooled positions in row-major order at their chosen windows
__global__ void __launch_bounds__(256) k_conv1_wgrad(const uint8_t *__restrict__ hwc, int C, const float *__restrict__ dp1,
                                                     const float *__restrict__ p1, const uint8_t *__restrict__ ch1, int relu,
                                                     float *__restrict__ part) {
  extern __shared__ __align__(16) unsigned char dyn[];
  float *sg = reinterpret_cast<float *>(dyn);  // [20][784]
  short *spos = reinterpret_cast<short *>(sg + NF1 * P1 * P1);
  uint8_t *simg = reinterpret_cast<uint8_t *>(spos + NF1 * P1 * P1);  // [C][60][60]
  const int im = blockIdx.x, nw = NF1 * C * 25;
  const uint8_t *g = hwc + (size_t)im * S * S * C;
  for (int k = threadIdx.x; k < S * S * C; k += blockDim.x) {
    const int pix = k / C, c = k - pix * C;
    simg[c * S * S + pix] = g[k];
  }
  for (int k = threadIdx.x; k < NF1 * P1 * P1; k += blockDim.x) {
    const size_t at = (size_t)im * NF1 * P1 * P1 + k;
    const int p = k % (P1 * P1), a = ch1[at];
    sg[k] = pooled_grad(dp1[at], p1[at], relu);
    spos[k] = (short)((2 * (p / P1) + (a >> 1)) * S + 2 * (p % P1) + (a & 1));
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nw + NF1; e += blockDim.x) {
    float acc = 0.0f;
    if (e < nw) {
      const int o = e / (C * 25), c = (e / 25) % C, kh = (e % 25) / 5, kw = e % 5;
      const uint8_t *x = simg + c * S * S + kh * S + kw;
      const float *gg = sg + o * P1 * P1;
      const short *q = spos + o * P1 * P1;
      for (int p = 0; p < P1 * P1; p++) acc = fmaf(gg[p], (float)x[q[p]], acc);
    } else {
      const float *gg = sg + (e - nw) * P1 * P1;
      for (int p = 0; p < P1 * P1; p++) acc += gg[p];
    }
    part[(size_t)im * (nw + NF1) + e] = acc;
  }
}

__global__ void k_sgd(float *__restrict__ w, const float *__restrict__ g, float *__restrict__ buf, size_t n, float lr,
                      float mu, float wd, int first) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) gpdb_train_sgd(w + e, g[e], buf + e, lr, mu, wd, first != 0);
}

__global__ void k_adam(float *__restrict__ w, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v,
                       size_t n, float b1, float omb1, float b2, float omb2, float eps, float wd, float step, float r) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) gpdb_train_adam(w + e, g[e], m + e, v + e, b1, omb1, b2, omb2, eps, wd, step, r);
}

__global__ void k_check_labels(const int32_t *__restrict__ labels, int n, unsigned long long *first_bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && labels[i] != 0 && labels[i] != 1) atomicMin(first_bad, (unsigned long long)i);
}

size_t param_sizes(int C, size_t *off, size_t *len) {
  const size_t sz[8] = {(size_t)NF1 * C * 25, NF1, (size_t)NF2 * NF1 * 25, NF2, (size_t)NH * K, NH, 2 * NH, 2};
  off[0] = 0;
  for (int i = 0; i < 8; i++) {
    len[i] = sz[i];
    off[i + 1] = (off[i] + sz[i] + 3) / 4 * 4;
  }
  return off[8];
}

// the scratch of one chunk of nb images (SCR_TRAIN): 483 024 + 2 000 C bytes per image, plus alignment
struct ChunkBufs {
  uint8_t *p16, *ch1, *ch2;
  float *p1, *p2, *h3, *scores, *logits, *loss, *dz, *dh, *dx, *dc2, *dp1, *part2, *part1;
};
auto chunk_layout(ChunkBufs &b, int nb, int C) {
  return [&b, nb, C](Carve &c) {
    const size_t n = (size_t)nb;
    b.p16 = c.take<uint8_t>(n * S * S * 16, 16);
    b.p1 = c.take<float>(n * NF1 * P1 * P1, 16);
    b.p2 = c.take<float>(n * K, 16);
    b.h3 = c.take<float>(n * NH, 16);
    b.scores = c.take<float>(n);
    b.logits = c.take<float>(2 * n);
    b.loss = c.take<float>(n);
    b.dz = c.take<float>(2 * n);
    b.dh = c.take<float>(n * NH);
    b.dx = c.take<float>(n * K);
    b.dc2 = c.take<float>(n * NF2 * O2 * O2);
    b.dp1 = c.take<float>(n * NF1 * P1 * P1);
    b.part2 = c.take<float>(n * NW2);
    b.part1 = c.take<float>(n * ((size_t)NF1 * C * 25 + NF1));
    b.ch1 = c.take<uint8_t>(n * NF1 * P1 * P1);
    b.ch2 = c.take<uint8_t>(n * K);
  };
}

int gemm(gpdb_ctx *ctx, const float *A, long am, long ar, const float *B, long br, long bc, float *Cm, int ldc, int M,
         int N, int R, int acc) {
  dim3 grid((M + 63) / 64, (N + 63) / 64);
  k_gemm<<<grid, 256, 0, ctx->stream>>>(A, am, ar, B, br, bc, Cm, ldc, M, N, R, acc);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int colsum(gpdb_ctx *ctx, const float *X, int rows, int ld, int cols, float *out, int acc) {
  k_colsum<<<(cols + 127) / 128, 128, 0, ctx->stream>>>(X, rows, ld, cols, out, acc);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int relayout(gpdb_ctx *ctx, TrainState &ts, int dir) {
  const int n = NF1 * ts.C * 25 + NF2 * NF1 * 25;
  k_relayout<<<(n + 255) / 256, 256, 0, ctx->stream>>>(ts.w + ts.off[0], ts.w + ts.off[2], ts.C, ts.c1t, ts.c2t, dir);
  LAUNCH_CHECK();
  return GPDB_OK;
}

#define TRY(x)                          \
  do {                                  \
    const int rc__ = (x);               \
    if (rc__ != GPDB_OK) return rc__;   \
  } while (0)

// forward, pooling choices, loss and every gradient of one chunk (images b0 .. b0 + nb of a step of n), the parameter
// gradients chained onto ts.g unless first
int chunk(gpdb_ctx *ctx, TrainState &ts, ChunkBufs &b, const uint8_t *d_img, const int32_t *d_lab, int nb, int n,
          bool first, bool last, float *d_loss_out) {
  const int C = ts.C, relu = ctx->prm.relu_after_conv, acc = first ? 0 : 1;
  const float *w = ts.w;
  float *g = ts.g;
  const size_t *off = ts.off;
  TRY(geo_hwc_to_p16(ctx, d_img, nb, b.p16));
  const LenetWeights lw = {ts.c1t, ts.w + off[1], ts.c2t, ts.w + off[3], ts.w + off[4], ts.w + off[5], ts.w + off[6],
                           ts.w + off[7], C, true};
  TRY(lenet_simt_run(ctx, lw, b.p16, nb, b.p1, b.p2, b.h3, b.scores, b.logits));
  const size_t sm1 = sizeof(float) * NF1 * C * 25 + (size_t)C * S * S, sm2 = sizeof(float) * (NF2 * NF1 * 25 + NF1 * P1 * P1);
  CUDA_TRY(cudaFuncSetAttribute(k_choice1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
  CUDA_TRY(cudaFuncSetAttribute(k_choice2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
  k_choice1<<<nb, 256, sm1, ctx->stream>>>(d_img, C, w + off[0], w + off[1], b.ch1);
  LAUNCH_CHECK();
  k_choice2<<<nb, 256, sm2, ctx->stream>>>(b.p1, w + off[2], w + off[3], b.ch2);
  LAUNCH_CHECK();
  k_loss<<<(nb + 127) / 128, 128, 0, ctx->stream>>>(b.logits, d_lab, nb, (float)n, b.loss, b.dz);
  LAUNCH_CHECK();
  k_loss_sum<<<1, 1, 0, ctx->stream>>>(b.loss, nb, first, last, (float)n, ts.loss, d_loss_out);
  LAUNCH_CHECK();
  // ip2: dW2[o + 2k] = sum_i dz[i][o] h[i][k]; db2
  TRY(gemm(ctx, b.h3, 1, NH, b.dz, 2, 1, g + off[6], 2, NH, 2, nb, acc));
  TRY(colsum(ctx, b.dz, nb, 2, 2, g + off[7], acc));
  k_dh<<<(nb * NH + 255) / 256, 256, 0, ctx->stream>>>(b.h3, b.dz, w + off[6], nb, b.dh);
  LAUNCH_CHECK();
  // ip1: dW1[k][o] = sum_i x[i][k] dh[i][o]; db1; dx[i][k] = sum_o dh[i][o] W1[k][o]
  TRY(gemm(ctx, b.p2, 1, K, b.dh, NH, 1, g + off[4], NH, K, NH, nb, acc));
  TRY(colsum(ctx, b.dh, nb, NH, NH, g + off[5], acc));
  TRY(gemm(ctx, b.dh, NH, 1, w + off[4], 1, NH, b.dx, K, nb, K, NH, 0));
  // pool2 -> conv2
  k_dconv2<<<(nb * NF2 * O2 * O2 + 255) / 256, 256, 0, ctx->stream>>>(b.dx, b.p2, b.ch2, relu, nb, b.dc2);
  LAUNCH_CHECK();
  const size_t smw2 = sizeof(float) * (NF1 * P1 * P1 + K) + sizeof(short) * K;
  CUDA_TRY(cudaFuncSetAttribute(k_conv2_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smw2));
  k_conv2_wgrad<<<nb, 256, smw2, ctx->stream>>>(b.p1, b.dx, b.p2, b.ch2, relu, b.part2);
  LAUNCH_CHECK();
  TRY(colsum(ctx, b.part2, nb, NW2, NW2, g + off[2], acc));
  const size_t smd1 = sizeof(float) * NF2 * O2 * O2;
  CUDA_TRY(cudaFuncSetAttribute(k_dpool1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smd1));
  k_dpool1<<<nb, 256, smd1, ctx->stream>>>(b.dc2, w + off[2], b.dp1);
  LAUNCH_CHECK();
  // pool1 -> conv1
  const int nw1 = NF1 * C * 25 + NF1;
  const size_t smw1 = (sizeof(float) + sizeof(short)) * NF1 * P1 * P1 + (size_t)C * S * S;
  CUDA_TRY(cudaFuncSetAttribute(k_conv1_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smw1));
  k_conv1_wgrad<<<nb, 256, smw1, ctx->stream>>>(d_img, C, b.dp1, b.p1, b.ch1, relu, b.part1);
  LAUNCH_CHECK();
  TRY(colsum(ctx, b.part1, nb, nw1, nw1, g + off[0], acc));
  return GPDB_OK;
}

// gpdb_debug_train_step: the per-image arrays of the chunk that just ran (images b0 .. b0 + nb of the step) to the
// caller's arrays at image offset b0, before the next chunk overwrites the buffers
int debug_copy_chunk(gpdb_ctx *ctx, const ChunkBufs &b, const gpdb_train_debug &dbg, int b0, int nb) {
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  auto get = [&](auto *dst, const void *src, size_t per_image) {
    return dst ? cudaMemcpy(dst + per_image * b0, src, sizeof(*dst) * per_image * nb, cudaMemcpyDeviceToHost)
               : cudaSuccess;
  };
  CUDA_TRY(get(dbg.pool1, b.p1, NF1 * P1 * P1));
  CUDA_TRY(get(dbg.pool2, b.p2, K));
  CUDA_TRY(get(dbg.ip1, b.h3, NH));
  CUDA_TRY(get(dbg.logits, b.logits, 2));
  CUDA_TRY(get(dbg.choice1, b.ch1, NF1 * P1 * P1));
  CUDA_TRY(get(dbg.choice2, b.ch2, K));
  CUDA_TRY(get(dbg.loss, b.loss, 1));
  CUDA_TRY(get(dbg.dlogits, b.dz, 2));
  CUDA_TRY(get(dbg.dip1, b.dh, NH));
  CUDA_TRY(get(dbg.dpool2, b.dx, K));
  CUDA_TRY(get(dbg.dpool1, b.dp1, NF1 * P1 * P1));
  return GPDB_OK;
}

bool params_ok(const gpdb_train_params &p) {
  auto nonneg = [](float x) { return std::isfinite(x) && x >= 0.0f; };
  if (p.optimizer != 0 && p.optimizer != 1) return false;
  if (!nonneg(p.lr) || !nonneg(p.weight_decay)) return false;
  if (p.optimizer == 0) return nonneg(p.momentum);
  return nonneg(p.eps) && nonneg(p.beta1) && p.beta1 < 1.0f && nonneg(p.beta2) && p.beta2 < 1.0f;
}

}  // namespace

static bool train_started(const gpdb_ctx *ctx) { return ctx->train != nullptr; }

void train_free(gpdb_ctx *ctx) {
  if (!ctx->train) return;
  cudaFree(ctx->train->w);
  delete ctx->train;
  ctx->train = nullptr;
}

static int train_begin(gpdb_ctx *ctx, const gpdb_train_params *p, const float *const init[8]) {
  if (!p || !params_ok(*p)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_train_begin: bad training parameters");
    return GPDB_ERR_INVALID;
  }
  if (init) {
    for (int i = 0; i < 8; i++)
      if (!init[i]) {
        gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_train_begin: null weight array %d", i);
        return GPDB_ERR_INVALID;
      }
  } else if (!ctx->w.set) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "gpdb_train_begin: no classifier weights to start from: pass init or call "
                                        "gpdb_load_weights_dir / gpdb_set_weights first");
    return GPDB_ERR_STATE;
  }
  const int C = ctx->prm.image_num_channels;
  TrainState *ts = new TrainState{};
  const size_t np = param_sizes(C, ts->off, ts->len), nt1 = (size_t)NF1 * C * 25, nt2 = (size_t)NF2 * NF1 * 25;
  ts->C = C;
  ts->p = *p;
  float *base = nullptr;
  if (cudaMalloc(&base, sizeof(float) * (4 * np + nt1 + nt2 + 2)) != cudaSuccess) {
    cudaGetLastError();
    delete ts;
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "gpdb_train_begin: out of device memory");
    return GPDB_ERR_CUDA;
  }
  ts->w = base;
  ts->m = base + np;
  ts->v = base + 2 * np;
  ts->g = base + 3 * np;
  ts->c1t = base + 4 * np;
  ts->c2t = ts->c1t + nt1;
  ts->loss = ts->c2t + nt2;
  auto fail = [&](int rc) {
    cudaFree(base);
    delete ts;
    return rc;
  };
  if (cudaMemsetAsync(base, 0, sizeof(float) * 4 * np, ctx->stream) != cudaSuccess) return fail(GPDB_ERR_CUDA);
  int rc = GPDB_OK;
  if (init) {
    for (int i = 0; i < 8 && rc == GPDB_OK; i++)
      if (cudaMemcpyAsync(ts->w + ts->off[i], init[i], sizeof(float) * ts->len[i], cudaMemcpyHostToDevice,
                          ctx->stream) != cudaSuccess)
        rc = GPDB_ERR_CUDA;
  } else {
    const LenetWeights &w = ctx->w;
    const float *src[8] = {nullptr, w.c1b, nullptr, w.c2b, w.i1w, w.i1b, w.i2w, w.i2b};
    for (int i = 0; i < 8 && rc == GPDB_OK; i++)
      if (src[i] && cudaMemcpyAsync(ts->w + ts->off[i], src[i], sizeof(float) * ts->len[i],
                                    cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess)
        rc = GPDB_ERR_CUDA;
    if (rc == GPDB_OK &&
        (cudaMemcpyAsync(ts->c1t, w.c1w, sizeof(float) * nt1, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess ||
         cudaMemcpyAsync(ts->c2t, w.c2w, sizeof(float) * nt2, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess))
      rc = GPDB_ERR_CUDA;
    if (rc == GPDB_OK) rc = relayout(ctx, *ts, 1);
  }
  if (rc == GPDB_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = GPDB_ERR_CUDA;
  if (rc != GPDB_OK) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "gpdb_train_begin: %s", cudaGetErrorString(cudaGetLastError()));
    return fail(rc);
  }
  train_free(ctx);
  ctx->train = ts;
  return GPDB_OK;
}

// the label check of a step: lowers *d_bad to the first label outside {0, 1}
static int train_check_labels(gpdb_ctx *ctx, const int32_t *d_labels, int n, unsigned long long *d_bad) {
  k_check_labels<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_labels, n, d_bad);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// one step on n device images / labels (labels already checked); d_loss_out / h_loss_out: device / host float or null;
// dbg: host outputs of a debug step (any n, copied chunk by chunk), which updates nothing
static int train_step(gpdb_ctx *ctx, const uint8_t *d_images, const int32_t *d_labels, int n, float *d_loss_out,
                      float *h_loss_out, const gpdb_train_debug *dbg) {
  TrainState &ts = *ctx->train;
  const int C = ts.C, chunk_n = std::min(n, GPDB_TRAIN_CHUNK);
  ChunkBufs b;
  if (!gpdb_carve(ctx, SCR_TRAIN, chunk_layout(b, chunk_n, C))) return GPDB_ERR_CUDA;
  TRY(relayout(ctx, ts, 0));
  const size_t isz = (size_t)S * S * C;
  for (int b0 = 0; b0 < n; b0 += GPDB_TRAIN_CHUNK) {
    const int nb = std::min(GPDB_TRAIN_CHUNK, n - b0);
    TRY(chunk(ctx, ts, b, d_images + isz * b0, d_labels + b0, nb, n, b0 == 0, b0 + nb == n, d_loss_out));
    if (dbg) TRY(debug_copy_chunk(ctx, b, *dbg, b0, nb));
  }
  if (dbg) {  // the gradients once, after the last chunk has chained onto them
    for (int i = 0; i < 8; i++)
      if (dbg->grad[i])
        CUDA_TRY(cudaMemcpy(dbg->grad[i], ts.g + ts.off[i], sizeof(float) * ts.len[i], cudaMemcpyDeviceToHost));
    return GPDB_OK;
  }
  const gpdb_train_params &p = ts.p;
  float step = 0.0f, r = 0.0f;
  if (p.optimizer == 1) gpdb_train_adam_scalars(p.lr, p.beta1, p.beta2, ts.t + 1, &step, &r);
  for (int i = 0; i < 8; i++) {  // the arrays only, not the padding between them
    const size_t o = ts.off[i], len = ts.len[i];
    const unsigned blocks = (unsigned)((len + 255) / 256);
    if (p.optimizer == 0)
      k_sgd<<<blocks, 256, 0, ctx->stream>>>(ts.w + o, ts.g + o, ts.m + o, len, p.lr, p.momentum, p.weight_decay, ts.t == 0);
    else
      k_adam<<<blocks, 256, 0, ctx->stream>>>(ts.w + o, ts.g + o, ts.m + o, ts.v + o, len, p.beta1, 1.0f - p.beta1, p.beta2,
                                              1.0f - p.beta2, p.eps, p.weight_decay, step, r);
    LAUNCH_CHECK();
  }
  ts.t++;
  if (h_loss_out) {
    CUDA_TRY(cudaMemcpyAsync(h_loss_out, ts.loss + 1, sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  return GPDB_OK;
}

static int train_weights(gpdb_ctx *ctx, float *const out[8]) {
  const TrainState &ts = *ctx->train;
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < 8; i++)
    CUDA_TRY(cudaMemcpy(out[i], ts.w + ts.off[i], sizeof(float) * ts.len[i], cudaMemcpyDeviceToHost));
  return GPDB_OK;
}

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

extern "C" {

int gpdb_train_begin(gpdb_ctx *ctx, const gpdb_train_params *p, const float *const init[8]) {
  int rc = gpdb_check_state(ctx, false, false);
  if (rc != GPDB_OK) return rc;
  return train_begin(ctx, p, init);
}

namespace {

// the checks of a training step before any device work: begun, a 60 x 60 network, n >= 1, the arrays given
int train_step_args(gpdb_ctx *ctx, const char *name, const void *images, const void *labels, int32_t n) {
  int rc = gpdb_check_state(ctx, false, false);
  if (rc != GPDB_OK) return rc;
  if (!train_started(ctx)) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "%s: call gpdb_train_begin first", name);
    return GPDB_ERR_STATE;
  }
  if (ctx->prm.image_size != 60) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: LeNet expects image_size 60, got %d", name, ctx->prm.image_size);
    return GPDB_ERR_INVALID;
  }
  if (n <= 0 || !images || !labels) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: bad arguments (n = %d)", name, n);
    return GPDB_ERR_INVALID;
  }
  return GPDB_OK;
}

// the device check of the labels, then the step: a label outside {0, 1} fails the step before anything changes
int train_step_checked(gpdb_ctx *ctx, const char *name, const uint8_t *d_images, const int32_t *d_labels, int32_t n,
                       float *d_loss_out, float *h_loss_out, const gpdb_train_debug *dbg) {
  unsigned long long bad;
  int rc = first_bad(ctx, 0, &bad, [&](unsigned long long *d_bad, void *) {
    return train_check_labels(ctx, d_labels, n, d_bad);
  });
  if (rc != GPDB_OK) return rc;
  if (bad != NO_BAD) {
    int32_t v = 0;
    CUDA_TRY(cudaMemcpy(&v, d_labels + bad, sizeof(v), cudaMemcpyDeviceToHost));
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: labels[%llu] = %d is not 0 or 1", name, bad, v);
    return GPDB_ERR_INVALID;
  }
  return train_step(ctx, d_images, d_labels, n, d_loss_out, h_loss_out, dbg);
}

// host twins: upload images and labels (SCR_HWC / SCR_LABELS), then the device path
int train_step_host(gpdb_ctx *ctx, const char *name, const uint8_t *images_hwc, const int32_t *labels, int32_t n,
                    float *loss_out, const gpdb_train_debug *dbg) {
  const size_t isz = (size_t)60 * 60 * ctx->prm.image_num_channels * n;
  uint8_t *d_img = (uint8_t *)gpdb_scratch(ctx, SCR_HWC, isz);
  int32_t *d_lab = (int32_t *)gpdb_scratch(ctx, SCR_LABELS, sizeof(int32_t) * (size_t)n);
  if (!d_img || !d_lab) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(d_img, images_hwc, isz, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(d_lab, labels, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  return train_step_checked(ctx, name, d_img, d_lab, n, nullptr, loss_out, dbg);
}

}  // namespace

int gpdb_train_step(gpdb_ctx *ctx, const uint8_t *images_hwc, const int32_t *labels, int32_t n, float *loss_out) {
  const char *name = "gpdb_train_step";
  int rc = train_step_args(ctx, name, images_hwc, labels, n);
  if (rc != GPDB_OK) return rc;
  return train_step_host(ctx, name, images_hwc, labels, n, loss_out, nullptr);
}

int gpdb_train_step_device(gpdb_ctx *ctx, const uint8_t *d_images_hwc, const int32_t *d_labels, int32_t n,
                           float *d_loss_out) {
  const char *name = "gpdb_train_step_device";
  int rc = train_step_args(ctx, name, d_images_hwc, d_labels, n);
  if (rc != GPDB_OK) return rc;
  rc = gpdb_check_device_ptrs(ctx, name, {{"d_images_hwc", d_images_hwc}, {"d_labels", d_labels}, {"d_loss_out", d_loss_out}});
  if (rc != GPDB_OK) return rc;
  return train_step_checked(ctx, name, d_images_hwc, d_labels, n, d_loss_out, nullptr, nullptr);
}

int gpdb_debug_train_step(gpdb_ctx *ctx, const uint8_t *images_hwc, const int32_t *labels, int32_t n,
                          gpdb_train_debug *out) {
  const char *name = "gpdb_debug_train_step";
  int rc = train_step_args(ctx, name, images_hwc, labels, n);
  if (rc != GPDB_OK) return rc;
  if (!out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need an output struct", name);
    return GPDB_ERR_INVALID;
  }
  return train_step_host(ctx, name, images_hwc, labels, n, nullptr, out);
}

int gpdb_train_weights(gpdb_ctx *ctx, float *const out[8]) {
  int rc = gpdb_check_state(ctx, false, false);
  if (rc != GPDB_OK) return rc;
  if (!train_started(ctx)) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "gpdb_train_weights: call gpdb_train_begin first");
    return GPDB_ERR_STATE;
  }
  if (!out || !out[0] || !out[1] || !out[2] || !out[3] || !out[4] || !out[5] || !out[6] || !out[7]) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_train_weights: null output array");
    return GPDB_ERR_INVALID;
  }
  return train_weights(ctx, out);
}

}  // extern "C"
