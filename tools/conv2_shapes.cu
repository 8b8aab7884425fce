// conv2_shapes.cu — tensor-clock rate of the wgmma shapes conv2 can be written with, in isolation (development aid; run it
// through tools/conv2_shapes.sh). One CTA per SM, two warpgroups; each issues back-to-back batches of one conv2 tile (the
// 65 K-chunks of `c2_off`, paired per k16 step) from shared-memory operands laid out as in lenet_tc.cu, and waits for
// them before the next batch, so one warpgroup's wait overlaps the other's instructions. Operand values are a fixed
// pattern: only the rates matter.
//   pix-M  : today's kernel: A = a Hankel pixel plane (two m64 halves of a 128-row tile), B = [w_hi | w_lo]:
//            per half and k16 step m64n112k16 (a_hi) + m64n56k16 (a_lo)
//   f-M N  : transposed: A = a 64-row weight block [chunk][hi|lo][64][16 B], B = N pixels of the Hankel plane:
//            per k16 step three m64nNk16 (w_hi a_hi, w_lo a_hi, w_hi a_lo), N = 224, 256, 112
// It reports SM cycles per instruction against the dense f16 rate (2 048 MAC per clock per SM: m64nNk16 = N / 2 clocks),
// and the cycles per valid conv2 output pixel (24 of every 28 GEMM pixels). The SM clock is the cycle count over the
// CUDA-event time of the same launch.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "wgmma.cuh"

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      fprintf(stderr, "%s:%d %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)

constexpr int W = 28, NCH = 65, NMMA = 33;

// byte offset of K-chunk c inside a stage of six planes of `plane` bytes (lenet_tc.cu's c2_off)
__host__ __device__ constexpr uint32_t chunk_off(int c, uint32_t plane) {
  const int cc = c >= NCH ? NCH - 1 : c;
  return cc < 50 ? (uint32_t)((cc / 25) * plane + (((cc / 5) % 5) * W + cc % 5) * 16)
                 : (uint32_t)(2 * plane + (((cc - 50) / 3) * W + 2 * ((cc - 50) % 3)) * 16);
}

// variant V: 0 = pix-M (n112 + n56), 1 = f-M n224, 2 = f-M n256, 3 = f-M n112
template <int V>
struct Shape {
  static constexpr int N = V == 0 ? 112 : V == 1 ? 224 : V == 2 ? 256 : 112;
  static constexpr int NPIX = V == 0 ? 256 : N + 120;                   // plane pixels, incl. the tail the Hankel reads
  static constexpr int PLANE = NPIX * 16, STAGE = 6 * PLANE;
  static constexpr int W_BYTES = V == 0 ? 2 * NMMA * 112 * 16 : 2 * NMMA * 2 * 64 * 16;
  static constexpr int SMEM = W_BYTES + 2 * STAGE;
  static constexpr int NACC = V == 0 ? 112 : N / 2;
  static constexpr int INSTR = V == 0 ? 4 * NMMA : 3 * NMMA;            // per warpgroup batch
  static constexpr int IDEAL = V == 0 ? 2 * NMMA * (56 + 28) : 3 * NMMA * N / 2;  // dense tensor clocks per batch
  static constexpr int VALID_PIX = V == 0 ? 96 : (N / W) * 24 + (N % W < 24 ? N % W : 24);
};

template <int V>
__device__ __forceinline__ void batch(float *d, uint32_t sw, uint32_t pl) {
  using S = Shape<V>;
#pragma unroll
  for (int i = 0; i < NMMA; i++) {
    const uint32_t a0 = chunk_off(2 * i, S::PLANE), a1 = chunk_off(2 * i + 1, S::PLANE);
    const uint32_t lbo = (2 * i + 1 >= NCH) ? 16u : (a1 - a0);
    if constexpr (V == 0) {
      const uint64_t db = wg::desc(sw + (uint32_t)(2 * i) * 112 * 16, 112 * 16, 128);
      wg::mma_f16_n112(d, wg::desc(pl + a0, lbo, 128), db, i > 0);
      wg::mma_f16_n112(d + 56, wg::desc(pl + 64 * 16 + a0, lbo, 128), db, i > 0);
    } else {
      const uint64_t whi = wg::desc(sw + (uint32_t)(2 * i) * 2048, 2048, 128), wlo = whi + (1024 >> 4);
      const uint64_t ahi = wg::desc(pl + a0, lbo, 128), alo = wg::desc(pl + 3 * S::PLANE + a0, lbo, 128);
      if constexpr (S::N == 224) {
        wg::mma_f16_n224(d, whi, ahi, i > 0);
        wg::mma_f16_n224(d, wlo, ahi, true);
        wg::mma_f16_n224(d, whi, alo, true);
      } else if constexpr (S::N == 256) {
        wg::mma_f16_n256(d, whi, ahi, i > 0);
        wg::mma_f16_n256(d, wlo, ahi, true);
        wg::mma_f16_n256(d, whi, alo, true);
      } else {
        wg::mma_f16_n112(d, whi, ahi, i > 0);
        wg::mma_f16_n112(d, wlo, ahi, true);
        wg::mma_f16_n112(d, whi, alo, true);
      }
    }
  }
  if constexpr (V == 0) {
#pragma unroll
    for (int i = 0; i < NMMA; i++) {
      const uint32_t a0 = chunk_off(2 * i, S::PLANE), a1 = chunk_off(2 * i + 1, S::PLANE);
      const uint32_t lbo = (2 * i + 1 >= NCH) ? 16u : (a1 - a0);
      const uint64_t db = wg::desc(sw + (uint32_t)(2 * i) * 112 * 16, 112 * 16, 128);
      wg::mma_f16_n56(d, wg::desc(pl + 3 * S::PLANE + a0, lbo, 128), db, true);
      wg::mma_f16_n56(d + 56, wg::desc(pl + 3 * S::PLANE + 64 * 16 + a0, lbo, 128), db, true);
    }
  }
}

template <int V>
__global__ void __launch_bounds__(256, 1) k_shape(int reps, long long *cycles, float *sink) {
  using S = Shape<V>;
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, wgi = tid >> 7;
  // a fixed pattern of f16 values in [-1, 1): finite, non-zero, every bit position toggling
  uint16_t *h = reinterpret_cast<uint16_t *>(smem);
  for (int i = tid; i < S::SMEM / 2; i += blockDim.x) {
    const uint32_t x = (uint32_t)i * 2654435761u;
    h[i] = (uint16_t)(0x3800u | (x >> 22)) ^ (uint16_t)((x >> 15) & 0x8000u);
  }
  wg::fence_async_smem();
  __syncthreads();
  uint32_t sw = wg::smem_u32(smem), pl = sw + S::W_BYTES + (uint32_t)wgi * S::STAGE;
  float d[S::NACC];
#pragma unroll
  for (int i = 0; i < S::NACC; i++) d[i] = 0.0f;
  const long long t0 = clock64();
  for (int r = 0; r < reps; r++) {
    // the descriptors are formed per batch, as in the kernel, instead of being hoisted into (spilled) registers
    asm volatile("" : "+r"(sw), "+r"(pl));
    wg::fence();
    batch<V>(d, sw, pl);
    wg::commit();
    wg::wait<0>();
    wg::reg_fence(d);
  }
  __syncthreads();
  const long long t1 = clock64();
  if (tid == 0) cycles[blockIdx.x] = t1 - t0;
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < S::NACC; i++) s += d[i];
  if (s == 12345.0f) sink[tid] = s;  // keeps the results live
}

template <int V>
static void run(const char *name, int sms, int reps) {
  using S = Shape<V>;
  CK(cudaFuncSetAttribute(k_shape<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::SMEM));
  long long *cyc;
  float *sink;
  CK(cudaMalloc(&cyc, sms * sizeof(long long)));
  CK(cudaMalloc(&sink, 256 * sizeof(float)));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  k_shape<V><<<sms, 256, S::SMEM>>>(reps / 10, cyc, sink);  // warm-up
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(e0));
  k_shape<V><<<sms, 256, S::SMEM>>>(reps, cyc, sink);
  CK(cudaEventRecord(e1));
  CK(cudaGetLastError());
  CK(cudaEventSynchronize(e1));
  float ms = 0.0f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  long long *h = (long long *)malloc(sms * sizeof(long long));
  CK(cudaMemcpy(h, cyc, sms * sizeof(long long), cudaMemcpyDeviceToHost));
  double mean = 0.0;
  long long mx = 0;
  for (int i = 0; i < sms; i++) mean += (double)h[i] / sms, mx = h[i] > mx ? h[i] : mx;
  const double batches = 2.0 * reps;  // per SM: two warpgroups
  const double per_instr = mean / (batches * S::INSTR), ideal = (double)S::IDEAL / S::INSTR;
  printf("%-10s %4d instr/batch  %7.1f cycles/instr  (dense %6.1f)  %5.1f %% of dense  %6.2f cycles/valid px  "
         "%7.1f ms  SM clock %5.0f MHz\n",
         name, S::INSTR, per_instr, ideal, 100.0 * ideal / per_instr, mean / (batches * S::VALID_PIX), ms,
         (double)mx / (ms * 1e3));
  free(h);
  CK(cudaFree(cyc));
  CK(cudaFree(sink));
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
}

int main(int argc, char **argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 4000;
  cudaDeviceProp p;
  CK(cudaGetDeviceProperties(&p, 0));
  printf("%s, %d SMs, %d batches per warpgroup\n", p.name, p.multiProcessorCount, reps);
  for (int pass = 0; pass < 2; pass++) {  // the second pass shows the spread
    run<0>("pix-M", p.multiProcessorCount, reps);
    run<1>("f-M n224", p.multiProcessorCount, reps);
    run<2>("f-M n256", p.multiProcessorCount, reps);
    run<3>("f-M n112", p.multiProcessorCount, reps);
  }
  return 0;
}
