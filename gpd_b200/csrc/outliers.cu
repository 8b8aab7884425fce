// outliers.cu — Cloud::removeStatisticalOutliers on the device (include/gpd_b200_outliers.h).
//
//   k_refine_knn     (refine.cu, through refine_knn_lists) the mean_k + 1 nearest neighbours of every point (rule 1)
//   k_outlier_mean   one thread per point: the distances to list entries 1..mean_k and their mean (rule 2)
//   k_outlier_stats  one CTA per cloud: the two sequential double sums (one thread adds, the others stage the means in
//                    shared memory), then the statistics (rules 3 and 5)
//   k_outlier_mark   one thread per point: the decision (rule 4), the keep flags and bytes, per-cloud kept counts and
//                    whether a kept point misses a camera
//   k_outlier_gather one thread per point: the kept points, normals, camera masks and source indices at their scanned
//                    positions (rule 6)
// The gathered arrays go back into the store's arenas and the store is reinstalled with the new offsets, which rebuilds
// the grids and the nonunit flags; each cloud's all_seen flag is recomputed from the kept masks. Whatever step fails, the
// store is left without a cloud, as a failed install leaves it. Compiled with -fmad=false: every operation of the
// specification is rounded on its own.
#include <cmath>
#include <cub/cub.cuh>
#include <vector>

#include "../../include/gpd_b200_outliers.h"
#include "common.cuh"
#include "grid.cuh"

namespace {

constexpr int TB = 256;
constexpr int STATS_THREADS = 256;
constexpr int STATS_CHUNK = 4096;  // mean distances per shared-memory stage of k_outlier_stats

// rule 2 for concatenated point g: its list nbr[g*k ..], k = mean_k + 1, holds min(k, N_b) cloud-local indices
__global__ void __launch_bounds__(TB) k_outlier_mean(const CloudDesc *d, int B, int N, const float *xyz, const int *nbr,
                                                     int mean_k, float *dist) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const CloudDesc &D = d[b_cloud_of_point(d, B, g)];
  if (D.N <= mean_k) {  // rule 5: the cloud keeps every point
    dist[g] = NAN;
    return;
  }
  const float q[3] = {xyz[3 * (size_t)g], xyz[3 * (size_t)g + 1], xyz[3 * (size_t)g + 2]};
  const int *lst = nbr + (size_t)g * (mean_k + 1);
  double s = 0.0;
  for (int r = 1; r <= mean_k; r++) {
    const float *p = xyz + 3 * ((size_t)D.off + __ldg(lst + r));
    const float pp[3] = {__ldg(p), __ldg(p + 1), __ldg(p + 2)};
    s = gpdb_outlier_dist_add(s, gpdb_refine_l2(q, pp));
  }
  dist[g] = gpdb_outlier_mean(s, mean_k);
}

// rules 3 and 5 for cloud b = blockIdx.x: stats[3b ..] = mean, stddev, threshold. Thread 0 adds chunk c from shared memory
// while warps 1.. stage chunk c + 1, so the two chains wait on shared loads only.
__global__ void __launch_bounds__(STATS_THREADS) k_outlier_stats(const CloudDesc *d, const float *dist, int mean_k,
                                                                 double stddev_mul, double *stats) {
  __shared__ __align__(16) float s_d[2][STATS_CHUNK];
  const int b = blockIdx.x;
  const int n = d[b].N;
  if (n <= mean_k) {
    if (threadIdx.x == 0) gpdb_outlier_stats(0.0, 0.0, n, mean_k, stddev_mul, stats + 3 * (size_t)b);
    return;
  }
  const float *e = dist + d[b].off;
  const int nc = (n + STATS_CHUNK - 1) / STATS_CHUNK;
  for (int j = threadIdx.x; j < min(n, STATS_CHUNK); j += STATS_THREADS) s_d[0][j] = __ldg(e + j);
  __syncthreads();
  double sum = 0.0, sq = 0.0;
  for (int c = 0; c < nc; c++) {
    const int base = c * STATS_CHUNK;
    if (threadIdx.x == 0) {
      const float *p = s_d[c & 1];
      const int len = min(STATS_CHUNK, n - base);
      int j = 0;
#pragma unroll 2
      for (; j + 4 <= len; j += 4) {
        const float4 v = *reinterpret_cast<const float4 *>(p + j);
        gpdb_outlier_stats_add(&sum, &sq, v.x);
        gpdb_outlier_stats_add(&sum, &sq, v.y);
        gpdb_outlier_stats_add(&sum, &sq, v.z);
        gpdb_outlier_stats_add(&sum, &sq, v.w);
      }
      for (; j < len; j++) gpdb_outlier_stats_add(&sum, &sq, p[j]);
    } else if (threadIdx.x >= 32 && c + 1 < nc) {
      const int nb = base + STATS_CHUNK, nl = min(STATS_CHUNK, n - nb);
      for (int j = threadIdx.x - 32; j < nl; j += STATS_THREADS - 32) s_d[(c + 1) & 1][j] = __ldg(e + nb + j);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) gpdb_outlier_stats(sum, sq, n, mean_k, stddev_mul, stats + 3 * (size_t)b);
}

// rule 4: flag[g] (the scan's input) and kept[g] = 1 for a kept point. Per cloud b (both zeroed by the caller): cnt[b]
// counts the kept points, partial[b] becomes 1 when a kept point misses one of the cloud's cameras (the all_seen flag an
// install of the kept points computes is !partial[b])
__global__ void __launch_bounds__(TB) k_outlier_mark(const CloudDesc *d, int B, int N, const float *dist,
                                                     const double *stats, const uint8_t *cam, int *flag, uint8_t *kept,
                                                     int *cnt, int *partial) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = g < N;
  int b = 0, keep = 0;
  bool miss = false;
  if (in) {
    b = b_cloud_of_point(d, B, g);
    keep = !gpdb_outlier_removed(dist[g], stats[3 * (size_t)b + 2]);  // a NaN threshold (rule 5) keeps the point
    flag[g] = keep;
    kept[g] = (uint8_t)keep;
    const unsigned all = (1u << d[b].K) - 1;
    miss = keep && (cam[g] & all) != all;
  }
  // one atomic per cloud and warp
  const unsigned peers = __match_any_sync(0xffffffffu, in ? b : -1);
  const int n = __popc(peers & __ballot_sync(0xffffffffu, keep));
  const bool any_miss = (peers & __ballot_sync(0xffffffffu, miss)) != 0;
  if (in && (threadIdx.x & 31) == __ffs(peers) - 1) {
    if (n > 0) atomicAdd(cnt + b, n);
    if (any_miss) partial[b] = 1;
  }
}

// rule 6: kept point g to position pos[g] of the gathered arrays
__global__ void __launch_bounds__(TB) k_outlier_gather(int N, const int *flag, const int *pos, const float *xyz,
                                                       const double *nrm, const uint8_t *cam, const int *src, float *xyz2,
                                                       double *nrm2, uint8_t *cam2, int *src2) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N || !flag[g]) return;
  const size_t j = (size_t)pos[g];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    xyz2[3 * j + a] = xyz[3 * (size_t)g + a];
    nrm2[3 * j + a] = nrm[3 * (size_t)g + a];
  }
  cam2[j] = cam[g];
  src2[j] = src[g];
}

}  // namespace

#define LAUNCH_CHECK()                                   \
  do {                                                   \
    ctx->launches++;                                     \
    cudaError_t e__ = cudaGetLastError();                \
    if (e__ != cudaSuccess) {                            \
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return GPDB_ERR_CUDA;                              \
    }                                                    \
  } while (0)

namespace {

// SCR_OUTLIERS, in this order (8-byte blocks first): stats double[3B], gathered normals double[3N], gathered xyz
// float[3N], mean distances float[N], flags and scan int[N+1] each, gathered src int[N], counts and camera flags int[B]
// each, keep bytes [N], gathered camera masks [N]. The lists are SCR_NBR, shared with the normal refinement.
struct OutlierScratch {
  double *stats, *nrm2;
  float *xyz2, *dist;
  int *nbr, *flag, *pos, *src2, *cnt, *partial;
  uint8_t *kept, *cam2;
};

int outlier_scratch(gpdb_ctx *ctx, size_t N, int B, int k, OutlierScratch &w) {
  const size_t bytes = sizeof(double) * (3 * (size_t)B + 3 * N) + sizeof(float) * 4 * N +
                       sizeof(int) * (2 * (N + 1) + N + 2 * (size_t)B) + 2 * N;
  unsigned char *p = (unsigned char *)gpdb_scratch(ctx, SCR_OUTLIERS, bytes);
  w.nbr = (int *)gpdb_scratch(ctx, SCR_NBR, sizeof(int) * N * k);
  if (!p || !w.nbr) return GPDB_ERR_CUDA;
  w.stats = (double *)p;
  w.nrm2 = w.stats + 3 * (size_t)B;
  w.xyz2 = (float *)(w.nrm2 + 3 * N);
  w.dist = w.xyz2 + 3 * N;
  w.flag = (int *)(w.dist + N);
  w.pos = w.flag + N + 1;
  w.src2 = w.pos + N + 1;
  w.cnt = w.src2 + N;
  w.partial = w.cnt + B;
  w.kept = (uint8_t *)(w.partial + B);
  w.cam2 = w.kept + N;
  return GPDB_OK;
}

// outliers_remove_batch up to its result; an error may come after the store has been partly rewritten
int remove_batch(gpdb_ctx *ctx, CloudSet &s, int mean_k, double stddev_mul, int *off, double *stats, uint8_t *kept) {
  const int B = s.n, N = s.points(), k = mean_k + 1;
  OutlierScratch w;
  int rc = outlier_scratch(ctx, (size_t)N, B, k, w);
  if (rc != GPDB_OK) return rc;
  // the camera fields of the descriptors, for the reinstall; read back with the counts
  std::vector<CloudDesc> desc((size_t)B);
  std::vector<int> cnt(2 * (size_t)B);  // counts, then the camera flags
  CUDA_TRY(cudaMemcpyAsync(desc.data(), s.desc, sizeof(CloudDesc) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(w.cnt, 0, sizeof(int) * 2 * (size_t)B, ctx->stream));
  const int nb = (N + TB - 1) / TB;
  if ((rc = refine_knn_lists(ctx, s, k, w.nbr)) != GPDB_OK) return rc;
  if (N > 0) {
    k_outlier_mean<<<nb, TB, 0, ctx->stream>>>(s.desc, B, N, s.xyz, w.nbr, mean_k, w.dist);
    LAUNCH_CHECK();
  }
  k_outlier_stats<<<B, STATS_THREADS, 0, ctx->stream>>>(s.desc, w.dist, mean_k, stddev_mul, w.stats);
  LAUNCH_CHECK();
  if (N > 0) {
    k_outlier_mark<<<nb, TB, 0, ctx->stream>>>(s.desc, B, N, w.dist, w.stats, s.cam, w.flag, w.kept, w.cnt, w.partial);
    LAUNCH_CHECK();
    CUDA_TRY(cudaMemsetAsync(w.flag + N, 0, sizeof(int), ctx->stream));
    size_t tmp_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, w.flag, w.pos, N + 1, ctx->stream);
    void *tmp = gpdb_scratch(ctx, SCR_CUB, tmp_bytes);
    if (!tmp) return GPDB_ERR_CUDA;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, w.flag, w.pos, N + 1, ctx->stream));
    ctx->launches += 2;
    k_outlier_gather<<<nb, TB, 0, ctx->stream>>>(N, w.flag, w.pos, s.xyz, s.nrm, s.cam, s.src, w.xyz2, w.nrm2, w.cam2,
                                                 w.src2);
    LAUNCH_CHECK();
  }
  CUDA_TRY(cudaMemcpyAsync(cnt.data(), w.cnt, sizeof(int) * 2 * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  if (stats) CUDA_TRY(cudaMemcpyAsync(stats, w.stats, sizeof(double) * 3 * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  if (kept && N > 0) CUDA_TRY(cudaMemcpyAsync(kept, w.kept, (size_t)N, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  off[0] = 0;
  for (int b = 0; b < B; b++) {
    off[b + 1] = off[b] + cnt[b];
    desc[b].all_seen = !cnt[B + b];  // as gpdb_pack_cameras computes it for the kept points
  }
  const size_t n2 = (size_t)off[B];
  const bool has_src = s.has_src;
  CUDA_TRY(cudaMemcpyAsync(s.xyz, w.xyz2, sizeof(float) * 3 * n2, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(s.nrm, w.nrm2, sizeof(double) * 3 * n2, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(s.cam, w.cam2, n2, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(s.src, w.src2, sizeof(int) * n2, cudaMemcpyDeviceToDevice, ctx->stream));
  if ((rc = gpdb_install_clouds(ctx, s, desc.data(), off, B, true)) != GPDB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  s.has_src = has_src;  // the raw offsets stay: src still indexes each cloud's raw points
  return B;
}

}  // namespace

int outliers_remove_batch(gpdb_ctx *ctx, CloudSet &s, int mean_k, double stddev_mul, int *off, double *stats,
                          uint8_t *kept) {
  const int rc = remove_batch(ctx, s, mean_k, stddev_mul, off, stats, kept);
  if (rc < 0) {  // whatever step failed, the store holds no cloud, as after a failed install
    s.n = 0;
    s.has_src = false;
  }
  return rc;
}
