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
// specification is rounded on its own. The entry points gpdb_remove_outliers and gpdb_remove_outliers_clouds, with their
// checks, follow the kernels.
#include <algorithm>
#include <cmath>
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

// rules 3 and 5 for cloud b = blockIdx.x: stats[3b ..] = mean, stddev, threshold
__global__ void __launch_bounds__(STATS_THREADS) k_outlier_stats(const CloudDesc *d, const float *dist, int mean_k,
                                                                 double stddev_mul, double *stats) {
  __shared__ __align__(16) float s_d[2][STATS_CHUNK];
  const int b = blockIdx.x;
  const int n = d[b].N;
  if (n <= mean_k) {
    if (threadIdx.x == 0) gpdb_outlier_stats(0.0, 0.0, n, mean_k, stddev_mul, stats + 3 * (size_t)b);
    return;
  }
  double sum = 0.0, sq = 0.0;
  ordered_fold<STATS_THREADS, STATS_CHUNK>(dist + d[b].off, n, s_d,
                                           [&](float v) { gpdb_outlier_stats_add(&sum, &sq, v); });
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

// outliers_remove_batch up to its result; an error may come after the store has been partly rewritten
int remove_batch(gpdb_ctx *ctx, CloudSet &s, int mean_k, double stddev_mul, int *off, double *stats, uint8_t *kept) {
  const int B = s.n, N = s.points(), k = mean_k + 1;
  const size_t n = (size_t)N;
  double *d_stats, *nrm2;
  float *xyz2, *dist;
  int *flag, *pos, *src2, *d_cnt;
  uint8_t *d_kept, *cam2;
  // xyz2 / nrm2 / src2 / cam2: the kept points, gathered
  if (!gpdb_carve(ctx, SCR_OUTLIERS, [&](Carve &c) {
        d_stats = c.take<double>(3 * (size_t)B); nrm2 = c.take<double>(3 * n); xyz2 = c.take<float>(3 * n);
        dist = c.take<float>(n); flag = c.take<int>(n + 1); pos = c.take<int>(n + 1); src2 = c.take<int>(n);
        d_cnt = c.take<int>(2 * (size_t)B);  // kept counts [B], then the camera flags [B]: one memset, one read-back
        d_kept = c.take<uint8_t>(n); cam2 = c.take<uint8_t>(n);
      }))
    return GPDB_ERR_CUDA;
  int *partial = d_cnt + B;
  int *nbr = (int *)gpdb_scratch(ctx, SCR_NBR, sizeof(int) * n * k);  // shared with the normal refinement
  if (!nbr) return GPDB_ERR_CUDA;
  int rc;
  // the camera fields of the descriptors, for the reinstall; read back with the counts
  std::vector<CloudDesc> desc((size_t)B);
  std::vector<int> cnt(2 * (size_t)B);  // counts, then the camera flags
  CUDA_TRY(cudaMemcpyAsync(desc.data(), s.desc, sizeof(CloudDesc) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(d_cnt, 0, sizeof(int) * 2 * (size_t)B, ctx->stream));
  const int nb = (N + TB - 1) / TB;
  if ((rc = refine_knn_lists(ctx, s, k, nbr)) != GPDB_OK) return rc;
  if (N > 0) {
    k_outlier_mean<<<nb, TB, 0, ctx->stream>>>(s.desc, B, N, s.xyz, nbr, mean_k, dist);
    LAUNCH_CHECK();
  }
  k_outlier_stats<<<B, STATS_THREADS, 0, ctx->stream>>>(s.desc, dist, mean_k, stddev_mul, d_stats);
  LAUNCH_CHECK();
  if (N > 0) {
    k_outlier_mark<<<nb, TB, 0, ctx->stream>>>(s.desc, B, N, dist, d_stats, s.cam, flag, d_kept, d_cnt, partial);
    LAUNCH_CHECK();
    if ((rc = scan_flags(ctx, flag, pos, N)) != GPDB_OK) return rc;
    k_outlier_gather<<<nb, TB, 0, ctx->stream>>>(N, flag, pos, s.xyz, s.nrm, s.cam, s.src, xyz2, nrm2, cam2, src2);
    LAUNCH_CHECK();
  }
  CUDA_TRY(cudaMemcpyAsync(cnt.data(), d_cnt, sizeof(int) * 2 * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  if (stats) CUDA_TRY(cudaMemcpyAsync(stats, d_stats, sizeof(double) * 3 * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  if (kept && N > 0) CUDA_TRY(cudaMemcpyAsync(kept, d_kept, (size_t)N, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  off[0] = 0;
  for (int b = 0; b < B; b++) {
    off[b + 1] = off[b] + cnt[b];
    desc[b].all_seen = !cnt[B + b];  // as batch_pack_cameras computes it for the kept points
  }
  const size_t n2 = (size_t)off[B];
  const bool has_src = s.has_src;
  CUDA_TRY(cudaMemcpyAsync(s.xyz, xyz2, sizeof(float) * 3 * n2, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(s.nrm, nrm2, sizeof(double) * 3 * n2, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(s.cam, cam2, n2, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(s.src, src2, sizeof(int) * n2, cudaMemcpyDeviceToDevice, ctx->stream));
  if ((rc = gpdb_install_clouds(ctx, s, desc.data(), off, B, true)) != GPDB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  s.has_src = has_src;  // the raw offsets stay: src still indexes each cloud's raw points
  return B;
}

// Removes the statistical outliers of every cloud of store s with mean_k neighbours (1..127) and reinstalls the kept
// points (grids, nonunit and all_seen flags as an install of them computes them; sample positions dropped; the source
// indices and has_src kept). off[B+1] (host) receives the new point offsets; stats[3B] (host, may be null) each cloud's
// mean, stddev and threshold; kept (host, may be null) one byte per point before the call. Returns B, or an error after
// which s holds no cloud (s.n = 0), as after a failed install.
int outliers_remove_batch(gpdb_ctx *ctx, CloudSet &s, int mean_k, double stddev_mul, int *off, double *stats,
                          uint8_t *kept) {
  const int rc = remove_batch(ctx, s, mean_k, stddev_mul, off, stats, kept);
  if (rc < 0) {  // whatever step failed, the store holds no cloud, as after a failed install
    s.n = 0;
    s.has_src = false;
  }
  return rc;
}

}  // namespace

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

// gpdb_remove_outliers / gpdb_remove_outliers_clouds: the state and argument checks, then outliers_remove_batch on the
// single cloud (single) or the batch. It reinstalls the store: the batch loses its SIS record, and any failure after the
// checks leaves no cloud (no batch: gpdb_drop_batch), as a failed install does. Returns the kept points (single) or B.
static int outliers_entry(gpdb_ctx *ctx, const char *name, bool single, int32_t mean_k, double stddev_mul,
                          int32_t *offsets_out, double *stats_out, uint8_t *kept_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  CloudSet &s = single ? ctx->one : ctx->many;
  int rc = single ? gpdb_check_state(ctx, true, false)
                  : gpdb_need_batch(ctx, name, "gpdb_set_clouds / gpdb_preprocess_clouds / gpdb_preprocess_depth");
  if (rc != GPDB_OK) return rc;
  if (mean_k < 1 || mean_k > GPDB_OUTLIERS_MAX_K) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: mean_k must lie in 1..%d (got %d)", name, GPDB_OUTLIERS_MAX_K, (int)mean_k);
    return GPDB_ERR_INVALID;
  }
  if (!std::isfinite(stddev_mul)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: stddev_mul must be finite", name);
    return GPDB_ERR_INVALID;
  }
  std::vector<int> off((size_t)s.n + 1);
  const cudaError_t e = cudaSetDevice(ctx->device);
  if (e != cudaSuccess) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "%s: cudaSetDevice -> %s", name, cudaGetErrorString(e));
    rc = GPDB_ERR_CUDA;
  } else {
    rc = outliers_remove_batch(ctx, s, mean_k, stddev_mul, off.data(), stats_out, kept_out);
  }
  if (rc < 0) {
    s.n = 0;
    s.has_src = false;
    if (!single) gpdb_drop_batch(ctx);
    return rc;
  }
  if (!single) sis_forget(ctx);  // the SIS positions describe clouds that are gone
  if (offsets_out) std::copy(off.begin(), off.end(), offsets_out);
  if (!single) return rc;
  if (off[1] == 0) s.n = 0;  // no point kept: no cloud, as gpdb_preprocess when its filter keeps none
  return off[1];
}

extern "C" {

int gpdb_remove_outliers(gpdb_ctx *ctx, int32_t mean_k, double stddev_mul, double stats_out[3], uint8_t *kept_out) {
  return outliers_entry(ctx, "gpdb_remove_outliers", true, mean_k, stddev_mul, nullptr, stats_out, kept_out);
}

int gpdb_remove_outliers_clouds(gpdb_ctx *ctx, int32_t mean_k, double stddev_mul, int32_t *offsets_out,
                                double *stats_out, uint8_t *kept_out) {
  return outliers_entry(ctx, "gpdb_remove_outliers_clouds", false, mean_k, stddev_mul, offsets_out, stats_out, kept_out);
}

}  // extern "C"
