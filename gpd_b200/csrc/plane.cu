// plane.cu — the support-plane segmentation of Cloud::sampleAbovePlane on the device (include/gpd_b200_plane.h).
//
//   k_plane_hyp    one thread per (cloud, hypothesis): its first good sample of 1000 attempts and the plane through it.
//                  Hypotheses do not depend on one another, so every one a call may evaluate is drawn at once.
//   k_plane_count  a grid of (cloud, point tile): each CTA holds all of its cloud's hypotheses in shared memory and counts
//                  the inliers of each over its tile; block sums go to integer atomics, so the counts are exact.
//   k_plane_pick   one thread per cloud: RandomSampleConsensus::computeModel's loop replayed over the counts.
//   k_plane_refit  one CTA per cloud: the inliers of the best hypothesis gathered in index order, the ordered float32
//                  sums of computeMeanAndCovarianceMatrix and pcl::eigen33 (the k_normals code, pcl_eigen33.cuh).
//   k_plane_mark   one thread per point: the final threshold test, the eligible bytes, per-cloud inlier counts.
// Compiled with -fmad=false: every float32 / float64 operation of the specification is rounded on its own.
// The entry points gpdb_segment_plane and gpdb_segment_planes[_device], with their checks, follow the kernels.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cub/cub.cuh>
#include <vector>

#include "../../include/gpd_b200_plane.h"
#include "common.cuh"

namespace {

#include "pcl_eigen33.cuh"

constexpr int CNT_THREADS = 256;
constexpr int CNT_PPT = 8;                            // points per thread of k_plane_count
constexpr int CNT_TILE = CNT_THREADS * CNT_PPT;       // points per CTA
constexpr int HMAX = GPDB_PLANE_MAX_ITERATIONS + 1;   // hypotheses a call may evaluate
constexpr int REFIT_THREADS = 256;
constexpr int REFIT_PPT = 8;
constexpr int REFIT_CHUNK = REFIT_THREADS * REFIT_PPT;

// inlier test of rule 3: (double)dist < threshold is dist <= tf, tf the largest float below the threshold (host)
__device__ __forceinline__ bool plane_inlier(const float4 &c, float x, float y, float z, float tf) {
  const float cf[4] = {c.x, c.y, c.z, c.w};
  return gpdb_plane_dist(cf, x, y, z) <= tf;
}

// hyp[b*H + h] = the plane of hypothesis h; cnt[b*H + h] = 0, or -1 when its 1000 attempts are all bad (or N < 3);
// nh[b] (H on entry) drops to the first such h
__global__ void k_plane_hyp(const float *xyz, const int *off, int B, int H, unsigned long long seed, float4 *hyp, int *cnt,
                            int *nh) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)B * H) return;
  const int b = (int)(t / H), h = (int)(t % H);
  const int o = off[b], n = off[b + 1] - o;
  const unsigned long long key = seed + (unsigned long long)b;
  bool good = false;
  float coef[4] = {0.f, 0.f, 0.f, 0.f};
  if (n >= 3) {
    for (uint32_t a = 0; a < GPDB_PLANE_SAMPLE_CHECKS && !good; a++) {
      uint32_t idx[3];
      gpdb_plane_sample(gpdb_plane_draw(key, (uint32_t)h, a), (uint32_t)n, idx);
      float p[3][3];
      for (int k = 0; k < 3; k++)
        for (int r = 0; r < 3; r++) p[k][r] = xyz[3 * ((size_t)o + idx[k]) + r];
      good = gpdb_plane_model(p[0], p[1], p[2], coef);
    }
  }
  hyp[t] = make_float4(coef[0], coef[1], coef[2], coef[3]);
  cnt[t] = good ? 0 : -1;
  if (!good) atomicMin(nh + b, h);
}

// cnt[b*H + h] += inliers of hypothesis h < nh[b] among points [tile * CNT_TILE, +CNT_TILE) of cloud b = blockIdx.x
__global__ void __launch_bounds__(CNT_THREADS) k_plane_count(const float *xyz, const int *off, int H, const float4 *hyp,
                                                            const int *nh, float tf, int *cnt) {
  __shared__ float4 s_hyp[HMAX];
  __shared__ int s_cnt[HMAX];
  const int b = blockIdx.x;
  const int o = off[b], n = off[b + 1] - o;
  const int base = blockIdx.y * CNT_TILE;
  if (base >= n) return;
  const int nb = nh[b];
  for (int h = threadIdx.x; h < nb; h += CNT_THREADS) {
    s_hyp[h] = hyp[(size_t)b * H + h];
    s_cnt[h] = 0;
  }
  float px[CNT_PPT], py[CNT_PPT], pz[CNT_PPT];
#pragma unroll
  for (int k = 0; k < CNT_PPT; k++) {
    const int j = base + k * CNT_THREADS + threadIdx.x;
    if (j < n) {
      const float *q = xyz + 3 * ((size_t)o + j);
      px[k] = q[0], py[k] = q[1], pz[k] = q[2];
    } else {
      px[k] = py[k] = pz[k] = __int_as_float(0x7fc00000);  // NaN: never an inlier
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int h = 0; h < nb; h++) {
    const float4 c = s_hyp[h];
    unsigned m = 0;
#pragma unroll
    for (int k = 0; k < CNT_PPT; k++) m += plane_inlier(c, px[k], py[k], pz[k], tf) ? 1u : 0u;
    m = __reduce_add_sync(0xffffffffu, m);
    if (lane == 0 && m) atomicAdd(s_cnt + h, (int)m);
  }
  __syncthreads();
  for (int h = threadIdx.x; h < nb; h += CNT_THREADS)
    if (s_cnt[h]) atomicAdd(cnt + (size_t)b * H + h, s_cnt[h]);
}

// rule 4 per cloud: pick[2b] = the best hypothesis (-1: the fit failed), pick[2b+1] = hypotheses evaluated
__global__ void k_plane_pick(const int *off, int B, int H, const int *cnt, int max_iterations, double one_minus_p,
                             int *pick) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int n = off[b + 1] - off[b];
  int best = INT_MIN, bh = -1, ev = 0;
  double q = 1.0, qp = 1.0;  // qp = q^(h+1)
  for (int h = 0; h < H; h++) {
    const int c = cnt[(size_t)b * H + h];
    if (c < 0) break;
    ev = h + 1;
    if (c > best) {
      best = c;
      bh = h;
      const double w = (double)c * (1.0 / (double)n);
      q = 1.0 - (w * w) * w;
      q = fmin(fmax(q, DBL_EPSILON), 1.0 - DBL_EPSILON);
      qp = 1.0;
      for (int i = 0; i <= h; i++) qp = qp * q;
    } else {
      qp = qp * q;
    }
    if (h + 1 > max_iterations || !(qp > one_minus_p)) break;
  }
  pick[2 * b] = bh;
  pick[2 * b + 1] = ev;
}

// rule 5 per cloud (blockIdx.x): planes[b] = the refined plane of the best hypothesis, the hypothesis itself with 3 or
// fewer inliers, NaN when the fit failed
__global__ void __launch_bounds__(REFIT_THREADS) k_plane_refit(const float *xyz, const int *off, int H, const float4 *hyp,
                                                              const int *pick, float tf, float4 *planes) {
  typedef cub::BlockScan<int, REFIT_THREADS> Scan;
  __shared__ typename Scan::TempStorage s_scan;
  __shared__ __align__(16) float s_p[3][REFIT_CHUNK];
  __shared__ int s_n;
  __shared__ float s_acc[9];
  const int b = blockIdx.x;
  const int o = off[b], n = off[b + 1] - o;
  const int bh = pick[2 * b];
  if (bh < 0) {
    if (threadIdx.x == 0) {
      const float nan = __int_as_float(0x7fc00000);
      planes[b] = make_float4(nan, nan, nan, nan);
    }
    return;
  }
  const float4 c = hyp[(size_t)b * H + bh];
  // lanes 0..8 of warp 0 own accu[0..8] = xx xy xz yy yz zz x y z (computeMeanAndCovarianceMatrix); the plain sums
  // multiply by 1.0f, which is exact
  const int lane = threadIdx.x;
  const int ia = (lane == 3 || lane == 4 || lane == 7) ? 1 : ((lane == 5 || lane == 8) ? 2 : 0);
  const int ib = (lane == 1 || lane == 3) ? 1 : ((lane == 2 || lane == 4 || lane == 5) ? 2 : (lane == 0 ? 0 : -1));
  float acc = 0.0f;
  int total = 0;
  for (int c0 = 0; c0 < n; c0 += REFIT_CHUNK) {
    // thread t owns points c0 + t*PPT .. +PPT-1: the exclusive scan of its inlier count is where they go, in index order
    float q[REFIT_PPT][3];
    bool in[REFIT_PPT];
    int m = 0;
#pragma unroll
    for (int k = 0; k < REFIT_PPT; k++) {
      const int j = c0 + threadIdx.x * REFIT_PPT + k;
      in[k] = false;
      if (j < n) {
        const float *p = xyz + 3 * ((size_t)o + j);
        q[k][0] = p[0], q[k][1] = p[1], q[k][2] = p[2];
        in[k] = plane_inlier(c, q[k][0], q[k][1], q[k][2], tf);
      }
      m += in[k];
    }
    int at, chunk_n;
    Scan(s_scan).ExclusiveSum(m, at, chunk_n);
#pragma unroll
    for (int k = 0; k < REFIT_PPT; k++)
      if (in[k]) {
        s_p[0][at] = q[k][0], s_p[1][at] = q[k][1], s_p[2][at] = q[k][2];
        at++;
      }
    __syncthreads();
    if (lane < 9) {
      const float *pa = s_p[ia];
      const float *pb = s_p[ib < 0 ? 0 : ib];
      const bool prod = ib >= 0;
      // strictly ascending k, four at a time from 16-byte loads; every product rounded before it is added
      int k = 0;
      for (; k + 4 <= chunk_n; k += 4) {
        const float4 a4 = *reinterpret_cast<const float4 *>(pa + k);
        float4 b4 = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
        if (prod) b4 = *reinterpret_cast<const float4 *>(pb + k);
        acc += a4.x * b4.x;
        acc += a4.y * b4.y;
        acc += a4.z * b4.z;
        acc += a4.w * b4.w;
      }
      for (; k < chunk_n; k++) acc += pa[k] * (prod ? pb[k] : 1.0f);
    }
    total += chunk_n;
    __syncthreads();
  }
  if (lane < 9) s_acc[lane] = acc / (float)total;
  if (threadIdx.x == 0) s_n = total;
  __syncthreads();
  if (threadIdx.x != 0) return;
  if (s_n <= 3) {  // optimizeModelCoefficients: not enough inliers, the coefficients stay
    planes[b] = c;
    return;
  }
  const float *a9 = s_acc;
  float cov[3][3];
  cov[0][0] = a9[0] - a9[6] * a9[6];
  cov[0][1] = a9[1] - a9[6] * a9[7];
  cov[0][2] = a9[2] - a9[6] * a9[8];
  cov[1][1] = a9[3] - a9[7] * a9[7];
  cov[1][2] = a9[4] - a9[7] * a9[8];
  cov[2][2] = a9[5] - a9[8] * a9[8];
  cov[1][0] = cov[0][1];
  cov[2][0] = cov[0][2];
  cov[2][1] = cov[1][2];
  float nv[3];
  pcl_eigen33_smallest(cov, nv);
  const float d = -((nv[0] * a9[6] + nv[1] * a9[7]) + nv[2] * a9[8]);
  planes[b] = make_float4(nv[0], nv[1], nv[2], d);
}

// rule 6: eligible[g] = point g is not a final inlier of its cloud's plane (a failed fit's NaN plane has none);
// fin[b] += the final inliers of cloud b
__global__ void __launch_bounds__(256) k_plane_mark(const float *xyz, const int *off, int B, int N, const float4 *planes,
                                                    float tf, uint8_t *eligible, int *fin) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = g < N;
  int b = -1;
  bool in = false;
  if (live) {
    b = csr_owner(off, B, g);
    const float *p = xyz + 3 * (size_t)g;
    in = plane_inlier(planes[b], p[0], p[1], p[2], tf);
    if (eligible) eligible[g] = in ? 0 : 1;
  }
  // one atomic per run of a cloud's points in the warp
  const unsigned same = __match_any_sync(0xffffffffu, b);
  const unsigned hits = __ballot_sync(0xffffffffu, in) & same;
  if (live && hits && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(fin + b, __popc(hits));
}

// Segments every cloud of store s (cloud b with key pp.seed + b): planes[4B], n_inliers[B] and n_hyp[B] (may be null) are
// host arrays, d_eligible (N bytes or null) device memory. Returns B.
int plane_segment_batch(gpdb_ctx *ctx, const CloudSet &s, const gpdb_plane_params &pp, float *planes, int *n_inliers,
                        int *n_hyp, uint8_t *d_eligible) {
  const int B = s.n, N = s.points(), H = pp.max_iterations + 1;
  // (double)dist < threshold <=> dist <= tf for every float dist
  float tf = (float)pp.distance_threshold;
  if ((double)tf >= pp.distance_threshold) tf = nextafterf(tf, -INFINITY);
  int largest = 0;
  for (int b = 0; b < B; b++) largest = std::max(largest, s.off[b + 1] - s.off[b]);
  const size_t BH = (size_t)B * H;
  float4 *hyp, *d_planes;
  int *cnt, *d_off, *nh, *pick, *fin;
  if (!gpdb_carve(ctx, SCR_PLANE, [&](Carve &c) {
        hyp = c.take<float4>(BH); d_planes = c.take<float4>(B); cnt = c.take<int>(BH);
        d_off = c.take<int>((size_t)B + 1); nh = c.take<int>(B); pick = c.take<int>(2 * (size_t)B);
        fin = c.take<int>(B);
      }))
    return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(d_off, s.off, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  std::vector<int> h_nh((size_t)B, H);
  CUDA_TRY(cudaMemcpyAsync(nh, h_nh.data(), sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(fin, 0, sizeof(int) * (size_t)B, ctx->stream));
  const int tb = 256;
  k_plane_hyp<<<(unsigned)((BH + tb - 1) / tb), tb, 0, ctx->stream>>>(s.xyz, d_off, B, H, pp.seed, hyp, cnt, nh);
  LAUNCH_CHECK();
  if (largest > 0) {
    k_plane_count<<<dim3(B, (largest + CNT_TILE - 1) / CNT_TILE), CNT_THREADS, 0, ctx->stream>>>(s.xyz, d_off, H, hyp, nh,
                                                                                                tf, cnt);
    LAUNCH_CHECK();
  }
  k_plane_pick<<<(B + 127) / 128, 128, 0, ctx->stream>>>(d_off, B, H, cnt, pp.max_iterations, 1.0 - pp.probability, pick);
  LAUNCH_CHECK();
  k_plane_refit<<<B, REFIT_THREADS, 0, ctx->stream>>>(s.xyz, d_off, H, hyp, pick, tf, d_planes);
  LAUNCH_CHECK();
  if (N > 0) {
    k_plane_mark<<<(N + 255) / 256, 256, 0, ctx->stream>>>(s.xyz, d_off, B, N, d_planes, tf, d_eligible, fin);
    LAUNCH_CHECK();
  }
  std::vector<int> h_pick(2 * (size_t)B);
  CUDA_TRY(cudaMemcpyAsync(planes, d_planes, sizeof(float4) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(n_inliers, fin, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(h_pick.data(), pick, sizeof(int) * 2 * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  for (int b = 0; b < B; b++) {
    if (n_hyp) n_hyp[b] = h_pick[2 * b + 1];
    const int nb = s.off[b + 1] - s.off[b];
    // no point off the plane: every point stays eligible (a failed fit has no inlier and needs nothing)
    if (d_eligible && nb > 0 && n_inliers[b] == nb)
      CUDA_TRY(cudaMemsetAsync(d_eligible + s.off[b], 1, (size_t)nb, ctx->stream));
  }
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return B;
}

}  // namespace

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

// gpdb_segment_plane / gpdb_segment_planes[_device]: the state and argument checks, then plane_segment_batch on the
// single cloud (single) or the batch. The host twins let the eligible bytes come back through SCR_UPLOAD.
static int segment_entry(gpdb_ctx *ctx, const char *name, bool single, const gpdb_plane_params *pl, float *planes_out,
                         int32_t *n_inliers_out, int32_t *n_hyp_out, uint8_t *eligible_out, bool device) {
  if (!ctx) return GPDB_ERR_INVALID;
  CloudSet &s = single ? ctx->one : ctx->many;
  int rc = single ? gpdb_check_state(ctx, true, false)
                  : gpdb_need_batch(ctx, name, "gpdb_set_clouds / gpdb_preprocess_clouds / gpdb_preprocess_depth");
  if (rc != GPDB_OK) return rc;
  if (!pl || !planes_out || !n_inliers_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need params, %s and n_inliers_out", name, single ? "plane_out" : "planes_out");
    return GPDB_ERR_INVALID;
  }
  const char *bad = nullptr;
  if (!std::isfinite(pl->distance_threshold) || !(pl->distance_threshold > 0.0))
    bad = "distance_threshold must be finite and positive";
  else if (pl->max_iterations < 1 || pl->max_iterations > GPDB_PLANE_MAX_ITERATIONS)
    bad = "max_iterations must lie in 1..1024";
  else if (!(pl->probability > 0.0 && pl->probability < 1.0))
    bad = "probability must lie in (0, 1)";
  if (bad) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: %s", name, bad);
    return GPDB_ERR_INVALID;
  }
  if (device && (rc = gpdb_check_device_ptrs(ctx, name, {{"d_eligible_out", eligible_out}})) != GPDB_OK) return rc;
  CUDA_TRY(cudaSetDevice(ctx->device));
  const int N = s.points();
  uint8_t *d_elig = eligible_out;
  if (!device && eligible_out) {
    d_elig = (uint8_t *)gpdb_scratch(ctx, SCR_UPLOAD, (size_t)N + 16);
    if (!d_elig) return GPDB_ERR_CUDA;
  }
  rc = plane_segment_batch(ctx, s, *pl, planes_out, n_inliers_out, n_hyp_out, d_elig);
  if (rc < 0) return rc;
  if (!device && eligible_out && N > 0) {
    CUDA_TRY(cudaMemcpyAsync(eligible_out, d_elig, (size_t)N, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  return rc;
}

extern "C" {

void gpdb_plane_params_default(gpdb_plane_params *p) {
  if (!p) return;
  p->distance_threshold = 0.01;
  p->max_iterations = 50;
  p->probability = 0.99;
  p->seed = 0;
}

int gpdb_segment_plane(gpdb_ctx *ctx, const gpdb_plane_params *pl, float plane_out[4], int32_t *n_inliers_out,
                       uint8_t *eligible_out) {
  return segment_entry(ctx, "gpdb_segment_plane", true, pl, plane_out, n_inliers_out, nullptr, eligible_out, false);
}

int gpdb_segment_planes(gpdb_ctx *ctx, const gpdb_plane_params *pl, float *planes_out, int32_t *n_inliers_out,
                        int32_t *n_hypotheses_out, uint8_t *eligible_out) {
  return segment_entry(ctx, "gpdb_segment_planes", false, pl, planes_out, n_inliers_out, n_hypotheses_out, eligible_out,
                       false);
}

int gpdb_segment_planes_device(gpdb_ctx *ctx, const gpdb_plane_params *pl, float *planes_out, int32_t *n_inliers_out,
                               int32_t *n_hypotheses_out, uint8_t *d_eligible_out) {
  return segment_entry(ctx, "gpdb_segment_planes_device", false, pl, planes_out, n_inliers_out, n_hypotheses_out,
                       d_eligible_out, true);
}

}  // extern "C"
