// refine.cu — Cloud::refineNormals on the device (include/gpd_b200_refine.h).
//
//   k_refine_knn     one warp per point: shells of grid cells around the point's cell, an exact top-k of
//                    (float32 distance bits, cloud-local index) keys in shared memory, no radius bound (rule 1)
//   k_refine_cast    the float32 input normals (rule 2)
//   k_refine_iter    one thread per point of a cloud still iterating: the ordered neighbour sums, the refined normal and
//                    its error (rules 3 and 4)
//   k_refine_stop    one CTA per cloud still iterating: the sequential float32 mean of rule 4 (ordered_fold), the
//                    iteration count and the cloud's done flag, so that a batch runs its 15 iterations without reading
//                    back to the host
//   k_refine_commit  the last iterate of every cloud, cast to double, into the store (rule 5)
// The lists are N x k int32; the iterates ping-pong between two float4 arrays: iteration t reads buf[(t - 1) & 1] and
// writes buf[t & 1], so a cloud done after m iterations holds its result in buf[m & 1]. Nothing in the store changes
// before k_refine_commit. Compiled with -fmad=false: every float32 operation of the specification is rounded on its own.
// The entry points gpdb_refine_normals and gpdb_refine_normals_clouds, with their checks, follow the kernels.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <vector>

#include "../../include/gpd_b200_refine.h"
#include "common.cuh"
#include "grid.cuh"

namespace {

constexpr int KNN_WARPS = 8;
constexpr int STOP_THREADS = 256;
constexpr int STOP_CHUNK = 4096;  // errors per shared-memory stage of k_refine_stop
constexpr int KNN_SLOTS = (GPDB_REFINE_MAX_K + 31) / 32;  // list entries per lane
constexpr unsigned FULL = 0xffffffffu;
constexpr unsigned long long NO_KEY = ~0ull;

// Inserts the keys of the warp's 32 lanes (NO_KEY: none) into the ascending list keys[0..cnt) of at most L entries.
// Every lane holds cnt; a key no smaller than the L-th is dropped. Keys are distinct (they carry the point index).
__device__ __forceinline__ void knn_insert(unsigned long long *keys, int &cnt, int L, unsigned long long key, int lane) {
  unsigned m = __ballot_sync(FULL, key < (cnt < L ? NO_KEY : keys[L - 1]));
  while (m) {
    const int j = __ffs(m) - 1;
    m &= m - 1;
    const unsigned long long kk = __shfl_sync(FULL, key, j);
    if (cnt == L && kk >= keys[L - 1]) continue;  // warp-uniform: an earlier insert of this batch raised the bar
    int pos = 0;
    for (int e = lane; e < cnt; e += 32) pos += keys[e] < kk;
    pos = __reduce_add_sync(FULL, pos);
    const int nc = min(cnt + 1, L);
    unsigned long long v[KNN_SLOTS];
#pragma unroll
    for (int i = 0; i < KNN_SLOTS; i++) {
      const int e = lane + 32 * i;
      if (e < nc) v[i] = e < pos ? keys[e] : (e == pos ? kk : keys[e - 1]);
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < KNN_SLOTS; i++) {
      const int e = lane + 32 * i;
      if (e < nc) keys[e] = v[i];
    }
    __syncwarp();
    cnt = nc;
  }
}

// Rule 1 for concatenated point g = one warp: nbr[g*k + r], r < min(k, N_b), the cloud-local index of its r-th neighbour.
//
// Shell s is the set of cells whose Chebyshev distance from the point's cell c is s, clipped to the grid. A row (cy, cz)
// of the clipped cube with |cy - c.y| = s or |cz - c.z| = s lies wholly in shell s (one contiguous pts4 segment);
// any other row adds only its two end cells c.x - s and c.x + s. Every cell is visited once.
//
// Stop test after shell s, once the list is full. A point p not yet visited lies in a cell beyond the clipped cube on
// some axis a whose cube side is not at the grid's edge. With cell = 1 / inv_cell (exact in double), cell_of computes
// floor(fl(fl(v - lo) * inv_cell)): two roundings of relative error u = 2^-24 each, so a point filed under cell i lies
// within [lo + i*cell - e, lo + (i+1)*cell + e], e <= 2.1u * dim * cell, and a clamp to the grid only moves a point
// further from the cube. So |p_a - q_a| >= gap, gap = the distance in double from q to the nearest open side of the
// cube, less pad = 1e-6 * dim * cell (more than 2e). L2_Simple of p then rounds five times over non-negative terms:
// fl(d) >= gap^2 (1 - u)^5 > gap^2 (1 - 1e-6). When (double)kth < gap^2 (1 - 1e-6), every unvisited point has a float
// distance strictly above the k-th key's, whatever its index. gap must exceed 1e-12, far above the float32 subnormal
// range where the relative bounds fail. A cube that covers the whole grid has visited every point: a cloud with
// N < k and an isolated point end there.
__global__ void __launch_bounds__(KNN_WARPS * 32) k_refine_knn(DevCloud cl0, CloudTable tab, int N, int k, int *nbr) {
  __shared__ unsigned long long s_keys[KNN_WARPS][GPDB_REFINE_MAX_K];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * KNN_WARPS + warp;
  if (g >= N) return;  // warp-uniform
  const CloudDesc &D = point_cloud(tab, g);
  const DevCloud cl = local_cloud(D, cl0);
  unsigned long long *keys = s_keys[warp];
  const int L = min(k, D.N);
  const float q[3] = {cl0.xyz[3 * (size_t)g], cl0.xyz[3 * (size_t)g + 1], cl0.xyz[3 * (size_t)g + 2]};
  int c[3], dim[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    c[a] = cell_of(D, q[a], a);
    dim[a] = D.dim[a];
  }
  const double cell = 1.0 / (double)D.inv_cell;
  const double pad = 1e-6 * cell * (double)max(dim[0], max(dim[1], dim[2]));
  int cnt = 0;
  for (int s = 0;; s++) {
    int lo[3], hi[3];
    bool whole = true;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      lo[a] = max(c[a] - s, 0);
      hi[a] = min(c[a] + s, dim[a] - 1);
      whole = whole && lo[a] == 0 && hi[a] == dim[a] - 1;
    }
    const int ny = hi[1] - lo[1] + 1, nrows = ny * (hi[2] - lo[2] + 1);
    for (int r0 = 0; r0 < nrows; r0 += 32) {
      const int r = r0 + lane;
      int st[2] = {0, 0}, len[2] = {0, 0};
      if (r < nrows) {
        const int cy = lo[1] + r % ny, cz = lo[2] + r / ny;
        const int *cs = cl.cell_start + ((size_t)cz * dim[1] + cy) * dim[0];
        if (abs(cy - c[1]) == s || abs(cz - c[2]) == s) {
          st[0] = __ldg(cs + lo[0]);
          len[0] = __ldg(cs + hi[0] + 1) - st[0];
        } else {  // s > 0: the row's two end cells
          if (c[0] - s >= 0) {
            st[0] = __ldg(cs + c[0] - s);
            len[0] = __ldg(cs + c[0] - s + 1) - st[0];
          }
          if (c[0] + s < dim[0]) {
            st[1] = __ldg(cs + c[0] + s);
            len[1] = __ldg(cs + c[0] + s + 1) - st[1];
          }
        }
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        unsigned nonempty = __ballot_sync(FULL, len[h] > 0);
        while (nonempty) {
          const int j = __ffs(nonempty) - 1;
          nonempty &= nonempty - 1;
          const int rs = __shfl_sync(FULL, st[h], j), rl = __shfl_sync(FULL, len[h], j);
          for (int k0 = 0; k0 < rl; k0 += 32) {
            unsigned long long key = NO_KEY;
            if (k0 + lane < rl) {
              const float4 p = __ldg(cl0.pts4 + rs + k0 + lane);
              const float pp[3] = {p.x, p.y, p.z};
              key = ((unsigned long long)__float_as_uint(gpdb_refine_l2(q, pp)) << 32) | (unsigned)__float_as_int(p.w);
            }
            knn_insert(keys, cnt, L, key, lane);
          }
        }
      }
    }
    if (whole) break;
    if (cnt == L) {
      double gap = INFINITY;
#pragma unroll
      for (int a = 0; a < 3; a++) {
        if (lo[a] > 0) gap = fmin(gap, (double)q[a] - ((double)D.lo[a] + (double)lo[a] * cell));
        if (hi[a] < dim[a] - 1) gap = fmin(gap, ((double)D.lo[a] + (double)(hi[a] + 1) * cell) - (double)q[a]);
      }
      gap -= pad;
      const double kth = (double)__uint_as_float((unsigned)(keys[L - 1] >> 32));
      if (gap > 1e-12 && kth < gap * gap * (1.0 - 1e-6)) break;
    }
  }
  int *out = nbr + (size_t)g * k;
  for (int r = lane; r < L; r += 32) out[r] = (int)(unsigned)keys[r];
}

__global__ void k_refine_cast(const double *nrm, int N, float4 *m0) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const double *n = nrm + 3 * (size_t)g;
  m0[g] = make_float4((float)n[0], (float)n[1], (float)n[2], 0.0f);
}

// rules 3 and 4, one iteration, for every point of a cloud that is not done
__global__ void __launch_bounds__(256) k_refine_iter(const CloudDesc *d, int B, int N, const int *nbr, int k,
                                                     const int *done, const float4 *in, float4 *out, float *err) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const int b = b_cloud_of_point(d, B, g);
  if (done[b]) return;
  const int off = d[b].off, L = min(k, d[b].N);
  const int *lst = nbr + (size_t)g * k;
  float sx = 0.0f, sy = 0.0f, sz = 0.0f;
  for (int r = 0; r < L; r++) {
    const float4 m = in[off + __ldg(lst + r)];
    const float mm[3] = {m.x, m.y, m.z};
    if (gpdb_refine_finite3(mm)) {
      sx = sx + m.x;
      sy = sy + m.y;
      sz = sz + m.z;
    }
  }
  const float4 o4 = in[g];
  const float o[3] = {o4.x, o4.y, o4.z};
  float m[3];
  gpdb_refine_normal(sx, sy, sz, m);
  out[g] = make_float4(m[0], m[1], m[2], 0.0f);
  err[g] = gpdb_refine_error(o, m);
}

// rule 4 after iteration t for cloud b = blockIdx.x, unless it is done: the float32 sum of its errors in index order (one
// sequential chain, as std::accumulate), the mean, the count, the flag. A cloud without points is done at once (0).
__global__ void __launch_bounds__(STOP_THREADS) k_refine_stop(const CloudDesc *d, const float *err, int t, int *done,
                                                              int *iters) {
  __shared__ __align__(16) float s_e[2][STOP_CHUNK];
  const int b = blockIdx.x;
  if (done[b]) return;  // block-uniform: thread 0 writes the flag only after every thread has read it
  const int n = d[b].N;
  if (n == 0) {
    if (threadIdx.x == 0) done[b] = 1;
    return;
  }
  float s = 0.0f;
  ordered_fold<STOP_THREADS, STOP_CHUNK>(err + d[b].off, n, s_e, [&](float v) { s = s + v; });
  if (threadIdx.x == 0) {
    iters[b] = t;
    if (s / (float)n < GPDB_REFINE_CONVERGENCE || t >= GPDB_REFINE_MAX_ITERATIONS) done[b] = 1;
  }
}

__global__ void k_refine_commit(const CloudDesc *d, int B, int N, const int *iters, const float4 *buf0, const float4 *buf1,
                                double *nrm) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const float4 m = (iters[b_cloud_of_point(d, B, g)] & 1) ? buf1[g] : buf0[g];
  double *n = nrm + 3 * (size_t)g;
  n[0] = (double)m.x;
  n[1] = (double)m.y;
  n[2] = (double)m.z;
}

}  // namespace

int refine_knn_lists(gpdb_ctx *ctx, const CloudSet &s, int k, int *nbr) {
  const int N = s.points();
  if (N > 0) {
    k_refine_knn<<<(N + KNN_WARPS - 1) / KNN_WARPS, KNN_WARPS * 32, 0, ctx->stream>>>(s.view, s.table(), N, k, nbr);
    LAUNCH_CHECK();
  }
  return GPDB_OK;
}

// Refines the normals of every cloud of store s with k neighbours (1..128) and refreshes the descriptors' nonunit flags;
// iters[B] (host) receives each cloud's iteration count. The stored normals change only once every step before the final
// cast has succeeded. Returns B.
static int refine_normals_batch(gpdb_ctx *ctx, CloudSet &s, int k, int *iters) {
  const int B = s.n, N = s.points();
  const size_t n = (size_t)N;
  float4 *buf0, *buf1;
  float *err;
  int *done;
  if (!gpdb_carve(ctx, SCR_REFINE, [&](Carve &c) {
        buf0 = c.take<float4>(n); buf1 = c.take<float4>(n); err = c.take<float>(n);
        done = c.take<int>(2 * (size_t)B);  // done flags [B], then iteration counts [B]: one memset
      }))
    return GPDB_ERR_CUDA;
  int *d_iters = done + B;
  int *nbr = (int *)gpdb_scratch(ctx, SCR_NBR, sizeof(int) * n * k);
  if (!nbr) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemsetAsync(done, 0, sizeof(int) * 2 * (size_t)B, ctx->stream));
  const int tb = 256, nb = (N + tb - 1) / tb;
  const int rc0 = refine_knn_lists(ctx, s, k, nbr);
  if (rc0 != GPDB_OK) return rc0;
  if (N > 0) {
    k_refine_cast<<<nb, tb, 0, ctx->stream>>>(s.nrm, N, buf0);
    LAUNCH_CHECK();
  }
  for (int t = 1; t <= GPDB_REFINE_MAX_ITERATIONS; t++) {
    if (N > 0) {
      k_refine_iter<<<nb, tb, 0, ctx->stream>>>(s.desc, B, N, nbr, k, done, (t & 1) ? buf0 : buf1, (t & 1) ? buf1 : buf0,
                                                err);
      LAUNCH_CHECK();
    }
    k_refine_stop<<<B, STOP_THREADS, 0, ctx->stream>>>(s.desc, err, t, done, d_iters);
    LAUNCH_CHECK();
  }
  if (N > 0) {
    k_refine_commit<<<nb, tb, 0, ctx->stream>>>(s.desc, B, N, d_iters, buf0, buf1, s.nrm);
    LAUNCH_CHECK();
  }
  const int rc = pre_nonunit_batch(ctx, s);
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaMemcpyAsync(iters, d_iters, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return B;
}

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

// gpdb_refine_normals / gpdb_refine_normals_clouds: the state and argument checks, then refine_normals_batch on the single
// cloud (single) or the batch
static int refine_entry(gpdb_ctx *ctx, const char *name, bool single, int32_t k, int32_t *iterations_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  CloudSet &s = single ? ctx->one : ctx->many;
  int rc = single ? gpdb_check_state(ctx, true, false)
                  : gpdb_need_batch(ctx, name, "gpdb_set_clouds / gpdb_preprocess_clouds / gpdb_preprocess_depth");
  if (rc != GPDB_OK) return rc;
  if (k < 1 || k > GPDB_REFINE_MAX_K) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: k must lie in 1..%d (got %d)", name, GPDB_REFINE_MAX_K, (int)k);
    return GPDB_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(ctx->device));
  std::vector<int> iters((size_t)s.n);
  rc = refine_normals_batch(ctx, s, k, iters.data());
  if (rc < 0) return rc;
  if (iterations_out) std::copy(iters.begin(), iters.end(), iterations_out);
  return rc;
}

extern "C" {

int gpdb_refine_normals(gpdb_ctx *ctx, int32_t k, int32_t *iterations_out) {
  return refine_entry(ctx, "gpdb_refine_normals", true, k, iterations_out);
}

int gpdb_refine_normals_clouds(gpdb_ctx *ctx, int32_t k, int32_t *iterations_out) {
  return refine_entry(ctx, "gpdb_refine_normals_clouds", false, k, iterations_out);
}

}  // extern "C"
