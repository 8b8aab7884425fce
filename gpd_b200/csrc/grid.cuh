// grid.cuh — the uniform-grid neighbour search shared by geometry.cu and preprocess.cu (sm_90a).
// Cells are ordered x-fastest, so a row of cells is ONE contiguous segment of the cell-sorted point array; the
// predicate is FLANN L2_Simple<float> (frame_estimator.cpp:74, hand_search.cpp:178, image_generator.cpp:61 and
// pcl::search::KdTree inside pcl::NormalEstimationOMP, cloud.cpp:497-535).
#pragma once
#include "common.cuh"

namespace {

// G: a CloudDesc
template <class G>
__device__ __forceinline__ int cell_of(const G &P, float v, int a) {
  int c = (int)floorf((v - P.lo[a]) * P.inv_cell);
  return min(max(c, 0), P.dim[a] - 1);
}

// position of a sample: a cloud point (index < n_points: Cloud::getSampleIndices) or an arbitrary float64 position
// (index >= n_points: Cloud::setSamples / gpdb_set_samples / gpdb_set_clouds_samples)
__device__ __forceinline__ void sample_position(const DevCloud &cl, int si, double out[3]) {
  if (si < cl.n_points) {
    out[0] = (double)cl.xyz[3 * (size_t)si];
    out[1] = (double)cl.xyz[3 * (size_t)si + 1];
    out[2] = (double)cl.xyz[3 * (size_t)si + 2];
  } else {
    const double *s = cl.samples + 3 * (size_t)(si - cl.n_points);
    out[0] = s[0];
    out[1] = s[1];
    out[2] = s[2];
  }
}

// The arrays of a cloud: indices (sample indices, pts4 w bits) are local to it; pts4 positions and cell_start values
// stay store-wide.
__device__ __forceinline__ DevCloud local_cloud(const CloudDesc &D, DevCloud cl) {
  cl.xyz += 3 * (size_t)D.off;
  cl.nrm += 3 * (size_t)D.off;
  cl.cam += D.off;
  cl.cell_start += D.cell_base;
  cl.samples += 3 * (size_t)D.pos;
  cl.n_points = D.N;
  return cl;
}

// The cloud of a sample slot (get) and its arrays (local). A store of one cloud (BATCH = false): descriptor 0, whose offset
// and cell_base are 0, so its arrays are the store's own and `local` is the identity; the one-cloud instantiations carry
// no slot search and no offset arithmetic (k_hands spills more with them). Batch: the descriptor of the cloud whose CSR
// sample range holds the slot (binary search over soff), its arrays offset to that cloud.
template <bool BATCH>
struct CloudSel {
  static __device__ __forceinline__ const CloudDesc &get(const CloudTable &t, int) { return t.d[0]; }
  static __device__ __forceinline__ DevCloud local(const CloudDesc &, const DevCloud &cl) { return cl; }
};
template <>
struct CloudSel<true> {
  static __device__ __forceinline__ const CloudDesc &get(const CloudTable &t, int slot) {
    int lo = 0, hi = t.n;  // largest b with soff[b] <= slot
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(t.soff + mid) <= slot) lo = mid; else hi = mid;
    }
    return t.d[lo];
  }
  static __device__ __forceinline__ DevCloud local(const CloudDesc &D, const DevCloud &cl) { return local_cloud(D, cl); }
};
// the cloud holding concatenated point g: largest b with d[b].off <= g. A cloud without points shares its offset with the
// next cloud, so the search passes over it to the cloud that holds g.
__device__ __forceinline__ int b_cloud_of_point(const CloudDesc *d, int B, int g) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (d[mid].off <= g) lo = mid; else hi = mid;
  }
  return lo;
}
// The cloud of a concatenated point (kernels with one thread or warp per point).
__device__ __forceinline__ const CloudDesc &point_cloud(const CloudTable &t, int g) {
  return t.d[b_cloud_of_point(t.d, t.n, g)];
}

// FLANN L2_Simple<float> (float32, accumulated x,y,z in order)
__device__ __forceinline__ float l2_simple(const float q[3], float x, float y, float z) {
  float dx = q[0] - x, dy = q[1] - y, dz = q[2] - z;
  float d = dx * dx;
  d += dy * dy;
  d += dz * dz;
  return d;
}


// ------------------------------------------------------------------------------------------------
// Row segments of the grid cube around q: rows (cy,cz), each one contiguous run [start, start+len).
// Block-wide; NT threads; at most NT rows per batch. Returns total candidates of the batch.
// ------------------------------------------------------------------------------------------------
struct SegRange {
  int c0[3], c1[3], ny, nrows;
};
template <class G>
__device__ __forceinline__ SegRange seg_range(const G &P, const float q[3], float rf) {
  SegRange s;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    s.c0[a] = cell_of(P, q[a] - rf, a);
    s.c1[a] = cell_of(P, q[a] + rf, a);
  }
  s.ny = s.c1[1] - s.c0[1] + 1;
  s.nrows = s.ny * (s.c1[2] - s.c0[2] + 1);
  return s;
}
template <class G>
__device__ __forceinline__ void seg_row(const G &P, const int *cell_start, const SegRange &s, int row, int &start,
                                        int &len) {
  int cy = s.c0[1] + row % s.ny, cz = s.c0[2] + row / s.ny;
  size_t base = ((size_t)cz * P.dim[1] + cy) * P.dim[0];
  start = __ldg(cell_start + base + s.c0[0]);
  len = __ldg(cell_start + base + s.c1[0] + 1) - start;
}

// Ball scan, one warp per grid row: lanes stride over the row's contiguous point segment (coalesced float4 loads).
// body(in_range, point) is called by all 32 lanes together, so it may use warp collectives.
template <int NT, class G, class F>
__device__ __forceinline__ void scan_rows(const G &P, const DevCloud &cl, const SegRange &sr, F &&body) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int NW = NT / 32;
  // this warp owns rows warp, warp + NW, ...; the bounds of 32 of them are fetched at once (one lane each) so that
  // the dependent cell_start -> point loads cost one round trip per 32 rows, and empty rows are skipped by ballot
  for (int j0 = 0; warp + NW * j0 < sr.nrows; j0 += 32) {
    const int myrow = warp + NW * (j0 + lane);
    int st = 0, len = 0;
    if (myrow < sr.nrows) seg_row(P, cl.cell_start, sr, myrow, st, len);
    unsigned nonempty = __ballot_sync(0xffffffffu, len > 0);
    while (nonempty) {
      const int j = __ffs(nonempty) - 1;
      nonempty &= nonempty - 1;
      const int rs = __shfl_sync(0xffffffffu, st, j), rl = __shfl_sync(0xffffffffu, len, j);
      for (int k0 = 0; k0 < rl; k0 += 32) {
        const int k = k0 + lane;
        const bool in = k < rl;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in) p = __ldg(cl.pts4 + rs + k);
        body(in, p);
      }
    }
  }
}

}  // namespace
