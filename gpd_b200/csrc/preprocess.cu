// preprocess.cu — cloud preprocessing on the device (SURVEY.md 8(f).1), the step immediately before the path:
//
//   CandidatesGenerator::preprocessPointCloud (candidates_generator.cpp:14-37)
//     removeNans          (cloud.cpp:154-164)   \  k_pre_flag + scan + k_pre_compact
//     filterWorkspace     (cloud.cpp:207-266)   /
//     voxelizeCloud       (cloud.cpp:286-348)      k_bpre_bounds, k_bvox_keys, radix sorts, k_bvox_heads, k_bvox_emit
//     calculateNormalsOMP (cloud.cpp:497-535)   \  k_normals (one warp per point)
//     reverseNormals      (cloud.cpp:573-604)   /
//
// Design (not a translation of the std::set / kd-tree / OpenMP loops of the reference):
//   * voxelisation is a 63-bit key sort: points of one voxel become one run, the stable sort keeps them in index
//     order so the run head is the first-inserted point (whose camera source the reference keeps) and the normal
//     average is summed in the reference's order; the voxel set is an EXACT set (include/gpd_b200.h);
//   * normal estimation reuses the uniform grid of the hot path: one warp gathers the r-ball of its point with
//     FLANN's float32 predicate, sorts the (dist, index) keys in shared memory (bucketed rank sort) — PCL accumulates the
//     float32 covariance sums in the kd-tree's sorted order, and float32 addition does not commute — then
//     nine lanes walk the sorted list with one accumulator each (computeMeanAndCovarianceMatrix), lane 0 runs
//     pcl::eigen33's closed-form float32 solver, the viewpoint flip and reverseNormals.
// Compiled with -fmad=false: every float32 operation is rounded separately, like the oracle's.
#include <cfloat>
#include <cstdio>
#include <cstdlib>
#include <cub/cub.cuh>
#include <vector>

#include "common.cuh"
#include "grid.cuh"

namespace {

constexpr int NRM_WARPS = 4;       // warps per CTA, tier 1
constexpr int NRM_CAP1 = 1024;     // neighbours per point, tier 1 (4 warps x 26 B x 1024 = 104 KB per CTA, 2 CTAs per SM)
constexpr int NRM_CAP2 = 8192;     // tier 2: one warp per CTA (208 KB)
constexpr int NRM_BYTES_PER = 26;  // key 8 + xyz 12 + bucket group 2 + pad 2 + rank 2 (keys / group / pad are reused: sorted xyz)
constexpr int NRM_NB1 = 32;        // distance buckets, tier 1
constexpr int NRM_NB2 = 256;       // tier 2

// monotone float <-> int encoding for atomicMin / atomicMax
__device__ __forceinline__ int f2ord(float f) {
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__host__ __device__ __forceinline__ float ord2f(int i) {
  int j = i >= 0 ? i : i ^ 0x7fffffff;
#ifdef __CUDA_ARCH__
  return __int_as_float(j);
#else
  float f;
  memcpy(&f, &j, 4);
  return f;
#endif
}

// removeNans + filterWorkspace: strict inequalities of the float32 coordinates against the double bounds
__global__ void k_pre_flag(const float *xyz, int M, const double *ws, int *flag) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
  bool ok = isfinite(x) && isfinite(y) && isfinite(z);
  ok = ok && (double)x > ws[0] && (double)x < ws[1] && (double)y > ws[2] && (double)y < ws[3] && (double)z > ws[4] &&
       (double)z < ws[5];
  flag[i] = ok ? 1 : 0;
}
__global__ void k_pre_compact(const float *xyz, const int *flag, const int *pos, int M, int *keep, float *xyz1) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M || !flag[i]) return;
  int k = pos[i];
  keep[k] = i;
  xyz1[3 * (size_t)k] = xyz[3 * (size_t)i];
  xyz1[3 * (size_t)k + 1] = xyz[3 * (size_t)i + 1];
  xyz1[3 * (size_t)k + 2] = xyz[3 * (size_t)i + 2];
}
// voxel index of a point: floorVector((pt - min_pt) / cell_size), float32 (cloud.cpp:299-301)
__device__ __forceinline__ int voxel_of(float v, float mn, float cell) { return (int)floorf((v - mn) / cell); }

#include "pcl_eigen33.cuh"

// ---- k_normals -------------------------------------------------------------------------------------------
// pcl::NormalEstimationOMP::computeFeature (radius search on the whole cloud, computePointNormal,
// flipNormalTowardsViewpoint) for the first camera that sees the point (convertCameraSourceMatrixToLists,
// cloud.cpp:606-621), then reverseNormals (cloud.cpp:573-604). One warp per point.
//   tier 0: point i = blockIdx.x * WARPS + warp, capacity cap; overflowing points are appended to `ovf`
//   tier 1: the points of `ovf` (one warp per CTA, large capacity); overflow -> err[4]
// Sorting the ball by (dist, index): the squared distance is quantised into NB monotone buckets (on a surface the
// neighbour count grows linearly in d^2, so the buckets fill evenly), the arrival positions are grouped by
// bucket with a counting pass, and each key is ranked inside its own bucket only: n^2 / NB comparisons, not n^2.
// Per-warp shared memory, 26 B per neighbour: keys u64[cap] + pc float[3][cap] (arrival order), grp u16[cap]
// (arrival positions grouped by bucket) + 2 B pad, rk u16[cap] (rank of each arrival position). Once the ranks are
// known, keys / grp / pad are dead and receive the coordinates IN SORTED ORDER (sx, sy over the keys, sz over grp + pad),
// so that the ordered accumulation reads three plain arrays sequentially (16-byte loads, no index chain).
// One warp per point of the store's concatenated clouds (N = all points); the warp resolves its cloud and works on that
// cloud's arrays, grid, view points and cameras only. pts4 carries cloud-local indices in its w bits, so the (dist, index)
// keys, their order and the float32 sums do not depend on the clouds beside it. `ovf` and `nrm_out` are indexed by
// concatenated point.
template <int WARPS, int NB>
__global__ void __launch_bounds__(WARPS * 32) k_normals(DevCloud cl0, CloudTable tab, int N, float r2, float rf, int cap,
                                                        double *nrm_out, int *ovf, int *ovf_count, int tier, int *err) {
  extern __shared__ __align__(16) unsigned char nrm_dyn[];
  __shared__ int s_hist[WARPS][2 * NB + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char *base = nrm_dyn + (size_t)warp * cap * NRM_BYTES_PER;
  unsigned long long *keys = reinterpret_cast<unsigned long long *>(base);
  float *pc = reinterpret_cast<float *>(keys + cap);  // [3][cap]
  unsigned short *grp = reinterpret_cast<unsigned short *>(pc + 3 * (size_t)cap);
  unsigned short *rk = grp + 2 * (size_t)cap;                       // after grp[cap] and the pad[cap]
  float *sxy = reinterpret_cast<float *>(keys);                     // sorted x [cap] | sorted y [cap] (over keys)
  float *sz = reinterpret_cast<float *>(grp);                       // sorted z [cap] (over grp + pad)
  int *hist = s_hist[warp];      // [0..NB]: bucket starts after the scan
  int *fill = hist + NB + 1;     // [0..NB): per-bucket cursor of the grouping pass
  int g;  // concatenated point
  if (tier == 0) {
    g = blockIdx.x * WARPS + warp;
    if (g >= N) return;
  } else {
    if ((int)blockIdx.x >= *ovf_count) return;
    g = ovf[blockIdx.x];
  }
  const CloudDesc &G = point_cloud(tab, g);
  const DevCloud cl = local_cloud(G, cl0);
  const int i = g - G.off;  // index in its cloud
  const uint8_t camm = cl.cam[i];
  double *out = nrm_out + 3 * (size_t)g;
  if (camm == 0) {  // seen by no camera: the reference leaves the column uninitialised; specified as 0
    if (lane < 3) out[lane] = 0.0;
    return;
  }
  for (int b = lane; b < 2 * NB + 1; b += 32) hist[b] = 0;
  __syncwarp();
  const float q[3] = {cl.xyz[3 * (size_t)i], cl.xyz[3 * (size_t)i + 1], cl.xyz[3 * (size_t)i + 2]};
  const float bscale = (float)NB / r2;
  const SegRange sr = seg_range(G, q, rf);
  int cnt = 0;
  for (int j0 = 0; j0 < sr.nrows; j0 += 32) {
    int st = 0, len = 0;
    if (j0 + lane < sr.nrows) seg_row(G, cl.cell_start, sr, j0 + lane, st, len);
    unsigned nonempty = __ballot_sync(0xffffffffu, len > 0);
    while (nonempty) {
      const int j = __ffs(nonempty) - 1;
      nonempty &= nonempty - 1;
      const int rs = __shfl_sync(0xffffffffu, st, j), rl = __shfl_sync(0xffffffffu, len, j);
      // four 32-point chunks of the row in flight at once: the gather is bound by L2 latency, not bandwidth
      for (int k0 = 0; k0 < rl; k0 += 128) {
        float4 pv[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const int k = k0 + 32 * u + lane;
          pv[u] = (k < rl) ? __ldg(cl.pts4 + rs + k) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
          if (k0 + 32 * u >= rl) break;
          const float4 p = pv[u];
          const float d = l2_simple(q, p.x, p.y, p.z);
          const bool hit = (k0 + 32 * u + lane < rl) && d < r2;
          const unsigned m = __ballot_sync(0xffffffffu, hit);
          const int pos = cnt + __popc(m & ((1u << lane) - 1));
          if (hit && pos < cap) {
            keys[pos] = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)__float_as_int(p.w);
            pc[pos] = p.x;
            pc[cap + pos] = p.y;
            pc[2 * cap + pos] = p.z;
            atomicAdd(hist + 1 + min((int)(d * bscale), NB - 1), 1);
          }
          cnt += __popc(m);
        }
      }
    }
  }
  if (cnt > cap) {
    if (lane == 0) {
      if (tier == 0) ovf[atomicAdd(ovf_count, 1)] = g;
      else atomicAdd(err + 4, 1);
    }
    if (tier == 0) return;
    cnt = cap;
  }
  __syncwarp();
  float n[3];
  if (cnt < 3) {  // computePointNormal: fewer than 3 neighbours -> NaN normal
    n[0] = n[1] = n[2] = __int_as_float(0x7fc00000);
  } else {
    // inclusive scan of the bucket counts in place: hist[1 + b] = end of bucket b, so hist[b] = start of bucket b
    int carry = 0;
    for (int b0 = 0; b0 < NB; b0 += 32) {
      const int b = b0 + lane;
      int incl = (b < NB) ? hist[1 + b] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      if (b < NB) hist[1 + b] = carry + incl;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    __syncwarp();
    // grouping pass: arrival positions grouped by bucket (unordered inside a bucket)
    for (int a = lane; a < cnt; a += 32) {
      const int b = min((int)(__uint_as_float((unsigned)(keys[a] >> 32)) * bscale), NB - 1);
      grp[hist[b] + atomicAdd(fill + b, 1)] = (unsigned short)a;
    }
    __syncwarp();
    // rank of every key inside its bucket -> rk[arrival position] = rank in ascending (dist, index) order
    for (int s = lane; s < cnt; s += 32) {
      const int a = grp[s];
      const unsigned long long ka = keys[a];
      const int b = min((int)(__uint_as_float((unsigned)(ka >> 32)) * bscale), NB - 1);
      const int lo = hist[b], hi = hist[b + 1];
      int rank = lo;
      for (int t = lo; t < hi; t++) rank += (keys[grp[t]] < ka);
      rk[a] = (unsigned short)rank;
    }
    __syncwarp();
    // keys / grp are dead: permute the coordinates into sorted order
    for (int a = lane; a < cnt; a += 32) {
      const int r = rk[a];
      sxy[r] = pc[a];
      sxy[cap + r] = pc[cap + a];
      sz[r] = pc[2 * cap + a];
    }
    __syncwarp();
    // computeMeanAndCovarianceMatrix (float32, single pass, sorted order): lanes 0..8 own accu[0..8]
    const int ia = (lane == 3 || lane == 4 || lane == 7) ? 1 : ((lane == 5 || lane == 8) ? 2 : 0);
    const int ib = (lane == 1 || lane == 3) ? 1 : ((lane == 2 || lane == 4 || lane == 5) ? 2 : (lane == 0 ? 0 : -1));
    float acc = 0.0f;
    if (lane < 9) {
      // one loop for all nine accumulators: lanes 6..8 (plain sums) multiply by 1.0f, which is exact. Strictly
      // ascending k; every product is rounded before it is added (-fmad=false): the reference's arithmetic.
      const float *pa = ia == 2 ? sz : sxy + (size_t)ia * cap;
      const float *pb = ib == 2 ? sz : sxy + (size_t)max(ib, 0) * cap;
      const bool prod = ib >= 0;
      int k = 0;
      for (; k + 4 <= cnt; k += 4) {
        const float4 a4 = *reinterpret_cast<const float4 *>(pa + k);
        float4 b4 = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
        if (prod) b4 = *reinterpret_cast<const float4 *>(pb + k);
        acc += a4.x * b4.x;
        acc += a4.y * b4.y;
        acc += a4.z * b4.z;
        acc += a4.w * b4.w;
      }
      for (; k < cnt; k++) acc += pa[k] * (prod ? pb[k] : 1.0f);
    }
    const float fc = (float)cnt;
    acc = acc / fc;
    float a9[9];
#pragma unroll
    for (int k = 0; k < 9; k++) a9[k] = __shfl_sync(0xffffffffu, acc, k);
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
    if (lane != 0) return;
    pcl_eigen33_smallest(cov, n);
    // flipNormalTowardsViewpoint, float32, view point of the first camera that sees the point
    const int camera = __ffs((unsigned)camm) - 1;
    const float vx = (float)G.vp[camera][0] - q[0], vy = (float)G.vp[camera][1] - q[1], vz = (float)G.vp[camera][2] - q[2];
    const float cos_theta = vx * n[0] + vy * n[1] + vz * n[2];
    if (cos_theta < 0) {
      n[0] *= -1;
      n[1] *= -1;
      n[2] *= -1;
    }
  }
  if (lane != 0) return;
  double nd[3] = {(double)n[0], (double)n[1], (double)n[2]};
  bool needs_reverse = true;
  for (int j = 0; j < G.K; j++)
    if ((camm >> j) & 1) {
      const double d0 = (double)q[0] - G.vp[j][0], d1 = (double)q[1] - G.vp[j][1], d2 = (double)q[2] - G.vp[j][2];
      if (nd[0] * d0 + nd[1] * d1 + nd[2] * d2 < 0) {
        needs_reverse = false;
        break;
      }
    }
  if (needs_reverse) {
    nd[0] *= -1.0;
    nd[1] *= -1.0;
    nd[2] *= -1.0;
  }
  out[0] = nd[0];
  out[1] = nd[1];
  out[2] = nd[2];
}

// ---- filter + voxelise a batch of raw clouds (gpdb_preprocess: a batch of one) ------------------------------------

// largest b < B with off[b] <= k: the cloud of point k of a concatenation (an emptied cloud repeats its successor's offset)
__device__ __forceinline__ int seg_of(const int *off, int B, int k) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= k) lo = mid; else hi = mid;
  }
  return lo;
}
// filtered offsets: the exclusive scan of the filter flags (M + 1 entries) read at the raw offsets
__global__ void k_bpre_offsets(const int *pos, const int *roff, int B, int *foff) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b <= B) foff[b] = pos[roff[b]];
}
// pcl::getMinMax3D of every cloud, bounds[6b .. 6b+5] = min x y z, max x y z as ordered ints (atomicMin / atomicMax):
// blockIdx.x = cloud, the gridDim.y CTAs of a cloud share its points, so that one large cloud is reduced by many SMs
__global__ void __launch_bounds__(256) k_bpre_bounds(const float *xyz1, const int *foff, int *bounds) {
  __shared__ int s_b[6];
  const int b = blockIdx.x;
  if (threadIdx.x < 6) s_b[threadIdx.x] = threadIdx.x < 3 ? INT_MAX : INT_MIN;
  __syncthreads();
  int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {INT_MIN, INT_MIN, INT_MIN};
  const int end = foff[b + 1];
  for (int i = foff[b] + blockIdx.y * blockDim.x + threadIdx.x; i < end; i += gridDim.y * blockDim.x)
    for (int a = 0; a < 3; a++) {
      const int o = f2ord(xyz1[3 * (size_t)i + a]);
      mn[a] = min(mn[a], o);
      mx[a] = max(mx[a], o);
    }
  for (int a = 0; a < 3; a++) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
  }
  if ((threadIdx.x & 31) == 0)
    for (int a = 0; a < 3; a++) {
      atomicMin(s_b + a, mn[a]);
      atomicMax(s_b + 3 + a, mx[a]);
    }
  __syncthreads();
  if (threadIdx.x < 3) atomicMin(bounds + 6 * b + threadIdx.x, s_b[threadIdx.x]);
  else if (threadIdx.x < 6) atomicMax(bounds + 6 * b + threadIdx.x, s_b[threadIdx.x]);
}
// 63-bit voxel key of every filtered point, against its cloud's own minimum; cl_of[k] = cloud of filtered point k; err[0]
// counts out-of-range voxel indices, err[1] = the first cloud that has one
__global__ void k_bvox_keys(const float *xyz1, int n, const int *foff, int B, const int *bounds, float cell,
                            unsigned long long *keys, int *vals, int *cl_of, int *err) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int b = seg_of(foff, B, k);
  unsigned long long key = 0;
  for (int a = 0; a < 3; a++) {
    int c = voxel_of(xyz1[3 * (size_t)k + a], ord2f(bounds[6 * b + a]), cell);
    if (c < 0 || c >= (1 << 21)) {
      atomicAdd(err, 1);
      atomicMin(err + 1, b);
      c = max(0, min(c, (1 << 21) - 1));
    }
    key = (key << 21) | (unsigned long long)c;
  }
  keys[k] = key;
  vals[k] = k;
  cl_of[k] = b;
}
// the cloud of each entry after the (stable) key sort: the key of the second sort
__global__ void k_bvox_cloud_keys(const int *vals, const int *cl_of, int n, unsigned *ck) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) ck[s] = (unsigned)cl_of[vals[s]];
}
// the keys in the order of the cloud sort: ks[s] = keys[vals[s]]
__global__ void k_bvox_gather_keys(const unsigned long long *keys, const int *vals, int n, unsigned long long *ks) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) ks[s] = keys[vals[s]];
}
// run heads in (cloud, key, index) order, ks = the keys in that order: a new voxel where the cloud OR the key changes (two
// clouds may share a key)
__global__ void k_bvox_heads(const unsigned long long *ks, const unsigned *ck, int n, int *head) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  head[s] = (s == 0 || ck[s] != ck[s - 1] || ks[s] != ks[s - 1]) ? 1 : 0;
}
// one entry per voxel: first point (run head = smallest index: the sorts are stable) and run start; the group order key
// is the cloud above the descending first index
__global__ void k_bvox_groups(const int *head, const int *gid_incl, const int *vals, const unsigned *ck, int n, int *gfirst,
                              int *gbegin, unsigned long long *gorder_key, int *gorder_val) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || !head[s]) return;
  int g = gid_incl[s] - 1;
  gfirst[g] = vals[s];
  gbegin[g] = s;
  gorder_key[g] = ((unsigned long long)ck[s] << 32) | (0x7fffffffu - (unsigned)vals[s]);
  gorder_val[g] = g;
}
// processed offsets: cloud b's sorted entries are foff[b] .. foff[b+1]-1, so its voxels start after the heads before foff[b]
__global__ void k_bvox_offsets(const int *gid_incl, const int *foff, int B, int *poff) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b <= B) poff[b] = foff[b] == 0 ? 0 : gid_incl[foff[b] - 1];
}
// voxel point = min_pt + cell_size * v.cast<float>() (cloud.cpp:322) with the cloud's own minimum, camera source of the
// first point (cloud.cpp:325-327), src local to the cloud's raw points, normal = mean of the voxel's normals summed in
// index order (cloud.cpp:307-311,331-333) over the run in ks (the keys in sorted order), bounded by the cloud's range
__global__ void k_bvox_emit(const int *gsorted, const unsigned long long *gkeys, int U, const int *gfirst, const int *gbegin,
                            const int *vals, const unsigned long long *ks, const int *foff, const int *roff, const int *keep,
                            const float *xyz1, const int *bounds, float cell, const uint8_t *cam_in, const double *nrm_in,
                            float *xyz_out, uint8_t *cam_out, double *nrm_out, int *src_out) {
  int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= U) return;
  const int g = gsorted[o], b = (int)(gkeys[o] >> 32), k = gfirst[g], i = keep[k];
  for (int a = 0; a < 3; a++) {
    const float mn = ord2f(bounds[6 * b + a]);
    const int c = voxel_of(xyz1[3 * (size_t)k + a], mn, cell);
    const float t = cell * (float)c;
    xyz_out[3 * (size_t)o + a] = mn + t;
  }
  cam_out[o] = cam_in[i];
  src_out[o] = i - roff[b];
  if (nrm_in) {
    double acc[3] = {0.0, 0.0, 0.0};
    const unsigned long long key = ks[gbegin[g]];
    const int end = foff[b + 1];
    int s = gbegin[g];
    for (; s < end && ks[s] == key; s++) {
      const double *nn = nrm_in + 3 * (size_t)keep[vals[s]];
      acc[0] += nn[0];
      acc[1] += nn[1];
      acc[2] += nn[2];
    }
    const double cnt = (double)(s - gbegin[g]);
    nrm_out[3 * (size_t)o] = acc[0] / cnt;
    nrm_out[3 * (size_t)o + 1] = acc[1] / cnt;
    nrm_out[3 * (size_t)o + 2] = acc[2] / cnt;
  }
}
// voxelize = 0: the filtered points themselves (src local to the cloud)
__global__ void k_bgather_plain(const int *keep, int n1, const int *foff, const int *roff, int B, const float *xyz1,
                                const uint8_t *cam_in, const double *nrm_in, float *xyz_out, uint8_t *cam_out, double *nrm_out,
                                int *src_out) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n1) return;
  const int i = keep[k];
  for (int a = 0; a < 3; a++) xyz_out[3 * (size_t)k + a] = xyz1[3 * (size_t)k + a];
  cam_out[k] = cam_in[i];
  src_out[k] = i - roff[seg_of(foff, B, k)];
  if (nrm_in)
    for (int a = 0; a < 3; a++) nrm_out[3 * (size_t)k + a] = nrm_in[3 * (size_t)i + a];
}
// per cloud: any normal not of unit length (unit_normal, common.cuh) -> the descriptor's nonunit flag, cleared first
__global__ void k_bnonunit_clear(CloudDesc *d, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) d[b].nonunit = 0;
}
__global__ void k_bnonunit(const double *nrm, CloudDesc *d, int B, int N) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < N && !unit_normal(nrm + 3 * (size_t)g)) d[b_cloud_of_point(d, B, g)].nonunit = 1;
}

}  // namespace

// Normal estimation over the N points of store s (grids built): writes s.nrm.
int pre_normals_batch(gpdb_ctx *ctx, CloudSet &s, double radius) {
  const int N = s.points();
  if (N == 0) return GPDB_OK;
  const CloudTable tab = s.table();
  const float r2 = (float)(radius * radius);
  const float rf = (float)radius * 1.0001f + 1e-6f;
  int *ovf, *ovf_count;
  if (!gpdb_carve(ctx, SCR_OVF, [&](Carve &c) { ovf = c.take<int>(N); ovf_count = c.take<int>(1); }))
    return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemsetAsync(ovf_count, 0, sizeof(int), ctx->stream));
  const size_t sm1 = (size_t)NRM_WARPS * NRM_CAP1 * NRM_BYTES_PER, sm2 = (size_t)NRM_CAP2 * NRM_BYTES_PER;
  CUDA_TRY(cudaFuncSetAttribute(k_normals<NRM_WARPS, NRM_NB1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
  CUDA_TRY(cudaFuncSetAttribute(k_normals<1, NRM_NB2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
  k_normals<NRM_WARPS, NRM_NB1><<<(N + NRM_WARPS - 1) / NRM_WARPS, NRM_WARPS * 32, sm1, ctx->stream>>>(
      s.view, tab, N, r2, rf, NRM_CAP1, s.nrm, ovf, ovf_count, 0, ctx->d_err);
  LAUNCH_CHECK();
  int h_ovf = 0;
  CUDA_TRY(cudaMemcpyAsync(&h_ovf, ovf_count, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (h_ovf > 0) {
    k_normals<1, NRM_NB2><<<h_ovf, 32, sm2, ctx->stream>>>(s.view, tab, N, r2, rf, NRM_CAP2, s.nrm, ovf, ovf_count, 1,
                                                           ctx->d_err);
    LAUNCH_CHECK();
    int e4 = 0;
    CUDA_TRY(cudaMemcpyAsync(&e4, ctx->d_err + 4, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (e4) {
      CUDA_TRY(cudaMemsetAsync(ctx->d_err + 4, 0, sizeof(int), ctx->stream));
      gpdb_set_error(ctx, GPDB_ERR_CAPACITY, "normal estimation: %d points have more than %d neighbours within normals_radius %g",
                     e4, NRM_CAP2, radius);
      return GPDB_ERR_CAPACITY;
    }
  }
  return GPDB_OK;
}

int pre_bounds_batch(gpdb_ctx *ctx, const float *xyz, const int *d_off, int B, int largest, int *bounds) {
  std::vector<int> init((size_t)6 * B);
  for (int b = 0; b < B; b++)
    for (int a = 0; a < 3; a++) {
      init[6 * (size_t)b + a] = INT_MAX;
      init[6 * (size_t)b + 3 + a] = INT_MIN;
    }
  CUDA_TRY(cudaMemcpyAsync(bounds, init.data(), sizeof(int) * init.size(), cudaMemcpyHostToDevice, ctx->stream));
  const int ysplit = std::min(64, std::max(1, (largest + 8191) / 8192));  // ~8 K points per CTA in the largest cloud
  k_bpre_bounds<<<dim3(B, ysplit), 256, 0, ctx->stream>>>(xyz, d_off, bounds);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// The header of a preprocessing call in SCR_WORK_A, then `extra` bytes for the caller (h.extra, 8-byte aligned).
// Uploads the workspace, the raw offsets and the voxel error words.
int pre_batch_header(gpdb_ctx *ctx, int B, const int *roff, const gpdb_preprocess_params &pp, size_t extra, PreBatch &h) {
  if (!gpdb_carve(ctx, SCR_WORK_A, [&](Carve &c) {
        h.ws = c.take<double>(6); h.roff = c.take<int>((size_t)B + 1); h.foff = c.take<int>((size_t)B + 1);
        h.poff = c.take<int>((size_t)B + 1); h.bounds = c.take<int>(6 * (size_t)B); h.verr = c.take<int>(2);
        h.extra = c.take<unsigned char>(extra, 8);
      }))
    return GPDB_ERR_CUDA;
  const int verr0[2] = {0, INT_MAX};
  CUDA_TRY(cudaMemcpyAsync(h.ws, pp.workspace, sizeof(double) * 6, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(h.roff, roff, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(h.verr, verr0, sizeof(verr0), cudaMemcpyHostToDevice, ctx->stream));
  return GPDB_OK;
}

int scan_flags(gpdb_ctx *ctx, int *flag, int *pos, int n) {
  CUDA_TRY(cudaMemsetAsync(flag + n, 0, sizeof(int), ctx->stream));
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, flag, pos, n + 1, ctx->stream);
  void *tmp = gpdb_scratch(ctx, SCR_CUB, tmp_bytes);
  if (!tmp) return GPDB_ERR_CUDA;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flag, pos, n + 1, ctx->stream));
  ctx->launches += 2;
  return GPDB_OK;
}

// filtered offsets h.foff[b] = pos[roff[b]] from the exclusive scan pos (M + 1 entries) of the filter flags
int pre_filter_offsets(gpdb_ctx *ctx, const int *pos, const PreBatch &h, int B) {
  const int tb = 256;
  k_bpre_offsets<<<(B + 1 + tb - 1) / tb, tb, 0, ctx->stream>>>(pos, h.roff, B, h.foff);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// Filter + voxelise the raw batch (M points; cloud b owns raw points roff[b] .. roff[b+1]-1, host offsets) into the arenas
// of store s (reserved here once the output size is known). poff[B+1] (host) receives the processed offsets; a cloud the
// filter empties keeps its place with no points. d_nrm_raw may be null. Every cloud goes through the steps on its own:
// the filter keeps the clouds contiguous (the compaction preserves order), the voxel sort orders by (cloud, voxel key,
// index), each cloud's voxels are emitted with its own minimum, and src is an index into the cloud's own raw points.
int pre_filter_voxelize_batch(gpdb_ctx *ctx, CloudSet &s, const float *d_xyz_raw, const uint8_t *d_cam_raw,
                              const double *d_nrm_raw, int M, int B, const int *roff, const gpdb_preprocess_params &pp,
                              int *poff, cudaEvent_t ev_filter_done) {
  const int tb = 256;
  // ---- removeNans + filterWorkspace, one scan for all clouds
  PreBatch h;
  int rc = pre_batch_header(ctx, B, roff, pp, 0, h);
  if (rc != GPDB_OK) return rc;
  int *flag, *pos, *keep;
  float *xyz1;
  if (!gpdb_carve(ctx, SCR_WORK_B, [&](Carve &c) {
        flag = c.take<int>((size_t)M + 1); pos = c.take<int>((size_t)M + 1); keep = c.take<int>(M);
        xyz1 = c.take<float>(3 * (size_t)M);
      }))
    return GPDB_ERR_CUDA;
  k_pre_flag<<<(M + tb - 1) / tb, tb, 0, ctx->stream>>>(d_xyz_raw, M, h.ws, flag);
  LAUNCH_CHECK();
  if ((rc = scan_flags(ctx, flag, pos, M)) != GPDB_OK) return rc;  // pos[M] = number of filtered points
  k_pre_compact<<<(M + tb - 1) / tb, tb, 0, ctx->stream>>>(d_xyz_raw, flag, pos, M, keep, xyz1);
  LAUNCH_CHECK();
  if ((rc = pre_filter_offsets(ctx, pos, h, B)) != GPDB_OK) return rc;
  std::vector<int> foff((size_t)B + 1);
  CUDA_TRY(cudaMemcpyAsync(foff.data(), h.foff, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, ctx->stream));
  cudaEventRecord(ev_filter_done, ctx->stream);
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return pre_voxelize_back(ctx, s, h, foff.data(), keep, xyz1, d_cam_raw, d_nrm_raw, B, pp, poff);
}

// The back of pre_filter_voxelize_batch, after the filter: voxelise (or, with voxelize = 0, gather) the filtered points
// into the arenas of store s. foff[B+1] (host) = filtered offsets (also in h.foff), keep[k] = the raw index of filtered
// point k in the call's numbering (made cloud-local with h.roff), xyz1 [3 * foff[B]] its coordinates; d_cam_raw /
// d_nrm_raw are indexed by raw index.
int pre_voxelize_back(gpdb_ctx *ctx, CloudSet &s, const PreBatch &h, const int *foff, const int *keep, const float *xyz1,
                      const uint8_t *d_cam_raw, const double *d_nrm_raw, int B, const gpdb_preprocess_params &pp, int *poff) {
  const int tb = 256;
  const int *d_roff = h.roff, *d_foff = h.foff;
  int *d_poff = h.poff, *d_bounds = h.bounds, *d_verr = h.verr;
  const int M1 = foff[B];

  if (!pp.voxelize || M1 == 0) {
    memcpy(poff, foff, sizeof(int) * ((size_t)B + 1));
    int rc = gpdb_cloud_reserve(ctx, s, (size_t)M1, B);
    if (rc != GPDB_OK || M1 == 0) return rc;
    k_bgather_plain<<<(M1 + tb - 1) / tb, tb, 0, ctx->stream>>>(keep, M1, d_foff, d_roff, B, xyz1, d_cam_raw, d_nrm_raw,
                                                                s.xyz, s.cam, s.nrm, s.src);
    LAUNCH_CHECK();
    return GPDB_OK;
  }
  // ---- voxelizeCloud of every cloud
  const float cell = (float)pp.voxel_size;
  int largest = 0;
  for (int b = 0; b < B; b++) largest = std::max(largest, foff[b + 1] - foff[b]);
  int rc = pre_bounds_batch(ctx, xyz1, d_foff, B, largest, d_bounds);
  if (rc != GPDB_OK) return rc;
  // sort buffers: voxel keys and point indices, cloud keys, group heads / ids / first points / begins, group order
  unsigned long long *keys, *keys2, *gord_k, *gord_k2;
  int *vals, *vals2, *vals3, *cl_of, *head, *gid, *gfirst, *gbegin, *gord_v, *gord_v2;
  unsigned *ck, *ck2;
  if (!gpdb_carve(ctx, SCR_WORK_C, [&](Carve &c) {
        const size_t m = (size_t)M1;
        keys = c.take<unsigned long long>(m); keys2 = c.take<unsigned long long>(m);
        gord_k = c.take<unsigned long long>(m); gord_k2 = c.take<unsigned long long>(m); vals = c.take<int>(m);
        vals2 = c.take<int>(m); vals3 = c.take<int>(m); cl_of = c.take<int>(m); ck = c.take<unsigned>(m);
        ck2 = c.take<unsigned>(m); head = c.take<int>(m); gid = c.take<int>(m); gfirst = c.take<int>(m);
        gbegin = c.take<int>(m); gord_v = c.take<int>(m); gord_v2 = c.take<int>(m);
      }))
    return GPDB_ERR_CUDA;
  int cloud_bits = 0;
  while ((1 << cloud_bits) < B) cloud_bits++;
  k_bvox_keys<<<(M1 + tb - 1) / tb, tb, 0, ctx->stream>>>(xyz1, M1, d_foff, B, d_bounds, cell, keys, vals, cl_of, d_verr);
  LAUNCH_CHECK();
  size_t t1 = 0, t2 = 0, t3 = 0, t4 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t1, keys, keys2, vals, vals2, M1, 0, 63, ctx->stream);
  if (cloud_bits) cub::DeviceRadixSort::SortPairs(nullptr, t2, ck, ck2, vals2, vals3, M1, 0, cloud_bits, ctx->stream);
  cub::DeviceScan::InclusiveSum(nullptr, t3, head, gid, M1, ctx->stream);
  cub::DeviceRadixSort::SortPairs(nullptr, t4, gord_k, gord_k2, gord_v, gord_v2, M1, 0, 32 + cloud_bits, ctx->stream);
  void *tmp = gpdb_scratch(ctx, SCR_CUB, std::max(std::max(t1, t2), std::max(t3, t4)));
  if (!tmp) return GPDB_ERR_CUDA;
  // (cloud, key, index) order: the key sort keeps index order among equal keys, the cloud sort keeps key order. keys2
  // holds the keys in the final order: the key sort leaves them so, and after a cloud sort they are gathered into its order.
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, t1, keys, keys2, vals, vals2, M1, 0, 63, ctx->stream));
  ctx->launches += 9;
  if (cloud_bits) {
    k_bvox_cloud_keys<<<(M1 + tb - 1) / tb, tb, 0, ctx->stream>>>(vals2, cl_of, M1, ck);
    LAUNCH_CHECK();
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, t2, ck, ck2, vals2, vals3, M1, 0, cloud_bits, ctx->stream));
    ctx->launches += 5;
    k_bvox_gather_keys<<<(M1 + tb - 1) / tb, tb, 0, ctx->stream>>>(keys, vals3, M1, keys2);
    LAUNCH_CHECK();
  } else {
    vals3 = vals2;
    CUDA_TRY(cudaMemsetAsync(ck2, 0, sizeof(unsigned) * (size_t)M1, ctx->stream));
  }
  k_bvox_heads<<<(M1 + tb - 1) / tb, tb, 0, ctx->stream>>>(keys2, ck2, M1, head);
  LAUNCH_CHECK();
  CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp, t3, head, gid, M1, ctx->stream));
  ctx->launches += 2;
  k_bvox_groups<<<(M1 + tb - 1) / tb, tb, 0, ctx->stream>>>(head, gid, vals3, ck2, M1, gfirst, gbegin, gord_k, gord_v);
  LAUNCH_CHECK();
  k_bvox_offsets<<<(B + 1 + tb - 1) / tb, tb, 0, ctx->stream>>>(gid, d_foff, B, d_poff);
  LAUNCH_CHECK();
  int verr[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(poff, d_poff, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(verr, d_verr, sizeof(verr), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (verr[0]) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "voxelisation: %d points fall outside the 2^21-voxel range, the first in cloud %d "
                   "(voxel_size %g too small for the cloud extent)", verr[0], verr[1], (double)cell);
    return GPDB_ERR_INVALID;
  }
  const int U = poff[B];
  // output order: cloud, then descending index of each voxel's first point
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, t4, gord_k, gord_k2, gord_v, gord_v2, U, 0, 32 + cloud_bits, ctx->stream));
  ctx->launches += 8;
  rc = gpdb_cloud_reserve(ctx, s, (size_t)U, B);
  if (rc != GPDB_OK) return rc;
  k_bvox_emit<<<(U + tb - 1) / tb, tb, 0, ctx->stream>>>(gord_v2, gord_k2, U, gfirst, gbegin, vals3, keys2, d_foff, d_roff, keep,
                                                         xyz1, d_bounds, cell, d_cam_raw, d_nrm_raw, s.xyz, s.cam, s.nrm, s.src);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// the nonunit flag of every cloud of store s, in its descriptor
int pre_nonunit_batch(gpdb_ctx *ctx, CloudSet &s) {
  const int B = s.n, N = s.points();
  k_bnonunit_clear<<<(B + 255) / 256, 256, 0, ctx->stream>>>(s.desc, B);
  LAUNCH_CHECK();
  if (N > 0) {
    k_bnonunit<<<(N + 255) / 256, 256, 0, ctx->stream>>>(s.nrm, s.desc, B, N);
    LAUNCH_CHECK();
  }
  return GPDB_OK;
}
