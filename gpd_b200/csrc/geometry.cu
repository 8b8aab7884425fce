// geometry.cu — the point-geometry kernels of the grasp-candidate path (sm_90a).
//
//   k_frames  : FrameEstimator::calculateLocalFrames  (frame_estimator.cpp:6-86, local_frame.cpp:14-41)
//   k_hands   : HandSearch::evalHands / HandSet::evalHands / FingerHand / Antipodal / Hand::construct
//               (hand_search.cpp:144-188, hand_set.cpp:31-116,235-261, finger_hand.cpp, antipodal.cpp:10-96,
//               hand.cpp:24-45) + GraspDetector::filterGraspsWorkspace/Direction (grasp_detector.cpp:334-456)
//   k_images  : ImageGenerator::createImages + Image{1,3,12,15}ChannelsStrategy (image_generator.cpp:17-99,
//               image_strategy.cpp:32-233, image_*_channels_strategy.cpp) + HandSet::calculateShadow in the
//               deterministic variant of include/gpd_b200_shadow.h
//
// Design (not a translation of the reference's per-sample OpenMP loops over Eigen temporaries):
//   * the two KdTreeFLANN builds are replaced by ONE uniform grid whose cells are ordered x-fastest, so
//     a row of cells is one contiguous segment of the cell-sorted point array: a radius search is a
//     handful of coalesced segment reads with FLANN's exact float32 predicate; no sorted result list
//     is ever materialised because every consumer is reformulated as an order-free reduction
//     (OR / min / max / arg-max / integer sums), SURVEY.md 9.6;
//   * one CTA owns one sample, its neighbourhood is staged once in shared memory and ONE WARP OWNS ONE
//     HAND POSE: all finger / deepen / closing-region / antipodal tests are warp-shuffle reductions;
//   * one CTA owns one grasp image: rasterisation into shared-memory tiles with 64-bit integer
//     atomics (arg-max key, fixed-point sum+count) => bit-reproducible, then dilate / min-max /
//     quantise in-tile.
// All float64 geometry is evaluated in the oracle's operation order; this file is compiled with
// -fmad=false so that no multiply-add is contracted (strict '<' on doubles, SURVEY.md 9.3).
#include <cfloat>
#include <climits>
#include <cstdlib>
#include <vector>
#include <cub/cub.cuh>

#include "common.cuh"
#include "grid.cuh"

namespace {

constexpr int NT_HANDS = 256;
#ifndef GPDB_NT_IMG
#define GPDB_NT_IMG 512
#endif
constexpr int NT_IMG = GPDB_NT_IMG;  // threads of k_images (one CTA per SM: 214 KB of shared memory)
constexpr int LRF_WARPS = 4;
constexpr int LRF_CAP_GLOBAL = 16384;  // last tier of k_frames: lists in global memory
constexpr int LRF_CAP = 1024;  // points of the r = nn_radius ball (dynamic shared memory: 2 x 8 B x LRF_CAP per warp)
constexpr int BOX_CAP = 2048;  // points inside one image box
constexpr int MAXPIX = 64 * 64;  // image_size <= 64

// o = frame^T v, frame column-major, summed left to right (PointList::transformToHandFrame, point_list.cpp:22-33)
__device__ __forceinline__ void to_frame(const double *F, double v0, double v1, double v2, double &o0, double &o1,
                                         double &o2) {
  o0 = (F[0] * v0 + F[1] * v1) + F[2] * v2;
  o1 = (F[3] * v0 + F[4] * v1) + F[5] * v2;
  o2 = (F[6] * v0 + F[7] * v1) + F[8] * v2;
}
__device__ __forceinline__ void mat3_mul(const double *A, const double *B, double *Cm) {
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++) Cm[c * 3 + r] = (A[r] * B[c * 3] + A[3 + r] * B[c * 3 + 1]) + A[6 + r] * B[c * 3 + 2];
}

__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_sum(int v) { return __reduce_add_sync(0xffffffffu, v); }

template <int NT>
struct SegScan {
  typedef cub::BlockScan<int, NT> Scan;
  typename Scan::TempStorage tmp;
  int start[NT];
  int prefix[NT + 1];
};
// fills seg.start/prefix for rows [row0, row0+NT) ; returns batch total. Contains __syncthreads.
template <int NT, class G>
__device__ __forceinline__ int seg_batch(const G &P, const int *cell_start, const SegRange &s, int row0,
                                         SegScan<NT> &seg) {
  int row = row0 + threadIdx.x, st = 0, len = 0;
  if (row < s.nrows) seg_row(P, cell_start, s, row, st, len);
  int excl, total;
  SegScan<NT>::Scan(seg.tmp).ExclusiveSum(len, excl, total);
  seg.start[threadIdx.x] = st;
  seg.prefix[threadIdx.x] = excl;
  if (threadIdx.x == 0) seg.prefix[NT] = total;
  __syncthreads();
  return total;
}
// Ball scan with exact load balance: the row bounds are fetched once (one thread per row), prefix-summed across
// the CTA, and every warp walks an equal share [T w / NW, T (w+1) / NW) of the flattened candidate range, row by row
// (rows are contiguous segments of the cell-sorted point array -> coalesced float4 loads, no per-candidate search).
// body(in_range, point, position in the cell-sorted array) is called by all 32 lanes together. Contains __syncthreads:
// call from uniform control flow.
template <int NT, class G, class F>
__device__ __forceinline__ void scan_balanced(const G &P, const DevCloud &cl, const SegRange &sr, SegScan<NT> &seg,
                                              F &&body) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int NW = NT / 32;
  for (int row0 = 0; row0 < sr.nrows; row0 += NT) {
    __syncthreads();
    const int total = seg_batch<NT>(P, cl.cell_start, sr, row0, seg);  // fills seg.start / seg.prefix, syncs
    const int nr = min(NT, sr.nrows - row0);
    const int c_begin = (int)(((long long)total * warp) / NW), c_end = (int)(((long long)total * (warp + 1)) / NW);
    if (c_begin >= c_end) continue;
    int lo = 0, hi = nr;  // largest r with prefix[r] <= c_begin
    while (hi - lo > 1) {
      int mid = (lo + hi) >> 1;
      if (seg.prefix[mid] <= c_begin) lo = mid; else hi = mid;
    }
    // software pipeline: the load of chunk i+1 is issued before chunk i is processed (the scan is latency bound:
    // ~10 short row segments per warp, each a dependent L2 round trip)
    int r = lo, c = c_begin;
    auto fetch = [&](bool &have, bool &in, float4 &p, int &where) {
      have = false;
      in = false;
      where = 0;
      p = make_float4(0.f, 0.f, 0.f, 0.f);
      while (c < c_end) {
        const int pe = (r + 1 < nr) ? seg.prefix[r + 1] : total;
        const int seg_end = min(pe, c_end);
        if (c >= seg_end) {  // row exhausted (or empty): next row
          r++;
          continue;
        }
        const int k = c + lane;
        in = k < seg_end;
        where = (seg.start[r] - seg.prefix[r]) + k;
        if (in) p = __ldg(cl.pts4 + where);
        c = min(c + 32, seg_end);
        have = true;
        return;
      }
    };
    bool have0, in0, have1, in1;
    float4 p0, p1;
    int w0, w1;
    fetch(have0, in0, p0, w0);
    while (have0) {
      fetch(have1, in1, p1, w1);
      body(in0, p0, w0);
      have0 = have1;
      in0 = in1;
      p0 = p1;
      w0 = w1;
    }
  }
}

template <int NT>
__device__ __forceinline__ int seg_lookup(const SegScan<NT> &seg, int c) {
  // largest r with prefix[r] <= c
  int lo = 0, hi = NT;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (seg.prefix[mid] <= c) lo = mid; else hi = mid;
  }
  return seg.start[lo] + (c - seg.prefix[lo]);
}

// ------------------------------------------------------------------------------------------------
// 3x3 symmetric eigen-solver: Eigen::SelfAdjointEigenSolver<Matrix3d>::compute restated
// (same sequence of operations as oracle/gpd_oracle.cpp eigen3 -> identical bits).
// ------------------------------------------------------------------------------------------------
__device__ void make_givens(double p, double q, double &c, double &s) {
  if (q == 0.0) {
    c = p < 0.0 ? -1.0 : 1.0;
    s = 0.0;
  } else if (p == 0.0) {
    c = 0.0;
    s = q < 0.0 ? 1.0 : -1.0;
  } else if (fabs(p) > fabs(q)) {
    double t = q / p;
    double u = sqrt(1.0 + t * t);
    if (p < 0.0) u = -u;
    c = 1.0 / u;
    s = -t * c;
  } else {
    double t = p / q;
    double u = sqrt(1.0 + t * t);
    if (q < 0.0) u = -u;
    s = -1.0 / u;
    c = -t * s;
  }
}
__device__ double eigen_hypot(double x, double y) {
  double ax = fabs(x), ay = fabs(y);
  double p = fmax(ax, ay);
  if (p == 0.0) return 0.0;
  double qp = fmin(ax, ay) / p;
  return p * sqrt(1.0 + qp * qp);
}
// m: lower triangle used, column-major; eval ascending, Q column-major
__device__ void eigen3(const double *Min, double *eval, double *Q) {
  double m00 = Min[0], m10 = Min[1], m20 = Min[2], m11 = Min[4], m21 = Min[5], m22 = Min[8];
  double scale = fmax(fmax(fmax(fabs(m00), fabs(m10)), fmax(fabs(m20), fabs(m11))), fmax(fabs(m21), fabs(m22)));
  if (scale == 0.0) scale = 1.0;
  m00 /= scale; m10 /= scale; m20 /= scale; m11 /= scale; m21 /= scale; m22 /= scale;
  double diag[3], sub[2];
  const double tol = DBL_MIN;
  diag[0] = m00;
  double v1norm2 = m20 * m20;
  if (v1norm2 <= tol) {
    diag[1] = m11;
    diag[2] = m22;
    sub[0] = m10;
    sub[1] = m21;
    for (int i = 0; i < 9; i++) Q[i] = (i % 4 == 0) ? 1.0 : 0.0;
  } else {
    double beta = sqrt(m10 * m10 + v1norm2);
    double invBeta = 1.0 / beta;
    double m01 = m10 * invBeta;
    double m02 = m20 * invBeta;
    double q = 2.0 * m01 * m21 + m02 * (m22 - m11);
    diag[1] = m11 + m02 * q;
    diag[2] = m22 - m02 * q;
    sub[0] = beta;
    sub[1] = m21 - m01 * q;
    Q[0] = 1; Q[1] = 0;   Q[2] = 0;
    Q[3] = 0; Q[4] = m01; Q[5] = m02;
    Q[6] = 0; Q[7] = m02; Q[8] = -m01;
  }
  const int n = 3;
  int end = n - 1, start = 0, iter = 0;
  const int maxIterations = 30;
  const double precision_inv = 1.0 / DBL_EPSILON;
  while (end > 0) {
    for (int i = start; i < end; ++i) {
      if (fabs(sub[i]) < DBL_MIN) {
        sub[i] = 0.0;
      } else {
        const double scaled = precision_inv * sub[i];
        if (scaled * scaled <= (fabs(diag[i]) + fabs(diag[i + 1]))) sub[i] = 0.0;
      }
    }
    while (end > 0 && sub[end - 1] == 0.0) end--;
    if (end <= 0) break;
    iter++;
    if (iter > maxIterations * n) break;
    start = end - 1;
    while (start > 0 && sub[start - 1] != 0.0) start--;
    double td = (diag[end - 1] - diag[end]) * 0.5;
    double e = sub[end - 1];
    double mu = diag[end];
    if (td == 0.0) {
      mu -= fabs(e);
    } else if (e != 0.0) {
      const double e2 = e * e;
      const double h = eigen_hypot(td, e);
      if (e2 == 0.0)
        mu -= e / ((td + (td > 0.0 ? h : -h)) / e);
      else
        mu -= e2 / (td + (td > 0.0 ? h : -h));
    }
    double x = diag[start] - mu;
    double z = sub[start];
    for (int k = start; k < end && z != 0.0; ++k) {
      double c, s;
      make_givens(x, z, c, s);
      double sdk = s * diag[k] + c * sub[k];
      double dkp1 = s * sub[k] + c * diag[k + 1];
      diag[k] = c * (c * diag[k] - s * sub[k]) - s * (c * sub[k] - s * diag[k + 1]);
      diag[k + 1] = s * sdk + c * dkp1;
      sub[k] = c * sdk - s * dkp1;
      if (k > start) sub[k - 1] = c * sub[k - 1] - s * z;
      x = sub[k];
      if (k < end - 1) {
        z = -s * sub[k + 1];
        sub[k + 1] = c * sub[k + 1];
      }
      for (int r = 0; r < 3; r++) {
        double xi = Q[k * 3 + r], yi = Q[(k + 1) * 3 + r];
        Q[k * 3 + r] = c * xi - s * yi;
        Q[(k + 1) * 3 + r] = s * xi + c * yi;
      }
    }
  }
  for (int i = 0; i < n - 1; ++i) {
    int k = 0;
    for (int j = 1; j < n - i; j++)
      if (diag[i + j] < diag[i + k]) k = j;
    if (k > 0) {
      double t = diag[i]; diag[i] = diag[k + i]; diag[k + i] = t;
      for (int r = 0; r < 3; r++) { t = Q[i * 3 + r]; Q[i * 3 + r] = Q[(k + i) * 3 + r]; Q[(k + i) * 3 + r] = t; }
    }
  }
  for (int i = 0; i < 3; i++) eval[i] = diag[i] * scale;
}

// ------------------------------------------------------------------------------------------------
// k_frames: one warp per sample. The r = nn_radius ball (~44 points) is gathered as 64-bit keys
// (dist bits << 32 | index), rank-sorted so that N*N^T and sum(n) are accumulated in exactly the
// (dist, index) order the reference's sorted radiusSearch yields -> bit-identical to the oracle.
// ------------------------------------------------------------------------------------------------
// Three tiers: tier 0 runs every sample with a small per-warp list (cap0 keys: 16 CTAs per SM instead of 3); samples whose
// ball does not fit are appended to `ovf` and re-run by tier 1 with LRF_CAP keys in shared memory; what still does not fit
// goes to `ovf2` and tier 2, whose lists live in a per-warp slice of global memory (`gkeys`, LRF_CAP_GLOBAL keys, a
// grid-stride loop over the list). Beyond that: err[0]. The reference has no limit (frame_estimator.cpp:6-86); a voxelised
// cloud never leaves tier 0 (at most ~155 voxels of 3 mm in a 1 cm ball).
template <bool BATCH>
__device__ __forceinline__ bool lrf_sample(const DevParams &P, const DevCloud &cl, const CloudTable &tab, const int *sidx, int i,
                                           unsigned long long *keys, unsigned long long *sorted, int cap, bool last, double *frames,
                                           uint8_t *valid, int *err, double *s_acc_w);

template <bool BATCH>
__global__ void __launch_bounds__(LRF_WARPS * 32) k_frames(const DevParams *Pp, DevCloud cl, CloudTable tab, const int *sidx, int n,
                                                            double *frames, uint8_t *valid, int *err, int cap, int *ovf,
                                                            int *ovf_count, int *ovf2, int *ovf2_count, unsigned long long *gkeys,
                                                            int tier) {
  const DevParams &P = *Pp;
  extern __shared__ __align__(16) unsigned char lrf_dyn[];
  __shared__ double s_acc[LRF_WARPS][9];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (tier == 2) {
    const int gw = blockIdx.x * LRF_WARPS + warp, nw = gridDim.x * LRF_WARPS, cnt2 = *ovf2_count;
    unsigned long long *keys = gkeys + (size_t)gw * 2 * cap;
    for (int j = gw; j < cnt2; j += nw) {
      lrf_sample<BATCH>(P, cl, tab, sidx, ovf2[j], keys, keys + cap, cap, true, frames, valid, err, s_acc[warp]);
      __syncwarp();
    }
    return;
  }
  int i = blockIdx.x * LRF_WARPS + warp;
  if (tier == 0) {
    if (i >= n) return;
  } else {
    if (i >= *ovf_count) return;
    i = ovf[i];
  }
  unsigned long long *keys = reinterpret_cast<unsigned long long *>(lrf_dyn) + (size_t)warp * cap;
  unsigned long long *sorted = reinterpret_cast<unsigned long long *>(lrf_dyn) + (size_t)(LRF_WARPS + warp) * cap;
  if (!lrf_sample<BATCH>(P, cl, tab, sidx, i, keys, sorted, cap, false, frames, valid, err, s_acc[warp]) && lane == 0) {
    if (tier == 0) ovf[atomicAdd(ovf_count, 1)] = i;  // re-run with the large list
    else ovf2[atomicAdd(ovf2_count, 1)] = i;          // ... with the global-memory list
  }
}

// one sample by one warp; false when the ball holds more than `cap` points and this is not the last tier (nothing written)
template <bool BATCH>
__device__ __forceinline__ bool lrf_sample(const DevParams &P, const DevCloud &cl0, const CloudTable &tab, const int *sidx, int i,
                                           unsigned long long *keys, unsigned long long *sorted, int cap, bool last, double *frames,
                                           uint8_t *valid, int *err, double *s_acc_w) {
  const int lane = threadIdx.x & 31;
  const int si = sidx[i];
  const auto &G = CloudSel<BATCH>::get(tab, i);  // geo_frames runs over the whole call: slot = i
  const DevCloud cl = CloudSel<BATCH>::local(G, cl0);
  double sp[3];
  sample_position(cl, si, sp);
  float q[3] = {(float)sp[0], (float)sp[1], (float)sp[2]};
  SegRange sr = seg_range(G, q, P.rf_lrf);
  int cnt = 0;
  for (int row = 0; row < sr.nrows; row++) {
    int st, len;
    seg_row(G, cl.cell_start, sr, row, st, len);
    for (int k0 = 0; k0 < len; k0 += 32) {
      int k = k0 + lane;
      bool hit = false;
      unsigned long long key = 0;
      if (k < len) {
        float4 p = __ldg(cl.pts4 + st + k);
        float d = l2_simple(q, p.x, p.y, p.z);
        hit = d < P.r2_lrf;
        key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)__float_as_int(p.w);
      }
      unsigned m = __ballot_sync(0xffffffffu, hit);
      int pos = cnt + __popc(m & ((1u << lane) - 1));
      if (hit && pos < cap) keys[pos] = key;
      cnt += __popc(m);
    }
  }
  if (cnt > cap) {
    if (!last) return false;
    if (lane == 0) atomicAdd(err + 0, 1);
    cnt = cap;
  }
  __syncwarp();
  if (cnt == 0) {
    if (lane == 0) valid[i] = 0;
    if (lane < 9) frames[9 * (size_t)i + lane] = 0.0;
    return true;
  }
  for (int a = lane; a < cnt; a += 32) {
    unsigned long long ka = keys[a];
    int rank = 0;
    for (int b = 0; b < cnt; b++) rank += (keys[b] < ka);
    sorted[rank] = ka;
  }
  __syncwarp();
  // lanes 0..5: lower-triangle entries of M = N N^T ; lanes 6..8: sum of normals
  if (lane < 9) {
    const int rr[9] = {0, 1, 2, 1, 2, 2, 0, 1, 2}, cc[9] = {0, 0, 0, 1, 1, 2, 0, 0, 0};
    int r = rr[lane], c = cc[lane];
    double acc = 0.0;
    for (int a = 0; a < cnt; a++) {
      int idx = (int)(unsigned)(sorted[a] & 0xffffffffu);
      const double *nn = cl.nrm + 3 * (size_t)idx;
      if (lane < 6) acc += nn[r] * nn[c]; else acc += nn[r];
    }
    s_acc_w[lane] = acc;
  }
  __syncwarp();
  if (lane == 0) {
    const double *a = s_acc_w;
    double M[9] = {a[0], a[1], a[2], a[1], a[3], a[4], a[2], a[4], a[5]};
    double eval[3], evec[9];
    eigen3(M, eval, evec);
    int mn = 0, mx = 0;
    for (int k = 1; k < 3; k++) {
      if (eval[k] < eval[mn]) mn = k;
      if (eval[k] > eval[mx]) mx = k;
    }
    double curv[3] = {evec[mn * 3], evec[mn * 3 + 1], evec[mn * 3 + 2]};
    double normal[3] = {evec[mx * 3], evec[mx * 3 + 1], evec[mx * 3 + 2]};
    double nrm = sqrt((a[6] * a[6] + a[7] * a[7]) + a[8] * a[8]);
    double avg[3] = {a[6] / nrm, a[7] / nrm, a[8] / nrm};
    if ((avg[0] * normal[0] + avg[1] * normal[1]) + avg[2] * normal[2] < 0) {
      normal[0] *= -1.0; normal[1] *= -1.0; normal[2] *= -1.0;
    }
    double *f = frames + 9 * (size_t)i;
    f[0] = normal[0]; f[1] = normal[1]; f[2] = normal[2];
    f[3] = curv[1] * normal[2] - curv[2] * normal[1];
    f[4] = curv[2] * normal[0] - curv[0] * normal[2];
    f[5] = curv[0] * normal[1] - curv[1] * normal[0];
    f[6] = curv[0]; f[7] = curv[1]; f[8] = curv[2];
    valid[i] = 1;
  }
  return true;
}

// ------------------------------------------------------------------------------------------------
// k_hands
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned slot_mask(const DevParams &P, const double *sfs, const double *sfsw, double y) {
  unsigned m = 0;
  const int F = 2 * P.nfp;
  if (P.slots_disjoint) {
    // slots within each half are disjoint, ascending and (nearly) equally spaced: estimate the slot index
    // arithmetically and test the estimate and its two neighbours with the exact table values
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const double *fs = sfs + half * P.nfp, *fsw = sfsw + half * P.nfp;
      const double tq = (y - fs[0]) * P.inv_slot_step;
      const double tf = floor(tq);
      if (tq - tf > 1e-9 && tf + 1.0 - tq > 1e-9) {
        // clearly inside one slot pitch: only that slot can contain y (one exact test)
        const int i = (int)tf;
        if (i >= 0 && i < P.nfp && y > fs[i] && y < fsw[i]) m |= 1u << (half * P.nfp + i);
      } else {
        // within rounding distance of a pitch boundary: test the estimate and both neighbours exactly
        const int e = min(max((int)tf, 1), P.nfp - 2 > 1 ? P.nfp - 2 : 1);
#pragma unroll
        for (int d = -1; d <= 1; d++) {
          const int i = e + d;
          if (i >= 0 && i < P.nfp && y > fs[i] && y < fsw[i]) m |= 1u << (half * P.nfp + i);
        }
      }
    }
  } else {
    for (int f = 0; f < F; f++)
      if (y > sfs[f] && y < sfsw[f]) m |= 1u << f;
  }
  return m;
}

constexpr int SURV_CAP = 1024;
struct HandsSmem {
  SegScan<NT_HANDS> seg;
  unsigned short surv[NT_HANDS / 32][SURV_CAP];  // per-warp closing-region member indices
  double fs[GPDB_MAX_SLOTS], fsw[GPDB_MAX_SLOTS];  // finger slot tables (copied from DevParams)
  int count;      // staged (slab) points
  int n_ball;     // all points of the r ball
  unsigned long long nb0_key;
  double T[9];    // frame * ROT_BINORMAL
  double frame[9];
  double sample[3];
  int cap;
};

// one CTA per sample; dynamic smem: float4 list[cap]
// tiers: in_list == nullptr: every sample, else the samples in_list[0 .. *in_count) (the overflow of the previous tier);
// samples whose slab does not fit `cap` go to out_list (next tier) or, in the last tier (out_list == nullptr), are an error.
// glist != nullptr: the staged neighbourhood lives in a per-CTA slice of global memory (last tier, any density up to cap).
template <bool BATCH>
__global__ void __launch_bounds__(NT_HANDS, 4) k_hands(const DevParams *Pp, DevCloud cl0, CloudTable tab, const int *sidx, int n, int slot0,
                                                    const double *frames, const uint8_t *fvalid, gpdb_pose *poses,
                                                    uint8_t *flags, int cap, const int *in_list, const int *in_count,
                                                    int *out_list, int *out_count, float4 *glist, int *err,
                                                    unsigned long long *prof) {
  const DevParams &P = *Pp;
  extern __shared__ __align__(16) unsigned char dyn[];
  float4 *list = glist ? glist + (size_t)blockIdx.x * cap : reinterpret_cast<float4 *>(dyn);
  __shared__ HandsSmem S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int work_n = in_list ? *in_count : n;
  if (tid < 2 * P.nfp) {
    S.fs[tid] = P.fs[tid];
    S.fsw[tid] = P.fsw[tid];
  }
  for (int w = blockIdx.x; w < work_n; w += gridDim.x) {
    const int i = in_list ? in_list[w] : w;
    const int si = sidx[i];
    const auto &G = CloudSel<BATCH>::get(tab, slot0 + i);
    const DevCloud cl = CloudSel<BATCH>::local(G, cl0);
    __syncthreads();
    if (tid == 0) {
      S.count = 0;
      S.n_ball = 0;
      S.nb0_key = ~0ull;
    }
    if (tid < 9) S.frame[tid] = frames[9 * (size_t)i + tid];
    if (tid == 0) sample_position(cl, si, S.sample);
    __syncthreads();
    if (tid == 0) mat3_mul(S.frame, P.rotb, S.T);
    const bool fv = fvalid[i] != 0;
    if (!fv) {
      // no local frame (calculateFrame returned nullptr): no hand set for this sample
      for (int p = tid; p < P.P; p += NT_HANDS) {
        gpdb_pose *h = poses + (size_t)i * P.P + p;
        memset(h, 0, sizeof(gpdb_pose));
        h->sample_index = si;
        h->sample_slot = slot0 + i;
        h->pose_slot = (int16_t)p;
        h->finger_idx = -1;
        h->score = __int_as_float(0x7fc00000);
        flags[(size_t)i * P.P + p] = 0;
      }
      continue;
    }
    __syncthreads();
    // ---- stage the neighbourhood: ball r = nn_radius_hs, kept if inside the (slightly widened)
    // height slab when every rotation axis is the curvature axis (z is then pose independent)
    float q[3] = {(float)S.sample[0], (float)S.sample[1], (float)S.sample[2]};
    SegRange sr = seg_range(G, q, P.rf_hs);
    const double hz = P.hand_height * 1.001 + 1e-9;
    unsigned long long best = ~0ull;
    int nball = 0;
    scan_balanced<NT_HANDS>(G, cl, sr, S.seg, [&](bool in, const float4 &p, int) {
      bool keep = false;
      if (in) {
        float d = l2_simple(q, p.x, p.y, p.z);
        if (d < P.r2_hs) {
          nball++;
          unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)__float_as_int(p.w);
          best = key < best ? key : best;
          keep = true;
          if (P.all_axes_z) {
            double z0 = (S.T[6] * ((double)p.x - S.sample[0]) + S.T[7] * ((double)p.y - S.sample[1])) +
                        S.T[8] * ((double)p.z - S.sample[2]);
            keep = fabs(z0) < hz;
          }
        }
      }
      unsigned m = __ballot_sync(0xffffffffu, keep);
      if (m) {
        int leader = __ffs(m) - 1, base = 0;
        if (lane == leader) base = atomicAdd(&S.count, __popc(m));
        base = __shfl_sync(0xffffffffu, base, leader);
        int pos = base + __popc(m & ((1u << lane) - 1));
        if (keep && pos < cap) list[pos] = p;
      }
    });
    nball = warp_sum(nball);
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
      best = ob < best ? ob : best;
    }
    if (lane == 0) {
      atomicAdd(&S.n_ball, nball);
      atomicMin(&S.nb0_key, best);
    }
    __syncthreads();
    const int m = S.count;
    if (m > cap) {
      // does not fit this tier: defer to the next one (or report)
      if (tid == 0) {
        if (out_list) {
          int k = atomicAdd(out_count, 1);
          out_list[k] = i;
          if (!in_list) atomicAdd(err + 3, 1);
        } else {
          atomicAdd(err + 1, 1);
        }
      }
      if (!out_list) {
        for (int p = tid; p < P.P; p += NT_HANDS) flags[(size_t)i * P.P + p] = 0;
      }
      continue;
    }
    const int n_ball = S.n_ball;
    // nb0 = nearest neighbour (first of the sorted radius search): pads the cropped list
    // (PointList::cropByHandHeight quirk, point_list.cpp:44-55)
    const int nb0 = (int)(unsigned)(S.nb0_key & 0xffffffffu);
    double nbx = 0, nby = 0, nbz = 0;
    if (n_ball > 0) {
      nbx = (double)cl.xyz[3 * (size_t)nb0] - S.sample[0];
      nby = (double)cl.xyz[3 * (size_t)nb0 + 1] - S.sample[1];
      nbz = (double)cl.xyz[3 * (size_t)nb0 + 2] - S.sample[2];
    }
    // ---- one warp per pose
    for (int pose = warp; pose < P.P; pose += NT_HANDS / 32) {
      gpdb_pose *h = poses + (size_t)i * P.P + pose;
      double R[9];
      mat3_mul(S.T, P.rot[pose], R);
      const double hh = P.hand_height;
      uint8_t fl = 0;
      double top = 0, bottom = 0, center = 0, width = 0;
      int fidx = -1, fpi = -1;
      bool half = false, full = false;
      double x0, y0, z0;
      to_frame(R, nbx, nby, nbz, x0, y0, z0);
      if (n_ball > 0) {
        // pass A: crop + finger masks (FingerHand::evaluateFingers, finger_hand.cpp:26-73)
        const double b0 = P.init_bite, bot0 = P.init_bite - P.hand_depth;
        int k = 0;
        unsigned anyA = 0, anyB = 0, fmask = 0;
        for (int a = lane; a < m; a += 32) {
          float4 p = list[a];
          double x, y, z;
          to_frame(R, (double)p.x - S.sample[0], (double)p.y - S.sample[1], (double)p.z - S.sample[2], x, y, z);
          if (z > -1.0 * hh && z < hh) {
            k++;
            if (x < b0) {
              anyA = 1;
              if (x < bot0) anyB = 1;
              fmask |= slot_mask(P, S.fs, S.fsw, y);
            }
          }
        }
        k = warp_sum(k);
        const int npad = n_ball - k;
        if (npad > 0 && x0 < b0) {
          anyA = 1;
          if (x0 < bot0) anyB = 1;
          fmask |= slot_mask(P, S.fs, S.fsw, y0);
        }
        anyA = __reduce_or_sync(0xffffffffu, anyA);
        anyB = __reduce_or_sync(0xffffffffu, anyB);
        fmask = __reduce_or_sync(0xffffffffu, fmask);
        const unsigned allF = (2 * P.nfp >= 32) ? 0xffffffffu : ((1u << (2 * P.nfp)) - 1);
        unsigned freef = (anyA && !anyB) ? (~fmask & allF) : 0u;
        unsigned hand = freef & (freef >> P.nfp) & ((1u << P.nfp) - 1);  // evaluateHand (:75-81)
        if (hand) {
          // chooseMiddleHand (:89-105): hand_idx[ceil(m/2) - 1]
          int cntb = __popc(hand);
          int target = (cntb + 1) / 2;  // 1-based ordinal of the chosen set bit
          unsigned hm = hand;
          while (--target) hm &= hm - 1;
          fidx = __ffs(hm) - 1;
          // Hand::construct (hand.cpp:33-38): finger_placement_index_ = FIRST set bit of hand_; deepenHand
          // resets hand_ to the eroded index only (finger_hand.cpp:134-136), chooseMiddleHand does not
          fpi = P.deepen ? fidx : (__ffs(hand) - 1);
          top = b0;
          bottom = bot0;
          if (P.deepen) {
            // deepenHand (:107-139) as one min-reduction over the first failing step
            int jf = P.J;  // 0-based index of the first failing step; J = none fails
            const double sl0 = P.fs[fidx], sl1 = P.fsw[fidx], sr0 = P.fs[P.nfp + fidx], sr1 = P.fsw[P.nfp + fidx];
            const int J = P.J;
            auto visitB = [&](double x, double y) {
              if (J > 0 && x < P.botj[J - 1]) {
                int j = 0;
                while (!(x < P.botj[j])) j++;
                jf = min(jf, j);
              }
              if ((y > sl0 && y < sl1) || (y > sr0 && y < sr1)) {
                if (J > 0 && x < P.topj[J - 1]) {
                  int j = 0;
                  while (!(x < P.topj[j])) j++;
                  jf = min(jf, j);
                }
              }
            };
            for (int a = lane; a < m; a += 32) {
              float4 p = list[a];
              double x, y, z;
              to_frame(R, (double)p.x - S.sample[0], (double)p.y - S.sample[1], (double)p.z - S.sample[2], x, y, z);
              if (z > -1.0 * hh && z < hh) visitB(x, y);
            }
            if (npad > 0) visitB(x0, y0);
            jf = __reduce_min_sync(0xffffffffu, jf);
            if (jf > 0) {
              top = P.topj[jf - 1];
              bottom = P.botj[jf - 1];
            }
          }
          // computePointsInClosingRegion (:141-171)
          const double left = P.fsw[fidx], right = P.fs[P.nfp + fidx];
          center = 0.5 * (left + right);
          int cnt = 0;
          double mny = DBL_MAX, mxy = -DBL_MAX;
          // the closing-region members (~10 % of the slab) are remembered per warp so that the two Antipodal passes
          // below visit only them instead of re-transforming the whole slab
          unsigned short *surv = S.surv[warp];
          int nsurv = 0;
          for (int a0 = 0; a0 < m; a0 += 32) {
            const int a = a0 + lane;
            bool inr = false;
            if (a < m) {
              float4 p = list[a];
              double x, y, z;
              to_frame(R, (double)p.x - S.sample[0], (double)p.y - S.sample[1], (double)p.z - S.sample[2], x, y, z);
              if (z > -1.0 * hh && z < hh && x > bottom && x < top && y > left && y < right) {
                inr = true;
                cnt++;
                mny = fmin(mny, y);
                mxy = fmax(mxy, y);
              }
            }
            const unsigned mk = __ballot_sync(0xffffffffu, inr);
            const int pos = nsurv + __popc(mk & ((1u << lane) - 1));
            if (inr && pos < SURV_CAP) surv[pos] = (unsigned short)a;
            nsurv += __popc(mk);
          }
          const bool surv_ok = nsurv <= SURV_CAP && m <= 65535;
          __syncwarp();
          const bool nb_in = npad > 0 && x0 > bottom && x0 < top && y0 > left && y0 < right;
          cnt = warp_sum(cnt) + (nb_in ? npad : 0);
          mny = warp_min(mny);
          mxy = warp_max(mxy);
          if (nb_in) {
            mny = fmin(mny, y0);
            mxy = fmax(mxy, y0);
          }
          if (cnt > 0) {
            fl |= GPDB_POSE_VALID;
            width = mxy - mny;  // modifyCandidate (hand_set.cpp:245-247)
            // Antipodal::evaluateGrasp (antipodal.cpp:10-96), lateral = 1, forward = 0, vertical = 2
            const double min_x = mny + 0.003, max_x = mxy - 0.003;
            int cl_ = 0, cr_ = 0;
            double lmaxx = -DBL_MAX, lminx = DBL_MAX, lmaxz = -DBL_MAX, lminz = DBL_MAX;
            double rmaxx = -DBL_MAX, rminx = DBL_MAX, rmaxz = -DBL_MAX, rminz = DBL_MAX;
            auto visitD = [&](double x, double y, double z, int idx, int wgt) {
              const double *nn = cl.nrm + 3 * (size_t)idx;
              double n0, n1, n2;
              to_frame(R, nn[0], nn[1], nn[2], n0, n1, n2);
              double ldot = (0.0 * n0 + -1.0 * n1) + 0.0 * n2;
              double rdot = (0.0 * n0 + 1.0 * n1) + 0.0 * n2;
              if (ldot > P.cosf && y < min_x) {
                cl_ += wgt;
                lmaxx = fmax(lmaxx, x); lminx = fmin(lminx, x); lmaxz = fmax(lmaxz, z); lminz = fmin(lminz, z);
              }
              if (rdot > P.cosf && y > max_x) {
                cr_ += wgt;
                rmaxx = fmax(rmaxx, x); rminx = fmin(rminx, x); rmaxz = fmax(rmaxz, z); rminz = fmin(rminz, z);
              }
            };
            if (surv_ok) {
              for (int sidx_ = lane; sidx_ < nsurv; sidx_ += 32) {
                float4 p = list[surv[sidx_]];
                double x, y, z;
                to_frame(R, (double)p.x - S.sample[0], (double)p.y - S.sample[1], (double)p.z - S.sample[2], x, y, z);
                visitD(x, y, z, __float_as_int(p.w), 1);
              }
            } else {
              if (prof && lane == 0) atomicAdd(prof + GPDB_PROF_PATH + PATH_HANDS_SLAB, 1ull);
              for (int a = lane; a < m; a += 32) {
                float4 p = list[a];
                double x, y, z;
                to_frame(R, (double)p.x - S.sample[0], (double)p.y - S.sample[1], (double)p.z - S.sample[2], x, y, z);
                if (z > -1.0 * hh && z < hh && x > bottom && x < top && y > left && y < right)
                  visitD(x, y, z, __float_as_int(p.w), 1);
              }
            }
            if (nb_in && lane == 0) visitD(x0, y0, z0, nb0, npad);
            cl_ = warp_sum(cl_);
            cr_ = warp_sum(cr_);
            half = cl_ > 0 || cr_ > 0;
            if (cl_ > 0 && cr_ > 0) {
              lmaxx = warp_max(lmaxx); lminx = warp_min(lminx); lmaxz = warp_max(lmaxz); lminz = warp_min(lminz);
              rmaxx = warp_max(rmaxx); rminx = warp_min(rminx); rmaxz = warp_max(rmaxz); rminz = warp_min(rminz);
              const double top_y = fmin(lmaxx, rmaxx), bot_y = fmax(lminx, rminx);
              const double top_z = fmin(lmaxz, rmaxz), bot_z = fmax(lminz, rminz);
              int nl = 0, nr = 0;
              auto visitE = [&](double x, double y, double z, int idx, int wgt) {
                const double *nn = cl.nrm + 3 * (size_t)idx;
                double n0, n1, n2;
                to_frame(R, nn[0], nn[1], nn[2], n0, n1, n2);
                double ldot = (0.0 * n0 + -1.0 * n1) + 0.0 * n2;
                double rdot = (0.0 * n0 + 1.0 * n1) + 0.0 * n2;
                bool inw = x >= bot_y && x <= top_y && z >= bot_z && z <= top_z;
                if (ldot > P.cosf && y < min_x && inw) nl += wgt;
                if (rdot > P.cosf && y > max_x && inw) nr += wgt;
              };
              if (surv_ok) {
                for (int sidx_ = lane; sidx_ < nsurv; sidx_ += 32) {
                  float4 p = list[surv[sidx_]];
                  double x, y, z;
                  to_frame(R, (double)p.x - S.sample[0], (double)p.y - S.sample[1], (double)p.z - S.sample[2], x, y, z);
                  visitE(x, y, z, __float_as_int(p.w), 1);
                }
              } else {
                for (int a = lane; a < m; a += 32) {
                  float4 p = list[a];
                  double x, y, z;
                  to_frame(R, (double)p.x - S.sample[0], (double)p.y - S.sample[1], (double)p.z - S.sample[2], x, y, z);
                  if (z > -1.0 * hh && z < hh && x > bottom && x < top && y > left && y < right)
                    visitE(x, y, z, __float_as_int(p.w), 1);
                }
              }
              if (nb_in && lane == 0) visitE(x0, y0, z0, nb0, npad);
              nl = warp_sum(nl);
              nr = warp_sum(nr);
              full = nl >= P.min_viable && nr >= P.min_viable;
            }
            if (half) fl |= GPDB_POSE_HALF;
            if (full) fl |= GPDB_POSE_FULL;
          }
        }
      }
      // ---- record (Hand::construct, hand.cpp:24-45) + A15 filters, by lane 0
      if (lane == 0) {
        gpdb_pose o;
        memset(&o, 0, sizeof(o));
        for (int r = 0; r < 3; r++) o.sample[r] = S.sample[r];
        for (int r = 0; r < 9; r++) o.frame[r] = R[r];
        o.sample_index = si;
        o.sample_slot = slot0 + i;
        o.pose_slot = (int16_t)pose;
        o.finger_idx = -1;
        o.score = __int_as_float(0x7fc00000);
        if (fl & GPDB_POSE_VALID) {
          o.top = top;
          o.bottom = bottom;
          o.center = center;
          o.width = width;
          o.finger_idx = (int16_t)fpi;
          o.half_antipodal = half;
          o.full_antipodal = full;
          for (int r = 0; r < 3; r++)
            o.position[r] = ((R[r] * bottom + R[3 + r] * center) + R[6 + r] * 0.0) + S.sample[r];
          // filterGraspsWorkspace (grasp_detector.cpp:334-398; right_top uses left_bottom, :362-363)
          const double half_width = 0.5 * P.hand_outer_diameter;
          bool ok = width >= P.min_ap && width <= P.max_ap;
          for (int r = 0; r < 3; r++) {
            double lb = o.position[r] + half_width * R[3 + r];
            double rb = o.position[r] - half_width * R[3 + r];
            double lt = lb + P.hand_depth * R[r];
            double rt = lb + P.hand_depth * R[r];
            double ap = o.position[r] - 0.05 * R[r];
            double mn = fmin(fmin(fmin(lb, rb), fmin(lt, rt)), ap);
            double mx = fmax(fmax(fmax(lb, rb), fmax(lt, rt)), ap);
            ok = ok && mn >= P.ws[2 * r] && mx <= P.ws[2 * r + 1];
          }
          if (ok && P.filt_dir) {  // filterGraspsDirection (:422-456): acos(dot) > thresh as the host evaluates it
            double dot = (P.dir[0] * R[0] + P.dir[1] * R[1]) + P.dir[2] * R[2];
            if (dot >= -1.0 && dot <= 1.0 && dot < P.dir_keep) ok = false;
          }
          if (ok) fl |= GPDB_POSE_FILTERED;
        }
        *h = o;
        flags[(size_t)i * P.P + pose] = fl;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// compaction of candidate poses (hands_out order of image_generator.cpp:91-98)
// ------------------------------------------------------------------------------------------------
__global__ void k_flag01(const uint8_t *flags, int n, int *f01) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) f01[i] = (flags[i] & 3) == 3;
}
__global__ void k_scatter(const gpdb_pose *poses, const int *f01, const int *pos, int n, gpdb_pose *cand, int *count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (f01[i]) cand[pos[i]] = poses[i];
  if (i == n - 1) *count = pos[i] + f01[i];
}
__global__ void k_scatter_scores(const gpdb_pose *cand, const float *scores, int nc, int slot0, int P, float *pose_scores,
                                 gpdb_pose *cand_out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  float s = scores[i];
  pose_scores[(size_t)(cand[i].sample_slot - slot0) * P + cand[i].pose_slot] = s;
  cand_out[i].score = s;
}

// selectGrasps (grasp_detector.cpp:405-420) on the device: sort key = descending score, stable in candidate order
__global__ void k_select_keys(const gpdb_pose *cand, int n, unsigned *keys, int *vals) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned u = __float_as_uint(cand[i].score);
  u ^= (u >> 31) ? 0xFFFFFFFFu : 0x80000000u;  // ascending float order as unsigned
  keys[i] = ~u;                                // descending
  vals[i] = i;
}
__global__ void k_gather_poses(const gpdb_pose *cand, const int *order, int k, gpdb_pose *out) {
  // one warp per record: 176-byte pose = 44 words
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= k) return;
  const int *src = reinterpret_cast<const int *>(cand + order[w]);
  int *dst = reinterpret_cast<int *>(out + w);
  for (int j = lane; j < (int)(sizeof(gpdb_pose) / 4); j += 32) dst[j] = src[j];
}

// ------------------------------------------------------------------------------------------------
// HandSearch::reevaluateHypotheses (hand_search.cpp:66-134,190-228): the given hands are re-labelled against a cloud of
// the store (GraspDetector::evalGroundTruth: a ground-truth mesh cloud). One WARP per hand; hand i belongs to the cloud
// whose group holds it (the group offsets sit in the store's soff, CloudSel). The closing-region bounds depend only on
// the record (bottom / top from its top, left / right from its finger placement), so ONE walk of the r = nn_radius_hs
// ball does the work of the reference's first two passes: neighbour 0, crop count, back-of-hand and finger tests of the
// hand's own slot at its own depth, and the closing-region count and y-extent. The same walk records the closing-region
// members (their positions in pts4) in a per-warp list in shared memory; the two Antipodal passes read that list and the
// normals. A hand whose closing region holds more than LABEL_CAP points (the neighbour-0 padding is not a member) walks
// the grid for the Antipodal passes instead (path counter 15). Every reduction is a count, a min, a max or an or, and the
// neighbour-0 padding weights are applied after them as in k_hands, so the result does not depend on the visit order.
// ------------------------------------------------------------------------------------------------
constexpr int LABEL_NT = 128;
constexpr int LABEL_CAP = 1024;  // closing-region members per warp, as k_hands' SURV_CAP

// body(in, point, pts4 position) for every grid candidate of the ball's cube, called by all 32 lanes together (so it may
// use warp collectives); in: the lane holds a point of the ball
template <class F>
__device__ __forceinline__ void warp_scan_ball(const CloudDesc &G, const DevCloud &cl, const SegRange &sr, const float q[3], float r2,
                                               F &&body) {
  const int lane = threadIdx.x & 31;
  for (int j0 = 0; j0 < sr.nrows; j0 += 32) {
    const int myrow = j0 + lane;
    int st = 0, len = 0;
    if (myrow < sr.nrows) seg_row(G, cl.cell_start, sr, myrow, st, len);
    unsigned nonempty = __ballot_sync(0xffffffffu, len > 0);
    while (nonempty) {
      const int j = __ffs(nonempty) - 1;
      nonempty &= nonempty - 1;
      const int rs = __shfl_sync(0xffffffffu, st, j), rl = __shfl_sync(0xffffffffu, len, j);
      for (int k0 = 0; k0 < rl; k0 += 32) {
        const int k = k0 + lane;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < rl) p = __ldg(cl.pts4 + rs + k);
        body(k < rl && l2_simple(q, p.x, p.y, p.z) < r2, p, rs + k);
      }
    }
  }
}

template <bool BATCH>
__global__ void __launch_bounds__(LABEL_NT) k_label(const DevParams *Pp, DevCloud cl0, CloudTable tab, gpdb_pose *hands, int n,
                                                    int *labels, unsigned long long *prof) {
  __shared__ int members[LABEL_NT / 32][LABEL_CAP];  // per warp: pts4 positions of the closing-region members
  const DevParams &P = *Pp;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n) return;
  const auto &G = CloudSel<BATCH>::get(tab, i);
  const DevCloud cl = CloudSel<BATCH>::local(G, cl0);
  int *memb = members[(threadIdx.x >> 5)];
  gpdb_pose &h = hands[i];
  double R[9], smp[3];
#pragma unroll
  for (int r = 0; r < 9; r++) R[r] = h.frame[r];
#pragma unroll
  for (int r = 0; r < 3; r++) smp[r] = h.sample[r];
  const int idx = h.finger_idx;
  const double top = h.top, bottom = top - P.hand_depth, hh = P.hand_height;  // evaluateFingers(points, hand.getTop(), idx)
  const float q[3] = {(float)smp[0], (float)smp[1], (float)smp[2]};            // eigenVectorToPcl (:136-142)
  const SegRange sr = seg_range(G, q, P.rf_hs);
  int label = 0;
  bool half = false, full = false;
  if (idx >= 0 && idx < P.nfp) {
    const double s0 = P.fs[idx], s0w = P.fsw[idx], s1 = P.fs[P.nfp + idx], s1w = P.fsw[P.nfp + idx];
    const double left = s0w, right = s1;  // computePointsInClosingRegion (finger_hand.cpp:141-171)
    auto in_region = [&](double x, double y) { return x > bottom && x < top && y > left && y < right; };
    // the walk: neighbour 0, crop count, back-of-hand collision, the two finger gaps, and the closing region
    int nball = 0, k = 0, cnt = 0, nmemb = 0;
    unsigned long long best = ~0ull;
    unsigned anyA = 0, anyB = 0, blocked = 0;
    double mny = DBL_MAX, mxy = -DBL_MAX;
    auto finger_test = [&](double x, double y) {
      if (x < top) {
        anyA = 1;
        if (x < bottom) anyB = 1;
        if ((y > s0 && y < s0w) || (y > s1 && y < s1w)) blocked = 1;
      }
    };
    warp_scan_ball(G, cl, sr, q, P.r2_hs, [&](bool in, const float4 &p, int g) {
      bool inr = false;
      if (in) {
        nball++;
        const unsigned long long key = ((unsigned long long)__float_as_uint(l2_simple(q, p.x, p.y, p.z)) << 32) | (unsigned)__float_as_int(p.w);
        best = key < best ? key : best;
        double x, y, z;
        to_frame(R, (double)p.x - smp[0], (double)p.y - smp[1], (double)p.z - smp[2], x, y, z);
        if (z > -1.0 * hh && z < hh) {
          k++;
          finger_test(x, y);
          if (in_region(x, y)) {
            inr = true;
            cnt++;
            mny = fmin(mny, y);
            mxy = fmax(mxy, y);
          }
        }
      }
      const unsigned mk = __ballot_sync(0xffffffffu, inr);
      const int pos = nmemb + __popc(mk & ((1u << lane) - 1));
      if (inr && pos < LABEL_CAP) memb[pos] = g;
      nmemb += __popc(mk);
    });
    __syncwarp();
    nball = warp_sum(nball);
    k = warp_sum(k);
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
      best = ob < best ? ob : best;
    }
    const int npad = nball - k;  // cropByHandHeight pads with copies of neighbour 0 (point_list.cpp:44-55)
    const int nb0 = (int)(unsigned)(best & 0xffffffffull);
    double x0 = 0, y0 = 0, z0 = 0;
    if (nball > 0)
      to_frame(R, (double)cl.xyz[3 * (size_t)nb0] - smp[0], (double)cl.xyz[3 * (size_t)nb0 + 1] - smp[1],
               (double)cl.xyz[3 * (size_t)nb0 + 2] - smp[2], x0, y0, z0);
    if (npad > 0 && lane == 0) finger_test(x0, y0);
    anyA = __reduce_or_sync(0xffffffffu, anyA);
    anyB = __reduce_or_sync(0xffffffffu, anyB);
    blocked = __reduce_or_sync(0xffffffffu, blocked);
    if (nball > 0 && anyA && !anyB && !blocked) {
      const bool nb_in = npad > 0 && in_region(x0, y0);
      cnt = warp_sum(cnt) + (nb_in ? npad : 0);
      mny = warp_min(mny);
      mxy = warp_max(mxy);
      if (nb_in) {
        mny = fmin(mny, y0);
        mxy = fmax(mxy, y0);
      }
      if (cnt > 0) {
        // the Antipodal passes: Antipodal::evaluateGrasp (antipodal.cpp:10-96), as in k_hands, over the members
        const bool listed = nmemb <= LABEL_CAP;
        if (!listed && prof && lane == 0) atomicAdd(prof + GPDB_PROF_PATH + PATH_LABEL_WALK, 1ull);
        auto members_do = [&](auto &&visit) {  // visit(x, y, z, cloud-local index, 1) for every member
          if (listed) {
            for (int j = lane; j < nmemb; j += 32) {
              const float4 p = __ldg(cl.pts4 + memb[j]);
              double x, y, z;
              to_frame(R, (double)p.x - smp[0], (double)p.y - smp[1], (double)p.z - smp[2], x, y, z);
              visit(x, y, z, __float_as_int(p.w), 1);
            }
          } else {
            warp_scan_ball(G, cl, sr, q, P.r2_hs, [&](bool in, const float4 &p, int) {
              if (!in) return;
              double x, y, z;
              to_frame(R, (double)p.x - smp[0], (double)p.y - smp[1], (double)p.z - smp[2], x, y, z);
              if (z > -1.0 * hh && z < hh && in_region(x, y)) visit(x, y, z, __float_as_int(p.w), 1);
            });
          }
        };
        const double min_x = mny + 0.003, max_x = mxy - 0.003;
        int cl_ = 0, cr_ = 0;
        double lmaxx = -DBL_MAX, lminx = DBL_MAX, lmaxz = -DBL_MAX, lminz = DBL_MAX;
        double rmaxx = -DBL_MAX, rminx = DBL_MAX, rmaxz = -DBL_MAX, rminz = DBL_MAX;
        auto dots = [&](int pidx, double &ldot, double &rdot) {
          const double *nn = cl.nrm + 3 * (size_t)pidx;
          double n0, n1, n2;
          to_frame(R, nn[0], nn[1], nn[2], n0, n1, n2);
          ldot = (0.0 * n0 + -1.0 * n1) + 0.0 * n2;
          rdot = (0.0 * n0 + 1.0 * n1) + 0.0 * n2;
        };
        auto visitD = [&](double x, double y, double z, int pidx, int wgt) {
          double ldot, rdot;
          dots(pidx, ldot, rdot);
          if (ldot > P.cosf && y < min_x) {
            cl_ += wgt;
            lmaxx = fmax(lmaxx, x); lminx = fmin(lminx, x); lmaxz = fmax(lmaxz, z); lminz = fmin(lminz, z);
          }
          if (rdot > P.cosf && y > max_x) {
            cr_ += wgt;
            rmaxx = fmax(rmaxx, x); rminx = fmin(rminx, x); rmaxz = fmax(rmaxz, z); rminz = fmin(rminz, z);
          }
        };
        members_do(visitD);
        if (nb_in && lane == 0) visitD(x0, y0, z0, nb0, npad);
        cl_ = warp_sum(cl_);
        cr_ = warp_sum(cr_);
        half = cl_ > 0 || cr_ > 0;
        if (cl_ > 0 && cr_ > 0) {
          lmaxx = warp_max(lmaxx); lminx = warp_min(lminx); lmaxz = warp_max(lmaxz); lminz = warp_min(lminz);
          rmaxx = warp_max(rmaxx); rminx = warp_min(rminx); rmaxz = warp_max(rmaxz); rminz = warp_min(rminz);
          const double top_y = fmin(lmaxx, rmaxx), bot_y = fmax(lminx, rminx);
          const double top_z = fmin(lmaxz, rmaxz), bot_z = fmax(lminz, rminz);
          int nl = 0, nr = 0;
          auto visitE = [&](double x, double y, double z, int pidx, int wgt) {
            double ldot, rdot;
            dots(pidx, ldot, rdot);
            const bool inw = x >= bot_y && x <= top_y && z >= bot_z && z <= top_z;
            if (ldot > P.cosf && y < min_x && inw) nl += wgt;
            if (rdot > P.cosf && y > max_x && inw) nr += wgt;
          };
          members_do(visitE);
          if (nb_in && lane == 0) visitE(x0, y0, z0, nb0, npad);
          nl = warp_sum(nl);
          nr = warp_sum(nr);
          full = nl >= P.min_viable && nr >= P.min_viable;
        }
        if (full) label = 1;
      }
    }
  }
  if (lane == 0) {
    h.half_antipodal = half ? 1 : 0;
    h.full_antipodal = full ? 1 : 0;
    labels[i] = label;
  }
}

// ------------------------------------------------------------------------------------------------
// Clustering::findClusters (clustering.cpp:5-105, remove_inliers = false): hand i becomes a cluster when at least
// min_inliers OTHER hands have an axis within 12 degrees, a position within 5 cm and an axis-orthogonal offset within
// 5 mm; cluster position = mean inlier position, score = lower bound of the 99 % confidence interval of the inlier
// scores (Welford update in index order, :62-70). One warp per hand: the lanes test 32 hands j at a time, lane 0 folds
// the inliers of the ballot IN INDEX ORDER, so the float64 running mean / variance are the reference's sequential ones.
// Groups (goff[G+1]): hand i is clustered against the hands of its own group only, as findClusters on that group alone;
// gcount[g] counts the group's clusters.
// ------------------------------------------------------------------------------------------------
__global__ void k_clusters(const gpdb_pose *__restrict__ hands, int n, const int *__restrict__ goff, int G, int min_inliers,
                           double cos_thresh, gpdb_pose *__restrict__ out, uint8_t *__restrict__ keep, int *gcount) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n) return;
  int g = 0, gh = G;  // largest g with goff[g] <= i: empty groups share their offset with the next group
  while (gh - g > 1) {
    const int mid = (g + gh) >> 1;
    if (__ldg(goff + mid) <= i) g = mid; else gh = mid;
  }
  const int lo = __ldg(goff + g), hi = __ldg(goff + g + 1);
  const double AXIS_ALIGN_DIST_THRESH = 0.005, MAX_DIST_THRESH = 0.05;
  const double ai[3] = {hands[i].frame[6], hands[i].frame[7], hands[i].frame[8]};
  const double pi[3] = {hands[i].position[0], hands[i].position[1], hands[i].position[2]};
  double outer[3][3];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) outer[r][c] = ai[r] * ai[c];
  int num_inliers = 0;
  double pd[3] = {0.0, 0.0, 0.0}, mean = 0.0, sd = 0.0;
  for (int j0 = lo; j0 < hi; j0 += 32) {
    const int j = j0 + lane;
    bool inl = false;
    if (j < hi && j != i) {
      const double aj[3] = {hands[j].frame[6], hands[j].frame[7], hands[j].frame[8]};
      const double axis_aligned = ai[0] * aj[0] + ai[1] * aj[1] + ai[2] * aj[2];
      const double d[3] = {pi[0] - hands[j].position[0], pi[1] - hands[j].position[1], pi[2] - hands[j].position[2]};
      double proj[3];
#pragma unroll
      for (int r = 0; r < 3; r++)
        proj[r] = ((r == 0 ? 1.0 : 0.0) - outer[r][0]) * d[0] + ((r == 1 ? 1.0 : 0.0) - outer[r][1]) * d[1] +
                  ((r == 2 ? 1.0 : 0.0) - outer[r][2]) * d[2];
      inl = fabs(axis_aligned) > cos_thresh && sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) <= MAX_DIST_THRESH &&
            sqrt(proj[0] * proj[0] + proj[1] * proj[1] + proj[2] * proj[2]) <= AXIS_ALIGN_DIST_THRESH;
    }
    unsigned m = __ballot_sync(0xffffffffu, inl);
    if (lane == 0)
      while (m) {
        const int jj = j0 + __ffs(m) - 1;
        m &= m - 1;
        num_inliers++;
#pragma unroll
        for (int r = 0; r < 3; r++) pd[r] += hands[jj].position[r];
        const double old_mean = mean, sj = (double)hands[jj].score;
        mean += (sj - mean) / (double)num_inliers;
        sd += (sj - mean) * (sj - old_mean);
      }
  }
  if (lane == 0) {
    gpdb_pose o = hands[i];
    uint8_t k = 0;
    if (num_inliers >= min_inliers) {
      const double dn = (double)num_inliers;
#pragma unroll
      for (int r = 0; r < 3; r++) pd[r] = pd[r] / dn - pi[r];
      sd /= dn;
      if (sd != 0) sd = sqrt(sd);
      const double conf_lb = mean - 2.576 * sd / sqrt((double)num_inliers);
#pragma unroll
      for (int r = 0; r < 3; r++) o.position[r] = pi[r] + pd[r];
      o.score = (float)conf_lb;
      k = 3;  // VALID | FILTERED: geo_compact keeps it
      atomicAdd(gcount + g, 1);
    }
    out[i] = o;
    keep[i] = k;
  }
}

// ------------------------------------------------------------------------------------------------
// k_images (round 2): one CTA per grasp image.
//
// Output stage. The reference post-processes every channel group as cv::dilate(3x3) -> cv::normalize(NORM_MINMAX over the
// group's channels) -> convertTo(CV_8U, 255) (image_strategy.cpp:145-153,179-187,222-230). The affine map + rounding is
// monotone non-decreasing, so it commutes with the max filter: the kernel quantises the OCCUPIED cells only (a few
// hundred per projection) into uint8 planes in shared memory and dilates the bytes afterwards with packed 4-pixel SIMD
// (__vmaxu4), while assembling the pixels. What the normalisation needs from the dilated float image is its max (= the
// max over the occupied cells: dilation moves maxima, it does not change them) and its min, which is 0 whenever the
// image has an all-empty 3x3 window (every value is >= 0 and the background is 0); the occupancy bitmap decides that
// with a few word operations. Images without such a window (fully covered: very dense clouds) take a general path that
// evaluates the min over the dilated float image explicitly (points_minmax_general / dilated_min), so the result is
// the reference's for every input.
//
// Pixel layout written to HBM ("P16"): one 16-byte group per pixel = channels 0..C-1 in the reference's order, bytes
// C..15 zero, pixels row-major — exactly the K-chunk the tensor-core conv1 reads (lenet_tc.cu), so the classifier
// bulk-copies an image straight into its operand plane; k_p16_to_hwc produces the cv::Mat layout for callers that
// want the images themselves (gpdb_images, keep_images).
// ------------------------------------------------------------------------------------------------
// Shared memory of both image kernels; NCAM: the most cameras whose shadows one CTA casts (k_images2: 2).
template <int NCAM>
struct ImgSmemT {
  SegScan<NT_IMG> seg;
  gpdb_pose h;
  double red[NT_IMG / 32][4];
  double center[3];
  double sv[NCAM][3];              // shadow vectors
  unsigned occf[MAXPIX / 32 + 2];  // occupancy of the image cells, flat (bit = pixel index), written by warp ballots
  unsigned lcgA[GPDB_MAX_NSP], lcgC[GPDB_MAX_NSP];  // LCG skip-ahead tables (DevParams), staged once per CTA
  int cam_or, n_img, box_n;
  int wl_n;     // shadow work list, then the voxel list
  union {
    int nonunit;  // scan 1 of k_images2: a box point has a normal of other than unit length (the image goes to k_images)
    int dl_n;     // shadow phase: draws that passed the window test (draw list)
  };
  int ball_n;   // in-ball points recorded by scan 1 (positions in the cell-sorted array)
  int bm_org[3], bm_dims[3];
  float fred[NT_IMG / 32][8];
  // shadow phase invariants of the image, read from here rather than held in registers (k_images2 runs at 64 registers):
  // the float frame and sample, the box widened by the jitter (voxel test) and by the margin (slab cull), and per camera
  // the slab reciprocals of the shadow vector (0: the vector is parallel to that slab)
  float fR[9], fs[3], fbx_lo[3], fbx_hi[3], cull_lo[3], cull_hi[3];
  float cull_inv[NCAM][3];
};
using ImgSmem = ImgSmemT<GPDB_MAX_CAMERAS>;

__device__ __forceinline__ bool in_image_box(const DevParams &P, const gpdb_pose &h, double x, double y, double z) {
  const double half_od = P.vol_w / 2.0;
  return (x > h.bottom) && (x < h.bottom + P.vol_d) && (y > h.center - half_od) && (y < h.center + half_od) &&
         (z > -1.0 * P.vol_h) && (z < P.vol_h);
}
// unit coordinate + cell of one axis without the two float64 divisions of the reference formulas
// ((v - lo) / extent, floor(u / (1.0 / S))) in the common case: a reciprocal multiply gives u to ~2 ulp, and the cell is
// floor(u * S) unless u * S lies within 1e-9 of an integer — only then are the exact divisions evaluated, so the
// cell index is always the reference's. u feeds the per-cell MEAN only (float32 result, 2 ulp of float64 are invisible).
__device__ __forceinline__ void unit_axis(double v, double lo, double extent, double inv_extent, int S, double &u, int &cell) {
  u = (v - lo) * inv_extent;
  double q = u * (double)S;
  double fq = floor(q);
  const double fr = q - fq;  // in [0, 1): exact (Sterbenz) for q >= 1
  if (fr < 1e-9 || fr > 1.0 - 1e-9) {
    u = (v - lo) / extent;
    double cellsize = 1.0 / (double)S;
    fq = floor(u / cellsize);
  }
  cell = min((int)fq, S - 1);
}
__device__ __forceinline__ unsigned unit_q32(double u) {
  return __double2uint_rz(u * 4294967296.0);  // cvt.rzi.u32.f64 saturates: the same result as clamping to [0, 2^32 - 1] first
}

// mean of a cell from its packed accumulator (count << 48 | fixed-point sum, 32 fractional bits): sum / (count 2^32). The
// per-count reciprocals 1 / (c 2^32), c < RCP_N, are tabulated once per image in the (then idle) reduction scratch of the
// ball scan: one multiplication instead of a float64 division per occupied cell (count 1: an exact scaling either way).
constexpr int RCP_N = (NT_IMG / 32) * 4;
__device__ __forceinline__ double cell_mean(unsigned long long acc, const double *rcp) {
  const unsigned c = (unsigned)(acc >> 48);
  const double sum = (double)(acc & 0xffffffffffffull);
  return c < (unsigned)RCP_N ? sum * rcp[c] : sum / ((double)c * 4294967296.0);
}
// The image tiles hold 64-bit cells (low word at the lower address) but are updated with 32-bit shared-memory atomics:
// sm_90 has no native 64-bit shared atomic add or max, and the compare-and-swap loop the compiler emits instead
// serialises lanes that hit the same cell (common for shadow voxels, which collapse along each projection axis).
//
// cell_add: one entry into a cell accumulator (count << 48 | fixed-point sum). Each adder carries its own overflow of the
// low word into the high word, so the final 64-bit value is the exact sum whatever order the adders run in. Returns
// whether this entry carried.
__device__ __forceinline__ bool cell_add(unsigned long long *cell, unsigned q) {
  unsigned *w = reinterpret_cast<unsigned *>(cell);
  const unsigned lo_old = atomicAdd(w, q);
  const bool carry = lo_old + q < lo_old;
  atomicAdd(w + 1, (1u << 16) + (carry ? 1u : 0u));
  return carry;
}
// key_max_dist, barrier, key_max_index: the cell ends up holding the largest key (distance bits << 32 | index), as one
// 64-bit atomicMax would leave it. The index word is only raised by keys whose distance equals the cell's maximum.
__device__ __forceinline__ void key_max_dist(unsigned long long *cell, unsigned long long key) {
  atomicMax(reinterpret_cast<unsigned *>(cell) + 1, (unsigned)(key >> 32));
}
__device__ __forceinline__ void key_max_index(unsigned long long *cell, unsigned long long key) {
  unsigned *w = reinterpret_cast<unsigned *>(cell);
  if (w[1] == (unsigned)(key >> 32)) atomicMax(w, (unsigned)key);
}

__device__ __forceinline__ bool fully_covered(const unsigned *occf, int S);
// block-wide reduction of up to eight floats with max (use negated values for min). Contains two barriers. With `occf`
// non-null, warp 0 also evaluates fully_covered(occf) between the barriers (the occupancy words were written before the
// call) and every thread receives the verdict in *covered — one evaluation per CTA, no extra barrier.
template <int NT, int NV>
__device__ __forceinline__ void block_max(float (&v)[NV], float (*red)[8], const unsigned *occf = nullptr, int S = 0,
                                          bool *covered = nullptr) {
#pragma unroll
  for (int o = 16; o; o >>= 1)
#pragma unroll
    for (int i = 0; i < NV; i++) v[i] = fmaxf(v[i], __shfl_xor_sync(0xffffffffu, v[i], o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int i = 0; i < NV; i++) red[threadIdx.x >> 5][i] = v[i];
  if (occf && threadIdx.x < 32) {
    const bool c = fully_covered(occf, S);
    if (threadIdx.x == 0) red[0][7] = c ? 1.0f : 0.0f;  // slot 7 is never used by a reduction (NV <= 6)
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NV; i++) v[i] = red[0][i];
  for (int w = 1; w < NT / 32; w++)
#pragma unroll
    for (int i = 0; i < NV; i++) v[i] = fmaxf(v[i], red[w][i]);
  if (covered) *covered = red[0][7] != 0.0f;
}

// cv::normalize(NORM_MINMAX, 0..1) + convertTo(CV_8U, 255) of one value, as OpenCV evaluates it: scale / shift in double,
// cast to float, one fused multiply-add, round-half-even, saturate.
struct Quant {
  float a, b;
  __device__ __forceinline__ Quant(float mn, float mx) {
    const double smin = (double)mn, smax = (double)mx;
    const double scale = (1.0 - 0.0) * (smax - smin > DBL_EPSILON ? 1.0 / (smax - smin) : 0.0);
    const double shift = 0.0 - smin * scale;
    a = (float)scale;
    b = (float)shift;
  }
  __device__ __forceinline__ unsigned operator()(float v) const {
    const float t = fmaf(v, a, b);
    const int q = __float2int_rn(t * 255.0f);
    return (unsigned)min(max(q, 0), 255);
  }
};

// true when the S x S occupancy has NO all-empty 3x3 window. occf: flat bitmap (bit = row * S + col) followed by two
// zero-readable words. One warp (32 rows per pass, a few word operations per row); block_max distributes the verdict.
__device__ __forceinline__ bool fully_covered(const unsigned *occf, int S) {
  const int lane = threadIdx.x & 31;
  const unsigned long long mask = S >= 64 ? ~0ull : ((1ull << S) - 1ull);
  auto row_bits = [&](int r) -> unsigned long long {
    if (r < 0 || r >= S) return 0ull;
    const int b = r * S, w = b >> 5, sh = b & 31;
    unsigned long long x = ((unsigned long long)occf[w] | ((unsigned long long)occf[w + 1] << 32)) >> sh;
    if (sh + S > 64) x |= (unsigned long long)occf[w + 2] << (64 - sh);
    return x & mask;
  };
  bool empty = false;
  for (int r = lane; r < S; r += 32) {
    const unsigned long long o = row_bits(r - 1) | row_bits(r) | row_bits(r + 1);
    const unsigned long long d = (o | (o << 1) | (o >> 1)) & mask;
    empty = empty || (d != mask);
  }
  return !__any_sync(0xffffffffu, empty);
}
// one bit per cell from a per-thread predicate over pix = tid + t * NT (warp-aligned): word (pix >> 5) of the flat bitmap
template <int NT>
__device__ __forceinline__ void occ_ballot(unsigned *occf, int t, bool occupied) {
  const unsigned word = __ballot_sync(0xffffffffu, occupied);
  if ((threadIdx.x & 31) == 0) occf[(threadIdx.x >> 5) + t * (NT / 32)] = word;
}

// min over the 3x3-dilated (border ignored) image of channel plane F[SS] (float, row-major): general path only
template <int NT>
__device__ __noinline__ float dilated_min(const float *F, int S) {
  float mn = FLT_MAX;
  for (int pix = threadIdx.x; pix < S * S; pix += NT) {
    const int r = pix / S, c = pix - r * S;
    float m = -FLT_MAX;
    for (int dr = -1; dr <= 1; dr++)
      for (int dc = -1; dc <= 1; dc++) {
        const int rr = r + dr, cc = c + dc;
        if (rr >= 0 && rr < S && cc >= 0 && cc < S) m = fmaxf(m, F[rr * S + cc]);
      }
    mn = fminf(mn, m);
  }
  return mn;
}

// optional phase timing (development aid, gpdb_debug_phase_cycles): thread 0 accumulates clock64() deltas
#define PHASE(i)                                                        \
  do {                                                                  \
    if (prof && threadIdx.x == 0) {                                     \
      long long now__ = clock64();                                      \
      if ((i) > 1) atomicAdd(prof + (i), (unsigned long long)(now__ - t_phase)); \
      t_phase = now__;                                                  \
    }                                                                   \
  } while (0)
// sub-phase timing of the shadow half (gpdb_debug_phase_cycles [16 + i]): thread 0 adds the cycles since t, restarts t
__device__ __forceinline__ void sub_phase(unsigned long long *prof, int i, long long &t) {
  if (prof && threadIdx.x == 0) {
    const long long now = clock64();
    atomicAdd(prof + GPDB_PROF_SUB + i, (unsigned long long)(now - t));
    t = now;
  }
}
enum SubPhase { SUB_CULL, SUB_WINDOW, SUB_EXPAND, SUB_CHANNELS, SUB_STASH, SUB_CLEARS, SUB_PROBE, SUB_EVT_SHARED };

// ---- phases shared by the two image kernels (k_images, k_images2). Every function is called by all threads of the CTA
// together unless it says otherwise.

// Warp-aggregated slot reservation (one shared-memory atomic per warp): this lane's slot among the lanes with `pred`, in
// lane order. Called by all 32 lanes together; the result means nothing where pred is false.
__device__ __forceinline__ int warp_append(bool pred, int *counter) {
  const unsigned mk = __ballot_sync(0xffffffffu, pred);
  if (!mk) return 0;
  const int lane = threadIdx.x & 31, leader = __ffs(mk) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(counter, __popc(mk));
  base = __shfl_sync(0xffffffffu, base, leader);
  return base + __popc(mk & ((1u << lane) - 1));
}

// Balanced expansion of the set bits of one bitmap word per lane (shadow voxels are spatially clustered, so a loop over
// each lane's own word would hold the warp for the densest word's popcount): the warp's set bits, in lane then bit order,
// are handed out 32 at a time. Each lane finds its slot's word by a binary search over the inclusive popcount scan, and
// the bit with __fns. reserve(total) is called once by all lanes and returns the warp's first output position;
// emit(position, code | bit) runs once per set bit. Called by all 32 lanes together.
template <class R, class E>
__device__ __forceinline__ void warp_expand_bits(unsigned bits, unsigned code, R &&reserve, E &&emit) {
  const int lane = threadIdx.x & 31;
  if (!__any_sync(0xffffffffu, bits != 0u)) return;  // most words of a bitmap are empty
  const int cnt = __popc(bits);
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  const int base = reserve(total);
  for (int j0 = 0; j0 < total; j0 += 32) {
    const int j = j0 + lane;
    int w = 0;  // first lane whose inclusive count exceeds j
#pragma unroll
    for (int s = 16; s; s >>= 1) {
      const int v = __shfl_sync(0xffffffffu, incl, w + s - 1);
      if (v <= j) w += s;
    }
    const unsigned wbits = __shfl_sync(0xffffffffu, bits, w), wcode = __shfl_sync(0xffffffffu, code, w);
    const int wexcl = __shfl_sync(0xffffffffu, incl - cnt, w);
    if (j < total) emit(base + j, wcode | __fns(wbits, 0, j - wexcl + 1));
  }
}

// The set bits of a shadow bitmap (rows of 64 bits along x, nbits bits), expanded into voxel codes b0 | b1 << 8 | b2 << 16:
// emit(position, code) once per set bit, positions reserved from *counter (null: every position is 0).
template <class E>
__device__ __forceinline__ void expand_bitmap(const unsigned *bitmap, int nbits, int d1, int *counter, E &&emit) {
  const int lane = threadIdx.x & 31;
  for (int wd0 = 0; wd0 * 32 < nbits; wd0 += NT_IMG) {
    const int wd = wd0 + threadIdx.x;
    const unsigned bits = (wd * 32 < nbits) ? bitmap[wd] : 0u;
    const int rowi = wd >> 1;  // b2 * d1 + b1 (words past the bitmap's end are empty)
    const unsigned code = ((unsigned)(rowi % d1) << 8) | ((unsigned)(rowi / d1) << 16) | ((unsigned)(wd & 1) << 5);
    warp_expand_bits(
        bits, code,
        [&](int total) {
          int base = 0;
          if (counter && lane == 0 && total) base = atomicAdd(counter, total);
          return __shfl_sync(0xffffffffu, base, 0);
        },
        emit);
  }
}

// Coordinate orders of the three projections, (x,y,z), (z,y,x), (z,x,y): rows cumulatively swapped {0<->2}, {1<->2}
// (image_15_channels_strategy.cpp:57-64). Axis a0 gives the row (flipped), a1 the column, a2 the depth.
struct Proj {
  int a0, a1, a2;
  __device__ __forceinline__ explicit Proj(int pj) : a0(pj == 0 ? 0 : 2), a1(pj == 2 ? 0 : 1), a2(pj == 0 ? 2 : (pj == 1 ? 0 : 1)) {}
  __device__ __forceinline__ int row(unsigned cells, int S) const { return S - 1 - (int)((cells >> (8 * a0)) & 255); }
  __device__ __forceinline__ int col(unsigned cells) const { return (int)((cells >> (8 * a1)) & 255); }
  __device__ __forceinline__ int pix(unsigned cells, int S) const { return row(cells, S) * S + col(cells); }
};

// The points inside the image box: key (distance bits << 32 | index), coordinates [3][cap] (raw float after scan 1, then
// fixed point in the unit cube) and cells (packed 3 x 8 bit), in one block of memory.
struct BoxList {
  unsigned long long *keys;
  unsigned *q, *cell;
  int cap;
  __device__ __forceinline__ BoxList(unsigned char *base, int cap_)
      : keys(reinterpret_cast<unsigned long long *>(base)), q(reinterpret_cast<unsigned *>(keys + cap_)), cell(q + 3 * cap_),
        cap(cap_) {}
};

// the cell and unit coordinates of a hand-frame point (ImageStrategy::transformToUnitImage); inv: the reciprocal extents
__device__ __forceinline__ void unit_cells(const DevParams &P, const gpdb_pose &h, const double (&inv)[3], int S, double x,
                                           double y, double z, double (&u)[3], int (&cell)[3]) {
  unit_axis(x, h.bottom, P.vol_d, inv[0], S, u[0], cell[0]);
  unit_axis(y, h.center - P.vol_w / 2.0, P.vol_w, inv[1], S, u[1], cell[1]);
  unit_axis(z, -P.vol_h, 2.0 * P.vol_h, inv[2], S, u[2], cell[2]);
}

// per CTA: the LCG skip-ahead tables and a clean occupancy bitmap
template <class Sm>
__device__ __forceinline__ void img_cta_init(Sm &sm, const DevParams &P) {
  for (int k = threadIdx.x; k < GPDB_MAX_NSP; k += NT_IMG) {
    sm.lcgA[k] = P.lcgA[k];
    sm.lcgC[k] = P.lcgC[k];
  }
  for (int k = threadIdx.x; k < MAXPIX / 32 + 2; k += NT_IMG) sm.occf[k] = 0u;
}

// per image: the pose into shared memory, the counters of scan 1 cleared (visible after the caller's next barrier)
template <class Sm>
__device__ __forceinline__ void img_begin(Sm &sm, const gpdb_pose *pose) {
  __syncthreads();
  const int *src = reinterpret_cast<const int *>(pose);
  int *dst = reinterpret_cast<int *>(&sm.h);
  for (int k = threadIdx.x; k < (int)(sizeof(gpdb_pose) / 4); k += NT_IMG) dst[k] = src[k];
  if (threadIdx.x == 0) {
    sm.cam_or = 0;
    sm.n_img = 0;
    sm.box_n = 0;
    sm.ball_n = 0;
    sm.nonunit = 0;
  }
}

// Ball scan 1: the neighbourhood centre and camera set (HandSet::calculateShadow, hand_set.cpp:131-136), at 15 channels
// the positions of the in-ball points in the cell-sorted array (the first ball_cap of them: the shadow casting re-reads
// the neighbourhood from that list as independent loads instead of walking the grid again), and the first bl.cap points
// inside the image box. The scan only APPENDS the raw box points (few lanes qualify: doing the per-point work here would
// run it at ~6 % lane utilisation); box_units does it densely afterwards. on_box(index) runs for every box point. Thread
// 0 finishes with sm.center and sm.cam_or set (the caller's barrier publishes them); sm.box_n and sm.ball_n count every
// point, including those past the capacities.
template <class Sm, class G, class OnBox>
__device__ __forceinline__ void ball_scan1(const DevParams &P, const G &Gd, const DevCloud &cl, const SegRange &sr,
                                           const float (&q)[3], Sm &sm, int C, int *ball, int ball_cap, const BoxList &bl,
                                           OnBox &&on_box) {
  const gpdb_pose &h = sm.h;
  const int tid = threadIdx.x, lane = tid & 31;
  const bool need_cam = (C == 15) && !Gd.all_seen;  // the camera set of the neighbourhood is only read by the shadow
  double sx = 0, sy = 0, sz = 0;
  int cnt = 0, cam_or = 0;
  scan_balanced<NT_IMG>(Gd, cl, sr, sm.seg, [&](bool in, const float4 &p, int where) {
    bool inb = false, inball = false;
    unsigned long long key = 0;
    if (in) {
      float d = l2_simple(q, p.x, p.y, p.z);
      if (d < P.r2_img) {
        inball = true;
        const int idx = __float_as_int(p.w);
        sx += (double)p.x;
        sy += (double)p.y;
        sz += (double)p.z;
        cnt++;
        if (need_cam) cam_or |= cl.cam[idx];
        double x, y, z;
        to_frame(h.frame, (double)p.x - h.sample[0], (double)p.y - h.sample[1], (double)p.z - h.sample[2], x, y, z);
        if (in_image_box(P, h, x, y, z)) {
          inb = true;
          key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)idx;
          on_box(idx);
        }
      }
    }
    if (C == 15) {
      const int pos = warp_append(inball, &sm.ball_n);
      if (inball && pos < ball_cap) ball[pos] = where;
    }
    const int pos = warp_append(inb, &sm.box_n);
    if (inb && pos < bl.cap) {
      bl.keys[pos] = key;
      bl.q[pos] = __float_as_uint(p.x);
      bl.q[bl.cap + pos] = __float_as_uint(p.y);
      bl.q[2 * bl.cap + pos] = __float_as_uint(p.z);
    }
  });
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
    sy += __shfl_xor_sync(0xffffffffu, sy, o);
    sz += __shfl_xor_sync(0xffffffffu, sz, o);
  }
  cnt = warp_sum(cnt);
  cam_or = __reduce_or_sync(0xffffffffu, (unsigned)cam_or);
  __syncthreads();
  if (lane == 0) {
    sm.red[tid >> 5][0] = sx;
    sm.red[tid >> 5][1] = sy;
    sm.red[tid >> 5][2] = sz;
    atomicAdd(&sm.n_img, cnt);
    atomicOr(&sm.cam_or, cam_or);
  }
  __syncthreads();
  if (tid == 0) {
    double a0 = 0, a1 = 0, a2 = 0;
    for (int w = 0; w < NT_IMG / 32; w++) {
      a0 += sm.red[w][0];
      a1 += sm.red[w][1];
      a2 += sm.red[w][2];
    }
    double nn = (double)sm.n_img;
    if (!need_cam && sm.n_img > 0) sm.cam_or = (1 << Gd.K) - 1;  // every point is seen by every camera (set at upload)
    sm.center[0] = a0 / nn;
    sm.center[1] = a1 / nn;
    sm.center[2] = a2 / nn;
  }
}

// Dense pass over the bn listed box points (all lanes busy): raw coordinates -> hand frame -> fixed-point unit coordinates
// and packed cells. on_point(k) runs after point k. No barrier. Not inlined (nor is shadow_setup): inlined, the two
// raise the spills of k_images2, which runs at 64 registers.
template <class F>
__device__ __noinline__ void box_units(const DevParams &P, const gpdb_pose &h, const double (&inv)[3], const BoxList &bl,
                                          int bn, int S, F &&on_point) {
  for (int k = threadIdx.x; k < bn; k += NT_IMG) {
    const double px = (double)__uint_as_float(bl.q[k]), py = (double)__uint_as_float(bl.q[bl.cap + k]),
                 pz = (double)__uint_as_float(bl.q[2 * bl.cap + k]);
    double x, y, z, u[3];
    int c[3];
    to_frame(h.frame, px - h.sample[0], py - h.sample[1], pz - h.sample[2], x, y, z);
    unit_cells(P, h, inv, S, x, y, z, u, c);
    bl.q[k] = unit_q32(u[0]);
    bl.q[bl.cap + k] = unit_q32(u[1]);
    bl.q[2 * bl.cap + k] = unit_q32(u[2]);
    bl.cell[k] = (unsigned)c[0] | ((unsigned)c[1] << 8) | ((unsigned)c[2] << 16);
    on_point(k);
  }
}

// One projection of the box points: tile A gets each cell's arg-max key (= the last writer in (distance, index) order,
// createNormalsImage :124-143), tile B its depth sum (the mean, createDepthImage :158-176), occf its occupancy bit. The
// tiles and occf are clean on entry. Ends behind a barrier.
__device__ __forceinline__ void raster_projection(const BoxList &bl, int bn, int S, const Proj &pr, unsigned long long *tileA,
                                                  unsigned long long *tileB, unsigned *occf) {
  for (int k = threadIdx.x; k < bn; k += NT_IMG) {
    const int pix = pr.pix(bl.cell[k], S);
    key_max_dist(tileA + pix, bl.keys[k]);
    atomicOr(&occf[pix >> 5], 1u << (pix & 31));
  }
  __syncthreads();
  for (int k = threadIdx.x; k < bn; k += NT_IMG) {
    const int pix = pr.pix(bl.cell[k], S);
    key_max_index(tileA + pix, bl.keys[k]);
    cell_add(tileB + pix, bl.q[pr.a2 * bl.cap + k]);
  }
  __syncthreads();
}

// clears the cells of one projection that the box points touched (tiles A, B, occupancy) for the next projection
__device__ __forceinline__ void wipe_cells(const BoxList &bl, int bn, int S, const Proj &pr, unsigned long long *tileA,
                                           unsigned long long *tileB, unsigned *occf) {
  for (int k = threadIdx.x; k < bn; k += NT_IMG) {
    const int pix = pr.pix(bl.cell[k], S);
    tileA[pix] = 0ull;
    tileB[pix] = 0ull;
    occf[pix >> 5] = 0u;
  }
}

// general path of the point channels (no all-empty 3x3 window): the min over the dilations of the float images F[4][S S]
// of one projection, normals (channels 0..2) in mnv[0] and depth in mnv[1]
__device__ __forceinline__ void points_dilated_min(const float *F, int S, float (*fred)[8], float (&mnv)[2]) {
  const int SS = S * S;
  float neg[2];
  neg[0] = -fminf(fminf(dilated_min<NT_IMG>(F, S), dilated_min<NT_IMG>(F + SS, S)), dilated_min<NT_IMG>(F + 2 * SS, S));
  neg[1] = -dilated_min<NT_IMG>(F + 3 * SS, S);
  block_max<NT_IMG, 2>(neg, fred);
  mnv[0] = -neg[0];
  mnv[1] = -neg[1];
}

// The quantised point planes of one projection: normals in planes cb .. cb + 2, depth in plane cd, planes plb bytes apart,
// rows of rs bytes. The winners of the projection's cells are quantised with min mnv / max mxv. With `background` (the
// general path: the image has no all-empty 3x3 window, so its minimum need not be 0) the planes are first filled with the
// quantised 0. for_each_winner(emit) calls emit(byte offset in the plane, |n0|, |n1|, |n2|, 1 - mean depth) once per winner.
struct PointPlanes {
  uint8_t *base;
  int plb, rs, cb, cd;
  bool nrm, dep;
};
template <class W>
__device__ __forceinline__ void winners_to_planes(const PointPlanes &pp, const float (&mnv)[2], const float (&mxv)[2],
                                                  bool background, W &&for_each_winner) {
  const Quant qn(mnv[0], mxv[0]), qd(mnv[1], mxv[1]);
  if (background) {
    const unsigned bg_n = qn(0.0f) * 0x01010101u, bg_d = qd(0.0f) * 0x01010101u;
    for (int k = threadIdx.x; k < (pp.plb >> 2); k += NT_IMG) {
      if (pp.nrm)
#pragma unroll
        for (int c = 0; c < 3; c++) reinterpret_cast<unsigned *>(pp.base + (size_t)(pp.cb + c) * pp.plb)[k] = bg_n;
      if (pp.dep) reinterpret_cast<unsigned *>(pp.base + (size_t)pp.cd * pp.plb)[k] = bg_d;
    }
    __syncthreads();  // the background is in place before the winners overwrite their cells
  }
  for_each_winner([&](int o, float n0, float n1, float n2, float dv) {
    if (pp.nrm) {
      pp.base[(size_t)(pp.cb + 0) * pp.plb + o] = (uint8_t)qn(n0);
      pp.base[(size_t)(pp.cb + 1) * pp.plb + o] = (uint8_t)qn(n1);
      pp.base[(size_t)(pp.cb + 2) * pp.plb + o] = (uint8_t)qn(n2);
    }
    if (pp.dep) pp.base[(size_t)pp.cd * pp.plb + o] = (uint8_t)qd(dv);
  });
}

// ---- shadow phase (15 channels): HandSet::calculateShadow, deterministic variant

// Shadow setup (thread 0 and threads < K): the bitmap AABB (voxel indices of the image box widened by the largest jitter),
// the float32 invariants of the pre-test and of the slab cull, and per camera the shadow vector shadow_length (center -
// view_point) / norm (hand_set.cpp:146-150) with the slab reciprocals of its hand-frame image. Clears the bitmaps
// (bm_total words). No barrier.
template <class Sm, class G>
__device__ __noinline__ void shadow_setup(const DevParams &P, const G &Gd, Sm &sm, double gmax, unsigned *bitmap,
                                             int bm_total) {
  const gpdb_pose &h = sm.h;
  const int tid = threadIdx.x;
  const double voxel = GPDB_SHADOW_VOXEL;
  if (tid < 32) {
    const double half_od = P.vol_w / 2.0;
    // lane 3 cr + r (< 24): world coordinate r of box corner cr; lanes r < 3 then take the min / max over the corners in
    // corner order
    double wv = 0.0;
    if (tid < 24) {
      const int cr = tid / 3, r = tid - 3 * cr;
      double cx = (cr & 1) ? h.bottom + P.vol_d : h.bottom;
      double cy = (cr & 2) ? h.center + half_od : h.center - half_od;
      double cz = (cr & 4) ? P.vol_h : -P.vol_h;
      wv = h.frame[r] * cx + h.frame[3 + r] * cy + h.frame[6 + r] * cz + h.sample[r];
    }
    double mn = DBL_MAX, mx = -DBL_MAX;
#pragma unroll
    for (int cr = 0; cr < 8; cr++) {
      const double v = __shfl_sync(0xffffffffu, wv, 3 * cr + tid % 3);
      mn = fmin(mn, v);
      mx = fmax(mx, v);
    }
    if (tid < 3) {
      const int a = tid;
      const double jmax = gmax * voxel * 0.3 + 1e-9;
      int lo = (int)floor((mn - jmax) * P.vox_mult) - 1;
      int hi = (int)floor((mx + jmax) * P.vox_mult) + 1;
      sm.bm_org[a] = lo;
      sm.bm_dims[a] = min(hi - lo + 1, P.bm_dim);
      // pre-test: float32 frame and sample, box widened by the jitter (gmax 0.0009 sqrt 3) + 2e-5 slack
      sm.fs[a] = (float)h.sample[a];
      const float jm = (float)(gmax * voxel * 0.3 * 1.7320508075688772 + 2e-5);
      sm.fbx_lo[a] = (a == 0 ? (float)h.bottom : a == 1 ? (float)(h.center - P.vol_w / 2.0) : (float)(-P.vol_h)) - jm;
      sm.fbx_hi[a] = (a == 0 ? (float)(h.bottom + P.vol_d) : a == 1 ? (float)(h.center + P.vol_w / 2.0) : (float)P.vol_h) + jm;
      // slab cull: the image box in the hand frame, widened by voxel truncation (<= 0.003 sqrt 3) + jitter (<= gmax
      // 0.0009 sqrt 3), + 1e-5 for the float32 rounding of the cull
      const double wm = 0.0105;
      const double bx_lo = a == 0 ? h.bottom - wm : a == 1 ? h.center - P.vol_w / 2.0 - wm : -P.vol_h - wm;
      const double bx_hi = a == 0 ? h.bottom + P.vol_d + wm : a == 1 ? h.center + P.vol_w / 2.0 + wm : P.vol_h + wm;
      sm.cull_lo[a] = (float)bx_lo - 1e-5f;
      sm.cull_hi[a] = (float)bx_hi + 1e-5f;
    }
    if (tid < 9) sm.fR[tid] = (float)h.frame[tid];
    if (tid == 0) sm.wl_n = 0;  // the work-list count of the first camera's casting
  }
  if (tid < Gd.K) {
    double s0 = sm.center[0] - Gd.vp[tid][0], s1 = sm.center[1] - Gd.vp[tid][1], s2 = sm.center[2] - Gd.vp[tid][2];
    double nn = sqrt((s0 * s0 + s1 * s1) + s2 * s2);
    sm.sv[tid][0] = P.shadow_length * s0 / nn;
    sm.sv[tid][1] = P.shadow_length * s1 / nn;
    sm.sv[tid][2] = P.shadow_length * s2 / nn;
    double svh[3];
    to_frame(h.frame, sm.sv[tid][0], sm.sv[tid][1], sm.sv[tid][2], svh[0], svh[1], svh[2]);
    for (int a = 0; a < 3; a++) {
      // 0: the segment moves this coordinate by < 1e-6 (below the margin): parallel to the slab
      const float dv = (float)svh[a];
      sm.cull_inv[tid][a] = fabsf(dv) < 1e-6f ? 0.0f : 1.0f / dv;
    }
  }
  for (int k = tid; k < bm_total; k += NT_IMG) bitmap[k] = 0u;
}

// the bitmap AABB of the image (origin and extent in voxels), read once after the setup
struct VoxelBox {
  int o0, o1, o2, d0, d1, d2;
  template <class Sm>
  __device__ __forceinline__ explicit VoxelBox(const Sm &sm)
      : o0(sm.bm_org[0]), o1(sm.bm_org[1]), o2(sm.bm_org[2]), d0(sm.bm_dims[0]), d1(sm.bm_dims[1]), d2(sm.bm_dims[2]) {}
};

// voxel -> jittered point -> hand frame -> inside the image box?
__device__ __forceinline__ bool voxel_point_in_box(const DevParams &P, const gpdb_pose &h, const double *qtab, int v0, int v1,
                                                   int v2, double &x, double &y, double &z) {
  const double voxel = GPDB_SHADOW_VOXEL;
  double g = qtab[gpdb_voxel_hash(v0, v1, v2) & (GPDB_QTAB_SIZE - 1)];
  double jit = 1.0 * g * voxel * 0.3;
  double w0 = (double)v0 * voxel + jit, w1 = (double)v1 * voxel + jit, w2 = (double)v2 * voxel + jit;
  to_frame(h.frame, w0 - h.sample[0], w1 - h.sample[1], w2 - h.sample[2], x, y, z);
  return in_image_box(P, h, x, y, z);
}

// one shadow draw of camera k -> bit index in its bitmap, or -1 (outside the bitmap AABB / fails the pre-test)
template <class Sm>
__device__ __forceinline__ int draw_bit(const DevParams &P, const Sm &sm, const VoxelBox &vb, double px, double py, double pz,
                                        unsigned seed, int k) {
  const double s0 = sm.sv[k][0], s1 = sm.sv[k][1], s2 = sm.sv[k][2];
  double u = (double)((seed >> 16) & 0x7FFFu) * (1.0 / 32767.0);
  int v0 = (int)((px + u * s0) * P.vox_mult);
  int v1 = (int)((py + u * s1) * P.vox_mult);
  int v2 = (int)((pz + u * s2) * P.vox_mult);
  int b0 = v0 - vb.o0, b1 = v1 - vb.o1, b2 = v2 - vb.o2;
  if ((unsigned)b0 >= (unsigned)vb.d0 || (unsigned)b1 >= (unsigned)vb.d1 || (unsigned)b2 >= (unsigned)vb.d2) return -1;
  // conservative float32 pre-test of the voxel's lattice point against the image box widened by the largest jitter
  // (+ rounding slack): rejects most out-of-box voxels for ~20 instructions. The exact float64 test (jitter + frame
  // transform, the oracle's operation order) runs once per UNIQUE surviving voxel (eval_voxel).
  const float *fR = sm.fR, *fs = sm.fs;
  const float wx = fmaf((float)v0, 0.003f, -fs[0]), wy = fmaf((float)v1, 0.003f, -fs[1]), wz = fmaf((float)v2, 0.003f, -fs[2]);
  const float hx = fmaf(fR[0], wx, fmaf(fR[1], wy, fR[2] * wz));
  const float hy = fmaf(fR[3], wx, fmaf(fR[4], wy, fR[5] * wz));
  const float hz = fmaf(fR[6], wx, fmaf(fR[7], wy, fR[8] * wz));
  if (hx < sm.fbx_lo[0] || hx > sm.fbx_hi[0] || hy < sm.fbx_lo[1] || hy > sm.fbx_hi[1] || hz < sm.fbx_lo[2] ||
      hz > sm.fbx_hi[2])
    return -1;
  return ((b2 * vb.d1 + b1) << 6) + b0;
}

__device__ __forceinline__ void set_bit(unsigned *bm, int bit) {
  if (bit >= 0) atomicOr(bm + (bit >> 5), 1u << (bit & 31));
}

// Conservative slab cull of camera k's shadow segment p + u sv, u in [0,1], against the widened image box (hand frame):
// only draws whose 15-bit LCG value falls in rg = [r0, r1] (r0 | r1 << 16) can produce a voxel point inside the box.
// float32 is enough here: its rounding (~1e-7 of coordinates < 0.2 m, 3e-7 of t) is covered by the extra 1e-5 of box
// margin and by the +-1 of slack on r0 / r1 (1 / 32767 = 3e-5); the draws themselves are evaluated in the reference's
// float64.
template <class Sm>
__device__ __forceinline__ bool cull(const Sm &sm, int k, const float4 &p, unsigned &rg) {
  const float *fR = sm.fR, *cull_inv = sm.cull_inv[k];
  const float wx = p.x - sm.fs[0], wy = p.y - sm.fs[1], wz = p.z - sm.fs[2];
  const float o3[3] = {fmaf(fR[0], wx, fmaf(fR[1], wy, fR[2] * wz)), fmaf(fR[3], wx, fmaf(fR[4], wy, fR[5] * wz)),
                       fmaf(fR[6], wx, fmaf(fR[7], wy, fR[8] * wz))};
  float tmin = 0.0f, tmax = 1.0f;
  bool hit = true;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (cull_inv[a] == 0.0f) {  // segment (numerically) parallel to the slab: inside or outside for every u
      hit = hit && o3[a] >= sm.cull_lo[a] && o3[a] <= sm.cull_hi[a];
    } else {
      const float t1 = (sm.cull_lo[a] - o3[a]) * cull_inv[a], t2 = (sm.cull_hi[a] - o3[a]) * cull_inv[a];
      tmin = fmaxf(tmin, fminf(t1, t2));
      tmax = fminf(tmax, fmaxf(t1, t2));
    }
  }
  if (!hit || tmin > tmax) return false;
  const int r0 = max((int)floorf(tmin * 32767.0f) - 1, 0), r1 = min((int)ceilf(tmax * 32767.0f) + 1, 32767);
  rg = (unsigned)r0 | ((unsigned)r1 << 16);
  return true;
}

// Where the shadow casting of one camera keeps its lists, and the path-counter slots of their in-place fallbacks.
struct CastLists {
  float4 *wl;        // work list: x, y, z, LCG seed of the points whose segment passes the cull
  unsigned *wrange;  // ... and their LCG windows (cull)
  int wl_cap;
  unsigned *dlist;   // draw list: item << 7 | t of the draws inside their point's window
  int dl_cap;
  int path_cast, path_draw;
};

// Shadow casting of camera k into its bitmap bm, load-balanced in two steps. (1) The in-ball points whose shadow segment
// can reach the bitmap go to the work list: from the list scan 1 recorded (use_ball; ball_at(i): the position of the i-th
// of the nball points) or by walking the grid again. Past the work list's capacity a point's draws are cast in place.
// (2) The (point, draw) pairs are spread evenly over all threads — draw t of a point comes from the closed-form LCG
// skip-ahead seed_t = A^(t+1) seed_0 + C_(t+1) (mod 2^32) — in two dense steps: the cheap window test of every pair,
// which ~60 % of the draws fail, with the survivors compacted into the draw list, then the float64 voxel arithmetic of the
// survivors only, all lanes busy (doing it in place kept the 70-instruction body running at ~40 % lane utilisation).
// count_walks: event slot 14 counts the grid walks.
template <class Sm, class G, class BallAt>
__device__ __forceinline__ void cast_camera(const DevParams &P, const G &Gd, const DevCloud &cl, const SegRange &sr,
                                            const float (&q)[3], Sm &sm, const VoxelBox &vb, int k, unsigned *bm,
                                            const CastLists &L, bool use_ball, int nball, BallAt &&ball_at,
                                            unsigned long long *prof, bool count_walks) {
  const int tid = threadIdx.x;
  long long t_sub = 0;
  if (prof && tid == 0) t_sub = clock64();
  __syncthreads();  // the previous camera's lists have been read
  // sm.wl_n is 0 on entry (shadow_setup, or the previous camera behind its window-test barrier); sm.dl_n, read by the
  // previous camera before the barrier above, is first counted behind the append's barrier
  if (tid == 0) sm.dl_n = 0;
  // appends the point to the work list; called by all 32 lanes together
  auto append = [&](bool ok, const float4 &p, unsigned rg) {
    const int pos = warp_append(ok, &sm.wl_n);
    if (!ok) return;
    const unsigned seed0 = gpdb_shadow_seed((unsigned)sm.h.sample_index, (unsigned)__float_as_int(p.w), (unsigned)k);
    if (pos < L.wl_cap) {
      L.wl[pos] = make_float4(p.x, p.y, p.z, __uint_as_float(seed0));
      L.wrange[pos] = rg;
    } else {  // work list full (very dense neighbourhood): cast this point's draws in place
      unsigned seed = seed0;
      const int r0 = (int)(rg & 0xFFFFu), r1 = (int)(rg >> 16);
      for (int t = 0; t < P.nsp; t++) {
        int r = (int)gpdb_fastrand(&seed);
        if (r >= r0 && r <= r1) set_bit(bm, draw_bit(P, sm, vb, (double)p.x, (double)p.y, (double)p.z, seed, k));
      }
    }
  };
  if (use_ball) {  // independent loads, all lanes busy (uniform)
    for (int i0 = 0; i0 < nball; i0 += NT_IMG) {
      const int i = i0 + tid;
      float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
      unsigned rg = 0;
      bool ok = false;
      if (i < nball) {
        p = __ldg(cl.pts4 + ball_at(i));
        ok = cull(sm, k, p, rg);
      }
      append(ok, p, rg);
    }
  } else {
    scan_balanced<NT_IMG>(Gd, cl, sr, sm.seg, [&](bool in, const float4 &p, int) {
      unsigned rg = 0;
      const bool ok = in && l2_simple(q, p.x, p.y, p.z) < P.r2_img && cull(sm, k, p, rg);
      append(ok, p, rg);
    });
    if (count_walks && prof && tid == 0) atomicAdd(prof + 14, 1ull);
  }
  __syncthreads();
  sub_phase(prof, SUB_CULL, t_sub);
  const int nw = min(sm.wl_n, L.wl_cap);
  if (prof && tid == 0) {
    atomicAdd(prof + 9, (unsigned long long)nw);
    if (sm.wl_n > L.wl_cap) atomicAdd(prof + GPDB_PROF_PATH + L.path_cast, (unsigned long long)(sm.wl_n - L.wl_cap));
  }
  const int nsp = P.nsp;
  const unsigned nsp_magic = nsp > 1 ? (unsigned)((0x100000000ull + (unsigned)nsp - 1) / (unsigned)nsp) : 0u;  // ceil(2^32 / nsp)
  const int nd = nw * nsp;
  // window test of every draw, survivors compacted: WT draws per thread between two slot reservations, so that a warp
  // takes one scan and one shared-memory atomic per 32 WT draws (the loop was bound by that chain, not by the test)
  constexpr int WT = 4;
  const int lane = tid & 31;
  for (int w0 = 0; w0 < nd; w0 += WT * NT_IMG) {
    unsigned code[WT], pm = 0;
#pragma unroll
    for (int j = 0; j < WT; j++) {
      const int w = w0 + j * NT_IMG + tid;
      code[j] = 0;
      if (w < nd) {
        // w / nsp by multiply-high: exact for w < 2^32 / nsp (w < WL_CAP * nsp < 2^20)
        const int item = nsp > 1 ? (int)__umulhi((unsigned)w, nsp_magic) : w, t = w - item * nsp;
        const unsigned seed = sm.lcgA[t] * __float_as_uint(L.wl[item].w) + sm.lcgC[t];
        const unsigned rg = L.wrange[item];
        const int r = (int)((seed >> 16) & 0x7FFFu);
        if (r >= (int)(rg & 0xFFFFu) && r <= (int)(rg >> 16)) pm |= 1u << j;
        code[j] = ((unsigned)item << 7) | (unsigned)t;
      }
    }
    const int cnt = __popc(pm);
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    int pos = 0;
    if (lane == 31 && incl) pos = atomicAdd(&sm.dl_n, incl);
    pos = __shfl_sync(0xffffffffu, pos, 31) + incl - cnt;
#pragma unroll
    for (int j = 0; j < WT; j++) {
      if (!((pm >> j) & 1u)) continue;
      if (pos < L.dl_cap) L.dlist[pos] = code[j];
      else {  // list full: evaluate in place
        const float4 e = L.wl[code[j] >> 7];
        const int t = (int)(code[j] & 127u);
        const unsigned seed = sm.lcgA[t] * __float_as_uint(e.w) + sm.lcgC[t];
        set_bit(bm, draw_bit(P, sm, vb, (double)e.x, (double)e.y, (double)e.z, seed, k));
      }
      pos++;
    }
  }
  __syncthreads();
  sub_phase(prof, SUB_WINDOW, t_sub);
  const int ndl = min(sm.dl_n, L.dl_cap);
  if (tid == 0) sm.wl_n = 0;  // for the next camera: every read of this camera's count lies before the barrier above
  if (prof && tid == 0) {
    atomicAdd(prof + 10, (unsigned long long)sm.dl_n);
    if (sm.dl_n > L.dl_cap) atomicAdd(prof + GPDB_PROF_PATH + L.path_draw, (unsigned long long)(sm.dl_n - L.dl_cap));
  }
  auto list_bit = [&](int i) -> int {
    if (i >= ndl) return -1;
    const unsigned code = L.dlist[i];
    const float4 e = L.wl[code >> 7];
    const int t = (int)(code & 127u);
    const unsigned seed = sm.lcgA[t] * __float_as_uint(e.w) + sm.lcgC[t];
    return draw_bit(P, sm, vb, (double)e.x, (double)e.y, (double)e.z, seed, k);
  };
  for (int i = tid; i < ndl; i += 2 * NT_IMG) {  // two independent float64 chains per thread
    const int bit_a = list_bit(i), bit_b = list_bit(i + NT_IMG);
    set_bit(bm, bit_a);
    set_bit(bm, bit_b);
  }
}

// set intersection over the cameras that see the neighbourhood, into bitmap 0, starting from camera 0's set even when it
// is empty (hand_set.cpp:153-176)
__device__ __forceinline__ void intersect_bitmaps(unsigned *bitmap, int bm_words, int K, int cam_set) {
  if (K < 2) return;
  for (int wd = threadIdx.x; wd < bm_words; wd += NT_IMG) {
    unsigned acc = bitmap[wd];
    for (int k = 1; k < K; k++)
      if ((cam_set >> k) & 1) acc &= bitmap[(size_t)k * bm_words + wd];
    bitmap[wd] = acc;
  }
}

// One shadow voxel (code b0 | b1 << 8 | b2 << 16 in the bitmap AABB): the exact float64 box test of its jittered point,
// then its entry into the sum tiles of projections [pj_lo, pj_hi) (tile pj - pj_lo, S S cells each). Returns projection
// 2's entry (cell | 1 << 31, fixed-point coordinate), zero when the point lies outside the box. evt (may be null) counts
// the entries whose cell another active lane of the warp hits in the same update.
__device__ __forceinline__ uint2 eval_voxel(const DevParams &P, const gpdb_pose &h, const double *qtab, const double (&inv)[3],
                                            int S, const VoxelBox &vb, unsigned long long *tiles, unsigned code, int pj_lo,
                                            int pj_hi, unsigned long long *evt = nullptr) {
  int b0 = code & 255, b1 = (code >> 8) & 255, b2 = code >> 16;
  double x, y, z;
  if (!voxel_point_in_box(P, h, qtab, b0 + vb.o0, b1 + vb.o1, b2 + vb.o2, x, y, z)) return make_uint2(0u, 0u);
  double u[3];
  int cellv[3];
  unit_cells(P, h, inv, S, x, y, z, u, cellv);
  uint2 st = make_uint2(0u, 0u);
#pragma unroll
  for (int pj = 0; pj < 3; pj++) {
    const Proj pr(pj);
    const int pix = (S - 1 - cellv[pr.a0]) * S + cellv[pr.a1];
    const unsigned qv = unit_q32(u[pr.a2]);
    if (pj >= pj_lo && pj < pj_hi) {
      if (evt && __popc(__match_any_sync(__activemask(), pj * S * S + pix)) > 1) atomicAdd(evt, 1ull);
      cell_add(tiles + (size_t)(pj - pj_lo) * S * S + pix, qv);
    }
    if (pj == 2) st = make_uint2((unsigned)pix | 0x80000000u, qv);
  }
  return st;
}

// createShadowImage (image_strategy.cpp:193-233) of one sum tile into one plane (rows of rs bytes): mean per cell, value =
// max over the occupied cells - mean on the occupied cells. The general path writes its float image over the tile.
template <class Sm>
__device__ __forceinline__ void shadow_channel(Sm &sm, const double *rcp, int S, unsigned long long *tile, uint8_t *plane,
                                               int rs) {
  constexpr int PIXT = (MAXPIX + NT_IMG - 1) / NT_IMG;
  const int tid = threadIdx.x, SS = S * S;
  float avgr[PIXT];
  unsigned occm = 0;
  float mm[2] = {-FLT_MAX, -FLT_MAX};  // max avg, -(min avg) over the occupied cells
#pragma unroll
  for (int t = 0; t < PIXT; t++) {
    const int pix = tid + t * NT_IMG;
    avgr[t] = 0.0f;
    bool oc = false;
    if (pix < SS) {
      const unsigned long long acc = tile[pix];
      const unsigned cntc = (unsigned)(acc >> 48);
      if (cntc) {
        avgr[t] = (float)cell_mean(acc, rcp);
        occm |= 1u << t;
        oc = true;
        mm[0] = fmaxf(mm[0], avgr[t]);
        mm[1] = fmaxf(mm[1], -avgr[t]);
      }
    }
    if (t * NT_IMG < SS) occ_ballot<NT_IMG>(sm.occf, t, oc);
  }
  bool covered;
  block_max<NT_IMG, 2>(mm, sm.fred, sm.occf, S, &covered);  // (its barriers publish the occupancy words)
  const bool any = mm[0] != -FLT_MAX;
  const float maxf = any ? mm[0] : 0.0f;
  const float vmax = any ? maxf - (-mm[1]) : 0.0f;  // largest cell value = max avg - min avg
  float vmin = 0.0f;
  if (covered) {  // general path: min over the dilated float image
    float *srcF = reinterpret_cast<float *>(tile);
    __syncthreads();
#pragma unroll
    for (int t = 0; t < PIXT; t++) {
      const int pix = tid + t * NT_IMG;
      if (pix < SS) srcF[pix] = ((occm >> t) & 1) ? (maxf - avgr[t]) : 0.0f;
    }
    __syncthreads();
    float neg[1] = {-dilated_min<NT_IMG>(srcF, S)};
    block_max<NT_IMG, 1>(neg, sm.fred);
    vmin = -neg[0];
  }
  const Quant qs(vmin, vmax);
  const unsigned bg = qs(0.0f);
#pragma unroll
  for (int t = 0; t < PIXT; t++) {
    const int pix = tid + t * NT_IMG;
    if (pix < SS) {
      const bool oc = (occm >> t) & 1;
      if (oc || bg) plane[pix + (pix / S) * (rs - S)] = (uint8_t)(oc ? qs(maxf - avgr[t]) : bg);  // row * rs + column
    }
  }
}

// Dilate (3x3 max, border ignored) the quantised planes four pixels at a time and assemble the 16-byte pixels (gout: S x
// S). plane(ch): the plane of reference channel ch, rows of RW words; pixels past column S - 1 are not stored.
template <class PL>
__device__ __forceinline__ void dilate_assemble(int S, int RW, int C, PL &&plane, uint4 *gout) {
  for (int g = threadIdx.x; g < S * RW; g += NT_IMG) {
    const int row = g / RW, c4 = g - row * RW;
    // 3x3 max of 4 pixels x 1 channel per word. Bytes are split into their even / odd 16-bit lanes (E = [b0, b2],
    // O = [b1, b3]) so that every max is ONE native VIMNMX3.U16x2 (the 8-bit SIMD max is emulated): vertical
    // max of the three rows first (centre word: E and O; left word: only O, whose high lane is pixel -1; right word:
    // only E, whose low lane is pixel +4), then the horizontal neighbours by lane shifts.
    unsigned res[16];
    const bool up = row > 0, dn = row + 1 < S, lf = c4 > 0, rt = c4 + 1 < RW;
#pragma unroll
    for (int ch = 0; ch < 16; ch++) {
      res[ch] = 0u;
      if (ch < C) {
        const unsigned *W = reinterpret_cast<const unsigned *>(plane(ch)) + row * RW + c4;
        const unsigned m0 = W[0], u0 = up ? W[-RW] : 0u, d0 = dn ? W[RW] : 0u;
        const unsigned ml = lf ? W[-1] : 0u, ul = (up && lf) ? W[-RW - 1] : 0u, dl = (dn && lf) ? W[RW - 1] : 0u;
        const unsigned mr = rt ? W[1] : 0u, ur = (up && rt) ? W[-RW + 1] : 0u, dr = (dn && rt) ? W[RW + 1] : 0u;
        const unsigned E = __vimax3_u16x2(__byte_perm(u0, 0u, 0x4240), __byte_perm(m0, 0u, 0x4240), __byte_perm(d0, 0u, 0x4240));
        const unsigned O = __vimax3_u16x2(__byte_perm(u0, 0u, 0x4341), __byte_perm(m0, 0u, 0x4341), __byte_perm(d0, 0u, 0x4341));
        const unsigned LO = __vimax3_u16x2(__byte_perm(ul, 0u, 0x4341), __byte_perm(ml, 0u, 0x4341), __byte_perm(dl, 0u, 0x4341));
        const unsigned RE = __vimax3_u16x2(__byte_perm(ur, 0u, 0x4240), __byte_perm(mr, 0u, 0x4240), __byte_perm(dr, 0u, 0x4240));
        const unsigned En = __vimax3_u16x2(E, O, __byte_perm(LO, O, 0x5432));   // [max(p-1,p0,p1), max(p1,p2,p3)]
        const unsigned On = __vimax3_u16x2(O, E, __byte_perm(E, RE, 0x5432));   // [max(p0,p1,p2), max(p2,p3,p4)]
        res[ch] = __byte_perm(En, On, 0x6240);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if (c4 * 4 + i < S) {
        const unsigned sel = (unsigned)i | ((unsigned)(4 + i) << 4);
        uint4 o;
        o.x = __byte_perm(__byte_perm(res[0], res[1], sel), __byte_perm(res[2], res[3], sel), 0x5410);
        o.y = __byte_perm(__byte_perm(res[4], res[5], sel), __byte_perm(res[6], res[7], sel), 0x5410);
        o.z = __byte_perm(__byte_perm(res[8], res[9], sel), __byte_perm(res[10], res[11], sel), 0x5410);
        o.w = __byte_perm(__byte_perm(res[12], res[13], sel), __byte_perm(res[14], res[15], sel), 0x5410);
        gout[row * S + c4 * 4 + i] = o;
      }
    }
  }
}

// ---- k_images: the general tier (and the overflow tier of k_images2), one CTA per SM.
// dynamic shared memory: planes C x S x RS bytes (RS = S rounded up to 4) | tiles 3 x 8 S S | box list 36 B x BOX_CAP
// (the shadow bitmaps + voxel list alias the box list; the shadow work list aliases the tiles)
// GL = true is the last tier: the box list (and the float images of the general min path) live in a per-CTA slice of global
// memory (`gl_base`, `gl_cap` points: L2-resident scratch) instead of shared memory, for clouds so dense that an image box
// holds more than BOX_CAP points (the reference has no limit; image_generator.cpp:54-64).
template <int S_T, bool GL, bool BATCH>
__global__ void __launch_bounds__(NT_IMG, 1) k_images(const DevParams *Pp, DevCloud cl0, CloudTable tab, const gpdb_pose *cand, int nc,
                                                      uint8_t *p16, const double *qtab, int *err, int plane_bytes,
                                                      int list_bytes, unsigned long long *prof, const int *work,
                                                      const int *work_n, unsigned char *gl_base, int gl_cap, int *ovf2,
                                                      int *ovf2_count) {
  // work != nullptr: only the images work[0 .. *work_n) (the overflow list of the previous tier); ovf2 != nullptr: images
  // whose box list overflows THIS tier are appended there (and redone by the next one) instead of being an error
  long long t_phase = 0;
  const DevParams &P = *Pp;
  extern __shared__ __align__(16) unsigned char dyn[];
  __shared__ ImgSmem sm;
  const int S = S_T > 0 ? S_T : P.S, C = P.C, SS = S * S;
  const int RS = (S + 3) & ~3, PLB = S * RS;
  uint8_t *planes = dyn;
  unsigned long long *tileA = reinterpret_cast<unsigned long long *>(dyn + plane_bytes);
  unsigned long long *tileB = tileA + SS;
  unsigned long long *tileC = tileB + SS;
  unsigned char *lbase = reinterpret_cast<unsigned char *>(tileC + SS);
  const int BC = GL ? gl_cap : BOX_CAP;
  const BoxList bl(GL ? gl_base + (size_t)blockIdx.x * ((size_t)gl_cap * 36 + (size_t)16 * SS) : lbase, BC);
  float *bnrm = reinterpret_cast<float *>(bl.cell + BC);  // [3][CAP]: |R^T n| of each box point
  float *gF = bnrm + 3 * BC;                              // GL: 4 float images of the general min path
  unsigned *bitmap = reinterpret_cast<unsigned *>(lbase);  // aliases the list (shadow phase)
  // the in-ball list of scan 1 lives in tile C, which nothing else touches before the shadow phase
  int *ball = reinterpret_cast<int *>(tileC);
  const int BALL_CAP = 2 * SS;  // 8 S S bytes / 4
  const int tid = threadIdx.x;
  const int nproj = (C >= 12) ? 3 : 1;
  const int per = (C == 15) ? 5 : 4;
  const bool do_nrm = C != 1, do_dep = C == 1 || C >= 12;
  img_cta_init(sm, P);

  const int n_work = work ? *work_n : nc;
  for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
    const int b = work ? work[wi] : wi;
    img_begin(sm, cand + b);
    for (int k = tid; k < plane_bytes >> 4; k += NT_IMG) reinterpret_cast<uint4 *>(planes)[k] = make_uint4(0, 0, 0, 0);
    for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(tileA)[k] = make_uint4(0, 0, 0, 0);  // tiles A, B: clean
    __syncthreads();
    PHASE(1);   // image start
    const gpdb_pose &h = sm.h;
    const auto &G = CloudSel<BATCH>::get(tab, h.sample_slot);
    const DevCloud cl = CloudSel<BATCH>::local(G, cl0);
    const double inv[3] = {1.0 / P.vol_d, 1.0 / P.vol_w, 1.0 / (2.0 * P.vol_h)};
    const float q[3] = {(float)h.sample[0], (float)h.sample[1], (float)h.sample[2]};
    const SegRange sr = seg_range(G, q, P.rf_img);
    ball_scan1(P, G, cl, sr, q, sm, C, ball, BALL_CAP, bl, [](int) {});
    if (tid == 0 && sm.box_n > BC) {
      if (ovf2) ovf2[atomicAdd(ovf2_count, 1)] = b;  // redone by the next tier (larger list)
      else {
        atomicAdd(err + 2, 1);
        sm.box_n = BC;
      }
    }
    __syncthreads();
    PHASE(2);  // scan 1 + reductions done
    if (sm.box_n > BC) continue;  // handed to the next tier (uniform; without a next tier box_n was clamped)
    const int bn = sm.box_n;
    double *rcp = &sm.red[0][0];  // the scan's reduction scratch is idle from here to the next image: reciprocal table (cell_mean)
    if (tid < RCP_N) rcp[tid] = 1.0 / ((double)tid * 4294967296.0);  // visible after the barrier that ends the box-point pass
    bool nonunit = false;
    box_units(P, h, inv, bl, bn, S, [&](int k) {
      const double *nn = cl.nrm + 3 * (size_t)(unsigned)(bl.keys[k] & 0xffffffffull);
      double n0, n1, n2;
      to_frame(h.frame, nn[0], nn[1], nn[2], n0, n1, n2);
      bnrm[k] = (float)fabs(n0);
      bnrm[BC + k] = (float)fabs(n1);
      bnrm[2 * BC + k] = (float)fabs(n2);
      if (!unit_normal(nn)) nonunit = true;
    });
    // a normal of other than unit length in the box: the cells replay createNormalsImage's fold (unit_normal, common.cuh)
    const bool exact_fold = __syncthreads_or(nonunit) != 0;

    // ---- points phase
    for (int pj = 0; pj < nproj; pj++) {
      const Proj pr(pj);
      raster_projection(bl, bn, S, pr, tileA, tileB, sm.occf);
      // the winner of a cell (its point with the largest key) carries the cell's values: |n| of that point, 1 - mean depth
      auto cell_values = [&](int k, int &row, int &col, float &n0, float &n1, float &n2, float &dv) -> bool {
        const unsigned cc = bl.cell[k];
        row = pr.row(cc, S);
        col = pr.col(cc);
        const int pix = row * S + col;
        if (tileA[pix] != bl.keys[k]) return false;
        n0 = bnrm[k];
        n1 = bnrm[BC + k];
        n2 = bnrm[2 * BC + k];
        if (exact_fold) {
          // replay the cell's writers in ascending key ((dist, index)) order, ending with this winner: v = |n| into an
          // empty cell, else v += (|n| - v) * (1 / sqrt(v.v)) in the oracle's float / double steps. O(writers x bn), only
          // for images that hold a normal of other than unit length.
          float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
          unsigned long long cur = 0ull;
          bool first = true;
          for (;;) {
            unsigned long long nxt = ~0ull;
            int jn = k;
            for (int j = 0; j < bn; j++) {
              const unsigned long long kj = bl.keys[j];
              if (pr.pix(bl.cell[j], S) == pix && (first || kj > cur) && kj < nxt) {
                nxt = kj;
                jn = j;
              }
            }
            const float b0 = bnrm[jn], b1 = bnrm[BC + jn], b2 = bnrm[2 * BC + jn];
            if (v0 == 0.0f && v1 == 0.0f && v2 == 0.0f) {
              v0 = b0;
              v1 = b1;
              v2 = b2;
            } else {
              const double f = 1.0 / (double)sqrtf(v0 * v0 + v1 * v1 + v2 * v2);
              const float d0 = (float)((double)(b0 - v0) * f), d1 = (float)((double)(b1 - v1) * f),
                          d2 = (float)((double)(b2 - v2) * f);
              v0 += d0;
              v1 += d1;
              v2 += d2;
            }
            if (jn == k) break;
            cur = nxt;
            first = false;
          }
          n0 = v0;
          n1 = v1;
          n2 = v2;
        }
        const float avg = (float)cell_mean(tileB[pix], rcp);
        dv = (float)(1.0 - (double)avg);
        return true;
      };
      // every winner of the box list, re-derived: emit(byte offset in the plane, values)
      auto listed_winners = [&](auto &&emit) {
        for (int k = tid; k < bn; k += NT_IMG) {
          int row, col;
          float n0, n1, n2, dv;
          if (cell_values(k, row, col, n0, n1, n2, dv)) emit(row * RS + col, n0, n1, n2, dv);
        }
      };
      float mxv[2] = {0.0f, 0.0f};  // max of the normals group / of the depth channel (all values are >= 0)
      listed_winners([&](int, float n0, float n1, float n2, float dv) {
        mxv[0] = fmaxf(mxv[0], fmaxf(fmaxf(n0, n1), n2));
        mxv[1] = fmaxf(mxv[1], dv);
      });
      bool covered;
      block_max<NT_IMG, 2>(mxv, sm.fred, sm.occf, S, &covered);  // (its barriers publish the occupancy words)
      float mnv[2] = {0.0f, 0.0f};  // min over the dilated image: 0 when an all-empty 3x3 window exists
      const int cb = (C == 1) ? 0 : pj * per;
      const PointPlanes pp = {planes, PLB, RS, cb, cb + (C == 1 ? 0 : 3), do_nrm, do_dep};
      if (!covered) {
        winners_to_planes(pp, mnv, mxv, false, listed_winners);
        __syncthreads();  // every winner has read its cell
        wipe_cells(bl, bn, S, pr, tileA, tileB, sm.occf);
      } else {
        if constexpr (GL) {
          // general path, global-list tier: the float images live in the CTA's global slice, the tiles stay intact and the
          // winners are simply re-derived (cell_values) — no per-thread value cache sized by the list capacity
          for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(gF)[k] = make_uint4(0, 0, 0, 0);
          __syncthreads();
          for (int k = tid; k < bn; k += NT_IMG) {
            int row, col;
            float v[4];
            if (cell_values(k, row, col, v[0], v[1], v[2], v[3]))
#pragma unroll
              for (int c = 0; c < 4; c++) gF[c * SS + row * S + col] = v[c];
          }
          __syncthreads();
          points_dilated_min(gF, S, sm.fred, mnv);
          winners_to_planes(pp, mnv, mxv, true, listed_winners);
          __syncthreads();
        } else {
          // general path: materialise the four float channel images over the (now dead) tiles and take the min of their
          // dilations. Winners keep their values in registers across the rewrite of the tiles.
          constexpr int JMAX = (BOX_CAP + NT_IMG - 1) / NT_IMG;
          float wv[JMAX][4];
          int wpix[JMAX];
#pragma unroll
          for (int j = 0; j < JMAX; j++) {
            const int k = tid + j * NT_IMG;
            wpix[j] = -1;
            int row, col;
            if (k < bn && cell_values(k, row, col, wv[j][0], wv[j][1], wv[j][2], wv[j][3])) wpix[j] = row * S + col;
          }
          __syncthreads();
          float *F = reinterpret_cast<float *>(tileA);  // 4 x SS floats = tileA + tileB
          for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(F)[k] = make_uint4(0, 0, 0, 0);
          __syncthreads();
#pragma unroll
          for (int j = 0; j < JMAX; j++)
            if (wpix[j] >= 0)
#pragma unroll
              for (int c = 0; c < 4; c++) F[c * SS + wpix[j]] = wv[j][c];
          __syncthreads();
          points_dilated_min(F, S, sm.fred, mnv);
          winners_to_planes(pp, mnv, mxv, true, [&](auto &&emit) {
#pragma unroll
            for (int j = 0; j < JMAX; j++)
              if (wpix[j] >= 0) emit(wpix[j] / S * RS + wpix[j] % S, wv[j][0], wv[j][1], wv[j][2], wv[j][3]);
          });
        }
        for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(tileA)[k] = make_uint4(0, 0, 0, 0);  // clean tiles A, B
        for (int k = tid; k < MAXPIX / 32; k += NT_IMG) sm.occf[k] = 0u;
      }
      __syncthreads();
    }

    PHASE(3);  // points phase (3 projections) done
    if (C == 15) {
      const int K = G.K, bm_words = 2 * P.bm_dim * P.bm_dim;  // rows of 64 bits along x (bm_dim <= 64)
      shadow_setup(P, G, sm, qtab[GPDB_QTAB_SIZE - 1], bitmap, bm_words * K);
      __syncthreads();
      PHASE(4);  // shadow setup done
      const VoxelBox vb(sm);
      const int cam_set = sm.cam_or;
      // work list over tiles A + B (tile C holds the ball list until the first camera's casting is done), then the
      // draw list over tile C
      float4 *wl = reinterpret_cast<float4 *>(tileA);
      const int WL_CAP = (2 * SS * 8) / 20;
      const CastLists L = {wl, reinterpret_cast<unsigned *>(wl + WL_CAP), WL_CAP, reinterpret_cast<unsigned *>(tileC), 2 * SS,
                           PATH_IMG_CAST, PATH_IMG_DRAW};
      bool use_ball = sm.ball_n <= BALL_CAP;
      for (int k = 0; k < K; k++) {
        if (!((cam_set >> k) & 1)) continue;  // camera_set(i) >= 1 (hand_set.cpp:141)
        cast_camera(P, G, cl, sr, q, sm, vb, k, bitmap + (size_t)k * bm_words, L, use_ball, sm.ball_n,
                    [&](int i) { return ball[i]; }, prof, false);
        use_ball = false;  // the draw list has overwritten the ball list: a further camera walks the grid again
      }
      __syncthreads();
      PHASE(5);  // S1 (casting) done
      intersect_bitmaps(bitmap, bm_words, K, cam_set);
      for (int k = tid; k < (3 * SS) >> 1; k += NT_IMG) reinterpret_cast<uint4 *>(tileA)[k] = make_uint4(0, 0, 0, 0);
      // odd image size: the 16-byte stores stop one cell short of tile C's end (its last pixel would keep the ball /
      // draw list or the previous image's sums); the bitmaps follow, so no store may go further
      if ((SS & 1) && tid == 0) tileA[3 * SS - 1] = 0ull;
      if (tid == 0) sm.wl_n = 0;
      __syncthreads();
      // the voxel list (4 B codes) behind bitmap 0, over the other (dead) bitmaps and the box list
      unsigned *blist = bitmap + bm_words;
      const int BL_CAP = list_bytes / 4 - bm_words;
      expand_bitmap(bitmap, 64 * vb.d1 * vb.d2, vb.d1, &sm.wl_n, [&](int pos, unsigned code) {
        if (pos < BL_CAP) blist[pos] = code;
        else eval_voxel(P, h, qtab, inv, S, vb, tileA, code, 0, 3);  // list full: evaluate in place
      });
      __syncthreads();
      const int nset = min(sm.wl_n, BL_CAP);
      if (prof && tid == 0) {
        atomicAdd(prof + 11, (unsigned long long)sm.wl_n);
        atomicAdd(prof + 12, (unsigned long long)bn);
        atomicAdd(prof + 13, (unsigned long long)sm.n_img);
        if (sm.wl_n > BL_CAP) atomicAdd(prof + GPDB_PROF_PATH + PATH_IMG_STASH, 1ull);
        if (sm.ball_n > BALL_CAP) atomicAdd(prof + GPDB_PROF_PATH + PATH_IMG_BALL, 1ull);
      }
      for (int i = tid; i < nset; i += NT_IMG) eval_voxel(P, h, qtab, inv, S, vb, tileA, blist[i], 0, 3);
      __syncthreads();
      PHASE(6);  // S2 bitmap pass done
      for (int pj = 0; pj < 3; pj++) shadow_channel(sm, rcp, S, tileA + (size_t)pj * SS, planes + (size_t)(pj * 5 + 4) * PLB, RS);
      // the points phase of the next image expects a clean occupancy bitmap
      __syncthreads();
      for (int k = tid; k < MAXPIX / 32; k += NT_IMG) sm.occf[k] = 0u;
    }
    __syncthreads();
    PHASE(7);  // shadow images done
    dilate_assemble(S, RS >> 2, C, [&](int ch) { return planes + (size_t)ch * PLB; }, reinterpret_cast<uint4 *>(p16) + (size_t)b * SS);
    PHASE(8);  // assembled image stored
  }
}

// ------------------------------------------------------------------------------------------------
// k_images2: the fast path of the image stage — the same algorithm as k_images in 103 KB of shared memory and 64
// registers, so that TWO 512-thread CTAs share an SM (k_images needs 214 KB: one CTA per SM, 16 warps, issue slots idle
// behind barriers and dependent-issue stalls). What makes the footprint fit:
//   * the box list holds 1024 points (24 B each: key, unit coordinates, cells; the normal of a WINNER is re-read from the
//     cloud); images with more box points are appended to `ovf` and redone by k_images (2048 points, one CTA per SM);
//   * two 64-bit tiles instead of three: the shadow sums of projections 0 and 1 are taken first, the per-voxel result for
//     projection 2 (cell + fixed-point coordinate) is stashed next to the voxel code and summed in a second, cheap pass;
//   * the quantised POINT channels are scattered straight into the image's own (still unused) 57.6 KB of HBM / L2 as twelve
//     byte planes and read back into the dead tiles before the dilation; only the three shadow planes stay in shared memory.
// Requires image_size 60 and, at 15 channels, at most two cameras whose shadow bitmaps fit the box list with 2 KB to spare
// (see geo_images; otherwise k_images does all the work). Images with a normal of other than unit length in the box are
// handed to k_images too (its exact fold). Results are bit-identical to k_images.
// ------------------------------------------------------------------------------------------------
constexpr int BOX_CAP2 = 1024;
// the in-ball list of the shadow casting fills the image's 57.6 KB slot behind the 43.2 KB of point planes
constexpr int IMG2_S = 60;  // the only image size of the fast path
constexpr int BALL_CAP2 = (IMG2_S * IMG2_S * 16 - 12 * IMG2_S * IMG2_S) / 4;
using Img2Smem = ImgSmemT<2>;
// two CTAs per SM: 2 x (dynamic + static + the 1 KB the hardware reserves per CTA) within Hopper's 228 KB per SM
constexpr size_t IMG2_DYN_SMEM = (size_t)2 * 8 * IMG2_S * IMG2_S + (size_t)3 * IMG2_S * IMG2_S + (size_t)BOX_CAP2 * 36;
static_assert(2 * (IMG2_DYN_SMEM + sizeof(Img2Smem) + 1024) <= 228 * 1024, "k_images2 no longer fits two CTAs per SM");

template <bool BATCH>
__global__ void __launch_bounds__(NT_IMG, 2) k_images2(const DevParams *Pp, DevCloud cl0, CloudTable tab, const gpdb_pose *cand, int nc,
                                                       uint8_t *p16, const double *qtab, int *ovf, int *ovf_count,
                                                       unsigned long long *prof) {
  long long t_phase = 0, t_sub = 0;
  const DevParams &P = *Pp;
  extern __shared__ __align__(16) unsigned char dyn[];
  __shared__ Img2Smem sm;
  constexpr int S = IMG2_S, SS = S * S, RW = S / 4, PLB = SS;  // 15 words per row, 3600-byte planes
  constexpr int JW = (BOX_CAP2 + NT_IMG - 1) / NT_IMG;  // box points per thread
  const int C = P.C;
  unsigned long long *tileA = reinterpret_cast<unsigned long long *>(dyn);
  unsigned long long *tileB = tileA + SS;
  uint8_t *splanes = reinterpret_cast<uint8_t *>(tileB + SS);       // 3 shadow planes
  unsigned char *lbase = splanes + 3 * PLB;
  constexpr int LIST_BYTES = BOX_CAP2 * 36;                         // 24 B per box point + room for the shadow phase
  const BoxList bl(lbase, BOX_CAP2);
  unsigned *bitmap = reinterpret_cast<unsigned *>(lbase);           // shadow phase: aliases the (dead) box list
  uint8_t *tplanes = reinterpret_cast<uint8_t *>(tileA);            // final stage: the 12 point planes over the dead tiles
  const int tid = threadIdx.x;
  const int nproj = (C >= 12) ? 3 : 1;
  const bool do_nrm = C != 1, do_dep = C == 1 || C >= 12;
  const int npp = (C == 15 || C == 12) ? 12 : C;  // point planes (C = 1: the depth plane is plane 0)
  img_cta_init(sm, P);

  for (int b = blockIdx.x; b < nc; b += gridDim.x) {
    img_begin(sm, cand + b);
    uint8_t *gimg = p16 + (size_t)b * SS * 16;  // the image's own memory: first the point planes, finally the pixels
    // ... and behind the twelve point planes, the list of in-ball points that the shadow casting walks once per camera
    int *ball = reinterpret_cast<int *>(gimg + 12 * PLB);
    for (int k = tid; k < (npp * PLB) >> 4; k += NT_IMG) reinterpret_cast<uint4 *>(gimg)[k] = make_uint4(0, 0, 0, 0);
    for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(tileA)[k] = make_uint4(0, 0, 0, 0);  // tiles A, B
    for (int k = tid; k < (3 * PLB) >> 4; k += NT_IMG) reinterpret_cast<uint4 *>(splanes)[k] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    PHASE(1);
    const gpdb_pose &h = sm.h;
    const auto &G = CloudSel<BATCH>::get(tab, h.sample_slot);
    const DevCloud cl = CloudSel<BATCH>::local(G, cl0);
    const double inv[3] = {1.0 / P.vol_d, 1.0 / P.vol_w, 1.0 / (2.0 * P.vol_h)};
    const float q[3] = {(float)h.sample[0], (float)h.sample[1], (float)h.sample[2]};
    const SegRange sr = seg_range(G, q, P.rf_img);
    ball_scan1(P, G, cl, sr, q, sm, C, ball, BALL_CAP2, bl, [&](int idx) {
      if (G.nonunit && !unit_normal(cl.nrm + 3 * (size_t)idx)) sm.nonunit = 1;
    });
    if (tid == 0 && (sm.box_n > BOX_CAP2 || sm.nonunit)) {
      ovf[atomicAdd(ovf_count, 1)] = b;  // redone by k_images (larger list / exact fold)
      if (prof) atomicAdd(prof + GPDB_PROF_PATH + (sm.box_n > BOX_CAP2 ? PATH_IMG2_BOX : PATH_IMG2_NONUNIT), 1ull);
    }
    __syncthreads();
    PHASE(2);
    if (sm.box_n > BOX_CAP2 || sm.nonunit) continue;  // uniform
    const int bn = sm.box_n;
    double *rcp = &sm.red[0][0];  // the scan's reduction scratch is idle from here to the next image: reciprocal table (cell_mean)
    if (tid < RCP_N) rcp[tid] = 1.0 / ((double)tid * 4294967296.0);  // visible after the barrier that ends the box-point pass
    box_units(P, h, inv, bl, bn, S, [](int) {});
    __syncthreads();

    // ---- points phase
    for (int pj = 0; pj < nproj; pj++) {
      const Proj pr(pj);
      raster_projection(bl, bn, S, pr, tileA, tileB, sm.occf);
      // winners (largest key of their cell) carry the cell's values; each thread owns <= JW box points
      float wv[JW][4];
      int wpix[JW];
      float mxv[2] = {0.0f, 0.0f};
#pragma unroll
      for (int j = 0; j < JW; j++) {
        const int k = tid + j * NT_IMG;
        wpix[j] = -1;
        if (k < bn) {
          const int pix = pr.pix(bl.cell[k], S);
          const unsigned long long key = bl.keys[k];
          if (tileA[pix] == key) {
            wpix[j] = pix;
            const double *nn = cl.nrm + 3 * (size_t)(unsigned)(key & 0xffffffffull);
            double n0, n1, n2;
            to_frame(h.frame, nn[0], nn[1], nn[2], n0, n1, n2);
            wv[j][0] = (float)fabs(n0);
            wv[j][1] = (float)fabs(n1);
            wv[j][2] = (float)fabs(n2);
            const float avg = (float)cell_mean(tileB[pix], rcp);
            wv[j][3] = (float)(1.0 - (double)avg);
            mxv[0] = fmaxf(mxv[0], fmaxf(fmaxf(wv[j][0], wv[j][1]), wv[j][2]));
            mxv[1] = fmaxf(mxv[1], wv[j][3]);
          }
        }
      }
      bool covered;
      block_max<NT_IMG, 2>(mxv, sm.fred, sm.occf, S, &covered);
      float mnv[2] = {0.0f, 0.0f};
      if (covered) {  // general path: no all-empty 3x3 window -> min over the dilated float images
        float *F = reinterpret_cast<float *>(tileA);  // 4 x SS floats = tiles A + B (every winner holds its values)
        for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(F)[k] = make_uint4(0, 0, 0, 0);
        __syncthreads();
#pragma unroll
        for (int j = 0; j < JW; j++)
          if (wpix[j] >= 0)
#pragma unroll
            for (int c = 0; c < 4; c++) F[c * SS + wpix[j]] = wv[j][c];
        __syncthreads();
        points_dilated_min(F, S, sm.fred, mnv);
      }
      const int cb = (C == 1) ? 0 : pj * 4;  // first point plane of the projection
      const PointPlanes pp = {gimg, PLB, S, cb, cb + (C == 1 ? 0 : 3), do_nrm, do_dep};
      winners_to_planes(pp, mnv, mxv, covered, [&](auto &&emit) {
#pragma unroll
        for (int j = 0; j < JW; j++)
          if (wpix[j] >= 0) emit(wpix[j], wv[j][0], wv[j][1], wv[j][2], wv[j][3]);
      });
      // clean tiles / occupancy for the next projection
      if (covered) {
        for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(tileA)[k] = make_uint4(0, 0, 0, 0);
        for (int k = tid; k < MAXPIX / 32; k += NT_IMG) sm.occf[k] = 0u;
      } else {
        __syncthreads();  // every winner has read its cell
        wipe_cells(bl, bn, S, pr, tileA, tileB, sm.occf);
      }
      __syncthreads();
    }
    PHASE(3);

    if (C == 15) {
      const int K = G.K, bm_words = 2 * P.bm_dim * P.bm_dim;
      shadow_setup(P, G, sm, qtab[GPDB_QTAB_SIZE - 1], bitmap, bm_words * K);
      __syncthreads();
      PHASE(4);
      const VoxelBox vb(sm);
      const int cam_set = sm.cam_or, nball = sm.ball_n;
      // work list over tile A, draw list over tile B
      float4 *wl = reinterpret_cast<float4 *>(tileA);
      constexpr int WL_CAP = (SS * 8) / 20;
      const CastLists L = {wl, reinterpret_cast<unsigned *>(wl + WL_CAP), WL_CAP, reinterpret_cast<unsigned *>(tileB), 2 * SS,
                           PATH_IMG2_CAST, PATH_IMG2_DRAW};
      for (int k = 0; k < K; k++) {
        if (!((cam_set >> k) & 1)) continue;
        cast_camera(P, G, cl, sr, q, sm, vb, k, bitmap + (size_t)k * bm_words, L, nball <= BALL_CAP2, nball,
                    [&](int i) { return __ldcg(ball + i); },  // the list was written by this CTA: L2, not L1
                    prof, true);
      }
      __syncthreads();
      PHASE(5);
      t_sub = t_phase;
      intersect_bitmaps(bitmap, bm_words, K, cam_set);
      for (int k = tid; k < SS; k += NT_IMG) reinterpret_cast<uint4 *>(tileA)[k] = make_uint4(0, 0, 0, 0);  // tiles A, B
      if (tid == 0) sm.wl_n = 0;
      __syncthreads();
      // voxel list (8 B per voxel behind the bitmaps): .x = voxel code, later the stash for projection 2
      const int nbits = 64 * vb.d1 * vb.d2;
      // continued past the shared memory in the image's HBM slot, over the in-ball list (dead once the casting is done)
      uint2 *stash = reinterpret_cast<uint2 *>(bitmap + (((size_t)bm_words * (K > 1 ? K : 1) + 1) & ~(size_t)1));
      const int ST_SM = (LIST_BYTES - (int)((reinterpret_cast<unsigned char *>(stash)) - lbase)) / 8;
      uint2 *gstash = reinterpret_cast<uint2 *>(ball);
      const int ST_CAP = ST_SM + BALL_CAP2 / 2;
      auto st_put = [&](int i, uint2 v) {
        if (i < ST_SM) stash[i] = v;
        else __stcg(gstash + (i - ST_SM), v);
      };
      auto st_get = [&](int i) -> uint2 { return i < ST_SM ? stash[i] : __ldcg(gstash + (i - ST_SM)); };  // L2, not L1
      expand_bitmap(bitmap, nbits, vb.d1, &sm.wl_n, [&](int pos, unsigned code) {
        if (pos < ST_CAP) st_put(pos, make_uint2(code, 0u));
        else eval_voxel(P, h, qtab, inv, S, vb, tileA, code, 0, 2);  // list full: projections 0 and 1 in place (2: second walk below)
      });
      __syncthreads();
      sub_phase(prof, SUB_EXPAND, t_sub);
      const int nset_all = sm.wl_n, nset = min(nset_all, ST_CAP);
      if (prof && tid == 0) {
        atomicAdd(prof + 11, (unsigned long long)nset_all);
        atomicAdd(prof + 12, (unsigned long long)bn);
        atomicAdd(prof + 13, (unsigned long long)sm.n_img);
        if (nset_all > ST_CAP) atomicAdd(prof + GPDB_PROF_PATH + PATH_IMG2_STASH, 1ull);
      }
      unsigned long long *evt = prof ? prof + GPDB_PROF_SUB + SUB_EVT_SHARED : nullptr;
      for (int i = tid; i < nset; i += NT_IMG) st_put(i, eval_voxel(P, h, qtab, inv, S, vb, tileA, st_get(i).x, 0, 2, evt));
      __syncthreads();
      PHASE(6);
      t_sub = t_phase;
      shadow_channel(sm, rcp, S, tileA, splanes, S);
      shadow_channel(sm, rcp, S, tileB, splanes + PLB, S);
      __syncthreads();
      sub_phase(prof, SUB_CHANNELS, t_sub);
      for (int k = tid; k < SS / 2; k += NT_IMG) reinterpret_cast<uint4 *>(tileA)[k] = make_uint4(0, 0, 0, 0);  // tile A
      __syncthreads();
      sub_phase(prof, SUB_CLEARS, t_sub);
      // projection 2: from the stash, or — when the voxel list overflowed — by a second walk over the whole bitmap
      if (nset_all <= ST_CAP) {
        for (int i = tid; i < nset; i += NT_IMG) {
          const uint2 st = st_get(i);
          if (st.x & 0x80000000u) {
            if (evt && __popc(__match_any_sync(__activemask(), st.x)) > 1) atomicAdd(evt, 1ull);
            const bool carry = cell_add(tileA + (st.x & 0x7fffffffu), st.y);
            if (prof && carry) atomicAdd(prof + 0, 1ull);
          }
        }
      } else {
        expand_bitmap(bitmap, nbits, vb.d1, nullptr, [&](int, unsigned code) { eval_voxel(P, h, qtab, inv, S, vb, tileA, code, 2, 3); });
      }
      __syncthreads();
      sub_phase(prof, SUB_STASH, t_sub);
      if (prof) {  // the most shadow voxels summed into one cell of projection 2
        unsigned most = 0;
        for (int k = tid; k < SS; k += NT_IMG) most = max(most, (unsigned)(tileA[k] >> 48));
        most = __reduce_max_sync(0xffffffffu, most);
        if ((tid & 31) == 0 && most) atomicMax(prof + 1, (unsigned long long)most);
      }
      sub_phase(prof, SUB_PROBE, t_sub);
      shadow_channel(sm, rcp, S, tileA, splanes + 2 * PLB, S);
      __syncthreads();
      sub_phase(prof, SUB_CHANNELS, t_sub);
      for (int k = tid; k < MAXPIX / 32; k += NT_IMG) sm.occf[k] = 0u;
    }
    __syncthreads();
    if (C == 15) sub_phase(prof, SUB_CLEARS, t_sub);
    PHASE(7);
    // ---- the point planes come back from the image's memory into the dead tiles, then dilation + pixel assembly
    for (int k = tid; k < (npp * PLB) >> 4; k += NT_IMG)
      reinterpret_cast<uint4 *>(tplanes)[k] = __ldcg(reinterpret_cast<const uint4 *>(gimg) + k);  // written by this CTA: L2, not L1
    __syncthreads();
    // reference channel ch -> its plane: point channels in the tile region, shadow channels in splanes
    dilate_assemble(S, RW, C, [&](int ch) {
      return (C == 15) ? ((ch % 5 == 4) ? splanes + (size_t)(ch / 5) * PLB : tplanes + (size_t)(4 * (ch / 5) + ch % 5) * PLB)
                       : tplanes + (size_t)ch * PLB;
    }, reinterpret_cast<uint4 *>(gimg));
    PHASE(8);
  }
}

// P16 (16-byte pixels) <-> HWC (the cv::Mat layout, C bytes per pixel)
__global__ void k_p16_to_hwc(const uint8_t *__restrict__ p16, size_t npix, int C, uint8_t *__restrict__ hwc) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one output byte per thread
  if (i >= npix * (size_t)C) return;
  const size_t pix = i / C;
  hwc[i] = p16[pix * 16 + (i - pix * C)];
}
__global__ void k_hwc_to_p16(const uint8_t *__restrict__ hwc, size_t npix, int C, uint8_t *__restrict__ p16) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one pixel per thread
  if (i >= npix) return;
  unsigned w[4] = {0u, 0u, 0u, 0u};
  for (int c = 0; c < C; c++) w[c >> 2] |= (unsigned)hwc[i * C + c] << (8 * (c & 3));
  reinterpret_cast<uint4 *>(p16)[i] = make_uint4(w[0], w[1], w[2], w[3]);
}

// ------------------------------------------------------------------------------------------------
// batch of clouds (gpdb_set_clouds): one grid per cloud, built for all clouds in one segmented pass
// ------------------------------------------------------------------------------------------------
// per cloud: the grid over its bounds (pre_bounds_batch; float32 steps: 2 cm cells, grown x1.5 while the grid has more than
// 48e6 cells). ncell[b] = cells of cloud b. A cloud without points (gpdb_preprocess_clouds keeps a view the filter
// emptied) gets the grid of bounds 0..0: 2 x 2 x 2 cells that no search reads, since no sample and no point belongs to it
// (b_cloud_of_point passes over it).
__global__ void k_batch_desc(const int *bounds, CloudDesc *d, int B, long long *ncell) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  CloudDesc &D = d[b];
  float lo[3], hi[3];
  for (int a = 0; a < 3; a++) {
    const int mn = bounds[6 * b + a], mx = bounds[6 * b + 3 + a];  // order-preserving ints
    lo[a] = D.N > 0 ? __int_as_float(mn >= 0 ? mn : mn ^ 0x7fffffff) : 0.0f;
    hi[a] = D.N > 0 ? __int_as_float(mx >= 0 ? mx : mx ^ 0x7fffffff) : 0.0f;
  }
  float cell = 0.02f;
  double nc;
  for (;;) {
    nc = 1;
    for (int a = 0; a < 3; a++) {
      D.dim[a] = (int)floorf((hi[a] - lo[a]) / cell) + 2;
      nc *= D.dim[a];
    }
    if (nc <= 48e6) break;
    cell *= 1.5f;
  }
  for (int a = 0; a < 3; a++) D.lo[a] = lo[a];
  D.inv_cell = 1.0f / cell;
  ncell[b] = (long long)nc;
}
__global__ void k_batch_base(CloudDesc *d, const long long *base, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) d[b].cell_base = (int)base[b];
}
// cell id of every point in the store-wide numbering (cloud b's cells start at its cell_base): sorting by it orders the
// points by (cloud, cell), stable in point order
__global__ void k_batch_cell_ids(const float *xyz, const CloudDesc *d, int B, int N, int *cid, int *idx, int *counts) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const CloudDesc &D = d[b_cloud_of_point(d, B, g)];
  const int c = D.cell_base +
                (cell_of(D, xyz[3 * g + 2], 2) * D.dim[1] + cell_of(D, xyz[3 * g + 1], 1)) * D.dim[0] + cell_of(D, xyz[3 * g], 0);
  cid[g] = c;
  idx[g] = g;
  atomicAdd(counts + c + 1, 1);
}
__global__ void k_batch_fill_sorted(const float *xyz, const int *idx_sorted, const CloudDesc *d, int B, int N, float4 *pts4) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= N) return;
  const int g = idx_sorted[k];
  const int local = g - d[b_cloud_of_point(d, B, g)].off;
  pts4[k] = make_float4(xyz[3 * g], xyz[3 * g + 1], xyz[3 * g + 2], __int_as_float(local));
}
// first candidate of every cloud: candidates are in sample-slot order, cloud b owns the slots [soff[b], soff[b+1])
__global__ void k_batch_cand_off(const gpdb_pose *cand, int n, const int *soff, int B, int *cand_off) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > B) return;
  const int slot = soff[b];
  int lo = 0, hi = n;  // first candidate with sample_slot >= slot
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cand[mid].sample_slot < slot) lo = mid + 1; else hi = mid;
  }
  cand_off[b] = lo;
}
// selection keys of a batch: cloud in the high word (clouds in order), descending score below (as k_select_keys); one
// stable device-wide radix sort then orders every cloud's candidates as gpdb_detect_select would, ties in candidate order
__global__ void k_batch_select_keys(const gpdb_pose *cand, int n, const int *soff, int B, unsigned long long *keys, int *vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int slot = cand[i].sample_slot;
  int lo = 0, hi = B;  // largest b with soff[b] <= slot
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (soff[mid] <= slot) lo = mid; else hi = mid;
  }
  unsigned u = __float_as_uint(cand[i].score);
  u ^= (u >> 31) ? 0xFFFFFFFFu : 0x80000000u;
  keys[i] = ((unsigned long long)lo << 32) | ~u;
  vals[i] = i;
}
// the selected records in output order: the first sel_off[b+1] - sel_off[b] of cloud b's sorted segment
__global__ void k_batch_sel_order(const int *sorted_vals, const int *cand_off, const int *sel_off, int B, int k, int *order) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= k) return;
  int lo = 0, hi = B;  // largest b with sel_off[b] <= j
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sel_off[mid] <= j) lo = mid; else hi = mid;
  }
  order[j] = sorted_vals[cand_off[lo] + (j - sel_off[lo])];
}

}  // namespace

// ================================================================================================
// host launchers
// ================================================================================================
__global__ void k_path_add(unsigned long long *prof, int e0, const int *n0, int e1, const int *n1) {
  // atomic: the hand search of the next chunk may run on its own stream beside the image kernels of this one
  atomicAdd(prof + GPDB_PROF_PATH + e0, (unsigned long long)(unsigned)*n0);
  if (n1) atomicAdd(prof + GPDB_PROF_PATH + e1, (unsigned long long)(unsigned)*n1);
}

// path counters on: adds the lengths of the overflow lists of a tiered launch (n1 may be null) to the path counters. A
// development aid, so not counted in ctx->launches (the launch count of a call is the same with the counters on or off).
static int path_add(gpdb_ctx *ctx, int e0, const int *n0, int e1, const int *n1) {
  if (!ctx->d_prof) return GPDB_OK;
  k_path_add<<<1, 1, 0, ctx->stream>>>(ctx->d_prof, e0, n0, e1, n1);
  CUDA_TRY(cudaGetLastError());
  return GPDB_OK;
}

// SCR_OVF for a tiered launch over n samples: the tier-1 overflow list and its count, the tier-2 list and its count
static bool overflow_lists(gpdb_ctx *ctx, int n, int *&ovf, int *&ovf_count, int *&ovf2, int *&ovf2_count) {
  return gpdb_carve(ctx, SCR_OVF, [&](Carve &c) {
    ovf = c.take<int>(n); ovf_count = c.take<int>(1); ovf2 = c.take<int>(n); ovf2_count = c.take<int>(1);
  });
}

template <bool BATCH>
static int launch_frames(gpdb_ctx *ctx, const CloudSet &s, const int *d_sidx, int n, double *d_frames, uint8_t *d_valid) {
  const int cap0 = 128;  // ~44 points at the default nn_radius on a 3 mm cloud
  const size_t smem0 = (size_t)2 * LRF_WARPS * cap0 * sizeof(unsigned long long);
  const size_t smem1 = (size_t)2 * LRF_WARPS * LRF_CAP * sizeof(unsigned long long);
  CUDA_TRY(cudaFuncSetAttribute(k_frames<BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
  int *ovf, *ovf_count, *ovf2, *ovf2_count;
  if (!overflow_lists(ctx, n, ovf, ovf_count, ovf2, ovf2_count)) return GPDB_ERR_CUDA;
  const int g2 = 37;  // tier 2: 148 warps, 2 x 8 B x LRF_CAP_GLOBAL each (38 MB of scratch)
  unsigned long long *gkeys =
      (unsigned long long *)gpdb_scratch(ctx, SCR_FRAMES_GL, sizeof(unsigned long long) * 2 * LRF_CAP_GLOBAL * (size_t)g2 * LRF_WARPS);
  if (!gkeys) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemsetAsync(ovf_count, 0, sizeof(int), ctx->stream));
  CUDA_TRY(cudaMemsetAsync(ovf2_count, 0, sizeof(int), ctx->stream));
  const DevCloud &cl = s.view;
  const CloudTable tab = s.table();
  const int grid = (n + LRF_WARPS - 1) / LRF_WARPS;
  k_frames<BATCH><<<grid, LRF_WARPS * 32, smem0, ctx->stream>>>(ctx->dp, cl, tab, d_sidx, n, d_frames, d_valid, ctx->d_err, cap0,
                                                                ovf, ovf_count, ovf2, ovf2_count, nullptr, 0);
  LAUNCH_CHECK();
  // overflow tiers over the (usually empty) lists: the tier-1 grid is sized for the worst case (every sample overflowed) so
  // no host round trip is needed; warps beyond the list length exit at once
  k_frames<BATCH><<<grid, LRF_WARPS * 32, smem1, ctx->stream>>>(ctx->dp, cl, tab, d_sidx, n, d_frames, d_valid, ctx->d_err,
                                                                LRF_CAP, ovf, ovf_count, ovf2, ovf2_count, nullptr, 1);
  LAUNCH_CHECK();
  k_frames<BATCH><<<g2, LRF_WARPS * 32, 0, ctx->stream>>>(ctx->dp, cl, tab, d_sidx, n, d_frames, d_valid, ctx->d_err,
                                                          LRF_CAP_GLOBAL, ovf, ovf_count, ovf2, ovf2_count, gkeys, 2);
  LAUNCH_CHECK();
  return path_add(ctx, PATH_FRAMES_T1, ovf_count, PATH_FRAMES_T2, ovf2_count);
}

// The geometry launchers run the one-cloud instantiations (BATCH = false) when the store holds one cloud: they carry no
// per-sample cloud search and spill less.
int geo_frames(gpdb_ctx *ctx, const CloudSet &s, const int *d_sidx, int n, double *d_frames, uint8_t *d_valid) {
  if (n <= 0) return GPDB_OK;
  return s.n > 1 ? launch_frames<true>(ctx, s, d_sidx, n, d_frames, d_valid)
                 : launch_frames<false>(ctx, s, d_sidx, n, d_frames, d_valid);
}

static const int HANDS_CAP1 = 2176, HANDS_CAP2 = 12800;  // tier 1: 4 CTAs per SM (34 KB + 20 KB static each, <= 64 registers)
static const int HANDS_CAP3 = 131072;                    // last tier: neighbourhood staged in global memory (2 MB per CTA)

template <bool BATCH>
static int launch_hands(gpdb_ctx *ctx, const CloudSet &s, const int *d_sidx, int n, int slot0, const double *d_frames,
                        const uint8_t *d_valid, gpdb_pose *d_poses, uint8_t *d_flags) {
  // per call, not once per process: function attributes belong to the current device's context (one context per GPU)
  CUDA_TRY(cudaFuncSetAttribute(k_hands<BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, HANDS_CAP2 * 16));
  int *ovf, *ovf_count, *ovf2, *ovf2_count;
  if (!overflow_lists(ctx, n, ovf, ovf_count, ovf2, ovf2_count)) return GPDB_ERR_CUDA;
  float4 *glist = (float4 *)gpdb_scratch(ctx, SCR_HANDS_GL, sizeof(float4) * (size_t)HANDS_CAP3 * ctx->sm_count);
  if (!glist) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemsetAsync(ovf_count, 0, sizeof(int), ctx->stream));
  CUDA_TRY(cudaMemsetAsync(ovf2_count, 0, sizeof(int), ctx->stream));
  const DevCloud &cl = s.view;
  const CloudTable tab = s.table();
  k_hands<BATCH><<<n, NT_HANDS, HANDS_CAP1 * 16, ctx->stream>>>(ctx->dp, cl, tab, d_sidx, n, slot0, d_frames, d_valid, d_poses,
                                                                d_flags, HANDS_CAP1, nullptr, nullptr, ovf, ovf_count, nullptr,
                                                                ctx->d_err, ctx->d_prof);
  LAUNCH_CHECK();
  // large-tile pass over the samples whose neighbourhood did not fit tier 1 (persistent CTAs) ...
  k_hands<BATCH><<<ctx->sm_count, NT_HANDS, HANDS_CAP2 * 16, ctx->stream>>>(ctx->dp, cl, tab, d_sidx, n, slot0, d_frames,
                                                                            d_valid, d_poses, d_flags, HANDS_CAP2, ovf,
                                                                            ovf_count, ovf2, ovf2_count, nullptr, ctx->d_err,
                                                                            ctx->d_prof);
  LAUNCH_CHECK();
  // ... and the last tier over what did not fit that either: neighbourhood in global memory (usually an empty list)
  k_hands<BATCH><<<ctx->sm_count, NT_HANDS, 16, ctx->stream>>>(ctx->dp, cl, tab, d_sidx, n, slot0, d_frames, d_valid, d_poses,
                                                               d_flags, HANDS_CAP3, ovf2, ovf2_count, nullptr, nullptr, glist,
                                                               ctx->d_err, ctx->d_prof);
  LAUNCH_CHECK();
  return path_add(ctx, PATH_HANDS_T2, ovf_count, PATH_HANDS_T3, ovf2_count);
}

int geo_hands(gpdb_ctx *ctx, const CloudSet &s, const int *d_sidx, int n, int slot0, const double *d_frames,
              const uint8_t *d_valid, gpdb_pose *d_poses, uint8_t *d_flags) {
  if (n <= 0) return GPDB_OK;
  return s.n > 1 ? launch_hands<true>(ctx, s, d_sidx, n, slot0, d_frames, d_valid, d_poses, d_flags)
                 : launch_hands<false>(ctx, s, d_sidx, n, slot0, d_frames, d_valid, d_poses, d_flags);
}

int geo_compact(gpdb_ctx *ctx, const gpdb_pose *d_poses, const uint8_t *d_flags, int n_poses, gpdb_pose *d_cand,
                int *d_count) {
  if (n_poses <= 0) {
    CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int), ctx->stream));
    return GPDB_OK;
  }
  int *f01, *pos;
  if (!gpdb_carve(ctx, SCR_KEYS, [&](Carve &c) { f01 = c.take<int>(n_poses); pos = c.take<int>(n_poses); }))
    return GPDB_ERR_CUDA;
  const int tb = 256, gb = (n_poses + tb - 1) / tb;
  k_flag01<<<gb, tb, 0, ctx->stream>>>(d_flags, n_poses, f01);
  LAUNCH_CHECK();
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, f01, pos, n_poses, ctx->stream);
  void *tmp = gpdb_scratch(ctx, SCR_CUB, tmp_bytes);
  if (!tmp) return GPDB_ERR_CUDA;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, f01, pos, n_poses, ctx->stream));
  ctx->launches += 2;
  k_scatter<<<gb, tb, 0, ctx->stream>>>(d_poses, f01, pos, n_poses, d_cand, d_count);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// `d_p16`: nc images of S*S 16-byte pixels (see k_images). Fast path: k_images2 (two CTAs per SM) over every image, then
// k_images over the images whose box list (1 024 points) overflowed, then its global-list instance over the images whose box
// holds more than 2 048 points (up to 32 768; the overflow lists are usually empty: those launches return at once);
// k_images alone when the geometry is outside the fast path's limits (image_size != 60; at 15 channels more than two
// cameras, or shadow bitmaps that leave less than 2 KB of the box list: two cameras at the default image volume) or when
// GPD_B200_IMAGES_KERNEL=1 forces it (tests compare the kernels).
// the two k_images tiers: the box list in shared memory over `work` (every image when null), its overflow (`ovf2`)
// redone with the list in global memory (32 768 points; beyond: GPDB_ERR_CAPACITY)
template <int S_T, bool BATCH>
static int launch_general(gpdb_ctx *ctx, const CloudSet &s, const gpdb_pose *d_cand, int nc, uint8_t *d_p16, size_t smem,
                          size_t plane_bytes, size_t list_bytes, int grid, const int *d_work, const int *d_work_n,
                          unsigned char *gl, int gl_cap, int *ovf2, int *ovf2_count) {
  const DevCloud &cl = s.view;
  const CloudTable tab = s.table();
  CUDA_TRY(cudaFuncSetAttribute(k_images<S_T, false, BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CUDA_TRY(cudaFuncSetAttribute(k_images<S_T, true, BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_images<S_T, false, BATCH><<<grid, NT_IMG, smem, ctx->stream>>>(ctx->dp, cl, tab, d_cand, nc, d_p16, ctx->d_qtab, ctx->d_err,
                                                                  (int)plane_bytes, (int)list_bytes, ctx->d_prof, d_work,
                                                                  d_work_n, nullptr, 0, ovf2, ovf2_count);
  LAUNCH_CHECK();
  k_images<S_T, true, BATCH><<<ctx->sm_count, NT_IMG, smem, ctx->stream>>>(ctx->dp, cl, tab, d_cand, nc, d_p16, ctx->d_qtab,
                                                                          ctx->d_err, (int)plane_bytes, (int)list_bytes,
                                                                          ctx->d_prof, ovf2, ovf2_count, gl, gl_cap, nullptr,
                                                                          nullptr);
  LAUNCH_CHECK();
  return GPDB_OK;
}

template <bool BATCH>
static int launch_images(gpdb_ctx *ctx, const CloudSet &s, const gpdb_pose *d_cand, int nc, uint8_t *d_p16) {
  const DevParams &hp = ctx->hp;
  const int K = s.maxk;  // a batch is sized for its largest camera count
  const DevCloud &cl = s.view;
  const CloudTable tab = s.table();
  const int S = hp.S, RS = (S + 3) & ~3;
  const size_t plane_bytes = ((size_t)hp.C * S * RS + 15) / 16 * 16;
  const size_t tiles = (size_t)3 * 8 * S * S;
  const size_t bm = (size_t)K * (2 * (size_t)hp.bm_dim * hp.bm_dim) * 4;
  // shadow phase: the bitmaps alias the box list and the compacted voxel list follows them: room for >= 4 k voxels
  const size_t list_bytes = (std::max((size_t)BOX_CAP * 36, hp.C == 15 ? bm + 4096 * 4 : (size_t)0) + 15) / 16 * 16;
  const size_t smem = plane_bytes + tiles + list_bytes;
  // dynamic + static shared memory may not pass the device's opt-in maximum per block (232 448 B on H100)
  const size_t smem_max = (size_t)ctx->smem_optin - sizeof(ImgSmem);
  if (smem > smem_max) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "image geometry needs %zu B of shared memory per CTA (max %zu)", smem, smem_max);
    return GPDB_ERR_INVALID;
  }
  const char *force = getenv("GPD_B200_IMAGES_KERNEL");
  const bool fast = S == 60 && (hp.C != 15 || (K <= 2 && bm + 2048 <= (size_t)BOX_CAP2 * 36)) && !(force && force[0] == '1');
  const int *d_work = nullptr, *d_work_n = nullptr;
  if (fast) {
    int *ovf, *ovf_count;  // not SCR_OVF: the hand search of the next chunk may be writing it
    if (!gpdb_carve(ctx, SCR_IMG_OVF, [&](Carve &c) { ovf = c.take<int>(nc); ovf_count = c.take<int>(1); }))
      return GPDB_ERR_CUDA;
    CUDA_TRY(cudaMemsetAsync(ovf_count, 0, sizeof(int), ctx->stream));
    const size_t smem2 = IMG2_DYN_SMEM;
    CUDA_TRY(cudaFuncSetAttribute(k_images2<BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    k_images2<BATCH><<<std::min(nc, ctx->sm_count * 64), NT_IMG, smem2, ctx->stream>>>(ctx->dp, cl, tab, d_cand, nc, d_p16, ctx->d_qtab, ovf,
                                                                               ovf_count, ctx->d_prof);
    LAUNCH_CHECK();
    d_work = ovf;
    d_work_n = ovf_count;
  }
  // general tier (2 048-point box list in shared memory): everything, or the overflow list of the fast path; its own
  // overflow goes to a second list ...
  int *ovf2, *ovf2_count;
  if (!gpdb_carve(ctx, SCR_IMG_OVF2, [&](Carve &c) { ovf2 = c.take<int>(nc); ovf2_count = c.take<int>(1); }))
    return GPDB_ERR_CUDA;
  const int gl_cap = 32768;
  const size_t gl_slice = (size_t)gl_cap * 36 + (size_t)16 * S * S;
  unsigned char *gl = (unsigned char *)gpdb_scratch(ctx, SCR_IMG_GL, gl_slice * (size_t)ctx->sm_count);
  if (!gl) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemsetAsync(ovf2_count, 0, sizeof(int), ctx->stream));
  const int grid = fast ? ctx->sm_count : std::min(nc, ctx->sm_count * 64);
  const int err = S == 60 ? launch_general<60, BATCH>(ctx, s, d_cand, nc, d_p16, smem, plane_bytes, list_bytes, grid, d_work,
                                                      d_work_n, gl, gl_cap, ovf2, ovf2_count)
                          : launch_general<0, BATCH>(ctx, s, d_cand, nc, d_p16, smem, plane_bytes, list_bytes, grid, d_work,
                                                     d_work_n, gl, gl_cap, ovf2, ovf2_count);
  if (err != GPDB_OK) return err;
  return path_add(ctx, PATH_IMG_GL, ovf2_count, 0, nullptr);
}

int geo_images(gpdb_ctx *ctx, const CloudSet &s, const gpdb_pose *d_cand, int nc, uint8_t *d_p16) {
  if (nc <= 0) return GPDB_OK;
  return s.n > 1 ? launch_images<true>(ctx, s, d_cand, nc, d_p16) : launch_images<false>(ctx, s, d_cand, nc, d_p16);
}

int geo_p16_to_hwc(gpdb_ctx *ctx, const uint8_t *d_p16, int n, uint8_t *d_hwc) {
  if (n <= 0) return GPDB_OK;
  const size_t npix = (size_t)n * ctx->hp.S * ctx->hp.S, nb = npix * ctx->hp.C;
  k_p16_to_hwc<<<(unsigned)((nb + 255) / 256), 256, 0, ctx->stream>>>(d_p16, npix, ctx->hp.C, d_hwc);
  LAUNCH_CHECK();
  return GPDB_OK;
}
int geo_hwc_to_p16(gpdb_ctx *ctx, const uint8_t *d_hwc, int n, uint8_t *d_p16) {
  if (n <= 0) return GPDB_OK;
  const size_t npix = (size_t)n * ctx->hp.S * ctx->hp.S;
  k_hwc_to_p16<<<(unsigned)((npix + 255) / 256), 256, 0, ctx->stream>>>(d_hwc, npix, ctx->hp.C, d_p16);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int geo_label(gpdb_ctx *ctx, const CloudSet &s, gpdb_pose *d_hands, int n, int *d_labels) {
  if (n <= 0) return GPDB_OK;
  const unsigned grid = (unsigned)(((size_t)n * 32 + LABEL_NT - 1) / LABEL_NT);
  if (s.n > 1)
    k_label<true><<<grid, LABEL_NT, 0, ctx->stream>>>(ctx->dp, s.view, s.table(), d_hands, n, d_labels, ctx->d_prof);
  else
    k_label<false><<<grid, LABEL_NT, 0, ctx->stream>>>(ctx->dp, s.view, s.table(), d_hands, n, d_labels, ctx->d_prof);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int geo_clusters(gpdb_ctx *ctx, const gpdb_pose *d_hands, int n, const int *d_goff, int G, int min_inliers, gpdb_pose *d_dense,
                 uint8_t *d_keep, int *d_gcount) {
  CUDA_TRY(cudaMemsetAsync(d_gcount, 0, sizeof(int) * (size_t)G, ctx->stream));
  if (n <= 0) return GPDB_OK;
  const double cos_thresh = std::cos(12.0 * M_PI / 180.0);  // AXIS_ALIGN_ANGLE_THRESH (clustering.cpp:9)
  k_clusters<<<(n * 32 + 255) / 256, 256, 0, ctx->stream>>>(d_hands, n, d_goff, G, min_inliers, cos_thresh, d_dense, d_keep,
                                                            d_gcount);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int geo_select(gpdb_ctx *ctx, const gpdb_pose *d_cand, int n, int k, gpdb_pose *d_out) {
  if (n <= 0 || k <= 0) return GPDB_OK;
  unsigned *keys, *keys2;
  int *vals, *vals2;
  if (!gpdb_carve(ctx, SCR_KEYS, [&](Carve &c) {
        keys = c.take<unsigned>(n); keys2 = c.take<unsigned>(n); vals = c.take<int>(n); vals2 = c.take<int>(n);
      }))
    return GPDB_ERR_CUDA;
  k_select_keys<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_cand, n, keys, vals);
  LAUNCH_CHECK();
  size_t tmp_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys2, vals, vals2, n, 0, 32, ctx->stream);
  void *tmp = gpdb_scratch(ctx, SCR_CUB, tmp_bytes);
  if (!tmp) return GPDB_ERR_CUDA;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys2, vals, vals2, n, 0, 32, ctx->stream));
  ctx->launches += 4;
  k_gather_poses<<<(k * 32 + 255) / 256, 256, 0, ctx->stream>>>(d_cand, vals2, k, d_out);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int geo_scatter_scores(gpdb_ctx *ctx, const gpdb_pose *d_cand, const float *d_scores, int nc, int slot0, int P,
                       float *d_pose_scores, gpdb_pose *d_cand_out) {
  if (nc <= 0) return GPDB_OK;
  k_scatter_scores<<<(nc + 255) / 256, 256, 0, ctx->stream>>>(d_cand, d_scores, nc, slot0, P, d_pose_scores, d_cand_out);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// The grids of store s (s.n clouds whose descriptors hold off / N): per-cloud bounds with many CTAs per cloud, dims and
// cell bases on the device, one sort over (cloud, cell) for all clouds.
int geo_build_grid_batch(gpdb_ctx *ctx, CloudSet &s) {
  const int B = s.n, N = s.points();
  long long *ncell, *base;  // cells per cloud and their scan
  int *d_off, *bounds;
  if (!gpdb_carve(ctx, SCR_WORK_B, [&](Carve &c) {
        ncell = c.take<long long>((size_t)B + 1); base = c.take<long long>((size_t)B + 1);
        d_off = c.take<int>((size_t)B + 1); bounds = c.take<int>(6 * (size_t)B);
      }))
    return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(d_off, s.off, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  int largest = 0;
  for (int b = 0; b < B; b++) largest = std::max(largest, s.off[b + 1] - s.off[b]);
  int rc = pre_bounds_batch(ctx, s.xyz, d_off, B, largest, bounds);
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaMemsetAsync(ncell + B, 0, sizeof(long long), ctx->stream));
  k_batch_desc<<<(B + 255) / 256, 256, 0, ctx->stream>>>(bounds, s.desc, B, ncell);
  LAUNCH_CHECK();
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, ncell, base, B + 1, ctx->stream);
  void *tmp = gpdb_scratch(ctx, SCR_CUB, tmp_bytes);
  if (!tmp) return GPDB_ERR_CUDA;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, ncell, base, B + 1, ctx->stream));
  ctx->launches += 1;
  long long total = 0;
  CUDA_TRY(cudaMemcpyAsync(&total, base + B, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (total + 1 > (long long)INT_MAX) {
    gpdb_set_error(ctx, GPDB_ERR_CAPACITY, "gpdb_set_clouds: the grids of the batch need %lld cells (max %d)", total, INT_MAX - 1);
    return GPDB_ERR_CAPACITY;
  }
  k_batch_base<<<(B + 255) / 256, 256, 0, ctx->stream>>>(s.desc, base, B);
  LAUNCH_CHECK();
  const size_t ncells = (size_t)total;
  if (ncells + 1 > s.cell_cap) {
    cudaStreamSynchronize(ctx->stream);
    cudaFree(s.cell_start);
    s.cell_start = nullptr;
    s.cell_cap = 0;
    CUDA_TRY(cudaMalloc(&s.cell_start, sizeof(int) * (ncells + 1 + ncells / 4)));
    s.cell_cap = ncells + 1 + ncells / 4;
  }
  CUDA_TRY(cudaMemsetAsync(s.cell_start, 0, sizeof(int) * (ncells + 1), ctx->stream));
  int *cid, *idx, *cid2, *idx2;
  if (!gpdb_carve(ctx, SCR_P16, [&](Carve &c) {
        cid = c.take<int>(N); idx = c.take<int>(N); cid2 = c.take<int>(N); idx2 = c.take<int>(N);
      }))
    return GPDB_ERR_CUDA;
  const int tb = 256, gb = (N + tb - 1) / tb;
  size_t tmp2 = 0;
  tmp_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, cid, cid2, idx, idx2, N, 0, 32, ctx->stream);
  cub::DeviceScan::InclusiveSum(nullptr, tmp2, s.cell_start, s.cell_start, (int)(ncells + 1), ctx->stream);
  tmp = gpdb_scratch(ctx, SCR_CUB, std::max(tmp_bytes, tmp2));
  if (!tmp) return GPDB_ERR_CUDA;
  if (N > 0) {  // a preprocessed batch may hold no point at all (every view filtered out)
    k_batch_cell_ids<<<gb, tb, 0, ctx->stream>>>(s.xyz, s.desc, B, N, cid, idx, s.cell_start);
    LAUNCH_CHECK();
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, cid, cid2, idx, idx2, N, 0, 32, ctx->stream));
    ctx->launches += 4;
    k_batch_fill_sorted<<<gb, tb, 0, ctx->stream>>>(s.xyz, idx2, s.desc, B, N, s.pts4);
    LAUNCH_CHECK();
  }
  CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp, tmp2, s.cell_start, s.cell_start, (int)(ncells + 1), ctx->stream));
  ctx->launches += 2;
  s.view.cell_start = s.cell_start;
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return GPDB_OK;
}

// gpdb_detect_select per cloud of the running batch: the n classified candidates (sample-slot order) are sorted by
// (cloud, descending score) with one stable device-wide radix sort, so ties keep candidate order and one large cloud is
// sorted by the whole device; the first min(k, count) of every cloud are gathered to d_out in cloud order.
// sel_off[B+1] (host) receives the output offsets; returns the total.
int geo_select_batch(gpdb_ctx *ctx, CloudSet &s, const gpdb_pose *d_cand, int n, int k, gpdb_pose **d_out) {
  const int B = s.n;
  int *sel_off = s.sel;
  *d_out = nullptr;
  unsigned long long *keys, *keys2;
  int *vals, *vals2, *order, *cand_off, *d_sel_off;
  if (!gpdb_carve(ctx, SCR_KEYS, [&](Carve &c) {
        keys = c.take<unsigned long long>(n); keys2 = c.take<unsigned long long>(n); vals = c.take<int>(n);
        vals2 = c.take<int>(n); order = c.take<int>(n); cand_off = c.take<int>((size_t)B + 1);
        d_sel_off = c.take<int>((size_t)B + 1);
      }))
    return GPDB_ERR_CUDA;
  k_batch_cand_off<<<(B + 1 + 255) / 256, 256, 0, ctx->stream>>>(d_cand, n, s.soff, B, cand_off);
  LAUNCH_CHECK();
  std::vector<int> coff((size_t)B + 1);
  CUDA_TRY(cudaMemcpyAsync(coff.data(), cand_off, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, ctx->stream));
  if (n > 0) {
    k_batch_select_keys<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_cand, n, s.soff, B, keys, vals);
    LAUNCH_CHECK();
    int cloud_bits = 0;
    while ((1ll << cloud_bits) < B) cloud_bits++;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys2, vals, vals2, n, 0, 32 + cloud_bits, ctx->stream);
    void *tmp = gpdb_scratch(ctx, SCR_CUB, tmp_bytes);
    if (!tmp) return GPDB_ERR_CUDA;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys2, vals, vals2, n, 0, 32 + cloud_bits, ctx->stream));
    ctx->launches += 4;
  }
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  sel_off[0] = 0;
  for (int b = 0; b < B; b++) sel_off[b + 1] = sel_off[b] + std::min(k, coff[b + 1] - coff[b]);
  const int total = sel_off[B];
  if (total == 0) return 0;
  CUDA_TRY(cudaMemcpyAsync(d_sel_off, sel_off, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  k_batch_sel_order<<<(total + 255) / 256, 256, 0, ctx->stream>>>(vals2, cand_off, d_sel_off, B, total, order);
  LAUNCH_CHECK();
  gpdb_pose *out = (gpdb_pose *)gpdb_scratch(ctx, SCR_POSES, sizeof(gpdb_pose) * (size_t)total);
  if (!out) return GPDB_ERR_CUDA;
  k_gather_poses<<<(total * 32 + 255) / 256, 256, 0, ctx->stream>>>(d_cand, order, total, out);
  LAUNCH_CHECK();
  *d_out = out;
  return total;
}

int geo_batch_cand_off(gpdb_ctx *ctx, const CloudSet &s, const gpdb_pose *d_cand, int n, int *cand_off) {
  const int B = s.n;
  int *d_off = (int *)gpdb_scratch(ctx, SCR_KEYS, sizeof(int) * ((size_t)B + 1));
  if (!d_off) return GPDB_ERR_CUDA;
  k_batch_cand_off<<<(B + 1 + 255) / 256, 256, 0, ctx->stream>>>(d_cand, n, s.soff, B, d_off);
  LAUNCH_CHECK();
  CUDA_TRY(cudaMemcpyAsync(cand_off, d_off, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return GPDB_OK;
}
