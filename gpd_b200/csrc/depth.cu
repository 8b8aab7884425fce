// depth.cu — the depth-image front of preprocessing and Cloud::subsample on the device (include/gpd_b200_depth.h).
//
//   gpdb_preprocess_depth: k_depth_flag (back-projection + removeNans + filterWorkspace, one thread per pixel) + scan +
//     k_depth_compact, then the voxelise / emit back of pre_filter_voxelize_batch (preprocess.cu). The raw cloud of a view
//     is never materialised: per pixel only the filter flag, its scan and a one-byte camera mask exist; the coordinates
//     are written for the filtered points only.
//   gpdb_subsample_clouds: k_sub_flag (eligible points, the mask read through src) + scan + k_sub_compact (keys), a
//     segmented radix sort of (key, eligible position) per cloud, k_sub_pick (each cloud's first k) and a scan +
//     k_sub_gather of the picks, which restores ascending j.
// Compiled with -fmad=false: every float32 / float64 operation of the back-projection is rounded on its own.
#include <cfloat>
#include <climits>
#include <cub/cub.cuh>
#include <vector>

#include "../../include/gpd_b200_depth.h"
#include "common.cuh"

namespace {

// one camera of a call as the kernels read it (filled by pre_depth_batch)
struct DepthCam {
  double R[9], t[3];
  double min_depth, max_depth;
  float fx, fy, cx, cy, scale;
  int width;
  uint8_t bit;  // 1 << (camera index in its view): the camera mask of its pixels
};

// pixel i of the call: its camera c (csr_owner over the pixel offsets), its world point and validity. Returns whether the
// pixel has a valid depth; xyz is the back-projected point (gpd_b200_depth.h 2)
__device__ __forceinline__ bool depth_point(const void *depth, int format, const DepthCam &K, int p, float xyz[3], long long i) {
  float z;
  bool ret;
  if (format == GPDB_DEPTH_U16) {
    const uint16_t raw = static_cast<const uint16_t *>(depth)[i];
    ret = raw != 0;
    z = (float)raw * K.scale;
  } else {
    const float raw = static_cast<const float *>(depth)[i];
    ret = isfinite(raw) && raw > 0.0f;
    z = raw * K.scale;
  }
  const bool valid = ret && (double)z >= K.min_depth && (double)z <= K.max_depth;
  const int u = p % K.width, v = p / K.width;
  const float xc = (((float)u - K.cx) * z) / K.fx, yc = (((float)v - K.cy) * z) / K.fy, zc = z;
  for (int r = 0; r < 3; r++)
    xyz[r] = (float)(((K.R[3 * r] * (double)xc + K.R[3 * r + 1] * (double)yc) + K.R[3 * r + 2] * (double)zc) + K.t[r]);
  return valid;
}

// removeNans + filterWorkspace of the back-projected pixel: k_pre_flag's test on its float32 point
__device__ __forceinline__ bool in_workspace(const float *q, const double *ws) {
  return isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]) && (double)q[0] > ws[0] && (double)q[0] < ws[1] &&
         (double)q[1] > ws[2] && (double)q[1] < ws[3] && (double)q[2] > ws[4] && (double)q[2] < ws[5];
}

__global__ void __launch_bounds__(256) k_depth_flag(const void *depth, int format, int M, const int *cam_off, int C,
                                                    const DepthCam *cams, const double *ws, int *flag, uint8_t *cam_raw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int c = csr_owner(cam_off, C, i);
  const DepthCam &K = cams[c];
  float q[3];
  const bool valid = depth_point(depth, format, K, i - cam_off[c], q, i);
  flag[i] = valid && in_workspace(q, ws) ? 1 : 0;
  cam_raw[i] = K.bit;
}

// the filtered pixels again: keep[k] = pixel index in the call, xyz1[3k..] its point
__global__ void __launch_bounds__(256) k_depth_compact(const void *depth, int format, int M, const int *cam_off, int C,
                                                       const DepthCam *cams, const int *flag, const int *pos, int *keep,
                                                       float *xyz1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M || !flag[i]) return;
  const int c = csr_owner(cam_off, C, i);
  float q[3];
  depth_point(depth, format, cams[c], i - cam_off[c], q, i);
  const int k = pos[i];
  keep[k] = i;
  xyz1[3 * (size_t)k] = q[0];
  xyz1[3 * (size_t)k + 1] = q[1];
  xyz1[3 * (size_t)k + 2] = q[2];
}

// ---- Cloud::subsample ----------------------------------------------------------------------------------------------
// flag[g] = point g of the store is eligible: no mask, or the mask byte of its source raw point (raw offsets roff)
__global__ void k_sub_flag(int N, const int *off, int B, const int *src, const int *roff, const uint8_t *mask, int *flag) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  int e = 1;
  if (mask) {
    const int b = csr_owner(off, B, g);
    e = mask[(size_t)roff[b] + src[g]] != 0;
  }
  flag[g] = e;
}
// flag[g] = the mask byte of point g itself (a mask over the installed points)
__global__ void k_sub_flag_points(int N, const uint8_t *mask, int *flag) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < N) flag[g] = mask[g] != 0;
}
// eligible point g -> position e = pos[g]: its key under seed + b, its cloud-local index j, and e itself (the sort's value)
__global__ void k_sub_compact(int N, const int *off, int B, const int *flag, const int *pos, unsigned long long seed,
                              unsigned long long *keys, int *vals, int *ev) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N || !flag[g]) return;
  const int b = csr_owner(off, B, g);
  const int j = g - off[b], e = pos[g];
  keys[e] = gpdb_subsample_key(seed + (unsigned long long)b, (uint32_t)j);
  vals[e] = j;
  if (ev) ev[e] = e;
}
// sorted entry s of cloud b (eoff): pick[e] = 1 for the eligible position e of each of the cloud's first k_b = soff[b+1] -
// soff[b] entries (pick zeroed by the caller)
__global__ void k_sub_pick(int E, const int *eoff, const int *soff, int B, const int *ev_sorted, int *pick) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= E) return;
  const int b = csr_owner(eoff, B, s);
  if (s - eoff[b] < soff[b + 1] - soff[b]) pick[ev_sorted[s]] = 1;
}
// the picked positions in ascending order (within a cloud: ascending j) -> out
__global__ void k_sub_gather(int E, const int *pick, const int *ppos, const int *vals, int *out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < E && pick[e]) out[ppos[e]] = vals[e];
}

}  // namespace

// Back-projection + filter of the pixels of B views (camera descriptions cams, view b has n_cameras[b] of them; raw
// offsets roff = cumulative pixels per view), then the voxelise / emit back of preprocess.cu
int pre_depth_batch(gpdb_ctx *ctx, CloudSet &s, const void *d_depth, int format, const gpdb_depth_camera *cams,
                    const int *n_cameras, int B, const int *roff, const gpdb_preprocess_params &pp, int *poff,
                    cudaEvent_t ev_filter_done) {
  const int tb = 256;
  const int M = roff[B];
  int C = 0;
  for (int b = 0; b < B; b++) C += n_cameras[b];
  // the camera table: the cameras, then their pixel offsets [C+1]; staged on the host, copied behind the call's header
  DepthCam *tab;
  int *cam_off;
  const auto table = [&](Carve &c) { tab = c.take<DepthCam>(C); cam_off = c.take<int>((size_t)C + 1); };
  std::vector<unsigned char> h_tab(carve_bytes(table));
  carve_at(h_tab.data(), table);
  cam_off[0] = 0;
  for (int b = 0, c = 0; b < B; b++)
    for (int k = 0; k < n_cameras[b]; k++, c++) {
      const gpdb_depth_camera &D = cams[c];
      DepthCam &K = tab[c];
      for (int r = 0; r < 3; r++) {
        for (int q = 0; q < 3; q++) K.R[3 * r + q] = D.pose[4 * r + q];
        K.t[r] = D.pose[4 * r + 3];
      }
      K.min_depth = D.min_depth;
      K.max_depth = D.max_depth;
      K.fx = (float)D.fx, K.fy = (float)D.fy, K.cx = (float)D.cx, K.cy = (float)D.cy, K.scale = (float)D.depth_scale;
      K.width = D.width;
      K.bit = (uint8_t)(1u << k);
      cam_off[c + 1] = cam_off[c] + D.width * D.height;
    }
  PreBatch h;
  int rc = pre_batch_header(ctx, B, roff, pp, h_tab.size(), h);
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaMemcpyAsync(h.extra, h_tab.data(), h_tab.size(), cudaMemcpyHostToDevice, ctx->stream));
  carve_at(h.extra, table);  // tab and cam_off now address the device copy
  const DepthCam *d_cams = tab;
  const int *d_cam_off = cam_off;
  // per pixel: filter flag + its scan, the camera mask
  int *flag, *pos;
  if (!gpdb_carve(ctx, SCR_KEYS, [&](Carve &c) {
        flag = c.take<int>((size_t)M + 1); pos = c.take<int>((size_t)M + 1);
      }))
    return GPDB_ERR_CUDA;
  uint8_t *cam_raw = (uint8_t *)gpdb_scratch(ctx, SCR_SIDX, (size_t)M + 16);
  if (!cam_raw) return GPDB_ERR_CUDA;
  k_depth_flag<<<(M + tb - 1) / tb, tb, 0, ctx->stream>>>(d_depth, format, M, d_cam_off, C, d_cams, h.ws, flag, cam_raw);
  LAUNCH_CHECK();
  if ((rc = scan_flags(ctx, flag, pos, M)) != GPDB_OK) return rc;  // pos[M] = number of filtered points
  if ((rc = pre_filter_offsets(ctx, pos, h, B)) != GPDB_OK) return rc;
  std::vector<int> foff((size_t)B + 1);
  CUDA_TRY(cudaMemcpyAsync(foff.data(), h.foff, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  // the filtered points alone: keep + xyz1, sized by the count just read back
  const int M1 = foff[B];
  int *keep;
  float *xyz1;
  if (!gpdb_carve(ctx, SCR_WORK_B, [&](Carve &c) { keep = c.take<int>(M1); xyz1 = c.take<float>(3 * (size_t)M1); }))
    return GPDB_ERR_CUDA;
  if (M1 > 0) {
    k_depth_compact<<<(M + tb - 1) / tb, tb, 0, ctx->stream>>>(d_depth, format, M, d_cam_off, C, d_cams, flag, pos, keep,
                                                               xyz1);
    LAUNCH_CHECK();
  }
  cudaEventRecord(ev_filter_done, ctx->stream);
  return pre_voxelize_back(ctx, s, h, foff.data(), keep, xyz1, cam_raw, nullptr, B, pp, poff);
}

int sub_draw_batch(gpdb_ctx *ctx, const CloudSet &s, int num_samples, unsigned long long seed, const uint8_t *d_mask,
                   bool per_point, int *d_out, int *soff) {
  const int tb = 256;
  const int B = s.n, N = s.points();
  // device: point offsets, raw offsets, eligible offsets, output offsets
  int *d_off, *d_roff, *d_eoff, *d_soff;
  if (!gpdb_carve(ctx, SCR_WORK_A, [&](Carve &c) {
        d_off = c.take<int>((size_t)B + 1); d_roff = c.take<int>((size_t)B + 1); d_eoff = c.take<int>((size_t)B + 1);
        d_soff = c.take<int>((size_t)B + 1);
      }))
    return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(d_off, s.off, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  if (d_mask && !per_point)
    CUDA_TRY(cudaMemcpyAsync(d_roff, s.raw_off, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  std::vector<int> eoff((size_t)B + 1, 0);
  int *flag = nullptr, *pos = nullptr;
  if (N > 0) {
    if (!gpdb_carve(ctx, SCR_KEYS, [&](Carve &c) {
          flag = c.take<int>((size_t)N + 1); pos = c.take<int>((size_t)N + 1);
        }))
      return GPDB_ERR_CUDA;
    if (d_mask && per_point) k_sub_flag_points<<<(N + tb - 1) / tb, tb, 0, ctx->stream>>>(N, d_mask, flag);
    else k_sub_flag<<<(N + tb - 1) / tb, tb, 0, ctx->stream>>>(N, d_off, B, s.src, d_roff, d_mask, flag);
    LAUNCH_CHECK();
    int rc = scan_flags(ctx, flag, pos, N);
    if (rc != GPDB_OK) return rc;
    // eligible offsets eoff[b] = pos[off[b]] (the filtered-offsets kernel of preprocessing, on the point offsets)
    PreBatch h{};
    h.roff = d_off;
    h.foff = d_eoff;
    if ((rc = pre_filter_offsets(ctx, pos, h, B)) != GPDB_OK) return rc;
    CUDA_TRY(cudaMemcpyAsync(eoff.data(), d_eoff, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  const int E = eoff[B];
  bool all = true;  // every cloud takes all its eligible points: the compacted indices are the answer
  soff[0] = 0;
  for (int b = 0; b < B; b++) {
    const int cnt = eoff[b + 1] - eoff[b];
    const int k = num_samples == 0 ? cnt : std::min(num_samples, cnt);
    all = all && k == cnt;
    soff[b + 1] = soff[b] + k;
  }
  const int n = soff[B];
  if (E == 0) return 0;
  // keys, sorted keys; j, e, sorted e; pick flags and their scan
  unsigned long long *keys, *keys2;
  int *vals, *ev, *ev2, *pick, *ppos;
  if (!gpdb_carve(ctx, SCR_WORK_C, [&](Carve &c) {
        keys = c.take<unsigned long long>(E); keys2 = c.take<unsigned long long>(E); vals = c.take<int>(E);
        ev = c.take<int>(E); ev2 = c.take<int>(E); pick = c.take<int>((size_t)E + 1); ppos = c.take<int>((size_t)E + 1);
      }))
    return GPDB_ERR_CUDA;
  k_sub_compact<<<(N + tb - 1) / tb, tb, 0, ctx->stream>>>(N, d_off, B, flag, pos, seed, keys, all ? d_out : vals,
                                                           all ? nullptr : ev);
  LAUNCH_CHECK();
  if (all) {
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return n;
  }
  CUDA_TRY(cudaMemcpyAsync(d_soff, soff, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  // (key, e) order per cloud: the radix sort is LSD (stable) and e ascends with j inside a cloud, so equal keys stay in
  // ascending j. The first k_b entries of each cloud are picked, and the picks compacted in e order: ascending j again.
  size_t t1 = 0, t2 = 0;
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, t1, keys, keys2, ev, ev2, E, B, d_eoff, d_eoff + 1, 0, 64, ctx->stream);
  cub::DeviceScan::ExclusiveSum(nullptr, t2, pick, ppos, E + 1, ctx->stream);
  void *tmp = gpdb_scratch(ctx, SCR_CUB, std::max(t1, t2));
  if (!tmp) return GPDB_ERR_CUDA;
  CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairs(tmp, t1, keys, keys2, ev, ev2, E, B, d_eoff, d_eoff + 1, 0, 64,
                                                    ctx->stream));
  ctx->launches++;
  CUDA_TRY(cudaMemsetAsync(pick, 0, sizeof(int) * ((size_t)E + 1), ctx->stream));
  k_sub_pick<<<(E + tb - 1) / tb, tb, 0, ctx->stream>>>(E, d_eoff, d_soff, B, ev2, pick);
  LAUNCH_CHECK();
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, t2, pick, ppos, E + 1, ctx->stream));
  ctx->launches += 2;
  k_sub_gather<<<(E + tb - 1) / tb, tb, 0, ctx->stream>>>(E, pick, ppos, vals, d_out);
  LAUNCH_CHECK();
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return n;
}
