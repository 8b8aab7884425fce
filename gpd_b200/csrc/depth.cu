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
// The entry points gpdb_preprocess_depth[_organized][_device] and gpdb_subsample_clouds[_points][_device], with their
// argument checks, follow the kernels; the depth-format and camera checks are render.cu's too.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
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

// Cloud::subsample of every cloud of store s: cloud b's draw to d_out at soff[b] (host, B + 1); returns the total or an
// error. d_mask: one byte per installed point (per_point), or per raw point indexed by the store's raw_off (has_src)
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

}  // namespace

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

int check_depth_format(gpdb_ctx *ctx, const char *name, int32_t format) {
  if (format == GPDB_DEPTH_U16 || format == GPDB_DEPTH_F32) return GPDB_OK;
  gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: unknown depth format %d (GPDB_DEPTH_U16 = 0, GPDB_DEPTH_F32 = 1)", name, format);
  return GPDB_ERR_INVALID;
}

int check_depth_cameras(gpdb_ctx *ctx, const char *name, int32_t B, const int32_t *n_cameras,
                        const gpdb_depth_camera *cams, std::vector<int> &roff) {
  roff.assign((size_t)B + 1, 0);
  long long total = 0;
  for (int b = 0, c = 0; b < B; b++) {
    if (n_cameras[b] <= 0 || n_cameras[b] > GPDB_MAX_CAMERAS) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: view %d has %d cameras (1 <= cameras <= %d)", name, b, n_cameras[b],
                     GPDB_MAX_CAMERAS);
      return GPDB_ERR_INVALID;
    }
    for (int k = 0; k < n_cameras[b]; k++, c++) {
      const gpdb_depth_camera &D = cams[c];
      const char *bad = nullptr;
      bool finite = std::isfinite(D.fx) && std::isfinite(D.fy) && std::isfinite(D.cx) && std::isfinite(D.cy);
      for (int e = 0; e < 12; e++) finite = finite && std::isfinite(D.pose[e]);
      if (D.width < 1 || D.height < 1) bad = "width and height must be at least 1";
      else if (!finite) bad = "non-finite intrinsics or pose";
      else if (!(D.fx > 0.0) || !(D.fy > 0.0)) bad = "fx and fy must be positive";
      else if (!(D.depth_scale > 0.0) || !std::isfinite(D.depth_scale)) bad = "depth_scale must be finite and positive";
      else if (!(D.min_depth >= 0.0)) bad = "min_depth must be >= 0";
      else if (!(D.max_depth > D.min_depth)) bad = "max_depth must exceed min_depth";
      if (bad) {
        gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: view %d camera %d (camera %d of the call): %s", name, b, k, c, bad);
        return GPDB_ERR_INVALID;
      }
      total += (long long)D.width * D.height;
      if (total >= (1ll << 31)) {
        gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: view %d camera %d: the call holds 2^31 or more pixels", name, b, k);
        return GPDB_ERR_INVALID;
      }
    }
    roff[b + 1] = (int)total;
  }
  return GPDB_OK;
}

// the argument checks of gpdb_preprocess_depth[_device]; roff[B+1] receives the raw offsets (cumulative pixels per view)
static int check_depth_args(gpdb_ctx *ctx, const char *name, int32_t B, const int32_t *n_cameras, const gpdb_depth_camera *cams,
                            int32_t format, const void *depth, const gpdb_preprocess_params *pp, const int32_t *poff,
                            std::vector<int> &roff) {
  if (B <= 0 || !n_cameras || !cams || !depth || !pp || !poff) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need n_views > 0, n_cameras, cameras, depth, params, processed_offsets_out",
                   name);
    return GPDB_ERR_INVALID;
  }
  if (check_depth_format(ctx, name, format) != GPDB_OK) return GPDB_ERR_INVALID;
  if (!pp->estimate_normals) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: estimate_normals must be 1 (depth images carry no normals)", name);
    return GPDB_ERR_INVALID;
  }
  const int rc = gpdb_check_preprocess_params(ctx, name, pp, nullptr);
  if (rc != GPDB_OK) return rc;
  return check_depth_cameras(ctx, name, B, n_cameras, cams, roff);
}

// gpdb_preprocess_depth[_device] after the argument checks: d_depth in device memory (the host twin has uploaded it)
// organized: the normals of gpd_b200_organized.h rule 7 replace the radius estimates (n_fallback[B], host, may be null)
static int preprocess_depth(gpdb_ctx *ctx, const char *name, CloudSet &s, int32_t B, const int32_t *n_cameras,
                            const gpdb_depth_camera *cams, int32_t format, const void *depth, bool device,
                            const gpdb_preprocess_params *pp, const std::vector<int> &roff, int32_t *poff, bool organized,
                            int32_t *n_fallback) {
  cudaEvent_t *ev = ctx->ev;
  const int M = roff[B];
  CUDA_TRY(cudaSetDevice(ctx->device));
  cudaEventRecord(ev[0], ctx->stream);
  const void *d_depth = depth;
  if (!device) {
    const size_t bytes = (size_t)M * (format == GPDB_DEPTH_U16 ? sizeof(uint16_t) : sizeof(float));
    void *up = gpdb_scratch(ctx, SCR_UPLOAD, bytes);
    if (!up) return GPDB_ERR_CUDA;
    CUDA_TRY(cudaMemcpyAsync(up, depth, bytes, cudaMemcpyHostToDevice, ctx->stream));
    d_depth = up;
  }
  // the camera fields of the descriptors: view point k = t of camera k; one-hot camera sources, as a cam_source matrix
  std::vector<CloudDesc> desc((size_t)B);
  for (int b = 0, c = 0; b < B; b++) {
    CloudDesc &D = desc[b];
    memset(&D, 0, sizeof(D));
    D.K = n_cameras[b];
    for (int k = 0; k < D.K; k++, c++)
      for (int r = 0; r < 3; r++) D.vp[k][r] = cams[c].pose[4 * r + 3];
  }
  cudaEventRecord(ev[1], ctx->stream);
  int rc = pre_depth_batch(ctx, s, d_depth, format, cams, n_cameras, B, roff.data(), *pp, poff, ev[2]);
  if (rc != GPDB_OK) return rc;
  if (!organized) return gpdb_preprocess_install(ctx, s, desc.data(), B, roff.data(), pp, poff);
  // the host twin's images stay in SCR_UPLOAD until here: the install does not use that slot
  return gpdb_preprocess_install(ctx, s, desc.data(), B, roff.data(), pp, poff, [&]() {
    return org_depth_normals(ctx, name, s, d_depth, format, cams, n_cameras, B, n_fallback);
  });
}

static int depth_entry(gpdb_ctx *ctx, const char *name, int32_t n_views, const int32_t *n_cameras,
                       const gpdb_depth_camera *cameras, int32_t depth_format, const void *depth,
                       const gpdb_preprocess_params *pp, int32_t *processed_offsets_out, bool device,
                       bool organized = false, int32_t *n_fallback = nullptr) {
  if (!ctx) return GPDB_ERR_INVALID;
  gpdb_drop_batch(ctx);
  std::vector<int> roff;
  int rc = check_depth_args(ctx, name, n_views, n_cameras, cameras, depth_format, depth, pp, processed_offsets_out, roff);
  if (rc == GPDB_OK && device) rc = gpdb_check_device_ptrs(ctx, name, {{"d_depth", depth}});
  if (rc != GPDB_OK) return rc;
  return preprocess_depth(ctx, name, ctx->many, n_views, n_cameras, cameras, depth_format, depth, device, pp, roff,
                          processed_offsets_out, organized, n_fallback);
}

// gpdb_subsample_clouds[_device]: the state and argument checks, then the device draw (the host twin uploads the mask and
// copies the indices back)
static int subsample_entry(gpdb_ctx *ctx, const char *name, int32_t num_samples, uint64_t seed, const uint8_t *mask,
                           int32_t *idx_out, int32_t *offsets_out, bool device, bool per_point = false) {
  if (!ctx) return GPDB_ERR_INVALID;
  CloudSet &s = ctx->many;
  int rc = gpdb_need_batch(ctx, name, "gpdb_preprocess_depth / gpdb_preprocess_clouds");
  if (rc != GPDB_OK) return rc;
  if (num_samples < 0 || !offsets_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need num_samples >= 0 (got %d) and sample_offsets_out", name, num_samples);
    return GPDB_ERR_INVALID;
  }
  if (mask && !per_point && !s.has_src) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "%s: a mask needs the source indices of a preprocessing call (gpdb_preprocess_depth "
                   "/ gpdb_preprocess_clouds); the batch was installed by gpdb_set_clouds", name);
    return GPDB_ERR_STATE;
  }
  const int B = s.n;
  long long room = 0;
  for (int b = 0; b < B; b++) {
    const int nb = s.off[b + 1] - s.off[b];
    room += num_samples == 0 ? nb : std::min(num_samples, nb);
  }
  if (room > 0 && !idx_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null %s", name, device ? "d_sample_idx_out" : "sample_idx_out");
    return GPDB_ERR_INVALID;
  }
  if (device && (rc = gpdb_check_device_ptrs(ctx, name, {{"d_mask", mask}, {"d_sample_idx_out", idx_out}})) != GPDB_OK)
    return rc;
  CUDA_TRY(cudaSetDevice(ctx->device));
  const uint8_t *d_mask = mask;
  int *d_out = idx_out;
  if (!device) {
    if (mask) {
      const size_t M = per_point ? (size_t)s.points() : (size_t)s.raw_off[B];
      uint8_t *up = (uint8_t *)gpdb_scratch(ctx, SCR_UPLOAD, M);
      if (!up) return GPDB_ERR_CUDA;
      CUDA_TRY(cudaMemcpyAsync(up, mask, M, cudaMemcpyHostToDevice, ctx->stream));
      d_mask = up;
    }
    d_out = (int *)gpdb_scratch(ctx, SCR_SIDX, sizeof(int) * (size_t)room);
    if (!d_out) return GPDB_ERR_CUDA;
  }
  std::vector<int> soff((size_t)B + 1);
  const int n = sub_draw_batch(ctx, s, num_samples, seed, d_mask, per_point, d_out, soff.data());
  if (n < 0) return n;
  if (!device && n > 0) {
    CUDA_TRY(cudaMemcpyAsync(idx_out, d_out, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  memcpy(offsets_out, soff.data(), sizeof(int) * ((size_t)B + 1));
  return n;
}

extern "C" {

int gpdb_preprocess_depth(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras, const gpdb_depth_camera *cameras,
                          int32_t depth_format, const void *depth, const gpdb_preprocess_params *pp,
                          int32_t *processed_offsets_out) {
  return depth_entry(ctx, "gpdb_preprocess_depth", n_views, n_cameras, cameras, depth_format, depth, pp,
                     processed_offsets_out, false);
}

int gpdb_preprocess_depth_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras, const gpdb_depth_camera *cameras,
                                 int32_t depth_format, const void *d_depth, const gpdb_preprocess_params *pp,
                                 int32_t *processed_offsets_out) {
  return depth_entry(ctx, "gpdb_preprocess_depth_device", n_views, n_cameras, cameras, depth_format, d_depth, pp,
                     processed_offsets_out, true);
}

int gpdb_preprocess_depth_organized(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras,
                                    const gpdb_depth_camera *cameras, int32_t depth_format, const void *depth,
                                    const gpdb_preprocess_params *pp, int32_t *processed_offsets_out,
                                    int32_t *n_fallback_out) {
  return depth_entry(ctx, "gpdb_preprocess_depth_organized", n_views, n_cameras, cameras, depth_format, depth, pp,
                     processed_offsets_out, false, true, n_fallback_out);
}

int gpdb_preprocess_depth_organized_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras,
                                           const gpdb_depth_camera *cameras, int32_t depth_format, const void *d_depth,
                                           const gpdb_preprocess_params *pp, int32_t *processed_offsets_out,
                                           int32_t *n_fallback_out) {
  return depth_entry(ctx, "gpdb_preprocess_depth_organized_device", n_views, n_cameras, cameras, depth_format, d_depth, pp,
                     processed_offsets_out, true, true, n_fallback_out);
}

int gpdb_subsample_clouds(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *mask, int32_t *sample_idx_out,
                          int32_t *sample_offsets_out) {
  return subsample_entry(ctx, "gpdb_subsample_clouds", num_samples, seed, mask, sample_idx_out, sample_offsets_out, false);
}

int gpdb_subsample_clouds_device(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *d_mask,
                                 int32_t *d_sample_idx_out, int32_t *sample_offsets_out) {
  return subsample_entry(ctx, "gpdb_subsample_clouds_device", num_samples, seed, d_mask, d_sample_idx_out,
                         sample_offsets_out, true);
}

int gpdb_subsample_clouds_points(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *point_mask,
                                 int32_t *sample_idx_out, int32_t *sample_offsets_out) {
  return subsample_entry(ctx, "gpdb_subsample_clouds_points", num_samples, seed, point_mask, sample_idx_out,
                         sample_offsets_out, false, true);
}

int gpdb_subsample_clouds_points_device(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *d_point_mask,
                                        int32_t *d_sample_idx_out, int32_t *sample_offsets_out) {
  return subsample_entry(ctx, "gpdb_subsample_clouds_points_device", num_samples, seed, d_point_mask, d_sample_idx_out,
                         sample_offsets_out, true, true);
}

}  // extern "C"
