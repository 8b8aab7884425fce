// organized.cu — pcl::IntegralImageNormalEstimation (COVARIANCE_MATRIX) on the device (include/gpd_b200_organized.h):
// Cloud::calculateNormalsOrganized for organized clouds (gpdb_normals_organized[_device]).
//
//   k_org_change    the depth-change map (rule 2), one thread per pixel, written as the initial distance map
//   k_org_dist      the two chamfer passes (rule 3), one CTA per image, each pass a wavefront
//   k_org_integral  the nine float64 integral tables and the count table (rule 4), one CTA per image, a wavefront
//   k_org_normals   the per-pixel estimate (rule 5)
//
// The images of a call are processed in groups whose tables fit ORG_GROUP_BYTES; a group's points (host twin), distance
// map, normals (host twin) and tables are carved from one scratch slot (SCR_ORGANIZED), sized once for the largest group.
// Compiled with -fmad=false: every float32 / float64 operation is rounded on its own. The entry points
// gpdb_normals_organized[_device], with their argument checks, follow the kernels.
#include <cfloat>
#include <algorithm>
#include <climits>
#include <vector>

#include "../../include/gpd_b200_depth.h"
#include "../../include/gpd_b200_organized.h"
#include "common.cuh"
#include "grid.cuh"

namespace {

#include "pcl_eigen33.cuh"

constexpr int ORG_THREADS = 512;                    // threads of the wavefront CTAs (one image each)
constexpr size_t ORG_GROUP_BYTES = size_t(512) << 20;  // scratch of one group: pixels, distances, tables

// One image of a group. Its pixels are pix .. pix + W*H - 1 of the group's pixel arrays, its table entries
// tab .. tab + (W+1)*(H+1) - 1 of each of the group's ten tables (nine float64, one int32).
struct OrgImg {
  int pix, tab, W, H;
  float vp[3];
};
// The tables of a group: T entries each; channel ch of entry e is sum[ch * T + e] (x y z, xx xy xz yy yz zz)
struct OrgTabs {
  double *sum;
  int *cnt;
  int T;
};

// Rules 2 and 3: pixel i of the group starts the distance map at 0 (a pair test that touches it fails) or W + H.
__global__ void __launch_bounds__(256) k_org_change(const float *xyz, const int *pix_off, const OrgImg *im, int n_img, int P,
                                                    float *dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const OrgImg &I = im[csr_owner(pix_off, n_img, i)];
  const int W = I.W, H = I.H, p = i - I.pix, r = p / W, c = p % W;
  const float *z = xyz + 3 * (size_t)I.pix + 2;
  const auto Z = [&](int rr, int cc) { return z[3 * ((size_t)rr * W + cc)]; };
  const float zc = Z(r, c);
  bool brk = false;
  if (r < H - 1 && c < W - 1) brk = gpdb_org_pair_breaks(zc, Z(r, c + 1)) || gpdb_org_pair_breaks(zc, Z(r + 1, c));
  if (r < H - 1 && c >= 1) brk = brk || gpdb_org_pair_breaks(Z(r, c - 1), zc);  // the pair (r, c-1) - (r, c)
  if (r >= 1 && c < W - 1) brk = brk || gpdb_org_pair_breaks(Z(r - 1, c), zc);  // the pair (r-1, c) - (r, c)
  dist[i] = brk ? 0.0f : (float)(W + H);
}

// Rule 3, the two sequential passes, bit for bit. Pass 1 updates (r, c) from (r, c-1) and (r-1, c-1 .. c+1); at step
// t = (c-1) + 2(r-1) those were final at steps t-1, t-2, t-3 and t-1, so one step is a set of independent pixels (one per
// row) and a __syncthreads between steps orders every read after the write it needs. Each value is computed from the
// same operands with the same rounded operations as the sequential loop. The wrap read of the last column (UR = element 0
// of the current row) sees the initial value, which pass 1 never changes. Pass 2 is the mirror image: (r, c) at
// t = (W-2-c) + 2(H-2-r) reads (r, c+1) and (r+1, c-1 .. c+1), final at t-1 .. t-3; column 0 reads the current row's last
// element, which pass 2 never changes.
__global__ void __launch_bounds__(ORG_THREADS) k_org_dist(const OrgImg *im, float *dist) {
  const OrgImg I = im[blockIdx.x];
  const int W = I.W, H = I.H;
  float *d = dist + I.pix;
  const int steps = W >= 2 && H >= 2 ? (W - 2) + 2 * (H - 2) + 1 : 0;
  for (int t = 0; t < steps; t++) {
    for (int r = 1 + threadIdx.x; r < H; r += blockDim.x) {
      const int c = t - 2 * (r - 1) + 1;
      if (c >= 1 && c < W) {
        float *row = d + (size_t)r * W, *prev = row - W;
        const float m = gpdb_org_chamfer(prev[c - 1], prev[c], row[c - 1], prev[c + 1]);
        if (m < row[c]) row[c] = m;
      }
    }
    __syncthreads();
  }
  for (int t = 0; t < steps; t++) {
    for (int j = threadIdx.x; j < H - 1; j += blockDim.x) {
      const int r = H - 2 - j, c = W - 2 - t + 2 * j;
      if (c >= 0 && c <= W - 2) {
        float *row = d + (size_t)r * W, *next = row + W;
        const float m = gpdb_org_chamfer(next[c - 1], next[c], row[c + 1], next[c + 1]);
        if (m < row[c]) row[c] = m;
      }
    }
    __syncthreads();
  }
}

// Rule 4, bit for bit: pixel (r, c) writes entry (r+1, c+1) from (r, c+1), (r+1, c) and (r, c), the entries of pixels
// (r-1, c), (r, c-1) and (r-1, c-1), final at steps t-1, t-1 and t-2 of t = r + c. The count is an exact integer sum.
__global__ void __launch_bounds__(ORG_THREADS) k_org_integral(const OrgImg *im, const float *xyz, OrgTabs tb) {
  const OrgImg I = im[blockIdx.x];
  const int W = I.W, H = I.H, W1 = W + 1;
  double *S = tb.sum + I.tab;
  int *N = tb.cnt + I.tab;
  const size_t T = (size_t)tb.T;
  for (int e = threadIdx.x; e < W1 + H; e += blockDim.x) {  // row 0 and column 0
    const size_t k = e < W1 ? (size_t)e : (size_t)(e - W) * W1;
    for (int ch = 0; ch < 9; ch++) S[ch * T + k] = 0.0;
    N[k] = 0;
  }
  __syncthreads();
  const float *pts = xyz + 3 * (size_t)I.pix;
  for (int t = 0; t < W + H - 1; t++) {
    for (int r = threadIdx.x; r < H; r += blockDim.x) {
      const int c = t - r;
      if (c < 0 || c >= W) continue;
      const float *p = pts + 3 * ((size_t)r * W + c);
      const float q[3] = {p[0], p[1], p[2]};
      const bool f = gpdb_org_finite_point(q);
      const size_t ul = (size_t)r * W1 + c, up = ul + 1, left = ul + W1, me = left + 1;
      const double add[9] = {(double)q[0], (double)q[1], (double)q[2], (double)(q[0] * q[0]), (double)(q[0] * q[1]),
                             (double)(q[0] * q[2]), (double)(q[1] * q[1]), (double)(q[1] * q[2]), (double)(q[2] * q[2])};
#pragma unroll
      for (int ch = 0; ch < 9; ch++) {
        double *s = S + ch * T;
        double v = gpdb_org_integral(s[up], s[left], s[ul]);
        if (f) v += add[ch];
        s[me] = v;
      }
      N[me] = N[up] + N[left] - N[ul] + (f ? 1 : 0);
    }
    __syncthreads();
  }
}

// Rule 5 at pixel (r, c) of image I (pts, dist: the image's own arrays): the normal in the cloud's frame, NaN where the
// rule says so
__device__ void org_normal(const OrgImg &I, const float *pts, const float *dist, const OrgTabs &tb, int r, int c,
                           float n[3]) {
  const float nan = __int_as_float(0x7fc00000);
  n[0] = n[1] = n[2] = nan;
  const int W = I.W, H = I.H, B = GPDB_ORG_BORDER;
  if (r < B || r >= H - B || c < B || c >= W - B) return;
  const size_t p = (size_t)r * W + c;
  const float q[3] = {pts[3 * p], pts[3 * p + 1], pts[3 * p + 2]};
  if (!isfinite(q[2])) return;
  const float dm = dist[p];
  const float s = GPDB_ORG_SMOOTHING < dm ? GPDB_ORG_SMOOTHING : dm;  // std::min(dist, 20.0f)
  if (!(s > 2.0f)) return;
  const int w = (int)s, x0 = c - w / 2, y0 = r - w / 2, W1 = W + 1;
  const size_t ul = (size_t)y0 * W1 + x0, ur = ul + w, ll = (size_t)(y0 + w) * W1 + x0, lr = ll + w;
  const int *N = tb.cnt + I.tab;
  const int count = ((N[lr] + N[ul]) - N[ur]) - N[ll];
  if (count == 0) return;
  const double *S = tb.sum + I.tab;
  const size_t T = (size_t)tb.T;
  double sum[9];
#pragma unroll
  for (int ch = 0; ch < 9; ch++) {
    const double *t = S + ch * T;
    sum[ch] = gpdb_org_window(t[lr], t[ul], t[ur], t[ll]);
  }
  float cov[3][3];
  gpdb_org_covariance(sum, sum + 3, count, cov);
  pcl_eigen33_smallest(cov, n);
  gpdb_org_flip(q, I.vp, n);
}

// every pixel of the group: nrm[3i ..] = rule 5
__global__ void __launch_bounds__(256) k_org_normals(const float *xyz, const float *dist, const int *pix_off, const OrgImg *im,
                                                     int n_img, int P, OrgTabs tb, float *nrm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const OrgImg &I = im[csr_owner(pix_off, n_img, i)];
  const int p = i - I.pix;
  float n[3];
  org_normal(I, xyz + 3 * (size_t)I.pix, dist + I.pix, tb, p / I.W, p % I.W, n);
  nrm[3 * (size_t)i] = n[0];
  nrm[3 * (size_t)i + 1] = n[1];
  nrm[3 * (size_t)i + 2] = n[2];
}

// ---- depth views ---------------------------------------------------------------------------------------------------

// one camera of a depth call as the organized kernels read it
struct OrgCam {
  double R[9];
  double min_depth, max_depth;
  float fx, fy, cx, cy, scale;
  long long depth_pix;  // first pixel of the camera's image in the call's depth array
  int W, view_pix;      // width; first pixel of the camera in its view's raw numbering
};

// rule 6: the camera-frame point of group pixel i (gpd_b200_depth.h rule 2 without the pose), NaN when invalid
__global__ void __launch_bounds__(256) k_org_backproject(const void *depth, int format, const OrgCam *cams, int c0,
                                                         const int *pix_off, const OrgImg *im, int n_img, int P, float *xyz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const int k = csr_owner(pix_off, n_img, i);
  const OrgCam &K = cams[c0 + k];
  const int p = i - im[k].pix;
  const long long di = K.depth_pix + p;
  float z;
  bool ret;
  if (format == GPDB_DEPTH_U16) {
    const uint16_t raw = static_cast<const uint16_t *>(depth)[di];
    ret = raw != 0;
    z = (float)raw * K.scale;
  } else {
    const float raw = static_cast<const float *>(depth)[di];
    ret = isfinite(raw) && raw > 0.0f;
    z = raw * K.scale;
  }
  const bool valid = ret && (double)z >= K.min_depth && (double)z <= K.max_depth;
  float *o = xyz + 3 * (size_t)i;
  if (!valid) {
    o[0] = o[1] = o[2] = __int_as_float(0x7fc00000);
    return;
  }
  const int u = p % K.W, v = p / K.W;
  o[0] = (((float)u - K.cx) * z) / K.fx;
  o[1] = (((float)v - K.cy) * z) / K.fy;
  o[2] = z;
}

// rule 7 for the processed points whose representative pixel belongs to a camera of the group (cameras c0 .. c0+n_img-1
// of the call; view b's cameras start at cam0[b]): a finite world normal replaces the radius estimate in nrm_out, then
// reverseNormals as k_normals applies it, and the point is flagged organized
__global__ void __launch_bounds__(256) k_org_depth_normals(DevCloud cl, CloudTable tab, int N, const int *src, const int *cam0,
                                                           const OrgCam *cams, int c0, const float *xyz, const float *dist,
                                                           const OrgImg *im, int n_img, OrgTabs tb, double *nrm_out,
                                                           uint8_t *organized) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const int b = b_cloud_of_point(tab.d, tab.n, g);
  const CloudDesc &G = tab.d[b];
  const int raw = src[g];
  int c = cam0[b];
  for (int k = 1; k < G.K && raw >= cams[cam0[b] + k].view_pix; k++) c = cam0[b] + k;
  if (c < c0 || c >= c0 + n_img) return;
  const uint8_t camm = cl.cam[g];
  if (camm == 0) return;
  const OrgImg &I = im[c - c0];
  const OrgCam &K = cams[c];
  const int p = raw - K.view_pix;
  float nc[3], nw[3];
  org_normal(I, xyz + 3 * (size_t)I.pix, dist + I.pix, tb, p / I.W, p % I.W, nc);
  gpdb_org_rotate(K.R, nc, nw);
  if (!isfinite(nw[0]) || !isfinite(nw[1]) || !isfinite(nw[2])) return;
  const float q[3] = {cl.xyz[3 * (size_t)g], cl.xyz[3 * (size_t)g + 1], cl.xyz[3 * (size_t)g + 2]};
  double nd[3] = {(double)nw[0], (double)nw[1], (double)nw[2]};
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
  double *out = nrm_out + 3 * (size_t)g;
  out[0] = nd[0];
  out[1] = nd[1];
  out[2] = nd[2];
  organized[g] = 1;
}

// fallback points per view: count[b] += 1 for every point without an organized normal
__global__ void k_org_fallback_count(CloudTable tab, int N, const uint8_t *organized, int *count) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < N && !organized[g]) atomicAdd(count + b_cloud_of_point(tab.d, tab.n, g), 1);
}

// ---- groups ------------------------------------------------------------------------------------------------------

// the images [first, last) of one group
struct OrgGroup {
  int first, last, pixels;
  long long entries;
};

size_t org_table_bytes(long long entries) { return entries * (9 * sizeof(double) + sizeof(int)); }

// consecutive images, each group's tables within ORG_GROUP_BYTES (an image larger than that is a group of its own)
std::vector<OrgGroup> org_groups(int n, const int *W, const int *H) {
  std::vector<OrgGroup> g;
  OrgGroup cur{0, 0, 0, 0};
  for (int i = 0; i < n; i++) {
    const int px = W[i] * H[i];
    const long long en = (long long)(W[i] + 1) * (H[i] + 1);
    if (cur.last > cur.first && org_table_bytes(cur.entries + en) > ORG_GROUP_BYTES) {
      g.push_back(cur);
      cur = OrgGroup{i, i, 0, 0};
    }
    cur.last = i + 1;
    cur.pixels += px;
    cur.entries += en;
  }
  g.push_back(cur);
  return g;
}

// The scratch of one group: the images and their pixel offsets, the group's points, distance map and normals where the
// call does not use the caller's arrays, and its tables; sized for the largest of the groups
struct OrgScratch {
  OrgImg *im;
  int *pix_off;
  float *xyz, *dist, *nrm;
  OrgTabs tb;
};
bool org_carve(gpdb_ctx *ctx, int n_img, int pixels, int entries, bool own_xyz, bool own_dist, bool own_nrm, OrgScratch &o) {
  return gpdb_carve(ctx, SCR_ORGANIZED, [&](Carve &c) {
    o.im = c.take<OrgImg>(n_img);
    o.pix_off = c.take<int>((size_t)n_img + 1);
    o.xyz = own_xyz ? c.take<float>(3 * (size_t)pixels) : nullptr;
    o.dist = own_dist ? c.take<float>(pixels) : nullptr;
    o.nrm = own_nrm ? c.take<float>(3 * (size_t)pixels) : nullptr;
    o.tb.sum = c.take<double>(9 * (size_t)entries);
    o.tb.cnt = c.take<int>(entries);
    o.tb.T = entries;
  });
}

// The image table of a group (view points vp[3i..] per image of the call) into o.im / o.pix_off
int org_upload(gpdb_ctx *ctx, const OrgGroup &G, const int *W, const int *H, const float *vp, const OrgScratch &o) {
  const int n = G.last - G.first;
  std::vector<OrgImg> im(n);
  std::vector<int> pix_off((size_t)n + 1, 0);
  for (int k = 0, tab = 0; k < n; k++) {
    const int i = G.first + k;
    im[k] = OrgImg{pix_off[k], tab, W[i], H[i], {vp[3 * i], vp[3 * i + 1], vp[3 * i + 2]}};
    pix_off[k + 1] = pix_off[k] + W[i] * H[i];
    tab += (W[i] + 1) * (H[i] + 1);
  }
  CUDA_TRY(cudaMemcpyAsync(o.im, im.data(), sizeof(OrgImg) * n, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(o.pix_off, pix_off.data(), sizeof(int) * ((size_t)n + 1), cudaMemcpyHostToDevice, ctx->stream));
  return GPDB_OK;
}

// rules 2 - 4 on the group's points xyz (its image table uploaded), with its distance map in dist
int org_maps(gpdb_ctx *ctx, const OrgGroup &G, const OrgScratch &o, const float *xyz, float *dist) {
  const int n = G.last - G.first, P = G.pixels;
  k_org_change<<<(P + 255) / 256, 256, 0, ctx->stream>>>(xyz, o.pix_off, o.im, n, P, dist);
  LAUNCH_CHECK();
  k_org_dist<<<n, ORG_THREADS, 0, ctx->stream>>>(o.im, dist);
  LAUNCH_CHECK();
  k_org_integral<<<n, ORG_THREADS, 0, ctx->stream>>>(o.im, xyz, o.tb);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// the scratch of the largest group; GPDB_ERR_INVALID when one image's tables exceed the int32 entry range
int org_scratch(gpdb_ctx *ctx, const char *name, const std::vector<OrgGroup> &groups, bool own_xyz, bool own_dist,
                bool own_nrm, OrgScratch &o) {
  int n_max = 0, p_max = 0;
  long long e_max = 0;
  for (const OrgGroup &G : groups) {
    n_max = std::max(n_max, G.last - G.first);
    p_max = std::max(p_max, G.pixels);
    e_max = std::max(e_max, G.entries);
  }
  if (e_max > INT_MAX) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: an image of %lld integral-table entries (2^31 or more)", name, e_max);
    return GPDB_ERR_INVALID;
  }
  return org_carve(ctx, n_max, p_max, (int)e_max, own_xyz, own_dist, own_nrm, o) ? GPDB_OK : GPDB_ERR_CUDA;
}

// Rules 2 - 5 on B organized clouds (cloud b: W[b] x H[b] points, view point vp[3b..], concatenated in xyz): nrm_out
// [3 * pixels] and dist_out [pixels] (may be null). device: xyz and the outputs are device arrays, else host arrays.
// `name` is the entry point the errors name.
int org_normals_batch(gpdb_ctx *ctx, const char *name, int B, const int *W, const int *H, const float *xyz, const float *vp,
                      float *nrm_out, float *dist_out, bool device) {
  const std::vector<OrgGroup> groups = org_groups(B, W, H);
  OrgScratch o;
  int rc = org_scratch(ctx, name, groups, !device, !device || !dist_out, !device, o);
  if (rc != GPDB_OK) return rc;
  long long pix0 = 0;
  for (const OrgGroup &G : groups) {
    const int P = G.pixels;
    const float *gx = device ? xyz + 3 * pix0 : o.xyz;
    float *gd = device && dist_out ? dist_out + pix0 : o.dist;
    float *gn = device ? nrm_out + 3 * pix0 : o.nrm;
    if (!device)
      CUDA_TRY(cudaMemcpyAsync(o.xyz, xyz + 3 * pix0, sizeof(float) * 3 * (size_t)P, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = org_upload(ctx, G, W, H, vp, o)) != GPDB_OK || (rc = org_maps(ctx, G, o, gx, gd)) != GPDB_OK) return rc;
    k_org_normals<<<(P + 255) / 256, 256, 0, ctx->stream>>>(gx, gd, o.pix_off, o.im, G.last - G.first, P, o.tb, gn);
    LAUNCH_CHECK();
    if (!device) {
      CUDA_TRY(cudaMemcpyAsync(nrm_out + 3 * pix0, o.nrm, sizeof(float) * 3 * (size_t)P, cudaMemcpyDeviceToHost, ctx->stream));
      if (dist_out)
        CUDA_TRY(cudaMemcpyAsync(dist_out + pix0, o.dist, sizeof(float) * (size_t)P, cudaMemcpyDeviceToHost, ctx->stream));
    }
    pix0 += P;
  }
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return GPDB_OK;
}

}  // namespace

int org_depth_normals(gpdb_ctx *ctx, const char *name, CloudSet &s, const void *d_depth, int format,
                      const gpdb_depth_camera *cams, const int *n_cameras, int B, int *n_fallback) {
  const int tb = 256, N = s.points();
  int C = 0;
  for (int b = 0; b < B; b++) C += n_cameras[b];
  // host tables: the cameras, each view's first camera, widths / heights, and view points at the camera origin
  std::vector<OrgCam> hc(C);
  std::vector<int> cam0((size_t)B), W(C), H(C);
  std::vector<float> vp(3 * (size_t)C, 0.0f);
  long long dpix = 0;
  for (int b = 0, c = 0; b < B; b++) {
    cam0[b] = c;
    for (int k = 0, vpix = 0; k < n_cameras[b]; k++, c++) {
      const gpdb_depth_camera &D = cams[c];
      OrgCam &K = hc[c];
      for (int r = 0; r < 3; r++)
        for (int q = 0; q < 3; q++) K.R[3 * r + q] = D.pose[4 * r + q];
      K.min_depth = D.min_depth;
      K.max_depth = D.max_depth;
      K.fx = (float)D.fx, K.fy = (float)D.fy, K.cx = (float)D.cx, K.cy = (float)D.cy, K.scale = (float)D.depth_scale;
      K.depth_pix = dpix;
      K.W = D.width;
      K.view_pix = vpix;
      W[c] = D.width;
      H[c] = D.height;
      vpix += D.width * D.height;
      dpix += (long long)D.width * D.height;
    }
  }
  const std::vector<OrgGroup> groups = org_groups(C, W.data(), H.data());
  OrgScratch o;
  int rc = org_scratch(ctx, name, groups, true, true, false, o);
  if (rc != GPDB_OK) return rc;
  // the call's cameras, the views' first cameras, the fallback counts and the organized flags
  OrgCam *d_cams;
  int *d_cam0, *d_fb;
  uint8_t *d_org;
  if (!gpdb_carve(ctx, SCR_ORGANIZED_DEPTH, [&](Carve &c) {
        d_cams = c.take<OrgCam>(C); d_cam0 = c.take<int>(B); d_fb = c.take<int>(B); d_org = c.take<uint8_t>((size_t)N + 1);
      }))
    return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(d_cams, hc.data(), sizeof(OrgCam) * (size_t)C, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(d_cam0, cam0.data(), sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(d_fb, 0, sizeof(int) * (size_t)B, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(d_org, 0, (size_t)N + 1, ctx->stream));
  const CloudTable tab = s.table();
  for (const OrgGroup &G : groups) {
    const int n = G.last - G.first, P = G.pixels;
    if ((rc = org_upload(ctx, G, W.data(), H.data(), vp.data(), o)) != GPDB_OK) return rc;
    k_org_backproject<<<(P + tb - 1) / tb, tb, 0, ctx->stream>>>(d_depth, format, d_cams, G.first, o.pix_off, o.im, n, P,
                                                                 o.xyz);
    LAUNCH_CHECK();
    if ((rc = org_maps(ctx, G, o, o.xyz, o.dist)) != GPDB_OK) return rc;
    if (N > 0) {
      k_org_depth_normals<<<(N + tb - 1) / tb, tb, 0, ctx->stream>>>(s.view, tab, N, s.src, d_cam0, d_cams, G.first, o.xyz,
                                                                     o.dist, o.im, n, o.tb, s.nrm, d_org);
      LAUNCH_CHECK();
    }
  }
  if (N > 0) {
    k_org_fallback_count<<<(N + tb - 1) / tb, tb, 0, ctx->stream>>>(tab, N, d_org, d_fb);
    LAUNCH_CHECK();
  }
  if (n_fallback) CUDA_TRY(cudaMemcpyAsync(n_fallback, d_fb, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return GPDB_OK;
}

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

// gpdb_normals_organized[_device]: the argument checks, then rules 2 - 5 of gpd_b200_organized.h on every cloud
static int organized_entry(gpdb_ctx *ctx, const char *name, int32_t B, const int32_t *W, const int32_t *H, const float *xyz,
                           const float *view_points, float *normals_out, float *distance_out, bool device) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (B <= 0 || !W || !H || !xyz || !view_points || !normals_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need n_clouds > 0, widths, heights, xyz, view_points, normals_out", name);
    return GPDB_ERR_INVALID;
  }
  long long total = 0;
  for (int b = 0; b < B; b++) {
    if (W[b] < 1 || H[b] < 1) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: cloud %d is %d x %d (width and height must be at least 1)", name, b, W[b],
                     H[b]);
      return GPDB_ERR_INVALID;
    }
    total += (long long)W[b] * H[b];
    if (total >= (1ll << 31)) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: cloud %d: the call holds 2^31 or more points", name, b);
      return GPDB_ERR_INVALID;
    }
  }
  int rc = device ? gpdb_check_device_ptrs(ctx, name, {{"d_xyz", xyz}, {"d_normals_out", normals_out},
                                                       {"d_distance_out", distance_out}})
                  : GPDB_OK;
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaSetDevice(ctx->device));
  rc = org_normals_batch(ctx, name, B, W, H, xyz, view_points, normals_out, distance_out, device);
  return rc == GPDB_OK ? B : rc;
}

extern "C" {

int gpdb_normals_organized(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *widths, const int32_t *heights, const float *xyz,
                           const float *view_points, float *normals_out, float *distance_out) {
  return organized_entry(ctx, "gpdb_normals_organized", n_clouds, widths, heights, xyz, view_points, normals_out,
                         distance_out, false);
}

int gpdb_normals_organized_device(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *widths, const int32_t *heights,
                                  const float *d_xyz, const float *view_points, float *d_normals_out,
                                  float *d_distance_out) {
  return organized_entry(ctx, "gpdb_normals_organized_device", n_clouds, widths, heights, d_xyz, view_points,
                         d_normals_out, d_distance_out, true);
}

}  // extern "C"
