// api.cu — the C-ABI of libgpd_b200.so (include/gpd_b200.h): the context, the cloud store, the checks the other entry
// points share (common.cuh), the chunked detect pipeline and the detect / hand-search / frames / images / classify /
// reevaluate / cluster entry points. Host-side logic only; their kernels live in geometry.cu / lenet_simt.cu /
// lenet_tc.cu. The depth, mesh, organized-normal, plane, refinement, outlier, training and SIS entry points sit beside
// their kernels, in depth.cu / render.cu / organized.cu / plane.cu / refine.cu / outliers.cu / train.cu / sis.cu.
// There is no CPU fallback anywhere in this library.
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>

#include "common.cuh"

static char g_create_err[512] = "";

struct StageTimes {
  struct Span { int stage; cudaEvent_t b, e; };
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  std::vector<Span> spans;
  cudaEvent_t get() {
    if (used == pool.size()) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      pool.push_back(e);
    }
    return pool[used++];
  }
  ~StageTimes() { for (cudaEvent_t e : pool) cudaEventDestroy(e); }
};
cudaEvent_t gpdb_st_begin(gpdb_ctx *ctx) {
  cudaEvent_t e = ctx->st->get();
  cudaEventRecord(e, ctx->stream);
  return e;
}
void gpdb_st_end(gpdb_ctx *ctx, int stage, cudaEvent_t begin) {
  cudaEvent_t e = ctx->st->get();
  cudaEventRecord(e, ctx->stream);
  ctx->st->spans.push_back({stage, begin, e});
}

static void st_collect(gpdb_ctx *ctx, double *ms) {
  for (auto &sp : ctx->st->spans) {
    float t = 0;
    if (cudaEventElapsedTime(&t, sp.b, sp.e) == cudaSuccess) ms[sp.stage] += t;
  }
  ctx->st->spans.clear();
  ctx->st->used = 0;
}



void gpdb_set_error(gpdb_ctx *ctx, int code, const char *fmt, ...) {
  char buf[480];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  char *dst = ctx ? ctx->err : g_create_err;
  snprintf(dst, 512, "gpd_b200 error %d: %s", code, buf);
  fprintf(stderr, "%s\n", dst);  // reference convention: errors are also printed
}

void *gpdb_scratch(gpdb_ctx *ctx, ScratchSlot slot, size_t bytes) {
  if (bytes == 0) bytes = 16;
  if (ctx->scratch_sz[slot] >= bytes) return ctx->scratch[slot];
  if (ctx->scratch[slot]) {
    cudaStreamSynchronize(ctx->stream);
    cudaFree(ctx->scratch[slot]);
    ctx->scratch[slot] = nullptr;
    ctx->scratch_sz[slot] = 0;
  }
  size_t want = bytes + bytes / 4 + 256;
  if (cudaMalloc(&ctx->scratch[slot], want) != cudaSuccess) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "cudaMalloc(%zu) failed for scratch slot %d: %s", want, slot,
                   cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  ctx->scratch_sz[slot] = want;
  return ctx->scratch[slot];
}

// ---- host restatements of the Eigen helpers that define the rotation set --------------------------
// Eigen::AngleAxisd(angle, axis).toRotationMatrix(), column-major (hand_set.cpp:52-53,68-69)
static void angle_axis_matrix(double angle, const double axis[3], double *R) {
  double s = std::sin(angle), c = std::cos(angle);
  double sa[3] = {s * axis[0], s * axis[1], s * axis[2]};
  double c1[3] = {(1.0 - c) * axis[0], (1.0 - c) * axis[1], (1.0 - c) * axis[2]};
  double t;
  t = c1[0] * axis[1]; R[1 * 3 + 0] = t - sa[2]; R[0 * 3 + 1] = t + sa[2];
  t = c1[0] * axis[2]; R[2 * 3 + 0] = t + sa[1]; R[0 * 3 + 2] = t - sa[1];
  t = c1[1] * axis[2]; R[2 * 3 + 1] = t - sa[0]; R[1 * 3 + 2] = t + sa[0];
  R[0] = c1[0] * axis[0] + c;
  R[4] = c1[1] * axis[1] + c;
  R[8] = c1[2] * axis[2] + c;
}
// Eigen 3.3 VectorXd::LinSpaced(size, low, high)(i)
static double linspaced(int size, double low, double high, int i) {
  int size1 = size == 1 ? 1 : size - 1;
  double step = size == 1 ? 0.0 : (high - low) / (double)(size - 1);
  bool flip = std::fabs(high) < std::fabs(low);
  if (flip) return (i == 0) ? low : (high - (double)(size1 - i) * step);
  return (i == size1) ? high : (low + (double)i * step);
}

// doubles <-> integers in the same order (-0 and +0 share key 0), so that bisection can walk adjacent doubles
static long long ordered_key(double x) {
  long long b;
  memcpy(&b, &x, sizeof(b));
  return b < 0 ? -(b & 0x7fffffffffffffffLL) : b;
}
static double from_ordered_key(long long k) {
  long long b = k < 0 ? (-k) | (long long)0x8000000000000000ULL : k;
  double x;
  memcpy(&x, &b, sizeof(x));
  return x;
}

// filterGraspsDirection (grasp_detector.cpp:437-438) erases a grasp when std::acos(dot) > thresh_rad. CUDA's acos is not
// correctly rounded (2 ulp), so the kernel must not evaluate it: acos is non-increasing on [-1, 1], and the predicate
// becomes dot < d*, with d* the smallest double in [-1, 1] that the host's acos keeps (2 when it keeps none, -1 when it
// keeps all, as for a NaN or >= pi threshold). |dot| > 1 and NaN give acos = NaN, which the reference keeps.
static int direction_keep_edge(gpdb_ctx *ctx, double thresh, double *d_star) {
  auto rejects = [thresh](long long k) { return std::acos(from_ordered_key(k)) > thresh; };
  long long lo = ordered_key(-1.0), hi = ordered_key(1.0);
  if (!rejects(lo)) {
    *d_star = -1.0;
    return GPDB_OK;
  }
  if (rejects(hi)) {
    *d_star = 2.0;
    return GPDB_OK;
  }
  while (hi - lo > 1) {  // rejects(lo), !rejects(hi)
    long long mid = lo + (hi - lo) / 2;
    (rejects(mid) ? lo : hi) = mid;
  }
  // the bisection is right only if the host acos is non-increasing over all of [-1, 1], which libm's acos is; this
  // check is local: it confirms one switch across the 256 doubles either side of it and catches a libm that is not
  for (long long k = 1; k <= 256; k++)
    if ((hi - k >= ordered_key(-1.0) && !rejects(hi - k)) || (hi + k <= ordered_key(1.0) && rejects(hi + k))) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "the host acos is not monotone near thresh_rad = %.17g", thresh);
      return GPDB_ERR_INVALID;
    }
  *d_star = from_ordered_key(hi);
  return GPDB_OK;
}

static int fill_dev_params(gpdb_ctx *ctx) {
  const gpdb_params &p = ctx->prm;
  DevParams &d = ctx->hp;
  memset(&d, 0, sizeof(d));
  if (p.num_orientations < 1 || p.num_orientations > GPDB_MAX_ORIENT || p.num_hand_axes < 1 ||
      p.num_hand_axes > GPDB_MAX_HAND_AXES || p.num_finger_placements < 1 || 2 * p.num_finger_placements > GPDB_MAX_SLOTS ||
      p.image_size < 8 || p.image_size > 64 ||
      !(p.image_num_channels == 1 || p.image_num_channels == 3 || p.image_num_channels == 12 || p.image_num_channels == 15)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID,
                   "unsupported parameters (num_orientations 1..%d, hand_axes 1..3, num_finger_placements 1..%d, "
                   "image_size 8..64, image_num_channels 1/3/12/15)", GPDB_MAX_ORIENT, GPDB_MAX_SLOTS / 2);
    return GPDB_ERR_INVALID;
  }
  d.finger_width = p.finger_width;
  d.hand_outer_diameter = p.hand_outer_diameter;
  d.hand_depth = p.hand_depth;
  d.hand_height = p.hand_height;
  d.init_bite = p.init_bite;
  d.n_axes = p.num_hand_axes;
  d.n_orient = p.num_orientations;
  d.P = d.n_axes * d.n_orient;
  d.nfp = p.num_finger_placements;
  d.deepen = p.deepen_hand;
  d.all_axes_z = 1;
  for (int a = 0; a < d.n_axes; a++) {
    if (p.hand_axes[a] < 0 || p.hand_axes[a] > 2) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "hand_axes[%d] = %d out of range 0..2", a, p.hand_axes[a]);
      return GPDB_ERR_INVALID;
    }
    d.axes[a] = p.hand_axes[a];
    if (p.hand_axes[a] != 2) d.all_axes_z = 0;
  }
  // FingerHand::FingerHand (finger_hand.cpp:6-24)
  for (int i = 0; i < d.nfp; i++) {
    double h = linspaced(d.nfp, 0.0, p.hand_outer_diameter - p.finger_width, i);
    d.fs[i] = (h - p.hand_outer_diameter) + p.finger_width;
    d.fs[d.nfp + i] = h;
  }
  for (int i = 0; i < 2 * d.nfp; i++) d.fsw[i] = d.fs[i] + p.finger_width;
  d.slots_disjoint = d.nfp >= 3 ? 1 : 0;  // the arithmetic slot lookup needs >= 3 equally spaced slots; else linear scan
  d.inv_slot_step = d.nfp >= 2 ? 1.0 / (d.fs[1] - d.fs[0]) : 0.0;
  for (int i = 0; i + 1 < d.nfp; i++)
    if (!(d.fsw[i] <= d.fs[i + 1]) || !(d.fsw[d.nfp + i] <= d.fs[d.nfp + i + 1])) d.slots_disjoint = 0;
  // deepenHand steps (finger_hand.cpp:118-121): repeated += 0.005 in double
  d.J = 0;
  for (double depth = p.init_bite + 0.005; depth <= p.hand_depth; depth += 0.005) {
    if (d.J >= GPDB_MAX_DEEPEN) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "more than %d deepen steps", GPDB_MAX_DEEPEN);
      return GPDB_ERR_INVALID;
    }
    d.topj[d.J] = depth;
    d.botj[d.J] = depth - p.hand_depth;
    d.J++;
  }
  d.cosf = std::cos(p.friction_coeff * M_PI / 180.0);
  d.min_viable = p.min_viable;
  d.min_ap = p.min_aperture;
  d.max_ap = p.max_aperture;
  for (int i = 0; i < 6; i++) d.ws[i] = p.workspace_grasps[i];
  d.filt_dir = p.filter_approach_direction;
  for (int i = 0; i < 3; i++) d.dir[i] = p.direction[i];
  d.thresh = p.thresh_rad;
  if (direction_keep_edge(ctx, p.thresh_rad, &d.dir_keep) != GPDB_OK) return GPDB_ERR_INVALID;
  const double uy[3] = {0, 1, 0};
  angle_axis_matrix(M_PI, uy, d.rotb);
  static const double AXES[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int a = 0; a < d.n_axes; a++)
    for (int i = 0; i < d.n_orient; i++) {
      // angles = LinSpaced(n+1, -pi/2, pi/2).head(n) (hand_search.cpp:151-155)
      double ang = linspaced(d.n_orient + 1, -1.0 * M_PI / 2.0, M_PI / 2.0, i);
      angle_axis_matrix(ang, AXES[d.axes[a]], d.rot[a * d.n_orient + i]);
    }
  d.vol_w = p.volume_width;
  d.vol_d = p.volume_depth;
  d.vol_h = p.volume_height;
  d.S = p.image_size;
  d.C = p.image_num_channels;
  // radii: hand_search.cpp:13-17, image_generator.cpp:43-46, image_15_channels_strategy.h:72-75
  double r_hs = std::max(std::max(p.hand_outer_diameter - p.finger_width, p.hand_depth), p.hand_height / 2.0);
  double r_img = std::max(std::max(p.volume_depth, p.volume_height / 2.0), p.volume_width);
  double r_lrf = p.nn_radius;
  d.r2_lrf = (float)(r_lrf * r_lrf);
  d.r2_hs = (float)(r_hs * r_hs);
  d.r2_img = (float)(r_img * r_img);
  d.rf_lrf = (float)r_lrf * 1.0001f + 1e-6f;
  d.rf_hs = (float)r_hs * 1.0001f + 1e-6f;
  d.rf_img = (float)r_img * 1.0001f + 1e-6f;
  d.shadow_length = r_img;
  d.vox_mult = 1.0 / GPDB_SHADOW_VOXEL;
  d.nsp = (int)std::floor(d.shadow_length / GPDB_SHADOW_VOXEL);
  if (d.nsp > GPDB_MAX_NSP) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "image volume too large: %d shadow draws per point (max %d)", d.nsp, GPDB_MAX_NSP);
    return GPDB_ERR_INVALID;
  }
  {  // closed-form skip-ahead of HandSet::fastrand (hand_set.cpp:263-266), mod 2^32
    unsigned A = 1u, Cc = 0u;
    for (int t = 0; t < GPDB_MAX_NSP; t++) {
      Cc = 214013u * Cc + 2531011u;
      A = 214013u * A;
      d.lcgA[t] = A;
      d.lcgC[t] = Cc;
    }
  }
  double diag = std::sqrt(p.volume_depth * p.volume_depth + p.volume_width * p.volume_width +
                          4.0 * p.volume_height * p.volume_height);
  d.bm_dim = (int)std::ceil((diag + 2.0 * 3.2 * GPDB_SHADOW_VOXEL * 0.3) / GPDB_SHADOW_VOXEL) + 4;
  if (d.bm_dim > 64 && d.C == 15) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "image volume too large for the shadow bitmap (%d > 64 voxels across)", d.bm_dim);
    return GPDB_ERR_INVALID;
  }
  d.relu_after_conv = p.relu_after_conv;
  return GPDB_OK;
}

static void cloud_free(CloudSet &s) {
  void *dev[] = {s.pts4, s.xyz, s.nrm, s.cam, s.src, s.cell_start, s.desc, s.soff, s.samples};
  for (void *p : dev) cudaFree(p);
  free(s.off);
  free(s.sel);
  free(s.pos);
  free(s.raw_off);
}

extern "C" {

void gpdb_params_default(gpdb_params *p) {
  memset(p, 0, sizeof(*p));
  p->finger_width = 0.01;
  p->hand_outer_diameter = 0.12;
  p->hand_depth = 0.06;
  p->hand_height = 0.02;
  p->init_bite = 0.01;
  p->volume_width = 0.10;
  p->volume_depth = 0.06;
  p->volume_height = 0.02;
  p->image_size = 60;
  p->image_num_channels = 15;
  p->nn_radius = 0.01;
  p->num_orientations = 8;
  p->num_finger_placements = 10;
  p->num_hand_axes = 1;
  p->hand_axes[0] = 2;
  p->deepen_hand = 1;
  p->friction_coeff = 20.0;
  p->min_viable = 6;
  p->min_aperture = 0.0;
  p->max_aperture = 0.085;
  const double ws[6] = {-1, 1, -1, 1, -1, 1};
  for (int i = 0; i < 6; i++) p->workspace_grasps[i] = ws[i];
  p->filter_approach_direction = 0;
  p->direction[0] = 1.0;
  p->thresh_rad = 2.3;
}

const char *gpdb_build_info(void) {
  return "gpd_b200 v1, sm_90a, kernels: k_frames k_hands k_images k_normals (fp64 / PCL-order fp32, -fmad=false), lenet: "
         "conv1 wgmma u8 x s8 implicit GEMM (uint8 image x 3 int8 weight digit planes, exact int32 accumulators), conv2 wgmma "
         "f16 implicit GEMM + ip1 TMA-fed wgmma GEMM (fp16 hi/lo split operands, fp32 accumulate), ip2 simt; "
         "lenet_impl=1 forces the simt-fp32 kernels";
}

const char *gpdb_last_error(const gpdb_ctx *ctx) { return ctx ? ctx->err : g_create_err; }

int gpdb_create(const gpdb_params *params, gpdb_ctx **ctx_out) {
  if (!params || !ctx_out) {
    gpdb_set_error(nullptr, GPDB_ERR_INVALID, "gpdb_create: null argument");
    return GPDB_ERR_INVALID;
  }
  *ctx_out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    gpdb_set_error(nullptr, GPDB_ERR_CUDA, "no CUDA device: libgpd_b200 has no CPU fallback");
    return GPDB_ERR_CUDA;
  }
  if (params->device < 0 || params->device >= ndev) {
    gpdb_set_error(nullptr, GPDB_ERR_INVALID, "device %d out of range (have %d)", params->device, ndev);
    return GPDB_ERR_INVALID;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, params->device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
    gpdb_set_error(nullptr, GPDB_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a (H100) only",
                   params->device, prop.major, prop.minor);
    return GPDB_ERR_CUDA;
  }
  gpdb_ctx *ctx = new gpdb_ctx();
  memset(ctx, 0, sizeof(*ctx));
  ctx->st = new StageTimes();
  ctx->own_stream = true;
  ctx->prm = *params;
  ctx->device = params->device;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->smem_optin = (int)prop.sharedMemPerBlockOptin;
  int rc = fill_dev_params(ctx);
  if (rc != GPDB_OK) {
    strncpy(g_create_err, ctx->err, sizeof(g_create_err) - 1);
    delete ctx->st;
    delete ctx;
    return rc;
  }
  bool ok = cudaSetDevice(ctx->device) == cudaSuccess &&
            cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) == cudaSuccess &&
            cudaMalloc(&ctx->dp, sizeof(DevParams)) == cudaSuccess &&
            cudaMalloc(&ctx->d_err, sizeof(int) * GPDB_NERR) == cudaSuccess &&
            cudaMalloc(&ctx->d_qtab, sizeof(double) * GPDB_QTAB_SIZE) == cudaSuccess;
  if (ok) {
    double qt[GPDB_QTAB_SIZE];
    gpdb_build_qtab(qt);
    ok = cudaMemcpy(ctx->d_qtab, qt, sizeof(qt), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(ctx->dp, &ctx->hp, sizeof(DevParams), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemset(ctx->d_err, 0, sizeof(int) * GPDB_NERR) == cudaSuccess;
  }
  for (cudaEvent_t &e : ctx->ev) ok = ok && cudaEventCreate(&e) == cudaSuccess;
  ok = ok && gpdb_pipe_create(ctx) == GPDB_OK;
  ctx->overlap_hands = !(getenv("GPD_B200_OVERLAP") && getenv("GPD_B200_OVERLAP")[0] == '0');
  if (!ok) {
    gpdb_set_error(nullptr, GPDB_ERR_CUDA, "context setup failed: %s", cudaGetErrorString(cudaGetLastError()));
    gpdb_destroy(ctx);
    return GPDB_ERR_CUDA;
  }
  *ctx_out = ctx;
  return GPDB_OK;
}

void gpdb_destroy(gpdb_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  gpdb_comm_destroy(ctx);
  train_free(ctx);
  gpdb_pipe_destroy(ctx);
  cudaFree(ctx->dp);
  cudaFree(ctx->d_err);
  cudaFree(ctx->d_prof);
  cudaFree(ctx->d_qtab);
  cudaFree(ctx->d_sel);
  sis_free(ctx);
  cloud_free(ctx->one);
  cloud_free(ctx->many);
  float *w[8] = {ctx->w.c1w, ctx->w.c1b, ctx->w.c2w, ctx->w.c2b, ctx->w.i1w, ctx->w.i1b, ctx->w.i2w, ctx->w.i2b};
  for (float *p : w) cudaFree(p);
  cudaFree(ctx->tc.b1);
  cudaFree(ctx->tc.b2);
  cudaFree(ctx->tc.b3);
  for (int i = 0; i < SCR_N; i++) cudaFree(ctx->scratch[i]);
  for (cudaEvent_t e : ctx->ev)
    if (e) cudaEventDestroy(e);
  if (ctx->stream && ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx->st;
  delete ctx;
}

int gpdb_set_weights(gpdb_ctx *ctx, const float *conv1_w, const float *conv1_b, const float *conv2_w,
                     const float *conv2_b, const float *ip1_w, const float *ip1_b, const float *ip2_w,
                     const float *ip2_b) {
  if (!ctx) return GPDB_ERR_INVALID;
  const float *w[8] = {conv1_w, conv1_b, conv2_w, conv2_b, ip1_w, ip1_b, ip2_w, ip2_b};
  for (const float *p : w)
    if (!p) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_set_weights: null weight array");
      return GPDB_ERR_INVALID;
    }
  CUDA_TRY(cudaSetDevice(ctx->device));
  return lenet_upload(ctx, w);
}

// readBinaryFileIntoVector (eigen_classifier.cpp:185-205)
int gpdb_load_weights_dir(gpdb_ctx *ctx, const char *dir) {
  if (!ctx || !dir) return GPDB_ERR_INVALID;
  const int C = ctx->prm.image_num_channels;
  const char *names[8] = {"conv1_weights", "conv1_biases", "conv2_weights", "conv2_biases",
                          "ip1_weights",   "ip1_biases",   "ip2_weights",   "ip2_biases"};
  const size_t sizes[8] = {(size_t)20 * C * 25, 20, 50 * 20 * 25, 50, (size_t)500 * 7200, 500, 1000, 2};
  std::vector<std::vector<float>> bufs(8);
  for (int i = 0; i < 8; i++) {
    std::string path = std::string(dir) + names[i] + ".bin";
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) {
      gpdb_set_error(ctx, GPDB_ERR_IO, "Cannot open file: %s", path.c_str());
      return GPDB_ERR_IO;
    }
    bufs[i].resize(sizes[i]);
    size_t got = fread(bufs[i].data(), sizeof(float), sizes[i], f);
    char extra;
    bool more = fread(&extra, 1, 1, f) == 1;
    fclose(f);
    if (got != sizes[i] || more) {
      gpdb_set_error(ctx, GPDB_ERR_IO, "%s: expected %zu float32 values for %d channels", path.c_str(), sizes[i], C);
      return GPDB_ERR_IO;
    }
  }
  return gpdb_set_weights(ctx, bufs[0].data(), bufs[1].data(), bufs[2].data(), bufs[3].data(), bufs[4].data(),
                          bufs[5].data(), bufs[6].data(), bufs[7].data());
}

}  // extern "C"

int gpdb_cloud_reserve(gpdb_ctx *ctx, CloudSet &s, size_t n, int n_clouds) {
  if (n > s.point_cap) {
    cudaStreamSynchronize(ctx->stream);
    cudaFree(s.pts4); s.pts4 = nullptr;
    cudaFree(s.xyz); s.xyz = nullptr;
    cudaFree(s.nrm); s.nrm = nullptr;
    cudaFree(s.cam); s.cam = nullptr;
    cudaFree(s.src); s.src = nullptr;
    s.point_cap = 0;
    const size_t cap = n + n / 8 + 1024;
    CUDA_TRY(cudaMalloc(&s.pts4, sizeof(float4) * cap));
    CUDA_TRY(cudaMalloc(&s.xyz, sizeof(float) * 3 * cap));
    CUDA_TRY(cudaMalloc(&s.nrm, sizeof(double) * 3 * cap));
    CUDA_TRY(cudaMalloc(&s.cam, cap));
    CUDA_TRY(cudaMalloc(&s.src, sizeof(int) * cap));
    s.point_cap = cap;
  }
  if ((size_t)n_clouds + 1 > s.desc_cap) {
    cudaStreamSynchronize(ctx->stream);
    cudaFree(s.desc); s.desc = nullptr;
    cudaFree(s.soff); s.soff = nullptr;
    free(s.off); s.off = nullptr;
    free(s.sel); s.sel = nullptr;
    free(s.pos); s.pos = nullptr;
    free(s.raw_off); s.raw_off = nullptr;
    s.desc_cap = 0;
    const size_t cap = (size_t)n_clouds + 1 + n_clouds / 4;
    CUDA_TRY(cudaMalloc(&s.desc, sizeof(CloudDesc) * cap));
    CUDA_TRY(cudaMalloc(&s.soff, sizeof(int) * cap));
    s.off = (int *)malloc(sizeof(int) * cap);
    s.sel = (int *)malloc(sizeof(int) * cap);
    s.pos = (int *)malloc(sizeof(int) * cap);
    s.raw_off = (int *)malloc(sizeof(int) * cap);
    if (!s.off || !s.sel || !s.pos || !s.raw_off) {
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "cloud store: host allocation failed");
      return GPDB_ERR_CUDA;
    }
    s.desc_cap = cap;
  }
  return GPDB_OK;
}

int gpdb_install_clouds(gpdb_ctx *ctx, CloudSet &s, CloudDesc *desc, const int *off, int B, bool nonunit) {
  int maxk = 0;
  for (int b = 0; b < B; b++) {
    desc[b].off = off[b];
    desc[b].N = off[b + 1] - off[b];
    maxk = std::max(maxk, desc[b].K);
  }
  CUDA_TRY(cudaMemcpyAsync(s.desc, desc, sizeof(CloudDesc) * (size_t)B, cudaMemcpyHostToDevice, ctx->stream));
  memcpy(s.off, off, sizeof(int) * ((size_t)B + 1));
  s.n = B;
  s.maxk = maxk;
  s.has_src = false;  // preprocessing sets it once the source indices of these clouds are in place
  s.n_samples = 0;    // a new cloud drops the sample positions
  s.view = DevCloud{s.pts4, s.xyz, s.nrm, s.cam, s.cell_start, nullptr, off[B]};
  int rc = geo_build_grid_batch(ctx, s);
  if (rc == GPDB_OK && nonunit) rc = pre_nonunit_batch(ctx, s);
  if (rc != GPDB_OK) s.n = 0;
  return rc;
}

// ---- the device-resident entry points (gpdb_*_device): bulk arrays in device memory, sizes and offsets on the host ----

int gpdb_check_device_ptrs(gpdb_ctx *ctx, const char *name,
                           std::initializer_list<std::pair<const char *, const void *>> ptrs) {
  for (const auto &p : ptrs) {
    if (!p.second) continue;
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, p.second);
    if (e != cudaSuccess) cudaGetLastError();
    if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != ctx->device) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: %s is not device memory of device %d", name, p.first, ctx->device);
      return GPDB_ERR_INVALID;
    }
  }
  return GPDB_OK;
}

// ---- the checks shared by the batch entry points and their _device twins ----------------------------------------------

void gpdb_drop_batch(gpdb_ctx *ctx) {
  ctx->many.n = 0;
  ctx->many.has_src = false;
  ctx->many.n_samples = 0;
  sis_forget(ctx);
}

int gpdb_need_batch(gpdb_ctx *ctx, const char *name, const char *hint) {
  if (ctx->many.n) return GPDB_OK;
  gpdb_set_error(ctx, GPDB_ERR_STATE, "%s: no batch of clouds: call %s first", name, hint);
  return GPDB_ERR_STATE;
}

int gpdb_check_offsets(gpdb_ctx *ctx, const char *name, const char *label, const int32_t *off, int B, const char *unit) {
  if (!off || off[0] != 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need %s[%d] starting at 0", name, label, B + 1);
    return GPDB_ERR_INVALID;
  }
  for (int b = 0; b < B; b++)
    if (off[b + 1] < off[b]) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: %s decrease at %s %d", name, label, unit, b);
      return GPDB_ERR_INVALID;
    }
  return GPDB_OK;
}

int gpdb_check_cloud_indices(gpdb_ctx *ctx, const char *name, bool init, const int32_t *off, const int32_t *d_idx,
                             const int *d_off) {
  const CloudSet &s = ctx->many;
  const int B = s.n, n = off[B];
  if (n == 0) return GPDB_OK;
  std::vector<int> lim((size_t)B);
  for (int b = 0; b < B; b++) lim[b] = s.off[b + 1] - s.off[b] + s.positions(b);
  unsigned long long bad;
  const int rc = first_bad(ctx, sizeof(int) * (size_t)B, &bad, [&](unsigned long long *d_bad, void *d_lim) -> int {
    CUDA_TRY(cudaMemcpyAsync(d_lim, lim.data(), sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, ctx->stream));
    return batch_check_samples(ctx, d_idx, n, d_off, B, (const int *)d_lim, d_bad);
  });
  if (rc != GPDB_OK || bad == NO_BAD) return rc;
  const int i = (int)bad;
  int b = 0, v = 0;
  while (off[b + 1] <= i) b++;
  CUDA_TRY(cudaMemcpyAsync(&v, d_idx + i, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  const int nb = s.off[b + 1] - s.off[b];
  if (init)
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: init index %d at position %d outside cloud %d (N = %d)", name, v, i, b, nb);
  else
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: sample index %d at position %d outside cloud %d (N = %d, + %d sample "
                   "positions)", name, v, i, b, nb, s.positions(b));
  return GPDB_ERR_INVALID;
}

// Packs the camera-source matrices of B clouds (cloud b: off[b+1] - off[b] rows of n_cameras[b] entries, concatenated
// in device memory as d_rows, or null: every camera sees every point) into d_cam, one bit per camera
// (batch_pack_cameras), and fills desc[b].K / vp / all_seen. A camera sees a point when its entry is > 0 (eq1 false)
// or == 1 (eq1 true); strict01 refuses entries other than 0 and 1 and names the first.
static int pack_cameras(gpdb_ctx *ctx, const char *name, int B, const int32_t *off, const int32_t *d_rows,
                        const int32_t *n_cameras, const double *view_points, bool eq1, bool strict01, uint8_t *d_cam,
                        CloudDesc *desc) {
  // behind the check word: element offsets of the cam_source blocks [B+1], point offsets [B+1], K_b [B], all_seen [B]
  const size_t bytes = sizeof(long long) * ((size_t)B + 1) + sizeof(int) * (3 * (size_t)B + 1);
  std::vector<unsigned char> h(bytes);
  long long *h_roff = (long long *)h.data();
  int *h_off = (int *)(h_roff + B + 1), *h_k = h_off + B + 1, *h_all = h_k + B;
  h_roff[0] = 0;
  size_t vs = 0;  // running offset into view_points: cloud b's 3 x K_b block follows cloud b-1's
  for (int b = 0; b < B; b++) {
    CloudDesc &D = desc[b];
    memset(&D, 0, sizeof(D));
    D.K = n_cameras[b];
    for (int k = 0; k < D.K; k++)
      for (int r = 0; r < 3; r++) D.vp[k][r] = view_points[vs + 3 * k + r];
    vs += 3 * (size_t)D.K;
    h_roff[b + 1] = h_roff[b] + (long long)(off[b + 1] - off[b]) * D.K;
    h_k[b] = D.K;
    h_all[b] = 1;
  }
  memcpy(h_off, off, sizeof(int) * ((size_t)B + 1));
  unsigned long long e;
  const int rc = first_bad(ctx, bytes, &e, [&](unsigned long long *d_bad, void *d) -> int {
    long long *d_roff = (long long *)d;
    int *d_off = (int *)(d_roff + B + 1), *d_k = d_off + B + 1, *d_all = d_k + B;
    CUDA_TRY(cudaMemcpyAsync(d, h.data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
    const int r = batch_pack_cameras(ctx, d_rows, d_off, d_roff, d_k, B, off[B], eq1, strict01, d_cam, d_all, d_bad);
    if (r == GPDB_OK) CUDA_TRY(cudaMemcpyAsync(h_all, d_all, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
    return r;
  });
  if (rc != GPDB_OK) return rc;
  if (e != NO_BAD) {
    int b = 0;
    while ((unsigned long long)h_roff[b + 1] <= e) b++;
    int32_t v = 0;
    CUDA_TRY(cudaMemcpyAsync(&v, d_rows + e, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const long long r = (long long)e - h_roff[b];
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: cloud %d: cam_source[%d][%d] = %d; without voxelisation entries must be 0 or 1",
                   name, b, (int)(r / n_cameras[b]), (int)(r % n_cameras[b]), v);
    return GPDB_ERR_INVALID;
  }
  for (int b = 0; b < B; b++) desc[b].all_seen = h_all[b];
  return GPDB_OK;
}

// The camera-source matrices of B clouds on the device (*d_rows): the caller's device array as it is (device, or null),
// else the host matrices uploaded into SCR_UPLOAD
static int cam_source_on_device(gpdb_ctx *ctx, int B, const int32_t *off, const int32_t *cam_source,
                                const int32_t *n_cameras, bool device, const int32_t **d_rows) {
  *d_rows = cam_source;
  if (device || !cam_source) return GPDB_OK;
  size_t n = 0;
  for (int b = 0; b < B; b++) n += (size_t)(off[b + 1] - off[b]) * n_cameras[b];
  int32_t *up = (int32_t *)gpdb_scratch(ctx, SCR_UPLOAD, sizeof(int32_t) * n);
  if (!up) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(up, cam_source, sizeof(int32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
  *d_rows = up;
  return GPDB_OK;
}

int gpdb_stage_clouds(gpdb_ctx *ctx, CloudSet &s, const char *name, int B, const int32_t *off, const float *xyz,
                      const double *normals, const int32_t *cam_source, const int32_t *n_cameras,
                      const double *view_points, bool device, CloudDesc *desc) {
  const int N = off[B];
  const cudaMemcpyKind kind = device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  CUDA_TRY(cudaSetDevice(ctx->device));
  int rc = gpdb_cloud_reserve(ctx, s, (size_t)N, B);
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaMemcpyAsync(s.xyz, xyz, sizeof(float) * 3 * (size_t)N, kind, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(s.nrm, normals, sizeof(double) * 3 * (size_t)N, kind, ctx->stream));
  const int32_t *d_rows;
  if ((rc = cam_source_on_device(ctx, B, off, cam_source, n_cameras, device, &d_rows)) != GPDB_OK) return rc;
  unsigned long long bad;
  rc = first_bad(ctx, 0, &bad, [&](unsigned long long *d_bad, void *) {
    return batch_first_nonfinite(ctx, s.xyz, 3 * (long long)N, d_bad);
  });
  if (rc != GPDB_OK) return rc;
  if (bad != NO_BAD) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: point %llu has a non-finite coordinate (run removeNans / gpdb_preprocess first)",
                   name, bad);
    return GPDB_ERR_INVALID;
  }
  return pack_cameras(ctx, name, B, off, d_rows, n_cameras, view_points, false, false, s.cam, desc);
}

// gpdb_set_clouds[_device] into store s after the argument checks (gpdb_set_cloud: `one`, a batch of one); `name` is
// the entry point the errors name
static int set_clouds(gpdb_ctx *ctx, CloudSet &s, const char *name, int32_t B, const int32_t *off, const float *xyz,
                      const double *normals, const int32_t *cam_source, const int32_t *n_cameras,
                      const double *view_points, bool device) {
  std::vector<CloudDesc> desc((size_t)B);
  int rc = gpdb_stage_clouds(ctx, s, name, B, off, xyz, normals, cam_source, n_cameras, view_points, device, desc.data());
  if (rc == GPDB_OK) rc = gpdb_install_clouds(ctx, s, desc.data(), off, B, true);
  return rc == GPDB_OK ? B : rc;
}

// gpdb_preprocess_clouds into store s after the argument checks (gpdb_preprocess: `one`, a batch of one); a failed call
// leaves no cloud in s. device: xyz, normals and cam_source are the caller's device arrays, read in place; else host
// arrays uploaded here. Either way the camera masks are packed on the device.
static int preprocess_clouds(gpdb_ctx *ctx, CloudSet &s, const char *name, int32_t B, const int32_t *roff, const float *xyz,
                             const double *normals, const int32_t *cam_source, const int32_t *n_cameras,
                             const double *view_points, const gpdb_preprocess_params *pp, int32_t *poff,
                             bool device = false) {
  s.n = 0;
  s.has_src = false;
  // the stage boundaries are recorded in the context's events: preprocessing calls on one context are serialised by the
  // stream synchronisation that ends this function, and a call that fails before it reads no event
  cudaEvent_t *ev = ctx->ev;
  const int M = roff[B];
  // ---- camera masks, packed per cloud with its own K_b. A camera sees a point when its entry is exactly 1: the
  // reference's voxelisation keeps only those entries (cloud.cpp:327) and its normal estimation and reverseNormals test
  // == 1 (cloud.cpp:581,611). Without voxelisation the reference keeps the raw values, which its normals read as == 1 and
  // the grasp path as >= 1; one bit cannot hold both, so other values are rejected there.
  std::vector<CloudDesc> desc((size_t)B);
  const float *d_xyz_raw = xyz;
  const double *d_nrm_raw = normals;
  float *xyz_up = nullptr;
  double *nrm_up = nullptr;
  uint8_t *d_cam_raw;
  CUDA_TRY(cudaSetDevice(ctx->device));
  if (!gpdb_carve(ctx, SCR_SIDX, [&](Carve &c) {
        if (!device) {
          if (normals) nrm_up = c.take<double>(3 * (size_t)M);
          xyz_up = c.take<float>(3 * (size_t)M);
        }
        d_cam_raw = c.take<uint8_t>((size_t)M + 16);
      }))
    return GPDB_ERR_CUDA;
  cudaEventRecord(ev[0], ctx->stream);
  if (!device) {  // ---- one upload of the concatenated raw arrays
    CUDA_TRY(cudaMemcpyAsync(xyz_up, xyz, sizeof(float) * 3 * (size_t)M, cudaMemcpyHostToDevice, ctx->stream));
    if (normals) CUDA_TRY(cudaMemcpyAsync(nrm_up, normals, sizeof(double) * 3 * (size_t)M, cudaMemcpyHostToDevice, ctx->stream));
    d_xyz_raw = xyz_up;
    d_nrm_raw = nrm_up;
  }
  const int32_t *d_rows;
  int rc = cam_source_on_device(ctx, B, roff, cam_source, n_cameras, device, &d_rows);
  if (rc == GPDB_OK)
    rc = pack_cameras(ctx, name, B, roff, d_rows, n_cameras, view_points, true, !pp->voxelize, d_cam_raw, desc.data());
  if (rc != GPDB_OK) return rc;
  for (CloudDesc &D : desc) D.all_seen = cam_source ? 0 : 1;  // without a camera-source matrix every camera sees every point
  cudaEventRecord(ev[1], ctx->stream);
  // ---- removeNans + filterWorkspace + voxelizeCloud of every cloud, into the store's arenas
  rc = pre_filter_voxelize_batch(ctx, s, d_xyz_raw, d_cam_raw, d_nrm_raw, M, B, roff, *pp, poff, ev[2]);
  if (rc != GPDB_OK) return rc;
  return gpdb_preprocess_install(ctx, s, desc.data(), B, roff, pp, poff);
}

int gpdb_preprocess_install(gpdb_ctx *ctx, CloudSet &s, CloudDesc *desc, int B, const int32_t *roff,
                            const gpdb_preprocess_params *pp, int32_t *poff, const std::function<int()> &after_normals) {
  cudaEvent_t *ev = ctx->ev;
  cudaEventRecord(ev[3], ctx->stream);
  // ---- install, one grid per cloud
  int rc = gpdb_install_clouds(ctx, s, desc, poff, B, false);
  if (rc != GPDB_OK) return rc;
  cudaEventRecord(ev[4], ctx->stream);
  // ---- calculateNormalsOMP + reverseNormals, every cloud against its own grid; then the per-cloud nonunit flags: zero
  // normals (points no camera sees) and voxel averages of supplied normals are not of unit length. The store holds the
  // clouds by now: a failure drops them again.
  auto tail = [&]() -> int {
    if (pp->estimate_normals) {
      const int r = pre_normals_batch(ctx, s, pp->normals_radius);
      if (r != GPDB_OK) return r;
    }
    if (after_normals) {
      const int r = after_normals();
      if (r != GPDB_OK) return r;
    }
    const int r = pre_nonunit_batch(ctx, s);
    if (r != GPDB_OK) return r;
    cudaEventRecord(ev[5], ctx->stream);
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return GPDB_OK;
  };
  if ((rc = tail()) != GPDB_OK) {
    s.n = 0;
    return rc;
  }
  memset(ctx->pre_ms, 0, sizeof(ctx->pre_ms));
  float t;
  for (int i = 0; i < 5; i++)
    if (cudaEventElapsedTime(&t, ev[i], ev[i + 1]) == cudaSuccess) ctx->pre_ms[i] = t;
  if (cudaEventElapsedTime(&t, ev[0], ev[5]) == cudaSuccess) ctx->pre_ms[5] = t;
  memcpy(s.raw_off, roff, sizeof(int) * ((size_t)B + 1));
  s.has_src = true;
  return B;
}

// the arrays of store s to the host; the camera masks are expanded on the host, each cloud with its own camera count
static int get_clouds(gpdb_ctx *ctx, CloudSet &s, float *xyz_out, double *normals_out, int32_t *cam_source_out,
                      int32_t *src_out) {
  CUDA_TRY(cudaSetDevice(ctx->device));
  const int B = s.n;
  const size_t N = (size_t)s.points();
  if (xyz_out) CUDA_TRY(cudaMemcpyAsync(xyz_out, s.xyz, sizeof(float) * 3 * N, cudaMemcpyDeviceToHost, ctx->stream));
  if (normals_out) CUDA_TRY(cudaMemcpyAsync(normals_out, s.nrm, sizeof(double) * 3 * N, cudaMemcpyDeviceToHost, ctx->stream));
  if (src_out) CUDA_TRY(cudaMemcpyAsync(src_out, s.src, sizeof(int) * N, cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<uint8_t> cam(cam_source_out ? N : 0);
  std::vector<CloudDesc> desc(cam_source_out ? (size_t)B : 0);
  if (cam_source_out) {
    CUDA_TRY(cudaMemcpyAsync(cam.data(), s.cam, N, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(desc.data(), s.desc, sizeof(CloudDesc) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (cam_source_out) {
    size_t o = 0;
    for (int b = 0; b < B; b++)
      for (int i = s.off[b]; i < s.off[b + 1]; i++)
        for (int k = 0; k < desc[b].K; k++) cam_source_out[o++] = (cam[i] >> k) & 1;
  }
  return (int)N;
}

int gpdb_reserve_samples(gpdb_ctx *ctx, CloudSet &s, int n) {
  CUDA_TRY(cudaSetDevice(ctx->device));
  s.n_samples = 0;
  if ((size_t)n > s.samples_cap) {
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    cudaFree(s.samples);
    s.samples = nullptr;
    s.samples_cap = 0;
    s.view.samples = nullptr;
    CUDA_TRY(cudaMalloc(&s.samples, sizeof(double) * 3 * (size_t)n));
    s.samples_cap = (size_t)n;
  }
  s.view.samples = s.samples;  // an install (gpdb_install_clouds) resets the kernels' view of the arena
  return GPDB_OK;
}

// replaces the sample positions of store s by n host positions (3 x n, column-major; n == 0: none)
static int upload_samples(gpdb_ctx *ctx, CloudSet &s, const double *samples, int n) {
  const int rc = gpdb_reserve_samples(ctx, s, n);
  if (rc != GPDB_OK || n == 0) return rc;
  CUDA_TRY(cudaMemcpyAsync(s.samples, samples, sizeof(double) * 3 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  s.n_samples = n;
  return GPDB_OK;
}

int gpdb_check_preprocess_params(gpdb_ctx *ctx, const char *name, const gpdb_preprocess_params *pp, const double *normals) {
  if (!pp->estimate_normals && !normals) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: estimate_normals = 0 needs the caller's normals", name);
    return GPDB_ERR_INVALID;
  }
  if ((pp->voxelize && !(pp->voxel_size > 0.0)) || (pp->estimate_normals && !(pp->normals_radius > 0.0))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: voxel_size and normals_radius must be positive", name);
    return GPDB_ERR_INVALID;
  }
  return GPDB_OK;
}

extern "C" {

int gpdb_set_cloud(gpdb_ctx *ctx, const float *xyz, const double *normals, const int32_t *cam_source, int32_t N,
                   const double *view_points, int32_t K) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (!xyz || !normals || !view_points || N <= 0 || K <= 0 || K > GPDB_MAX_CAMERAS) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_set_cloud: need xyz, normals, view_points, N > 0, 1 <= cameras <= %d",
                   GPDB_MAX_CAMERAS);
    return GPDB_ERR_INVALID;
  }
  ctx->one.n = 0;  // past the argument checks, a failed call leaves no cloud behind
  const int32_t off[2] = {0, N};
  const int rc = set_clouds(ctx, ctx->one, "gpdb_set_cloud", 1, off, xyz, normals, cam_source, &K, view_points, false);
  return rc < 0 ? rc : GPDB_OK;
}

void gpdb_preprocess_params_default(gpdb_preprocess_params *p) {
  memset(p, 0, sizeof(*p));
  const double ws[6] = {-1, 1, -1, 1, -1, 1};
  for (int i = 0; i < 6; i++) p->workspace[i] = ws[i];
  p->voxel_size = 0.003;
  p->normals_radius = 0.03;
  p->voxelize = 1;
  p->estimate_normals = 1;
}

int gpdb_preprocess(gpdb_ctx *ctx, const float *xyz, const double *normals, const int32_t *cam_source, int32_t M,
                    const double *view_points, int32_t K, const gpdb_preprocess_params *pp) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (!xyz || !view_points || !pp || M <= 0 || K <= 0 || K > GPDB_MAX_CAMERAS) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_preprocess: need xyz, view_points, params, n_points > 0, 1 <= cameras <= %d",
                   GPDB_MAX_CAMERAS);
    return GPDB_ERR_INVALID;
  }
  int rc = gpdb_check_preprocess_params(ctx, "gpdb_preprocess", pp, normals);
  if (rc != GPDB_OK) return rc;
  const int32_t roff[2] = {0, M};
  int32_t poff[2] = {0, 0};
  rc = preprocess_clouds(ctx, ctx->one, "gpdb_preprocess", 1, roff, xyz, normals, cam_source, &K, view_points, pp, poff);
  if (rc < 0) return rc;
  if (poff[1] == 0) {  // the filter kept no point: no cloud
    ctx->one.n = 0;
    memset(ctx->pre_ms, 0, sizeof(ctx->pre_ms));
  }
  return poff[1];
}

int gpdb_set_samples(gpdb_ctx *ctx, const double *samples, int32_t n) {
  if (!ctx || n < 0 || (n > 0 && !samples)) return GPDB_ERR_INVALID;
  CloudSet &s = ctx->one;
  if (!s.n && ctx->many.n > 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_set_samples: sample positions address the single cloud; a batch of clouds "
                   "(gpdb_set_clouds) takes cloud-local point indices only");
    return GPDB_ERR_INVALID;
  }
  if (!s.n) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "no point cloud: call gpdb_set_cloud / gpdb_preprocess first");
    return GPDB_ERR_STATE;
  }
  const int rc = upload_samples(ctx, s, samples, n);
  return rc < 0 ? rc : s.points();  // the first sample index that addresses samples[0]
}

}  // extern "C"

// gpdb_set_clouds_samples[_device]: `name` is the entry point the errors name; device: samples is a device array, copied
// device to device into the store's sample arena
static int set_clouds_samples(gpdb_ctx *ctx, const char *name, const int32_t *pos_offsets, const double *samples,
                              bool device) {
  if (!ctx) return GPDB_ERR_INVALID;
  CloudSet &s = ctx->many;
  s.n_samples = 0;  // past this point, a failed call leaves no positions behind
  int rc = gpdb_need_batch(ctx, name, "gpdb_set_clouds / gpdb_preprocess_clouds");
  if (rc != GPDB_OK) return rc;
  const int B = s.n;
  if ((rc = gpdb_check_offsets(ctx, name, "pos_offsets", pos_offsets, B, "cloud")) != GPDB_OK) return rc;
  const int M = pos_offsets[B];
  if (M > 0 && !samples) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null samples_xyz for %d positions", name, M);
    return GPDB_ERR_INVALID;
  }
  if (device && (rc = gpdb_check_device_ptrs(ctx, name, {{"d_samples_xyz", samples}})) != GPDB_OK) return rc;
  memcpy(s.pos, pos_offsets, sizeof(int) * ((size_t)B + 1));
  // each descriptor's first position: one strided copy into the pos field of the B device descriptors
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaMemcpy2DAsync(&s.desc[0].pos, sizeof(CloudDesc), s.pos, sizeof(int), sizeof(int), (size_t)B,
                             cudaMemcpyHostToDevice, ctx->stream));
  if (!device) {
    rc = upload_samples(ctx, s, samples, M);
    return rc < 0 ? rc : M;
  }
  if ((rc = gpdb_reserve_samples(ctx, s, M)) != GPDB_OK) return rc;
  if (M > 0)
    CUDA_TRY(cudaMemcpyAsync(s.samples, samples, sizeof(double) * 3 * (size_t)M, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  s.n_samples = M;
  return M;
}

extern "C" {

int gpdb_set_clouds_samples(gpdb_ctx *ctx, const int32_t *pos_offsets, const double *samples) {
  return set_clouds_samples(ctx, "gpdb_set_clouds_samples", pos_offsets, samples, false);
}

int gpdb_set_clouds_samples_device(gpdb_ctx *ctx, const int32_t *pos_offsets, const double *d_samples_xyz) {
  return set_clouds_samples(ctx, "gpdb_set_clouds_samples_device", pos_offsets, d_samples_xyz, true);
}

int gpdb_get_cloud(gpdb_ctx *ctx, float *xyz_out, double *normals_out, int32_t *cam_source_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (!ctx->one.n) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "no point cloud: call gpdb_set_cloud / gpdb_preprocess first");
    return GPDB_ERR_STATE;
  }
  return get_clouds(ctx, ctx->one, xyz_out, normals_out, cam_source_out, nullptr);
}

int gpdb_get_cloud_source_index(gpdb_ctx *ctx, int32_t *src_out) {
  if (!ctx || !src_out) return GPDB_ERR_INVALID;
  if (!ctx->one.n || !ctx->one.has_src) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "no preprocessed cloud: call gpdb_preprocess first");
    return GPDB_ERR_STATE;
  }
  return get_clouds(ctx, ctx->one, nullptr, nullptr, nullptr, src_out);
}

int gpdb_preprocess_timings(const gpdb_ctx *ctx, double ms_out[6]) {
  if (!ctx || !ms_out) return GPDB_ERR_INVALID;
  for (int i = 0; i < 6; i++) ms_out[i] = ctx->pre_ms[i];
  return GPDB_OK;
}

}  // extern "C"

// ---- pipeline ------------------------------------------------------------------------------------

// Page-locked host memory of one gpdb_result. The device writes the result arrays straight into it (no pageable
// bounce, no second copy), chunk by chunk on the copy stream while the next chunk computes; gpdb_free_result hands it
// back to the context for the next call. Reference-counted: a result may outlive its context.
struct HostArena {
  std::atomic<int> refs{1};        // the owning context + an outstanding result
  std::atomic<bool> in_use{false};
  void *buf[4] = {nullptr, nullptr, nullptr, nullptr};  // 0: per-sample / per-pose arrays, 1: candidate records, 2: images,
  size_t cap[4] = {0, 0, 0, 0};                         // 3: extra (gathered per-pose arrays of gpdb_detect_sharded)
};
static void arena_unref(HostArena *a) {
  if (a->refs.fetch_sub(1) == 1) {
    for (void *b : a->buf)
      if (b) cudaFreeHost(b);
    delete a;
  }
}
// grows buffer `which` to at least `bytes`, keeping the first `keep` bytes (the caller has drained the copies into it)
static bool arena_reserve(HostArena *a, int which, size_t bytes, size_t keep) {
  if (a->cap[which] >= bytes) return true;
  const size_t want = bytes + bytes / 2 + 4096;
  void *nb = nullptr;
  if (cudaHostAlloc(&nb, want, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  if (a->buf[which]) {
    if (keep) memcpy(nb, a->buf[which], keep);
    cudaFreeHost(a->buf[which]);
  }
  a->buf[which] = nb;
  a->cap[which] = want;
  return true;
}

struct PipeState {
  cudaStream_t copy = nullptr;  // D2H of finished chunks + the per-chunk candidate count, concurrent with compute
  cudaStream_t hands = nullptr; // hand search + compaction of the chunks ahead, concurrent with images / LeNet of the current one
  cudaEvent_t ev_compact[2], ev_count[2], ev_scored[2], ev_copied[2], ev_frames, ev_consumed[2], ev_hands_done;
  int *h_count = nullptr;       // pinned [2]
  std::vector<HostArena *> arenas;
  bool ok = false;
};
int gpdb_pipe_create(gpdb_ctx *ctx) {
  PipeState *ps = new PipeState();
  ctx->pipe = ps;
  bool ok = cudaStreamCreateWithFlags(&ps->copy, cudaStreamNonBlocking) == cudaSuccess &&
            cudaStreamCreateWithFlags(&ps->hands, cudaStreamNonBlocking) == cudaSuccess &&
            cudaHostAlloc((void **)&ps->h_count, 2 * sizeof(int), cudaHostAllocDefault) == cudaSuccess;
  cudaEvent_t *evs[12] = {&ps->ev_compact[0], &ps->ev_compact[1], &ps->ev_count[0], &ps->ev_count[1], &ps->ev_scored[0],
                          &ps->ev_scored[1], &ps->ev_copied[0], &ps->ev_copied[1], &ps->ev_frames, &ps->ev_consumed[0],
                          &ps->ev_consumed[1], &ps->ev_hands_done};
  for (cudaEvent_t *e : evs) {
    *e = nullptr;
    ok = ok && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess;
  }
  ps->ok = ok;
  return ok ? GPDB_OK : GPDB_ERR_CUDA;
}
void gpdb_pipe_destroy(gpdb_ctx *ctx) {
  PipeState *ps = ctx->pipe;
  if (!ps) return;
  if (ps->copy) {
    cudaStreamSynchronize(ps->copy);
    cudaStreamDestroy(ps->copy);
  }
  if (ps->hands) {
    cudaStreamSynchronize(ps->hands);
    cudaStreamDestroy(ps->hands);
  }
  cudaEvent_t evs[12] = {ps->ev_compact[0], ps->ev_compact[1], ps->ev_count[0], ps->ev_count[1], ps->ev_scored[0],
                         ps->ev_scored[1], ps->ev_copied[0], ps->ev_copied[1], ps->ev_frames, ps->ev_consumed[0],
                         ps->ev_consumed[1], ps->ev_hands_done};
  for (cudaEvent_t e : evs)
    if (e) cudaEventDestroy(e);
  if (ps->h_count) cudaFreeHost(ps->h_count);
  for (HostArena *a : ps->arenas) arena_unref(a);
  delete ps;
  ctx->pipe = nullptr;
}
// pinned memory that lives and dies with a result (gpdb_detect_sharded: the gathered per-pose arrays of all ranks)
void *gpdb_result_extra(gpdb_result *r, size_t bytes) {
  if (!r || !r->owner_) return nullptr;
  HostArena *a = (HostArena *)r->owner_;
  return arena_reserve(a, 3, bytes, 0) ? a->buf[3] : nullptr;
}

static HostArena *arena_acquire(gpdb_ctx *ctx) {
  PipeState &ps = *ctx->pipe;
  for (HostArena *a : ps.arenas) {
    bool expect = false;
    if (a->in_use.compare_exchange_strong(expect, true)) {
      a->refs.fetch_add(1);
      return a;
    }
  }
  if (ps.arenas.size() >= 8) {  // results that were never freed: do not pin host memory without bound
    gpdb_set_error(ctx, GPDB_ERR_STATE, "8 results of this context are outstanding: release them with gpdb_free_result");
    return nullptr;
  }
  HostArena *a = new HostArena();
  a->in_use = true;
  a->refs = 2;
  ps.arenas.push_back(a);
  return a;
}

int gpdb_check_state(gpdb_ctx *ctx, bool need_cloud, bool need_weights) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (need_cloud && !ctx->one.n) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "no point cloud: call gpdb_set_cloud first");
    return GPDB_ERR_STATE;
  }
  if (need_weights && !ctx->w.set) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "no classifier weights: call gpdb_load_weights_dir / gpdb_set_weights first");
    return GPDB_ERR_STATE;
  }
  CUDA_TRY(cudaSetDevice(ctx->device));
  return GPDB_OK;
}

namespace {

int check_device_errors(gpdb_ctx *ctx) {
  int e[GPDB_NERR];
  CUDA_TRY(cudaMemcpyAsync(e, ctx->d_err, sizeof(e), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (e[0] || e[1] || e[2]) {
    CUDA_TRY(cudaMemsetAsync(ctx->d_err, 0, sizeof(e), ctx->stream));
    gpdb_set_error(ctx, GPDB_ERR_CAPACITY,
                   "neighbourhood exceeded an on-chip tile (frame ball: %d samples, hand-search ball: %d samples, "
                   "image box: %d images): the cloud is denser than the supported %d / %d / %d points",
                   e[0], e[1], e[2], 16384, 131072, 32768);
    return GPDB_ERR_CAPACITY;
  }
  return GPDB_OK;
}

}  // namespace

// The chunked device pipeline behind the detect and hand-search entry points, single cloud, batch and sharded; the request
// (PipeRequest, common.cuh) says where the samples are and where the results go. With device samples and a destination on
// the device nothing but the per-chunk candidate count (and for PIPE_ALL_CALLER the per-cloud offsets) crosses PCIe. A
// selecting call (PIPE_TOP_*) keeps the classified
// candidates of all chunks on the device, sorts the select_k best out there and delivers only them; no per-sample /
// per-pose array is returned.
//
// Stream schedule (H = hand search + compaction of a chunk, I/L/S = images, LeNet, score scatter):
//   compute: F  H0  H1  I0 L0 S0  H2  I1 L1 S1  ...      copy:  frames | n0 | n1 | cand0 flags0 scores0 | n2 | cand1 ...
// The candidate count of chunk i is read back on the copy stream while H(i+1) runs, so the device never waits for the
// host; every chunk is ONE k_images / LeNet launch sized to its candidate count (no tail launches), and the results of
// chunk i go to the pinned arena while chunk i+1 computes.
int gpdb_run_pipeline(gpdb_ctx *ctx, PipeRequest &rq, gpdb_result *out) {
  CloudSet &s = *rq.store;
  const int n = rq.n;
  const bool to_host = rq.dest == PIPE_TO_HOST;  // per-sample / per-pose arrays + all candidate records go to the host
  const bool selecting = rq.dest == PIPE_TOP_HOST || rq.dest == PIPE_TOP_DEVICE;
  memset(out, 0, sizeof(*out));
  PipeState &ps = *ctx->pipe;
  const int P = ctx->hp.P, S = ctx->hp.S, C = ctx->hp.C;
  const size_t isz = (size_t)S * S * C;    // one image in the cv::Mat layout (what the caller receives)
  const size_t psz = (size_t)S * S * 16;   // one image in the device layout (16-byte pixels, see k_images)
  out->n_samples = n;
  out->poses_per_sample = P;
  if (!rq.samples_on_device && !rq.per_cloud)
    for (int i = 0; i < n; i++)
      if (rq.sample_idx[i] < 0 || rq.sample_idx[i] >= s.points() + s.n_samples) {
        gpdb_set_error(ctx, GPDB_ERR_INVALID, "sample index %d at position %d outside the cloud (N = %d, + %d sample positions)",
                       rq.sample_idx[i], i, s.points(), s.n_samples);
        return GPDB_ERR_INVALID;
      }
  const int64_t launches0 = ctx->launches;
  double ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int chunk = ctx->prm.chunk_samples > 0 ? ctx->prm.chunk_samples : 16384;
  const int batch_cap = ctx->prm.batch_size > 0 ? ctx->prm.batch_size : 32768;  // images per k_images / LeNet launch
  const bool keep = rq.classify && ctx->prm.keep_images && to_host;
  const size_t nP = (size_t)n * P;
  const int cmax = std::min(chunk, std::max(n, 1));
  int *d_sidx = rq.samples_on_device && rq.sample_idx ? const_cast<int *>(rq.sample_idx)
                                                      : (int *)gpdb_scratch(ctx, SCR_SIDX, sizeof(int) * (size_t)n);
  double *d_frames = (double *)gpdb_scratch(ctx, SCR_FRAMES, sizeof(double) * 9 * (size_t)n);
  uint8_t *d_valid = (uint8_t *)gpdb_scratch(ctx, SCR_VALID, (size_t)n);
  uint8_t *d_flags = rq.d_flags ? rq.d_flags : (uint8_t *)gpdb_scratch(ctx, SCR_FLAGS, nP);
  float *d_pscores = rq.d_scores ? rq.d_scores : (float *)gpdb_scratch(ctx, SCR_PSCORES, sizeof(float) * nP);
  gpdb_pose *d_poses = (gpdb_pose *)gpdb_scratch(ctx, SCR_POSES, sizeof(gpdb_pose) * (size_t)cmax * P);
  gpdb_pose *d_cand2 = (gpdb_pose *)gpdb_scratch(ctx, SCR_CAND, 2 * sizeof(gpdb_pose) * (size_t)cmax * P);  // double-buffered
  int *d_count = (int *)gpdb_scratch(ctx, SCR_COUNT, 64);
  if (!d_sidx || !d_frames || !d_valid || !d_flags || !d_pscores || !d_poses || !d_cand2 || !d_count) return GPDB_ERR_CUDA;
  gpdb_pose *d_cand[2] = {d_cand2, d_cand2 + (size_t)cmax * P};
  rq.d_flags = d_flags;
  rq.d_scores = d_pscores;

  HostArena *ar = nullptr;
  int rc = GPDB_OK;
  // every exit after this point goes through finish(): drains both streams, clears the device error counters, collects
  // the stage timers and releases the arena on failure, so that a failed call leaves no state behind
  auto finish = [&](int code) -> int {
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ps.hands);
    cudaStreamSynchronize(ps.copy);
    if (code >= 0) {
      int e = check_device_errors(ctx);
      if (e != GPDB_OK) code = e;
    } else {
      cudaMemsetAsync(ctx->d_err, 0, sizeof(int) * GPDB_NERR, ctx->stream);
      cudaStreamSynchronize(ctx->stream);
    }
    st_collect(ctx, ms);
    for (int i = 0; i < 8; i++) ctx->last_ms[i] = ms[i];
    if (code < 0) {
      if (ar) {
        ar->in_use = false;
        arena_unref(ar);
      }
      memset(out, 0, sizeof(*out));
    }
    return code;
  };
#define PIPE_TRY(expr)                                \
  do {                                                \
    if ((rc = (expr)) != GPDB_OK) return finish(rc);  \
  } while (0)
#define PIPE_CUDA(expr)                                                                                           \
  do {                                                                                                            \
    cudaError_t e__ = (expr);                                                                                     \
    if (e__ != cudaSuccess) {                                                                                     \
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__));   \
      return finish(GPDB_ERR_CUDA);                                                                               \
    }                                                                                                             \
  } while (0)

  // host-side layout of the fixed-size arrays inside arena buffer 0
  const size_t off_valid = 0, off_frames = ((size_t)n + 63) / 64 * 64, off_flags = off_frames + sizeof(double) * 9 * (size_t)n,
               off_scores = (off_flags + nP + 63) / 64 * 64, fixed_bytes = off_scores + sizeof(float) * nP + 64;
  if (to_host || rq.dest == PIPE_TOP_HOST) {
    ar = arena_acquire(ctx);
    if (!ar) return GPDB_ERR_STATE;
    const size_t guess = std::max((size_t)1024, nP / 8);  // grown on demand
    if (!arena_reserve(ar, 0, to_host ? fixed_bytes : 64, 0) ||
        !arena_reserve(ar, 1, sizeof(gpdb_pose) * (selecting ? (size_t)std::max(rq.select_k, 1) : guess), 0)) {
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "cudaHostAlloc of the result arena failed");
      return finish(GPDB_ERR_CUDA);
    }
  }
  uint8_t *h_fixed = ar ? (uint8_t *)ar->buf[0] : nullptr;

  ctx->st->spans.clear();
  ctx->st->used = 0;
  cudaEvent_t t_all = gpdb_st_begin(ctx);
  if (n > 0) {
    if (!rq.samples_on_device)
      PIPE_CUDA(cudaMemcpyAsync(d_sidx, rq.sample_idx, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    PIPE_CUDA(cudaMemsetAsync(d_pscores, 0xFF, sizeof(float) * nP, ctx->stream));  // 0xFFFFFFFF = NaN
  }
  cudaEvent_t t0 = gpdb_st_begin(ctx);
  PIPE_TRY(geo_frames(ctx, s, d_sidx, n, d_frames, d_valid));
  gpdb_st_end(ctx, 0, t0);
  // The hand search of the chunks AHEAD runs on its own stream: its CTAs (54 KB, 64 registers) fill what the tensor-core
  // kernels of the current chunk leave idle (conv1: one 162 KB CTA per SM at 42 % issue utilisation).
  // gpdb_set_overlap(ctx, 0) / GPD_B200_OVERLAP=0 put everything on one stream (exclusive stage timers, A/B).
  const bool overlap = ctx->overlap_hands;
  cudaStream_t const main_stream = ctx->stream, hs = overlap ? ps.hands : ctx->stream;
  PIPE_CUDA(cudaEventRecord(ps.ev_frames, main_stream));
  if (overlap) PIPE_CUDA(cudaStreamWaitEvent(hs, ps.ev_frames, 0));
  if (to_host && n > 0) {
    PIPE_CUDA(cudaStreamWaitEvent(ps.copy, ps.ev_frames, 0));
    PIPE_CUDA(cudaMemcpyAsync(h_fixed + off_valid, d_valid, (size_t)n, cudaMemcpyDeviceToHost, ps.copy));
    PIPE_CUDA(cudaMemcpyAsync(h_fixed + off_frames, d_frames, sizeof(double) * 9 * (size_t)n, cudaMemcpyDeviceToHost, ps.copy));
  }
  const int nchunks = (n + chunk - 1) / chunk;
  int total_nc = 0;
  size_t img_host = 0;  // bytes of images already placed in arena buffer 2
  bool cand_busy[2] = {false, false};      // a D2H copy out of d_cand[b] has been issued (ev_copied[b] marks its end)
  bool cand_consumed[2] = {false, false};  // ev_consumed[b] marks the end of the main stream's reads of d_cand[b]
  auto launch_hands = [&](int ci) -> int {
    const int c0 = ci * chunk, nn = std::min(chunk, n - c0), b = ci & 1;
    if (cand_busy[b]) CUDA_TRY(cudaStreamWaitEvent(hs, ps.ev_copied[b], 0));  // chunk ci-2 has left d_cand[b] for the host
    if (overlap && cand_consumed[b]) CUDA_TRY(cudaStreamWaitEvent(hs, ps.ev_consumed[b], 0));  // ... and images / scatter read it
    ctx->stream = hs;  // the launchers (and the stage timers) use the context's current stream
    cudaEvent_t t1 = gpdb_st_begin(ctx);
    int r = geo_hands(ctx, s, d_sidx + c0, nn, c0 + rq.slot_base, d_frames + 9 * (size_t)c0, d_valid + c0, d_poses,
                      d_flags + (size_t)c0 * P);
    if (r == GPDB_OK) r = geo_compact(ctx, d_poses, d_flags + (size_t)c0 * P, nn * P, d_cand[b], d_count + b);
    if (r == GPDB_OK) gpdb_st_end(ctx, 1, t1);
    ctx->stream = main_stream;
    if (r != GPDB_OK) return r;
    CUDA_TRY(cudaEventRecord(ps.ev_compact[b], hs));
    CUDA_TRY(cudaStreamWaitEvent(ps.copy, ps.ev_compact[b], 0));
    CUDA_TRY(cudaMemcpyAsync(ps.h_count + b, d_count + b, sizeof(int), cudaMemcpyDeviceToHost, ps.copy));
    CUDA_TRY(cudaEventRecord(ps.ev_count[b], ps.copy));
    return GPDB_OK;
  };
  if (nchunks > 0) PIPE_TRY(launch_hands(0));
  for (int ci = 0; ci < nchunks; ci++) {
    const int c0 = ci * chunk, nn = std::min(chunk, n - c0), b = ci & 1;
    if (ci + 1 < nchunks) PIPE_TRY(launch_hands(ci + 1));  // queued BEHIND which the host now waits for chunk ci's count
    PIPE_CUDA(cudaEventSynchronize(ps.ev_count[b]));
    const int nc = ps.h_count[b];
    if (overlap) PIPE_CUDA(cudaStreamWaitEvent(main_stream, ps.ev_compact[b], 0));  // d_cand[b], flags of chunk ci are ready
    total_nc += nc;
    uint8_t *d_img = nullptr;  // keep_images: the chunk's images in the cv::Mat layout
    if (rq.classify && nc > 0) {
      float *d_scores = (float *)gpdb_scratch(ctx, SCR_SCORES, sizeof(float) * (size_t)nc);
      const int ib = std::min(nc, batch_cap);
      uint8_t *d_p16 = (uint8_t *)gpdb_scratch(ctx, SCR_P16, psz * (size_t)ib);
      if (keep) d_img = (uint8_t *)gpdb_scratch(ctx, SCR_HWC, isz * (size_t)nc);
      if (!d_scores || !d_p16 || (keep && !d_img)) return finish(GPDB_ERR_CUDA);
      if (keep && ci > 0) PIPE_CUDA(cudaStreamWaitEvent(ctx->stream, ps.ev_copied[b ^ 1], 0));  // d_img is being read
      for (int b0 = 0; b0 < nc; b0 += batch_cap) {
        const int bn = std::min(batch_cap, nc - b0);
        cudaEvent_t t2 = gpdb_st_begin(ctx);
        PIPE_TRY(geo_images(ctx, s, d_cand[b] + b0, bn, d_p16));
        if (keep) PIPE_TRY(geo_p16_to_hwc(ctx, d_p16, bn, d_img + isz * (size_t)b0));
        gpdb_st_end(ctx, 2, t2);
        cudaEvent_t t3 = gpdb_st_begin(ctx);
        PIPE_TRY(lenet_forward(ctx, d_p16, bn, d_scores + b0, nullptr));
        gpdb_st_end(ctx, 3, t3);
      }
      PIPE_TRY(geo_scatter_scores(ctx, d_cand[b], d_scores, nc, c0 + rq.slot_base, P, d_pscores + (size_t)c0 * P, d_cand[b]));
      if (keep) {
        PIPE_CUDA(cudaStreamSynchronize(ps.copy));  // growing moves the buffer: earlier image copies must have landed
        if (!arena_reserve(ar, 2, img_host + isz * (size_t)nc, img_host)) {
          gpdb_set_error(ctx, GPDB_ERR_CUDA, "cudaHostAlloc of %zu B for the images failed", img_host + isz * (size_t)nc);
          return finish(GPDB_ERR_CUDA);
        }
      }
    }
    if (nc > 0 && (selecting || rq.dest == PIPE_ALL_DEVICE)) {  // keep the chunk's scored candidates on the device
      if ((size_t)total_nc > ctx->sel_cap) {
        const size_t cap = std::max((size_t)total_nc * 2, (size_t)65536);
        gpdb_pose *grown = nullptr;
        PIPE_CUDA(cudaMalloc(&grown, sizeof(gpdb_pose) * cap));
        if (ctx->d_sel && total_nc > nc)
          cudaMemcpyAsync(grown, ctx->d_sel, sizeof(gpdb_pose) * (size_t)(total_nc - nc), cudaMemcpyDeviceToDevice, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
        cudaFree(ctx->d_sel);
        ctx->d_sel = grown;
        ctx->sel_cap = cap;
      }
      PIPE_CUDA(cudaMemcpyAsync(ctx->d_sel + (total_nc - nc), d_cand[b], sizeof(gpdb_pose) * (size_t)nc, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    if (nc > 0 && rq.dest == PIPE_ALL_CALLER)  // the caller's buffer holds n * P records: no growth, ordered as above
      PIPE_CUDA(cudaMemcpyAsync(rq.d_selected + (total_nc - nc), d_cand[b], sizeof(gpdb_pose) * (size_t)nc,
                                cudaMemcpyDeviceToDevice, ctx->stream));
    if (overlap) {
      PIPE_CUDA(cudaEventRecord(ps.ev_consumed[b], main_stream));
      cand_consumed[b] = true;
    }
    if (to_host) {  // this chunk's results leave for the pinned arena while the next chunk computes
      if (sizeof(gpdb_pose) * (size_t)total_nc > ar->cap[1]) {
        PIPE_CUDA(cudaStreamSynchronize(ps.copy));
        if (!arena_reserve(ar, 1, sizeof(gpdb_pose) * (size_t)total_nc, sizeof(gpdb_pose) * (size_t)(total_nc - nc))) {
          gpdb_set_error(ctx, GPDB_ERR_CUDA, "cudaHostAlloc of the candidate arena failed");
          return finish(GPDB_ERR_CUDA);
        }
      }
      PIPE_CUDA(cudaEventRecord(ps.ev_scored[b], ctx->stream));
      PIPE_CUDA(cudaStreamWaitEvent(ps.copy, ps.ev_scored[b], 0));
      if (nc > 0)
        PIPE_CUDA(cudaMemcpyAsync((gpdb_pose *)ar->buf[1] + (total_nc - nc), d_cand[b], sizeof(gpdb_pose) * (size_t)nc,
                                  cudaMemcpyDeviceToHost, ps.copy));
      PIPE_CUDA(cudaMemcpyAsync(h_fixed + off_flags + (size_t)c0 * P, d_flags + (size_t)c0 * P, (size_t)nn * P,
                                cudaMemcpyDeviceToHost, ps.copy));
      PIPE_CUDA(cudaMemcpyAsync(h_fixed + off_scores + sizeof(float) * (size_t)c0 * P, d_pscores + (size_t)c0 * P,
                                sizeof(float) * (size_t)nn * P, cudaMemcpyDeviceToHost, ps.copy));
      if (keep && d_img) {
        PIPE_CUDA(cudaMemcpyAsync((uint8_t *)ar->buf[2] + img_host, d_img, isz * (size_t)nc,
                                  cudaMemcpyDeviceToHost, ps.copy));
        img_host += isz * (size_t)nc;
      }
      PIPE_CUDA(cudaEventRecord(ps.ev_copied[b], ps.copy));
      cand_busy[b] = true;
    }
  }
  int n_sel = 0;
  if (selecting && rq.per_cloud) {  // the top select_k of every cloud
    gpdb_pose *d_top = nullptr;
    rc = geo_select_batch(ctx, s, ctx->d_sel, total_nc, rq.select_k, &d_top);
    if (rc < 0) return finish(rc);
    n_sel = rc;
    // sample slots are positions in the whole stream on the device: make them cloud-local, as a single-cloud call has them
    PIPE_TRY(batch_local_slots(ctx, d_top, n_sel, s.soff, s.n, rq.dest == PIPE_TOP_DEVICE ? rq.d_selected : d_top));
    if (n_sel > 0 && rq.dest == PIPE_TOP_HOST) {
      PIPE_CUDA(cudaStreamSynchronize(ps.copy));
      if (!arena_reserve(ar, 1, sizeof(gpdb_pose) * (size_t)n_sel, 0)) {
        gpdb_set_error(ctx, GPDB_ERR_CUDA, "cudaHostAlloc of the candidate arena failed");
        return finish(GPDB_ERR_CUDA);
      }
      PIPE_CUDA(cudaMemcpyAsync(ar->buf[1], d_top, sizeof(gpdb_pose) * (size_t)n_sel, cudaMemcpyDeviceToHost, ctx->stream));
    }
  } else if (selecting) {
    n_sel = std::min(rq.select_k, total_nc);
    if (n_sel > 0) {
      gpdb_pose *d_top = (gpdb_pose *)gpdb_scratch(ctx, SCR_POSES, sizeof(gpdb_pose) * (size_t)std::max(n_sel, cmax * P));
      if (!d_top) return finish(GPDB_ERR_CUDA);
      PIPE_TRY(geo_select(ctx, ctx->d_sel, total_nc, n_sel, d_top));
      PIPE_CUDA(cudaMemcpyAsync(ar->buf[1], d_top, sizeof(gpdb_pose) * (size_t)n_sel, cudaMemcpyDeviceToHost, ctx->stream));
    }
  } else if (rq.dest == PIPE_ALL_CALLER) {
    // the per-cloud offsets are found on the stream slots; then the slots are made cloud-local in place
    PIPE_TRY(geo_batch_cand_off(ctx, s, rq.d_selected, total_nc, s.sel));
    PIPE_TRY(batch_local_slots(ctx, rq.d_selected, total_nc, s.soff, s.n, rq.d_selected));
  }
  gpdb_st_end(ctx, 4, t_all);
  rc = finish(total_nc);
  if (rc < 0) return rc;
#undef PIPE_TRY
#undef PIPE_CUDA
  out->n_candidates = selecting ? n_sel : total_nc;
  out->n_total_candidates = total_nc;
  if (ar) {
    out->owner_ = ar;
    out->candidates = (gpdb_pose *)ar->buf[1];
    if (to_host) {
      out->frame_valid = h_fixed + off_valid;
      out->frames = (double *)(h_fixed + off_frames);
      out->pose_flags = h_fixed + off_flags;
      out->pose_scores = (float *)(h_fixed + off_scores);
      if (keep) out->images = (uint8_t *)ar->buf[2];
    }
  }
  out->ms_candidates = ms[0] + ms[1];
  out->ms_images = ms[2];
  out->ms_classify = ms[3];
  out->kernel_launches = ctx->launches - launches0;
  return out->n_candidates;
}

extern "C" {

int gpdb_detect(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n, gpdb_result *out) {
  int rc = gpdb_check_state(ctx, true, true);
  if (rc != GPDB_OK) return rc;
  if (!out || (n > 0 && !sample_idx) || n < 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect: bad arguments");
    return GPDB_ERR_INVALID;
  }
  PipeRequest rq = {.store = &ctx->one, .sample_idx = sample_idx, .n = n, .classify = true, .dest = PIPE_TO_HOST};
  return gpdb_run_pipeline(ctx, rq, out);
}

int gpdb_detect_select(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n, int32_t num_selected, gpdb_result *out) {
  int rc = gpdb_check_state(ctx, true, true);
  if (rc != GPDB_OK) return rc;
  if (!out || (n > 0 && !sample_idx) || n < 0 || num_selected < 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_select: bad arguments");
    return GPDB_ERR_INVALID;
  }
  PipeRequest rq = {.store = &ctx->one, .sample_idx = sample_idx, .n = n, .classify = true, .dest = PIPE_TOP_HOST,
                    .select_k = num_selected};
  return gpdb_run_pipeline(ctx, rq, out);
}

int gpdb_detect_resident(gpdb_ctx *ctx, const int32_t *d_sample_idx, int32_t n, uint8_t *d_flags_out,
                         float *d_scores_out, gpdb_result *stats) {
  int rc = gpdb_check_state(ctx, true, true);
  if (rc != GPDB_OK) return rc;
  if (!stats || n < 0 || (n > 0 && (!d_sample_idx || !d_flags_out || !d_scores_out))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_resident: bad arguments");
    return GPDB_ERR_INVALID;
  }
  PipeRequest rq = {.store = &ctx->one, .sample_idx = d_sample_idx, .n = n, .samples_on_device = true, .classify = true,
                    .d_flags = d_flags_out, .d_scores = d_scores_out, .dest = PIPE_STAY};
  return gpdb_run_pipeline(ctx, rq, stats);
}

}  // extern "C"

// gpdb_set_clouds[_device] and, raw, gpdb_preprocess_clouds[_device]: drop the batch, check the arguments (device: the d_*
// pointers too), then install or preprocess into the batch store
static int clouds_entry(gpdb_ctx *ctx, const char *name, int32_t n_clouds, const int32_t *point_offsets, const float *xyz,
                        const double *normals, const int32_t *cam_source, const int32_t *n_cameras, const double *view_points,
                        const gpdb_preprocess_params *pp, int32_t *processed_offsets_out, bool raw, bool device) {
  if (!ctx) return GPDB_ERR_INVALID;
  gpdb_drop_batch(ctx);
  if (n_clouds <= 0 || !point_offsets || !n_cameras || !xyz || !view_points || point_offsets[0] != 0 ||
      (raw ? !pp || !processed_offsets_out : !normals)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need n_clouds > 0, point_offsets (starting at 0), n_cameras, xyz, %s", name,
                   raw ? "view_points, params, processed_offsets_out" : "normals, view_points");
    return GPDB_ERR_INVALID;
  }
  for (int b = 0; b < n_clouds; b++) {
    if (point_offsets[b + 1] <= point_offsets[b]) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: %s %d has %d points (offsets must increase)", name, raw ? "raw cloud" : "cloud",
                     b, point_offsets[b + 1] - point_offsets[b]);
      return GPDB_ERR_INVALID;
    }
    if (n_cameras[b] <= 0 || n_cameras[b] > GPDB_MAX_CAMERAS) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: cloud %d has %d cameras (1 <= cameras <= %d)", name, b, n_cameras[b],
                     GPDB_MAX_CAMERAS);
      return GPDB_ERR_INVALID;
    }
  }
  int rc = raw ? gpdb_check_preprocess_params(ctx, name, pp, normals) : GPDB_OK;
  if (rc == GPDB_OK && device)
    rc = gpdb_check_device_ptrs(ctx, name, {{"d_xyz", xyz}, {"d_normals", normals}, {"d_cam_source", cam_source}});
  if (rc != GPDB_OK) return rc;
  CloudSet &s = ctx->many;
  if (raw)
    return preprocess_clouds(ctx, s, name, n_clouds, point_offsets, xyz, normals, cam_source, n_cameras, view_points, pp,
                             processed_offsets_out, device);
  return set_clouds(ctx, s, name, n_clouds, point_offsets, xyz, normals, cam_source, n_cameras, view_points, device);
}

extern "C" {

int gpdb_set_clouds(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *xyz, const double *normals,
                    const int32_t *cam_source, const int32_t *n_cameras, const double *view_points) {
  return clouds_entry(ctx, "gpdb_set_clouds", n_clouds, point_offsets, xyz, normals, cam_source, n_cameras, view_points,
                      nullptr, nullptr, false, false);
}

int gpdb_set_clouds_device(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *d_xyz,
                           const double *d_normals, const int32_t *d_cam_source, const int32_t *n_cameras,
                           const double *view_points) {
  return clouds_entry(ctx, "gpdb_set_clouds_device", n_clouds, point_offsets, d_xyz, d_normals, d_cam_source, n_cameras,
                      view_points, nullptr, nullptr, false, true);
}

int gpdb_preprocess_clouds(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *xyz,
                           const double *normals, const int32_t *cam_source, const int32_t *n_cameras,
                           const double *view_points, const gpdb_preprocess_params *pp, int32_t *processed_offsets_out) {
  return clouds_entry(ctx, "gpdb_preprocess_clouds", n_clouds, point_offsets, xyz, normals, cam_source, n_cameras,
                      view_points, pp, processed_offsets_out, true, false);
}

int gpdb_preprocess_clouds_device(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *d_xyz,
                                  const double *d_normals, const int32_t *d_cam_source, const int32_t *n_cameras,
                                  const double *view_points, const gpdb_preprocess_params *pp,
                                  int32_t *processed_offsets_out) {
  return clouds_entry(ctx, "gpdb_preprocess_clouds_device", n_clouds, point_offsets, d_xyz, d_normals, d_cam_source,
                      n_cameras, view_points, pp, processed_offsets_out, true, true);
}

int gpdb_get_clouds(gpdb_ctx *ctx, float *xyz_out, double *normals_out, int32_t *cam_source_out, int32_t *src_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  const int rc = gpdb_need_batch(ctx, "gpdb_get_clouds", "gpdb_set_clouds / gpdb_preprocess_clouds");
  if (rc != GPDB_OK) return rc;
  if (src_out && !ctx->many.has_src) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "gpdb_get_clouds: source indices exist after gpdb_preprocess_clouds only");
    return GPDB_ERR_STATE;
  }
  return get_clouds(ctx, ctx->many, xyz_out, normals_out, cam_source_out, src_out);
}

}  // extern "C"

namespace {

// gpdb_detect_batch / gpdb_detect_batch_select / gpdb_hand_search_batch: checks the CSR sample lists against the installed
// batch and runs them as ONE sample stream through the chunk pipeline (chunks span cloud boundaries); the records come back
// with cloud-local sample slots, grouped by cloud (offsets_out). Only the classifying calls (with_images_and_scores) need
// weights. The sample lists are checked on the device; host lists are uploaded first. device (gpdb_*_batch*_device):
// sample_idx and sel_out are device arrays and the records stay there: the selection (select_k >= 0), or every record
// (select_k < 0, PIPE_ALL_CALLER) with the dense flags / scores in the caller's d_flags / d_scores when those are
// given. sel_name names sel_out in the messages.
int run_batch(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *sample_idx, gpdb_result *out, int32_t *offsets_out,
              bool with_images_and_scores, int select_k, const char *name, bool device = false, gpdb_pose *sel_out = nullptr,
              const char *sel_name = "d_selected_out", uint8_t *d_flags = nullptr, float *d_scores = nullptr) {
  int rc = gpdb_check_state(ctx, false, with_images_and_scores);
  if (rc != GPDB_OK) return rc;
  CloudSet &s = ctx->many;
  if ((rc = gpdb_need_batch(ctx, name, "gpdb_set_clouds")) != GPDB_OK) return rc;
  const int B = s.n;
  if (!out || !sample_offsets || sample_offsets[0] != 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need out and sample_offsets[%d] starting at 0", name, B + 1);
    return GPDB_ERR_INVALID;
  }
  if ((rc = gpdb_check_offsets(ctx, name, "sample_offsets", sample_offsets, B, "cloud")) != GPDB_OK) return rc;
  const int n = sample_offsets[B];
  if (n > 0 && !sample_idx) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null sample_idx", name);
    return GPDB_ERR_INVALID;
  }
  if (device) {
    if (n > 0 && select_k != 0 && !sel_out) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null %s", name, sel_name);
      return GPDB_ERR_INVALID;
    }
    if ((rc = gpdb_check_device_ptrs(ctx, name, {{"d_sample_idx", sample_idx}, {sel_name, sel_out}, {"d_flags_out", d_flags},
                                                 {"d_scores_out", d_scores}})) != GPDB_OK)
      return rc;
  } else if (n > 0) {  // host lists go through SCR_SIDX, where the pipeline reads them
    int *d_sidx = (int *)gpdb_scratch(ctx, SCR_SIDX, sizeof(int) * (size_t)n);
    if (!d_sidx) return GPDB_ERR_CUDA;
    CUDA_TRY(cudaMemcpyAsync(d_sidx, sample_idx, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    sample_idx = d_sidx;
  }
  CUDA_TRY(cudaMemcpyAsync(s.soff, sample_offsets, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = gpdb_check_cloud_indices(ctx, name, false, sample_offsets, sample_idx, s.soff)) != GPDB_OK) return rc;
  PipeRequest rq = {.store = &s, .sample_idx = sample_idx, .n = n, .samples_on_device = true, .per_cloud = true,
                    .classify = with_images_and_scores, .d_flags = d_flags, .d_scores = d_scores,
                    .dest = select_k < 0 ? (device ? PIPE_ALL_CALLER : PIPE_TO_HOST) : device ? PIPE_TOP_DEVICE : PIPE_TOP_HOST,
                    .select_k = select_k, .d_selected = sel_out};
  rc = gpdb_run_pipeline(ctx, rq, out);
  if (rc < 0) return rc;
  if (rq.dest != PIPE_TO_HOST) {  // the pipeline has made the records' sample slots cloud-local
    memcpy(offsets_out, s.sel, sizeof(int) * ((size_t)B + 1));
  } else {  // sample slots are positions in the whole stream on the device: make them cloud-local, as a single-cloud call has them
    int b = 0;
    offsets_out[0] = 0;
    for (int j = 0; j < out->n_candidates; j++) {
      while (out->candidates[j].sample_slot >= sample_offsets[b + 1]) offsets_out[++b] = j;
      out->candidates[j].sample_slot -= sample_offsets[b];
    }
    while (b < B) offsets_out[++b] = out->n_candidates;
  }
  return rc;
}

}  // namespace

extern "C" {

int gpdb_detect_batch(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *sample_idx, gpdb_result *out,
                      int32_t *cand_offsets_out) {
  if (ctx && !cand_offsets_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_batch: null cand_offsets_out");
    return GPDB_ERR_INVALID;
  }
  return run_batch(ctx, sample_offsets, sample_idx, out, cand_offsets_out, true, -1, "gpdb_detect_batch");
}

int gpdb_hand_search_batch(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *sample_idx, gpdb_result *out,
                           int32_t *cand_offsets_out) {
  if (ctx && !cand_offsets_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_hand_search_batch: null cand_offsets_out");
    return GPDB_ERR_INVALID;
  }
  return run_batch(ctx, sample_offsets, sample_idx, out, cand_offsets_out, false, -1, "gpdb_hand_search_batch");
}

int gpdb_detect_batch_select(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *sample_idx, int32_t num_selected,
                             gpdb_result *out, int32_t *sel_offsets_out) {
  if (ctx && (!sel_offsets_out || num_selected < 0)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_batch_select: need sel_offsets_out and num_selected >= 0");
    return GPDB_ERR_INVALID;
  }
  return run_batch(ctx, sample_offsets, sample_idx, out, sel_offsets_out, true, num_selected, "gpdb_detect_batch_select");
}

int gpdb_detect_batch_select_device(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *d_sample_idx,
                                    int32_t num_selected, gpdb_pose *d_selected_out, int32_t *sel_offsets_out,
                                    gpdb_result *stats) {
  if (ctx && (!sel_offsets_out || num_selected < 0)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_batch_select_device: need sel_offsets_out and num_selected >= 0");
    return GPDB_ERR_INVALID;
  }
  return run_batch(ctx, sample_offsets, d_sample_idx, stats, sel_offsets_out, true, num_selected,
                   "gpdb_detect_batch_select_device", true, d_selected_out);
}

int gpdb_hand_search_batch_device(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *d_sample_idx,
                                  uint8_t *d_flags_out, gpdb_pose *d_hands_out, int32_t *cand_offsets_out, gpdb_result *stats) {
  if (ctx && !cand_offsets_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_hand_search_batch_device: null cand_offsets_out");
    return GPDB_ERR_INVALID;
  }
  return run_batch(ctx, sample_offsets, d_sample_idx, stats, cand_offsets_out, false, -1, "gpdb_hand_search_batch_device",
                   true, d_hands_out, "d_hands_out", d_flags_out);
}

int gpdb_detect_batch_device(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *d_sample_idx, uint8_t *d_flags_out,
                             float *d_scores_out, gpdb_pose *d_candidates_out, int32_t *cand_offsets_out, gpdb_result *stats) {
  if (ctx && !cand_offsets_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_batch_device: null cand_offsets_out");
    return GPDB_ERR_INVALID;
  }
  return run_batch(ctx, sample_offsets, d_sample_idx, stats, cand_offsets_out, true, -1, "gpdb_detect_batch_device", true,
                   d_candidates_out, "d_candidates_out", d_flags_out, d_scores_out);
}

// ImageGenerator::createImages for given hands of the installed batch. The image kernels find a record's cloud from its
// sample slot through the store's soff (CloudSel<true>); here soff holds the hand offsets and every hand is copied into
// the candidate scratch with its position in d_hands as its slot (batch_image_hands), so hand j is imaged against the cloud
// whose group holds it. That slot is the only record field the image kernels index memory with; sample, frame and box only
// feed arithmetic, and sample_index seeds the shadow draws as in gpdb_detect_batch. Every batch call uploads its own
// offsets to soff before it reads them, so borrowing soff here leaves nothing behind. A batch of one runs the one-cloud
// kernels, as gpdb_detect_batch does.
int gpdb_images_batch_device(gpdb_ctx *ctx, const int32_t *hand_offsets, const gpdb_pose *d_hands, uint8_t *d_images_out) {
  const char *name = "gpdb_images_batch_device";
  int rc = gpdb_check_state(ctx, false, false);
  if (rc != GPDB_OK) return rc;
  CloudSet &s = ctx->many;
  if ((rc = gpdb_need_batch(ctx, name, "gpdb_set_clouds")) != GPDB_OK) return rc;
  const int B = s.n;
  if ((rc = gpdb_check_offsets(ctx, name, "hand_offsets", hand_offsets, B, "cloud")) != GPDB_OK) return rc;
  const int n = hand_offsets[B];
  if (n > 0 && (!d_hands || !d_images_out)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null d_hands or d_images_out", name);
    return GPDB_ERR_INVALID;
  }
  if ((rc = gpdb_check_device_ptrs(ctx, name, {{"d_hands", d_hands}, {"d_images_out", d_images_out}})) != GPDB_OK) return rc;
  if (n == 0) return 0;
  CUDA_TRY(cudaMemcpyAsync(s.soff, hand_offsets, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  const size_t isz = (size_t)ctx->hp.S * ctx->hp.S * ctx->hp.C, psz = (size_t)ctx->hp.S * ctx->hp.S * 16;
  const int batch = ctx->prm.batch_size > 0 ? ctx->prm.batch_size : 8192;
  for (int b0 = 0; b0 < n; b0 += batch) {
    const int bn = std::min(batch, n - b0);
    gpdb_pose *d_cand = (gpdb_pose *)gpdb_scratch(ctx, SCR_CAND, sizeof(gpdb_pose) * (size_t)bn);
    uint8_t *d_p16 = (uint8_t *)gpdb_scratch(ctx, SCR_P16, psz * (size_t)bn);
    if (!d_cand || !d_p16) return GPDB_ERR_CUDA;
    if ((rc = batch_image_hands(ctx, d_hands + b0, bn, b0, d_cand)) != GPDB_OK) return rc;
    if ((rc = geo_images(ctx, s, d_cand, bn, d_p16)) != GPDB_OK) return rc;
    if ((rc = geo_p16_to_hwc(ctx, d_p16, bn, d_images_out + isz * (size_t)b0)) != GPDB_OK) return rc;
  }
  if ((rc = check_device_errors(ctx)) != GPDB_OK) return rc;  // drains the stream
  return n;
}

int gpdb_set_overlap(gpdb_ctx *ctx, int32_t enable) {
  if (!ctx) return GPDB_ERR_INVALID;
  ctx->overlap_hands = enable != 0;
  return GPDB_OK;
}

int gpdb_set_stream(gpdb_ctx *ctx, void *cuda_stream) {
  if (!ctx) return GPDB_ERR_INVALID;
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  ctx->stream = (cudaStream_t)cuda_stream;
  ctx->own_stream = false;
  return GPDB_OK;
}

int gpdb_hand_search(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n, gpdb_result *out) {
  int rc = gpdb_check_state(ctx, true, false);
  if (rc != GPDB_OK) return rc;
  if (!out || (n > 0 && !sample_idx) || n < 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_hand_search: bad arguments");
    return GPDB_ERR_INVALID;
  }
  PipeRequest rq = {.store = &ctx->one, .sample_idx = sample_idx, .n = n, .classify = false, .dest = PIPE_TO_HOST};
  return gpdb_run_pipeline(ctx, rq, out);
}

int gpdb_frames(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n, double *frames_out, uint8_t *valid_out) {
  int rc = gpdb_check_state(ctx, true, false);
  if (rc != GPDB_OK) return rc;
  if (n < 0 || (n > 0 && (!sample_idx || !frames_out || !valid_out))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_frames: bad arguments");
    return GPDB_ERR_INVALID;
  }
  if (n == 0) return 0;
  for (int i = 0; i < n; i++)
    if (sample_idx[i] < 0 || sample_idx[i] >= ctx->one.points()) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "sample index %d outside the cloud (N = %d)", sample_idx[i], ctx->one.points());
      return GPDB_ERR_INVALID;
    }
  int *d_sidx = (int *)gpdb_scratch(ctx, SCR_SIDX, sizeof(int) * (size_t)n);
  double *d_frames = (double *)gpdb_scratch(ctx, SCR_FRAMES, sizeof(double) * 9 * (size_t)n);
  uint8_t *d_valid = (uint8_t *)gpdb_scratch(ctx, SCR_VALID, (size_t)n);
  if (!d_sidx || !d_frames || !d_valid) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(d_sidx, sample_idx, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = geo_frames(ctx, ctx->one, d_sidx, n, d_frames, d_valid)) != GPDB_OK) return rc;
  CUDA_TRY(cudaMemcpyAsync(frames_out, d_frames, sizeof(double) * 9 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(valid_out, d_valid, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  if ((rc = check_device_errors(ctx)) != GPDB_OK) return rc;
  return n;
}

int gpdb_images(gpdb_ctx *ctx, const gpdb_pose *poses, int32_t n, uint8_t *images_out) {
  int rc = gpdb_check_state(ctx, true, false);
  if (rc != GPDB_OK) return rc;
  if (n < 0 || (n > 0 && (!poses || !images_out))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_images: bad arguments");
    return GPDB_ERR_INVALID;
  }
  const size_t isz = (size_t)ctx->hp.S * ctx->hp.S * ctx->hp.C, psz = (size_t)ctx->hp.S * ctx->hp.S * 16;
  const int batch = 8192;
  for (int b0 = 0; b0 < n; b0 += batch) {
    const int bn = std::min(batch, n - b0);
    gpdb_pose *d_cand = (gpdb_pose *)gpdb_scratch(ctx, SCR_CAND, sizeof(gpdb_pose) * (size_t)bn);
    uint8_t *d_p16 = (uint8_t *)gpdb_scratch(ctx, SCR_P16, psz * (size_t)bn);
    uint8_t *d_img = (uint8_t *)gpdb_scratch(ctx, SCR_HWC, isz * (size_t)bn);
    if (!d_cand || !d_p16 || !d_img) return GPDB_ERR_CUDA;
    CUDA_TRY(cudaMemcpyAsync(d_cand, poses + b0, sizeof(gpdb_pose) * (size_t)bn, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = geo_images(ctx, ctx->one, d_cand, bn, d_p16)) != GPDB_OK) return rc;
    if ((rc = geo_p16_to_hwc(ctx, d_p16, bn, d_img)) != GPDB_OK) return rc;
    CUDA_TRY(cudaMemcpyAsync(images_out + isz * (size_t)b0, d_img, isz * (size_t)bn, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  if ((rc = check_device_errors(ctx)) != GPDB_OK) return rc;
  return n;
}

namespace {

// The classify loop of gpdb_classify and gpdb_debug_lenet_layers: HWC -> P16 and lenet_forward in batches of batch_size.
// scores_out / logits_out may be null; layers (null for gpdb_classify) receives every layer's output at offset b0.
// device (gpdb_classify_device): images and outputs are device arrays; the images are converted in place and LeNet writes
// the outputs directly, with one synchronisation at the end.
int classify_batches(gpdb_ctx *ctx, const uint8_t *images_hwc, int32_t n, float *scores_out, float *logits_out,
                     const LenetLayers *layers, bool device = false) {
  int rc;
  const size_t isz = (size_t)ctx->hp.S * ctx->hp.S * ctx->hp.C, psz = (size_t)ctx->hp.S * ctx->hp.S * 16;
  const int batch = ctx->prm.batch_size > 0 ? ctx->prm.batch_size : 8192;
  if (device) {
    for (int b0 = 0; b0 < n; b0 += batch) {
      const int bn = std::min(batch, n - b0);
      uint8_t *d_p16 = (uint8_t *)gpdb_scratch(ctx, SCR_P16, psz * (size_t)bn);
      if (!d_p16) return GPDB_ERR_CUDA;
      if ((rc = geo_hwc_to_p16(ctx, images_hwc + isz * (size_t)b0, bn, d_p16)) != GPDB_OK) return rc;
      if ((rc = lenet_forward(ctx, d_p16, bn, scores_out + b0, logits_out ? logits_out + 2 * (size_t)b0 : nullptr)) != GPDB_OK)
        return rc;
    }
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return n;
  }
  for (int b0 = 0; b0 < n; b0 += batch) {
    const int bn = std::min(batch, n - b0);
    uint8_t *d_img = (uint8_t *)gpdb_scratch(ctx, SCR_HWC, isz * (size_t)bn);
    uint8_t *d_p16 = (uint8_t *)gpdb_scratch(ctx, SCR_P16, psz * (size_t)bn);
    float *d_scores = (float *)gpdb_scratch(ctx, SCR_SCORES, sizeof(float) * (size_t)bn * 3);
    if (!d_img || !d_p16 || !d_scores) return GPDB_ERR_CUDA;
    float *d_logits = d_scores + bn;
    CUDA_TRY(cudaMemcpyAsync(d_img, images_hwc + isz * (size_t)b0, isz * (size_t)bn, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = geo_hwc_to_p16(ctx, d_img, bn, d_p16)) != GPDB_OK) return rc;  // cv::Mat bytes -> 16-byte pixels
    LenetLayers at = {};
    if (layers)
      at = {layers->pool1 ? layers->pool1 + (size_t)b0 * 20 * 28 * 28 : nullptr,
            layers->pool2 ? layers->pool2 + (size_t)b0 * 7200 : nullptr, layers->ip1 ? layers->ip1 + (size_t)b0 * 500 : nullptr};
    if ((rc = lenet_forward(ctx, d_p16, bn, d_scores, d_logits, layers ? &at : nullptr)) != GPDB_OK) return rc;
    if (scores_out)
      CUDA_TRY(cudaMemcpyAsync(scores_out + b0, d_scores, sizeof(float) * (size_t)bn, cudaMemcpyDeviceToHost, ctx->stream));
    if (logits_out)
      CUDA_TRY(cudaMemcpyAsync(logits_out + 2 * (size_t)b0, d_logits, sizeof(float) * 2 * (size_t)bn,
                               cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  return n;
}

}  // namespace

int gpdb_classify(gpdb_ctx *ctx, const uint8_t *images_hwc, int32_t n, float *scores_out, float *logits_out) {
  int rc = gpdb_check_state(ctx, false, true);
  if (rc != GPDB_OK) return rc;
  if (n < 0 || (n > 0 && (!images_hwc || !scores_out))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_classify: bad arguments");
    return GPDB_ERR_INVALID;
  }
  return classify_batches(ctx, images_hwc, n, scores_out, logits_out, nullptr);
}

int gpdb_classify_device(gpdb_ctx *ctx, const uint8_t *d_images_hwc, int32_t n, float *d_scores_out, float *d_logits_out) {
  const char *name = "gpdb_classify_device";
  int rc = gpdb_check_state(ctx, false, true);
  if (rc != GPDB_OK) return rc;
  if (n < 0 || (n > 0 && (!d_images_hwc || !d_scores_out))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: bad arguments", name);
    return GPDB_ERR_INVALID;
  }
  rc = gpdb_check_device_ptrs(ctx, name, {{"d_images_hwc", d_images_hwc}, {"d_scores_out", d_scores_out},
                                          {"d_logits_out", d_logits_out}});
  if (rc != GPDB_OK) return rc;
  return classify_batches(ctx, d_images_hwc, n, d_scores_out, d_logits_out, nullptr, true);
}

int gpdb_debug_lenet_layers(gpdb_ctx *ctx, const uint8_t *images_hwc, int32_t n, float *pool1_out, double *pool2_out,
                            float *ip1_out, float *logits_out) {
  int rc = gpdb_check_state(ctx, false, true);
  if (rc != GPDB_OK) return rc;
  if (n < 0 || (n > 0 && !images_hwc)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_debug_lenet_layers: bad arguments");
    return GPDB_ERR_INVALID;
  }
  const LenetLayers layers = {pool1_out, pool2_out, ip1_out};
  return classify_batches(ctx, images_hwc, n, nullptr, logits_out, &layers);
}

namespace {

// gpdb_reevaluate[_batch][_device] after their checks: HandSearch::reevaluateHypotheses of the hand_offsets[B] hands,
// group b (hand_offsets[b] .. hand_offsets[b+1]) against cloud b of store s, in one k_label launch. The store is only
// read: a batch borrows its soff for the group offsets, as gpdb_images_batch_device does. device: hands and labels are
// device arrays, labelled in place; else they go through SCR_HANDS / SCR_LABELS.
int label_hands(gpdb_ctx *ctx, const CloudSet &s, const int32_t *hand_offsets, gpdb_pose *hands, int32_t *labels,
                bool device) {
  const int n = hand_offsets[s.n];
  if (n == 0) return 0;
  gpdb_pose *d_h = hands;
  int *d_l = labels;
  if (!device) {
    d_h = (gpdb_pose *)gpdb_scratch(ctx, SCR_HANDS, sizeof(gpdb_pose) * (size_t)n);
    d_l = (int *)gpdb_scratch(ctx, SCR_LABELS, sizeof(int) * (size_t)n);
    if (!d_h || !d_l) return GPDB_ERR_CUDA;
    CUDA_TRY(cudaMemcpyAsync(d_h, hands, sizeof(gpdb_pose) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (s.n > 1)
    CUDA_TRY(cudaMemcpyAsync(s.soff, hand_offsets, sizeof(int) * ((size_t)s.n + 1), cudaMemcpyHostToDevice, ctx->stream));
  int rc;
  if ((rc = geo_label(ctx, s, d_h, n, d_l)) != GPDB_OK) return rc;
  if (!device) {
    CUDA_TRY(cudaMemcpyAsync(hands, d_h, sizeof(gpdb_pose) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(labels, d_l, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return n;
}

int reevaluate_batch(gpdb_ctx *ctx, const char *name, const int32_t *hand_offsets, gpdb_pose *hands, int32_t *labels_out,
                     bool device) {
  int rc = gpdb_check_state(ctx, false, false);
  if (rc != GPDB_OK) return rc;
  if ((rc = gpdb_need_batch(ctx, name, "gpdb_set_clouds / gpdb_preprocess_clouds / gpdb_preprocess_depth")) != GPDB_OK)
    return rc;
  if ((rc = gpdb_check_offsets(ctx, name, "hand_offsets", hand_offsets, ctx->many.n, "cloud")) != GPDB_OK) return rc;
  if (hand_offsets[ctx->many.n] > 0 && (!hands || !labels_out)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null %s or %s", name, device ? "d_hands" : "hands",
                   device ? "d_labels_out" : "labels_out");
    return GPDB_ERR_INVALID;
  }
  if (device && (rc = gpdb_check_device_ptrs(ctx, name, {{"d_hands", hands}, {"d_labels_out", labels_out}})) != GPDB_OK)
    return rc;
  return label_hands(ctx, ctx->many, hand_offsets, hands, labels_out, device);
}

}  // namespace

int gpdb_reevaluate(gpdb_ctx *ctx, gpdb_pose *hands, int32_t n, int32_t *labels_out) {
  int rc = gpdb_check_state(ctx, true, false);
  if (rc != GPDB_OK) return rc;
  if (n < 0 || (n > 0 && (!hands || !labels_out))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_reevaluate: bad arguments");
    return GPDB_ERR_INVALID;
  }
  const int32_t hand_offsets[2] = {0, n};
  return label_hands(ctx, ctx->one, hand_offsets, hands, labels_out, false);
}

int gpdb_reevaluate_batch(gpdb_ctx *ctx, const int32_t *hand_offsets, gpdb_pose *hands, int32_t *labels_out) {
  return reevaluate_batch(ctx, "gpdb_reevaluate_batch", hand_offsets, hands, labels_out, false);
}

int gpdb_reevaluate_batch_device(gpdb_ctx *ctx, const int32_t *hand_offsets, gpdb_pose *d_hands, int32_t *d_labels_out) {
  return reevaluate_batch(ctx, "gpdb_reevaluate_batch_device", hand_offsets, d_hands, d_labels_out, true);
}

}  // extern "C"

int gpdb_cluster_groups(gpdb_ctx *ctx, int G, const int32_t *hand_offsets, const gpdb_pose *hands, int min_inliers,
                        gpdb_pose *clusters_out, int32_t *cluster_offsets_out, bool device) {
  const int n = hand_offsets[G];
  for (int g = 0; g <= G; g++) cluster_offsets_out[g] = 0;
  if (n == 0) return 0;
  CUDA_TRY(cudaSetDevice(ctx->device));
  gpdb_pose *d_dense, *d_out, *d_up = nullptr;  // dense records, compacted records, the uploaded hands
  int *d_goff, *d_gcount;
  uint8_t *d_keep;
  const bool ok = gpdb_carve(ctx, SCR_HANDS, [&](Carve &c) {
                    d_dense = c.take<gpdb_pose>(n); d_out = c.take<gpdb_pose>(n);
                    if (!device) d_up = c.take<gpdb_pose>(n);
                  }) &&
                  gpdb_carve(ctx, SCR_LABELS, [&](Carve &c) {
                    d_goff = c.take<int>((size_t)G + 1); d_gcount = c.take<int>(G); d_keep = c.take<uint8_t>(n);
                  });
  int *d_count = (int *)gpdb_scratch(ctx, SCR_COUNT, 64);
  if (!ok || !d_count) return GPDB_ERR_CUDA;
  const gpdb_pose *d_in = hands;
  if (!device) {
    d_in = d_up;
    CUDA_TRY(cudaMemcpyAsync(d_up, hands, sizeof(gpdb_pose) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  }
  CUDA_TRY(cudaMemcpyAsync(d_goff, hand_offsets, sizeof(int) * ((size_t)G + 1), cudaMemcpyHostToDevice, ctx->stream));
  int rc;
  if ((rc = geo_clusters(ctx, d_in, n, d_goff, G, min_inliers, d_dense, d_keep, d_gcount)) != GPDB_OK) return rc;
  if ((rc = geo_compact(ctx, d_dense, d_keep, n, d_out, d_count + 2)) != GPDB_OK) return rc;  // order of i kept
  // per-group counts -> exclusive scan: the groups' slices of the compacted list
  CUDA_TRY(cudaMemcpyAsync(cluster_offsets_out + 1, d_gcount, sizeof(int) * (size_t)G, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  for (int g = 0; g < G; g++) cluster_offsets_out[g + 1] += cluster_offsets_out[g];
  const int nc = cluster_offsets_out[G];
  if (nc > 0) {
    CUDA_TRY(cudaMemcpyAsync(clusters_out, d_out, sizeof(gpdb_pose) * (size_t)nc, cudaMemcpyDefault, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  return nc;
}

extern "C" {

int gpdb_find_clusters(gpdb_ctx *ctx, const gpdb_pose *hands, int32_t n, int32_t min_inliers, gpdb_pose *clusters_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (n < 0 || (n > 0 && (!hands || !clusters_out))) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_find_clusters: bad arguments");
    return GPDB_ERR_INVALID;
  }
  const int32_t hand_offsets[2] = {0, n};
  int32_t cluster_offsets[2];
  return gpdb_cluster_groups(ctx, 1, hand_offsets, hands, min_inliers, clusters_out, cluster_offsets);
}

}  // extern "C"

// the argument checks of gpdb_find_clusters_batch[_device]
static int check_groups_args(gpdb_ctx *ctx, const char *name, int32_t n_groups, const int32_t *hand_offsets,
                             const gpdb_pose *hands, const gpdb_pose *clusters_out, const int32_t *cluster_offsets_out) {
  if (n_groups < 0 || !hand_offsets || !cluster_offsets_out || hand_offsets[0] != 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need n_groups >= 0, hand_offsets[n_groups + 1] starting at 0 and "
                   "cluster_offsets_out", name);
    return GPDB_ERR_INVALID;
  }
  const int rc = gpdb_check_offsets(ctx, name, "hand_offsets", hand_offsets, n_groups, "group");
  if (rc != GPDB_OK) return rc;
  if (hand_offsets[n_groups] > 0 && (!hands || !clusters_out)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null hands or clusters_out", name);
    return GPDB_ERR_INVALID;
  }
  return GPDB_OK;
}

extern "C" {

int gpdb_find_clusters_batch(gpdb_ctx *ctx, int32_t n_groups, const int32_t *hand_offsets, const gpdb_pose *hands,
                             int32_t min_inliers, gpdb_pose *clusters_out, int32_t *cluster_offsets_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  const int rc = check_groups_args(ctx, "gpdb_find_clusters_batch", n_groups, hand_offsets, hands, clusters_out,
                                   cluster_offsets_out);
  if (rc != GPDB_OK) return rc;
  return gpdb_cluster_groups(ctx, n_groups, hand_offsets, hands, min_inliers, clusters_out, cluster_offsets_out);
}

int gpdb_find_clusters_batch_device(gpdb_ctx *ctx, int32_t n_groups, const int32_t *hand_offsets, const gpdb_pose *d_hands,
                                    int32_t min_inliers, gpdb_pose *d_clusters_out, int32_t *cluster_offsets_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  const char *name = "gpdb_find_clusters_batch_device";
  int rc = check_groups_args(ctx, name, n_groups, hand_offsets, d_hands, d_clusters_out, cluster_offsets_out);
  if (rc == GPDB_OK) rc = gpdb_check_device_ptrs(ctx, name, {{"d_hands", d_hands}, {"d_clusters_out", d_clusters_out}});
  if (rc != GPDB_OK) return rc;
  return gpdb_cluster_groups(ctx, n_groups, hand_offsets, d_hands, min_inliers, d_clusters_out, cluster_offsets_out, true);
}

void gpdb_free_result(gpdb_result *r) {
  if (!r) return;
  if (r->owner_) {  // the arrays live in a pinned arena of the context that produced them: hand it back
    HostArena *a = (HostArena *)r->owner_;
    a->in_use = false;
    arena_unref(a);
  } else {
    free(r->frame_valid);
    free(r->frames);
    free(r->pose_flags);
    free(r->pose_scores);
    free(r->candidates);
    free(r->images);
  }
  memset(r, 0, sizeof(*r));
}

int gpdb_debug_phase_cycles(gpdb_ctx *ctx, int enable, uint64_t cycles_out[32]) {
  if (!ctx) return GPDB_ERR_INVALID;
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  // slots 0..15: phase cycles and image events; 16..31: the path counters of gpdb_debug_path_counts (GPDB_PROF_PATH);
  // 32..47: the shadow sub-phases and their events (GPDB_PROF_SUB), returned as cycles_out[16..31]
  if (ctx->d_prof && cycles_out) {
    CUDA_TRY(cudaMemcpy(cycles_out, ctx->d_prof, sizeof(uint64_t) * 16, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(cycles_out + 16, ctx->d_prof + GPDB_PROF_SUB, sizeof(uint64_t) * 16, cudaMemcpyDeviceToHost));
  }
  if (enable && !ctx->d_prof) CUDA_TRY(cudaMalloc(&ctx->d_prof, sizeof(uint64_t) * GPDB_PROF_SLOTS));
  if (enable) CUDA_TRY(cudaMemset(ctx->d_prof, 0, sizeof(uint64_t) * GPDB_PROF_SLOTS));
  if (!enable && ctx->d_prof) {
    cudaFree(ctx->d_prof);
    ctx->d_prof = nullptr;
  }
  return GPDB_OK;
}

int gpdb_debug_path_counts(gpdb_ctx *ctx, uint64_t counts_out[16]) {
  if (!ctx || !counts_out) return GPDB_ERR_INVALID;
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (ctx->d_prof)
    CUDA_TRY(cudaMemcpy(counts_out, ctx->d_prof + GPDB_PROF_PATH, sizeof(uint64_t) * 16, cudaMemcpyDeviceToHost));
  else
    memset(counts_out, 0, sizeof(uint64_t) * 16);
  return GPDB_OK;
}

int gpdb_last_timings(const gpdb_ctx *ctx, double ms_out[8]) {
  if (!ctx || !ms_out) return GPDB_ERR_INVALID;
  for (int i = 0; i < 8; i++) ms_out[i] = ctx->last_ms[i];
  return GPDB_OK;
}

}  // extern "C"
