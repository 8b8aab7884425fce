// comm.cu — multi-GPU sharding of the path INSIDE the C-ABI (SURVEY.md 8(e)): one context per GPU, the cloud broadcast
// with ncclBroadcast, every rank runs the chunk pipeline on its contiguous slice of the sample indices, ONE ncclAllGather of
// fixed-stride {score f32, flags u8} slots. The reference's counterpart is the OpenMP loop over samples
// (hand_search.cpp:168-182, image_generator.cpp:83-89, eigen_classifier.cpp:67-76): samples are independent.
//
// NCCL is bound at run time with dlopen: the copy already loaded in the process (PyTorch ships its own libnccl.so.2) is
// reused, otherwise the system library is opened; libgpd_b200.so itself has no link-time dependency on NCCL, so the
// single-GPU boundary loads on machines without it.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace {

struct NcclApi {
  void *handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int *) = nullptr;
};
NcclApi g_nccl;

const char *load_nccl_once() {
  void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);  // the process's own copy first (PyTorch's)
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return "libnccl.so.2 not found (dlopen)";
  NcclApi a;
  a.handle = h;
#define SYM(field, name)                                          \
  a.field = reinterpret_cast<decltype(a.field)>(dlsym(h, name));  \
  if (!a.field) return "libnccl.so.2 lacks " name;
  SYM(GetUniqueId, "ncclGetUniqueId")
  SYM(CommInitRank, "ncclCommInitRank")
  SYM(CommDestroy, "ncclCommDestroy")
  SYM(Broadcast, "ncclBroadcast")
  SYM(AllGather, "ncclAllGather")
  SYM(GroupStart, "ncclGroupStart")
  SYM(GroupEnd, "ncclGroupEnd")
  SYM(GetErrorString, "ncclGetErrorString")
  SYM(GetVersion, "ncclGetVersion")
#undef SYM
  g_nccl = a;
  return nullptr;
}
// returns nullptr on success, else the reason. Thread-safe (one context per host thread in the multi-GPU shim): the
// function-local static is initialised exactly once, and g_nccl is complete before any caller sees the result.
const char *load_nccl() {
  static const char *const why = load_nccl_once();
  return why;
}

}  // namespace

struct CommState {
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1;
  int32_t count = 0;  // this rank's candidate count of the last sharded call (staged into its slot)
};

#define NCCL_TRY(expr)                                                                                              \
  do {                                                                                                              \
    ncclResult_t r__ = (expr);                                                                                      \
    if (r__ != ncclSuccess) {                                                                                       \
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "%s:%d %s -> NCCL: %s", __FILE__, __LINE__, #expr, g_nccl.GetErrorString(r__)); \
      return GPDB_ERR_CUDA;                                                                                         \
    }                                                                                                               \
  } while (0)

static int need_comm(gpdb_ctx *ctx) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (!ctx->comm || !ctx->comm->comm) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "no communicator: call gpdb_comm_init first");
    return GPDB_ERR_STATE;
  }
  return GPDB_OK;
}

extern "C" {

int gpdb_comm_unique_id(char id_out[GPDB_COMM_ID_BYTES]) {
  static_assert(sizeof(ncclUniqueId) == GPDB_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  if (!id_out) return GPDB_ERR_INVALID;
  if (const char *why = load_nccl()) {
    gpdb_set_error(nullptr, GPDB_ERR_STATE, "%s", why);
    return GPDB_ERR_STATE;
  }
  ncclUniqueId id;
  if (g_nccl.GetUniqueId(&id) != ncclSuccess) {
    gpdb_set_error(nullptr, GPDB_ERR_CUDA, "ncclGetUniqueId failed");
    return GPDB_ERR_CUDA;
  }
  memcpy(id_out, &id, sizeof(id));
  return GPDB_OK;
}

int gpdb_comm_init(gpdb_ctx *ctx, const char id[GPDB_COMM_ID_BYTES], int32_t rank, int32_t nranks) {
  if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_comm_init: need id, 0 <= rank < nranks");
    return GPDB_ERR_INVALID;
  }
  if (const char *why = load_nccl()) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "%s", why);
    return GPDB_ERR_STATE;
  }
  CUDA_TRY(cudaSetDevice(ctx->device));
  gpdb_comm_destroy(ctx);
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  CommState *cs = new CommState();
  cs->rank = rank;
  cs->nranks = nranks;
  ncclResult_t r = g_nccl.CommInitRank(&cs->comm, nranks, uid, rank);
  if (r != ncclSuccess) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "ncclCommInitRank(rank %d of %d) -> %s", rank, nranks, g_nccl.GetErrorString(r));
    delete cs;
    return GPDB_ERR_CUDA;
  }
  ctx->comm = cs;
  return GPDB_OK;
}

int gpdb_comm_destroy(gpdb_ctx *ctx) {
  if (!ctx || !ctx->comm) return GPDB_OK;
  if (ctx->comm->comm && g_nccl.CommDestroy) {
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    g_nccl.CommDestroy(ctx->comm->comm);
  }
  delete ctx->comm;
  ctx->comm = nullptr;
  return GPDB_OK;
}

void gpdb_shard_bounds(int32_t n, int32_t rank, int32_t nranks, int32_t *lo, int32_t *hi, int32_t *slot_samples) {
  if (nranks < 1 || rank < 0 || rank >= nranks || n < 0) {  // malformed request: an empty slice
    if (lo) *lo = 0;
    if (hi) *hi = 0;
    if (slot_samples) *slot_samples = 0;
    return;
  }
  const int64_t a = ((int64_t)rank * n) / nranks, b = ((int64_t)(rank + 1) * n) / nranks;
  if (lo) *lo = (int32_t)a;
  if (hi) *hi = (int32_t)b;
  if (slot_samples) {
    int64_t m = 0;
    for (int r = 0; r < nranks; r++) m = std::max(m, ((int64_t)(r + 1) * n) / nranks - ((int64_t)r * n) / nranks);
    *slot_samples = (int32_t)m;
  }
}

// slot = [scores f32 np][flags u8 np, padded to 16 B][int32 candidate count of the rank, 12 B pad]
int64_t gpdb_slot_bytes(int32_t slot_samples, int32_t P) {
  const int64_t np = (int64_t)slot_samples * P;
  return np * 4 + (np + 15) / 16 * 16 + 16;
}

int gpdb_set_cloud_bcast(gpdb_ctx *ctx, int32_t root, const float *xyz, const double *normals, const int32_t *cam_source,
                         int32_t N, const double *view_points, int32_t K) {
  int rc = need_comm(ctx);
  if (rc != GPDB_OK) return rc;
  CommState &cs = *ctx->comm;
  if (root < 0 || root >= cs.nranks) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_set_cloud_bcast: root %d outside 0..%d", root, cs.nranks - 1);
    return GPDB_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(ctx->device));
  const bool is_root = cs.rank == root;
  // header: N, K, validity of the root's arguments, the view points
  double hdr[4 + 3 * GPDB_MAX_CAMERAS] = {0};
  double *d_hdr = (double *)gpdb_scratch(ctx, SCR_WORK_A, sizeof(hdr));
  if (!d_hdr) return GPDB_ERR_CUDA;
  CloudSet &s = ctx->one;
  s.n = 0;
  CloudDesc desc;
  if (is_root) {
    // the root stages its cloud in its own store, checked and packed as gpdb_set_cloud does it; a failure is reported
    // through the header too: every rank waits in its broadcast
    const int32_t off[2] = {0, N};
    const bool ok = xyz && normals && view_points && N > 0 && K > 0 && K <= GPDB_MAX_CAMERAS &&
                    gpdb_stage_clouds(ctx, s, "gpdb_set_cloud_bcast", 1, off, xyz, normals, cam_source, &K, view_points,
                                      false, &desc) == GPDB_OK;
    hdr[0] = ok ? N : -1;
    hdr[1] = K;
    if (ok) {
      hdr[2] = desc.all_seen;
      memcpy(hdr + 4, view_points, sizeof(double) * 3 * (size_t)K);
    }
  }
  if (is_root) CUDA_TRY(cudaMemcpyAsync(d_hdr, hdr, sizeof(hdr), cudaMemcpyHostToDevice, ctx->stream));
  NCCL_TRY(g_nccl.Broadcast(d_hdr, d_hdr, sizeof(hdr), ncclUint8, root, cs.comm, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(hdr, d_hdr, sizeof(hdr), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (hdr[0] < 1) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_set_cloud_bcast: the root's cloud is invalid (need finite xyz, normals, "
                   "view_points, N > 0, 1 <= cameras <= %d)", GPDB_MAX_CAMERAS);
    return GPDB_ERR_INVALID;
  }
  N = (int32_t)hdr[0];
  K = (int32_t)hdr[1];
  if (!is_root && (rc = gpdb_cloud_reserve(ctx, s, (size_t)N, 1)) != GPDB_OK) return rc;
  NCCL_TRY(g_nccl.GroupStart());
  NCCL_TRY(g_nccl.Broadcast(s.xyz, s.xyz, sizeof(float) * 3 * (size_t)N, ncclUint8, root, cs.comm, ctx->stream));
  NCCL_TRY(g_nccl.Broadcast(s.nrm, s.nrm, sizeof(double) * 3 * (size_t)N, ncclUint8, root, cs.comm, ctx->stream));
  NCCL_TRY(g_nccl.Broadcast(s.cam, s.cam, (size_t)N, ncclUint8, root, cs.comm, ctx->stream));
  NCCL_TRY(g_nccl.GroupEnd());
  memset(&desc, 0, sizeof(desc));
  desc.K = K;
  desc.all_seen = (int)hdr[2];
  for (int k = 0; k < K; k++)
    for (int r = 0; r < 3; r++) desc.vp[k][r] = hdr[4 + 3 * k + r];
  const int off[2] = {0, N};
  if ((rc = gpdb_install_clouds(ctx, s, &desc, off, 1, true)) != GPDB_OK) return rc;
  return N;
}

int gpdb_detect_sharded_resident(gpdb_ctx *ctx, const int32_t *d_sample_idx_local, int32_t n_local, int32_t slot_samples,
                                 uint8_t *d_gathered, gpdb_result *stats) {
  int rc = need_comm(ctx);
  if (rc != GPDB_OK) return rc;
  if ((rc = gpdb_check_state(ctx, true, true)) != GPDB_OK) return rc;
  CommState &cs = *ctx->comm;
  if (!stats || n_local < 0 || n_local > slot_samples || !d_gathered || (n_local > 0 && !d_sample_idx_local)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_sharded_resident: bad arguments");
    return GPDB_ERR_INVALID;
  }
  const int P = ctx->hp.P;
  const size_t slot = (size_t)gpdb_slot_bytes(slot_samples, P);
  uint8_t *mine = d_gathered + slot * (size_t)cs.rank;
  float *d_scores = reinterpret_cast<float *>(mine);
  uint8_t *d_flags = mine + sizeof(float) * (size_t)slot_samples * P;
  if (n_local < slot_samples) {  // padding of a short slice: NaN scores, zero flags
    const size_t a = (size_t)n_local * P, b = (size_t)slot_samples * P;
    CUDA_TRY(cudaMemsetAsync(d_scores + a, 0xFF, sizeof(float) * (b - a), ctx->stream));
    CUDA_TRY(cudaMemsetAsync(d_flags + a, 0, b - a, ctx->stream));
  }
  PipeRequest rq = {.store = &ctx->one, .sample_idx = d_sample_idx_local, .n = n_local, .samples_on_device = true,
                    .classify = true, .d_flags = d_flags, .d_scores = d_scores, .dest = PIPE_STAY};
  int nc = gpdb_run_pipeline(ctx, rq, stats);
  if (nc < 0) return nc;
  cs.count = nc;
  CUDA_TRY(cudaMemcpyAsync(mine + slot - 16, &cs.count, sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
  NCCL_TRY(g_nccl.AllGather(mine, d_gathered, slot, ncclUint8, cs.comm, ctx->stream));  // in place
  ctx->launches++;
  stats->kernel_launches++;
  return nc;
}

int gpdb_detect_sharded(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n, gpdb_result *out) {
  int rc = need_comm(ctx);
  if (rc != GPDB_OK) return rc;
  if ((rc = gpdb_check_state(ctx, true, true)) != GPDB_OK) return rc;
  CommState &cs = *ctx->comm;
  if (!out || n < 0 || (n > 0 && !sample_idx)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_detect_sharded: bad arguments");
    return GPDB_ERR_INVALID;
  }
  const int P = ctx->hp.P;
  int32_t lo, hi, slot_samples;
  gpdb_shard_bounds(n, cs.rank, cs.nranks, &lo, &hi, &slot_samples);
  // this rank's slice through the host-buffer pipeline (pose records of the slice -> pinned arena, sample_slot global)
  PipeRequest rq = {.store = &ctx->one, .sample_idx = sample_idx + lo, .n = hi - lo, .classify = true, .dest = PIPE_TO_HOST,
                    .slot_base = lo};
  int nc = gpdb_run_pipeline(ctx, rq, out);
  if (nc < 0) return nc;
  // the request now names the device arrays holding the slice's dense flags / scores: pack them into this rank's slot
  // and all-gather
  const size_t slot = (size_t)gpdb_slot_bytes(slot_samples, P);
  const size_t np_l = (size_t)(hi - lo) * P, np_s = (size_t)slot_samples * P;
  uint8_t *d_gath = (uint8_t *)gpdb_scratch(ctx, SCR_WORK_B, slot * (size_t)cs.nranks);
  if (!d_gath) { gpdb_free_result(out); return GPDB_ERR_CUDA; }
  uint8_t *mine = d_gath + slot * (size_t)cs.rank;
  int err = GPDB_OK;
  auto cu = [&](cudaError_t e) { if (e != cudaSuccess && err == GPDB_OK) { gpdb_set_error(ctx, GPDB_ERR_CUDA, "gpdb_detect_sharded: %s", cudaGetErrorString(e)); err = GPDB_ERR_CUDA; } };
  cu(cudaMemsetAsync(mine, 0xFF, sizeof(float) * np_s, ctx->stream));
  cu(cudaMemsetAsync(mine + sizeof(float) * np_s, 0, slot - sizeof(float) * np_s, ctx->stream));
  if (np_l) {
    cu(cudaMemcpyAsync(mine, rq.d_scores, sizeof(float) * np_l, cudaMemcpyDeviceToDevice, ctx->stream));
    cu(cudaMemcpyAsync(mine + sizeof(float) * np_s, rq.d_flags, np_l, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  cs.count = nc;
  cu(cudaMemcpyAsync(mine + slot - 16, &cs.count, sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
  if (err == GPDB_OK && g_nccl.AllGather(mine, d_gath, slot, ncclUint8, cs.comm, ctx->stream) != ncclSuccess) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "ncclAllGather failed");
    err = GPDB_ERR_CUDA;
  }
  ctx->launches++;
  // the gathered arrays [n*P] of all ranks go to pinned memory owned by the result (freed with it), the per-rank
  // candidate counts ride in the slot tails
  const size_t nP = (size_t)n * P, off_flags = (sizeof(float) * nP + 63) / 64 * 64, off_counts = (off_flags + nP + 63) / 64 * 64;
  uint8_t *h = (uint8_t *)gpdb_result_extra(out, off_counts + 16 * (size_t)cs.nranks + 64);
  if (!h && err == GPDB_OK) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "cudaHostAlloc of the gathered result arrays failed");
    err = GPDB_ERR_CUDA;
  }
  for (int r = 0; r < cs.nranks && err == GPDB_OK; r++) {
    int32_t a, b;
    gpdb_shard_bounds(n, r, cs.nranks, &a, &b, nullptr);
    const uint8_t *src = d_gath + slot * (size_t)r;
    if (b > a) {
      cu(cudaMemcpyAsync(h + sizeof(float) * (size_t)a * P, src, sizeof(float) * (size_t)(b - a) * P, cudaMemcpyDeviceToHost, ctx->stream));
      cu(cudaMemcpyAsync(h + off_flags + (size_t)a * P, src + sizeof(float) * np_s, (size_t)(b - a) * P, cudaMemcpyDeviceToHost, ctx->stream));
    }
    cu(cudaMemcpyAsync(h + off_counts + 16 * (size_t)r, src + slot - 16, 16, cudaMemcpyDeviceToHost, ctx->stream));
  }
  cu(cudaStreamSynchronize(ctx->stream));
  if (err != GPDB_OK) {
    gpdb_free_result(out);
    return err;
  }
  int total = 0;
  for (int r = 0; r < cs.nranks; r++) total += *reinterpret_cast<const int32_t *>(h + off_counts + 16 * (size_t)r);
  // the slice-sized per-pose arrays of the arena are replaced by the gathered ones; frames stay per-slice -> not returned
  out->frame_valid = nullptr;
  out->frames = nullptr;
  out->pose_scores = reinterpret_cast<float *>(h);
  out->pose_flags = h + off_flags;
  out->n_samples = n;
  out->n_total_candidates = total;
  out->kernel_launches++;
  return nc;
}

}  // extern "C"
