// sis.cu — gpdb_sis_batch[_device] and gpdb_sis_positions: SequentialImportanceSampling's draws (include/gpd_b200_sis.h),
// the kept-set bookkeeping of every round, the installation of a round's positions and the final score filter. Everything
// between two hand searches stays on the device; the host reads back one count per cloud and round to size the next
// pipeline call. The entry points, their checks, the rounds (sis_run) and the record gpdb_sis_positions reads (SisState)
// follow the kernels.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <cub/block/block_scan.cuh>
#include <vector>

#include "../../include/gpd_b200_sis.h"
#include "grid.cuh"

// Per cloud b of a batch with R rounds of S positions and initial offsets init_off[B+1] (device), the kept arena holds
// room for init_off[b+1] - init_off[b] + R*S positions from position init_off[b] + b*R*S, the evaluated arena S positions
// per (cloud, round) from (b*R + r)*S; kcount[b] counts the kept positions, ecount[r*B + b] the positions of round r.
struct SisDraw {
  int R, S, n_gauss, n_rand, method, round;
  double sigma, ws[6];
  unsigned long long seed;
};

namespace {

constexpr int NT_SIS = 256;
using Scan = cub::BlockScan<int, NT_SIS>;

// d2 = (dx*dx + dy*dy) + dz*dz, each operation rounded on its own
__device__ __forceinline__ double d2_rn(const double *x, const double *k) {
  const double dx = __dsub_rn(x[0], k[0]), dy = __dsub_rn(x[1], k[1]), dz = __dsub_rn(x[2], k[2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// Appends the accepted proposals of one wave (this thread's proposal: acc, x) behind the `filled` slots already written,
// in proposal order, up to `need`; returns the slots filled after the wave (the same on every thread).
__device__ __forceinline__ int take(Scan::TempStorage &tmp, bool acc, const double *x, double *out, int filled, int need) {
  int rank, total;
  Scan(tmp).ExclusiveSum(acc ? 1 : 0, rank, total);
  if (acc && filled + rank < need)
    for (int k = 0; k < 3; k++) out[3 * (size_t)(filled + rank) + k] = x[k];
  __syncthreads();  // tmp is reused by the next wave
  return min(need, filled + total);
}

// One CTA per cloud. The Gaussian proposals of the round, then the uniform ones, in waves of NT_SIS proposals; the first
// accepted proposals in t order fill the slots. Kept positions are staged in shared memory when they fit.
__global__ void __launch_bounds__(NT_SIS) k_sis_draw(SisDraw q, DevCloud cl, const CloudDesc *desc, const int *init_off,
                                                     const int *init_idx, const double *kept, const int *kcount, int stage_cap,
                                                     double *eval, int *ecount) {
  extern __shared__ __align__(16) double sk[];
  __shared__ Scan::TempStorage tmp;
  const int b = blockIdx.x, B = gridDim.x, tid = threadIdx.x;
  const int m = kcount[b];
  if (m == 0) {  // inactive: no initial hand
    if (tid == 0) ecount[q.round * B + b] = 0;
    return;
  }
  const double *K = kept + 3 * ((size_t)init_off[b] + (size_t)b * q.R * q.S);
  if (m <= stage_cap) {
    for (int i = tid; i < 3 * m; i += NT_SIS) sk[i] = K[i];
    K = sk;
    __syncthreads();
  }
  double *out = eval + 3 * ((size_t)b * q.R + q.round) * q.S;
  const unsigned long long key = q.seed + (unsigned long long)b;
  const uint32_t r = (uint32_t)q.round;
  int filled = 0;
  for (int t0 = 0; filled < q.n_gauss && t0 < GPDB_SIS_MAX_PROPOSALS; t0 += NT_SIS) {
    const uint32_t t = (uint32_t)(t0 + tid);
    const gpdb_u32x4 c0 = gpdb_sis_draw(key, t, r, GPDB_SIS_GAUSS, 0), c1 = gpdb_sis_draw(key, t, r, GPDB_SIS_GAUSS, 1);
    const double *pk = K + 3 * (size_t)(c0.x % (uint32_t)m);
    const double r01 = sqrt(-2.0 * log(gpdb_sis_unit(c0.y))), a01 = 2.0 * gpdb_sis_unit(c0.z);
    const double z[3] = {r01 * cospi(a01), r01 * sinpi(a01),
                         sqrt(-2.0 * log(gpdb_sis_unit(c0.w))) * cospi(2.0 * gpdb_sis_unit(c1.x))};
    double x[3];
    for (int k = 0; k < 3; k++) x[k] = __dadd_rn(pk[k], __dmul_rn(q.sigma, z[k]));
    bool acc = true;
    if (q.method == 1) {  // max of Gaussians: the parent must be (one of) the nearest kept positions
      const double dp = d2_rn(x, pk);
      for (int j = 0; j < m && acc; j++) acc = dp <= d2_rn(x, K + 3 * (size_t)j);
    }
    filled = take(tmp, acc, x, out, filled, q.n_gauss);
  }
  const int n_init = init_off[b + 1] - init_off[b], N = desc[b].N, off = desc[b].off;
  int rfill = 0;
  for (int t0 = 0; rfill < q.n_rand && t0 < GPDB_SIS_MAX_PROPOSALS; t0 += NT_SIS) {
    const uint32_t t = (uint32_t)(t0 + tid);
    const gpdb_u32x4 c = gpdb_sis_draw(key, t, r, GPDB_SIS_UNIFORM, 0);
    const int pi = n_init > 0 ? init_idx[init_off[b] + (int)(c.x % (uint32_t)n_init)] : (int)(c.x % (uint32_t)N);
    const float *p = cl.xyz + 3 * ((size_t)off + pi);
    const double x[3] = {(double)p[0], (double)p[1], (double)p[2]};
    const bool acc = x[0] >= q.ws[0] && x[0] <= q.ws[1] && x[1] >= q.ws[2] && x[1] <= q.ws[3] && x[2] >= q.ws[4] &&
                     x[2] <= q.ws[5];
    rfill = take(tmp, acc, x, out + 3 * (size_t)filled, rfill, q.n_rand);
  }
  if (tid == 0) ecount[q.round * B + b] = filled + rfill;
}

// One CTA per cloud: the samples of the cloud's range of the CSR list, in order, whose poses include one with VALID and
// FILTERED set append their position (the hand set's sample_) to the kept positions.
__global__ void __launch_bounds__(NT_SIS) k_sis_keep(const uint8_t *flags, int P, const int *sidx, const int *soff,
                                                     const CloudDesc *desc, DevCloud cl, const int *init_off, int RS,
                                                     double *kept, int *kcount) {
  __shared__ Scan::TempStorage tmp;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int i0 = soff[b], i1 = soff[b + 1];
  const CloudDesc &D = desc[b];
  const DevCloud lc = local_cloud(D, cl);
  double *K = kept + 3 * ((size_t)init_off[b] + (size_t)b * RS);
  int cnt = kcount[b];
  for (int c = i0; c < i1; c += NT_SIS) {
    const int i = c + tid;
    bool keep = false;
    if (i < i1)
      for (int p = 0; p < P && !keep; p++) keep = (flags[(size_t)i * P + p] & 3) == 3;
    int rank, total;
    Scan(tmp).ExclusiveSum(keep ? 1 : 0, rank, total);
    if (keep) sample_position(lc, sidx[i], K + 3 * (size_t)(cnt + rank));
    cnt += total;
    __syncthreads();
  }
  if (tid == 0) kcount[b] = cnt;
}

__global__ void k_sis_install(const double *src, int stride, int add, const int *init_off, const int *cnt, const int *soff,
                              CloudDesc *desc, double *dst, int *sidx) {
  const int b = blockIdx.x, n = cnt[b], o = soff[b], N = desc[b].N;
  const double *S = src + 3 * ((size_t)b * stride + add + (init_off ? init_off[b] : 0));
  if (threadIdx.x == 0) desc[b].pos = o;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    for (int k = 0; k < 3; k++) dst[3 * (size_t)(o + j) + k] = S[3 * (size_t)j + k];
    sidx[o + j] = N + j;
  }
}

__global__ void k_sis_filter(gpdb_pose *rec, int n, const int *soff, int B, double min_score, uint8_t *keep, int *hcount) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int b = csr_owner(soff, B, rec[j].sample_slot);
  rec[j].sample_slot -= soff[b];
  const bool k = (double)rec[j].score > min_score;  // pruneGraspCandidates (grasp_detector.cpp:544-548)
  keep[j] = k ? 3 : 0;
  if (k) atomicAdd(hcount + b, 1);
}

// the draws of round q.round for every cloud with a kept position (one CTA per cloud); stage_cap: kept positions a CTA may
// stage in shared memory
int sis_draw(gpdb_ctx *ctx, const SisDraw &q, int B, const CloudSet &s, const int *d_init_off, const int *d_init_idx,
             const double *d_kept, const int *d_kcount, int stage_cap, double *d_eval, int *d_ecount) {
  if (B == 0) return GPDB_OK;
  k_sis_draw<<<B, NT_SIS, sizeof(double) * 3 * (size_t)stage_cap, ctx->stream>>>(q, s.view, s.desc, d_init_off, d_init_idx,
                                                                                  d_kept, d_kcount, stage_cap, d_eval,
                                                                                  d_ecount);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// appends, per cloud and in sample order, the position of every sample of the CSR list d_sidx (offsets s.soff) with a
// VALID|FILTERED pose in the dense flags [n * P] to the cloud's kept positions
int sis_keep(gpdb_ctx *ctx, const CloudSet &s, const uint8_t *d_flags, const int *d_sidx, const int *d_init_off, int RS,
             double *d_kept, int *d_kcount) {
  if (s.n == 0) return GPDB_OK;
  k_sis_keep<<<s.n, NT_SIS, 0, ctx->stream>>>(d_flags, ctx->hp.P, d_sidx, s.soff, s.desc, s.view, d_init_off, RS, d_kept,
                                               d_kcount);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// the positions to install, as gpdb_set_clouds_samples would lay them out: cloud b's d_cnt[b] positions from position
// b*stride + add (+ d_init_off[b] when given) of d_src go to d_dst (the store's sample arena) at d_soff[b],
// d_sidx[d_soff[b] + j] = N_b + j, and the descriptors' first position becomes d_soff[b]
int sis_install(gpdb_ctx *ctx, CloudSet &s, const double *d_src, int stride, int add, const int *d_init_off,
                const int *d_cnt, const int *d_soff, double *d_dst, int *d_sidx) {
  if (s.n == 0) return GPDB_OK;
  k_sis_install<<<s.n, 128, 0, ctx->stream>>>(d_src, stride, add, d_init_off, d_cnt, d_soff, s.desc, d_dst, d_sidx);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// the final score filter over n records of a batch call (stream sample slots, offsets d_soff): keep flag 3 where
// score > min_score, sample slots made cloud-local, d_hcount[b] (zeroed by the caller) counts cloud b's kept records
int sis_filter(gpdb_ctx *ctx, gpdb_pose *d_rec, int n, const int *d_soff, int B, double min_score, uint8_t *d_keep,
               int *d_hcount) {
  if (n == 0) return GPDB_OK;
  k_sis_filter<<<(n + 127) / 128, 128, 0, ctx->stream>>>(d_rec, n, d_soff, B, min_score, d_keep, d_hcount);
  LAUNCH_CHECK();
  return GPDB_OK;
}

}  // namespace

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

// What the last SIS call evaluated and kept, for gpdb_sis_positions (gpdb_sis_batch): the counts on
// the host, the positions in SCR_SIS
struct SisState {
  bool valid = false;
  int B = 0, R = 0, S = 0;
  std::vector<int> init_off;  // [B + 1] initial samples per cloud (they size the kept arena)
  std::vector<int> ecount;    // [R * B] round-major, as the device holds them
  std::vector<int> koff;      // [B + 1] kept positions per cloud
};

void sis_forget(gpdb_ctx *ctx) {
  if (ctx->sis) ctx->sis->valid = false;
}

void sis_free(gpdb_ctx *ctx) { delete ctx->sis; }

// The arrays of SCR_SIS for B clouds, R rounds of S positions and n_init initial samples: kept positions (KC = n_init +
// B*R*S of them) and evaluated positions, the initial offsets and indices, the kept counts [B] followed by the round
// counts [R*B] (ecount, zeroed with them), the hand counts and the installed sample list
struct SisArena {
  double *kept, *eval;
  int *init_off, *init_idx, *kcount, *ecount, *hcount, *sidx;
};
static void sis_layout(Carve &c, int B, int R, int S, int n_init, SisArena &a) {
  const size_t RS = (size_t)R * S, KC = (size_t)n_init + (size_t)B * RS;
  a.kept = c.take<double>(3 * KC);
  a.eval = c.take<double>(3 * (size_t)B * RS);
  a.init_off = c.take<int>((size_t)B + 1);
  a.init_idx = c.take<int>(n_init);
  a.kcount = c.take<int>((size_t)B * (R + 1));
  a.ecount = c.base ? a.kcount + B : nullptr;
  a.hcount = c.take<int>(B);
  a.sidx = c.take<int>(KC);
}

// The argument checks of gpdb_sis_batch[_device] after the state checks: parameters and offsets
static int check_sis_args(gpdb_ctx *ctx, const char *name, int B, const gpdb_sis_params *sp, const int32_t *init_offsets,
                          const void *init_idx, const void *out, const int32_t *hand_offsets_out) {
  if (!sp || !init_offsets || init_offsets[0] != 0 || !out || !hand_offsets_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need params, init_offsets[%d] starting at 0, a result and hand_offsets_out",
                   name, B + 1);
    return GPDB_ERR_INVALID;
  }
  if (sp->num_iterations < 0 || sp->num_samples_per_iteration < 0 || sp->min_inliers < 0) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: num_iterations, num_samples_per_iteration and min_inliers must not be negative",
                   name);
    return GPDB_ERR_INVALID;
  }
  if (!(sp->prob_rand_samples >= 0.0 && sp->prob_rand_samples <= 1.0)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: prob_rand_samples = %g outside [0, 1]", name, sp->prob_rand_samples);
    return GPDB_ERR_INVALID;
  }
  if (!(std::isfinite(sp->standard_deviation) && sp->standard_deviation > 0.0)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: standard_deviation = %g must be finite and positive", name,
                   sp->standard_deviation);
    return GPDB_ERR_INVALID;
  }
  if (sp->sampling_method != 0 && sp->sampling_method != 1) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: sampling_method = %d (0 sum of Gaussians, 1 max of Gaussians)", name,
                   sp->sampling_method);
    return GPDB_ERR_INVALID;
  }
  const int rc = gpdb_check_offsets(ctx, name, "init_offsets", init_offsets, B, "cloud");
  if (rc != GPDB_OK) return rc;
  if (init_offsets[B] > 0 && !init_idx) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null init_idx", name);
    return GPDB_ERR_INVALID;
  }
  const long long kc = (long long)init_offsets[B] + (long long)B * sp->num_iterations * sp->num_samples_per_iteration;
  if (kc * ctx->hp.P > INT32_MAX) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: %lld positions of %d poses exceed the 2^31 records of one call", name, kc,
                   ctx->hp.P);
    return GPDB_ERR_INVALID;
  }
  return GPDB_OK;
}

// The hand search of the CSR list d_sidx (offsets in s.soff, n samples) and the kept-set update it implies
static int sis_search(gpdb_ctx *ctx, CloudSet &s, const int *d_sidx, int n, const SisArena &a, int RS) {
  gpdb_result r;
  PipeRequest rq = {.store = &s, .sample_idx = d_sidx, .n = n, .samples_on_device = true, .per_cloud = true,
                    .classify = false, .dest = PIPE_STAY};
  const int rc = gpdb_run_pipeline(ctx, rq, &r);
  if (rc < 0) return rc;
  return sis_keep(ctx, s, rq.d_flags, d_sidx, a.init_off, RS, a.kept, a.kcount);
}

// Installs, as gpdb_set_clouds_samples would, cloud b's cnt[b] positions of src (see sis_install) straight into the
// store's sample arena, with the sample list N_b + j; h_cnt (host) gives the offsets. Returns the number of positions.
static int sis_install_positions(gpdb_ctx *ctx, CloudSet &s, const SisArena &a, const int *h_cnt, const double *src,
                                 int stride, int add, const int *init_off, const int *d_cnt) {
  const int B = s.n;
  s.pos[0] = 0;
  for (int b = 0; b < B; b++) s.pos[b + 1] = s.pos[b] + h_cnt[b];
  int rc = gpdb_reserve_samples(ctx, s, s.pos[B]);
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaMemcpyAsync(s.soff, s.pos, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = sis_install(ctx, s, src, stride, add, init_off, d_cnt, s.soff, s.samples, a.sidx)) != GPDB_OK) return rc;
  s.n_samples = s.pos[B];
  return s.n_samples;
}

// gpdb_sis_batch[_device] after the checks: d_init_idx already in the arena. dest (host or device) receives the records,
// out the counts and timings.
static int sis_run(gpdb_ctx *ctx, const gpdb_sis_params *sp, const int32_t *init_offsets, const SisArena &a, gpdb_pose *dest,
                   bool dest_on_host, int32_t *hand_offsets_out, gpdb_result *out) {
  CloudSet &s = ctx->many;
  SisState &st = *ctx->sis;
  const int B = s.n, R = sp->num_iterations, S = sp->num_samples_per_iteration, RS = R * S, P = ctx->hp.P;
  const int64_t launches0 = ctx->launches;
  // 1. the initial hand sets (:68-79)
  CUDA_TRY(cudaMemcpyAsync(s.soff, init_offsets, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  int rc = sis_search(ctx, s, a.init_idx, init_offsets[B], a, RS);
  if (rc != GPDB_OK) return rc;
  std::vector<int> h_cnt((size_t)B);
  CUDA_TRY(cudaMemcpyAsync(h_cnt.data(), a.kcount, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  bool any_active = false;
  for (int c : h_cnt) any_active |= c > 0;
  // 2. the rounds (:109-160): draws, then the hand search at the drawn positions
  SisDraw q = {R, S, 0, 0, sp->sampling_method, 0, sp->standard_deviation, {}, sp->seed};
  q.n_rand = (int)(sp->prob_rand_samples * S);
  q.n_gauss = S - q.n_rand;
  for (int k = 0; k < 6; k++) q.ws[k] = sp->workspace[k];
  int max_init = 0;
  for (int b = 0; b < B; b++) max_init = std::max(max_init, init_offsets[b + 1] - init_offsets[b]);
  for (int r = 0; r < R && any_active; r++) {
    q.round = r;
    const int stage_cap = std::min(max_init + r * S, 1920);  // 45 KB: with the scan storage inside the 48 KB default
    if ((rc = sis_draw(ctx, q, B, s, a.init_off, a.init_idx, a.kept, a.kcount, stage_cap, a.eval, a.ecount)) != GPDB_OK)
      return rc;
    CUDA_TRY(cudaMemcpyAsync(h_cnt.data(), a.ecount + (size_t)r * B, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost,
                             ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const int n = sis_install_positions(ctx, s, a, h_cnt.data(), a.eval, RS, r * S, nullptr, a.ecount + (size_t)r * B);
    if (n < 0) return n;
    if (n > 0 && (rc = sis_search(ctx, s, a.sidx, n, a, RS)) != GPDB_OK) return rc;
  }
  // 3. classify at every kept position (:168-170), keep score > min_score
  st.ecount.resize((size_t)R * B);
  CUDA_TRY(cudaMemcpyAsync(h_cnt.data(), a.kcount, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(st.ecount.data(), a.ecount, sizeof(int) * st.ecount.size(), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  const int M = sis_install_positions(ctx, s, a, h_cnt.data(), a.kept, RS, 0, a.init_off, a.kcount);
  if (M < 0) return M;
  st.koff.assign(s.pos, s.pos + B + 1);
  PipeRequest rq = {.store = &s, .sample_idx = a.sidx, .n = M, .samples_on_device = true, .per_cloud = true, .classify = true,
                    .dest = PIPE_ALL_DEVICE};
  if ((rc = gpdb_run_pipeline(ctx, rq, out)) < 0) return rc;
  const int total = out->n_total_candidates;
  uint8_t *d_keep = (uint8_t *)gpdb_scratch(ctx, SCR_FLAGS, (size_t)total);
  gpdb_pose *d_filt = (gpdb_pose *)gpdb_scratch(ctx, SCR_POSES, sizeof(gpdb_pose) * (size_t)total);
  int *d_count = (int *)gpdb_scratch(ctx, SCR_COUNT, 64);
  if (!d_keep || !d_filt || !d_count) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemsetAsync(a.hcount, 0, sizeof(int) * (size_t)B, ctx->stream));
  if ((rc = sis_filter(ctx, ctx->d_sel, total, s.soff, B, sp->min_score, d_keep, a.hcount)) != GPDB_OK) return rc;
  if ((rc = geo_compact(ctx, ctx->d_sel, d_keep, total, d_filt, d_count)) != GPDB_OK) return rc;
  std::vector<int32_t> hoff((size_t)B + 1, 0);
  CUDA_TRY(cudaMemcpyAsync(hoff.data() + 1, a.hcount, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  for (int b = 0; b < B; b++) hoff[b + 1] += hoff[b];
  int n_out = hoff[B];
  if (dest_on_host) dest = n_out ? (gpdb_pose *)malloc(sizeof(gpdb_pose) * (size_t)n_out) : nullptr;
  if (n_out && !dest) {
    gpdb_set_error(ctx, GPDB_ERR_CUDA, "out of host memory for %d records", n_out);
    return GPDB_ERR_CUDA;
  }
  // 4. cluster (:177-179)
  if (sp->min_inliers > 0) {
    n_out = gpdb_cluster_groups(ctx, B, hoff.data(), d_filt, sp->min_inliers, dest, hand_offsets_out, true);
  } else {
    memcpy(hand_offsets_out, hoff.data(), sizeof(int32_t) * ((size_t)B + 1));
    if (n_out) {
      cudaError_t e = cudaMemcpyAsync(dest, d_filt, sizeof(gpdb_pose) * (size_t)n_out, cudaMemcpyDefault, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      if (e != cudaSuccess) {
        gpdb_set_error(ctx, GPDB_ERR_CUDA, "copy of the %d records: %s", n_out, cudaGetErrorString(e));
        n_out = GPDB_ERR_CUDA;
      }
    }
  }
  if (n_out < 0) {
    if (dest_on_host) free(dest);
    return n_out;
  }
  st.valid = true;
  out->n_samples = M;
  out->poses_per_sample = P;
  out->n_candidates = n_out;
  out->candidates = dest_on_host ? dest : nullptr;
  out->kernel_launches = ctx->launches - launches0;
  return n_out;
}

// gpdb_sis_batch[_device]: checks, the initial indices into the arena (checked there, on the device), sis_run
static int sis_batch(gpdb_ctx *ctx, const char *name, const gpdb_sis_params *sp, const int32_t *init_offsets,
                     const int32_t *init_idx, bool device, gpdb_pose *d_hands_out, int32_t *hand_offsets_out,
                     gpdb_result *out) {
  if (!ctx) return GPDB_ERR_INVALID;
  CloudSet &s = ctx->many;
  s.n_samples = 0;  // a failed call leaves no positions behind, and no SIS positions to read back
  sis_forget(ctx);
  int rc = gpdb_check_state(ctx, false, true);
  if (rc != GPDB_OK) return rc;
  if (!ctx->sis) ctx->sis = new SisState();
  if ((rc = gpdb_need_batch(ctx, name, "gpdb_set_clouds / gpdb_preprocess_clouds")) != GPDB_OK) return rc;
  const int B = s.n;
  if ((rc = check_sis_args(ctx, name, B, sp, init_offsets, init_idx, out, hand_offsets_out)) != GPDB_OK) return rc;
  const int n0 = init_offsets[B];
  if (device) {
    if ((rc = gpdb_check_device_ptrs(ctx, name, {{"d_init_idx", init_idx}, {"d_hands_out", d_hands_out}})) != GPDB_OK)
      return rc;
    const long long kc = (long long)n0 + (long long)B * sp->num_iterations * sp->num_samples_per_iteration;
    if (kc > 0 && !d_hands_out) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null d_hands_out", name);
      return GPDB_ERR_INVALID;
    }
  }
  SisState &st = *ctx->sis;
  const int R = sp->num_iterations, S = sp->num_samples_per_iteration;
  SisArena a;
  if (!gpdb_carve(ctx, SCR_SIS, [&](Carve &c) { sis_layout(c, B, R, S, n0, a); })) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(a.init_off, init_offsets, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  if (n0 > 0)
    CUDA_TRY(cudaMemcpyAsync(a.init_idx, init_idx, sizeof(int) * (size_t)n0,
                             device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(a.kcount, 0, sizeof(int) * (size_t)B * (R + 1), ctx->stream));  // kept and round counts
  if ((rc = gpdb_check_cloud_indices(ctx, name, true, init_offsets, a.init_idx, a.init_off)) != GPDB_OK) return rc;
  st.B = B;
  st.R = R;
  st.S = S;
  st.init_off.assign(init_offsets, init_offsets + B + 1);
  rc = sis_run(ctx, sp, init_offsets, a, d_hands_out, !device, hand_offsets_out, out);
  if (rc < 0) {
    s.n_samples = 0;
    st.valid = false;
  }
  return rc;
}

extern "C" {

void gpdb_sis_params_default(gpdb_sis_params *p) {
  memset(p, 0, sizeof(*p));
  p->num_iterations = 5;
  p->num_samples_per_iteration = 50;
  p->prob_rand_samples = 0.3;
  p->standard_deviation = 0.02;
  const double ws[6] = {-1, 1, -1, 1, -1, 1};
  for (int i = 0; i < 6; i++) p->workspace[i] = ws[i];
  p->min_inliers = 1;
}

int gpdb_sis_batch(gpdb_ctx *ctx, const gpdb_sis_params *sp, const int32_t *init_offsets, const int32_t *init_idx,
                   gpdb_result *out, int32_t *hand_offsets_out) {
  return sis_batch(ctx, "gpdb_sis_batch", sp, init_offsets, init_idx, false, nullptr, hand_offsets_out, out);
}

int gpdb_sis_batch_device(gpdb_ctx *ctx, const gpdb_sis_params *sp, const int32_t *init_offsets, const int32_t *d_init_idx,
                          gpdb_pose *d_hands_out, int32_t *hand_offsets_out, gpdb_result *stats) {
  return sis_batch(ctx, "gpdb_sis_batch_device", sp, init_offsets, d_init_idx, true, d_hands_out, hand_offsets_out, stats);
}

int gpdb_sis_positions(gpdb_ctx *ctx, int32_t *eval_offsets_out, int32_t *eval_round_counts_out, double *eval_xyz_out,
                       int32_t *kept_offsets_out, double *kept_xyz_out) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (!ctx->sis || !ctx->sis->valid) {
    gpdb_set_error(ctx, GPDB_ERR_STATE, "gpdb_sis_positions: no successful gpdb_sis_batch call on this context");
    return GPDB_ERR_STATE;
  }
  const SisState &st = *ctx->sis;
  const int B = st.B, R = st.R, S = st.S, RS = R * S;
  SisArena a;
  carve_at(ctx->scratch[SCR_SIS], [&](Carve &c) { sis_layout(c, B, R, S, st.init_off[B], a); });
  CUDA_TRY(cudaSetDevice(ctx->device));
  // the evaluated and kept arenas, read once on the context's stream and unpacked on the host
  std::vector<double> ev(eval_xyz_out ? 3 * (size_t)B * RS : 0), kp(kept_xyz_out ? 3 * ((size_t)st.init_off[B] + (size_t)B * RS) : 0);
  if (!ev.empty()) CUDA_TRY(cudaMemcpyAsync(ev.data(), a.eval, sizeof(double) * ev.size(), cudaMemcpyDeviceToHost, ctx->stream));
  if (!kp.empty()) CUDA_TRY(cudaMemcpyAsync(kp.data(), a.kept, sizeof(double) * kp.size(), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (eval_offsets_out || eval_round_counts_out || eval_xyz_out) {
    size_t o = 0;
    if (eval_offsets_out) eval_offsets_out[0] = 0;
    for (int b = 0; b < B; b++) {
      for (int r = 0; r < R; r++) {
        const int c = st.ecount[(size_t)r * B + b];
        if (eval_round_counts_out) eval_round_counts_out[(size_t)b * R + r] = c;
        if (eval_xyz_out) memcpy(eval_xyz_out + 3 * o, ev.data() + 3 * ((size_t)b * R + r) * S, sizeof(double) * 3 * c);
        o += c;
      }
      if (eval_offsets_out) eval_offsets_out[b + 1] = (int32_t)o;
    }
  }
  if (kept_offsets_out) memcpy(kept_offsets_out, st.koff.data(), sizeof(int32_t) * ((size_t)B + 1));
  if (kept_xyz_out)  // cloud b's kept positions start at position init_off[b] + b*R*S of the arena
    for (int b = 0; b < B; b++)
      memcpy(kept_xyz_out + 3 * (size_t)st.koff[b], kp.data() + 3 * ((size_t)st.init_off[b] + (size_t)b * RS),
             sizeof(double) * 3 * (size_t)(st.koff[b + 1] - st.koff[b]));
  return B;
}

}  // extern "C"
