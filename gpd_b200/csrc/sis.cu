// sis.cu — kernels of gpdb_sis_batch (api.cu): SequentialImportanceSampling's draws (include/gpd_b200_sis.h), the kept-set
// bookkeeping of every round, the installation of a round's positions and the final score filter. Everything between two
// hand searches stays on the device; the host reads back one count per cloud and round to size the next pipeline call.
#include <cub/block/block_scan.cuh>

#include "../../include/gpd_b200_sis.h"
#include "grid.cuh"

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

}  // namespace

int sis_draw(gpdb_ctx *ctx, const SisDraw &q, int B, const CloudSet &s, const int *d_init_off, const int *d_init_idx,
             const double *d_kept, const int *d_kcount, int stage_cap, double *d_eval, int *d_ecount) {
  if (B == 0) return GPDB_OK;
  k_sis_draw<<<B, NT_SIS, sizeof(double) * 3 * (size_t)stage_cap, ctx->stream>>>(q, s.view, s.desc, d_init_off, d_init_idx,
                                                                                  d_kept, d_kcount, stage_cap, d_eval,
                                                                                  d_ecount);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int sis_keep(gpdb_ctx *ctx, const CloudSet &s, const uint8_t *d_flags, const int *d_sidx, const int *d_init_off, int RS,
             double *d_kept, int *d_kcount) {
  if (s.n == 0) return GPDB_OK;
  k_sis_keep<<<s.n, NT_SIS, 0, ctx->stream>>>(d_flags, ctx->hp.P, d_sidx, s.soff, s.desc, s.view, d_init_off, RS, d_kept,
                                               d_kcount);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int sis_install(gpdb_ctx *ctx, CloudSet &s, const double *d_src, int stride, int add, const int *d_init_off,
                const int *d_cnt, const int *d_soff, double *d_dst, int *d_sidx) {
  if (s.n == 0) return GPDB_OK;
  k_sis_install<<<s.n, 128, 0, ctx->stream>>>(d_src, stride, add, d_init_off, d_cnt, d_soff, s.desc, d_dst, d_sidx);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int sis_filter(gpdb_ctx *ctx, gpdb_pose *d_rec, int n, const int *d_soff, int B, double min_score, uint8_t *d_keep,
               int *d_hcount) {
  if (n == 0) return GPDB_OK;
  k_sis_filter<<<(n + 127) / 128, 128, 0, ctx->stream>>>(d_rec, n, d_soff, B, min_score, d_keep, d_hcount);
  LAUNCH_CHECK();
  return GPDB_OK;
}
