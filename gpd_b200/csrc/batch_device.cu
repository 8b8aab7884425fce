// batch_device.cu — kernels of the installs and batch entry points (api.cu), host calls and gpdb_*_device twins
// alike: camera-mask packing, the finiteness and sample-index checks, cloud-local sample slots of records, and the
// caller's hands made addressable by the image kernels. The checks write the lowest
// offending position (atomicMin into a word the caller set to all ones), so that their error messages name the first
// offending point, entry or sample, as a sequential loop over the input would.
#include <algorithm>

#include "common.cuh"

namespace {

// one thread per point: bit k of cam[g] set when entry k of the point's row counts as seen (== 1 with eq1, else > 0); a
// null rows means every camera sees every point. all_seen[b] (set to 1 by the caller) drops to 0 when a point of cloud b
// misses a camera; with strict01, entries other than 0 / 1 report their index in the concatenated blocks.
__global__ void k_pack_cameras(const int32_t *rows, const int *off, const long long *row_off, const int *ks, int B, int N,
                               int eq1, int strict01, uint8_t *cam, int *all_seen, unsigned long long *first_bad) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const int b = csr_owner(off, B, g);
  const int K = ks[b];
  const unsigned all = (1u << K) - 1;
  unsigned m = all;
  if (rows) {
    const long long e0 = row_off[b] + (long long)(g - off[b]) * K;
    m = 0;
    for (int k = 0; k < K; k++) {
      const int32_t v = rows[e0 + k];
      m |= (unsigned)(eq1 ? v == 1 : v > 0) << k;
      if (strict01 && v != 0 && v != 1) atomicMin(first_bad, (unsigned long long)(e0 + k));
    }
  }
  cam[g] = (uint8_t)m;
  if (m != all) all_seen[b] = 0;
}

// the first point (index of float / 3) with a non-finite coordinate
__global__ void k_first_nonfinite(const float *v, long long n, unsigned long long *first_bad) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (!isfinite(v[i])) atomicMin(first_bad, (unsigned long long)(i / 3));
}

// the first position of the CSR sample list whose cloud-local index lies outside its cloud: lim[b] = N_b + M_b
__global__ void k_check_samples(const int *sidx, int n, const int *soff, int B, const int *lim, unsigned long long *first_bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int v = sidx[i];
  if (v < 0 || v >= lim[csr_owner(soff, B, i)]) atomicMin(first_bad, (unsigned long long)i);
}

// sample slots are positions in the whole sample stream: subtract the first slot of the record's cloud (in may equal out)
__global__ void k_local_slots(const gpdb_pose *in, int n, const int *soff, int B, gpdb_pose *out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  gpdb_pose p = in[j];
  p.sample_slot -= soff[csr_owner(soff, B, p.sample_slot)];
  out[j] = p;
}

// the caller's hands as the image kernels address them: sample slot = the hand's position in the caller's array, which
// the hand offsets (uploaded as the store's soff) assign to its cloud. No other field of a record indexes memory there.
__global__ void k_image_hands(const gpdb_pose *in, int n, int base, gpdb_pose *out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  gpdb_pose p = in[j];
  p.sample_slot = base + j;
  out[j] = p;
}

}  // namespace

int batch_pack_cameras(gpdb_ctx *ctx, const int32_t *d_rows, const int *d_off, const long long *d_row_off, const int *d_k,
                       int B, int N, bool eq1, bool strict01, uint8_t *d_cam, int *d_all_seen,
                       unsigned long long *d_first_bad) {
  if (N == 0) return GPDB_OK;
  k_pack_cameras<<<(N + 255) / 256, 256, 0, ctx->stream>>>(d_rows, d_off, d_row_off, d_k, B, N, eq1, strict01, d_cam,
                                                           d_all_seen, d_first_bad);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int batch_first_nonfinite(gpdb_ctx *ctx, const float *d_v, long long n, unsigned long long *d_first_bad) {
  if (n == 0) return GPDB_OK;
  const long long blocks = std::min((n + 255) / 256, (long long)ctx->sm_count * 16);
  k_first_nonfinite<<<(int)blocks, 256, 0, ctx->stream>>>(d_v, n, d_first_bad);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int batch_check_samples(gpdb_ctx *ctx, const int *d_sidx, int n, const int *d_soff, int B, const int *d_lim,
                        unsigned long long *d_first_bad) {
  if (n == 0) return GPDB_OK;
  k_check_samples<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_sidx, n, d_soff, B, d_lim, d_first_bad);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int batch_local_slots(gpdb_ctx *ctx, const gpdb_pose *d_in, int n, const int *d_soff, int B, gpdb_pose *d_out) {
  if (n == 0) return GPDB_OK;
  k_local_slots<<<(n + 127) / 128, 128, 0, ctx->stream>>>(d_in, n, d_soff, B, d_out);
  LAUNCH_CHECK();
  return GPDB_OK;
}

int batch_image_hands(gpdb_ctx *ctx, const gpdb_pose *d_in, int n, int base, gpdb_pose *d_out) {
  if (n == 0) return GPDB_OK;
  k_image_hands<<<(n + 127) / 128, 128, 0, ctx->stream>>>(d_in, n, base, d_out);
  LAUNCH_CHECK();
  return GPDB_OK;
}
