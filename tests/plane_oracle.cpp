// plane_oracle.cpp — the CPU oracle of include/gpd_b200_plane.h: a C++ restatement of the support-plane fit, written
// from the header's rules, with every intermediate the tests compare (attempts, samples, coefficients, counts, the picked
// hypothesis, hypotheses evaluated, the refined plane and the final mask). The sample shuffle runs on an explicit sparse
// permutation, not the header's closed form. The refit uses the oracle's pcl::eigen33 (gpdo_pcl_eigen33 of
// oracle/libgpd_oracle.so); the covariance is the ordered single float32 pass of computeMeanAndCovarianceMatrix.
// Test infrastructure only: tests/plane_oracle.py builds it (g++ -ffp-contract=off) into a temporary directory.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <thread>
#include <vector>

#include "gpd_b200_sis.h"  // gpdb_philox4x32_10

extern "C" void gpdo_pcl_eigen33(const float *cov9, float *eigenvalue, float *evec);

namespace {

bool model(const float *p0, const float *p1, const float *p2, float c[4]) {
  float a[3], b[3];
  for (int k = 0; k < 3; k++) a[k] = p1[k] - p0[k], b[k] = p2[k] - p0[k];
  const float rx = a[0] / b[0], ry = a[1] / b[1], rz = a[2] / b[2];
  if (rx == ry && rz == ry) return false;
  float n[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
  const float s = std::sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  if (s > 0.0f)
    for (float &v : n) v = v / s;
  c[0] = n[0], c[1] = n[1], c[2] = n[2];
  c[3] = -((n[0] * p0[0] + n[1] * p0[1]) + n[2] * p0[2]);
  return true;
}

bool inlier(const float c[4], const float *p, double thr) {
  const float d = std::fabs(((c[0] * p[0] + c[1] * p[1]) + c[2] * p[2]) + c[3]);
  return (double)d < thr;
}

}  // namespace

extern "C" {

// One cloud of n points with key `key`. Per hypothesis h < max_iterations + 1 (arrays of that length): attempt_out[h]
// (-1: no good sample, or not drawn), sample_out[3h..], coef_out[4h..], count_out[h] (-1 where not evaluated).
// Returns the hypotheses evaluated; *best_out = the picked h (-1: failed).
int plane_oracle_segment(const float *xyz, int n, uint64_t key, double thr, int max_iterations, double probability,
                         int32_t *attempt_out, int32_t *sample_out, float *coef_out, int32_t *count_out, int32_t *best_out,
                         float *plane_out, int32_t *n_inliers_out, uint8_t *eligible_out) {
  const int H = max_iterations + 1;
  for (int h = 0; h < H; h++) attempt_out[h] = -1, count_out[h] = -1;
  int best = -1, best_count = 0, ev = 0;
  double q = 1.0, qp = 1.0;
  for (int h = 0; n >= 3 && h < H; h++) {
    int attempt = -1;
    float c[4];
    int idx[3];
    for (uint32_t a = 0; a < 1000 && attempt < 0; a++) {
      const gpdb_u32x4 ctr = {(uint32_t)h, a, 3u, 0u};
      const gpdb_u32x4 r = gpdb_philox4x32_10(ctr, (uint32_t)key, (uint32_t)(key >> 32));
      const uint32_t w[3] = {r.x, r.y, r.z};
      std::map<uint32_t, uint32_t> perm;  // position -> value where the swaps moved it
      auto at = [&](uint32_t p) { auto it = perm.find(p); return it == perm.end() ? p : it->second; };
      for (uint32_t i = 0; i < 3; i++) {
        const uint32_t j = i + w[i] % ((uint32_t)n - i);
        const uint32_t vi = at(i), vj = at(j);
        perm[i] = vj, perm[j] = vi;
        idx[i] = (int)vj;
      }
      if (model(xyz + 3 * (size_t)idx[0], xyz + 3 * (size_t)idx[1], xyz + 3 * (size_t)idx[2], c)) attempt = (int)a;
    }
    if (attempt < 0) break;
    attempt_out[h] = attempt;
    for (int k = 0; k < 3; k++) sample_out[3 * h + k] = idx[k];
    for (int k = 0; k < 4; k++) coef_out[4 * h + k] = c[k];
    int cnt = 0;
    for (int j = 0; j < n; j++) cnt += inlier(c, xyz + 3 * (size_t)j, thr);
    count_out[h] = cnt;
    ev = h + 1;
    if (best < 0 || cnt > best_count) {
      best = h, best_count = cnt;
      const double w = (double)cnt * (1.0 / (double)n);
      q = std::fmin(std::fmax(1.0 - (w * w) * w, DBL_EPSILON), 1.0 - DBL_EPSILON);
      qp = 1.0;
      for (int i = 0; i <= h; i++) qp = qp * q;
    } else {
      qp = qp * q;
    }
    if (h + 1 > max_iterations || !(qp > 1.0 - probability)) break;
  }
  *best_out = best;
  if (best < 0) {
    for (int k = 0; k < 4; k++) plane_out[k] = NAN;
    *n_inliers_out = 0;
    std::memset(eligible_out, 1, (size_t)n);
    return ev;
  }
  const float *c = coef_out + 4 * best;
  float plane[4] = {c[0], c[1], c[2], c[3]};
  float acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  int m = 0;
  for (int j = 0; j < n; j++) {
    const float *p = xyz + 3 * (size_t)j;
    if (!inlier(c, p, thr)) continue;
    acc[0] += p[0] * p[0], acc[1] += p[0] * p[1], acc[2] += p[0] * p[2];
    acc[3] += p[1] * p[1], acc[4] += p[1] * p[2], acc[5] += p[2] * p[2];
    acc[6] += p[0], acc[7] += p[1], acc[8] += p[2];
    m++;
  }
  if (m > 3) {
    for (float &a : acc) a = a / (float)m;
    float cov[9];
    cov[0] = acc[0] - acc[6] * acc[6];
    cov[1] = acc[1] - acc[6] * acc[7];
    cov[2] = acc[2] - acc[6] * acc[8];
    cov[4] = acc[3] - acc[7] * acc[7];
    cov[5] = acc[4] - acc[7] * acc[8];
    cov[8] = acc[5] - acc[8] * acc[8];
    cov[3] = cov[1], cov[6] = cov[2], cov[7] = cov[5];
    float ev33, nv[3];
    gpdo_pcl_eigen33(cov, &ev33, nv);
    plane[0] = nv[0], plane[1] = nv[1], plane[2] = nv[2];
    plane[3] = -((nv[0] * acc[6] + nv[1] * acc[7]) + nv[2] * acc[8]);
  }
  int fin = 0;
  for (int j = 0; j < n; j++) {
    const bool in = inlier(plane, xyz + 3 * (size_t)j, thr);
    eligible_out[j] = in ? 0 : 1;
    fin += in;
  }
  if (fin == n) std::memset(eligible_out, 1, (size_t)n);
  for (int k = 0; k < 4; k++) plane_out[k] = plane[k];
  *n_inliers_out = fin;
  return ev;
}

// Every cloud of a batch (cloud b: points off[b] .. off[b+1]-1, key seed + b), clouds spread over `threads` host threads:
// planes [4B], n_inliers [B], n_hypotheses [B], eligible [N].
void plane_oracle_batch(int B, const int32_t *off, const float *xyz, uint64_t seed, double thr, int max_iterations,
                        double probability, float *planes, int32_t *n_inliers, int32_t *n_hyp, uint8_t *eligible, int threads) {
  auto work = [&](int t) {
    const int H = max_iterations + 1;
    std::vector<int32_t> att(H), smp(3 * H), cnt(H);
    std::vector<float> coef(4 * H);
    for (int b = t; b < B; b += threads) {
      int32_t best;
      n_hyp[b] = plane_oracle_segment(xyz + 3 * (size_t)off[b], off[b + 1] - off[b], seed + (uint64_t)b, thr, max_iterations,
                                      probability, att.data(), smp.data(), coef.data(), cnt.data(), &best, planes + 4 * b,
                                      n_inliers + b, eligible + off[b]);
    }
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; t++) pool.emplace_back(work, t);
  for (auto &th : pool) th.join();
}

}  // extern "C"
