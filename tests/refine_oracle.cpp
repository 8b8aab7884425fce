// refine_oracle.cpp — the CPU oracle of include/gpd_b200_refine.h: a C++ restatement of Cloud::refineNormals, written from
// the header's rules, for clouds too large for the numpy restatement. The neighbour lists are a brute-force partial sort
// of every point's (float32 distance bits, index) keys; the iterations follow the rules point by point, one cloud per
// host thread. Test infrastructure only: tests/refine_oracle.py builds it (g++ -ffp-contract=off) into a temporary
// directory.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "gpd_b200_refine.h"

namespace {

uint64_t key(const float *xyz, int i, int j) {
  float d = gpdb_refine_l2(xyz + 3 * (size_t)i, xyz + 3 * (size_t)j);
  uint32_t bits;
  std::memcpy(&bits, &d, 4);
  return ((uint64_t)bits << 32) | (uint32_t)j;
}

// rule 1 for points [a, e) of one cloud of n points: nbr[i*k + r], r < min(k, n)
void knn_rows(const float *xyz, int n, int k, int a, int e, int32_t *nbr) {
  const int L = std::min(k, n);
  std::vector<uint64_t> kk((size_t)n);
  for (int i = a; i < e; i++) {
    for (int j = 0; j < n; j++) kk[j] = key(xyz, i, j);
    std::partial_sort(kk.begin(), kk.begin() + L, kk.end());
    for (int r = 0; r < L; r++) nbr[(size_t)i * k + r] = (int32_t)(uint32_t)kk[r];
  }
}

// rules 2-5 for one cloud given its lists; returns the iterations run
int iterate(int n, int k, const int32_t *nbr, double *normals) {
  if (n == 0) return 0;
  const int L = std::min(k, n);
  std::vector<float> m(3 * (size_t)n), next(3 * (size_t)n);
  std::vector<float> err((size_t)n);
  for (size_t i = 0; i < 3 * (size_t)n; i++) m[i] = (float)normals[i];
  int t = 0;
  while (t < GPDB_REFINE_MAX_ITERATIONS) {
    for (int i = 0; i < n; i++) {
      float sx = 0.0f, sy = 0.0f, sz = 0.0f;
      for (int r = 0; r < L; r++) {
        const float *q = m.data() + 3 * (size_t)nbr[(size_t)i * k + r];
        if (!gpdb_refine_finite3(q)) continue;
        sx = sx + q[0];
        sy = sy + q[1];
        sz = sz + q[2];
      }
      gpdb_refine_normal(sx, sy, sz, next.data() + 3 * (size_t)i);
      err[i] = gpdb_refine_error(m.data() + 3 * (size_t)i, next.data() + 3 * (size_t)i);
    }
    m.swap(next);
    t++;
    float s = 0.0f;
    for (int i = 0; i < n; i++) s = s + err[i];
    if (s / (float)n < GPDB_REFINE_CONVERGENCE) break;
  }
  for (size_t i = 0; i < 3 * (size_t)n; i++) normals[i] = (double)m[i];
  return t;
}

}  // namespace

extern "C" {

// One cloud: its lists nbr [n * k] (rows of min(k, n) entries) on `threads` host threads.
void refine_oracle_knn(const float *xyz, int n, int k, int32_t *nbr, int threads) {
  std::vector<std::thread> pool;
  const int T = std::max(1, std::min(threads, n));
  for (int t = 0; t < T; t++)
    pool.emplace_back([=] { knn_rows(xyz, n, k, (int)((long long)n * t / T), (int)((long long)n * (t + 1) / T), nbr); });
  for (auto &th : pool) th.join();
}

// One cloud with given lists: normals [3n] refined in place; returns the iterations run.
int refine_oracle_iterate(int n, int k, const int32_t *nbr, double *normals) { return iterate(n, k, nbr, normals); }

// A CSR batch (off [B + 1]): every cloud on its own, the clouds spread over `threads` host threads. normals [3N] are
// refined in place, iters [B] receives the iteration counts.
void refine_oracle_batch(int B, const int32_t *off, const float *xyz, double *normals, int k, int32_t *iters, int threads) {
  std::atomic<int> next{0};
  std::vector<std::thread> pool;
  for (int t = 0; t < std::max(1, threads); t++)
    pool.emplace_back([&] {
      for (int b; (b = next++) < B;) {
        const int o = off[b], n = off[b + 1] - o;
        std::vector<int32_t> nbr((size_t)n * k);
        knn_rows(xyz + 3 * (size_t)o, n, k, 0, n, nbr.data());
        iters[b] = iterate(n, k, nbr.data(), normals + 3 * (size_t)o);
      }
    });
  for (auto &th : pool) th.join();
}

}  // extern "C"
