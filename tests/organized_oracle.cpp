// organized_oracle.cpp — the sequential C++ restatement of include/gpd_b200_organized.h rules 2 - 5 (test infrastructure
// only), over the header's helpers compiled for the host. The eigenvector is the oracle's pcl::eigen33
// (gpdo_pcl_eigen33 of libgpd_oracle.so): pcl_eigen33.cuh is device-only.
#include <math.h>
#include <stdint.h>

#include <vector>

#include "gpd_b200_organized.h"

extern "C" void gpdo_pcl_eigen33(const float *cov9, float *eigenvalue, float *evec);

// one W x H cloud: nrm [3 W H], dist [W H]
extern "C" void org_oracle_normals(int W, int H, const float *xyz, const float *vp, float *nrm, float *dist) {
  const size_t P = (size_t)W * H;
  // rule 2
  std::vector<uint8_t> change(P, 1);
  for (int r = 0; r < H - 1; r++)
    for (int c = 0; c < W - 1; c++) {
      const size_t i = (size_t)r * W + c;
      const float z = xyz[3 * i + 2];
      if (gpdb_org_pair_breaks(z, xyz[3 * (i + 1) + 2])) change[i] = change[i + 1] = 0;
      if (gpdb_org_pair_breaks(z, xyz[3 * (i + W) + 2])) change[i] = change[i + W] = 0;
    }
  // rule 3, the flat array as PCL indexes it
  for (size_t i = 0; i < P; i++) dist[i] = change[i] ? (float)(W + H) : 0.0f;
  for (int r = 1; r < H; r++) {
    float *row = dist + (size_t)r * W, *prev = row - W;
    for (int c = 1; c < W; c++) {
      const float m = gpdb_org_chamfer(prev[c - 1], prev[c], row[c - 1], prev[c + 1]);
      if (m < row[c]) row[c] = m;
    }
  }
  for (int r = H - 2; r >= 0; r--) {
    float *row = dist + (size_t)r * W, *next = row + W;
    for (int c = W - 2; c >= 0; c--) {
      const float m = gpdb_org_chamfer(next[c - 1], next[c], row[c + 1], next[c + 1]);
      if (m < row[c]) row[c] = m;
    }
  }
  // rule 4
  const size_t W1 = (size_t)W + 1, T = W1 * ((size_t)H + 1);
  std::vector<double> S(9 * T, 0.0);
  std::vector<int> N(T, 0);
  for (int r = 0; r < H; r++)
    for (int c = 0; c < W; c++) {
      const float *q = xyz + 3 * ((size_t)r * W + c);
      const bool f = gpdb_org_finite_point(q);
      const double add[9] = {(double)q[0], (double)q[1], (double)q[2], (double)(q[0] * q[0]), (double)(q[0] * q[1]),
                             (double)(q[0] * q[2]), (double)(q[1] * q[1]), (double)(q[1] * q[2]), (double)(q[2] * q[2])};
      const size_t ul = (size_t)r * W1 + c, up = ul + 1, left = ul + W1, me = left + 1;
      for (int ch = 0; ch < 9; ch++) {
        double *s = S.data() + ch * T;
        double v = gpdb_org_integral(s[up], s[left], s[ul]);
        if (f) v += add[ch];
        s[me] = v;
      }
      N[me] = N[up] + N[left] - N[ul] + (f ? 1 : 0);
    }
  // rule 5
  const float nan = NAN;
  for (int r = 0; r < H; r++)
    for (int c = 0; c < W; c++) {
      const size_t p = (size_t)r * W + c;
      float *n = nrm + 3 * p;
      n[0] = n[1] = n[2] = nan;
      const int B = GPDB_ORG_BORDER;
      if (r < B || r >= H - B || c < B || c >= W - B) continue;
      const float *q = xyz + 3 * p;
      if (!isfinite(q[2])) continue;
      const float s = GPDB_ORG_SMOOTHING < dist[p] ? GPDB_ORG_SMOOTHING : dist[p];
      if (!(s > 2.0f)) continue;
      const int w = (int)s, x0 = c - w / 2, y0 = r - w / 2;
      const size_t ul = (size_t)y0 * W1 + x0, ur = ul + w, ll = (size_t)(y0 + w) * W1 + x0, lr = ll + w;
      const int count = ((N[lr] + N[ul]) - N[ur]) - N[ll];
      if (count == 0) continue;
      double sum[9];
      for (int ch = 0; ch < 9; ch++) {
        const double *t = S.data() + ch * T;
        sum[ch] = gpdb_org_window(t[lr], t[ul], t[ur], t[ll]);
      }
      float cov[3][3], ev;
      gpdb_org_covariance(sum, sum + 3, count, cov);
      gpdo_pcl_eigen33(&cov[0][0], &ev, n);
      gpdb_org_flip(q, vp, n);
    }
}

// rule 6: camera-frame normals rotated by R (row-major 3 x 3), finite or not
extern "C" void org_oracle_rotate(int n, const double *R, const float *nc, float *nw) {
  for (int i = 0; i < n; i++) gpdb_org_rotate(R, nc + 3 * i, nw + 3 * i);
}
