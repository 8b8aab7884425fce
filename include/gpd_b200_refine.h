/*
 * gpd_b200_refine.h — SPECIFICATION of the normal refinement on the device (gpdb_refine_normals,
 * gpdb_refine_normals_clouds); the entry points are declared in gpd_b200.h.
 *
 * Cloud::refineNormals(k) (cloud.cpp:176-204) runs after calculateNormals when refine_normals_k > 0: a
 * pcl::search::KdTree k-nearest-neighbour search over the processed cloud, then pcl::NormalRefinement<pcl::Normal> with
 * its default settings. This file restates both step by step. Every float32 operation is rounded on its own, with no
 * FMA. The NormalRefinement details are recalled from PCL 1.9.1's published normal_refinement.h/.hpp; the ones marked
 * UNPINNED AGAINST UPSTREAM BINARIES below could not be read from that source (DESIGN.md 6c names every departure).
 *
 * Cloud b of a call has N points (cloud-local indices j = 0..N-1, float32 coordinates p_j as installed, float64 normals
 * as installed). Every point takes part, whatever its camera; each cloud is refined on its own.
 *
 *  1. Neighbour lists (nearestKSearch(cloud, {}, k)). key(i, j) = (bits of l2_simple(p_i, p_j), j), l2_simple the FLANN
 *     L2_Simple<float> distance ((dx*dx + dy*dy) + dz*dz) with d = p_i - p_j (gpdb_refine_l2). The list of point i is
 *     the L = min(k, N) points j with the smallest keys, in ascending key order: nearest first, ties by index. Point i is
 *     in its own list at distance 0 (first unless an earlier index shares its coordinates). The tie-break by index is
 *     FLANN's behaviour as SURVEY 9.7 assumes it for the radius searches (unpinned).
 *  2. Input normals: m0_j = (float)n_j per component (normals_.col(j).cast<float>()).
 *  3. Iteration t = 1, 2, ... (refineNormal, Jacobi: every point from the previous iterate m_{t-1}). For point i, the
 *     sums (sx, sy, sz) start at 0.0f and add the neighbours' normals in list order, each weighted by 1.0f
 *     (assignNormalWeights' uniform default; a product by 1.0f is exact, so it is left out); a neighbour whose normal has
 *     a non-finite component is skipped. norm = sqrtf((sx*sx + sy*sy) + sz*sz); m_t,i = (sx/norm, sy/norm, sz/norm) when
 *     norm is finite and norm > FLT_EPSILON, else NaN in all three (gpdb_refine_normal). The pairing of the squared
 *     terms is unpinned.
 *  4. Stop statistic (applyFilter's convergence test, convergence_threshold_ = 1e-5f). The error of point i is
 *     e_i = acos(clamp(dot, -1, 1)), dot = ((o.x*m.x + o.y*m.y) + o.z*m.z) of its previous normal o = m_{t-1},i and its
 *     new normal m = m_t,i, and e_i = 0 when either has a non-finite component (gpdb_refine_error). The mean is the
 *     float32 sum s = ((0 + e_0) + e_1) + ... in index order (std::accumulate), divided by (float)N. The loop stops after
 *     iteration t when mean < 1e-5f, and after iteration GPDB_REFINE_MAX_ITERATIONS in any case. Unpinned: that the error
 *     is this angle (in radians) and not another difference measure, the clamp, and the zero for non-finite normals.
 *     Departure: PCL calls the host libm acosf, which a device cannot reproduce bit for bit; the contract replaces it by
 *     gpdb_refine_acosf, a fixed sequence of float32 operations (the Cephes asinf polynomial) that the oracles and the
 *     kernels share. It is within a few ulp of acos.
 *  5. Output: the normals of the last iteration run, cast to double (reverseNormals is not applied again); the count of
 *     iterations run (1..15; 0 for a cloud without points, whose applyFilter returns at once).
 *
 * tests/refine_reference.py restates this file in numpy, tests/refine_oracle.cpp in C++.
 */
#ifndef GPD_B200_REFINE_H_
#define GPD_B200_REFINE_H_

#include <float.h>
#include <math.h>
#include <stdint.h>

#include "gpd_b200_shadow.h" /* GPDB_HD */

#define GPDB_REFINE_MAX_K 128           /* largest k: the lists take N * k int32 of device memory */
#define GPDB_REFINE_MAX_ITERATIONS 15   /* NormalRefinement's default max_iterations_            */
#define GPDB_REFINE_CONVERGENCE 1e-5f   /* NormalRefinement's default convergence_threshold_     */

/* rule 1: FLANN L2_Simple<float> between points a and b */
GPDB_HD float gpdb_refine_l2(const float a[3], const float b[3]) {
  const float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  float d = dx * dx;
  d = d + dy * dy;
  d = d + dz * dz;
  return d;
}

GPDB_HD bool gpdb_refine_finite3(const float n[3]) { return isfinite(n[0]) && isfinite(n[1]) && isfinite(n[2]); }

/* rule 3: the refined normal from the neighbour sums */
GPDB_HD void gpdb_refine_normal(float sx, float sy, float sz, float out[3]) {
  const float norm = sqrtf((sx * sx + sy * sy) + sz * sz);
  if (isfinite(norm) && norm > FLT_EPSILON) {
    out[0] = sx / norm;
    out[1] = sy / norm;
    out[2] = sz / norm;
  } else {
    out[0] = out[1] = out[2] = NAN;
  }
}

/* rule 4: acos of x in [-1, 1] as a fixed sequence of float32 operations. Cephes' asinf polynomial
 * P(z) = (((c4 z + c3) z + c2) z + c1) z + c0 gives asin(s) = s + (P(z) z) s with z = s*s for s <= 0.5; above 0.5,
 * acos(a) = 2 asin(sqrt((1 - a) / 2)), and acos(-a) = pi - acos(a). */
GPDB_HD float gpdb_refine_acosf(float x) {
  const float a = fabsf(x);
  float s, z;
  if (a > 0.5f) {
    z = 0.5f * (1.0f - a);
    s = sqrtf(z);
  } else {
    s = a;
    z = a * a;
  }
  float p = 4.2163199048e-2f * z + 2.4181311049e-2f;
  p = p * z + 4.5470025998e-2f;
  p = p * z + 7.4953002686e-2f;
  p = p * z + 1.6666752422e-1f;
  const float r = s + (p * z) * s;  // asin(s)
  if (a > 0.5f) {
    const float t = r + r;  // acos(a)
    return x < 0.0f ? 3.14159265358979f - t : t;
  }
  return x < 0.0f ? 1.57079632679490f + r : 1.57079632679490f - r;
}

/* rule 4: the error of one point between its previous normal o and its new normal m */
GPDB_HD float gpdb_refine_error(const float o[3], const float m[3]) {
  if (!gpdb_refine_finite3(o) || !gpdb_refine_finite3(m)) return 0.0f;
  float d = (o[0] * m[0] + o[1] * m[1]) + o[2] * m[2];
  d = fminf(fmaxf(d, -1.0f), 1.0f);
  return gpdb_refine_acosf(d);
}

#endif /* GPD_B200_REFINE_H_ */
