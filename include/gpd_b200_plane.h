/*
 * gpd_b200_plane.h — SPECIFICATION of the support-plane segmentation on the device (gpdb_segment_plane,
 * gpdb_segment_planes[_device]); the entry points and gpdb_plane_params are declared in gpd_b200.h.
 *
 * Cloud::sampleAbovePlane (cloud.cpp:407-435) fits the table plane with pcl::SACSegmentation (SACMODEL_PLANE, SAC_RANSAC,
 * setDistanceThreshold(0.01), setOptimizeCoefficients(true)) and keeps only the points off that plane as sample
 * candidates. This file restates PCL 1.9.1's published algorithm step by step, with its random draws replaced by
 * counter-based ones. The defaults and the PCL details are recalled from the published algorithm and are UNPINNED AGAINST
 * UPSTREAM BINARIES (DESIGN.md 6c names every departure). Every operation is rounded on its own, with no FMA.
 *
 * Cloud b of a call has N points (cloud-local indices j = 0..N-1, float32 coordinates as installed); key = seed + b.
 *
 *  1. Sample draw (SampleConsensusModel::getSamples / drawIndexSample). Hypothesis h, attempt a (0 <= a < 1000, PCL's
 *     max_sample_checks_) draws c = gpdb_plane_draw(key, h, a) = philox({h, a, 3, 0}, key); stream word 3 keeps these
 *     draws apart from SIS (0, 1) and subsampling (2). The three indices are a partial Fisher-Yates shuffle of the
 *     identity permutation of 0..N-1 with r0 = c.x % N, r1 = c.y % (N-1), r2 = c.z % (N-2) (gpdb_plane_sample). PCL
 *     shuffles a persistent permutation instead of starting from the identity each time: a departure.
 *  2. Good sample and coefficients (isSampleGood / computeModelCoefficients, gpdb_plane_model), float32:
 *     p1p0 = p1 - p0, p2p0 = p2 - p0; the sample is bad iff p1p0.x/p2p0.x == p1p0.y/p2p0.y and p1p0.z/p2p0.z ==
 *     p1p0.y/p2p0.y (NaN compares unequal); n = (p1p0.y*p2p0.z - p1p0.z*p2p0.y, p1p0.z*p2p0.x - p1p0.x*p2p0.z,
 *     p1p0.x*p2p0.y - p1p0.y*p2p0.x); s = sqrtf((n.x*n.x + n.y*n.y) + n.z*n.z) and n /= s when s > 0; d =
 *     -((n.x*p0.x + n.y*p0.y) + n.z*p0.z). The guard s > 0 is a deliberate amendment of an unconditional n /= s: Eigen's
 *     normalize leaves a zero vector as it is, so a "good" triple with a zero normal (three points of one lattice row,
 *     whose coordinate ratios are NaN) counts every point as an inlier, as in PCL, instead of none. The pairing of the
 *     squared terms, and whether PCL's 4-vector squared norm adds its zero w term, are unpinned. Hypothesis h takes its
 *     first good attempt; when all 1000 attempts are bad the loop of rule 4 ends before h. The same predicate guards
 *     computeModelCoefficients, so PCL's skip counter never moves.
 *  3. Distance (countWithinDistance / selectWithinDistance, gpdb_plane_dist): dist = fabsf(((a*x + b*y) + c*z) + d) in
 *     float32; a point is an inlier iff (double)dist < distance_threshold. PCL's vectorised dot may round its last bit
 *     differently: only points within an ulp of the threshold can tell (unpinned).
 *  4. Loop (RandomSampleConsensus::computeModel). Hypotheses h = 0, 1, ... are evaluated, at most max_iterations + 1 of
 *     them. h becomes the best when its inlier count is strictly larger than the best so far (h = 0 always does). After
 *     each new best, w = n_best * (1.0 / N) and q = 1 - (w*w)*w in float64, clamped to [DBL_EPSILON, 1 - DBL_EPSILON].
 *     After h the loop stops when h + 1 > max_iterations or unless q^(h+1) > 1 - probability, q^(h+1) being h + 1
 *     sequential float64 multiplications (1 * q * q * ...). PCL's test is iterations < log(1 - p) / log(q): the same
 *     inequality up to rounding, written without log or pow (a departure). N < 3: no hypothesis, the fit fails.
 *  5. Refit (SampleConsensusModelPlane::optimizeModelCoefficients, PCL 1.9.1). Input: the inliers of the best hypothesis
 *     in index order. More than 3 of them: computeMeanAndCovarianceMatrix as one float32 pass in index order (accu[0..8]
 *     = xx, xy, xz, yy, yz, zz, x, y, z, each product rounded before it is added, then accu /= (float)count, cov = accu -
 *     centroid products, as k_normals and DESIGN.md 4b), the smallest eigenvector of pcl::eigen33 (k_normals' restatement)
 *     as n, and d = -((n.x*cx + n.y*cy) + n.z*cz) with the centroid c. 3 or fewer: the hypothesis' coefficients stay.
 *     The final inliers are the points within the threshold of the refined plane (rule 3).
 *  6. Output (sampleAbovePlane). plane[b] = (a, b, c, d) float32, all NaN when the fit failed; n_inliers[b] = the final
 *     inliers (0 when the fit failed); eligible[j] = 1 for every point that is not a final inlier, and 1 for every point
 *     of a cloud whose fit failed or that has no point off the plane (cloud.cpp:427-433). n_hypotheses[b] = hypotheses
 *     evaluated (0 when N < 3 or hypothesis 0 found no good sample). A cloud's result depends only on (key, its points,
 *     the parameters).
 *
 * tests/plane_reference.py restates this file in numpy, tests/plane_oracle.cpp in C++.
 */
#ifndef GPD_B200_PLANE_H_
#define GPD_B200_PLANE_H_

#include <stdint.h>

#include "gpd_b200_sis.h" /* gpdb_philox4x32_10, GPDB_HD */

#define GPDB_PLANE_STREAM 3u          /* the stream word of the sample draws                */
#define GPDB_PLANE_SAMPLE_CHECKS 1000 /* attempts per hypothesis (PCL's max_sample_checks_) */
#define GPDB_PLANE_MAX_ITERATIONS 1024

/* rule 1: the draw of attempt a of hypothesis h for the cloud whose key is seed + b */
GPDB_HD gpdb_u32x4 gpdb_plane_draw(uint64_t key, uint32_t h, uint32_t a) {
  const gpdb_u32x4 c = {h, a, GPDB_PLANE_STREAM, 0u};
  return gpdb_philox4x32_10(c, (uint32_t)key, (uint32_t)(key >> 32));
}

/* rule 1: the first three entries of the identity permutation of 0..n-1 (n >= 3) after the swaps (0, r0), (1, 1 + r1),
 * (2, 2 + r2). Position 1 + r1 >= 1 still holds its own value unless it is r0 (then 0); position 2 + r2 holds what the
 * second swap left there, or 0 when it is r0, or its own value. */
GPDB_HD void gpdb_plane_sample(gpdb_u32x4 c, uint32_t n, uint32_t idx[3]) {
  const uint32_t r0 = c.x % n, j1 = 1u + c.y % (n - 1u), j2 = 2u + c.z % (n - 2u);
  const uint32_t left1 = r0 == 1u ? 0u : 1u;  // the value the second swap moves to position j1
  idx[0] = r0;
  idx[1] = j1 == r0 ? 0u : j1;
  idx[2] = j2 == j1 ? left1 : (j2 == r0 ? 0u : j2);
}

/* rule 2: false for a bad sample; else the normalised coefficients */
GPDB_HD bool gpdb_plane_model(const float p0[3], const float p1[3], const float p2[3], float coef[4]) {
  const float ax = p1[0] - p0[0], ay = p1[1] - p0[1], az = p1[2] - p0[2];
  const float bx = p2[0] - p0[0], by = p2[1] - p0[1], bz = p2[2] - p0[2];
  const float rx = ax / bx, ry = ay / by, rz = az / bz;
  if (rx == ry && rz == ry) return false;
  float n0 = ay * bz - az * by, n1 = az * bx - ax * bz, n2 = ax * by - ay * bx;
  const float s = sqrtf((n0 * n0 + n1 * n1) + n2 * n2);
  if (s > 0.0f) {
    n0 = n0 / s;
    n1 = n1 / s;
    n2 = n2 / s;
  }
  coef[0] = n0;
  coef[1] = n1;
  coef[2] = n2;
  coef[3] = -((n0 * p0[0] + n1 * p0[1]) + n2 * p0[2]);
  return true;
}

/* rule 3: the distance of (x, y, z) from the plane coef */
GPDB_HD float gpdb_plane_dist(const float coef[4], float x, float y, float z) {
  return fabsf(((coef[0] * x + coef[1] * y) + coef[2] * z) + coef[3]);
}

#endif /* GPD_B200_PLANE_H_ */
