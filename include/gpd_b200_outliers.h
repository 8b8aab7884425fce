/*
 * gpd_b200_outliers.h — SPECIFICATION of the statistical outlier removal on the device (gpdb_remove_outliers,
 * gpdb_remove_outliers_clouds); the entry points are declared in gpd_b200.h.
 *
 * Cloud::removeStatisticalOutliers (cloud.cpp:166-174) runs pcl::StatisticalOutlierRemoval with setMeanK(50) and
 * setStddevMulThresh(1.0) on the processed cloud. This file restates PCL 1.9.1's applyFilterIndices rule by rule. The
 * rules are recalled from PCL's published statistical_outlier_removal.hpp; the details marked UNPINNED AGAINST UPSTREAM
 * BINARIES below could not be checked against a PCL build (DESIGN.md 6c names every departure). Every float32 and
 * float64 operation is rounded on its own, with no FMA.
 *
 * Cloud b of a call has N points (cloud-local indices i = 0..N-1, float32 coordinates as installed; every installed point
 * is finite, installs reject the others). Parameters: mean_k (1..GPDB_OUTLIERS_MAX_K) and stddev_mul (finite).
 *
 *  1. Neighbours (nearestKSearch(i, mean_k + 1)). The mean_k + 1 smallest keys of gpd_b200_refine.h rule 1
 *     ((bits of gpdb_refine_l2, index), ties by index, no radius bound). The point itself is one of them, at distance 0.
 *  2. Mean distance. With l2_1 <= ... <= l2_{k+1} the key distances in ascending order (k = mean_k),
 *     dist_sum = ((0 + sqrtf(l2_2)) + sqrtf(l2_3)) + ... + sqrtf(l2_{k+1}) in double, each float32 root widened and added
 *     (gpdb_outlier_dist_add), and d_i = (float)(dist_sum / mean_k) (gpdb_outlier_mean). Entry 1 is skipped: it is 0,
 *     the point itself or a duplicate of it. The sequence l2_1..l2_{k+1} is the same whichever way ties are broken, so
 *     d_i does not depend on the tie-break. UNPINNED: that PCL's unqualified sqrt of a float resolves to the float
 *     overload; the contract fixes sqrtf.
 *  3. Cloud statistics. Two double sums, each one sequential chain in index order, as PCL's loop runs:
 *     sum += d_i and sq_sum += (float)(d_i * d_i) (the product rounded in float32, then widened; gpdb_outlier_stats_add).
 *     Then, with n = N: mean = sum / n, variance = (sq_sum - sum * sum / n) / (n - 1), stddev = sqrt(variance),
 *     threshold = mean + stddev_mul * stddev (gpdb_outlier_stats). A variance made negative by cancellation gives a NaN
 *     stddev and threshold, and rule 4 then keeps every point, as PCL does. UNPINNED: the float32 product of sq_sum
 *     (distances is a std::vector<float>), and PCL >= 1.9's search of mean_k + 1 neighbours with the first skipped
 *     (older releases searched mean_k and kept the zero).
 *  4. Decision. Point i is removed iff (double)d_i > threshold (strict; gpdb_outlier_removed): a point exactly at the
 *     threshold stays.
 *  5. Small clouds. DEPARTURE: when N <= mean_k, PCL reads past the neighbour lists (undefined behaviour). The contract
 *     keeps every point and reports NaN for mean, stddev and threshold. A cloud without points stays empty (NaN too).
 *  6. Output. The kept points in their original order, with their normals, camera masks and source indices.
 *
 * tests/outliers_reference.py restates this file in numpy.
 */
#ifndef GPD_B200_OUTLIERS_H_
#define GPD_B200_OUTLIERS_H_

#include <math.h>
#include <stdint.h>

#include "gpd_b200_refine.h" /* rule 1: gpdb_refine_l2, GPDB_HD */

/* largest mean_k: the lists take N * (mean_k + 1) int32 of device memory, within the refinement's N * 128 */
#define GPDB_OUTLIERS_MAX_K (GPDB_REFINE_MAX_K - 1)

/* rule 2: one neighbour's distance added to the running double sum */
GPDB_HD double gpdb_outlier_dist_add(double dist_sum, float l2) { return dist_sum + (double)sqrtf(l2); }

/* rule 2: the point's mean distance from the sum over its mean_k neighbours */
GPDB_HD float gpdb_outlier_mean(double dist_sum, int mean_k) { return (float)(dist_sum / (double)mean_k); }

/* rule 3: one point's mean distance added to the two running sums */
GPDB_HD void gpdb_outlier_stats_add(double *sum, double *sq_sum, float d) {
  *sum = *sum + (double)d;
  *sq_sum = *sq_sum + (double)(d * d);
}

/* rules 3 and 5: out = {mean, stddev, threshold} of a cloud of n points; NaN when n <= mean_k */
GPDB_HD void gpdb_outlier_stats(double sum, double sq_sum, int n, int mean_k, double stddev_mul, double out[3]) {
  if (n <= mean_k) {
    out[0] = out[1] = out[2] = NAN;
    return;
  }
  const double dn = (double)n;
  const double mean = sum / dn;
  const double variance = (sq_sum - sum * sum / dn) / (dn - 1.0);
  const double stddev = sqrt(variance);
  out[0] = mean;
  out[1] = stddev;
  out[2] = mean + stddev_mul * stddev;
}

/* rule 4: a NaN threshold removes nothing */
GPDB_HD bool gpdb_outlier_removed(float d, double threshold) { return (double)d > threshold; }

#endif /* GPD_B200_OUTLIERS_H_ */
