/*
 * gpd_b200_organized.h — SPECIFICATION of the integral-image normal estimation of organized clouds on the device
 * (gpdb_normals_organized[_device], gpdb_preprocess_depth_organized[_device]); the entry points are declared in
 * gpd_b200.h.
 *
 * Cloud::calculateNormalsOrganized (cloud.cpp:479-495) runs pcl::IntegralImageNormalEstimation with COVARIANCE_MATRIX,
 * setNormalSmoothingSize(20.0f) and PCL's defaults otherwise: max_depth_change_factor_ = 0.02f, BORDER_POLICY_IGNORE, no
 * depth-dependent smoothing. This file restates PCL 1.9.1's integral_image_normal.hpp and integral_image2D.hpp rule by
 * rule. The rules are recalled from PCL's published source; EVERY rule below is UNPINNED AGAINST UPSTREAM BINARIES (no
 * PCL build was available to check them against; DESIGN.md 6c names every departure). Every float32 and float64
 * operation is rounded on its own, with no FMA.
 *
 *  1. Input. An organized cloud of W x H float32 points, row-major (pixel (r, c) is point r * W + c). A missing point
 *     has NaN coordinates. The view point is float32 (setViewPoint takes floats).
 *  2. Depth-change map. Every pixel starts at 1. For each pixel (r, c) with r < H-1 and c < W-1, with z its depth and
 *     t = (0.02f * (fabsf(z) + 1.0f)) * 2.0f: if fabsf(z - z_right) > t or either z is not finite, both pixels become 0
 *     (gpdb_org_pair_breaks); the same test against the pixel below. The result does not depend on evaluation order.
 *  3. Distance map (a float32 chamfer). 0 where the change map is 0, else (float)(W + H). Pass 1: rows 1..H-1 ascending,
 *     columns 1..W-1 ascending, m = min(min(UL + 1.4f, U + 1.0f), min(L + 1.0f, UR + 1.4f)), stored when m < centre
 *     (gpdb_org_chamfer). Pass 2: rows H-2..0 descending, columns W-2..0 descending, the same form over lower-left,
 *     lower, right and lower-right. PCL indexes one flat array, so the edge neighbours wrap: in pass 1 the UR of the last
 *     column is element 0 of the current row (which pass 1 never updates); in pass 2 the lower-left of column 0 is the
 *     last element of the current row (which pass 2 never updates). These sequential float32 passes are the
 *     specification.
 *  4. Integral images (float64). (W+1) x (H+1) tables with row 0 and column 0 zero:
 *     I[r+1][c+1] = ((I[r][c+1] + I[r+1][c]) - I[r][c]) (gpdb_org_integral), then, when the float32 sum (x + y) + z is
 *     finite (gpdb_org_finite_point), += (double) of each coordinate, += (double) of the six float32 products xx, xy,
 *     xz, yy, yz, zz, and the integer count += 1. The window sum over [x0, x0+w) x [y0, y0+h) is
 *     ((I[lr] + I[ul]) - I[ur]) - I[ll] (gpdb_org_window). The double sums are not exact, so this order is the
 *     specification.
 *  5. Per pixel. Pixels within GPDB_ORG_BORDER = 20 of any image edge are NaN; an image with W <= 40 or H <= 40 is all
 *     NaN. DEPARTURE: PCL's unsigned loop bounds write out of range for W < 20 or H < 20. Otherwise the normal is NaN
 *     when z is not finite, when s = min(dist, 20.0f) is not > 2.0f, or when the window count is 0. Else w = (int)s, the
 *     window starts at (c - w/2, r - w/2) (integer division) and is w x w, centre_i = (float) first-order sum i (not
 *     divided by the count), C_ij = (float)so_ij - (centre_i * centre_j) / (float)count (gpdb_org_covariance), the
 *     normal is pcl::eigen33's smallest eigenvector of C (the solver k_normals uses), flipped towards the view point in
 *     float32 as flipNormalTowardsViewpoint does (gpdb_org_flip). The output is float32; no curvature.
 *  6. Depth views. Camera k's organized cloud is its pixels in the CAMERA frame: (xc, yc, zc) of gpd_b200_depth.h rule
 *     2 for a valid pixel, NaN for an invalid one; the view point is the origin. The workspace filter does not apply:
 *     PCL sees the whole image, and the z of the depth-change test is depth. The normal goes to the world frame by the
 *     pose's R: n_i = (float)(((R_i0 * nx + R_i1 * ny) + R_i2 * nz)) in double, one rounding (gpdb_org_rotate).
 *  7. Processed point p of a depth view. Its representative pixel is the voxel's first point (src of gpdb_get_clouds),
 *     or the pixel itself when voxelize = 0. When that pixel's world normal is finite, p's normal is it, widened to
 *     double, then the float64 reverseNormals test at p with p's camera mask, as k_normals applies it. Otherwise p is a
 *     fallback: its normal is exactly the one gpdb_preprocess_depth gives p (the radius estimate). Points, camera
 *     sources, source indices and offsets equal gpdb_preprocess_depth's on the same call bit for bit.
 *
 * tests/organized_reference.py restates this file in numpy, tests/organized_oracle.cpp in C++ over these helpers.
 */
#ifndef GPD_B200_ORGANIZED_H_
#define GPD_B200_ORGANIZED_H_

#include <math.h>
#include <stdint.h>

#include "gpd_b200_shadow.h" /* GPDB_HD */

#define GPDB_ORG_BORDER 20      /* (int)normal_smoothing_size_, BORDER_POLICY_IGNORE */
#define GPDB_ORG_SMOOTHING 20.0f /* setNormalSmoothingSize(20.0f) (cloud.cpp:485) */

/* rule 2: the pair (a, b), a the pixel the loop stands on, breaks the surface */
GPDB_HD bool gpdb_org_pair_breaks(float a, float b) {
  const float t = (0.02f * (fabsf(a) + 1.0f)) * 2.0f;
  return fabsf(a - b) > t || !isfinite(a) || !isfinite(b);
}

/* rule 3: min(min(d0 + 1.4f, d1 + 1.0f), min(d2 + 1.0f, d3 + 1.4f)); pass 1: (UL, U, L, UR), pass 2: (LL, Lo, R, LR) */
GPDB_HD float gpdb_org_chamfer(float diag0, float straight0, float straight1, float diag1) {
  const float a = diag0 + 1.4f, b = straight0 + 1.0f, c = straight1 + 1.0f, d = diag1 + 1.4f;
  const float m0 = b < a ? b : a, m1 = d < c ? d : c; /* std::min(x, y): y if y < x, else x */
  return m1 < m0 ? m1 : m0;
}

/* rule 4: the recurrence before the pixel's own terms, I[r+1][c+1] from up = I[r][c+1], left = I[r+1][c], ul = I[r][c] */
GPDB_HD double gpdb_org_integral(double up, double left, double ul) { return (up + left) - ul; }

/* rule 4: a point counts when the float32 sum (x + y) + z is finite */
GPDB_HD bool gpdb_org_finite_point(const float p[3]) { return isfinite((p[0] + p[1]) + p[2]); }

/* rule 4: the window sum from the four corners */
GPDB_HD double gpdb_org_window(double lr, double ul, double ur, double ll) { return ((lr + ul) - ur) - ll; }

/* rule 5: the covariance matrix from the window's first-order sums s[3], second-order sums so[6] (xx xy xz yy yz zz)
 * and count */
GPDB_HD void gpdb_org_covariance(const double s[3], const double so[6], int count, float cov[3][3]) {
  const float c[3] = {(float)s[0], (float)s[1], (float)s[2]};
  const float n = (float)count;
  const int ij[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
  for (int e = 0; e < 6; e++) {
    const int i = ij[e][0], j = ij[e][1];
    cov[i][j] = cov[j][i] = (float)so[e] - (c[i] * c[j]) / n;
  }
}

/* rule 5: flipNormalTowardsViewpoint in float32 */
GPDB_HD void gpdb_org_flip(const float p[3], const float vp[3], float n[3]) {
  const float vx = vp[0] - p[0], vy = vp[1] - p[1], vz = vp[2] - p[2];
  const float cos_theta = vx * n[0] + vy * n[1] + vz * n[2];
  if (cos_theta < 0) {
    n[0] *= -1;
    n[1] *= -1;
    n[2] *= -1;
  }
}

/* rule 6: the camera-frame normal n in the world frame (R row-major 3 x 3) */
GPDB_HD void gpdb_org_rotate(const double R[9], const float n[3], float out[3]) {
  for (int i = 0; i < 3; i++)
    out[i] = (float)(((R[3 * i] * (double)n[0] + R[3 * i + 1] * (double)n[1]) + R[3 * i + 2] * (double)n[2]));
}

#endif /* GPD_B200_ORGANIZED_H_ */
