/*
 * gpd_b200_sensor.h — SPECIFICATION of the structured-light sensor model of gpdb_render_sensor_depth[_device] (declared in
 * gpd_b200.h): the depth images gpdb_render_depth renders, seen as a projector-camera sensor (a PrimeSense, the sensor of
 * the BigBird captures the reference trained on) sees them. Three artefacts of such a sensor shape GPD's inputs: no return
 * where the projector cannot see the surface (a band beside every occluding edge), no return at grazing angles, and depth
 * quantised in disparity (a step that grows with z^2). Every operation is rounded on its own, with no FMA. The parameters
 * are one gpdb_sensor_params per call (gpd_b200.h); gpdb_sensor_params_default sets every field to 0, and with every field
 * 0 the call equals gpdb_render_depth bit for bit.
 *
 * For pixel (u, v) of camera k (0-based within its view) of view b; "no return" writes the no-hit value of
 * gpd_b200_render.h rule 5 (raw 0) and the face -1.
 *
 *  1. Draws. r_w = philox({v*width + u, k, GPDB_SENSOR_STREAM, w}, key) for w = 0 and 1, key = seed + b split as in
 *     gpd_b200_depth.h rule 5 (gpdb_sensor_draw). Stream word 5 keeps these draws apart from SIS (0, 1), subsampling (2),
 *     the plane fit (3) and the mesh samples (4). Uniforms are built from word pairs as gpdb_mesh_unit builds them:
 *     g0 from (r_0.x, r_0.y), g1 from (r_0.z, r_0.w), g2 from (r_1.x, r_1.y) through rule 2, and U = unit(r_1.z, r_1.w).
 *     View b's images depend only on seed + b, its mesh and its cameras, not on the batch it is rendered in.
 *  2. Gaussian draws without device transcendentals (the device's log and cos are not the host's). T is a float64
 *     inverse-normal table of GPDB_SENSOR_TABLE = 4097 entries: T[i] = Phi^-1(i / 4096) for 1 <= i <= 2047, found by
 *     bisection on 0.5*erfc(-x/sqrt(2)) in the host's libm; T[2048] = 0; T[4096 - i] = -T[i] (exact odd symmetry);
 *     T[0] = T[1] and T[4096] = T[4095] (the infinite ends clamped to their neighbours). The library builds it once on
 *     the host (gpdb_sensor_table_build) and gpdb_debug_sensor_table exports it. The draw of a uniform U in [0, 1) is
 *     s = U*4096, i = floor(s), f = s - i, g = T[i] + f*(T[i+1] - T[i]) (gpdb_sensor_gauss). Consequence: draws are
 *     truncated at |g| <= T[4095] = 3.4871 (about 3.5 sigma), and their standard deviation is that of the table's
 *     piecewise-linear distribution (0.99957), not exactly 1.
 *  3. Lateral jitter. The pixel reads (u', v') = (u + rint(lateral_sigma*g0), v + rint(lateral_sigma*g1)) (in float64;
 *     rint is half to even). Outside the image: no return. There it reads the clean hit (t, face) of gpd_b200_render.h
 *     rules 2-5, t in float64 before the format conversion; no hit: no return. The surface point in the camera frame is
 *     X = (t*dx, t*dy, t), (dx, dy) the ray of (u', v') by render rule 3.
 *  4. Grazing angle (only when min_cos_incidence > 0). n = the face's world normal by render rule 1 in float64 from its
 *     float32 vertices (n = (b - a) x (c - a)), rotated into the camera frame by R^T in render rule 2's operand order
 *     without the translation: m_i = (R0i*n.x + R1i*n.y) + R2i*n.z. c = |m.X| / (sqrt(m.m)*sqrt(X.X)), each dot product
 *     (a.x*b.x + a.y*b.y) + a.z*b.z. If c < min_cos_incidence: no return (a NaN c, from a face of zero area, passes).
 *  5. Projector shadow (only when baseline > 0). The projector is a pinhole with the camera's intrinsics and size; its
 *     pose is the camera's with the translation t_i + baseline*R_i0 in float64 (gpdb_sensor_projector_pose), and its clean
 *     image is rendered by the same rules. X_p = (X.x - baseline, X.y, X.z) lands on (pu, pv) = (rint((fx*X_p.x)/X.z + cx),
 *     rint((fy*X_p.y)/X.z + cy)). No return if (pu, pv) lies outside the image, the projector has no hit there, or its
 *     hit t_p < X.z*(1 - shadow_tolerance). The projector shares the camera's z axis, so t_p and X.z are both depths.
 *  6. Disparity (only when baseline > 0). D = (fx*baseline)/X.z, D' = D + disparity_sigma*g2; if disparity_step > 0,
 *     D' = disparity_step*rint(D'/disparity_step). If D' <= 0 or D' is not finite: no return; else z' = (fx*baseline)/D'.
 *     Without a baseline z' = X.z (= t).
 *  7. Dropout. If U < dropout: no return.
 *  8. Output. The stored value of z' by render rule 5 (F32 or U16), in the layout gpdb_render_depth writes; the optional
 *     face image holds the face of the hit that was read, or -1 wherever the pixel is not a return. min_depth and
 *     max_depth are left to preprocessing, as for the render.
 *  9. Errors (GPDB_ERR_INVALID with a message; nothing is written): every error of render rule 7; a parameter that is
 *     negative or not finite; dropout > 1; shadow_tolerance >= 1; min_cos_incidence > 1; disparity_sigma or
 *     disparity_step > 0 with baseline = 0.
 *
 * Rules 3-7 run in this order and stop at the first "no return" (gpdb_sensor_pixel), so the draws are made for every
 * pixel whether or not they are used. tests/sensor_reference.py restates this file in numpy float64, bit for bit.
 */
#ifndef GPD_B200_SENSOR_H_
#define GPD_B200_SENSOR_H_

#include <math.h>
#include <stdint.h>

#include "gpd_b200_render.h" /* gpdb_render_*, gpdb_mesh_unit, gpdb_philox4x32_10, gpdb_sensor_params, GPDB_HD */

/* the stream word of the sensor draws (SIS 0 and 1, subsampling 2, plane fit 3, mesh samples 4) */
#define GPDB_SENSOR_STREAM 5u
/* rule 2: the entries of the inverse-normal table */
#define GPDB_SENSOR_TABLE 4097

/* rule 2: the table, built on the host (libm's erfc) */
static inline void gpdb_sensor_table_build(double T[GPDB_SENSOR_TABLE]) {
  for (int i = 1; i < 2048; i++) {
    const double p = (double)i / 4096.0;
    double lo = -40.0, hi = 0.0;  // 0.5*erfc(-x/sqrt(2)) < p at lo, >= p at hi
    for (;;) {
      const double mid = 0.5 * (lo + hi);
      if (!(mid > lo && mid < hi)) break;
      if (0.5 * erfc(-mid * 0.70710678118654752440) < p) lo = mid;
      else hi = mid;
    }
    const double elo = p - 0.5 * erfc(-lo * 0.70710678118654752440), ehi = 0.5 * erfc(-hi * 0.70710678118654752440) - p;
    T[i] = elo < ehi ? lo : hi;
    T[4096 - i] = -T[i];
  }
  T[2048] = 0.0;
  T[0] = T[1];
  T[4096] = T[4095];
}

/* rule 1: draw w (0 or 1) of pixel index pix (v*width + u) of camera k of the view whose key is seed + b */
GPDB_HD gpdb_u32x4 gpdb_sensor_draw(uint64_t key, uint32_t pix, uint32_t k, uint32_t w) {
  const gpdb_u32x4 c = {pix, k, GPDB_SENSOR_STREAM, w};
  return gpdb_philox4x32_10(c, (uint32_t)key, (uint32_t)(key >> 32));
}

/* rule 2: the Gaussian draw of the uniform U in [0, 1) */
GPDB_HD double gpdb_sensor_gauss(const double *T, double U) {
  const double s = U * 4096.0;
  const int i = (int)s;
  const double f = s - (double)i;
  return T[i] + f * (T[i + 1] - T[i]);
}

/* rule 5: the projector's pose (camera-to-world, row-major 3 x 4) of the camera pose `pose` */
GPDB_HD void gpdb_sensor_projector_pose(const double pose[12], double baseline, double out[12]) {
  for (int e = 0; e < 12; e++) out[e] = pose[e];
  for (int i = 0; i < 3; i++) out[4 * i + 3] = pose[4 * i + 3] + baseline * pose[4 * i];
}

/* rules 1 and 3-7 for pixel (u, v) of a W x H camera (intrinsics fx, fy, cx, cy, pose `pose`), camera k of the view
 * whose key is seed + b. ct / cf: the camera's clean image (t, face; face -1 where there is no hit), row-major; pt / pf:
 * the projector's (read only when baseline > 0); vtx / faces: the view's vertices and faces. Returns the face of the hit
 * read, *z receiving z', or -1 for no return. */
GPDB_HD int gpdb_sensor_pixel(const gpdb_sensor_params *s, const double *T, uint64_t key, uint32_t k, int u, int v,
                              int W, int H, double fx, double fy, double cx, double cy, const double pose[12],
                              const double *ct, const int *cf, const double *pt, const int *pf, const float *vtx,
                              const int *faces, double *z) {
  // rule 1
  const gpdb_u32x4 r0 = gpdb_sensor_draw(key, (uint32_t)v * (uint32_t)W + (uint32_t)u, k, 0u);
  const gpdb_u32x4 r1 = gpdb_sensor_draw(key, (uint32_t)v * (uint32_t)W + (uint32_t)u, k, 1u);
  const double g0 = gpdb_sensor_gauss(T, gpdb_mesh_unit(r0.x, r0.y)), g1 = gpdb_sensor_gauss(T, gpdb_mesh_unit(r0.z, r0.w));
  const double g2 = gpdb_sensor_gauss(T, gpdb_mesh_unit(r1.x, r1.y)), U = gpdb_mesh_unit(r1.z, r1.w);
  // rule 3
  const double su = (double)u + rint(s->lateral_sigma * g0), sv = (double)v + rint(s->lateral_sigma * g1);
  if (!(su >= 0.0 && su < (double)W && sv >= 0.0 && sv < (double)H)) return -1;
  const int ru = (int)su, rv = (int)sv;
  const int f = cf[(long long)rv * W + ru];
  if (f < 0) return -1;
  const double t = ct[(long long)rv * W + ru];
  double d[2];
  gpdb_render_ray(ru, rv, fx, fy, cx, cy, d);
  const double X[3] = {t * d[0], t * d[1], t};
  // rule 4
  if (s->min_cos_incidence > 0.0) {
    const float *a = vtx + 3 * (long long)faces[3 * (long long)f], *b = vtx + 3 * (long long)faces[3 * (long long)f + 1];
    const float *c = vtx + 3 * (long long)faces[3 * (long long)f + 2];
    const double ba[3] = {(double)b[0] - (double)a[0], (double)b[1] - (double)a[1], (double)b[2] - (double)a[2]};
    const double ca[3] = {(double)c[0] - (double)a[0], (double)c[1] - (double)a[1], (double)c[2] - (double)a[2]};
    double n[3], m[3];
    gpdb_render_cross(ba, ca, n);
    for (int i = 0; i < 3; i++) m[i] = (pose[i] * n[0] + pose[4 + i] * n[1]) + pose[8 + i] * n[2];
    const double mx = (m[0] * X[0] + m[1] * X[1]) + m[2] * X[2];
    const double mm = (m[0] * m[0] + m[1] * m[1]) + m[2] * m[2], xx = (X[0] * X[0] + X[1] * X[1]) + X[2] * X[2];
    const double cs = fabs(mx) / (sqrt(mm) * sqrt(xx));
    if (cs < s->min_cos_incidence) return -1;
  }
  double zz = X[2];
  if (s->baseline > 0.0) {
    // rule 5
    const double pu = rint((fx * (X[0] - s->baseline)) / X[2] + cx), pv = rint((fy * X[1]) / X[2] + cy);
    if (!(pu >= 0.0 && pu < (double)W && pv >= 0.0 && pv < (double)H)) return -1;
    const long long pi = (long long)pv * W + (long long)pu;
    if (pf[pi] < 0 || pt[pi] < X[2] * (1.0 - s->shadow_tolerance)) return -1;
    // rule 6
    const double fb = fx * s->baseline;
    double D = fb / X[2] + s->disparity_sigma * g2;
    if (s->disparity_step > 0.0) D = s->disparity_step * rint(D / s->disparity_step);
    if (!(D > 0.0) || !isfinite(D)) return -1;
    zz = fb / D;
  }
  // rule 7
  if (U < s->dropout) return -1;
  *z = zz;
  return f;
}

#endif /* GPD_B200_SENSOR_H_ */
