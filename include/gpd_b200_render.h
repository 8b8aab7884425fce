/*
 * gpd_b200_render.h — SPECIFICATION of the depth rendering of triangle meshes (gpdb_render_depth[_device]) and of the
 * surface sampling of the same meshes (gpdb_sample_meshes[_device]); the entry points are declared in gpd_b200.h.
 *
 * A user who retrains the classifier for a new gripper usually has meshes of their objects and no captured dataset.
 * These two calls make the training views (depth images that gpdb_preprocess_depth[_device] consumes as they are) and
 * the ground-truth clouds that gpdb_reevaluate_batch[_device] labels against, from the same meshes. Every operation is
 * rounded on its own, with no FMA.
 *
 *  1. Mesh. View (or mesh) b has the float32 xyz vertices vertex_offsets[b] .. vertex_offsets[b+1]-1 (world frame) and
 *     the int32 index triples faces face_offsets[b] .. face_offsets[b+1]-1, 0-based into the view's own vertices. Face
 *     (a, b, c) has the normal n = (b - a) x (c - a); a cross product is x = a.y*b.z - a.z*b.y and cyclically
 *     (gpdb_render_cross). A mesh may have no faces.
 *  2. Camera frame. gpdb_depth_camera (gpd_b200_depth.h) unchanged; the pose is camera-to-world [R | t]. A vertex p goes
 *     to the camera frame in float64: dx = (double)p.x - t0 (likewise dy, dz), q_i = (R0i*dx + R1i*dy) + R2i*dz
 *     (gpdb_render_to_camera). Each vertex is transformed once per camera, so a shared vertex has identical camera-frame
 *     values in every face that uses it.
 *  3. Pixel ray. d = (((double)u - cx) / fx, ((double)v - cy) / fy, 1): the pixel convention of gpd_b200_depth.h rule 1,
 *     no half-pixel offset (gpdb_render_ray).
 *  4. Coverage. A face with camera-frame vertices A, B, C has m0 = A x B, m1 = B x C, m2 = C x A, n = (B - A) x (C - A)
 *     and h = (n.x*A.x + n.y*A.y) + n.z*A.z (gpdb_render_setup). For the ray d, e_i = (m_i.x*d.x + m_i.y*d.y) + m_i.z and
 *     s = (n.x*d.x + n.y*d.y) + n.z. The face covers the pixel iff s != 0, (e0, e1, e2) are all >= 0 or all <= 0, and
 *     t = h / s is finite and > 0 (gpdb_render_hit). The test does not depend on the winding: both sides of a face render.
 *     Watertightness. Let two faces share an edge whose two vertices have identical coordinates (in the world frame, hence
 *     by rule 2 in the camera frame). If the faces traverse the edge in opposite directions, one has m = P x Q and the
 *     other m' = Q x P. Each component of Q x P is Q.y*P.z - Q.z*P.y; IEEE multiplication commutes exactly, so its two
 *     products are those of P x Q swapped, and IEEE subtraction satisfies fl(a - b) = -fl(b - a) exactly: m' = -m bit for
 *     bit. e for the ray d is then formed from negated operands, and rounding to nearest is symmetric, so e' = -e exactly.
 *     (Same direction: m' = m and e' = e.) Hence the shared edge splits the rays identically for both faces: a ray with
 *     e > 0 is on one face's inner side of the edge and on the other's outer side when the faces lie on opposite sides of
 *     it, as in any unfolded mesh, and a ray with e = 0 passes the edge test of both. A ray through the edge's interior
 *     therefore fails the edge test of at most one face and passes that of the other, which its remaining two edges
 *     accept (they are bounded away from the edge's interior); a ray through a shared vertex passes e = 0 on the two edges
 *     of each face that meet there. No ray through a shared edge or vertex falls between the faces. tests/
 *     test_render_reference.py checks fans and strips whose shared edges and vertices pass exactly through pixel centres.
 *  5. Depth. A pixel's hit is the covering face with the smallest t, ties to the smallest face index (view-local). Every
 *     camera's image is written back to back in the layout gpdb_preprocess_depth reads: view by view, camera by camera,
 *     height x width row-major. GPDB_DEPTH_F32: raw = (float)(t / depth_scale). GPDB_DEPTH_U16: r = rint(t / depth_scale)
 *     in float64 (half to even), raw = r if 1 <= r <= 65535, else 0. No hit: raw = 0. min_depth and max_depth are not
 *     applied (preprocessing applies them). The optional face image holds the hit's view-local face index, or -1 wherever
 *     the pixel is not a return by gpd_b200_depth.h rule 2 (U16: raw = 0; F32: raw not finite or <= 0), so the depth image
 *     and the face image always agree (gpdb_render_raw).
 *  6. Surface samples. Face f of mesh b (view-local index) in the world frame, in float64 from the float32 vertices a, b,
 *     c: n by rule 1, L = sqrt((n.x*n.x + n.y*n.y) + n.z*n.z), area = 0.5*L (gpdb_mesh_face). Draw j of the face is
 *     philox({f, j, GPDB_MESH_STREAM, 0}, key) with key = seed + b split as in gpd_b200_depth.h rule 5 (gpdb_mesh_draw);
 *     stream word 4 keeps these draws apart from SIS (0, 1), subsampling (2) and the plane fit (3). A uniform from two
 *     words (x, y) is ((x << 32 | y) >> 11) * 2^-53 (gpdb_mesh_unit). The count is floor(area*density + U), U the uniform
 *     of draw j = 0 from (x, y); a face with L = 0 or a non-finite L has count 0 (gpdb_mesh_count). Point k of the face
 *     uses draw j = k + 1: r1 from (x, y), r2 from (z, w), s = sqrt(r1), w0 = 1 - s, w1 = s*(1 - r2), w2 = s*r2, and p =
 *     (w0*a + w1*b) + w2*c per component (gpdb_mesh_point); xyz = (float)p, normal = n / L per component in float64
 *     (following the winding), face = f. Mesh b's points come face by face in face order, and its offsets are the exact
 *     integer exclusive scan of the counts. A mesh's draw depends only on (seed + b, mesh b, density).
 *  7. Errors (GPDB_ERR_INVALID, the message naming the view or mesh; nothing is written): a face index outside the view's
 *     vertices or a non-finite vertex (checked on the device, the host twins upload first); malformed offsets; the camera
 *     checks of gpdb_preprocess_depth; 2^31 or more pixels in a render call; a density that is not finite and > 0; 2^31
 *     or more sampled points.
 *
 * tests/render_reference.py restates this file in numpy float64 (single IEEE roundings, so it is the oracle bit for bit).
 */
#ifndef GPD_B200_RENDER_H_
#define GPD_B200_RENDER_H_

#include <math.h>
#include <stdint.h>

#include "gpd_b200_depth.h" /* gpdb_depth_camera, GPDB_DEPTH_*, gpdb_philox4x32_10, GPDB_HD */

/* the stream word of the surface-sample draws (SIS 0 and 1, subsampling 2, plane fit 3) */
#define GPDB_MESH_STREAM 4u

/* rule 1: o = a x b */
GPDB_HD void gpdb_render_cross(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

/* rule 2: q = R^T (p - t) for the camera-to-world pose [R | t] (row-major 3 x 4) */
GPDB_HD void gpdb_render_to_camera(const double pose[12], const float p[3], double q[3]) {
  const double dx = (double)p[0] - pose[3], dy = (double)p[1] - pose[7], dz = (double)p[2] - pose[11];
  for (int i = 0; i < 3; i++) q[i] = (pose[i] * dx + pose[4 + i] * dy) + pose[8 + i] * dz;
}

/* rule 3: the x and y of the ray of pixel (u, v) (its z is 1) */
GPDB_HD void gpdb_render_ray(int u, int v, double fx, double fy, double cx, double cy, double d[2]) {
  d[0] = ((double)u - cx) / fx;
  d[1] = ((double)v - cy) / fy;
}

/* rule 4: the setup of a face with camera-frame vertices A, B, C: rec = m0, m1, m2, n (3 each), h */
#define GPDB_RENDER_REC 13
GPDB_HD void gpdb_render_setup(const double A[3], const double B[3], const double C[3], double rec[GPDB_RENDER_REC]) {
  gpdb_render_cross(A, B, rec);
  gpdb_render_cross(B, C, rec + 3);
  gpdb_render_cross(C, A, rec + 6);
  const double ba[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]};
  const double ca[3] = {C[0] - A[0], C[1] - A[1], C[2] - A[2]};
  gpdb_render_cross(ba, ca, rec + 9);
  rec[12] = (rec[9] * A[0] + rec[10] * A[1]) + rec[11] * A[2];
}

/* rule 4: true iff the face covers the ray (dx, dy, 1); *t receives h / s */
GPDB_HD bool gpdb_render_hit(const double rec[GPDB_RENDER_REC], double dx, double dy, double *t) {
  const double e0 = (rec[0] * dx + rec[1] * dy) + rec[2];
  const double e1 = (rec[3] * dx + rec[4] * dy) + rec[5];
  const double e2 = (rec[6] * dx + rec[7] * dy) + rec[8];
  const double s = (rec[9] * dx + rec[10] * dy) + rec[11];
  if (s == 0.0) return false;
  if (!((e0 >= 0.0 && e1 >= 0.0 && e2 >= 0.0) || (e0 <= 0.0 && e1 <= 0.0 && e2 <= 0.0))) return false;
  *t = rec[12] / s;
  return isfinite(*t) && *t > 0.0;
}

/* rule 5: the stored value of a hit at distance t (F32: the float's bits in the low 32 bits; U16: the value); *ret is
 * whether the value is a return by gpd_b200_depth.h rule 2 */
GPDB_HD uint32_t gpdb_render_raw(double t, double depth_scale, int format, bool *ret) {
  const double q = t / depth_scale;
  if (format == GPDB_DEPTH_F32) {
    const float f = (float)q;
    *ret = isfinite(f) && f > 0.0f;
    union {
      float f;
      uint32_t u;
    } b;
    b.f = f;
    return b.u;
  }
  const double r = rint(q);
  *ret = r >= 1.0 && r <= 65535.0;
  return *ret ? (uint32_t)r : 0u;
}

/* rule 6: draw j of face f of the mesh whose key is seed + b */
GPDB_HD gpdb_u32x4 gpdb_mesh_draw(uint64_t key, uint32_t f, uint32_t j) {
  const gpdb_u32x4 c = {f, j, GPDB_MESH_STREAM, 0u};
  return gpdb_philox4x32_10(c, (uint32_t)key, (uint32_t)(key >> 32));
}

/* rule 6: the uniform in [0, 1) of the words (x, y) */
GPDB_HD double gpdb_mesh_unit(uint32_t x, uint32_t y) {
  return (double)((((uint64_t)x << 32) | y) >> 11) * 1.1102230246251565e-16;
}

/* rule 6: the world-frame normal n and its length L of the face (a, b, c); returns L */
GPDB_HD double gpdb_mesh_face(const float a[3], const float b[3], const float c[3], double n[3]) {
  const double ba[3] = {(double)b[0] - (double)a[0], (double)b[1] - (double)a[1], (double)b[2] - (double)a[2]};
  const double ca[3] = {(double)c[0] - (double)a[0], (double)c[1] - (double)a[1], (double)c[2] - (double)a[2]};
  gpdb_render_cross(ba, ca, n);
  return sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
}

/* rule 6: the face's point count as a double (floor(area*density + U), 0 for L = 0 or a non-finite L); the caller
 * compares it with 2^31 before converting */
GPDB_HD double gpdb_mesh_count(double L, double density, double U) {
  if (!(L > 0.0) || !isfinite(L)) return 0.0;
  return floor((0.5 * L) * density + U);
}

/* rule 6: the point of the face (a, b, c) at the uniforms r1, r2 */
GPDB_HD void gpdb_mesh_point(const float a[3], const float b[3], const float c[3], double r1, double r2, double p[3]) {
  const double s = sqrt(r1), w0 = 1.0 - s, w1 = s * (1.0 - r2), w2 = s * r2;
  for (int i = 0; i < 3; i++) p[i] = (w0 * (double)a[i] + w1 * (double)b[i]) + w2 * (double)c[i];
}

#endif /* GPD_B200_RENDER_H_ */
