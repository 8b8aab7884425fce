// render_oracle.cpp — include/gpd_b200_render.h's helpers compiled for the host (test infrastructure only), so the numpy
// restatement (tests/render_reference.py) can be held against the header's own code.
#include <stdint.h>

#include "gpd_b200_render.h"

// rule 2 of n vertices under one pose
extern "C" void ro_to_camera(int n, const double *pose, const float *p, double *q) {
  for (int i = 0; i < n; i++) gpdb_render_to_camera(pose, p + 3 * i, q + 3 * i);
}

// rule 4 of n (face, ray) pairs: abc [9n] camera-frame vertices, d [2n] rays; rec [13n], t [n], covers [n]
extern "C" void ro_setup_hit(int n, const double *abc, const double *d, double *rec, double *t, int32_t *covers) {
  for (int i = 0; i < n; i++) {
    gpdb_render_setup(abc + 9 * i, abc + 9 * i + 3, abc + 9 * i + 6, rec + GPDB_RENDER_REC * i);
    t[i] = 0.0;
    covers[i] = gpdb_render_hit(rec + GPDB_RENDER_REC * i, d[2 * i], d[2 * i + 1], t + i);
  }
}

// rule 5 of n hit distances
extern "C" void ro_raw(int n, const double *t, double scale, int format, uint32_t *raw, int32_t *ret) {
  for (int i = 0; i < n; i++) {
    bool r = false;
    raw[i] = gpdb_render_raw(t[i], scale, format, &r);
    ret[i] = r;
  }
}

// rule 6 of n faces abc [9n] (face i is face index i of a mesh with key `key`): count [n], and the first point [3n] and
// normal [3n] of each face (draw j = 1)
extern "C" void ro_mesh(int n, const float *abc, uint64_t key, double density, double *count, double *point, double *normal,
                        double *L) {
  for (int i = 0; i < n; i++) {
    const float *a = abc + 9 * i, *b = a + 3, *c = a + 6;
    double nn[3];
    L[i] = gpdb_mesh_face(a, b, c, nn);
    const gpdb_u32x4 r0 = gpdb_mesh_draw(key, (uint32_t)i, 0u);
    count[i] = gpdb_mesh_count(L[i], density, gpdb_mesh_unit(r0.x, r0.y));
    const gpdb_u32x4 r1 = gpdb_mesh_draw(key, (uint32_t)i, 1u);
    gpdb_mesh_point(a, b, c, gpdb_mesh_unit(r1.x, r1.y), gpdb_mesh_unit(r1.z, r1.w), point + 3 * i);
    for (int k = 0; k < 3; k++) normal[3 * i + k] = nn[k] / L[i];
  }
}
