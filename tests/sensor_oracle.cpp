// sensor_oracle.cpp — include/gpd_b200_sensor.h's helpers compiled for the host (test infrastructure only), so the numpy
// restatement (tests/sensor_reference.py) can be held against the header's own code.
#include <stdint.h>

#include "gpd_b200_sensor.h"

// rule 2's table
extern "C" void so_table(double *T) { gpdb_sensor_table_build(T); }

// rule 2 of n uniforms
extern "C" void so_gauss(int n, const double *T, const double *U, double *g) {
  for (int i = 0; i < n; i++) g[i] = gpdb_sensor_gauss(T, U[i]);
}

// rules 1 and 3-7 of every pixel of camera k (cam) of a view with key `key`, from the clean images (ct, cf) and (pt, pf):
// face [W*H] (-1: no return) and z [W*H]
extern "C" void so_pixels(const gpdb_sensor_params *sp, const double *T, uint64_t key, uint32_t k, const gpdb_depth_camera *cam,
                          const double *ct, const int32_t *cf, const double *pt, const int32_t *pf, const float *vtx,
                          const int32_t *faces, int32_t *face, double *z) {
  const int W = cam->width, H = cam->height;
  for (int v = 0; v < H; v++)
    for (int u = 0; u < W; u++) {
      double zz = 0.0;
      face[v * W + u] = gpdb_sensor_pixel(sp, T, key, k, u, v, W, H, cam->fx, cam->fy, cam->cx, cam->cy, cam->pose, ct, cf,
                                          pt, pf, vtx, faces, &zz);
      z[v * W + u] = zz;
    }
}
