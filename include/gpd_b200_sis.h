/*
 * gpd_b200_sis.h — SPECIFICATION of the random draws of gpdb_sis_batch (SequentialImportanceSampling on the device).
 *
 * The reference draws its proposals with rand() / a std::normal_distribution inside loops that stop when enough proposals
 * were accepted (sequential_importance_sampling.cpp:187-270), so a run cannot be reproduced on a GPU that draws many
 * proposals at once. gpdb_sis_batch keeps the reference's loop (drawRound of the host shim) and replaces the generator by
 * a counter-based one, so that every proposal is a pure function of (seed, cloud, round, proposal number):
 *
 *  1. Philox4x32-10 (Salmon et al., SC'11; the Random123 constants below). Cloud b's key is seed + b as (low word, high
 *     word); the counter of proposal t of round r is (t, r, stream, half), stream 0 for Gaussian proposals, 1 for uniform.
 *  2. A Gaussian proposal t draws c0 = philox(t, r, 0, 0) and c1 = philox(t, r, 0, 1). Its parent is kept position
 *     c0.x % m, m = the cloud's kept positions when the round started. With u(w) = (w + 0.5) * 2^-32 (in (0, 1)):
 *        z0, z1 = sqrt(-2 log u(c0.y)) * (cospi, sinpi)(2 u(c0.z))      z2 = sqrt(-2 log u(c0.w)) * cospi(2 u(c1.x))
 *     and x_k = parent_k + sigma * z_k, each operation rounded on its own (no FMA).
 *  3. Sum of Gaussians accepts every Gaussian proposal. Max of Gaussians accepts x iff d2(x, parent) <= d2(x, kept_j) for
 *     every kept j < m, d2 = (dx*dx + dy*dy) + dz*dz rounded per operation: the reference's `p >= maxp` test
 *     (:213-234) without the exp, which can only differ where exp rounds two distances to the same density or underflows.
 *  4. A uniform proposal t draws c = philox(t, r, 1, 0); its point is init[c.x % n_init] (the cloud's initial sample
 *     indices), or point c.x % N_b when the cloud has no initial list, accepted when (double) of each float coordinate
 *     lies inside the inclusive workspace (drawUniformSamples, :263-265).
 *  5. Accepted proposals fill the round's slots in increasing t: the Gaussian slots first, then the uniform ones. Each of
 *     the two loops stops after GPDB_SIS_MAX_PROPOSALS proposals; slots still empty then are dropped, not evaluated (the
 *     reference would loop forever there).
 *
 * So cloud b's result depends only on (parameters, seed + b, cloud b, its initial list): not on the batch size, the other
 * clouds or how the library splits its work. tests/test_sis_generator.py restates this file in numpy.
 */
#ifndef GPD_B200_SIS_H_
#define GPD_B200_SIS_H_

#include <math.h>
#include <stdint.h>

#include "gpd_b200_shadow.h" /* GPDB_HD */

#define GPDB_SIS_MAX_PROPOSALS (1 << 20)
#define GPDB_SIS_GAUSS 0u
#define GPDB_SIS_UNIFORM 1u

typedef struct gpdb_u32x4 {
  uint32_t x, y, z, w;
} gpdb_u32x4;

GPDB_HD gpdb_u32x4 gpdb_philox4x32_10(gpdb_u32x4 c, uint32_t k0, uint32_t k1) {
  for (int i = 0; i < 10; i++) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c.x, p1 = (uint64_t)0xCD9E8D57u * c.z;
    const gpdb_u32x4 n = {(uint32_t)(p1 >> 32) ^ c.y ^ k0, (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c.w ^ k1, (uint32_t)p0};
    c = n;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

/* the draw of proposal t of round r, stream s, half h, for cloud key `key` = seed + b */
GPDB_HD gpdb_u32x4 gpdb_sis_draw(uint64_t key, uint32_t t, uint32_t r, uint32_t s, uint32_t h) {
  const gpdb_u32x4 c = {t, r, s, h};
  return gpdb_philox4x32_10(c, (uint32_t)key, (uint32_t)(key >> 32));
}

/* u(w) = (w + 0.5) * 2^-32: exact in double, never 0 or 1 */
GPDB_HD double gpdb_sis_unit(uint32_t w) { return ((double)w + 0.5) * 2.3283064365386963e-10; }

#endif /* GPD_B200_SIS_H_ */
