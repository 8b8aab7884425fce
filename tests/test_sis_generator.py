"""The SIS generator of include/gpd_b200_sis.h without a GPU: the numpy restatement (sis_reference.py) against the Random123
known-answer vectors of Philox4x32-10, the header's own C code against the restatement, the restated draw procedure on toy
kept sets, and the layout of gpdb_sis_params against the ctypes mirror."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import sis_reference as sr
from gpd_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_philox_known_answers():
    # Random123 kat_vectors, philox4x32_10: counter / key -> output
    kat = [([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
           ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
           ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
            [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1])]
    for ctr, key, want in kat:
        assert sr.philox(np.array([ctr], np.uint32), key)[0].tolist() == want


def compile_and_run(src):
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-O1", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"),
                               os.path.join(d, "t.c"), "-lm"])
        return subprocess.check_output([os.path.join(d, "t")]).decode().split()


def test_header_draws_equal_the_restatement():
    """gpdb_sis_draw of the header (the code the kernels run) for keys with both words set, both streams and halves."""
    src = r'''
#include <stdio.h>
#include "gpd_b200_sis.h"
int main(void) {
  const uint64_t keys[3] = {0ull, 0x0123456789ABCDEFull, 0xFFFFFFFFFFFFFFFFull};
  for (int k = 0; k < 3; k++)
    for (uint32_t t = 0; t < 70000; t += 6911)
      for (uint32_t s = 0; s < 2; s++)
        for (uint32_t h = 0; h < 2; h++) {
          gpdb_u32x4 c = gpdb_sis_draw(keys[k], t, 3u, s, h);
          printf("%u %u %u %u\n", c.x, c.y, c.z, c.w);
        }
  printf("%.17g %.17g\n", gpdb_sis_unit(0u), gpdb_sis_unit(0xFFFFFFFFu));
  return 0;
}'''
    out = list(map(float, compile_and_run(src)))
    got = np.array(out[:-2], np.uint64).reshape(-1, 4)
    rows = []
    for key in (0, 0x0123456789ABCDEF, 0xFFFFFFFFFFFFFFFF):
        for t in range(0, 70000, 6911):
            for s in range(2):
                for h in range(2):
                    rows.append(sr.draws(key, [t], 3, s, h)[0])
    assert np.array_equal(got, np.array(rows, np.uint64))
    assert out[-2:] == [0.5 * 2.0 ** -32, 1.0 - 0.5 * 2.0 ** -32]


def test_sis_params_layout_matches_the_header():
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "gpd_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(gpdb_sis_params), offsetof(gpdb_sis_params, num_iterations),
         offsetof(gpdb_sis_params, num_samples_per_iteration), offsetof(gpdb_sis_params, prob_rand_samples),
         offsetof(gpdb_sis_params, standard_deviation), offsetof(gpdb_sis_params, sampling_method),
         offsetof(gpdb_sis_params, workspace), offsetof(gpdb_sis_params, min_score), offsetof(gpdb_sis_params, min_inliers),
         offsetof(gpdb_sis_params, seed));
  return 0;
}'''
    nums = list(map(int, compile_and_run(src)))
    names = [n for n, _ in abi.SisParams._fields_]
    assert nums == [C.sizeof(abi.SisParams)] + [getattr(abi.SisParams, n).offset for n in names]
    assert nums[0] == 104


def toy():
    rng = np.random.default_rng(5)
    xyz = rng.uniform(-0.2, 0.2, (500, 3)).astype(np.float32)
    kept = xyz[:7].astype(np.float64)
    return xyz, kept


def test_sum_of_gaussians_takes_the_first_proposals():
    xyz, kept = toy()
    key, sigma = 12345 + (7 << 32), 0.02
    pos, par, ng = sr.draw_round(kept, 2, key, 50, 0.3, sigma, 0, [-1, 1, -1, 1, -1, 1], xyz, np.arange(40))
    assert ng == 35 and len(pos) == 50
    p, z = sr.gaussian(key, np.arange(35), 2, 7)
    assert np.array_equal(par, p) and np.array_equal(pos[:35], kept[p] + sigma * z)
    # the uniform slots are initial points, taken in proposal order
    c = sr.draws(key, np.arange(15), 2, 1, 0)[:, 0]
    assert np.array_equal(pos[35:], xyz[(c % 40).astype(np.int64)].astype(np.float64))


def test_max_of_gaussians_keeps_only_nearest_parent_proposals():
    xyz, kept = toy()
    kept = np.vstack([kept, kept[:2] + 0.001])  # near-duplicates: many proposals fall closer to another kept position
    pos, par, ng = sr.draw_round(kept, 0, 99, 40, 0.0, 0.02, 1, [-1, 1, -1, 1, -1, 1], xyz, np.arange(9))
    assert ng == 40
    assert np.all(sr.d2(pos, kept[par]) <= sr.d2(pos[:, None, :], kept[None]).min(axis=1))
    # the accepted ones are the first proposals that satisfy the rule: the rejected ones before them violate it
    p, z = sr.gaussian(99, np.arange(4096), 0, len(kept))
    x = kept[p] + 0.02 * z
    ok = sr.d2(x, kept[p]) <= sr.d2(x[:, None, :], kept[None]).min(axis=1)
    assert 40 < np.flatnonzero(ok)[39] + 1 < 4096 and np.array_equal(x[ok][:40], pos)


def test_uniform_draws_respect_the_inclusive_workspace():
    xyz, kept = toy()
    ws = [float(xyz[3, 0]), 1, -1, 1, -1, 1]  # point 3 lies exactly on the lower x bound: inside
    pos, _, ng = sr.draw_round(kept, 1, 4, 30, 1.0, 0.02, 0, ws, xyz, [])
    assert ng == 0 and len(pos) == 30 and np.all(pos[:, 0] >= ws[0])
    # a workspace that holds no point: the loop stops after MAX_PROPOSALS and the slots are dropped
    pos, _, _ = sr.draw_round(kept, 1, 4, 10, 1.0, 0.02, 0, [5, 6, 5, 6, 5, 6], xyz, [], wave=1 << 18)
    assert len(pos) == 0
