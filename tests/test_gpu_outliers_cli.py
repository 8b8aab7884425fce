"""Cloud::removeStatisticalOutliers in the host shim (-m gpu): on a processed cloud installed in a context it prints the
reference's message and leaves the util::Cloud equal to the library call (gpdb_remove_outliers with mean_k = 50 and
stddev_mul = 1.0); detect_grasps with remove_outliers = 1 reports the key as ignored and detects as without it."""
import os
import subprocess

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from test_host_cpp import HOST, ROOT, _write_detector_cfg, cli, write_pcd  # noqa: F401 (cli: the fixture that builds the CLI)
from test_outliers_reference import noisy_table
from test_refine_reference import random_normals

pytestmark = pytest.mark.gpu

_PROG = r"""
#include <cstdio>
#include <vector>
#include "gpd/gpd.h"
// stdin: N, then N rows x y z nx ny nz cam (hex floats). Installs the cloud, removes its outliers through the shim and
// prints the cloud left behind.
int main() {
  int n;
  if (scanf("%d", &n) != 1) return 1;
  std::vector<float> xyz(3 * (size_t)n);
  std::vector<double> nrm(3 * (size_t)n);
  std::vector<int> cam((size_t)n);
  for (int i = 0; i < n; i++) {
    double v[6];
    for (int a = 0; a < 6; a++) scanf("%la", &v[a]);
    scanf("%d", &cam[i]);
    for (int a = 0; a < 3; a++) xyz[3 * i + a] = (float)v[a], nrm[3 * i + a] = v[3 + a];
  }
  gpd::util::Cloud cloud(xyz, nrm, cam, {0.0, 0.0, 0.0});
  cloud.setSampleIndices({0, 1, 2});
  gpdb_params p;
  gpdb_params_default(&p);
  gpdb_ctx *ctx = nullptr;
  if (gpdb_create(&p, &ctx) != GPDB_OK) return 1;
  if (gpdb_set_cloud(ctx, xyz.data(), nrm.data(), cam.data(), n, cloud.getViewPoints().data(), 1) != GPDB_OK) return 1;
  if (!cloud.removeStatisticalOutliers(ctx)) return 1;
  printf("SAMPLES %zu\n", cloud.getSampleIndices().size());
  for (size_t i = 0; i < cloud.size(); i++)
    printf("P %a %a %a %a %a %a %d\n", cloud.getPoints()[3 * i], cloud.getPoints()[3 * i + 1], cloud.getPoints()[3 * i + 2],
           cloud.getNormals()[3 * i], cloud.getNormals()[3 * i + 1], cloud.getNormals()[3 * i + 2], cloud.getCameraSource()[i]);
  gpdb_destroy(ctx);
  return 0;
}
"""


@pytest.fixture(scope="module")
def prog(cli, tmp_path_factory):  # noqa: F811
    d = tmp_path_factory.mktemp("outliers_prog")
    src, exe = d / "prog.cpp", d / "prog"
    src.write_text(_PROG)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(HOST, "include"), "-I", os.path.join(ROOT, "include"),
                           "-o", str(exe), str(src), "-L", HOST, "-lgpd_host", "-L", os.path.join(ROOT, "gpd_b200"),
                           "-lgpd_b200", "-Wl,-rpath," + HOST, "-Wl,-rpath," + os.path.join(ROOT, "gpd_b200")])
    return str(exe)


def test_shim_equals_the_library_call(prog):
    xyz = noisy_table()
    nrm = random_normals(len(xyz), 31)
    cam = (np.arange(len(xyz)) % 3 != 0).astype(np.int32)
    rows = "\n".join(" ".join([float(v).hex() for v in (*x, *m)] + [str(c)]) for x, m, c in zip(xyz, nrm, cam))
    out = subprocess.run([prog], input=f"{len(xyz)}\n{rows}\n", capture_output=True, text=True, check=True).stdout
    ctx = lib.Context(lib.default_params())
    ctx.set_cloud(xyz, nrm, cam[:, None], np.zeros((1, 3)))
    r = ctx.remove_outliers()
    want = ctx.get_cloud()
    ctx.close()
    assert f"Cloud after removing statistical outliers: {r['n_kept']}\n" in out
    assert 0 < r["n_kept"] < len(xyz)
    assert "SAMPLES 0" in out  # the sample indices are invalidated
    got = np.array([[float.fromhex(v) for v in l.split()[1:7]] for l in out.splitlines() if l.startswith("P ")])
    gcam = np.array([int(l.split()[7]) for l in out.splitlines() if l.startswith("P ")])
    assert np.array_equal(got[:, :3].astype(np.float32), want["xyz"])
    assert np.array_equal(got[:, 3:], want["normals"])
    assert np.array_equal(gcam, want["cam_source"][:, 0])


def test_detect_grasps_ignores_remove_outliers(cli, tmp_path):  # noqa: F811
    w, _ = load_weights(15)
    xyz = np.asarray(scenes.synthetic_raw_scene(12, n_points=15000)["xyz"], np.float32)
    pcd = tmp_path / "view.pcd"
    write_pcd(pcd, xyz, binary=True)
    outs = []
    for i, extra in enumerate(("", "remove_outliers = 1\n")):
        d = tmp_path / f"cfg{i}"
        d.mkdir()
        cfg = _write_detector_cfg(d, w, "num_samples = 100\nnum_selected = 20\n" + extra)
        outs.append(subprocess.check_output([cli, cfg, str(pcd)]).decode())
    assert "NOTE: remove_outliers is not part of the accelerated preprocessing: ignored" in outs[1]
    assert "statistical outliers" not in outs[1]
    res = [[l for l in o.splitlines() if l.startswith("RESULT")] for o in outs]
    assert res[0] == res[1] and len(res[0]) == 1
