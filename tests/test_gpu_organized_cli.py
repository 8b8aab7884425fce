"""Cloud::calculateNormalsOrganized in the host shim (-m gpu): an organized .pcd (WIDTH x HEIGHT with NaN points) keeps
its layout, and the shim prints the reference's message and leaves the normals gpdb_normals_organized gives, widened to
double; an unorganized cloud prints the reference's error and keeps its normals."""
import os
import subprocess

import numpy as np
import pytest

import depth_reference as dr
import organized_reference as orf
from gpd_b200 import lib
from test_host_cpp import HOST, ROOT, cli  # noqa: F401 (cli: the fixture that builds the shim)

pytestmark = pytest.mark.gpu

_PROG = r"""
#include <cstdio>
#include "gpd/gpd.h"
// argv[1]: a .pcd file. Loads it with view point (0.1, -0.2, 0.3), estimates organized normals and prints them.
int main(int argc, char **argv) {
  gpd::util::Cloud cloud(argv[1], {0.1, -0.2, 0.3});
  gpdb_params p;
  gpdb_params_default(&p);
  gpdb_ctx *ctx = nullptr;
  if (gpdb_create(&p, &ctx) != GPDB_OK) return 1;
  printf("ORGANIZED %d %d %d\n", (int)cloud.isOrganized(), cloud.width(), cloud.height());
  const bool ok = cloud.calculateNormalsOrganized(ctx);
  printf("OK %d\n", (int)ok);
  for (size_t i = 0; i < cloud.getNormals().size(); i++) printf("N %a\n", cloud.getNormals()[i]);
  gpdb_destroy(ctx);
  return 0;
}
"""


@pytest.fixture(scope="module")
def prog(cli, tmp_path_factory):  # noqa: F811
    d = tmp_path_factory.mktemp("organized_prog")
    src, exe = d / "prog.cpp", d / "prog"
    src.write_text(_PROG)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(HOST, "include"), "-I", os.path.join(ROOT, "include"),
                           "-o", str(exe), str(src), "-L", HOST, "-lgpd_host", "-L", os.path.join(ROOT, "gpd_b200"),
                           "-lgpd_b200", "-Wl,-rpath," + HOST, "-Wl,-rpath," + os.path.join(ROOT, "gpd_b200")])
    return str(exe)


def _write(path, xyz, W, H):
    rows = np.asarray(xyz, np.float32).reshape(-1, 3)
    hdr = (f"VERSION .7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\nWIDTH {W}\nHEIGHT {H}\nVIEWPOINT 0 0 0 1 0 0 0\n"
           f"POINTS {W * H}\nDATA binary\n")
    with open(path, "wb") as f:
        f.write(hdr.encode() + rows.tobytes())


def test_shim_equals_the_library_call(prog, tmp_path):
    v = dr.render_views([4], [1], 0, width=120, height=90, f=140.0)[0][0]
    xyz = orf.camera_cloud(v[0], v[1], 0)
    assert np.isnan(xyz).any()
    pcd = tmp_path / "organized.pcd"
    _write(pcd, xyz, 120, 90)
    out = subprocess.run([prog, str(pcd)], capture_output=True, text=True, check=True).stdout
    assert "ORGANIZED 1 120 90" in out and "OK 1" in out
    assert "Using integral images for surface normals estimation ...\n" in out
    got = np.array([float.fromhex(l.split()[1]) for l in out.splitlines() if l.startswith("N ")]).reshape(90, 120, 3)
    ctx = lib.Context(lib.default_params())
    want, _ = ctx.normals_organized([xyz], np.array([[0.1, -0.2, 0.3]]))
    ctx.close()
    assert np.array_equal(got, want[0].astype(np.float64), equal_nan=True)
    assert np.isfinite(got[..., 0]).sum() > 100


def test_unorganized_cloud_keeps_its_normals(prog, tmp_path):
    from test_organized_reference import plane
    pcd = tmp_path / "flat.pcd"
    _write(pcd, plane(50, 60), 3000, 1)
    out = subprocess.run([prog, str(pcd)], capture_output=True, text=True, check=True).stdout
    assert "ORGANIZED 0 3000 1" in out and "OK 0" in out
    assert "Error: point cloud is not organized!\n" in out
