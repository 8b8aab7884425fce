"""refine_normals_k in the host shim (-m gpu): GraspDetector::preprocessPointCloud / preprocessPointClouds refine the
normals on the device, and the normals they leave in util::Cloud equal the library calls composed by hand
(gpdb_preprocess[_clouds] then gpdb_refine_normals[_clouds]); detect_grasps prints the reference's message and no
NOTE for the key."""
import os
import subprocess

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from test_host_cpp import HOST, ROOT, _write_detector_cfg, cli, write_pcd  # noqa: F401 (cli: the fixture that builds the CLI)

pytestmark = pytest.mark.gpu
K = 12

_PROG = r"""
#include <cstdio>
#include "gpd/gpd.h"
// argv: cfg pcd... ; one file: preprocessPointCloud, several: preprocessPointClouds. Prints each cloud's normals.
int main(int argc, char **argv) {
  gpd::GraspDetector det(argv[1]);
  std::vector<gpd::util::Cloud> clouds;
  for (int i = 2; i < argc; i++) clouds.emplace_back(argv[i], std::vector<double>{0.0, 0.0, 0.0});
  if (clouds.size() == 1) det.preprocessPointCloud(clouds[0]);
  else if (!det.preprocessPointClouds(clouds)) return 1;
  for (size_t b = 0; b < clouds.size(); b++) {
    printf("NRM %zu", b);
    for (double v : clouds[b].getNormals()) printf(" %a", v);
    printf("\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def prog(cli, tmp_path_factory):  # noqa: F811
    d = tmp_path_factory.mktemp("refine_prog")
    src, exe = d / "prog.cpp", d / "prog"
    src.write_text(_PROG)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(HOST, "include"), "-I", os.path.join(ROOT, "include"),
                           "-o", str(exe), str(src), "-L", HOST, "-lgpd_host", "-L", os.path.join(ROOT, "gpd_b200"),
                           "-lgpd_b200", "-Wl,-rpath," + HOST, "-Wl,-rpath," + os.path.join(ROOT, "gpd_b200")])
    return str(exe)


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    """A config file with refine_normals_k set and two raw table views as binary PCD files."""
    d = tmp_path_factory.mktemp("refine_scene")
    w, _ = load_weights(15)
    cfg = _write_detector_cfg(d, w, f"num_samples = 100\nnum_selected = 20\nrefine_normals_k = {K}\n")
    raws, files = [], []
    for i, seed in enumerate((9, 10)):
        xyz = np.asarray(scenes.synthetic_raw_scene(seed, n_points=15000)["xyz"], np.float32)
        p = d / f"view{i}.pcd"
        write_pcd(p, xyz, binary=True)
        raws.append(xyz)
        files.append(str(p))
    return cfg, raws, files


def by_hand(raws):
    ctx = lib.Context(lib.default_params(channels=15))
    ctx.preprocess_clouds([{"xyz": x, "view_points": np.zeros((1, 3))} for x in raws], pp=lib.preprocess_params(voxelize=0))
    ctx.refine_normals_clouds(K)
    out = [c["normals"] for c in ctx.get_clouds()]
    ctx.close()
    return out


def nrm_lines(out):
    return {int(l.split()[1]): np.array([float.fromhex(v) for v in l.split()[2:]]).reshape(-1, 3)
            for l in out.splitlines() if l.startswith("NRM ")}


def test_preprocessing_refines_the_normals(prog, scene):
    cfg, raws, files = scene
    hand = by_hand(raws)
    out = subprocess.check_output([prog, cfg, files[0]]).decode()
    assert "Refining surface normals ..." in out and "refine_normals_k are not part" not in out
    got = nrm_lines(out)[0]
    assert np.array_equal(got, hand[0], equal_nan=True)
    out = subprocess.check_output([prog, cfg] + files).decode()
    got = nrm_lines(out)
    for b in range(len(files)):
        assert np.array_equal(got[b], hand[b], equal_nan=True)


def test_cli_routes_refine(cli, scene):  # noqa: F811
    cfg, _, files = scene
    for args in ([files[0]], ["--batch"] + files):
        out = subprocess.check_output([cli, cfg] + args).decode()
        assert "Refining surface normals ..." in out and "RESULT n_grasps=" in out
        assert "refine_normals_k are not part" not in out
