"""sample_above_plane in the host shim (-m gpu): GraspDetector::preprocessPointCloud / preprocessPointClouds and the
detect_grasps command line (also --sis and --batch) run Cloud::sampleAbovePlane on the device. The sample indices they
draw equal the library calls composed by hand (gpdb_preprocess, gpdb_segment_plane[s], subsampleSampleIndices' fixed-seed
draws), and every one of them is off the plane."""
import os
import subprocess

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from test_host_cpp import HOST, ROOT, _write_detector_cfg, cli, write_pcd  # noqa: F401 (cli: the fixture that builds the CLI)

pytestmark = pytest.mark.gpu
NUM_SAMPLES = 200

_PROG = r"""
#include <cstdio>
#include "gpd/gpd.h"
// argv: cfg pcd... ; one file: preprocessPointCloud, several: preprocessPointClouds. Prints each cloud's sample indices.
int main(int argc, char **argv) {
  gpd::GraspDetector det(argv[1]);
  std::vector<gpd::util::Cloud> clouds;
  for (int i = 2; i < argc; i++) clouds.emplace_back(argv[i], std::vector<double>{0.0, 0.0, 0.0});
  if (clouds.size() == 1) det.preprocessPointCloud(clouds[0]);
  else if (!det.preprocessPointClouds(clouds)) return 1;
  for (size_t b = 0; b < clouds.size(); b++) {
    printf("IDX %zu", b);
    for (int j : clouds[b].getSampleIndices()) printf(" %d", j);
    printf("\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def prog(cli, tmp_path_factory):  # noqa: F811
    d = tmp_path_factory.mktemp("plane_prog")
    src, exe = d / "prog.cpp", d / "prog"
    src.write_text(_PROG)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(HOST, "include"), "-I", os.path.join(ROOT, "include"),
                           "-o", str(exe), str(src), "-L", HOST, "-lgpd_host", "-L", os.path.join(ROOT, "gpd_b200"),
                           "-lgpd_b200", "-Wl,-rpath," + HOST, "-Wl,-rpath," + os.path.join(ROOT, "gpd_b200")])
    return str(exe)


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    """A config file with sample_above_plane = 1 and two raw table views as binary PCD files."""
    d = tmp_path_factory.mktemp("plane_scene")
    w, _ = load_weights(15)
    cfg = _write_detector_cfg(d, w, f"num_samples = {NUM_SAMPLES}\nnum_selected = 20\nmin_inliers = 1\nsample_above_plane = 1\n"
                              "num_init_samples = 50\nnum_iterations = 1\nnum_samples_per_iteration = 30\n")
    raws, files = [], []
    for i, seed in enumerate((7, 8)):
        xyz = np.asarray(scenes.synthetic_raw_scene(seed, n_points=15000)["xyz"], np.float32)
        p = d / f"view{i}.pcd"
        write_pcd(p, xyz, binary=True)
        raws.append(xyz)
        files.append(str(p))
    return cfg, raws, files


def draws(pool, n):
    """subsampleSampleIndices with the shim's fixed-seed generator: n draws with replacement (none when n >= |pool|)."""
    if n <= 0 or n >= len(pool):
        return list(pool)
    s, out = 42, []
    for _ in range(n):
        s = (s * 1664525 + 1013904223) & 0xFFFFFFFF
        out.append(int(pool[s % len(pool)]))
    return out


def by_hand(raws):
    """gpdb_preprocess_clouds (voxelize = 0, as the cfg) + gpdb_segment_planes, cloud b with key b: each cloud's pool of
    points off its plane (empty when the fit failed or no point is off it) and eligible bytes."""
    ctx = lib.Context(lib.default_params(channels=15))
    ctx.preprocess_clouds([{"xyz": x, "view_points": np.zeros((1, 3))} for x in raws], pp=lib.preprocess_params(voxelize=0))
    r = ctx.segment_planes()
    off = np.concatenate([[0], np.cumsum([len(c["xyz"]) for c in ctx.get_clouds()])])
    out = []
    for b in range(len(raws)):
        e = r["eligible"][off[b]:off[b + 1]]
        n = off[b + 1] - off[b]
        pool = np.flatnonzero(e) if 0 < r["n_inliers"][b] < n else np.zeros(0, np.int64)
        out.append((pool, e))
    ctx.close()
    return out


def idx_lines(out):
    return {int(l.split()[1]): [int(v) for v in l.split()[2:]] for l in out.splitlines() if l.startswith("IDX ")}


def test_single_and_batch_preprocessing_sample_above_the_plane(prog, scene):
    cfg, raws, files = scene
    hand = by_hand(raws)
    for b, f in enumerate(files[:1]):
        out = subprocess.check_output([prog, cfg, f]).decode()
        pool, e = hand[b]
        assert len(pool) > NUM_SAMPLES
        assert f"Plane fit succeeded. {len(pool)} samples above plane." in out
        got = idx_lines(out)[0]
        assert got == draws(pool, NUM_SAMPLES) and all(e[j] == 1 for j in got)
    out = subprocess.check_output([prog, cfg] + files).decode()
    got = idx_lines(out)
    for b in range(len(files)):
        pool, e = hand[b]
        assert f"Plane fit succeeded. {len(pool)} samples above plane." in out
        assert got[b] == draws(pool, NUM_SAMPLES) and all(e[j] == 1 for j in got[b])
    assert "sample_above_plane are not part" not in out


def test_cli_routes_report_the_fit(cli, scene):  # noqa: F811
    """detect_grasps, --sis and --batch print the reference's message with the count the library calls give, and find
    grasps."""
    cfg, raws, files = scene
    hand = by_hand(raws)
    n0 = len(hand[0][0])
    for extra in ([], ["--sis", "3"]):
        out = subprocess.check_output([cli, cfg, files[0]] + extra).decode()
        assert "Sampling above plane ..." in out and f"Plane fit succeeded. {n0} samples above plane." in out
        assert "RESULT n_grasps=" in out
    out = subprocess.check_output([cli, cfg, "--batch"] + files).decode()
    for pool, _ in hand:
        assert f"Plane fit succeeded. {len(pool)} samples above plane." in out
