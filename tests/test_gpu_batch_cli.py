"""detect_grasps CONFIG --batch PCD... (GraspDetector / SequentialImportanceSampling over a batch of clouds, -m gpu): per
file, the result lines equal those of a run on that file alone; with --sis SEED, cloud b's equal the run with SEED + b."""
import subprocess

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import scenes
from test_host_cpp import _write_detector_cfg, cli, write_pcd  # noqa: F401 (cli: the fixture that builds the CLI)

pytestmark = pytest.mark.gpu


def raw_files(tmp_path):
    """Three raw views (no normals: each is preprocessed and its normals estimated on the device)."""
    k = scenes.krylon_cloud()
    clouds = [k["xyz"], scenes.synthetic_raw_scene(7, n_points=15000)["xyz"], scenes.synthetic_raw_scene(8, n_points=15000)["xyz"]]
    paths = []
    for i, xyz in enumerate(clouds):
        p = tmp_path / f"view{i}.pcd"
        write_pcd(p, np.asarray(xyz, np.float32), binary=True)
        paths.append(str(p))
    return paths


def blocks(out):
    """{file: the lines after its CLOUD header} of a --batch run."""
    res, cur = {}, None
    for line in out.splitlines():
        if line.startswith("CLOUD "):
            cur = line.split(" ", 2)[2]
            res[cur] = []
        elif cur is not None:
            res[cur].append(line)
    return res


def result_lines(out):
    """The lines a single-file run prints from its first grasp (or its RESULT line) on."""
    lines = out.splitlines()
    first = next(i for i, l in enumerate(lines) if l.startswith("--- grasp ") or l.startswith("RESULT"))
    return lines[first:]


def test_batch_cli_equals_single_file_runs(cli, tmp_path):  # noqa: F811
    w, _ = load_weights(15)
    cfg = _write_detector_cfg(tmp_path, w, "num_samples = 300\nmin_inliers = 1\nnum_selected = 40\n")
    files = raw_files(tmp_path)
    out = subprocess.check_output([cli, cfg, "--batch"] + files).decode()
    got = blocks(out)
    assert list(got) == files
    n_grasps = 0
    for f in files:
        one = subprocess.check_output([cli, cfg, f]).decode()
        assert got[f] == result_lines(one), f
        n_grasps += int([l for l in got[f] if l.startswith("RESULT")][0].split("n_grasps=")[1].split()[0])
    assert n_grasps > 0


def test_batch_sis_cli_equals_single_file_runs_with_shifted_seeds(cli, tmp_path):  # noqa: F811
    w, _ = load_weights(15)
    cfg = _write_detector_cfg(tmp_path, w, "num_samples = 100\nnum_init_samples = 30\nnum_iterations = 2\n"
                              "num_samples_per_iteration = 40\nprob_rand_samples = 0.25\nstandard_deviation = 0.01\n"
                              "min_score = -1000000\nmin_inliers = 1\nnum_selected = 1000\n")
    files = raw_files(tmp_path)
    out = subprocess.check_output([cli, cfg, "--batch"] + files + ["--sis", "7"]).decode()
    got = blocks(out)
    assert list(got) == files
    sis = lambda lines: [l for l in lines if l.startswith("SIS_") or l.startswith("RESULT")]  # noqa: E731
    for b, f in enumerate(files):
        one = subprocess.check_output([cli, cfg, f, "--sis", str(7 + b)]).decode()
        assert sis(got[f]) == sis(one.splitlines()), f
        assert any(l.startswith("SIS_SAMPLE") for l in got[f])
