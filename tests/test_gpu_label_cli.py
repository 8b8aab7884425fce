"""label_grasps CONFIG_FILE PCD_FILE MESH_FILE (-m gpu): the program prints the labels the same steps give through the
Python binding: the view preprocessed (workspace, 3 mm voxels, normals) with its normals flipped, samples drawn above the
support plane with the shim's fixed-seed draws, the hand search's candidates; the mesh's normals estimated without
voxelisation and flipped; gpdb_reevaluate of the candidates against the mesh."""
import re
import subprocess

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from test_gpu_plane_cli import draws
from test_host_cpp import _write_detector_cfg, cli, write_pcd  # noqa: F401 (cli: the fixture that builds the programs)
from test_label_cli import LABEL

pytestmark = pytest.mark.gpu
CAMS4 = np.array([[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.6, 0.0, 0.0], [0.0, 0.6, 0.0]])
NUM_SAMPLES = 150
VP = np.zeros((1, 3))


def flipped(ctx, xyz, pp):
    c = ctx.preprocess(xyz, None, VP, pp)
    ctx.set_cloud(c["xyz"], -c["normals"], c["cam_source"], VP)
    return c


def test_label_grasps_prints_the_binding_labels(cli, tmp_path):  # noqa: F811
    view = scenes.synthetic_raw_scene(6, n_points=20000)["xyz"]
    mesh = scenes.synthetic_raw_scene(6, n_points=20000, step=0.003, cameras=CAMS4, mark_all_cameras=True)["xyz"]
    write_pcd(tmp_path / "view.pcd", view, binary=True)
    write_pcd(tmp_path / "mesh.pcd", mesh, binary=True)
    w, _ = load_weights(15)
    cfg = _write_detector_cfg(tmp_path, w, f"num_samples = {NUM_SAMPLES}\n")
    r = subprocess.run([LABEL, cfg, str(tmp_path / "view.pcd"), str(tmp_path / "mesh.pcd")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = r.stdout
    assert f"num_threads: 1, num_samples: {NUM_SAMPLES}\nsample_above_plane: 1\nnormals_radius: 0.030\n" in out

    ctx = lib.Context(lib.default_params(channels=15))
    v = flipped(ctx, view, lib.preprocess_params(voxelize=1, voxel_size=0.003, normals_radius=0.03))
    _, n_in, elig = ctx.segment_plane()
    assert 0 < n_in < len(v["xyz"])
    sidx = np.array(draws(np.flatnonzero(elig), NUM_SAMPLES), np.int32)
    cand = ctx.hand_search(sidx)["candidates"]
    assert len(cand) > 0
    inf = float("inf")
    flipped(ctx, mesh, lib.preprocess_params(voxelize=0, normals_radius=0.03, workspace=[-inf, inf, -inf, inf, -inf, inf]))
    labels, recs = ctx.reevaluate(cand)
    ctx.close()

    assert f"labels: {len(cand)}\n" in out
    lines = re.findall(r"^\((\d+)\) label: (\d)$", out, re.M)
    seen = np.zeros(len(cand), int)
    for i, lb in lines:
        assert int(lb) == labels[int(i)], i
        seen[int(i)] += 1
    assert np.array_equal(seen, 1 + recs["full_antipodal"])  # a full antipodal hand's line comes twice, as upstream
