"""label_grasps (the reference's src/label_grasps.cpp over the shim, CPU): too few arguments print the usage text and a
missing file its message, each returning -1 before any device is touched."""
import os
import subprocess

from test_host_cpp import HOST, cli  # noqa: F401 (cli: the fixture that builds the host programs)

LABEL = os.path.join(HOST, "label_grasps")
USAGE = ("Error: Not enough input arguments!\n\nUsage: label_grasps CONFIG_FILE PCD_FILE MESH_FILE\n\n"
         "Find grasp poses for a point cloud, PCD_FILE (*.pcd), using parameters from CONFIG_FILE (*.cfg), and check them "
         "against a mesh, MESH_FILE (*.pcd).\n\n")


def run(*args):
    r = subprocess.run([LABEL, *map(str, args)], capture_output=True, text=True)
    return r.returncode, r.stdout


def test_usage_and_missing_files(cli, tmp_path):  # noqa: F811
    for args in ((), ("a.cfg",), ("a.cfg", "b.pcd")):
        assert run(*args) == (255, USAGE)
    cfg, pcd, mesh = tmp_path / "main.cfg", tmp_path / "view.pcd", tmp_path / "mesh.pcd"
    for f in (cfg, pcd, mesh):
        f.write_text("")
    missing = tmp_path / "missing"
    assert run(missing, pcd, mesh) == (255, f"File {missing} could not be found!\nError: CONFIG_FILE not found!\n")
    assert run(cfg, missing, mesh) == (255, f"File {missing} could not be found!\nError: PCD_FILE not found!\n")
    assert run(cfg, pcd, missing) == (255, f"File {missing} could not be found!\nError: MESH_FILE not found!\n")
