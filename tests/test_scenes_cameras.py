"""Camera options of the synthetic table scene (CPU): an explicit camera list reproduces the built-in camera sets byte for
byte (bench configs 3-5 and the GPU tests depend on those arrays), and mark_all_cameras only adds cameras to cam_source."""
import numpy as np

from gpd_b200 import scenes

KEYS = ("xyz", "normals", "cam_source", "view_points")


def _same(a, b):
    return all(a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes() for k in KEYS)


def test_camera_list_reproduces_the_builtin_camera_sets():
    assert _same(scenes.synthetic_table_scene(7, n_points=60000),
                 scenes.synthetic_table_scene(7, n_points=60000, cameras=[[0.0, 0.0, 0.0]]))
    assert _same(scenes.synthetic_table_scene(5, n_points=60000, two_cameras=True),
                 scenes.synthetic_table_scene(5, n_points=60000, cameras=[[0.0, 0.0, 0.0], [0.6, 0.0, 0.0]]))


def test_raw_scene_camera_list_reproduces_the_builtin_camera_sets():
    keys = ("xyz", "cam_source", "view_points")
    for kw, cams in (({}, [[0.0, 0.0, 0.0]]), ({"two_cameras": True}, [[0.0, 0.0, 0.0], [0.6, 0.0, 0.0]])):
        a = scenes.synthetic_raw_scene(7, n_points=20000, nan_fraction=0.01, **kw)
        b = scenes.synthetic_raw_scene(7, n_points=20000, nan_fraction=0.01, cameras=cams)
        assert all(a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes() for k in keys)
    cams = [[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.5, 0.1, 0.05]]
    one = scenes.synthetic_raw_scene(5, n_points=20000, cameras=cams)
    allc = scenes.synthetic_raw_scene(5, n_points=20000, cameras=cams, mark_all_cameras=True)
    assert np.array_equal(one["xyz"], allc["xyz"]) and (one["cam_source"].sum(1) == 1).all()
    assert (allc["cam_source"] >= one["cam_source"]).all() and (allc["cam_source"].sum(1) >= 2).mean() > 0.2


def test_mark_all_cameras_adds_every_seeing_camera():
    cams = [[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.5, 0.1, 0.05]]
    one = scenes.synthetic_table_scene(5, n_points=60000, cameras=cams)
    allc = scenes.synthetic_table_scene(5, n_points=60000, cameras=cams, mark_all_cameras=True)
    for k in ("xyz", "normals", "view_points"):
        assert np.array_equal(one[k], allc[k])
    assert (one["cam_source"].sum(1) == 1).all()
    assert ((allc["cam_source"] >= one["cam_source"]).all() and set(np.unique(allc["cam_source"])) == {0, 1})
    assert np.array_equal(np.argmax(allc["cam_source"], axis=1), np.argmax(one["cam_source"], axis=1))
    assert (allc["cam_source"].sum(1) >= 2).mean() > 0.2
    assert one["cam_source"].sum(0).min() > 0  # every camera is the first to see some points
