"""pack_clouds for raw clouds (gpdb_preprocess_clouds): clouds without normals, on the CPU."""
import numpy as np
import pytest

from gpd_b200 import lib


def raw(n, k, seed, normals=False):
    rng = np.random.default_rng(seed)
    c = {"xyz": rng.random((n, 3)).astype(np.float32), "cam_source": rng.integers(0, 2, (n, k)).astype(np.int32),
         "view_points": rng.random((k, 3))}
    if normals:
        c["normals"] = rng.random((n, 3))
    return c


def test_clouds_without_normals_pack_to_none():
    cs = [raw(5, 1, 0), raw(3, 2, 1), dict(raw(4, 1, 2), normals=None)]
    pk = lib.pack_clouds(cs)
    assert pk["normals"] is None
    assert list(pk["offsets"]) == [0, 5, 8, 12] and list(pk["n_cameras"]) == [1, 2, 1]
    assert np.array_equal(pk["xyz"], np.concatenate([c["xyz"] for c in cs]))
    assert np.array_equal(pk["cam_source"], np.concatenate([c["cam_source"].ravel() for c in cs]))
    assert pk["view_points"].shape == (4, 3)


def test_clouds_with_normals_pack_as_before():
    cs = [raw(5, 1, 0, normals=True), raw(3, 2, 1, normals=True)]
    pk = lib.pack_clouds(cs)
    assert pk["normals"].dtype == np.float64 and np.array_equal(pk["normals"], np.concatenate([c["normals"] for c in cs]))


def test_normals_on_some_clouds_only_are_refused():
    with pytest.raises(ValueError, match="clouds \\[1\\] have no normals"):
        lib.pack_clouds([raw(5, 1, 0, normals=True), raw(3, 2, 1)])
