"""CPU: the packing of a list of clouds and of per-cloud sample lists into the CSR arrays of gpdb_set_clouds /
gpdb_detect_batch, and the per-cloud views of a batch result."""
import numpy as np
import pytest

from gpd_b200 import abi, lib


def cloud(n, k, seed, cam=True):
    rng = np.random.default_rng(seed)
    return {"xyz": rng.random((n, 3)).astype(np.float32), "normals": rng.random((n, 3)),
            "cam_source": rng.integers(0, 2, (n, k)).astype(np.int32) if cam else None, "view_points": rng.random((k, 3))}


def test_pack_clouds_concatenates_in_cloud_order():
    cs = [cloud(5, 2, 0), cloud(3, 1, 1, cam=False), cloud(4, 3, 2)]
    pk = lib.pack_clouds(cs)
    assert pk["offsets"].tolist() == [0, 5, 8, 12] and pk["offsets"].dtype == np.int32
    assert pk["n_cameras"].tolist() == [2, 1, 3]
    assert np.array_equal(pk["xyz"], np.concatenate([c["xyz"] for c in cs])) and pk["xyz"].dtype == np.float32
    assert np.array_equal(pk["normals"], np.concatenate([c["normals"] for c in cs])) and pk["normals"].dtype == np.float64
    assert np.array_equal(pk["view_points"], np.concatenate([c["view_points"] for c in cs]))
    # cam_source: the N_b x K_b blocks one after the other; a cloud without one is seen by all its cameras
    want = np.concatenate([cs[0]["cam_source"].ravel(), np.ones(3, np.int32), cs[2]["cam_source"].ravel()])
    assert np.array_equal(pk["cam_source"], want) and pk["cam_source"].dtype == np.int32
    assert pk["xyz"].flags.c_contiguous and pk["cam_source"].flags.c_contiguous


def test_pack_clouds_without_camera_sources():
    pk = lib.pack_clouds([cloud(2, 1, 0, cam=False), {"xyz": np.zeros((1, 3)), "normals": np.zeros((1, 3))}])
    assert pk["cam_source"] is None
    assert pk["n_cameras"].tolist() == [1, 1] and pk["view_points"].shape == (2, 3)


def test_pack_samples_csr():
    off, idx = lib.pack_samples([[3, 1], [], np.array([7], np.int64), [0, 0, 2]])
    assert off.tolist() == [0, 2, 2, 3, 6] and idx.tolist() == [3, 1, 7, 0, 0, 2]
    assert off.dtype == np.int32 and idx.dtype == np.int32
    off, idx = lib.pack_samples([[]])
    assert off.tolist() == [0, 0] and len(idx) == 0


def test_split_batch_result_views():
    n, P = 6, 2
    cands = np.zeros(5, dtype=abi.POSE_DTYPE)
    cands["sample_index"] = [0, 1, 2, 3, 4]
    out = {"poses_per_sample": P, "frame_valid": np.arange(n, dtype=np.uint8), "frames": np.arange(n * 9.0).reshape(n, 9),
           "pose_flags": np.zeros((n, P), np.uint8), "pose_scores": np.arange(n * P, dtype=np.float32).reshape(n, P),
           "candidates": cands, "images": np.arange(5)[:, None].repeat(3, 1)}
    v = lib.split_batch_result(out, [0, 2, 2, 6], [0, 3, 3, 5])
    assert [x["n_samples"] for x in v] == [2, 0, 4] and [x["n_candidates"] for x in v] == [3, 0, 2]
    assert v[2]["frame_valid"].tolist() == [2, 3, 4, 5]
    assert v[0]["candidates"]["sample_index"].tolist() == [0, 1, 2] and v[2]["images"][:, 0].tolist() == [3, 4]
    assert np.shares_memory(v[2]["pose_scores"], out["pose_scores"])  # views, not copies


def test_sample_lists_must_match_the_installed_batch():
    """The C-ABI reads B + 1 offsets for the B installed clouds: the binding refuses any other number of lists before the
    call (a context object without a device behind it: the check runs first)."""
    ctx = lib.Context.__new__(lib.Context)
    ctx.h, ctx._n_clouds = None, 2
    for lists in ([[1]], [[1], [2], [3]], []):
        with pytest.raises(ValueError, match="batch of 2 clouds"):
            ctx.detect_batch(lists)
        with pytest.raises(ValueError, match="batch of 2 clouds"):
            ctx.detect_batch_select(lists, 4)
    with pytest.raises(ValueError):
        ctx.detect_batch_raw(np.zeros(2, np.int32), np.zeros(0, np.int32), abi.Result(), np.zeros(3, np.int32))
    ctx._n_clouds = 0  # no batch installed
    with pytest.raises(ValueError, match="batch of 0 clouds"):
        ctx.detect_batch([[1]])
