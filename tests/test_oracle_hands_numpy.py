"""Second, independent restatement of the hand search (A3-A7) in numpy, written from the reference sources
(hand_set.cpp:31-116,235-261, finger_hand.cpp, antipodal.cpp:10-96, hand.cpp:24-45, point_list.cpp:22-55; filters: grasp_detector.cpp:334-398,422-456) separately from
the C++ oracle, and compared with it pose by pose. The reference cannot run here (Eigen / PCL are absent), so this is a
cross-check between two restatements, not a pin against upstream binaries; it guards the oracle — the checker of every GPU
parity test — against transcription errors. The local frames and the neighbourhoods come from the oracle (pinned
separately: eigen-solver against numpy.linalg.eigh, radius search against brute force)."""
import numpy as np
import pytest

from gpd_b200 import abi, scenes
from hand_reference import filtered, hand_set
from oracle import oracle


@pytest.mark.parametrize("scene,over", [
    ("krylon", {}), ("table", {}), ("table", {"hand_axes": [0, 1, 2], "num_orientations": 4, "deepen_hand": 0}),
    ("table", {"filter_approach_direction": 1, "direction": [0.0, 0.0, 1.0], "thresh_rad": 1.2, "max_aperture": 0.07,
               "workspace_grasps": [-0.5, 0.5, -0.4, 0.4, 0.0, 0.95]})])
def test_hand_search_oracle_matches_the_numpy_restatement(scene, over):
    c = scenes.krylon_cloud() if scene == "krylon" else scenes.synthetic_table_scene(7, n_points=60000)
    oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    p = abi.default_params(15, **over)
    sidx = scenes.sample_indices(2 if scene == "krylon" else 3, len(c["xyz"]), 40)
    frames, valid = oc.frames(p, sidx)
    poses, flags = oc.hand_search(p, sidx, frames, valid)
    n_valid = mism = 0
    for i, si in enumerate(sidx):
        if not valid[i]:
            continue
        q = c["xyz"][si]
        idx, _ = oc.radius_search(q, 0.11)                                       # hand_search.cpp:13-17,178
        ref = hand_set(p, q.astype(np.float64), frames[i], c["xyz"][idx].astype(np.float64), c["normals"][idx])
        for j, r in enumerate(ref):
            got_valid = bool(flags[i, j] & abi.POSE_VALID)
            if (r is not None) != got_valid:
                mism += 1
                continue
            if r is None:
                continue
            n_valid += 1
            g = poses[i, j]
            assert list(g["frame"]) == r["frame"] and list(g["position"]) == r["position"]
            assert g["top"] == r["top"] and g["bottom"] == r["bottom"] and g["center"] == r["center"]
            assert g["width"] == r["width"] and g["finger_idx"] == r["finger_idx"]
            assert bool(g["half_antipodal"]) == r["half"] and bool(g["full_antipodal"]) == r["full"]
            assert bool(flags[i, j] & abi.POSE_HALF) == r["half"] and bool(flags[i, j] & abi.POSE_FULL) == r["full"]
            assert bool(flags[i, j] & abi.POSE_FILTERED) == filtered(p, r)                          # A15
    # the restatement evaluates every hand-frame product and sum in the oracle's order: records equal bit for bit
    assert mism == 0 and n_valid >= 20, (mism, n_valid)


def test_local_frames_against_numpy_eigh():
    """LocalFrame::findAverageNormalAxis (local_frame.cpp:14-41) against numpy.linalg.eigh on the same r = nn_radius
    balls: the normal (largest eigenvalue, flipped to agree with the summed normals) must match, the curvature axis
    (smallest eigenvalue) up to the sign that only Eigen's iterative solver fixes (restated in the oracle, SURVEY 9.1),
    and binormal = curvature x normal."""
    c = scenes.synthetic_table_scene(7, n_points=60000)
    oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    p = abi.default_params(15)
    sidx = scenes.sample_indices(3, 60000, 200)
    frames, valid = oc.frames(p, sidx)
    checked = 0
    for i, si in enumerate(sidx):
        idx, _ = oc.radius_search(c["xyz"][si], p.nn_radius)
        assert bool(valid[i]) == (len(idx) > 0)
        if not valid[i]:
            continue
        Nn = c["normals"][idx]
        w, v = np.linalg.eigh(Nn.T @ Nn)
        if (w[1] - w[0]) < 1e-6 * w[2] or (w[2] - w[1]) < 1e-6 * w[2]:
            continue  # (near-)degenerate spectrum: the eigenvectors are not unique
        normal = v[:, 2] if v[:, 2] @ Nn.sum(0) >= 0 else -v[:, 2]
        f = frames[i].reshape(3, 3)                      # rows: normal | binormal | curvature axis (column-major 3x3)
        assert np.allclose(f[0], normal, atol=1e-9)
        s = np.sign(f[2] @ v[:, 0])
        assert np.allclose(f[2], s * v[:, 0], atol=1e-9)
        assert np.allclose(f[1], np.cross(f[2], f[0]), atol=1e-12)
        checked += 1
    assert checked >= 150
