"""GPU parity off the default geometry (-m gpu): camera counts and camera sets, image sizes, finger placements, hand and
image-volume parameters, each against the CPU oracle under the contract of test_gpu_parity.py (flags, frames and pose
records exact; images <= 1 LSB on <= 1e-3 of the pixels; scores within 1e-4 of max |score|).

Which image kernel ran is read from `kernel_launches` of gpdb_detect: the fast path (k_images2, then k_images over its
overflow list) launches one kernel more per image batch than the general tier alone, which GPD_B200_IMAGES_KERNEL=1
forces. Every case here has a single image batch.
"""
import os

import numpy as np
import pytest

from gpd_b200 import lib, scenes
from oracle import oracle
from test_gpu_parity import assert_parity, make

pytestmark = pytest.mark.gpu

# cameras in front of the table (z = 0.9), looking along +z
CAMS = [[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.5, 0.1, 0.05], [0.0, 0.5, 0.0], [0.1, -0.5, 0.1], [0.45, 0.45, 0.0],
        [-0.4, -0.4, 0.0], [0.3, -0.2, -0.2]]
# the largest image depth at which two cameras' 15-channel shadow bitmaps fit k_images2 (bm_dim 46 instead of 48)
FAST_2CAM_DEPTH = 0.05


def scene(k, mark_all=False, seed=5):
    return scenes.synthetic_table_scene(seed, n_points=60000, cameras=CAMS[:k], mark_all_cameras=mark_all)


def detect_both_tiers(ctx, sidx, monkeypatch):
    """(default result, result with the general image tier forced, extra launches of the default path)."""
    monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    general = ctx.detect(sidx)
    monkeypatch.delenv("GPD_B200_IMAGES_KERNEL")
    default = ctx.detect(sidx)
    assert np.array_equal(default["pose_flags"], general["pose_flags"])
    if default["images"] is not None:
        assert np.array_equal(default["images"], general["images"])
    assert np.array_equal(default["pose_scores"], general["pose_scores"], equal_nan=True)
    return default, general, default["kernel_launches"] - general["kernel_launches"]


def check_against_oracle(cloud, ch, sidx, monkeypatch, fast, **over):
    p, ctx, oc, w = make(cloud, ch, keep_images=1, **over)
    rg, _, extra = detect_both_tiers(ctx, sidx, monkeypatch)
    ro = oc.detect(p, w, sidx)
    assert_parity(ro, rg, ch)
    assert rg["n_candidates"] >= 20
    assert extra == (1 if fast else 0)
    ctx.close()
    return ro


def test_two_cameras_15ch_fast_path_matches_oracle(monkeypatch):
    """k_images2's two-camera shadow: at the default image volume two 15-channel bitmaps (2 x 2 x 48^2 x 4 B) fill the
    whole box list and only the general tier runs; 5 mm less depth and the fast path takes them."""
    s = scenes.synthetic_table_scene(5, n_points=60000, two_cameras=True)
    sidx = scenes.sample_indices(5, 60000, 250)
    p, ctx, _, _ = make(s, 15)
    assert detect_both_tiers(ctx, sidx, monkeypatch)[2] == 0
    ctx.close()
    check_against_oracle(s, 15, sidx, monkeypatch, True, volume_depth=FAST_2CAM_DEPTH)


def test_three_cameras_15ch_matches_oracle(monkeypatch):
    check_against_oracle(scene(3), 15, scenes.sample_indices(5, 60000, 250), monkeypatch, False)


@pytest.mark.parametrize("k", [4, 6, 8])
def test_many_cameras_12ch_match_oracle(k, monkeypatch):
    """12 channels cast no shadows: any camera count (up to GPDB_MAX_CAMERAS) runs the fast path."""
    check_against_oracle(scene(k), 12, scenes.sample_indices(5, 60000, 200), monkeypatch, True)


def test_four_cameras_15ch_is_a_clean_error():
    """Four 15-channel shadow bitmaps do not fit the general tier's shared memory: GPDB_ERR_INVALID, no fault, and the
    context keeps working with a cloud of two cameras."""
    sidx = scenes.sample_indices(5, 60000, 100)
    p, ctx, _, w = make(scene(4), 15)
    for call in (ctx.detect, lambda i: ctx.images(ctx.hand_search(i)["candidates"])):
        with pytest.raises(lib.GpdbError) as e:
            call(sidx)
        assert e.value.code == -1 and "shared memory" in str(e.value)
    s2 = scene(2)
    ctx.set_cloud(s2["xyz"], s2["normals"], s2["cam_source"], s2["view_points"])
    oc = oracle.OracleCloud(s2["xyz"], s2["normals"], s2["cam_source"], s2["view_points"])
    rg = ctx.detect(sidx)
    ro = oc.detect(p, w, sidx)
    assert rg["n_candidates"] > 0
    assert np.array_equal(ro["pose_flags"], rg["pose_flags"])
    m = ~np.isnan(ro["pose_scores"])
    assert np.abs(ro["pose_scores"][m] - rg["pose_scores"][m]).max() <= 1e-4 * np.abs(ro["pose_scores"][m]).max()
    ctx.close()


@pytest.mark.parametrize("width,bm_dim", [(0.116, 52), (0.12, 53)])
def test_general_tier_shared_memory_bound(width, bm_dim):
    """Three 15-channel shadow bitmaps at the edge of k_images' shared memory: dynamic + static may not pass the device's
    opt-in maximum per block (232 448 B on H100, of which the static part takes 9 520 B). bm_dim 52 needs 221 680 B of
    dynamic memory and runs; bm_dim 53 needs 224 208 B and is refused with GPDB_ERR_INVALID, after which the same
    context still makes images."""
    s = scene(3)
    sidx = scenes.sample_indices(5, 60000, 100)
    p, ctx, oc, _ = make(s, 15, volume_width=width)
    cand = ctx.hand_search(sidx)["candidates"]
    assert len(cand) > 20
    if bm_dim == 53:
        with pytest.raises(lib.GpdbError) as e:
            ctx.images(cand)
        assert e.value.code == -1 and "shared memory" in str(e.value), str(e.value)
        s = scene(2)
        ctx.set_cloud(s["xyz"], s["normals"], s["cam_source"], s["view_points"])
        oc = oracle.OracleCloud(s["xyz"], s["normals"], s["cam_source"], s["view_points"])
        cand = ctx.hand_search(sidx)["candidates"]
    io, ig = oc.images(p, cand), ctx.images(cand)
    d = np.abs(io.astype(np.int32).reshape(ig.shape) - ig.astype(np.int32))
    assert io.max() > 0 and d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    ctx.close()


@pytest.mark.parametrize("k,fast", [(2, True), (3, False)])
def test_multi_camera_and_unseen_points_15ch(k, fast, monkeypatch):
    """cam_source rows with several cameras (every camera that sees the point) and with none: the shadow's camera set."""
    s = scene(k, mark_all=True)
    bits = s["cam_source"].sum(1)
    s["cam_source"][np.random.default_rng(k).random(60000) < 0.1] = 0
    assert (bits >= 2).mean() > 0.2 and (s["cam_source"].sum(1) == 0).mean() > 0.05
    over = {"volume_depth": FAST_2CAM_DEPTH} if fast else {}
    check_against_oracle(s, 15, scenes.sample_indices(5, 60000, 250), monkeypatch, fast, **over)


@pytest.mark.parametrize("ch", [12, 15])
@pytest.mark.parametrize("size", [57, 61, 48, 64])
def test_image_sizes(size, ch):
    """Image sizes other than 60 through hand search + images against the oracle: odd sizes (an odd number of 8-byte
    cells per projection tile), sizes that are not multiples of 4 (padded plane rows), 61 = the largest that fits at 15
    channels. LeNet needs 60 (61 would also reach ip1 with 7200 inputs), so gpdb_detect reports GPDB_ERR_INVALID.
    64 x 64 x 15 does not fit shared memory: GPDB_ERR_INVALID."""
    s = scenes.synthetic_table_scene(7, n_points=60000)
    p, ctx, oc, w = make(s, ch, image_size=size)
    sidx = scenes.sample_indices(3, 60000, 150)
    cand = ctx.hand_search(sidx)["candidates"]
    assert len(cand) > 100
    if size == 64 and ch == 15:
        with pytest.raises(lib.GpdbError) as e:
            ctx.images(cand)
        assert e.value.code == -1 and "shared memory" in str(e.value)
    else:
        io, ig = oc.images(p, cand), ctx.images(cand)
        d = np.abs(io.astype(np.int32).reshape(ig.shape) - ig.astype(np.int32))
        assert io.max() > 0 and d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect(sidx)
    assert e.value.code == -1
    assert len(ctx.hand_search(sidx)["candidates"]) == len(cand)  # the context still works
    ctx.close()


@pytest.mark.parametrize("nfp", [1, 2, 13, 16])
def test_finger_placements_linear_slot_scan(nfp, monkeypatch):
    """Finger placements whose slots overlap (13, 16 with the default hand) or are too few (1, 2) for the arithmetic
    slot lookup: the hand search scans the slots linearly. With one or two placements a finger always starts at the
    sample, so only a few dozen points of the scene (edges) have a collision-free placement: those take every point."""
    s = scenes.synthetic_table_scene(7, n_points=60000)
    if nfp <= 2:  # one chunk: one image batch
        check_against_oracle(s, 15, np.arange(60000, dtype=np.int32), monkeypatch, True, num_finger_placements=nfp,
                             chunk_samples=60000)
    else:
        check_against_oracle(s, 15, scenes.sample_indices(3, 60000, 200), monkeypatch, True, num_finger_placements=nfp)


def _cfg(path):
    out = {}
    for line in open(path):
        line = line.split("#")[0].strip()
        if "=" in line:
            k, v = (t.strip() for t in line.split("=", 1))
            out[k] = float(v)
    return out


HANDS = {
    "ur5": {},  # filled from tests/golden/cfg/ur5_hand_geometry.cfg
    "ur5_all_axes": {"hand_axes": [0, 1, 2], "num_orientations": 4},
    "deep_tall": {"hand_depth": 0.08, "init_bite": 0.015, "hand_height": 0.03},
    "large_volume": {"volume_width": 0.12, "volume_depth": 0.08, "volume_height": 0.03},
    "nn_radius_2cm": {"nn_radius": 0.02},
}


@pytest.mark.parametrize("name", list(HANDS))
def test_hand_and_volume_parameters(name, golden_dir, monkeypatch):
    """Hand geometry, image volume and normal radius off their defaults: slab height, deepen steps, search / image
    radii, shadow draws and bitmap size all follow from them."""
    over = dict(HANDS[name])
    if name.startswith("ur5"):
        c = _cfg(os.path.join(golden_dir, "cfg", "ur5_hand_geometry.cfg"))
        over.update({k: c[k] for k in ("finger_width", "hand_outer_diameter", "hand_depth", "hand_height", "init_bite")})
    s = scenes.synthetic_table_scene(7, n_points=60000)
    ro = check_against_oracle(s, 15, scenes.sample_indices(3, 60000, 200), monkeypatch, True, **over)
    if name == "ur5_all_axes":
        assert (ro["pose_flags"].reshape(-1, 3, 4) & 3 == 3).any(axis=(0, 2)).all()  # candidates on every hand axis
