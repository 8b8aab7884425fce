"""Batches of clouds (gpdb_set_clouds / gpdb_detect_batch / gpdb_detect_batch_select) off the defaults, on the GPU.

Every case holds each cloud's slice of the batch bit-equal to gpdb_detect on that cloud alone (test_gpu_batch's
contract), at least one cloud of the batch against the CPU oracle at the bars of test_gpu_parity.assert_parity, and
checks from its own inputs that it reaches the path it names: camera counts and image tiers (mixed K_b, all_seen per
cloud), hand geometry and search parameters, finger placements, the orientation count at 1 and 32, grids whose cell
grew past 2 cm (batch_param_cases.py), the batch-wide cell-count guard, and exact ties in selection.
"""
import ctypes as C
import os

import numpy as np
import pytest

from batch_param_cases import (GUARD_CLOUDS, cam_scene, guard_clouds, partial_tie_weights, table, tie_weights,
                               with_outliers)
from conftest import load_weights
from gpd_b200 import abi, lib, scenes
from preprocess_cases import grid_of
from test_gpu_batch import ERR_CAPACITY, ERR_STATE, assert_same, check_batch, check_oracle, context, nonunit, raw_detect_batch
from test_gpu_geometry_params import FAST_2CAM_DEPTH, HANDS, _cfg
from test_gpu_parity import _lattice_cloud, assert_parity, make

pytestmark = pytest.mark.gpu


def run_batch(ctx, samples):
    """detect_batch, plus the kernel launches of the call."""
    offsets, sidx = ctx._pack_batch_samples(samples)
    res = abi.Result()
    coff = np.zeros(len(offsets), np.int32)
    ctx._check(lib.lib().gpdb_detect_batch(ctx.h, offsets.ctypes.data_as(C.c_void_p), sidx.ctypes.data_as(C.c_void_p),
                                           C.byref(res), coff.ctypes.data_as(C.c_void_p)))
    S, Cc = ctx.params.image_size, ctx.params.image_num_channels
    out = abi.result_to_numpy(res, S * S * Cc)
    lib.free_result(res)
    return lib.split_batch_result(out, offsets, coff), out["kernel_launches"]


def batch_both_tiers(ctx, samples, monkeypatch):
    """(default views, extra launches of the default run over the general image tier forced), the two bit-equal."""
    monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    general, lg = run_batch(ctx, samples)
    monkeypatch.delenv("GPD_B200_IMAGES_KERNEL")
    default, ld = run_batch(ctx, samples)
    for d, g in zip(default, general):
        assert_same(d, g)
    return default, ld - lg


# ---- camera counts ----------------------------------------------------------------------------------------------------
def camera_case(name):
    """(channels, parameter overrides, clouds, whether the fast image tier runs, cloud held against the oracle)."""
    if name == "15ch_k123":  # b_maxk = 3: the general tier for every cloud
        return 15, {}, [cam_scene(1, seed=5), cam_scene(2, seed=6), cam_scene(3, seed=7)], False, 2
    if name == "15ch_k12_fast":  # two cameras' bitmaps fit k_images2 at 5 mm less depth
        return 15, {"volume_depth": FAST_2CAM_DEPTH}, [cam_scene(1, seed=5), cam_scene(2, seed=6)], True, 1
    if name == "12ch_k1468":  # no shadows at 12 channels: the fast tier at any camera count
        return 12, {}, [cam_scene(k, seed=4 + k) for k in (1, 4, 6, 8)], True, 3
    # all_seen differs between clouds: marked clouds with ~10 % unseen rows beside clouds without a camera-source matrix
    clouds = [cam_scene(2, seed=5, mark_all=True, zero_rows=0.1), dict(cam_scene(2, seed=6), cam_source=None),
              cam_scene(1, seed=7, mark_all=True, zero_rows=0.1), dict(cam_scene(1, seed=8), cam_source=None)]
    return 15, {"volume_depth": FAST_2CAM_DEPTH}, clouds, True, 0


@pytest.mark.parametrize("name", ["15ch_k123", "15ch_k12_fast", "12ch_k1468", "15ch_all_seen_mix"])
def test_mixed_camera_counts(name, monkeypatch):
    ch, over, clouds, fast, o = camera_case(name)
    p, ctx, w = context(ch, **over)
    ks = [len(c["view_points"]) for c in clouds]
    assert (max(ks) <= 2) == fast or ch == 12
    seen = [c["cam_source"] is None or bool((c["cam_source"] > 0).all()) for c in clouds]
    if name == "15ch_all_seen_mix":
        assert seen == [False, True, False, True]
        for c in clouds[::2]:
            bits = c["cam_source"].sum(1)
            assert (bits == 0).mean() > 0.05 and (len(c["view_points"]) == 1 or (bits >= 2).mean() > 0.2)
    samples = [scenes.sample_indices(5, len(c["xyz"]), 150) for c in clouds]
    ctx.set_clouds(clouds)
    views, extra = batch_both_tiers(ctx, samples, monkeypatch)
    assert (extra > 0) == fast
    for rb, rs in zip(views, check_batch(ctx, clouds, samples)):
        assert_same(rb, rs)
    assert views[o]["n_candidates"] >= 20
    check_oracle(p, w, clouds[o], samples[o], views[o], ch)
    ctx.close()


def test_four_camera_cloud_in_a_15ch_batch_is_a_clean_error():
    """The shadow bitmaps of a batch are sized for its largest camera count: one 4-camera cloud among 2-camera clouds
    does not fit the general tier's shared memory at 15 channels. GPDB_ERR_INVALID, and the context then runs a valid batch."""
    p, ctx, w = context(15)
    clouds = [cam_scene(2, seed=6), cam_scene(4, seed=5)]
    samples = [scenes.sample_indices(5, len(c["xyz"]), 80) for c in clouds]
    ctx.set_clouds(clouds)
    for call in (ctx.detect_batch, lambda s: ctx.detect_batch_select(s, 5)):
        with pytest.raises(lib.GpdbError) as e:
            call(samples)
        assert e.value.code == -1 and "shared memory" in str(e.value)
    good = [cam_scene(3, seed=7), cam_scene(1, seed=5)]
    samples = [scenes.sample_indices(5, len(c["xyz"]), 120) for c in good]
    views = check_batch(ctx, good, samples)
    assert views[0]["n_candidates"] >= 20
    check_oracle(p, w, good[0], samples[0], views[0])
    ctx.close()


# ---- hand geometry, search parameters, finger placements ------------------------------------------------------------
HAND_CASES = dict(HANDS, all_axes_filters={
    "hand_axes": [0, 1, 2], "num_orientations": 4, "num_finger_placements": 7, "deepen_hand": 0,
    "filter_approach_direction": 1, "direction": [0.0, 0.0, 1.0], "thresh_rad": 1.2, "max_aperture": 0.07,
    "workspace_grasps": [-0.5, 0.5, -0.4, 0.4, 0.0, 1.0]})


@pytest.mark.parametrize("name", list(HAND_CASES))
def test_hand_and_search_parameters(name, golden_dir):
    over = dict(HAND_CASES[name])
    if name.startswith("ur5"):
        c = _cfg(os.path.join(golden_dir, "cfg", "ur5_hand_geometry.cfg"))
        over.update({k: c[k] for k in ("finger_width", "hand_outer_diameter", "hand_depth", "hand_height", "init_bite")})
    p, ctx, w = context(15, **over)
    clouds = [table(7, n=30000), scenes.krylon_cloud(), table(4, two_cameras=True), nonunit(table(6))]
    samples = [scenes.sample_indices(3, len(c["xyz"]), n) for c, n in zip(clouds, (200, 100, 120, 100))]
    views = check_batch(ctx, clouds, samples)
    assert views[0]["n_candidates"] >= 20
    check_oracle(p, w, clouds[0], samples[0], views[0])
    flags = np.concatenate([v["pose_flags"] for v in views])
    if "hand_axes" in over:
        assert (flags.reshape(-1, 3, 4) & 3 == 3).any(axis=(0, 2)).all()  # candidates on every hand axis
    if name == "all_axes_filters":
        assert (flags & 1).sum() > (flags & 2).sum() // 2 > 0  # the filters actually filter
    ctx.close()


@pytest.mark.parametrize("nfp", [1, 2, 13, 16])
def test_finger_placements(nfp):
    """The linear slot scan of the hand search. With one or two placements few points have a collision-free placement:
    every point of small clouds is a sample. Chunks of chunk_samples end inside clouds."""
    k = scenes.krylon_cloud()
    if nfp <= 2:
        chunk, clouds = 1400, [table(7, n=6000), k, table(3, n=6000)]
        samples = [np.arange(len(c["xyz"]), dtype=np.int32) for c in clouds]
    else:
        chunk, clouds = 64, [table(7, n=30000), k, table(3)]
        samples = [scenes.sample_indices(3, len(c["xyz"]), 150) for c in clouds]
    p, ctx, w = context(15, num_finger_placements=nfp, chunk_samples=chunk)
    ends = np.cumsum([len(s) for s in samples])
    assert ends[-1] > 2 * chunk and (ends[:-1] % chunk != 0).all()
    views = check_batch(ctx, clouds, samples)
    o = int(np.argmax([v["n_candidates"] for v in views]))
    assert views[o]["n_candidates"] > 0
    check_oracle(p, w, clouds[o], samples[o], views[o])
    ctx.close()


# ---- orientation count ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("axes,n_orient", [([2], 1), ([0, 1, 2], 32)])
def test_orientation_count_edges(axes, n_orient):
    """P = 1 (one axis, one orientation) and P = 96 (three axes, GPDB_MAX_ORIENT = 32): the single cloud and a batch."""
    over = {"hand_axes": axes, "num_orientations": n_orient}
    s = table(7, n=30000)
    p, ctx, oc, w = make(s, 15, keep_images=1, **over)
    sidx = scenes.sample_indices(3, len(s["xyz"]), 250 if n_orient == 1 else 80)
    rg = ctx.detect(sidx)
    assert rg["poses_per_sample"] == len(axes) * n_orient and rg["n_candidates"] > 0
    assert_parity(oc.detect(p, w, sidx), rg, 15)
    ctx.close()
    p, ctx, w = context(15, **over)
    k = scenes.krylon_cloud()
    clouds = [table(3), k, table(4, two_cameras=True)]
    samples = [scenes.sample_indices(1, 20000, 100), scenes.sample_indices(2, len(k["xyz"]), 60),
               scenes.sample_indices(1, 20000, 80)]
    views = check_batch(ctx, clouds, samples)
    assert views[1]["n_candidates"] > 0
    check_oracle(p, w, k, samples[1], views[1])
    ctx.close()


def test_orientation_count_above_the_limit():
    with pytest.raises(lib.GpdbError) as e:
        lib.Context(lib.default_params(num_orientations=33))
    assert e.value.code == -1 and "num_orientations" in str(e.value)


# ---- grown grid cells ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist,steps", [(8.0, 1), (12.0, 2)])
def test_grown_cells_single_cloud_matches_oracle(dist, steps):
    """Outliers 8 / 12 m away: the grid's cell grows to 3 / 4.5 cm. Frames, hands, images and scores as the oracle's."""
    s = with_outliers(table(7, n=30000), dist)
    assert grid_of(s["xyz"])[4] == steps
    p, ctx, oc, w = make(s, 15, keep_images=1)
    sidx = scenes.sample_indices(3, 30000, 200)
    rg = ctx.detect(sidx)
    assert rg["n_candidates"] >= 20
    assert_parity(oc.detect(p, w, sidx), rg, 15)
    ctx.close()


def test_grown_cells_in_a_batch():
    """Clouds of 2, 3 and 4.5 cm cells in one batch; then the dense lattice of test_overflow_tiers_inside_a_batch inside
    a 3 cm grid (more points per cell: more candidates per scanned row for every tier)."""
    p, ctx, w = context(15)
    k = scenes.krylon_cloud()
    clouds = [table(3), with_outliers(table(4), 8.0), k, with_outliers(table(6, two_cameras=True), 12.0), table(8)]
    assert [grid_of(c["xyz"])[4] for c in clouds] == [0, 1, 0, 2, 0]
    samples = [scenes.sample_indices(1, 20000, 120), scenes.sample_indices(2, 20000, 120),
               scenes.sample_indices(2, len(k["xyz"]), 80), scenes.sample_indices(1, 20000, 120), []]
    views = check_batch(ctx, clouds, samples)
    assert all(v["n_candidates"] > 0 for v in views[:4])
    check_oracle(p, w, clouds[3], samples[3], views[3])
    dense, rng = _lattice_cloud(0.0012)
    center = np.argsort(np.linalg.norm(dense["xyz"][:, :2], axis=1))[:2000]
    sd = center[rng.choice(2000, 40, replace=False)].astype(np.int32)
    dg = with_outliers(dense, 8.0)
    assert grid_of(dg["xyz"])[4] == 1
    views = check_batch(ctx, [table(3), dg, k], [scenes.sample_indices(1, 20000, 100), sd,
                                                 scenes.sample_indices(2, len(k["xyz"]), 80)])
    assert views[1]["n_candidates"] > 0
    check_oracle(p, w, dg, sd, views[1])
    ctx.close()


def test_batch_cell_guard():
    """46 two-point clouds of 7.2 m: each grid keeps its 2 cm cell (just under 48e6 cells), together they exceed
    INT_MAX - 1 cells. gpdb_set_clouds refuses them before it allocates the cell table and leaves no batch."""
    p, ctx, w = context(15)
    clouds = guard_clouds()
    total = sum(grid_of(c["xyz"])[3] for c in clouds)
    assert len(clouds) == GUARD_CLOUDS and total > 2 ** 31 - 2
    with pytest.raises(lib.GpdbError) as e:
        ctx.set_clouds(clouds)
    assert e.value.code == ERR_CAPACITY and f"need {int(total)} cells" in str(e.value)
    assert raw_detect_batch(ctx, [0, 0], np.zeros(0, np.int32)) == ERR_STATE  # no batch is left
    k = scenes.krylon_cloud()
    samples = [scenes.sample_indices(1, 20000, 100), scenes.sample_indices(2, len(k["xyz"]), 80)]
    views = check_batch(ctx, [table(3), k], samples)
    check_oracle(p, w, k, samples[1], views[1])
    ctx.close()


# ---- ties in selection ------------------------------------------------------------------------------------------------
def tie_context(weights, impl):
    w, relu = load_weights(15)
    p = lib.default_params(channels=15, relu_after_conv=relu, lenet_impl=impl, chunk_samples=64)
    ctx = lib.Context(p)
    ctx.set_weights(weights(w))
    return ctx


def tie_clouds():
    k = scenes.krylon_cloud()
    return ([table(3), k, table(4, two_cameras=True)],
            [scenes.sample_indices(1, 20000, 200), scenes.sample_indices(2, len(k["xyz"]), 150),
             scenes.sample_indices(1, 20000, 150)])


def assert_select_is_sorted_detect(ctx, sidx, want_order):
    """detect_select(k) = the first k candidates of detect in want_order(candidates), for k at the edges and inside a
    chunk (chunk_samples = 64), field by field."""
    cand = ctx.detect(sidx)["candidates"]
    order = want_order(cand)
    first_chunk = int((cand["sample_slot"] < 64).sum())
    second_chunk = int((cand["sample_slot"] < 128).sum())
    assert 0 < first_chunk < second_chunk < len(cand)
    n_pos = int((cand["score"] > 0).sum())  # partial ties: the zeros follow the positive scores
    for k in (0, 1, (first_chunk + second_chunk) // 2, n_pos + (len(cand) - n_pos) // 2, len(cand), len(cand) + 7):
        r = ctx.detect_select(sidx, k)
        kk = min(k, len(cand))
        assert r["n_candidates"] == kk and r["n_total_candidates"] == len(cand)
        for f in cand.dtype.names:
            assert np.array_equal(r["candidates"][f], cand[order[:kk]][f]), (k, f)
    return cand


def assert_batch_select_is_single_select(ctx, clouds, samples, k):
    ctx.set_clouds(clouds)
    got = ctx.detect_batch_select(samples, k)
    for g, c, s in zip(got, clouds, samples):
        ctx.set_cloud(c["xyz"], c["normals"], c.get("cam_source"), c.get("view_points"))
        want = ctx.detect_select(np.asarray(s, np.int32), k)["candidates"]
        assert len(want) > 0 and g.tobytes() == want.tobytes()


@pytest.mark.parametrize("impl", [0, 1])  # 0 = wgmma convolutions, 1 = SIMT float32
def test_exact_ties_select_in_candidate_order(impl):
    """Equal ip2 rows and biases: every score is exactly +0.0, so selection is candidate order alone."""
    ctx = tie_context(tie_weights, impl)
    clouds, samples = tie_clouds()
    c = clouds[0]
    ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    cand = assert_select_is_sorted_detect(ctx, samples[0], lambda cd: np.arange(len(cd)))
    assert (cand["score"].view(np.uint32) == 0).all(), f"lenet_impl {impl}: equal ip2 rows gave unequal logits"
    for k in (1, 40, 10000):
        assert_batch_select_is_single_select(ctx, clouds, samples, k)
    ctx.close()


@pytest.mark.parametrize("impl", [0, 1])
def test_partial_ties_follow_the_stable_sort(impl):
    """ip2 rows equal but for one ip1 unit: exact zeros wherever that unit is 0 after the ReLU, distinct scores
    elsewhere; selection is the host's stable sort on descending score."""
    ctx = tie_context(partial_tie_weights, impl)
    clouds, samples = tie_clouds()
    c = clouds[0]
    ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    cand = assert_select_is_sorted_detect(ctx, samples[0], lambda cd: np.argsort(-cd["score"], kind="stable"))
    s = cand["score"]
    assert (s == 0).sum() >= 0.2 * len(s) and len(np.unique(s[s != 0])) >= 0.2 * len(s)
    for k in (1, 40, 10000):
        assert_batch_select_is_single_select(ctx, clouds, samples, k)
    ctx.close()
