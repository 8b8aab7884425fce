"""Sample positions in a batch of clouds (gpdb_set_clouds_samples) and the batch hand search (gpdb_hand_search_batch).

Cloud-local index N_b + j addresses position j of cloud b. The oracle of a batch is the library itself, cloud by cloud: each
cloud's slice of gpdb_detect_batch, gpdb_detect_batch_select and gpdb_hand_search_batch must be bit-equal to gpdb_set_cloud
+ gpdb_set_samples + the single-cloud call on that cloud (frames, flags, score bytes, pose records, images). One small
batch is also held against the CPU oracle's set_samples, and the float64-ulp position cases of hand_cases.py run as the
middle cloud of a batch.
"""
import ctypes as C

import numpy as np
import pytest

import hand_cases as hc
import hand_reference as hr
from conftest import load_weights
from gpd_b200 import abi, lib, scenes
from oracle import oracle
from test_gpu_batch import outside_workspace, table
from test_gpu_parity import assert_parity

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
# an off-default hand (every field moved; still inside the 15-channel shadow bitmap)
HAND = dict(finger_width=0.008, hand_outer_diameter=0.105, hand_depth=0.05, hand_height=0.025, init_bite=0.008)
FIELDS = ("frame", "position", "top", "bottom", "center", "width", "finger_idx", "half_antipodal", "full_antipodal",
          "sample", "sample_index", "sample_slot", "pose_slot")


def assert_same(rb, rs):
    """A batch slice against the single-cloud result, bit for bit (hand-search results carry no images)."""
    assert rb["n_candidates"] == rs["n_candidates"]
    assert np.array_equal(rb["frame_valid"], rs["frame_valid"])
    assert rb["frames"].tobytes() == rs["frames"].tobytes()
    assert np.array_equal(rb["pose_flags"], rs["pose_flags"])
    assert rb["pose_scores"].tobytes() == rs["pose_scores"].tobytes()
    assert rb["candidates"].tobytes() == rs["candidates"].tobytes()
    if rs["images"] is None or not rs["n_candidates"]:
        assert rb["images"] is None or not rb["n_candidates"]
    else:
        assert rb["images"].tobytes() == rs["images"].tobytes()


def context(ch, weights=True, **over):
    w, relu = load_weights(ch)
    p = lib.default_params(channels=ch, relu_after_conv=relu, keep_images=1, **over)
    ctx = lib.Context(p)
    if weights:
        ctx.set_weights(w)
    return p, ctx, oracle.WeightPack(w)


def positions_near(cloud, seed, m):
    """m float64 positions a few millimetres off cloud points: most of them carry hands."""
    rng = np.random.default_rng(seed)
    pts = cloud["xyz"][rng.choice(len(cloud["xyz"]), m, replace=False)].astype(np.float64)
    return pts + rng.normal(0.0, 0.002, pts.shape)


def mixed(n_points, m, seed, n_pts):
    """n_pts point indices and all m position indices (N + j), shuffled together."""
    rng = np.random.default_rng(seed)
    s = np.concatenate([rng.choice(n_points, n_pts, replace=False), n_points + np.arange(m)]).astype(np.int32)
    return rng.permutation(s).astype(np.int32)


def single(ctx, cloud, pos, sidx, call):
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud.get("cam_source"), cloud.get("view_points"))
    if len(pos):
        assert ctx.set_samples(pos)[0] == len(cloud["xyz"])
    return call(sidx)


def scenario():
    """krylon (one camera), a two-camera table, a table without positions, a cloud outside the workspace with positions, a
    table with positions and an empty sample range."""
    k = scenes.krylon_cloud()
    clouds = [k, table(4, two_cameras=True), table(5), outside_workspace(), table(6)]
    pos = [positions_near(k, 1, 40), positions_near(clouds[1], 2, 50), np.zeros((0, 3)), positions_near(clouds[3], 4, 12),
           positions_near(clouds[4], 5, 7)]
    n = [len(c["xyz"]) for c in clouds]
    samples = [mixed(n[0], 40, 11, 30), mixed(n[1], 50, 12, 40), mixed(n[2], 0, 13, 50), mixed(n[3], 12, 14, 10),
               np.zeros(0, np.int32)]
    return clouds, pos, samples


def check_scenario(ctx, clouds, pos, samples, with_images=True):
    ctx.set_clouds(clouds)
    idx = ctx.set_clouds_samples(pos)
    for b, c in enumerate(clouds):
        assert np.array_equal(idx[b], len(c["xyz"]) + np.arange(len(pos[b])))
    calls = [("hand_search", ctx.hand_search_batch, ctx.hand_search)]
    if with_images:
        calls.append(("detect", ctx.detect_batch, ctx.detect))
    views = {name: batch_call(samples) for name, batch_call, _ in calls}
    sel = ctx.detect_batch_select(samples, 25) if with_images else None
    for name, _, single_call in calls:  # the single cloud's calls leave the batch and its positions alone
        for b, c in enumerate(clouds):
            assert_same(views[name][b], single(ctx, c, pos[b], samples[b], single_call))
    if with_images:
        for b, c in enumerate(clouds):
            rs = single(ctx, c, pos[b], samples[b], lambda s: ctx.detect_select(s, 25))
            assert sel[b].tobytes() == rs["candidates"].tobytes()
    return views


@pytest.mark.parametrize("ch,over", [(15, {}), (3, {}), (15, HAND)], ids=["15ch", "3ch", "15ch-hand"])
def test_positions_in_a_batch_equal_single_clouds(ch, over):
    p, ctx, w = context(ch, **over)
    clouds, pos, samples = scenario()
    views = check_scenario(ctx, clouds, pos, samples)
    v = views["detect"]
    # positions carry hands: some candidate of krylon and of the two-camera table sits at a position index
    for b in (0, 1):
        assert np.any(v[b]["candidates"]["sample_index"] >= len(clouds[b]["xyz"]))
    assert v[3]["n_candidates"] == 0 and v[4]["n_samples"] == 0
    assert np.all(np.isnan(views["hand_search"][0]["pose_scores"]))
    ctx.close()


def test_hand_search_batch_needs_no_weights():
    p, ctx, _ = context(15, weights=False)
    clouds, pos, samples = scenario()
    check_scenario(ctx, clouds, pos, samples, with_images=False)
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect_batch(samples)
    assert e.value.code == ERR_STATE
    ctx.close()


def test_positions_in_a_preprocessed_batch_with_an_emptied_cloud():
    """gpdb_preprocess_clouds, one raw cloud emptied by the workspace filter (it keeps positions, takes an empty range)."""
    p, ctx, _ = context(15)
    pp = lib.preprocess_params()
    r7 = scenes.synthetic_raw_scene(7, n_points=20000)
    r8 = scenes.synthetic_raw_scene(8, n_points=20000, two_cameras=True)
    far = dict(xyz=(r7["xyz"][:5000] + np.float32([5.0, 0.0, 0.0])).astype(np.float32), cam_source=None,
               view_points=np.zeros((1, 3)))
    raws = [dict(xyz=r7["xyz"], cam_source=r7["cam_source"], view_points=r7["view_points"]), far,
            dict(xyz=r8["xyz"], cam_source=r8["cam_source"], view_points=r8["view_points"])]
    got = ctx.preprocess_clouds(raws, pp)
    assert len(got[1]["xyz"]) == 0 and len(got[0]["xyz"]) > 1000 and len(got[2]["xyz"]) > 1000
    pos = [positions_near(got[0], 21, 30), np.array([[5.0, 0.0, 0.9], [5.1, 0.0, 0.9]]), positions_near(got[2], 22, 30)]
    samples = [mixed(len(got[0]["xyz"]), 30, 31, 40), np.zeros(0, np.int32), mixed(len(got[2]["xyz"]), 30, 32, 40)]
    idx = ctx.set_clouds_samples(pos)
    assert list(idx[1]) == [0, 1]
    views = ctx.detect_batch(samples)
    hs = ctx.hand_search_batch(samples)
    assert views[1]["n_samples"] == 0 and hs[1]["n_samples"] == 0
    for b in (0, 2):
        assert_same(views[b], single(ctx, got[b], pos[b], samples[b], ctx.detect))
        assert_same(hs[b], single(ctx, got[b], pos[b], samples[b], ctx.hand_search))
        assert views[b]["n_candidates"] > 0
    ctx.close()


def test_hand_case_positions_as_the_middle_cloud_of_a_batch():
    """The float64-ulp position cases of hand_cases.py (every sample kind of each geometry case), as cloud 1 of three, equal
    the case's cloud alone: frames, flags and every field of every record."""
    w, _ = load_weights(15)
    other = hc.single_object().case("other")
    n_pos = 0
    for case in hc.geometry_cases():
        if not any(kind == "position" for kind, _ in case["samples"]):
            continue
        p = abi.default_params(15, **case["over"])
        ctx = lib.Context(p)
        ctx.set_weights(w)
        c = case["cloud"]
        ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        sidx = hr.case_samples(case, ctx)
        one_hs, one_d = ctx.hand_search(sidx), ctx.detect(sidx)
        pos = np.array([s for kind, s in case["samples"] if kind == "position"], np.float64)
        oc = other["cloud"]
        ctx.set_clouds([oc, c, oc])
        ctx.set_clouds_samples([np.zeros((0, 3)), pos, oc["xyz"][:2].astype(np.float64)])
        no = len(oc["xyz"])
        lists = [[4], sidx, [no, 4, no + 1]]
        mid_d = ctx.detect_batch(lists)[1]
        for mid, one in ((ctx.hand_search_batch(lists)[1], one_hs), (mid_d, one_d)):
            assert np.array_equal(mid["pose_flags"], one["pose_flags"]), case["name"]
            assert mid["frames"].tobytes() == one["frames"].tobytes(), case["name"]
            assert mid["n_candidates"] == one["n_candidates"]
            for f in FIELDS:
                assert np.array_equal(mid["candidates"][f], one["candidates"][f]), (case["name"], f)
        assert mid_d["pose_scores"].tobytes() == one_d["pose_scores"].tobytes()
        n_pos += len(pos)
        ctx.close()
    assert n_pos > 0


def test_small_batch_against_the_oracle():
    """krylon with positions as cloud 0 of two, against the CPU oracle's set_samples at the parity bars."""
    p, ctx, w = context(15)
    k = scenes.krylon_cloud()
    t = table(3)
    pos = positions_near(k, 41, 40)
    sidx = mixed(len(k["xyz"]), 40, 42, 40)
    ctx.set_clouds([k, t])
    ctx.set_clouds_samples([pos, positions_near(t, 43, 5)])
    views = ctx.detect_batch([sidx, len(t["xyz"]) + np.arange(5, dtype=np.int32)])
    oc = oracle.OracleCloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    assert oc.set_samples(pos)[0] == len(k["xyz"])
    assert_parity(oc.detect(p, w, sidx), views[0], 15)
    assert views[0]["n_candidates"] > 0
    ctx.close()


def raw_set(ctx, poff, samples):
    poff = None if poff is None else np.ascontiguousarray(poff, np.int32)
    sm = None if samples is None else np.ascontiguousarray(samples, np.float64)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    return lib.lib().gpdb_set_clouds_samples(ctx.h, p(poff), p(sm))


def test_position_errors_and_lifetime():
    p, ctx, _ = context(15)
    k, t = scenes.krylon_cloud(), table(3, n=8000)
    nk, nt = len(k["xyz"]), len(t["xyz"])
    pk, pt = positions_near(k, 51, 6), positions_near(t, 52, 4)
    assert raw_set(ctx, [0, 6, 10], np.vstack([pk, pt])) == ERR_STATE  # no batch installed
    ctx.set_clouds([k, t])
    assert raw_set(ctx, [0, 6, 10], np.vstack([pk, pt])) == 10
    ctx.detect_batch([[nk + 5], [nt + 3]])  # the last position of each cloud
    for bad in ([[nk + 6], []], [[], [nt + 4]], [[-1], []]):  # N_b + M_b is outside cloud b
        with pytest.raises(lib.GpdbError) as e:
            ctx.detect_batch(bad)
        assert e.value.code == ERR_INVALID
        with pytest.raises(lib.GpdbError) as e:
            ctx.hand_search_batch(bad)
        assert e.value.code == ERR_INVALID
    # malformed offsets: not starting at 0, decreasing, positions missing; a failed call leaves no positions
    for poff, sm in (([1, 6, 10], np.vstack([pk, pt])), ([0, 6, 5], np.vstack([pk, pt])), ([0, 6, 10], None)):
        assert raw_set(ctx, [0, 6, 10], np.vstack([pk, pt])) == 10
        assert raw_set(ctx, poff, sm) == ERR_INVALID
        with pytest.raises(lib.GpdbError):
            ctx.detect_batch([[nk], []])
    assert raw_set(ctx, None, None) == ERR_INVALID
    # each call replaces every position; an empty set is allowed
    ctx.set_clouds_samples([pk, pt])
    ctx.set_clouds_samples([np.zeros((0, 3)), pt[:1]])
    ctx.detect_batch([[], [nt]])
    with pytest.raises(lib.GpdbError):
        ctx.detect_batch([[nk], []])
    # a reinstall drops them: gpdb_set_clouds (successful or failed) and gpdb_preprocess_clouds
    ctx.set_clouds_samples([pk, pt])
    ctx.set_clouds([k, t])
    with pytest.raises(lib.GpdbError):
        ctx.detect_batch([[nk], []])
    ctx.set_clouds_samples([pk, pt])
    bad = dict(t, xyz=t["xyz"].copy())
    bad["xyz"][0, 0] = np.nan
    with pytest.raises(lib.GpdbError):
        ctx.set_clouds([k, bad])
    ctx.set_clouds([k, t])
    with pytest.raises(lib.GpdbError):
        ctx.detect_batch([[nk], []])
    ctx.set_clouds_samples([pk, pt])
    poff = ctx.preprocess_clouds([dict(xyz=k["xyz"], cam_source=None, view_points=k["view_points"])] * 2,
                                 lib.preprocess_params(), read_back=False)
    ctx.detect_batch([[int(poff[1]) - 1], []])
    with pytest.raises(lib.GpdbError):
        ctx.detect_batch([[int(poff[1])], []])
    # gpdb_set_samples with only a batch installed keeps its error
    with pytest.raises(lib.GpdbError) as e:
        ctx.set_samples(pk)
    assert e.value.code == ERR_INVALID
    ctx.close()


def test_single_and_batch_positions_are_independent():
    p, ctx, _ = context(15)
    k, t = scenes.krylon_cloud(), table(3, n=8000)
    nk = len(k["xyz"])
    ps, pb = positions_near(k, 61, 8), positions_near(k, 62, 8)
    ctx.set_cloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    first = ctx.set_samples(ps)
    before = ctx.detect(first)
    ctx.set_clouds([k, t])
    ctx.set_clouds_samples([pb, np.zeros((0, 3))])
    batch_before = ctx.detect_batch([nk + np.arange(8, dtype=np.int32), []])
    assert_same(ctx.detect(first), before)  # the single cloud's positions are untouched by the batch's
    ctx.set_samples(ps[::-1])  # ... and the batch's by the single cloud's
    assert_same(ctx.detect_batch([nk + np.arange(8, dtype=np.int32), []])[0], batch_before[0])
    assert before["n_candidates"] > 0 and batch_before[0]["n_candidates"] > 0
    assert before["candidates"]["sample"].tobytes() != batch_before[0]["candidates"]["sample"].tobytes()
    ctx.close()
