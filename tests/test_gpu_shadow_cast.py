"""GPU tests of the shadow casting of the 15-channel images at exact counts (-m gpu). Every case of
tests/shadow_cases.py (whose counts test_shadow_cast_reference.py proves on the CPU) runs once under the default kernel
choice and once with GPD_B200_IMAGES_KERNEL=1 (k_images alone), and with gpdb_debug_phase_cycles:

* slots 9, 10 and 11 (work-list entries, draws in their window, voxel-list size) equal the restatement's sums;
* every shadow path counter equals the restatement's excess past its capacity;
* the images equal image_reference.image(..., "kernel") bit for bit, all 15 channels, and the two kernels agree.

Further: the image at the stash's last entry made together with neighbours on both sides (its HBM stash ends exactly at
the end of its 57.6 KB slot), and the bench scene's counts over a few hundred candidates at one and two cameras."""
import numpy as np
import pytest

import capacity_cases as cc
import image_reference as ir
import shadow_cases as sc
import shadow_cast_reference as scr
from gpd_b200 import lib, scenes
from shadow_counters import IMAGES2_EVENTS, IMAGES_EVENTS, assert_counters, counted_images, expected

pytestmark = pytest.mark.gpu

def make_context(cloud, **over):
    ctx = lib.Context(lib.default_params(**over))
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    return ctx


@pytest.fixture(scope="session")
def reference_images():
    cache = {}

    def get(i):
        if i not in cache:
            case = sc.build(i)
            cache[i] = ir.image(case["cloud"], case["pose"][0], case["geometry"], "kernel")
        return cache[i]
    return get


@pytest.mark.parametrize("i", range(len(sc.EDGES)), ids=sc.IDS)
def test_shadow_lists_at_their_edges(i, reference_images, monkeypatch):
    case = sc.build(i)
    r, g = case["counts"], case["geometry"]
    box_n = cc.box_count(case["cloud"], case["pose"], g.w, g.d, g.h, g.radius)
    ctx = make_context(case["cloud"], **sc.params_of(case))
    images = {}
    for forced in (False, True):
        img, paths, slots = counted_images(ctx, case["pose"], forced, monkeypatch)
        exp = expected(r, g, box_n, forced)
        assert exp["s10"][0] == exp["s10"][1], "every case's draw count is exact"
        assert_counters(exp, paths, slots)
        images[forced] = img[0]
    ctx.close()
    if case["name"] != "voxel_list":
        assert expected(r, g, box_n, False)["fast"]  # the default choice ran k_images2
    assert np.array_equal(images[False], images[True])
    ref = reference_images(i)
    assert np.array_equal(images[False], ref), int(np.count_nonzero(images[False] != ref))
    if case["name"] == "no_camera0":
        assert not images[False][..., 4::5].any()
    else:
        assert images[False][..., 4::5].any()


def _neighbour(xyz_shift, seed):
    cloud, pose = cc.image_box(150, n_outside=30, seed=seed)
    obj = len(cloud["xyz"]) - 400  # image_box: the object, then the 20 x 20 plane
    pose["sample"][0] += xyz_shift
    pose["sample_index"] = seed
    return (cloud["xyz"][:obj].astype(np.float64) + xyz_shift).astype(np.float32), cloud["normals"][:obj], pose


def test_stash_edge_image_beside_its_neighbours(monkeypatch):
    """The image at ST_CAP (its stash ends at the end of its HBM slot) made in one call between two small images of
    their own objects, 0.5 m away: each image equals the one made alone."""
    i = sc.IDS.index("stash_cap_1cam-st_cap")
    case = sc.build(i)
    c = case["cloud"]
    (xa, na, pa), (xb, nb, pb) = _neighbour(np.array([0.5, 0.0, 0.0]), 3), _neighbour(np.array([-0.5, 0.0, 0.0]), 4)
    cloud = {"xyz": np.vstack([c["xyz"], xa, xb]), "normals": np.vstack([c["normals"], na, nb]),
             "view_points": c["view_points"]}
    cloud["cam_source"] = np.ones((len(cloud["xyz"]), 1), np.int32)
    ctx = make_context(cloud, **sc.params_of(case))
    poses = np.concatenate([pa, case["pose"], pb])
    r = scr.cast(cloud, case["pose"][0], case["geometry"])
    assert r["nset_all"] == case["target"] == cc.st_cap2(48, 1)
    for forced in (False, True):
        img, paths, slots = counted_images(ctx, poses, forced, monkeypatch)
        if not forced:  # k_images2 made all three, and the edge image's stash was exactly full
            assert paths["images2_box"] == 0 and paths["images2_stash_full"] == 0, paths
            assert int(slots[11]) >= case["target"], int(slots[11])
        for k in range(3):
            alone, _, _ = counted_images(ctx, poses[k:k + 1], forced, monkeypatch)
            assert np.array_equal(img[k], alone[0]), (forced, k)
        assert np.array_equal(img[1], ir.image(cloud, case["pose"][0], case["geometry"], "kernel"))
    ctx.close()


@pytest.mark.parametrize("two_cameras", [False, True], ids=["1cam", "2cam"])
def test_bench_scene_counts(two_cameras, monkeypatch):
    """The bench cloud and 250 of its candidates: slots 9 / 10 / 11 over one gpdb_images call equal the restatement
    summed over the same candidates, and so does every shadow path counter."""
    s = scenes.synthetic_table_scene(3, two_cameras=two_cameras)
    cloud = {"xyz": s["xyz"], "normals": s["normals"], "cam_source": s["cam_source"], "view_points": s["view_points"]}
    ctx = make_context(cloud, channels=15)
    sidx = np.random.default_rng(5).choice(len(s["xyz"]), 1000, replace=False).astype(np.int32)
    cand = ctx.hand_search(sidx)["candidates"]
    g = ir.Geometry(C=15)
    xyz = np.asarray(cloud["xyz"], np.float32)
    cams = np.asarray(cloud["cam_source"]).reshape(len(xyz), -1)
    keep, subs = [], []
    for j in range(len(cand)):
        if len(keep) == 250:
            break
        # the restatement runs on the points near the sample, under their cloud indices (the LCG seeds)
        near = np.flatnonzero(np.abs(xyz - cand["sample"][j].astype(np.float32)).max(1) < 0.11)
        sub = {"xyz": xyz[near], "cam_source": cams[near], "view_points": cloud["view_points"]}
        idx, _ = ir.neighbourhood(sub, cand["sample"][j], g.radius)
        if scr.centre_is_exact(sub["xyz"][idx]):  # the restatement's condition; nearly every candidate meets it
            keep.append(j)
            subs.append((sub, near))
    assert len(keep) >= 200
    poses = cand[keep]
    rs = [scr.cast(sub, poses[j], g, index=near) for j, (sub, near) in enumerate(subs)]
    boxes = [cc.box_count(sub, poses[j:j + 1], g.w, g.d, g.h, g.radius) for j, (sub, _) in enumerate(subs)]
    for forced in (False, True):
        img, paths, slots = counted_images(ctx, poses, forced, monkeypatch)
        exp = [expected(r, g, box_n, forced) for r, box_n in zip(rs, boxes)]
        assert int(slots[9]) == sum(e["s9"] for e in exp)
        assert sum(e["s10"][0] for e in exp) <= int(slots[10]) <= sum(e["s10"][1] for e in exp)
        assert int(slots[11]) == sum(e["s11"] for e in exp)
        assert int(slots[14]) == sum(e["walks"] for e in exp)
        for k in IMAGES2_EVENTS + IMAGES_EVENTS:
            if not k.endswith("draw_in_place") or all(e["s10"][0] == e["s10"][1] for e in exp):
                assert paths[k] == sum(e["events"][k] for e in exp), k
    ctx.close()


# ---- batches: the edge clouds through gpdb_images_batch_device (the BATCH instantiations of both kernels)

def _small(seed, view_points):
    cloud, pose = cc.image_box(150, n_outside=30, seed=seed)
    cloud["view_points"] = np.asarray(view_points, np.float64)
    cloud["cam_source"] = np.ones((len(cloud["xyz"]), len(cloud["view_points"])), np.int32)
    pose["sample_index"] = seed
    return cloud, pose


def batch_vs_singles(clouds, poses, geometry, monkeypatch):
    """One images_batch_tensors call over the clouds (one pose each) against one single-cloud gpdb_images call per
    cloud, under both kernel choices: the images equal, and the batch's counters equal the restatement summed over
    the clouds, with the launch sized for the batch's largest camera count."""
    import torch
    g = ir.Geometry(**geometry)
    over = dict(channels=15, volume_width=g.w, volume_depth=g.d, volume_height=g.h)
    maxk = max(len(c["view_points"]) for c in clouds)
    rs = [scr.cast(c, p[0], g) for c, p in zip(clouds, poses)]
    boxes = [cc.box_count(c, p, g.w, g.d, g.h, g.radius) for c, p in zip(clouds, poses)]
    ctx = lib.Context(lib.default_params(**over))
    ctx.set_clouds(clouds)
    recs = torch.from_numpy(np.concatenate(poses).view(np.uint8).reshape(len(poses), -1).copy()).cuda()
    hoff = np.arange(len(poses) + 1, dtype=np.int32)
    for forced in (False, True):
        if forced:
            monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
        try:
            ctx.phase_cycles(1)
            img = ctx.images_batch_tensors(hoff, recs).cpu().numpy()
            paths = ctx.path_counts()
            slots = ctx.phase_cycles(0)
        finally:
            monkeypatch.delenv("GPD_B200_IMAGES_KERNEL", raising=False)
        exp = [expected(r, g, box_n, forced, maxk) for r, box_n in zip(rs, boxes)]
        tot = {"s9": sum(e["s9"] for e in exp), "s10": (sum(e["s10"][0] for e in exp), sum(e["s10"][1] for e in exp)),
               "s11": sum(e["s11"] for e in exp), "walks": sum(e["walks"] for e in exp),
               "events": {k: sum(e["events"][k] for e in exp) for k in IMAGES2_EVENTS + IMAGES_EVENTS}}
        assert tot["s10"][0] == tot["s10"][1]
        assert_counters(tot, paths, slots)
        for b, (c, p) in enumerate(zip(clouds, poses)):
            ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
            alone, _, _ = counted_images(ctx, p, forced, monkeypatch)
            assert np.array_equal(img[b], alone[0]), (forced, b)
    ctx.close()
    return rs


BATCH_EDGES = ["stash_sm_1cam-st_sm", "stash_sm_1cam-st_sm+1", "stash_cap_1cam-st_cap", "stash_cap_1cam-st_cap+1",
               "work_list_1cam-wl_cap2+1", "draw_list-dl_cap+1", "ball-ball_cap+1"]


@pytest.mark.parametrize("edge", BATCH_EDGES)
def test_batch_middle_cloud_at_the_edge(edge, monkeypatch):
    case = sc.build(sc.IDS.index(edge))
    (a, pa), (b, pb) = _small(11, [[0.0, 0.0, 0.0]]), _small(12, [[0.1, 0.0, 0.0]])
    batch_vs_singles([a, case["cloud"], b], [pa, case["pose"], pb], sc.GEOMETRIES["default"], monkeypatch)


@pytest.mark.parametrize("one,two", [("st_sm", "st_sm+1"), ("st_sm+1", "st_sm")])
def test_batch_mixes_one_and_two_cameras_at_their_stash_edges(one, two, monkeypatch):
    """volume_depth 0.05: the launch is sized for two cameras, but each image lays out its stash behind its own bitmaps:
    ST_SM is 2 492 for the one-camera cloud and 376 for the two-camera cloud, each at or one past its own edge."""
    c1 = sc.build(sc.IDS.index(f"stash_sm_1cam_d05-{one}"))
    c2 = sc.build(sc.IDS.index(f"stash_sm_2cam-{two}"))
    assert c1["target"] - cc.st_sm2(46, 1) in (0, 1) and c2["target"] - cc.st_sm2(46, 2) in (0, 1)
    s, ps = _small(13, [[0.0, 0.0, 0.0]])
    rs = batch_vs_singles([s, c1["cloud"], c2["cloud"]], [ps, c1["pose"], c2["pose"]], sc.GEOMETRIES["depth05"],
                          monkeypatch)
    assert [r["K"] for r in rs] == [1, 1, 2] and rs[1]["nset_all"] == c1["target"] and rs[2]["nset_all"] == c2["target"]
