"""Batches of clouds (gpdb_set_clouds / gpdb_detect_batch / gpdb_detect_batch_select) on the GPU.

The oracle of a batch is the library itself, cloud by cloud: every cloud's slice of a batch result must be bit-equal to
gpdb_detect on that cloud alone (flags, frames, pose records with cloud-local sample index and slot, images, scores). The
heterogeneous, isolation and overflow-tier tests also hold one cloud of the batch against the CPU oracle at the parity bars
of test_gpu_parity (krylon; krylon moved into the table scene; the dense lattice).
"""
import ctypes as C

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import abi, lib, scenes
from oracle import oracle
from test_gpu_parity import _lattice_cloud, _random_cube, assert_parity

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE, ERR_CAPACITY = -1, -3, -5


def context(ch, **over):
    w, relu = load_weights(ch)
    p = lib.default_params(channels=ch, relu_after_conv=relu, keep_images=1, **over)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    return p, ctx, oracle.WeightPack(w)


def singles(ctx, clouds, samples):
    out = []
    for c, s in zip(clouds, samples):
        ctx.set_cloud(c["xyz"], c["normals"], c.get("cam_source"), c.get("view_points"))
        out.append(ctx.detect(np.asarray(s, np.int32)))
    return out


def assert_same(rb, rs):
    """A batch slice against the single-cloud result, bit for bit."""
    assert rb["n_candidates"] == rs["n_candidates"]
    assert np.array_equal(rb["frame_valid"], rs["frame_valid"])
    assert rb["frames"].tobytes() == rs["frames"].tobytes()
    assert np.array_equal(rb["pose_flags"], rs["pose_flags"])
    assert rb["pose_scores"].tobytes() == rs["pose_scores"].tobytes()
    assert rb["candidates"].tobytes() == rs["candidates"].tobytes()
    if rs["n_candidates"]:
        assert rb["images"].tobytes() == rs["images"].tobytes()


def check_oracle(p, w, cloud, sidx, view, ch=15):
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    assert_parity(oc.detect(p, w, np.asarray(sidx, np.int32)), view, ch)


def check_batch(ctx, clouds, samples):
    ctx.set_clouds(clouds)
    views = ctx.detect_batch(samples)
    assert len(views) == len(clouds)
    for rb, rs in zip(views, singles(ctx, clouds, samples)):
        assert_same(rb, rs)
    return views


def table(seed, n=20000, **kw):
    return scenes.synthetic_table_scene(seed, n_points=n, **kw)


def nonunit(cloud):
    """Voxel-average-like normals: a third of them shortened, so images take the exact-fold path."""
    c = dict(cloud)
    n = c["normals"].copy()
    n[::3] *= 0.6
    c["normals"] = n
    return c


def outside_workspace():
    """A table patch 5 m away: every hand lies outside workspace_grasps (-1..1), so the cloud yields no candidates."""
    t = table(9, n=8000)
    return dict(t, xyz=(t["xyz"] + np.float32([5.0, 0.0, 0.0])).astype(np.float32), view_points=t["view_points"] + [5.0, 0.0, 0.0])


def heterogeneous():
    k = scenes.krylon_cloud()
    clouds = [k, table(3), table(4, two_cameras=True), nonunit(table(6)), outside_workspace(), table(8)]
    samples = [scenes.sample_indices(2, len(k["xyz"]), 120), scenes.sample_indices(1, 20000, 150),
               scenes.sample_indices(1, 20000, 150), scenes.sample_indices(1, 20000, 120),
               scenes.sample_indices(1, 8000, 60), []]
    return clouds, samples


@pytest.mark.parametrize("ch", [15, 12, 3])
def test_heterogeneous_batch_equals_single_clouds(ch):
    p, ctx, w = context(ch)
    clouds, samples = heterogeneous()
    views = check_batch(ctx, clouds, samples)
    assert views[0]["n_candidates"] > 0 and views[4]["n_candidates"] == 0 and views[5]["n_samples"] == 0
    assert any(v["n_candidates"] > 0 for v in views[1:4])
    check_oracle(p, w, clouds[0], samples[0], views[0], ch)
    ctx.close()


def test_overlapping_clouds_stay_isolated():
    """krylon moved into the table scene's workspace, and one cloud twice: a search that crossed a cloud boundary would
    see the other cloud's points."""
    p, ctx, w = context(15)
    t = table(3)
    k = dict(scenes.krylon_cloud())
    kx = k["xyz"].astype(np.float64)
    target = t["xyz"][np.argmin(np.abs(t["xyz"][:, 0]) + np.abs(t["xyz"][:, 1]))].astype(np.float64)
    k["xyz"] = (kx - kx.mean(0) + target).astype(np.float32)
    lo, hi = t["xyz"].min(0), t["xyz"].max(0)
    assert np.all(k["xyz"].min(0) >= lo - 0.2) and np.all(k["xyz"].max(0) <= hi + 0.2)
    sk, st = scenes.sample_indices(2, len(k["xyz"]), 120), scenes.sample_indices(1, 20000, 150)
    views = check_batch(ctx, [t, k], [st, sk])
    check_oracle(p, w, k, sk, views[1])
    check_batch(ctx, [t, t], [st, st[::-1]])
    ctx.close()


def test_order_single_and_many_small_clouds():
    p, ctx, _ = context(15, chunk_samples=64)  # chunk boundaries fall inside clouds
    clouds = [table(3), scenes.krylon_cloud(), table(4, two_cameras=True)]
    samples = [scenes.sample_indices(1, 20000, 100), scenes.sample_indices(2, len(clouds[1]["xyz"]), 90),
               scenes.sample_indices(1, 20000, 80)]
    a = check_batch(ctx, clouds, samples)
    perm = [2, 0, 1]
    ctx.set_clouds([clouds[i] for i in perm])
    b = ctx.detect_batch([samples[i] for i in perm])
    for j, i in enumerate(perm):
        assert_same(b[j], a[i])
    one = check_batch(ctx, clouds[:1], samples[:1])  # B = 1
    assert_same(one[0], a[0])
    # ~200 small clouds: random crops of a few base scenes
    rng = np.random.default_rng(11)
    base = [table(s, n=8000) for s in (3, 4, 5, 6)]
    small, ss = [], []
    for i in range(200):
        c = base[i % 4]
        keep = np.sort(rng.choice(len(c["xyz"]), int(rng.integers(1500, 4000)), replace=False))
        small.append({"xyz": c["xyz"][keep], "normals": c["normals"][keep], "cam_source": c["cam_source"][keep],
                      "view_points": c["view_points"]})
        ss.append(rng.choice(len(keep), int(rng.integers(0, 40)), replace=False).astype(np.int32))
    views = check_batch(ctx, small, ss)
    assert sum(v["n_candidates"] for v in views) > 0
    ctx.close()


def test_overflow_tiers_inside_a_batch():
    """One dense unvoxelised lattice (hand slabs and image boxes beyond the shared-memory tiers, frames beyond the first)
    among voxelised clouds."""
    p, ctx, w = context(15)
    dense, rng = _lattice_cloud(0.0012)
    center = np.argsort(np.linalg.norm(dense["xyz"][:, :2], axis=1))[:2000]
    sd = center[rng.choice(2000, 40, replace=False)].astype(np.int32)
    k = scenes.krylon_cloud()
    views = check_batch(ctx, [table(3), dense, k], [scenes.sample_indices(1, 20000, 100), sd,
                                                    scenes.sample_indices(2, len(k["xyz"]), 80)])
    assert views[1]["n_candidates"] > 0
    check_oracle(p, w, dense, sd, views[1])
    ctx.close()


def test_batch_select_equals_per_cloud_select():
    p, ctx, _ = context(15)
    clouds, samples = heterogeneous()
    ctx.set_clouds(clouds)
    got = ctx.detect_batch_select(samples, 12)
    for g, c, s in zip(got, clouds, samples):
        ctx.set_cloud(c["xyz"], c["normals"], c.get("cam_source"), c.get("view_points"))
        want = ctx.detect_select(np.asarray(s, np.int32), 12)["candidates"]
        assert g.tobytes() == want.tobytes()
    assert len(got[0]) == 12 and len(got[4]) == 0
    ctx.close()


def raw_detect_batch(ctx, offsets, sidx):
    res = abi.Result()
    coff = np.zeros(len(offsets), np.int32)
    offsets, sidx = np.asarray(offsets, np.int32), np.asarray(sidx, np.int32)
    rc = lib.lib().gpdb_detect_batch(ctx.h, offsets.ctypes.data_as(C.c_void_p), sidx.ctypes.data_as(C.c_void_p), C.byref(res),
                                     coff.ctypes.data_as(C.c_void_p))
    lib.free_result(res)
    return rc


def test_errors_leave_the_context_usable():
    p, ctx, _ = context(15)
    k, t = scenes.krylon_cloud(), table(3)
    sk = scenes.sample_indices(2, len(k["xyz"]), 60)

    def still_works():
        ctx.set_clouds([t, k])
        for rb, rs in zip(ctx.detect_batch([sk, sk]), singles(ctx, [t, k], [sk, sk])):
            assert_same(rb, rs)

    ctx.set_clouds([t, k])
    for lists in ([sk], [sk, sk, sk]):  # one list per installed cloud: refused before the call
        with pytest.raises(ValueError):
            ctx.detect_batch(lists)
        with pytest.raises(ValueError):
            ctx.detect_batch_select(lists, 4)
    assert raw_detect_batch(ctx, [0, 70, 60], np.concatenate([sk, sk])) == ERR_INVALID  # decreasing offsets
    assert raw_detect_batch(ctx, [1, 60, 120], np.concatenate([sk, sk])) == ERR_INVALID  # not starting at 0
    bad = sk.copy()
    bad[5] = len(k["xyz"])  # local index == N_b (valid in the table scene, not in krylon)
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect_batch([sk, bad])
    assert e.value.code == ERR_INVALID
    still_works()
    nine = dict(k, cam_source=None, view_points=np.zeros((9, 3)))
    with pytest.raises(lib.GpdbError) as e:
        ctx.set_clouds([t, nine])
    assert e.value.code == ERR_INVALID
    with pytest.raises(ValueError, match="batch of 0 clouds"):  # the failed call left no batch
        ctx.detect_batch([sk, sk])
    assert raw_detect_batch(ctx, [0, 60, 120], np.concatenate([sk, sk])) == ERR_STATE  # ... in the library too
    still_works()
    # sample positions belong to the single cloud: with only a batch installed they are rejected
    p2, ctx2, _ = context(3)
    ctx2.set_clouds([t])
    with pytest.raises(lib.GpdbError) as e:
        ctx2.set_samples(np.zeros((2, 3)))
    assert e.value.code == ERR_INVALID
    ctx2.close()
    # a neighbourhood beyond the last tier anywhere in the batch fails the whole call
    xyz, nrm = _random_cube(400000, 0.03)
    cube = {"xyz": xyz, "normals": nrm, "cam_source": None, "view_points": np.zeros((1, 3))}
    mid = np.argsort(np.linalg.norm(xyz - 0.015, axis=1))[:8].astype(np.int32)
    ctx.set_clouds([t, cube])
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect_batch([sk, mid])
    assert e.value.code == ERR_CAPACITY
    still_works()
    ctx.set_cloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    assert ctx.detect(sk)["n_candidates"] > 0
    ctx.close()
