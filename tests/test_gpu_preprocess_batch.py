"""Preprocessing a batch of raw clouds in one call (gpdb_preprocess_clouds / gpdb_get_clouds) on the GPU.

The oracle of a batch is the library itself, cloud by cloud: every processed cloud must be bit-equal to gpdb_preprocess on
that raw cloud alone (points, camera sources, source indices and normals, estimated or voxel-averaged, compared with
tobytes()), and every cloud's slice of a following gpdb_detect_batch bit-equal to gpdb_preprocess + gpdb_detect on that
cloud. The krylon cloud is also held against the CPU oracle at the bars of test_gpu_preprocess.
"""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from oracle import oracle
from test_gpu_batch import assert_same
from test_gpu_preprocess import assert_cloud_parity

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE, ERR_CAPACITY = -1, -3, -5
VP0 = np.zeros((1, 3))


def context(ch=15):
    w, relu = load_weights(ch)
    ctx = lib.Context(lib.default_params(channels=ch, relu_after_conv=relu, keep_images=1))
    ctx.set_weights(w)
    return ctx


def raw(xyz, cam_source=None, view_points=VP0, normals=None):
    return {"xyz": np.ascontiguousarray(xyz, dtype=np.float32), "cam_source": cam_source, "view_points": view_points,
            "normals": normals}


def raw_scene(seed, n=30000, **kw):
    s = scenes.synthetic_raw_scene(seed, n_points=n, **kw)
    return raw(s["xyz"], s["cam_source"], s["view_points"])


def krylon_raw(golden_dir):
    return raw(np.load(os.path.join(golden_dir, "krylon_preprocess.npz"))["raw"])


def single(ctx, c, pp):
    return ctx.preprocess(c["xyz"], c["cam_source"], c["view_points"], pp, normals=c["normals"])


def assert_bit_equal(b, s):
    assert b["xyz"].shape == s["xyz"].shape and b["xyz"].tobytes() == s["xyz"].tobytes()
    assert b["cam_source"].shape == s["cam_source"].shape and np.array_equal(b["cam_source"], s["cam_source"])
    assert np.array_equal(b["src"], s["src"])
    assert b["normals"].tobytes() == s["normals"].tobytes()


def check(ctx, clouds, pp):
    """preprocess_clouds against preprocess of every cloud alone; the batch must survive the single-cloud calls."""
    got = ctx.preprocess_clouds(clouds, pp)
    assert len(got) == len(clouds)
    for g, c in zip(got, clouds):
        assert_bit_equal(g, single(ctx, c, pp))
    for g, a in zip(got, ctx.get_clouds()):  # gpdb_preprocess leaves the installed batch alone
        assert_bit_equal(a, g)
    return got


def samples_of(got, n=60):
    return [np.random.default_rng(b).choice(len(g["xyz"]), min(n, len(g["xyz"])), replace=False).astype(np.int32)
            for b, g in enumerate(got)]


def detect_equals_singles(ctx, clouds, got, pp, samples):
    views = ctx.detect_batch(samples)  # the batch preprocess_clouds installed
    for v, c, s, g in zip(views, clouds, samples, got):
        if len(g["xyz"]) == 0:  # gpdb_preprocess leaves no cloud to detect on: the batch slice is empty
            assert v["n_samples"] == v["n_candidates"] == 0
            continue
        single(ctx, c, pp)
        assert_same(v, ctx.detect(s))
    return views


def has_batch(ctx):
    return lib.lib().gpdb_get_clouds(ctx.h, None, None, None, None) >= 0


def test_heterogeneous_batch(golden_dir):
    """krylon, one- and two-camera raw scenes with 1 % NaNs, and a view lying outside the workspace (kept, empty)."""
    ctx = context()
    pp = lib.preprocess_params()
    far = raw_scene(5, n=8000)
    far["xyz"] = far["xyz"] + np.float32([5.0, 0.0, 0.0])
    clouds = [krylon_raw(golden_dir), raw_scene(7, nan_fraction=0.01), far,
              raw_scene(8, two_cameras=True, nan_fraction=0.01)]
    got = check(ctx, clouds, pp)
    assert len(got[2]["xyz"]) == 0 and all(len(got[b]["xyz"]) > 0 for b in (0, 1, 3))
    g = np.load(os.path.join(golden_dir, "krylon_preprocess.npz"))
    assert_cloud_parity(oracle.preprocess(g["raw"], None, VP0, pp), got[0])
    assert np.array_equal(got[0]["xyz"], g["xyz"])
    poff = ctx.preprocess_clouds(clouds, pp, read_back=False)
    assert np.array_equal(np.diff(poff), [len(c["xyz"]) for c in got])
    samples = samples_of(got)
    assert len(samples[2]) == 0
    views = detect_equals_singles(ctx, clouds, got, pp, samples)
    assert views[0]["n_candidates"] > 0 and views[2]["n_samples"] == 0
    ctx.preprocess_clouds(clouds, pp, read_back=False)
    bad = list(samples)
    bad[2] = np.zeros(1, np.int32)  # the empty cloud takes only an empty range
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect_batch(bad)
    assert e.value.code == ERR_INVALID
    ctx.close()


def test_supplied_normals_are_voxel_averaged_per_cloud():
    """estimate_normals = 0: bit-equal voxel averages, and two clouds whose single voxels share one key stay apart."""
    ctx = context()
    rng = np.random.default_rng(11)
    a, b = raw_scene(9, n=20000), raw_scene(10, n=15000, two_cameras=True)
    a["normals"], b["normals"] = rng.standard_normal((len(a["xyz"]), 3)), rng.standard_normal((len(b["xyz"]), 3))
    corner = np.float32([0.1, 0.2, 0.5])
    pair = [raw(corner + rng.uniform(0, 0.001, (4, 3)).astype(np.float32), normals=rng.standard_normal((4, 3)))
            for _ in range(2)]
    pair[1]["xyz"] = pair[0]["xyz"].copy()  # same coordinates, so both clouds have the same single voxel key
    for vox in (1, 0):
        pp = lib.preprocess_params(estimate_normals=0, voxelize=vox, voxel_size=0.004)
        got = check(ctx, [a, pair[0], pair[1], b], pp)
        if vox:
            assert len(got[1]["xyz"]) == len(got[2]["xyz"]) == 1
            for g, c in zip(got[1:3], pair):
                acc = np.zeros(3)
                for n in c["normals"]:
                    acc = acc + n
                assert g["normals"][0].tobytes() == (acc / 4).tobytes()
            assert not np.array_equal(got[1]["normals"], got[2]["normals"])
    ctx.close()


def test_clouds_stay_isolated(golden_dir):
    """The same raw cloud twice, and krylon moved into a raw table scene: normals and voxels from each cloud's own points."""
    ctx = context()
    pp = lib.preprocess_params()
    t = raw_scene(3)
    check(ctx, [t, t], pp)
    k = krylon_raw(golden_dir)
    fin = np.isfinite(t["xyz"]).all(1)
    tx = t["xyz"][fin]
    target = tx[np.argmin(np.abs(tx[:, 0]) + np.abs(tx[:, 1]))].astype(np.float64)
    kx = k["xyz"].astype(np.float64)
    k["xyz"] = (kx - np.nanmean(kx, axis=0) + target).astype(np.float32)
    got = check(ctx, [t, k], pp)
    lo, hi = got[0]["xyz"].min(0), got[0]["xyz"].max(0)
    assert np.all(got[1]["xyz"].min(0) >= lo - 0.2) and np.all(got[1]["xyz"].max(0) <= hi + 0.2)
    ctx.close()


def test_capacity_tiers_inside_a_batch(golden_dir):
    """The dense blob of test_gpu_preprocess (8 192-neighbour tier) inside a batch; 8 193 neighbours at one point fail
    the call with GPDB_ERR_CAPACITY, leave no batch, and the next call succeeds."""
    ctx = context()
    rng = np.random.default_rng(3)
    blob = raw((rng.uniform(-0.02, 0.02, (3000, 3)) + [0, 0, 0.5]).astype(np.float32))
    pp = lib.preprocess_params(voxelize=0)
    clouds = [raw_scene(4, n=20000), blob, krylon_raw(golden_dir)]
    got = check(ctx, clouds, pp)
    assert_cloud_parity(oracle.preprocess(blob["xyz"], None, VP0, pp), got[1])
    cluster = raw((rng.uniform(-0.004, 0.004, (9000, 3)) + [0.3, 0.0, 0.5]).astype(np.float32))
    with pytest.raises(lib.GpdbError) as e:
        ctx.preprocess_clouds([clouds[0], cluster], pp)
    assert e.value.code == ERR_CAPACITY
    assert not has_batch(ctx)
    with pytest.raises(ValueError, match="batch of 0 clouds"):
        ctx.detect_batch([[], []])
    check(ctx, clouds, pp)
    ctx.close()


def test_scale_and_order(golden_dir):
    ctx = context()
    pp = lib.preprocess_params()
    rng = np.random.default_rng(11)
    base = [scenes.synthetic_raw_scene(s, n_points=8000) for s in (3, 4, 5, 6)]
    small = []
    for i in range(200):
        s = base[i % 4]
        keep = np.sort(rng.choice(len(s["xyz"]), int(rng.integers(1500, 4000)), replace=False))
        small.append(raw(s["xyz"][keep], s["cam_source"][keep], s["view_points"]))
    got = check(ctx, small, pp)
    samples = samples_of(got, 20)
    detect_equals_singles(ctx, small[:200], got, pp, samples)
    big = scenes.synthetic_raw_scene(3)  # ~0.9 M raw points
    check(ctx, [small[0], raw(big["xyz"], big["cam_source"], big["view_points"]), small[1]], pp)
    clouds = [krylon_raw(golden_dir), raw_scene(7), raw_scene(8, two_cameras=True)]
    a = ctx.preprocess_clouds(clouds, pp)
    perm = [2, 0, 1]
    b = ctx.preprocess_clouds([clouds[i] for i in perm], pp)
    for j, i in enumerate(perm):
        assert_bit_equal(b[j], a[i])
    ctx.close()


def raw_call(ctx, offsets, xyz, n_cameras, pp, cam=None, normals=None):
    offsets, ncam = np.asarray(offsets, np.int32), np.asarray(n_cameras, np.int32)
    xyz = np.ascontiguousarray(xyz, np.float32)
    vp = np.zeros((int(ncam.sum()), 3))
    poff = np.zeros(len(offsets), np.int32)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    return lib.lib().gpdb_preprocess_clouds(ctx.h, len(offsets) - 1, p(offsets), p(xyz), p(normals), p(cam), p(ncam), p(vp),
                                            C.byref(pp), p(poff))


def test_errors_leave_no_batch(golden_dir):
    ctx = context()
    pp = lib.preprocess_params()
    k = krylon_raw(golden_dir)
    good = [k, raw_scene(4, n=10000)]
    xyz = np.random.default_rng(0).uniform(-0.1, 0.1, (20, 3)).astype(np.float32)

    def refused(code, call):
        ctx.preprocess_clouds(good, pp, read_back=False)
        assert has_batch(ctx)
        assert call() == code
        msg = lib.lib().gpdb_last_error(ctx.h).decode()
        assert not has_batch(ctx)
        return msg

    refused(ERR_INVALID, lambda: raw_call(ctx, [1, 10, 20], xyz, [1, 1], pp))   # not starting at 0
    refused(ERR_INVALID, lambda: raw_call(ctx, [0, 15, 10], xyz, [1, 1], pp))   # decreasing
    refused(ERR_INVALID, lambda: raw_call(ctx, [0, 10, 10], xyz, [1, 1], pp))   # an empty raw cloud
    refused(ERR_INVALID, lambda: raw_call(ctx, [0], xyz, [], pp))               # no cloud
    refused(ERR_INVALID, lambda: raw_call(ctx, [0, 10, 20], xyz, [1, 9], pp))   # K_b = 9
    refused(ERR_INVALID, lambda: raw_call(ctx, [0, 10, 20], xyz, [1, 1], lib.preprocess_params(estimate_normals=0)))
    refused(ERR_INVALID, lambda: raw_call(ctx, [0, 10, 20], xyz, [1, 1], lib.preprocess_params(voxel_size=0.0)))
    refused(ERR_INVALID, lambda: raw_call(ctx, [0, 10, 20], xyz, [1, 1], lib.preprocess_params(normals_radius=-1.0)))
    cam = np.ones((20, 1), np.int32)
    cam[13, 0] = 2
    msg = refused(ERR_INVALID, lambda: raw_call(ctx, [0, 10, 20], xyz, [1, 1], lib.preprocess_params(voxelize=0), cam=cam))
    assert "cloud 1: cam_source[3][0] = 2" in msg
    wide = xyz.copy()
    wide[15] = [0.5, 0.0, 0.0]  # >= 0.5 m / 0.15 um = 3.3e6 voxels > 2^21 along x in cloud 1; cloud 0 spans < 1.4e6
    msg = refused(ERR_INVALID, lambda: raw_call(ctx, [0, 10, 20], wide, [1, 1], lib.preprocess_params(voxel_size=1.5e-7)))
    assert "voxel" in msg and "cloud 1" in msg
    with pytest.raises(ValueError):  # normals on some clouds only
        ctx.preprocess_clouds([dict(k, normals=np.zeros((len(k["xyz"]), 3))), good[1]], pp)
    check(ctx, good, pp)  # the context stays usable
    # read-back without a batch, and source indices of a batch gpdb_set_clouds installed
    ctx2 = context()
    with pytest.raises(lib.GpdbError) as e:
        ctx2.get_clouds()
    assert e.value.code == ERR_STATE
    kc = scenes.krylon_cloud()
    ctx2.set_clouds([kc])
    src = np.zeros(len(kc["xyz"]), np.int32)
    assert lib.lib().gpdb_get_clouds(ctx2.h, None, None, None, src.ctypes.data_as(C.c_void_p)) == ERR_STATE
    back = ctx2.get_clouds()[0]
    assert np.array_equal(back["xyz"], kc["xyz"]) and back["normals"].tobytes() == kc["normals"].tobytes()
    assert np.array_equal(back["cam_source"], kc["cam_source"]) and "src" not in back
    ctx2.close()
    ctx.close()


def test_single_cloud_untouched(golden_dir):
    ctx = context()
    pp = lib.preprocess_params()
    k, t = krylon_raw(golden_dir), raw_scene(7)
    s1 = single(ctx, k, pp)
    sidx = scenes.sample_indices(2, len(s1["xyz"]), 64)
    d1 = ctx.detect(sidx)
    got = ctx.preprocess_clouds([t, k, t], pp)
    assert_bit_equal(dict(ctx.get_cloud(), src=_src(ctx, len(s1["xyz"]))), s1)
    assert_same(ctx.detect(sidx), d1)
    # and the reverse: gpdb_preprocess leaves the installed batch alone
    samples = samples_of(got)
    v1 = ctx.detect_batch(samples)
    single(ctx, t, pp)
    for a, g in zip(ctx.get_clouds(), got):
        assert_bit_equal(a, g)
    for a, b in zip(ctx.detect_batch(samples), v1):
        assert_same(a, b)
    ctx.close()


def _src(ctx, n):
    src = np.zeros(n, np.int32)
    assert lib.lib().gpdb_get_cloud_source_index(ctx.h, src.ctypes.data_as(C.c_void_p)) == n
    return src
