"""The statistical outlier removal on the device: gpdb_remove_outliers and gpdb_remove_outliers_clouds against the numpy
restatement of include/gpd_b200_outliers.h (tests/outliers_reference.py), bit for bit: kept bytes, statistics and the
compacted store for mean_k = 1, 2, 10, 50, 127 and stddev_mul = 1, 0, -0.5, 2 on the krylon fixture, a table scene with
flying pixels, duplicates, a lattice and clouds of at most mean_k points. Then the batch (every install route, an empty
cloud, a cloud that loses nothing, composed source indices), the equivalence with a fresh install of the kept points
(detection, refinement, plane fit) and the state rules."""
import ctypes as C

import numpy as np
import pytest

import depth_reference as dr
import outliers_reference as orf
from conftest import load_weights
from gpd_b200 import lib, scenes
from test_outliers_reference import noisy_table, pairs
from test_refine_reference import lattice, random_normals, with_duplicates

pytestmark = pytest.mark.gpu
ERR_INVALID, ERR_STATE = -1, -3
F = np.float32
KS = [1, 2, 10, 50, 127]
MULS = [1.0, 0.0, -0.5, 2.0]


def context(weights=False, channels=15):
    w, relu = load_weights(channels)
    ctx = lib.Context(lib.default_params(channels=channels, relu_after_conv=relu))
    if weights:
        ctx.set_weights(w)
    return ctx


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def clouds():
    """name -> (xyz, normals, cam_source, view_points)."""
    rng = np.random.default_rng(21)
    kr = scenes.krylon_cloud()
    one = lambda x, s: (np.asarray(x, F), random_normals(len(x), s), None, np.zeros((1, 3)))  # noqa: E731
    return {
        "krylon": (kr["xyz"], kr["normals"], kr["cam_source"], kr["view_points"]),
        "flying_pixels": one(noisy_table(), 1),
        "duplicates": one(with_duplicates(3), 2),
        "lattice": one(lattice(7), 3),
        "small": one(rng.uniform(0, 0.1, (40, 3)), 4),
    }


_D = {}


def restated(name, xyz, k, mul):
    """(kept bools, stats) of the restatement, the mean distances cached per cloud and mean_k."""
    if len(xyz) <= k:
        return orf.remove(xyz, k, mul)[:2]
    if (name, k) not in _D:
        _D[(name, k)] = orf.mean_distances(xyz, k)
    d = _D[(name, k)]
    st = orf.stats(d, k, mul)
    return orf.keep(d, st[2]), np.array(st)


def check_single(ctx, name, cl, k, mul):
    xyz, nrm, cam, vp = cl
    ctx.set_cloud(xyz, nrm, cam, vp)
    before = ctx.get_cloud()
    r = ctx.remove_outliers(k, mul)
    kept, st = restated(name, xyz, k, mul)
    assert np.array_equal(r["kept"], kept.astype(np.uint8)), (name, k, mul)
    assert np.array_equal(bits([r["mean"], r["stddev"], r["threshold"]]), bits(st)), (name, k, mul)
    assert r["n_kept"] == kept.sum()
    if r["n_kept"] == 0:  # no point kept: no cloud
        with pytest.raises(lib.GpdbError) as ei:
            ctx.get_cloud()
        assert ei.value.code == ERR_STATE
        return
    got = ctx.get_cloud()
    for f in ("xyz", "cam_source"):
        assert np.array_equal(got[f], before[f][kept]), (name, f)
    assert np.array_equal(bits(got["normals"]), bits(before["normals"][kept]))


@pytest.mark.parametrize("k", KS)
def test_single_cloud_equals_the_restatement(k):
    ctx = context()
    n_removed = 0
    for name, cl in clouds().items():
        for mul in MULS:
            check_single(ctx, name, cl, k, mul)
            n_removed += int(len(cl[0]) > k)
    assert n_removed > 0
    ctx.close()


def test_small_clouds_and_the_threshold():
    """N <= mean_k keeps every point with NaN statistics; N = mean_k + 1 has statistics; a point exactly at the threshold
    stays; a cloud of equal mean distances whose variance residue is negative keeps every point."""
    ctx = context()
    rng = np.random.default_rng(22)
    x = rng.uniform(0, 0.1, (11, 3)).astype(F)
    for k in (10, 11, 50):
        ctx.set_cloud(x, random_normals(11, 5))
        r = ctx.remove_outliers(k, 1.0)
        kept, st = orf.remove(x, k, 1.0)[:2]
        assert np.array_equal(r["kept"], kept.astype(np.uint8))
        assert np.array_equal(bits([r["mean"], r["stddev"], r["threshold"]]), bits(st))
        assert np.isnan(r["threshold"]) == (k >= 11)
    for xyz, mul, want in ((pairs([0.25, 0.5, 0.75], 1.0), 0.0, [1, 1, 1, 1, 0, 0]),
                           (pairs([0.3] * 777, 1.0), -1.0, [1] * 1554)):
        ctx.set_cloud(xyz, np.tile([0, 0, 1.0], (len(xyz), 1)))
        r = ctx.remove_outliers(1, mul)
        assert list(r["kept"]) == want
    ctx.close()


def batch_list():
    cl = clouds()
    return [cl["krylon"][:2], cl["small"][:2], cl["flying_pixels"][:2], cl["lattice"][:2]]


@pytest.mark.parametrize("k,mul", [(1, 1.0), (10, 0.0), (50, 1.0), (50, -0.5)])
def test_batch_equals_single_cloud_calls(k, mul):
    """Each cloud of a batch as the single-cloud call on it; the 40-point cloud loses nothing at mean_k = 50."""
    torch = pytest.importorskip("torch")
    cl = batch_list()
    off = np.concatenate([[0], np.cumsum([len(x) for x, _ in cl])]).astype(np.int32)
    ctx = context()
    for route in ("host", "tensors"):
        if route == "host":
            ctx.set_clouds([{"xyz": x, "normals": n, "view_points": np.zeros((1, 3))} for x, n in cl])
        else:
            ctx.set_clouds_tensors(off, torch.from_numpy(np.concatenate([x for x, _ in cl])).cuda(),
                                   torch.from_numpy(np.concatenate([n for _, n in cl])).cuda(), [1] * len(cl),
                                   np.zeros((len(cl), 3)))
        r = ctx.remove_outliers_clouds(k, mul)
        got = ctx.get_clouds()
        kept, st, noff = orf.remove_batch(off, np.concatenate([x for x, _ in cl]), k, mul)
        assert np.array_equal(r["offsets"], noff) and np.array_equal(r["kept"], kept.astype(np.uint8))
        assert np.array_equal(bits(r["stats"]), bits(st))
        if k == 50:
            assert noff[2] - noff[1] == len(cl[1][0])
        for b, (x, n) in enumerate(cl):
            ctx.set_cloud(x, n)
            s = ctx.remove_outliers(k, mul)
            assert np.array_equal(s["kept"], r["kept"][off[b]:off[b + 1]]), b
            assert np.array_equal(bits([s["mean"], s["stddev"], s["threshold"]]), bits(r["stats"][b])), b
            if s["n_kept"]:
                one = ctx.get_cloud()
                assert np.array_equal(one["xyz"], got[b]["xyz"]) and np.array_equal(bits(one["normals"]), bits(got[b]["normals"]))
            else:
                assert len(got[b]["xyz"]) == 0
    ctx.close()


def test_preprocessed_batch_with_an_empty_cloud_keeps_source_indices():
    rng = np.random.default_rng(23)
    raws = [scenes.synthetic_raw_scene(6, n_points=20000)["xyz"], rng.uniform(5, 6, (100, 3)), rng.uniform(0, 0.05, (9, 3))]
    raws = [{"xyz": np.asarray(r, F)[np.all(np.isfinite(r), axis=1)], "view_points": np.zeros((1, 3))} for r in raws]
    ctx = context()
    before = ctx.preprocess_clouds(raws)
    assert len(before[1]["xyz"]) == 0
    r = ctx.remove_outliers_clouds(50, 1.0)
    got = ctx.get_clouds()
    assert np.isnan(r["stats"][1]).all() and np.isnan(r["stats"][2]).all() and len(got[1]["xyz"]) == 0
    o = 0
    for b in range(3):
        kept, st = orf.remove(before[b]["xyz"], 50, 1.0)[:2]
        n = len(before[b]["xyz"])
        assert np.array_equal(r["kept"][o:o + n], kept.astype(np.uint8)) and np.array_equal(bits(r["stats"][b]), bits(st))
        for f in ("xyz", "cam_source", "src"):
            assert np.array_equal(got[b][f], before[b][f][kept]), (b, f)
        assert np.array_equal(bits(got[b]["normals"]), bits(before[b]["normals"][kept]))
        o += n
    assert len(got[0]["xyz"]) < len(before[0]["xyz"])
    ctx.close()


def test_depth_install_composes_the_source_indices():
    """After gpdb_preprocess_depth_device, the kept points keep their pixel indices: subsample_clouds with a pixel mask
    equals the restatement over the compacted store."""
    torch = pytest.importorskip("torch")
    views = dr.render_views([71, 72, 73], [2, 1, 1], 0)
    ks, cams = [len(v) for v in views], [c for v in views for _, c in v]
    depth = np.concatenate([np.asarray(img).ravel() for v in views for img, _ in v]).view(np.int16)
    ctx = context()
    ctx.preprocess_depth_tensors(ks, cams, torch.from_numpy(depth).cuda(), lib.preprocess_params())
    before = ctx.get_clouds()
    r = ctx.remove_outliers_clouds(50, 1.0)
    got = ctx.get_clouds()
    assert r["offsets"][-1] < sum(len(c["xyz"]) for c in before)
    o = 0
    for b in range(len(views)):
        n = len(before[b]["xyz"])
        kept, st = orf.remove(before[b]["xyz"], 50, 1.0)[:2]
        assert np.array_equal(r["kept"][o:o + n], kept.astype(np.uint8)) and np.array_equal(bits(r["stats"][b]), bits(st))
        assert np.array_equal(got[b]["src"], before[b]["src"][kept]) and np.array_equal(got[b]["xyz"], before[b]["xyz"][kept])
        o += n
    mask = (np.random.default_rng(3).random(len(depth)) < 0.5).astype(np.uint8)
    view_off = np.concatenate([[0], np.cumsum([sum(i.size for i, _ in v) for v in views])])
    src = np.concatenate([g["src"] for g in got])
    for num in (0, 40):
        lists = ctx.subsample_clouds(num, 5, mask)
        want = dr.subsample_batch(r["offsets"], num, 5, src, view_off, mask)
        assert all(np.array_equal(a, w) for a, w in zip(lists, want))
    ctx.close()


def kept_clouds(ctx_clouds):
    return [{"xyz": c["xyz"], "normals": c["normals"], "cam_source": c["cam_source"], "view_points": c["view_points"]}
            for c in ctx_clouds]


def test_batch_equals_a_fresh_install_of_the_kept_points():
    """detect_batch_select, refine_normals_clouds and segment_planes on the compacted store equal the same calls on a
    store installed with gpdb_set_clouds from the kept points."""
    cl = clouds()
    batch = [{"xyz": x, "normals": n, "cam_source": c, "view_points": v}
             for x, n, c, v in (cl["krylon"], cl["flying_pixels"])]
    batch[1]["cam_source"] = None
    a, f = context(weights=True), context(weights=True)
    a.set_clouds([{k: v for k, v in c.items() if v is not None} for c in batch])
    a.remove_outliers_clouds(50, 1.0)
    got = a.get_clouds()
    f.set_clouds(kept_clouds(got))
    samples = [scenes.sample_indices(b + 3, len(g["xyz"]), 40) for b, g in enumerate(got)]
    for x, y in zip(a.detect_batch_select(samples, 10), f.detect_batch_select(samples, 10)):
        assert len(x) > 0 and x.tobytes() == y.tobytes()
    pa, pf = a.segment_planes(), f.segment_planes()
    for key in ("planes", "n_inliers", "n_hypotheses", "eligible"):
        assert np.array_equal(pa[key], pf[key]), key
    assert np.array_equal(a.refine_normals_clouds(10), f.refine_normals_clouds(10))
    assert all(np.array_equal(bits(x["normals"]), bits(y["normals"])) for x, y in zip(a.get_clouds(), f.get_clouds()))
    a.close()
    f.close()


def test_single_cloud_detect_equals_a_fresh_install_and_the_oracle():
    from oracle import oracle
    cloud = scenes.krylon_cloud()
    rng = np.random.default_rng(24)
    fly = (cloud["xyz"][rng.choice(len(cloud["xyz"]), 30, replace=False)] * rng.uniform(0.85, 1.15, (30, 1))).astype(F)
    xyz = np.concatenate([cloud["xyz"], fly])
    nrm = np.concatenate([cloud["normals"], random_normals(30, 24)])
    cam = np.concatenate([cloud["cam_source"], np.ones((30, 1), np.int32)])
    w, relu = load_weights(15)
    p = lib.default_params(channels=15, relu_after_conv=relu, keep_images=1)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    ctx.set_cloud(xyz, nrm, cam, cloud["view_points"])
    r = ctx.remove_outliers()
    assert r["kept"][len(cloud["xyz"]):].sum() < 30
    k = r["kept"].astype(bool)
    sidx = scenes.sample_indices(2, r["n_kept"], 48)
    rg = ctx.detect(sidx)
    ref = lib.Context(p)
    ref.set_weights(w)
    ref.set_cloud(xyz[k], nrm[k], cam[k], cloud["view_points"])
    rf = ref.detect(sidx)
    assert np.array_equal(rg["pose_flags"], rf["pose_flags"]) and np.array_equal(rg["images"], rf["images"])
    assert rg["candidates"].tobytes() == rf["candidates"].tobytes()
    oc = oracle.OracleCloud(xyz[k], nrm[k], cam[k], cloud["view_points"])
    ro = oc.detect(p, oracle.WeightPack(w), sidx)
    assert np.array_equal(ro["pose_flags"], rg["pose_flags"]) and rg["n_candidates"] == ro["n_candidates"] > 0
    d = np.abs(ro["images"].astype(np.int32) - rg["images"].astype(np.int32))
    assert d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    ctx.close()
    ref.close()


def test_preprocessed_single_cloud_keeps_source_indices():
    raw = np.asarray(scenes.synthetic_raw_scene(8, n_points=20000)["xyz"], F)
    raw = raw[np.all(np.isfinite(raw), axis=1)]
    ctx = context()
    pc = ctx.preprocess(raw)
    r = ctx.remove_outliers(50, 1.0)
    k = r["kept"].astype(bool)
    assert r["n_kept"] < len(pc["xyz"])
    src = np.zeros(r["n_kept"], np.int32)
    assert lib.lib().gpdb_get_cloud_source_index(ctx.h, src.ctypes.data_as(C.c_void_p)) >= 0
    assert np.array_equal(src, pc["src"][k]) and np.array_equal(ctx.get_cloud()["xyz"], pc["xyz"][k])
    ctx.close()


def test_errors_and_state():
    ctx = context(weights=True)
    for fn in (ctx.remove_outliers, ctx.remove_outliers_clouds):
        with pytest.raises(lib.GpdbError) as ei:
            fn(10)
        assert ei.value.code == ERR_STATE
    cl = clouds()
    x, n = cl["flying_pixels"][:2]
    x2, n2 = cl["krylon"][:2]
    ctx.set_cloud(x, n)
    ctx.set_clouds([{"xyz": x2, "normals": n2, "view_points": np.zeros((1, 3))}])

    def snapshot():
        one, many = ctx.get_cloud(), ctx.get_clouds()[0]
        return [one["xyz"].tobytes(), one["normals"].tobytes(), one["cam_source"].tobytes(), many["xyz"].tobytes(),
                many["normals"].tobytes(), many["cam_source"].tobytes()]

    s0 = snapshot()
    for k, mul in ((0, 1.0), (128, 1.0), (-1, 1.0), (10, float("nan")), (10, float("inf")), (10, -float("inf"))):
        for fn in (ctx.remove_outliers, ctx.remove_outliers_clouds):
            with pytest.raises(lib.GpdbError) as ei:
                fn(k, mul)
            assert ei.value.code == ERR_INVALID
            assert snapshot() == s0
    # the single cloud leaves the batch alone and the other way round; sample positions are dropped
    sidx = ctx.set_samples(np.asarray(x[:5], np.float64))
    ctx.remove_outliers(10, 1.0)
    assert snapshot()[3:] == s0[3:]
    with pytest.raises(lib.GpdbError) as ei:
        ctx.hand_search(sidx)
    assert ei.value.code == ERR_INVALID
    single = snapshot()[:3]
    ctx.sis_batch([scenes.sample_indices(1, len(x2), 20)], num_iterations=1)
    ctx.sis_positions()
    ctx.remove_outliers_clouds(10, 1.0)
    assert snapshot()[:3] == single
    with pytest.raises(lib.GpdbError) as ei:
        ctx.sis_positions()
    assert ei.value.code == ERR_STATE
    n_b = len(ctx.get_clouds()[0]["xyz"])
    idx = ctx.set_clouds_samples([np.asarray(x2[:5], np.float64)])
    assert idx[0][0] == n_b
    ctx.remove_outliers_clouds(10, 1.0)
    with pytest.raises(lib.GpdbError) as ei:
        ctx.hand_search_batch([idx[0]])
    assert ei.value.code == ERR_INVALID
    ctx.close()
