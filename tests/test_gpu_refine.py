"""The normal refinement on the device: gpdb_refine_normals and gpdb_refine_normals_clouds against the numpy restatement of
include/gpd_b200_refine.h (tests/refine_reference.py) and its C++ oracle (tests/refine_oracle.cpp), bit for bit: refined
normals and iteration counts for k = 1, 2, 10, 50, 128 and k >= N, on the krylon fixture, table scenes, an unvoxelised
cloud with duplicates, NaN normals from the normal estimation, and clouds built so that a wrong neighbour set or order
changes the result (a k-th neighbour several cells away, ties at the k-th place, an isolated point). Then the batch
(every install route), detection downstream of the refined normals, and the errors and state rules."""
import numpy as np
import pytest

import refine_oracle as ro
import refine_reference as rr
import depth_reference as dr
from conftest import load_weights
from gpd_b200 import lib, scenes
from test_refine_reference import lattice, random_normals, two_clusters, with_duplicates

pytestmark = pytest.mark.gpu
ERR_INVALID, ERR_STATE = -1, -3
F = np.float32
KS = [1, 2, 10, 50, 128]


def context(weights=False, channels=12):
    w, relu = load_weights(channels)
    ctx = lib.Context(lib.default_params(channels=channels, relu_after_conv=relu))
    if weights:
        ctx.set_weights(w)
    return ctx


def same_search(a, b):
    """Two hand-search results agree on every frame, pose flag and candidate record."""
    for k in ("frame_valid", "frames", "pose_flags"):
        if a[k] is not None or b[k] is not None:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k
    assert a["candidates"].tobytes() == b["candidates"].tobytes()


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def special_clouds():
    """name -> (xyz, normals): the shapes where the search or the list order decides the float32 result."""
    rng = np.random.default_rng(11)
    table = scenes.synthetic_table_scene(4, n_points=20000)
    sparse = rng.uniform(0, 1.0, (400, 3)).astype(F)  # neighbours several 2 cm cells away
    line = (np.arange(300)[:, None] * np.array([[0.013, 0.0007, 0.0]])).astype(F)  # the k-th often one shell further
    isolated = np.concatenate([rng.uniform(0, 0.05, (300, 3)), [[0.9, 0.8, 0.7]]]).astype(F)
    return {
        "krylon": (scenes.krylon_cloud()["xyz"], scenes.krylon_cloud()["normals"]),
        "table": (table["xyz"], table["normals"]),
        "duplicates": (with_duplicates(3), random_normals(450, 3)),
        "lattice_ties": (lattice(9), random_normals(729, 4)),
        "sparse": (sparse, random_normals(400, 5)),
        "line": (line, random_normals(300, 6)),
        "isolated": (isolated, random_normals(301, 7)),
        "two_clusters": two_clusters(),
    }


_REF = {}


def reference(name, xyz, nrm, k):
    """The restatement (numpy below 5 000 points, the C++ oracle above, which the CPU suite pins to numpy)."""
    key = (name, k)
    if key not in _REF:
        _REF[key] = rr.refine(xyz, nrm, k) if len(xyz) < 5000 else ro.refine(xyz, nrm, k)
    return _REF[key]


@pytest.mark.parametrize("k", KS)
def test_single_cloud_equals_the_restatement(k):
    ctx = context()
    for name, (xyz, nrm) in special_clouds().items():
        ctx.set_cloud(xyz, nrm)
        it = ctx.refine_normals(k)
        want, wit = reference(name, xyz, nrm, k)
        got = ctx.get_cloud()
        assert it == wit, name
        assert np.array_equal(bits(got["normals"]), bits(want)), name
        assert np.array_equal(got["xyz"], np.asarray(xyz, F)), name
    ctx.close()


def test_k_at_least_n_and_lattice_ties():
    """k >= N lists every point; on a lattice k = 5 and 9 cut through the six face and twelve edge neighbours that tie."""
    ctx = context()
    rng = np.random.default_rng(12)
    small = rng.uniform(0, 0.3, (40, 3)).astype(F), random_normals(40, 12)
    for xyz, nrm, k in [(*small, 40), (*small, 41), (*small, 128), (lattice(6), random_normals(216, 13), 5),
                        (lattice(6), random_normals(216, 13), 9)]:
        ctx.set_cloud(xyz, nrm)
        it = ctx.refine_normals(k)
        want, wit = rr.refine(xyz, nrm, k)
        assert it == wit and np.array_equal(bits(ctx.get_cloud()["normals"]), bits(want))
    ctx.close()


def test_nan_normals_from_the_normal_estimation():
    """gpdb_preprocess with a small radius leaves NaN normals at points with fewer than 3 neighbours; refinement skips
    them as neighbours and gives finite normals to NaN points with finite neighbours."""
    rng = np.random.default_rng(14)
    raw = np.concatenate([scenes.synthetic_raw_scene(5, n_points=20000)["xyz"], rng.uniform(-0.5, 0.5, (300, 3)) + [0, 0, 1]])
    raw = raw[np.all(np.isfinite(raw), axis=1)].astype(F)
    ctx = context()
    pc = ctx.preprocess(raw, pp=lib.preprocess_params(normals_radius=0.008))
    nan = ~np.isfinite(pc["normals"]).all(axis=1)
    assert nan.sum() > 50
    it = ctx.refine_normals(10)
    want, wit = ro.refine(pc["xyz"], pc["normals"], 10)
    got = ctx.get_cloud()["normals"]
    assert it == wit and np.array_equal(bits(got), bits(want))
    assert np.isfinite(got[nan]).all(axis=1).any()
    ctx.close()


def batch_clouds():
    sc = special_clouds()
    rng = np.random.default_rng(15)
    return [sc["krylon"], (rng.uniform(0, 0.1, (7, 3)).astype(F), random_normals(7, 15)),
            sc["two_clusters"], sc["table"], sc["isolated"], (rng.uniform(0, 0.1, (50, 3)).astype(F), np.tile([0, 0, 1.0], (50, 1)))]


@pytest.mark.parametrize("k", [1, 10, 50])
def test_batch_equals_single_cloud_calls(k):
    """A cloud smaller than k, clouds that stop at 1, 2 and 15 iterations: each as the single-cloud call."""
    cl = batch_clouds()
    ctx = context()
    ctx.set_clouds([{"xyz": x, "normals": n, "view_points": np.zeros((1, 3))} for x, n in cl])
    its = ctx.refine_normals_clouds(k)
    got = ctx.get_clouds()
    if k == 10:
        assert len({int(its[2]), int(its[5]), int(its[0])}) == 3  # different stop iterations in one batch
    for b, (x, n) in enumerate(cl):
        ctx.set_cloud(x, n)
        assert ctx.refine_normals(k) == its[b], b
        assert np.array_equal(bits(ctx.get_cloud()["normals"]), bits(got[b]["normals"])), b
    want, wits = ro.refine_batch(np.concatenate([[0], np.cumsum([len(x) for x, _ in cl])]), np.concatenate([x for x, _ in cl]),
                                 np.concatenate([n for _, n in cl]), k)
    assert np.array_equal(its, wits)
    assert np.array_equal(bits(np.concatenate([g["normals"] for g in got])), bits(want))
    ctx.close()


def test_empty_cloud_in_a_preprocessed_batch():
    """A cloud the workspace filter empties stays in the batch with no points: 0 iterations, the others unaffected."""
    rng = np.random.default_rng(16)
    raws = [scenes.synthetic_raw_scene(6, n_points=20000)["xyz"], rng.uniform(5, 6, (100, 3)), rng.uniform(0, 0.05, (9, 3))]
    raws = [{"xyz": np.asarray(r, F)[np.all(np.isfinite(r), axis=1)], "view_points": np.zeros((1, 3))} for r in raws]
    ctx = context()
    before = ctx.preprocess_clouds(raws)
    assert len(before[1]["xyz"]) == 0
    its = ctx.refine_normals_clouds(10)
    got = ctx.get_clouds()
    assert its[1] == 0
    for b in (0, 2):
        w, wit = ro.refine(before[b]["xyz"], before[b]["normals"], 10)
        assert its[b] == wit and np.array_equal(bits(got[b]["normals"]), bits(w))
    ctx.close()


def test_device_installs():
    """gpdb_set_clouds_device and gpdb_preprocess_depth_device installs, refined in place."""
    torch = pytest.importorskip("torch")
    cl = batch_clouds()[1:4]
    off = np.concatenate([[0], np.cumsum([len(x) for x, _ in cl])]).astype(np.int32)
    ctx = context()
    ctx.set_clouds_tensors(off, torch.from_numpy(np.concatenate([x for x, _ in cl])).cuda(),
                           torch.from_numpy(np.concatenate([n for _, n in cl])).cuda(), [1] * 3, np.zeros((3, 3)))
    its = ctx.refine_normals_clouds(10)
    want, wits = ro.refine_batch(off, np.concatenate([x for x, _ in cl]), np.concatenate([n for _, n in cl]), 10)
    assert np.array_equal(its, wits)
    assert np.array_equal(bits(np.concatenate([g["normals"] for g in ctx.get_clouds()])), bits(want))
    views = dr.render_views([61, 62], [2, 1], 0)
    ks, cams = [len(v) for v in views], [c for v in views for _, c in v]
    depth = np.concatenate([np.asarray(img).ravel() for v in views for img, _ in v]).view(np.int16)
    poff = ctx.preprocess_depth_tensors(ks, cams, torch.from_numpy(depth).cuda(), lib.preprocess_params())
    before = ctx.get_clouds()
    its = ctx.refine_normals_clouds(20)
    got = ctx.get_clouds()
    for b in range(len(views)):
        w, wit = ro.refine(before[b]["xyz"], before[b]["normals"], 20)
        assert its[b] == wit and np.array_equal(bits(got[b]["normals"]), bits(w))
        assert np.array_equal(got[b]["src"], before[b]["src"]) and np.array_equal(got[b]["xyz"], before[b]["xyz"])
    assert poff[-1] == sum(len(g["xyz"]) for g in got)
    ctx.close()


def test_detect_on_the_refined_cloud_equals_the_oracle():
    """The refined store detects as a cloud installed with the refined normals (GPU, bit for bit) and as the CPU oracle's
    detect on that cloud (the smoke tolerances): the nonunit flags and every other derived copy follow the normals."""
    from oracle import oracle
    cloud = scenes.krylon_cloud()
    sidx = scenes.sample_indices(2, len(cloud["xyz"]), 48)
    w, relu = load_weights(15)
    p = lib.default_params(channels=15, relu_after_conv=relu, keep_images=1)
    nrm = cloud["normals"].copy()
    nrm[::37] = np.nan  # NaN normals make the flags matter: refinement removes most of them
    ctx = lib.Context(p)
    ctx.set_weights(w)
    ctx.set_cloud(cloud["xyz"], nrm, cloud["cam_source"], cloud["view_points"])
    ctx.refine_normals(10)
    refined = ctx.get_cloud()["normals"]
    rg = ctx.detect(sidx)
    ref = lib.Context(p)
    ref.set_weights(w)
    ref.set_cloud(cloud["xyz"], refined, cloud["cam_source"], cloud["view_points"])
    rr_ = ref.detect(sidx)
    assert np.array_equal(rg["pose_flags"], rr_["pose_flags"]) and np.array_equal(rg["images"], rr_["images"])
    same_search(rg, rr_)
    oc = oracle.OracleCloud(cloud["xyz"], refined, cloud["cam_source"], cloud["view_points"])
    ro_ = oc.detect(p, oracle.WeightPack(w), sidx)
    assert np.array_equal(ro_["pose_flags"], rg["pose_flags"]) and rg["n_candidates"] == ro_["n_candidates"] > 0
    d = np.abs(ro_["images"].astype(np.int32) - rg["images"].astype(np.int32))
    assert d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    ctx.close()
    ref.close()


def test_errors_and_state():
    ctx = context()
    for fn in (ctx.refine_normals, ctx.refine_normals_clouds):
        with pytest.raises(lib.GpdbError) as ei:
            fn(10)
        assert ei.value.code == ERR_STATE
    x, n = special_clouds()["table"]
    x2, n2 = batch_clouds()[2]
    ctx.set_cloud(x, n)
    ctx.set_clouds([{"xyz": x2, "normals": n2, "view_points": np.zeros((1, 3))}])
    for k in (0, 129, -1):
        for fn in (ctx.refine_normals, ctx.refine_normals_clouds):
            with pytest.raises(lib.GpdbError) as ei:
                fn(k)
            assert ei.value.code == ERR_INVALID
    assert np.array_equal(bits(ctx.get_cloud()["normals"]), bits(n))  # unchanged after the errors
    assert np.array_equal(bits(ctx.get_clouds()[0]["normals"]), bits(n2))
    # the single cloud leaves the batch alone and the other way round
    ctx.refine_normals(10)
    assert np.array_equal(bits(ctx.get_clouds()[0]["normals"]), bits(n2))
    single = ctx.get_cloud()["normals"]
    ctx.refine_normals_clouds(3)
    assert np.array_equal(bits(ctx.get_cloud()["normals"]), bits(single))
    ctx.close()


def test_sample_positions_stay():
    """The call is not a reinstall: positions of gpdb_set_samples / gpdb_set_clouds_samples still address the same
    places, and searches from them equal those on a cloud installed with the refined normals."""
    x, n = special_clouds()["krylon"]
    pos = np.asarray(x[:20], np.float64) + 0.001
    ctx = context(weights=True)
    ctx.set_clouds([{"xyz": x, "normals": n, "view_points": np.zeros((1, 3))}])
    idx = ctx.set_clouds_samples([pos])
    ctx.refine_normals_clouds(10)
    got = ctx.hand_search_batch([idx[0]])
    ctx.set_cloud(x, n)
    sidx = ctx.set_samples(pos)
    ctx.refine_normals(10)
    single = ctx.hand_search(sidx)
    ref = context(weights=True)
    refined = ctx.get_cloud()["normals"]
    ref.set_clouds([{"xyz": x, "normals": refined, "view_points": np.zeros((1, 3))}])
    ridx = ref.set_clouds_samples([pos])
    want = ref.hand_search_batch([ridx[0]])
    same_search(got[0], want[0])
    assert got[0]["n_candidates"] > 0
    ref.set_cloud(x, refined)
    same_search(single, ref.hand_search(ref.set_samples(pos)))
    ctx.close()
    ref.close()
