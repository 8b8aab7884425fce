"""GPU parity tests (-m gpu): the CUDA path, called through the C-ABI, against the CPU oracle on identical
seeded inputs, plus size-independent properties at BASELINE's full sizes.

Tolerances (SURVEY.md 8(d)): integer / boolean outputs exact; float64 geometry within 1e-9 absolute (the kernels
follow the oracle's operation order with FMA contraction off, so in practice bit-equal); images uint8-equal except
<= 1 LSB on <= 0.1 % of pixels (the per-cell means are exact fixed-point sums on the GPU, a float32 running mean in
the reference); scores within 1e-4 relative to the largest |score| (float32 accumulation order).
"""
import ctypes

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import abi, lib, scenes
from oracle import oracle

pytestmark = pytest.mark.gpu


def make(cloud, ch, **over):
    w, relu = load_weights(ch)
    p = lib.default_params(channels=ch, relu_after_conv=relu, **over)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    return p, ctx, oc, oracle.WeightPack(w)


def assert_parity(ro, rg, ch, equal_nan=False):
    """equal_nan: frames may be NaN (clouds with NaN normals), at the same entries on both sides."""
    assert np.array_equal(ro["frame_valid"], rg["frame_valid"])
    assert np.array_equal(np.isnan(ro["frames"]), np.isnan(rg["frames"]))
    assert np.allclose(ro["frames"], rg["frames"], atol=1e-9, rtol=0, equal_nan=equal_nan)
    assert np.array_equal(ro["pose_flags"], rg["pose_flags"])
    assert ro["n_candidates"] == rg["n_candidates"]
    co, cg = ro["candidates"], rg["candidates"]
    for f in ("sample_index", "sample_slot", "pose_slot", "finger_idx", "half_antipodal", "full_antipodal"):
        assert np.array_equal(co[f], cg[f]), f
    for f in ("sample", "frame", "position", "top", "bottom", "center", "width"):
        assert np.allclose(co[f], cg[f], atol=1e-9, rtol=0), f
    if ro["images"] is not None and len(co):
        d = np.abs(ro["images"].astype(np.int32) - rg["images"].astype(np.int32))
        assert d.max() <= 1
        assert np.count_nonzero(d) <= 1e-3 * d.size
    if len(co):
        so, sg = co["score"], cg["score"]
        assert np.abs(so - sg).max() <= 1e-4 * np.abs(so).max()
        assert np.array_equal(np.isnan(ro["pose_scores"]), np.isnan(rg["pose_scores"]))


@pytest.mark.parametrize("ch,n", [(15, 160), (3, 96), (1, 40)])
def test_krylon_matches_oracle(ch, n):
    k = scenes.krylon_cloud()  # ch == 1: random-init LeNet (conftest.load_weights), the reference ships none
    p, ctx, oc, w = make(k, ch, keep_images=1)
    sidx = scenes.sample_indices(2, len(k["xyz"]), n)
    assert_parity(oc.detect(p, w, sidx), ctx.detect(sidx), ch)
    ctx.close()


def test_synthetic_table_15ch_matches_oracle():
    s = scenes.synthetic_table_scene(7, n_points=60000)
    p, ctx, oc, w = make(s, 15, keep_images=1)
    sidx = scenes.sample_indices(3, 60000, 400)
    assert_parity(oc.detect(p, w, sidx), ctx.detect(sidx), 15)
    ctx.close()


def test_two_view_12ch_relu_net_matches_oracle():
    s = scenes.synthetic_table_scene(5, n_points=60000, two_cameras=True)
    p, ctx, oc, w = make(s, 12, keep_images=1)
    sidx = scenes.sample_indices(5, 60000, 300)
    assert_parity(oc.detect(p, w, sidx), ctx.detect(sidx), 12)
    ctx.close()


def test_two_view_15ch_all_axes_and_filters():
    s = scenes.synthetic_table_scene(5, n_points=60000, two_cameras=True)
    p, ctx, oc, w = make(s, 15, keep_images=1, hand_axes=[0, 1, 2], num_orientations=4, num_finger_placements=7,
                         deepen_hand=0, filter_approach_direction=1, direction=[0.0, 0.0, 1.0], thresh_rad=1.2,
                         max_aperture=0.07, workspace_grasps=[-0.5, 0.5, -0.4, 0.4, 0.0, 1.0])
    sidx = scenes.sample_indices(5, 60000, 120)
    ro, rg = oc.detect(p, w, sidx), ctx.detect(sidx)
    assert (ro["pose_flags"] & 1).sum() > (ro["pose_flags"] & 2).sum() // 2 > 0  # the filters actually filter
    assert_parity(ro, rg, 15)
    ctx.close()


def test_stage_entry_points():
    k = scenes.krylon_cloud()
    p, ctx, oc, w = make(k, 15)
    sidx = scenes.sample_indices(2, len(k["xyz"]), 64)
    fo, vo = oc.frames(p, sidx)
    fg, vg = ctx.frames(sidx)
    assert np.array_equal(vo, vg) and np.array_equal(fo, fg)
    hs = ctx.hand_search(sidx)
    po, flo = oc.hand_search(p, sidx, fo, vo)
    assert np.array_equal(hs["pose_flags"], flo)
    cand = hs["candidates"]
    assert len(cand) == ((flo & 3) == 3).sum() and np.isnan(cand["score"]).all()
    io, ig = oc.images(p, cand[:40]), ctx.images(cand[:40])
    d = np.abs(io.astype(int) - ig.astype(int))
    assert d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    sg, lg = ctx.classify(io)
    so, lo = oracle.classify(p, w, io)
    assert np.abs(lg - lo).max() <= 1e-4 * np.abs(lo).max()
    ctx.close()


@pytest.mark.parametrize("ch", [1, 3, 12])
def test_images_entry_point_other_channel_counts(ch):
    k = scenes.krylon_cloud()
    p3, ctx3, oc, _ = make(k, 3)
    cand = ctx3.hand_search(scenes.sample_indices(2, len(k["xyz"]), 24))["candidates"][:48]
    ctx3.close()
    p = lib.default_params(channels=ch)
    ctx = lib.Context(p)
    ctx.set_cloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    io, ig = oc.images(p, cand), ctx.images(cand)
    d = np.abs(io.astype(int) - ig.astype(int))
    assert io.max() > 0 and d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    ctx.close()


@pytest.mark.parametrize("impl", [0, 1])  # 0 = wgmma convolutions, 1 = SIMT float32
@pytest.mark.parametrize("name,ch", [("lenet_caffe_15ch", 15), ("lenet_caffe_3ch", 3), ("lenet_ir_12ch", 12)])
def test_classifier_against_reference_model_goldens(golden_dir, name, ch, impl):
    import os
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    w, relu = load_weights(ch)
    p = lib.default_params(channels=ch, relu_after_conv=relu, lenet_impl=impl)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    s, lg = ctx.classify(g["images"])
    assert np.abs(lg - g["logits"]).max() <= 1e-4 * np.abs(g["logits"]).max()
    ctx.close()


def test_edge_cases_and_errors():
    k = scenes.krylon_cloud()
    p, ctx, oc, w = make(k, 15)
    r = ctx.detect(np.zeros(0, np.int32))
    assert r["n_candidates"] == 0 and r["pose_flags"].shape == (0, 8)
    r = ctx.detect(np.array([100, 100, 7], np.int32))
    assert np.array_equal(r["pose_flags"][0], r["pose_flags"][1])
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect(np.array([len(k["xyz"])], np.int32))
    assert e.value.code == -1
    ctx2 = lib.Context(p)
    with pytest.raises(lib.GpdbError) as e:
        ctx2.detect(np.array([0], np.int32))
    assert e.value.code == -3
    with pytest.raises(lib.GpdbError) as e:
        ctx2.load_weights_dir("/nonexistent/")
    assert e.value.code == -4
    ctx2.close()
    # isolated point: the hand closes on the single point, outside the workspace
    xyz = np.vstack([k["xyz"], [[5.0, 5.0, 5.0]]]).astype(np.float32)
    nrm = np.vstack([k["normals"], [[0.0, 0.0, 1.0]]])
    ctx.set_cloud(xyz, nrm, None, np.zeros((1, 3)))
    oc2 = oracle.OracleCloud(xyz, nrm, None, np.zeros((1, 3)))
    sidx = np.array([len(xyz) - 1, 3], np.int32)
    assert_parity(oc2.detect(p, w, sidx), ctx.detect(sidx), 15)
    ctx.close()


def test_full_size_properties_config3():
    """BASELINE config 3 at full size (300k points, 100k samples): properties that need no oracle at that size —
    determinism, chunk-size independence, permutation equivariance, device-resident == host path — plus exact
    parity on a random subset small enough for the oracle."""
    import torch
    s = scenes.synthetic_table_scene(3)
    sidx = scenes.sample_indices(3, len(s["xyz"]))
    p, ctx, oc, w = make(s, 15)
    a = ctx.detect(sidx)
    b = ctx.detect(sidx)
    assert np.array_equal(a["pose_flags"], b["pose_flags"]) and np.array_equal(a["pose_scores"], b["pose_scores"], equal_nan=True)
    assert a["n_candidates"] > 50000
    # chunking does not change results
    p2, ctx2, _, _ = make(s, 15, chunk_samples=4096, batch_size=1000)
    sub = sidx[:20000]
    c = ctx2.detect(sub)
    assert np.array_equal(c["pose_flags"], a["pose_flags"][:20000])
    assert np.array_equal(c["pose_scores"], a["pose_scores"][:20000], equal_nan=True)
    ctx2.close()
    # permutation equivariance
    perm = np.random.default_rng(0).permutation(20000)
    d = ctx.detect(sub[perm])
    assert np.array_equal(d["pose_flags"], a["pose_flags"][:20000][perm])
    assert np.array_equal(d["pose_scores"], a["pose_scores"][:20000][perm], equal_nan=True)
    # device-resident entry point gives the same flags / scores
    from gpd_b200 import abi
    dev = torch.device("cuda", 0)
    d_sidx = torch.from_numpy(sidx).to(dev)
    d_flags = torch.zeros(len(sidx) * 8, dtype=torch.uint8, device=dev)
    d_scores = torch.zeros(len(sidx) * 8, dtype=torch.float32, device=dev)
    st = abi.Result()
    nc = ctx.detect_resident(d_sidx.data_ptr(), len(sidx), d_flags.data_ptr(), d_scores.data_ptr(), st)
    torch.cuda.synchronize()
    assert nc == a["n_candidates"]
    assert np.array_equal(d_flags.cpu().numpy().reshape(-1, 8), a["pose_flags"])
    assert np.array_equal(d_scores.cpu().numpy().reshape(-1, 8), a["pose_scores"], equal_nan=True)
    # exact parity on a subset
    pick = np.random.default_rng(1).choice(len(sidx), 300, replace=False)
    ro = oc.detect(p, w, sidx[pick])
    assert np.array_equal(ro["pose_flags"], a["pose_flags"][pick])
    m = ~np.isnan(ro["pose_scores"])
    assert np.abs(ro["pose_scores"][m] - a["pose_scores"][pick][m]).max() <= 1e-4 * np.abs(ro["pose_scores"][m]).max()
    ctx.close()


@pytest.mark.parametrize("ch", [15, 3, 12])
def test_tensor_core_lenet_matches_simt_and_oracle_on_many_images(ch):
    """wgmma implicit-GEMM convolutions (int8 digit planes / fp16x2 split operands) vs the float32 SIMT kernels vs the oracle
    on a few thousand images, random-init weights of the reference's architecture and scale."""
    rng = np.random.default_rng(ch)
    n = 1500
    imgs = rng.integers(0, 256, (n, 60, 60, ch), dtype=np.uint8)
    imgs[: n // 2] = ((rng.random((n // 2, 60, 60, ch)) < 0.2) * imgs[: n // 2]).astype(np.uint8)
    imgs[0] = 0
    imgs[1] = 255
    w = scenes.random_lenet_weights(ch, seed=ch)
    out = {}
    for impl in (0, 1):
        p = lib.default_params(channels=ch, lenet_impl=impl, relu_after_conv=int(ch == 12))
        ctx = lib.Context(p)
        ctx.set_weights(w)
        out[impl] = ctx.classify(imgs)[1]
        ctx.close()
    so, lo = oracle.classify(p, oracle.WeightPack(w), imgs[:200])
    scale = np.abs(lo).max()
    assert np.abs(out[1][:200] - lo).max() <= 1e-4 * scale
    assert np.abs(out[0][:200] - lo).max() <= 1e-4 * scale
    assert np.abs(out[0] - out[1]).max() <= 1e-4 * np.abs(out[1]).max()


def _random_cube(n, edge, seed=0):
    rng = np.random.default_rng(seed)
    xyz = (rng.random((n, 3)) * edge).astype(np.float32)
    nrm = rng.standard_normal((n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return xyz, nrm.astype(np.float32).astype(np.float64)


def test_frames_of_an_unvoxelised_cloud_use_the_global_tier():
    """500 k points in a 10 cm cube: ~2 100 points per r = 1 cm ball, more than the 1 024-key shared-memory list of
    k_frames. The global-memory tier (16 384 keys per warp) must give the oracle's frames (same sorted accumulation order)."""
    xyz, nrm = _random_cube(500000, 0.1)
    p = lib.default_params(channels=3)
    ctx = lib.Context(p)
    ctx.set_cloud(xyz, nrm, None, np.zeros((1, 3)))
    oc = oracle.OracleCloud(xyz, nrm, None, np.zeros((1, 3)))
    sidx = np.arange(0, 500000, 2500, dtype=np.int32)
    assert max(len(oc.radius_search(xyz[i], 0.01)[0]) for i in sidx[:40]) > 1024
    fo, vo = oc.frames(p, sidx)
    fg, vg = ctx.frames(sidx)
    assert np.array_equal(vo.astype(bool), vg.astype(bool))
    assert np.array_equal(fo.reshape(fg.shape), fg)
    ctx.close()


def test_capacity_error_is_reported_not_crashed():
    """A cloud denser than every tier (16 384 points in the r = 1 cm ball) must fail with GPDB_ERR_CAPACITY (-5), and the
    context must stay usable."""
    xyz, nrm = _random_cube(400000, 0.03)  # ~62 k points per ball in the interior
    p = lib.default_params(channels=3)
    ctx = lib.Context(p)
    ctx.set_cloud(xyz, nrm, None, np.zeros((1, 3)))
    mid = np.argsort(np.linalg.norm(xyz - 0.015, axis=1))[:8].astype(np.int32)
    with pytest.raises(lib.GpdbError) as e:
        ctx.frames(mid)
    assert e.value.code == -5 and "denser" in str(e.value)
    k = scenes.krylon_cloud()
    ctx.set_cloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    f, v = ctx.frames(np.arange(10, dtype=np.int32))
    assert v.all()
    ctx.close()


def _lattice_cloud(step, half=0.09):
    g = np.arange(-half, half, step)
    X, Y = np.meshgrid(g, g, indexing="ij")
    Z = 0.6 + 0.01 * np.sin(40 * X) * np.cos(30 * Y)
    xyz = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1).astype(np.float32)
    rng = np.random.default_rng(1)
    nrm = np.tile([0.0, 0.0, -1.0], (len(xyz), 1)) + rng.normal(0, 0.05, (len(xyz), 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return {"xyz": xyz, "normals": nrm.astype(np.float32).astype(np.float64), "cam_source": None, "view_points": np.zeros((1, 3))}, rng


def test_dense_clouds_go_through_the_overflow_tiers():
    """Lattices 6x / 9x denser than a 3 mm voxelised cloud. The hand-search slab leaves the 2 176-point tile (12 800-point
    pass) and then shared memory altogether (global-memory tier, 31 k points); the image boxes leave the 1 024- and
    2 048-point lists (global-list tier of k_images, ~3 400 points). The reference has no capacity limit: frames, hands,
    images and scores must still equal the oracle."""
    cloud, rng = _lattice_cloud(0.0012)
    xyz = cloud["xyz"]
    p, ctx, oc, w = make(cloud, 15, keep_images=1)
    center = np.argsort(np.linalg.norm(xyz[:, :2], axis=1))[:2000]
    sidx = center[rng.choice(2000, 60, replace=False)].astype(np.int32)
    assert len(oc.radius_search(xyz[sidx[0]], 0.11)[0]) > 12800
    ro, rg = oc.detect(p, w, sidx), ctx.detect(sidx)
    assert rg["n_candidates"] > 0
    assert_parity(ro, rg, 15)
    ctx.close()
    # image stage on a 1 mm lattice, for hands found on its 3 mm subset (enough of them, with large boxes)
    dense, rng = _lattice_cloud(0.001)
    coarse, _ = _lattice_cloud(0.003)
    for ch in (15, 12):
        pc, ctx_c, oc_c, wc = make(coarse, ch)
        poses = ctx_c.hand_search(np.arange(0, len(coarse["xyz"]), 7, dtype=np.int32))["candidates"][::6]
        ctx_c.close()
        assert len(poses) >= 40
        pd, ctx_d, oc_d, wd = make(dense, ch)
        assert len(oc_d.radius_search(dense["xyz"][len(dense["xyz"]) // 2 + 90], 0.11)[0]) > 12800
        box = []  # points inside the image volume of each hand: all three list tiers (<= 1 024, <= 2 048, global) must occur
        for c in poses:
            loc = (dense["xyz"].astype(np.float64) - c["sample"]) @ c["frame"].reshape(3, 3).T
            box.append(np.count_nonzero((loc[:, 0] > c["bottom"]) & (loc[:, 0] < c["bottom"] + 0.06) & (np.abs(loc[:, 1] - c["center"]) < 0.05)
                                        & (np.abs(loc[:, 2]) < 0.02)))
        box = np.array(box)
        assert (box > 2048).sum() >= 10 and ((box > 1024) & (box <= 2048)).sum() >= 5 and (box <= 1024).sum() >= 1, np.percentile(box, [0, 50, 100])
        io, ig = oc_d.images(pd, poses), ctx_d.images(poses)
        d = np.abs(io.astype(np.int32).reshape(ig.shape) - ig.astype(np.int32))
        assert d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
        so = oracle.classify(pd, wd, io.reshape(len(poses), -1))[0]
        sg = ctx_d.classify(ig)[0]
        assert np.abs(so - sg).max() <= 1e-4 * np.abs(so).max()
        # re-labelling of the same hands against the dense cloud (one warp per hand, straight from the grid)
        lo, ho = oc_d.reevaluate(pd, poses)
        lg, hg = ctx_d.reevaluate(poses)
        assert np.array_equal(lo, lg) and np.array_equal(ho["half_antipodal"], hg["half_antipodal"])
        ctx_d.close()


def test_config2_krylon_with_replacement():
    """BASELINE config 2: krylon, 10 000 samples drawn with replacement, 15 channels."""
    k = scenes.krylon_cloud()
    p, ctx, oc, w = make(k, 15)
    sidx = scenes.sample_indices(2, len(k["xyz"]))
    assert len(sidx) == 10000
    r = ctx.detect(sidx)
    # duplicated sample indices must give identical rows
    order = np.argsort(sidx, kind="stable")
    s_sorted = sidx[order]
    dup = np.where(s_sorted[1:] == s_sorted[:-1])[0]
    assert len(dup) > 1000
    a, b = order[dup], order[dup + 1]
    assert np.array_equal(r["pose_flags"][a], r["pose_flags"][b])
    assert np.array_equal(r["pose_scores"][a], r["pose_scores"][b], equal_nan=True)
    pick = np.random.default_rng(2).choice(len(sidx), 200, replace=False)
    ro = oc.detect(p, w, sidx[pick])
    assert np.array_equal(ro["pose_flags"], r["pose_flags"][pick])
    m = ~np.isnan(ro["pose_scores"])
    assert np.abs(ro["pose_scores"][m] - r["pose_scores"][pick][m]).max() <= 1e-4 * np.abs(ro["pose_scores"][m]).max()
    ctx.close()


def test_config5_two_view_12ch_full_cloud():
    """BASELINE config 5 cloud (300 k points, two cameras, 12-channel ReLU net): 20 000 samples on the GPU,
    exact parity on a subset."""
    s = scenes.synthetic_table_scene(5, two_cameras=True)
    p, ctx, oc, w = make(s, 12)
    sidx = scenes.sample_indices(5, len(s["xyz"]), 20000)
    r = ctx.detect(sidx)
    assert r["n_candidates"] > 5000
    pick = np.random.default_rng(3).choice(len(sidx), 250, replace=False)
    ro = oc.detect(p, w, sidx[pick])
    assert np.array_equal(ro["pose_flags"], r["pose_flags"][pick])
    m = ~np.isnan(ro["pose_scores"])
    assert m.sum() > 50
    assert np.abs(ro["pose_scores"][m] - r["pose_scores"][pick][m]).max() <= 1e-4 * np.abs(ro["pose_scores"][m]).max()
    ctx.close()


def test_detect_select_is_detect_plus_select_grasps():
    """gpdb_detect_select = detectGrasps steps 1-4 + selectGrasps (grasp_detector.cpp:405-420): the k best candidate
    records, descending score, ties in candidate order; bit-equal to sorting gpdb_detect's candidates on the host."""
    s = scenes.synthetic_table_scene(7, n_points=60000)
    p, ctx, oc, w = make(s, 15, chunk_samples=512)  # several chunks: candidates of all chunks compete
    sidx = scenes.sample_indices(3, 60000, 3000)
    full = ctx.detect(sidx)
    cand = full["candidates"]
    order = np.argsort(-cand["score"].astype(np.float64), kind="stable")
    for k in (0, 1, 50, len(cand), len(cand) + 10):
        r = ctx.detect_select(sidx, k)
        kk = min(k, len(cand))
        assert r["n_candidates"] == kk and r["n_total_candidates"] == len(cand) and r["frames"] is None
        for f in cand.dtype.names:  # field by field: the struct's trailing padding bytes are not part of the contract
            assert np.array_equal(r["candidates"][f], cand[order[:kk]][f]), (k, f)
    # against the oracle's scores (selection is a pure sort, so the same tolerance as the scores applies)
    ro = oc.detect(p, w, sidx)
    oo = np.argsort(-ro["candidates"]["score"].astype(np.float64), kind="stable")[:20]
    r = ctx.detect_select(sidx, 20)
    assert np.abs(r["candidates"]["score"] - ro["candidates"]["score"][oo]).max() <= 1e-4 * np.abs(ro["candidates"]["score"]).max()
    ctx.close()


def test_sample_positions_match_oracle():
    """gpdb_set_samples (Cloud::setSamples): arbitrary float64 sample positions addressed by indices >= N, against the
    oracle; positions that coincide with cloud points reproduce the index-mode poses and flags."""
    s = scenes.synthetic_table_scene(7, n_points=60000)
    p, ctx, oc, w = make(s, 15, keep_images=1)
    sidx = scenes.sample_indices(3, 60000, 300)
    pos = s["xyz"][sidx].astype(np.float64) + np.random.default_rng(1).normal(0, 1e-3, (300, 3))
    gi, oi = ctx.set_samples(pos), oc.set_samples(pos)
    assert np.array_equal(gi, oi) and gi[0] == 60000
    rg = ctx.detect(gi)
    assert_parity(oc.detect(p, w, oi), rg, 15)
    assert np.array_equal(rg["candidates"]["sample"], pos[rg["candidates"]["sample_slot"]])
    # on-cloud positions == index mode; mixed indices in one call
    gj = ctx.set_samples(s["xyz"][sidx].astype(np.float64))
    a, b = ctx.detect(sidx), ctx.detect(gj)
    assert np.array_equal(a["frames"], b["frames"]) and np.array_equal(a["pose_flags"], b["pose_flags"])
    for f in ("sample", "frame", "position", "top", "bottom", "center", "width", "finger_idx"):
        assert np.array_equal(a["candidates"][f], b["candidates"][f]), f
    with pytest.raises(lib.GpdbError):
        ctx.detect(np.array([60000 + 300], np.int32))  # beyond the sample positions
    ctx.set_cloud(s["xyz"], s["normals"], s["cam_source"], s["view_points"])  # a new cloud drops the positions
    with pytest.raises(lib.GpdbError):
        ctx.detect(np.array([60000], np.int32))
    ctx.close()


@pytest.mark.gpu
def test_sharded_entry_points_on_one_rank_equal_detect():
    """The multi-GPU code path of the library (gpdb_comm_init -> ncclCommInitRank, gpdb_set_cloud_bcast -> ncclBroadcast,
    gpdb_detect_sharded -> ncclAllGather) with a one-rank communicator: results bit-equal to gpdb_detect on the same samples.
    (N > 1: tools/multi_gpu_check.py under torchrun, and bench.py's parity_check.)"""
    s = scenes.krylon_cloud()
    sidx = scenes.sample_indices(2, len(s["xyz"]), 300)
    p, ctx, oc, w = make(s, 15)
    ref = ctx.detect(sidx)
    ctx.comm_init(lib.comm_unique_id(), 0, 1)
    # a preprocessed cloud has source indices; the broadcast cloud that replaces it has none
    wide = lib.preprocess_params(workspace=(-1e3, 1e3, -1e3, 1e3, -1e3, 1e3), voxelize=0, estimate_normals=0)
    assert ctx.preprocess(s["xyz"], s["cam_source"], s["view_points"], wide, normals=s["normals"])["src"].size > 0
    n = ctx.set_cloud_bcast(0, s["xyz"], s["normals"], s["cam_source"], s["view_points"])
    assert n == len(s["xyz"])
    src = np.zeros(n, np.int32)
    assert lib.lib().gpdb_get_cloud_source_index(ctx.h, src.ctypes.data_as(ctypes.c_void_p)) == -3  # GPDB_ERR_STATE
    with pytest.raises(lib.GpdbError):  # refused arguments leave the installed cloud in place
        ctx.preprocess(s["xyz"], s["cam_source"], s["view_points"], lib.preprocess_params(voxel_size=0.0))
    sh = ctx.detect_sharded(sidx)
    assert np.array_equal(sh["pose_flags"], ref["pose_flags"])
    assert np.array_equal(sh["pose_scores"].view(np.uint32), ref["pose_scores"].view(np.uint32))
    assert sh["n_candidates"] == ref["n_candidates"] == sh["n_total_candidates"]
    assert sh["candidates"].tobytes() == ref["candidates"].tobytes()
    ctx.close()


@pytest.mark.gpu
def test_result_arena_is_reused_and_outlives_the_context():
    """Results live in pinned host arenas of the context: freed results hand the arena back (same pointers on the next call),
    two outstanding results get distinct arenas, and a result may be freed after gpdb_destroy."""
    import ctypes as C
    s = scenes.krylon_cloud()
    sidx = np.ascontiguousarray(scenes.sample_indices(2, len(s["xyz"]), 200))
    p, ctx, oc, w = make(s, 15, chunk_samples=64)
    r1, r2 = abi.Result(), abi.Result()
    n1 = ctx.detect_raw(sidx, r1)
    a1 = C.cast(r1.candidates, C.c_void_p).value
    snap = C.string_at(r1.candidates, n1 * C.sizeof(abi.Pose))
    n2 = ctx.detect_raw(sidx, r2)  # r1 still outstanding -> another arena
    a2 = C.cast(r2.candidates, C.c_void_p).value
    assert n1 == n2 > 0 and a1 != a2
    assert C.string_at(r1.candidates, n1 * C.sizeof(abi.Pose)) == snap == C.string_at(r2.candidates, n2 * C.sizeof(abi.Pose))
    lib.free_result(r1)
    assert not r1.candidates
    n3 = ctx.detect_raw(sidx, r1)
    assert n3 == n1 and C.cast(r1.candidates, C.c_void_p).value == a1  # the freed arena is reused
    ctx.close()
    assert C.string_at(r2.candidates, n2 * C.sizeof(abi.Pose)) == snap  # still readable after gpdb_destroy
    lib.free_result(r1)
    lib.free_result(r2)


@pytest.mark.gpu
@pytest.mark.parametrize("ch,two_cams", [(15, False), (15, True), (12, True), (3, False), (1, False)])
def test_image_kernels_agree(ch, two_cams, monkeypatch):
    """The two image kernels — k_images2 (fast path: two CTAs per SM, 1024-point box list, two-pass shadow sums, point
    planes parked in the image's own memory) and k_images (general tier, also the overflow tier of the fast path) — must
    produce bit-identical images; both are compared with the oracle elsewhere. The fast path must actually have run: it
    launches one kernel more per image batch (one batch here) than the general tier alone. Two cameras' 15-channel shadow
    bitmaps fit k_images2 only at an image depth below the default 0.06 (DESIGN §4)."""
    s = scenes.synthetic_table_scene(5 if two_cams else 7, n_points=60000, two_cameras=two_cams)
    p, ctx, oc, w = make(s, ch, keep_images=1, **({"volume_depth": 0.05} if ch == 15 and two_cams else {}))
    sidx = scenes.sample_indices(3, 60000, 1500)
    monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    general = ctx.detect(sidx)
    monkeypatch.delenv("GPD_B200_IMAGES_KERNEL")
    fast = ctx.detect(sidx)
    assert general["n_candidates"] > 300
    assert fast["kernel_launches"] == general["kernel_launches"] + 1
    assert np.array_equal(general["images"], fast["images"])
    ctx.close()


@pytest.mark.gpu
def test_reevaluate_hypotheses_matches_oracle():
    """gpdb_reevaluate (HandSearch::reevaluateHypotheses / GraspDetector::evalGroundTruth): labels and half / full flags of
    given hands against the installed cloud — the same cloud, and a thinned "ground-truth" cloud — equal the oracle's."""
    s = scenes.synthetic_table_scene(7, n_points=60000)
    p, ctx, oc, w = make(s, 15)
    c = ctx.hand_search(scenes.sample_indices(3, 60000, 1200))["candidates"]
    assert len(c) > 300
    lo, ho = oc.reevaluate(p, c)
    lg, hg = ctx.reevaluate(c)
    assert np.array_equal(lo, lg) and np.array_equal(lg, c["full_antipodal"].astype(np.int32))
    for f in ("half_antipodal", "full_antipodal"):
        assert np.array_equal(ho[f], hg[f]), f
    keep = np.arange(60000) % 4 != 1
    ctx.set_cloud(s["xyz"][keep], s["normals"][keep], s["cam_source"][keep], s["view_points"])
    thin = oracle.OracleCloud(s["xyz"][keep], s["normals"][keep], s["cam_source"][keep], s["view_points"])
    lo, ho = thin.reevaluate(p, c)
    lg, hg = ctx.reevaluate(c)
    assert np.array_equal(lo, lg)
    for f in ("half_antipodal", "full_antipodal"):
        assert np.array_equal(ho[f], hg[f]), f
    assert not np.array_equal(hg["half_antipodal"], c["half_antipodal"])  # the thinner cloud does change labels
    ctx.close()
