"""GPU tests of the geometry kernels' list capacities at their exact edges (-m gpu). Each case of tests/capacity_cases.py
(whose counts tests/test_capacity_cases.py proves on the CPU) fills one list to its capacity and one point past it, and
is checked three ways: against the CPU oracle under the contract of test_gpu_parity.py (frames and pose records exact,
images <= 1 LSB on <= 1e-3 of the pixels); where both image kernels apply, k_images2 against k_images
(GPD_B200_IMAGES_KERNEL=1) bit for bit; and with gpdb_debug_path_counts, which must show the next tier unused at the
capacity and used one point past it. Which store-guard and tier-decision mutations of the kernels these tests catch is
listed in DESIGN.md section 0 (capacity row)."""
import numpy as np
import pytest

import capacity_cases as cc
import image_reference as ir
import shadow_cast_reference as scr
import shadow_counters as gsc
from gpd_b200 import lib
from conftest import load_weights
from oracle import oracle
from test_gpu_batch import assert_same

pytestmark = pytest.mark.gpu


def context(cloud, **over):
    p = lib.default_params(**over)
    ctx = lib.Context(p)
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    return p, ctx, oc


def counted(ctx, call, *args):
    """(result of call(*args), path counters of that call)."""
    ctx.phase_cycles(1)
    out = call(*args)
    counts = ctx.path_counts()
    ctx.phase_cycles(0)
    return out, counts


GPDB_ERR_CAPACITY = -5


def assert_capacity_error(call, arg, what):
    """call(arg) fails with GPDB_ERR_CAPACITY, and the message names exactly one over-full neighbourhood of kind `what`."""
    with pytest.raises(lib.GpdbError) as e:
        call(arg)
    assert e.value.code == GPDB_ERR_CAPACITY and what in str(e.value), str(e.value)


# ---- k_frames: 128 (tier 0) / 1 024 (tier 1) / 16 384 (tier 2) ball keys

@pytest.mark.parametrize("n,at_position", [(cc.FRAMES_CAP0, False), (cc.FRAMES_CAP0 + 1, False), (cc.FRAMES_CAP1, False),
                                           (cc.FRAMES_CAP1 + 1, False), (cc.FRAMES_CAP2, False),
                                           (cc.FRAMES_CAP1, True), (cc.FRAMES_CAP1 + 1, True)])
def test_frames_at_the_ball_capacities(n, at_position):
    cloud, si, pos, plane = cc.frames_ball(n, at_position)
    p, ctx, oc = context(cloud)
    if at_position:
        si = ctx.set_samples(pos[None])[0]
        assert oc.set_samples(pos[None])[0] == si
    sidx = np.concatenate([[si], plane]).astype(np.int32)
    if at_position:  # gpdb_frames takes cloud points only: the frames of a sample position come with the hand search
        rg, counts = counted(ctx, ctx.hand_search, sidx)
        fg, vg = rg["frames"].reshape(-1, 9), rg["frame_valid"]
    else:
        (fg, vg), counts = counted(ctx, ctx.frames, sidx)
    fo, vo = oc.frames(p, sidx)
    assert np.array_equal(vg, vo) and vg[0] == 1
    assert np.array_equal(fg, fo)
    t1 = n > cc.FRAMES_CAP0
    t2 = n > cc.FRAMES_CAP1
    assert counts["frames_tier1"] == int(t1), counts  # the plane samples stay in tier 0
    assert counts["frames_tier2"] == int(t2), counts
    ctx.close()


def test_frames_past_the_last_tier_is_a_capacity_error():
    cloud, si, _, plane = cc.frames_ball(cc.FRAMES_CAP2 + 1)
    p, ctx, oc = context(cloud)
    sidx = np.concatenate([[si], plane]).astype(np.int32)
    assert_capacity_error(ctx.frames, sidx, "frame ball: 1 samples, hand-search ball: 0 samples, image box: 0 images")
    # the context recovers: the plane samples alone give the oracle's frames
    fg, vg = ctx.frames(plane)
    fo, vo = oc.frames(p, plane)
    assert np.array_equal(vg, vo) and np.array_equal(fg, fo)
    ctx.close()


# ---- k_hands: 2 176 (tier 1) / 12 800 (tile) / 131 072 (global memory) staged points

def hands_both(cloud, si, axes):
    over = {"hand_axes": axes, "num_orientations": 8 if len(axes) == 1 else 4}
    p, ctx, oc = context(cloud, **over)
    (rg, counts) = counted(ctx, ctx.hand_search, np.array([si], np.int32))
    fo, vo = oc.frames(p, [si])
    po, flo = oc.hand_search(p, [si], fo, vo)
    assert np.array_equal(rg["frames"].reshape(-1, 9), fo)
    assert np.array_equal(rg["pose_flags"].reshape(flo.shape), flo)
    assert ((flo & 3) == 3).any()
    cand_o = po.ravel()[(flo.ravel() & 3) == 3]
    assert rg["n_candidates"] == len(cand_o)
    for f in ("frame", "position", "top", "bottom", "center", "width", "finger_idx", "half_antipodal", "full_antipodal"):
        assert np.array_equal(rg["candidates"][f], cand_o[f]), f
    return ctx, counts


@pytest.mark.parametrize("axes", [[2], [0, 1, 2]], ids=["slab", "ball"])
@pytest.mark.parametrize("n", [cc.HANDS_CAP1, cc.HANDS_CAP1 + 1, cc.HANDS_CAP2, cc.HANDS_CAP2 + 1])
def test_hands_at_the_staging_capacities(n, axes):
    cloud, si = cc.hand_cylinder(n)
    ctx, counts = hands_both(cloud, si, axes)
    assert counts["hands_tile"] == int(n > cc.HANDS_CAP1), counts
    assert counts["hands_global"] == int(n > cc.HANDS_CAP2), counts
    ctx.close()


def test_hands_last_tier_edge_and_full_slab_passes():
    """131 072 staged points run in the global-memory tier; the slab is over 65 535 points, so every valid pose takes the
    Antipodal passes over the whole slab. One point more is GPDB_ERR_CAPACITY, and the context recovers."""
    cloud, si = cc.hand_cylinder(cc.HANDS_CAP3)
    ctx, counts = hands_both(cloud, si, [2])
    assert counts["hands_tile"] == 1 and counts["hands_global"] == 1, counts
    assert counts["hands_full_slab"] >= 1, counts
    ctx.close()
    cloud, si = cc.hand_cylinder(cc.HANDS_CAP3 + 1)
    p, ctx, oc = context(cloud)
    assert_capacity_error(ctx.hand_search, np.array([si], np.int32),
                          "frame ball: 0 samples, hand-search ball: 1 samples, image box: 0 images")
    far = np.array([len(cloud["xyz"]) - 1], np.int32)  # a plane point: far from the cylinder
    rg = ctx.hand_search(far)
    fo, vo = oc.frames(p, far)
    po, flo = oc.hand_search(p, far, fo, vo)
    assert np.array_equal(rg["pose_flags"].reshape(flo.shape), flo)
    ctx.close()


# ---- images: box lists of 1 024 (k_images2) / 2 048 (k_images) / 32 768 (global memory), in-ball list of 3 600

def images_checked(cloud, pose, ch, monkeypatch, oracle_check=True):
    p, ctx, oc = context(cloud, channels=ch)
    ig, counts = counted(ctx, ctx.images, pose)
    monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    ig1, counts1 = counted(ctx, ctx.images, pose)
    monkeypatch.delenv("GPD_B200_IMAGES_KERNEL")
    assert np.array_equal(ig, ig1)
    if oracle_check:
        io = oc.images(p, pose)
        d = np.abs(io.astype(np.int32).reshape(ig.shape) - ig.astype(np.int32))
        assert io.max() > 0 and d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    return ctx, counts, counts1


@pytest.mark.parametrize("ch", [15, 12])
@pytest.mark.parametrize("n", [cc.BOX_CAP2, cc.BOX_CAP2 + 1, cc.BOX_CAP, cc.BOX_CAP + 1])
def test_images_at_the_box_capacities(n, ch, monkeypatch):
    cloud, pose = cc.image_box(n, n_outside=100)
    ctx, counts, forced = images_checked(cloud, pose, ch, monkeypatch)
    assert counts["images2_box"] == int(n > cc.BOX_CAP2), counts
    assert counts["images2_nonunit"] == 0
    assert counts["images_global"] == int(n > cc.BOX_CAP), counts
    assert forced["images_global"] == int(n > cc.BOX_CAP), forced
    ctx.close()


@pytest.mark.parametrize("ch", [15, 12])
def test_images_last_tier_edge(ch, monkeypatch):
    cloud, pose = cc.image_box(cc.BOX_CAP_GL, n_outside=100)
    ctx, counts, _ = images_checked(cloud, pose, ch, monkeypatch)
    assert counts["images_global"] == 1
    ctx.close()
    cloud, pose = cc.image_box(cc.BOX_CAP_GL + 1, n_outside=100)
    p, ctx, oc = context(cloud, channels=ch)
    assert_capacity_error(ctx.images, pose, "frame ball: 0 samples, hand-search ball: 0 samples, image box: 1 images")
    small, spose = cc.image_box(500, n_outside=100)  # the context recovers
    ctx.set_cloud(small["xyz"], small["normals"], small["cam_source"], small["view_points"])
    oc = oracle.OracleCloud(small["xyz"], small["normals"], small["cam_source"], small["view_points"])
    ig, io = ctx.images(spose), oc.images(p, spose)
    d = np.abs(io.astype(np.int32).reshape(ig.shape) - ig.astype(np.int32))
    assert d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    ctx.close()


@pytest.mark.parametrize("n_ball", [cc.BALL_CAP2, cc.BALL_CAP2 + 1])
def test_images2_in_ball_list_capacity(n_ball, monkeypatch):
    """15 channels, 1 000 box points: the in-ball list of k_images2 holds 3 600 points; one more and the shadow casting
    walks the grid (phase counter [14])."""
    cloud, pose = cc.image_box(1000, n_outside=n_ball - 1000)
    p, ctx, oc = context(cloud, channels=15)
    ctx.phase_cycles(1)
    ig = ctx.images(pose)
    walks = int(ctx.phase_cycles(0)[14])
    assert walks == int(n_ball > cc.BALL_CAP2)
    monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    assert np.array_equal(ig, ctx.images(pose))
    monkeypatch.delenv("GPD_B200_IMAGES_KERNEL")
    io = oc.images(p, pose)
    d = np.abs(io.astype(np.int32).reshape(ig.shape) - ig.astype(np.int32))
    assert d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    ctx.close()


# ---- k_hands: closing-region members remembered per warp (SURV_CAP = 1 024, staged list <= 65 535)

@pytest.mark.parametrize("n", [cc.SURV_CAP, cc.SURV_CAP + 1])
def test_hands_closing_region_capacity(n):
    """The whole cylinder lies in the closing region of every valid pose (test_capacity_cases.py proves the count): at
    1 024 members the Antipodal passes visit the remembered list, at 1 025 every valid pose walks the whole slab."""
    cloud, si = cc.hand_cylinder(n)
    ctx, counts = hands_both(cloud, si, [2])
    p = lib.default_params(hand_axes=[2])
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    fo, vo = oc.frames(p, [si])
    po, flo = oc.hand_search(p, [si], fo, vo)
    n_valid = int(np.count_nonzero(flo & 1))
    assert (cc.closing_counts(cloud, si, po[0], flo[0])[flo[0] & 1 == 1] == n).all()
    assert counts["hands_tile"] == 0
    assert counts["hands_full_slab"] == (n_valid if n > cc.SURV_CAP else 0), counts
    ctx.close()


# ---- shadow phase of the 15-channel images: in-place fallbacks of the work list, the draw list and the voxel stash,
# counted exactly against tests/shadow_cast_reference.py (test_gpu_shadow_cast.py pins each list at its edge)

SHADOW = {
    # name: (box points, out-of-box points, cameras, overrides)
    "small": (40, 0, 1, {}),
    "work_list": (1000, 900, 1, {}),
    "draw_list": (1000, 100, 1, {}),
    "stash_1cam": (1000, 100, 1, {}),
    "stash_2cam": (1000, 100, 2, {"volume_depth": 0.05}),
}


@pytest.mark.parametrize("name", list(SHADOW))
def test_images2_shadow_fallbacks(name, monkeypatch):
    n_box, n_out, k, over = SHADOW[name]
    cloud, pose = cc.image_box(n_box, n_outside=n_out)
    if k == 2:
        cloud["view_points"] = np.array([[0.0, 0.0, 0.0], [0.3, 0.0, 0.0]])
        cloud["cam_source"] = np.ones((len(cloud["xyz"]), 2), np.int32)
    p, ctx, oc = context(cloud, channels=15, **over)
    g = ir.Geometry(C=15, d=over.get("volume_depth", 0.06))
    r = scr.cast(cloud, pose[0], g)
    ig, counts, slots = gsc.counted_images(ctx, pose, False, monkeypatch)
    ig1, forced, slots1 = gsc.counted_images(ctx, pose, True, monkeypatch)
    assert counts["images2_box"] == 0  # the fast kernel made this image itself
    assert np.array_equal(ig, ig1)
    io = oc.images(p, pose)
    d = np.abs(io.astype(np.int32).reshape(ig.shape) - ig.astype(np.int32))
    assert io[..., 14].max() > 0 and d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    box_n = cc.box_count(cloud, pose, g.w, g.d, g.h, g.radius)
    gsc.assert_counters(gsc.expected(r, g, box_n, False), counts, slots)
    gsc.assert_counters(gsc.expected(r, g, box_n, True), forced, slots1)
    ctx.close()


# ---- batches: the edge cloud in the middle of three, chunks ending inside clouds

def batch_context():
    w, relu = load_weights(15)
    p = lib.default_params(channels=15, relu_after_conv=relu, keep_images=1, chunk_samples=4)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    return ctx


def outer_clouds():
    a, sa = cc.hand_cylinder(600, seed=1)
    b, sb, _, pb = cc.frames_ball(200, seed=2)
    return (a, [sa, 1, 2, 3, 4]), (b, [sb, *pb[:4]])


def batch_vs_singles(ctx, clouds, samples):
    """detect_batch bit-equal to the single-cloud detects; returns (batch path counters, summed single-cloud counters)."""
    ctx.set_clouds(clouds)
    views, cb = counted(ctx, ctx.detect_batch, samples)
    single, cs = [], {}
    for c, s in zip(clouds, samples):
        ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        r, k = counted(ctx, ctx.detect, np.asarray(s, np.int32))
        single.append(r)
        cs = {e: cs.get(e, 0) + v for e, v in k.items()}
    for rb, rs in zip(views, single):
        assert_same(rb, rs)
    # which points a full shadow work list leaves to be cast in place follows the order of the grid walk, which differs
    # between a batch and a single cloud: the draws of the listed points (in place past the draw list) differ in number,
    # not in the bits they set (the images above are equal)
    for e in ("images2_draw_in_place", "images_draw_in_place"):
        assert (cb.pop(e) > 0) == (cs.pop(e) > 0), e
    return cb, cs


BATCH_EDGES = [("frames", cc.FRAMES_CAP1), ("frames", cc.FRAMES_CAP1 + 1), ("frames", cc.FRAMES_CAP2),
               ("hands", cc.HANDS_CAP1), ("hands", cc.HANDS_CAP1 + 1), ("hands", cc.HANDS_CAP2), ("hands", cc.HANDS_CAP2 + 1)]


@pytest.mark.parametrize("kind,n", BATCH_EDGES)
def test_batch_middle_cloud_at_the_edge(kind, n):
    """The frame and hand edges as the middle cloud of a three-cloud batch: every cloud bit-equal to its single-cloud
    call, and the batch takes exactly the tiers (and image tiers) the single-cloud calls take."""
    ctx = batch_context()
    (a, sa), (b, sb) = outer_clouds()
    if kind == "frames":
        mid, si, _, plane = cc.frames_ball(n)
        sm = [si, *plane[:4]]
    else:
        mid, si = cc.hand_cylinder(n)
        sm = [si, 5, 6, 7, 8]
    cb, cs = batch_vs_singles(ctx, [a, mid, b], [sa, sm, sb])
    assert cb == cs, (cb, cs)
    if kind == "frames":
        assert cb["frames_tier2"] == int(n > cc.FRAMES_CAP1), cb  # the outer clouds stay below tier 2
    else:
        # every sampled cylinder point with a frame stages the whole cylinder
        assert (cb["hands_tile"] >= 1) == (n > cc.HANDS_CAP1) and (cb["hands_global"] >= 1) == (n > cc.HANDS_CAP2), cb
        assert cb["images2_box"] >= 1 and cb["images_global"] >= 1, cb  # the cylinder's images overflow both box lists
    ctx.close()


def test_batch_capacity_error_then_usable():
    ctx = batch_context()
    (a, sa), (b, sb) = outer_clouds()
    mid, si = cc.hand_cylinder(cc.HANDS_CAP3 + 1)
    ctx.set_clouds([a, mid, b])
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect_batch([sa, [si], sb])
    assert e.value.code == GPDB_ERR_CAPACITY and "hand-search ball: 1 samples" in str(e.value)
    far = [len(mid["xyz"]) - 1, len(mid["xyz"]) - 2]  # plane points, far from the cylinder
    views = ctx.detect_batch([sa, far, sb])
    ctx.set_clouds([a, mid, b])  # the same batch reinstalled: the results of a fresh context's call
    for rb, rs in zip(views, ctx.detect_batch([sa, far, sb])):
        assert_same(rb, rs)
    ctx.close()
