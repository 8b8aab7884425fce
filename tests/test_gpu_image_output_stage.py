"""The image kernels pixel for pixel at the edges of the output stage (-m gpu): for every case of tests/image_cases.py,
under the default kernel choice and with GPD_B200_IMAGES_KERNEL=1 (k_images for every image), the device's images equal
the kernel-mode restatement (tests/image_reference.py) bit for bit, every pixel where the device differs from the
oracle is one where the kernel and reference restatements differ, and gpdb_debug_path_counts shows the intended tier.
test_image_cases.py proves on the CPU that the cases reach what they claim and that the oracle equals the reference
mode."""
import functools

import numpy as np
import pytest

import image_cases as ic
import image_reference as ir
from gpd_b200 import lib
from oracle import oracle

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def cases():
    return {c["name"]: c for c in ic.all_cases()}


def _params(case):
    g = case["geometry"]
    return lib.default_params(channels=g.C, image_size=g.S, volume_width=g.w, volume_depth=g.d, volume_height=g.h)


@pytest.mark.parametrize("forced", [False, True], ids=["default", "k_images"])
@pytest.mark.parametrize("name", [c["name"] for c in ic.all_cases()])
def test_device_images_equal_the_kernel_restatement(name, forced, monkeypatch):
    case = cases()[name]
    c, g = case["cloud"], case["geometry"]
    ctx = lib.Context(_params(case))
    ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    if forced:
        monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    ctx.phase_cycles(1)
    dev = ctx.images(case["poses"]).reshape(len(case["poses"]), g.S, g.S, g.C)
    counts = ctx.path_counts()
    ctx.phase_cycles(0)
    ctx.close()
    oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    io = oc.images(ic.params_of(case), case["poses"])
    qt = oracle.qtab()
    for i, pose in enumerate(case["poses"]):
        ker = ir.image(c, pose, g, "kernel", qtab=qt)
        assert np.array_equal(dev[i], ker), (name, i, case["claims"][i], np.argwhere(dev[i] != ker)[:8])
        ref = ir.image(c, pose, g, "reference", qtab=qt)
        assert not np.any((dev[i] != io[i]) & (ker == ref)), (name, i)
    # the tiers: k_images2 (S = 60, unit normals) hands larger boxes to k_images, whose global list takes > 2 048 points
    tiers = [cl["tier"] for cl in case["claims"]]
    n_gl = sum(t == "gl" for t in tiers)
    fast = g.S == 60 and not forced
    n_over = sum(t in ("shared", "gl") for t in tiers) if fast else 0
    n_nonunit = sum(bool(cl.get("nonunit")) and cl["tier"] == "images2" for cl in case["claims"]) if fast else 0
    assert counts["images2_box"] == n_over, counts
    assert counts["images2_nonunit"] == n_nonunit, counts
    assert counts["images_global"] == n_gl, counts


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_cta_reuse_alternating_covered_and_uncovered():
    """More images than CTAs: k_images runs one CTA per SM as k_images2's overflow tier, so each CTA makes several
    images in turn. 3 x SM-count + 7 poses of 1 025 - 2 048 box points, two in every five uncovered (5 divides
    neither 132 nor 114 SMs, so each CTA meets both kinds), the rest covered lattices; the one-call images equal the images made one call per
    pose."""
    g = ir.Geometry(C=12, **ic.DEFAULT)
    b = ic.Builder(g, seed=60)
    S = g.S
    n = 3 * _sm_count() + 7
    for k in range(n):
        hole = {(S - 1 - 30, 30)} if k % 5 in (1, 3) else set()
        cells = ic.lattice(S, 2, 0, 1, np.arange(3, S - 3), b.rng, hole)
        cells = np.vstack([cells, cells[::2] + np.array([0, 0, 1])])
        b.add(b.cells_to_hand(cells), b.tilted(len(cells)), {"tier": "shared"})
    case = b.case("reuse")
    c = case["cloud"]
    ctx = lib.Context(_params(case))
    ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    ctx.phase_cycles(1)
    all_at_once = ctx.images(case["poses"])
    counts = ctx.path_counts()
    ctx.phase_cycles(0)
    assert counts["images2_box"] == n and counts["images_global"] == 0, counts
    for i in range(n):
        assert np.array_equal(all_at_once[i], ctx.images(case["poses"][i:i + 1])[0]), i
    ctx.close()


def test_images2_cta_reuse_in_one_detect_chunk():
    """k_images2 launches min(images, 64 x SM-count) CTAs and gpdb_images makes at most 8 192 images per call, so only a
    gpdb_detect chunk of more candidates hands a k_images2 CTA a second image. One chunk of the bench cloud with more
    than 64 x SM-count candidates, images kept: they equal the same candidates' images made by gpdb_images 300 at a
    time (one image per CTA)."""
    from conftest import load_weights
    from gpd_b200 import scenes
    cloud = scenes.synthetic_table_scene(3)
    w, relu = load_weights(15)
    sidx = scenes.sample_indices(3, len(cloud["xyz"]), 30000)
    ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu, keep_images=1, chunk_samples=len(sidx)))
    ctx.set_weights(w)
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    r = ctx.detect(sidx)
    nc = r["n_candidates"]
    assert nc > 64 * _sm_count(), nc
    kept = np.asarray(r["images"]).reshape(nc, -1)
    for b0 in range(0, nc, 300):
        one = np.asarray(ctx.images(r["candidates"][b0:b0 + 300])).reshape(-1, kept.shape[1])
        assert np.array_equal(one, kept[b0:b0 + 300]), b0
    ctx.close()
