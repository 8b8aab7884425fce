"""SHA-256 digests of the grasp images on fixed, seeded workloads, for both image kernels (-m gpu).

k_images2 and k_images share their phase code, so comparing the two kernels with each other cannot see a fault inside a
shared phase, and the oracle comparisons allow +-1 LSB on 1e-3 of the pixels. The images are integer and exact
fixed-point results (DESIGN.md section 4), so they are deterministic: tests/golden/image_digests.json holds their digests,
and every workload must reproduce them bit for bit, by default and with GPD_B200_IMAGES_KERNEL=1 (the general tier does
every image). The workloads reach the fast path, the general tier at 1, 3, 12 and 15 channels, image size 48, one and two
cameras, non-unit normals (k_images2 hands those images to k_images), the global-memory box list and a batch of clouds.

    python tests/test_gpu_image_digests.py [out.json]   # records the digests (default: the golden file) with the library
                                                        # in the tree, or the one GPD_B200_LIB names
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT, load_weights  # noqa: E402  (puts the repository root on sys.path)
import capacity_cases as cc  # noqa: E402
from gpd_b200 import lib, scenes  # noqa: E402
from test_gpu_image_paths import bench_cloud  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "image_digests.json")
MODES = {"default": None, "general": "1"}  # value of GPD_B200_IMAGES_KERNEL


def _context(cloud, ch, **over):
    w, relu = load_weights(ch)
    ctx = lib.Context(lib.default_params(channels=ch, relu_after_conv=relu, keep_images=1, **over))
    ctx.set_weights(w)
    if cloud is not None:
        ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    return ctx


def _detect(make_cloud, ch, **over):
    """make_cloud() -> (cloud, sample indices); built when the workload runs, not when the module is collected."""
    def run():
        cloud, sidx = make_cloud()
        ctx = _context(cloud, ch, **over)
        r = ctx.detect(sidx)
        ctx.close()
        assert r["n_candidates"] > 0
        return [r["images"]]
    return run


def _table(seed, ch, two_cameras=False, **over):
    return _detect(lambda: (scenes.synthetic_table_scene(seed, n_points=60000, two_cameras=two_cameras),
                            scenes.sample_indices(3, 60000, 1500)), ch, **over)


def _sized(size, ch):
    """LeNet takes 60 x 60 images only: other sizes go through hand search + gpdb_images."""
    def run():
        ctx = _context(scenes.synthetic_table_scene(7, n_points=60000), ch, image_size=size)
        ig = ctx.images(ctx.hand_search(scenes.sample_indices(3, 60000, 400))["candidates"])
        ctx.close()
        return [ig]
    return run


def _bench(copies=1, turn=False):
    return _detect(lambda: bench_cloud(copies, turn), 15)


def _nonunit():
    def run():
        s = scenes.synthetic_table_scene(7, n_points=60000)
        nrm = s["normals"].copy()
        nrm[::3] *= 0.97  # every third normal 3 % short: the exact fold of createNormalsImage
        ctx = _context({**s, "normals": np.ascontiguousarray(nrm)}, 15)
        ctx.phase_cycles(1)
        r = ctx.detect(scenes.sample_indices(3, 60000, 600))
        handed = ctx.path_counts()["images2_nonunit"]
        ctx.close()
        assert r["n_candidates"] > 0 and (handed > 0) == ("GPD_B200_IMAGES_KERNEL" not in os.environ)
        return [r["images"]]
    return run


def _global_box(ch):
    def run():
        cloud, pose = cc.image_box(3000, n_outside=100)
        ctx = _context(cloud, ch)
        ig = ctx.images(pose)
        ctx.close()
        return [ig]
    return run


def _batch():
    def run():
        clouds = [scenes.synthetic_table_scene(seed, n_points=30000, two_cameras=seed == 5) for seed in (4, 5, 6)]
        ctx = _context(None, 15, volume_depth=0.05)
        ctx.set_clouds(clouds)
        views = ctx.detect_batch([scenes.sample_indices(3, 30000, 400 + 50 * i) for i in range(3)])
        ctx.close()
        assert all(v["n_candidates"] > 0 for v in views)
        return [v["images"] for v in views]
    return run


WORKLOADS = {
    "bench_15ch": _bench(),
    "bench_doubled_turned_15ch": _bench(2, True),
    "two_cameras_12ch": _table(5, 12, two_cameras=True),
    "two_cameras_15ch_depth_0.05": _table(5, 15, two_cameras=True, volume_depth=0.05),
    "table_1ch": _table(7, 1),
    "table_3ch": _table(7, 3),
    "image_size_48_15ch": _sized(48, 15),
    "image_size_57_12ch": _sized(57, 12),
    "nonunit_normals_15ch": _nonunit(),
    "global_box_list_15ch": _global_box(15),
    "global_box_list_12ch": _global_box(12),
    "batch_of_3_15ch": _batch(),
}


def digest(name, mode):
    old = os.environ.pop("GPD_B200_IMAGES_KERNEL", None)
    if MODES[mode] is not None:
        os.environ["GPD_B200_IMAGES_KERNEL"] = MODES[mode]
    try:
        images = WORKLOADS[name]()
    finally:
        os.environ.pop("GPD_B200_IMAGES_KERNEL", None)
        if old is not None:
            os.environ["GPD_B200_IMAGES_KERNEL"] = old
    h = hashlib.sha256()
    for im in images:
        h.update(repr(im.shape).encode())
        h.update(np.ascontiguousarray(im).tobytes())
    return h.hexdigest()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(WORKLOADS))
def test_image_digest(name, mode):
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert digest(name, mode) == golden[name][mode]


if __name__ == "__main__":
    out = {name: {mode: digest(name, mode) for mode in MODES} for name in WORKLOADS}
    with open(sys.argv[1] if len(sys.argv) > 1 else GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(out, indent=1))
