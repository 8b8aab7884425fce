"""The numpy restatement of include/gpd_b200_depth.h (tests/depth_reference.py) and the ctypes mirror of its camera struct,
without a GPU: struct layout against the header, the float32 back-projection against float64, the raw-cloud numbering, and
the sampling rule. tests/test_abi.py holds the prototypes of the depth entry points against include/gpd_b200.h."""
import ctypes as C
import os
import re

import numpy as np

import depth_reference as dr
from gpd_b200 import abi, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header(name):
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", name)).read(), flags=re.S)


def test_camera_struct_matches_the_header():
    body = re.search(r"struct gpdb_depth_camera\s*\{(.*?)\};", header("gpd_b200_depth.h"), flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = " ".join(decl.split())
        if not decl:
            continue
        ctype, names = decl.split(" ", 1)
        for n in names.split(","):
            n = n.strip()
            m = re.match(r"(\w+)\[(\d+)\]", n)
            fields.append((m.group(1), ctype, int(m.group(2))) if m else (n, ctype, 1))
    size = {"int32_t": 4, "double": 8}
    mine = abi.DepthCamera._fields_
    assert [f[0] for f in fields] == [f[0] for f in mine]
    off = 0
    for (name, ctype, n), (_, t) in zip(fields, mine):
        al = size[ctype]
        off = (off + al - 1) // al * al
        assert getattr(abi.DepthCamera, name).offset == off, name
        assert C.sizeof(t) == size[ctype] * n, name
        off += size[ctype] * n
    assert C.sizeof(abi.DepthCamera) == off
    h = header("gpd_b200_depth.h")
    assert re.search(r"#define GPDB_DEPTH_U16 0\b", h) and re.search(r"#define GPDB_DEPTH_F32 1\b", h)
    assert (abi.DEPTH_U16, abi.DEPTH_F32) == (0, 1)


def test_float32_back_projection_within_a_few_ulps_of_float64():
    for fmt in (0, 1):
        view = dr.render_views([3], [2], fmt)[0]
        for img, cam in view:
            p32 = dr.back_project(img, cam, fmt).astype(np.float64)
            p64 = dr.back_project_f64(img, cam, fmt)
            ok = np.isfinite(p64[:, 0])
            assert ok.sum() > 0.5 * len(ok)
            assert np.array_equal(np.isfinite(p32[:, 0]), ok)
            # float32 camera coordinates (three roundings each, |value| < 2 m) through a float64 transform of a rotation,
            # then one rounding to float32: a few float32 ulps at 2 m
            assert np.abs(p32[ok] - p64[ok]).max() <= 6 * np.spacing(np.float32(2.0)), fmt


def test_validity_rules():
    z, v = dr.pixel_valid(np.array([0, 1, 500, 65535], np.uint16), 0, 0.001, 0.0005, 100.0)
    assert v.tolist() == [False, True, True, True] and z.dtype == np.float32
    raw = np.array([0.0, -1.0, np.nan, np.inf, -np.inf, 0.5, 2.0, 1.0], np.float32)
    z, v = dr.pixel_valid(raw, 1, 1.0, 0.5, 1.5)
    assert v.tolist() == [False, False, False, False, False, True, False, True]
    _, v = dr.pixel_valid(np.array([3.0e38], np.float32), 1, 10.0, 0.0, np.inf)  # overflows to inf: valid, point not finite
    assert v.tolist() == [True]


def test_raw_cloud_numbering_one_hot_and_view_points():
    cams = [lib.depth_camera(5, 4, 10, 10, 2, 1.5, dr.pose(dr.rot_y(0.1), (0.1, 0.2, 0.3))),
            lib.depth_camera(3, 2, 8, 9, 1, 0.5, dr.pose(dr.rot_x(-0.2), (-0.4, 0.0, 0.05)))]
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 3, (c.height, c.width)).astype(np.uint16) * 400 for c in cams]
    view = list(zip(imgs, cams))
    rc = dr.raw_cloud(view, 0)
    assert rc["xyz"].shape == (26, 3) and rc["cam_source"].shape == (26, 2)
    assert np.array_equal(rc["cam_source"].sum(1), np.ones(26))
    assert np.array_equal(rc["cam_source"][:20, 0], np.ones(20)) and np.array_equal(rc["cam_source"][20:, 1], np.ones(6))
    assert np.allclose(rc["view_points"], [[0.1, 0.2, 0.3], [-0.4, 0.0, 0.05]], atol=0, rtol=0)
    flat = np.concatenate([i.ravel() for i in imgs])
    assert np.array_equal(np.isnan(rc["xyz"][:, 0]), flat == 0)
    for i in range(26):
        k, v, u = dr.decode_pixel(cams, i)
        assert imgs[k][v, u] == flat[i]
        p = dr.back_project(imgs[k], cams[k], 0)[v * cams[k].width + u]
        assert np.array_equal(p, rc["xyz"][i], equal_nan=True)
    # pixel (u, v) = column u, row v, no half-pixel offset: the principal point back-projects onto the optical axis
    c = lib.depth_camera(3, 3, 50, 50, 1, 1)
    img = np.full((3, 3), 1000, np.uint16)
    p = dr.back_project(img, c, 0).reshape(3, 3, 3)
    assert p[1, 1].tolist() == [0.0, 0.0, 1.0] and p[1, 2, 0] > 0 and p[2, 1, 1] > 0


def test_sampling_ascending_unique_and_all_when_enough():
    for n in (0, 1, 7, 300):
        for k in (0, 1, 5, 299, 300, 1000):
            s = dr.subsample(n, k, 11, 2)
            assert np.all(np.diff(s) > 0) and (len(s) == 0 or (s.min() >= 0 and s.max() < n))
            assert len(s) == (n if k == 0 else min(k, n))
            if k == 0 or k >= n:
                assert np.array_equal(s, np.arange(n))


def test_sampling_respects_the_mask():
    rng = np.random.default_rng(4)
    el = rng.random(500) < 0.3
    for k in (0, 10, 149, 10000):
        s = dr.subsample(500, k, 5, 0, el)
        assert el[s].all() and np.all(np.diff(s) > 0)
        assert len(s) == (el.sum() if k == 0 else min(k, el.sum()))
    assert len(dr.subsample(500, 10, 5, 0, np.zeros(500, bool))) == 0
    # through src and the raw offsets of a batch
    off, roff = np.array([0, 3, 3, 6]), np.array([0, 10, 12, 20])
    src = np.array([9, 0, 4, 7, 1, 0])
    mask = np.zeros(20, np.uint8)
    mask[[9, 4, 12 + 7, 12]] = 1
    got = dr.subsample_batch(off, 0, 1, src, roff, mask)
    assert [g.tolist() for g in got] == [[0, 2], [], [0, 2]]


def test_sampling_draw_is_a_uniform_choice():
    """The key order is a permutation that does not favour low or high indices."""
    hits = np.zeros(200)
    for seed in range(300):
        hits[dr.subsample(200, 20, seed, 0)] += 1
    assert abs(hits[:100].sum() - hits[100:].sum()) < 0.1 * hits.sum()
    assert hits.min() > 0


def test_a_clouds_draw_does_not_depend_on_the_others():
    off_a = np.array([0, 400, 900, 1300])
    a = dr.subsample_batch(off_a, 37, 99)
    # drop the last cloud, or add one behind: cloud b keeps its draw as long as it keeps its index b (key seed + b)
    off_b = np.array([0, 400, 900])
    b = dr.subsample_batch(off_b, 37, 99)
    assert all(np.array_equal(x, y) for x, y in zip(a[:2], b))
    off_c = np.array([0, 400, 900, 1300, 2000])
    c = dr.subsample_batch(off_c, 37, 99)
    assert all(np.array_equal(x, y) for x, y in zip(a, c[:3]))
    # cloud 1 of seed s is cloud 0 of seed s + 1
    d = dr.subsample_batch(np.array([0, 500]), 37, 100)
    assert np.array_equal(d[0], a[1])
