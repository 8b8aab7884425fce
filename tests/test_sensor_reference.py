"""CPU tests of include/gpd_b200_sensor.h's restatement (tests/sensor_reference.py): the clean fixed point, the
inverse-normal table, the projector shadow and the grazing-angle cut on analytic scenes, the disparity quantisation, the
statistics of the draws on a flat wall, the header's helpers compiled for the host held bit for bit against numpy, and
the parameter checks (which run before any device work, so they need no GPU)."""
import ctypes as C

import numpy as np
import pytest
from scipy.stats import norm

import render_reference as rr
import sensor_reference as sr
from gpd_b200 import abi, lib, scenes

FX = 570.0


@pytest.fixture(scope="module")
def T():
    return sr.table()


@pytest.fixture(scope="module")
def host():
    return sr.cpp()


def camera(W=640, H=480, fx=FX, scale=1.0, pose=None):
    return lib.depth_camera(W, H, fx, fx, (W - 1) / 2, (H - 1) / 2, pose, scale)


def quad(x0, y0, x1, y1, z0, z1=None, zy=None):
    """two faces spanning x0..x1, y0..y1: z0 at x0, z1 at x1 (a plane tilted about y), or z0 at y0, zy at y1"""
    z1 = z0 if z1 is None else z1
    if zy is not None:
        v = np.array([[x0, y0, z0], [x1, y0, z0], [x1, y1, zy], [x0, y1, zy]], np.float32)
    else:
        v = np.array([[x0, y0, z0], [x1, y0, z1], [x1, y1, z1], [x0, y1, z0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def merge(*meshes):
    vs, fs, o = [], [], 0
    for v, f in meshes:
        vs.append(v)
        fs.append(f + o)
        o += len(v)
    return np.concatenate(vs), np.concatenate(fs)


def wall_and_plate():
    """a wall at z = 1.0 and a 0.2 m plate at z = 0.8 in front of it"""
    return merge(quad(-3, -3, 3, 3, 1.0), quad(-0.1, -0.1, 0.1, 0.1, 0.8))


def test_zero_parameters_give_the_render_bit_for_bit(T):
    sp = lib.sensor_params()
    assert all(getattr(sp, f) == 0.0 for f in sr.FIELDS)
    rng = np.random.default_rng(1)
    meshes = [scenes.mesh_table_scene(s, n_objects=4, segments=8)[:2] for s in (1, 2)]
    cams = [[lib.depth_camera(96, 72, 110.0, 112.0, 47.3, 35.8, rr_pose(rng), sc) for sc in (0.001, 0.0005)]
            for _ in meshes]
    for fmt in (0, 1):
        got, ref = sr.render(meshes, cams, sp, 7, fmt, T), rr.render(meshes, cams, fmt)
        for b in range(2):
            for k in range(2):
                assert np.array_equal(got[b][0][k], ref[b][0][k]) and np.array_equal(got[b][1][k], ref[b][1][k])
                assert (got[b][1][k] >= 0).sum() > 1000


def rr_pose(rng):
    import depth_reference as dr
    return dr.pose(dr.rot_x(0.1 * rng.normal()) @ dr.rot_y(0.1 * rng.normal()), rng.normal(0, 0.02, 3))


def test_table_symmetry_monotonicity_accuracy_and_host_bytes(T, host):
    assert T.shape == (4097,) and T[2048] == 0.0
    assert np.array_equal(T[::-1], -T)  # exact odd symmetry
    assert np.all(np.diff(T) >= 0) and np.all(np.diff(T[1:-1]) > 0)
    assert T[0] == T[1] and T[4096] == T[4095]
    ref = norm.ppf(np.arange(1, 4096) / 4096.0)
    assert np.abs(T[1:-1] - ref).max() <= 1e-12
    h = np.zeros(4097)
    host.so_table(rr.p_(h))
    assert np.array_equal(h.view(np.uint64), T.view(np.uint64))
    U = np.random.default_rng(2).random(20000)
    U[:4] = [0.0, 0.5, 4095 / 4096, np.nextafter(1.0, 0.0)]
    g = np.zeros_like(U)
    host.so_gauss(len(U), rr.p_(T), rr.p_(U), rr.p_(g))
    assert np.array_equal(g.view(np.uint64), sr.gauss(T, U).view(np.uint64))
    assert np.abs(g).max() <= T[4095] < 3.5


@pytest.mark.parametrize("case", ["clean", "lateral", "grazing", "shadow", "disparity", "quantised", "dropout", "all"])
def test_host_helpers_equal_the_restatement(case, T, host):
    sp = {"clean": {}, "lateral": dict(lateral_sigma=1.7), "grazing": dict(min_cos_incidence=0.4),
          "shadow": dict(baseline=0.075, shadow_tolerance=0.01), "disparity": dict(baseline=0.075, disparity_sigma=0.3),
          "quantised": dict(baseline=0.075, disparity_step=0.125), "dropout": dict(dropout=0.3),
          "all": dict(baseline=0.075, lateral_sigma=0.8, disparity_sigma=0.2, disparity_step=0.125, min_cos_incidence=0.3,
                      shadow_tolerance=0.02, dropout=0.05)}[case]
    sp = lib.sensor_params(**sp)
    v, f, _ = scenes.mesh_table_scene(3, n_objects=5, segments=10)
    import depth_reference as dr
    cam = dr.default_cameras(2, width=80, height=60, f=100.0)[1]
    key = 2 ** 63 + 11
    pose = rr.pose_of(cam)
    ct, cf = sr.clean(v, f, cam, pose)
    pt, pf = sr.clean(v, f, cam, sr.projector_pose(pose, sp.baseline)) if sp.baseline > 0 else (ct, cf)
    ref = sr.sensor_pixels(sp, T, key, 1, cam, ct, cf, pt, pf, v, f)
    face, z = sr.host_pixels(host, sp, T, key, 1, cam, ct, cf, pt, pf, v, f)
    assert np.array_equal(face, ref["face"])
    assert np.array_equal(z.view(np.uint64), ref["z"].view(np.uint64))
    assert 0 < (face >= 0).sum() < len(face)


def test_projector_shadow_band_of_an_occluding_plate(T):
    """the projector at +x casts the plate's shadow on the wall on the plate's -x side: rint(fx b (1/0.8 - 1/1.0)) = 11
    pixels wide, give or take one; the +x side and the plate itself keep their returns"""
    v, f = wall_and_plate()
    cam = camera()
    sp = lib.sensor_params(baseline=0.075, shadow_tolerance=0.01)
    img, face = sr.sensor_camera(v, f, cam, 0, 5, sp, T, 1)
    _, clean_face = rr.render_camera(v, f, cam, 1)
    expect = int(np.rint(FX * 0.075 * (1 / 0.8 - 1 / 1.0)))
    assert expect == 11
    plate = np.flatnonzero(clean_face[240] >= 2)
    u0, u1 = plate[0], plate[-1]
    for row in range(200, 281):  # rows through the plate
        lost = np.flatnonzero((face[row] < 0) & (clean_face[row] >= 0))
        # away from the image's left border, where the projector sees nothing at all
        band = lost[lost >= int(np.ceil(FX * 0.075))]
        assert len(band) and band.max() == u0 - 1 and abs(len(band) - expect) <= 1, (row, band)
        assert np.array_equal(band, np.arange(band[0], u0)), row  # one contiguous band against the plate
        assert (face[row, u0:u1 + 1] >= 2).all() and (face[row, u1 + 1:] >= 0).all()
    # the projector sees nothing left of fx b / z pixels: the left border band
    assert (face[:, :int(FX * 0.075) - 1] < 0).all()


@pytest.mark.parametrize("deg", [55.0, 70.0, 80.0])
def test_grazing_cut_on_tilted_planes(deg, T):
    """a plane through (0, 0, 1) tilted about the y axis by `deg`: exactly the pixels whose incidence cosine lies below
    min_cos_incidence lose their return"""
    a = np.radians(deg)
    x = 3.0
    v, f = quad(-x, -2, x, 2, 1.0 - x * np.tan(a), 1.0 + x * np.tan(a))
    cam = camera(160, 120, 150.0)
    thr = np.cos(np.radians(75.0))
    sp = lib.sensor_params(min_cos_incidence=thr)
    _, face = sr.sensor_camera(v, f, cam, 0, 1, sp, T, 1)
    _, clean_face = rr.render_camera(v, f, cam, 1)
    # the incidence cosine from the float32 plane's exact normal and the pixel ray
    vv = v.astype(np.float64)
    n = np.cross(vv[1] - vv[0], vv[2] - vv[0])
    dx, dy = rr.rays(cam)
    d = np.stack([dx, dy, np.ones_like(dx)], 1)
    c = np.abs(d @ n) / (np.linalg.norm(d, axis=1) * np.linalg.norm(n))
    hit = clean_face.ravel() >= 0
    sure = hit & (np.abs(c - thr) > 1e-9)
    assert np.array_equal((face.ravel() < 0)[sure], (c < thr)[sure])
    assert (c[hit] < thr).any() and (c[hit] >= thr).any()


def test_quantised_disparity_is_a_multiple_of_the_step(T):
    v, f, _ = scenes.mesh_table_scene(4, n_objects=6, segments=12)
    import depth_reference as dr
    cam = dr.default_cameras(1, width=160, height=120, f=200.0, scale=1.0)[0]
    for step in (0.125, 1 / 3, 0.5):
        sp = lib.sensor_params(baseline=0.075, disparity_sigma=0.4, disparity_step=step, shadow_tolerance=0.02)
        img, face, px = sr.sensor_camera(v, f, cam, 0, 3, sp, T, 1, detail=True)
        ret = face.ravel() >= 0
        assert ret.sum() > 5000
        Dp = px["Dp"][ret]
        assert np.array_equal(Dp, step * np.rint(Dp / step))
        assert len(np.unique(Dp)) > 10
        # and the returned depth is fx b / D'
        assert np.array_equal(px["z"][ret], (cam.fx * 0.075) / Dp)


def test_statistics_on_a_flat_wall(T):
    W, H = 640, 480  # 307 200 pixels
    v, f = quad(-5, -5, 5, 5, 1.2)
    cam = camera(W, H)
    sd = sr.table_std(T)
    assert abs(sd - 1.0) < 1e-3
    # disparity noise: D' - D has the spread sigma * sd and mean 0
    sigma = 0.35
    sp = lib.sensor_params(baseline=0.075, disparity_sigma=sigma)
    _, face, px = sr.sensor_camera(v, f, cam, 0, 17, sp, T, 1, detail=True)
    ret = face.ravel() >= 0
    n = int(ret.sum())
    assert n > 250000
    e = (px["Dp"] - px["D"])[ret]
    assert abs(e.std() / (sigma * sd) - 1.0) < 0.02
    assert abs(e.mean()) < 3 * sigma * sd / np.sqrt(n)
    # dropout: binomial within 4 sigma
    p = 0.1
    _, face, _ = sr.sensor_camera(v, f, cam, 1, 18, lib.sensor_params(dropout=p), T, 1, detail=True)
    lost = (face < 0).sum()
    assert abs(lost - p * W * H) < 4 * np.sqrt(W * H * p * (1 - p))
    # lateral jitter: the pixel each return reads, recovered from its depth on planes tilted along x and along y, is
    # shifted by rint(sigma * g) with g the table's distribution
    sig = 1.4
    sp = lib.sensor_params(lateral_sigma=sig)
    probs = {j: sr.table_cdf(T, (j + 0.5) / sig) - sr.table_cdf(T, (j - 0.5) / sig) for j in range(-6, 7)}
    for axis, plane in ((0, quad(-5, -5, 5, 5, 1.0 - 5 * 0.2, 1.0 + 5 * 0.2)), (1, quad(-5, -5, 5, 5, 1.0 - 5 * 0.2, zy=1.0 + 5 * 0.2))):
        img, face, px = sr.sensor_camera(*plane, cam, 0, 19, sp, T, 1, detail=True)
        t = img.ravel().astype(np.float64)
        ok = face.ravel() >= 0
        d = (1.0 - 1.0 / t[ok]) / 0.2  # the ray slope along the tilt
        read = np.rint(d * FX + (W - 1 if axis == 0 else H - 1) / 2)
        vv, uu = np.divmod(np.flatnonzero(ok), W)
        shift = (read - (uu if axis == 0 else vv)).astype(int)
        assert np.array_equal(shift, px["du" if axis == 0 else "dv"][ok].astype(int))
        interior = (uu >= 8) & (uu < W - 8) & (vv >= 8) & (vv < H - 8)
        m = int(interior.sum())
        for j, pj in probs.items():
            cnt = int((shift[interior] == j).sum())
            assert abs(cnt - m * pj) <= 5 * np.sqrt(m * pj * (1 - pj)) + 1, (axis, j, cnt, m * pj)


ERROR_CASES = [(dict(baseline=-0.1), "baseline must be finite and >= 0"),
               (dict(lateral_sigma=np.inf), "lateral_sigma must be finite and >= 0"),
               (dict(baseline=0.1, disparity_sigma=np.nan), "disparity_sigma must be finite and >= 0"),
               (dict(dropout=1.5), "dropout must lie in [0, 1]"),
               (dict(shadow_tolerance=1.0), "shadow_tolerance must be < 1"),
               (dict(min_cos_incidence=1.01), "min_cos_incidence must be <= 1"),
               (dict(disparity_sigma=0.1), "disparity_sigma and disparity_step need a baseline > 0"),
               (dict(disparity_step=0.1), "disparity_sigma and disparity_step need a baseline > 0")]


@pytest.mark.parametrize("fields,msg", ERROR_CASES)
def test_each_parameter_rule_is_refused(fields, msg):
    assert sr.param_error(lib.sensor_params(**fields)) == msg


def test_parameter_struct_and_edges():
    assert C.sizeof(abi.SensorParams) == 7 * 8
    with pytest.raises(TypeError):
        lib.sensor_params(base_line=1.0)
    for ok in (dict(), dict(dropout=1.0, min_cos_incidence=1.0, shadow_tolerance=0.999), dict(baseline=1e-9, disparity_step=2.0)):
        assert sr.param_error(lib.sensor_params(**ok)) is None
