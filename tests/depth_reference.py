"""numpy restatement of include/gpd_b200_depth.h: back-projection, the raw cloud of a view and Cloud::subsample; plus a
z-buffer renderer that turns gpd_b200.scenes tables into depth images.

The back-projection is float32 per rounded operation, the world transform float64 per rounded operation with one final
rounding to float32 (numpy's elementwise ufuncs never fuse a multiply and an add), so the points match the library's bit
for bit. The sampling keys are sis_reference.philox with stream word 2.
"""
import numpy as np

from gpd_b200 import lib, scenes
from sis_reference import philox

F32 = np.float32


def rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1.0, 0, 0], [0, c, -s], [0, s, c]])


def rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1.0, 0], [-s, 0, c]])


def pose(R, t):
    """The 3 x 4 camera-to-world matrix [R | t]."""
    return np.hstack([np.asarray(R, np.float64), np.asarray(t, np.float64).reshape(3, 1)])


def pixel_valid(raw, fmt, scale, min_depth, max_depth):
    """(z float32, valid) of raw depth values (gpd_b200_depth.h 2)."""
    raw = np.asarray(raw)
    if fmt == 0:
        z = raw.astype(F32) * F32(scale)
        ret = raw != 0
    else:
        raw = raw.astype(F32)
        with np.errstate(over="ignore", invalid="ignore"):
            z = raw * F32(scale)
            ret = np.isfinite(raw) & (raw > 0)
    zd = z.astype(np.float64)
    with np.errstate(invalid="ignore"):
        valid = ret & (zd >= min_depth) & (zd <= max_depth)
    return z, valid


def back_project(raw, cam, fmt):
    """The points [H*W, 3] float32 of one camera's image in row-major pixel order (NaN where the pixel is not valid)."""
    H, W = int(cam.height), int(cam.width)
    z, valid = pixel_valid(np.asarray(raw).reshape(H * W), fmt, cam.depth_scale, cam.min_depth, cam.max_depth)
    v, u = np.divmod(np.arange(H * W), W)
    with np.errstate(over="ignore", invalid="ignore"):
        xc = ((u.astype(F32) - F32(cam.cx)) * z) / F32(cam.fx)
        yc = ((v.astype(F32) - F32(cam.cy)) * z) / F32(cam.fy)
        c = [xc.astype(np.float64), yc.astype(np.float64), z.astype(np.float64)]
        P = np.array(cam.pose[:], np.float64).reshape(3, 4)
        out = np.stack([(((P[r, 0] * c[0] + P[r, 1] * c[1]) + P[r, 2] * c[2]) + P[r, 3]).astype(F32) for r in range(3)], 1)
    out[~valid] = np.nan
    return out


def back_project_f64(raw, cam, fmt):
    """The same points in float64 throughout (for the rounding bound of the float32 arithmetic)."""
    H, W = int(cam.height), int(cam.width)
    z32, valid = pixel_valid(np.asarray(raw).reshape(H * W), fmt, cam.depth_scale, cam.min_depth, cam.max_depth)
    z = z32.astype(np.float64)
    v, u = np.divmod(np.arange(H * W), W)
    c = np.stack([(u - cam.cx) * z / cam.fx, (v - cam.cy) * z / cam.fy, z], 1)
    P = np.array(cam.pose[:], np.float64).reshape(3, 4)
    out = c @ P[:, :3].T + P[:, 3]
    out[~valid] = np.nan
    return out


def raw_cloud(view, fmt):
    """The raw cloud of one view, a list of (image, camera) (gpd_b200_depth.h 3): xyz [N, 3] (NaN for invalid pixels),
    one-hot cam_source [N, K] int32, view_points [K, 3] = the t vectors."""
    K = len(view)
    xyz, cam = [], []
    for k, (img, c) in enumerate(view):
        p = back_project(img, c, fmt)
        xyz.append(p)
        oh = np.zeros((len(p), K), np.int32)
        oh[:, k] = 1
        cam.append(oh)
    vps = np.array([[c.pose[3], c.pose[7], c.pose[11]] for _, c in view], np.float64)
    return {"xyz": np.concatenate(xyz), "cam_source": np.concatenate(cam), "view_points": vps}


def decode_pixel(view_cams, i):
    """(camera, v, u) of raw point i of a view with cameras view_cams."""
    for k, c in enumerate(view_cams):
        n = int(c.width) * int(c.height)
        if i < n:
            return k, i // int(c.width), i % int(c.width)
        i -= n
    raise IndexError("raw index beyond the view's pixels")


def sample_keys(seed, b, j):
    """The 64-bit keys (uint64) of cloud-local points j of cloud b."""
    key = (int(seed) + int(b)) & 0xFFFFFFFFFFFFFFFF
    j = np.asarray(j, np.uint32)
    ctr = np.stack([j, np.zeros_like(j), np.full_like(j, 2), np.zeros_like(j)], axis=1)
    c = philox(ctr, (key & 0xFFFFFFFF, key >> 32)) if len(j) else np.zeros((0, 4), np.uint32)
    return (c[:, 0].astype(np.uint64) << np.uint64(32)) | c[:, 1].astype(np.uint64)


def subsample(n_points, num_samples, seed, b, eligible=None):
    """Cloud::subsample of cloud b with n_points points (gpd_b200_depth.h 5): ascending cloud-local indices."""
    j = np.arange(n_points) if eligible is None else np.flatnonzero(eligible)
    if num_samples == 0 or num_samples >= len(j):
        return j.astype(np.int32)
    keys = sample_keys(seed, b, j)
    order = np.lexsort((j, keys))
    return np.sort(j[order[:num_samples]]).astype(np.int32)


def subsample_batch(offsets, num_samples, seed, src=None, raw_offsets=None, mask=None):
    """subsample() of every cloud of a batch (point offsets [B+1]); with a mask, point g of cloud b is eligible when
    mask[raw_offsets[b] + src[g]] != 0."""
    out = []
    for b in range(len(offsets) - 1):
        o0, o1 = int(offsets[b]), int(offsets[b + 1])
        el = None if mask is None else np.asarray(mask)[int(raw_offsets[b]) + np.asarray(src[o0:o1], np.int64)] != 0
        out.append(subsample(o1 - o0, num_samples, seed, b, el))
    return out


# ---- renderer -----------------------------------------------------------------------------------------------------------

def default_cameras(K, width=120, height=90, f=150.0, scale=0.001, min_depth=0.0, max_depth=float("inf")):
    """K cameras looking at the table scene (at z ~ 0.9 in front of the origin) from different places, none with an
    identity pose."""
    places = [(rot_x(0.04) @ rot_y(-0.03), (0.02, -0.01, 0.0)), (rot_y(-0.25), (0.25, 0.0, 0.03)),
              (rot_x(0.2), (0.0, -0.18, 0.02)), (rot_y(0.22) @ rot_x(-0.05), (-0.2, 0.03, 0.01))]
    return [lib.depth_camera(width, height, f, f * 1.02, (width - 1) / 2 + 0.3, (height - 1) / 2 - 0.2,
                             pose(*places[k % len(places)]), scale, min_depth, max_depth) for k in range(K)]


def render(points, cam, fmt):
    """Z-buffer splat of world points into camera cam: the nearest point per pixel, as uint16 units of depth_scale
    (fmt 0) or float32 metres times 1 / depth_scale (fmt 1); 0 where nothing lands."""
    P = np.array(cam.pose[:], np.float64).reshape(3, 4)
    pc = (np.asarray(points, np.float64) - P[:, 3]) @ P[:, :3]
    z = pc[:, 2]
    ok = z > 1e-3
    u = np.rint(cam.fx * pc[ok, 0] / z[ok] + cam.cx).astype(np.int64)
    v = np.rint(cam.fy * pc[ok, 1] / z[ok] + cam.cy).astype(np.int64)
    z = z[ok]
    inside = (u >= 0) & (u < cam.width) & (v >= 0) & (v < cam.height)
    u, v, z = u[inside], v[inside], z[inside]
    depth = np.full(int(cam.width) * int(cam.height), np.inf)
    np.minimum.at(depth, v * int(cam.width) + u, z)
    hole = ~np.isfinite(depth)
    depth[hole] = 0.0
    units = depth / cam.depth_scale
    img = np.rint(units).astype(np.uint16) if fmt == 0 else units.astype(F32)
    return img.reshape(int(cam.height), int(cam.width))


def render_views(seeds, cams_per_view, fmt, n_points=20000, **cam_kw):
    """One rendered view per seed: a list of (image, camera) per view, cameras_per_view[b] cameras each."""
    views = []
    for seed, K in zip(seeds, cams_per_view):
        pts = scenes.synthetic_raw_scene(seed, n_points=n_points)["xyz"]
        pts = pts[np.all(np.isfinite(pts), axis=1)]
        views.append([(render(pts, c, fmt), c) for c in default_cameras(K, **cam_kw)])
    return views
