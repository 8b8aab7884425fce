"""Seeded INPUT generators for the hot path (host-side, numpy): the tutorial cloud fixture and the
synthetic "cluttered table" clouds of BASELINE.json's configs (SURVEY.md 8(d)).

This is input preparation (what util::Cloud preprocessing produces before the path starts,
candidates_generator.cpp:14-37) — NOT part of the accelerated path and not timed.
Outputs follow the C-ABI of gpdb_set_cloud: xyz float32 [N,3], normals float64 [N,3] (float32
values, as PCL normals are, cloud.cpp:531-532), cam_source int32 [N,K], view_points float64 [K,3].
"""
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DIR = os.path.join(os.path.dirname(_HERE), "tests", "golden")


def voxelize(points, cell=0.003):
    """Cloud::voxelizeCloud (cloud.cpp:286-348): voxel corner min_pt + cell*floor((p-min)/cell),
    one point per occupied voxel, ordered lexicographically by voxel index."""
    pts = np.asarray(points, np.float32)
    mn = pts.min(axis=0)
    vox = np.floor((pts - mn) / np.float32(cell)).astype(np.int64)
    _, first = np.unique(vox, axis=0, return_index=True)
    v = vox[first]
    order = np.lexsort((v[:, 2], v[:, 1], v[:, 0]))
    first = first[order]
    out = (mn + np.float32(cell) * vox[first].astype(np.float32)).astype(np.float32)
    return out, first


def pca_normals(points, radius, view_point, flip_away=False):
    """pcl::NormalEstimation restated loosely (PCA of the r-ball, flipped towards the view
    point); only used to prepare the small tutorial fixture."""
    from scipy.spatial import cKDTree

    pts = np.asarray(points, np.float64)
    tree = cKDTree(pts)
    nn = tree.query_ball_point(pts, radius)
    normals = np.zeros_like(pts)
    for i, idx in enumerate(nn):
        q = pts[idx]
        c = np.cov((q - q.mean(0)).T) if len(idx) >= 3 else np.eye(3)
        w, v = np.linalg.eigh(c)
        n = v[:, 0]
        if np.dot(n, view_point - pts[i]) < 0:
            n = -n
        normals[i] = n
    if flip_away:
        normals = -normals
    return normals.astype(np.float32).astype(np.float64)


def load_pcd_ascii(path):
    """Minimal ASCII PCD reader (x y z [rgb]) for tutorials/*.pcd."""
    with open(path) as f:
        lines = f.read().split("\n")
    k = next(i for i, l in enumerate(lines) if l.startswith("DATA"))
    rows = [l.split()[:3] for l in lines[k + 1:] if l.strip()]
    a = np.array(rows, dtype=np.float64)
    return a[np.isfinite(a).all(axis=1)].astype(np.float32)


def krylon_cloud(pcd_path=None):
    """Config 1/2 cloud: tutorials/krylon.pcd voxelised at 0.003 (2 373 points), normals PCA
    r=0.03 towards camera_position = origin then negated (test_grasp_image.cpp:117-118: the
    object surrounds the origin). Loaded from the committed fixture when present."""
    fx = os.path.join(GOLDEN_DIR, "krylon_voxel.npz")
    if pcd_path is None and os.path.exists(fx):
        d = np.load(fx)
        return {k: d[k] for k in ("xyz", "normals", "cam_source", "view_points")}
    pcd_path = pcd_path or "/root/reference/tutorials/krylon.pcd"
    pts = load_pcd_ascii(pcd_path)
    xyz, _ = voxelize(pts, 0.003)
    vp = np.zeros((1, 3))
    normals = pca_normals(xyz, 0.03, vp[0], flip_away=True)
    return {"xyz": xyz, "normals": normals, "cam_source": np.ones((len(xyz), 1), np.int32), "view_points": vp}


# ------------------------------------------------------------------------------------------------
# synthetic cluttered table (configs 3-5)
# ------------------------------------------------------------------------------------------------
def _lattice_rect(origin, eu, ev, lu, lv, step):
    nu, nv = max(int(lu / step), 1), max(int(lv / step), 1)
    u, v = np.meshgrid(np.arange(nu) * step, np.arange(nv) * step, indexing="ij")
    return origin + u.reshape(-1, 1) * eu + v.reshape(-1, 1) * ev


def _box(rng, cx, cy, z0, step):
    sx, sy, sz = rng.uniform(0.05, 0.25, 3)
    yaw = rng.uniform(0, np.pi)
    ex = np.array([np.cos(yaw), np.sin(yaw), 0.0])
    ey = np.array([-np.sin(yaw), np.cos(yaw), 0.0])
    ez = np.array([0.0, 0.0, -1.0])  # "up" is -z: camera looks along +z, table at larger z
    c = np.array([cx, cy, z0])
    P, Nn = [], []
    faces = [
        (c - ex * sx / 2 - ey * sy / 2 + ez * sz, ex, ey, sx, sy, ez),  # top
        (c - ex * sx / 2 - ey * sy / 2, ex, ez, sx, sz, -ey),
        (c - ex * sx / 2 + ey * sy / 2, ex, ez, sx, sz, ey),
        (c - ex * sx / 2 - ey * sy / 2, ey, ez, sy, sz, -ex),
        (c + ex * sx / 2 - ey * sy / 2, ey, ez, sy, sz, ex),
    ]
    for o, eu, ev, lu, lv, n in faces:
        p = _lattice_rect(o, eu, ev, lu, lv, step)
        P.append(p)
        Nn.append(np.tile(n, (len(p), 1)))
    return np.vstack(P), np.vstack(Nn)


def _cylinder(rng, cx, cy, z0, step):
    r, h = rng.uniform(0.025, 0.09), rng.uniform(0.05, 0.25)
    nth = max(int(2 * np.pi * r / step), 8)
    th = np.arange(nth) * (2 * np.pi / nth)
    zz = np.arange(max(int(h / step), 1)) * step
    T, Z = np.meshgrid(th, zz, indexing="ij")
    side = np.stack([cx + r * np.cos(T), cy + r * np.sin(T), z0 - Z], -1).reshape(-1, 3)
    nside = np.stack([np.cos(T), np.sin(T), np.zeros_like(T)], -1).reshape(-1, 3)
    g = np.arange(-r, r, step)
    X, Y = np.meshgrid(g, g, indexing="ij")
    m = X * X + Y * Y < r * r
    top = np.stack([cx + X[m], cy + Y[m], np.full(m.sum(), z0 - h)], -1)
    ntop = np.tile([0.0, 0.0, -1.0], (len(top), 1))
    return np.vstack([side, top]), np.vstack([nside, ntop])


def _sphere(rng, cx, cy, z0, step):
    r = rng.uniform(0.03, 0.10)
    n = max(int(4 * np.pi * r * r / (step * step)), 16)
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = np.pi * (1 + 5 ** 0.5) * i
    d = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], -1)
    return np.array([cx, cy, z0 - r]) + r * d, d


def _visible(points, cam, ang_res):
    """Hidden-surface culling with a spherical z-buffer seen from `cam`."""
    d = points - cam
    rng_ = np.linalg.norm(d, axis=1)
    az = np.arctan2(d[:, 0], d[:, 2])
    el = np.arcsin(np.clip(d[:, 1] / rng_, -1, 1))
    iu = np.floor(az / ang_res).astype(np.int64)
    iv = np.floor(el / ang_res).astype(np.int64)
    key = (iu - iu.min()) * (iv.max() - iv.min() + 1) + (iv - iv.min())
    order = np.lexsort((rng_, key))
    ks = key[order]
    first = np.ones(len(ks), bool)
    first[1:] = ks[1:] != ks[:-1]
    grp = np.cumsum(first) - 1
    minr = rng_[order][first][grp]
    vis = np.zeros(len(points), bool)
    vis[order] = rng_[order] <= minr + 0.004
    return vis


def synthetic_raw_scene(seed, n_points=300000, two_cameras=False, step=0.002, nan_fraction=0.0, cameras=None,
                        mark_all_cameras=False):
    """RAW (unprocessed) cloud of the same cluttered-table scene family: the hidden-surface-culled noisy surface
    samples BEFORE voxelisation and normal estimation (several points per 3 mm voxel at the default 2 mm
    lattice), i.e. what CandidatesGenerator::preprocessPointCloud receives (candidates_generator.cpp:14-37).
    `n_points` sizes the scene like synthetic_table_scene (the voxelised cloud has roughly that many points);
    `nan_fraction` of the points get a NaN coordinate (depth-camera dropouts, cloud.cpp:154-164); `cameras` and
    `mark_all_cameras` as in synthetic_table_scene."""
    d = synthetic_table_scene(seed, n_points=n_points, two_cameras=two_cameras, step=step, _raw=True, cameras=cameras,
                              mark_all_cameras=mark_all_cameras)
    if nan_fraction > 0:
        rng = np.random.default_rng(seed + 1000)
        bad = rng.random(len(d["xyz"])) < nan_fraction
        d["xyz"][bad, rng.integers(0, 3, int(bad.sum()))] = np.nan
    return d


def synthetic_table_scene(seed, n_points=300000, two_cameras=False, step=0.003, _raw=False, cameras=None,
                          mark_all_cameras=False):
    """Config 3/4/5 cloud: a table plane at z ~ 0.9 m in front of a camera at the origin looking
    along +z, 30-60 boxes / cylinders / spheres (5-25 cm) resting on it, surfaces on a 3 mm
    lattice with sigma = 0.5 mm noise, hidden-surface culled per camera, voxelised at 0.003 and
    cut to exactly n_points. Normals are the analytic surface normals perturbed by ~3 degrees of
    noise (stand-in for PCA r=0.03), flipped towards the seeing camera, stored as float32 values.

    `cameras` ([K, 3] positions, looking along +z from z < 0.9) replaces the default camera set (the origin, plus
    (0.6, 0, 0) with `two_cameras`). cam_source marks the first camera that sees a point, or every camera that sees
    it with `mark_all_cameras`; normals are flipped towards the first one either way.
    """
    rng = np.random.default_rng(seed)
    scale = (n_points / 300000.0) ** 0.5
    tx, ty, tz = 2.0 * scale, 1.5 * scale, 0.9
    if cameras is None:
        cams = [np.zeros(3)] + ([np.array([0.6, 0.0, 0.0])] if two_cameras else [])
    else:
        cams = [np.asarray(c, dtype=np.float64).reshape(3) for c in cameras]
    table = _lattice_rect(np.array([-tx / 2, -ty / 2, tz]), np.array([1.0, 0, 0]), np.array([0, 1.0, 0]), tx, ty, step)
    P, Nn = [table], [np.tile([0.0, 0.0, -1.0], (len(table), 1))]
    n_obj = int(rng.integers(30, 61) * scale * scale) + 1
    for _ in range(n_obj):
        cx, cy = rng.uniform(-tx / 2 + 0.1, tx / 2 - 0.1), rng.uniform(-ty / 2 + 0.1, ty / 2 - 0.1)
        kind = rng.integers(0, 3)
        p, n = (_box, _cylinder, _sphere)[kind](rng, cx, cy, tz, step)
        P.append(p)
        Nn.append(n)
    pts = np.vstack(P)
    nrm = np.vstack(Nn)
    pts = pts + rng.normal(0, 0.0005, pts.shape)
    seen = np.zeros((len(pts), len(cams)), bool)
    for k, cam in enumerate(cams):
        facing = ((cam - pts) * nrm).sum(1) > 0
        seen[:, k] = facing & _visible(pts, cam, 0.6 * step / tz)
    keep = seen.any(1)
    pts, nrm, seen = pts[keep], nrm[keep], seen[keep]
    if _raw:
        order = rng.permutation(len(pts))  # scan order is not voxel order
        pts, seen = pts[order], seen[order]
        firstcam = np.argmax(seen, axis=1)
        cam_source = np.zeros((len(pts), len(cams)), np.int32)
        cam_source[np.arange(len(pts)), firstcam] = 1
        if mark_all_cameras:
            cam_source = seen.astype(np.int32)
        return {"xyz": np.ascontiguousarray(pts.astype(np.float32)), "cam_source": cam_source,
                "view_points": np.array(cams, dtype=np.float64)}
    xyz, first = voxelize(pts.astype(np.float32), step)
    nrm, seen = nrm[first], seen[first]
    if len(xyz) < n_points:
        raise RuntimeError(f"synthetic scene produced only {len(xyz)} < {n_points} points")
    sel = np.sort(rng.choice(len(xyz), n_points, replace=False))
    xyz, nrm, seen = xyz[sel], nrm[sel], seen[sel]
    nrm = nrm + rng.normal(0, 0.05, nrm.shape)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    firstcam = np.argmax(seen, axis=1)
    cam_source = np.zeros((n_points, len(cams)), np.int32)
    cam_source[np.arange(n_points), firstcam] = 1
    if mark_all_cameras:
        cam_source = seen.astype(np.int32)
    vp = np.array(cams, dtype=np.float64)
    to_cam = vp[firstcam] - xyz.astype(np.float64)
    flip = (to_cam * nrm).sum(1) < 0
    nrm[flip] *= -1
    normals = nrm.astype(np.float32).astype(np.float64)
    return {"xyz": np.ascontiguousarray(xyz), "normals": np.ascontiguousarray(normals),
            "cam_source": np.ascontiguousarray(cam_source), "view_points": vp}


def sample_indices(config, n_cloud, n_samples=None):
    """Seeded sample indices of BASELINE.json's configs (SURVEY.md 8(d))."""
    if config == 1:
        return np.random.default_rng(1).choice(n_cloud, n_samples or 500, replace=False).astype(np.int32)
    if config == 2:
        return np.random.default_rng(2).integers(0, n_cloud, n_samples or 10000).astype(np.int32)
    if config == 3:
        return np.random.default_rng(3).choice(n_cloud, n_samples or 100000, replace=False).astype(np.int32)
    if config == 4:
        return np.random.default_rng(4).integers(0, n_cloud, n_samples or 1000000).astype(np.int32)
    if config == 5:
        return np.random.default_rng(5).integers(0, n_cloud, n_samples or 200000).astype(np.int32)
    raise ValueError(config)


def random_lenet_weights(channels, seed=0):
    """Random-init LeNet of the reference's architecture (A14) in the .bin layout, with weight
    scales close to the shipped models' (|w|max ~ 0.17 / 0.10 / 0.045 / 0.24)."""
    rng = np.random.default_rng(seed)
    f = np.float32
    return [
        (rng.standard_normal(20 * channels * 25) * 0.04).astype(f), (rng.standard_normal(20) * 0.1).astype(f),
        (rng.standard_normal(50 * 500) * 0.025).astype(f), (rng.standard_normal(50) * 0.1).astype(f),
        (rng.standard_normal(500 * 7200) * 0.008).astype(f), (rng.standard_normal(500) * 0.1).astype(f),
        (rng.standard_normal(2 * 500) * 0.05).astype(f), (rng.standard_normal(2) * 0.1).astype(f),
    ]


def load_weights_dir(d):
    """Read the reference's raw float32 .bin weight directory (eigen_classifier.cpp:185-205)."""
    names = ["conv1_weights", "conv1_biases", "conv2_weights", "conv2_biases", "ip1_weights", "ip1_biases",
             "ip2_weights", "ip2_biases"]
    return [np.fromfile(os.path.join(d, n + ".bin"), dtype=np.float32) for n in names]


# ---- triangle-mesh scenes (gpdb_render_depth / gpdb_sample_meshes) -------------------------------------------------------

def _outward(v, f, centre):
    """faces f of the convex solid v wound so that (b - a) x (c - a) points away from its centre"""
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    flip = (np.cross(b - a, c - a) * ((a + b + c) / 3 - centre)).sum(1) < 0
    f = f.copy()
    f[flip] = f[flip][:, [0, 2, 1]]
    return f


def _mesh_box(centre, half, yaw):
    s = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64) * half
    c, si = np.cos(yaw), np.sin(yaw)
    R = np.array([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]])
    v = s @ R.T + centre
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for q in quads for t in ((q[0], q[1], q[2]), (q[0], q[2], q[3]))], np.int64)
    return v, _outward(v, f, centre)


def _mesh_cylinder(cx, cy, z0, r, h, n):
    th = np.arange(n) * (2 * np.pi / n)
    ring = np.stack([cx + r * np.cos(th), cy + r * np.sin(th)], 1)
    v = np.vstack([np.column_stack([ring, np.full(n, z0)]), np.column_stack([ring, np.full(n, z0 - h)]),
                   [[cx, cy, z0], [cx, cy, z0 - h]]])
    i, j = np.arange(n), (np.arange(n) + 1) % n
    f = np.vstack([np.stack([i, j, n + j], 1), np.stack([i, n + j, n + i], 1),
                   np.stack([np.full(n, 2 * n), j, i], 1), np.stack([np.full(n, 2 * n + 1), n + i, n + j], 1)])
    return v, _outward(v, f, np.array([cx, cy, z0 - h / 2]))


def _mesh_sphere(centre, r, n):
    nu, nv = 2 * n, n
    ph = np.arange(1, nv) * (np.pi / nv)
    th = np.arange(nu) * (2 * np.pi / nu)
    P, T = np.meshgrid(ph, th, indexing="ij")
    ring = np.stack([np.sin(P) * np.cos(T), np.sin(P) * np.sin(T), np.cos(P)], -1).reshape(-1, 3)
    v = centre + r * np.vstack([ring, [[0, 0, 1.0], [0, 0, -1.0]]])
    top, bot = len(ring), len(ring) + 1
    f = []
    for a in range(nv - 1):
        for k in range(nu):
            p, q = a * nu + k, a * nu + (k + 1) % nu
            if a == 0:
                f.append((top, p, q))
            if a == nv - 2:
                f.append((bot, q, p))
            else:
                f.append((p, p + nu, q + nu))
                f.append((p, q + nu, q))
    return v, _outward(v, np.array(f, np.int64), centre)


def mesh_table_scene(seed, n_objects=8, segments=24, table=(0.6, 0.45), tz=0.9):
    """A seeded tabletop of triangle meshes in the frame of synthetic_table_scene (up is -z, the table top at z = tz,
    cameras near the origin looking along +z): a 3 cm table slab plus n_objects closed, outward-wound boxes, cylinders
    and UV spheres resting on it, 3-8 cm across, so the default hand (aperture up to 8.5 cm) fits most of them.
    `segments` sets the tessellation (cylinder sides, sphere rings), the knob of the face count. Returns (vertices [V, 3]
    float32, faces [F, 3] int32, object_id [F] int32: 0 for the table, 1..n_objects for the objects)."""
    rng = np.random.default_rng(seed)
    tx, ty = table
    parts = [_mesh_box(np.array([0.0, 0.0, tz + 0.015]), np.array([tx / 2, ty / 2, 0.015]), 0.0)]
    for _ in range(n_objects):
        cx, cy = rng.uniform(-tx / 2 + 0.06, tx / 2 - 0.06), rng.uniform(-ty / 2 + 0.06, ty / 2 - 0.06)
        kind = rng.integers(0, 3)
        if kind == 0:
            half = np.array([rng.uniform(0.015, 0.04), rng.uniform(0.015, 0.04), rng.uniform(0.02, 0.07)])
            parts.append(_mesh_box(np.array([cx, cy, tz - half[2]]), half, rng.uniform(0, np.pi)))
        elif kind == 1:
            parts.append(_mesh_cylinder(cx, cy, tz, rng.uniform(0.015, 0.035), rng.uniform(0.04, 0.14), 2 * segments))
        else:
            r = rng.uniform(0.02, 0.04)
            parts.append(_mesh_sphere(np.array([cx, cy, tz - r]), r, segments))
    V, Fs, ids, base = [], [], [], 0
    for k, (v, f) in enumerate(parts):
        V.append(v)
        Fs.append(f + base)
        ids.append(np.full(len(f), k, np.int32))
        base += len(v)
    return (np.ascontiguousarray(np.vstack(V).astype(np.float32)), np.ascontiguousarray(np.vstack(Fs).astype(np.int32)),
            np.concatenate(ids))
