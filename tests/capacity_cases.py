"""Inputs that put an exact number of points into the fixed-size neighbourhood lists of the geometry kernels
(test_gpu_capacity_edges.py on the device, test_capacity_cases.py on the CPU), so that each list is filled to its
capacity and one point past it.

Every coordinate is a multiple of a power of two (2^-14 for the small balls, 2^-12 for the image boxes) and lies within
1 m of the origin: every float32 difference, square and sum of squares between two points is exact, so the float32 ball
count of numpy with FLANN's predicate (dx^2 + dy^2 + dz^2 < float32(r^2)) is the kernels' count, whatever the order of
the additions. The counted neighbourhood is an isolated object; the rest of the cloud (a sparse plane) lies beyond every
search radius of it.
"""
import numpy as np

from gpd_b200 import abi

# list capacities, as the kernels define them (gpd_b200/csrc/geometry.cu, by symbol)
FRAMES_CAP0 = 128          # launch_frames: cap0, tier 0 of k_frames
FRAMES_CAP1 = 1024         # LRF_CAP: tier 1 (shared memory)
FRAMES_CAP2 = 16384        # LRF_CAP_GLOBAL: tier 2 (global memory); beyond: GPDB_ERR_CAPACITY
HANDS_CAP1 = 2176          # HANDS_CAP1: first k_hands tier
HANDS_CAP2 = 12800         # HANDS_CAP2: the large shared-memory tile
HANDS_CAP3 = 131072        # HANDS_CAP3: global-memory tier; beyond: GPDB_ERR_CAPACITY
SURV_CAP = 1024            # SURV_CAP: closing-region members remembered per warp
IMG2_S = 60                # IMG2_S: the only image size of k_images2
BOX_CAP2 = 1024            # BOX_CAP2: k_images2's box list; beyond: the image is redone by k_images
BALL_CAP2 = (IMG2_S * IMG2_S * 16 - 12 * IMG2_S * IMG2_S) // 4  # BALL_CAP2: in-ball list of k_images2 (3 600)
BOX_CAP = 2048             # BOX_CAP: k_images' shared-memory box list; beyond: its global-memory instance
BOX_CAP_GL = 32768         # launch_images: gl_cap; beyond: GPDB_ERR_CAPACITY
WL_CAP2 = (IMG2_S * IMG2_S * 8) // 20   # k_images2: WL_CAP, the shadow work list (1 440)
WL_CAP = (2 * IMG2_S * IMG2_S * 8) // 20  # k_images: WL_CAP, the shadow work list (2 880)
DL_CAP = 2 * IMG2_S * IMG2_S            # CastLists::dl_cap, the draw list of either kernel (7 200)


def st_sm2(bm_dim, n_cameras):
    """The shared-memory part of k_images2's voxel stash (ST_SM): what LIST_BYTES (BOX_CAP2 x 36 B) leaves behind the
    cameras' shadow bitmaps (2 bm_dim^2 words each) and one word of alignment, in 8-byte entries."""
    bm_words = 2 * bm_dim * bm_dim
    used = ((bm_words * max(n_cameras, 1) + 1) & ~1) * 4
    return (BOX_CAP2 * 36 - used) // 8


def st_cap2(bm_dim, n_cameras):
    """k_images2's voxel stash (ST_CAP): ST_SM entries in shared memory, then BALL_CAP2 / 2 more in the image's own
    HBM slot over the in-ball list; past it the voxels of projection 2 take a second walk over the bitmap."""
    return st_sm2(bm_dim, n_cameras) + BALL_CAP2 // 2


BOX_CAP2_BYTES = BOX_CAP2 * 36   # k_images2's LIST_BYTES


def list_bytes(bm_dim, n_cameras):
    """launch_images: k_images' box-list region at 15 channels, which the shadow bitmaps and the voxel list alias."""
    bm = n_cameras * (2 * bm_dim * bm_dim) * 4
    return (max(BOX_CAP * 36, bm + 4096 * 4) + 15) // 16 * 16


def bl_cap(bm_dim, n_cameras):
    """k_images' voxel list (BL_CAP): the 4-byte entries of list_bytes behind bitmap 0."""
    return list_bytes(bm_dim, n_cameras) // 4 - 2 * bm_dim * bm_dim


def fast_path_15(bm_dim, n_cameras):
    """launch_images: whether a 15-channel image of size 60 goes to k_images2, whose shadow bitmaps must leave 2 KB of
    its list free."""
    return n_cameras <= 2 and n_cameras * (2 * bm_dim * bm_dim) * 4 + 2048 <= BOX_CAP2_BYTES


def bm_dim(volume_width=0.10, volume_depth=0.06, volume_height=0.02):
    """api.cu fill_dev_params: the shadow bitmap's extent in voxels."""
    import math
    diag = math.sqrt(volume_depth * volume_depth + volume_width * volume_width + 4.0 * volume_height * volume_height)
    return int(math.ceil((diag + 2.0 * 3.2 * 0.003 * 0.3) / 0.003)) + 4


# search radii at the default hand and image geometry (api.cu fill_dev_params)
R_LRF = 0.01   # nn_radius
R_HS = 0.11    # max(hand_outer_diameter - finger_width, hand_depth, hand_height / 2)
R_IMG = 0.10   # max(volume_depth, volume_height / 2, volume_width)


def ball_count(xyz, q, r):
    """Points of xyz in the r-ball of q by FLANN's float32 predicate (L2_Simple, then < float32(r^2))."""
    d = np.asarray(q, np.float32)[None] - np.asarray(xyz, np.float32)
    dist = d[:, 0] * d[:, 0]
    dist = dist + d[:, 1] * d[:, 1]
    dist = dist + d[:, 2] * d[:, 2]
    return int(np.count_nonzero(dist < np.float32(r * r)))


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _tilted_normals(n, rng, spread=0.3):
    return _unit(np.array([0.0, 0.0, 1.0]) + spread * rng.standard_normal((n, 3)))


def _plane(z, q, rng):
    """The rest of the cloud: 20 x 20 points at about 3 mm on the plane at height z, x in [0.3, 0.36]."""
    k = np.stack(np.meshgrid(np.arange(20), np.arange(20), indexing="ij"), -1).reshape(-1, 2) * round(0.003 / q)
    xyz = np.zeros((len(k), 3))
    xyz[:, 0] = 0.3 + k[:, 0] * q
    xyz[:, 1] = k[:, 1] * q
    xyz[:, 2] = z
    return xyz.astype(np.float32), _tilted_normals(len(k), rng)


def _distinct_offsets(n, lim, rng, keep):
    """n distinct integer offsets in [-lim, lim]^3 that satisfy keep(k) (float64 array [m, 3] -> bool [m])."""
    out = np.zeros((0, 3), np.int64)
    while len(out) < n:
        k = rng.integers(-lim, lim + 1, (max(4 * (n - len(out)), 1024), 3))
        k = k[keep(k.astype(np.float64))]
        out = np.unique(np.concatenate([out, k]), axis=0)
    return out[rng.permutation(len(out))[:n]]


def frames_ball(n, at_position=False, seed=0):
    """A cloud whose sample has exactly n points in its r = nn_radius ball: the sample point itself (unless at_position)
    and n - 1 (n) distinct lattice points within 0.9 r of it, behind a shell of 300 points between 1.01 r and 1.2 r.
    Returns (cloud dict, sample index or None, sample position [3] float64, indices of a few plane samples)."""
    q = 2.0 ** -14
    rng = np.random.default_rng(seed)
    c = np.array([0.0, 0.0, 0.5])
    rq = R_LRF / q
    inner = _distinct_offsets(n if at_position else n - 1, int(0.9 * rq), rng,
                              lambda k: ((k * k).sum(1) <= (0.9 * rq) ** 2) & (k != 0).any(1))
    shell = _distinct_offsets(300, int(1.2 * rq), rng,
                              lambda k: ((k * k).sum(1) >= (1.01 * rq) ** 2) & ((k * k).sum(1) <= (1.2 * rq) ** 2))
    ks = inner if at_position else np.vstack([np.zeros((1, 3), np.int64), inner])
    obj = (c + np.vstack([ks, shell]) * q).astype(np.float32)
    bg, bgn = _plane(0.5, q, rng)
    xyz = np.vstack([obj, bg])
    nrm = np.vstack([_tilted_normals(len(obj), rng), bgn])
    cloud = {"xyz": xyz, "normals": nrm, "cam_source": np.ones((len(xyz), 1), np.int32), "view_points": np.zeros((1, 3))}
    plane_samples = np.arange(len(obj), len(xyz), 37, dtype=np.int32)
    return cloud, (None if at_position else 0), c.copy(), plane_samples


def hand_cylinder(n, seed=0):
    """A cloud whose sample has exactly n points in its hand-search ball (r = 0.11) and in its hand-height slab: a 5 cm
    cylinder along y (|y| <= 12 mm) of n distinct lattice points with radial normals, the sample at the point facing the
    camera (-z). Every normal lies in the x-z plane, so the curvature axis of the sample's frame is y and the slab of
    hand_axes = [2] (|z| < hand_height along it) holds the whole cylinder. The hand closes across it. The plane is more
    than 0.2 m away. Returns (cloud dict, sample index)."""
    q = 2.0 ** -14
    rng = np.random.default_rng(seed)
    c = np.array([0.0, 0.0, 0.5])
    rad, half = 0.025, 0.012
    ks = [np.round(np.array([0.0, 0.0, -rad]) / q).astype(np.int64)[None]]
    nr = [np.array([[0.0, 0.0, -1.0]])]
    have = {tuple(ks[0][0])}
    while len(have) < n:
        m = 2 * (n - len(have)) + 64
        th = rng.uniform(0, 2 * np.pi, m)
        y = rng.uniform(-half, half, m)
        k = np.round(np.stack([rad * np.cos(th), y, rad * np.sin(th)], 1) / q).astype(np.int64)
        sel = []
        for i in range(m):
            t = tuple(k[i])
            if t not in have and len(have) < n:
                have.add(t)
                sel.append(i)
        ks.append(k[sel])
        nr.append(np.stack([np.cos(th[sel]), np.zeros(len(sel)), np.sin(th[sel])], 1))
    obj = (c + np.vstack(ks) * q).astype(np.float32)
    bg, bgn = _plane(0.75, q, rng)
    xyz = np.vstack([obj, bg])
    nrm = np.vstack([_unit(np.vstack(nr)), bgn])
    cloud = {"xyz": xyz, "normals": nrm, "cam_source": np.ones((len(xyz), 1), np.int32), "view_points": np.zeros((1, 3))}
    return cloud, 0


def slab_count(cloud, sample_idx, frame, hand_height=0.02, r=R_HS):
    """Points k_hands stages for hand_axes = [2]: in the float32 r-ball of the sample and inside the widened hand-height
    slab, z0 = T[6] dx + T[7] dy + T[8] dz (float64, the kernel's order) with T = frame x rot_binormal, |z0| < hz."""
    xyz = np.asarray(cloud["xyz"], np.float32)
    s = xyz[sample_idx].astype(np.float64)
    d = np.asarray(s, np.float32)[None] - xyz
    dist = d[:, 0] * d[:, 0]
    dist = dist + d[:, 1] * d[:, 1]
    dist = dist + d[:, 2] * d[:, 2]
    inb = dist < np.float32(r * r)
    # frame: column-major 3 x 3 (normal, binormal, curvature axis); rot_binormal = rotation by pi about y
    F = np.asarray(frame, np.float64).reshape(3, 3).T
    cp, sp = np.cos(np.pi), np.sin(np.pi)
    rotb = np.array([[cp, 0.0, sp], [0.0, 1.0, 0.0], [-sp, 0.0, cp]])
    T = (F @ rotb).T.ravel()  # column-major again: T[6..8] = third column
    p = xyz.astype(np.float64) - s
    z0 = (T[6] * p[:, 0] + T[7] * p[:, 1]) + T[8] * p[:, 2]
    hz = hand_height * 1.001 + 1e-9
    return int(np.count_nonzero(inb & (np.abs(z0) < hz)))


def closing_counts(cloud, sample_idx, poses, flags, hand_height=0.02, fw=0.01, od=0.12, nfp=10, r=R_HS):
    """Closing-region members of each valid pose (what k_hands remembers per warp, SURV_CAP): staged points with
    |z| < hand_height, bottom < x < top and left < y < right in the pose's frame, in float64 in the kernel's operation
    order (to_frame of p - sample). left = fsw[f], right = fs[nfp + f] of the pose's finger placement f, as
    api.cu fill_dev_params builds the slot tables (deepen_hand on: finger_idx is f). Every point of these cases is
    staged (ball and slab), so the staged list is the ball. -1: pose not valid."""
    xyz = np.asarray(cloud["xyz"], np.float32)
    s = xyz[sample_idx].astype(np.float64)
    step = (od - fw) / (nfp - 1)
    d = np.asarray(s, np.float32)[None] - xyz
    dist = d[:, 0] * d[:, 0]
    dist = dist + d[:, 1] * d[:, 1]
    dist = dist + d[:, 2] * d[:, 2]
    p = xyz[dist < np.float32(r * r)].astype(np.float64) - s
    out = np.full(len(poses), -1)
    for k, (h, f) in enumerate(zip(poses, flags)):
        if not f & 1:
            continue
        R = h["frame"]
        x = (R[0] * p[:, 0] + R[1] * p[:, 1]) + R[2] * p[:, 2]
        y = (R[3] * p[:, 0] + R[4] * p[:, 1]) + R[5] * p[:, 2]
        z = (R[6] * p[:, 0] + R[7] * p[:, 1]) + R[8] * p[:, 2]
        f_ = int(h["finger_idx"])
        right = (od - fw) if f_ == nfp - 1 else 0.0 + f_ * step  # linspaced(nfp, 0, od - fw, f)
        left = ((right - od) + fw) + fw
        assert h["center"] == 0.5 * (left + right)
        out[k] = np.count_nonzero((z > -1.0 * hand_height) & (z < hand_height) & (x > h["bottom"]) & (x < h["top"]) &
                                  (y > left) & (y < right))
    return out


def image_box(n_box, n_outside=0, seed=0):
    """Points for one hand-built candidate: n_box distinct lattice points inside its image box and n_outside more in
    its image ball but outside the box, on the camera side (nearer the camera at the origin). The candidate: sample
    (0, 0, 0.5), identity frame, bottom 0, center 0: the box is x in (0, 0.06), |y| < 0.05, |z - 0.5| < 0.02.
    Returns (cloud dict, poses [1] POSE_DTYPE)."""
    q = 2.0 ** -12
    rng = np.random.default_rng(seed)
    s = np.array([0.0, 0.0, 0.5])

    def box(lo, hi, n):
        lo_k, hi_k = np.ceil(np.array(lo) / q).astype(np.int64), np.floor(np.array(hi) / q).astype(np.int64)
        out = np.zeros((0, 3), np.int64)
        while len(out) < n:
            k = rng.integers(lo_k, hi_k + 1, (2 * (n - len(out)) + 64, 3))
            out = np.unique(np.concatenate([out, k]), axis=0)
        return out[rng.permutation(len(out))[:n]]

    kin = box([0.002, -0.048, -0.018], [0.058, 0.048, 0.018], n_box)
    kout = box([0.002, -0.04, -0.06], [0.05, 0.04, -0.025], n_outside)
    obj = (s + np.vstack([kin, kout]) * q).astype(np.float32)
    bg, bgn = _plane(0.65, q, rng)
    xyz = np.vstack([obj, bg])
    nrm = np.vstack([_unit(rng.standard_normal((len(obj), 3))), bgn])
    cloud = {"xyz": xyz, "normals": nrm, "cam_source": np.ones((len(xyz), 1), np.int32), "view_points": np.zeros((1, 3))}
    pose = np.zeros(1, dtype=abi.POSE_DTYPE)
    pose["sample"][0] = s
    pose["frame"][0] = np.eye(3).ravel()
    pose["bottom"], pose["top"], pose["center"] = 0.0, 0.06, 0.0
    pose["sample_index"] = 0
    pose["finger_idx"] = 4
    pose["score"] = np.nan
    return cloud, pose


def box_count(cloud, pose, vol_w=0.10, vol_d=0.06, vol_h=0.02, r=R_IMG):
    """Points in the candidate's image box (in_image_box in float64, the kernels' order) among those of its float32
    image ball."""
    h = pose[0]
    xyz = np.asarray(cloud["xyz"], np.float32)
    sf = h["sample"].astype(np.float32)
    d = sf[None] - xyz
    dist = d[:, 0] * d[:, 0]
    dist = dist + d[:, 1] * d[:, 1]
    dist = dist + d[:, 2] * d[:, 2]
    inb = dist < np.float32(r * r)
    R = h["frame"]
    p = xyz.astype(np.float64) - h["sample"]
    x = (R[0] * p[:, 0] + R[1] * p[:, 1]) + R[2] * p[:, 2]
    y = (R[3] * p[:, 0] + R[4] * p[:, 1]) + R[5] * p[:, 2]
    z = (R[6] * p[:, 0] + R[7] * p[:, 1]) + R[8] * p[:, 2]
    half = vol_w / 2.0
    box = (x > h["bottom"]) & (x < h["bottom"] + vol_d) & (y > h["center"] - half) & (y < h["center"] + half) & \
        (z > -1.0 * vol_h) & (z < vol_h)
    return int(np.count_nonzero(inb & box))
