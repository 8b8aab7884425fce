"""Hand-built candidates for gpdb_images that reach the edges of the image stage's output (test_image_cases.py proves the
reach on the CPU from the restatement's intermediates, test_gpu_image_output_stage.py checks the kernels pixel for pixel):
covered projections (no all-empty 3 x 3 window: the general min path) at each kernel tier, marginal coverage at the image
border and where a row straddles three occupancy words, constant groups (Quant's DBL_EPSILON branch), points on and 1 ulp
either side of cell boundaries and box faces, stacks of 1 to 200 points in one cell, image sizes 8 to 64, 1 to 15
channels, covered shadow channels and non-unit normals.

Each candidate is an isolated object around its own sample (objects 0.25 m apart, beyond every image ball) with a
caller-made pose: an exact permutation frame and a set sample_index. The points are placed in hand coordinates, so
every case states which cells it fills. The rest of the cloud is a sparse plane beyond the image balls."""
import numpy as np

import capacity_cases as cc
from gpd_b200 import abi
from image_reference import Geometry, unit_cells

DEFAULT = dict(S=60, w=0.10, d=0.06, h=0.02)
DYADIC = dict(S=32, w=0.125, d=0.0625, h=0.03125)   # every cell boundary is an exact float32
# permutation frames (rows: the hand axes in world coordinates): identity and the two cyclic rotations
FRAMES = [np.eye(3), np.array([[0.0, 1, 0], [0, 0, 1], [1, 0, 0]]), np.array([[0.0, 0, 1], [1, 0, 0], [0, 1, 0]])]
PROJ = [(0, 1, 2), (2, 1, 0), (2, 0, 1)]


class Builder:
    """Objects one per pose: add() takes hand-frame points and normals and returns the pose."""

    def __init__(self, g, seed=0):
        self.g = g
        self.rng = np.random.default_rng(seed)
        self.xyz, self.nrm, self.poses, self.claims = [], [], [], []

    def origin(self):
        k = len(self.poses)
        return np.array([0.25 * (k % 12), 0.25 * (k // 12), 0.5])

    def pose(self, sample, frame=0, bottom=0.0, center=0.0):
        p = np.zeros(1, dtype=abi.POSE_DTYPE)
        p["sample"][0] = sample
        p["frame"][0] = FRAMES[frame].ravel()
        p["bottom"], p["top"], p["center"] = bottom, bottom + self.g.d, center
        p["sample_index"] = 1000 + len(self.poses)
        p["finger_idx"] = 4
        p["score"] = np.nan
        return p

    def add(self, hand_pts, normals_hand, claims, frame=0, pose=None, world=None):
        pose = self.pose(self.origin(), frame) if pose is None else pose
        Fm = np.asarray(pose["frame"][0], np.float64).reshape(3, 3)
        if world is None:
            world = (pose["sample"][0][None] + np.asarray(hand_pts, np.float64) @ Fm).astype(np.float32)
        self.xyz.append(np.asarray(world, np.float32))
        self.nrm.append(np.asarray(normals_hand, np.float64) @ Fm)
        self.poses.append(pose)
        self.claims.append(claims)
        return pose

    def cells_to_hand(self, cells, frac=None, pose=None):
        g = self.g
        frac = self.rng.uniform(0.25, 0.75, np.shape(cells)) if frac is None else frac
        b, c = (0.0, 0.0) if pose is None else (float(pose["bottom"][0]), float(pose["center"][0]))
        lo = np.array([b, c - g.w / 2.0, -g.h])
        ext = np.array([g.d, g.w, 2.0 * g.h])
        return lo + (np.asarray(cells, np.float64) + frac) * ext / g.S

    def tilted(self, n):
        return cc._unit(np.array([0.55, 0.5, 0.6]) + 0.15 * self.rng.uniform(-1, 1, (n, 3)))

    def cloud(self, K=1, view_points=None):
        bg, bgn = cc._plane(-0.5, 2.0 ** -12, self.rng)
        xyz = np.vstack(self.xyz + [bg])
        nrm = np.vstack(self.nrm + [bgn])
        vp = np.zeros((1, 3)) if view_points is None else np.asarray(view_points, np.float64)
        return {"xyz": xyz, "normals": nrm, "cam_source": np.ones((len(xyz), len(vp)), np.int32), "view_points": vp}

    def case(self, name, **cloud_kw):
        return {"name": name, "geometry": self.g, "cloud": self.cloud(**cloud_kw), "poses": np.concatenate(self.poses),
                "claims": self.claims}


def lattice(S, step, a0, a1, depth_cells, rng, skip=()):
    """Cells [n, 3] of a lattice every `step` cells of rows (axis a0) and columns (axis a1), offset so that every clipped
    3 x 3 window of the projection holds a lattice cell; depth cells (axis a2) drawn from depth_cells. `skip`: (r, c)
    cells of the projection plane left out (image rows: r is S - 1 - cell of a0)."""
    off = 1 if step == 3 else 0
    ks = np.arange(off, S, step)
    if step == 3 and ks[-1] < S - 2:
        ks = np.append(ks, S - 1)
    rr, cc_ = np.meshgrid(ks, ks, indexing="ij")
    rr, cc_ = rr.ravel(), cc_.ravel()
    keep = np.array([(S - 1 - r, c) not in skip for r, c in zip(rr, cc_)], bool)
    rr, cc_ = rr[keep], cc_[keep]
    a2 = 3 - a0 - a1
    cells = np.zeros((len(rr), 3), np.int64)
    cells[:, a0], cells[:, a1], cells[:, a2] = rr, cc_, rng.choice(depth_cells, len(rr))
    return cells


def dense(S, a0, a1, rng, empty=()):
    """Every cell of the projection plane (one point each) except the image cells (row, col) in `empty`."""
    a2 = 3 - a0 - a1
    rows, cols = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    rows, cols = rows.ravel(), cols.ravel()
    keep = np.array([(r, c) not in empty for r, c in zip(rows, cols)], bool)
    cells = np.zeros((int(keep.sum()), 3), np.int64)
    cells[:, a0], cells[:, a1] = S - 1 - rows[keep], cols[keep]
    cells[:, a2] = rng.integers(2, S - 2, len(cells))
    return cells


def patch(r0, r1, c0, c1):
    return {(r, c) for r in range(r0, r1 + 1) for c in range(c0, c1 + 1)}


def _covered_claims(pj, tier, covered=True, extra=None):
    cl = {"tier": tier, "covered": {(pj, "n"): covered, (pj, "d"): covered}}
    if covered:
        cl["min_positive"] = [(pj, "n"), (pj, "d")]
    cl.update(extra or {})
    return cl


def covered_cases():
    """Projection pj's poses use frame pj. The covered projections at each tier (every 3rd cell: k_images2; every 2nd cell, some cells twice: k_images'
    shared list; every cell: its global list), once per projection, with one cell emptied of every lattice as the
    uncovered twin (k_images2 and shared list)."""
    g = Geometry(C=12, **DEFAULT)
    b = Builder(g, seed=1)
    S = g.S
    for pj in range(3):
        a0, a1, _ = PROJ[pj]
        for step, tier in ((3, "images2"), (2, "shared"), (1, "gl")):
            for hole in ((False, True) if step > 1 else (False,)):
                skip = {(S - 1 - (31 if step == 3 else 30), 31 if step == 3 else 30)} if hole else set()
                cells = lattice(S, step, a0, a1, np.arange(3, S - 3), b.rng, skip) if step > 1 else dense(S, a0, a1, b.rng)
                if step == 2:   # every other lattice cell holds a second point: 1 025 - 2 048 box points
                    cells = np.vstack([cells, cells[::2] + np.eye(3, dtype=np.int64)[3 - a0 - a1]])
                b.add(b.cells_to_hand(cells), b.tilted(len(cells)), _covered_claims(pj, tier, covered=not hole), frame=pj)
    return b.case("covered")


# image cells emptied in the dense lattice of projection 0 (an empty 3 x 3 window: not covered; a thinner patch: covered)
HOLES = {
    "interior_3x3": (patch(29, 31, 29, 31), False), "interior_2x3": (patch(29, 30, 29, 31), True),
    "interior_3x2": (patch(29, 31, 29, 30), True),
    "row0_2x3": (patch(0, 1, 20, 22), False), "row0_1x3": (patch(0, 0, 20, 22), True),
    "rowS1_2x3": (patch(58, 59, 20, 22), False), "rowS1_1x3": (patch(59, 59, 20, 22), True),
    "col0_3x2": (patch(20, 22, 0, 1), False), "col0_3x1": (patch(20, 22, 0, 0), True),
    "colS1_3x2": (patch(20, 22, 58, 59), False), "colS1_3x1": (patch(20, 22, 59, 59), True),
    "corner_2x2": (patch(0, 1, 0, 1), False), "corner_1x2": (patch(0, 0, 0, 1), True),
    # rows 1-3 of a 60-wide bitmap start at bits 28, 24, 20 of their word: their high columns lie in a third word
    "straddle_3x3": (patch(1, 3, 50, 52), False), "straddle_2x3": (patch(1, 2, 50, 52), True),
}


def hole_cases():
    g = Geometry(C=12, **DEFAULT)
    b = Builder(g, seed=2)
    for name, (empty, covered) in HOLES.items():
        cells = dense(g.S, 0, 1, b.rng, empty)
        cl = _covered_claims(0, "gl", covered)
        cl["hole"] = name
        b.add(b.cells_to_hand(cells), b.tilted(len(cells)), cl)
    return b.case("holes")


def constant_cases():
    """A covered plane perpendicular to each projection axis with identical normals: every group constant (the
    DBL_EPSILON branch), and the same plane with one empty 3 x 3 window (min 0, max the constant)."""
    g = Geometry(C=12, **DEFAULT)
    b = Builder(g, seed=3)
    S = g.S
    n = cc._unit(np.ones((1, 3)))
    for pj in range(3):
        a0, a1, a2 = PROJ[pj]
        for hole in (False, True):
            cells = lattice(S, 3, a0, a1, [S // 2], b.rng, {(S - 1 - 31, 31)} if hole else set())
            frac = np.full(cells.shape, 0.5)
            grp = [(pj, "n"), (pj, "d")]
            cl = {"tier": "images2", "covered": {k: not hole for k in grp}}
            cl["constant" if not hole else "min_zero_max_constant"] = grp
            b.add(b.cells_to_hand(cells, frac), np.repeat(n, len(cells), 0), cl, frame=pj)
    return b.case("constant")


def stack_cases():
    """Stacks of 1, 63, 64, 65 and 200 points with distinct depths in single cells of projection 0 (the reciprocal
    table of cell_mean ends at 64), isolated 6 cells apart, at both geometries."""
    out = []
    for geo, seed in ((DEFAULT, 4), (DYADIC, 5)):
        g = Geometry(C=12, **geo)
        b = Builder(g, seed=seed)
        pts = []
        for i, n in enumerate((1, 2, 63, 64, 65, 200)):
            c0, c1 = 2 + 5 * i, 3 + 5 * i
            z = np.linspace(0.05, 0.95, n) * 2 * g.h - g.h
            h = b.cells_to_hand(np.tile([[c0, c1, 0]], (n, 1)), np.tile([[0.4, 0.6, 0.0]], (n, 1)))
            h[:, 2] = z
            pts.append(h)
        pts = np.vstack(pts)
        b.add(pts, b.tilted(len(pts)), {"tier": "images2" if g.S == 60 else "shared",
                                        "stack_counts": [1, 2, 63, 64, 65, 200]})
        out.append(b.case(f"stacks_S{g.S}"))
    return out


def size_cases():
    """Image sizes 8, 57, 64 (12 channels; 64 takes fully_covered's full-word mask) and the dyadic geometry at 32, and 1,
    3, 15 channels at size 60: a covered projection 0 and its uncovered twin each."""
    out = []
    for geo, C in ((dict(DEFAULT, S=8), 12), (dict(DEFAULT, S=57), 12), (dict(DEFAULT, S=64), 12), (DYADIC, 12),
                   (DEFAULT, 1), (DEFAULT, 3), (DEFAULT, 15)):
        g = Geometry(C=C, **geo)
        b = Builder(g, seed=6 + C + g.S)
        S = g.S
        grp = [(0, k) for k in (("n", "d") if C >= 12 else ("d",) if C == 1 else ("n",))]
        tier = "images2" if S == 60 else "shared"
        for hole in (False, True):
            cells = lattice(S, 3 if S > 8 else 1, 0, 1, np.arange(1, S - 1), b.rng,
                            {(S - 1 - 31, 31)} if hole and S > 8 else set())
            if hole and S == 8:
                cells = cells[~((cells[:, 0] >= 3) & (cells[:, 0] <= 5) & (cells[:, 1] >= 3) & (cells[:, 1] <= 5))]
            cl = {"tier": tier, "covered": {k: not hole for k in grp}}
            if not hole:
                cl["min_positive"] = grp
            b.add(b.cells_to_hand(cells), b.tilted(len(cells)), cl)
        out.append(b.case(f"size_S{S}_C{C}" + ("_dyadic" if geo is DYADIC else "")))
    return out


def shadow_cases():
    """15 channels: a dense plane 1 cm in front of the box (between the box and the camera) whose shadow fills the box,
    so that the shadow channels take the covered path; one camera, and two cameras at volume_depth 0.05 (k_images2)."""
    out = []
    for K, geo in ((1, DEFAULT), (2, dict(DEFAULT, d=0.05))):
        g = Geometry(C=15, **geo)
        b = Builder(g, seed=20 + K)
        q = 2.0 ** -9
        xs = np.arange(-0.004, g.d + 0.004, q)
        ys = np.arange(-g.w / 2 - 0.004, g.w / 2 + 0.004, q)
        X, Y = np.meshgrid(xs, ys, indexing="ij")
        pts = np.stack([X.ravel(), Y.ravel(), np.full(X.size, -g.h - 0.0078125)], 1)
        pose = b.pose(np.array([0.0, 0.0, 0.5]))
        b.add(pts, b.tilted(len(pts)), {"tier": "images2", "shadow_covered": True}, pose=pose)
        vp = [[0.0, 0.0, 0.0]] if K == 1 else [[0.0, 0.0, 0.0], [0.02, 0.0, 0.0]]
        out.append(b.case(f"shadow_K{K}", view_points=vp))
    return out


def nonunit_cases():
    """Normals of other than unit length: a covered k_images2-size lattice with two points in every other cell (the
    exact fold, run by k_images), the same at the global-list tier, and normals of length 1e-40 (a group whose max -
    min is positive but below DBL_EPSILON)."""
    g = Geometry(C=12, **DEFAULT)
    b = Builder(g, seed=30)
    S = g.S
    cells = lattice(S, 3, 0, 1, np.arange(3, S - 3), b.rng)
    cells = np.vstack([cells, cells[::2] + np.array([0, 0, 1])])
    n = b.tilted(len(cells)) * b.rng.uniform(0.3, 1.7, (len(cells), 1))
    b.add(b.cells_to_hand(cells), n, {"tier": "images2", "nonunit": True, "covered": {(0, "n"): True, (0, "d"): True},
                                     "min_positive": [(0, "n"), (0, "d")]})
    cells = dense(S, 0, 1, b.rng)
    n = b.tilted(len(cells)) * b.rng.uniform(0.3, 1.7, (len(cells), 1))
    b.add(b.cells_to_hand(cells), n, {"tier": "gl", "nonunit": True, "covered": {(0, "n"): True, (0, "d"): True}})
    cells = lattice(S, 3, 0, 1, np.arange(3, S - 3), b.rng, {(28, 31)})
    n = np.abs(b.rng.uniform(1e-40, 2e-40, (len(cells), 3)))
    b.add(b.cells_to_hand(cells), n, {"tier": "images2", "nonunit": True, "tiny": [(0, "n")]})
    return b.case("nonunit")


# ---------------------------------------------------------------------------------------------------- boundaries

def _f32_step(v, k):
    v = np.float32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf))
    return v


def _kernel_cells(g, pose, hand, fault=None):
    u, cell = unit_cells(g, pose[0], np.asarray(hand, np.float64)[None], "kernel", fault)
    return u[0], cell[0]


def boundary_cases(geo=DEFAULT, seed=40):
    """Isolated points (plus one anchor point 10 cells away) on cell boundaries and box faces. Each pose is tuned (its
    bottom along x, its center along y, its sample along z) so that the boundary lies exactly on a float32 world
    coordinate v; the points sit at v and 1 ulp either side. Where the reciprocal product alone (no exact-division
    fallback) gives another cell than unit_axis, a further pose stepped from such a tuning holds the point ("fault_e").
    Faces: the point on the face (excluded) and 1 ulp inside; the z faces with the point a few cm from the origin,
    where the sample at exactly volume_height from it is a float64. Below the upper x face: poses whose bottom is negative, so
    that x - bottom rounds up to volume_depth for a point strictly inside the box (u = 1: the fixed-point coordinate
    saturates, the cell clamps to S - 1)."""
    g = Geometry(C=12, **geo)
    b = Builder(g, seed=seed)
    S = g.S
    ext = [g.d, g.w, 2.0 * g.h]
    tier = "images2" if S == 60 else "shared"

    def tuned(axis, tune, z_origin=None):
        """A pose whose boundary at `tune` from the low face lies at the float32 coordinate vv along `axis`."""
        o = b.origin()
        if z_origin is not None:
            o[2] = z_origin
        pose = b.pose(o)
        vv = np.float32(o[axis] + 0.3 * ext[axis] + (0.0 if axis != 2 else -g.h))
        hv = float(vv) - o[axis]
        if axis == 0:
            pose["bottom"] = hv - tune
            pose["top"] = pose["bottom"] + g.d
        elif axis == 1:
            pose["center"] = hv - tune + g.w / 2.0
        else:
            pose["sample"][0][2] = float(vv) - (tune - g.h)
        return pose, vv

    def add(pose, axis, vv, claim, rel=0, hand0=None):
        cells = np.full((2, 3), 10)
        cells[1] = [S - 12, S - 12, S - 12]
        hand = b.cells_to_hand(cells, np.full((2, 3), 0.5), pose=pose[0:1])
        world = (pose["sample"][0][None] + hand).astype(np.float32)
        if hand0 is not None:
            world[0] = hand0
        else:
            world[0, axis] = _f32_step(vv, rel)
        b.add(None, b.tilted(2), claim, pose=pose, world=world)

    ks = (1, 7, 13, 22, 29, 37, 44, 51, S - 1) if S == 60 else (1, 5, 11, 16, 23, S - 1)
    for axis in range(3):
        for k in ks:
            for rel in (-1, 0, 1):
                pose, vv = tuned(axis, k * ext[axis] / S)
                add(pose, axis, vv, {"tier": tier, "boundary": (axis, k, rel)}, rel)
    # fault (e): step the tuned bottom / center until the product and the exact divisions disagree on the point's cell
    if S == 60:
        for axis in (0, 1):
            for k in ks[:-1]:
                pose, vv = tuned(axis, k * ext[axis] / S)
                field = "bottom" if axis == 0 else "center"
                hv = float(vv) - pose["sample"][0][axis]
                for step in range(64):
                    hand = np.array([0.0, 0.0, 0.0])
                    hand[axis] = hv
                    if _kernel_cells(g, pose, hand)[1][axis] != _kernel_cells(g, pose, hand, "e")[1][axis]:
                        pose["top"] = pose["bottom"] + g.d
                        add(pose, axis, vv, {"tier": tier, "fault_e": axis})
                        break
                    pose[field] = np.nextafter(pose[field][0], np.inf if step % 2 else -np.inf)
                    for _ in range(step // 2):
                        pose[field] = np.nextafter(pose[field][0], np.inf if step % 2 else -np.inf)
    # faces: on the face (excluded) and 1 ulp inside
    for axis in range(3):
        for upper in (False, True):
            for rel in (0, 1):
                if axis < 2:
                    pose, vv = tuned(axis, ext[axis] if upper else 0.0)
                    hv = float(vv) - pose["sample"][0][axis]
                    field = "bottom" if axis == 0 else "center"
                    off = (g.d if upper else 0.0) if axis == 0 else (g.w / 2.0 if upper else -g.w / 2.0)
                    for _ in range(200):   # step the pose until the face lies exactly at hv in float64
                        face = pose[field][0] + off
                        if face == hv:
                            break
                        pose[field] = np.nextafter(pose[field][0], np.inf if hv > face else -np.inf)
                    assert pose[field][0] + off == hv
                    pose["top"] = pose["bottom"] + g.d
                else:
                    # z: the point near 0.03 m (upper face) or 0.008 m (lower face), where the sample vv -+ volume_height is an
                    # exact float64 and so is the difference
                    want = g.h if upper else -1.0 * g.h
                    pose, vv = tuned(axis, ext[axis] if upper else 0.0, z_origin=0.04 if upper else 0.016)
                    for _ in range(200):
                        sz = float(vv) - want
                        if float(vv) - sz == want:
                            break
                        vv = _f32_step(vv, 1)
                    pose["sample"][0][2] = sz
                    assert float(vv) - pose["sample"][0][2] == want
                add(pose, axis, vv, {"tier": tier, "face": (axis, upper, rel)}, -rel if upper else rel)
    # saturation: bottom < 0 and x the largest float64 below bottom + volume_depth; x - bottom rounds to volume_depth,
    # so u = 1 exactly. The sample is float32(2 x) - x, so that the float32 world coordinate float32(2 x) gives x exactly.
    if S == 60:
        rng = np.random.default_rng(seed)
        found = 0
        while found < 3:
            bt = -rng.uniform(0.005, 0.055)
            x = np.nextafter(bt + g.d, -np.inf)
            wx = np.float32(2.0 * x)
            sx = float(wx) - x
            if not (x > bt and x < bt + g.d and float(wx) - sx == x):
                continue
            o = np.array([sx, 5.0 + 0.25 * found, 0.5])
            pose = b.pose(o)
            pose["bottom"], pose["top"] = bt, bt + g.d
            u, cell = _kernel_cells(g, pose, [x, 0.0, 0.0])
            if u[0] < 1.0:
                continue
            hand = b.cells_to_hand(np.array([[0, 10, 10]]), np.full((1, 3), 0.5), pose=pose[0:1])[0]
            w0 = (o + hand).astype(np.float32)
            w0[0] = wx
            add(pose, 0, None, {"tier": tier, "saturate": True}, hand0=w0)
            found += 1
    return b.case("boundaries" if S == 60 else "boundaries_dyadic")


def all_cases():
    return ([covered_cases(), hole_cases(), constant_cases(), nonunit_cases(), boundary_cases(), boundary_cases(DYADIC, 41)]
            + stack_cases() + size_cases() + shadow_cases())


def params_of(case):
    from gpd_b200 import abi as _abi
    g = case["geometry"]
    return _abi.default_params(g.C, image_size=g.S, volume_width=g.w, volume_depth=g.d, volume_height=g.h)
