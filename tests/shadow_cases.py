"""Inputs that put an exact number of entries into the lists of the shadow casting of the 15-channel images
(test_shadow_cast_reference.py proves the counts on the CPU with tests/shadow_cast_reference.py, test_gpu_shadow_cast.py
checks the kernels' counters against them).

One hand-built candidate in the style of capacity_cases.image_box: sample (0, 0, 0.5), identity frame, bottom 0,
center 0, so hand coordinates are world coordinates minus the sample. Every coordinate is a multiple of 2^-12, so the
float32 ball and the float64 centre are exact in any order. The cameras stand 16 m away along -y, so every shadow
segment runs (almost exactly) along +y, the long axis of the image box. The points come from four regions:

* FULL: just outside the box on the camera side (y in [-0.058, -0.0505]): the whole segment lies inside the cull box,
  so the cull passes and every one of the nsp draws passes its window; the segment crosses the box along y;
* FINE: just past the box's far face (y in [0.0505, 0.058]): the cull passes, one to four draws pass the window and
  at most two voxels of the point's column pass the pre-test, which lets a count grow by 0, 1 or 2 per point;
* BOX: inside the box, y in [-0.048, -0.042] (a full window too): the points of the image's point channels;
* BALLAST: in the ball with |z| >= 3.5 cm in hand coordinates (1.5 cm beyond the box's faces at +-2 cm, 0.45 cm
  beyond the cull box): its segment misses the cull box.

A builder adds FULL points (one per voxel column first) until a count is near its target and FINE points, one at a
time, until it hits the target exactly; a point that would overshoot is left out. Work-list and draw-list counts are
additive per point and are reached directly. Each case records its counts as shadow_cast_reference.cast gives them."""
import functools

import numpy as np

import capacity_cases as cc
import shadow_cast_reference as scr
from gpd_b200 import abi
from image_reference import Geometry

Q = 2.0 ** -12
SAMPLE = np.array([0.0, 0.0, 0.5])
VP = [[0.03125, -16.0, 0.5], [0.09375, -16.0, 0.5]]  # cameras 0 and 1: shadow segments along +y, 0.2 degrees apart

# the kernels' capacities (gpd_b200/csrc/geometry.cu, by symbol); k_images2's stash: capacity_cases.st_sm2 / st_cap2
WL_CAP2, WL_CAP, DL_CAP = cc.WL_CAP2, cc.WL_CAP, cc.DL_CAP
BALL_CAP = 2 * cc.IMG2_S * cc.IMG2_S   # k_images: the in-ball list over tile C (7 200)

GEOMETRIES = {
    "default": dict(S=60, C=15, w=0.10, d=0.06, h=0.02),
    "depth05": dict(S=60, C=15, w=0.10, d=0.05, h=0.02),  # two cameras still take k_images2 (bm_dim 46)
    "tall": dict(S=60, C=15, w=0.10, d=0.06, h=0.04),     # bm_dim 54: k_images' voxel list shrinks to 12 600
}


def params_of(case):
    g = case["geometry"]
    return dict(channels=15, image_size=g.S, volume_width=g.w, volume_depth=g.d, volume_height=g.h)


class Builder:
    def __init__(self, geo, K, seed, cam0_sees=True):
        self.g = Geometry(**GEOMETRIES[geo])
        self.geo, self.K, self.cam0_sees = geo, K, cam0_sees
        self.rng = np.random.default_rng(seed)
        self.pts = []          # hand coordinates in units of Q (int64 [3])
        self.have = set()
        d, h = self.g.d, self.g.h
        lo_x, hi_x = 0.001, d - 0.001
        self.regions = {
            "full": ([lo_x, -0.058, -h + 0.001], [hi_x, -0.0505, h - 0.001]),
            "fine": ([lo_x, 0.0505, -h + 0.001], [hi_x, 0.058, h - 0.001]),
            "box": ([lo_x, -0.048, -h + 0.001], [hi_x, -0.042, h - 0.001]),
        }
        self.columns = None
        self.pose = np.zeros(1, dtype=abi.POSE_DTYPE)
        self.pose["sample"][0] = SAMPLE
        self.pose["frame"][0] = np.eye(3).ravel()
        self.pose["bottom"], self.pose["top"], self.pose["center"] = 0.0, d, 0.0
        self.pose["sample_index"] = 7
        self.pose["finger_idx"] = 4
        self.pose["score"] = np.nan

    def _draw(self, lo, hi, n, keep=None):
        lo_k = np.ceil(np.asarray(lo) / Q).astype(np.int64)
        hi_k = np.floor(np.asarray(hi) / Q).astype(np.int64)
        out = []
        while len(out) < n:
            k = self.rng.integers(lo_k, hi_k + 1, (2 * (n - len(out)) + 16, 3))
            for t in map(tuple, k):
                if t not in self.have and (keep is None or keep(np.array(t) * Q)) and len(out) < n:
                    self.have.add(t)
                    out.append(t)
        return out

    def add(self, region, n):
        if region == "ballast":
            def keep(p):  # inside the ball (r = 0.1) with room to spare, away from the cull box
                return p @ p < 0.0095 and abs(p[2]) >= 0.035
            new = []
            while len(new) < n:
                sign = 1.0 if self.rng.random() < 0.5 else -1.0
                zlo, zhi = sorted([sign * 0.035, sign * 0.06])
                new += self._draw([-0.04, -0.05, zlo], [0.04, 0.05, zhi], 1, keep)
        elif region == "full" and self.columns is not None and len(self.columns):
            new = []
            while len(new) < n and len(self.columns):
                vx, vz = self.columns[-1]
                self.columns = self.columns[:-1]
                lo, hi = self.regions["full"]
                x0, x1 = max(lo[0], vx * 0.003 + 0.0003), min(hi[0], vx * 0.003 + 0.0027)
                z0, z1 = max(lo[2], vz * 0.003 + 0.0003 - 0.5), min(hi[2], vz * 0.003 + 0.0027 - 0.5)
                if x0 < x1 and z0 < z1:
                    new += self._draw([x0, lo[1], z0], [x1, hi[1], z1], 1)
            new += self._draw(*self.regions["full"], n - len(new))
        else:
            new = self._draw(*self.regions[region], n)
        self.pts += new
        return len(new)

    def spread_columns(self):
        """FULL points go one per voxel column (x, z) first, in a random order."""
        lo, hi = self.regions["full"]
        vx = np.arange(int(lo[0] / 0.003), int(hi[0] / 0.003) + 1)
        vz = np.arange(int((0.5 + lo[2]) / 0.003), int((0.5 + hi[2]) / 0.003) + 1)
        cols = np.stack(np.meshgrid(vx, vz, indexing="ij"), -1).reshape(-1, 2)
        self.columns = cols[self.rng.permutation(len(cols))]

    def cloud(self):
        obj = (SAMPLE + np.array(self.pts, np.float64) * Q).astype(np.float32)
        bg, bgn = cc._plane(-0.5, Q, self.rng)
        xyz = np.vstack([obj, bg])
        nrm = np.vstack([cc._unit(np.random.default_rng(len(obj)).standard_normal((len(obj), 3))), bgn])
        vp = np.array(VP[:self.K], np.float64)
        cam = np.ones((len(xyz), self.K), np.int32)
        if not self.cam0_sees:
            cam[:, 0] = 0
        return {"xyz": xyz, "normals": nrm, "cam_source": cam, "view_points": vp}

    def counts(self):
        return scr.cast(self.cloud(), self.pose[0], self.g)

    def reach(self, metric, target, per_point):
        """FULL points in chunks while the count is well below target, then FINE points one by one to hit it."""
        r = self.counts()
        while metric(r) < target - 3 * per_point:
            self.add("full", max(1, int((target - metric(r)) / per_point / 2)))
            r = self.counts()
        tries = 0
        while metric(r) < target:
            self.add("fine", 1)
            r2 = self.counts()
            if metric(r2) > target:
                self.have.discard(self.pts.pop())
            else:
                r = r2
            tries += 1
            assert tries < 2000, "no FINE point reaches the target"
        assert metric(r) == target, (metric(r), target)
        return r

    def case(self, name, edge, target, r):
        return {"name": name, "edge": edge, "target": target, "geometry": self.g, "geo": self.geo, "K": self.K,
                "cloud": self.cloud(), "pose": self.pose, "counts": r}


def _stash(geo, K, target, seed):
    b = Builder(geo, K, seed)
    b.add("box", 30 if target > 1000 else 10)
    b.spread_columns()
    return b, b.reach(lambda r: r["nset_all"], target, 12 if K == 2 else 20)


def _work_list(geo, K, target, seed):
    """target FULL and BOX points (every one cast, every draw in its window), ballast for a realistic ball."""
    b = Builder(geo, K, seed)
    b.add("box", 200)
    b.add("full", target - 200)
    b.add("ballast", 300)
    return b, b.counts()


def _draw_list(target, seed):
    b = Builder("default", 1, seed)
    b.add("box", 150)
    b.spread_columns()
    return b, b.reach(lambda r: r["dl_n"][0], target, 33)


def _ball(target, seed):
    """target in-ball points: 150 BOX points, 20 FULL points, the rest ballast (no list but the ball list fills)."""
    b = Builder("default", 1, seed)
    b.add("box", 150)
    b.add("full", 20)
    b.add("ballast", target - 170)
    return b, b.counts()


def _no_camera0(seed):
    b = Builder("depth05", 2, seed, cam0_sees=False)
    b.add("box", 100)
    b.add("full", 50)
    return b, b.counts()


EDGES = [
    # (name, edge, kernel count, target, builder)
    ("stash_sm_1cam", "st_sm", cc.st_sm2(48, 1)),
    ("stash_sm_1cam", "st_sm+1", cc.st_sm2(48, 1) + 1),
    ("stash_cap_1cam", "st_cap", cc.st_cap2(48, 1)),
    ("stash_cap_1cam", "st_cap+1", cc.st_cap2(48, 1) + 1),
    ("stash_sm_2cam", "st_sm", cc.st_sm2(46, 2)),
    ("stash_sm_2cam", "st_sm+1", cc.st_sm2(46, 2) + 1),
    ("stash_cap_2cam", "st_cap", cc.st_cap2(46, 2)),
    ("stash_cap_2cam", "st_cap+1", cc.st_cap2(46, 2) + 1),
    ("voxel_list", "bl_cap", cc.bl_cap(54, 1)),
    ("voxel_list", "bl_cap+1", cc.bl_cap(54, 1) + 1),
    ("work_list_1cam", "wl_cap2", WL_CAP2),
    ("work_list_1cam", "wl_cap2+1", WL_CAP2 + 1),
    ("work_list_1cam", "wl_cap", WL_CAP),
    ("work_list_1cam", "wl_cap+1", WL_CAP + 1),
    ("work_list_2cam", "wl_cap2", WL_CAP2),
    ("work_list_2cam", "wl_cap2+1", WL_CAP2 + 1),
    ("work_list_2cam", "wl_cap", WL_CAP),
    ("work_list_2cam", "wl_cap+1", WL_CAP + 1),
    ("draw_list", "dl_cap", DL_CAP),
    ("draw_list", "dl_cap+1", DL_CAP + 1),
    ("ball", "ball_cap", BALL_CAP),
    ("ball", "ball_cap+1", BALL_CAP + 1),
    ("no_camera0", "empty", 0),
    # one camera at volume_depth 0.05 (ST_SM 2 492): in a batch beside a two-camera cloud, whose ST_SM is 376
    ("stash_sm_1cam_d05", "st_sm", cc.st_sm2(46, 1)),
    ("stash_sm_1cam_d05", "st_sm+1", cc.st_sm2(46, 1) + 1),
]
IDS = [f"{n}-{e}" for n, e, _ in EDGES]


@functools.lru_cache(maxsize=None)
def build(i):
    """The case of EDGES[i]: a dict with the cloud, the pose and the restatement's counts ("counts")."""
    name, edge, target = EDGES[i]
    seed = 100 + i
    if name.startswith("stash"):
        geo, K = {"1cam": ("default", 1), "1cam_d05": ("depth05", 1), "2cam": ("depth05", 2)}[name.split("_", 2)[2]]
        b, r = _stash(geo, K, target, seed)
    elif name == "voxel_list":
        b = Builder("tall", 1, seed)
        b.add("box", 150)
        b.regions["full"] = ([0.001, -0.058, -0.039], [0.059, -0.0505, 0.039])
        b.regions["fine"] = ([0.001, 0.0505, -0.039], [0.059, 0.058, 0.039])
        b.spread_columns()
        r = b.reach(lambda r: r["nset_all"], target, 20)
    elif name.startswith("work_list"):
        geo, K = ("default", 1) if name.endswith("1cam") else ("depth05", 2)
        b, r = _work_list(geo, K, target, seed)
    elif name == "draw_list":
        b, r = _draw_list(target, seed)
    elif name == "ball":
        b, r = _ball(target, seed)
    else:
        b, r = _no_camera0(seed)
    return b.case(name, edge, target, r)
