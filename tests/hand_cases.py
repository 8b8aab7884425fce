"""Hand-built clouds whose hand-frame coordinates land on the predicates of the hand search and the grasp filters
(test_hand_cases.py proves the reach on the CPU from hand_reference.py's intermediates, test_gpu_hand_edges.py checks
k_frames / k_hands against the oracle bit for bit).

Every object is isolated (objects 1 m apart, beyond every search ball) around its own sample. Within the r = nn_radius
frame ball it is a 3 x 3 patch of points 2^-8 m apart whose normals are all +z, so that the local frame is exactly the
permutation normal = +z, binormal = -y, curvature axis = +x. With 8 orientations about the curvature axis, pose 4 has
angle 0 and rot = I, and its hand frame is that permutation times AngleAxis(pi, y): a world offset v has the hand
coordinates x = -s vx - vz, y = -vy, z = -vx + s vz with s = sin(pi) = 1.22e-16, every product and sum evaluated
exactly as hand_reference.to_frame does. The approach of pose 4 is (-s, 0, -1), so direction = (0, 0, -d) gives
dot = d exactly.

Probe points sit outside the frame ball in hand coordinates. Edges that need a coordinate exactly on a float64 bound
take a gpdb_set_samples position as the sample: the hand transform subtracts the float64 position from the float32
point, and the position is chosen so that the difference is the bound itself or one float64 ulp either side."""
import math

import numpy as np

import hand_reference as hr
from gpd_b200 import abi

POSE0 = 4                     # angle 0 of 8 orientations about the curvature axis
PATCH_STEP = 2.0 ** -8
Y_SLOT7 = 0.09                # inside right finger slot 7 (0.0856, 0.0956) at the default hand, far from slots 0-6


def default_over(**kw):
    over = {"hand_axes": [2], "num_orientations": 8}
    over.update(kw)
    return over


def exact_sample(w, t):
    """A float64 s near w - t with float64(w) - s == t exactly, or None."""
    s = float(w) - t
    for k in (0, 1, -1, 2, -2, 3, -3):
        c = hr.ulp_step(s, k)
        if float(w) - c == t:
            return c
    return None


def exact_pair(t):
    """(w float32, s float64) within 0.12 m of 0 with float64(w) - s == t exactly."""
    for w in np.arange(1, 123, dtype=np.float32) * np.float32(2.0 ** -10):
        s = exact_sample(w, t)
        if s is not None:
            return w, s
    raise AssertionError(t)


class Builder:
    def __init__(self):
        self.xyz, self.nrm, self.samples, self.claims = [], [], [], []

    def _patch(self, f):
        g = np.array([(i, j) for i in (-1, 0, 1) for j in (-1, 0, 1)], np.float64) * PATCH_STEP
        pts = np.zeros((9, 3), np.float32)
        pts[:, 0] = np.float32(f[0]) + g[:, 0]
        pts[:, 1] = np.float32(f[1]) + g[:, 1]
        pts[:, 2] = np.float32(f[2])
        pts[4] = np.asarray(f, np.float32)       # the patch centre is the float32 image of the sample
        return pts

    def add(self, sample, probes, claim, position=False):
        """sample: float64 [3]; probes: float32 world points [k, 3]. position: the sample is a float64 position
        (gpdb_set_samples), else it is the patch centre, a cloud point."""
        f = np.asarray(sample, np.float64).astype(np.float32)
        pts = self._patch(f)
        base = sum(len(x) for x in self.xyz)
        self.xyz.append(np.vstack([pts, np.asarray(probes, np.float32).reshape(-1, 3)]))
        n = np.zeros((len(self.xyz[-1]), 3))
        n[:, 2] = 1.0
        self.nrm.append(n)
        self.samples.append(("position", np.asarray(sample, np.float64)) if position else ("point", base + 4))
        self.claims.append(claim)

    def case(self, name, over=None):
        xyz = np.vstack(self.xyz)
        return {"name": name, "over": default_over(**(over or {})),
                "cloud": {"xyz": xyz, "normals": np.vstack(self.nrm), "cam_source": np.ones((len(xyz), 1), np.int32),
                          "view_points": np.zeros((1, 3))},
                "samples": self.samples, "claims": self.claims}


def origin(k):
    return np.array([0.0, 0.5 + 1.0 * k, 0.0])


def _hand_probe(sample, x, y, z):
    """Float32 world point at the hand coordinates (x, y, z) of pose 4, to float32 rounding."""
    return np.array([sample[0] - z, sample[1] - y, sample[2] - x], np.float32)


def crop_cases():
    """A probe in right slot 7 at z = +-hand_height, on the bound and one float64 ulp either side (float64 sample
    positions), and at the nearest float32 steps either side (cloud-point samples). Kept (|z| < hand_height), it blocks
    hand 7, and the middle of the free hands 1-6 is hand 3; cropped, the free hands are 1-7 and the middle is hand 4."""
    hh = 0.02
    b = Builder()
    k = 0
    for sign in (1.0, -1.0):
        for rel in (-1, 0, 1):
            t = hr.ulp_step(sign * hh, rel)                  # target z
            wx, sx = exact_pair(-t)                          # vx = wx - sx = -z
            o = origin(k)
            sample = np.array([sx, o[1], o[2]])
            probe = _hand_probe(sample, 0.0, Y_SLOT7, t)
            probe[0] = wx
            kept = -hh < t < hh
            b.add(sample, probe[None], {"pred": "crop", "z": t, "kept": kept, "finger_idx": 3 if kept else 4},
                  position=True)
            k += 1
    for sign in (1.0, -1.0):
        for side in (-1, 1):                                 # the float32 step just inside / just outside
            o = origin(k)
            sample = np.array([0.5, o[1], o[2]])
            wx = np.float32(0.5 - sign * hh)
            while not (-(float(wx) - 0.5) * sign < hh if side < 0 else -(float(wx) - 0.5) * sign > hh):
                wx = np.nextafter(wx, np.float32(np.inf if (side < 0) == (sign > 0) else -np.inf))
            probe = _hand_probe(sample, 0.0, Y_SLOT7, 0.0)
            probe[0] = wx
            z = -(float(wx) - 0.5)
            kept = -hh < z < hh
            b.add(sample, probe[None], {"pred": "crop", "z": z, "kept": kept, "finger_idx": 3 if kept else 4})
            k += 1
    return b.case("crop")


def bite_cases():
    """A probe in right slot 7 with x on init_bite (in front of the fingers: x < init_bite) and on init_bite -
    hand_depth (the back: x < bottom ends evaluateFingers with no finger free), on and one float64 ulp either side."""
    b = Builder()
    k = 0
    for pred, bound in (("bite", 0.01), ("back", 0.01 - 0.06)):
        for rel in (-1, 0, 1):
            t = hr.ulp_step(bound, rel)                      # target x = -vz
            wz, sz = exact_pair(-t)                          # vz = wz - sz = -x
            o = origin(k)
            sample = np.array([o[0], o[1], sz])
            probe = _hand_probe(sample, t, Y_SLOT7, 0.0)
            probe[2] = wz
            if pred == "bite":
                claim = {"pred": "bite", "x": t, "front": t < 0.01, "finger_idx": 3 if t < 0.01 else 4}
            else:
                claim = {"pred": "back", "x": t, "collides": t < bound, "finger_idx": None if t < bound else 3}
            b.add(sample, probe[None], claim, position=True)
            k += 1
    # the same bounds at the nearest float32 steps either side, with cloud-point samples (so that they also run in a
    # batch): the sample at z = 0.5, the probe at the float32 z = w, x = 0.5 - w
    for pred, bound in (("bite", 0.01), ("back", 0.01 - 0.06)):
        w0 = np.float32(0.5 - bound)
        ws = [np.float32(w0 + np.float32(i) * np.spacing(w0)) for i in range(-3, 4)]
        xs = sorted((0.5 - float(w), w) for w in ws)
        for t, w in (max(v for v in xs if v[0] < bound), min(v for v in xs if v[0] > bound)):
            o = origin(k)
            sample = np.array([o[0], o[1], 0.5])
            probe = _hand_probe(sample, t, Y_SLOT7, 0.0)
            probe[2] = w
            if pred == "bite":
                claim = {"pred": "bite", "x": t, "front": t < 0.01, "finger_idx": 3 if t < 0.01 else 4}
            else:
                claim = {"pred": "back", "x": t, "collides": t < bound, "finger_idx": None if t < bound else 3}
            b.add(sample, probe[None], claim)
            k += 1
    return b.case("bite")


def single_object(sample=(0.25, 0.5, 0.0)):
    b = Builder()
    b.add(np.array(sample, np.float64), np.zeros((0, 3)), {})
    return b


def _record(case, p):
    """The restatement's pose records of the case's first sample, with the oracle's frame."""
    return hr.run_case(case, p)[5][0]


def filter_cases():
    """Cases of the aperture and workspace filters at their bounds and of the right_top quirk, each one context on a
    single object: the bound is set from the exact record of pose 4 (hand_reference), on it and one ulp beyond."""
    out = []
    base = single_object().case("filter_base")
    p = abi.default_params(15, **base["over"])
    recs = _record(base, p)
    r = recs[POSE0]
    w = r["width"]
    for name, rel, keep in (("max_aperture", 0, True), ("max_aperture", -1, False),
                            ("min_aperture", 0, True), ("min_aperture", 1, False)):
        c = single_object().case(f"aperture_{name}_{rel}", {name: hr.ulp_step(w, rel)})
        c["claims"] = [{"pred": "aperture", "pose": POSE0, "filtered": keep}]
        out.append(c)
    hw = 0.5 * 0.12
    a, bn, pos = r["frame"][0:3], r["frame"][3:6], r["position"]
    for k in range(3):
        lb = pos[k] + hw * bn[k]
        rb = pos[k] - hw * bn[k]
        lt = lb + 0.06 * a[k]
        ap = pos[k] - 0.05 * a[k]
        mn, mx = min(min(min(lb, rb), min(lt, lt)), ap), max(max(max(lb, rb), max(lt, lt)), ap)
        for upper, bound in ((False, mn), (True, mx)):
            for rel, keep in ((0, True), ((-1 if upper else 1), False)):
                ws = [-1.0, 1.0, -1.0, 1.0, -1.0, 1.0]
                ws[2 * k + upper] = hr.ulp_step(bound, rel)
                c = single_object().case(f"workspace_{k}{'+' if upper else '-'}_{rel}", {"workspace_grasps": ws})
                c["claims"] = [{"pred": "workspace", "pose": POSE0, "filtered": keep}]
                out.append(c)
    # right_top: at angle -pi/4 (pose 2) the true right-top corner is the largest y of the hand, the quirk's is not
    r2 = recs[2]
    a, bn, pos = r2["frame"][0:3], r2["frame"][3:6], r2["position"]
    lb = pos[1] + hw * bn[1]
    rb = pos[1] - hw * bn[1]
    ap = pos[1] - 0.05 * a[1]
    mx = max(max(max(lb, rb), lb + 0.06 * a[1]), ap)
    assert rb + 0.06 * a[1] > mx
    c = single_object().case("right_top_quirk", {"workspace_grasps": [-1.0, 1.0, -1.0, mx, -1.0, 1.0]})
    c["claims"] = [{"pred": "right_top", "pose": 2, "filtered": True}]
    out.append(c)
    return out


def direction_case(d, thresh, name=None):
    c = single_object().case(name or f"dir_{d!r}_{thresh!r}", {"filter_approach_direction": 1, "direction": [0.0, 0.0, -d],
                                                               "thresh_rad": thresh})
    angle = math.acos(d) if -1.0 <= d <= 1.0 else math.nan
    c["claims"] = [{"pred": "direction", "pose": POSE0, "dot": d, "filtered": not (angle > thresh)}]
    return c


# thresholds of the acos sweep: default, and values whose switch point lies in each range of the device acos
SWEEP_THRESH = [2.3, 0.05, 0.3, 0.7, 1.0, 1.2, 1.5, 1.5707963267948966, 1.6, 2.0, 2.6, 2.9, 3.1, 3.14]
SWEEP_HALF = 100              # doubles either side of each switch point
SWEEP_ANGLE = 8               # angle ulps either side of each threshold


def sweep_dots(t, half=SWEEP_HALF, angle=SWEEP_ANGLE):
    """The dots of the sweep at threshold t: the 2 half doubles around the switch point d*, and the switch points of
    the thresholds up to `angle` ulps either side of t. The second set covers what an acos a few ulps off could
    misjudge where one angle ulp spans many doubles of dot (near pi / 2, d* is close to 0)."""
    ds = hr.d_star(t)
    dots = {hr.ulp_step(ds, k) for k in range(-half, half)}
    dots |= {hr.d_star(hr.ulp_step(t, j)) for j in range(-angle, angle + 1)}
    return sorted(dots)


def direction_cases(thresholds=SWEEP_THRESH, half=SWEEP_HALF, angle=SWEEP_ANGLE):
    """sweep_dots at each threshold; then |dot| > 1 (acos NaN: kept), dot = +-1, a negative threshold (every dot in
    [-1, 1] rejected) and thresholds at and above pi and NaN (none rejected)."""
    out = []
    for t in thresholds:
        for d in sweep_dots(t, half, angle):
            out.append(direction_case(d, t))
    for d in (hr.ulp_step(1.0, 1), 1.5, hr.ulp_step(-1.0, -1), -3.0, 1.0, -1.0):
        for t in (0.5, 2.3):
            out.append(direction_case(d, t))
    for t in (-0.1, -0.0, math.pi, 4.0, math.nan):
        for d in (-1.0, -0.5, 0.0, 0.5, 1.0, 1.25):
            out.append(direction_case(d, t))
    return out


def geometry_cases():
    return [crop_cases(), bite_cases()]


# the geometry cases off their defaults: deepenHand off (finger_idx is the first free hand) and all three hand axes
# (24 poses; the slab prefilter is off). The claims hold for the default only; off it the cases are compared only.
VARIANTS = {"default": {}, "no_deepen": {"deepen_hand": 0}, "all_axes": {"hand_axes": [0, 1, 2]}}


def variant(case, name):
    if name == "default":
        return case
    return dict(case, name=f"{case['name']}_{name}", over=dict(case["over"], **VARIANTS[name]),
                claims=[{} for _ in case["claims"]])
