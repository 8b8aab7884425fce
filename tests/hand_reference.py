"""Restatement of the hand search (A3-A7) and the grasp filters (A15) in Python, written from the reference sources
(hand_set.cpp:31-116,235-261, finger_hand.cpp, antipodal.cpp:10-96, hand.cpp:24-45, point_list.cpp:22-55;
grasp_detector.cpp:334-398,422-456) separately from the C++ oracle.

Every hand-frame quantity is computed with the association of the kernels and the oracle: to_frame(F, v) is
(F0 v0 + F1 v1) + F2 v2, frame_rot = mat3_mul(mat3_mul(frame, rot_binormal), rot), both on column-major 3 x 3 matrices,
evaluated element by element on float64 (numpy ufuncs round every product and sum, nothing is contracted). No matrix
product (`@`) is used, so the restatement is exact: the oracle's records equal it bit for bit.

`fault` names one deliberate deviation of a predicate (FAULTS): test_hand_cases.py shows that some case of
hand_cases.py tells each one apart from the exact restatement."""
import ctypes as C
import math
import struct

import numpy as np

from oracle import oracle

# deliberate deviations, each the way a kernel could get a predicate subtly wrong
FAULTS = {
    "crop_le": "cropByHandHeight with |z| <= hand_height instead of <",
    "back_le": "back collision x <= bottom instead of x < bottom",
    "bite_le": "points at x <= init_bite count as in front of the fingers",
    "middle_floor": "chooseMiddleHand with floor instead of ceil",
    "aperture_strict": "strict aperture bounds",
    "workspace_strict": "strict workspace bounds",
    "rt_from_rb": "right_top from right_bottom instead of the reference's left_bottom",
    "dir_nan_rejected": "the direction filter rejects a NaN angle (|dot| > 1)",
}


def derived(p):
    """(angles [num_orientations], rot_binormal as 9 column-major floats) as the oracle derives them."""
    drv = np.zeros(4 + p.num_orientations + 9)
    oracle.lib().gpdo_derived(C.byref(p), drv.ctypes.data_as(C.c_void_p))
    return [float(a) for a in drv[4:4 + p.num_orientations]], [float(v) for v in drv[4 + p.num_orientations:]]


def angle_axis9(angle, axis):
    """Eigen::AngleAxisd(angle, axis).toRotationMatrix() as 9 column-major floats (the oracle's host restatement)."""
    R = np.zeros(9)
    oracle.lib().gpdo_angle_axis(C.c_double(angle), np.asarray(axis, np.float64).ctypes.data_as(C.c_void_p),
                                 R.ctypes.data_as(C.c_void_p))
    return [float(v) for v in R]


def mat3_mul(A, B):
    return [(A[r] * B[c * 3] + A[3 + r] * B[c * 3 + 1]) + A[6 + r] * B[c * 3 + 2] for c in range(3) for r in range(3)]


def to_frame(F, v0, v1, v2):
    """F^T v for a column-major frame F; v0, v1, v2 scalars or float64 arrays."""
    return ((F[0] * v0 + F[1] * v1) + F[2] * v2, (F[3] * v0 + F[4] * v1) + F[5] * v2, (F[6] * v0 + F[7] * v1) + F[8] * v2)


def frame_rot(frame9, rotb, angle, axis):
    return mat3_mul(mat3_mul([float(v) for v in frame9], rotb), angle_axis9(angle, np.eye(3)[axis]))


class FingerHand:
    def __init__(self, fw, od, depth, n, fault=None):
        # Eigen's LinSpaced(n, 0, od - fw): low + i * step, step = (high - low) / (n - 1)
        fs_half = np.array([0.0 + i * (((od - fw) - 0.0) / (n - 1)) if i < n - 1 else od - fw for i in range(n)])
        self.fs = np.concatenate([(fs_half - od) + fw, fs_half])
        self.fw, self.depth, self.n, self.fault = fw, depth, n, fault
        self.fingers = np.zeros(2 * n, bool)
        self.hand = np.zeros(n, bool)
        self.top = self.bottom = self.center = 0.0

    def copy(self):
        o = FingerHand.__new__(FingerHand)
        o.__dict__ = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.__dict__.items()}
        return o

    def gap_free(self, pts, cropped, idx):
        y = pts[1, cropped]
        return not np.any((y > self.fs[idx]) & (y < self.fs[idx] + self.fw))

    def evaluate_fingers(self, pts, bite, idx=-1):
        self.top, self.bottom, self.center = bite, bite - self.depth, 0.0
        self.fingers[:] = False
        cropped = []
        for i in range(pts.shape[1]):
            if pts[0, i] < bite or (self.fault == "bite_le" and pts[0, i] == bite):
                if pts[0, i] < self.bottom or (self.fault == "back_le" and pts[0, i] == self.bottom):
                    return
                cropped.append(i)
        if not cropped:
            return
        cropped = np.array(cropped)
        for i in (range(2 * self.n) if idx == -1 else (idx, self.n + idx)):
            if self.gap_free(pts, cropped, i):
                self.fingers[i] = True

    def evaluate_hand(self):
        self.hand = self.fingers[:self.n] & self.fingers[self.n:]

    def choose_middle(self):
        h = np.nonzero(self.hand)[0]
        if len(h) == 0:
            return -1
        k = len(h) // 2 if self.fault == "middle_floor" else int(np.ceil(len(h) / 2.0))
        return int(h[max(k, 1) - 1])


def deepen(fh, pts, min_depth, max_depth):
    idx = fh.choose_middle()
    new, last = fh.copy(), fh.copy()
    depth = min_depth + 0.005
    while depth <= max_depth:
        new.evaluate_fingers(pts, depth, idx)
        if not new.fingers[idx] or not new.fingers[fh.n + idx]:
            break
        last = new.copy()
        depth += 0.005
    last.hand = np.zeros(fh.n, bool)
    last.hand[idx] = True
    return last, idx


def antipodal(pts, nrm, friction_coeff, min_viable):
    cosf = math.cos(friction_coeff * math.pi / 180.0)
    min_x, max_x = pts[1].min() + 0.003, pts[1].max() - 0.003
    ldot = (0.0 * nrm[0] + -1.0 * nrm[1]) + 0.0 * nrm[2]          # l = (0,-1,0), r = (0,1,0)
    rdot = (0.0 * nrm[0] + 1.0 * nrm[1]) + 0.0 * nrm[2]
    left, right = np.nonzero((ldot > cosf) & (pts[1] < min_x))[0], np.nonzero((rdot > cosf) & (pts[1] > max_x))[0]
    half = len(left) > 0 or len(right) > 0
    full = False
    if len(left) > 0 and len(right) > 0:
        L, R = pts[:, left], pts[:, right]
        top_y, bot_y = min(L[0].max(), R[0].max()), max(L[0].min(), R[0].min())
        top_z, bot_z = min(L[2].max(), R[2].max()), max(L[2].min(), R[2].min())
        inside = lambda Q: int(np.count_nonzero((Q[0] >= bot_y) & (Q[0] <= top_y) & (Q[2] >= bot_z) & (Q[2] <= top_z)))
        full = inside(L) >= min_viable and inside(R) >= min_viable
    return half, full


def hand_set(p, sample, frame9, pts, nrm, fault=None):
    """HandSet::evalHands for one sample: `pts` [n, 3] float64 (the float32 cloud points) and `nrm` [n, 3] of the
    hand-search ball in the sorted radius search's order (neighbour 0 first). -> list over (axis, angle) of None (not
    valid) or a dict of Hand fields."""
    angles, rotb = derived(p)
    axes = list(p.hand_axes[:p.num_hand_axes])
    sx, sy, sz = (float(v) for v in sample)
    out = []
    for ax in axes:
        fh0 = FingerHand(p.finger_width, p.hand_outer_diameter, p.hand_depth, p.num_finger_placements, fault)
        for ang in angles:
            fh = fh0.copy()                                   # evaluateFingers resets the state that matters
            R = frame_rot(frame9, rotb, ang, ax)
            P = np.array(to_frame(R, pts[:, 0] - sx, pts[:, 1] - sy, pts[:, 2] - sz))
            N = np.array(to_frame(R, nrm[:, 0], nrm[:, 1], nrm[:, 2]))
            hh = p.hand_height
            if fault == "crop_le":
                inr = np.nonzero((P[2] >= -1.0 * hh) & (P[2] <= hh))[0]
            else:
                inr = np.nonzero((P[2] > -1.0 * hh) & (P[2] < hh))[0]
            pad = P.shape[1] - len(inr)
            idx = np.concatenate([inr, np.zeros(pad, np.int64)]).astype(np.int64)   # cropByHandHeight quirk
            Pc, Nc = P[:, idx], N[:, idx]
            fh.evaluate_fingers(Pc, p.init_bite)
            fh.evaluate_hand()
            if not fh.hand.any():
                out.append(None)
                continue
            if p.deepen_hand:
                fh, fidx = deepen(fh, Pc, p.init_bite, p.hand_depth)
            else:
                fidx = fh.choose_middle()
            left, right = fh.fs[fidx] + fh.fw, fh.fs[fh.n + fidx]
            fh.center = 0.5 * (left + right)
            closing = np.nonzero((Pc[0] > fh.bottom) & (Pc[0] < fh.top) & (Pc[1] > left) & (Pc[1] < right))[0]
            if len(closing) == 0:
                out.append(None)
                continue
            half, full = antipodal(Pc[:, closing], Nc[:, closing], p.friction_coeff, p.min_viable)
            pb = (fh.bottom, fh.center, 0.0)
            position = [((R[r] * pb[0] + R[3 + r] * pb[1]) + R[6 + r] * pb[2]) + float(sample[r]) for r in range(3)]
            out.append({"frame": R, "position": position, "top": fh.top, "bottom": fh.bottom, "center": fh.center,
                        "finger_idx": int(np.nonzero(fh.hand)[0][0]),
                        "width": Pc[1, closing].max() - Pc[1, closing].min(), "half": half, "full": full})
    return out


def direction_angle(p, r):
    a = r["frame"]
    dot = (p.direction[0] * a[0] + p.direction[1] * a[1]) + p.direction[2] * a[2]
    return dot, (math.acos(dot) if -1.0 <= dot <= 1.0 else math.nan)


def filtered(p, r, fault=None):
    """GraspDetector::filterGraspsWorkspace (grasp_detector.cpp:334-398; right_top is computed from left_bottom there)
    followed by filterGraspsDirection (:422-456) when enabled: erased when acos(dot) > thresh, so a NaN angle
    (|dot| > 1) keeps the grasp."""
    a, b, pos = r["frame"][0:3], r["frame"][3:6], r["position"]
    hw = 0.5 * p.hand_outer_diameter
    ws = list(p.workspace_grasps)
    if fault == "aperture_strict":
        ok = p.min_aperture < r["width"] < p.max_aperture
    else:
        ok = p.min_aperture <= r["width"] <= p.max_aperture
    for k in range(3):
        lb = pos[k] + hw * b[k]
        rb = pos[k] - hw * b[k]
        lt = lb + p.hand_depth * a[k]
        rt = (rb if fault == "rt_from_rb" else lb) + p.hand_depth * a[k]
        ap = pos[k] - 0.05 * a[k]
        mn, mx = min(min(min(lb, rb), min(lt, rt)), ap), max(max(max(lb, rb), max(lt, rt)), ap)
        if fault == "workspace_strict":
            ok = ok and mn > ws[2 * k] and mx < ws[2 * k + 1]
        else:
            ok = ok and mn >= ws[2 * k] and mx <= ws[2 * k + 1]
    if ok and p.filter_approach_direction:
        dot, angle = direction_angle(p, r)
        if fault == "dir_nan_rejected":
            ok = angle <= p.thresh_rad
        else:
            ok = not (angle > p.thresh_rad)
    return bool(ok)


# ---- the direction filter as the kernel evaluates it: one comparison against the switch point d* of the host acos

def _key(x):
    b = struct.unpack("<q", struct.pack("<d", x))[0]
    return -(b & 0x7FFFFFFFFFFFFFFF) if b < 0 else b


def _from_key(k):
    return struct.unpack("<d", struct.pack("<q", (-k) | -0x8000000000000000 if k < 0 else k))[0]


def ulp_step(x, k):
    """The double k steps away from x in the order of the doubles."""
    return _from_key(_key(x) + k)


def d_star(thresh):
    """Smallest double in [-1, 1] with not (acos(d) > thresh), by bisection over the ordered doubles; 2.0 when every
    d in [-1, 1] is rejected, -1.0 when none is."""
    rej = lambda k: math.acos(_from_key(k)) > thresh
    lo, hi = _key(-1.0), _key(1.0)
    if not rej(lo):
        return -1.0
    if rej(hi):
        return 2.0
    while hi - lo > 1:
        mid = lo + (hi - lo) // 2
        if rej(mid):
            lo = mid
        else:
            hi = mid
    return _from_key(hi)


def direction_rejects_kernel(dot, dstar):
    return -1.0 <= dot <= 1.0 and dot < dstar


# ---- a whole case: the oracle's frames, flags and records beside the restatement's

def hand_ball_radius(p):
    return max(max(p.hand_outer_diameter - p.finger_width, p.hand_depth), p.hand_height / 2.0)


def case_samples(case, oc):
    """Sample indices of a hand_cases case for an OracleCloud (or a lib.Context) holding its cloud: cloud points by
    index, float64 positions installed with set_samples."""
    pos = [s for kind, s in case["samples"] if kind == "position"]
    first = list(oc.set_samples(np.array(pos))) if pos else []
    out, k = [], 0
    for kind, s in case["samples"]:
        if kind == "position":
            out.append(first[k])
            k += 1
        else:
            out.append(s)
    return np.array(out, np.int32)


def run_case(case, p, fault=None):
    """(sample indices, oracle frames, valid, poses [n, P], flags [n, P], restated records [n][P], restated flags)."""
    from gpd_b200 import abi
    c = case["cloud"]
    oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    sidx = case_samples(case, oc)
    frames, valid = oc.frames(p, sidx)
    poses, flags = oc.hand_search(p, sidx, frames, valid)
    xyz = np.vstack([c["xyz"].astype(np.float64)])
    recs, rflags = [], np.zeros_like(flags)
    for i, si in enumerate(sidx):
        kind, s = case["samples"][i]
        sample = np.asarray(s, np.float64) if kind == "position" else xyz[s]
        idx, _ = oc.radius_search(sample.astype(np.float32), hand_ball_radius(p))
        rs = hand_set(p, sample, frames[i], xyz[idx], c["normals"][idx], fault) if valid[i] and len(idx) else \
            [None] * flags.shape[1]
        recs.append(rs)
        for j, r in enumerate(rs):
            if r is not None:
                rflags[i, j] = (abi.POSE_VALID | (abi.POSE_HALF if r["half"] else 0) | (abi.POSE_FULL if r["full"] else 0)
                                | (abi.POSE_FILTERED if filtered(p, r, fault) else 0))
    return sidx, frames, valid, poses, flags, recs, rflags
