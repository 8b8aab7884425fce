"""The hand-search edge cases of hand_cases.py on the CPU: the oracle equals the exact restatement of hand_reference.py
bit for bit on every case, each case reaches the predicate edge it claims, and every fault of hand_reference.FAULTS
changes a flag or a record field on at least one case."""
import math

import numpy as np
import pytest

import hand_cases as hc
import hand_reference as hr
from gpd_b200 import abi

FIELDS = ("top", "bottom", "center", "width", "finger_idx")


def params(case):
    return abi.default_params(15, **case["over"])


def assert_oracle_equals_restatement(case):
    p = params(case)
    sidx, frames, valid, poses, flags, recs, rflags = hr.run_case(case, p)
    assert valid.all(), case["name"]
    assert np.array_equal(flags, rflags), (case["name"], flags, rflags)
    for i in range(len(sidx)):
        for j, r in enumerate(recs[i]):
            if r is None:
                continue
            g = poses[i, j]
            assert list(g["frame"]) == r["frame"] and list(g["position"]) == r["position"], (case["name"], i, j)
            for f in FIELDS:
                assert g[f] == r[f], (case["name"], i, j, f)
            assert bool(g["half_antipodal"]) == r["half"] and bool(g["full_antipodal"]) == r["full"]
    return p, frames, recs, flags


def check_claims(case, p, frames, recs, flags):
    for i, cl in enumerate(case["claims"]):
        if not cl:
            continue
        j = cl.get("pose", hc.POSE0)
        # the frame is the exact permutation the cases are built on
        assert list(frames[i]) == [0.0, 0.0, 1.0, 0.0, -1.0, 0.0, 1.0, 0.0, 0.0], frames[i]
        pred = cl["pred"]
        if pred in ("crop", "bite", "back"):
            kind, s = case["samples"][i]
            c = case["cloud"]
            sample = np.asarray(s, np.float64) if kind == "position" else c["xyz"][s].astype(np.float64)
            pw = c["xyz"][10 * i + 9].astype(np.float64)   # each object: the 9 patch points, then its probe
            angles, rotb = hr.derived(p)
            R = hr.frame_rot(frames[i], rotb, angles[j], 2)
            x, y, z = hr.to_frame(R, pw[0] - sample[0], pw[1] - sample[1], pw[2] - sample[2])
            fh = hr.FingerHand(p.finger_width, p.hand_outer_diameter, p.hand_depth, p.num_finger_placements)
            assert fh.fs[17] < y < fh.fs[17] + fh.fw and not fh.fs[16] + fh.fw > y   # right slot 7 only
            if pred == "crop":
                assert z == cl["z"] and (-p.hand_height < z < p.hand_height) == cl["kept"], (z, cl)
            else:
                assert x == cl["x"] and -p.hand_height < z < p.hand_height, (x, z, cl)
            r = recs[i][j]
            if cl["finger_idx"] is None:
                assert r is None, (case["name"], i)
            else:
                assert r is not None and r["finger_idx"] == cl["finger_idx"], (case["name"], i, r and r["finger_idx"], cl)
        else:
            assert recs[i][j] is not None, (case["name"], i)
            assert bool(flags[i, j] & abi.POSE_FILTERED) == cl["filtered"], (case["name"], cl, flags[i, j])
            if pred == "direction":
                dot, angle = hr.direction_angle(p, recs[i][j])
                assert dot == cl["dot"], (dot, cl)


@pytest.mark.parametrize("var", list(hc.VARIANTS))
@pytest.mark.parametrize("case", hc.geometry_cases(), ids=lambda c: c["name"])
def test_geometry_cases_oracle_equals_restatement_and_reach_their_edges(case, var):
    case = hc.variant(case, var)
    check_claims(case, *assert_oracle_equals_restatement(case))


def test_filter_cases_oracle_equals_restatement_and_reach_their_edges():
    cases = hc.filter_cases()
    assert len(cases) == 4 + 12 + 1
    for case in cases:
        check_claims(case, *assert_oracle_equals_restatement(case))


def test_direction_cases_oracle_equals_restatement_and_reach_their_edges():
    cases = hc.direction_cases()
    for case in cases:
        check_claims(case, *assert_oracle_equals_restatement(case))
    # each sweep straddles its switch point: kept at d* and above, rejected below
    for t in hc.SWEEP_THRESH:
        ds = hr.d_star(t)
        assert not (math.acos(ds) > t) and math.acos(hr.ulp_step(ds, -1)) > t, t


def test_d_star_is_the_switch_of_the_host_acos():
    """d* (the kernel's comparison value) against acos itself, over the sweep and at the special thresholds."""
    rng = np.random.default_rng(5)
    for t in list(rng.uniform(0.0, math.pi, 200)) + hc.SWEEP_THRESH:
        ds = hr.d_star(t)
        for k in range(-8, 8):
            d = hr.ulp_step(ds, k)
            assert hr.direction_rejects_kernel(d, ds) == (math.acos(d) > t), (t, k)
    assert hr.d_star(-0.1) == 2.0 and hr.d_star(math.pi) == -1.0 and hr.d_star(4.0) == -1.0
    assert hr.d_star(math.nan) == -1.0
    for d in (1.5, hr.ulp_step(1.0, 1), -2.0, math.nan):
        assert not hr.direction_rejects_kernel(d, hr.d_star(0.3)) and not hr.direction_rejects_kernel(d, 2.0)


def _differs(case, fault):
    p = params(case)
    _, _, _, poses, flags, recs, rflags = hr.run_case(case, p)
    _, _, _, _, _, frecs, fflags = hr.run_case(case, p, fault)
    if not np.array_equal(rflags, fflags):
        return True
    for a, b in zip(recs, frecs):
        for r, f in zip(a, b):
            if (r is None) != (f is None):
                return True
            if r is not None and any(r[k] != f[k] for k in FIELDS + ("position", "half", "full")):
                return True
    return False


def test_every_fault_is_caught_by_a_case():
    cases = hc.geometry_cases() + hc.filter_cases() + hc.direction_cases(thresholds=[0.3], half=2)
    caught = {}
    for fault in hr.FAULTS:
        for case in cases:
            if _differs(case, fault):
                caught[fault] = case["name"]
                break
    print("\n".join(f"{f}: {caught.get(f, 'NOT CAUGHT')}" for f in hr.FAULTS))
    assert sorted(caught) == sorted(hr.FAULTS), sorted(set(hr.FAULTS) - set(caught))
