"""The image stage's output at its edges, on the CPU: the oracle equals the reference-mode restatement
(tests/image_reference.py) bit for bit on every case of tests/image_cases.py, each case reaches what it claims, and
each emulated kernel fault of image_reference.FAULTS changes a pixel of a named case against the fault-free kernel mode
(fault b, which no output can show: the verdict the case was built to reach)."""
import functools

import numpy as np
import pytest

import capacity_cases as cc
import image_cases as ic
import image_reference as ir
from oracle import oracle


@functools.lru_cache(maxsize=None)
def cases():
    return {c["name"]: c for c in ic.all_cases()}


@functools.lru_cache(maxsize=None)
def qtab():
    return oracle.qtab()


@functools.lru_cache(maxsize=None)
def restated(name, i, mode, fault=None):
    case = cases()[name]
    info = {}
    img = ir.image(case["cloud"], case["poses"][i], case["geometry"], mode, fault=fault, qtab=qtab(), info=info)
    return img, info


def test_jitter_table_agrees_with_the_restated_table():
    t, mine = qtab(), ir.norm_quantile_table()
    assert np.all(np.abs(t - mine) <= np.spacing(np.abs(t)))


@pytest.mark.parametrize("name", [c["name"] for c in ic.all_cases()])
def test_oracle_equals_the_reference_restatement(name):
    case = cases()[name]
    c = case["cloud"]
    oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    io = oc.images(ic.params_of(case), case["poses"])
    for i in range(len(case["poses"])):
        ref, _ = restated(name, i, "reference")
        assert np.array_equal(ref, io[i]), (name, i, case["claims"][i], np.argwhere(ref != io[i])[:8])
        assert io[i].max() > 0 or restated(name, i, "reference")[1]["box"] == 0


TIER_BOX = {"images2": (0, cc.BOX_CAP2), "shared": (cc.BOX_CAP2 + 1, cc.BOX_CAP), "gl": (cc.BOX_CAP + 1, cc.BOX_CAP_GL)}


@pytest.mark.parametrize("name", [c["name"] for c in ic.all_cases()])
def test_cases_reach_what_they_claim(name):
    case = cases()[name]
    g = case["geometry"]
    for i, (pose, cl) in enumerate(zip(case["poses"], case["claims"])):
        _, info = restated(name, i, "kernel")
        grp = info["groups"]
        where = (name, i, cl)
        n = cc.box_count(case["cloud"], case["poses"][i:i + 1], g.w, g.d, g.h, g.radius)
        assert n == info["box"], where
        lo, hi = TIER_BOX[cl["tier"]]
        if g.S != 60 and cl["tier"] == "shared":
            lo = 0 if not cl.get("shadow_covered") else lo
        if not cl.get("shadow_covered"):
            assert lo <= n <= hi, (where, n)
        for k, v in cl.get("covered", {}).items():
            assert grp[k]["covered"] == v, (where, k, grp[k])
        for k in cl.get("min_positive", []):
            assert grp[k]["min"] > 0, (where, k, grp[k])
        for k in cl.get("constant", []):
            assert grp[k]["constant"] and grp[k]["covered"] and grp[k]["max"] > 0, (where, k, grp[k])
        for k in cl.get("min_zero_max_constant", []):
            assert grp[k]["min"] == 0 and grp[k]["max"] == grp[(k[0], k[1])]["max"] > 0, (where, k, grp[k])
        for k in cl.get("tiny", []):
            assert 0 < grp[k]["max"] - grp[k]["min"] <= ir.DBL_EPSILON, (where, k, grp[k])
        if cl.get("nonunit"):
            assert info["nonunit"], where
        if cl.get("shadow_covered"):
            assert all(grp[(pj, "s")]["covered"] and grp[(pj, "s")]["min"] > 0 for pj in range(3)), (where, grp)
        if "stack_counts" in cl:
            pix = (g.S - 1 - info["cells"][:, 0]) * g.S + info["cells"][:, 1]
            assert sorted(np.bincount(pix)[np.bincount(pix) > 0]) == sorted(cl["stack_counts"]), where
        if "boundary" in cl:
            axis, k, rel = cl["boundary"]
            ref_info = restated(name, i, "reference")[1]
            assert np.array_equal(info["cells"], ref_info["cells"]), where   # unit_axis gives the reference's cells
            got = info["cells"][info["box_index"] == info["box_index"].min(), axis][0]
            assert got in (k - 1, k), (where, got)
        if "face" in cl:
            axis, upper, rel = cl["face"]
            faulty = restated(name, i, "kernel", "h")[1]
            if rel == 0:   # on the face: excluded, and included by non-strict faces
                assert faulty["box"] == info["box"] + 1, where
            else:          # 1 ulp inside: included either way
                assert faulty["box"] == info["box"] >= 1, where
        if "fault_e" in cl:   # the reciprocal product alone puts the point in another cell than unit_axis
            k = np.flatnonzero(info["box_index"] == info["box_index"].min())[0]
            axis = cl["fault_e"]
            assert info["cells"][k, axis] != restated(name, i, "kernel", "e")[1]["cells"][k, axis], where
        if cl.get("saturate"):   # strictly inside the box with u = 1: q = 2^32 - 1, cell S - 1
            k = np.flatnonzero(info["box_index"] == info["box_index"].min())[0]
            assert info["units"][k, 0] == 1.0 and info["cells"][k, 0] == g.S - 1, where
    if name == "boundaries":
        assert any("fault_e" in cl for cl in case["claims"]) and any(cl.get("saturate") for cl in case["claims"])
    if name.startswith("boundaries"):
        # both sides of every boundary are reached: the point at the boundary lies in cell k, 1 ulp below in k - 1
        sides = {}
        for i, cl in enumerate(case["claims"]):
            if "boundary" in cl:
                _, info = restated(name, i, "kernel")
                axis, k, rel = cl["boundary"]
                sides.setdefault((axis, k), set()).add(int(info["cells"][info["box_index"] == info["box_index"].min(), axis][0]))
        assert all(s == {k - 1, k} for (axis, k), s in sides.items()), sides


# the case and the claim of its first pose that exposes each emulated fault
FAULT_CASES = {
    "a": ("covered", "min_positive"),       # a covered lattice: its dilated minimum is > 0
    "c": ("covered", "min_positive"),       # rows 1-3 of the 60-wide bitmap straddle three words
    "d": ("nonunit", "tiny"),               # normals of length 1e-40: 0 < max - min <= DBL_EPSILON
    "e": ("boundaries", "fault_e"),         # a tuned boundary where the reciprocal product gives another cell
    "f": ("boundaries", "saturate"),        # u = 1 strictly inside the box: q saturates at 2^32 - 1
    "g": ("stacks_S60", "stack_counts"),    # stacks of 2 to 63 points use the table
    "g2": ("stacks_S60", "stack_counts"),   # the stack of 64 points is the first past the table
    "h": ("boundaries", "face"),            # a point on the lower x face
    "i": ("covered", "min_positive"),       # covered projection 0, then projection 1
}


def fault_pose(fault):
    name, key = FAULT_CASES[fault]
    return name, next(i for i, cl in enumerate(cases()[name]["claims"]) if key in cl)


@pytest.mark.parametrize("fault", sorted(FAULT_CASES))
def test_each_fault_changes_a_pixel(fault):
    name, i = fault_pose(fault)
    good, _ = restated(name, i, "kernel")
    bad, _ = restated(name, i, "kernel", fault)
    assert not np.array_equal(good, bad), (fault, ir.FAULTS[fault])


def test_border_window_fault_flips_the_verdict_only():
    """Fault (b) turns the clipped border windows of the hole cases into occupied ones: the verdict flips to covered,
    and the general path then finds the same minimum 0 (the empty window's dilated value), so no pixel changes. The
    kernels' verdict is an optimisation whose one-sided errors (covered reported as not covered: faults a, c) show."""
    case = cases()["holes"]
    flipped = 0
    for i, cl in enumerate(case["claims"]):
        good, gi = restated("holes", i, "kernel")
        bad, bi = restated("holes", i, "kernel", "b")
        assert np.array_equal(good, bad)
        flipped += int(gi["groups"][(0, "d")]["covered"] != bi["groups"][(0, "d")]["covered"])
    assert flipped == 5   # row 0, row S - 1, column 0, column S - 1 and the corner
