"""k_frames / k_hands on the cases of hand_cases.py (-m gpu): the height crop, init_bite and back edges, the aperture and
workspace bounds and the direction filter. Frames, the flags of every pose and every field of every candidate record
equal the oracle bit for bit (test_hand_cases.py proves on the CPU that the oracle equals the
exact restatement and that each case sits on its edge). The direction filter is swept over the doubles around the
switch point of acos(dot) > thresh at several thresholds, and past |dot| = 1. The geometry cases also run as the middle
cloud of a three-cloud batch (k_frames<true> / k_hands<true>) and through gpdb_detect in small chunks with the hand
search overlapped and not."""
import numpy as np
import pytest

import hand_cases as hc
import hand_reference as hr
from conftest import load_weights
from gpd_b200 import abi, lib

pytestmark = pytest.mark.gpu

FIELDS = ("frame", "position", "top", "bottom", "center", "width", "finger_idx", "half_antipodal", "full_antipodal",
          "sample", "sample_index", "sample_slot", "pose_slot")


def on_device(case, p, weights=None):
    ctx = lib.Context(p)
    if weights is not None:
        ctx.set_weights(weights)
    c = case["cloud"]
    ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    sidx = hr.case_samples(case, ctx)
    return ctx, sidx


def mismatches(case, p):
    """Poses whose flags differ from the oracle's; frames and candidate records must match exactly regardless."""
    sidx_o, fo, vo, po, flo, _, _ = hr.run_case(case, p)
    ctx, sidx = on_device(case, p)
    assert np.array_equal(sidx, sidx_o)
    rg = ctx.hand_search(sidx)
    ctx.close()
    assert np.array_equal(rg["frame_valid"], vo) and np.array_equal(rg["frames"].reshape(-1, 9), fo), case["name"]
    fg = rg["pose_flags"].reshape(flo.shape)
    bad = np.argwhere(fg != flo)
    if len(bad) == 0:
        cand_o = po.ravel()[(flo.ravel() & 3) == 3]
        assert rg["n_candidates"] == len(cand_o)
        for f in FIELDS:
            assert np.array_equal(rg["candidates"][f], cand_o[f]), (case["name"], f)
    return [(case["name"], int(i), int(j), int(fg[i, j]), int(flo[i, j])) for i, j in bad]


@pytest.mark.parametrize("case", [hc.variant(c, v) for c in hc.geometry_cases() for v in hc.VARIANTS] + hc.filter_cases(),
                         ids=lambda c: c["name"])
def test_hand_search_at_the_edges_equals_the_oracle(case):
    p = abi.default_params(15, **case["over"])
    assert mismatches(case, p) == []


def test_direction_filter_at_the_acos_switch_equals_the_oracle():
    """At 14 thresholds, every dot within 100 doubles of the switch point and the switch points of the thresholds 8 angle
    ulps either side (hand_cases.sweep_dots); |dot| > 1, +-1 and the special thresholds: the FILTERED flag is the
    host's acos(dot) > thresh."""
    cases = hc.direction_cases()
    bad = []
    for case in cases:
        bad += mismatches(case, abi.default_params(15, **case["over"]))
    print(f"{len(cases)} direction cases, {len(bad)} flag mismatches")
    assert bad == [], bad[:20]


def _point_samples(case):
    return [s for kind, s in case["samples"] if kind == "point"]


def test_geometry_cases_as_the_middle_cloud_of_a_batch():
    """The cloud-point samples of every geometry case, detected as cloud 1 of three, equal the case's cloud alone.
    Batches take cloud points only (no gpdb_set_samples positions): the float64-ulp edges run in single-cloud calls,
    their float32-step twins here."""
    w, _ = load_weights(15)
    other = hc.single_object().case("other")
    for case in hc.geometry_cases():
        pts = _point_samples(case)
        if not pts:
            continue
        p = abi.default_params(15, **case["over"])
        ctx, _ = on_device(case, p, w)
        one = ctx.detect(np.array(pts, np.int32))
        ctx.set_clouds([other["cloud"], case["cloud"], other["cloud"]])
        views = ctx.detect_batch([[4], pts, [4]])
        ctx.close()
        mid = views[1]
        assert np.array_equal(mid["pose_flags"], one["pose_flags"]) and np.array_equal(mid["frames"], one["frames"])
        assert mid["n_candidates"] == one["n_candidates"]
        for f in FIELDS:
            assert np.array_equal(mid["candidates"][f], one["candidates"][f]), (case["name"], f)


@pytest.mark.parametrize("overlap", [1, 0])
def test_detect_in_small_chunks_gives_the_hand_search_flags(overlap):
    """gpdb_detect with chunk_samples 2, the hand search of the next chunk overlapped or not: the same flags and candidate
    records as gpdb_hand_search (results are identical either way)."""
    w, _ = load_weights(15)
    for case in hc.geometry_cases():
        p = abi.default_params(15, **case["over"])
        ctx, sidx = on_device(case, p, w)
        hs = ctx.hand_search(sidx)
        ctx.close()
        p2 = abi.default_params(15, chunk_samples=2, **case["over"])
        ctx, sidx2 = on_device(case, p2, w)
        ctx.set_overlap(overlap)
        rd = ctx.detect(sidx2)
        ctx.close()
        assert np.array_equal(sidx, sidx2)
        assert np.array_equal(rd["pose_flags"], hs["pose_flags"]), case["name"]
        assert np.array_equal(rd["frames"], hs["frames"]), case["name"]
        assert rd["n_candidates"] == hs["n_candidates"] > 0
        for f in FIELDS:
            assert np.array_equal(rd["candidates"][f], hs["candidates"][f]), (case["name"], f)
