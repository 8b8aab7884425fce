"""gpdb_reevaluate_batch[_device] (-m gpu): HandSearch::reevaluateHypotheses for every cloud of a batch in one k_label
launch. The candidates of several synthetic camera views are labelled against ground-truth clouds of the same scenes
(four cameras, every camera marked); each group must be bit-equal to gpdb_reevaluate with its cloud installed alone, and
equal to the CPU oracle. Also: the closing-region list of k_label at its exact capacity (1 024 members) and one past it,
the grid-walking tier on a dense unvoxelised ground truth, records gpdb_reevaluate labels 0 without a walk, the device
twin, errors and the store left as it was."""
import ctypes as C

import numpy as np
import pytest

import capacity_cases as cc
from conftest import load_weights
from gpd_b200 import lib, scenes
from oracle import oracle

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
CAMS4 = np.array([[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.6, 0.0, 0.0], [0.0, 0.6, 0.0]])
N = 20000
WIDE = [-10.0, 10.0, -10.0, 10.0, -10.0, 10.0]
FAR = {"xyz": np.array([[50.0, 50.0, 50.0]], np.float32), "normals": np.array([[0.0, 0.0, 1.0]]),
       "cam_source": np.ones((1, 1), np.int32), "view_points": np.zeros((1, 3))}


def gt_pp(**over):
    """Installs ground-truth clouds as given (voxelize = 0, their own normals, a workspace that keeps every point)."""
    return lib.preprocess_params(**{"voxelize": 0, "estimate_normals": 0, "workspace": WIDE, **over})


def candidates(p, cloud, n_samples=200):
    ctx = lib.Context(p)
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    c = ctx.hand_search(np.random.default_rng(len(cloud["xyz"])).choice(len(cloud["xyz"]), n_samples, replace=False)
                        .astype(np.int32))["candidates"]
    ctx.close()
    return c


@pytest.fixture(scope="module")
def world():
    """Params, three ground-truth clouds (seeds 3, 4, 5 seen by four cameras) and the candidates of one camera's view of
    each scene."""
    p = lib.default_params(channels=15)
    gts, cands = [], []
    for s in (3, 4, 5):
        view = scenes.synthetic_table_scene(s, n_points=N)
        gts.append(scenes.synthetic_table_scene(s, n_points=N, cameras=CAMS4, mark_all_cameras=True))
        cands.append(candidates(p, view))
        assert len(cands[-1]) > 50
    return p, gts, cands


def single(p, clouds, groups):
    """gpdb_reevaluate of every group with its cloud installed alone (an empty cloud: a cloud with no point near any
    hand, which is what an empty cloud is to the ball search)."""
    ctx = lib.Context(p)
    out = []
    for c, h in zip(clouds, groups):
        c = FAR if len(c["xyz"]) == 0 else c
        ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        out.append(ctx.reevaluate(h))
    ctx.close()
    return out


def assert_groups_equal(got_labels, got_recs, want):
    for g, (lb, rec, (lw, rw)) in enumerate(zip(got_labels, got_recs, want)):
        assert np.array_equal(lb, lw), g
        assert rec.tobytes() == rw.tobytes(), g


def edge_batch(gts, cands):
    """Raw ground-truth clouds and hand groups: two scenes, a thinned copy of the second (which must change labels), an
    empty cloud (its one point lies outside the workspace), an empty group, and a group of another view's hands."""
    g1 = gts[1]
    keep = np.arange(len(g1["xyz"])) % 4 != 1
    thin = {k: (v[keep] if k != "view_points" else v) for k, v in g1.items()}
    empty = dict(FAR, xyz=np.array([[0.0, 0.0, 50.0]], np.float32))
    clouds = [gts[0], g1, thin, empty, gts[2], gts[2]]
    groups = [cands[0], cands[1], cands[1], cands[0][:20], cands[2][:0], cands[0]]
    return clouds, groups


def test_batch_equals_single_and_the_oracle(world):
    p, gts, cands = world
    raw, groups = edge_batch(gts, cands)
    ctx = lib.Context(p)
    ctx.preprocess_clouds(raw, pp=gt_pp(), read_back=False)
    clouds = ctx.get_clouds()
    assert len(clouds[3]["xyz"]) == 0 and len(clouds[2]["xyz"]) < len(clouds[1]["xyz"])
    labels, recs = ctx.reevaluate_batch(groups)
    want = single(p, clouds, groups)
    assert_groups_equal(labels, recs, want)
    # the thinner cloud changes some labels; the empty cloud and the empty group label nothing
    assert any(not np.array_equal(recs[1][f], recs[2][f]) for f in ("half_antipodal", "full_antipodal"))
    assert not labels[3].any() and not recs[3]["half_antipodal"].any() and len(labels[4]) == 0
    for g in (0, 1, 2, 5):
        oc = oracle.OracleCloud(clouds[g]["xyz"], clouds[g]["normals"], clouds[g]["cam_source"], clouds[g]["view_points"])
        lo, ho = oc.reevaluate(p, groups[g])
        assert np.array_equal(lo, labels[g]), g
        for f in ("half_antipodal", "full_antipodal"):
            assert np.array_equal(ho[f], recs[g][f]), (g, f)
    ctx.close()


def test_device_twin_across_contexts_and_streams(world):
    """Context A holds the views and finds the candidates on the device; context B holds the ground truth, installed
    once, and labels A's record tensor in place, on the current and on a side stream, bit-equal to the host twin."""
    import torch
    p, gts, cands = world
    views = [scenes.synthetic_table_scene(s, n_points=N) for s in (3, 4, 5)]
    a = lib.Context(p)
    a.set_clouds(views)
    sidx = [np.random.default_rng(b).choice(N, 150, replace=False).astype(np.int32) for b in range(3)]
    soff, idx = lib.pack_samples(sidx)
    rec, _, hoff = a.hand_search_batch_tensors(soff, torch.from_numpy(idx).cuda())
    host = lib.poses_from_tensor(rec)
    b = lib.Context(p)
    b.set_clouds(gts)
    lw, rw = b.reevaluate_batch([host[hoff[g]:hoff[g + 1]] for g in range(3)])
    for stream in (None, torch.cuda.Stream()):
        t = rec.clone()
        if stream is None:
            labels = b.reevaluate_batch_tensors(hoff, t)
        else:
            stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(stream):
                labels = b.reevaluate_batch_tensors(hoff, t)
            torch.cuda.current_stream().wait_stream(stream)
        assert labels.dtype == torch.int32 and labels.is_cuda
        assert np.array_equal(labels.cpu().numpy(), np.concatenate(lw))
        assert lib.poses_from_tensor(t).tobytes() == np.concatenate(rw).tobytes()
    assert np.concatenate(lw).any()
    # the same error codes as the host twin
    L = lib.lib()
    bad = np.array([0, 5, 3, int(hoff[-1])], np.int32)
    for fn, h_ptr, l_ptr in ((L.gpdb_reevaluate_batch, host.ctypes.data_as(C.c_void_p), np.zeros(len(host), np.int32).ctypes.data_as(C.c_void_p)),
                             (L.gpdb_reevaluate_batch_device, C.c_void_p(rec.data_ptr()), C.c_void_p(labels.data_ptr()))):
        assert fn(b.h, bad.ctypes.data_as(C.c_void_p), h_ptr, l_ptr) == ERR_INVALID
    # a host pointer where a device array belongs
    lab = np.zeros(len(host), np.int32)
    assert L.gpdb_reevaluate_batch_device(b.h, hoff.ctypes.data_as(C.c_void_p), host.ctypes.data_as(C.c_void_p),
                                          lab.ctypes.data_as(C.c_void_p)) == ERR_INVALID
    assert "not device memory" in L.gpdb_last_error(b.h).decode()
    a.close()
    b.close()


def test_errors_leave_outputs_and_store_untouched(world):
    p, gts, cands = world
    L = lib.lib()
    ctx = lib.Context(p)
    with pytest.raises(lib.GpdbError) as e:
        ctx.reevaluate_batch([])
    assert e.value.code == ERR_STATE
    ctx.set_cloud(gts[0]["xyz"], gts[0]["normals"], gts[0]["cam_source"], gts[0]["view_points"])  # a single cloud is no batch
    with pytest.raises(lib.GpdbError) as e:
        ctx.reevaluate_batch([cands[0]])
    assert e.value.code == ERR_STATE
    assert L.gpdb_reevaluate_batch_device(ctx.h, None, None, None) == ERR_STATE

    w, _ = load_weights(15)
    ctx.set_weights(w)
    views = [scenes.synthetic_table_scene(s, n_points=N) for s in (3, 4)]  # one camera: the SIS call makes 15-channel images
    ctx.set_clouds(views)
    ctx.set_clouds_samples([views[0]["xyz"][:5].astype(np.float64) + 0.001, np.zeros((0, 3))])
    hands = np.ascontiguousarray(np.concatenate([cands[0], cands[1]]))
    before = hands.tobytes()
    labels = np.full(len(hands), 7, np.int32)
    n0 = len(cands[0])
    for off in ([1, n0, len(hands)], [0, n0 + 1, n0], [0, -1, len(hands)]):
        o = np.array(off, np.int32)
        assert L.gpdb_reevaluate_batch(ctx.h, o.ctypes.data_as(C.c_void_p), hands.ctypes.data_as(C.c_void_p),
                                       labels.ctypes.data_as(C.c_void_p)) == ERR_INVALID
        assert hands.tobytes() == before and (labels == 7).all()
    o = np.array([0, n0, len(hands)], np.int32)
    assert L.gpdb_reevaluate_batch(ctx.h, o.ctypes.data_as(C.c_void_p), None, None) == ERR_INVALID
    assert L.gpdb_reevaluate_batch(ctx.h, None, None, None) == ERR_INVALID

    # the store: the clouds, the sample positions (they still address the same hands) and the SIS record
    sidx = [np.array([0, 7, N, N + 4], np.int32), np.array([3, 9], np.int32)]
    det = ctx.hand_search_batch(sidx)
    clouds = ctx.get_clouds()
    ctx.reevaluate_batch([cands[0], cands[1]])
    for c0, c1 in zip(clouds, ctx.get_clouds()):
        for k in ("xyz", "normals", "cam_source", "view_points"):
            assert np.array_equal(c0[k], c1[k]), k
    for v0, v1 in zip(det, ctx.hand_search_batch(sidx)):
        assert v0["candidates"].tobytes() == v1["candidates"].tobytes()
    sis = ctx.sis_batch([np.arange(0, 2000, 40, dtype=np.int32), np.arange(0, 2000, 50, dtype=np.int32)],
                        num_iterations=2, num_samples_per_iteration=20)
    ctx.reevaluate_batch([cands[0], cands[1]])
    again = ctx.sis_positions()
    for k in ("evaluated", "kept"):
        assert all(np.array_equal(x, y) for x, y in zip(sis[k], again[k])), k
    assert np.array_equal(sis["round_counts"], again["round_counts"])
    ctx.close()


def test_records_without_a_walk_label_zero(world):
    """finger_idx -1 or nfp, or a NaN sample: gpdb_reevaluate gives label 0 and clears both flags; the batch call gives
    the same, in every group."""
    p, gts, cands = world
    c = cands[0][:6].copy()
    c["half_antipodal"] = 1
    c["full_antipodal"] = 1
    c["finger_idx"][0:2] = -1
    c["finger_idx"][2:4] = p.num_finger_placements
    c["sample"][4:6, 1] = np.nan
    want = single(p, gts[:2], [c, c])
    for lw, rw in want:
        assert not lw.any() and not rw["half_antipodal"].any() and not rw["full_antipodal"].any()
    ctx = lib.Context(p)
    ctx.set_clouds(gts[:2])
    labels, recs = ctx.reevaluate_batch([c, c])
    assert_groups_equal(labels, recs, want)
    ctx.close()


def closing_hands(n):
    """The cylinder of capacity_cases.hand_cylinder(n) and the valid hands of its sample: every one holds exactly n
    closing-region members (counted in float64 as k_hands' list is)."""
    cloud, si = cc.hand_cylinder(n)
    p = lib.default_params(hand_axes=[2], num_orientations=8)
    ctx = lib.Context(p)
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    r = ctx.hand_search(np.array([si], np.int32))
    ctx.close()
    hands = r["candidates"]
    assert len(hands) > 0
    assert (cc.closing_counts(cloud, si, hands, np.ones(len(hands), np.int32)) == n).all()
    return p, cloud, hands


def counted(ctx, call, *args):
    ctx.phase_cycles(1)
    out = call(*args)
    k = ctx.path_counts()["label_walk"]
    ctx.phase_cycles(0)
    return out, k


@pytest.mark.parametrize("n", [cc.SURV_CAP, cc.SURV_CAP + 1])
def test_closing_region_list_capacity(n):
    """At 1 024 members the Antipodal passes read the list, at 1 025 they walk the grid (path counter 15); both equal
    the oracle, alone and as the middle group of a three-group call."""
    p, cloud, hands = closing_hands(n)
    ctx = lib.Context(p)
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    (l1, h1), k1 = counted(ctx, ctx.reevaluate, hands[:1])
    assert k1 == (1 if n > cc.SURV_CAP else 0)
    (la, ha), ka = counted(ctx, ctx.reevaluate, hands)
    assert ka == (len(hands) if n > cc.SURV_CAP else 0)
    lo, ho = oc.reevaluate(p, hands)
    assert np.array_equal(lo, la) and np.array_equal(l1, la[:1])
    for f in ("half_antipodal", "full_antipodal"):
        assert np.array_equal(ho[f], ha[f]), f
    assert ha["half_antipodal"].any()
    k = scenes.krylon_cloud()
    kh = candidates(p, k, 100)
    want, ks = [], []
    for c, h in ((k, kh[:40]), (cloud, hands), (k, kh[40:])):
        ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        out, kc = counted(ctx, ctx.reevaluate, h)
        want.append(out)
        ks.append(kc)
    ctx.set_clouds([k, cloud, k])
    (labels, recs), kb = counted(ctx, ctx.reevaluate_batch, [kh[:40], hands, kh[40:]])
    assert kb == sum(ks) and ks[1] == ka
    assert_groups_equal(labels, recs, want)
    ctx.close()


def test_dense_unvoxelised_ground_truth_walks_and_equals_the_oracle(world):
    """A 2 mm unvoxelised ground truth (normals estimated on the device): some closing regions hold more than 1 024
    points, and the labels of both tiers equal the oracle's."""
    p, gts, cands = world
    raw = scenes.synthetic_raw_scene(5, n_points=N, step=0.002, cameras=CAMS4, mark_all_cameras=True)
    ctx = lib.Context(p)
    gt = ctx.preprocess_clouds([raw], pp=lib.preprocess_params(voxelize=0, workspace=WIDE))[0]
    (labels, recs), k = counted(ctx, ctx.reevaluate_batch, [cands[2]])
    assert 0 < k < len(cands[2]), k
    oc = oracle.OracleCloud(gt["xyz"], gt["normals"], gt["cam_source"], gt["view_points"])
    lo, ho = oc.reevaluate(p, cands[2])
    assert np.array_equal(lo, labels[0])
    for f in ("half_antipodal", "full_antipodal"):
        assert np.array_equal(ho[f], recs[0][f]), f
    assert labels[0].any()
    ctx.close()
