"""gpdb_sis_batch / gpdb_sis_batch_device: SequentialImportanceSampling::detectGrasps on the device.

The oracle of a call is the library's existing batch calls fed with the positions the call exports (replay): the initial
hand search, then gpdb_set_clouds_samples + gpdb_hand_search_batch per round must give the kept positions bit for bit and
in order, and gpdb_set_clouds_samples(kept) + gpdb_detect_batch + the score filter + gpdb_find_clusters_batch the records
byte for byte. The draws themselves are held against the numpy restatement of include/gpd_b200_sis.h (sis_reference.py).
"""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

import sis_reference as sr
from conftest import load_weights
from gpd_b200 import abi, lib, scenes
from oracle import oracle
from test_gpu_batch import outside_workspace, table
from test_gpu_parity import assert_parity

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
WS = [-1, 1, -1, 1, -1, 1]


def context(ch=15, **over):
    w, relu = load_weights(ch)
    p = lib.default_params(channels=ch, relu_after_conv=relu, **over)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    return p, ctx, oracle.WeightPack(w)


def inits(clouds, n, seed):
    rng = np.random.default_rng(seed)
    return [rng.choice(len(c["xyz"]), min(n, len(c["xyz"])), replace=False).astype(np.int32) for c in clouds]


def scenario():
    """krylon, a two-camera table, a cloud with an empty initial list, a cloud far outside the grasp workspace (inactive:
    its initial search finds no hand) and a plain table."""
    clouds = [scenes.krylon_cloud(), table(4, n=8000, two_cameras=True), table(5, n=6000), outside_workspace(),
              table(6, n=8000)]
    init = inits(clouds, 40, 1)
    init[2] = np.zeros(0, np.int32)
    return clouds, init


def hand_set_positions(view):
    c = view["candidates"]
    _, first = np.unique(c["sample_slot"], return_index=True)
    return c["sample"][np.sort(first)].astype(np.float64)


def replay(ctx, clouds, init, sis, res):
    """Feeds the exported positions through the existing batch calls; returns the kept positions at the start of every
    round (for the generator checks) after asserting the kept set and the records."""
    B, R = len(clouds), sis.get("num_iterations", 5)
    pos = ctx.sis_positions()
    kept = [hand_set_positions(v) for v in ctx.hand_search_batch(init)]
    starts = []
    ro = [np.concatenate([[0], np.cumsum(pos["round_counts"][b])]) for b in range(B)]
    for r in range(R):
        starts.append([k.copy() for k in kept])
        rp = [pos["evaluated"][b][ro[b][r]:ro[b][r + 1]] for b in range(B)]
        for b, v in enumerate(ctx.hand_search_batch(ctx.set_clouds_samples(rp))):
            kept[b] = np.vstack([kept[b], hand_set_positions(v)])
    for b in range(B):
        assert kept[b].tobytes() == pos["kept"][b].tobytes(), f"cloud {b}: kept positions"
    assert res["n_samples"] == sum(len(k) for k in kept)
    det = [v["candidates"] for v in ctx.detect_batch(ctx.set_clouds_samples(kept))]
    ms = sis.get("min_score", 0.0)
    filt = [d[d["score"].astype(np.float64) > ms] for d in det]
    mi = sis.get("min_inliers", 1)
    want = ctx.find_clusters_batch(filt, mi) if mi > 0 else filt
    for b in range(B):
        assert res["hands"][b].tobytes() == want[b].tobytes(), f"cloud {b}: records"
    assert res["n_total_candidates"] == sum(len(d) for d in det)
    return starts, pos, det


def check_generator(clouds, init, sis, starts, pos):
    """Every round's positions against the restatement: parents and uniform points exactly, offsets to 1e-13."""
    B = len(clouds)
    S, R = sis.get("num_samples_per_iteration", 50), sis.get("num_iterations", 5)
    sigma, seed = sis.get("standard_deviation", 0.02), sis.get("seed", 0)
    for b in range(B):
        ro = np.concatenate([[0], np.cumsum(pos["round_counts"][b])])
        for r in range(R):
            got = pos["evaluated"][b][ro[r]:ro[r + 1]]
            k = starts[r][b]
            if len(k) == 0:
                assert len(got) == 0
                continue
            want, par, ng = sr.draw_round(k, r, seed + b, S, sis.get("prob_rand_samples", 0.3), sigma,
                                          sis.get("sampling_method", 0), sis.get("workspace", WS), clouds[b]["xyz"], init[b])
            assert len(got) == len(want), (b, r)
            assert got[ng:].tobytes() == want[ng:].tobytes()
            tol = 1e-13 * sigma * np.maximum(1.0, np.abs(want[:ng] - k[par]) / sigma) + 2 * np.spacing(np.abs(k[par]))
            assert np.all(np.abs(got[:ng] - want[:ng]) <= tol), (b, r)
            if sis.get("sampling_method", 0) == 1 and ng:  # the device's own positions obey the exact d2 rule
                assert np.all(sr.d2(got[:ng], k[par]) <= sr.d2(got[:ng, None, :], k[None]).min(axis=1))


CASES = {
    "sum-0.3-cl1": dict(),
    "max-0.3-cl3": dict(sampling_method=1, min_inliers=3, seed=7),
    "sum-0-flat": dict(prob_rand_samples=0.0, min_inliers=0, seed=11),
    "max-1-flat": dict(sampling_method=1, prob_rand_samples=1.0, min_inliers=0, num_samples_per_iteration=20),
    "ws-part": dict(workspace="half", prob_rand_samples=0.5, num_iterations=3, seed=3),
    "rounds-0": dict(num_iterations=0),
    "score-low": dict(min_score=-1e9, num_iterations=2),
    "score-high": dict(min_score=1e9, num_iterations=2),
}


@pytest.mark.parametrize("name", list(CASES))
def test_sis_replays_through_the_batch_calls(name):
    sis = dict(CASES[name])
    p, ctx, _ = context()
    clouds, init = scenario()
    if sis.get("workspace") == "half":  # excludes the half of krylon's initial points with the larger x
        sis["workspace"] = [-1, float(np.median(clouds[0]["xyz"][init[0], 0])), -1, 1, -1, 1]
    ctx.set_clouds(clouds)
    res = ctx.sis_batch(init, **sis)
    starts, pos, _ = replay(ctx, clouds, init, sis, res)
    check_generator(clouds, init, sis, starts, pos)
    rc = pos["round_counts"]
    assert rc.shape == (5, sis.get("num_iterations", 5))
    assert np.all(rc[2] == 0) and np.all(rc[3] == 0) and len(res["hands"][3]) == 0  # empty init list, inactive cloud
    if sis.get("num_iterations", 5):
        assert rc[0].sum() > 0
    if name == "score-high":
        assert all(len(h) == 0 for h in res["hands"])
    if name == "score-low":
        assert sum(len(h) for h in res["hands"]) > 0
    ctx.close()


@pytest.mark.parametrize("ch", [12, 15])
def test_min_score_at_a_typical_score(ch):
    """min_score equal to a score that occurs: the hands with exactly that score are dropped (score > min_score)."""
    p, ctx, _ = context(ch)
    clouds, init = scenario()
    ctx.set_clouds(clouds)
    base = ctx.sis_batch(init, min_inliers=0, num_iterations=2)
    s = np.concatenate([h["score"] for h in base["hands"]]).astype(np.float64)
    assert len(s) > 4
    sis = dict(min_inliers=1, num_iterations=2, min_score=float(np.sort(s)[len(s) // 2]))
    res = ctx.sis_batch(init, **sis)
    replay(ctx, clouds, init, sis, res)
    ctx.close()


def test_offsets_are_normal():
    """10^5 Gaussian offsets of the device draws (parents from the restatement) against N(0, sigma)."""
    p, ctx, _ = context()
    k = scenes.krylon_cloud()
    ctx.set_clouds([k])
    init = inits([k], 60, 2)
    sis = dict(num_iterations=1, num_samples_per_iteration=34000, prob_rand_samples=0.0, seed=2024)
    ctx.sis_batch(init, **sis)
    pos = ctx.sis_positions()
    kept0 = hand_set_positions(ctx.hand_search_batch(init)[0])
    par, _ = sr.gaussian(2024, np.arange(34000), 0, len(kept0))
    off = (pos["evaluated"][0] - kept0[par]).ravel() / 0.02
    assert len(off) >= 100000
    assert stats.kstest(off, "norm").pvalue > 1e-3
    ctx.close()


def test_clouds_are_independent_of_the_batch_and_the_pipeline():
    clouds = [table(20 + i, n=8000) for i in range(16)]
    init = inits(clouds, 30, 3)
    sis = dict(num_iterations=3, num_samples_per_iteration=30, seed=1000, min_inliers=1)
    p, ctx, _ = context()
    ctx.set_clouds(clouds)
    ref = ctx.sis_batch(init, **sis)
    assert sum(len(h) for h in ref["hands"]) > 0
    for b in (0, 5, 15):
        ctx.set_clouds([clouds[b]])
        one = ctx.sis_batch([init[b]], **dict(sis, seed=1000 + b))
        assert one["hands"][0].tobytes() == ref["hands"][b].tobytes()
        assert one["kept"][0].tobytes() == ref["kept"][b].tobytes()
        assert one["evaluated"][0].tobytes() == ref["evaluated"][b].tobytes()
    ctx.close()
    for over, overlap in (({"chunk_samples": 64}, 1), ({"chunk_samples": 1000}, 0)):
        p, ctx, _ = context(**over)
        ctx.set_overlap(overlap)
        ctx.set_clouds(clouds)
        r = ctx.sis_batch(init, **sis)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(r["hands"], ref["hands"]))
        assert all(a.tobytes() == b.tobytes() for a, b in zip(r["kept"], ref["kept"]))
        ctx.close()


def test_device_twin_is_bit_equal_also_on_a_side_stream():
    import torch
    p, ctx, _ = context()
    clouds, init = scenario()
    ctx.set_clouds(clouds)
    for sis in (dict(), dict(sampling_method=1, min_inliers=0, seed=5)):
        host = ctx.sis_batch(init, **sis)
        off, idx = lib.pack_samples(init)
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            d_idx = torch.from_numpy(idx).cuda()
            rec, hoff, st = ctx.sis_batch_tensors(off, d_idx, **sis)
            recs = lib.poses_from_tensor(rec)
        for b in range(len(clouds)):
            assert recs[hoff[b]:hoff[b + 1]].tobytes() == host["hands"][b].tobytes()
        pos = ctx.sis_positions()
        assert all(a.tobytes() == b.tobytes() for a, b in zip(pos["kept"], host["kept"]))
        assert st["n_samples"] == host["n_samples"] and st["n_total_candidates"] == host["n_total_candidates"]
    # the same errors and messages
    off, idx = lib.pack_samples(init)
    bad_idx = idx.copy()
    bad_idx[off[4] + 3] = len(clouds[4]["xyz"])
    cases = [(dict(standard_deviation=0.0), idx), (dict(prob_rand_samples=1.5), idx), (dict(sampling_method=2), idx),
             (dict(num_iterations=-1), idx), (dict(), bad_idx)]
    for sis, ii in cases:
        with pytest.raises(lib.GpdbError) as eh:
            ctx.sis_batch([ii[off[b]:off[b + 1]] for b in range(len(clouds))], **sis)
        with pytest.raises(lib.GpdbError) as ed:
            ctx.sis_batch_tensors(off, torch.from_numpy(ii).cuda(), **sis)
        assert eh.value.code == ed.value.code == ERR_INVALID
        assert str(eh.value).replace("gpdb_sis_batch", "X") == str(ed.value).replace("gpdb_sis_batch_device", "X")
    hoff = np.zeros(len(off), np.int32)  # a host pointer where device memory is required
    rc = lib.lib().gpdb_sis_batch_device(ctx.h, C.byref(lib.sis_params()), lib._p(off), lib._p(idx), None, lib._p(hoff),
                                         C.byref(abi.Result()))
    assert rc == ERR_INVALID and b"d_init_idx is not device memory" in lib.lib().gpdb_last_error(ctx.h)
    ctx.close()


def test_state_after_the_call():
    p, ctx, w = context()
    clouds, init = scenario()
    k = clouds[0]
    ctx.set_cloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    single = ctx.detect(init[0])
    ctx.set_clouds(clouds)
    sis = dict(num_iterations=2)
    res = ctx.sis_batch(init, **sis)
    # the batch holds the kept positions: gpdb_detect_batch at N_b + j is the final step
    n = [len(c["xyz"]) for c in clouds]
    det = ctx.detect_batch([n[b] + np.arange(len(res["kept"][b]), dtype=np.int32) for b in range(len(clouds))])
    _, _, det_replay = replay(ctx, clouds, init, sis, res)
    assert all(a["candidates"].tobytes() == b.tobytes() for a, b in zip(det, det_replay))
    # the single cloud is untouched
    assert ctx.detect(init[0])["candidates"].tobytes() == single["candidates"].tobytes()
    # a failed call leaves no positions, and no SIS positions to read back
    bad = [i.copy() for i in init]
    bad[0][0] = -1
    with pytest.raises(lib.GpdbError) as e:
        ctx.sis_batch(bad, **sis)
    assert e.value.code == ERR_INVALID and "init index -1 at position 0 outside cloud 0" in str(e.value)
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect_batch([[n[0]], [], [], [], []])
    assert e.value.code == ERR_INVALID
    with pytest.raises(lib.GpdbError) as e:
        ctx.sis_positions()
    assert e.value.code == ERR_STATE
    ctx.close()
    # weights are required
    q = lib.Context(lib.default_params(channels=15))
    q.set_clouds(clouds)
    with pytest.raises(lib.GpdbError) as e:
        q.sis_batch(init)
    assert e.value.code == ERR_STATE
    q.close()


def test_kept_positions_against_the_oracle():
    p, ctx, w = context()
    k, t = scenes.krylon_cloud(), table(3, n=6000)
    ctx.set_clouds([k, t])
    init = inits([k, t], 30, 9)
    res = ctx.sis_batch(init, num_iterations=2, num_samples_per_iteration=20, min_inliers=0)
    kept = res["kept"]
    assert len(kept[0]) > 0
    views = ctx.detect_batch(ctx.set_clouds_samples(kept))
    for b, c in enumerate((k, t)):
        oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        sidx = oc.set_samples(kept[b])
        assert_parity(oc.detect(p, w, sidx), views[b], 15)
    ctx.close()


def test_positions_are_dropped_by_a_new_batch():
    """gpdb_sis_positions describes the batch of the last SIS call: any install after it (smaller or larger batch, host or
    device, set or preprocess) leaves nothing to read, and the library writes nothing into the caller's arrays."""
    import torch
    p, ctx, _ = context()
    clouds = [table(20 + i, n=8000) for i in range(16)]
    init = inits(clouds, 30, 4)
    raw = [{"xyz": c["xyz"], "view_points": c["view_points"]} for c in clouds[:2]]
    off = np.array([0, len(clouds[0]["xyz"])], np.int32)
    reinstalls = [
        lambda: ctx.set_clouds(clouds[:1]),
        lambda: ctx.set_clouds(clouds + clouds[:4]),
        lambda: ctx.preprocess_clouds(raw, read_back=False),
        lambda: ctx.set_clouds_tensors(off, torch.from_numpy(clouds[0]["xyz"]).cuda(),
                                       torch.from_numpy(np.ascontiguousarray(clouds[0]["normals"], np.float64)).cuda(),
                                       [len(clouds[0]["view_points"])], clouds[0]["view_points"]),
    ]
    for reinstall in reinstalls:
        ctx.set_clouds(clouds)
        res = ctx.sis_batch(init, num_iterations=2, num_samples_per_iteration=20)
        assert len(res["kept"]) == 16 and sum(len(k) for k in res["kept"]) > 0
        reinstall()
        with pytest.raises(lib.GpdbError) as e:
            ctx.sis_positions()
        assert e.value.code == ERR_STATE
        # the raw call with arrays sized for one cloud: refused before any write
        eoff, koff, rcount = np.full(2, -7, np.int32), np.full(2, -7, np.int32), np.full(2, -7, np.int32)
        rc = lib.lib().gpdb_sis_positions(ctx.h, lib._p(eoff), lib._p(rcount), None, lib._p(koff), None)
        assert rc == ERR_STATE and np.all(eoff == -7) and np.all(koff == -7) and np.all(rcount == -7)
    # after a SIS call on the new batch, the positions have its shape
    ctx.set_clouds(clouds[:3])
    res = ctx.sis_batch(init[:3], num_iterations=2, num_samples_per_iteration=20)
    assert res["round_counts"].shape == (3, 2) and len(res["kept"]) == 3
    # a call that fails its checks after a successful one leaves nothing to read either
    with pytest.raises(lib.GpdbError):
        ctx.sis_batch(init[:3], standard_deviation=-1.0)
    with pytest.raises(lib.GpdbError) as e:
        ctx.sis_positions()
    assert e.value.code == ERR_STATE
    ctx.close()
