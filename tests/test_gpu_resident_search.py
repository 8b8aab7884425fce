"""Device-resident sample positions, hand search, detection, grasp images and classification of a batch of clouds
(gpdb_set_clouds_samples_device, gpdb_hand_search_batch_device, gpdb_detect_batch_device, gpdb_images_batch_device,
gpdb_classify_device) through the tensor methods of lib.Context.

The oracle of every device route is its host route on the same seeded inputs, bit for bit: the records (cloud-local
sample slots), the per-cloud offsets, the dense flags and the score bit patterns of hand_search_batch / detect_batch, the
images of detect_batch with keep_images = 1 and the scores and logits of classify. The errors must be the host twin's
(code and message, up to the entry point's name). tests/test_abi.py holds the ctypes prototypes of the five calls
against their declarations in include/gpd_b200.h.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import abi, lib, scenes

ERR_INVALID, ERR_STATE = -1, -3
K1 = [(0.0, 0.0, 0.0)]
K2 = [(0.0, 0.0, 0.0), (0.3, 0.0, 0.0)]
K3 = [(0.0, 0.0, 0.0), (0.3, 0.0, 0.0), (-0.3, 0.1, 0.0)]
K8 = [(-0.3, -0.2, 0.0), (0.0, -0.2, 0.0), (0.3, -0.2, 0.0), (-0.3, 0.2, 0.0), (0.0, 0.2, 0.0), (0.3, 0.2, 0.0),
      (0.0, 0.0, 0.0), (0.15, 0.0, 0.1)]


# ---- GPU ---------------------------------------------------------------------------------------------------------------

def torch_():
    return pytest.importorskip("torch")


def context(channels=12, weights=True, **over):
    w, relu = load_weights(channels)
    ctx = lib.Context(lib.default_params(channels=channels, relu_after_conv=relu, **over))
    if weights:
        ctx.set_weights(w)
    return ctx


def dev(a):
    return torch_().from_numpy(np.ascontiguousarray(a)).cuda()


def tables(cams, n=9000, seed=60):
    """One table scene per camera set (K_b = len(cams[b])), all cameras marked."""
    return [scenes.synthetic_table_scene(seed + b, n_points=n, cameras=k, mark_all_cameras=True) for b, k in enumerate(cams)]


def positions_near(cloud, seed, m):
    """m float64 positions a few millimetres off cloud points (Gaussian offsets): most of them carry hands."""
    rng = np.random.default_rng(seed)
    if m == 0:
        return np.zeros((0, 3))
    return cloud["xyz"][rng.choice(len(cloud["xyz"]), m, replace=False)].astype(np.float64) + rng.normal(0, 0.002, (m, 3))


def scenario(clouds, seed=0):
    """Positions in some clouds only, sample lists that mix points and positions, and an empty last sample range."""
    B = len(clouds)
    m = [(25, 0, 15, 8)[b % 4] for b in range(B)]
    pos = [positions_near(c, seed + 10 + b, m[b]) for b, c in enumerate(clouds)]
    samples = []
    for b, c in enumerate(clouds):
        rng = np.random.default_rng(seed + b)
        n = len(c["xyz"])
        s = np.concatenate([rng.choice(n, 40, replace=False), n + np.arange(m[b])]) if b < B - 1 or B == 1 else []
        samples.append(rng.permutation(np.asarray(s, np.int64)).astype(np.int32))
    return pos, samples


def install_positions(ctx, pos):
    """set_clouds_samples_tensors from one [M, 3] tensor; returns N_b."""
    poff = np.zeros(len(pos) + 1, np.int32)
    poff[1:] = np.cumsum([len(p) for p in pos])
    first = ctx.set_clouds_samples_tensors(poff, dev(np.concatenate(pos)))
    return first


def search_both(ctx, samples, detect):
    """The host batch call and its device twin on the installed batch; asserts they agree and returns (host per-cloud
    results, device records, device offsets)."""
    host = ctx.detect_batch(samples) if detect else ctx.hand_search_batch(samples)
    offsets, sidx = lib.pack_samples(samples)
    if detect:
        rec, flags, scores, coff = ctx.detect_batch_tensors(offsets, dev(sidx))
    else:
        rec, flags, coff = ctx.hand_search_batch_tensors(offsets, dev(sidx))
    assert rec.is_cuda and rec.dtype == torch_().uint8 and rec.shape[1] == lib.POSE_BYTES
    assert np.array_equal(np.diff(coff), [h["n_candidates"] for h in host]) and coff[0] == 0
    assert lib.poses_from_tensor(rec).tobytes() == b"".join(h["candidates"].tobytes() for h in host)
    P = ctx.params.num_hand_axes * ctx.params.num_orientations
    assert flags.shape == (len(sidx), P)
    assert np.array_equal(flags.cpu().numpy(), np.concatenate([h["pose_flags"] for h in host]).reshape(-1, P))
    if detect:
        hs = np.concatenate([h["pose_scores"] for h in host]).reshape(-1, P)
        assert scores.cpu().numpy().view(np.int32).tobytes() == hs.view(np.int32).tobytes()
    return host, rec, coff


SEARCH_CASES = {
    "12ch_mixed_K": dict(channels=12, cams=[K1, K3, K8, K1]),
    "15ch_fast_tier": dict(channels=15, cams=[K1, K2, K1]),
    "15ch_general_tier": dict(channels=15, cams=[K1, K3, K2]),
    "12ch_straddling_chunks_no_overlap": dict(channels=12, cams=[K1, K3, K1, K2], chunk_samples=37, overlap=False),
    "15ch_straddling_chunks_overlap": dict(channels=15, cams=[K2, K1, K1], chunk_samples=29, overlap=True),
    "batch_of_one": dict(channels=15, cams=[K1]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SEARCH_CASES))
def test_search_and_detect_equal_the_host_routes(case):
    cfg = dict(SEARCH_CASES[case])
    cams, overlap = cfg.pop("cams"), cfg.pop("overlap", None)
    ctx = context(**cfg)
    if overlap is not None:
        ctx.set_overlap(overlap)
    clouds = tables(cams)
    ctx.set_clouds(clouds)
    pos, samples = scenario(clouds)
    ctx.set_clouds_samples(pos)
    search_both(ctx, samples, False)
    host, rec, _ = search_both(ctx, samples, True)
    assert sum(h["n_candidates"] for h in host) > 0
    assert any(np.any(h["candidates"]["sample_index"] >= len(c["xyz"])) for h, c in zip(host, clouds))  # at positions
    # positions installed from a tensor address the same hands
    assert np.array_equal(install_positions(ctx, pos), [len(c["xyz"]) for c in clouds])
    search_both(ctx, samples, False)
    assert lib.poses_from_tensor(search_both(ctx, samples, True)[1]).tobytes() == lib.poses_from_tensor(rec).tobytes()
    ctx.close()


@pytest.mark.gpu
def test_positions_from_a_side_stream_and_their_lifetime():
    """Positions written by torch on a side stream with no synchronisation are the host positions; a second call replaces
    them; a failed call and a reinstall drop them; without a batch the call is GPDB_ERR_STATE, as its host twin."""
    torch = torch_()
    ctx = context(channels=12)
    # no batch: GPDB_ERR_STATE with the host twin's message
    off0 = np.array([0, 3], np.int32)
    d3 = dev(np.zeros((3, 3)))
    assert lib.lib().gpdb_set_clouds_samples(ctx.h, lib._p(off0), lib._p(np.zeros((3, 3)))) == ERR_STATE
    msg_h = lib.lib().gpdb_last_error(ctx.h).decode()
    assert lib.lib().gpdb_set_clouds_samples_device(ctx.h, lib._p(off0), C.c_void_p(d3.data_ptr())) == ERR_STATE
    msg_d = lib.lib().gpdb_last_error(ctx.h).decode()
    assert msg_d.replace("gpdb_set_clouds_samples_device", "gpdb_set_clouds_samples") == msg_h
    clouds = tables([K1, K3, K1])
    ctx.set_clouds(clouds)
    pos, samples = scenario(clouds, seed=3)
    ctx.set_clouds_samples(pos)
    host, _, _ = search_both(ctx, samples, True)
    # positions written on a side stream, installed and used there with no synchronisation in between
    poff = np.zeros(len(pos) + 1, np.int32)
    poff[1:] = np.cumsum([len(p) for p in pos])
    offsets, sidx = lib.pack_samples(samples)
    src_pos = torch.from_numpy(np.concatenate(pos)).pin_memory()
    src_idx = torch.from_numpy(sidx).pin_memory()
    ctx.set_clouds_samples([np.zeros((0, 3))] * len(clouds))  # nothing installed before the side-stream call
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d_pos = torch.zeros(src_pos.shape, dtype=torch.float64, device="cuda")
        d_idx = torch.zeros(src_idx.shape, dtype=torch.int32, device="cuda")
        torch.cuda._sleep(200_000_000)  # the copies land long after the calls below are queued behind them
        d_pos.copy_(src_pos, non_blocking=True)
        d_idx.copy_(src_idx, non_blocking=True)
        ctx.set_clouds_samples_tensors(poff, d_pos)
        rec, flags, scores, coff = ctx.detect_batch_tensors(offsets, d_idx)
    torch.cuda.synchronize()
    assert lib.poses_from_tensor(rec).tobytes() == b"".join(h["candidates"].tobytes() for h in host)
    assert np.array_equal(np.diff(coff), [h["n_candidates"] for h in host])
    # a second call replaces the positions: the host route with the same replacement agrees
    pos2 = [p + 0.001 for p in pos]
    install_positions(ctx, pos2)
    dev2 = ctx.hand_search_batch_tensors(offsets, dev(sidx))
    ctx.set_clouds_samples(pos2)
    host2 = ctx.hand_search_batch(samples)
    assert lib.poses_from_tensor(dev2[0]).tobytes() == b"".join(h["candidates"].tobytes() for h in host2)
    assert lib.poses_from_tensor(dev2[0]).tobytes() != lib.poses_from_tensor(rec).tobytes()
    n0 = len(clouds[0]["xyz"])

    def position_refused():
        with pytest.raises(lib.GpdbError) as e:
            ctx.hand_search_batch_tensors(np.array([0, 1, 1, 1], np.int32), dev(np.array([n0], np.int32)))
        assert e.value.code == ERR_INVALID and f"sample index {n0} at position 0 outside cloud 0 (N = {n0}, + 0" in str(e.value)

    # a failed call (decreasing offsets) leaves no positions
    install_positions(ctx, pos)
    bad = np.array([0, 5, 3, poff[-1]], np.int32)
    with pytest.raises(lib.GpdbError) as e:
        ctx.set_clouds_samples_tensors(bad, dev(np.concatenate(pos)))
    assert e.value.code == ERR_INVALID and "pos_offsets decrease at cloud 1" in str(e.value)
    position_refused()
    # a reinstall drops them
    install_positions(ctx, pos)
    ctx.set_clouds(clouds)
    position_refused()
    ctx.close()


def image_case(channels, cams):
    """A keep_images context with a batch, positions and the hand-search records of the device route."""
    ctx = context(channels=channels, keep_images=1)
    clouds = tables(cams, seed=80)
    ctx.set_clouds(clouds)
    pos, samples = scenario(clouds, seed=21)
    ctx.set_clouds_samples(pos)
    return ctx, clouds, pos, samples


def subset(rec, coff, keep):
    """The records with keep[j] set, regrouped: (records tensor, offsets)."""
    torch = torch_()
    idx = np.flatnonzero(keep)
    off = np.searchsorted(idx, coff).astype(np.int32)
    return rec[torch.from_numpy(idx).cuda()].contiguous(), off


@pytest.mark.gpu
@pytest.mark.parametrize("channels,cams", [(1, [K1, K3, K1]), (3, [K2, K1]), (12, [K1, K8, K3]), (15, [K1, K2, K1]),
                                           (15, [K3, K1])], ids=["1ch", "3ch", "12ch", "15ch_fast_tier", "15ch_general_tier"])
def test_images_equal_detect_batch_images(channels, cams):
    ctx, clouds, _, samples = image_case(channels, cams)
    det = ctx.detect_batch(samples)
    offsets, sidx = lib.pack_samples(samples)
    rec, _, coff = ctx.hand_search_batch_tensors(offsets, dev(sidx))
    assert lib.poses_from_tensor(rec)["frame"].tobytes() == b"".join(d["candidates"]["frame"].tobytes() for d in det)
    img = ctx.images_batch_tensors(coff, rec)
    S = ctx.params.image_size
    assert img.is_cuda and img.shape == (coff[-1], S, S, channels)
    want = np.concatenate([d["images"] for d in det if d["n_candidates"]]).reshape(-1, S, S, channels)
    assert coff[-1] > 0 and img.cpu().numpy().tobytes() == want.tobytes()
    # a filtered subset (every third record, and none of cloud 0)
    keep = np.arange(coff[-1]) % 3 == 1
    keep[:coff[1]] = False
    sub, soff = subset(rec, coff, keep)
    assert soff[1] == 0 and soff[-1] == keep.sum()
    assert ctx.images_batch_tensors(soff, sub).cpu().numpy().tobytes() == want[keep].tobytes()
    ctx.close()


@pytest.mark.gpu
def test_images_of_one_cloud_equal_the_single_cloud_call():
    ctx, clouds, pos, samples = image_case(15, [K2])
    offsets, sidx = lib.pack_samples(samples)
    rec, _, coff = ctx.hand_search_batch_tensors(offsets, dev(sidx))
    img = ctx.images_batch_tensors(coff, rec).cpu().numpy()
    c = clouds[0]
    ctx.set_cloud(c["xyz"], c["normals"], c.get("cam_source"), c.get("view_points"))
    ctx.set_samples(pos[0])
    assert coff[-1] > 0 and img.tobytes() == ctx.images(lib.poses_from_tensor(rec)).tobytes()
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("lenet_impl", [0, 1], ids=["tensor_cores", "simt"])
@pytest.mark.parametrize("channels", [12, 15])
def test_classify_equals_host_classify_and_detect_scores(channels, lenet_impl):
    """classify_tensors equals classify of the same host images (scores and logits bit for bit) and the scores detect_batch
    gave those records. The second holds exactly: the image kernels write the P16 pixels with bytes C..15 zero, and
    k_hwc_to_p16 rebuilds every pixel from its C bytes with the same zero padding, so hwc_to_p16(p16_to_hwc(x)) is x and
    LeNet reads the bytes it read inside detect_batch."""
    ctx = context(channels=channels, keep_images=1, lenet_impl=lenet_impl, batch_size=100)
    clouds = tables([K1, K2, K1], seed=80)
    ctx.set_clouds(clouds)
    pos, samples = scenario(clouds, seed=21)
    ctx.set_clouds_samples(pos)
    det = ctx.detect_batch(samples)
    offsets, sidx = lib.pack_samples(samples)
    rec, _, _, coff = ctx.detect_batch_tensors(offsets, dev(sidx))
    img = ctx.images_batch_tensors(coff, rec)
    scores, logits = ctx.classify_tensors(img)
    hs, hl = ctx.classify(img.cpu().numpy())
    assert coff[-1] > 100  # more than one classifier batch
    assert scores.cpu().numpy().tobytes() == hs.tobytes() and logits.cpu().numpy().tobytes() == hl.tobytes()
    want = np.concatenate([d["candidates"]["score"] for d in det])
    assert scores.cpu().numpy().tobytes() == want.tobytes()
    assert lib.poses_from_tensor(rec)["score"].tobytes() == want.tobytes()
    empty = ctx.classify_tensors(img[:0])
    assert empty[0].shape == (0,) and empty[1].shape == (0, 2)
    ctx.close()


def refused(call, code=ERR_INVALID):
    with pytest.raises(lib.GpdbError) as e:
        call()
    assert e.value.code == code
    return str(e.value)


def last_error(ctx):
    return lib.lib().gpdb_last_error(ctx.h).decode()


@pytest.mark.gpu
def test_errors_match_the_host_twins():
    ctx = context(channels=12)
    L = lib.lib()
    clouds = tables([K1, K3, K1, K2])
    ctx.set_clouds(clouds)
    pos, samples = scenario(clouds, seed=5)
    ctx.set_clouds_samples(pos)
    n = [len(c["xyz"]) + len(p) for c, p in zip(clouds, pos)]
    # an index outside its cloud in a middle cloud
    bad = [s.copy() for s in samples]
    bad[2][7] = n[2]
    offsets, sidx = lib.pack_samples(bad)
    for host_call, dev_call, name in ((ctx.detect_batch, ctx.detect_batch_tensors, "gpdb_detect_batch"),
                                      (ctx.hand_search_batch, ctx.hand_search_batch_tensors, "gpdb_hand_search_batch")):
        msg_h = refused(lambda: host_call(bad))
        msg_d = refused(lambda: dev_call(offsets, dev(sidx)))
        assert msg_d.replace(name + "_device", name) == msg_h
        assert f"sample index {n[2]} at position {offsets[2] + 7} outside cloud 2" in msg_h
    # malformed offsets
    good_off, good_idx = lib.pack_samples(samples)
    dec = good_off.copy()
    dec[2] = dec[3] + 1
    d_idx = dev(good_idx)
    P = ctx.params.num_hand_axes * ctx.params.num_orientations
    d_rec = torch_().empty((len(good_idx) * P, lib.POSE_BYTES), dtype=torch_().uint8, device="cuda")
    coff = np.zeros(len(dec), np.int32)
    res = abi.Result()
    for host_fn, dev_fn, name in ((L.gpdb_detect_batch, L.gpdb_detect_batch_device, "gpdb_detect_batch"),
                                  (L.gpdb_hand_search_batch, L.gpdb_hand_search_batch_device, "gpdb_hand_search_batch")):
        assert host_fn(ctx.h, lib._p(dec), lib._p(good_idx), C.byref(res), lib._p(coff)) == ERR_INVALID
        msg_h = last_error(ctx)
        dense = [None, None] if name == "gpdb_detect_batch" else [None]
        assert dev_fn(ctx.h, lib._p(dec), C.c_void_p(d_idx.data_ptr()), *dense, C.c_void_p(d_rec.data_ptr()), lib._p(coff),
                      C.byref(res)) == ERR_INVALID
        assert last_error(ctx).replace(name + "_device", name) == msg_h and "sample_offsets decrease at cloud 2" in msg_h
    # host pointers where device memory is expected: refused before any device work
    assert L.gpdb_detect_batch_device(ctx.h, lib._p(good_off), lib._p(good_idx), None, None, C.c_void_p(d_rec.data_ptr()),
                                      lib._p(coff), C.byref(res)) == ERR_INVALID
    assert "gpdb_detect_batch_device: d_sample_idx is not device memory of device 0" in last_error(ctx)
    host_rec = np.zeros(len(good_idx) * P * lib.POSE_BYTES, np.uint8)
    assert L.gpdb_hand_search_batch_device(ctx.h, lib._p(good_off), C.c_void_p(d_idx.data_ptr()), None, lib._p(host_rec),
                                           lib._p(coff), C.byref(res)) == ERR_INVALID
    assert "d_hands_out is not device memory" in last_error(ctx)
    poff = np.array([0, 1, 1, 1, 1], np.int32)
    assert L.gpdb_set_clouds_samples_device(ctx.h, lib._p(poff), lib._p(np.zeros((1, 3)))) == ERR_INVALID
    assert "d_samples_xyz is not device memory" in last_error(ctx)
    ctx.set_clouds_samples(pos)  # the refused call dropped the positions, as its host twin's failures do
    rec, _, coff = ctx.hand_search_batch_tensors(good_off, d_idx)
    img = ctx.images_batch_tensors(coff, rec)
    host_img = np.zeros(img.numel(), np.uint8)
    assert L.gpdb_images_batch_device(ctx.h, lib._p(coff), C.c_void_p(rec.data_ptr()), lib._p(host_img)) == ERR_INVALID
    assert "gpdb_images_batch_device: d_images_out is not device memory" in last_error(ctx)
    scores = torch_().empty(len(img), dtype=torch_().float32, device="cuda")
    assert L.gpdb_classify_device(ctx.h, lib._p(host_img), len(img), C.c_void_p(scores.data_ptr()), None) == ERR_INVALID
    assert "gpdb_classify_device: d_images_hwc is not device memory" in last_error(ctx)
    # hand offsets: decreasing, or of the wrong length
    hdec = coff.copy()
    hdec[1] = hdec[2] + 1
    assert "gpdb_images_batch_device: hand_offsets decrease at cloud 1" in refused(lambda: ctx.images_batch_tensors(hdec, rec))
    with pytest.raises(ValueError, match="hand_offsets"):
        ctx.images_batch_tensors(coff[:-1], rec)
    with pytest.raises(ValueError, match="sample_offsets"):
        ctx.detect_batch_tensors(good_off[:-1], d_idx)
    # the batch and its positions stay after refused calls, and the calls still agree with their host twins
    search_both(ctx, samples, True)
    ctx.close()
