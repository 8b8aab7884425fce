"""world_size-2 gloo test (CPU) of the multi-GPU host logic: contiguous slices of the sample indices over a
broadcast cloud, one all-gather of fixed-stride score slots (gpd_b200/sharding.py). The per-rank compute is
stood in by the oracle here (no GPU in this container); on a GPU machine the same code runs with NCCL."""
import os
import socket

import numpy as np
import pytest

from gpd_b200 import sharding


def test_slices_partition_the_samples():
    for n in (0, 1, 7, 100, 100001):
        for world in (1, 2, 3, 8):
            b = [sharding.slice_bounds(n, r, world) for r in range(world)]
            assert b[0][0] == 0 and b[-1][1] == n
            assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
            assert max(hi - lo for lo, hi in b) - min(hi - lo for lo, hi in b) <= 1
            assert sharding.slot_stride(n, world) == max(hi - lo for lo, hi in b)


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist

    from gpd_b200 import abi, scenes
    from oracle import oracle

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cloud = scenes.krylon_cloud() if rank == 0 else None
    cloud = sharding.broadcast_cloud(cloud, rank, dist)
    n = 21  # uneven split on purpose
    sidx = scenes.sample_indices(2, len(cloud["xyz"]), n)
    lo, hi = sharding.slice_bounds(n, rank, world)
    p = abi.default_params(3)
    z = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpd_b200", "weights",
                             "lenet_3ch.npz"))
    w = oracle.WeightPack([z[k] for k in oracle.WeightPack.NAMES])
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    local = oc.detect(p, w, sidx[lo:hi], nthreads=2)
    full = sharding.gather_scores(local["pose_scores"].reshape(-1), n, 8, rank, world, dist)
    # global top-k: local top-k per rank (what gpdb_detect_select returns), one all-gather of record slots, merge
    k = 5
    lc = local["candidates"]
    lc = lc[np.argsort(-lc["score"].astype(np.float64), kind="stable")[:k]]
    top = sharding.select_global(lc, k, n, rank, world, dist)
    if rank == 0:
        ref = oc.detect(p, w, sidx, nthreads=2)
        q.put((full.numpy(), ref["pose_scores"], top, ref["candidates"]))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_allgather_matches_single_rank():
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    full, ref, top, ref_cand = q.get(timeout=240)
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    assert full.shape == ref.shape == (21, 8)
    assert np.array_equal(np.isnan(full), np.isnan(ref))
    m = ~np.isnan(ref)
    assert m.any() and np.array_equal(full[m], ref[m])
    # sharded selectGrasps == single-rank selectGrasps (same records, same order, sample slots rebased)
    want = ref_cand[np.argsort(-ref_cand["score"].astype(np.float64), kind="stable")[:5]]
    assert len(top) == len(want) == 5
    for f in top.dtype.names:
        if f != "pad_":
            assert np.array_equal(top[f], want[f]), f


def test_reference_arm_prints_one_contract_line():
    """`bench.py --impl reference` (the CPU restatement timed on the host cores, no GPU): exactly one JSON line on stdout
    with the keys of the bench contract."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=600, env={**os.environ, "RANK": "0", "WORLD_SIZE": "1"})
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, out.stdout[-400:] + out.stderr[-400:]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["value"] > 0 and d["higher_is_better"] is True and d["n_gpus"] == 1
    assert d["metric"].startswith("grasp candidates/sec") and d["unit"].startswith("samples/s")
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    # a non-zero rank of a torchrun launch does no work and prints nothing
    out2 = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--gpus", "2"],
                          capture_output=True, text=True, timeout=60, env={**os.environ, "RANK": "1", "WORLD_SIZE": "2"})
    assert out2.returncode == 0 and out2.stdout.strip() == ""


def test_c_abi_shard_bounds_match_the_python_plumbing():
    """gpdb_shard_bounds / gpdb_slot_bytes (the slices gpdb_detect_sharded uses inside the library; pure host arithmetic, no
    GPU needed) against sharding.slice_bounds / slot_stride, incl. n < nranks, n = 0 and n not divisible by nranks."""
    from gpd_b200 import lib
    for n in (0, 1, 5, 7, 100000, 100001, 1000000, 2 ** 31 - 1):
        for world in (1, 2, 3, 4, 8):
            covered = 0
            for r in range(world):
                lo, hi, st = lib.shard_bounds(n, r, world)
                assert (lo, hi) == sharding.slice_bounds(n, r, world)
                assert lo == covered and hi >= lo
                covered = hi
                if n < 2 ** 30:
                    assert st == sharding.slot_stride(n, world)
            assert covered == n
    assert lib.slot_bytes(12501, 8) == 12501 * 8 * 4 + (12501 * 8 + 15) // 16 * 16 + 16
    # malformed requests give an empty slice instead of dividing by zero
    for bad in ((10, 0, 0), (10, -1, 4), (10, 4, 4), (-5, 0, 2)):
        assert lib.shard_bounds(*bad) == (0, 0, 0)
