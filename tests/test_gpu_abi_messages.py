"""Every argument and state check of the batch entry points, host call and _device twin alike, pinned to its return code,
its exact full message and the state a failed call leaves behind, on the GPU.

Each row of the table is one bad call: null and negative arguments, offsets that do not start at 0 or decrease at a
middle cloud or group, no installed batch, a host pointer where device memory is expected, an index outside a middle
cloud (a point index, and one past the sample positions), a non-finite point and cam_source = 2 without voxelisation.
After the call the test reads which state survived: the batch, its sample positions and the record of the last SIS call.
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import abi, lib, scenes

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

INVALID, STATE = -1, -3
K3 = [(0.0, 0.0, 0.0), (0.3, 0.0, 0.0), (-0.3, 0.1, 0.0)]
FULL = (True, True, True)    # (batch, sample positions, SIS record) after the setup of a row
KEPT_NO_POS = (True, False, True)
KEPT_NO_SIS = (True, False, False)
NONE = (False, False, False)
L = lib.lib


def ptr(x):
    """A host (numpy) or device (torch) array as the void * of the C-ABI."""
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return C.c_void_p(x.data_ptr())
    return x.ctypes.data_as(C.c_void_p)


def context():
    w, relu = load_weights(12)
    ctx = lib.Context(lib.default_params(channels=12, relu_after_conv=relu))
    ctx.set_weights(w)
    return ctx


def raw_view(seed, n, cameras=None):
    s = scenes.synthetic_raw_scene(seed, n_points=n, cameras=cameras, mark_all_cameras=cameras is not None)
    return {"xyz": s["xyz"].astype(np.float32), "cam_source": s["cam_source"], "view_points": s["view_points"],
            "normals": None}


@pytest.fixture(scope="module")
def env():
    ctx, empty = context(), context()
    views = [raw_view(41, 6000), raw_view(42, 6000, cameras=K3), raw_view(43, 6000)]
    e = SimpleNamespace(ctx=ctx, empty=empty, views=views, pp=lib.preprocess_params())
    clouds = ctx.preprocess_clouds(views, e.pp)
    e.N = [len(c["xyz"]) for c in clouds]
    assert min(e.N) > 10
    e.pk, e.rk = lib.pack_clouds(clouds), lib.pack_clouds(views)
    e.dpk = {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in e.pk.items()}
    e.drk = {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in e.rk.items()}
    # the positions of the setup: two per cloud, at each cloud's first two points
    e.pos_off = np.array([0, 2, 4, 6], np.int32)
    e.pos = np.ascontiguousarray(np.concatenate([c["xyz"][:2] for c in clouds]).astype(np.float64))
    e.d_pos = torch.from_numpy(e.pos).cuda()
    e.fmt = {"n0": e.N[0], "n1": e.N[1], "n2": e.N[2], "n1p": e.N[1] + 2, "p1": int(e.pk["offsets"][1]) + 5}
    yield e
    ctx.close()
    empty.close()


def sis_call(c, sp, ioff, iidx, dev=False, hands=None):
    r = abi.Result()
    hoff = np.zeros(4, np.int32)
    if dev:
        return L().gpdb_sis_batch_device(c.h, C.byref(sp) if sp else None, ptr(ioff), ptr(iidx), ptr(hands), ptr(hoff),
                                         C.byref(r)), r
    return L().gpdb_sis_batch(c.h, C.byref(sp) if sp else None, ptr(ioff), ptr(iidx), C.byref(r), ptr(hoff)), r


def setup_full(e):
    """The batch (preprocessed, so it has source indices), a successful SIS call, then two positions per cloud."""
    c = e.ctx
    c.preprocess_clouds(e.views, e.pp, read_back=False)
    rc, r = sis_call(c, lib.sis_params(num_iterations=1, num_samples_per_iteration=4), np.array([0, 3, 6, 9], np.int32),
                     np.array([0, 1, 2] * 3, np.int32))
    assert rc >= 0, L().gpdb_last_error(c.h).decode()
    L().gpdb_free_result(C.byref(r))
    rc = L().gpdb_set_clouds_samples(c.h, ptr(e.pos_off), ptr(e.pos))
    assert rc == 6, L().gpdb_last_error(c.h).decode()


def state(e, c):
    """(batch installed, sample positions installed, SIS record readable)"""
    sis = L().gpdb_sis_positions(c.h, None, None, None, None, None) >= 0
    batch = L().gpdb_get_clouds(c.h, None, None, None, None) >= 0
    pos = False
    if batch:  # index N_0 addresses cloud 0's first position: in range only while positions are installed
        r = abi.Result()
        rc = L().gpdb_hand_search_batch(c.h, ptr(np.array([0, 1, 1, 1], np.int32)), ptr(np.array([e.N[0]], np.int32)),
                                        C.byref(r), ptr(np.zeros(4, np.int32)))
        pos = rc >= 0
        if pos:
            L().gpdb_free_result(C.byref(r))
    return batch, pos, sis


# ---- the calls of the table: `o` overrides the good arguments, dev selects the _device twin ------------------------------

def set_clouds(c, e, dev=False, **o):
    src = e.dpk if dev else e.pk
    a = dict(n=3, off=e.pk["offsets"], xyz=src["xyz"], nrm=src["normals"], cam=src["cam_source"], ks=e.pk["n_cameras"],
             vp=e.pk["view_points"])
    a.update(o)
    f = L().gpdb_set_clouds_device if dev else L().gpdb_set_clouds
    return f(c.h, a["n"], ptr(a["off"]), ptr(a["xyz"]), ptr(a["nrm"]), ptr(a["cam"]), ptr(a["ks"]), ptr(a["vp"]))


def preprocess(c, e, dev=False, **o):
    src = e.drk if dev else e.rk
    a = dict(n=3, off=e.rk["offsets"], xyz=src["xyz"], nrm=None, cam=src["cam_source"], ks=e.rk["n_cameras"],
             vp=e.rk["view_points"], pp=e.pp, out=np.zeros(4, np.int32))
    a.update(o)
    f = L().gpdb_preprocess_clouds_device if dev else L().gpdb_preprocess_clouds
    return f(c.h, a["n"], ptr(a["off"]), ptr(a["xyz"]), ptr(a["nrm"]), ptr(a["cam"]), ptr(a["ks"]), ptr(a["vp"]),
             C.byref(a["pp"]) if a["pp"] is not None else None, ptr(a["out"]))


def depth(c, e, dev=False, n=1, d=None):
    cams = (abi.DepthCamera * 1)(lib.depth_camera(8, 6, 10.0, 10.0, 4.0, 3.0))
    img = np.full(48, 500, np.uint16) if d is None else d
    f = L().gpdb_preprocess_depth_device if dev else L().gpdb_preprocess_depth
    return f(c.h, n, ptr(np.array([1], np.int32)), cams, abi.DEPTH_U16, ptr(img), C.byref(e.pp), ptr(np.zeros(2, np.int32)))


def set_samples(c, e, dev=False, **o):
    a = dict(off=e.pos_off, pos=e.d_pos if dev else e.pos)
    a.update(o)
    f = L().gpdb_set_clouds_samples_device if dev else L().gpdb_set_clouds_samples
    return f(c.h, ptr(a["off"]), ptr(a["pos"]))


def bad_samples(e, at=None, v=None):
    """Three samples per cloud; sample `at` of cloud 1 (position 3 + at) replaced by v."""
    idx = np.array([0, 1, 2] * 3, np.int32)
    if at is not None:
        idx[3 + at] = v
    return idx


SOFF = np.array([0, 3, 6, 9], np.int32)


def batch(which, c, e, dev=False, **o):
    """the six run_batch entry points: detect / hand_search / select, host and device"""
    rec = torch.zeros(64 * C.sizeof(abi.Pose), dtype=torch.uint8, device="cuda") if dev else None
    a = dict(off=SOFF, idx=bad_samples(e), out=np.zeros(4, np.int32), sel=rec, flags=None, scores=None, hands=rec)
    a.update(o)
    if dev and isinstance(a["idx"], np.ndarray) and "host_idx" not in o:
        a["idx"] = torch.from_numpy(a["idx"]).cuda()
    r = abi.Result()
    rc = {
        "detect_batch": lambda: L().gpdb_detect_batch(c.h, ptr(a["off"]), ptr(a["idx"]), C.byref(r), ptr(a["out"])),
        "hand_search_batch": lambda: L().gpdb_hand_search_batch(c.h, ptr(a["off"]), ptr(a["idx"]), C.byref(r), ptr(a["out"])),
        "detect_batch_select": lambda: L().gpdb_detect_batch_select(c.h, ptr(a["off"]), ptr(a["idx"]), 2, C.byref(r),
                                                                    ptr(a["out"])),
        "detect_batch_select_device": lambda: L().gpdb_detect_batch_select_device(c.h, ptr(a["off"]), ptr(a["idx"]), 2,
                                                                                  ptr(a["sel"]), ptr(a["out"]), C.byref(r)),
        "hand_search_batch_device": lambda: L().gpdb_hand_search_batch_device(c.h, ptr(a["off"]), ptr(a["idx"]),
                                                                              ptr(a["flags"]), ptr(a["hands"]), ptr(a["out"]),
                                                                              C.byref(r)),
        "detect_batch_device": lambda: L().gpdb_detect_batch_device(c.h, ptr(a["off"]), ptr(a["idx"]), ptr(a["flags"]),
                                                                    ptr(a["scores"]), ptr(a["hands"]), ptr(a["out"]),
                                                                    C.byref(r)),
    }[which]()
    assert rc < 0, "the row's call must fail"
    return rc


def images(c, e, **o):
    a = dict(off=np.array([0, 1, 2, 3], np.int32), hands=torch.zeros(3 * C.sizeof(abi.Pose), dtype=torch.uint8, device="cuda"),
             out=torch.zeros(1, dtype=torch.uint8, device="cuda"))
    a.update(o)
    return L().gpdb_images_batch_device(c.h, ptr(a["off"]), ptr(a["hands"]), ptr(a["out"]))


def clusters(c, e, dev=False, **o):
    a = dict(n=3, off=np.array([0, 1, 2, 3], np.int32), hands=np.zeros(3 * C.sizeof(abi.Pose), np.uint8),
             out=np.zeros(3 * C.sizeof(abi.Pose), np.uint8), coff=np.zeros(4, np.int32))
    a.update(o)
    f = L().gpdb_find_clusters_batch_device if dev else L().gpdb_find_clusters_batch
    return f(c.h, a["n"], ptr(a["off"]), ptr(a["hands"]), 1, ptr(a["out"]), ptr(a["coff"]))


def sis(c, e, dev=False, **o):
    a = dict(sp=lib.sis_params(num_iterations=1, num_samples_per_iteration=4), off=SOFF, idx=bad_samples(e),
             hands=torch.zeros(64 * C.sizeof(abi.Pose), dtype=torch.uint8, device="cuda"))
    a.update(o)
    if dev and isinstance(a["idx"], np.ndarray) and "host_idx" not in o:
        a["idx"] = torch.from_numpy(a["idx"]).cuda()
    rc, _ = sis_call(c, a["sp"], a["off"], a["idx"], dev, a["hands"])
    assert rc < 0, "the row's call must fail"
    return rc


def subsample(c, e, dev=False, n=2, **o):
    a = dict(mask=None, idx=torch.zeros(64, dtype=torch.int32, device="cuda") if dev else np.zeros(64, np.int32),
             off=np.zeros(4, np.int32))
    a.update(o)
    f = L().gpdb_subsample_clouds_device if dev else L().gpdb_subsample_clouds
    return f(c.h, n, 7, ptr(a["mask"]), ptr(a["idx"]), ptr(a["off"]))


def classify(c, e, n=1, images_hwc=None):
    img = torch.zeros(12 * 60 * 60, dtype=torch.uint8, device="cuda") if images_hwc is None else images_hwc
    return L().gpdb_classify_device(c.h, ptr(img), n, ptr(torch.zeros(1, device="cuda")), None)


def nan_xyz(e, dev):
    x = e.pk["xyz"].copy()
    x[int(e.pk["offsets"][1]) + 5, 1] = np.nan
    return torch.from_numpy(x).cuda() if dev else x


def cam2(e, dev):
    """cloud 1 (3 cameras): cam_source[7][1] = 2"""
    cs = e.rk["cam_source"].copy()
    cs[int(e.rk["offsets"][1]) * int(e.rk["n_cameras"][0]) + 7 * 3 + 1] = 2
    return torch.from_numpy(cs).cuda() if dev else cs


I32 = lambda *v: np.array(v, np.int32)  # noqa: E731
HOST = np.zeros(64, np.uint8)
SETC = "need n_clouds > 0, point_offsets (starting at 0), n_cameras, xyz, normals, view_points"
PREC = "need n_clouds > 0, point_offsets (starting at 0), n_cameras, xyz, view_points, params, processed_offsets_out"
NOBATCH = "no batch of clouds: call gpdb_set_clouds / gpdb_preprocess_clouds first"
NOBATCH_SET = "no batch of clouds: call gpdb_set_clouds first"
NOBATCH_DEPTH = "no batch of clouds: call gpdb_preprocess_depth / gpdb_preprocess_clouds first"
NODEV = "is not device memory of device 0"
RUN_BATCH = ["detect_batch", "hand_search_batch", "detect_batch_select", "detect_batch_select_device",
             "hand_search_batch_device", "detect_batch_device"]
CAND_OUT = {"detect_batch": "null cand_offsets_out", "hand_search_batch": "null cand_offsets_out",
            "detect_batch_select": "need sel_offsets_out and num_selected >= 0",
            "detect_batch_select_device": "need sel_offsets_out and num_selected >= 0",
            "hand_search_batch_device": "null cand_offsets_out", "detect_batch_device": "null cand_offsets_out"}
SEL_NAME = {"detect_batch_select_device": "d_selected_out", "hand_search_batch_device": "d_hands_out",
            "detect_batch_device": "d_candidates_out"}


def rows():
    """(id, setup, call, return code, message after "gpd_b200 error <code>: ", state afterwards)"""
    R = []
    for dev, nm in ((False, "gpdb_set_clouds"), (True, "gpdb_set_clouds_device")):
        R += [
            (f"{nm}-n0", "full", lambda c, e, d=dev: set_clouds(c, e, d, n=0), INVALID, f"{nm}: {SETC}", NONE),
            (f"{nm}-neg", "full", lambda c, e, d=dev: set_clouds(c, e, d, n=-1), INVALID, f"{nm}: {SETC}", NONE),
            (f"{nm}-null-off", "full", lambda c, e, d=dev: set_clouds(c, e, d, off=None), INVALID, f"{nm}: {SETC}", NONE),
            (f"{nm}-off0", "full", lambda c, e, d=dev: set_clouds(c, e, d, off=e.pk["offsets"] + 1), INVALID, f"{nm}: {SETC}",
             NONE),
            (f"{nm}-decrease", "full", lambda c, e, d=dev: set_clouds(c, e, d, off=I32(0, 20, 10, 30)), INVALID,
             f"{nm}: cloud 1 has -10 points (offsets must increase)", NONE),
            (f"{nm}-cameras", "full", lambda c, e, d=dev: set_clouds(c, e, d, ks=I32(1, 9, 1)), INVALID,
             f"{nm}: cloud 1 has 9 cameras (1 <= cameras <= 8)", NONE),
            (f"{nm}-nonfinite", "full", lambda c, e, d=dev: set_clouds(c, e, d, xyz=nan_xyz(e, d)), INVALID,
             f"{nm}: point {{p1}} has a non-finite coordinate (run removeNans / gpdb_preprocess first)", NONE),
        ]
    R += [("gpdb_set_clouds_device-host-xyz", "full", lambda c, e: set_clouds(c, e, True, xyz=e.pk["xyz"]), INVALID,
           f"gpdb_set_clouds_device: d_xyz {NODEV}", NONE),
          ("gpdb_set_clouds_device-host-cam", "full",
           lambda c, e: set_clouds(c, e, True, cam=np.ones(len(e.pk["xyz"]), np.int32)), INVALID,
           f"gpdb_set_clouds_device: d_cam_source {NODEV}", NONE)]
    for dev, nm in ((False, "gpdb_preprocess_clouds"), (True, "gpdb_preprocess_clouds_device")):
        R += [
            (f"{nm}-n0", "full", lambda c, e, d=dev: preprocess(c, e, d, n=0), INVALID, f"{nm}: {PREC}", NONE),
            (f"{nm}-null-params", "full", lambda c, e, d=dev: preprocess(c, e, d, pp=None), INVALID, f"{nm}: {PREC}", NONE),
            (f"{nm}-null-out", "full", lambda c, e, d=dev: preprocess(c, e, d, out=None), INVALID, f"{nm}: {PREC}", NONE),
            (f"{nm}-off0", "full", lambda c, e, d=dev: preprocess(c, e, d, off=e.rk["offsets"] + 1), INVALID,
             f"{nm}: {PREC}", NONE),
            (f"{nm}-decrease", "full", lambda c, e, d=dev: preprocess(c, e, d, off=I32(0, 20, 10, 30)), INVALID,
             f"{nm}: raw cloud 1 has -10 points (offsets must increase)", NONE),
            (f"{nm}-normals", "full", lambda c, e, d=dev: preprocess(c, e, d, pp=lib.preprocess_params(estimate_normals=0)),
             INVALID, f"{nm}: estimate_normals = 0 needs the caller's normals", NONE),
            (f"{nm}-voxel", "full", lambda c, e, d=dev: preprocess(c, e, d, pp=lib.preprocess_params(voxel_size=0.0)),
             INVALID, f"{nm}: voxel_size and normals_radius must be positive", NONE),
            (f"{nm}-cam2", "full",
             lambda c, e, d=dev: preprocess(c, e, d, cam=cam2(e, d), pp=lib.preprocess_params(voxelize=0)), INVALID,
             f"{nm}: cloud 1: cam_source[7][1] = 2; without voxelisation entries must be 0 or 1", NONE),
        ]
    R += [("gpdb_preprocess_clouds_device-host-xyz", "full", lambda c, e: preprocess(c, e, True, xyz=e.rk["xyz"]), INVALID,
           f"gpdb_preprocess_clouds_device: d_xyz {NODEV}", NONE)]
    DEP = "need n_views > 0, n_cameras, cameras, depth, params, processed_offsets_out"
    R += [("gpdb_preprocess_depth-n0", "full", lambda c, e: depth(c, e, n=0), INVALID, f"gpdb_preprocess_depth: {DEP}", NONE),
          ("gpdb_preprocess_depth_device-neg", "full", lambda c, e: depth(c, e, True, n=-1), INVALID,
           f"gpdb_preprocess_depth_device: {DEP}", NONE),
          ("gpdb_preprocess_depth_device-host-depth", "full", lambda c, e: depth(c, e, True), INVALID,
           f"gpdb_preprocess_depth_device: d_depth {NODEV}", NONE)]
    for dev, nm in ((False, "gpdb_set_clouds_samples"), (True, "gpdb_set_clouds_samples_device")):
        R += [
            (f"{nm}-nobatch", "empty", lambda c, e, d=dev: set_samples(c, e, d), STATE, f"{nm}: {NOBATCH}", NONE),
            (f"{nm}-null-off", "full", lambda c, e, d=dev: set_samples(c, e, d, off=None), INVALID,
             f"{nm}: need pos_offsets[4] starting at 0", KEPT_NO_POS),
            (f"{nm}-off0", "full", lambda c, e, d=dev: set_samples(c, e, d, off=I32(1, 2, 4, 6)), INVALID,
             f"{nm}: need pos_offsets[4] starting at 0", KEPT_NO_POS),
            (f"{nm}-decrease", "full", lambda c, e, d=dev: set_samples(c, e, d, off=I32(0, 2, 1, 6)), INVALID,
             f"{nm}: pos_offsets decrease at cloud 1", KEPT_NO_POS),
            (f"{nm}-null-samples", "full", lambda c, e, d=dev: set_samples(c, e, d, pos=None), INVALID,
             f"{nm}: null samples_xyz for 6 positions", KEPT_NO_POS),
        ]
    R += [("gpdb_set_clouds_samples_device-host-samples", "full", lambda c, e: set_samples(c, e, True, pos=e.pos), INVALID,
           f"gpdb_set_clouds_samples_device: d_samples_xyz {NODEV}", KEPT_NO_POS)]
    for which in RUN_BATCH:
        nm, dev = "gpdb_" + which, which.endswith("_device")
        R += [
            (f"{nm}-nobatch", "empty", lambda c, e, w=which, d=dev: batch(w, c, e, d), STATE, f"{nm}: {NOBATCH_SET}", NONE),
            (f"{nm}-null-cand-out", "full", lambda c, e, w=which, d=dev: batch(w, c, e, d, out=None), INVALID,
             f"{nm}: {CAND_OUT[which]}", FULL),
            (f"{nm}-null-off", "full", lambda c, e, w=which, d=dev: batch(w, c, e, d, off=None), INVALID,
             f"{nm}: need out and sample_offsets[4] starting at 0", FULL),
            (f"{nm}-off0", "full", lambda c, e, w=which, d=dev: batch(w, c, e, d, off=I32(1, 3, 6, 9)), INVALID,
             f"{nm}: need out and sample_offsets[4] starting at 0", FULL),
            (f"{nm}-decrease", "full", lambda c, e, w=which, d=dev: batch(w, c, e, d, off=I32(0, 3, 2, 9)), INVALID,
             f"{nm}: sample_offsets decrease at cloud 1", FULL),
            (f"{nm}-null-idx", "full", lambda c, e, w=which, d=dev: batch(w, c, e, d, idx=None), INVALID,
             f"{nm}: null sample_idx", FULL),
            (f"{nm}-sample-index", "full", lambda c, e, w=which, d=dev: batch(w, c, e, d, idx=bad_samples(e, 1, -1)), INVALID,
             f"{nm}: sample index -1 at position 4 outside cloud 1 (N = {{n1}}, + 2 sample positions)", FULL),
            (f"{nm}-position-index", "full",
             lambda c, e, w=which, d=dev: batch(w, c, e, d, idx=bad_samples(e, 2, e.N[1] + 2)), INVALID,
             f"{nm}: sample index {{n1p}} at position 5 outside cloud 1 (N = {{n1}}, + 2 sample positions)", FULL),
        ]
        if dev:
            R += [
                (f"{nm}-host-idx", "full", lambda c, e, w=which: batch(w, c, e, True, host_idx=1), INVALID,
                 f"{nm}: d_sample_idx {NODEV}", FULL),
                (f"{nm}-host-out", "full", lambda c, e, w=which: batch(w, c, e, True, sel=HOST, hands=HOST), INVALID,
                 f"{nm}: {SEL_NAME[which]} {NODEV}", FULL),
                (f"{nm}-null-records", "full", lambda c, e, w=which: batch(w, c, e, True, sel=None, hands=None), INVALID,
                 f"{nm}: null {SEL_NAME[which]}", FULL),
            ]
            if which != "detect_batch_select_device":  # the one device batch call without dense flags
                R += [(f"{nm}-host-flags", "full", lambda c, e, w=which: batch(w, c, e, True, flags=HOST), INVALID,
                       f"{nm}: d_flags_out {NODEV}", FULL)]
    R += [
        ("gpdb_images_batch_device-nobatch", "empty", lambda c, e: images(c, e), STATE,
         f"gpdb_images_batch_device: {NOBATCH_SET}", NONE),
        ("gpdb_images_batch_device-null-off", "full", lambda c, e: images(c, e, off=None), INVALID,
         "gpdb_images_batch_device: need hand_offsets[4] starting at 0", FULL),
        ("gpdb_images_batch_device-off0", "full", lambda c, e: images(c, e, off=I32(1, 1, 2, 3)), INVALID,
         "gpdb_images_batch_device: need hand_offsets[4] starting at 0", FULL),
        ("gpdb_images_batch_device-decrease", "full", lambda c, e: images(c, e, off=I32(0, 2, 1, 3)), INVALID,
         "gpdb_images_batch_device: hand_offsets decrease at cloud 1", FULL),
        ("gpdb_images_batch_device-null-hands", "full", lambda c, e: images(c, e, hands=None), INVALID,
         "gpdb_images_batch_device: null d_hands or d_images_out", FULL),
        ("gpdb_images_batch_device-host-hands", "full", lambda c, e: images(c, e, hands=HOST), INVALID,
         f"gpdb_images_batch_device: d_hands {NODEV}", FULL),
        ("gpdb_images_batch_device-host-out", "full", lambda c, e: images(c, e, out=HOST), INVALID,
         f"gpdb_images_batch_device: d_images_out {NODEV}", FULL),
    ]
    GRP = "need n_groups >= 0, hand_offsets[n_groups + 1] starting at 0 and cluster_offsets_out"
    for dev, nm in ((False, "gpdb_find_clusters_batch"), (True, "gpdb_find_clusters_batch_device")):
        R += [
            (f"{nm}-neg", "full", lambda c, e, d=dev: clusters(c, e, d, n=-1), INVALID, f"{nm}: {GRP}", FULL),
            (f"{nm}-null-coff", "full", lambda c, e, d=dev: clusters(c, e, d, coff=None), INVALID, f"{nm}: {GRP}", FULL),
            (f"{nm}-off0", "full", lambda c, e, d=dev: clusters(c, e, d, off=I32(1, 1, 2, 3)), INVALID, f"{nm}: {GRP}", FULL),
            (f"{nm}-decrease", "full", lambda c, e, d=dev: clusters(c, e, d, off=I32(0, 2, 1, 3)), INVALID,
             f"{nm}: hand_offsets decrease at group 1", FULL),
            (f"{nm}-null-hands", "full", lambda c, e, d=dev: clusters(c, e, d, hands=None), INVALID,
             f"{nm}: null hands or clusters_out", FULL),
        ]
    R += [("gpdb_find_clusters_batch_device-host-hands", "full", lambda c, e: clusters(c, e, True), INVALID,
           f"gpdb_find_clusters_batch_device: d_hands {NODEV}", FULL)]
    SISA = "need params, init_offsets[4] starting at 0, a result and hand_offsets_out"
    for dev, nm in ((False, "gpdb_sis_batch"), (True, "gpdb_sis_batch_device")):
        R += [
            (f"{nm}-nobatch", "empty", lambda c, e, d=dev: sis(c, e, d), STATE, f"{nm}: {NOBATCH}", NONE),
            (f"{nm}-null-params", "full", lambda c, e, d=dev: sis(c, e, d, sp=None), INVALID, f"{nm}: {SISA}", KEPT_NO_SIS),
            (f"{nm}-off0", "full", lambda c, e, d=dev: sis(c, e, d, off=I32(1, 3, 6, 9)), INVALID, f"{nm}: {SISA}",
             KEPT_NO_SIS),
            (f"{nm}-negative", "full", lambda c, e, d=dev: sis(c, e, d, sp=lib.sis_params(num_iterations=-1)), INVALID,
             f"{nm}: num_iterations, num_samples_per_iteration and min_inliers must not be negative", KEPT_NO_SIS),
            (f"{nm}-decrease", "full", lambda c, e, d=dev: sis(c, e, d, off=I32(0, 3, 2, 9)), INVALID,
             f"{nm}: init_offsets decrease at cloud 1", KEPT_NO_SIS),
            (f"{nm}-null-idx", "full", lambda c, e, d=dev: sis(c, e, d, idx=None), INVALID, f"{nm}: null init_idx",
             KEPT_NO_SIS),
            (f"{nm}-init-index", "full", lambda c, e, d=dev: sis(c, e, d, idx=bad_samples(e, 1, e.N[1])), INVALID,
             f"{nm}: init index {{n1}} at position 4 outside cloud 1 (N = {{n1}})", KEPT_NO_SIS),
            (f"{nm}-negative-index", "full", lambda c, e, d=dev: sis(c, e, d, idx=bad_samples(e, 2, -3)), INVALID,
             f"{nm}: init index -3 at position 5 outside cloud 1 (N = {{n1}})", KEPT_NO_SIS),
        ]
    R += [("gpdb_sis_batch_device-host-idx", "full", lambda c, e: sis(c, e, True, host_idx=1), INVALID,
           f"gpdb_sis_batch_device: d_init_idx {NODEV}", KEPT_NO_SIS),
          ("gpdb_sis_batch_device-host-hands", "full", lambda c, e: sis(c, e, True, hands=HOST), INVALID,
           f"gpdb_sis_batch_device: d_hands_out {NODEV}", KEPT_NO_SIS),
          ("gpdb_sis_batch_device-null-hands", "full", lambda c, e: sis(c, e, True, hands=None), INVALID,
           "gpdb_sis_batch_device: null d_hands_out", KEPT_NO_SIS)]
    for dev, nm in ((False, "gpdb_subsample_clouds"), (True, "gpdb_subsample_clouds_device")):
        out = "d_sample_idx_out" if dev else "sample_idx_out"
        R += [
            (f"{nm}-nobatch", "empty", lambda c, e, d=dev: subsample(c, e, d), STATE, f"{nm}: {NOBATCH_DEPTH}", NONE),
            (f"{nm}-neg", "full", lambda c, e, d=dev: subsample(c, e, d, n=-1), INVALID,
             f"{nm}: need num_samples >= 0 (got -1) and sample_offsets_out", FULL),
            (f"{nm}-null-off", "full", lambda c, e, d=dev: subsample(c, e, d, off=None), INVALID,
             f"{nm}: need num_samples >= 0 (got 2) and sample_offsets_out", FULL),
            (f"{nm}-null-idx", "full", lambda c, e, d=dev: subsample(c, e, d, idx=None), INVALID, f"{nm}: null {out}", FULL),
        ]
    R += [("gpdb_subsample_clouds_device-host-mask", "full", lambda c, e: subsample(c, e, True, mask=HOST), INVALID,
           f"gpdb_subsample_clouds_device: d_mask {NODEV}", FULL),
          ("gpdb_subsample_clouds_device-host-idx", "full", lambda c, e: subsample(c, e, True, idx=np.zeros(64, np.int32)),
           INVALID, f"gpdb_subsample_clouds_device: d_sample_idx_out {NODEV}", FULL),
          ("gpdb_get_clouds-nobatch", "empty", lambda c, e: L().gpdb_get_clouds(c.h, None, None, None, None), STATE,
           f"gpdb_get_clouds: {NOBATCH}", NONE),
          ("gpdb_classify_device-neg", "full", lambda c, e: classify(c, e, n=-1), INVALID, "gpdb_classify_device: bad arguments",
           FULL),
          ("gpdb_classify_device-host-images", "full", lambda c, e: classify(c, e, images_hwc=HOST), INVALID,
           f"gpdb_classify_device: d_images_hwc {NODEV}", FULL)]
    return R


ROWS = rows()


def test_rows_are_unique():
    ids = [r[0] for r in ROWS]
    assert len(ids) == len(set(ids))


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_message(env, row):
    _, setup, call, code, msg, after = row
    c = env.empty if setup == "empty" else env.ctx
    if setup == "full":
        setup_full(env)
        assert state(env, c) == FULL
    rc = call(c, env)
    assert rc == code
    assert L().gpdb_last_error(c.h).decode() == f"gpd_b200 error {code}: " + msg.format(**env.fmt)
    assert state(env, c) == after
