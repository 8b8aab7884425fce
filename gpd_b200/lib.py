"""ctypes binding of libgpd_b200.so — the CUDA product library (include/gpd_b200.h).

The library is built in-tree (gpd_b200/csrc/Makefile, __graft_entry__.build()). There is no CPU
fallback: if the shared object is missing this module raises, and every compute call returns
GPDB_ERR_CUDA when no sm_90 device is present.
"""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
# GPD_B200_LIB overrides the library path (A/B comparison of builds during development); default: the in-tree build
SO_PATH = os.environ.get("GPD_B200_LIB") or os.path.join(_HERE, "libgpd_b200.so")
_LIB = None

EXPORTS = list(abi.PROTOTYPES)

# gpdb_debug_path_counts: index of each event in the returned array (include/gpd_b200.h)
PATH_EVENTS = ["frames_tier1", "frames_tier2", "hands_tile", "hands_global", "hands_full_slab", "images2_box",
               "images2_nonunit", "images_global", "images2_cast_in_place", "images2_draw_in_place", "images2_stash_full",
               "images_cast_in_place", "images_draw_in_place", "images_voxel_list_full", "images_ball_record_full",
               "label_walk"]


class GpdbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[{code}] {msg}")
        self.code = code


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(SO_PATH):
        raise RuntimeError(
            f"{SO_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). gpd_b200 has no CPU fallback.")
    L = C.CDLL(SO_PATH)
    for name, (restype, argtypes) in abi.PROTOTYPES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _LIB = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def default_params(**over):
    p = abi.Params()
    lib().gpdb_params_default(C.byref(p))
    chan = over.pop("channels", None)
    if chan is not None:
        p.image_num_channels = chan
    return abi.set_fields(p, **over)


def preprocess_params(**over):
    """gpdb_preprocess_params with the reference defaults (cfg/eigen_params.cfg:16-21), overridden by keyword."""
    p = abi.PreprocessParams()
    lib().gpdb_preprocess_params_default(C.byref(p))
    return abi.set_fields(p, **over)


def sis_params(**over):
    """gpdb_sis_params with the reference defaults (gpdb_sis_params_default), overridden by keyword (cfg key names)."""
    p = abi.SisParams()
    lib().gpdb_sis_params_default(C.byref(p))
    return abi.set_fields(p, **over)


def plane_params(**over):
    """gpdb_plane_params with the reference's values (gpdb_plane_params_default: threshold 0.01, 50 iterations,
    probability 0.99, seed 0), overridden by keyword."""
    p = abi.PlaneParams()
    lib().gpdb_plane_params_default(C.byref(p))
    return abi.set_fields(p, **over)


def sensor_params(**fields):
    """gpdb_sensor_params (include/gpd_b200_sensor.h): every field 0 (a clean render, gpdb_sensor_params_default),
    overridden by keyword: baseline (m), lateral_sigma, disparity_sigma, disparity_step (pixels), min_cos_incidence,
    shadow_tolerance, dropout."""
    p = abi.SensorParams()
    lib().gpdb_sensor_params_default(C.c_void_p(C.addressof(p)))
    for k in fields:
        if k not in dict(abi.SensorParams._fields_):
            raise TypeError(f"sensor_params: unknown field {k!r}")
    return abi.set_fields(p, **fields)


def debug_sensor_table():
    """gpdb_debug_sensor_table: the float64 inverse-normal table [4097] the sensor draws interpolate (gpd_b200_sensor.h 2).
    Needs no device."""
    t = np.zeros(4097, np.float64)
    rc = lib().gpdb_debug_sensor_table(_p(t))
    if rc != len(t):
        raise GpdbError(rc, "gpdb_debug_sensor_table failed")
    return t


def read_weights_file(weights_file, channels, model_file=None):
    """Host-side import of a .caffemodel or an OpenVINO IR into the eight arrays of the .bin layout (no device needed).
    Returns (arrays, relu_layers)."""
    sizes = [20 * channels * 25, 20, 50 * 20 * 25, 50, 500 * 7200, 500, 1000, 2]
    arrs = [np.zeros(s, np.float32) for s in sizes]
    ptrs = (C.c_void_p * 8)(*[a.ctypes.data for a in arrs])
    relu = C.c_int32(-1)
    err = C.create_string_buffer(512)
    rc = lib().gpdb_read_weights_file(None if model_file is None else model_file.encode(), weights_file.encode(), channels, ptrs,
                                      C.byref(relu), err, 512)
    if rc != 0:
        raise GpdbError(rc, err.value.decode())
    return arrs, relu.value


def weight_sizes(channels):
    """Values in each of the eight arrays of the .bin layout (gpdb_set_weights) for a network of `channels` inputs."""
    return [20 * channels * 25, 20, 50 * 20 * 25, 50, 500 * 7200, 500, 1000, 2]


def train_params(optimizer="sgd", lr=1e-5, momentum=0.9, weight_decay=0.0, betas=(0.9, 0.999), eps=1e-8):
    """gpdb_train_params: optimizer "sgd" (torch.optim.SGD, dampening 0) or "adam" (torch.optim.Adam, L2 weight decay).
    The defaults are the reference's pytorch/train_net.py (SGD, lr 1e-5, momentum 0.9)."""
    opt = {"sgd": 0, "adam": 1}.get(optimizer)
    if opt is None:
        raise ValueError(f"optimizer: 'sgd' or 'adam', got {optimizer!r}")
    return abi.TrainParams(opt, lr, momentum, weight_decay, betas[0], betas[1], eps)


def _weight_ptrs(arrays, channels):
    sizes = weight_sizes(channels)
    if len(arrays) != 8:
        raise ValueError(f"need 8 weight arrays, got {len(arrays)}")
    arrs = [np.ascontiguousarray(a, dtype=np.float32).ravel() for a in arrays]
    for i, (a, s) in enumerate(zip(arrs, sizes)):
        if a.size != s:
            raise ValueError(f"weight array {i}: {a.size} values, need {s} for {channels} channels")
    return arrs, (C.c_void_p * 8)(*[a.ctypes.data for a in arrs])


def write_weights_dir(d, channels, arrays):
    """gpdb_write_weights_dir: the eight arrays as {conv1,conv2,ip1,ip2}_{weights,biases}.bin in the directory d, what
    Context.load_weights_dir and the reference's EigenClassifier read."""
    _, ptrs = _weight_ptrs(arrays, channels)
    rc = lib().gpdb_write_weights_dir(os.fspath(d).encode(), int(channels), ptrs)
    if rc != 0:
        raise GpdbError(rc, f"gpdb_write_weights_dir({os.fspath(d)!r}, {channels}) failed")


def pack_clouds(clouds):
    """The CSR arrays of gpdb_set_clouds / gpdb_preprocess_clouds for a list of cloud dicts (xyz [N, 3], normals [N, 3],
    optional cam_source [N, K], optional view_points [K, 3]): point offsets [B+1], xyz, normals (None when no cloud has
    them, as raw clouds whose normals are estimated; ValueError when only some have them), cam_source (None when no
    cloud has one; a cloud without one is seen by all its cameras), camera counts [B] and view points, each concatenated
    in cloud order."""
    if not clouds:
        raise ValueError("pack_clouds: need at least one cloud")
    xyz = [np.asarray(c["xyz"], dtype=np.float32).reshape(-1, 3) for c in clouds]
    has_nrm = [c.get("normals") is not None for c in clouds]
    if any(has_nrm) and not all(has_nrm):
        raise ValueError(f"pack_clouds: clouds {[i for i, h in enumerate(has_nrm) if not h]} have no normals; either every "
                         "cloud has normals or none has")
    nrm = [np.asarray(c["normals"], dtype=np.float64).reshape(-1, 3) for c in clouds] if all(has_nrm) else None
    vps = [np.asarray(c.get("view_points") if c.get("view_points") is not None else np.zeros((1, 3)), dtype=np.float64).reshape(-1, 3)
           for c in clouds]
    ks = np.array([len(v) for v in vps], dtype=np.int32)
    offsets = np.zeros(len(clouds) + 1, np.int32)
    offsets[1:] = np.cumsum([len(x) for x in xyz])
    cam = None
    if any(c.get("cam_source") is not None for c in clouds):
        blocks = []
        for c, x, k in zip(clouds, xyz, ks):
            cs = c.get("cam_source")
            blocks.append(np.ones((len(x), k), np.int32) if cs is None else np.asarray(cs, dtype=np.int32).reshape(len(x), k))
        cam = np.ascontiguousarray(np.concatenate([b.ravel() for b in blocks]))
    return {"offsets": offsets, "xyz": np.ascontiguousarray(np.concatenate(xyz)),
            "normals": None if nrm is None else np.ascontiguousarray(np.concatenate(nrm)),
            "cam_source": cam, "n_cameras": ks, "view_points": np.ascontiguousarray(np.concatenate(vps))}


def pack_meshes(meshes):
    """The CSR arrays of gpdb_render_depth / gpdb_sample_meshes for a list of (vertices [V, 3], faces [F, 3]) meshes, faces
    indexing their own mesh's vertices from 0: {"vertex_offsets" [B+1], "vertices" float32 [sum V, 3], "face_offsets"
    [B+1], "faces" int32 [sum F, 3]}, each concatenated in mesh order."""
    if not meshes:
        raise ValueError("pack_meshes: need at least one mesh")
    vs = [np.asarray(v, dtype=np.float32).reshape(-1, 3) for v, _ in meshes]
    fs = [np.asarray(f, dtype=np.int32).reshape(-1, 3) for _, f in meshes]
    voff = np.zeros(len(meshes) + 1, np.int32)
    voff[1:] = np.cumsum([len(v) for v in vs])
    foff = np.zeros(len(meshes) + 1, np.int32)
    foff[1:] = np.cumsum([len(f) for f in fs])
    return {"vertex_offsets": voff, "vertices": np.ascontiguousarray(np.concatenate(vs)),
            "face_offsets": foff, "faces": np.ascontiguousarray(np.concatenate(fs))}


def depth_camera(width, height, fx, fy, cx, cy, pose=None, depth_scale=0.001, min_depth=0.0, max_depth=float("inf")):
    """A gpdb_depth_camera (include/gpd_b200_depth.h): pinhole intrinsics in pixels, pose = camera-to-world [R | t] as a
    3 x 4 (or 4 x 4) array, identity when None; depth_scale in metres per stored unit (0.001 for uint16 millimetres, 1.0
    for float32 metres); a pixel is valid iff min_depth <= z <= max_depth."""
    c = abi.DepthCamera()
    c.width, c.height = int(width), int(height)
    c.fx, c.fy, c.cx, c.cy = float(fx), float(fy), float(cx), float(cy)
    P = np.eye(4)[:3] if pose is None else np.asarray(pose, dtype=np.float64)[:3, :4]
    c.pose[:] = [float(v) for v in P.ravel()]
    c.depth_scale, c.min_depth, c.max_depth = float(depth_scale), float(min_depth), float(max_depth)
    return c


def _depth_cameras(n_cameras, cameras):
    ks = _host_i32("n_cameras", n_cameras)
    cams = list(cameras)
    if len(cams) != int(ks.sum()):
        raise ValueError(f"cameras: {len(cams)} descriptions, need sum(n_cameras) = {int(ks.sum())}")
    arr = (abi.DepthCamera * max(len(cams), 1))(*cams)
    vps = np.array([[c.pose[3], c.pose[7], c.pose[11]] for c in cams], dtype=np.float64).reshape(-1, 3)
    return ks, arr, vps


def _depth_views(views, name):
    """(n_cameras, cameras, format, concatenated images) of the host depth views of preprocess_depth[_organized]."""
    imgs, cams, ks = [], [], []
    for view in views:
        ks.append(len(view))
        for img, cam in view:
            imgs.append(np.asarray(img))
            cams.append(cam)
    dts = {a.dtype for a in imgs}
    if len(dts) != 1 or next(iter(dts)) not in (np.dtype(np.uint16), np.dtype(np.float32)):
        raise TypeError(f"{name}: need every image uint16 or every image float32, got {sorted(map(str, dts))}")
    fmt = abi.DEPTH_U16 if next(iter(dts)) == np.uint16 else abi.DEPTH_F32
    for i, (a, c) in enumerate(zip(imgs, cams)):
        if a.shape != (c.height, c.width):
            raise ValueError(f"{name}: image {i} has shape {a.shape}, its camera is {c.height} x {c.width}")
    return ks, cams, fmt, np.ascontiguousarray(np.concatenate([a.ravel() for a in imgs]))


def _organized_shapes(clouds, view_points):
    """widths [B], heights [B] (int32) and view points [B, 3] (float32) of [H, W, 3] organized clouds."""
    for i, c in enumerate(clouds):
        if len(c.shape) != 3 or c.shape[2] != 3:
            raise ValueError(f"clouds[{i}]: shape {tuple(c.shape)}, need [H, W, 3]")
    H = np.array([c.shape[0] for c in clouds], np.int32)
    W = np.array([c.shape[1] for c in clouds], np.int32)
    B = len(clouds)
    vp = np.zeros((B, 3), np.float32) if view_points is None else np.ascontiguousarray(view_points, np.float32).reshape(-1, 3)
    if len(vp) != B:
        raise ValueError(f"view_points: {len(vp)} rows, need one per cloud ({B})")
    return W, H, np.ascontiguousarray(vp)


def _organized_split(nrm, dist, W, H):
    """The concatenated outputs of gpdb_normals_organized[_device] as per-cloud [H, W, 3] normals and [H, W] distances."""
    ns, ds, o = [], [], 0
    for w, h in zip(W.tolist(), H.tolist()):
        ns.append(nrm[3 * o:3 * (o + w * h)].reshape(h, w, 3))
        ds.append(None if dist is None else dist[o:o + w * h].reshape(h, w))
        o += w * h
    return ns, ds


def pack_samples(sample_lists):
    """The CSR arrays of gpdb_detect_batch for one list of cloud-local sample indices per cloud: (offsets [B+1], indices)."""
    arrs = [np.asarray(s, dtype=np.int32).ravel() for s in sample_lists]
    offsets = np.zeros(len(arrs) + 1, np.int32)
    offsets[1:] = np.cumsum([len(a) for a in arrs])
    return offsets, np.ascontiguousarray(np.concatenate(arrs) if arrs else np.zeros(0, np.int32))


def split_batch_result(out, sample_offsets, cand_offsets):
    """Per-cloud views of one batch result (abi.result_to_numpy dict): the slices of every per-sample / per-pose array at
    sample_offsets and of the candidates (and images) at cand_offsets."""
    views = []
    for b in range(len(sample_offsets) - 1):
        s0, s1, c0, c1 = sample_offsets[b], sample_offsets[b + 1], cand_offsets[b], cand_offsets[b + 1]
        v = {"n_samples": s1 - s0, "poses_per_sample": out["poses_per_sample"], "n_candidates": c1 - c0,
             "candidates": out["candidates"][c0:c1], "images": None if out["images"] is None else out["images"][c0:c1]}
        for k in ("frame_valid", "frames", "pose_flags", "pose_scores"):
            v[k] = None if out[k] is None else out[k][s0:s1]
        views.append(v)
    return views


POSE_BYTES = C.sizeof(abi.Pose)


def poses_from_tensor(t):
    """The gpdb_pose records of a uint8 tensor [n, POSE_BYTES] (as the *_tensors methods return them) as a host
    abi.POSE_DTYPE array."""
    return t.detach().cpu().numpy().reshape(-1).view(abi.POSE_DTYPE).copy()


def _host_i32(name, a, n=None):
    a = np.ascontiguousarray(a, dtype=np.int32).ravel()
    if n is not None and len(a) != n:
        raise ValueError(f"{name}: {len(a)} entries, need {n}")
    return a


def _device_arg(name, t, dtype, device, numel, optional=False):
    """The device pointer of a tensor argument of the gpdb_*_device calls, after the checks the library cannot make
    (dtype, contiguity, size); ValueError / TypeError before any library call. An empty tensor passes NULL."""
    import torch
    if t is None:
        if optional:
            return None
        raise ValueError(f"{name}: a CUDA tensor is required")
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda" or t.device.index != device:
        where = t.device if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"{name}: need a tensor on cuda:{device}, got {where}")
    if t.dtype != dtype:
        raise TypeError(f"{name}: need {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: need a contiguous tensor")
    if t.numel() != numel:
        raise ValueError(f"{name}: {t.numel()} elements, need {numel}")
    return C.c_void_p(t.data_ptr()) if numel else None


class Context:
    """One gpdb_ctx: one CUDA device + stream (gpdb_create ... gpdb_destroy)."""

    def __init__(self, params):
        self.params = params
        self.h = C.c_void_p()
        rc = lib().gpdb_create(C.byref(params), C.byref(self.h))
        if rc != 0:
            self.h = None
            raise GpdbError(rc, lib().gpdb_last_error(None).decode())
        self._keep = []
        self._n_clouds = 0  # clouds of the installed batch (gpdb_detect_batch reads that many + 1 sample offsets)
        self._batch = None  # (point offsets, camera counts, view point blocks, has source indices) of the installed batch
        self._stream = None  # the torch stream the *_tensors methods last moved the context to
        self._sis_shape = None  # (B, num_iterations) of the last successful SIS call: sizes sis_positions' arrays
        self._n_raw = None  # raw points (pixels) of the preprocessing call that installed the batch: the length of a mask

    def close(self):
        if getattr(self, "h", None):
            lib().gpdb_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _check(self, rc):
        if rc < 0:
            raise GpdbError(rc, lib().gpdb_last_error(self.h).decode())
        return rc

    def load_weights_dir(self, d):
        if not d.endswith("/"):
            d += "/"
        self._check(lib().gpdb_load_weights_dir(self.h, d.encode()))

    def load_weights_file(self, weights_file, model_file=None):
        """.bin directory, .caffemodel or OpenVINO IR (.bin + .xml), as Classifier::create's weights_file / model_file."""
        self._check(lib().gpdb_load_weights_file(self.h, None if model_file is None else model_file.encode(), weights_file.encode()))

    def set_weights(self, arrays):
        arrs = [np.ascontiguousarray(a, dtype=np.float32).ravel() for a in arrays]
        self._check(lib().gpdb_set_weights(self.h, *[_p(a) for a in arrs]))

    def set_cloud(self, xyz, normals, cam_source=None, view_points=None):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32)
        normals = np.ascontiguousarray(normals, dtype=np.float64)
        vp = np.ascontiguousarray(view_points if view_points is not None else np.zeros((1, 3)), dtype=np.float64)
        cam = None if cam_source is None else np.ascontiguousarray(cam_source, dtype=np.int32)
        self._check(lib().gpdb_set_cloud(self.h, _p(xyz), _p(normals), _p(cam), xyz.shape[0], _p(vp), vp.shape[0]))

    def preprocess(self, xyz, cam_source=None, view_points=None, pp=None, normals=None, read_back=True):
        """CandidatesGenerator::preprocessPointCloud on the device (gpdb_preprocess): NaN / workspace filter,
        voxelisation, normal estimation; installs the processed cloud. Returns the processed cloud as a dict
        (xyz, normals, cam_source, view_points, src) or just N' when read_back is False."""
        xyz = np.ascontiguousarray(xyz, dtype=np.float32)
        vp = np.ascontiguousarray(view_points if view_points is not None else np.zeros((1, 3)), dtype=np.float64)
        cam = None if cam_source is None else np.ascontiguousarray(cam_source, dtype=np.int32)
        nrm = None if normals is None else np.ascontiguousarray(normals, dtype=np.float64)
        if pp is None:
            pp = preprocess_params()
        n = self._check(lib().gpdb_preprocess(self.h, _p(xyz), _p(nrm), _p(cam), xyz.shape[0], _p(vp), vp.shape[0],
                                              C.byref(pp)))
        if not read_back:
            return n
        out = self.get_cloud() if n > 0 else {"xyz": np.zeros((0, 3), np.float32), "normals": np.zeros((0, 3)),
                                              "cam_source": np.zeros((0, vp.shape[0]), np.int32)}
        out["view_points"] = vp
        if n > 0:
            src = np.zeros(n, np.int32)
            self._check(lib().gpdb_get_cloud_source_index(self.h, _p(src)))
            out["src"] = src
        else:
            out["src"] = np.zeros(0, np.int32)
        return out

    # ---- multi-GPU sharding inside the boundary (gpdb_comm_*, SURVEY.md 8(e)) ----
    def comm_init(self, unique_id, rank, nranks):
        """ncclCommInitRank on this context's device; unique_id = 128 bytes from comm_unique_id() of one rank."""
        buf = C.create_string_buffer(bytes(unique_id), 128)
        self._check(lib().gpdb_comm_init(self.h, buf, int(rank), int(nranks)))
        self.rank, self.nranks = int(rank), int(nranks)

    def set_cloud_bcast(self, root, xyz=None, normals=None, cam_source=None, view_points=None):
        """gpdb_set_cloud on every rank from the root's host arrays (ncclBroadcast of the device copies)."""
        if xyz is None:
            return self._check(lib().gpdb_set_cloud_bcast(self.h, int(root), None, None, None, 0, None, 0))
        xyz = np.ascontiguousarray(xyz, dtype=np.float32)
        normals = np.ascontiguousarray(normals, dtype=np.float64)
        vp = np.ascontiguousarray(view_points if view_points is not None else np.zeros((1, 3)), dtype=np.float64)
        cam = None if cam_source is None else np.ascontiguousarray(cam_source, dtype=np.int32)
        return self._check(lib().gpdb_set_cloud_bcast(self.h, int(root), _p(xyz), _p(normals), _p(cam), xyz.shape[0], _p(vp), vp.shape[0]))

    def detect_sharded(self, sample_idx):
        """gpdb_detect over sharded samples: gathered pose_flags / pose_scores of all ranks + this rank's pose records."""
        sidx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        res = abi.Result()
        self._check(lib().gpdb_detect_sharded(self.h, _p(sidx), len(sidx), C.byref(res)))
        n, P, nc = res.n_samples, res.poses_per_sample, res.n_candidates
        out = {"pose_flags": np.ctypeslib.as_array(res.pose_flags, (n, P)).copy(),
               "pose_scores": np.ctypeslib.as_array(res.pose_scores, (n, P)).copy(),
               "n_candidates": nc, "n_total_candidates": res.n_total_candidates,
               "candidates": np.frombuffer(C.string_at(res.candidates, nc * C.sizeof(abi.Pose)), dtype=abi.POSE_DTYPE).copy()
               if nc else np.zeros(0, dtype=abi.POSE_DTYPE)}
        lib().gpdb_free_result(C.byref(res))
        return out

    def detect_sharded_raw(self, sidx_i32, res):
        return self._check(lib().gpdb_detect_sharded(self.h, _p(sidx_i32), len(sidx_i32), C.byref(res)))

    def detect_sharded_resident(self, d_sidx_local_ptr, n_local, slot_samples, d_gathered_ptr, stats):
        return self._check(lib().gpdb_detect_sharded_resident(self.h, C.c_void_p(d_sidx_local_ptr), int(n_local), int(slot_samples),
                                                              C.c_void_p(d_gathered_ptr), C.byref(stats)))

    def reevaluate(self, hands):
        """HandSearch::reevaluateHypotheses against the installed cloud: (labels int32, re-labelled records)."""
        hands = np.array(hands, dtype=abi.POSE_DTYPE, copy=True)
        labels = np.zeros(len(hands), np.int32)
        self._check(lib().gpdb_reevaluate(self.h, _p(hands), len(hands), _p(labels)))
        return labels, hands

    def find_clusters(self, hands, min_inliers):
        """Clustering::findClusters (remove_inliers = false) on the device; hands / result: abi.POSE_DTYPE records."""
        hands = np.ascontiguousarray(hands, dtype=abi.POSE_DTYPE)
        out = np.zeros(len(hands), dtype=abi.POSE_DTYPE)
        n = self._check(lib().gpdb_find_clusters(self.h, _p(hands), len(hands), int(min_inliers), _p(out)))
        return out[:n].copy()

    # ---- batch bookkeeping: what the library installed, kept here to size the outputs of later batch calls ----
    def _drop_batch(self):
        self._n_clouds, self._batch, self._sis_shape, self._n_raw = 0, None, None, None

    def _install(self, call, offsets, n_cameras, view_points, n_raw=None):
        """Runs call(), which installs a batch of len(n_cameras) clouds, and records that batch: offsets [B+1] are its
        point offsets (read by set_clouds, written by the preprocessing calls), n_raw the raw points of a preprocessing
        call, whose clouds keep source indices (None after set_clouds). A failed install leaves no batch in the library,
        so none is recorded. Returns offsets."""
        self._drop_batch()
        self._check(call())
        self._n_clouds = len(n_cameras)
        self._batch = (offsets, n_cameras, view_points, n_raw is not None)
        self._n_raw = n_raw
        return offsets

    def _n_points(self):
        return int(self._batch[0][-1]) if self._batch is not None else 0

    def set_clouds(self, clouds):
        """gpdb_set_clouds: installs a batch of processed clouds (list of dicts as set_cloud takes) beside the single cloud."""
        pk = pack_clouds(clouds)
        self._install(lambda: lib().gpdb_set_clouds(self.h, len(clouds), _p(pk["offsets"]), _p(pk["xyz"]), _p(pk["normals"]),
                                                    _p(pk["cam_source"]), _p(pk["n_cameras"]), _p(pk["view_points"])),
                      pk["offsets"], pk["n_cameras"], pk["view_points"])

    def preprocess_clouds(self, raw_clouds, pp=None, read_back=True):
        """gpdb_preprocess_clouds: preprocess() of every raw cloud (list of dicts: xyz, optional normals, optional
        cam_source, view_points) in one call, the processed clouds installed as the batch (detect_batch works straight
        after it). Returns one dict per cloud as preprocess() returns (xyz, normals, cam_source, view_points, src), or the
        processed point offsets [B+1] when read_back is False. A cloud the filter empties stays, with no points."""
        pk = pack_clouds(raw_clouds)
        if pp is None:
            pp = preprocess_params()
        poff = np.zeros(len(raw_clouds) + 1, np.int32)
        self._install(lambda: lib().gpdb_preprocess_clouds(self.h, len(raw_clouds), _p(pk["offsets"]), _p(pk["xyz"]),
                                                           _p(pk["normals"]), _p(pk["cam_source"]), _p(pk["n_cameras"]),
                                                           _p(pk["view_points"]), C.byref(pp), _p(poff)),
                      poff, pk["n_cameras"], pk["view_points"], int(pk["offsets"][-1]))
        return self.get_clouds() if read_back else poff

    def get_clouds(self):
        """gpdb_get_clouds: the installed batch as one dict per cloud (xyz, normals, cam_source [N_b, K_b], view_points,
        and src, the index into the cloud's raw points, after preprocess_clouds)."""
        if self._batch is None:
            self._check(lib().gpdb_get_clouds(self.h, None, None, None, None))  # raises: no batch installed
        offsets, ks, vps, has_src = self._batch
        n = int(offsets[-1])
        xyz = np.zeros((n, 3), np.float32)
        nrm = np.zeros((n, 3), np.float64)
        cam = np.zeros(int(np.sum(np.diff(offsets) * ks)), np.int32)
        src = np.zeros(n, np.int32) if has_src else None
        self._check(lib().gpdb_get_clouds(self.h, _p(xyz), _p(nrm), _p(cam), _p(src)))
        out, c0, v0 = [], 0, 0
        for b in range(len(ks)):
            o0, o1, k = int(offsets[b]), int(offsets[b + 1]), int(ks[b])
            d = {"xyz": xyz[o0:o1].copy(), "normals": nrm[o0:o1].copy(), "cam_source": cam[c0:c0 + (o1 - o0) * k].reshape(o1 - o0, k).copy(),
                 "view_points": vps[v0:v0 + k].copy()}
            if has_src:
                d["src"] = src[o0:o1].copy()
            out.append(d)
            c0, v0 = c0 + (o1 - o0) * k, v0 + k
        return out

    def _pack_batch_samples(self, sample_lists):
        # the C-ABI takes no cloud count: it reads and writes B + 1 offsets for the B installed clouds
        if len(sample_lists) != self._n_clouds:
            raise ValueError(f"{len(sample_lists)} sample lists for a batch of {self._n_clouds} clouds (one list per cloud)")
        return pack_samples(sample_lists)

    def _batch_result(self, fn, sample_lists):
        offsets, sidx = self._pack_batch_samples(sample_lists)
        res = abi.Result()
        coff = np.zeros(len(offsets), np.int32)
        self._check(fn(self.h, _p(offsets), _p(sidx), C.byref(res), _p(coff)))
        S, Cc = self.params.image_size, self.params.image_num_channels
        out = abi.result_to_numpy(res, S * S * Cc)
        lib().gpdb_free_result(C.byref(res))
        return split_batch_result(out, offsets, coff)

    def detect_batch(self, sample_lists):
        """gpdb_detect_batch: one list of cloud-local sample indices per installed cloud; returns one result dict per
        cloud (views of the single batch result), each as detect() would return for that cloud alone."""
        return self._batch_result(lib().gpdb_detect_batch, sample_lists)

    def hand_search_batch(self, sample_lists):
        """gpdb_hand_search_batch: hand_search() of every installed cloud in one call (no images, NaN scores, no weights
        needed); returns one result dict per cloud, as detect_batch does."""
        return self._batch_result(lib().gpdb_hand_search_batch, sample_lists)

    def set_clouds_samples(self, positions):
        """gpdb_set_clouds_samples: Cloud::setSamples for every installed cloud (one [m_b, 3] float64 array per cloud,
        m_b may be 0); returns per cloud the cloud-local sample indices N_b .. N_b + m_b - 1 that address them."""
        if len(positions) != self._n_clouds:
            raise ValueError(f"{len(positions)} position arrays for a batch of {self._n_clouds} clouds (one per cloud)")
        arrs = [np.asarray(p, dtype=np.float64).reshape(-1, 3) for p in positions]
        poff = np.zeros(len(arrs) + 1, np.int32)
        poff[1:] = np.cumsum([len(a) for a in arrs])
        sm = np.ascontiguousarray(np.concatenate(arrs) if arrs else np.zeros((0, 3)))
        self._check(lib().gpdb_set_clouds_samples(self.h, _p(poff), _p(sm)))
        npts = np.diff(self._batch[0])
        return [np.arange(npts[b], npts[b] + len(a), dtype=np.int32) for b, a in enumerate(arrs)]

    def find_clusters_batch(self, groups, min_inliers):
        """gpdb_find_clusters_batch: find_clusters() on every group of hands (list of abi.POSE_DTYPE arrays) in one call;
        returns one cluster array per group."""
        arrs = [np.asarray(g, dtype=abi.POSE_DTYPE).ravel() for g in groups]
        hoff = np.zeros(len(arrs) + 1, np.int32)
        hoff[1:] = np.cumsum([len(a) for a in arrs])
        hands = np.ascontiguousarray(np.concatenate(arrs) if arrs else np.zeros(0, abi.POSE_DTYPE))
        out = np.zeros(len(hands), dtype=abi.POSE_DTYPE)
        coff = np.zeros(len(arrs) + 1, np.int32)
        self._check(lib().gpdb_find_clusters_batch(self.h, len(arrs), _p(hoff), _p(hands), int(min_inliers), _p(out), _p(coff)))
        return [out[coff[g]:coff[g + 1]].copy() for g in range(len(arrs))]

    def reevaluate_batch(self, hand_lists):
        """gpdb_reevaluate_batch: reevaluate() of every group of hands (one abi.POSE_DTYPE array per installed cloud, may
        be empty) against its cloud in one call. Returns (labels, records): one int32 array and one re-labelled record
        array per group."""
        if self._batch is not None and len(hand_lists) != self._n_clouds:  # no batch: the library names the state error
            raise ValueError(f"{len(hand_lists)} hand lists for a batch of {self._n_clouds} clouds (one list per cloud)")
        arrs = [np.asarray(h, dtype=abi.POSE_DTYPE).ravel() for h in hand_lists]
        hoff = np.zeros(len(arrs) + 1, np.int32)
        hoff[1:] = np.cumsum([len(a) for a in arrs])
        hands = np.ascontiguousarray(np.concatenate(arrs) if arrs else np.zeros(0, abi.POSE_DTYPE))
        labels = np.zeros(len(hands), np.int32)
        self._check(lib().gpdb_reevaluate_batch(self.h, _p(hoff), _p(hands), _p(labels)))
        return ([labels[hoff[g]:hoff[g + 1]].copy() for g in range(len(arrs))],
                [hands[hoff[g]:hoff[g + 1]].copy() for g in range(len(arrs))])

    def detect_batch_select(self, sample_lists, num_selected):
        """gpdb_detect_batch_select: the num_selected best candidates of every cloud; returns one record array per cloud."""
        offsets, sidx = self._pack_batch_samples(sample_lists)
        res = abi.Result()
        soff = np.zeros(len(offsets), np.int32)
        self._check(lib().gpdb_detect_batch_select(self.h, _p(offsets), _p(sidx), int(num_selected), C.byref(res), _p(soff)))
        out = abi.result_to_numpy(res, 0)
        lib().gpdb_free_result(C.byref(res))
        return [out["candidates"][soff[b]:soff[b + 1]] for b in range(len(offsets) - 1)]

    def sis_batch(self, init_lists, **sis):
        """gpdb_sis_batch: SequentialImportanceSampling::detectGrasps on every installed cloud in one call, from one list of
        cloud-local initial point indices per cloud; keywords are gpdb_sis_params fields (sis_params). Returns a dict:
        "hands" one record array per cloud (hands with score > min_score, or their clusters when min_inliers > 0),
        "n_samples" the kept positions, "n_total_candidates" the classified candidates, and the positions of
        sis_positions()."""
        offsets, idx = self._pack_batch_samples(init_lists)
        sp = sis_params(**sis)
        res = abi.Result()
        hoff = np.zeros(len(offsets), np.int32)
        self._sis_shape = None  # a failed call leaves nothing to read back
        self._check(lib().gpdb_sis_batch(self.h, C.byref(sp), _p(offsets), _p(idx), C.byref(res), _p(hoff)))
        self._sis_shape = (len(hoff) - 1, sp.num_iterations)
        out = abi.result_to_numpy(res, 0)
        lib().gpdb_free_result(C.byref(res))
        return {"hands": [out["candidates"][hoff[b]:hoff[b + 1]] for b in range(len(hoff) - 1)], "n_samples": out["n_samples"],
                "n_total_candidates": out["n_total_candidates"], **self.sis_positions()}

    def sis_positions(self):
        """gpdb_sis_positions: per cloud, "evaluated" the positions of every round [n, 3] in round order, "round_counts"
        [B, num_iterations], and "kept" the positions that carried a hand [k, 3], initial samples first. The arrays are
        sized by the batch of that call; after a new batch is installed there is nothing to read (GpdbError)."""
        if self._sis_shape is None:  # the library holds no record either: let it name the error
            self._check(lib().gpdb_sis_positions(self.h, None, None, None, None, None))
            raise GpdbError(-3, "sis_positions: no successful SIS call on the installed batch")
        B, R = self._sis_shape
        eoff, koff, rcount = np.zeros(B + 1, np.int32), np.zeros(B + 1, np.int32), np.zeros(B * R, np.int32)
        self._check(lib().gpdb_sis_positions(self.h, _p(eoff), _p(rcount), None, _p(koff), None))
        ev, kept = np.zeros((int(eoff[-1]), 3)), np.zeros((int(koff[-1]), 3))
        self._check(lib().gpdb_sis_positions(self.h, None, None, _p(ev), None, _p(kept)))
        return {"evaluated": [ev[eoff[b]:eoff[b + 1]] for b in range(B)], "round_counts": rcount.reshape(B, R),
                "kept": [kept[koff[b]:koff[b + 1]] for b in range(B)]}

    # ---- device-resident batches (gpdb_*_device): CUDA tensors in, CUDA tensors out -----------------------------------
    # Every method checks device, dtype, contiguity and size of its tensors before the library call, moves the context
    # to torch.cuda.current_stream() (inputs made ready on it need no synchronisation; later calls of this context run
    # there too) and allocates its outputs with torch. Sizes and offsets are host arrays.

    def _torch_stream(self):
        import torch
        s = torch.cuda.current_stream(self.params.device).cuda_stream
        if s != self._stream:
            self.set_stream(s)
            self._stream = s

    def _cloud_tensors(self, point_offsets, xyz, normals, cam_source, n_cameras, view_points, normals_optional):
        off = _host_i32("point_offsets", point_offsets)
        B = len(off) - 1
        if B < 1:
            raise ValueError("point_offsets: need at least two entries (one cloud)")
        ks = _host_i32("n_cameras", n_cameras, B)
        vp = np.ascontiguousarray(view_points, dtype=np.float64).reshape(-1, 3)
        if len(vp) != int(ks.sum()):
            raise ValueError(f"view_points: {len(vp)} rows, need sum(n_cameras) = {int(ks.sum())}")
        import torch
        dev = self.params.device
        M = int(off[-1])
        ptrs = (_device_arg("xyz", xyz, torch.float32, dev, 3 * M),
                _device_arg("normals", normals, torch.float64, dev, 3 * M, optional=normals_optional),
                _device_arg("cam_source", cam_source, torch.int32, dev, int(np.sum(np.diff(off).astype(np.int64) * ks)),
                            optional=True))
        self._torch_stream()
        return off, ks, vp, ptrs

    def preprocess_clouds_tensors(self, point_offsets, xyz, n_cameras, view_points, cam_source=None, normals=None, pp=None):
        """gpdb_preprocess_clouds_device: preprocess_clouds() of raw clouds held in CUDA tensors, concatenated (cloud b:
        rows point_offsets[b] .. point_offsets[b+1]-1 of xyz [M, 3] float32 and normals [M, 3] float64 or None; cam_source
        int32 holding the N_b x K_b blocks one after the other, or None). point_offsets [B+1], n_cameras [B] and
        view_points [sum K_b, 3] are host arrays. Installs the processed batch; returns its point offsets [B+1]."""
        off, ks, vp, (px, pn, pc) = self._cloud_tensors(point_offsets, xyz, normals, cam_source, n_cameras, view_points, True)
        if pp is None:
            pp = preprocess_params()
        poff = np.zeros(len(ks) + 1, np.int32)
        return self._install(lambda: lib().gpdb_preprocess_clouds_device(self.h, len(ks), _p(off), px, pn, pc, _p(ks), _p(vp),
                                                                         C.byref(pp), _p(poff)),
                             poff, ks, vp, int(off[-1]))

    def _install_depth(self, fn, n_cameras, cameras, fmt, ptr, pp, fallback=None):
        # fallback: the n_fallback_out array of the organized entry points, which take it as one more argument
        ks, arr, vps = _depth_cameras(n_cameras, cameras)
        if pp is None:
            pp = preprocess_params()
        poff = np.zeros(len(ks) + 1, np.int32)
        extra = () if fallback is None else (_p(fallback),)
        return self._install(lambda: fn(self.h, len(ks), _p(ks), C.cast(arr, C.c_void_p), int(fmt), ptr, C.byref(pp), _p(poff),
                                        *extra),
                             poff, ks, vps, sum(int(c.width) * int(c.height) for c in arr[:len(cameras)]))

    def preprocess_depth(self, views, pp=None, read_back=True):
        """gpdb_preprocess_depth: preprocess_clouds() of views given as depth images. views: one list per view of
        (image, camera) pairs, image a [height, width] uint16 or float32 array (one dtype for the whole call, which selects
        GPDB_DEPTH_U16 / GPDB_DEPTH_F32), camera a depth_camera(). View b's raw cloud is its cameras' pixels concatenated
        (include/gpd_b200_depth.h), so src indexes those pixels. Installs the processed batch; returns one dict per view as
        preprocess_clouds() does, or the processed point offsets [B+1] when read_back is False."""
        ks, cams, fmt, depth = _depth_views(views, "preprocess_depth")
        poff = self._install_depth(lib().gpdb_preprocess_depth, ks, cams, fmt, _p(depth), pp)
        return self.get_clouds() if read_back else poff

    def preprocess_depth_organized(self, views, pp=None, read_back=True):
        """gpdb_preprocess_depth_organized: preprocess_depth() with the integral-image normals of each camera's image
        (include/gpd_b200_organized.h rule 7); a point without a finite one keeps its radius estimate. Returns
        (what preprocess_depth() returns, the fallback points per view [B])."""
        ks, cams, fmt, depth = _depth_views(views, "preprocess_depth_organized")
        fb = np.zeros(len(ks), np.int32)
        poff = self._install_depth(lib().gpdb_preprocess_depth_organized, ks, cams, fmt, _p(depth), pp, fb)
        return (self.get_clouds() if read_back else poff), fb

    def preprocess_depth_tensors(self, n_cameras, cameras, d_depth, pp=None):
        """gpdb_preprocess_depth_device: preprocess_depth() of depth images held in ONE CUDA tensor, every camera's image
        back to back in camera order (n_cameras [B] per view, cameras the sum(n_cameras) depth_camera()s, view by view).
        The tensor's dtype selects the format: torch.uint16 (or int16 holding the same bits) or torch.float32. Installs the
        processed batch; returns its point offsets [B+1]."""
        cams = list(cameras)
        fmt, ptr = self._depth_tensor(cams, d_depth)
        return self._install_depth(lib().gpdb_preprocess_depth_device, n_cameras, cams, fmt, ptr, pp)

    def preprocess_depth_organized_tensors(self, n_cameras, cameras, d_depth, pp=None):
        """gpdb_preprocess_depth_organized_device: preprocess_depth_organized() of depth images held in one CUDA tensor,
        as preprocess_depth_tensors() takes them. Returns (the processed point offsets [B+1], the fallback points per view
        [B])."""
        cams = list(cameras)
        fmt, ptr = self._depth_tensor(cams, d_depth)
        fb = np.zeros(len(_host_i32("n_cameras", n_cameras)), np.int32)
        return self._install_depth(lib().gpdb_preprocess_depth_organized_device, n_cameras, cams, fmt, ptr, pp, fb), fb

    def _depth_tensor(self, cams, d_depth):
        """(format, device pointer) of the depth tensor of a *_tensors call whose cameras are cams."""
        import torch
        n = sum(int(c.width) * int(c.height) for c in cams)
        if not isinstance(d_depth, torch.Tensor):
            raise ValueError(f"d_depth: need a tensor on cuda:{self.params.device}, got {type(d_depth).__name__}")
        u16 = [d for d in (getattr(torch, "uint16", None), torch.int16) if d is not None]
        if d_depth.dtype in u16:
            fmt, dt = abi.DEPTH_U16, d_depth.dtype
        elif d_depth.dtype == torch.float32:
            fmt, dt = abi.DEPTH_F32, torch.float32
        else:
            raise TypeError(f"d_depth: need torch.uint16 or torch.float32, got {d_depth.dtype}")
        ptr = _device_arg("d_depth", d_depth, dt, self.params.device, n)
        self._torch_stream()
        return fmt, ptr

    # ---- triangle meshes (include/gpd_b200_render.h): depth images and surface samples; nothing is installed ----

    def render_depth(self, meshes, cameras_per_view, dtype=np.float32, face_ids=False):
        """gpdb_render_depth: depth images of mesh scenes. meshes: one (vertices [V, 3], faces [F, 3]) per view;
        cameras_per_view: one list of depth_camera()s per view. dtype np.float32 (GPDB_DEPTH_F32) or np.uint16
        (GPDB_DEPTH_U16). Returns one list of (image [height, width], camera) per view, what preprocess_depth() takes,
        and with face_ids also one list of int32 face images per view (the view-local face each return hit, -1 where
        the pixel has none)."""
        return self._render_views("render_depth", lib().gpdb_render_depth, (), meshes, cameras_per_view, dtype, face_ids)

    def render_sensor_depth(self, meshes, cameras_per_view, sensor, seed, dtype=np.float32, face_ids=False):
        """gpdb_render_sensor_depth: render_depth() seen by the structured-light sensor `sensor` (a sensor_params()),
        view b with the key seed + b (include/gpd_b200_sensor.h): projector shadows, grazing-angle dropouts, disparity
        noise and quantisation, lateral jitter and dropout. Returns what render_depth() returns; with sensor_params()'s
        zeros it equals render_depth() bit for bit."""
        return self._render_views("render_sensor_depth", lib().gpdb_render_sensor_depth, self._sensor_args(sensor, seed),
                                  meshes, cameras_per_view, dtype, face_ids)

    @staticmethod
    def _sensor_args(sensor, seed):
        if not isinstance(sensor, abi.SensorParams):
            raise TypeError(f"sensor: need a sensor_params(), got {type(sensor).__name__}")
        return (C.c_void_p(C.addressof(sensor)), C.c_uint64(int(seed) % 2 ** 64))

    def _render_views(self, name, fn, extra, meshes, cameras_per_view, dtype, face_ids):
        fmt = {np.dtype(np.float32): abi.DEPTH_F32, np.dtype(np.uint16): abi.DEPTH_U16}.get(np.dtype(dtype))
        if fmt is None:
            raise TypeError(f"{name}: dtype must be float32 or uint16, got {np.dtype(dtype)}")
        if len(cameras_per_view) != len(meshes):
            raise ValueError(f"cameras_per_view: {len(cameras_per_view)} lists, need one per mesh ({len(meshes)})")
        m = pack_meshes(meshes)
        ks, arr, _ = _depth_cameras([len(c) for c in cameras_per_view], [c for cs in cameras_per_view for c in cs])
        cams = list(arr[:int(ks.sum())])
        n = sum(int(c.width) * int(c.height) for c in cams)
        depth = np.zeros(n, dtype)
        face = np.zeros(n, np.int32) if face_ids else None
        self._check(fn(self.h, len(ks), _p(m["vertex_offsets"]), _p(m["vertices"]), _p(m["face_offsets"]), _p(m["faces"]),
                       _p(ks), C.cast(arr, C.c_void_p), fmt, _p(depth), _p(face), *extra))
        views, faces, o, k = [], [], 0, 0
        for cs in cameras_per_view:
            views.append([])
            faces.append([])
            for _ in cs:
                c = cams[k]
                h, w = int(c.height), int(c.width)
                views[-1].append((depth[o:o + h * w].reshape(h, w), c))
                faces[-1].append(None if face is None else face[o:o + h * w].reshape(h, w))
                o, k = o + h * w, k + 1
        return (views, faces) if face_ids else views

    def render_depth_tensors(self, vertex_offsets, vertices, face_offsets, faces, n_cameras, cameras, dtype=None,
                             face_ids=False):
        """gpdb_render_depth_device: render_depth() of meshes held in CUDA tensors (vertices [V, 3] float32, faces
        [F, 3] int32, concatenated as pack_meshes() lays them out; the offsets, n_cameras [B] and the sum(n_cameras)
        cameras are host arrays). dtype torch.float32 (default) or torch.uint16. Returns ONE depth tensor holding every
        camera's image back to back, as preprocess_depth_tensors() takes it, and with face_ids also the int32 face
        tensor of the same length."""
        return self._render_tensors("render_depth_tensors", lib().gpdb_render_depth_device, (), vertex_offsets, vertices,
                                    face_offsets, faces, n_cameras, cameras, dtype, face_ids)

    def render_sensor_depth_tensors(self, vertex_offsets, vertices, face_offsets, faces, n_cameras, cameras, sensor, seed,
                                    dtype=None, face_ids=False):
        """gpdb_render_sensor_depth_device: render_sensor_depth() of meshes held in CUDA tensors, laid out as
        render_depth_tensors() takes them. Returns what render_depth_tensors() returns."""
        return self._render_tensors("render_sensor_depth_tensors", lib().gpdb_render_sensor_depth_device,
                                    self._sensor_args(sensor, seed), vertex_offsets, vertices, face_offsets, faces,
                                    n_cameras, cameras, dtype, face_ids)

    def _render_tensors(self, name, fn, extra, vertex_offsets, vertices, face_offsets, faces, n_cameras, cameras, dtype,
                        face_ids):
        import torch
        dtype = torch.float32 if dtype is None else dtype
        fmt = {torch.float32: abi.DEPTH_F32, torch.uint16: abi.DEPTH_U16}.get(dtype)
        if fmt is None:
            raise TypeError(f"{name}: dtype must be torch.float32 or torch.uint16, got {dtype}")
        voff, foff = _host_i32("vertex_offsets", vertex_offsets), _host_i32("face_offsets", face_offsets)
        if len(voff) < 2 or len(foff) != len(voff):
            raise ValueError(f"vertex_offsets / face_offsets: {len(voff)} / {len(foff)} entries, need B + 1 each (B >= 1)")
        ks, arr, _ = _depth_cameras(n_cameras, cameras)
        if len(ks) != len(voff) - 1:
            raise ValueError(f"n_cameras: {len(ks)} entries, need one per view ({len(voff) - 1})")
        dev = self.params.device
        pv = _device_arg("vertices", vertices, torch.float32, dev, 3 * int(voff[-1]))
        pf = _device_arg("faces", faces, torch.int32, dev, 3 * int(foff[-1]))
        n = sum(int(c.width) * int(c.height) for c in arr[:int(ks.sum())])
        depth = torch.empty(n, dtype=dtype, device=f"cuda:{dev}")
        face = torch.empty(n, dtype=torch.int32, device=f"cuda:{dev}") if face_ids else None
        self._torch_stream()
        self._check(fn(self.h, len(ks), _p(voff), pv, _p(foff), pf, _p(ks), C.cast(arr, C.c_void_p), fmt,
                       C.c_void_p(depth.data_ptr()), None if face is None else C.c_void_p(face.data_ptr()), *extra))
        return (depth, face) if face_ids else depth

    def sample_meshes(self, meshes, density, seed, face_ids=False):
        """gpdb_sample_meshes: ground-truth clouds sampled from the surfaces of (vertices, faces) meshes at `density`
        points per square metre, mesh b with the key seed + b. Returns (point_offsets [B+1], xyz [n, 3] float32, normals
        [n, 3] float64 unit face normals[, face [n] int32 mesh-local faces]): what set_clouds() takes as clouds."""
        m = pack_meshes(meshes)
        B = len(meshes)
        poff = np.zeros(B + 1, np.int32)
        args = (self.h, B, _p(m["vertex_offsets"]), _p(m["vertices"]), _p(m["face_offsets"]), _p(m["faces"]),
                C.c_double(float(density)), C.c_uint64(int(seed)), _p(poff))
        n = self._check(lib().gpdb_sample_meshes(*args, None, None, None))
        xyz, nrm = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float64)
        face = np.zeros(n, np.int32) if face_ids else None
        if n:
            self._check(lib().gpdb_sample_meshes(*args, _p(xyz), _p(nrm), _p(face)))
        return (poff, xyz, nrm, face) if face_ids else (poff, xyz, nrm)

    def sample_meshes_tensors(self, vertex_offsets, vertices, face_offsets, faces, density, seed, face_ids=False):
        """gpdb_sample_meshes_device: sample_meshes() of meshes held in CUDA tensors (as render_depth_tensors() takes
        them). Returns (point_offsets [B+1] host, xyz [n, 3] float32, normals [n, 3] float64[, face [n] int32]) with the
        point arrays on the device: what set_clouds_tensors() takes."""
        import torch
        voff, foff = _host_i32("vertex_offsets", vertex_offsets), _host_i32("face_offsets", face_offsets)
        if len(voff) < 2 or len(foff) != len(voff):
            raise ValueError(f"vertex_offsets / face_offsets: {len(voff)} / {len(foff)} entries, need B + 1 each (B >= 1)")
        dev = self.params.device
        pv = _device_arg("vertices", vertices, torch.float32, dev, 3 * int(voff[-1]))
        pf = _device_arg("faces", faces, torch.int32, dev, 3 * int(foff[-1]))
        self._torch_stream()
        poff = np.zeros(len(voff), np.int32)
        args = (self.h, len(voff) - 1, _p(voff), pv, _p(foff), pf, C.c_double(float(density)), C.c_uint64(int(seed)),
                _p(poff))
        n = self._check(lib().gpdb_sample_meshes_device(*args, None, None, None))
        xyz = torch.empty((n, 3), dtype=torch.float32, device=f"cuda:{dev}")
        nrm = torch.empty((n, 3), dtype=torch.float64, device=f"cuda:{dev}")
        face = torch.empty(n, dtype=torch.int32, device=f"cuda:{dev}") if face_ids else None
        if n:
            self._check(lib().gpdb_sample_meshes_device(*args, C.c_void_p(xyz.data_ptr()), C.c_void_p(nrm.data_ptr()),
                                                        None if face is None else C.c_void_p(face.data_ptr())))
        return (poff, xyz, nrm, face) if face_ids else (poff, xyz, nrm)

    def normals_organized(self, clouds, view_points=None):
        """gpdb_normals_organized: Cloud::calculateNormalsOrganized (include/gpd_b200_organized.h) of organized clouds,
        each a [H, W, 3] float32 array (NaN coordinates for a missing point), view_points [B, 3] (None: the origin).
        Nothing installed changes. Returns (normals, distance maps): one [H, W, 3] float32 and one [H, W] float32 array
        per cloud, NaN normals where the estimator gives none."""
        arrs = [np.asarray(c, dtype=np.float32) for c in clouds]
        W, H, vp = _organized_shapes(arrs, view_points)
        xyz = np.ascontiguousarray(np.concatenate([a.ravel() for a in arrs])) if arrs else np.zeros(0, np.float32)
        n = int((W.astype(np.int64) * H).sum())
        nrm, dist = np.zeros(3 * n, np.float32), np.zeros(n, np.float32)
        self._check(lib().gpdb_normals_organized(self.h, len(arrs), _p(W), _p(H), _p(xyz), _p(vp), _p(nrm), _p(dist)))
        return _organized_split(nrm, dist, W, H)

    def normals_organized_tensors(self, clouds, view_points=None, distance=True):
        """gpdb_normals_organized_device: normals_organized() of [H, W, 3] float32 CUDA tensors (several are copied back to
        back into one first). Returns lists of [H, W, 3] normal and [H, W] distance tensors (views of one output each;
        distances None when distance is False)."""
        import torch
        ts = list(clouds)
        W, H, vp = _organized_shapes(ts, view_points)
        dev = self.params.device
        for i, t in enumerate(ts):
            _device_arg(f"clouds[{i}]", t, torch.float32, dev, t.numel())
        xyz = ts[0].contiguous() if len(ts) == 1 else torch.cat([t.reshape(-1) for t in ts])
        n = int((W.astype(np.int64) * H).sum())
        nrm = torch.empty(3 * n, dtype=torch.float32, device=f"cuda:{dev}")
        dist = torch.empty(n, dtype=torch.float32, device=f"cuda:{dev}") if distance else None
        self._torch_stream()
        self._check(lib().gpdb_normals_organized_device(self.h, len(ts), _p(W), _p(H), _device_arg("clouds", xyz, torch.float32, dev, 3 * n),
                                                        _p(vp), _device_arg("normals", nrm, torch.float32, dev, 3 * n),
                                                        _device_arg("distance", dist, torch.float32, dev, n, optional=True)))
        return _organized_split(nrm, dist, W, H)

    def _subsample_room(self, num_samples):
        npts = np.diff(self._batch[0]).astype(np.int64) if self._batch is not None else np.zeros(0, np.int64)
        return int(npts.sum()) if num_samples == 0 else int(np.minimum(npts, max(int(num_samples), 0)).sum())

    def _subsample(self, fn, num_samples, seed, name, mask, need, per):
        # the host twins: a mask of `need` bytes (None: nothing to size it by, and the library reports the state error)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8).ravel()
        if m is not None and need is not None and len(m) != need:
            raise ValueError(f"{name}: {len(m)} bytes, need one per {per} ({need})")
        idx = np.zeros(max(self._subsample_room(num_samples), 1), np.int32)
        soff = np.zeros(self._n_clouds + 1, np.int32)
        self._check(fn(self.h, int(num_samples), C.c_uint64(int(seed)), _p(m), _p(idx), _p(soff)))
        return [idx[soff[b]:soff[b + 1]].copy() for b in range(self._n_clouds)]

    def _subsample_tensors(self, fn, num_samples, seed, name, d_mask, need):
        import torch
        dev = self.params.device
        pm = None if d_mask is None else _device_arg(name, d_mask, torch.uint8, dev, need)
        self._torch_stream()
        room = self._subsample_room(num_samples)
        out = torch.empty(room, dtype=torch.int32, device=f"cuda:{dev}")
        soff = np.zeros(self._n_clouds + 1, np.int32)
        n = self._check(fn(self.h, int(num_samples), C.c_uint64(int(seed)), pm, C.c_void_p(out.data_ptr()) if room else None,
                           _p(soff)))
        return soff, out[:n]

    def subsample_clouds(self, num_samples, seed, mask=None):
        """gpdb_subsample_clouds: Cloud::subsample of every installed cloud (include/gpd_b200_depth.h 5): num_samples
        cloud-local point indices per cloud without replacement, ascending (0: every eligible point), drawn with key
        seed + b. mask: one uint8 per raw point (pixel) of the preprocessing call that installed the batch, concatenated
        by view, or None; only points whose source raw point has a nonzero byte are eligible. Returns one int32 array per
        cloud, as detect_batch takes them."""
        return self._subsample(lib().gpdb_subsample_clouds, num_samples, seed, "mask", mask, self._n_raw, "raw point")

    def subsample_clouds_tensors(self, num_samples, seed, d_mask=None):
        """gpdb_subsample_clouds_device: subsample_clouds() with the mask (uint8 CUDA tensor, one byte per raw point, or
        None) on the device. Returns (offsets, indices): the host offsets [B+1] and an int32 CUDA tensor of the cloud-local
        indices (cloud b's at offsets[b] .. offsets[b+1]-1), the CSR pair detect_batch_select_tensors / sis_batch_tensors
        take."""
        import torch
        n_raw = self._n_raw if self._n_raw is not None else (d_mask.numel() if isinstance(d_mask, torch.Tensor) else 0)
        return self._subsample_tensors(lib().gpdb_subsample_clouds_device, num_samples, seed, "d_mask", d_mask, int(n_raw))

    def subsample_clouds_points(self, num_samples, seed, point_mask=None):
        """gpdb_subsample_clouds_points: subsample_clouds() with the mask over the installed points (one uint8 per point
        of the batch, concatenated by cloud, e.g. segment_planes()' eligible bytes), so it also works after set_clouds().
        Returns one int32 array per cloud."""
        need = self._n_points() if self._batch is not None else None
        return self._subsample(lib().gpdb_subsample_clouds_points, num_samples, seed, "point_mask", point_mask, need,
                               "installed point")

    def subsample_clouds_points_tensors(self, num_samples, seed, d_point_mask=None):
        """gpdb_subsample_clouds_points_device: subsample_clouds_points() with the mask (uint8 CUDA tensor, one byte per
        installed point, or None) on the device. Returns (offsets, indices) as subsample_clouds_tensors()."""
        return self._subsample_tensors(lib().gpdb_subsample_clouds_points_device, num_samples, seed, "d_point_mask",
                                       d_point_mask, self._n_points())

    def segment_plane(self, pl=None):
        """gpdb_segment_plane: the support plane of the single installed cloud (include/gpd_b200_plane.h). Returns
        (plane [4] float32, NaN when the fit failed; n_inliers; eligible [N] uint8, 1 for the points off the plane)."""
        pl = plane_params() if pl is None else pl
        n = self._check(lib().gpdb_get_cloud(self.h, None, None, None))
        plane = np.zeros(4, np.float32)
        cnt = np.zeros(1, np.int32)
        elig = np.zeros(max(n, 1), np.uint8)
        self._check(lib().gpdb_segment_plane(self.h, C.byref(pl), _p(plane), _p(cnt), _p(elig)))
        return plane, int(cnt[0]), elig[:n]

    def _segment_planes(self, fn, pl, eligible, p_eligible):
        pl = plane_params() if pl is None else pl
        n = max(self._n_clouds, 1)
        planes, cnt, nh = np.zeros((n, 4), np.float32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        B = self._check(fn(self.h, C.byref(pl), _p(planes), _p(cnt), _p(nh), p_eligible))
        return {"planes": planes[:B], "n_inliers": cnt[:B], "n_hypotheses": nh[:B], "eligible": eligible}

    def segment_planes(self, pl=None):
        """gpdb_segment_planes: the support plane of every installed cloud (cloud b with key seed + b). Returns a dict:
        planes [B, 4] float32, n_inliers [B], n_hypotheses [B] (RANSAC hypotheses evaluated) and eligible [N] uint8
        (concatenated by cloud, the point_mask subsample_clouds_points() takes)."""
        n_pts = self._n_points()
        elig = np.zeros(max(n_pts, 1), np.uint8)
        return self._segment_planes(lib().gpdb_segment_planes, pl, elig[:n_pts], _p(elig))

    def segment_planes_tensors(self, pl=None):
        """gpdb_segment_planes_device: segment_planes() with the eligible bytes in a uint8 CUDA tensor [N], on torch's
        current stream; planes and counts are host arrays as in segment_planes()."""
        import torch
        n_pts = self._n_points()
        self._torch_stream()
        elig = torch.empty(n_pts, dtype=torch.uint8, device=f"cuda:{self.params.device}")
        return self._segment_planes(lib().gpdb_segment_planes_device, pl, elig, C.c_void_p(elig.data_ptr()) if n_pts else None)

    def refine_normals(self, k):
        """gpdb_refine_normals: refines the normals of the single installed cloud in place with k nearest neighbours
        (Cloud::refineNormals, include/gpd_b200_refine.h). Returns the iterations run; get_cloud() reads the normals."""
        it = np.zeros(1, np.int32)
        self._check(lib().gpdb_refine_normals(self.h, int(k), _p(it)))
        return int(it[0])

    def refine_normals_clouds(self, k):
        """gpdb_refine_normals_clouds: refine_normals() for every installed cloud, each on its own. Returns the
        iterations run per cloud, int32 [B]."""
        it = np.zeros(max(self._n_clouds, 1), np.int32)
        B = self._check(lib().gpdb_refine_normals_clouds(self.h, int(k), _p(it)))
        return it[:B]

    def remove_outliers(self, mean_k=50, stddev_mul=1.0):
        """gpdb_remove_outliers: removes the statistical outliers of the single installed cloud and reinstalls the kept
        points (Cloud::removeStatisticalOutliers, include/gpd_b200_outliers.h). Returns n_kept, the cloud's mean, stddev
        and threshold, and kept, one byte per point before the call; get_cloud() reads the kept cloud."""
        n = self._check(lib().gpdb_get_cloud(self.h, None, None, None))
        stats = np.zeros(3, np.float64)
        kept = np.zeros(n, np.uint8)
        n_kept = self._check(lib().gpdb_remove_outliers(self.h, int(mean_k), float(stddev_mul), _p(stats), _p(kept)))
        return {"n_kept": n_kept, "mean": float(stats[0]), "stddev": float(stats[1]), "threshold": float(stats[2]),
                "kept": kept}

    def remove_outliers_clouds(self, mean_k=50, stddev_mul=1.0):
        """gpdb_remove_outliers_clouds: remove_outliers() for every installed cloud, each on its own. Returns offsets, the
        new point offsets [B+1], stats [B, 3] (mean, stddev, threshold) and kept, one byte per point before the call.
        Sample positions and the SIS record are dropped."""
        B = self._n_clouds
        off = np.zeros(B + 1, np.int32)
        stats = np.zeros((max(B, 1), 3), np.float64)
        kept = np.zeros(self._n_points(), np.uint8)
        try:
            self._check(lib().gpdb_remove_outliers_clouds(self.h, int(mean_k), float(stddev_mul), _p(off), _p(stats),
                                                          _p(kept)))
        except GpdbError as e:
            # GPDB_ERR_INVALID / GPDB_ERR_STATE come before any device work and change nothing; after any other error the
            # library holds no batch, and neither may this bookkeeping, which sizes the output buffers of later calls
            if e.code not in (-1, -3):
                self._drop_batch()
            raise
        self._batch = (off,) + self._batch[1:]
        self._sis_shape = None
        return {"offsets": off, "stats": stats[:B], "kept": kept}

    def set_clouds_tensors(self, point_offsets, xyz, normals, n_cameras, view_points, cam_source=None):
        """gpdb_set_clouds_device: set_clouds() from CUDA tensors, laid out as preprocess_clouds_tensors takes them
        (normals required)."""
        off, ks, vp, (px, pn, pc) = self._cloud_tensors(point_offsets, xyz, normals, cam_source, n_cameras, view_points, False)
        self._install(lambda: lib().gpdb_set_clouds_device(self.h, len(ks), _p(off), px, pn, pc, _p(ks), _p(vp)), off, ks, vp)

    def detect_batch_select_tensors(self, sample_offsets, d_sample_idx, k):
        """gpdb_detect_batch_select_device: the k best candidates of every installed cloud, for cloud-local sample indices
        in an int32 CUDA tensor (CSR: cloud b's at sample_offsets[b] .. sample_offsets[b+1]-1, sample_offsets a host array
        of B+1 entries). Returns (records, offsets): a uint8 CUDA tensor [n, POSE_BYTES] of gpdb_pose records (cloud b's
        rows offsets[b] .. offsets[b+1]-1, as detect_batch_select returns them; poses_from_tensor reads them) and the host
        offsets [B+1]."""
        import torch
        off = _host_i32("sample_offsets", sample_offsets, self._n_clouds + 1)
        ps = _device_arg("d_sample_idx", d_sample_idx, torch.int32, self.params.device, int(off[-1]))
        self._torch_stream()
        out = torch.empty((self._n_clouds * max(int(k), 0), POSE_BYTES), dtype=torch.uint8, device=f"cuda:{self.params.device}")
        soff = np.zeros(len(off), np.int32)
        stats = abi.Result()
        n = self._check(lib().gpdb_detect_batch_select_device(self.h, _p(off), ps, int(k),
                                                               C.c_void_p(out.data_ptr()) if out.numel() else None, _p(soff),
                                                               C.byref(stats)))
        return out[:n], soff

    def sis_batch_tensors(self, init_offsets, d_init_idx, **sis):
        """gpdb_sis_batch_device: sis_batch() from cloud-local initial indices in an int32 CUDA tensor (CSR: cloud b's at
        init_offsets[b] .. init_offsets[b+1]-1, init_offsets a host array of B+1 entries). Returns (records, offsets, stats):
        a uint8 CUDA tensor [n, POSE_BYTES] of gpdb_pose records (cloud b's rows offsets[b] .. offsets[b+1]-1, as sis_batch
        returns them; poses_from_tensor reads them), the host offsets [B+1] and a dict of n_samples, n_total_candidates
        and kernel_launches."""
        import torch
        off = _host_i32("init_offsets", init_offsets, self._n_clouds + 1)
        pi = _device_arg("d_init_idx", d_init_idx, torch.int32, self.params.device, int(off[-1]))
        sp = sis_params(**sis)
        self._torch_stream()
        P = self.params.num_hand_axes * self.params.num_orientations
        cap = (int(off[-1]) + self._n_clouds * max(sp.num_iterations, 0) * max(sp.num_samples_per_iteration, 0)) * P
        out = torch.empty((cap, POSE_BYTES), dtype=torch.uint8, device=f"cuda:{self.params.device}")
        hoff = np.zeros(len(off), np.int32)
        stats = abi.Result()
        self._sis_shape = None
        n = self._check(lib().gpdb_sis_batch_device(self.h, C.byref(sp), _p(off), pi,
                                                     C.c_void_p(out.data_ptr()) if cap else None, _p(hoff), C.byref(stats)))
        self._sis_shape = (len(hoff) - 1, sp.num_iterations)
        return out[:n], hoff, {"n_samples": stats.n_samples, "n_total_candidates": stats.n_total_candidates,
                               "kernel_launches": stats.kernel_launches}

    def find_clusters_batch_tensors(self, hand_offsets, hands, min_inliers):
        """gpdb_find_clusters_batch_device: find_clusters_batch() on groups of gpdb_pose records held in a uint8 CUDA tensor
        [n, POSE_BYTES] (group g: rows hand_offsets[g] .. hand_offsets[g+1]-1, hand_offsets a host array). Returns
        (clusters, offsets): a uint8 CUDA tensor [nc, POSE_BYTES] and the host offsets [G+1]."""
        import torch
        hoff = _host_i32("hand_offsets", hand_offsets)
        n = int(hoff[-1]) if len(hoff) else 0
        ph = _device_arg("hands", hands, torch.uint8, self.params.device, n * POSE_BYTES)
        self._torch_stream()
        out = torch.empty((n, POSE_BYTES), dtype=torch.uint8, device=f"cuda:{self.params.device}")
        coff = np.zeros(max(len(hoff), 1), np.int32)
        nc = self._check(lib().gpdb_find_clusters_batch_device(self.h, len(hoff) - 1, _p(hoff), ph, int(min_inliers),
                                                               C.c_void_p(out.data_ptr()) if n else None, _p(coff)))
        return out[:nc], coff

    def set_clouds_samples_tensors(self, pos_offsets, xyz):
        """gpdb_set_clouds_samples_device: set_clouds_samples() from a float64 CUDA tensor xyz [M, 3] (cloud b's positions
        at rows pos_offsets[b] .. pos_offsets[b+1]-1, pos_offsets a host array of B+1 entries), e.g. drawn by a model on the
        GPU. Returns each cloud's first position index N_b (int32 [B]): cloud-local index N_b + j addresses its position j."""
        import torch
        off = _host_i32("pos_offsets", pos_offsets, self._n_clouds + 1)
        px = _device_arg("xyz", xyz, torch.float64, self.params.device, 3 * int(off[-1]))
        self._torch_stream()
        self._check(lib().gpdb_set_clouds_samples_device(self.h, _p(off), px))
        return np.diff(self._batch[0]).astype(np.int32)

    def _all_records(self, fn, sample_offsets, d_sample_idx, scores):
        import torch
        off = _host_i32("sample_offsets", sample_offsets, self._n_clouds + 1)
        dev = self.params.device
        n, P = int(off[-1]), self.params.num_hand_axes * self.params.num_orientations
        ps = _device_arg("d_sample_idx", d_sample_idx, torch.int32, dev, n)
        self._torch_stream()
        rec = torch.empty((n * P, POSE_BYTES), dtype=torch.uint8, device=f"cuda:{dev}")
        flags = torch.empty((n, P), dtype=torch.uint8, device=f"cuda:{dev}")
        dense = [flags] + ([torch.empty((n, P), dtype=torch.float32, device=f"cuda:{dev}")] if scores else [])
        coff = np.zeros(len(off), np.int32)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t.numel() else None  # noqa: E731
        stats = abi.Result()
        nc = self._check(fn(self.h, _p(off), ps, *[ptr(t) for t in dense], ptr(rec), _p(coff), C.byref(stats)))
        return (rec[:nc], *dense, coff)

    def hand_search_batch_tensors(self, sample_offsets, d_sample_idx):
        """gpdb_hand_search_batch_device: hand_search_batch() for cloud-local sample indices in an int32 CUDA tensor (CSR,
        sample_offsets a host array of B+1 entries). Returns (records, flags, offsets): every VALID|FILTERED record as a uint8
        CUDA tensor [nc, POSE_BYTES] (cloud b's rows offsets[b] .. offsets[b+1]-1, cloud-local sample slots, as
        hand_search_batch returns them; poses_from_tensor reads them), the pose flags [n, P] uint8 on the device and the host
        offsets [B+1]."""
        return self._all_records(lib().gpdb_hand_search_batch_device, sample_offsets, d_sample_idx, False)

    def detect_batch_tensors(self, sample_offsets, d_sample_idx):
        """gpdb_detect_batch_device: detect_batch() on the device, as hand_search_batch_tensors. Returns (records, flags,
        scores, offsets): the scored records, the pose flags [n, P] uint8 and scores [n, P] float32 (NaN where no image was
        classified) on the device, and the host offsets [B+1]. No images: images_batch_tensors makes them."""
        return self._all_records(lib().gpdb_detect_batch_device, sample_offsets, d_sample_idx, True)

    def images_batch_tensors(self, hand_offsets, hands):
        """gpdb_images_batch_device: the grasp images of gpdb_pose records in a uint8 CUDA tensor [n, POSE_BYTES] (cloud b's
        at rows hand_offsets[b] .. hand_offsets[b+1]-1, hand_offsets a host array of B+1 entries), as a uint8 CUDA tensor
        [n, S, S, C] in the cv::Mat layout, byte-equal to detect_batch's images of the same records."""
        import torch
        hoff = _host_i32("hand_offsets", hand_offsets, self._n_clouds + 1)
        dev = self.params.device
        n = int(hoff[-1])
        ph = _device_arg("hands", hands, torch.uint8, dev, n * POSE_BYTES)
        self._torch_stream()
        S, Cc = self.params.image_size, self.params.image_num_channels
        out = torch.empty((n, S, S, Cc), dtype=torch.uint8, device=f"cuda:{dev}")
        self._check(lib().gpdb_images_batch_device(self.h, _p(hoff), ph, C.c_void_p(out.data_ptr()) if n else None))
        return out

    def reevaluate_batch_tensors(self, hand_offsets, hands):
        """gpdb_reevaluate_batch_device: reevaluate_batch() of gpdb_pose records in a uint8 CUDA tensor [n, POSE_BYTES]
        (group b, labelled against cloud b: rows hand_offsets[b] .. hand_offsets[b+1]-1, hand_offsets a host array of B+1
        entries), e.g. detect_batch_tensors' records of another context. The records' half / full flags are updated in
        place; returns the labels as an int32 CUDA tensor [n]."""
        import torch
        hoff = _host_i32("hand_offsets", hand_offsets, self._n_clouds + 1 if self._batch is not None else None)
        dev = self.params.device
        n = int(hoff[-1]) if len(hoff) else 0
        ph = _device_arg("hands", hands, torch.uint8, dev, n * POSE_BYTES)
        self._torch_stream()
        labels = torch.empty(n, dtype=torch.int32, device=f"cuda:{dev}")
        self._check(lib().gpdb_reevaluate_batch_device(self.h, _p(hoff), ph, C.c_void_p(labels.data_ptr()) if n else None))
        return labels

    def classify_tensors(self, images):
        """gpdb_classify_device: classify() of uint8 CUDA images [n, S, S, C] (cv::Mat layout). Returns (scores [n], logits
        [n, 2]), float32 CUDA tensors, bit-equal to classify() of the same images."""
        import torch
        dev = self.params.device
        S, Cc = self.params.image_size, self.params.image_num_channels
        n = images.shape[0] if isinstance(images, torch.Tensor) and images.dim() > 0 else 0
        pi = _device_arg("images", images, torch.uint8, dev, n * S * S * Cc)
        self._torch_stream()
        scores = torch.empty(n, dtype=torch.float32, device=f"cuda:{dev}")
        logits = torch.empty((n, 2), dtype=torch.float32, device=f"cuda:{dev}")
        self._check(lib().gpdb_classify_device(self.h, pi, n, C.c_void_p(scores.data_ptr()) if n else None,
                                               C.c_void_p(logits.data_ptr()) if n else None))
        return scores, logits

    def detect_batch_raw(self, offsets_i32, sidx_i32, res, cand_offsets_i32):
        """Timed path for tools/bench_batch.py: no numpy conversion; caller frees `res`."""
        if len(offsets_i32) != self._n_clouds + 1 or len(cand_offsets_i32) != self._n_clouds + 1:
            raise ValueError(f"offsets need {self._n_clouds + 1} entries for a batch of {self._n_clouds} clouds")
        return self._check(lib().gpdb_detect_batch(self.h, _p(offsets_i32), _p(sidx_i32), C.byref(res), _p(cand_offsets_i32)))

    def set_samples(self, samples):
        """Cloud::setSamples: arbitrary float64 positions [n, 3]; returns the sample indices that address them."""
        sm = np.ascontiguousarray(samples, dtype=np.float64)
        first = self._check(lib().gpdb_set_samples(self.h, _p(sm), len(sm)))
        return np.arange(first, first + len(sm), dtype=np.int32)

    def get_cloud(self):
        n = self._check(lib().gpdb_get_cloud(self.h, None, None, None))
        xyz = np.zeros((n, 3), np.float32)
        nrm = np.zeros((n, 3), np.float64)
        self._check(lib().gpdb_get_cloud(self.h, _p(xyz), _p(nrm), None))
        return {"xyz": xyz, "normals": nrm, "cam_source": self._cam_source(n)}

    def _cam_source(self, n, kmax=8):
        # the camera count is not exported separately: read k x N into a buffer sized for GPDB_MAX_CAMERAS
        buf = np.full(n * kmax, -1, np.int32)
        self._check(lib().gpdb_get_cloud(self.h, None, None, _p(buf)))
        k = int(np.count_nonzero(buf >= 0)) // max(n, 1)
        return buf[: n * k].reshape(n, k).copy()

    def preprocess_timings(self):
        ms = np.zeros(6)
        lib().gpdb_preprocess_timings(self.h, _p(ms))
        return ms

    def _result(self, fn, sample_idx, *args):
        sidx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        res = abi.Result()
        self._check(fn(self.h, _p(sidx), len(sidx), *args, C.byref(res)))
        S, Cc = self.params.image_size, self.params.image_num_channels
        out = abi.result_to_numpy(res, S * S * Cc)
        lib().gpdb_free_result(C.byref(res))
        return out

    def detect(self, sample_idx):
        return self._result(lib().gpdb_detect, sample_idx)

    def detect_select(self, sample_idx, num_selected):
        """detectGrasps + selectGrasps: the num_selected best candidates, sorted on the device (gpdb_detect_select)."""
        return self._result(lib().gpdb_detect_select, sample_idx, int(num_selected))

    def detect_select_raw(self, sidx_i32, num_selected, res):
        """Timed path for bench.py; caller frees `res`."""
        return self._check(lib().gpdb_detect_select(self.h, _p(sidx_i32), len(sidx_i32), int(num_selected), C.byref(res)))

    def detect_raw(self, sidx_i32, res):
        """Timed path for bench.py: no numpy conversion; caller frees `res`."""
        return self._check(lib().gpdb_detect(self.h, _p(sidx_i32), len(sidx_i32), C.byref(res)))

    def detect_resident(self, d_sidx_ptr, n, d_flags_ptr, d_scores_ptr, stats):
        """Device-resident path (raw device pointers as ints); returns n_candidates."""
        return self._check(lib().gpdb_detect_resident(self.h, C.c_void_p(d_sidx_ptr), n, C.c_void_p(d_flags_ptr),
                                                      C.c_void_p(d_scores_ptr), C.byref(stats)))

    def set_overlap(self, enable):
        """Hand search of the chunks ahead on its own stream (default on); off = one stream, exclusive stage timers."""
        self._check(lib().gpdb_set_overlap(self.h, int(bool(enable))))

    def set_stream(self, cuda_stream_ptr):
        self._check(lib().gpdb_set_stream(self.h, C.c_void_p(cuda_stream_ptr)))

    def hand_search(self, sample_idx):
        return self._result(lib().gpdb_hand_search, sample_idx)

    def frames(self, sample_idx):
        sidx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        n = len(sidx)
        frames = np.zeros((n, 9))
        valid = np.zeros(n, np.uint8)
        self._check(lib().gpdb_frames(self.h, _p(sidx), n, _p(frames), _p(valid)))
        return frames, valid

    def images(self, poses):
        poses = np.ascontiguousarray(poses, dtype=abi.POSE_DTYPE)
        n = len(poses)
        S, Cc = self.params.image_size, self.params.image_num_channels
        out = np.zeros((n, S, S, Cc), np.uint8)
        self._check(lib().gpdb_images(self.h, _p(poses), n, _p(out)))
        return out

    def classify(self, images):
        images = np.ascontiguousarray(images, dtype=np.uint8)
        n = images.shape[0]
        scores = np.zeros(n, np.float32)
        logits = np.zeros((n, 2), np.float32)
        self._check(lib().gpdb_classify(self.h, _p(images), n, _p(scores), _p(logits)))
        return scores, logits

    def train_begin(self, params, init=None):
        """gpdb_train_begin: start (or restart) training from the eight arrays `init`, or from the loaded weights when
        None. The optimiser state and step count start at zero."""
        C_ = self.params.image_num_channels
        if init is None:
            self._check(lib().gpdb_train_begin(self.h, C.c_void_p(C.addressof(params)), None))
        else:
            arrs, ptrs = _weight_ptrs(init, C_)
            self._check(lib().gpdb_train_begin(self.h, C.c_void_p(C.addressof(params)), ptrs))

    def train_step(self, images, labels):
        """gpdb_train_step: one optimiser step on uint8 images [n, S, S, C] (cv::Mat layout) and labels in {0, 1};
        returns the step's mean loss."""
        images = np.ascontiguousarray(images, dtype=np.uint8)
        labels = _host_i32("labels", labels, images.shape[0] if images.ndim else 0)
        loss = C.c_float()
        self._check(lib().gpdb_train_step(self.h, _p(images), _p(labels), len(labels), C.byref(loss)))
        return loss.value

    def train_step_tensors(self, images, labels):
        """gpdb_train_step_device: train_step() on a uint8 CUDA tensor [n, S, S, C] and int32 CUDA labels [n]; returns
        the loss as a 0-d float32 CUDA tensor, written on the device (no synchronisation)."""
        import torch
        dev = self.params.device
        S, Cc = self.params.image_size, self.params.image_num_channels
        n = images.shape[0] if isinstance(images, torch.Tensor) and images.dim() > 0 else 0
        pi = _device_arg("images", images, torch.uint8, dev, n * S * S * Cc)
        pl = _device_arg("labels", labels, torch.int32, dev, n)
        self._torch_stream()
        loss = torch.empty((), dtype=torch.float32, device=f"cuda:{dev}")
        self._check(lib().gpdb_train_step_device(self.h, pi, pl, n, C.c_void_p(loss.data_ptr())))
        return loss

    def train_weights(self):
        """gpdb_train_weights: the trained weights as eight float32 arrays in the .bin layout (set_weights takes them)."""
        arrs = [np.zeros(s, np.float32) for s in weight_sizes(self.params.image_num_channels)]
        self._check(lib().gpdb_train_weights(self.h, (C.c_void_p * 8)(*[a.ctypes.data for a in arrs])))
        return arrs

    def debug_train_step(self, images, labels):
        """gpdb_debug_train_step: one step's forward state, backward intermediates and gradients (nothing updated), as a
        dict of numpy arrays named as the fields of gpdb_train_debug; "grad" holds the eight gradients."""
        images = np.ascontiguousarray(images, dtype=np.uint8)
        n = images.shape[0]
        labels = _host_i32("labels", labels, n)
        shapes = {"pool1": ((n, 20, 28, 28), np.float32), "pool2": ((n, 7200), np.float32), "ip1": ((n, 500), np.float32),
                  "logits": ((n, 2), np.float32), "choice1": ((n, 20, 28, 28), np.uint8), "choice2": ((n, 7200), np.uint8),
                  "loss": ((n,), np.float32), "dlogits": ((n, 2), np.float32), "dip1": ((n, 500), np.float32),
                  "dpool2": ((n, 7200), np.float32), "dpool1": ((n, 20, 28, 28), np.float32)}
        out = {k: np.zeros(s, t) for k, (s, t) in shapes.items()}
        out["grad"] = [np.zeros(s, np.float32) for s in weight_sizes(self.params.image_num_channels)]
        dbg = abi.TrainDebug(*[out[k].ctypes.data for k in shapes], (C.c_void_p * 8)(*[a.ctypes.data for a in out["grad"]]))
        self._check(lib().gpdb_debug_train_step(self.h, _p(images), _p(labels), n, C.c_void_p(C.addressof(dbg))))
        return out

    def lenet_layers(self, images):
        """gpdb_debug_lenet_layers: classify() that also returns every layer the selected implementation computed, as a
        dict: pool1 [n, 20, 28, 28] float32, pool2 [n, 7200] float64 (k = c + 50 j, the values ip1 multiplies), ip1
        [n, 500] float32, logits [n, 2] float32."""
        images = np.ascontiguousarray(images, dtype=np.uint8)
        n = images.shape[0]
        out = {"pool1": np.zeros((n, 20, 28, 28), np.float32), "pool2": np.zeros((n, 7200), np.float64),
               "ip1": np.zeros((n, 500), np.float32), "logits": np.zeros((n, 2), np.float32)}
        self._check(lib().gpdb_debug_lenet_layers(self.h, _p(images), n, _p(out["pool1"]), _p(out["pool2"]), _p(out["ip1"]),
                                                  _p(out["logits"])))
        return out

    def phase_cycles(self, enable=1):
        out = np.zeros(32, np.uint64)
        self._check(lib().gpdb_debug_phase_cycles(self.h, enable, _p(out)))
        return out

    def path_counts(self):
        """gpdb_debug_path_counts as a dict (PATH_EVENTS): how often each tier or in-place fallback of the geometry kernels
        ran since phase_cycles(1) enabled the counters (all zero while they are off)."""
        out = np.zeros(16, np.uint64)
        self._check(lib().gpdb_debug_path_counts(self.h, _p(out)))
        return {name: int(out[i]) for i, name in enumerate(PATH_EVENTS)}

    def last_timings(self):
        ms = np.zeros(8)
        lib().gpdb_last_timings(self.h, _p(ms))
        return ms


def comm_unique_id():
    """ncclGetUniqueId (128 bytes): call on one rank and distribute to the others."""
    buf = C.create_string_buffer(128)
    rc = lib().gpdb_comm_unique_id(buf)
    if rc != 0:
        raise GpdbError(rc, lib().gpdb_last_error(None).decode())
    return buf.raw


def shard_bounds(n, rank, nranks):
    """(lo, hi, slot_samples) of gpdb_shard_bounds: the slice of `rank` and the fixed slot size of the all-gather."""
    lo, hi, st = C.c_int32(), C.c_int32(), C.c_int32()
    lib().gpdb_shard_bounds(int(n), int(rank), int(nranks), C.byref(lo), C.byref(hi), C.byref(st))
    return lo.value, hi.value, st.value


def slot_bytes(slot_samples, P):
    return int(lib().gpdb_slot_bytes(int(slot_samples), int(P)))


def free_result(res):
    lib().gpdb_free_result(C.byref(res))
