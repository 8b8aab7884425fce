"""ctypes mirror of include/gpd_b200.h (the C-ABI types of the grasp-candidate hot path).

Only type definitions live here; they are shared by the product loader (gpd_b200/lib.py) and by
the test-only oracle loader (oracle/oracle.py) because both speak the same boundary structs.
"""
import ctypes as C

import numpy as np

MAX_HAND_AXES = 3
POSE_VALID, POSE_FILTERED, POSE_HALF, POSE_FULL = 1, 2, 4, 8


class Params(C.Structure):
    """gpdb_params — field names are the reference's cfg keys (grasp_detector.cpp:48-185)."""

    _fields_ = [
        ("finger_width", C.c_double),
        ("hand_outer_diameter", C.c_double),
        ("hand_depth", C.c_double),
        ("hand_height", C.c_double),
        ("init_bite", C.c_double),
        ("volume_width", C.c_double),
        ("volume_depth", C.c_double),
        ("volume_height", C.c_double),
        ("image_size", C.c_int32),
        ("image_num_channels", C.c_int32),
        ("nn_radius", C.c_double),
        ("num_orientations", C.c_int32),
        ("num_finger_placements", C.c_int32),
        ("num_hand_axes", C.c_int32),
        ("hand_axes", C.c_int32 * MAX_HAND_AXES),
        ("deepen_hand", C.c_int32),
        ("friction_coeff", C.c_double),
        ("min_viable", C.c_int32),
        ("min_aperture", C.c_double),
        ("max_aperture", C.c_double),
        ("workspace_grasps", C.c_double * 6),
        ("filter_approach_direction", C.c_int32),
        ("direction", C.c_double * 3),
        ("thresh_rad", C.c_double),
        ("batch_size", C.c_int32),
        ("relu_after_conv", C.c_int32),
        ("shadow_mode", C.c_int32),
        ("device", C.c_int32),
        ("chunk_samples", C.c_int32),
        ("keep_images", C.c_int32),
        ("lenet_impl", C.c_int32),
    ]


class Pose(C.Structure):
    """gpdb_pose = candidate::Hand (include/gpd/candidate/hand.h:267-276)."""

    _fields_ = [
        ("sample", C.c_double * 3),
        ("frame", C.c_double * 9),
        ("position", C.c_double * 3),
        ("top", C.c_double),
        ("bottom", C.c_double),
        ("center", C.c_double),
        ("width", C.c_double),
        ("score", C.c_float),
        ("sample_index", C.c_int32),
        ("sample_slot", C.c_int32),
        ("pose_slot", C.c_int16),
        ("finger_idx", C.c_int16),
        ("half_antipodal", C.c_uint8),
        ("full_antipodal", C.c_uint8),
        ("pad_", C.c_uint8 * 6),
    ]


POSE_DTYPE = np.dtype(
    [
        ("sample", "<f8", (3,)),
        ("frame", "<f8", (9,)),
        ("position", "<f8", (3,)),
        ("top", "<f8"),
        ("bottom", "<f8"),
        ("center", "<f8"),
        ("width", "<f8"),
        ("score", "<f4"),
        ("sample_index", "<i4"),
        ("sample_slot", "<i4"),
        ("pose_slot", "<i2"),
        ("finger_idx", "<i2"),
        ("half_antipodal", "u1"),
        ("full_antipodal", "u1"),
        ("pad_", "u1", (6,)),
    ],
    align=True,
)
assert POSE_DTYPE.itemsize == C.sizeof(Pose), (POSE_DTYPE.itemsize, C.sizeof(Pose))


class Result(C.Structure):
    """gpdb_result — callee-allocated SoA result."""

    _fields_ = [
        ("n_samples", C.c_int32),
        ("poses_per_sample", C.c_int32),
        ("frame_valid", C.POINTER(C.c_uint8)),
        ("frames", C.POINTER(C.c_double)),
        ("pose_flags", C.POINTER(C.c_uint8)),
        ("pose_scores", C.POINTER(C.c_float)),
        ("n_candidates", C.c_int32),
        ("candidates", C.POINTER(Pose)),
        ("images", C.POINTER(C.c_uint8)),
        ("ms_candidates", C.c_double),
        ("ms_images", C.c_double),
        ("ms_classify", C.c_double),
        ("kernel_launches", C.c_int64),
        ("n_total_candidates", C.c_int32),
        ("owner_", C.c_void_p),
    ]


class PreprocessParams(C.Structure):
    """gpdb_preprocess_params — cfg keys of CandidatesGenerator::preprocessPointCloud
    (candidates_generator.cpp:14-37, grasp_detector.cpp:50-66)."""

    _fields_ = [
        ("workspace", C.c_double * 6),
        ("voxel_size", C.c_double),
        ("normals_radius", C.c_double),
        ("voxelize", C.c_int32),
        ("estimate_normals", C.c_int32),
    ]


class SisParams(C.Structure):
    """gpdb_sis_params — cfg keys of SequentialImportanceSampling (sequential_importance_sampling.cpp:19-31)."""

    _fields_ = [
        ("num_iterations", C.c_int32),
        ("num_samples_per_iteration", C.c_int32),
        ("prob_rand_samples", C.c_double),
        ("standard_deviation", C.c_double),
        ("sampling_method", C.c_int32),
        ("workspace", C.c_double * 6),
        ("min_score", C.c_double),
        ("min_inliers", C.c_int32),
        ("seed", C.c_uint64),
    ]


DEPTH_U16, DEPTH_F32 = 0, 1  # GPDB_DEPTH_U16 / GPDB_DEPTH_F32


class DepthCamera(C.Structure):
    """gpdb_depth_camera (include/gpd_b200_depth.h): one pinhole depth camera of a view."""

    _fields_ = [
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("fx", C.c_double),
        ("fy", C.c_double),
        ("cx", C.c_double),
        ("cy", C.c_double),
        ("pose", C.c_double * 12),  # camera-to-world [R | t], row-major 3 x 4
        ("depth_scale", C.c_double),
        ("min_depth", C.c_double),
        ("max_depth", C.c_double),
    ]


class SensorParams(C.Structure):
    """gpdb_sensor_params (include/gpd_b200.h, rules in include/gpd_b200_sensor.h): every field 0 is a clean render."""

    _fields_ = [(f, C.c_double) for f in ("baseline", "lateral_sigma", "disparity_sigma", "disparity_step",
                                          "min_cos_incidence", "shadow_tolerance", "dropout")]


class PlaneParams(C.Structure):
    """gpdb_plane_params (include/gpd_b200.h, rules in include/gpd_b200_plane.h)."""

    _fields_ = [
        ("distance_threshold", C.c_double),
        ("max_iterations", C.c_int32),
        ("probability", C.c_double),
        ("seed", C.c_uint64),
    ]


class TrainParams(C.Structure):
    """gpdb_train_params (include/gpd_b200.h, rules in include/gpd_b200_train.h)."""

    _fields_ = [
        ("optimizer", C.c_int32),
        ("lr", C.c_float),
        ("momentum", C.c_float),
        ("weight_decay", C.c_float),
        ("beta1", C.c_float),
        ("beta2", C.c_float),
        ("eps", C.c_float),
    ]


class TrainDebug(C.Structure):
    """gpdb_train_debug (include/gpd_b200.h): host buffers of gpdb_debug_train_step, any of them NULL."""

    _fields_ = [(f, C.c_void_p) for f in ("pool1", "pool2", "ip1", "logits", "choice1", "choice2", "loss", "dlogits",
                                          "dip1", "dpool2", "dpool1")] + [("grad", C.c_void_p * 8)]


_vp, _i32, _int = C.c_void_p, C.c_int32, C.c_int
_res, _pp, _sp, _pl = C.POINTER(Result), C.POINTER(PreprocessParams), C.POINTER(SisParams), C.POINTER(PlaneParams)

# Every function of include/gpd_b200.h, in its order: name -> (restype, argtypes). A pointer is c_void_p (a host or
# device address) unless it points to a boundary struct; tests/test_abi.py holds each entry against the declaration.
PROTOTYPES = {
    "gpdb_params_default": (None, [C.POINTER(Params)]),
    "gpdb_create": (_int, [C.POINTER(Params), C.POINTER(_vp)]),
    "gpdb_destroy": (None, [_vp]),
    "gpdb_last_error": (C.c_char_p, [_vp]),
    "gpdb_load_weights_dir": (_int, [_vp, C.c_char_p]),
    "gpdb_load_weights_file": (_int, [_vp, C.c_char_p, C.c_char_p]),
    "gpdb_read_weights_file": (_int, [C.c_char_p, C.c_char_p, _i32, _vp, _vp, C.c_char_p, _i32]),
    "gpdb_set_weights": (_int, [_vp] * 9),
    "gpdb_set_cloud": (_int, [_vp, _vp, _vp, _vp, _i32, _vp, _i32]),
    "gpdb_set_samples": (_int, [_vp, _vp, _i32]),
    "gpdb_detect": (_int, [_vp, _vp, _i32, _res]),
    "gpdb_detect_select": (_int, [_vp, _vp, _i32, _i32, _res]),
    "gpdb_detect_resident": (_int, [_vp, _vp, _i32, _vp, _vp, _res]),
    "gpdb_set_clouds": (_int, [_vp, _i32] + [_vp] * 6),
    "gpdb_detect_batch": (_int, [_vp, _vp, _vp, _res, _vp]),
    "gpdb_detect_batch_select": (_int, [_vp, _vp, _vp, _i32, _res, _vp]),
    "gpdb_set_clouds_samples": (_int, [_vp, _vp, _vp]),
    "gpdb_hand_search_batch": (_int, [_vp, _vp, _vp, _res, _vp]),
    "gpdb_set_stream": (_int, [_vp, _vp]),
    "gpdb_set_overlap": (_int, [_vp, _i32]),
    "gpdb_frames": (_int, [_vp, _vp, _i32, _vp, _vp]),
    "gpdb_hand_search": (_int, [_vp, _vp, _i32, _res]),
    "gpdb_images": (_int, [_vp, _vp, _i32, _vp]),
    "gpdb_classify": (_int, [_vp, _vp, _i32, _vp, _vp]),
    "gpdb_preprocess_params_default": (None, [_pp]),
    "gpdb_preprocess": (_int, [_vp, _vp, _vp, _vp, _i32, _vp, _i32, _pp]),
    "gpdb_get_cloud": (_int, [_vp, _vp, _vp, _vp]),
    "gpdb_get_cloud_source_index": (_int, [_vp, _vp]),
    "gpdb_preprocess_clouds": (_int, [_vp, _i32] + [_vp] * 6 + [_pp, _vp]),
    "gpdb_get_clouds": (_int, [_vp] * 5),
    "gpdb_preprocess_timings": (_int, [_vp, _vp]),
    "gpdb_reevaluate": (_int, [_vp, _vp, _i32, _vp]),
    "gpdb_reevaluate_batch": (_int, [_vp] * 4),
    "gpdb_find_clusters": (_int, [_vp, _vp, _i32, _i32, _vp]),
    "gpdb_find_clusters_batch": (_int, [_vp, _i32, _vp, _vp, _i32, _vp, _vp]),
    "gpdb_preprocess_clouds_device": (_int, [_vp, _i32] + [_vp] * 6 + [_pp, _vp]),
    "gpdb_set_clouds_device": (_int, [_vp, _i32] + [_vp] * 6),
    "gpdb_detect_batch_select_device": (_int, [_vp, _vp, _vp, _i32, _vp, _vp, _res]),
    "gpdb_find_clusters_batch_device": (_int, [_vp, _i32, _vp, _vp, _i32, _vp, _vp]),
    "gpdb_set_clouds_samples_device": (_int, [_vp, _vp, _vp]),
    "gpdb_hand_search_batch_device": (_int, [_vp] * 6 + [_res]),
    "gpdb_detect_batch_device": (_int, [_vp] * 7 + [_res]),
    "gpdb_images_batch_device": (_int, [_vp] * 4),
    "gpdb_classify_device": (_int, [_vp, _vp, _i32, _vp, _vp]),
    "gpdb_reevaluate_batch_device": (_int, [_vp] * 4),
    "gpdb_sis_params_default": (None, [_sp]),
    "gpdb_sis_batch": (_int, [_vp, _sp, _vp, _vp, _res, _vp]),
    "gpdb_sis_batch_device": (_int, [_vp, _sp, _vp, _vp, _vp, _vp, _res]),
    "gpdb_sis_positions": (_int, [_vp] * 6),
    "gpdb_preprocess_depth": (_int, [_vp, _i32, _vp, _vp, _i32, _vp, _pp, _vp]),
    "gpdb_preprocess_depth_device": (_int, [_vp, _i32, _vp, _vp, _i32, _vp, _pp, _vp]),
    "gpdb_normals_organized": (_int, [_vp, _i32] + [_vp] * 6),
    "gpdb_normals_organized_device": (_int, [_vp, _i32] + [_vp] * 6),
    "gpdb_preprocess_depth_organized": (_int, [_vp, _i32, _vp, _vp, _i32, _vp, _pp, _vp, _vp]),
    "gpdb_preprocess_depth_organized_device": (_int, [_vp, _i32, _vp, _vp, _i32, _vp, _pp, _vp, _vp]),
    "gpdb_subsample_clouds": (_int, [_vp, _i32, C.c_uint64, _vp, _vp, _vp]),
    "gpdb_subsample_clouds_device": (_int, [_vp, _i32, C.c_uint64, _vp, _vp, _vp]),
    "gpdb_plane_params_default": (None, [_pl]),
    "gpdb_segment_plane": (_int, [_vp, _pl, _vp, _vp, _vp]),
    "gpdb_segment_planes": (_int, [_vp, _pl, _vp, _vp, _vp, _vp]),
    "gpdb_segment_planes_device": (_int, [_vp, _pl, _vp, _vp, _vp, _vp]),
    "gpdb_refine_normals": (_int, [_vp, _i32, _vp]),
    "gpdb_refine_normals_clouds": (_int, [_vp, _i32, _vp]),
    "gpdb_remove_outliers": (_int, [_vp, _i32, C.c_double, _vp, _vp]),
    "gpdb_remove_outliers_clouds": (_int, [_vp, _i32, C.c_double, _vp, _vp, _vp]),
    "gpdb_subsample_clouds_points": (_int, [_vp, _i32, C.c_uint64, _vp, _vp, _vp]),
    "gpdb_subsample_clouds_points_device": (_int, [_vp, _i32, C.c_uint64, _vp, _vp, _vp]),
    "gpdb_render_depth": (_int, [_vp, _i32] + [_vp] * 5 + [_vp, _i32, _vp, _vp]),
    "gpdb_render_depth_device": (_int, [_vp, _i32] + [_vp] * 5 + [_vp, _i32, _vp, _vp]),
    "gpdb_sample_meshes": (_int, [_vp, _i32] + [_vp] * 4 + [C.c_double, C.c_uint64] + [_vp] * 4),
    "gpdb_sample_meshes_device": (_int, [_vp, _i32] + [_vp] * 4 + [C.c_double, C.c_uint64] + [_vp] * 4),
    "gpdb_sensor_params_default": (None, [_vp]),
    "gpdb_render_sensor_depth": (_int, [_vp, _i32] + [_vp] * 5 + [_vp, _i32, _vp, _vp, _vp, C.c_uint64]),
    "gpdb_render_sensor_depth_device": (_int, [_vp, _i32] + [_vp] * 5 + [_vp, _i32, _vp, _vp, _vp, C.c_uint64]),
    "gpdb_debug_sensor_table": (_int, [_vp]),
    "gpdb_free_result": (None, [_res]),
    "gpdb_comm_unique_id": (_int, [_vp]),
    "gpdb_comm_init": (_int, [_vp, _vp, _i32, _i32]),
    "gpdb_comm_destroy": (_int, [_vp]),
    "gpdb_shard_bounds": (None, [_i32, _i32, _i32, _vp, _vp, _vp]),
    "gpdb_set_cloud_bcast": (_int, [_vp, _i32, _vp, _vp, _vp, _i32, _vp, _i32]),
    "gpdb_detect_sharded": (_int, [_vp, _vp, _i32, _res]),
    "gpdb_detect_sharded_resident": (_int, [_vp, _vp, _i32, _i32, _vp, _res]),
    "gpdb_slot_bytes": (C.c_int64, [_i32, _i32]),
    "gpdb_last_timings": (_int, [_vp, _vp]),
    "gpdb_debug_phase_cycles": (_int, [_vp, _int, _vp]),
    "gpdb_debug_path_counts": (_int, [_vp, _vp]),
    "gpdb_debug_lenet_layers": (_int, [_vp, _vp, _i32, _vp, _vp, _vp, _vp]),
    "gpdb_train_begin": (_int, [_vp] * 3),
    "gpdb_train_step": (_int, [_vp, _vp, _vp, _i32, _vp]),
    "gpdb_train_step_device": (_int, [_vp, _vp, _vp, _i32, _vp]),
    "gpdb_train_weights": (_int, [_vp, _vp]),
    "gpdb_write_weights_dir": (_int, [C.c_char_p, _i32, _vp]),
    "gpdb_debug_train_step": (_int, [_vp, _vp, _vp, _i32, _vp]),
    "gpdb_build_info": (C.c_char_p, []),
}


def set_fields(p, **over):
    """Sets fields of a params struct by keyword and returns it. An array field takes all its values, except hand_axes,
    which takes 1..MAX_HAND_AXES axes and sets num_hand_axes to their count."""
    for k, v in over.items():
        if k == "hand_axes":
            p.num_hand_axes = len(v)
            p.hand_axes[:len(v)] = list(v)
        elif isinstance(getattr(p, k, None), C.Array):
            getattr(p, k)[:] = list(v)
        else:
            setattr(p, k, v)
    return p


def default_preprocess_params(**over):
    """Reference defaults (cfg/eigen_params.cfg:16-21, grasp_detector.cpp:56-66)."""
    p = PreprocessParams()
    p.workspace[:] = [-1.0, 1.0, -1.0, 1.0, -1.0, 1.0]
    p.voxel_size = 0.003
    p.normals_radius = 0.03
    p.voxelize = 1
    p.estimate_normals = 1
    return set_fields(p, **over)


def default_params(channels=15, **over):
    """The reference defaults (gpdb_params_default in C), restated for the oracle loader.

    cfg/hand_geometry.cfg:8-12, cfg/image_geometry_15channels.cfg:8-12, cfg/eigen_params.cfg:36-42,
    grasp_detector.cpp:158-174.
    """
    p = Params()
    p.finger_width, p.hand_outer_diameter, p.hand_depth = 0.01, 0.12, 0.06
    p.hand_height, p.init_bite = 0.02, 0.01
    p.volume_width, p.volume_depth, p.volume_height = 0.10, 0.06, 0.02
    p.image_size, p.image_num_channels = 60, channels
    p.nn_radius = 0.01
    p.num_orientations, p.num_finger_placements = 8, 10
    p.num_hand_axes = 1
    p.hand_axes[0] = 2
    p.deepen_hand = 1
    p.friction_coeff, p.min_viable = 20.0, 6
    p.min_aperture, p.max_aperture = 0.0, 0.085
    for i, v in enumerate([-1, 1, -1, 1, -1, 1]):
        p.workspace_grasps[i] = v
    p.filter_approach_direction = 0
    p.direction[0], p.direction[1], p.direction[2] = 1.0, 0.0, 0.0
    p.thresh_rad = 2.3
    p.batch_size = 0
    p.relu_after_conv = 0
    p.shadow_mode = 0
    p.device = 0
    p.chunk_samples = 0
    p.keep_images = 0
    p.lenet_impl = 0
    return set_fields(p, **over)


def result_to_numpy(res, image_bytes):
    """Copy a gpdb_result into numpy arrays (so the C result can be freed)."""
    n, P = res.n_samples, res.poses_per_sample
    nc = res.n_candidates
    full = bool(res.frames)  # gpdb_detect_select returns the selected pose records only
    out = {
        "n_samples": n,
        "poses_per_sample": P,
        "frame_valid": None if not full else np.ctypeslib.as_array(res.frame_valid, (n,)).copy() if n else np.zeros(0, np.uint8),
        "frames": None if not full else np.ctypeslib.as_array(res.frames, (n, 9)).copy() if n else np.zeros((0, 9)),
        "pose_flags": None if not full else np.ctypeslib.as_array(res.pose_flags, (n, P)).copy() if n else np.zeros((0, P), np.uint8),
        "pose_scores": None if not full else np.ctypeslib.as_array(res.pose_scores, (n, P)).copy() if n else np.zeros((0, P), np.float32),
        "n_candidates": nc,
        "n_total_candidates": res.n_total_candidates,
        "ms": (res.ms_candidates, res.ms_images, res.ms_classify),
        "kernel_launches": res.kernel_launches,
    }
    if nc:
        buf = C.string_at(res.candidates, nc * C.sizeof(Pose))
        out["candidates"] = np.frombuffer(buf, dtype=POSE_DTYPE).copy()
    else:
        out["candidates"] = np.zeros(0, dtype=POSE_DTYPE)
    if res.images and nc:
        out["images"] = np.ctypeslib.as_array(res.images, (nc, image_bytes)).copy()
    else:
        out["images"] = None
    return out
