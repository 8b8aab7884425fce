#!/usr/bin/env python
"""Generate tests/golden/cfg_reference_parse.json: what the reference's own util::ConfigFile, candidate::HandGeometry and
descriptor::ImageGeometry return for the cfg files under tests/golden/cfg/ (the reference's shipped files plus tricky.cfg,
the format's corner cases). Needs oracle/_ref/libgpd_ref_config.so (`make -C oracle _ref`, from the reference sources).
tests/test_host_cpp.py::test_cfg_parser_against_the_references_own_parser checks the shim's parser against this file."""
import ctypes as C
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "tests", "golden", "cfg")
OUT = os.path.join(ROOT, "tests", "golden", "cfg_reference_parse.json")

KEYS_TRICKY = ["alpha", "beta", "gamma", "delta", "vec", "flag0", "flag1", "empty_after_hash", "int_as_float", "weights_file",
               "spaced", "spaced key", "missing"]
KEYS_SHIPPED = ["hand_geometry_filename", "image_geometry_filename", "weights_file", "model_file", "workspace", "workspace_grasps",
                "num_samples", "num_threads", "voxelize", "voxel_size", "hand_axes", "finger_width", "hand_outer_diameter",
                "volume_width", "image_num_channels", "camera_position", "min_inliers", "num_selected", "direction", "thresh_rad"]
SHIPPED = ["eigen_params.cfg", "caffe_params.cfg", "vino_params_12channels.cfg", "hand_geometry.cfg",
           "image_geometry_15channels.cfg", "ros_eigen_params.cfg"]
GEOMETRY = ["tricky.cfg", "does_not_exist.cfg", "hand_geometry.cfg", "ur5_hand_geometry.cfg", "image_geometry_15channels.cfg",
            "image_geometry_12channels.cfg", "image_geometry_3channels.cfg", "image_geometry_1channels.cfg", "eigen_params.cfg"]


def bind(L, pre, names):
    """names = suffixes of the (double, int, bool, doubles) getters."""
    getattr(L, pre).argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
    for suf, t in zip(names[:3], (C.c_double, C.c_int, C.c_int)):
        f = getattr(L, pre + suf)
        f.argtypes, f.restype = [C.c_char_p, C.c_char_p, t], t
    getattr(L, pre + names[3]).argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int]


def get(L, pre, names, path, key):
    """(found, string value, getDouble, getInt, getBool, number of doubles, the doubles) of one key."""
    buf = C.create_string_buffer(512)
    found = getattr(L, pre)(path.encode(), key.encode(), b"<default>", buf, 512)
    vec = (C.c_double * 16)()
    nv = getattr(L, pre + names[3])(path.encode(), key.encode(), b"1.5 2.5", vec, 16)
    return [found, buf.value.decode(), getattr(L, pre + names[0])(path.encode(), key.encode(), -7.25),
            getattr(L, pre + names[1])(path.encode(), key.encode(), -7), getattr(L, pre + names[2])(path.encode(), key.encode(), 1),
            nv, list(vec[:min(nv, 16)])]


def geometry(L, hg, ig, path):
    a, b, c = (C.c_double * 5)(), (C.c_double * 3)(), (C.c_int * 2)()
    getattr(L, hg)(path.encode(), a)
    getattr(L, ig)(path.encode(), b, c)
    return [list(a), list(b), list(c)]


def main():
    R = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libgpd_ref_config.so"))
    names = ("_double", "_int", "_bool", "_doubles")
    bind(R, "gpdref_config_get", names)
    out = {"keys": {}, "geometry": {}}
    for name, keys in [("tricky.cfg", KEYS_TRICKY)] + [(n, KEYS_SHIPPED) for n in SHIPPED] + [("does_not_exist.cfg", ["alpha"])]:
        out["keys"][name] = {k: get(R, "gpdref_config_get", names, os.path.join(CFG, name), k) for k in keys}
    for name in GEOMETRY:
        out["geometry"][name] = geometry(R, "gpdref_hand_geometry", "gpdref_image_geometry", os.path.join(CFG, name))
    with open(OUT, "w") as f:  # one line per key
        f.write('{"keys": {\n' + ',\n'.join(f' {json.dumps(n)}: {{\n' + ',\n'.join(f'  {json.dumps(k)}: {json.dumps(v)}' for k, v in ks.items())
                                            + '}' for n, ks in out["keys"].items()) + '},\n')
        f.write('"geometry": {\n' + ',\n'.join(f' {json.dumps(n)}: {json.dumps(v)}' for n, v in out["geometry"].items()) + '}}\n')


if __name__ == "__main__":
    main()
