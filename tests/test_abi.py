"""CPU tests of the drop-in boundary: libgpd_b200.so loads, exports every symbol include/gpd_b200.h declares,
its structs have the layout the bindings assume, and it fails loudly (no CPU fallback) without a GPU."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import pytest

from gpd_b200 import abi, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    h = open(os.path.join(ROOT, "include", "gpd_b200.h")).read()
    h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
    return sorted(set(re.findall(r"\b(gpdb_[a-z0-9_]+)\s*\(", h)))


def test_library_exports_every_declared_symbol():
    L = lib.lib()
    syms = header_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/gpd_b200.h but not exported"
    assert set(lib.EXPORTS) == set(syms)


# the structs passed by reference, typed as pointers to their mirrors; arrays of records (gpdb_pose, gpdb_depth_camera)
# and every other pointer, host or device memory, are c_void_p, and a char * string is c_char_p
BY_REF = {"gpdb_params": abi.Params, "gpdb_result": abi.Result, "gpdb_preprocess_params": abi.PreprocessParams,
          "gpdb_sis_params": abi.SisParams, "gpdb_plane_params": abi.PlaneParams}
SCALARS = {"void": None, "int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
           "double": C.c_double}


def header_prototypes():
    """{name: (return type, [parameter declarations])} of every function include/gpd_b200.h declares."""
    h = open(os.path.join(ROOT, "include", "gpd_b200.h")).read()
    h = re.sub(r"/\*.*?\*/|//[^\n]*|^\s*#[^\n]*", "", h, flags=re.S | re.M)
    out = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\s*\b(gpdb_\w+)\s*\(([^)]*)\)\s*;", h):
        params = [" ".join(p.split()) for p in params.split(",")]
        out[name] = (" ".join(ret.split()), [] if params == ["void"] else params)
    return out


def ctype_of(decl):
    """The ctypes type that passes a C value declared as `decl` (a parameter or a return type)."""
    base = next(w for w in re.sub(r"[*\[\]]", " ", decl).split() if w != "const")
    depth = decl.count("*") + decl.count("[")
    if depth == 0:
        return SCALARS[base]
    if depth == 2:  # gpdb_ctx **ctx_out; float *const out[8]
        return C.POINTER(C.c_void_p) if base == "gpdb_ctx" else C.c_void_p
    if base in BY_REF:
        return C.POINTER(BY_REF[base])
    return C.c_char_p if base == "char" and "*" in decl else C.c_void_p


def test_prototypes_match_the_header():
    decls = header_prototypes()
    assert len(decls) >= 70 and set(decls) == set(abi.PROTOTYPES)
    for name, (ret, params) in decls.items():
        restype, argtypes = abi.PROTOTYPES[name]
        assert restype is ctype_of(ret), (name, ret, restype)
        assert len(argtypes) == len(params), (name, params, argtypes)
        for p, t in zip(params, argtypes):
            assert t is ctype_of(p), (name, p, t)


def test_struct_layouts_match_the_header():
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "gpd_b200.h"
int main(void) {
  printf("%zu %zu %zu\n", sizeof(gpdb_params), sizeof(gpdb_pose), sizeof(gpdb_result));
  printf("%zu %zu %zu %zu\n", offsetof(gpdb_params, nn_radius), offsetof(gpdb_params, workspace_grasps),
         offsetof(gpdb_params, batch_size), offsetof(gpdb_params, lenet_impl));
  printf("%zu %zu %zu %zu\n", offsetof(gpdb_pose, position), offsetof(gpdb_pose, score), offsetof(gpdb_pose, pose_slot),
         offsetof(gpdb_pose, half_antipodal));
  printf("%zu %zu %zu\n", offsetof(gpdb_result, candidates), offsetof(gpdb_result, ms_candidates),
         offsetof(gpdb_result, kernel_launches));
  printf("%zu %zu %zu\n", sizeof(gpdb_preprocess_params), offsetof(gpdb_preprocess_params, voxelize),
         offsetof(gpdb_result, n_total_candidates));
  return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        out = subprocess.check_output([os.path.join(d, "t")]).decode().split()
    nums = list(map(int, out))
    assert nums[0:3] == [C.sizeof(abi.Params), C.sizeof(abi.Pose), C.sizeof(abi.Result)]
    assert nums[3:7] == [abi.Params.nn_radius.offset, abi.Params.workspace_grasps.offset, abi.Params.batch_size.offset,
                         abi.Params.lenet_impl.offset]
    assert nums[7:11] == [abi.Pose.position.offset, abi.Pose.score.offset, abi.Pose.pose_slot.offset,
                          abi.Pose.half_antipodal.offset]
    assert nums[11:14] == [abi.Result.candidates.offset, abi.Result.ms_candidates.offset, abi.Result.kernel_launches.offset]
    assert nums[14:17] == [C.sizeof(abi.PreprocessParams), abi.PreprocessParams.voxelize.offset,
                           abi.Result.n_total_candidates.offset]
    assert abi.POSE_DTYPE.itemsize == C.sizeof(abi.Pose)


def test_defaults_are_the_reference_defaults():
    p = lib.default_params()
    q = abi.default_params(15)
    for name, _ in abi.Params._fields_:
        a, b = getattr(p, name), getattr(q, name)
        if hasattr(a, "__len__"):
            a, b = list(a), list(b)
        assert a == b, name
    # cfg/hand_geometry.cfg:8-12, cfg/image_geometry_15channels.cfg:8-12, cfg/eigen_params.cfg:36-42
    assert (p.finger_width, p.hand_outer_diameter, p.hand_depth, p.hand_height, p.init_bite) == (0.01, 0.12, 0.06, 0.02, 0.01)
    assert (p.volume_width, p.volume_depth, p.volume_height, p.image_size, p.image_num_channels) == (0.10, 0.06, 0.02, 60, 15)
    assert (p.num_orientations, p.num_finger_placements, p.friction_coeff, p.min_viable) == (8, 10, 20.0, 6)


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback_without_a_device():
    p = lib.default_params()
    with pytest.raises(lib.GpdbError) as e:
        lib.Context(p)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)


def test_product_never_touches_the_oracle():
    """The product path must not import, link or execute anything under oracle/."""
    bad = re.compile(r"(from\s+oracle|import\s+oracle|libgpd_oracle|#include\s+\".*oracle|oracle\.(lib|OracleCloud|classify)\()")
    for dirpath, _, files in os.walk(os.path.join(ROOT, "gpd_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")) or f == "Makefile":
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert not bad.search(txt), f
    out = subprocess.check_output(["ldd", lib.SO_PATH]).decode()
    assert "oracle" not in out
