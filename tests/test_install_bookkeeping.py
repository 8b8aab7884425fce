"""Every Context method that installs a batch keeps its batch bookkeeping in step with the library (CPU, a stand-in
library): a failed install leaves no batch, in the library as here, and a successful one records the batch's point
offsets, camera counts, view points, whether its clouds keep source indices and how many raw points they came from."""
import numpy as np
import pytest

from gpd_b200 import abi, lib

PP = abi.default_preprocess_params()
CLOUDS = [{"xyz": np.zeros((n, 3)), "normals": np.zeros((n, 3))} for n in (3, 2)]
CAMERAS = [lib.depth_camera(4, 2, 1, 1, 0, 0), lib.depth_camera(3, 1, 1, 1, 0, 0)]
PROCESSED = [0, 2, 3]  # the point offsets the stand-in preprocessing calls write


class FakeLib:
    def __init__(self, rc):
        self.rc = rc

    def _install(self, *args):
        return self.rc

    def _preprocess(self, *args):  # the processed point offsets are the last argument
        if self.rc >= 0:
            np.ctypeslib.as_array(lib.C.cast(args[-1], lib.C.POINTER(lib.C.c_int32)), (3,))[:] = PROCESSED
        return self.rc

    gpdb_set_clouds = gpdb_set_clouds_device = _install
    gpdb_preprocess_clouds = gpdb_preprocess_clouds_device = gpdb_preprocess_depth = _preprocess

    def gpdb_last_error(self, h):
        return b"stand-in error"


# method -> (the install, the point offsets it records, the raw points of a preprocessing call)
INSTALLS = {
    "set_clouds": (lambda ctx: ctx.set_clouds(CLOUDS), [0, 3, 5], None),
    "set_clouds_tensors": (lambda ctx: ctx.set_clouds_tensors([0, 3, 5], None, None, [1, 1], np.zeros((2, 3))),
                           [0, 3, 5], None),
    "preprocess_clouds": (lambda ctx: ctx.preprocess_clouds(CLOUDS, PP, read_back=False), PROCESSED, 5),
    "preprocess_clouds_tensors": (lambda ctx: ctx.preprocess_clouds_tensors([0, 3, 5], None, [1, 1], np.zeros((2, 3)),
                                                                            pp=PP), PROCESSED, 5),
    "_install_depth": (lambda ctx: ctx._install_depth(lib.lib().gpdb_preprocess_depth, [1, 1], CAMERAS, abi.DEPTH_U16,
                                                      None, PP), PROCESSED, 4 * 2 + 3 * 1),
}


def installed_context(monkeypatch, rc):
    monkeypatch.setattr(lib, "lib", lambda: FakeLib(rc))
    # the tensor methods' device checks and stream switch need a GPU; the bookkeeping does not
    monkeypatch.setattr(lib, "_device_arg", lambda *args, **kw: None)
    monkeypatch.setattr(lib.Context, "_torch_stream", lambda self: None)
    ctx = object.__new__(lib.Context)
    ctx.h = None  # no library context: close() has nothing to free
    ctx.params = abi.default_params(15)
    ctx._n_clouds = 2  # a batch installed earlier, which any install replaces
    ctx._batch = (np.array([0, 5, 9], np.int32), np.array([1, 1], np.int32), np.zeros((2, 3)), True)
    ctx._sis_shape = (2, 3)
    ctx._n_raw = 20
    return ctx


@pytest.mark.parametrize("method", INSTALLS)
@pytest.mark.parametrize("rc", [-1, -2, 0])
def test_install_records_the_batch_or_none(monkeypatch, method, rc):
    install, offsets, n_raw = INSTALLS[method]
    ctx = installed_context(monkeypatch, rc)
    if rc < 0:
        with pytest.raises(lib.GpdbError):
            install(ctx)
        assert ctx._n_clouds == 0 and ctx._batch is None and ctx._sis_shape is None and ctx._n_raw is None
        return
    install(ctx)
    assert ctx._n_clouds == 2 and ctx._sis_shape is None and ctx._n_raw == n_raw
    off, ks, vps, has_src = ctx._batch
    assert list(off) == offsets and list(ks) == [1, 1] and vps.shape == (2, 3) and has_src == (n_raw is not None)
