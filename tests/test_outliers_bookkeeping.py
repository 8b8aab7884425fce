"""Context.remove_outliers_clouds keeps its batch bookkeeping in step with the library (CPU, a stand-in library): after
GPDB_ERR_INVALID or GPDB_ERR_STATE, which change nothing, the batch stays; after any other error the library holds no
batch, so the bookkeeping that sizes the output buffers of later batch calls holds none either; after success the
offsets are the new ones and the SIS record is gone."""
import numpy as np
import pytest

from gpd_b200 import lib


class FakeLib:
    def __init__(self, rc):
        self.rc = rc

    def gpdb_remove_outliers_clouds(self, h, mean_k, mul, off, stats, kept):
        if self.rc >= 0:
            np.ctypeslib.as_array(lib.C.cast(off, lib.C.POINTER(lib.C.c_int32)), (3,))[:] = [0, 4, 6]
        return self.rc

    def gpdb_last_error(self, h):
        return b"stand-in error"


def batch_context(monkeypatch, rc):
    monkeypatch.setattr(lib, "lib", lambda: FakeLib(rc))
    ctx = object.__new__(lib.Context)
    ctx.h = None  # no library context: close() has nothing to free
    ctx._n_clouds = 2
    ctx._batch = (np.array([0, 5, 9], np.int32), np.array([1, 1], np.int32), np.zeros((2, 3)), True)
    ctx._sis_shape = (2, 3)
    ctx._n_raw = 20
    return ctx


@pytest.mark.parametrize("rc", [-1, -3])
def test_errors_before_device_work_keep_the_batch(monkeypatch, rc):
    ctx = batch_context(monkeypatch, rc)
    with pytest.raises(lib.GpdbError):
        ctx.remove_outliers_clouds(10)
    assert ctx._n_clouds == 2 and list(ctx._batch[0]) == [0, 5, 9] and ctx._sis_shape == (2, 3) and ctx._n_raw == 20


@pytest.mark.parametrize("rc", [-2, -5])
def test_other_errors_drop_the_batch(monkeypatch, rc):
    ctx = batch_context(monkeypatch, rc)
    with pytest.raises(lib.GpdbError):
        ctx.remove_outliers_clouds(10)
    assert ctx._n_clouds == 0 and ctx._batch is None and ctx._sis_shape is None and ctx._n_raw is None


def test_success_installs_the_new_offsets(monkeypatch):
    ctx = batch_context(monkeypatch, 2)
    r = ctx.remove_outliers_clouds(10)
    assert list(r["offsets"]) == [0, 4, 6] and list(ctx._batch[0]) == [0, 4, 6]
    assert ctx._n_clouds == 2 and ctx._sis_shape is None and ctx._n_raw == 20 and ctx._batch[3]
