"""Context.reevaluate_batch / reevaluate_batch_tensors against a stand-in library (CPU): the group offsets passed to
gpdb_reevaluate_batch[_device] are built from the hand lists, the records are labelled in place (the host method hands
back the re-labelled copies per group, the tensor method updates the caller's tensor) and the labels come back per
group."""
import ctypes as C

import numpy as np
import pytest

from gpd_b200 import abi, lib


class FakeLib:
    """Labels hand i with i % 2 and sets its full flag to match, as the library writes both."""

    def __init__(self):
        self.offsets = None

    def _label(self, h, hoff, hands, labels, B=3):
        self.offsets = np.ctypeslib.as_array(C.cast(hoff, C.POINTER(C.c_int32)), (B + 1,)).copy()
        n = int(self.offsets[-1])
        if n:
            rec = np.ctypeslib.as_array(C.cast(hands, C.POINTER(C.c_uint8)), (n * lib.POSE_BYTES,)).view(abi.POSE_DTYPE)
            lab = np.ctypeslib.as_array(C.cast(labels, C.POINTER(C.c_int32)), (n,))
            lab[:] = np.arange(n) % 2
            rec["full_antipodal"] = lab
        return n

    gpdb_reevaluate_batch = gpdb_reevaluate_batch_device = _label

    def gpdb_last_error(self, h):
        return b"stand-in error"


def context(monkeypatch, fake):
    monkeypatch.setattr(lib, "lib", lambda: fake)
    ctx = object.__new__(lib.Context)
    ctx.h = None
    ctx.params = abi.default_params(15)
    ctx._n_clouds = 3
    ctx._batch = (np.array([0, 5, 9, 12], np.int32), np.array([1, 1, 1], np.int32), np.zeros((3, 3)), False)
    return ctx


def hands(n, start):
    h = np.zeros(n, abi.POSE_DTYPE)
    h["sample_index"] = np.arange(start, start + n)
    return h


def test_reevaluate_batch_offsets_and_records(monkeypatch):
    fake = FakeLib()
    ctx = context(monkeypatch, fake)
    groups = [hands(3, 0), hands(0, 3), hands(2, 3)]
    labels, recs = ctx.reevaluate_batch(groups)
    assert list(fake.offsets) == [0, 3, 3, 5]
    assert [list(x) for x in labels] == [[0, 1, 0], [], [1, 0]]
    for g, r in zip(groups, recs):
        assert np.array_equal(r["sample_index"], g["sample_index"])
    assert [list(r["full_antipodal"]) for r in recs] == [[0, 1, 0], [], [1, 0]]
    assert not any(g["full_antipodal"].any() for g in groups)  # the caller's arrays are not written
    with pytest.raises(ValueError):
        ctx.reevaluate_batch(groups[:2])  # one list per installed cloud


def test_reevaluate_batch_tensors_updates_in_place(monkeypatch):
    torch = pytest.importorskip("torch")
    fake = FakeLib()
    ctx = context(monkeypatch, fake)
    # the device checks, the stream switch and the CUDA allocation need a GPU; the bookkeeping does not
    monkeypatch.setattr(lib, "_device_arg", lambda name, t, *a, **k: C.c_void_p(t.data_ptr()))
    monkeypatch.setattr(lib.Context, "_torch_stream", lambda self: None)
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, device=None, **k: empty(*a, **k))
    h = np.concatenate([hands(4, 0), hands(1, 4)])
    t = torch.from_numpy(h.view(np.uint8).reshape(5, lib.POSE_BYTES).copy())
    labels = ctx.reevaluate_batch_tensors([0, 4, 4, 5], t)
    assert list(fake.offsets) == [0, 4, 4, 5]
    assert labels.dtype == torch.int32 and labels.tolist() == [0, 1, 0, 1, 0]
    assert list(lib.poses_from_tensor(t)["full_antipodal"]) == [0, 1, 0, 1, 0]
    with pytest.raises(ValueError):
        ctx.reevaluate_batch_tensors([0, 5], t)  # B + 1 offsets
