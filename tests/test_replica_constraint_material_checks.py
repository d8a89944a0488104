"""The Python checks in front of the per-constraint replica material calls (Engine.set_replica_constraint_materials, its device form and
get_replica_materials).  The engine here is a stand-in whose library records what reaches it: no GPU is needed, and a refused argument
never reaches the library."""
import numpy as np
import pytest

from positionbaseddynamics_b200 import _capi

K, COUNT, NMAT = 3, 5, 2


class Iface:
    def __init__(self, shape, typestr="<f4", strides=None, ptr=0x7f0000000000, readonly=False):
        self.__cuda_array_interface__ = dict(shape=shape, typestr=typestr, strides=strides, data=(ptr, readonly), version=3)


class Lib:
    """Records every call of the library; each returns 0 (success)."""
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return 0
        return call


@pytest.fixture
def eng(monkeypatch):
    lib = Lib()
    monkeypatch.setattr(_capi, "lib", lambda: lib)
    e = object.__new__(_capi.Engine)
    e._h, e.K, e.n, e._nc = None, K, 4, 0
    e._constraint_materials_shape = lambda ctype: (K, COUNT, NMAT)
    e.calls = lib.calls
    return e


def names(eng):
    return [c[0] for c in eng.calls]


def test_host_form_takes_float32_c_contiguous_arrays_of_the_exact_shape(eng):
    mat = np.zeros((K, COUNT, NMAT), np.float32)
    eng.set_replica_constraint_materials(_capi.FEMTET, mat)
    assert names(eng) == ["pbd_set_replica_constraint_materials"]
    assert eng.calls[0][1][1] == _capi.FEMTET and eng.calls[0][1][2].value == mat.ctypes.data


def test_host_form_none_selects_the_shared_parameters(eng):
    eng.set_replica_constraint_materials(_capi.DISTANCE, None)
    assert names(eng) == ["pbd_set_replica_constraint_materials"] and eng.calls[0][1][2] is None


@pytest.mark.parametrize("bad, error, match", [
    (np.zeros((K, COUNT, NMAT), np.float64), ValueError, "element type float64"),
    (np.zeros((K, COUNT, NMAT), np.int32), ValueError, "element type int32"),
    (np.zeros((K * COUNT * NMAT,), np.float32), ValueError, "shape"),
    (np.zeros((K, COUNT + 1, NMAT), np.float32), ValueError, "shape"),
    (np.zeros((K - 1, COUNT, NMAT), np.float32), ValueError, "shape"),
    (np.zeros((NMAT, COUNT, K), np.float32).T, ValueError, "C-contiguous"),
    (np.zeros((K, COUNT, 2 * NMAT), np.float32)[:, :, ::2], ValueError, "C-contiguous"),
    (np.zeros((K, COUNT, NMAT)).tolist(), TypeError, "numpy array"),
    (Iface((K, COUNT, NMAT)), TypeError, "set_replica_constraint_materials_device"),
], ids=["f64", "i32", "flat", "count", "replicas", "fortran", "strided", "list", "device"])
def test_host_form_refusals_never_reach_the_library(eng, bad, error, match):
    with pytest.raises(error, match=match):
        eng.set_replica_constraint_materials(_capi.FEMTET, bad)
    assert eng.calls == []


def test_device_form_takes_any_shape_of_the_right_size_and_a_mask(eng):
    eng.set_replica_constraint_materials_device(_capi.FEMTET, Iface((K * COUNT * NMAT,)))
    eng.set_replica_constraint_materials_device(_capi.FEMTET, Iface((K, COUNT, NMAT), readonly=True),
                                                replicas=Iface((K,), "|b1", ptr=0x7f0000001000), stream=0)
    assert names(eng) == ["pbd_set_replica_constraint_materials_device"] * 2
    args = eng.calls[1][1]
    assert args[2].value == 0x7f0000000000 and args[3].value == 0x7f0000001000 and args[4].value == 1  # 0: the legacy default stream
    assert eng.calls[0][1][3] is None and eng.calls[0][1][4] is None


@pytest.mark.parametrize("bad, mask, error, match", [
    (None, None, TypeError, "mat is None"),
    (np.zeros((K, COUNT, NMAT), np.float32), None, TypeError, "__cuda_array_interface__"),
    (Iface((K, COUNT, NMAT), "<f8"), None, ValueError, "element type"),
    (Iface((K, COUNT, NMAT + 1)), None, ValueError, "elements"),
    (Iface((K * COUNT * NMAT,), strides=(8,)), None, ValueError, "C-contiguous"),
    (Iface((K, COUNT, NMAT)), Iface((K + 1,), "|u1"), ValueError, "replicas: .*elements"),
    (Iface((K, COUNT, NMAT)), Iface((K,), "<i4"), ValueError, "replicas: element type"),
], ids=["none", "host", "f64", "size", "strided", "mask-size", "mask-type"])
def test_device_form_refusals_never_reach_the_library(eng, bad, mask, error, match):
    with pytest.raises(error, match=match):
        eng.set_replica_constraint_materials_device(_capi.FEMTET, bad, replicas=mask)
    assert eng.calls == []


def test_get_fills_a_new_array_or_a_given_one(eng):
    got = eng.get_replica_materials(_capi.FEMTET)
    assert got.shape == (K, COUNT, NMAT) and got.dtype == np.float32
    out = np.empty((K, COUNT, NMAT), np.float32)
    assert eng.get_replica_materials(_capi.FEMTET, out=out) is out
    assert names(eng) == ["pbd_get_replica_materials"] * 2 and eng.calls[1][1][2].value == out.ctypes.data


@pytest.mark.parametrize("make, match", [
    (lambda: np.empty((K, COUNT, NMAT), np.float64), "element type"),
    (lambda: np.empty((K, COUNT), np.float32), "shape"),
    (lambda: np.empty((NMAT, COUNT, K), np.float32).T, "C-contiguous"),
    (lambda: np.frombuffer(bytes(K * COUNT * NMAT * 4), np.float32).reshape(K, COUNT, NMAT), "read-only"),
], ids=["f64", "shape", "fortran", "read-only"])
def test_get_refuses_an_output_it_cannot_write_in_place(eng, make, match):
    with pytest.raises(ValueError, match=match):
        eng.get_replica_materials(_capi.FEMTET, out=make())
    assert eng.calls == []
