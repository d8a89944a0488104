"""The Python checks in front of the device-memory state calls (_capi._device_ptr, _capi._stream), on objects that only carry a
__cuda_array_interface__: they need no GPU, and a refused argument never reaches the library."""
import pytest

from positionbaseddynamics_b200 import _capi


class Iface:
    def __init__(self, shape, typestr="<f4", strides=None, ptr=0x7f0000000000, readonly=False):
        self.__cuda_array_interface__ = dict(shape=shape, typestr=typestr, strides=strides, data=(ptr, readonly), version=3)


def test_accepts_contiguous_arrays_of_the_right_size():
    assert _capi._device_ptr("x", Iface((4, 5, 3)), ("<f4",), 60) == 0x7f0000000000
    assert _capi._device_ptr("x", Iface((60,), strides=(4,)), ("<f4",), 60)
    assert _capi._device_ptr("x", Iface((4, 1, 15), strides=(60, 4, 4)), ("<f4",), 60)  # the stride of an extent-1 axis is free
    assert _capi._device_ptr("mask", Iface((3,), "|b1"), ("|b1", "|u1"), 3)
    assert _capi._device_ptr("mask", Iface((3,), "|u1"), ("|b1", "|u1"), 3)


def test_refusals():
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        _capi._device_ptr("x", [0.0] * 60, ("<f4",), 60)
    with pytest.raises(ValueError, match="element type"):
        _capi._device_ptr("x", Iface((60,), "<f8"), ("<f4",), 60)
    with pytest.raises(ValueError, match="element type"):
        _capi._device_ptr("mask", Iface((3,), "<i4"), ("|b1", "|u1"), 3)
    with pytest.raises(ValueError, match="C-contiguous"):
        _capi._device_ptr("x", Iface((60,), strides=(8,)), ("<f4",), 60)
    with pytest.raises(ValueError, match="C-contiguous"):
        _capi._device_ptr("x", Iface((20, 3), strides=(4, 80)), ("<f4",), 60)  # Fortran order
    with pytest.raises(ValueError, match="elements"):
        _capi._device_ptr("x", Iface((59,)), ("<f4",), 60)
    with pytest.raises(ValueError, match="read-only"):
        _capi._device_ptr("out", Iface((60,), readonly=True), ("<f4",), 60, writable=True)
    assert _capi._device_ptr("src", Iface((60,), readonly=True), ("<f4",), 60)  # a source may be read-only


def test_stream_handles():
    assert _capi._stream(None) is None
    assert _capi._stream(0).value == 1  # torch's default stream: the legacy default stream, not the engine's (NULL)
    assert _capi._stream(0x1234).value == 0x1234
