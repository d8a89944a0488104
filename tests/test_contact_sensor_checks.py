"""The Python checks in front of pbd_set_replica_collider_poses_device and pbd_get_contact_sensors_device, on objects that only carry a
__cuda_array_interface__: they need no GPU, and a refused argument never reaches the library."""
import ctypes as C

import pytest

from positionbaseddynamics_b200 import _capi
from test_device_array_checks import Iface

K, NR = 3, 2


def engine():
    """An Engine as the checks see it after set_replicas(K) and set_replica_colliders with NR colliders per replica; no device handle."""
    e = object.__new__(_capi.Engine)
    e._h = C.c_void_p()
    e.K, e.n, e.n_rigid_colliders, e._replica_colliders = K, 10, NR, True
    return e


def test_collider_pose_refusals():
    e = engine()
    pose, bx = Iface((K, NR, 21)), Iface((K * NR * 3,))
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        e.set_replica_collider_poses_device([0.0] * (K * NR * 21), bx)
    with pytest.raises(ValueError, match="elements"):
        e.set_replica_collider_poses_device(Iface((K, NR, 20)), bx)
    with pytest.raises(ValueError, match="element type"):
        e.set_replica_collider_poses_device(Iface((K, NR, 21), "<f8"), bx)
    with pytest.raises(ValueError, match="body_x: .*elements"):
        e.set_replica_collider_poses_device(pose, Iface((K * NR * 3 - 1,)))
    with pytest.raises(ValueError, match="body_v: .*elements"):
        e.set_replica_collider_poses_device(pose, bx, body_v=Iface((K * NR,)))
    with pytest.raises(TypeError, match="body_x is required"):
        e.set_replica_collider_poses_device(pose, None)
    with pytest.raises(ValueError, match="replicas: .*element type"):
        e.set_replica_collider_poses_device(pose, bx, replicas=Iface((K,), "<i4"))


def test_contact_sensor_buffer_refusals():
    e = engine()
    with pytest.raises(ValueError, match="count: element type <i4, wants <u4"):
        e.get_contact_sensors_device(count=Iface((K * NR,), "<i4"))
    with pytest.raises(ValueError, match="count: .*elements"):
        e.get_contact_sensors_device(count=Iface((K * NR + 1,), "<u4"))
    with pytest.raises(ValueError, match="count: read-only"):
        e.get_contact_sensors_device(count=Iface((K * NR,), "<u4", readonly=True))
    with pytest.raises(ValueError, match="impulse: .*elements"):
        e.get_contact_sensors_device(impulse=Iface((K * NR,)))
    with pytest.raises(ValueError, match="impulse: read-only"):
        e.get_contact_sensors_device(impulse=Iface((K, NR, 3), readonly=True))
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        e.get_contact_sensors_device(impulse=[0.0] * (K * NR * 3))
    # the accepted shapes: any C-contiguous shape of the right size
    assert _capi._device_ptr("count", Iface((K, NR), "<u4"), ("<u4",), K * NR, writable=True)
    assert _capi._device_ptr("impulse", Iface((K, NR, 3)), ("<f4",), K * NR * 3, writable=True)
