"""The Python checks in front of the per-replica and device-memory rigid-body calls (Engine.set_replica_rigid_bodies,
set_rigid_bodies_device, get_rigid_bodies_device): on the CPU, on an Engine shell that never reaches the library."""
import ctypes as C

import numpy as np
import pytest

from positionbaseddynamics_b200 import _capi
from test_device_array_checks import Iface

K, NB = 3, 4


def shell():
    e = _capi.Engine.__new__(_capi.Engine)
    e._h, e.K, e.n, e.n_rb, e._nc = C.c_void_p(), K, 0, NB, 0
    return e


def test_set_replica_rigid_bodies_shapes():
    e = shell()
    good = dict(mass=np.ones((K, NB)), x=np.zeros((K, NB, 3)), q=np.zeros((K, NB, 4)), inertia=np.ones((K, NB, 3)))
    for name, bad in (("mass", np.ones(K * NB)), ("mass", np.ones((K + 1, NB))), ("x", np.zeros((K, NB, 4))), ("q", np.zeros((K, NB, 3))),
                      ("inertia", np.ones((K, NB + 1, 3)))):
        with pytest.raises(ValueError, match=name):
            e.set_replica_rigid_bodies(**dict(good, **{name: bad}))
    for name in ("v", "omega"):
        with pytest.raises(ValueError, match=name):
            e.set_replica_rigid_bodies(**good, **{name: np.zeros((K, NB, 4))})


def test_device_calls_check_every_array():
    e = shell()
    x, q = Iface((K * NB * 3,)), Iface((K, NB, 4))
    with pytest.raises(TypeError, match="x and q are required"):
        e.set_rigid_bodies_device(x, None)
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        e.set_rigid_bodies_device(np.zeros(K * NB * 3, np.float32), q)
    with pytest.raises(ValueError, match="q: .*elements"):
        e.set_rigid_bodies_device(x, Iface((K * NB * 3,)))
    with pytest.raises(ValueError, match="mass: .*elements"):
        e.set_rigid_bodies_device(x, q, mass=Iface((K * NB * 3,)))
    with pytest.raises(ValueError, match="inertia: element type"):
        e.set_rigid_bodies_device(x, q, inertia=Iface((K * NB * 3,), "<f8"))
    with pytest.raises(ValueError, match="omega: not C-contiguous"):
        e.set_rigid_bodies_device(x, q, omega=Iface((K * NB * 3,), strides=(8,)))
    with pytest.raises(ValueError, match="replicas: element type"):
        e.set_rigid_bodies_device(x, q, replicas=Iface((K,), "<i4"))
    with pytest.raises(ValueError, match="x: read-only"):
        e.get_rigid_bodies_device(x=Iface((K * NB * 3,), readonly=True))
    with pytest.raises(ValueError, match="v: .*elements"):
        e.get_rigid_bodies_device(v=Iface((K * NB * 4,)))
