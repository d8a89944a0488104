"""CPU checks of external forces (pbd_set_external_forces): the fp64 checker the GPU tests hold the engine to (the C restatement with an
external acceleration, tests/oracle_ext/external_accel.c), pinned bit for bit against the restatement's own step and gravity path, and the
Python checks in front of the host and device calls, which need no GPU and never let a refused argument reach the library."""
import ctypes as C

import numpy as np
import pytest

import resident_meshes as rm
import scenes
from external_forces_util import checker, ext_acceleration
from positionbaseddynamics_b200 import _capi
from test_device_array_checks import Iface

G = (0.0, -9.81, 0.0)
DT, SUB, ITER = 0.005, 3, 4
STATE = ("x", "v", "oldX", "lastX")


def _perturbed(cpu):
    rng = np.random.default_rng(5)
    x = cpu.get("x")
    _, w = cpu.masses()
    x[w != 0] += rng.uniform(-0.01, 0.01, x[w != 0].shape)
    cpu.set("x", x)
    return x


def _cloth(cpu, gravity):
    scenes.cloth(cpu, 12, 12, 4, 3, dist_k=1.0e5, bend_k=100.0, sub_steps=SUB, max_iter=ITER)
    cpu.set_params(dt=DT, sub_steps=SUB, max_iter=ITER, gravity=gravity)
    return _perturbed(cpu)


def _run(cpu, gravity, ext=None, build=_cloth, steps=3):
    """`steps` steps of the scene on `cpu` (the restatement keeps one model per library: each run builds it again); returns x, v, oldX,
    lastX, the start positions and the rigid bodies."""
    x0 = build(cpu, gravity)
    if ext is not None:
        cpu.set_ext_accel(np.broadcast_to(ext, (cpu.num_particles(), 3)))
    cpu.step(steps)
    return [cpu.get(k) for k in STATE] + [x0, cpu.rigid_bodies().copy()]


def _rig(cpu, gravity):
    rm.builder("solid", "small", rig=True)(cpu)
    cpu.set_params(dt=DT, sub_steps=2, max_iter=3, gravity=gravity)
    return _perturbed(cpu)


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("scene", ["cloth", "rig"])
def test_without_and_with_zero_acceleration_the_step_is_the_restatements(cpu_libs, precision, scene):
    """No acceleration set, and an acceleration of zero: the bits of the restatement's own step (orc_step), bodies included."""
    build = _cloth if scene == "cloth" else _rig
    ref = _run(cpu_libs.CpuPbd("oracle", precision), G, build=build, steps=2)
    for ext in (None, np.zeros(3)):
        got = _run(checker(cpu_libs, precision), G, ext, build=build, steps=2)
        for name, u, w in zip(STATE + ("x0", "bodies"), got, ref):
            assert np.array_equal(u, w), (scene, precision, ext, name)


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_uniform_acceleration_is_shifted_gravity(cpu_libs, precision):
    """A uniform external acceleration c under gravity g gives the bits of gravity g + c (the sum in the restatement's precision); the
    opposite acceleration does not."""
    dt = np.float64 if precision == "f64" else np.float32
    c = np.array([1.5, 4.0, -2.5])
    shifted = tuple(float(v) for v in np.asarray(G, dt) + np.asarray(c, dt))
    a = _run(cpu_libs.CpuPbd("oracle", precision), shifted)
    b = _run(checker(cpu_libs, precision), G, c)
    for name, u, w in zip(STATE, a, b):
        assert np.array_equal(u, w), (precision, name)
    flip = _run(checker(cpu_libs, precision), G, -c)
    moved = np.abs(a[0] - a[4]).max()
    assert moved > 1e-2 and np.abs(flip[0] - a[0]).max() / moved > 0.03


def test_per_particle_acceleration_and_clearing(cpu_libs):
    """Different accelerations per particle move the particles apart from the uniform case; static particles ignore theirs; clearing
    returns to the restatement's step."""
    rng = np.random.default_rng(3)
    cpu = checker(cpu_libs, "f64")
    x0 = _cloth(cpu, G)
    _, w = cpu.masses()
    cpu.set_ext_accel(rng.uniform(-10.0, 10.0, (cpu.num_particles(), 3)))
    cpu.step(2)
    x = cpu.get("x")
    assert np.array_equal(x[w == 0], x0[w == 0])
    cpu.set_ext_accel(None)
    state = [cpu.get(k) for k in STATE]
    cpu.step(1)
    got = [cpu.get(k) for k in STATE]
    plain = cpu_libs.CpuPbd("oracle", "f64")
    _cloth(plain, G)
    for k, s in zip(STATE, state):
        plain.set(k, s)
    plain.step(1)
    for name, u in zip(STATE, got):
        assert np.array_equal(u, plain.get(name)), name


def test_ext_acceleration_skips_static_particles():
    f = np.array([[2.0, 0.0, -4.0], [1.0, 1.0, 1.0]])
    assert np.array_equal(ext_acceleration(f, [2.0, 0.0]), [[1.0, 0.0, -2.0], [0.0, 0.0, 0.0]])


# ---- Python argument checks ----------------------------------------------------------------------------------------------------------
K, N = 3, 10


class _Lib:
    """Records the calls the checks let through."""
    def __init__(self):
        self.calls = []

    def pbd_set_external_forces(self, h, p):
        self.calls.append(("host", p)); return 0

    def pbd_set_external_forces_device(self, h, p, mask, stream):
        self.calls.append(("device", p.value, mask, stream)); return 0


@pytest.fixture
def fake(monkeypatch):
    lib = _Lib()
    monkeypatch.setattr(_capi, "lib", lambda: lib)
    return lib


def engine(k=K):
    e = object.__new__(_capi.Engine)
    e._h = C.c_void_p()
    e.K, e.n = k, N
    return e


def test_host_call_checks(fake):
    e = engine()
    with pytest.raises(TypeError, match="numpy array"):
        e.set_external_forces([[0.0] * 3] * (K * N))
    with pytest.raises(TypeError, match="numpy array"):
        e.set_external_forces(Iface((K, N, 3)))
    with pytest.raises(ValueError, match="element type float64"):
        e.set_external_forces(np.zeros((K, N, 3)))
    with pytest.raises(ValueError, match="shape"):
        e.set_external_forces(np.zeros((K * N, 3), np.float32))
    with pytest.raises(ValueError, match="shape"):
        e.set_external_forces(np.zeros((K, N + 1, 3), np.float32))
    with pytest.raises(ValueError, match="C-contiguous"):
        e.set_external_forces(np.zeros((3, N, K), np.float32).T)
    assert fake.calls == []
    e.set_external_forces(np.zeros((K, N, 3), np.float32))
    e.set_external_forces(None)
    assert fake.calls[0][0] == "host" and fake.calls[0][1] is not None
    assert fake.calls[1] == ("host", None)  # None clears
    one = engine(1)
    with pytest.raises(ValueError, match="shape"):
        one.set_external_forces(np.zeros((1, N, 3), np.float32))
    one.set_external_forces(np.zeros((N, 3), np.float32))  # (n, 3) at K = 1
    assert len(fake.calls) == 3


def test_device_call_checks(fake):
    e = engine()
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        e.set_external_forces_device(np.zeros((K, N, 3), np.float32))
    with pytest.raises(TypeError, match="set_external_forces\\(None\\)"):
        e.set_external_forces_device(None)
    with pytest.raises(ValueError, match="element type"):
        e.set_external_forces_device(Iface((K, N, 3), "<f8"))
    with pytest.raises(ValueError, match="elements"):
        e.set_external_forces_device(Iface((K, N - 1, 3)))
    with pytest.raises(ValueError, match="C-contiguous"):
        e.set_external_forces_device(Iface((K * N, 3), strides=(4, 4 * K * N)))
    with pytest.raises(ValueError, match="replicas: .*element type"):
        e.set_external_forces_device(Iface((K, N, 3)), replicas=Iface((K,), "<i4"))
    with pytest.raises(ValueError, match="replicas: .*elements"):
        e.set_external_forces_device(Iface((K, N, 3)), replicas=Iface((K + 1,), "|u1"))
    assert fake.calls == []
    e.set_external_forces_device(Iface((K * N * 3,)), replicas=Iface((K,), "|b1"), stream=0)
    kind, ptr, mask, stream = fake.calls[0]
    assert (kind, ptr, mask.value, stream.value) == ("device", 0x7f0000000000, 0x7f0000000000, 1)
    e.set_external_forces_device(Iface((K, N, 3)))
    assert fake.calls[1][2] is None and fake.calls[1][3] is None
