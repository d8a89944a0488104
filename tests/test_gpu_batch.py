"""Replica batches on the GPU (pbd_set_replicas): replica r of a batch must advance bit for bit as an engine of its own started from
replica r's state, in every mode, including the XPBD multipliers."""
import numpy as np
import pytest

import scenes
from batch_util import AUTO, GRAPH, JACOBI, MODES, RESIDENT, SCENES, engine, model, replica_state, run, set_state

pytestmark = pytest.mark.gpu

_solo = {}


def solo(name, r):
    """Replica r stepped by an engine that never heard of batches."""
    from positionbaseddynamics_b200 import _capi
    if (name, r) not in _solo:
        m = model(name)
        x, v, mass = replica_state(m, r)
        eng = engine(m, GRAPH)
        eng.set_attr(_capi.ATTR_X, x); eng.set_attr(_capi.ATTR_V, v); eng.set_masses(mass)
        _solo[(name, r)] = run(eng, m)
        eng.close()
    return _solo[(name, r)]


@MODES
@pytest.mark.parametrize("k", [1, 3, 300])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_batch_equals_solo_runs(name, k, mode):
    """Replica r of a batch of k equals its solo run bit for bit (x, v, multipliers).  300 replicas are more than the device runs at
    once in the resident mode: its clusters step several replicas one after the other."""
    from positionbaseddynamics_b200 import _capi
    m = model(name)
    states = [replica_state(m, r) for r in range(k)]
    eng = engine(m, mode, replicas=k)
    assert eng.replicas() == k
    set_state(eng, states)
    x, v, lam = run(eng, m)
    st = eng.stats()
    eng.close()
    n = len(m["x"])
    assert x.shape == ((k, n, 3) if k > 1 else (n, 3))
    x, v = x.reshape(k, n, 3), v.reshape(k, n, 3)
    for r in sorted({0, 1, k // 2, k - 1} & set(range(k))):
        xs, vs, ls = solo(name, r)
        assert np.array_equal(x[r], xs), (name, k, mode, r)
        assert np.array_equal(v[r], vs), (name, k, mode, r)
        for t, l in ls.items():
            assert np.array_equal(lam[t].reshape(k, -1)[r], l), (name, k, mode, r, t)
    assert st.num_particles == n and st.num_constraints == len(m["types"])
    steps = [(m["sub"], m["it"])] * 2 + [(m["sub"] + 1, m["it"] + 1)] * 3
    assert st.projections == k * len(m["types"]) * sum(s * i for s, i in steps)


def test_replicas_start_as_copies_of_replica_zero():
    """set_replicas copies replica 0's current state into every replica; a batch of equal replicas steps them equally."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    x, v, mass = replica_state(m, 0)
    eng = engine(m, GRAPH)
    eng.set_attr(_capi.ATTR_X, x); eng.set_attr(_capi.ATTR_V, v)
    eng.step(1)
    want = {a: eng.get_attr(a).copy() for a in (_capi.ATTR_X, _capi.ATTR_V, _capi.ATTR_X0, _capi.ATTR_OLDX, _capi.ATTR_LASTX)}
    eng.set_replicas(4)
    for a, w in want.items():
        got = eng.get_attr(a)
        assert got.shape == (4,) + w.shape and all(np.array_equal(g, w) for g in got), a
    eng.step(2); eng.sync()
    xb = eng.get_attr(_capi.ATTR_X)
    assert all(np.array_equal(xb[r], xb[0]) for r in range(4))
    lam, _ = eng.lambdas(_capi.DISTANCE_XPBD)
    assert lam.shape[0] == 4 and all(np.array_equal(lam[r], lam[0]) for r in range(4))
    eng.close()
    # a batch size set while the engine holds no particles: the particles set afterwards start every replica
    empty = _capi.Engine(0)
    empty.set_replicas(3)
    empty.set_particles(x, mass, v=v)
    assert empty.replicas() == 3
    for a, w in ((_capi.ATTR_X, x), (_capi.ATTR_V, v), (_capi.ATTR_X0, x)):
        assert all(np.array_equal(g, w) for g in empty.get_attr(a)), a
    empty.close()


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_host_buffer_steps_equal_device_steps(mode):
    """step_host and step_host_async with K*n buffers compute what set_attr + step + get_attr compute."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k = 3
    states = [replica_state(m, r) for r in range(k)]
    xs = np.ascontiguousarray(np.stack([s[0] for s in states])); vs = np.ascontiguousarray(np.stack([s[1] for s in states]))
    outs = []
    for how in ("device", "host", "async"):
        eng = engine(m, mode, replicas=k)
        x_out = np.empty_like(xs); v_out = np.empty_like(vs)
        if how == "device":
            eng.set_attr(_capi.ATTR_X, xs); eng.set_attr(_capi.ATTR_V, vs)
            eng.step(3); eng.sync()
            x_out[:] = eng.get_attr(_capi.ATTR_X); v_out[:] = eng.get_attr(_capi.ATTR_V)
        elif how == "host":
            eng.step_host(3, xs, vs, x_out, v_out)
        else:
            eng.step_host_async(3, xs, vs, x_out, v_out)
            eng.step_host_wait(0)
        outs.append((x_out, v_out))
        eng.close()
    for x_out, v_out in outs[1:]:
        assert np.array_equal(x_out, outs[0][0]) and np.array_equal(v_out, outs[0][1])


def test_batch_refusals():
    """Rigid bodies, colliders and the Jacobi mode are refused at K > 1 before anything changes; a replica too big for one cluster is
    refused by the resident mode and runs in graph mode under AUTO."""
    from positionbaseddynamics_b200 import _capi
    m = model("cfg1")
    eng = engine(m, GRAPH, replicas=2)
    with pytest.raises(_capi.PbdError, match="rigid bodies"):
        eng.set_rigid_bodies([1.0], [[0, 0, 0]], [[1, 0, 0, 0]], [[1, 1, 1]])
    with pytest.raises(_capi.PbdError, match="colliders"):
        eng.set_colliders([_capi.ParticleCollider(0, len(m["x"]), 0.5, 0.1)], [])
    with pytest.raises(_capi.PbdError, match="PBD_MODE_JACOBI"):
        eng.set_mode(JACOBI)
    assert eng.get_mode()[0] == GRAPH and eng.replicas() == 2
    eng.step(1); eng.sync()
    eng.close()
    one = engine(m, GRAPH)
    one.set_rigid_bodies([1.0], [[0, 0, 0]], [[1, 0, 0, 0]], [[1, 1, 1]])
    with pytest.raises(_capi.PbdError, match="rigid bodies"):
        one.set_replicas(2)
    assert one.replicas() == 1
    with pytest.raises(_capi.PbdError, match="at least one replica"):
        one.set_replicas(0)
    one.close()

    from positionbaseddynamics_b200.model import HostModel
    hm = HostModel()
    scenes.cloth(hm, 500, 500, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=1, max_iter=2)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    big = dict(types=types, bodies=bodies, params=params, off=off, ids=ids, x=hm.get("x"), x0=hm.get("x0"), mass=mass, dt=0.005, sub=1, it=2)
    hm.close()
    res = engine(big, RESIDENT, replicas=2)
    with pytest.raises(_capi.PbdError, match="does not fit one cluster"):
        res.step(1)
    res.close()
    auto = engine(big, AUTO, replicas=2)
    auto.step(1); auto.sync()
    assert auto.get_mode() == (AUTO, GRAPH)
    x = auto.get_attr(_capi.ATTR_X)
    assert np.isfinite(x).all() and np.array_equal(x[0], x[1])
    auto.close()
