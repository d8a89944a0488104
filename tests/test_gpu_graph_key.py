"""The graph mode replays a captured step only while everything the capture read is unchanged (graph_key in engine.cu).  One scripted
sequence of state changes, with a few steps after each, runs on a graph-mode engine and on a launch-mode engine.  Both run the same
kernels with the same arguments, so after every segment their positions must be bit-identical.  The sequence covers every call that
changes what the captured step reads."""
import numpy as np
import pytest

import scenes
from batch_util import GRAPH, LAUNCH, RESIDENT, engine, model, replica_state, set_state

pytestmark = pytest.mark.gpu

STIFFNESS = {1: 1.0e5, 4: 100.0}  # xpbd_cloth64: Distance_XPBD and IsometricBending_XPBD, whose one material parameter is the stiffness
EXTRA = 37  # free particles the engines start with, beyond the cloth's


def segment(engines, what, change, steps=2):
    """change(engine) on both engines, `steps` steps, then the same positions."""
    from positionbaseddynamics_b200 import _capi
    for e in engines:
        change(e)
    for e in engines:
        e.step(steps)
    xg, xl = (e.get_attr(_capi.ATTR_X) for e in engines)
    assert np.array_equal(xg, xl), what


def test_graph_follows_every_state_change():
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    assert {int(t) for t in np.unique(m["types"])} == set(STIFFNESS)
    rng = np.random.default_rng(7)
    free = (rng.normal(0.0, 1.0, (EXTRA, 3)) + (0.0, 5.0, 0.0)).astype(np.float32)
    big = dict(m, x=np.concatenate([m["x"], free]), x0=np.concatenate([m["x0"], free]), mass=np.concatenate([m["mass"], np.ones(EXTRA, np.float32)]))
    engines = (engine(big, GRAPH), engine(big, LAUNCH))
    sub, it = m["sub"], m["it"]

    def on_graph(change):  # the graph engine alone: the launch engine stays in its mode
        return lambda e: change(e) if e is engines[0] else None

    segment(engines, "first steps", lambda e: None)
    segment(engines, "set_params: new dt", lambda e: e.set_params(dt=0.004, sub_steps=sub, max_iter=it))
    segment(engines, "set_params: the same values", lambda e: e.set_params(dt=0.004, sub_steps=sub, max_iter=it))
    segment(engines, "set_params: everything else", lambda e: e.set_params(dt=0.004, sub_steps=sub + 1, max_iter=it + 1, vel_method=1, gravity=(0.5, -9.0, 0.0)))
    pinned = big["mass"].copy(); pinned[::5] = 0.0
    segment(engines, "set_masses", lambda e: e.set_masses(pinned))
    segment(engines, "set_particles: fewer particles", lambda e: e.set_particles(m["x"], m["mass"], x0=m["x0"]))

    for k in (4, 2):
        segment(engines, "set_replicas %d" % k, lambda e: (e.set_replicas(k), set_state(e, [replica_state(m, r) for r in range(k)])))
    k = 2  # the batch size from here on

    def materials(scale):
        return lambda e: [e.set_replica_materials(t, None if scale is None else [[s * scale(r)] for r in range(k)]) for t, s in STIFFNESS.items()]
    segment(engines, "set_replica_materials on", materials(lambda r: 0.5 + r))
    segment(engines, "set_replica_materials rewritten", materials(lambda r: 2.0 - 0.75 * r))
    segment(engines, "set_replica_materials off", materials(None))

    segment(engines, "set_replica_gravity on", lambda e: e.set_replica_gravity([(0.0, -9.81, 0.0), (1.5, -7.0, -2.5)]))
    segment(engines, "set_replica_gravity rewritten", lambda e: e.set_replica_gravity([(0.0, 0.0, 0.0), (-1.0, -12.0, 0.5)]))
    segment(engines, "set_replica_gravity off", lambda e: e.set_replica_gravity(None))

    c = m["x0"].mean(axis=0)

    def rest(scales):
        return lambda e: e.set_replica_rest_positions(None if scales is None else np.stack([c + (m["x0"] - c) * np.float32(s) for s in scales]).astype(np.float32))
    segment(engines, "set_replica_rest_positions on", rest((1.05, 0.9)))
    segment(engines, "set_replica_rest_positions rewritten", rest((0.95, 1.1)))
    segment(engines, "set_replica_rest_positions off", rest(None))

    pairs = np.array([(i, i + 65) for i in range(0, 63, 3)], dtype=np.uint32)  # diagonals of the 64 x 64 grid
    params = np.zeros((len(pairs), _capi.num_params(1)), np.float32)
    params[:, 0] = np.linalg.norm(m["x0"][pairs[:, 0]] - m["x0"][pairs[:, 1]], axis=1)
    params[:, 1] = STIFFNESS[1]
    segment(engines, "add_constraints after a step", lambda e: e.add_constraints(1, pairs, params))

    segment(engines, "set_mode resident", on_graph(lambda e: e.set_mode(RESIDENT)))
    assert engines[0].get_mode() == (RESIDENT, RESIDENT)
    segment(engines, "set_mode graph", on_graph(lambda e: e.set_mode(GRAPH)))
    for e in engines:
        e.close()


def test_graph_follows_set_rigid_bodies():
    """A single scene with ball joints: new rigid-body state between steps (pbd_set_rigid_bodies)."""
    from positionbaseddynamics_b200 import _capi
    from positionbaseddynamics_b200.model import HostModel
    hm = HostModel()
    scenes.cfg4(hm, 16, (5, 3, 3))
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x, x0, rb = hm.get("x").copy(), hm.get("x0").copy(), hm.rigid_bodies().copy()
    hm.close()
    assert (types == _capi.BALLJOINT).any()
    rb_mass = np.array([0.0 if i % 3 == 0 else 1.0 for i in range(len(rb))], np.float32)  # scenes.coupling_rig
    inertia = [scenes.box_inertia(1.0, 0.5, 0.5, 0.5) if i % 3 == 0 else scenes.box_inertia(1.0, 0.4, 2.0, 0.4) for i in range(len(rb))]
    engines = []
    for mode in (GRAPH, LAUNCH):
        e = _capi.Engine(0)
        e.set_particles(x, mass, x0=x0)
        e.set_rigid_bodies(rb_mass, rb[:, :3], rb[:, 3:7], inertia)
        e.add_flat(types, bodies, params)
        e.set_groups(off, ids)
        e.set_params(dt=0.005, sub_steps=5, max_iter=1)
        e.set_mode(mode)
        engines.append(e)

    def kick(e):
        s = e.get_rigid_bodies()
        e.set_rigid_bodies(rb_mass, s[:, :3], s[:, 3:7], inertia, v=s[:, 7:10] + (rb_mass[:, None] > 0) * np.float32(0.5), omega=s[:, 10:])
    segment(engines, "first steps", lambda e: None, steps=3)
    for n in range(2):
        segment(engines, "set_rigid_bodies %d" % n, kick, steps=3)
        assert np.array_equal(engines[0].get_rigid_bodies(), engines[1].get_rigid_bodies())
    for e in engines:
        e.close()
