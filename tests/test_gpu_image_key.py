"""The device image is planned again whenever something it is planned from changes, and only then (image_key in engine.cu).  One
scripted sequence of state changes, with a few steps after each, runs on one engine.  After every segment an engine built fresh through
the C ABI in that segment's state, and stepped the same way, must reach the same positions bit for bit and report the same mode.  A new
plan zeroes the XPBD multipliers, so reading them straight after a call tells whether the call had the image planned again."""
import numpy as np
import pytest

import scenes
from batch_util import AUTO, GRAPH, JACOBI, LAUNCH, RESIDENT, XPBD_TYPES, engine, model, replica_state

pytestmark = pytest.mark.gpu

EXTRA = 37  # free particles beyond the cloth's, for a particle set of another size


def flat_adds(types, bodies, params):
    """The add_constraints calls of Engine.add_flat: (type, bodies, params, insertion ids) per type."""
    from positionbaseddynamics_b200 import _capi
    return [(t, bodies[sel][:, :_capi.num_bodies(t)], params[sel][:, :_capi.num_params(t)], sel.astype(np.uint32))
            for t in range(_capi.NUM_TYPES) for sel in [np.nonzero(types == t)[0]] if len(sel)]


def multipliers(eng):
    st = eng.stats()
    return [eng.lambdas(t)[0].copy() for t in XPBD_TYPES if st.constraints_per_type[t]]


def fresh(d, eng):
    """An engine built through the C ABI from the description d (the model as handed in, the batch and its overrides), started from
    eng's particle and rigid-body state and colour groups."""
    from positionbaseddynamics_b200 import _capi
    attrs = (_capi.ATTR_X, _capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX, _capi.ATTR_X0)
    state = {a: eng.get_attr(a).reshape(d["K"], -1, 3) for a in attrs}
    f = _capi.Engine(0)
    f.set_particles(state[_capi.ATTR_X][0], d["mass"][0])
    if d["rb"] is not None:
        s = eng.get_rigid_bodies()
        f.set_rigid_bodies(d["rb"][0], s[:, :3], s[:, 3:7], d["rb"][1], v=s[:, 7:10], omega=s[:, 10:])
    for t, b, p, ids in d["adds"]:
        f.add_constraints(t, b, p, ids=ids)
    f.set_groups(*eng.groups())
    f.set_params(**d["params"])
    f.set_mode(d["mode"])
    f.set_replicas(d["K"])
    f.set_masses(d["mass"])
    for t, rows in d["mats"].items():
        f.set_replica_materials(t, rows)
    if d["gravity"] is not None:
        f.set_replica_gravity(d["gravity"])
    if d["rest"] is not None:
        f.set_replica_rest_positions(d["rest"])
    for a in attrs:
        f.set_attr(a, state[a])
    return f


def segment(d, eng, what, change, planned=None, steps=2):
    """change(eng); planned: None = not checked, False = the multipliers of the last step are kept, True = they are zero.  Then eng and
    a fresh engine in its state step alike."""
    from positionbaseddynamics_b200 import _capi
    before = multipliers(eng)
    change(eng)
    after = multipliers(eng)
    if planned is not None:
        assert before and all(b.any() for b in before), what
        assert all(np.array_equal(b, a) != planned for b, a in zip(before, after)), what
        if planned:
            assert not any(a.any() for a in after), what
    f = fresh(d, eng)
    eng.step(steps); f.step(steps)
    x, y = eng.get_attr(_capi.ATTR_X), f.get_attr(_capi.ATTR_X)
    if d["mode"] == JACOBI:  # float atomics: the order of a particle's corrections differs from run to run
        np.testing.assert_allclose(x, y, rtol=0, atol=1e-5, err_msg=what)
    else:
        assert np.array_equal(x, y), what
    assert eng.get_mode() == f.get_mode(), what
    if d["rb"] is not None:
        assert np.array_equal(eng.get_rigid_bodies(), f.get_rigid_bodies()), what
    f.close()


def test_image_follows_every_model_change():
    from positionbaseddynamics_b200 import _capi
    m = model("femtri_dihedral_cloth")  # a 40 x 40 cloth: FEMTriangle, Dihedral, IsometricBending_XPBD
    eng = engine(m, GRAPH)
    d = dict(mass=m["mass"][None], adds=flat_adds(m["types"], m["bodies"], m["params"]), params=dict(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"]),
             mode=GRAPH, K=1, mats={}, gravity=None, rest=None, rb=None)

    def do(**changes):  # the change to the description, then the calls on the engine
        def change(e, calls=changes.pop("calls")):
            d.update(changes)
            calls(e)
        return change

    segment(d, eng, "first steps", lambda e: None)
    params = dict(d["params"], dt=0.004, vel_method=1)
    segment(d, eng, "set_params", do(params=params, calls=lambda e: e.set_params(**params)), planned=False)
    pinned = m["mass"].copy(); pinned[::5] = 0.0
    segment(d, eng, "set_masses", do(mass=pinned[None], calls=lambda e: e.set_masses(pinned)), planned=False)
    segment(d, eng, "set_attr", do(calls=lambda e: e.set_attr(_capi.ATTR_V, e.get_attr(_capi.ATTR_V) * np.float32(0.5))), planned=False)
    for mode in (LAUNCH, JACOBI, GRAPH):
        segment(d, eng, "set_mode %d" % mode, do(mode=mode, calls=lambda e: e.set_mode(mode)), planned=False)
    segment(d, eng, "set_mode resident", do(mode=RESIDENT, calls=lambda e: e.set_mode(RESIDENT)), planned=True)
    assert eng.get_mode() == (RESIDENT, RESIDENT)

    # a new particle set while the tile-major image is current: the same n, another n, the cloth again
    x, _, mass = replica_state(m, 0)
    free = (np.random.default_rng(7).normal(0.0, 1.0, (EXTRA, 3)) + (0.0, 5.0, 0.0)).astype(np.float32)
    big = np.concatenate([m["x"], free]), np.concatenate([m["mass"], np.ones(EXTRA, np.float32)])
    for what, (px, pm) in (("same n", (x, mass)), ("another n", big), ("the cloth again", (m["x"], m["mass"]))):
        segment(d, eng, "set_particles: " + what, do(mass=pm[None], calls=lambda e: e.set_particles(px, pm)), planned=True)
    segment(d, eng, "set_mode graph", do(mode=GRAPH, calls=lambda e: e.set_mode(GRAPH)), planned=True)
    segment(d, eng, "set_mode auto", do(mode=AUTO, calls=lambda e: e.set_mode(AUTO)), planned=False)
    assert eng.get_mode() == (AUTO, GRAPH)

    # a batch and each of its overrides
    k = 4
    states = [replica_state(m, r) for r in range(k)]

    def batch(e):
        e.set_replicas(k)
        e.set_attr(_capi.ATTR_X, np.stack([s[0] for s in states])); e.set_attr(_capi.ATTR_V, np.stack([s[1] for s in states]))
        e.set_masses(np.stack([s[2] for s in states]))
    segment(d, eng, "set_replicas 4", do(K=k, mass=np.stack([s[2] for s in states]), calls=batch), planned=True)
    stiffness = {4: 100.0}  # IsometricBending_XPBD: the stiffness is its one material parameter
    for what, scale in (("on", lambda r: 0.5 + r), ("rewritten", lambda r: 2.0 - 0.3 * r), ("off", None)):
        rows = {t: None if scale is None else np.array([[s * scale(r)] for r in range(k)], np.float32) for t, s in stiffness.items()}
        segment(d, eng, "set_replica_materials " + what, do(mats={t: r for t, r in rows.items() if r is not None},
                                                            calls=lambda e: [e.set_replica_materials(t, r) for t, r in rows.items()]), planned=False)
    g = np.array([(0.0, -9.81, 0.0), (1.5, -7.0, -2.5), (0.0, 0.0, 0.0), (-1.0, -12.0, 0.5)], np.float32)
    segment(d, eng, "set_replica_gravity on", do(gravity=g, calls=lambda e: e.set_replica_gravity(g)), planned=False)
    segment(d, eng, "set_replica_gravity off", do(gravity=None, calls=lambda e: e.set_replica_gravity(None)), planned=False)

    c = m["x0"].mean(axis=0)
    shapes = {s: np.stack([c + (m["x0"] - c) * np.float32(1.0 + s * (r - 1.5)) for r in range(k)]).astype(np.float32) for s in (0.05, -0.04)}
    tri = m["bodies"][np.nonzero(m["types"] == 5)[0][7]][:3]
    collapsed = shapes[0.05].copy(); collapsed[2][tri] = collapsed[2][tri[0]]  # replica 2: one FEMTriangle collapsed to a point

    def refused(e):
        with pytest.raises(_capi.PbdError, match="degenerate"):
            e.set_replica_rest_positions(collapsed)
    segment(d, eng, "set_replica_rest_positions on", do(rest=shapes[0.05], calls=lambda e: e.set_replica_rest_positions(shapes[0.05])), planned=True)
    segment(d, eng, "set_replica_rest_positions rewritten", do(rest=shapes[-0.04], calls=lambda e: e.set_replica_rest_positions(shapes[-0.04])), planned=False)
    segment(d, eng, "set_replica_rest_positions refused while on", do(calls=refused), planned=False)
    segment(d, eng, "set_replica_rest_positions off", do(rest=None, calls=lambda e: e.set_replica_rest_positions(None)), planned=True)
    segment(d, eng, "set_replica_rest_positions refused while off", do(calls=refused), planned=True)  # the call plans what a derivation reads
    segment(d, eng, "set_replica_rest_positions refused again", do(calls=refused), planned=False)
    segment(d, eng, "set_replicas 1", do(K=1, mass=states[0][2][None], mats={}, gravity=None, calls=lambda e: e.set_replicas(1)), planned=True)

    # the constraints and the colour groups
    pairs = np.array([(i, i + 41) for i in range(0, 39, 3)], dtype=np.uint32)  # Distance_XPBD diagonals of the 40 x 40 grid
    params = np.zeros((len(pairs), _capi.num_params(1)), np.float32)
    params[:, 0] = np.linalg.norm(m["x0"][pairs[:, 0]] - m["x0"][pairs[:, 1]], axis=1)
    params[:, 1] = 1.0e5
    adds = d["adds"] + [(1, pairs, params, None)]

    def replace(e):
        e.clear_constraints()
        for t, b, p, ids in adds:
            e.add_constraints(t, b, p, ids=ids)
    segment(d, eng, "clear_constraints + add_constraints", do(adds=adds, calls=replace), planned=True)
    segment(d, eng, "set_groups", do(calls=lambda e: e.set_groups(*e.groups())), planned=True)
    segment(d, eng, "color_first_fit", do(calls=lambda e: e.color_first_fit()), planned=True)
    segment(d, eng, "color_first_fit_device", do(calls=lambda e: e.color_first_fit_device()), planned=True)

    # mode round trips: AUTO resolves to graph for this model
    for mode, planned in ((GRAPH, False), (AUTO, False), (RESIDENT, True), (AUTO, True), (RESIDENT, True), (GRAPH, True)):
        segment(d, eng, "set_mode %d" % mode, do(mode=mode, calls=lambda e: e.set_mode(mode)), planned=planned)
    eng.close()


def test_image_follows_set_rigid_bodies():
    """A scene with ball joints that fits one cluster, in the resident mode: new rigid-body state with the same body count keeps the
    image (the joint arrays point at the same bodies), another body count plans it again."""
    from positionbaseddynamics_b200 import _capi
    from positionbaseddynamics_b200.model import HostModel
    hm = HostModel()
    scenes.mixed(hm, n_cloth=24, bar_dims=(7, 4, 4), cloth_method=4, bending_method=3)
    scenes.coupling_rig(hm, 24, 24)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x, rb = hm.get("x").copy(), hm.rigid_bodies().copy()
    hm.close()
    assert (types == _capi.BALLJOINT).any() and (types == 1).any()
    rb_mass = np.array([0.0 if i % 3 == 0 else 1.0 for i in range(len(rb))], np.float32)  # scenes.coupling_rig
    inertia = np.array([scenes.box_inertia(1.0, 0.5, 0.5, 0.5) if i % 3 == 0 else scenes.box_inertia(1.0, 0.4, 2.0, 0.4) for i in range(len(rb))], np.float32)
    eng = _capi.Engine(0)
    eng.set_particles(x, mass)
    eng.set_rigid_bodies(rb_mass, rb[:, :3], rb[:, 3:7], inertia)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=0.005, sub_steps=5, max_iter=1)
    eng.set_mode(RESIDENT)
    d = dict(mass=mass[None], adds=flat_adds(types, bodies, params), params=dict(dt=0.005, sub_steps=5, max_iter=1), mode=RESIDENT, K=1,
             mats={}, gravity=None, rest=None, rb=(rb_mass, inertia))

    def bodies_(count):  # the current state of the first `count` bodies, dynamic ones kicked upwards; a new body rests above the rig
        def change(e):
            s = e.get_rigid_bodies()
            while len(s) < count:
                s = np.concatenate([s, [[0.0, 9.0, 0.0, 1.0, 0, 0, 0, 0, 0, 0, 0, 0, 0]]]).astype(np.float32)
            s = s[:count]
            m_ = np.concatenate([rb_mass, np.ones(count - len(rb_mass), np.float32)])[:count]
            i_ = np.concatenate([inertia, np.ones((count - len(inertia), 3), np.float32)])[:count]
            d["rb"] = (m_, i_)
            e.set_rigid_bodies(m_, s[:, :3], s[:, 3:7], i_, v=s[:, 7:10] + (m_[:, None] > 0) * np.float32(0.5), omega=s[:, 10:])
        return change
    segment(d, eng, "first steps", lambda e: None, steps=3)
    assert eng.get_mode() == (RESIDENT, RESIDENT)
    for what, count, planned in (("same count", len(rb), False), ("one more body", len(rb) + 1, True), ("same count", len(rb) + 1, False),
                                 ("the rig again", len(rb), True)):
        segment(d, eng, "set_rigid_bodies: " + what, bodies_(count), planned=planned, steps=3)
    eng.close()


def test_auto_decides_again_after_set_particles(monkeypatch):
    """A cloth of 40,000 particles whose rest positions are scrambled, tiled into 64 independent CTAs: every tile's X items reach more than
    32 others, so the resident mode refuses it and AUTO runs the graph image.  set_particles with the grid's own rest positions gives the
    same constraints a tiling the resident mode takes, and AUTO takes it."""
    from positionbaseddynamics_b200 import _capi
    from positionbaseddynamics_b200.model import HostModel
    monkeypatch.setenv("PBD_B200_CLUSTERS", "64x1")
    hm = HostModel()
    scenes.cloth(hm, 200, 200, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=1, max_iter=4)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x = hm.get("x").copy()
    hm.close()
    assert len(x) >= 40000
    scrambled = x[np.random.default_rng(7).permutation(len(x))]
    eng = _capi.Engine(0)
    eng.set_particles(x, mass, x0=scrambled)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=0.005, sub_steps=1, max_iter=4)
    eng.step(1)
    assert eng.get_mode() == (AUTO, GRAPH)
    d = dict(mass=mass[None], adds=flat_adds(types, bodies, params), params=dict(dt=0.005, sub_steps=1, max_iter=4), mode=AUTO, K=1,
             mats={}, gravity=None, rest=None, rb=None)
    segment(d, eng, "set_particles: the grid's rest positions", lambda e: e.set_particles(x, mass), planned=True)
    assert eng.get_mode() == (AUTO, RESIDENT)
    eng.close()
