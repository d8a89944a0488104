"""Per-replica rest shapes of a batch (pbd_set_replica_rest_positions / pbd_get_replica_geometry): the geometry every replica's constraints
are stepped with is derived on the GPU from that replica's own rest positions, as the host mirror's add*Constraint derives it, and replica r
then advances bit for bit as a single-scene engine whose constraints carry that geometry.  The scenes are the six batch
scenes of batch_util.py (all six resident type masks) and small tet bars with the solid methods those lack (FEMTet_XPBD, StrainTet,
ShapeMatching, Distance_XPBD + Volume_XPBD), so that every particle constraint type is derived."""
import numpy as np
import pytest

import batch_util
import scenes
from batch_util import GRAPH, LAUNCH, MODES, RESIDENT, engine, replica_state, results, run, set_state

pytestmark = pytest.mark.gpu

PARTICLE_TYPES = range(13)
DIHEDRAL = 2
GEO_FIRST = {3: 1, 4: 1, 12: 1}  # the geometry columns start behind the stiffness for these types, at column 0 for the others

SCENES = {**batch_util.SCENES,  # name: (builder, dt, sub_steps, max_iter)
    "femtet_xpbd_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=3, k=1.0e5, sub_steps=2, max_iter=3), 0.005, 2, 3),
    "straintet_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=4, k=1.0, sub_steps=2, max_iter=3), 0.005, 2, 3),
    "shapematching_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=5, k=1.0, sub_steps=2, max_iter=3), 0.005, 2, 3),
    "xpbd_distance_volume_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=6, k=1.0e4, vol_k=1.0e4, sub_steps=2, max_iter=3), 0.005, 2, 3),
}


class _Shaped:
    """The host model mirror with its rest positions and masses replaced by a replica's as soon as its particles exist, so that the scene
    builder's add*Constraint calls derive that replica's geometry."""
    def __init__(self, hm, x0, mass):
        self.hm, self.x0, self.mass = hm, x0, mass

    def __getattr__(self, name):
        return getattr(self.hm, name)

    def _shape(self):
        n = self.hm.num_particles()
        self.hm.set("x0", self.x0[:n])
        for i in range(n):
            self.hm.set_mass(i, float(self.mass[i]))

    def add_regular_triangle_model(self, *a, **k):
        self.hm.add_regular_triangle_model(*a, **k); self._shape()

    def add_regular_tet_model(self, *a, **k):
        self.hm.add_regular_tet_model(*a, **k); self._shape()

    def set_mass(self, i, m):  # the replica's masses stand
        pass


def model(name):
    return batch_util.model(name, SCENES)


def present(m):
    return [t for t in PARTICLE_TYPES if (m["types"] == t).any()]


def geo_cols(t):
    from positionbaseddynamics_b200 import _capi
    g0 = GEO_FIRST.get(t, 0)
    return list(range(g0, g0 + _capi.num_geometry(t)))


def rest_shape(m, r, scale=None):
    """Replica r's rest positions: the model's, rotated, anisotropically scaled in [0.8, 1.25] and moved by 1 % noise (seeded by r);
    `scale`: a uniform scale only."""
    x0 = m["x0"].astype(np.float64)
    c = x0.mean(axis=0)
    if scale is not None:
        return (c + (x0 - c) * scale).astype(np.float32)
    rng = np.random.default_rng(500 + r)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    if (m["types"] == 6).any():  # StrainTriangle takes its rest triangle in the x-z plane: turn the cloth about y only, keeping it there
        q[1] = q[3] = 0.0; q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    s = rng.uniform(0.8, 1.25, 3)
    size = float(np.ptp(x0, axis=0).max())
    edge = size / max(10.0, np.cbrt(len(x0)) * 3.0)
    return (c + ((x0 - c) * s) @ R.T + rng.normal(0.0, 0.01 * edge, x0.shape)).astype(np.float32)


def host_geometry(m, x0, mass):
    """{type: (count, nGeo)} the host mirror's geometry of the model built on these rest positions and masses."""
    from positionbaseddynamics_b200.model import HostModel
    hm = HostModel()
    SCENES[m["name"]][0](_Shaped(hm, x0, mass))
    types, _, params, _ = hm.constraints()
    hm.close()
    assert np.array_equal(np.asarray(types), m["types"]), "the replica's rest shape lost a constraint on the host"
    return {t: np.asarray(params)[np.asarray(types) == t][:, geo_cols(t)].copy() for t in present(m)}


def with_geometry(m, geo):
    """The model with every constraint of type t carrying the geometry rows geo[t]."""
    params = m["params"].copy()
    for t, rows in geo.items():
        sel = np.nonzero(m["types"] == t)[0]
        params[np.ix_(sel, geo_cols(t))] = rows
    return dict(m, params=params)


def ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def assert_geometry_equal(got, want, t, what):
    if t == DIHEDRAL:  # acos: CUDA's double acos is not promised to round like glibc's
        d = ulps(got, want)
        print("%s: Dihedral rest angles differing from the host's: %d of %d (max %d ulp)" % (what, int((d != 0).sum()), d.size, int(d.max(initial=0))))
        assert d.max(initial=0) <= 1, what
    else:
        assert np.array_equal(got, want), (what, t, int((got != want).sum()))


def solo(m, geo_r, state):
    """One replica stepped by a single-scene engine whose constraints carry the replica's read-back geometry."""
    ms = with_geometry(m, geo_r)
    eng = engine(ms, GRAPH)
    set_state(eng, [state])
    out = run(eng, ms)
    eng.close()
    return out


@MODES
@pytest.mark.parametrize("k", [3, 300])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_rest_shapes_equal_host_mirror_and_solo_runs(name, k, mode):
    """Every replica with its own rest shape (and its own state): its geometry equals the host mirror's built on that rest shape, and its
    trajectory (x, v, multipliers) the solo run with that geometry."""
    m = model(name)
    states = [replica_state(m, r) for r in range(k)]
    rest = np.stack([rest_shape(m, r) for r in range(k)])
    eng = engine(m, mode, replicas=k)
    set_state(eng, states)
    eng.set_replica_rest_positions(rest)
    geo = {t: eng.replica_geometry(t) for t in present(m)}
    x, v, lam = run(eng, m)
    eng.close()
    assert np.isfinite(x).all()
    for r in sorted({0, 1, k // 2, k - 1}):
        want = host_geometry(m, rest[r], states[r][2])
        for t in present(m):
            assert_geometry_equal(geo[t][r], want[t], t, "%s K=%d mode=%d replica %d" % (name, k, mode, r))
        xs, vs, ls = solo(m, {t: geo[t][r] for t in present(m)}, states[r])
        assert np.array_equal(x[r], xs), (name, k, mode, r)
        assert np.array_equal(v[r], vs), (name, k, mode, r)
        for t, l in ls.items():
            assert np.array_equal(lam[t][r], l), (name, k, mode, r, t)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
@pytest.mark.parametrize("name", ["cfg1", "fem_volume_bar", "femtri_dihedral_cloth", "shapematching_bar"])
def test_model_rest_positions_are_a_no_op(name, mode):
    """Replicas whose rest positions are the model's own x0 step exactly as a batch without the override -- except with Dihedral
    constraints, whose rest angle may differ by one ulp (acos), so there only the geometry is held to that."""
    m = model(name)
    k = 3
    states = [replica_state(m, r)[:2] + (m["mass"],) for r in range(k)]  # the model's masses: ShapeMatching freezes the inverse masses
    plain = engine(m, mode, replicas=k)
    set_state(plain, states)
    shared = {t: plain.replica_geometry(t) for t in present(m)}
    xp, vp, lp = run(plain, m)
    plain.close()
    eng = engine(m, mode, replicas=k)
    set_state(eng, states)
    eng.set_replica_rest_positions(np.stack([m["x0"]] * k))
    for t in present(m):
        got = eng.replica_geometry(t)
        if t == DIHEDRAL:
            assert_geometry_equal(got, shared[t], t, name)
        else:
            assert np.array_equal(got, shared[t]), (name, t)
    if name == "femtri_dihedral_cloth":
        print("%s: trajectories not compared -- the Dihedral rest angles may differ from the host's by an ulp" % name)
        eng.close()
        return
    x, v, lam = run(eng, m)
    eng.close()
    assert np.array_equal(x, xp) and np.array_equal(v, vp), name
    for t in lam:
        assert np.array_equal(lam[t], lp[t]), (name, t)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT, LAUNCH], ids=["graph", "resident", "launch"])
def test_switching_on_off_and_new_positions_between_steps(mode):
    """NULL restores the shared geometry bit for bit; new positions between two steps count from the next step on: the batch then equals
    solo engines with the new geometry started from the batch's intermediate state."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k = 3
    states = [replica_state(m, r) for r in range(k)]
    plain = engine(m, mode, replicas=k); set_state(plain, states)
    xp, vp, lp = run(plain, m); plain.close()
    back = engine(m, mode, replicas=k); set_state(back, states)
    back.set_replica_rest_positions(np.stack([rest_shape(m, r) for r in range(k)]))
    back.step(1)
    back.set_replica_rest_positions(None)
    set_state(back, states)
    xb, vb, lb = run(back, m); back.close()
    assert np.array_equal(xb, xp) and np.array_equal(vb, vp) and all(np.array_equal(lb[t], lp[t]) for t in lp)

    attrs = (_capi.ATTR_X, _capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX)
    eng = engine(m, mode, replicas=k)
    eng.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], vel_method=1)
    set_state(eng, states)
    eng.set_replica_rest_positions(np.stack([rest_shape(m, r) for r in range(k)]))
    eng.step(2); eng.sync()
    mid = {a: eng.get_attr(a).copy() for a in attrs}
    eng.set_replica_rest_positions(np.stack([rest_shape(m, r + 10) for r in range(k)]))
    geo = {t: eng.replica_geometry(t) for t in present(m)}
    assert np.array_equal(eng.get_attr(_capi.ATTR_X0), np.stack([rest_shape(m, r + 10) for r in range(k)]))
    eng.step(2)
    x, v, lam = results(eng, m)
    eng.close()
    for r in range(k):
        ms = with_geometry(m, {t: geo[t][r] for t in present(m)})
        twin = engine(ms, GRAPH)
        twin.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], vel_method=1)
        twin.set_masses(states[r][2])
        for a in attrs:
            twin.set_attr(a, mid[a][r])
        twin.step(2)
        xs, vs, ls = results(twin, ms)
        twin.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)
        for t, l in ls.items():
            assert np.array_equal(lam[t][r], l), (mode, r, t)


def test_a_new_plan_keeps_the_rest_shapes():
    """A mode switch and an added constraint mid-simulation re-plan the image; its geometry is derived again from the kept rest positions
    (the added constraint's too), and every replica stays equal to its solo engine."""
    m = model("fem_volume_bar")
    k = 3
    states = [replica_state(m, r) for r in range(k)]
    rest = np.stack([rest_shape(m, r) for r in range(k)])
    eng = engine(m, GRAPH, replicas=k)
    set_state(eng, states)
    eng.set_replica_rest_positions(rest)
    eng.step(1)
    eng.set_mode(RESIDENT)
    eng.step(1)
    extra = np.array([[0, len(m["x"]) - 1]], np.uint32)
    eng.add_constraints(0, extra, np.array([[1.0, 0.5]], np.float32))
    eng.set_groups(np.array([0] + [int(o) for o in m["off"][1:]] + [len(m["types"]) + 1], np.uint32), np.append(m["ids"], len(m["types"])).astype(np.uint32))
    eng.step(1)
    geo = {t: eng.replica_geometry(t) for t in present(m) + ([0] if 0 not in present(m) else [])}
    x, v, _ = results(eng, m)
    eng.close()
    m2 = dict(m, types=np.append(m["types"], 0), bodies=np.vstack([m["bodies"], np.array([[0, len(m["x"]) - 1, 0, 0]], np.uint32)]),
              params=np.vstack([m["params"], np.pad(np.array([[0.0, 0.5]], np.float32), ((0, 0), (0, m["params"].shape[1] - 2)))]))
    for r in range(k):
        d = [float(rest[r][len(m["x"]) - 1][c]) - float(rest[r][0][c]) for c in range(3)]
        assert geo[0][r][-1, 0] == np.float32(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])), r
        ms = with_geometry(m2, {t: geo[t][r] for t in geo})
        one = _solo_engine(ms, m, states[r])
        one.step(2)
        one.add_constraints(0, extra, ms["params"][-1:, :2])
        one.set_groups(np.array([0] + [int(o) for o in m["off"][1:]] + [len(m["types"]) + 1], np.uint32), np.append(m["ids"], len(m["types"])).astype(np.uint32))
        one.step(1)
        xs, vs, _ = results(one, m)
        one.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), r


def _solo_engine(ms, m, state):
    """A single-scene engine of the model's constraints (without the ones appended to `ms`) carrying ms's geometry."""
    n0 = len(m["types"])
    mm = dict(m, params=ms["params"][:n0])
    eng = engine(mm, GRAPH)
    set_state(eng, [state])
    return eng


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_rest_shapes_compose_with_materials_and_gravity(mode):
    """Per-replica rest shapes, material rows and gravity together: replica r = the solo engine with all three of its own."""
    m = model("strain_cloth")
    k = 4
    states = [replica_state(m, r) for r in range(k)]
    rest = np.stack([rest_shape(m, r) for r in range(k)])
    mats = {6: np.stack([np.array([1.0 + r, 1.0 + 0.5 * r, 1.0, 0.0, 1.0], np.float32) for r in range(k)]), 4: np.array([[50.0 * (r + 1)] for r in range(k)], np.float32)}
    grav = np.array([[0.0, -9.81 + r, 0.5 * r] for r in range(k)], np.float32)
    eng = engine(m, mode, replicas=k)
    set_state(eng, states)
    for t, rows in mats.items():
        eng.set_replica_materials(t, rows)
    eng.set_replica_gravity(grav)
    eng.set_replica_rest_positions(rest)
    geo = {t: eng.replica_geometry(t) for t in present(m)}
    x, v, lam = run(eng, m)
    eng.close()
    cols = {6: [4, 5, 6, 7, 8], 4: [0]}
    for r in range(k):
        ms = with_geometry(m, {t: geo[t][r] for t in present(m)})
        for t, rows in mats.items():
            sel = np.nonzero(ms["types"] == t)[0]
            ms["params"][np.ix_(sel, cols[t])] = rows[r]
        one = engine(ms, GRAPH, gravity=grav[r])
        set_state(one, [states[r]])
        one.step(2)
        one.set_params(dt=m["dt"], sub_steps=m["sub"] + 1, max_iter=m["it"] + 1, vel_method=1, gravity=grav[r])
        from positionbaseddynamics_b200 import _capi
        one.step(2)
        one.set_attr(_capi.ATTR_V, one.get_attr(_capi.ATTR_V) * np.float32(0.5))
        one.step(1)
        xs, vs, ls = results(one, ms)
        one.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)
        for t, l in ls.items():
            assert np.array_equal(lam[t][r], l), (mode, r, t)


def test_refusals_leave_the_state_unchanged():
    """Refused before anything changes: a single-scene engine, a collapsed triangle or a flat tet in one replica (the message names the
    replica and the constraint); steps after a refused call equal those of an engine that never saw it.  pbd_set_replicas and
    pbd_set_particles drop the override."""
    from positionbaseddynamics_b200 import _capi
    m = model("femtri_dihedral_cloth")
    one = engine(m, GRAPH)
    with pytest.raises(_capi.PbdError, match="single-scene engine"):
        one.set_replica_rest_positions(m["x0"][None])
    one.close()
    k = 3
    states = [replica_state(m, r) for r in range(k)]
    rest = np.stack([rest_shape(m, r) for r in range(k)])
    tri = m["bodies"][np.nonzero(m["types"] == 5)[0][7]][:3]
    bad = rest.copy()
    bad[2][tri] = bad[2][tri[0]]  # replica 2: one triangle collapsed to a point
    eng = engine(m, GRAPH, replicas=k)
    set_state(eng, states)
    eng.set_replica_rest_positions(rest)
    eng.step(1)
    with pytest.raises(_capi.PbdError, match="replica 2 .*constraint [0-9]+"):
        eng.set_replica_rest_positions(bad)
    ref = engine(m, GRAPH, replicas=k)
    set_state(ref, states)
    ref.set_replica_rest_positions(rest)
    ref.step(1)
    for e in (eng, ref):
        e.step(2)
    xa, va, _ = results(eng, m); xb, vb, _ = results(ref, m)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb)
    assert np.array_equal(eng.get_attr(_capi.ATTR_X0), rest)
    eng.set_replicas(2)  # the override ends with the batch size
    ref.close()
    shared = m["params"][m["types"] == 5][:, :5]
    assert np.array_equal(eng.replica_geometry(5)[0], shared) and np.array_equal(eng.replica_geometry(5)[1], shared)
    eng.set_replica_rest_positions(np.stack([rest_shape(m, r) for r in range(2)]))
    assert not np.array_equal(eng.replica_geometry(5)[1], shared)
    eng.set_particles(m["x"], m["mass"], x0=m["x0"])  # ... and with set_particles
    assert np.array_equal(eng.replica_geometry(5)[1], shared)
    eng.close()

    bar = model("fem_volume_bar")
    tet = bar["bodies"][np.nonzero(bar["types"] == 9)[0][3]]
    flat = np.stack([rest_shape(bar, r) for r in range(2)])
    flat[1][tet[3]] = flat[1][tet[0]] + 0.5 * (flat[1][tet[1]] - flat[1][tet[0]])  # replica 1: one tet flattened onto an edge
    eng = engine(bar, GRAPH, replicas=2)
    with pytest.raises(_capi.PbdError, match="replica 1 .*constraint [0-9]+"):
        eng.set_replica_rest_positions(flat)
    assert np.array_equal(eng.replica_geometry(9)[1], bar["params"][bar["types"] == 9][:, :10])
    eng.close()


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_rest_shapes_decide_the_result(mode):
    """Negative control: rest shapes scaled by 1.3 move the batch far from the shared-geometry batch, which proves that the projections
    read the per-replica arrays.  Sanity: under a uniform scale s the rest lengths are s x the model's and the volumes s^3 x."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_distance_volume_bar")
    k = 3
    plain = engine(m, mode, replicas=k)
    plain.step(5); plain.sync()
    xp = plain.get_attr(_capi.ATTR_X).copy(); plain.close()
    eng = engine(m, mode, replicas=k)
    eng.set_replica_rest_positions(np.stack([rest_shape(m, 0, scale=s) for s in (1.3, 1.3, 0.9)]))
    lengths, volumes = eng.replica_geometry(1), eng.replica_geometry(8)
    eng.step(5); eng.sync()
    x = eng.get_attr(_capi.ATTR_X)
    eng.close()
    assert np.array_equal(x[0], x[1])
    assert np.abs(x[0] - xp[0]).max() > 1e-2 and np.abs(x[2] - xp[2]).max() > 1e-3
    base_l = m["params"][m["types"] == 1][:, 0].astype(np.float64)
    base_v = m["params"][m["types"] == 8][:, 0].astype(np.float64)
    for r, s in enumerate((1.3, 1.3, 0.9)):
        np.testing.assert_allclose(lengths[r][:, 0], s * base_l, rtol=1e-5)
        np.testing.assert_allclose(volumes[r][:, 0], s ** 3 * base_v, rtol=3e-5)


def test_a_degenerate_added_constraint_is_refused_at_add_time():
    """With per-replica rest shapes on, a constraint that some replica's kept rest shape makes degenerate is refused by
    pbd_add_constraints itself (the next steps still run, as if it had never been offered); a sound one is taken."""
    from positionbaseddynamics_b200 import _capi
    m = model("fem_volume_bar")
    k = 3
    states = [replica_state(m, r) for r in range(k)]
    rest = np.stack([rest_shape(m, r) for r in range(k)])
    tet = m["bodies"][np.nonzero(m["types"] == 9)[0][0]].copy()
    eng = engine(m, GRAPH, replicas=k)
    ref = engine(m, GRAPH, replicas=k)
    for e in (eng, ref):
        set_state(e, states)
        e.set_replica_rest_positions(rest)
        e.step(1)
    flat = np.array([[tet[0], tet[1], tet[2], tet[0]]], np.uint32)  # two bodies the same particle: singular in every replica
    with pytest.raises(_capi.PbdError, match="pbd_add_constraints: .*replica 0 .*constraint %d" % len(m["types"])):
        eng.add_constraints(9, flat, np.array([[0.0] * 10 + [1.0e5, 0.3]], np.float32))
    for e in (eng, ref):
        e.step(2)
    xa, va, _ = results(eng, m); xb, vb, _ = results(ref, m)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb)
    eng.add_constraints(7, tet[None], np.array([[0.0, 1.0]], np.float32))  # a sound Volume constraint is taken
    assert eng.replica_geometry(7).shape[1] == int((m["types"] == 7).sum()) + 1
    eng.close(); ref.close()
