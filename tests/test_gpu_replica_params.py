"""Per-replica material parameters and gravity of a batch (pbd_set_replica_materials / pbd_set_replica_gravity): replica r must advance
bit for bit as a single-scene engine whose constraints were added with replica r's row and whose gravity is replica r's vector, in every
mode.  The scenes are the batch scenes of batch_util.py: between them they run all six resident type masks and every type with more than one
material parameter."""
import numpy as np
import pytest

from batch_util import DEFAULT_G, GRAPH, MODES, RESIDENT, SCENES, engine, model, replica_state, results, run, set_state

pytestmark = pytest.mark.gpu

# include/pbd_b200.h: the material columns of every type's parameter layout, and what each is: s = stiffness / modulus, n = Poisson
# ratio, f = flag
MAT = {0: ([1], "s"), 1: ([1], "s"), 2: ([1], "s"), 3: ([0], "s"), 4: ([0], "s"), 5: ([5, 6, 7, 8, 9], "sssnn"), 6: ([4, 5, 6, 7, 8], "sssff"),
       7: ([1], "s"), 8: ([1], "s"), 9: ([10, 11], "sn"), 10: ([10, 11], "sn"), 11: ([9, 10, 11, 12], "ssff"), 12: ([0], "s")}

_solo = {}


def present(m):
    return [t for t in sorted(MAT) if (m["types"] == t).any()]


def material_row(m, t, r, zero=False):
    """Replica r's material parameters of type t, derived from the model's own: stiffnesses and moduli scaled, Poisson ratios moved
    inside [0, 0.49], flags kept; `zero`: a stiffness of exactly 0 where the type has a single stiffness."""
    cols, kinds = MAT[t]
    base = m["params"][np.nonzero(m["types"] == t)[0][0], cols]
    row = base.copy()
    for k, kind in enumerate(kinds):
        if kind == "s":
            row[k] = np.float32(base[k]) * np.float32(0.25 + 1.5 * ((r * 0.6180339887) % 1.0))
        elif kind == "n":
            row[k] = np.float32(0.01 + 0.48 * ((r * 0.3819660113 + 0.1 * k) % 1.0))
    if zero and kinds == "s":
        row[0] = 0.0
    return row.astype(np.float32)


def gravity_row(r):
    return [(0.0, 0.0, 0.0), (1.5 + 0.01 * r, -7.0, -2.5), DEFAULT_G][r % 3]


def with_materials(m, rows):
    """The model with every constraint of type t carrying rows[t]."""
    params = m["params"].copy()
    for t, row in rows.items():
        sel = np.nonzero(m["types"] == t)[0]
        params[np.ix_(sel, MAT[t][0])] = row
    return dict(m, params=params)


def solo(name, r, zero, own_gravity):
    """Replica r stepped by a single-scene engine whose constraints were added with replica r's rows."""
    if (name, r, zero, own_gravity) not in _solo:
        m = model(name)
        g = gravity_row(r) if own_gravity else DEFAULT_G
        ms = with_materials(m, {t: material_row(m, t, r, zero) for t in present(m)})
        eng = engine(ms, GRAPH, gravity=g)
        set_state(eng, [replica_state(m, r)])
        _solo[(name, r, zero, own_gravity)] = run(eng, ms, gravity=g)
        eng.close()
    return _solo[(name, r, zero, own_gravity)]


def check_against_solo(name, k, mode, own_gravity):
    m = model(name)
    eng = engine(m, mode, replicas=k)
    set_state(eng, [replica_state(m, r) for r in range(k)])
    for t in present(m):  # the last replica takes the zero-stiffness branch
        eng.set_replica_materials(t, np.stack([material_row(m, t, r, r == k - 1) for r in range(k)]))
    if own_gravity:
        eng.set_replica_gravity(np.asarray([gravity_row(r) for r in range(k)], np.float32))
    x, v, lam = run(eng, m)
    eng.close()
    assert np.isfinite(x).all()
    for r in sorted({0, 1, k // 2, k - 1}):
        xs, vs, ls = solo(name, r, r == k - 1, own_gravity)
        assert np.array_equal(x[r], xs), (name, k, mode, r)
        assert np.array_equal(v[r], vs), (name, k, mode, r)
        for t, l in ls.items():
            assert np.array_equal(lam[t][r], l), (name, k, mode, r, t)


@MODES
@pytest.mark.parametrize("k", [3, 300])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_replica_materials_equal_solo_runs(name, k, mode):
    """Every replica with its own row for every type present and its own perturbed state equals its solo run (x, v, multipliers)."""
    check_against_solo(name, k, mode, own_gravity=False)


@MODES
@pytest.mark.parametrize("k", [3, 300])
@pytest.mark.parametrize("name", ["xpbd_cloth64", "fem_volume_bar", "femtri_dihedral_cloth"])
def test_replica_gravity_equals_solo_runs(name, k, mode):
    """Per-replica gravity (zero, an off-axis vector, the shared default) on top of per-replica materials and replica 1's pinned masses."""
    check_against_solo(name, k, mode, own_gravity=True)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_override_of_a_type_with_per_constraint_materials(mode):
    """A cloth whose Distance constraints carry two stiffnesses has a per-constraint stiffness array in its image.  An override replaces
    it (replica r = the solo engine with the uniform value); without the override the array counts again."""
    m = model("cfg1")
    params = m["params"].copy()
    dist = np.nonzero(m["types"] == 0)[0]
    params[dist[::2], 1] = 0.6
    two = dict(m, params=params)
    k = 3
    states = [replica_state(m, r) for r in range(k)]
    rows = np.asarray([[0.3], [0.6], [1.0]], np.float32)

    eng = engine(two, mode, replicas=k)
    set_state(eng, states)
    eng.set_replica_materials(0, rows)
    x, v, _ = run(eng, two)
    eng.close()
    for r in range(k):
        one = engine(with_materials(m, {0: rows[r]}), GRAPH)
        set_state(one, [states[r]])
        xs, vs, _ = run(one, m)
        one.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)

    plain = engine(two, mode, replicas=k)
    set_state(plain, states)
    xp, vp, _ = run(plain, two)
    plain.close()
    back = engine(two, mode, replicas=k)
    set_state(back, states)
    back.set_replica_materials(0, rows)
    back.step(1)
    back.set_replica_materials(0, None)
    set_state(back, states)  # (run starts with two first-order steps: oldX and lastX of the step above do not reach its result)
    xb, vb, _ = run(back, two)
    back.close()
    assert not np.array_equal(xp, x)
    assert np.array_equal(xb, xp) and np.array_equal(vb, vp)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_rows_change_between_steps(mode):
    """A row changed between two steps counts from the next step on (in the graph mode without a new capture): the batch then equals
    single-scene engines built with the new values and started from the batch's intermediate state -- x, v, oldX and lastX, because the
    second-order velocity update reads lastX (the multipliers are zeroed at each substep's first sweep)."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k = 3
    attrs = (_capi.ATTR_X, _capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX)
    eng = engine(m, mode, replicas=k)
    eng.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], vel_method=1)
    set_state(eng, [replica_state(m, r) for r in range(k)])
    for t in (1, 4):
        eng.set_replica_materials(t, np.stack([material_row(m, t, r) for r in range(k)]))
    eng.set_replica_gravity(np.asarray([gravity_row(r) for r in range(k)], np.float32))
    eng.step(2); eng.sync()
    mid = {a: eng.get_attr(a).copy() for a in attrs}
    masses = [replica_state(m, r)[2] for r in range(k)]
    new_rows = {t: np.stack([material_row(m, t, r + 10) for r in range(k)]) for t in (1, 4)}
    new_g = np.asarray([gravity_row(r + 1) for r in range(k)], np.float32)
    for t in (1, 4):
        eng.set_replica_materials(t, new_rows[t])
    eng.set_replica_gravity(new_g)
    eng.step(2)
    x, v, lam = results(eng, m)
    eng.close()
    for r in range(k):
        ms = with_materials(m, {t: new_rows[t][r] for t in (1, 4)})
        twin = engine(ms, GRAPH)
        twin.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], vel_method=1, gravity=new_g[r])
        twin.set_masses(masses[r])
        for a in attrs:
            twin.set_attr(a, mid[a][r])
        twin.step(2)
        xs, vs, ls = results(twin, ms)
        twin.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)
        for t, l in ls.items():
            assert np.array_equal(lam[t][r], l), (mode, r, t)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_rows_decide_the_result(mode):
    """Replicas with the same state: different rows end in different positions, equal rows bit-equal."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    for what in ("materials", "gravity"):
        eng = engine(m, mode, replicas=4)
        if what == "materials":
            eng.set_replica_materials(1, np.asarray([[1.0e5], [1.0e3], [1.0e5], [1.0e3]], np.float32))
        else:
            eng.set_replica_gravity(np.asarray([DEFAULT_G, (3.0, -9.81, 0.0), DEFAULT_G, (3.0, -9.81, 0.0)], np.float32))
        eng.step(3); eng.sync()
        x = eng.get_attr(_capi.ATTR_X)
        eng.close()
        assert np.array_equal(x[0], x[2]) and np.array_equal(x[1], x[3]), (mode, what)
        assert not np.array_equal(x[0], x[1]), (mode, what)


def test_rows_outlive_a_new_plan_and_end_with_the_batch_size():
    """Planning the image again (here: another mode) keeps the rows; set_replicas drops them: the batch then runs with the shared
    parameters like a batch that never had any."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k = 3
    rows = np.stack([material_row(m, 1, r) for r in range(k)])
    g = np.asarray([gravity_row(r) for r in range(k)], np.float32)
    eng = engine(m, GRAPH, replicas=k)
    eng.set_replica_materials(1, rows)
    eng.set_replica_gravity(g)
    eng.step(1)
    eng.set_mode(RESIDENT)
    eng.step(1)
    assert eng.get_mode() == (RESIDENT, RESIDENT)
    x, v, lam = results(eng, m)
    for r in range(k):
        ms = with_materials(m, {1: rows[r]})
        one = engine(ms, GRAPH, gravity=g[r])
        one.step(2)
        xs, vs, ls = results(one, ms)
        one.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs) and np.array_equal(lam[1][r], ls[1]), r

    eng.set_replicas(2)  # both replicas: copies of replica 0's state
    eng.step(2)
    x2, v2, _ = results(eng, m)
    eng.close()
    assert np.array_equal(x2[0], x2[1])
    one = engine(m, GRAPH)  # first-order velocity update: x and v are the whole state
    one.set_attr(_capi.ATTR_X, x[0]); one.set_attr(_capi.ATTR_V, v[0])
    one.step(2)
    xs, vs, _ = results(one, m)
    one.close()
    assert np.array_equal(x2[0], xs) and np.array_equal(v2[0], vs)


def test_replica_parameter_refusals():
    """Refused before anything changes: a single-scene engine, a joint type, an unknown type; a wrong shape is caught in Python."""
    from positionbaseddynamics_b200 import _capi
    assert [_capi.num_materials(t) for t in range(15)] == [1, 1, 1, 1, 1, 5, 5, 1, 1, 2, 2, 4, 1, 0, 0]
    assert _capi.num_materials(99) == 0
    m = model("cfg1")
    one = engine(m, GRAPH)
    with pytest.raises(_capi.PbdError, match="single-scene engine"):
        one.set_replica_materials(_capi.DISTANCE, np.ones((1, 1), np.float32))
    with pytest.raises(_capi.PbdError, match="single-scene engine"):
        one.set_replica_gravity(np.zeros((1, 3), np.float32))
    one.close()
    eng = engine(m, GRAPH, replicas=2)
    with pytest.raises(_capi.PbdError, match="no material parameters"):
        eng.set_replica_materials(_capi.BALLJOINT, np.zeros((2, 0), np.float32))
    with pytest.raises(_capi.PbdError, match="unknown constraint type"):
        eng.set_replica_materials(99, None)
    with pytest.raises(ValueError):
        eng.set_replica_materials(_capi.DISTANCE, np.ones((3, 1), np.float32))
    with pytest.raises(ValueError):
        eng.set_replica_materials(_capi.FEMTRIANGLE, np.ones((2, 1), np.float32))
    with pytest.raises(ValueError):
        eng.set_replica_gravity(np.zeros((2, 2), np.float32))
    eng.step(1); eng.sync()
    x = eng.get_attr(_capi.ATTR_X)
    assert np.isfinite(x).all() and np.array_equal(x[0], x[1])  # nothing changed: both replicas still share every parameter
    eng.close()
