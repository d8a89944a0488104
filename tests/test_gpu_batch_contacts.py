"""Contacts of a replica batch (pbd_set_replica_colliders): every replica against its own static colliders, one launch of
k_contacts_batch per step.  Replica r must advance bit for bit as a single-scene engine given its bodies (pbd_set_rigid_bodies, masses 0)
and its colliders (pbd_set_colliders, collider k on body k), and record the same contacts with the particle index shifted by r n."""
import ctypes as C
import numpy as np
import pytest

import contact_util as cu
import scenes
from batch_util import AUTO, GRAPH, LAUNCH, MODES, RESIDENT, model, replica_state, set_state

pytestmark = pytest.mark.gpu

SCENES = {  # name: (builder, dt, sub_steps, max_iter)
    "contact_cloth24": (lambda m: (m.add_regular_triangle_model(24, 24, t=(-2.5, 2.2, -2.5), R=scenes.RX90, scale=(5.0, 5.0)),
                                   m.add_cloth_constraints(0, 4, dist_k=1.0e5), m.add_bending_constraints(0, 3, 100.0)), 0.005, 1, 4),
    "contact_bar": (lambda m: (m.add_regular_tet_model(9, 4, 4, t=(0.0, 2.0, 0.0), R=np.eye(3), scale=(3.0, 0.6, 0.6)),
                               m.add_solid_constraints(0, 2, k=1.0e5, nu=0.3)), 0.005, 2, 3),
}
PC = {"contact_cloth24": (0.5, 0.1), "contact_bar": (0.4, 0.3)}  # the model's restitution and friction
STEPS = 120
CAP = 1 << 20
REC = np.dtype([("particle", "<u4"), ("body", "<u4"), ("cp0", "<f4", 3), ("cp1", "<f4", 3), ("n", "<f4", 3), ("dist", "<f4")])


def _model(name):
    return model(name, SCENES)


def _pc(m, name):
    from positionbaseddynamics_b200 import _capi
    return [_capi.ParticleCollider(0, len(m["x"]), *PC[name])]


def contacts(eng):
    """The last step's contact records, sorted by (particle, body)."""
    from positionbaseddynamics_b200 import _capi
    buf = np.zeros(CAP, REC); cnt = C.c_uint(0)
    _capi._ck(_capi.lib().pbd_get_contacts(eng._h, buf.ctypes.data_as(C.c_void_p), CAP, C.byref(cnt)))
    assert cnt.value <= CAP
    return buf[:cnt.value].copy()


def batch_engine(m, name, mode, k, scene):
    from batch_util import engine
    eng = engine(m, mode, replicas=k)
    set_state(eng, [replica_state(m, r) for r in range(k)])
    cols, bx, bv, bw = scene
    eng.set_replica_colliders(_pc(m, name), [[cu.to_capi(d) for d in c] for c in cols], bx, bv, bw)
    eng.set_contact_params(tolerance=cu.TOL, stiffness=100.0, max_iter_v=5)
    eng.record_contacts(CAP)
    return eng


def solo_engine(m, name, r, cols, bx, bv, bw, gravity=None, params=None):
    """Replica r as a single-scene engine: its bodies as static rigid bodies (set before the groups, which cover them), collider k on body k."""
    from positionbaseddynamics_b200 import _capi
    eng = _capi.Engine(0)
    eng.set_particles(m["x"], m["mass"], x0=m["x0"])
    set_solo_bodies(eng, bx, bv, bw)
    eng.add_flat(m["types"], m["bodies"], m["params"] if params is None else params)
    eng.set_groups(m["off"], m["ids"])
    eng.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], gravity=(0.0, -9.81, 0.0) if gravity is None else gravity)
    eng.set_mode(GRAPH)
    set_state(eng, [replica_state(m, r)])
    eng.set_colliders(_pc(m, name), [cu.to_capi(dict(d, body=j)) for j, d in enumerate(cols)])
    eng.set_contact_params(tolerance=cu.TOL, stiffness=100.0, max_iter_v=5)
    eng.record_contacts(CAP)
    return eng


def set_solo_bodies(eng, bx, bv, bw):
    nr = len(bx)
    eng.set_rigid_bodies([0.0] * nr, bx, [(1.0, 0.0, 0.0, 0.0)] * nr, [(1.0, 1.0, 1.0)] * nr, v=bv, omega=bw)


def final(eng):
    from positionbaseddynamics_b200 import _capi
    eng.sync()
    return eng.get_attr(_capi.ATTR_X).copy(), eng.get_attr(_capi.ATTR_V).copy()


_solo = {}


def solo_run(name, r, empty):
    """(x, v, per-step contact lists) of replica r's solo run over STEPS steps."""
    key = (name, r, empty)
    if key not in _solo:
        m = _model(name)
        cols, bx, bv, bw = cu.replica_scene(r, cu.footprint(m["x"]), empty)
        eng = solo_engine(m, name, r, cols, bx, bv, bw)
        lists = []
        for _ in range(STEPS):
            eng.step(1)
            lists.append(contacts(eng))
        _solo[key] = final(eng) + (lists,)
        eng.close()
    return _solo[key]


def compared(k):
    return sorted({0, 1, k // 2, k - 1} & set(range(k)))


@MODES
@pytest.mark.parametrize("k", [2, 3, 300])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_batch_contacts_equal_solo_runs(name, k, mode):
    """Replicas {0, 1, k/2, k-1} of a batch with per-replica colliders equal their solo runs bit for bit after STEPS steps (x, v), and
    record the solo contact lists at every step.  The colliders cover every shape, inverted distance fields, rotated frames, differing
    coefficients and moving body surfaces; the last replica (k >= 3) has only empty boxes.  300 replicas are more than the resident mode
    runs at once."""
    from positionbaseddynamics_b200 import _capi
    m = _model(name)
    n = len(m["x"])
    scene = cu.batch_scene(k, cu.footprint(m["x"]))
    empty = k - 1 if k >= 3 else -1
    eng = batch_engine(m, name, mode, k, scene)
    launches0 = eng.stats().kernel_launches
    eng.step(1); eng.sync()
    launches1 = eng.stats().kernel_launches - launches0
    lists = [contacts(eng)]
    for _ in range(STEPS - 1):
        eng.step(1)
        lists.append(contacts(eng))
    x, v = final(eng)
    eng.close()
    x, v = x.reshape(k, n, 3), v.reshape(k, n, 3)
    events = np.zeros(k, np.int64)
    for l in lists:
        assert np.all(np.diff(l["particle"].astype(np.int64)) >= 0)  # replica-major
        events += np.bincount(l["particle"] // n, minlength=k)
    print("%s K=%d mode %d: contact events per compared replica %s, %d in all; %d launches in the first step" % (
        name, k, mode, {r: int(events[r]) for r in compared(k)}, int(events.sum()), launches1))
    for r in compared(k):
        xs, vs, ls = solo_run(name, r, r == empty)
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (name, k, mode, r)
        for s, (l, want) in enumerate(zip(lists, ls)):
            mine = l[l["particle"] // n == r].copy()
            mine["particle"] -= r * n
            assert np.array_equal(mine.view(np.uint8), want.view(np.uint8)), (name, k, mode, r, s)
        assert events[r] == 0 if r == empty else events[r] >= 100, (r, events[r])
    assert np.isfinite(x).all()


def _moved(k, m, t):
    """Per-replica body moves at time t: each replica's obstacles slide along their own direction."""
    d = np.stack([np.array([np.cos(1.3 * r), 0.3, np.sin(1.3 * r)]) for r in range(k)])
    return 0.02 * t * d


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_moving_obstacles_between_steps(mode):
    """set_replica_colliders between steps, with step and with step_host_async + step_host_wait(1): the same as solo engines that call
    set_rigid_bodies + set_colliders at the same points."""
    from positionbaseddynamics_b200 import _capi
    name, k = "contact_cloth24", 3
    m = _model(name)
    n = len(m["x"])
    fp = cu.footprint(m["x"])
    eng = batch_engine(m, name, mode, k, cu.batch_scene(k, fp, empty=-1))
    xo = [np.empty((k, n, 3), np.float32) for _ in range(2)]; vo = [np.empty((k, n, 3), np.float32) for _ in range(2)]
    for t in range(1, 61):
        if t % 5 == 0:
            cols, bx, bv, bw = cu.batch_scene(k, fp, empty=-1, shift=_moved(k, m, t))
            eng.set_replica_colliders(_pc(m, name), [[cu.to_capi(d) for d in c] for c in cols], bx, bv, bw)
        if t <= 30:
            eng.step(1)
        else:
            eng.step_host_async(1, None, None, xo[t & 1], vo[t & 1])
            eng.step_host_wait(1)
    eng.step_host_wait(0)
    x, v = final(eng)
    assert np.array_equal(x, xo[0]) and np.array_equal(v, vo[0])  # the last call's output
    eng.close()
    for r in range(k):
        cols, bx, bv, bw = cu.replica_scene(r, fp)
        one = solo_engine(m, name, r, cols, bx, bv, bw)
        for t in range(1, 61):
            if t % 5 == 0:
                cols, bx, bv, bw = cu.replica_scene(r, fp, shift=_moved(k, m, t)[r])
                set_solo_bodies(one, bx, bv, bw)
                one.set_colliders(_pc(m, name), [cu.to_capi(dict(d, body=j)) for j, d in enumerate(cols)])
            one.step(1)
        xs, vs = final(one)
        one.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_colliders_with_gravity_materials_and_rest_shapes(mode):
    """Per-replica gravity, material rows and rest shapes together with per-replica colliders: replica r = the solo engine with all of
    its own."""
    from positionbaseddynamics_b200 import _capi
    name, k = "contact_cloth24", 3
    m = _model(name)
    n = len(m["x"])
    fp = cu.footprint(m["x"])
    scene = cu.batch_scene(k, fp)
    c = m["x0"].mean(axis=0)
    rest = np.stack([(c + (m["x0"] - c) * np.float32(0.92 + 0.06 * r)).astype(np.float32) for r in range(k)])
    mats = {_capi.DISTANCE_XPBD: np.array([[1.0e4 * (r + 1)] for r in range(k)], np.float32), _capi.ISOBENDING_XPBD: np.array([[40.0 * (r + 1)] for r in range(k)], np.float32)}
    mat_col = {_capi.DISTANCE_XPBD: 1, _capi.ISOBENDING_XPBD: 0}
    geo_first = {_capi.DISTANCE_XPBD: 0, _capi.ISOBENDING_XPBD: 1}
    grav = np.array([[0.3 * r, -9.81 + r, -0.2 * r] for r in range(k)], np.float32)
    eng = batch_engine(m, name, mode, k, scene)
    for t, rows in mats.items():
        eng.set_replica_materials(t, rows)
    eng.set_replica_gravity(grav)
    eng.set_replica_rest_positions(rest)
    geo = {t: eng.replica_geometry(t) for t in mats}
    eng.step(80)
    x, v = final(eng)
    eng.close()
    for r in range(k):
        params = m["params"].copy()
        for t in mats:
            sel = np.nonzero(m["types"] == t)[0]
            params[np.ix_(sel, list(range(geo_first[t], geo_first[t] + _capi.num_geometry(t))))] = geo[t][r]
            params[sel, mat_col[t]] = mats[t][r, 0]
        cols, bx, bv, bw = cu.replica_scene(r, fp, r == k - 1)
        one = solo_engine(m, name, r, cols, bx, bv, bw, gravity=grav[r], params=params)
        one.step(80)
        xs, vs = final(one)
        one.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)


def test_negative_controls():
    """Each of these changes the compared replicas: swapping the collider lists of replicas 1 and 2, zeroing one replica's body omega, a
    batch without colliders."""
    name, k = "contact_cloth24", 4
    m = _model(name)
    n = len(m["x"])
    fp = cu.footprint(m["x"])
    scene = cu.batch_scene(k, fp, empty=-1)

    def run(sc):
        eng = batch_engine(m, name, GRAPH, k, sc) if sc is not None else None
        if eng is None:
            from batch_util import engine
            eng = engine(m, GRAPH, replicas=k)
            set_state(eng, [replica_state(m, r) for r in range(k)])
        eng.step(STEPS)
        x, v = final(eng)
        eng.close()
        return x, v

    base = run(scene)
    cols, bx, bv, bw = scene
    swapped = ([cols[0], cols[2], cols[1], cols[3]], bx[[0, 2, 1, 3]], bv[[0, 2, 1, 3]], bw[[0, 2, 1, 3]])
    bw0 = bw.copy(); bw0[1] = 0.0
    for what, sc, rs in (("swapped colliders of replicas 1 and 2", swapped, (1, 2)), ("omega of replica 1 zeroed", (cols, bx, bv, bw0), (1,)),
                         ("no colliders", None, (0, 1, 2, 3))):
        x, v = run(sc)
        for r in rs:
            dx = float(np.abs(x[r] - base[0][r]).max()); dv = float(np.abs(v[r] - base[1][r]).max())
            print("%s: replica %d moves by up to %.3e m, %.3e m/s" % (what, r, dx, dv))
            assert dx > 1e-4, (what, r)
        if sc is not None and what.startswith("omega"):
            for r in (0, 2, 3):
                assert np.array_equal(x[r], base[0][r]), (what, r)


def test_refusals_keep_the_previous_colliders():
    """K = 1, more than 8 rigid colliders, an unknown shape, a particle range beyond n and body_x = None are refused, and the next step
    still equals the solo runs; set_replicas drops the colliders; wrong shapes raise ValueError."""
    from positionbaseddynamics_b200 import _capi
    name, k = "contact_cloth24", 3
    m = _model(name)
    n = len(m["x"])
    fp = cu.footprint(m["x"])
    scene = cu.batch_scene(k, fp)
    cols, bx, bv, bw = scene
    eng = batch_engine(m, name, GRAPH, k, scene)
    caps = lambda c: [[cu.to_capi(d) for d in l] for l in c]
    nine = [l + [cu.empty_box()] * 5 for l in cols]
    bx9 = np.concatenate([bx, np.zeros((k, 5, 3), np.float32)], axis=1)
    bad_shape = [list(l) for l in cols]; bad_shape[1] = [dict(bad_shape[1][0], shape=7)] + bad_shape[1][1:]
    for match, args in (("9 rigid colliders", (_pc(m, name), caps(nine), bx9)),
                        ("unknown shape 7", (_pc(m, name), caps(bad_shape), bx, bv, bw)),
                        ("covers", ([_capi.ParticleCollider(10, n, 0.5, 0.1)], caps(cols), bx, bv, bw)),
                        ("body_x == NULL", (_pc(m, name), caps(cols), None, bv, bw))):
        with pytest.raises(_capi.PbdError, match=match):
            eng.set_replica_colliders(*args)
    with pytest.raises(ValueError):
        eng.set_replica_colliders(_pc(m, name), caps(cols)[:2], bx[:2])
    with pytest.raises(ValueError):
        eng.set_replica_colliders(_pc(m, name), caps(cols), bx[:, :2])
    eng.step(STEPS)
    x, v = final(eng)
    for r in range(k):
        xs, vs, _ = solo_run(name, r, r == k - 1)
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), r
    # set_replicas drops them: the next steps equal a batch that never had colliders
    eng.set_replicas(2)
    set_state(eng, [replica_state(m, r) for r in range(2)])
    eng.step(STEPS)
    xa, va = final(eng)
    eng.close()
    from batch_util import engine
    plain = engine(m, GRAPH, replicas=2)
    set_state(plain, [replica_state(m, r) for r in range(2)])
    plain.step(STEPS)
    xb, vb = final(plain)
    plain.close()
    assert np.array_equal(xa, xb) and np.array_equal(va, vb)
    one = engine(m, GRAPH)
    with pytest.raises(_capi.PbdError, match="single-scene"):
        one.set_replica_colliders(_pc(m, name), [[cu.to_capi(d) for d in cols[0]]], bx[:1], bv[:1], bw[:1])
    one.close()


def test_example_runs():
    """examples/cloth_collision_batch.py with a small K: every cloth ends above its own obstacle."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "examples", "cloth_collision_batch.py"), "--replicas", "4", "--steps", "200"],
                         capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stderr
    assert "every cloth above its obstacle: yes" in out.stdout
