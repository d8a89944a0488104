"""Replica batches with rigid bodies and ball joints (pbd_set_replica_rigid_bodies): replica r advances bit for bit like a single-scene engine
given replica r's bodies through pbd_set_rigid_bodies, in every mode -- particle x and v, the XPBD multipliers, body x, q, v and omega --
alone and with per-replica gravity, materials, rest shapes and colliders; the device-memory body calls and the lifetime of the bodies."""
import numpy as np
import pytest

import rigid_batch_util as rb
from batch_util import AUTO, GRAPH, LAUNCH, MODES, RESIDENT

pytestmark = pytest.mark.gpu


def solo_run(m, mode, r, k, gravity=rb.DEFAULT_G, extra=None):
    eng = rb.engine(m, mode, bodies=rb.replica_bodies(m, r), gravity=gravity)
    rb.set_particles(eng, [rb.particle_state(m, r)])
    if extra:
        extra(eng, r)
    out = rb.run(eng, m, gravity=gravity)
    eng.close()
    return out


def batch_run(m, mode, k, gravity=rb.DEFAULT_G, extra=None):
    eng = rb.engine(m, mode, replicas=k, bodies=[rb.replica_bodies(m, r) for r in range(k)], gravity=gravity)
    rb.set_particles(eng, [rb.particle_state(m, r) for r in range(k)])
    if extra:
        extra(eng, None)
    out = rb.run(eng, m, gravity=gravity)
    active = eng.get_mode()[1]
    eng.close()
    return out, active


@pytest.mark.parametrize("name", ["rig", "rigid_cases", "strain_rig"])
@pytest.mark.parametrize("k", [2, 3, 300])
@MODES
def test_replica_equals_solo(name, k, mode):
    m = rb.model(name)
    out, active = batch_run(m, mode, k)
    if mode != AUTO:
        assert active == mode
    for r in rb.sampled(k):
        rb.same(out, solo_run(m, mode, r, k), r, (name, k, mode))


def test_free_bodies_beyond_the_block_under_auto():
    """700 free bodies beside an XPBD cloth, K = 32 under AUTO: the resident batch on the solid instantiation, more bodies than threads."""
    m = rb.free_body_cloth()
    k = 32
    out, active = batch_run(m, AUTO, k)
    assert active == RESIDENT
    for r in rb.sampled(k):
        rb.same(out, solo_run(m, RESIDENT, r, k), r)


def test_replica_gravity_moves_the_bodies():
    m = rb.model("rig")
    k = 3
    g = np.array([(0.0, -9.81, 0.0), (2.0, -4.0, 1.0), (0.0, -20.0, -3.0)], np.float32)
    for mode in (GRAPH, RESIDENT):
        out, _ = batch_run(m, mode, k, extra=lambda e, r: e.set_replica_gravity(g))
        for r in range(k):
            rb.same(out, solo_run(m, mode, r, k, gravity=tuple(g[r])), r, mode)
        plain, _ = batch_run(m, mode, k)
        for r in (1, 2):  # the rows moved these replicas' bodies off where the shared gravity takes them
            assert not np.array_equal(out[3][r][:, :3], plain[3][r][:, :3]), (mode, r)


def test_replica_materials_and_rest_shapes_beside_joints():
    """Per-replica material rows and rest shapes on the particle constraints of the rig: replica r equals a single-scene engine whose
    constraints were added with replica r's material values and with the geometry the batch derived from replica r's rest positions
    (read back through replica_geometry), and whose x0 are those rest positions."""
    from positionbaseddynamics_b200 import _capi
    from test_gpu_replica_params import MAT, with_materials
    from test_gpu_replica_rest_shape import with_geometry
    m = rb.model("rig")
    k = 3
    types = sorted({int(t) for t in np.unique(m["types"])} - {_capi.BALLJOINT, _capi.RB_PARTICLE_BALLJOINT})
    t = types[0]
    rows = (np.arange(1, k + 1, dtype=np.float32)[:, None] * np.float32(0.3) * m["params"][np.nonzero(m["types"] == t)[0][0], MAT[t][0]][None]).astype(np.float32)
    c = m["x0"].mean(axis=0)
    rest = np.stack([c + (m["x0"] - c) * np.float32(s) for s in (1.0, 0.97, 1.03)]).astype(np.float32)
    for mode in (GRAPH, LAUNCH, RESIDENT):
        eng = rb.engine(m, mode, replicas=k, bodies=[rb.replica_bodies(m, r) for r in range(k)])
        rb.set_particles(eng, [rb.particle_state(m, r) for r in range(k)])
        eng.set_replica_materials(t, rows)
        eng.set_replica_rest_positions(rest)
        geo = {tt: eng.replica_geometry(tt) for tt in types}
        out = rb.run(eng, m)
        eng.close()
        for r in range(k):
            ms = with_geometry(with_materials(m, {t: rows[r]}), {tt: geo[tt][r] for tt in types})
            solo = rb.engine(dict(ms, x0=rest[r]), mode, bodies=rb.replica_bodies(m, r))
            rb.set_particles(solo, [rb.particle_state(m, r)])
            rb.same(out, rb.run(solo, ms), r, mode)
            solo.close()


def test_replica_colliders_beside_joint_bodies():
    """pbd_set_replica_colliders' static bodies and the joint bodies in one batch: replica r equals a solo engine given the joint bodies
    followed by the collider bodies (rc.body offset to match) and the colliders through set_colliders."""
    from positionbaseddynamics_b200 import _capi
    m = rb.model("rig")
    k = 3
    n = len(m["x"])
    nb = len(m["bm"])
    floor = [(0.0, -0.2 - 0.1 * r, 0.0) for r in range(k)]

    def collider(body):
        c = _capi.RigidCollider()
        c.shape, c.body = _capi.SHAPE_BOX, body
        c.dim[:] = (20.0, 0.2, 20.0)
        c.thickness, c.restitution, c.friction = 0.0, 0.5, 0.1
        c.R[:] = (1, 0, 0, 0, 1, 0, 0, 0, 1)
        c.aabb_min[:] = (-25.0, -2.0, -25.0); c.aabb_max[:] = (25.0, 2.0, 25.0)
        return c
    ranges = [_capi.ParticleCollider(0, n, 0.5, 0.1)]

    def batch_extra(e, _):
        e.set_replica_colliders(ranges, [[collider(0)] for _ in range(k)], body_x=np.array(floor, np.float32).reshape(k, 1, 3))
    for mode in (GRAPH, RESIDENT):
        out, _ = batch_run(m, mode, k, extra=batch_extra)
        for r in range(k):
            mass, x, q, inertia, v, w = rb.replica_bodies(m, r)
            bodies = (np.append(mass, 0.0).astype(np.float32), np.vstack([x, floor[r]]).astype(np.float32), np.vstack([q, (1, 0, 0, 0)]).astype(np.float32),
                      np.vstack([inertia, (1, 1, 1)]).astype(np.float32), np.vstack([v, (0, 0, 0)]).astype(np.float32), np.vstack([w, (0, 0, 0)]).astype(np.float32))
            eng = rb.engine(m, mode, bodies=bodies)
            rb.set_particles(eng, [rb.particle_state(m, r)])
            eng.set_colliders(ranges, [collider(nb)])
            sx, sv, sl, sb = rb.run(eng, m)
            eng.close()
            rb.same(out, (sx, sv, sl, sb[:nb]), r, mode)


def test_set_replicas_copies_replica0_bodies_and_keeps_joints():
    from positionbaseddynamics_b200 import _capi
    m = rb.model("rig")
    eng = rb.engine(m, GRAPH, replicas=3, bodies=[rb.replica_bodies(m, r) for r in range(3)])
    eng.step(1)
    b0 = eng.get_rigid_bodies()[0].copy()
    eng.set_replicas(5)
    got = eng.get_rigid_bodies()
    assert got.shape == (5, len(m["bm"]), 13)
    assert all(np.array_equal(got[r], b0) for r in range(5))
    eng.step(2)
    got = eng.get_rigid_bodies()
    assert all(np.array_equal(got[r], got[0]) for r in range(5))
    assert all(np.array_equal(x, eng.get_attr(_capi.ATTR_X)[0]) for x in eng.get_attr(_capi.ATTR_X))
    eng.close()
    # the old refusals hold
    one = rb.engine(m, GRAPH, bodies=rb.replica_bodies(m, 0))
    with pytest.raises(_capi.PbdError, match="rigid bodies"):
        one.set_replicas(2)
    with pytest.raises(_capi.PbdError, match="pbd_set_replicas first"):
        one.set_replica_rigid_bodies(*[a[None] for a in rb.replica_bodies(m, 0)])
    one.close()
    two = rb.engine(m, GRAPH, replicas=2, bodies=[rb.replica_bodies(m, r) for r in range(2)])
    with pytest.raises(_capi.PbdError, match="rigid bodies"):
        two.set_rigid_bodies(*rb.replica_bodies(m, 0))
    with pytest.raises(_capi.PbdError, match="PBD_MODE_JACOBI"):
        two.set_mode(3)
    two.step(1); two.sync()
    two.close()
