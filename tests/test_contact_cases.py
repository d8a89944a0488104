"""The contact path's case set and fp64 restatement (tests/contact_cases.py) on the CPU: every branch the restatement tags is taken in
every configuration, the restatement is the C restatement's contact step to 1e-12 and the unmodified reference's (where oracle/_ref
is present) to 1e-9, and the contact kernel compiled for the host
(tests/host_shim/run_contacts.cpp, run_contact_sensors.cpp) is within the gate of the fp64 answer on every case.  The GPU gate is
tests/test_gpu_contact_answers.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import contact_cases as cc
import contact_util as cu
from test_contacts_host_shim import _RC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_layouts = None


def layouts():
    global _layouts
    if _layouts is None:
        _layouts = cc.make_layouts()
    return _layouts


@pytest.mark.parametrize("config", cc.CONFIGS, ids=["tol%g_k%g_it%d_sub%d" % c for c in cc.CONFIGS])
def test_every_branch_is_taken(config):
    tags = {}
    for L in layouts():
        cc.run_reference(L, L.x, L.v, config, tags=tags)
    need = set(cc.BRANCHES_DETECT)
    if config[2] > 0:
        need |= set(cc.BRANCHES_SOLVE)
    if config[2] < 2:  # a contact's impulse turns negative only in a later sweep
        need.discard("friction_lo")
    assert need <= set(tags), sorted(need - set(tags))


def test_case_set_covers_every_class():
    classes = set()
    for L in layouts():
        classes |= set(L.cls.tolist())
        assert len(L.x) == cc.N and cc.N % 128 and cc.N > 4 * 128
        assert len(L.cols) == 8
    assert set(cc.DETECTION + cc.SOLVE + cc.STRUCTURE + cc.THRESHOLD) == classes
    keys = set()
    for L in layouts():
        keys |= set(zip(L.shape.tolist(), L.cls.tolist()))
    assert set(cc.TOL) == {k for k in keys if k[1] not in cc.THRESHOLD}  # every gated (shape, class) has its measured threshold
    S, I, M = layouts()
    assert {c["invert"] for c in S.cols[:6]} == {False} and {c["invert"] for c in I.cols[:6]} == {True}
    assert S.cols[6]["body"] == S.cols[7]["body"]


def _rows(cols):
    return [[c["shape"], c["body"], *c["dim"], c["thickness"], float(c["invert"]), c["restitution"], c["friction"], *c["R"], *c["v1"], *c["v2"],
             *c["aabb_min"], *c["aabb_max"]] for c in cols]


@pytest.mark.parametrize("config", cc.CONFIGS, ids=["tol%g_k%g_it%d_sub%d" % c for c in cc.CONFIGS])
def test_restatement_is_the_c_restatements_contact_step(config, cpu_libs):
    """The C restatement (fp64) steps every layout once: colliders from set_colliders, bodies with set_rigid_body_velocity.  reference()
    applied to its own state after the substeps (v_pre = (x - oldX) / h) gives its post-step velocities to 1e-12 of max(|v|, 1 m/s)."""
    tol, stiff, iters, sub = config
    worst = 0.0
    for L in layouts():
        m = cpu_libs.CpuPbd("oracle", "f64")
        m.add_triangle_model(L.x_pre.astype(np.float64), np.zeros((0, 3), np.uint32))
        for i, mass in enumerate(L.mass):
            m.set_mass(i, float(mass))
        m.set("v", L.v)
        for b in range(len(L.bx)):
            m.add_rigid_body(0.0, L.bx[b], (1.0, 1.0, 1.0))
            m.set_rigid_body_velocity(b, L.bv[b], L.bw[b])
        m.set_colliders(cc.RANGES, _rows(L.cols))
        m.set_oracle_contact_params(float(np.float32(tol)), float(np.float32(stiff)), iters)
        m.set_params(dt=cc.DT, sub_steps=sub, max_iter=1, vel_method=0, gravity=(0.0, 0.0, 0.0))
        m.step(1)
        h = cc.DT / sub
        x, old = m.get("x"), m.get("oldX")
        v_pre = (x - old) * (1.0 / h)
        v_pre[L.mass == 0] = L.v[L.mass == 0]  # the velocity update skips static particles
        mass, w = m.masses()
        v, rec, _, _ = cc.reference(x, v_pre, w, mass, cc.RANGES, L.cols, (L.bx, L.bv, L.bw), float(np.float32(tol)), float(np.float32(stiff)), iters)
        want = m.get("v")
        fin = np.isfinite(want).all(1)
        assert np.array_equal(fin, np.isfinite(v).all(1)), L.name
        worst = max(worst, float((np.abs(v[fin] - want[fin]).max(1) / np.maximum(np.abs(want[fin]).max(1), 1.0)).max()))
        p, b, _ = m.oracle_contacts()
        assert sorted(zip(p.tolist(), b.tolist())) == sorted((int(r["particle"]), L.cols[r["collider"]]["body"]) for r in rec), L.name
    print("restatement vs the C restatement (%s): worst relative |dv| %.1e" % (config, worst))
    assert worst <= 1e-12


def _ref_collider_dict(row):
    """A collision_objects() row (the pbd_rigid_collider layout, 30 doubles) as a contact_util collider dict."""
    d = [float(v) for v in row]
    return dict(shape=int(d[0]), body=int(d[1]), dim=d[2:5], thickness=d[5], invert=d[6] != 0.0, restitution=d[7], friction=d[8], R=d[9:18],
                v1=d[18:21], v2=d[21:24], aabb_min=d[24:27], aabb_max=d[27:30])


@pytest.mark.parametrize("config", [(0.05, 100.0, 5, 1), (0.05, 0.0, 20, 2)], ids=["tol0.05_k100_it5_sub1", "tol0.05_k0_it20_sub2"])
def test_restatement_is_the_references_contact_step(config, cpu_libs):
    """The unmodified reference (oracle/_ref, fp64) steps once: seven particle models registered as collision objects, each with its own
    restitution and friction, some particles static, against inverted and upright colliders of every shape on static bodies that move
    and spin, in rotated frames.  reference(), given the colliders as collision_objects() reports them, the bodies after the step and
    v_pre = (x - oldX) / h of the reference's own state, gives its contact list and post-step velocities to 1e-9 of max(|v|, 1 m/s)."""
    from conftest import have_ref
    import scenes
    if not have_ref("f64"):
        pytest.skip("prebuilt oracle/_ref/libpbdref_f64.so not present")
    tol, stiff, iters, sub = config
    rng = np.random.default_rng(77)
    ref = cpu_libs.CpuPbd("ref", "f64")
    shapes = [(0, (1.0, 0.6, 0.8)), (1, (0.9,)), (2, (0.8, 0.3)), (3, (0.6, 1.0)), (4, (0.9,)), (5, (1.0, 0.7, 0.9))]
    cols = []
    for j, (shape, dims) in enumerate(shapes * 2):
        invert = j >= len(shapes)
        centre = np.array([4.0 * (j % len(shapes)) - 10.0, 6.0 * invert, 0.0])
        rot = cu.rotation(rng.normal(size=3), rng.uniform(0.2, 1.2))
        half = cu.half_extents(shape, list(dims) + [0.0] * (3 - len(dims)), 0.15)
        cols.append((centre, rot, half, shape, dims, invert))
    # The reference tests a particle model's bounding-sphere leaves against a collider's box and then every particle of a touching leaf,
    # so a particle outside an inverted collider's box may still get a contact there, depending on how the hierarchy grouped it; the
    # kernel tests each particle against the box.  Each inverted collider therefore gets a model of its own, inside its box.
    groups = [np.concatenate([c[0] + rng.uniform(-1.2, 1.2, (60, 3)) * (np.abs(c[1]) @ c[2]) for c in cols if not c[5]])]
    groups += [c[0] + rng.uniform(-0.9, 0.9, (40, 3)) * (np.abs(c[1]) @ c[2]) for c in cols if c[5]]
    pts = np.concatenate(groups)
    n = len(pts)
    vel = rng.normal(0.0, 1.0, (n, 3))
    for g in groups:  # one particle model per group, each its own collision object with its own coefficients
        ref.add_triangle_model(g, np.zeros((0, 3), np.uint32))
    mass = rng.uniform(0.2, 3.0, n); mass[::9] = 0.0
    for i in range(n):
        ref.set_mass(i, float(mass[i]))
    ref.set("v", vel)
    ref.set_params(dt=cc.DT, sub_steps=sub, max_iter=1, vel_method=0, gravity=(0.0, 0.0, 0.0))
    ref.use_distance_field_cd(tol)
    for j, (centre, rot, half, shape, dims, invert) in enumerate(cols):
        b, _ = ref.add_rigid_body_mesh(1.0, scenes.BOX_VERTS, scenes.BOX_FACES, x=centre, R=rot, scale=2.0 * half)
        ref.set_rigid_body_mass(b, 0.0)
        ref.set_rigid_body_velocity(b, rng.normal(0.0, 0.4, 3), rng.normal(0.0, 0.8, 3))
        ref.add_rigid_collider(b, shape, dims, thickness=0.15, invert=invert, restitution=rng.uniform(0.2, 0.9), friction=rng.uniform(0.05, 0.4))
    for k in range(len(groups)):
        ref.add_model_collider(0, k, restitution=rng.uniform(0.2, 0.9), friction=rng.uniform(0.05, 0.4))
    ref.set_contact_params(stiffness=stiff, max_iter_v=iters)
    ref.step(1)
    models, rigid = ref.collision_objects()
    assert len(models) == len(groups) and len(rigid) == len(cols) and sum(r[6] != 0 for r in rigid) == len(shapes)
    x, old = ref.get("x"), ref.get("oldX")
    v_pre = (x - old) * (1.0 / (cc.DT / sub))
    m, w = ref.masses()
    v_pre[m == 0] = vel[m == 0]  # the velocity update skips static particles
    rb = ref.rigid_bodies()
    assert np.abs(rb[:, 7:13]).max() > 0  # the static bodies move and spin
    v, rec, _, _ = cc.reference(x, v_pre, w, m, models, [_ref_collider_dict(r) for r in rigid], (rb[:, :3], rb[:, 7:10], rb[:, 10:13]), tol, stiff, iters)
    p, b, _, _, _ = ref.contacts()
    assert sorted(zip(p.tolist(), b.tolist())) == sorted((int(q["particle"]), int(rigid[q["collider"]][1])) for q in rec)
    assert len(rec) > 200 and len({int(rigid[q["collider"]][1]) for q in rec}) == len(cols) and (m[rec["particle"]] == 0).any()
    want = ref.get("v")
    worst = float((np.abs(v - want).max(1) / np.maximum(np.abs(want).max(1), 1.0)).max())
    print("restatement vs the reference (%s): %d contacts, worst relative |dv| %.1e" % (config, len(rec), worst))
    assert worst <= 1e-9


# ---------------------------------------------------------------------------------------------------------------------------------
# the contact kernel on the host
# ---------------------------------------------------------------------------------------------------------------------------------
def _shim(tmp_path, name):
    so = str(tmp_path / ("lib%s.so" % name))
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "tests", "host_shim"), "-I" + os.path.join(ROOT, "positionbaseddynamics_b200", "csrc"),
                           "-o", so, os.path.join(ROOT, "tests", "host_shim", name + ".cpp")])
    return C.CDLL(so)


def kernel_inputs(L, x, v, bodies_per_collider=False):
    """pos / vel float4 rows, body rows and kernel colliders of layout L.  bodies_per_collider: collider k on body k (the batch layout)."""
    from positionbaseddynamics_b200 import _capi
    n = len(x)
    pos = np.zeros((n, 4), np.float32); pos[:, :3] = x; pos[:, 3] = cc.inv_mass(L.mass)
    vel = np.zeros((n, 4), np.float32); vel[:, :3] = v; vel[:, 3] = L.mass
    idx = [c["body"] for c in L.cols] if bodies_per_collider else list(range(len(L.bx)))
    body = lambda a: np.concatenate([np.asarray(a, np.float32)[idx], np.zeros((len(idx), 1), np.float32)], 1).copy()
    rcs = (_RC * len(L.cols))()
    for k, c in enumerate(L.cols):
        rc = rcs[k]; rc.shape = c["shape"]; rc.body = k if bodies_per_collider else c["body"]; rc.dim[:] = c["dim"]; rc.thickness = c["thickness"]
        rc.invert = -1.0 if c["invert"] else 1.0; rc.restitution = c["restitution"]; rc.friction = c["friction"]; rc.R[:] = c["R"]
        rc.v1[:] = c["v1"]; rc.v2[:] = c["v2"]; rc.aabbMin[:] = c["aabb_min"]; rc.aabbMax[:] = c["aabb_max"]
    pcs = (_capi.ParticleCollider * len(cc.RANGES))(*[_capi.ParticleCollider(*r) for r in cc.RANGES])
    return pos, vel, body(L.bx), body(L.bv), body(L.bw), rcs, pcs


class ContactSense(C.Structure):  # pbdk::ContactSense
    _fields_ = [("count", C.c_uint * 8), ("p", C.c_float * 24)]


def test_host_kernel_within_the_gate(tmp_path):
    """run_contacts (k_contacts) and run_contact_sensors (the sensing instantiation, one replica per layout) on every layout and
    configuration: the velocity gate (contact_cases.velocity_gate), the contact set exactly, the sensors' counts exactly and their
    impulses within TOL_SENSORS of the fp64 sum (contact_cases.sensor_errors, as on the GPU); the sensing run moves the particles bit
    for bit as the plain one.  The gate fails against each mutated restatement (contact_cases.MUTATIONS)."""
    from positionbaseddynamics_b200 import _capi
    lib, sense = _shim(tmp_path, "run_contacts"), _shim(tmp_path, "run_contact_sensors")
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    worst, results = {}, {}
    for config in cc.CONFIGS:
        tol, stiff, iters, _ = config
        for L in layouts():
            pos, vel, bX, bV, bW, rcs, pcs = kernel_inputs(L, L.x, L.v)
            rec = (_capi.Contact * 8192)(); cnt = C.c_uint(0)
            lib.run_contacts(cc.N, vp(pos), vp(vel), vp(bX), vp(bV), vp(bW), 8, C.cast(rcs, C.c_void_p), len(cc.RANGES), C.cast(pcs, C.c_void_p),
                             C.c_float(tol), C.c_float(stiff), iters, C.cast(rec, C.c_void_p), C.byref(cnt), 8192)
            v_ref, rref, count, impulse = cc.run_reference(L, L.x, L.v, config)
            got = vel[:, :3]
            results[(L.name, config)] = got.copy()
            for key, err, limit in cc.velocity_gate(L, got, L.x, L.v, config):
                worst[key] = max(worst.get(key, 0.0), err)
                assert err <= limit, (config, L.name, key, err, limit)
            g = cc.gated(L)
            mine = sorted((rec[i].particle, rec[i].body) for i in range(cnt.value) if g[rec[i].particle])
            assert mine == sorted((int(r["particle"]), L.cols[r["collider"]]["body"]) for r in rref if g[r["particle"]]), (config, L.name)
            # the sensing instantiation: the same bits; the sensors, also with the degenerate normals made static (every impulse finite)
            for M in (L, cc.without_degenerate(L)):
                pos2, vel2, bX, bV, bW, rcs, pcs = kernel_inputs(M, M.x, M.v, bodies_per_collider=True)
                s = (ContactSense * cc.N)(); c2 = C.c_uint(0)
                slot = np.arange(cc.N, dtype=np.uint32)
                sense.run_contact_sensors(1, cc.N, vp(slot), vp(pos2), vp(vel2), vp(bX), vp(bV), vp(bW), 8, C.cast(rcs, C.c_void_p), len(cc.RANGES),
                                          C.cast(pcs, C.c_void_p), C.c_float(tol), C.c_float(stiff), iters, None, C.byref(c2), 0, C.cast(s, C.c_void_p))
                if M is L:
                    assert np.array_equal(vel2.view(np.uint32), vel.view(np.uint32)), (config, L.name)
                _, _, count, impulse = cc.run_reference(M, M.x, M.v, config)
                sc = np.array([list(s[i].count) for i in range(cc.N)]).sum(0)
                sp = -np.array([list(s[i].p) for i in range(cc.N)], np.float64).reshape(cc.N, 8, 3).sum(0)
                same_count, same_fin, err = cc.sensor_errors(sc, sp, count, impulse)
                assert same_count and same_fin and err <= cc.TOL_SENSORS, (config, L.name, M is L, sc, count, err)
                if M is not L:
                    assert np.isfinite(impulse).all()
                worst[("sensors", L.name)] = max(worst.get(("sensors", L.name), 0.0), err)
    print("HOST-MEASURED %r" % worst)
    # negative controls: the same gate fails against each mutated restatement
    caught = {mut: sum(not err <= limit for L in layouts() for config in cc.CONFIGS
                       for _, err, limit in cc.velocity_gate(L, results[(L.name, config)], L.x, L.v, config, mut=mut)) for mut in cc.MUTATIONS}
    print("negative controls, (shape, class) outside the gate: %s" % caught)
    assert all(caught.values()), caught
