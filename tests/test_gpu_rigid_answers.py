"""Rigid bodies and both ball joints against the fp64 restatement, through the engine's execution paths.

Cases and the fp64 restatement of the rigid parts of a substep are in tests/rigid_cases.py.  The CPU test pins the restatement to the
checker's own time step.  The GPU tests give the engine what the checker built -- constraint rows, colour groups and body state -- and run

  launch        MODE_LAUNCH, every configuration of projection_cases.CONFIGS
  graph         MODE_GRAPH, the same configurations
  resident1x1   MODE_RESIDENT, one CTA: the joints in its colour phases, the bodies stepped by CTA 0
  resident1x4   MODE_RESIDENT, one cluster of four CTAs on rest positions in a random order, so that a body's particle joints run in
                CTAs 1-3 (the tile of the particle) while its BallJoints run in tile 0

and compare body x, q, v, omega and the particles' x, v with the restatement; every path must be bit-identical to MODE_LAUNCH.  Error
measures, per case: positions and velocities (times h) relative to max(|correction|, 1e-3) plus 16 fp32 ulps of |x|; the rotation as
the angle between the two quaternions relative to max(angle moved, 1e-3); omega relative to max(|omega|, 1e-3).  Each run prints the
worst error per (kind, class, path).  Negative controls: the gate must fail against the restatement without the gyroscopic term, with
the world inertia built as R^T D R, with omega from conj(q_old) q, without the particle's inverse mass in K, and with a first-order
linear velocity update of the bodies under velocity method 1.

Three tests hold the resident kernel to the other modes on more bodies than it has shared-memory threads:
test_resident_steps_every_body_in_one_cluster (700 bodies in particle joints, one cluster), test_auto_resident_steps_free_bodies_beyond_the_block
(700 free bodies beside a cloth big enough for MODE_AUTO to choose the resident mode: one cluster of 16 CTAs) and
test_independent_ctas_step_free_bodies_beyond_the_block (the same scene as independent CTAs, where CTA 0 also runs X threads).
"""
import os

import numpy as np
import pytest

import projection_cases as pc
import rigid_cases as rc

PER_CLASS = 10
STEPS = 2
# (kind, class): (position / velocity threshold, worst measured, rotation threshold, worst measured, omega threshold, worst measured)
# over every path and configuration; measured on an H100 80GB HBM3 at its 700 W power limit, thresholds 3x the measured worst (two
# significant digits, rounded up; an exact zero stays zero).
TOL = {
    ('BallJoint', 'both_static'): (0, 0.00e+00, 0, 0.00e+00, 0, 0.00e+00),
    ('BallJoint', 'large'): (4.5e-06, 1.47e-06, 3e-05, 9.77e-06, 6e-05, 1.99e-05),
    ('BallJoint', 'lever0'): (2.7e-05, 8.70e-06, 0.00067, 2.20e-04, 0.0011, 3.39e-04),
    ('BallJoint', 'lever10'): (2.5e-05, 8.03e-06, 7.7e-05, 2.54e-05, 0.00013, 4.10e-05),
    ('BallJoint', 'ratio1e3'): (4.8e-05, 1.59e-05, 0.0003, 9.89e-05, 0.00075, 2.49e-04),
    ('BallJoint', 'rotated'): (2.1e-05, 6.84e-06, 0.00026, 8.62e-05, 0.00031, 1.03e-04),
    ('BallJoint', 'shift1e2'): (0.0028, 9.20e-04, 0.0068, 2.25e-03, 0.0081, 2.67e-03),
    ('BallJoint', 'shift1e3'): (0.016, 5.23e-03, 0.034, 1.11e-02, 0.062, 2.06e-02),
    ('BallJoint', 'small'): (0.00085, 2.83e-04, 0.0013, 4.19e-04, 0.0029, 9.47e-04),
    ('BallJoint', 'spinning'): (2.5e-05, 8.14e-06, 3.1e-05, 1.03e-05, 9.5e-05, 3.16e-05),
    ('BallJoint', 'static0'): (8.5e-05, 2.81e-05, 0.00019, 6.26e-05, 0.00029, 9.39e-05),
    ('BallJoint', 'static1'): (0.00028, 9.04e-05, 6.1e-05, 2.02e-05, 7.5e-05, 2.48e-05),
    ('RigidBodyParticleBallJoint', 'both_static'): (0, 0.00e+00, 0, 0.00e+00, 0, 0.00e+00),
    ('RigidBodyParticleBallJoint', 'large'): (2.2e-06, 7.24e-07, 8.7e-06, 2.89e-06, 1.2e-05, 3.79e-06),
    ('RigidBodyParticleBallJoint', 'lever0'): (5.3e-05, 1.75e-05, 0.00077, 2.55e-04, 0.0046, 1.53e-03),
    ('RigidBodyParticleBallJoint', 'lever10'): (4e-05, 1.32e-05, 3.2e-05, 1.05e-05, 0.00019, 6.04e-05),
    ('RigidBodyParticleBallJoint', 'ratio1e3'): (5.5e-05, 1.81e-05, 4.6e-05, 1.51e-05, 8.4e-05, 2.78e-05),
    ('RigidBodyParticleBallJoint', 'rotated'): (3.9e-05, 1.28e-05, 5.5e-05, 1.81e-05, 0.0001, 3.31e-05),
    ('RigidBodyParticleBallJoint', 'shift1e2'): (0.0032, 1.06e-03, 0.0015, 4.82e-04, 0.0022, 7.31e-04),
    ('RigidBodyParticleBallJoint', 'shift1e3'): (0.028, 9.05e-03, 0.016, 5.17e-03, 0.024, 7.71e-03),
    ('RigidBodyParticleBallJoint', 'small'): (0.00057, 1.88e-04, 0.00043, 1.41e-04, 0.00075, 2.49e-04),
    ('RigidBodyParticleBallJoint', 'spinning'): (2.7e-05, 8.76e-06, 3.4e-05, 1.11e-05, 5.1e-05, 1.69e-05),
    ('RigidBodyParticleBallJoint', 'static_body'): (0.00041, 1.34e-04, 0, 0.00e+00, 0, 0.00e+00),
    ('RigidBodyParticleBallJoint', 'static_particle'): (4.3e-05, 1.42e-05, 2.5e-05, 8.05e-06, 6.7e-05, 2.21e-05),
    ('chain', 'chain'): (0.00018, 5.98e-05, 0.012, 3.90e-03, 0.0044, 1.44e-03),
    ('free', 'free'): (0.0008, 2.66e-04, 3.2e-05, 1.04e-05, 7.1e-05, 2.35e-05),
}

# the fp64 gate of the two tests with more bodies than a block has threads: one bound for all three measures, the largest threshold
# of TOL outside the translated classes, on other seeds
REGRESSION_TOL = 0.012

_model = None


def model():
    global _model
    if _model is None:
        _model = rc.make_model(PER_CLASS, 4242)
    return _model


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU: the restatement
# ---------------------------------------------------------------------------------------------------------------------------------
def _rel(a, b):
    """Largest difference of x, q, v, omega (bodies) or x, v (particles) relative to the largest magnitude of the quantity (at least 1)."""
    return max(np.abs(a[:, k] - b[:, k]).max() / max(np.abs(b[:, k]).max(), 1.0) for k in (slice(0, 3), slice(3, 7), slice(7, 10), slice(10, 13)))


@pytest.mark.parametrize("config", pc.CONFIGS, ids=["%dx%d_v%d" % c for c in pc.CONFIGS])
def test_restatement_is_the_checkers_time_step(config):
    """The numpy restatement against the checker's own TimeStepController step on the whole case set, two steps: the same bodies and
    particles to 1e-9 of each quantity's scale."""
    m = model()
    ck = rc.load(m, rc.checker())
    ck.set_params(dt=rc.DT, sub_steps=config[0], max_iter=config[1], vel_method=config[2], gravity=rc.GRAVITY)
    ck.step(STEPS)
    px, pv, rb = rc.reference(m, *config, steps=STEPS)
    e_rb = _rel(ck.rigid_bodies(), rb)
    e_p = max(np.abs(ck.get("x") - px).max() / np.abs(px).max(), np.abs(ck.get("v") - pv).max() / np.abs(pv).max())
    print("restatement vs the checker's step (%s): bodies %.1e, particles %.1e" % (rc.checker().kind, e_rb, e_p))
    assert e_rb <= 1e-9 and e_p <= 1e-9


def test_case_set_covers_every_class():
    m = model()
    for kind in rc.KINDS:
        for cls in rc.CLASSES[kind]:
            assert ((m.kind == kind) & (m.cls == cls)).sum() == PER_CLASS, (kind, cls)
    assert set(np.unique(m.types)) == {rc.BJ, rc.RBP}
    chain = np.nonzero(m.kind == "chain")[0]
    per_body = np.bincount(m.bodies[np.isin(m.jcase, chain)][:, 0], minlength=m.nb) + \
        np.bincount(m.bodies[np.isin(m.jcase, chain) & (m.types == rc.BJ)][:, 1], minlength=m.nb)
    assert per_body.max() == 4  # one body in four joints, each in a colour of its own
    assert m.nb < 512  # the block size of the resident kernel's solid mask: test_resident_steps_every_body_in_one_cluster goes beyond it


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
def engine(m, mode, x0=None, particles=None):
    """m's bodies and joints in an engine; particles: (x, masses, constraints) of a particle model that takes the place of m's particles."""
    from positionbaseddynamics_b200 import _capi
    eng = _capi.Engine(0)
    if particles is None:
        eng.set_particles(m.px, m.pm, x0=x0)
        types, bodies, params, off, ids = m.types, m.bodies, m.params, m.off, m.ids
    else:
        x, mass, (types, bodies, params, off, ids) = particles
        eng.set_particles(x, mass)
    eng.set_rigid_bodies(m.bm, m.bx, m.bq, m.bI, v=m.bv, omega=m.bw)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_mode(mode)
    return eng


def run(eng, m, config, steps=STEPS, particles=None):
    """`steps` steps of config from m's initial state: particles (x, v) and bodies (n, 13)."""
    from positionbaseddynamics_b200 import _capi
    sub, it, vel = config
    x, v = (m.px, m.pv) if particles is None else particles
    for a, val in ((_capi.ATTR_X, x), (_capi.ATTR_V, v), (_capi.ATTR_OLDX, x), (_capi.ATTR_LASTX, x)):
        eng.set_attr(a, np.asarray(val, np.float32))
    eng.set_rigid_bodies(m.bm, m.bx, m.bq, m.bI, v=m.bv, omega=m.bw)
    eng.set_params(dt=rc.DT, sub_steps=sub, max_iter=it, vel_method=vel, gravity=rc.GRAVITY)
    eng.step(steps); eng.sync()
    return (eng.get_attr(_capi.ATTR_X).astype(np.float64), eng.get_attr(_capi.ATTR_V).astype(np.float64),
            eng.get_rigid_bodies().astype(np.float64))


def _qangle(a, b):
    """Angle between rotations a and b (rows (w, x, y, z))."""
    w = np.abs((a * b).sum(1))
    p = a[:, :1] * b[:, 1:] - b[:, :1] * a[:, 1:] + np.cross(a[:, 1:], b[:, 1:])
    return 2.0 * np.arctan2(np.linalg.norm(p, axis=1), w)


def errors(m, got, ref, config):
    """Per case: (position / velocity, rotation, omega) errors."""
    h = rc.DT / config[0]
    px, pv, rb = got
    rpx, rpv, rrb = ref
    nc = len(m.cases)
    moved, ulp = np.zeros(nc), np.zeros(nc)
    np.maximum.at(moved, m.pcase, np.abs(rpx - m.px).max(1))
    np.maximum.at(moved, m.bcase, np.abs(rrb[:, :3] - m.bx).max(1))
    f32 = float(np.spacing(np.float32(1.0)))
    np.maximum.at(ulp, m.pcase, f32 * np.abs(rpx).max(1))
    np.maximum.at(ulp, m.bcase, f32 * np.abs(rrb[:, :3]).max(1))
    sc = np.maximum(moved, 1e-3) + 16.0 * ulp
    e_pos, e_rot, e_om = np.zeros(nc), np.zeros(nc), np.zeros(nc)
    np.maximum.at(e_pos, m.pcase, np.maximum(np.abs(px - rpx).max(1), np.abs(pv - rpv).max(1) * h) / sc[m.pcase])
    np.maximum.at(e_pos, m.bcase, np.maximum(np.abs(rb[:, :3] - rrb[:, :3]).max(1), np.abs(rb[:, 7:10] - rrb[:, 7:10]).max(1) * h) / sc[m.bcase])
    np.maximum.at(e_rot, m.bcase, _qangle(rb[:, 3:7], rrb[:, 3:7]) / np.maximum(_qangle(m.bq, rrb[:, 3:7]), 1e-3))
    np.maximum.at(e_om, m.bcase, np.linalg.norm(rb[:, 10:] - rrb[:, 10:], axis=1) / np.maximum(np.linalg.norm(rrb[:, 10:], axis=1), 1e-3))
    bad = ~(np.isfinite(e_pos) & np.isfinite(e_rot) & np.isfinite(e_om))
    return [np.where(bad, np.inf, e) for e in (e_pos, e_rot, e_om)]


def over(m, errs):
    """Indices of the cases outside the gate."""
    tol = np.array([TOL[(k, c)] for k, c in zip(m.kind, m.cls)]).reshape(len(m.kind), 6)
    return np.nonzero((errs[0] > tol[:, 0]) | (errs[1] > tol[:, 2]) | (errs[2] > tol[:, 4]))[0]


class Table:
    def __init__(self):
        self.worst = {}
        self.bad = []

    def check(self, m, got, ref, config, path):
        errs = errors(m, got, ref, config)
        for i in range(len(m.cases)):
            k = (str(m.kind[i]), str(m.cls[i]), path)
            self.worst[k] = tuple(max(a, float(e[i])) for a, e in zip(self.worst.get(k, (0.0, 0.0, 0.0)), errs))
        self.bad += [(str(m.kind[i]), str(m.cls[i]), path, config, [float(e[i]) for e in errs]) for i in over(m, errs)]

    def show(self):
        print("\nworst error per (kind, class, path): position/velocity, rotation, omega")
        for k in sorted(self.worst):
            print("  %-28s %-16s %-12s %.2e %.2e %.2e" % (k + self.worst[k]))
        per_class = {}
        for (kind, cls, _), v in self.worst.items():
            per_class[(kind, cls)] = tuple(max(a, b) for a, b in zip(per_class.get((kind, cls), (0.0, 0.0, 0.0)), v))
        print("TOL-MEASURED", repr(per_class))


def _with_clusters(shape, fn):
    old = os.environ.pop("PBD_B200_CLUSTERS", None)
    if shape:
        os.environ["PBD_B200_CLUSTERS"] = shape
    try:
        return fn()
    finally:
        os.environ.pop("PBD_B200_CLUSTERS", None)
        if old is not None:
            os.environ["PBD_B200_CLUSTERS"] = old


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_rigid_answers_every_path():
    from positionbaseddynamics_b200 import _capi
    m = model()
    table = Table()
    refs = {}

    def ref(config, mut=None):
        if (config, mut) not in refs:
            with np.errstate(invalid="ignore", divide="ignore"):
                refs[(config, mut)] = rc.reference(m, *config, steps=STEPS, mut=mut)
        return refs[(config, mut)]

    launch = {}
    for mode, path in ((_capi.MODE_LAUNCH, "launch"), (_capi.MODE_GRAPH, "graph")):
        eng = engine(m, mode)
        for config in pc.CONFIGS:
            got = run(eng, m, config)
            assert eng.get_mode()[1] == mode
            table.check(m, got, ref(config), config, path)
            if mode == _capi.MODE_LAUNCH:
                launch[config] = got
            else:
                assert _same(got, launch[config]), (path, config)
        eng.close()

    x0 = rc.tile_x0(m, np.random.default_rng(5))
    for shape in ("1x1", "1x4"):
        def resident():
            eng = engine(m, _capi.MODE_RESIDENT, x0=x0)
            out = {config: run(eng, m, config) for config in ((2, 3, 1), (1, 1, 0), (1, 3, 1))}
            assert eng.get_mode() == (_capi.MODE_RESIDENT, _capi.MODE_RESIDENT), shape
            eng.close()
            return out
        for config, got in _with_clusters(shape, resident).items():
            table.check(m, got, ref(config), config, "resident" + shape)
            assert _same(got, launch[config]), ("resident" + shape, config)
    table.show()
    assert {k[:2] for k in table.worst} == set(TOL)  # every gated class ran
    assert not table.bad, (len(table.bad), table.bad[:20])

    # negative controls: the gate fails against each mutated restatement on the classes it must catch
    both_dynamic = ["small", "large", "rotated", "spinning", "ratio1e3", "lever0", "lever10", "shift1e2", "shift1e3"]
    controls = (("no_gyro", (2, 3, 1), [("BallJoint", "spinning"), ("free", "free")]),
                ("RtDR", (2, 3, 1), [("BallJoint", "rotated"), ("RigidBodyParticleBallJoint", "rotated"), ("free", "free")]),
                ("omega_conj", (2, 3, 1), [(k, c) for k in ("BallJoint", "RigidBodyParticleBallJoint") for c in ("rotated", "spinning")]),
                ("no_particle_w", (1, 3, 0), [("RigidBodyParticleBallJoint", c) for c in both_dynamic] + [("chain", "chain")]),
                ("first_order_rb", (2, 3, 1), [("BallJoint", c) for c in both_dynamic] + [("free", "free")]))
    for mut, config, must in controls:
        with np.errstate(invalid="ignore", divide="ignore"):
            errs = errors(m, launch[config], ref(config, mut), config)
        bad = over(m, errs)
        print("negative control %-15s cases outside the gate per named class: %s" % (mut, ", ".join(
            "%s/%s %d/%d" % (k, c, np.isin(bad, np.nonzero((m.kind == k) & (m.cls == c))[0]).sum(), ((m.kind == k) & (m.cls == c)).sum())
            for k, c in must)))
        print("  every class with a case outside the gate: %s" % sorted({(str(m.kind[i]), str(m.cls[i])) for i in bad}))
        for k, c in must:
            assert np.isin(bad, np.nonzero((m.kind == k) & (m.cls == c))[0]).any(), ("negative control passed the gate", mut, k, c)


def _bodies_with_particle_joints(n, seed):
    rng = np.random.default_rng(seed)
    m = rc.Model()
    for i in range(n):
        rc.add_case(m, rng, "RigidBodyParticleBallJoint", ("rotated", "spinning", "small", "large")[i % 4])
    return m.finish()


@pytest.mark.gpu
def test_resident_steps_every_body_in_one_cluster():
    """700 bodies, each in a particle joint, in one resident cluster: more bodies than the kernel has threads per CTA.  The resident
    result equals MODE_LAUNCH bit for bit, and both are within the gate of the fp64 restatement."""
    from positionbaseddynamics_b200 import _capi
    m = _bodies_with_particle_joints(700, 77)
    config = (2, 3, 1)
    eng = engine(m, _capi.MODE_LAUNCH)
    want = run(eng, m, config); eng.close()
    eng = engine(m, _capi.MODE_RESIDENT)
    got = run(eng, m, config)
    assert eng.get_mode() == (_capi.MODE_RESIDENT, _capi.MODE_RESIDENT)
    eng.close()
    stepped = (got[2][:, :3] != m.bx).any(1)
    print("resident, one cluster: %d of %d bodies moved; bodies differing from MODE_LAUNCH: %s" %
          (stepped.sum(), m.nb, np.nonzero((got[2] != want[2]).any(1))[0][:8]))
    assert _same(got, want)
    e = [float(x.max()) for x in errors(m, got, rc.reference(m, *config, steps=STEPS), config)]
    print("against fp64: position / velocity %.2e, rotation %.2e, omega %.2e" % tuple(e))
    assert max(e) <= REGRESSION_TOL


def cloth_and_free_bodies():
    """A 210 x 210 XPBD cloth (the checker's cfg2 model, 4 iterations) and 700 free dynamic bodies: (bodies as a Model, the cloth's
    (x, masses, (types, bodies, params, group offsets, group ids)))."""
    import scenes
    rng = np.random.default_rng(99)
    m = rc.Model()
    for _ in range(350):
        rc.add_case(m, rng, "free", "free")
    m = m.finish()
    assert m.nb == 700
    cpu = rc.po.CpuPbd("oracle", "f64")
    scenes.cfg2(cpu, 210, 4)
    mass, _ = cpu.masses()
    return m, (cpu.get("x").astype(np.float32), mass, tuple(cpu.constraints()[:3]) + tuple(cpu.groups()))


# forced on the free-body scene: independent resident CTAs, which give some of their threads to the X items
INDEPENDENT_CTAS = "8x1"


def _free_bodies_against_graph(mode, shape, path):
    """The scene of cloth_and_free_bodies in `mode` (PBD_B200_CLUSTERS = shape, or the planner's choice) and in MODE_GRAPH: the active
    mode, both results, and the worst fp64 errors of the bodies."""
    from positionbaseddynamics_b200 import _capi
    m, cloth = cloth_and_free_bodies()
    v = np.zeros((len(cloth[0]), 3), np.float32)
    config = (1, 4, 0)

    def one(md):
        eng = engine(m, md, particles=cloth)
        got = run(eng, m, config, particles=(cloth[0], v))
        active = eng.get_mode()[1]
        eng.close()
        return got, active

    got, active = _with_clusters(shape, lambda: one(mode))
    want, _ = one(_capi.MODE_GRAPH)
    print("%s: bodies differing from MODE_GRAPH: %d of %d" % (path, (got[2] != want[2]).any(1).sum(), m.nb))
    e = [float(x.max()) for x in errors(m, (m.px, m.pv, got[2]), (m.px, m.pv, rc.reference(m, *config, steps=STEPS)[2]), config)]
    print("%s: bodies against fp64: position / velocity %.2e, rotation %.2e, omega %.2e" % ((path,) + tuple(e)))
    return active, got, want, e


@pytest.mark.gpu
def test_auto_resident_steps_free_bodies_beyond_the_block():
    """The cloth and 700 free bodies under MODE_AUTO: the resident mode, as one cluster of 16 CTAs of 640 threads
    (tests/test_image_plan.py::test_free_bodies_beyond_the_block_are_planned_as_intended).  Bodies and cloth equal MODE_GRAPH bit for bit;
    the bodies are within the fp64 bound."""
    from positionbaseddynamics_b200 import _capi
    active, got, want, e = _free_bodies_against_graph(_capi.MODE_AUTO, None, "resident (AUTO), one cluster")
    assert active == _capi.MODE_RESIDENT
    assert _same(got, want)
    assert max(e) <= REGRESSION_TOL


@pytest.mark.gpu
def test_independent_ctas_step_free_bodies_beyond_the_block():
    """The same scene as 8 independent resident CTAs (PBD_B200_CLUSTERS; the planner admits bodies without joints there): CTA 0's
    threads past the X-item share are X threads, so fewer shared-memory threads than bodies step them.  Bodies and cloth equal MODE_GRAPH
    bit for bit; the bodies are within the fp64 bound."""
    from positionbaseddynamics_b200 import _capi
    active, got, want, e = _free_bodies_against_graph(_capi.MODE_RESIDENT, INDEPENDENT_CTAS, "resident %s" % INDEPENDENT_CTAS)
    assert active == _capi.MODE_RESIDENT
    assert _same(got, want)
    assert max(e) <= REGRESSION_TOL
