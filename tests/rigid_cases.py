"""Seeded rigid-body cases for both joint types and the fp64 restatement of what the engine does with the rigid parts of a substep
(tests/test_gpu_rigid_answers.py).

A case is a small independent group of rigid bodies and particles; many cases share one model, and every case carries the name of its edge
class.  Everything either side sees -- x, q, v, omega, masses, principal inertias and the joint point -- is rounded to fp32 once: the engine
gets those values, the fp64 restatement gets them promoted.  The joints' local connectors are what the checker's own initConstraint derives
from the bodies' poses at construction, so every joint starts satisfied; a case's velocities violate it by the time the first projection
runs (one full step's worth: a fraction of the lever arm over DT).  Classes:

  BallJoint                    small / large (violated by 1e-3 / 0.5 of the lever arm), rotated (random q, principal inertias up to
                               1:10:100), spinning (|omega| up to 20 rad/s about a non-principal axis), static0 / static1 / both_static,
                               ratio1e3 (masses 1 and 1024), lever0 (the joint at body 0's centre of mass) / lever10 (lever arms of 10),
                               shift1e2 / shift1e3 (the whole case translated by 1e2 / 1e3)
  RigidBodyParticleBallJoint   the same, with static_body / static_particle / both_static
  chain                        body B in four joints across colours (BallJoints to bodies A and C, two particle joints), C in a
                               particle joint: the joints of one body in consecutive colours
  free                         bodies in no joint: integration with the gyroscopic term and the velocity update alone

The restatement (`reference`) follows the checker's TimeStepController step (oracle/pbd_oracle.c step_once): per substep the bodies'
semi-implicit Euler with the term omega x (I_w omega) and the quaternion update, the particles' Euler step, max_iter sweeps of the joints in
the checker's colour-group order (both lever arms taken before either body moves), then the first- or second-order linear velocity update
and the first-order angular one in both modes (TimeIntegration.cpp:82-95).  `mut` names a deliberate error for the negative controls.
"""
import numpy as np

from oracle import pyoracle as po

BJ, RBP = po.BALLJOINT, po.RB_PARTICLE_BALLJOINT
KINDS = ("BallJoint", "RigidBodyParticleBallJoint", "chain", "free")
COMMON = ["small", "large", "rotated", "spinning", "ratio1e3", "lever0", "lever10", "shift1e2", "shift1e3"]
CLASSES = {"BallJoint": COMMON + ["static0", "static1", "both_static"],
           "RigidBodyParticleBallJoint": COMMON + ["static_body", "static_particle", "both_static"],
           "chain": ["chain"], "free": ["free"]}
DT = float(np.float32(0.005))
GRAVITY = (0.0, -9.81, 0.0)
MUTATIONS = ("no_gyro", "RtDR", "omega_conj", "no_particle_w", "first_order_rb")

_checker = None


def checker():
    """The fp64 checker the cases are built in: the unmodified reference when oracle/_ref travelled here and exports the velocity setter,
    else the C restatement."""
    global _checker
    if _checker is None:
        kind = "ref" if po.available("ref", "f64") and hasattr(po.CpuPbd("ref", "f64").lib, "ref_set_rigid_body_velocity") else "oracle"
        if not po.available(kind, "f64"):
            po.build(ref=False)
        _checker = po.CpuPbd(kind, "f64")
    return _checker


def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def _unit(rng):
    d = rng.normal(size=3)
    return d / np.linalg.norm(d)


def _quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q) * np.sign(q[0])


class Model:
    """Particles (x, v, m), bodies (mass, x, q (w, x, y, z), v, omega, principal inertia), joints (type, two body indices, joint point),
    and the case (kind, class) of every body, particle and joint; fp32 values held as float64."""

    def __init__(self):
        self.px, self.pv, self.pm, self.pcase = [], [], [], []
        self.bm, self.bx, self.bq, self.bv, self.bw, self.bI, self.bcase = [], [], [], [], [], [], []
        self.joints = []  # (type, a, b, point, case)
        self.cases = []   # (kind, class)

    def particle(self, x, v, m):
        self.px.append(x); self.pv.append(v); self.pm.append(m); self.pcase.append(len(self.cases))
        return len(self.px) - 1

    def body(self, m, x, q, v, w, inertia):
        self.bm.append(m); self.bx.append(x); self.bq.append(q); self.bv.append(v); self.bw.append(w); self.bI.append(inertia)
        self.bcase.append(len(self.cases))
        return len(self.bm) - 1

    def finish(self):
        """fp32-rounded arrays, then built in the checker: its constraint rows (the local connectors) and colour groups."""
        for f in ("pm", "bm"):
            setattr(self, f, _f32(np.array(getattr(self, f), np.float64).reshape(-1)))
        for f in ("px", "pv", "bx", "bq", "bv", "bw", "bI"):
            setattr(self, f, _f32(np.array(getattr(self, f), np.float64).reshape(-1, 4 if f == "bq" else 3)))
        self.pcase, self.bcase = np.array(self.pcase, int), np.array(self.bcase, int)
        self.kind = np.array([k for k, _ in self.cases]); self.cls = np.array([c for _, c in self.cases])
        self.joints = [(t, a, b, _f32(p), c) for t, a, b, p, c in self.joints]
        ck = load(self, checker())
        self.types, self.bodies, self.params, _ = ck.constraints()
        self.off, self.ids = ck.groups()
        assert len(self.types) == len(self.joints), "the checker refused a joint"
        self.jcase = np.array([j[4] for j in self.joints], int)
        return self

    @property
    def n(self):
        return len(self.px)

    @property
    def nb(self):
        return len(self.bm)


def load(m, ck):
    """The model's particles, bodies and joints in checker `ck` (reset first)."""
    ck.reset()
    ck.add_triangle_model(m.px if m.n else np.zeros((1, 3)), np.zeros((0, 3), np.uint32))
    for i in range(m.n):
        ck.set_mass(i, m.pm[i])
    if m.n:
        ck.set("v", m.pv)
    else:
        ck.set_mass(0, 0.0)  # a placeholder particle nothing touches
    for i in range(m.nb):
        assert ck.add_rigid_body(m.bm[i], m.bx[i], m.bI[i], m.bq[i]) == i
        ck.set_rigid_body_velocity(i, m.bv[i], m.bw[i])
    for t, a, b, p, _ in m.joints:
        assert ck.add_ball_joint(a, b, p) if t == BJ else ck.add_rb_particle_ball_joint(a, b)
    return ck


def _inertia(rng, cls):
    if cls in ("rotated", "free"):  # ratios up to 1:10:100 in a random order
        return rng.permutation([1.0, float(rng.choice([3.0, 10.0])), float(rng.choice([30.0, 100.0]))]) * rng.uniform(0.02, 0.2)
    return rng.uniform(0.05, 0.15, 3)


def _omega(rng, cls):
    if cls in ("spinning", "free"):
        return _unit(rng) * rng.uniform(5.0, 20.0)
    return _unit(rng) * rng.uniform(0.0, 1.0)


def add_case(m, rng, kind, cls):
    """One case of (kind, class) into model m."""
    c = len(m.cases)
    shift = np.zeros(3)
    if cls.startswith("shift"):
        shift = _unit(rng) * float(cls[5:])
    base = shift + rng.uniform(-1.0, 1.0, 3)
    lever = {"lever0": 0.0, "lever10": 10.0}.get(cls, rng.uniform(0.5, 1.5))
    viol = {"small": 1e-3, "large": 0.5}.get(cls, 0.05) * max(lever, 1.0) / DT  # relative velocity that violates the joint over one step
    q0 = _quat(rng) if cls != "lever0" or rng.random() < 0.5 else np.array([1.0, 0, 0, 0])
    v0 = rng.uniform(-0.3, 0.3, 3)
    if kind == "free":
        for _ in range(2):
            m.body(rng.uniform(0.5, 2.0), base + rng.uniform(-1, 1, 3), _quat(rng), v0, _omega(rng, "free"), _inertia(rng, "free"))
        m.cases.append((kind, cls))
        return
    if kind == "chain":
        A = m.body(0.0 if rng.random() < 0.5 else 1.0, base, _quat(rng), np.zeros(3), np.zeros(3), _inertia(rng, "rotated"))
        if m.bm[A] != 0.0:
            m.bv[A] = v0; m.bw[A] = _omega(rng, "spinning")
        jab = base + _unit(rng) * 0.8
        B = m.body(1.0, jab + _unit(rng) * 0.8, _quat(rng), rng.uniform(-1, 1, 3), _omega(rng, "spinning"), _inertia(rng, "rotated"))
        jbc = m.bx[B] + _unit(rng) * 0.8
        C = m.body(rng.choice([0.5, 2.0]), jbc + _unit(rng) * 0.8, _quat(rng), rng.uniform(-1, 1, 3), _omega(rng, "rotated"), _inertia(rng, "rotated"))
        m.joints.append((BJ, A, B, jab, c)); m.joints.append((BJ, B, C, jbc, c))
        for body in (B, B, C):
            p = m.particle(m.bx[body] + _unit(rng) * rng.uniform(0.5, 1.0), rng.uniform(-1, 1, 3), rng.choice([0.5, 1.0]))
            m.joints.append((RBP, body, p, None, c))
        m.cases.append((kind, cls))
        return
    m0, m1 = rng.uniform(0.5, 2.0), rng.uniform(0.5, 2.0)
    if cls == "ratio1e3":
        m0, m1 = (1.0, 1024.0) if rng.random() < 0.5 else (1024.0, 1.0)
    if cls in ("static0", "static_body", "both_static"):
        m0 = 0.0
    if cls in ("static1", "static_particle", "both_static"):
        m1 = 0.0
    w0 = _omega(rng, cls) if m0 else np.zeros(3)
    v0 = v0 if m0 else np.zeros(3)
    A = m.body(m0, base, q0, v0, w0, _inertia(rng, cls))
    point = base + _unit(rng) * lever
    # the second side drifts away from the joint at `viol` (the first side when the second is static)
    drift = _unit(rng) * viol
    v1 = rng.uniform(-0.3, 0.3, 3) + (drift if m1 else 0.0)
    if not m1 and m0:
        m.bv[A] = m.bv[A] - drift
    if kind == "BallJoint":
        arm1 = {"lever10": 10.0}.get(cls, rng.uniform(0.5, 1.5))
        B = m.body(m1, point + _unit(rng) * arm1, _quat(rng), v1 if m1 else np.zeros(3), _omega(rng, cls) if m1 else np.zeros(3),
                   _inertia(rng, cls))
        m.joints.append((BJ, A, B, point, c))
    else:
        p = m.particle(point, v1 if m1 else np.zeros(3), m1)
        m.joints.append((RBP, A, p, None, c))
    m.cases.append((kind, cls))


def make_model(per_class, seed, kinds=KINDS):
    rng = np.random.default_rng(seed)
    m = Model()
    for kind in kinds:
        for cls in CLASSES[kind]:
            for _ in range(per_class):
                add_case(m, rng, kind, cls)
    return m.finish()


def tile_x0(m, rng):
    """Rest positions on a line in a random order: the resident planner bisects them into tiles, so a case's particles (and the particles
    of a body's joints) land in different tiles of a cluster."""
    x0 = np.zeros((max(m.n, 1), 3), np.float32)
    x0[:m.n, 0] = rng.permutation(m.n)
    return x0


# ---------------------------------------------------------------------------------------------------------------------------------
# fp64 restatement
# ---------------------------------------------------------------------------------------------------------------------------------
def qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
                     a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def qconj(a):
    return np.array([a[0], -a[1], -a[2], -a[3]])


def qmatrix(q):
    """Eigen's toRotationMatrix (no normalisation: the fp32-rounded inputs are unit to rounding only, on both sides)."""
    w, x, y, z = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    return np.array([[1 - (ty * y + tz * z), ty * x - tz * w, tz * x + ty * w],
                     [ty * x + tz * w, 1 - (tx * x + tz * z), tz * y - tx * w],
                     [tz * x - ty * w, tz * y + tx * w, 1 - (tx * x + ty * y)]])


def skew(r):
    return np.array([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])


class _State:
    def __init__(self, m):
        self.px, self.pv = m.px.copy(), m.pv.copy()
        self.pold, self.plast = m.px.copy(), m.px.copy()
        self.bx, self.bq, self.bv, self.bw = m.bx.copy(), m.bq.copy(), m.bv.copy(), m.bw.copy()
        self.bold, self.blast, self.qold, self.qlast = m.bx.copy(), m.bx.copy(), m.bq.copy(), m.bq.copy()


def _world(m, i, q, d, mut):
    R = qmatrix(q)
    return (R.T @ np.diag(d) @ R) if mut == "RtDR" else (R @ np.diag(d) @ R.T)


def _k(w, r, J):
    """computeMatrixK: w 1 - [r]x J [r]x (zero for a static side)."""
    if w == 0.0:
        return np.zeros((3, 3))
    S = skew(r)
    return w * np.eye(3) - S @ J @ S


def _correct(m, s, i, r, pt, mut):
    """BallJoint::solvePositionConstraint's body update: x += w pt; q += 1/2 (0, J (r x pt)) q; normalise."""
    J = _world(m, i, s.bq[i], 1.0 / m.bI[i], mut)
    ot = J @ np.cross(r, pt)
    s.bx[i] = s.bx[i] + pt / m.bm[i]
    q = s.bq[i] + 0.5 * qmul(np.array([0.0, *ot]), s.bq[i])
    s.bq[i] = q / np.linalg.norm(q)


def _project(m, s, j, mut):
    t, (a, b) = int(m.types[j]), m.bodies[j][:2]
    p = m.params[j]
    wa = 1.0 / m.bm[a] if m.bm[a] else 0.0
    ca = qmatrix(s.bq[a]) @ p[0:3] + s.bx[a]
    ra = ca - s.bx[a]
    K = _k(wa, ra, _world(m, a, s.bq[a], 1.0 / m.bI[a], mut))
    if t == BJ:
        wb = 1.0 / m.bm[b] if m.bm[b] else 0.0
        cb = qmatrix(s.bq[b]) @ p[3:6] + s.bx[b]
        rb = cb - s.bx[b]
        K = K + _k(wb, rb, _world(m, b, s.bq[b], 1.0 / m.bI[b], mut))
        if wa == 0.0 and wb == 0.0:
            return
        pt = np.linalg.solve(K, cb - ca)
        if wa:
            _correct(m, s, a, ra, pt, mut)
        if wb:
            _correct(m, s, b, rb, -pt, mut)
    else:
        wp = 1.0 / m.pm[b] if m.pm[b] else 0.0
        if wp and (mut != "no_particle_w" or wa == 0.0):
            K = K + wp * np.eye(3)
        if wa == 0.0 and wp == 0.0:
            return
        pt = np.linalg.solve(K, s.px[b] - ca)
        if wa:
            _correct(m, s, a, ra, pt, mut)
        if wp:
            s.px[b] = s.px[b] - wp * pt


def reference(m, sub, iters, vel, dt=DT, steps=1, gravity=GRAVITY, mut=None):
    """Particles (x, v) and bodies (n, 13: x, q (w, x, y, z), v, omega) after `steps` steps of model m."""
    s = _State(m)
    g = np.asarray(gravity, np.float64)
    h = dt / sub
    pdyn, bdyn = m.pm != 0, m.bm != 0
    order = [int(j) for j in m.ids]
    groups = [order[m.off[k]:m.off[k + 1]] for k in range(len(m.off) - 1)]
    for _ in range(steps):
        for _ in range(sub):
            s.blast, s.bold = s.bold.copy(), s.bx.copy()
            s.qlast, s.qold = s.qold.copy(), s.bq.copy()
            for i in np.nonzero(bdyn)[0]:
                s.bv[i] = s.bv[i] + g * h
                s.bx[i] = s.bx[i] + s.bv[i] * h
                om = s.bw[i]
                if mut != "no_gyro":
                    om = om + _world(m, i, s.bq[i], 1.0 / m.bI[i], mut) @ (-np.cross(om, _world(m, i, s.bq[i], m.bI[i], mut) @ om)) * h
                s.bw[i] = om
                q = s.bq[i] + 0.5 * h * qmul(np.array([0.0, *om]), s.bq[i])
                s.bq[i] = q / np.linalg.norm(q)
            s.plast, s.pold = s.pold.copy(), s.px.copy()
            s.pv[pdyn] += g * h
            s.px[pdyn] += s.pv[pdyn] * h
            for _ in range(iters):
                for grp in groups:
                    for j in grp:
                        _project(m, s, j, mut)
            for i in np.nonzero(bdyn)[0]:
                if vel == 0 or mut == "first_order_rb":
                    s.bv[i] = (s.bx[i] - s.bold[i]) / h
                else:
                    s.bv[i] = (1.5 * s.bx[i] - 2.0 * s.bold[i] + 0.5 * s.blast[i]) / h
                rel = qmul(qconj(s.qold[i]), s.bq[i]) if mut == "omega_conj" else qmul(s.bq[i], qconj(s.qold[i]))
                s.bw[i] = rel[1:] * (2.0 / h)
            if vel == 0:
                s.pv[pdyn] = (s.px[pdyn] - s.pold[pdyn]) / h
            else:
                s.pv[pdyn] = (1.5 * s.px[pdyn] - 2.0 * s.pold[pdyn] + 0.5 * s.plast[pdyn]) / h
    return s.px, s.pv, np.concatenate([s.bx, s.bq, s.bv, s.bw], axis=1)
