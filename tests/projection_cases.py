"""Seeded one-constraint stencils for every particle constraint type and the fp64 restatement of what the engine does with them
(tests/test_gpu_projection_answers.py).

A case is one constraint on four private particles (the unused ones of 2- and 3-body types are free particles nothing touches).  Its
rest geometry is what the checker's own initConstraint derives from a rest stencil (a one-constraint model's constraints() row), and
everything either side sees -- x, v, masses, parameters, dt -- is rounded to fp32 once: the engine gets those values, the fp64 reference
gets them promoted.  Every case carries the name of its edge class; `branches` records which of the solver branches that DESIGN.md
section 5 keeps literally the case takes, decided from the fp64 inputs.  A case whose deciding quantity lies within 1e-3 (relative) of a
branch threshold is drawn again: there fp32 and fp64 may legitimately decide differently.

The reference (`reference`, `reference_jacobi`) restates the engine's loop on a free stencil with gravity 0 around the checker's
stateless solver entry point kat_solve (the unmodified reference's when oracle/_ref is present, else the C restatement, which
tests/test_oracle_golden.py pins to the reference): sub_steps x max_iter sweeps, lambda carried across the sweeps of a substep and zeroed
at each substep's first sweep, FEMTet's handleInversion recomputed from the current volume at every sweep, ShapeMatching's raw answer
scaled by 1/numClusters, corrections applied to dynamic particles only, integration and the velocity update between substeps.
"""
import numpy as np

from oracle import pyoracle as po

TYPES = list(range(13))  # every particle constraint type (the joints have no kat_solve entry)
NB = po.NBODIES
NP = po.NPARAMS
XPBD = (po.DISTANCE_XPBD, po.ISOBENDING_XPBD, po.VOLUME_XPBD, po.FEMTET_XPBD)
ISO = (po.ISOBENDING, po.ISOBENDING_XPBD)
FEMTETS = (po.FEMTET, po.FEMTET_XPBD)
# material columns of a parameter row (include/pbd_b200.h); the others are rest geometry, contiguous
MAT = {0: [1], 1: [1], 2: [1], 3: [0], 4: [0], 5: [5, 6, 7, 8, 9], 6: [4, 5, 6, 7, 8], 7: [1], 8: [1], 9: [10, 11], 10: [10, 11],
       11: [9, 10, 11, 12], 12: [0]}
GEO = {t: [c for c in range(NP[t]) if c not in MAT[t]] for t in TYPES}
# the stiffness-like columns (what a "stiffness x 1.01" mutation scales and the "k0" class zeroes); FEMTriangle: the first Young's
# modulus only, because scaling all three together leaves the PBD answer unchanged (as scaling E does for FEMTet)
STIFF = {0: [1], 1: [1], 2: [1], 3: [0], 4: [0], 5: [5], 6: [4, 5, 6], 7: [1], 8: [1], 9: [10], 10: [10], 11: [9, 10], 12: [0]}
# the material arguments of add_constraint (their order is the order of MAT's columns); ShapeMatching: k + four numClusters
DEFAULT_U = {0: [0.8], 1: [1.0e5], 2: [0.5], 3: [0.5], 4: [100.0], 5: [1000.0, 800.0, 400.0, 0.3, 0.25], 6: [1.0, 0.8, 0.6, 0.0, 0.0],
             7: [0.7], 8: [1.0e5], 9: [1000.0, 0.3], 10: [1.0e4, 0.3], 11: [1.0, 0.7, 0.0, 0.0], 12: [0.6]}
DT = float(np.float32(0.005))
CONFIGS = [(1, 1, 0), (1, 1, 1), (1, 3, 0), (1, 3, 1), (2, 3, 0), (2, 3, 1)]  # (sub_steps, max_iter, velocity method)

_checker = None


def checker():
    """The fp64 kat_solve provider: the unmodified reference when oracle/_ref travelled here, else the C restatement."""
    global _checker
    if _checker is None:
        kind = "ref" if po.available("ref", "f64") else "oracle"
        if not po.available(kind, "f64"):
            po.build(ref=False)
        _checker = po.CpuPbd(kind, "f64")
    return _checker


def classes_of(t):
    c = ["small", "large", "shift1e2", "shift1e3", "some_static", "all_static", "ratio1e3", "k0"]
    if t in XPBD:
        c += ["k1e2", "k1e5", "k1e9"]
    if t in (po.DISTANCE, po.DISTANCE_XPBD):
        c += ["coincident"]
    if t in (po.VOLUME, po.VOLUME_XPBD):
        c += ["flat", "collinear"]
    if t == po.DIHEDRAL:
        c += ["planar0", "planar_pi"]
    if t in (po.FEMTRIANGLE, po.STRAINTRIANGLE):
        c += ["collinear"]
    if t in FEMTETS:
        c += ["inverted", "compressed", "flat", "nu_out"]
    if t == po.STRAINTET:
        c += ["inverted", "flat"]
    if t == po.SHAPEMATCHING:
        c += ["rotated", "reflected"]
    return c


def _rot(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def _rest(rng, t):
    """A well-conditioned O(1) rest stencil (4 points; unused ones free), randomly rotated and scaled."""
    if t in (po.DISTANCE, po.DISTANCE_XPBD):
        x = np.array([[0.0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]])
    elif t in (po.DIHEDRAL,) + ISO:  # two triangles sharing the edge (x2, x3); x0, x1 opposite
        x = np.array([[0.0, 1.0, 0.0], [0.0, -1.0, 0.3], [-1.0, 0.0, 0.0], [1.0, 0.0, 0.0]])
    elif t in (po.FEMTRIANGLE, po.STRAINTRIANGLE):
        x = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.2], [0.2, 0.0, 1.0], [0.5, 0.5, 0.5]])
    else:
        x = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    x = x + rng.uniform(-0.15, 0.15, (4, 3))
    return (x @ _rot(rng).T) * rng.uniform(0.6, 1.6)


def _material(rng, t, cls):
    u = list(DEFAULT_U[t])
    if t == po.SHAPEMATCHING:
        u = [u[0] if rng.random() < 0.5 else float(rng.choice([0.2, 1.0]))] + [float(rng.integers(1, 8)) for _ in range(4)]
    elif t in (po.STRAINTRIANGLE, po.STRAINTET):  # all four normalize-flag combinations
        f = len(u) - 2
        u[f], u[f + 1] = float(rng.integers(2)), float(rng.integers(2))
        if rng.random() < 0.5:
            u[0] *= float(rng.choice([0.3, 2.0]))
    elif t in FEMTETS:
        if rng.random() < 0.5:
            u = [u[0] * float(rng.choice([0.1, 100.0])), float(rng.choice([0.1, 0.45]))]
    elif t == po.FEMTRIANGLE:
        if rng.random() < 0.5:
            u = [float(rng.choice([1.0, 500.0])), float(rng.choice([1.0, 2000.0])), float(rng.choice([10.0, 400.0])), 0.2, 0.35]
    elif t not in XPBD and rng.random() < 0.5:
        u[0] = float(rng.choice([0.1, 0.3, 1.0]))
    if cls == "k0":  # stiffness 0; FEM: E = 0 or below (the E <= 0 early-out)
        if t in FEMTETS:
            u[0] = float(rng.choice([0.0, -1000.0]))
        else:
            for c in STIFF[t]:
                u[MAT[t].index(c)] = 0.0
    if t in XPBD and cls in ("k1e2", "k1e5", "k1e9"):
        u[0] = float(cls[1:])
    if cls == "nu_out":
        u[1] = float(rng.choice([-0.1, 0.6]))
    return u


def _tet_volume(x):
    return np.dot(np.cross(x[1] - x[0], x[2] - x[0]), x[3] - x[0]) / 6.0


def _dihedral_sign(x):
    """sin of the dihedral angle's sign test (n1 x n2) . e, normalised -- the kernel flips lambda on its sign."""
    p0, p1, p2, p3 = x
    e = p3 - p2
    n1 = np.cross(p2 - p0, p3 - p0); n2 = np.cross(p3 - p1, p2 - p1)
    return np.dot(np.cross(n1, n2), e) / max(np.linalg.norm(n1) * np.linalg.norm(n2) * np.linalg.norm(e), 1e-300)


def _state(rng, t, cls, x0):
    """Current positions and masses of one case of class `cls` around rest stencil x0."""
    nb = NB[t]
    m = np.ones(4)
    amp = {"small": 1e-3, "large": 0.3}.get(cls, 0.1)
    x = x0 + rng.uniform(-amp, amp, (4, 3))
    if cls == "some_static":
        k = int(rng.integers(1, nb))
        m[rng.choice(nb, k, replace=False)] = 0.0
    elif cls == "all_static":
        m[:] = 0.0
    elif cls == "ratio1e3":  # inverse masses 1 and 1/1024 (exact in fp32), both present
        m[:nb] = rng.permutation([1.0] + [1024.0] + list(rng.choice([1.0, 1024.0], nb - 2)))
    elif cls == "coincident":
        x[1] = x[0]
    elif cls in ("flat", "collinear", "planar0", "planar_pi"):
        # exact zeros: the decisions these classes test are taken on exactly degenerate geometry on both sides
        x = np.round(x0 + rng.uniform(-0.2, 0.2, (4, 3)), 3)
        x[:, 2] = 0.0
        if cls == "collinear":
            x[:, 1] = 0.0
        if cls == "planar0":  # the opposite vertices on either side of the edge: dihedral angle 0
            x[2] = [-1.0, 0.0, 0.0]; x[3] = [1.0, 0.0, 0.0]; x[0, 1] = abs(x[0, 1]) + 0.5; x[1, 1] = -abs(x[1, 1]) - 0.5
        if cls == "planar_pi":  # both on one side: folded flat, angle pi
            x[2] = [-1.0, 0.0, 0.0]; x[3] = [1.0, 0.0, 0.0]; x[0, 1] = abs(x[0, 1]) + 0.5; x[1, 1] = abs(x[1, 1]) + 0.9
    elif cls == "inverted":
        x[3] = x[0] + (x[0] - x[3]) * rng.uniform(0.3, 1.0)
    elif cls == "compressed":  # 0 < V/V0 < 0.2: handleInversion set, but no SVD branch
        x[3] = x[0] + (x[3] - x[0]) * rng.uniform(0.03, 0.15)
    elif cls == "rotated":
        x = (x0 - x0.mean(0)) @ _rot(rng).T + x0.mean(0) + rng.uniform(-0.05, 0.05, (4, 3))
    elif cls == "reflected":
        x = (x0 - x0.mean(0)) * np.array([-1.0, 1.0, 1.0]) @ _rot(rng).T + x0.mean(0)
    return x, m


def _near_threshold(t, cls, x, x0, p, m):
    """True when a deciding quantity of the first sweep lies within 1e-3 (relative) of its branch threshold."""
    if t in FEMTETS + (po.VOLUME, po.VOLUME_XPBD, po.STRAINTET) and cls not in ("flat", "collinear"):
        r = _tet_volume(x) / _tet_volume(x0)
        if abs(r) < 1e-3 or abs(r - 0.2) < 2e-4:
            return True
    if t == po.DIHEDRAL and cls not in ("planar0", "planar_pi"):
        if abs(_dihedral_sign(x)) < 1e-3:
            return True
    if t == po.SHAPEMATCHING:
        A = sum(np.outer(x[i] - x.mean(0), x0[i] - x0.mean(0)) for i in range(4))
        if abs(np.linalg.det(A)) < 1e-3 * np.linalg.norm(A) ** 3:
            return True
    return False


def branches_of(t, x, w, p, cls, fullq=False):
    """The literally kept branches (DESIGN.md section 5) this case takes at its first sweep, from the fp64 inputs."""
    b = {cls}
    nb = NB[t]
    if (w[:nb] == 0).all():
        b.add("wsum0")
    if t in (po.DISTANCE, po.DISTANCE_XPBD) and (x[0] == x[1]).all():
        b.add("d0")
    if any(p[c] == 0.0 for c in STIFF[t]) and t not in FEMTETS:
        b.add("k0")
    if t in XPBD:
        b.add("alpha0" if p[MAT[t][0]] == 0.0 else "alpha>0")
    if t in (po.VOLUME, po.VOLUME_XPBD):
        g = [np.cross(x[1] - x[2], x[3] - x[2]), np.cross(x[2] - x[0], x[3] - x[0]), np.cross(x[3] - x[0], x[1] - x[0]), np.cross(x[1] - x[0], x[2] - x[0])]
        b.add("K<=eps" if sum(w[i] * np.dot(g[i], g[i]) for i in range(4)) <= 1e-6 else "K>eps")
    if t in FEMTETS:
        r = _tet_volume(x) / p[0]
        b.add("E<=0" if p[10] <= 0 else ("nu_out" if not (0.0 <= p[11] <= 0.49) else "fem_solved"))
        b.add("svd" if r <= 0 else ("hinv_no_svd" if r < 0.2 else "no_hinv"))
    if t in FEMTETS + (po.STRAINTET,):
        v = _tet_volume(x)
        b.add("tet_flat" if v == 0 else ("tet_inverted" if v < 0 else "tet_upright"))  # the generator's rest tets are upright
    if t in (po.FEMTRIANGLE, po.STRAINTRIANGLE) and np.linalg.norm(np.cross(x[1] - x[0], x[2] - x[0])) == 0:
        b.add("tri_collinear")
    if t == po.DIHEDRAL:
        s = _dihedral_sign(x)
        n1 = np.cross(x[2] - x[0], x[3] - x[0]); n2 = np.cross(x[3] - x[1], x[2] - x[1])
        c = np.dot(n1, n2) / (np.linalg.norm(n1) * np.linalg.norm(n2))
        if s == 0 and c > 0:
            b.add("angle0")
        elif s == 0:
            b.add("angle_pi")
    if t == po.STRAINTRIANGLE:
        b.add("norm%d%d" % (p[7] != 0, p[8] != 0))
    if t == po.STRAINTET:
        b.add("norm%d%d" % (p[11] != 0, p[12] != 0))
    if t in ISO:
        b.add("fullq" if fullq else "rank1")
    if t == po.SHAPEMATCHING:
        if (p[20:24] > 1).any():
            b.add("numClusters>1")
        A = sum(np.outer(x[i] - x.mean(0), p[4 + 3 * i:7 + 3 * i] - p[1:4]) for i in range(4))
        if np.linalg.det(A) < 0:
            b.add("reflection")
    return b


REQUIRED = {  # branches every stencil set must take at least once
    "all": {"wsum0", "k0", "shift1e2", "shift1e3", "small", "large", "some_static", "ratio1e3"},
    po.DISTANCE: {"d0"}, po.DISTANCE_XPBD: {"d0", "alpha0", "alpha>0"},
    po.VOLUME: {"K<=eps", "K>eps"}, po.VOLUME_XPBD: {"K<=eps", "K>eps", "alpha0", "alpha>0"},
    po.DIHEDRAL: {"angle0", "angle_pi"},
    po.ISOBENDING: {"rank1"}, po.ISOBENDING_XPBD: {"rank1", "alpha0", "alpha>0"},
    po.FEMTRIANGLE: {"tri_collinear"},
    po.STRAINTRIANGLE: {"tri_collinear", "norm00", "norm01", "norm10", "norm11"},
    po.FEMTET: {"E<=0", "nu_out", "fem_solved", "svd", "hinv_no_svd", "no_hinv", "tet_flat", "tet_inverted"},
    po.FEMTET_XPBD: {"E<=0", "nu_out", "fem_solved", "svd", "hinv_no_svd", "no_hinv", "tet_flat", "tet_inverted", "alpha0", "alpha>0"},
    po.STRAINTET: {"norm00", "norm01", "norm10", "norm11", "tet_flat", "tet_inverted"},
    po.SHAPEMATCHING: {"numClusters>1", "reflection"},
}


class Cases:
    """Struct of arrays, one row per case: type, class, x / v (4, 3), masses (4), parameter row (24), fp32 values held as float64;
    `fullq`: an IsometricBending case whose Q is not of the rank-one form."""
    FIELDS = ("t", "cls", "x", "v", "m", "p", "fullq", "x0")

    def __init__(self, **kw):
        for f in self.FIELDS:
            setattr(self, f, kw[f])

    def __len__(self):
        return len(self.t)

    def take(self, sel):
        return Cases(**{f: getattr(self, f)[sel] for f in self.FIELDS})

    @staticmethod
    def cat(parts):
        return Cases(**{f: np.concatenate([getattr(c, f) for c in parts]) for f in Cases.FIELDS})

    def w(self):
        return np.where(self.m != 0, 1.0 / np.where(self.m != 0, self.m, 1.0), 0.0)

    def branches(self):
        w = self.w()
        return [branches_of(int(self.t[i]), self.x[i], w[i], self.p[i], self.cls[i], bool(self.fullq[i])) for i in range(len(self))]


def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def make_cases(t, per_class, seed, fullq=False):
    """per_class cases of every edge class of type t (fp32-representable values).  fullq: IsometricBending with a user-edited Q that
    is not rank one; the translated classes are left out there (see EXCLUDED in the test)."""
    ck = checker()
    rng = np.random.default_rng(seed)
    rows = []
    classes = [c for c in classes_of(t) if not (fullq and c.startswith("shift"))]
    for cls in classes:
        made = tries = 0
        while made < per_class:
            tries += 1
            assert tries < 50 * per_class, ("the generator cannot draw class", t, cls)
            x0 = _rest(rng, t)
            u = _material(rng, t, cls)
            x, m = _state(rng, t, cls, x0)
            if cls.startswith("shift"):
                d = rng.normal(size=3); d *= float(cls[5:]) / np.linalg.norm(d)
                x0 = x0 + d; x = x + d
            x0 = _f32(x0); x = _f32(x)
            ck.reset()
            ck.add_triangle_model(x0, np.zeros((0, 3), np.uint32))
            for i in range(4):
                ck.set_mass(i, m[i])  # ShapeMatching freezes the inverse masses now: the live ones of both sides
            if not ck.add_constraint(t, list(range(NB[t])), u[:8] if t != po.SHAPEMATCHING else u):
                continue
            p = np.zeros(24)
            p[:NP[t]] = ck.constraints()[2][0][:NP[t]]
            if fullq:
                a, b = rng.choice(4, 2, replace=False)
                Q = p[1:17].reshape(4, 4)
                Q[a, b] += 0.3; Q[b, a] += 0.3
                Q[a, a] += 0.2
            p = _f32(p)
            if _near_threshold(t, cls, x, x0, p, m):
                continue
            v = _f32(rng.uniform(-0.2, 0.2, (4, 3)))
            rows.append((t, cls, x, v, m, p, fullq, x0))
            made += 1
    return Cases(t=np.array([r[0] for r in rows], np.int32), cls=np.array([r[1] for r in rows]), x=np.array([r[2] for r in rows]),
                 v=np.array([r[3] for r in rows]), m=np.array([r[4] for r in rows]), p=np.array([r[5] for r in rows]),
                 fullq=np.array([r[6] for r in rows]), x0=np.array([r[7] for r in rows]))


def restate_state(cases, seed):
    """The same constraints (types, parameters) with another x, v and masses of the same edge classes: a replica's own state.  The
    masses of ShapeMatching cases stay, because the constraint froze them."""
    rng = np.random.default_rng(seed)
    out = Cases(**{f: getattr(cases, f).copy() for f in Cases.FIELDS})
    for i in range(len(cases)):
        t, cls = int(cases.t[i]), str(cases.cls[i])
        for _ in range(200):
            x, m = _state(rng, t, cls, cases.x0[i])  # x0 of a translated class is translated already
            x = _f32(x)
            if t == po.SHAPEMATCHING:
                m = cases.m[i]
            elif cls not in ("some_static", "all_static", "ratio1e3"):
                m = np.where(rng.random(4) < 0.2, 2.0, 1.0) if cls not in ("small",) else cases.m[i]
            if not _near_threshold(t, cls, x, cases.x0[i], cases.p[i], m):
                break
        out.x[i] = x; out.m[i] = m
        out.v[i] = _f32(rng.uniform(-0.2, 0.2, (4, 3)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# fp64 reference
# ---------------------------------------------------------------------------------------------------------------------------------
def _solve(ck, t, x, w, p, h, lam, mut, fullq=False):
    hinv = False
    if t in ISO and not fullq:
        # A rank-one Q annihilates translations, but its fp32-rounded entries do not quite: evaluated on absolute positions the
        # rounding of Q alone would move the answer of a stencil at |x| = 1e3 by O(0.1).  The engine's rank-one form is translation
        # invariant, so the reference takes the stencil about its own centroid (the corrections are unchanged by a translation).
        x = x - x.mean(0)
    if t in FEMTETS:
        hinv = bool(_tet_volume(x) / p[0] < 0.2)  # FEMTetConstraint::solvePositionConstraint, every sweep
    if mut == "q_off" and t in ISO:
        p = p.copy(); p[1] *= 1.0 + 1e-3
    res, corr, lam = ck.kat_solve(t, x, w, p, dt=h, handle_inversion=hinv, lam=lam)
    if not res:
        corr[:] = 0.0
    if t == po.SHAPEMATCHING:
        if mut != "sm_no_average":
            corr = corr / p[20:24, None]
        w = p[16:20]  # written where the frozen inverse mass is not zero (equal to the live one here)
    corr[w == 0] = 0.0
    return bool(res), corr, lam


def mutate_params(cases, mut):
    p = cases.p.copy()
    if mut == "stiffness_1.01":
        for i, t in enumerate(cases.t):
            for c in STIFF[int(t)]:
                p[i, c] *= 1.01
    return p


def reference(cases, sub, iters, vel, dt=DT, mut=None, ck=None, fp32_state=False):
    """x, v (N, 4, 3) and lambda (N) after one step of every case on its own.  ck: another kat_solve provider (the fp32 build of the C
    restatement); fp32_state: positions and velocities stored in fp32 after every update, as the engine stores them -- with both, the
    loop is an fp32 restatement of the engine, which tells how far fp32 itself is from fp64 on a case."""
    ck = ck or checker()
    rnd = _f32 if fp32_state else (lambda a: a)
    n = len(cases)
    X = cases.x.copy(); V = cases.v.copy(); L = np.zeros(n)
    W = cases.w()
    P = mutate_params(cases, mut)
    h = dt / sub
    for i in range(n):
        t = int(cases.t[i]); nb = NB[t]
        x = X[i]; v = V[i]; w = W[i]; p = P[i]
        dyn = cases.m[i] != 0
        old = x.copy(); last = x.copy()
        lam = 0.0
        for s in range(sub):
            last = old.copy(); old = x.copy()
            x[dyn] = rnd(x[dyn] + v[dyn] * h)
            for it in range(iters):
                if it == 0 and not (mut == "no_lambda_reset" and s > 0):
                    lam = 0.0
                _, corr, lam = _solve(ck, t, x, w, p, h, lam, mut, bool(cases.fullq[i]))
                x[:nb] = rnd(x[:nb] + corr[:nb])
            if vel == 0:
                v[dyn] = rnd((x[dyn] - old[dyn]) / h)
            else:
                v[dyn] = rnd((1.5 * x[dyn] - 2.0 * old[dyn] + 0.5 * last[dyn]) / h)
        L[i] = lam
    return X, V, L


def reference_jacobi(cases, bodies, n, x, v, m, sub, iters, vel, dt=DT, count_failed=True):
    """The engine's Jacobi mode in fp64 on constraints that share particles: every projection of a sweep reads the sweep-start
    positions; each store to a dynamic particle adds the correction (zero where the solve early-outs) and one count; the particle
    moves by the average.  count_failed False: the rule without the failed solves (a negative control)."""
    ck = checker()
    X = x.copy(); V = v.copy()
    w = np.where(m != 0, 1.0 / np.where(m != 0, m, 1.0), 0.0)
    dyn = m != 0
    h = dt / sub
    lam = np.zeros(len(cases))
    old = X.copy()
    for s in range(sub):
        last = old.copy(); old = X.copy()
        X[dyn] += V[dyn] * h
        for it in range(iters):
            if it == 0:
                lam[:] = 0.0
            acc = np.zeros_like(X); cnt = np.zeros(n)
            for c in range(len(cases)):
                t = int(cases.t[c]); b = bodies[c]
                xs = np.zeros((4, 3)); ws = np.zeros(4)
                xs[:NB[t]] = X[b]; ws[:NB[t]] = w[b]
                res, corr, lam[c] = _solve(ck, t, xs, ws, cases.p[c], h, lam[c], None, bool(cases.fullq[c]))
                for k in range(NB[t]):
                    if dyn[b[k]] and (res or count_failed):
                        acc[b[k]] += corr[k]; cnt[b[k]] += 1
            moved = cnt > 0
            X[moved] += acc[moved] / cnt[moved, None]
        if vel == 0:
            V[dyn] = (X[dyn] - old[dyn]) / h
        else:
            V[dyn] = (1.5 * X[dyn] - 2.0 * old[dyn] + 0.5 * last[dyn]) / h
    return X, V, lam
