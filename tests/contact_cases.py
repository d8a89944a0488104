"""Edge cases of the contact path and its fp64 restatement (tests/test_contact_cases.py on the CPU, tests/test_gpu_contact_answers.py on
the GPU).

Three layouts of at most kMaxRigidColliders = 8 static colliders each, built with contact_util.collider, every collider on a body with its
own centre, velocity and angular velocity:

  S  the six shapes with invert = 0 (box and sphere axis-aligned, the others in random frames), bodies 1, 3, 5 moving, and an
     overlapping sphere and box that share one body (shared_body; wedge: inside both, where their normals oppose)
  I  the six shapes with invert = 1, bodies 0, 2, 4 moving, and a box translated by 1e2 and a torus by 1e3 (shift1e2 / shift1e3)
  M  eight nested colliders around one centre (spheres and cylinders inside two boxes): particles inside 2 .. 8 of them (multi2 .. multi8)

Every layout has the same number of particles, N (several 128-thread blocks, not a multiple of 128), so that the three make the replicas of
one batch.  Particles 0 .. UNRANGED-1 belong to no particle range (they sit inside colliders and must be left alone); the rest are split
into three ranges with their own restitution and friction, listed out of offset order, one of them empty.  Every particle carries the
(shape, class) of its case; inputs are rounded to fp32 once, and the restatement takes them promoted to fp64.

The positions are designed as the positions after one step without gravity, so a case lands where it was placed: x_pre = x - v dt.

reference() restates, in numpy, what the contact kernel computes after the substeps: the bounding-box test, the local transform,
collisionTest (the analytic sphere and hollow-sphere overrides, otherwise central differences of the distance function with eps = 1e-6 in
double precision), the contact initialisation and max_iter_v Gauss-Seidel sweeps over each particle's contacts in collider order.
dtype = np.float32 runs the same operations in fp32 (the distance function stays fp64, as in the kernel); `mut` names a deliberate error
for the negative controls (MUTATIONS)."""
import numpy as np

import contact_util as cu

DT = 0.005
N = 701                # particles per layout
UNRANGED = 6           # particles 0 .. UNRANGED-1 are in no particle range
# (offset, count, restitution, friction): one range not starting at 0, an empty one, listed out of offset order
RANGES = [(o, c, float(np.float32(e)), float(np.float32(f))) for o, c, e, f in ((400, N - 400, 0.8, 0.3), (400, 0, 0.1, 0.9), (UNRANGED, 400 - UNRANGED, 0.5, 0.1))]
# (tolerance, stiffness, max_iter_v) x sub_steps
CONTACT = [(0.05, 100.0, 5), (0.05, 100.0, 1), (0.05, 0.0, 20), (0.0, 1.0e4, 5), (0.05, 100.0, 0)]
CONFIGS = [c + (s,) for c in CONTACT for s in (1, 2)]
LAYOUTS = ("S", "I", "M")
SHAPE_NAMES = dict(enumerate(cu.SHAPES))

DETECTION = ("deep", "shell", "outside", "aabb_cut", "crease", "axis", "hollow_in", "hollow_out")
SOLVE = ("approach", "separating", "stick", "slide", "normal_only", "tangent_zero", "static_particle", "moving_body")
STRUCTURE = tuple("multi%d" % k for k in range(2, 9)) + ("shared_body", "wedge", "shift1e2", "shift1e3", "unranged", "pad")
THRESHOLD = ("grazing", "on_crease", "aabb_face", "degenerate_normal")
MUTATIONS = ("no_omega", "omega_sign", "friction_swap", "no_sum_clamp", "restitution_always", "no_hollow_flip", "forward_diff", "reverse_order")

# every branch reference() tags (BRANCHES_SOLVE only run when max_iter_v > 0)
BRANCHES_DETECT = ("aabb_out", "aabb_in", "analytic_contact", "analytic_none", "analytic_hollow_flip", "analytic_n_zero", "fd_contact", "fd_none",
                   "fd_n_zero", "init_t_normalised", "init_t_unnormalised", "init_approach", "init_no_restitution", "static_particle")
BRANCHES_SOLVE = ("sum_clamp", "penalty", "friction_hi", "friction_lo", "friction_cone")


# ---------------------------------------------------------------------------------------------------------------------------------
# distance functions (fp64) and the restatement
# ---------------------------------------------------------------------------------------------------------------------------------
def sdf(c, x, tol):
    """The kernel's sdf_distance for collider c at local points x (M, 3), in float64."""
    x = np.asarray(x, np.float64)
    inv, d, th = (-1.0 if c["invert"] else 1.0), np.asarray(c["dim"], np.float64), float(c["thickness"])
    s = c["shape"]
    if s in (cu.BOX, cu.HOLLOW_BOX):
        q = np.abs(x) - d
        b = np.minimum(q.max(1), 0.0) + np.linalg.norm(np.maximum(q, 0.0), axis=1)
        return inv * (b if s == cu.BOX else np.abs(b) - th) - tol
    if s == cu.SPHERE:
        return inv * (np.linalg.norm(x, axis=1) - d[0]) - tol
    if s == cu.HOLLOW_SPHERE:
        return inv * (np.abs(np.linalg.norm(x, axis=1) - d[0]) - th) - tol
    if s == cu.TORUS:
        qx = np.sqrt(x[:, 0] ** 2 + x[:, 2] ** 2) - d[0]
        return inv * (np.sqrt(qx * qx + x[:, 1] ** 2) - d[1]) - tol
    l = np.sqrt(x[:, 0] ** 2 + x[:, 2] ** 2)  # cylinder
    q = np.stack([np.abs(l) - d[0], np.abs(x[:, 1]) - d[1]], 1)
    return inv * (np.minimum(q.max(1), 0.0) + np.linalg.norm(np.maximum(q, 0.0), axis=1)) - tol


def _tag(tags, name, count):
    if tags is not None and count:
        tags[name] = tags.get(name, 0) + int(count)


def detect(x, c, com, tol, dtype=np.float64, mut=None, tags=None):
    """One collider against every particle: (hit (M,), cp1 (M,3), n (M,3), dist (M,)) in world space."""
    f = dtype
    x = np.asarray(x, f); com = np.asarray(com, f)
    R = np.asarray(c["R"], f).reshape(3, 3); v1 = np.asarray(c["v1"], f); v2 = np.asarray(c["v2"], f)
    lo, hi = np.asarray(c["aabb_min"], f), np.asarray(c["aabb_max"], f)
    inbox = ~((x < lo) | (x > hi)).any(1)
    _tag(tags, "aabb_out", (~inbox).sum()); _tag(tags, "aabb_in", inbox.sum())
    d = x - com
    xl = (d[:, 0:1] * R[:, 0] + d[:, 1:2] * R[:, 1] + d[:, 2:3] * R[:, 2]) + v1  # R (x - com) + v1
    M = len(x)
    n = np.zeros((M, 3), f); cp = np.zeros((M, 3), f)
    tolf = f(tol)
    inv = f(-1.0 if c["invert"] else 1.0)
    if c["shape"] in (cu.SPHERE, cu.HOLLOW_SPHERE):
        hollow = c["shape"] == cu.HOLLOW_SPHERE
        r, th = f(c["dim"][0]), f(c["thickness"])
        dl = np.sqrt((xl * xl).sum(1))
        dist = inv * (np.abs(dl - r) - th) - tolf if hollow else inv * (dl - r) - tolf
        hit = inbox & (dist < 0)
        sgn = np.full(M, inv, f)
        if hollow and mut != "no_hollow_flip":
            flip = dl < r
            sgn = np.where(flip, -inv, inv).astype(f)
            _tag(tags, "analytic_hollow_flip", (hit & flip).sum())
        zero = dl < f(1e-6)
        with np.errstate(invalid="ignore", divide="ignore"):
            n = np.where(zero[:, None], f(0.0), sgn[:, None] * xl / dl[:, None]).astype(f)
        cp = (xl - dist[:, None] * n) if hollow else (r + tolf) * n
        _tag(tags, "analytic_contact", hit.sum()); _tag(tags, "analytic_none", (inbox & ~hit).sum()); _tag(tags, "analytic_n_zero", (hit & zero).sum())
    else:
        xd = xl.astype(np.float64)
        dist = sdf(c, xd, float(tolf)).astype(f)
        hit = inbox & (dist < 0)
        eps = 1e-6
        g = np.zeros((M, 3))
        for j in range(3):
            e = np.zeros(3); e[j] = eps
            if mut == "forward_diff":
                g[:, j] = (sdf(c, xd + e, float(tolf)) - sdf(c, xd, float(tolf))) * (1.0 / eps)
            else:
                g[:, j] = (sdf(c, xd + e, float(tolf)) - sdf(c, xd - e, float(tolf))) * (1.0 / (2.0 * eps))
        n = g.astype(f)
        norm2 = (n * n).sum(1)
        zero = norm2 < f(1e-6)
        with np.errstate(invalid="ignore", divide="ignore"):
            n = np.where(zero[:, None], f(0.0), n / np.sqrt(norm2)[:, None]).astype(f)
        cp = xl - dist[:, None] * n
        _tag(tags, "fd_contact", hit.sum()); _tag(tags, "fd_none", (inbox & ~hit).sum()); _tag(tags, "fd_n_zero", (hit & zero).sum())
    cpw = cp[:, 0:1] * R[0] + cp[:, 1:2] * R[1] + cp[:, 2:3] * R[2] + v2  # R^T cp + v2
    nw = n[:, 0:1] * R[0] + n[:, 1:2] * R[1] + n[:, 2:3] * R[2]
    return hit, cpw.astype(f), nw.astype(f), dist.astype(f)


def _u1(bv, bw, r1, mut):
    if mut == "no_omega":
        return np.broadcast_to(bv, r1.shape)
    w = -bw if mut == "omega_sign" else bw
    return bv + np.cross(np.broadcast_to(w, r1.shape), r1)


def reference(x, v_pre, inv_mass, mass, ranges, colliders, bodies, tol, stiffness, max_iter_v, dtype=np.float64, mut=None, tags=None):
    """What the contact kernel computes for particles x (N, 3) with velocities v_pre (N, 3) after the substeps, against `colliders`
    (contact_util dicts; colliders[k]["body"] indexes bodies = (X, V, W), each (nb, 3)), particle `ranges` [(offset, count, restitution,
    friction)].  Returns (v, contacts, count, impulse): the velocity after contact; the contact list as a structured array (particle,
    collider, cp1, n, dist) in the kernel's order per particle; per collider the contact count and -sum p over the particles with
    mass != 0.  tags: a dict that receives the number of times each branch (BRANCHES_*) was taken."""
    f = dtype
    x = np.asarray(x, f); V = np.array(v_pre, f); w = np.asarray(inv_mass, f); m = np.asarray(mass, f)
    BX, BV, BW = (np.asarray(b, f).reshape(-1, 3) for b in bodies)
    Np, nR = len(x), len(colliders)
    rest, fric, inr = np.zeros(Np, f), np.zeros(Np, f), np.zeros(Np, bool)
    for off, cnt, e, mu in ranges:
        rest[off:off + cnt] = e; fric[off:off + cnt] = mu; inr[off:off + cnt] = True
    live = []
    for k, c in enumerate(colliders):
        b = c["body"]
        hit, cp1, n, dist = detect(x, c, BX[b], tol, f, mut, tags)
        hit &= inr
        r1 = cp1 - BX[b]
        ur = V - _u1(BV[b], BW[b], r1, mut)
        urn = (n * ur).sum(1)
        t = ur - urn[:, None] * n
        tl2 = (t * t).sum(1)
        big = tl2 > f(1e-6)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            t = np.where(big[:, None], t * (f(1.0) / np.sqrt(tl2))[:, None], t).astype(f)
            kd = np.where(w != 0, w, f(0.0)).astype(f)
            nKnInv = (f(1.0) / (kd * (n * n).sum(1))).astype(f)
            pMax = (f(1.0) / (kd * (t * t).sum(1)) * (ur * t).sum(1)).astype(f)
        e = rest * f(c["restitution"])
        approach = urn < 0
        goal = np.where(approach | (mut == "restitution_always"), -e * urn, f(0.0)).astype(f)
        _tag(tags, "init_t_normalised", (hit & big).sum()); _tag(tags, "init_t_unnormalised", (hit & ~big).sum())
        _tag(tags, "init_approach", (hit & approach).sum()); _tag(tags, "init_no_restitution", (hit & ~approach).sum())
        _tag(tags, "static_particle", (hit & (w == 0)).sum())
        live.append(dict(k=k, hit=hit, cp0=x, cp1=cp1, n=n, t=t, nKnInv=nKnInv, pMax=pMax, goal=goal, sum=np.zeros(Np, f),
                         mu=(fric + f(c["friction"])).astype(f), body=b, dist=dist))
    count = np.array([int(L["hit"].sum()) for L in live], np.int64)
    impulse = np.zeros((nR, 3), np.float64)
    solve = np.zeros(Np, bool)
    for L in live:
        solve |= L["hit"]
    solve &= w != 0
    order = live[::-1] if mut == "reverse_order" else live
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for _ in range(max_iter_v):
            for L in order:
                a = L["hit"] & solve
                if not a.any():
                    continue
                n, t, b = L["n"][a], L["t"][a], L["body"]
                d = (n * (L["cp0"][a] - L["cp1"][a])).sum(1)
                r1 = L["cp1"][a] - BX[b]
                ur = V[a] - _u1(BV[b], BW[b], r1, mut)
                urn = (ur * n).sum(1)
                mag = L["nKnInv"][a] * (L["goal"][a] - urn)
                s = L["sum"][a]
                clamp = mag < -s
                if mut != "no_sum_clamp":
                    mag = np.where(clamp, -s, mag)
                pen = d < 0
                mag = np.where(pen, mag - f(stiffness) * L["nKnInv"][a] * d, mag).astype(f)
                p = mag[:, None] * n
                L["sum"][a] = s + mag
                pn = (p * n).sum(1)
                mu, pm = L["mu"][a], L["pMax"][a]
                hi_, lo_ = mu * pn > pm, mu * pn < -pm
                if mut == "friction_swap":
                    ft = np.where(hi_, pm, np.where(lo_, -pm, -mu * pn))
                else:
                    ft = np.where(hi_, -pm, np.where(lo_, pm, -mu * pn))
                p = (p + ft.astype(f)[:, None] * t).astype(f)
                moving = m[a] != 0
                V[np.nonzero(a)[0][moving]] += (w[a][moving, None] * p[moving]).astype(f)
                impulse[L["k"]] -= p[moving].astype(np.float64).sum(0)
                _tag(tags, "sum_clamp", (clamp).sum()); _tag(tags, "penalty", pen.sum())
                _tag(tags, "friction_hi", hi_.sum()); _tag(tags, "friction_lo", (lo_ & ~hi_).sum()); _tag(tags, "friction_cone", (~hi_ & ~lo_).sum())
    rec = []
    for i in range(Np):
        for L in live:
            if L["hit"][i]:
                rec.append((i, L["k"], L["cp1"][i], L["n"][i], L["dist"][i]))
    out = np.zeros(len(rec), CONTACT_DTYPE)
    for j, r in enumerate(rec):
        out[j] = r
    return V, out, count, impulse


CONTACT_DTYPE = np.dtype([("particle", "<u4"), ("collider", "<u4"), ("cp1", "<f8", 3), ("n", "<f8", 3), ("dist", "<f8")])


# ---------------------------------------------------------------------------------------------------------------------------------
# the case set
# ---------------------------------------------------------------------------------------------------------------------------------
class Layout:
    """One layout: colliders (dicts, body = index into the body arrays), bodies (bx, bv, bw (nb, 3) float32), particles x (after the
    step), v, mass (float32) and the (shape, class) of each."""

    def __init__(self, name):
        self.name = name
        self.cols, self.bx, self.bv, self.bw = [], [], [], []
        self.x, self.v, self.mass, self.shape, self.cls = [], [], [], [], []

    def add_body(self, x, v, w):
        self.bx.append(np.asarray(x, np.float64)); self.bv.append(np.asarray(v, np.float64)); self.bw.append(np.asarray(w, np.float64))
        return len(self.bx) - 1

    def add(self, x, v, shape, cls, mass=1.0):
        self.x.append(np.asarray(x, np.float64)); self.v.append(np.asarray(v, np.float64)); self.mass.append(mass)
        self.shape.append(shape); self.cls.append(cls)


def _f32(a):
    return np.asarray(a, np.float32)


def _rounded(c):
    """A collider dict with every float field rounded to fp32 (what the engine and the restatement both see)."""
    c = dict(c)
    for k in ("dim", "R", "v1", "v2", "aabb_min", "aabb_max"):
        c[k] = [float(v) for v in _f32(c[k])]
    for k in ("thickness", "restitution", "friction"):
        c[k] = float(np.float32(c[k]))
    return c


def _local(c, xw, com):
    R = np.asarray(c["R"]).reshape(3, 3)
    return (np.asarray(xw) - com) @ R.T + np.asarray(c["v1"])


def _world(c, xl, com):
    R = np.asarray(c["R"]).reshape(3, 3)
    return (np.asarray(xl) - np.asarray(c["v1"])) @ R + com


def _normal(c, xl):
    """fp64 outward normal (world) of the field at local points: central differences."""
    g = np.zeros((len(xl), 3))
    for j in range(3):
        e = np.zeros(3); e[j] = 1e-6
        g[:, j] = (sdf(c, xl + e, 0.0) - sdf(c, xl - e, 0.0)) / 2e-6
    g /= np.maximum(np.linalg.norm(g, axis=1), 1e-300)[:, None]
    return g @ np.asarray(c["R"]).reshape(3, 3)


def _sample(c, rng, pred, count, spread=1.3):
    """`count` local points in the collider's (spread-scaled) local box whose tolerance-free field value s satisfies pred(s, x)."""
    half = cu.half_extents(c["shape"], c["dim"], c["thickness"]) + 0.06
    out = []
    for _ in range(200):
        x = rng.uniform(-1, 1, (4000, 3)) * half * spread
        s = sdf(c, x, 0.0)
        out += list(x[pred(s, x)])
        if len(out) >= count:
            return np.array(out[:count])
    raise RuntimeError("no points for %s" % c)


def _rel_v(rng, n, kind):
    """A relative velocity for solve class `kind` against normal n."""
    t = np.cross(n, rng.normal(size=3)); t /= np.linalg.norm(t)
    a = rng.uniform(0.3, 1.5)
    return {"approach": -a * n + rng.uniform(0, 0.5) * t, "separating": a * n + rng.uniform(0, 0.5) * t, "stick": -a * n + 0.002 * a * t,
            "slide": -a * n + 3.0 * a * t, "normal_only": -a * n + 3e-4 * t}.get(kind, rng.normal(0, 0.5, 3))


def _collider_cases(L, k, rng, per, tol=cu.TOL):
    """The detection and solve cases of collider k of layout L."""
    c = L.cols[k]; b = c["body"]; com = L.bx[b]
    shape = SHAPE_NAMES[c["shape"]]
    inside = lambda s, x: (s < -0.005)
    shell = lambda s, x: (s > 0.002) & (s < tol - 0.002)
    hollow = c["shape"] in (cu.HOLLOW_SPHERE, cu.HOLLOW_BOX)

    def put(xl, cls, vkind=None, mass=1.0, vzero=False):
        xw = _world(c, xl, com)
        nw = _normal(c, xl)
        for i in range(len(xw)):
            u1 = L.bv[b] + np.cross(L.bw[b], xw[i] - com)
            v = np.zeros(3) if vzero else u1 + _rel_v(rng, nw[i], vkind or cls)
            L.add(xw[i], v, shape, cls, mass)

    put(_sample(c, rng, inside, per), "deep")
    put(_sample(c, rng, shell, per), "shell")
    lo, hi = np.asarray(c["aabb_min"]), np.asarray(c["aabb_max"])
    xo = _sample(c, rng, lambda s, x: s > tol + 0.005, 4 * per)
    wo = _world(c, xo, com)
    keep = ~((wo < lo) | (wo > hi)).any(1)
    put(xo[keep][:per], "outside")
    if c["invert"]:  # outside the bounding box, inside the (inverted) field
        for i in range(per):
            p = lo + rng.uniform(0.1, 0.9, 3) * (hi - lo)
            j = i % 3
            p[j] = hi[j] + rng.uniform(0.01, 0.05) if i % 2 else lo[j] - rng.uniform(0.01, 0.05)
            L.add(p, rng.normal(0, 0.3, 3), shape, "aabb_cut")
    dim, th = np.asarray(c["dim"], np.float64), float(c["thickness"])
    if c["shape"] in (cu.BOX, cu.HOLLOW_BOX, cu.CYLINDER):
        pts = []
        for _ in range(per):
            sg = rng.choice([-1.0, 1.0], 3)
            off = rng.uniform(1e-4, 0.015, 3) * rng.choice([-1.0, 1.0], 3)
            if c["shape"] == cu.BOX:
                p = sg * dim + off
                if rng.uniform() < 0.5:  # an edge instead of a corner
                    j = rng.integers(3); p[j] = rng.uniform(-0.8, 0.8) * dim[j]
            elif c["shape"] == cu.HOLLOW_BOX:  # the edges of the inner wall
                p = sg * (dim - th) + off
                j = rng.integers(3); p[j] = rng.uniform(-0.5, 0.5) * dim[j]
            else:  # the cylinder's rim
                a = rng.uniform(0, 2 * np.pi)
                rr = dim[0] + off[0]
                p = np.array([rr * np.cos(a), sg[1] * dim[1] + off[1], rr * np.sin(a)])
            pts.append(p)
        pts = np.array(pts)
        pts = pts[sdf(c, pts, 0.0) < tol - 0.002]
        put(pts, "crease")
    if c["shape"] in (cu.TORUS, cu.CYLINDER):
        ys = rng.uniform(0.5, 0.95, per) * (dim[1] if c["shape"] == cu.CYLINDER else 1.5 * dim[1] + dim[0]) * rng.choice([-1.0, 1.0], per)
        if c["shape"] == cu.TORUS and not c["invert"]:
            ys = ys * 0.5
        # near the axis, at least 1e-4 from it: closer than eps = 1e-6 the normal is set by the fp32 rounding of the local transform
        a, rr = rng.uniform(0, 2 * np.pi, per), rng.uniform(1e-4, 1e-3, per)
        put(np.stack([rr * np.cos(a), ys, rr * np.sin(a)], 1), "axis")
    if hollow:
        inner = (lambda s, x: (s < -0.002) & (np.linalg.norm(x, axis=1) < dim[0])) if c["shape"] == cu.HOLLOW_SPHERE else \
            (lambda s, x: (s < -0.002) & (sdf(dict(c, shape=cu.BOX, invert=False), x, 0.0) < 0))
        outer = (lambda s, x: (s < -0.002) & (np.linalg.norm(x, axis=1) > dim[0])) if c["shape"] == cu.HOLLOW_SPHERE else \
            (lambda s, x: (s < -0.002) & (sdf(dict(c, shape=cu.BOX, invert=False), x, 0.0) > 0))
        put(_sample(c, rng, inner, per), "hollow_in")
        put(_sample(c, rng, outer, per), "hollow_out")
    for kind in ("approach", "separating", "stick", "slide", "normal_only"):
        put(_sample(c, rng, inside if kind != "separating" else shell, per), kind)
    if not (L.bv[b].any() or L.bw[b].any()):
        put(_sample(c, rng, inside, per), "tangent_zero", vzero=True)
    else:
        put(_sample(c, rng, inside, per), "moving_body", vkind="approach")
    put(_sample(c, rng, inside, per), "static_particle", vkind="approach", mass=0.0)


def _frame(rng):
    return cu.rotation(rng.normal(size=3), rng.uniform(0.3, 1.2))


def _dims(shape, s):
    return {cu.BOX: (s, 0.6 * s, 0.8 * s), cu.SPHERE: (s,), cu.TORUS: (s, 0.35 * s), cu.CYLINDER: (0.6 * s, s),
            cu.HOLLOW_SPHERE: (s,), cu.HOLLOW_BOX: (s, 0.7 * s, 0.9 * s)}[shape]


def layout_S(rng, per):
    L = Layout("S")
    for j in range(6):
        centre = np.array([6.0 * j - 15.0, 0.0, 2.0])
        moving = j % 2 == 1
        b = L.add_body(centre, rng.normal(0, 0.4, 3) if moving else np.zeros(3), rng.normal(0, 0.8, 3) if moving else np.zeros(3))
        rot = np.eye(3) if j in (cu.BOX, cu.SPHERE) else _frame(rng)
        L.cols.append(cu.collider(j, _dims(j, 1.0), centre, rot, thickness=0.15 if j in (cu.HOLLOW_SPHERE, cu.HOLLOW_BOX) else 0.0,
                                  restitution=rng.uniform(0.2, 0.9), friction=rng.uniform(0.05, 0.4), body=b))
    # two colliders on one body, overlapping: between them the normals oppose (wedge)
    b = L.add_body([0.0, 8.0, 0.0], rng.normal(0, 0.4, 3), rng.normal(0, 0.8, 3))
    L.cols.append(cu.collider(cu.SPHERE, (0.8,), [-0.5, 8.0, 0.0], _frame(rng), restitution=0.4, friction=0.2, body=b))
    L.cols.append(cu.collider(cu.BOX, (0.7, 0.5, 0.6), [0.6, 8.0, 0.0], cu.rotation((0.0, 0.0, 1.0), 0.2), restitution=0.7, friction=0.15, body=b))
    for c in L.cols[6:]:  # off the centre of mass: x_local = R (x - com) + v1 with v1 = R (com - centre)
        c["v1"] = (np.asarray(c["R"]).reshape(3, 3) @ (L.bx[b] - np.asarray(c["v2"]))).tolist()
    L.cols = [_rounded(c) for c in L.cols]
    for k in range(6):
        _collider_cases(L, k, rng, per)
    com = L.bx[b]
    for k in (6, 7):
        c = L.cols[k]
        xl = _sample(c, rng, lambda s, x: s < -0.005, 2 * per)
        xw = _world(c, xl, com)
        for i in range(len(xw)):
            u1 = L.bv[b] + np.cross(L.bw[b], xw[i] - com)
            L.add(xw[i], u1 + rng.normal(0, 0.5, 3), "shared", "shared_body")
    # wedge: inside both, approaching the sphere and separating from the box; the sphere's impulse then drives the particle into the
    # box, whose goal must stay 0 (restitution only where the contact began approaching)
    sph6, box7 = L.cols[6], L.cols[7]
    xl = _sample(sph6, rng, lambda s, x: s < -0.005, 40 * per)
    xw = _world(sph6, xl, com)
    inside7 = sdf(box7, _local(box7, xw, com), 0.0) < -0.005
    xw, xl = xw[inside7], xl[inside7]
    n6, n7 = _normal(sph6, xl), _normal(box7, _local(box7, xw, com))
    got = 0
    for i in range(len(xw)):
        ur = -rng.uniform(0.3, 1.0) * n6[i]
        if got < 2 * per and ur @ n7[i] > 0.05:
            L.add(xw[i], L.bv[b] + np.cross(L.bw[b], xw[i] - com) + ur, "shared", "wedge")
            got += 1
    assert got == 2 * per, got
    # at threshold: the box (axis-aligned, at rest) and the sphere (axis-aligned) of S
    box, sph = L.cols[cu.BOX], L.cols[cu.SPHERE]
    cb, cs = L.bx[box["body"]], L.bx[sph["body"]]
    d = np.asarray(box["dim"], np.float64)
    for i in range(per):
        # grazing: on the tolerance surface of a face, |dist| < 1e-6; v tangent to the face keeps the coordinate exact
        j = i % 3
        p = rng.uniform(-0.7, 0.7, 3) * d; p[j] = float(np.float32(d[j] + cu.TOL)) * (1 if i % 2 else -1)
        v = rng.normal(0, 0.5, 3); v[j] = 0.0
        L.add(cb + p, v, "box", "grazing")
        # on the crease: within eps of an edge
        q = np.sign(rng.normal(size=3)) * d + rng.uniform(-5e-7, 5e-7, 3)
        L.add(cb + q, np.zeros(3), "box", "on_crease")
    L.add(cb, np.zeros(3), "box", "degenerate_normal")
    L.add(cs, np.zeros(3), "sphere", "degenerate_normal")
    L.add(cs, np.zeros(3), "sphere", "degenerate_normal", mass=0.0)
    return L


def layout_I(rng, per):
    L = Layout("I")
    for j in range(6):
        centre = np.array([7.0 * j - 18.0, -6.0, -3.0])
        moving = j % 2 == 0
        b = L.add_body(centre, rng.normal(0, 0.4, 3) if moving else np.zeros(3), rng.normal(0, 0.8, 3) if moving else np.zeros(3))
        L.cols.append(cu.collider(j, _dims(j, 1.2), centre, _frame(rng), thickness=0.2 if j in (cu.HOLLOW_SPHERE, cu.HOLLOW_BOX) else 0.0,
                                  invert=True, restitution=rng.uniform(0.2, 0.9), friction=rng.uniform(0.05, 0.4), body=b))
    for shift, shape, cls in ((1e2, cu.BOX, "shift1e2"), (1e3, cu.TORUS, "shift1e3")):
        centre = np.array([shift, shift * 0.5, -shift])
        b = L.add_body(centre, rng.normal(0, 0.4, 3), rng.normal(0, 0.8, 3))
        L.cols.append(cu.collider(shape, _dims(shape, 1.0), centre, _frame(rng), restitution=0.5, friction=0.25, body=b))
    L.cols = [_rounded(c) for c in L.cols]
    for k in range(6):
        _collider_cases(L, k, rng, per)
    for k, cls in ((6, "shift1e2"), (7, "shift1e3")):
        c = L.cols[k]; com = L.bx[c["body"]]
        xl = _sample(c, rng, lambda s, x: s < cu.TOL - 0.005, 2 * per)
        xw = _world(c, xl, com)
        for i in range(len(xw)):
            L.add(xw[i], L.bv[c["body"]] + np.cross(L.bw[c["body"]], xw[i] - com) + rng.normal(0, 0.5, 3), SHAPE_NAMES[c["shape"]], cls)
    # at threshold: exactly on a face of the inverted box's bounding box (the velocity along that axis is zero)
    c = L.cols[cu.BOX]
    lo, hi = np.asarray(c["aabb_min"], np.float64), np.asarray(c["aabb_max"], np.float64)
    for i in range(per):
        j = i % 3
        p = lo + rng.uniform(0.05, 0.95, 3) * (hi - lo); p[j] = hi[j] if i % 2 else lo[j]
        v = rng.normal(0, 0.5, 3); v[j] = 0.0
        L.add(p, v, "box", "aabb_face")
    return L


def layout_M(rng, per):
    L = Layout("M")
    centre = np.array([0.0, 20.0, 0.0])
    rho = [1.2 * 1.6 ** j for j in range(8)]
    shapes = [cu.SPHERE, cu.CYLINDER, cu.SPHERE, cu.CYLINDER, cu.SPHERE, cu.CYLINDER, cu.BOX, cu.BOX]
    for j in range(8):
        moving = j % 3 == 1
        b = L.add_body(centre, rng.normal(0, 0.05, 3) if moving else np.zeros(3), rng.normal(0, 0.05, 3) if moving else np.zeros(3))
        dim = {cu.SPHERE: (rho[j],), cu.CYLINDER: (rho[j], rho[j]), cu.BOX: (rho[j],) * 3}[shapes[j]]
        L.cols.append(cu.collider(shapes[j], dim, centre, _frame(rng), restitution=rng.uniform(0.2, 0.9), friction=rng.uniform(0.05, 0.4), body=b))
    L.cols = [_rounded(c) for c in L.cols]
    for k in range(2, 9):  # inside colliders 8-k .. 7, outside 0 .. 7-k (with their corners)
        lo = (rho[7 - k] * np.sqrt(2.0) + 2 * cu.TOL) if k < 8 else 0.05
        hi = rho[8 - k] - 0.1
        for i in range(per):
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            xw = centre + d * rng.uniform(lo, hi)
            # mostly along the normals: the other contacts of the particle then pull a contact's impulse below zero (friction_lo)
            L.add(xw, -rng.uniform(0.3, 1.0) * d + rng.normal(0, 0.01, 3), "multi", "multi%d" % k)
    return L


def _finish(L, rng):
    """Unranged particles at the front, padding far away; x_pre = x - v dt; fp32."""
    n_case = len(L.x)
    assert n_case + UNRANGED <= N, (L.name, n_case)
    # unranged: inside a collider, moving, but outside every particle range
    c = L.cols[0]; com = L.bx[c["body"]]
    xu = _world(c, _sample(c, rng, lambda s, x: (s < -0.005) if not c["invert"] else (s < cu.TOL - 0.005), UNRANGED), com)
    xs = list(xu) + L.x
    vs = [rng.normal(0, 0.5, 3) for _ in range(UNRANGED)] + L.v
    ms = [1.0] * UNRANGED + L.mass
    sh = ["range"] * UNRANGED + L.shape
    cl = ["unranged"] * UNRANGED + L.cls
    # padding, far from every collider: the same particles in every layout (the replicas of a batch share the constraints on them)
    pad = np.random.default_rng(99)
    px, pv, pm = np.array([500.0, -500.0, 500.0]) + pad.uniform(-1, 1, (N, 3)), pad.normal(0, 0.5, (N, 3)), pad.uniform(0.2, 3.0, N)
    n_case = len(xs)
    xs += list(px[n_case:]); vs += list(pv[n_case:]); ms += [1.0] * (N - n_case)
    sh += ["none"] * (N - n_case); cl += ["pad"] * (N - n_case)
    x = np.array(xs); v = np.array(vs)
    mass = np.array(ms)
    # particles in the ranges get random masses (static ones stay 0)
    mass = np.where(mass != 0, rng.uniform(0.2, 3.0, N), 0.0)
    mass[n_case:] = pm[n_case:]
    L.x, L.v, L.mass = _f32(x), _f32(v), _f32(mass)
    L.x_pre = _f32(np.where(mass[:, None] != 0, x - v * DT, x))  # static particles do not move
    L.shape, L.cls = np.array(sh), np.array(cl)
    L.bx, L.bv, L.bw = _f32(L.bx), _f32(L.bv), _f32(L.bw)
    return L


def make_layouts(per=4, seed=2024):
    rng = np.random.default_rng(seed)
    return [_finish(f(rng, per), rng) for f in (layout_S, layout_I, layout_M)]


def inv_mass(mass):
    m = np.asarray(mass, np.float32)
    return np.where(m != 0, np.float32(1.0) / np.where(m != 0, m, np.float32(1.0)), np.float32(0.0)).astype(np.float32)


def run_reference(L, x, v_pre, config, dtype=np.float64, mut=None, tags=None):
    tol, stiff, iters, _ = config
    return reference(np.asarray(x, np.float64 if dtype == np.float64 else np.float32), v_pre, inv_mass(L.mass), L.mass, RANGES, L.cols,
                     (L.bx, L.bv, L.bw), np.float32(tol), np.float32(stiff), iters, dtype=dtype, mut=mut, tags=tags)


# ---------------------------------------------------------------------------------------------------------------------------------
# the gate
# ---------------------------------------------------------------------------------------------------------------------------------
def velocity_errors(v_got, v_ref, v_pre):
    """Per particle: |v_got - v_ref| relative to max(|v_ref - v_pre|, 1e-3 m/s) plus 16 fp32 ulps of |v_ref|; NaN where either is
    non-finite (the degenerate normals, compared by their non-finite set instead)."""
    v_got, v_ref, v_pre = (np.asarray(a, np.float64) for a in (v_got, v_ref, v_pre))
    scale = np.maximum(np.linalg.norm(v_ref - v_pre, axis=1), 1e-3) + 16.0 * float(np.spacing(np.float32(1.0))) * np.linalg.norm(v_ref, axis=1)
    with np.errstate(invalid="ignore"):
        return np.linalg.norm(v_got - v_ref, axis=1) / scale


def gated(L):
    """The particles held to TOL: every class but the at-threshold ones."""
    return ~np.isin(L.cls, THRESHOLD)


def finite_sets_agree(v_got, v_ref):
    return np.array_equal(np.isfinite(v_got).all(1), np.isfinite(v_ref).all(1))


def velocity_gate(L, v_got, x, v_pre, config, mut=None):
    """The velocity gate of v_got (the kernel's velocities after contact, from x and v_pre) against reference(mut): per (shape, class) of
    L, (key, worst error, limit).  Gated classes: velocity_errors within TOL.  At-threshold classes: within 4x the fp32 restatement's own
    error (at least TOL_DEFAULT), so that the inputs, not the kernel, set the error; the degenerate normals: the same particles
    non-finite as the restatement (error 0 or inf, limit 0)."""
    v_ref = run_reference(L, x, v_pre, config, mut=mut)[0]
    e = velocity_errors(v_got, v_ref, v_pre)
    e32 = None
    out = []
    for key in sorted(set(zip(L.shape.tolist(), L.cls.tolist()))):
        sel = (L.shape == key[0]) & (L.cls == key[1])
        if key[1] == "degenerate_normal":
            out.append((key, 0.0 if finite_sets_agree(v_got[sel], v_ref[sel]) else np.inf, 0.0))
            continue
        worst = float(np.max(e[sel])) if np.isfinite(e[sel]).all() else np.inf
        if key[1] in THRESHOLD:
            if e32 is None:
                e32 = velocity_errors(run_reference(L, x, v_pre, config, dtype=np.float32, mut=mut)[0], v_ref, v_pre)
            out.append((key, worst, max(4.0 * float(np.nanmax(e32[sel])), TOL_DEFAULT)))
        else:
            out.append((key, worst, tol(*key)))
    return out


def sensor_errors(count_got, impulse_got, count_ref, impulse_ref):
    """(counts equal, non-finite colliders the same, worst impulse error relative to max(|sum|, 1e-2))."""
    fin = np.isfinite(impulse_ref).all(1)
    same_fin = np.array_equal(np.isfinite(impulse_got).all(1), fin)
    imp = np.asarray(impulse_got, np.float64)
    err = np.abs(imp[fin] - impulse_ref[fin]).max(1) / np.maximum(np.abs(impulse_ref[fin]).max(1), 1e-2) if fin.any() else np.zeros(1)
    return np.array_equal(np.asarray(count_got), np.asarray(count_ref)), same_fin, float(err.max())


def without_degenerate(L):
    """L with the degenerate-normal particles static: their contacts are recorded and counted but not solved, so every collider's
    impulse stays finite and the sensors can be compared on every collider."""
    import copy
    M = copy.copy(L)
    M.mass = np.where(L.cls == "degenerate_normal", np.float32(0.0), L.mass).astype(np.float32)
    return M


# (shape, class): (velocity threshold of the gate (velocity_errors), worst measured), for every gated (shape, class) of the case set.
# Measured over every path and configuration on an H100 80GB HBM3 at its 700 W power limit and by the host build of the kernel
# (test_contact_cases.py), the larger of the two; thresholds 3x that worst (two significant digits, rounded up; an exact zero stays zero).
# normal_only: the tangent is left unnormalised (tl2 <= 1e-6), so pMax and the friction impulse come from a difference of nearly equal
# fp32 velocities; shift1e3: positions near 1e3 m carry fp32 ulps of 6e-5 m into the normals.  The at-threshold classes (THRESHOLD) are
# held to the fp32 restatement instead (H100 worst: grazing 7.8e-2, on_crease 7.9e-6, aabb_face 2.9e-6).
TOL_MEASURED = {
    ('box', 'aabb_cut'): (0, 0.00e+00),
    ('box', 'approach'): (3.5e-05, 1.14e-05),
    ('box', 'crease'): (0.00027, 8.94e-05),
    ('box', 'deep'): (3.1e-05, 1.01e-05),
    ('box', 'moving_body'): (2e-05, 6.48e-06),
    ('box', 'normal_only'): (3e-05, 9.87e-06),
    ('box', 'outside'): (0, 0.00e+00),
    ('box', 'separating'): (0.00099, 3.27e-04),
    ('box', 'shell'): (0.00014, 4.49e-05),
    ('box', 'shift1e2'): (0.00073, 2.43e-04),
    ('box', 'slide'): (2.6e-05, 8.64e-06),
    ('box', 'static_particle'): (0, 0.00e+00),
    ('box', 'stick'): (0.00022, 7.08e-05),
    ('box', 'tangent_zero'): (5e-06, 1.65e-06),
    ('cylinder', 'aabb_cut'): (0, 0.00e+00),
    ('cylinder', 'approach'): (1.1e-05, 3.52e-06),
    ('cylinder', 'axis'): (2.4e-06, 7.85e-07),
    ('cylinder', 'crease'): (9e-05, 2.99e-05),
    ('cylinder', 'deep'): (1.3e-05, 4.30e-06),
    ('cylinder', 'moving_body'): (2e-06, 6.63e-07),
    ('cylinder', 'normal_only'): (0.009, 2.98e-03),
    ('cylinder', 'outside'): (0, 0.00e+00),
    ('cylinder', 'separating'): (0.00015, 4.70e-05),
    ('cylinder', 'shell'): (3.8e-05, 1.26e-05),
    ('cylinder', 'slide'): (2.1e-05, 6.88e-06),
    ('cylinder', 'static_particle'): (0, 0.00e+00),
    ('cylinder', 'stick'): (0.00014, 4.65e-05),
    ('cylinder', 'tangent_zero'): (2.5e-05, 8.26e-06),
    ('hollow_box', 'aabb_cut'): (0, 0.00e+00),
    ('hollow_box', 'approach'): (1.1e-05, 3.60e-06),
    ('hollow_box', 'crease'): (0.00071, 2.36e-04),
    ('hollow_box', 'deep'): (4.5e-05, 1.50e-05),
    ('hollow_box', 'hollow_in'): (9.5e-06, 3.15e-06),
    ('hollow_box', 'hollow_out'): (3.9e-05, 1.28e-05),
    ('hollow_box', 'moving_body'): (2.6e-05, 8.52e-06),
    ('hollow_box', 'normal_only'): (0.0012, 3.91e-04),
    ('hollow_box', 'outside'): (0, 0.00e+00),
    ('hollow_box', 'separating'): (0.00027, 8.86e-05),
    ('hollow_box', 'shell'): (5.7e-05, 1.87e-05),
    ('hollow_box', 'slide'): (2.6e-05, 8.45e-06),
    ('hollow_box', 'static_particle'): (0, 0.00e+00),
    ('hollow_box', 'stick'): (8.4e-05, 2.79e-05),
    ('hollow_box', 'tangent_zero'): (4.2e-06, 1.38e-06),
    ('hollow_sphere', 'aabb_cut'): (0, 0.00e+00),
    ('hollow_sphere', 'approach'): (2.3e-05, 7.58e-06),
    ('hollow_sphere', 'deep'): (2.1e-05, 6.95e-06),
    ('hollow_sphere', 'hollow_in'): (7.2e-05, 2.38e-05),
    ('hollow_sphere', 'hollow_out'): (2.6e-05, 8.61e-06),
    ('hollow_sphere', 'moving_body'): (4.1e-05, 1.35e-05),
    ('hollow_sphere', 'normal_only'): (0.0049, 1.62e-03),
    ('hollow_sphere', 'outside'): (0, 0.00e+00),
    ('hollow_sphere', 'separating'): (0.00013, 4.18e-05),
    ('hollow_sphere', 'shell'): (3.3e-05, 1.09e-05),
    ('hollow_sphere', 'slide'): (0.0001, 3.32e-05),
    ('hollow_sphere', 'static_particle'): (0, 0.00e+00),
    ('hollow_sphere', 'stick'): (0.00019, 6.12e-05),
    ('hollow_sphere', 'tangent_zero'): (9.6e-06, 3.19e-06),
    ('multi', 'multi2'): (1.8e-06, 5.79e-07),
    ('multi', 'multi3'): (8.5e-07, 2.82e-07),
    ('multi', 'multi4'): (1.1e-06, 3.46e-07),
    ('multi', 'multi5'): (4.8e-06, 1.60e-06),
    ('multi', 'multi6'): (4.5e-05, 1.48e-05),
    ('multi', 'multi7'): (2.1e-06, 6.99e-07),
    ('multi', 'multi8'): (6.5e-05, 2.15e-05),
    ('none', 'pad'): (0, 0.00e+00),
    ('range', 'unranged'): (0, 0.00e+00),
    ('shared', 'shared_body'): (5.4e-05, 1.80e-05),
    ('shared', 'wedge'): (4.8e-06, 1.60e-06),
    ('sphere', 'aabb_cut'): (0, 0.00e+00),
    ('sphere', 'approach'): (3.7e-06, 1.22e-06),
    ('sphere', 'deep'): (5.3e-05, 1.75e-05),
    ('sphere', 'moving_body'): (3e-06, 9.75e-07),
    ('sphere', 'normal_only'): (9.3e-06, 3.07e-06),
    ('sphere', 'outside'): (0, 0.00e+00),
    ('sphere', 'separating'): (0.00025, 8.06e-05),
    ('sphere', 'shell'): (1.7e-05, 5.66e-06),
    ('sphere', 'slide'): (2.7e-06, 8.72e-07),
    ('sphere', 'static_particle'): (0, 0.00e+00),
    ('sphere', 'stick'): (0.00025, 8.15e-05),
    ('sphere', 'tangent_zero'): (7.4e-07, 2.46e-07),
    ('torus', 'aabb_cut'): (0, 0.00e+00),
    ('torus', 'approach'): (4.7e-06, 1.54e-06),
    ('torus', 'axis'): (0, 0.00e+00),
    ('torus', 'deep'): (1.7e-05, 5.38e-06),
    ('torus', 'moving_body'): (1.1e-05, 3.56e-06),
    ('torus', 'normal_only'): (0.014, 4.65e-03),
    ('torus', 'outside'): (0, 0.00e+00),
    ('torus', 'separating'): (6.2e-05, 2.04e-05),
    ('torus', 'shell'): (0.00012, 3.67e-05),
    ('torus', 'shift1e3'): (0.0082, 2.73e-03),
    ('torus', 'slide'): (3.6e-06, 1.20e-06),
    ('torus', 'static_particle'): (0, 0.00e+00),
    ('torus', 'stick'): (0.00011, 3.59e-05),
    ('torus', 'tangent_zero'): (9.9e-06, 3.28e-06),
}
TOL = {k: t for k, (t, _) in TOL_MEASURED.items()}
TOL_DEFAULT = 1e-3  # the floor of the at-threshold classes' fp32-conditioning bound (velocity_gate)


TOL_RECORDS = 2e-4   # cp1 relative to max(|cp1|, 1 m), n absolute, dist relative to max(|dist|, 1e-3 m); H100 worst 6.6e-5
TOL_SENSORS = 2.8e-3  # impulse relative to max(|sum|, 1e-2); worst 9.2e-4 (H100), 7.9e-4 (host build)


def tol(shape, cls):
    """The velocity threshold of a gated (shape, class)."""
    return TOL[(str(shape), str(cls))]
