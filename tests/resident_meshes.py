"""Mesh scenes for the resident kernel, one per type mask, on the builder surface of tests/scenes.py (so that the host model mirror and the
CPU checkers build identical models), and the cluster shapes they run in.  Unlike the separated stencils of tests/projection_cases.py,
every constraint here shares particles with constraints of other colours and types, so a resident item that reads a particle before an
earlier colour's store to it is visible changes the answer.  Each scene comes in two sizes: a small one of about 2,000-2,600 particles,
which fits one CTA, and a large one of 20,000-23,000 particles, whose tiles at 2x1 hold slots above 8,191, close to a tile's capacity.

Used by tests/test_resident_meshes_plan.py (the plans, on the CPU) and tests/test_gpu_resident_meshes.py (the kernel against the launch
mode, bit for bit)."""
import numpy as np

import scenes

VOLUME, VOLUME_XPBD = 7, 8
FEMTET_XPBD = 10
BALLJOINT, RB_PARTICLE_BALLJOINT = 13, 14
# the type masks of csrc/device_image.h
_B = lambda *ts: sum(1 << t for t in ts)
MASK_CLOTH_XPBD = _B(1, 4)
MASK_CLOTH = MASK_CLOTH_XPBD | _B(0, 3)
MASK_LIGHT = _B(0, 1, 2, 3, 4, 5, 7, 8)
MASK_FEM = _B(7, 8, 9, 10)
MASK_SOLID = MASK_CLOTH | MASK_FEM | _B(5, 13, 14)
MASK_ALL = (1 << 15) - 1

# cluster shapes, "GxC" as PBD_B200_CLUSTERS takes them; "default": the planner's own choice
REGIMES = ["1x1", "1x2", "1x4", "1x16", "2x1", "7x1", "37x1", "default"]
SIZES = ["small", "large"]


def regimes(size):
    """The regimes a scene of `size` runs in: a large scene does not fit one CTA."""
    return [r for r in REGIMES if not (size == "large" and r == "1x1")]


def shape(regime):
    """(G, C) forced by `regime`, (0, 0) for the planner's default."""
    return (0, 0) if regime == "default" else tuple(int(v) for v in regime.split("x"))


def independent(regime):
    """Independent CTAs (G > 1): the X items and the neighbour flags.  Every other regime is one cluster (the default is one for every
    scene here: none exceeds what 16 CTAs hold)."""
    return shape(regime)[0] > 1


SPAN = 5.0  # every model spans x in [0, SPAN]: the planner bisects along x first, so every model is cut into every tile


class _Placer:
    """Lays models out over one region, cloths above one another and bars side by side in z, and keeps the particle offset of each
    (models are numbered per kind, particles in creation order)."""
    def __init__(self, m):
        self.m, self.n, self.tri, self.tet = m, 0, 0, 0

    def cloth(self, nx, cloth_method, bending_methods, dist_k=1.0e5, bend_k=(100.0,), fem=(1000.0, 1000.0, 500.0, 0.3, 0.3)):
        """nx x nx sheet in the x-z plane, two corners pinned."""
        m, off, tm = self.m, self.n, self.tri
        m.add_regular_triangle_model(nx, nx, t=(0.0, 2.0 + 0.3 * tm, 0.0), R=scenes.RX90, scale=(SPAN, SPAN))
        m.set_mass(off, 0.0); m.set_mass(off + nx - 1, 0.0)
        m.add_cloth_constraints(tm, cloth_method, dist_k=dist_k, xx=fem[0], yy=fem[1], xy=fem[2], pxy=fem[3], pyx=fem[4])
        for b, k in zip(bending_methods, bend_k):
            m.add_bending_constraints(tm, b, k)
        self.n += nx * nx; self.tri += 1
        return off

    def bar(self, dims, solid_method, k, vol_k=1.0, extra=None, extra_k=1.0):
        """dims[0] x dims[1] x dims[2] tet bar along x, its first slab pinned; `extra`: one more constraint of that type per tet."""
        m, off, tm = self.m, self.n, self.tet
        w, h, d = dims
        m.add_regular_tet_model(w, h, d, t=(0.0, 0.0, 0.8 * tm), R=np.eye(3), scale=(SPAN, SPAN * h / w, SPAN * d / w))
        for i in range(h * d):
            m.set_mass(off + i, 0.0)
        m.add_solid_constraints(tm, solid_method, k=k, nu=0.3, vol_k=vol_k)
        if extra is not None:
            for t in m.tet_tets(tm):
                m.add_constraint(extra, [int(v) + off for v in t], [extra_k])
        self.n += w * h * d; self.tet += 1
        return off


# per scene: (small, large) sizes
_CLOTH_XPBD = {"small": 50, "large": 150}
_CLOTH = {"small": 36, "large": 106}
_LIGHT = {"small": (30, (12, 5, 5)), "large": (100, (20, 8, 8))}
_FEM = {"small": (20, 8, 8), "large": (40, 16, 16)}
_SOLID = {"small": (40, (12, 6, 6)), "large": (140, (20, 8, 8))}
_ALL = {"small": (20, (9, 4, 4)), "large": (80, (16, 6, 6))}


def cloth_xpbd(m, size):
    """ClothXPBD: an XPBD cloth (Distance_XPBD + IsometricBending_XPBD)."""
    _Placer(m).cloth(_CLOTH_XPBD[size], 4, (3,))
    m.set_params(dt=0.005, sub_steps=1, max_iter=5)


def cloth(m, size):
    """Cloth: a PBD cloth (Distance + IsometricBending) and an XPBD cloth, in one model."""
    p = _Placer(m)
    p.cloth(_CLOTH[size], 1, (2,), dist_k=1.0, bend_k=(0.5,))
    p.cloth(_CLOTH[size], 4, (3,))
    m.set_params(dt=0.005, sub_steps=1, max_iter=5)


def light(m, size):
    """Light: a FEMTriangle + Dihedral cloth, a Distance + IsometricBending_XPBD + IsometricBending cloth, and a Distance_XPBD +
    Volume_XPBD bar with a Volume constraint on every tet: every type of the light mask."""
    n, dims = _LIGHT[size]
    p = _Placer(m)
    p.cloth(n, 2, (1,), bend_k=(0.5,))
    p.cloth(n, 1, (3, 2), dist_k=1.0, bend_k=(100.0, 0.5))
    p.bar(dims, 6, k=1.0e5, vol_k=1.0e5, extra=VOLUME, extra_k=1.0)
    m.set_params(dt=0.005, sub_steps=2, max_iter=3)


def fem(m, size):
    """Fem: a FEMTet bar (solid method 2) with a Volume constraint per tet and a FEMTet_XPBD bar (method 3, E = 1e4) with a Volume_XPBD
    constraint per tet."""
    p = _Placer(m)
    p.bar(_FEM[size], 2, k=1.0e6, extra=VOLUME, extra_k=1.0)
    p.bar(_FEM[size], 3, k=1.0e4, extra=VOLUME_XPBD, extra_k=1.0e4)
    m.set_params(dt=0.005, sub_steps=2, max_iter=3)


def solid(m, size, rig=False):
    """Solid: a FEMTriangle + IsometricBending cloth and a FEMTet bar in one model, plus the rigid coupling rig with `rig` (BallJoint and
    RigidBodyParticleBallJoint, their particles the cloth's corners; the planner admits joints in one cluster only)."""
    n, dims = _SOLID[size]
    p = _Placer(m)
    p.cloth(n, 2, (2,), bend_k=(0.01,))
    p.bar(dims, 2, k=1.0e6)
    if rig:
        scenes.coupling_rig(m, n, n)
    m.set_params(dt=0.005, sub_steps=2, max_iter=3)


def all_types(m, size):
    """All: cloths of methods 2, 3 and 4 with the three bending methods, and bars of solid methods 1 to 6 (FEMTet_XPBD at E = 1e4), every
    mesh its own particle range: every particle constraint type."""
    n, dims = _ALL[size]
    p = _Placer(m)
    p.cloth(n, 2, (1,), bend_k=(0.5,))
    p.cloth(n, 3, (2,), bend_k=(0.5,), fem=(1.0, 1.0, 1.0, 0.3, 0.3))
    p.cloth(n, 4, (3,))
    for method, k, vol_k in ((1, 1.0, 1.0), (2, 1.0e6, 1.0), (3, 1.0e4, 1.0), (4, 1.0, 1.0), (5, 0.5, 1.0), (6, 1.0e5, 1.0e5)):
        p.bar(dims, method, k=k, vol_k=vol_k)
    m.set_params(dt=0.005, sub_steps=2, max_iter=3)


SCENES = {  # name: (builder(m, size), the mask the planner must choose)
    "cloth_xpbd": (cloth_xpbd, MASK_CLOTH_XPBD),
    "cloth": (cloth, MASK_CLOTH),
    "light": (light, MASK_LIGHT),
    "fem": (fem, MASK_FEM),
    "solid": (solid, MASK_SOLID),
    "all": (all_types, MASK_ALL),
}


def has_rig(name, regime):
    """The solid scene carries the coupling rig in the one-cluster regimes."""
    return name == "solid" and not independent(regime)


def builder(name, size, rig=False):
    build = SCENES[name][0]
    if rig:
        return lambda m: build(m, size, rig=True)
    return lambda m: build(m, size)


def xpbd_fem(name):
    """Scenes with FEMTet_XPBD: held to the fp64 checker after one step (DESIGN.md section 5)."""
    return name in ("fem", "all")


def flat(name, size, rig=False, amplitude=0.01):
    """Scene (name, size) from the host model mirror as flat arrays, its particles perturbed by parity_util.perturb (pinned ones stay):
    constraints, groups, x (perturbed), x0, masses, parameters and, with `rig`, the rig's bodies."""
    from parity_util import perturb
    from positionbaseddynamics_b200.model import HostModel
    hm = HostModel()
    builder(name, size, rig)(hm)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x = perturb([hm], amplitude)
    p = hm._params
    out = dict(name=name, size=size, types=np.asarray(types).copy(), bodies=np.asarray(bodies).copy(), params=np.asarray(params, np.float32).copy(),
               off=np.asarray(off).copy(), ids=np.asarray(ids).copy(), x=np.asarray(x, np.float32).copy(),
               x0=np.asarray(hm.get("x0"), np.float32).copy(), mass=np.asarray(mass, np.float32).copy(), dt=p["dt"], sub=p["sub_steps"], it=p["max_iter"])
    if rig:
        rb = hm.rigid_bodies().copy()
        anchor, box = scenes.box_inertia(1.0, 0.5, 0.5, 0.5), scenes.box_inertia(1.0, 0.4, 2.0, 0.4)
        out.update(bm=np.float32([0.0, 1.0, 1.0] * 4), bI=np.float32([anchor, box, box] * 4), bx=rb[:, :3].copy(), bq=rb[:, 3:7].copy(),
                   bv=rb[:, 7:10].copy(), bw=rb[:, 10:13].copy())
    hm.close()
    return out
