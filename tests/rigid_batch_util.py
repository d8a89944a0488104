"""Scaffolding of the rigid-body replica-batch tests (test_gpu_batch_rigid.py, test_gpu_batch_rigid_device.py): scenes with rigid bodies and
joints as flat arrays, every replica's own body state, and batch and single-scene engines fed the same way.  A batch gets its bodies from
set_replica_rigid_bodies, the single-scene engine of replica r from set_rigid_bodies with replica r's rows."""
import numpy as np

import scenes
from batch_util import DEFAULT_G, XPBD_TYPES, replica_state

RIG_N = 20  # cloth of the coupling rig: RIG_N x RIG_N particles, its corners pinned to the rig's top boxes


def _rig_bodies():
    """Masses and principal inertias of scenes.coupling_rig's 12 bodies, in the order it adds them."""
    anchor, box = scenes.box_inertia(1.0, 0.5, 0.5, 0.5), scenes.box_inertia(1.0, 0.4, 2.0, 0.4)
    return [0.0, 1.0, 1.0] * 4, [anchor, box, box] * 4


def _from_host(build, dt, sub, it, bodies=None, name=""):
    """A HostModel scene as flat arrays; `bodies` (masses, inertias) of the rigid bodies it added, else read from it with unit inertias."""
    from positionbaseddynamics_b200.model import HostModel
    hm = HostModel()
    build(hm)
    hm.init_groups()
    types, bodies_, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    rb = hm.rigid_bodies().copy()
    if bodies is None:
        bodies = ([hm.rigid_body_mass(i) for i in range(len(rb))], [(1.0, 1.0, 1.0)] * len(rb))
    m = dict(types=np.asarray(types).copy(), bodies=np.asarray(bodies_).copy(), params=np.asarray(params, np.float32).copy(), off=off, ids=ids,
             x=np.asarray(hm.get("x"), np.float32).copy(), x0=np.asarray(hm.get("x0"), np.float32).copy(), mass=np.asarray(mass, np.float32).copy(),
             dt=dt, sub=sub, it=it, name=name,
             bm=np.asarray(bodies[0], np.float32), bx=rb[:, :3].copy(), bq=rb[:, 3:7].copy(), bI=np.asarray(bodies[1], np.float32),
             bv=rb[:, 7:10].copy(), bw=rb[:, 10:13].copy())
    hm.close()
    return m


def _rigid_cases(seed=77):
    import rigid_cases as rc
    c = rc.make_model(1, seed)
    f = np.float32
    x = c.px.astype(f) if c.n else np.zeros((1, 3), f)
    return dict(types=np.asarray(c.types), bodies=np.asarray(c.bodies), params=np.asarray(c.params, f), off=c.off, ids=c.ids,
                x=x, x0=rc.tile_x0(c, np.random.default_rng(seed)), mass=c.pm.astype(f) if c.n else np.zeros(1, f),
                dt=rc.DT, sub=2, it=2, name="rigid_cases", bm=c.bm.astype(f), bx=c.bx.astype(f), bq=c.bq.astype(f), bI=c.bI.astype(f),
                bv=c.bv.astype(f), bw=c.bw.astype(f), pv=c.pv.astype(f), case=c)


def _free_bodies(m, count=700, seed=3):
    """`count` free bodies (no joint) spread over the cloth, unit masses, inertias up to 1:10:100."""
    rng = np.random.default_rng(seed)
    return rng.uniform(-1.0, 1.0, (count, 3)) * (5.0, 1.0, 5.0) + (0.0, 3.0, 0.0)


SCENES = {  # name: builder of the flat arrays
    # the coupling rig (both joint types; the resident batch runs the solid instantiation)
    "rig": lambda: _from_host(lambda m: (scenes.cloth(m, RIG_N, RIG_N, sub_steps=2, max_iter=2), scenes.coupling_rig(m, RIG_N, RIG_N)),
                              0.005, 2, 2, _rig_bodies(), "rig"),
    # every edge class of rigid_cases.py: spinning bodies, inertia ratios up to 1:10:100, static sides, mass ratio 1e3, a body in four
    # joints across colours, free bodies
    "rigid_cases": _rigid_cases,
    # StrainTriangle cloth and the rig: the all-types instantiation
    "strain_rig": lambda: _from_host(lambda m: (scenes.cloth(m, RIG_N, RIG_N, cloth_method=3, bending_method=3, bend_k=100.0, sub_steps=2, max_iter=2),
                                                scenes.coupling_rig(m, RIG_N, RIG_N)), 0.005, 2, 2, _rig_bodies(), "strain_rig"),
}
_models = {}


def model(name):
    if name not in _models:
        _models[name] = SCENES[name]()
    return _models[name]


def free_body_cloth():
    """An XPBD cloth with 700 free bodies beside it: more bodies than a CTA has threads; AUTO runs a batch of 32 or more resident."""
    if "free" not in _models:
        m = _from_host(lambda h: scenes.cloth(h, 30, 30, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=1, max_iter=3),
                       0.005, 1, 3, name="free")
        rng = np.random.default_rng(11)
        nb = 700
        m.update(bm=np.ones(nb, np.float32), bx=_free_bodies(m, nb).astype(np.float32), bq=np.tile(np.float32([1, 0, 0, 0]), (nb, 1)),
                 bI=(rng.permutation([1.0, 10.0, 100.0] * nb).reshape(nb, 3) * 0.01).astype(np.float32),
                 bv=np.zeros((nb, 3), np.float32), bw=np.zeros((nb, 3), np.float32))
        _models["free"] = m
    return _models["free"]


def replica_bodies(m, r):
    """Replica r's bodies (mass, x, q, inertia, v, omega): seeded offsets, velocities and spins, dynamic masses and inertias scaled per
    replica; in replica 1 the first dynamic body is static."""
    rng = np.random.default_rng(500 + r)
    nb = len(m["bm"])
    mass = m["bm"].copy()
    dyn = mass != 0
    scale = np.float32(1.0 + 0.25 * (r % 4))
    mass[dyn] *= scale
    inertia = m["bI"] * np.where(dyn[:, None], scale, np.float32(1.0))
    if r == 1 and dyn.any():
        mass[np.argmax(dyn)] = 0.0
    x = (m["bx"] + rng.normal(0.0, 0.01, (nb, 3))).astype(np.float32)
    q = m["bq"] + rng.normal(0.0, 0.02, (nb, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    v = (m["bv"] + rng.normal(0.0, 0.2, (nb, 3))).astype(np.float32)
    w = (m["bw"] + rng.normal(0.0, 1.0, (nb, 3))).astype(np.float32)
    return mass.astype(np.float32), x, q, inertia.astype(np.float32), v, w


def engine(m, mode, replicas=None, bodies=None, gravity=DEFAULT_G):
    """A batch of `replicas` with bodies[r] = replica_bodies of replica r, or (replicas None) a single scene with the bodies `bodies`."""
    from positionbaseddynamics_b200 import _capi
    eng = _capi.Engine(0)
    eng.set_particles(m["x"], m["mass"], x0=m["x0"])
    if replicas is not None:
        eng.set_replicas(replicas)
        eng.set_replica_rigid_bodies(*[np.stack([b[k] for b in bodies]) for k in range(6)])
    else:
        eng.set_rigid_bodies(*bodies)
    eng.add_flat(m["types"], m["bodies"], m["params"])
    eng.set_groups(m["off"], m["ids"])
    eng.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], gravity=gravity)
    eng.set_mode(mode)
    return eng


def results(eng, m):
    """x, v, the multipliers of every XPBD type present (by insertion id) and the bodies (x, q, v, omega)."""
    from positionbaseddynamics_b200 import _capi
    eng.sync()
    lam = {}
    for t in XPBD_TYPES:
        if (m["types"] == t).any():
            l, ids = eng.lambdas(t)
            lam[t] = l[..., np.argsort(ids)].copy()
    return eng.get_attr(_capi.ATTR_X).copy(), eng.get_attr(_capi.ATTR_V).copy(), lam, eng.get_rigid_bodies().copy()


def run(eng, m, gravity=DEFAULT_G):
    """batch_util.run's step sequence (other subSteps / maxIter / velocity method mid-run, an edit of v), returning results()."""
    from positionbaseddynamics_b200 import _capi
    eng.step(2)
    eng.set_params(dt=m["dt"], sub_steps=m["sub"] + 1, max_iter=m["it"] + 1, vel_method=1, gravity=gravity)
    eng.step(2)
    eng.set_attr(_capi.ATTR_V, eng.get_attr(_capi.ATTR_V) * np.float32(0.5))
    eng.step(1)
    return results(eng, m)


def set_particles(eng, states):
    from positionbaseddynamics_b200 import _capi
    eng.set_attr(_capi.ATTR_X, np.stack([s[0] for s in states]))
    eng.set_attr(_capi.ATTR_V, np.stack([s[1] for s in states]))
    eng.set_masses(np.stack([s[2] for s in states]))


def same(batch, solo, r, what=""):
    """Replica r of batch results() bit for bit equal to single-scene results()."""
    xb, vb, lb, bb = batch
    xs, vs, ls, bs = solo
    assert np.array_equal(xb[r], xs), ("x", r, what)
    assert np.array_equal(vb[r], vs), ("v", r, what)
    for t in ls:
        assert np.array_equal(lb[t][r], ls[t]), ("lambda", t, r, what)
    assert np.array_equal(bb[r], bs), ("bodies", r, what)


def sampled(k):
    return sorted({0, 1, k // 2, k - 1} & set(range(k)))


def particle_state(m, r):
    return replica_state(m, r)
