"""Scaffolding shared by the replica-batch GPU tests (test_gpu_batch.py, test_gpu_replica_params.py, test_gpu_replica_rest_shape.py).
Each scene is built by tests/scenes.py on a HostModel and handed to _capi.Engine through add_flat / set_groups / set_particles, the batch
and the single-scene engines alike."""
import numpy as np
import pytest

import scenes

GRAPH, RESIDENT, LAUNCH, JACOBI, AUTO = 0, 1, 2, 3, 4
MODES = pytest.mark.parametrize("mode", [GRAPH, LAUNCH, RESIDENT, AUTO], ids=["graph", "launch", "resident", "auto"])
XPBD_TYPES = (1, 4, 8, 10)
DEFAULT_G = (0.0, -9.81, 0.0)

# Between them the scenes run all six resident type masks and every type with more than one material parameter.
SCENES = {  # name: (builder, dt, sub_steps, max_iter)
    "cfg1": (lambda m: scenes.cfg1(m), 0.005, 1, 5),
    "xpbd_cloth64": (lambda m: scenes.cloth(m, 64, 64, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=1, max_iter=5), 0.005, 1, 5),
    "fem_volume_bar": (lambda m: scenes.bar(m, 9, 4, 4, solid_method=2, k=1.0e5, extra_volume=True, sub_steps=2, max_iter=3), 0.005, 2, 3),
    "mixed": (lambda m: scenes.mixed(m), 0.005, 5, 1),
    # the light-mask resident kernels (FEMTriangle + Dihedral + IsometricBending_XPBD) and the all-types ones (StrainTriangle)
    "femtri_dihedral_cloth": (lambda m: (scenes.cloth(m, 40, 40, cloth_method=2, bending_method=1, sub_steps=2, max_iter=3),
                                         m.add_bending_constraints(0, 3, 100.0)), 0.005, 2, 3),
    "strain_cloth": (lambda m: scenes.cloth(m, 40, 40, cloth_method=3, bending_method=3, bend_k=100.0, sub_steps=2, max_iter=3), 0.005, 2, 3),
}
_models = {}


def model(name, table=SCENES):
    """Scene `name` of `table` as flat arrays (copies, the host model is closed), built once per session."""
    if name not in _models:
        from positionbaseddynamics_b200.model import HostModel
        build, dt, sub, it = table[name]
        hm = HostModel()
        build(hm)
        hm.init_groups()
        types, bodies, params, _ = hm.constraints()
        off, ids = hm.groups()
        mass, _ = hm.masses()
        _models[name] = dict(types=np.asarray(types).copy(), bodies=np.asarray(bodies).copy(), params=np.asarray(params, np.float32).copy(), off=off, ids=ids,
                             x=np.asarray(hm.get("x"), np.float32).copy(), x0=np.asarray(hm.get("x0"), np.float32).copy(),
                             mass=np.asarray(mass, np.float32).copy(), dt=dt, sub=sub, it=it, name=name)
        hm.close()
    return _models[name]


def replica_state(m, r):
    """Replica r's own seeded perturbation of x and v; replica 1 also pins every 7th particle through its masses."""
    rng = np.random.default_rng(1000 + r)
    scale = float(np.ptp(m["x"], axis=0).max())
    x = (m["x"] + rng.normal(0.0, 0.01 * scale, m["x"].shape)).astype(np.float32)
    v = rng.normal(0.0, 0.1, m["x"].shape).astype(np.float32)
    mass = m["mass"].copy()
    if r == 1:
        mass[::7] = 0.0
    return x, v, mass


def engine(m, mode, replicas=None, gravity=DEFAULT_G):
    from positionbaseddynamics_b200 import _capi
    eng = _capi.Engine(0)
    eng.set_particles(m["x"], m["mass"], x0=m["x0"])
    eng.add_flat(m["types"], m["bodies"], m["params"])
    eng.set_groups(m["off"], m["ids"])
    eng.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], gravity=gravity)
    eng.set_mode(mode)
    if replicas is not None:
        eng.set_replicas(replicas)
    return eng


def results(eng, m):
    """x, v and the multipliers of every XPBD type present."""
    from positionbaseddynamics_b200 import _capi
    eng.sync()
    lam = {}
    for t in XPBD_TYPES:
        if (m["types"] == t).any():
            l, ids = eng.lambdas(t)
            lam[t] = l[..., np.argsort(ids)].copy()  # by insertion id: the resident image orders a colour's constraints by tile
    return eng.get_attr(_capi.ATTR_X).copy(), eng.get_attr(_capi.ATTR_V).copy(), lam


def run(eng, m, gravity=DEFAULT_G):
    """The step sequence every engine of these tests runs: steps, then other subSteps / maxIter / velocity method, then an edit of the
    velocities with set_attr, then a last step; returns results().  `gravity` is what set_params carries: a batch's per-replica rows
    must outlive that call."""
    from positionbaseddynamics_b200 import _capi
    eng.step(2)
    eng.set_params(dt=m["dt"], sub_steps=m["sub"] + 1, max_iter=m["it"] + 1, vel_method=1, gravity=gravity)
    eng.step(2)
    eng.set_attr(_capi.ATTR_V, eng.get_attr(_capi.ATTR_V) * np.float32(0.5))
    eng.step(1)
    return results(eng, m)


def set_state(eng, states):
    """Every replica's (x, v, mass), replica after replica."""
    from positionbaseddynamics_b200 import _capi
    eng.set_attr(_capi.ATTR_X, np.stack([s[0] for s in states]))
    eng.set_attr(_capi.ATTR_V, np.stack([s[1] for s in states]))
    eng.set_masses(np.stack([s[2] for s in states]))
