"""The X items of the resident mode's many-CTA regime are ordered across CTAs by per-CTA arrival flags that each CTA polls for its
neighbouring tiles only.  These tests hold that protocol to the graph mode bit for bit over several tile counts, substep / iteration
counts that change between steps (the flags carry a launch ordinal), the second-order velocity update, and check that a model whose
tiles have too many neighbours is refused by the resident mode and runs in graph mode under the automatic choice."""
import os

import numpy as np
import pytest

import scenes

pytestmark = pytest.mark.gpu


def _run(mode, clusters=None, steps=((1, 8, 3),), vel_method=0, n=300):
    """n x n XPBD cloth, perturbed; `steps`: (sub_steps, max_iter, number of steps) run one after the other."""
    from positionbaseddynamics_b200.model import HostModel
    from parity_util import perturb
    if clusters:
        os.environ["PBD_B200_CLUSTERS"] = clusters
    try:
        m = HostModel()
        scenes.cloth(m, n, n, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=steps[0][0], max_iter=steps[0][1],
                     vel_method=vel_method)
        perturb([m], 2.0e-3)
        m.time_step().set_mode(mode)
        for sub, it, k in steps:
            m.set_params(**dict(m._params, sub_steps=sub, max_iter=it))
            m.step(k)
        out = m.get("x").copy(), m.get("v").copy()
        m.close()
    finally:
        os.environ.pop("PBD_B200_CLUSTERS", None)
    assert np.isfinite(out[0]).all()
    return out


def _same(a, b):
    return (a[0] == b[0]).all() and (a[1] == b[1]).all()


@pytest.mark.parametrize("clusters", ["132x1", "37x1", "7x1"])
def test_resident_neighbour_flags_match_graph(clusters):
    assert _same(_run(0), _run(1, clusters))


@pytest.mark.parametrize("clusters", ["132x1", "37x1"])
def test_resident_neighbour_flags_substeps_and_changing_parameters(clusters):
    """Several substeps, the second-order velocity update, and maxIter / subSteps changed between steps (a launch whose phase count
    differs from the previous one's must still wait for exactly the arrivals of its own launch)."""
    steps = ((3, 4, 2), (1, 9, 1), (4, 2, 2), (2, 7, 1))
    assert _same(_run(0, steps=steps, vel_method=1), _run(1, clusters, steps=steps, vel_method=1))


def test_too_many_neighbours_is_refused_and_auto_falls_back(monkeypatch):
    """40,000 particles with long-range random distance constraints, in 64 independent tiles (a model this small would otherwise fit
    one cluster, which has no X items): every tile reaches far more than 32 others through global-homed particles.  The resident mode
    refuses the model with a message; the automatic choice runs it in graph mode with the same bits."""
    from positionbaseddynamics_b200 import _capi
    monkeypatch.setenv("PBD_B200_CLUSTERS", "64x1")
    rng = np.random.default_rng(7)
    side = 200
    g = np.stack(np.meshgrid(np.arange(side), np.arange(side), indexing="ij"), -1).reshape(-1, 2).astype(np.float32) * 0.05
    x = np.zeros((side * side, 3), np.float32); x[:, 0] = g[:, 0]; x[:, 2] = g[:, 1]
    mass = np.ones(side * side, np.float32); mass[0] = 0.0
    pairs = rng.integers(0, side * side, size=(30000, 2))
    pairs = pairs[pairs[:, 0] != pairs[:, 1]].astype(np.uint32)
    rest = np.linalg.norm(x[pairs[:, 0]] - x[pairs[:, 1]], axis=1) * np.float32(0.9)
    params = np.stack([rest, np.full_like(rest, 1.0e4)], 1)

    def engine(mode):
        eng = _capi.Engine(0)
        eng.set_particles(x, mass)
        eng.add_constraints(_capi.TYPE_NAMES.index("Distance_XPBD"), pairs, params)
        eng.color_first_fit()
        eng.set_params(dt=0.005, sub_steps=1, max_iter=4)
        if mode is not None:
            eng.set_mode(mode)
        return eng

    eng = engine(_capi.MODE_RESIDENT)
    with pytest.raises(_capi.PbdError, match="more than 32 other tiles"):
        eng.step(1)
    eng.close()

    res = []
    for mode in (None, _capi.MODE_GRAPH):
        eng = engine(mode)
        eng.step(2); eng.sync()
        res.append((eng.get_attr(_capi.ATTR_X).copy(), eng.get_mode()[1]))
        eng.close()
    assert res[0][1] == _capi.MODE_GRAPH
    assert (res[0][0] == res[1][0]).all()
