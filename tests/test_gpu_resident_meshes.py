"""The resident kernel against the launch mode, bit for bit, on the mesh scenes of tests/resident_meshes.py: one scene per type mask, in
which constraints of every type share particles with other colours and types across tiles, in every regime -- one CTA, one cluster of
2, 4 or 16 CTAs (DSMEM items), 2, 7 or 37 independent CTAs (X items and neighbour flags) and the planner's default.  A missing cluster
barrier, an X item that passes its neighbour wait too early, a DSMEM store that lands after the next colour's gather or a wrong split of
a colour's runs changes these answers.  Controls: the colour groups reversed change them too (the answers depend on the order the
barriers protect), and the launch mode itself is held to the fp64 checker.  Replica batches of every mask run at C = 2 and C = 4 with
more replicas than the device runs clusters at once."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import resident_meshes as rm
from batch_util import DEFAULT_G, XPBD_TYPES, replica_state, set_state

pytestmark = pytest.mark.gpu

GRAPH, RESIDENT, LAUNCH = 0, 1, 2
HERE = os.path.dirname(os.path.abspath(__file__))


def schedule(m):
    """(sub_steps, max_iter, vel_method, steps): the step counts change between steps, and both velocity updates run."""
    sub, it = m["sub"], m["it"]
    return [(sub, it, 0, 2), (sub + 1, it + 2, 1, 1), (1, it, 1, 1), (sub, it + 1, 0, 1)]


def engine(m, mode, groups=None):
    from positionbaseddynamics_b200 import _capi
    eng = _capi.Engine(0)
    eng.set_particles(m["x"], m["mass"], x0=m["x0"])
    if "bm" in m:
        eng.set_rigid_bodies(m["bm"], m["bx"], m["bq"], m["bI"], m["bv"], m["bw"])
    eng.add_flat(m["types"], m["bodies"], m["params"])
    eng.set_groups(*(groups or (m["off"], m["ids"])))
    eng.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"])
    eng.set_mode(mode)
    return eng


def results(eng, m):
    """x, v, the multipliers of every XPBD type (by insertion id) and the rigid bodies."""
    from positionbaseddynamics_b200 import _capi
    eng.sync()
    lam = {}
    for t in XPBD_TYPES:
        if (m["types"] == t).any():
            l, ids = eng.lambdas(t)
            lam[t] = l[..., np.argsort(ids)].copy()
    rb = eng.get_rigid_bodies().copy() if "bm" in m else None
    return eng.get_attr(_capi.ATTR_X).copy(), eng.get_attr(_capi.ATTR_V).copy(), lam, rb


def run(eng, m, modes=None):
    """The schedule, segment k in modes[k] where given; returns results()."""
    for k, (sub, it, vel, steps) in enumerate(schedule(m)):
        if modes:
            eng.set_mode(modes[k])
        eng.set_params(dt=m["dt"], sub_steps=sub, max_iter=it, vel_method=vel, gravity=DEFAULT_G)
        eng.step(steps)
    return results(eng, m)


def same(a, b, r=None):
    """results() a (replica r of a batch's, if given) and b bit for bit: a list of what differs."""
    pick = (lambda v: v) if r is None else (lambda v: v[r])
    bad = [k for k, u, w in (("x", a[0], b[0]), ("v", a[1], b[1])) if not np.array_equal(pick(u), w)]
    bad += ["lambda%d" % t for t in b[2] if not np.array_equal(pick(a[2][t]), b[2][t])]
    if b[3] is not None and not np.array_equal(pick(a[3]), b[3]):
        bad.append("bodies")
    return bad


def with_clusters(regime):
    """Set PBD_B200_CLUSTERS for `regime` (read at every plan); returns what to restore."""
    old = os.environ.pop("PBD_B200_CLUSTERS", None)
    if regime != "default":
        os.environ["PBD_B200_CLUSTERS"] = regime
    return old


def restore(old):
    os.environ.pop("PBD_B200_CLUSTERS", None)
    if old is not None:
        os.environ["PBD_B200_CLUSTERS"] = old


def resident_run(m, regime, modes=None):
    old = with_clusters(regime)
    try:
        eng = engine(m, RESIDENT if modes is None else modes[0])
        out = run(eng, m, modes)
        if modes is None:
            assert eng.get_mode()[1] == RESIDENT, (m["name"], m["size"], regime)
        eng.close()
    finally:
        restore(old)
    return out


def launch_run(m, groups=None):
    eng = engine(m, LAUNCH, groups)
    out = run(eng, m)
    eng.close()
    assert np.isfinite(out[0]).all() and np.isfinite(out[1]).all(), (m["name"], m["size"])
    return out


def reversed_groups(off, ids):
    """The colour groups in the opposite order."""
    parts = [ids[off[g]:off[g + 1]] for g in range(len(off) - 1)][::-1]
    return np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint32), np.concatenate(parts).astype(np.uint32)


_flats = {}


def flat(name, size, rig):
    key = (name, size, rig)
    if key not in _flats:
        _flats[key] = rm.flat(name, size, rig)
    return _flats[key]


def fp64_gate(name, cpu_libs):
    """The launch mode's small scene after two steps against the fp64 restatement and, where it was built, the fp64 reference; the start
    state and a twin without projections must fail the gate.  Scenes with FEMTet_XPBD (E = 1e4) run one step (DESIGN.md section 5) and
    are held to 1e-3 on positions: their bars are ill-conditioned near the rest state, and the fp32 and fp64 restatements of the fem
    scene's bar differ by 2.2e-3 after that step.  Measured on an H100 80GB HBM3 (700 W): fem 7.4e-4, all 4.7e-4; both controls 0.94
    and more."""
    from parity_util import assert_gate_rejects, assert_parity, parity_errors
    from conftest import have_ref
    m = flat(name, "small", False)
    steps, tol = (1, 1e-3) if rm.xpbd_fem(name) else (2, 1e-4)
    eng = engine(m, LAUNCH)
    eng.step(steps); eng.sync()
    from positionbaseddynamics_b200 import _capi
    x = eng.get_attr(_capi.ATTR_X).copy()
    eng.close()

    def checker(kind, max_iter=None):
        cpu = cpu_libs.CpuPbd(kind, "f64")
        rm.builder(name, "small")(cpu)
        t, b, _, _ = cpu.constraints()
        assert np.array_equal(t, m["types"]) and np.array_equal(b, m["bodies"])
        cpu.set("x", m["x"])
        if max_iter is not None:
            cpu.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=max_iter)
        cpu.step(steps)
        return np.asarray(cpu.get("x"), np.float64).copy()

    xc = checker("oracle")
    e_pos, e_disp = assert_parity(x, xc, m["x"], tol_pos=tol, what="%s launch vs fp64" % name)
    line = "%s: fp64 rel pos %.2e, rel disp %.2e" % (name, e_pos, e_disp)
    if have_ref("f64"):
        e_ref = assert_parity(x, checker("ref"), m["x"], tol_pos=tol, what="%s launch vs fp64 reference" % name)
        line += "; reference %.2e / %.2e" % e_ref
    free = checker("oracle", max_iter=0)
    assert_gate_rejects(m["x"], xc, m["x"], what="%s start state" % name)
    assert_gate_rejects(free, xc, m["x"], what="%s without projections" % name)
    return line + "; controls: start %.2e / %.2e, no projections %.2e / %.2e" % (parity_errors(m["x"], xc, m["x"]) + parity_errors(free, xc, m["x"]))


@pytest.mark.parametrize("name", sorted(rm.SCENES))
def test_resident_meshes_match_launch(name, cpu_libs):
    t0 = time.time()
    print()
    print(fp64_gate(name, cpu_libs))
    for size in rm.SIZES:
        ref = {}
        for regime in rm.regimes(size):
            rig = rm.has_rig(name, regime)
            m = flat(name, size, rig)
            if rig not in ref:
                ref[rig] = launch_run(m)
                if not rig:  # control: the answers depend on the colour order
                    rev = launch_run(m, reversed_groups(m["off"], m["ids"]))
                    d = float(np.abs(rev[0].astype(np.float64) - ref[rig][0]).max())
                    print("%s %s: colour groups reversed move x by up to %.2e" % (name, size, d))
                    assert d > 0.0, (name, size, "reversing the colours changes nothing")
            bad = same(resident_run(m, regime), ref[rig])
            assert not bad, (name, size, regime, "resident", bad)
            bad = same(resident_run(m, regime, modes=(LAUNCH, RESIDENT, RESIDENT, LAUNCH)), ref[rig])
            assert not bad, (name, size, regime, "launch -> resident -> launch", bad)
    print("%s: every regime bit-identical to the launch mode, %.1f s" % (name, time.time() - t0))


_SHAPE_WORKER = r"""
import os, sys
import resident_meshes as rm
import test_gpu_resident_meshes as t
for name in sorted(rm.SCENES):
    for size in rm.SIZES:
        for regime in rm.regimes(size):
            m = t.flat(name, size, rm.has_rig(name, regime))
            old = t.with_clusters(regime)
            sys.stderr.write("@@ %s %s %s\n" % (name, size, regime)); sys.stderr.flush()
            eng = t.engine(m, t.RESIDENT)
            eng.step(1); eng.sync(); eng.close()
            sys.stderr.flush()
            t.restore(old)
"""


def test_resident_meshes_ran_the_intended_shapes():
    """One process with PBD_B200_VERBOSE (read once per process) plans every (scene, size, regime): the shape each image ran is the one
    asked for, and the default is one cluster."""
    t0 = time.time()
    env = dict(os.environ, PBD_B200_VERBOSE="1", PYTHONPATH=os.pathsep.join([os.path.dirname(HERE), HERE]))
    env.pop("PBD_B200_CLUSTERS", None)
    out = subprocess.run([sys.executable, "-c", _SHAPE_WORKER], cwd=HERE, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    got, cur = {}, None
    for line in out.stderr.splitlines():
        if line.startswith("@@ "):
            cur = tuple(line.split()[1:])
        elif "] resident: " in line and " clusters x " in line:
            w = line.split("resident: ")[1].split()
            got.setdefault(cur, []).append((int(w[0]), int(w[3])))
    for name in sorted(rm.SCENES):
        for size in rm.SIZES:
            for regime in rm.regimes(size):
                shapes = got.get((name, size, regime))
                assert shapes, (name, size, regime, "no resident image")
                G, C = shapes[-1]
                print("%s %s %s: ran %d clusters x %d CTAs" % (name, size, regime, G, C))
                assert (G, C) == rm.shape(regime) if regime != "default" else G == 1, (name, size, regime, G, C)
    print("shapes checked in %.1f s" % (time.time() - t0))


def _batch(m, K, C, mode, states, bodies, extra=None):
    from positionbaseddynamics_b200 import _capi  # noqa: F401
    old = with_clusters("1x%d" % C)
    try:
        eng = _capi.Engine(0)
        eng.set_particles(m["x"], m["mass"], x0=m["x0"])
        eng.set_replicas(K)
        if bodies:
            eng.set_replica_rigid_bodies(*[np.stack([b[k] for b in bodies]) for k in range(6)])
        eng.add_flat(m["types"], m["bodies"], m["params"])
        eng.set_groups(m["off"], m["ids"])
        eng.set_params(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"])
        eng.set_mode(mode)
        set_state(eng, states)
        if extra:
            extra(eng)
        out = run(eng, m)
        if mode == RESIDENT:
            assert eng.get_mode()[1] == RESIDENT
        eng.close()
    finally:
        restore(old)
    return out


@pytest.mark.parametrize("C", [2, 4])
@pytest.mark.parametrize("name", sorted(rm.SCENES))
def test_resident_mesh_batches_match_single_scenes(name, C):
    """K = 2 x 132 / C + 1 replicas of the small scene, each with its own state (and, for the solid scene, its own rig bodies), at a forced
    cluster of C CTAs: clusters step several replicas in turn.  Replica r equals a single-scene launch engine given replica r's state."""
    import rigid_batch_util as rbu
    t0 = time.time()
    rig = name == "solid"
    m = flat(name, "small", rig)
    K = 2 * (132 // C) + 1
    states = [replica_state(m, r) for r in range(K)]
    bodies = [rbu.replica_bodies(m, r) for r in range(K)] if rig else None
    batch = _batch(m, K, C, RESIDENT, states, bodies)
    for r in sorted({0, 1, 2, K // 2, K - 2, K - 1}):
        eng = engine(m, LAUNCH)
        if rig:
            eng.set_rigid_bodies(*bodies[r])
        from positionbaseddynamics_b200 import _capi
        eng.set_attr(_capi.ATTR_X, states[r][0]); eng.set_attr(_capi.ATTR_V, states[r][1]); eng.set_masses(states[r][2])
        solo = run(eng, m)
        eng.close()
        bad = same(batch, solo, r)
        assert not bad, (name, C, K, r, bad)
    print("%s: %d replicas at C = %d match single scenes, %.1f s" % (name, K, C, time.time() - t0))


@pytest.mark.parametrize("C", [2, 4])
def test_resident_all_types_batch_with_replica_overrides(C):
    """The all-types scene's batch with per-replica rest shapes (the geometry offsets), per-constraint materials of every type (the
    material offsets) and gravity: the resident batch at C = 2 and 4 equals the launch batch given the same, replica by replica."""
    from positionbaseddynamics_b200 import _capi
    m = flat("all", "small", False)
    K = 2 * (132 // C) + 1
    states = [replica_state(m, r) for r in range(K)]
    c = m["x0"].mean(axis=0)
    x0 = np.stack([c + (m["x0"] - c) * np.float32(1.0 + 0.04 * ((r % 5) - 2)) for r in range(K)]).astype(np.float32)
    scale = np.float32(1.0) + np.float32(0.1) * ((np.arange(K) % 3) - 1).astype(np.float32)
    g = np.stack([0.5 * np.sin(np.arange(K)), -9.81 + 0.1 * (np.arange(K) % 7), np.zeros(K)], 1).astype(np.float32)
    present = [t for t in range(13) if (m["types"] == t).any() and _capi.num_materials(t)]

    def overrides(eng):
        eng.set_replica_rest_positions(x0)
        for t in present:
            eng.set_replica_constraint_materials(t, np.ascontiguousarray(eng.get_replica_materials(t) * scale[:, None, None]))
        eng.set_replica_gravity(g)

    res = _batch(m, K, C, RESIDENT, states, None, overrides)
    lau = _batch(m, K, C, LAUNCH, states, None, overrides)
    for r in range(K):
        bad = same(res, (lau[0][r], lau[1][r], {t: v[r] for t, v in lau[2].items()}, None), r)
        assert not bad, (C, K, r, bad)
    assert not np.array_equal(res[0][0], res[0][3])  # the replicas differ
