"""The contact kernels against the fp64 restatement of tests/contact_cases.py, in every execution mode.

Each layout's particles start from x_pre with their velocities, no gravity, and step once.  A twin engine without colliders, stepped
from the same state in MODE_LAUNCH, gives the state the contact launch starts from (positions do not depend on contacts); its fp32 x and
v go to contact_cases.reference, so the comparison measures the contact kernel alone.  Paths:

  launch / graph / resident   one layout per single-scene engine (pbd_set_colliders), every configuration of contact_cases.CONFIGS
  batch_*                     the three layouts as the replicas of one K = 3 batch (pbd_set_replica_colliders), replica r held to
                              its own answer, in the same three modes
  poses_*                     the same batch after its rows were moved away and back with pbd_set_replica_collider_poses_device

Sensors are on in one run of each path and off in another; the velocities must be the same bits.  Compared per case: the contact set
exactly (by particle and body), cp1, n and dist of each record, the velocity (contact_cases.velocity_errors), the sensor counts exactly
and the impulses relative to max(|sum|, 1e-2).  Every path must be bit-identical to MODE_LAUNCH.  The at-threshold classes are held
to bit identity with MODE_LAUNCH and, for the degenerate normals, to the restatement's set of non-finite particles; their velocity
error must be within a few times the fp32 restatement's.  The sensors of every collider are compared in one more run, with the
degenerate-normal particles static (otherwise their NaN velocities make their colliders' impulses NaN).  Negative controls: the gate
must fail against each mutated restatement."""
import numpy as np
import pytest

import contact_cases as cc
import contact_util as cu

pytestmark = pytest.mark.gpu
REC = np.dtype([("particle", "<u4"), ("body", "<u4"), ("cp0", "<f4", 3), ("cp1", "<f4", 3), ("n", "<f4", 3), ("dist", "<f4")])
CAP = 1 << 16
PATCH = 64  # the last PATCH particles (far from every collider) carry distance constraints, so that the resident mode admits the model


def _layouts():
    global _L
    try:
        return _L
    except NameError:
        _L = cc.make_layouts()
        return _L


def _patch():
    i = np.arange(cc.N - PATCH, cc.N, 2)
    return np.stack([i, i + 1], 1).astype(np.uint32)


def engine(L_or_list, mode, colliders=True, sense=False):
    """A single-scene engine (one layout) or a K = 3 batch (a list of layouts)."""
    from positionbaseddynamics_b200 import _capi
    batch = isinstance(L_or_list, list)
    Ls = L_or_list if batch else [L_or_list]
    L0 = Ls[0]
    eng = _capi.Engine(0)
    eng.set_particles(L0.x_pre, L0.mass, x0=L0.x_pre)
    pairs = _patch()
    rest = np.linalg.norm(L0.x_pre[pairs[:, 0]] - L0.x_pre[pairs[:, 1]], axis=1)
    eng.add_constraints(_capi.DISTANCE, pairs, np.stack([rest, np.ones_like(rest)], 1))
    eng.color_first_fit()
    if not batch and colliders:
        eng.set_rigid_bodies([0.0] * len(L0.bx), L0.bx, [(1.0, 0.0, 0.0, 0.0)] * len(L0.bx), [(1.0, 1.0, 1.0)] * len(L0.bx), v=L0.bv, omega=L0.bw)
    eng.set_mode(mode)
    if batch:
        eng.set_replicas(len(Ls))
        eng.set_masses(np.stack([L.mass for L in Ls]))
    pcs = [_capi.ParticleCollider(*r) for r in cc.RANGES]
    if colliders:
        if batch:
            eng.set_replica_colliders(pcs, [[cu.to_capi(c) for c in L.cols] for L in Ls], *body_rows(Ls))
        else:
            eng.set_colliders(pcs, [cu.to_capi(c) for c in L0.cols])
        eng.record_contacts(CAP)
        if sense:
            eng.sense_contacts(True)
    return eng


def body_rows(Ls):
    """(K, 8, 3) body x, v, omega: collider k of replica r on body k."""
    idx = lambda L: [c["body"] for c in L.cols]
    return tuple(np.stack([np.asarray(getattr(L, a))[idx(L)] for L in Ls]).astype(np.float32) for a in ("bx", "bv", "bw"))


def step(eng, Ls, config, sense=False):
    """One step of config from the layouts' x_pre and v: x, v (K, N, 3) and, with colliders, the contact records and the sensors
    (None unless `sense`)."""
    from positionbaseddynamics_b200 import _capi
    tol, stiff, iters, sub = config
    x = np.stack([L.x_pre for L in Ls]); v = np.stack([L.v for L in Ls])
    if len(Ls) == 1:
        x, v = x[0], v[0]
    for a, val in ((_capi.ATTR_X, x), (_capi.ATTR_V, v), (_capi.ATTR_OLDX, x), (_capi.ATTR_LASTX, x)):
        eng.set_attr(a, val)
    eng.set_params(dt=cc.DT, sub_steps=sub, max_iter=1, vel_method=0, gravity=(0.0, 0.0, 0.0))
    eng.set_contact_params(tolerance=tol, stiffness=stiff, max_iter_v=iters)
    eng.step(1); eng.sync()
    K = len(Ls)
    out = [eng.get_attr(_capi.ATTR_X).reshape(K, cc.N, 3).copy(), eng.get_attr(_capi.ATTR_V).reshape(K, cc.N, 3).copy()]
    if eng.n_rigid_colliders:
        recs, found = eng.contacts(CAP)
        assert found <= CAP
        out.append(np.array([(c.particle, c.body, tuple(c.cp0), tuple(c.cp1), tuple(c.normal), c.dist) for c in recs], REC))
        out.append(eng.contact_sensors() if sense else None)
    return out


class Table:
    def __init__(self):
        self.worst, self.bad = {}, []

    def note(self, key, path, value, limit, what):
        k = key + (path,)
        self.worst[k] = max(self.worst.get(k, 0.0), value)
        if not value <= limit:
            self.bad.append((key, path, what, value, limit))

    def show(self):
        print("\nworst velocity error per (shape, class, path)")
        for k in sorted(self.worst):
            print("  %-10s %-18s %-16s %.2e" % (k + (self.worst[k],)))
        per = {}
        for (s, c, _), v in self.worst.items():
            per[(s, c)] = max(per.get((s, c), 0.0), v)
        print("TOL-MEASURED", repr(per))


def check(table, L, config, path, got_x, got_v, rec, sensors, twin_x, twin_v, r=0):
    """One replica / layout of one run against its fp64 answer."""
    assert np.array_equal(got_x, twin_x), (path, L.name, config)
    for key, err, limit in cc.velocity_gate(L, got_v, twin_x, twin_v, config):
        table.note(key, path, err, limit, "velocity")
    _, rref, count, impulse = cc.run_reference(L, twin_x, twin_v, config)
    # the contact set (by particle and body) and the records
    n, g = cc.N, cc.gated(L)
    mine = rec[rec["particle"] // n == r]
    gp = g[mine["particle"] - r * n]
    got_set = sorted(zip((mine["particle"][gp] - r * n).tolist(), mine["body"][gp].tolist()))
    bid = [c["body"] for c in L.cols]
    want = [(int(q["particle"]), bid[int(q["collider"])]) for q in rref if g[q["particle"]]]
    assert got_set == sorted(want), (path, L.name, config, len(got_set), len(want))
    keyed = {}  # cp1, n, dist where a (particle, body) pair is unique
    for q in rref:
        keyed.setdefault((int(q["particle"]), bid[int(q["collider"])]), []).append(q)
    worst_rec = 0.0
    for m_ in mine[gp]:
        lst = keyed[(int(m_["particle"]) - r * n, int(m_["body"]))]
        if len(lst) != 1:
            continue
        q = lst[0]
        worst_rec = max(worst_rec, float(np.abs(m_["cp1"] - q["cp1"]).max() / max(np.abs(q["cp1"]).max(), 1.0)),
                        float(np.abs(m_["n"] - q["n"]).max()), float(abs(m_["dist"] - q["dist"]) / max(abs(q["dist"]), 1e-3)))
    table.note(("records", L.name), path, worst_rec, cc.TOL_RECORDS, "records")
    if sensors is not None:
        same_count, same_fin, err = cc.sensor_errors(sensors[0][r], sensors[1][r], count, impulse)
        assert same_count and same_fin, (path, L.name, config, sensors[0][r], count)
        table.note(("sensors", L.name), path, err, cc.TOL_SENSORS, "sensor impulse")


def test_contact_answers_every_path():
    import subprocess
    from positionbaseddynamics_b200 import _capi
    Ls = _layouts()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("measured on: %s" % gpu)
    table = Table()
    launch = {}
    # twins: the pre-contact state of every layout and configuration
    twins = {}
    for i, L in enumerate(Ls):
        tw = engine(L, _capi.MODE_LAUNCH, colliders=False)
        for config in cc.CONFIGS:
            x, v = step(tw, [L], config)[:2]
            twins[(i, config)] = (x[0], v[0])
        tw.close()
    for mode, path in ((_capi.MODE_LAUNCH, "launch"), (_capi.MODE_GRAPH, "graph"), (_capi.MODE_RESIDENT, "resident")):
        for sense in (False, True):
            for i, L in enumerate(Ls):
                eng = engine(L, mode, sense=sense)
                for config in cc.CONFIGS:
                    x, v, rec, sensors = step(eng, [L], config, sense)
                    assert eng.get_mode()[1] == mode, (path, eng.get_mode())
                    key = (i, config)
                    if key not in launch:
                        launch[key] = (x, v)
                    assert np.array_equal(x, launch[key][0]) and np.array_equal(v.view(np.uint32), launch[key][1].view(np.uint32)), (path, sense, L.name, config)
                    check(table, L, config, path, x[0], v[0], rec, sensors, *twins[key])
                eng.close()
    # the K = 3 batch: replica r = layout r, in three modes, and after a device write of the rows
    import torch
    for mode, path in ((_capi.MODE_LAUNCH, "batch_launch"), (_capi.MODE_GRAPH, "batch_graph"), (_capi.MODE_RESIDENT, "batch_resident")):
        for sense in (False, True):
            for poses in (False, True):
                eng = engine(list(Ls), mode, sense=sense)
                name = path.replace("batch", "poses") if poses else path
                if poses:
                    bx, bv, bw = body_rows(Ls)
                    away = [[dict(c, v2=(np.asarray(c["v2"]) + 7.0).tolist(), aabb_min=(np.asarray(c["aabb_min"]) + 7.0).tolist(),
                                  aabb_max=(np.asarray(c["aabb_max"]) + 7.0).tolist()) for c in L.cols] for L in Ls]
                    eng.set_replica_colliders([_capi.ParticleCollider(*r) for r in cc.RANGES], [[cu.to_capi(c) for c in l] for l in away],
                                              bx + 7.0, bv * 0.0, bw * 0.0)
                    pose = np.concatenate([np.stack([np.concatenate([c["R"], c["v1"], c["v2"], c["aabb_min"], c["aabb_max"]]) for c in L.cols]) for L in Ls])
                    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda()
                    eng.set_replica_collider_poses_device(dev(pose), dev(bx), dev(bv), dev(bw), stream=torch.cuda.current_stream().cuda_stream)
                for config in cc.CONFIGS:
                    x, v, rec, sensors = step(eng, list(Ls), config, sense)
                    assert eng.get_mode()[1] == mode, (name, eng.get_mode())
                    for r, L in enumerate(Ls):
                        lx, lv = launch[(r, config)]
                        assert np.array_equal(x[r], lx[0]) and np.array_equal(v[r].view(np.uint32), lv[0].view(np.uint32)), (name, sense, L.name, config)
                        check(table, L, config, name, x[r], v[r], rec, sensors, *twins[(r, config)], r=r)
                eng.close()
    # the sensors of every collider: the degenerate normals (whose NaN velocities make their colliders' impulses NaN) made static
    for i, L in enumerate(Ls):
        M = cc.without_degenerate(L)
        tw = engine(M, _capi.MODE_LAUNCH, colliders=False)
        eng = engine(M, _capi.MODE_LAUNCH, sense=True)
        for config in cc.CONFIGS:
            tx, tv = step(tw, [M], config)
            x, v, rec, sensors = step(eng, [M], config, True)
            _, _, count, impulse = cc.run_reference(M, tx[0], tv[0], config)
            assert np.isfinite(impulse).all(), (L.name, config)
            check(table, M, config, "launch_static_degenerate", x[0], v[0], rec, sensors, tx[0], tv[0])
        tw.close(); eng.close()
    table.show()
    assert not table.bad, (len(table.bad), table.bad[:20])

    # negative controls: the gate (gated and at-threshold classes alike) fails against each mutated restatement
    caught = {}
    for mut in cc.MUTATIONS:
        for i, L in enumerate(Ls):
            for config in cc.CONFIGS:
                x, v = launch[(i, config)]
                tx, tv = twins[(i, config)]
                caught[mut] = caught.get(mut, 0) + sum(not err <= limit for _, err, limit in cc.velocity_gate(L, v[0], tx, tv, config, mut=mut))
    print("negative controls, (shape, class) outside the gate: %s" % caught)
    for mut in cc.MUTATIONS:
        assert caught[mut] > 0, ("negative control passed the gate", mut)


def test_overlapping_ranges_are_refused():
    """Two particle ranges over one particle are refused by both collider calls, with the previous colliders still in force; adjacent and
    empty ranges are accepted."""
    from positionbaseddynamics_b200 import _capi
    Ls = _layouts()
    L = Ls[0]
    config = cc.CONFIGS[0]
    one = engine(L, _capi.MODE_GRAPH)
    want = step(one, [L], config)[:2]
    cols = [cu.to_capi(c) for c in L.cols]
    for bad in ([(10, 20, 0.5, 0.1), (29, 5, 0.5, 0.1)], [(0, cc.N, 0.5, 0.1), (0, cc.N, 0.5, 0.1)], [(100, 50, 0.5, 0.1), (0, 300, 0.5, 0.1)]):
        with pytest.raises(_capi.PbdError, match="overlap"):
            one.set_colliders([_capi.ParticleCollider(*r) for r in bad], cols)
    got = step(one, [L], config)[:2]
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
    one.set_colliders([_capi.ParticleCollider(*r) for r in ((0, 30, 0.5, 0.1), (30, 0, 0.5, 0.1), (30, 10, 0.5, 0.1), (35, 0, 0.1, 0.1))], cols)
    one.close()
    b = engine(list(Ls), _capi.MODE_GRAPH)
    want = step(b, list(Ls), config)[:2]
    rows = [[cu.to_capi(c) for c in l.cols] for l in Ls]
    with pytest.raises(_capi.PbdError, match="overlap"):
        b.set_replica_colliders([_capi.ParticleCollider(0, 30, 0.5, 0.1), _capi.ParticleCollider(29, 1, 0.5, 0.1)], rows, *body_rows(Ls))
    got = step(b, list(Ls), config)[:2]
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
    b.set_replica_colliders([_capi.ParticleCollider(0, 30, 0.5, 0.1), _capi.ParticleCollider(30, 1, 0.5, 0.1)], rows, *body_rows(Ls))
    b.close()
