"""Per-constraint material parameters of every replica of a batch (pbd_set_replica_constraint_materials, its device form and
pbd_get_replica_materials): replica r advances bit for bit as a single-scene engine whose constraints were added with replica r's values,
in every mode, next to the other per-replica parameters, across source switches, re-plans and added constraints; the device form writes
only the masked replicas, in the caller's stream order.  The scenes are the six batch scenes of batch_util.py (all six resident type masks)
and the tet bars with the solid methods they lack, so that every material-bearing type is overridden."""
import numpy as np
import pytest

import batch_util
import scenes
from batch_util import AUTO, GRAPH, LAUNCH, MODES, RESIDENT, engine, replica_state, results, run, set_state

pytestmark = pytest.mark.gpu

X, V, X0, OLDX, LASTX = range(5)
STATE = (X, V, OLDX, LASTX)
SPIN = 100_000_000  # torch.cuda._sleep cycles: some 50 ms on an H100
# the material columns of every particle type's parameter layout (include/pbd_b200.h), and which of them are Poisson ratios and flags
MAT_COLS = {0: [1], 1: [1], 2: [1], 3: [0], 4: [0], 5: [5, 6, 7, 8, 9], 6: [4, 5, 6, 7, 8], 7: [1], 8: [1], 9: [10, 11], 10: [10, 11],
            11: [9, 10, 11, 12], 12: [0]}
POISSON = {5: (3, 4), 9: (1,), 10: (1,)}  # material slots
FLAGS = {11: (2, 3)}  # (StrainTriangle keeps the model's normalisation flags: random ones made some solo runs diverge)

SCENES = {**batch_util.SCENES,
    "femtet_xpbd_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=3, k=1.0e5, sub_steps=2, max_iter=3), 0.005, 2, 3),
    "straintet_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=4, k=1.0, sub_steps=2, max_iter=3), 0.005, 2, 3),
    "shapematching_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=5, k=1.0, sub_steps=2, max_iter=3), 0.005, 2, 3),
    "xpbd_distance_volume_bar": (lambda m: scenes.bar(m, 8, 3, 3, solid_method=6, k=1.0e4, vol_k=1.0e4, sub_steps=2, max_iter=3), 0.005, 2, 3),
}


def model(name):
    return batch_util.model(name, SCENES)


def present(m):
    return [t for t in MAT_COLS if (m["types"] == t).any()]


def field(m, t, k, seed):
    """(k, count, nMat): a distinct value for every constraint of type t in every replica -- the model's values scaled by 0.5 .. 1.5,
    every 11th constraint of a stiffness type at zero stiffness, Poisson ratios spread over [0, 0.49], flags 0 / 1."""
    rng = np.random.default_rng(seed * 100 + t)
    base = m["params"][m["types"] == t][:, MAT_COLS[t]].astype(np.float64)
    out = base[None] * rng.uniform(0.5, 1.5, (k,) + base.shape)
    for s in POISSON.get(t, ()):
        out[:, :, s] = rng.uniform(0.0, 0.49, out.shape[:2])
    for s in FLAGS.get(t, ()):
        out[:, :, s] = rng.integers(0, 2, out.shape[:2])
    if len(MAT_COLS[t]) == 1:
        out[:, ::11, 0] = 0.0
    return out.astype(np.float32)


def with_materials(m, mats, r):
    """The model with every constraint of type t carrying replica r's values mats[t][r]."""
    params = m["params"].copy()
    for t, f in mats.items():
        params[np.ix_(np.nonzero(m["types"] == t)[0], MAT_COLS[t])] = f[r]
    return dict(m, params=params)


def solo(m, state, gravity=batch_util.DEFAULT_G):
    eng = engine(m, GRAPH, gravity=gravity)
    set_state(eng, [state])
    out = run(eng, m, gravity)
    eng.close()
    return out


def assert_replica(got, want, what):
    x, v, lam = got
    xs, vs, ls = want
    assert np.isfinite(xs).all(), what
    assert np.array_equal(x, xs), what
    assert np.array_equal(v, vs), what
    for t, l in ls.items():
        assert np.array_equal(lam[t], l), (what, t)


def batch_vs_solo(m, mode, k, mats, seed_states=0):
    """The batch with mats set per constraint, run(), against solo runs of replicas 0, 1, K/2, K-1."""
    states = [replica_state(m, r + seed_states) for r in range(k)]
    eng = engine(m, mode, replicas=k)
    set_state(eng, states)
    for t, f in mats.items():
        eng.set_replica_constraint_materials(t, f)
        assert np.array_equal(eng.get_replica_materials(t), f), t
    x, v, lam = run(eng, m)
    active = eng.get_mode()[1]
    eng.close()
    for r in sorted({0, 1, k // 2, k - 1}):
        assert_replica((x[r], v[r], {t: l[r] for t, l in lam.items()}), solo(with_materials(m, mats, r), states[r]), (m["name"], k, mode, r))
    return active


@MODES
@pytest.mark.parametrize("k", [3, 300])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_replicas_equal_solo_runs(name, k, mode):
    m = model(name)
    batch_vs_solo(m, mode, k, {t: field(m, t, k, 1) for t in present(m)})


def test_forced_cluster_shape_on_cfg3(monkeypatch):
    """cfg3 as a batch of one-replica clusters of 8 CTAs (FEMTet + Volume, the FEM instantiation with DSMEM accesses)."""
    monkeypatch.setenv("PBD_B200_CLUSTERS", "1x8")
    table = {"cfg3": (lambda hm: scenes.cfg3(hm), 0.005, 2, 2)}
    m = batch_util.model("cfg3", table)
    assert batch_vs_solo(m, RESIDENT, 3, {t: field(m, t, 3, 2) for t in present(m)}) == RESIDENT


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_with_rest_shapes_gravity_and_rows(mode):
    """Per-constraint materials of StrainTriangle, rows of IsometricBending_XPBD, per-replica rest shapes and gravity together."""
    from test_gpu_replica_rest_shape import rest_shape, with_geometry
    m = model("strain_cloth")
    k = 4
    states = [replica_state(m, r) for r in range(k)]
    mats = {6: field(m, 6, k, 3)}
    rows = np.array([[50.0 * (r + 1)] for r in range(k)], np.float32)
    grav = np.array([[0.0, -9.81 + r, 0.5 * r] for r in range(k)], np.float32)
    eng = engine(m, mode, replicas=k)
    set_state(eng, states)
    eng.set_replica_rest_positions(np.stack([rest_shape(m, r) for r in range(k)]))
    eng.set_replica_constraint_materials(6, mats[6])
    eng.set_replica_materials(4, rows)
    eng.set_replica_gravity(grav)
    geo = {t: eng.replica_geometry(t) for t in (4, 6)}
    assert np.array_equal(eng.get_replica_materials(4), np.repeat(rows[:, None, :], (m["types"] == 4).sum(), axis=1))
    x, v, lam = run(eng, m)
    eng.close()
    for r in range(k):
        ms = with_materials(with_geometry(m, {t: g[r] for t, g in geo.items()}), {**mats, 4: np.repeat(rows[:, None, :], (m["types"] == 4).sum(), axis=1)}, r)
        assert_replica((x[r], v[r], {t: l[r] for t, l in lam.items()}), solo(ms, states[r], gravity=grav[r]), (mode, r))


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_with_replica_colliders(mode):
    """Per-constraint FEMTet materials and every replica against its own static colliders."""
    import contact_util as cu
    from test_gpu_batch_contacts import SCENES as CSCENES, batch_engine, final, solo_engine
    m = batch_util.model("contact_bar", CSCENES)
    k = 3
    mats = {9: field(m, 9, k, 4)}
    fp = cu.footprint(m["x"])
    eng = batch_engine(m, "contact_bar", mode, k, cu.batch_scene(k, fp, -1))
    eng.set_replica_constraint_materials(9, mats[9])
    eng.step(60)
    x, v = final(eng)
    eng.close()
    for r in range(k):
        cols, bx, bv, bw = cu.replica_scene(r, fp, False)
        one = solo_engine(m, "contact_bar", r, cols, bx, bv, bw, params=with_materials(m, mats, r)["params"])
        one.step(60)
        xs, vs = final(one)
        one.close()
        assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)


def twin(m, mid, r, mass, steps):
    """Replica r from the batch's intermediate state `mid` as a single-scene engine of model m, `steps` steps: x, v, multipliers."""
    eng = engine(m, GRAPH)
    eng.set_masses(mass)
    for a in STATE:
        eng.set_attr(a, mid[a][r])
    eng.step(steps)
    out = results(eng, m)
    eng.close()
    return out


def segments(m, eng, k, states, changes, steps=2):
    """For every (change, params of replica r) in `changes`: change(eng), `steps` steps; each replica against its twin from the state the
    segment started in."""
    for i, (change, params_of) in enumerate(changes):
        eng.sync()
        mid = {a: eng.get_attr(a).copy() for a in STATE}
        change(eng)
        eng.step(steps)
        x, v, lam = results(eng, m)
        for r in range(k):
            assert_replica((x[r], v[r], {t: l[r] for t, l in lam.items()}), twin(dict(m, params=params_of(r)), mid, r, states[r][2], steps), (i, r))


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT, LAUNCH], ids=["graph", "resident", "launch"])
def test_source_switching(mode):
    """rows -> per-constraint -> rows -> shared: each call selects its source, each segment equals its twins, and
    pbd_get_replica_materials reports the source in force."""
    m = model("fem_volume_bar")
    k = 3
    t = 9
    cnt = int((m["types"] == t).sum())
    states = [replica_state(m, r) for r in range(k)]
    eng = engine(m, mode, replicas=k)
    set_state(eng, states)
    rows = np.array([[1.0e5 * (1 + r), 0.1 * r] for r in range(k)], np.float32)
    rows2 = rows[::-1].copy()
    f = field(m, t, k, 5)
    per = lambda rr: (lambda r: with_materials(m, {t: np.repeat(rr[:, None], cnt, axis=1)}, r)["params"])
    changes = [(lambda e: e.set_replica_materials(t, rows), per(rows)),
               (lambda e: e.set_replica_constraint_materials(t, f), lambda r: with_materials(m, {t: f}, r)["params"]),
               (lambda e: e.set_replica_materials(t, rows2), per(rows2)),
               (lambda e: e.set_replica_materials(t, None), lambda r: m["params"])]
    reported = []
    for change, params_of in changes:
        segments(m, eng, k, states, [(change, params_of)])
        reported.append(eng.get_replica_materials(t))
    shared = m["params"][m["types"] == t][:, MAT_COLS[t]]
    assert np.array_equal(reported[0], np.repeat(rows[:, None], cnt, axis=1))
    assert np.array_equal(reported[1], f)
    assert np.array_equal(reported[2], np.repeat(rows2[:, None], cnt, axis=1))
    assert np.array_equal(reported[3], np.stack([shared] * k))
    # NULL of the per-constraint call: the shared parameters as well
    eng.set_replica_constraint_materials(t, f)
    eng.set_replica_constraint_materials(t, None)
    assert np.array_equal(eng.get_replica_materials(t), np.stack([shared] * k))
    eng.close()


def test_lifetime():
    """A mode switch mid-run gives the same bits; added constraints keep the old per-replica values and carry their own in every replica;
    pbd_set_replicas drops the override."""
    m = model("fem_volume_bar")
    k = 3
    t = 9
    states = [replica_state(m, r) for r in range(k)]
    f = field(m, t, k, 6)
    runs = []
    for switch in (False, True):
        eng = engine(m, GRAPH, replicas=k)
        set_state(eng, states)
        eng.set_replica_constraint_materials(t, f)
        eng.step(2)
        if switch:
            eng.set_mode(RESIDENT)
            eng.step(1)
            eng.set_mode(LAUNCH)
        else:
            eng.step(1)
        eng.step(1)
        runs.append(results(eng, m))
        eng.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])

    # an added FEMTet constraint: its parameters in every replica, the old constraints their per-replica values
    tet = m["bodies"][np.nonzero(m["types"] == t)[0][5]]
    added = np.array([[0.0] * 10 + [3.0e4, 0.2]], np.float32)
    added[0, :10] = m["params"][np.nonzero(m["types"] == t)[0][5]][:10]
    n0 = len(m["types"])
    m2 = dict(m, types=np.append(m["types"], t), bodies=np.vstack([m["bodies"], tet[None]]),
              params=np.vstack([m["params"], np.pad(added, ((0, 0), (0, m["params"].shape[1] - 12)))]))
    groups = (np.array([0] + [int(o) for o in m["off"][1:]] + [n0 + 1], np.uint32), np.append(m["ids"], n0).astype(np.uint32))
    for mode in (GRAPH, RESIDENT):
        eng = engine(m, mode, replicas=k)
        set_state(eng, states)
        eng.set_replica_constraint_materials(t, f)
        eng.step(1)
        eng.sync()
        mid = {a: eng.get_attr(a).copy() for a in STATE}
        eng.add_constraints(t, tet[None], added)
        eng.set_groups(*groups)
        want = np.concatenate([f, np.repeat(added[None, :, 10:12], k, axis=0)], axis=1)
        assert np.array_equal(eng.get_replica_materials(t), want)
        eng.step(2)
        x, v, lam = results(eng, m)
        eng.close()
        for r in range(k):
            mr = dict(m2, params=with_materials(m2, {t: want}, r)["params"], off=groups[0], ids=groups[1])
            xs, vs, _ = twin(mr, mid, r, states[r][2], 2)
            assert np.array_equal(x[r], xs) and np.array_equal(v[r], vs), (mode, r)

    eng = engine(m, GRAPH, replicas=k)
    eng.set_replica_constraint_materials(t, f)
    eng.set_replicas(2)
    shared = m["params"][m["types"] == t][:, MAT_COLS[t]]
    assert np.array_equal(eng.get_replica_materials(t), np.stack([shared] * 2))
    eng.set_replica_constraint_materials(t, f[:2])
    eng.clear_constraints()
    eng.add_flat(m["types"], m["bodies"], m["params"])
    eng.set_groups(m["off"], m["ids"])
    assert np.array_equal(eng.get_replica_materials(t), np.stack([shared] * 2))
    eng.close()


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda()


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
@pytest.mark.parametrize("before", ["shared", "rows", "constraint"])
def test_masked_device_writes(mode, before):
    """NaN in the rows of the replicas left out: they keep exactly the parameters they had (shared, rows or per-constraint); the written
    ones take theirs.  Each replica equals its twin over the segment after the write."""
    import torch
    m = model("xpbd_cloth64")
    k = 5
    t = 1
    cnt = int((m["types"] == t).sum())
    states = [replica_state(m, r) for r in range(k)]
    eng = engine(m, mode, replicas=k)
    set_state(eng, states)
    rows = np.array([[1.0e4 * (r + 1)] for r in range(k)], np.float32)
    old = {"shared": np.stack([m["params"][m["types"] == t][:, [1]]] * k), "rows": np.repeat(rows[:, None], cnt, axis=1), "constraint": field(m, t, k, 7)}[before]
    if before == "rows":
        eng.set_replica_materials(t, rows)
    elif before == "constraint":
        eng.set_replica_constraint_materials(t, old)
    eng.step(1)
    new = field(m, t, k, 8)
    mask = np.array([1, 0, 1, 0, 0], bool)
    src = new.copy()
    src[~mask] = np.nan
    eng.set_replica_constraint_materials_device(t, dev(src), replicas=torch.from_numpy(mask).cuda(), stream=torch.cuda.current_stream().cuda_stream)
    want = np.where(mask[:, None, None], new, old)
    assert np.array_equal(eng.get_replica_materials(t), want)
    segments(m, eng, k, states, [(lambda e: None, lambda r: with_materials(m, {t: want}, r)["params"])])
    eng.close()


def test_stream_order_without_host_sync():
    """The device form behind a spinning caller stream: the engine reads what the caller wrote after the spin, the host is not held, and
    the source may be freed and reused on the caller's stream right after the call."""
    import time
    import torch
    m = model("xpbd_cloth64")
    k = 3
    t = 1
    states = [replica_state(m, r) for r in range(k)]
    eng = engine(m, GRAPH, replicas=k)
    set_state(eng, states)
    eng.set_replica_constraint_materials(t, field(m, t, k, 9))  # on: the calls below switch nothing
    eng.step(1); eng.sync()
    want = field(m, t, k, 10)
    side = torch.cuda.Stream()
    src, staged = torch.zeros(want.size, device="cuda"), dev(want)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        src.copy_(staged)
        t0 = time.perf_counter()
        eng.set_replica_constraint_materials_device(t, src, stream=side.cuda_stream)
        held = time.perf_counter() - t0
        del src
        junk = torch.full((want.size,), float("nan"), device="cuda")  # the freed block handed out again on the caller's stream
    assert held < 0.02, held  # the spin lasts some 50 ms
    assert np.array_equal(eng.get_replica_materials(t), want)
    side.synchronize()
    del junk
    eng.close()


def test_no_replan_when_values_change_and_replan_when_switched():
    """Repeat calls keep the image -- the multipliers of the last step survive them -- and the graph engine stays bit-identical to a launch
    engine; switching the override on or off plans the image again (multipliers back to zero), so the captured step is captured again."""
    import torch
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k = 3
    t = 1
    states = [replica_state(m, r) for r in range(k)]
    engines = [engine(m, mode, replicas=k) for mode in (GRAPH, LAUNCH)]
    for e in engines:
        set_state(e, states)
        e.step(1)
        assert e.lambdas(_capi.DISTANCE_XPBD)[0].any()
        e.set_replica_constraint_materials(t, field(m, t, k, 11))
        assert not e.lambdas(_capi.DISTANCE_XPBD)[0].any()  # switched on: planned again
        e.step(1)
    for rnd in range(3):
        f = field(m, t, k, 20 + rnd)
        for e in engines:
            before = e.lambdas(_capi.DISTANCE_XPBD)[0].copy()
            assert before.any()
            if rnd % 2:
                e.set_replica_constraint_materials(t, f)
            else:
                e.set_replica_constraint_materials_device(t, dev(f), stream=torch.cuda.current_stream().cuda_stream)
            assert np.array_equal(e.lambdas(_capi.DISTANCE_XPBD)[0], before), rnd
            e.step(2)
        xs = [e.get_attr(X) for e in engines]
        assert np.array_equal(xs[0], xs[1]), rnd
    for e in engines:
        e.set_replica_constraint_materials(t, None)
        e.lambdas(_capi.DISTANCE_XPBD)
        assert not e.lambdas(_capi.DISTANCE_XPBD)[0].any()  # switched off: planned again
        e.close()


def test_refusals_leave_the_state_unchanged():
    import torch
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k = 3
    t = 1
    states = [replica_state(m, r) for r in range(k)]
    f = field(m, t, k, 12)
    one = engine(m, GRAPH)
    with pytest.raises(_capi.PbdError, match="single-scene engine"):
        _capi._ck(_capi.lib().pbd_set_replica_constraint_materials(one._h, t, f.ctypes.data))
    one.close()
    eng, ref = engine(m, GRAPH, replicas=k), engine(m, GRAPH, replicas=k)
    for e in (eng, ref):
        set_state(e, states)
        e.set_replica_constraint_materials(t, f)
        e.step(1)
    h = eng._h
    lib = _capi.lib()
    good = dev(f)
    mask = torch.ones(k, dtype=torch.bool, device="cuda")
    for call, match in ((lambda: lib.pbd_set_replica_constraint_materials(h, 99, f.ctypes.data), "unknown constraint type"),
                        (lambda: lib.pbd_set_replica_constraint_materials(h, _capi.BALLJOINT, f.ctypes.data), "no material parameters"),
                        (lambda: lib.pbd_set_replica_constraint_materials(h, _capi.FEMTET, f.ctypes.data), "no constraints of type"),
                        (lambda: lib.pbd_set_replica_constraint_materials_device(h, t, None, None, None), "mat == NULL"),
                        (lambda: lib.pbd_set_replica_constraint_materials_device(h, t, f.ctypes.data, None, None), "pageable host memory"),
                        (lambda: lib.pbd_set_replica_constraint_materials_device(h, t, good.data_ptr(), f.ctypes.data, None), "replicas is pageable host memory"),
                        (lambda: lib.pbd_set_replica_constraint_materials_device(h, _capi.RB_PARTICLE_BALLJOINT, good.data_ptr(), mask.data_ptr(), None),
                         "no material parameters"),
                        (lambda: lib.pbd_get_replica_materials(h, _capi.BALLJOINT, f.ctypes.data), "no material parameters")):
        assert call() != 0, match
        assert match in lib.pbd_last_error().decode(), (match, lib.pbd_last_error())
    # a stream being captured into a graph
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        s = torch.cuda.current_stream().cuda_stream
        rc = lib.pbd_set_replica_constraint_materials_device(h, t, good.data_ptr(), None, _capi.C.c_void_p(s))
    assert rc != 0 and "captured" in lib.pbd_last_error().decode()
    assert np.array_equal(eng.get_replica_materials(t), f)
    for e in (eng, ref):
        e.step(2)
    xa, va, la = results(eng, m); xb, vb, lb = results(ref, m)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and all(np.array_equal(la[q], lb[q]) for q in la)
    eng.close(); ref.close()


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_negative_controls_fail_the_gate(mode):
    """The comparison detects wrong values: rows shifted by one replica, the values given in device order instead of the order the
    constraints were added, and replica 0's values for every replica each move some compared replica away from its solo run."""
    m = model("xpbd_cloth64")
    k = 3
    t = 1
    f = field(m, t, k, 13)
    probe = engine(m, mode, replicas=k)
    probe.step(1)
    _, ids = probe.lambdas(t)  # the device order of the type's constraints (insertion ids; the type's ids are 0 .. count-1 in order)
    probe.close()
    local = np.argsort(np.argsort(ids))  # insertion id -> local index is the identity here; device position -> local index
    assert not np.array_equal(local, np.arange(len(ids)))
    wrong = {"shifted": np.roll(f, 1, axis=0), "device order": np.ascontiguousarray(f[:, local]), "replica 0": np.stack([f[0]] * k)}
    states = [replica_state(m, r) for r in range(k)]
    for what, given in wrong.items():
        eng = engine(m, mode, replicas=k)
        set_state(eng, states)
        eng.set_replica_constraint_materials(t, given)
        x, v, lam = run(eng, m)
        eng.close()
        with pytest.raises(AssertionError):
            for r in range(k):
                assert_replica((x[r], v[r], {q: l[r] for q, l in lam.items()}), solo(with_materials(m, {t: f}, r), states[r]), (what, r))
        print("negative control '%s' fails the gate" % what)
