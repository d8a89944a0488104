"""Contact sensors (pbd_sense_contacts, pbd_get_contact_sensors, pbd_get_contact_sensors_device): per replica and rigid collider, the contacts
the step found and the impulse the particles exerted.  The impulses balance the momentum the contacts gave the particles (checked in lockstep
against a twin without colliders), the counts are those of the contact record, the values are the same bits in every mode, in every run and
for a replica of a batch as for the single scene given its rows, and sensing changes no state."""
import re

import numpy as np
import pytest

import contact_util as cu
from batch_util import AUTO, GRAPH, LAUNCH, RESIDENT, engine, replica_state, set_state
from test_gpu_batch_contacts import CAP, _model, _pc, batch_engine, contacts, final, solo_engine

pytestmark = pytest.mark.gpu

NAME = "contact_cloth24"
SPIN = 100_000_000  # torch.cuda._sleep cycles: some 50 ms on an H100
X, V, X0, OLDX, LASTX = range(5)


def sensing_batch(m, mode, k, scene):
    eng = batch_engine(m, NAME, mode, k, scene)
    eng.sense_contacts(True)
    return eng


def run_sensors(eng, steps):
    """The sensors after each of `steps` steps."""
    out = []
    for _ in range(steps):
        eng.step(1)
        c, i = eng.contact_sensors()
        out.append((c.copy(), i.copy()))
    return out


def test_impulses_balance_the_particles_momentum_in_lockstep():
    """Every step, a twin without colliders takes the sensing batch's X, V, OLDX and LASTX and both step once while the cloth falls onto
    and slides over the obstacles.  Positions stay bit-identical (contacts change velocities only); per replica, -sum_k impulse equals
    sum_i m_i (v_with - v_without), and per collider too where no particle touched two colliders."""
    m = _model(NAME)
    k, n = 3, len(m["x"])
    scene = cu.batch_scene(k, cu.footprint(m["x"]), empty=-1)
    eng = sensing_batch(m, GRAPH, k, scene)
    twin = engine(m, GRAPH, replicas=k)
    set_state(twin, [replica_state(m, r) for r in range(k)])
    mass = np.stack([replica_state(m, r)[2] for r in range(k)]).astype(np.float64)
    per_collider_checked, touched = 0, 0
    for step in range(150):
        for a in (X, V, OLDX, LASTX):
            twin.set_attr(a, eng.get_attr(a))
        eng.step(1); twin.step(1)
        xw, vw = final(eng); xo, vo = final(twin)
        assert np.array_equal(xw, xo), step
        count, impulse = eng.contact_sensors()
        rec = contacts(eng)
        dp = mass[..., None] * (vw.astype(np.float64) - vo.astype(np.float64))  # (K, n, 3)
        for r in range(k):
            scale = max(np.abs(dp[r]).sum(), 1e-6)
            assert np.abs(-impulse[r].astype(np.float64).sum(axis=0) - dp[r].sum(axis=0)).max() <= 5e-5 * scale + 1e-6, (step, r)
            mine = rec[rec["particle"] // n == r]
            assert np.array_equal(count[r], np.bincount(mine["body"], minlength=len(count[r]))), (step, r)
            parts = mine["particle"] - r * n
            if len(parts) and len(np.unique(parts)) == len(parts):  # each particle touches at most one collider
                for j in range(count.shape[1]):
                    sel = parts[mine["body"] == j]
                    want = dp[r][sel].sum(axis=0)
                    assert np.abs(-impulse[r, j] - want).max() <= 5e-5 * max(np.abs(dp[r][sel]).sum(), 1e-6) + 1e-6, (step, r, j)
                per_collider_checked += 1
            touched += int(count[r].sum() > 0)
    print("lockstep: %d replica-steps with contacts, %d checked per collider" % (touched, per_collider_checked))
    assert touched > 100 and per_collider_checked > 20
    eng.close(); twin.close()


def test_counts_equal_the_contact_record():
    """Every step: count[r][k] is the number of pbd_get_contacts entries of replica r on collider k's body id (distinct ids)."""
    m = _model(NAME)
    k, n = 4, len(m["x"])
    scene = cu.batch_scene(k, cu.footprint(m["x"]))
    eng = sensing_batch(m, RESIDENT, k, scene)
    total = 0
    for step in range(120):
        eng.step(1)
        count, _ = eng.contact_sensors()
        rec = contacts(eng)
        for r in range(k):
            mine = rec[rec["particle"] // n == r]
            assert np.array_equal(count[r], np.bincount(mine["body"], minlength=4)), (step, r)
        total += int(count.sum())
    assert total > 1000 and not count[k - 1].any()  # the last replica has only empty boxes
    eng.close()


_solo = {}


def solo_sensors(r, steps):
    if (r, steps) not in _solo:
        m = _model(NAME)
        cols, bx, bv, bw = cu.replica_scene(r, cu.footprint(m["x"]))
        eng = solo_engine(m, NAME, r, cols, bx, bv, bw)
        eng.sense_contacts(True)
        _solo[(r, steps)] = run_sensors(eng, steps)
        eng.close()
    return _solo[(r, steps)]


@pytest.mark.parametrize("k", [2, 3, 300])
def test_bit_identity_across_modes_runs_and_single_scenes(k):
    """The sensors of every step are the same bits in GRAPH, RESIDENT, LAUNCH and AUTO and in a second GRAPH run, and replicas
    {0, 1, k/2, k-1} report what a single-scene engine given their rows reports."""
    m = _model(NAME)
    scene = cu.batch_scene(k, cu.footprint(m["x"]), empty=-1)
    steps = 80
    runs = []
    for mode in (GRAPH, RESIDENT, LAUNCH, AUTO, GRAPH):
        eng = sensing_batch(m, mode, k, scene)
        runs.append(run_sensors(eng, steps))
        eng.close()
    for other in runs[1:]:
        for (c0, i0), (c1, i1) in zip(runs[0], other):
            assert np.array_equal(c0, c1) and np.array_equal(i0.view(np.uint32), i1.view(np.uint32))
    for r in sorted({0, 1, k // 2, k - 1}):
        for s, ((c, i), (cs, is_)) in enumerate(zip(runs[0], solo_sensors(r, steps))):
            assert np.array_equal(c[r], cs[0]) and np.array_equal(i[r].view(np.uint32), is_[0].view(np.uint32)), (k, r, s)
    assert sum(int(c.sum()) for c, _ in runs[0]) > 0


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_sensing_changes_no_state(mode):
    """The state is bit-identical with sensing on and off; sensing adds one launch per step and plans and captures nothing again."""
    m = _model(NAME)
    k = 3
    scene = cu.batch_scene(k, cu.footprint(m["x"]))
    on, off = sensing_batch(m, mode, k, scene), batch_engine(m, NAME, mode, k, scene)
    for e in (on, off):
        e.step(1); e.sync()
    before = [(e.stats().images_planned, e.stats().graph_captures, e.stats().kernel_launches) for e in (on, off)]
    on.step(100); off.step(100)
    after = [(e.stats().images_planned, e.stats().graph_captures, e.stats().kernel_launches) for e in (on, off)]
    assert before[0][:2] == after[0][:2] and before[1][:2] == after[1][:2]
    assert after[0][2] - before[0][2] == after[1][2] - before[1][2] + 100
    xa, va = final(on); xb, vb = final(off)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb)
    # switching sensing off and on again plans and captures nothing either, and zeroes the sensors
    on.sense_contacts(False); off.sense_contacts(True)
    c, i = off.contact_sensors()
    assert not c.any() and not i.any()
    on.step(20); off.step(20)
    xa, va = final(on); xb, vb = final(off)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb)
    assert (on.stats().images_planned, on.stats().graph_captures) == after[0][:2]
    on.close(); off.close()


def test_negative_controls():
    """A replica whose colliders are moved far away reports count 0 and impulse exactly 0; a higher friction of one replica's colliders
    changes the tangential part of its impulses."""
    m = _model(NAME)
    k = 4
    fp = cu.footprint(m["x"])
    scene = cu.batch_scene(k, fp, empty=-1)
    steps = 60

    def sensors(sc):
        eng = sensing_batch(m, GRAPH, k, sc)
        out = run_sensors(eng, steps)
        eng.close()
        return out
    base = sensors(scene)
    cols, bx, bv, bw = scene
    away = cu.batch_scene(k, fp, empty=-1, shift=np.array([[0.0, 0.0, 0.0], [0.0, 50.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]]))
    far = sensors(away)
    for c, i in far:
        assert not c[1].any() and not i[1].view(np.uint32).any()
    assert sum(int(c[1].sum()) for c, _ in base) > 0
    rough = [list(c) for c in cols]
    rough[2] = [dict(d, friction=d["friction"] + 0.5) for d in rough[2]]
    fr = sensors((rough, bx, bv, bw))
    assert any(not np.array_equal(i0[2], i1[2]) for (_, i0), (_, i1) in zip(base, fr))
    for (c0, i0), (c1, i1) in zip(base, fr):
        assert np.array_equal(c0[0], c1[0]) and np.array_equal(i0[0], i1[0])  # the other replicas are untouched


def test_swapped_rows_swap_the_sensors():
    """Two replicas with the same particle state and swapped collider rows report swapped sensors, bit for bit, at every step."""
    m = _model(NAME)
    k = 3
    fp = cu.footprint(m["x"])
    cols, bx, bv, bw = cu.batch_scene(k, fp, empty=-1)
    order = [0, 2, 1]
    runs = []
    for sc in ((cols, bx, bv, bw), ([cols[j] for j in order], bx[order], bv[order], bw[order])):
        from batch_util import engine as plain
        eng = plain(m, GRAPH, replicas=k)
        st = replica_state(m, 0)
        set_state(eng, [st] * k)
        eng.set_replica_colliders(_pc(m, NAME), [[cu.to_capi(d) for d in c] for c in sc[0]], sc[1], sc[2], sc[3])
        eng.set_contact_params(tolerance=cu.TOL, stiffness=100.0, max_iter_v=5)
        eng.sense_contacts(True)
        runs.append(run_sensors(eng, 60))
        eng.close()
    seen = 0
    for (c0, i0), (c1, i1) in zip(*runs):
        assert np.array_equal(c0[order], c1) and np.array_equal(i0[order].view(np.uint32), i1.view(np.uint32))
        seen += int(c0[1].sum() + c0[2].sum())
    assert seen > 0


def test_device_get_in_stream_order():
    """A device get behind a spinning caller stream delivers the sensors of the steps enqueued before it, into torch tensors, without a host
    synchronisation; a count buffer is uint32."""
    import torch
    m = _model(NAME)
    k = 3
    eng = sensing_batch(m, GRAPH, k, cu.batch_scene(k, cu.footprint(m["x"]), empty=-1))
    eng.step(40)
    want_c, want_i = eng.contact_sensors()
    assert want_c.sum() > 0
    side = torch.cuda.Stream()
    count = torch.zeros(k * 4, dtype=torch.int32, device="cuda").view(torch.uint32)
    impulse = torch.full((k * 4 * 3,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        impulse.fill_(float("nan"))
        eng.get_contact_sensors_device(count, impulse, stream=side.cuda_stream)
        c2, i2 = count.view(torch.int32).clone(), impulse.clone()
    eng.step(5)  # enqueued after the get: not part of what it delivers
    side.synchronize()
    assert np.array_equal(c2.cpu().numpy().view(np.uint32).reshape(k, 4), want_c)
    assert np.array_equal(i2.cpu().numpy().reshape(k, 4, 3), want_i)
    eng.close()


def test_single_scene_sensors_and_refusals():
    """A single scene (pbd_set_colliders) has sensors too; the get calls are refused while sensing is off, without colliders, for host
    memory and on a capturing stream; set_replicas keeps the switch."""
    import torch
    from positionbaseddynamics_b200 import _capi
    L = _capi.lib()
    m = _model(NAME)
    cols, bx, bv, bw = cu.replica_scene(0, cu.footprint(m["x"]))
    eng = solo_engine(m, NAME, 0, cols, bx, bv, bw)

    def refused(rc, pattern):
        assert rc != 0
        assert re.search(pattern, L.pbd_last_error().decode()), L.pbd_last_error().decode()
    buf = torch.zeros(4 * 3, device="cuda")
    with pytest.raises(_capi.PbdError, match="sensing is off"):
        eng.contact_sensors()
    refused(L.pbd_get_contact_sensors_device(eng._h, None, buf.data_ptr(), None), "sensing is off")
    eng.sense_contacts(True)
    eng.step(60)
    c, i = eng.contact_sensors()
    assert c.shape == (1, 4) and i.shape == (1, 4, 3) and c.sum() > 0
    host_np = np.zeros(12, np.float32)
    pinned = torch.zeros(12).pin_memory()
    refused(L.pbd_get_contact_sensors_device(eng._h, None, host_np.ctypes.data, None), "pageable")
    refused(L.pbd_get_contact_sensors_device(eng._h, None, pinned.data_ptr(), None), "pinned")
    with pytest.raises(ValueError, match="element type"):
        eng.get_contact_sensors_device(count=torch.zeros(4, dtype=torch.int32, device="cuda"))
    g = torch.cuda.CUDAGraph()
    y = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        with pytest.raises(_capi.PbdError, match="captured"):
            eng.get_contact_sensors_device(impulse=buf, stream=torch.cuda.current_stream().cuda_stream)
        y += 1
    g.replay()
    torch.cuda.synchronize()
    c2, i2 = eng.contact_sensors()
    assert np.array_equal(c, c2) and np.array_equal(i, i2)
    eng.set_colliders([], [])
    with pytest.raises(_capi.PbdError, match="no rigid colliders"):
        eng.contact_sensors()
    eng.close()
    # a batch: set_replicas keeps the switch, and sensors come back with the next colliders
    k = 2
    b = engine(m, GRAPH)
    b.sense_contacts(True)
    b.set_replicas(k)
    with pytest.raises(_capi.PbdError, match="no rigid colliders"):
        b.contact_sensors()
    set_state(b, [replica_state(m, r) for r in range(k)])
    sc = cu.batch_scene(k, cu.footprint(m["x"]), empty=-1)
    b.set_replica_colliders(_pc(m, NAME), [[cu.to_capi(d) for d in l] for l in sc[0]], sc[1], sc[2], sc[3])
    c, i = b.contact_sensors()
    assert c.shape == (k, 4) and not c.any() and not i.any()
    b.step(60)
    assert b.contact_sensors()[0].sum() > 0
    b.close()


def test_example_runs():
    """examples/cloth_pusher_batch.py with a small K ends where the same loop on the host calls ends."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "examples", "cloth_pusher_batch.py"), "--replicas", "6", "--steps", "240"],
                         capture_output=True, text=True, timeout=900)
    print(out.stdout)
    assert out.returncode == 0, out.stderr
    assert "device loop = host loop, bit for bit: yes" in out.stdout
