"""Rigid-body state of a batch in device memory (pbd_set_rigid_bodies_device / pbd_get_rigid_bodies_device) and repeat host sets of the
same bodies: round trips against the host calls, masked writes, restarts, stream order, no re-plan or re-capture, and every refusal."""
import re

import numpy as np
import pytest

import rigid_batch_util as rb
from batch_util import GRAPH, LAUNCH, RESIDENT

pytestmark = pytest.mark.gpu
SPIN = 200_000_000  # torch.cuda._sleep cycles: long enough that the engine would overtake the caller's stream if it did not wait


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).to("cuda")


def cur():
    import torch
    return torch.cuda.current_stream().cuda_stream


def batch(m, mode, k):
    eng = rb.engine(m, mode, replicas=k, bodies=[rb.replica_bodies(m, r) for r in range(k)])
    rb.set_particles(eng, [rb.particle_state(m, r) for r in range(k)])
    return eng


def stacked(m, rs):
    return [np.stack([rb.replica_bodies(m, r)[j] for r in rs]) for j in range(6)]


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT])
def test_round_trip_and_device_set_equals_host_set(mode):
    """get_rigid_bodies_device returns what get_rigid_bodies does; a device set and a host set of the same rows leave identical bits
    (masses and inertias converted with the same IEEE divisions) and step identically."""
    import torch
    m = rb.model("rig")
    k, nb = 3, len(m["bm"])
    rows = stacked(m, [2, 0, 1])
    engines = [batch(m, mode, k) for _ in range(2)]
    for e in engines:
        e.step(1)
    engines[0].set_replica_rigid_bodies(*rows)
    mass, x, q, inertia, v, w = rows
    engines[1].set_rigid_bodies_device(dev(x), dev(q), v=dev(v), omega=dev(w), mass=dev(mass), inertia=dev(inertia), stream=cur())
    outs = [tuple(torch.empty(k * nb * c, device="cuda") for c in (3, 4, 3, 3)) for _ in engines]
    for e, o in zip(engines, outs):
        e.get_rigid_bodies_device(*o, stream=cur())
        torch.cuda.synchronize()
        host = e.get_rigid_bodies()
        got = np.concatenate([a.cpu().numpy().reshape(k, nb, -1) for a in o], axis=2)
        assert np.array_equal(got, host)
    assert np.array_equal(engines[0].get_rigid_bodies(), engines[1].get_rigid_bodies())
    res = [rb.run(e, m) for e in engines]
    for r in range(k):
        rb.same(res[0], tuple(a[r] if not isinstance(a, dict) else {t: l[r] for t, l in a.items()} for a in res[1]), r)
    for e in engines:
        e.close()


@pytest.mark.parametrize("mode", [GRAPH, LAUNCH, RESIDENT])
def test_masked_restart_matches_fresh_solo_engines(mode):
    """A mid-run restart of replicas 0 and 2 through masked device writes of particles (x, v, oldX, lastX) and bodies, with NaN in the rows
    of the replica left out: the restarted replicas equal fresh single-scene engines, the other one is untouched."""
    import torch
    from positionbaseddynamics_b200 import _capi
    m = rb.model("rig")
    k = 3
    eng = batch(m, mode, k)
    eng.step(3)
    before = rb.results(eng, m)
    mask = torch.tensor([1, 0, 1], dtype=torch.uint8, device="cuda")
    fresh = [rb.particle_state(m, 10 + r) for r in range(k)]
    fb = stacked(m, [10, 11, 12])
    nan = np.float32(np.nan)
    px = np.stack([s[0] for s in fresh]); pv = np.stack([s[1] for s in fresh])
    px[1] = nan; pv[1] = nan
    for j in range(6):
        fb[j] = fb[j].copy(); fb[j][1] = nan
    for a, src in ((_capi.ATTR_X, px), (_capi.ATTR_V, pv), (_capi.ATTR_OLDX, px), (_capi.ATTR_LASTX, px)):
        eng.set_attr_device(a, dev(src), replicas=mask, stream=cur())
    masses = np.stack([s[2] for s in fresh]); masses[1] = nan
    eng.set_masses_device(dev(masses), replicas=mask, stream=cur())
    mass, x, q, inertia, v, w = fb
    eng.set_rigid_bodies_device(dev(x), dev(q), v=dev(v), omega=dev(w), mass=dev(mass), inertia=dev(inertia), replicas=mask, stream=cur())
    torch.cuda.synchronize()
    mid = rb.results(eng, m)
    assert np.array_equal(mid[0][1], before[0][1]) and np.array_equal(mid[3][1], before[3][1])
    out = rb.run(eng, m)
    eng.close()
    for r in (0, 2):
        solo = rb.engine(m, mode, bodies=rb.replica_bodies(m, 10 + r))
        rb.set_particles(solo, [fresh[r]])
        rb.same(out, rb.run(solo, m), r, mode)
        solo.close()


def test_moving_anchors_each_step_without_replan_or_recapture():
    """The static anchors of the rig moved before every step, by a device set on a batch and by set_rigid_bodies on single-scene
    engines: bit for bit the same.  Neither the device sets nor a repeat host set of the same n plans the image again or captures the step
    graph again (pbd_stats images_planned / graph_captures stay where the first step left them)."""
    import torch
    m = rb.model("rig")
    k, steps = 3, 6
    anchors = np.nonzero(m["bm"] == 0)[0]
    engines = [batch(m, mode, k) for mode in (GRAPH, LAUNCH, RESIDENT)]
    solos = [rb.engine(m, GRAPH, bodies=rb.replica_bodies(m, r)) for r in range(k)]
    for r, s in enumerate(solos):
        rb.set_particles(s, [rb.particle_state(m, r)])
    for e in engines:
        e.step(1)
    for s in solos:
        s.step(1)
    counters = [(e.stats().images_planned, e.stats().graph_captures) for e in engines]
    assert counters[0][1] == 1 and counters[1][1] == 0 and all(c[0] >= 1 for c in counters), counters
    for i in range(steps):
        state = engines[0].get_rigid_bodies()
        x = state[..., :3].copy(); q = state[..., 3:7].copy()
        x[:, anchors, 1] += np.float32(0.01 * (i + 1))
        for e in engines:
            e.set_rigid_bodies_device(dev(x), dev(q), v=dev(state[..., 7:10]), omega=dev(state[..., 10:13]), stream=cur())
        for r, s in enumerate(solos):
            own = s.get_rigid_bodies()
            xs = own[:, :3].copy(); xs[anchors, 1] = x[r, anchors, 1]
            mass, _, _, inertia, _, _ = rb.replica_bodies(m, r)
            s.set_rigid_bodies(mass, xs, own[:, 3:7], inertia, v=own[:, 7:10], omega=own[:, 10:13])
        if i == steps // 2:  # a repeat host set of the same n, stream-ordered too
            for e in engines:
                cur_state = e.get_rigid_bodies()
                mass = np.stack([rb.replica_bodies(m, r)[0] for r in range(k)]); inertia = np.stack([rb.replica_bodies(m, r)[3] for r in range(k)])
                e.set_replica_rigid_bodies(mass, cur_state[..., :3], cur_state[..., 3:7], inertia, cur_state[..., 7:10], cur_state[..., 10:13])
        for e in engines + solos:
            e.step(1)
        torch.cuda.synchronize()
    res = [rb.results(e, m) for e in engines]
    for r in range(k):
        solo = rb.results(solos[r], m)
        for out in res:
            rb.same(out, solo, r)
    assert [(e.stats().images_planned, e.stats().graph_captures) for e in engines] == counters
    assert engines[0].stats().kernel_launches == engines[1].stats().kernel_launches
    for e in engines + solos:
        e.close()


def test_caller_stream_order_without_host_sync():
    """A caller stream held back by a spin: the engine reads the body rows written on it after the spin, and a get is read on that stream
    after the copy."""
    import torch
    m = rb.model("rig")
    k, nb = 3, len(m["bm"])
    eng = batch(m, GRAPH, k)
    eng.step(1); eng.sync()
    want = eng.get_rigid_bodies().copy()
    want[..., :3] += np.float32(0.25)
    side = torch.cuda.Stream()
    x, q = torch.zeros(k * nb * 3, device="cuda"), dev(want[..., 3:7])
    staged = dev(want[..., :3])
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        x.copy_(staged)
        eng.set_rigid_bodies_device(x, q, v=dev(want[..., 7:10]), omega=dev(want[..., 10:13]), stream=side.cuda_stream)
    assert np.array_equal(eng.get_rigid_bodies(), want)
    out = torch.zeros(k * nb * 3, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        out.fill_(float("nan"))
        eng.get_rigid_bodies_device(x=out, stream=side.cuda_stream)
        copy = out.clone()
    side.synchronize()
    assert np.array_equal(copy.cpu().numpy().reshape(k, nb, 3), want[..., :3])
    eng.close()


def test_refusals_leave_the_state_unchanged():
    import torch
    from positionbaseddynamics_b200 import _capi
    L = _capi.lib()
    m = rb.model("rig")
    k, nb = 3, len(m["bm"])
    eng = batch(m, GRAPH, k)
    eng.step(1)
    snap = eng.get_rigid_bodies().copy()
    x, q = dev(snap[..., :3] + 1), dev(snap[..., 3:7])
    host_np = np.zeros(k * nb * 4, np.float32)
    pinned = torch.zeros(k * nb * 4).pin_memory()

    def refused(rc, pattern):
        assert rc != 0
        assert re.search(pattern, L.pbd_last_error().decode()), L.pbd_last_error().decode()
    for p, kind in ((host_np.ctypes.data, "pageable"), (pinned.data_ptr(), "pinned")):
        refused(L.pbd_set_rigid_bodies_device(eng._h, None, p, q.data_ptr(), None, None, None, None, None), kind)
        refused(L.pbd_set_rigid_bodies_device(eng._h, None, x.data_ptr(), p, None, None, None, None, None), kind)
        refused(L.pbd_set_rigid_bodies_device(eng._h, p, x.data_ptr(), q.data_ptr(), None, None, None, None, None), kind)
        refused(L.pbd_set_rigid_bodies_device(eng._h, None, x.data_ptr(), q.data_ptr(), None, None, None, p, None), kind)
        refused(L.pbd_get_rigid_bodies_device(eng._h, p, None, None, None, None), kind)
    refused(L.pbd_set_rigid_bodies_device(eng._h, None, None, q.data_ptr(), None, None, None, None, None), "x == NULL")
    refused(L.pbd_set_rigid_bodies_device(eng._h, None, x.data_ptr(), None, None, None, None, None, None), "q == NULL")
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        eng.set_rigid_bodies_device(host_np, q)
    with pytest.raises(ValueError, match="elements"):
        eng.set_rigid_bodies_device(x[:-3], q)
    g = torch.cuda.CUDAGraph()
    y = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        s = torch.cuda.current_stream().cuda_stream
        with pytest.raises(_capi.PbdError, match="captured"):
            eng.set_rigid_bodies_device(x, q, stream=s)
        with pytest.raises(_capi.PbdError, match="captured"):
            eng.get_rigid_bodies_device(x=x, stream=s)
        y += 1
    g.replay()
    torch.cuda.synchronize()
    # the host batch call: K*n >= 2^31 and null arrays
    refused(L.pbd_set_replica_rigid_bodies(eng._h, (1 << 31) // k + 1, host_np.ctypes.data, host_np.ctypes.data, host_np.ctypes.data, host_np.ctypes.data, None, None), "2\\^31")
    refused(L.pbd_set_replica_rigid_bodies(eng._h, nb, None, host_np.ctypes.data, host_np.ctypes.data, host_np.ctypes.data, None, None), "null argument")
    assert np.array_equal(eng.get_rigid_bodies(), snap)
    eng.step(1)
    assert np.isfinite(eng.get_rigid_bodies()).all()
    eng.close()
    one = rb.engine(m, GRAPH, bodies=rb.replica_bodies(m, 0))
    refused(L.pbd_set_replica_rigid_bodies(one._h, nb, *[a.ctypes.data for a in rb.replica_bodies(m, 0)[:4]], None, None), "pbd_set_replicas first")
    one.close()


def test_device_mass_writes_reach_the_collider_checks():
    """A single scene: a device write that makes a collider's static body dynamic is refused by the next step and by set_colliders, one
    that makes a dynamic body static lets set_colliders put a collider on it (the contact path reads the written masses back)."""
    import torch
    from positionbaseddynamics_b200 import _capi
    m = rb.model("rig")
    eng = rb.engine(m, GRAPH, bodies=rb.replica_bodies(m, 0))
    nb = len(m["bm"])
    anchor, box = int(np.nonzero(m["bm"] == 0)[0][0]), int(np.nonzero(m["bm"] != 0)[0][0])

    def collider(body):
        c = _capi.RigidCollider()
        c.shape, c.body = _capi.SHAPE_SPHERE, body
        c.dim[:] = (0.3, 0.0, 0.0)
        c.R[:] = (1, 0, 0, 0, 1, 0, 0, 0, 1)
        c.aabb_min[:] = (-1.0, -1.0, -1.0); c.aabb_max[:] = (1.0, 1.0, 1.0)
        return c
    ranges = [_capi.ParticleCollider(0, len(m["x"]), 0.5, 0.1)]
    eng.set_colliders(ranges, [collider(anchor)])
    eng.step(1)
    st = eng.get_rigid_bodies()
    x, q = dev(st[:, :3]), dev(st[:, 3:7])
    mass = rb.replica_bodies(m, 0)[0].copy()
    mass[anchor] = 1.0  # the collider's body made dynamic
    eng.set_rigid_bodies_device(x, q, mass=dev(mass), stream=cur())
    with pytest.raises(_capi.PbdError, match="not static any more"):
        eng.step(1)
    with pytest.raises(_capi.PbdError, match="has mass"):
        eng.set_colliders(ranges, [collider(anchor)])
    mass[anchor], mass[box] = 0.0, 0.0  # static again, and a dynamic box made static
    eng.set_rigid_bodies_device(x, q, mass=dev(mass), stream=cur())
    eng.set_colliders(ranges, [collider(anchor), collider(box)])
    eng.step(1); eng.sync()
    assert np.isfinite(eng.get_rigid_bodies()).all() and nb == len(eng.get_rigid_bodies())
    eng.close()
