"""Collider placement from device memory (pbd_set_replica_collider_poses_device): a batch whose obstacles move every step through the device
call steps bit for bit like one moved through pbd_set_replica_colliders with the same rows, writes only the masked replicas, keeps the
caller's stream order without a host synchronisation, plans and captures nothing again, and refuses what it cannot take with the colliders
in force left as they were."""
import ctypes as C
import re

import numpy as np
import pytest

import contact_util as cu
from batch_util import GRAPH, LAUNCH, RESIDENT, engine
from test_gpu_batch_contacts import _model, _pc, batch_engine, final

pytestmark = pytest.mark.gpu

NAME = "contact_cloth24"
SPIN = 100_000_000  # torch.cuda._sleep cycles: some 50 ms on an H100
# pbd_rigid_collider as a numpy record: a whole batch of rows goes to pbd_set_replica_colliders in one array
RC = np.dtype([("shape", "<i4"), ("body", "<u4"), ("dim", "<f4", 3), ("thickness", "<f4"), ("invert_sdf", "<i4"), ("restitution", "<f4"),
               ("friction", "<f4"), ("R", "<f4", 9), ("v1", "<f4", 3), ("v2", "<f4", 3), ("aabb_min", "<f4", 3), ("aabb_max", "<f4", 3)])
POSE = ["R", "v1", "v2", "aabb_min", "aabb_max"]


def rows(cols):
    """K lists of collider dicts -> (K*nR) RC records."""
    flat = [d for c in cols for d in c]
    a = np.zeros(len(flat), RC)
    for i, d in enumerate(flat):
        a[i] = (d["shape"], d["body"], d["dim"], d["thickness"], int(d["invert"]), d["restitution"], d["friction"], d["R"], d["v1"], d["v2"],
                d["aabb_min"], d["aabb_max"])
    return a


def pose(a):
    """The K*nR*21 placement floats of RC records."""
    return np.concatenate([a[f].reshape(len(a), -1) for f in POSE], axis=1).astype(np.float32)


def moved(a, bx, shift):
    """Records and body centres moved by shift (K, 3): v2, the bounding box and the centre of mass."""
    a = a.copy()
    K = len(shift); nR = len(a) // K
    s = np.repeat(shift.astype(np.float32), nR, axis=0)
    for f in ("v2", "aabb_min", "aabb_max"):
        a[f] += s
    return a, (bx.reshape(-1, 3) + s).reshape(bx.shape).astype(np.float32)


def shift_at(K, t):
    d = np.stack([np.array([np.cos(1.3 * r), 0.3 * np.sin(0.1 * t + r), np.sin(1.3 * r)]) for r in range(K)])
    return (0.01 * t * d).astype(np.float32)


def host_set(eng, m, a, bx, bv, bw):
    from positionbaseddynamics_b200 import _capi
    pcs = _pc(m, NAME)
    pa = (_capi.ParticleCollider * 1)(*pcs)
    nr = len(a) // eng.K
    p = lambda x: None if x is None else np.ascontiguousarray(x, np.float32).ctypes.data_as(C.c_void_p)
    _capi._ck(_capi.lib().pbd_set_replica_colliders(eng._h, 1, C.cast(pa, C.c_void_p), nr, a.ctypes.data_as(C.c_void_p), p(bx), p(bv), p(bw)))


def dev(a, dtype=np.float32):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype).reshape(-1)).cuda()


def cur():
    import torch
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT, LAUNCH], ids=["graph", "resident", "launch"])
@pytest.mark.parametrize("k", [2, 3, 300])
def test_device_poses_step_like_host_calls(k, mode):
    """Obstacles moved before every one of 110 steps: by the host call in one batch, by the device call with the same rows in the other.
    x and v are bit-identical after every 10 steps and at the end, and the device batch planned and captured nothing again."""
    m = _model(NAME)
    scene = cu.batch_scene(k, cu.footprint(m["x"]), empty=-1)
    base, bx, bv, bw = rows(scene[0]), scene[1], scene[2], scene[3]
    host, devb = batch_engine(m, NAME, mode, k, scene), batch_engine(m, NAME, mode, k, scene)
    for e in (host, devb):
        e.step(1); e.sync()
    counters = (devb.stats().images_planned, devb.stats().graph_captures)
    bvd, bwd = dev(bv), dev(bw)
    contacts = 0
    for t in range(1, 111):
        a, x = moved(base, bx, shift_at(k, t))
        host_set(host, m, a, x, bv, bw)
        devb.set_replica_collider_poses_device(dev(pose(a)), dev(x), bvd, bwd, stream=cur())
        host.step(1); devb.step(1)
        if t % 10 == 0:
            xh, vh = final(host); xd, vd = final(devb)
            assert np.array_equal(xh, xd) and np.array_equal(vh, vd), (k, mode, t)
            contacts += len(host.contacts(1 << 20)[0])
    assert contacts > 0
    assert (devb.stats().images_planned, devb.stats().graph_captures) == counters
    host.close(); devb.close()


def test_masked_write_leaves_the_other_replicas():
    """A masked write whose unmasked rows are NaN: the masked replicas take the new rows, the others step bit for bit like an engine whose
    colliders were not moved."""
    import torch
    m = _model(NAME)
    k = 4
    scene = cu.batch_scene(k, cu.footprint(m["x"]), empty=-1)
    base, bx, bv, bw = rows(scene[0]), scene[1], scene[2], scene[3]
    mask = np.array([1, 0, 1, 0], np.uint8)
    a, x = moved(base, bx, shift_at(k, 30))
    p, xx, vv = pose(a).reshape(k, -1), x.copy(), bv.copy()
    p[mask == 0] = np.nan; xx[mask == 0] = np.nan; vv[mask == 0] = np.nan
    engines = [batch_engine(m, NAME, GRAPH, k, scene) for _ in range(3)]
    still, moved_host, dmask = engines
    want, want_x = base.copy(), bx.copy()
    sel = np.repeat(mask, len(base) // k).astype(bool)
    want[sel] = a[sel]; want_x[mask == 1] = x[mask == 1]
    host_set(moved_host, m, want, want_x, bv, bw)
    dmask.set_replica_collider_poses_device(dev(p), dev(xx), dev(vv), dev(bw), replicas=torch.from_numpy(mask).cuda(), stream=cur())
    for e in engines:
        e.step(60)
    (xs, vs), (xm, vm), (xd, vd) = [final(e) for e in engines]
    assert np.array_equal(xd, xm) and np.array_equal(vd, vm)
    for r in range(k):
        if mask[r] == 0:
            assert np.array_equal(xd[r], xs[r]) and np.array_equal(vd[r], vs[r]), r
    assert any(not np.array_equal(xd[r], xs[r]) for r in range(k) if mask[r])
    assert np.isfinite(xd).all()
    for e in engines:
        e.close()


def test_caller_stream_order_without_host_sync():
    """A caller stream held back by a spin: the engine steps with the rows written on that stream after the spin."""
    import torch
    m = _model(NAME)
    k = 3
    scene = cu.batch_scene(k, cu.footprint(m["x"]), empty=-1)
    base, bx, bv, bw = rows(scene[0]), scene[1], scene[2], scene[3]
    host, devb = batch_engine(m, NAME, GRAPH, k, scene), batch_engine(m, NAME, GRAPH, k, scene)
    a, x = moved(base, bx, shift_at(k, 40))
    host_set(host, m, a, x, bv, bw)
    side = torch.cuda.Stream()
    src, staged = torch.zeros(len(a) * 21, device="cuda"), dev(pose(a))
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        src.copy_(staged)
        devb.set_replica_collider_poses_device(src, dev(x), dev(bv), dev(bw), stream=side.cuda_stream)
        del src
        torch.full((len(a) * 21,), float("nan"), device="cuda")  # the block handed out again on the caller's stream
    host.step(40); devb.step(40)
    xh, vh = final(host); xd, vd = final(devb)
    assert np.array_equal(xh, xd) and np.array_equal(vh, vd)
    side.synchronize()
    host.close(); devb.close()


def test_refusals_keep_the_colliders_in_force():
    import torch
    from positionbaseddynamics_b200 import _capi
    L = _capi.lib()
    m = _model(NAME)
    k = 3
    scene = cu.batch_scene(k, cu.footprint(m["x"]), empty=-1)
    base, bx, bv, bw = rows(scene[0]), scene[1], scene[2], scene[3]
    ref, eng = batch_engine(m, NAME, GRAPH, k, scene), batch_engine(m, NAME, GRAPH, k, scene)
    a, x = moved(base, bx, shift_at(k, 50))
    p, xd = dev(pose(a)), dev(x)
    host_np = pose(a).reshape(-1).copy()
    pinned = torch.zeros(len(a) * 21).pin_memory()
    host_mask = np.ones(k, np.uint8)

    def refused(rc, pattern):
        assert rc != 0
        assert re.search(pattern, L.pbd_last_error().decode()), L.pbd_last_error().decode()
    for ptr, kind in ((host_np.ctypes.data, "pageable"), (pinned.data_ptr(), "pinned")):
        refused(L.pbd_set_replica_collider_poses_device(eng._h, ptr, xd.data_ptr(), None, None, None, None), kind)
        refused(L.pbd_set_replica_collider_poses_device(eng._h, p.data_ptr(), ptr, None, None, None, None), kind)
        refused(L.pbd_set_replica_collider_poses_device(eng._h, p.data_ptr(), xd.data_ptr(), ptr, None, None, None), kind)
    refused(L.pbd_set_replica_collider_poses_device(eng._h, p.data_ptr(), xd.data_ptr(), None, None, host_mask.ctypes.data, None), "replicas is pageable")
    refused(L.pbd_set_replica_collider_poses_device(eng._h, None, xd.data_ptr(), None, None, None, None), "pose == NULL")
    refused(L.pbd_set_replica_collider_poses_device(eng._h, p.data_ptr(), None, None, None, None, None), "body_x == NULL")
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        eng.set_replica_collider_poses_device(host_np, xd)
    with pytest.raises(ValueError, match="elements"):
        eng.set_replica_collider_poses_device(p[:-1], xd)
    g = torch.cuda.CUDAGraph()
    y = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        with pytest.raises(_capi.PbdError, match="captured"):
            eng.set_replica_collider_poses_device(p, xd, stream=torch.cuda.current_stream().cuda_stream)
        y += 1
    g.replay()
    torch.cuda.synchronize()
    for e in (ref, eng):
        e.step(40)
    xr, vr = final(ref); xe, ve = final(eng)
    assert np.array_equal(xr, xe) and np.array_equal(vr, ve)
    # without replica colliders in force, and at K = 1
    eng.set_replica_colliders(_pc(m, NAME), None)
    refused(L.pbd_set_replica_collider_poses_device(eng._h, p.data_ptr(), xd.data_ptr(), None, None, None, None), "no replica colliders in force")
    ref.close(); eng.close()
    one = engine(m, GRAPH)
    refused(L.pbd_set_replica_collider_poses_device(one._h, p.data_ptr(), xd.data_ptr(), None, None, None, None), "single-scene")
    one.close()
