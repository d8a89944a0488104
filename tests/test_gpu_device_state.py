"""Particle state in device memory (pbd_set_attr_device / pbd_get_attr_device / pbd_set_masses_device), with torch CUDA tensors as the
caller's buffers: the device calls move the same bits as the host calls in every slot layout, step alike, write only the masked replicas,
restart replicas as fresh engines, keep the caller's stream order without a host synchronisation, plan and capture nothing again, and
refuse what they cannot take with the state unchanged."""
import re

import numpy as np
import pytest

from batch_util import AUTO, GRAPH, LAUNCH, MODES, RESIDENT, XPBD_TYPES, engine, model, replica_state, run, set_state

pytestmark = pytest.mark.gpu

X, V, X0, OLDX, LASTX = range(5)
ATTRS = (X, V, X0, OLDX, LASTX)
SPIN = 100_000_000  # torch.cuda._sleep cycles: some 50 ms on an H100, long enough for the host to enqueue everything behind it


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda()


def cur():
    import torch
    return torch.cuda.current_stream().cuda_stream  # 0 on torch's default stream: the legacy default stream


def empty(n):
    import torch
    return torch.full((n,), float("nan"), device="cuda")


# (layout, K): before the first step (the formula slots), a graph image, a resident image (tile-major slots), and a single scene forced
# into four independent resident CTAs, whose shared particles live in global memory
LAYOUTS = [(lay, k) for lay in ("formula", "graph", "resident") for k in (1, 3)] + [("resident_4x1", 1)]


def laid_out(m, layout, k, monkeypatch):
    if layout == "resident_4x1":
        monkeypatch.setenv("PBD_B200_CLUSTERS", "4x1")
    mode = RESIDENT if layout.startswith("resident") else GRAPH
    eng = engine(m, mode, replicas=k if k > 1 else None)
    if layout != "formula":
        eng.step(1)
        assert eng.get_mode()[1] == mode
    return eng


@pytest.mark.parametrize("layout,k", LAYOUTS)
def test_round_trip_equals_host_calls(layout, k, monkeypatch):
    """Every attribute: a device set read back by the host get equals a host set; a device get equals the host get.  Masses: a device set
    steps like a host set."""
    m = model("xpbd_cloth64")
    n = len(m["x"])
    host, device = laid_out(m, layout, k, monkeypatch), laid_out(m, layout, k, monkeypatch)
    rng = np.random.default_rng(11)
    for attr in ATTRS:
        vals = rng.normal(size=(k * n, 3)).astype(np.float32)
        host.set_attr(attr, vals)
        device.set_attr_device(attr, dev(vals), stream=cur())
        want = host.get_attr(attr)
        assert np.array_equal(device.get_attr(attr), want), attr
        out = device.get_attr_device(attr, empty(k * n * 3), stream=cur())
        assert np.array_equal(out.cpu().numpy().reshape(want.shape), want), attr
    states = [replica_state(m, r) for r in range(k)]
    xs, vs = np.stack([s[0] for s in states]), np.stack([s[1] for s in states])
    mass = np.stack([s[2] for s in states])
    mass[:, 3::11] = 0.0
    for e in (host, device):
        for attr, a in ((X, xs), (OLDX, xs), (LASTX, xs), (X0, np.repeat(m["x0"][None], k, 0)), (V, vs)):
            e.set_attr(attr, a)
    host.set_masses(mass)
    device.set_masses_device(dev(mass), stream=cur())
    for e in (host, device):
        e.step(2)
    for attr in (X, V):
        assert np.array_equal(host.get_attr(attr), device.get_attr(attr)), attr
    host.close(); device.close()


def device_run(eng, m, states):
    """batch_util.run with every state transfer through the device calls on torch's current stream."""
    import torch
    k, n = len(states), len(m["x"])
    eng.set_attr_device(X, dev(np.stack([s[0] for s in states])), stream=cur())
    eng.set_attr_device(V, dev(np.stack([s[1] for s in states])), stream=cur())
    eng.set_masses_device(dev(np.stack([s[2] for s in states])), stream=cur())
    eng.step(2)
    eng.set_params(dt=m["dt"], sub_steps=m["sub"] + 1, max_iter=m["it"] + 1, vel_method=1)
    eng.step(2)
    v = eng.get_attr_device(V, empty(k * n * 3), stream=cur())
    eng.set_attr_device(V, v * 0.5, stream=cur())
    eng.step(1)
    x, v = (eng.get_attr_device(a, empty(k * n * 3), stream=cur()) for a in (X, V))
    torch.cuda.synchronize()
    lam = {}
    for t in XPBD_TYPES:
        if (m["types"] == t).any():
            l, ids = eng.lambdas(t)
            lam[t] = l[..., np.argsort(ids)].copy()
    return x.cpu().numpy().reshape(k, n, 3), v.cpu().numpy().reshape(k, n, 3), lam


@MODES
@pytest.mark.parametrize("name", ["xpbd_cloth64", "fem_volume_bar"])
def test_device_fed_batch_steps_like_host_fed(name, mode):
    """A batch fed and read through the device calls advances bit for bit like one fed and read through the host calls (x, v, multipliers)."""
    m = model(name)
    k = 3
    states = [replica_state(m, r) for r in range(k)]
    host = engine(m, mode, replicas=k)
    set_state(host, states)
    xh, vh, lh = run(host, m)
    host.close()
    device = engine(m, mode, replicas=k)
    xd, vd, ld = device_run(device, m, states)
    device.close()
    assert np.array_equal(xd, xh) and np.array_equal(vd, vh)
    assert lh.keys() == ld.keys() and all(np.array_equal(lh[t], ld[t]) for t in lh)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT], ids=["graph", "resident"])
def test_masked_writes_touch_only_the_masked_replicas(mode):
    """The unmasked replicas' rows of the source are NaN: they must be neither written nor read.  The result steps like a host engine given
    the merged state."""
    import torch
    m = model("xpbd_cloth64")
    k, n = 4, len(m["x"])
    mask = np.array([False, True, False, True])
    states = [replica_state(m, r) for r in range(k)]
    eng, host = engine(m, mode, replicas=k), engine(m, mode, replicas=k)
    for e in (eng, host):
        set_state(e, states)
        e.step(2)
    rng = np.random.default_rng(3)
    for i, attr in enumerate(ATTRS):
        before = eng.get_attr(attr)
        new = before + rng.normal(0.0, 1e-3, before.shape).astype(np.float32)
        merged = np.where(mask[:, None, None], new, before)
        new[~mask] = np.nan
        replicas = torch.from_numpy(mask).cuda() if i % 2 else torch.from_numpy(mask.astype(np.uint8)).cuda()  # |b1 and |u1
        eng.set_attr_device(attr, dev(new), replicas=replicas, stream=cur())
        host.set_attr(attr, merged)
        got = eng.get_attr(attr)
        assert np.array_equal(got, merged), attr
    mass = np.stack([replica_state(m, r + 1)[2] for r in range(k)])  # replica r gets replica r + 1's pins
    merged = np.where(mask[:, None], mass, np.stack([s[2] for s in states]))
    mass[~mask] = np.nan
    eng.set_masses_device(dev(mass), replicas=torch.from_numpy(mask).cuda(), stream=cur())
    host.set_masses(merged)
    for e in (eng, host):
        e.step(2)
    for attr in ATTRS:
        got = eng.get_attr(attr)
        assert np.isfinite(got).all() and np.array_equal(got, host.get_attr(attr)), attr
    eng.close(); host.close()


def test_mask_of_one_replica():
    """At K = 1 the mask has one byte: zero leaves the scene as it was, nonzero writes it."""
    import torch
    m = model("xpbd_cloth64")
    eng = engine(m, GRAPH)
    eng.step(1)
    before = eng.get_attr(X)
    new = before + np.float32(0.25)
    eng.set_attr_device(X, dev(new), replicas=torch.zeros(1, dtype=torch.bool, device="cuda"), stream=cur())
    assert np.array_equal(eng.get_attr(X), before)
    eng.set_attr_device(X, dev(new), replicas=torch.ones(1, dtype=torch.uint8, device="cuda"), stream=cur())
    assert np.array_equal(eng.get_attr(X), new)
    eng.close()


def solo_from(m, x, v, mass, params):
    """A single-scene engine started from (x, v, mass) by set_particles, so that oldX = lastX = x."""
    from positionbaseddynamics_b200 import _capi
    eng = _capi.Engine(0)
    eng.set_particles(x, mass, x0=m["x0"], v=v)
    eng.add_flat(m["types"], m["bodies"], m["params"])
    eng.set_groups(m["off"], m["ids"])
    eng.set_params(**params)
    eng.set_mode(GRAPH)
    return eng


@MODES
def test_restart_replicas_mid_run(mode):
    """Replicas 1 and 3 restarted after 3 steps through masked device writes of X, V, OLDX = X, LASTX = X and the masses, with the
    second-order velocity update (which reads lastX): each then matches a fresh single-scene engine, and replicas 0 and 2 an uninterrupted
    run, bit for bit, multipliers included."""
    import torch
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k, n = 4, len(m["x"])
    params = dict(dt=m["dt"], sub_steps=m["sub"], max_iter=m["it"], vel_method=1)
    states = [replica_state(m, r) for r in range(k)]
    runs = []
    for restart in (False, True):
        eng = engine(m, mode, replicas=k)
        eng.set_params(**params)
        set_state(eng, states)
        eng.step(3)
        if restart:
            mask = np.array([False, True, False, True])
            fresh = [replica_state(m, 20 + r) for r in range(k)]
            x = np.stack([f[0] for f in fresh]); x[~mask] = np.nan
            v = np.stack([f[1] for f in fresh]); v[~mask] = np.nan
            mass = np.stack([f[2] for f in fresh]); mass[~mask] = np.nan
            replicas = torch.from_numpy(mask).cuda()
            xd = dev(x)
            for attr, src in ((X, xd), (V, dev(v)), (OLDX, xd), (LASTX, xd)):
                eng.set_attr_device(attr, src, replicas=replicas, stream=cur())
            eng.set_masses_device(dev(mass), replicas=replicas, stream=cur())
        eng.step(2)
        eng.sync()
        lam, ids = eng.lambdas(_capi.DISTANCE_XPBD)
        runs.append((eng.get_attr(X), eng.get_attr(V), lam[:, np.argsort(ids)]))
        eng.close()
    (xu, vu, lu), (xr, vr, lr) = runs
    for r in (0, 2):
        assert np.array_equal(xr[r], xu[r]) and np.array_equal(vr[r], vu[r]) and np.array_equal(lr[r], lu[r]), r
    for r in (1, 3):
        x, v, mass = replica_state(m, 20 + r)
        solo = solo_from(m, x, v, mass, params)
        solo.step(2)
        solo.sync()
        lam, ids = solo.lambdas(_capi.DISTANCE_XPBD)
        assert np.array_equal(xr[r], solo.get_attr(X)) and np.array_equal(vr[r], solo.get_attr(V)), r
        assert np.array_equal(lr[r], lam[np.argsort(ids)]), r
        solo.close()


def test_caller_stream_order_without_host_sync():
    """A caller stream held back by a spin: the engine reads the buffer written on it after the spin; a get is read by torch on that stream
    after the copy; the source can be freed and its block handed out again on that stream right after the call; and the engine's steps in
    between stay in order."""
    import torch
    m = model("xpbd_cloth64")
    k, n = 3, len(m["x"])
    states = [replica_state(m, r) for r in range(k)]
    eng = engine(m, GRAPH, replicas=k)
    set_state(eng, states)
    eng.step(1); eng.sync()
    side = torch.cuda.Stream()
    rng = np.random.default_rng(5)
    # the write after the spin is what the engine reads
    want = (eng.get_attr(X) + rng.normal(0.0, 1e-3, (k, n, 3))).astype(np.float32)
    src, staged = torch.zeros(k * n * 3, device="cuda"), dev(want)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        src.copy_(staged)
        eng.set_attr_device(X, src, stream=side.cuda_stream)
    assert np.array_equal(eng.get_attr(X), want)
    # a get read on the caller's stream right behind it
    out = torch.zeros(k * n * 3, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        out.fill_(float("nan"))
        eng.get_attr_device(X, out, stream=side.cuda_stream)
        copy = out.clone()
    side.synchronize()
    assert np.array_equal(copy.cpu().numpy().reshape(k, n, 3), want)
    # the source freed and its block reused on the caller's stream while the engine stream is still busy with steps
    vals = rng.normal(0.0, 0.1, (k, n, 3)).astype(np.float32)
    with torch.cuda.stream(side):
        src = torch.from_numpy(vals.reshape(-1)).to("cuda")
        ptr = src.data_ptr()
        eng.step(50)
        eng.set_attr_device(V, src, stream=side.cuda_stream)
        del src
        junk = torch.full((k * n * 3,), float("nan"), device="cuda")
        assert junk.data_ptr() == ptr  # the caching allocator handed the block out again
    assert np.array_equal(eng.get_attr(V), vals)
    side.synchronize()
    eng.close()


def test_interleaved_with_step_host_async():
    """Device calls between pbd_step_host_async calls compute what host calls between synchronised ones compute."""
    import torch
    m = model("xpbd_cloth64")
    k, n = 3, len(m["x"])
    states = [replica_state(m, r) for r in range(k)]
    xin = np.ascontiguousarray(np.stack([s[0] for s in states])); vin = np.ascontiguousarray(np.stack([s[1] for s in states]))
    outs = []
    for how in ("host", "device"):
        eng = engine(m, GRAPH, replicas=k)
        eng.set_masses(np.stack([s[2] for s in states]))
        x1, v1, x2, x3 = (np.empty_like(xin) for _ in range(4))
        eng.step_host_async(1, xin, vin, x1, v1)
        if how == "host":
            eng.step_host_wait(0)
            eng.set_attr(V, eng.get_attr(V) * np.float32(0.5))
        else:
            v = eng.get_attr_device(V, empty(k * n * 3), stream=cur())
            eng.set_attr_device(V, v * 0.5, stream=cur())
        eng.step_host_async(2, None, None, x2, None)
        got = eng.get_attr_device(X, empty(k * n * 3), stream=cur()) if how == "device" else None
        eng.step_host_async(1, None, None, x3, None)
        eng.step_host_wait(0)
        if how == "host":
            got = x2
        else:
            torch.cuda.synchronize()
            got = got.cpu().numpy().reshape(k, n, 3)
        outs.append((x1, v1, x2, x3, got))
        eng.close()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_no_replan_and_no_recapture():
    """Device calls between steps keep the image (the multipliers of the last step survive them) and the captured graph (the graph engine
    stays bit-identical to a launch engine and launches as many kernels)."""
    from positionbaseddynamics_b200 import _capi
    m = model("xpbd_cloth64")
    k, n = 2, len(m["x"])
    states = [replica_state(m, r) for r in range(k)]
    engines = [engine(m, mode, replicas=k) for mode in (GRAPH, LAUNCH, RESIDENT)]
    rng = np.random.default_rng(9)
    for e in engines:
        set_state(e, states)
        e.step(2)
    for rnd in range(3):
        vals = (engines[0].get_attr(V) * np.float32(0.5)).astype(np.float32)
        mass = np.stack([s[2] for s in states]); mass[:, rng.integers(0, n, 10)] = 0.0
        for e in engines:
            before = e.lambdas(_capi.DISTANCE_XPBD)[0].copy()
            assert before.any()
            e.set_attr_device(V, dev(vals), stream=cur())
            e.set_masses_device(dev(mass), stream=cur())
            e.get_attr_device(X, empty(k * n * 3), stream=cur())
            assert np.array_equal(e.lambdas(_capi.DISTANCE_XPBD)[0], before), (rnd, e.get_mode())
        for e in engines:
            e.step(2)
        xs = [e.get_attr(X) for e in engines]
        assert all(np.array_equal(x, xs[0]) for x in xs), rnd
    assert engines[0].stats().kernel_launches == engines[1].stats().kernel_launches
    for e in engines:
        e.close()


@pytest.mark.parametrize("switch", [(GRAPH, RESIDENT), (RESIDENT, GRAPH), (AUTO, LAUNCH)], ids=["graph-resident", "resident-graph", "auto-launch"])
def test_replan_waits_for_a_pending_get(switch):
    """A get enqueued behind a spinning caller stream, then a mode change that plans the image again in another slot layout, then a step:
    the get still delivers the state from before the change, in host order."""
    import torch
    m = model("xpbd_cloth64")
    k, n = 3, len(m["x"])
    states = [replica_state(m, r) for r in range(k)]
    eng = engine(m, switch[0], replicas=k)
    set_state(eng, states)
    eng.step(2)
    want = eng.get_attr(X)
    side = torch.cuda.Stream()
    out = empty(k * n * 3)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        eng.get_attr_device(X, out, stream=side.cuda_stream)
    eng.set_mode(switch[1])
    eng.step(1)
    side.synchronize()
    assert np.array_equal(out.cpu().numpy().reshape(k, n, 3), want)
    eng.close()


def test_refusals_leave_the_state_unchanged():
    import torch
    from positionbaseddynamics_b200 import _capi
    L = _capi.lib()
    m = model("xpbd_cloth64")
    k, n = 3, len(m["x"])
    eng = engine(m, GRAPH, replicas=k)
    set_state(eng, [replica_state(m, r) for r in range(k)])
    eng.step(1)
    snapshot = {a: eng.get_attr(a) for a in ATTRS}
    good = dev(snapshot[X] + np.float32(1.0))
    good_mass = torch.ones(k * n, device="cuda")
    mask = torch.ones(k, dtype=torch.bool, device="cuda")
    host_np = np.zeros(k * n * 3, np.float32)
    pinned = torch.zeros(k * n * 3).pin_memory()
    host_mask = np.ones(k, np.bool_)

    def refused(rc, pattern):
        assert rc != 0
        assert re.search(pattern, L.pbd_last_error().decode()), L.pbd_last_error().decode()

    # the Python layer: no device array, wrong element type, size, layout, a read-only output
    for a in (host_np, pinned):
        with pytest.raises(TypeError, match="__cuda_array_interface__"):
            eng.set_attr_device(X, a)
        with pytest.raises(TypeError, match="__cuda_array_interface__"):
            eng.get_attr_device(X, a)
    with pytest.raises(TypeError, match="__cuda_array_interface__"):
        eng.set_attr_device(X, good, replicas=host_mask)
    with pytest.raises(ValueError, match="element type"):
        eng.set_attr_device(X, good.double())
    with pytest.raises(ValueError, match="element type"):
        eng.set_attr_device(X, good, replicas=mask.int())
    with pytest.raises(ValueError, match="elements"):
        eng.set_attr_device(X, good[:-3])
    with pytest.raises(ValueError, match="elements"):
        eng.set_masses_device(good_mass, replicas=mask[:2])
    with pytest.raises(ValueError, match="C-contiguous"):
        eng.set_attr_device(X, torch.zeros(2 * k * n * 3, device="cuda")[::2])

    class ReadOnly:
        __cuda_array_interface__ = dict(good.__cuda_array_interface__, data=(good.data_ptr(), True))
    with pytest.raises(ValueError, match="read-only"):
        eng.get_attr_device(X, ReadOnly())

    # the C calls: host memory (pageable, pinned), a host mask, attributes out of range, null pointers
    for p, kind in ((host_np.ctypes.data, "pageable"), (pinned.data_ptr(), "pinned")):
        refused(L.pbd_set_attr_device(eng._h, X, p, None, None), kind)
        refused(L.pbd_get_attr_device(eng._h, X, p, None), kind)
        refused(L.pbd_set_masses_device(eng._h, p, None, None), kind)
    refused(L.pbd_set_attr_device(eng._h, X, good.data_ptr(), host_mask.ctypes.data, None), "replicas is pageable host memory")
    refused(L.pbd_set_masses_device(eng._h, good_mass.data_ptr(), pinned.data_ptr(), None), "replicas is pinned host memory")
    for attr in (-1, 5):
        refused(L.pbd_set_attr_device(eng._h, attr, good.data_ptr(), None, None), "bad attribute")
        refused(L.pbd_get_attr_device(eng._h, attr, good.data_ptr(), None), "bad attribute")
    refused(L.pbd_set_attr_device(eng._h, X, None, None, None), "src == NULL")
    refused(L.pbd_get_attr_device(eng._h, X, None, None), "dst == NULL")
    refused(L.pbd_set_masses_device(eng._h, None, None, None), "mass == NULL")

    # a stream being captured into a graph
    g = torch.cuda.CUDAGraph()
    y = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        s = torch.cuda.current_stream().cuda_stream
        with pytest.raises(_capi.PbdError, match="captured"):
            eng.set_attr_device(X, good, stream=s)
        with pytest.raises(_capi.PbdError, match="captured"):
            eng.get_attr_device(X, good, stream=s)
        with pytest.raises(_capi.PbdError, match="captured"):
            eng.set_masses_device(good_mass, replicas=mask, stream=s)
        y += 1
    g.replay()
    torch.cuda.synchronize()
    assert y.item() == 1.0

    for a in ATTRS:
        assert np.array_equal(eng.get_attr(a), snapshot[a]), a
    assert np.array_equal(good.cpu().numpy().reshape(k, n, 3), snapshot[X] + np.float32(1.0))  # the refused get wrote nothing either
    eng.step(1)
    assert np.isfinite(eng.get_attr(X)).all()
    eng.close()
