"""Replica batches on one GPU (pbd_set_replicas): ms per batched step and aggregate projections/s for batches of cfg1-, cfg3-,
100x100-XPBD-cloth and 100x100-FEMTriangle-cloth replicas over a sweep of K, in graph and resident mode, against the same K replicas
stepped one after another by a K = 1 engine; the resident cluster size C swept on the cfg1- and cfg3-class batches; the card name and
power limit read in the same run.  The four scenes run four different resident instantiations (cloth, FEM, cloth-XPBD and light type
masks).

    python tools/bench_batch.py [--out results.json] [--quick] [--replica-rows] [--sweep] [--rest-shapes] [--colliders] [--constraint-materials]
                                [--rigid] [--contact-sensors] [--forces] [--ks 8,132] [--no-baseline]

--replica-rows measures every batch twice in a row: with the shared parameters, and with per-replica material rows and gravity
(pbd_set_replica_materials / pbd_set_replica_gravity) equal to the shared values, so that the work is identical and the difference is what
the tables cost.  --sweep adds one real sweep: 132 cfg1 replicas, each with its own Distance and IsometricBending stiffness.
--rest-shapes measures every batch twice in a row with the shared geometry and with per-replica rest shapes
(pbd_set_replica_rest_positions) equal to the model's own rest positions, so that the work is identical and the difference is what the
per-replica geometry arrays cost (they are K times the shared ones and leave L2 for large batches).  It also times the device derivation of
the geometry of K rest shapes against building K host models (the host mirror's add*Constraint) for cfg1 K = 1056 and cfg3 K = 66.
--colliders measures only the contact path of batches: cfg1 at K = 8, 132, 1056 and the 100x100 XPBD cloth at K = 33, 264, each in graph
and resident mode, without and with three per-replica colliders (pbd_set_replica_colliders: a sphere, a rotated box and a torus cutting
through the cloth's plane at random places, every replica its own), alternating.  The difference is the cost of the contact launch.
--constraint-materials measures every batch four times in a row: with the shared parameters, with per-constraint materials of every replica
(pbd_set_replica_constraint_materials) equal to the shared values, and both again, so that the work is identical and the difference is
what reading the K x count material arrays costs; their size is printed beside each row.  It also times the device form of the call
(pbd_set_replica_constraint_materials_device) for every replica and for a 10 % mask, 200 calls enqueued behind a spin so that the
gathers run back to back, against the algorithmic bytes of the gather.
--rigid measures only batches of the rigid-body cloth coupling rig (a 20 x 20 cloth, 12 bodies, 8 BallJoints, 4 RigidBodyParticleBallJoints,
tests/rigid_batch_util.py), every replica with its own bodies (pbd_set_replica_rigid_bodies): ms per batched step at K = 1, 33, 132, 528 in
graph and in forced resident mode, against the K replicas stepped one after another by a K = 1 engine (per replica its particles and bodies
uploaded, one step, both read back), and the cost of one masked device write of the bodies per step (pbd_set_rigid_bodies_device, half the
replicas): the write alone, 200 enqueued back to back, and steps with a write before each against steps without, wall clock after a sync.
--contact-sensors measures the contact path's device interface on the --colliders workloads, in graph and resident mode: steps with the
three per-replica colliders and the contact sensors off, on, off, on (pbd_sense_contacts; device time), and 200 steps each preceded by a move
of every replica's colliders (wall clock after a sync), the rows drawn by a torch op on the GPU: no move, the host call
pbd_set_replica_colliders after copying the rows to the host, and the device call pbd_set_replica_collider_poses_device.
--forces measures external forces (pbd_set_external_forces) on the cfg2 single scene, cfg1 at K = 132 and 1056 and the 100x100 XPBD cloth
at K = 264, in graph and resident mode: steps with forces off, on, off, on, the forces all zero so that the work is identical but the force
read (device time), and, on the batches, 200 steps each preceded by a write of every particle's force drawn by a torch op on the GPU (wall
clock after a sync): no write, the host call after copying the forces to the host, and the device call pbd_set_external_forces_device.
--ks replaces the K sweep of every scene; --no-baseline skips the one-after-another baseline and the C sweep.  Without --rest-shapes or
--replica-rows the script also runs against a build without those calls, so that shared-parameter batches can be compared across builds.

Batch times are device times (CUDA events on the engine's stream around `steps` steps, after warm-up steps).  The baseline is measured:
a K = 1 engine in its faster mode (graph or resident) steps K replicas one after another -- K pbd_step calls, each replica's state
uploaded before its step and read back after it (pbd_set_attr / pbd_get_attr of x and v), wall clock around the whole sequence.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import scenes  # noqa: E402
from positionbaseddynamics_b200 import _capi  # noqa: E402
from positionbaseddynamics_b200.model import HostModel  # noqa: E402

SCENES = {  # name: (builder, sub_steps, max_iter, K sweep)
    "cfg1": (lambda m: scenes.cfg1(m), 1, 5, [1, 8, 33, 132, 264, 528, 1056]),
    "cfg3": (lambda m: scenes.cfg3(m), 10, 5, [1, 4, 8, 16, 33, 66]),
    "cloth100_xpbd": (lambda m: scenes.cloth(m, 100, 100, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=1, max_iter=20),
                      1, 20, [1, 8, 33, 66, 132, 264]),
    "cloth100_femtri": (lambda m: scenes.cloth(m, 100, 100, cloth_method=2, bending_method=1, sub_steps=1, max_iter=5), 1, 5, [1, 8, 33, 66, 132, 264]),
}
C_SWEEP = {"cfg1": [8, 132, 528], "cfg3": [8, 33, 66]}  # K at which every cluster size C is measured
RIGID_KS = [1, 33, 132, 528]


def rigid_engine(m, mode, k):
    import rigid_batch_util as rb
    if k == 1:
        return rb.engine(m, mode, bodies=rb.replica_bodies(m, 0))
    return rb.engine(m, mode, replicas=k, bodies=[rb.replica_bodies(m, r) for r in range(k)])


def rigid_one_after_another(m, k):
    """ms for K rig replicas stepped one after another by one K = 1 engine in graph mode: per replica its x, v and bodies uploaded, one
    step, x, v and bodies read back; wall clock around the sequence, after one warm-up pass."""
    import rigid_batch_util as rb
    eng = rigid_engine(m, _capi.MODE_GRAPH, 1)
    try:
        xs = np.repeat(np.asarray(m["x"], np.float32)[None], k, 0)
        vs = np.zeros_like(xs)
        mass, _, _, inertia, _, _ = rb.replica_bodies(m, 0)
        bodies = np.repeat(eng.get_rigid_bodies()[None], k, 0)
        for passes in range(2):  # the first pass warms up
            eng.sync()
            t0 = time.perf_counter()
            for r in range(k):
                eng.set_attr(_capi.ATTR_X, xs[r]); eng.set_attr(_capi.ATTR_V, vs[r])
                b = bodies[r]
                eng.set_rigid_bodies(mass, b[:, :3], b[:, 3:7], inertia, v=b[:, 7:10], omega=b[:, 10:13])
                eng.step(1)
                eng.get_attr(_capi.ATTR_X, xs[r]); eng.get_attr(_capi.ATTR_V, vs[r]); bodies[r] = eng.get_rigid_bodies()
            eng.sync()
            ms = (time.perf_counter() - t0) * 1e3
        return ms
    finally:
        eng.close()


def rigid_write_timing(m, k, calls=200):
    """A masked device write of every body of half the replicas (pbd_set_rigid_bodies_device, x and q from torch): ms per write alone
    (`calls` enqueued back to back), and ms per step with and without a write before each step (graph mode), wall clock after a sync."""
    import torch
    eng = rigid_engine(m, _capi.MODE_GRAPH, k)
    try:
        st = eng.get_rigid_bodies()
        x = torch.from_numpy(np.ascontiguousarray(st[..., :3]).reshape(-1)).cuda()
        q = torch.from_numpy(np.ascontiguousarray(st[..., 3:7]).reshape(-1)).cuda()
        mask = (torch.arange(k, device="cuda") % 2 == 0).to(torch.uint8)
        s = torch.cuda.current_stream().cuda_stream

        def wall(f, n):
            f(); torch.cuda.synchronize(); eng.sync()
            t0 = time.perf_counter()
            for _ in range(n):
                f()
            torch.cuda.synchronize(); eng.sync()
            return (time.perf_counter() - t0) * 1e3 / n
        write = lambda: eng.set_rigid_bodies_device(x, q, replicas=mask, stream=s)
        alone = wall(write, calls)
        steps = [wall(lambda: eng.step(1), 100), wall(lambda: (write(), eng.step(1)), 100), wall(lambda: eng.step(1), 100), wall(lambda: (write(), eng.step(1)), 100)]
        return {"K": k, "write_ms": alone, "step_ms": steps[0::2], "step_with_write_ms": steps[1::2]}
    finally:
        eng.close()


def rigid_main(a, res):
    import rigid_batch_util as rb
    m = rb.model("rig")
    print("rig: %d particles, %d bodies, %d constraints, %d x %d" % (len(m["x"]), len(m["bm"]), len(m["types"]), m["sub"], m["it"]), flush=True)
    for k in ([int(v) for v in a.ks.split(",")] if a.ks else RIGID_KS):
        row = {"K": k, "baseline_ms": float("nan") if a.no_baseline else rigid_one_after_another(m, k)}
        for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
            eng = None
            try:
                eng = rigid_engine(m, md, k)
                ms, steps = timed(eng)
                row[label] = {"ms": ms, "steps": steps, "active": eng.get_mode()[1]}
            except _capi.PbdError as ex:
                row[label] = {"error": str(ex)}
            finally:
                if eng is not None:
                    eng.close()
        if k > 1:
            row["write"] = rigid_write_timing(m, k)
        res["rigid"].append(row)
        fmt = lambda r: ("%8.4f ms" % r["ms"]) if "ms" in r else ("refused: " + r["error"][:60])
        w = row.get("write")
        print("  rig K=%4d  graph %s | resident %s | one after another %9.3f ms%s" % (
            k, fmt(row["graph"]), fmt(row["resident"]), row["baseline_ms"],
            (" | masked body write %.4f ms alone, step %.4f %.4f ms, with a write %.4f %.4f ms" % (w["write_ms"], *w["step_ms"], *w["step_with_write_ms"])) if w else ""),
            flush=True)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as ex:  # the numbers are worth less without it: say so in the output
        return "unknown (%s)" % ex


def model(name, table=SCENES):
    build, sub, it, _ = table[name]
    hm = HostModel()
    build(hm)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    m = dict(types=types, bodies=bodies, params=np.array(params, np.float32), off=off, ids=ids, x0=hm.get("x0"), mass=mass, sub=sub, it=it)
    hm.close()
    return m


def topology(name):
    """The model's triangles or tets, for building a host model on other rest positions."""
    build, sub, it, _ = SCENES[name]
    hm = HostModel()
    build(hm)
    topo = hm.tri_faces(0) if name.startswith("cfg1") or name.startswith("cloth") else hm.tet_tets(0)
    hm.close()
    return topo


def host_build(name, x0, mass, topo):
    """One host model of scene `name` built on rest positions x0 (what a replica's geometry costs without the device derivation)."""
    hm = HostModel()
    if name == "cfg3":
        hm.add_tet_model(x0, topo)
        for i in np.nonzero(mass == 0)[0]:
            hm.set_mass(int(i), 0.0)
        hm.add_solid_constraints(0, 2, k=1.0e6, nu=0.3, vol_k=1.0)
        for t in topo:
            hm.add_constraint(scenes.VOLUME, [int(v) for v in t], [1.0])
    else:
        hm.add_triangle_model(x0, topo)
        for i in np.nonzero(mass == 0)[0]:
            hm.set_mass(int(i), 0.0)
        hm.add_cloth_constraints(0, 1, dist_k=1.0)
        hm.add_bending_constraints(0, 2, 0.01)
    n = hm.num_constraints()
    hm.close()
    return n


def derive_timing(name, m, k):
    """Seconds to give K replicas their own rest shapes on the device (pbd_set_replica_rest_positions: upload, derivation, check, copy)
    against building K host models on those rest positions (three built and timed, scaled to K)."""
    rng = np.random.default_rng(7)
    x0 = np.asarray(m["x0"], np.float32)
    rest = (x0[None] * rng.uniform(0.9, 1.1, (k, 1, 3))).astype(np.float32)
    eng = engine(m, _capi.MODE_GRAPH, k)
    try:
        eng.step(1); eng.sync()
        t = []
        for _ in range(3):
            t0 = time.perf_counter()
            eng.set_replica_rest_positions(rest)
            t.append(time.perf_counter() - t0)
            eng.set_replica_rest_positions(None)
    finally:
        eng.close()
    topo = topology(name)
    h = []
    for r in range(3):
        t0 = time.perf_counter()
        host_build(name, rest[r], np.asarray(m["mass"]), topo)
        h.append(time.perf_counter() - t0)
    return {"scene": name, "K": k, "device_s": min(t), "host_one_s": min(h), "host_K_s": min(h) * k}


def shared_rows(m, k):
    """Per-replica rows that restate the shared parameters: {type: (k, nMat)} from each type's first constraint, and (k, 3) gravity."""
    rows = {}
    for t in range(_capi.NUM_TYPES):
        sel = np.nonzero(np.asarray(m["types"]) == t)[0]
        if len(sel) and _capi.num_materials(t):
            cols = MAT_FIRST_COLUMN[t] + np.arange(_capi.num_materials(t))
            rows[t] = np.repeat(np.asarray(m["params"], np.float32)[sel[0], cols][None], k, 0)
    return rows, np.repeat(np.asarray([[0.0, -9.81, 0.0]], np.float32), k, 0)


# bytes of packed geometry per constraint (the image's float4 and scalar geometry arrays; IsometricBending: the rank-one Kp)
GEO_BYTES = {0: 4, 1: 4, 2: 4, 3: 16, 4: 16, 5: 20, 6: 16, 7: 4, 8: 4, 9: 40, 10: 40, 11: 36, 12: 96}
DERIVE_K = {"cfg1": 1056, "cfg3": 66}
# include/pbd_b200.h: where a type's material parameters start in its parameter layout
MAT_FIRST_COLUMN = {0: 1, 1: 1, 2: 1, 3: 0, 4: 0, 5: 5, 6: 4, 7: 1, 8: 1, 9: 10, 10: 10, 11: 9, 12: 0}


COLLIDER_KS = {"cfg1": [8, 132, 1056], "cloth100_xpbd": [33, 264]}


def replica_colliders(m, k):
    """Three static colliders per replica across the cloth's plane, each replica's at its own random places: (rigid lists, body_x)."""
    x0 = np.asarray(m["x0"], np.float64)
    lo, hi = x0.min(axis=0), x0.max(axis=0)
    c, h = (lo + hi) / 2.0, (hi - lo) / 2.0
    size = float(min(h[0], h[2]))
    rng = np.random.default_rng(3)
    rigid, body_x = [], np.zeros((k, 3, 3), np.float32)
    for r in range(k):
        cols = []
        for j, shape in enumerate((_capi.SHAPE_SPHERE, _capi.SHAPE_BOX, _capi.SHAPE_TORUS)):
            centre = c + np.array([rng.uniform(-0.6, 0.6) * h[0], -0.1 * size, rng.uniform(-0.6, 0.6) * h[2]])
            a = rng.normal(size=3); a /= np.linalg.norm(a); t = rng.uniform(0.0, 1.0)
            kx = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
            rot = np.eye(3) + np.sin(t) * kx + (1.0 - np.cos(t)) * (kx @ kx)
            s = 0.2 * size
            dim = {_capi.SHAPE_SPHERE: (s, 0.0, 0.0), _capi.SHAPE_BOX: (s, 0.5 * s, s), _capi.SHAPE_TORUS: (s, 0.4 * s, 0.0)}[shape]
            half = {_capi.SHAPE_SPHERE: np.full(3, s), _capi.SHAPE_BOX: np.array(dim), _capi.SHAPE_TORUS: np.array([1.4 * s, 0.4 * s, 1.4 * s])}[shape]
            half = np.abs(rot) @ half + 0.05
            rc = _capi.RigidCollider(); rc.shape = shape; rc.body = j; rc.dim[:] = list(dim); rc.restitution = 0.6; rc.friction = 0.2
            rc.R[:] = rot.T.reshape(-1).tolist(); rc.v2[:] = centre.tolist(); rc.aabb_min[:] = (centre - half).tolist(); rc.aabb_max[:] = (centre + half).tolist()
            cols.append(rc); body_x[r, j] = centre
        rigid.append(cols)
    return rigid, body_x


def constraint_materials(m, k):
    """{type: (k, count, nMat)}: every material-bearing type's per-constraint values, the shared ones in every replica."""
    out = {}
    for t in range(_capi.NUM_TYPES):
        sel = np.nonzero(np.asarray(m["types"]) == t)[0]
        if len(sel) and _capi.num_materials(t):
            cols = MAT_FIRST_COLUMN[t] + np.arange(_capi.num_materials(t))
            out[t] = np.ascontiguousarray(np.repeat(np.asarray(m["params"], np.float32)[sel][:, cols][None], k, 0))
    return out


def gather_timing(m, k, calls=200):
    """µs per pbd_set_replica_constraint_materials_device call's gather, for every replica and for every tenth, against the algorithmic
    bytes: per written (replica, constraint) nMat floats read, written to the device-ordered arrays and to the engine's copy, and one
    4-byte map entry read."""
    import torch
    mats = constraint_materials(m, k)
    eng = engine(m, _capi.MODE_GRAPH, k, cmat=mats)
    out = []
    try:
        eng.step(1); eng.sync()
        src = {t: torch.from_numpy(f.reshape(-1)).cuda() for t, f in mats.items()}
        for label, mask in (("all", None), ("10 %", np.arange(k) % 10 == 0)):
            dm = None if mask is None else torch.from_numpy(mask).cuda()
            written = k if mask is None else int(mask.sum())
            for t, f in mats.items():
                nbytes = written * f.shape[1] * (3 * 4 * f.shape[2] + 4)
                torch.cuda.synchronize()
                s = torch.cuda.current_stream()
                torch.cuda._sleep(50_000_000)  # the calls below are enqueued while this spins, then run back to back
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(s)
                for _ in range(calls):
                    eng.set_replica_constraint_materials_device(t, src[t], replicas=dm, stream=s.cuda_stream)
                e1.record(s)
                e1.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / calls
                out.append({"K": k, "type": t, "mask": label, "us": us, "bytes": nbytes, "tb_s": nbytes / (us * 1e-6) / 1e12})
    finally:
        eng.close()
    return out


def engine(m, mode, k, clusters=None, rows=None, rest=False, colliders=False, cmat=None, sense=False, forces=False):
    if clusters:
        os.environ["PBD_B200_CLUSTERS"] = "1x%d" % clusters  # the planner's cluster-size override (read when the image is planned)
    else:
        os.environ.pop("PBD_B200_CLUSTERS", None)
    eng = _capi.Engine(0)
    eng.set_particles(m["x0"], m["mass"])
    eng.add_flat(m["types"], m["bodies"], m["params"])
    eng.set_groups(m["off"], m["ids"])
    eng.set_params(dt=0.005, sub_steps=m["sub"], max_iter=m["it"])
    eng.set_mode(mode)
    if k > 1:
        eng.set_replicas(k)
    if rows is not None:
        for t, mat in rows[0].items():
            eng.set_replica_materials(t, mat)
        eng.set_replica_gravity(rows[1])
    if rest:  # every replica's rest shape = the model's: the same geometry, from the per-replica arrays
        eng.set_replica_rest_positions(np.repeat(np.asarray(m["x0"], np.float32)[None], k, 0))
    if cmat is not None:
        for t, f in cmat.items():
            eng.set_replica_constraint_materials(t, f)
    if colliders:
        rigid, body_x = replica_colliders(m, k)
        eng.set_replica_colliders([_capi.ParticleCollider(0, len(m["x0"]), 0.5, 0.1)], rigid, body_x)
        eng.set_contact_params(0.05, 100.0, 5)
        eng.sense_contacts(sense)
    if forces:  # zero forces: the same answer as none, through the integration's force form
        eng.set_external_forces(np.zeros(((k,) if k > 1 else ()) + (len(m["x0"]), 3), np.float32))
    return eng


def timed(eng, warmup=3, min_s=0.4):
    """ms per step: warm-up steps, a probe to size the window, then a window of at least min_s seconds of device time."""
    eng.step(warmup); eng.sync()
    eng.step(2); eng.sync()
    probe = max(eng.stats().last_step_ms / 2, 1e-3)
    steps = int(min(2000, max(10, min_s * 1e3 / probe)))
    eng.step(steps); eng.sync()
    st = eng.stats()
    return st.last_step_ms / steps, steps


def measure(m, mode, k, clusters=None, rows=None, rest=False, colliders=False, cmat=None, sense=False, forces=False):
    t0 = time.time()
    eng = None
    try:
        eng = engine(m, mode, k, clusters, rows, rest, colliders, cmat, sense, forces)
        ms, steps = timed(eng)
        _, active = eng.get_mode()
    except _capi.PbdError as ex:
        return {"error": str(ex)}
    finally:
        if eng is not None:
            eng.close()
    return {"ms": ms, "steps": steps, "active": active, "wall_s": time.time() - t0}


def pose_write_timing(m, mode, k, steps=200):
    """ms per step (wall clock, after a sync) of `steps` steps, each preceded by a move of every replica's colliders drawn by a torch op on the
    GPU: {"none": rows drawn but not written, "host": rows copied to the host and written by pbd_set_replica_colliders, "device": written by
    pbd_set_replica_collider_poses_device}."""
    import ctypes as C
    import torch
    eng = engine(m, mode, k, colliders=True)
    try:
        rigid, body_x = replica_colliders(m, k)
        nr = len(rigid[0])
        ra = (_capi.RigidCollider * (k * nr))(*[c for r in rigid for c in r])
        fields = np.frombuffer(ra, np.float32).reshape(k * nr, 30)  # the 21 placement floats are columns 9 .. 29
        pc = (_capi.ParticleCollider * 1)(_capi.ParticleCollider(0, len(m["x0"]), 0.5, 0.1))
        base, bx0 = torch.from_numpy(fields[:, 9:].copy()).cuda(), torch.from_numpy(body_x.reshape(-1, 3).copy()).cuda()
        shift = torch.zeros(k * nr, 21, device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        out = {}
        for how in ("none", "host", "device", "none", "host", "device"):
            for passes in range(2):  # the first pass warms up
                torch.cuda.synchronize(); eng.sync()
                t0 = time.perf_counter()
                for t in range(steps):
                    d = 1e-4 * (t % 50)
                    pose = base + shift.fill_(d)   # stands for a policy's action: the rows are born on the GPU
                    bx = bx0 + d
                    if how == "host":
                        fields[:, 9:] = pose.cpu().numpy()
                        host_x = bx.cpu().numpy()
                        _capi._ck(_capi.lib().pbd_set_replica_colliders(eng._h, 1, C.cast(pc, C.c_void_p), nr, C.cast(ra, C.c_void_p),
                                                                        C.c_void_p(host_x.ctypes.data), None, None))
                    elif how == "device":
                        eng.set_replica_collider_poses_device(pose, bx, stream=s)
                    eng.step(1)
                torch.cuda.synchronize(); eng.sync()
                ms = (time.perf_counter() - t0) * 1e3 / steps
            out.setdefault(how, []).append(ms)
        return out
    finally:
        eng.close()


# --forces: (scene, K) rows; cfg2 is the single-scene flagship (bench.py)
FORCE_SCENES = dict(SCENES, cfg2=(lambda m: scenes.cfg2(m), 1, 20, [1]))
FORCE_ROWS = [("cfg2", 1), ("cfg1", 132), ("cfg1", 1056), ("cloth100_xpbd", 264)]


def force_write_timing(m, mode, k, steps=200):
    """ms per step (wall clock, after a sync) of `steps` steps, each preceded by a write of every particle's force drawn by a torch op on the
    GPU: {"none": forces drawn but not written, "host": copied to the host and written by pbd_set_external_forces, "device": written by
    pbd_set_external_forces_device}."""
    import torch
    eng = engine(m, mode, k, forces=True)
    try:
        shape = ((k,) if k > 1 else ()) + (len(m["x0"]), 3)
        base = torch.zeros(shape, device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        out = {}
        for how in ("none", "host", "device", "none", "host", "device"):
            for passes in range(2):  # the first pass warms up
                torch.cuda.synchronize(); eng.sync()
                t0 = time.perf_counter()
                for t in range(steps):
                    f = base + 1e-3 * (t % 50)  # stands for a policy's action: the forces are born on the GPU
                    if how == "host":
                        eng.set_external_forces(f.cpu().numpy())
                    elif how == "device":
                        eng.set_external_forces_device(f, stream=s)
                    eng.step(1)
                torch.cuda.synchronize(); eng.sync()
                ms = (time.perf_counter() - t0) * 1e3 / steps
            out.setdefault(how, []).append(ms)
        return out
    finally:
        eng.close()


def forces_main(a, res):
    res["forces"], res["force_writes"] = [], []
    for name, k in FORCE_ROWS:
        m = model(name, FORCE_SCENES)
        for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
            # off, on, off, on with zero forces: the same work but the force read; the spread of each pair is next to the difference
            ms = [measure(m, md, k, forces=bool(i & 1)).get("ms", float("nan")) for i in range(4)]
            extra = min(ms[1::2]) - min(ms[0::2])
            res["forces"].append({"scene": name, "K": k, "mode": label, "off_ms": ms[0::2], "on_ms": ms[1::2], "forces_ms": extra})
            print("  forces %-13s K=%5d %-8s off %.4f %.4f ms | on %.4f %.4f ms | forces %+.4f ms (%+.1f %%)"
                  % (name, k, label, ms[0], ms[2], ms[1], ms[3], extra, 100.0 * extra / min(ms[0::2])), flush=True)
            if name != "cfg2":
                w = force_write_timing(m, md, k)
                res["force_writes"].append({"scene": name, "K": k, "mode": label, **{h + "_ms": v for h, v in w.items()}})
                print("  force writes %-13s K=%5d %-8s per step: no write %.4f %.4f ms | host call %.4f %.4f ms | device call %.4f %.4f ms"
                      % (name, k, label, *w["none"], *w["host"], *w["device"]), flush=True)


def one_after_another(m, mode, k):
    """ms for K replicas stepped one after another by one K = 1 engine: per replica, its x and v uploaded, one step, x and v read
    back (the replicas' states are kept on the host between their steps); wall clock around the sequence, after one warm-up pass."""
    eng = engine(m, mode, 1)
    try:
        n = len(m["x0"])
        xs = np.repeat(np.asarray(m["x0"], np.float32)[None], k, 0)
        vs = np.zeros_like(xs)
        for passes in range(2):  # the first pass warms up
            eng.sync()
            t0 = time.perf_counter()
            for r in range(k):
                eng.set_attr(_capi.ATTR_X, xs[r]); eng.set_attr(_capi.ATTR_V, vs[r])
                eng.step(1)
                eng.get_attr(_capi.ATTR_X, xs[r]); eng.get_attr(_capi.ATTR_V, vs[r])
            eng.sync()
            ms = (time.perf_counter() - t0) * 1e3
        assert xs.shape == (k, n, 3)
        return ms
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    ap.add_argument("--quick", action="store_true", help="first two K of every sweep, no C sweep (a rehearsal)")
    ap.add_argument("--scenes", default=",".join(SCENES))
    ap.add_argument("--replica-rows", action="store_true", help="every batch also with per-replica rows equal to the shared parameters")
    ap.add_argument("--sweep", action="store_true", help="132 cfg1 replicas, each with its own stiffnesses")
    ap.add_argument("--rest-shapes", action="store_true", help="every batch also with per-replica rest shapes; device derivation against host builds")
    ap.add_argument("--colliders", action="store_true", help="only the contact path: batches without and with three per-replica colliders")
    ap.add_argument("--constraint-materials", action="store_true", help="every batch also with per-constraint materials equal to the shared ones; gather timing")
    ap.add_argument("--contact-sensors", action="store_true", help="only the contact path: sensing off / on, and per-step collider moves by host and device calls")
    ap.add_argument("--forces", action="store_true", help="only external forces: zero forces off / on, and per-step force writes by host and device calls")
    ap.add_argument("--rigid", action="store_true", help="only batches of the rigid-body coupling rig and the masked device body write")
    ap.add_argument("--ks", default=None, help="comma-separated K to measure instead of each scene's sweep")
    ap.add_argument("--no-baseline", action="store_true", help="skip the one-after-another baseline and the C sweep")
    a = ap.parse_args()
    res = {"card": card(), "rows": [], "c_sweep": [], "replica_rows": [], "sweep": [], "rest_shapes": [], "derive": [], "colliders": [],
           "constraint_materials": [], "gather": [], "rigid": []}
    print("card: %s" % res["card"], flush=True)
    if a.rigid or a.forces:
        (rigid_main if a.rigid else forces_main)(a, res)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
        return
    if a.contact_sensors:
        res["contact_sensors"], res["pose_writes"] = [], []
        for name, ks in COLLIDER_KS.items():
            m = model(name)
            for k in ([int(v) for v in a.ks.split(",")] if a.ks else ks):
                for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
                    # off, on, off, on: the spread of each pair is next to the difference between them
                    ms = [measure(m, md, k, colliders=True, sense=bool(i & 1)).get("ms", float("nan")) for i in range(4)]
                    extra = min(ms[1::2]) - min(ms[0::2])
                    res["contact_sensors"].append({"scene": name, "K": k, "mode": label, "off_ms": ms[0::2], "on_ms": ms[1::2], "sensing_ms": extra})
                    print("  sensors %-13s K=%5d %-8s off %.4f %.4f ms | on %.4f %.4f ms | sensing %+.4f ms (%+.1f %%)"
                          % (name, k, label, ms[0], ms[2], ms[1], ms[3], extra, 100.0 * extra / min(ms[0::2])), flush=True)
                    w = pose_write_timing(m, md, k)
                    res["pose_writes"].append({"scene": name, "K": k, "mode": label, **{h + "_ms": v for h, v in w.items()}})
                    print("  pose writes %-13s K=%5d %-8s per step: no move %.4f %.4f ms | host call %.4f %.4f ms | device call %.4f %.4f ms"
                          % (name, k, label, *w["none"], *w["host"], *w["device"]), flush=True)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
        return
    if a.colliders:
        for name, ks in COLLIDER_KS.items():
            m = model(name)
            for k in ([int(v) for v in a.ks.split(",")] if a.ks else ks):
                for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
                    # without, with, without, with: the spread of each pair is next to the difference between them
                    ms = [measure(m, md, k, colliders=bool(i & 1)).get("ms", float("nan")) for i in range(4)]
                    launch = min(ms[1::2]) - min(ms[0::2])
                    res["colliders"].append({"scene": name, "K": k, "mode": label, "without_ms": ms[0::2], "with_ms": ms[1::2], "contact_launch_ms": launch})
                    print("  colliders %-13s K=%5d %-8s without %.4f %.4f ms | with 3 per replica %.4f %.4f ms | contact launch %.4f ms (%.1f %% of the step)"
                          % (name, k, label, ms[0], ms[2], ms[1], ms[3], launch, 100.0 * launch / min(ms[0::2])), flush=True)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
        return
    for name in a.scenes.split(","):
        m = model(name)
        ncons = len(m["types"])
        proj = ncons * m["sub"] * m["it"]
        solo = {md: measure(m, md, 1) for md in (_capi.MODE_GRAPH, _capi.MODE_RESIDENT)}
        solo_mode = min((r["ms"], md) for md, r in solo.items() if "ms" in r)[1]
        ks = [int(v) for v in a.ks.split(",")] if a.ks else (SCENES[name][3][:2] if a.quick else SCENES[name][3])
        print("%s: %d particles, %d constraints, %d x %d; K = 1: graph %.3f ms, resident %s ms" % (
            name, len(m["x0"]), ncons, m["sub"], m["it"], solo[0]["ms"], "%.3f" % solo[1]["ms"] if "ms" in solo[1] else solo[1]["error"]), flush=True)
        for k in ks:
            row = {"scene": name, "K": k, "baseline_ms": float("nan") if a.no_baseline else one_after_another(m, solo_mode, k)}
            for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT), ("auto", _capi.MODE_AUTO)):
                r = measure(m, md, k)
                row[label] = r
                if "ms" in r:
                    r["proj_per_s"] = k * proj / (r["ms"] * 1e-3)
            res["rows"].append(row)
            fmt = lambda r: ("%9.3f ms %8.2e/s" % (r["ms"], r["proj_per_s"])) if "ms" in r else ("refused: " + r["error"][:60])
            print("  K=%5d  graph %s | resident %s | auto(%s) %s | one after another %9.3f ms" % (
                k, fmt(row["graph"]), fmt(row["resident"]), row["auto"].get("active"), fmt(row["auto"]), row["baseline_ms"]), flush=True)
        for k in (ks if a.replica_rows else []):
            if k == 1:
                continue
            rows = shared_rows(m, k)
            for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
                # shared, rows, shared, rows: the spread of each pair is next to the difference between them
                ms = [measure(m, md, k, rows=rows if i & 1 else None).get("ms", float("nan")) for i in range(4)]
                res["replica_rows"].append({"scene": name, "K": k, "mode": label, "shared_ms": ms[0::2], "rows_ms": ms[1::2]})
                print("  rows K=%5d %-8s shared %.4f %.4f ms | per-replica rows %.4f %.4f ms" % (k, label, ms[0], ms[2], ms[1], ms[3]), flush=True)
        for k in (ks if a.rest_shapes else []):
            if k == 1:
                continue
            for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
                # shared, per-replica, shared, per-replica: the spread of each pair is next to the difference between them
                ms = [measure(m, md, k, rest=bool(i & 1)).get("ms", float("nan")) for i in range(4)]
                geo_mb = sum(k * int((np.asarray(m["types"]) == t).sum()) * GEO_BYTES.get(t, 0) for t in range(_capi.NUM_TYPES)) * 1e-6
                res["rest_shapes"].append({"scene": name, "K": k, "mode": label, "shared_ms": ms[0::2], "rest_ms": ms[1::2], "geometry_mb": geo_mb})
                print("  rest shapes K=%5d %-8s shared %.4f %.4f ms | per-replica %.4f %.4f ms (%.0f MB of geometry)" % (k, label, ms[0], ms[2], ms[1], ms[3], geo_mb), flush=True)
        for k in (ks if a.constraint_materials else []):
            if k == 1:
                continue
            cm = constraint_materials(m, k)
            mb = sum(f.size for f in cm.values()) * 4 * 1e-6  # the device-ordered arrays the kernels read (the engine's copy is as large)
            for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
                # shared, per-constraint, shared, per-constraint: the spread of each pair is next to the difference between them
                ms = [measure(m, md, k, cmat=cm if i & 1 else None).get("ms", float("nan")) for i in range(4)]
                res["constraint_materials"].append({"scene": name, "K": k, "mode": label, "shared_ms": ms[0::2], "constraint_ms": ms[1::2], "arrays_mb": mb})
                print("  constraint materials K=%5d %-8s shared %.4f %.4f ms | per-constraint %.4f %.4f ms (%.0f MB of material arrays)"
                      % (k, label, ms[0], ms[2], ms[1], ms[3], mb), flush=True)
            for g in gather_timing(m, k):
                g["scene"] = name
                res["gather"].append(g)
                print("  gather K=%5d type %2d %-4s %8.1f us  %.1f MB  %.2f TB/s (%.0f %% of 3.35 TB/s)"
                      % (k, g["type"], g["mask"], g["us"], g["bytes"] * 1e-6, g["tb_s"], 100.0 * g["tb_s"] / 3.35), flush=True)
        if a.rest_shapes and name in DERIVE_K:
            d = derive_timing(name, m, DERIVE_K[name])
            res["derive"].append(d)
            print("  derive K=%5d: device %.3f s, host models %.3f s each -> %.1f s for K" % (d["K"], d["device_s"], d["host_one_s"], d["host_K_s"]), flush=True)
        if a.sweep and name == "cfg1":
            k = 132
            rows = shared_rows(m, k)
            scale = np.linspace(0.1, 1.0, k, dtype=np.float32)[:, None]
            swept = ({t: mat * scale for t, mat in rows[0].items()}, rows[1])
            for label, md in (("graph", _capi.MODE_GRAPH), ("resident", _capi.MODE_RESIDENT)):
                r = measure(m, md, k, rows=swept)
                r.update({"scene": name, "K": k, "mode": label})
                res["sweep"].append(r)
                print("  stiffness sweep K=%5d %-8s %s" % (k, label, ("%.4f ms" % r["ms"]) if "ms" in r else r["error"][:80]), flush=True)
        if a.quick or a.no_baseline or name not in C_SWEEP:
            continue
        for k in C_SWEEP[name]:
            for c in (1, 2, 4, 8, 16):
                r = measure(m, _capi.MODE_RESIDENT, k, clusters=c)
                r.update({"scene": name, "K": k, "C": c})
                res["c_sweep"].append(r)
                print("  C sweep K=%5d C=%2d: %s" % (k, c, ("%.3f ms" % r["ms"]) if "ms" in r else r["error"][:80]), flush=True)
    os.environ.pop("PBD_B200_CLUSTERS", None)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
