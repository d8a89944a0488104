"""CPU-side guard of the batched contact kernel: csrc/contacts.cuh compiled for the host through the test-only shim (tests/host_shim/),
k_contacts_batch over K = 5 replicas with colliders that differ in every field (blockIdx.y = replica), against k_contacts run on each
replica alone.  Every replica must match bit for bit: velocities, and the contact records with the particle index shifted by r n.  The GPU
tests proper are in tests/test_gpu_batch_contacts.py; this one runs without a GPU and is not a product path."""
import ctypes as C
import os
import subprocess
import numpy as np

import contact_util as cu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REC = np.dtype([("particle", "<u4"), ("body", "<u4"), ("cp0", "<f4", 3), ("cp1", "<f4", 3), ("n", "<f4", 3), ("dist", "<f4")])


class _RC(C.Structure):  # pbdk::RigidCollider
    _fields_ = [("shape", C.c_int), ("body", C.c_uint), ("dim", C.c_float * 3), ("thickness", C.c_float), ("invert", C.c_float), ("restitution", C.c_float),
                ("friction", C.c_float), ("R", C.c_float * 9), ("v1", C.c_float * 3), ("v2", C.c_float * 3), ("aabbMin", C.c_float * 3), ("aabbMax", C.c_float * 3)]


class _PC(C.Structure):  # pbdk::ParticleCollider
    _fields_ = [("offset", C.c_uint), ("count", C.c_uint), ("restitution", C.c_float), ("friction", C.c_float)]


def _rc(d):
    rc = _RC()
    rc.shape = d["shape"]; rc.body = d["body"]; rc.dim[:] = d["dim"]; rc.thickness = d["thickness"]; rc.invert = -1.0 if d["invert"] else 1.0
    rc.restitution = d["restitution"]; rc.friction = d["friction"]; rc.R[:] = d["R"]; rc.v1[:] = d["v1"]; rc.v2[:] = d["v2"]
    rc.aabbMin[:] = d["aabb_min"]; rc.aabbMax[:] = d["aabb_max"]
    return rc


def _f4(xyz, w):
    a = np.zeros(xyz.shape[:-1] + (4,), np.float32); a[..., :3] = xyz; a[..., 3] = w
    return a


def test_batched_contact_kernel_equals_one_scene_per_replica(tmp_path):
    so = str(tmp_path / "libcontacts_batch_host.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "tests", "host_shim"), "-I" + os.path.join(ROOT, "positionbaseddynamics_b200", "csrc"),
                           "-o", so, os.path.join(ROOT, "tests", "host_shim", "run_contacts_batch.cpp")])
    lib = C.CDLL(so)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    K, n, cap = 5, 3000, 1 << 16
    rng = np.random.default_rng(11)
    fp = (np.array([0.0, 2.2, 0.0]), np.array([2.5, 0.05, 2.5]))
    cols, bx, bv, bw = cu.batch_scene(K, fp, empty=3)
    nR = len(cols[0])
    # particles over the obstacles' region: many inside a shape or its tolerance shell; two ranges, some particles pinned
    lo = fp[0] - fp[1] - np.array([0.0, 2.0, 0.0]); hi = fp[0] + fp[1]
    x = rng.uniform(lo, hi, (K, n, 3)).astype(np.float32)
    v = rng.normal(0.0, 1.0, (K, n, 3)).astype(np.float32)
    mass = rng.uniform(0.5, 2.0, (K, n)).astype(np.float32); mass[:, ::11] = 0.0
    inv = np.where(mass != 0, 1.0 / np.where(mass != 0, mass, 1.0), 0.0).astype(np.float32)
    slot = rng.permutation(n).astype(np.uint32)  # host index -> slot within a replica
    pos = np.zeros((K, n, 4), np.float32); vel = np.zeros((K, n, 4), np.float32)
    for r in range(K):
        pos[r, slot] = _f4(x[r], inv[r]); vel[r, slot] = _f4(v[r], mass[r])
    ranges = (_PC * 2)(_PC(0, 1800, 0.5, 0.1), _PC(2000, 1000, 0.3, 0.25))
    rigid = (_RC * (K * nR))(*[_rc(d) for c in cols for d in c])
    X, V, W = _f4(bx, 0.0), _f4(bv, 0.0), _f4(bw, 0.0)
    args = (C.c_float(cu.TOL), C.c_float(100.0), 5)

    bpos, bvel = pos.copy(), vel.copy()
    rec = np.zeros(cap, REC); cnt = C.c_uint(0)
    lib.run_contacts_batch(K, n, vp(slot), vp(bpos), vp(bvel), vp(X), vp(V), vp(W), nR, C.cast(rigid, C.c_void_p), 2, C.cast(ranges, C.c_void_p), *args,
                           vp(rec), C.byref(cnt), cap)
    assert cnt.value < cap
    got = np.sort(rec[:cnt.value], order=["particle", "body"])
    events = np.bincount(got["particle"] // n, minlength=K)
    print("host shim, batch of %d: contacts per replica %s" % (K, events.tolist()))
    assert events[3] == 0 and all(events[r] > 100 for r in (0, 1, 2, 4))
    assert set(got["body"].tolist()) == set(range(nR))
    for r in range(K):
        spos, svel = pos[r].copy(), vel[r].copy()
        one = (_RC * nR)(*[_rc(dict(d, body=k)) for k, d in enumerate(cols[r])])  # body k carries collider k
        srec = np.zeros(cap, REC); scnt = C.c_uint(0)
        lib.run_contacts_solo(vp(slot), vp(spos), vp(svel), vp(X[r]), vp(V[r]), vp(W[r]), nR, C.cast(one, C.c_void_p), 2, C.cast(ranges, C.c_void_p), *args,
                              vp(srec), C.byref(scnt), cap)
        assert np.array_equal(bvel[r].view(np.uint32), svel.view(np.uint32)), r
        assert np.array_equal(bpos[r].view(np.uint32), spos.view(np.uint32)), r
        want = np.sort(srec[:scnt.value], order=["particle", "body"])
        want["particle"] += r * n
        mine = got[got["particle"] // n == r]
        assert np.array_equal(mine.view(np.uint8), want.view(np.uint8)), r
        assert not np.array_equal(svel, vel[r]) or events[r] == 0, r  # the contacts changed the velocities
