"""CPU-side guard of the contact sensors: csrc/contacts.cuh compiled for the host through the test-only shim (tests/host_shim/), the sensing
instantiation contacts_particle<true, true> over K = 5 replicas against the batched kernel without sensing.  The sensors must count exactly
the contact records of each collider, their impulses must balance the momentum the contacts gave the particles, and sensing must not change
a velocity bit.  The block sums of the GPU kernel and the GPU runs are in tests/test_gpu_contact_sensors.py."""
import ctypes as C
import os
import subprocess

import numpy as np

import contact_util as cu
from test_contacts_batch_host_shim import REC, _PC, _RC, _f4, _rc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENSE = np.dtype([("count", "<u4", 8), ("p", "<f4", (8, 3))])  # pbdk::ContactSense


def _lib(tmp_path, name):
    so = str(tmp_path / ("lib%s.so" % name))
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-std=c++17", "-I" + os.path.join(ROOT, "tests", "host_shim"),
                           "-I" + os.path.join(ROOT, "positionbaseddynamics_b200", "csrc"), "-o", so, os.path.join(ROOT, "tests", "host_shim", name + ".cpp")])
    return C.CDLL(so)


def test_sensors_count_the_records_and_balance_the_momentum(tmp_path):
    sensing, plain = _lib(tmp_path, "run_contact_sensors"), _lib(tmp_path, "run_contacts_batch")
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    K, n, cap = 5, 3000, 1 << 16
    rng = np.random.default_rng(23)
    fp = (np.array([0.0, 2.2, 0.0]), np.array([2.5, 0.05, 2.5]))
    cols, bx, bv, bw = cu.batch_scene(K, fp, empty=3)
    nR = len(cols[0])
    lo = fp[0] - fp[1] - np.array([0.0, 2.0, 0.0]); hi = fp[0] + fp[1]
    x = rng.uniform(lo, hi, (K, n, 3)).astype(np.float32)
    v = rng.normal(0.0, 1.0, (K, n, 3)).astype(np.float32)
    mass = rng.uniform(0.5, 2.0, (K, n)).astype(np.float32); mass[:, ::11] = 0.0
    inv = np.where(mass != 0, 1.0 / np.where(mass != 0, mass, 1.0), 0.0).astype(np.float32)
    slot = rng.permutation(n).astype(np.uint32)
    pos = np.zeros((K, n, 4), np.float32); vel = np.zeros((K, n, 4), np.float32)
    for r in range(K):
        pos[r, slot] = _f4(x[r], inv[r]); vel[r, slot] = _f4(v[r], mass[r])
    ranges = (_PC * 2)(_PC(0, 1800, 0.5, 0.1), _PC(2000, 1000, 0.3, 0.25))
    total = 2800
    rigid = (_RC * (K * nR))(*[_rc(d) for c in cols for d in c])
    X, V, W = _f4(bx, 0.0), _f4(bv, 0.0), _f4(bw, 0.0)
    args = (C.c_float(cu.TOL), C.c_float(100.0), 5)

    runs = []
    for lib in (sensing, plain):
        bpos, bvel = pos.copy(), vel.copy()
        rec = np.zeros(cap, REC); cnt = C.c_uint(0)
        common = (K, n, vp(slot), vp(bpos), vp(bvel), vp(X), vp(V), vp(W), nR, C.cast(rigid, C.c_void_p), 2, C.cast(ranges, C.c_void_p), *args,
                  vp(rec), C.byref(cnt), cap)
        if lib is sensing:
            sense = np.zeros(K * total, SENSE)
            lib.run_contact_sensors(*common, vp(sense))
        else:
            lib.run_contacts_batch(*common)
        assert cnt.value < cap
        runs.append((bpos, bvel, np.sort(rec[:cnt.value], order=["particle", "body"])))
    (spos, svel, srec), (ppos, pvel, prec) = runs
    # sensing changes nothing: velocities, positions and records bit for bit
    assert np.array_equal(svel.view(np.uint32), pvel.view(np.uint32))
    assert np.array_equal(spos.view(np.uint32), ppos.view(np.uint32))
    assert np.array_equal(srec.view(np.uint8), prec.view(np.uint8))

    sense = sense.reshape(K, total)
    count = sense["count"][:, :, :nR].sum(axis=1, dtype=np.int64)           # (K, nR)
    impulse = -sense["p"][:, :, :nR].astype(np.float64).sum(axis=1)          # (K, nR, 3)
    assert not sense["count"][:, :, nR:].any() and not sense["p"][:, :, nR:].any()
    for r in range(K):
        mine = srec[srec["particle"] // n == r]
        want = np.bincount(mine["body"], minlength=nR)  # collider j sits on body j in cu.batch_scene
        assert np.array_equal(count[r], want), (r, count[r], want)
        # the impulse on the colliders balances the momentum the particles gained: sum_i m_i (v_after - v_before)
        dv = svel[r][slot][:, :3].astype(np.float64) - v[r].astype(np.float64)
        gained = (mass[r][:, None].astype(np.float64) * dv).sum(axis=0)
        scale = (mass[r].astype(np.float64) * np.linalg.norm(dv, axis=1)).sum()
        print("replica %d: contacts per collider %s, impulse on the colliders %s, particles' momentum gain %s (scale %.3e)"
              % (r, count[r].tolist(), np.round(impulse[r].sum(axis=0), 4).tolist(), np.round(gained, 4).tolist(), scale))
        assert np.abs(-impulse[r].sum(axis=0) - gained).max() <= 1e-5 * max(scale, 1.0), r
        if r == 3:
            assert count[r].sum() == 0 and not impulse[r].any()
        else:
            assert count[r].sum() > 100 and np.abs(impulse[r]).sum() > 0.0
        # a particle of mass 0 is counted but receives no impulse
        pinned = np.nonzero(mass[r] == 0)[0]
        gids = np.concatenate([np.arange(0, 1800), np.arange(2000, 3000)])
        at = np.isin(gids, pinned)
        assert not sense["p"][r][at].any()
        assert r == 3 or sense["count"][r][at].any(), r
