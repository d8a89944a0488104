"""K copies of the rigid-body cloth coupling rig of rigid_body_cloth_coupling.py stepped as one replica batch and driven from PyTorch: a
20 x 20 cloth hung between four three-body chains (static anchor + two dynamic boxes joined by BallJoints), its corners tied to the top
box of each chain by RigidBodyParticleBallJoints.  Every replica has its own box masses (pbd_set_replica_rigid_bodies) and its own gravity
(pbd_set_replica_gravity).  Every step torch moves each replica's static anchors up and down on a replica's own phase -- the action of a
policy that acts through grippers -- by reading the bodies (pbd_get_rigid_bodies_device) and writing them back with the new anchor
positions (pbd_set_rigid_bodies_device).  A replica whose episode has run its length is restarted from its initial state by masked device
writes of its particles (x, v, oldX = x, lastX = x) and its bodies.  Nothing crosses to the host inside the loop.  The same loop written on
the host calls (pbd_get_rigid_bodies / pbd_set_replica_rigid_bodies, pbd_get_attr / pbd_set_attr of all K replicas) runs next to it and
must end in the same state bit for bit.  Needs a CUDA device and torch.

    python examples/rigid_body_cloth_coupling_batch.py [--replicas K] [--steps S] [--seed N]"""
import argparse
import math
import os
import sys
import time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel

N_ROWS, N_COLS = 20, 20
WIDTH, HEIGHT, DEPTH = 0.4, 2.0, 0.4  # the dynamic boxes (RigidBodyClothCouplingDemo.cpp:33-35)
CORNERS = ((-5.0, -5.0), (5.0, -5.0), (5.0, 5.0), (-5.0, 5.0))
ANCHORS = np.array([0, 3, 6, 9])      # the static body of each chain
AMPLITUDE = 0.5                       # of the anchors' vertical motion


def box_inertia(mass, w, h, d):
    return (mass / 12.0 * (h * h + d * d), mass / 12.0 * (w * w + d * d), mass / 12.0 * (w * w + h * h))


def rig():
    """The model (one replica) as flat arrays, and its 12 bodies: mass, x, q (w, x, y, z), principal inertia."""
    hm = HostModel()
    c, s = math.cos(math.pi * 0.5), math.sin(math.pi * 0.5)
    hm.add_regular_triangle_model(N_COLS, N_ROWS, t=(-5.0, 4.0, -5.0), R=np.array([[1, 0, 0], [0, c, -s], [0, s, c]]), scale=(10.0, 10.0))
    hm.add_cloth_constraints(0, 2, dist_k=1.0)
    hm.add_bending_constraints(0, 2, 0.01)
    mass, x, inertia = [], [], []
    for cx, cz in CORNERS:
        for m, y, I in ((0.0, 0.0, box_inertia(1.0, 0.5, 0.5, 0.5)), (1.0, 1.0, box_inertia(1.0, WIDTH, HEIGHT, DEPTH)),
                        (1.0, 3.0, box_inertia(1.0, WIDTH, HEIGHT, DEPTH))):
            hm.add_rigid_body(m, (cx, y, cz), I)
            mass.append(m); x.append((cx, y, cz)); inertia.append(I)
    for chain, (cx, cz) in enumerate(CORNERS):
        hm.add_ball_joint(3 * chain, 3 * chain + 1, (cx, 0.0, cz))
        hm.add_ball_joint(3 * chain + 1, 3 * chain + 2, (cx, 2.0, cz))
    for chain, particle in enumerate((0, N_COLS - 1, N_ROWS * N_COLS - 1, (N_ROWS - 1) * N_COLS)):
        hm.add_rb_particle_ball_joint(3 * chain + 2, particle)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    pmass, _ = hm.masses()
    px = np.asarray(hm.get("x"), np.float32).copy()
    hm.close()
    nb = len(mass)
    q = np.tile(np.float32([1, 0, 0, 0]), (nb, 1))
    return (types, bodies, params, off, ids, px, np.asarray(pmass, np.float32),
            (np.asarray(mass, np.float32), np.asarray(x, np.float32), q, np.asarray(inertia, np.float32)))


def setup(K, seed):
    """The batch engine and every replica's initial state: its own box masses (scaled by 0.5 .. 2), gravity, anchor phase and episode length."""
    types, bodies, params, off, ids, px, pmass, (bm, bx, bq, bI) = rig()
    rng = np.random.default_rng(seed)
    scale = rng.uniform(0.5, 2.0, (K, 1)).astype(np.float32)
    mass = np.where(bm[None] != 0, bm[None] * scale, np.float32(0)).astype(np.float32)
    inertia = (bI[None] * np.where(bm[None] != 0, scale, np.float32(1))[..., None]).astype(np.float32)
    init = dict(x=np.repeat(px[None], K, 0), v=np.zeros((K, len(px), 3), np.float32), bmass=mass, bx=np.repeat(bx[None], K, 0),
                bq=np.repeat(bq[None], K, 0), binertia=inertia)
    gravity = np.stack([np.float32([0.0, -9.81, 0.0]) + rng.normal(0.0, 1.0, 3).astype(np.float32) for _ in range(K)]).astype(np.float32)
    phase = rng.uniform(0.0, 2.0 * math.pi, K)
    episode = rng.integers(30, 60, K)
    eng = _capi.Engine(0)
    eng.set_particles(px, pmass)
    eng.set_replicas(K)
    eng.set_replica_rigid_bodies(mass, init["bx"], init["bq"], inertia)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=0.005, sub_steps=5, max_iter=1, vel_method=0)
    eng.set_replica_gravity(gravity)
    return eng, init, phase, episode


def anchor_heights(phase, step):
    """(K,) the anchors' height at `step`, in float32 as both loops write it."""
    return (AMPLITUDE * np.sin(phase + 0.05 * step)).astype(np.float32)


def run_device(K, steps, seed):
    eng, init, phase, episode = setup(K, seed)
    nb, n = init["bx"].shape[1], init["x"].shape[1]
    dev = torch.device("cuda")
    s = torch.cuda.current_stream().cuda_stream
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).to(dev)
    X0, BX0, BQ0, BM0, BI0 = t(init["x"]), t(init["bx"]), t(init["bq"]), t(init["bmass"]), t(init["binertia"])
    V0, BZ = torch.zeros_like(X0), torch.zeros(K * nb * 3, device=dev)
    heights = torch.from_numpy(np.stack([anchor_heights(phase, i) for i in range(steps)])).to(dev)  # (steps, K)
    episode = torch.from_numpy(episode).to(dev)
    anchors = torch.from_numpy(ANCHORS).to(dev)
    age = torch.zeros(K, dtype=torch.int64, device=dev)
    restarts = torch.zeros(K, dtype=torch.int64, device=dev)
    bx, bq, bv, bw = (torch.empty(K * nb * c, device=dev) for c in (3, 4, 3, 3))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        eng.get_rigid_bodies_device(bx, bq, bv, bw, stream=s)  # the action: every replica's anchors at their height of this step
        bx.view(K, nb, 3)[:, anchors, 1] = heights[i][:, None]
        eng.set_rigid_bodies_device(bx, bq, v=bv, omega=bw, stream=s)
        eng.step(1)
        age += 1
        done = age >= episode
        restarts += done
        age[done] = 0
        for attr, src in ((_capi.ATTR_X, X0), (_capi.ATTR_V, V0), (_capi.ATTR_OLDX, X0), (_capi.ATTR_LASTX, X0)):
            eng.set_attr_device(attr, src, replicas=done, stream=s)
        eng.set_rigid_bodies_device(BX0, BQ0, v=BZ, omega=BZ, mass=BM0, inertia=BI0, replicas=done, stream=s)
    xs = eng.get_attr_device(_capi.ATTR_X, torch.empty(K * n * 3, device=dev), stream=s)
    vs = eng.get_attr_device(_capi.ATTR_V, torch.empty(K * n * 3, device=dev), stream=s)
    eng.get_rigid_bodies_device(bx, bq, bv, bw, stream=s)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    eng.close()
    body = np.concatenate([a.cpu().numpy().reshape(K, nb, -1) for a in (bx, bq, bv, bw)], axis=2)
    return xs.cpu().numpy().reshape(K, n, 3), vs.cpu().numpy().reshape(K, n, 3), body, restarts.cpu().numpy(), ms


def run_host(K, steps, seed):
    eng, init, phase, episode = setup(K, seed)
    age = np.zeros(K, np.int64)
    restarts = np.zeros(K, np.int64)
    t0 = time.perf_counter()
    for i in range(steps):
        b = eng.get_rigid_bodies()
        b[:, ANCHORS, 1] = anchor_heights(phase, i)[:, None]
        eng.set_replica_rigid_bodies(init["bmass"], b[..., :3], b[..., 3:7], init["binertia"], b[..., 7:10], b[..., 10:13])
        eng.step(1)
        age += 1
        done = age >= episode
        restarts += done
        age[done] = 0
        if done.any():  # the host calls write every replica: read the state back, patch the done rows, write it all
            state = {a: eng.get_attr(a) for a in (_capi.ATTR_X, _capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX)}
            for a, src in ((_capi.ATTR_X, init["x"]), (_capi.ATTR_V, init["v"]), (_capi.ATTR_OLDX, init["x"]), (_capi.ATTR_LASTX, init["x"])):
                state[a][done] = src[done]
                eng.set_attr(a, state[a])
            b = eng.get_rigid_bodies()
            bx, bq, bv, bw = b[..., :3].copy(), b[..., 3:7].copy(), b[..., 7:10].copy(), b[..., 10:13].copy()
            bx[done], bq[done], bv[done], bw[done] = init["bx"][done], init["bq"][done], 0.0, 0.0
            eng.set_replica_rigid_bodies(init["bmass"], bx, bq, init["binertia"], bv, bw)
    x_end, v_end, body = eng.get_attr(_capi.ATTR_X), eng.get_attr(_capi.ATTR_V), eng.get_rigid_bodies()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    eng.close()
    return x_end, v_end, body, restarts, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=64)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    xd, vd, bd, rd, msd = run_device(a.replicas, a.steps, a.seed)
    xh, vh, bh, rh, msh = run_host(a.replicas, a.steps, a.seed)
    same = np.array_equal(xd, xh) and np.array_equal(vd, vh) and np.array_equal(bd, bh) and np.array_equal(rd, rh)
    print("%d rig replicas, %d steps: %d restarts; device-memory loop %.3f ms/step, host loop %.3f ms/step (wall clock, small scene: "
          "launch-bound)" % (a.replicas, a.steps, rd.sum(), msd, msh))
    print("final state of the device-memory loop equals the host-call loop bit for bit: %s" % ("yes" if same else "NO"))
    return 0 if same and rd.sum() > 0 and np.isfinite(xd).all() else 1


if __name__ == "__main__":
    sys.exit(main())
