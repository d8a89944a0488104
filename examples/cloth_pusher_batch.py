"""A batch of pushers sweeping through cloths, driven from PyTorch without a host round trip (pbd_set_replica_collider_poses_device and the
contact sensors): K cloths lie on a floor; each replica has a sphere or a turning box that sweeps through its cloth along a path drawn in
torch, at its own speed.  Every step torch computes the pushers' placement rows, writes them under a mask (the pushers still moving, and the
ones just restarted), and reads every collider's contact count and impulse into tensors.  A replica whose pusher force exceeds a threshold,
or whose episode ended, restarts from the initial cloth through the device state calls under the same mask.

The same loop then runs on the host calls (pbd_set_replica_colliders with the rows copied to the host, pbd_get_contacts summed per collider,
pbd_get_contact_sensors) and the two must end bit for bit in the same state.  Needs a CUDA device.

    python examples/cloth_pusher_batch.py [--replicas K] [--steps S] [--episode T] [--force F]"""
import argparse
import ctypes as C
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel

TOL, DT = 0.05, 0.005
RX90 = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])
FLOOR_C, FLOOR_HALF = (0.0, -0.5, 0.0), (10.0, 0.5, 10.0)
SPHERE_R, BOX_HALF, START_X, HEIGHT = 0.25, 0.25, -1.6, 0.3   # the pushers skim the floor: their lowest point 0.05 above it


def cloth():
    hm = HostModel()
    hm.add_regular_triangle_model(24, 24, t=(-1.0, 0.03, -1.0), R=RX90, scale=(2.0, 2.0))
    hm.add_cloth_constraints(0, 4, dist_k=1.0e5)
    hm.add_bending_constraints(0, 3, 100.0)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x = np.asarray(hm.get("x"), np.float32).copy()
    hm.close()
    return types, bodies, params, off, ids, np.asarray(mass, np.float32), x


def placement(t, speed, box, z):
    """The pushers' placement at step t (all (K,) tensors on the GPU): pose rows (K, 21) = R (rot^T, row-major), v1 = 0, v2 = centre,
    bounding box = the rotated half extents + tolerance; centre, velocity and angular velocity (K, 3)."""
    tf = t.to(torch.float32) * DT
    centre = torch.stack([START_X + speed * tf, torch.full_like(tf, HEIGHT), z], 1)
    w = 2.0 * box.to(torch.float32)                    # boxes turn about y at 2 rad/s, spheres do not turn
    c, s = torch.cos(w * tf), torch.sin(w * tf)
    one, zero = torch.ones_like(tf), torch.zeros_like(tf)
    rot = torch.stack([c, zero, s, zero, one, zero, -s, zero, c], 1).view(-1, 3, 3)   # about y
    half_local = torch.where(box[:, None], torch.full((len(t), 3), BOX_HALF, device=t.device), torch.full((len(t), 3), SPHERE_R, device=t.device))
    half = (rot.abs() @ half_local[:, :, None])[:, :, 0] + TOL
    pose = torch.cat([rot.transpose(1, 2).reshape(-1, 9), torch.zeros_like(centre), centre, centre - half, centre + half], 1)
    vel = torch.stack([speed, zero, zero], 1)
    omega = torch.stack([zero, w, zero], 1)
    return pose, centre, vel, omega


def rigid_colliders(K, box, pose):
    """The K x [floor, pusher] pbd_rigid_colliders, placements from pose (K, 2, 21) on the host."""
    out = (_capi.RigidCollider * (2 * K))()
    for r in range(K):
        for j in range(2):
            rc = out[2 * r + j]
            if j == 0:
                rc.shape, rc.dim[:], rc.friction = _capi.SHAPE_BOX, FLOOR_HALF, 0.3
            elif box[r]:
                rc.shape, rc.dim[:], rc.friction = _capi.SHAPE_BOX, (BOX_HALF,) * 3, 0.2
            else:
                rc.shape, rc.dim[:], rc.friction = _capi.SHAPE_SPHERE, (SPHERE_R, 0.0, 0.0), 0.2
            rc.body, rc.restitution = j, 0.2
            p = pose[r, j]
            rc.R[:] = p[0:9].tolist(); rc.v1[:] = p[9:12].tolist(); rc.v2[:] = p[12:15].tolist()
            rc.aabb_min[:] = p[15:18].tolist(); rc.aabb_max[:] = p[18:21].tolist()
    return out


def run(device_loop, K, steps, episode, force_limit):
    types, bodies, params, off, ids, mass, x = cloth()
    n = len(x)
    eng = _capi.Engine(0)
    eng.set_particles(x, mass)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=DT, sub_steps=1, max_iter=5)
    eng.set_replicas(K)
    eng.set_contact_params(tolerance=TOL, stiffness=100.0, max_iter_v=5)
    eng.sense_contacts(True)
    if not device_loop:
        eng.record_contacts(1 << 20)
    dev = torch.device("cuda")
    r_idx = torch.arange(K, device=dev)
    box = (r_idx % 2) == 1
    z = 0.4 * torch.sin(1.7 * r_idx.to(torch.float32))
    episodes = torch.zeros(K, dtype=torch.int64, device=dev)
    speed = lambda: 1.0 + 1.5 * torch.frac(0.618034 * (r_idx + 7 * episodes).to(torch.float32))   # m/s, per replica and episode
    t = torch.zeros(K, dtype=torch.int64, device=dev)
    floor_pose = torch.tensor([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, *FLOOR_C, *(np.subtract(FLOOR_C, FLOOR_HALF) - TOL), *(np.add(FLOOR_C, FLOOR_HALF) + TOL)],
                              dtype=torch.float32, device=dev)
    init = torch.from_numpy(np.tile(x, (K, 1))).to(dev).reshape(-1)
    zeros = torch.zeros(K * n * 3, device=dev)

    def rows(t):
        pose, centre, vel, omega = placement(t, speed(), box, z)
        P = torch.stack([floor_pose.expand(K, 21), pose], 1).contiguous()                                             # (K, 2, 21)
        bx = torch.stack([torch.tensor(FLOOR_C, device=dev).expand(K, 3), centre], 1).contiguous()
        bv = torch.stack([torch.zeros(K, 3, device=dev), vel], 1).contiguous()
        bw = torch.stack([torch.zeros(K, 3, device=dev), omega], 1).contiguous()
        return P, bx, bv, bw

    P, bx, bv, bw = rows(t)
    host_rows = [a.cpu().numpy() for a in (P, bx, bv, bw)]
    pc = [_capi.ParticleCollider(0, n, 0.5, 0.1)]
    first = rigid_colliders(K, box.cpu().numpy(), host_rows[0])
    eng.set_replica_colliders(pc, [list(first[2 * r:2 * r + 2]) for r in range(K)], *host_rows[1:])
    count = torch.zeros(K * 2, dtype=torch.int32, device=dev).view(torch.uint32)
    impulse = torch.zeros(K * 2 * 3, device=dev)
    restarts, peak = torch.zeros((), dtype=torch.int64, device=dev), torch.zeros((), device=dev)
    for step in range(steps):
        moving = (t * DT * speed() < 2 * abs(START_X)) | (t == 0)      # pushers still crossing their cloth, and those just restarted
        P, bx, bv, bw = rows(t)
        if device_loop:
            eng.set_replica_collider_poses_device(P, bx, bv, bw, replicas=moving.to(torch.uint8), stream=torch.cuda.current_stream().cuda_stream)
        else:
            m = moving.cpu().numpy()
            new = [a.cpu().numpy() for a in (P, bx, bv, bw)]   # what a host-call driver must copy and wait for every step
            for old, a in zip(host_rows, new):
                old[m] = a[m]
            rc = rigid_colliders(K, box.cpu().numpy(), host_rows[0])
            _capi._ck(_capi.lib().pbd_set_replica_colliders(eng._h, 1, C.cast((_capi.ParticleCollider * 1)(*pc), C.c_void_p), 2, C.cast(rc, C.c_void_p),
                                                            *[C.c_void_p(a.ctypes.data) for a in host_rows[1:]]))
        eng.step(1)
        if device_loop:
            eng.get_contact_sensors_device(count, impulse, stream=torch.cuda.current_stream().cuda_stream)
            imp = impulse.view(K, 2, 3)
        else:
            got, _ = eng.contacts(1 << 20)
            per = np.zeros((K, 2), np.int32)
            for c in got:
                per[c.particle // n, c.body] += 1
            c_host, i_host = eng.contact_sensors()
            assert np.array_equal(per, c_host.astype(np.int32)), "contact record and sensors disagree"
            imp = torch.from_numpy(i_host).to(dev)
        force = imp[:, 1].norm(dim=1) / DT                               # the pusher's mean force over the step
        peak = torch.maximum(peak, force.max())
        t += 1
        done = (force > force_limit) | (t >= episode)
        restarts += done.sum()
        mask = done.to(torch.uint8)
        if device_loop:
            s = torch.cuda.current_stream().cuda_stream
            for a, src in ((_capi.ATTR_X, init), (_capi.ATTR_V, zeros), (_capi.ATTR_OLDX, init), (_capi.ATTR_LASTX, init)):
                eng.set_attr_device(a, src, replicas=mask, stream=s)
        elif done.any():
            d = done.cpu().numpy()
            for a, src in ((_capi.ATTR_X, x), (_capi.ATTR_V, np.zeros_like(x)), (_capi.ATTR_OLDX, x), (_capi.ATTR_LASTX, x)):
                cur = eng.get_attr(a)
                cur[d] = src
                eng.set_attr(a, cur)
        episodes += done.to(torch.int64)
        t = torch.where(done, torch.zeros_like(t), t)
    eng.sync()
    out = eng.get_attr(_capi.ATTR_X).copy(), eng.get_attr(_capi.ATTR_V).copy(), eng.contact_sensors()
    eng.close()
    return out, int(restarts), episodes.cpu().numpy(), float(peak)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=16)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--episode", type=int, default=150, help="steps before a replica restarts")
    ap.add_argument("--force", type=float, default=2000.0, help="pusher force (N) above which a replica restarts")
    a = ap.parse_args()
    (xd, vd, (cd, idv)), restarts, episodes, peak = run(True, a.replicas, a.steps, a.episode, a.force)
    (xh, vh, (ch, ih)), restarts_h, episodes_h, _ = run(False, a.replicas, a.steps, a.episode, a.force)
    for r in range(a.replicas):
        print("replica %3d (%s): %d restarts, last step: %3d floor contacts, %3d pusher contacts, pusher impulse (%.3f, %.3f, %.3f) N s"
              % (r, "box" if r % 2 else "sphere", episodes[r], cd[r, 0], cd[r, 1], *idv[r, 1]))
    same = (np.array_equal(xd, xh) and np.array_equal(vd, vh) and np.array_equal(cd, ch) and np.array_equal(idv.view(np.uint32), ih.view(np.uint32))
            and np.array_equal(episodes, episodes_h))
    print("%d replicas, %d steps, %d restarts (device) / %d (host), peak pusher force %.1f N" % (a.replicas, a.steps, restarts, restarts_h, peak))
    finite = bool(np.isfinite(xd).all() and np.isfinite(vd).all())
    print("every cloth finite: %s" % ("yes" if finite else "no"))
    print("device loop = host loop, bit for bit: %s" % ("yes" if same else "no"))
    return 0 if same and finite else 1


if __name__ == "__main__":
    sys.exit(main())
