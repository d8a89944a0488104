"""A batch of cloth drops (pbd_set_replicas + pbd_set_replica_colliders): K copies of a 32 x 32 XPBD cloth, each falling onto its own
randomly placed and rotated box and sphere above a floor, all K stepped by one engine with one contact launch per step.  The kind of
batch a dataset generator or a domain-randomised environment runs.  Headless: prints the contacts of the last step per replica and whether
every cloth came to rest above its own box.  Needs a CUDA device.

    python examples/cloth_collision_batch.py [--replicas K] [--steps S] [--seed N]"""
import argparse
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel

TOL = 0.05
RX90 = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])


def rotation(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.eye(3) + np.sin(angle) * k + (1.0 - np.cos(angle)) * (k @ k)


def collider(shape, dims, centre, rot, body, friction):
    """A collider on a static body whose frame is rotated by `rot` about its centre: x_local = rot^T (x - centre)."""
    rc = _capi.RigidCollider()
    rc.shape, rc.body = shape, body
    rc.dim[:] = list(dims) + [0.0] * (3 - len(dims))
    rc.restitution, rc.friction = 0.4, friction
    rc.R[:] = rot.T.reshape(-1).tolist(); rc.v2[:] = list(centre)
    half = {_capi.SHAPE_BOX: np.array(rc.dim[:]), _capi.SHAPE_SPHERE: np.full(3, dims[0])}[shape]
    half = np.abs(rot) @ half + TOL
    rc.aabb_min[:] = (np.asarray(centre) - half).tolist(); rc.aabb_max[:] = (np.asarray(centre) + half).tolist()
    return rc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=16)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    K = a.replicas
    hm = HostModel()
    hm.add_regular_triangle_model(32, 32, t=(-2.0, 3.0, -2.0), R=RX90, scale=(4.0, 4.0))
    hm.add_cloth_constraints(0, 4, dist_k=1.0e5)
    hm.add_bending_constraints(0, 3, 100.0)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x = np.asarray(hm.get("x"), np.float32).copy()
    hm.close()
    n = len(x)

    eng = _capi.Engine(0)
    eng.set_particles(x, mass)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=0.005, sub_steps=1, max_iter=5)
    eng.set_replicas(K)
    # replica r: a floor (top at y = 0), a box turned about a random axis and a sphere, each at its own random place under the cloth
    rng = np.random.default_rng(a.seed)
    rigid, body_x, boxes = [], np.zeros((K, 3, 3), np.float32), []
    for r in range(K):
        box_c = np.array([rng.uniform(-0.8, 0.8), rng.uniform(0.6, 1.2), rng.uniform(-0.8, 0.8)])
        box_half = rng.uniform(0.3, 0.6, 3)
        sph_c = np.array([rng.uniform(-1.5, 1.5), rng.uniform(0.3, 0.6), rng.uniform(-1.5, 1.5)])
        sph_r = rng.uniform(0.3, 0.6)
        rot = rotation(rng.normal(size=3), rng.uniform(0.0, 1.0))
        floor_c = np.array([0.0, -0.5, 0.0])
        rigid.append([collider(_capi.SHAPE_BOX, (10.0, 0.5, 10.0), floor_c, np.eye(3), 0, 0.3),
                      collider(_capi.SHAPE_BOX, box_half, box_c, rot, 1, 0.4),
                      collider(_capi.SHAPE_SPHERE, (sph_r,), sph_c, rotation((0, 1, 0), rng.uniform(0, 6.3)), 2, 0.2)])
        body_x[r] = [floor_c, box_c, sph_c]
        boxes.append(box_c)
    eng.set_replica_colliders([_capi.ParticleCollider(0, n, 0.5, 0.1)], rigid, body_x)
    eng.set_contact_params(tolerance=TOL, stiffness=100.0, max_iter_v=5)
    eng.record_contacts(1 << 20)
    eng.step(a.steps)
    eng.sync()
    xs = eng.get_attr(_capi.ATTR_X).reshape(K, n, 3)
    got, found = eng.contacts(1 << 20)
    per = np.bincount(np.array([c.particle // n for c in got], np.int64), minlength=K)
    above = []
    for r in range(K):
        near = np.argmin(np.linalg.norm(xs[r][:, [0, 2]] - boxes[r][[0, 2]], axis=1))  # the cloth particle right over the box
        above.append(bool(xs[r][near, 1] > boxes[r][1]))
        print("replica %3d: %4d contacts in the last step, cloth over its box at y = %.3f (box centre y = %.3f), lowest particle y = %.3f"
              % (r, per[r], xs[r][near, 1], boxes[r][1], xs[r][:, 1].min()))
    print("%d replicas, %d steps, %d contacts in the last step; every cloth above its obstacle: %s" % (K, a.steps, found, "yes" if all(above) else "no"))
    eng.close()
    return 0 if all(above) else 1


if __name__ == "__main__":
    sys.exit(main())
