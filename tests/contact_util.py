"""Static colliders of the replica-batch contact tests (test_contacts_batch_host_shim.py on the host, test_gpu_batch_contacts.py on the GPU)
and of examples/cloth_collision_batch.py: analytic shapes in rotated frames over a particle model's footprint, as plain dicts that convert
to the engine's pbd_rigid_collider (to_capi) and to the kernel's RigidCollider (the host shim).

A body rotated by `rot` about its centre of mass c carries its collider in the frame x_local = rot^T (x_world - c): R = rot^T (row-major),
v1 = 0, v2 = c.  The bounding box is the world box of the rotated local box, extended by the contact tolerance."""
import numpy as np

SHAPES = ("box", "sphere", "torus", "cylinder", "hollow_sphere", "hollow_box")
BOX, SPHERE, TORUS, CYLINDER, HOLLOW_SPHERE, HOLLOW_BOX = range(6)
TOL = 0.05


def rotation(axis, angle):
    """Rotation matrix about `axis` (Rodrigues)."""
    a = np.asarray(axis, np.float64); a = a / np.linalg.norm(a)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.eye(3) + np.sin(angle) * k + (1.0 - np.cos(angle)) * (k @ k)


def half_extents(shape, dim, thickness):
    """The shape's local bounding half extents (dims as include/pbd_b200.h lists them)."""
    if shape == BOX:
        return np.array(dim[:3])
    if shape == SPHERE:
        return np.full(3, dim[0])
    if shape == TORUS:
        return np.array([dim[0] + dim[1], dim[1], dim[0] + dim[1]])
    if shape == CYLINDER:
        return np.array([dim[0], dim[1], dim[0]])
    if shape == HOLLOW_SPHERE:
        return np.full(3, dim[0] + thickness)
    return np.array(dim[:3]) + thickness  # HOLLOW_BOX


def collider(shape, dim, centre, rot=np.eye(3), thickness=0.0, invert=False, restitution=0.6, friction=0.2, body=0, tol=TOL):
    dim = list(dim) + [0.0] * (3 - len(dim))
    centre = np.asarray(centre, np.float64)
    half = np.abs(rot) @ half_extents(shape, dim, thickness) + tol
    return dict(shape=shape, body=body, dim=dim, thickness=thickness, invert=bool(invert), restitution=restitution, friction=friction,
                R=rot.T.reshape(-1).tolist(), v1=[0.0, 0.0, 0.0], v2=centre.tolist(), aabb_min=(centre - half).tolist(), aabb_max=(centre + half).tolist())


def empty_box(body=0):
    """A collider no particle passes: its bounding box is empty (aabb_min > aabb_max)."""
    return dict(shape=BOX, body=body, dim=[1.0, 1.0, 1.0], thickness=0.0, invert=False, restitution=0.5, friction=0.1,
                R=np.eye(3).reshape(-1).tolist(), v1=[0.0, 0.0, 0.0], v2=[0.0, 0.0, 0.0], aabb_min=[1.0, 1.0, 1.0], aabb_max=[-1.0, -1.0, -1.0])


def replica_scene(r, footprint, empty=False, shift=(0.0, 0.0, 0.0)):
    """Replica r's four colliders over `footprint` = (centre (3,), half extents (3,)) of the particle model, and the state of the bodies
    carrying them: (colliders, body_x (4, 3), body_v (4, 3), body_omega (4, 3)).  Three obstacles below the model, shapes
    SHAPES[(3r + j) % 6] (replicas 0 and 1 cover all six), each in its own random frame, with its own coefficients and body velocities;
    the fourth is an inverted sphere around the model (a bowl whose rim the model's corners touch) in odd replicas, an empty box in
    even ones.  empty: four empty boxes.  shift moves every body (a moving obstacle)."""
    rng = np.random.default_rng(7000 + r)
    c, h = np.asarray(footprint[0], np.float64), np.asarray(footprint[1], np.float64)
    size = float(min(h[0], h[2]))
    cols, xs = [], []
    for j in range(3):
        shape = (3 * r + j) % 6
        centre = c + np.array([rng.uniform(-0.5, 0.5) * h[0], -h[1] - rng.uniform(0.3, 0.6) * size, rng.uniform(-0.5, 0.5) * h[2]]) + shift
        rot = rotation(rng.normal(size=3), rng.uniform(0.2, 1.2))
        s = rng.uniform(0.25, 0.4) * size
        dim = {BOX: (s, 0.5 * s, s), SPHERE: (s,), TORUS: (s, 0.4 * s), CYLINDER: (0.6 * s, s), HOLLOW_SPHERE: (s,), HOLLOW_BOX: (s, 0.6 * s, s)}[shape]
        cols.append(collider(shape, dim, centre, rot, thickness=0.08 * s if shape in (HOLLOW_SPHERE, HOLLOW_BOX) else 0.0,
                             restitution=rng.uniform(0.2, 0.8), friction=rng.uniform(0.05, 0.4), body=j))
        xs.append(centre)
    if r % 2:
        centre = c + np.array([0.0, 0.3 * size, 0.0]) + shift
        radius = 0.97 * float(np.linalg.norm(h))
        cols.append(collider(SPHERE, (radius,), centre, rotation((0.0, 1.0, 0.0), 0.4), invert=True, restitution=0.3, friction=0.3, body=3))
        xs.append(centre)
    else:
        cols.append(empty_box(3))
        xs.append(c + shift)
    if empty:
        cols = [empty_box(j) for j in range(4)]
    body_v = rng.normal(0.0, 0.2, (4, 3))
    body_w = rng.normal(0.0, 0.8, (4, 3))
    return cols, np.asarray(xs, np.float32), body_v.astype(np.float32), body_w.astype(np.float32)


def batch_scene(K, footprint, empty=None, shift=None):
    """replica_scene of every replica: (K lists of colliders, body_x, body_v, body_omega as (K, 4, 3)).  empty: the replica given only
    empty boxes (default: the last one when K >= 3).  shift: (K, 3) per-replica body moves."""
    if empty is None:
        empty = K - 1 if K >= 3 else -1
    parts = [replica_scene(r, footprint, r == empty, (0.0, 0.0, 0.0) if shift is None else shift[r]) for r in range(K)]
    return [p[0] for p in parts], np.stack([p[1] for p in parts]), np.stack([p[2] for p in parts]), np.stack([p[3] for p in parts])


def footprint(x):
    """(centre, half extents) of a particle cloud."""
    lo, hi = np.min(x, axis=0), np.max(x, axis=0)
    return (lo + hi) / 2.0, (hi - lo) / 2.0


def to_capi(d):
    from positionbaseddynamics_b200 import _capi
    rc = _capi.RigidCollider()
    rc.shape, rc.body = d["shape"], d["body"]
    rc.dim[:] = d["dim"]; rc.thickness = d["thickness"]; rc.invert_sdf = int(d["invert"])
    rc.restitution, rc.friction = d["restitution"], d["friction"]
    rc.R[:] = d["R"]; rc.v1[:] = d["v1"]; rc.v2[:] = d["v2"]; rc.aabb_min[:] = d["aabb_min"]; rc.aabb_max[:] = d["aabb_max"]
    return rc
