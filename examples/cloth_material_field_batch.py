"""A batch of falling cloths, each with its own random stiffness field (pbd_set_replica_constraint_materials): K copies of a 24 x 24 XPBD
cloth whose every stretch edge has its own stiffness, drawn per replica by torch on the GPU (log-uniform over 1e2 .. 1e5).  Every step torch
reads the positions on the GPU, marks the replicas whose centre fell below the floor height as done, and restarts those from their initial
state with a freshly drawn field -- masked device writes of the state (pbd_set_attr_device) and of the field
(pbd_set_replica_constraint_materials_device), the loop of a driver that randomises materials per episode.  Nothing crosses to the host
inside the loop.  The same loop written on the host calls (every replica's state and field through pbd_get_attr / pbd_set_attr and
pbd_set_replica_constraint_materials) runs next to it and must end in the same state bit for bit.  Needs a CUDA device and torch.

    python examples/cloth_material_field_batch.py [--replicas K] [--steps S] [--seed N]"""
import argparse
import os
import sys
import time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel

FLOOR = -1.0  # a replica whose centre falls below this height is done and starts again with a new field
STATE = (_capi.ATTR_X, _capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX)


def cloth_engine(K):
    hm = HostModel()
    hm.add_regular_triangle_model(24, 24, scale=(2.0, 2.0))
    hm.add_cloth_constraints(0, 4, dist_k=1.0e5)
    hm.add_bending_constraints(0, 3, 100.0)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x = np.asarray(hm.get("x"), np.float32).copy()
    edges = int((np.asarray(types) == _capi.DISTANCE_XPBD).sum())
    hm.close()
    eng = _capi.Engine(0)
    eng.set_particles(x, mass)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=0.005, sub_steps=1, max_iter=5, vel_method=1)
    eng.set_replicas(K)
    return eng, x, np.asarray(mass, np.float32), edges


def initial_state(x, mass, K, seed):
    """Replica r: the cloth at its own height, moving sideways at its own speed, nothing pinned (every cloth falls)."""
    rng = np.random.default_rng(seed)
    x0 = np.repeat(x[None], K, 0) + np.stack([np.array([0.0, rng.uniform(0.5, 3.0), 0.0], np.float32) for _ in range(K)])[:, None, :]
    v0 = np.repeat(rng.uniform(-1.0, 1.0, (K, 1, 3)).astype(np.float32), len(x), 1)
    m = np.repeat(np.where(mass == 0.0, np.float32(1.0), mass)[None], K, 0)
    return x0.astype(np.float32), v0, m


class Fields:
    """Stiffness fields drawn by torch on the GPU: (K, edges, 1) per draw, log-uniform over 1e2 .. 1e5.  Both loops draw once per step
    from the same seed, so they see the same sequence of fields."""
    def __init__(self, K, edges, seed):
        self.shape = (K, edges, 1)
        self.gen = torch.Generator(device="cuda")
        self.gen.manual_seed(seed)

    def draw(self):
        u = torch.rand(self.shape, generator=self.gen, device="cuda")
        return torch.pow(10.0, 2.0 + 3.0 * u).contiguous()


def run_device(K, steps, seed):
    eng, x, mass, edges = cloth_engine(K)
    x0, v0, m = initial_state(x, mass, K, seed)
    dev = torch.device("cuda")
    X0, V0 = torch.from_numpy(x0.reshape(-1)).to(dev), torch.from_numpy(v0.reshape(-1)).to(dev)
    s = torch.cuda.current_stream().cuda_stream
    for attr, src in ((_capi.ATTR_X, X0), (_capi.ATTR_OLDX, X0), (_capi.ATTR_LASTX, X0), (_capi.ATTR_V, V0)):
        eng.set_attr_device(attr, src, stream=s)
    eng.set_masses_device(torch.from_numpy(m.reshape(-1)).to(dev), stream=s)
    fields = Fields(K, edges, seed)
    eng.set_replica_constraint_materials_device(_capi.DISTANCE_XPBD, fields.draw(), stream=s)
    xs = torch.empty(K * len(x) * 3, device=dev)
    restarts = torch.zeros(K, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        eng.step(1)
        eng.get_attr_device(_capi.ATTR_X, xs, stream=s)
        done = xs.view(K, -1, 3)[:, :, 1].mean(dim=1) < FLOOR
        restarts += done
        eng.set_replica_constraint_materials_device(_capi.DISTANCE_XPBD, fields.draw(), replicas=done, stream=s)
        for attr, src in ((_capi.ATTR_X, X0), (_capi.ATTR_V, V0), (_capi.ATTR_OLDX, X0), (_capi.ATTR_LASTX, X0)):
            eng.set_attr_device(attr, src, replicas=done, stream=s)
    eng.get_attr_device(_capi.ATTR_X, xs, stream=s)
    v = eng.get_attr_device(_capi.ATTR_V, torch.empty_like(xs), stream=s)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    k_end = eng.get_replica_materials(_capi.DISTANCE_XPBD)
    eng.close()
    return xs.cpu().numpy().reshape(K, -1, 3), v.cpu().numpy().reshape(K, -1, 3), k_end, restarts.cpu().numpy(), ms


def run_host(K, steps, seed):
    eng, x, mass, edges = cloth_engine(K)
    x0, v0, m = initial_state(x, mass, K, seed)
    for attr, src in ((_capi.ATTR_X, x0), (_capi.ATTR_OLDX, x0), (_capi.ATTR_LASTX, x0), (_capi.ATTR_V, v0)):
        eng.set_attr(attr, src)
    eng.set_masses(m)
    fields = Fields(K, edges, seed)
    field = fields.draw().cpu().numpy()
    eng.set_replica_constraint_materials(_capi.DISTANCE_XPBD, field)
    restarts = np.zeros(K, np.int64)
    t0 = time.perf_counter()
    for _ in range(steps):
        eng.step(1)
        xs = eng.get_attr(_capi.ATTR_X)
        done = xs[:, :, 1].mean(axis=1) < FLOOR
        restarts += done
        fresh = fields.draw().cpu().numpy()
        if done.any():  # the host calls write every replica: patch the done rows of the field and of all four state arrays
            field[done] = fresh[done]
            eng.set_replica_constraint_materials(_capi.DISTANCE_XPBD, field)
            state = {a: eng.get_attr(a) for a in (_capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX)}
            state[_capi.ATTR_X] = xs
            for a, init in ((_capi.ATTR_X, x0), (_capi.ATTR_V, v0), (_capi.ATTR_OLDX, x0), (_capi.ATTR_LASTX, x0)):
                state[a][done] = init[done]
                eng.set_attr(a, state[a])
    x_end, v_end = eng.get_attr(_capi.ATTR_X), eng.get_attr(_capi.ATTR_V)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    eng.close()
    return x_end, v_end, field, restarts, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=64)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    xd, vd, kd, rd, msd = run_device(a.replicas, a.steps, a.seed)
    xh, vh, kh, rh, msh = run_host(a.replicas, a.steps, a.seed)
    same = np.array_equal(xd, xh) and np.array_equal(vd, vh) and np.array_equal(kd, kh) and np.array_equal(rd, rh)
    print("%d replicas, %d steps: %d restarts with a new stiffness field (%d replicas restarted at least once); device-memory loop %.3f ms/step, "
          "host loop %.3f ms/step (wall clock, small scene: launch-bound)" % (a.replicas, a.steps, rd.sum(), (rd > 0).sum(), msd, msh))
    print("final state and fields of the device-memory loop equal the host-call loop bit for bit: %s" % ("yes" if same else "NO"))
    return 0 if same and rd.sum() > 0 else 1


if __name__ == "__main__":
    sys.exit(main())
