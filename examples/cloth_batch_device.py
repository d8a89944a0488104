"""A batch of falling cloths driven from PyTorch without a host round trip (pbd_set_replicas + the device-memory state calls): K copies
of a 24 x 24 XPBD cloth, each dropped from its own height with its own sideways velocity.  Every step torch reads the positions on the GPU
(pbd_get_attr_device), marks the replicas whose centre fell below the floor height as done, and restarts those from their initial state by
masked device writes of x, v, oldX = x and lastX = x (pbd_set_attr_device) -- the loop an RL or Monte-Carlo driver runs.  Nothing crosses
to the host inside the loop.  The same loop written on the host calls (pbd_get_attr / pbd_set_attr of all K replicas) runs next to it and
must end in the same state bit for bit.  Needs a CUDA device and torch.

    python examples/cloth_batch_device.py [--replicas K] [--steps S] [--seed N]"""
import argparse
import os
import sys
import time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel

FLOOR = -1.0  # a replica whose centre falls below this height is done and starts again


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
    hm.close()
    eng = _capi.Engine(0)
    eng.set_particles(x, mass)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=0.005, sub_steps=1, max_iter=5, vel_method=1)
    eng.set_replicas(K)
    return eng, x, np.asarray(mass, np.float32)


def initial_state(x, mass, K, seed):
    """Replica r: the cloth at its own height, moving sideways at its own speed, nothing pinned (every cloth falls)."""
    rng = np.random.default_rng(seed)
    x0 = np.repeat(x[None], K, 0) + np.stack([np.array([0.0, rng.uniform(0.5, 3.0), 0.0], np.float32) for _ in range(K)])[:, None, :]
    v0 = np.repeat(rng.uniform(-1.0, 1.0, (K, 1, 3)).astype(np.float32), len(x), 1)
    m = np.repeat(np.where(mass == 0.0, np.float32(1.0), mass)[None], K, 0)
    return x0.astype(np.float32), v0, m


def run_device(K, steps, seed):
    eng, x, mass = cloth_engine(K)
    x0, v0, m = initial_state(x, mass, K, seed)
    dev = torch.device("cuda")
    X0, V0 = torch.from_numpy(x0.reshape(-1)).to(dev), torch.from_numpy(v0.reshape(-1)).to(dev)
    s = torch.cuda.current_stream().cuda_stream
    for attr, src in ((_capi.ATTR_X, X0), (_capi.ATTR_OLDX, X0), (_capi.ATTR_LASTX, X0), (_capi.ATTR_V, V0)):
        eng.set_attr_device(attr, src, stream=s)
    eng.set_masses_device(torch.from_numpy(m.reshape(-1)).to(dev), stream=s)
    xs = torch.empty(K * len(x) * 3, device=dev)
    restarts = torch.zeros(K, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        eng.step(1)
        eng.get_attr_device(_capi.ATTR_X, xs, stream=s)
        done = xs.view(K, -1, 3)[:, :, 1].mean(dim=1) < FLOOR
        restarts += done
        for attr, src in ((_capi.ATTR_X, X0), (_capi.ATTR_V, V0), (_capi.ATTR_OLDX, X0), (_capi.ATTR_LASTX, X0)):
            eng.set_attr_device(attr, src, replicas=done, stream=s)
    eng.get_attr_device(_capi.ATTR_X, xs, stream=s)
    v = eng.get_attr_device(_capi.ATTR_V, torch.empty_like(xs), stream=s)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    eng.close()
    return xs.cpu().numpy().reshape(K, -1, 3), v.cpu().numpy().reshape(K, -1, 3), restarts.cpu().numpy(), ms


def run_host(K, steps, seed):
    eng, x, mass = cloth_engine(K)
    x0, v0, m = initial_state(x, mass, K, seed)
    for attr, src in ((_capi.ATTR_X, x0), (_capi.ATTR_OLDX, x0), (_capi.ATTR_LASTX, x0), (_capi.ATTR_V, v0)):
        eng.set_attr(attr, src)
    eng.set_masses(m)
    restarts = np.zeros(K, np.int64)
    t0 = time.perf_counter()
    for _ in range(steps):
        eng.step(1)
        xs = eng.get_attr(_capi.ATTR_X)
        done = xs[:, :, 1].mean(axis=1) < FLOOR
        restarts += done
        if done.any():  # the host calls write every replica: read the other three arrays back, patch the done rows, write all four
            state = {a: eng.get_attr(a) for a in (_capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX)}
            state[_capi.ATTR_X] = xs
            for a, init in ((_capi.ATTR_X, x0), (_capi.ATTR_V, v0), (_capi.ATTR_OLDX, x0), (_capi.ATTR_LASTX, x0)):
                state[a][done] = init[done]
                eng.set_attr(a, state[a])
    x_end, v_end = eng.get_attr(_capi.ATTR_X), eng.get_attr(_capi.ATTR_V)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    eng.close()
    return x_end, v_end, restarts, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=64)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    xd, vd, rd, msd = run_device(a.replicas, a.steps, a.seed)
    xh, vh, rh, msh = run_host(a.replicas, a.steps, a.seed)
    same = np.array_equal(xd, xh) and np.array_equal(vd, vh) and np.array_equal(rd, rh)
    print("%d replicas, %d steps: %d restarts (%d replicas restarted at least once); device-memory loop %.3f ms/step, host loop %.3f ms/step "
          "(wall clock, small scene: launch-bound)" % (a.replicas, a.steps, rd.sum(), (rd > 0).sum(), msd, msh))
    print("final state of the device-memory loop equals the host-call loop bit for bit: %s" % ("yes" if same else "NO"))
    return 0 if same and rd.sum() > 0 else 1


if __name__ == "__main__":
    sys.exit(main())
