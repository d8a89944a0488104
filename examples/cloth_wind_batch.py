"""A batch of cloths in the wind, the wind force computed by PyTorch on the GPU every step (pbd_set_external_forces_device): K copies of a
32 x 32 XPBD cloth pinned at two corners, each replica in its own wind.  Every step torch reads the positions on the GPU
(pbd_get_attr_device), computes each triangle's pressure force c (n . w) n A from its normal n, area A and the replica's wind w, and hands
every particle the sum over its triangles, a third each, as its external force.  The wind turns slowly, replica by replica.  Nothing
crosses to the host inside the loop.  The same loop through the host calls (pbd_get_attr / pbd_set_external_forces) runs next to it and
must end in the same state bit for bit.  Needs a CUDA device and torch.

    python examples/cloth_wind_batch.py [--replicas K] [--steps S] [--check]"""
import argparse
import os
import sys
import time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel

N = 32
DRAG = 500.0  # N s^2 / m^4: pressure per (m/s)^2 of wind along the normal, on particles of 1 kg


def cloth_engine(K):
    hm = HostModel()
    hm.add_regular_triangle_model(N, N, t=(0, 1, 0), R=np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], float), scale=(2.0, 2.0))
    hm.set_mass(0, 0.0)
    hm.set_mass(N - 1, 0.0)
    hm.add_cloth_constraints(0, 4, dist_k=1.0e5)
    hm.add_bending_constraints(0, 3, 100.0)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    off, ids = hm.groups()
    mass, _ = hm.masses()
    x = np.asarray(hm.get("x"), np.float32).copy()
    faces = np.asarray(hm.tri_faces(0), np.int64).reshape(-1, 3).copy()
    hm.close()
    eng = _capi.Engine(0)
    eng.set_particles(x, mass)
    eng.add_flat(types, bodies, params)
    eng.set_groups(off, ids)
    eng.set_params(dt=0.005, sub_steps=2, max_iter=5)
    eng.set_replicas(K)
    return eng, len(x), faces


class Wind:
    """Per-replica wind and the pressure force on every particle, as fixed-order torch operations on the GPU (no atomics), so that both
    loops compute the same bits from the same positions."""
    def __init__(self, K, n, faces, dev):
        self.K, self.n = K, n
        self.faces = torch.from_numpy(faces).to(dev)
        incident = [[] for _ in range(n)]
        for t, f in enumerate(faces):
            for i in f:
                incident[i].append(t)
        width = max(len(i) for i in incident)
        table = np.full((n, width), len(faces), np.int64)  # padded with a triangle of zero force
        for i, ts in enumerate(incident):
            table[i, :len(ts)] = ts
        self.incident = torch.from_numpy(table).to(dev)
        phase = torch.arange(K, device=dev, dtype=torch.float32)
        self.speed = 4.0 + 0.5 * (phase % 5)
        self.heading = 0.7 * phase

    def forces(self, x, step):
        """(K*n*3,) float32 forces from positions x (K*n*3,) on the GPU."""
        p = x.view(self.K, self.n, 3)
        a, b, c = p[:, self.faces[:, 0]], p[:, self.faces[:, 1]], p[:, self.faces[:, 2]]
        area_n = 0.5 * torch.cross(b - a, c - a, dim=2)                      # normal times area
        unit = area_n / torch.linalg.norm(area_n, dim=2, keepdim=True).clamp_min(1e-12)
        ang = self.heading + 0.01 * step
        w = torch.stack([torch.cos(ang), 0.5 * torch.sin(3.0 * ang), torch.sin(ang)], 1) * self.speed[:, None]
        un = (unit * w[:, None, :]).sum(dim=2, keepdim=True)                # n . w
        f_tri = (DRAG / 3.0) * un * un.abs() * area_n                        # a third to each corner
        f_tri = torch.cat([f_tri, torch.zeros_like(f_tri[:, :1])], dim=1)
        return f_tri[:, self.incident].sum(dim=2).reshape(-1).contiguous()


def run_device(K, steps):
    eng, n, faces = cloth_engine(K)
    dev = torch.device("cuda")
    wind = Wind(K, n, faces, dev)
    s = torch.cuda.current_stream().cuda_stream
    xs = torch.empty(K * n * 3, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(steps):
        eng.get_attr_device(_capi.ATTR_X, xs, stream=s)
        eng.set_external_forces_device(wind.forces(xs, k), stream=s)
        eng.step(1)
    eng.get_attr_device(_capi.ATTR_X, xs, stream=s)
    v = eng.get_attr_device(_capi.ATTR_V, torch.empty_like(xs), stream=s)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    eng.close()
    return xs.cpu().numpy().reshape(K, n, 3), v.cpu().numpy().reshape(K, n, 3), ms


def run_host(K, steps):
    eng, n, faces = cloth_engine(K)
    dev = torch.device("cuda")
    wind = Wind(K, n, faces, dev)
    t0 = time.perf_counter()
    for k in range(steps):
        x = torch.from_numpy(eng.get_attr(_capi.ATTR_X).reshape(-1)).to(dev)
        eng.set_external_forces(wind.forces(x, k).cpu().numpy().reshape(K, n, 3))
        eng.step(1)
    x_end, v_end = eng.get_attr(_capi.ATTR_X), eng.get_attr(_capi.ATTR_V)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    eng.close()
    return x_end, v_end, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=64)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--check", action="store_true", help="also require that the wind moved the cloths apart")
    a = ap.parse_args()
    xd, vd, msd = run_device(a.replicas, a.steps)
    xh, vh, msh = run_host(a.replicas, a.steps)
    same = np.array_equal(xd, xh) and np.array_equal(vd, vh)
    spread = float(np.abs(xd - xd[:1]).max())
    print("%d replicas, %d steps: the cloths end up to %.3f m apart; device-memory loop %.3f ms/step, host loop %.3f ms/step (wall clock)"
          % (a.replicas, a.steps, spread, msd, msh))
    print("final state of the device-memory loop equals the host-call loop bit for bit: %s" % ("yes" if same else "NO"))
    ok = same and np.isfinite(xd).all() and (not a.check or spread > 1e-2)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
