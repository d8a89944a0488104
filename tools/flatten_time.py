"""Development aid: time to the first step of cfg2 from nothing (C++ host model -> engine), one fresh model per execution mode.
Run on the GPU box: [PBD_B200_VERBOSE=1] python tools/flatten_time.py [size]"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, scenes
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
# one-time costs of the process, outside the timings: library load, CUDA context, lazy loading of the kernels (a 64 x 64 cloth in every mode)
import torch; torch.cuda.init(); torch.zeros(1, device="cuda")
for mode in (_capi.MODE_RESIDENT, _capi.MODE_GRAPH):
    w = HostModel(); scenes.cfg2(w, 64, 2); w.time_step(device=0).set_mode(mode); w.step(2); w.time_step().sync(); w.close()
for mode, name in ((_capi.MODE_RESIDENT, "resident"), (_capi.MODE_GRAPH, "graph"), (_capi.MODE_AUTO, "auto")):
    t0 = time.perf_counter(); hm = HostModel()
    hm.add_regular_triangle_model(n, n, t=(0, 1, 0), R=scenes.RX90, scale=(10, 10)); t1 = time.perf_counter()
    hm.set_mass(0, 0.0); hm.set_mass(n - 1, 0.0)
    hm.add_cloth_constraints(0, 4, dist_k=1e5); t2 = time.perf_counter()
    hm.add_bending_constraints(0, 3, 100.0); t3 = time.perf_counter()
    hm.set_params(dt=0.005, sub_steps=1, max_iter=20)
    ts = hm.time_step(device=0); ts.set_mode(mode); t4 = time.perf_counter()
    hm.step(1); ts.sync(); t5 = time.perf_counter(); hm.step(1); ts.sync(); t6 = time.perf_counter()
    print("%-8s: mesh %.3f | distance %.3f | bending %.3f | engine %.3f | first step (upload + colouring + flatten + launch) %.3f  => time to first step %.3f s; second step %.4f s"
          % (name, t1 - t0, t2 - t1, t3 - t2, t4 - t3, t5 - t4, t5 - t0, t6 - t5))
    hm.close()
