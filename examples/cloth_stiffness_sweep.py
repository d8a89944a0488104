"""A stiffness sweep of the cloth of cloth_model.py in one replica batch: K copies of the 50 x 50 XPBD cloth, each with its own
Distance_XPBD stiffness and, for show, its own gravity tilt, advanced together by one engine (Engine.set_replicas +
set_replica_materials / set_replica_gravity).  Headless: prints how far each cloth's free edge has dropped.  Needs a CUDA device."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel
from cloth_model import nCols, nRows, width, height, rotation_matrix


def main(K=12, steps=200):
    hm = HostModel()
    hm.add_regular_triangle_model(nCols, nRows, t=(0, 0, 0), R=rotation_matrix(np.pi * 0.5, [1.0, 0.0, 0.0]), scale=(width, height))
    hm.set_mass(0, 0.0); hm.set_mass(nRows - 1, 0.0)
    hm.add_cloth_constraints(0, 4, dist_k=1.0e5)   # Distance_XPBD; the sweep replaces this stiffness per replica
    hm.add_bending_constraints(0, 3, 50.0)
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    eng = _capi.Engine(0)
    eng.set_particles(hm.get("x"), hm.masses()[0])
    eng.add_flat(types, bodies, params)
    eng.set_groups(*hm.groups())
    eng.set_params(dt=0.005, sub_steps=3, max_iter=5)
    eng.set_replicas(K)
    stiffness = np.logspace(2, 6, K, dtype=np.float32)
    eng.set_replica_materials(_capi.DISTANCE_XPBD, stiffness[:, None])
    eng.set_replica_gravity(np.stack([(0.5 * np.sin(r), -9.81, 0.0) for r in range(K)]))
    eng.step(steps); eng.sync()
    x = eng.get_attr(_capi.ATTR_X)
    for r in range(K):
        print("stiffness %9.3g: lowest particle at y = %.3f" % (stiffness[r], x[r, :, 1].min()))
    eng.close(); hm.close()
    return x


if __name__ == "__main__":
    main()
