"""A rest-shape sweep of the cloth of cloth_model.py in one replica batch: K copies of the 50 x 50 XPBD cloth, all hanging from the same
two corners, whose rest shapes are the cloth scaled in its plane from 0.8 (pre-stretched: the rest state is smaller than the hung cloth) to
1.2 (slack), advanced together by one engine (Engine.set_replicas + set_replica_rest_positions: every replica's rest lengths and bending Q
are derived on the GPU from its own rest shape).  Headless: prints each cloth's sag and mean edge strain.  Needs a CUDA device."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from positionbaseddynamics_b200 import _capi
from positionbaseddynamics_b200.model import HostModel
from cloth_model import nCols, nRows, width, height, rotation_matrix


def main(K=9, steps=300):
    hm = HostModel()
    hm.add_regular_triangle_model(nCols, nRows, t=(0, 0, 0), R=rotation_matrix(np.pi * 0.5, [1.0, 0.0, 0.0]), scale=(width, height))
    hm.set_mass(0, 0.0); hm.set_mass(nRows - 1, 0.0)
    hm.add_cloth_constraints(0, 4, dist_k=1.0e5)   # Distance_XPBD
    hm.add_bending_constraints(0, 3, 50.0)         # IsometricBending_XPBD
    hm.init_groups()
    types, bodies, params, _ = hm.constraints()
    x0 = np.asarray(hm.get("x0"), np.float32)
    eng = _capi.Engine(0)
    eng.set_particles(hm.get("x"), hm.masses()[0])
    eng.add_flat(types, bodies, params)
    eng.set_groups(*hm.groups())
    eng.set_params(dt=0.005, sub_steps=3, max_iter=5)
    eng.set_replicas(K)
    scale = np.linspace(0.8, 1.2, K)
    centre = x0.mean(axis=0)
    rest = np.stack([centre + (x0 - centre) * s for s in scale]).astype(np.float32)  # the cloth lies in the x-z plane: a uniform scale keeps it there
    eng.set_replica_rest_positions(rest)
    eng.step(steps); eng.sync()
    x = eng.get_attr(_capi.ATTR_X)
    edges = np.asarray(bodies)[np.asarray(types) == _capi.DISTANCE_XPBD][:, :2]
    rest_len = eng.replica_geometry(_capi.DISTANCE_XPBD)[:, :, 0]  # (K, edges), the constraints in the order they were added
    for r in range(K):
        length = np.linalg.norm(x[r, edges[:, 0]] - x[r, edges[:, 1]], axis=1)
        strain = np.mean(length / rest_len[r] - 1.0)
        print("rest scale %.2f: sag %.3f, mean edge strain %+.4f" % (scale[r], x0[:, 1].max() - x[r, :, 1].min(), strain))
    eng.close(); hm.close()
    return x


if __name__ == "__main__":
    main()
