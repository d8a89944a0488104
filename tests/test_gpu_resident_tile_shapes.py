"""The resident mode against the graph mode, bit for bit, in the shapes of the one-CTA-per-cluster regime that the cloth tests do not
reach: 2-, 3- and 4-body types in the shared-memory runs (Distance_XPBD, FEMTriangle, Dihedral, Volume_XPBD), tiles large enough to
use slots above 8,191, a whole scene in a single CTA, and the rigid-body joints in a single CTA."""
import os

import numpy as np
import pytest

import scenes

pytestmark = pytest.mark.gpu


def _run(mode, build, clusters=None, steps=3):
    from positionbaseddynamics_b200.model import HostModel
    from parity_util import perturb
    if clusters:
        os.environ["PBD_B200_CLUSTERS"] = clusters
    try:
        m = HostModel()
        build(m)
        perturb([m], 2.0e-3)
        m.time_step().set_mode(mode)
        m.step(steps)
        out = m.get("x").copy(), m.get("v").copy(), m.rigid_bodies().copy()
        m.close()
    finally:
        os.environ.pop("PBD_B200_CLUSTERS", None)
    assert np.isfinite(out[0]).all()
    return out


def _same(a, b):
    return all((u == v).all() for u, v in zip(a, b))


def _cloth_and_block(n_cloth, bar_dims):
    """FEMTriangle cloth with Dihedral bending, and a tet block with Distance_XPBD edges and Volume_XPBD tets, in one model."""
    def build(m):
        scenes.mixed(m, n_cloth=n_cloth, bar_dims=bar_dims, cloth_method=2, bending_method=1, solid_method=6, sub_steps=2, max_iter=4)
    return build


@pytest.mark.parametrize("clusters", ["2x1", "5x1"])
def test_tile_slots_match_graph_large_tiles(clusters):
    """150 x 150 cloth + 20 x 8 x 8 block = 23,780 particles: two tiles of about 11,900 particles (slots above 8,191, close to the
    ~13,800 a tile of 227 KB holds), or five smaller ones with more X items between them."""
    build = _cloth_and_block(150, (20, 8, 8))
    assert _same(_run(0, build), _run(1, build, clusters))


def test_tile_slots_match_graph_one_cta():
    """A scene small enough for one CTA (one cluster of one CTA: no X items, every item in shared memory)."""
    build = _cloth_and_block(40, (8, 4, 4))
    assert _same(_run(0, build), _run(1, build, "1x1"))


def test_joints_in_one_cta_match_graph():
    """Cloth + tet solid + the rigid coupling rig in one CTA: the joints index rigid bodies in global memory next to particles in
    shared memory."""
    def build(m):
        scenes.mixed(m, n_cloth=24, bar_dims=(7, 4, 4))
        scenes.coupling_rig(m, 24, 24)
    assert _same(_run(0, build), _run(1, build, "1x1"))
