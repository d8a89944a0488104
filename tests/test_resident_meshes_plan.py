"""The resident plans of the mesh scenes of tests/resident_meshes.py, on the CPU: every (scene, size, regime) is admitted with the type
mask meant for it and the forced G x C, holds every invariant of plan_util.check_plan, and gives every particle type of the scene items of
the regime's kind -- X items with independent CTAs, DSMEM items in a cluster of several CTAs -- so that the GPU test compares the kernel
with the launch mode exactly where a wrong order across tiles would show.  Also the planner's refusal of resident batches whose
per-replica rows the kernel's 32-bit offsets cannot address."""
import numpy as np
import pytest

import resident_meshes as rm
from plan_util import AUTO, GRAPH, RESIDENT, Scene, build_driver, check_plan, item_kinds_by_type, mode_of, plan, same_image, u32

JOINTS = (rm.BALLJOINT, rm.RB_PARTICLE_BALLJOINT)


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_driver(tmp_path_factory.mktemp("plan"))


_scenes = {}


def scene(name, size, rig):
    key = (name, size, rig)
    if key not in _scenes:
        _scenes[key] = Scene.of(rm.builder(name, size, rig))
    return _scenes[key]


@pytest.mark.parametrize("size", rm.SIZES)
@pytest.mark.parametrize("name", sorted(rm.SCENES))
def test_mesh_scene_plans(driver, tmp_path, name, size):
    mask = rm.SCENES[name][1]
    for regime in rm.regimes(size):
        rig = rm.has_rig(name, regime)
        sc = scene(name, size, rig)
        present = [t for t in range(15) if len(sc.store[t][0])]
        assert sum(1 << t for t in present) & ~mask == 0
        p = plan(driver, tmp_path, sc, RESIDENT, rm.shape(regime), tag=regime)
        assert p["error"] == b"", (name, size, regime, p["error"])
        G, C = check_plan(sc, p, True)
        res = u32(p, "res")
        assert int(res[4]) == mask, (name, size, regime, hex(int(res[4])))
        if regime != "default":
            assert (G, C) == rm.shape(regime), (name, size, regime, G, C)
        else:
            assert G == 1, (name, size, G, C)  # one cluster: every scene here fits 16 CTAs
        kinds = item_kinds_by_type(sc, p)
        print("%s %s %s: %d particles, %d x %d, mask %#x, per type (X, DSMEM, own tile) %s" % (name, size, regime, sc.n, G, C, mask, kinds))
        for t in present:
            if t in JOINTS:
                continue  # rigid-body indices: a BallJoint runs in tile 0, a particle joint in its particle's tile
            nx, nd, _ = kinds[t]
            if G > 1:
                assert nx > 0, (name, size, regime, "type %d has no X items" % t)
            elif C > 1:
                assert nd > 0, (name, size, regime, "type %d has no DSMEM items" % t)
        if size == "large" and regime == "2x1":
            tstart = u32(p, "tileStart").astype(np.int64)
            assert np.diff(tstart).min() > 8192 and int(res[5]) - np.diff(tstart).max() < 2048, (np.diff(tstart), int(res[5]))


def _distance_scene(n, count, rng):
    """`count` Distance constraints between random pairs of n particles on a line, coloured first-fit."""
    from positionbaseddynamics_b200.model import first_fit_colouring
    x = np.zeros((n, 3), np.float32); x[:, 0] = np.arange(n) * 0.01
    i = rng.integers(0, n, count)
    pairs = np.stack([i, (i + 1 + rng.integers(0, 64, count)) % n], 1).astype(np.uint32)
    ncol, col = first_fit_colouring(n, np.arange(count + 1, dtype=np.uint32) * 2, pairs.reshape(-1))
    ids = np.argsort(col, kind="stable")
    off = np.searchsorted(col[ids], np.arange(ncol + 1))
    bodies = np.zeros((count, 4), np.uint32); bodies[:, :2] = pairs
    params = np.zeros((count, 24), np.float32); params[:, 0] = 0.01; params[:, 1] = 1.0
    return Scene(n, 0, np.zeros(count, np.int64), bodies, params, off, ids, x)


@pytest.mark.parametrize("replicas,count", [(32768, 131072), (65535, 65537)], ids=["2^32", "2^32-1"])
def test_replica_offsets_beyond_32_bits_are_refused(driver, tmp_path, replicas, count):
    """A resident batch with per-replica rest shapes or materials addresses replica r's rows of a type at r x count + i in 32 bits: at K x
    count = 2^32 the resident mode refuses it and AUTO plans the graph image; at 2^32 - 1, and without the per-replica tables, it is
    admitted."""
    n = (1 << 31) // replicas - 1  # the largest replica a batch of K admits: K x n < 2^31
    sc = _distance_scene(n, count, np.random.default_rng(9))
    over = replicas * count >= 1 << 32
    p = plan(driver, tmp_path, sc, RESIDENT, replicas=replicas, rest_tables=True, tag="r")
    if over:
        assert p["error"] == (b"resident mode: %d replicas of %d constraints of type 0 with per-replica rest shapes or materials exceed the "
                              b"2^32 rows the resident kernel addresses (use PBD_MODE_GRAPH)" % (replicas, count))
        q = plan(driver, tmp_path, sc, AUTO, replicas=replicas, rest_tables=True, tag="a")
        assert mode_of(q) == GRAPH and q["residentRefusal"] == p["error"]
        assert same_image(q, plan(driver, tmp_path, sc, GRAPH, replicas=replicas, rest_tables=True, tag="g"))
    else:
        assert mode_of(p) == RESIDENT
        check_plan(sc, p, True)
    shared = plan(driver, tmp_path, sc, RESIDENT, replicas=replicas, rest_tables=False, tag="s")
    assert mode_of(shared) == RESIDENT
