"""The device image as the planner (csrc/host/image_plan.cpp) builds it, checked on the CPU: a small driver linked against the built
libpbd_b200.so (tests/host_shim/plan_image.cpp) plans scenes of tests/scenes.py, and every expectation here is derived from the
host model's constraints, groups and rest positions and from the raw plan -- slot map and tiles, buckets, index decoding, tile runs, and
the X-neighbour tables whose errors the resident kernel would turn into a hang rather than a failure."""
import numpy as np
import pytest

import scenes

from plan_util import AUTO, GRAPH, JACOBI, LAUNCH, RESIDENT, Scene, build_driver, check_plan, mode_of, plan, same_image


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_driver(tmp_path_factory.mktemp("plan"))


def cloth(n):
    return lambda m: scenes.cloth(m, n, n, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=1, max_iter=8)


def mixed(m):
    scenes.mixed(m, n_cloth=60, bar_dims=(12, 5, 5), cloth_method=2, bending_method=1, solid_method=6, sub_steps=2, max_iter=4)


def rig(m):
    scenes.mixed(m, n_cloth=24, bar_dims=(7, 4, 4))
    scenes.coupling_rig(m, 24, 24)


@pytest.mark.parametrize("build,shape", [(cloth(40), "graph"), (cloth(60), "1x1"), (cloth(100), "1x4"), (cloth(100), "7x1"),
                                         (cloth(300), "37x1"), (mixed, "5x1"), (rig, "1x1")],
                         ids=["cloth-graph", "cloth-1x1", "cloth-1x4", "cloth-7x1", "cloth-37x1", "mixed-5x1", "rig-1x1"])
def test_plan_invariants(driver, tmp_path, build, shape):
    sc = Scene.of(build)
    tiled = shape != "graph"
    G, C = (int(v) for v in shape.split("x")) if tiled else (0, 0)
    got = check_plan(sc, plan(driver, tmp_path, sc, RESIDENT if tiled else GRAPH, (G, C)), tiled)
    if tiled:
        assert got == (G, C)


def test_auto_mode_resolution(driver, tmp_path):
    """PBD_MODE_AUTO: the resident image for a cloth of at least 40,000 particles, the graph image for a smaller cloth and for rigid
    coupling.  The explicit modes get what they ask for; graph, launch and Jacobi share one image."""
    big = Scene.of(cloth(210))
    p = plan(driver, tmp_path, big, AUTO)
    assert mode_of(p) == RESIDENT and p["residentRefusal"] == b""
    check_plan(big, p, True)
    assert same_image(p, plan(driver, tmp_path, big, RESIDENT, tag="r"))
    graph = plan(driver, tmp_path, big, GRAPH, tag="g")
    check_plan(big, graph, False)
    for mode in (LAUNCH, JACOBI):
        q = plan(driver, tmp_path, big, mode, tag="m%d" % mode)
        assert mode_of(q) == mode and same_image(q, graph, "mode")
    for build in (cloth(40), rig):
        sc = Scene.of(build)
        q = plan(driver, tmp_path, sc, AUTO, tag="a")
        assert mode_of(q) == GRAPH and q["residentRefusal"] == b""
        assert same_image(q, plan(driver, tmp_path, sc, GRAPH, tag="g"))


def test_too_few_coresident_clusters(driver, tmp_path):
    """A device that keeps 8 clusters co-resident refuses 37 of them: an error under PBD_MODE_RESIDENT, the graph image under AUTO."""
    sc = Scene.of(cloth(210))
    assert sc.n >= 40000
    p = plan(driver, tmp_path, sc, RESIDENT, (37, 1), max_clusters=8, tag="r")
    assert p["error"] == b"resident mode: the device runs 8 clusters of 1 CTAs at a time, the scene needs 37 co-resident"
    q = plan(driver, tmp_path, sc, AUTO, (37, 1), max_clusters=8, tag="a")
    assert mode_of(q) == GRAPH and q["residentRefusal"] == p["error"]
    assert same_image(q, plan(driver, tmp_path, sc, GRAPH, (37, 1), max_clusters=8, tag="g"))


def test_auto_mode_without_coresident_clusters(driver, tmp_path):
    """A device that keeps no cluster co-resident: AUTO plans the graph image and says why."""
    sc = Scene.of(cloth(210))
    p = plan(driver, tmp_path, sc, AUTO, max_clusters=0, tag="a")
    assert mode_of(p) == GRAPH and b"the device runs 0 clusters" in p["residentRefusal"]
    assert same_image(p, plan(driver, tmp_path, sc, GRAPH, tag="g"))


def test_long_range_scene_is_refused(driver, tmp_path):
    """The random long-range distance constraints of test_gpu_resident_neighbours.py in 64 independent tiles: refused by the resident
    mode, planned in graph mode under AUTO."""
    from positionbaseddynamics_b200.model import first_fit_colouring
    rng = np.random.default_rng(7)
    side = 200
    g = np.stack(np.meshgrid(np.arange(side), np.arange(side), indexing="ij"), -1).reshape(-1, 2).astype(np.float32) * 0.05
    x = np.zeros((side * side, 3), np.float32); x[:, 0] = g[:, 0]; x[:, 2] = g[:, 1]
    pairs = rng.integers(0, side * side, size=(30000, 2))
    pairs = pairs[pairs[:, 0] != pairs[:, 1]].astype(np.uint32)
    rest = np.linalg.norm(x[pairs[:, 0]] - x[pairs[:, 1]], axis=1) * np.float32(0.9)
    N = len(pairs)
    ncol, col = first_fit_colouring(side * side, np.arange(N + 1, dtype=np.uint32) * 2, pairs.reshape(-1))
    ids = np.argsort(col, kind="stable")
    off = np.searchsorted(col[ids], np.arange(ncol + 1))
    bodies = np.zeros((N, 4), np.uint32); bodies[:, :2] = pairs
    params = np.zeros((N, 24), np.float32); params[:, 0] = rest; params[:, 1] = 1.0e4
    sc = Scene(side * side, 0, np.full(N, 1), bodies, params, off, ids, x)
    p = plan(driver, tmp_path, sc, RESIDENT, (64, 1))
    assert b"more than 32 other tiles" in p["error"]
    q = plan(driver, tmp_path, sc, AUTO, (64, 1), tag="a")
    assert mode_of(q) == GRAPH and b"more than 32 other tiles" in q["residentRefusal"]
    assert same_image(q, plan(driver, tmp_path, sc, GRAPH, (64, 1), tag="g"))


def test_modified_bending_q(driver, tmp_path):
    """A bending Q that is not of the rank-one form: refused by the resident mode, the literal 4x4 form (variant 1) in graph mode."""
    sc = Scene.of(lambda m: scenes.cloth(m, 20, 20, cloth_method=1, bending_method=2))
    ids, b, prm = sc.store[3]
    prm[5, 1:17] += np.eye(4, dtype=np.float32).reshape(-1) * 0.5
    assert b"user-modified Q" in plan(driver, tmp_path, sc, RESIDENT, (1, 1))["error"]
    p = plan(driver, tmp_path, sc, GRAPH)
    assert int(np.frombuffer(p["variant3"], np.int32)[0]) == 1
    check_plan(sc, p, False)


def test_modified_bending_q_under_auto(driver, tmp_path):
    """The same in a cloth big enough for AUTO to try the resident mode: refused, and planned in graph mode instead."""
    sc = Scene.of(lambda m: scenes.cloth(m, 200, 200, cloth_method=1, bending_method=2))
    assert sc.n >= 40000
    ids, b, prm = sc.store[3]
    prm[5, 1:17] += np.eye(4, dtype=np.float32).reshape(-1) * 0.5
    p = plan(driver, tmp_path, sc, AUTO)
    assert mode_of(p) == GRAPH and b"user-modified Q" in p["residentRefusal"]
    assert int(np.frombuffer(p["variant3"], np.int32)[0]) == 1
    check_plan(sc, p, False)


def test_plan_is_deterministic(driver, tmp_path):
    """Byte-identical plans with one host thread and with four (each in a process of its own: the thread count is read once)."""
    sc = Scene.of(cloth(300))
    one = plan(driver, tmp_path, sc, RESIDENT, (37, 1), threads=1, tag="t1")
    four = plan(driver, tmp_path, sc, RESIDENT, (37, 1), threads=4, tag="t4")
    assert one["error"] == b"" and one["raw"] == four["raw"]


def test_joints_in_one_cluster_only(driver, tmp_path):
    """The rigid-body cases of tests/rigid_cases.py on rest positions in a random order.  Independent CTAs (a forced G > 1) are refused:
    a joint's bodies are stepped by CTA 0 alone.  One cluster of four is admitted: every BallJoint runs in tile 0, every particle joint in
    the tile of its particle, so the joints of one body run in several CTAs, ordered by the cluster barrier."""
    import rigid_cases as rc
    from plan_util import u32
    m = rc.make_model(3, 8)
    sc = Scene(m.n, m.nb, m.types, m.bodies, m.params, m.off, m.ids, rc.tile_x0(m, np.random.default_rng(5)))
    p = plan(driver, tmp_path, sc, RESIDENT, (4, 1), tag="g4")
    assert p["error"] == b"resident mode: rigid-body coupling is supported for scenes that fit one cluster (use PBD_MODE_GRAPH)"
    p = plan(driver, tmp_path, sc, RESIDENT, (1, 4), tag="c4")
    assert check_plan(sc, p, True) == (1, 4)
    buckets = np.frombuffer(p["buckets"], np.int32).reshape(-1, 4)
    tile_off = u32(p, "tileOff").astype(np.int64).reshape(len(buckets), 9)
    tstart = u32(p, "tileStart").astype(np.int64)
    ptile = np.searchsorted(tstart, u32(p, "slot"), "right") - 1
    for t in (rc.BJ, rc.RBP):
        ids, b, _ = sc.store[t]
        b = b[np.searchsorted(ids, u32(p, "order%d" % t))]  # device order
        ex = np.full(len(ids), -1)
        for bi in np.nonzero(buckets[:, 0] == t)[0]:
            lab = np.repeat(np.arange(8), np.diff(tile_off[bi]))
            assert (lab % 2 == 1).all()  # shared-memory items only
            ex[buckets[bi, 1]:buckets[bi, 1] + buckets[bi, 2]] = lab // 2
        if t == rc.BJ:
            assert (ex == 0).all()
        else:
            assert np.array_equal(ex, ptile[b[:, 1]]) and set(ex) == {0, 1, 2, 3}


def test_free_bodies_beyond_the_block_are_planned_as_intended(driver, tmp_path):
    """The 210 x 210 cloth and 700 free bodies of tests/test_gpu_rigid_answers.py: MODE_AUTO plans one resident cluster whose CTAs have
    fewer threads than there are bodies, and the forced independent CTAs give part of every CTA to X threads, so fewer still step bodies
    in CTA 0.  Both shapes the GPU tests run are admitted as intended."""
    from plan_util import u32
    from test_gpu_rigid_answers import INDEPENDENT_CTAS, cloth_and_free_bodies
    m, (x, _, (types, bodies, params, off, ids)) = cloth_and_free_bodies()
    sc = Scene(len(x), m.nb, types, bodies, params, off, ids, x)
    shapes = {"auto": (0, 0), "forced": tuple(int(v) for v in INDEPENDENT_CTAS.split("x"))}
    res = {}
    for name, shape in shapes.items():
        p = plan(driver, tmp_path, sc, AUTO if name == "auto" else RESIDENT, shape, tag=name)
        assert mode_of(p) == RESIDENT and p["residentRefusal"] == b""
        G, C = check_plan(sc, p, True)
        threads, xthreads = (int(v) for v in u32(p, "res")[2:4])
        res[name] = (G, C, threads, xthreads)
        print("%s: %d x %d, %d threads, %d for X items; %d bodies" % (name, G, C, threads, xthreads, m.nb))
        assert threads - xthreads < m.nb
    assert res["auto"][0] == 1 and res["auto"][3] == 0
    assert res["forced"][:2] == shapes["forced"] and res["forced"][3] > 0
