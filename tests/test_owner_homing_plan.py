"""Homing by constraint owner (csrc/host/image_plan.cpp: home_by_owner), checked on the CPU for independent CTAs (G > 1, C = 1).  The
tiles are the recursive coordinate bisection of the particles' rest positions; a constraint's owner is the tile that holds most of its
particles (ties: the lowest) and runs it.  A particle stays in its tile's shared memory when every constraint through it is owned there,
else it is global-homed in its tile.  Every expectation is re-derived here from the scene's rest positions and constraints, and every
plan also holds plan_util.check_plan (neighbour sets and masks included)."""
import numpy as np
import pytest

import resident_meshes as rm
import scenes
from plan_util import NB, NUM_TYPES, RESIDENT, Scene, build_driver, check_plan, indices, is_rb, item_kinds, item_kinds_by_type, plan, u32


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_driver(tmp_path_factory.mktemp("plan"))


def bisect(pts, parts):
    """The planner's recursive coordinate bisection of the float32 points `pts` into `parts` parts of equal counts: the longest axis of the
    bounding box (ties: the lower axis), split at the count's share of the left half, points ordered by coordinate, then by index."""
    lab = np.zeros(len(pts), np.int64)

    def rec(ix, t0, nt):
        if nt == 1:
            lab[ix] = t0
            return
        q = pts[ix]
        ext = q.max(0) - q.min(0)
        ax = 0
        for k in (1, 2):
            if ext[k] > ext[ax]:
                ax = k
        ntl = nt // 2
        mid = len(ix) * ntl // nt
        o = ix[np.lexsort((ix, q[:, ax]))]
        rec(o[:mid], t0, ntl)
        rec(o[mid:], t0 + ntl, nt - ntl)

    rec(np.arange(len(pts)), 0, parts)
    return lab


def owners(sc, region):
    """Owner tile of every constraint, by type in the scene's row order: the tile of most of its particles, ties to the lowest."""
    out = []
    for t in range(NUM_TYPES):
        b = sc.store[t][1]
        pk = [k for k in range(NB[t]) if not is_rb(t, k)]
        if not len(b) or not pk:
            out.append(np.zeros(len(b), np.int64)); continue
        reg = region[b[:, pk]]
        cnt = (reg[:, :, None] == reg[:, None, :]).sum(2)
        score = cnt * (1 << 20) - reg  # most particles first, then the lowest tile
        out.append(reg[np.arange(len(b)), score.argmax(1)])
    return out


def check_owner_homing(sc, p):
    """check_plan, and the homing of an independent-CTA plan re-derived from the scene; returns (X item share, global-homed share)."""
    G, C = check_plan(sc, p, True)
    assert G > 1 and C == 1
    n = sc.n
    slot = u32(p, "slot").astype(np.int64)
    tstart, tsmem = u32(p, "tileStart").astype(np.int64), u32(p, "tileSmem").astype(np.int64)
    ptile = np.searchsorted(tstart, slot, "right") - 1
    homed_global = (slot - tstart[ptile]) >= tsmem[ptile]
    region = bisect(np.asarray(sc.x0, np.float32), G)
    assert np.array_equal(ptile, region), "a particle is not in its tile of the bisection"
    buckets = np.frombuffer(p["buckets"], np.int32).reshape(-1, 4)
    tile_off = u32(p, "tileOff").astype(np.int64).reshape(len(buckets), 2 * G + 1)
    own = owners(sc, region)
    foreign = np.zeros(n, bool)  # touched by a constraint owned by another tile
    for t in range(NUM_TYPES):
        ids, b, _ = sc.store[t]
        if not len(ids):
            continue
        pk = [k for k in range(NB[t]) if not is_rb(t, k)]
        for k in pk:
            foreign[b[own[t] != region[b[:, k]], k]] = True
        pos = np.searchsorted(ids, u32(p, "order%d" % t))  # host rows in device order
        ex, isx = np.zeros(len(ids), np.int64), np.zeros(len(ids), bool)
        for bi in np.nonzero(buckets[:, 0] == t)[0]:
            lab = np.repeat(np.arange(2 * G), np.diff(tile_off[bi]))
            ex[buckets[bi, 1]:buckets[bi, 1] + buckets[bi, 2]], isx[buckets[bi, 1]:buckets[bi, 1] + buckets[bi, 2]] = lab // 2, lab % 2 == 0
        assert np.array_equal(ex, own[t][pos]), "type %d: an item does not run in its owner" % t
        bd = b[pos][:, pk]
        hg = homed_global[bd]
        assert np.array_equal(isx, hg.any(1)), "type %d: an item is an X item exactly when it touches a global-homed particle" % t
        assert (ptile[bd][~hg] == np.broadcast_to(ex[:, None], bd.shape)[~hg]).all(), \
            "type %d: a shared-memory particle of an item is homed in another tile than the item's owner" % t
        # the encoded indices of shared-memory particles address the owner's tile (rank 0 of a cluster of one)
        idx = indices(p, t, len(ids)).astype(np.int64)[:, pk]
        assert (((idx >> 27) & 15)[idx >= 1 << 31] == 0).all()
    assert np.array_equal(homed_global, foreign)
    return item_kinds(sc, p)[0] / sc.N, homed_global.mean()


def cloth(n):
    return lambda m: scenes.cfg2(m, n, 20)


_big = {}


def big(n):
    if n not in _big:
        _big[n] = Scene.of(cloth(n))
    return _big[n]


@pytest.mark.parametrize("n,x_max,global_max", [(1000, 0.07, 0.05), (500, 0.14, 0.10)], ids=["cfg2", "cfg5"])
def test_big_cloths(driver, tmp_path, n, x_max, global_max):
    """cfg2 (1000 x 1000) and cfg5 (500 x 500) in the planner's own shape, 132 independent CTAs: homed by owner, with at most 7 % X items
    and 5 % global-homed particles at cfg2, 14 % and 10 % at cfg5 (global wherever a constraint spans two tiles: 10.4 % and 6.5 % at
    cfg2, 20.4 % and 12.9 % at cfg5)."""
    sc = big(n)
    p = plan(driver, tmp_path, sc, RESIDENT)
    assert p["error"] == b""
    res = u32(p, "res")
    G, C, threads, xthreads = (int(v) for v in res[:4])
    assert (G, C) == (132, 1)
    x_share, g_share = check_owner_homing(sc, p)
    tsmem = u32(p, "tileSmem")
    print("%dx%d: %.2f %% X items, %.2f %% global-homed, %d of %d threads for X items, largest tile %d shared-memory particles (cap %d), "
          "smallest %d" % (n, n, 100 * x_share, 100 * g_share, xthreads, threads, tsmem.max(), int(res[5]), tsmem.min()))
    assert x_share <= x_max and g_share <= global_max
    assert xthreads == max(64, min((int(threads * x_share * 3.1) + 31) & ~31, (threads // 2) & ~31))


@pytest.mark.parametrize("regime", ["2x1", "7x1", "37x1"])
@pytest.mark.parametrize("name", sorted(rm.SCENES))
def test_mesh_scenes(driver, tmp_path, name, regime):
    """The large mesh scenes of tests/resident_meshes.py with independent CTAs: homed by owner, and every particle type has X items."""
    sc = Scene.of(rm.builder(name, "large"))
    p = plan(driver, tmp_path, sc, RESIDENT, rm.shape(regime), tag=regime)
    assert p["error"] == b"", p["error"]
    check_owner_homing(sc, p)
    for t, (nx, _, _) in item_kinds_by_type(sc, p).items():
        assert nx > 0, "type %d has no X items" % t


def test_particles_without_constraints(driver, tmp_path):
    """A cloth with a grid of free particles beside it: the free particles live in their tile's shared memory."""
    def build(m):
        scenes.cfg2(m, 120, 5)
    sc = Scene.of(build)
    free = np.stack(np.meshgrid(np.linspace(0, 10, 60), np.linspace(-3, 3, 40), indexing="ij"), -1).reshape(-1, 2)
    x0 = np.concatenate([np.asarray(sc.x0, np.float32), np.stack([free[:, 0], np.full(len(free), 1.0), free[:, 1]], 1).astype(np.float32)])
    sc2 = Scene.__new__(Scene)
    sc2.__dict__.update(sc.__dict__)
    sc2.n, sc2.x0 = len(x0), x0
    p = plan(driver, tmp_path, sc2, RESIDENT, (7, 1))
    assert p["error"] == b"", p["error"]
    check_owner_homing(sc2, p)


def test_straddling_stencils(tmp_path, driver):
    """The resident image of tests/test_gpu_projection_answers.py in seven independent CTAs: stencils that share no particle, with
    particle k of every stencil in the k-th quarter of a line.  Each stencil runs in the tile of most of its particles, and its particles
    in other tiles are global-homed, so it is an X item."""
    from test_gpu_projection_answers import plan_scene, resident_set
    sc = plan_scene(resident_set())
    p = plan(driver, tmp_path, sc, RESIDENT, (7, 1))
    assert p["error"] == b"", p["error"]
    check_owner_homing(sc, p)
    assert item_kinds(sc, p)[0] > 0
