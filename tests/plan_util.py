"""The device-image planner (csrc/host/image_plan.cpp) run on the CPU through a small driver linked against the built libpbd_b200.so
(tests/host_shim/plan_image.cpp), and the invariants of its plans: shared by tests/test_image_plan.py and
tests/test_gpu_projection_answers.py.  Every expectation is derived from the host model's constraints, groups and rest positions and from
the raw plan -- slot map and tiles, buckets, index decoding, tile runs, and the X-neighbour tables whose errors the resident kernel would
turn into a hang rather than a failure."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "positionbaseddynamics_b200")
NUM_TYPES = 15
NB = [2, 2, 4, 4, 4, 3, 3, 4, 4, 4, 4, 4, 4, 2, 2]
NP = [2, 2, 2, 17, 17, 10, 9, 2, 2, 12, 12, 13, 24, 12, 6]
XPBD = {1, 4, 8, 10}
ISOBENDING, BALLJOINT, RB_PARTICLE_BALLJOINT = (3, 4), 13, 14
SMEM_FLAG, RANK_SHIFT = 0x80000000, 27
MAX_SMEM, MAX_NBR = 227 * 1024, 32
GRAPH, RESIDENT, LAUNCH, JACOBI, AUTO = range(5)  # pbd_solver_mode
# Parameter columns of the SoA arrays (the layout of include/pbd_b200.h): float4 geometry arrays (-1: zero), scalar arrays, material slots
_C4 = lambda *cs: [tuple(range(c, c + 4)) for c in cs]
COLUMNS = {0: ([], [0], [1]), 1: ([], [0], [1]), 2: ([], [0], [1]), 7: ([], [0], [1]), 8: ([], [0], [1]),
           3: (_C4(1, 5, 9, 13), [], [0]), 4: (_C4(1, 5, 9, 13), [], [0]),
           5: (_C4(1), [0], [5, 6, 7, 8, 9]), 6: (_C4(0), [], [4, 5, 6, 7, 8]),
           9: (_C4(1, 5), [9, 0], [10, 11]), 10: (_C4(1, 5), [9, 0], [10, 11]), 11: (_C4(0, 4), [8], [9, 10, 11, 12]),
           12: ([(1, 2, 3, -1)] + _C4(4, 8, 12, 16, 20), [], [0]),
           13: ([(0, 1, 2, -1), (3, 4, 5, -1)], [], []), 14: ([(0, 1, 2, -1)], [], [])}


def is_rb(t, k):
    return t == BALLJOINT or (t == RB_PARTICLE_BALLJOINT and k == 0)


def build_driver(out_dir):
    """Compile the planner driver (tests/host_shim/plan_image.cpp) against the built libpbd_b200.so into out_dir; returns its path."""
    from positionbaseddynamics_b200 import _capi
    _capi.lib()  # fails loudly when the library has not been built
    exe = os.path.join(str(out_dir), "plan_image")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")  # the compiler the library is built with (csrc/Makefile)
    subprocess.check_call([nvcc, "-std=c++17", "-O1", "-ccbin", "/usr/bin/g++", "-I" + os.path.join(PKG, "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "host_shim", "plan_image.cpp"), "-L" + PKG, "-lpbd_b200", "-Xlinker", "-rpath," + PKG])
    return exe


class Scene:
    """Constraints by type (insertion ids, bodies, parameters), colour groups and rest positions of a model."""
    def __init__(self, n, nrb, types, bodies, params, off, ids, x0):
        self.n, self.nrb, self.off, self.ids, self.x0 = n, nrb, np.asarray(off, np.uint32), np.asarray(ids, np.uint32), x0
        self.N = len(types)
        self.store = []
        for t in range(NUM_TYPES):
            sel = np.nonzero(types == t)[0].astype(np.uint32)
            self.store.append((sel, np.ascontiguousarray(bodies[sel, :NB[t]], np.uint32), np.ascontiguousarray(params[sel, :NP[t]], np.float32)))

    @classmethod
    def of(cls, build):
        from positionbaseddynamics_b200.model import HostModel
        m = HostModel()
        build(m)
        m.init_groups()
        types, bodies, params, _ = m.constraints()
        off, ids = m.groups()
        s = cls(m.num_particles(), len(m.rigid_bodies()), types, bodies, params, off, ids, m.get("x0"))
        m.close()
        return s

    def colour_of(self):
        col = np.zeros(self.N, np.int64)
        for g in range(len(self.off) - 1):
            col[self.ids[self.off[g]:self.off[g + 1]]] = g
        return col


def plan(driver, tmp_path, sc, mode, shape=(0, 0), threads=None, tag="p", max_clusters=132, replicas=1, rest_tables=False):
    """The plan of `replicas` replicas of `sc` in `mode` on a device of 132 SMs that keeps `max_clusters` clusters of any shape co-resident."""
    x0 = np.zeros((sc.n, 4), np.float32); x0[:, :3] = sc.x0
    head = [replicas, sc.n, sc.nrb, sc.N, mode, int(rest_tables), shape[0], shape[1], 132, max_clusters, len(sc.off) - 1]
    parts = [np.asarray(head, np.uint32), sc.off, sc.ids, x0]
    for ids, b, p in sc.store:
        parts += [np.asarray([len(ids)], np.uint32), ids, b, p]
    fin, fout = str(tmp_path / (tag + ".in")), str(tmp_path / (tag + ".out"))
    with open(fin, "wb") as f:
        for a in parts:
            f.write(np.ascontiguousarray(a).tobytes())
    env = dict(os.environ)
    if threads:
        env["PBD_B200_HOST_THREADS"] = str(threads)
    subprocess.check_call([driver, fin, fout], env=env)
    raw = open(fout, "rb").read()
    out, at = {}, 0
    while at < len(raw):
        name = raw[at:at + 32].split(b"\0")[0].decode(); size = int(np.frombuffer(raw[at + 32:at + 40], np.uint64)[0])
        out[name] = raw[at + 40:at + 40 + size]; at += 40 + size
    out["raw"] = raw
    return out


def u32(p, k):
    return np.frombuffer(p[k], np.uint32)


def mode_of(p):
    assert p["error"] == b""
    return int(np.frombuffer(p["mode"], np.int32)[0])


def same_image(a, b, *skip):
    """The plans `a` and `b` are byte-identical, apart from the refusal, the layout (its multipliers and X flags are sized by the batch and
    the clusters launched, not by the image) and the records in `skip`."""
    drop = {"raw", "residentRefusal", "layout"} | set(skip)
    return {k: v for k, v in a.items() if k not in drop} == {k: v for k, v in b.items() if k not in drop}


def indices(p, t, cnt):
    if NB[t] == 2:
        return u32(p, "idx2_%d" % t).reshape(cnt, 2)
    if NB[t] == 4:
        return u32(p, "idx4_%d" % t).reshape(cnt, 4)
    return np.stack([u32(p, "idx3_%d_%d" % (t, k)) for k in range(3)], 1)


def check_plan(sc, p, tiled):
    """Every invariant of the plan `p` of scene `sc`; returns (G, C)."""
    assert p["error"] == b""
    assert (mode_of(p) == RESIDENT) == tiled
    n = sc.n
    slot = u32(p, "slot")
    assert np.array_equal(np.sort(slot), np.arange(n))                        # a permutation
    inv = np.empty(n, np.int64); inv[slot] = np.arange(n)
    buckets = np.frombuffer(p["buckets"], np.int32).reshape(-1, 4)          # type, first, count, colour
    G, C, threads, xthreads, mask, tile_cap, n_col = (int(v) for v in u32(p, "res"))
    T = G * C
    smem = int(np.frombuffer(p["smem"], np.uint64)[0])
    colour = sc.colour_of()

    # buckets: colour after colour, each exactly its colour group's constraints of its type, no body twice in a colour
    assert (np.diff(buckets[:, 3]) >= 0).all()
    order = {t: u32(p, "order%d" % t) for t in range(NUM_TYPES)}
    nxt = np.zeros(NUM_TYPES, np.int64)
    for t, first, cnt, g in buckets:
        assert first == nxt[t]; nxt[t] += cnt
        got = order[t][first:first + cnt]
        want = sc.ids[sc.off[g]:sc.off[g + 1]]
        assert np.array_equal(np.sort(got), np.sort(want[np.isin(want, sc.store[t][0])]))
    for t in range(NUM_TYPES):
        assert nxt[t] == len(sc.store[t][0]) == len(order[t])
    for g in range(len(sc.off) - 1):
        members = sc.ids[sc.off[g]:sc.off[g + 1]]
        part, rb = [], []
        for t in range(NUM_TYPES):
            ids, b, _ = sc.store[t]
            sel = np.isin(ids, members)
            for k in range(NB[t]):
                (rb if is_rb(t, k) else part).append(b[sel, k])
        for lst in (part, rb):
            if lst:
                allb = np.concatenate(lst)
                assert len(np.unique(allb)) == len(allb), "colour %d uses a body twice" % g

    if tiled:
        tstart, tsmem = u32(p, "tileStart").astype(np.int64), u32(p, "tileSmem").astype(np.int64)
        assert len(tstart) == T + 1 and tstart[0] == 0 and tstart[-1] == n and (np.diff(tstart) >= 0).all()
        assert (tsmem <= np.diff(tstart)).all() and (tsmem <= tile_cap).all() and tile_cap % 64 == 0
        assert tile_cap * 16 + len(buckets) * 32 + (2 * n_col + 2 + MAX_NBR) * 4 <= MAX_SMEM
        assert smem == tile_cap * 16 + len(buckets) * 32 + (2 * n_col + 2 + MAX_NBR) * 4  # what the kernel lays out
        assert 16 * tile_cap <= smem <= MAX_SMEM
        ptile = np.searchsorted(tstart, slot, "right") - 1                   # tile of every host particle
        homed_global = (slot - tstart[ptile]) >= tsmem[ptile]
        assert n_col == len(np.unique(buckets[:, 3]))
        tile_off = u32(p, "tileOff").astype(np.int64).reshape(len(buckets), 2 * T + 1)
        touch = [np.stack([np.nonzero(homed_global)[0], ptile[homed_global]], 1)]  # (global-homed particle, tile)
        has_x = np.zeros((T, 1 + n_col), bool)
        has_x[:, 0] = tsmem < np.diff(tstart)
        col_index = {c: i for i, c in enumerate(np.unique(buckets[:, 3]))}

    for t in range(NUM_TYPES):
        ids, bod, par = sc.store[t]
        cnt = len(ids)
        if not cnt:
            continue
        pos = np.searchsorted(ids, order[t])                                  # host rows in device order
        b, prm = bod[pos], par[pos]
        idx = indices(p, t, cnt).astype(np.int64)
        # executing tile and kind of every item, from the runs of the buckets
        ex, isx = np.zeros(cnt, np.int64), np.zeros(cnt, bool)
        for bi in np.nonzero(buckets[:, 0] == t)[0]:
            first, bc = buckets[bi, 1], buckets[bi, 2]
            if tiled:
                runs = tile_off[bi]
                assert runs[0] == 0 and runs[-1] == bc and (np.diff(runs) >= 0).all()
                lab = np.repeat(np.arange(2 * T), np.diff(runs))
                ex[first:first + bc], isx[first:first + bc] = lab // 2, lab % 2 == 0
                for tile in np.unique(lab[lab % 2 == 0] // 2):
                    has_x[tile, 1 + col_index[buckets[bi, 3]]] = True
        pk = [k for k in range(NB[t]) if not is_rb(t, k)]
        for k in range(NB[t]):
            v = idx[:, k]
            if is_rb(t, k):
                assert np.array_equal(v, b[:, k]); continue
            if not tiled:
                assert np.array_equal(v, slot[b[:, k]]); continue
            sm = (v & SMEM_FLAG) != 0
            rank, local = (v >> RANK_SHIFT) & 15, v & ((1 << RANK_SHIFT) - 1)
            in_tile = local ^ ((local >> 3) & 7)                                # the swizzle is its own inverse
            tile = (ex // C) * C + rank
            assert (in_tile[sm] < tsmem[tile[sm]]).all()
            assert np.array_equal(inv[tstart[tile[sm]] + in_tile[sm]], b[sm, k])
            assert np.array_equal(inv[v[~sm]], b[~sm, k]) and homed_global[b[~sm, k]].all()
            assert not homed_global[b[sm, k]].any()
        if tiled and pk:
            hg = homed_global[b[:, pk]]
            assert hg[isx].any(1).all(), "an X item touches no global-homed particle"
            assert not hg[~isx].any(), "a shared-memory item touches a global-homed particle"
            home = ptile[b[:, pk]]
            assert ((home[~isx] // C) == (ex[~isx] // C)[:, None]).all()
            if C == 1:
                assert (home[~isx] == ex[~isx][:, None]).all()
            for k in pk:
                sel = isx & homed_global[b[:, k]]
                touch.append(np.stack([b[sel, k], ex[sel]], 1))
        # geometry and material columns
        gvc, gsc, matc = COLUMNS[t]
        variant = int(np.frombuffer(p["variant%d" % t], np.int32)[0])
        gv = {k: np.frombuffer(p["gv%d_%d" % (t, k)], np.float32).reshape(-1, 4) for k in range(6)}
        if t in ISOBENDING and variant == 0:
            Q = prm[:, 1:17].reshape(cnt, 4, 4).astype(np.float64)
            kp = gv[0].astype(np.float64)
            assert np.abs(Q + kp[:, :, None] * kp[:, None, :]).max() <= 1e-4 * max(np.abs(Q).max(), 1e-30)
            assert all(len(gv[k]) == 0 for k in range(1, 6))
        else:
            for k, cols in enumerate(gvc):
                want = np.stack([prm[:, c] if c >= 0 else np.zeros(cnt, np.float32) for c in cols], 1)
                assert np.array_equal(gv[k], want)
        for k, c in enumerate(gsc):
            assert np.array_equal(np.frombuffer(p["gs%d_%d" % (t, k)], np.float32), prm[:, c])
        matu = np.frombuffer(p["matU%d" % t], np.float32)
        for k, c in enumerate(matc):
            arr = np.frombuffer(p["mat%d_%d" % (t, k)], np.float32)
            assert np.array_equal(arr, prm[:, c]) if len(arr) else (prm[:, c] == matu[k]).all()

    if tiled:
        # neighbours: tiles that share a global-homed particle through their X items or its home, symmetric and complete
        tp = np.unique(np.concatenate(touch), axis=0)
        want = [set() for _ in range(T)]
        for part in np.split(tp[:, 1], np.nonzero(np.diff(tp[:, 0]))[0] + 1):
            for i in part:
                want[i].update(int(j) for j in part if j != i)
        nbr = u32(p, "xNbr").reshape(T, MAX_NBR)
        xmask = u32(p, "xMask").reshape(T, 1 + n_col)
        for i in range(T):
            k_used = [k for k in range(MAX_NBR) if nbr[i, k] != i]
            got = [int(nbr[i, k]) for k in k_used]
            assert len(set(got)) == len(got) and set(got) == want[i], "tile %d" % i
            assert k_used == list(range(len(got)))
            for ph in range(1 + n_col):
                for k in range(MAX_NBR):
                    bit = (int(xmask[i, ph]) >> k) & 1
                    assert bit == (k < len(got) and has_x[got[k], ph]), (i, ph, k)
        assert all(i in want[j] for i in range(T) for j in want[i])
    else:
        assert smem == 0
    return G, C


def item_kinds(sc, p):
    """(X items, shared-memory items whose particles live in another CTA of the cluster (DSMEM), shared-memory items of the executing
    CTA's own tile) of a resident plan."""
    return tuple(int(v) for v in np.sum(list(item_kinds_by_type(sc, p).values()) or [(0, 0, 0)], axis=0))


def item_kinds_by_type(sc, p):
    """item_kinds of every type the scene has: {type: (X items, DSMEM items, own-tile items)}."""
    G, C = (int(v) for v in u32(p, "res")[:2])
    buckets = np.frombuffer(p["buckets"], np.int32).reshape(-1, 4)
    tile_off = u32(p, "tileOff").astype(np.int64).reshape(len(buckets), 2 * G * C + 1)
    kinds = {}
    for t in range(NUM_TYPES):
        cnt = len(sc.store[t][0])
        if not cnt:
            continue
        idx = indices(p, t, cnt).astype(np.int64)
        ex, isx = np.zeros(cnt, np.int64), np.zeros(cnt, bool)
        for bi in np.nonzero(buckets[:, 0] == t)[0]:
            first, bc = buckets[bi, 1], buckets[bi, 2]
            lab = np.repeat(np.arange(2 * G * C), np.diff(tile_off[bi]))
            ex[first:first + bc], isx[first:first + bc] = lab // 2, lab % 2 == 0
        pk = [k for k in range(NB[t]) if not is_rb(t, k)]
        remote = np.zeros(cnt, bool)
        for k in pk:
            v = idx[:, k]
            remote |= ((v & SMEM_FLAG) != 0) & (((v >> RANK_SHIFT) & 15) != ex % C)
        kinds[t] = (int(isx.sum()), int((~isx & remote).sum()), int((~isx & ~remote).sum()))
    return kinds
