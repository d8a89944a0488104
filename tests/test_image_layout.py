"""The layout of the device image (csrc/host/image_plan.cpp: image_layout), checked on the CPU through the planner drivers.  The engine
uploads the image into one allocation at these offsets and binds every pointer from the same list, so: every array on a 256-byte
boundary, no two overlapping, each followed by 16 bytes of its own allocation (the resident kernel's L2 prefetch rounds the end of a
run up to 16 bytes), the zeroed regions last (one memset) and of their sizes, and every array the plan holds or a present type reads
listed exactly once."""
import numpy as np
import pytest

from plan_util import (BALLJOINT, COLUMNS, ISOBENDING, NB, NUM_TYPES, RESIDENT, GRAPH, MAX_NBR, XPBD, Scene, build_driver, check_plan,
                       plan, u32)
from test_batch_plan import batch_driver  # noqa: F401  (fixture)
from test_image_plan import cloth, mixed, rig

X_FLAG_STRIDE = 16  # device_image.h: kXFlagStride
ROW = np.dtype([("name", "S32"), ("offset", "<u8"), ("bytes", "<u8")])


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_driver(tmp_path_factory.mktemp("plan"))


def layout_of(p):
    """(size of the allocation, [(name, offset, bytes)] of every listed array)."""
    raw = p["layout"]
    rows = np.frombuffer(raw[8:], ROW)
    return int(np.frombuffer(raw[:8], np.uint64)[0]), [(r["name"].decode(), int(r["offset"]), int(r["bytes"])) for r in rows]


def layout_errors(total, rows):
    """What breaks the layout rules in the arrays `rows` of an allocation of `total` bytes."""
    errs = []
    spans = sorted((o, b, name) for name, o, b in rows if b)
    for i, (o, b, name) in enumerate(spans):
        end = spans[i + 1][0] if i + 1 < len(spans) else total
        if o % 256:
            errs.append("%s starts at %d, not on a 256-byte boundary" % (name, o))
        if o + b > end:
            errs.append("%s overlaps the next region" % name)
        elif o + b + 16 > end:
            errs.append("%s has %d bytes of slack" % (name, end - o - b))
    return errs


def expected_arrays(sc, p, replicas, rest_tables):
    """{name: bytes} of every array the image must hold, from the scene; only the plan's bending variant and tables' shapes are read."""
    want = {}
    colour = sc.colour_of()
    pairs = set()
    for t in range(NUM_TYPES):
        ids = sc.store[t][0]
        cnt = len(ids)
        pairs |= {(int(g), t) for g in colour[ids]}
        if not cnt:
            continue
        if NB[t] == 3:
            want.update({"idx3_%d_%d" % (t, k): cnt * 4 for k in range(3)})
        else:
            want["idx%d_%d" % (NB[t], t)] = cnt * 4 * NB[t]
        gvc, gsc, matc = COLUMNS[t]
        variant = int(np.frombuffer(p["variant%d" % t], np.int32)[0])
        n_gv = 1 if t in ISOBENDING and variant == 0 else len(gvc)
        want.update({"gv%d_%d" % (t, k): cnt * 16 for k in range(n_gv)})
        want.update({"gs%d_%d" % (t, k): cnt * 4 for k in range(len(gsc))})
        prm = sc.store[t][2]
        want.update({"mat%d_%d" % (t, k): cnt * 4 for k, c in enumerate(matc) if (prm[:, c] != prm[0, c]).any()})
        if t in XPBD:
            want["lambda%d" % t] = replicas * cnt * 4
        if rest_tables and t < BALLJOINT:
            want.update({"restBodies%d" % t: cnt * NB[t] * 4, "restLocal%d" % t: cnt * 4, "restIds%d" % t: cnt * 4})
    want["buckets"] = len(pairs) * 16
    if int(np.frombuffer(p["mode"], np.int32)[0]) == RESIDENT:
        G, C, n_col = (int(v) for v in u32(p, "res")[[0, 1, 6]])
        launched = int(u32(p, "batch")[1])
        T = G * C  # the tiles of the tables: one replica's in a batch
        want.update({"colourStart": (n_col + 1) * 4, "tileOff": len(pairs) * (2 * T + 1) * 4, "tileStart": (T + 1) * 4,
                     "tileSmem": T * 4, "xNbr": T * MAX_NBR * 4, "xMask": T * (1 + n_col) * 4,
                     "xFlags": launched * C * X_FLAG_STRIDE * 8})
    return want


def check_layout(sc, p, replicas=1, rest_tables=False):
    total, rows = layout_of(p)
    assert layout_errors(total, rows) == []
    names = [name for name, _, _ in rows]
    assert len(set(names)) == len(names)
    listed = {name: b for name, _, b in rows if b}
    assert listed == expected_arrays(sc, p, replicas, rest_tables)
    zeroed = [o for name, o, b in rows if b and (name.startswith("lambda") or name == "xFlags")]
    data = [o for name, o, b in rows if b and name not in ("xFlags",) and not name.startswith("lambda")]
    assert not zeroed or not data or max(data) < min(zeroed)  # the zeroed regions last: one memset clears them
    for name, _, b in rows:  # the arrays with a host source are the plan's records
        if not (name.startswith("lambda") or name == "xFlags"):
            assert len(p[name]) == b
    return total, rows


@pytest.mark.parametrize("build,shape", [(cloth(40), "graph"), (mixed, "graph"), (rig, "graph"), (cloth(60), "1x1"), (cloth(100), "1x4"),
                                         (cloth(100), "7x1"), (mixed, "5x1"), (rig, "1x1")],
                         ids=["cloth-graph", "mixed-graph", "rig-graph", "cloth-1x1", "cloth-1x4", "cloth-7x1", "mixed-5x1", "rig-1x1"])
def test_layout(driver, tmp_path, build, shape):
    sc = Scene.of(build)
    tiled = shape != "graph"
    G, C = (int(v) for v in shape.split("x")) if tiled else (0, 0)
    p = plan(driver, tmp_path, sc, RESIDENT if tiled else GRAPH, (G, C))
    check_plan(sc, p, tiled)
    check_layout(sc, p)


@pytest.mark.parametrize("mode", [GRAPH, RESIDENT])
def test_batch_layout_with_rest_tables(batch_driver, tmp_path, mode):  # noqa: F811
    """A batch of 3 with per-replica rest shapes: the multipliers of every replica, and the tables their geometry is derived from."""
    sc = Scene.of(cloth(40))
    p = plan(batch_driver, tmp_path, sc, mode, rest_tables=True, replicas=3, max_clusters=40)
    assert p["error"] == b""
    check_layout(sc, p, replicas=3, rest_tables=True)
    assert np.array_equal(u32(p, "restIds1"), u32(p, "order1"))  # the insertion ids in device order
    assert np.array_equal(u32(p, "restLocal1"), np.searchsorted(sc.store[1][0], u32(p, "order1")))


def test_layout_check_rejects_missing_slack(driver, tmp_path):
    """Negative control: the same layout with the slack after one array taken away fails the check."""
    sc = Scene.of(cloth(60))
    total, rows = check_layout(sc, plan(driver, tmp_path, sc, RESIDENT, (1, 1)))
    spans = sorted((o, name) for name, o, b in rows if b)
    for (o, name), nxt in zip(spans, [s[0] for s in spans[1:]] + [total]):
        tight = [(nm, oo, (nxt - o) if nm == name else b) for nm, oo, b in rows]
        assert any("0 bytes of slack" in err for err in layout_errors(total, tight)), name
