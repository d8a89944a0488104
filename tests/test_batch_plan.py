"""The image of a replica batch as the planner (csrc/host/image_plan.cpp) builds it, checked on the CPU with a driver of its own
(tests/host_shim/plan_batch.cpp): the graph image is the one-scene image (the replicas share it), the resident image is the tiling of one
replica into one cluster with as many clusters as the device runs at once, and what a batch cannot run is refused."""
import os
import subprocess

import numpy as np
import pytest

import scenes
from plan_util import AUTO, GRAPH, JACOBI, LAUNCH, RESIDENT, Scene, check_plan, mode_of, same_image, u32
from test_image_plan import cloth, mixed, rig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "positionbaseddynamics_b200")
SM_COUNT = 132
LIGHT_MASK = 447  # device_image.h: kMaskLight


@pytest.fixture(scope="module")
def batch_driver(tmp_path_factory):
    from positionbaseddynamics_b200 import _capi
    _capi.lib()  # fails loudly when the library has not been built
    exe = str(tmp_path_factory.mktemp("plan") / "plan_batch")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-std=c++17", "-O1", "-ccbin", "/usr/bin/g++", "-I" + os.path.join(PKG, "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "host_shim", "plan_batch.cpp"), "-L" + PKG, "-lpbd_b200", "-Xlinker", "-rpath," + PKG])
    return exe


def plan(driver, tmp_path, sc, mode, replicas, shape=(0, 0), max_clusters=40, tag="p"):
    """The plan of `replicas` replicas of `sc` in `mode` on a device of 132 SMs that runs `max_clusters` clusters of any shape at once."""
    x0 = np.zeros((sc.n, 4), np.float32); x0[:, :3] = sc.x0
    head = [replicas, sc.n, sc.nrb, sc.N, mode, 0, shape[0], shape[1], SM_COUNT, max_clusters, len(sc.off) - 1]
    parts = [np.asarray(head, np.uint32), sc.off, sc.ids, x0]
    for ids, b, p in sc.store:
        parts += [np.asarray([len(ids)], np.uint32), ids, b, p]
    fin, fout = str(tmp_path / (tag + ".in")), str(tmp_path / (tag + ".out"))
    with open(fin, "wb") as f:
        for a in parts:
            f.write(np.ascontiguousarray(a).tobytes())
    subprocess.check_call([driver, fin, fout])
    raw = open(fout, "rb").read()
    out, at = {}, 0
    while at < len(raw):
        name = raw[at:at + 32].split(b"\0")[0].decode(); size = int(np.frombuffer(raw[at + 32:at + 40], np.uint64)[0])
        out[name] = raw[at + 40:at + 40 + size]; at += 40 + size
    out["raw"] = raw
    return out


@pytest.mark.parametrize("build", [cloth(40), mixed], ids=["cloth", "mixed"])
@pytest.mark.parametrize("mode", [GRAPH, LAUNCH])
def test_graph_image_is_shared(batch_driver, tmp_path, build, mode):
    """The graph and launch images of a batch are byte for byte the image of one replica: uploaded once, shared by all."""
    sc = Scene.of(build)
    one = plan(batch_driver, tmp_path, sc, mode, 1, tag="one")
    check_plan(sc, one, False)
    for k in (3, 300):
        assert same_image(plan(batch_driver, tmp_path, sc, mode, k, tag="k%d" % k), one)


@pytest.mark.parametrize("build", [cloth(40), cloth(100), mixed], ids=["cloth40", "cloth100", "mixed"])
def test_resident_batch_is_one_cluster_per_replica(batch_driver, tmp_path, build):
    """The batched resident image: the one-cluster tiling of one replica with the same C (no X items, no global-homed particles),
    launched as G = min(K, what the cluster query answers) clusters."""
    sc = Scene.of(build)
    for k, mc in ((3, 40), (300, 40), (300, 7)):
        p = plan(batch_driver, tmp_path, sc, RESIDENT, k, max_clusters=mc, tag="b")
        G, C = check_plan(sc, p, True)
        assert G == 1 and 1 <= C <= 16 and C & (C - 1) == 0
        replicas, launched = (int(v) for v in u32(p, "batch"))
        assert replicas == k and launched == min(k, mc)
        res = u32(p, "res")
        assert res[3] == 0                                                    # no X threads
        assert np.array_equal(u32(p, "tileSmem"), np.diff(u32(p, "tileStart")))  # every particle in shared memory
        solo = plan(batch_driver, tmp_path, sc, RESIDENT, 1, shape=(1, C), max_clusters=mc, tag="s")
        assert same_image(p, solo, "batch", "res")
        solo_res = u32(solo, "res")                   # the same shape, apart from the batched light kernel's block size
        assert np.array_equal(np.delete(res, 2), np.delete(solo_res, 2))
        assert res[2] == (384 if res[4] == LIGHT_MASK else solo_res[2])


def test_cluster_size_follows_the_batch(batch_driver, tmp_path):
    """A replica that fits one CTA gets clusters of one at every K.  A bigger one keeps the single-scene cluster size while the device
    runs all K clusters of that size at once, and otherwise the smallest cluster that holds it."""
    small = Scene.of(cloth(100))                                  # 10,000 particles: one CTA holds them
    assert check_plan(small, plan(batch_driver, tmp_path, small, RESIDENT, 1, tag="s"), True)[1] > 1
    for k in (2, 1000):
        assert check_plan(small, plan(batch_driver, tmp_path, small, RESIDENT, k, tag="k"), True)[1] == 1
    bar = Scene.of(lambda m: scenes.bar(m, 41, 21, 21, extra_volume=True))  # 18,081 particles: two CTAs at least
    solo = check_plan(bar, plan(batch_driver, tmp_path, bar, RESIDENT, 1, tag="bs"), True)[1]
    assert solo == 16
    assert check_plan(bar, plan(batch_driver, tmp_path, bar, RESIDENT, 30, max_clusters=40, tag="b30"), True)[1] == 16
    assert check_plan(bar, plan(batch_driver, tmp_path, bar, RESIDENT, 30, max_clusters=20, tag="b20"), True)[1] == 2
    assert check_plan(bar, plan(batch_driver, tmp_path, bar, RESIDENT, 100, max_clusters=40, tag="b100"), True)[1] == 2


def test_auto_mode_of_a_batch(batch_driver, tmp_path):
    """AUTO: a small cloth or FEM model runs a batch of 32 or more replicas in the resident mode, fewer in the graph mode."""
    sc = Scene.of(cloth(40))
    assert mode_of(plan(batch_driver, tmp_path, sc, AUTO, 8, tag="a8")) == GRAPH
    p = plan(batch_driver, tmp_path, sc, AUTO, 32, tag="a32")
    assert mode_of(p) == RESIDENT and same_image(p, plan(batch_driver, tmp_path, sc, RESIDENT, 32, tag="r32"))
    # a model only the light instantiation covers: from 64 replicas on
    light = Scene.of(lambda m: scenes.cloth(m, 40, 40, cloth_method=2, bending_method=1))
    assert mode_of(plan(batch_driver, tmp_path, light, AUTO, 32, tag="l32")) == GRAPH
    assert mode_of(plan(batch_driver, tmp_path, light, AUTO, 64, tag="l64")) == RESIDENT


def test_replica_too_big_for_one_cluster(batch_driver, tmp_path):
    """A replica that does not fit one cluster: refused under RESIDENT, the graph image under AUTO."""
    sc = Scene.of(cloth(500))
    p = plan(batch_driver, tmp_path, sc, RESIDENT, 4, tag="r")
    assert b"does not fit one cluster" in p["error"]
    q = plan(batch_driver, tmp_path, sc, AUTO, 4, tag="a")
    assert mode_of(q) == GRAPH and q["residentRefusal"] == p["error"]
    assert same_image(q, plan(batch_driver, tmp_path, sc, GRAPH, 4, tag="g"))


def test_batch_refusals(batch_driver, tmp_path):
    """No replicas, more particles than 2^31, rigid bodies / joints and the Jacobi mode are refused; one replica of a rigid scene is not."""
    sc = Scene.of(cloth(40))
    assert plan(batch_driver, tmp_path, sc, GRAPH, 0)["error"] == b"replica batch: at least one replica"
    k = (1 << 31) // sc.n + 1
    assert b"exceed 2^31 particles" in plan(batch_driver, tmp_path, sc, GRAPH, k)["error"]
    assert b"at most 65535" in plan(batch_driver, tmp_path, sc, GRAPH, 65536)["error"]
    assert plan(batch_driver, tmp_path, sc, GRAPH, 65535)["error"] == b""
    assert b"PBD_MODE_JACOBI" in plan(batch_driver, tmp_path, sc, JACOBI, 2)["error"]
    assert plan(batch_driver, tmp_path, sc, JACOBI, 1)["error"] == b""
    r = Scene.of(rig)
    for mode in (GRAPH, RESIDENT, AUTO):
        assert b"rigid bodies and joints" in plan(batch_driver, tmp_path, r, mode, 2)["error"]
    assert plan(batch_driver, tmp_path, r, GRAPH, 1)["error"] == b""
