"""The planner (csrc/host/image_plan.cpp) on replica batches with rigid bodies, on the CPU: a batch whose every replica has bodies of its
own (PlanInput::replicaBodies, tests/host_shim/plan_rigid_batch.cpp) is admitted with its joints, keeps the one-replica colouring and joint
buckets, and runs the resident mode on an instantiation that steps bodies; without the flag it stays refused."""
import os
import subprocess

import numpy as np
import pytest

import scenes
from plan_util import AUTO, GRAPH, LAUNCH, RESIDENT, Scene, check_plan, mode_of, same_image, u32
from test_batch_plan import PKG, ROOT, plan
from test_image_plan import cloth, rig

SOLID_MASK, ALL_MASK = 26555, 32767  # device_image.h: kMaskSolid, kMaskAll
BJ, RBP = 13, 14


def _driver(tmp_path_factory, name):
    from positionbaseddynamics_b200 import _capi
    _capi.lib()  # fails loudly when the library has not been built
    exe = str(tmp_path_factory.mktemp("plan") / name)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-std=c++17", "-O1", "-ccbin", "/usr/bin/g++", "-I" + os.path.join(PKG, "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "host_shim", name + ".cpp"), "-L" + PKG, "-lpbd_b200", "-Xlinker", "-rpath," + PKG])
    return exe


@pytest.fixture(scope="module")
def rigid_driver(tmp_path_factory):
    return _driver(tmp_path_factory, "plan_rigid_batch")


@pytest.fixture(scope="module")
def batch_driver(tmp_path_factory):
    return _driver(tmp_path_factory, "plan_batch")


def free_bodies(nb):
    """A 40 x 40 XPBD cloth and `nb` free bodies (no joint): what AUTO runs resident from 32 replicas on."""
    def build(m):
        scenes.cloth(m, 40, 40, cloth_method=4, bending_method=3, dist_k=1.0e5, bend_k=100.0, sub_steps=1, max_iter=3)
        for i in range(nb):
            m.add_rigid_body(1.0, (0.01 * i, 2.0, 0.0), (1.0, 1.0, 1.0))
    return build


def strain_rig(m):
    scenes.cloth(m, 12, 12, cloth_method=3, bending_method=3, bend_k=100.0)
    scenes.coupling_rig(m, 12, 12)


def test_joints_admitted_only_with_replica_bodies(rigid_driver, batch_driver, tmp_path):
    """The rig batch: refused without per-replica bodies, admitted with them in every mode but Jacobi; the graph image is the image of
    one replica, byte for byte."""
    r = Scene.of(rig)
    assert r.nrb and (np.asarray(r.store[BJ][0]).size and np.asarray(r.store[RBP][0]).size)
    for mode in (GRAPH, RESIDENT, AUTO):
        assert b"rigid bodies and joints" in plan(batch_driver, tmp_path, r, mode, 2)["error"]
    for mode in (GRAPH, LAUNCH):
        one = plan(batch_driver, tmp_path, r, mode, 1, tag="one")
        for k in (2, 300):
            p = plan(rigid_driver, tmp_path, r, mode, k, tag="k")
            assert p["error"] == b"", p["error"]
            check_plan(r, p, False)
            assert same_image(p, one)
    assert b"PBD_MODE_JACOBI" in plan(rigid_driver, tmp_path, r, 3, 2)["error"]


def test_resident_rig_batch_is_one_cluster_with_the_joints(rigid_driver, tmp_path):
    """The resident rig batch: one cluster per replica on the solid instantiation, the joint buckets and the colouring of one replica,
    every joint in a tile of that one cluster; a StrainTriangle cloth with the rig takes the all-types instantiation.  AUTO keeps joint
    models in graph mode."""
    for build, mask in ((rig, SOLID_MASK), (strain_rig, ALL_MASK)):
        sc = Scene.of(build)
        for k, mc in ((3, 40), (300, 40), (300, 7)):
            p = plan(rigid_driver, tmp_path, sc, RESIDENT, k, max_clusters=mc, tag="b")
            assert p["error"] == b"", p["error"]
            G, C = check_plan(sc, p, True)
            assert G == 1
            res = u32(p, "res")
            assert res[4] == mask and res[3] == 0
            assert [int(v) for v in u32(p, "batch")] == [k, min(k, mc)]
            # the joint buckets: every joint item is a shared-memory item of one of the cluster's C tiles
            buckets = u32(p, "buckets").reshape(-1, 4)
            toff = u32(p, "tileOff").reshape(len(buckets), 2 * C + 1)
            for b, off in zip(buckets, toff):
                if b[0] in (BJ, RBP):
                    assert off[0] == 0 and off[-1] == b[2]
                    assert all(off[2 * t] == off[2 * t + 1] for t in range(C))  # no X items
        assert mode_of(plan(rigid_driver, tmp_path, sc, AUTO, 300, tag="a")) == GRAPH


def test_cloth_batch_with_free_bodies_steps_them_resident(rigid_driver, batch_driver, tmp_path):
    """An XPBD cloth batch with free bodies under AUTO: resident from 32 replicas on, on the solid instantiation (the batched cloth kernel
    has no body path); without bodies the same cloth takes the cloth instantiation."""
    for nb in (1, 700):
        sc = Scene.of(free_bodies(nb))
        assert sc.nrb == nb
        assert mode_of(plan(rigid_driver, tmp_path, sc, AUTO, 8, tag="a8")) == GRAPH
        p = plan(rigid_driver, tmp_path, sc, AUTO, 32, tag="a32")
        assert mode_of(p) == RESIDENT
        assert u32(p, "res")[4] == SOLID_MASK
    bare = Scene.of(cloth(40))
    assert u32(plan(batch_driver, tmp_path, bare, AUTO, 32, tag="c32"), "res")[4] != SOLID_MASK
