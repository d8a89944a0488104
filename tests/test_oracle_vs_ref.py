"""Oracle pinned against the reference itself: on scenes larger than the golden fixtures of test_oracle_golden.py, against
what the reference computed for them (tests/golden/reference_runs.npz, recorded by tests/golden/make_golden.py runs); and,
where a build of the reference is present (oracle/_ref), against the live reference."""
import os
import numpy as np
import pytest

import scenes
from conftest import have_ref
from parity_util import digest, perturb

RUNS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_runs.npz")

needs_ref = pytest.mark.skipif(not (have_ref("f32") and have_ref("f64")), reason="oracle/_ref not built (no /root/reference here)")

CASES = {
    "cfg1": lambda m: scenes.cfg1(m, 50),
    "cloth_xpbd_64": lambda m: scenes.cfg2(m, 64, 8),
    "cloth_fem_dihedral": lambda m: scenes.cloth(m, 30, 30, 2, 1, fem=(1000.0, 1000.0, 500.0, 0.3, 0.3)),
    "cfg3_small": lambda m: scenes.cfg3(m, 14, 5, 5),
    "bar_xpbd": lambda m: scenes.bar(m, 10, 4, 4, 6, k=1e5, vol_k=1e5),
    "bar_strain": lambda m: scenes.bar(m, 10, 4, 4, 4, k=1.0),
    "bar_femx_1step": lambda m: scenes.bar(m, 7, 4, 4, 3, k=1.0e4, sub_steps=2, max_iter=3),
}


def steps_of(name):
    return 1 if name.endswith("1step") else 3  # XPBD-FEM amplifies rounding differences chaotically after a step


@pytest.mark.parametrize("name", sorted(CASES))
def test_structure_and_trajectory(name, cpu_libs):
    """Constraints, colour groups, constraint parameters and the positions after `steps_of(name)` steps of the oracle, against
    those the reference produced for the same scene (golden, both precisions)."""
    g = np.load(RUNS)
    for prec, tol in (("f64", 1e-9), ("f32", 5e-5)):
        key = "ovr/%s/%s/" % (name, prec)
        o = cpu_libs.CpuPbd("oracle", prec)
        CASES[name](o)
        to, bo, po, _ = o.constraints()
        go = o.groups()
        assert digest(to, np.int32) == str(g[key + "types"]) and digest(bo, np.uint32) == str(g[key + "bodies"])
        assert digest(go[0], np.uint32) == str(g[key + "group_off"]) and digest(go[1], np.uint32) == str(g[key + "group_ids"])
        pr = g[key + "params"].astype(np.float64)
        assert np.abs(po - pr).max() <= tol * max(np.abs(pr).max(), 1.0)
        perturb([o], 0.01)
        o.step(steps_of(name))
        xo, xr = o.get("x"), g[key + "x"].astype(np.float64)
        err = np.abs(xo - xr).max() / np.abs(xr).max()
        limit = tol
        if prec == "f32" and name in ("cfg1", "cloth_xpbd_64"):
            limit = 3e-3  # isometric bending in fp32: both sides are inside the reference's own cancellation noise
        if prec == "f32" and name == "bar_femx_1step":
            limit = 2e-3  # sqrt(2U') constraint near the rest state: ill-conditioned in fp32 (reference fp32 vs fp64 differ by 7e-5 here)
        assert err <= limit, (name, prec, err)


@needs_ref
def test_thread_count_does_not_change_results(cpu_libs):
    """Colours make the parallel Gauss-Seidel deterministic (SURVEY.md F6)."""
    r = cpu_libs.CpuPbd("ref", "f32")
    out = []
    for threads in (1, 4):
        r.reset(); r.set_threads(threads)
        scenes.cfg1(r, 40)
        r.step(5)
        out.append(r.get("x"))
    assert (out[0] == out[1]).all()


def test_reference_side_adapter_is_built_and_fails_loudly_without_a_gpu():
    """oracle/_ref/libpbdref_gpu_*.so = the unmodified reference + integration/GpuTimeStepController.h (the PBD::TimeStep subclass
    that binds libpbd_b200.so).  Here (no GPU) installing it must fail with the engine's "no CUDA device" message, never fall
    back to a CPU path; the GPU parity of the adapter is tests/test_gpu_parity.py::test_reference_side_adapter."""
    import torch
    from oracle import pyoracle
    for precision in ("f32", "f64"):
        if not pyoracle.available("refgpu", precision):
            pytest.skip("oracle/_ref/libpbdref_gpu_%s.so not built (no /root/reference here)" % precision)
        m = pyoracle.CpuPbd("refgpu", precision)
        scenes.cloth(m, 6, 6, 4, 3, dist_k=1e5, bend_k=100.0)
        if torch.cuda.is_available():
            m.use_gpu_timestep(0, 0)
            m.step(1)
            assert m.gpu_error() == ""
        else:
            with pytest.raises(RuntimeError, match="no CUDA device"):
                m.use_gpu_timestep(0, 0)
            x0 = m.get("x").copy()
            m.step(1)  # the reference's own TimeStepController is still installed and still works
            assert np.abs(m.get("x") - x0).max() > 0


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_contact_path_restatement_is_pinned_to_the_reference(precision, cpu_libs):
    """The C restatement of the contact path (oracle/pbd_oracle.c: distance functions, collisionTest, contact initialisation, velocity-level
    solve) against the reference's DistanceFieldCollisionDetection + ParticleRigidBodyContactConstraint in the same precision: in lockstep
    (the oracle takes the reference's state before every step) over 110 steps of a cloth falling onto all six analytic shapes -- the same
    contact list, and velocities that agree to rounding (the two sides evaluate the same formulas in the same precision)."""
    if not have_ref(precision):
        pytest.skip("prebuilt oracle/_ref/libpbdref_%s.so not present" % precision)
    ref = cpu_libs.CpuPbd("ref", precision); orc = cpu_libs.CpuPbd("oracle", precision)
    # Real = float: the reference takes the torus' ring distance from a float norm (Vector2r(x, z).norm(), DistanceFieldCollisionDetection.cpp:635);
    # the central differences of approximateNormal (eps = 1e-6) then differentiate rounding noise and the normal is off by percent in a
    # rounding-dependent direction -- nothing to pin there, so the float run leaves the torus out (the double run has all six shapes)
    shapes = ("box", "sphere", "torus", "cylinder", "hollow_sphere", "hollow_box") if precision == "f64" else ("box", "sphere", "cylinder", "hollow_sphere", "hollow_box")
    scenes.cloth_on_colliders(ref, 24, shapes=shapes)
    orc.add_regular_triangle_model(24, 24, t=(-2.5, 2.2, -2.5), R=scenes.RX90, scale=(5.0, 5.0))
    orc.add_cloth_constraints(0, 4, dist_k=1.0e5)
    orc.add_bending_constraints(0, 3, 100.0)
    orc.set_params(dt=0.005, sub_steps=1, max_iter=4)
    for row in ref.rigid_bodies():
        orc.add_rigid_body(0.0, row[:3], (1.0, 1.0, 1.0), row[3:7])
    models, rigid = ref.collision_objects()
    orc.set_colliders(models, rigid)
    orc.set_oracle_contact_params(tolerance=0.05, stiffness=100.0, max_iter_v=5)
    events = 0; worst_dv = 0.0; worst_x = 0.0; grazing = 0
    tol_v = 1e-9 if precision == "f64" else 5e-3  # float: the penalty impulse (stiffness 100 x depth) amplifies the rounding of the positions; a flipped contact would be 0.1 - 2 m/s
    for step in range(110):
        orc.set("x", ref.get("x")); orc.set("v", ref.get("v"))
        ref.step(1); orc.step(1)
        p, b, info, rr, pt = ref.contacts()
        po, bo, io = orc.oracle_contacts()
        a, c = set(zip(p.tolist(), b.tolist())), set(zip(po.tolist(), bo.tolist()))
        if a != c:  # only a contact whose signed distance is at the rounding level may be on one side only (never in fp64)
            assert precision == "f32" and len(a ^ c) <= 2, "step %d: contact lists differ: %s" % (step, sorted(a ^ c))
            grazing += len(a ^ c)
        events += len(p)
        worst_x = max(worst_x, float(np.abs(orc.get("x") - ref.get("x")).max()))
        dv = np.abs(orc.get("v") - ref.get("v")).max(axis=1)
        dv[[q for q, _ in a ^ c]] = 0.0
        worst_dv = max(worst_dv, float(dv.max()))
    print("contact restatement, %s: %d contact events, %d grazing, worst |dx| %.2e, worst |dv| %.2e" % (precision, events, grazing, worst_x, worst_dv))
    assert events > 2000 and grazing <= 4 and worst_dv <= tol_v


@needs_ref
@pytest.mark.parametrize("config", [(1, 1, 0), (2, 3, 1)], ids=["1x1_v0", "2x3_v1"])
def test_rigid_cases_in_lockstep(cpu_libs, config):
    """The rigid-body cases of tests/rigid_cases.py (both ball joints, chains, free spinning bodies; initial v and omega through
    set_rigid_body_velocity) in the reference and the C restatement, both fp64, in lockstep: bodies and particles equal to 1e-9 of each
    quantity's scale after every step."""
    import rigid_cases as rc
    ref = cpu_libs.CpuPbd("ref", "f64")
    if not hasattr(ref.lib, "ref_set_rigid_body_velocity"):
        pytest.skip("the prebuilt oracle/_ref predates set_rigid_body_velocity")
    m = rc.make_model(4, 31)
    orc = cpu_libs.CpuPbd("oracle", "f64")
    for ck in (ref, orc):
        rc.load(m, ck)
        ck.set_params(dt=rc.DT, sub_steps=config[0], max_iter=config[1], vel_method=config[2], gravity=rc.GRAVITY)
    (tr, br, pr, _), (to, bo, po_, _) = ref.constraints(), orc.constraints()
    assert np.array_equal(tr, to) and np.array_equal(br, bo) and np.abs(pr - po_).max() <= 1e-12 * np.abs(pr).max()
    assert all(np.array_equal(a, b) for a, b in zip(ref.groups(), orc.groups()))
    for _ in range(3):
        ref.step(1); orc.step(1)
        rr, ro = ref.rigid_bodies(), orc.rigid_bodies()
        for k in (slice(0, 3), slice(3, 7), slice(7, 10), slice(10, 13)):
            assert np.abs(rr[:, k] - ro[:, k]).max() <= 1e-9 * max(np.abs(rr[:, k]).max(), 1.0), k
        for name in ("x", "v"):
            assert np.abs(ref.get(name) - orc.get(name)).max() <= 1e-9 * max(np.abs(ref.get(name)).max(), 1.0), name
