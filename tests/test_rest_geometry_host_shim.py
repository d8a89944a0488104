"""CPU-side guard of the rest-geometry arithmetic a batch derives on the GPU for every replica (csrc/rest_geometry.cuh, k_derive_geometry):
the header compiled for the host through the test-only shim of tests/host_shim/, held against the unmodified reference in fp64 (oracle/_ref):
every type's geometry columns and initConstraint's verdict, on rigidly moved, anisotropically scaled and noisy rest shapes of a cloth (every
cloth and bending method) and a tet bar (every solid method), and on degenerate ones.  Runs without a GPU; not a product path."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest

import scenes
from conftest import have_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEO_FIRST = {3: 1, 4: 1, 12: 1}
NUM_GEO = {0: 1, 1: 1, 2: 1, 3: 16, 4: 16, 5: 5, 6: 4, 7: 1, 8: 1, 9: 10, 10: 10, 11: 9, 12: 23}
NUM_BODIES = {0: 2, 1: 2, 2: 4, 3: 4, 4: 4, 5: 3, 6: 3, 7: 4, 8: 4, 9: 4, 10: 4, 11: 4, 12: 4}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rest_geometry") / "librest_geometry_host.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "tests", "host_shim"), "-I" + os.path.join(ROOT, "positionbaseddynamics_b200", "csrc"),
                           "-o", so, os.path.join(ROOT, "tests", "host_shim", "rest_geometry.cpp")])
    lib = C.CDLL(so)
    lib.derive_rest_geometry.argtypes = [C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def derive(lib, t, bodies, x0, inv_mass):
    bodies = np.ascontiguousarray(np.asarray(bodies, np.uint32)[:, :NUM_BODIES[t]])
    x = np.zeros((len(x0), 4), np.float32); x[:, :3] = x0; x[:, 3] = inv_mass
    geo = np.zeros((len(bodies), NUM_GEO[t]), np.float32)
    ok = np.zeros(len(bodies), np.uint8); rank1 = np.zeros(len(bodies), np.uint8)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib.derive_rest_geometry(t, len(bodies), vp(bodies), vp(x), vp(geo), vp(ok), vp(rank1))
    return geo, ok.astype(bool), rank1.astype(bool)


def rest_shapes(x0, seed):
    """The model's rest positions rigidly moved, anisotropically scaled, and with 1 % noise."""
    rng = np.random.default_rng(seed)
    c = x0.mean(axis=0)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    s = rng.uniform(0.8, 1.25, 3)
    edge = float(np.ptp(x0, axis=0).max()) / 30.0
    return {"rigid": (x0 - c) @ R.T + c + rng.normal(0, 1.0, 3), "scaled": (x0 - c) * s + c,
            "noisy": ((x0 - c) * s) @ R.T + c + rng.normal(0.0, 0.01 * edge, x0.shape)}


def reference(cpu_libs, kind, x0, topo, inv_mass, candidates):
    """Every candidate (type, bodies) added one by one to the reference model on rest positions x0: initConstraint's verdict, and the
    parameters of the accepted ones."""
    m = cpu_libs.CpuPbd("ref", "f64")
    (m.add_triangle_model if kind == "cloth" else m.add_tet_model)(x0.astype(np.float64), topo)
    for i, w in enumerate(inv_mass):
        m.set_mass(i, 0.0 if w == 0 else 1.0 / float(w))
    verdict = []
    for t, b in candidates:
        args = {12: [1.0, 1, 1, 1, 1]}.get(t, [1.0, 1.0, 1.0, 0.3, 0.3])
        verdict.append(bool(m.add_constraint(t, [int(v) for v in b[:NUM_BODIES[t]]], args)))
    types, _, params, _ = m.constraints()
    return np.array(verdict), types, params


def compare(lib, cpu_libs, kind, x0, topo, inv_mass, model_types, model_bodies, what):
    """Our columns and verdicts against the reference's, constraint by constraint; returns the number of constraints compared."""
    x0 = x0.astype(np.float32)  # the fp32 rest positions both evaluate in double
    cands = [(int(t), b) for t, b in zip(model_types, model_bodies) if int(t) in NUM_GEO]
    verdict, rtypes, rparams = reference(cpu_libs, kind, x0, topo, inv_mass, cands)
    seen = 0
    for t in sorted({t for t, _ in cands}):
        sel = [i for i, (tt, _) in enumerate(cands) if tt == t]
        geo, ok, rank1 = derive(lib, t, np.array([cands[i][1] for i in sel]), x0.astype(np.float32), inv_mass)
        assert np.array_equal(ok, verdict[sel]), (what, t, "accept flags differ")
        ref = rparams[rtypes == t][:, GEO_FIRST.get(t, 0):GEO_FIRST.get(t, 0) + NUM_GEO[t]]
        mine = geo[ok].astype(np.float64)
        if t == 12:  # numClusters is topology, copied by the caller
            mine, ref = mine[:, :19], ref[:, :19]
        # relative to the largest column of the constraint; a rest angle near 0 (flat cloth: acos near 1) relative to one radian
        scale = np.maximum(np.abs(ref).max(axis=1, keepdims=True), 1.0 if t == 2 else 1e-30)
        err = float((np.abs(mine - ref) / scale).max(initial=0.0))
        assert err <= 1e-6, (what, t, err)
        if t in (3, 4):
            assert rank1[ok].all(), (what, "factor_rank1 rejects a derived Q")
        seen += len(sel)
    return seen


@pytest.mark.parametrize("seed", [1, 2])
def test_rest_geometry_matches_the_reference(shim, cpu_libs, seed):
    if not have_ref("f64"):
        pytest.skip("prebuilt oracle/_ref/libpbdref_f64.so not present")
    from positionbaseddynamics_b200.model import HostModel
    total = 0
    for kind, methods in (("cloth", [(c, b) for c in (1, 2, 3, 4) for b in (1, 2, 3)]), ("bar", [(s, 0) for s in (1, 2, 3, 4, 5, 6)])):
        for m1, m2 in methods:
            hm = HostModel()
            if kind == "cloth":
                scenes.cloth(hm, 12, 10, cloth_method=m1, bending_method=m2)
                topo = hm.tri_faces(0)
            else:
                scenes.bar(hm, 6, 3, 3, solid_method=m1, extra_volume=True)
                topo = hm.tet_tets(0)
            types, bodies, _, _ = hm.constraints()
            _, inv_mass = hm.masses()
            x0 = np.asarray(hm.get("x0"), np.float64)
            hm.close()
            for name, xs in rest_shapes(x0, seed + 10 * m1 + m2).items():
                total += compare(shim, cpu_libs, kind, xs, topo, inv_mass.astype(np.float32), types, bodies, "%s %d/%d %s" % (kind, m1, m2, name))
    print("rest geometry: %d constraints compared with the reference" % total)
    assert total > 10000


def test_degenerate_rest_shapes_are_refused_where_the_reference_refuses(shim, cpu_libs):
    if not have_ref("f64"):
        pytest.skip("prebuilt oracle/_ref/libpbdref_f64.so not present")
    x = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 1], [0, 1, 0], [1, 1, 1], [0.5, 0, 0], [0.5, 0, 0.0000001]], np.float32)
    inv = np.ones(len(x), np.float32)
    cases = [(5, [0, 1, 5]), (5, [0, 1, 2]), (6, [0, 1, 3]), (6, [0, 1, 2]), (6, [0, 5, 6]),  # collinear / in the x-y plane for the strain triangle
             (2, [0, 1, 5, 5]), (2, [0, 1, 2, 3]), (2, [2, 3, 0, 1]), (9, [0, 1, 5, 2]), (9, [0, 1, 2, 3]), (11, [0, 1, 5, 3]), (11, [0, 1, 2, 3]),
             (10, [0, 1, 2, 6]), (12, [0, 1, 2, 3]), (7, [0, 1, 2, 3]), (0, [0, 5]), (3, [0, 1, 2, 3])]
    verdict, _, _ = reference(cpu_libs, "bar", x.astype(np.float64), np.array([[0, 1, 2, 3]], np.uint32), inv, [(t, np.array(b, np.uint32)) for t, b in cases])
    for (t, b), want in zip(cases, verdict):
        _, ok, _ = derive(shim, t, np.array([b], np.uint32), x, inv)
        assert bool(ok[0]) == bool(want), (t, b, want)
    assert not verdict.all() and verdict.any()
    # ShapeMatching with every particle pinned (w = 0): wsum = 4 / eps, accepted
    _, ok, _ = derive(shim, 12, np.array([[0, 1, 2, 3]], np.uint32), x, np.zeros(len(x), np.float32))
    assert ok[0]
