"""Every constraint projection against the fp64 solver functions, through the engine's execution paths.

Stencil sets and the fp64 restatement of the engine's loop are in tests/projection_cases.py.  The CPU tests check the generator (every
literally kept branch is taken by some case) and pin the restatement to the checker's own time step.  The GPU tests run the sets through

  launch_type   one type per engine, MODE_LAUNCH: k_project<T, VAR, false> (one bucket per colour)
  launch_multi  all types in one engine, MODE_LAUNCH: one colour of at most 65,536 constraints, k_project_multi<false>
  graph         the same engines, MODE_GRAPH
  uniform       per type the cases that share one material row: the uniform kernel argument instead of per-constraint arrays
  resident      the rank-one types, MODE_RESIDENT (the full-Q IsometricBending layout is refused there and stays out)
  jacobi        MODE_JACOBI; the stencils share no particle, so every particle has one store per sweep
  batch_*       K = 3 replicas, each with its own x, v, masses and, for a subset of types, material row (set_replica_materials):
                k_project<T, VAR, true> (one type per engine) and k_project_multi<true> (all types), launch and graph; resident K = 3

and compare x, v and the XPBD multipliers (by insertion id) with the reference; every path but Jacobi must also be bit-identical to
MODE_LAUNCH.  test_resident_shapes_and_masks runs the resident kernel as one CTA, one cluster of four (DSMEM items) and seven
independent CTAs (X items), and once per type mask, on stencils laid across tile boundaries; test_resident_images_are_planned_as_intended
proves those images on the CPU through the planner driver.  test_jacobi_on_shared_particles holds MODE_JACOBI to reference_jacobi on a
chain of all 13 types whose stencils share particles.  test_batch_many_replicas_and_rest_shapes runs K = 150 resident replicas and
per-replica rest shapes (launch and resident), the reference reading each replica's geometry back through replica_geometry.  Error measures: positions relative to max(|correction|, 1e-3) plus 16 fp32 ulps of |x| (the translated stencils);
velocities the same times h; lambda relative to max(|lambda|, 1e-3 / (1 + alpha)).  Each run prints the worst error per (type, edge
class, path); the thresholds below are within 4x of the worst value measured on an H100 80GB HBM3 (the measured value beside each).
Negative controls: the same gate must fail against a reference mutated by stiffness x 1.01, by lambda not reset at the second substep,
by ShapeMatching without the 1/numClusters averaging, and by one full-Q entry off by 1e-3 relative.
"""

import numpy as np
import pytest

import projection_cases as pc
from oracle import pyoracle as po

PER_CLASS = 20
# Excluded from the gate (still run, printed and held bit-identical to MODE_LAUNCH), because the fp32 build of the C restatement is as
# far from fp64 as the kernels are -- the inputs, not the kernels, decide the answer there:
#  * ShapeMatching "some_static" (20 cases): a static particle weighs 1/(0 + 1e-6) = 1e6 in the centre of mass, so x - cm cancels;
#    fp32 restatement vs fp64: 62x the correction.
#  * StrainTriangle "collinear" (20 cases): once the first sweep moves the points off their line, the strain gradients of the
#    degenerate triangle amplify rounding; fp32 restatement vs fp64 at 1x3 / 2x3: 0.29 - 1.5 of the correction (1x1: 1.6e-4).
# (type, class): (position / velocity threshold, worst measured, lambda threshold, worst measured) over every path and every GPU test of
# this file; measured on an H100 80GB HBM3 at its 700 W power limit, thresholds 3x the measured worst (2 significant digits up; an exact
# zero stays zero).  Loosened: every class whose threshold exceeds 1e-2 -- the stencils translated by 1e2 / 1e3 (O(10) fp32 ulps of |x|
# accumulated over the sweeps, against corrections that can be a few ulps of |x| themselves), the exactly planar dihedral at angle 0
# (acos at 1 loses half the digits), and the FEM / strain tets whose replica states are badly conditioned.  For each of them
# test_loosened_classes_are_fp32_conditioning checks that the fp32 restatement of the same loop on the same inputs is off from fp64 by
# at least a twelfth of what the kernels are: the inputs, not a kernel, set the error there.
TOL = {
    ('Dihedral', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('Dihedral', 'k0'): (0.00098, 3.24e-04, 0, 0.00e+00),
    ('Dihedral', 'large'): (0.00068, 2.25e-04, 0, 0.00e+00),
    ('Dihedral', 'planar0'): (0.037, 1.22e-02, 0, 0.00e+00),
    ('Dihedral', 'planar_pi'): (0.00072, 2.37e-04, 0, 0.00e+00),
    ('Dihedral', 'ratio1e3'): (0.0011, 3.50e-04, 0, 0.00e+00),
    ('Dihedral', 'shift1e2'): (0.076, 2.53e-02, 0, 0.00e+00),
    ('Dihedral', 'shift1e3'): (0.19, 6.12e-02, 0, 0.00e+00),
    ('Dihedral', 'small'): (0.0019, 6.03e-04, 0, 0.00e+00),
    ('Dihedral', 'some_static'): (0.00078, 2.57e-04, 0, 0.00e+00),
    ('Distance', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('Distance', 'coincident'): (0.00039, 1.28e-04, 0, 0.00e+00),
    ('Distance', 'k0'): (0.0011, 3.66e-04, 0, 0.00e+00),
    ('Distance', 'large'): (0.00065, 2.14e-04, 0, 0.00e+00),
    ('Distance', 'ratio1e3'): (0.00057, 1.89e-04, 0, 0.00e+00),
    ('Distance', 'shift1e2'): (0.044, 1.46e-02, 0, 0.00e+00),
    ('Distance', 'shift1e3'): (0.18, 5.71e-02, 0, 0.00e+00),
    ('Distance', 'small'): (0.0012, 3.75e-04, 0, 0.00e+00),
    ('Distance', 'some_static'): (0.00049, 1.63e-04, 0, 0.00e+00),
    ('Distance_XPBD', 'all_static'): (0, 0.00e+00, 0.0032, 1.03e-03),
    ('Distance_XPBD', 'coincident'): (0.00082, 2.70e-04, 3.2e-06, 1.06e-06),
    ('Distance_XPBD', 'k0'): (0.0013, 4.01e-04, 0.00049, 1.63e-04),
    ('Distance_XPBD', 'k1e2'): (0.0013, 4.22e-04, 0.00051, 1.68e-04),
    ('Distance_XPBD', 'k1e5'): (0.0013, 4.27e-04, 0.00023, 7.40e-05),
    ('Distance_XPBD', 'k1e9'): (0.0013, 4.11e-04, 0.00032, 1.06e-04),
    ('Distance_XPBD', 'large'): (0.0013, 4.28e-04, 0.00019, 6.27e-05),
    ('Distance_XPBD', 'ratio1e3'): (0.00073, 2.40e-04, 0.0015, 4.68e-04),
    ('Distance_XPBD', 'shift1e2'): (0.084, 2.78e-02, 0.032, 1.06e-02),
    ('Distance_XPBD', 'shift1e3'): (0.31, 1.02e-01, 0.39, 1.27e-01),
    ('Distance_XPBD', 'small'): (0.0012, 3.81e-04, 0.0019, 6.13e-04),
    ('Distance_XPBD', 'some_static'): (0.0014, 4.56e-04, 0.00088, 2.92e-04),
    ('FEMTet', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('FEMTet', 'compressed'): (0.00026, 8.39e-05, 0, 0.00e+00),
    ('FEMTet', 'inverted'): (0.13, 4.28e-02, 0, 0.00e+00),
    ('FEMTet', 'k0'): (0.0027, 8.95e-04, 0, 0.00e+00),
    ('FEMTet', 'large'): (0.18, 5.84e-02, 0, 0.00e+00),
    ('FEMTet', 'nu_out'): (0.0062, 2.05e-03, 0, 0.00e+00),
    ('FEMTet', 'ratio1e3'): (0.0018, 5.76e-04, 0, 0.00e+00),
    ('FEMTet', 'shift1e2'): (0.06, 1.99e-02, 0, 0.00e+00),
    ('FEMTet', 'shift1e3'): (0.22, 7.00e-02, 0, 0.00e+00),
    ('FEMTet', 'small'): (0.13, 4.04e-02, 0, 0.00e+00),
    ('FEMTet', 'some_static'): (0.0021, 6.90e-04, 0, 0.00e+00),
    ('FEMTet_XPBD', 'all_static'): (0, 0.00e+00, 1.2e-05, 3.78e-06),
    ('FEMTet_XPBD', 'compressed'): (0.0041, 1.36e-03, 0.0008, 2.65e-04),
    ('FEMTet_XPBD', 'inverted'): (0.00026, 8.48e-05, 0.0004, 1.31e-04),
    ('FEMTet_XPBD', 'k0'): (0.0012, 3.95e-04, 0, 0.00e+00),
    ('FEMTet_XPBD', 'k1e2'): (0.00066, 2.18e-04, 7.9e-05, 2.60e-05),
    ('FEMTet_XPBD', 'k1e5'): (0.00027, 8.78e-05, 0.00022, 7.16e-05),
    ('FEMTet_XPBD', 'k1e9'): (0.0069, 2.27e-03, 0.0029, 9.58e-04),
    ('FEMTet_XPBD', 'large'): (0.00039, 1.30e-04, 0.00026, 8.34e-05),
    ('FEMTet_XPBD', 'nu_out'): (0.00084, 2.80e-04, 0, 0.00e+00),
    ('FEMTet_XPBD', 'ratio1e3'): (0.00052, 1.71e-04, 8.1e-05, 2.68e-05),
    ('FEMTet_XPBD', 'shift1e2'): (0.16, 5.17e-02, 2.5, 8.20e-01),
    ('FEMTet_XPBD', 'shift1e3'): (0.22, 7.21e-02, 0.24, 7.96e-02),
    ('FEMTet_XPBD', 'small'): (0.0063, 2.08e-03, 0.0015, 4.77e-04),
    ('FEMTet_XPBD', 'some_static'): (0.00028, 9.09e-05, 0.0039, 1.29e-03),
    ('FEMTriangle', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('FEMTriangle', 'collinear'): (0.0015, 4.85e-04, 0, 0.00e+00),
    ('FEMTriangle', 'k0'): (0.0016, 5.09e-04, 0, 0.00e+00),
    ('FEMTriangle', 'large'): (3.8e-05, 1.24e-05, 0, 0.00e+00),
    ('FEMTriangle', 'ratio1e3'): (0.023, 7.56e-03, 0, 0.00e+00),
    ('FEMTriangle', 'shift1e2'): (0.015, 4.71e-03, 0, 0.00e+00),
    ('FEMTriangle', 'shift1e3'): (0.13, 4.29e-02, 0, 0.00e+00),
    ('FEMTriangle', 'small'): (0.02, 6.60e-03, 0, 0.00e+00),
    ('FEMTriangle', 'some_static'): (0.0031, 1.02e-03, 0, 0.00e+00),
    ('IsometricBending', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('IsometricBending', 'k0'): (0.0011, 3.37e-04, 0, 0.00e+00),
    ('IsometricBending', 'large'): (8.8e-05, 2.92e-05, 0, 0.00e+00),
    ('IsometricBending', 'ratio1e3'): (0.0028, 9.31e-04, 0, 0.00e+00),
    ('IsometricBending', 'shift1e2'): (0.013, 4.13e-03, 0, 0.00e+00),
    ('IsometricBending', 'shift1e3'): (0.13, 4.08e-02, 0, 0.00e+00),
    ('IsometricBending', 'small'): (0.0012, 3.67e-04, 0, 0.00e+00),
    ('IsometricBending', 'some_static'): (0.00056, 1.86e-04, 0, 0.00e+00),
    ('IsometricBending/fullq', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('IsometricBending/fullq', 'k0'): (0.00071, 2.36e-04, 0, 0.00e+00),
    ('IsometricBending/fullq', 'large'): (0.00016, 5.04e-05, 0, 0.00e+00),
    ('IsometricBending/fullq', 'ratio1e3'): (0.0016, 5.19e-04, 0, 0.00e+00),
    ('IsometricBending/fullq', 'small'): (0.00027, 8.87e-05, 0, 0.00e+00),
    ('IsometricBending/fullq', 'some_static'): (0.00042, 1.38e-04, 0, 0.00e+00),
    ('IsometricBending_XPBD', 'all_static'): (0, 0.00e+00, 8.5e-05, 2.82e-05),
    ('IsometricBending_XPBD', 'k0'): (0.00079, 2.60e-04, 0.00062, 2.04e-04),
    ('IsometricBending_XPBD', 'k1e2'): (0.0012, 3.98e-04, 3.7e-05, 1.23e-05),
    ('IsometricBending_XPBD', 'k1e5'): (0.00094, 3.11e-04, 0.0014, 4.55e-04),
    ('IsometricBending_XPBD', 'k1e9'): (0.00072, 2.39e-04, 0.00071, 2.36e-04),
    ('IsometricBending_XPBD', 'large'): (0.00096, 3.19e-04, 1.9e-05, 6.29e-06),
    ('IsometricBending_XPBD', 'ratio1e3'): (0.00096, 3.19e-04, 4.5e-05, 1.48e-05),
    ('IsometricBending_XPBD', 'shift1e2'): (0.067, 2.21e-02, 0.0015, 4.83e-04),
    ('IsometricBending_XPBD', 'shift1e3'): (0.34, 1.12e-01, 0.014, 4.34e-03),
    ('IsometricBending_XPBD', 'small'): (0.0011, 3.51e-04, 0.00012, 3.88e-05),
    ('IsometricBending_XPBD', 'some_static'): (0.0011, 3.37e-04, 0.0002, 6.61e-05),
    ('IsometricBending_XPBD/fullq', 'all_static'): (0, 0.00e+00, 0.00022, 7.05e-05),
    ('IsometricBending_XPBD/fullq', 'k0'): (0.00019, 6.18e-05, 0.00038, 1.24e-04),
    ('IsometricBending_XPBD/fullq', 'k1e2'): (0.0012, 3.99e-04, 0.00068, 2.26e-04),
    ('IsometricBending_XPBD/fullq', 'k1e5'): (0.00047, 1.55e-04, 0.00054, 1.80e-04),
    ('IsometricBending_XPBD/fullq', 'k1e9'): (0.002, 6.64e-04, 0.012, 3.96e-03),
    ('IsometricBending_XPBD/fullq', 'large'): (0.00095, 3.15e-04, 5.1e-05, 1.69e-05),
    ('IsometricBending_XPBD/fullq', 'ratio1e3'): (0.001, 3.33e-04, 0.00085, 2.83e-04),
    ('IsometricBending_XPBD/fullq', 'small'): (0.0013, 4.07e-04, 0.00011, 3.51e-05),
    ('IsometricBending_XPBD/fullq', 'some_static'): (0.00085, 2.81e-04, 3.7e-05, 1.21e-05),
    ('ShapeMatching', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('ShapeMatching', 'k0'): (0.00059, 1.95e-04, 0, 0.00e+00),
    ('ShapeMatching', 'large'): (3.7e-05, 1.23e-05, 0, 0.00e+00),
    ('ShapeMatching', 'ratio1e3'): (0.0019, 6.31e-04, 0, 0.00e+00),
    ('ShapeMatching', 'reflected'): (0.0015, 4.76e-04, 0, 0.00e+00),
    ('ShapeMatching', 'rotated'): (0.00015, 4.97e-05, 0, 0.00e+00),
    ('ShapeMatching', 'shift1e2'): (0.005, 1.65e-03, 0, 0.00e+00),
    ('ShapeMatching', 'shift1e3'): (0.044, 1.46e-02, 0, 0.00e+00),
    ('ShapeMatching', 'small'): (0.0016, 5.04e-04, 0, 0.00e+00),
    ('StrainTet', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('StrainTet', 'flat'): (0.0029, 9.39e-04, 0, 0.00e+00),
    ('StrainTet', 'inverted'): (1.9e-05, 6.07e-06, 0, 0.00e+00),
    ('StrainTet', 'k0'): (0.0011, 3.54e-04, 0, 0.00e+00),
    ('StrainTet', 'large'): (0.074, 2.46e-02, 0, 0.00e+00),
    ('StrainTet', 'ratio1e3'): (0.00025, 8.05e-05, 0, 0.00e+00),
    ('StrainTet', 'shift1e2'): (0.0021, 6.70e-04, 0, 0.00e+00),
    ('StrainTet', 'shift1e3'): (0.023, 7.57e-03, 0, 0.00e+00),
    ('StrainTet', 'small'): (0.0027, 8.87e-04, 0, 0.00e+00),
    ('StrainTet', 'some_static'): (6.8e-05, 2.24e-05, 0, 0.00e+00),
    ('StrainTriangle', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('StrainTriangle', 'k0'): (0.00063, 2.07e-04, 0, 0.00e+00),
    ('StrainTriangle', 'large'): (3.6e-05, 1.17e-05, 0, 0.00e+00),
    ('StrainTriangle', 'ratio1e3'): (3.6e-05, 1.19e-05, 0, 0.00e+00),
    ('StrainTriangle', 'shift1e2'): (0.0031, 1.01e-03, 0, 0.00e+00),
    ('StrainTriangle', 'shift1e3'): (0.03, 9.70e-03, 0, 0.00e+00),
    ('StrainTriangle', 'small'): (4.9e-05, 1.63e-05, 0, 0.00e+00),
    ('StrainTriangle', 'some_static'): (0.035, 1.16e-02, 0, 0.00e+00),
    ('Volume', 'all_static'): (0, 0.00e+00, 0, 0.00e+00),
    ('Volume', 'collinear'): (0.00057, 1.88e-04, 0, 0.00e+00),
    ('Volume', 'flat'): (5.6e-05, 1.85e-05, 0, 0.00e+00),
    ('Volume', 'k0'): (0.0011, 3.50e-04, 0, 0.00e+00),
    ('Volume', 'large'): (0.00037, 1.21e-04, 0, 0.00e+00),
    ('Volume', 'ratio1e3'): (0.00089, 2.96e-04, 0, 0.00e+00),
    ('Volume', 'shift1e2'): (0.049, 1.63e-02, 0, 0.00e+00),
    ('Volume', 'shift1e3'): (0.33, 1.10e-01, 0, 0.00e+00),
    ('Volume', 'small'): (0.0015, 4.71e-04, 0, 0.00e+00),
    ('Volume', 'some_static'): (0.00061, 2.02e-04, 0, 0.00e+00),
    ('Volume_XPBD', 'all_static'): (0, 0.00e+00, 5.4e-05, 1.77e-05),
    ('Volume_XPBD', 'collinear'): (0.00097, 3.23e-04, 4.1e-07, 1.34e-07),
    ('Volume_XPBD', 'flat'): (1.6e-05, 5.25e-06, 1.9e-05, 6.01e-06),
    ('Volume_XPBD', 'k0'): (0.0011, 3.41e-04, 0.00012, 3.95e-05),
    ('Volume_XPBD', 'k1e2'): (0.0013, 4.13e-04, 0.00033, 1.08e-04),
    ('Volume_XPBD', 'k1e5'): (0.00072, 2.37e-04, 0.00025, 8.22e-05),
    ('Volume_XPBD', 'k1e9'): (0.00078, 2.57e-04, 0.00016, 5.04e-05),
    ('Volume_XPBD', 'large'): (0.00038, 1.24e-04, 0.00015, 4.91e-05),
    ('Volume_XPBD', 'ratio1e3'): (0.00057, 1.87e-04, 0.00015, 4.68e-05),
    ('Volume_XPBD', 'shift1e2'): (0.059, 1.94e-02, 0.012, 3.99e-03),
    ('Volume_XPBD', 'shift1e3'): (0.35, 1.15e-01, 0.12, 3.87e-02),
    ('Volume_XPBD', 'small'): (0.0015, 4.70e-04, 0.0002, 6.45e-05),
    ('Volume_XPBD', 'some_static'): (0.00068, 2.24e-04, 0.00025, 8.15e-05),
}
#  * FEMTet and FEMTet_XPBD "flat" (20 cases each): an exactly flat tet takes the SVD branch with a zero singular value; fp32
#    restatement vs fp64: 0.16 and 0.47 of the correction (lambda 0.14) -- a gate there could not tell a zero correction from a right one.
EXCLUDED = {("ShapeMatching", "some_static"), ("StrainTriangle", "collinear"), ("FEMTet", "flat"), ("FEMTet_XPBD", "flat")}
# Excluded by construction: full-Q IsometricBending translated by 1e2 / 1e3 (make_cases(fullq=True) does not make them).  The full-Q
# form evaluates the quadratic form on absolute positions, literally as the reference does (DESIGN.md section 5): at |x| = 1e3 its
# fp32 energy is cancellation noise.

_sets = {}


def case_set(kind):
    """'main': every type's classes; 'fullq': IsometricBending with user-edited Q; built once per session."""
    if kind not in _sets:
        if kind == "main":
            _sets[kind] = pc.Cases.cat([pc.make_cases(t, PER_CLASS, 1000 + t) for t in pc.TYPES])
        else:
            _sets[kind] = pc.Cases.cat([pc.make_cases(t, PER_CLASS, 2000 + t, fullq=True) for t in pc.ISO])
    return _sets[kind]


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU: generator and restatement
# ---------------------------------------------------------------------------------------------------------------------------------
def test_every_kept_branch_is_taken():
    for kind in ("main", "fullq"):
        c = case_set(kind)
        br = c.branches()
        counts = {}
        for b, t in zip(br, c.t):
            for name in b:
                counts[(int(t), name)] = counts.get((int(t), name), 0) + 1
        types = pc.TYPES if kind == "main" else list(pc.ISO)
        for t in types:
            need = pc.REQUIRED["all"] | pc.REQUIRED.get(t, set())
            if kind == "fullq":
                need = (need - {"rank1", "shift1e2", "shift1e3"}) | {"fullq"}
            missing = [n for n in need if counts.get((t, n), 0) == 0]
            assert not missing, (kind, po.TYPE_NAMES[t], missing)
        print(kind, {po.TYPE_NAMES[t]: len(c.take(c.t == t)) for t in types})
    assert all((case_set("main").t == t).sum() >= 150 for t in pc.TYPES)


@pytest.mark.parametrize("config", pc.CONFIGS, ids=["%dx%d_v%d" % c for c in pc.CONFIGS])
def test_restatement_is_the_checkers_time_step(config):
    """The numpy loop of the reference against the checker's own TimeStepController step on a one-constraint model with gravity 0
    (the model's own parameter row), for a sample of every type and class: same x and v to 1e-9 of the scale."""
    sub, it, vel = config
    c = case_set("main").take(slice(0, None, 5))
    ck = pc.checker()
    worst = 0.0
    for i in range(len(c)):
        t = int(c.t[i])
        ck.reset()
        ck.add_triangle_model(c.x0[i], np.zeros((0, 3), np.uint32))
        for k in range(4):
            ck.set_mass(k, c.m[i, k])
        u = [c.p[i, col] for col in pc.MAT[t]] if t != po.SHAPEMATCHING else [c.p[i, 0]] + list(c.p[i, 20:24])
        assert ck.add_constraint(t, list(range(pc.NB[t])), u)
        one = c.take([i])
        one.p[0, :pc.NP[t]] = ck.constraints()[2][0][:pc.NP[t]]
        X, V, _ = pc.reference(one, sub, it, vel)
        ck.set("x", c.x[i]); ck.set("v", c.v[i]); ck.set("oldX", c.x[i]); ck.set("lastX", c.x[i])
        ck.set_params(dt=pc.DT, sub_steps=sub, max_iter=it, vel_method=vel, gravity=(0, 0, 0))
        ck.step(1)
        sc = max(np.abs(X[0] - c.x[i]).max(), 1e-3)
        e = max(np.abs(ck.get("x") - X[0]).max(), np.abs(ck.get("v") - V[0]).max() * pc.DT / sub) / sc
        worst = max(worst, e)
        # the checker's step evaluates IsometricBending's 16-term quadratic form (entries up to ~10) on absolute positions, the
        # restatement about the centroid: fp64 cancellation of up to 1e-14 |x|^2 between them at |x| = 1e3
        assert e <= 1e-9 + 1e-14 * np.abs(c.x[i]).max() ** 2 / sc, (po.TYPE_NAMES[t], c.cls[i], e)
    print("restatement vs the checker's step, worst %.1e" % worst)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
def engine(c, mode, K=1, states=None, rows=None, x0=None):
    """c's cases on private particles 4i .. 4i+3, constraint insertion id = case index; x0: rest positions (the resident tiling)."""
    from positionbaseddynamics_b200 import _capi
    eng = _capi.Engine(0)
    n = 4 * len(c)
    eng.set_particles(c.x.reshape(n, 3), c.m.reshape(n), x0=x0)
    for t in range(13):
        sel = np.nonzero(c.t == t)[0]
        if len(sel):
            b = (4 * sel[:, None] + np.arange(pc.NB[t])[None, :]).astype(np.uint32)
            eng.add_constraints(t, b, c.p[sel, :pc.NP[t]], ids=sel.astype(np.uint32))
    eng.color_first_fit()
    eng.set_mode(mode)
    if K > 1:
        eng.set_replicas(K)
        eng.set_masses(np.stack([s.m.reshape(n) for s in states]))
        for t, r in (rows or {}).items():
            if (c.t == t).any():
                eng.set_replica_materials(t, r)
    return eng


def run(eng, states, config):
    """One step of config from each state; x, v (K, N, 4, 3) and lambda (K, N)."""
    from positionbaseddynamics_b200 import _capi
    sub, it, vel = config
    K = len(states); N = len(states[0]); n = 4 * N
    x = np.stack([s.x.reshape(n, 3) for s in states]).astype(np.float32)
    v = np.stack([s.v.reshape(n, 3) for s in states]).astype(np.float32)
    for a, val in ((_capi.ATTR_X, x), (_capi.ATTR_V, v), (_capi.ATTR_OLDX, x), (_capi.ATTR_LASTX, x)):
        eng.set_attr(a, val if K > 1 else val[0])
    eng.set_params(dt=pc.DT, sub_steps=sub, max_iter=it, vel_method=vel, gravity=(0.0, 0.0, 0.0))
    eng.step(1); eng.sync()
    X = eng.get_attr(_capi.ATTR_X).reshape(K, N, 4, 3).astype(np.float64)
    V = eng.get_attr(_capi.ATTR_V).reshape(K, N, 4, 3).astype(np.float64)
    L = np.zeros((K, N))
    for t in pc.XPBD:
        if (states[0].t == t).any():
            lam, ids = eng.lambdas(t)
            L[:, ids] = np.asarray(lam, np.float64).reshape(K, -1)
    return X, V, L


def errors(c, got, ref, config):
    """Per case: position / velocity error and lambda error (0 for the non-XPBD types)."""
    sub = config[0]
    h = pc.DT / sub
    X, V, L = got
    Xr, Vr, Lr = ref
    ulp = np.spacing(np.float32(1.0)) * np.abs(c.x).reshape(len(c), -1).max(1)
    sc = np.maximum(np.abs(Xr - c.x).reshape(len(c), -1).max(1), 1e-3) + 16.0 * ulp
    ex = np.abs(X - Xr).reshape(len(c), -1).max(1) / sc
    ev = np.abs(V - Vr).reshape(len(c), -1).max(1) * h / sc
    k = np.array([c.p[i, pc.MAT[int(t)][0]] if int(t) in pc.XPBD else 0.0 for i, t in enumerate(c.t)])
    alpha = np.where(k > 0, 1.0 / np.where(k > 0, k, 1.0) / (h * h), 0.0)
    el = np.abs(L - Lr) / np.maximum(np.abs(Lr), 1e-3 / (1.0 + alpha))
    el[~np.isin(c.t, pc.XPBD)] = 0.0
    return np.maximum(ex, ev), el


def key(c, i, fullq):
    return po.TYPE_NAMES[int(c.t[i])] + ("/fullq" if fullq else ""), str(c.cls[i])


def over(c, e_pos, e_lam, fullq=False):
    """Indices of the cases outside the gate."""
    lim = [(np.inf, None, np.inf, None) if key(c, i, fullq) in EXCLUDED else TOL[key(c, i, fullq)] for i in range(len(c))]
    tol = np.array([x[0] for x in lim]); tl = np.array([x[2] for x in lim])
    return np.nonzero((e_pos > tol) | (e_lam > tl) | ~np.isfinite(e_pos) | ~np.isfinite(e_lam))[0]


class Table:
    def __init__(self):
        self.worst = {}
        self.bad = []

    def add(self, c, path, e_pos, e_lam, fullq=False):
        for i in range(len(c)):
            k = key(c, i, fullq) + (path,)
            a, b = self.worst.get(k, (0.0, 0.0))
            self.worst[k] = (max(a, float(e_pos[i])), max(b, float(e_lam[i])))

    def show(self):
        print("\nworst error per (type, class, path): position/velocity, lambda")
        for key in sorted(self.worst):
            print("  %-26s %-12s %-14s %.2e %.2e" % (key + self.worst[key]))
        per_type = {}
        for (t, _, _), (a, b) in self.worst.items():
            x, y = per_type.get(t, (0.0, 0.0)); per_type[t] = (max(x, a), max(y, b))
        print("worst per type:", {t: "%.2e / %.2e" % v for t, v in sorted(per_type.items())})
        per_class = {}
        for (t, cls, _), (a, b) in self.worst.items():
            x, y = per_class.get((t, cls), (0.0, 0.0)); per_class[(t, cls)] = (max(x, a), max(y, b))
        print("TOL-MEASURED", repr({k: v for k, v in sorted(per_class.items())}))


def _check(c, got, ref, config, path, table, fullq=False):
    """Gate one run; violations are collected in the table and asserted after it has been printed."""
    e_pos, e_lam = errors(c, got, ref, config)
    table.add(c, path, e_pos, e_lam, fullq)
    table.bad += [(po.TYPE_NAMES[int(c.t[i])], str(c.cls[i]), path, config, float(e_pos[i]), float(e_lam[i])) for i in over(c, e_pos, e_lam, fullq)]


REPLICA_ROWS_TYPES = (po.DISTANCE_XPBD, po.FEMTET, po.STRAINTRIANGLE, po.SHAPEMATCHING)


def replica_rows(K):
    """Material rows of REPLICA_ROWS_TYPES for K replicas (ShapeMatching: its stiffness)."""
    rows = {po.DISTANCE_XPBD: [[1e5], [1e2], [1e9]], po.FEMTET: [[1000.0, 0.3], [50.0, 0.1], [2e4, 0.45]],
            po.STRAINTRIANGLE: [[1.0, 0.8, 0.6, 0, 0], [0.5, 1.0, 0.3, 1, 0], [0.9, 0.2, 0.9, 1, 0]], po.SHAPEMATCHING: [[0.6], [0.25], [1.0]]}
    return {t: np.asarray(r[:K], np.float32) for t, r in rows.items()}


def with_rows(c, rows, r):
    out = pc.Cases(**{f: getattr(c, f).copy() for f in pc.Cases.FIELDS})
    for t, rr in rows.items():
        sel = c.t == t
        out.p[np.ix_(sel, pc.MAT[t])] = rr[r].astype(np.float64)
    return out


@pytest.mark.gpu
def test_projection_answers_every_path():
    from positionbaseddynamics_b200 import _capi
    table = Table()
    main, fullq = case_set("main"), case_set("fullq")
    refs = {}

    def ref(c, config, key, mut=None):
        k = (key, config, mut)
        if k not in refs:
            refs[k] = pc.reference(c, *config, mut=mut)
        return refs[k]

    # launch_multi + graph on every config: the launch result is what the other paths must reproduce bit for bit
    launch = {}
    for name, c, fq in (("main", main, False), ("fullq", fullq, True)):
        for mode, path in ((_capi.MODE_LAUNCH, "launch_multi"), (_capi.MODE_GRAPH, "graph")):
            eng = engine(c, mode)
            assert eng.get_mode()[0] == mode
            for config in pc.CONFIGS:
                got = run(eng, [c], config)
                assert eng.get_mode()[1] == mode
                _check(c, [a[0] for a in got], ref(c, config, name), config, path, table, fq)
                if mode == _capi.MODE_LAUNCH:
                    launch[(name, config)] = got
                else:
                    assert all((a == b).all() for a, b in zip(got, launch[(name, config)])), (name, path, config)
            eng.close()

    def same_as_launch(name, sel, got, config, path):
        ref_l = launch[(name, config)]
        for a, b in zip(got, ref_l):
            assert (a[0] == b[0][sel]).all(), (name, path, config)

    # one type per engine (k_project), every config; the uniform material argument on the cases of the modal row
    for name, c, fq in (("main", main, False), ("fullq", fullq, True)):
        for t in np.unique(c.t):
            sel = np.nonzero(c.t == t)[0]
            ct = c.take(sel)
            eng = engine(ct, _capi.MODE_LAUNCH)
            for config in pc.CONFIGS:
                got = run(eng, [ct], config)
                same_as_launch(name, sel, got, config, "launch_type")
                table.add(ct, "launch_type", *errors(ct, [a[0] for a in got], [a[sel] for a in ref(c, config, name)], config), fullq=fq)
            eng.close()
            rows, inv, cnt = np.unique(ct.p[:, pc.MAT[int(t)]], axis=0, return_inverse=True, return_counts=True)
            usel = sel[inv.reshape(-1) == np.argmax(cnt)]
            cu = c.take(usel)
            eng = engine(cu, _capi.MODE_LAUNCH)
            config = (2, 3, 1)
            same_as_launch(name, usel, run(eng, [cu], config), config, "uniform")
            eng.close()

    # resident (rank-one types only) and Jacobi
    for config in ((2, 3, 1), (1, 3, 0)):
        eng = engine(main, _capi.MODE_RESIDENT)
        got = run(eng, [main], config)
        assert eng.get_mode() == (_capi.MODE_RESIDENT, _capi.MODE_RESIDENT)
        same_as_launch("main", np.arange(len(main)), got, config, "resident")
        eng.close()
    for name, c, fq in (("main", main, False), ("fullq", fullq, True)):
        eng = engine(c, _capi.MODE_JACOBI)
        for config in pc.CONFIGS:
            got = run(eng, [c], config)
            assert eng.get_mode()[1] == _capi.MODE_JACOBI
            _check(c, [a[0] for a in got], ref(c, config, name), config, "jacobi", table, fq)
        eng.close()

    # batches: every replica its own state, masses and (for some types) material row; reference of replica r with row r
    K = 3
    rows = replica_rows(K)
    config = (2, 3, 1)
    for name, c, fq in (("main", main, False), ("fullq", fullq, True)):
        states = [c] + [pc.restate_state(c, 50 + r) for r in range(1, K)]
        rrefs = [pc.reference(with_rows(s, rows, r), *config) for r, s in enumerate(states)]
        solo = []
        for r, s in enumerate(states):  # the same replica alone, its row baked into the parameters: the launch bits
            eng = engine(with_rows(s, rows, r), _capi.MODE_LAUNCH)
            solo.append(run(eng, [s], config)); eng.close()
        modes = ((_capi.MODE_LAUNCH, "batch_launch"), (_capi.MODE_GRAPH, "batch_graph")) + (((_capi.MODE_RESIDENT, "batch_resident"),) if not fq else ())
        for mode, path in modes:
            eng = engine(c, mode, K, states, rows)
            got = run(eng, states, config)
            assert eng.get_mode()[1] == mode
            eng.close()
            for r in range(K):
                _check(states[r], [a[r] for a in got], rrefs[r], config, path, table, fq)
                assert all((a[r] == b[0]).all() for a, b in zip(got, solo[r])), (name, path, r)
        for t in np.unique(c.t):  # one type per engine: k_project<T, VAR, true>, launched and captured
            sel = np.nonzero(c.t == t)[0]
            for mode in (_capi.MODE_LAUNCH, _capi.MODE_GRAPH):
                eng = engine(c.take(sel), mode, K, [s.take(sel) for s in states], rows)
                got = run(eng, [s.take(sel) for s in states], config)
                assert eng.get_mode()[1] == mode
                eng.close()
                for r in range(K):
                    assert all((a[r] == b[0][sel]).all() for a, b in zip(got, solo[r])), (name, "batch_type", mode, po.TYPE_NAMES[int(t)], r)
    table.show()
    assert {k[:2] for k in table.worst} >= set(TOL) | EXCLUDED  # every gated class ran
    assert not table.bad, (len(table.bad), table.bad[:20])

    # negative controls: the gate fails against each mutated reference
    base = launch[("main", (2, 3, 1))]
    stiff_types = [t for t in pc.TYPES if t != po.FEMTET]  # PBD FEMTet's correction does not depend on the scale of E
    for mut, types in (("stiffness_1.01", stiff_types), ("no_lambda_reset", pc.XPBD), ("sm_no_average", (po.SHAPEMATCHING,))):
        wrong = ref(main, (2, 3, 1), "main", mut)
        e_pos, e_lam = errors(main, [a[0] for a in base], wrong, (2, 3, 1))
        bad = over(main, e_pos, e_lam)
        for t in types:
            assert np.isin(bad, np.nonzero(main.t == t)[0]).any(), ("negative control passed the gate", mut, po.TYPE_NAMES[t])
    wrong = ref(fullq, (1, 1, 0), "fullq", "q_off")
    e_pos, e_lam = errors(fullq, [a[0] for a in launch[("fullq", (1, 1, 0))]], wrong, (1, 1, 0))
    for t in pc.ISO:
        assert np.isin(over(fullq, e_pos, e_lam, True), np.nonzero(fullq.t == t)[0]).any(), ("negative control passed the gate", "q_off", t)


# ---------------------------------------------------------------------------------------------------------------------------------
# Resident images: three cluster shapes and the six type masks, on stencils laid across tile boundaries
# ---------------------------------------------------------------------------------------------------------------------------------
# the type subsets of the resident kernel's masks (csrc/device_image.h); the planner picks the leanest mask that covers a model
_B = lambda *ts: sum(1 << t for t in ts)
MASKS = {"ClothXPBD": ([1, 4], _B(1, 4)), "Cloth": ([0, 1, 3, 4], _B(0, 1, 3, 4)),
         "Light": ([0, 1, 2, 3, 4, 5, 7, 8], _B(0, 1, 2, 3, 4, 5, 7, 8)),
         "Fem": ([7, 8, 9, 10], _B(7, 8, 9, 10)), "Solid": ([0, 1, 3, 4, 5, 7, 8, 9, 10], _B(0, 1, 3, 4, 5, 7, 8, 9, 10, 13, 14)),
         "All": (pc.TYPES, (1 << 15) - 1)}
SHAPES = {(1, 1): "one CTA", (1, 4): "one cluster of four CTAs (DSMEM items)", (7, 1): "independent CTAs (X items)"}


def resident_set(types=pc.TYPES):
    """Every third case of the main set restricted to `types`: small enough for one tile."""
    c = case_set("main").take(slice(0, None, 3))
    return c.take(np.isin(c.t, types))


def straddling_x0(c):
    """Rest positions that put particle k of every stencil into the k-th quarter of a line: tiles follow x0 (the projections read their
    geometry from the parameters), so every stencil spans several tiles of a cluster, or several clusters."""
    N = len(c)
    x0 = np.zeros((N, 4, 3))
    x0[:, :, 0] = np.arange(4)[None, :] * N + np.arange(N)[:, None]
    return x0.reshape(-1, 3).astype(np.float32)


def plan_scene(c):
    import plan_util
    N = len(c)
    bodies = (4 * np.arange(N)[:, None] + np.arange(4)[None, :]).astype(np.uint32)
    params = c.p.astype(np.float32)
    return plan_util.Scene(4 * N, 0, c.t, bodies, params, [0, N], np.arange(N, dtype=np.uint32), straddling_x0(c))


def resident_images():
    """(name, types, forced shape or (0, 0), mask) of every resident image the GPU test runs."""
    out = [("All %dx%d" % s, pc.TYPES, s, MASKS["All"][1]) for s in SHAPES]
    return out + [("mask " + m, ts, (0, 0), mask) for m, (ts, mask) in MASKS.items()]


def test_resident_images_are_planned_as_intended(tmp_path):
    """The planner (through tests/host_shim/plan_image.cpp) admits every resident image the GPU test runs, with the intended mask, all
    plan invariants, and the intended item kinds: one CTA holds everything in its own tile, a cluster of four reaches its neighbours'
    tiles through DSMEM, independent CTAs exchange X items."""
    import plan_util
    drv = plan_util.build_driver(tmp_path)
    for name, types, shape, mask in resident_images():
        sc = plan_scene(resident_set(types))
        p = plan_util.plan(drv, tmp_path, sc, plan_util.RESIDENT, shape, tag=name.replace(" ", "_"))
        assert p["error"] == b"", (name, p["error"])
        G, C = plan_util.check_plan(sc, p, True)
        assert int(plan_util.u32(p, "res")[4]) == mask, name
        nx, nd, nl = plan_util.item_kinds(sc, p)
        print("%-16s G x C = %d x %d: %d X items, %d DSMEM items, %d own-tile items" % (name, G, C, nx, nd, nl))
        if shape == (1, 1):
            assert (G, C) == shape and nx == 0 and nd == 0
        elif shape == (1, 4):
            assert (G, C) == shape and nx == 0 and nd > 0
        elif shape == (7, 1):
            assert (G, C) == shape and nx > 0


@pytest.mark.gpu
def test_resident_shapes_and_masks():
    """Each image of test_resident_images_are_planned_as_intended on the GPU, bit-identical to MODE_LAUNCH on the same cases and
    within the gate of the fp64 reference."""
    import os
    from positionbaseddynamics_b200 import _capi
    table = Table()
    config = (2, 3, 1)
    for name, types, shape, mask in resident_images():
        c = resident_set(types)
        eng = engine(c, _capi.MODE_LAUNCH)
        want = run(eng, [c], config); eng.close()
        old = os.environ.pop("PBD_B200_CLUSTERS", None)
        if shape != (0, 0):
            os.environ["PBD_B200_CLUSTERS"] = "%dx%d" % shape
        try:
            eng = engine(c, _capi.MODE_RESIDENT, x0=straddling_x0(c))
            got = run(eng, [c], config)
            assert eng.get_mode() == (_capi.MODE_RESIDENT, _capi.MODE_RESIDENT), name
            eng.close()
        finally:
            os.environ.pop("PBD_B200_CLUSTERS", None)
            if old is not None:
                os.environ["PBD_B200_CLUSTERS"] = old
        assert all((a == b).all() for a, b in zip(got, want)), name
        _check(c, [a[0] for a in got], pc.reference(c, *config), config, "resident " + name, table)
    table.show()
    assert not table.bad, table.bad[:20]


# ---------------------------------------------------------------------------------------------------------------------------------
# Jacobi on constraints that share particles
# ---------------------------------------------------------------------------------------------------------------------------------
# worst error of the GPU against reference_jacobi over the six configurations (positions / velocities, lambda), H100 80GB HBM3 at 700 W;
# the threshold is 3x that
JACOBI_TOL = (2.1e-3, 6.82e-4, 1.1e-3, 3.46e-4)


def shared_scene():
    """A chain of constraints of all 13 types in which each stencil's first particle is the previous stencil's last one: the case is
    translated so that the two coincide (every projection is translation invariant; rank-one bending is taken about its centroid by
    the reference).  All masses 1 (ShapeMatching's frozen weights are 1 too).  Coincident Distance / Distance_XPBD and PBD Volume with
    stiffness 0 are solves that early-out: their stores still count in the kernel's average."""
    main = case_set("main")
    pick = []
    for t in pc.TYPES:
        pick += list(np.nonzero((main.t == t) & (main.cls == "large"))[0][:3])
    for t, cls in ((po.DISTANCE, "coincident"), (po.DISTANCE_XPBD, "coincident"), (po.VOLUME, "k0")):
        pick += list(np.nonzero((main.t == t) & (main.cls == cls) & (main.m == 1).all(1))[0][:2])
    pick = np.random.default_rng(7).permutation(pick)
    c = main.take(pick)
    c.x = c.x.copy()
    bodies, x, v = [], [], []
    for i in range(len(c)):
        nb = pc.NB[int(c.t[i])]
        b = list(range(len(x), len(x) + nb))
        if i:
            c.x[i] += x[bodies[-1][-1]] - c.x[i][0]  # translate onto the previous stencil's last particle
            b = [bodies[-1][-1]] + list(range(len(x), len(x) + nb - 1))
            x += list(c.x[i][1:nb]); v += list(c.v[i][1:nb])
        else:
            x += list(c.x[i][:nb]); v += list(c.v[i][:nb])
        bodies.append(b)
    x = pc._f32(np.array(x)); v = np.array(v)
    for i in range(len(c)):  # the translated positions, rounded once, as both sides see them
        c.x[i][:pc.NB[int(c.t[i])]] = x[bodies[i]]
    return c, [np.array(b) for b in bodies], x, v, np.ones(len(x))


def jacobi_errors(got, ref, x, h):
    X, V, L = got
    Xr, Vr, Lr = ref
    sc = max(np.abs(Xr - x).max(), 1e-3)
    return max(np.abs(X - Xr).max(), np.abs(V - Vr).max() * h) / sc, float((np.abs(L - Lr) / np.maximum(np.abs(Lr), 1e-3)).max())


@pytest.mark.gpu
def test_jacobi_on_shared_particles():
    from positionbaseddynamics_b200 import _capi
    c, bodies, x, v, m = shared_scene()
    assert len(np.unique(c.t)) == 13
    shared = np.bincount(np.concatenate(bodies))
    assert (shared > 1).sum() >= len(c) - 1
    eng = _capi.Engine(0)
    eng.set_particles(x, m)
    for t in range(13):
        sel = np.nonzero(c.t == t)[0]
        eng.add_constraints(t, np.array([bodies[i] for i in sel], np.uint32), c.p[sel, :pc.NP[t]], ids=sel.astype(np.uint32))
    eng.color_first_fit()
    eng.set_mode(_capi.MODE_JACOBI)
    worst = [0.0, 0.0]; control = []
    for config in pc.CONFIGS:
        sub, it, vel = config
        for a, val in ((_capi.ATTR_X, x), (_capi.ATTR_V, v), (_capi.ATTR_OLDX, x), (_capi.ATTR_LASTX, x)):
            eng.set_attr(a, val)
        eng.set_params(dt=pc.DT, sub_steps=sub, max_iter=it, vel_method=vel, gravity=(0.0, 0.0, 0.0))
        eng.step(1); eng.sync()
        assert eng.get_mode()[1] == _capi.MODE_JACOBI
        L = np.zeros(len(c))
        for t in pc.XPBD:
            lam, ids = eng.lambdas(t); L[ids] = lam
        got = (eng.get_attr(_capi.ATTR_X).astype(np.float64), eng.get_attr(_capi.ATTR_V).astype(np.float64), L)
        h = pc.DT / sub
        e = jacobi_errors(got, pc.reference_jacobi(c, bodies, len(x), x, v, m, sub, it, vel), x, h)
        worst = [max(worst[0], e[0]), max(worst[1], e[1])]
        control.append(jacobi_errors(got, pc.reference_jacobi(c, bodies, len(x), x, v, m, sub, it, vel, count_failed=False), x, h))
    eng.close()
    print("Jacobi on shared particles: worst %.2e (x, v), %.2e (lambda); without the failed solves' counts: %.2e" % (*worst, max(e[0] for e in control)))
    assert worst[0] <= JACOBI_TOL[0] and worst[1] <= JACOBI_TOL[2], worst
    # negative control: the counting rule without the early-out solves' stores fails the same gate
    assert max(e[0] for e in control) > JACOBI_TOL[0]


# ---------------------------------------------------------------------------------------------------------------------------------
# Batches: clusters stepping many replicas in turn, and per-replica rest shapes
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batch_many_replicas_and_rest_shapes():
    """K = 150 replicas in the resident mode (clusters step several replicas in turn), each with its own state and material row; and
    K = 3 replicas with rest shapes of their own (set_replica_rest_positions), launched (replica_arrays moves the geometry pointers)
    and resident (a geometry offset), the reference reading every replica's geometry back through replica_geometry."""
    from positionbaseddynamics_b200 import _capi
    table = Table()
    config = (2, 3, 1)
    rows3 = replica_rows(3)
    c = case_set("main").take(slice(0, None, 20))
    K = 150
    rows = {t: r[np.arange(K) % 3] for t, r in rows3.items()}
    states = [c] + [pc.restate_state(c, 300 + r) for r in range(1, K)]
    eng = engine(c, _capi.MODE_RESIDENT, K, states, rows)
    got = run(eng, states, config)
    assert eng.get_mode()[1] == _capi.MODE_RESIDENT and eng.replicas() == K
    eng.close()
    eng = engine(c, _capi.MODE_LAUNCH, K, states, rows)  # the per-bucket kernels, one replica per blockIdx.y: the same bits
    assert all((a == b).all() for a, b in zip(got, run(eng, states, config)))
    eng.close()
    for r in range(K):
        _check(states[r], [a[r] for a in got], pc.reference(with_rows(states[r], rows, r), *config), config, "batch_resident_K150", table)

    c = case_set("main")
    K = 3
    states = [c] + [pc.restate_state(c, 500 + r) for r in range(1, K)]
    rest = []
    for r in range(K):  # replica r's rest stencils: the cases' own, scaled about their centroids by 1 + 0.03 r
        ctr = c.x0.mean(1, keepdims=True)
        rest.append((ctr + (c.x0 - ctr) * (1.0 + 0.03 * r)).reshape(-1, 3))
    rest = np.stack(rest).astype(np.float32)
    for mode, path in ((_capi.MODE_LAUNCH, "batch_rest_launch"), (_capi.MODE_RESIDENT, "batch_rest_resident")):
        eng = engine(c, mode, K, states, rows3)
        eng.set_replica_rest_positions(rest)
        got = run(eng, states, config)
        assert eng.get_mode()[1] == mode
        geo = {t: eng.replica_geometry(t) for t in pc.TYPES}
        eng.close()
        for r in range(K):
            s = with_rows(states[r], rows3, r)
            for t in pc.TYPES:
                sel = np.nonzero(c.t == t)[0]
                s.p[np.ix_(sel, pc.GEO[t])] = geo[t][r].astype(np.float64)
            if r:
                assert not (s.p == with_rows(states[r], rows3, r).p).all()  # the replica's own geometry, not the shared one
            _check(states[r], [a[r] for a in got], pc.reference(s, *config), config, path, table)
    table.show()
    assert not table.bad, (len(table.bad), table.bad[:20])


def test_loosened_classes_are_fp32_conditioning():
    """Every class whose threshold exceeds 1e-2, and every excluded class: the fp32 restatement (the fp32 build of the C restatement's
    solver functions, positions and velocities stored in fp32) on the same inputs -- the main set in all six configurations and the
    K = 150 replica states of test_batch_many_replicas_and_rest_shapes -- is at least a twelfth as far from fp64 as the kernels were
    measured to be; for the excluded classes it is at least 0.1 of the correction."""
    f32 = po.CpuPbd("oracle", "f32") if po.available("oracle", "f32") else None
    if f32 is None:
        po.build(ref=False); f32 = po.CpuPbd("oracle", "f32")
    loose = {k for k, v in TOL.items() if v[0] > 1e-2 or v[2] > 1e-2}
    want = loose | EXCLUDED
    worst = {}

    def add(c, config, fullq=False):
        ep, el = errors(c, pc.reference(c, *config, ck=f32, fp32_state=True), pc.reference(c, *config), config)
        for i in range(len(c)):
            k = key(c, i, fullq); x, y = worst.get(k, (0.0, 0.0)); worst[k] = (max(x, ep[i]), max(y, el[i]))

    main = case_set("main")
    sel = np.array([key(main, i, False) in want for i in range(len(main))])
    fq = case_set("fullq")
    selq = np.array([key(fq, i, True) in want for i in range(len(fq))])
    for config in pc.CONFIGS:
        add(main.take(sel), config)
        if selq.any():
            add(fq.take(selq), config, True)
    c = main.take(slice(0, None, 20))
    keep = np.array([key(c, i, False) in want for i in range(len(c))])
    rows = replica_rows(3)
    for r in range(1, 150):  # the states of the GPU test: restated from the whole subset, as there
        add(with_rows(pc.restate_state(c, 300 + r), {t: v[[r % 3]] for t, v in rows.items()}, 0).take(keep), (2, 3, 1))
    for k in sorted(want):
        f = worst.get(k, (0.0, 0.0))
        if k in EXCLUDED:
            print("excluded %-40s fp32 restatement %.2e" % (k, f[0]))
            assert f[0] >= 0.1, (k, f)
        else:
            g = TOL[k]
            print("loosened %-40s fp32 restatement %.2e / %.2e, kernels %.2e / %.2e" % (k, f[0], f[1], g[1], g[3]))
            assert 12.0 * f[0] >= g[1] and (g[3] <= 1e-2 or 12.0 * f[1] >= g[3]), (k, f, g)
