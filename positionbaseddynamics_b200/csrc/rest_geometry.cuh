// positionbaseddynamics_b200/csrc/rest_geometry.cuh
//
// The rest geometry of every particle constraint type, described once for the host and the device: what the reference's
// initConstraint / init_* derive from the rest positions (rest lengths and angles, the bending Q, inverse rest matrices, areas, volumes,
// the frozen shape-matching cluster), and how those parameter columns are packed into the SoA arrays of the image.
//   * host/pbd_model.cpp builds its constraints with these functions (the host model mirror, SimulationModel::add*Constraint);
//   * host/image_plan.cpp packs the parameter table with pack_columns and factor_rank1;
//   * engine.cu's k_derive_geometry derives every replica's geometry of a batch from its own rest positions
//     (pbd_set_replica_rest_positions).
// Evaluated in double from the fp32 rest positions and rounded to float once, as the host mirror always has.  The library is compiled
// with -fmad=false, so the device evaluation has no contracted multiply-adds: IEEE add, multiply, divide and sqrt in double give the
// host's bits.  The one libm call is Dihedral's acos, whose rounding CUDA does not promise to match glibc's.
#pragma once
#include <math.h>
#include "device_image.h"

#if defined(__CUDACC__)
#define PBD_HD __host__ __device__
#else
#define PBD_HD
#endif

namespace pbdk {

constexpr double kRestEps = 1e-6;  // PositionBasedDynamics.cpp:7 (absolute, not scale aware -- kept literally)

// The geometry columns of a type: every parameter column that is not a material parameter (include/pbd_b200.h), in layout order.
// They start at column geo_first(t); the material columns sit in front of them (IsometricBending, ShapeMatching) or behind them.
PBD_HD constexpr int geo_first(int t) { return (t == PBD_ISOBENDING || t == PBD_ISOBENDING_XPBD || t == PBD_SHAPEMATCHING) ? 1 : 0; }
PBD_HD constexpr int num_geo(int t) { return type_shape(t).nParams - type_shape(t).nMat; }
constexpr int kMaxGeoColumns = 23;  // ShapeMatching: restCm[3], x0[12], w[4], numClusters[4]

struct RD3 { double x, y, z; };
PBD_HD inline RD3 rd3(const float4 &p) { return RD3{(double)p.x, (double)p.y, (double)p.z}; }
PBD_HD inline RD3 operator-(RD3 a, RD3 b) { return RD3{a.x - b.x, a.y - b.y, a.z - b.z}; }
PBD_HD inline RD3 operator-(RD3 a) { return RD3{-a.x, -a.y, -a.z}; }
PBD_HD inline double dotd(RD3 a, RD3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
PBD_HD inline RD3 crossd(RD3 a, RD3 b) { return RD3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
PBD_HD inline double normd(RD3 a) { return ::sqrt(dotd(a, a)); }
PBD_HD inline RD3 normalizedd(RD3 a) { const double z = dotd(a, a); if (z > 0) { const double s = 1.0 / ::sqrt(z); return RD3{a.x * s, a.y * s, a.z * s}; } return a; }
PBD_HD inline double cot_theta(RD3 v, RD3 w) { return dotd(v, w) / normd(crossd(v, w)); }  // MathFunctions.cpp:391-396

PBD_HD inline bool invert3d(const double m[9], double inv[9]) {
    const double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
    if (!(::fabs(det) > kRestEps)) return false;
    const double id = 1.0 / det;
    inv[0] = (m[4] * m[8] - m[5] * m[7]) * id; inv[1] = (m[2] * m[7] - m[1] * m[8]) * id; inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    inv[3] = (m[5] * m[6] - m[3] * m[8]) * id; inv[4] = (m[0] * m[8] - m[2] * m[6]) * id; inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    inv[6] = (m[3] * m[7] - m[4] * m[6]) * id; inv[7] = (m[1] * m[6] - m[0] * m[7]) * id; inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    return true;
}

// DistanceConstraint(_XPBD)::initConstraint (Constraints.cpp:1166-1181, 1211-1227): restLength
PBD_HD inline bool rest_distance(const float4 *x, float *geo) {
    geo[0] = (float)normd(rd3(x[1]) - rd3(x[0]));
    return true;
}
// DihedralConstraint::initConstraint (Constraints.cpp:1264-1300): restAngle; refused when the shared edge is shorter than 1e-6
PBD_HD inline bool rest_dihedral(const float4 *x, float *geo) {
    const RD3 p0 = rd3(x[0]), p1 = rd3(x[1]), p2 = rd3(x[2]), p3 = rd3(x[3]);
    geo[0] = 0.0f;
    if (normd(p3 - p2) < 1e-6) return false;
    const RD3 n1 = normalizedd(crossd(p2 - p0, p3 - p0)), n2 = normalizedd(crossd(p3 - p1, p2 - p1));
    double dot = dotd(n1, n2);
    dot = ::fmin(::fmax(dot, -1.0), 1.0);
    geo[0] = (float)::acos(dot);
    return true;
}
// init_IsometricBendingConstraint (PositionBasedDynamics.cpp:145-183): Q[16] = coef K K^T over the stencil x = {p2, p3, p0, p1}
PBD_HD inline bool rest_isobending(const float4 *x, float *geo) {
    const RD3 s[4] = {rd3(x[2]), rd3(x[3]), rd3(x[0]), rd3(x[1])};
    const RD3 e0 = s[1] - s[0], e1 = s[2] - s[0], e2 = s[3] - s[0], e3 = s[2] - s[1], e4 = s[3] - s[1];
    const double c01 = cot_theta(e0, e1), c02 = cot_theta(e0, e2), c03 = cot_theta(-e0, e3), c04 = cot_theta(-e0, e4);
    const double A0 = 0.5 * normd(crossd(e0, e1)), A1 = 0.5 * normd(crossd(e0, e2));
    const double coef = -3.0 / (2.0 * (A0 + A1));
    const double K[4] = {c03 + c04, c01 + c02, -c01 - c03, -c02 - c04};
    for (int j = 0; j < 4; j++)
        for (int k = 0; k < 4; k++) geo[4 * j + k] = (float)(K[j] * coef * K[k]);
    return true;
}
// init_FEMTriangleConstraint (PositionBasedDynamics.cpp:808-841): area, invRestMat[4]; refused when !(|det| > eps)
PBD_HD inline bool rest_femtriangle(const float4 *x, float *geo) {
    const RD3 p0 = rd3(x[0]), p1 = rd3(x[1]), p2 = rd3(x[2]);
    const RD3 normal0 = crossd(p1 - p0, p2 - p0);
    const double area = normd(normal0) * 0.5;
    const RD3 axis1 = normalizedd(p1 - p0), axis2 = normalizedd(crossd(normal0, axis1));
    const double q00 = dotd(p0, axis2), q01 = dotd(p0, axis1), q10 = dotd(p1, axis2), q11 = dotd(p1, axis1), q20 = dotd(p2, axis2), q21 = dotd(p2, axis1);
    const double P00 = q00 - q20, P10 = q01 - q21, P01 = q10 - q20, P11 = q11 - q21;
    const double det = P00 * P11 - P01 * P10;
    geo[0] = (float)area; geo[1] = geo[2] = geo[3] = geo[4] = 0.0f;
    if (!(::fabs(det) > kRestEps)) return false;
    geo[1] = (float)(P11 / det); geo[2] = (float)(-P01 / det); geo[3] = (float)(-P10 / det); geo[4] = (float)(P00 / det);
    return true;
}
// StrainTriangleConstraint::initConstraint (Constraints.cpp:1544-1569: the rest triangle is taken in the x-z plane)
// + init_StrainTriangleConstraint (PositionBasedDynamics.cpp:562-581): invRestMat[4]; refused when |det| < eps
PBD_HD inline bool rest_straintriangle(const float4 *x, float *geo) {
    const double a = (double)x[1].x - x[0].x, b = (double)x[2].x - x[0].x, c = (double)x[1].z - x[0].z, d = (double)x[2].z - x[0].z;
    const double det = a * d - b * c;
    geo[0] = geo[1] = geo[2] = geo[3] = 0.0f;
    if (::fabs(det) < kRestEps) return false;
    const double s = 1.0 / det;
    geo[0] = (float)(d * s); geo[1] = (float)(-b * s); geo[2] = (float)(-c * s); geo[3] = (float)(a * s);
    return true;
}
PBD_HD inline double rest_volume6(const float4 *x) {
    const RD3 p0 = rd3(x[0]), p1 = rd3(x[1]), p2 = rd3(x[2]), p3 = rd3(x[3]);
    return ::fabs((1.0 / 6.0) * dotd(p3 - p0, crossd(p2 - p0, p1 - p0)));
}
// VolumeConstraint(_XPBD)::initConstraint (Constraints.cpp:1617-1635, 1683-1702): restVolume
PBD_HD inline bool rest_volume(const float4 *x, float *geo) {
    geo[0] = (float)rest_volume6(x);
    return true;
}
// init_FEMTetraConstraint (PositionBasedDynamics.cpp:933-955): volume, invRestMat[9] of the columns p0-p3, p1-p3, p2-p3; refused when singular
PBD_HD inline bool rest_femtet(const float4 *x, float *geo) {
    geo[0] = (float)rest_volume6(x);
    const RD3 p3 = rd3(x[3]), a = rd3(x[0]) - p3, b = rd3(x[1]) - p3, c = rd3(x[2]) - p3;
    const double m[9] = {a.x, b.x, c.x, a.y, b.y, c.y, a.z, b.z, c.z};
    double inv[9];
    const bool ok = invert3d(m, inv);
    for (int k = 0; k < 9; k++) geo[1 + k] = ok ? (float)inv[k] : 0.0f;
    return ok;
}
// init_StrainTetraConstraint (PositionBasedDynamics.cpp:691-710): invRestMat[9] of the columns p1-p0, p2-p0, p3-p0; refused when singular
PBD_HD inline bool rest_straintet(const float4 *x, float *geo) {
    const RD3 p0 = rd3(x[0]), a = rd3(x[1]) - p0, b = rd3(x[2]) - p0, c = rd3(x[3]) - p0;
    const double m[9] = {a.x, b.x, c.x, a.y, b.y, c.y, a.z, b.z, c.z};
    double inv[9];
    const bool ok = invert3d(m, inv);
    for (int k = 0; k < 9; k++) geo[k] = ok ? (float)inv[k] : 0.0f;
    return ok;
}
// ShapeMatchingConstraint::initConstraint (Constraints.cpp:1985-2001) + init_ShapeMatchingConstraint (PositionBasedDynamics.cpp:479-497):
// restCm[3], x0[4][3], w[4] -- the rest positions and inverse masses (x[i].w) are frozen into the constraint; refused when wsum == 0.
// (numClusters, the last four geometry columns, is topology: the caller copies it.)
PBD_HD inline bool rest_shapematching(const float4 *x, float *geo) {
    double cm[3] = {0, 0, 0}, wsum = 0.0;
    for (int i = 0; i < 4; i++) {
        const float p[3] = {x[i].x, x[i].y, x[i].z};
        const float w = x[i].w;
        const double wi = 1.0 / ((double)w + kRestEps);
        for (int k = 0; k < 3; k++) { cm[k] += p[k] * wi; geo[3 + 3 * i + k] = p[k]; }
        wsum += wi;
        geo[15 + i] = w;
    }
    const bool ok = wsum != 0.0;
    for (int k = 0; k < 3; k++) geo[k] = ok ? (float)(cm[k] / wsum) : 0.0f;
    return ok;
}

// The geometry columns of a constraint of type t (num_geo(t) floats; ShapeMatching: all but numClusters) from the rest positions of its
// bodies, and whether the reference's initConstraint accepts them.  Joints: no rest geometry of particles (false).
PBD_HD inline bool rest_geometry(int t, const float4 *x, float *geo) {
    switch (t) {
    case PBD_DISTANCE: case PBD_DISTANCE_XPBD: return rest_distance(x, geo);
    case PBD_DIHEDRAL: return rest_dihedral(x, geo);
    case PBD_ISOBENDING: case PBD_ISOBENDING_XPBD: return rest_isobending(x, geo);
    case PBD_FEMTRIANGLE: return rest_femtriangle(x, geo);
    case PBD_STRAINTRIANGLE: return rest_straintriangle(x, geo);
    case PBD_VOLUME: case PBD_VOLUME_XPBD: return rest_volume(x, geo);
    case PBD_FEMTET: case PBD_FEMTET_XPBD: return rest_femtet(x, geo);
    case PBD_STRAINTET: return rest_straintet(x, geo);
    case PBD_SHAPEMATCHING: return rest_shapematching(x, geo);
    default: return false;
    }
}

// Q (row-major 4x4, solver order) = -Kp Kp^T ?  Returns true and Kp when the rank-one negative-semidefinite form of
// init_IsometricBendingConstraint (PositionBasedDynamics.cpp:169-180) reproduces Q to fp32 accuracy.
PBD_HD inline bool factor_rank1(const float *Q, float Kp[4]) {
    int piv = 0; float best = 0.0f, maxAbs = 0.0f;
    for (int j = 0; j < 4; j++) { if (-Q[5 * j] > best) { best = -Q[5 * j]; piv = j; } }
    for (int i = 0; i < 16; i++) { const float a = ::fabsf(Q[i]); maxAbs = (maxAbs < a) ? a : maxAbs; }
    if (maxAbs == 0.0f) { Kp[0] = Kp[1] = Kp[2] = Kp[3] = 0.0f; return true; }
    if (!(best > 0.0f)) return false;
    const double kp = ::sqrt((double)best);
    double K[4];
    for (int k = 0; k < 4; k++) K[k] = -(double)Q[4 * piv + k] / kp;
    for (int j = 0; j < 4; j++)
        for (int k = 0; k < 4; k++)
            if (::fabs((double)Q[4 * j + k] + K[j] * K[k]) > 1e-5 * (double)maxAbs) return false;
    for (int k = 0; k < 4; k++) Kp[k] = (float)K[k];
    return true;
}

// Parameter columns (include/pbd_b200.h) of a type's SoA arrays: float4 geometry array k = columns gv[k][0..3], scalar geometry
// array k = column gs[k], material slot k = column mat[k]; -1 = zero-filled component, or no such array / slot.
// IsometricBending: the full-Q layout (variant 1); the rank-one layout (variant 0) holds factor_rank1's Kp in gv[0] instead.
struct PackColumns { signed char gv[kMaxGeoV][4], gs[kMaxGeoS], mat[kMaxMat]; };
PBD_HD inline PackColumns pack_columns(int t) {
    PackColumns p;
    for (int k = 0; k < kMaxGeoV; k++) p.gv[k][0] = p.gv[k][1] = p.gv[k][2] = p.gv[k][3] = -1;
    for (int k = 0; k < kMaxGeoS; k++) p.gs[k] = -1;
    for (int k = 0; k < kMaxMat; k++) p.mat[k] = -1;
    auto gv = [&](int k, int c0, int c1, int c2, int c3) { p.gv[k][0] = (signed char)c0; p.gv[k][1] = (signed char)c1; p.gv[k][2] = (signed char)c2; p.gv[k][3] = (signed char)c3; };
    auto mat = [&](int first, int count) { for (int k = 0; k < count; k++) p.mat[k] = (signed char)(first + k); };
    switch (t) {
    case PBD_DISTANCE: case PBD_DISTANCE_XPBD: case PBD_DIHEDRAL: case PBD_VOLUME: case PBD_VOLUME_XPBD: p.gs[0] = 0; mat(1, 1); break;
    case PBD_ISOBENDING: case PBD_ISOBENDING_XPBD: for (int r = 0; r < 4; r++) gv(r, 1 + 4 * r, 2 + 4 * r, 3 + 4 * r, 4 + 4 * r); mat(0, 1); break;
    case PBD_FEMTRIANGLE: p.gs[0] = 0; gv(0, 1, 2, 3, 4); mat(5, 5); break;
    case PBD_STRAINTRIANGLE: gv(0, 0, 1, 2, 3); mat(4, 5); break;
    case PBD_FEMTET: case PBD_FEMTET_XPBD: gv(0, 1, 2, 3, 4); gv(1, 5, 6, 7, 8); p.gs[0] = 9; p.gs[1] = 0; mat(10, 2); break;
    case PBD_STRAINTET: gv(0, 0, 1, 2, 3); gv(1, 4, 5, 6, 7); p.gs[0] = 8; mat(9, 4); break;
    // local connectors (jointInfo columns 0 [and 1]); the global columns are recomputed per solve
    case PBD_BALLJOINT: gv(0, 0, 1, 2, -1); gv(1, 3, 4, 5, -1); break;
    case PBD_RB_PARTICLE_BALLJOINT: gv(0, 0, 1, 2, -1); break;
    // restCm | x0[0..3] packed in 3 float4 | w | numClusters ; stiffness is the material slot
    case PBD_SHAPEMATCHING: gv(0, 1, 2, 3, -1); for (int k = 1; k < 6; k++) gv(k, 4 * k, 4 * k + 1, 4 * k + 2, 4 * k + 3); mat(0, 1); break;
    default: break;
    }
    return p;
}

}  // namespace pbdk
