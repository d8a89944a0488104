/* oracle/pbd_oracle.c -- TEST INFRASTRUCTURE, not product code (see pbd_oracle.h).
 *
 * CPU restatement, in plain C, of the reference's PBD/XPBD constraint-projection path.  Every function
 * cites the reference file:line it follows (paths relative to the reference root).  Written from the
 * reference's behaviour; data structures are flat arrays, not the reference's class hierarchy.
 *
 * PINNING: the reference has no tests for this path.  This file is pinned against the reference itself
 * (oracle/_ref, built from the unmodified sources) by tests/test_oracle_vs_ref.py and against the
 * fixtures generated from it under tests/golden/ by tests/test_oracle_golden.py.
 */
#define _POSIX_C_SOURCE 199309L
#include "pbd_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#ifdef ORACLE_DOUBLE
#define RSQRT sqrt
#define RFABS fabs
#define RACOS acos
#define REAL_MAX DBL_MAX
#else
#define RSQRT sqrtf
#define RFABS fabsf
#define RACOS acosf
#define REAL_MAX FLT_MAX
#endif
#define R(x) ((real)(x))
#define NOFACE 0xffffffffu
#define MIN_PARALLEL_SIZE 64 /* Common/Common.h:8 */

static const real EPS = R(1e-6); /* PositionBasedDynamics.cpp:7, XPBD.cpp:8 */

/* ------------------------------------------------------------------------------------------------ */
/* small vector helpers                                                                              */
/* ------------------------------------------------------------------------------------------------ */
typedef struct { real v[3]; } vec3;
static inline vec3 V(real x, real y, real z) { vec3 r = {{x, y, z}}; return r; }
static inline vec3 vadd(vec3 a, vec3 b) { return V(a.v[0] + b.v[0], a.v[1] + b.v[1], a.v[2] + b.v[2]); }
static inline vec3 vsub(vec3 a, vec3 b) { return V(a.v[0] - b.v[0], a.v[1] - b.v[1], a.v[2] - b.v[2]); }
static inline vec3 vmul(vec3 a, real s) { return V(a.v[0] * s, a.v[1] * s, a.v[2] * s); }
static inline vec3 vneg(vec3 a) { return V(-a.v[0], -a.v[1], -a.v[2]); }
static inline real vdot(vec3 a, vec3 b) { return a.v[0] * b.v[0] + a.v[1] * b.v[1] + a.v[2] * b.v[2]; }
static inline vec3 vcross(vec3 a, vec3 b) {
    return V(a.v[1] * b.v[2] - a.v[2] * b.v[1], a.v[2] * b.v[0] - a.v[0] * b.v[2], a.v[0] * b.v[1] - a.v[1] * b.v[0]);
}
static inline real vsq(vec3 a) { return vdot(a, a); }
static inline real vnorm(vec3 a) { return RSQRT(vsq(a)); }
/* Eigen's normalize(): leaves a zero vector untouched (extern/eigen/Eigen/src/Core/Dot.h:145-151) */
static inline vec3 vnormalize(vec3 a) {
    real z = vsq(a);
    if (z > R(0.0)) return vmul(a, R(1.0) / RSQRT(z));
    return a;
}
static const vec3 VZERO = {{0, 0, 0}};

typedef struct { real m[3][3]; } mat3;
static inline real det3(const mat3 *a) {
    return a->m[0][0] * (a->m[1][1] * a->m[2][2] - a->m[1][2] * a->m[2][1]) -
           a->m[0][1] * (a->m[1][0] * a->m[2][2] - a->m[1][2] * a->m[2][0]) +
           a->m[0][2] * (a->m[1][0] * a->m[2][1] - a->m[1][1] * a->m[2][0]);
}
static inline mat3 inv3(const mat3 *a, real det) {
    mat3 r;
    real id = R(1.0) / det;
    r.m[0][0] = (a->m[1][1] * a->m[2][2] - a->m[1][2] * a->m[2][1]) * id;
    r.m[0][1] = (a->m[0][2] * a->m[2][1] - a->m[0][1] * a->m[2][2]) * id;
    r.m[0][2] = (a->m[0][1] * a->m[1][2] - a->m[0][2] * a->m[1][1]) * id;
    r.m[1][0] = (a->m[1][2] * a->m[2][0] - a->m[1][0] * a->m[2][2]) * id;
    r.m[1][1] = (a->m[0][0] * a->m[2][2] - a->m[0][2] * a->m[2][0]) * id;
    r.m[1][2] = (a->m[0][2] * a->m[1][0] - a->m[0][0] * a->m[1][2]) * id;
    r.m[2][0] = (a->m[1][0] * a->m[2][1] - a->m[1][1] * a->m[2][0]) * id;
    r.m[2][1] = (a->m[0][1] * a->m[2][0] - a->m[0][0] * a->m[2][1]) * id;
    r.m[2][2] = (a->m[0][0] * a->m[1][1] - a->m[0][1] * a->m[1][0]) * id;
    return r;
}
static inline mat3 mul3(const mat3 *a, const mat3 *b) {
    mat3 r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r.m[i][j] = a->m[i][0] * b->m[0][j] + a->m[i][1] * b->m[1][j] + a->m[i][2] * b->m[2][j];
    return r;
}
static inline mat3 transpose3(const mat3 *a) {
    mat3 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[i][j] = a->m[j][i];
    return r;
}
static inline vec3 mcol(const mat3 *a, int c) { return V(a->m[0][c], a->m[1][c], a->m[2][c]); }

/* quaternion (w, x, y, z); Eigen semantics for product, conjugate, matrix() and normalize() */
typedef struct { real w, x, y, z; } quat;
static inline quat qmul(quat a, quat b) {
    quat r;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
    r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
    return r;
}
static inline quat qconj(quat a) { quat r = {a.w, -a.x, -a.y, -a.z}; return r; }
static inline quat qnormalize(quat a) {
    real n = RSQRT(a.w * a.w + a.x * a.x + a.y * a.y + a.z * a.z);
    quat r = {a.w / n, a.x / n, a.y / n, a.z / n};
    return r;
}
static inline mat3 qmatrix(quat q) {
    mat3 m;
    const real tx = R(2.0) * q.x, ty = R(2.0) * q.y, tz = R(2.0) * q.z;
    const real twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    m.m[0][0] = R(1.0) - (tyy + tzz); m.m[0][1] = txy - twz; m.m[0][2] = txz + twy;
    m.m[1][0] = txy + twz; m.m[1][1] = R(1.0) - (txx + tzz); m.m[1][2] = tyz - twx;
    m.m[2][0] = txz - twy; m.m[2][1] = tyz + twx; m.m[2][2] = R(1.0) - (txx + tyy);
    return m;
}
static inline vec3 mvec(const mat3 *a, vec3 v) {
    return V(a->m[0][0] * v.v[0] + a->m[0][1] * v.v[1] + a->m[0][2] * v.v[2], a->m[1][0] * v.v[0] + a->m[1][1] * v.v[1] + a->m[1][2] * v.v[2],
             a->m[2][0] * v.v[0] + a->m[2][1] * v.v[1] + a->m[2][2] * v.v[2]);
}

/* ------------------------------------------------------------------------------------------------ */
/* MathFunctions (PositionBasedDynamics/MathFunctions.cpp)                                           */
/* ------------------------------------------------------------------------------------------------ */

/* MathFunctions::cotTheta, MathFunctions.cpp:391-396 */
static real cot_theta(vec3 v, vec3 w) { return vdot(v, w) / vnorm(vcross(v, w)); }

/* MathFunctions::jacobiRotate, MathFunctions.cpp:11-43 */
static void jacobi_rotate(mat3 *A, mat3 *Rm, int p, int q) {
    if (A->m[p][q] == R(0.0)) return;
    real d = (A->m[p][p] - A->m[q][q]) / (R(2.0) * A->m[p][q]);
    real t = R(1.0) / (RFABS(d) + RSQRT(d * d + R(1.0)));
    if (d < R(0.0)) t = -t;
    real c = R(1.0) / RSQRT(t * t + 1);
    real s = t * c;
    A->m[p][p] += t * A->m[p][q];
    A->m[q][q] -= t * A->m[p][q];
    A->m[p][q] = A->m[q][p] = R(0.0);
    for (int k = 0; k < 3; k++) {
        if (k != p && k != q) {
            real Akp = c * A->m[k][p] + s * A->m[k][q];
            real Akq = -s * A->m[k][p] + c * A->m[k][q];
            A->m[k][p] = A->m[p][k] = Akp;
            A->m[k][q] = A->m[q][k] = Akq;
        }
    }
    for (int k = 0; k < 3; k++) {
        real Rkp = c * Rm->m[k][p] + s * Rm->m[k][q];
        real Rkq = -s * Rm->m[k][p] + c * Rm->m[k][q];
        Rm->m[k][p] = Rkp;
        Rm->m[k][q] = Rkq;
    }
}

/* MathFunctions::eigenDecomposition, MathFunctions.cpp:46-75 (<=10 Jacobi rotations, 1e-15 stop) */
static void eigen_decomposition(const mat3 *A, mat3 *vecs, vec3 *vals) {
    const real epsilon = R(1e-15);
    mat3 D = *A;
    memset(vecs, 0, sizeof(*vecs));
    vecs->m[0][0] = vecs->m[1][1] = vecs->m[2][2] = R(1.0);
    for (int iter = 0; iter < 10; iter++) {
        int p = 0, q = 1;
        real mx = RFABS(D.m[0][1]);
        real a = RFABS(D.m[0][2]);
        if (a > mx) { p = 0; q = 2; mx = a; }
        a = RFABS(D.m[1][2]);
        if (a > mx) { p = 1; q = 2; mx = a; }
        if (mx < epsilon) break;
        jacobi_rotate(&D, vecs, p, q);
    }
    vals->v[0] = D.m[0][0]; vals->v[1] = D.m[1][1]; vals->v[2] = D.m[2][2];
}

/* MathFunctions::svdWithInversionHandling, MathFunctions.cpp:261-388 */
static void svd_inversion(const mat3 *A, vec3 *sigma, mat3 *U, mat3 *VT) {
    mat3 At = transpose3(A);
    mat3 AtA = mul3(&At, A);
    mat3 Vm; vec3 S;
    eigen_decomposition(&AtA, &Vm, &S);
    if (det3(&Vm) < R(0.0)) {
        real minL = REAL_MAX; int pos = 0;
        for (int l = 0; l < 3; l++) if (S.v[l] < minL) { pos = l; minL = S.v[l]; }
        for (int r = 0; r < 3; r++) Vm.m[r][pos] = -Vm.m[r][pos];
    }
    for (int l = 0; l < 3; l++) if (S.v[l] < R(0.0)) S.v[l] = R(0.0);
    for (int l = 0; l < 3; l++) sigma->v[l] = RSQRT(S.v[l]);
    *VT = transpose3(&Vm);

    int chk = 0, pos = 0;
    for (int l = 0; l < 3; l++) if (RFABS(sigma->v[l]) < 1.0e-4) { pos = l; chk++; }
    if (chk > 0) {
        if (chk > 1) {
            memset(U, 0, sizeof(*U));
            U->m[0][0] = U->m[1][1] = U->m[2][2] = R(1.0);
        } else {
            *U = mul3(A, &Vm);
            for (int l = 0; l < 3; l++)
                if (l != pos) for (int m = 0; m < 3; m++) U->m[m][l] *= R(1.0) / sigma->v[l];
            vec3 v[2]; int idx = 0;
            for (int l = 0; l < 3; l++) if (l != pos) v[idx++] = mcol(U, l);
            vec3 vec = vnormalize(vcross(v[0], v[1]));
            for (int m = 0; m < 3; m++) U->m[m][pos] = vec.v[m];
        }
    } else {
        vec3 si = V(R(1.0) / sigma->v[0], R(1.0) / sigma->v[1], R(1.0) / sigma->v[2]);
        *U = mul3(A, &Vm);
        for (int l = 0; l < 3; l++) for (int m = 0; m < 3; m++) U->m[m][l] *= si.v[l];
    }
    if (det3(U) < R(0.0)) {
        real minL = REAL_MAX; int p2 = 0;
        for (int l = 0; l < 3; l++) if (sigma->v[l] < minL) { p2 = l; minL = sigma->v[l]; }
        sigma->v[p2] = -sigma->v[p2];
        for (int m = 0; m < 3; m++) U->m[m][p2] = -U->m[m][p2];
    }
}

/* MathFunctions::oneNorm / infNorm, MathFunctions.cpp:148-178 */
static real one_norm(const mat3 *A) {
    real m = R(0.0);
    for (int c = 0; c < 3; c++) { real s = RFABS(A->m[0][c]) + RFABS(A->m[1][c]) + RFABS(A->m[2][c]); if (c == 0 || s > m) m = s; }
    return m;
}
static real inf_norm(const mat3 *A) {
    real m = R(0.0);
    for (int r = 0; r < 3; r++) { real s = RFABS(A->m[r][0]) + RFABS(A->m[r][1]) + RFABS(A->m[r][2]); if (r == 0 || s > m) m = s; }
    return m;
}
static inline vec3 mrow(const mat3 *a, int r) { return V(a->m[r][0], a->m[r][1], a->m[r][2]); }
static inline void set_row(mat3 *a, int r, vec3 v) { a->m[r][0] = v.v[0]; a->m[r][1] = v.v[1]; a->m[r][2] = v.v[2]; }

/* MathFunctions::polarDecompositionStable, MathFunctions.cpp:180-255 */
static void polar_decomposition_stable(const mat3 *M, real tolerance, mat3 *Rm) {
    mat3 Mt = transpose3(M);
    real Mone = one_norm(M), Minf = inf_norm(M), Eone;
    mat3 MadjTt, Et;
    do {
        set_row(&MadjTt, 0, vcross(mrow(&Mt, 1), mrow(&Mt, 2)));
        set_row(&MadjTt, 1, vcross(mrow(&Mt, 2), mrow(&Mt, 0)));
        set_row(&MadjTt, 2, vcross(mrow(&Mt, 0), mrow(&Mt, 1)));
        real det = Mt.m[0][0] * MadjTt.m[0][0] + Mt.m[0][1] * MadjTt.m[0][1] + Mt.m[0][2] * MadjTt.m[0][2];
        if (RFABS(det) < 1.0e-12) {
            int index = -1;
            for (int i = 0; i < 3; i++) { if (vsq(mrow(&MadjTt, i)) > 1.0e-12) { index = i; break; } }
            if (index < 0) { memset(Rm, 0, sizeof(*Rm)); Rm->m[0][0] = Rm->m[1][1] = Rm->m[2][2] = R(1.0); return; }
            set_row(&Mt, index, vcross(mrow(&Mt, (index + 1) % 3), mrow(&Mt, (index + 2) % 3)));
            set_row(&MadjTt, (index + 1) % 3, vcross(mrow(&Mt, (index + 2) % 3), mrow(&Mt, index)));
            set_row(&MadjTt, (index + 2) % 3, vcross(mrow(&Mt, index), mrow(&Mt, (index + 1) % 3)));
            mat3 M2 = transpose3(&Mt);
            Mone = one_norm(&M2); Minf = inf_norm(&M2);
            det = Mt.m[0][0] * MadjTt.m[0][0] + Mt.m[0][1] * MadjTt.m[0][1] + Mt.m[0][2] * MadjTt.m[0][2];
        }
        const real MadjTone = one_norm(&MadjTt), MadjTinf = inf_norm(&MadjTt);
        const real gamma = RSQRT(RSQRT((MadjTone * MadjTinf) / (Mone * Minf)) / RFABS(det));
        const real g1 = gamma * R(0.5);
        const real g2 = R(0.5) / (gamma * det);
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                Et.m[i][j] = Mt.m[i][j];
                Mt.m[i][j] = g1 * Mt.m[i][j] + g2 * MadjTt.m[i][j];
                Et.m[i][j] -= Mt.m[i][j];
            }
        Eone = one_norm(&Et);
        Mone = one_norm(&Mt); Minf = inf_norm(&Mt);
    } while (Eone > Mone * tolerance);
    *Rm = transpose3(&Mt);
}

/* ------------------------------------------------------------------------------------------------ */
/* Stateless solver functions                                                                        */
/* ------------------------------------------------------------------------------------------------ */

/* PositionBasedDynamics::solve_DistanceConstraint, PositionBasedDynamics.cpp:13-34 */
static int solve_distance(vec3 p0, real w0, vec3 p1, real w1, real restLength, real k, vec3 *c0, vec3 *c1) {
    real wSum = w0 + w1;
    if (wSum == R(0.0)) return 0;
    vec3 n = vsub(p1, p0);
    real d = vnorm(n);
    n = vnormalize(n);
    /* stiffness * n * (d - restLength) / wSum, evaluated left to right */
    vec3 corr = vmul(vmul(n, k), d - restLength);
    corr = V(corr.v[0] / wSum, corr.v[1] / wSum, corr.v[2] / wSum);
    *c0 = vmul(corr, w0);
    *c1 = vmul(corr, -w1);
    return 1;
}

/* XPBD::solve_DistanceConstraint, XPBD.cpp:14-60 */
static int solve_distance_xpbd(vec3 p0, real w0, vec3 p1, real w1, real restLength, real k, real dt, real *lambda,
                               vec3 *c0, vec3 *c1) {
    real K = w0 + w1;
    vec3 n = vsub(p0, p1);
    real d = vnorm(n);
    real C = d - restLength;
    if (d > R(1e-6)) n = V(n.v[0] / d, n.v[1] / d, n.v[2] / d);
    else { *c0 = VZERO; *c1 = VZERO; return 1; }
    real alpha = R(0.0);
    if (k != R(0.0)) { alpha = R(1.0) / (k * dt * dt); K += alpha; }
    real Kinv;
    if (RFABS(K) > R(1e-6)) Kinv = R(1.0) / K;
    else { *c0 = VZERO; *c1 = VZERO; return 1; }
    const real dl = -Kinv * (C + alpha * *lambda);
    *lambda += dl;
    vec3 pt = vmul(n, dl);
    *c0 = vmul(pt, w0);
    *c1 = vmul(pt, -w1);
    return 1;
}

/* PositionBasedDynamics::solve_DihedralConstraint, PositionBasedDynamics.cpp:37-102 */
static int solve_dihedral(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, real restAngle,
                          real k, vec3 *c0, vec3 *c1, vec3 *c2, vec3 *c3) {
    if (w0 == R(0.0) && w1 == R(0.0)) return 0;
    vec3 e = vsub(p3, p2);
    real elen = vnorm(e);
    if (elen < EPS) return 0;
    real invElen = R(1.0) / elen;
    vec3 n1 = vcross(vsub(p2, p0), vsub(p3, p0)); { real s = vsq(n1); n1 = V(n1.v[0] / s, n1.v[1] / s, n1.v[2] / s); }
    vec3 n2 = vcross(vsub(p3, p1), vsub(p2, p1)); { real s = vsq(n2); n2 = V(n2.v[0] / s, n2.v[1] / s, n2.v[2] / s); }
    vec3 d0 = vmul(n1, elen);
    vec3 d1 = vmul(n2, elen);
    vec3 d2 = vadd(vmul(n1, vdot(vsub(p0, p3), e) * invElen), vmul(n2, vdot(vsub(p1, p3), e) * invElen));
    vec3 d3 = vadd(vmul(n1, vdot(vsub(p2, p0), e) * invElen), vmul(n2, vdot(vsub(p2, p1), e) * invElen));
    n1 = vnormalize(n1);
    n2 = vnormalize(n2);
    real dot = vdot(n1, n2);
    if (dot < R(-1.0)) dot = R(-1.0);
    if (dot > R(1.0)) dot = R(1.0);
    real phi = RACOS(dot);
    real lambda = w0 * vsq(d0) + w1 * vsq(d1) + w2 * vsq(d2) + w3 * vsq(d3);
    if (lambda == R(0.0)) return 0;
    lambda = (phi - restAngle) / lambda * k;
    if (vdot(vcross(n1, n2), e) > R(0.0)) lambda = -lambda;
    *c0 = vmul(d0, -w0 * lambda);
    *c1 = vmul(d1, -w1 * lambda);
    *c2 = vmul(d2, -w2 * lambda);
    *c3 = vmul(d3, -w3 * lambda);
    return 1;
}

/* PositionBasedDynamics::solve_VolumeConstraint, PositionBasedDynamics.cpp:104-142 */
static int solve_volume(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, real restVolume, real k,
                        vec3 *c0, vec3 *c1, vec3 *c2, vec3 *c3) {
    real volume = R(1.0 / 6.0) * vdot(vcross(vsub(p1, p0), vsub(p2, p0)), vsub(p3, p0));
    *c0 = *c1 = *c2 = *c3 = VZERO;
    if (k == R(0.0)) return 0;
    vec3 g0 = vcross(vsub(p1, p2), vsub(p3, p2));
    vec3 g1 = vcross(vsub(p2, p0), vsub(p3, p0));
    vec3 g2 = vcross(vsub(p0, p1), vsub(p3, p1));
    vec3 g3 = vcross(vsub(p1, p0), vsub(p2, p0));
    real lambda = w0 * vsq(g0) + w1 * vsq(g1) + w2 * vsq(g2) + w3 * vsq(g3);
    if (RFABS(lambda) < EPS) return 0;
    lambda = k * (volume - restVolume) / lambda;
    *c0 = vmul(g0, -lambda * w0);
    *c1 = vmul(g1, -lambda * w1);
    *c2 = vmul(g2, -lambda * w2);
    *c3 = vmul(g3, -lambda * w3);
    return 1;
}

/* XPBD::solve_VolumeConstraint, XPBD.cpp:63-109 */
static int solve_volume_xpbd(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, real restVolume,
                             real k, real dt, real *lambda, vec3 *c0, vec3 *c1, vec3 *c2, vec3 *c3) {
    real volume = R(1.0 / 6.0) * vdot(vcross(vsub(p1, p0), vsub(p2, p0)), vsub(p3, p0));
    *c0 = *c1 = *c2 = *c3 = VZERO;
    vec3 g0 = vcross(vsub(p1, p2), vsub(p3, p2));
    vec3 g1 = vcross(vsub(p2, p0), vsub(p3, p0));
    vec3 g2 = vcross(vsub(p0, p1), vsub(p3, p1));
    vec3 g3 = vcross(vsub(p1, p0), vsub(p2, p0));
    real K = w0 * vsq(g0) + w1 * vsq(g1) + w2 * vsq(g2) + w3 * vsq(g3);
    real alpha = R(0.0);
    if (k != R(0.0)) { alpha = R(1.0) / (k * dt * dt); K += alpha; }
    if (RFABS(K) < EPS) return 0;
    const real C = volume - restVolume;
    const real dl = -(C + alpha * *lambda) / K;
    *lambda += dl;
    *c0 = vmul(g0, dl * w0);
    *c1 = vmul(g1, dl * w1);
    *c2 = vmul(g2, dl * w2);
    *c3 = vmul(g3, dl * w3);
    return 1;
}

/* PositionBasedDynamics::init_IsometricBendingConstraint, PositionBasedDynamics.cpp:145-183
 * (XPBD::init_IsometricBendingConstraint, XPBD.cpp:112-150, is identical).  Q row-major 4x4. */
static int init_isobending(vec3 p0, vec3 p1, vec3 p2, vec3 p3, real *Q) {
    const vec3 x[4] = {p2, p3, p0, p1};
    const vec3 e0 = vsub(x[1], x[0]);
    const vec3 e1 = vsub(x[2], x[0]);
    const vec3 e2 = vsub(x[3], x[0]);
    const vec3 e3 = vsub(x[2], x[1]);
    const vec3 e4 = vsub(x[3], x[1]);
    const real c01 = cot_theta(e0, e1);
    const real c02 = cot_theta(e0, e2);
    const real c03 = cot_theta(vneg(e0), e3);
    const real c04 = cot_theta(vneg(e0), e4);
    const real A0 = R(0.5) * vnorm(vcross(e0, e1));
    const real A1 = R(0.5) * vnorm(vcross(e0, e2));
    const real coef = -3.f / (2.f * (A0 + A1));
    const real K[4] = {c03 + c04, c01 + c02, -c01 - c03, -c02 - c04};
    const real K2[4] = {coef * K[0], coef * K[1], coef * K[2], coef * K[3]};
    for (int j = 0; j < 4; j++) {
        for (int k = 0; k < j; k++) Q[4 * j + k] = Q[4 * k + j] = K[j] * K2[k];
        Q[4 * j + j] = K[j] * K2[j];
    }
    return 1;
}

/* shared part of the isometric bending solvers: energy, gradients, weighted gradient norm */
static real isobending_terms(const vec3 *x, const real *w, const real *Q, vec3 *grad, real *sumNorm) {
    real energy = R(0.0);
    for (int k = 0; k < 4; k++) for (int j = 0; j < 4; j++) energy += Q[4 * j + k] * vdot(x[k], x[j]);
    energy *= R(0.5);
    for (int j = 0; j < 4; j++) grad[j] = VZERO;
    for (int k = 0; k < 4; k++) for (int j = 0; j < 4; j++) grad[j] = vadd(grad[j], vmul(x[k], Q[4 * j + k]));
    real s = R(0.0);
    for (int j = 0; j < 4; j++) if (w[j] != R(0.0)) s += w[j] * vsq(grad[j]);
    *sumNorm = s;
    return energy;
}

/* PositionBasedDynamics::solve_IsometricBendingConstraint, PositionBasedDynamics.cpp:186-236 */
static int solve_isobending(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, const real *Q,
                            real k, vec3 *c0, vec3 *c1, vec3 *c2, vec3 *c3) {
    const vec3 x[4] = {p2, p3, p0, p1};
    const real w[4] = {w2, w3, w0, w1};
    vec3 g[4]; real sum;
    real energy = isobending_terms(x, w, Q, g, &sum);
    if (RFABS(sum) > EPS) {
        const real s = energy / sum;
        *c0 = vmul(g[2], -k * (s * w[2]));
        *c1 = vmul(g[3], -k * (s * w[3]));
        *c2 = vmul(g[0], -k * (s * w[0]));
        *c3 = vmul(g[1], -k * (s * w[1]));
        return 1;
    }
    return 0;
}

/* XPBD::solve_IsometricBendingConstraint, XPBD.cpp:153-213 */
static int solve_isobending_xpbd(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, const real *Q,
                                 real k, real dt, real *lambda, vec3 *c0, vec3 *c1, vec3 *c2, vec3 *c3) {
    const vec3 x[4] = {p2, p3, p0, p1};
    const real w[4] = {w2, w3, w0, w1};
    vec3 g[4]; real sum;
    real energy = isobending_terms(x, w, Q, g, &sum);
    real alpha = R(0.0);
    if (k != R(0.0)) { alpha = R(1.0) / (k * dt * dt); sum += alpha; }
    if (RFABS(sum) > EPS) {
        const real dl = -(energy + alpha * *lambda) / sum;
        *lambda += dl;
        *c0 = vmul(g[2], dl * w[2]);
        *c1 = vmul(g[3], dl * w[3]);
        *c2 = vmul(g[0], dl * w[0]);
        *c3 = vmul(g[1], dl * w[1]);
        return 1;
    }
    return 0;
}

/* PositionBasedDynamics::init_FEMTriangleConstraint, PositionBasedDynamics.cpp:808-841. inv row-major 2x2 */
static int init_femtriangle(vec3 p0, vec3 p1, vec3 p2, real *area, real *inv) {
    vec3 normal0 = vcross(vsub(p1, p0), vsub(p2, p0));
    *area = vnorm(normal0) * R(0.5);
    vec3 axis1 = vnormalize(vsub(p1, p0));
    vec3 axis2 = vnormalize(vcross(normal0, axis1));
    real q[3][2] = {{vdot(p0, axis2), vdot(p0, axis1)}, {vdot(p1, axis2), vdot(p1, axis1)}, {vdot(p2, axis2), vdot(p2, axis1)}};
    real P00 = q[0][0] - q[2][0], P10 = q[0][1] - q[2][1], P01 = q[1][0] - q[2][0], P11 = q[1][1] - q[2][1];
    const real det = P00 * P11 - P01 * P10;
    if (RFABS(det) > EPS) {
        real id = R(1.0) / det;
        inv[0] = P11 * id; inv[1] = -P01 * id; inv[2] = -P10 * id; inv[3] = P00 * id;
        return 1;
    }
    return 0;
}

/* PositionBasedDynamics::solve_FEMTriangleConstraint, PositionBasedDynamics.cpp:844-930 */
static int solve_femtriangle(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, real area, const real *inv, real Ex,
                             real Ey, real Exy, real nuxy, real nuyx, vec3 *c0, vec3 *c1, vec3 *c2) {
#define IM(r, c) inv[2 * (r) + (c)]
    real C[3][3]; memset(C, 0, sizeof(C));
    C[0][0] = Ex / (R(1.0) - nuxy * nuyx);
    C[0][1] = Ex * nuyx / (R(1.0) - nuxy * nuyx);
    C[1][1] = Ey / (R(1.0) - nuxy * nuyx);
    C[1][0] = Ey * nuxy / (R(1.0) - nuxy * nuyx);
    C[2][2] = Exy;
    const vec3 p13 = vsub(p0, p2), p23 = vsub(p1, p2);
    real F[3][2];
    for (int r = 0; r < 3; r++) {
        F[r][0] = p13.v[r] * IM(0, 0) + p23.v[r] * IM(1, 0);
        F[r][1] = p13.v[r] * IM(0, 1) + p23.v[r] * IM(1, 1);
    }
    real e00 = R(0.5) * (F[0][0] * F[0][0] + F[1][0] * F[1][0] + F[2][0] * F[2][0] - R(1.0));
    real e11 = R(0.5) * (F[0][1] * F[0][1] + F[1][1] * F[1][1] + F[2][1] * F[2][1] - R(1.0));
    real e01 = R(0.5) * (F[0][0] * F[0][1] + F[1][0] * F[1][1] + F[2][0] * F[2][1]);
    real s00 = C[0][0] * e00 + C[0][1] * e11 + C[0][2] * e01;
    real s11 = C[1][0] * e00 + C[1][1] * e11 + C[1][2] * e01;
    real s01 = C[2][0] * e00 + C[2][1] * e11 + C[2][2] * e01;
    real PK[3][2];
    for (int r = 0; r < 3; r++) { PK[r][0] = F[r][0] * s00 + F[r][1] * s01; PK[r][1] = F[r][0] * s01 + F[r][1] * s11; }
    real psi = e00 * s00 + e01 * s01 + e01 * s01 + e11 * s11;
    psi = R(0.5) * psi;
    real energy = area * psi;
    /* H = area * PK * invRestMat^T */
    vec3 g[3];
    for (int r = 0; r < 3; r++) {
        real a0 = area * PK[r][0], a1 = area * PK[r][1];
        g[0].v[r] = a0 * IM(0, 0) + a1 * IM(0, 1);
        g[1].v[r] = a0 * IM(1, 0) + a1 * IM(1, 1);
    }
    g[2] = vsub(vneg(g[0]), g[1]);
    real sum = w0 * vsq(g[0]);
    sum += w1 * vsq(g[1]);
    sum += w2 * vsq(g[2]);
    if (RFABS(sum) > EPS) {
        const real s = energy / sum;
        *c0 = vmul(g[0], -(s * w0));
        *c1 = vmul(g[1], -(s * w1));
        *c2 = vmul(g[2], -(s * w2));
        return 1;
    }
    return 0;
#undef IM
}

/* PositionBasedDynamics::init_StrainTriangleConstraint, PositionBasedDynamics.cpp:562-581 */
static int init_straintriangle(vec3 p0, vec3 p1, vec3 p2, real *inv) {
    real a = p1.v[0] - p0.v[0], b = p2.v[0] - p0.v[0];
    real c = p1.v[1] - p0.v[1], d = p2.v[1] - p0.v[1];
    real det = a * d - b * c;
    if (RFABS(det) < EPS) return 0;
    real s = R(1.0) / det;
    inv[0] = d * s; inv[1] = -b * s; inv[2] = -c * s; inv[3] = a * s;
    return 1;
}

/* PositionBasedDynamics::solve_StrainTriangleConstraint, PositionBasedDynamics.cpp:584-688 */
static int solve_straintriangle(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, const real *inv, real kxx, real kyy,
                                real kxy, int normStretch, int normShear, vec3 *c0, vec3 *c1, vec3 *c2) {
#define IM(r, c) inv[2 * (r) + (c)]
    vec3 c[2] = {V(IM(0, 0), IM(1, 0), R(0.0)), V(IM(0, 1), IM(1, 1), R(0.0))};
    vec3 r[3];
    *c0 = *c1 = *c2 = VZERO;
    for (int i = 0; i < 2; i++) {
        for (int j = 0; j <= i; j++) {
            for (int a = 0; a < 3; a++)
                r[a] = V((p1.v[a] + c1->v[a]) - (p0.v[a] + c0->v[a]), (p2.v[a] + c2->v[a]) - (p0.v[a] + c0->v[a]), R(0.0));
            real Sij = R(0.0);
            for (int k = 0; k < 3; k++) Sij += vdot(r[k], c[i]) * vdot(r[k], c[j]);
            vec3 d[3];
            d[0] = VZERO;
            vec3 rci = V(vdot(r[0], c[i]), vdot(r[1], c[i]), vdot(r[2], c[i]));
            vec3 rcj = V(vdot(r[0], c[j]), vdot(r[1], c[j]), vdot(r[2], c[j]));
            for (int k = 0; k < 2; k++) {
                d[k + 1] = vmul(rcj, IM(k, i));
                d[k + 1] = vadd(d[k + 1], vmul(rci, IM(k, j)));
                d[0] = vsub(d[0], d[k + 1]);
            }
            if (i != j && normShear) {
                real fi2 = R(0.0), fj2 = R(0.0);
                for (int k = 0; k < 3; k++) { fi2 += vdot(r[k], c[i]) * vdot(r[k], c[i]); fj2 += vdot(r[k], c[j]) * vdot(r[k], c[j]); }
                real fi = RSQRT(fi2), fj = RSQRT(fj2);
                d[0] = VZERO;
                real s = Sij / (fi2 * fi * fj2 * fj);
                for (int k = 0; k < 2; k++) {
                    real q = fi * fj;
                    d[k + 1] = V(d[k + 1].v[0] / q, d[k + 1].v[1] / q, d[k + 1].v[2] / q);
                    d[k + 1] = vsub(d[k + 1], vmul(vmul(vmul(rci, fj * fj), IM(k, i)), s));
                    d[k + 1] = vsub(d[k + 1], vmul(vmul(vmul(rcj, fi * fi), IM(k, j)), s));
                    d[0] = vsub(d[0], d[k + 1]);
                }
                Sij = Sij / (fi * fj);
            }
            real lambda = w0 * vsq(d[0]) + w1 * vsq(d[1]) + w2 * vsq(d[2]);
            if (lambda == R(0.0)) continue;
            if (i == 0 && j == 0) {
                if (normStretch) { real s = RSQRT(Sij); lambda = R(2.0) * s * (s - R(1.0)) / lambda * kxx; }
                else lambda = (Sij - R(1.0)) / lambda * kxx;
            } else if (i == 1 && j == 1) {
                if (normStretch) { real s = RSQRT(Sij); lambda = R(2.0) * s * (s - R(1.0)) / lambda * kyy; }
                else lambda = (Sij - R(1.0)) / lambda * kyy;
            } else {
                lambda = Sij / lambda * kxy;
            }
            *c0 = vsub(*c0, vmul(d[0], lambda * w0));
            *c1 = vsub(*c1, vmul(d[1], lambda * w1));
            *c2 = vsub(*c2, vmul(d[2], lambda * w2));
        }
    }
    return 1;
#undef IM
}

/* PositionBasedDynamics::init_ShapeMatchingConstraint, PositionBasedDynamics.cpp:479-497 */
static int init_shapematching(const vec3 *x0, const real *w, int n, vec3 *restCm) {
    *restCm = VZERO;
    real wsum = R(0.0);
    for (int i = 0; i < n; i++) { real wi = R(1.0) / (w[i] + EPS); *restCm = vadd(*restCm, vmul(x0[i], wi)); wsum += wi; }
    if (wsum == R(0.0)) return 0;
    *restCm = V(restCm->v[0] / wsum, restCm->v[1] / wsum, restCm->v[2] / wsum);
    return 1;
}

/* PositionBasedDynamics::solve_ShapeMatchingConstraint, PositionBasedDynamics.cpp:500-558 (allowStretch = false) */
static int solve_shapematching(const vec3 *x0, const vec3 *x, const real *w, int n, vec3 restCm, real k, vec3 *corr) {
    for (int i = 0; i < n; i++) corr[i] = VZERO;
    vec3 cm = VZERO; real wsum = R(0.0);
    for (int i = 0; i < n; i++) { real wi = R(1.0) / (w[i] + EPS); cm = vadd(cm, vmul(x[i], wi)); wsum += wi; }
    if (wsum == R(0.0)) return 0;
    cm = V(cm.v[0] / wsum, cm.v[1] / wsum, cm.v[2] / wsum);
    mat3 A; memset(&A, 0, sizeof(A));
    for (int i = 0; i < n; i++) {
        vec3 q = vsub(x0[i], restCm), pp = vsub(x[i], cm);
        real wi = R(1.0) / (w[i] + EPS);
        pp = vmul(pp, wi);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) A.m[r][c] += pp.v[r] * q.v[c];
    }
    mat3 Rm;
    polar_decomposition_stable(&A, EPS, &Rm);
    for (int i = 0; i < n; i++) {
        vec3 q = vsub(x0[i], restCm);
        vec3 goal = vadd(cm, V(Rm.m[0][0] * q.v[0] + Rm.m[0][1] * q.v[1] + Rm.m[0][2] * q.v[2], Rm.m[1][0] * q.v[0] + Rm.m[1][1] * q.v[1] + Rm.m[1][2] * q.v[2],
                               Rm.m[2][0] * q.v[0] + Rm.m[2][1] * q.v[1] + Rm.m[2][2] * q.v[2]));
        corr[i] = vmul(vsub(goal, x[i]), k);
    }
    return 1;
}

/* PositionBasedDynamics::init_StrainTetraConstraint, PositionBasedDynamics.cpp:691-710 */
static int init_straintet(vec3 p0, vec3 p1, vec3 p2, vec3 p3, mat3 *inv) {
    mat3 m; vec3 a = vsub(p1, p0), b = vsub(p2, p0), c = vsub(p3, p0);
    for (int r = 0; r < 3; r++) { m.m[r][0] = a.v[r]; m.m[r][1] = b.v[r]; m.m[r][2] = c.v[r]; }
    real det = det3(&m);
    if (RFABS(det) > EPS) { *inv = inv3(&m, det); return 1; }
    return 0;
}

/* PositionBasedDynamics::solve_StrainTetraConstraint, PositionBasedDynamics.cpp:713-805 */
static int solve_straintet(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, const mat3 *inv,
                           vec3 stretchK, vec3 shearK, int normStretch, int normShear, vec3 *c0, vec3 *c1, vec3 *c2, vec3 *c3) {
    *c0 = *c1 = *c2 = *c3 = VZERO;
    vec3 c[3] = {mcol(inv, 0), mcol(inv, 1), mcol(inv, 2)};
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j <= i; j++) {
            vec3 P0 = vsub(vadd(p1, *c1), vadd(p0, *c0));
            vec3 P1 = vsub(vadd(p2, *c2), vadd(p0, *c0));
            vec3 P2 = vsub(vadd(p3, *c3), vadd(p0, *c0));
            /* fi = P * c[i] (P has columns P0,P1,P2) */
            vec3 fi = vadd(vadd(vmul(P0, c[i].v[0]), vmul(P1, c[i].v[1])), vmul(P2, c[i].v[2]));
            vec3 fj = vadd(vadd(vmul(P0, c[j].v[0]), vmul(P1, c[j].v[1])), vmul(P2, c[j].v[2]));
            real Sij = vdot(fi, fj);
            real wi = 0, wj = 0, s1 = 0, s3 = 0;
            if (normShear && i != j) {
                wi = vnorm(fi); wj = vnorm(fj);
                s1 = R(1.0) / (wi * wj);
                s3 = s1 * s1 * s1;
            }
            vec3 d[4];
            d[0] = VZERO;
            for (int k = 0; k < 3; k++) {
                d[k + 1] = vadd(vmul(fj, inv->m[k][i]), vmul(fi, inv->m[k][j]));
                if (normShear && i != j) {
                    vec3 t = vadd(vmul(vmul(fi, wj * wj), inv->m[k][i]), vmul(vmul(fj, wi * wi), inv->m[k][j]));
                    d[k + 1] = vsub(vmul(d[k + 1], s1), vmul(t, Sij * s3));
                }
                d[0] = vsub(d[0], d[k + 1]);
            }
            if (normShear && i != j) Sij *= s1;
            real lambda = w0 * vsq(d[0]) + w1 * vsq(d[1]) + w2 * vsq(d[2]) + w3 * vsq(d[3]);
            if (RFABS(lambda) < EPS) continue;
            if (i == j) {
                if (normStretch) { real s = RSQRT(Sij); lambda = R(2.0) * s * (s - R(1.0)) / lambda * stretchK.v[i]; }
                else lambda = (Sij - R(1.0)) / lambda * stretchK.v[i];
            } else {
                lambda = Sij / lambda * shearK.v[i + j - 1];
            }
            *c0 = vsub(*c0, vmul(d[0], lambda * w0));
            *c1 = vsub(*c1, vmul(d[1], lambda * w1));
            *c2 = vsub(*c2, vmul(d[2], lambda * w2));
            *c3 = vsub(*c3, vmul(d[3], lambda * w3));
        }
    }
    return 1;
}

/* PositionBasedDynamics::init_FEMTetraConstraint, PositionBasedDynamics.cpp:933-955 */
static int init_femtet(vec3 p0, vec3 p1, vec3 p2, vec3 p3, real *volume, mat3 *inv) {
    *volume = RFABS(R(1.0 / 6.0) * vdot(vsub(p3, p0), vcross(vsub(p2, p0), vsub(p1, p0))));
    mat3 m; vec3 a = vsub(p0, p3), b = vsub(p1, p3), c = vsub(p2, p3);
    for (int r = 0; r < 3; r++) { m.m[r][0] = a.v[r]; m.m[r][1] = b.v[r]; m.m[r][2] = c.v[r]; }
    real det = det3(&m);
    if (RFABS(det) > EPS) { *inv = inv3(&m, det); return 1; }
    return 0;
}

static void deformation_gradient(vec3 x1, vec3 x2, vec3 x3, vec3 x4, const mat3 *inv, mat3 *F) {
    const vec3 p14 = vsub(x1, x4), p24 = vsub(x2, x4), p34 = vsub(x3, x4);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) F->m[r][c] = p14.v[r] * inv->m[0][c] + p24.v[r] * inv->m[1][c] + p34.v[r] * inv->m[2][c];
}

/* PositionBasedDynamics::computeGreenStrainAndPiolaStress, PositionBasedDynamics.cpp:958-1008 */
static void green_strain_piola(vec3 x1, vec3 x2, vec3 x3, vec3 x4, const mat3 *inv, real restVolume, real mu, real lambda,
                               mat3 *epsilon, mat3 *sigma, real *energy) {
    mat3 F;
    deformation_gradient(x1, x2, x3, x4, inv, &F);
    for (int a = 0; a < 3; a++)
        for (int b = a; b < 3; b++) {
            real s = F.m[0][a] * F.m[0][b] + F.m[1][a] * F.m[1][b] + F.m[2][a] * F.m[2][b];
            if (a == b) s -= R(1.0);
            epsilon->m[a][b] = epsilon->m[b][a] = R(0.5) * s;
        }
    const real trace = epsilon->m[0][0] + epsilon->m[1][1] + epsilon->m[2][2];
    const real ltrace = lambda * trace;
    mat3 s2;
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) s2.m[a][b] = (real)(epsilon->m[a][b] * 2.0) * mu;
    s2.m[0][0] += ltrace; s2.m[1][1] += ltrace; s2.m[2][2] += ltrace;
    *sigma = mul3(&F, &s2);
    real psi = R(0.0);
    for (int j = 0; j < 3; j++) for (int k = 0; k < 3; k++) psi += epsilon->m[j][k] * epsilon->m[j][k];
    psi = mu * psi + R(0.5) * lambda * trace * trace;
    *energy = restVolume * psi;
}

/* PositionBasedDynamics::computeGradCGreen, PositionBasedDynamics.cpp:1011-1031 */
static void grad_c_green(real restVolume, const mat3 *inv, const mat3 *sigma, vec3 *J) {
    mat3 T = transpose3(inv);
    mat3 H = mul3(sigma, &T);
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) H.m[a][b] *= restVolume;
    for (int r = 0; r < 3; r++) { J[0].v[r] = H.m[r][0]; J[1].v[r] = H.m[r][1]; J[2].v[r] = H.m[r][2]; }
    J[3] = vsub(vsub(vneg(J[0]), J[1]), J[2]);
}

/* PositionBasedDynamics::computeGreenStrainAndPiolaStressInversion, PositionBasedDynamics.cpp:1034-1104 */
static void green_strain_piola_inversion(vec3 x1, vec3 x2, vec3 x3, vec3 x4, const mat3 *inv, real restVolume, real mu,
                                         real lambda, mat3 *epsilon, mat3 *sigma, real *energy) {
    mat3 F, U, VT; vec3 hatF;
    deformation_gradient(x1, x2, x3, x4, inv, &F);
    svd_inversion(&F, &hatF, &U, &VT);
    const real minXVal = R(0.577);
    for (int j = 0; j < 3; j++) if (hatF.v[j] < minXVal) hatF.v[j] = minXVal;
    vec3 eh = V(R(0.5) * (hatF.v[0] * hatF.v[0] - R(1.0)), R(0.5) * (hatF.v[1] * hatF.v[1] - R(1.0)),
                R(0.5) * (hatF.v[2] * hatF.v[2] - R(1.0)));
    const real trace = eh.v[0] + eh.v[1] + eh.v[2];
    const real ltrace = lambda * trace;
    vec3 sv;
    for (int j = 0; j < 3; j++) { sv.v[j] = (real)(eh.v[j] * 2.0) * mu; sv.v[j] += ltrace; sv.v[j] = hatF.v[j] * sv.v[j]; }
    mat3 sd, ed; memset(&sd, 0, sizeof(sd)); memset(&ed, 0, sizeof(ed));
    for (int j = 0; j < 3; j++) { sd.m[j][j] = sv.v[j]; ed.m[j][j] = eh.v[j]; }
    mat3 t = mul3(&U, &ed); *epsilon = mul3(&t, &VT);
    t = mul3(&U, &sd); *sigma = mul3(&t, &VT);
    real psi = R(0.0);
    for (int j = 0; j < 3; j++) for (int k = 0; k < 3; k++) psi += epsilon->m[j][k] * epsilon->m[j][k];
    psi = mu * psi + R(0.5) * lambda * trace * trace;
    *energy = restVolume * psi;
}

/* PositionBasedDynamics::solve_FEMTetraConstraint, PositionBasedDynamics.cpp:1109-1169 */
static int solve_femtet(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, real restVolume,
                        const mat3 *inv, real E, real nu, int handleInversion, vec3 *c0, vec3 *c1, vec3 *c2, vec3 *c3) {
    *c0 = *c1 = *c2 = *c3 = VZERO;
    if (E <= R(0.0)) return 1;
    if (nu < R(0.0) || nu > 0.49) return 0;
    real C = R(0.0);
    vec3 g[4]; mat3 eps_, sig;
    real volume = vdot(vcross(vsub(p1, p0), vsub(p2, p0)), vsub(p3, p0)) / R(6.0);
    real mu = E / R(2.0) / (R(1.0) + nu);
    real lambda = E * nu / (R(1.0) + nu) / (R(1.0) - R(2.0) * nu);
    if (!handleInversion || volume > R(0.0)) green_strain_piola(p0, p1, p2, p3, inv, restVolume, mu, lambda, &eps_, &sig, &C);
    else green_strain_piola_inversion(p0, p1, p2, p3, inv, restVolume, mu, lambda, &eps_, &sig, &C);
    grad_c_green(restVolume, inv, &sig, g);
    real sum = w0 * vsq(g[0]) + w1 * vsq(g[1]) + w2 * vsq(g[2]) + w3 * vsq(g[3]);
    if (sum < EPS) return 0;
    const real s = C / sum;
    *c0 = vmul(g[0], -s * w0);
    *c1 = vmul(g[1], -s * w1);
    *c2 = vmul(g[2], -s * w2);
    *c3 = vmul(g[3], -s * w3);
    return 1;
}

/* XPBD::solve_FEMTetraConstraint, XPBD.cpp:217-294 */
static int solve_femtet_xpbd(vec3 p0, real w0, vec3 p1, real w1, vec3 p2, real w2, vec3 p3, real w3, real restVolume,
                             const mat3 *inv, real E, real nu, int handleInversion, real dt, real *multiplier, vec3 *c0,
                             vec3 *c1, vec3 *c2, vec3 *c3) {
    *c0 = *c1 = *c2 = *c3 = VZERO;
    if (E <= R(0.0)) return 1;
    if (nu < R(0.0) || nu > 0.49) return 0;
    vec3 g[4]; mat3 eps_, sig;
    real volume = vdot(vcross(vsub(p1, p0), vsub(p2, p0)), vsub(p3, p0)) / R(6.0);
    real mu_ = (real)(1.0 / R(2.0) / (R(1.0) + nu));
    real lambda_ = (real)(1.0 * nu / (R(1.0) + nu) / (R(1.0) - R(2.0) * nu));
    real U_ = R(0.0);
    if (!handleInversion || volume > R(0.0)) green_strain_piola(p0, p1, p2, p3, inv, restVolume, mu_, lambda_, &eps_, &sig, &U_);
    else green_strain_piola_inversion(p0, p1, p2, p3, inv, restVolume, mu_, lambda_, &eps_, &sig, &U_);
    grad_c_green(restVolume, inv, &sig, g);
    const real C = (real)sqrt(2.0 * U_);
    real sum = w0 * vsq(g[0]) + w1 * vsq(g[1]) + w2 * vsq(g[2]) + w3 * vsq(g[3]);
    real alpha = R(1.0) / (E * dt * dt);
    sum += C * C * alpha;
    if (sum < EPS) return 0;
    const real lambda = -C * (C + alpha * *multiplier) / sum;
    *multiplier += lambda;
    *c0 = vmul(g[0], lambda * w0);
    *c1 = vmul(g[1], lambda * w1);
    *c2 = vmul(g[2], lambda * w2);
    *c3 = vmul(g[3], lambda * w3);
    return 1;
}

/* ------------------------------------------------------------------------------------------------ */
/* Model state (flat restatement of ParticleData.h:86-311 + SimulationModel's constraint vector)     */
/* ------------------------------------------------------------------------------------------------ */
typedef struct {
    int type;
    unsigned nb;
    unsigned b[4];
    real p[ORC_MAX_PARAMS];
    real lambda;
} Constraint;

typedef struct { unsigned v[2]; unsigned f[2]; } TriEdge;
typedef struct {
    unsigned offset, nVerts, nFaces, nEdges;
    unsigned *faces; /* 3 per face */
    TriEdge *edges;
} TriModel;
typedef struct {
    unsigned offset, nVerts, nTets, nEdges;
    unsigned *tets;     /* 4 per tet */
    unsigned *edges;    /* 2 per edge */
    unsigned *vertTets; /* number of tets per vertex */
} TetModel;

/* Simulation/RigidBody.h:17-68 (state used on this path) */
typedef struct {
    real mass, invMass;
    vec3 x, lastX, oldX, x0, v, a, omega, torque;
    vec3 inertia, inertiaInv;
    mat3 rot, inertiaW, inertiaInvW;
    quat q, lastQ, oldQ, q0;
} RigidBody;

/* contact path: DistanceFieldCollisionDetection objects as an adapter would hand them over (same layout as pbd_rigid_collider of
 * include/pbd_b200.h): shape, body, dimensions, m_invertSDF, the body's coefficients, RigidBody::getTransformationR / V1 / V2 and m_aabb */
struct RigidColl { int shape; unsigned body; double dim[3], thickness, invert; real restitution, friction; real Rm[9], v1[3], v2[3], lo[3], hi[3]; };
struct PartColl { unsigned offset, count; real restitution, friction; };
/* ParticleRigidBodyContactConstraint (Constraints.h): m_bodies, m_constraintInfo (3x5), m_sum_impulses, m_stiffness, m_frictionCoeff */
struct Contact { unsigned particle, body; vec3 cp0, cp1, n, t; real nKnInv, pMax, goal, sum, stiffness, friction; };

typedef struct {
    unsigned n, cap;
    RigidBody *rbs; unsigned nRb;
    vec3 *x0, *x, *v, *a, *oldX, *lastX;
    real *mass, *invMass;
    Constraint *cons; unsigned nCons, capCons;
    TriModel *tris; unsigned nTris;
    TetModel *tets; unsigned nTetModels;
    unsigned *groupOff, *groupIds; unsigned nGroups; int groupsInit;
    real dt, time; unsigned subSteps, maxIter; int velMethod; vec3 gravity;
    /* contact path (static analytic colliders) */
    struct RigidColl *rigidColl; unsigned nRigidColl;
    struct PartColl *partColl; unsigned nPartColl;
    struct Contact *contacts; unsigned nContacts, capContacts;
    real contactTolerance, contactStiffness; unsigned maxIterV;
} Model;

static Model *G = NULL;

static void model_free(Model *m) {
    if (!m) return;
    free(m->x0); free(m->x); free(m->v); free(m->a); free(m->oldX); free(m->lastX); free(m->mass); free(m->invMass);
    free(m->cons);
    for (unsigned i = 0; i < m->nTris; i++) { free(m->tris[i].faces); free(m->tris[i].edges); }
    for (unsigned i = 0; i < m->nTetModels; i++) { free(m->tets[i].tets); free(m->tets[i].edges); free(m->tets[i].vertTets); }
    free(m->tris); free(m->tets); free(m->groupOff); free(m->groupIds); free(m->rbs);
    free(m->rigidColl); free(m->partColl); free(m->contacts);
    free(m);
}

int orc_real_size(void) { return (int)sizeof(real); }
void orc_set_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}
int orc_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* defaults: TimeStepController.cpp:23-32 (subSteps 5, maxIterations 1, first-order velocity update),
 * TimeManager.cpp:10 / Simulation.cpp:56 (h = 0.005), Simulation.cpp:16 (gravity) */
void orc_reset(void) {
    model_free(G);
    G = (Model *)calloc(1, sizeof(Model));
    G->dt = R(0.005); G->subSteps = 5; G->maxIter = 1; G->velMethod = 0;
    G->contactTolerance = R(0.01); G->contactStiffness = R(100.0); G->maxIterV = 5; /* CollisionDetection.cpp:25, SimulationModel.cpp:57, TimeStepController.cpp:29 */
    G->gravity = V(R(0.0), R(-9.81), R(0.0));
}

/* ParticleData::addVertex, ParticleData.h:127-137 (mass = invMass = 1) */
static unsigned add_vertex(Model *m, vec3 p) {
    if (m->n == m->cap) {
        unsigned nc = m->cap ? m->cap * 2 : 1024;
#define GROW(f, T) m->f = (T *)realloc(m->f, (size_t)nc * sizeof(T))
        GROW(x0, vec3); GROW(x, vec3); GROW(v, vec3); GROW(a, vec3); GROW(oldX, vec3); GROW(lastX, vec3);
        GROW(mass, real); GROW(invMass, real);
#undef GROW
        m->cap = nc;
    }
    unsigned i = m->n++;
    m->x0[i] = m->x[i] = m->oldX[i] = m->lastX[i] = p;
    m->v[i] = m->a[i] = VZERO;
    m->mass[i] = m->invMass[i] = R(1.0);
    return i;
}

/* ParticleData::setMass, ParticleData.h:239-246 */
void orc_set_mass(unsigned i, double mass) {
    G->mass[i] = (real)mass;
    G->invMass[i] = ((real)mass != R(0.0)) ? R(1.0) / (real)mass : R(0.0);
}

/* IndexedFaceMesh::buildNeighbors, Utils/IndexedFaceMesh.cpp:118-226.
 * Edges are discovered face by face in the order (v0,v1), (v1,v2), (v2,v0); the first sighting fixes the
 * orientation and m_face[0]; a later sighting sets m_face[1].  The search list of the reference
 * (pEdges[a]) holds every edge touching a, so "find an edge with endpoints {a,b}" is a lookup among the
 * edges incident to a in discovery order - reproduced here with per-vertex incidence lists. */
static void build_tri_edges(TriModel *t) {
    unsigned nv = t->nVerts, nf = t->nFaces;
    unsigned cap = 3 * nf;
    t->edges = (TriEdge *)malloc((size_t)(cap ? cap : 1) * sizeof(TriEdge));
    t->nEdges = 0;
    /* incidence lists: head per vertex, (edge, next) nodes; appended at tail to keep discovery order */
    unsigned *head = (unsigned *)malloc((size_t)nv * sizeof(unsigned));
    unsigned *tail = (unsigned *)malloc((size_t)nv * sizeof(unsigned));
    unsigned *nodeEdge = (unsigned *)malloc((size_t)2 * (cap ? cap : 1) * sizeof(unsigned));
    unsigned *nodeNext = (unsigned *)malloc((size_t)2 * (cap ? cap : 1) * sizeof(unsigned));
    unsigned nNodes = 0;
    for (unsigned i = 0; i < nv; i++) head[i] = tail[i] = NOFACE;
    for (unsigned f = 0; f < nf; f++) {
        const unsigned *vv = t->faces + 3 * f;
        for (unsigned j = 0; j < 3; j++) {
            unsigned a = vv[j], b = vv[(j + 1) % 3];
            unsigned edge = NOFACE;
            for (unsigned nd = head[a]; nd != NOFACE; nd = nodeNext[nd]) {
                const TriEdge *e = &t->edges[nodeEdge[nd]];
                if ((e->v[0] == a || e->v[0] == b) && (e->v[1] == a || e->v[1] == b)) { edge = nodeEdge[nd]; break; }
            }
            if (edge == NOFACE) {
                TriEdge e; e.v[0] = a; e.v[1] = b; e.f[0] = f; e.f[1] = NOFACE;
                edge = t->nEdges;
                t->edges[t->nEdges++] = e;
                unsigned ends[2] = {a, b};
                for (int s = 0; s < 2; s++) {
                    unsigned nd = nNodes++;
                    nodeEdge[nd] = edge; nodeNext[nd] = NOFACE;
                    if (head[ends[s]] == NOFACE) head[ends[s]] = nd; else nodeNext[tail[ends[s]]] = nd;
                    tail[ends[s]] = nd;
                }
            } else {
                t->edges[edge].f[1] = f;
            }
        }
    }
    free(head); free(tail); free(nodeEdge); free(nodeNext);
}

/* SimulationModel::addTriangleModel, SimulationModel.cpp:808-829 (+TriangleModel::initMesh, TriangleModel.cpp:30-43) */
static unsigned add_triangle_model(Model *m, unsigned nPoints, unsigned nFaces, const vec3 *pts, const unsigned *idx) {
    m->tris = (TriModel *)realloc(m->tris, (size_t)(m->nTris + 1) * sizeof(TriModel));
    TriModel *t = &m->tris[m->nTris];
    t->offset = m->n; t->nVerts = nPoints; t->nFaces = nFaces;
    for (unsigned i = 0; i < nPoints; i++) add_vertex(m, pts[i]);
    t->faces = (unsigned *)malloc((size_t)3 * (nFaces ? nFaces : 1) * sizeof(unsigned));
    memcpy(t->faces, idx, (size_t)3 * nFaces * sizeof(unsigned));
    build_tri_edges(t);
    return m->nTris++;
}

static vec3 rot_apply(const double *Rm, vec3 p, vec3 t) {
    real r[9]; for (int i = 0; i < 9; i++) r[i] = (real)Rm[i];
    return vadd(V(r[0] * p.v[0] + r[1] * p.v[1] + r[2] * p.v[2], r[3] * p.v[0] + r[4] * p.v[1] + r[5] * p.v[2],
                  r[6] * p.v[0] + r[7] * p.v[1] + r[8] * p.v[2]), t);
}

/* SimulationModel::addRegularTriangleModel, SimulationModel.cpp:831-901 */
void orc_add_regular_triangle_model(int width, int height, const double *t, const double *Rm, const double *scale) {
    const real sx = (real)scale[0], sy = (real)scale[1];
    const real dy = sy / (real)(height - 1);
    const real dx = sx / (real)(width - 1);
    vec3 tr = V((real)t[0], (real)t[1], (real)t[2]);
    vec3 *pts = (vec3 *)malloc((size_t)width * height * sizeof(vec3));
    for (int i = 0; i < height; i++)
        for (int j = 0; j < width; j++) {
            const real y = (real)dy * i;
            const real x = (real)dx * j;
            pts[i * width + j] = rot_apply(Rm, V(x, y, R(0.0)), tr);
        }
    const int nIdx = 6 * (height - 1) * (width - 1);
    unsigned *idx = (unsigned *)malloc((size_t)(nIdx ? nIdx : 1) * sizeof(unsigned));
    int k = 0;
    for (int i = 0; i < height - 1; i++)
        for (int j = 0; j < width - 1; j++) {
            int helper = (i % 2 == j % 2) ? 1 : 0;
            idx[k++] = i * width + j; idx[k++] = i * width + j + 1; idx[k++] = (i + 1) * width + j + helper;
            idx[k++] = (i + 1) * width + j + 1; idx[k++] = (i + 1) * width + j; idx[k++] = i * width + j + 1 - helper;
        }
    unsigned tm = add_triangle_model(G, (unsigned)(width * height), (unsigned)(nIdx / 3), pts, idx);
    for (unsigned i = G->tris[tm].offset; i < G->tris[tm].offset + G->tris[tm].nVerts; i++) orc_set_mass(i, 1.0);
    free(pts); free(idx);
}

void orc_add_triangle_model(unsigned nPoints, unsigned nFaces, const double *pts, const unsigned *idx) {
    vec3 *p = (vec3 *)malloc((size_t)(nPoints ? nPoints : 1) * sizeof(vec3));
    for (unsigned i = 0; i < nPoints; i++) p[i] = V((real)pts[3 * i], (real)pts[3 * i + 1], (real)pts[3 * i + 2]);
    add_triangle_model(G, nPoints, nFaces, p, idx);
    free(p);
}

/* IndexedTetMesh::buildNeighbors, Utils/IndexedTetMesh.cpp:55-182: edges per tet in the order
 * {0,1 0,2 0,3 1,2 1,3 2,3}, first sighting wins; vertex->tet incidence counts (for shape matching). */
static void build_tet_edges(TetModel *t) {
    unsigned nv = t->nVerts, nt = t->nTets;
    unsigned cap = 6 * nt;
    t->edges = (unsigned *)malloc((size_t)2 * (cap ? cap : 1) * sizeof(unsigned));
    t->nEdges = 0;
    t->vertTets = (unsigned *)calloc(nv ? nv : 1, sizeof(unsigned));
    unsigned *head = (unsigned *)malloc((size_t)(nv ? nv : 1) * sizeof(unsigned));
    unsigned *tail = (unsigned *)malloc((size_t)(nv ? nv : 1) * sizeof(unsigned));
    unsigned *nodeEdge = (unsigned *)malloc((size_t)2 * (cap ? cap : 1) * sizeof(unsigned));
    unsigned *nodeNext = (unsigned *)malloc((size_t)2 * (cap ? cap : 1) * sizeof(unsigned));
    unsigned nNodes = 0;
    for (unsigned i = 0; i < nv; i++) head[i] = tail[i] = NOFACE;
    static const int EP[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
    for (unsigned ti = 0; ti < nt; ti++) {
        const unsigned *vv = t->tets + 4 * ti;
        for (int j = 0; j < 4; j++) t->vertTets[vv[j]]++;
        for (int j = 0; j < 6; j++) {
            unsigned a = vv[EP[j][0]], b = vv[EP[j][1]];
            unsigned edge = NOFACE;
            for (unsigned nd = head[a]; nd != NOFACE; nd = nodeNext[nd]) {
                const unsigned *e = t->edges + 2 * nodeEdge[nd];
                if ((e[0] == a || e[0] == b) && (e[1] == a || e[1] == b)) { edge = nodeEdge[nd]; break; }
            }
            if (edge == NOFACE) {
                edge = t->nEdges++;
                t->edges[2 * edge] = a; t->edges[2 * edge + 1] = b;
                unsigned ends[2] = {a, b};
                for (int s = 0; s < 2; s++) {
                    unsigned nd = nNodes++;
                    nodeEdge[nd] = edge; nodeNext[nd] = NOFACE;
                    if (head[ends[s]] == NOFACE) head[ends[s]] = nd; else nodeNext[tail[ends[s]]] = nd;
                    tail[ends[s]] = nd;
                }
            }
        }
    }
    free(head); free(tail); free(nodeEdge); free(nodeNext);
}

/* SimulationModel::addTetModel, SimulationModel.cpp:903-919 */
static unsigned add_tet_model(Model *m, unsigned nPoints, unsigned nTets, const vec3 *pts, const unsigned *idx) {
    m->tets = (TetModel *)realloc(m->tets, (size_t)(m->nTetModels + 1) * sizeof(TetModel));
    TetModel *t = &m->tets[m->nTetModels];
    t->offset = m->n; t->nVerts = nPoints; t->nTets = nTets;
    for (unsigned i = 0; i < nPoints; i++) add_vertex(m, pts[i]);
    t->tets = (unsigned *)malloc((size_t)4 * (nTets ? nTets : 1) * sizeof(unsigned));
    memcpy(t->tets, idx, (size_t)4 * nTets * sizeof(unsigned));
    build_tet_edges(t);
    return m->nTetModels++;
}

/* SimulationModel::addRegularTetModel, SimulationModel.cpp:921-1005 */
void orc_add_regular_tet_model(int width, int height, int depth, const double *t, const double *Rm, const double *scale) {
    const real s0 = (real)scale[0], s1 = (real)scale[1], s2 = (real)scale[2];
    const real dx = s0 / (real)(width - 1), dy = s1 / (real)(height - 1), dz = s2 / (real)(depth - 1);
    /* translation - 0.5*scale: the 0.5 is a double literal applied to a Real vector */
    vec3 tr = V((real)t[0] - (real)(0.5 * s0), (real)t[1] - (real)(0.5 * s1), (real)t[2] - (real)(0.5 * s2));
    vec3 *pts = (vec3 *)malloc((size_t)width * height * depth * sizeof(vec3));
    for (int i = 0; i < width; i++)
        for (int j = 0; j < height; j++)
            for (int k = 0; k < depth; k++) {
                const real x = (real)dx * i, y = (real)dy * j, z = (real)dz * k;
                pts[i * height * depth + j * depth + k] = rot_apply(Rm, V(x, y, z), tr);
            }
    size_t nCells = (size_t)(width - 1) * (height - 1) * (depth - 1);
    unsigned *idx = (unsigned *)malloc((nCells ? nCells : 1) * 20 * sizeof(unsigned));
    size_t n = 0;
    for (int i = 0; i < width - 1; i++)
        for (int j = 0; j < height - 1; j++)
            for (int k = 0; k < depth - 1; k++) {
                unsigned p0 = i * height * depth + j * depth + k;
                unsigned p1 = p0 + 1;
                unsigned p3 = (i + 1) * height * depth + j * depth + k;
                unsigned p2 = p3 + 1;
                unsigned p7 = (i + 1) * height * depth + (j + 1) * depth + k;
                unsigned p6 = p7 + 1;
                unsigned p4 = i * height * depth + (j + 1) * depth + k;
                unsigned p5 = p4 + 1;
                if ((i + j + k) % 2 == 1) {
                    const unsigned q[20] = {p2, p1, p6, p3, p6, p3, p4, p7, p4, p1, p6, p5, p3, p1, p4, p0, p6, p1, p4, p3};
                    memcpy(idx + n, q, sizeof(q));
                } else {
                    const unsigned q[20] = {p0, p2, p5, p1, p7, p2, p0, p3, p5, p2, p7, p6, p7, p0, p5, p4, p0, p2, p7, p5};
                    memcpy(idx + n, q, sizeof(q));
                }
                n += 20;
            }
    unsigned tm = add_tet_model(G, (unsigned)(width * height * depth), (unsigned)(n / 4), pts, idx);
    for (unsigned i = G->tets[tm].offset; i < G->tets[tm].offset + G->tets[tm].nVerts; i++) orc_set_mass(i, 1.0);
    free(pts); free(idx);
}

void orc_add_tet_model(unsigned nPoints, unsigned nTets, const double *pts, const unsigned *idx) {
    vec3 *p = (vec3 *)malloc((size_t)(nPoints ? nPoints : 1) * sizeof(vec3));
    for (unsigned i = 0; i < nPoints; i++) p[i] = V((real)pts[3 * i], (real)pts[3 * i + 1], (real)pts[3 * i + 2]);
    add_tet_model(G, nPoints, nTets, p, idx);
    free(p);
}

/* ------------------------------------------------------------------------------------------------ */
/* rigid bodies and the two joints that couple them to particles (SURVEY.md 8f-1)                     */
/* ------------------------------------------------------------------------------------------------ */
/* RigidBody::rotationUpdated + updateInertiaW, RigidBody.h:190-207 */
static void rb_rotation_updated(RigidBody *b) {
    if (b->mass == R(0.0)) return;
    b->rot = qmatrix(b->q);
    mat3 rt = transpose3(&b->rot), d, t;
    memset(&d, 0, sizeof(d));
    for (int k = 0; k < 3; k++) d.m[k][k] = b->inertia.v[k];
    t = mul3(&b->rot, &d); b->inertiaW = mul3(&t, &rt);
    for (int k = 0; k < 3; k++) d.m[k][k] = b->inertiaInv.v[k];
    t = mul3(&b->rot, &d); b->inertiaInvW = mul3(&t, &rt);
}

/* RigidBody::initBody(mass, x, inertiaTensor, rotation, ...), RigidBody.h:84-120 */
unsigned orc_add_rigid_body(double mass, const double *x, const double *inertia, const double *q) {
    Model *m = G;
    m->rbs = (RigidBody *)realloc(m->rbs, (size_t)(m->nRb + 1) * sizeof(RigidBody));
    RigidBody *b = &m->rbs[m->nRb];
    memset(b, 0, sizeof(*b));
    b->mass = (real)mass; b->invMass = ((real)mass != R(0.0)) ? R(1.0) / (real)mass : R(0.0);
    b->x = b->x0 = b->lastX = b->oldX = V((real)x[0], (real)x[1], (real)x[2]);
    b->inertia = V((real)inertia[0], (real)inertia[1], (real)inertia[2]);
    b->inertiaInv = V(R(1.0) / b->inertia.v[0], R(1.0) / b->inertia.v[1], R(1.0) / b->inertia.v[2]);
    quat qq = {(real)q[0], (real)q[1], (real)q[2], (real)q[3]};
    b->q = b->q0 = b->lastQ = b->oldQ = qq;
    b->rot = qmatrix(qq);
    rb_rotation_updated(b);
    m->groupsInit = 0;
    return m->nRb++;
}
unsigned orc_num_rigid_bodies(void) { return G->nRb; }
void orc_get_rigid_bodies(double *out) {
    for (unsigned i = 0; i < G->nRb; i++) {
        const RigidBody *b = &G->rbs[i];
        double *o = out + 13 * i;
        for (int k = 0; k < 3; k++) { o[k] = b->x.v[k]; o[7 + k] = b->v.v[k]; o[10 + k] = b->omega.v[k]; }
        o[3] = b->q.w; o[4] = b->q.x; o[5] = b->q.y; o[6] = b->q.z;
    }
}

void orc_set_rigid_body_velocity(unsigned i, const double *v, const double *omega) {
    RigidBody *b = &G->rbs[i];
    b->v = V((real)v[0], (real)v[1], (real)v[2]);
    b->omega = V((real)omega[0], (real)omega[1], (real)omega[2]);
}

/* PositionBasedRigidBodyDynamics::computeMatrixK, PositionBasedRigidBodyDynamics.cpp:11-45 */
static void compute_matrix_k(vec3 connector, real invMass, vec3 x, const mat3 *J, mat3 *K) {
    if (invMass != R(0.0)) {
        const vec3 v = vsub(connector, x);
        const real a = v.v[0], b = v.v[1], c = v.v[2];
        const real j11 = J->m[0][0], j12 = J->m[0][1], j13 = J->m[0][2], j22 = J->m[1][1], j23 = J->m[1][2], j33 = J->m[2][2];
        K->m[0][0] = c * c * j22 - b * c * (j23 + j23) + b * b * j33 + invMass;
        K->m[0][1] = -(c * c * j12) + a * c * j23 + b * c * j13 - a * b * j33;
        K->m[0][2] = b * c * j12 - a * c * j22 - b * b * j13 + a * b * j23;
        K->m[1][0] = K->m[0][1];
        K->m[1][1] = c * c * j11 - a * c * (j13 + j13) + a * a * j33 + invMass;
        K->m[1][2] = -(b * c * j11) + a * c * j12 + a * b * j13 - a * a * j23;
        K->m[2][0] = K->m[0][2];
        K->m[2][1] = K->m[1][2];
        K->m[2][2] = b * b * j11 - a * b * (j12 + j12) + a * a * j22 + invMass;
    } else memset(K, 0, sizeof(*K));
}
/* (K1 + K2).llt().solve(rhs): 3x3 Cholesky */
static vec3 llt_solve(const mat3 *A, vec3 rhs) {
    real l00 = RSQRT(A->m[0][0]);
    real l10 = A->m[1][0] / l00, l20 = A->m[2][0] / l00;
    real l11 = RSQRT(A->m[1][1] - l10 * l10);
    real l21 = (A->m[2][1] - l20 * l10) / l11;
    real l22 = RSQRT(A->m[2][2] - l20 * l20 - l21 * l21);
    real y0 = rhs.v[0] / l00;
    real y1 = (rhs.v[1] - l10 * y0) / l11;
    real y2 = (rhs.v[2] - l20 * y0 - l21 * y1) / l22;
    real z2 = y2 / l22;
    real z1 = (y1 - l21 * z2) / l11;
    real z0 = (y0 - l10 * z1 - l20 * z2) / l00;
    return V(z0, z1, z2);
}
/* apply a positional + rotational correction to a rigid body (BallJoint::solvePositionConstraint, Constraints.cpp:106-121) */
static void rb_apply(RigidBody *b, vec3 r, vec3 pt) { /* r = connector - x, pt = impulse-like vector (sign included) */
    if (b->mass == R(0.0)) return;
    const vec3 ot = mvec(&b->inertiaInvW, vcross(r, pt));
    quat otQ = {R(0.0), ot.v[0], ot.v[1], ot.v[2]};
    quat dq = qmul(otQ, b->q);
    b->x = vadd(b->x, vmul(pt, b->invMass));
    b->q.w += (real)(0.5 * dq.w); b->q.x += (real)(0.5 * dq.x); b->q.y += (real)(0.5 * dq.y); b->q.z += (real)(0.5 * dq.z);
    b->q = qnormalize(b->q);
    rb_rotation_updated(b);
}

/* ------------------------------------------------------------------------------------------------ */
/* constraint factories: <X>Constraint::initConstraint + SimulationModel::add<X>Constraint            */
/* (SimulationModel.cpp:565-806: push_back only when initConstraint returned true; groups invalidated)*/
/* ------------------------------------------------------------------------------------------------ */
static Constraint *new_constraint(Model *m) {
    if (m->nCons == m->capCons) {
        m->capCons = m->capCons ? m->capCons * 2 : 4096;
        m->cons = (Constraint *)realloc(m->cons, (size_t)m->capCons * sizeof(Constraint));
    }
    Constraint *c = &m->cons[m->nCons];
    memset(c, 0, sizeof(*c));
    return c;
}
static void mat3_to_params(const mat3 *a, real *p) { for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) p[3 * r + c] = a->m[r][c]; }
static mat3 params_to_mat3(const real *p) { mat3 a; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) a.m[r][c] = p[3 * r + c]; return a; }

/* p: per-type user parameters (the add*Constraint arguments after the particle indices) */
static int add_constraint(Model *m, int type, const unsigned *b, const real *u) {
    Constraint *c = new_constraint(m);
    c->type = type;
    const vec3 *x0 = m->x0;
    int ok = 1;
    switch (type) {
    case ORC_DISTANCE: case ORC_DISTANCE_XPBD: /* Constraints.cpp:1166-1181, 1211-1227 */
        c->nb = 2; c->p[0] = vnorm(vsub(x0[b[1]], x0[b[0]])); c->p[1] = u[0]; break;
    case ORC_DIHEDRAL: { /* Constraints.cpp:1264-1300 */
        c->nb = 4;
        vec3 p0 = x0[b[0]], p1 = x0[b[1]], p2 = x0[b[2]], p3 = x0[b[3]];
        vec3 e = vsub(p3, p2);
        real elen = vnorm(e);
        if (elen < 1e-6) { ok = 0; break; }
        vec3 n1 = vcross(vsub(p2, p0), vsub(p3, p0)); { real s = vsq(n1); n1 = V(n1.v[0] / s, n1.v[1] / s, n1.v[2] / s); }
        vec3 n2 = vcross(vsub(p3, p1), vsub(p2, p1)); { real s = vsq(n2); n2 = V(n2.v[0] / s, n2.v[1] / s, n2.v[2] / s); }
        n1 = vnormalize(n1); n2 = vnormalize(n2);
        real dot = vdot(n1, n2);
        if (dot < R(-1.0)) dot = R(-1.0);
        if (dot > R(1.0)) dot = R(1.0);
        c->p[0] = RACOS(dot); c->p[1] = u[0];
        break; }
    case ORC_ISOBENDING: case ORC_ISOBENDING_XPBD: /* Constraints.cpp:1345-1364, 1407-1427 */
        c->nb = 4; c->p[0] = u[0];
        ok = init_isobending(x0[b[0]], x0[b[1]], x0[b[2]], x0[b[3]], c->p + 1); break;
    case ORC_FEMTRIANGLE: /* Constraints.cpp:1476-1496 */
        c->nb = 3;
        ok = init_femtriangle(x0[b[0]], x0[b[1]], x0[b[2]], &c->p[0], c->p + 1);
        c->p[5] = u[0]; c->p[6] = u[1]; c->p[7] = u[2]; c->p[8] = u[3]; c->p[9] = u[4]; break;
    case ORC_STRAINTRIANGLE: { /* Constraints.cpp:1544-1569: "bring triangles to xy plane" = take (x, z) */
        c->nb = 3;
        vec3 y1 = V(x0[b[0]].v[0], x0[b[0]].v[2], R(0.0)), y2 = V(x0[b[1]].v[0], x0[b[1]].v[2], R(0.0)),
             y3 = V(x0[b[2]].v[0], x0[b[2]].v[2], R(0.0));
        ok = init_straintriangle(y1, y2, y3, c->p);
        c->p[4] = u[0]; c->p[5] = u[1]; c->p[6] = u[2]; c->p[7] = u[3]; c->p[8] = u[4]; break; }
    case ORC_VOLUME: case ORC_VOLUME_XPBD: { /* Constraints.cpp:1617-1635, 1683-1702 */
        c->nb = 4;
        vec3 p0 = x0[b[0]], p1 = x0[b[1]], p2 = x0[b[2]], p3 = x0[b[3]];
        c->p[0] = RFABS(R(1.0 / 6.0) * vdot(vsub(p3, p0), vcross(vsub(p2, p0), vsub(p1, p0))));
        c->p[1] = u[0]; break; }
    case ORC_FEMTET: case ORC_FEMTET_XPBD: { /* Constraints.cpp:1755-1775, 1830-1852 */
        c->nb = 4; mat3 inv; memset(&inv, 0, sizeof(inv));
        ok = init_femtet(x0[b[0]], x0[b[1]], x0[b[2]], x0[b[3]], &c->p[0], &inv);
        mat3_to_params(&inv, c->p + 1); c->p[10] = u[0]; c->p[11] = u[1]; break; }
    case ORC_STRAINTET: { /* Constraints.cpp:1912-1935 */
        c->nb = 4; mat3 inv; memset(&inv, 0, sizeof(inv));
        ok = init_straintet(x0[b[0]], x0[b[1]], x0[b[2]], x0[b[3]], &inv);
        mat3_to_params(&inv, c->p); c->p[9] = u[0]; c->p[10] = u[1]; c->p[11] = u[2]; c->p[12] = u[3]; break; }
    case ORC_BALLJOINT: { /* BallJoint::initConstraint, Constraints.cpp:54-70 + init_BallJoint, PositionBasedRigidBodyDynamics.cpp:160-186; u = joint position */
        c->nb = 2;
        if (b[0] >= m->nRb || b[1] >= m->nRb) { ok = 0; break; }
        const RigidBody *r0 = &m->rbs[b[0]], *r1 = &m->rbs[b[1]];
        vec3 pos = V(u[0], u[1], u[2]);
        mat3 r0T = qmatrix(r0->q), r1T = qmatrix(r1->q); r0T = transpose3(&r0T); r1T = transpose3(&r1T);
        vec3 l0 = mvec(&r0T, vsub(pos, r0->x)), l1 = mvec(&r1T, vsub(pos, r1->x));
        for (int k = 0; k < 3; k++) { c->p[k] = l0.v[k]; c->p[3 + k] = l1.v[k]; c->p[6 + k] = pos.v[k]; c->p[9 + k] = pos.v[k]; }
        break; }
    case ORC_RB_PARTICLE_BALLJOINT: { /* RigidBodyParticleBallJoint::initConstraint, Constraints.cpp:925-938 + init (PositionBasedRigidBodyDynamics.cpp:2130-2147) */
        c->nb = 2;
        if (b[0] >= m->nRb || b[1] >= m->n) { ok = 0; break; }
        const RigidBody *r0 = &m->rbs[b[0]];
        mat3 r0T = qmatrix(r0->q); r0T = transpose3(&r0T);
        vec3 l0 = mvec(&r0T, vsub(m->x[b[1]], r0->x));
        for (int k = 0; k < 3; k++) { c->p[k] = l0.v[k]; c->p[3 + k] = m->x[b[1]].v[k]; }
        break; }
    case ORC_SHAPEMATCHING: { /* Constraints.cpp:1985-2001: copies of x0 and invMass are frozen into the constraint; u = [k, nc0..nc3] */
        c->nb = 4; c->p[0] = u[0];
        vec3 q[4]; real w[4];
        for (int i = 0; i < 4; i++) { q[i] = x0[b[i]]; w[i] = m->invMass[b[i]]; }
        vec3 rc; ok = init_shapematching(q, w, 4, &rc);
        for (int k = 0; k < 3; k++) c->p[1 + k] = rc.v[k];
        for (int i = 0; i < 4; i++) { for (int k = 0; k < 3; k++) c->p[4 + 3 * i + k] = q[i].v[k]; c->p[16 + i] = w[i]; c->p[20 + i] = u[1 + i]; }
        break; }
    default: ok = 0; break;
    }
    for (unsigned k = 0; k < c->nb; k++) c->b[k] = b[k];
    if (ok) { m->nCons++; m->groupsInit = 0; }
    return ok;
}

int orc_add_constraint(int type, const unsigned *bodies, const double *p) {
    real u[8];
    for (int i = 0; i < 8; i++) u[i] = (real)p[i];
    return add_constraint(G, type, bodies, u);
}

/* SimulationModel::addClothConstraints, SimulationModel.cpp:1125-1184 */
void orc_add_cloth_constraints(unsigned tmIdx, unsigned method, double distK, double xx, double yy, double xy, double pxy,
                               double pyx, int normStretch, int normShear) {
    const TriModel *tm = &G->tris[tmIdx];
    const unsigned off = tm->offset;
    if (method == 1 || method == 4) {
        real u[8] = {(real)distK};
        for (unsigned i = 0; i < tm->nEdges; i++) {
            unsigned b[2] = {tm->edges[i].v[0] + off, tm->edges[i].v[1] + off};
            add_constraint(G, method == 1 ? ORC_DISTANCE : ORC_DISTANCE_XPBD, b, u);
        }
    } else if (method == 2) {
        real u[8] = {(real)xx, (real)yy, (real)xy, (real)pxy, (real)pyx};
        for (unsigned i = 0; i < tm->nFaces; i++) {
            unsigned b[3] = {tm->faces[3 * i] + off, tm->faces[3 * i + 1] + off, tm->faces[3 * i + 2] + off};
            add_constraint(G, ORC_FEMTRIANGLE, b, u);
        }
    } else if (method == 3) {
        real u[8] = {(real)xx, (real)yy, (real)xy, (real)(normStretch != 0), (real)(normShear != 0)};
        for (unsigned i = 0; i < tm->nFaces; i++) {
            unsigned b[3] = {tm->faces[3 * i] + off, tm->faces[3 * i + 1] + off, tm->faces[3 * i + 2] + off};
            add_constraint(G, ORC_STRAINTRIANGLE, b, u);
        }
    }
}

/* SimulationModel::addBendingConstraints, SimulationModel.cpp:1186-1240 */
void orc_add_bending_constraints(unsigned tmIdx, unsigned method, double k) {
    if (method < 1 || method > 3) return;
    const TriModel *tm = &G->tris[tmIdx];
    const unsigned off = tm->offset;
    real u[8] = {(real)k};
    for (unsigned i = 0; i < tm->nEdges; i++) {
        const unsigned tri1 = tm->edges[i].f[0], tri2 = tm->edges[i].f[1];
        if (tri1 == NOFACE || tri2 == NOFACE) continue;
        const unsigned a1 = tm->edges[i].v[0], a2 = tm->edges[i].v[1];
        int point1 = -1, point2 = -1;
        for (int j = 0; j < 3; j++) if (tm->faces[3 * tri1 + j] != a1 && tm->faces[3 * tri1 + j] != a2) { point1 = (int)tm->faces[3 * tri1 + j]; break; }
        for (int j = 0; j < 3; j++) if (tm->faces[3 * tri2 + j] != a1 && tm->faces[3 * tri2 + j] != a2) { point2 = (int)tm->faces[3 * tri2 + j]; break; }
        if (point1 != -1 && point2 != -1) {
            unsigned b[4] = {(unsigned)point1 + off, (unsigned)point2 + off, a1 + off, a2 + off};
            add_constraint(G, method == 1 ? ORC_DIHEDRAL : (method == 2 ? ORC_ISOBENDING : ORC_ISOBENDING_XPBD), b, u);
        }
    }
}

/* SimulationModel::addSolidConstraints, SimulationModel.cpp:1242-1349 */
void orc_add_solid_constraints(unsigned tmIdx, unsigned method, double k, double nu, double volK, int normStretch, int normShear) {
    const TetModel *tm = &G->tets[tmIdx];
    const unsigned off = tm->offset;
    (void)normShear; /* method 4 passes normalizeStretch for both flags, SimulationModel.cpp:1308 */
    if (method == 1 || method == 6) {
        real u[8] = {(real)k};
        for (unsigned i = 0; i < tm->nEdges; i++) {
            unsigned b[2] = {tm->edges[2 * i] + off, tm->edges[2 * i + 1] + off};
            add_constraint(G, method == 1 ? ORC_DISTANCE : ORC_DISTANCE_XPBD, b, u);
        }
        real uv[8] = {(real)volK};
        for (unsigned i = 0; i < tm->nTets; i++) {
            unsigned b[4] = {tm->tets[4 * i] + off, tm->tets[4 * i + 1] + off, tm->tets[4 * i + 2] + off, tm->tets[4 * i + 3] + off};
            add_constraint(G, method == 1 ? ORC_VOLUME : ORC_VOLUME_XPBD, b, uv);
        }
    } else if (method == 2 || method == 3) {
        real u[8] = {(real)k, (real)nu};
        for (unsigned i = 0; i < tm->nTets; i++) {
            unsigned b[4] = {tm->tets[4 * i] + off, tm->tets[4 * i + 1] + off, tm->tets[4 * i + 2] + off, tm->tets[4 * i + 3] + off};
            add_constraint(G, method == 2 ? ORC_FEMTET : ORC_FEMTET_XPBD, b, u);
        }
    } else if (method == 5) { /* one 4-particle cluster per tet; corrections are divided by the number of clusters at the vertex */
        for (unsigned i = 0; i < tm->nTets; i++) {
            unsigned b[4] = {tm->tets[4 * i] + off, tm->tets[4 * i + 1] + off, tm->tets[4 * i + 2] + off, tm->tets[4 * i + 3] + off};
            real u[8] = {(real)k, (real)tm->vertTets[b[0] - off], (real)tm->vertTets[b[1] - off], (real)tm->vertTets[b[2] - off], (real)tm->vertTets[b[3] - off]};
            add_constraint(G, ORC_SHAPEMATCHING, b, u);
        }
    } else if (method == 4) {
        real u[8] = {(real)k, (real)k, (real)(normStretch != 0), (real)(normStretch != 0)};
        for (unsigned i = 0; i < tm->nTets; i++) {
            unsigned b[4] = {tm->tets[4 * i] + off, tm->tets[4 * i + 1] + off, tm->tets[4 * i + 2] + off, tm->tets[4 * i + 3] + off};
            add_constraint(G, ORC_STRAINTET, b, u);
        }
    }
}

void orc_set_params(double dt, unsigned subSteps, unsigned maxIter, int velMethod, const double *g) {
    G->dt = (real)dt; G->subSteps = subSteps; G->maxIter = maxIter; G->velMethod = velMethod;
    G->gravity = V((real)g[0], (real)g[1], (real)g[2]);
}

/* SimulationModel::initConstraintGroups, SimulationModel.cpp:1033-1094: greedy first fit in insertion order,
 * one byte map per colour over the bodies. */
void orc_init_groups(void) {
    Model *m = G;
    if (m->groupsInit) return;
    /* rigid-body and particle indices share ONE index space without offset (SimulationModel.cpp:1041,1058,1070) */
    const unsigned nc = m->nCons, nb = m->n + m->nRb;
    unsigned char **mapping = NULL; unsigned nGroups = 0, capGroups = 0;
    unsigned *colour = (unsigned *)malloc((size_t)(nc ? nc : 1) * sizeof(unsigned));
    unsigned *count = NULL;
    for (unsigned i = 0; i < nc; i++) {
        const Constraint *c = &m->cons[i];
        unsigned g = nGroups;
        for (unsigned j = 0; j < nGroups; j++) {
            int fits = 1;
            for (unsigned k = 0; k < c->nb; k++) if (mapping[j][c->b[k]] != 0) { fits = 0; break; }
            if (fits) { g = j; break; }
        }
        if (g == nGroups) {
            if (nGroups == capGroups) {
                capGroups = capGroups ? capGroups * 2 : 16;
                mapping = (unsigned char **)realloc(mapping, capGroups * sizeof(*mapping));
                count = (unsigned *)realloc(count, capGroups * sizeof(unsigned));
            }
            mapping[nGroups] = (unsigned char *)calloc(nb ? nb : 1, 1);
            count[nGroups] = 0;
            nGroups++;
        }
        for (unsigned k = 0; k < c->nb; k++) mapping[g][c->b[k]] = 1;
        colour[i] = g; count[g]++;
    }
    free(m->groupOff); free(m->groupIds);
    m->groupOff = (unsigned *)malloc((size_t)(nGroups + 1) * sizeof(unsigned));
    m->groupIds = (unsigned *)malloc((size_t)(nc ? nc : 1) * sizeof(unsigned));
    unsigned o = 0;
    for (unsigned g = 0; g < nGroups; g++) { m->groupOff[g] = o; o += count[g]; count[g] = m->groupOff[g]; }
    m->groupOff[nGroups] = o;
    for (unsigned i = 0; i < nc; i++) m->groupIds[count[colour[i]]++] = i;
    m->nGroups = nGroups; m->groupsInit = 1;
    for (unsigned g = 0; g < nGroups; g++) free(mapping[g]);
    free(mapping); free(count); free(colour);
}

unsigned orc_num_particles(void) { return G->n; }
unsigned orc_num_constraints(void) { return G->nCons; }
unsigned orc_num_groups(void) { return G->nGroups; }
void orc_get_groups(unsigned *offsets, unsigned *ids) {
    memcpy(offsets, G->groupOff, (size_t)(G->nGroups + 1) * sizeof(unsigned));
    memcpy(ids, G->groupIds, (size_t)G->nCons * sizeof(unsigned));
}
static vec3 *attr_ptr(int which) {
    switch (which) { case 0: return G->x; case 1: return G->v; case 2: return G->x0; case 3: return G->oldX; case 4: return G->lastX; default: return G->a; }
}
void orc_get_attr(int which, double *out) {
    const vec3 *p = attr_ptr(which);
    for (unsigned i = 0; i < G->n; i++) for (int k = 0; k < 3; k++) out[3 * i + k] = p[i].v[k];
}
void orc_set_attr(int which, const double *in) {
    vec3 *p = attr_ptr(which);
    for (unsigned i = 0; i < G->n; i++) for (int k = 0; k < 3; k++) p[i].v[k] = (real)in[3 * i + k];
}
void orc_get_masses(double *mass, double *invMass) {
    for (unsigned i = 0; i < G->n; i++) { mass[i] = G->mass[i]; invMass[i] = G->invMass[i]; }
}
unsigned orc_tri_num_edges(unsigned tm) { return G->tris[tm].nEdges; }
unsigned orc_tri_num_faces(unsigned tm) { return G->tris[tm].nFaces; }
unsigned orc_tri_index_offset(unsigned tm) { return G->tris[tm].offset; }
void orc_tri_get_edges(unsigned tm, unsigned *out) {
    const TriModel *t = &G->tris[tm];
    for (unsigned i = 0; i < t->nEdges; i++) { out[4 * i] = t->edges[i].v[0]; out[4 * i + 1] = t->edges[i].v[1]; out[4 * i + 2] = t->edges[i].f[0]; out[4 * i + 3] = t->edges[i].f[1]; }
}
void orc_tri_get_faces(unsigned tm, unsigned *out) { memcpy(out, G->tris[tm].faces, (size_t)3 * G->tris[tm].nFaces * sizeof(unsigned)); }
unsigned orc_tet_num_edges(unsigned tm) { return G->tets[tm].nEdges; }
unsigned orc_tet_num_tets(unsigned tm) { return G->tets[tm].nTets; }
unsigned orc_tet_index_offset(unsigned tm) { return G->tets[tm].offset; }
void orc_tet_get_edges(unsigned tm, unsigned *out) { memcpy(out, G->tets[tm].edges, (size_t)2 * G->tets[tm].nEdges * sizeof(unsigned)); }
void orc_tet_get_tets(unsigned tm, unsigned *out) { memcpy(out, G->tets[tm].tets, (size_t)4 * G->tets[tm].nTets * sizeof(unsigned)); }

static int nparams_of(int type) {
    static const int n[ORC_NUM_TYPES] = {2, 2, 2, 17, 17, 10, 9, 2, 2, 12, 12, 13, 24, 12, 6};
    return (type >= 0 && type < ORC_NUM_TYPES) ? n[type] : 0;
}
int orc_get_constraint(unsigned i, unsigned *bodies, double *p, double *lambda) {
    const Constraint *c = &G->cons[i];
    for (unsigned k = 0; k < c->nb; k++) bodies[k] = c->b[k];
    for (int k = 0; k < nparams_of(c->type); k++) p[k] = c->p[k];
    *lambda = c->lambda;
    return c->type;
}
void orc_get_constraints(int *types, unsigned *bodies, double *params, int *nbodies) {
    for (unsigned i = 0; i < G->nCons; i++) {
        const Constraint *c = &G->cons[i];
        types[i] = c->type; nbodies[i] = (int)c->nb;
        for (unsigned k = 0; k < 4; k++) bodies[4 * i + k] = k < c->nb ? c->b[k] : NOFACE;
        for (int k = 0; k < ORC_MAX_PARAMS; k++) params[(size_t)ORC_MAX_PARAMS * i + k] = k < nparams_of(c->type) ? c->p[k] : 0.0;
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* <X>Constraint::solvePositionConstraint: gather, call the solver, scatter x += corr where invMass!=0 */
/* ------------------------------------------------------------------------------------------------ */
static void solve_position_constraint(Model *m, Constraint *c, unsigned iter, real dt) {
    vec3 *x = m->x; const real *w = m->invMass;
    const unsigned *b = c->b;
    vec3 corr[4] = {VZERO, VZERO, VZERO, VZERO};
    int res = 0;
    switch (c->type) {
    case ORC_DISTANCE: /* Constraints.cpp:1183-1206 */
        res = solve_distance(x[b[0]], w[b[0]], x[b[1]], w[b[1]], c->p[0], c->p[1], &corr[0], &corr[1]); break;
    case ORC_DISTANCE_XPBD: /* Constraints.cpp:1227-1258: lambda reset at iter 0, dt = TimeManager step (substep h) */
        if (iter == 0) c->lambda = R(0.0);
        res = solve_distance_xpbd(x[b[0]], w[b[0]], x[b[1]], w[b[1]], c->p[0], c->p[1], dt, &c->lambda, &corr[0], &corr[1]); break;
    case ORC_DIHEDRAL: /* Constraints.cpp:1302-1339 */
        res = solve_dihedral(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], x[b[3]], w[b[3]], c->p[0], c->p[1], &corr[0], &corr[1], &corr[2], &corr[3]); break;
    case ORC_ISOBENDING: /* Constraints.cpp:1366-1402 */
        res = solve_isobending(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], x[b[3]], w[b[3]], c->p + 1, c->p[0], &corr[0], &corr[1], &corr[2], &corr[3]); break;
    case ORC_ISOBENDING_XPBD: /* Constraints.cpp:1429-1471 */
        if (iter == 0) c->lambda = R(0.0);
        res = solve_isobending_xpbd(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], x[b[3]], w[b[3]], c->p + 1, c->p[0], dt, &c->lambda, &corr[0], &corr[1], &corr[2], &corr[3]); break;
    case ORC_FEMTRIANGLE: /* Constraints.cpp:1498-1538 */
        res = solve_femtriangle(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], c->p[0], c->p + 1, c->p[5], c->p[6], c->p[7], c->p[8], c->p[9], &corr[0], &corr[1], &corr[2]); break;
    case ORC_STRAINTRIANGLE: /* Constraints.cpp:1565-1610 */
        res = solve_straintriangle(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], c->p, c->p[4], c->p[5], c->p[6], c->p[7] != 0, c->p[8] != 0, &corr[0], &corr[1], &corr[2]); break;
    case ORC_VOLUME: /* Constraints.cpp:1637-1677 */
        res = solve_volume(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], x[b[3]], w[b[3]], c->p[0], c->p[1], &corr[0], &corr[1], &corr[2], &corr[3]); break;
    case ORC_VOLUME_XPBD: /* Constraints.cpp:1704-1750 */
        if (iter == 0) c->lambda = R(0.0);
        res = solve_volume_xpbd(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], x[b[3]], w[b[3]], c->p[0], c->p[1], dt, &c->lambda, &corr[0], &corr[1], &corr[2], &corr[3]); break;
    case ORC_FEMTET: case ORC_FEMTET_XPBD: { /* Constraints.cpp:1777-1825, 1854-1906 */
        vec3 x1 = x[b[0]], x2 = x[b[1]], x3 = x[b[2]], x4 = x[b[3]];
        real currentVolume = -R(1.0 / 6.0) * vdot(vsub(x4, x1), vcross(vsub(x3, x1), vsub(x2, x1)));
        int handleInversion = 0;
        if (currentVolume / c->p[0] < 0.2) handleInversion = 1;
        mat3 inv = params_to_mat3(c->p + 1);
        if (c->type == ORC_FEMTET)
            res = solve_femtet(x1, w[b[0]], x2, w[b[1]], x3, w[b[2]], x4, w[b[3]], c->p[0], &inv, c->p[10], c->p[11], handleInversion, &corr[0], &corr[1], &corr[2], &corr[3]);
        else {
            if (iter == 0) c->lambda = R(0.0);
            res = solve_femtet_xpbd(x1, w[b[0]], x2, w[b[1]], x3, w[b[2]], x4, w[b[3]], c->p[0], &inv, c->p[10], c->p[11], handleInversion, dt, &c->lambda, &corr[0], &corr[1], &corr[2], &corr[3]);
        }
        break; }
    case ORC_STRAINTET: { /* Constraints.cpp:1937-1980: scalar stiffness * Vector3r::Ones() */
        mat3 inv = params_to_mat3(c->p);
        vec3 ks = V(c->p[9], c->p[9], c->p[9]), kh = V(c->p[10], c->p[10], c->p[10]);
        res = solve_straintet(x[b[0]], w[b[0]], x[b[1]], w[b[1]], x[b[2]], w[b[2]], x[b[3]], w[b[3]], &inv, ks, kh, c->p[11] != 0, c->p[12] != 0, &corr[0], &corr[1], &corr[2], &corr[3]);
        break; }
    case ORC_BALLJOINT: { /* BallJoint::updateConstraint + solvePositionConstraint (Constraints.cpp:72-125), solve_BallJoint (PositionBasedRigidBodyDynamics.cpp:212-262) */
        RigidBody *r0 = &m->rbs[b[0]], *r1 = &m->rbs[b[1]];
        mat3 R0 = qmatrix(r0->q), R1 = qmatrix(r1->q);
        vec3 c0 = vadd(mvec(&R0, V(c->p[0], c->p[1], c->p[2])), r0->x), c1 = vadd(mvec(&R1, V(c->p[3], c->p[4], c->p[5])), r1->x);
        for (int k = 0; k < 3; k++) { c->p[6 + k] = c0.v[k]; c->p[9 + k] = c1.v[k]; }
        mat3 K1, K2, K;
        compute_matrix_k(c0, r0->invMass, r0->x, &r0->inertiaInvW, &K1);
        compute_matrix_k(c1, r1->invMass, r1->x, &r1->inertiaInvW, &K2);
        for (int a = 0; a < 3; a++) for (int d = 0; d < 3; d++) K.m[a][d] = K1.m[a][d] + K2.m[a][d];
        vec3 pt = llt_solve(&K, vsub(c1, c0));
        const vec3 ra = vsub(c0, r0->x), rb_ = vsub(c1, r1->x);  /* both lever arms from the state before either body moves */
        if (r0->invMass != R(0.0)) rb_apply(r0, ra, pt);
        if (r1->invMass != R(0.0)) rb_apply(r1, rb_, vneg(pt));
        return; }
    case ORC_RB_PARTICLE_BALLJOINT: { /* Constraints.cpp:940-987, solve_RigidBodyParticleBallJoint (PositionBasedRigidBodyDynamics.cpp:2168-2217) */
        RigidBody *r0 = &m->rbs[b[0]];
        const unsigned pi = b[1];
        mat3 R0 = qmatrix(r0->q);
        vec3 c0 = vadd(mvec(&R0, V(c->p[0], c->p[1], c->p[2])), r0->x);
        for (int k = 0; k < 3; k++) c->p[3 + k] = c0.v[k];
        mat3 K;
        compute_matrix_k(c0, r0->invMass, r0->x, &r0->inertiaInvW, &K);
        if (w[pi] != R(0.0)) { K.m[0][0] += w[pi]; K.m[1][1] += w[pi]; K.m[2][2] += w[pi]; }
        vec3 pt = llt_solve(&K, vsub(x[pi], c0));
        if (r0->invMass != R(0.0)) rb_apply(r0, vsub(c0, r0->x), pt);
        if (m->mass[pi] != R(0.0) && w[pi] != R(0.0)) x[pi] = vadd(x[pi], vmul(pt, -w[pi]));
        return; }
    case ORC_SHAPEMATCHING: { /* Constraints.cpp:2003-2028: uses the frozen m_x0 / m_w copies; 1/numClusters averaging */
        vec3 q0[4], xs[4]; real ws[4];
        for (int i = 0; i < 4; i++) { q0[i] = V(c->p[4 + 3 * i], c->p[5 + 3 * i], c->p[6 + 3 * i]); xs[i] = x[b[i]]; ws[i] = c->p[16 + i]; }
        if (solve_shapematching(q0, xs, ws, 4, V(c->p[1], c->p[2], c->p[3]), c->p[0], corr))
            for (int i = 0; i < 4; i++)
                if (ws[i] != R(0.0)) x[b[i]] = vadd(x[b[i]], vmul(corr[i], (real)(1.0 / (unsigned)c->p[20 + i])));
        return; }
    default: break;
    }
    if (res)
        for (unsigned k = 0; k < c->nb; k++)
            if (w[b[k]] != R(0.0)) x[b[k]] = vadd(x[b[k]], corr[k]);
}

/* TimeStepController::positionConstraintProjection, TimeStepController.cpp:251-295 */
static void position_constraint_projection(Model *m, real h) {
    orc_init_groups();
    for (unsigned iter = 0; iter < m->maxIter; iter++) {
        for (unsigned g = 0; g < m->nGroups; g++) {
            const int first = (int)m->groupOff[g], size = (int)(m->groupOff[g + 1] - m->groupOff[g]);
#pragma omp parallel for schedule(static) if (size > MIN_PARALLEL_SIZE)
            for (int i = 0; i < size; i++) solve_position_constraint(m, &m->cons[m->groupIds[first + i]], iter, h);
        }
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* contact path: particles against analytic distance fields on static rigid bodies                   */
/* ------------------------------------------------------------------------------------------------ */
/* DistanceFieldCollision{Box,Sphere,Torus,Cylinder,HollowSphere,HollowBox}::distance, DistanceFieldCollisionDetection.cpp:598-682
 * (evaluated in double precision there as here) */
static double coll_distance(const struct RigidColl *c, const double x[3], double tol) {
    const double inv = c->invert;
    switch (c->shape) {
    case 0: { /* box, :598-605 */
        const double d[3] = {fabs(x[0]) - c->dim[0], fabs(x[1]) - c->dim[1], fabs(x[2]) - c->dim[2]};
        const double m[3] = {fmax(d[0], 0.0), fmax(d[1], 0.0), fmax(d[2], 0.0)};
        return inv * (fmin(fmax(d[0], fmax(d[1], d[2])), 0.0) + sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2])) - tol;
    }
    case 1: return inv * (sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]) - c->dim[0]) - tol; /* sphere, :607-612 */
    case 2: { /* torus, :632-637 (the ring distance is taken in Real precision there) */
        const real rx = (real)x[0], rz = (real)x[2];
        const double q0 = (double)RSQRT(rx * rx + rz * rz) - c->dim[0], q1 = x[1];
        return inv * (sqrt(q0 * q0 + q1 * q1) - c->dim[1]) - tol;
    }
    case 3: { /* cylinder, :639-645 */
        const double l = sqrt(x[0] * x[0] + x[2] * x[2]);
        const double d[2] = {fabs(l) - c->dim[0], fabs(x[1]) - c->dim[1]};
        const double m[2] = {fmax(d[0], 0.0), fmax(d[1], 0.0)};
        return inv * (fmin(fmax(d[0], d[1]), 0.0) + sqrt(m[0] * m[0] + m[1] * m[1])) - tol;
    }
    case 4: return inv * (fabs(sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]) - c->dim[0]) - c->thickness) - tol; /* hollow sphere, :648-653 */
    default: { /* hollow box, :675-682 */
        const double d[3] = {fabs(x[0]) - c->dim[0], fabs(x[1]) - c->dim[1], fabs(x[2]) - c->dim[2]};
        const double m[3] = {fmax(d[0], 0.0), fmax(d[1], 0.0), fmax(d[2], 0.0)};
        return inv * (fabs(fmin(fmax(d[0], fmax(d[1], d[2])), 0.0) + sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2])) - c->thickness) - tol;
    }
    }
}
/* collisionTest: the analytic overrides of the sphere (:614-630) and the hollow sphere (:655-673), else DistanceFieldCollisionObject::
 * collisionTest with approximateNormal (:684-728) */
static int coll_test(const struct RigidColl *c, vec3 x, real tol, vec3 *cp, vec3 *n, real *dist) {
    if (c->shape == 1 || c->shape == 4) {
        const real dl = vnorm(x), r = (real)c->dim[0], inv = (real)c->invert;
        *dist = (c->shape == 4) ? inv * (RFABS(dl - r) - (real)c->thickness) - tol : inv * (dl - r) - tol;
        if (!(*dist < R(0.0))) return 0;
        if (dl < R(1.e-6)) *n = V(0, 0, 0);
        else if (c->shape == 4 && dl < r) *n = vmul(vmul(x, -inv), R(1.0) / dl);
        else *n = vmul(vmul(x, inv), R(1.0) / dl);
        *cp = (c->shape == 4) ? vsub(x, vmul(*n, *dist)) : vmul(*n, r + tol);
        return 1;
    }
    const double xd[3] = {(double)x.v[0], (double)x.v[1], (double)x.v[2]};
    *dist = (real)coll_distance(c, xd, (double)tol);
    if (!(*dist < R(0.0))) return 0;
    const double eps = 1.e-6;
    double xt[3] = {xd[0], xd[1], xd[2]};
    for (int j = 0; j < 3; j++) {
        xt[j] = xd[j] + eps; const double ep = coll_distance(c, xt, (double)tol);
        xt[j] = xd[j] - eps; const double em = coll_distance(c, xt, (double)tol);
        xt[j] = xd[j];
        n->v[j] = (real)((ep - em) * (1.0 / (2.0 * eps)));
    }
    const real norm2 = vsq(*n);
    if (norm2 < R(1.e-6)) *n = V(0, 0, 0); else *n = vmul(*n, R(1.0) / RSQRT(norm2));
    *cp = vsub(x, vmul(*n, *dist));
    return 1;
}
/* DistanceFieldCollisionDetection::collisionDetection + collisionDetectionRBSolid (:26-197, :290-357) for static bodies, every point tested
 * (the bounding-sphere hierarchy only prunes), then ParticleRigidBodyContactConstraint::initConstraint (Constraints.cpp:2115-2145) +
 * init_ParticleRigidBodyContactConstraint (PositionBasedRigidBodyDynamics.cpp:2386-2451) */
static void contact_detection(Model *m) {
    m->nContacts = 0;  /* SimulationModel::resetContacts */
    for (unsigned pi = 0; pi < m->nPartColl; pi++)
        for (unsigned k = 0; k < m->nRigidColl; k++) {
            const struct PartColl *pc = &m->partColl[pi];
            const struct RigidColl *c = &m->rigidColl[k];
            const RigidBody *rb = &m->rbs[c->body];
            for (unsigned i = pc->offset; i < pc->offset + pc->count; i++) {
                const vec3 xw = m->x[i];
                if (xw.v[0] < c->lo[0] || xw.v[1] < c->lo[1] || xw.v[2] < c->lo[2] || xw.v[0] > c->hi[0] || xw.v[1] > c->hi[1] || xw.v[2] > c->hi[2]) continue;
                const vec3 d = vsub(xw, rb->x);
                vec3 xl, cp, nl; real dist;
                for (int r = 0; r < 3; r++) xl.v[r] = c->Rm[3 * r] * d.v[0] + c->Rm[3 * r + 1] * d.v[1] + c->Rm[3 * r + 2] * d.v[2] + c->v1[r];
                if (!coll_test(c, xl, m->contactTolerance, &cp, &nl, &dist)) continue;
                if (m->nContacts == m->capContacts) { m->capContacts = m->capContacts ? 2 * m->capContacts : 256; m->contacts = (struct Contact *)realloc(m->contacts, (size_t)m->capContacts * sizeof(struct Contact)); }
                struct Contact *ct = &m->contacts[m->nContacts++];
                ct->particle = i; ct->body = c->body; ct->cp0 = xw; ct->sum = R(0.0); ct->stiffness = m->contactStiffness; ct->friction = pc->friction + c->friction;
                for (int r = 0; r < 3; r++) {  /* cp_w = R^T cp + v2, n_w = R^T n */
                    ct->cp1.v[r] = c->Rm[r] * cp.v[0] + c->Rm[3 + r] * cp.v[1] + c->Rm[6 + r] * cp.v[2] + c->v2[r];
                    ct->n.v[r] = c->Rm[r] * nl.v[0] + c->Rm[3 + r] * nl.v[1] + c->Rm[6 + r] * nl.v[2];
                }
                const real restitution = pc->restitution * c->restitution, invMass0 = m->invMass[i];
                const vec3 r1 = vsub(ct->cp1, rb->x);
                const vec3 u1 = vadd(rb->v, vcross(rb->omega, r1));
                const vec3 urel = vsub(m->v[i], u1);
                const real urn = vdot(ct->n, urel);
                ct->t = vsub(urel, vmul(ct->n, urn));
                const real tl2 = vsq(ct->t);
                if (tl2 > R(1.0e-6)) ct->t = vmul(ct->t, R(1.0) / RSQRT(tl2));
                /* computeMatrixK of a static body is zero: K = invMass0 * I */
                const real kd = (invMass0 != R(0.0)) ? invMass0 : R(0.0);
                ct->nKnInv = R(1.0) / (kd * vsq(ct->n));
                ct->pMax = R(1.0) / (kd * vsq(ct->t)) * vdot(urel, ct->t);
                ct->goal = (urn < R(0.0)) ? -restitution * urn : R(0.0);
            }
        }
}
/* TimeStepController::velocityConstraintProjection (TimeStepController.cpp:298-357; the particle constraints' velocity hooks are no-ops) over the
 * contact list + velocitySolve_ParticleRigidBodyContactConstraint (PositionBasedRigidBodyDynamics.cpp:2454-2537) */
static void contact_velocity_projection(Model *m) {
    for (unsigned it = 0; it < m->maxIterV; it++)
        for (unsigned k = 0; k < m->nContacts; k++) {
            struct Contact *ct = &m->contacts[k];
            const unsigned i = ct->particle;
            const RigidBody *rb = &m->rbs[ct->body];
            const real invMass0 = m->invMass[i];
            if (invMass0 == R(0.0) && rb->invMass == R(0.0)) continue;
            const real d = vdot(ct->n, vsub(ct->cp0, ct->cp1));
            const vec3 r1 = vsub(ct->cp1, rb->x);
            const vec3 u1 = vadd(rb->v, vcross(rb->omega, r1));
            const vec3 urel = vsub(m->v[i], u1);
            const real urn = vdot(urel, ct->n);
            real mag = ct->nKnInv * (ct->goal - urn);
            if (mag < -ct->sum) mag = -ct->sum;
            if (d < R(0.0)) mag -= ct->stiffness * ct->nKnInv * d;
            vec3 p = vmul(ct->n, mag);
            ct->sum += mag;
            const real pn = vdot(p, ct->n);
            if (ct->friction * pn > ct->pMax) p = vsub(p, vmul(ct->t, ct->pMax));
            else if (ct->friction * pn < -ct->pMax) p = vadd(p, vmul(ct->t, ct->pMax));
            else p = vsub(p, vmul(ct->t, ct->friction * pn));
            if (m->mass[i] != R(0.0)) m->v[i] = vadd(m->v[i], vmul(p, invMass0));
        }
}

/* TimeStepController::step, TimeStepController.cpp:75-241, particle part only
 * (no rigid bodies / orientations / collision detection; velocity constraints are no-ops for particle constraints) */
static void step_once(Model *m) {
    const real hOld = m->dt;
    const int n = (int)m->n;
    /* TimeStep::clearAccelerations, TimeStep.cpp:28-62 */
    for (int i = 0; i < n; i++) if (m->mass[i] != R(0.0)) m->a[i] = m->gravity;
    for (unsigned i = 0; i < m->nRb; i++) if (m->rbs[i].mass != R(0.0)) m->rbs[i].a = m->gravity;
    const real h = hOld / (real)m->subSteps;
    for (unsigned s = 0; s < m->subSteps; s++) {
        for (unsigned i = 0; i < m->nRb; i++) { /* TimeStepController.cpp:97-107, TimeIntegration.cpp:7-19, 22-39 */
            RigidBody *b = &m->rbs[i];
            b->lastX = b->oldX; b->oldX = b->x;
            if (b->mass != R(0.0)) { b->v = vadd(b->v, vmul(b->a, h)); b->x = vadd(b->x, vmul(b->v, h)); }
            b->lastQ = b->oldQ; b->oldQ = b->q;
            if (b->mass != R(0.0)) {
                vec3 t = vsub(b->torque, vcross(b->omega, mvec(&b->inertiaW, b->omega)));
                b->omega = vadd(b->omega, vmul(mvec(&b->inertiaInvW, t), h));
                quat wq = {R(0.0), b->omega.v[0], b->omega.v[1], b->omega.v[2]};
                quat dq = qmul(wq, b->q);
                const double hh = (double)h * 0.5;
                b->q.w += (real)(hh * dq.w); b->q.x += (real)(hh * dq.x); b->q.y += (real)(hh * dq.y); b->q.z += (real)(hh * dq.z);
                b->q = qnormalize(b->q);
            }
            rb_rotation_updated(b);
        }
#pragma omp parallel for schedule(static)
        for (int i = 0; i < n; i++) { /* :112-118 + TimeIntegration::semiImplicitEuler, TimeIntegration.cpp:7-19 */
            m->lastX[i] = m->oldX[i];
            m->oldX[i] = m->x[i];
            if (m->mass[i] != R(0.0)) {
                m->v[i] = vadd(m->v[i], vmul(m->a[i], h));
                m->x[i] = vadd(m->x[i], vmul(m->v[i], h));
            }
        }
        position_constraint_projection(m, h);
        for (unsigned i = 0; i < m->nRb; i++) { /* TimeStepController.cpp:139-152, TimeIntegration.cpp:42-66, 69-95 (angular: first order in both modes) */
            RigidBody *b = &m->rbs[i];
            if (b->mass == R(0.0)) continue;
            if (m->velMethod == 0) b->v = vmul(vsub(b->x, b->oldX), (real)(1.0 / h));
            else {
                vec3 t;
                for (int k = 0; k < 3; k++) t.v[k] = (real)(1.5 * b->x.v[k]) - (real)(2.0 * b->oldX.v[k]) + (real)(0.5 * b->lastX.v[k]);
                b->v = vmul(t, (real)(1.0 / h));
            }
            quat rel = qmul(b->q, qconj(b->oldQ));
            b->omega = vmul(V(rel.x, rel.y, rel.z), (real)(2.0 / h));
        }
#pragma omp parallel for schedule(static)
        for (int i = 0; i < n; i++) { /* :155-162 + TimeIntegration.cpp:42-51 / 69-79 */
            if (m->mass[i] == R(0.0)) continue;
            if (m->velMethod == 0) {
                m->v[i] = vmul(vsub(m->x[i], m->oldX[i]), (real)(1.0 / h));
            } else {
                vec3 t;
                for (int k = 0; k < 3; k++)
                    t.v[k] = (real)(1.5 * m->x[i].v[k]) - (real)(2.0 * m->oldX[i].v[k]) + (real)(0.5 * m->lastX[i].v[k]);
                m->v[i] = vmul(t, (real)(1.0 / h));
            }
        }
    }
    if (m->nRigidColl && m->nPartColl) { contact_detection(m); contact_velocity_projection(m); } /* TimeStepController.cpp:189-196 */
    m->time += hOld; /* TimeStepController.cpp:239 */
}

/* colliders in the layout of oracle/ref_driver's ref_collision_object_info (what an adapter hands to pbd_set_colliders): models = 4 doubles
 * each (offset, count, restitution, friction), rigid = 30 doubles each */
void orc_set_colliders(unsigned nModels, const double *models, unsigned nRigid, const double *rigid) {
    Model *m = G;
    m->partColl = (struct PartColl *)realloc(m->partColl, (size_t)(nModels ? nModels : 1) * sizeof(struct PartColl)); m->nPartColl = nModels;
    m->rigidColl = (struct RigidColl *)realloc(m->rigidColl, (size_t)(nRigid ? nRigid : 1) * sizeof(struct RigidColl)); m->nRigidColl = nRigid;
    for (unsigned i = 0; i < nModels; i++) {
        struct PartColl *p = &m->partColl[i];
        p->offset = (unsigned)models[4 * i]; p->count = (unsigned)models[4 * i + 1]; p->restitution = (real)models[4 * i + 2]; p->friction = (real)models[4 * i + 3];
    }
    for (unsigned i = 0; i < nRigid; i++) {
        const double *d = rigid + 30 * (size_t)i;
        struct RigidColl *c = &m->rigidColl[i];
        c->shape = (int)d[0]; c->body = (unsigned)d[1];
        for (int k = 0; k < 3; k++) c->dim[k] = (double)(real)d[2 + k];  /* the reference stores the dimensions in Real */
        c->thickness = (double)(real)d[5]; c->invert = d[6] != 0.0 ? -1.0 : 1.0; c->restitution = (real)d[7]; c->friction = (real)d[8];
        for (int k = 0; k < 9; k++) c->Rm[k] = (real)d[9 + k];
        for (int k = 0; k < 3; k++) { c->v1[k] = (real)d[18 + k]; c->v2[k] = (real)d[21 + k]; c->lo[k] = (real)d[24 + k]; c->hi[k] = (real)d[27 + k]; }
    }
}
void orc_set_contact_params(double tolerance, double stiffness, unsigned maxIterV) {
    G->contactTolerance = (real)tolerance; G->contactStiffness = (real)stiffness; G->maxIterV = maxIterV;
}
unsigned orc_num_contacts(void) { return G->nContacts; }
void orc_get_contacts(unsigned *particle, unsigned *body, double *out) { /* 10 doubles per contact: cp0 | cp1 | n | 1/(n^T K n) */
    for (unsigned i = 0; i < G->nContacts; i++) {
        const struct Contact *c = &G->contacts[i];
        particle[i] = c->particle; body[i] = c->body;
        for (int k = 0; k < 3; k++) { out[10 * i + k] = c->cp0.v[k]; out[10 * i + 3 + k] = c->cp1.v[k]; out[10 * i + 6 + k] = c->n.v[k]; }
        out[10 * i + 9] = c->nKnInv;
    }
}

double orc_step(int n) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int i = 0; i < n; i++) step_once(G);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
double orc_time(void) { return G->time; }

/* ------------------------------------------------------------------------------------------------ */
/* known-answer entry points (same signatures as oracle/ref_driver/ref_driver.cpp)                    */
/* ------------------------------------------------------------------------------------------------ */
int orc_kat_solve(int type, const double *xd, const double *wd, const double *pd, double dtd, int handleInversion,
                  double *lambda, double *corr) {
    vec3 X[4], C[4] = {VZERO, VZERO, VZERO, VZERO};
    real W[4], p[ORC_MAX_PARAMS];
    for (int i = 0; i < 4; i++) { X[i] = V((real)xd[3 * i], (real)xd[3 * i + 1], (real)xd[3 * i + 2]); W[i] = (real)wd[i]; }
    for (int i = 0; i < nparams_of(type); i++) p[i] = (real)pd[i];
    real lam = (real)*lambda, dt = (real)dtd;
    int res = -1;
    switch (type) {
    case ORC_DISTANCE: res = solve_distance(X[0], W[0], X[1], W[1], p[0], p[1], &C[0], &C[1]); break;
    case ORC_DISTANCE_XPBD: res = solve_distance_xpbd(X[0], W[0], X[1], W[1], p[0], p[1], dt, &lam, &C[0], &C[1]); break;
    case ORC_DIHEDRAL: res = solve_dihedral(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], p[0], p[1], &C[0], &C[1], &C[2], &C[3]); break;
    case ORC_ISOBENDING: res = solve_isobending(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], p + 1, p[0], &C[0], &C[1], &C[2], &C[3]); break;
    case ORC_ISOBENDING_XPBD: res = solve_isobending_xpbd(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], p + 1, p[0], dt, &lam, &C[0], &C[1], &C[2], &C[3]); break;
    case ORC_FEMTRIANGLE: res = solve_femtriangle(X[0], W[0], X[1], W[1], X[2], W[2], p[0], p + 1, p[5], p[6], p[7], p[8], p[9], &C[0], &C[1], &C[2]); break;
    case ORC_STRAINTRIANGLE: res = solve_straintriangle(X[0], W[0], X[1], W[1], X[2], W[2], p, p[4], p[5], p[6], p[7] != 0, p[8] != 0, &C[0], &C[1], &C[2]); break;
    case ORC_VOLUME: res = solve_volume(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], p[0], p[1], &C[0], &C[1], &C[2], &C[3]); break;
    case ORC_VOLUME_XPBD: res = solve_volume_xpbd(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], p[0], p[1], dt, &lam, &C[0], &C[1], &C[2], &C[3]); break;
    case ORC_FEMTET: { mat3 inv = params_to_mat3(p + 1); res = solve_femtet(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], p[0], &inv, p[10], p[11], handleInversion, &C[0], &C[1], &C[2], &C[3]); break; }
    case ORC_FEMTET_XPBD: { mat3 inv = params_to_mat3(p + 1); res = solve_femtet_xpbd(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], p[0], &inv, p[10], p[11], handleInversion, dt, &lam, &C[0], &C[1], &C[2], &C[3]); break; }
    case ORC_STRAINTET: { mat3 inv = params_to_mat3(p); res = solve_straintet(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], &inv, V(p[9], p[9], p[9]), V(p[10], p[10], p[10]), p[11] != 0, p[12] != 0, &C[0], &C[1], &C[2], &C[3]); break; }
    case ORC_SHAPEMATCHING: { /* raw solver answer (before the 1/numClusters averaging of the constraint class); w argument ignored: frozen copies in p */
        vec3 q0[4]; real ws[4];
        for (int i = 0; i < 4; i++) { q0[i] = V(p[4 + 3 * i], p[5 + 3 * i], p[6 + 3 * i]); ws[i] = p[16 + i]; }
        res = solve_shapematching(q0, X, ws, 4, V(p[1], p[2], p[3]), p[0], C); break; }
    default: return -1;
    }
    *lambda = lam;
    for (int i = 0; i < 4; i++) for (int k = 0; k < 3; k++) corr[3 * i + k] = C[i].v[k];
    return res;
}

int orc_kat_init(int type, const double *xd, double *out) {
    vec3 X[4];
    for (int i = 0; i < 4; i++) X[i] = V((real)xd[3 * i], (real)xd[3 * i + 1], (real)xd[3 * i + 2]);
    switch (type) {
    case ORC_ISOBENDING: case ORC_ISOBENDING_XPBD: { real Q[16]; int r = init_isobending(X[0], X[1], X[2], X[3], Q); for (int i = 0; i < 16; i++) out[i] = Q[i]; return r; }
    case ORC_FEMTRIANGLE: { real area = 0, inv[4] = {0}; int r = init_femtriangle(X[0], X[1], X[2], &area, inv); out[0] = area; for (int i = 0; i < 4; i++) out[1 + i] = inv[i]; return r; }
    case ORC_STRAINTRIANGLE: { real inv[4] = {0}; int r = init_straintriangle(X[0], X[1], X[2], inv); for (int i = 0; i < 4; i++) out[i] = inv[i]; return r; }
    case ORC_FEMTET: case ORC_FEMTET_XPBD: { real vol = 0, q[9]; mat3 inv; memset(&inv, 0, sizeof(inv)); int r = init_femtet(X[0], X[1], X[2], X[3], &vol, &inv); mat3_to_params(&inv, q); out[0] = vol; for (int i = 0; i < 9; i++) out[1 + i] = q[i]; return r; }
    case ORC_STRAINTET: { real q[9]; mat3 inv; memset(&inv, 0, sizeof(inv)); int r = init_straintet(X[0], X[1], X[2], X[3], &inv); mat3_to_params(&inv, q); for (int i = 0; i < 9; i++) out[i] = q[i]; return r; }
    default: return -1;
    }
}

void orc_kat_svd(const double *Ad, double *sigma, double *Ud, double *VTd) {
    mat3 A, U, VT; vec3 s;
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) A.m[r][c] = (real)Ad[3 * r + c];
    svd_inversion(&A, &s, &U, &VT);
    for (int r = 0; r < 3; r++) { sigma[r] = s.v[r]; for (int c = 0; c < 3; c++) { Ud[3 * r + c] = U.m[r][c]; VTd[3 * r + c] = VT.m[r][c]; } }
}

/* TimeIntegration::semiImplicitEuler, TimeIntegration.cpp:7-19 */
void orc_kat_integrate(double h, double mass, double *x, double *v, const double *a) {
    if ((real)mass != R(0.0))
        for (int k = 0; k < 3; k++) {
            real vv = (real)v[k] + (real)a[k] * (real)h;
            real xx = (real)x[k] + vv * (real)h;
            v[k] = vv; x[k] = xx;
        }
}
/* TimeIntegration::velocityUpdateFirstOrder / SecondOrder, TimeIntegration.cpp:42-51, 69-79 */
void orc_kat_velocity_update(int order, double hd, double mass, const double *x, const double *oldX, const double *lastX, double *v) {
    if ((real)mass == R(0.0)) return;
    real h = (real)hd;
    for (int k = 0; k < 3; k++) {
        if (order == 0) v[k] = (real)(1.0 / h) * ((real)x[k] - (real)oldX[k]);
        else v[k] = (real)(1.0 / h) * ((real)(1.5 * (real)x[k]) - (real)(2.0 * (real)oldX[k]) + (real)(0.5 * (real)lastX[k]));
    }
}
