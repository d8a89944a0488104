// positionbaseddynamics_b200/csrc/kernels.cuh
//
// sm_90a kernels of the PBD/XPBD step.  One thread projects one constraint: it loads the constraint's particle
// indices (coalesced), gathers the particle float4s through L1 (plain ld.global, see ldp), runs the projection in
// registers and scatters the float4s back (st.global.cg).  Colours guarantee disjoint particle sets, so no atomics.
//
//   k_integrate   : TimeStepController.cpp:112-118 + TimeIntegration::semiImplicitEuler (TimeIntegration.cpp:7-19);
//                   gravity is a uniform (TimeStep::clearAccelerations sets a = g for every dynamic particle, TimeStep.cpp:28-62)
//   k_project<T>  : one (colour,type) bucket of TimeStepController::positionConstraintProjection (TimeStepController.cpp:270-286)
//   k_velocity    : TimeStepController.cpp:155-162 + TimeIntegration::velocityUpdateFirstOrder/SecondOrder (TimeIntegration.cpp:42-51, 69-79)
//   k_step_resident (resident.cuh): the whole step in one launch, positions resident in the shared memory of thread-block clusters
#pragma once
#include "device_image.h"
#include "rest_geometry.cuh"
#include "solvers.cuh"

namespace pbdk {

// Programmatic dependent launch (PDL): every kernel of the step is launched with the programmatic-stream-serialization
// attribute, announces "dependents may launch" immediately and waits for its predecessor only right before it touches
// particle data.  The next bucket's CTAs therefore get scheduled while the current bucket drains, and their coalesced
// streaming loads of indices / rest data (the HBM-latency part) overlap the predecessor's tail.  Without the launch
// attribute both instructions are no-ops.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// wait that is data-dependent on the streamed operands, so that ptxas cannot sink their loads below the wait
// (ptxas hoists an operand-less ACQBULK above independent loads; predicating the wait on the loaded data -- both
// predicate senses wait, so it always executes -- pins it behind them)
__device__ __forceinline__ void pdl_wait_after(unsigned a, float b) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %0, %1;\n\t@p griddepcontrol.wait;\n\t@!p griddepcontrol.wait;\n\t}" :: "r"(a), "r"(__float_as_uint(b)) : "memory");
}

// Particle gather of the per-bucket kernels: through L1, so the 2-4 gathers of one constraint and of neighbouring threads
// that fall into the same 32 B sector / 128 B line are served once.  Safe because L1 is invalidated at every kernel boundary.
__device__ __forceinline__ float4 ldp(const float4 *p) { return *p; }
__device__ __forceinline__ void stp(float4 *p, const float4 &v) { if (v.w != 0.0f) __stcg(p, v); }  // static particles never move

// A replica batch keeps the uniform material parameters of a type in a table row per replica (pbd_set_replica_materials; the shared
// values where a replica has none of its own).  MatRow: that row in registers, loaded once ahead of a kernel's projections like the
// other operands that do not depend on the previous colour; `on` false: the uniforms of the kernel arguments.
struct MatRow { bool on = false; float v[kMaxMat]; };
template <int T>
__device__ __forceinline__ MatRow load_mat_row(const float *row) {
    MatRow r;
    r.on = row != nullptr;
    if (r.on) {
#pragma unroll
        for (int k = 0; k < type_shape(T).nMat; k++) r.v[k] = row[k];
    }
    return r;
}
__device__ __forceinline__ float matv(const TypeArrays &a, int slot, unsigned i, const MatRow &row = MatRow{}) {
    return a.mat[slot] ? __ldg(a.mat[slot] + i) : (row.on ? row.v[slot] : a.matU[slot]);
}
__device__ __forceinline__ float xpbd_alpha(float k, float dt) { return (k != 0.0f) ? frcp(k * dt * dt) : 0.0f; }

// What a constraint streams from HBM before it touches any particle: indices + per-constraint constants.  These never
// change during a step, so they can be fetched ahead of the dependency on the previous colour phase (before the PDL
// wait in k_project, before the colour barrier in k_step_resident).
struct Streamed {
    uint4 b;        // particle indices (x,y[,z[,w]])
    float4 g0, g1;  // float4 geometry (Kp / invRestMat rows / joint connectors)
    float s0, s1;   // scalar geometry (rest length / angle / volume / area / invRestMat(2,2))
};

// the indices, the first nStreamV float4 and all nGeoS scalar geometry arrays of type T (type_shape); the geometry of constraint i at
// i + geoOff (a batch's replica with a rest shape of its own, resident.cuh: an offset costs the register-tight resident kernels less than
// moved array pointers)
template <int T>
__device__ __forceinline__ Streamed load_streamed(const TypeArrays &a, unsigned i, unsigned geoOff = 0u) {
    constexpr TypeShape sh = type_shape(T);
    static_assert(sh.nStreamV <= 2 && sh.nGeoS <= 2, "Streamed holds two float4 and two scalar geometry values");
    Streamed s;
    s.g0 = make_float4(0.f, 0.f, 0.f, 0.f); s.g1 = s.g0; s.s0 = 0.0f; s.s1 = 0.0f;
    if (sh.nBodies == 2) {
        const uint2 b = __ldg(a.idx2 + i);
        s.b = make_uint4(b.x, b.y, 0u, 0u);
    } else if (sh.nBodies == 3) {
        s.b = make_uint4(__ldg(a.idx3[0] + i), __ldg(a.idx3[1] + i), __ldg(a.idx3[2] + i), 0u);
    } else {
        s.b = __ldg(a.idx4 + i);
    }
    if (sh.nStreamV >= 1) s.g0 = __ldg(a.gv[0] + (i + geoOff));
    if (sh.nStreamV >= 2) s.g1 = __ldg(a.gv[1] + (i + geoOff));
    if (sh.nGeoS >= 1) s.s0 = __ldg(a.gs[0] + (i + geoOff));
    if (sh.nGeoS >= 2) s.s1 = __ldg(a.gs[1] + (i + geoOff));
    return s;
}

// Particle accessors: where a constraint's particle index points to.
//   GlobalAcc : the float4 array in global memory (L2-resident), index = device slot
//   ClusterAcc (resident.cuh): bit 31 set -> slot in the shared-memory tile of a CTA of the executing cluster (DSMEM), else global
// handle(idx) resolves the address once; ld / st take the handle (a particle is read and written through the same one)
struct GlobalAcc {
    typedef float4 *Handle;
    float4 *pos;
    __device__ __forceinline__ Handle handle(unsigned idx) const { return pos + idx; }
    __device__ __forceinline__ float4 ld(Handle h) const { return ldp(h); }
    __device__ __forceinline__ void st(Handle h, const float4 &v) const { stp(h, v); }
};

// Gather -> project -> scatter for constraint i (index into the type's arrays) whose streamed part is already here.
// Joints couple rigid bodies (their own small state arrays, L2 only) with each other or with a particle.  rbOff: a batch's replica
// reads its bodies at index + rbOff (resident.cuh, like geoOff)
template <int T, class Acc>
__device__ __forceinline__ void project_joint(const Acc &acc, const TypeArrays &a, const Streamed &s, unsigned rbOff = 0u) {
    const unsigned b0 = s.b.x + rbOff;
    float4 X0 = __ldcg(a.rbX + b0), Q0 = __ldcg(a.rbQ + b0);
    const float4 I0 = __ldg(a.rbIinv + b0);
    if (T == PBD_BALLJOINT) {
        const unsigned b1 = s.b.y + rbOff;
        float4 X1 = __ldcg(a.rbX + b1), Q1 = __ldcg(a.rbQ + b1);
        const float4 I1 = __ldg(a.rbIinv + b1);
        project_balljoint(X0, Q0, mk(I0.x, I0.y, I0.z), X1, Q1, mk(I1.x, I1.y, I1.z), mk(s.g0.x, s.g0.y, s.g0.z), mk(s.g1.x, s.g1.y, s.g1.z));
        if (X1.w != 0.0f) { __stcg(a.rbX + b1, X1); __stcg(a.rbQ + b1, Q1); }
    } else {
        const typename Acc::Handle hp = acc.handle(s.b.y);
        float4 p = acc.ld(hp);
        project_rb_particle_balljoint(X0, Q0, mk(I0.x, I0.y, I0.z), p, mk(s.g0.x, s.g0.y, s.g0.z));
        acc.st(hp, p);
    }
    if (X0.w != 0.0f) { __stcg(a.rbX + b0, X0); __stcg(a.rbQ + b0, Q0); }
}

// VAR: compile-time layout variant of the type (IsometricBending: 0 = rank-1 Kp, 1 = full Q), -1 = read a.variant at run time
// matOff: a batch's replica with per-constraint materials of its own reads them at i + matOff (resident.cuh, like geoOff); rbOff: its
// rigid bodies (project_joint)
template <int T, class Acc, int VAR = -1>
__device__ __forceinline__ void project_streamed_acc(const Acc &acc, const TypeArrays &a, unsigned i, const Streamed &s, float dt,
                                                     bool iterZero, bool lambdaGiven = false, float lambdaValue = 0.0f, const MatRow &matRow = MatRow{},
                                                     unsigned geoOff = 0u, unsigned matOff = 0u, unsigned rbOff = 0u) {
    if (T == PBD_BALLJOINT || T == PBD_RB_PARTICLE_BALLJOINT) { project_joint<T>(acc, a, s, rbOff); return; }
    constexpr bool XPBD = type_shape(T).xpbd;
    constexpr int NB = type_shape(T).nBodies;
    const unsigned mi = i + matOff;
    const typename Acc::Handle h0 = acc.handle(s.b.x), h1 = acc.handle(s.b.y), h2 = acc.handle(NB >= 3 ? s.b.z : s.b.x), h3 = acc.handle(NB >= 4 ? s.b.w : s.b.x);
    float4 p0 = acc.ld(h0), p1 = acc.ld(h1), p2, p3;
    if (NB >= 3) p2 = acc.ld(h2);
    if (NB >= 4) p3 = acc.ld(h3);
    float lam = 0.0f;
    if (XPBD && !iterZero) lam = lambdaGiven ? lambdaValue : __ldcg(a.lambda + i);  // m_lambda; zero at the first sweep of a substep (Constraints.cpp:1241-1242)

    if (T == PBD_DISTANCE) {
        project_distance(p0, p1, s.s0, matv(a, 0, mi, matRow));
    } else if (T == PBD_DISTANCE_XPBD) {
        project_distance_xpbd(p0, p1, s.s0, xpbd_alpha(matv(a, 0, mi, matRow), dt), lam);
    } else if (T == PBD_FEMTRIANGLE) {
        const FemTriMaterial m = femtri_material(matv(a, 0, mi, matRow), matv(a, 1, mi, matRow), matv(a, 2, mi, matRow), matv(a, 3, mi, matRow), matv(a, 4, mi, matRow));
        project_femtriangle(p0, p1, p2, s.s0, s.g0, m);
    } else if (T == PBD_STRAINTRIANGLE) {
        project_straintriangle(p0, p1, p2, s.g0, matv(a, 0, mi, matRow), matv(a, 1, mi, matRow), matv(a, 2, mi, matRow), matv(a, 3, mi, matRow) != 0.0f, matv(a, 4, mi, matRow) != 0.0f);
    } else if (T == PBD_DIHEDRAL) {
        project_dihedral(p0, p1, p2, p3, s.s0, matv(a, 0, mi, matRow));
    } else if (T == PBD_VOLUME) {
        project_volume<false>(p0, p1, p2, p3, s.s0, matv(a, 0, mi, matRow), 0.0f, lam);
    } else if (T == PBD_VOLUME_XPBD) {
        const float k = matv(a, 0, mi, matRow);
        project_volume<true>(p0, p1, p2, p3, s.s0, k, xpbd_alpha(k, dt), lam);
    } else if (T == PBD_ISOBENDING || T == PBD_ISOBENDING_XPBD) {
        constexpr bool X = (T == PBD_ISOBENDING_XPBD);
        const float k = matv(a, 0, mi, matRow);
        const float alpha = X ? xpbd_alpha(k, dt) : 0.0f;
        if (VAR == 0 || (VAR < 0 && a.variant == 0)) project_isobending_rank1<X>(p0, p1, p2, p3, s.g0, k, alpha, lam);
        else project_isobending_fullq<X>(p0, p1, p2, p3, s.g0, __ldg(a.gv[1] + (i + geoOff)), __ldg(a.gv[2] + (i + geoOff)), __ldg(a.gv[3] + (i + geoOff)), k, alpha, lam);
    } else if (T == PBD_FEMTET || T == PBD_FEMTET_XPBD || T == PBD_STRAINTET) {
        M3 inv;
        inv.m[0][0] = s.g0.x; inv.m[0][1] = s.g0.y; inv.m[0][2] = s.g0.z; inv.m[1][0] = s.g0.w;
        inv.m[1][1] = s.g1.x; inv.m[1][2] = s.g1.y; inv.m[2][0] = s.g1.z; inv.m[2][1] = s.g1.w;
        inv.m[2][2] = s.s0;
        if (T == PBD_STRAINTET) project_straintet(p0, p1, p2, p3, inv, matv(a, 0, mi, matRow), matv(a, 1, mi, matRow), matv(a, 2, mi, matRow) != 0.0f, matv(a, 3, mi, matRow) != 0.0f);
        else project_femtet<(T == PBD_FEMTET_XPBD)>(p0, p1, p2, p3, s.s1, inv, matv(a, 0, mi, matRow), matv(a, 1, mi, matRow), dt, lam);
    } else if (T == PBD_SHAPEMATCHING) {
        const unsigned g = i + geoOff;
        project_shapematching(p0, p1, p2, p3, __ldg(a.gv[0] + g), __ldg(a.gv[1] + g), __ldg(a.gv[2] + g), __ldg(a.gv[3] + g), __ldg(a.gv[4] + g),
                              __ldg(a.gv[5] + g), matv(a, 0, mi, matRow));
    }

    if (XPBD) __stcg(a.lambda + i, lam);
    acc.st(h0, p0); acc.st(h1, p1);
    if (NB >= 3) acc.st(h2, p2);
    if (NB >= 4) acc.st(h3, p3);
}

template <int T, int VAR = -1>
__device__ __forceinline__ void project_streamed(float4 *pos, const TypeArrays &a, unsigned i, const Streamed &s, float dt, bool iterZero, const MatRow &matRow) {
    project_streamed_acc<T, GlobalAcc, VAR>(GlobalAcc{pos}, a, i, s, dt, iterZero, false, 0.0f, matRow);
}

// The one list of all constraint types: dispatch a statement on the runtime type, restricted to the types of MASK (T is a
// constant inside the statement; a type outside the mask does nothing).
#define PBD_CASE_TYPE(MASK, TT, ...) case TT: if constexpr ((MASK) & type_bit(TT)) { constexpr int T = TT; __VA_ARGS__ } break;
#define PBD_FOR_TYPE(MASK, type, ...)                                                                                              \
    switch (type) {                                                                                                                \
        PBD_CASE_TYPE(MASK, PBD_DISTANCE, __VA_ARGS__) PBD_CASE_TYPE(MASK, PBD_DISTANCE_XPBD, __VA_ARGS__)                         \
        PBD_CASE_TYPE(MASK, PBD_DIHEDRAL, __VA_ARGS__) PBD_CASE_TYPE(MASK, PBD_ISOBENDING, __VA_ARGS__)                            \
        PBD_CASE_TYPE(MASK, PBD_ISOBENDING_XPBD, __VA_ARGS__) PBD_CASE_TYPE(MASK, PBD_FEMTRIANGLE, __VA_ARGS__)                    \
        PBD_CASE_TYPE(MASK, PBD_STRAINTRIANGLE, __VA_ARGS__) PBD_CASE_TYPE(MASK, PBD_VOLUME, __VA_ARGS__)                          \
        PBD_CASE_TYPE(MASK, PBD_VOLUME_XPBD, __VA_ARGS__) PBD_CASE_TYPE(MASK, PBD_FEMTET, __VA_ARGS__)                             \
        PBD_CASE_TYPE(MASK, PBD_FEMTET_XPBD, __VA_ARGS__) PBD_CASE_TYPE(MASK, PBD_STRAINTET, __VA_ARGS__)                          \
        PBD_CASE_TYPE(MASK, PBD_SHAPEMATCHING, __VA_ARGS__) PBD_CASE_TYPE(MASK, PBD_BALLJOINT, __VA_ARGS__)                        \
        PBD_CASE_TYPE(MASK, PBD_RB_PARTICLE_BALLJOINT, __VA_ARGS__)                                                                \
    default: break;                                                                                                                \
    }

constexpr int kProjectThreads = 256;
constexpr int kMultiSegments = 4;

// A replica batch (pbd_set_replicas) shares one constraint image; the BATCH instantiations of the projection kernels run replica
// blockIdx.y, whose particles start at slot y x nPos and whose multipliers of segment k's type start at y x nLambda[k] (k_project: [0]).
// mat[k]: segment k's type in replica 0's row of the batch's material table (rows of kMatRowFloats floats), or null: no replica has
// material parameters of its own for that type.  nGeo[k]: with per-replica rest shapes (pbd_set_replica_rest_positions) the geometry
// arrays hold every replica's, replica y's at y x nGeo[k]; 0: one geometry shared by all.  nMat[k]: with per-constraint materials of every
// replica (pbd_set_replica_constraint_materials) the material arrays hold every replica's, replica y's at y x nMat[k]; 0: shared.
// nRb: the rigid bodies of a replica (pbd_set_replica_rigid_bodies), replica y's at y x nRb of the joints' body arrays.
struct ReplicaStrides {
    unsigned nPos; unsigned nLambda[kMultiSegments]; const float *mat[kMultiSegments]; unsigned nGeo[kMultiSegments]; unsigned nMat[kMultiSegments];
    unsigned nRb;
    __device__ __forceinline__ const float *mat_row(int k, unsigned rep) const { return mat[k] ? mat[k] + (size_t)rep * kMatRowFloats : nullptr; }
};
// the type's arrays with the multipliers, the geometry, the per-constraint materials and the rigid bodies of replica `rep` (the body arrays
// are set for the joint types only)
__device__ __forceinline__ TypeArrays replica_arrays(const TypeArrays &a, unsigned rep, unsigned nLambda, unsigned nGeo, unsigned nMat = 0u, unsigned nRb = 0u) {
    TypeArrays r = a;
    if (r.lambda) r.lambda += (size_t)rep * nLambda;
    if (nRb && r.rbX) {
        const size_t o = (size_t)rep * nRb;
        r.rbX += o; r.rbQ += o; r.rbIinv += o;
    }
    if (nGeo) {
        const size_t o = (size_t)rep * nGeo;
#pragma unroll
        for (int k = 0; k < kMaxGeoV; k++) if (r.gv[k]) r.gv[k] += o;
#pragma unroll
        for (int k = 0; k < kMaxGeoS; k++) if (r.gs[k]) r.gs[k] += o;
    }
    if (nMat) {
        const size_t o = (size_t)rep * nMat;
#pragma unroll
        for (int k = 0; k < kMaxMat; k++) if (r.mat[k]) r.mat[k] += o;
    }
    return r;
}
template <int T, int VAR, bool BATCH>
__global__ void __launch_bounds__(kProjectThreads) k_project(float4 *pos, TypeArrays a, unsigned first,
                                                             unsigned count, float dt, int iterZero, ReplicaStrides rs) {
    pdl_launch_dependents();
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;  // an exited thread counts as having passed the dependency
    MatRow matRow;
    if (BATCH) { pos += (size_t)blockIdx.y * rs.nPos; a = replica_arrays(a, blockIdx.y, rs.nLambda[0], rs.nGeo[0], rs.nMat[0], rs.nRb); matRow = load_mat_row<T>(rs.mat_row(0, blockIdx.y)); }
    const Streamed s = load_streamed<T>(a, first + i);
    pdl_wait_after(s.b.x ^ s.b.y, s.g0.x + s.g1.x + s.s0 + s.s1);
    project_streamed<T, VAR>(pos, a, first + i, s, dt, iterZero != 0, matRow);
}

// ---- Jacobi comparison path (north_star: "a Jacobi path uses atomicAdd for comparison") -------------------------------------------
// One launch per constraint TYPE and sweep over ALL its constraints, colours ignored: every projection reads the positions of the
// sweep's start and adds its correction to a scratch float4 per particle with one vector atomicAdd (x, y, z, 1); k_jacobi_apply then
// moves every touched particle by the average of its corrections.  A different algorithm from the reference's Gauss-Seidel sweep
// (slower convergence, no ordering), so it is not parity-gated; it exists to price the colouring against atomics.
struct JacobiAcc {
    typedef unsigned Handle;
    const float4 *pos; float4 *delta;
    __device__ __forceinline__ Handle handle(unsigned idx) const { return idx; }
    __device__ __forceinline__ float4 ld(Handle h) const { return __ldg(pos + h); }
    __device__ __forceinline__ void st(Handle h, const float4 &v) const {
        if (v.w == 0.0f) return;
        const float4 o = __ldg(pos + h);
        atomicAdd(delta + h, make_float4(v.x - o.x, v.y - o.y, v.z - o.z, 1.0f));  // RED.E.ADD.F32x4 (sm_90+)
    }
};
template <int T, int VAR>
__global__ void __launch_bounds__(kProjectThreads) k_project_jacobi(const float4 *pos, float4 *delta, TypeArrays a, unsigned count, float dt, int iterZero) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const Streamed s = load_streamed<T>(a, i);
    project_streamed_acc<T, JacobiAcc, VAR>(JacobiAcc{pos, delta}, a, i, s, dt, iterZero != 0);
}
__global__ void __launch_bounds__(256) k_jacobi_apply(float4 *__restrict__ pos, float4 *__restrict__ delta, unsigned n) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 d = delta[i];
    if (d.w == 0.0f) return;
    const float inv = 1.0f / d.w;
    float4 x = pos[i];
    x.x = fmaf(d.x, inv, x.x); x.y = fmaf(d.y, inv, x.y); x.z = fmaf(d.z, inv, x.z);
    pos[i] = x;
    delta[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// Several (colour,type) buckets of ONE colour in a single launch: buckets of a colour touch disjoint particles, so they
// need no ordering among themselves (the reference runs a whole colour group under one `omp parallel for`,
// TimeStepController.cpp:275-285).  A CTA finds its segment from blockIdx and dispatches on the segment's type.
// Used when a colour holds more than one constraint type (e.g. FEMTet + Volume in cfg3: 112 buckets but 74 colours).
struct MultiArgs {
    int nSeg;
    int type[kMultiSegments];
    unsigned first[kMultiSegments], count[kMultiSegments], blockStart[kMultiSegments + 1];
    TypeArrays arrays[kMultiSegments];
};

template <bool BATCH>
__global__ void __launch_bounds__(kProjectThreads) k_project_multi(float4 *pos, const __grid_constant__ MultiArgs m, float dt, int iterZero, ReplicaStrides rs) {
    pdl_launch_dependents();
    int s = 0;
#pragma unroll
    for (int k = 1; k < kMultiSegments; k++)
        if (k < m.nSeg && blockIdx.x >= m.blockStart[k]) s = k;
    const unsigned i = (blockIdx.x - m.blockStart[s]) * blockDim.x + threadIdx.x;
    if (i >= m.count[s]) return;
    const unsigned ci = m.first[s] + i;
    TypeArrays batchArrays;
    if (BATCH) { pos += (size_t)blockIdx.y * rs.nPos; batchArrays = replica_arrays(m.arrays[s], blockIdx.y, rs.nLambda[s], rs.nGeo[s], rs.nMat[s], rs.nRb); }
    const TypeArrays &a = BATCH ? batchArrays : m.arrays[s];
    PBD_FOR_TYPE(kMaskAll, m.type[s],
        MatRow matRow;
        if (BATCH) matRow = load_mat_row<T>(rs.mat_row(s, blockIdx.y));
        const Streamed st = load_streamed<T>(a, ci);
        pdl_wait_after(st.b.x ^ st.b.y, st.g0.x + st.g1.x + st.s0 + st.s1);
        project_streamed<T>(pos, a, ci, st, dt, iterZero != 0, matRow);)
}

// The particle updates of a substep, shared by every execution mode and by the linear part of the rigid bodies, so that the modes
// agree bit for bit.  Arithmetic only: each caller loads and stores with the cache hints of its own memory layout.
// TimeIntegration::semiImplicitEuler (TimeIntegration.cpp:7-19) of a point with mass: v += g h; x += v h
__device__ __forceinline__ void semi_implicit_euler(float4 &x, float4 &v, float h, float gx, float gy, float gz) {
    v.x = fmaf(gx, h, v.x); v.y = fmaf(gy, h, v.y); v.z = fmaf(gz, h, v.z);
    x.x = fmaf(v.x, h, x.x); x.y = fmaf(v.y, h, x.y); x.z = fmaf(v.z, h, x.z);
}
// TimeIntegration::velocityUpdateFirstOrder / SecondOrder (TimeIntegration.cpp:42-51, 69-79): v.xyz = (1/h)(x - oldX)  or
// (1/h)(1.5 x - 2 oldX + 0.5 lastX); lastX() loads lastX, second order only
template <class LastX>
__device__ __forceinline__ void velocity_update(float4 &v, const float4 &x, const float4 &o, float invH, int secondOrder, LastX lastX) {
    if (!secondOrder) {
        v.x = invH * (x.x - o.x); v.y = invH * (x.y - o.y); v.z = invH * (x.z - o.z);
    } else {
        const float4 l = lastX();
        v.x = invH * (1.5f * x.x - 2.0f * o.x + 0.5f * l.x);
        v.y = invH * (1.5f * x.y - 2.0f * o.y + 0.5f * l.y);
        v.z = invH * (1.5f * x.z - 2.0f * o.z + 0.5f * l.z);
    }
}

// The acceleration of a particle with an external force (pbd_set_external_forces): a = g + f w per component, w = the particle's inverse
// mass (x.w) at integration time.  Every mode integrates through this one function, so they agree bit for bit; f = 0 gives exactly g.
__device__ __forceinline__ void external_acceleration(float &gx, float &gy, float &gz, const float4 &f, float w) {
    gx = fmaf(f.x, w, gx); gy = fmaf(f.y, w, gy); gz = fmaf(f.z, w, gz);
}

// lastX = oldX; oldX = x; if (mass != 0) { v += a h; x += v h }, a = g (+ f w with FORCE: `force` at the particle's slot)
// BATCH: the n particles of replica blockIdx.y under that replica's row of `replicaG` (pbd_set_replica_gravity)
template <bool BATCH, bool FORCE>
__device__ __forceinline__ void integrate_slot(float4 *__restrict__ pos, float4 *__restrict__ vel, float4 *__restrict__ oldp,
                                               float4 *__restrict__ lastp, unsigned n, float h, float gx, float gy, float gz,
                                               const float *__restrict__ replicaG, const float4 *__restrict__ force) {
    pdl_launch_dependents();
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (BATCH) {
        i += blockIdx.y * n;
        gx = __ldg(replicaG + 3u * blockIdx.y); gy = __ldg(replicaG + 3u * blockIdx.y + 1u); gz = __ldg(replicaG + 3u * blockIdx.y + 2u);
    }
    pdl_wait();
    float4 x = __ldcg(pos + i);
    __stcs(lastp + i, __ldcs(oldp + i));
    __stcg(oldp + i, x);
    float4 v = __ldcs(vel + i);
    if (v.w != 0.0f) {  // v.w carries the mass (TimeIntegration.cpp:14 tests mass != 0)
        if (FORCE) external_acceleration(gx, gy, gz, __ldcs(force + i), x.w);
        semi_implicit_euler(x, v, h, gx, gy, gz);
        __stcs(vel + i, v);
        __stcg(pos + i, x);
    }
}
template <bool BATCH>
__global__ void __launch_bounds__(256) k_integrate(float4 *__restrict__ pos, float4 *__restrict__ vel,
                                                   float4 *__restrict__ oldp, float4 *__restrict__ lastp, unsigned n,
                                                   float h, float gx, float gy, float gz, const float *__restrict__ replicaG) {
    integrate_slot<BATCH, false>(pos, vel, oldp, lastp, n, h, gx, gy, gz, replicaG, nullptr);
}
// k_integrate with every particle's external force (K x n float4 in slot order, .w unused); launched only while forces are set
template <bool BATCH>
__global__ void __launch_bounds__(256) k_integrate_force(float4 *__restrict__ pos, float4 *__restrict__ vel,
                                                         float4 *__restrict__ oldp, float4 *__restrict__ lastp, unsigned n,
                                                         float h, float gx, float gy, float gz, const float *__restrict__ replicaG,
                                                         const float4 *__restrict__ force) {
    integrate_slot<BATCH, true>(pos, vel, oldp, lastp, n, h, gx, gy, gz, replicaG, force);
}

// Rigid-body prologue / epilogue (a handful of bodies: one thread each).
//   integrate: TimeStepController.cpp:97-107 + TimeIntegration::semiImplicitEuler / semiImplicitEulerRotation (TimeIntegration.cpp:7-39)
//   velocity : TimeStepController.cpp:139-152 + velocityUpdate*/angularVelocityUpdate* (TimeIntegration.cpp:42-95; the angular update is
//              first order in both modes, as in the reference)
struct RbState { float4 *X, *Q, *V, *W, *oldX, *lastX, *oldQ, *lastQ; const float4 *I, *Iinv; unsigned n; };

__device__ __forceinline__ void rb_integrate_body(const RbState &r, unsigned i, float h, float gx, float gy, float gz) {
    float4 X = __ldcg(r.X + i), Q = __ldcg(r.Q + i), V = r.V[i], W = r.W[i];
    r.lastX[i] = r.oldX[i]; r.oldX[i] = X;
    r.lastQ[i] = r.oldQ[i]; r.oldQ[i] = Q;
    if (V.w != 0.0f) {  // V.w = mass
        semi_implicit_euler(X, V, h, gx, gy, gz);
        const M3 R = qmatrix(Q);
        const float4 I = r.I[i], Ii = r.Iinv[i];
        const M3 Iw = world_tensor(R, mk(I.x, I.y, I.z)), Jw = world_tensor(R, mk(Ii.x, Ii.y, Ii.z));
        V3 om = mk(W.x, W.y, W.z);
        const V3 t = -cross(om, mvec(Iw, om));  // torque = 0
        om = om + mvec(Jw, t) * h;
        const float4 dq = qmul(make_float4(om.x, om.y, om.z, 0.0f), Q);
        const float hh = h * 0.5f;
        Q = qnormalize(make_float4(Q.x + hh * dq.x, Q.y + hh * dq.y, Q.z + hh * dq.z, Q.w + hh * dq.w));
        W.x = om.x; W.y = om.y; W.z = om.z;
        __stcg(r.X + i, X); __stcg(r.Q + i, Q); r.V[i] = V; r.W[i] = W;
    }
}
__device__ __forceinline__ void rb_velocity_body(const RbState &r, unsigned i, float invH, float twoInvH, int secondOrder) {
    float4 V = r.V[i];
    if (V.w == 0.0f) return;
    const float4 X = __ldcg(r.X + i), Q = __ldcg(r.Q + i), o = r.oldX[i], oq = r.oldQ[i];
    velocity_update(V, X, o, invH, secondOrder, [&] { return r.lastX[i]; });
    const float4 rel = qmul(Q, make_float4(-oq.x, -oq.y, -oq.z, oq.w));
    float4 W = r.W[i];
    W.x = rel.x * twoInvH; W.y = rel.y * twoInvH; W.z = rel.z * twoInvH;
    r.V[i] = V; r.W[i] = W;
}

__global__ void k_rb_integrate(RbState r, float h, float gx, float gy, float gz) {
    pdl_launch_dependents();
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    pdl_wait();
    rb_integrate_body(r, i, h, gx, gy, gz);
}

__global__ void k_rb_velocity(RbState r, float invH, float twoInvH, int secondOrder) {
    pdl_launch_dependents();
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    pdl_wait();
    rb_velocity_body(r, i, invH, twoInvH, secondOrder);
}

// A replica batch's bodies (pbd_set_replica_rigid_bodies): r.n bodies per replica, replica blockIdx.y's at rows y n .. y n + n - 1; the
// integration under that replica's row of `replicaG` (pbd_set_replica_gravity; null: gx, gy, gz)
__global__ void k_rb_integrate_batch(RbState r, float h, float gx, float gy, float gz, const float *__restrict__ replicaG) {
    pdl_launch_dependents();
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    if (replicaG) { gx = __ldg(replicaG + 3u * blockIdx.y); gy = __ldg(replicaG + 3u * blockIdx.y + 1u); gz = __ldg(replicaG + 3u * blockIdx.y + 2u); }
    pdl_wait();
    rb_integrate_body(r, blockIdx.y * r.n + i, h, gx, gy, gz);
}
__global__ void k_rb_velocity_batch(RbState r, float invH, float twoInvH, int secondOrder) {
    pdl_launch_dependents();
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    pdl_wait();
    rb_velocity_body(r, blockIdx.y * r.n + i, invH, twoInvH, secondOrder);
}

// Rigid-body state <-> the host calls' layouts in device memory (pbd_set_rigid_bodies_device / pbd_get_rigid_bodies_device): rows of
// x(3), q(4, as w x y z), v(3), omega(3), mass(1), inertia(3), replica after replica (r.n bodies per replica; a single scene is replica 0).
// The set writes what pbd_set_rigid_bodies uploads, with the same IEEE divisions: X.w = 1/mass (0 for a static body), V.w = mass, the
// inverse of the principal inertia, oldX = lastX = X, oldQ = lastQ = Q.  mass / inertia null: each body keeps its own; v / omega null: 0.
// mask: as k_pack3 -- replica y is written only where mask[y] != 0, and otherwise its rows are not read.
struct BodyRows { float *x, *q, *v, *omega; const float *mass, *inertia; const unsigned char *mask; };
__global__ void k_set_bodies(RbState r, BodyRows s) {
    if (s.mask && !s.mask[blockIdx.y]) return;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    const size_t b = (size_t)blockIdx.y * r.n + i;
    float4 X = make_float4(s.x[3 * b], s.x[3 * b + 1], s.x[3 * b + 2], 0.0f), V = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s.mass) { const float m = s.mass[b]; X.w = (m != 0.0f) ? __fdiv_rn(1.0f, m) : 0.0f; V.w = m; }
    else { X.w = r.X[b].w; V.w = r.V[b].w; }
    if (s.v) { V.x = s.v[3 * b]; V.y = s.v[3 * b + 1]; V.z = s.v[3 * b + 2]; }
    const float4 Q = make_float4(s.q[4 * b + 1], s.q[4 * b + 2], s.q[4 * b + 3], s.q[4 * b]);
    const float4 W = s.omega ? make_float4(s.omega[3 * b], s.omega[3 * b + 1], s.omega[3 * b + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    r.X[b] = X; r.oldX[b] = X; r.lastX[b] = X;
    r.Q[b] = Q; r.oldQ[b] = Q; r.lastQ[b] = Q;
    r.V[b] = V; r.W[b] = W;
    if (s.inertia) {
        const float ix = s.inertia[3 * b], iy = s.inertia[3 * b + 1], iz = s.inertia[3 * b + 2];
        const_cast<float4 *>(r.I)[b] = make_float4(ix, iy, iz, 0.f);
        const_cast<float4 *>(r.Iinv)[b] = make_float4(__fdiv_rn(1.0f, ix), __fdiv_rn(1.0f, iy), __fdiv_rn(1.0f, iz), 0.f);
    }
}
__global__ void k_get_bodies(RbState r, unsigned rows, BodyRows d) {
    const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= rows) return;
    if (d.x) { const float4 X = r.X[b]; d.x[3 * b] = X.x; d.x[3 * b + 1] = X.y; d.x[3 * b + 2] = X.z; }
    if (d.q) { const float4 Q = r.Q[b]; d.q[4 * b] = Q.w; d.q[4 * b + 1] = Q.x; d.q[4 * b + 2] = Q.y; d.q[4 * b + 3] = Q.z; }
    if (d.v) { const float4 V = r.V[b]; d.v[3 * b] = V.x; d.v[3 * b + 1] = V.y; d.v[3 * b + 2] = V.z; }
    if (d.omega) { const float4 W = r.W[b]; d.omega[3 * b] = W.x; d.omega[3 * b + 1] = W.y; d.omega[3 * b + 2] = W.z; }
}

// v = (1/h)(x - oldX)   or   (1/h)(1.5 x - 2 oldX + 0.5 lastX)
__global__ void __launch_bounds__(256) k_velocity(const float4 *__restrict__ pos, float4 *__restrict__ vel,
                                                  const float4 *__restrict__ oldp, const float4 *__restrict__ lastp,
                                                  unsigned n, float invH, int secondOrder) {
    pdl_launch_dependents();
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pdl_wait();
    const float4 x = __ldcg(pos + i);
    if (x.w == 0.0f) return;  // invMass == 0  <=>  mass == 0 (ParticleData::setMass keeps them consistent)
    const float4 o = __ldcg(oldp + i);
    float4 v;
    velocity_update(v, x, o, invH, secondOrder, [&] { return __ldcs(lastp + i); });
    // keep the mass in .w: re-read only that lane's .w would cost a full sector anyway, so read-modify-write the float4
    v.w = __ldcs(vel + i).w;
    __stcs(vel + i, v);
}

// host AoS-3 <-> device float4 conversion (std::vector<Vector3r> layout on the host side); particle i of the host lives
// in device slot slot[i] (de-interleaved formula of device_image.h, or the tile-major permutation of the tiled mode).  Replica
// blockIdx.y of a batch: host arrays at y x n particles, device arrays at slot y x n + slot[i].  `mask` (k_pack3, k_set_w; nullptr: every
// replica): replica y is written only where mask[y] != 0 -- one load per block, the same for all its threads -- and otherwise its row of
// the source is not read.
__global__ void k_relayout(const float4 *__restrict__ src, float4 *__restrict__ dst, unsigned n, const unsigned *__restrict__ oldSlot,
                           const unsigned *__restrict__ newSlot) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t r = (size_t)blockIdx.y * n;
    if (i < n) dst[r + newSlot[i]] = src[r + oldSlot[i]];
}
__global__ void k_pack3(const float *__restrict__ src, float4 *__restrict__ dst, unsigned n, int keepW, const unsigned *__restrict__ slot,
                        const unsigned char *__restrict__ mask) {
    if (mask && !mask[blockIdx.y]) return;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    src += (size_t)blockIdx.y * 3 * n; dst += (size_t)blockIdx.y * n;
    const unsigned s = slot[i];
    float4 d = keepW ? dst[s] : make_float4(0.f, 0.f, 0.f, 0.f);
    d.x = src[3 * i]; d.y = src[3 * i + 1]; d.z = src[3 * i + 2];
    dst[s] = d;
}
__global__ void k_unpack3(const float4 *__restrict__ src, float *__restrict__ dst, unsigned n, const unsigned *__restrict__ slot) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    src += (size_t)blockIdx.y * n; dst += (size_t)blockIdx.y * 3 * n;
    const float4 s = src[slot[i]];
    dst[3 * i] = s.x; dst[3 * i + 1] = s.y; dst[3 * i + 2] = s.z;
}
// the rest positions of pbd_set_replica_rest_positions: host AoS-3 of K replicas -> K x n float4 BY HOST INDEX, .w = the replica's
// inverse mass now (ShapeMatching freezes it into the constraint)
__global__ void k_pack_rest(const float *__restrict__ src, const float4 *__restrict__ pos, float4 *__restrict__ dst, unsigned n, const unsigned *__restrict__ slot) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    src += (size_t)blockIdx.y * 3 * n; pos += (size_t)blockIdx.y * n; dst += (size_t)blockIdx.y * n;
    dst[i] = make_float4(src[3 * i], src[3 * i + 1], src[3 * i + 2], pos[slot[i]].w);
}

// k_derive_geometry: the rest geometry of a batch's replicas (pbd_set_replica_rest_positions), one thread per (constraint i of type T in
// device order, replica blockIdx.y), with the arithmetic of the host mirror (rest_geometry.cuh).  Replica r's constraint i is packed into
// the image's layout at r x count + i of the K x count long arrays gv / gs -- or, with `rows`, written as the parameter layout's geometry
// columns at row r x count + local[i] (pbd_get_replica_geometry).  A constraint the reference's initConstraint would refuse (and an
// IsometricBending Q that factor_rank1 rejects) lowers *fail to (replica << 32 | insertion id).
struct DeriveArgs {
    const float4 *rest;          // K x n rest positions by host index, .w = inverse mass
    unsigned n, count;
    const unsigned *bodies;      // [count][nBodies] host particle indices, device order
    const unsigned *ids;         // [count] insertion ids
    const unsigned *local;       // [count] position among the type's constraints in the order they were added
    const float4 *clusters;      // ShapeMatching: numClusters of the shared image (its gv[5]), device order
    int variant;                 // IsometricBending: 0 = rank-one Kp in gv[0], 1 = full Q in gv[0..3]
    float4 *gv[kMaxGeoV]; float *gs[kMaxGeoS];
    float *rows;
    unsigned long long *fail;
};
template <int T>
__global__ void __launch_bounds__(128) k_derive_geometry(const __grid_constant__ DeriveArgs d) {
    constexpr TypeShape sh = type_shape(T);
    constexpr int g0 = geo_first(T), nGeo = num_geo(T);
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (i >= d.count) return;
    float4 x[4];
#pragma unroll
    for (int k = 0; k < sh.nBodies; k++) x[k] = __ldg(d.rest + (size_t)r * d.n + __ldg(d.bodies + (size_t)i * sh.nBodies + k));
    float p[24];  // the parameter row; its material columns stay zero and are never read
#pragma unroll
    for (int k = 0; k < 24; k++) p[k] = 0.0f;
    bool ok = rest_geometry(T, x, p + g0);
    if (T == PBD_SHAPEMATCHING) { const float4 c = __ldg(d.clusters + i); p[20] = c.x; p[21] = c.y; p[22] = c.z; p[23] = c.w; }
    float Kp[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (T == PBD_ISOBENDING || T == PBD_ISOBENDING_XPBD) ok = factor_rank1(p + 1, Kp) && ok;
    if (!ok) atomicMin(d.fail, ((unsigned long long)r << 32) | __ldg(d.ids + i));
    if (d.rows) {
        float *row = d.rows + ((size_t)r * d.count + __ldg(d.local + i)) * nGeo;
#pragma unroll
        for (int j = 0; j < nGeo; j++) row[j] = p[g0 + j];
        return;
    }
    const size_t o = (size_t)r * d.count + i;
    if ((T == PBD_ISOBENDING || T == PBD_ISOBENDING_XPBD) && d.variant == 0) { d.gv[0][o] = make_float4(Kp[0], Kp[1], Kp[2], Kp[3]); return; }
    const PackColumns pc = pack_columns(T);
    auto col = [&](int c) { return c < 0 ? 0.0f : p[c]; };
#pragma unroll
    for (int k = 0; k < kMaxGeoV; k++)
        if (d.gv[k]) d.gv[k][o] = make_float4(col(pc.gv[k][0]), col(pc.gv[k][1]), col(pc.gv[k][2]), col(pc.gv[k][3]));
#pragma unroll
    for (int k = 0; k < kMaxGeoS; k++)
        if (d.gs[k]) d.gs[k][o] = col(pc.gs[k]);
}

// k_gather_materials: per-constraint material parameters of a batch (pbd_set_replica_constraint_materials), one thread per (constraint i of
// one type in device order, replica blockIdx.y).  Replica r's row local[i] of `src` (K x count rows of nMat floats, in the order the
// constraints were added) goes to dst[k][r count + i], the device-ordered arrays the projections read; with `keep` the row is also written
// there (the engine's copy in the order they were added).  mask: as k_pack3 -- a replica left out keeps its values, and its rows of src are
// not read.
struct GatherMatArgs {
    const float *src;
    float *keep;
    float *dst[kMaxMat];
    const unsigned *local;       // [count] device position -> position among the type's constraints in the order they were added
    const unsigned char *mask;
    unsigned count;
    int nMat;
};
__global__ void __launch_bounds__(128) k_gather_materials(const __grid_constant__ GatherMatArgs g) {
    if (g.mask && !g.mask[blockIdx.y]) return;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g.count) return;
    const size_t row = ((size_t)blockIdx.y * g.count + __ldg(g.local + i)) * (unsigned)g.nMat, o = (size_t)blockIdx.y * g.count + i;
#pragma unroll
    for (int k = 0; k < kMaxMat; k++)
        if (k < g.nMat) {
            const float v = g.src[row + k];
            g.dst[k][o] = v;
            if (g.keep) g.keep[row + k] = v;
        }
}

__global__ void k_set_w(float4 *__restrict__ pos, float4 *__restrict__ vel, const float *__restrict__ mass, unsigned n, const unsigned *__restrict__ slot,
                        const unsigned char *__restrict__ mask) {
    if (mask && !mask[blockIdx.y]) return;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pos += (size_t)blockIdx.y * n; vel += (size_t)blockIdx.y * n; mass += (size_t)blockIdx.y * n;
    const float m = mass[i];
    const unsigned s = slot[i];
    pos[s].w = (m != 0.0f) ? 1.0f / m : 0.0f;  // ParticleData::setMass (ParticleData.h:239-246)
    vel[s].w = m;
}

}  // namespace pbdk
