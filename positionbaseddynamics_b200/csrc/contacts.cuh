// Contact path (SURVEY.md section 8 row f-4, the part that is data-parallel): particles of triangle / tet models against rigid bodies
// that carry an analytic distance field, then the velocity-level contact solve.
//
// Follows  DistanceFieldCollisionDetection::collisionDetection / collisionDetectionRBSolid
//            (Simulation/DistanceFieldCollisionDetection.cpp:26-197, 290-357),
//          the distance functions and collisionTest / approximateNormal (:598-728),
//          ParticleRigidBodyContactConstraint::initConstraint / solveVelocityConstraint (Simulation/Constraints.cpp:2115-2186),
//          PositionBasedRigidBodyDynamics::init_ / velocitySolve_ParticleRigidBodyContactConstraint
//            (PositionBasedDynamics/PositionBasedRigidBodyDynamics.cpp:2386-2537),
//          TimeStepController::velocityConstraintProjection (Simulation/TimeStepController.cpp:298-357).
//
// Scope: the rigid bodies are static (mass 0: the reference's computeMatrixK is zero, a contact changes its particle's velocity only),
// so the contacts of different particles are independent and the reference's sequential loop over the contact list equals one thread
// per particle that walks ITS contacts in list order inside every velocity iteration.  The reference prunes candidates with a
// bounding-sphere hierarchy; with exact (1-Lipschitz) distance functions the set of points that pass collisionTest is the same as
// testing every point, which is what one thread per particle does.  Dynamic bodies in contact, rigid-rigid and particle-tet contacts
// stay on the reference's CPU time step (the engine and the adapter refuse them).
//
// A replica batch runs the same per-particle body as k_contacts_batch: replica r's particles against replica r's own colliders and
// static bodies, one grid row per replica, each replica computing what k_contacts computes for it alone.
#pragma once
#include <cuda_runtime.h>

namespace pbdk {

enum { kShapeBox = 0, kShapeSphere = 1, kShapeTorus = 2, kShapeCylinder = 3, kShapeHollowSphere = 4, kShapeHollowBox = 5, kNumShapes = 6 };
constexpr int kMaxRigidColliders = 8;

struct RigidCollider {     // one DistanceFieldCollisionObject on a rigid body
    int shape; unsigned body;
    float dim[3];          // box: half extents (m_box); sphere: radius; torus: radii; cylinder: radius, half height (m_dim); hollow: + thickness
    float thickness, invert;  // m_invertSDF (+1 / -1)
    float restitution, friction;
    float R[9], v1[3], v2[3];  // RigidBody::getTransformationR / V1 / V2 (row-major): x_local = R (x_w - com) + v1, x_w = R^T x_local + v2
    float aabbMin[3], aabbMax[3];  // CollisionObject::m_aabb after updateAABB (already extended by the tolerance)
};
struct ParticleCollider {  // one triangle / tet model registered as collision object (DistanceFieldCollisionObjectWithoutGeometry)
    unsigned offset, count;
    float restitution, friction;
};
struct ContactRecord { unsigned particle, body; float cp0[3], cp1[3], n[3], dist; };

struct ContactArgs {
    float4 *pos, *vel;             // pos.w = inverse mass, vel.w = mass
    const unsigned *slot;          // host particle index -> device slot
    const float4 *rbX, *rbV, *rbW; // rigid bodies: centre of mass (w: inverse mass), velocity, angular velocity
    const RigidCollider *rigid; unsigned nRigid;
    const ParticleCollider *ranges; unsigned nRanges;
    const unsigned *rangeStart;    // [nRanges + 1] prefix sums of the counts
    unsigned total;
    float tolerance, stiffness; unsigned maxIterV;
    ContactRecord *record; unsigned *recordCount; unsigned recordCap;
    // replica batch (k_contacts_batch): particles per replica.  Replica r's particles sit at slots r n + slot[i], its colliders at
    // rigid[r nRigid ..] and the bodies carrying them at rbX / rbV / rbW[r nRigid ..], one body per collider
    unsigned n = 0;
};

// ---- distance functions (double precision, as the reference evaluates them) ------------------------------------------------------
__device__ __forceinline__ double sdf_distance(const RigidCollider &c, double x, double y, double z, float tolerance) {
    const double inv = (double)c.invert, tol = (double)tolerance;
    switch (c.shape) {
    case kShapeBox: {
        const double dx = fabs(x) - (double)c.dim[0], dy = fabs(y) - (double)c.dim[1], dz = fabs(z) - (double)c.dim[2];
        const double mx = fmax(dx, 0.0), my = fmax(dy, 0.0), mz = fmax(dz, 0.0);
        return inv * (fmin(fmax(dx, fmax(dy, dz)), 0.0) + sqrt(mx * mx + my * my + mz * mz)) - tol;
    }
    case kShapeSphere: return inv * (sqrt(x * x + y * y + z * z) - (double)c.dim[0]) - tol;
    case kShapeTorus: {
        // The reference takes the ring distance from Vector2r(x, z).norm(), i.e. in Real precision.  In its default build Real is double;
        // in a Real = float build that cast quantises the central differences of approximateNormal (eps = 1e-6 against a float ulp of
        // 6e-8: normals off by percent).  Double here: identical to the default build, and what the float build means to compute.
        const double qx = sqrt(x * x + z * z) - (double)c.dim[0], qy = y;
        return inv * (sqrt(qx * qx + qy * qy) - (double)c.dim[1]) - tol;
    }
    case kShapeCylinder: {
        const double l = sqrt(x * x + z * z);
        const double dx = fabs(l) - (double)c.dim[0], dy = fabs(y) - (double)c.dim[1];
        const double mx = fmax(dx, 0.0), my = fmax(dy, 0.0);
        return inv * (fmin(fmax(dx, dy), 0.0) + sqrt(mx * mx + my * my)) - tol;
    }
    case kShapeHollowSphere: return inv * (fabs(sqrt(x * x + y * y + z * z) - (double)c.dim[0]) - (double)c.thickness) - tol;
    default: {  // kShapeHollowBox
        const double dx = fabs(x) - (double)c.dim[0], dy = fabs(y) - (double)c.dim[1], dz = fabs(z) - (double)c.dim[2];
        const double mx = fmax(dx, 0.0), my = fmax(dy, 0.0), mz = fmax(dz, 0.0);
        return inv * (fabs(fmin(fmax(dx, fmax(dy, dz)), 0.0) + sqrt(mx * mx + my * my + mz * mz)) - (double)c.thickness) - tol;
    }
    }
}

// collisionTest of the object at the local point x: closest point, normal and distance (all local); false = no contact (dist >= 0)
__device__ __forceinline__ bool collision_test(const RigidCollider &c, const float x[3], float tolerance, float cp[3], float n[3], float &dist) {
    if (c.shape == kShapeSphere || c.shape == kShapeHollowSphere) {  // analytic overrides (:614-630, :655-673)
        const float dl = sqrtf(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
        const bool hollow = (c.shape == kShapeHollowSphere);
        dist = hollow ? c.invert * (fabsf(dl - c.dim[0]) - c.thickness) - tolerance : c.invert * (dl - c.dim[0]) - tolerance;
        if (!(dist < 0.0f)) return false;
        float sgn = c.invert;
        if (hollow && dl < c.dim[0]) sgn = -c.invert;
        for (int k = 0; k < 3; k++) n[k] = (dl < 1.e-6f) ? 0.0f : sgn * x[k] / dl;
        for (int k = 0; k < 3; k++) cp[k] = hollow ? x[k] - dist * n[k] : (c.dim[0] + tolerance) * n[k];
        return true;
    }
    dist = (float)sdf_distance(c, (double)x[0], (double)x[1], (double)x[2], tolerance);
    if (!(dist < 0.0f)) return false;
    // approximateNormal: central differences of the distance function, eps = 1e-6, in double precision
    const double eps = 1.e-6;
    double xt[3] = {(double)x[0], (double)x[1], (double)x[2]};
    for (int j = 0; j < 3; j++) {
        const double keep = xt[j];
        xt[j] = keep + eps;
        const double ep = sdf_distance(c, xt[0], xt[1], xt[2], tolerance);
        xt[j] = (double)x[j] - eps;
        const double em = sdf_distance(c, xt[0], xt[1], xt[2], tolerance);
        xt[j] = (double)x[j];
        n[j] = (float)((ep - em) * (1.0 / (2.0 * eps)));
    }
    const float norm2 = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
    if (norm2 < 1.e-6f) n[0] = n[1] = n[2] = 0.0f;
    else { const float s = sqrtf(norm2); n[0] /= s; n[1] /= s; n[2] /= s; }
    for (int k = 0; k < 3; k++) cp[k] = x[k] - dist * n[k];
    return true;
}

struct LiveContact {  // ParticleRigidBodyContactConstraint: m_constraintInfo (3x5), m_sum_impulses, m_frictionCoeff
    float cp0[3], cp1[3], n[3], t[3];
    float nKnInv, pMax, goal, sum, friction;
    unsigned body;  // where the carrying body's state sits in rbX / rbV / rbW
};

// Contact sensors of one particle (contacts_particle<*, true>): per rigid collider k of its replica, whether the collision test found a
// contact, and the sum of the impulses p the solve added to the particle's velocity through that contact, sweep after sweep.
struct ContactSense {
    unsigned count[kMaxRigidColliders];
    float p[kMaxRigidColliders][3];
};

// One thread per particle of the registered triangle / tet models: collision test against every rigid collider in list order (the
// order of the reference's contact list for this particle), contact initialisation with the velocities before any contact impulse,
// then maxIterV sweeps over the particle's contacts.  BATCH: the particle, colliders and bodies of replica `replica` (ContactArgs::n);
// one scene: the body of a collider is its `body`, which indexes rbX / rbV / rbW.
// SENSE: also fills *sense (zeroed by the caller); the arithmetic that moves the particle is the same.
template <bool BATCH, bool SENSE = false>
__device__ __forceinline__ void contacts_particle(const ContactArgs &A, const unsigned gid, const unsigned replica, ContactSense *sense = nullptr) {
    if (gid >= A.total) return;
    unsigned r = 0;
    while (r + 1 < A.nRanges && gid >= A.rangeStart[r + 1]) r++;
    const ParticleCollider pc = A.ranges[r];
    const unsigned particle = pc.offset + (gid - A.rangeStart[r]);
    const unsigned first = BATCH ? replica * A.nRigid : 0u;      // the replica's first collider and body
    const unsigned shift = BATCH ? replica * A.n : 0u;           // the replica's first particle
    const unsigned slot = shift + A.slot[particle];
    const float4 X = A.pos[slot];
    float4 V; bool haveV = false;  // the velocity is fetched for candidates only: most particles leave after the bounding-box tests
    const float invMass0 = X.w;

    LiveContact live[kMaxRigidColliders];
    unsigned char liveCollider[SENSE ? kMaxRigidColliders : 1];  // SENSE: the collider of each live contact
    unsigned nLive = 0;
    for (unsigned k = 0; k < A.nRigid; k++) {
        const RigidCollider &c = A.rigid[first + k];
        const unsigned body = BATCH ? first + k : c.body;
        // candidates outside the collider's (tolerance-extended) bounding box never reach collisionTest in the reference either
        if (X.x < c.aabbMin[0] || X.y < c.aabbMin[1] || X.z < c.aabbMin[2] || X.x > c.aabbMax[0] || X.y > c.aabbMax[1] || X.z > c.aabbMax[2]) continue;
        if (!haveV) { V = A.vel[slot]; haveV = true; }
        const float4 com = A.rbX[body];
        const float d[3] = {X.x - com.x, X.y - com.y, X.z - com.z};
        float xl[3], cp[3], nl[3], dist;
        for (int i = 0; i < 3; i++) xl[i] = c.R[3 * i] * d[0] + c.R[3 * i + 1] * d[1] + c.R[3 * i + 2] * d[2] + c.v1[i];
        if (!collision_test(c, xl, A.tolerance, cp, nl, dist)) continue;
        LiveContact &L = live[nLive];
        for (int i = 0; i < 3; i++) {  // back to world space: R^T
            L.cp1[i] = c.R[i] * cp[0] + c.R[3 + i] * cp[1] + c.R[6 + i] * cp[2] + c.v2[i];
            L.n[i] = c.R[i] * nl[0] + c.R[3 + i] * nl[1] + c.R[6 + i] * nl[2];
        }
        L.cp0[0] = X.x; L.cp0[1] = X.y; L.cp0[2] = X.z;
        L.body = body; L.friction = pc.friction + c.friction; L.sum = 0.0f;
        const float restitution = pc.restitution * c.restitution;
        // init_ParticleRigidBodyContactConstraint (body 1 static: K = invMass0 * I)
        const float4 v1 = A.rbV[body], w1 = A.rbW[body];
        const float r1[3] = {L.cp1[0] - com.x, L.cp1[1] - com.y, L.cp1[2] - com.z};
        const float u1[3] = {v1.x + (w1.y * r1[2] - w1.z * r1[1]), v1.y + (w1.z * r1[0] - w1.x * r1[2]), v1.z + (w1.x * r1[1] - w1.y * r1[0])};
        const float ur[3] = {V.x - u1[0], V.y - u1[1], V.z - u1[2]};
        const float urn = L.n[0] * ur[0] + L.n[1] * ur[1] + L.n[2] * ur[2];
        for (int i = 0; i < 3; i++) L.t[i] = ur[i] - urn * L.n[i];
        const float tl2 = L.t[0] * L.t[0] + L.t[1] * L.t[1] + L.t[2] * L.t[2];
        if (tl2 > 1.0e-6f) { const float s = 1.0f / sqrtf(tl2); L.t[0] *= s; L.t[1] *= s; L.t[2] *= s; }
        const float kd = (invMass0 != 0.0f) ? invMass0 : 0.0f;
        L.nKnInv = 1.0f / (kd * (L.n[0] * L.n[0] + L.n[1] * L.n[1] + L.n[2] * L.n[2]));
        L.pMax = 1.0f / (kd * (L.t[0] * L.t[0] + L.t[1] * L.t[1] + L.t[2] * L.t[2])) * (ur[0] * L.t[0] + ur[1] * L.t[1] + ur[2] * L.t[2]);
        L.goal = (urn < 0.0f) ? -restitution * urn : 0.0f;
        if (A.record) {
            const unsigned at = atomicAdd(A.recordCount, 1u);
            if (at < A.recordCap) {
                ContactRecord rec; rec.particle = shift + particle; rec.body = c.body; rec.dist = dist;
                for (int i = 0; i < 3; i++) { rec.cp0[i] = L.cp0[i]; rec.cp1[i] = L.cp1[i]; rec.n[i] = L.n[i]; }
                A.record[at] = rec;
            }
        }
        if constexpr (SENSE) { liveCollider[nLive] = (unsigned char)k; sense->count[k] = 1u; }
        nLive++;
    }
    if (nLive == 0 || invMass0 == 0.0f) return;  // velocitySolve returns false when both sides are static
    const float mass0 = V.w;

    for (unsigned it = 0; it < A.maxIterV; it++) {
        for (unsigned k = 0; k < nLive; k++) {
            LiveContact &L = live[k];
            const float4 com = A.rbX[L.body], v1 = A.rbV[L.body], w1 = A.rbW[L.body];
            const float d = L.n[0] * (L.cp0[0] - L.cp1[0]) + L.n[1] * (L.cp0[1] - L.cp1[1]) + L.n[2] * (L.cp0[2] - L.cp1[2]);  // penetration depth
            const float r1[3] = {L.cp1[0] - com.x, L.cp1[1] - com.y, L.cp1[2] - com.z};
            const float u1[3] = {v1.x + (w1.y * r1[2] - w1.z * r1[1]), v1.y + (w1.z * r1[0] - w1.x * r1[2]), v1.z + (w1.x * r1[1] - w1.y * r1[0])};
            const float ur[3] = {V.x - u1[0], V.y - u1[1], V.z - u1[2]};
            const float urn = ur[0] * L.n[0] + ur[1] * L.n[1] + ur[2] * L.n[2];
            float mag = L.nKnInv * (L.goal - urn);
            if (mag < -L.sum) mag = -L.sum;
            if (d < 0.0f) mag -= A.stiffness * L.nKnInv * d;  // penalty impulse against the penetration
            float p[3] = {mag * L.n[0], mag * L.n[1], mag * L.n[2]};
            L.sum += mag;
            const float pn = p[0] * L.n[0] + p[1] * L.n[1] + p[2] * L.n[2];
            float ft;
            if (L.friction * pn > L.pMax) ft = -L.pMax;
            else if (L.friction * pn < -L.pMax) ft = L.pMax;
            else ft = -L.friction * pn;
            for (int i = 0; i < 3; i++) p[i] += ft * L.t[i];
            if (mass0 != 0.0f) {
                V.x += invMass0 * p[0]; V.y += invMass0 * p[1]; V.z += invMass0 * p[2];
                if constexpr (SENSE) { float *s = sense->p[liveCollider[k]]; s[0] += p[0]; s[1] += p[1]; s[2] += p[2]; }
            }
        }
    }
    A.vel[slot] = V;
}

__global__ void __launch_bounds__(128) k_contacts(const ContactArgs A) { contacts_particle<false>(A, blockIdx.x * blockDim.x + threadIdx.x, 0u); }
// grid (ceil(total / 128), K): replica = blockIdx.y, so that every collider and body load of a block is uniform
__global__ void __launch_bounds__(128) k_contacts_batch(const ContactArgs A) { contacts_particle<true>(A, blockIdx.x * blockDim.x + threadIdx.x, blockIdx.y); }

#ifdef __CUDACC__
// ---- contact sensors (pbd_sense_contacts) ------------------------------------------------------------------------------------------
// The contact launch with sensing on: the same grid as k_contacts / k_contacts_batch, each thread running contacts_particle<*, true>.  Each
// block then sums its 128 particles' sensors per collider in a fixed order -- within a warp by a shuffle tree (lane i takes lane i + 16,
// + 8, ..., + 1), then the four warp sums in warp order -- into partial[(replica * gridDim.x + block) * nRigid + k]: the impulse sum in
// xyz, the contact count in w (as bits).  k_contact_sensors_sum adds a collider's partials in block order.  The order depends only on
// the particle ranges, so replica r of a batch sums exactly as a single scene given its rows, in every mode.
constexpr unsigned kSenseThreads = 128;
template <bool BATCH>
__device__ __forceinline__ void contacts_sense(const ContactArgs &A, const unsigned replica, float4 *__restrict__ partial) {
    ContactSense s;
    for (int k = 0; k < kMaxRigidColliders; k++) { s.count[k] = 0u; s.p[k][0] = s.p[k][1] = s.p[k][2] = 0.0f; }
    contacts_particle<BATCH, true>(A, blockIdx.x * blockDim.x + threadIdx.x, replica, &s);
    __shared__ float4 warpSum[kSenseThreads / 32][kMaxRigidColliders];
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (unsigned k = 0; k < A.nRigid; k++) {
        float x = s.p[k][0], y = s.p[k][1], z = s.p[k][2];
        unsigned c = s.count[k];
        for (int off = 16; off > 0; off >>= 1) {
            x += __shfl_down_sync(0xffffffffu, x, off); y += __shfl_down_sync(0xffffffffu, y, off); z += __shfl_down_sync(0xffffffffu, z, off);
            c += __shfl_down_sync(0xffffffffu, c, off);
        }
        if (lane == 0) warpSum[warp][k] = make_float4(x, y, z, __uint_as_float(c));
    }
    __syncthreads();
    if (threadIdx.x < A.nRigid) {
        const unsigned k = threadIdx.x;
        float4 t = warpSum[0][k];
        unsigned c = __float_as_uint(t.w);
        for (unsigned w = 1; w < kSenseThreads / 32; w++) {
            const float4 u = warpSum[w][k];
            t.x += u.x; t.y += u.y; t.z += u.z; c += __float_as_uint(u.w);
        }
        t.w = __uint_as_float(c);
        partial[((size_t)replica * gridDim.x + blockIdx.x) * A.nRigid + k] = t;
    }
}
__global__ void __launch_bounds__(kSenseThreads) k_contacts_sense(const ContactArgs A, float4 *partial) { contacts_sense<false>(A, 0u, partial); }
__global__ void __launch_bounds__(kSenseThreads) k_contacts_sense_batch(const ContactArgs A, float4 *partial) { contacts_sense<true>(A, blockIdx.y, partial); }

// one thread per (replica, collider) row of K * nRigid: its `blocks` partials summed in block order; the impulse on the collider is the
// negated sum of what its contacts added to the particles
__global__ void __launch_bounds__(128) k_contact_sensors_sum(const float4 *__restrict__ partial, unsigned rows, unsigned nRigid, unsigned blocks,
                                                             unsigned *__restrict__ count, float *__restrict__ impulse) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const unsigned r = i / nRigid, k = i - r * nRigid;
    const float4 *p = partial + (size_t)r * blocks * nRigid + k;
    float x = 0.0f, y = 0.0f, z = 0.0f;
    unsigned c = 0u;
    for (unsigned b = 0; b < blocks; b++) {
        const float4 u = p[(size_t)b * nRigid];
        x += u.x; y += u.y; z += u.z; c += __float_as_uint(u.w);
    }
    count[i] = c;
    impulse[3 * i] = 0.0f - x; impulse[3 * i + 1] = 0.0f - y; impulse[3 * i + 2] = 0.0f - z;  // (+0 where nothing touched, not -0)
}

// pbd_set_replica_collider_poses_device: one grid row per replica (blockIdx.y), thread k < nRigid writes the placement of collider k and
// the body carrying it.  pose rows: R[9], v1[3], v2[3], aabbMin[3], aabbMax[3]; bodies: w = 0, as the host call writes them.
struct ColliderPoses { const float *pose, *x, *v, *omega; const unsigned char *mask; };
__global__ void k_set_collider_poses(RigidCollider *__restrict__ rigid, float4 *__restrict__ bX, float4 *__restrict__ bV, float4 *__restrict__ bW,
                                     unsigned nRigid, const ColliderPoses s) {
    if (s.mask && !s.mask[blockIdx.y]) return;
    const unsigned k = threadIdx.x;
    if (k >= nRigid) return;
    const size_t i = (size_t)blockIdx.y * nRigid + k;
    const float *p = s.pose + 21 * i;
    RigidCollider &c = rigid[i];
    for (int j = 0; j < 9; j++) c.R[j] = p[j];
    for (int j = 0; j < 3; j++) { c.v1[j] = p[9 + j]; c.v2[j] = p[12 + j]; c.aabbMin[j] = p[15 + j]; c.aabbMax[j] = p[18 + j]; }
    bX[i] = make_float4(s.x[3 * i], s.x[3 * i + 1], s.x[3 * i + 2], 0.f);
    bV[i] = s.v ? make_float4(s.v[3 * i], s.v[3 * i + 1], s.v[3 * i + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    bW[i] = s.omega ? make_float4(s.omega[3 * i], s.omega[3 * i + 1], s.omega[3 * i + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
}
#endif

}  // namespace pbdk
