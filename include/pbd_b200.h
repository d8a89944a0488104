/* include/pbd_b200.h -- C ABI of the H100-native PBD/XPBD constraint-projection engine (libpbd_b200.so).
 *
 * Drop-in seam: this is what a `PBD::TimeStep` subclass on the reference side binds to replace
 * `TimeStepController::step` (Simulation/TimeStepController.cpp:75-241; seam: Simulation/TimeStep.h:13-48,
 * installed via Simulation::setTimeStep, Simulation/Simulation.h:48-49).  The reference-side adapter that
 * flattens a `PBD::SimulationModel` into these calls is integration/GpuTimeStepController.h (compiled inside the
 * unmodified reference by oracle/Makefile and parity-tested; INTEGRATION.md section 1).
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success, non-zero on error
 * (the reference's own convention is bool/void with no exceptions, Simulation/SimulationModel.cpp:565-575);
 * pbd_last_error() returns the message of the last failure on the calling thread.  Nothing throws across
 * this boundary.  One engine <-> one CUDA device + one stream; engines are independent.
 * There is NO CPU fallback: without a CUDA device every entry point that needs one fails.
 */
#ifndef PBD_B200_H
#define PBD_B200_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct pbd_engine pbd_engine;

/* Flat constraint types and their per-constraint parameter layout (floats, in this order).  The layout is the
 * reference's own member set per constraint class (Simulation/Constraints.h:255-457), matrices row-major.
 *  type                     bodies  params                                                   reference class
 *  PBD_DISTANCE             2       restLength, stiffness                                    DistanceConstraint           Constraints.cpp:1166-1206
 *  PBD_DISTANCE_XPBD        2       restLength, stiffness                         (+lambda)  DistanceConstraint_XPBD      Constraints.cpp:1211-1258
 *  PBD_DIHEDRAL             4       restAngle, stiffness                                     DihedralConstraint           Constraints.cpp:1264-1339
 *  PBD_ISOBENDING           4       stiffness, Q[16]                                         IsometricBendingConstraint   Constraints.cpp:1345-1402
 *  PBD_ISOBENDING_XPBD      4       stiffness, Q[16]                              (+lambda)  IsometricBendingConstraint_XPBD :1407-1471
 *  PBD_FEMTRIANGLE          3       area, invRestMat[4], Exx, Eyy, Exy, nu_xy, nu_yx         FEMTriangleConstraint        Constraints.cpp:1476-1538
 *  PBD_STRAINTRIANGLE       3       invRestMat[4], kxx, kyy, kxy, normStretch, normShear     StrainTriangleConstraint     Constraints.cpp:1544-1610
 *  PBD_VOLUME               4       restVolume, stiffness                                    VolumeConstraint             Constraints.cpp:1617-1677
 *  PBD_VOLUME_XPBD          4       restVolume, stiffness                         (+lambda)  VolumeConstraint_XPBD        Constraints.cpp:1683-1750
 *  PBD_FEMTET               4       volume, invRestMat[9], E, nu                             FEMTetConstraint             Constraints.cpp:1755-1825
 *  PBD_FEMTET_XPBD          4       volume, invRestMat[9], E, nu                  (+lambda)  XPBD_FEMTetConstraint        Constraints.cpp:1830-1906
 *  PBD_STRAINTET            4       invRestMat[9], stretchK, shearK, normStretch, normShear  StrainTetConstraint          Constraints.cpp:1912-1980
 *  PBD_SHAPEMATCHING        4       stiffness, restCm[3], x0[4][3], w[4], numClusters[4]     ShapeMatchingConstraint (4-particle clusters) :1985-2028
 *  PBD_BALLJOINT            2 (rigid body, rigid body)      jointInfo[3x4] column by column  BallJoint                    Constraints.cpp:54-125
 *  PBD_RB_PARTICLE_BALLJOINT 2 (rigid body, particle)       jointInfo[3x2] column by column  RigidBodyParticleBallJoint   Constraints.cpp:925-987
 *  Material parameters (what pbd_set_replica_materials replaces per replica; everything else is geometry of the rest state):
 *    Distance(+XPBD), Dihedral, Volume(+XPBD), IsometricBending(+XPBD), ShapeMatching: stiffness;  FEMTriangle: Exx, Eyy, Exy, nu_xy,
 *    nu_yx;  StrainTriangle: kxx, kyy, kxy, normStretch, normShear;  FEMTet(+XPBD): E, nu;  StrainTet: stretchK, shearK, normStretch,
 *    normShear;  the two joint types: none.
 *  (joints: only the local connector columns are read, the global ones are recomputed at every solve as
 *   updateConstraint does; rigid bodies must be uploaded with pbd_set_rigid_bodies before joints are added)
 */
enum pbd_constraint_type {
    PBD_DISTANCE = 0, PBD_DISTANCE_XPBD = 1, PBD_DIHEDRAL = 2, PBD_ISOBENDING = 3, PBD_ISOBENDING_XPBD = 4,
    PBD_FEMTRIANGLE = 5, PBD_STRAINTRIANGLE = 6, PBD_VOLUME = 7, PBD_VOLUME_XPBD = 8, PBD_FEMTET = 9,
    PBD_FEMTET_XPBD = 10, PBD_STRAINTET = 11, PBD_SHAPEMATCHING = 12,
    PBD_BALLJOINT = 13, PBD_RB_PARTICLE_BALLJOINT = 14, PBD_NUM_TYPES = 15
};

/* particle attributes (ParticleData, Simulation/ParticleData.h:91-100); host layout = packed 3 floats per particle,
 * exactly `std::vector<Vector3r>::data()` of the reference's fp32 build. */
enum pbd_attr { PBD_ATTR_X = 0, PBD_ATTR_V = 1, PBD_ATTR_X0 = 2, PBD_ATTR_OLDX = 3, PBD_ATTR_LASTX = 4 };

enum pbd_solver_mode {
    PBD_MODE_GRAPH = 0,      /* one kernel per (colour,type) bucket, whole step replayed as a CUDA graph */
    PBD_MODE_RESIDENT = 1,   /* one launch per step: positions resident in the distributed shared memory of thread-block clusters,
                                hardware cluster barrier between colours (csrc/resident.cuh); scenes up to ~1.5 M particles */
    PBD_MODE_LAUNCH = 2,     /* plain stream launches (debug / per-kernel profiling) */
    PBD_MODE_JACOBI = 3,     /* comparison path, NOT the reference's algorithm: colours ignored, one launch per type and sweep, corrections
                                accumulated with float4 atomicAdd and averaged per particle (rigid-body joints are not supported) */
    PBD_MODE_AUTO = 4        /* default: RESIDENT where it is the faster exact mode (cloth and FEM models of >= 40,000 particles, or batches of >= 32 replicas
                                of them -- 64 for FEMTriangle / Dihedral / Volume models, pbd_set_replicas), else GRAPH, and GRAPH for a model
                                RESIDENT refuses (decided when the model is flattened); both produce the same bits (pbd_get_mode reports the choice) */
};

typedef struct pbd_stats {
    unsigned long long projections;    /* solvePositionConstraint calls executed so far (reference counting: early-outs included) */
    unsigned long long kernel_launches; /* kernels (or graph kernel nodes) launched by pbd_step so far */
    unsigned long long steps;          /* TimeStepController::step equivalents executed */
    unsigned num_particles, num_constraints, num_groups, num_buckets;
    unsigned constraints_per_type[PBD_NUM_TYPES];
    double bytes_per_step;             /* algorithmic bytes of one step (DESIGN.md table) */
    float last_step_ms;                /* device time of the last pbd_step call (CUDA events on the engine stream), after pbd_sync */
    unsigned long long images_planned; /* device images planned so far (a new model, mode, batch size or body arrays plan one) */
    unsigned long long graph_captures; /* step graphs captured so far (PBD_MODE_GRAPH captures again when what the step reads changes) */
} pbd_stats;

const char *pbd_last_error(void);
int pbd_device_count(int *count);

/* stream: a cudaStream_t owned by the caller (e.g. torch.cuda.current_stream().cuda_stream) or NULL to let the
 * engine create its own non-blocking stream. */
int pbd_create(int device, void *stream, pbd_engine **out);
int pbd_destroy(pbd_engine *e);

/* ParticleData upload.  mass: n floats (invMass derived as ParticleData::setMass does, ParticleData.h:239-246).
 * x0/v may be NULL (x0 = x, v = 0); oldX = lastX = x as ParticleData::addVertex does (ParticleData.h:127-137). */
int pbd_set_particles(pbd_engine *e, unsigned n, const float *x, const float *x0, const float *v, const float *mass);
int pbd_set_attr(pbd_engine *e, int attr, const float *src);  /* host -> device, n*3 floats */
int pbd_get_attr(pbd_engine *e, int attr, float *dst);        /* device -> host, n*3 floats; synchronises */
int pbd_set_masses(pbd_engine *e, const float *mass);

/* Rigid bodies taking part in the coloured sweep through BallJoint / RigidBodyParticleBallJoint (SURVEY.md 8f-1;
 * Simulation/RigidBody.h:84-120 initBody with explicit mass and principal inertia).  mass[n], x[3n], q[4n] as (w,x,y,z),
 * inertia[3n] (principal moments), v[3n] / omega[3n] may be NULL (= 0).  old/last state = current, like initBody.
 * pbd_get_rigid_bodies: any output may be NULL. */
int pbd_set_rigid_bodies(pbd_engine *e, unsigned n, const float *mass, const float *x, const float *q, const float *inertia,
                         const float *v, const float *omega);
int pbd_get_rigid_bodies(pbd_engine *e, float *x, float *q, float *v, float *omega);

/* Constraints.  `bodies`: count*numBodies(type) particle indices; `params`: count*numParams(type) floats in the
 * layout above; `ids`: the constraint's index in the reference's SimulationModel::m_constraints (insertion order),
 * or NULL for "append after everything added so far".  Insertion order defines colouring and hence the result. */
int pbd_clear_constraints(pbd_engine *e);
int pbd_add_constraints(pbd_engine *e, int type, unsigned count, const unsigned *bodies, const float *params,
                        const unsigned *ids);
int pbd_num_bodies(int type);
int pbd_num_params(int type);
int pbd_num_materials(int type);  /* how many of the type's parameters are material parameters (table above); 0 for the joints */

/* Colour groups: either import the reference's SimulationModel::m_constraintGroups (offsets[nGroups+1], ids by
 * insertion index) or recompute them with the reference's greedy first-fit (SimulationModel.cpp:1033-1094). */
int pbd_set_groups(pbd_engine *e, unsigned nGroups, const unsigned *offsets, const unsigned *ids);
int pbd_color_first_fit(pbd_engine *e);
/* The same colouring computed on the GPU (exact: wavefronts over the insertion-order dependency DAG, csrc/colouring.cuh);
 * identical groups.  ms / wavefronts (may be NULL): device time of the colouring and number of wavefronts. */
int pbd_color_first_fit_device(pbd_engine *e, float *ms, unsigned *wavefronts);
int pbd_get_num_groups(pbd_engine *e, unsigned *nGroups);
int pbd_get_groups(pbd_engine *e, unsigned *offsets, unsigned *ids);

/* TimeStepController knobs (NUM_SUB_STEPS, MAX_ITERATIONS, VELOCITY_UPDATE_METHOD: TimeStepController.cpp:47-72),
 * TimeManager step size (TimeManager.h:26-27) and Simulation::GRAVITATION (Simulation.cpp:63). */
int pbd_set_params(pbd_engine *e, float dt, unsigned subSteps, unsigned maxIter, int velocityUpdateMethod,
                   const float gravity[3]);
int pbd_set_mode(pbd_engine *e, int mode);
int pbd_get_mode(pbd_engine *e, int *requested, int *active);  /* active = the mode the next step runs in (the image is brought up to date first) */

/* nSteps x TimeStepController::step, asynchronous on the engine's stream. */
int pbd_step(pbd_engine *e, unsigned nSteps);
int pbd_sync(pbd_engine *e);
/* Page-lock caller-owned host arrays (e.g. the reference's std::vector<Vector3r> storage) so that pbd_step_host copies at full
 * PCIe speed straight from / into them; unpin before the memory is freed or reallocated.  Thin wrappers over cudaHostRegister,
 * exported so that a reference-side adapter needs no CUDA headers. */
int pbd_pin_host(void *ptr, size_t bytes);
int pbd_unpin_host(void *ptr);
/* End-to-end convenience used by host-buffer callers (what the TimeStep adapter calls once per step): upload x and v
 * (3 floats/particle each, pinned or pageable; NULL = keep the device state), run nSteps, download x (and v if
 * v_out != NULL), synchronise.  Input and output buffers may be the same arrays. */
int pbd_step_host(pbd_engine *e, unsigned nSteps, const float *x_in, const float *v_in, float *x_out, float *v_out);
/* Pipelined form for callers that stream frames (a renderer reading frame k while frame k+1 is simulated, a batch driver): same
 * arguments and the same per-call copies, but the call only enqueues -- the upload of the next call and the download of the
 * previous one overlap the projection kernels (three streams, two staging slots).  The input arrays must stay untouched and the
 * output arrays unread until pbd_step_host_wait covers the call: lag = 0 waits for every call issued so far, lag = 1 for all but
 * the newest (so a loop "async(k); wait(1);" keeps exactly one call in flight behind the host).  Host arrays should be pinned
 * (pbd_pin_host), otherwise the copies are staged by the driver and do not overlap. */
int pbd_step_host_async(pbd_engine *e, unsigned nSteps, const float *x_in, const float *v_in, float *x_out, float *v_out);
int pbd_step_host_wait(pbd_engine *e, unsigned lag);

/* Particle state in device memory (PyTorch / CuPy buffers).  Same layouts as pbd_set_attr / pbd_get_attr / pbd_set_masses: K*n*3 floats
 * (K*n masses), replica after replica, host particle order -- the slot map and tile permutation stay invisible.  Pointers must be device
 * memory of the engine's device (or managed memory); host memory, pinned included, is refused (use the host calls).
 * stream: the caller's stream (e.g. torch.cuda.current_stream().cuda_stream; the legacy default stream is cudaStreamLegacy) or NULL = the
 * engine's stream.  The copy runs after the work already enqueued on `stream` and on the engine's stream (earlier steps included).  Later
 * work on `stream`, and every later engine call, runs after the copy, so `src` may be freed or reused on `stream` as soon as the call
 * returns.  No call blocks the host.  A stream being captured into a graph is refused.
 * replicas (set calls only): NULL = every replica; else K bytes in device memory.  Replica r is written iff replicas[r] != 0; the other
 * replicas are left bit for bit as they were and their rows of src/mass are not read.  At K = 1 `replicas` has one byte.
 * Refused, with nothing enqueued and the state unchanged: a null pointer, an attribute out of range, host memory, memory of another
 * device, a capturing stream.  K*n = 0 is a no-op.
 * Restarting replicas (episodes that ended, Monte-Carlo restarts): write X, V, OLDX = X and LASTX = X for the chosen replicas (masses too
 * if they change), all with the same `replicas` mask.  Each restarted replica then advances bit for bit as a single-scene engine that
 * pbd_set_particles started from that state; the XPBD multipliers need no reset (they are zeroed at the first sweep of every substep). */
int pbd_set_attr_device(pbd_engine *e, int attr, const float *src, const unsigned char *replicas, void *stream);
int pbd_get_attr_device(pbd_engine *e, int attr, float *dst, void *stream);
int pbd_set_masses_device(pbd_engine *e, const float *mass, const unsigned char *replicas, void *stream);

/* External forces on the particles (wind, drag, a pointer pulling a vertex, an action given as a force).  f: K*n*3 floats (N, world frame)
 * in the layout of pbd_set_attr, replica after replica.  In every substep of every step a particle with mass integrates with the
 * acceleration a = g + f * w, g its replica's gravity (pbd_set_params or pbd_set_replica_gravity), w its inverse mass when it is integrated:
 * a later pbd_set_masses[_device] changes the acceleration, not the force.  A particle with mass 0 ignores its force.  A force stays until
 * it is replaced or cleared, the same in every substep.  Zero forces step to the same bits as no forces.
 * pbd_set_external_forces: from host memory; synchronises.  f = NULL clears every force, and the steps run without the force read again.
 * pbd_set_external_forces_device: from device memory, with the stream contract, mask and refusals of pbd_set_attr_device.  The first set
 * after the forces were cleared zeroes the replicas the mask leaves out.
 * Both write a device table that keeps its address while n and K stand, so a new force between two steps neither plans the image again
 * nor captures the step graph again; setting or clearing forces captures it once.  Adding constraints keeps the forces (they move with
 * the particles); pbd_set_particles and pbd_set_replicas clear them.  bytes_per_step counts 16 more bytes per particle and substep while
 * forces are set. */
int pbd_set_external_forces(pbd_engine *e, const float *f);
int pbd_set_external_forces_device(pbd_engine *e, const float *f, const unsigned char *replicas, void *stream);

/* ---- Contact path (SURVEY.md section 8 row f-4, its data-parallel part) ----------------------------------------------------
 * Particles of triangle / tet models against analytic distance fields carried by STATIC rigid bodies, and the velocity-level
 * contact solve: DistanceFieldCollisionDetection::collisionDetection + collisionDetectionRBSolid
 * (Simulation/DistanceFieldCollisionDetection.cpp:26-197, 290-357; distance functions :598-728), TimeStep::contactCallbackFunction ->
 * SimulationModel::addParticleRigidBodyContactConstraint (Simulation/SimulationModel.cpp:538-549),
 * ParticleRigidBodyContactConstraint (Simulation/Constraints.cpp:2115-2186) and TimeStepController::velocityConstraintProjection
 * (Simulation/TimeStepController.cpp:189-196, 298-357).  Runs once per pbd_step after the substeps, as in the reference.
 * A collider on a rigid body with mass != 0 is refused (its contacts couple through the body and are inherently sequential);
 * rigid-rigid and particle-tet contacts are not covered -- such models stay on the reference's CPU time step.
 *   pbd_particle_collider: one DistanceFieldCollisionObjectWithoutGeometry (particles [offset, offset+count) of a model, the
 *                          model's restitution / friction coefficients).  The ranges of one call must not overlap: a particle
 *                          belongs to at most one range (empty ranges overlap nothing), and both collider calls refuse
 *                          overlapping ranges, with the colliders of the previous call left in force;
 *   pbd_rigid_collider:    one DistanceFieldCollision{Box,Sphere,Torus,Cylinder,HollowSphere,HollowBox} in the order of
 *                          CollisionDetection::getCollisionObjects(): `dim` = m_box (half extents) | m_radius | m_radii | m_dim
 *                          (radius, half height), m_thickness, m_invertSDF, the body's coefficients, RigidBody::getTransformationR
 *                          (row-major) / V1 / V2 and the object's m_aabb (after updateAABB, i.e. extended by the tolerance). */
enum pbd_collider_shape { PBD_SHAPE_BOX = 0, PBD_SHAPE_SPHERE = 1, PBD_SHAPE_TORUS = 2, PBD_SHAPE_CYLINDER = 3, PBD_SHAPE_HOLLOW_SPHERE = 4, PBD_SHAPE_HOLLOW_BOX = 5 };
typedef struct pbd_particle_collider { unsigned offset, count; float restitution, friction; } pbd_particle_collider;
typedef struct pbd_rigid_collider {
    int shape; unsigned body;
    float dim[3], thickness; int invert_sdf;
    float restitution, friction;
    float R[9], v1[3], v2[3];
    float aabb_min[3], aabb_max[3];
} pbd_rigid_collider;
typedef struct pbd_contact { unsigned particle, body; float cp0[3], cp1[3], normal[3], dist; } pbd_contact;
int pbd_set_colliders(pbd_engine *e, unsigned nParticleColliders, const pbd_particle_collider *pc, unsigned nRigidColliders, const pbd_rigid_collider *rc);
/* CollisionDetection::m_tolerance, SimulationModel::m_contactStiffnessParticleRigidBody, TimeStepController::m_maxIterationsV */
int pbd_set_contact_params(pbd_engine *e, float tolerance, float stiffness, unsigned maxIterationsV);
/* debug / rendering: keep the contacts of every step (up to `capacity`); pbd_get_contacts returns those of the last step sorted by
 * (particle, body) and the number found (which may exceed what was kept) */
int pbd_record_contacts(pbd_engine *e, unsigned capacity);
int pbd_get_contacts(pbd_engine *e, pbd_contact *out, unsigned capacity, unsigned *count);
/* Contacts of a replica batch (K > 1).  pc: nParticleColliders particle ranges of ONE replica's particles, shared by every replica
 * (as pbd_set_colliders).  rc: K*nRigidColliders rigid colliders, replica after replica; replica r's list may differ from the
 * others in everything: shape, dims, thickness, invert_sdf, coefficients, R, v1, v2, aabb.  body_x / body_v / body_omega:
 * K*nRigidColliders*3 floats each.  They are the centre of mass, velocity and angular velocity of the static body carrying each
 * collider.  body_v and body_omega may be NULL (= 0).  rc[i].body is only the id reported in pbd_contact.body.
 * Replica r then advances bit for bit as a single-scene engine given
 *   pbd_set_rigid_bodies(nR, masses 0, body_x of replica r, ..., body_v / body_omega of replica r)
 *   and pbd_set_colliders(nP, pc, nR, rc + r*nR) with rc[i].body = i.
 * nRigidColliders = 0 or rc = NULL: no contacts.  A replica that needs fewer colliders gives the others an empty box
 * (aabb_min > aabb_max), which no particle passes.
 * Refused, with the colliders of the previous call left in force: at K = 1, more than 8 rigid colliders per replica, an unknown shape,
 * a particle range beyond n, body_x = NULL with nRigidColliders > 0.  Calling again with the same nParticleColliders and
 * nRigidColliders copies the new rows in stream order into device tables that keep their address, without a host synchronisation: the
 * next step enqueued (pbd_step, pbd_step_host_async, ...) reads them, so obstacles may move per replica between any two steps.  A call
 * that changes either count, or switches the contacts on or off, may synchronise.  pbd_set_replicas drops them; nothing else does.
 * pbd_set_contact_params is shared by all replicas.  pbd_get_contacts reports particle = r*n + i (the index in the K*n state arrays)
 * and body = rc.body, sorted by (particle, body), i.e. replica after replica; the recording capacity is shared by all replicas. */
int pbd_set_replica_colliders(pbd_engine *e, unsigned nParticleColliders, const pbd_particle_collider *pc,
                              unsigned nRigidColliders, const pbd_rigid_collider *rc,
                              const float *body_x, const float *body_v, const float *body_omega);
/* Move the rigid colliders of a replica batch from device memory (K > 1, after pbd_set_replica_colliders switched them on with nR per
 * replica).  pose: K*nR*21 floats; each row is the float fields R[9], v1[3], v2[3], aabb_min[3], aabb_max[3] of a pbd_rigid_collider, in
 * that order (the struct from &rc.R[0] to its end).  body_x: K*nR*3 floats, required; body_v and body_omega: K*nR*3 floats or NULL (= 0).
 * All are the arrays of pbd_set_replica_colliders, replica after replica, colliders in list order.  Only where the obstacles are changes:
 * shape, dims, thickness, invert_sdf, coefficients, body ids, particle ranges and counts stay those of the host call.  The engine then
 * steps bit for bit as if pbd_set_replica_colliders had been called with the same ranges and counts and these placement floats and body
 * rows, so a device set and a host set of the same rows give identical bits.  The rows are written in place (the tables keep their
 * address): no host synchronisation, no new plan, no new graph capture.
 * Stream contract, mask and memory refusals of pbd_set_attr_device: a replica r with replicas[r] == 0 keeps its colliders and bodies bit
 * for bit and its rows are not read.  Refused, with the colliders in force left as they were: at K = 1, without replica colliders in force,
 * a null pose or body_x, host memory (pinned or pageable), memory of another device, a host-memory mask, a stream being captured. */
int pbd_set_replica_collider_poses_device(pbd_engine *e, const float *pose, const float *body_x, const float *body_v,
                                          const float *body_omega, const unsigned char *replicas, void *stream);
/* Contact sensors: per rigid collider of the colliders in force, the contacts found and the impulse received, kept on the device.
 * While sensing is on (pbd_sense_contacts(e, 1); off by default), the contact launch of every step also produces, for each replica r
 * (r = 0 for pbd_set_colliders' single scene) and each rigid collider k:
 *   count[r*nR + k]:         the contacts the collision test of that step found between collider k and replica r's particles -- the
 *                            entries pbd_get_contacts lists for that collider, static particles included;
 *   impulse[3*(r*nR + k)..]: the impulse the particles exerted on collider k during the step's velocity solve, in mass x velocity units
 *                            (divide by dt for the mean force): -sum p over the collider's contacts and the maxIterationsV sweeps, p being
 *                            every impulse (normal, penalty, friction) the solve adds to a particle's velocity (particles of mass 0 get
 *                            none); the -p the reference's velocitySolve_ParticleRigidBodyContactConstraint would apply to a dynamic body.
 * The values are those of the last step enqueued before the get; they are zero when sensing is switched on and when the collider or particle
 * range counts change.  Sums are taken in an order fixed by K, the particle ranges and the collider list (no floating-point atomics), so
 * they are the same bits in every mode and run, and replica r of a batch reports what a single-scene engine given replica r's rows reports.
 * Sensing changes no state; it costs one more launch per step (counted in pbd_stats.kernel_launches) and K*ceil(total/128)*nR*16 bytes of
 * device memory, allocated by this call and by the collider calls, never inside a step.  Switching it plans and captures nothing again;
 * pbd_set_replicas keeps the switch.
 * pbd_get_contact_sensors: host arrays, count K*nR unsigned, impulse K*nR*3 floats, either may be NULL; synchronises.
 * pbd_get_contact_sensors_device: the same into device memory, with the stream contract and memory refusals of pbd_get_attr_device.
 * Both are refused while sensing is off or no rigid colliders are in force. */
int pbd_sense_contacts(pbd_engine *e, int on);
int pbd_get_contact_sensors(pbd_engine *e, unsigned *count, float *impulse);
int pbd_get_contact_sensors_device(pbd_engine *e, unsigned *count, float *impulse, void *stream);

/* ---- Replica batch: K independent copies of one model's state stepped together on one device ---------------------------------
 * One engine holds one model (particles, constraints, groups, parameters) and K copies of its state; one pbd_step advances all K,
 * and replica r advances bit for bit as an engine of its own started from replica r's state would, in every mode.  The constraint
 * image is shared by the replicas and uploaded once.
 *  - Calls that DEFINE the model describe one replica: pbd_set_particles (n, and it sets EVERY replica to the given state),
 *    pbd_add_constraints, the colour groups, pbd_set_params.
 *  - Calls that MOVE state take the whole batch, replica after replica: pbd_set_attr / pbd_get_attr (K*n*3 floats), pbd_set_masses
 *    (K*n: each replica may pin other particles), their device-memory forms (whose set calls may write chosen replicas only),
 *    pbd_step_host / pbd_step_host_async (K*n*3 per array), pbd_get_lambdas (K*count multipliers, `ids` count insertion ids).
 *  - Constraint parameters, gravity and the geometry of the rest state (rest lengths and angles, Q, inverse rest matrices, areas,
 *    volumes, shape-matching rest shapes) are shared unless pbd_set_replica_materials / pbd_set_replica_gravity /
 *    pbd_set_replica_rest_positions (below) give every replica its own.
 *  - Contacts: every replica against its own static colliders through pbd_set_replica_colliders (contact section above); the
 *    colliders of pbd_set_colliders belong to one scene.
 *  - pbd_get_stats: projections and bytes_per_step count every replica; num_particles and num_constraints are per replica.
 *  - Rigid bodies and joints: every replica with its own bodies through pbd_set_replica_rigid_bodies (below); the bodies of
 *    pbd_set_rigid_bodies belong to one scene.
 *  - K > 1 is refused with pbd_set_rigid_bodies' bodies (and joints without per-replica bodies), with pbd_set_colliders' colliders and in
 *    PBD_MODE_JACOBI.  PBD_MODE_RESIDENT runs one cluster of CTAs per replica and refuses a replica that does not fit one cluster;
 *    PBD_MODE_AUTO then runs the graph mode.
 * pbd_set_replicas: 1 <= K <= 65535 and K*n < 2^31.  Every replica starts as a copy of replica 0's current state (x, v, x0, oldX,
 * lastX, masses), the XPBD multipliers at zero, and the image is planned again.  At K = 1 every call behaves as for one scene. */
int pbd_set_replicas(pbd_engine *e, unsigned K);
int pbd_get_replicas(pbd_engine *e, unsigned *K);
/* Per-replica parameters of a batch (K > 1; a single-scene engine takes its parameters from pbd_add_constraints / pbd_set_params and
 * refuses these calls).  Both copy their rows in stream order into device tables that keep their address, so a change between two steps
 * takes effect at the next step.  pbd_set_replicas drops every override (the rows belong to the old K); nothing else does -- adding
 * constraints or changing the mode keeps them.
 * pbd_set_replica_materials: replica r's constraints of `type` all carry the material parameters mat[r*nMat .. r*nMat+nMat), nMat =
 * pbd_num_materials(type), replacing whatever the constraints were added with (a per-constraint material array of that type is ignored
 * while the override is set).  mat = NULL: back to the shared parameters.  Replica r then advances bit for bit as a single-scene engine
 * whose constraints of `type` were added with those values.  Refused for an unknown type and for a type without material parameters.
 * pbd_set_replica_gravity: replica r integrates with gravity g[3r..3r+3) instead of pbd_set_params' vector.  g = NULL: back to it. */
int pbd_set_replica_materials(pbd_engine *e, int type, const float *mat /* K * pbd_num_materials(type) */);
int pbd_set_replica_gravity(pbd_engine *e, const float *g /* K*3 */);
/* Per-constraint material parameters of every replica (K > 1).  mat: K*count*nMat floats, count = the number of constraints of `type`,
 * nMat = pbd_num_materials(type); replica after replica, within a replica the constraints in the order they were added (the order of
 * pbd_get_replica_geometry), each constraint's nMat values in the order of the material columns above.  Replica r then advances bit for bit
 * as a single-scene engine whose constraints of `type` were added with replica r's values.  mat = NULL: back to the shared parameters.
 * One material source per type: the shared parameters, pbd_set_replica_materials' rows, or these per-constraint values -- each set call
 * selects its own, so pbd_set_replica_materials(type, rows or NULL) switches this override off.
 * Lifetime: pbd_set_replicas and pbd_clear_constraints drop it; changing the mode keeps it; pbd_add_constraints keeps it -- the constraints
 * there were keep every replica's values, the new ones carry the parameters they were added with in every replica.  A repeat call copies
 * in stream order into device arrays that keep their address (the next step enqueued reads the new values, a captured step graph stays
 * valid); a call that switches the override on plans the image again and may synchronise.
 * Refused, with nothing changed: at K = 1, an unknown type, the joint types (no material parameters), a type without constraints.
 * pbd_set_replica_constraint_materials_device: the same from device memory, with the stream contract and the refusals of
 * pbd_set_attr_device (mat = NULL included).  replicas: NULL = every replica, else K bytes in device memory; a replica r with
 * replicas[r] == 0 keeps exactly the parameters it was stepped with before the call (shared, rows or per-constraint) and its rows of mat
 * are not read.  No host synchronisation once the override is on.
 * pbd_get_replica_materials: K*count*nMat floats in that layout, the values every replica's constraints of `type` are stepped with,
 * whichever source is in force.  Synchronises. */
int pbd_set_replica_constraint_materials(pbd_engine *e, int type, const float *mat);
int pbd_set_replica_constraint_materials_device(pbd_engine *e, int type, const float *mat, const unsigned char *replicas, void *stream);
int pbd_get_replica_materials(pbd_engine *e, int type, float *dst);
/* Per-replica rest shape of a batch (K > 1, refused at K = 1 like the two calls above).  x0: K*n*3 floats, replica after replica.  Sets
 * PBD_ATTR_X0 of every replica and gives every constraint of replica r the rest geometry that the constraint class's initConstraint derives
 * from replica r's rest positions (ShapeMatching: and from replica r's inverse masses at the time of the call), computed on the GPU with the
 * arithmetic of the host mirror's add*Constraint (double precision, rounded to float; Dihedral's acos may differ from the host's by an ulp).
 * The geometry columns per type: Distance(+XPBD) restLength; Dihedral restAngle; IsometricBending(+XPBD) Q[16]; FEMTriangle area,
 * invRestMat[4]; StrainTriangle invRestMat[4] (rest triangle in the x-z plane, as the reference takes it); Volume(+XPBD) restVolume;
 * FEMTet(+XPBD) volume, invRestMat[9]; StrainTet invRestMat[9]; ShapeMatching restCm[3], x0[12], w[4], numClusters[4] (copied).
 * Refused, with nothing changed, when some replica's rest positions make a constraint degenerate -- where the reference's initConstraint
 * would return false, or an IsometricBending Q has no rank-one factor; the message names the first such replica and the constraint's
 * insertion id.  x0 = NULL: back to the shared geometry (PBD_ATTR_X0 is left as it is).
 * Lifetime: pbd_set_replicas and pbd_set_particles drop the override; adding constraints and changing the mode keep it (the image planned
 * again derives its geometry from the rest positions this call was given; pbd_add_constraints refuses a constraint that some replica's
 * kept rest shape makes degenerate, with the same message); a later pbd_set_attr(PBD_ATTR_X0) re-derives nothing, as
 * editing x0 after initConstraint moves no constraint in the reference.  Calling again with new positions takes effect at the next step. */
int pbd_set_replica_rest_positions(pbd_engine *e, const float *x0);
/* The geometry replica r's constraints of `type` are stepped with: K * count * nGeo floats, nGeo = pbd_num_params(type) -
 * pbd_num_materials(type) (the non-material columns of the type's parameter layout, in layout order), constraints in the order they were
 * added.  Without an override: the shared geometry, repeated for every replica.  Refused for the joint types. */
int pbd_get_replica_geometry(pbd_engine *e, int type, float *dst);
/* Rigid bodies of every replica (K > 1).  mass, x, q, inertia, v, omega: K*n rows each, replica after replica, in the layouts of
 * pbd_set_rigid_bodies (q as (w,x,y,z), principal inertia; v and omega may be NULL = 0).  Defines n bodies per replica: joints added
 * afterwards index 0 .. n-1 and mean "this replica's body i".  Each replica's old and last state equal its current state; each may have its
 * own masses and inertia, and a body may be static in one replica and dynamic in another.  Replica r then advances bit for bit as a
 * single-scene engine given replica r's rows through pbd_set_rigid_bodies and the same constraints and groups; per-replica gravity
 * (pbd_set_replica_gravity) moves replica r's bodies too.  pbd_get_rigid_bodies returns K*n rows.
 * A repeat call with the same n copies in stream order into device arrays that keep their address: no host synchronisation, no new plan
 * or graph capture.  A different n may synchronise and recolours (as pbd_set_rigid_bodies).  pbd_set_replicas(K') starts every replica
 * from replica 0's bodies (state, history, masses, inertia) and keeps them per-replica bodies; pbd_set_rigid_bodies makes them one
 * scene's again.  Contacts stay with static colliders (pbd_set_replica_colliders, whose bodies are its own).
 * Refused, with nothing changed: at K = 1, a null mass / x / q / inertia with n > 0, K*n >= 2^31, PBD_MODE_JACOBI. */
int pbd_set_replica_rigid_bodies(pbd_engine *e, unsigned n, const float *mass, const float *x, const float *q, const float *inertia,
                                 const float *v, const float *omega);
/* Rigid-body state in device memory, at any K where the engine holds bodies: the layouts above (K*n rows), the stream contract, mask
 * semantics and refusals of pbd_set_attr_device.  The set writes x and q (required), v and omega (NULL = 0), and mass / inertia (NULL = each
 * body keeps its own), converted on the device with the host call's IEEE divisions, so a device set and a host set of the same rows give
 * identical bits; every written replica's old and last state equal its new current state.  A replica outside `replicas` stays bit for bit
 * as it was and its rows are not read.  The contact path reads written masses back before it next checks that colliders of
 * pbd_set_colliders sit on static bodies.  The get writes any of x, q, v, omega that is not NULL. */
int pbd_set_rigid_bodies_device(pbd_engine *e, const float *mass, const float *x, const float *q, const float *inertia, const float *v,
                                const float *omega, const unsigned char *replicas, void *stream);
int pbd_get_rigid_bodies_device(pbd_engine *e, float *x, float *q, float *v, float *omega, void *stream);

int pbd_get_lambdas(pbd_engine *e, int type, float *dst, unsigned *ids); /* debug: per-type XPBD multipliers + insertion ids */
int pbd_get_stats(pbd_engine *e, pbd_stats *out);
/* per-type device time of one profiled step (plain launches bracketed by CUDA events; ms per type + prologue/epilogue) */
int pbd_profile_step(pbd_engine *e, float *ms_per_type /*PBD_NUM_TYPES*/, float *ms_integrate, float *ms_velocity,
                     unsigned *launches_per_type /*PBD_NUM_TYPES*/);

#ifdef __cplusplus
}
#endif
#endif
