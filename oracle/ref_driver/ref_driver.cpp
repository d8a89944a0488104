// oracle/ref_driver/ref_driver.cpp -- TEST INFRASTRUCTURE, not product code.
//
// Thin extern "C" wrapper that links against the UNMODIFIED reference sources compiled from
// /root/reference (see oracle/Makefile) so that tests and golden-vector generation can drive the
// reference's own SimulationModel / TimeStepController / solve_* functions headless.
// Built twice: libpbdref_f32.so (Real=float, parity oracle) and libpbdref_f64.so (-DUSE_DOUBLE,
// the reference's default precision).  All floating-point arguments cross this ABI as double so
// that one ctypes binding serves both builds (float->double is exact).
//
// Nothing here is copied from the reference; it only calls its public API
// (Simulation/SimulationModel.h:134-327, Simulation/TimeStepController.h, Simulation/Simulation.h:41-49).
#include "Simulation/Simulation.h"
#include "Simulation/SimulationModel.h"
#include "Simulation/TimeManager.h"
#include "Simulation/TimeStepController.h"
#include "Simulation/Constraints.h"
#include "Simulation/RigidBody.h"
#include "Simulation/DistanceFieldCollisionDetection.h"
#include "Utils/IndexedFaceMesh.h"
#include "PositionBasedDynamics/PositionBasedDynamics.h"
#include "PositionBasedDynamics/XPBD.h"
#include "PositionBasedDynamics/MathFunctions.h"
#include "PositionBasedDynamics/TimeIntegration.h"
#include "Utils/Logger.h"
#include "Utils/Timing.h"
#include <chrono>
#include <cstring>
#ifdef _OPENMP
#include <omp.h>
#endif

#ifdef PBD_WITH_GPU_ADAPTER
// the reference-side binding of libpbd_b200.so, compiled inside this reference build so that the parity tests can step a model
// the reference built and coloured through the GPU engine (integration/GpuTimeStepController.h)
#define PBD_GPU_TIMESTEP_IMPLEMENTATION
#include "GpuTimeStepController.h"
#endif

INIT_LOGGING
INIT_TIMING

using namespace PBD;

// shared flat-constraint type codes (same numbering as include/pbd_b200.h and oracle/pbd_oracle.h)
enum { T_DISTANCE = 0, T_DISTANCE_XPBD, T_DIHEDRAL, T_ISOBENDING, T_ISOBENDING_XPBD, T_FEMTRIANGLE,
       T_STRAINTRIANGLE, T_VOLUME, T_VOLUME_XPBD, T_FEMTET, T_FEMTET_XPBD, T_STRAINTET, T_SHAPEMATCHING,
       T_BALLJOINT, T_RB_PARTICLE_BALLJOINT, T_UNKNOWN = -1 };

static SimulationModel *g_model = nullptr;
static DistanceFieldCollisionDetection *g_cd = nullptr;  // the reference's collision detection, attached to whichever time step is installed
#ifdef PBD_WITH_GPU_ADAPTER
static GpuTimeStepController *g_gpuTs = nullptr;  // owned by Simulation once installed
static std::string g_gpuErr;
#endif

static Vector3r v3(const double *p) { return Vector3r((Real)p[0], (Real)p[1], (Real)p[2]); }
static Matrix3r m3(const double *p) {  // row-major in
    Matrix3r m;
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) m(r, c) = (Real)p[3 * r + c];
    return m;
}

extern "C" {

int ref_real_size() { return (int)sizeof(Real); }

void ref_set_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#endif
}
int ref_max_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

// fresh Simulation + SimulationModel (Demos/ClothDemo/main.cpp:46-73 does the same dance)
void ref_reset() {
    if (Simulation::hasCurrent()) {
        Simulation *s = Simulation::getCurrent();
        if (g_model) { g_model->cleanup(); delete g_model; g_model = nullptr; }
        delete s;  // deletes TimeStep and TimeManager (Simulation.cpp:22-28)
        TimeManager::setCurrent(nullptr);
        delete g_cd; g_cd = nullptr;
#ifdef PBD_WITH_GPU_ADAPTER
        g_gpuTs = nullptr;
#endif
    }
    g_model = new SimulationModel();
    g_model->init();
    Simulation::getCurrent()->setModel(g_model);
    TimeManager::getCurrent()->setTimeStepSize((Real)0.005);
}

void ref_add_regular_triangle_model(int w, int h, const double *t, const double *R, const double *scale) {
    g_model->addRegularTriangleModel(w, h, v3(t), m3(R), Vector2r((Real)scale[0], (Real)scale[1]));
}
void ref_add_regular_tet_model(int w, int h, int d, const double *t, const double *R, const double *scale) {
    g_model->addRegularTetModel(w, h, d, v3(t), m3(R), v3(scale));
}
void ref_add_triangle_model(unsigned nPoints, unsigned nFaces, const double *pts, const unsigned *idx) {
    std::vector<Vector3r> p(nPoints);
    for (unsigned i = 0; i < nPoints; i++) p[i] = v3(pts + 3 * i);
    std::vector<unsigned> ind(idx, idx + 3 * nFaces);
    TriangleModel::ParticleMesh::UVIndices uvi; TriangleModel::ParticleMesh::UVs uvs;
    g_model->addTriangleModel(nPoints, nFaces, p.data(), ind.data(), uvi, uvs);
}
void ref_add_tet_model(unsigned nPoints, unsigned nTets, const double *pts, const unsigned *idx) {
    std::vector<Vector3r> p(nPoints);
    for (unsigned i = 0; i < nPoints; i++) p[i] = v3(pts + 3 * i);
    std::vector<unsigned> ind(idx, idx + 4 * nTets);
    g_model->addTetModel(nPoints, nTets, p.data(), ind.data());
}
void ref_set_mass(unsigned i, double m) { g_model->getParticles().setMass(i, (Real)m); }

// RigidBody::initBody(mass, x, inertiaTensor, rotation, vertices, mesh) (Simulation/RigidBody.h:84-120); q = (w,x,y,z).
// The geometry is irrelevant on this path; a one-triangle mesh satisfies the signature.
unsigned ref_add_rigid_body(double mass, const double *x, const double *inertia, const double *q) {
    VertexData vd;
    vd.addVertex(Vector3r(0, 0, 0)); vd.addVertex(Vector3r(1, 0, 0)); vd.addVertex(Vector3r(0, 1, 0));
    Utilities::IndexedFaceMesh mesh;
    mesh.initMesh(3, 3, 1);
    const unsigned tri[3] = {0, 1, 2};
    mesh.addFace(tri);
    mesh.buildNeighbors();
    RigidBody *rb = new RigidBody();
    rb->initBody((Real)mass, v3(x), v3(inertia), Quaternionr((Real)q[0], (Real)q[1], (Real)q[2], (Real)q[3]), vd, mesh);
    g_model->getRigidBodies().push_back(rb);
    g_model->m_groupsInitialized = false;
    return (unsigned)g_model->getRigidBodies().size() - 1;
}
// RigidBody::initBody(density, x, rotation, vertices, mesh, scale) (Simulation/RigidBody.h:122-150): mass properties from the
// mesh (Utils/VolumeIntegration.cpp), body frame moved to the centre of mass and the principal axes.  R row-major.
unsigned ref_add_rigid_body_mesh(double density, unsigned nV, const double *verts, unsigned nF, const unsigned *faces,
                                 const double *x, const double *R, const double *scale) {
    VertexData vd;
    for (unsigned i = 0; i < nV; i++) vd.addVertex(v3(verts + 3 * i));
    Utilities::IndexedFaceMesh mesh;
    mesh.initMesh(nV, nF * 2, nF);
    for (unsigned i = 0; i < nF; i++) mesh.addFace(faces + 3 * i);
    mesh.buildNeighbors();
    RigidBody *rb = new RigidBody();
    rb->initBody((Real)density, v3(x), Quaternionr(m3(R)), vd, mesh, v3(scale));
    g_model->getRigidBodies().push_back(rb);
    g_model->m_groupsInitialized = false;
    return (unsigned)g_model->getRigidBodies().size() - 1;
}
// mass, principal inertia (3), position (3), rotation (w, x, y, z)
void ref_get_rigid_body_props(unsigned i, double *out) {
    RigidBody *rb = g_model->getRigidBodies()[i];
    out[0] = rb->getMass();
    for (int k = 0; k < 3; k++) { out[1 + k] = rb->getInertiaTensor()[k]; out[4 + k] = rb->getPosition()[k]; }
    const Quaternionr &q = rb->getRotation();
    out[7] = q.w(); out[8] = q.x(); out[9] = q.y(); out[10] = q.z();
}
void ref_set_rigid_body_velocity(unsigned i, const double *v, const double *omega) {
    RigidBody *rb = g_model->getRigidBodies()[i];
    rb->setVelocity(v3(v));
    rb->setAngularVelocity(v3(omega));
}
unsigned ref_num_rigid_bodies() { return (unsigned)g_model->getRigidBodies().size(); }
void ref_get_rigid_bodies(double *out) {
    auto &rbs = g_model->getRigidBodies();
    for (size_t i = 0; i < rbs.size(); i++) {
        double *o = out + 13 * i;
        const RigidBody &b = *rbs[i];
        for (int k = 0; k < 3; k++) { o[k] = b.getPosition()[k]; o[7 + k] = b.getVelocity()[k]; o[10 + k] = b.getAngularVelocity()[k]; }
        o[3] = b.getRotation().w(); o[4] = b.getRotation().x(); o[5] = b.getRotation().y(); o[6] = b.getRotation().z();
    }
}

void ref_add_cloth_constraints(unsigned triModel, unsigned method, double distK, double xx, double yy, double xy,
                               double pxy, double pyx, int normStretch, int normShear) {
    g_model->addClothConstraints(g_model->getTriangleModels()[triModel], method, (Real)distK, (Real)xx, (Real)yy,
                                 (Real)xy, (Real)pxy, (Real)pyx, normStretch != 0, normShear != 0);
}
void ref_add_bending_constraints(unsigned triModel, unsigned method, double k) {
    g_model->addBendingConstraints(g_model->getTriangleModels()[triModel], method, (Real)k);
}
void ref_add_solid_constraints(unsigned tetModel, unsigned method, double k, double nu, double volK, int normStretch,
                               int normShear) {
    g_model->addSolidConstraints(g_model->getTetModels()[tetModel], method, (Real)k, (Real)nu, (Real)volK,
                                 normStretch != 0, normShear != 0);
}
// single-constraint adders; params follow the flat layout documented in oracle/pbd_oracle.h
int ref_add_constraint(int type, const unsigned *b, const double *p) {
    SimulationModel &m = *g_model;
    switch (type) {
    case T_DISTANCE: return m.addDistanceConstraint(b[0], b[1], (Real)p[0]);
    case T_DISTANCE_XPBD: return m.addDistanceConstraint_XPBD(b[0], b[1], (Real)p[0]);
    case T_DIHEDRAL: return m.addDihedralConstraint(b[0], b[1], b[2], b[3], (Real)p[0]);
    case T_ISOBENDING: return m.addIsometricBendingConstraint(b[0], b[1], b[2], b[3], (Real)p[0]);
    case T_ISOBENDING_XPBD: return m.addIsometricBendingConstraint_XPBD(b[0], b[1], b[2], b[3], (Real)p[0]);
    case T_FEMTRIANGLE: return m.addFEMTriangleConstraint(b[0], b[1], b[2], (Real)p[0], (Real)p[1], (Real)p[2], (Real)p[3], (Real)p[4]);
    case T_STRAINTRIANGLE: return m.addStrainTriangleConstraint(b[0], b[1], b[2], (Real)p[0], (Real)p[1], (Real)p[2], p[3] != 0, p[4] != 0);
    case T_VOLUME: return m.addVolumeConstraint(b[0], b[1], b[2], b[3], (Real)p[0]);
    case T_VOLUME_XPBD: return m.addVolumeConstraint_XPBD(b[0], b[1], b[2], b[3], (Real)p[0]);
    case T_FEMTET: return m.addFEMTetConstraint(b[0], b[1], b[2], b[3], (Real)p[0], (Real)p[1]);
    case T_FEMTET_XPBD: return m.addFEMTetConstraint_XPBD(b[0], b[1], b[2], b[3], (Real)p[0], (Real)p[1]);
    case T_STRAINTET: return m.addStrainTetConstraint(b[0], b[1], b[2], b[3], (Real)p[0], (Real)p[1], p[2] != 0, p[3] != 0);
    case T_BALLJOINT: return m.addBallJoint(b[0], b[1], v3(p));
    case T_RB_PARTICLE_BALLJOINT: return m.addRigidBodyParticleBallJoint(b[0], b[1]);
    case T_SHAPEMATCHING: { const unsigned nc[4] = {(unsigned)p[1], (unsigned)p[2], (unsigned)p[3], (unsigned)p[4]}; return m.addShapeMatchingConstraint(4, b, nc, (Real)p[0]); }
    default: return -1;
    }
}

void ref_set_params(double dt, unsigned subSteps, unsigned maxIter, int velMethod, const double *g) {
    TimeManager::getCurrent()->setTimeStepSize((Real)dt);
#ifdef PBD_WITH_GPU_ADAPTER
    if (g_gpuTs) {
        g_gpuTs->setValue<unsigned int>(GpuTimeStepController::NUM_SUB_STEPS, subSteps);
        g_gpuTs->setValue<unsigned int>(GpuTimeStepController::MAX_ITERATIONS, maxIter);
        g_gpuTs->setValue<int>(GpuTimeStepController::VELOCITY_UPDATE_METHOD, velMethod);
    } else
#endif
    {
    TimeStepController *ts = static_cast<TimeStepController *>(Simulation::getCurrent()->getTimeStep());
    ts->setValue<unsigned int>(TimeStepController::NUM_SUB_STEPS, subSteps);
    ts->setValue<unsigned int>(TimeStepController::MAX_ITERATIONS, maxIter);
    ts->setValue<int>(TimeStepController::VELOCITY_UPDATE_METHOD, velMethod);
    }
    Real gg[3] = {(Real)g[0], (Real)g[1], (Real)g[2]};
    Simulation::getCurrent()->setVecValue<Real>(Simulation::GRAVITATION, gg);
}

void ref_init_groups() { g_model->initConstraintGroups(); }
unsigned ref_num_particles() { return g_model->getParticles().size(); }
unsigned ref_num_constraints() { return (unsigned)g_model->getConstraints().size(); }
unsigned ref_num_groups() { return (unsigned)g_model->getConstraintGroups().size(); }
// offsets has nGroups+1 entries, ids has nConstraints entries
void ref_get_groups(unsigned *offsets, unsigned *ids) {
    auto &g = g_model->getConstraintGroups();
    unsigned o = 0;
    for (size_t i = 0; i < g.size(); i++) {
        offsets[i] = o;
        for (unsigned id : g[i]) ids[o++] = id;
    }
    offsets[g.size()] = o;
}

// which: 0 x, 1 v, 2 x0, 3 oldX, 4 lastX, 5 a
static Vector3r &attr(ParticleData &pd, int which, unsigned i) {
    switch (which) {
    case 0: return pd.getPosition(i);
    case 1: return pd.getVelocity(i);
    case 2: return pd.getPosition0(i);
    case 3: return pd.getOldPosition(i);
    case 4: return pd.getLastPosition(i);
    default: return pd.getAcceleration(i);
    }
}
void ref_get_attr(int which, double *out) {
    ParticleData &pd = g_model->getParticles();
    for (unsigned i = 0; i < pd.size(); i++) { const Vector3r &v = attr(pd, which, i); out[3*i] = v[0]; out[3*i+1] = v[1]; out[3*i+2] = v[2]; }
}
void ref_set_attr(int which, const double *in) {
    ParticleData &pd = g_model->getParticles();
    for (unsigned i = 0; i < pd.size(); i++) attr(pd, which, i) = v3(in + 3 * i);
}
void ref_get_masses(double *mass, double *invMass) {
    ParticleData &pd = g_model->getParticles();
    for (unsigned i = 0; i < pd.size(); i++) { mass[i] = pd.getMass(i); invMass[i] = pd.getInvMass(i); }
}

unsigned ref_tri_num_edges(unsigned tm) { return g_model->getTriangleModels()[tm]->getParticleMesh().numEdges(); }
unsigned ref_tri_num_faces(unsigned tm) { return g_model->getTriangleModels()[tm]->getParticleMesh().numFaces(); }
unsigned ref_tri_index_offset(unsigned tm) { return g_model->getTriangleModels()[tm]->getIndexOffset(); }
// per edge: v0 v1 f0 f1
void ref_tri_get_edges(unsigned tm, unsigned *out) {
    auto &e = g_model->getTriangleModels()[tm]->getParticleMesh().getEdges();
    for (size_t i = 0; i < e.size(); i++) { out[4*i] = e[i].m_vert[0]; out[4*i+1] = e[i].m_vert[1]; out[4*i+2] = e[i].m_face[0]; out[4*i+3] = e[i].m_face[1]; }
}
void ref_tri_get_faces(unsigned tm, unsigned *out) {
    auto &f = g_model->getTriangleModels()[tm]->getParticleMesh().getFaces();
    memcpy(out, f.data(), f.size() * sizeof(unsigned));
}
unsigned ref_tet_num_edges(unsigned tm) { return g_model->getTetModels()[tm]->getParticleMesh().numEdges(); }
unsigned ref_tet_num_tets(unsigned tm) { return g_model->getTetModels()[tm]->getParticleMesh().numTets(); }
unsigned ref_tet_index_offset(unsigned tm) { return g_model->getTetModels()[tm]->getIndexOffset(); }
void ref_tet_get_edges(unsigned tm, unsigned *out) {
    auto &e = g_model->getTetModels()[tm]->getParticleMesh().getEdges();
    for (size_t i = 0; i < e.size(); i++) { out[2*i] = e[i].m_vert[0]; out[2*i+1] = e[i].m_vert[1]; }
}
void ref_tet_get_tets(unsigned tm, unsigned *out) {
    auto &t = g_model->getTetModels()[tm]->getParticleMesh().getTets();
    memcpy(out, t.data(), t.size() * sizeof(unsigned));
}

static int typeCode(Constraint *c) {
    const int id = c->getTypeId();
    if (id == DistanceConstraint::TYPE_ID) return T_DISTANCE;
    if (id == DistanceConstraint_XPBD::TYPE_ID) return T_DISTANCE_XPBD;
    if (id == DihedralConstraint::TYPE_ID) return T_DIHEDRAL;
    if (id == IsometricBendingConstraint::TYPE_ID) return T_ISOBENDING;
    if (id == IsometricBendingConstraint_XPBD::TYPE_ID) return T_ISOBENDING_XPBD;
    if (id == FEMTriangleConstraint::TYPE_ID) return T_FEMTRIANGLE;
    if (id == StrainTriangleConstraint::TYPE_ID) return T_STRAINTRIANGLE;
    if (id == VolumeConstraint::TYPE_ID) return T_VOLUME;
    if (id == VolumeConstraint_XPBD::TYPE_ID) return T_VOLUME_XPBD;
    if (id == FEMTetConstraint::TYPE_ID) return T_FEMTET;
    if (id == XPBD_FEMTetConstraint::TYPE_ID) return T_FEMTET_XPBD;
    if (id == StrainTetConstraint::TYPE_ID) return T_STRAINTET;
    if (id == ShapeMatchingConstraint::TYPE_ID) return T_SHAPEMATCHING;
    if (id == BallJoint::TYPE_ID) return T_BALLJOINT;
    if (id == RigidBodyParticleBallJoint::TYPE_ID) return T_RB_PARTICLE_BALLJOINT;
    return T_UNKNOWN;
}

// Flat export of constraint i: returns type code; bodies[<=4]; params[<=24] (layout: oracle/pbd_oracle.h)
int ref_get_constraint(unsigned i, unsigned *bodies, double *p, double *lambda) {
    Constraint *c = g_model->getConstraints()[i];
    const int t = typeCode(c);
    for (unsigned k = 0; k < c->numberOfBodies() && k < 4; k++) bodies[k] = c->m_bodies[k];
    *lambda = 0.0;
    int n = 0;
    auto putM = [&](const auto &M, int rows, int cols) { for (int r = 0; r < rows; r++) for (int cc = 0; cc < cols; cc++) p[n++] = M(r, cc); };
    switch (t) {
    case T_DISTANCE: { auto *d = static_cast<DistanceConstraint *>(c); p[n++] = d->m_restLength; p[n++] = d->m_stiffness; break; }
    case T_DISTANCE_XPBD: { auto *d = static_cast<DistanceConstraint_XPBD *>(c); p[n++] = d->m_restLength; p[n++] = d->m_stiffness; *lambda = d->m_lambda; break; }
    case T_DIHEDRAL: { auto *d = static_cast<DihedralConstraint *>(c); p[n++] = d->m_restAngle; p[n++] = d->m_stiffness; break; }
    case T_ISOBENDING: { auto *d = static_cast<IsometricBendingConstraint *>(c); p[n++] = d->m_stiffness; putM(d->m_Q, 4, 4); break; }
    case T_ISOBENDING_XPBD: { auto *d = static_cast<IsometricBendingConstraint_XPBD *>(c); p[n++] = d->m_stiffness; putM(d->m_Q, 4, 4); *lambda = d->m_lambda; break; }
    case T_FEMTRIANGLE: { auto *d = static_cast<FEMTriangleConstraint *>(c); p[n++] = d->m_area; putM(d->m_invRestMat, 2, 2);
        p[n++] = d->m_xxStiffness; p[n++] = d->m_yyStiffness; p[n++] = d->m_xyStiffness; p[n++] = d->m_xyPoissonRatio; p[n++] = d->m_yxPoissonRatio; break; }
    case T_STRAINTRIANGLE: { auto *d = static_cast<StrainTriangleConstraint *>(c); putM(d->m_invRestMat, 2, 2);
        p[n++] = d->m_xxStiffness; p[n++] = d->m_yyStiffness; p[n++] = d->m_xyStiffness; p[n++] = d->m_normalizeStretch; p[n++] = d->m_normalizeShear; break; }
    case T_VOLUME: { auto *d = static_cast<VolumeConstraint *>(c); p[n++] = d->m_restVolume; p[n++] = d->m_stiffness; break; }
    case T_VOLUME_XPBD: { auto *d = static_cast<VolumeConstraint_XPBD *>(c); p[n++] = d->m_restVolume; p[n++] = d->m_stiffness; *lambda = d->m_lambda; break; }
    case T_FEMTET: { auto *d = static_cast<FEMTetConstraint *>(c); p[n++] = d->m_volume; putM(d->m_invRestMat, 3, 3); p[n++] = d->m_stiffness; p[n++] = d->m_poissonRatio; break; }
    case T_FEMTET_XPBD: { auto *d = static_cast<XPBD_FEMTetConstraint *>(c); p[n++] = d->m_volume; putM(d->m_invRestMat, 3, 3); p[n++] = d->m_stiffness; p[n++] = d->m_poissonRatio; *lambda = d->m_lambda; break; }
    case T_STRAINTET: { auto *d = static_cast<StrainTetConstraint *>(c); putM(d->m_invRestMat, 3, 3);
        p[n++] = d->m_stretchStiffness; p[n++] = d->m_shearStiffness; p[n++] = d->m_normalizeStretch; p[n++] = d->m_normalizeShear; break; }
    case T_BALLJOINT: { auto *d = static_cast<BallJoint *>(c); for (int col = 0; col < 4; col++) for (int k = 0; k < 3; k++) p[n++] = d->m_jointInfo(k, col); break; }
    case T_RB_PARTICLE_BALLJOINT: { auto *d = static_cast<RigidBodyParticleBallJoint *>(c); for (int col = 0; col < 2; col++) for (int k = 0; k < 3; k++) p[n++] = d->m_jointInfo(k, col); break; }
    case T_SHAPEMATCHING: { auto *d = static_cast<ShapeMatchingConstraint *>(c); p[n++] = d->m_stiffness;
        for (int k = 0; k < 3; k++) p[n++] = d->m_restCm[k];
        for (int q = 0; q < 4; q++) for (int k = 0; k < 3; k++) p[n++] = d->m_x0[q][k];
        for (int q = 0; q < 4; q++) p[n++] = d->m_w[q];
        for (int q = 0; q < 4; q++) p[n++] = d->m_numClusters[q];
        break; }
    default: break;
    }
    return t;
}

// Bulk export: types[n], bodies[4n] (unused = 0xffffffff), params[24n], nparams[n]
void ref_get_constraints(int *types, unsigned *bodies, double *params, int *nbodies) {
    auto &cs = g_model->getConstraints();
    for (size_t i = 0; i < cs.size(); i++) {
        unsigned b[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
        double p[32] = {0}; double lam;
        types[i] = ref_get_constraint((unsigned)i, b, p, &lam);
        nbodies[i] = (int)cs[i]->numberOfBodies();
        memcpy(bodies + 4 * i, b, sizeof(b));
        memcpy(params + 24 * i, p, 24 * sizeof(double));
    }
}

// n x TimeStepController::step (Simulation/TimeStepController.cpp:75); returns wall seconds of the n steps
double ref_step(int n) {
    TimeStep *ts = Simulation::getCurrent()->getTimeStep();
    auto t0 = std::chrono::steady_clock::now();
    for (int i = 0; i < n; i++) ts->step(*g_model);
    auto t1 = std::chrono::steady_clock::now();
    return std::chrono::duration<double>(t1 - t0).count();
}
double ref_time() { return TimeManager::getCurrent()->getTime(); }

// model-wide parameter setter (SimulationModel.cpp:1351-1485): rewrites the member of every constraint of the type, does not clear
// m_groupsInitialized -- what a GPU time step has to notice on its own
void ref_set_cloth_stiffness(double k) { g_model->setClothStiffness((Real)k); }

// ---------------------------------------------------------------------------------------------
// Contact path: the reference's DistanceFieldCollisionDetection set up the way Demos/DistanceFieldDemos/ClothCollisionDemo.cpp:120-182
// does -- static rigid bodies with analytic distance fields, triangle / tet models as point clouds.
// ---------------------------------------------------------------------------------------------
void ref_use_distance_field_cd(double tolerance) {
    if (!g_cd) { g_cd = new DistanceFieldCollisionDetection(); g_cd->init(); }
    Simulation::getCurrent()->getTimeStep()->setCollisionDetection(*g_model, g_cd);
    g_cd->setTolerance((Real)tolerance);
}
void ref_set_rigid_body_mass(unsigned i, double m) { g_model->getRigidBodies()[i]->setMass((Real)m); }
// shape: 0 box (dims = full extents), 1 sphere (radius), 2 torus (radii), 3 cylinder (radius, height), 4 hollow sphere (radius; thickness),
// 5 hollow box (full extents; thickness) -- the arguments of DistanceFieldCollisionDetection::addCollision* (:498-582)
int ref_add_rigid_collider(unsigned body, int shape, const double *dims, double thickness, int invert, double restitution, double friction) {
    if (!g_cd) return 1;
    RigidBody *rb = g_model->getRigidBodies()[body];
    rb->setRestitutionCoeff((Real)restitution); rb->setFrictionCoeff((Real)friction);
    const std::vector<Vector3r> &v = rb->getGeometry().getVertexDataLocal().getVertices();
    const unsigned nv = (unsigned)v.size();
    const unsigned type = CollisionDetection::CollisionObject::RigidBodyCollisionObjectType;
    switch (shape) {
    case 0: g_cd->addCollisionBox(body, type, v.data(), nv, v3(dims), true, invert != 0); break;
    case 1: g_cd->addCollisionSphere(body, type, v.data(), nv, (Real)dims[0], true, invert != 0); break;
    case 2: g_cd->addCollisionTorus(body, type, v.data(), nv, Vector2r((Real)dims[0], (Real)dims[1]), true, invert != 0); break;
    case 3: g_cd->addCollisionCylinder(body, type, v.data(), nv, Vector2r((Real)dims[0], (Real)dims[1]), true, invert != 0); break;
    case 4: g_cd->addCollisionHollowSphere(body, type, v.data(), nv, (Real)dims[0], (Real)thickness, true, invert != 0); break;
    case 5: g_cd->addCollisionHollowBox(body, type, v.data(), nv, v3(dims), (Real)thickness, true, invert != 0); break;
    default: return 2;
    }
    return 0;
}
// kind 0: triangle model, 1: tet model
int ref_add_model_collider(int kind, unsigned modelIndex, double restitution, double friction) {
    if (!g_cd) return 1;
    ParticleData &pd = g_model->getParticles();
    if (kind == 0) {
        TriangleModel *tm = g_model->getTriangleModels()[modelIndex];
        tm->setRestitutionCoeff((Real)restitution); tm->setFrictionCoeff((Real)friction);
        g_cd->addCollisionObjectWithoutGeometry(modelIndex, CollisionDetection::CollisionObject::TriangleModelCollisionObjectType,
                                                &pd.getPosition(tm->getIndexOffset()), tm->getParticleMesh().numVertices(), true);
    } else {
        TetModel *tm = g_model->getTetModels()[modelIndex];
        tm->setRestitutionCoeff((Real)restitution); tm->setFrictionCoeff((Real)friction);
        g_cd->addCollisionObjectWithoutGeometry(modelIndex, CollisionDetection::CollisionObject::TetModelCollisionObjectType,
                                                &pd.getPosition(tm->getIndexOffset()), tm->getParticleMesh().numVertices(), true);
    }
    return 0;
}
void ref_set_contact_params(double stiffnessParticleRigidBody, unsigned maxIterV) {
    g_model->setContactStiffnessParticleRigidBody((Real)stiffnessParticleRigidBody);
    TimeStep *ts = Simulation::getCurrent()->getTimeStep();
    ts->setValue<unsigned int>(TimeStepController::MAX_ITERATIONS_V, maxIterV);
}
// the contact list of the last step (SimulationModel::getParticleRigidBodyContactConstraints); out: 10 doubles per contact = cp0 | cp1 | n | 1/(n^T K n)
unsigned ref_num_contacts(unsigned *rigidRigid, unsigned *particleTet) {
    if (rigidRigid) *rigidRigid = (unsigned)g_model->getRigidBodyContactConstraints().size();
    if (particleTet) *particleTet = (unsigned)g_model->getParticleSolidContactConstraints().size();
    return (unsigned)g_model->getParticleRigidBodyContactConstraints().size();
}
void ref_get_contacts(unsigned *particle, unsigned *body, double *out) {
    auto &cs = g_model->getParticleRigidBodyContactConstraints();
    for (size_t i = 0; i < cs.size(); i++) {
        particle[i] = cs[i].m_bodies[0]; body[i] = cs[i].m_bodies[1];
        for (int col = 0; col < 3; col++) for (int k = 0; k < 3; k++) out[10 * i + 3 * col + k] = (double)cs[i].m_constraintInfo(k, col);
        out[10 * i + 9] = (double)cs[i].m_constraintInfo(0, 4);
    }
}
// what an adapter hands to pbd_set_colliders for collision object i: returns its kind (0 rigid analytic, 1 triangle model, 2 tet model,
// -1 other); out (rigid): shape, body, dim[3], thickness, invert, restitution, friction, R[9] row-major, v1[3], v2[3], aabbMin[3], aabbMax[3]
// = 30 doubles; out (model): offset, count, restitution, friction
unsigned ref_num_collision_objects() { return g_cd ? (unsigned)g_cd->getCollisionObjects().size() : 0u; }
int ref_collision_object_info(unsigned i, double *out) {
    typedef DistanceFieldCollisionDetection D;
    CollisionDetection::CollisionObject *co = g_cd->getCollisionObjects()[i];
    g_cd->updateAABB(*g_model, co);
    if (co->m_bodyType == CollisionDetection::CollisionObject::TriangleModelCollisionObjectType) {
        TriangleModel *tm = g_model->getTriangleModels()[co->m_bodyIndex];
        out[0] = tm->getIndexOffset(); out[1] = tm->getParticleMesh().numVertices(); out[2] = tm->getRestitutionCoeff(); out[3] = tm->getFrictionCoeff();
        return 1;
    }
    if (co->m_bodyType == CollisionDetection::CollisionObject::TetModelCollisionObjectType) {
        TetModel *tm = g_model->getTetModels()[co->m_bodyIndex];
        out[0] = tm->getIndexOffset(); out[1] = tm->getParticleMesh().numVertices(); out[2] = tm->getRestitutionCoeff(); out[3] = tm->getFrictionCoeff();
        return 2;
    }
    if (co->m_bodyType != CollisionDetection::CollisionObject::RigidBodyCollisionObjectType) return -1;
    int shape = -1; double dim[3] = {0, 0, 0}, thickness = 0;
    const int id = co->getTypeId();
    if (id == D::DistanceFieldCollisionBox::TYPE_ID) { shape = 0; auto *o = (D::DistanceFieldCollisionBox *)co; for (int k = 0; k < 3; k++) dim[k] = o->m_box[k]; }
    else if (id == D::DistanceFieldCollisionSphere::TYPE_ID) { shape = 1; dim[0] = ((D::DistanceFieldCollisionSphere *)co)->m_radius; }
    else if (id == D::DistanceFieldCollisionTorus::TYPE_ID) { shape = 2; auto *o = (D::DistanceFieldCollisionTorus *)co; dim[0] = o->m_radii[0]; dim[1] = o->m_radii[1]; }
    else if (id == D::DistanceFieldCollisionCylinder::TYPE_ID) { shape = 3; auto *o = (D::DistanceFieldCollisionCylinder *)co; dim[0] = o->m_dim[0]; dim[1] = o->m_dim[1]; }
    else if (id == D::DistanceFieldCollisionHollowSphere::TYPE_ID) { shape = 4; auto *o = (D::DistanceFieldCollisionHollowSphere *)co; dim[0] = o->m_radius; thickness = o->m_thickness; }
    else if (id == D::DistanceFieldCollisionHollowBox::TYPE_ID) { shape = 5; auto *o = (D::DistanceFieldCollisionHollowBox *)co; for (int k = 0; k < 3; k++) dim[k] = o->m_box[k]; thickness = o->m_thickness; }
    else return -1;
    RigidBody *rb = g_model->getRigidBodies()[co->m_bodyIndex];
    auto *dco = (D::DistanceFieldCollisionObject *)co;
    int n = 0;
    out[n++] = shape; out[n++] = co->m_bodyIndex; for (int k = 0; k < 3; k++) out[n++] = dim[k];
    out[n++] = thickness; out[n++] = (dco->m_invertSDF < 0) ? 1 : 0; out[n++] = rb->getRestitutionCoeff(); out[n++] = rb->getFrictionCoeff();
    const Matrix3r &R = rb->getTransformationR();
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) out[n++] = R(r, c);
    for (int k = 0; k < 3; k++) out[n++] = rb->getTransformationV1()[k];
    for (int k = 0; k < 3; k++) out[n++] = rb->getTransformationV2()[k];
    for (int k = 0; k < 3; k++) out[n++] = co->m_aabb.m_p[0][k];
    for (int k = 0; k < 3; k++) out[n++] = co->m_aabb.m_p[1][k];
    return 0;
}

#ifdef PBD_WITH_GPU_ADAPTER
// Install the GPU time step the way a user of the reference would (Simulation.h:48-49), carrying over the solver parameters.
// mode: PBD_MODE_* of include/pbd_b200.h.  Returns 0 on success.
int ref_use_gpu_timestep(int device, int mode) {
    Simulation *sim = Simulation::getCurrent();
    TimeStepController *old = static_cast<TimeStepController *>(sim->getTimeStep());
    const unsigned subSteps = old->getValue<unsigned int>(TimeStepController::NUM_SUB_STEPS);
    const unsigned maxIter = old->getValue<unsigned int>(TimeStepController::MAX_ITERATIONS);
    const int velMethod = old->getValue<int>(TimeStepController::VELOCITY_UPDATE_METHOD);
    GpuTimeStepController *ts = new GpuTimeStepController(device);
    ts->init();
    if (!ts->ok()) { g_gpuErr = ts->lastError(); delete ts; return 1; }
    ts->setMode(mode);
    ts->setValue<unsigned int>(GpuTimeStepController::NUM_SUB_STEPS, subSteps);
    ts->setValue<unsigned int>(GpuTimeStepController::MAX_ITERATIONS, maxIter);
    ts->setValue<int>(GpuTimeStepController::VELOCITY_UPDATE_METHOD, velMethod);
    delete old;
    sim->setTimeStep(ts);
    if (g_cd) ts->setCollisionDetection(*g_model, g_cd);  // what the user of the reference does after installing a time step
    g_gpuTs = ts;
    g_gpuErr.clear();
    return 0;
}
const char *ref_gpu_error() { if (g_gpuTs) g_gpuErr = g_gpuTs->lastError(); return g_gpuErr.c_str(); }
// Attach a collision detection with one collision object to the installed time step, the way the reference's demos do
// (TimeStep::setCollisionDetection, CollisionDetection::addCollisionObject): the GPU time step must then refuse to step.
namespace { struct NullCollisionDetection : public CollisionDetection { void collisionDetection(SimulationModel &) override {} }; }
int ref_attach_collision_object() {
    TimeStep *ts = Simulation::getCurrent()->getTimeStep();
    CollisionDetection *cd = new NullCollisionDetection();
    cd->addCollisionObject(0, CollisionDetection::CollisionObject::TriangleModelCollisionObjectType);
    ts->setCollisionDetection(*g_model, cd);
    return (int)cd->getCollisionObjects().size();
}
void ref_invalidate_gpu() { if (g_gpuTs) g_gpuTs->invalidate(); }
void ref_set_host_state_authoritative(int on) { if (g_gpuTs) g_gpuTs->setHostStateAuthoritative(on != 0); }
void ref_invalidate_state_gpu() { if (g_gpuTs) g_gpuTs->invalidateState(); }
int ref_download_history() { return (g_gpuTs && g_gpuTs->downloadHistory(*g_model)) ? 0 : 1; }
#endif

// ---------------------------------------------------------------------------------------------
// Known-answer entry points: call the stateless static solver functions directly.
// x: 4x3 positions, w: 4 inverse masses, p: params in the flat layout, corr: 4x3 out. Returns the bool result.
int ref_kat_solve(int type, const double *x, const double *w, const double *p, double dt, int handleInversion,
                  double *lambda, double *corr) {
    Vector3r X[4], C[4];
    Real W[4];
    for (int i = 0; i < 4; i++) { X[i] = v3(x + 3 * i); W[i] = (Real)w[i]; C[i].setZero(); }
    Real lam = (Real)*lambda;
    bool res = false;
    auto M2 = [&](const double *q) { Matrix2r m; m(0,0) = (Real)q[0]; m(0,1) = (Real)q[1]; m(1,0) = (Real)q[2]; m(1,1) = (Real)q[3]; return m; };
    auto M4 = [&](const double *q) { Matrix4r m; for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) m(r, c) = (Real)q[4*r+c]; return m; };
    switch (type) {
    case T_DISTANCE: res = PositionBasedDynamics::solve_DistanceConstraint(X[0], W[0], X[1], W[1], (Real)p[0], (Real)p[1], C[0], C[1]); break;
    case T_DISTANCE_XPBD: res = XPBD::solve_DistanceConstraint(X[0], W[0], X[1], W[1], (Real)p[0], (Real)p[1], (Real)dt, lam, C[0], C[1]); break;
    case T_DIHEDRAL: res = PositionBasedDynamics::solve_DihedralConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], (Real)p[0], (Real)p[1], C[0], C[1], C[2], C[3]); break;
    case T_ISOBENDING: res = PositionBasedDynamics::solve_IsometricBendingConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], M4(p + 1), (Real)p[0], C[0], C[1], C[2], C[3]); break;
    case T_ISOBENDING_XPBD: res = XPBD::solve_IsometricBendingConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], M4(p + 1), (Real)p[0], (Real)dt, lam, C[0], C[1], C[2], C[3]); break;
    case T_FEMTRIANGLE: { Real area = (Real)p[0]; res = PositionBasedDynamics::solve_FEMTriangleConstraint(X[0], W[0], X[1], W[1], X[2], W[2], area, M2(p + 1), (Real)p[5], (Real)p[6], (Real)p[7], (Real)p[8], (Real)p[9], C[0], C[1], C[2]); break; }
    case T_STRAINTRIANGLE: res = PositionBasedDynamics::solve_StrainTriangleConstraint(X[0], W[0], X[1], W[1], X[2], W[2], M2(p), (Real)p[4], (Real)p[5], (Real)p[6], p[7] != 0, p[8] != 0, C[0], C[1], C[2]); break;
    case T_VOLUME: res = PositionBasedDynamics::solve_VolumeConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], (Real)p[0], (Real)p[1], C[0], C[1], C[2], C[3]); break;
    case T_VOLUME_XPBD: res = XPBD::solve_VolumeConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], (Real)p[0], (Real)p[1], (Real)dt, lam, C[0], C[1], C[2], C[3]); break;
    case T_FEMTET: res = PositionBasedDynamics::solve_FEMTetraConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], (Real)p[0], m3(p + 1), (Real)p[10], (Real)p[11], handleInversion != 0, C[0], C[1], C[2], C[3]); break;
    case T_FEMTET_XPBD: res = XPBD::solve_FEMTetraConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], (Real)p[0], m3(p + 1), (Real)p[10], (Real)p[11], handleInversion != 0, (Real)dt, lam, C[0], C[1], C[2], C[3]); break;
    case T_STRAINTET: res = PositionBasedDynamics::solve_StrainTetraConstraint(X[0], W[0], X[1], W[1], X[2], W[2], X[3], W[3], m3(p), (Real)p[9] * Vector3r::Ones(), (Real)p[10] * Vector3r::Ones(), p[11] != 0, p[12] != 0, C[0], C[1], C[2], C[3]); break;
    case T_SHAPEMATCHING: {  // raw solver answer; frozen x0 / w copies come from p (layout of ref_get_constraint)
        Vector3r q0[4]; Real ws[4];
        for (int i = 0; i < 4; i++) { q0[i] = v3(p + 4 + 3 * i); ws[i] = (Real)p[16 + i]; }
        res = PositionBasedDynamics::solve_ShapeMatchingConstraint(q0, X, ws, 4, v3(p + 1), (Real)p[0], false, C); break; }
    default: return -1;
    }
    *lambda = lam;
    for (int i = 0; i < 4; i++) for (int k = 0; k < 3; k++) corr[3 * i + k] = C[i][k];
    return res ? 1 : 0;
}

// init_* known answers: out receives the rest data in the flat layout (without stiffness fields)
int ref_kat_init(int type, const double *x, double *out) {
    Vector3r X[4];
    for (int i = 0; i < 4; i++) X[i] = v3(x + 3 * i);
    int n = 0;
    switch (type) {
    case T_ISOBENDING: case T_ISOBENDING_XPBD: { Matrix4r Q; bool r = PositionBasedDynamics::init_IsometricBendingConstraint(X[0], X[1], X[2], X[3], Q);
        for (int a = 0; a < 4; a++) for (int b = 0; b < 4; b++) out[n++] = Q(a, b); return r; }
    case T_FEMTRIANGLE: { Real area; Matrix2r m; bool r = PositionBasedDynamics::init_FEMTriangleConstraint(X[0], X[1], X[2], area, m);
        out[n++] = area; out[n++] = m(0,0); out[n++] = m(0,1); out[n++] = m(1,0); out[n++] = m(1,1); return r; }
    case T_STRAINTRIANGLE: { Matrix2r m; bool r = PositionBasedDynamics::init_StrainTriangleConstraint(X[0], X[1], X[2], m);
        out[n++] = m(0,0); out[n++] = m(0,1); out[n++] = m(1,0); out[n++] = m(1,1); return r; }
    case T_FEMTET: case T_FEMTET_XPBD: { Real vol; Matrix3r m; bool r = PositionBasedDynamics::init_FEMTetraConstraint(X[0], X[1], X[2], X[3], vol, m);
        out[n++] = vol; for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) out[n++] = m(a, b); return r; }
    case T_STRAINTET: { Matrix3r m; bool r = PositionBasedDynamics::init_StrainTetraConstraint(X[0], X[1], X[2], X[3], m);
        for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) out[n++] = m(a, b); return r; }
    default: return -1;
    }
}

// MathFunctions::svdWithInversionHandling (MathFunctions.cpp:261-388); A row-major in; out: sigma[3], U[9], VT[9]
void ref_kat_svd(const double *A, double *sigma, double *U, double *VT) {
    Matrix3r a = m3(A), u, vt; Vector3r s;
    MathFunctions::svdWithInversionHandling(a, s, u, vt);
    for (int r = 0; r < 3; r++) { sigma[r] = s[r]; for (int c = 0; c < 3; c++) { U[3*r+c] = u(r, c); VT[3*r+c] = vt(r, c); } }
}

// TimeIntegration known answers (TimeIntegration.cpp:7-19, 42-51, 69-79)
void ref_kat_integrate(double h, double mass, double *x, double *v, const double *a) {
    Vector3r X = v3(x), V = v3(v);
    TimeIntegration::semiImplicitEuler((Real)h, (Real)mass, X, V, v3(a));
    for (int k = 0; k < 3; k++) { x[k] = X[k]; v[k] = V[k]; }
}
void ref_kat_velocity_update(int order, double h, double mass, const double *x, const double *oldX, const double *lastX, double *v) {
    Vector3r V = v3(v);
    if (order == 0) TimeIntegration::velocityUpdateFirstOrder((Real)h, (Real)mass, v3(x), v3(oldX), V);
    else TimeIntegration::velocityUpdateSecondOrder((Real)h, (Real)mass, v3(x), v3(oldX), v3(lastX), V);
    for (int k = 0; k < 3; k++) v[k] = V[k];
}

} // extern "C"
