// positionbaseddynamics_b200/csrc/host/pbd_model.h
//
// Host-side mirror of the reference's model interface for the constraint-projection path: the same class and
// method names, argument meaning and bool/void error behaviour as
//   Simulation/ParticleData.h:86-311, Utils/IndexedFaceMesh.h, Utils/IndexedTetMesh.h, Simulation/TriangleModel.h,
//   Simulation/TetModel.h, Simulation/SimulationModel.h:134-327, Simulation/TimeStepController.h, Simulation/TimeManager.h
// so that scene-building code written against the reference drives the H100 engine unchanged.  The storage behind
// the interface is NOT the reference's: constraints live in per-type structure-of-arrays stores (no heap object and
// no vtable per constraint), which is what the device image is flattened from.
#pragma once
#include <array>
#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <vector>
#include "../../../include/pbd_b200.h"

namespace pbd_b200 {

using Real = float;  // the engine is fp32 (Common/Common.h:7-28 with USE_DOUBLE undefined)

struct Vector3r {
    Real v[3];
    Vector3r() : v{0, 0, 0} {}
    Vector3r(Real x, Real y, Real z) : v{x, y, z} {}
    Real &operator[](int i) { return v[i]; }
    const Real &operator[](int i) const { return v[i]; }
};
static_assert(sizeof(Vector3r) == 12, "Vector3r must be 3 packed floats (Eigen::DontAlign layout, Common/Common.h:31)");
struct Vector2r { Real v[2]; Real &operator[](int i) { return v[i]; } const Real &operator[](int i) const { return v[i]; } };
struct Matrix3r {  // row-major
    Real m[9];
    static Matrix3r Identity() { Matrix3r r{}; r.m[0] = r.m[4] = r.m[8] = 1; return r; }
    Real operator()(int r, int c) const { return m[3 * r + c]; }
    Real &operator()(int r, int c) { return m[3 * r + c]; }
};

// ---------------------------------------------------------------------------------------------------------
// ParticleData (Simulation/ParticleData.h:86-311)
// ---------------------------------------------------------------------------------------------------------
class SimulationModel;
class ParticleData {
public:
    void addVertex(const Vector3r &vertex);  // mass = invMass = 1, v = a = 0, x0 = x = oldX = lastX (ParticleData.h:127-137)
    void addVertices(const Vector3r *vertices, unsigned int n);  // n x addVertex in one go
    unsigned int size() const { return (unsigned int)m_x.size(); }
    unsigned int getNumberOfParticles() const { return size(); }
    void reserve(unsigned int n);
    void release();

    // Non-const accessors hand out lvalues exactly like the reference; they first pull that attribute from the device
    // when the engine is ahead and mark it as modified on the host (the next step re-uploads it).
    Vector3r &getPosition(unsigned int i) { touch(PBD_ATTR_X); return m_x[i]; }
    Vector3r &getPosition0(unsigned int i) { touch(PBD_ATTR_X0); return m_x0[i]; }
    Vector3r &getVelocity(unsigned int i) { touch(PBD_ATTR_V); return m_v[i]; }
    Vector3r &getAcceleration(unsigned int i) { return m_a[i]; }
    Vector3r &getOldPosition(unsigned int i) { touch(PBD_ATTR_OLDX); return m_oldX[i]; }
    Vector3r &getLastPosition(unsigned int i) { touch(PBD_ATTR_LASTX); return m_lastX[i]; }
    const Vector3r &getPosition(unsigned int i) const { pull(PBD_ATTR_X); return m_x[i]; }
    const Vector3r &getPosition0(unsigned int i) const { return m_x0[i]; }
    const Vector3r &getVelocity(unsigned int i) const { pull(PBD_ATTR_V); return m_v[i]; }
    const Vector3r &getOldPosition(unsigned int i) const { pull(PBD_ATTR_OLDX); return m_oldX[i]; }
    const Vector3r &getLastPosition(unsigned int i) const { pull(PBD_ATTR_LASTX); return m_lastX[i]; }
    void setPosition(unsigned int i, const Vector3r &p) { touch(PBD_ATTR_X); m_x[i] = p; }
    void setPosition0(unsigned int i, const Vector3r &p) { touch(PBD_ATTR_X0); m_x0[i] = p; }
    void setVelocity(unsigned int i, const Vector3r &p) { touch(PBD_ATTR_V); m_v[i] = p; }
    void setAcceleration(unsigned int i, const Vector3r &p) { m_a[i] = p; }
    Real getMass(unsigned int i) const { return m_masses[i]; }
    Real getInvMass(unsigned int i) const { return m_invMasses[i]; }
    void setMass(unsigned int i, Real mass);  // keeps invMass consistent (ParticleData.h:239-246)
    const std::vector<Vector3r> &getVertices() const { pull(PBD_ATTR_X); return m_x; }  // pyPBD getVertices (ParticleDataModule.cpp:54-58)

    // raw storage (reference member names)
    std::vector<Real> m_masses, m_invMasses;
    std::vector<Vector3r> m_x0, m_x, m_v, m_a, m_oldX, m_lastX;

    // coherence with the device image: one bit per pbd_attr
    mutable unsigned int dirtyMask = 0x1f;  // host copy of the attribute modified since the last upload
    mutable unsigned int aheadMask = 0;     // device copy of the attribute newer than the host copy
    mutable bool massDirty = true;
    std::function<bool(int)> pullAttr;      // installed by the TimeStepController that owns the engine
    void touch(int attr) const { pull(attr); dirtyMask |= 1u << attr; }
    void pull(int attr) const { if ((aheadMask >> attr) & 1u) { if (pullAttr && pullAttr(attr)) aheadMask &= ~(1u << attr); } }
    void pullAll() const { for (int a = 0; a < 5; a++) pull(a); }
};

// ---------------------------------------------------------------------------------------------------------
// Mesh topology (Utils/IndexedFaceMesh.{h,cpp}, Utils/IndexedTetMesh.{h,cpp}); the edge DISCOVERY ORDER defines the
// constraint order, hence the colouring and the Gauss-Seidel order.
// ---------------------------------------------------------------------------------------------------------
// std::vector whose resize() leaves new trivially-constructible elements uninitialised: the bulk builders size a store once and fill it
// from all threads (first touch in parallel instead of one thread zeroing hundreds of megabytes first)
template <class T> struct DefaultInitAllocator : std::allocator<T> {
    template <class U> struct rebind { typedef DefaultInitAllocator<U> other; };
    DefaultInitAllocator() = default;
    template <class U> DefaultInitAllocator(const DefaultInitAllocator<U> &) {}
    template <class U> void construct(U *p) { ::new (static_cast<void *>(p)) U; }
    template <class U, class... Args> void construct(U *p, Args &&...args) { ::new (static_cast<void *>(p)) U(std::forward<Args>(args)...); }
};
template <class T> using PodVector = std::vector<T, DefaultInitAllocator<T>>;
class IndexedFaceMesh {
public:
    struct Edge { std::array<unsigned int, 2> m_face; std::array<unsigned int, 2> m_vert; };  // IndexedFaceMesh.h:14-18
    typedef std::vector<unsigned int> Faces;
    typedef PodVector<Edge> Edges;
    void initMesh(unsigned int nPoints, unsigned int nEdges, unsigned int nFaces);
    void addFace(const unsigned int *indices);
    void addFaces(const unsigned int *indices, unsigned int nFaces);
    void buildNeighbors();  // IndexedFaceMesh.cpp:118-226
    const Faces &getFaces() const { return m_indices; }
    const Edges &getEdges() const { return m_edges; }
    unsigned int numVertices() const { return m_numPoints; }
    unsigned int numFaces() const { return (unsigned int)m_indices.size() / 3; }
    unsigned int numEdges() const { return (unsigned int)m_edges.size(); }
    bool isClosed() const { return m_closed; }
private:
    unsigned int m_numPoints = 0;
    Faces m_indices;
    Edges m_edges;
    bool m_closed = false;
};

class IndexedTetMesh {
public:
    struct Edge { std::array<unsigned int, 2> m_vert; };
    typedef std::vector<unsigned int> Tets;
    typedef std::vector<Edge> Edges;
    void initMesh(unsigned int nPoints, unsigned int nEdges, unsigned int nFaces, unsigned int nTets);
    void addTet(const unsigned int *indices);
    void buildNeighbors();  // IndexedTetMesh.cpp:55-182 (edges + vertex->tet incidence; faces are not needed on this path)
    const Tets &getTets() const { return m_tetIndices; }
    const Edges &getEdges() const { return m_edges; }
    const std::vector<unsigned int> &getVertexTetCounts() const { return m_vertexTetCount; }
    unsigned int numVertices() const { return m_numPoints; }
    unsigned int numTets() const { return (unsigned int)m_tetIndices.size() / 4; }
    unsigned int numEdges() const { return (unsigned int)m_edges.size(); }
private:
    unsigned int m_numPoints = 0;
    Tets m_tetIndices;
    Edges m_edges;
    std::vector<unsigned int> m_vertexTetCount;
};

class TriangleModel {
public:
    typedef IndexedFaceMesh ParticleMesh;
    void initMesh(unsigned int nPoints, unsigned int nFaces, unsigned int indexOffset, const unsigned int *indices);  // TriangleModel.cpp:30-43
    ParticleMesh &getParticleMesh() { return m_particleMesh; }
    const ParticleMesh &getParticleMesh() const { return m_particleMesh; }
    unsigned int getIndexOffset() const { return m_indexOffset; }
    Real getRestitutionCoeff() const { return m_restitutionCoeff; }   // TriangleModel.cpp constructor: 0.6 / 0.2
    void setRestitutionCoeff(Real v) { m_restitutionCoeff = v; }
    Real getFrictionCoeff() const { return m_frictionCoeff; }
    void setFrictionCoeff(Real v) { m_frictionCoeff = v; }
private:
    unsigned int m_indexOffset = 0;
    ParticleMesh m_particleMesh;
    Real m_restitutionCoeff = static_cast<Real>(0.6), m_frictionCoeff = static_cast<Real>(0.2);
};

class TetModel {
public:
    typedef IndexedTetMesh ParticleMesh;
    void initMesh(unsigned int nPoints, unsigned int nTets, unsigned int indexOffset, const unsigned int *indices);  // TetModel.cpp
    ParticleMesh &getParticleMesh() { return m_particleMesh; }
    const ParticleMesh &getParticleMesh() const { return m_particleMesh; }
    unsigned int getIndexOffset() const { return m_indexOffset; }
    Real getRestitutionCoeff() const { return m_restitutionCoeff; }   // TetModel.cpp constructor: 0.6 / 0.2
    void setRestitutionCoeff(Real v) { m_restitutionCoeff = v; }
    Real getFrictionCoeff() const { return m_frictionCoeff; }
    void setFrictionCoeff(Real v) { m_frictionCoeff = v; }
private:
    unsigned int m_indexOffset = 0;
    ParticleMesh m_particleMesh;
    Real m_restitutionCoeff = static_cast<Real>(0.6), m_frictionCoeff = static_cast<Real>(0.2);
};

// ---------------------------------------------------------------------------------------------------------
// RigidBody (Simulation/RigidBody.h): the state that takes part in the coloured sweep through BallJoint /
// RigidBodyParticleBallJoint (SURVEY.md 8f-1).  Geometry, contacts and the other joint types stay with the reference.
// ---------------------------------------------------------------------------------------------------------
struct Quaternionr { Real w, x, y, z; Quaternionr(Real w_ = 1, Real x_ = 0, Real y_ = 0, Real z_ = 0) : w(w_), x(x_), y(y_), z(z_) {} };
class RigidBody {
public:
    // initBody(mass, x, inertiaTensor, rotation, ...) of the reference without the mesh arguments (RigidBody.h:84-120)
    void initBody(Real mass, const Vector3r &x, const Vector3r &inertiaTensor, const Quaternionr &rotation);
    Real getMass() const { return m_mass; }
    Real getInvMass() const { return m_invMass; }
    const Vector3r &getPosition() const { return m_x; }
    const Vector3r &getPosition0() const { return m_x0; }
    const Vector3r &getVelocity() const { return m_v; }
    const Vector3r &getAngularVelocity() const { return m_omega; }
    const Quaternionr &getRotation() const { return m_q; }
    const Vector3r &getInertiaTensor() const { return m_inertiaTensor; }
    Real getRestitutionCoeff() const { return m_restitutionCoeff; }   // RigidBody.h:115-116: 0.6 / 0.2
    void setRestitutionCoeff(Real v) { m_restitutionCoeff = v; }
    Real getFrictionCoeff() const { return m_frictionCoeff; }
    void setFrictionCoeff(Real v) { m_frictionCoeff = v; }
    Real m_restitutionCoeff = static_cast<Real>(0.6), m_frictionCoeff = static_cast<Real>(0.2);
    // Frame of the body's geometry (what the reference keeps as m_x0_mat / m_q_mat / m_q_initial, RigidBody.h:172-188): a distance field
    // attached to the body is evaluated at  x_local = frameR * R(q)^T (x_world - x) + frameT.  Identity / zero for bodies created in their
    // own frame; a body moved to its centre of mass and principal axes sets the principal-axes matrix and the centre of mass here.
    Matrix3r m_frameR = Matrix3r::Identity();
    Vector3r m_frameT;
    Real m_mass = 0, m_invMass = 0;
    Vector3r m_x, m_x0, m_v, m_omega, m_inertiaTensor;
    Quaternionr m_q, m_q0;
};

// ---------------------------------------------------------------------------------------------------------
// Constraint storage: per-type SoA in the flat parameter layout of include/pbd_b200.h, plus the global insertion
// order (the reference's m_constraints vector) as (type, local index) pairs.
// ---------------------------------------------------------------------------------------------------------
struct ConstraintRef { int type; unsigned int local; };
struct ConstraintView {  // what `model.getConstraints()[i]` exposes
    int type; unsigned int numberOfBodies; const unsigned int *m_bodies; const Real *params; unsigned int numParams;
};
struct TypeStore { PodVector<unsigned int> ids, bodies; PodVector<Real> params; };

class SimulationModel {
public:
    typedef std::vector<RigidBody *> RigidBodyVector;
    typedef std::vector<TriangleModel *> TriangleModelVector;
    typedef std::vector<TetModel *> TetModelVector;
    typedef std::vector<std::vector<unsigned int>> ConstraintGroupVector;

    SimulationModel();
    ~SimulationModel();
    void init() {}
    void reset();    // SimulationModel.cpp:270-304: x = x0 = oldX = lastX, v = a = 0
    void cleanup();  // SimulationModel.cpp:105-126

    RigidBodyVector &getRigidBodies() { return m_rigidBodies; }  // the caller pushes bodies, the model deletes them (SimulationModel.cpp:105-126)
    bool addBallJoint(unsigned int rbIndex1, unsigned int rbIndex2, const Vector3r &pos);                  // SimulationModel.cpp:306-317
    bool addRigidBodyParticleBallJoint(unsigned int rbIndex, unsigned int particleIndex);                  // SimulationModel.cpp:449-460
    mutable bool rigidBodiesDirty = true;   // host copy newer than the device copy
    ParticleData &getParticles() { return m_particles; }
    TriangleModelVector &getTriangleModels() { return m_triangleModels; }
    TetModelVector &getTetModels() { return m_tetModels; }
    ConstraintGroupVector &getConstraintGroups() { return m_constraintGroups; }
    unsigned int numConstraints() const { return (unsigned int)m_order.size(); }
    ConstraintView getConstraint(unsigned int i) const;
    bool m_groupsInitialized = false;

    void addTriangleModel(unsigned int nPoints, unsigned int nFaces, const Vector3r *points, const unsigned int *indices);
    void addRegularTriangleModel(int width, int height, const Vector3r &translation = Vector3r(), const Matrix3r &rotation = Matrix3r::Identity(),
                                 const Vector2r &scale = Vector2r{{1, 1}});
    void addTetModel(unsigned int nPoints, unsigned int nTets, const Vector3r *points, const unsigned int *indices);
    void addRegularTetModel(int width, int height, int depth, const Vector3r &translation = Vector3r(), const Matrix3r &rotation = Matrix3r::Identity(),
                            const Vector3r &scale = Vector3r(1, 1, 1));

    void initConstraintGroups();  // SimulationModel.cpp:1033-1094 (greedy first fit, insertion order)

    // each returns false (and adds nothing) when the rest configuration is degenerate, like the reference
    bool addDistanceConstraint(unsigned int p1, unsigned int p2, Real stiffness);
    bool addDistanceConstraint_XPBD(unsigned int p1, unsigned int p2, Real stiffness);
    bool addDihedralConstraint(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stiffness);
    bool addIsometricBendingConstraint(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stiffness);
    bool addIsometricBendingConstraint_XPBD(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stiffness);
    bool addFEMTriangleConstraint(unsigned int p1, unsigned int p2, unsigned int p3, Real xxStiffness, Real yyStiffness, Real xyStiffness,
                                  Real xyPoissonRatio, Real yxPoissonRatio);
    bool addStrainTriangleConstraint(unsigned int p1, unsigned int p2, unsigned int p3, Real xxStiffness, Real yyStiffness, Real xyStiffness,
                                     bool normalizeStretch, bool normalizeShear);
    bool addVolumeConstraint(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stiffness);
    bool addVolumeConstraint_XPBD(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stiffness);
    bool addFEMTetConstraint(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stiffness, Real poissonRatio);
    bool addFEMTetConstraint_XPBD(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stiffness, Real poissonRatio);
    bool addStrainTetConstraint(unsigned int p1, unsigned int p2, unsigned int p3, unsigned int p4, Real stretchStiffness, Real shearStiffness,
                                bool normalizeStretch, bool normalizeShear);
    // clusters of exactly 4 particles (what addSolidConstraints method 5 creates); other cluster sizes are rejected
    bool addShapeMatchingConstraint(unsigned int numberOfParticles, const unsigned int particleIndices[], const unsigned int numClusters[], Real stiffness);

    void addClothConstraints(const TriangleModel *tm, unsigned int clothMethod, Real distanceStiffness, Real xxStiffness, Real yyStiffness,
                             Real xyStiffness, Real xyPoissonRatio, Real yxPoissonRatio, bool normalizeStretch, bool normalizeShear);
    void addBendingConstraints(const TriangleModel *tm, unsigned int bendingMethod, Real stiffness);
    void addSolidConstraints(const TetModel *tm, unsigned int solidMethod, Real stiffness, Real poissonRatio, Real volumeStiffness,
                             bool normalizeStretch, bool normalizeShear);

    // global stiffness setters (SimulationModel.cpp:1351-1485); reference quirk kept: YY and XY write the XX member (:1365-1377)
    void setClothStiffness(Real val);
    void setClothStiffnessXX(Real val);
    void setClothStiffnessYY(Real val);
    void setClothStiffnessXY(Real val);
    void setClothPoissonRatioXY(Real val);
    void setClothPoissonRatioYX(Real val);
    void setClothBendingStiffness(Real val);
    void setClothNormalizeStretch(bool val);
    void setClothNormalizeShear(bool val);
    void setSolidStiffness(Real val);
    void setSolidPoissonRatio(Real val);
    void setSolidVolumeStiffness(Real val);
    void setSolidNormalizeStretch(bool val);
    void setSolidNormalizeShear(bool val);

    // SimulationModel.h:253-254, SimulationModel.cpp:57
    Real getContactStiffnessParticleRigidBody() const { return m_contactStiffnessParticleRigidBody; }
    void setContactStiffnessParticleRigidBody(Real val) { m_contactStiffnessParticleRigidBody = val; }

    // flat view for the engine
    const TypeStore &store(int type) const { return m_store[type]; }
    uint64_t constraintGeneration() const { return m_generation; }  // bumps whenever constraints or their parameters change

private:
    bool pushConstraint(int type, const unsigned int *bodies, const Real *params, bool ok);
    void reserveConstraints(int type, size_t count);
    void setParam(int type, int slot, Real val);
    ParticleData m_particles;
    RigidBodyVector m_rigidBodies;
    TriangleModelVector m_triangleModels;
    TetModelVector m_tetModels;
    TypeStore m_store[PBD_NUM_TYPES];
    PodVector<ConstraintRef> m_order;
    ConstraintGroupVector m_constraintGroups;
    uint64_t m_generation = 1;
    Real m_contactStiffnessParticleRigidBody = static_cast<Real>(100.0);
};

// OpenMP team size of the host-side model build and of the engine's flatten (capped; PBD_B200_HOST_THREADS sets the cap)
int host_threads();

// Greedy first-fit colouring shared by SimulationModel::initConstraintGroups and pbd_color_first_fit: constraint c uses
// bodies[bodyOff[c] .. bodyOff[c+1]); returns per-constraint colour and the number of colours.
unsigned int firstFitColouring(unsigned int numBodies, unsigned int numConstraints, const unsigned int *bodyOff,
                               const unsigned int *bodies, std::vector<unsigned int> &colour);

// ---------------------------------------------------------------------------------------------------------
// TimeManager / TimeStepController (Simulation/TimeManager.h, Simulation/TimeStepController.{h,cpp})
// ---------------------------------------------------------------------------------------------------------
// ---------------------------------------------------------------------------------------------------------
// CollisionDetection / DistanceFieldCollisionDetection (Simulation/CollisionDetection.h:15-104,
// Simulation/DistanceFieldCollisionDetection.h): the registry of collision objects with the reference's add* signatures.  The
// tests themselves run on the GPU (csrc/contacts.cuh); this class only holds what pbd_set_colliders needs.  The reference takes
// a collision object's bounding box from the rigid body's mesh; the bodies of this mirror carry no mesh, so the box is taken
// from the vertices handed to add* (the same local vertices the reference builds its bounding-sphere hierarchy from).
// ---------------------------------------------------------------------------------------------------------
class CollisionDetection {
public:
    struct CollisionObject {
        static const unsigned int RigidBodyCollisionObjectType = 0, TriangleModelCollisionObjectType = 1, TetModelCollisionObjectType = 2;
        unsigned int m_bodyIndex = 0, m_bodyType = 0;
        int shape = -1;                       // pbd_collider_shape, -1 = object without geometry
        Real dim[3] = {0, 0, 0}, thickness = 0;
        bool m_testMesh = true; bool invertSDF = false;
        std::vector<Vector3r> vertices;       // local vertices (bounding box source)
    };
    virtual ~CollisionDetection() {}
    Real getTolerance() const { return m_tolerance; }
    void setTolerance(Real v) { m_tolerance = v; }
    std::vector<CollisionObject> &getCollisionObjects() { return m_collisionObjects; }
    void cleanup() { m_collisionObjects.clear(); }
protected:
    Real m_tolerance = static_cast<Real>(0.01);  // CollisionDetection.cpp:25
    std::vector<CollisionObject> m_collisionObjects;
};
class DistanceFieldCollisionDetection : public CollisionDetection {
public:
    // DistanceFieldCollisionDetection.cpp:498-582 (box / hollow box take the full extents, cylinder radius and full height)
    void addCollisionBox(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector3r &box, bool testMesh = true, bool invertSDF = false);
    void addCollisionSphere(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, Real radius, bool testMesh = true, bool invertSDF = false);
    void addCollisionTorus(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector2r &radii, bool testMesh = true, bool invertSDF = false);
    void addCollisionCylinder(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector2r &dim, bool testMesh = true, bool invertSDF = false);
    void addCollisionHollowSphere(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, Real radius, Real thickness, bool testMesh = true, bool invertSDF = false);
    void addCollisionHollowBox(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector3r &box, Real thickness, bool testMesh = true, bool invertSDF = false);
    void addCollisionObjectWithoutGeometry(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, bool testMesh);
private:
    CollisionObject &add(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, int shape, bool testMesh, bool invertSDF);
};

class TimeManager {
public:
    Real getTime() const { return time; }
    void setTime(Real t) { time = t; }
    Real getTimeStepSize() const { return h; }
    void setTimeStepSize(Real tss) { h = tss; }
private:
    Real time = 0; Real h = static_cast<Real>(0.005);  // TimeManager.cpp:10
};

class TimeStepController {
public:
    // parameter ids with the reference's names (TimeStepController.h:16-22, .cpp:47-72)
    static const int NUM_SUB_STEPS = 0, MAX_ITERATIONS = 1, MAX_ITERATIONS_V = 2, VELOCITY_UPDATE_METHOD = 3;
    static const int ENUM_VUPDATE_FIRST_ORDER = 0, ENUM_VUPDATE_SECOND_ORDER = 1;

    explicit TimeStepController(int device = 0, void *stream = nullptr);
    ~TimeStepController();
    bool valid() const { return m_engine != nullptr; }
    const std::string &error() const { return m_error; }

    void init() {}
    void reset();                         // TimeStepController.cpp:243-249
    bool step(SimulationModel &model);    // TimeStepController.cpp:75-241; false + error() on CUDA failure (reference: void)

    unsigned int getValueUInt(int id) const;
    bool setValueUInt(int id, unsigned int v);
    int getValueInt(int id) const { return id == VELOCITY_UPDATE_METHOD ? m_velocityUpdateMethod : 0; }
    bool setValueInt(int id, int v);
    void setGravitation(const Vector3r &g) { m_gravitation = g; }  // Simulation::GRAVITATION (Simulation.cpp:63)
    const Vector3r &getGravitation() const { return m_gravitation; }
    TimeManager &timeManager() { return m_tm; }
    pbd_engine *engine() { return m_engine; }
    void setSolverMode(int mode) { m_mode = mode; }
    // TimeStep::setCollisionDetection (TimeStep.cpp:63-68).  Covered on the GPU: particles of triangle / tet models against analytic
    // distance fields on static rigid bodies; step() fails with error() for anything else (dynamic collision bodies, two tet models).
    void setCollisionDetection(SimulationModel &model, CollisionDetection *cd) { (void)model; m_collisionDetection = cd; }
    CollisionDetection *getCollisionDetection() { return m_collisionDetection; }

private:
    bool uploadModel(SimulationModel &model);
    bool uploadColliders(SimulationModel &model);
    bool fail(const char *what);
    CollisionDetection *m_collisionDetection = nullptr;
    std::vector<unsigned char> m_collidersSent;  // byte image of the last pbd_set_colliders arguments
    pbd_engine *m_engine = nullptr;
    std::string m_error;
    TimeManager m_tm;
    unsigned int m_subSteps = 5, m_maxIterations = 1, m_maxIterationsV = 5;  // TimeStepController.cpp:28-30
    int m_velocityUpdateMethod = 0;
    Vector3r m_gravitation = Vector3r(0, static_cast<Real>(-9.81), 0);  // Simulation.cpp:16
    int m_mode = PBD_MODE_AUTO, m_modeSent = -1;
    const SimulationModel *m_boundModel = nullptr;
    uint64_t m_boundGeneration = 0;
    unsigned int m_boundParticles = 0, m_boundRigidBodies = 0;
};

}  // namespace pbd_b200
