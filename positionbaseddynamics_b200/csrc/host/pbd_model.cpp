// positionbaseddynamics_b200/csrc/host/pbd_model.cpp -- see pbd_model.h.
#include "pbd_model.h"
#include "../rest_geometry.cuh"
#include <algorithm>
#include <cstdlib>
#include <omp.h>
#include <parallel/algorithm>
#include <cmath>
#include <cstring>
#include <unordered_map>

namespace pbd_b200 {

// ============================================================================================================
// ParticleData
// ============================================================================================================
void ParticleData::addVertex(const Vector3r &vertex) {
    m_x0.push_back(vertex); m_x.push_back(vertex); m_oldX.push_back(vertex); m_lastX.push_back(vertex);
    m_masses.push_back(1.0f); m_invMasses.push_back(1.0f);
    m_v.push_back(Vector3r()); m_a.push_back(Vector3r());
    dirtyMask = 0x1f; massDirty = true;
}
void ParticleData::addVertices(const Vector3r *vertices, unsigned int n) {
    for (auto *v : {&m_x0, &m_x, &m_oldX, &m_lastX}) v->insert(v->end(), vertices, vertices + n);
    m_masses.insert(m_masses.end(), n, 1.0f); m_invMasses.insert(m_invMasses.end(), n, 1.0f);
    m_v.insert(m_v.end(), n, Vector3r()); m_a.insert(m_a.end(), n, Vector3r());
    dirtyMask = 0x1f; massDirty = true;
}
void ParticleData::reserve(unsigned int n) {
    m_masses.reserve(n); m_invMasses.reserve(n); m_x0.reserve(n); m_x.reserve(n); m_v.reserve(n); m_a.reserve(n);
    m_oldX.reserve(n); m_lastX.reserve(n);
}
void ParticleData::release() {
    m_masses.clear(); m_invMasses.clear(); m_x0.clear(); m_x.clear(); m_v.clear(); m_a.clear(); m_oldX.clear(); m_lastX.clear();
    dirtyMask = 0x1f; aheadMask = 0; massDirty = true;
}
void ParticleData::setMass(unsigned int i, Real mass) {
    m_masses[i] = mass;
    m_invMasses[i] = (mass != 0.0f) ? 1.0f / mass : 0.0f;
    massDirty = true;
}

// ============================================================================================================
// Mesh topology
// ============================================================================================================
static inline uint64_t edgeKey(unsigned int a, unsigned int b) {
    return a < b ? ((uint64_t)a << 32) | b : ((uint64_t)b << 32) | a;
}

void IndexedFaceMesh::initMesh(unsigned int nPoints, unsigned int nEdges, unsigned int nFaces) {
    m_numPoints = nPoints; m_indices.clear(); m_indices.reserve((size_t)nFaces * 3); m_edges.clear(); m_edges.reserve(nEdges);
}
void IndexedFaceMesh::addFace(const unsigned int *indices) { m_indices.insert(m_indices.end(), indices, indices + 3); }
void IndexedFaceMesh::addFaces(const unsigned int *indices, unsigned int nFaces) { m_indices.insert(m_indices.end(), indices, indices + 3 * (size_t)nFaces); }

// The reference looks an undirected edge {a,b} up among the edges already incident to a, in discovery order, and creates
// it (oriented a->b, m_face[0] = current face) when absent; a later sighting overwrites m_face[1]
// (IndexedFaceMesh.cpp:146-205).  A hash map keyed on the unordered pair gives the same edge numbering.
// Edge lookup of buildNeighbors: open addressing with linear probing over a power-of-two table (the reference walks per-vertex
// edge lists, Utils/IndexedFaceMesh.cpp:118-226; only the ORDER of first occurrence matters, and that is the scan order).
// Replaces std::unordered_map: mesh construction of cfg2 0.49 s -> 0.31 s.
namespace {
struct FlatEdgeMap {
    std::vector<uint64_t> keys; std::vector<unsigned int> vals; size_t mask;
    explicit FlatEdgeMap(size_t expected) {
        size_t cap = 16; while (cap < expected * 2) cap <<= 1;
        keys.assign(cap, ~uint64_t(0)); vals.resize(cap); mask = cap - 1;
    }
    // returns the stored value; inserts `fresh` when the key is new (inserted = true)
    unsigned int findOrInsert(uint64_t key, unsigned int fresh, bool &inserted) {
        size_t h = (size_t)((key * 0x9E3779B97F4A7C15ull) >> 20) & mask;
        while (keys[h] != ~uint64_t(0)) { if (keys[h] == key) { inserted = false; return vals[h]; } h = (h + 1) & mask; }
        keys[h] = key; vals[h] = fresh; inserted = true; return fresh;
    }
};
}  // namespace

// OpenMP team of the host-side model build and of the engine's flatten.  GPU hosts expose far more hardware threads (128 here)
// than a process may actually use (measured: a 128-thread team made flatten 9x slower than the serial code, 8-16 threads 3x
// faster), so the team is capped at 8, or at PBD_B200_HOST_THREADS.
int host_threads() {
    static const int n = [] { const char *g = getenv("PBD_B200_HOST_THREADS"); const int want = g ? atoi(g) : 8; return std::max(1, std::min(want, omp_get_max_threads())); }();
    return n;
}

// Edge discovery in the reference's order (IndexedFaceMesh.cpp:118-226: faces in order, their three edges in order, an edge is
// created by the first half-edge that mentions it), computed without a sequential hash walk: sort the half-edges by (vertex
// pair, position), the first of every run creates the edge, the edge's index is the rank of that creating position.
// exclusive prefix sum of flags[0..count) into pos[0..count] (pos[count] = total), two passes over per-thread chunks
static void parallel_prefix(const unsigned char *flags, size_t count, unsigned int *pos) {
    const int T = std::max(1, host_threads());
    std::vector<size_t> chunkSum((size_t)T + 1, 0);
    #pragma omp parallel num_threads(T)
    {
        const int t = omp_get_thread_num(), nt = omp_get_num_threads();
        const size_t lo = count * (size_t)t / nt, hi = count * (size_t)(t + 1) / nt;
        size_t sum = 0;
        for (size_t i = lo; i < hi; i++) sum += flags[i];
        chunkSum[(size_t)t + 1] = sum;
        #pragma omp barrier
        #pragma omp single
        for (int k = 0; k < nt; k++) chunkSum[(size_t)k + 1] += chunkSum[k];
        size_t run = chunkSum[t];
        for (size_t i = lo; i < hi; i++) { pos[i] = (unsigned int)run; run += flags[i]; }
        if (t == nt - 1) pos[count] = (unsigned int)run;
    }
    if (count == 0) pos[0] = 0;
}

void IndexedFaceMesh::buildNeighbors() {
    m_edges.clear();
    const size_t nH = (size_t)numFaces() * 3;
    if (nH < 4096) {  // tiny meshes: the sequential walk
        FlatEdgeMap lookup((size_t)numFaces() * 3 / 2 + 16);
        m_edges.reserve((size_t)numFaces() * 3 / 2 + 16);
        for (unsigned int f = 0; f < numFaces(); f++) {
            const unsigned int *v = &m_indices[3 * (size_t)f];
            for (int j = 0; j < 3; j++) {
                const unsigned int a = v[j], b = v[(j + 1) % 3];
                bool inserted;
                const unsigned int id = lookup.findOrInsert(edgeKey(a, b), (unsigned int)m_edges.size(), inserted);
                if (inserted) { Edge e; e.m_vert = {a, b}; e.m_face = {f, 0xffffffffu}; m_edges.push_back(e); }
                else m_edges[id].m_face[1] = f;
            }
        }
    } else {
        struct Half { uint64_t key; unsigned int pos; };
        std::unique_ptr<Half[]> hbuf(new Half[nH]);  // uninitialised: filled from all threads
        Half *h = hbuf.get();
        const int threads = host_threads();
        #pragma omp parallel for schedule(static) num_threads(threads)
        for (long long p = 0; p < (long long)nH; p++) {
            const unsigned int f = (unsigned int)(p / 3), j = (unsigned int)(p % 3);
            h[p] = Half{edgeKey(m_indices[3 * (size_t)f + j], m_indices[3 * (size_t)f + (j + 1) % 3]), (unsigned int)p};
        }
        __gnu_parallel::sort(h, h + nH, [](const Half &a, const Half &b) { return a.key < b.key || (a.key == b.key && a.pos < b.pos); },
                             __gnu_parallel::default_parallel_tag(threads));
        // creating position of every run -> rank among the creating positions = edge index
        std::unique_ptr<unsigned char[]> creates(new unsigned char[nH]);
        std::unique_ptr<unsigned int[]> rank(new unsigned int[nH + 1]);
        #pragma omp parallel for schedule(static) num_threads(threads)
        for (long long k = 0; k < (long long)nH; k++) creates[k] = 0;
        #pragma omp parallel for schedule(static) num_threads(threads)
        for (long long k = 0; k < (long long)nH; k++) if (k == 0 || h[k].key != h[k - 1].key) creates[h[k].pos] = 1;
        parallel_prefix(creates.get(), nH, rank.get());
        m_edges.resize(rank[nH]);
        #pragma omp parallel for schedule(static) num_threads(threads)
        for (long long k = 0; k < (long long)nH; k++) {
            if (k != 0 && h[k].key == h[k - 1].key) continue;
            size_t last = (size_t)k;
            while (last + 1 < nH && h[last + 1].key == h[k].key) last++;  // the LAST later half-edge wins m_face[1], as in the sequential walk
            const unsigned int p = h[k].pos, f = p / 3, j = p % 3;
            Edge e; e.m_vert = {m_indices[3 * (size_t)f + j], m_indices[3 * (size_t)f + (j + 1) % 3]};
            e.m_face = {f, last == (size_t)k ? 0xffffffffu : h[last].pos / 3};
            m_edges[rank[p]] = e;
        }
    }
    int open = 0;
    #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(| : open)
    for (long long i = 0; i < (long long)m_edges.size(); i++) open |= (m_edges[i].m_face[1] == 0xffffffffu) ? 1 : 0;
    m_closed = !open;
}

void IndexedTetMesh::initMesh(unsigned int nPoints, unsigned int nEdges, unsigned int, unsigned int nTets) {
    m_numPoints = nPoints; m_tetIndices.clear(); m_tetIndices.reserve((size_t)nTets * 4); m_edges.clear(); m_edges.reserve(nEdges);
}
void IndexedTetMesh::addTet(const unsigned int *indices) { m_tetIndices.insert(m_tetIndices.end(), indices, indices + 4); }

void IndexedTetMesh::buildNeighbors() {
    static const int EP[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};  // IndexedTetMesh.cpp:77-82
    m_edges.clear();
    m_vertexTetCount.assign(m_numPoints, 0u);
    FlatEdgeMap lookup((size_t)numTets() * 2 + 16);
    for (unsigned int t = 0; t < numTets(); t++) {
        const unsigned int *v = &m_tetIndices[4 * (size_t)t];
        for (int j = 0; j < 4; j++) m_vertexTetCount[v[j]]++;
        for (int j = 0; j < 6; j++) {
            const unsigned int a = v[EP[j][0]], b = v[EP[j][1]];
            bool inserted;
            lookup.findOrInsert(edgeKey(a, b), (unsigned int)m_edges.size(), inserted);
            if (inserted) { Edge e; e.m_vert = {a, b}; m_edges.push_back(e); }
        }
    }
}

void TriangleModel::initMesh(unsigned int nPoints, unsigned int nFaces, unsigned int indexOffset, const unsigned int *indices) {
    m_indexOffset = indexOffset;
    m_particleMesh.initMesh(nPoints, nFaces * 2, nFaces);
    m_particleMesh.addFaces(indices, nFaces);
    m_particleMesh.buildNeighbors();
}
void TetModel::initMesh(unsigned int nPoints, unsigned int nTets, unsigned int indexOffset, const unsigned int *indices) {
    m_indexOffset = indexOffset;
    m_particleMesh.initMesh(nPoints, nTets * 6, nTets * 4, nTets);
    for (unsigned int i = 0; i < nTets; i++) m_particleMesh.addTet(&indices[4 * (size_t)i]);
    m_particleMesh.buildNeighbors();
}

// ============================================================================================================
// colouring
// ============================================================================================================
// Greedy first fit in insertion order (SimulationModel.cpp:1033-1094).  The reference keeps one byte map per colour and
// scans the colours in creation order; here every body carries a bit set of the colours already using it, so the first
// admissible colour is the lowest zero bit of the OR of the constraint's bodies.  Identical result.
unsigned int firstFitColouring(unsigned int numBodies, unsigned int numConstraints, const unsigned int *bodyOff,
                               const unsigned int *bodies, std::vector<unsigned int> &colour) {
    unsigned int words = 1, nColours = 0;
    std::vector<uint64_t> mask((size_t)numBodies * words, 0);
    colour.resize(numConstraints);
    for (unsigned int c = 0; c < numConstraints; c++) {
        const unsigned int *b = bodies + bodyOff[c];
        const unsigned int nb = bodyOff[c + 1] - bodyOff[c];
        unsigned int col = 0;
        bool found = false;
        for (unsigned int w = 0; w < words && !found; w++) {
            uint64_t m = 0;
            for (unsigned int k = 0; k < nb; k++) m |= mask[(size_t)b[k] * words + w];
            if (~m) { col = w * 64 + (unsigned int)__builtin_ctzll(~m); found = true; }
        }
        if (!found) {  // every colour representable so far is taken: add a word per body
            const unsigned int nw = words + 1;
            std::vector<uint64_t> m2((size_t)numBodies * nw, 0);
            for (size_t p = 0; p < numBodies; p++) for (unsigned int w = 0; w < words; w++) m2[p * nw + w] = mask[p * words + w];
            mask.swap(m2);
            col = words * 64; words = nw;
        }
        for (unsigned int k = 0; k < nb; k++) mask[(size_t)b[k] * words + col / 64] |= (uint64_t)1 << (col % 64);
        colour[c] = col;
        if (col + 1 > nColours) nColours = col + 1;
    }
    return nColours;
}

// ============================================================================================================
// SimulationModel
// ============================================================================================================
SimulationModel::SimulationModel() {}
SimulationModel::~SimulationModel() { cleanup(); }

void SimulationModel::cleanup() {
    for (auto *b : m_rigidBodies) delete b;
    m_rigidBodies.clear(); rigidBodiesDirty = true;
    for (auto *t : m_triangleModels) delete t;
    for (auto *t : m_tetModels) delete t;
    m_triangleModels.clear(); m_tetModels.clear();
    for (auto &s : m_store) { s.ids.clear(); s.bodies.clear(); s.params.clear(); }
    m_order.clear(); m_constraintGroups.clear(); m_groupsInitialized = false;
    m_particles.release();
    m_generation++;
}

void SimulationModel::reset() {
    for (auto *b : m_rigidBodies) { b->m_x = b->m_x0; b->m_q = b->m_q0; b->m_v = Vector3r(); b->m_omega = Vector3r(); }
    rigidBodiesDirty = true;
    ParticleData &pd = m_particles;
    for (unsigned int i = 0; i < pd.size(); i++) {
        pd.m_x[i] = pd.m_x0[i]; pd.m_oldX[i] = pd.m_x0[i]; pd.m_lastX[i] = pd.m_x0[i];
        pd.m_v[i] = Vector3r(); pd.m_a[i] = Vector3r();
    }
    pd.aheadMask = 0; pd.dirtyMask = 0x1f;
}

ConstraintView SimulationModel::getConstraint(unsigned int i) const {
    const ConstraintRef r = m_order[i];
    const int nb = pbd_num_bodies(r.type), np = pbd_num_params(r.type);
    ConstraintView v;
    v.type = r.type; v.numberOfBodies = (unsigned int)nb; v.numParams = (unsigned int)np;
    v.m_bodies = &m_store[r.type].bodies[(size_t)r.local * nb];
    v.params = &m_store[r.type].params[(size_t)r.local * np];
    return v;
}

void SimulationModel::addTriangleModel(unsigned int nPoints, unsigned int nFaces, const Vector3r *points, const unsigned int *indices) {
    TriangleModel *tm = new TriangleModel();
    m_triangleModels.push_back(tm);
    const unsigned int startIndex = m_particles.size();
    m_particles.reserve(startIndex + nPoints);
    m_particles.addVertices(points, nPoints);
    tm->initMesh(nPoints, nFaces, startIndex, indices);
}

static inline Vector3r rotTrans(const Matrix3r &R, const Vector3r &p, const Vector3r &t) {
    return Vector3r(R(0, 0) * p[0] + R(0, 1) * p[1] + R(0, 2) * p[2] + t[0], R(1, 0) * p[0] + R(1, 1) * p[1] + R(1, 2) * p[2] + t[1],
                    R(2, 0) * p[0] + R(2, 1) * p[1] + R(2, 2) * p[2] + t[2]);
}

// SimulationModel.cpp:831-901: grid point (i,j) -> index i*width+j; cell (i,j) split along alternating diagonals.
void SimulationModel::addRegularTriangleModel(int width, int height, const Vector3r &translation, const Matrix3r &rotation, const Vector2r &scale) {
    const Real dy = scale[1] / (Real)(height - 1);
    const Real dx = scale[0] / (Real)(width - 1);
    std::vector<Vector3r> points((size_t)width * height);
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (int i = 0; i < height; i++)
        for (int j = 0; j < width; j++) points[(size_t)i * width + j] = rotTrans(rotation, Vector3r(dx * j, dy * i, 0.0f), translation);
    PodVector<unsigned int> indices((size_t)6 * (height - 1) * (width - 1));
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (int i = 0; i < height - 1; i++)
        for (int j = 0; j < width - 1; j++) {
            const unsigned int helper = (i % 2 == j % 2) ? 1u : 0u;
            const unsigned int a = i * width + j, b = (i + 1) * width + j;
            const unsigned int tri[6] = {a, a + 1, b + helper, b + 1, b, a + 1 - helper};
            std::memcpy(&indices[6 * ((size_t)i * (width - 1) + j)], tri, sizeof(tri));
        }
    const size_t modelIndex = m_triangleModels.size();
    addTriangleModel((unsigned int)points.size(), (unsigned int)indices.size() / 3, points.data(), indices.data());
    const unsigned int offset = m_triangleModels[modelIndex]->getIndexOffset();
    for (unsigned int i = offset; i < offset + (unsigned int)points.size(); i++) m_particles.setMass(i, 1.0f);  // SimulationModel.cpp:897-900
}

void SimulationModel::addTetModel(unsigned int nPoints, unsigned int nTets, const Vector3r *points, const unsigned int *indices) {
    TetModel *tm = new TetModel();
    m_tetModels.push_back(tm);
    const unsigned int startIndex = m_particles.size();
    m_particles.reserve(startIndex + nPoints);
    m_particles.addVertices(points, nPoints);
    tm->initMesh(nPoints, nTets, startIndex, indices);
}

// SimulationModel.cpp:921-1005: point (i,j,k) -> i*height*depth + j*depth + k, five tets per cell, parity flipped so that
// neighbouring cells share faces.
void SimulationModel::addRegularTetModel(int width, int height, int depth, const Vector3r &translation, const Matrix3r &rotation, const Vector3r &scale) {
    const Real dx = scale[0] / (Real)(width - 1), dy = scale[1] / (Real)(height - 1), dz = scale[2] / (Real)(depth - 1);
    const Vector3r t((Real)(translation[0] - 0.5 * scale[0]), (Real)(translation[1] - 0.5 * scale[1]), (Real)(translation[2] - 0.5 * scale[2]));
    std::vector<Vector3r> points((size_t)width * height * depth);
    for (int i = 0; i < width; i++)
        for (int j = 0; j < height; j++)
            for (int k = 0; k < depth; k++) points[(size_t)i * height * depth + (size_t)j * depth + k] = rotTrans(rotation, Vector3r(dx * i, dy * j, dz * k), t);
    std::vector<unsigned int> indices;
    indices.reserve((size_t)20 * (width - 1) * (height - 1) * (depth - 1));
    for (int i = 0; i < width - 1; i++)
        for (int j = 0; j < height - 1; j++)
            for (int k = 0; k < depth - 1; k++) {
                // cell corners: 0=(i,j,k) 1=(i,j,k+1) 3=(i+1,j,k) 2=(i+1,j,k+1) 4=(i,j+1,k) 5=(i,j+1,k+1) 7=(i+1,j+1,k) 6=(i+1,j+1,k+1)
                unsigned int p[8];
                p[0] = i * height * depth + j * depth + k; p[1] = p[0] + 1;
                p[3] = (i + 1) * height * depth + j * depth + k; p[2] = p[3] + 1;
                p[7] = (i + 1) * height * depth + (j + 1) * depth + k; p[6] = p[7] + 1;
                p[4] = i * height * depth + (j + 1) * depth + k; p[5] = p[4] + 1;
                static const int odd[20] = {2, 1, 6, 3, 6, 3, 4, 7, 4, 1, 6, 5, 3, 1, 4, 0, 6, 1, 4, 3};
                static const int even[20] = {0, 2, 5, 1, 7, 2, 0, 3, 5, 2, 7, 6, 7, 0, 5, 4, 0, 2, 7, 5};
                const int *pat = ((i + j + k) % 2 == 1) ? odd : even;
                for (int q = 0; q < 20; q++) indices.push_back(p[pat[q]]);
            }
    const size_t modelIndex = m_tetModels.size();
    addTetModel((unsigned int)points.size(), (unsigned int)indices.size() / 4, points.data(), indices.data());
    const unsigned int offset = m_tetModels[modelIndex]->getIndexOffset();
    for (unsigned int i = offset; i < offset + (unsigned int)points.size(); i++) m_particles.setMass(i, 1.0f);
}

void RigidBody::initBody(Real mass, const Vector3r &x, const Vector3r &inertiaTensor, const Quaternionr &rotation) {
    m_mass = mass; m_invMass = (mass != 0.0f) ? 1.0f / mass : 0.0f;  // RigidBody::setMass (RigidBody.h:277-284)
    m_x = m_x0 = x; m_v = Vector3r(); m_omega = Vector3r();
    m_inertiaTensor = inertiaTensor; m_q = m_q0 = rotation;
}

// world -> body space of a point, R(q)^T (p - x), evaluated in double
static void toLocal(const RigidBody &b, const double p[3], Real out[3]) {
    const double w = b.m_q.w, x = b.m_q.x, y = b.m_q.y, z = b.m_q.z;
    const double R[3][3] = {{1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)},
                            {2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)},
                            {2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)}};
    const double d[3] = {p[0] - b.m_x[0], p[1] - b.m_x[1], p[2] - b.m_x[2]};
    for (int c = 0; c < 3; c++) out[c] = (Real)(R[0][c] * d[0] + R[1][c] * d[1] + R[2][c] * d[2]);
}

// BallJoint::initConstraint + init_BallJoint (Constraints.cpp:54-70, PositionBasedRigidBodyDynamics.cpp:160-186):
// jointInfo = [connector in body 0 | connector in body 1 | global | global]
bool SimulationModel::addBallJoint(unsigned int rbIndex1, unsigned int rbIndex2, const Vector3r &pos) {
    if (rbIndex1 >= m_rigidBodies.size() || rbIndex2 >= m_rigidBodies.size()) return false;
    const double p[3] = {pos[0], pos[1], pos[2]};
    Real info[12];
    toLocal(*m_rigidBodies[rbIndex1], p, info); toLocal(*m_rigidBodies[rbIndex2], p, info + 3);
    for (int k = 0; k < 3; k++) info[6 + k] = info[9 + k] = pos[k];
    const unsigned int b[2] = {rbIndex1, rbIndex2};
    return pushConstraint(PBD_BALLJOINT, b, info, true);
}
// RigidBodyParticleBallJoint::initConstraint (Constraints.cpp:925-938): connector = the particle's CURRENT position
bool SimulationModel::addRigidBodyParticleBallJoint(unsigned int rbIndex, unsigned int particleIndex) {
    if (rbIndex >= m_rigidBodies.size() || particleIndex >= m_particles.size()) return false;
    const Vector3r &x = static_cast<const ParticleData &>(m_particles).getPosition(particleIndex);
    const double p[3] = {x[0], x[1], x[2]};
    Real info[6];
    toLocal(*m_rigidBodies[rbIndex], p, info);
    for (int k = 0; k < 3; k++) info[3 + k] = x[k];
    const unsigned int b[2] = {rbIndex, particleIndex};
    return pushConstraint(PBD_RB_PARTICLE_BALLJOINT, b, info, true);
}

void SimulationModel::initConstraintGroups() {
    if (m_groupsInitialized) return;
    const unsigned int N = numConstraints();
    std::vector<unsigned int> off(N + 1, 0), bodies;
    bodies.reserve((size_t)N * 4);
    for (unsigned int c = 0; c < N; c++) {
        const ConstraintView v = getConstraint(c);
        bodies.insert(bodies.end(), v.m_bodies, v.m_bodies + v.numberOfBodies);
        off[c + 1] = (unsigned int)bodies.size();
    }
    std::vector<unsigned int> colour;
    // rigid-body and particle indices share one index space without offset (SimulationModel.cpp:1041,1058,1070)
    const unsigned int nColours = firstFitColouring(m_particles.size() + (unsigned int)m_rigidBodies.size(), N, off.data(), bodies.data(), colour);
    m_constraintGroups.assign(nColours, std::vector<unsigned int>());
    for (unsigned int c = 0; c < N; c++) m_constraintGroups[colour[c]].push_back(c);
    m_groupsInitialized = true;
}

// ------------------------------------------------------------------------------------------------------------
// constraint factories.  Rest-state data is evaluated in double from the fp32 rest positions and rounded once.
// ------------------------------------------------------------------------------------------------------------
// The geometry columns of a constraint of `type` on `bodies` from the rest positions (and, ShapeMatching, the inverse masses) into its
// parameter row, and whether the constraint class's initConstraint accepts them: rest_geometry.cuh, the description the device derivation
// of a batch's per-replica rest shapes (pbd_set_replica_rest_positions) shares.
static bool restParams(const ParticleData &pd, int type, const unsigned int *bodies, Real *params) {
    float4 x[4];
    for (int k = 0; k < pbdk::type_shape(type).nBodies; k++) {
        const Vector3r &p = pd.m_x0[bodies[k]];
        x[k] = make_float4(p[0], p[1], p[2], pd.m_invMasses[bodies[k]]);
    }
    return pbdk::rest_geometry(type, x, params + pbdk::geo_first(type));
}

// the batch builders know how many constraints they are about to add: one allocation instead of repeated vector growth
// (cfg2: addBendingConstraints 0.48 s -> 0.30 s)
void SimulationModel::reserveConstraints(int type, size_t count) {
    TypeStore &s = m_store[type];
    s.ids.reserve(s.ids.size() + count);
    s.bodies.reserve(s.bodies.size() + count * (size_t)pbd_num_bodies(type));
    s.params.reserve(s.params.size() + count * (size_t)pbd_num_params(type));
    m_order.reserve(m_order.size() + count);
}

bool SimulationModel::pushConstraint(int type, const unsigned int *bodies, const Real *params, bool ok) {
    if (!ok) return false;  // reference: constraint deleted, nothing added, groups untouched (SimulationModel.cpp:565-575)
    TypeStore &s = m_store[type];
    const int nb = pbd_num_bodies(type), np = pbd_num_params(type);
    s.ids.push_back((unsigned int)m_order.size());
    s.bodies.insert(s.bodies.end(), bodies, bodies + nb);
    s.params.insert(s.params.end(), params, params + np);
    m_order.push_back({type, (unsigned int)s.ids.size() - 1});
    m_groupsInitialized = false;
    m_generation++;
    return true;
}

// Order-preserving bulk construction (SURVEY.md 8 f-3, host part): candidate i of `count` is computed by fill(i, bodies, params) ->
// bool (the constraint class's initConstraint result), independently of the others and therefore in parallel; the accepted ones
// are appended in candidate order, i.e. exactly as the reference's sequential add loop would have inserted them.
template <class A, class F>
static void push_bulk(TypeStore &s, PodVector<ConstraintRef> &order, int type, size_t count, A &&accept, F &&fill) {
    const int nb = pbd_num_bodies(type), np = pbd_num_params(type);
    std::unique_ptr<unsigned char[]> flag(new unsigned char[count + 1]);
    std::unique_ptr<unsigned int[]> pos(new unsigned int[count + 1]);
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (long long i = 0; i < (long long)count; i++) flag[i] = accept((size_t)i) ? 1 : 0;  // cheap topological test
    parallel_prefix(flag.get(), count, pos.get());
    const size_t add = pos[count], base = s.ids.size(), obase = order.size();
    s.ids.resize(base + add); s.bodies.resize((base + add) * nb); s.params.resize((base + add) * np); order.resize(obase + add);  // uninitialised: filled below
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (long long i = 0; i < (long long)count; i++) {
        if (!flag[i]) continue;
        const size_t k = pos[i];
        s.ids[base + k] = (unsigned int)(obase + k);
        fill((size_t)i, &s.bodies[(base + k) * nb], &s.params[(base + k) * np]);  // straight into the store: no staging copy
        order[obase + k] = ConstraintRef{type, (unsigned int)(base + k)};
    }
}

// DistanceConstraint::initConstraint (Constraints.cpp:1166-1181): rest length from x0
bool SimulationModel::addDistanceConstraint(unsigned int p1, unsigned int p2, Real stiffness) {
    const unsigned int b[2] = {p1, p2};
    Real p[2] = {0, stiffness};
    return pushConstraint(PBD_DISTANCE, b, p, restParams(m_particles, PBD_DISTANCE, b, p));
}
bool SimulationModel::addDistanceConstraint_XPBD(unsigned int p1, unsigned int p2, Real stiffness) {  // Constraints.cpp:1211-1227
    const unsigned int b[2] = {p1, p2};
    Real p[2] = {0, stiffness};
    return pushConstraint(PBD_DISTANCE_XPBD, b, p, restParams(m_particles, PBD_DISTANCE_XPBD, b, p));
}

// DihedralConstraint::initConstraint (Constraints.cpp:1264-1300)
bool SimulationModel::addDihedralConstraint(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stiffness) {
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[2] = {0, stiffness};
    return pushConstraint(PBD_DIHEDRAL, b, p, restParams(m_particles, PBD_DIHEDRAL, b, p));
}

// init_IsometricBendingConstraint (PositionBasedDynamics.cpp:145-183): Q = coef K K^T over x = {p2, p3, p0, p1}
bool SimulationModel::addIsometricBendingConstraint(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stiffness) {
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[17]; p[0] = stiffness;
    return pushConstraint(PBD_ISOBENDING, b, p, restParams(m_particles, PBD_ISOBENDING, b, p));
}
bool SimulationModel::addIsometricBendingConstraint_XPBD(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stiffness) {
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[17]; p[0] = stiffness;
    return pushConstraint(PBD_ISOBENDING_XPBD, b, p, restParams(m_particles, PBD_ISOBENDING_XPBD, b, p));
}

// init_FEMTriangleConstraint (PositionBasedDynamics.cpp:808-841)
bool SimulationModel::addFEMTriangleConstraint(unsigned int i1, unsigned int i2, unsigned int i3, Real xx, Real yy, Real xy, Real nuxy, Real nuyx) {
    const unsigned int b[3] = {i1, i2, i3};
    Real p[10] = {0, 0, 0, 0, 0, xx, yy, xy, nuxy, nuyx};
    return pushConstraint(PBD_FEMTRIANGLE, b, p, restParams(m_particles, PBD_FEMTRIANGLE, b, p));
}

// StrainTriangleConstraint::initConstraint (Constraints.cpp:1544-1569: the rest triangle is taken in the x-z plane)
// + init_StrainTriangleConstraint (PositionBasedDynamics.cpp:562-581)
bool SimulationModel::addStrainTriangleConstraint(unsigned int i1, unsigned int i2, unsigned int i3, Real xx, Real yy, Real xy, bool normalizeStretch, bool normalizeShear) {
    const unsigned int b[3] = {i1, i2, i3};
    Real p[9] = {0, 0, 0, 0, xx, yy, xy, normalizeStretch ? 1.0f : 0.0f, normalizeShear ? 1.0f : 0.0f};
    return pushConstraint(PBD_STRAINTRIANGLE, b, p, restParams(m_particles, PBD_STRAINTRIANGLE, b, p));
}

bool SimulationModel::addVolumeConstraint(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stiffness) {  // Constraints.cpp:1617-1635
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[2] = {0, stiffness};
    return pushConstraint(PBD_VOLUME, b, p, restParams(m_particles, PBD_VOLUME, b, p));
}
bool SimulationModel::addVolumeConstraint_XPBD(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stiffness) {  // Constraints.cpp:1683-1702
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[2] = {0, stiffness};
    return pushConstraint(PBD_VOLUME_XPBD, b, p, restParams(m_particles, PBD_VOLUME_XPBD, b, p));
}

// init_FEMTetraConstraint (PositionBasedDynamics.cpp:933-955): columns p0-p3, p1-p3, p2-p3
bool SimulationModel::addFEMTetConstraint(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stiffness, Real poissonRatio) {
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[12]; p[10] = stiffness; p[11] = poissonRatio;
    return pushConstraint(PBD_FEMTET, b, p, restParams(m_particles, PBD_FEMTET, b, p));
}
bool SimulationModel::addFEMTetConstraint_XPBD(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stiffness, Real poissonRatio) {
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[12]; p[10] = stiffness; p[11] = poissonRatio;
    return pushConstraint(PBD_FEMTET_XPBD, b, p, restParams(m_particles, PBD_FEMTET_XPBD, b, p));
}

// init_StrainTetraConstraint (PositionBasedDynamics.cpp:691-710): columns p1-p0, p2-p0, p3-p0
bool SimulationModel::addStrainTetConstraint(unsigned int i1, unsigned int i2, unsigned int i3, unsigned int i4, Real stretchStiffness, Real shearStiffness,
                                             bool normalizeStretch, bool normalizeShear) {
    const unsigned int b[4] = {i1, i2, i3, i4};
    Real p[13];
    p[9] = stretchStiffness; p[10] = shearStiffness; p[11] = normalizeStretch ? 1.0f : 0.0f; p[12] = normalizeShear ? 1.0f : 0.0f;
    return pushConstraint(PBD_STRAINTET, b, p, restParams(m_particles, PBD_STRAINTET, b, p));
}

// ShapeMatchingConstraint::initConstraint (Constraints.cpp:1985-2001) + init_ShapeMatchingConstraint
// (PositionBasedDynamics.cpp:479-497): rest positions and inverse masses are frozen into the constraint.
bool SimulationModel::addShapeMatchingConstraint(unsigned int numberOfParticles, const unsigned int particleIndices[], const unsigned int numClusters[], Real stiffness) {
    if (numberOfParticles != 4) return false;  // the accelerated path covers the tetrahedral clusters of addSolidConstraints
    Real p[24];
    p[0] = stiffness;
    for (int i = 0; i < 4; i++) p[20 + i] = (Real)numClusters[i];
    return pushConstraint(PBD_SHAPEMATCHING, particleIndices, p, restParams(m_particles, PBD_SHAPEMATCHING, particleIndices, p));
}

// SimulationModel::addClothConstraints (SimulationModel.cpp:1125-1184)
void SimulationModel::addClothConstraints(const TriangleModel *tm, unsigned int clothMethod, Real distanceStiffness, Real xxStiffness, Real yyStiffness,
                                          Real xyStiffness, Real xyPoissonRatio, Real yxPoissonRatio, bool normalizeStretch, bool normalizeShear) {
    const unsigned int offset = tm->getIndexOffset();
    const IndexedFaceMesh &mesh = tm->getParticleMesh();
    if (clothMethod == 1 || clothMethod == 4) {
        const int type = clothMethod == 1 ? PBD_DISTANCE : PBD_DISTANCE_XPBD;
        const IndexedFaceMesh::Edges &edges = mesh.getEdges();
        const ParticleData &pd = m_particles;
        push_bulk(m_store[type], m_order, type, edges.size(), [](size_t) { return true; }, [&](size_t i, unsigned int *b, Real *p) {
            b[0] = edges[i].m_vert[0] + offset; b[1] = edges[i].m_vert[1] + offset;
            restParams(pd, type, b, p); p[1] = distanceStiffness;  // DistanceConstraint::initConstraint
        });
        if (!edges.empty()) { m_groupsInitialized = false; m_generation++; }
    } else if (clothMethod == 2 || clothMethod == 3) {
        const unsigned int *tris = mesh.getFaces().data();
        reserveConstraints(clothMethod == 2 ? PBD_FEMTRIANGLE : PBD_STRAINTRIANGLE, mesh.numFaces());
        for (unsigned int i = 0; i < mesh.numFaces(); i++) {
            const unsigned int v1 = tris[3 * i] + offset, v2 = tris[3 * i + 1] + offset, v3 = tris[3 * i + 2] + offset;
            if (clothMethod == 2) addFEMTriangleConstraint(v1, v2, v3, xxStiffness, yyStiffness, xyStiffness, xyPoissonRatio, yxPoissonRatio);
            else addStrainTriangleConstraint(v1, v2, v3, xxStiffness, yyStiffness, xyStiffness, normalizeStretch, normalizeShear);
        }
    }
}

// SimulationModel::addBendingConstraints (SimulationModel.cpp:1186-1240): one constraint per interior edge,
// bodies = (opposite vertex of face 0, opposite vertex of face 1, edge v0, edge v1)
void SimulationModel::addBendingConstraints(const TriangleModel *tm, unsigned int bendingMethod, Real stiffness) {
    if (bendingMethod < 1 || bendingMethod > 3) return;
    const unsigned int offset = tm->getIndexOffset();
    const IndexedFaceMesh &mesh = tm->getParticleMesh();
    const unsigned int *tris = mesh.getFaces().data();
    if (bendingMethod == 2 || bendingMethod == 3) {
        const int type = bendingMethod == 2 ? PBD_ISOBENDING : PBD_ISOBENDING_XPBD;
        const IndexedFaceMesh::Edges &edges = mesh.getEdges();
        const ParticleData &pd = m_particles;
        const size_t before = m_order.size();
        auto opposite = [&](const IndexedFaceMesh::Edge &e, int &point1, int &point2) {
            const unsigned int tri1 = e.m_face[0], tri2 = e.m_face[1];
            point1 = point2 = -1;
            if (tri1 == 0xffffffffu || tri2 == 0xffffffffu) return false;
            const unsigned int a1 = e.m_vert[0], a2 = e.m_vert[1];
            for (int j = 0; j < 3; j++) if (tris[3 * tri1 + j] != a1 && tris[3 * tri1 + j] != a2) { point1 = (int)tris[3 * tri1 + j]; break; }
            for (int j = 0; j < 3; j++) if (tris[3 * tri2 + j] != a1 && tris[3 * tri2 + j] != a2) { point2 = (int)tris[3 * tri2 + j]; break; }
            return point1 != -1 && point2 != -1;
        };
        push_bulk(m_store[type], m_order, type, edges.size(),
                  [&](size_t i) { int p1, p2; return opposite(edges[i], p1, p2); },
                  [&](size_t i, unsigned int *b, Real *p) {
                      int point1, point2;
                      opposite(edges[i], point1, point2);
                      b[0] = point1 + offset; b[1] = point2 + offset; b[2] = edges[i].m_vert[0] + offset; b[3] = edges[i].m_vert[1] + offset;
                      p[0] = stiffness;
                      restParams(pd, type, b, p);
                  });
        if (m_order.size() != before) { m_groupsInitialized = false; m_generation++; }
        return;
    }
    reserveConstraints(PBD_DIHEDRAL, mesh.getEdges().size());
    for (const IndexedFaceMesh::Edge &e : mesh.getEdges()) {
        const unsigned int tri1 = e.m_face[0], tri2 = e.m_face[1];
        if (tri1 == 0xffffffffu || tri2 == 0xffffffffu) continue;
        const unsigned int a1 = e.m_vert[0], a2 = e.m_vert[1];
        int point1 = -1, point2 = -1;
        for (int j = 0; j < 3; j++) if (tris[3 * tri1 + j] != a1 && tris[3 * tri1 + j] != a2) { point1 = (int)tris[3 * tri1 + j]; break; }
        for (int j = 0; j < 3; j++) if (tris[3 * tri2 + j] != a1 && tris[3 * tri2 + j] != a2) { point2 = (int)tris[3 * tri2 + j]; break; }
        if (point1 == -1 || point2 == -1) continue;
        const unsigned int v1 = point1 + offset, v2 = point2 + offset, v3 = a1 + offset, v4 = a2 + offset;
        if (bendingMethod == 1) addDihedralConstraint(v1, v2, v3, v4, stiffness);
        else if (bendingMethod == 2) addIsometricBendingConstraint(v1, v2, v3, v4, stiffness);
        else addIsometricBendingConstraint_XPBD(v1, v2, v3, v4, stiffness);
    }
}

// SimulationModel::addSolidConstraints (SimulationModel.cpp:1242-1349)
void SimulationModel::addSolidConstraints(const TetModel *tm, unsigned int solidMethod, Real stiffness, Real poissonRatio, Real volumeStiffness,
                                          bool normalizeStretch, bool /*normalizeShear*/) {
    const IndexedTetMesh &mesh = tm->getParticleMesh();
    const unsigned int nTets = mesh.numTets();
    const unsigned int *tets = mesh.getTets().data();
    const unsigned int offset = tm->getIndexOffset();
    if (solidMethod == 1 || solidMethod == 6) {
        for (const IndexedTetMesh::Edge &e : mesh.getEdges()) {
            if (solidMethod == 1) addDistanceConstraint(e.m_vert[0] + offset, e.m_vert[1] + offset, stiffness);
            else addDistanceConstraint_XPBD(e.m_vert[0] + offset, e.m_vert[1] + offset, stiffness);
        }
        for (unsigned int i = 0; i < nTets; i++) {
            if (solidMethod == 1) addVolumeConstraint(tets[4 * i] + offset, tets[4 * i + 1] + offset, tets[4 * i + 2] + offset, tets[4 * i + 3] + offset, volumeStiffness);
            else addVolumeConstraint_XPBD(tets[4 * i] + offset, tets[4 * i + 1] + offset, tets[4 * i + 2] + offset, tets[4 * i + 3] + offset, volumeStiffness);
        }
    } else if (solidMethod == 5) {
        const std::vector<unsigned int> &vt = mesh.getVertexTetCounts();
        for (unsigned int i = 0; i < nTets; i++) {
            const unsigned int v[4] = {tets[4 * i] + offset, tets[4 * i + 1] + offset, tets[4 * i + 2] + offset, tets[4 * i + 3] + offset};
            // divide the correction by the number of clusters containing the vertex (SimulationModel.cpp:1322-1325)
            const unsigned int nc[4] = {vt[v[0] - offset], vt[v[1] - offset], vt[v[2] - offset], vt[v[3] - offset]};
            addShapeMatchingConstraint(4, v, nc, stiffness);
        }
    } else if (solidMethod >= 2 && solidMethod <= 4) {
        for (unsigned int i = 0; i < nTets; i++) {
            const unsigned int v1 = tets[4 * i] + offset, v2 = tets[4 * i + 1] + offset, v3 = tets[4 * i + 2] + offset, v4 = tets[4 * i + 3] + offset;
            if (solidMethod == 2) addFEMTetConstraint(v1, v2, v3, v4, stiffness, poissonRatio);
            else if (solidMethod == 3) addFEMTetConstraint_XPBD(v1, v2, v3, v4, stiffness, poissonRatio);
            else addStrainTetConstraint(v1, v2, v3, v4, stiffness, stiffness, normalizeStretch, normalizeStretch);  // :1308 passes normalizeStretch twice
        }
    }
}

void SimulationModel::setParam(int type, int slot, Real val) {
    TypeStore &s = m_store[type];
    const int np = pbd_num_params(type);
    for (size_t i = 0; i < s.ids.size(); i++) s.params[i * np + slot] = val;
    if (!s.ids.empty()) m_generation++;
}
void SimulationModel::setClothStiffness(Real v) { setParam(PBD_DISTANCE, 1, v); setParam(PBD_DISTANCE_XPBD, 1, v); }
void SimulationModel::setClothStiffnessXX(Real v) { setParam(PBD_FEMTRIANGLE, 5, v); setParam(PBD_STRAINTRIANGLE, 4, v); }
// SimulationModel.cpp:1365-1377: the YY and XY setters of the reference write m_xxStiffness; kept so that identical
// parameter scripts give identical scenes.
void SimulationModel::setClothStiffnessYY(Real v) { setParam(PBD_FEMTRIANGLE, 5, v); setParam(PBD_STRAINTRIANGLE, 4, v); }
void SimulationModel::setClothStiffnessXY(Real v) { setParam(PBD_FEMTRIANGLE, 5, v); setParam(PBD_STRAINTRIANGLE, 4, v); }
void SimulationModel::setClothPoissonRatioXY(Real v) { setParam(PBD_FEMTRIANGLE, 8, v); }
void SimulationModel::setClothPoissonRatioYX(Real v) { setParam(PBD_FEMTRIANGLE, 9, v); }
void SimulationModel::setClothBendingStiffness(Real v) { setParam(PBD_DIHEDRAL, 1, v); setParam(PBD_ISOBENDING, 0, v); setParam(PBD_ISOBENDING_XPBD, 0, v); }
void SimulationModel::setClothNormalizeStretch(bool v) { setParam(PBD_STRAINTRIANGLE, 7, v ? 1.0f : 0.0f); }
void SimulationModel::setClothNormalizeShear(bool v) { setParam(PBD_STRAINTRIANGLE, 8, v ? 1.0f : 0.0f); }
void SimulationModel::setSolidStiffness(Real v) {
    setParam(PBD_FEMTET, 10, v); setParam(PBD_FEMTET_XPBD, 10, v); setParam(PBD_STRAINTET, 9, v); setParam(PBD_STRAINTET, 10, v);
    setParam(PBD_SHAPEMATCHING, 0, v);
}
void SimulationModel::setSolidPoissonRatio(Real v) { setParam(PBD_FEMTET, 11, v); setParam(PBD_FEMTET_XPBD, 11, v); }
void SimulationModel::setSolidVolumeStiffness(Real v) { setParam(PBD_VOLUME, 1, v); setParam(PBD_VOLUME_XPBD, 1, v); }
void SimulationModel::setSolidNormalizeStretch(bool v) { setParam(PBD_STRAINTET, 11, v ? 1.0f : 0.0f); }
void SimulationModel::setSolidNormalizeShear(bool v) { setParam(PBD_STRAINTET, 12, v ? 1.0f : 0.0f); }

// ============================================================================================================
// TimeStepController
// ============================================================================================================
TimeStepController::TimeStepController(int device, void *stream) {
    if (pbd_create(device, stream, &m_engine) != 0) { m_engine = nullptr; m_error = pbd_last_error(); }
}
TimeStepController::~TimeStepController() { if (m_engine) pbd_destroy(m_engine); }

bool TimeStepController::fail(const char *what) { m_error = std::string(what) + ": " + pbd_last_error(); return false; }

void TimeStepController::reset() {}

unsigned int TimeStepController::getValueUInt(int id) const {
    switch (id) { case NUM_SUB_STEPS: return m_subSteps; case MAX_ITERATIONS: return m_maxIterations; case MAX_ITERATIONS_V: return m_maxIterationsV; default: return 0; }
}
bool TimeStepController::setValueUInt(int id, unsigned int v) {
    switch (id) {
    case NUM_SUB_STEPS: if (v < 1) return false; m_subSteps = v; return true;          // min 1 (TimeStepController.cpp:50)
    case MAX_ITERATIONS: if (v < 1) return false; m_maxIterations = v; return true;    // min 1 (:55)
    case MAX_ITERATIONS_V: m_maxIterationsV = v; return true;                          // velocity constraints: no-ops for particle constraints
    default: return false;
    }
}
bool TimeStepController::setValueInt(int id, int v) {
    if (id != VELOCITY_UPDATE_METHOD || (v != 0 && v != 1)) return false;
    m_velocityUpdateMethod = v; return true;
}

bool TimeStepController::uploadModel(SimulationModel &model) {
    static const bool verbose = getenv("PBD_B200_VERBOSE") != nullptr;
    double tPrev = omp_get_wtime();
    auto lap = [&](const char *what) { if (verbose) { const double t = omp_get_wtime(); fprintf(stderr, "[pbd_b200] upload:  %-34s %.3f s\n", what, t - tPrev); tPrev = t; } };
    ParticleData &pd = model.getParticles();
    const unsigned int n = pd.size();
    const bool rebind = (m_boundModel != &model) || (m_boundParticles != n);
    if (rebind) {
        if (pbd_set_particles(m_engine, n, n ? &pd.m_x[0][0] : nullptr, n ? &pd.m_x0[0][0] : nullptr, n ? &pd.m_v[0][0] : nullptr, pd.m_masses.data())) return fail("pbd_set_particles");
        if (n) {
            if (pbd_set_attr(m_engine, PBD_ATTR_OLDX, &pd.m_oldX[0][0])) return fail("pbd_set_attr");
            if (pbd_set_attr(m_engine, PBD_ATTR_LASTX, &pd.m_lastX[0][0])) return fail("pbd_set_attr");
        }
        pd.dirtyMask = 0; pd.massDirty = false; pd.aheadMask = 0;
        m_boundParticles = n; m_boundGeneration = 0;
    } else if (n) {
        if (pd.massDirty) { if (pbd_set_masses(m_engine, pd.m_masses.data())) return fail("pbd_set_masses"); pd.massDirty = false; }
        const std::vector<Vector3r> *src[5] = {&pd.m_x, &pd.m_v, &pd.m_x0, &pd.m_oldX, &pd.m_lastX};
        for (int a = 0; a < 5; a++)
            if ((pd.dirtyMask >> a) & 1u) { if (pbd_set_attr(m_engine, a, &(*src[a])[0][0])) return fail("pbd_set_attr"); }
        pd.dirtyMask = 0;
    }
    if (rebind) lap("particles");
    SimulationModel::RigidBodyVector &rbs = model.getRigidBodies();
    if (rebind || model.rigidBodiesDirty || rbs.size() != m_boundRigidBodies) {
        const unsigned int nr = (unsigned int)rbs.size();
        std::vector<float> mass(nr), x(3 * nr), q(4 * nr), I(3 * nr), v(3 * nr), w(3 * nr);
        for (unsigned int i = 0; i < nr; i++) {
            const RigidBody &b = *rbs[i];
            mass[i] = b.m_mass;
            for (int k = 0; k < 3; k++) { x[3 * i + k] = b.m_x[k]; I[3 * i + k] = b.m_inertiaTensor[k]; v[3 * i + k] = b.m_v[k]; w[3 * i + k] = b.m_omega[k]; }
            q[4 * i] = b.m_q.w; q[4 * i + 1] = b.m_q.x; q[4 * i + 2] = b.m_q.y; q[4 * i + 3] = b.m_q.z;
        }
        if (pbd_set_rigid_bodies(m_engine, nr, mass.data(), x.data(), q.data(), I.data(), v.data(), w.data())) return fail("pbd_set_rigid_bodies");
        if (nr != m_boundRigidBodies) m_boundGeneration = 0;  // joints reference the body arrays: re-send the constraints
        m_boundRigidBodies = nr; model.rigidBodiesDirty = false;
    }
    if (rebind || m_boundGeneration != model.constraintGeneration()) {
        if (pbd_clear_constraints(m_engine)) return fail("pbd_clear_constraints");
        for (int t = 0; t < PBD_NUM_TYPES; t++) {
            const TypeStore &s = model.store(t);
            if (s.ids.empty()) continue;
            if (pbd_add_constraints(m_engine, t, (unsigned int)s.ids.size(), s.bodies.data(), s.params.data(), s.ids.data())) return fail("pbd_add_constraints");
        }
        // Colour groups (TimeStepController.cpp:256 -> SimulationModel::initConstraintGroups).  When the model has not been coloured yet the
        // engine does it on the GPU (pbd_color_first_fit_device: the same greedy first fit, identical groups) and the result is mirrored
        // into the model, so getConstraintGroups() shows what is simulated; the host colouring is the fallback.
        lap("constraints (pbd_add_constraints)");
        bool coloured = false;
        if (!model.m_groupsInitialized && model.numConstraints() > 0 && pbd_color_first_fit_device(m_engine, nullptr, nullptr) == 0) {
            unsigned int ng = 0;
            if (pbd_get_num_groups(m_engine, &ng) == 0) {
                std::vector<unsigned int> off(ng + 1), ids(model.numConstraints());
                if (pbd_get_groups(m_engine, off.data(), ids.data()) == 0) {
                    SimulationModel::ConstraintGroupVector &groups = model.getConstraintGroups();
                    groups.assign(ng, std::vector<unsigned int>());
                    #pragma omp parallel for schedule(dynamic, 1) num_threads(host_threads())
                    for (long long g = 0; g < (long long)ng; g++) groups[g].assign(ids.begin() + off[g], ids.begin() + off[g + 1]);
                    model.m_groupsInitialized = true;
                    coloured = true;
                }
            }
        }
        if (!coloured) {
            model.initConstraintGroups();
            const SimulationModel::ConstraintGroupVector &groups = model.getConstraintGroups();
            std::vector<unsigned int> off(groups.size() + 1, 0), ids;
            ids.reserve(model.numConstraints());
            for (size_t g = 0; g < groups.size(); g++) { ids.insert(ids.end(), groups[g].begin(), groups[g].end()); off[g + 1] = (unsigned int)ids.size(); }
            if (pbd_set_groups(m_engine, (unsigned int)groups.size(), off.data(), ids.data())) return fail("pbd_set_groups");
        }
        lap("colouring + groups into the model");
        m_boundGeneration = model.constraintGeneration();
    }
    m_boundModel = &model;
    // lazy per-attribute download installed on the model's particle container
    pbd_engine *eng = m_engine;
    ParticleData *pdp = &pd;
    pd.pullAttr = [eng, pdp](int attr) -> bool {
        std::vector<Vector3r> *dst[5] = {&pdp->m_x, &pdp->m_v, &pdp->m_x0, &pdp->m_oldX, &pdp->m_lastX};
        if (pdp->size() == 0) return true;
        return pbd_get_attr(eng, attr, &(*dst[attr])[0][0]) == 0;
    };
    return true;
}

// ---------------------------------------------------------------------------------------------------------
// DistanceFieldCollisionDetection: registry only (the tests run in csrc/contacts.cuh)
// ---------------------------------------------------------------------------------------------------------
CollisionDetection::CollisionObject &DistanceFieldCollisionDetection::add(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices,
                                                                          unsigned int numVertices, int shape, bool testMesh, bool invertSDF) {
    m_collisionObjects.emplace_back();
    CollisionObject &co = m_collisionObjects.back();
    co.m_bodyIndex = bodyIndex; co.m_bodyType = bodyType; co.shape = shape; co.m_testMesh = testMesh; co.invertSDF = invertSDF;
    if (vertices && bodyType == CollisionObject::RigidBodyCollisionObjectType) co.vertices.assign(vertices, vertices + numVertices);
    return co;
}
void DistanceFieldCollisionDetection::addCollisionBox(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector3r &box, bool testMesh, bool invertSDF) {
    CollisionObject &co = add(bodyIndex, bodyType, vertices, numVertices, PBD_SHAPE_BOX, testMesh, invertSDF);
    for (int k = 0; k < 3; k++) co.dim[k] = static_cast<Real>(0.5) * box[k];  // the distance function takes half extents (:503)
}
void DistanceFieldCollisionDetection::addCollisionSphere(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, Real radius, bool testMesh, bool invertSDF) {
    add(bodyIndex, bodyType, vertices, numVertices, PBD_SHAPE_SPHERE, testMesh, invertSDF).dim[0] = radius;
}
void DistanceFieldCollisionDetection::addCollisionTorus(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector2r &radii, bool testMesh, bool invertSDF) {
    CollisionObject &co = add(bodyIndex, bodyType, vertices, numVertices, PBD_SHAPE_TORUS, testMesh, invertSDF);
    co.dim[0] = radii[0]; co.dim[1] = radii[1];
}
void DistanceFieldCollisionDetection::addCollisionCylinder(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector2r &dim, bool testMesh, bool invertSDF) {
    CollisionObject &co = add(bodyIndex, bodyType, vertices, numVertices, PBD_SHAPE_CYLINDER, testMesh, invertSDF);
    co.dim[0] = dim[0]; co.dim[1] = static_cast<Real>(0.5) * dim[1];  // height / 2 (:545)
}
void DistanceFieldCollisionDetection::addCollisionHollowSphere(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, Real radius, Real thickness, bool testMesh, bool invertSDF) {
    CollisionObject &co = add(bodyIndex, bodyType, vertices, numVertices, PBD_SHAPE_HOLLOW_SPHERE, testMesh, invertSDF);
    co.dim[0] = radius; co.thickness = thickness;
}
void DistanceFieldCollisionDetection::addCollisionHollowBox(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, const Vector3r &box, Real thickness, bool testMesh, bool invertSDF) {
    CollisionObject &co = add(bodyIndex, bodyType, vertices, numVertices, PBD_SHAPE_HOLLOW_BOX, testMesh, invertSDF);
    for (int k = 0; k < 3; k++) co.dim[k] = static_cast<Real>(0.5) * box[k];
    co.thickness = thickness;
}
void DistanceFieldCollisionDetection::addCollisionObjectWithoutGeometry(unsigned int bodyIndex, unsigned int bodyType, const Vector3r *vertices, unsigned int numVertices, bool testMesh) {
    add(bodyIndex, bodyType, vertices, numVertices, -1, testMesh, false);
}

// The pair dispatch of DistanceFieldCollisionDetection::collisionDetection (DistanceFieldCollisionDetection.cpp:96-165) reduced to what the GPU
// path covers; everything else is an error (the reference would run it, this engine cannot).
bool TimeStepController::uploadColliders(SimulationModel &model) {
    std::vector<pbd_particle_collider> pcs;
    std::vector<pbd_rigid_collider> rcs;
    if (m_collisionDetection) {
        unsigned int tetObjects = 0;
        for (const CollisionDetection::CollisionObject &co : m_collisionDetection->getCollisionObjects()) {
            typedef CollisionDetection::CollisionObject CO;
            if (co.m_bodyType == CO::TriangleModelCollisionObjectType || co.m_bodyType == CO::TetModelCollisionObjectType) {
                const bool tet = (co.m_bodyType == CO::TetModelCollisionObjectType);
                if (tet && ++tetObjects > 1) { m_error = "two tet models as collision objects produce particle-tet contacts, which are not on the GPU path"; return false; }
                if (!co.m_testMesh) continue;
                pbd_particle_collider pc;
                if (tet) {
                    if (co.m_bodyIndex >= model.getTetModels().size()) { m_error = "collision object refers to a tet model that does not exist"; return false; }
                    const TetModel *tm = model.getTetModels()[co.m_bodyIndex];
                    pc.offset = tm->getIndexOffset(); pc.count = tm->getParticleMesh().numVertices(); pc.restitution = tm->getRestitutionCoeff(); pc.friction = tm->getFrictionCoeff();
                } else {
                    if (co.m_bodyIndex >= model.getTriangleModels().size()) { m_error = "collision object refers to a triangle model that does not exist"; return false; }
                    const TriangleModel *tm = model.getTriangleModels()[co.m_bodyIndex];
                    pc.offset = tm->getIndexOffset(); pc.count = tm->getParticleMesh().numVertices(); pc.restitution = tm->getRestitutionCoeff(); pc.friction = tm->getFrictionCoeff();
                }
                pcs.push_back(pc);
                continue;
            }
            if (co.m_bodyType != CO::RigidBodyCollisionObjectType || co.shape < 0) continue;
            if (co.m_bodyIndex >= model.getRigidBodies().size()) { m_error = "collision object refers to a rigid body that does not exist"; return false; }
            const RigidBody &rb = *model.getRigidBodies()[co.m_bodyIndex];
            if (rb.getMass() != 0) { m_error = "rigid body " + std::to_string(co.m_bodyIndex) + " is a dynamic collision object; contacts with dynamic bodies are not on the GPU path (static colliders only)"; return false; }
            if (co.invertSDF) { m_error = "collision objects with an inverted distance field are not on the GPU path"; return false; }
            pbd_rigid_collider rc;
            std::memset(&rc, 0, sizeof(rc));
            rc.shape = co.shape; rc.body = co.m_bodyIndex; rc.thickness = co.thickness; rc.invert_sdf = 0;
            for (int k = 0; k < 3; k++) rc.dim[k] = co.dim[k];
            rc.restitution = rb.getRestitutionCoeff(); rc.friction = rb.getFrictionCoeff();
            // x_local = frameR * R(q)^T (x_w - x) + frameT  (RigidBody::updateInverseTransformation, RigidBody.h:172-188)
            const Quaternionr &q = rb.getRotation();
            const Real Rq[9] = {1 - 2 * (q.y * q.y + q.z * q.z), 2 * (q.x * q.y - q.w * q.z), 2 * (q.x * q.z + q.w * q.y),
                                2 * (q.x * q.y + q.w * q.z), 1 - 2 * (q.x * q.x + q.z * q.z), 2 * (q.y * q.z - q.w * q.x),
                                2 * (q.x * q.z - q.w * q.y), 2 * (q.y * q.z + q.w * q.x), 1 - 2 * (q.x * q.x + q.y * q.y)};
            Real T[9];  // transformation R = frameR * R(q)^T
            for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { Real a = 0; for (int k = 0; k < 3; k++) a += rb.m_frameR.m[3 * r + k] * Rq[3 * c + k]; T[3 * r + c] = a; }
            for (int k = 0; k < 9; k++) rc.R[k] = T[k];
            for (int k = 0; k < 3; k++) {
                rc.v1[k] = rb.m_frameT[k];
                rc.v2[k] = rb.getPosition()[k] - (T[k] * rb.m_frameT[0] + T[3 + k] * rb.m_frameT[1] + T[6 + k] * rb.m_frameT[2]);  // x - T^T frameT
            }
            // bounding box: the object's vertices in world space (CollisionDetection::updateAABB), else the shape's own box
            Real lo[3] = {1e30f, 1e30f, 1e30f}, hi[3] = {-1e30f, -1e30f, -1e30f};
            auto extend = [&](const Real v[3]) {  // x_w = T^T v + v2
                for (int r = 0; r < 3; r++) {
                    const Real w = T[r] * v[0] + T[3 + r] * v[1] + T[6 + r] * v[2] + rc.v2[r];
                    lo[r] = std::min(lo[r], w); hi[r] = std::max(hi[r], w);
                }
            };
            if (!co.vertices.empty()) { for (const Vector3r &v : co.vertices) { const Real t[3] = {v[0], v[1], v[2]}; extend(t); } }
            else {
                Real h[3] = {co.dim[0], co.dim[1], co.dim[2]};
                if (co.shape == PBD_SHAPE_SPHERE || co.shape == PBD_SHAPE_HOLLOW_SPHERE) h[0] = h[1] = h[2] = co.dim[0] + co.thickness;
                else if (co.shape == PBD_SHAPE_TORUS) { h[0] = h[2] = co.dim[0] + co.dim[1]; h[1] = co.dim[1]; }
                else if (co.shape == PBD_SHAPE_CYLINDER) { h[0] = h[2] = co.dim[0]; h[1] = co.dim[1]; }
                else if (co.shape == PBD_SHAPE_HOLLOW_BOX) for (int k = 0; k < 3; k++) h[k] += co.thickness;
                for (int corner = 0; corner < 8; corner++) { const Real t[3] = {(corner & 1) ? h[0] : -h[0], (corner & 2) ? h[1] : -h[1], (corner & 4) ? h[2] : -h[2]}; extend(t); }
            }
            const Real tol = m_collisionDetection->getTolerance();
            for (int k = 0; k < 3; k++) { rc.aabb_min[k] = lo[k] - tol; rc.aabb_max[k] = hi[k] + tol; }
            rcs.push_back(rc);
        }
    }
    // send only when something changed (byte image of the arguments)
    std::vector<unsigned char> image(pcs.size() * sizeof(pbd_particle_collider) + rcs.size() * sizeof(pbd_rigid_collider) + 1, 0);
    if (!pcs.empty()) std::memcpy(image.data(), pcs.data(), pcs.size() * sizeof(pbd_particle_collider));
    if (!rcs.empty()) std::memcpy(image.data() + pcs.size() * sizeof(pbd_particle_collider), rcs.data(), rcs.size() * sizeof(pbd_rigid_collider));
    image.back() = (unsigned char)pcs.size();
    if (image != m_collidersSent) {
        if (pbd_set_colliders(m_engine, (unsigned)pcs.size(), pcs.data(), (unsigned)rcs.size(), rcs.data())) return fail("pbd_set_colliders");
        m_collidersSent.swap(image);
    }
    if (m_collisionDetection && pbd_set_contact_params(m_engine, m_collisionDetection->getTolerance(), model.getContactStiffnessParticleRigidBody(), m_maxIterationsV)) return fail("pbd_set_contact_params");
    return true;
}

bool TimeStepController::step(SimulationModel &model) {
    if (!m_engine) { if (m_error.empty()) m_error = "no engine"; return false; }
    if (!uploadModel(model)) return false;
    if ((m_collisionDetection || !m_collidersSent.empty()) && !uploadColliders(model)) return false;
    const float g[3] = {m_gravitation[0], m_gravitation[1], m_gravitation[2]};
    if (m_mode != m_modeSent) { if (pbd_set_mode(m_engine, m_mode)) return fail("pbd_set_mode"); m_modeSent = m_mode; }
    if (pbd_set_params(m_engine, m_tm.getTimeStepSize(), m_subSteps, m_maxIterations, m_velocityUpdateMethod, g)) return fail("pbd_set_params");
    if (pbd_step(m_engine, 1)) return fail("pbd_step");
    if (!model.getRigidBodies().empty()) {  // a handful of bodies: mirror their state right away
        SimulationModel::RigidBodyVector &rbs = model.getRigidBodies();
        const unsigned int nr = (unsigned int)rbs.size();
        std::vector<float> x(3 * nr), q(4 * nr), v(3 * nr), w(3 * nr);
        if (pbd_get_rigid_bodies(m_engine, x.data(), q.data(), v.data(), w.data())) return fail("pbd_get_rigid_bodies");
        for (unsigned int i = 0; i < nr; i++) {
            RigidBody &b = *rbs[i];
            for (int k = 0; k < 3; k++) { b.m_x[k] = x[3 * i + k]; b.m_v[k] = v[3 * i + k]; b.m_omega[k] = w[3 * i + k]; }
            b.m_q = Quaternionr(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]);
        }
    }
    ParticleData &pd = model.getParticles();
    pd.aheadMask |= (1u << PBD_ATTR_X) | (1u << PBD_ATTR_V) | (1u << PBD_ATTR_OLDX) | (1u << PBD_ATTR_LASTX);
    m_tm.setTime(m_tm.getTime() + m_tm.getTimeStepSize());  // TimeStepController.cpp:239
    return true;
}

}  // namespace pbd_b200
