// positionbaseddynamics_b200/csrc/engine.cu
//
// Host side of the H100 PBD/XPBD engine behind the C ABI of include/pbd_b200.h:
//   * the device image: colour groups (device colouring), the image planned by host/image_plan.cpp, and its upload,
//   * the step driver that replaces TimeStepController::step (Simulation/TimeStepController.cpp:75-241) for
//     particle constraints: per substep  integrate -> maxIterations x (colour by colour, bucket by bucket) -> velocity update,
//     executed as plain launches, as a replayed CUDA graph, or as one cluster launch with the positions resident in
//     distributed shared memory (resident.cuh).
// There is no CPU fallback: every path that computes needs the CUDA device.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <array>
#include <string>
#include <vector>
#include "kernels.cuh"
#include "resident.cuh"
#include "colouring.cuh"
#include "contacts.cuh"
#include <cub/cub.cuh>
#include <omp.h>
#include "host/image_plan.h"

using namespace pbdk;
using pbd_b200::host_threads;
using pbd_b200::verbose;
using pbd_b200::is_rb_body;

// ------------------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(const char *fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_err = buf;
    return 1;
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)
#define CKE(e) do { int r_ = (e); if (r_) return r_; } while (0)

extern "C" const char *pbd_last_error(void) { return g_err.c_str(); }

// ------------------------------------------------------------------------------------------------------------
// engine state
// ------------------------------------------------------------------------------------------------------------
using pbd_b200::PodVector;        // std::vector whose resize() does not zero (filled from all threads right after)
using pbd_b200::TypeStore;        // constraints of one type as handed in through pbd_add_constraints (ids: insertion index)

struct DevBuf {                   // one device allocation, freed with its owner
    void *p = nullptr; size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    int alloc(size_t b) {
        if (b <= bytes && p) return 0;
        if (p) cudaFree(p);
        p = nullptr; bytes = 0;
        if (b == 0) return 0;
        cudaError_t e = cudaMalloc(&p, b);
        if (e != cudaSuccess) return fail("cudaMalloc(%zu) -> %s", b, cudaGetErrorString(e));
        bytes = b;
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
};

constexpr int kNumAttrs = PBD_ATTR_LASTX + 1;  // x, v, x0, oldX, lastX

struct DevType {
    // replica batch: the geometry arrays every replica's projections read while per-replica rest shapes are on (K x count; they keep
    // their address while it stays on)
    DevBuf repGv[kMaxGeoV], repGs[kMaxGeoS];
    // replica batch with per-constraint materials of every replica (pbd_set_replica_constraint_materials): the values in the order the
    // constraints were added (K x count x nMat), and what the projections read, gathered from them into device order (one K x count array
    // per material slot).  Both keep their address while K and count stay.
    DevBuf cmat, repMat[kMaxMat];
    PodVector<unsigned> order;    // position in the device arrays -> insertion id
    unsigned count = 0;
    // pointers into the image (upload_image): the arrays the kernels read, and what a batch's per-replica geometry is derived from
    TypeArrays arrays{};
    pbd_b200::RestTables rest{};
};

struct pbd_engine {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool ownsStream = false;
    int smCount = 132;                    // H100 SXM; read from the device in pbd_create
    size_t l2Bytes = 50u << 20;           // likewise
    // particles: batch.K replicas of n (pbd_set_replicas), replica r at device slots [r n, (r + 1) n); one float4 array per attribute,
    // indexed by pbd_attr (attr_ptr).  stage: the host copies' staging areas, K n 3 floats each (upload_attr / download_attr; set_w's
    // masses in stage[0]); stage[1] only for pbd_step_host, so that its x and v uploads do not wait on each other.
    unsigned n = 0;
    DevBuf attr[kNumAttrs], stage[2], jacobiDelta;
    // external forces (pbd_set_external_forces): K x n float4 in slot order like the particle arrays (.w unused), null while none is set.
    // Not an attribute: it keeps its address while n and K stand, is moved by relayout with them, and is released by pbd_set_particles and
    // pbd_set_replicas.
    DevBuf force;
    // A replica batch and what its replicas have of their own (batch_arrays, replica_mat and replica_geo turn it into what the kernels see).
    // mat [K][kMatRowFloats]: the uniform material parameters of every type, replica by replica -- the shared ones of the image, or a
    // replica's own (pbd_set_replica_materials, the types of matMask); gravity [K][3] (pbd_set_replica_gravity).
    // restX: per-replica rest shapes (pbd_set_replica_rest_positions), the rest positions the call was given, K x n float4 by host index
    // with .w = the inverse mass at the time of the call; every image planned while restShapes is on derives its geometry from them.
    // restTables: images carry what a derivation reads (TypePlan::restBodies / restLocal), from the first pbd_set_replica_rest_positions
    // until the override is dropped, so that batches without it do not pay for them.
    // cmatMask: the types whose materials are per constraint and per replica (pbd_set_replica_constraint_materials; DevType::cmat).  A type
    // takes its materials from one source: the shared parameters, its rows of `mat` (matMask) or its per-constraint arrays (cmatMask).  The
    // gather reads the image's restTables too, so images carry them while any type has the override on (rest_tables).
    struct Batch {
        unsigned K = 1, matMask = 0, cmatMask = 0;
        DevBuf mat, gravity, restX;
        bool gravitySet = false, restShapes = false, restTables = false;
    } batch;
    // rigid bodies coupled through joints (SURVEY.md 8f-1): float4 arrays X(xyz,invMass) Q(x,y,z,w) V(xyz,mass) W(omega) + history + inertia.
    // nRb bodies per replica, K x nRb rows, replica r's at [r nRb, (r + 1) nRb).  rbReplica: the bodies came from
    // pbd_set_replica_rigid_bodies (every replica has its own; a batch admits them), not from pbd_set_rigid_bodies (one scene's).
    unsigned nRb = 0;
    bool rbReplica = false;
    bool rbMassStale = false;  // rbMass (contact path, below) predates a device write of the masses: read back before it is used
    DevBuf rbX, rbQ, rbV, rbW, rbOldX, rbLastX, rbOldQ, rbLastQ, rbI, rbIinv;
    // constraints (host copy, insertion order) and groups
    TypeStore host[PBD_NUM_TYPES];
    unsigned numConstraints = 0;
    std::vector<unsigned> groupOff, groupIds;
    bool groupsSet = false; unsigned long long modelGen = 0;  // modelGen: counts model_changed (particles, constraints or groups replaced)
    // device image: one allocation (upload_image), and the image_key it was planned under
    DevType dev[PBD_NUM_TYPES];
    std::vector<Bucket> buckets;
    DevBuf image, dTrace;
    pbd_b200::ImageTables tables{};
    std::vector<unsigned char> imageKey; unsigned long long imageGen = 0;  // imageGen: images planned so far
    // parameters
    float dt = 0.005f; unsigned subSteps = 5, maxIter = 1; int velMethod = 0; float g[3] = {0.f, -9.81f, 0.f};
    int mode = PBD_MODE_AUTO;             // requested (pbd_set_mode); what the image runs in: active_mode
    // graph cache: the captured step and the graph_key it was captured under
    cudaGraphExec_t graphExec = nullptr;
    std::vector<unsigned char> graphKey;
    unsigned long long graphLaunches = 0;  // kernel nodes of the captured step
    // stats
    pbd_stats stats{};
    cudaEvent_t evStart = nullptr, evStop = nullptr;
    // the device-memory state calls (pbd_set_attr_device ...) on a caller's stream: the engine stream waits for evCaller, recorded on the
    // caller's stream, before the copy; the caller's stream waits for evEngine, recorded on the engine stream, after it
    cudaEvent_t evCaller = nullptr, evEngine = nullptr;
    // pbd_step_host_async: two staging slots, one upload and one download stream next to the compute stream
    struct HostPipe {
        cudaStream_t up = nullptr, down = nullptr;
        DevBuf inX[2], inV[2], outX[2], outV[2];
        cudaEvent_t uploaded[2] = {nullptr, nullptr}, consumed[2] = {nullptr, nullptr}, produced[2] = {nullptr, nullptr}, downloaded[2] = {nullptr, nullptr};
        unsigned long long issued = 0;
        bool ready = false;
    } pipe;
    // contact path (contacts.cuh): colliders, parameters, optional record of the last step's contacts
    std::vector<float> rbMass;
    std::vector<ParticleCollider> pColliders;
    std::vector<RigidCollider> rColliders;
    DevBuf dPColliders, dRColliders, dRangeStart, dContacts, dContactCount;
    unsigned contactTotal = 0, contactCap = 0;
    float contactTolerance = 0.01f, contactStiffness = 100.0f; unsigned maxIterV = 5;  // CollisionDetection.cpp:25, SimulationModel.cpp:34, TimeStepController.cpp:23
    // contacts of a replica batch (pbd_set_replica_colliders): one replica's particle ranges, K x nRigid colliders and the bodies carrying
    // them, replica after replica (rbX / rbV / rbW as float4, one body per collider).  The device tables keep their address while nP and
    // nRigid stay, so that new rows are copied in stream order between steps.  nRigid == 0: off.
    struct ReplicaColliders {
        std::vector<ParticleCollider> ranges;
        unsigned nRigid = 0, total = 0;
        DevBuf dRanges, dStart, dRigid, dX, dV, dW;
    } repColliders;
    // contact sensors (pbd_sense_contacts): per replica and rigid collider, the contacts found and the impulse received in the last step.
    // partial: the contact launch's per-block sums (K x blocks x nRigid float4), summed into count / impulse by k_contact_sensors_sum.
    // Sized for the colliders in force (K, nRigid, blocks) by size_sensors, outside the steps; all zero when nRigid == 0.
    struct Sensors {
        bool on = false;
        unsigned K = 0, nRigid = 0, blocks = 0;
        DevBuf partial, count, impulse;
    } sensors;
    bool timingPending = false;
    std::vector<unsigned> slot;          // host particle index -> device slot (formula layouts or the tile-major permutation)
    DevBuf dSlot, dSlotOld, relayoutTmp;
    // resident mode (resident.cuh): the launch shape of the current image (res.G == 0: the image is not tiled)
    pbd_b200::ResidentShape res;
    unsigned long long xLaunch = 0;       // resident launches so far: the high word of the X arrival flags
};

static int use(pbd_engine *e) { CK(cudaSetDevice(e->device)); return 0; }
static bool rest_tables(const pbd_engine *e) { return e->batch.restTables || e->batch.cmatMask; }

static void model_changed(pbd_engine *e) { e->modelGen++; }  // what the device image is planned from (image_key) replaced
static void drop_replica_geometry(pbd_engine *e) {
    e->batch.restShapes = e->batch.restTables = false;
    e->batch.restX.release();
    for (DevType &d : e->dev) {
        for (DevBuf &b : d.repGv) b.release();
        for (DevBuf &b : d.repGs) b.release();
    }
}

// per-constraint materials of the types in `types` back to their other source (what matMask says); the steps in flight are done first
static int drop_constraint_materials(pbd_engine *e, unsigned types) {
    if (!(e->batch.cmatMask & types)) return 0;
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    for (int t = 0; t < PBD_NUM_TYPES; t++)
        if ((types >> t) & 1u) {
            e->dev[t].cmat.release();
            for (DevBuf &b : e->dev[t].repMat) b.release();
        }
    e->batch.cmatMask &= ~types;
    return 0;
}

extern "C" int pbd_device_count(int *count) {
    cudaError_t err = cudaGetDeviceCount(count);
    if (err != cudaSuccess) { *count = 0; return fail("cudaGetDeviceCount -> %s", cudaGetErrorString(err)); }
    return 0;
}
extern "C" int pbd_num_bodies(int type) { return type_shape(type).nBodies; }
extern "C" int pbd_num_params(int type) { return type_shape(type).nParams; }
extern "C" int pbd_num_materials(int type) { return type_shape(type).nMat; }

extern "C" int pbd_create(int device, void *stream, pbd_engine **out) {
    if (!out) return fail("pbd_create: out == NULL");
    int count = 0;
    cudaError_t err = cudaGetDeviceCount(&count);
    if (err != cudaSuccess || count == 0)
        return fail("pbd_create: no CUDA device available (%s); this engine has no CPU fallback",
                    err != cudaSuccess ? cudaGetErrorString(err) : "device count 0");
    if (device < 0 || device >= count) return fail("pbd_create: device %d out of range [0,%d)", device, count);
    pbd_engine *e = new pbd_engine();
    e->device = device;
    if (use(e)) { delete e; return 1; }
    cudaDeviceProp prop;
    err = cudaGetDeviceProperties(&prop, device);
    if (err != cudaSuccess) { delete e; return fail("cudaGetDeviceProperties -> %s", cudaGetErrorString(err)); }
    e->smCount = prop.multiProcessorCount;
    e->l2Bytes = (size_t)prop.l2CacheSize;
    if (stream) { e->stream = (cudaStream_t)stream; e->ownsStream = false; }
    else {
        err = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
        if (err != cudaSuccess) { delete e; return fail("cudaStreamCreate -> %s", cudaGetErrorString(err)); }
        e->ownsStream = true;
    }
    cudaEventCreate(&e->evStart); cudaEventCreate(&e->evStop);
    cudaEventCreateWithFlags(&e->evCaller, cudaEventDisableTiming); cudaEventCreateWithFlags(&e->evEngine, cudaEventDisableTiming);
    *out = e;
    return 0;
}

extern "C" int pbd_destroy(pbd_engine *e) {
    if (!e) return 0;
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    if (e->graphExec) cudaGraphExecDestroy(e->graphExec);
    if (e->evStart) cudaEventDestroy(e->evStart);
    if (e->evStop) cudaEventDestroy(e->evStop);
    if (e->evCaller) cudaEventDestroy(e->evCaller);
    if (e->evEngine) cudaEventDestroy(e->evEngine);
    if (e->pipe.ready) {
        cudaStreamSynchronize(e->pipe.up); cudaStreamSynchronize(e->pipe.down);
        for (int s = 0; s < 2; s++)
            for (cudaEvent_t ev : {e->pipe.uploaded[s], e->pipe.consumed[s], e->pipe.produced[s], e->pipe.downloaded[s]}) cudaEventDestroy(ev);
        cudaStreamDestroy(e->pipe.up); cudaStreamDestroy(e->pipe.down);
    }
    if (e->ownsStream) cudaStreamDestroy(e->stream);
    delete e;  // the DevBufs free the device memory (on the device selected above)
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// particles
// ------------------------------------------------------------------------------------------------------------
static inline unsigned nblk(unsigned n, unsigned t) { return (n + t - 1) / t; }

static float4 *attr_ptr(const pbd_engine *e, int a) { return (float4 *)e->attr[a].p; }

static int upload_slot_map(pbd_engine *e) {
    if (e->n == 0) return 0;
    CKE(e->dSlot.alloc((size_t)e->n * sizeof(unsigned)));
    CK(cudaMemcpy(e->dSlot.p, e->slot.data(), (size_t)e->n * sizeof(unsigned), cudaMemcpyHostToDevice));
    return 0;
}
// move every particle array, and the external forces if any are set, from the current slot map to `newSlot`
static int relayout(pbd_engine *e, const std::vector<unsigned> &newSlot) {
    if (e->n == 0 || newSlot == e->slot) { e->slot = newSlot; return 0; }
    const size_t nb = (size_t)e->n * sizeof(unsigned);
    CKE(e->dSlotOld.alloc(nb));
    CK(cudaMemcpy(e->dSlotOld.p, e->slot.data(), nb, cudaMemcpyHostToDevice));
    e->slot = newSlot;
    CKE(upload_slot_map(e));
    CKE(e->relayoutTmp.alloc((size_t)e->batch.K * e->n * sizeof(float4)));
    std::vector<DevBuf *> moved;
    for (DevBuf &b : e->attr) moved.push_back(&b);
    if (e->force.p) moved.push_back(&e->force);
    for (DevBuf *b : moved) {
        k_relayout<<<dim3((e->n + 255) / 256, e->batch.K), 256, 0, e->stream>>>((const float4 *)b->p, (float4 *)e->relayoutTmp.p, e->n, (const unsigned *)e->dSlotOld.p, (const unsigned *)e->dSlot.p);
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(e->stream));
        std::swap(b->p, e->relayoutTmp.p); std::swap(b->bytes, e->relayoutTmp.bytes);
    }
    return 0;
}

// grid of a per-particle kernel over `replicas` replicas: blockIdx.y = replica (kernels.cuh: k_pack3 ...)
static dim3 replica_grid(const pbd_engine *e, unsigned replicas) { return dim3(nblk(e->n, 256), replicas); }

// The per-particle copies between AoS-3 device buffers (K n 3 floats, host particle order) and the particle arrays, on the engine stream.
// mask: the replicas written (k_pack3 / k_set_w), nullptr for all of them.
static int pack_attr(pbd_engine *e, int a, const float *src, int keepW, unsigned replicas, const unsigned char *mask) {
    k_pack3<<<replica_grid(e, replicas), 256, 0, e->stream>>>(src, attr_ptr(e, a), e->n, keepW, (const unsigned *)e->dSlot.p, mask);
    CK(cudaGetLastError());
    return 0;
}
static int unpack_attr(pbd_engine *e, int a, float *dst) {
    k_unpack3<<<replica_grid(e, e->batch.K), 256, 0, e->stream>>>(attr_ptr(e, a), dst, e->n, (const unsigned *)e->dSlot.p);
    CK(cudaGetLastError());
    return 0;
}
static int pack_w(pbd_engine *e, const float *mass, unsigned replicas, const unsigned char *mask) {
    k_set_w<<<replica_grid(e, replicas), 256, 0, e->stream>>>(attr_ptr(e, PBD_ATTR_X), attr_ptr(e, PBD_ATTR_V), mass, e->n, (const unsigned *)e->dSlot.p, mask);
    CK(cudaGetLastError());
    return 0;
}

// Host AoS-3 of the first `replicas` replicas -> `staging` on stream `copy` -> attribute `a` by k_pack3 on the engine stream (.w kept
// with keepW).  host == nullptr: `staging` holds the copy already.  A copy stream other than the engine's comes with `copied`, through
// which the pack waits for the copy.
static int upload_attr(pbd_engine *e, int a, const float *host, int keepW, unsigned replicas, const DevBuf &staging, cudaStream_t copy,
                       cudaEvent_t copied = nullptr) {
    if (host) CK(cudaMemcpyAsync(staging.p, host, (size_t)replicas * e->n * 3 * sizeof(float), cudaMemcpyHostToDevice, copy));
    if (copied) { CK(cudaEventRecord(copied, copy)); CK(cudaStreamWaitEvent(e->stream, copied, 0)); }
    return pack_attr(e, a, (const float *)staging.p, keepW, replicas, nullptr);
}
// Attribute `a` of every replica -> `staging` by k_unpack3 on the engine stream -> host AoS-3 on stream `copy`.  A copy stream other
// than the engine's comes with `unpacked`, through which the copy waits for the unpack.
static int download_attr(pbd_engine *e, int a, float *host, const DevBuf &staging, cudaStream_t copy, cudaEvent_t unpacked = nullptr) {
    CKE(unpack_attr(e, a, (float *)staging.p));
    if (unpacked) { CK(cudaEventRecord(unpacked, e->stream)); CK(cudaStreamWaitEvent(copy, unpacked, 0)); }
    CK(cudaMemcpyAsync(host, staging.p, (size_t)e->batch.K * e->n * 3 * sizeof(float), cudaMemcpyDeviceToHost, copy));
    return 0;
}

// masses of the first `replicas` replicas (n floats each), staged in stage[0]
static int set_w(pbd_engine *e, const float *mass, unsigned replicas) {
    CK(cudaMemcpyAsync(e->stage[0].p, mass, (size_t)replicas * e->n * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    CKE(pack_w(e, (const float *)e->stage[0].p, replicas, nullptr));
    CK(cudaStreamSynchronize(e->stream));  // staging buffers are reused by the next call
    return 0;
}

extern "C" int pbd_set_masses(pbd_engine *e, const float *mass) {
    if (!e || !mass) return fail("pbd_set_masses: null argument");
    CKE(use(e));
    if (e->n == 0) return 0;
    return set_w(e, mass, e->batch.K);
}

// the first `one` bytes of `p` copied to the K - 1 places after them (doubling copies)
static int broadcast_rows(pbd_engine *e, void *p, size_t one, unsigned K) {
    for (size_t have = 1; have < K; have *= 2)
        CK(cudaMemcpyAsync((char *)p + have * one, p, std::min(have, (size_t)K - have) * one, cudaMemcpyDeviceToDevice, e->stream));
    return 0;
}
// replica 0 of every particle array copied to replicas 1 .. K-1
static int broadcast_replica0(pbd_engine *e, unsigned K) {
    for (DevBuf &b : e->attr) CKE(broadcast_rows(e, b.p, (size_t)e->n * sizeof(float4), K));
    return 0;
}
// The particle arrays sized for K replicas of n, and stage[0] for their host copies.  keepReplica0: replica 0 moves into fresh arrays
// (the old ones are freed) and replicas 1 .. K-1 become copies of it; otherwise what the arrays hold is the caller's to write.
static int size_particles(pbd_engine *e, unsigned K, bool keepReplica0) {
    const size_t one = (size_t)e->n * sizeof(float4);
    const bool keep = keepReplica0 && one;
    for (DevBuf &b : e->attr) {
        if (!keep) { CKE(b.alloc(one * K)); continue; }
        DevBuf grown;
        CKE(grown.alloc(one * K));
        CK(cudaMemcpyAsync(grown.p, b.p, one, cudaMemcpyDeviceToDevice, e->stream));
        std::swap(b.p, grown.p); std::swap(b.bytes, grown.bytes);
        CK(cudaStreamSynchronize(e->stream));  // before `grown` frees the old array
    }
    CKE(e->stage[0].alloc((size_t)K * e->n * 3 * sizeof(float)));
    return keep ? broadcast_replica0(e, K) : 0;
}

// the rigid-body arrays, in the order of rb_state's members
static std::array<DevBuf *, 10> rb_bufs(pbd_engine *e) {
    return {&e->rbX, &e->rbQ, &e->rbV, &e->rbW, &e->rbOldX, &e->rbLastX, &e->rbOldQ, &e->rbLastQ, &e->rbI, &e->rbIinv};
}
// A batch's per-replica bodies resized for K replicas: replica 0 moves into fresh arrays, replicas 1 .. K-1 become copies of it.
static int size_bodies(pbd_engine *e, unsigned K) {
    const size_t one = (size_t)e->nRb * sizeof(float4);
    if (!e->rbReplica || !one) return 0;
    for (DevBuf *b : rb_bufs(e)) {
        DevBuf grown;
        CKE(grown.alloc(one * K));
        CK(cudaMemcpyAsync(grown.p, b->p, one, cudaMemcpyDeviceToDevice, e->stream));
        CKE(broadcast_rows(e, grown.p, one, K));
        CK(cudaStreamSynchronize(e->stream));  // before `grown` frees the old array
        std::swap(b->p, grown.p); std::swap(b->bytes, grown.bytes);
    }
    std::vector<float> mass((size_t)K * e->nRb);
    for (size_t i = 0; i < mass.size(); i++) mass[i] = e->rbMass[i % e->nRb];
    e->rbMass.swap(mass);
    return 0;
}

extern "C" int pbd_set_particles(pbd_engine *e, unsigned n, const float *x, const float *x0, const float *v, const float *mass) {
    if (!e || (n && (!x || !mass))) return fail("pbd_set_particles: null argument");
    const std::string why = pbd_b200::batch_refusal(e->batch.K, n, e->mode, e->nRb, e->host, e->rbReplica);
    if (!why.empty()) return fail("pbd_set_particles: %s", why.c_str());
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    e->n = n; model_changed(e);  // and the formula slot map below
    CKE(size_particles(e, e->batch.K, false));
    drop_replica_geometry(e);  // every replica's state is redefined
    e->force.release();        // forces of the old particles
    e->slot.resize(n);
    for (unsigned i = 0; i < n; i++) e->slot[i] = particle_slot(i, n);
    if (n == 0) return 0;
    CKE(upload_slot_map(e));
    const size_t b4 = (size_t)n * sizeof(float4);
    CK(cudaMemsetAsync(attr_ptr(e, PBD_ATTR_V), 0, b4, e->stream));
    CKE(upload_attr(e, PBD_ATTR_X, x, 0, 1, e->stage[0], e->stream)); CK(cudaStreamSynchronize(e->stream));
    if (v) { CKE(upload_attr(e, PBD_ATTR_V, v, 0, 1, e->stage[0], e->stream)); CK(cudaStreamSynchronize(e->stream)); }
    CKE(set_w(e, mass, 1));
    // oldX = lastX = x, x0 = x unless given (ParticleData::addVertex, ParticleData.h:127-137)
    for (int a : {PBD_ATTR_OLDX, PBD_ATTR_LASTX, PBD_ATTR_X0}) CK(cudaMemcpyAsync(attr_ptr(e, a), attr_ptr(e, PBD_ATTR_X), b4, cudaMemcpyDeviceToDevice, e->stream));
    if (x0) CKE(upload_attr(e, PBD_ATTR_X0, x0, 1, 1, e->stage[0], e->stream));
    CKE(broadcast_replica0(e, e->batch.K));  // every replica of a batch starts here
    CK(cudaStreamSynchronize(e->stream));
    e->stats.num_particles = n;
    return 0;
}

// pbd_set_colliders' colliders belong to one scene; a batch takes its own per replica (pbd_set_replica_colliders)
static int collider_refusal(const pbd_engine *e, unsigned K, size_t nColliders) {
    if (K > 1 && nColliders)
        return fail("replica batch: colliders of pbd_set_colliders are stepped one scene per engine (pbd_set_replicas 1); a batch takes per-replica colliders from pbd_set_replica_colliders");
    return 0;
}
static void drop_replica_colliders(pbd_engine *e) {
    pbd_engine::ReplicaColliders &c = e->repColliders;
    c.ranges.clear(); c.nRigid = c.total = 0;
    for (DevBuf *b : {&c.dRanges, &c.dStart, &c.dRigid, &c.dX, &c.dV, &c.dW}) b->release();
}
// The contact sensors sized for the colliders in force: a batch's replica colliders, else pbd_set_colliders' one scene.  New sizes (sensing
// switched on, other collider or particle counts, another K) zero the outputs once the steps in flight are done; the same sizes keep them.
static int size_sensors(pbd_engine *e) {
    pbd_engine::Sensors &s = e->sensors;
    const pbd_engine::ReplicaColliders &rep = e->repColliders;
    const bool batch = rep.nRigid != 0;
    unsigned K = 0, nR = 0, blocks = 0;
    if (s.on && (batch || !e->rColliders.empty())) {
        K = batch ? e->batch.K : 1u;
        nR = batch ? rep.nRigid : (unsigned)e->rColliders.size();
        blocks = nblk(batch ? rep.total : e->contactTotal, kSenseThreads);
    }
    if (K == s.K && nR == s.nRigid && blocks == s.blocks) return 0;
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    s.K = K; s.nRigid = nR; s.blocks = blocks;
    for (DevBuf *b : {&s.partial, &s.count, &s.impulse}) b->release();
    if (!nR) return 0;
    const size_t rows = (size_t)K * nR;
    CKE(s.partial.alloc(std::max<size_t>(rows * blocks, 1) * sizeof(float4)));
    CKE(s.count.alloc(rows * sizeof(unsigned)));
    CKE(s.impulse.alloc(rows * 3 * sizeof(float)));
    CK(cudaMemsetAsync(s.count.p, 0, rows * sizeof(unsigned), e->stream));
    CK(cudaMemsetAsync(s.impulse.p, 0, rows * 3 * sizeof(float), e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

extern "C" int pbd_set_replicas(pbd_engine *e, unsigned K) {
    if (!e) return fail("null engine");
    const std::string why = pbd_b200::batch_refusal(K, e->n, e->mode, e->nRb, e->host, e->rbReplica);
    if (!why.empty()) return fail("pbd_set_replicas: %s", why.c_str());
    CKE(collider_refusal(e, K, e->pColliders.size() + e->rColliders.size()));
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    CKE(size_particles(e, K, true));  // replica 0 kept, the others copies of it
    CKE(size_bodies(e, K));           // likewise
    e->batch.K = K;
    CKE(drop_constraint_materials(e, ~0u));
    e->batch.mat.release(); e->batch.gravity.release(); e->batch.matMask = 0; e->batch.gravitySet = false;  // rows of the old K
    e->force.release();  // likewise
    drop_replica_geometry(e);
    drop_replica_colliders(e);
    CKE(size_sensors(e));  // sensing stays on; the one scene's colliders, if any, keep their sensors
    CK(cudaStreamSynchronize(e->stream));
    model_changed(e);  // every replica is redefined: planned again, with the shared material rows and zero multipliers
    return 0;
}

static int replica_params_refusal(const pbd_engine *e, const char *what) {
    if (!e) return fail("%s: null engine", what);
    if (e->batch.K == 1) return fail("%s: a single-scene engine takes its parameters from pbd_add_constraints / pbd_set_params (pbd_set_replicas first)", what);
    return 0;
}
// type's columns of the K rows of the material table <- rows of nMat floats `pitch` bytes apart (0: the same row for every replica)
static int write_replica_materials(pbd_engine *e, int type, const float *rows, size_t pitch) {
    if (!e->batch.mat.p) {
        CKE(e->batch.mat.alloc((size_t)e->batch.K * kMatRowFloats * sizeof(float)));
        CK(cudaMemsetAsync(e->batch.mat.p, 0, e->batch.mat.bytes, e->stream));
    }
    const size_t width = type_shape(type).nMat * sizeof(float);
    std::vector<float> same;
    if (!pitch) {
        same.resize((size_t)e->batch.K * type_shape(type).nMat);
        for (size_t i = 0; i < same.size(); i++) same[i] = rows[i % type_shape(type).nMat];
        rows = same.data(); pitch = width;
    }
    CK(cudaMemcpy2DAsync((float *)e->batch.mat.p + mat_offset(type), kMatRowFloats * sizeof(float), rows, pitch, width, e->batch.K, cudaMemcpyHostToDevice, e->stream));
    return 0;
}
extern "C" int pbd_set_replica_materials(pbd_engine *e, int type, const float *mat) {
    if (type < 0 || type >= PBD_NUM_TYPES) return fail("pbd_set_replica_materials: unknown constraint type %d", type);
    const int nMat = type_shape(type).nMat;
    if (nMat == 0) return fail("pbd_set_replica_materials: constraint type %d has no material parameters", type);
    CKE(replica_params_refusal(e, "pbd_set_replica_materials"));
    CKE(use(e));
    const unsigned bit = 1u << type;
    CKE(drop_constraint_materials(e, bit));  // one source per type: this call's
    if (mat) CKE(write_replica_materials(e, type, mat, nMat * sizeof(float)));
    else if (e->batch.matMask & bit) CKE(write_replica_materials(e, type, e->dev[type].arrays.matU, 0));  // (an image planned again writes them too)
    if (mat) e->batch.matMask |= bit; else e->batch.matMask &= ~bit;
    return 0;
}
extern "C" int pbd_set_replica_gravity(pbd_engine *e, const float *g) {
    CKE(replica_params_refusal(e, "pbd_set_replica_gravity"));
    CKE(use(e));
    if (g) {
        CKE(e->batch.gravity.alloc((size_t)e->batch.K * 3 * sizeof(float)));
        CK(cudaMemcpyAsync(e->batch.gravity.p, g, (size_t)e->batch.K * 3 * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    }
    e->batch.gravitySet = (g != nullptr);
    return 0;
}
// What a batch's per-bucket kernels get for type t: where the replicas have parameters of their own, its place in replica 0's row of the
// material table (without them the kernel arguments' uniforms do: reading the table for every launch cost the small shared-parameter
// batches of DESIGN.md section 6 7-17 % in graph mode); and its arrays -- without the per-constraint material arrays in that case.
// With per-replica rest shapes the geometry arrays are the K x count ones, replica r's at r x replica_geo (0: the shared image's).
static const float *replica_mat(const pbd_engine *e, int t) { return ((e->batch.matMask >> t) & 1u) ? (const float *)e->batch.mat.p + mat_offset(t) : nullptr; }
static unsigned replica_geo(const pbd_engine *e, int t) { return e->batch.restShapes && t < PBD_BALLJOINT ? e->dev[t].count : 0u; }  // (joints: no rest shape)
// with per-constraint materials of every replica the material arrays are the K x count ones, replica r's at r x replica_cmat (0: shared)
static unsigned replica_cmat(const pbd_engine *e, int t) { return ((e->batch.cmatMask >> t) & 1u) ? e->dev[t].count : 0u; }
static TypeArrays batch_arrays(const pbd_engine *e, int t) {
    TypeArrays a = e->dev[t].arrays;
    if ((e->batch.matMask >> t) & 1u) for (int k = 0; k < kMaxMat; k++) a.mat[k] = nullptr;
    if ((e->batch.cmatMask >> t) & 1u) for (int k = 0; k < type_shape(t).nMat; k++) a.mat[k] = (const float *)e->dev[t].repMat[k].p;
    if (replica_geo(e, t)) {
        for (int k = 0; k < kMaxGeoV; k++) if (a.gv[k]) a.gv[k] = (const float4 *)e->dev[t].repGv[k].p;
        for (int k = 0; k < kMaxGeoS; k++) if (a.gs[k]) a.gs[k] = (const float *)e->dev[t].repGs[k].p;
    }
    return a;
}

extern "C" int pbd_get_replicas(pbd_engine *e, unsigned *K) {
    if (!e || !K) return fail("pbd_get_replicas: null argument");
    *K = e->batch.K;
    return 0;
}

extern "C" int pbd_set_attr(pbd_engine *e, int attr, const float *src) {
    if (!e || !src) return fail("pbd_set_attr: null argument");
    CKE(use(e));
    if (attr < 0 || attr >= kNumAttrs) return fail("pbd_set_attr: bad attribute %d", attr);
    if (e->n == 0) return 0;
    CKE(upload_attr(e, attr, src, 1, e->batch.K, e->stage[0], e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

extern "C" int pbd_get_attr(pbd_engine *e, int attr, float *dst) {
    if (!e || !dst) return fail("pbd_get_attr: null argument");
    CKE(use(e));
    if (attr < 0 || attr >= kNumAttrs) return fail("pbd_get_attr: bad attribute %d", attr);
    if (e->n == 0) return 0;
    CKE(download_attr(e, attr, dst, e->stage[0], e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

// ---- particle state in device memory (pbd_set_attr_device, pbd_get_attr_device, pbd_set_masses_device) -----------------------------
// `p` must be device or managed memory of the engine's device; host memory, pinned or not, is what the host calls take.
static int device_memory_refusal(const pbd_engine *e, const char *what, const char *arg, const void *p) {
    cudaPointerAttributes a{};
    const cudaError_t err = cudaPointerGetAttributes(&a, p);
    if (err != cudaSuccess) { cudaGetLastError(); return fail("%s: %s: cudaPointerGetAttributes -> %s", what, arg, cudaGetErrorString(err)); }
    const bool onDevice = a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
    if (onDevice && a.device == e->device) return 0;
    if (onDevice) return fail("%s: %s is memory of device %d, the engine runs on device %d", what, arg, a.device, e->device);
    return fail("%s: %s is %s host memory; the device calls take device memory (host arrays go through pbd_set_attr / pbd_get_attr / pbd_set_masses)",
                what, arg, a.type == cudaMemoryTypeHost ? "pinned" : "pageable");
}
// A device-memory state call: every check before anything is enqueued, then `copy` on the engine stream, ordered after the work enqueued
// so far on the caller's stream and before the work enqueued on it later.  The second wait is what lets a caching allocator hand `data`
// out again on the caller's stream while the copy is still pending.  No staging and no host synchronisation.
// `prepare` runs after the checks and before the wait for the caller's stream (work that may synchronise the host goes there).
// `rows`: what the call moves; none is a no-op.
template <class P, class F>
static int device_call(pbd_engine *e, const char *what, const char *arg, const void *data, const unsigned char *mask, void *stream, size_t rows,
                       P &&prepare, F &&copy) {
    if (!data) return fail("%s: %s == NULL", what, arg);
    CKE(use(e));
    const cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
    cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
    CK(cudaStreamIsCapturing(s, &capturing));
    if (capturing != cudaStreamCaptureStatusNone)
        return fail("%s: the stream is being captured into a graph; the copy would run at every replay, outside the engine's order (call it outside the capture)", what);
    CKE(device_memory_refusal(e, what, arg, data));
    if (mask) CKE(device_memory_refusal(e, what, "replicas", mask));
    if (!rows) return 0;
    CKE(prepare());
    const bool other = s != e->stream;
    if (other) { CK(cudaEventRecord(e->evCaller, s)); CK(cudaStreamWaitEvent(e->stream, e->evCaller, 0)); }
    CKE(copy());
    if (other) { CK(cudaEventRecord(e->evEngine, e->stream)); CK(cudaStreamWaitEvent(s, e->evEngine, 0)); }
    return 0;
}
template <class F>
static int device_call(pbd_engine *e, const char *what, const char *arg, const void *data, const unsigned char *mask, void *stream, F &&copy) {
    return device_call(e, what, arg, data, mask, stream, e->n, [] { return 0; }, copy);
}

extern "C" int pbd_set_attr_device(pbd_engine *e, int attr, const float *src, const unsigned char *replicas, void *stream) {
    if (!e) return fail("pbd_set_attr_device: null engine");
    if (attr < 0 || attr >= kNumAttrs) return fail("pbd_set_attr_device: bad attribute %d", attr);
    return device_call(e, "pbd_set_attr_device", "src", src, replicas, stream, [&] { return pack_attr(e, attr, src, 1, e->batch.K, replicas); });
}
extern "C" int pbd_get_attr_device(pbd_engine *e, int attr, float *dst, void *stream) {
    if (!e) return fail("pbd_get_attr_device: null engine");
    if (attr < 0 || attr >= kNumAttrs) return fail("pbd_get_attr_device: bad attribute %d", attr);
    return device_call(e, "pbd_get_attr_device", "dst", dst, nullptr, stream, [&] { return unpack_attr(e, attr, dst); });
}
extern "C" int pbd_set_masses_device(pbd_engine *e, const float *mass, const unsigned char *replicas, void *stream) {
    if (!e) return fail("pbd_set_masses_device: null engine");
    return device_call(e, "pbd_set_masses_device", "mass", mass, replicas, stream, [&] { return pack_w(e, mass, e->batch.K, replicas); });
}

// ---- external forces (pbd_set_external_forces, pbd_set_external_forces_device) ----------------------------------------------------------
// The table is allocated and zeroed by the first set of the current n and K, so replicas a masked set leaves out have zero force; later
// sets write it in place (k_pack3 through the slot map, .w = 0), so its address -- what a captured step reads -- stays.
static int ensure_forces(pbd_engine *e) {
    if (e->force.p) return 0;
    CKE(e->force.alloc((size_t)e->batch.K * e->n * sizeof(float4)));
    CK(cudaMemsetAsync(e->force.p, 0, e->force.bytes, e->stream));
    return 0;
}
static int pack_forces(pbd_engine *e, const float *f, const unsigned char *mask) {
    k_pack3<<<replica_grid(e, e->batch.K), 256, 0, e->stream>>>(f, (float4 *)e->force.p, e->n, 0, (const unsigned *)e->dSlot.p, mask);
    CK(cudaGetLastError());
    return 0;
}
extern "C" int pbd_set_external_forces(pbd_engine *e, const float *f) {
    if (!e) return fail("pbd_set_external_forces: null engine");
    CKE(use(e));
    if (!f) {  // cleared: the steps go back to the integration without forces
        if (e->force.p) { CK(cudaStreamSynchronize(e->stream)); e->force.release(); }
        return 0;
    }
    if (e->n == 0) return 0;
    CKE(ensure_forces(e));
    CK(cudaMemcpyAsync(e->stage[0].p, f, (size_t)e->batch.K * e->n * 3 * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    CKE(pack_forces(e, (const float *)e->stage[0].p, nullptr));
    CK(cudaStreamSynchronize(e->stream));  // staging buffers are reused by the next call
    return 0;
}
extern "C" int pbd_set_external_forces_device(pbd_engine *e, const float *f, const unsigned char *replicas, void *stream) {
    if (!e) return fail("pbd_set_external_forces_device: null engine");
    return device_call(e, "pbd_set_external_forces_device", "f", f, replicas, stream, e->n, [&] { return ensure_forces(e); },
                       [&] { return pack_forces(e, f, replicas); });
}

// ------------------------------------------------------------------------------------------------------------
// rigid bodies (host arrays are tiny: plain synchronous copies)
// ------------------------------------------------------------------------------------------------------------
// `rows` bodies in the layouts of pbd_set_rigid_bodies -> the device arrays' float4 rows (v / omega may be null: 0)
struct BodyUpload { std::vector<float4> X, Q, V, W, I, Ii; };
static void convert_bodies(size_t rows, const float *mass, const float *x, const float *q, const float *inertia, const float *v, const float *omega, BodyUpload &u) {
    u.X.resize(rows); u.Q.resize(rows); u.V.resize(rows); u.W.resize(rows); u.I.resize(rows); u.Ii.resize(rows);
    for (size_t i = 0; i < rows; i++) {
        const float m = mass[i];
        u.X[i] = make_float4(x[3 * i], x[3 * i + 1], x[3 * i + 2], (m != 0.0f) ? 1.0f / m : 0.0f);
        u.Q[i] = make_float4(q[4 * i + 1], q[4 * i + 2], q[4 * i + 3], q[4 * i]);  // (w,x,y,z) -> (x,y,z,w)
        u.V[i] = v ? make_float4(v[3 * i], v[3 * i + 1], v[3 * i + 2], m) : make_float4(0.f, 0.f, 0.f, m);
        u.W[i] = omega ? make_float4(omega[3 * i], omega[3 * i + 1], omega[3 * i + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        u.I[i] = make_float4(inertia[3 * i], inertia[3 * i + 1], inertia[3 * i + 2], 0.f);
        u.Ii[i] = make_float4(1.0f / inertia[3 * i], 1.0f / inertia[3 * i + 1], 1.0f / inertia[3 * i + 2], 0.f);  // RigidBody::setInertiaTensor (RigidBody.h:416-420)
    }
}
// the converted rows into the body arrays (sized first when `size`), old and last state = the current state (RigidBody::initBody)
static int upload_bodies(pbd_engine *e, const BodyUpload &u, bool size) {
    const size_t b = u.X.size() * sizeof(float4);
    const std::vector<float4> *src[10] = {&u.X, &u.Q, &u.V, &u.W, &u.X, &u.X, &u.Q, &u.Q, &u.I, &u.Ii};
    const std::array<DevBuf *, 10> dst = rb_bufs(e);
    for (int k = 0; k < 10; k++) {
        if (size) CKE(dst[k]->alloc(b));
        // Stream-ordered: the next step enqueued reads the new rows.  The sources are pageable, so the driver has staged them when the
        // call returns and the vectors may go.
        CK(cudaMemcpyAsync(dst[k]->p, src[k]->data(), b, cudaMemcpyHostToDevice, e->stream));
    }
    return 0;
}

extern "C" int pbd_set_rigid_bodies(pbd_engine *e, unsigned n, const float *mass, const float *x, const float *q, const float *inertia,
                                    const float *v, const float *omega) {
    if (!e || (n && (!mass || !x || !q || !inertia))) return fail("pbd_set_rigid_bodies: null argument");
    const std::string why = pbd_b200::batch_refusal(e->batch.K, e->n, e->mode, n, e->host);
    if (!why.empty()) return fail("pbd_set_rigid_bodies: %s", why.c_str());
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    if (n != e->nRb) e->groupsSet = false;  // the colouring covers the bodies
    e->nRb = n; e->rbReplica = false;
    e->rbMass.assign(mass, mass + n); e->rbMassStale = false;
    if (n == 0) return 0;
    BodyUpload u;
    convert_bodies(n, mass, x, q, inertia, v, omega, u);
    CKE(upload_bodies(e, u, true));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

extern "C" int pbd_set_replica_rigid_bodies(pbd_engine *e, unsigned n, const float *mass, const float *x, const float *q, const float *inertia,
                                            const float *v, const float *omega) {
    const char *what = "pbd_set_replica_rigid_bodies";
    if (!e) return fail("%s: null engine", what);
    if (e->batch.K == 1) return fail("%s: a single-scene engine takes its bodies from pbd_set_rigid_bodies (pbd_set_replicas first)", what);
    if (n && (!mass || !x || !q || !inertia)) return fail("%s: null argument", what);
    const size_t rows = (size_t)e->batch.K * n;
    if (rows >= (1ull << 31)) return fail("%s: %u replicas of %u bodies exceed 2^31 bodies", what, e->batch.K, n);
    const std::string why = pbd_b200::batch_refusal(e->batch.K, e->n, e->mode, n, e->host, true);
    if (!why.empty()) return fail("%s: %s", what, why.c_str());
    CKE(use(e));
    BodyUpload u;
    convert_bodies(rows, mass, x, q, inertia, v, omega, u);
    // the same n: copies in stream order into arrays that keep their address (no re-plan, no new graph capture); else what
    // pbd_set_rigid_bodies does
    const bool keep = e->rbReplica && n == e->nRb;
    if (!keep) {
        CK(cudaStreamSynchronize(e->stream));
        if (n != e->nRb) e->groupsSet = false;
        e->nRb = n; e->rbReplica = true;
    }
    e->rbMass.assign(mass, mass + rows); e->rbMassStale = false;
    return rows ? upload_bodies(e, u, !keep) : 0;
}

extern "C" int pbd_get_rigid_bodies(pbd_engine *e, float *x, float *q, float *v, float *omega) {
    if (!e) return fail("null engine");
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    const size_t n = (size_t)e->batch.K * e->nRb;  // every replica's
    if (n == 0) return 0;
    std::vector<float4> t(n);
    const size_t b = n * sizeof(float4);
    if (x) { CK(cudaMemcpy(t.data(), e->rbX.p, b, cudaMemcpyDeviceToHost)); for (size_t i = 0; i < n; i++) { x[3 * i] = t[i].x; x[3 * i + 1] = t[i].y; x[3 * i + 2] = t[i].z; } }
    if (q) { CK(cudaMemcpy(t.data(), e->rbQ.p, b, cudaMemcpyDeviceToHost)); for (size_t i = 0; i < n; i++) { q[4 * i] = t[i].w; q[4 * i + 1] = t[i].x; q[4 * i + 2] = t[i].y; q[4 * i + 3] = t[i].z; } }
    if (v) { CK(cudaMemcpy(t.data(), e->rbV.p, b, cudaMemcpyDeviceToHost)); for (size_t i = 0; i < n; i++) { v[3 * i] = t[i].x; v[3 * i + 1] = t[i].y; v[3 * i + 2] = t[i].z; } }
    if (omega) { CK(cudaMemcpy(t.data(), e->rbW.p, b, cudaMemcpyDeviceToHost)); for (size_t i = 0; i < n; i++) { omega[3 * i] = t[i].x; omega[3 * i + 1] = t[i].y; omega[3 * i + 2] = t[i].z; } }
    return 0;
}

// ---- rigid-body state in device memory (pbd_set_rigid_bodies_device, pbd_get_rigid_bodies_device): device_call's stream contract -------
static RbState rb_state(const pbd_engine *e);
// the optional arrays of a device body call: device memory of the engine's device, checked before anything is enqueued
static int body_arrays_refusal(const pbd_engine *e, const char *what, std::initializer_list<std::pair<const char *, const void *>> arrays) {
    for (const auto &a : arrays) if (a.second) CKE(device_memory_refusal(e, what, a.first, a.second));
    return 0;
}
extern "C" int pbd_set_rigid_bodies_device(pbd_engine *e, const float *mass, const float *x, const float *q, const float *inertia, const float *v,
                                           const float *omega, const unsigned char *replicas, void *stream) {
    const char *what = "pbd_set_rigid_bodies_device";
    if (!e) return fail("%s: null engine", what);
    if (!e->nRb) return fail("%s: the engine holds no rigid bodies (pbd_set_rigid_bodies / pbd_set_replica_rigid_bodies first)", what);
    if (!q) return fail("%s: q == NULL", what);
    CKE(body_arrays_refusal(e, what, {{"q", q}, {"mass", mass}, {"inertia", inertia}, {"v", v}, {"omega", omega}}));
    return device_call(e, what, "x", x, replicas, stream, (size_t)e->batch.K * e->nRb, [] { return 0; }, [&]() -> int {
        k_set_bodies<<<dim3(nblk(e->nRb, 128), e->batch.K), 128, 0, e->stream>>>(rb_state(e), BodyRows{(float *)x, (float *)q, (float *)v, (float *)omega, mass, inertia, replicas});
        CK(cudaGetLastError());
        if (mass) e->rbMassStale = true;
        return 0;
    });
}
extern "C" int pbd_get_rigid_bodies_device(pbd_engine *e, float *x, float *q, float *v, float *omega, void *stream) {
    const char *what = "pbd_get_rigid_bodies_device";
    if (!e) return fail("%s: null engine", what);
    const float *first = x ? x : q ? q : v ? v : omega;
    if (!first) return 0;  // nothing asked for
    CKE(body_arrays_refusal(e, what, {{"x", x}, {"q", q}, {"v", v}, {"omega", omega}}));
    const unsigned rows = e->batch.K * e->nRb;
    return device_call(e, what, x ? "x" : q ? "q" : v ? "v" : "omega", first, nullptr, stream, rows, [] { return 0; }, [&]() -> int {
        k_get_bodies<<<nblk(rows, 128), 128, 0, e->stream>>>(rb_state(e), rows, BodyRows{x, q, v, omega, nullptr, nullptr, nullptr});
        CK(cudaGetLastError());
        return 0;
    });
}

template <class V> static int upload_vec(DevBuf &buf, const V &v, cudaStream_t s) {  // V: std::vector / PodVector of PODs
    typedef typename V::value_type T;
    if (v.empty()) return 0;
    if (buf.alloc(v.size() * sizeof(T))) return 1;
    cudaError_t e = cudaMemcpyAsync(buf.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return fail("upload -> %s", cudaGetErrorString(e));
    e = cudaStreamSynchronize(s);  // the host vector dies with the caller's scope
    if (e != cudaSuccess) return fail("upload sync -> %s", cudaGetErrorString(e));
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// constraints and groups
// ------------------------------------------------------------------------------------------------------------
extern "C" int pbd_clear_constraints(pbd_engine *e) {
    if (!e) return fail("null engine");
    CKE(drop_constraint_materials(e, ~0u));
    for (auto &h : e->host) { h.ids.clear(); h.bodies.clear(); h.params.clear(); }
    e->numConstraints = 0;
    e->groupOff.clear(); e->groupIds.clear(); e->groupsSet = false;
    model_changed(e);
    return 0;
}

// With per-replica rest shapes on, a constraint added later gets its geometry from every replica's kept rest positions when the image is
// planned again.  Checked here, on the host and with the arithmetic of the device derivation (rest_geometry.cuh), so that a constraint some
// replica's rest shape makes degenerate is refused by this call instead of failing the next step.
static int check_added_geometry(pbd_engine *e, int type, unsigned count, const unsigned *bodies, const unsigned *ids) {
    if (!e->batch.restShapes || !count || !e->n || type >= PBD_BALLJOINT) return 0;
    CKE(use(e));
    std::vector<float4> rest((size_t)e->batch.K * e->n);
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy(rest.data(), e->batch.restX.p, rest.size() * sizeof(float4), cudaMemcpyDeviceToHost));
    const int nb = type_shape(type).nBodies;
    for (unsigned r = 0; r < e->batch.K; r++)
        for (unsigned i = 0; i < count; i++) {
            float4 x[4];
            for (int k = 0; k < nb; k++) x[k] = rest[(size_t)r * e->n + bodies[(size_t)i * nb + k]];
            float geo[kMaxGeoColumns], Kp[4];
            bool ok = rest_geometry(type, x, geo);
            if (type == PBD_ISOBENDING || type == PBD_ISOBENDING_XPBD) ok = factor_rank1(geo, Kp) && ok;
            if (!ok)
                return fail("pbd_add_constraints: the rest positions of replica %u make constraint %u (type %d) degenerate; the reference's "
                            "initConstraint would refuse it, and the replicas of a batch share one constraint set", r, ids ? ids[i] : e->numConstraints + i, type);
        }
    return 0;
}

// With per-constraint materials of every replica on for `type`, `count` constraints added: every replica's values of the constraints there
// are stay, the new ones carry the parameters they are added with in every replica (the image planned again gathers them)
static int grow_constraint_materials(pbd_engine *e, int type, unsigned count, const float *params) {
    if (!((e->batch.cmatMask >> type) & 1u) || !count) return 0;
    CKE(use(e));
    const TypeShape s = type_shape(type);
    const PackColumns pc = pack_columns(type);
    const size_t K = e->batch.K, c0 = e->host[type].ids.size(), c1 = c0 + count, w = (size_t)s.nMat * sizeof(float);
    std::vector<float> added(K * count * s.nMat);
    for (size_t r = 0; r < K; r++)
        for (size_t i = 0; i < count; i++)
            for (int k = 0; k < s.nMat; k++) added[(r * count + i) * s.nMat + k] = params[i * s.nParams + pc.mat[k]];
    DevBuf grown;
    CKE(grown.alloc(K * c1 * w));
    CK(cudaMemcpy2DAsync(grown.p, c1 * w, e->dev[type].cmat.p, c0 * w, c0 * w, K, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpy2DAsync((char *)grown.p + c0 * w, c1 * w, added.data(), count * w, count * w, K, cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));  // before the old array is freed
    std::swap(e->dev[type].cmat.p, grown.p); std::swap(e->dev[type].cmat.bytes, grown.bytes);
    return 0;
}

extern "C" int pbd_add_constraints(pbd_engine *e, int type, unsigned count, const unsigned *bodies, const float *params, const unsigned *ids) {
    if (!e) return fail("null engine");
    if (type < 0 || type >= PBD_NUM_TYPES) return fail("pbd_add_constraints: unknown constraint type %d", type);
    if (count && (!bodies || !params)) return fail("pbd_add_constraints: null arrays");
    const TypeShape s = type_shape(type);
    const long long badAt = pbd_b200::bad_body_index(type, bodies, count, e->n, e->nRb);
    if (badAt >= 0) {
        if (is_rb_body(type, (int)(badAt % s.nBodies))) return fail("pbd_add_constraints: rigid-body index %u out of range (%u bodies; call pbd_set_rigid_bodies first)", bodies[badAt], e->nRb);
        return fail("pbd_add_constraints: particle index %u out of range (n=%u)", bodies[badAt], e->n);
    }
    CKE(check_added_geometry(e, type, count, bodies, ids));
    CKE(grow_constraint_materials(e, type, count, params));
    TypeStore &h = e->host[type];
    {
        const size_t b0 = h.ids.size();
        h.ids.resize(b0 + count); h.bodies.resize((b0 + count) * s.nBodies); h.params.resize((b0 + count) * s.nParams);  // uninitialised, filled below
        unsigned *idDst = h.ids.data() + b0, *bDst = h.bodies.data() + b0 * s.nBodies; float *pDst = h.params.data() + b0 * s.nParams;
        const unsigned firstId = e->numConstraints;
        #pragma omp parallel for schedule(static) num_threads(host_threads()) if (count > 50000)
        for (long long i = 0; i < (long long)count; i++) {
            idDst[i] = ids ? ids[i] : firstId + (unsigned)i;
            std::memcpy(bDst + (size_t)i * s.nBodies, bodies + (size_t)i * s.nBodies, sizeof(unsigned) * s.nBodies);
            std::memcpy(pDst + (size_t)i * s.nParams, params + (size_t)i * s.nParams, sizeof(float) * s.nParams);
        }
    }
    e->numConstraints += count;
    e->groupsSet = false;  // any add invalidates the groups (SimulationModel: m_groupsInitialized = false)
    model_changed(e);
    return 0;
}

extern "C" int pbd_set_groups(pbd_engine *e, unsigned nGroups, const unsigned *offsets, const unsigned *ids) {
    if (!e || (nGroups && (!offsets || !ids))) return fail("pbd_set_groups: null argument");
    const unsigned N = e->numConstraints;
    if (nGroups == 0 && N != 0) return fail("pbd_set_groups: %u constraints but no groups", N);
    if (nGroups && offsets[nGroups] != N) return fail("pbd_set_groups: groups cover %u constraints, model has %u", offsets[nGroups], N);
    if (nGroups && offsets[0] != 0) return fail("pbd_set_groups: offsets[0] must be 0");
    for (unsigned g = 0; g < nGroups; g++)
        if (offsets[g] > offsets[g + 1]) return fail("pbd_set_groups: offsets must be non-decreasing (group %u)", g);
    std::vector<unsigned char> seen(N, 0);
    for (unsigned i = 0; i < N; i++) {
        if (ids[i] >= N || seen[ids[i]]) return fail("pbd_set_groups: ids are not a permutation of 0..%u", N);
        seen[ids[i]] = 1;
    }
    e->groupOff.assign(offsets, offsets + nGroups + 1);
    e->groupIds.assign(ids, ids + N);
    if (nGroups == 0) e->groupOff.assign(1, 0u);
    e->groupsSet = true;
    model_changed(e);
    return 0;
}

// insertion-ordered CSR of the constraint bodies (the colouring's input)
static int build_id_csr(pbd_engine *e, std::vector<unsigned> &off, std::vector<unsigned> &bodies) {
    std::vector<std::pair<int, unsigned>> map;
    const std::string err = pbd_b200::build_id_map(e->host, e->numConstraints, map);
    if (!err.empty()) return fail("%s", err.c_str());
    const unsigned N = e->numConstraints;
    off.resize((size_t)N + 1);
    // off = exclusive prefix sum of the body counts (chunked two-pass scan), then every constraint copies its bodies
    const int T = std::max(1, host_threads());
    std::vector<unsigned long long> chunk((size_t)T + 1, 0ull);
    #pragma omp parallel num_threads(T)
    {
        const int t = omp_get_thread_num(), nt = omp_get_num_threads();
        const size_t lo = (size_t)N * t / nt, hi = (size_t)N * (t + 1) / nt;
        unsigned long long sum = 0;
        for (size_t id = lo; id < hi; id++) sum += (unsigned)type_shape(map[id].first).nBodies;
        chunk[(size_t)t + 1] = sum;
        #pragma omp barrier
        #pragma omp single
        for (int k = 0; k < nt; k++) chunk[(size_t)k + 1] += chunk[k];
        unsigned long long run = chunk[t];
        for (size_t id = lo; id < hi; id++) { off[id] = (unsigned)run; run += (unsigned)type_shape(map[id].first).nBodies; }
        if (t == nt - 1) off[N] = (unsigned)run;
    }
    if (N == 0) off[0] = 0;
    bodies.resize(off[N]);
    #pragma omp parallel for schedule(static) num_threads(T)
    for (long long id = 0; id < (long long)N; id++) {
        const int t = map[id].first;
        const int nb = type_shape(t).nBodies;
        std::memcpy(&bodies[off[id]], &e->host[t].bodies[(size_t)map[id].second * nb], sizeof(unsigned) * nb);
    }
    return 0;
}
// colour per constraint -> groups in insertion order (what SimulationModel::getConstraintGroups holds)
static void groups_from_colours(pbd_engine *e, const std::vector<unsigned> &colour, unsigned nColours) {
    const unsigned N = e->numConstraints;
    // stable counting sort by colour: per-thread histograms over contiguous id ranges, then every thread scatters its range
    const int T = std::max(1, host_threads());
    std::vector<unsigned> hist((size_t)T * nColours, 0u), goff(nColours + 1, 0u);
    e->groupIds.resize(N);
    #pragma omp parallel num_threads(T)
    {
        const int t = omp_get_thread_num(), nt = omp_get_num_threads();
        const size_t lo = (size_t)N * t / nt, hi = (size_t)N * (t + 1) / nt;
        unsigned *h = &hist[(size_t)t * nColours];
        for (size_t id = lo; id < hi; id++) h[colour[id]]++;
        #pragma omp barrier
        #pragma omp single
        {
            unsigned run = 0;
            for (unsigned c = 0; c < nColours; c++) {
                goff[c] = run;
                for (int k = 0; k < nt; k++) { const unsigned cntk = hist[(size_t)k * nColours + c]; hist[(size_t)k * nColours + c] = run; run += cntk; }
            }
            goff[nColours] = run;
        }
        for (size_t id = lo; id < hi; id++) e->groupIds[h[colour[id]]++] = (unsigned)id;
    }
    e->groupOff = goff;
    e->groupsSet = true; model_changed(e);
}

// Greedy first fit in insertion order == SimulationModel::initConstraintGroups (Simulation/SimulationModel.cpp:1033-1094);
// the colouring itself is host/pbd_model.cpp:firstFitColouring (shared with the host model mirror).
extern "C" int pbd_color_first_fit(pbd_engine *e) {
    if (!e) return fail("null engine");
    std::vector<unsigned> off, bodies, colour;
    CKE(build_id_csr(e, off, bodies));
    // rigid-body and particle indices share one index space without offset (SimulationModel.cpp:1041,1058,1070)
    const unsigned nColours = pbd_b200::firstFitColouring(e->n + e->nRb, e->numConstraints, off.data(), bodies.data(), colour);
    groups_from_colours(e, colour, nColours);
    return 0;
}

// The same colouring computed on the device (colouring.cuh): identical groups, SURVEY.md section 8 f-3.
extern "C" int pbd_color_first_fit_device(pbd_engine *e, float *ms, unsigned *wavefronts) {
    if (!e) return fail("null engine");
    CKE(use(e));
    const unsigned N = e->numConstraints, V = e->n + e->nRb;
    if (ms) *ms = 0.0f;
    if (wavefronts) *wavefronts = 0;
    if (N == 0) { e->groupOff.assign(1, 0u); e->groupIds.clear(); e->groupsSet = true; model_changed(e); return 0; }
    std::vector<unsigned> off, bodies;
    CKE(build_id_csr(e, off, bodies));
    const unsigned M = (unsigned)bodies.size();
    cudaStream_t s = e->stream;
    // one device allocation for all the work arrays (a dozen cudaMalloc / cudaFree pairs cost more than the colouring kernels of a small scene)
    int endBit = 1; while (endBit < 32 && (1ull << endBit) < (unsigned long long)V) endBit++;
    size_t tmpBytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmpBytes, (const unsigned *)nullptr, (unsigned *)nullptr, (const unsigned *)nullptr, (unsigned *)nullptr, (int)M, 0, endBit, s));
    struct View { void *p = nullptr; };
    View dOff, dBody, dBody4, dNext4, dKeys, dVals, dKeysS, dValsS, dIndeg, dColour, dA, dB, dCnt, dTmp;
    DevBuf dAll, dUsed;
    {
        struct Want { View *v; size_t bytes; } want[] = {{&dOff, ((size_t)N + 1) * sizeof(unsigned)}, {&dBody, (size_t)M * sizeof(unsigned)}, {&dKeys, (size_t)M * sizeof(unsigned)},
            {&dVals, (size_t)M * sizeof(unsigned)}, {&dKeysS, (size_t)M * sizeof(unsigned)}, {&dValsS, (size_t)M * sizeof(unsigned)}, {&dBody4, (size_t)N * sizeof(uint4)},
            {&dNext4, (size_t)N * sizeof(uint4)}, {&dIndeg, (size_t)N * sizeof(unsigned)}, {&dColour, (size_t)N * sizeof(unsigned)}, {&dA, (size_t)N * sizeof(unsigned)},
            {&dB, (size_t)N * sizeof(unsigned)}, {&dCnt, 4 * sizeof(unsigned)}, {&dTmp, tmpBytes}};
        size_t total = 0;
        for (auto &w : want) total += (w.bytes + 255) & ~(size_t)255;
        CKE(dAll.alloc(total));
        size_t at = 0;
        for (auto &w : want) { w.v->p = (char *)dAll.p + at; at += (w.bytes + 255) & ~(size_t)255; }
    }
    CK(cudaMemcpyAsync(dOff.p, off.data(), ((size_t)N + 1) * sizeof(unsigned), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(dBody.p, bodies.data(), (size_t)M * sizeof(unsigned), cudaMemcpyHostToDevice, s));
    cudaEvent_t ev0, ev1;
    CK(cudaEventCreate(&ev0)); CK(cudaEventCreate(&ev1));
    CK(cudaEventRecord(ev0, s));
    // incidence lists: stable sort of (body, incidence) by body, then successor / in-degree of every constraint
    k_colour_expand<<<nblk(N, 256), 256, 0, s>>>((const unsigned *)dOff.p, (const unsigned *)dBody.p, (uint4 *)dBody4.p, (unsigned *)dKeys.p, (unsigned *)dVals.p, N);
    CK(cub::DeviceRadixSort::SortPairs(dTmp.p, tmpBytes, (const unsigned *)dKeys.p, (unsigned *)dKeysS.p, (const unsigned *)dVals.p, (unsigned *)dValsS.p, (int)M, 0, endBit, s));
    CK(cudaMemsetAsync(dNext4.p, 0xff, (size_t)N * sizeof(uint4), s));
    std::vector<unsigned> colour(N);
    unsigned cnt[4] = {0, 0, 0, 0};
    for (unsigned words = 2;; words *= 2) {  // 128 colours to begin with; doubled when a constraint finds none free
        CKE(dUsed.alloc((size_t)V * words * sizeof(unsigned long long)));
        CK(cudaMemsetAsync(dUsed.p, 0, (size_t)V * words * sizeof(unsigned long long), s));
        CK(cudaMemsetAsync(dIndeg.p, 0, (size_t)N * sizeof(unsigned), s));
        CK(cudaMemsetAsync(dCnt.p, 0, 4 * sizeof(unsigned), s));
        k_colour_links<<<nblk(M, 256), 256, 0, s>>>((const unsigned *)dKeysS.p, (const unsigned *)dValsS.p, M, (unsigned *)dNext4.p, (unsigned *)dIndeg.p);
        ColourArgs a{N, V, words, (const uint4 *)dBody4.p, (const uint4 *)dNext4.p, (unsigned *)dIndeg.p, (unsigned long long *)dUsed.p,
                     (unsigned *)dColour.p, (unsigned *)dA.p, (unsigned *)dB.p, (unsigned *)dCnt.p};
        k_colour_seed<<<nblk(N, 256), 256, 0, s>>>(a);
        k_colour_wavefronts<<<1, kColourThreads, 0, s>>>(a);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(cnt, dCnt.p, sizeof(cnt), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        if (!cnt[1]) break;
        if (words >= 1024) return fail("device colouring: more than %u colours needed", words * 64);
    }
    CK(cudaEventRecord(ev1, s));
    CK(cudaMemcpyAsync(colour.data(), dColour.p, (size_t)N * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    float t = 0.0f; cudaEventElapsedTime(&t, ev0, ev1);
    cudaEventDestroy(ev0); cudaEventDestroy(ev1);
    if (cnt[2] != N) return fail("device colouring: coloured %u of %u constraints (dependency cycle?)", cnt[2], N);
    unsigned nColours = 0;
    #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(max : nColours)
    for (long long id = 0; id < (long long)N; id++) nColours = std::max(nColours, colour[id] + 1);
    groups_from_colours(e, colour, nColours);
    if (ms) *ms = t;
    if (wavefronts) *wavefronts = cnt[3];
    return 0;
}

extern "C" int pbd_get_num_groups(pbd_engine *e, unsigned *nGroups) {
    if (!e || !nGroups) return fail("null argument");
    if (!e->groupsSet) return fail("groups not initialised (call pbd_set_groups or pbd_color_first_fit)");
    *nGroups = (unsigned)e->groupOff.size() - 1;
    return 0;
}
extern "C" int pbd_get_groups(pbd_engine *e, unsigned *offsets, unsigned *ids) {
    if (!e || !offsets || !ids) return fail("null argument");
    if (!e->groupsSet) return fail("groups not initialised");
    memcpy(offsets, e->groupOff.data(), e->groupOff.size() * sizeof(unsigned));
    memcpy(ids, e->groupIds.data(), e->groupIds.size() * sizeof(unsigned));
    return 0;
}

extern "C" int pbd_set_params(pbd_engine *e, float dt, unsigned subSteps, unsigned maxIter, int velMethod, const float gravity[3]) {
    if (!e) return fail("null engine");
    if (subSteps < 1) return fail("subSteps must be >= 1 (TimeStepController.cpp:50)");
    if (maxIter < 1) return fail("maxIterations must be >= 1 (TimeStepController.cpp:55)");
    if (velMethod != 0 && velMethod != 1) return fail("velocityUpdateMethod must be 0 or 1");
    if (!(dt > 0.0f)) return fail("time step size must be positive");
    e->dt = dt; e->subSteps = subSteps; e->maxIter = maxIter; e->velMethod = velMethod;
    if (gravity) { e->g[0] = gravity[0]; e->g[1] = gravity[1]; e->g[2] = gravity[2]; }
    return 0;
}
extern "C" int pbd_set_mode(pbd_engine *e, int mode) {
    if (!e) return fail("null engine");
    if (mode != PBD_MODE_GRAPH && mode != PBD_MODE_RESIDENT && mode != PBD_MODE_LAUNCH && mode != PBD_MODE_JACOBI && mode != PBD_MODE_AUTO) return fail("unknown solver mode %d", mode);
    const std::string why = pbd_b200::batch_refusal(e->batch.K, e->n, mode, e->nRb, e->host, e->rbReplica);
    if (!why.empty()) return fail("pbd_set_mode: %s", why.c_str());
    e->mode = mode;
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// the device image: planned on the host (host/image_plan.cpp), uploaded here
// ------------------------------------------------------------------------------------------------------------
template <unsigned M, bool BATCH, class F> static int resident_kernel(bool single, F &&f) {
    return single ? f(k_step_resident<M, resident_threads(M, BATCH), true, BATCH>) : f(k_step_resident<M, resident_threads(M, BATCH), false, BATCH>);
}
template <unsigned M, class F> static int resident_kernel(bool single, bool batch, F &&f) {
    return batch ? resident_kernel<M, true>(single, f) : resident_kernel<M, false>(single, f);
}
// the compiled instantiations of k_step_resident: F(kernel pointer) for a type mask, one CTA per cluster or not, a replica batch or not
template <class F> static int with_resident_kernel(unsigned mask, unsigned C, bool batch, F &&f) {
    const bool single = (C == 1);
    switch (mask) {
    case kMaskClothXPBD: return resident_kernel<kMaskClothXPBD>(single, batch, f);
    case kMaskCloth: return resident_kernel<kMaskCloth>(single, batch, f);
    case kMaskLight: return resident_kernel<kMaskLight>(single, batch, f);
    case kMaskFem: return resident_kernel<kMaskFem>(single, batch, f);
    case kMaskSolid: return resident_kernel<kMaskSolid>(single, batch, f);
    default: return resident_kernel<kMaskAll>(single, batch, f);
    }
}

static void resident_launch_config(unsigned mask, unsigned C, bool batch, unsigned grid, size_t smem, cudaStream_t s, cudaLaunchConfig_t &cfg, cudaLaunchAttribute *attr) {
    cfg = cudaLaunchConfig_t{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(resident_threads(mask, batch)); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
}

// how many clusters of C CTAs (one CTA per SM, `smem` bytes each) of the instantiation for `mask` the device keeps resident at the same time
static int resident_max_clusters(const pbd_engine *e, unsigned mask, unsigned C, size_t smem, int *out) {
    return with_resident_kernel(mask, C, e->batch.K > 1, [&](auto kernel) -> int {
        CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxDynamicSmem));
        CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
        cudaLaunchConfig_t cfg; cudaLaunchAttribute attr[1];
        resident_launch_config(mask, C, e->batch.K > 1, C, smem, e->stream, cfg, attr);
        cudaError_t err = cudaOccupancyMaxActiveClusters(out, kernel, &cfg);
        if (err != cudaSuccess) { cudaGetLastError(); *out = 0; }
        return 0;
    });
}
// colour groups when none were given: the reference-order-preserving first fit on the GPU (colouring.cuh), the host version as the fallback
static int colour_if_needed(pbd_engine *e) {
    if (e->groupsSet) return 0;
    if (pbd_color_first_fit_device(e, nullptr, nullptr)) CKE(pbd_color_first_fit(e));
    return 0;
}

// The planned image in its one allocation (pbd_b200::image_layout): `ptr` pointed at every array (nullptr: the arrays without bytes), each
// copied to its place, the zeroed regions -- the layout puts them last -- cleared by one memset.  Returns once the copies have read the plan.
static int upload_image(pbd_engine *e, const pbd_b200::ImagePlan &plan, pbd_b200::ImagePointers &ptr) {
    const pbd_b200::ImageLayout l = pbd_b200::image_layout(plan, e->batch.K);
    CKE(e->image.alloc(l.bytes));
    ptr = pbd_b200::ImagePointers{};
    size_t zeroed = l.bytes;
    for (const pbd_b200::ImageArray &a : l.arrays) {
        if (!a.bytes) continue;
        char *at = (char *)e->image.p + a.offset;
        std::memcpy((char *)&ptr + a.slot, &at, sizeof(at));
        if (a.zeroed) zeroed = std::min(zeroed, a.offset);
        else CK(cudaMemcpyAsync(at, a.src, a.bytes, cudaMemcpyHostToDevice, e->stream));
    }
    if (zeroed < l.bytes) CK(cudaMemsetAsync((char *)e->image.p + zeroed, 0, l.bytes - zeroed, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}
// one type of the uploaded image: its TypeArrays and rest tables, what of them is not an array, and a batch's shared material rows
static int upload_type(pbd_engine *e, int t, pbd_b200::TypePlan &p, const pbd_b200::ImagePointers &ptr) {
    DevType &d = e->dev[t];
    const unsigned cnt = (unsigned)p.order.size();
    d.count = cnt;
    e->stats.constraints_per_type[t] = cnt;
    d.arrays = ptr.types[t]; d.rest = ptr.rest[t];
    d.order.swap(p.order);
    if (cnt == 0) return 0;
    TypeArrays &a = d.arrays;
    for (int k = 0; k < kMaxMat; k++) a.matU[k] = p.matU[k];
    a.variant = p.variant;
    if (e->batch.K > 1 && type_shape(t).nMat && !((e->batch.matMask >> t) & 1u)) CKE(write_replica_materials(e, t, a.matU, 0));  // the shared parameters, for every replica
    if (t == PBD_BALLJOINT || t == PBD_RB_PARTICLE_BALLJOINT) {
        a.rbX = (float4 *)e->rbX.p; a.rbQ = (float4 *)e->rbQ.p; a.rbIinv = (const float4 *)e->rbIinv.p;
    }
    return 0;
}

// ---- per-replica rest shapes of a batch (pbd_set_replica_rest_positions) ------------------------------------------------------
template <class F> static int with_geometry_type(int type, F &&f) {
    PBD_FOR_TYPE(kMaskAll & ~(type_bit(PBD_BALLJOINT) | type_bit(PBD_RB_PARTICLE_BALLJOINT)), type, return f(std::integral_constant<int, T>{});)
    return fail("constraint type %d has no rest geometry of particles", type);
}
struct GeoBufs { DevBuf gv[kMaxGeoV], gs[kMaxGeoS]; };  // one type's geometry arrays in the image's layout
// Every particle type's geometry of the K replicas derived from `rest` (K x n float4 by host index, k_pack_rest) on the device: packed into
// the image's layout in fresh[type], or with `rows` type rowsType's parameter-layout geometry rows (K x count x num_geo).  *bad: the
// first constraint refused (replica << 32 | insertion id), ~0 for none.
static int derive_geometry(pbd_engine *e, const float4 *rest, GeoBufs *fresh, int rowsType, float *rows, unsigned long long *bad) {
    DevBuf failed;
    CKE(failed.alloc(sizeof(unsigned long long)));
    CK(cudaMemsetAsync(failed.p, 0xff, sizeof(unsigned long long), e->stream));
    for (int t = 0; t < PBD_BALLJOINT; t++) {
        DevType &d = e->dev[t];
        if (!d.count || (rows && t != rowsType)) continue;
        DeriveArgs a{};
        a.rest = rest; a.n = e->n; a.count = d.count;
        a.bodies = d.rest.bodies; a.ids = d.rest.ids; a.local = d.rest.local;
        a.clusters = d.arrays.gv[5]; a.variant = d.arrays.variant; a.rows = rows; a.fail = (unsigned long long *)failed.p;
        if (!rows) {
            const size_t cnt = (size_t)e->batch.K * d.count;
            for (int k = 0; k < kMaxGeoV; k++) if (d.arrays.gv[k]) { CKE(fresh[t].gv[k].alloc(pbd_b200::padded_bytes(cnt * sizeof(float4)))); a.gv[k] = (float4 *)fresh[t].gv[k].p; }
            for (int k = 0; k < kMaxGeoS; k++) if (d.arrays.gs[k]) { CKE(fresh[t].gs[k].alloc(pbd_b200::padded_bytes(cnt * sizeof(float)))); a.gs[k] = (float *)fresh[t].gs[k].p; }
        }
        CKE(with_geometry_type(t, [&](auto T) -> int {
            k_derive_geometry<decltype(T)::value><<<dim3(nblk(d.count, 128), e->batch.K), 128, 0, e->stream>>>(a);
            CK(cudaGetLastError());
            return 0;
        }));
    }
    CK(cudaMemcpyAsync(bad, failed.p, sizeof(*bad), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}
// The geometry derived from `rest` becomes what the projections read -- only when no constraint refuses it: otherwise the error names the
// first replica and constraint, and nothing has changed.  It is copied into the live arrays in stream order, so that they keep their
// address and the captured graph stays valid.  The scratch arrays are as large as the live ones: they are freed on return.
static int apply_replica_geometry(pbd_engine *e, const float4 *rest, const char *what) {
    unsigned long long bad = ~0ull;
    GeoBufs fresh[PBD_BALLJOINT];
    CKE(derive_geometry(e, rest, fresh, -1, nullptr, &bad));
    if (bad != ~0ull) {
        const unsigned rep = (unsigned)(bad >> 32), id = (unsigned)bad;
        int type = -1;
        for (int t = 0; t < PBD_NUM_TYPES && type < 0; t++)
            for (unsigned id2 : e->host[t].ids) if (id2 == id) { type = t; break; }
        return fail("%s: the rest positions of replica %u make constraint %u (type %d) degenerate; the reference's initConstraint would refuse "
                    "it, and the replicas of a batch share one constraint set", what, rep, id, type);
    }
    for (int t = 0; t < PBD_BALLJOINT; t++) {
        DevType &d = e->dev[t];
        const size_t cnt = (size_t)e->batch.K * d.count;
        if (!cnt) continue;
        for (int k = 0; k < kMaxGeoV; k++)
            if (d.arrays.gv[k]) { CKE(d.repGv[k].alloc(pbd_b200::padded_bytes(cnt * sizeof(float4)))); CK(cudaMemcpyAsync(d.repGv[k].p, fresh[t].gv[k].p, cnt * sizeof(float4), cudaMemcpyDeviceToDevice, e->stream)); }
        for (int k = 0; k < kMaxGeoS; k++)
            if (d.arrays.gs[k]) { CKE(d.repGs[k].alloc(pbd_b200::padded_bytes(cnt * sizeof(float)))); CK(cudaMemcpyAsync(d.repGs[k].p, fresh[t].gs[k].p, cnt * sizeof(float), cudaMemcpyDeviceToDevice, e->stream)); }
    }
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

// ---- per-constraint materials of every replica of a batch (pbd_set_replica_constraint_materials) ---------------------------------
// The device-ordered arrays of type t (sized here: they keep their address while K and count stay) <- `src`, K x count rows of nMat floats in
// the order the constraints were added, through the image's device position -> insertion position map (restTables); with `keep` the rows
// also go to DevType::cmat.  mask: the replicas written (nullptr: all).  Enqueued on the engine stream, no host synchronisation.
static int gather_materials(pbd_engine *e, int t, const float *src, bool keep, const unsigned char *mask) {
    DevType &d = e->dev[t];
    if (!d.count) return 0;
    if (!d.rest.local) return fail("per-constraint materials of type %d: the image lacks the device order tables", t);
    const size_t cnt = (size_t)e->batch.K * d.count;
    GatherMatArgs g{};
    g.src = src; g.keep = keep ? (float *)d.cmat.p : nullptr; g.local = d.rest.local; g.mask = mask; g.count = d.count; g.nMat = type_shape(t).nMat;
    for (int k = 0; k < g.nMat; k++) { CKE(d.repMat[k].alloc(pbd_b200::padded_bytes(cnt * sizeof(float)))); g.dst[k] = (float *)d.repMat[k].p; }
    k_gather_materials<<<dim3(nblk(d.count, 128), e->batch.K), 128, 0, e->stream>>>(g);
    CK(cudaGetLastError());
    return 0;
}

template <class... V> static void append_bytes(std::vector<unsigned char> &key, const V &...v) {
    static_assert((std::is_scalar_v<std::remove_all_extents_t<V>> && ...), "padding bytes would make equal states compare unequal");
    size_t at = key.size();
    key.resize(at + (sizeof(V) + ...));
    ((std::memcpy(&key[at], &v, sizeof(V)), at += sizeof(V)), ...);
}
// Everything the image is planned and uploaded from; the joint arrays hold the rigid-body pointers.  The mode counts where it asks for a
// tiled image: AUTO then falls back to graph where the resident mode refuses the model, RESIDENT fails.  Left out: the rest positions the
// tiling bisects (they decide how fast a tiled image runs, not what it computes) and PBD_B200_CLUSTERS (a knob read at planning time).
static std::vector<unsigned char> image_key(const pbd_engine *e) {
    std::vector<unsigned char> key;
    const bool tiled = pbd_b200::preferred_mode(e->mode, e->host, e->n, e->numConstraints, e->batch.K) == PBD_MODE_RESIDENT;
    append_bytes(key, e->modelGen, e->n, e->nRb, e->rbReplica, e->rbX.p, e->rbQ.p, e->rbIinv.p, e->batch.K, tiled ? e->mode : -1, rest_tables(e));
    return key;
}

// The device image of the requested mode (the planner resolves PBD_MODE_AUTO), planned again whenever image_key changes: colour groups
// made where none were given, the planner's inputs gathered, the plan uploaded.
static int flatten(pbd_engine *e) {
    pbd_b200::Lap lap;
    CKE(colour_if_needed(e));  // before the key: the groups it makes are the model's from now on
    std::vector<unsigned char> key = image_key(e);
    if (key == e->imageKey) return 0;
    CKE(use(e));
    // Work still pending on the engine stream -- a device get or set enqueued behind a caller's stream included -- reads the particle
    // arrays and the slot map that relayout replaces, and upload_slot_map's copy is not ordered against the engine stream.
    CK(cudaStreamSynchronize(e->stream));
    e->imageGen++;
    e->stats.images_planned++;
    std::vector<float4> x0;  // resident: rest positions by host index
    if (pbd_b200::preferred_mode(e->mode, e->host, e->n, e->numConstraints, e->batch.K) == PBD_MODE_RESIDENT && e->n) {
        std::vector<float4> raw(e->n);
        CK(cudaMemcpy(raw.data(), attr_ptr(e, PBD_ATTR_X0), (size_t)e->n * sizeof(float4), cudaMemcpyDeviceToHost));
        x0.resize(e->n);
        for (unsigned i = 0; i < e->n; i++) x0[i] = raw[e->slot[i]];
    }
    lap("colouring + rest positions");
    pbd_b200::PlanInput in{e->host, e->numConstraints, e->n, e->nRb, &e->groupOff, &e->groupIds, e->mode, x0.data(), 0u, 0u, e->smCount, nullptr,
                           rest_tables(e), e->batch.K, e->rbReplica};
    if (const char *g = getenv("PBD_B200_CLUSTERS")) {  // development knob "GxC"
        unsigned gg = 0, cc = 0;
        if (sscanf(g, "%ux%u", &gg, &cc) == 2 && gg >= 1 && cc >= 1 && cc <= (unsigned)kMaxClusterCtas && (cc & (cc - 1)) == 0) { in.forcedG = gg; in.forcedC = cc; }
    }
    in.maxClusters = [&](unsigned mask, unsigned C, size_t smem) { int mc = 0; return resident_max_clusters(e, mask, C, smem, &mc) ? 0 : mc; };
    pbd_b200::ImagePlan plan;
    const std::string err = pbd_b200::plan_image(in, plan);
    if (!plan.residentRefusal.empty() && verbose()) fprintf(stderr, "[pbd_b200] auto mode: resident refused (%s), using the graph mode\n", plan.residentRefusal.c_str());
    if (!err.empty()) return fail("%s", err.c_str());
    CKE(relayout(e, plan.slot));
    pbd_b200::ImagePointers ptr;
    CKE(upload_image(e, plan, ptr));
    for (int t = 0; t < PBD_NUM_TYPES; t++) CKE(upload_type(e, t, plan.types[t], ptr));
    e->buckets.swap(plan.buckets);
    e->tables = ptr.tables;
    e->res = plan.res;
    CK(cudaStreamSynchronize(e->stream));
    lap("relayout + upload");
    if (e->batch.restShapes) CKE(apply_replica_geometry(e, (const float4 *)e->batch.restX.p, "pbd_set_replica_rest_positions (image planned again)"));  // the new image's geometry, from the rest positions the override was given
    for (int t = 0; t < PBD_NUM_TYPES; t++)  // the new image's device order of the per-constraint materials
        if ((e->batch.cmatMask >> t) & 1u) CKE(gather_materials(e, t, (const float *)e->dev[t].cmat.p, false, nullptr));

    e->stats.num_constraints = e->numConstraints;  // per replica, like num_particles
    e->stats.num_groups = (unsigned)e->groupOff.size() - 1;
    e->stats.num_buckets = (unsigned)e->buckets.size();
    e->imageKey.swap(key);
    return 0;
}
// What the current image runs in: a tiled image the resident mode, any other the requested mode, PBD_MODE_AUTO resolved to graph.
static int active_mode(const pbd_engine *e) { return e->res.G ? PBD_MODE_RESIDENT : e->mode == PBD_MODE_AUTO ? PBD_MODE_GRAPH : e->mode; }

extern "C" int pbd_get_mode(pbd_engine *e, int *requested, int *active) {
    if (!e) return fail("null engine");
    CKE(flatten(e));
    if (requested) *requested = e->mode;
    if (active) *active = active_mode(e);
    return 0;
}

// The rest positions go to a buffer of their own (and PBD_ATTR_X0) only after the geometry derived from them has been accepted; the engine
// keeps them, so that an image planned again (constraints added, another mode) derives its geometry from them too.
extern "C" int pbd_set_replica_rest_positions(pbd_engine *e, const float *x0) {
    CKE(replica_params_refusal(e, "pbd_set_replica_rest_positions"));
    CKE(use(e));
    if (!x0) { drop_replica_geometry(e); return 0; }
    e->batch.restTables = true;  // planned again, if need be, with the bodies the derivation reads
    CKE(flatten(e));  // the device order of the constraints the geometry is derived for
    for (int t = 0; t < PBD_BALLJOINT; t++)  // the resident kernel addresses replica r's geometry as i + r count in 32 bits
        if ((unsigned long long)e->batch.K * e->dev[t].count >= (1ull << 32))
            return fail("pbd_set_replica_rest_positions: %u replicas of %u constraints of type %d exceed 2^32 geometry rows", e->batch.K, e->dev[t].count, t);
    if (e->n) {
        DevBuf rest;
        CKE(rest.alloc((size_t)e->batch.K * e->n * sizeof(float4)));
        CK(cudaMemcpyAsync(e->stage[0].p, x0, (size_t)e->batch.K * e->n * 3 * sizeof(float), cudaMemcpyHostToDevice, e->stream));
        k_pack_rest<<<replica_grid(e, e->batch.K), 256, 0, e->stream>>>((const float *)e->stage[0].p, attr_ptr(e, PBD_ATTR_X), (float4 *)rest.p, e->n, (const unsigned *)e->dSlot.p);
        CK(cudaGetLastError());
        CKE(apply_replica_geometry(e, (const float4 *)rest.p, "pbd_set_replica_rest_positions"));
        std::swap(e->batch.restX.p, rest.p); std::swap(e->batch.restX.bytes, rest.bytes);
        CKE(upload_attr(e, PBD_ATTR_X0, nullptr, 1, e->batch.K, e->stage[0], e->stream));  // PBD_ATTR_X0 of every replica, from x0 still in stage[0]
        CK(cudaStreamSynchronize(e->stream));
    }
    e->batch.restShapes = true;
    return 0;
}

// The values replica r's constraints of `type` are stepped with while the type has no per-constraint override: its rows (matMask) or the
// shared parameters, K x count x nMat in the order the constraints were added.  Reading the rows back synchronises.
static int stepped_materials(pbd_engine *e, int type, std::vector<float> &out) {
    const TypeStore &h = e->host[type];
    const TypeShape s = type_shape(type);
    const PackColumns pc = pack_columns(type);
    const size_t K = e->batch.K, cnt = h.ids.size();
    std::vector<float> rows;
    if ((e->batch.matMask >> type) & 1u) {
        rows.resize(K * s.nMat);
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaMemcpy2D(rows.data(), s.nMat * sizeof(float), (const float *)e->batch.mat.p + mat_offset(type), kMatRowFloats * sizeof(float),
                        s.nMat * sizeof(float), K, cudaMemcpyDeviceToHost));
    }
    out.resize(K * cnt * s.nMat);
    for (size_t r = 0; r < K; r++)
        for (size_t i = 0; i < cnt; i++)
            for (int k = 0; k < s.nMat; k++) out[(r * cnt + i) * s.nMat + k] = rows.empty() ? h.params[i * s.nParams + pc.mat[k]] : rows[r * s.nMat + k];
    return 0;
}
static int constraint_materials_refusal(const pbd_engine *e, const char *what, int type) {
    CKE(replica_params_refusal(e, what));
    if (type < 0 || type >= PBD_NUM_TYPES) return fail("%s: unknown constraint type %d", what, type);
    if (type_shape(type).nMat == 0) return fail("%s: constraint type %d has no material parameters", what, type);
    const size_t cnt = e->host[type].ids.size();
    if (!cnt) return fail("%s: the model has no constraints of type %d", what, type);
    if ((unsigned long long)e->batch.K * cnt >= (1ull << 32))  // the resident kernel addresses replica r's materials as i + r count in 32 bits
        return fail("%s: %u replicas of %zu constraints of type %d exceed 2^32 material rows", what, e->batch.K, cnt, type);
    return 0;
}
// Type `type` takes its materials from DevType::cmat from now on.  Switching the override on (may synchronise): `fill` -- the rows keep the
// values the replicas were stepped with (a masked call leaves the other replicas as they were) -- and the image planned with the tables the
// gather reads.  Every call: the image brought up to date, so that the gather runs in its device order.
static int constraint_materials_on(pbd_engine *e, int type, bool fill) {
    const unsigned bit = 1u << type;
    if (!(e->batch.cmatMask & bit)) {
        const size_t bytes = (size_t)e->batch.K * e->host[type].ids.size() * type_shape(type).nMat * sizeof(float);
        CKE(e->dev[type].cmat.alloc(bytes));
        if (fill) {
            std::vector<float> now;
            CKE(stepped_materials(e, type, now));
            CK(cudaMemcpyAsync(e->dev[type].cmat.p, now.data(), bytes, cudaMemcpyHostToDevice, e->stream));
            CK(cudaStreamSynchronize(e->stream));  // `now` dies here
        }
        if (e->batch.matMask & bit) {  // rows off: the table holds the shared parameters again (the resident batch kernels read it)
            CKE(write_replica_materials(e, type, e->dev[type].arrays.matU, 0));
            e->batch.matMask &= ~bit;
        }
        e->batch.cmatMask |= bit;  // image_key: planned again with the tables, if they were not there
        CKE(flatten(e));
        CKE(gather_materials(e, type, (const float *)e->dev[type].cmat.p, false, nullptr));  // (where flatten did not plan: the values now in force)
    }
    return flatten(e);
}

extern "C" int pbd_set_replica_constraint_materials(pbd_engine *e, int type, const float *mat) {
    const char *what = "pbd_set_replica_constraint_materials";
    CKE(constraint_materials_refusal(e, what, type));
    CKE(use(e));
    if (!mat) {  // the shared parameters
        CKE(drop_constraint_materials(e, 1u << type));
        return pbd_set_replica_materials(e, type, nullptr);
    }
    CKE(constraint_materials_on(e, type, false));
    DevType &d = e->dev[type];
    CK(cudaMemcpyAsync(d.cmat.p, mat, (size_t)e->batch.K * d.count * type_shape(type).nMat * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    return gather_materials(e, type, (const float *)d.cmat.p, false, nullptr);
}
extern "C" int pbd_set_replica_constraint_materials_device(pbd_engine *e, int type, const float *mat, const unsigned char *replicas, void *stream) {
    const char *what = "pbd_set_replica_constraint_materials_device";
    CKE(constraint_materials_refusal(e, what, type));
    return device_call(e, what, "mat", mat, replicas, stream, e->n, [&] { return constraint_materials_on(e, type, replicas != nullptr); },
                       [&] { return gather_materials(e, type, mat, true, replicas); });
}
extern "C" int pbd_get_replica_materials(pbd_engine *e, int type, float *dst) {
    if (!e || !dst) return fail("pbd_get_replica_materials: null argument");
    if (type < 0 || type >= PBD_NUM_TYPES) return fail("pbd_get_replica_materials: unknown constraint type %d", type);
    if (type_shape(type).nMat == 0) return fail("pbd_get_replica_materials: constraint type %d has no material parameters", type);
    CKE(use(e));
    const DevType &d = e->dev[type];
    if ((e->batch.cmatMask >> type) & 1u) {
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaMemcpy(dst, d.cmat.p, (size_t)e->batch.K * e->host[type].ids.size() * type_shape(type).nMat * sizeof(float), cudaMemcpyDeviceToHost));
        return 0;
    }
    std::vector<float> now;
    CKE(stepped_materials(e, type, now));
    if (!now.empty()) memcpy(dst, now.data(), now.size() * sizeof(float));
    return 0;
}

extern "C" int pbd_get_replica_geometry(pbd_engine *e, int type, float *dst) {
    if (!e || !dst) return fail("pbd_get_replica_geometry: null argument");
    if (type < 0 || type >= PBD_BALLJOINT) return fail("pbd_get_replica_geometry: constraint type %d has no rest geometry of particles", type);
    CKE(use(e)); CKE(flatten(e));
    const unsigned cnt = e->dev[type].count;
    const int nGeo = num_geo(type), g0 = geo_first(type), np = type_shape(type).nParams;
    if (cnt == 0) return 0;
    const size_t one = (size_t)cnt * nGeo;
    if (!e->batch.restShapes) {  // the shared geometry, for every replica
        const TypeStore &h = e->host[type];
        for (size_t i = 0; i < cnt; i++)
            for (int j = 0; j < nGeo; j++) dst[i * nGeo + j] = h.params[i * np + g0 + j];
        for (unsigned r = 1; r < e->batch.K; r++) memcpy(dst + r * one, dst, one * sizeof(float));
        return 0;
    }
    DevBuf rows;
    CKE(rows.alloc((size_t)e->batch.K * one * sizeof(float)));
    unsigned long long bad = ~0ull;
    CKE(derive_geometry(e, (const float4 *)e->batch.restX.p, nullptr, type, (float *)rows.p, &bad));
    CK(cudaMemcpy(dst, rows.p, (size_t)e->batch.K * one * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// step drivers
// ------------------------------------------------------------------------------------------------------------
// Block size of a projection launch (kProjectThreads is only the compiled upper bound).  128 threads rather than 256: more,
// smaller CTAs ramp up and drain faster in each dependent launch (H100 80GB HBM3, 400 W, graph mode: cfg3 8.48 ms against 11.14 ms
// with 256; cfg2 5.60 / 5.57 ms); a launch that would not even give every SM one CTA is spread
// further, down to one warp per CTA, because such phases are pure latency chains (cfg1, cfg3).
static unsigned project_block(const pbd_engine *e, unsigned count) {
    const unsigned perSM = (count + (unsigned)e->smCount - 1) / (unsigned)e->smCount;
    return std::max(32u, std::min(128u, (perSM + 31u) & ~31u));
}

// One kernel of a step.  With `pdl` the launch carries the programmatic-stream-serialization attribute, so that the whole step is one
// programmatic dependency chain (kernels.cuh); pbd_profile_step launches without it, so that each kernel's duration is its own.
template <typename... KArgs, typename... Args>
static cudaError_t launch_step_kernel(void (*kernel)(KArgs...), dim3 grid, unsigned block, cudaStream_t s, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3(block); cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// (constraint type, layout variant) -> f(T, VAR): the compile-time arguments of the k_project / k_project_jacobi instantiation
template <int V> using IntC = std::integral_constant<int, V>;
template <class F> static int with_project_type(int type, int variant, F &&f) {
    PBD_FOR_TYPE(kMaskAll, type,
        if constexpr (T == PBD_ISOBENDING || T == PBD_ISOBENDING_XPBD)
            if (variant) return f(IntC<T>{}, IntC<1>{});
        return f(IntC<T>{}, IntC<0>{});)
    return fail("no kernel for constraint type %d", type);
}

// A batch's projection launches run replica blockIdx.y (the BATCH instantiations); their block size follows the whole batch's count.
static int launch_bucket(pbd_engine *e, const Bucket &b, float h, int iterZero, cudaStream_t s, bool pdl) {
    const TypeArrays a = batch_arrays(e, b.type);
    const unsigned block = project_block(e, b.count * e->batch.K);
    const ReplicaStrides rs{e->n, {e->dev[b.type].count}, {replica_mat(e, b.type)}, {replica_geo(e, b.type)}, {replica_cmat(e, b.type)}, e->nRb};
    return with_project_type(b.type, a.variant, [&](auto T, auto V) -> int {
        constexpr int TT = decltype(T)::value, VAR = decltype(V)::value;
        if (e->batch.K > 1) CK(launch_step_kernel(k_project<TT, VAR, true>, dim3(nblk(b.count, block), e->batch.K), block, s, pdl, attr_ptr(e, PBD_ATTR_X), a, b.first, b.count, h, iterZero, rs));
        else CK(launch_step_kernel(k_project<TT, VAR, false>, nblk(b.count, block), block, s, pdl, attr_ptr(e, PBD_ATTR_X), a, b.first, b.count, h, iterZero, rs));
        return 0;
    });
}

// Per-kernel timing (pbd_profile_step): an event recorded after every launch and what the launch was -- a constraint type,
// kLaunchIntegrate or kLaunchVelocity; ev[0] marks the start.
enum { kLaunchStart = -3, kLaunchVelocity = -2, kLaunchIntegrate = -1 };
struct LaunchLog {
    std::vector<cudaEvent_t> ev;
    std::vector<int> what;
    ~LaunchLog() { for (cudaEvent_t x : ev) cudaEventDestroy(x); }
    int mark(cudaStream_t s, int kind) {
        cudaEvent_t x;
        CK(cudaEventCreate(&x));
        ev.push_back(x); what.push_back(kind);
        CK(cudaEventRecord(x, s));
        return 0;
    }
};

// all buckets [b0, b1) belong to one colour: one launch for up to kMultiSegments of them; with `log` one launch per bucket
static int launch_colour(pbd_engine *e, size_t b0, size_t b1, float h, int iterZero, cudaStream_t s, LaunchLog *log, unsigned long long *launches) {
    // One launch per colour pays off when the colour is small (latency-bound phases; H100 80GB HBM3, 400 W, graph mode: cfg3 11.0 ->
    // 7.95 ms); a large colour keeps the specialised single-type kernels (cfg2, 250k-constraint colours: 5.59 ms either way).
    constexpr unsigned kMergeMaxConstraints = 65536;
    unsigned colourTotal = 0;
    for (size_t i = b0; i < b1; i++) colourTotal += e->buckets[i].count;
    colourTotal *= e->batch.K;
    if (b1 - b0 == 1 || log || colourTotal > kMergeMaxConstraints) {
        for (size_t i = b0; i < b1; i++) {
            CKE(launch_bucket(e, e->buckets[i], h, iterZero, s, !log));
            (*launches)++;
            if (log) CKE(log->mark(s, e->buckets[i].type));
        }
        return 0;
    }
    for (size_t c0 = b0; c0 < b1; c0 += kMultiSegments) {
        const size_t c1 = std::min(b1, c0 + (size_t)kMultiSegments);
        MultiArgs m{};
        ReplicaStrides rs{e->n, {}, {}, {}, {}, e->nRb};
        m.nSeg = (int)(c1 - c0);
        unsigned blocks = 0, total = 0;
        for (size_t i = c0; i < c1; i++) total += e->buckets[i].count;
        const unsigned block = project_block(e, total * e->batch.K);
        for (size_t i = c0; i < c1; i++) {
            const Bucket &b = e->buckets[i];
            const int k = (int)(i - c0);
            m.type[k] = b.type; m.first[k] = b.first; m.count[k] = b.count; m.blockStart[k] = blocks;
            m.arrays[k] = batch_arrays(e, b.type);
            rs.nLambda[k] = e->dev[b.type].count; rs.mat[k] = replica_mat(e, b.type); rs.nGeo[k] = replica_geo(e, b.type); rs.nMat[k] = replica_cmat(e, b.type);
            blocks += nblk(b.count, block);
        }
        for (int k = m.nSeg; k <= kMultiSegments; k++) m.blockStart[k] = blocks;
        if (e->batch.K > 1) CK(launch_step_kernel(k_project_multi<true>, dim3(blocks, e->batch.K), block, s, true, attr_ptr(e, PBD_ATTR_X), m, h, iterZero, rs));
        else CK(launch_step_kernel(k_project_multi<false>, blocks, block, s, true, attr_ptr(e, PBD_ATTR_X), m, h, iterZero, rs));
        (*launches)++;
    }
    return 0;
}

static RbState rb_state(const pbd_engine *e) {
    return RbState{(float4 *)e->rbX.p, (float4 *)e->rbQ.p, (float4 *)e->rbV.p, (float4 *)e->rbW.p, (float4 *)e->rbOldX.p, (float4 *)e->rbLastX.p,
                   (float4 *)e->rbOldQ.p, (float4 *)e->rbLastQ.p, (const float4 *)e->rbI.p, (const float4 *)e->rbIinv.p, e->nRb};
}

// One TimeStepController::step as individual launches on stream s; returns the number of kernels launched.  With `log`
// (pbd_profile_step): one launch per bucket, no PDL, and an event after every launch.
static int enqueue_step_launches(pbd_engine *e, cudaStream_t s, unsigned long long *launches, LaunchLog *log = nullptr) {
    const float h = e->dt / (float)e->subSteps;  // TimeStepController.cpp:91
    const float invH = (float)(1.0 / (double)h);
    const unsigned n = e->n * e->batch.K;  // the particle updates run over every replica's slots at once
    const bool pdl = !log;
    const RbState rb = rb_state(e);
    float4 *x = attr_ptr(e, PBD_ATTR_X), *v = attr_ptr(e, PBD_ATTR_V), *oldX = attr_ptr(e, PBD_ATTR_OLDX), *lastX = attr_ptr(e, PBD_ATTR_LASTX);
    const float4 *force = (const float4 *)e->force.p;  // the integration's force form only while forces are set
    unsigned long long L = 0;
    auto launched = [&](int kind) { L++; return log ? log->mark(s, kind) : 0; };
    for (unsigned sub = 0; sub < e->subSteps; sub++) {
        if (e->nRb) {
            if (e->batch.K > 1)  // replica blockIdx.y's bodies, under its own gravity row where it has one
                CK(launch_step_kernel(k_rb_integrate_batch, dim3(nblk(e->nRb, 256), e->batch.K), 256, s, pdl, rb, h, e->g[0], e->g[1], e->g[2],
                                      e->batch.gravitySet ? (const float *)e->batch.gravity.p : (const float *)nullptr));
            else CK(launch_step_kernel(k_rb_integrate, nblk(e->nRb, 256), 256, s, pdl, rb, h, e->g[0], e->g[1], e->g[2]));
            CKE(launched(kLaunchIntegrate));
        }
        if (n) {
            if (e->batch.gravitySet && force)  // replica blockIdx.y under its own row
                CK(launch_step_kernel(k_integrate_force<true>, replica_grid(e, e->batch.K), 256, s, pdl, x, v, oldX, lastX, e->n, h, 0.0f, 0.0f, 0.0f,
                                      (const float *)e->batch.gravity.p, force));
            else if (e->batch.gravitySet)
                CK(launch_step_kernel(k_integrate<true>, replica_grid(e, e->batch.K), 256, s, pdl, x, v, oldX, lastX, e->n, h, 0.0f, 0.0f, 0.0f,
                                      (const float *)e->batch.gravity.p));
            else if (force)
                CK(launch_step_kernel(k_integrate_force<false>, nblk(n, 256), 256, s, pdl, x, v, oldX, lastX, n, h, e->g[0], e->g[1], e->g[2],
                                      (const float *)nullptr, force));
            else
                CK(launch_step_kernel(k_integrate<false>, nblk(n, 256), 256, s, pdl, x, v, oldX, lastX, n, h, e->g[0], e->g[1], e->g[2],
                                      (const float *)nullptr));
            CKE(launched(kLaunchIntegrate));
        }
        for (unsigned it = 0; it < e->maxIter; it++)
            for (size_t b0 = 0; b0 < e->buckets.size();) {
                size_t b1 = b0 + 1;
                while (b1 < e->buckets.size() && e->buckets[b1].colour == e->buckets[b0].colour) b1++;
                CKE(launch_colour(e, b0, b1, h, it == 0, s, log, &L));
                b0 = b1;
            }
        if (n) {
            CK(launch_step_kernel(k_velocity, nblk(n, 256), 256, s, pdl, x, v, oldX, lastX, n, invH, e->velMethod));
            CKE(launched(kLaunchVelocity));
        }
        if (e->nRb) {
            if (e->batch.K > 1) CK(launch_step_kernel(k_rb_velocity_batch, dim3(nblk(e->nRb, 256), e->batch.K), 256, s, pdl, rb, invH, (float)(2.0 / (double)h), e->velMethod));
            else CK(launch_step_kernel(k_rb_velocity, nblk(e->nRb, 256), 256, s, pdl, rb, invH, (float)(2.0 / (double)h), e->velMethod));
            CKE(launched(kLaunchVelocity));
        }
    }
    *launches = L;
    return 0;
}

// One step as one launch of k_step_resident: grid = G x C CTAs in clusters of C, one CTA per SM, all co-resident
// (the X items of different clusters wait for each other; the planner admitted the image only if the device keeps them so).
static int enqueue_step_resident(pbd_engine *e, cudaStream_t s, unsigned long long *launches) {
    const float h = e->dt / (float)e->subSteps;
    ResidentArgs ra;
    ra.pos = attr_ptr(e, PBD_ATTR_X); ra.vel = attr_ptr(e, PBD_ATTR_V); ra.oldp = attr_ptr(e, PBD_ATTR_OLDX); ra.lastp = attr_ptr(e, PBD_ATTR_LASTX);
    const pbd_b200::ImageTables &tb = e->tables;
    ra.buckets = tb.buckets; ra.colourStart = tb.colourStart; ra.tileOff = tb.tileOff; ra.tileStart = tb.tileStart; ra.tileSmem = tb.tileSmem;
    ra.xNbr = tb.xNbr; ra.xMask = tb.xMask; ra.xFlags = tb.xFlags;
    const bool batch = e->res.replicas > 1;  // the tables hold the C tiles of one replica
    ra.nBuckets = (unsigned)e->buckets.size(); ra.nColours = e->res.nColours; ra.nTiles = batch ? e->res.C : e->res.G * e->res.C; ra.subSteps = e->subSteps; ra.maxIter = e->maxIter;
    ra.tileCap = e->res.tileCap; ra.xThreads = e->res.xThreads; ra.clusterSize = e->res.C;
    {   // L2 prefetch of the operand runs pays when the constraint stream of a sweep does not stay in L2 anyway (above ~0.38 x the L2).
        // H100 80GB HBM3 (400 W, 50 MB L2), prefetch off / on: cfg2 (192 MB per sweep) 2.28 / 2.08 ms, cfg5 (48 MB) 1.246 / 1.216 ms,
        // 300x300 cloth (below the threshold) 1.015 / 1.016 ms.
        double streamBytes = 0.0;
        for (int t = 0; t < PBD_NUM_TYPES; t++) {
            const TypeShape sh = type_shape(t);
            streamBytes += (double)e->dev[t].count * (4.0 * sh.nBodies + 16.0 * sh.nGeoV + 4.0 * sh.nGeoS + (sh.xpbd ? 4.0 : 0.0));
        }
        ra.l2Prefetch = streamBytes > 0.38 * (double)e->l2Bytes ? 1 : 0;
    }
    ra.h = h; ra.invH = (float)(1.0 / (double)h); ra.twoInvH = (float)(2.0 / (double)h); ra.gx = e->g[0]; ra.gy = e->g[1]; ra.gz = e->g[2];
    ra.secondOrder = e->velMethod;
    ra.xLaunch = (++e->xLaunch) << 32;  // above every flag value of the earlier launches, whatever subSteps / maxIter they ran with
    ra.rb = rb_state(e);
    for (int t = 0; t < PBD_NUM_TYPES; t++) { ra.types[t] = batch_arrays(e, t); ra.lamCount[t] = e->dev[t].count; ra.geoCount[t] = replica_geo(e, t); ra.matCount[t] = replica_cmat(e, t); }
    ra.replicas = e->res.replicas; ra.replicaStride = e->n;
    ra.repMat = (const float *)e->batch.mat.p; ra.repGravity = e->batch.gravitySet ? (const float *)e->batch.gravity.p : nullptr;
    ra.force = (const float4 *)e->force.p;
    *launches = 1;
    ra.trace = nullptr; ra.tracePhases = 0;
    static const char *tracePath = getenv("PBD_B200_TRACE");  // development aid: dump per-phase timelines of one step (tools/trace_resident.py)
    const unsigned kTracePhases = 256;
    if (tracePath && !batch) {  // (a batch's clusters step different replicas through the same tiles: no per-CTA timeline to record)
        CKE(e->dTrace.alloc((size_t)kTracePhases * ra.nTiles * kTraceSlots * sizeof(unsigned long long)));
        CK(cudaMemsetAsync(e->dTrace.p, 0, e->dTrace.bytes, s));
        ra.trace = (unsigned long long *)e->dTrace.p; ra.tracePhases = kTracePhases;
    }
    struct TraceDump {  // runs after the launch below has been enqueued (scope exit)
        pbd_engine *e; cudaStream_t s; const char *path; size_t words;
        ~TraceDump() {
            if (!path) return;
            cudaStreamSynchronize(s);
            std::vector<unsigned long long> h(words);
            cudaMemcpy(h.data(), e->dTrace.p, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
            if (FILE *f = fopen(path, "wb")) { fwrite(h.data(), sizeof(unsigned long long), h.size(), f); fclose(f); }
        }
    } dump{e, s, batch ? nullptr : tracePath, (size_t)kTracePhases * ra.nTiles * kTraceSlots};
    const pbd_b200::ResidentShape &r = e->res;
    CKE(with_resident_kernel(r.mask, r.C, batch, [&](auto kernel) -> int {
        CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxDynamicSmem));
        if (r.C > 8) CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
        cudaLaunchConfig_t cfg; cudaLaunchAttribute attr[1];
        resident_launch_config(r.mask, r.C, batch, r.G * r.C, r.smem, s, cfg, attr);
        CK(cudaLaunchKernelEx(&cfg, kernel, ra));
        return 0;
    }));
    if (batch && e->nRb) {  // a batch's body velocities of the last substep (resident.cuh: the others at the head of the next substep)
        k_rb_velocity_batch<<<dim3(nblk(e->nRb, 256), e->batch.K), 256, 0, s>>>(ra.rb, ra.invH, ra.twoInvH, ra.secondOrder);
        CK(cudaGetLastError());
        *launches = 2;
    }
    return 0;
}

// Jacobi comparison path (kernels.cuh): per sweep one launch per type over all its constraints + the averaging pass
static int enqueue_step_jacobi(pbd_engine *e, cudaStream_t s, unsigned long long *launches) {
    if (e->nRb || e->dev[PBD_BALLJOINT].count || e->dev[PBD_RB_PARTICLE_BALLJOINT].count)
        return fail("PBD_MODE_JACOBI does not cover rigid-body coupling (use PBD_MODE_GRAPH)");
    const float h = e->dt / (float)e->subSteps;
    const float invH = (float)(1.0 / (double)h);
    const unsigned n = e->n;
    if (n == 0) { *launches = 0; return 0; }
    if (!e->jacobiDelta.p || e->jacobiDelta.bytes < (size_t)n * sizeof(float4)) {
        CKE(e->jacobiDelta.alloc((size_t)n * sizeof(float4)));
        CK(cudaMemsetAsync(e->jacobiDelta.p, 0, (size_t)n * sizeof(float4), s));
    }
    float4 *x = attr_ptr(e, PBD_ATTR_X), *v = attr_ptr(e, PBD_ATTR_V), *oldX = attr_ptr(e, PBD_ATTR_OLDX), *lastX = attr_ptr(e, PBD_ATTR_LASTX);
    float4 *delta = (float4 *)e->jacobiDelta.p;
    unsigned long long L = 0;
    for (unsigned sub = 0; sub < e->subSteps; sub++) {
        if (e->force.p) k_integrate_force<false><<<nblk(n, 256), 256, 0, s>>>(x, v, oldX, lastX, n, h, e->g[0], e->g[1], e->g[2], nullptr, (const float4 *)e->force.p);
        else k_integrate<false><<<nblk(n, 256), 256, 0, s>>>(x, v, oldX, lastX, n, h, e->g[0], e->g[1], e->g[2], nullptr);
        L++;
        for (unsigned it = 0; it < e->maxIter; it++) {
            for (int t = 0; t < PBD_BALLJOINT; t++) {
                const unsigned cnt = e->dev[t].count;
                if (!cnt) continue;
                const TypeArrays &a = e->dev[t].arrays;
                CKE(with_project_type(t, a.variant, [&](auto T, auto V) -> int {
                    constexpr int TT = decltype(T)::value, VAR = decltype(V)::value;
                    if constexpr (TT < PBD_BALLJOINT)  // the joints are refused above
                        k_project_jacobi<TT, VAR><<<nblk(cnt, 128), 128, 0, s>>>(x, delta, a, cnt, h, it == 0);
                    return 0;
                }));
                L++;
            }
            k_jacobi_apply<<<nblk(n, 256), 256, 0, s>>>(x, delta, n); L++;
        }
        k_velocity<<<nblk(n, 256), 256, 0, s>>>(x, v, oldX, lastX, n, invH, e->velMethod); L++;
    }
    CK(cudaGetLastError());
    *launches = L;
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// contact path (contacts.cuh)
// ------------------------------------------------------------------------------------------------------------
// the kernel's form of a pbd_rigid_collider; refused: an unknown shape
static int convert_collider(const char *what, unsigned i, const pbd_rigid_collider &c, RigidCollider &d) {
    if (c.shape < 0 || c.shape >= kNumShapes) return fail("%s: rigid collider %u has unknown shape %d", what, i, c.shape);
    d.shape = c.shape; d.body = c.body; d.thickness = c.thickness; d.invert = c.invert_sdf ? -1.0f : 1.0f; d.restitution = c.restitution; d.friction = c.friction;
    for (int k = 0; k < 3; k++) { d.dim[k] = c.dim[k]; d.v1[k] = c.v1[k]; d.v2[k] = c.v2[k]; d.aabbMin[k] = c.aabb_min[k]; d.aabbMax[k] = c.aabb_max[k]; }
    for (int k = 0; k < 9; k++) d.R[k] = c.R[k];
    return 0;
}
// one replica's particle ranges and the prefix sums of their counts; refused: a range beyond the engine's n particles, and two ranges
// that share a particle (the contact kernel runs one thread per range entry: two threads would solve the same particle and one store
// would be lost)
static int convert_ranges(const pbd_engine *e, const char *what, unsigned nP, const pbd_particle_collider *pc, std::vector<ParticleCollider> &P,
                          std::vector<unsigned> &start) {
    P.resize(nP); start.assign(nP + 1, 0u);
    std::vector<unsigned> byOffset;
    for (unsigned i = 0; i < nP; i++) {
        if ((unsigned long long)pc[i].offset + pc[i].count > e->n) return fail("%s: particle collider %u covers [%u, %u), the engine holds %u particles", what, i, pc[i].offset, pc[i].offset + pc[i].count, e->n);
        P[i].offset = pc[i].offset; P[i].count = pc[i].count; P[i].restitution = pc[i].restitution; P[i].friction = pc[i].friction;
        start[i + 1] = start[i] + pc[i].count;
        if (pc[i].count) byOffset.push_back(i);
    }
    std::sort(byOffset.begin(), byOffset.end(), [&](unsigned a, unsigned b) { return pc[a].offset < pc[b].offset; });
    for (size_t j = 1; j < byOffset.size(); j++) {
        const pbd_particle_collider &a = pc[byOffset[j - 1]], &b = pc[byOffset[j]];
        if (b.offset < a.offset + a.count)
            return fail("%s: particle colliders %u [%u, %u) and %u [%u, %u) overlap (each particle may belong to one range only)", what, byOffset[j - 1],
                        a.offset, a.offset + a.count, byOffset[j], b.offset, b.offset + b.count);
    }
    return 0;
}

// the host copy of the body masses the contact path checks: read back (V.w, in stream order) after a device write of the masses
static int body_masses(pbd_engine *e) {
    if (!e->rbMassStale) return 0;
    const size_t rows = (size_t)e->batch.K * e->nRb;
    std::vector<float4> V(rows);
    CK(cudaStreamSynchronize(e->stream));
    if (rows) CK(cudaMemcpy(V.data(), e->rbV.p, rows * sizeof(float4), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < rows; i++) e->rbMass[i] = V[i].w;
    e->rbMassStale = false;
    return 0;
}

extern "C" int pbd_set_colliders(pbd_engine *e, unsigned nP, const pbd_particle_collider *pc, unsigned nR, const pbd_rigid_collider *rc) {
    if (!e || (nP && !pc) || (nR && !rc)) return fail("pbd_set_colliders: null argument");
    CKE(collider_refusal(e, e->batch.K, (size_t)nP + nR));
    CKE(use(e));
    if (nR > (unsigned)kMaxRigidColliders) return fail("pbd_set_colliders: %u rigid colliders (the contact kernel keeps up to %d contacts per particle)", nR, kMaxRigidColliders);
    std::vector<ParticleCollider> P;
    std::vector<RigidCollider> R(nR);
    std::vector<unsigned> start;
    CKE(convert_ranges(e, "pbd_set_colliders", nP, pc, P, start));
    CKE(body_masses(e));
    for (unsigned i = 0; i < nR; i++) {
        const pbd_rigid_collider &c = rc[i];
        CKE(convert_collider("pbd_set_colliders", i, c, R[i]));
        if (c.body >= e->nRb) return fail("pbd_set_colliders: rigid collider %u refers to rigid body %u, the engine holds %u (pbd_set_rigid_bodies first)", i, c.body, e->nRb);
        if (e->rbMass[c.body] != 0.0f)
            return fail("pbd_set_colliders: rigid body %u has mass %g; contacts with dynamic bodies couple through the body and stay on the CPU time step (static colliders only)", c.body, e->rbMass[c.body]);
    }
    CK(cudaStreamSynchronize(e->stream));
    e->pColliders.swap(P); e->rColliders.swap(R);
    e->contactTotal = start[nP];
    if (nP) { CKE(upload_vec(e->dPColliders, e->pColliders, e->stream)); CKE(upload_vec(e->dRangeStart, start, e->stream)); }
    if (nR) CKE(upload_vec(e->dRColliders, e->rColliders, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return size_sensors(e);
}
extern "C" int pbd_set_replica_colliders(pbd_engine *e, unsigned nP, const pbd_particle_collider *pc, unsigned nR, const pbd_rigid_collider *rc,
                                         const float *body_x, const float *body_v, const float *body_omega) {
    CKE(replica_params_refusal(e, "pbd_set_replica_colliders"));
    if (!rc) nR = 0;
    if (nP && !pc) return fail("pbd_set_replica_colliders: null argument");
    if (nR && !body_x) return fail("pbd_set_replica_colliders: body_x == NULL with %u rigid colliders per replica", nR);
    if (nR > (unsigned)kMaxRigidColliders) return fail("pbd_set_replica_colliders: %u rigid colliders per replica (the contact kernel keeps up to %d contacts per particle)", nR, kMaxRigidColliders);
    CKE(use(e));
    const unsigned K = e->batch.K;
    const size_t rows = (size_t)K * nR;
    std::vector<ParticleCollider> P;
    std::vector<unsigned> start;
    CKE(convert_ranges(e, "pbd_set_replica_colliders", nP, pc, P, start));
    std::vector<RigidCollider> R(rows);
    for (size_t i = 0; i < rows; i++) CKE(convert_collider("pbd_set_replica_colliders", (unsigned)i, rc[i], R[i]));
    std::vector<float4> X(rows), V(rows), W(rows);  // the static bodies: w = inverse mass / mass / unused, all 0
    for (size_t i = 0; i < rows; i++) {
        X[i] = make_float4(body_x[3 * i], body_x[3 * i + 1], body_x[3 * i + 2], 0.f);
        V[i] = body_v ? make_float4(body_v[3 * i], body_v[3 * i + 1], body_v[3 * i + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        W[i] = body_omega ? make_float4(body_omega[3 * i], body_omega[3 * i + 1], body_omega[3 * i + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    pbd_engine::ReplicaColliders &c = e->repColliders;
    if (nR == 0) {  // off
        CK(cudaStreamSynchronize(e->stream));
        drop_replica_colliders(e);
        return size_sensors(e);
    }
    const struct { DevBuf *d; const void *h; size_t bytes; } up[] = {
        {&c.dRanges, P.data(), nP * sizeof(ParticleCollider)}, {&c.dStart, start.data(), (nP + 1) * sizeof(unsigned)},
        {&c.dRigid, R.data(), rows * sizeof(RigidCollider)}, {&c.dX, X.data(), rows * sizeof(float4)}, {&c.dV, V.data(), rows * sizeof(float4)},
        {&c.dW, W.data(), rows * sizeof(float4)}};
    if (nP != c.ranges.size() || nR != c.nRigid) {  // new table sizes: allocated again once the steps in flight are done
        CK(cudaStreamSynchronize(e->stream));
        drop_replica_colliders(e);
        for (const auto &u : up) CKE(u.d->alloc(u.bytes));
    }
    // Stream-ordered copies into tables that keep their address: the next step enqueued reads the new rows, the steps before it the old
    // ones.  The sources are pageable, so the driver has staged them when the call returns and the vectors may go.
    for (const auto &u : up) if (u.bytes) CK(cudaMemcpyAsync(u.d->p, u.h, u.bytes, cudaMemcpyHostToDevice, e->stream));
    c.ranges.swap(P); c.nRigid = nR; c.total = start[nP];
    return size_sensors(e);  // the same counts: nothing to do, no synchronisation
}

// pbd_set_replica_collider_poses_device: the placement rows of a batch's colliders and their bodies, written in place by
// k_set_collider_poses under device_call's stream contract
extern "C" int pbd_set_replica_collider_poses_device(pbd_engine *e, const float *pose, const float *body_x, const float *body_v,
                                                     const float *body_omega, const unsigned char *replicas, void *stream) {
    const char *what = "pbd_set_replica_collider_poses_device";
    if (!e) return fail("%s: null engine", what);
    if (e->batch.K == 1) return fail("%s: a single-scene engine places its colliders through pbd_set_colliders (pbd_set_replicas first)", what);
    pbd_engine::ReplicaColliders &c = e->repColliders;
    if (!c.nRigid) return fail("%s: no replica colliders in force (pbd_set_replica_colliders first)", what);
    if (!body_x) return fail("%s: body_x == NULL", what);
    CKE(body_arrays_refusal(e, what, {{"body_x", body_x}, {"body_v", body_v}, {"body_omega", body_omega}}));
    return device_call(e, what, "pose", pose, replicas, stream, (size_t)e->batch.K * c.nRigid, [] { return 0; }, [&]() -> int {
        k_set_collider_poses<<<dim3(1, e->batch.K), kMaxRigidColliders, 0, e->stream>>>((RigidCollider *)c.dRigid.p, (float4 *)c.dX.p, (float4 *)c.dV.p,
                                                                                   (float4 *)c.dW.p, c.nRigid, ColliderPoses{pose, body_x, body_v, body_omega, replicas});
        CK(cudaGetLastError());
        return 0;
    });
}

// ---- contact sensors -----------------------------------------------------------------------------------------------------------------
extern "C" int pbd_sense_contacts(pbd_engine *e, int on) {
    if (!e) return fail("pbd_sense_contacts: null engine");
    e->sensors.on = on != 0;
    return size_sensors(e);
}
static int sensors_refusal(const pbd_engine *e, const char *what) {
    if (!e->sensors.on) return fail("%s: contact sensing is off (pbd_sense_contacts)", what);
    if (!e->sensors.nRigid) return fail("%s: no rigid colliders in force (pbd_set_colliders / pbd_set_replica_colliders)", what);
    return 0;
}
extern "C" int pbd_get_contact_sensors(pbd_engine *e, unsigned *count, float *impulse) {
    const char *what = "pbd_get_contact_sensors";
    if (!e) return fail("%s: null engine", what);
    CKE(sensors_refusal(e, what));
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    const size_t rows = (size_t)e->sensors.K * e->sensors.nRigid;
    if (count) CK(cudaMemcpy(count, e->sensors.count.p, rows * sizeof(unsigned), cudaMemcpyDeviceToHost));
    if (impulse) CK(cudaMemcpy(impulse, e->sensors.impulse.p, rows * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
}
extern "C" int pbd_get_contact_sensors_device(pbd_engine *e, unsigned *count, float *impulse, void *stream) {
    const char *what = "pbd_get_contact_sensors_device";
    if (!e) return fail("%s: null engine", what);
    CKE(sensors_refusal(e, what));
    if (!count && !impulse) return 0;  // nothing asked for
    CKE(body_arrays_refusal(e, what, {{"count", count}, {"impulse", impulse}}));
    const size_t rows = (size_t)e->sensors.K * e->sensors.nRigid;
    return device_call(e, what, count ? "count" : "impulse", count ? (const void *)count : (const void *)impulse, nullptr, stream, rows, [] { return 0; },
                       [&]() -> int {
        if (count) CK(cudaMemcpyAsync(count, e->sensors.count.p, rows * sizeof(unsigned), cudaMemcpyDeviceToDevice, e->stream));
        if (impulse) CK(cudaMemcpyAsync(impulse, e->sensors.impulse.p, rows * 3 * sizeof(float), cudaMemcpyDeviceToDevice, e->stream));
        return 0;
    });
}
extern "C" int pbd_set_contact_params(pbd_engine *e, float tolerance, float stiffness, unsigned maxIterationsV) {
    if (!e) return fail("null engine");
    e->contactTolerance = tolerance; e->contactStiffness = stiffness; e->maxIterV = maxIterationsV;
    return 0;
}
extern "C" int pbd_record_contacts(pbd_engine *e, unsigned capacity) {
    if (!e) return fail("null engine");
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    e->contactCap = capacity;
    if (capacity) {
        CKE(e->dContacts.alloc((size_t)capacity * sizeof(ContactRecord)));
        CKE(e->dContactCount.alloc(sizeof(unsigned)));
        CK(cudaMemset(e->dContactCount.p, 0, sizeof(unsigned)));
    }
    return 0;
}
extern "C" int pbd_get_contacts(pbd_engine *e, pbd_contact *out, unsigned capacity, unsigned *count) {
    if (!e || !count) return fail("pbd_get_contacts: null argument");
    CKE(use(e));
    *count = 0;
    if (!e->contactCap) return fail("pbd_get_contacts: recording is off (pbd_record_contacts)");
    CK(cudaStreamSynchronize(e->stream));
    unsigned found = 0;
    CK(cudaMemcpy(&found, e->dContactCount.p, sizeof(unsigned), cudaMemcpyDeviceToHost));
    *count = found;
    const unsigned kept = std::min(found, e->contactCap);
    static_assert(sizeof(pbd_contact) == sizeof(ContactRecord), "pbd_contact mirrors ContactRecord");
    std::vector<pbd_contact> tmp(kept);
    if (kept) CK(cudaMemcpy(tmp.data(), e->dContacts.p, (size_t)kept * sizeof(pbd_contact), cudaMemcpyDeviceToHost));
    std::sort(tmp.begin(), tmp.end(), [](const pbd_contact &a, const pbd_contact &b) { return a.particle != b.particle ? a.particle < b.particle : a.body < b.body; });
    if (out) for (unsigned i = 0; i < std::min(kept, capacity); i++) out[i] = tmp[i];
    return 0;
}
// after the substeps of a step: collision detection + velocity-level contact solve (TimeStepController.cpp:189-196)
// A batch's replica colliders (pbd_set_replica_colliders) run k_contacts_batch, one grid row per replica; pbd_set_colliders' k_contacts.
static int enqueue_contacts(pbd_engine *e, cudaStream_t s, unsigned long long *launches) {
    const pbd_engine::ReplicaColliders &rep = e->repColliders;
    const bool batch = rep.nRigid != 0;
    if (batch ? rep.total == 0 : (e->rColliders.empty() || e->contactTotal == 0)) return 0;
    if (!batch) CKE(body_masses(e));
    if (!batch)
        for (const RigidCollider &c : e->rColliders)  // the bodies may have been replaced since pbd_set_colliders
            if (c.body >= e->nRb || e->rbMass[c.body] != 0.0f) return fail("contact path: collider on rigid body %u, which is missing or not static any more (pbd_set_colliders again)", c.body);
    for (const ParticleCollider &c : batch ? rep.ranges : e->pColliders)
        if ((unsigned long long)c.offset + c.count > e->n) return fail("contact path: a particle collider covers particles beyond the %u the engine holds", e->n);
    ContactArgs a;
    a.pos = attr_ptr(e, PBD_ATTR_X); a.vel = attr_ptr(e, PBD_ATTR_V); a.slot = (const unsigned *)e->dSlot.p;
    if (batch) {
        a.rbX = (const float4 *)rep.dX.p; a.rbV = (const float4 *)rep.dV.p; a.rbW = (const float4 *)rep.dW.p;
        a.rigid = (const RigidCollider *)rep.dRigid.p; a.nRigid = rep.nRigid;
        a.ranges = (const ParticleCollider *)rep.dRanges.p; a.nRanges = (unsigned)rep.ranges.size();
        a.rangeStart = (const unsigned *)rep.dStart.p; a.total = rep.total; a.n = e->n;
    } else {
        a.rbX = (const float4 *)e->rbX.p; a.rbV = (const float4 *)e->rbV.p; a.rbW = (const float4 *)e->rbW.p;
        a.rigid = (const RigidCollider *)e->dRColliders.p; a.nRigid = (unsigned)e->rColliders.size();
        a.ranges = (const ParticleCollider *)e->dPColliders.p; a.nRanges = (unsigned)e->pColliders.size();
        a.rangeStart = (const unsigned *)e->dRangeStart.p; a.total = e->contactTotal;
    }
    a.tolerance = e->contactTolerance; a.stiffness = e->contactStiffness; a.maxIterV = e->maxIterV;
    a.record = e->contactCap ? (ContactRecord *)e->dContacts.p : nullptr; a.recordCount = (unsigned *)e->dContactCount.p; a.recordCap = e->contactCap;
    if (e->contactCap) CK(cudaMemsetAsync(e->dContactCount.p, 0, sizeof(unsigned), s));
    const dim3 grid((a.total + 127u) / 128u, batch ? e->batch.K : 1u);
    const pbd_engine::Sensors &S = e->sensors;
    if (!S.on) {
        if (batch) k_contacts_batch<<<grid, 128, 0, s>>>(a);
        else k_contacts<<<grid, 128, 0, s>>>(a);
        CK(cudaGetLastError());
        *launches += 1;
        return 0;
    }
    // sensing: the same contacts with per-block sensor sums, then their sum per collider in block order (size_sensors sized the buffers)
    if (S.K != grid.y || S.nRigid != a.nRigid || S.blocks != grid.x) return fail("contact sensors sized for %u x %u colliders and %u blocks, the launch has %u x %u and %u", S.K, S.nRigid, S.blocks, grid.y, a.nRigid, grid.x);
    float4 *partial = (float4 *)S.partial.p;
    if (batch) k_contacts_sense_batch<<<grid, kSenseThreads, 0, s>>>(a, partial);
    else k_contacts_sense<<<grid, kSenseThreads, 0, s>>>(a, partial);
    const unsigned rows = S.K * S.nRigid;
    k_contact_sensors_sum<<<nblk(rows, 128), 128, 0, s>>>(partial, rows, S.nRigid, S.blocks, (unsigned *)S.count.p, (float *)S.impulse.p);
    CK(cudaGetLastError());
    *launches += 2;
    return 0;
}

// Everything enqueue_step_launches reads, which a captured step bakes in, as the bytes of scalars and arrays of them (no padding).
// imageGen stands for the bucket table.  The structured bindings do not compile once RbState or TypeArrays gains a member not listed here.
static std::vector<unsigned char> graph_key(const pbd_engine *e) {
    std::vector<unsigned char> key;
    key.reserve(4096);
    const auto [X, Q, V, W, oldX, lastX, oldQ, lastQ, I, Iinv, nRb] = rb_state(e);
    append_bytes(key, e->imageGen, e->n, e->batch.K, e->dt, e->subSteps, e->maxIter, e->velMethod, e->g,
                 attr_ptr(e, PBD_ATTR_X), attr_ptr(e, PBD_ATTR_V), attr_ptr(e, PBD_ATTR_OLDX), attr_ptr(e, PBD_ATTR_LASTX),
                 e->batch.gravitySet ? e->batch.gravity.p : nullptr, e->force.p, X, Q, V, W, oldX, lastX, oldQ, lastQ, I, Iinv, nRb);
    for (int t = 0; t < PBD_NUM_TYPES; t++) {
        const auto [idx2, idx4, idx3, gv, gs, mat, matU, lambda, rbX, rbQ, rbIinv, variant] = batch_arrays(e, t);
        append_bytes(key, idx2, idx4, idx3, gv, gs, mat, matU, lambda, rbX, rbQ, rbIinv, variant, replica_mat(e, t), replica_geo(e, t), replica_cmat(e, t),
                     e->dev[t].count);
    }
    return key;
}

static int ensure_graph(pbd_engine *e) {
    std::vector<unsigned char> key = graph_key(e);
    if (e->graphExec && key == e->graphKey) return 0;
    if (e->graphExec) { cudaGraphExecDestroy(e->graphExec); e->graphExec = nullptr; }
    cudaGraph_t graph = nullptr;
    CK(cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
    unsigned long long L = 0;
    int rc = enqueue_step_launches(e, e->stream, &L);
    cudaError_t err = cudaStreamEndCapture(e->stream, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (err != cudaSuccess) return fail("cudaStreamEndCapture -> %s", cudaGetErrorString(err));
    err = cudaGraphInstantiate(&e->graphExec, graph, 0);
    cudaGraphDestroy(graph);
    if (err != cudaSuccess) { e->graphExec = nullptr; return fail("cudaGraphInstantiate -> %s", cudaGetErrorString(err)); }
    e->graphKey.swap(key);
    e->graphLaunches = L;
    e->stats.graph_captures++;
    return 0;
}

extern "C" int pbd_step(pbd_engine *e, unsigned nSteps) {
    if (!e) return fail("null engine");
    CKE(use(e));
    CKE(flatten(e));
    const int active = active_mode(e);
    CK(cudaEventRecord(e->evStart, e->stream));
    for (unsigned s = 0; s < nSteps; s++) {
        unsigned long long L = 0;
        if (active == PBD_MODE_LAUNCH) CKE(enqueue_step_launches(e, e->stream, &L));
        else if (active == PBD_MODE_RESIDENT) CKE(enqueue_step_resident(e, e->stream, &L));
        else if (active == PBD_MODE_JACOBI) CKE(enqueue_step_jacobi(e, e->stream, &L));
        else { if (s == 0) CKE(ensure_graph(e)); CK(cudaGraphLaunch(e->graphExec, e->stream)); L = e->graphLaunches; }
        CKE(enqueue_contacts(e, e->stream, &L));
        e->stats.kernel_launches += L;
        e->stats.steps++;
        e->stats.projections += (unsigned long long)e->numConstraints * e->subSteps * e->maxIter * e->batch.K;
    }
    CK(cudaEventRecord(e->evStop, e->stream));
    e->timingPending = true;
    return 0;
}

extern "C" int pbd_sync(pbd_engine *e) {
    if (!e) return fail("null engine");
    CKE(use(e));
    CK(cudaStreamSynchronize(e->stream));
    if (e->timingPending) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, e->evStart, e->evStop) == cudaSuccess) e->stats.last_step_ms = ms;
        e->timingPending = false;
    }
    return 0;
}

extern "C" int pbd_pin_host(void *ptr, size_t bytes) {
    if (!ptr || !bytes) return fail("pbd_pin_host: null argument");
    const cudaError_t err = cudaHostRegister(ptr, bytes, cudaHostRegisterPortable);
    if (err != cudaSuccess) { cudaGetLastError(); return fail("cudaHostRegister -> %s", cudaGetErrorString(err)); }  // clear the sticky per-thread error: a later CK(cudaGetLastError()) must not see it
    return 0;
}
extern "C" int pbd_unpin_host(void *ptr) {
    if (!ptr) return 0;
    const cudaError_t err = cudaHostUnregister(ptr);
    if (err != cudaSuccess) { cudaGetLastError(); return fail("cudaHostUnregister -> %s", cudaGetErrorString(err)); }
    return 0;
}

extern "C" int pbd_step_host(pbd_engine *e, unsigned nSteps, const float *x_in, const float *v_in, float *x_out, float *v_out) {
    if (!e) return fail("null engine");
    CKE(use(e));
    if (e->n == 0) return pbd_step(e, nSteps);
    // two staging areas so that x and v uploads do not serialise on a host sync
    for (DevBuf &b : e->stage) CKE(b.alloc((size_t)e->batch.K * e->n * 3 * sizeof(float)));
    if (x_in) CKE(upload_attr(e, PBD_ATTR_X, x_in, 1, e->batch.K, e->stage[0], e->stream));
    if (v_in) CKE(upload_attr(e, PBD_ATTR_V, v_in, 1, e->batch.K, e->stage[1], e->stream));
    CKE(pbd_step(e, nSteps));
    if (x_out) CKE(download_attr(e, PBD_ATTR_X, x_out, e->stage[0], e->stream));
    if (v_out) CKE(download_attr(e, PBD_ATTR_V, v_out, e->stage[1], e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

// Pipelined form of pbd_step_host: the upload of call k+1 and the download of call k-1 overlap the projection kernels of call k
// (three streams, two staging slots, ordering by events only -- the host never blocks here).
extern "C" int pbd_step_host_async(pbd_engine *e, unsigned nSteps, const float *x_in, const float *v_in, float *x_out, float *v_out) {
    if (!e) return fail("null engine");
    CKE(use(e));
    if (e->n == 0) return pbd_step(e, nSteps);
    const size_t bytes = (size_t)e->batch.K * e->n * 3 * sizeof(float);
    auto &P = e->pipe;
    if (!P.ready) {
        CK(cudaStreamCreateWithFlags(&P.up, cudaStreamNonBlocking));
        CK(cudaStreamCreateWithFlags(&P.down, cudaStreamNonBlocking));
        for (int s = 0; s < 2; s++)
            for (cudaEvent_t *ev : {&P.uploaded[s], &P.consumed[s], &P.produced[s], &P.downloaded[s]}) CK(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
        P.ready = true;
    }
    const int s = (int)(P.issued & 1);
    const bool reuse = P.issued >= 2;  // the slot was used by call k-2: its consumers are ordered before us by events
    if (reuse && (x_in || v_in)) CK(cudaStreamWaitEvent(P.up, P.consumed[s], 0));
    if (x_in) { CKE(P.inX[s].alloc(bytes)); CKE(upload_attr(e, PBD_ATTR_X, x_in, 1, e->batch.K, P.inX[s], P.up, P.uploaded[s])); }
    if (v_in) { CKE(P.inV[s].alloc(bytes)); CKE(upload_attr(e, PBD_ATTR_V, v_in, 1, e->batch.K, P.inV[s], P.up, P.uploaded[s])); }
    CK(cudaEventRecord(P.consumed[s], e->stream));
    CKE(pbd_step(e, nSteps));
    if (reuse && (x_out || v_out)) CK(cudaStreamWaitEvent(e->stream, P.downloaded[s], 0));
    if (x_out) { CKE(P.outX[s].alloc(bytes)); CKE(download_attr(e, PBD_ATTR_X, x_out, P.outX[s], P.down, P.produced[s])); }
    if (v_out) { CKE(P.outV[s].alloc(bytes)); CKE(download_attr(e, PBD_ATTR_V, v_out, P.outV[s], P.down, P.produced[s])); }
    CK(cudaEventRecord(P.downloaded[s], P.down));
    P.issued++;
    return 0;
}

extern "C" int pbd_step_host_wait(pbd_engine *e, unsigned lag) {
    if (!e) return fail("null engine");
    CKE(use(e));
    auto &P = e->pipe;
    if (!P.ready || P.issued == 0) return 0;
    if (lag > 1) return fail("pbd_step_host_wait: lag %u (the pipeline has two slots: 0 = everything, 1 = all but the newest call)", lag);
    if (lag == 0) {
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaStreamSynchronize(P.down));
        return 0;
    }
    if (P.issued < 2) return 0;
    CK(cudaEventSynchronize(P.downloaded[(P.issued - 2) & 1]));
    return 0;
}

extern "C" int pbd_get_lambdas(pbd_engine *e, int type, float *dst, unsigned *ids) {
    if (!e || !dst) return fail("null argument");
    if (type < 0 || type >= PBD_NUM_TYPES || !type_shape(type).xpbd) return fail("type %d has no multipliers", type);
    CKE(use(e)); CKE(flatten(e));
    DevType &d = e->dev[type];
    if (d.count == 0) return 0;
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy(dst, d.arrays.lambda, (size_t)e->batch.K * d.count * sizeof(float), cudaMemcpyDeviceToHost));  // replica after replica
    if (ids) memcpy(ids, d.order.data(), (size_t)d.count * sizeof(unsigned));
    return 0;
}

extern "C" int pbd_get_stats(pbd_engine *e, pbd_stats *out) {
    if (!e || !out) return fail("null argument");
    CKE(use(e)); CKE(flatten(e));
    double sweep = 0.0;
    for (int t = 0; t < PBD_NUM_TYPES; t++) sweep += (double)e->dev[t].count * algorithmic_bytes(t, e->dev[t].arrays.variant);
    // per particle per substep: integrate 48 read + 64 write = 112, velocity update 32 read + 16 write = 48 (SURVEY.md 8d); the force
    // read while external forces are set, 16
    const double perParticle = 112.0 + 48.0 + (e->velMethod ? 16.0 : 0.0) + (e->force.p ? 16.0 : 0.0);
    e->stats.bytes_per_step = (sweep * e->maxIter + (double)e->n * perParticle) * e->subSteps * e->batch.K;
    *out = e->stats;
    return 0;
}

extern "C" int pbd_profile_step(pbd_engine *e, float *msPerType, float *msIntegrate, float *msVelocity, unsigned *launchesPerType) {
    if (!e) return fail("null engine");
    CKE(use(e)); CKE(flatten(e));
    if (e->mode != PBD_MODE_GRAPH && e->mode != PBD_MODE_LAUNCH) return fail("pbd_profile_step: per-bucket launches do not exist in this mode (select PBD_MODE_GRAPH or PBD_MODE_LAUNCH first)");
    CK(cudaStreamSynchronize(e->stream));
    // One event after every launch, all recorded in stream order without host synchronisation (a host sync per launch would time
    // the idle-launch latency, not the kernel); read back after one final sync.
    LaunchLog log;
    CKE(log.mark(e->stream, kLaunchStart));
    unsigned long long L = 0;
    const int rc = enqueue_step_launches(e, e->stream, &L, &log);
    const cudaError_t se = cudaStreamSynchronize(e->stream);
    if (msPerType) for (int t = 0; t < PBD_NUM_TYPES; t++) msPerType[t] = 0.0f;
    if (launchesPerType) for (int t = 0; t < PBD_NUM_TYPES; t++) launchesPerType[t] = 0;
    float mi = 0.0f, mv = 0.0f;
    if (!rc && se == cudaSuccess)
        for (size_t i = 1; i < log.ev.size(); i++) {
            float ms = 0.0f;
            cudaEventElapsedTime(&ms, log.ev[i - 1], log.ev[i]);
            const int what = log.what[i];
            if (what == kLaunchIntegrate) mi += ms;
            else if (what == kLaunchVelocity) mv += ms;
            else { if (msPerType) msPerType[what] += ms; if (launchesPerType) launchesPerType[what]++; }
        }
    if (rc) return rc;
    if (se != cudaSuccess) return fail("pbd_profile_step: %s", cudaGetErrorString(se));
    if (msIntegrate) *msIntegrate = mi;
    if (msVelocity) *msVelocity = mv;
    e->stats.steps++;
    e->stats.projections += (unsigned long long)e->numConstraints * e->subSteps * e->maxIter * e->batch.K;
    return 0;
}
