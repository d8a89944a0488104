// positionbaseddynamics_b200/csrc/host/image_plan.h
//
// The planner of the device image: constraints + colour groups (+ rest positions for the resident mode) -> every array the
// engine uploads, in host memory.  Host-only C++ (no CUDA API call): the engine gathers its inputs, plans, and uploads the
// result (engine.cu:flatten); the CPU tests run the same code on scenes of their own (tests/test_image_plan.py).
#pragma once
#include <functional>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>
#include "../device_image.h"
#include "pbd_model.h"

namespace pbd_b200 {

// PBD_B200_VERBOSE: flatten and the resident planner report their stages and timings on stderr
bool verbose();
// stage timings on stderr (PBD_B200_VERBOSE)
struct Lap {
    double prev;
    Lap();
    void operator()(const char *what);
};

// body k of a constraint of this type is a rigid body (else a particle)
inline bool is_rb_body(int type, int k) { return type == PBD_BALLJOINT || (type == PBD_RB_PARTICLE_BALLJOINT && k == 0); }
// Body indices of `count` constraints of one type against the particle and rigid-body counts, all threads.  Returns the position in
// `bodies` of the last index out of range, or -1.
long long bad_body_index(int type, const unsigned *bodies, size_t count, unsigned n, unsigned nRb);
// insertion id -> (type, local index) of the N constraints in store[PBD_NUM_TYPES]; "" or why the ids are not a permutation of 0..N-1
std::string build_id_map(const TypeStore *store, unsigned N, std::vector<std::pair<int, unsigned>> &map);

// The mode an image is planned for: `requested`, or for PBD_MODE_AUTO the resident mode where it is faster, else graph (plan_image falls
// back to graph where the resident mode refuses the model).  `replicas`: the size of the replica batch the image serves (pbd_set_replicas).
int preferred_mode(int requested, const TypeStore *store, unsigned n, unsigned numConstraints, unsigned replicas = 1);

// Clusters of C CTAs with `smem` bytes each the device keeps co-resident; a query of the type mask alone answers for every cluster shape.
struct ClusterQuery : std::function<int(unsigned mask, unsigned C, size_t smem)> {
    using function::function;
    template <class F, class = std::enable_if_t<std::is_invocable_r_v<int, F, unsigned>>> ClusterQuery(F f) : function([f](unsigned m, unsigned, size_t) { return f(m); }) {}
};

// What the planner needs to know about the model and, for the resident mode, about the device.
struct PlanInput {
    const TypeStore *store;                        // [PBD_NUM_TYPES] constraints by type, as added
    unsigned numConstraints, n, nRb;
    const std::vector<unsigned> *groupOff, *groupIds;  // the colour groups (CSR over insertion ids)
    int mode;                                      // the requested pbd_solver_mode (PBD_MODE_GRAPH = 0, PBD_MODE_RESIDENT = 1, ...)
    const float4 *x0;                              // resident: rest positions by host index
    unsigned forcedG, forcedC;                     // resident: G x C clusters x CTAs (PBD_B200_CLUSTERS), 0 = chosen from the model
    int smCount;
    ClusterQuery maxClusters;                      // resident: what the device keeps co-resident
    bool restTables = false;                       // replica batch with per-replica rest shapes: also TypePlan::restBodies / restLocal
    unsigned replicas = 1;                         // replica batch: every replica runs this one image (n, the constraints: one replica)
    bool replicaBodies = false;                    // replica batch: every replica has nRb rigid bodies of its own (pbd_set_replica_rigid_bodies)
};

// One constraint type's arrays in device order (the host side of pbdk::TypeArrays).
struct TypePlan {
    PodVector<unsigned> order;                     // device position -> insertion id
    PodVector<uint2> idx2; PodVector<uint4> idx4; PodVector<unsigned> idx3[3];
    PodVector<float4> gv[pbdk::kMaxGeoV];
    PodVector<float> gs[pbdk::kMaxGeoS], mat[pbdk::kMaxMat];  // mat[k] empty: every constraint has matU[k]
    float matU[pbdk::kMaxMat] = {};
    int variant = 0;
    // PlanInput::restTables: device position -> host particle indices of the bodies, and -> position among the type's constraints in the
    // order they were added (the per-replica geometry of pbd_set_replica_rest_positions is derived from these)
    PodVector<unsigned> restBodies, restLocal;
};

// Launch shape of a resident image: G clusters x C CTAs (one tile each), block size and type mask of the instantiation, smem per CTA.
// A replica batch (replicas > 1): the tables describe the C tiles of one replica, and each of the G clusters steps every G-th replica.
struct ResidentShape { unsigned G = 0, C = 0, threads = 0, xThreads = 0, mask = 0, tileCap = 0, nColours = 0, replicas = 1; size_t smem = 0; };

struct ImagePlan {
    int mode = PBD_MODE_GRAPH;                     // what the image runs in: the requested mode, PBD_MODE_AUTO resolved
    std::string residentRefusal;                   // PBD_MODE_AUTO fell back to the graph mode: why the resident mode refused the model
    std::vector<unsigned> slot;                    // host particle index -> device slot
    std::vector<pbdk::Bucket> buckets;             // colour after colour
    TypePlan types[PBD_NUM_TYPES];
    // resident only (resident.cuh: ResidentArgs)
    ResidentShape res;
    std::vector<unsigned> colourStart, tileOff, tileStart, tileSmem, xNbr, xMask;
};

// Why a batch of `replicas` replicas of n particles cannot run `mode` with these rigid bodies and constraints, or "" (also for one replica
// within the size limits).  plan_image checks it first; the engine also before it changes the batch size, the mode or the rigid bodies.
// Bodies and joints are admitted in a batch only where every replica has bodies of its own (replicaBodies).
std::string batch_refusal(unsigned replicas, unsigned n, int mode, unsigned nRb, const TypeStore *store, bool replicaBodies = false);

// Plans the image of `in` into `out`; returns "" or why the model cannot be flattened (for this mode and, resident, this device).
std::string plan_image(const PlanInput &in, ImagePlan &out);

// Device bytes an array of `bytes` takes: the L2 prefetch of a run (resident.cuh: l2_prefetch_bytes) rounds its end up to 16 bytes, so
// every streamed array is followed by 16 bytes of its own allocation.
inline size_t padded_bytes(size_t bytes) { return bytes + 16; }

// What the device addresses of an image's arrays become: every type's TypeArrays, the tables a batch's per-replica geometry is derived
// from (pbdk::DeriveArgs: TypePlan::restBodies / restLocal, and the insertion ids in device order), and the image-wide tables.  Every
// pointer in it has the representation of a char *.
struct RestTables { const unsigned *bodies, *local, *ids; };
struct ImageTables { const pbdk::Bucket *buckets; const unsigned *colourStart, *tileOff, *tileStart, *tileSmem, *xNbr, *xMask; unsigned long long *xFlags; };
struct ImagePointers { pbdk::TypeArrays types[PBD_NUM_TYPES]; RestTables rest[PBD_NUM_TYPES]; ImageTables tables; };

// One device array of an image: its name (the record of the CPU planner drivers), its host source or `zeroed` (the region starts zeroed),
// its place in the image's allocation, and the pointer of ImagePointers it becomes (`slot`: its byte offset there).
struct ImageArray { std::string name; const void *src; size_t bytes; bool zeroed; size_t slot, offset; };
struct ImageLayout { std::vector<ImageArray> arrays; size_t bytes = 0; };
// Every array the image `p` of a batch of `replicas` may hold, laid out in one allocation of `bytes` (arrays without bytes take no room):
// the plan's arrays, then the zeroed regions -- the XPBD multipliers and the resident mode's X arrival flags.  The sources point into `p`.
ImageLayout image_layout(const ImagePlan &p, unsigned replicas);

}  // namespace pbd_b200
