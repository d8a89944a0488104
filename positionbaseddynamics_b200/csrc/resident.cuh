// positionbaseddynamics_b200/csrc/resident.cuh
//
// k_step_resident: one TimeStepController::step (Simulation/TimeStepController.cpp:75-241) with the particle positions
// RESIDENT IN THE DISTRIBUTED SHARED MEMORY of thread-block clusters for the whole step.
//
// Why.  The per-bucket kernels are bound by L2 sector throughput on big scenes
// (every projection gathers and scatters 2-4 half-used 32-byte sectors through L2) and by the colour-phase dependency
// chain on small ones (cfg3: 3,700 dependent phases per step, however they are launched).  Both come
// from the same thing: positions live in L2 and every colour phase is a device-wide round trip.  Here
//   * the particles are partitioned spatially (host, recursive coordinate bisection) into G cluster regions x C tiles; CTA
//     (g, r) keeps its tile's positions in shared memory from the first integration to the last velocity update;
//   * a projection reaches a particle of a sibling tile of the same cluster through DSMEM (mapa + ld/st.shared::cluster),
//     so inside a cluster a colour phase ends with the hardware cluster barrier (barrier.cluster) instead of a
//     grid-wide atomic barrier or a kernel boundary;
//   * only particles touched by a constraint that spans two clusters stay in global memory ("global-homed").  The constraints
//     touching them ("X items") are run by dedicated warps of every CTA, which order themselves across CTAs through per-CTA
//     arrival flags: after its X items of phase p a CTA publishes its arrival count with st.release.gpu on its own flag, and
//     before its X items of phase p+1 it spins (ld.acquire.gpu, one lane per neighbour) on the flags of its NEIGHBOURS only --
//     the CTAs whose X items share a global-homed particle with its own, or touch one it is the home of (flatten time, at most
//     32).  A phase is thus no grid-wide barrier: a CTA waits for the few tiles around it, not for the slowest of all.  The
//     round trip overlaps the shared-memory work the other warps do in the meantime; those never touch the flags.  A scene that
//     fits one cluster (G = 1) has no X items.
//   Two regimes are used (host/image_plan.cpp:choose_resident_shape): ONE cluster of up to 16 CTAs for scenes whose colour phases are small
//   (cfg1 / cfg3 / cfg4), and G = #SMs clusters of ONE CTA for big scenes (cfg2 / cfg5: 132 independent CTAs on an H100; the SINGLE
//   instantiations: plain LDS / STS, __syncthreads).  A replica batch (pbd_set_replicas, the BATCH instantiations) tiles one replica
//   into one cluster of C CTAs and launches G such clusters; cluster g steps replicas g, g + G, ... one after the other.  The tables
//   are tile-local and shared by every cluster; only the particle and multiplier bases move with the replica.  No cluster waits for
//   another, so nothing beyond one cluster needs to be co-resident.
//   The order of the items inside a tile's run is chosen at flatten time so that the lanes of a quarter-warp hit distinct 16-byte
//   bank groups (host/image_plan.cpp:bank_group_fill).
//
// Exactness.  Colour phases are kept: inside a colour no two constraints share a particle (checked at flatten time),
// across colours every constraint reads exactly what the reference's sequential sweep would have produced, whichever CTA
// executes it.  The projection code is the one the per-bucket kernels inline (project_streamed_acc), compiled with
// -fmad=false + explicit fmaf, so the result is bit-identical to the graph / launch modes (tested).
//
// Index encoding: device_image.h (kSmemFlag).
// Constraint order inside a (colour,type) bucket: by executing tile, inside a tile the X items (touching a global-homed
// particle) first; tileOff[bucket][2t], [2t+1], [2t+2] delimit the two runs of tile t (relative to the bucket's `first`).
#pragma once
#include <type_traits>
#include <utility>
#include "kernels.cuh"

namespace pbdk {

// (the index encoding, tile swizzle, run table and shared-memory layout of the image are defined in device_image.h)
// PBD_B200_TRACE record per (phase, CTA): [0] phase start, [1] X items done, [2] other items done + colour arrive issued,
// [3] colour wait returned, [4] X wait returned (0 where the CTA has no X items in the phase); tools/trace_resident.py
constexpr unsigned kTraceSlots = 5;

struct ResidentArgs {
    float4 *pos, *vel, *oldp, *lastp;
    const Bucket *buckets;        // colour after colour
    const unsigned *colourStart;  // [nColours + 1] bucket ranges of the colours that own buckets
    const unsigned *tileOff;      // [nBuckets][2 nTiles + 1], relative to the bucket's `first`: tile t = [2t] X items.. [2t+1] others.. [2t+2]
    const unsigned *tileStart;    // [nTiles + 1] device slots: tile t owns [tileStart[t], tileStart[t+1])
    const unsigned *tileSmem;     // [nTiles] leading slots of the tile that live in shared memory; the rest is global-homed
    const unsigned *xNbr;         // [nTiles][kMaxXNeighbours] neighbours of every CTA (the CTAs whose X items it has to wait for)
    const unsigned *xMask;        // [nTiles][1 + nColours] bit k: neighbour k arrives in the integration phase / in colour c
    unsigned nBuckets, nColours, nTiles, subSteps, maxIter;
    unsigned tileCap;             // float4 slots reserved for the tile in every CTA's shared memory (>= the largest tileSmem)
    unsigned xThreads;            // the last xThreads threads of every CTA run the X items (and nothing else); 0 when there is one cluster
    unsigned clusterSize;         // CTAs per cluster (1: the colour barrier is a plain __syncthreads)
    int l2Prefetch;               // prefetch the next colour's operand runs into L2 (scenes whose constraint stream exceeds L2)
    float h, invH, twoInvH, gx, gy, gz;
    int secondOrder;
    unsigned long long *xFlags;   // [nTiles][kXFlagStride] arrival flag of every CTA: (launch ordinal << 32) | arrivals in this launch
    unsigned long long xLaunch;   // this launch's ordinal << 32 (the host counts resident launches: flags stay monotone across launches)
    RbState rb;                   // rigid bodies coupled through joints (global memory; single-cluster scenes only); a batch's replica r
                                  // at rows r x rb.n (pbd_set_replica_rigid_bodies)
    unsigned long long *trace;    // development aid (PBD_B200_TRACE): globaltimer per (phase, CTA, kTraceSlots)
    unsigned tracePhases;
    TypeArrays types[PBD_NUM_TYPES];
    // replica batch (BATCH instantiations): cluster g runs replicas g, g + G, ... of `replicas`; replica r's particles start at slot
    // r x replicaStride, its multipliers of type t at r x lamCount[t]
    unsigned replicas, replicaStride;
    unsigned lamCount[PBD_NUM_TYPES];
    // per-replica parameters of a batch (pbd_set_replica_materials / pbd_set_replica_gravity): rows of kMatRowFloats floats (the uniform
    // material parameters of every type) and rows of 3 floats (null: gx, gy, gz for every replica)
    const float *repMat, *repGravity;
    // per-replica rest shapes (pbd_set_replica_rest_positions): replica r's geometry of type t at r x geoCount[t] (0: shared)
    unsigned geoCount[PBD_NUM_TYPES];
    // per-constraint materials of every replica (pbd_set_replica_constraint_materials): replica r's of type t at r x matCount[t] (0: shared)
    unsigned matCount[PBD_NUM_TYPES];
    // external forces (pbd_set_external_forces): K x n float4 in slot order, read at integration only; null while none is set
    const float4 *force;
};

// ---- cluster primitives --------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned cluster_ctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ unsigned cluster_nctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}

// Particle accessors of the resident kernel.
//   ClusterAcc: an X item -- each particle is in the shared memory of a CTA of the cluster (DSMEM) or global-homed;
//   SmemAcc   : every other item -- shared memory only (the flag bit of the index is known to be set).
__device__ __forceinline__ unsigned dsmem_addr(unsigned tileBase, unsigned idx) {
    unsigned a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(tileBase + ((idx & kLocalMask) << 4)), "r"((idx >> kRankShift) & 15u));
    return a;
}
__device__ __forceinline__ float4 dsmem_ld(unsigned a) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void dsmem_st(unsigned a, const float4 &v) {
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" :: "r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
struct SmemAcc {
    typedef unsigned Handle;  // shared::cluster address
    unsigned tileBase;        // shared::cta address of this CTA's tile; the same offset in every CTA of the cluster
    __device__ __forceinline__ Handle handle(unsigned idx) const { return dsmem_addr(tileBase, idx); }
    __device__ __forceinline__ float4 ld(Handle h) const { return dsmem_ld(h); }
    __device__ __forceinline__ void st(Handle h, const float4 &v) const { if (v.w != 0.0f) dsmem_st(h, v); }  // static particles never move
};
struct ClusterAcc {
    typedef unsigned long long Handle;  // bit 63: shared::cluster address in the low word, else a global pointer
    float4 *pos;
    unsigned tileBase;
    __device__ __forceinline__ Handle handle(unsigned idx) const {
        return (idx & kSmemFlag) ? ((1ull << 63) | dsmem_addr(tileBase, idx)) : (unsigned long long)(pos + idx);
    }
    __device__ __forceinline__ float4 ld(Handle h) const { return (h >> 63) ? dsmem_ld((unsigned)h) : __ldcg((const float4 *)h); }
    __device__ __forceinline__ void st(Handle h, const float4 &v) const {
        if (v.w == 0.0f) return;
        if (h >> 63) dsmem_st((unsigned)h, v); else __stcg((float4 *)h, v);
    }
};

// One CTA per cluster (SINGLE instantiations: big scenes, one independent CTA per SM; tiny scenes, one CTA): every shared-memory
// particle is in this CTA's own tile -- plain LDS.128 / STS.128, no mapa, no cluster address space.
struct LocalAcc {
    typedef float4 *Handle;
    float4 *tile;
    __device__ __forceinline__ Handle handle(unsigned idx) const { return tile + (idx & kLocalMask); }
    __device__ __forceinline__ float4 ld(Handle h) const { return *h; }
    __device__ __forceinline__ void st(Handle h, const float4 &v) const { if (v.w != 0.0f) *h = v; }
};
struct LocalXAcc {
    typedef unsigned long long Handle;  // bit 63: offset into the tile in the low word, else a global pointer
    float4 *pos, *tile;
    __device__ __forceinline__ Handle handle(unsigned idx) const { return (idx & kSmemFlag) ? ((1ull << 63) | (idx & kLocalMask)) : (unsigned long long)(pos + idx); }
    __device__ __forceinline__ float4 ld(Handle h) const { return (h >> 63) ? tile[(unsigned)h] : __ldcg((const float4 *)h); }
    __device__ __forceinline__ void st(Handle h, const float4 &v) const {
        if (v.w == 0.0f) return;
        if (h >> 63) tile[(unsigned)h] = v; else __stcg((float4 *)h, v);
    }
};

__device__ __forceinline__ Bucket load_bucket(const Bucket *buckets, unsigned bi) {
    Bucket b;
    const int4 raw = __ldg(reinterpret_cast<const int4 *>(buckets) + bi);  // Bucket is 16 bytes
    b.type = raw.x; b.first = (unsigned)raw.y; b.count = (unsigned)raw.z; b.colour = (unsigned)raw.w;
    return b;
}

// L2 prefetch of a contiguous piece of a streamed array (cp.async.bulk.prefetch.L2: one instruction per <= 32 KB, no registers, no
// shared memory): issued one colour ahead, so that the operand loads of the next phase hit L2 instead of paying the DRAM latency on
// the dependency chain of every item (the per-sweep constraint stream of a big scene does not stay in L2 between sweeps).
__device__ __forceinline__ void l2_prefetch_bytes(const void *p, size_t bytes) {
    if (!p || !bytes) return;
    unsigned long long a = (unsigned long long)p, end = (a + bytes + 15ull) & ~15ull;
    a &= ~15ull;
    while (a < end) {
        const unsigned chunk = (unsigned)((end - a) < 32768ull ? (end - a) : 32768ull);
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(a), "r"(chunk) : "memory");
        a += chunk;
    }
}
// the per-constraint arrays of one type (indices, every geometry array, the multipliers from a.lambda + lamOff): array k of items
// [first, first + n), one array per calling lane
// (geoOff: a batch's replica with geometry of its own starts its geometry arrays there -- an offset rather than a replica_arrays copy,
// because the arrays are picked by the lane: a copy indexed at run time would live on the stack)
template <int T>
__device__ __forceinline__ void l2_prefetch_run(const TypeArrays &a, unsigned first, unsigned n, unsigned lane, size_t lamOff, size_t geoOff = 0) {
    constexpr TypeShape sh = type_shape(T);
    if (lane == 0) {
        if (sh.nBodies == 2) l2_prefetch_bytes(a.idx2 + first, (size_t)n * 8u);
        else if (sh.nBodies == 3) l2_prefetch_bytes(a.idx3[0] + first, (size_t)n * 4u);
        else l2_prefetch_bytes(a.idx4 + first, (size_t)n * 16u);
    } else if (lane <= 2) {
        if (sh.nBodies == 3) l2_prefetch_bytes(a.idx3[lane] + first, (size_t)n * 4u);
    } else if (lane < 3 + (unsigned)kMaxGeoV) {
        const unsigned k = lane - 3u;
        if ((int)k < sh.nGeoV && a.gv[k]) l2_prefetch_bytes(a.gv[k] + geoOff + first, (size_t)n * 16u);
    } else if (lane < 3 + (unsigned)kMaxGeoV + (unsigned)kMaxGeoS) {
        const unsigned k = lane - 3u - (unsigned)kMaxGeoV;
        if ((int)k < sh.nGeoS && a.gs[k]) l2_prefetch_bytes(a.gs[k] + geoOff + first, (size_t)n * 4u);
    } else if (lane == 3 + (unsigned)kMaxGeoV + (unsigned)kMaxGeoS) {
        if (sh.xpbd && a.lambda) l2_prefetch_bytes(a.lambda + lamOff + first, (size_t)n * 4u);
    }
}
constexpr unsigned kPrefetchLanes = 3u + (unsigned)kMaxGeoV + (unsigned)kMaxGeoS + 1u;

// What a thread fetched ahead of the colour barrier for its first item of the next phase: the streamed operands (immutable) and
// the XPBD multiplier (last written by this very thread one sweep ago), so that after the barrier only the gathers remain.
struct Prefetched { Streamed s; float lam; unsigned bucket; };

// types whose item loop keeps the next item's operands in flight (the register-heavy projections would spill with a second operand set)
template <int T> __device__ __forceinline__ constexpr bool is_pipelined() {
    return T == PBD_DISTANCE || T == PBD_DISTANCE_XPBD || T == PBD_ISOBENDING || T == PBD_ISOBENDING_XPBD || T == PBD_VOLUME || T == PBD_VOLUME_XPBD || T == PBD_FEMTRIANGLE || T == PBD_DIHEDRAL;
}
// ... and the ones light enough to keep TWO items ahead in flight (an L2 hit is ~300 cycles, one cloth projection ~60 issue slots)
template <int T> __device__ __forceinline__ constexpr bool is_pipelined2() { return T == PBD_DISTANCE_XPBD || T == PBD_ISOBENDING_XPBD || T == PBD_DISTANCE || T == PBD_ISOBENDING; }

// the multipliers of type T of replica `rep` of a batch start at A.types[T].lambda + lambda_offset
template <int T> __device__ __forceinline__ size_t lambda_offset(const ResidentArgs &A, unsigned rep) { return (size_t)rep * A.lamCount[T]; }

template <unsigned MASK, bool BATCH>
__device__ __forceinline__ void prefetch_first(const ResidentArgs &A, const RunEntry &r, unsigned bi, bool iterZero, unsigned tid, bool xRun, Prefetched &pre,
                                               unsigned rep) {
    pre.bucket = 0xffffffffu;
    const unsigned first = xRun ? r.firstX : r.firstR, n = xRun ? r.nX : r.nR;
    if (tid >= n) return;
    PBD_FOR_TYPE(MASK, r.type,
        pre.s = load_streamed<T>(A.types[T], first + tid, BATCH ? rep * A.geoCount[T] : 0u);
        if (type_shape(T).xpbd && !iterZero) pre.lam = __ldcg((BATCH ? A.types[T].lambda + lambda_offset<T>(A, rep) : A.types[T].lambda) + first + tid);
        pre.bucket = bi;)
}

// items [first, first + n) of a type's arrays: item tid, tid + stride, ... on this thread; with usePre the first one is in `pre`.
// Software pipelined: the streamed operands (and multiplier) of the next item are in flight while the current one is projected.
// A batch: `rows` is replica rep's material row, staged in shared memory (a global load at the head of every run would sit on the
// critical path of the colour phase); a batch's resident kernels take every uniform from it.
template <unsigned MASK, bool DEEP, bool BATCH, class Acc>
__device__ __forceinline__ void run_items(const ResidentArgs &A, const Acc &acc, int type, unsigned first, unsigned n, bool iterZero, unsigned tid, unsigned stride,
                                          bool usePre, const Prefetched &pre, unsigned rep, const float *rows) {
    PBD_FOR_TYPE(MASK, type,
        TypeArrays batchArrays;  // a batch: the arrays with replica rep's multipliers
        if (BATCH) batchArrays = replica_arrays(A.types[T], rep, A.lamCount[T], 0u);
        const unsigned go = BATCH ? rep * A.geoCount[T] : 0u;  // replica rep's geometry (pbd_set_replica_rest_positions; 0: shared)
        const unsigned mo = BATCH ? rep * A.matCount[T] : 0u;  // ... and materials (pbd_set_replica_constraint_materials; 0: shared)
        const unsigned ro = BATCH ? rep * A.rb.n : 0u;         // ... and rigid bodies (pbd_set_replica_rigid_bodies)
        MatRow matRow;
        if (BATCH) { matRow = load_mat_row<T>(rows + mat_offset(T)); matRow.on = true; }
        const TypeArrays &ta = BATCH ? batchArrays : A.types[T];
        unsigned i = tid;
        if (DEEP && is_pipelined2<T>()) {
            if (i < n) {
                auto fetch = [&](unsigned k, Streamed &sx, float &lx) { sx = load_streamed<T>(ta, first + k, go); if (type_shape(T).xpbd && !iterZero) lx = __ldcg(ta.lambda + first + k); };
                Streamed s0, s1, s2; float l0 = 0.0f, l1 = 0.0f, l2 = 0.0f;
                if (usePre) { s0 = pre.s; l0 = pre.lam; } else fetch(i, s0, l0);
                bool h1 = i + stride < n;
                if (h1) fetch(i + stride, s1, l1);
                _Pragma("unroll 1")
                for (;;) {
                    const unsigned j2 = i + 2u * stride;
                    const bool h2 = j2 < n;
                    if (h2) fetch(j2, s2, l2);
                    project_streamed_acc<T, Acc, 0>(acc, ta, first + i, s0, A.h, iterZero, true, l0, matRow, go, mo, ro);
                    if (!h1) break;
                    s0 = s1; l0 = l1; s1 = s2; l1 = l2; h1 = h2; i += stride;
                }
            }
        } else
        if (i < n) {
            Streamed cur; float lam = 0.0f;
            if (usePre) { cur = pre.s; lam = pre.lam; }
            else { cur = load_streamed<T>(ta, first + i, go); if (type_shape(T).xpbd && !iterZero) lam = __ldcg(ta.lambda + first + i); }
            _Pragma("unroll 1")
            for (;;) {
                const unsigned j = i + stride;
                const bool more = j < n;
                Streamed nxt; float lamN = 0.0f;
                if (is_pipelined<T>() && more) { nxt = load_streamed<T>(ta, first + j, go); if (type_shape(T).xpbd && !iterZero) lamN = __ldcg(ta.lambda + first + j); }
                project_streamed_acc<T, Acc, 0>(acc, ta, first + i, cur, A.h, iterZero, true, lam, matRow, go, mo, ro);  // variant 0 only: flatten refuses the full-Q bending layout in this mode
                if (!more) break;
                if (!is_pipelined<T>()) { nxt = load_streamed<T>(ta, first + j, go); if (type_shape(T).xpbd && !iterZero) lamN = __ldcg(ta.lambda + first + j); }
                cur = nxt; lam = lamN; i = j;
            }
        })
}

// semi-implicit Euler of one particle whose position is `x` (TimeStepController.cpp:112-118, TimeIntegration.cpp:7-19), with its external
// force at `slot` while forces are set (the substep prologue is the only place that tests A.force)
__device__ __forceinline__ bool integrate_particle(const ResidentArgs &A, unsigned slot, float4 &x, float gx, float gy, float gz) {
    __stcs(A.lastp + slot, __ldcs(A.oldp + slot));
    __stcs(A.oldp + slot, x);
    float4 v = __ldcs(A.vel + slot);
    if (v.w == 0.0f) return false;  // v.w carries the mass
    if (A.force) external_acceleration(gx, gy, gz, __ldcs(A.force + slot), x.w);
    semi_implicit_euler(x, v, A.h, gx, gy, gz);
    __stcs(A.vel + slot, v);
    return true;
}
// velocity update of one particle whose position is `x` (TimeIntegration.cpp:42-51, 69-79)
__device__ __forceinline__ void velocity_particle(const ResidentArgs &A, unsigned slot, const float4 &x) {
    if (x.w == 0.0f) return;
    const float4 o = __ldcs(A.oldp + slot);
    float4 v = __ldcs(A.vel + slot);
    velocity_update(v, x, o, A.invH, A.secondOrder, [&] { return __ldcs(A.lastp + slot); });
    __stcs(A.vel + slot, v);
}

// X warps of a CTA act as one party of the flag protocol (one arrival per CTA and phase, one poller per neighbour).  Named barrier 1
// synchronises the CTA's XT threads (whole warps).
//   wait  : lane k of the first X warp spins until neighbour k's flag shows every arrival of the earlier phases this CTA depends on
//           (ld.acquire.gpu; `target` = launch ordinal | arrivals, `spin` false when there is none), then the barrier releases the X warps;
//   arrive: after the X warps' stores -- barrier (orders them before the first X thread), then that thread publishes its CTA's arrival
//           count with st.release.gpu (the fence is cumulative over what the barrier ordered: the cooperative-groups grid.sync pattern).
__device__ __forceinline__ void x_bar(unsigned xThreads) { asm volatile("bar.sync 1, %0;" :: "r"(xThreads) : "memory"); }
__device__ __forceinline__ void x_wait(const unsigned long long *peer, unsigned long long target, bool spin, unsigned xThreads) {
    if (spin)
        while (ld_acquire_u64(peer) < target) { }
    x_bar(xThreads);
}
__device__ __forceinline__ void x_arrive(unsigned long long *flag, unsigned long long value, unsigned xtid, unsigned xThreads) {
    x_bar(xThreads);
    if (xtid == 0) st_release_u64(flag, value);
}

// colour barrier of the cluster: arrive (publishes this thread's shared-memory stores), then wait; one CTA: a block barrier
__device__ __forceinline__ void colour_arrive(bool single) { if (!single) cluster_arrive(); }
__device__ __forceinline__ void colour_wait(bool single) { if (single) __syncthreads(); else cluster_wait(); }

// BATCH: a replica batch (one cluster's tiling of ONE replica, no X items); cluster g steps replicas g, g + G, ... one after the other,
// each a whole step from the tile load to the tile store, and never waits for another cluster.
template <unsigned MASK, int THREADS, bool SINGLE, bool BATCH>
__global__ void __launch_bounds__(THREADS, 1) k_step_resident(const __grid_constant__ ResidentArgs A) {
    extern __shared__ float4 tile[];
    RunEntry *runs = reinterpret_cast<RunEntry *>(tile + A.tileCap);
    unsigned *sMask = reinterpret_cast<unsigned *>(runs + A.nBuckets);  // [1 + nColours]
    unsigned *sColour = sMask + 1 + A.nColours;                         // [nColours + 1]
    unsigned *sNbr = sColour + 1 + A.nColours;                          // [kMaxXNeighbours]
    float *const sRep = reinterpret_cast<float *>(sNbr);                // a batch (no X items): the current replica's material row, then its gravity
    const unsigned cta = BATCH ? blockIdx.x % A.clusterSize : blockIdx.x;  // tile id = cluster * C + rank (1-D grid, cluster dimension C); a batch: the rank
    const unsigned tile0 = __ldg(A.tileStart + cta), nSm = __ldg(A.tileSmem + cta), nAll = __ldg(A.tileStart + cta + 1) - tile0;
    unsigned rep = BATCH ? blockIdx.x / A.clusterSize : 0u;  // the replica this cluster steps
    unsigned t0 = tile0 + (BATCH ? rep * A.replicaStride : 0u);
    const unsigned nGl = nAll - nSm;
    // thread roles: the first RT threads run the shared-memory items; the last XT threads (whole warps) run the X items and the
    // global-homed particles and are the only ones that ever wait for another cluster
    // (a batch tiles one replica into one cluster: it has no X items, and its instantiations no X path -- that is where the registers
    // for the replica's parameters come from)
    const unsigned XT = BATCH ? 0u : A.xThreads, RT = THREADS - XT;
    const bool isX = !BATCH && threadIdx.x >= RT;
    const unsigned xtid = threadIdx.x - RT;
    // rigid bodies: stepped by CTA 0 of the cluster, replica rep's at rows rep x rb.n.  A batch's instantiations without the joint types
    // have no body path (the planner gives a batch with bodies the solid or the all-types instantiation).  A batch updates a substep's body
    // velocities at the head of the next substep, in the thread that integrates the body next, and the last substep's after the launch
    // (k_rb_velocity_batch, engine.cu): the same arithmetic, but no body code after the colour phases, where the batched solid kernel
    // would spill more.
    constexpr bool bodies = !BATCH || (MASK & (type_bit(PBD_BALLJOINT) | type_bit(PBD_RB_PARTICLE_BALLJOINT))) != 0u;
    constexpr bool single = SINGLE;  // one CTA per cluster: plain shared-memory accesses, __syncthreads between colours
    typedef typename std::conditional<SINGLE, LocalXAcc, ClusterAcc>::type XAcc;
    typedef typename std::conditional<SINGLE, LocalAcc, SmemAcc>::type RAcc;
    XAcc accX; RAcc accR;
    if constexpr (SINGLE) { accX.pos = A.pos; accX.tile = tile; accR.tile = tile; }
    else { accX.pos = A.pos; accX.tileBase = smem_u32(tile); accR.tileBase = smem_u32(tile); }
    // flag protocol (X threads only): lane k of the first X warp counts the arrivals of neighbour k up to the current phase
    unsigned xNeed = 0, xArrivals = 0;  // ... and every X thread this CTA's own
    unsigned long long *const xFlag = A.xFlags + (size_t)cta * kXFlagStride;
    const bool xLane = isX && xtid < kMaxXNeighbours;
    auto x_count = [&](unsigned p) { if (xLane) xNeed += (sMask[p] >> xtid) & 1u; };  // after phase p (0: integration, 1 + c: colour c)
    auto x_publish = [&]() { x_arrive(xFlag, A.xLaunch | ++xArrivals, xtid, XT); };
    auto x_peer = [&]() { return A.xFlags + (size_t)sNbr[xtid & (kMaxXNeighbours - 1u)] * kXFlagStride; };  // neighbour xtid's flag
    unsigned phase = 0;
    auto stamp = [&](unsigned k) {
        if (A.trace && phase < A.tracePhases && (threadIdx.x == 0 || ((k == 1 || k == 4) && threadIdx.x == RT)))
            A.trace[((size_t)phase * gridDim.x + cta) * kTraceSlots + k] = globaltimer_ns();
    };
    auto x_sync = [&]() { x_wait(x_peer(), A.xLaunch | xNeed, xLane && xNeed != 0u, XT); stamp(4); };

    // ---- once per launch: the tile and this CTA's view of the phase structure go to shared memory (after a cluster barrier L1 is
    // invalid, so anything read per phase from global memory would cost an L2 round trip on the critical path of every colour)
    for (unsigned i = threadIdx.x; i < nSm; i += THREADS) tile[tile_swizzle(i)] = __ldcg(A.pos + t0 + i);
    for (unsigned bi = threadIdx.x; bi < A.nBuckets; bi += THREADS) {
        const Bucket b = load_bucket(A.buckets, bi);
        const unsigned *off = A.tileOff + (size_t)bi * (2u * A.nTiles + 1u) + 2u * cta;
        const unsigned o0 = __ldg(off), o1 = __ldg(off + 1), o2 = __ldg(off + 2);
        RunEntry r; r.type = b.type; r.firstX = b.first + o0; r.nX = o1 - o0; r.firstR = b.first + o1; r.nR = o2 - o1; r.rotR = r.pad0 = r.pad1 = 0u;
        runs[bi] = r;
    }
    for (unsigned i = threadIdx.x; i < 1u + A.nColours; i += THREADS) { sMask[i] = __ldg(A.xMask + (size_t)cta * (1u + A.nColours) + i); sColour[i] = __ldg(A.colourStart + i); }
    if (!BATCH && threadIdx.x < kMaxXNeighbours) sNbr[threadIdx.x] = __ldg(A.xNbr + (size_t)cta * kMaxXNeighbours + threadIdx.x);
    auto stage_replica = [&]() {  // once per replica, so that no colour phase starts with a load from global memory
        if (A.repMat && threadIdx.x < (unsigned)kMatRowFloats) sRep[threadIdx.x] = __ldg(A.repMat + (size_t)rep * kMatRowFloats + threadIdx.x);
        if (threadIdx.x < 3u)
            sRep[kMatRowFloats + threadIdx.x] = A.repGravity ? __ldg(A.repGravity + 3u * rep + threadIdx.x) : (threadIdx.x == 0u ? A.gx : (threadIdx.x == 1u ? A.gy : A.gz));
    };
    if (BATCH) stage_replica();
    __syncthreads();
    for (unsigned c = threadIdx.x; c < A.nColours; c += THREADS) {  // rotations: bucket k of a colour starts where bucket k-1 ended
        unsigned accR = 0;
        for (unsigned bi = sColour[c]; bi < sColour[c + 1]; bi++) {
            runs[bi].rotR = (accR % RT) & ~7u; accR += runs[bi].nR;  // multiple of 8: the quarter-warps of a run stay aligned with its item order
        }
    }
    __syncthreads();
    Prefetched pre;
    pre.bucket = 0xffffffffu; pre.lam = 0.0f;
    for (;;) {  // the replicas of this cluster (one pass outside a batch)
        if (!single) { cluster_arrive(); cluster_wait(); }  // every tile of the cluster is loaded (and every CTA has started) before the first DSMEM access

        for (unsigned sub = 0; sub < A.subSteps; sub++) {
            // ---- prologue: lastX = oldX; oldX = x; semi-implicit Euler
            stamp(0);
            const float gx = BATCH ? sRep[kMatRowFloats] : A.gx, gy = BATCH ? sRep[kMatRowFloats + 1] : A.gy, gz = BATCH ? sRep[kMatRowFloats + 2] : A.gz;
            if (isX) {  // global-homed particles: what other clusters wait for
                for (unsigned i = xtid; i < nGl; i += XT) {
                    float4 x = __ldcg(A.pos + t0 + nSm + i);
                    if (integrate_particle(A, t0 + nSm + i, x, gx, gy, gz)) __stcg(A.pos + t0 + nSm + i, x);
                }
                if (nGl) x_publish();
                stamp(1);
            } else {
                for (unsigned i = threadIdx.x; i < nSm; i += RT) {
                    float4 x = tile[tile_swizzle(i)];
                    if (integrate_particle(A, t0 + i, x, gx, gy, gz)) tile[tile_swizzle(i)] = x;
                }
                if (bodies && cta == 0) {  // every body, in CTA 0: with G > 1 no joint reads them, in one cluster the cluster barrier orders them
                    const unsigned r0 = BATCH ? rep * A.rb.n : 0u;
                    for (unsigned i = threadIdx.x; i < A.rb.n; i += RT) {
                        if (BATCH && sub) rb_velocity_body(A.rb, r0 + i, A.invH, A.twoInvH, A.secondOrder);  // the previous substep's
                        rb_integrate_body(A.rb, r0 + i, A.h, gx, gy, gz);
                    }
                }
            }
            x_count(0);
            colour_arrive(single);
            if (A.nColours) prefetch_first<MASK, BATCH>(A, runs[sColour[0]], sColour[0], true, isX ? xtid : threadIdx.x, isX, pre, rep);
            stamp(2); colour_wait(single); stamp(3);
            phase++;

            // ---- coloured Gauss-Seidel sweeps (TimeStepController.cpp:270-286)
            for (unsigned it = 0; it < A.maxIter; it++) {
                const bool iterZero = (it == 0);
                for (unsigned c = 0; c < A.nColours; c++) {
                    const unsigned b0 = sColour[c], b1 = sColour[c + 1];
                    stamp(0);
                    if (A.l2Prefetch && !isX && (threadIdx.x & 31u) == 0u) {  // the next colour's operand runs of this CTA start travelling DRAM -> L2 now
                        // one array per R warp (lane 0): the colour barrier waits for the slowest warp, and the arrays issued by the lanes of
                        // one warp would go one divergent path after the other; the X warps stay free for their cross-tile chain
                        const unsigned cn = (c + 1 == A.nColours) ? 0u : c + 1u;
                        for (unsigned k = threadIdx.x >> 5; k < kPrefetchLanes; k += RT >> 5)
                            for (unsigned bi = sColour[cn]; bi < sColour[cn + 1]; bi++) {
                                const RunEntry r = runs[bi];
                                PBD_FOR_TYPE(MASK, r.type, l2_prefetch_run<T>(A.types[T], r.firstX, r.nX + r.nR, k, BATCH ? lambda_offset<T>(A, rep) : 0u,
                                                                              BATCH ? (size_t)rep * A.geoCount[T] : 0u);)
                            }
                    }
                    if (isX) {
                        // X items of every bucket of the colour: they touch global-homed particles and are ordered across CTAs by the flags
                        bool mine = false;  // CTA-uniform: does this CTA own an X item of this colour?
                        for (unsigned bi = b0; bi < b1; bi++) mine = mine || (runs[bi].nX != 0u);
                        if (mine) {
                            x_sync();
    #pragma unroll 1
                            for (unsigned bi = b0; bi < b1; bi++) run_items<MASK, false, BATCH>(A, accX, runs[bi].type, runs[bi].firstX, runs[bi].nX, iterZero, xtid, XT, pre.bucket == bi, pre,
                                                                                         BATCH ? rep : 0u, sRep);
                            x_publish();
                        }
                        stamp(1);
                    } else {
                        // everything else: shared memory of this cluster only
    #pragma unroll 1
                        for (unsigned bi = b0; bi < b1; bi++) {
                            const unsigned rot = runs[bi].rotR;  // 0 for the first bucket of a colour (the one prefetch_first serves)
                            run_items<MASK, SINGLE && MASK == kMaskClothXPBD, BATCH>(A, accR, runs[bi].type, runs[bi].firstR, runs[bi].nR, iterZero,
                                                                               threadIdx.x >= rot ? threadIdx.x - rot : threadIdx.x + RT - rot, RT, pre.bucket == bi, pre,
                                                                               BATCH ? rep : 0u, sRep);
                        }
                    }
                    x_count(1u + c);
                    colour_arrive(single);
                    {   // this thread's first item of the next colour streams in while the CTAs synchronise
                        const bool lastColour = (c + 1 == A.nColours);
                        if (!lastColour || it + 1 < A.maxIter) {
                            const unsigned nb = sColour[lastColour ? 0u : c + 1u];
                            prefetch_first<MASK, BATCH>(A, runs[nb], nb, false, isX ? xtid : threadIdx.x, isX, pre, rep);
                        } else pre.bucket = 0xffffffffu;
                    }
                    stamp(2); colour_wait(single); stamp(3);
                    phase++;
                }
            }

            // ---- epilogue: velocity update (own particles only; the global-homed ones need the last X items of every neighbour)
            if (isX) {
                if (nGl) x_wait(x_peer(), A.xLaunch | xNeed, xLane && xNeed != 0u, XT);
                for (unsigned i = xtid; i < nGl; i += XT) velocity_particle(A, t0 + nSm + i, __ldcg(A.pos + t0 + nSm + i));
            } else {
                for (unsigned i = threadIdx.x; i < nSm; i += RT) velocity_particle(A, t0 + i, tile[tile_swizzle(i)]);
                if (!BATCH && cta == 0)  // (a batch: at the head of the next substep)
                    for (unsigned i = threadIdx.x; i < A.rb.n; i += RT) rb_velocity_body(A.rb, i, A.invH, A.twoInvH, A.secondOrder);
            }
        }
        for (unsigned i = threadIdx.x; i < nSm; i += THREADS) __stcg(A.pos + t0 + i, tile[tile_swizzle(i)]);
        if (!BATCH) break;
        rep += gridDim.x / A.clusterSize;
        if (rep >= A.replicas) break;
        t0 = tile0 + rep * A.replicaStride;
        __syncthreads();  // the last replica's tile is stored before the next one overwrites it (no other CTA reads it after the last colour barrier)
        stage_replica();
        for (unsigned i = threadIdx.x; i < nSm; i += THREADS) tile[tile_swizzle(i)] = __ldcg(A.pos + t0 + i);
        __syncthreads();
    }
}

}  // namespace pbdk
