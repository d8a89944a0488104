// positionbaseddynamics_b200/csrc/host/image_plan.cpp
//
// The image planner (image_plan.h): a constraint list + the reference's colour groups -> (colour,type) buckets of SoA arrays; for the
// resident mode (resident.cuh) also the tiling of the particles, the per-tile runs and the X-neighbour tables.  No CUDA API call.
#include "image_plan.h"
#include "../rest_geometry.cuh"
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <omp.h>
#include <parallel/algorithm>  // libstdc++ parallel mode (OpenMP): the per-bucket sorts

namespace pbd_b200 {
using namespace pbdk;

bool verbose() {
    static const bool v = getenv("PBD_B200_VERBOSE") != nullptr;
    return v;
}
Lap::Lap() : prev(omp_get_wtime()) {}
void Lap::operator()(const char *what) {
    if (!verbose()) return;
    const double t = omp_get_wtime();
    fprintf(stderr, "[pbd_b200] flatten: %-34s %.3f s\n", what, t - prev);
    prev = t;
}

static std::string fmt(const char *f, ...) {
    char buf[1024];
    va_list ap; va_start(ap, f); vsnprintf(buf, sizeof(buf), f, ap); va_end(ap);
    return buf;
}

long long bad_body_index(int type, const unsigned *bodies, size_t count, unsigned n, unsigned nRb) {
    const int nb = type_shape(type).nBodies;
    long long badAt = -1;
    #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(max : badAt) if (count * nb > 100000)
    for (long long c = 0; c < (long long)count; c++)
        for (int k = 0; k < nb; k++) {
            const long long i = c * nb + k;
            if (bodies[i] >= (is_rb_body(type, k) ? nRb : n)) badAt = std::max(badAt, i);
        }
    return badAt;
}

std::string build_id_map(const TypeStore *store, unsigned N, std::vector<std::pair<int, unsigned>> &map) {
    map.resize(N);
    PodVector<int> seenType(N);
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (long long i = 0; i < (long long)N; i++) seenType[i] = -1;
    for (int t = 0; t < PBD_NUM_TYPES; t++) {
        const TypeStore &h = store[t];
        long long bad = -1; int dup = 0;
        #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(max : bad) reduction(| : dup) if (h.ids.size() > 50000)
        for (long long i = 0; i < (long long)h.ids.size(); i++) {
            const unsigned id = h.ids[i];
            if (id >= N) { bad = std::max(bad, (long long)id); continue; }
            if (__atomic_exchange_n(&seenType[id], t, __ATOMIC_RELAXED) != -1) { dup = 1; bad = std::max(bad, (long long)id); continue; }
            map[id] = std::make_pair(t, (unsigned)i);
        }
        if (bad >= 0 && !dup) return fmt("constraint id %u out of range (N=%u)", (unsigned)bad, N);
        if (dup) return fmt("constraint id %u used twice", (unsigned)bad);
    }
    return "";  // N ids, all below N, none twice: a permutation
}

// the particle / rigid-body counts may have shrunk since the constraints were added (pbd_set_particles, pbd_set_rigid_bodies)
static std::string validate_bodies(const PlanInput &in) {
    for (int t = 0; t < PBD_NUM_TYPES; t++) {
        const TypeStore &h = in.store[t];
        const long long badAt = bad_body_index(t, h.bodies.data(), h.ids.size(), in.n, in.nRb);
        if (badAt < 0) continue;
        const bool isRb = is_rb_body(t, (int)(badAt % type_shape(t).nBodies));
        return fmt("constraint of type %d refers to %s %u, but the engine holds %u: re-add the constraints after shrinking the model", t,
                   isRb ? "rigid body" : "particle", h.bodies[badAt], isRb ? in.nRb : in.n);
    }
    return "";
}

// The planner's state: its input, the plan being built, and for the resident mode where every host particle lives.
struct Ctx {
    const PlanInput &in;
    ImagePlan &out;
    bool tiled;                               // the resident mode's image
    std::vector<unsigned> tileOf;             // host particle -> tile (cluster = tile / C, rank = tile % C)
    std::vector<unsigned char> homedGlobal;   // host particle lives in global memory (touched by a constraint run in another tile)
    std::vector<unsigned> owner[PBD_NUM_TYPES];  // independent CTAs: local index of a constraint -> its owner tile (else empty)
    unsigned nTiles() const { return out.res.G * out.res.C; }
};

// Resident mode (resident.cuh): the particles are partitioned into G cluster regions x C tiles by recursive coordinate
// bisection of the rest positions; the device arrays are permuted to tile-major order.
static void bisect(std::vector<unsigned> &idx, size_t lo, size_t hi, unsigned t0, unsigned nt, const float4 *x, std::vector<unsigned> &tileOf) {
    if (nt == 1) { for (size_t i = lo; i < hi; i++) tileOf[idx[i]] = t0; return; }
    float mn[3] = {3.4e38f, 3.4e38f, 3.4e38f}, mx[3] = {-3.4e38f, -3.4e38f, -3.4e38f};
    for (size_t i = lo; i < hi; i++) {
        const float4 &p = x[idx[i]];
        const float c[3] = {p.x, p.y, p.z};
        for (int k = 0; k < 3; k++) { mn[k] = std::min(mn[k], c[k]); mx[k] = std::max(mx[k], c[k]); }
    }
    int ax = 0;
    for (int k = 1; k < 3; k++) if (mx[k] - mn[k] > mx[ax] - mn[ax]) ax = k;
    const unsigned ntL = nt / 2;
    const size_t mid = lo + (size_t)((double)(hi - lo) * ntL / nt);
    auto key = [&](unsigned i) { const float4 &p = x[i]; return ax == 0 ? p.x : (ax == 1 ? p.y : p.z); };
    std::nth_element(idx.begin() + lo, idx.begin() + mid, idx.begin() + hi, [&](unsigned a, unsigned b) { const float ka = key(a), kb = key(b); return ka < kb || (ka == kb && a < b); });
    // the two halves are independent: run them as tasks while they are big enough to pay for it
    #pragma omp task shared(idx, x, tileOf) if (hi - lo > 65536)
    bisect(idx, lo, mid, t0, ntL, x, tileOf);
    bisect(idx, mid, hi, t0 + ntL, nt - ntL, x, tileOf);
    #pragma omp taskwait
}

// Executing tile of constraint `local` of type t: its owner with independent CTAs (every shared-memory particle of it is homed there);
// else the tile that holds most of its shared-memory particles (ties: the lowest tile); none -> the tile of its first particle (0 for a
// joint between rigid bodies).  *touchesGlobal: one of its particles is global-homed.
static inline unsigned exec_tile(const Ctx &c, int t, unsigned local, bool *touchesGlobal) {
    const int nb = type_shape(t).nBodies;
    const unsigned *b = &c.in.store[t].bodies[(size_t)local * nb];
    const std::vector<unsigned> &tileOf = c.tileOf;
    const std::vector<unsigned char> &homedGlobal = c.homedGlobal;
    bool x = false;
    unsigned best = 0xffffffffu, bestCnt = 0, first = 0xffffffffu;
    for (int k = 0; k < nb; k++) {
        if (is_rb_body(t, k)) continue;
        if (first == 0xffffffffu) first = tileOf[b[k]];
        if (homedGlobal[b[k]]) { x = true; continue; }
        unsigned cnt = 0;
        for (int j = 0; j < nb; j++) cnt += (!is_rb_body(t, j) && !homedGlobal[b[j]] && tileOf[b[j]] == tileOf[b[k]]);
        if (cnt > bestCnt || (cnt == bestCnt && tileOf[b[k]] < best)) { best = tileOf[b[k]]; bestCnt = cnt; }
    }
    *touchesGlobal = x;
    if (!c.owner[t].empty()) return c.owner[t][local];
    return (best != 0xffffffffu) ? best : (first != 0xffffffffu ? first : 0u);
}

// Independent CTAs (G > 1, C = 1): homing by constraint owner.  A constraint's owner is the tile that holds most of its particles
// (ties: the lowest tile; rigid bodies do not count), and the owner runs it.  A particle stays in the shared memory of its tile when
// every constraint through it is owned there, else it is global-homed (its tile still integrates it and updates its velocity).  So an
// item's shared-memory particles are always its owner's, and a constraint across a cut makes global only its particles outside its
// owner.  Making global every particle of a constraint whose particles lie in two tiles (the cluster regimes' rule) puts a band as wide
// as the widest stencil (a bending constraint: two cells) on both sides of every cut: at cfg2 10.4 % X items and 6.5 % global-homed
// particles, against 6.4 % and 3.3 % here (DESIGN.md section 6).  The tiles stay the particles' bisection, so each holds its share of
// the particles whatever the constraints are.
static void home_by_owner(Ctx &c) {
    const unsigned *tileOf = c.tileOf.data();
    unsigned char *hg = c.homedGlobal.data();
    for (int t = 0; t < PBD_NUM_TYPES; t++) {
        const TypeStore &h = c.in.store[t];
        const int nb = type_shape(t).nBodies;
        std::vector<unsigned> &owner = c.owner[t];
        owner.assign(h.ids.size(), 0u);
        #pragma omp parallel for schedule(static) num_threads(host_threads())
        for (long long k0 = 0; k0 < (long long)h.ids.size(); k0++) {
            const unsigned *b = &h.bodies[(size_t)k0 * nb];
            unsigned best = 0xffffffffu, bestCnt = 0;
            for (int k = 0; k < nb; k++) {
                if (is_rb_body(t, k)) continue;
                unsigned cnt = 0;
                for (int j = 0; j < nb; j++) cnt += (!is_rb_body(t, j) && tileOf[b[j]] == tileOf[b[k]]);
                if (cnt > bestCnt || (cnt == bestCnt && tileOf[b[k]] < best)) { best = tileOf[b[k]]; bestCnt = cnt; }
            }
            if (best == 0xffffffffu) continue;  // no particle (a joint between rigid bodies): tile 0
            owner[k0] = best;
            for (int k = 0; k < nb; k++)
                if (!is_rb_body(t, k) && tileOf[b[k]] != best) hg[b[k]] = 1;  // every writer stores the same byte
        }
    }
}

// shape of the launch: type mask / block size of the instantiation, clusters x CTAs per cluster
static std::string choose_resident_shape(const PlanInput &in, ResidentShape &r) {
    unsigned present = 0, nTypes = 0;
    for (int t = 0; t < PBD_NUM_TYPES; t++) if (!in.store[t].ids.empty()) { present |= 1u << t; nTypes++; }
    // the leanest instantiation that covers the model; a batch with rigid bodies one with the joint types, whose batched form steps them
    constexpr unsigned joints = type_bit(PBD_BALLJOINT) | type_bit(PBD_RB_PARTICLE_BALLJOINT);
    const bool batchBodies = in.replicas > 1 && (in.nRb || (present & joints));
    r.mask = kMaskAll;
    for (unsigned m : {kMaskClothXPBD, kMaskCloth, kMaskFem, kMaskLight, kMaskSolid})
        if ((present & ~m) == 0 && (!batchBodies || (m & joints) == joints)) { r.mask = m; break; }
    r.threads = resident_threads(r.mask, in.replicas > 1);
    const unsigned nGroups = (unsigned)std::max<size_t>(in.groupOff->size(), 2) - 1;
    const unsigned perPhase = in.numConstraints / std::max(1u, nGroups);
    // particles a tile can hold: what is left of the CTA's shared memory after the phase tables (bound: one bucket per colour and type)
    const size_t tables = resident_smem_bytes(0u, nGroups * std::max(1u, nTypes), nGroups);
    if (tables + 1024 * sizeof(float4) > kMaxDynamicSmem) return fmt("resident mode: %u colour groups need %zu bytes of phase tables (use PBD_MODE_GRAPH)", nGroups, tables);
    const unsigned cap = (unsigned)(0.97 * (double)((kMaxDynamicSmem - tables) / sizeof(float4)));  // bisection splits counts evenly; slack for rounding
    unsigned G = 1, C = 1;
    const bool oneCluster = in.n <= (unsigned)kMaxClusterCtas * cap && perPhase <= (unsigned)kMaxClusterCtas * 1024u;
    if (in.replicas > 1) {
        // A batch tiles one replica into one cluster of C CTAs; G clusters (plan_mode) step the replicas one after the other.  Smaller
        // clusters run more replicas at once, larger ones step each replica faster.  C: one CTA when a replica fits one (no cluster
        // barrier at all); else the largest C up to the single-scene choice below whose clusters the device runs all at once, else the
        // smallest C that holds the replica.  H100 80GB HBM3 (700 W), ms per batched step (tools/bench_batch.py, C forced):
        //   cfg1 (2,500 particles, fits one CTA), C = 1 / 2 / 4 / 8 / 16:  K = 8  0.147 / 0.193 / 0.186 / 0.185 / 0.342,
        //        K = 132  0.151 / 0.394 / 0.923 / 1.640 / 3.270,  K = 528  0.628 / 1.600 / 3.346 / 6.572 / 13.098;
        //   cfg3 (44,541 particles, C >= 4; the single scene takes 16), C = 4 / 8 / 16:  K = 4 (C = 16 only) 7.82,  K = 8  14.38 / 10.12 /
        //        15.54 (16-CTA clusters: fewer than 8 at once),  K = 33  29.28 / 30.69 / 39.60,  K = 66  44.38 / 51.50 / 78.25.
        if (!oneCluster)
            return fmt("resident mode: a replica of %u particles (%u constraints per colour) does not fit one cluster of %d CTAs (use PBD_MODE_GRAPH)", in.n, perPhase, kMaxClusterCtas);
        unsigned fit = 1;
        while (in.n > fit * cap) fit *= 2;
        C = fit;
        if (fit > 1) {
            unsigned solo = fit;
            while (solo < (unsigned)kMaxClusterCtas && (perPhase > solo * 256u || in.n > solo * cap)) solo *= 2;
            for (unsigned c = solo; c > fit; c /= 2)
                if (in.maxClusters(r.mask, c, kMaxDynamicSmem) >= (int)in.replicas) { C = c; break; }
        }
        if (in.forcedC) C = in.forcedC;
    } else if (oneCluster) {
        // one cluster: enough CTAs that a colour phase is about one item per thread, and that the tiles fit
        while (C < (unsigned)kMaxClusterCtas && (perPhase > C * 256u || in.n > C * cap)) C *= 2;
    } else {
        // Too big for one cluster: one independent CTA per SM (clusters of 1).  Larger clusters have fewer X items but idle SMs (a
        // cluster must fit a GPC) and a colour barrier that waits for the slowest of C CTAs; with C = 1 the colour barrier is a
        // __syncthreads.
        const int mc = in.maxClusters(r.mask, 1u, kMaxDynamicSmem);
        if (mc < 1) return fmt("resident mode: a CTA with %zu bytes of shared memory is not schedulable on this device", kMaxDynamicSmem);
        C = 1; G = (unsigned)std::min(mc, in.smCount);
    }
    if (in.forcedG && in.replicas == 1) { G = in.forcedG; C = in.forcedC; }
    if ((unsigned long long)G * C * cap < in.n)
        return fmt("resident mode: %u particles do not fit %u x %u tiles of %u (use PBD_MODE_GRAPH)", in.n, G, C, cap);
    // (bodies without joints -- e.g. the static colliders of the contact path -- are integrated by CTA 0 and touch no constraint)
    if (G > 1 && (!in.store[PBD_BALLJOINT].ids.empty() || !in.store[PBD_RB_PARTICLE_BALLJOINT].ids.empty()))
        return "resident mode: rigid-body coupling is supported for scenes that fit one cluster (use PBD_MODE_GRAPH)";
    r.G = G; r.C = C;
    r.xThreads = (G > 1) ? 128u : 0u;  // refined in place_in_tiles once the share of X items is known
    return "";
}

static std::string place_in_tiles(Ctx &c) {
    const PlanInput &in = c.in;
    ImagePlan &pl = c.out;
    const std::string err = choose_resident_shape(in, pl.res);
    if (!err.empty()) return err;
    const unsigned n = in.n, G = pl.res.G, C = pl.res.C, T = c.nTiles();
    c.tileOf.assign(n, 0); c.homedGlobal.assign(n, 0); pl.tileStart.assign(T + 1, 0); pl.tileSmem.assign(T, 0);
    if (n) {
        const float4 *x = in.x0;  // rest positions by host index
        std::vector<unsigned> idx(n), region(n);
        for (unsigned i = 0; i < n; i++) idx[i] = i;
        #pragma omp parallel num_threads(host_threads())
        #pragma omp single
        bisect(idx, 0, n, 0, G, x, region);  // cluster regions; idx is now grouped region by region
        size_t lo = 0;
        for (unsigned g = 0; g < G; g++) {
            size_t hi = lo;
            while (hi < n && region[idx[hi]] == g) hi++;
            if (C == 1) { for (size_t i = lo; i < hi; i++) c.tileOf[idx[i]] = g; }
            else {
                #pragma omp parallel num_threads(host_threads())
                #pragma omp single
                bisect(idx, lo, hi, g * C, C, x, c.tileOf);
            }
            lo = hi;
        }
        // global-homed: independent CTAs, touched by a constraint owned by another tile; clusters of several CTAs, touched by a
        // constraint whose particles lie in more than one cluster
        if (G > 1 && C == 1) home_by_owner(c);
        else if (G > 1)
            for (int t = 0; t < PBD_NUM_TYPES; t++) {
                const TypeStore &h = in.store[t];
                const int nb = type_shape(t).nBodies;
                unsigned char *hg = c.homedGlobal.data();
                #pragma omp parallel for schedule(static) num_threads(host_threads())
                for (long long k0 = 0; k0 < (long long)h.ids.size(); k0++) {
                    const unsigned *b = &h.bodies[(size_t)k0 * nb];
                    bool spans = false;
                    for (int k = 1; k < nb; k++) spans |= (c.tileOf[b[k]] / C != c.tileOf[b[0]] / C);
                    if (spans) for (int k = 0; k < nb; k++) hg[b[k]] = 1;  // every writer stores the same byte
                }
            }
        // threads of a CTA dedicated to the X items: in proportion to their share, times 3.1 because an X item waits for L2 where
        // the others read shared memory.  The factor is carried over from an earlier GPU.  H100 80GB HBM3 (700 W), ms per step at 128 /
        // 160 / 192 / 224 X threads, two alternating runs each, with a first homing by owner of nearly the same X share (DESIGN.md
        // section 6): cfg2 1.694 / 1.675 / 1.699 / 1.739 (this rule: 128), cfg5 1.142-1.145 / 1.136-1.145 / 1.124-1.140 / 1.128-1.140
        // (this rule: 256).
        if (G > 1) {
            unsigned long long xItems = 0;
            for (int t = 0; t < PBD_NUM_TYPES; t++) {
                const TypeStore &h = in.store[t];
                const int nb = type_shape(t).nBodies;
                #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(+ : xItems)
                for (long long k0 = 0; k0 < (long long)h.ids.size(); k0++) {
                    bool x = false;
                    for (int k = 0; k < nb; k++) x |= (!is_rb_body(t, k) && c.homedGlobal[h.bodies[(size_t)k0 * nb + k]]);
                    xItems += x;
                }
            }
            const double share = (double)xItems / std::max(1u, in.numConstraints);
            unsigned xt = ((unsigned)(pl.res.threads * share * 3.1) + 31u) & ~31u;
            pl.res.xThreads = std::max(64u, std::min(xt, (pl.res.threads / 2u) & ~31u));
        }
        // tile-major slots: shared-memory particles first (host order), global-homed behind them
        std::vector<unsigned> cntS(T, 0), cntG(T, 0);
        for (unsigned i = 0; i < n; i++) (c.homedGlobal[i] ? cntG : cntS)[c.tileOf[i]]++;
        for (unsigned t = 0; t < T; t++) {
            pl.tileStart[t + 1] = pl.tileStart[t] + cntS[t] + cntG[t];
            pl.tileSmem[t] = cntS[t];
        }
        std::vector<unsigned> curS(T), curG(T);
        for (unsigned t = 0; t < T; t++) { curS[t] = pl.tileStart[t]; curG[t] = pl.tileStart[t] + cntS[t]; }
        pl.slot.resize(n);
        for (unsigned i = 0; i < n; i++) pl.slot[i] = c.homedGlobal[i] ? curG[c.tileOf[i]]++ : curS[c.tileOf[i]]++;
        if (verbose()) {
            unsigned long long nGl = 0;
            for (unsigned i = 0; i < n; i++) nGl += c.homedGlobal[i];
            fprintf(stderr, "[pbd_b200] resident: %u clusters x %u CTAs, %u threads (%u for X items), %u particles, %.2f %% global-homed, max tile %u\n", G, C, pl.res.threads, pl.res.xThreads, n,
                    100.0 * nGl / n, *std::max_element(cntS.begin(), cntS.end()));
        }
    }
    pl.res.tileCap = 64u;  // multiple of 64: the bank swizzle permutes inside aligned 64-slot blocks
    for (unsigned t = 0; t < T; t++) pl.res.tileCap = std::max(pl.res.tileCap, (pl.tileSmem[t] + 63u) & ~63u);
    return "";
}

typedef std::pair<unsigned long long, unsigned> KeyedItem;  // (sort key, local host index of the constraint)
struct Wavefronts { double before = 0, after = 0, requests = 0; };

// Shared-memory bank groups of one run of a resident tile.  The eight lanes of a quarter-warp (eight consecutive items of the run) read
// operand k of their items with one LDS.128; it takes as many wavefronts as the fullest 16-byte bank group (slot & 7 after the swizzle).
// Greedy re-ordering: each group of eight is filled with the items, out of the next `kWindow` unused ones, that add the fewest
// collisions over all operands.  The order inside a colour is free; results are bit-identical.  H100 80GB HBM3 (400 W), without / with
// the fill: cfg2 2.14 / 2.08 ms, cfg5 1.221 / 1.216 ms, cfg3 7.81 / 7.69 ms (bank group taken inside the CTA that holds the particle).
// With `wf`: the wavefronts of the run's quarter-warp gathers before and after, and their number.
static void bank_group_fill(KeyedItem *run, size_t cnt, int t, const Ctx &c, Wavefronts *wf) {
    constexpr int kWindow = 64;
    const int nb = type_shape(t).nBodies, nk = std::min(nb, 4);
    const unsigned *bod = c.in.store[t].bodies.data();
    std::vector<unsigned char> bg(cnt * 4, 0);
    for (size_t i = 0; i < cnt; i++) {
        const unsigned *b = bod + (size_t)run[i].second * nb;
        for (int k = 0; k < nk; k++) bg[i * 4 + k] = (unsigned char)(tile_swizzle(c.out.slot[b[k]] - c.out.tileStart[c.tileOf[b[k]]]) & 7u);  // bank group inside the CTA that holds the particle
    }
    // greedy fill from a sliding pool of the next kWindow unused items (kept in run order)
    std::vector<unsigned> out; out.reserve(cnt);
    unsigned pool[kWindow]; int nPool = 0; size_t head = 0;
    while (out.size() < cnt) {
        unsigned char load[4][8] = {};
        for (int j = 0; j < 8 && out.size() < cnt; j++) {
            while (nPool < kWindow && head < cnt) pool[nPool++] = (unsigned)head++;
            int best = 0, bestCost = 1 << 30;
            for (int p = 0; p < nPool; p++) {
                const unsigned char *g4 = &bg[(size_t)pool[p] * 4];
                int cost = 0;
                for (int k = 0; k < nk; k++) cost += load[k][g4[k]];
                if (cost < bestCost) { bestCost = cost; best = p; if (!cost) break; }
            }
            const unsigned pick = pool[best];
            for (int p = best; p + 1 < nPool; p++) pool[p] = pool[p + 1];
            nPool--;
            out.push_back(pick);
            for (int k = 0; k < nk; k++) load[k][bg[(size_t)pick * 4 + k]]++;
        }
    }
    if (wf) {
        auto wavefronts = [&](const std::vector<unsigned> &ord) {
            double w = 0;
            for (size_t g8 = 0; g8 + 8 <= cnt; g8 += 8)
                for (int k = 0; k < nk; k++) {
                    unsigned char c8[8] = {0, 0, 0, 0, 0, 0, 0, 0}; unsigned mx = 0;
                    for (int j = 0; j < 8; j++) mx = std::max<unsigned>(mx, ++c8[bg[ord[g8 + j] * 4 + k]]);
                    w += mx;
                }
            return w;
        };
        std::vector<unsigned> asSorted(cnt);
        std::iota(asSorted.begin(), asSorted.end(), 0u);
        wf->before += wavefronts(asSorted); wf->after += wavefronts(out); wf->requests += (double)(cnt / 8) * nk;
    }
    const std::vector<KeyedItem> sorted(run, run + cnt);
    for (size_t i = 0; i < cnt; i++) run[i] = sorted[out[i]];
}

// The items (local host indices) of the bucket (colour g, type t), re-ordered.  The order inside a colour is free: sorted by lowest
// particle slot for gather locality (joints keep their order); resident: major key = executing tile, then the X items (touching a
// global-homed particle) before the others, the shared-memory runs bank-group filled, and the runs of every tile appended to tileOff:
// [2 tile] X items, [2 tile + 1] the others.
static void sort_bucket(const Ctx &c, unsigned g, int t, std::vector<unsigned> &items, std::vector<unsigned> &tileOff) {
    const bool tiled = c.tiled;
    const bool joint = (t == PBD_BALLJOINT || t == PBD_RB_PARTICLE_BALLJOINT);
    const int nb = type_shape(t).nBodies;
    const unsigned *bod = c.in.store[t].bodies.data();
    std::vector<KeyedItem> keyed(items.size());
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (long long i = 0; i < (long long)items.size(); i++) {
        const unsigned *b = bod + (size_t)items[i] * nb;
        unsigned mn = 0xffffffffu;
        for (int k = 0; k < nb; k++) if (!is_rb_body(t, k)) mn = std::min(mn, c.out.slot[b[k]]);
        if (joint) mn = (unsigned)i;
        // resident: run = executing tile and kind (X items first) in key bits 51 and up.  Ordering a run by kind of element as well
        // (constraints with the same slot offsets between their particles first) made no difference on an H100 80GB HBM3 (700 W):
        // cfg3 7.66 / 7.62 ms, cfg4 0.625 / 0.625 ms with / without.
        unsigned long long run = 0;
        if (tiled) {
            bool x = false;
            const unsigned exec = exec_tile(c, t, items[i], &x);
            run = 2ull * exec + (x ? 0u : 1u);
        }
        keyed[i] = std::make_pair((run << 51) | mn, items[i]);
    }
    __gnu_parallel::stable_sort(keyed.begin(), keyed.end(), [](const KeyedItem &a, const KeyedItem &b) { return a.first < b.first; },
                                __gnu_parallel::default_parallel_tag(host_threads()));
    if (tiled && !joint) {
        std::vector<size_t> runStart;
        for (size_t i = 0; i < keyed.size(); i++) if (i == 0 || (keyed[i].first >> 51) != (keyed[i - 1].first >> 51)) runStart.push_back(i);
        runStart.push_back(keyed.size());
        double before = 0, after = 0, requests = 0;
        const long long nRuns = (long long)runStart.size() - 1;
        #pragma omp parallel for schedule(dynamic, 1) num_threads(host_threads()) reduction(+ : before, after, requests)
        for (long long r = 0; r < nRuns; r++) {
            const size_t lo = runStart[r], cnt = runStart[r + 1] - lo;
            if (!((keyed[lo].first >> 51) & 1ull) || cnt < 16) continue;  // X runs gather from global memory: left alone
            Wavefronts w;
            bank_group_fill(&keyed[lo], cnt, t, c, verbose() ? &w : nullptr);
            before += w.before; after += w.after; requests += w.requests;
        }
        if (verbose() && requests > 0) fprintf(stderr, "[pbd_b200] flatten:   colour %u type %d: %.2f wavefronts per quarter-warp gather as sorted, %.2f after the bank-group fill\n", g, t,
                                               before / requests, after / requests);
    }
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (long long i = 0; i < (long long)keyed.size(); i++) items[i] = keyed[i].second;
    if (tiled) {
        const size_t base = tileOff.size();
        tileOff.resize(base + 2 * c.nTiles() + 1, 0u);
        for (size_t i = 0; i < keyed.size(); i++) tileOff[base + (keyed[i].first >> 51) + 1]++;
        for (unsigned k = 0; k < 2 * c.nTiles(); k++) tileOff[base + k + 1] += tileOff[base + k];
    }
}

// every colour group split by type into (colour, type) buckets; order[t]: device position -> local host index
static void order_buckets(Ctx &c, const std::vector<std::pair<int, unsigned>> &map, std::vector<unsigned> (&order)[PBD_NUM_TYPES]) {
    const std::vector<unsigned> &groupOff = *c.in.groupOff, &groupIds = *c.in.groupIds;
    const unsigned nGroups = (unsigned)groupOff.size() - 1;
    c.out.buckets.clear();
    std::vector<unsigned> items[PBD_NUM_TYPES];
    for (unsigned g = 0; g < nGroups; g++) {
        for (auto &v : items) v.clear();
        for (unsigned i = groupOff[g]; i < groupOff[g + 1]; i++) {
            const auto &m = map[groupIds[i]];
            items[m.first].push_back(m.second);
        }
        for (int t = 0; t < PBD_NUM_TYPES; t++) {
            if (items[t].empty()) continue;
            const bool joint = (t == PBD_BALLJOINT || t == PBD_RB_PARTICLE_BALLJOINT);
            if (!joint || c.tiled) sort_bucket(c, g, t, items[t], c.out.tileOff);
            Bucket b; b.type = t; b.first = (unsigned)order[t].size(); b.count = (unsigned)items[t].size(); b.colour = g;
            c.out.buckets.push_back(b);
            order[t].insert(order[t].end(), items[t].begin(), items[t].end());
        }
    }
}

// Debug-grade safety: inside a colour no particle may be used twice (race freedom by construction, SURVEY.md section 5).  Particles
// and rigid bodies are stamped in separate index spaces (the reference's colouring shares one, which only ever over-separates; a body
// really used twice in a colour would be a race here).
static std::string check_colouring(const Ctx &c, const std::vector<unsigned> (&order)[PBD_NUM_TYPES]) {
    const unsigned n = c.in.n;
    std::vector<unsigned> stamp((size_t)n + c.in.nRb, 0xffffffffu);
    for (const Bucket &b : c.out.buckets) {  // colour after colour
        const unsigned g = b.colour;
        const int nb = type_shape(b.type).nBodies;
        long long bad = -1;  // items of a bucket in parallel: the stamp of a slot is exchanged atomically
        #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(max : bad) if (b.count > 20000)
        for (long long i = 0; i < (long long)b.count; i++) {
            const unsigned *bd = &c.in.store[b.type].bodies[(size_t)order[b.type][b.first + i] * nb];
            for (int k = 0; k < nb; k++) {
                const size_t slot = is_rb_body(b.type, k) ? (size_t)n + bd[k] : bd[k];
                if (__atomic_exchange_n(&stamp[slot], g, __ATOMIC_RELAXED) == g) bad = std::max(bad, (long long)slot);
            }
        }
        if (bad >= 0) {
            const bool isRb = (size_t)bad >= n;
            return fmt("colour group %u uses %s %u twice: the groups are not a valid colouring", g, isRb ? "rigid body" : "particle", (unsigned)(isRb ? bad - n : bad));
        }
    }
    return "";
}

// (pack_columns and factor_rank1: rest_geometry.cuh, shared with the device derivation of a batch's per-replica geometry)
// the SoA arrays of type t in device order (order: device position -> local host index)
static std::string pack_type(Ctx &c, int t, const std::vector<unsigned> &order, Lap &lap) {
    TypePlan &d = c.out.types[t];
    const TypeStore &h = c.in.store[t];
    const TypeShape s = type_shape(t);
    const unsigned cnt = (unsigned)order.size();
    const bool tiled = c.tiled;
    d.order.resize(cnt);
    if (cnt == 0) return "";
    #pragma omp parallel for schedule(static) num_threads(host_threads())
    for (long long i = 0; i < (long long)cnt; i++) d.order[i] = h.ids[order[i]];
    if (c.in.restTables && t < PBD_BALLJOINT) {  // what a batch's per-replica geometry is derived from (k_derive_geometry)
        d.restBodies.resize((size_t)cnt * s.nBodies); d.restLocal.resize(cnt);
        #pragma omp parallel for schedule(static) num_threads(host_threads())
        for (long long i = 0; i < (long long)cnt; i++) {
            d.restLocal[i] = order[i];
            for (int k = 0; k < s.nBodies; k++) d.restBodies[(size_t)i * s.nBodies + k] = h.bodies[(size_t)order[i] * s.nBodies + k];
        }
    }
    auto P = [&](unsigned i, int k) { return h.params[(size_t)order[i] * s.nParams + k]; };
    auto B = [&](unsigned i, int k) {
        const unsigned raw = h.bodies[(size_t)order[i] * s.nBodies + k];
        if (is_rb_body(t, k)) return raw;
        if (tiled && !c.homedGlobal[raw]) {  // lives in the shared memory of CTA (tile % C) of the executing cluster
            const unsigned tl = c.tileOf[raw];
            return kSmemFlag | ((tl % c.out.res.C) << kRankShift) | tile_swizzle(c.out.slot[raw] - c.out.tileStart[tl]);
        }
        return c.out.slot[raw];
    };

    if (verbose()) fprintf(stderr, "[pbd_b200] flatten:   type %d (%u constraints)\n", t, cnt);
    lap("  order ids");
    // indices
    if (s.nBodies == 2) {
        d.idx2.resize(cnt);
        #pragma omp parallel for schedule(static) num_threads(host_threads())
        for (long long i = 0; i < (long long)cnt; i++) d.idx2[i] = make_uint2(B(i, 0), B(i, 1));
    } else if (s.nBodies == 4) {
        d.idx4.resize(cnt);
        #pragma omp parallel for schedule(static) num_threads(host_threads())
        for (long long i = 0; i < (long long)cnt; i++) d.idx4[i] = make_uint4(B(i, 0), B(i, 1), B(i, 2), B(i, 3));
    } else {
        for (int k = 0; k < 3; k++) {
            d.idx3[k].resize(cnt);
            #pragma omp parallel for schedule(static) num_threads(host_threads())
            for (long long i = 0; i < (long long)cnt; i++) d.idx3[k][i] = B(i, k);
        }
    }

    lap("  indices");
    // geometry: the parameter columns of the table, with two exceptions
    const PackColumns pc = pack_columns(t);
    bool fromColumns = true;
    if (t == PBD_ISOBENDING || t == PBD_ISOBENDING_XPBD) {
        // the rank-one form Q = -Kp Kp^T of init_IsometricBendingConstraint: gv[0] = Kp; a user-modified Q anywhere in this type:
        // the literal 4x4 evaluation (variant 1) for the whole type, Q row by row from the columns of the table
        d.gv[0].resize(cnt);
        int notRank1 = 0;
        #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(| : notRank1)
        for (long long i = 0; i < (long long)cnt; i++) {
            float Q[16], Kp[4] = {0.f, 0.f, 0.f, 0.f};
            for (int k = 0; k < 16; k++) Q[k] = P((unsigned)i, 1 + k);
            if (!factor_rank1(Q, Kp)) notRank1 |= 1;
            d.gv[0][i] = make_float4(Kp[0], Kp[1], Kp[2], Kp[3]);
        }
        if (notRank1 && tiled) return "resident mode: IsometricBending with a user-modified Q matrix (not of the rank-one form) is evaluated by the per-bucket kernels only (use PBD_MODE_GRAPH)";
        d.variant = notRank1 ? 1 : 0;
        fromColumns = notRank1 != 0;
    }
    if (t == PBD_SHAPEMATCHING)
        for (unsigned i = 0; i < cnt; i++)
            for (int k = 20; k < 24; k++) if (!(P(i, k) >= 1.0f)) return "ShapeMatching constraint: numClusters must be >= 1";
    auto col = [&](unsigned i, int k) { return k < 0 ? 0.0f : P(i, k); };
    for (int k = 0; k < kMaxGeoV && fromColumns; k++) {
        const signed char *cc = pc.gv[k];
        if (cc[0] < 0 && cc[1] < 0 && cc[2] < 0 && cc[3] < 0) continue;
        d.gv[k].resize(cnt);
        #pragma omp parallel for schedule(static) num_threads(host_threads())
        for (long long i = 0; i < (long long)cnt; i++) d.gv[k][i] = make_float4(col(i, cc[0]), col(i, cc[1]), col(i, cc[2]), col(i, cc[3]));
    }
    for (int k = 0; k < kMaxGeoS; k++) {
        if (pc.gs[k] < 0) continue;
        d.gs[k].resize(cnt);
        #pragma omp parallel for schedule(static) num_threads(host_threads())
        for (long long i = 0; i < (long long)cnt; i++) d.gs[k][i] = P(i, pc.gs[k]);
    }
    lap("  geometry");
    // material parameters: one uniform per type when every constraint agrees, else a per-constraint array
    for (int k = 0; k < kMaxMat; k++) {
        const int cm = pc.mat[k];
        if (cm < 0) continue;
        const float first = P(0, cm);
        int differs = 0;
        #pragma omp parallel for schedule(static) num_threads(host_threads()) reduction(| : differs) if (cnt > 100000)
        for (long long i = 1; i < (long long)cnt; i++) differs |= (P((unsigned)i, cm) != first) ? 1 : 0;
        d.matU[k] = first;
        if (differs) {
            d.mat[k].resize(cnt);
            #pragma omp parallel for schedule(static) num_threads(host_threads())
            for (long long i = 0; i < (long long)cnt; i++) d.mat[k][i] = P(i, cm);
        }
    }
    lap("  material");
    return "";
}

// resident mode: colour ranges of the bucket table, the per-tile runs, and who waits for whom in the X flag protocol.  Tile j is a
// neighbour of tile i when an X item of i and an X item of j touch the same global-homed particle, or an X item of one of them touches
// a particle homed in the other: exactly the tiles whose global-memory accesses i's X items and i's global-homed particles have to be
// ordered with.  xMask[i][0] bit k: neighbour k has global-homed particles (arrives in the integration phase); xMask[i][1 + c] bit k:
// neighbour k has X items in colour c.
static std::string build_phase_tables(Ctx &c, const std::vector<unsigned> (&order)[PBD_NUM_TYPES]) {
    ImagePlan &pl = c.out;
    const std::vector<Bucket> &buckets = pl.buckets;
    const std::vector<unsigned> &tileOff = pl.tileOff;
    const unsigned T = c.nTiles();
    std::vector<unsigned> &colourStart = pl.colourStart;
    colourStart.clear();
    for (size_t i = 0; i < buckets.size(); i++)
        if (i == 0 || buckets[i].colour != buckets[i - 1].colour) colourStart.push_back((unsigned)i);
    pl.res.nColours = (unsigned)colourStart.size();
    colourStart.push_back((unsigned)buckets.size());
    if (tileOff.size() != buckets.size() * (2 * (size_t)T + 1)) return "flatten: internal error (tile runs)";
    const unsigned nC = pl.res.nColours;
    auto run = [&](size_t bi, unsigned t) { return &tileOff[bi * (2 * (size_t)T + 1) + 2 * t]; };  // [0] X items .. [1] others .. [2]
    // (global-homed particle, tile) pairs: its home tile and every tile that executes an X item touching it
    std::vector<std::pair<unsigned, unsigned>> touch;
    for (unsigned i = 0; i < c.in.n; i++) if (c.homedGlobal[i]) touch.emplace_back(i, c.tileOf[i]);
    for (size_t bi = 0; bi < buckets.size(); bi++) {
        const Bucket &b = buckets[bi];
        const int nb = type_shape(b.type).nBodies;
        for (unsigned t = 0; t < T; t++)
            for (unsigned k = run(bi, t)[0]; k < run(bi, t)[1]; k++) {
                const unsigned *bod = &c.in.store[b.type].bodies[(size_t)order[b.type][b.first + k] * nb];
                for (int j = 0; j < nb; j++) if (!is_rb_body(b.type, j) && c.homedGlobal[bod[j]]) touch.emplace_back(bod[j], t);
            }
    }
    std::sort(touch.begin(), touch.end());
    touch.erase(std::unique(touch.begin(), touch.end()), touch.end());
    std::vector<unsigned char> adj((size_t)T * T, 0);
    for (size_t lo = 0, hi; lo < touch.size(); lo = hi) {
        for (hi = lo + 1; hi < touch.size() && touch[hi].first == touch[lo].first; hi++) {}
        for (size_t a = lo; a < hi; a++)
            for (size_t cc = lo; cc < hi; cc++)
                if (touch[a].second != touch[cc].second) adj[(size_t)touch[a].second * T + touch[cc].second] = 1;
    }
    std::vector<unsigned char> hasX((size_t)T * (1 + nC), 0);  // [tile][phase]: the tile arrives in the phase
    for (unsigned t = 0; t < T; t++) {
        hasX[(size_t)t * (1 + nC)] = (pl.tileStart[t + 1] - pl.tileStart[t] - pl.tileSmem[t]) != 0;
        for (unsigned cl = 0; cl < nC; cl++)
            for (unsigned bi = colourStart[cl]; bi < colourStart[cl + 1]; bi++) hasX[(size_t)t * (1 + nC) + 1 + cl] |= run(bi, t)[1] != run(bi, t)[0];
    }
    std::vector<unsigned> &nbr = pl.xNbr, &mask = pl.xMask, nNbr(T, 0u);
    nbr.assign((size_t)T * kMaxXNeighbours, 0u); mask.assign((size_t)T * (1 + nC), 0u);
    for (unsigned i = 0; i < T; i++) {
        for (unsigned k = 0; k < kMaxXNeighbours; k++) nbr[(size_t)i * kMaxXNeighbours + k] = i;  // unused lanes: never polled (mask bit 0)
        for (unsigned j = 0; j < T; j++) {
            if (!adj[(size_t)i * T + j]) continue;
            if (nNbr[i] == kMaxXNeighbours)
                return fmt("resident mode: tile %u shares global-homed particles with more than %u other tiles (the constraints reach too far "
                           "across the scene for the resident mode; use PBD_MODE_GRAPH)", i, kMaxXNeighbours);
            const unsigned k = nNbr[i]++;
            nbr[(size_t)i * kMaxXNeighbours + k] = j;
            for (unsigned p = 0; p <= nC; p++) mask[(size_t)i * (1 + nC) + p] |= (unsigned)hasX[(size_t)j * (1 + nC) + p] << k;
        }
    }
    if (verbose()) {
        const unsigned numConstraints = c.in.numConstraints;
        unsigned long long xItems = 0, mxRun = 0;
        std::vector<unsigned long long> perTile(T, 0);  // items a tile executes over one sweep
        unsigned long long lockstep = 0;                // ... and the sum over the colours of the largest tile's items of the colour
        unsigned long long rLargest = 0, xLargest = 0;  // sum over the colours of the largest tile's R / X items of the colour
        for (unsigned cl = 0; cl < nC; cl++) {
            unsigned long long mx = 0, mxR = 0, mxX = 0;
            for (unsigned t = 0; t < T; t++) {
                unsigned long long items = 0, rItems = 0;
                for (unsigned bi = colourStart[cl]; bi < colourStart[cl + 1]; bi++) {
                    xItems += run(bi, t)[1] - run(bi, t)[0];
                    items += run(bi, t)[2] - run(bi, t)[0];
                    rItems += run(bi, t)[2] - run(bi, t)[1];
                    mxRun = std::max<unsigned long long>(mxRun, run(bi, t)[2] - run(bi, t)[0]);
                }
                perTile[t] += items; mx = std::max(mx, items); mxR = std::max(mxR, rItems); mxX = std::max(mxX, items - rItems);
            }
            lockstep += mx; rLargest += mxR; xLargest += mxX;
        }
        std::vector<unsigned> hist(kMaxXNeighbours + 1, 0u);
        for (unsigned t = 0; t < T; t++) hist[nNbr[t]]++;
        fprintf(stderr, "[pbd_b200] resident: %u colours, %zu buckets, %.2f %% X items, largest run of a tile in a bucket %llu (mean %.0f)\n",
                nC, buckets.size(), 100.0 * xItems / std::max(1u, numConstraints), mxRun, (double)numConstraints / std::max<size_t>(1, buckets.size()) / T);
        fprintf(stderr, "[pbd_b200] resident: X neighbours per tile (count x tiles):");
        for (unsigned k = 0; k <= kMaxXNeighbours; k++) if (hist[k]) fprintf(stderr, " %u x %u", k, hist[k]);
        const unsigned long long mxTile = T ? *std::max_element(perTile.begin(), perTile.end()) : 0;
        fprintf(stderr, "\n[pbd_b200] resident: items per sweep, sum over colours of the largest tile %llu, largest tile over all colours %llu (lockstep penalty %.2f %%)\n",
                lockstep, mxTile, mxTile ? 100.0 * ((double)lockstep / mxTile - 1.0) : 0.0);
        // what a colour phase waits for: the CTA with the most shared-memory (R) items, and the one with the most X items, of the colour
        fprintf(stderr, "[pbd_b200] resident: largest tile's items per colour (mean over colours): R %.1f (%.1f per R thread), X %.1f (%.2f per X thread)\n",
                (double)rLargest / std::max(1u, nC), (double)rLargest / std::max(1u, nC) / std::max(1u, pl.res.threads - pl.res.xThreads),
                (double)xLargest / std::max(1u, nC), (double)xLargest / std::max(1u, nC) / std::max(1u, pl.res.xThreads));
        // the constraint stream of one sweep as this image streams it from DRAM: the 32-bit indices, the per-constraint geometry and
        // material arrays, the multipliers (read and written)
        double idxBytes = 0, constBytes = 0;
        for (const Bucket &b : buckets) {
            const TypePlan &a = pl.types[b.type];
            double perItem = type_shape(b.type).xpbd ? 8.0 : 0.0;
            for (int k = 0; k < kMaxGeoV; k++) perItem += !a.gv[k].empty() ? 16.0 : 0.0;
            for (int k = 0; k < kMaxGeoS; k++) perItem += !a.gs[k].empty() ? 4.0 : 0.0;
            for (int k = 0; k < kMaxMat; k++) perItem += !a.mat[k].empty() ? 4.0 : 0.0;
            idxBytes += b.count * 4.0 * type_shape(b.type).nBodies; constBytes += b.count * perItem;
        }
        fprintf(stderr, "[pbd_b200] resident: constraint stream per sweep %.1f MB: indices %.1f MB, constants and multipliers %.1f MB\n",
                (idxBytes + constBytes) * 1e-6, idxBytes * 1e-6, constBytes * 1e-6);
    }
    return "";
}

// PBD_MODE_AUTO: the resident mode where it is the faster exact mode -- models made of cloth and FEM / volume constraints with at
// least kAutoResidentMinParticles particles (cfg2, cfg3, cfg5); small models (cfg1), mixed models with rigid coupling and the heavy
// solver families (cfg4) stay in graph mode, and so does a model the resident mode refuses (plan_image).
// Measured on an H100 80GB HBM3 (SXM, 400 W, 1980 MHz), XPBD cloth 1 x 20, ms per step graph / resident: 100x100 0.66 / 0.79,
// 200x200 0.93 / 0.92, 300x300 1.20 / 1.02; cfg1 (50x50) 0.129 / 0.183; cfg3 (44,541 particles) 8.03 / 7.69.
// Replica batches take the resident mode from kAutoResidentMinReplicas replicas on whatever the size of a replica, from twice as many
// for models only the light instantiation covers (FEMTriangle, Dihedral, Volume: per replica a longer step than the cloth and FEM
// kernels take).  H100 80GB HBM3 (SXM, 700 W), ms per batched step graph / resident (tools/bench_batch.py): cfg1 K = 8 0.146 / 0.147,
// K = 33 0.263 / 0.147, K = 528 1.447 / 0.628; 100x100 XPBD cloth 1 x 20 K = 8 1.09 / 1.44, K = 33 2.78 / 1.45, K = 264 15.82 / 3.21;
// cfg3 K = 4 13.42 / 7.88, K = 66 127.9 / 44.1; 100x100 FEMTriangle + Dihedral cloth 1 x 5 (light) K = 33 0.531 / 0.692, K = 66
// 0.838 / 0.717, K = 132 1.412 / 0.745.
constexpr unsigned kAutoResidentMinParticles = 40000, kAutoResidentMinReplicas = 32;
int preferred_mode(int requested, const TypeStore *store, unsigned n, unsigned numConstraints, unsigned replicas) {
    if (requested != PBD_MODE_AUTO) return requested;
    if (numConstraints == 0) return PBD_MODE_GRAPH;
    unsigned present = 0;
    for (int t = 0; t < PBD_NUM_TYPES; t++) if (!store[t].ids.empty()) present |= 1u << t;
    const bool clothFem = (present & ~(kMaskCloth | kMaskFem)) == 0, light = (present & ~kMaskLight) == 0;
    if (!clothFem && !light) return PBD_MODE_GRAPH;
    if (n >= kAutoResidentMinParticles) return PBD_MODE_RESIDENT;
    return replicas >= (clothFem ? 1u : 2u) * kAutoResidentMinReplicas ? PBD_MODE_RESIDENT : PBD_MODE_GRAPH;
}

// The resident batch kernels address replica r's per-replica rest geometry and per-constraint materials of type t as the element
// offset r x count + i in 32 bits (resident.cuh: run_items / prefetch_first, load_streamed's geoOff, project_streamed_acc's matOff; kept
// narrow for the registers, DESIGN.md section 3), where the per-bucket kernels move a pointer by a size_t offset.  A batch whose tables
// carry either override (PlanInput::restTables) therefore needs K x count < 2^32 for every particle type, else the resident mode would
// read another replica's rows.  The calls that switch the overrides on refuse such a batch, but constraints added afterwards grow the
// counts of a batch that is planned again; this keeps that batch out of the resident mode (AUTO: graph).
static std::string replica_offset_refusal(const PlanInput &in) {
    if (in.replicas < 2 || !in.restTables) return "";
    for (int t = 0; t < PBD_BALLJOINT; t++)
        if ((unsigned long long)in.replicas * in.store[t].ids.size() >= (1ull << 32))
            return fmt("resident mode: %u replicas of %zu constraints of type %d with per-replica rest shapes or materials exceed the "
                       "2^32 rows the resident kernel addresses (use PBD_MODE_GRAPH)", in.replicas, in.store[t].ids.size(), t);
    return "";
}

// the image of the resident mode (tiled) or of the others
static std::string plan_mode(const PlanInput &in, bool tiled, ImagePlan &out) {
    Lap lap;
    std::vector<std::pair<int, unsigned>> map;
    std::string err = validate_bodies(in);
    if (err.empty()) err = build_id_map(in.store, in.numConstraints, map);
    if (!err.empty()) return err;
    Ctx c{in, out, tiled, {}, {}};
    if (tiled) {
        if (!(err = replica_offset_refusal(in)).empty()) return err;
        if (!(err = place_in_tiles(c)).empty()) return err;
    } else {
        out.slot.resize(in.n);
        for (unsigned i = 0; i < in.n; i++) out.slot[i] = particle_slot(i, in.n);
    }
    lap("validation + placement");
    std::vector<unsigned> order[PBD_NUM_TYPES];
    order_buckets(c, map, order);
    lap("bucket ordering");
    if (!(err = check_colouring(c, order)).empty()) return err;
    lap("colouring validity check");
    for (int t = 0; t < PBD_NUM_TYPES; t++)
        if (!(err = pack_type(c, t, order[t], lap)).empty()) return err;
    lap("SoA arrays");
    if (tiled && !(err = build_phase_tables(c, order)).empty()) return err;
    lap("phase tables");
    if (!tiled) return "";
    // admitted when every CTA gets its shared memory and all G x C are co-resident (the X items of different clusters wait for each other)
    ResidentShape &r = out.res;
    r.smem = resident_smem_bytes(r.tileCap, (unsigned)out.buckets.size(), r.nColours);
    if (r.smem > kMaxDynamicSmem)
        return fmt("resident mode: a CTA needs %zu bytes of shared memory (tile of %u particles + phase tables), %zu available", r.smem, r.tileCap, kMaxDynamicSmem);
    const int mc = in.maxClusters(r.mask, r.C, r.smem);
    if (in.replicas > 1) {  // a batch: as many clusters as the device runs at once, up to one per replica; none waits for another
        if (mc < 1) return fmt("resident mode: the device cannot run a cluster of %u CTAs with %zu bytes of shared memory each", r.C, r.smem);
        r.G = std::min(in.replicas, (unsigned)mc);
        r.replicas = in.replicas;
        return "";
    }
    return (unsigned)mc < r.G ? fmt("resident mode: the device runs %d clusters of %u CTAs at a time, the scene needs %u co-resident", mc, r.C, r.G) : "";
}

std::string batch_refusal(unsigned replicas, unsigned n, int mode, unsigned nRb, const TypeStore *store, bool replicaBodies) {
    if (replicas == 0) return "replica batch: at least one replica";
    if ((unsigned long long)replicas * n >= (1ull << 31))
        return fmt("replica batch: %u replicas of %u particles exceed 2^31 particles", replicas, n);
    if (replicas == 1) return "";
    if (replicas > 65535u) return fmt("replica batch: %u replicas, at most 65535 (the projection kernels run one replica per grid row)", replicas);
    if (!replicaBodies && (nRb || !store[PBD_BALLJOINT].ids.empty() || !store[PBD_RB_PARTICLE_BALLJOINT].ids.empty()))
        return "replica batch: rigid bodies and joints are stepped one scene per engine (pbd_set_replicas 1); a batch takes per-replica bodies from pbd_set_replica_rigid_bodies";
    if (mode == PBD_MODE_JACOBI) return "replica batch: PBD_MODE_JACOBI steps one scene per engine (pbd_set_replicas 1)";
    return "";
}

std::string plan_image(const PlanInput &in, ImagePlan &out) {
    const std::string refusal = batch_refusal(in.replicas, in.n, in.mode, in.nRb, in.store, in.replicaBodies);
    if (!refusal.empty()) return refusal;
    out.mode = preferred_mode(in.mode, in.store, in.n, in.numConstraints, in.replicas);
    const std::string err = plan_mode(in, out.mode == PBD_MODE_RESIDENT, out);
    if (err.empty() || in.mode != PBD_MODE_AUTO || out.mode != PBD_MODE_RESIDENT) return err;
    // AUTO, and the resident mode refused the model (does not fit, user-modified bending Q, ...): the graph image, planned from scratch
    out = ImagePlan{};
    out.residentRefusal = err;
    return plan_mode(in, false, out);
}

ImageLayout image_layout(const ImagePlan &p, unsigned replicas) {
    ImageLayout l;
    static const ImagePointers at{};  // the slots: where each pointer sits in an ImagePointers
    auto add = [&](const std::string &name, const void *field, const void *src, size_t bytes, bool zeroed = false) {
        l.arrays.push_back({name, src, bytes, zeroed, (size_t)((const char *)field - (const char *)&at), 0});
    };
    auto vec = [&](const std::string &name, const void *field, const auto &v) { add(name, field, v.data(), v.size() * sizeof(v[0])); };
    for (int t = 0; t < PBD_NUM_TYPES; t++) {
        const TypePlan &d = p.types[t];
        const TypeArrays &a = at.types[t];
        const std::string s = std::to_string(t);
        vec("idx2_" + s, &a.idx2, d.idx2); vec("idx4_" + s, &a.idx4, d.idx4);
        for (int k = 0; k < 3; k++) vec("idx3_" + s + "_" + std::to_string(k), &a.idx3[k], d.idx3[k]);
        for (int k = 0; k < kMaxGeoV; k++) vec("gv" + s + "_" + std::to_string(k), &a.gv[k], d.gv[k]);
        for (int k = 0; k < kMaxGeoS; k++) vec("gs" + s + "_" + std::to_string(k), &a.gs[k], d.gs[k]);
        for (int k = 0; k < kMaxMat; k++) vec("mat" + s + "_" + std::to_string(k), &a.mat[k], d.mat[k]);
        vec("restBodies" + s, &at.rest[t].bodies, d.restBodies); vec("restLocal" + s, &at.rest[t].local, d.restLocal);
        add("restIds" + s, &at.rest[t].ids, d.order.data(), d.restBodies.empty() ? 0 : d.order.size() * sizeof(unsigned));
    }
    const ImageTables &r = at.tables;
    vec("buckets", &r.buckets, p.buckets); vec("colourStart", &r.colourStart, p.colourStart); vec("tileOff", &r.tileOff, p.tileOff);
    vec("tileStart", &r.tileStart, p.tileStart); vec("tileSmem", &r.tileSmem, p.tileSmem); vec("xNbr", &r.xNbr, p.xNbr); vec("xMask", &r.xMask, p.xMask);
    // the zeroed regions last, so that one memset clears them: replica r's multipliers of type t at [r count, (r + 1) count)
    for (int t = 0; t < PBD_NUM_TYPES; t++)
        if (type_shape(t).xpbd) add("lambda" + std::to_string(t), &at.types[t].lambda, nullptr, (size_t)replicas * p.types[t].order.size() * sizeof(float), true);
    if (p.mode == PBD_MODE_RESIDENT) add("xFlags", &r.xFlags, nullptr, (size_t)p.res.G * p.res.C * kXFlagStride * sizeof(unsigned long long), true);
    // Every array on a 256-byte boundary (what cudaMalloc guarantees a separate allocation), one of 1 MiB or more on a 2 MiB boundary, each
    // followed by padded_bytes of its own.  H100 80GB HBM3 (700 W), ms per step with one cudaMalloc per array / 256-byte boundaries only /
    // this, six alternating runs each: cfg2 1.815 / 1.820 / 1.818, cfg5 1.195 / 1.192 / 1.180.
    for (ImageArray &a : l.arrays) {
        if (!a.bytes) continue;
        const size_t align = a.bytes >= (1u << 20) ? (2u << 20) : 256;
        a.offset = (l.bytes + align - 1) & ~(align - 1);
        l.bytes = a.offset + padded_bytes(a.bytes);
    }
    return l;
}

}  // namespace pbd_b200
