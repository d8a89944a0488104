// TEST INFRASTRUCTURE: runs the image planner of libpbd_b200.so (csrc/host/image_plan.h) on a model read from a file and writes every
// array of the plan to another, for tests/test_image_plan.py.  Needs no GPU: the co-residency query answers a constant from the input.
//   plan_image <input> <output>
// input : u32 n, nRb, numConstraints, mode, restTables, forcedG, forcedC, smCount, maxClusters, nGroups; u32 groupOff[nGroups + 1];
//         u32 groupIds[numConstraints]; float4 x0[n]; per type: u32 count, u32 ids[count], u32 bodies[count nBodies], f32 params[count nParams]
// output: records of (char name[32], u64 bytes, bytes of data); "error" and "residentRefusal" first, the plan's mode and arrays after
//         them when the error is empty
#include "host/image_plan.h"
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
using namespace pbd_b200;

static FILE *fin, *fout;
template <class T> static void get(T *p, size_t n) {
    if (n && fread(p, sizeof(T), n, fin) != n) { fprintf(stderr, "plan_image: short input\n"); exit(2); }
}
static unsigned get1() { unsigned v; get(&v, 1); return v; }
template <class V> static void put(const char *name, const V &v) {
    char tag[32] = {};
    snprintf(tag, sizeof(tag), "%s", name);
    const uint64_t bytes = v.size() * sizeof(v[0]);
    fwrite(tag, 1, sizeof(tag), fout); fwrite(&bytes, sizeof(bytes), 1, fout); fwrite(v.data(), 1, bytes, fout);
}
template <class V> static void put(const char *name, int t, const V &v) { char s[32]; snprintf(s, sizeof(s), "%s%d", name, t); put(s, v); }
template <class V> static void put(const char *name, int t, int k, const V &v) { char s[32]; snprintf(s, sizeof(s), "%s%d_%d", name, t, k); put(s, v); }

int main(int argc, char **argv) {
    if (argc != 3 || !(fin = fopen(argv[1], "rb")) || !(fout = fopen(argv[2], "wb"))) { fprintf(stderr, "usage: plan_image <input> <output>\n"); return 2; }
    const unsigned n = get1(), nRb = get1(), N = get1(), mode = get1(), restTables = get1(), G = get1(), C = get1(), smCount = get1(), maxClusters = get1(),
                   nGroups = get1();
    std::vector<unsigned> groupOff(nGroups + 1), groupIds(N);
    get(groupOff.data(), groupOff.size()); get(groupIds.data(), N);
    std::vector<float4> x0(n);
    get(x0.data(), n);
    TypeStore store[PBD_NUM_TYPES];
    for (int t = 0; t < PBD_NUM_TYPES; t++) {
        const unsigned cnt = get1();
        const pbdk::TypeShape s = pbdk::type_shape(t);
        TypeStore &h = store[t];
        h.ids.resize(cnt); h.bodies.resize((size_t)cnt * s.nBodies); h.params.resize((size_t)cnt * s.nParams);
        get(h.ids.data(), h.ids.size()); get(h.bodies.data(), h.bodies.size()); get(h.params.data(), h.params.size());
    }
    const PlanInput in{store, N, n, nRb, &groupOff, &groupIds, (int)mode, x0.data(), G, C, (int)smCount, [=](unsigned) { return (int)maxClusters; },
                       restTables != 0};
    ImagePlan p;
    const std::string err = plan_image(in, p);
    put("error", err);
    put("residentRefusal", p.residentRefusal);
    if (err.empty()) {
        put("mode", std::vector<int>{p.mode});
        put("slot", p.slot);
        put("buckets", p.buckets);
        for (int t = 0; t < PBD_NUM_TYPES; t++) {
            const TypePlan &d = p.types[t];
            put("order", t, d.order); put("idx2_", t, d.idx2); put("idx4_", t, d.idx4);
            for (int k = 0; k < 3; k++) put("idx3_", t, k, d.idx3[k]);
            for (int k = 0; k < pbdk::kMaxGeoV; k++) put("gv", t, k, d.gv[k]);
            for (int k = 0; k < pbdk::kMaxGeoS; k++) put("gs", t, k, d.gs[k]);
            for (int k = 0; k < pbdk::kMaxMat; k++) put("mat", t, k, d.mat[k]);
            put("matU", t, std::vector<float>(d.matU, d.matU + pbdk::kMaxMat));
            put("variant", t, std::vector<int>{d.variant});
        }
        const ResidentShape &r = p.res;
        put("res", std::vector<unsigned>{r.G, r.C, r.threads, r.xThreads, r.mask, r.tileCap, r.nColours});
        put("smem", std::vector<uint64_t>{r.smem});
        put("colourStart", p.colourStart); put("tileOff", p.tileOff); put("tileStart", p.tileStart); put("tileSmem", p.tileSmem);
        put("xNbr", p.xNbr); put("xMask", p.xMask);
    }
    fclose(fout);
    return 0;
}
