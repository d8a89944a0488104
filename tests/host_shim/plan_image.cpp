// TEST INFRASTRUCTURE: runs the image planner of libpbd_b200.so (csrc/host/image_plan.h) on a model read from a file and writes every
// array of the plan to another, for tests/test_image_plan.py and, as plan_batch, tests/test_batch_plan.py.  Needs no GPU: the
// co-residency query answers a constant from the input.
//   plan_image <input> <output>
// input : u32 replicas, n, nRb, numConstraints, mode, restTables, forcedG, forcedC, smCount, maxClusters, nGroups; u32 groupOff[nGroups + 1];
//         u32 groupIds[numConstraints]; float4 x0[n]; per type: u32 count, u32 ids[count], u32 bodies[count nBodies], f32 params[count nParams]
// output: records of (char name[32], u64 bytes, bytes of data); "error" and "residentRefusal" first, the plan's mode and arrays after
//         them when the error is empty, and "layout": u64 size of the device allocation, then per array char name[32], u64 offset, u64
//         bytes (image_layout).  "res" describes the tiling of ONE replica of a batch (G = 1), "batch" = (replicas, clusters launched).
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
static void put(const std::string &name, const void *data, uint64_t bytes) {
    char tag[32] = {};
    snprintf(tag, sizeof(tag), "%s", name.c_str());
    fwrite(tag, 1, sizeof(tag), fout); fwrite(&bytes, sizeof(bytes), 1, fout); fwrite(data, 1, bytes, fout);
}
template <class V> static void put(const std::string &name, const V &v) { put(name, v.data(), v.size() * sizeof(v[0])); }

int main(int argc, char **argv) {
    if (argc != 3 || !(fin = fopen(argv[1], "rb")) || !(fout = fopen(argv[2], "wb"))) { fprintf(stderr, "usage: plan_image <input> <output>\n"); return 2; }
    const unsigned replicas = get1(), n = get1(), nRb = get1(), N = get1(), mode = get1(), restTables = get1(), G = get1(), C = get1(), smCount = get1(), maxClusters = get1(),
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
                       restTables != 0, replicas};
    ImagePlan p;
    const std::string err = plan_image(in, p);
    put("error", err);
    put("residentRefusal", p.residentRefusal);
    if (err.empty()) {
        put("mode", std::vector<int>{p.mode});
        put("slot", p.slot);
        for (int t = 0; t < PBD_NUM_TYPES; t++) {
            const TypePlan &d = p.types[t];
            put("order" + std::to_string(t), d.order);
            put("matU" + std::to_string(t), std::vector<float>(d.matU, d.matU + pbdk::kMaxMat));
            put("variant" + std::to_string(t), std::vector<int>{d.variant});
        }
        const ImageLayout l = image_layout(p, replicas);
        std::vector<uint64_t> layout{l.bytes};
        for (const ImageArray &a : l.arrays) {
            if (!a.zeroed) put(a.name, a.src, a.bytes);
            uint64_t row[6] = {0, 0, 0, 0, a.offset, a.bytes};
            snprintf((char *)row, 32, "%s", a.name.c_str());
            layout.insert(layout.end(), row, row + 6);
        }
        put("layout", layout);
        const ResidentShape &r = p.res;
        put("res", std::vector<unsigned>{r.replicas > 1 ? 1u : r.G, r.C, r.threads, r.xThreads, r.mask, r.tileCap, r.nColours});
        put("batch", std::vector<unsigned>{r.replicas, r.G});
        put("smem", std::vector<uint64_t>{r.smem});
    }
    fclose(fout);
    return 0;
}
