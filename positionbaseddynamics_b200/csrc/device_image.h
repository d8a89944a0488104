// positionbaseddynamics_b200/csrc/device_image.h
//
// The flattened device image of a simulation model that the sm_90a kernels consume (DESIGN.md "Data layout").
//  * particles : float4 SoA  pos = (x,y,z,invMass), vel = (vx,vy,vz,mass), oldPos, lastPos, pos0
//                (ParticleData::m_x/m_invMasses/m_v/m_masses/m_oldX/m_lastX/m_x0, Simulation/ParticleData.h:91-100)
//  * constraints: per type, SoA, ordered bucket after bucket in the reference's colour order
//                (SimulationModel::m_constraintGroups, Simulation/SimulationModel.h:99), each (colour,type) bucket
//                a contiguous range [first, first+count)
#pragma once
#include <cuda_runtime.h>
#include "../../include/pbd_b200.h"

namespace pbdk {

constexpr int kMaxMat = 5;   // material parameters per type (stiffness, Young's moduli, Poisson ratios, flags)
constexpr int kMaxGeoV = 6;  // float4 geometry arrays per type
constexpr int kMaxGeoS = 2;  // scalar geometry arrays per type

// Particle placement in the device arrays: the de-interleaved layout puts the even-numbered particles first and the
// odd-numbered ones behind them.  Reason: the graph-mode step is bound by L2 *sector* throughput, and
// constraints of one colour never share a particle, so consecutive constraints of a bucket touch particles 2 apart --
// with the identity layout a warp's gather then uses only one 16-byte half of every 32-byte sector.  After de-interleaving
// a stride-2 pattern becomes contiguous (full sectors) and a stride-1 pattern becomes two contiguous streams (also full
// sectors).  Simulated sectors per gather on cfg2: 0.94 -> 0.72 (ideal 0.5).
#if defined(__CUDACC__)
__host__ __device__
#endif
inline unsigned particle_slot(unsigned i, unsigned n) {
    return (i >> 1) + (i & 1u) * ((n + 1u) >> 1);
}

struct TypeArrays {
    const uint2 *idx2;         // 2-body types
    const uint4 *idx4;         // 4-body types
    const unsigned *idx3[3];   // 3-body types (SoA, 12 B per constraint)
    const float4 *gv[kMaxGeoV];
    const float *gs[kMaxGeoS];
    const float *mat[kMaxMat]; // per-constraint material arrays, or nullptr -> matU (uniform over the type)
    float matU[kMaxMat];
    float *lambda;             // XPBD multipliers (m_lambda), zeroed at the first sweep of each substep
    float4 *rbX, *rbQ;         // joint types only: rigid-body positions (xyz, invMass) and rotations (x,y,z,w)
    const float4 *rbIinv;      // joint types only: inverse principal moments
    int variant;               // PBD_ISOBENDING*: 0 = rank-1 Kp form, 1 = full 4x4 Q
};

struct Bucket {
    int type;
    unsigned first;   // offset into the type's arrays
    unsigned count;
    unsigned colour;  // index of the reference colour group
};

// static per-type shape of the image.  nStreamV: the leading float4 geometry arrays that load_streamed (kernels.cuh) fetches
// ahead of the dependency on the previous colour phase; a projection reads any further ones itself.
struct TypeShape { int nBodies, nParams, nGeoV, nStreamV, nGeoS, nMat; bool xpbd; };

#if defined(__CUDACC__)
__host__ __device__
#endif
constexpr TypeShape type_shape(int t) {
    switch (t) {
    case PBD_DISTANCE:        return {2, 2, 0, 0, 1, 1, false};
    case PBD_DISTANCE_XPBD:   return {2, 2, 0, 0, 1, 1, true};
    case PBD_DIHEDRAL:        return {4, 2, 0, 0, 1, 1, false};
    case PBD_ISOBENDING:      return {4, 17, 4, 1, 0, 1, false};  // nGeoV: 1 (rank-1) or 4 (full Q), decided at flatten
    case PBD_ISOBENDING_XPBD: return {4, 17, 4, 1, 0, 1, true};
    case PBD_FEMTRIANGLE:     return {3, 10, 1, 1, 1, 5, false};
    case PBD_STRAINTRIANGLE:  return {3, 9, 1, 1, 0, 5, false};
    case PBD_VOLUME:          return {4, 2, 0, 0, 1, 1, false};
    case PBD_VOLUME_XPBD:     return {4, 2, 0, 0, 1, 1, true};
    case PBD_FEMTET:          return {4, 12, 2, 2, 2, 2, false};
    case PBD_FEMTET_XPBD:     return {4, 12, 2, 2, 2, 2, true};
    case PBD_STRAINTET:       return {4, 13, 2, 2, 1, 4, false};
    case PBD_SHAPEMATCHING:   return {4, 24, 6, 0, 0, 1, false};
    case PBD_BALLJOINT:       return {2, 12, 2, 2, 0, 0, false};
    case PBD_RB_PARTICLE_BALLJOINT: return {2, 6, 1, 1, 0, 0, false};
    default:                  return {0, 0, 0, 0, 0, 0, false};
    }
}

// Per-replica material parameters of a batch (pbd_set_replica_materials): one row of kMatRowFloats floats per replica, type t's
// nMat parameters at mat_offset(t).
#if defined(__CUDACC__)
__host__ __device__
#endif
constexpr int mat_offset(int t) {
    int o = 0;
    for (int u = 0; u < t; u++) o += type_shape(u).nMat;
    return o;
}
constexpr int kMatRowFloats = mat_offset(PBD_NUM_TYPES);

// Algorithmic bytes per projection (SURVEY.md section 8d): indices + particle float4 read + per-constraint constants
// + particle float4 write (+ lambda read/write for XPBD).  Isometric bending uses the rank-1 figure (4 floats Kp).
inline double algorithmic_bytes(int t, int isoVariant) {
    switch (t) {
    case PBD_DISTANCE:        return 8 + 32 + 4 + 32;
    case PBD_DISTANCE_XPBD:   return 8 + 32 + 4 + 32 + 8;
    case PBD_DIHEDRAL:        return 16 + 64 + 4 + 64;
    case PBD_ISOBENDING:      return 16 + 64 + (isoVariant ? 64 : 16) + 64;
    case PBD_ISOBENDING_XPBD: return 16 + 64 + (isoVariant ? 64 : 16) + 64 + 8;
    case PBD_FEMTRIANGLE:     return 12 + 48 + 20 + 48;
    case PBD_STRAINTRIANGLE:  return 12 + 48 + 16 + 48;
    case PBD_VOLUME:          return 16 + 64 + 4 + 64;
    case PBD_VOLUME_XPBD:     return 16 + 64 + 4 + 64 + 8;
    case PBD_FEMTET:          return 16 + 64 + 40 + 64;
    case PBD_FEMTET_XPBD:     return 16 + 64 + 40 + 64 + 8;
    case PBD_STRAINTET:       return 16 + 64 + 36 + 64;
    case PBD_SHAPEMATCHING:   return 16 + 64 + 96 + 64;
    case PBD_BALLJOINT:       return 8 + 2 * 48 + 32 + 2 * 32;   // two rigid bodies (x, q, Iinv) read, (x, q) written
    case PBD_RB_PARTICLE_BALLJOINT: return 8 + 48 + 16 + 16 + 32 + 16;  // restCm + frozen x0[4] + w[4] + numClusters[4]
    default:                  return 0;
    }
}

// Sets of constraint types, one bit per type.  k_step_resident (resident.cuh) is instantiated per mask, the leanest that
// covers the model: the everything-kernel is 20k instructions and 226 registers, and every colour phase jumps through it.
constexpr unsigned type_bit(int t) { return 1u << t; }
constexpr unsigned kMaskClothXPBD = type_bit(PBD_DISTANCE_XPBD) | type_bit(PBD_ISOBENDING_XPBD);
constexpr unsigned kMaskCloth = kMaskClothXPBD | type_bit(PBD_DISTANCE) | type_bit(PBD_ISOBENDING);
constexpr unsigned kMaskLight = type_bit(PBD_DISTANCE) | type_bit(PBD_DISTANCE_XPBD) | type_bit(PBD_DIHEDRAL) | type_bit(PBD_ISOBENDING) |
                                type_bit(PBD_ISOBENDING_XPBD) | type_bit(PBD_VOLUME) | type_bit(PBD_VOLUME_XPBD) | type_bit(PBD_FEMTRIANGLE);
// FEM solids (cfg3): tets with FEM / volume constraints; and cloth + FEM solids + the coupling joints (cfg4)
constexpr unsigned kMaskFem = type_bit(PBD_FEMTET) | type_bit(PBD_FEMTET_XPBD) | type_bit(PBD_VOLUME) | type_bit(PBD_VOLUME_XPBD);
constexpr unsigned kMaskSolid = kMaskCloth | kMaskFem | type_bit(PBD_FEMTRIANGLE) | type_bit(PBD_BALLJOINT) | type_bit(PBD_RB_PARTICLE_BALLJOINT);
constexpr unsigned kMaskAll = (1u << PBD_NUM_TYPES) - 1u;

// Block size of the resident instantiation of a type mask: the largest it compiles for without spilling (cloth 96 registers,
// light 128, everything 236).  A replica batch's light instantiation keeps the replica loop's state as well: at 512 threads (128
// registers) it spilled 44-64 bytes where the single-scene one spills 32-36, so it runs 384 threads (up to 168 registers).
constexpr unsigned resident_threads(unsigned mask, bool batch = false) {
    return mask == kMaskClothXPBD ? 640u : (mask == kMaskAll ? 256u : (batch && mask == kMaskLight ? 384u : 512u));
}

// ---- the resident image (resident.cuh) ---------------------------------------------------------------------------------------
// Index encoding: bit 31 set -> shared memory: bits 30..27 = CTA rank inside the executing cluster, bits 26..0 = slot inside that
// CTA's tile;  bit 31 clear -> device slot in the global float4 array.
constexpr unsigned kSmemFlag = 0x80000000u;
constexpr unsigned kRankShift = 27u;
constexpr unsigned kLocalMask = (1u << kRankShift) - 1u;
constexpr size_t kMaxDynamicSmem = 227u * 1024u;  // what a CTA may opt in to on sm_90
// Bank swizzle of a tile: slot s lives at tile[s ^ ((s >> 3) & 7)] (a permutation inside every aligned 64-slot block; tileCap is a
// multiple of 64).  One colour's constraints touch slots 2 or 3 apart, i.e. only half of the eight 16-byte bank groups per
// quarter-warp; the swizzle spreads such strides over all eight.
__host__ __device__ __forceinline__ unsigned tile_swizzle(unsigned s) { return s ^ ((s >> 3) & 7u); }
constexpr int kMaxClusterCtas = 16;   // non-portable cluster size (opt-in attribute), one GPC
// Dynamic shared memory of a CTA: [tile: tileCap float4][run table: nBuckets x RunEntry][xMask: 1 + nColours][colourStart: nColours + 1]
// [xNbr: kMaxXNeighbours]
// A replica batch has no X items: there the xNbr words hold the material row and the gravity of the replica the cluster is stepping.
// this CTA's two runs of one bucket (absolute indices into the type's arrays); rotR: where the run of shared-memory items starts in the
// colour's concatenated item sequence, modulo the number of threads that share it (the buckets of one colour go to different threads)
struct RunEntry { int type; unsigned firstX, nX, firstR, nR, rotR, pad0, pad1; };
constexpr unsigned kMaxXNeighbours = 32;  // one lane of the first X warp per neighbour
constexpr unsigned kXFlagStride = 16;     // unsigned long longs: every CTA's arrival flag on its own 128-byte line
static_assert(kMatRowFloats + 3 <= (int)kMaxXNeighbours, "a replica's material row and gravity are staged in the xNbr words");
__host__ __device__ inline size_t resident_smem_bytes(unsigned tileCap, unsigned nBuckets, unsigned nColours) {
    return (size_t)tileCap * sizeof(float4) + (size_t)nBuckets * sizeof(RunEntry) + (size_t)(2u * nColours + 2u + kMaxXNeighbours) * sizeof(unsigned);
}

}  // namespace pbdk
