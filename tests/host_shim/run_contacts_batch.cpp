// TEST INFRASTRUCTURE (see cuda_runtime.h in this directory): runs pbdk::k_contacts_batch over K replicas, and pbdk::k_contacts on one
// scene, for every particle, sequentially, on the host.  blockIdx.y carries the replica as the batched launch's grid rows do.
#include "contacts.cuh"
#include <vector>
using namespace pbdk;
// pos / vel: K * n slots (replica r at [r n, (r + 1) n), slot[i] within a replica); rbX / rbV / rbW / rigid: K * nRigid, replica after replica
extern "C" void run_contacts_batch(unsigned K, unsigned n, const unsigned *slot, float4 *pos, float4 *vel, const float4 *rbX, const float4 *rbV,
                                   const float4 *rbW, unsigned nRigid, const RigidCollider *rigid, unsigned nRanges, const ParticleCollider *ranges,
                                   float tol, float stiff, unsigned iters, ContactRecord *rec, unsigned *recCount, unsigned recCap) {
    std::vector<unsigned> start(nRanges + 1, 0);
    for (unsigned r = 0; r < nRanges; r++) start[r + 1] = start[r] + ranges[r].count;
    ContactArgs A{pos, vel, slot, rbX, rbV, rbW, rigid, nRigid, ranges, nRanges, start.data(), start[nRanges], tol, stiff, iters, rec, recCount, recCap};
    A.n = n;
    blockDim.x = 1;
    for (unsigned r = 0; r < K; r++)
        for (unsigned g = 0; g < A.total; g++) { blockIdx.x = g; blockIdx.y = r; threadIdx.x = 0; k_contacts_batch(A); }
}
// one scene: collider k on body rigid[k].body of rbX / rbV / rbW
extern "C" void run_contacts_solo(const unsigned *slot, float4 *pos, float4 *vel, const float4 *rbX, const float4 *rbV, const float4 *rbW,
                                  unsigned nRigid, const RigidCollider *rigid, unsigned nRanges, const ParticleCollider *ranges,
                                  float tol, float stiff, unsigned iters, ContactRecord *rec, unsigned *recCount, unsigned recCap) {
    std::vector<unsigned> start(nRanges + 1, 0);
    for (unsigned r = 0; r < nRanges; r++) start[r + 1] = start[r] + ranges[r].count;
    ContactArgs A{pos, vel, slot, rbX, rbV, rbW, rigid, nRigid, ranges, nRanges, start.data(), start[nRanges], tol, stiff, iters, rec, recCount, recCap};
    blockDim.x = 1;
    for (unsigned g = 0; g < A.total; g++) { blockIdx.x = g; blockIdx.y = 0; threadIdx.x = 0; k_contacts(A); }
}
