// TEST INFRASTRUCTURE (see cuda_runtime.h in this directory): runs the sensing instantiation pbdk::contacts_particle<true, true> over K
// replicas, for every particle, sequentially, on the host.  Each particle's sensors go to sense[r * total + gid] (zeroed by the caller);
// the block sums of the GPU kernel are left to the caller.
#include "contacts.cuh"
#include <vector>
using namespace pbdk;
extern "C" void run_contact_sensors(unsigned K, unsigned n, const unsigned *slot, float4 *pos, float4 *vel, const float4 *rbX, const float4 *rbV,
                                    const float4 *rbW, unsigned nRigid, const RigidCollider *rigid, unsigned nRanges, const ParticleCollider *ranges,
                                    float tol, float stiff, unsigned iters, ContactRecord *rec, unsigned *recCount, unsigned recCap, ContactSense *sense) {
    std::vector<unsigned> start(nRanges + 1, 0);
    for (unsigned r = 0; r < nRanges; r++) start[r + 1] = start[r] + ranges[r].count;
    ContactArgs A{pos, vel, slot, rbX, rbV, rbW, rigid, nRigid, ranges, nRanges, start.data(), start[nRanges], tol, stiff, iters, rec, recCount, recCap};
    A.n = n;
    for (unsigned r = 0; r < K; r++)
        for (unsigned g = 0; g < A.total; g++) contacts_particle<true, true>(A, g, r, sense + (size_t)r * A.total + g);
}
