// TEST INFRASTRUCTURE (see cuda_runtime.h in this directory): the rest geometry of csrc/rest_geometry.cuh -- what k_derive_geometry runs
// for every replica of a batch and the host mirror's add*Constraint for one scene -- evaluated on the host, one constraint at a time.
#define __host__
struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
#include "rest_geometry.cuh"
using namespace pbdk;

extern "C" int geometry_columns(int type) { return num_geo(type); }

// count constraints of `type` on `bodies` (nBodies each) over the rest positions x (.w = inverse mass): the geometry columns into
// geo[count][num_geo(type)], the accept flag of initConstraint into ok[count]; IsometricBending also factor_rank1's verdict into rank1
extern "C" void derive_rest_geometry(int type, unsigned count, const unsigned *bodies, const float4 *x, float *geo, unsigned char *ok, unsigned char *rank1) {
    const int nb = type_shape(type).nBodies, ng = num_geo(type);
    for (unsigned c = 0; c < count; c++) {
        float4 p[4];
        for (int k = 0; k < nb; k++) p[k] = x[bodies[(size_t)c * nb + k]];
        float *g = geo + (size_t)c * ng;
        for (int j = 0; j < ng; j++) g[j] = 0.0f;
        ok[c] = rest_geometry(type, p, g) ? 1 : 0;
        float Kp[4];
        if (rank1) rank1[c] = (type == PBD_ISOBENDING || type == PBD_ISOBENDING_XPBD) ? (factor_rank1(g, Kp) ? 1 : 0) : 1;
    }
}
