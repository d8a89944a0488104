/* oracle/pbd_oracle.h -- TEST INFRASTRUCTURE, not product code.
 *
 * Plain-C restatement of the reference's CPU algorithm for the PBD/XPBD constraint-projection path
 * (TimeStepController::step and everything below it).  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it.  The product (libpbd_b200.so) never does.
 *
 * Pinning: the reference ships NO tests / golden vectors for this path (SURVEY.md F2).  The restatement is
 * therefore pinned against outputs of the reference itself: oracle/_ref/libpbdref_f{32,64}.so (the unmodified
 * reference sources compiled by oracle/Makefile) and the fixtures under tests/golden/ generated from it by
 * tests/golden/make_golden.py.  See tests/test_oracle_vs_ref.py and tests/test_oracle_golden.py.
 *
 * Build: `make -C oracle oracle` -> liboracle_f32.so (real=float) and liboracle_f64.so (-DORACLE_DOUBLE).
 * All floating-point values cross the ABI as double (float->double is exact) so one ctypes binding drives
 * this library and oracle/_ref alike (same function names, prefix orc_ instead of ref_).
 */
#ifndef PBD_ORACLE_H
#define PBD_ORACLE_H

#ifdef ORACLE_DOUBLE
typedef double real;
#else
typedef float real;
#endif

/* Flat constraint type codes (shared with include/pbd_b200.h and oracle/ref_driver) */
enum {
    ORC_DISTANCE = 0,        /* bodies 2; params [restLength, stiffness]                      Constraints.cpp:1166-1206 */
    ORC_DISTANCE_XPBD = 1,   /* bodies 2; params [restLength, stiffness]; lambda              Constraints.cpp:1211-1258 */
    ORC_DIHEDRAL = 2,        /* bodies 4; params [restAngle, stiffness]                       Constraints.cpp:1264-1339 */
    ORC_ISOBENDING = 3,      /* bodies 4; params [stiffness, Q(4x4 row-major)]                Constraints.cpp:1345-1402 */
    ORC_ISOBENDING_XPBD = 4, /* same + lambda                                                 Constraints.cpp:1407-1471 */
    ORC_FEMTRIANGLE = 5,     /* bodies 3; params [area, invRestMat(2x2 rm), xx, yy, xy, nu_xy, nu_yx]   :1476-1538 */
    ORC_STRAINTRIANGLE = 6,  /* bodies 3; params [invRestMat(2x2 rm), xx, yy, xy, normStretch, normShear] :1544-1610 */
    ORC_VOLUME = 7,          /* bodies 4; params [restVolume, stiffness]                      Constraints.cpp:1617-1677 */
    ORC_VOLUME_XPBD = 8,     /* same + lambda                                                 Constraints.cpp:1683-1750 */
    ORC_FEMTET = 9,          /* bodies 4; params [volume, invRestMat(3x3 rm), E, nu]          Constraints.cpp:1755-1825 */
    ORC_FEMTET_XPBD = 10,    /* same + lambda                                                 Constraints.cpp:1830-1906 */
    ORC_STRAINTET = 11,      /* bodies 4; params [invRestMat(3x3 rm), stretchK, shearK, normStretch, normShear] :1912-1980 */
    ORC_SHAPEMATCHING = 12,  /* bodies 4; params [stiffness, restCm(3), x0(4x3), w(4), numClusters(4)]  :1985-2028 */
    ORC_BALLJOINT = 13,      /* bodies (rb, rb); params [local connector 0 (3), local connector 1 (3)]   Constraints.cpp:54-125 */
    ORC_RB_PARTICLE_BALLJOINT = 14, /* bodies (rb, particle); params [local connector in the rigid body (3)]  Constraints.cpp:925-987 */
    ORC_NUM_TYPES = 15
};
#define ORC_MAX_PARAMS 24

#ifdef __cplusplus
extern "C" {
#endif

int orc_real_size(void);
void orc_set_threads(int n);
int orc_max_threads(void);
void orc_reset(void);

void orc_add_regular_triangle_model(int w, int h, const double *t, const double *R, const double *scale);
void orc_add_regular_tet_model(int w, int h, int d, const double *t, const double *R, const double *scale);
void orc_add_triangle_model(unsigned nPoints, unsigned nFaces, const double *pts, const unsigned *idx);
void orc_add_tet_model(unsigned nPoints, unsigned nTets, const double *pts, const unsigned *idx);
void orc_set_mass(unsigned i, double m);

void orc_add_cloth_constraints(unsigned triModel, unsigned method, double distK, double xx, double yy, double xy,
                               double pxy, double pyx, int normStretch, int normShear);
void orc_add_bending_constraints(unsigned triModel, unsigned method, double k);
void orc_add_solid_constraints(unsigned tetModel, unsigned method, double k, double nu, double volK,
                               int normStretch, int normShear);
int orc_add_constraint(int type, const unsigned *bodies, const double *p);
/* rigid bodies (Simulation/RigidBody.h:84-110 initBody with explicit mass / principal inertia); q = (w, x, y, z) */
unsigned orc_add_rigid_body(double mass, const double *x, const double *inertia, const double *q);
unsigned orc_num_rigid_bodies(void);
void orc_get_rigid_bodies(double *out); /* per body: x(3) q(w,x,y,z) v(3) omega(3) = 13 doubles */
void orc_set_rigid_body_velocity(unsigned i, const double *v, const double *omega); /* RigidBody::setVelocity / setAngularVelocity */

void orc_set_params(double dt, unsigned subSteps, unsigned maxIter, int velMethod, const double *g);
void orc_init_groups(void);
unsigned orc_num_particles(void);
unsigned orc_num_constraints(void);
unsigned orc_num_groups(void);
void orc_get_groups(unsigned *offsets, unsigned *ids);
void orc_get_attr(int which, double *out);      /* 0 x, 1 v, 2 x0, 3 oldX, 4 lastX, 5 a */
void orc_set_attr(int which, const double *in);
void orc_get_masses(double *mass, double *invMass);

unsigned orc_tri_num_edges(unsigned tm);
unsigned orc_tri_num_faces(unsigned tm);
unsigned orc_tri_index_offset(unsigned tm);
void orc_tri_get_edges(unsigned tm, unsigned *out); /* v0 v1 f0 f1 per edge */
void orc_tri_get_faces(unsigned tm, unsigned *out);
unsigned orc_tet_num_edges(unsigned tm);
unsigned orc_tet_num_tets(unsigned tm);
unsigned orc_tet_index_offset(unsigned tm);
void orc_tet_get_edges(unsigned tm, unsigned *out); /* v0 v1 per edge */
void orc_tet_get_tets(unsigned tm, unsigned *out);

int orc_get_constraint(unsigned i, unsigned *bodies, double *p, double *lambda);
void orc_get_constraints(int *types, unsigned *bodies, double *params, int *nbodies);

/* contact path (static analytic colliders): objects as an adapter hands them to pbd_set_colliders (see pbd_oracle.c) */
void orc_set_colliders(unsigned nModels, const double *models, unsigned nRigid, const double *rigid);
void orc_set_contact_params(double tolerance, double stiffness, unsigned maxIterV);
unsigned orc_num_contacts(void);
void orc_get_contacts(unsigned *particle, unsigned *body, double *out);

double orc_step(int n);
double orc_time(void);

int orc_kat_solve(int type, const double *x, const double *w, const double *p, double dt, int handleInversion,
                  double *lambda, double *corr);
int orc_kat_init(int type, const double *x, double *out);
void orc_kat_svd(const double *A, double *sigma, double *U, double *VT);
void orc_kat_integrate(double h, double mass, double *x, double *v, const double *a);
void orc_kat_velocity_update(int order, double h, double mass, const double *x, const double *oldX,
                             const double *lastX, double *v);

#ifdef __cplusplus
}
#endif
#endif
