/* tests/oracle_ext/external_accel.c -- TEST INFRASTRUCTURE: the C restatement (oracle/pbd_oracle.c, compiled here unmodified and
 * whole) plus a per-particle external acceleration, the fp64 statement of pbd_set_external_forces.
 *
 *   orc_set_ext_accel(a): a = n x 3 doubles, particle i's external acceleration (f_i / m_i); NULL clears it.
 *   orc_step_ext(n)     : n x TimeStepController::step as orc_step, where clearAccelerations sets a[i] = gravity + ext[i] (in real)
 *                         for every particle with mass while an acceleration is set.  Everything else -- substeps of dt / subSteps,
 *                         rigid bodies, projections, velocity updates, the contact step once per step -- is step_once's own code
 *                         and calls.  With no acceleration set it computes exactly what orc_step computes (pinned bit for bit in
 *                         tests/test_external_forces_checks.py).
 * Built by tests/external_forces_util.py with oracle/Makefile's CFLAGS (and -DORACLE_DOUBLE for fp64). */
#include "../../oracle/pbd_oracle.c"

static vec3 *extAccel = NULL;
static unsigned extCount = 0;

void orc_set_ext_accel(const double *a) {
    free(extAccel); extAccel = NULL; extCount = 0;
    if (!a) return;
    extCount = G->n;
    extAccel = (vec3 *)malloc((size_t)(extCount ? extCount : 1) * sizeof(vec3));
    for (unsigned i = 0; i < extCount; i++) extAccel[i] = V((real)a[3 * i], (real)a[3 * i + 1], (real)a[3 * i + 2]);
}

/* step_once (pbd_oracle.c) with the external acceleration in clearAccelerations; the rest of the body is step_once's, line for line */
static void step_once_ext(Model *m) {
    const real hOld = m->dt;
    const int n = (int)m->n;
    for (int i = 0; i < n; i++)
        if (m->mass[i] != R(0.0)) m->a[i] = (extAccel && (unsigned)i < extCount) ? vadd(m->gravity, extAccel[i]) : m->gravity;
    for (unsigned i = 0; i < m->nRb; i++) if (m->rbs[i].mass != R(0.0)) m->rbs[i].a = m->gravity;
    const real h = hOld / (real)m->subSteps;
    for (unsigned s = 0; s < m->subSteps; s++) {
        for (unsigned i = 0; i < m->nRb; i++) {
            RigidBody *b = &m->rbs[i];
            b->lastX = b->oldX; b->oldX = b->x;
            if (b->mass != R(0.0)) { b->v = vadd(b->v, vmul(b->a, h)); b->x = vadd(b->x, vmul(b->v, h)); }
            b->lastQ = b->oldQ; b->oldQ = b->q;
            if (b->mass != R(0.0)) {
                vec3 t = vsub(b->torque, vcross(b->omega, mvec(&b->inertiaW, b->omega)));
                b->omega = vadd(b->omega, vmul(mvec(&b->inertiaInvW, t), h));
                quat wq = {R(0.0), b->omega.v[0], b->omega.v[1], b->omega.v[2]};
                quat dq = qmul(wq, b->q);
                const double hh = (double)h * 0.5;
                b->q.w += (real)(hh * dq.w); b->q.x += (real)(hh * dq.x); b->q.y += (real)(hh * dq.y); b->q.z += (real)(hh * dq.z);
                b->q = qnormalize(b->q);
            }
            rb_rotation_updated(b);
        }
#pragma omp parallel for schedule(static)
        for (int i = 0; i < n; i++) {
            m->lastX[i] = m->oldX[i];
            m->oldX[i] = m->x[i];
            if (m->mass[i] != R(0.0)) {
                m->v[i] = vadd(m->v[i], vmul(m->a[i], h));
                m->x[i] = vadd(m->x[i], vmul(m->v[i], h));
            }
        }
        position_constraint_projection(m, h);
        for (unsigned i = 0; i < m->nRb; i++) {
            RigidBody *b = &m->rbs[i];
            if (b->mass == R(0.0)) continue;
            if (m->velMethod == 0) b->v = vmul(vsub(b->x, b->oldX), (real)(1.0 / h));
            else {
                vec3 t;
                for (int k = 0; k < 3; k++) t.v[k] = (real)(1.5 * b->x.v[k]) - (real)(2.0 * b->oldX.v[k]) + (real)(0.5 * b->lastX.v[k]);
                b->v = vmul(t, (real)(1.0 / h));
            }
            quat rel = qmul(b->q, qconj(b->oldQ));
            b->omega = vmul(V(rel.x, rel.y, rel.z), (real)(2.0 / h));
        }
#pragma omp parallel for schedule(static)
        for (int i = 0; i < n; i++) {
            if (m->mass[i] == R(0.0)) continue;
            if (m->velMethod == 0) {
                m->v[i] = vmul(vsub(m->x[i], m->oldX[i]), (real)(1.0 / h));
            } else {
                vec3 t;
                for (int k = 0; k < 3; k++)
                    t.v[k] = (real)(1.5 * m->x[i].v[k]) - (real)(2.0 * m->oldX[i].v[k]) + (real)(0.5 * m->lastX[i].v[k]);
                m->v[i] = vmul(t, (real)(1.0 / h));
            }
        }
    }
    if (m->nRigidColl && m->nPartColl) { contact_detection(m); contact_velocity_projection(m); }
    m->time += hOld;
}

double orc_step_ext(int n) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int i = 0; i < n; i++) step_once_ext(G);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
