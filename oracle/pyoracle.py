"""oracle/pyoracle.py -- TEST INFRASTRUCTURE (ctypes driver for the CPU checkers).

One binding for both CPU libraries, which export the same entry points under different prefixes:
  * oracle/liboracle_f{32,64}.so      prefix ``orc_``  -- the plain-C restatement (oracle/pbd_oracle.c)
  * oracle/_ref/libpbdref_f{32,64}.so prefix ``ref_``  -- the unmodified reference (oracle/ref_driver)

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
Each library holds ONE global model (mirroring the reference's Simulation singleton, Simulation.cpp:11),
so a CpuPbd object is a thin namespace, not an instance handle.
"""
import ctypes as C
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# flat constraint type codes (include/pbd_b200.h, oracle/pbd_oracle.h)
DISTANCE, DISTANCE_XPBD, DIHEDRAL, ISOBENDING, ISOBENDING_XPBD, FEMTRIANGLE, STRAINTRIANGLE, VOLUME, \
    VOLUME_XPBD, FEMTET, FEMTET_XPBD, STRAINTET, SHAPEMATCHING, BALLJOINT, RB_PARTICLE_BALLJOINT = range(15)
TYPE_NAMES = ["Distance", "Distance_XPBD", "Dihedral", "IsometricBending", "IsometricBending_XPBD", "FEMTriangle",
              "StrainTriangle", "Volume", "Volume_XPBD", "FEMTet", "FEMTet_XPBD", "StrainTet", "ShapeMatching", "BallJoint",
              "RigidBodyParticleBallJoint"]
NPARAMS = [2, 2, 2, 17, 17, 10, 9, 2, 2, 12, 12, 13, 24, 12, 6]
NBODIES = [2, 2, 4, 4, 4, 3, 3, 4, 4, 4, 4, 4, 4, 2, 2]
MAX_PARAMS = 24

_D = C.c_double
_dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
_up = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint))
_ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))


def _f64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


def build(ref=True):
    """Compile the C restatement and (when /root/reference is present) oracle/_ref."""
    subprocess.check_call(["make", "-s", "-C", HERE, "oracle"])
    if ref:
        subprocess.check_call(["make", "-s", "-j8", "-C", HERE, "ref"])


def lib_path(kind, precision):
    """kind: 'oracle' | 'ref' | 'refgpu' (reference build + integration/GpuTimeStepController.h); precision: 'f32' | 'f64'."""
    if kind == "oracle":
        return os.path.join(HERE, "liboracle_%s.so" % precision)
    if kind == "refgpu":
        return os.path.join(HERE, "_ref", "libpbdref_gpu_%s.so" % precision)
    return os.path.join(HERE, "_ref", "libpbdref_%s.so" % precision)


def available(kind, precision):
    return os.path.exists(lib_path(kind, precision))


def best_ref_variant():
    """(path, flag) of the fastest fp32 reference build this host can run: the AVX-512 build (-march=x86-64-v4) when the CPU has
    the x86-64-v4 feature set and the library travelled here, else the portable AVX2 build (-march=x86-64-v3)."""
    v4 = os.path.join(HERE, "_ref", "libpbdref_f32_v4.so")
    try:
        flags = set()
        for ln in open("/proc/cpuinfo"):
            if ln.startswith("flags"):
                flags = set(ln.split(":", 1)[1].split()); break
        if os.path.exists(v4) and {"avx512f", "avx512bw", "avx512cd", "avx512dq", "avx512vl"} <= flags:
            return v4, "-march=x86-64-v4"
    except OSError:
        pass
    return lib_path("ref", "f32"), "-march=x86-64-v3"


class CpuPbd:
    def __init__(self, kind="oracle", precision="f32", path=None):
        self.kind, self.precision = kind, precision
        self.prefix = "orc_" if kind == "oracle" else "ref_"
        self.lib = C.CDLL(path or lib_path(kind, precision))
        for name in ("step", "time"):
            getattr(self.lib, self.prefix + name).restype = C.c_double
        assert self.f("real_size")() == (4 if precision == "f32" else 8)
        # the reference forks an OpenMP team per colour group; on many-core hosts the default team (all hardware threads)
        # makes small scenes crawl.  Checkers default to a small team; bench.py picks its own.
        self.set_threads(min(8, os.cpu_count() or 1))
        self.reset()

    def f(self, name):
        return getattr(self.lib, self.prefix + name)

    # -- scene construction ---------------------------------------------------------------------
    def reset(self):
        self.f("reset")()

    def set_threads(self, n):
        self.f("set_threads")(int(n))

    def max_threads(self):
        return self.f("max_threads")()

    def add_regular_triangle_model(self, w, h, t=(0, 0, 0), R=np.eye(3), scale=(1, 1)):
        self.f("add_regular_triangle_model")(w, h, _dp(_f64(t)), _dp(_f64(R)), _dp(_f64(scale)))

    def add_regular_tet_model(self, w, h, d, t=(0, 0, 0), R=np.eye(3), scale=(1, 1, 1)):
        self.f("add_regular_tet_model")(w, h, d, _dp(_f64(t)), _dp(_f64(R)), _dp(_f64(scale)))

    def add_triangle_model(self, pts, faces):
        pts = _f64(pts); faces = np.ascontiguousarray(faces, dtype=np.uint32)
        self.f("add_triangle_model")(len(pts), len(faces), _dp(pts), _up(faces))

    def add_tet_model(self, pts, tets):
        pts = _f64(pts); tets = np.ascontiguousarray(tets, dtype=np.uint32)
        self.f("add_tet_model")(len(pts), len(tets), _dp(pts), _up(tets))

    def set_mass(self, i, m):
        self.f("set_mass")(int(i), _D(m))

    def add_cloth_constraints(self, tm, method, dist_k=1.0, xx=1.0, yy=1.0, xy=1.0, pxy=0.3, pyx=0.3,
                              norm_stretch=False, norm_shear=False):
        self.f("add_cloth_constraints")(tm, method, _D(dist_k), _D(xx), _D(yy), _D(xy), _D(pxy), _D(pyx),
                                        int(norm_stretch), int(norm_shear))

    def add_bending_constraints(self, tm, method, k):
        self.f("add_bending_constraints")(tm, method, _D(k))

    def add_solid_constraints(self, tm, method, k=1.0, nu=0.3, vol_k=1.0, norm_stretch=False, norm_shear=False):
        self.f("add_solid_constraints")(tm, method, _D(k), _D(nu), _D(vol_k), int(norm_stretch), int(norm_shear))

    def add_constraint(self, ctype, bodies, params):
        b = np.zeros(4, dtype=np.uint32); b[:len(bodies)] = bodies
        p = np.zeros(8, dtype=np.float64); p[:len(params)] = params
        return self.f("add_constraint")(ctype, _up(b), _dp(p))

    # -- rigid bodies and the joints coupling them to particles (SURVEY.md 8f-1) ---------------------------------
    def add_rigid_body(self, mass, x, inertia, q=(1, 0, 0, 0)):
        """q = (w, x, y, z); inertia = principal moments (RigidBody::initBody, RigidBody.h:84-120)."""
        self.f("add_rigid_body").restype = C.c_uint
        return self.f("add_rigid_body")(_D(mass), _dp(_f64(x)), _dp(_f64(inertia)), _dp(_f64(q)))

    def set_rigid_body_velocity(self, i, v, omega):
        """RigidBody::setVelocity / setAngularVelocity of body i."""
        self.f("set_rigid_body_velocity")(int(i), _dp(_f64(v)), _dp(_f64(omega)))

    def add_rigid_body_mesh(self, density, verts, faces, x=(0, 0, 0), R=np.eye(3), scale=(1, 1, 1)):
        """ref only: RigidBody::initBody(density, x, rotation, vertices, mesh, scale); returns (index, [mass, inertia(3), x(3), q(w,x,y,z)])."""
        assert self.kind != "oracle"
        v = _f64(verts).reshape(-1, 3); f = np.ascontiguousarray(faces, dtype=np.uint32).reshape(-1, 3)
        i = self.lib.ref_add_rigid_body_mesh(_D(density), len(v), _dp(v), len(f), f.ctypes.data_as(C.c_void_p), _dp(_f64(x)), _dp(_f64(R)), _dp(_f64(scale)))
        out = np.zeros(11); self.lib.ref_get_rigid_body_props(i, _dp(out))
        return i, out

    # -- contact path (reference builds only): DistanceFieldCollisionDetection as Demos/DistanceFieldDemos/ClothCollisionDemo.cpp sets it up
    def use_distance_field_cd(self, tolerance=0.01):
        assert self.kind != "oracle"
        self.lib.ref_use_distance_field_cd(_D(tolerance))

    def set_rigid_body_mass(self, i, m):
        self.lib.ref_set_rigid_body_mass(int(i), _D(m))

    def add_rigid_collider(self, body, shape, dims, thickness=0.0, invert=False, restitution=0.6, friction=0.2):
        """shape 0 box (full extents) | 1 sphere (radius) | 2 torus (radii) | 3 cylinder (radius, height) | 4 hollow sphere | 5 hollow box."""
        d = np.zeros(3); d[:len(np.atleast_1d(dims))] = np.atleast_1d(dims)
        rc = self.lib.ref_add_rigid_collider(int(body), int(shape), _dp(d), _D(thickness), int(bool(invert)), _D(restitution), _D(friction))
        assert rc == 0, rc

    def add_model_collider(self, kind, model_index, restitution=0.6, friction=0.2):
        """kind 0: triangle model, 1: tet model (addCollisionObjectWithoutGeometry, testMesh = true)."""
        assert self.lib.ref_add_model_collider(int(kind), int(model_index), _D(restitution), _D(friction)) == 0

    def set_contact_params(self, stiffness=100.0, max_iter_v=5):
        self.lib.ref_set_contact_params(_D(stiffness), int(max_iter_v))

    def contacts(self):
        """Particle / rigid-body contacts of the last step: (particle[n], body[n], info[n, 10] = cp0 | cp1 | normal | 1/(n^T K n)), plus the
        counts of the contact kinds the GPU path does not cover (rigid-rigid, particle-tet)."""
        rr = C.c_uint(0); pt = C.c_uint(0)
        self.lib.ref_num_contacts.restype = C.c_uint
        n = self.lib.ref_num_contacts(C.byref(rr), C.byref(pt))
        particle = np.zeros(max(n, 1), dtype=np.uint32); body = np.zeros(max(n, 1), dtype=np.uint32); info = np.zeros((max(n, 1), 10))
        self.lib.ref_get_contacts(particle.ctypes.data_as(C.c_void_p), body.ctypes.data_as(C.c_void_p), _dp(info))
        return particle[:n], body[:n], info[:n], rr.value, pt.value

    def collision_objects(self):
        """What an adapter passes to pbd_set_colliders: ([(offset, count, restitution, friction)], [30 doubles per rigid collider]) in list order."""
        self.lib.ref_num_collision_objects.restype = C.c_uint
        models, rigid = [], []
        for i in range(self.lib.ref_num_collision_objects()):
            out = np.zeros(32)
            kind = self.lib.ref_collision_object_info(i, _dp(out))
            if kind == 0: rigid.append(out[:30].copy())
            elif kind in (1, 2): models.append((int(out[0]), int(out[1]), float(out[2]), float(out[3])))
            else: raise RuntimeError("collision object %d is of a kind the contact path does not cover" % i)
        return models, rigid

    # -- contact path of the C restatement: colliders handed over the way an adapter hands them to pbd_set_colliders
    def set_colliders(self, models, rigid):
        """oracle only: `models` = [(offset, count, restitution, friction)], `rigid` = 30 doubles per collider (collision_objects() of a reference build)."""
        assert self.kind == "oracle"
        mo = _f64(np.asarray(models, dtype=np.float64).reshape(-1, 4)); ri = _f64(np.asarray(rigid, dtype=np.float64).reshape(-1, 30))
        self.lib.orc_set_colliders(len(mo), _dp(mo), len(ri), _dp(ri))

    def set_oracle_contact_params(self, tolerance=0.01, stiffness=100.0, max_iter_v=5):
        assert self.kind == "oracle"
        self.lib.orc_set_contact_params(_D(tolerance), _D(stiffness), int(max_iter_v))

    def oracle_contacts(self):
        self.lib.orc_num_contacts.restype = C.c_uint
        n = self.lib.orc_num_contacts()
        particle = np.zeros(max(n, 1), dtype=np.uint32); body = np.zeros(max(n, 1), dtype=np.uint32); info = np.zeros((max(n, 1), 10))
        self.lib.orc_get_contacts(particle.ctypes.data_as(C.c_void_p), body.ctypes.data_as(C.c_void_p), _dp(info))
        return particle[:n], body[:n], info[:n]

    def add_ball_joint(self, rb0, rb1, pos):
        return self.add_constraint(BALLJOINT, [rb0, rb1], list(pos))

    def add_rb_particle_ball_joint(self, rb, particle):
        return self.add_constraint(RB_PARTICLE_BALLJOINT, [rb, particle], [])

    def rigid_bodies(self):
        """[n, 13]: x(3) q(w,x,y,z) v(3) omega(3)."""
        self.f("num_rigid_bodies").restype = C.c_uint
        n = self.f("num_rigid_bodies")()
        out = np.zeros((max(n, 1), 13)); self.f("get_rigid_bodies")(_dp(out)); return out[:n]

    def use_gpu_timestep(self, device=0, mode=0):
        """refgpu only: install PBD::GpuTimeStepController (integration/GpuTimeStepController.h) as the reference's TimeStep."""
        assert self.kind == "refgpu"
        self.lib.ref_gpu_error.restype = C.c_char_p
        if self.lib.ref_use_gpu_timestep(int(device), int(mode)):
            raise RuntimeError(self.lib.ref_gpu_error().decode())

    def gpu_error(self):
        self.lib.ref_gpu_error.restype = C.c_char_p
        return self.lib.ref_gpu_error().decode()

    def attach_collision_object(self):
        """refgpu only: TimeStep::setCollisionDetection with one collision object, as the reference's collision demos do."""
        assert self.kind == "refgpu"
        return int(self.lib.ref_attach_collision_object())

    def set_cloth_stiffness(self, k):
        """SimulationModel::setClothStiffness (ref / refgpu): rewrites m_stiffness of every cloth constraint."""
        assert self.kind in ("ref", "refgpu")
        self.lib.ref_set_cloth_stiffness(_D(k))

    def set_host_state_authoritative(self, on):
        """refgpu only: GpuTimeStepController::setHostStateAuthoritative (false: no per-step upload of x and v)."""
        assert self.kind == "refgpu"
        self.lib.ref_set_host_state_authoritative(int(bool(on)))

    def invalidate_state(self):
        assert self.kind == "refgpu"
        self.lib.ref_invalidate_state_gpu()

    def download_history(self):
        assert self.kind == "refgpu"
        return int(self.lib.ref_download_history())

    def set_params(self, dt=0.005, sub_steps=5, max_iter=1, vel_method=0, gravity=(0, -9.81, 0)):
        self.f("set_params")(_D(dt), sub_steps, max_iter, vel_method, _dp(_f64(gravity)))

    # -- structure ------------------------------------------------------------------------------
    def init_groups(self):
        self.f("init_groups")()

    def num_particles(self):
        return self.f("num_particles")()

    def num_constraints(self):
        return self.f("num_constraints")()

    def groups(self):
        self.init_groups()
        ng, nc = self.f("num_groups")(), self.num_constraints()
        off = np.zeros(ng + 1, dtype=np.uint32); ids = np.zeros(max(nc, 1), dtype=np.uint32)
        self.f("get_groups")(_up(off), _up(ids))
        return off, ids[:nc]

    def constraints(self):
        nc = self.num_constraints()
        types = np.zeros(max(nc, 1), dtype=np.int32); nb = np.zeros(max(nc, 1), dtype=np.int32)
        bodies = np.zeros((max(nc, 1), 4), dtype=np.uint32); params = np.zeros((max(nc, 1), MAX_PARAMS), dtype=np.float64)
        self.f("get_constraints")(_ip(types), _up(bodies), _dp(params), _ip(nb))
        return types[:nc], bodies[:nc], params[:nc], nb[:nc]

    def tri_edges(self, tm=0):
        n = self.f("tri_num_edges")(tm)
        out = np.zeros((n, 4), dtype=np.uint32); self.f("tri_get_edges")(tm, _up(out)); return out

    def tri_faces(self, tm=0):
        n = self.f("tri_num_faces")(tm)
        out = np.zeros((n, 3), dtype=np.uint32); self.f("tri_get_faces")(tm, _up(out)); return out

    def tet_edges(self, tm=0):
        n = self.f("tet_num_edges")(tm)
        out = np.zeros((n, 2), dtype=np.uint32); self.f("tet_get_edges")(tm, _up(out)); return out

    def tet_tets(self, tm=0):
        n = self.f("tet_num_tets")(tm)
        out = np.zeros((n, 4), dtype=np.uint32); self.f("tet_get_tets")(tm, _up(out)); return out

    # -- state ----------------------------------------------------------------------------------
    ATTR = {"x": 0, "v": 1, "x0": 2, "oldX": 3, "lastX": 4, "a": 5}

    def get(self, name="x"):
        out = np.zeros((self.num_particles(), 3), dtype=np.float64)
        self.f("get_attr")(self.ATTR[name], _dp(out)); return out

    def set(self, name, arr):
        arr = _f64(arr); assert arr.shape == (self.num_particles(), 3)
        self.f("set_attr")(self.ATTR[name], _dp(arr))

    def masses(self):
        n = self.num_particles()
        m = np.zeros(n); w = np.zeros(n); self.f("get_masses")(_dp(m), _dp(w)); return m, w

    def step(self, n=1):
        """n x TimeStepController::step; returns wall seconds."""
        return self.f("step")(int(n))

    # -- known-answer entry points --------------------------------------------------------------
    def time(self):
        """TimeManager::getTime of the checker."""
        return self.f("time")()

    def kat_solve(self, ctype, x, w, params, dt=0.005, handle_inversion=False, lam=0.0):
        x = _f64(x).reshape(4, 3).copy(); w = _f64(w); p = np.zeros(MAX_PARAMS); p[:len(params)] = params
        lam_c = _D(lam); corr = np.zeros((4, 3))
        res = self.f("kat_solve")(ctype, _dp(x), _dp(w), _dp(p), _D(dt), int(handle_inversion), C.byref(lam_c), _dp(corr))
        return res, corr, lam_c.value

    def kat_init(self, ctype, x):
        x = _f64(x).reshape(4, 3).copy(); out = np.zeros(MAX_PARAMS)
        res = self.f("kat_init")(ctype, _dp(x), _dp(out)); return res, out

    def kat_svd(self, A):
        A = _f64(A).reshape(3, 3).copy(); s = np.zeros(3); U = np.zeros((3, 3)); VT = np.zeros((3, 3))
        self.f("kat_svd")(_dp(A), _dp(s), _dp(U), _dp(VT)); return s, U, VT

    def kat_integrate(self, h, mass, x, v, a):
        x = _f64(x).copy(); v = _f64(v).copy(); a = _f64(a)
        self.f("kat_integrate")(_D(h), _D(mass), _dp(x), _dp(v), _dp(a)); return x, v

    def kat_velocity_update(self, order, h, mass, x, old_x, last_x, v):
        v = _f64(v).copy()
        self.f("kat_velocity_update")(order, _D(h), _D(mass), _dp(_f64(x)), _dp(_f64(old_x)), _dp(_f64(last_x)), _dp(v))
        return v
