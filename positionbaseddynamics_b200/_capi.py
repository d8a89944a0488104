"""ctypes binding of the engine-level C ABI (include/pbd_b200.h) exported by libpbd_b200.so.

This is plumbing only: every call goes straight into the CUDA library.  There is no Python or CPU fallback --
if the shared library is missing or no CUDA device is present the calls raise.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PBD_B200_LIB") or os.path.join(_HERE, "libpbd_b200.so")  # the override is a development aid (A/B builds)

(DISTANCE, DISTANCE_XPBD, DIHEDRAL, ISOBENDING, ISOBENDING_XPBD, FEMTRIANGLE, STRAINTRIANGLE, VOLUME, VOLUME_XPBD,
 FEMTET, FEMTET_XPBD, STRAINTET, SHAPEMATCHING, BALLJOINT, RB_PARTICLE_BALLJOINT) = range(15)
NUM_TYPES = 15
TYPE_NAMES = ["Distance", "Distance_XPBD", "Dihedral", "IsometricBending", "IsometricBending_XPBD", "FEMTriangle",
              "StrainTriangle", "Volume", "Volume_XPBD", "FEMTet", "FEMTet_XPBD", "StrainTet", "ShapeMatching", "BallJoint",
              "RigidBodyParticleBallJoint"]
ATTR_X, ATTR_V, ATTR_X0, ATTR_OLDX, ATTR_LASTX = range(5)
MODE_GRAPH, MODE_RESIDENT, MODE_LAUNCH, MODE_JACOBI, MODE_AUTO = 0, 1, 2, 3, 4

# every symbol include/pbd_b200.h declares (checked by tests/test_capi_symbols.py)
SYMBOLS = ["pbd_last_error", "pbd_device_count", "pbd_create", "pbd_destroy", "pbd_set_particles", "pbd_set_attr",
           "pbd_get_attr", "pbd_set_masses", "pbd_set_rigid_bodies", "pbd_get_rigid_bodies", "pbd_clear_constraints", "pbd_add_constraints", "pbd_num_bodies",
           "pbd_num_params", "pbd_set_groups", "pbd_color_first_fit", "pbd_color_first_fit_device", "pbd_pin_host", "pbd_unpin_host", "pbd_get_num_groups", "pbd_get_groups",
           "pbd_set_params", "pbd_set_mode", "pbd_get_mode", "pbd_step", "pbd_sync", "pbd_step_host", "pbd_step_host_async", "pbd_step_host_wait",
           "pbd_get_lambdas", "pbd_get_stats", "pbd_profile_step", "pbd_set_replicas", "pbd_get_replicas",
           "pbd_num_materials", "pbd_set_replica_materials", "pbd_set_replica_gravity",
           "pbd_set_replica_rest_positions", "pbd_get_replica_geometry",
           "pbd_set_colliders", "pbd_set_contact_params", "pbd_record_contacts", "pbd_get_contacts", "pbd_set_replica_colliders",
           "pbd_set_attr_device", "pbd_get_attr_device", "pbd_set_masses_device", "pbd_set_external_forces", "pbd_set_external_forces_device",
           "pbd_set_replica_constraint_materials", "pbd_set_replica_constraint_materials_device", "pbd_get_replica_materials",
           "pbd_set_replica_rigid_bodies", "pbd_set_rigid_bodies_device", "pbd_get_rigid_bodies_device",
           "pbd_set_replica_collider_poses_device", "pbd_sense_contacts", "pbd_get_contact_sensors", "pbd_get_contact_sensors_device"]


SHAPE_BOX, SHAPE_SPHERE, SHAPE_TORUS, SHAPE_CYLINDER, SHAPE_HOLLOW_SPHERE, SHAPE_HOLLOW_BOX = range(6)


class ParticleCollider(C.Structure):
    _fields_ = [("offset", C.c_uint), ("count", C.c_uint), ("restitution", C.c_float), ("friction", C.c_float)]


class RigidCollider(C.Structure):
    _fields_ = [("shape", C.c_int), ("body", C.c_uint), ("dim", C.c_float * 3), ("thickness", C.c_float), ("invert_sdf", C.c_int),
                ("restitution", C.c_float), ("friction", C.c_float), ("R", C.c_float * 9), ("v1", C.c_float * 3), ("v2", C.c_float * 3),
                ("aabb_min", C.c_float * 3), ("aabb_max", C.c_float * 3)]


class Contact(C.Structure):
    _fields_ = [("particle", C.c_uint), ("body", C.c_uint), ("cp0", C.c_float * 3), ("cp1", C.c_float * 3), ("normal", C.c_float * 3), ("dist", C.c_float)]


class Stats(C.Structure):
    _fields_ = [("projections", C.c_ulonglong), ("kernel_launches", C.c_ulonglong), ("steps", C.c_ulonglong),
                ("num_particles", C.c_uint), ("num_constraints", C.c_uint), ("num_groups", C.c_uint),
                ("num_buckets", C.c_uint), ("constraints_per_type", C.c_uint * NUM_TYPES),
                ("bytes_per_step", C.c_double), ("last_step_ms", C.c_float), ("images_planned", C.c_ulonglong), ("graph_captures", C.c_ulonglong)]


class PbdError(RuntimeError):
    pass


_lib = None


def lib():
    """Load libpbd_b200.so (built in-tree by __graft_entry__.build()).  Fails loudly when it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PbdError("native library %s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no Python/CPU fallback)" % LIB_PATH)
        _lib = C.CDLL(LIB_PATH)
        _lib.pbd_last_error.restype = C.c_char_p
        _lib.pbd_create.argtypes = [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
        for name in SYMBOLS:
            fn = getattr(_lib, name)
            if name not in ("pbd_last_error",):
                fn.restype = C.c_int
        for name in ("pbd_destroy", "pbd_clear_constraints", "pbd_color_first_fit", "pbd_sync"):
            getattr(_lib, name).argtypes = [C.c_void_p]
        _lib.pbd_color_first_fit_device.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_uint)]
        _lib.pbd_set_particles.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_set_attr.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib.pbd_get_attr.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib.pbd_set_masses.argtypes = [C.c_void_p, C.c_void_p]
        _lib.pbd_set_rigid_bodies.argtypes = [C.c_void_p, C.c_uint] + [C.c_void_p] * 6
        _lib.pbd_get_rigid_bodies.argtypes = [C.c_void_p] + [C.c_void_p] * 4
        _lib.pbd_add_constraints.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_set_groups.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p]
        _lib.pbd_get_num_groups.argtypes = [C.c_void_p, C.POINTER(C.c_uint)]
        _lib.pbd_get_groups.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_set_params.argtypes = [C.c_void_p, C.c_float, C.c_uint, C.c_uint, C.c_int, C.c_void_p]
        _lib.pbd_set_mode.argtypes = [C.c_void_p, C.c_int]
        _lib.pbd_get_mode.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        _lib.pbd_step.argtypes = [C.c_void_p, C.c_uint]
        _lib.pbd_step_host.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_step_host_async.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_step_host_wait.argtypes = [C.c_void_p, C.c_uint]
        _lib.pbd_set_colliders.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p]
        _lib.pbd_set_replica_colliders.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_set_contact_params.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_uint]
        _lib.pbd_record_contacts.argtypes = [C.c_void_p, C.c_uint]
        _lib.pbd_get_contacts.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.POINTER(C.c_uint)]
        _lib.pbd_get_lambdas.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib.pbd_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        _lib.pbd_profile_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_set_replicas.argtypes = [C.c_void_p, C.c_uint]
        _lib.pbd_get_replicas.argtypes = [C.c_void_p, C.POINTER(C.c_uint)]
        _lib.pbd_set_replica_materials.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib.pbd_set_replica_gravity.argtypes = [C.c_void_p, C.c_void_p]
        _lib.pbd_set_replica_rest_positions.argtypes = [C.c_void_p, C.c_void_p]
        _lib.pbd_get_replica_geometry.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib.pbd_set_attr_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_get_attr_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib.pbd_set_masses_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_set_external_forces.argtypes = [C.c_void_p, C.c_void_p]
        _lib.pbd_set_external_forces_device.argtypes = [C.c_void_p] * 4
        _lib.pbd_set_replica_constraint_materials.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib.pbd_set_replica_constraint_materials_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.pbd_get_replica_materials.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib.pbd_set_replica_rigid_bodies.argtypes = [C.c_void_p, C.c_uint] + [C.c_void_p] * 6
        _lib.pbd_set_rigid_bodies_device.argtypes = [C.c_void_p] * 9
        _lib.pbd_get_rigid_bodies_device.argtypes = [C.c_void_p] * 6
        _lib.pbd_set_replica_collider_poses_device.argtypes = [C.c_void_p] * 7
        _lib.pbd_sense_contacts.argtypes = [C.c_void_p, C.c_int]
        _lib.pbd_get_contact_sensors.argtypes = [C.c_void_p] * 3
        _lib.pbd_get_contact_sensors_device.argtypes = [C.c_void_p] * 4
    return _lib


def _ck(rc):
    if rc != 0:
        raise PbdError(lib().pbd_last_error().decode())


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _device_ptr(what, a, typestrs, count, writable=False):
    """The device pointer of `a`, an object with __cuda_array_interface__ (a torch CUDA tensor, a CuPy array), after the checks the C
    calls cannot make: element type one of `typestrs`, C-contiguous, `count` elements, and not read-only where it is written."""
    iface = getattr(a, "__cuda_array_interface__", None)
    if iface is None:
        raise TypeError("%s: wants device memory, an object with __cuda_array_interface__ (a torch CUDA tensor, a CuPy array), got %s; "
                        "host arrays go through the host calls" % (what, type(a).__name__))
    if iface["typestr"] not in typestrs:
        raise ValueError("%s: element type %s, wants %s" % (what, iface["typestr"], " or ".join(typestrs)))
    shape, strides = tuple(iface["shape"]), iface.get("strides")
    if strides is not None:
        step = int(iface["typestr"][2:])
        for extent, stride in reversed(list(zip(shape, strides))):
            if extent != 1 and stride != step:
                raise ValueError("%s: not C-contiguous (shape %s, strides %s)" % (what, shape, tuple(strides)))
            step *= extent
    size = int(np.prod(shape, dtype=np.int64))
    if size != count:
        raise ValueError("%s: %d elements (shape %s), wants %d" % (what, size, shape, count))
    ptr, readonly = iface["data"]
    if writable and readonly:
        raise ValueError("%s: read-only" % what)
    return ptr


def _stream(stream):
    """A stream handle for the device calls: None = the engine's stream; 0, what torch reports for the legacy default stream, becomes
    cudaStreamLegacy (a NULL handle would mean the engine's stream)."""
    if stream is None:
        return None
    return C.c_void_p(int(stream) or 1)


def _host_materials(what, a, shape, writable=False):
    """The checks in front of the host calls of per-constraint replica materials: a float32 numpy array of exactly `shape`, C-contiguous (and
    writable where it is written).  Nothing is converted: a copy in another type or order would hide a caller's mistake in the layout."""
    if not isinstance(a, np.ndarray):
        raise TypeError("%s: wants a numpy array, got %s (device arrays go through set_replica_constraint_materials_device)" % (what, type(a).__name__))
    if a.dtype != np.float32:
        raise ValueError("%s: element type %s, wants float32" % (what, a.dtype))
    if a.shape != tuple(shape):
        raise ValueError("%s: shape %s, wants %s (replicas, constraints, material parameters)" % (what, a.shape, tuple(shape)))
    if not a.flags.c_contiguous:
        raise ValueError("%s: not C-contiguous" % what)
    if writable and not a.flags.writeable:
        raise ValueError("%s: read-only" % what)
    return a


def device_count():
    n = C.c_int(0)
    rc = lib().pbd_device_count(C.byref(n))
    return n.value if rc == 0 else 0


def num_bodies(t):
    return lib().pbd_num_bodies(t)


def num_params(t):
    return lib().pbd_num_params(t)


def num_materials(t):
    """How many of type t's parameters are material parameters (include/pbd_b200.h); what a row of set_replica_materials holds."""
    return lib().pbd_num_materials(t)


def num_geometry(t):
    """How many of type t's parameters are rest geometry (every column that is not a material parameter); a row of replica_geometry."""
    return lib().pbd_num_params(t) - lib().pbd_num_materials(t)


class Engine:
    """One engine <-> one CUDA device + one stream (pbd_create / pbd_destroy).

    A replica batch (set_replicas(K), K > 1) steps K independent copies of the model's state at once: the particle state calls then
    take and return (K, n, 3) / (K, n) arrays and lambdas() (K, count); at K = 1 the shapes are those of one scene.  The replicas share
    the model's parameters, gravity and rest geometry unless set_replica_materials / set_replica_gravity / set_replica_rest_positions
    give each its own; set_replica_colliders gives each replica its own static colliders, set_replica_rigid_bodies its own rigid bodies
    (get_rigid_bodies then returns (K, n, 13))."""

    def __init__(self, device=0, stream=None):
        self._h = C.c_void_p()
        _ck(lib().pbd_create(int(device), C.c_void_p(stream) if stream else None, C.byref(self._h)))
        self.n = 0
        self.K = 1
        self._nc = 0  # constraints added so far (sizes the buffer of groups())
        self.n_rigid_colliders = 0  # rigid colliders per replica in force (sizes the contact sensors)
        self._replica_colliders = False

    def _batch_shape(self, *tail):
        return ((self.K,) if self.K > 1 else ()) + (self.n,) + tail

    def close(self):
        if self._h:
            lib().pbd_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # particles -------------------------------------------------------------------------------------
    def set_particles(self, x, mass, x0=None, v=None):
        x = _f32(x).reshape(-1, 3); mass = _f32(mass).reshape(-1)
        x0 = _f32(x0).reshape(-1, 3) if x0 is not None else None
        v = _f32(v).reshape(-1, 3) if v is not None else None
        self.n = len(x)
        _ck(lib().pbd_set_particles(self._h, self.n, _ptr(x), _ptr(x0), _ptr(v), _ptr(mass)))

    def set_attr(self, attr, a):
        a = _f32(a).reshape(-1, 3); assert len(a) == self.K * self.n
        _ck(lib().pbd_set_attr(self._h, attr, _ptr(a)))

    def get_attr(self, attr=ATTR_X, out=None):
        if out is None:
            out = np.empty(self._batch_shape(3), dtype=np.float32)
        _ck(lib().pbd_get_attr(self._h, attr, _ptr(out)))
        return out

    def set_masses(self, mass):
        mass = _f32(mass).reshape(-1); assert len(mass) == self.K * self.n
        _ck(lib().pbd_set_masses(self._h, _ptr(mass)))

    # particle state in device memory ----------------------------------------------------------------
    # The arrays are objects with __cuda_array_interface__ on the engine's device (torch CUDA tensors, CuPy arrays), float32,
    # C-contiguous, laid out as the host calls' arrays: K*n*3 elements (K*n masses), replica after replica.  stream: an integer stream
    # handle (torch.cuda.current_stream().cuda_stream; 0 = the legacy default stream) or None for the engine's stream.  The copy is
    # ordered after the work enqueued so far on `stream` and before the work enqueued on it later; nothing blocks the host.
    # replicas: None for every replica, or K bools / uint8 in device memory, nonzero where the replica is written.
    def _mask(self, what, replicas):
        return None if replicas is None else C.c_void_p(_device_ptr(what + ": replicas", replicas, ("|b1", "|u1"), self.K))

    def set_attr_device(self, attr, src, replicas=None, stream=None):
        """pbd_set_attr_device: attribute `attr` of the replicas in `replicas` from src (K*n*3 floats)."""
        p = _device_ptr("set_attr_device: src", src, ("<f4",), self.K * self.n * 3)
        mask = self._mask("set_attr_device", replicas)
        if self.K * self.n:
            _ck(lib().pbd_set_attr_device(self._h, int(attr), C.c_void_p(p), mask, _stream(stream)))

    def get_attr_device(self, attr, out, stream=None):
        """pbd_get_attr_device: attribute `attr` of every replica into out (K*n*3 floats); returns out."""
        p = _device_ptr("get_attr_device: out", out, ("<f4",), self.K * self.n * 3, writable=True)
        if self.K * self.n:
            _ck(lib().pbd_get_attr_device(self._h, int(attr), C.c_void_p(p), _stream(stream)))
        return out

    def set_masses_device(self, mass, replicas=None, stream=None):
        """pbd_set_masses_device: the masses of the replicas in `replicas` from mass (K*n floats)."""
        p = _device_ptr("set_masses_device: mass", mass, ("<f4",), self.K * self.n)
        mask = self._mask("set_masses_device", replicas)
        if self.K * self.n:
            _ck(lib().pbd_set_masses_device(self._h, C.c_void_p(p), mask, _stream(stream)))

    # external forces -------------------------------------------------------------------------------
    # Particle i of replica r integrates with a = g_r + f[r, i] * w (w its inverse mass at that time) in every substep until the forces are
    # replaced or cleared; a particle with mass 0 ignores its force.  set_particles and set_replicas clear them.
    def set_external_forces(self, f):
        """pbd_set_external_forces: f, a float32 numpy array (K, n, 3) -- (n, 3) at K = 1 -- C-contiguous, in newtons; None clears every
        force.  Nothing is converted: a copy in another type or order would hide a caller's mistake in the layout."""
        if f is not None:
            if not isinstance(f, np.ndarray):
                raise TypeError("set_external_forces: wants a numpy array, got %s (device arrays go through set_external_forces_device)"
                                % type(f).__name__)
            if f.dtype != np.float32:
                raise ValueError("set_external_forces: element type %s, wants float32" % f.dtype)
            if f.shape != self._batch_shape(3):
                raise ValueError("set_external_forces: shape %s, wants %s" % (f.shape, self._batch_shape(3)))
            if not f.flags.c_contiguous:
                raise ValueError("set_external_forces: not C-contiguous")
            if not f.size:
                return
        _ck(lib().pbd_set_external_forces(self._h, _ptr(f)))

    def set_external_forces_device(self, f, replicas=None, stream=None):
        """pbd_set_external_forces_device: the forces of the replicas in `replicas` from f (K*n*3 floats, the layout of
        set_external_forces); stream and replicas as in set_attr_device.  Replicas left out keep their forces (zero after a clear)."""
        if f is None:
            raise TypeError("set_external_forces_device: f is None; forces are cleared with set_external_forces(None)")
        p = _device_ptr("set_external_forces_device: f", f, ("<f4",), self.K * self.n * 3)
        mask = self._mask("set_external_forces_device", replicas)
        if self.K * self.n:
            _ck(lib().pbd_set_external_forces_device(self._h, C.c_void_p(p), mask, _stream(stream)))

    # replica batch ---------------------------------------------------------------------------------
    def set_replicas(self, k):
        """K copies of replica 0's current state (x, v, x0, oldX, lastX, masses), multipliers zero; the image is re-planned."""
        _ck(lib().pbd_set_replicas(self._h, int(k)))
        self.K = int(k)
        if self._replica_colliders:  # dropped with the old K
            self.n_rigid_colliders, self._replica_colliders = 0, False

    def replicas(self):
        k = C.c_uint(0)
        _ck(lib().pbd_get_replicas(self._h, C.byref(k)))
        return k.value

    def set_replica_materials(self, ctype, mat):
        """Replica r's constraints of `ctype` all carry the material parameters mat[r] ((K, num_materials(ctype)) array); None: the
        shared parameters again.  K > 1 only."""
        if mat is not None:
            mat = _f32(mat)
            if mat.shape != (self.K, num_materials(ctype)):
                raise ValueError("set_replica_materials: type %d wants a (%d, %d) array, got %s" % (ctype, self.K, num_materials(ctype), mat.shape))
        _ck(lib().pbd_set_replica_materials(self._h, int(ctype), _ptr(mat)))

    def _constraint_materials_shape(self, ctype):
        return (self.K, self.stats().constraints_per_type[ctype], num_materials(ctype))

    def set_replica_constraint_materials(self, ctype, mat):
        """Replica r's constraint i of `ctype` (in the order the constraints were added) carries the material parameters mat[r, i]
        ((K, count, num_materials(ctype)) float32 numpy array, C-contiguous); None: the shared parameters again.  K > 1 only."""
        if mat is not None:
            _host_materials("set_replica_constraint_materials", mat, self._constraint_materials_shape(ctype))
        _ck(lib().pbd_set_replica_constraint_materials(self._h, int(ctype), _ptr(mat)))

    def set_replica_constraint_materials_device(self, ctype, mat, replicas=None, stream=None):
        """pbd_set_replica_constraint_materials_device: the per-constraint materials of the replicas in `replicas` from mat, an object with
        __cuda_array_interface__ holding K*count*num_materials(ctype) float32 in that layout (C-contiguous, any shape of that size); stream
        and replicas as in set_attr_device.  Nothing blocks the host once the override is on."""
        if mat is None:
            raise TypeError("set_replica_constraint_materials_device: mat is None; the shared parameters come back with "
                            "set_replica_constraint_materials(ctype, None)")
        p = _device_ptr("set_replica_constraint_materials_device: mat", mat, ("<f4",), int(np.prod(self._constraint_materials_shape(ctype))))
        mask = self._mask("set_replica_constraint_materials_device", replicas)
        _ck(lib().pbd_set_replica_constraint_materials_device(self._h, int(ctype), C.c_void_p(p), mask, _stream(stream)))

    def get_replica_materials(self, ctype, out=None):
        """(K, count, num_materials(ctype)): the material parameters every replica's constraints of `ctype` are stepped with (shared, rows of
        set_replica_materials or per constraint), constraints in the order they were added; into `out` if given (float32, C-contiguous,
        writable, that shape)."""
        shape = self._constraint_materials_shape(ctype)
        if out is None:
            out = np.zeros(shape, dtype=np.float32)
        else:
            _host_materials("get_replica_materials: out", out, shape, writable=True)
        if out.size:
            _ck(lib().pbd_get_replica_materials(self._h, int(ctype), _ptr(out)))
        return out

    def set_replica_gravity(self, g):
        """Replica r integrates with gravity g[r] ((K, 3) array); None: the vector of set_params again.  K > 1 only."""
        if g is not None:
            g = _f32(g)
            if g.shape != (self.K, 3):
                raise ValueError("set_replica_gravity: wants a (%d, 3) array, got %s" % (self.K, g.shape))
        _ck(lib().pbd_set_replica_gravity(self._h, _ptr(g)))

    def set_replica_rest_positions(self, x0):
        """Replica r's constraints get the rest geometry derived from its own rest positions x0[r] ((K, n, 3) array), which also become
        its x0; None: the shared geometry again.  K > 1 only; refused, with nothing changed, when a replica's rest shape makes a
        constraint degenerate."""
        if x0 is not None:
            x0 = _f32(x0)
            if x0.shape != (self.K, self.n, 3):
                raise ValueError("set_replica_rest_positions: wants a (%d, %d, 3) array, got %s" % (self.K, self.n, x0.shape))
        _ck(lib().pbd_set_replica_rest_positions(self._h, _ptr(x0)))

    def replica_geometry(self, ctype):
        """(K, count, num_geometry(ctype)): the geometry columns every replica's constraints of `ctype` are stepped with, constraints in
        the order they were added."""
        cnt = self.stats().constraints_per_type[ctype]
        out = np.zeros((self.K, cnt, num_geometry(ctype)), dtype=np.float32)
        if out.size:
            _ck(lib().pbd_get_replica_geometry(self._h, int(ctype), _ptr(out)))
        return out

    # rigid bodies ----------------------------------------------------------------------------------
    def set_rigid_bodies(self, mass, x, q, inertia, v=None, omega=None):
        """q rows = (w, x, y, z); inertia rows = principal moments."""
        mass = _f32(mass).reshape(-1); self.n_rb = len(mass)
        x = _f32(x).reshape(-1, 3); q = _f32(q).reshape(-1, 4); inertia = _f32(inertia).reshape(-1, 3)
        v = _f32(v).reshape(-1, 3) if v is not None else None
        omega = _f32(omega).reshape(-1, 3) if omega is not None else None
        _ck(lib().pbd_set_rigid_bodies(self._h, self.n_rb, _ptr(mass), _ptr(x), _ptr(q), _ptr(inertia), _ptr(v), _ptr(omega)))

    def set_replica_rigid_bodies(self, mass, x, q, inertia, v=None, omega=None):
        """pbd_set_replica_rigid_bodies: n bodies per replica, replica r's from row r of mass (K, n), x (K, n, 3), q (K, n, 4) as (w, x, y, z),
        inertia (K, n, 3) principal moments, v / omega (K, n, 3) or None (= 0).  Joints index a replica's bodies 0 .. n-1.  K > 1 only."""
        mass = _f32(mass)
        if mass.ndim != 2 or mass.shape[0] != self.K:
            raise ValueError("set_replica_rigid_bodies: mass wants a (%d, n) array, got %s" % (self.K, mass.shape))
        n = mass.shape[1]
        arrays = []
        for name, a, width in (("x", x, 3), ("q", q, 4), ("inertia", inertia, 3), ("v", v, 3), ("omega", omega, 3)):
            if a is not None:
                a = _f32(a)
                if a.shape != (self.K, n, width):
                    raise ValueError("set_replica_rigid_bodies: %s wants a (%d, %d, %d) array, got %s" % (name, self.K, n, width, a.shape))
            arrays.append(a)
        _ck(lib().pbd_set_replica_rigid_bodies(self._h, n, _ptr(mass), *[_ptr(a) for a in arrays]))
        self.n_rb = n

    def get_rigid_bodies(self):
        """[n, 13], or (K, n, 13) for a batch: x(3) q(w,x,y,z) v(3) omega(3)."""
        n = getattr(self, "n_rb", 0)
        rows = self.K * n
        x = np.zeros((max(rows, 1), 3), np.float32); q = np.zeros((max(rows, 1), 4), np.float32)
        v = np.zeros((max(rows, 1), 3), np.float32); w = np.zeros((max(rows, 1), 3), np.float32)
        _ck(lib().pbd_get_rigid_bodies(self._h, _ptr(x), _ptr(q), _ptr(v), _ptr(w)))
        out = np.concatenate([x, q, v, w], axis=1)[:rows]
        return out.reshape(self.K, n, 13) if self.K > 1 else out

    # rigid-body state in device memory: the layouts of the host calls (K*n rows, replica after replica; q as (w, x, y, z)), as objects
    # with __cuda_array_interface__; stream and replicas as in set_attr_device.
    def set_rigid_bodies_device(self, x, q, v=None, omega=None, mass=None, inertia=None, replicas=None, stream=None):
        """pbd_set_rigid_bodies_device: the bodies of the replicas in `replicas` from x (K*n*3 floats) and q (K*n*4); v / omega None = 0;
        mass (K*n) / inertia (K*n*3) None = each body keeps its own.  Old and last state become the new current state."""
        rows = self.K * getattr(self, "n_rb", 0)
        ptrs = [C.c_void_p(_device_ptr("set_rigid_bodies_device: " + name, a, ("<f4",), rows * width)) if a is not None else None
                for name, a, width in (("mass", mass, 1), ("x", x, 3), ("q", q, 4), ("inertia", inertia, 3), ("v", v, 3), ("omega", omega, 3))]
        if ptrs[1] is None or ptrs[2] is None:
            raise TypeError("set_rigid_bodies_device: x and q are required")
        mask = self._mask("set_rigid_bodies_device", replicas)
        _ck(lib().pbd_set_rigid_bodies_device(self._h, *ptrs, mask, _stream(stream)))

    def get_rigid_bodies_device(self, x=None, q=None, v=None, omega=None, stream=None):
        """pbd_get_rigid_bodies_device: every replica's bodies into x (K*n*3 floats), q (K*n*4, (w, x, y, z)), v, omega (K*n*3); any may be
        None.  Returns (x, q, v, omega)."""
        rows = self.K * getattr(self, "n_rb", 0)
        ptrs = [C.c_void_p(_device_ptr("get_rigid_bodies_device: " + name, a, ("<f4",), rows * width, writable=True)) if a is not None else None
                for name, a, width in (("x", x, 3), ("q", q, 4), ("v", v, 3), ("omega", omega, 3))]
        _ck(lib().pbd_get_rigid_bodies_device(self._h, *ptrs, _stream(stream)))
        return x, q, v, omega

    # constraints -----------------------------------------------------------------------------------
    def clear_constraints(self):
        _ck(lib().pbd_clear_constraints(self._h))
        self._nc = 0

    def add_constraints(self, ctype, bodies, params, ids=None):
        nb, npar = num_bodies(ctype), num_params(ctype)
        bodies = np.ascontiguousarray(bodies, dtype=np.uint32).reshape(-1, nb)
        params = _f32(params).reshape(-1, npar)
        assert len(bodies) == len(params)
        ids = np.ascontiguousarray(ids, dtype=np.uint32) if ids is not None else None
        _ck(lib().pbd_add_constraints(self._h, ctype, len(bodies), _ptr(bodies), _ptr(params), _ptr(ids)))
        self._nc += len(bodies)

    def add_flat(self, types, bodies, params):
        """Insert a whole flat constraint list (types[n], bodies[n,4], params[n,24]) keeping insertion ids."""
        types = np.asarray(types)
        for t in range(NUM_TYPES):
            sel = np.nonzero(types == t)[0]
            if len(sel):
                self.add_constraints(t, np.asarray(bodies)[sel][:, :num_bodies(t)], np.asarray(params)[sel][:, :num_params(t)],
                                     ids=sel.astype(np.uint32))

    def set_groups(self, offsets, ids):
        offsets = np.ascontiguousarray(offsets, dtype=np.uint32); ids = np.ascontiguousarray(ids, dtype=np.uint32)
        _ck(lib().pbd_set_groups(self._h, len(offsets) - 1, _ptr(offsets), _ptr(ids)))

    def color_first_fit(self):
        _ck(lib().pbd_color_first_fit(self._h))

    def color_first_fit_device(self):
        """Exact first-fit colouring on the GPU; returns (device ms, wavefronts)."""
        ms = C.c_float(0.0); wf = C.c_uint(0)
        _ck(lib().pbd_color_first_fit_device(self._h, C.byref(ms), C.byref(wf)))
        return ms.value, wf.value

    def groups(self):
        ng = C.c_uint(0)
        _ck(lib().pbd_get_num_groups(self._h, C.byref(ng)))
        off = np.zeros(ng.value + 1, dtype=np.uint32)
        ids = np.zeros(max(self._nc, 1), dtype=np.uint32)  # the groups partition all constraints added so far
        _ck(lib().pbd_get_groups(self._h, _ptr(off), _ptr(ids)))
        return off, ids[:off[-1]]

    # parameters / stepping -------------------------------------------------------------------------
    def set_params(self, dt=0.005, sub_steps=5, max_iter=1, vel_method=0, gravity=(0.0, -9.81, 0.0)):
        g = _f32(gravity)
        _ck(lib().pbd_set_params(self._h, float(dt), int(sub_steps), int(max_iter), int(vel_method), _ptr(g)))

    def set_mode(self, mode):
        _ck(lib().pbd_set_mode(self._h, int(mode)))

    def get_mode(self):
        """(requested, active): active is what the next step runs in (the resolution of MODE_AUTO for the current model)."""
        r, a = C.c_int(0), C.c_int(0)
        _ck(lib().pbd_get_mode(self._h, C.byref(r), C.byref(a)))
        return r.value, a.value

    def step(self, n=1):
        _ck(lib().pbd_step(self._h, int(n)))

    def sync(self):
        _ck(lib().pbd_sync(self._h))

    def step_host(self, n, x_in, v_in, x_out, v_out=None):
        """Host arrays of K * n * 3 floats (replica after replica), or None."""
        _ck(lib().pbd_step_host(self._h, int(n), _ptr(x_in), _ptr(v_in), _ptr(x_out), _ptr(v_out)))

    def step_host_async(self, n, x_in, v_in, x_out, v_out=None):
        """pbd_step_host_async: enqueue only; the arrays belong to the engine until step_host_wait covers the call."""
        _ck(lib().pbd_step_host_async(self._h, int(n), _ptr(x_in), _ptr(v_in), _ptr(x_out), _ptr(v_out)))

    def step_host_wait(self, lag=0):
        _ck(lib().pbd_step_host_wait(self._h, int(lag)))

    def set_colliders(self, particle_colliders, rigid_colliders):
        """pbd_set_colliders: lists of ParticleCollider / RigidCollider (rigid ones in the order of the reference's collision object list)."""
        pa = (ParticleCollider * max(len(particle_colliders), 1))(*particle_colliders)
        ra = (RigidCollider * max(len(rigid_colliders), 1))(*rigid_colliders)
        _ck(lib().pbd_set_colliders(self._h, len(particle_colliders), C.cast(pa, C.c_void_p), len(rigid_colliders), C.cast(ra, C.c_void_p)))
        self.n_rigid_colliders, self._replica_colliders = len(rigid_colliders), False

    def set_replica_colliders(self, particle_colliders, rigid_colliders, body_x=None, body_v=None, body_omega=None):
        """pbd_set_replica_colliders: every replica against its own static colliders.  particle_colliders: ParticleCollider ranges of
        one replica's particles, shared by all; rigid_colliders: K lists of nR RigidCollider, one per replica; body_x / body_v / body_omega:
        (K, nR, 3) centre of mass, velocity and angular velocity of the static body carrying each collider (v, omega: None = 0).
        rigid_colliders None: no contacts.  K > 1 only."""
        if rigid_colliders is None:
            _ck(lib().pbd_set_replica_colliders(self._h, 0, None, 0, None, None, None, None))
            self.n_rigid_colliders, self._replica_colliders = 0, False
            return
        if len(rigid_colliders) != self.K or len(set(len(r) for r in rigid_colliders)) > 1:
            raise ValueError("set_replica_colliders: wants %d lists of the same number of rigid colliders, got %s" % (self.K, [len(r) for r in rigid_colliders]))
        nr = len(rigid_colliders[0]) if len(rigid_colliders) else 0
        flat = [c for r in rigid_colliders for c in r]
        arrays = []
        for name, a in (("body_x", body_x), ("body_v", body_v), ("body_omega", body_omega)):
            if a is not None:
                a = _f32(a)
                if a.shape != (self.K, nr, 3):
                    raise ValueError("set_replica_colliders: %s wants a (%d, %d, 3) array, got %s" % (name, self.K, nr, a.shape))
            arrays.append(a)
        pa = (ParticleCollider * max(len(particle_colliders), 1))(*particle_colliders)
        ra = (RigidCollider * max(len(flat), 1))(*flat)
        _ck(lib().pbd_set_replica_colliders(self._h, len(particle_colliders), C.cast(pa, C.c_void_p), nr, C.cast(ra, C.c_void_p), *[_ptr(a) for a in arrays]))
        self.n_rigid_colliders, self._replica_colliders = nr, nr > 0

    def set_replica_collider_poses_device(self, pose, body_x, body_v=None, body_omega=None, replicas=None, stream=None):
        """pbd_set_replica_collider_poses_device: move the replica colliders of set_replica_colliders from device memory.  pose: K*nR*21
        float32, each row R[9], v1[3], v2[3], aabb_min[3], aabb_max[3] of a RigidCollider; body_x (required), body_v, body_omega: K*nR*3
        float32 (v, omega None = 0).  Objects with __cuda_array_interface__; stream and replicas as in set_attr_device.  Everything else
        about the colliders stays as set_replica_colliders left it."""
        rows = self.K * self.n_rigid_colliders
        p = _device_ptr("set_replica_collider_poses_device: pose", pose, ("<f4",), rows * 21)
        ptrs = [C.c_void_p(_device_ptr("set_replica_collider_poses_device: " + name, a, ("<f4",), rows * 3)) if a is not None else None
                for name, a in (("body_x", body_x), ("body_v", body_v), ("body_omega", body_omega))]
        if ptrs[0] is None:
            raise TypeError("set_replica_collider_poses_device: body_x is required")
        mask = self._mask("set_replica_collider_poses_device", replicas)
        _ck(lib().pbd_set_replica_collider_poses_device(self._h, C.c_void_p(p), *ptrs, mask, _stream(stream)))

    # contact sensors: per replica and rigid collider, the contacts found and the impulse received (mass x velocity) in the last step
    def sense_contacts(self, on=True):
        """pbd_sense_contacts: switch the contact sensors on or off (off by default)."""
        _ck(lib().pbd_sense_contacts(self._h, int(bool(on))))

    def contact_sensors(self):
        """pbd_get_contact_sensors: (counts (K, nR) uint32, impulses (K, nR, 3) float32) of the last step; synchronises."""
        count = np.zeros((self.K, self.n_rigid_colliders), np.uint32)
        impulse = np.zeros((self.K, self.n_rigid_colliders, 3), np.float32)
        _ck(lib().pbd_get_contact_sensors(self._h, _ptr(count), _ptr(impulse)))
        return count, impulse

    def get_contact_sensors_device(self, count=None, impulse=None, stream=None):
        """pbd_get_contact_sensors_device: the sensors into count (K*nR uint32) and impulse (K*nR*3 float32), objects with
        __cuda_array_interface__, writable; either may be None.  Stream as in get_attr_device.  Returns (count, impulse)."""
        rows = self.K * self.n_rigid_colliders
        pc = C.c_void_p(_device_ptr("get_contact_sensors_device: count", count, ("<u4",), rows, writable=True)) if count is not None else None
        pi = C.c_void_p(_device_ptr("get_contact_sensors_device: impulse", impulse, ("<f4",), rows * 3, writable=True)) if impulse is not None else None
        _ck(lib().pbd_get_contact_sensors_device(self._h, pc, pi, _stream(stream)))
        return count, impulse

    def set_contact_params(self, tolerance=0.01, stiffness=100.0, max_iter_v=5):
        _ck(lib().pbd_set_contact_params(self._h, float(tolerance), float(stiffness), int(max_iter_v)))

    def record_contacts(self, capacity):
        _ck(lib().pbd_record_contacts(self._h, int(capacity)))

    def contacts(self, capacity=1 << 16):
        buf = (Contact * capacity)(); cnt = C.c_uint(0)
        _ck(lib().pbd_get_contacts(self._h, C.cast(buf, C.c_void_p), capacity, C.byref(cnt)))
        return [buf[i] for i in range(min(cnt.value, capacity))], cnt.value

    def lambdas(self, ctype):
        """(multipliers, insertion ids): multipliers (count,), or (K, count) for a batch."""
        cnt = self.stats().constraints_per_type[ctype]
        lam = np.zeros(max(self.K * cnt, 1), dtype=np.float32); ids = np.zeros(max(cnt, 1), dtype=np.uint32)
        _ck(lib().pbd_get_lambdas(self._h, ctype, _ptr(lam), _ptr(ids)))
        lam = lam[:self.K * cnt]
        return (lam.reshape(self.K, cnt) if self.K > 1 else lam), ids[:cnt]

    def stats(self, flatten=True):
        s = Stats()
        _ck(lib().pbd_get_stats(self._h, C.byref(s)))
        return s

    def profile_step(self):
        ms = np.zeros(NUM_TYPES, dtype=np.float32); launches = np.zeros(NUM_TYPES, dtype=np.uint32)
        mi = C.c_float(0); mv = C.c_float(0)
        _ck(lib().pbd_profile_step(self._h, _ptr(ms), C.byref(mi), C.byref(mv), _ptr(launches)))
        return ms, mi.value, mv.value, launches
