"""The fp64 checker of external forces (pbd_set_external_forces): the C restatement with a per-particle external acceleration,
tests/oracle_ext/external_accel.c.  That file compiles oracle/pbd_oracle.c unmodified and adds orc_set_ext_accel / orc_step_ext, whose
clearAccelerations sets a[i] = gravity + ext[i] for every particle with mass while an acceleration is set; the engine's dt and subSteps,
the rigid bodies and the contact step run as in orc_step.  It is compiled once per process, with oracle/Makefile's flags, into a
temporary directory."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCE = os.path.join(HERE, "oracle_ext", "external_accel.c")
CFLAGS = ["-O2", "-march=x86-64-v3", "-std=c11", "-fPIC", "-Wall", "-Wno-unused-function", "-fopenmp"]  # oracle/Makefile's CFLAGS
_built = {}


def library(precision):
    """Path of the restatement with external accelerations in `precision` ("f32" | "f64"), built on first use."""
    if precision not in _built:
        where = tempfile.mkdtemp(prefix="pbd_oracle_ext_")
        atexit.register(shutil.rmtree, where, True)
        out = os.path.join(where, "liboracle_ext_%s.so" % precision)
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"  # oracle/Makefile's CC
        cmd = [cc] + CFLAGS + (["-DORACLE_DOUBLE"] if precision == "f64" else []) + ["-shared", "-o", out, SOURCE, "-lm"]
        subprocess.check_call(cmd)
        _built[precision] = out
    return _built[precision]


def checker(pyoracle, precision="f64"):
    """A pyoracle.CpuPbd on the restatement with external accelerations: set_ext_accel(a) sets them (None clears), step() steps with them."""
    class CpuPbdExt(pyoracle.CpuPbd):
        def __init__(self):
            super().__init__("oracle", precision, path=library(precision))
            self.lib.orc_step_ext.restype = C.c_double
            self.set_ext_accel(None)

        def set_ext_accel(self, a):
            """a: (n, 3) external acceleration of every particle (f / m), or None."""
            if a is None:
                self.lib.orc_set_ext_accel(None)
                return
            a = np.ascontiguousarray(a, dtype=np.float64)
            assert a.shape == (self.num_particles(), 3)
            self.lib.orc_set_ext_accel(a.ctypes.data_as(C.c_void_p))

        def step(self, n=1):
            return self.lib.orc_step_ext(int(n))

    return CpuPbdExt()


def ext_acceleration(f, mass):
    """The external acceleration f / m of every particle in fp64 (0 where the mass is 0, which the integration skips anyway)."""
    f = np.asarray(f, np.float64)
    m = np.asarray(mass, np.float64)
    out = np.zeros_like(f)
    moving = m != 0.0
    out[moving] = f[moving] / m[moving][:, None]
    return out
