"""What the velocity-fix tests share, on the CPU and the GPU: the bounds of DESIGN.md §8d and the host build of the
velocity core (tests/emu/velocity_emu.cu)."""
import ctypes as C

import numpy as np

import velocity_oracle as vo
from hostbuild import host_library

# bounds of DESIGN.md §8d, a small multiple of the spread measured by tests/test_velocity_cpu.py
VEL_MS, DRIFT_SS = 1e-6, 1e-12        # planted recovery
LAT_DEG, HEIGHT_M = 1e-9, 1e-4        # geodetic against the forward formula
DOP_REL = 1e-9                        # DOP and residual RMS against numpy
SV_VEL_MS, SV_DRIFT_SS = 3e-6, 1e-15  # satellite velocity against a central difference, h = 0.1 s


def velocity_emulator():
    """(satellite(params, tow) -> (vx, vy, vz, drift), compute(rows, r, rx) -> VELOCITY_DTYPE record,
    geodetic(x, y, z) -> (lat, lon, h)): the host build of the velocity core."""
    lib = host_library("velocity_emu")
    lib.velocity_emu_satellite.argtypes = [C.c_void_p, C.c_double, C.c_void_p]
    lib.velocity_emu_compute.restype = C.c_int
    lib.velocity_emu_compute.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p]
    lib.velocity_emu_geodetic.argtypes = [C.c_double, C.c_double, C.c_double, C.c_void_p]

    def satellite(params, tow):
        p = np.ascontiguousarray(params, dtype=np.float64)
        out = np.zeros(4)
        lib.velocity_emu_satellite(p.ctypes.data, float(tow), out.ctypes.data)
        return out

    def compute(rows, r, rx=0.0):
        rr = np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, 8)
        out = np.zeros(1, dtype=vo.VELOCITY_DTYPE)
        lib.velocity_emu_compute(rr.ctypes.data, len(rr), float(rx), float(r[0]), float(r[1]), float(r[2]), out.ctypes.data)
        return out[0]

    def geodetic(x, y, z):
        out = np.zeros(3)
        lib.velocity_emu_geodetic(float(x), float(y), float(z), out.ctypes.data)
        return out

    return satellite, compute, geodetic
