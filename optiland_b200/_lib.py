"""ctypes binding of the C ABI in ``include/olb.h`` (libolb.so, built in-tree).

There is no CPU fallback: ``load()`` raises if the shared library is missing or does
not export every symbol the header declares.
"""
from __future__ import annotations

import ctypes as C
import os
from functools import lru_cache

import numpy as np

from . import table as T

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libolb.so")

OK = 0
ERRORS = {-1: "OLB_ERR_INVALID_ARG", -2: "OLB_ERR_UNSUPPORTED", -3: "OLB_ERR_CUDA",
          -4: "OLB_ERR_ALIGNMENT", -5: "OLB_ERR_TABLE"}

TF_POLARIZED = 1 << 0
TF_NO_FINAL = 1 << 1
TF_POL_IDENTITY = 1 << 2
TF_MOMENTS = 1 << 3
TF_SHARED_INPUT = 1 << 4
TF_MOMENTS_GLOBAL = 1 << 5
TF_MOMENTS_ALL = 1 << 6
BP_TX, BP_TY, BP_TZ, BP_R, BP_CURV, BP_CONIC, BP_N1, BP_N2, BP_COEF, BP_MAX_COEF = 0, 1, 2, 3, 12, 13, 14, 15, 16, 12
BP_COUNT = BP_COEF + BP_MAX_COEF
GP_TX, GP_TY, GP_TZ, GP_CURV, GP_CONIC, GP_N1, GP_N2, GP_COEF, GP_MAX_COEF = 0, 1, 2, 3, 4, 5, 6, 7, 12
GP_R = GP_COEF + GP_MAX_COEF      # 9 entries: dLoss/dR of a tilted pose (row-major)
GP_COUNT = GP_R + 9
GT_DIM = 12
GT_PER_SURFACE = 2 * GT_DIM * GT_DIM


class OlbTable(C.Structure):
    _fields_ = [
        ("surfaces", C.c_void_p), ("n_surfaces", C.c_int32), ("n_wl", C.c_int32),
        ("wavelengths", C.c_void_p), ("pool", C.c_void_p), ("pool_len", C.c_int32),
        ("reserved", C.c_int32),
    ]


class OlbRays(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("x", "y", "z", "L", "M", "N", "i", "w", "opd", "L0", "M0", "N0", "p")]


class OlbRecords(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("x", "y", "z", "L", "M", "N", "intensity", "opd")] + [
        ("row_stride", C.c_int64)]


class OlbPupilLaunch(C.Structure):
    _fields_ = [("Px", C.c_void_p), ("Py", C.c_void_p), ("origin0", C.c_double * 3), ("origin_scale", C.c_double * 2),
                ("target0", C.c_double * 3), ("target_scale", C.c_double * 2), ("intensity", C.c_double),
                ("Hx", C.c_void_p), ("Hy", C.c_void_p), ("field_mode", C.c_int32), ("n_vig", C.c_int32),
                ("field_arg", C.c_double), ("origin_field", C.c_double * 2), ("target_field", C.c_double * 2),
                ("vig_power", C.c_int32), ("reserved", C.c_int32), ("vig", (C.c_double * 4) * 16)]


class OlbWavefrontRef(C.Structure):
    _fields_ = [("center", C.c_double * 3), ("radius", C.c_double), ("n_image", C.c_double), ("tilt", C.c_double * 2),
                ("opd_ref", C.c_double), ("wavelength_um", C.c_double)]


class OlbWavefrontOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("opd", "pupil_x", "pupil_y", "pupil_z", "intensity")]


class OlbPolarization(C.Structure):
    _fields_ = [("is_polarized", C.c_int32), ("reserved", C.c_int32), ("Ex", C.c_double), ("Ey", C.c_double),
                ("phase_x", C.c_double), ("phase_y", C.c_double), ("intensity", C.c_void_p)]


class OlbTraceCall(C.Structure):
    _fields_ = [("first", C.c_int32), ("last", C.c_int32), ("n_rays", C.c_int64), ("flags", C.c_uint32),
                ("rng_stream", C.c_uint32), ("rays", C.POINTER(OlbRays)), ("rec", C.POINTER(OlbRecords)),
                ("launch", C.POINTER(OlbPupilLaunch)), ("center", C.c_double * 2), ("moments", C.c_void_p),
                ("rays_per_system", C.c_int64), ("wavefront_ref", C.POINTER(OlbWavefrontRef)),
                ("wavefront_out", C.POINTER(OlbWavefrontOut)), ("pol", C.POINTER(OlbPolarization)),
                ("status", C.c_void_p)]


class OlbAimCall(C.Structure):
    _fields_ = [("first", C.c_int32), ("last", C.c_int32), ("n_rays", C.c_int64), ("rays", C.POINTER(OlbRays)),
                ("Px", C.c_void_p), ("Py", C.c_void_p), ("r_stop", C.c_double), ("J_factor", C.c_double),
                ("tol", C.c_double), ("max_iter", C.c_int32), ("infinite", C.c_int32), ("status", C.c_void_p)]


class OlbIrradiance(C.Structure):
    _fields_ = [("x", C.c_void_p), ("y", C.c_void_p), ("z", C.c_void_p), ("i", C.c_void_p), ("n_rays", C.c_int64),
                ("frame", C.c_int32), ("nx", C.c_int32), ("ny", C.c_int32), ("path", C.c_int32),
                ("t", C.c_double * 3), ("R", C.c_double * 9), ("x_edges", C.c_void_p), ("y_edges", C.c_void_p),
                ("edges", C.c_void_p), ("hist", C.c_void_p)]


IRR_FRAME_TRANSLATE, IRR_FRAME_AFFINE = 0, 1
IRR_PATH_AUTO, IRR_PATH_SHARED, IRR_PATH_GLOBAL = 0, 1, 2


class OlbDeviceTable(C.Structure):
    _fields_ = [
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64), ("magic", C.c_uint32),
        ("features", C.c_uint32), ("n_surfaces", C.c_int32), ("n_wl", C.c_int32),
        ("off_f64", C.c_int32), ("bytes_f64", C.c_int32), ("off_f32", C.c_int32),
        ("bytes_f32", C.c_int32), ("bwd_supported", C.c_int32), ("bwd_slots", C.c_int32),
        ("n_systems", C.c_int32), ("stride_f64", C.c_int32), ("stride_f32", C.c_int32), ("hints", C.c_int32),
    ]


# every symbol include/olb.h declares: name -> (restype, argtypes)
_P = C.POINTER
SYMBOLS = {
    "olb_version": (C.c_int, []),
    "olb_last_error": (C.c_int, [C.c_char_p, C.c_int]),
    "olb_launch_count": (C.c_int64, []),
    "olb_table_workspace_bytes": (C.c_int64, [_P(OlbTable)]),
    "olb_table_upload": (C.c_int, [_P(OlbTable), C.c_void_p, C.c_int64, C.c_void_p, _P(OlbDeviceTable)]),
    "olb_trace_call_f32": (C.c_int, [_P(OlbDeviceTable), _P(OlbTraceCall), C.c_void_p]),
    "olb_trace_call_f64": (C.c_int, [_P(OlbDeviceTable), _P(OlbTraceCall), C.c_void_p]),
    "olb_aim_f32": (C.c_int, [_P(OlbDeviceTable), _P(OlbAimCall), C.c_void_p]),
    "olb_aim_f64": (C.c_int, [_P(OlbDeviceTable), _P(OlbAimCall), C.c_void_p]),
    "olb_trace_bwd_f32": (C.c_int, [_P(OlbDeviceTable), C.c_int32, C.c_int32, _P(OlbRays), _P(OlbRecords),
                                    _P(OlbRecords), _P(OlbRays), C.c_void_p, C.c_void_p, C.c_int64, C.c_uint64,
                                    C.c_void_p]),
    "olb_trace_bwd_f64": (C.c_int, [_P(OlbDeviceTable), C.c_int32, C.c_int32, _P(OlbRays), _P(OlbRecords),
                                    _P(OlbRecords), _P(OlbRays), C.c_void_p, C.c_void_p, C.c_int64, C.c_uint64,
                                    C.c_void_p]),
    "olb_table_batch_workspace_bytes": (C.c_int64, [_P(OlbTable), C.c_int32]),
    "olb_table_upload_batch": (C.c_int, [_P(OlbTable), C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p,
                                         _P(OlbDeviceTable)]),
    "olb_huygens_psf_f64": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_double,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
    "olb_fft_pupil_f64": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "olb_fft_pupil_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "olb_fft_psf_accumulate_f64": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_void_p, C.c_void_p]),
    "olb_fft_psf_accumulate_f32": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_void_p, C.c_void_p]),
    "olb_irradiance_f32": (C.c_int, [_P(OlbIrradiance), C.c_void_p]),
    "olb_irradiance_f64": (C.c_int, [_P(OlbIrradiance), C.c_void_p]),
    "olb_host_scratch_bytes": (C.c_int64, [C.c_int32, C.c_int64]),
    "olb_trace_host_f32": (C.c_int, [_P(OlbDeviceTable), C.c_int32, C.c_int32, _P(OlbPupilLaunch), _P(OlbRays),
                                     _P(OlbRays), _P(OlbRecords), C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
                                     C.c_uint32, C.c_void_p]),
    "olb_trace_host_f64": (C.c_int, [_P(OlbDeviceTable), C.c_int32, C.c_int32, _P(OlbPupilLaunch), _P(OlbRays),
                                     _P(OlbRays), _P(OlbRecords), C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
                                     C.c_uint32, C.c_void_p]),
}


class OlbError(RuntimeError):
    pass


@lru_cache(maxsize=1)
def load() -> C.CDLL:
    """Load libolb.so and bind every declared symbol.  Fails loudly; no fallback."""
    if not os.path.exists(LIB_PATH):
        raise OlbError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  optiland_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the export is missing
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


def last_error() -> str:
    buf = C.create_string_buffer(512)
    load().olb_last_error(buf, len(buf))
    return buf.value.decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != OK:
        raise OlbError(f"{what} failed: {ERRORS.get(rc, rc)}: {last_error()}")


class HostTable:
    """Owns the packed numpy arrays an ``OlbTable`` points into."""

    def __init__(self, tab: T.SurfaceTable, packed=None):
        self.surf, self.pool = packed if packed is not None else tab.pack()
        self.surf = np.ascontiguousarray(self.surf)
        self.pool = np.ascontiguousarray(self.pool)
        self.wl = np.ascontiguousarray(tab.wavelengths, dtype=np.float64)
        self.c = OlbTable(
            surfaces=self.surf.ctypes.data, n_surfaces=len(self.surf), n_wl=len(self.wl),
            wavelengths=self.wl.ctypes.data, pool=self.pool.ctypes.data, pool_len=len(self.pool),
            reserved=0)
