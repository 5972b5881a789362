"""TEST INFRASTRUCTURE ONLY -- Python access to the CPU instantiation of the device arithmetic
(tests/hostcheck/hostcheck.cpp: olb_math.cuh + olb_prep.h compiled by g++).  Used by the CPU tests,
by the test-only oracle engine of the Optiland plugin tests and by the reference-test sweep.  Never
imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from optiland_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck.so")
CSRC = os.path.join(ROOT, "optiland_b200", "csrc")
REC = ("x", "y", "z", "L", "M", "N", "intensity", "opd")
_lib_cache = None


def load():
    """Build (if stale) and load the host-check library."""
    global _lib_cache
    if _lib_cache is not None:
        return _lib_cache
    deps = [SRC, os.path.join(CSRC, "olb_math.cuh"), os.path.join(CSRC, "olb_prep.h"), os.path.join(CSRC, "olb_fftpsf.cuh")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])
    _lib_cache = C.CDLL(SO)
    return _lib_cache

def run_hostcheck(hc, table, rays, dtype, first=0, last=None, want_l0=False, pmat=None):
    last = table.num_surfaces if last is None else last
    ht = _lib.HostTable(table)
    n = rays["x"].size
    keys = ("x", "y", "z", "L", "M", "N", "i", "w", "opd")
    arrs = [np.ascontiguousarray(rays.get(k, np.zeros(n)), dtype=dtype).copy() for k in keys]
    rows = last - first
    rec = [np.full((rows, n), np.nan, dtype=dtype) for _ in range(8)]
    l0 = [np.zeros(n, dtype=dtype) for _ in range(3)]
    PP = C.c_void_p * 9
    ray_ptrs = PP(*[a.ctypes.data for a in arrs])
    rec_ptrs = (C.c_void_p * 8)(*[a.ctypes.data for a in rec])
    l0_ptrs = (C.c_void_p * 3)(*[a.ctypes.data for a in l0])
    status = C.c_int(0)
    err = C.create_string_buffer(256)
    fn = hc.olbhc_trace_f64 if dtype == np.float64 else hc.olbhc_trace_f32
    fn.restype = C.c_int
    parr = None
    if pmat is not None:
        cdt = np.complex128 if dtype == np.float64 else np.complex64
        parr = np.ascontiguousarray(pmat, dtype=cdt).copy()
    rc = fn(C.byref(ht.c), C.c_int(first), C.c_int(last), C.c_int64(n), ray_ptrs, rec_ptrs,
            l0_ptrs if want_l0 else None, C.c_void_p(parr.ctypes.data) if parr is not None else None,
            C.byref(status), err, 256)
    assert rc == 0, err.value
    out = dict(zip(keys, arrs))
    if parr is not None:
        out["p"] = parr
    out.update(L0=l0[0], M0=l0[1], N0=l0[2])
    return out, dict(zip(REC, rec)), status.value


def run_backward(hc, table, rays, rec, grec, dtype=np.float64, tables=False, first=0, last=None):
    """The adjoint over surfaces [first, last): ``rays`` is the state in front of surface ``first``, ``rec`` / ``grec``
    hold rows first .. last-1 (row 0 = surface ``first``); gradients come back for every surface of the table."""
    ht = _lib.HostTable(table)
    n = rays["x"].size
    S = table.num_surfaces
    last = S if last is None else last
    keys = ("x", "y", "z", "L", "M", "N", "i", "w", "opd")
    rin = [np.ascontiguousarray(rays.get(k, np.zeros(n)), dtype=dtype) for k in keys]
    recs = [np.ascontiguousarray(rec[k], dtype=dtype) for k in REC]
    grecs = [None if grec.get(k) is None else np.ascontiguousarray(grec[k], dtype=dtype) for k in REC]
    gin = [np.zeros(n, dtype=dtype) for _ in range(8)]
    gpc = hc.olbhc_gp_count()
    gpar = np.zeros((S, gpc), dtype=np.float64)
    P9 = (C.c_void_p * 9)(*[a.ctypes.data for a in rin])
    P8 = lambda arrs: (C.c_void_p * 8)(*[(a.ctypes.data if a is not None else None) for a in arrs])  # noqa: E731
    err = C.create_string_buffer(256)
    if tables:
        gtab = np.zeros((S, 2, 12, 12), dtype=np.float64)
        fn = hc.olbhc_backward_tables_f64 if dtype == np.float64 else hc.olbhc_backward_tables_f32
        rc = fn(C.byref(ht.c), first, last, C.c_int64(n), P9, P8(recs), P8(grecs), P8(gin), C.c_void_p(gpar.ctypes.data),
                C.c_void_p(gtab.ctypes.data), err, 256)
        assert rc == 0, err.value
        return dict(zip(("x", "y", "z", "L", "M", "N", "i", "opd"), gin)), gpar, gtab
    fn = hc.olbhc_backward_f64 if dtype == np.float64 else hc.olbhc_backward_f32
    rc = fn(C.byref(ht.c), first, last, C.c_int64(n), P9, P8(recs), P8(grecs), P8(gin), C.c_void_p(gpar.ctypes.data), err, 256)
    assert rc == 0, err.value
    return dict(zip(("x", "y", "z", "L", "M", "N", "i", "opd"), gin)), gpar




def run_wavefront(hc, fin: dict, Px, Py, ref: dict) -> dict:
    """olb_math.cuh::wavefront_point (the kernel's wavefront epilogue) on the CPU."""
    n = np.size(fin["x"])
    arrs = [np.ascontiguousarray(fin[k], dtype=np.float64) for k in ("x", "y", "z", "L", "M", "N", "opd")]
    px, py = np.ascontiguousarray(Px, dtype=np.float64), np.ascontiguousarray(Py, dtype=np.float64)
    tilt = ref.get("tilt", (0.0, 0.0))
    r = np.array([*ref["center"], ref["radius"], ref["n_image"], tilt[0], tilt[1], ref["opd_ref"],
                  1.0 / (float(ref["wavelength_um"]) * 1e-3)], dtype=np.float64)
    out = [np.empty(n) for _ in range(4)]
    hc.olbhc_wavefront.restype = C.c_int
    rc = hc.olbhc_wavefront(C.c_int64(n), (C.c_void_p * 7)(*[a.ctypes.data for a in arrs]), C.c_void_p(px.ctypes.data),
                            C.c_void_p(py.ctypes.data), C.c_void_p(r.ctypes.data), (C.c_void_p * 4)(*[a.ctypes.data for a in out]))
    assert rc == 0
    return dict(zip(("opd", "pupil_x", "pupil_y", "pupil_z"), out))


def run_pol_intensity(hc, P, k0, i0, state=None):
    """olb_math.cuh::polarized_intensity (the polarized kernels' intensity epilogue) on the CPU.  ``P``: (n, 3, 3)
    complex, ``k0``: (3, n) launch direction, ``state``: None (unpolarized) or (Ex, Ey, phase_x, phase_y)."""
    n = P.shape[0]
    pm = np.ascontiguousarray(P, dtype=np.complex128).view(np.float64).reshape(n, 18)
    kx, ky, kz = (np.ascontiguousarray(v, dtype=np.float64) for v in k0)
    i0 = np.ascontiguousarray(i0, dtype=np.float64)
    out = np.empty(n)
    if state is None:
        mode, ax, ay = 2, np.zeros(2), np.zeros(2)
    else:
        Ex, Ey, phx, phy = state
        mag = np.hypot(Ex, Ey)
        mode = 1
        ax = np.array([Ex / mag * np.cos(phx), Ex / mag * np.sin(phx)])
        ay = np.array([Ey / mag * np.cos(phy), Ey / mag * np.sin(phy)])
    status = C.c_int(0)
    hc.olbhc_pol_intensity.restype = C.c_int
    rc = hc.olbhc_pol_intensity(C.c_int64(n), C.c_void_p(pm.ctypes.data), C.c_void_p(kx.ctypes.data),
                                C.c_void_p(ky.ctypes.data), C.c_void_p(kz.ctypes.data), C.c_void_p(i0.ctypes.data),
                                C.c_int(mode), C.c_void_p(ax.ctypes.data), C.c_void_p(ay.ctypes.data),
                                C.c_void_p(out.ctypes.data), C.byref(status))
    assert rc == 0
    return out, status.value
