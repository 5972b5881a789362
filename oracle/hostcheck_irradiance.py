"""TEST INFRASTRUCTURE ONLY -- Python access to the host build of the irradiance binning arithmetic
(tests/hostcheck/hostcheck_irradiance.cpp: csrc/olb_irradiance.cuh compiled with g++).  Never imported by the product
package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.hostcheck_api import CSRC, ROOT

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_irradiance.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_irradiance.so")
DEPS = [SRC, os.path.join(CSRC, "olb_irradiance.cuh"), os.path.join(ROOT, "include", "olb.h")]
_cache = None


def build(force: bool = False) -> None:
    """Compile _hostcheck_irradiance.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


def bin_rays(x, y, power, x_edges, y_edges, z=None, frame=None):
    """(bins, hist): the flat bin ``ix * ny + iy`` of every ray (-1 when dropped) and the fp64 ``(nx, ny)`` histogram the
    kernel's arithmetic gives.  ``x / y / z / power``: NumPy arrays of one precision (fp32 or fp64); ``frame``: None
    (no translation), ``("translate", t)`` or ``("affine", t, R)`` as in ``OlbIrradiance``."""
    dt = np.asarray(x).dtype
    if dt not in (np.float32, np.float64):
        raise TypeError(dt)
    x, y, p = (np.ascontiguousarray(a, dtype=dt) for a in (x, y, power))
    z = np.ascontiguousarray(np.zeros_like(x) if z is None else z, dtype=dt)
    xe, ye = (np.ascontiguousarray(e, dtype=np.float64) for e in (x_edges, y_edges))
    nx, ny = len(xe) - 1, len(ye) - 1
    t, R, kind = np.zeros(3), np.eye(3), 0
    if frame is not None:
        kind = 1 if frame[0] == "affine" else 0
        t = np.ascontiguousarray(frame[1], dtype=np.float64)
        if kind:
            R = np.ascontiguousarray(frame[2], dtype=np.float64)
    R = np.ascontiguousarray(R, dtype=np.float64).reshape(9)
    n = x.size
    bins = np.empty(n, dtype=np.int64)
    hist = np.zeros(nx * ny, dtype=np.float64)
    fn = getattr(load(), "olbhc_irradiance_" + ("f64" if dt == np.float64 else "f32"))
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    fn.restype = None
    fn(ptr(x), ptr(y), ptr(z), ptr(p), C.c_int64(n), C.c_int32(kind), ptr(t), ptr(R), ptr(xe), C.c_int32(nx), ptr(ye),
       C.c_int32(ny), ptr(bins), ptr(hist))
    return bins, hist.reshape(nx, ny)
