"""TEST INFRASTRUCTURE ONLY -- Python access to the CPU instantiation of the ray-aiming solve
(tests/hostcheck/hostcheck_aim.cpp: hostcheck_polygon.cpp plus olb_aim.cuh with the kernel variants the library picks).
Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.hostcheck_api import CSRC, ROOT
from optiland_b200 import _lib

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_aim.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_aim.so")
DEPS = [SRC] + [os.path.join(ROOT, "tests", "hostcheck", f) for f in
                ("hostcheck_polygon.cpp", "hostcheck_grid_sag.cpp", "hostcheck_coating.cpp", "hostcheck_grating.cpp",
                 "hostcheck_phase.cpp", "hostcheck.cpp")] + \
       [os.path.join(CSRC, f) for f in ("olb_aim.cuh", "olb_math.cuh", "olb_prep.h", "olb_fftpsf.cuh")] + \
       [os.path.join(ROOT, "include", "olb.h")]
_cache = None
VARIANTS = {0: "closed form", 1: "general", 2: "superset"}


def build(force: bool = False) -> None:
    """Compile _hostcheck_aim.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


def run_aim(table, guess: dict, Px, Py, first: int, last: int, r_stop: float, J_factor: float, tol: float,
            max_iter: int, infinite: bool, dtype=np.float64):
    """One solve on the CPU.  ``guess``: {"x" .. "N"} (+ "w") arrays; returns (solution dict of the six arrays, status
    bits, kernel variant name)."""
    ht = _lib.HostTable(table)
    n = np.size(guess["x"])
    keys = ("x", "y", "z", "L", "M", "N", "w")
    arrs = [np.ascontiguousarray(np.broadcast_to(np.asarray(guess.get(k, np.zeros(n)), dtype=np.float64), (n,)),
                                 dtype=dtype).copy() for k in keys]
    px = np.ascontiguousarray(np.broadcast_to(np.asarray(Px, dtype=np.float64), (n,)), dtype=dtype)
    py = np.ascontiguousarray(np.broadcast_to(np.asarray(Py, dtype=np.float64), (n,)), dtype=dtype)
    status, variant = C.c_int(0), C.c_int(-1)
    err = C.create_string_buffer(256)
    hc = load()
    fn = hc.olbhc_aim_f64 if dtype == np.float64 else hc.olbhc_aim_f32
    fn.restype = C.c_int
    rc = fn(C.byref(ht.c), C.c_int(first), C.c_int(last), C.c_int64(n), (C.c_void_p * 7)(*[a.ctypes.data for a in arrs]),
            C.c_void_p(px.ctypes.data), C.c_void_p(py.ctypes.data), C.c_double(r_stop), C.c_double(J_factor),
            C.c_double(tol), C.c_int(max_iter), C.c_int(1 if infinite else 0), C.byref(status), C.byref(variant),
            err, 256)
    if rc != 0:
        raise _lib.OlbError(f"olbhc_aim failed: {_lib.ERRORS.get(rc, rc)}: {err.value.decode()}")
    return dict(zip(keys[:6], arrs[:6])), status.value, VARIANTS[variant.value]
