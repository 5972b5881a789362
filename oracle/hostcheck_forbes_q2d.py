"""TEST INFRASTRUCTURE ONLY -- Python access to the host check built with the kernel variants of tables with a Forbes
Q-2D surface (tests/hostcheck/hostcheck_forbes_q2d.cpp: hostcheck_coating.cpp plus the FEAT_Q2D instantiations of
olb_math.cuh).  Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.hostcheck_api import CSRC, ROOT, run_hostcheck

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_forbes_q2d.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_forbes_q2d.so")
DEPS = [SRC] + [os.path.join(ROOT, "tests", "hostcheck", f) for f in
                ("hostcheck_coating.cpp", "hostcheck_grating.cpp", "hostcheck_phase.cpp", "hostcheck.cpp")] + \
       [os.path.join(CSRC, "olb_math.cuh"), os.path.join(CSRC, "olb_prep.h"), os.path.join(CSRC, "olb_fftpsf.cuh"),
        os.path.join(ROOT, "include", "olb.h")]
_cache = None


def build(force: bool = False) -> None:
    """Compile _hostcheck_forbes_q2d.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


class _Q2dEntryPoints:
    """The Q-2D-aware trace entry points under the names ``hostcheck_api.run_hostcheck`` calls."""

    def __init__(self, lib):
        self.olbhc_trace_f64 = lib.olbhc_forbes_q2d_trace_f64
        self.olbhc_trace_f32 = lib.olbhc_forbes_q2d_trace_f32


def run_hostcheck_forbes_q2d(table, rays, dtype, first=0, last=None, want_l0=False, pmat=None):
    """``hostcheck_api.run_hostcheck`` through the dispatch that also covers Q-2D tables."""
    return run_hostcheck(_Q2dEntryPoints(load()), table, rays, dtype, first, last, want_l0=want_l0, pmat=pmat)


def eval_surface(table, surf, x, y, dtype=np.float64):
    """(sag, fx, fy) of Q-2D surface ``surf`` at local points (x, y), in the kernel's arithmetic of ``dtype``."""
    from optiland_b200 import _lib

    lib = load()
    ht = _lib.HostTable(table)
    x = np.ascontiguousarray(x, dtype=np.float64).ravel()
    y = np.ascontiguousarray(y, dtype=np.float64).ravel()
    out = [np.zeros(x.size) for _ in range(3)]
    err = C.create_string_buffer(256)
    fn = lib.olbhc_forbes_q2d_eval_f64 if dtype == np.float64 else lib.olbhc_forbes_q2d_eval_f32
    P = C.c_void_p
    rc = fn(C.byref(ht.c), C.c_int(surf), C.c_int64(x.size), P(x.ctypes.data), P(y.ctypes.data),
            *[P(o.ctypes.data) for o in out], err, 256)
    assert rc == 0, err.value
    return tuple(out)
