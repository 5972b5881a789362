"""TEST INFRASTRUCTURE ONLY -- Python access to the host check built with the kernel variant of tables with a
thin-film, polarizer or retarder coating (tests/hostcheck/hostcheck_coating.cpp: hostcheck_grating.cpp plus the
FEAT_JONES instantiation of olb_math.cuh), and to the per-ray thin-film arithmetic on its own.  Never imported by the
product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.hostcheck_api import CSRC, ROOT, run_hostcheck

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_coating.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_coating.so")
DEPS = [SRC, os.path.join(ROOT, "tests", "hostcheck", "hostcheck_grating.cpp"),
        os.path.join(ROOT, "tests", "hostcheck", "hostcheck_phase.cpp"),
        os.path.join(ROOT, "tests", "hostcheck", "hostcheck.cpp"), os.path.join(CSRC, "olb_math.cuh"),
        os.path.join(CSRC, "olb_prep.h"), os.path.join(CSRC, "olb_fftpsf.cuh"), os.path.join(ROOT, "include", "olb.h")]
_cache = None


def build(force: bool = False) -> None:
    """Compile _hostcheck_coating.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


class _CoatingEntryPoints:
    """The coating-aware trace entry points under the names ``hostcheck_api.run_hostcheck`` calls."""

    def __init__(self, lib):
        self.olbhc_trace_f64 = lib.olbhc_coating_trace_f64
        self.olbhc_trace_f32 = lib.olbhc_coating_trace_f32


def run_hostcheck_coating(table, rays, dtype, first=0, last=None, want_l0=False, pmat=None):
    """``hostcheck_api.run_hostcheck`` through the dispatch that also covers thin-film / polarizer / retarder tables."""
    return run_hostcheck(_CoatingEntryPoints(load()), table, rays, dtype, first, last, want_l0=want_l0, pmat=pmat)


def film_rt(table, surface: int, widx, aoi, dtype=np.float64):
    """(r_s, t_s, r_p, t_p), complex arrays, of the thin-film coating on ``surface`` at wavelength indices ``widx`` and
    angles of incidence ``aoi`` (radians), in the convention of the reference's ``_tmm_coh``."""
    from optiland_b200 import _lib

    ht = _lib.HostTable(table)
    widx = np.ascontiguousarray(widx, dtype=np.int32)
    aoi = np.ascontiguousarray(aoi, dtype=np.float64)
    out = np.zeros((len(aoi), 8))
    err = C.create_string_buffer(256)
    lib = load()
    fn = lib.olbhc_film_rt_f64 if dtype == np.float64 else lib.olbhc_film_rt_f32
    fn.restype = C.c_int
    rc = fn(C.byref(ht.c), C.c_int(surface), C.c_int64(len(aoi)), C.c_void_p(widx.ctypes.data),
            C.c_void_p(aoi.ctypes.data), C.c_void_p(out.ctypes.data), err, 256)
    assert rc == 0, err.value
    c = out[:, 0::2] + 1j * out[:, 1::2]
    return c[:, 0], c[:, 1], c[:, 2], c[:, 3]
