"""TEST INFRASTRUCTURE ONLY -- Python access to the host check built with the kernel variants of tables with a grid-sag
surface (tests/hostcheck/hostcheck_grid_sag.cpp: hostcheck_coating.cpp plus the FEAT_GRID instantiations of
olb_math.cuh).  Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from oracle.hostcheck_api import CSRC, ROOT, run_hostcheck

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_grid_sag.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_grid_sag.so")
DEPS = [SRC] + [os.path.join(ROOT, "tests", "hostcheck", f) for f in
                ("hostcheck_coating.cpp", "hostcheck_grating.cpp", "hostcheck_phase.cpp", "hostcheck.cpp")] + \
       [os.path.join(CSRC, "olb_math.cuh"), os.path.join(CSRC, "olb_prep.h"), os.path.join(CSRC, "olb_fftpsf.cuh"),
        os.path.join(ROOT, "include", "olb.h")]
_cache = None


def build(force: bool = False) -> None:
    """Compile _hostcheck_grid_sag.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


class _GridSagEntryPoints:
    """The grid-aware trace entry points under the names ``hostcheck_api.run_hostcheck`` calls."""

    def __init__(self, lib):
        self.olbhc_trace_f64 = lib.olbhc_grid_sag_trace_f64
        self.olbhc_trace_f32 = lib.olbhc_grid_sag_trace_f32


def run_hostcheck_grid_sag(table, rays, dtype, first=0, last=None, want_l0=False, pmat=None):
    """``hostcheck_api.run_hostcheck`` through the dispatch that also covers grid-sag tables."""
    return run_hostcheck(_GridSagEntryPoints(load()), table, rays, dtype, first, last, want_l0=want_l0, pmat=pmat)
