"""TEST INFRASTRUCTURE ONLY -- Python access to the host check built with the kernel variants of ruled-grating tables
(tests/hostcheck/hostcheck_grating.cpp: hostcheck_phase.cpp plus the FEAT_GRATING instantiations of olb_math.cuh).
Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from oracle.hostcheck_api import CSRC, ROOT, run_hostcheck

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_grating.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_grating.so")
DEPS = [SRC, os.path.join(ROOT, "tests", "hostcheck", "hostcheck_phase.cpp"),
        os.path.join(ROOT, "tests", "hostcheck", "hostcheck.cpp"), os.path.join(CSRC, "olb_math.cuh"),
        os.path.join(CSRC, "olb_prep.h"), os.path.join(CSRC, "olb_fftpsf.cuh"), os.path.join(ROOT, "include", "olb.h")]
_cache = None


def build(force: bool = False) -> None:
    """Compile _hostcheck_grating.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


class _GratingEntryPoints:
    """The grating-aware trace entry points under the names ``hostcheck_api.run_hostcheck`` calls."""

    def __init__(self, lib):
        self.olbhc_trace_f64 = lib.olbhc_grating_trace_f64
        self.olbhc_trace_f32 = lib.olbhc_grating_trace_f32


def run_hostcheck_grating(table, rays, dtype, first=0, last=None, want_l0=False, pmat=None):
    """``hostcheck_api.run_hostcheck`` through the dispatch that also covers ruled-grating tables."""
    return run_hostcheck(_GratingEntryPoints(load()), table, rays, dtype, first, last, want_l0=want_l0, pmat=pmat)
