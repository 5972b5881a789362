"""TEST INFRASTRUCTURE ONLY -- Python access to the host check built with the kernel variant of tables with a BSDF
surface (tests/hostcheck/hostcheck_bsdf.cpp: hostcheck_polygon.cpp plus the FEAT_BSDF instantiation of olb_math.cuh
and olb_bsdf.cuh), and to the draw function the kernel uses.  Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.hostcheck_api import CSRC, ROOT, run_hostcheck

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_bsdf.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_bsdf.so")
DEPS = [SRC] + [os.path.join(ROOT, "tests", "hostcheck", f) for f in
                ("hostcheck_polygon.cpp", "hostcheck_grid_sag.cpp", "hostcheck_coating.cpp", "hostcheck_grating.cpp",
                 "hostcheck_phase.cpp", "hostcheck.cpp")] + \
       [os.path.join(CSRC, f) for f in ("olb_math.cuh", "olb_bsdf.cuh", "olb_prep.h", "olb_fftpsf.cuh")] + \
       [os.path.join(ROOT, "include", "olb.h")]
_cache = None


def cuda_include() -> str:
    """The CUDA toolkit's include directory (cuRAND's Philox header and the vector types), next to the nvcc that
    builds libolb.so."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")


def build(force: bool = False) -> None:
    """Compile _hostcheck_bsdf.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC",
                               "-I", cuda_include(), "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


class _BsdfEntryPoints:
    """The BSDF-aware trace entry points, with the ray offset and stream bound, under the names
    ``hostcheck_api.run_hostcheck`` calls."""

    def __init__(self, lib, ray0: int, stream: int):
        extra = (C.c_int64(ray0), C.c_uint32(stream))
        self.olbhc_trace_f64 = lambda *a: lib.olbhc_bsdf_trace_f64(*a, *extra)
        self.olbhc_trace_f32 = lambda *a: lib.olbhc_bsdf_trace_f32(*a, *extra)


def run_hostcheck_bsdf(table, rays, dtype, first=0, last=None, want_l0=False, ray0=0, stream=0):
    """``hostcheck_api.run_hostcheck`` through the dispatch that also covers tables with BSDF surfaces; ray k draws as
    ray ``ray0 + k`` with counter word ``stream``."""
    return run_hostcheck(_BsdfEntryPoints(load(), ray0, stream), table, rays, dtype, first, last, want_l0=want_l0)


def draws(seed: int, stream: int, ray: int, count: int, kind: int, sigma: float, dtype=np.float64, attempt0: int = 0):
    """Draws ``attempt0 .. attempt0 + count - 1`` of one ray, (count, 2), exactly as the kernel makes them."""
    out = np.empty(2 * count)
    lib = load()
    lib.olbhc_bsdf_draws(C.c_uint64(seed), C.c_uint32(stream), C.c_uint64(ray), C.c_uint32(attempt0), C.c_int(count),
                         C.c_int(kind), C.c_double(sigma), C.c_int(0 if dtype == np.float64 else 1),
                         C.c_void_p(out.ctypes.data))
    return out.reshape(count, 2)


def philox(ctr, key):
    """One Philox4x32-10 block of the host instantiation."""
    c = (C.c_uint32 * 4)(*ctr)
    k = (C.c_uint32 * 2)(*key)
    o = (C.c_uint32 * 4)()
    load().olbhc_philox(c, k, o)
    return list(o)
