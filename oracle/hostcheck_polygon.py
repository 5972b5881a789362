"""TEST INFRASTRUCTURE ONLY -- Python access to the host check built with the kernel variants of tables with a polygon
in an aperture program (tests/hostcheck/hostcheck_polygon.cpp: hostcheck_grid_sag.cpp plus the FEAT_POLYGON
instantiations of olb_math.cuh).  Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.hostcheck_api import CSRC, ROOT, run_hostcheck

SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_polygon.cpp")
SO = os.path.join(ROOT, "tests", "hostcheck", "_hostcheck_polygon.so")
DEPS = [SRC] + [os.path.join(ROOT, "tests", "hostcheck", f) for f in
                ("hostcheck_grid_sag.cpp", "hostcheck_coating.cpp", "hostcheck_grating.cpp", "hostcheck_phase.cpp",
                 "hostcheck.cpp")] + \
       [os.path.join(CSRC, "olb_math.cuh"), os.path.join(CSRC, "olb_prep.h"), os.path.join(CSRC, "olb_fftpsf.cuh"),
        os.path.join(ROOT, "include", "olb.h")]
_cache = None


def build(force: bool = False) -> None:
    """Compile _hostcheck_polygon.so if it is missing or older than its sources (the flags of hostcheck.cpp's build)."""
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=fast", "-shared", "-fPIC", "-o", SO, SRC])


def load():
    global _cache
    if _cache is None:
        build()
        _cache = C.CDLL(SO)
    return _cache


class _PolygonEntryPoints:
    """The polygon-aware trace entry points under the names ``hostcheck_api.run_hostcheck`` calls."""

    def __init__(self, lib):
        self.olbhc_trace_f64 = lib.olbhc_polygon_trace_f64
        self.olbhc_trace_f32 = lib.olbhc_polygon_trace_f32


def run_hostcheck_polygon(table, rays, dtype, first=0, last=None, want_l0=False, pmat=None):
    """``hostcheck_api.run_hostcheck`` through the dispatch that also covers tables with polygon apertures."""
    return run_hostcheck(_PolygonEntryPoints(load()), table, rays, dtype, first, last, want_l0=want_l0, pmat=pmat)


def polygon_block(table, surface, dtype=np.float64):
    """The prepared polygon of ``surface`` (olb_prep.h PG_*): (buckets, ymin, ymax, start[buckets + 1], records (m, 4)
    of {vx, vy, vy_next, slope})."""
    from optiland_b200 import _lib

    ht = _lib.HostTable(table)
    out = np.zeros(1 << 16)
    err = C.create_string_buffer(256)
    n = load().olbhc_polygon_block(C.byref(ht.c), int(surface), 0 if dtype == np.float64 else 1,
                                   C.c_void_p(out.ctypes.data), out.size, err, 256)
    assert n >= 0, err.value
    nb, m = int(out[0]), int(out[3])
    pad = (nb + 1 + 3) & ~3
    return nb, out[1], out[2], out[4:4 + nb + 1].astype(int), out[4 + pad:4 + pad + 4 * m].reshape(m, 4)
