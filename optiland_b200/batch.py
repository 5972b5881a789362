"""Batched many-systems traces (SURVEY.md 8f-4): B perturbed copies of one template system in ONE launch.

The reference evaluates such ensembles one system at a time: the tolerancing Monte-Carlo loop
(optiland/tolerancing/monte_carlo.py:86-123 -> optiland/tolerancing/core.py) applies the sampled
perturbations to the live Optic and re-traces it per sample, and the BatchedRayEvaluator
(optiland/optimization/batched_evaluator.py:277-705) groups ray bundles of ONE system.  Here the B
prepared tables live side by side in HBM and the trace kernel's grid.y picks the system, so the B small
traces (a few thousand rays each -- far too small to fill 132 SMs alone) become one full-width launch.

``params`` is a (B, S, BP_COUNT) fp64 array of ABSOLUTE values (include/olb.h, OLB_BP_*): pose (t, R),
curvature, conic, n1, n2, even-asphere coefficients.  ``template_params`` + a perturbation is the usual way
to fill it.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np
import torch

from . import _lib
from . import table as T
from .trace import RealRays, _REC_KEYS, _c_records, _out_buffer, _require_cuda, _trace


def template_params(table: T.SurfaceTable) -> np.ndarray:
    """(S, BP_COUNT) block of the template's own values."""
    if table.n_wl != 1:
        raise ValueError("batched tables support one wavelength")
    if any(s.interaction != T.INTERACT_REFRACT for s in table.surfaces):
        raise ValueError("batched tables with phase-profile or grating surfaces are not built")
    if any(s.coating in T.JONES_COATINGS for s in table.surfaces):
        raise ValueError("batched tables with thin-film, polarizer or retarder coatings are not built")
    if any(s.kind == T.GEOM_GRID_SAG for s in table.surfaces):
        raise ValueError("batched tables with grid-sag surfaces are not built")
    if any(s.bsdf != T.BSDF_NONE for s in table.surfaces):
        raise ValueError("batched tables with BSDF surfaces are not built")
    if any(s.kind == T.GEOM_FORBES_Q2D for s in table.surfaces):
        raise ValueError("batched tables with Forbes Q-2D surfaces are not built")
    p = np.zeros((table.num_surfaces, _lib.BP_COUNT))
    for s, spec in enumerate(table.surfaces):
        p[s, _lib.BP_TX:_lib.BP_TX + 3] = spec.t
        p[s, _lib.BP_R:_lib.BP_R + 9] = np.asarray(spec.R, dtype=np.float64).reshape(9)
        p[s, _lib.BP_CURV] = 0.0 if not np.isfinite(spec.radius) else 1.0 / spec.radius
        p[s, _lib.BP_CONIC] = spec.conic
        p[s, _lib.BP_N1], p[s, _lib.BP_N2] = spec.n1[0], spec.n2[0]
        if spec.kind == T.GEOM_EVEN_ASPHERE:
            k = len(spec.coefficients)
            if k > _lib.BP_MAX_COEF:
                raise ValueError(f"more than {_lib.BP_MAX_COEF} even-asphere coefficients")
            p[s, _lib.BP_COEF:_lib.BP_COEF + k] = spec.coefficients
    return p


def system_table(template: T.SurfaceTable, params_b: np.ndarray) -> T.SurfaceTable:
    """The single-system ``SurfaceTable`` that one (S, BP_COUNT) block describes (what
    olb_table_upload_batch builds internally for that system)."""
    p = np.asarray(params_b, dtype=np.float64)
    specs = []
    for s, spec in enumerate(template.surfaces):
        if spec.kind == T.GEOM_NOOP:
            specs.append(spec)
            continue
        ch = dict(t=p[s, _lib.BP_TX:_lib.BP_TX + 3].copy(), R=p[s, _lib.BP_R:_lib.BP_R + 9].reshape(3, 3).copy(),
                  n1=np.array([p[s, _lib.BP_N1]]), n2=np.array([p[s, _lib.BP_N2]]))
        if spec.kind != T.GEOM_PLANE:
            ch["radius"] = float("inf") if p[s, _lib.BP_CURV] == 0 else 1.0 / p[s, _lib.BP_CURV]
            if spec.kind != T.GEOM_TOROIDAL:
                ch["conic"] = float(p[s, _lib.BP_CONIC])
        if spec.kind == T.GEOM_EVEN_ASPHERE:
            ch["coefficients"] = p[s, _lib.BP_COEF:_lib.BP_COEF + len(spec.coefficients)].copy()
        specs.append(dataclasses.replace(spec, **ch))
    return T.SurfaceTable(specs, template.wavelengths)


class BatchedTable:
    """B prepared systems resident on one GPU (olb_table_upload_batch)."""

    def __init__(self, template: T.SurfaceTable, params, device=None):
        _require_cuda()
        self.lib = _lib.load()
        self.template = template
        self.params = np.ascontiguousarray(params, dtype=np.float64)
        if self.params.ndim != 3 or self.params.shape[1:] != (template.num_surfaces, _lib.BP_COUNT):
            raise ValueError(f"params must be (B, {template.num_surfaces}, {_lib.BP_COUNT})")
        self.n_systems = int(self.params.shape[0])
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.host = _lib.HostTable(template)
        nbytes = self.lib.olb_table_batch_workspace_bytes(C.byref(self.host.c), self.n_systems)
        if nbytes < 0:
            _lib.check(int(nbytes), "olb_table_batch_workspace_bytes")
        self.workspace = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        self.c = _lib.OlbDeviceTable()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            rc = self.lib.olb_table_upload_batch(C.byref(self.host.c), C.c_void_p(self.params.ctypes.data),
                                                 self.n_systems, self.workspace.data_ptr(), int(nbytes),
                                                 C.c_void_p(stream), C.byref(self.c))
        _lib.check(rc, "olb_table_upload_batch")


def trace_batch(btab: BatchedTable, rays: RealRays, rays_per_system: int | None = None, shared_input: bool = False,
                record: bool = True, moments: bool = False, center=(0.0, 0.0), first: int = 0, last: int | None = None):
    """All B systems in one launch (OlbTraceCall.rays_per_system).  ``rays`` holds either B * m launch rays
    (system b owns [b*m, (b+1)*m)) or, with ``shared_input``, m rays that EVERY system traces.  Returns ``(records, moments)``: records = dict of
    (rows, B, m) tensors or None; moments = (B, 8) fp64 tensor or None.  Without records and without
    ``shared_input`` the final state is written back into ``rays`` in place."""
    B = btab.n_systems
    n_in = len(rays)
    m = int(rays_per_system) if rays_per_system is not None else (n_in if shared_input else n_in // B)
    if (shared_input and n_in != m) or (not shared_input and n_in != m * B):
        raise ValueError("ray count does not match rays_per_system x n_systems")
    last = btab.template.num_surfaces if last is None else last
    rows = last - first
    n = B * m
    flags = 0
    recs, c_rec = None, None
    if record and rows > 0:
        buf = _out_buffer(8, rows, n, rays.dtype, rays.device)
        recs = {k: buf[j, :, :n].view(rows, B, m) for j, k in enumerate(_REC_KEYS)}
        c_rec = _c_records(buf)
        flags |= _lib.TF_NO_FINAL
    if shared_input:
        flags |= _lib.TF_SHARED_INPUT | _lib.TF_NO_FINAL
    mom = None
    if moments:
        mom = torch.zeros((B, 8), dtype=torch.float64, device=rays.device)
        flags |= _lib.TF_MOMENTS
        if not record:
            flags |= _lib.TF_NO_FINAL
    c_rays = _lib.OlbRays(x=rays.x.data_ptr(), y=rays.y.data_ptr(), z=rays.z.data_ptr(), L=rays.L.data_ptr(),
                          M=rays.M.data_ptr(), N=rays.N.data_ptr(), i=rays.i.data_ptr(), opd=rays.opd.data_ptr())
    # (no status word: out-of-range freeform coordinates are not reported on this path)
    _trace(btab, rays.device, rays.dtype, first, last, n, flags, rays=c_rays, rec=c_rec, center=center, moments=mom,
           rays_per_system=m, own_status=False)
    return recs, mom
