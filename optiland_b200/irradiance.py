"""Incoherent irradiance binning on the GPU (``olb_irradiance_*``), and its hook into the reference's
``IncoherentIrradiance._generate_field_data`` (optiland/analysis/irradiance.py:265-353).

The reference's non-differentiable branch copies the x, y and power of every ray to the host, masks ``power > 0`` and
calls ``np.histogram2d`` with the power as weights (irradiance.py:338-353): at 10^6 - 10^8 rays that binning costs about
three orders of magnitude more than the trace.  Here the rays stay on the device and one kernel localizes, masks, bins
and accumulates them in fp64; only the (nx, ny) grid comes back.  Semantics: include/olb.h, ``OlbIrradiance``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

_SFX = {torch.float64: "f64", torch.float32: "f32"}


def bin_irradiance(x, y, power, x_edges, y_edges, z=None, frame=None, out=None, path: int = _lib.IRR_PATH_AUTO):
    """fp64 ``(nx, ny)`` tensor ``hist[ix, iy]``: the summed ``power`` of the rays whose local position falls in pixel
    (ix, iy) (``np.histogram2d(x, y, [x_edges, y_edges], weights=power)`` over the rays with ``power > 0``).

    ``x / y / z / power``: 1-D CUDA tensors of one floating type (fp32 or fp64) and one length.  ``x_edges / y_edges``:
    finite, strictly increasing fp64 edges (host arrays).  ``frame``: None (the points are already local),
    ``("translate", t)`` -- the local point is ``(x - t[0], y - t[1])`` in the rays' precision -- or
    ``("affine", t, R)`` -- ``R^T (p - t)`` in fp64, which needs ``z``.  ``out``: an fp64 ``(nx, ny)`` tensor on the
    rays' device to accumulate into (zeroed here when None).  ``path``: ``_lib.IRR_PATH_*``; the default lets the library
    choose between its two accumulation paths, the others force one (scripts/bench_irradiance.py measures both)."""
    dtype = x.dtype
    if dtype not in _SFX or not x.is_cuda:
        raise _lib.OlbError("bin_irradiance: CUDA fp32 / fp64 rays expected; there is no CPU fallback")
    dev = x.device
    arrs = [x, y, power] + ([z] if z is not None else [])
    for t in arrs:
        if not torch.is_tensor(t) or t.dtype != dtype or t.device != dev or t.ndim != 1 or t.shape != x.shape:
            raise _lib.OlbError("bin_irradiance: x, y, z and power must be 1-D CUDA tensors of one type, device and length")
    xe = np.ascontiguousarray(x_edges, dtype=np.float64)
    ye = np.ascontiguousarray(y_edges, dtype=np.float64)
    nx, ny = xe.size - 1, ye.size - 1
    c = _lib.OlbIrradiance()
    kind = "translate" if frame is None else frame[0]
    if kind == "affine":
        if z is None:
            raise _lib.OlbError("bin_irradiance: an affine frame needs z")
        c.frame = _lib.IRR_FRAME_AFFINE
        c.t[:] = [float(v) for v in np.asarray(frame[1], dtype=np.float64).reshape(3)]
        c.R[:] = [float(v) for v in np.asarray(frame[2], dtype=np.float64).reshape(9)]
    elif kind == "translate":
        c.frame = _lib.IRR_FRAME_TRANSLATE
        if frame is not None:
            c.t[:] = [float(v) for v in np.asarray(frame[1], dtype=np.float64).reshape(3)]
    else:
        raise ValueError(f"bin_irradiance: unknown frame {kind!r}")
    if out is None:
        out = torch.zeros((max(nx, 0), max(ny, 0)), dtype=torch.float64, device=dev)
    elif out.dtype != torch.float64 or out.device != dev or tuple(out.shape) != (nx, ny) or not out.is_contiguous():
        raise _lib.OlbError("bin_irradiance: out must be a contiguous fp64 (nx, ny) tensor on the rays' device")
    scratch = torch.empty(max(nx + ny + 2, 1), dtype=torch.float64, device=dev)
    keep = [t.detach().contiguous() for t in arrs]
    c.x, c.y, c.i = keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr()
    c.z = keep[3].data_ptr() if z is not None else None
    c.n_rays, c.nx, c.ny, c.path = x.numel(), nx, ny, int(path)
    c.x_edges, c.y_edges = xe.ctypes.data, ye.ctypes.data
    c.edges, c.hist = scratch.data_ptr(), out.data_ptr()
    lib = _lib.load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = getattr(lib, f"olb_irradiance_{_SFX[dtype]}")(C.byref(c), C.c_void_p(stream))
    _lib.check(rc, f"olb_irradiance_{_SFX[dtype]}")
    return out


# ---- the hook into the reference's class ------------------------------------------------------------------------------

def _edges(self, surf):
    """(x_edges, y_edges, pixel_area, npix) exactly as irradiance.py:298-314 forms them; ``npix`` is the (nx, ny) the
    px_size branch would store (and announce) when it differs from ``(self.npix_x, self.npix_y)``, else None."""
    x_min, x_max, y_min, y_max = surf.aperture.extent
    if self.px_size is None:
        x_edges = np.linspace(x_min, x_max, self.npix_x + 1, dtype=float)
        y_edges = np.linspace(y_min, y_max, self.npix_y + 1, dtype=float)
        return x_edges, y_edges, (x_edges[1] - x_edges[0]) * (y_edges[1] - y_edges[0]), None
    dx, dy = self.px_size
    x_edges = np.arange(x_min, x_max + 0.5 * dx, dx, dtype=float)
    y_edges = np.arange(y_min, y_max + 0.5 * dy, dy, dtype=float)
    npix = (len(x_edges) - 1, len(y_edges) - 1)
    return x_edges, y_edges, dx * dy, (None if npix == (self.npix_x, self.npix_y) else npix)


def _proper(e) -> bool:
    return e.ndim == 1 and e.size >= 2 and bool(np.all(np.isfinite(e))) and bool(np.all(np.diff(e) > 0))


def _frame(be, surf, dtype):
    """The detector frame for the kernel (CoordinateSystem.localize, coordinate_system.py:73-89): a translation when the
    frame is unrotated, has no parent and its origin tensors do not widen the rays' precision (so that ``x - t`` in the
    rays' precision is the reference's ``translate`` bit for bit), else the effective (t, R) in fp64."""
    cs = surf.geometry.cs
    origin = (cs.x, cs.y, cs.z)

    def narrow(v):   # x + v keeps the rays' dtype (a 0-d tensor, a Python number, or a tensor of that dtype)
        return not torch.is_tensor(v) or v.ndim == 0 or v.dtype == dtype

    if cs.reference_cs is None and not (cs.rx or cs.ry or cs.rz) and all(narrow(v) for v in origin):
        return ("translate", [float(v) for v in origin])
    t, R = cs.get_effective_transform()
    return ("affine", np.asarray(be.to_numpy(t), dtype=np.float64), np.asarray(be.to_numpy(R), dtype=np.float64))


def install(P, registry, be):
    """Wrap ``IncoherentIrradiance._generate_field_data``; returns the original for ``uninstall``."""
    from optiland.analysis.irradiance import IncoherentIrradiance
    from optiland.rays import RealRays

    orig = IncoherentIrradiance._generate_field_data

    def host_bin(x_g, y_g, z_g, power, surf, x_edges, y_edges, pixel_area):
        """The reference's own binning of rays it has already traced (irradiance.py:294-296, 340-353)."""
        from optiland.visualization.system.utils import transform

        x_local, y_local, _ = transform(x_g, y_g, z_g, surf, is_global=True)
        x_np, y_np, p_np = be.to_numpy(x_local), be.to_numpy(y_local), be.to_numpy(power)
        keep = p_np > 0.0
        hist, _, _ = np.histogram2d(x_np[keep], y_np[keep], bins=[x_edges, y_edges], weights=p_np[keep])
        return be.array(hist / pixel_area)

    def generate_field_data(self, field, wavelength, distribution, user_initial_rays):
        eng = P._state.get("engine")
        if be.get_backend() != "torch":
            P._decline("irradiance: backend is not torch")
            return orig(self, field, wavelength, distribution, user_initial_rays)
        if be.grad_mode.requires_grad:
            P._decline("irradiance: gradients wanted (bilinear branch)")
            return orig(self, field, wavelength, distribution, user_initial_rays)
        if eng is None or not hasattr(eng, "irradiance"):
            P._decline("irradiance: engine has no irradiance kernel")
            return orig(self, field, wavelength, distribution, user_initial_rays)
        surf = self.optic.surfaces[self.detector_surface]
        x_edges, y_edges, pixel_area, npix = _edges(self, surf)
        if not (_proper(x_edges) and _proper(y_edges)):
            P._decline("irradiance: degenerate detector edges")
            return orig(self, field, wavelength, distribution, user_initial_rays)

        # the reference's own trace calls (irradiance.py:270-292), served by the plugin's trace capability
        rays_traced = None
        if not self.skip_trace:
            if user_initial_rays is None:
                Hx, Hy = field
                rays_traced = self.optic.trace(Hx, Hy, wavelength, self.num_rays, distribution)
            else:
                rays_traced = RealRays(**self._initial_ray_data)
                self.optic.surfaces.trace(rays_traced)
        if rays_traced is not None:
            x_g, y_g, z_g, power = rays_traced.x, rays_traced.y, rays_traced.z, rays_traced.i
        else:
            x_g, y_g, z_g, power = surf.x, surf.y, surf.z, surf.intensity
        if npix is not None:   # irradiance.py:308-314
            print(f"[IncoherentIrradiance] Warning: res parameter ignored - derived from px_size instead → "
                  f"({npix[0]},{npix[1]}) pixels")
            self.npix_x, self.npix_y = npix

        # the rays in the backend's precision, as transform() builds them (RealRays -> be.atleast_1d)
        x, y, z = (be.atleast_1d(v) for v in (x_g, y_g, z_g))
        hist = None
        if torch.is_tensor(power) and power.dtype in (torch.float32, torch.float64) and x.dtype.itemsize >= power.dtype.itemsize:
            p = power.to(x.dtype)           # exact: same or wider type
            hist = eng.irradiance(x, y, z, p, x_edges, y_edges, _frame(be, surf, x.dtype))
        if hist is None:
            P._decline("irradiance: rays not accepted by the engine")
            return host_bin(x_g, y_g, z_g, power, surf, x_edges, y_edges, pixel_area), x_edges, y_edges
        # the fp64 grid, divided on the host and handed to be.array as the reference does (irradiance.py:352-353)
        irr = hist.cpu().numpy() / pixel_area
        return be.array(irr), x_edges, y_edges

    IncoherentIrradiance._generate_field_data = generate_field_data
    return orig


def uninstall(saved):
    from optiland.analysis.irradiance import IncoherentIrradiance

    IncoherentIrradiance._generate_field_data = saved
