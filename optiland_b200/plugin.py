"""Drop-in for Optiland: the CUDA trace loop behind ``optiland.backend``'s registry.

``install()`` (SURVEY.md section 8b):

1. registers ``B200TorchBackend`` -- a subclass of the reference's ``TorchBackend``
   (optiland/backend/torch_backend.py:113) that keeps all of its ~140 array
   ops (so autograd interop and every ``be.*`` call are unchanged), still reports the name
   ``"torch"`` (28 call sites branch on ``be.get_backend() == "torch"``) and adds ONE
   capability, ``trace_surfaces(surface_group, rays, start, stop) -> bool``; it is installed
   the way the reference's own test registers a foreign backend
   (the reference's tests/test_backend.py:79-85): by assignment into ``_backends``;
2. wraps ``RealRayTracer.trace`` (optiland/raytrace/real_ray_tracer.py:58-118) so that a single-field
   ``Optic.trace`` on an infinite-object angle field generates its launch rays inside the kernel
   (SURVEY.md 8f-1), and wraps ``SurfaceGroup.trace`` (optiland/surfaces/surface_group.py:245-257) and ``Surface.trace``
   (optiland/surfaces/standard_surface.py:200-215, the per-surface entry the ray aimers use) so that
   they try the capability first and run the reference's own Python body when it declines
   (unsupported surface kind, CPU tensors, ...).  With ``be.grad_mode`` on, the capability runs
   the forward and the hand-derived adjoint kernel as ONE ``torch.autograd.Function`` whose inputs
   are the live parameter tensors, so ``TorchBaseOptimizer`` differentiates through it.

``Optic.trace``, ``SpotDiagram``, ``Wavefront``, PSF and the optimisers are untouched and call
the path unchanged.  Declining is NOT a CPU fallback of this package: it hands the call back to
the reference's own code, which is what runs today.
"""
from __future__ import annotations

import sys
import threading
from collections import OrderedDict

import numpy as np

from . import table as T
from ._lib import OlbError
from .pack import UnsupportedSurface, pack_surface, pack_surface_group

# what packing / uploading a table may raise for a system outside the kernel's scope (aperture tree deeper than the
# evaluator's stack, polynomial order beyond the prepared tables, table larger than shared memory ...): every one
# of them hands the call back to the reference's own Python body instead of escaping from SurfaceGroup.trace
_PACK_ERRORS = (UnsupportedSurface, ValueError, TypeError, OlbError)

_REC_ATTR = (("x", "x"), ("y", "y"), ("z", "z"), ("L", "L"), ("M", "M"), ("N", "N"),
             ("intensity", "intensity"), ("opd", "opd"))
_tls = threading.local()


class _FrozenTables:
    """Context in which the optic is known not to change -- one ``aim_rays`` call of the iterative / robust ray aimer
    (rays/ray_aiming/iterative.py, robust.py: hundreds to thousands of subset traces of the SAME system while only the
    launch parameters move; the robust aimer of ``WideAngle170FOV`` issues ~1500 per ``Optic.trace``).  Inside it a packed
    table is built once per (surfaces, range, wavelengths) instead of once per trace: packing the live objects (~1 ms) is
    what such a trace costs on a GPU, the kernel takes ~20 us.  Re-entrant; the outermost exit drops everything."""

    def __enter__(self):
        self.outer = getattr(_tls, "frozen", None)
        if self.outer is None:
            _tls.frozen = {}
        return self

    def __exit__(self, *exc):
        if self.outer is None:
            _tls.frozen = None
        return False


class _ParaxialMemo:
    """For the duration of a call in which the optic does not change (``RayGenerator.generate_rays``, the launch scalars of
    a fused launch) ``Paraxial.EPL / EPD`` and ``SurfaceGroup.positions`` hand out the tensors they computed first
    (installed by ``install``); re-entrant, the outermost exit drops the memo."""

    def __enter__(self):
        self.outer = getattr(_tls, "paraxial_memo", None)
        if self.outer is None:
            _tls.paraxial_memo = {}
        return self

    def __exit__(self, *exc):
        if self.outer is None:
            _tls.paraxial_memo = None
        return False


def _frozen(key, owner, build):
    """``build()`` memoised on ``key`` while a _FrozenTables context is active (``owner`` is kept alive with the entry so
    that an ``id()`` in the key cannot be recycled)."""
    fr = getattr(_tls, "frozen", None)
    if fr is None:
        return build()
    hit = fr.get(key)
    if hit is None:
        hit = fr[key] = (owner, build())
    return hit[1]


_state: dict = {"installed": False, "declines": {}}


def _decline(reason: str):
    """Count why a call went back to the reference's Python body (see ``stats()``)."""
    d = _state.setdefault("declines", {})
    d[reason] = d.get(reason, 0) + 1
    return False


_RESET_ATTRS = ("y", "u", "x", "z", "L", "M", "N", "intensity", "aoi", "opd")


def _reset_records(be, surface_group) -> None:
    """``SurfaceGroup.reset()`` (surfaces/surface_group.py:373-380 -> standard_surface.py:285-299) without its 11
    allocations per surface: every attribute gets ONE shared empty array (143 ``be.empty(0)`` calls on the Double-Gauss,
    0.5 ms on a CUDA device, were the largest single item of a small ``Optic.trace`` through the plugin)."""
    e = be.empty(0)
    for surf in surface_group.surfaces:
        for attr in _RESET_ATTRS:
            setattr(surf, attr, e)


def _fused_decline(reason: str):
    """A fused entry point (Optic.trace / trace_generic / Wavefront) hands the call to the next level down -- the
    reference's RayGenerator followed by the SurfaceGroup.trace capability -- and says why (``stats()``)."""
    _decline("fused launch: " + reason)
    return None


def stats(reset: bool = False) -> dict:
    """{reason: count} of the calls the capability declined since install / the last reset --
    the answer to "why was my trace not accelerated?"."""
    out = dict(_state.get("declines", {}))
    if reset:
        _state["declines"] = {}
    return out


def _dev_array(t):
    """Detached, contiguous and 16-byte aligned (a view into a larger tensor may start anywhere)."""
    t = t.detach().contiguous()
    return t.clone() if t.data_ptr() % 16 else t


class CudaEngine:
    """Runs a packed table on the GPU through libolb (``optiland_b200.trace``)."""

    def __init__(self, cache_size: int = 8):
        self._cache: OrderedDict[bytes, object] = OrderedDict()
        self._cache_size = cache_size
        # what went through the engine, newest last: (n_surfaces, n_rays) for a plain trace, otherwise
        # (kind, ...) with kind in {"pupil", "wavefront", "psf", "grad", "moments", "batch", "irradiance"} -- the answer to
        # "did my call really run on the kernel?" (tests, plugin.stats())
        self.calls: list = []

    def _note(self, *what):
        self.calls.append(what)
        if len(self.calls) > 65536:
            del self.calls[:32768]

    # (class attribute so that the CPU tests can exercise ``accepts`` on host tensors: tests/test_pack_fast_path.py)
    _on_device = staticmethod(lambda t: t.is_cuda)

    def accepts(self, rays) -> bool:
        """Can this ray object be handed to the kernels as it is?  Nine 1-D arrays of one floating type on one CUDA
        device and of one length -- except ``w``, which may be ONE value for the whole batch:
        ``RealRays(..., wavelength=0.55)`` keeps a 1-element array that the reference's ops broadcast (real_rays.py:79;
        the iterative ray aimer builds its rays that way, ray_aiming/iterative.py:361)."""
        import torch

        keys = ("x", "y", "z", "L", "M", "N", "i", "opd")
        ts = [getattr(rays, k, None) for k in keys]
        w = getattr(rays, "w", None)
        if any(not torch.is_tensor(t) for t in ts) or not torch.is_tensor(w):
            return False
        t0 = ts[0]
        dev = self._on_device
        if not dev(t0) or t0.dtype not in (torch.float32, torch.float64) or t0.ndim != 1:
            return False
        if not (dev(w) and w.dtype == t0.dtype and w.device == t0.device and w.ndim == 1
                and (w.shape == t0.shape or w.numel() == 1)):
            return False
        return all(dev(t) and t.dtype == t0.dtype and t.shape == t0.shape and t.device == t0.device for t in ts)

    def device_table(self, table: T.SurfaceTable, device):
        from .trace import DeviceTable

        key = table.content_key() + str(device).encode()
        dt = self._cache.get(key)
        if dt is None:
            dt = DeviceTable(table, device, packed=table.packed())
            self._cache[key] = dt
            while len(self._cache) > self._cache_size:
                self._cache.popitem(last=False)
        else:
            self._cache.move_to_end(key)
        return dt

    def trace(self, table: T.SurfaceTable, rays, first: int, last: int):
        """Trace Optiland's ``rays`` object in place; return {key: (rows, N) tensor}."""
        import torch

        from .trace import PolarizedRays, RealRays, trace_device

        polarized = type(rays).__name__ == "PolarizedRays"
        shell = (PolarizedRays if polarized else RealRays).__new__(PolarizedRays if polarized else RealRays)
        if polarized:
            # the reference starts from a REAL identity stack (polarized_rays.py:50); the kernel
            # always carries the complex form
            cdt = torch.complex64 if rays.x.dtype == torch.float32 else torch.complex128
            shell.p = rays.p.detach().to(cdt).contiguous()
        n = rays.x.numel()
        for k in ("x", "y", "z", "L", "M", "N", "i", "w", "opd"):
            t = getattr(rays, k).detach()
            if k == "w" and t.numel() == 1 and n != 1:
                t = t.expand(n)                    # one wavelength for the whole batch (accepts())
            t = t.contiguous()
            if t.data_ptr() % 16:
                t = t.clone()
            setattr(shell, k, t)
        shell.L0 = shell.M0 = shell.N0 = None
        shell.is_normalized = True
        dt = self.device_table(table, shell.x.device)
        self._note(table.num_surfaces, int(shell.x.numel()))
        rec = trace_device(dt, shell, first, last, record=True)
        for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
            setattr(rays, k, getattr(shell, k))
        if polarized:
            rays.p = shell.p
        return rec


    def aim(self, table: T.SurfaceTable, guess: dict, Px, Py, r_stop: float, J_factor: float, tol: float,
            max_iter: int, infinite: bool) -> int:
        """One ray-aiming solve through the whole ``table`` (olb_aim_*, one launch): ``guess`` holds the launch state
        {"x" .. "N"} (+ "w" for several wavelengths) as aligned device tensors and receives the solution in place.
        Returns the OLB_ST_* bits (one 4-byte read-back); any bit set is a failed solve."""
        from .trace import aim_device

        dt = self.device_table(table, guess["x"].device)
        self._note("aim", table.num_surfaces, int(guess["x"].numel()))
        st = aim_device(dt, guess, Px, Py, 0, table.num_surfaces, r_stop, J_factor, tol, max_iter, infinite)
        return int(st.item())

    def accepts_tensor(self, t) -> bool:
        import torch

        return torch.is_tensor(t) and t.is_cuda and t.dtype in (torch.float32, torch.float64) and t.ndim == 1

    def trace_pupil(self, table: T.SurfaceTable, Px, Py, affine: dict, wavelength=None, polarization=False):
        """Launch state generated in-kernel from the pupil samples (OlbTraceCall.launch; with ``affine["fields"]``
        also from per-ray field points).  ``wavelength``: per-ray array for a multi-wavelength table.  Returns the
        record dict; the final state is its last row.  ``polarization``: False, or the optic's polarization state
        (None = unpolarized, or (Ex, Ey, phase_x, phase_y)) -- PolarizedRays are traced (OLB_TF_POLARIZED, OlbTraceCall.pol) and
        the dict also holds ``"p"`` (the (N, 3, 3) complex matrices) and ``"i_pol"`` (update_intensity's result)."""
        from .trace import trace_pupil_device

        dt = self.device_table(table, Px.device)
        if affine.get("fields") is not None:
            affine = dict(affine, fields=tuple(_dev_array(t) for t in affine["fields"]))
        w = _dev_array(wavelength) if wavelength is not None else None
        self._note("pupil", table.num_surfaces, int(Px.numel()))
        rays, rec = trace_pupil_device(dt, _dev_array(Px), _dev_array(Py), affine, 0, table.num_surfaces, wavelength=w,
                                       polarization=polarization)
        if polarization is not False:
            rec = dict(rec, p=rays.p, i_pol=rays.i)
        return rec

    def trace_wavefront(self, table: T.SurfaceTable, Px, Py, affine: dict, ref: dict, polarized: bool = False) -> dict:
        """One field's pupil grid -> OPD map + exit-pupil intercepts + intensity, nothing else written
        (OlbTraceCall.wavefront_*); ``polarized``: PolarizedRays, the result also holds the P matrices ``"p"``."""
        from .trace import trace_wavefront_device

        dt = self.device_table(table, Px.device)
        self._note("wavefront", table.num_surfaces, int(Px.numel()))
        return trace_wavefront_device(dt, _dev_array(Px), _dev_array(Py), affine, ref, polarized=polarized)

    def spot_moments(self, table: T.SurfaceTable, Px, Py, affine: dict, center=(0.0, 0.0), last=None,
                     global_xy: bool = False, every_ray: bool = False) -> list:
        """Launch generation + trace + moment sums in ONE kernel, nothing written per ray (OlbTraceCall.moments):
        the 8 sums of include/olb.h as Python floats (one 64-byte read-back)."""
        from .trace import trace_moments_device

        dt = self.device_table(table, Px.device)
        self._note("moments", table.num_surfaces, int(Px.numel()))
        m = trace_moments_device(dt, int(Px.numel()), Px.dtype, pupil=(_dev_array(Px), _dev_array(Py), affine),
                                 center=center, last=last, global_xy=global_xy, every_ray=every_ray)
        return [float(v) for v in m.cpu()]

    def huygens_psf(self, image_x, image_y, image_z, pupil_x, pupil_y, pupil_z, pupil_amp, pupil_opd, wavelength, Rp):
        """Huygens-Fresnel summation on the GPU (olb_huygens_psf_f64); None to decline (CPU tensors)."""
        import torch

        from .psf import huygens_fresnel_psf

        if not (torch.is_tensor(image_x) and image_x.is_cuda):
            return None
        self._note("psf", int(image_x.numel()), int(pupil_x.numel()))
        return huygens_fresnel_psf(image_x, image_y, image_z, pupil_x, pupil_y, pupil_z, pupil_amp, pupil_opd,
                                   wavelength, Rp).to(image_x.dtype)

    def irradiance(self, x, y, z, power, x_edges, y_edges, frame):
        """fp64 (nx, ny) irradiance histogram of the rays in one pass (olb_irradiance_*, optiland_b200.irradiance);
        None to decline (not 1-D CUDA tensors of one type, device and length)."""
        from .irradiance import bin_irradiance

        ts = (x, y, z, power)
        if not all(self.accepts_tensor(t) and t.dtype == x.dtype and t.device == x.device and t.shape == x.shape
                   for t in ts):
            return None
        self._note("irradiance", len(x_edges) - 1, len(y_edges) - 1, int(x.numel()))
        return bin_irradiance(x, y, power, x_edges, y_edges, z=z, frame=frame)

    def fft_pupil(self, opd_waves, intensity, cell_ray, num_rays: int, grid_size: int):
        """Padded complex pupil function of one wavelength in one pass (olb_fft_pupil_*); None to decline."""
        from .psf import fft_pupil

        if not (self.accepts_tensor(opd_waves) and self.accepts_tensor(intensity)):
            return None
        self._note("fft_pupil", int(num_rays), int(grid_size))
        return fft_pupil(opd_waves, intensity, cell_ray, num_rays, grid_size)

    def fft_psf_accumulate(self, amp, psf, first: bool, last: bool, div: float, mul: float):
        """|spectrum|^2 + fftshift + sum over wavelengths + normalisation in one pass (olb_fft_psf_accumulate_*)."""
        from .psf import fft_psf_accumulate

        self._note("fft_psf", int(amp.shape[-1]))
        return fft_psf_accumulate(amp, psf, first, last, div, mul)

    def trace_grad(self, table: T.SurfaceTable, params, rays, coefs=None):
        """Differentiable trace of Optiland's ``rays``: records are autograd outputs of ``params`` and of
        the ray tensors.  None if the table is outside olb_trace_bwd_*'s scope."""
        from . import autograd as AG

        dt = self.device_table(table, rays.x.device)
        if not dt.c.bwd_supported:
            return None
        self._note("grad", table.num_surfaces, int(rays.x.numel()))
        ins = [getattr(rays, k) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")]
        # one (N,) output per (quantity, row): the backward pass then touches only the rows the loss reads
        # (a dense (S, N) output would make autograd zero-fill and the kernel re-read every row), and ``dt``
        # -- packed from the same live values ``params`` was read from -- is reused instead of re-preparing
        S = table.num_surfaces
        outs = AG._TraceFn.apply(table, [dt], tuple(range(S)), params, coefs, *ins)
        rec = {k: list(outs[j * S:(j + 1) * S]) for j, k in enumerate(("x", "y", "z", "L", "M", "N", "intensity", "opd"))}
        for k, key in (("x", "x"), ("y", "y"), ("z", "z"), ("L", "L"), ("M", "M"), ("N", "N"), ("i", "intensity"), ("opd", "opd")):
            setattr(rays, k, rec[key][-1])
        return rec


def _prepare(engine, table, device) -> None:
    """Prepare + upload ``table`` now (cached by content) so that a table the library rejects -- OLB_ERR_TABLE /
    OLB_ERR_UNSUPPORTED from olb_table_upload -- surfaces as an OlbError HERE, inside the caller's try block, and
    turns into a decline rather than an exception out of the reference's trace call."""
    dt = getattr(engine, "device_table", None)
    if dt is not None:
        dt(table, device)


_launch_cache: OrderedDict = OrderedDict()
_dist_cache: OrderedDict = OrderedDict()
_DETERMINISTIC_DISTRIBUTIONS = ("hexapolar", "uniform", "line_x", "line_y", "positive_line_x", "positive_line_y", "cross", "ring")


def _distribution(be, name: str, num_rays):
    """``create_distribution(name).generate_points(num_rays)`` (optiland/distribution.py:415-446), memoised for the
    deterministic patterns: the reference regenerates the same pupil grid on every ``Optic.trace`` call -- a Python loop
    over the rings of a hexapolar pattern (distribution.py:209-220), 64 iterations for SpotDiagram's 64 rings, 1 154
    for a 4 M-ray pupil -- which costs more than the fused launch it feeds.  The arrays are shared read-only (no
    consumer mutates ``distribution.x`` in place)."""
    from optiland.distribution import create_distribution

    if name not in _DETERMINISTIC_DISTRIBUTIONS:
        d = create_distribution(name)
        d.generate_points(num_rays)
        return d
    key = (name, int(num_rays), str(be.get_precision()), str(be.get_device()) if hasattr(be, "get_device") else "")
    d = _dist_cache.get(key)
    if d is None:
        d = create_distribution(name)
        d.generate_points(num_rays)
        _dist_cache[key] = d
        while len(_dist_cache) > 32:
            _dist_cache.popitem(last=False)
    else:
        _dist_cache.move_to_end(key)
    return d


def _object_key(obj) -> tuple:
    """What a finite object contributes to the launch state (its pose and shape are not part of the traced table)."""
    from .pack import _f

    if bool(obj.is_infinite):
        return ()
    g = obj.geometry
    cs = g.cs
    return (type(g).__name__, _f(cs.x), _f(cs.y), _f(cs.z), _f(cs.rx), _f(cs.ry), _f(cs.rz),
            _f(getattr(g, "radius", float("inf"))), _f(getattr(g, "k", 0.0)))


def _launch_scalars_cached(be, optic, table, hx: float, hy: float) -> dict:
    """``pack.launch_scalars`` memoised on everything it depends on.

    The scalars (entrance-pupil position / diameter, the object-space offset, the object point of a finite-object
    field) come from the reference's own paraxial layer -- ``optic.paraxial.EPL() / EPD()``,
    ``field_definition.get_ray_origins`` -- which walks the surface list in Python several times per call
    (``SurfaceGroup.positions`` alone builds a RealRays object per surface): ~15 ms per ``Optic.trace`` on the
    Double-Gauss, two orders of magnitude more than the fused launch it parameterises.  They are pure functions of the
    system prescription (the packed table's bytes: poses, curvatures, media), the system aperture, the field
    definition / field list with its vignetting factors, the primary wavelength and the field point, so that is the
    key; any change to the live objects changes the key."""
    from .pack import _f, launch_scalars

    try:
        ap = optic.aperture
        fd = optic.fields.field_definition
        key = (table.content_key(), type(ap).__name__, _f(ap.value), type(fd).__name__,
               tuple((_f(f.x), _f(f.y), _f(f.vx), _f(f.vy)) for f in optic.fields.fields),
               float(optic.primary_wavelength), bool(optic.obj_space_telecentric), bool(optic.object_surface.is_infinite),
               _object_key(optic.object_surface), float(hx), float(hy), str(be.get_precision()))
    except Exception:      # an attribute this build of the reference does not have: no caching
        return launch_scalars(optic, hx, hy)
    sc = _launch_cache.get(key)
    if sc is None:
        with _ParaxialMemo():          # EPL / EPD / offset each walk the positions and trace paraxially: once per call
            sc = launch_scalars(optic, hx, hy)
        _launch_cache[key] = sc
        while len(_launch_cache) > 256:
            _launch_cache.popitem(last=False)
    else:
        _launch_cache.move_to_end(key)
    return dict(sc)


def _unique_wavelengths(w):
    """Distinct wavelengths of the batch (exact values), or None if there are too many."""
    import torch

    if w.numel() == 0:
        return None
    w = w.detach()
    lo, hi = torch.aminmax(w)
    if bool(lo == hi):
        return np.array([float(lo)], dtype=np.float64)
    u = torch.unique(w)
    if u.numel() > T.MAX_WAVELENGTHS:
        return None
    return u.double().cpu().numpy()


def _set_pre_interaction_direction(rays, table, rec, first, last, launch_dir):
    """rays.L0/M0/N0: direction before the last interaction, in the last surface's local frame
    (optiland/rays/real_rays.py:170-172).  It equals the direction recorded after the previous
    surface (or the launch direction), rotated into that frame -- no kernel output needed."""
    if last - first >= 2:
        Lg, Mg, Ng = rec["L"][-2], rec["M"][-2], rec["N"][-2]
    else:
        Lg, Mg, Ng = launch_dir
    s = table.surfaces[last - 1]
    if s.kind == T.GEOM_NOOP:
        return
    if s.rotated:
        R = s.R
        L0 = R[0, 0] * Lg + R[1, 0] * Mg + R[2, 0] * Ng
        M0 = R[0, 1] * Lg + R[1, 1] * Mg + R[2, 1] * Ng
        N0 = R[0, 2] * Lg + R[1, 2] * Mg + R[2, 2] * Ng
    else:
        L0, M0, N0 = Lg, Mg, Ng
    rays.L0, rays.M0, rays.N0 = L0, M0, N0


def _tail_propagate(be, rays, last_surface, wavelengths, w=None) -> None:
    """Tail of ``RealRayTracer.trace`` / ``trace_generic`` (raytrace/real_ray_tracer.py:105-110, :145-152): propagate
    the traced rays by the image surface's ``thickness`` through ``material_post``.

    The reference's ``HomogeneousPropagation.propagate`` (propagation/homogeneous.py:30-57) asks the material for
    ``k(rays.w)`` with the PER-RAY wavelength array, whose cache key is ``tuple(np.ravel(to_numpy(w)))``
    (materials/base.py:73-79): a device-to-host copy and a 10^7-element Python tuple per call.  The same arithmetic
    with k looked up per DISTINCT wavelength (the values the kernel's table holds), and nothing at all for the usual
    thickness 0 in a transparent medium (x + 0 L == x).  Other propagation models run the reference's own code."""
    pm = last_surface.material_post.propagation_model
    if type(pm).__name__ != "HomogeneousPropagation":
        pm.propagate(rays, last_surface.thickness)
        return
    t = last_surface.thickness
    t_val = float(np.asarray(be.to_numpy(t)).reshape(-1)[0])
    ks = [float(np.asarray(be.to_numpy(last_surface.material_post.k(float(wl)))).reshape(-1)[0]) for wl in wavelengths]
    if t_val != 0.0 or getattr(t, "requires_grad", False):
        rays.x = rays.x + t * rays.L
        rays.y = rays.y + t * rays.M
        rays.z = rays.z + t * rays.N
    if any(k > 0 for k in ks) and t_val != 0.0:
        if len(ks) == 1 or w is None:
            alpha = 4 * np.pi * ks[0] / float(wavelengths[0])
            rays.i = rays.i * be.exp(-alpha * t * 1e3 * be.ones_like(rays.i))
        else:
            k = be.zeros_like(rays.i)
            for wl, kv in zip(wavelengths, ks):
                k = be.where(w == wl, kv * be.ones_like(k), k)
            rays.i = rays.i * be.exp(-(4 * np.pi * k / w) * t * 1e3)
    if not rays.is_normalized:
        rays.normalize()


def _pol_state(be, optic):
    """(polarized, state) of ``optic.polarization`` (optic/optic.py:189-207): (False, False) for "ignore";
    (True, None) for unpolarized light; (True, (Ex, Ey, phase_x, phase_y)) for a polarized state."""
    if optic.polarization == "ignore":
        return False, False
    st = optic.polarization_state
    if not st.is_polarized:
        return True, None

    def f(v):
        return float(np.asarray(be.to_numpy(v)).reshape(-1)[0])

    return True, (f(st.Ex), f(st.Ey), f(st.phase_x), f(st.phase_y))


def _apodization_factor(be, engine, optic, Px, Py):
    """Per-ray launch intensity of an apodized pupil (``RayGenerator.generate_rays``, rays/ray_generator.py:83-87:
    ``apodization.get_intensity(Px, Py)``), or None without apodization; False when it cannot be used on the device."""
    if not optic.apodization:
        return None
    a = optic.apodization.get_intensity(Px, Py)
    if not engine.accepts_tensor(a) or a.shape != Px.shape or a.dtype != Px.dtype:
        return False
    return a


def _apply_apodization(rec, apod) -> None:
    """The kernel launches with unit intensity; every operation on the intensity along the path is a multiplication
    (absorption, coating transmittance, the polarized epilogue's sum |P E|^2 i0) or a reset to 0 (clipping), so the
    records of an apodized launch are the unit-intensity records times the per-ray factor: one pass over the (S, N)
    intensity rows instead of a per-ray intensity input to the launch.  (Out of place: the polarized epilogue's
    result may alias the last intensity row.)"""
    if apod is None:
        return
    if "i_pol" in rec:
        rec["i_pol"] = rec["i_pol"] * apod
    rec["intensity"] = rec["intensity"] * apod


def _make_rays(be, rec, wl_arr, polarized: bool):
    """The reference's ray object for a fused launch: ``RealRays``, or ``PolarizedRays`` carrying the kernel's P
    matrices, the updated intensity and the launch state update_intensity / get_exit_fields refer to
    (rays/polarized_rays.py:47-55; record row 0 is the object surface's record of the launch state)."""
    from optiland.rays import PolarizedRays, RealRays

    if not polarized:
        rays = RealRays(rec["x"][-1], rec["y"][-1], rec["z"][-1], rec["L"][-1], rec["M"][-1], rec["N"][-1],
                        rec["intensity"][-1], wl_arr)
        rays.opd = rec["opd"][-1]
        return rays
    rays = PolarizedRays.__new__(PolarizedRays)      # (its __init__ would tile an (N, 3, 3) identity first)
    rays.x, rays.y, rays.z = rec["x"][-1], rec["y"][-1], rec["z"][-1]
    rays.L, rays.M, rays.N = rec["L"][-1], rec["M"][-1], rec["N"][-1]
    rays.i, rays.w, rays.opd = rec["i_pol"], wl_arr, rec["opd"][-1]
    rays.p = rec["p"]
    rays._i0 = rec["intensity"][0]
    rays._L0, rays._M0, rays._N0 = rec["L"][0], rec["M"][0], rec["N"][0]
    rays.L0 = rays.M0 = rays.N0 = None
    rays.is_normalized = True
    return rays


def _live_frame(cs, scalar, zero):
    """Effective pose of a (possibly nested) coordinate system as torch values built from its LIVE tensors:
    ``t`` (3,) and ``R`` (3, 3) or None for the identity -- ``get_effective_transform`` (coordinate_system.py:145-165)
    with autograd connectivity.  An angle that is exactly 0 enters as a constant (the reference's localize / globalize
    skip such rotations, ``if self.rz:`` coordinate_system.py:84-104, so it gets no gradient there either)."""
    import torch

    t = torch.stack([scalar(cs.x), scalar(cs.y), scalar(cs.z)])
    ang = [scalar(v) if float(scalar(v).detach()) != 0.0 else zero for v in (cs.rx, cs.ry, cs.rz)]
    R = None
    if any(a is not zero for a in ang):
        rx, ry, rz = ang
        cx, sx, cy, sy, cz, sz = torch.cos(rx), torch.sin(rx), torch.cos(ry), torch.sin(ry), torch.cos(rz), torch.sin(rz)
        R = torch.stack([cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx,
                         sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx,
                         -sy, cy * sx, cy * cx]).reshape(3, 3)
    parent = getattr(cs, "reference_cs", None)
    if parent is None:
        return t, R
    tp, Rp = _live_frame(parent, scalar, zero)
    t_eff = tp + (Rp @ t if Rp is not None else t)
    R_eff = Rp if R is None else (R if Rp is None else Rp @ R)
    return t_eff, R_eff


def _live_params(surfaces, table, wavelength):
    """(S, GP_COUNT) fp64 tensor of the differentiable parameters, built with torch ops FROM THE LIVE
    tensors of the Optiland objects (geometry.cs.x/y/z, geometry.radius, geometry.k,
    geometry.coefficients, material_pre/post.n(lambda)) so that gradients flow back to whatever leaves
    the optimiser owns (optic/optic_updater.py:38-157).  None if a surface is outside the adjoint's scope."""
    import torch

    from .autograd import GP_COEF, GP_CONIC, GP_COUNT, GP_CURV, GP_MAX_COEF, GP_N1, GP_N2, GP_R, GP_TX
    from .pack import catalogue_value

    def scalar(v, like):
        # (dtype given: torch.as_tensor(<Python float>) would be float32 -- a parameter set as a plain number,
        # e.g. by optic.updater.set_radius(22.89, 1), must not lose 8 digits on its way into the fp64 table)
        t = v if torch.is_tensor(v) else torch.as_tensor(float(v), dtype=torch.float64)
        return t.to(dtype=torch.float64, device=like.device).reshape(())

    like = None
    for surf in surfaces:
        r = getattr(getattr(surf, "geometry", None), "radius", None)
        if torch.is_tensor(r):
            like = r
            break
    if like is None:
        like = torch.zeros(())
    zero = torch.zeros((), dtype=torch.float64, device=like.device)
    one = torch.ones((), dtype=torch.float64, device=like.device)
    # ONE stack for all S x GP_COUNT scalars (the curvature column first holds the RADIUS, or 1 where the
    # curvature is zero), then one vectorised 1/radius: a handful of kernels instead of several per surface
    flat, flat_r = [], []
    for surf, spec in zip(surfaces, table.surfaces):
        vals = [zero] * GP_COUNT
        if spec.interaction != T.INTERACT_REFRACT:
            return None          # phase-profile and grating surfaces: the adjoint has neither interaction
        if spec.kind != T.GEOM_NOOP:
            g = surf.geometry
            cs = g.cs
            if spec.kind not in (T.GEOM_PLANE, T.GEOM_STANDARD, T.GEOM_EVEN_ASPHERE, T.GEOM_ODD_ASPHERE,
                                 T.GEOM_POLYNOMIAL, T.GEOM_ZERNIKE, T.GEOM_CHEBYSHEV, T.GEOM_FORBES_QBFS, T.GEOM_GRID_SAG):
                return None
            # normalisation radii are constants of the adjoint.  One that an optimiser drives (NormalizationRadiusVariable,
            # optimization/variable/norm_radius.py: the value written is an nn.Parameter or computed from one) needs the
            # reference's eager graph; a plain be.array leaf -- every array is one under be.grad_mode -- does not
            # the same rule for a grid's node coordinates and sag values (constants of the adjoint: olb.h has no
            # gradient slot for them)
            # and for the vertices of polygon apertures (the clip mask is a constant of the adjoint)
            for a in ("norm_radius", "norm_x", "norm_y", "x_grid", "y_grid", "sag_grid"):
                v = getattr(g, a, None)
                if getattr(v, "requires_grad", False) and (v.grad_fn is not None or isinstance(v, torch.nn.Parameter)):
                    return None
            # the vertices of polygon apertures are constants too (the clip mask has no gradient).  PolygonAperture
            # always COMPUTES them (column_stack of x and y; scale() multiplies them), so under be.grad_mode they carry
            # a grad_fn without anybody driving them: what declines is an nn.Parameter among the leaves of their graph
            if any(_parameter_driven(v) for v in _polygon_vertices(surf)):
                return None
            nested = cs.reference_cs is not None
            if nested:
                # a frame defined relative to another one (coordinate breaks of imported systems,
                # fileio/zemax/reader/converter.py:120-190): the effective pose t = t_p + R_p t_c, R = R_p R_c
                # (coordinate_system.py:145-165) composed from the LIVE tensors of every level
                t_eff, R_eff = _live_frame(cs, lambda v: scalar(v, like), zero)
            # pose rotation: constants (identity for an untilted surface -- the reference skips zero rotations
            # altogether, `if self.rz:` coordinate_system.py:84-89, so zero angles get no gradient there either);
            # for a tilted pose R = Rz Ry Rx is formed from the LIVE angle tensors (coordinate_system.py:121-143)
            # so that the adjoint kernel's dLoss/dR reaches tilt variables
            if nested:
                if spec.rotated and R_eff is not None:
                    Rm = tuple(R_eff[q // 3, q % 3] for q in range(9))
                else:
                    Rm = (one, zero, zero, zero, one, zero, zero, zero, one)
            elif spec.rotated:
                # (an angle that is exactly 0 is skipped by the reference even on a tilted surface: constant)
                rx, ry, rz = (scalar(v, like) if float(scalar(v, like).detach()) != 0.0 else zero for v in (cs.rx, cs.ry, cs.rz))
                cx, sx, cy, sy, cz, sz = torch.cos(rx), torch.sin(rx), torch.cos(ry), torch.sin(ry), torch.cos(rz), torch.sin(rz)
                Rm = (cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx,
                      sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx,
                      -sy, cy * sx, cy * cx)
            else:
                Rm = (one, zero, zero, zero, one, zero, zero, zero, one)
            for q in range(9):
                vals[GP_R + q] = Rm[q]
            if nested:
                vals[GP_TX], vals[GP_TX + 1], vals[GP_TX + 2] = t_eff[0], t_eff[1], t_eff[2]
            else:
                vals[GP_TX], vals[GP_TX + 1], vals[GP_TX + 2] = scalar(cs.x, like), scalar(cs.y, like), scalar(cs.z, like)
            curved = spec.kind != T.GEOM_PLANE and np.isfinite(spec.radius)
            if spec.kind not in (T.GEOM_PLANE, T.GEOM_GRID_SAG):      # (a grid has no radius and no conic)
                vals[GP_CONIC] = scalar(g.k, like)
            flat_r.append(scalar(g.radius, like) if curved else one)
            # (a catalogue glass is a constant: the packed table already holds its index at this wavelength -- asking the
            # material again would re-evaluate its dispersion formula, pack.catalogue_value)
            for slot, mat, packed in ((GP_N1, surf.material_pre, spec.n1), (GP_N2, surf.material_post, spec.n2)):
                known = catalogue_value(mat, "n", wavelength)
                vals[slot] = scalar(float(packed[0]) if known is not None and len(packed) == 1 else mat.n(wavelength), like)
            if spec.kind in (T.GEOM_EVEN_ASPHERE, T.GEOM_ODD_ASPHERE):
                if len(g.coefficients) > GP_MAX_COEF:
                    return None
                for j, cj in enumerate(g.coefficients):
                    vals[GP_COEF + j] = scalar(cj, like)
            elif spec.kind == T.GEOM_FORBES_QBFS:
                # radial_terms {order n: a_n} (forbes/geometry.py:242-274; ForbesQNormalSlopeCoeffVariable writes
                # geom.radial_terms[n]); missing orders are constant zeros
                terms = g.radial_terms or {}
                if terms and max(int(n_) for n_ in terms) + 1 > GP_MAX_COEF:
                    return None
                for n_, cj in terms.items():
                    vals[GP_COEF + int(n_)] = scalar(cj, like)
            vals[GP_CURV] = one if curved else zero      # selector: 1 -> 1/radius, 0 -> 0
        else:
            flat_r.append(one)
        flat.extend(vals)
    P = torch.stack(flat).reshape(len(table.surfaces), GP_COUNT)
    radius = torch.stack(flat_r)
    curv = P[:, GP_CURV] / radius
    return torch.cat([P[:, :GP_CURV], curv[:, None], P[:, GP_CURV + 1:]], dim=1)


def _polygon_vertices(surf) -> list:
    """The vertex arrays of every polygon in the surface's aperture tree (pack.pack_aperture)."""
    out, stack = [], [getattr(surf, "aperture", None)]
    while stack:
        a = stack.pop()
        if a is None:
            continue
        if type(a).__name__ in ("PolygonAperture", "FileAperture"):
            out.append(getattr(a, "vertices", None))
        stack += [u for u in (getattr(a, "a", None), getattr(a, "b", None)) if hasattr(u, "contains")]
    return out


def _parameter_driven(v) -> bool:
    """True when ``v`` is an nn.Parameter or is computed from one."""
    import torch

    if isinstance(v, torch.nn.Parameter):
        return True
    seen, stack = set(), [getattr(v, "grad_fn", None)]
    while stack:
        fn = stack.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        if isinstance(getattr(fn, "variable", None), torch.nn.Parameter):
            return True
        stack += [f for f, _ in fn.next_functions]
    return False


def _live_coefs(surfaces, table):
    """(S, K) fp64 tensor of the USER coefficients of the polynomial-family surfaces (Zernike ``geometry.zernike.coeffs``,
    polynomial / Chebyshev ``geometry.coefficients``), stacked from the LIVE tensors so that the table gradients of
    olb_trace_bwd_* (grad_tables) flow back to the optimiser's variables (optimization/variable/zernike_coeff.py,
    polynomial_coeff.py, chebyshev_coeff.py); None when the table has no such surface."""
    import torch

    rows, K, dev = [], 0, None
    for surf, spec in zip(surfaces, table.surfaces):
        r = None
        if spec.kind == T.GEOM_ZERNIKE:
            r = surf.geometry.zernike.coeffs
        elif spec.kind in (T.GEOM_POLYNOMIAL, T.GEOM_CHEBYSHEV):
            c = surf.geometry.coefficients
            r = c if torch.is_tensor(c) else torch.stack([torch.stack([
                v.to(torch.float64) if torch.is_tensor(v) else torch.as_tensor(float(v), dtype=torch.float64) for v in row])
                for row in c])
        if r is not None:
            r = (r if torch.is_tensor(r) else torch.as_tensor(np.asarray(r, dtype=np.float64))).reshape(-1).to(torch.float64)
            if spec.kind == T.GEOM_CHEBYSHEV and r.requires_grad:
                # the reference sums over ``argwhere(coefficients != 0)`` (geometries/chebyshev.py:146, 177): a coefficient
                # that is exactly 0 is not part of its graph and receives gradient 0 -- reproduced, not fixed
                r = torch.where(r != 0, r, r.detach())
            K = max(K, r.numel())
            dev = r.device
        rows.append(r)
    if K == 0:
        return None
    out = []
    for r in rows:
        if r is None:
            out.append(torch.zeros(K, dtype=torch.float64, device=dev))
        else:
            out.append(torch.cat([r.to(dev), torch.zeros(K - r.numel(), dtype=torch.float64, device=dev)]) if r.numel() < K else r.to(dev))
    return torch.stack(out)


def _wants_grad(backend, surfaces, rays=None) -> bool:
    """True when the call must stay differentiable: ``be.grad_mode`` is on, or some tensor involved --
    a ray array or a live surface parameter -- requires grad even though the global switch is off (the
    reference's eager ops would build a graph for it regardless)."""
    if backend.grad_mode.requires_grad:
        return True

    def rg(v):
        return bool(getattr(v, "requires_grad", False))

    if rays is not None and any(rg(getattr(rays, k, None)) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")):
        return True
    for surf in surfaces:
        g = getattr(surf, "geometry", None)
        if g is None:
            continue
        cs = g.cs
        vals = [getattr(g, "radius", None), getattr(g, "k", None), cs.x, cs.y, cs.z, cs.rx, cs.ry, cs.rz]
        # ruled-grating scalars (pack.pack_grating) and grid-sag arrays (pack.pack_grid_sag)
        vals += [getattr(g, k, None) for k in ("grating_order", "grating_period", "groove_orientation_angle",
                                               "x_grid", "y_grid", "sag_grid")]
        parent = getattr(cs, "reference_cs", None)
        while parent is not None:                    # nested frames: the pose depends on every level
            vals += [parent.x, parent.y, parent.z, parent.rx, parent.ry, parent.rz]
            parent = getattr(parent, "reference_cs", None)
        rt = getattr(g, "radial_terms", None)        # Forbes Q^bfs: {order: tensor}
        if isinstance(rt, dict):
            vals += list(rt.values())
        ff = getattr(g, "freeform_coeffs", None)     # Forbes Q-2D: {(kind, m, n): tensor} (pack.pack_forbes_q2d)
        if isinstance(ff, dict):
            vals += list(ff.values()) + [getattr(g, "norm_radius", None)]
        coefs = getattr(g, "coefficients", None)     # (Zernike: the property returns geometry.zernike.coeffs)
        if coefs is not None:
            vals += [coefs] if hasattr(coefs, "requires_grad") else list(np.ravel(np.asarray(coefs, dtype=object)))
        pp = getattr(getattr(surf, "interaction_model", None), "phase_profile", None)
        if pp is not None:                           # phase-profile terms (pack.pack_phase_profile)
            vals += [getattr(pp, k, None) for k in ("phase", "_K_x", "_K_y")]
            pc = getattr(pp, "coefficients", None)
            if pc is not None:
                vals += [pc] if hasattr(pc, "requires_grad") else list(np.ravel(np.asarray(pc, dtype=object)))
        vals += _polygon_vertices(surf)              # polygon apertures (pack.pack_aperture)
        jones = getattr(getattr(getattr(surf, "interaction_model", None), "coating", None), "jones", None)
        if jones is not None:                        # thin-film thicknesses, retardance (pack.pack_jones_coating)
            vals += [getattr(layer, "thickness_um", None) for layer in getattr(getattr(jones, "stack", None), "layers", [])]
            vals += [getattr(jones, "retardance", None), getattr(jones, "axis", None)]
        if any(rg(v) for v in vals):
            return True
    return False


def _trace_grad_per_wavelength(engine, surfaces, rays, table_builder, wl):
    """Differentiable trace of a batch that mixes several wavelengths (``trace_generic`` with a per-ray wavelength
    array while gradients are wanted).  The adjoint kernel works on one medium table per call, and the indices
    n(lambda_j) are DIFFERENT differentiable functions of the live material tensors (``AbbeMaterial.index / abbe``,
    ``IdealMaterial.index``), so the batch is split by wavelength: one forward + one adjoint launch per wavelength on
    the rays that carry it, each with its own live parameter block, and the records are put back in the caller's ray
    order by one differentiable gather per (quantity, row).  Returns the record dict of per-row tensors, or None when
    some wavelength's table is outside the adjoint's scope (nothing has been modified then)."""
    import torch

    from types import SimpleNamespace

    w = rays.w.detach()
    keys = ("x", "y", "z", "L", "M", "N", "i", "opd")
    groups = []
    for wj in wl:
        idx = torch.nonzero(w == float(wj)).reshape(-1)
        table_j = table_builder(np.array([float(wj)], dtype=np.float64))
        _prepare(engine, table_j, rays.x.device)
        params = _live_params(surfaces, table_j, float(wj))
        if params is None:
            return None
        groups.append((idx, table_j, params, _live_coefs(surfaces, table_j)))
    parts = []
    for idx, table_j, params, coefs in groups:
        sub = SimpleNamespace(**{k: getattr(rays, k)[idx] for k in keys}, w=rays.w[idx])
        rec_j = engine.trace_grad(table_j, params, sub, coefs) if coefs is not None else engine.trace_grad(table_j, params, sub)
        if rec_j is None:
            return None
        parts.append(rec_j)
    # position of every original ray inside the concatenation of the groups
    order = torch.cat([g[0] for g in groups])
    inv = torch.empty_like(order)
    inv[order] = torch.arange(order.numel(), device=order.device)
    S = len(surfaces)
    rec = {}
    for key in ("x", "y", "z", "L", "M", "N", "intensity", "opd"):
        rec[key] = [torch.cat([p[key][row] for p in parts])[inv] for row in range(S)]
    for k, key in (("x", "x"), ("y", "y"), ("z", "z"), ("L", "L"), ("M", "M"), ("N", "N"), ("i", "intensity"), ("opd", "opd")):
        setattr(rays, k, rec[key][-1])
    return rec


def _trace_check(rays, table_builder):
    """What every trace of ``rays`` through the capability needs: returns ``(table, wavelengths)``, or the reason (a
    str) to decline.  ``table_builder(wavelengths)`` packs the surfaces.  Shared by ``_try_trace`` and the device ray
    aimer, which launches on the table a subset trace would use."""
    polarized = type(rays).__name__ == "PolarizedRays"
    if type(rays).__name__ != "RealRays" and not polarized:
        return f"ray class {type(rays).__name__}"  # ParaxialRays etc.: reference path
    engine = _state["engine"]
    if not engine.accepts(rays):
        return "rays not resident on a CUDA device (or not fp32/fp64)"
    if not getattr(rays, "is_normalized", True):
        # a previous surface left un-normalised direction cosines (thin_lens_interaction_model.py:111) and
        # HomogeneousPropagation.propagate would renormalise them first (propagation/homogeneous.py:55-56); the
        # kernel assumes unit directions
        return "rays.is_normalized is False"
    wl = _unique_wavelengths(rays.w)
    if wl is None:
        return f"more than {T.MAX_WAVELENGTHS} distinct wavelengths"
    try:
        table = table_builder(wl)
        _prepare(engine, table, rays.x.device)         # upload errors (OlbError) decline as well
    except _PACK_ERRORS as e:
        return f"unsupported: {e}"
    if not polarized and any(s.coating == T.COAT_FRESNEL for s in table.surfaces):
        # the reference raises for this combination (ray_generator.py:90-94)
        return "Fresnel coating with unpolarized rays"
    if not polarized and any(s.coating in T.JONES_COATINGS for s in table.surfaces):
        # the reference's ray generator raises for these too (ray_generator.py:90-94); RealRays pass them unchanged
        return "thin-film, polarizer or retarder coating with unpolarized rays"
    return table, wl


def _try_trace(backend, surfaces, rays, table_builder) -> bool:
    """Common body of the two wrappers.  ``surfaces``: the Surface objects to be traced (in
    order); ``table_builder(wavelengths)`` packs them.  Returns False to decline."""
    polarized = type(rays).__name__ == "PolarizedRays"
    checked = _trace_check(rays, table_builder)
    if isinstance(checked, str):
        return _decline(checked)
    table, wl = checked
    engine = _state["engine"]
    if any(s.bsdf != T.BSDF_NONE for s in table.surfaces):
        if polarized:
            return _decline("BSDF scatter with polarized rays")
        if _wants_grad(backend, surfaces, rays):
            # the reference's eager path then runs its numba scatter (which does not take torch tensors)
            return _decline("gradients wanted: BSDF scatter")
    launch_dir = (rays.L, rays.M, rays.N)
    if _wants_grad(backend, surfaces, rays):
        # gradients wanted: the records must be autograd outputs of the live parameter tensors
        # (optimization/operand/ray.py:299-342 differentiates through a recorded row).  One custom
        # Function (forward kernel + adjoint kernel) replaces the eager graph; tables outside the
        # adjoint's scope go back to the reference's eager path.
        if polarized:
            return _decline("gradients wanted: polarized rays")
        if table.n_wl != 1:
            try:
                rec = _trace_grad_per_wavelength(engine, surfaces, rays, table_builder, wl)
            except _PACK_ERRORS as e:
                return _decline(f"unsupported: {e}")
            if rec is None:
                return _decline("gradients wanted: a surface / table outside the adjoint's scope")
        else:
            # (inside one aiming call the live tensors do not change either: one parameter block, one graph node)
            params = _frozen(("params", id(table)), table, lambda: _live_params(surfaces, table, float(wl[0])))
            if params is None:
                return _decline("gradients wanted: a surface outside the adjoint's scope")
            coefs = _frozen(("coefs", id(table)), table, lambda: _live_coefs(surfaces, table))
            rec = engine.trace_grad(table, params, rays, coefs) if coefs is not None else engine.trace_grad(table, params, rays)
            if rec is None:
                return _decline("gradients wanted: table outside the adjoint's scope")
    else:
        rec = engine.trace(table, rays, 0, table.num_surfaces)
    for row, surf in enumerate(surfaces):
        for attr, key in _REC_ATTR:
            setattr(surf, attr, rec[key][row])
    _set_pre_interaction_direction(rays, table, rec, 0, table.num_surfaces, launch_dir)
    return True


def _capture_warnings(caught) -> list:
    """``warnings.catch_warnings(record=True)`` records as (message, category, filename, lineno, module name, registry):
    enough to issue each again as the original ``warnings.warn`` call issued it, through the same filters and the
    once-per-location registry of the module it was attributed to."""
    by_file = {getattr(m, "__file__", None): m for m in list(sys.modules.values())}
    out = []
    for w in caught:
        mod = by_file.get(w.filename)
        reg = mod.__dict__.setdefault("__warningregistry__", {}) if mod is not None else None
        out.append((w.message, w.category, w.filename, w.lineno, getattr(mod, "__name__", None), reg))
    return out


class _DeviceAimSolver:
    """The solves of ONE ``RobustRayAimer.aim_rays`` call on the device.  Each is what ``IterativeRayAimer.aim_rays(...,
    initial_guess=guess)`` computes (rays/ray_aiming/iterative.py:60-281) as ONE ``engine.aim`` launch plus one status
    read.  The stop radius and the paraxial Jacobian factor depend on the optic alone, which does not change during the
    call (the premise of _FrozenTables), so they are computed once; warnings the stop-radius strategy issued are issued
    again on every solve, as the reference recomputes the radius per solve."""

    def __init__(self, engine, table, r_stop, J_factor, tol, max_iter, infinite, warned):
        self.engine, self.table = engine, table
        self.r_stop, self.J_factor, self.tol, self.max_iter, self.infinite = r_stop, J_factor, tol, max_iter, infinite
        self.warned = warned
        self.wavelengths = None

    def solve(self, pupil, guess):
        """The solution (x, y, z, L, M, N) for the pupil targets ``pupil`` from ``guess``, or None where the reference
        raises ValueError (NaN start, not converged, a freeform range error)."""
        import warnings

        import torch

        import optiland.backend as be

        for message, category, filename, lineno, module, registry in self.warned:
            warnings.warn_explicit(message, category, filename, lineno, module=module, registry=registry)
        ts = torch.broadcast_tensors(*[be.as_array_1d(v).detach() for v in guess])
        dt, n = ts[0].dtype, ts[0].numel()

        def fresh(t):               # a new, contiguous (hence 16-byte aligned) array: the caller's guess is not written
            return t.detach().to(dt).expand(n).clone(memory_format=torch.contiguous_format)

        sol = {k: fresh(t) for k, t in zip(("x", "y", "z", "L", "M", "N"), ts)}
        if self.table.n_wl > 1:
            sol["w"] = fresh(be.as_array_1d(self.wavelengths))
        Px, Py = (fresh(be.as_array_1d(p)) for p in pupil)
        status = self.engine.aim(self.table, sol, Px, Py, self.r_stop, self.J_factor, self.tol, self.max_iter,
                                 self.infinite)
        if status:
            return None
        return sol["x"], sol["y"], sol["z"], sol["L"], sol["M"], sol["N"]


def _device_aim_solver(backend, aimer, probe, wavelengths):
    """The ``_DeviceAimSolver`` of one ``RobustRayAimer.aim_rays`` call, or None to run the reference's body: an engine
    without ``aim``, gradients wanted (the eager Broyden loop over the adjoint), or a subset table the capability declines
    (the same checks as every trace, ``_trace_check``, on the table ``aimer_trace_subset`` would launch).  ``probe``: a
    launch state of the call's rays (the first guess)."""
    import warnings

    import optiland.backend as be
    from optiland.rays import RealRays
    from optiland.rays.ray_aiming.initialization import get_stop_radius_strategy

    engine = _state["engine"]
    if not hasattr(engine, "aim"):
        return None
    optic = aimer.optic
    group = optic.surfaces
    stop = group.stop_index
    infinite = bool(getattr(optic.object_surface, "is_infinite", False))
    start = 1 if infinite else 0
    surfaces = list(group.surfaces)[start:stop + 1]
    if not surfaces:
        return None
    x, y, z, L, M, N = (be.as_array_1d(v) for v in probe)
    rays = RealRays(x, y, z, L, M, N, intensity=be.ones_like(x), wavelength=wavelengths)
    if _wants_grad(backend, surfaces, rays):
        _decline("robust ray aiming: gradients wanted")
        return None
    checked = _trace_check(rays, _group_table_builder(group, start, stop + 1))
    if isinstance(checked, str):
        return None                     # the reference's body runs; its subset traces decline with this reason
    table = checked[0]
    if any(s.bsdf != T.BSDF_NONE for s in table.surfaces):
        _decline("robust ray aiming: BSDF surface before the stop")
        return None
    if any(s.kind == T.GEOM_FORBES_Q2D for s in table.surfaces):
        _decline("robust ray aiming: Forbes Q-2D surface before the stop")
        return None
    if table.surfaces[-1].kind == T.GEOM_NOOP:
        return None                     # the stop is the object surface: it has no local frame in the kernel
    it = aimer._iterative
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        r_stop = float(get_stop_radius_strategy(optic, "iterative").calculate_stop_radius())
    wl_mean = be.mean(wavelengths) if hasattr(wavelengths, "__len__") else wavelengths
    J_factor = it._get_paraxial_jacobian(float(wl_mean), stop, infinite)
    if abs(J_factor) < 1e-12:
        J_factor = 1e-12
    solver = _DeviceAimSolver(engine, table, r_stop, float(J_factor), it.tol, it.max_iter, infinite,
                              _capture_warnings(caught))
    solver.wavelengths = wavelengths
    return solver


def _robust_aim_device(backend, aimer, fields, wavelengths, pupil_coords, initial_guess):
    """``RobustRayAimer.aim_rays`` (rays/ray_aiming/robust.py:61-171) with every solve on the device (one launch and one
    status read each, ``_DeviceAimSolver``); the paraxial guesses, the predictor and the interval halving are the
    reference's.  None: the reference's body runs instead (``_device_aim_solver``).

    Side effect: afterwards the surfaces hold the records of the stop-radius strategy's one-ray trace, not those of the
    last subset trace as after the reference's body.  Every caller in the reference traces again before it reads
    records."""
    def paraxial_at(t):                 # targets and paraxial solution at continuation parameter t
        pt = (pupil_coords[0] * t, pupil_coords[1] * t)
        ft = (fields[0] * t, fields[1] * t) if aimer.scale_fields else fields
        return pt, aimer._paraxial.aim_rays(ft, wavelengths, pt)

    anchor = paraxial_at(0.0)[1] if initial_guess is None else None
    solver = _device_aim_solver(backend, aimer, initial_guess if initial_guess is not None else anchor, wavelengths)
    if solver is None:
        return None
    if initial_guess is not None:
        sol = solver.solve(pupil_coords, initial_guess)
        if sol is not None:
            return sol
        anchor = paraxial_at(0.0)[1]
    return _robust_interval(aimer, solver, paraxial_at, 0.0, 1.0, anchor, anchor)


def _robust_interval(aimer, solver, paraxial_at, t0, t1, sol0, par0):
    """``RobustRayAimer._solve``: the solution at t1 from the one at t0, halving [t0, t1] where a solve fails."""
    import optiland.backend as be

    if (t1 - t0) < 1e-3:
        return sol0
    pt, par1 = paraxial_at(t1)
    # predictor: the paraxial solution at t1 plus the real - paraxial difference at t0
    xg, yg, zg, Lg, Mg = (p1 + (s0 - p0) for p1, s0, p0 in zip(par1[:5], sol0[:5], par0[:5]))
    sq = Lg**2 + Mg**2
    if be.any(sq > 1.0):                # one decision for the whole batch, as in the reference
        f = be.sqrt(sq)
        Lg, Mg = Lg / f, Mg / f
        sq = Lg**2 + Mg**2
    Ng = be.sqrt(1.0 - sq)
    Ng = be.where(par1[5] >= 0, Ng, -Ng)
    if getattr(aimer.optic.object_surface, "is_infinite", False):
        Lg, Mg, Ng = par1[3], par1[4], par1[5]   # the field angle fixes the direction
    sol = solver.solve(pt, (xg, yg, zg, Lg, Mg, Ng))
    if sol is not None:
        return sol
    tm = (t0 + t1) / 2.0
    sol_m = _robust_interval(aimer, solver, paraxial_at, t0, tm, sol0, par0)
    return _robust_interval(aimer, solver, paraxial_at, tm, t1, sol_m, paraxial_at(tm)[1])


def _group_table_builder(surface_group, start: int, stop: int):
    """``table_builder`` of surfaces [start, stop) of a SurfaceGroup: the whole group packed, then sliced (memoised
    inside a _FrozenTables context)."""
    def build(wl):
        def pack():
            full = pack_surface_group(surface_group, wl)
            return T.SurfaceTable(full.surfaces[start:stop], full.wavelengths)

        return _frozen(("group", id(surface_group), start, stop, tuple(float(w) for w in wl)), surface_group, pack)

    return build


def install(engine=None, alias: str | None = None) -> None:
    """Register the backend and wrap the two trace entry points (idempotent)."""
    import optiland.backend as be
    from optiland.backend.torch_backend import TorchBackend
    from optiland.surfaces.standard_surface import Surface
    from optiland.surfaces.surface_group import SurfaceGroup

    if _state["installed"]:
        if engine is not None:
            _state["engine"] = engine
        return
    _state["engine"] = engine if engine is not None else CudaEngine()

    class B200TorchBackend(TorchBackend):
        """TorchBackend + one capability: the fused CUDA trace loop."""

        def trace_surfaces(self, surface_group, rays, start: int, stop: int) -> bool:
            surfaces = list(surface_group.surfaces)[start:stop]
            if not surfaces:
                return False
            return _try_trace(self, surfaces, rays, _group_table_builder(surface_group, start, stop))

        def trace_optic(self, tracer, Hx, Hy, wavelength, num_rays, distribution):
            """``RealRayTracer.trace`` for ONE field with the launch state generated on the device
            (SURVEY.md 8f-1): returns the traced rays or None to decline.  Covers what
            ``RayGenerator.generate_rays`` + ``ParaxialRayAimer`` + ``field_definition.get_ray_origins`` do for one
            field point (infinite-object angle field, finite object with an object-height / angle field,
            object-space telecentric system), apodized or not; with ``optic.polarization`` set the rays are
            ``PolarizedRays`` (Fresnel coatings included) and ``update_intensity`` runs as the kernel's epilogue."""
            import numpy as _np

            from .launch import pupil_affine

            optic = tracer.optic
            if getattr(_tls, "in_reference", False) or _wants_grad(self, list(optic.surfaces.surfaces)):
                return None
            try:
                hx, hy = float(_np.asarray(be.to_numpy(be.atleast_1d(Hx))).reshape(-1)[0]), \
                    float(_np.asarray(be.to_numpy(be.atleast_1d(Hy))).reshape(-1)[0])
                single = be.size(be.atleast_1d(Hx)) == 1 and be.size(be.atleast_1d(Hy)) == 1
            except Exception:
                return _fused_decline("field coordinates are not plain numbers")
            if not single:
                return _fused_decline("several field points in one Optic.trace call")
            # the aimer is (re)configured lazily inside generate_rays from this dict (ray_generator.py:67-71)
            if getattr(tracer, "ray_aiming_config", {}).get("mode", "paraxial") != "paraxial":
                return _fused_decline("non-paraxial ray aiming")
            tracer._validate_normalized_coordinates(Hx, Hy, "field")
            if isinstance(distribution, str):
                distribution = _distribution(be, distribution, num_rays)
            Px, Py = distribution.x, distribution.y
            engine = _state["engine"]
            if not (engine.accepts_tensor(Px) and engine.accepts_tensor(Py)):
                return _fused_decline("pupil samples not resident on a CUDA device (or not fp32/fp64)")
            apod = _apodization_factor(be, engine, optic, Px, Py)      # (the UNSCALED pupil: real_ray_tracer.py:86-101)
            if apod is False:
                return _fused_decline("apodization factor not resident on the device")
            polarized, state = _pol_state(be, optic)
            try:
                table = pack_surface_group(optic.surfaces, [float(wavelength)])
                sc = _launch_scalars_cached(be, optic, table, hx, hy)
                _prepare(engine, table, Px.device)
            except _PACK_ERRORS as e:
                return _fused_decline(f"unsupported: {e}")
            if not polarized and any(s.coating in T.POLARIZING_COATINGS for s in table.surfaces):
                return None          # the reference raises for this combination (ray_generator.py:90-94)
            if polarized and any(s.bsdf != T.BSDF_NONE for s in table.surfaces):
                return _fused_decline("BSDF scatter with polarized rays")
            if table.surfaces[0].kind != T.GEOM_NOOP:
                return _fused_decline("first surface is not an object surface")
            rec = engine.trace_pupil(table, Px, Py, pupil_affine(sc), polarization=state) if polarized else \
                engine.trace_pupil(table, Px, Py, pupil_affine(sc))
            _apply_apodization(rec, apod)
            _reset_records(be, optic.surfaces)
            for row, surf in enumerate(optic.surfaces.surfaces):
                for attr, key in _REC_ATTR:
                    setattr(surf, attr, rec[key][row])
            rays = _make_rays(be, rec, be.ones_like(rec["x"][-1]) * wavelength, polarized)
            _set_pre_interaction_direction(rays, table, rec, 0, table.num_surfaces,
                                           (rec["L"][0], rec["M"][0], rec["N"][0]))
            # tail of RealRayTracer.trace (raytrace/real_ray_tracer.py:105-118); update_intensity already ran in-kernel
            # (it overwrites rays.i from P and the launch intensity alone, so the order with the propagate is immaterial
            # unless the image space absorbs -- then the reference's own order is restored below)
            if optic.image_surface:
                i_before = rays.i
                _tail_propagate(be, rays, optic.surfaces[-1], [float(wavelength)])
                if polarized and rays.i is not i_before:
                    rays.i = i_before
            return rays

        def trace_optic_generic(self, tracer, Hx, Hy, Px, Py, wavelength):
            """``RealRayTracer.trace_generic`` (raytrace/real_ray_tracer.py:120-154) for per-ray (Hx, Hy, Px, Py[, lambda])
            arrays with the launch state generated on the device.  Needs the paraxial aimer (apodized pupils and
            vignetting factors are served, also together);
            ``optic.polarization`` set -> ``PolarizedRays`` (config 5's call shape).  Returns the traced rays or None."""
            import numpy as _np

            from .launch import pupil_affine_fields
            from .pack import launch_scalars

            optic = tracer.optic
            engine = _state["engine"]
            if getattr(_tls, "in_reference", False) or _wants_grad(self, list(optic.surfaces.surfaces)):
                return None
            if getattr(tracer, "ray_aiming_config", {}).get("mode", "paraxial") != "paraxial":
                return _fused_decline("non-paraxial ray aiming")
            try:
                has_vig = bool(_np.any(_np.asarray(be.to_numpy(optic.fields.vx)) != 0)
                               or _np.any(_np.asarray(be.to_numpy(optic.fields.vy)) != 0))
            except Exception:
                return _fused_decline("vignetting factors are not plain numbers")
            tracer._validate_normalized_coordinates(Hx, Hy, "field")
            tracer._validate_normalized_coordinates(Px, Py, "pupil")
            vig = None
            if has_vig:
                # vignetting factors (nearest-neighbour over the defined fields, fields/field_group.py:93-122) scale
                # the pupil point TWICE on this path: once in trace_generic (real_ray_tracer.py:134-137) and once
                # more in the aimer (ray_aiming/paraxial.py:72-96) -- reproduced, looked up per ray IN the kernel
                # from the table of defined fields (OlbPupilLaunch.vig, vig_power = 2)
                try:
                    from .pack import _f

                    mf = _f(optic.fields.max_field)
                    norm = mf if mf != 0 else 1.0
                    vig = (_np.array([[_f(f.x) / norm, _f(f.y) / norm, _f(f.vx), _f(f.vy)] for f in optic.fields.fields]), 2)
                    if len(vig[0]) > 16:
                        vig = None
                except Exception:
                    vig = None
                if vig is None:      # (more than 16 fields, exotic field objects): the factors as eager ops
                    vxf, vyf = optic.fields.get_vig_factor(Hx, Hy)
                    Px = Px * (1 - vxf) * (1 - vxf)
                    Py = Py * (1 - vyf) * (1 - vyf)
            Hx, Hy, Px, Py = tracer._validate_array_size(Hx, Hy, Px, Py)
            # _validate_array_size expands Python numbers only; a 0-d / 1-element ARRAY among longer ones (np.float32
            # field coordinates, be.array(0.7), ...) is left to the broadcasting of the reference's element-wise ops
            # (ray_generator.py:47-99).  Same values here: sizes 1 and n are brought to (n,) before the launch.
            try:
                sizes = [int(be.size(t)) for t in (Hx, Hy, Px, Py)]
                n_max = max(sizes)
                if all(sz in (1, n_max) for sz in sizes) and any(getattr(t, "ndim", 1) != 1 or sz != n_max
                                                                 for t, sz in zip((Hx, Hy, Px, Py), sizes)):
                    Hx, Hy, Px, Py = (t.reshape(-1).expand(n_max) if sz == 1 and n_max > 1 else t.reshape(-1)
                                      for t, sz in zip((Hx, Hy, Px, Py), sizes))
            except Exception:
                pass                                  # not tensors: the check below declines
            if not all(engine.accepts_tensor(t) for t in (Hx, Hy, Px, Py)) or len({t.shape for t in (Hx, Hy, Px, Py)}) != 1:
                return _fused_decline("field / pupil arrays not resident on a CUDA device (or of different shapes)")
            if any(t.dtype != Px.dtype for t in (Hx, Hy)):
                return _fused_decline("field and pupil arrays of different precision")
            if optic.apodization and has_vig:
                # the factor is evaluated on the pupil point scaled ONCE by the vignetting factor (real_ray_tracer.py:132-141
                # -> ray_generator.py:83-85) while the launch geometry sees it scaled twice, in the kernel: three eager
                # element-wise ops for the once-scaled point
                if vig is None:
                    return _fused_decline("apodization together with vignetting factors of more than 16 fields")
                vxf, vyf = optic.fields.get_vig_factor(Hx, Hy)
                apod = _apodization_factor(be, engine, optic, Px * (1 - vxf), Py * (1 - vyf))
            else:
                apod = _apodization_factor(be, engine, optic, Px, Py)
            if apod is False:
                return _fused_decline("apodization factor not resident on the device")
            w = None
            if be.is_array_like(wavelength) and be.size(wavelength) > 1:
                w = be.to_tensor(wavelength, device=Px.device) if hasattr(be, "to_tensor") else wavelength
                if not engine.accepts_tensor(w) or w.shape != Px.shape:
                    return _fused_decline("wavelength array not resident on the device / wrong shape")
                w = w.to(Px.dtype)
                wls = _unique_wavelengths(w)
                if wls is None:
                    return _fused_decline(f"more than {T.MAX_WAVELENGTHS} distinct wavelengths")
            else:
                wls = _np.array([float(_np.asarray(be.to_numpy(be.atleast_1d(wavelength))).reshape(-1)[0])])
            polarized, state = _pol_state(be, optic)
            try:
                obj_geom = getattr(optic.object_surface, "geometry", None)
                if not bool(optic.object_surface.is_infinite) and type(obj_geom).__name__ != "Plane":
                    return _fused_decline("curved object surface")          # (it makes z0 field dependent)
                table = pack_surface_group(optic.surfaces, wls)
                sc = _launch_scalars_cached(be, optic, table, 0.0, 0.0)
                sc["vx"] = sc["vy"] = 1.0            # (the factors are already in Px, Py)
                _prepare(engine, table, Px.device)
                aff = pupil_affine_fields(sc, Hx, Hy)
                if vig is not None:
                    aff["vig"] = vig
            except _PACK_ERRORS as e:
                return _fused_decline(f"unsupported: {e}")
            if not polarized and any(s.coating in T.POLARIZING_COATINGS for s in table.surfaces):
                return None          # the reference raises (ray_generator.py:90-94)
            if polarized and any(s.bsdf != T.BSDF_NONE for s in table.surfaces):
                return _fused_decline("BSDF scatter with polarized rays")
            if table.surfaces[0].kind != T.GEOM_NOOP:
                return _fused_decline("first surface is not an object surface")
            # (trace_generic does NOT run update_intensity, real_ray_tracer.py:143-152: P matrices only)
            kw = {"polarization": "matrix"} if polarized else {}
            rec = engine.trace_pupil(table, Px, Py, aff, wavelength=w if len(wls) > 1 else None, **kw)
            _apply_apodization(rec, apod)
            _reset_records(be, optic.surfaces)
            for row, surf in enumerate(optic.surfaces.surfaces):
                for attr, key in _REC_ATTR:
                    setattr(surf, attr, rec[key][row])
            wl_arr = w if w is not None else be.ones_like(rec["x"][-1]) * float(wls[0])
            rays = _make_rays(be, rec, wl_arr, polarized)
            _set_pre_interaction_direction(rays, table, rec, 0, table.num_surfaces,
                                           (rec["L"][0], rec["M"][0], rec["N"][0]))
            # tail of trace_generic (real_ray_tracer.py:145-152)
            _tail_propagate(be, rays, optic.surfaces[-1], [float(v) for v in wls], w if len(wls) > 1 else None)
            return rays

        def wavefront_chief_ray(self, strategy, field, wavelength):
            """``ChiefRayStrategy.compute_wavefront_data`` (wavefront/strategy.py:152-213) with steps 3-5 -- the
            full-grid trace, the path length to the reference sphere, the OPD in waves and the exit-pupil
            intercepts -- fused into one launch that writes 5 values per ray (SURVEY.md 8f-2).  Steps 1-2 (chief
            ray, reference sphere, reference OPD) run as in the reference; with ``optic.polarization`` set the launch
            also writes the P matrices and step 6 (exit fields, strategy.py:193-203) runs the reference's own code on
            them.  Returns WavefrontData or None.

            Side effect that differs from the reference: afterwards ``optic.surfaces`` holds the records of the 1-ray
            chief trace, not of the full pupil grid (the fused launch writes no records)."""
            import numpy as _np
            from optiland.wavefront.wavefront_data import WavefrontData

            from .launch import launch_from_affine, pupil_affine
            from .pack import launch_scalars

            optic = strategy.optic
            engine = _state["engine"]
            if not hasattr(engine, "trace_wavefront") or getattr(strategy, "reference_type", "sphere") != "sphere":
                return None
            if getattr(_tls, "in_reference", False) or _wants_grad(self, list(optic.surfaces.surfaces)):
                return None
            if optic.apodization and optic.polarization != "ignore":
                return _fused_decline("wavefront: apodization together with polarization")
            if getattr(optic.ray_tracer, "ray_aiming_config", {}).get("mode", "paraxial") != "paraxial":
                return _fused_decline("wavefront: non-paraxial ray aiming")
            try:
                # the reference propagates the traced rays by the image surface's thickness before the wavefront
                # strategy reads them (real_ray_tracer.py:105-110); the fused epilogue works on the image-surface
                # record, so a non-zero thickness goes back to the reference path
                if float(_np.asarray(be.to_numpy(optic.surfaces[-1].thickness)).reshape(-1)[0]) != 0.0:
                    return _fused_decline("wavefront: image surface with a thickness")
            except Exception:
                return None
            dist = strategy.distribution
            Px, Py = dist.x, dist.y
            if not (engine.accepts_tensor(Px) and engine.accepts_tensor(Py)):
                return _fused_decline("wavefront: pupil samples not resident on a CUDA device")
            apod = _apodization_factor(be, engine, optic, Px, Py)      # scales WavefrontData.intensity only (the OPD
            if apod is False:                                          # does not depend on the launch intensity)
                return _fused_decline("wavefront: apodization factor not resident on the device")
            polarized, state = _pol_state(be, optic)
            try:
                hx, hy = float(field[0]), float(field[1])
                table = pack_surface_group(optic.surfaces, [float(wavelength)])
                sc = _launch_scalars_cached(be, optic, table, hx, hy)
                _prepare(engine, table, Px.device)
            except _PACK_ERRORS as e:
                return _fused_decline(f"wavefront unsupported: {e}")
            if not polarized and any(s.coating in T.POLARIZING_COATINGS for s in table.surfaces):
                return None
            if polarized and any(s.bsdf != T.BSDF_NONE for s in table.surfaces):
                return _fused_decline("BSDF scatter with polarized rays")
            # steps 1-2, the reference's own code on ONE ray (strategy.py:160-170)
            chief = optic.trace_generic(*field, Px=0.0, Py=0.0, wavelength=wavelength)
            strategy._chief_ray = chief
            geometry = strategy._create_reference_geometry(chief)
            opd_ref = chief.opd - geometry.path_length(chief, strategy.n_image)
            opd_ref = strategy._correct_tilt(field, opd_ref, x=0, y=0)
            tilt = (0.0, 0.0)
            if type(optic.fields.field_definition).__name__ == "AngleField" and bool(optic.object_surface.is_infinite):
                # _correct_tilt (strategy.py:112-138): opd += ux X + uy Y with (X, Y) = (Px, Py) EPD / 2
                mf = float(_np.asarray(be.to_numpy(optic.fields.max_field)).reshape(-1)[0])
                tx, ty = _np.tan(_np.deg2rad(hx * mf)), _np.tan(_np.deg2rad(hy * mf))
                uz = 1.0 / _np.sqrt(1.0 + tx**2 + ty**2)
                epd = float(_np.asarray(be.to_numpy(optic.paraxial.EPD())).reshape(-1)[0])
                tilt = (tx * uz * epd / 2, ty * uz * epd / 2)

            def f(v):
                return float(_np.asarray(be.to_numpy(v)).reshape(-1)[0])

            ref = {"center": [f(c) for c in geometry.center], "radius": f(geometry.radius), "n_image": f(strategy.n_image),
                   "tilt": tilt, "opd_ref": f(opd_ref), "wavelength_um": float(wavelength)}
            # a degenerate system (chief ray lost: NaN reference sphere, tests/test_fft_psf.py::test_invalid_working_FNO
            # moves the object to z = -1e100) has no sphere to fuse against -- the C ABI rejects a non-positive / NaN
            # radius: the reference's own ops carry the NaNs on
            chk = ref["center"] + [ref["radius"], ref["n_image"], ref["opd_ref"], tilt[0], tilt[1]]
            if not all(_np.isfinite(v) for v in chk) or not (ref["radius"] > 0 and ref["n_image"] > 0):
                return _fused_decline("wavefront: chief-ray reference sphere not finite")
            aff = pupil_affine(sc)
            kwargs = {}
            if polarized:
                out = engine.trace_wavefront(table, Px, Py, aff, ref, polarized=True)
                # step 6 (strategy.py:193-203): the reference's own get_exit_fields on the kernel's P matrices
                from optiland.rays import PolarizedRays

                shell = PolarizedRays.__new__(PolarizedRays)
                _, _, _, shell._L0, shell._M0, shell._N0 = launch_from_affine(Px, Py, aff)
                shell._i0 = be.ones_like(Px) * float(aff.get("intensity", 1.0))
                shell.p = out["p"]
                kwargs = {"prt_matrix": out["p"], "E_exits": shell.get_exit_fields(optic.polarization_state)}
            else:
                out = engine.trace_wavefront(table, Px, Py, aff, ref)
                if apod is not None:
                    out = dict(out, intensity=out["intensity"] * apod)
            return WavefrontData(pupil_x=out["pupil_x"], pupil_y=out["pupil_y"], pupil_z=out["pupil_z"], opd=out["opd"],
                                 intensity=out["intensity"], radius=geometry.radius, **kwargs)

        def trace_surface(self, surface, rays) -> bool:
            if type(surface).__name__ not in ("Surface", "ImageSurface"):
                return False
            return _try_trace(self, [surface], rays,
                              lambda wl: _frozen(("surface", id(surface), tuple(float(w) for w in wl)), surface,
                                                 lambda: T.SurfaceTable([pack_surface(surface, wl)], wl)))

    registry = be.__getattr__.__globals__["_backends"]  # same hook as tests/test_backend.py:79-85
    old = registry.get("torch")
    new = B200TorchBackend()
    if old is not None and hasattr(old, "_config"):
        new._config = old._config  # keep device / precision / grad-mode settings
    registry["torch"] = new
    if alias:
        registry[alias] = new

    orig_group_trace = SurfaceGroup.trace
    orig_surface_trace = Surface.trace

    def group_trace(self, rays, skip=0):
        backend = registry.get(be.get_backend())
        if hasattr(backend, "trace_surfaces") and not getattr(_tls, "in_reference", False):
            _reset_records(be, self)
            if backend.trace_surfaces(self, rays, skip, len(self.surfaces)):
                return rays
        _tls.in_reference = True
        try:
            return orig_group_trace(self, rays, skip)
        finally:
            _tls.in_reference = False

    def surface_trace(self, rays):
        backend = registry.get(be.get_backend())
        if hasattr(backend, "trace_surface") and not getattr(_tls, "in_reference", False):
            self.reset()
            if backend.trace_surface(self, rays):
                return rays
        return orig_surface_trace(self, rays)

    from optiland.raytrace.real_ray_tracer import RealRayTracer

    orig_tracer_trace = RealRayTracer.trace

    def tracer_trace(self, Hx, Hy, wavelength, num_rays=100, distribution="hexapolar"):
        backend = registry.get(be.get_backend())
        if hasattr(backend, "trace_optic") and _state.get("fuse_launch", True):
            rays = backend.trace_optic(self, Hx, Hy, wavelength, num_rays, distribution)
            if rays is not None:
                return rays
        return orig_tracer_trace(self, Hx, Hy, wavelength, num_rays, distribution)

    orig_tracer_generic = RealRayTracer.trace_generic

    def tracer_generic(self, Hx, Hy, Px, Py, wavelength):
        backend = registry.get(be.get_backend())
        if hasattr(backend, "trace_optic_generic") and _state.get("fuse_launch", True):
            rays = backend.trace_optic_generic(self, Hx, Hy, Px, Py, wavelength)
            if rays is not None:
                return rays
        return orig_tracer_generic(self, Hx, Hy, Px, Py, wavelength)

    # f-4: the iterative ray aimer re-traces ALL its rays from the first surface to the stop on every Broyden
    # iteration, one ``Surface.trace`` call per surface (rays/ray_aiming/iterative.py:339-367): through the per-surface
    # wrapper that is (stop + 1) packs, uploads and launches per iteration.  Here the whole subset is ONE table and ONE
    # launch of the SurfaceGroup capability over [start, stop]; records land on the same Surface objects.
    from optiland.rays.ray_aiming.iterative import IterativeRayAimer

    orig_trace_subset = IterativeRayAimer._trace_subset

    def aimer_trace_subset(self, x, y, z, L, M, N, wl, stop, is_inf):
        backend = registry.get(be.get_backend())
        if (hasattr(backend, "trace_surfaces") and _state.get("fuse_aimer", True)
                and not getattr(_tls, "in_reference", False)):
            from optiland.rays import RealRays as _RefRealRays

            rays = _RefRealRays(x, y, z, L, M, N, intensity=be.ones_like(x), wavelength=wl)
            start = 1 if is_inf else 0
            group = self.optic.surfaces
            for surf in list(group.surfaces)[start:stop + 1]:
                surf.reset()                       # what every Surface.trace starts with (standard_surface.py:200-215)
            if backend.trace_surfaces(group, rays, start, stop + 1):
                return rays
        return orig_trace_subset(self, x, y, z, L, M, N, wl, stop, is_inf)

    IterativeRayAimer._trace_subset = aimer_trace_subset

    from optiland.rays.ray_aiming.robust import RobustRayAimer

    orig_aim = {cls: cls.aim_rays for cls in (IterativeRayAimer, RobustRayAimer)}

    def _make_aim(orig):
        def aim_rays(self, *args, **kwargs):
            with _FrozenTables():              # the optic does not change inside one aiming call
                return orig(self, *args, **kwargs)
        return aim_rays

    IterativeRayAimer.aim_rays = _make_aim(orig_aim[IterativeRayAimer])

    # the robust aimer (ProjectionLens120FOV / 160FOV, WideAngle170FOV): every solve of its continuation is ONE launch of
    # the aim kernel instead of an eager Newton-Broyden loop of subset traces (and a stop-radius trace per solve)
    def robust_aim_rays(self, fields, wavelengths, pupil_coords, initial_guess=None):
        with _FrozenTables():
            backend = registry.get(be.get_backend())
            if (hasattr(backend, "trace_surfaces") and _state.get("device_aim", True)
                    and not getattr(_tls, "in_reference", False)):
                sol = _robust_aim_device(backend, self, fields, wavelengths, pupil_coords, initial_guess)
                if sol is not None:
                    return sol
            return orig_aim[RobustRayAimer](self, fields, wavelengths, pupil_coords, initial_guess)

    RobustRayAimer.aim_rays = robust_aim_rays

    # f-3: the Huygens-Fresnel summation strategy of the torch backend (psf/huygens_fresnel_strategies.py:183-273)
    from optiland.psf.huygens_fresnel_strategies import TorchSummation

    from optiland.wavefront.strategy import ChiefRayStrategy

    orig_chief_compute = ChiefRayStrategy.compute_wavefront_data

    def chief_compute(self, field, wavelength):
        backend = registry.get(be.get_backend())
        if hasattr(backend, "wavefront_chief_ray") and _state.get("fuse_wavefront", True):
            data = backend.wavefront_chief_ray(self, field, wavelength)
            if data is not None:
                return data
        return orig_chief_compute(self, field, wavelength)

    ChiefRayStrategy.compute_wavefront_data = chief_compute
    orig_hf_compute = TorchSummation.compute

    def hf_compute(self, image_x, image_y, image_z, pupil_x, pupil_y, pupil_z, pupil_amp, pupil_opd, wavelength, Rp):
        engine = _state.get("engine")
        if engine is not None and hasattr(engine, "huygens_psf") and not self.grad_wanted(
                image_x, image_y, image_z, pupil_x, pupil_y, pupil_z, pupil_amp, pupil_opd):
            ix, iy, iz = (be.to_tensor(t, device=self.device) for t in (image_x, image_y, image_z))
            px, py, pz, po = (be.to_tensor(t, device=self.device) for t in (pupil_x, pupil_y, pupil_z, pupil_opd))
            out = engine.huygens_psf(ix, iy, iz, px, py, pz, pupil_amp, po, float(wavelength), float(Rp))
            if out is not None:
                return out
        return orig_hf_compute(self, image_x, image_y, image_z, pupil_x, pupil_y, pupil_z, pupil_amp, pupil_opd,
                               wavelength, Rp)

    def _grad_wanted(self, *tensors):
        backend = registry.get(be.get_backend())
        return bool(backend.grad_mode.requires_grad) or any(getattr(t, "requires_grad", False) for t in tensors)

    # A helper of the reference's paraxial layer that dominates every trace of a CHANGED system: the launch scalars
    # (EPL, EPD, the object-space offset) read ``SurfaceGroup.positions`` eight times, and each read builds one
    # RealRays object per surface just to globalize the point (0, 0, 0) (coordinate_system.py:109-120) -- most of the
    # host time of an Optic.trace after a parameter change.  For a frame without a
    # parent the globalized origin IS (cs.x, cs.y, cs.z) (rotating the zero vector changes nothing), with the same
    # autograd connectivity; nested frames keep the reference's code.
    from optiland.coordinate_system import CoordinateSystem

    orig_position = CoordinateSystem.position_in_gcs

    def _position_in_gcs(self):
        if self.reference_cs is None and _state.get("fast_positions", True):
            return be.atleast_1d(self.x) + 0.0, be.atleast_1d(self.y) + 0.0, be.atleast_1d(self.z) + 0.0
        return orig_position.fget(self)

    CoordinateSystem.position_in_gcs = property(_position_in_gcs)

    # Inside ONE ``RayGenerator.generate_rays`` call the optic does not change, yet the reference recomputes the entrance
    # pupil diameter three times and its location twice -- each a paraxial trace in Python -- and the surface positions a
    # dozen times (ray_aiming/paraxial.py:33-106, fields/field_types/angle.py:17-120): 40 % of a small differentiable
    # step on the CPU, more on a GPU where every one of those element-wise ops is a kernel launch.  For the duration of
    # that call the three are memoised per object -- the SAME tensors are handed out again, so values and autograd
    # connectivity are exactly the reference's.
    from optiland.paraxial import Paraxial
    from optiland.rays.ray_generator import RayGenerator

    orig_generate = RayGenerator.generate_rays
    orig_epl, orig_epd = Paraxial.EPL, Paraxial.EPD
    orig_positions = SurfaceGroup.positions

    def _memo(key, owner, compute):
        memo = getattr(_tls, "paraxial_memo", None)
        if memo is None or not _state.get("memo_paraxial", True):
            return compute()
        hit = memo.get(key)
        if hit is None:
            hit = memo[key] = (owner, compute())
        return hit[1]

    def generate_rays(self, *args, **kwargs):
        with _ParaxialMemo():
            return orig_generate(self, *args, **kwargs)

    RayGenerator.generate_rays = generate_rays
    Paraxial.EPL = lambda self: _memo(("EPL", id(self)), self, lambda: orig_epl(self))
    Paraxial.EPD = lambda self: _memo(("EPD", id(self)), self, lambda: orig_epd(self))
    SurfaceGroup.positions = property(lambda self: _memo(("positions", id(self)), self, lambda: orig_positions.fget(self)))

    # f-2: spot statistics from the moments epilogue (RayOperand.rms_spot_size, SpotDiagram.rms_spot_radius / centroid)
    from . import spot as _spot

    saved_spot = _spot.install(sys.modules[__name__], registry, be)

    # f-3 (second half): the FFT-PSF's gridding passes on either side of the library FFT (psf/fft.py:123-227)
    from . import fftpsf as _fftpsf

    saved_fft = _fftpsf.install(sys.modules[__name__], registry, be)

    # incoherent irradiance maps binned on the device (analysis/irradiance.py:265-353)
    from . import irradiance as _irradiance

    saved_irr = _irradiance.install(sys.modules[__name__], registry, be)

    TorchSummation.grad_wanted = _grad_wanted
    TorchSummation.compute = hf_compute
    SurfaceGroup.trace = group_trace
    Surface.trace = surface_trace
    RealRayTracer.trace = tracer_trace
    RealRayTracer.trace_generic = tracer_generic
    _state.update(installed=True, orig_group_trace=orig_group_trace, orig_surface_trace=orig_surface_trace,
                  orig_tracer_trace=orig_tracer_trace, orig_tracer_generic=orig_tracer_generic, orig_hf_compute=orig_hf_compute, orig_chief_compute=orig_chief_compute,
                  old_backend=old, alias=alias, fuse_launch=True, fuse_wavefront=True, fuse_spot=True, fuse_fft_psf=True, fuse_aimer=True, device_aim=True, orig_trace_subset=orig_trace_subset, orig_aim=orig_aim, saved_spot=saved_spot, saved_fft=saved_fft,
                  saved_irr=saved_irr,
                  orig_position=orig_position, fast_positions=True, memo_paraxial=True,
                  orig_paraxial=(orig_generate, orig_epl, orig_epd, orig_positions))


def uninstall() -> None:
    if not _state.get("installed"):
        return
    import optiland.backend as be
    from optiland.surfaces.standard_surface import Surface
    from optiland.surfaces.surface_group import SurfaceGroup

    registry = be.__getattr__.__globals__["_backends"]
    from optiland.raytrace.real_ray_tracer import RealRayTracer

    SurfaceGroup.trace = _state["orig_group_trace"]
    Surface.trace = _state["orig_surface_trace"]
    RealRayTracer.trace = _state["orig_tracer_trace"]
    RealRayTracer.trace_generic = _state["orig_tracer_generic"]
    from optiland.psf.huygens_fresnel_strategies import TorchSummation

    TorchSummation.compute = _state["orig_hf_compute"]
    from optiland.wavefront.strategy import ChiefRayStrategy

    ChiefRayStrategy.compute_wavefront_data = _state["orig_chief_compute"]
    if _state.get("saved_spot") is not None:
        from . import spot as _spot

        _spot.uninstall(_state["saved_spot"])
    if _state.get("orig_trace_subset") is not None:
        from optiland.rays.ray_aiming.iterative import IterativeRayAimer

        IterativeRayAimer._trace_subset = _state["orig_trace_subset"]
    for cls, orig in (_state.get("orig_aim") or {}).items():
        cls.aim_rays = orig
    if _state.get("saved_fft") is not None:
        from . import fftpsf as _fftpsf

        _fftpsf.uninstall(_state["saved_fft"])
    if _state.get("saved_irr") is not None:
        from . import irradiance as _irradiance

        _irradiance.uninstall(_state["saved_irr"])
    if _state.get("orig_position") is not None:
        from optiland.coordinate_system import CoordinateSystem

        CoordinateSystem.position_in_gcs = _state["orig_position"]
    if _state.get("orig_paraxial") is not None:
        from optiland.paraxial import Paraxial
        from optiland.rays.ray_generator import RayGenerator

        RayGenerator.generate_rays, Paraxial.EPL, Paraxial.EPD, SurfaceGroup.positions = _state["orig_paraxial"]
    if _state.get("old_backend") is not None:
        registry["torch"] = _state["old_backend"]
    if _state.get("alias"):
        registry.pop(_state["alias"], None)
    _state.clear()
    _state["installed"] = False
    _state["declines"] = {}
