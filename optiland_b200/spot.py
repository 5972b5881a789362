"""SURVEY.md 8f-2 wired into the reference's classes: spot STATISTICS from the fused moments epilogue
(OlbTraceCall.moments) -- launch generation + trace + moment sums in one kernel, nothing written per ray -- behind

* ``RayOperand.rms_spot_size``        optiland/optimization/operand/ray.py:299-342
* ``SpotDiagram.rms_spot_radius`` / ``.centroid``   optiland/analysis/spot_diagram/core.py:329-370

``SpotDiagram`` keeps per-ray data for plotting (``self.data``, generated at construction,
core.py:420-481).  Under the plugin each spot becomes a ``LazySpotData``: the table, launch form and pupil samples are
captured at construction (so a later change of the optic does not alter what the analysis holds, exactly as with the
reference's eager arrays); ``x`` / ``y`` / ``intensity`` are traced -- ONE launch with records -- only if something
reads them (``view()``, ``geometric_spot_radius``), while ``rms_spot_radius`` / ``centroid`` need two moment launches
per spot and no per-ray memory at all.  One side effect moves with it: the reference leaves each spot's records on
``optic.surfaces`` at construction; here they appear there when the spot's per-ray data is first read.

Second moments are taken about the FINAL centre in a second pass (pass 1: centroid about the frame origin), so no
large-offset cancellation enters: the value equals the reference's two-pass ``mean((x - cx)^2 + (y - cy)^2)`` to
rounding.  Installed / removed by ``optiland_b200.plugin.install`` / ``uninstall``.
"""
from __future__ import annotations

import numpy as np

from . import table as T


class LazySpotData:
    """Drop-in for ``SpotData`` (core.py:35-47): same three attributes, materialised on first access."""

    def __init__(self, engine, be, table, Px, Py, affine, coordinates: str, optic=None, apod=None):
        import weakref

        # per-ray launch intensity of an apodized pupil (strictly positive, checked by _fused_inputs): the mask i > 0 and
        # with it every moment is the unit-intensity launch's; the materialised records / intensities are scaled by it
        self._apod = apod

        self._engine, self._be = engine, be
        self._optic = weakref.ref(optic) if optic is not None else (lambda: None)
        self._table, self._Px, self._Py, self._affine = table, Px, Py, affine
        self._coordinates = coordinates
        self._xyz = None
        self._moments: dict = {}

    # ---- statistics without per-ray data ---------------------------------------------------------------
    def moments(self, center=(0.0, 0.0)):
        """8 moment sums of the masked (i > 0) intercepts about ``center`` (include/olb.h: OlbTraceCall.moments), in the
        image surface's local frame or in global coordinates, as the SpotDiagram was configured."""
        key = (float(center[0]), float(center[1]))
        m = self._moments.get(key)
        if m is None:
            m = self._engine.spot_moments(self._table, self._Px, self._Py, self._affine, center=key,
                                          global_xy=self._coordinates != "local")
            self._moments[key] = m
        return m

    def centroid(self):
        m = self.moments()
        if m[7] > 0 or m[0] == 0:
            return float("nan"), float("nan")
        return m[1] / m[0], m[2] / m[0]

    def rms_about(self, cx: float, cy: float) -> float:
        m = self.moments((cx, cy))
        if m[7] > 0 or m[0] == 0:
            return float("nan")        # be.mean over an array holding NaN / over an empty array
        return float(np.sqrt(m[3] / m[0]))

    @property
    def materialized(self) -> bool:
        return self._xyz is not None

    # ---- per-ray data on demand (core.py:462-481) ---------------------------------------------------------
    def _materialize(self):
        if self._xyz is None:
            rec = self._engine.trace_pupil(self._table, self._Px, self._Py, self._affine)
            if self._apod is not None:
                rec = dict(rec, intensity=rec["intensity"] * self._apod)
            optic = self._optic()
            if optic is not None and len(optic.surfaces.surfaces) == self._table.num_surfaces:
                # the reference's _generate_field_data leaves this trace's records on the optic's surfaces
                # (core.py:462-470); here that side effect happens when the per-ray data is first read
                optic.surfaces.reset()
                for row, surf in enumerate(optic.surfaces.surfaces):
                    for attr in ("x", "y", "z", "L", "M", "N", "intensity", "opd"):
                        setattr(surf, attr, rec[attr][row])
            x, y, z, inten = rec["x"][-1], rec["y"][-1], rec["z"][-1], rec["intensity"][-1]
            mask = inten > 0
            x, y, z, inten = x[mask], y[mask], z[mask], inten[mask]
            if self._coordinates == "local":
                s = self._table.surfaces[-1]
                tx, ty, tz = (float(v) for v in s.t)
                dx, dy, dz = x - tx, y - ty, z - tz
                if s.rotated:
                    R = s.R          # local = R^T (global - t)   (coordinate_system.py:73-89)
                    x = R[0, 0] * dx + R[1, 0] * dy + R[2, 0] * dz
                    y = R[0, 1] * dx + R[1, 1] * dy + R[2, 1] * dz
                else:
                    x, y = dx, dy
            self._xyz = (x, y, inten)
        return self._xyz

    x = property(lambda self: self._materialize()[0])
    y = property(lambda self: self._materialize()[1])
    intensity = property(lambda self: self._materialize()[2])


def _scalar(be, v) -> float:
    return float(np.asarray(be.to_numpy(be.atleast_1d(v))).reshape(-1)[0])


def _fused_inputs(P, backend, be, optic, Hx, Hy, wavelength, num_rays, distribution):
    """((table, Px, Py, affine), apodization factor or None) of a single-field, single-wavelength fused launch, or None
    (with the reason counted)."""
    from .launch import pupil_affine
    from .pack import pack_surface_group

    engine = P._state["engine"]
    if not hasattr(engine, "spot_moments"):
        return None
    if getattr(P._tls, "in_reference", False) or P._wants_grad(backend, list(optic.surfaces.surfaces)):
        return None
    try:
        if be.size(be.atleast_1d(Hx)) != 1 or be.size(be.atleast_1d(Hy)) != 1:
            return P._fused_decline("spot moments: several field points")
        hx, hy = _scalar(be, Hx), _scalar(be, Hy)
    except Exception:
        return P._fused_decline("spot moments: field coordinates are not plain numbers")
    if optic.polarization != "ignore":
        return P._fused_decline("spot moments: polarization")
    if getattr(optic.ray_tracer, "ray_aiming_config", {}).get("mode", "paraxial") != "paraxial":
        return P._fused_decline("spot moments: non-paraxial ray aiming")
    if isinstance(distribution, str):
        distribution = P._distribution(be, distribution, num_rays)
    Px, Py = distribution.x, distribution.y
    if not (engine.accepts_tensor(Px) and engine.accepts_tensor(Py)):
        return P._fused_decline("spot moments: pupil samples not resident on a CUDA device")
    # An apodized pupil (ray_generator.py:83-87, evaluated on the UNSCALED pupil point as in Optic.trace) only scales the
    # intensity: the statistics mask i > 0, so with a strictly positive factor they are the unit-intensity launch's.
    apod = P._apodization_factor(be, engine, optic, Px, Py)
    if apod is False or (apod is not None and not bool((apod > 0).all())):
        return P._fused_decline("spot moments: apodization factor not positive everywhere / not on the device")
    try:
        table = pack_surface_group(optic.surfaces, [float(wavelength)])
        sc = P._launch_scalars_cached(be, optic, table, hx, hy)
        P._prepare(engine, table, Px.device)
    except P._PACK_ERRORS as e:
        return P._fused_decline(f"spot moments unsupported: {e}")
    if any(s.coating in T.POLARIZING_COATINGS for s in table.surfaces) or table.surfaces[0].kind != T.GEOM_NOOP:
        return None
    return (table, Px, Py, pupil_affine(sc)), apod


def rms_spot_size(P, backend, be, optic, surface_number, Hx, Hy, num_rays, wavelength, distribution):
    """``RayOperand.rms_spot_size`` (operand/ray.py:299-342) from moment launches: the RMS radius, about the centroid of
    the primary wavelength's spot, of the GLOBAL (x, y) of EVERY ray on surface ``surface_number`` (no intensity mask, a
    NaN ray makes the result NaN -- the reference's ``be.mean`` over the record row).  Returns a backend scalar or None."""
    engine = P._state["engine"]
    S = optic.surfaces.num_surfaces
    try:
        last = range(S)[int(surface_number)] + 1
    except (IndexError, TypeError, ValueError):
        return None
    if isinstance(wavelength, str):
        if wavelength != "all":
            return None
        wls = [float(w) for w in optic.wavelengths.get_wavelengths()]
        ref = int(optic.wavelengths.primary_index)
    else:
        wls, ref = [float(wavelength)], 0
    if isinstance(distribution, str):
        distribution = P._distribution(be, distribution, num_rays)
    jobs = []
    for wl in wls:
        inp = _fused_inputs(P, backend, be, optic, Hx, Hy, wl, num_rays, distribution)
        if inp is None:
            return None
        jobs.append(inp[0])          # (every ray counts here, no intensity mask: the apodization factor does not enter)
    kw = dict(last=last, global_xy=True, every_ray=True)
    m = engine.spot_moments(*jobs[ref], center=(0.0, 0.0), **kw)
    if not np.isfinite(m[1]) or not np.isfinite(m[2]) or m[0] == 0:
        return be.array(float("nan"))
    cx, cy = m[1] / m[0], m[2] / m[0]
    s2 = n = 0.0
    for job in jobs:
        mm = engine.spot_moments(*job, center=(cx, cy), **kw)
        s2 += mm[3]
        n += mm[0]
    return be.array(float(np.sqrt(s2 / n)))


def install(P, registry, be):
    """Wrap the two consumers; returns the originals for ``uninstall``."""
    from optiland.analysis.spot_diagram.core import SpotDiagram
    from optiland.analysis.spot_diagram.reference import CentroidReference, ChiefRayReference
    from optiland.optimization.operand.ray import RayOperand

    orig_operand = RayOperand.__dict__["rms_spot_size"]          # the staticmethod object
    orig_fn = RayOperand.rms_spot_size

    def operand(optic, surface_number, Hx, Hy, num_rays, wavelength, distribution="hexapolar"):
        backend = registry.get(be.get_backend())
        if hasattr(backend, "trace_optic") and P._state.get("fuse_spot", True):
            out = rms_spot_size(P, backend, be, optic, surface_number, Hx, Hy, num_rays, wavelength, distribution)
            if out is not None:
                return out
        return orig_fn(optic, surface_number, Hx, Hy, num_rays, wavelength, distribution)

    orig_field_data = SpotDiagram._generate_field_data
    orig_rms = SpotDiagram.rms_spot_radius
    orig_centroid = SpotDiagram.centroid

    def field_data(self, field, wavelength, num_rays, distribution, coordinates):
        backend = registry.get(be.get_backend())
        if hasattr(backend, "trace_optic") and P._state.get("fuse_spot", True):
            inp = _fused_inputs(P, backend, be, self.optic, field[0], field[1], wavelength, num_rays, distribution)
            if inp is not None:
                return LazySpotData(P._state["engine"], be, *inp[0], coordinates, optic=self.optic, apod=inp[1])
        return orig_field_data(self, field, wavelength, num_rays, distribution, coordinates)

    def _all_lazy(self):
        return all(isinstance(sd, LazySpotData) and not sd.materialized for fd in self.data for sd in fd)

    def _centers(self):
        strat = self._reference_strategy
        if type(strat) is CentroidReference:
            return [fd[self._analysis_ref_wavelength_index].centroid() for fd in self.data]
        if type(strat) is ChiefRayReference:        # does not read the spot data (reference.py:91-116)
            return [(_scalar(be, cx), _scalar(be, cy)) for cx, cy in self._get_reference_centers(self.data)]
        return None

    def rms_spot_radius(self):
        if _all_lazy(self):
            centers = _centers(self)
            if centers is not None:
                return [[be.array(sd.rms_about(cx, cy)) for sd in fd] for fd, (cx, cy) in zip(self.data, centers)]
        return orig_rms(self)

    def centroid(self):
        if _all_lazy(self):
            ref = self._analysis_ref_wavelength_index
            return [tuple(be.array(v) for v in fd[ref].centroid()) for fd in self.data]
        return orig_centroid(self)

    RayOperand.rms_spot_size = staticmethod(operand)
    SpotDiagram._generate_field_data = field_data
    SpotDiagram.rms_spot_radius = rms_spot_radius
    SpotDiagram.centroid = centroid
    return {"operand": orig_operand, "field_data": orig_field_data, "rms": orig_rms, "centroid": orig_centroid}


def uninstall(saved):
    from optiland.analysis.spot_diagram.core import SpotDiagram
    from optiland.optimization.operand.ray import RayOperand

    RayOperand.rms_spot_size = saved["operand"]
    SpotDiagram._generate_field_data = saved["field_data"]
    SpotDiagram.rms_spot_radius = saved["rms"]
    SpotDiagram.centroid = saved["centroid"]
