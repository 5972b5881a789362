"""Flatten a live Optiland ``SurfaceGroup`` into a ``SurfaceTable``.

This is the only module that looks at Optiland objects; it imports nothing from
Optiland itself (it dispatches on class *names*), so it is importable on a box
without the reference.  What it reads per surface is exactly what the reference's
hot path reads (SURVEY.md Appendix B):

* pose           ``geometry.cs.get_effective_transform()``  optiland/coordinate_system.py:145-165
* geometry       ``type(geometry)``, ``radius``, ``k``, ``coefficients``, ``tol``, ``max_iter``
                 optiland/geometries/{plane,standard,newton_raphson,even_asphere,odd_asphere,
                 polynomial,zernike}.py
* media          ``material_pre.n/k(lambda)``, ``material_post.n(lambda)``  optiland/materials/base.py:98-149
* interaction    ``interaction_model.is_reflective``, ``coating``, ``bsdf``  optiland/interactions/base.py:26-128
* aperture       ``surface.aperture`` tree  optiland/physical_apertures/*.py

Anything outside the supported set raises ``UnsupportedSurface`` so the caller
(``optiland_b200.plugin``) can fall back to the reference's Python loop.
"""
from __future__ import annotations

import math
import threading

import numpy as np

from . import table as T


class UnsupportedSurface(Exception):
    """The surface (or one of its parts) is outside the CUDA path's scope."""


_tls = threading.local()


def _f(v) -> float:
    """Scalar backend value (numpy scalar / 0-d tensor / float) -> python float."""
    pre = getattr(_tls, "resolved", None)
    if pre is not None:
        r = pre.get(id(v))
        if r is not None:
            return r
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return float(np.asarray(v, dtype=np.float64).reshape(-1)[0]) if np.ndim(v) else float(v)


def _arr(v) -> np.ndarray:
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype=np.float64)


def _cls(obj) -> str:
    return type(obj).__name__


class _Prefetch:
    """One device->host copy for ALL scalar parameters of a surface group.

    With the torch backend on a CUDA device every radius / conic / pose component / refractive index is a
    0-d device tensor, and converting them one by one costs a stream synchronisation each (~150 per
    Double-Gauss, 2-3 ms).  This context walks the same attributes ``pack_surface`` reads, stacks the tensors
    it finds (grouped by device and dtype) and resolves them together; ``_f`` then answers from the table by
    object identity.  Anything not found falls back to the direct conversion, so this is purely a fast path.
    """

    force = False       # tests: take the stacked path for host tensors too
    last_count = 0      # scalars resolved by the most recent prefetch

    def __init__(self, surfaces, wavelengths):
        self.surfaces = surfaces
        self.wavelengths = wavelengths
        self.keep = []          # keeps the tensors alive so that id() stays unique while the table is in use
        self.arrays = set()     # ids of the whole arrays among them (resolved to numpy arrays, not to floats)
        import torch

        self._tensor = torch.Tensor

    def _add(self, v):
        if isinstance(v, self._tensor):
            if v.numel() == 1 and v.dtype.is_floating_point:
                self.keep.append(v)
        elif isinstance(v, (list, tuple)):
            for u in v:
                self._add(u)

    def _add_array(self, v):
        if isinstance(v, self._tensor) and v.dtype.is_floating_point and v.numel() > 0:
            self.keep.append(v)
            self.arrays.add(id(v))

    def _walk(self):
        for surf in self.surfaces:
            g = getattr(surf, "geometry", None)
            if g is None:
                continue
            cs = getattr(g, "cs", None)
            if cs is not None:
                for k in ("x", "y", "z", "rx", "ry", "rz"):
                    self._add(getattr(cs, k, None))
            for k in ("radius", "k", "norm_x", "norm_y", "norm_radius", "Ry", "ky", "R_rot", "k_yz",
                      "grating_order", "grating_period", "groove_orientation_angle"):
                self._add(getattr(g, k, None))
            if _cls(g) == "GridSagGeometry":       # the node coordinates and sag values (pack_grid_sag)
                for k in ("x_grid", "y_grid", "sag_grid"):
                    self._add_array(getattr(g, k, None))
            if _cls(g) == "ForbesQ2dGeometry":     # the grouped coefficient lists (pack_forbes_q2d)
                for k in ("cm0_coeffs", "ams_coeffs", "bms_coeffs"):
                    self._add(getattr(g, k, None))
            for k in ("coefficients", "coeffs_poly_y"):
                c = getattr(g, k, None)
                if isinstance(c, (list, tuple)):
                    self._add([u for row in c for u in (row if isinstance(row, (list, tuple)) else [row])])
            rt = getattr(g, "radial_terms", None)
            if isinstance(rt, dict):
                self._add(list(rt.values()))
            z = getattr(g, "zernike", None)
            if z is not None:
                self._add(list(getattr(z, "coeffs", [])))
            pp = getattr(getattr(surf, "interaction_model", None), "phase_profile", None)
            if pp is not None:      # phase-profile terms (pack_phase_profile)
                for k in ("phase", "_K_x", "_K_y", "coefficients"):
                    self._add(getattr(pp, k, None))
            ap = getattr(surf, "aperture", None)
            stack = [ap] if ap is not None else []
            while stack:
                a = stack.pop()
                for k in ("r_max", "r_min", "offset_x", "offset_y", "x_min", "x_max", "y_min", "y_max"):
                    self._add(getattr(a, k, None))
                if _cls(a) in ("PolygonAperture", "FileAperture"):      # the vertex array (pack_aperture)
                    self._add_array(getattr(a, "vertices", None))
                for k in ("a", "b"):
                    u = getattr(a, k, None)
                    if u is not None and hasattr(u, "contains"):
                        stack.append(u)
                    else:
                        self._add(u)
            mats = [getattr(surf, "material_pre", None), getattr(surf, "material_post", None)]
            coating = getattr(getattr(surf, "interaction_model", None), "coating", None)
            if _cls(coating) == "ThinFilmCoating":
                try:
                    mats += _film_materials(coating)
                    self._add([layer.thickness_um for layer in coating.jones.stack.layers])
                except Exception:
                    pass
            elif _cls(coating) == "RetarderCoating":
                self._add(getattr(getattr(coating, "jones", None), "retardance", None))
            for mat in mats:
                if mat is None:
                    continue
                for wl in self.wavelengths:
                    for what in ("n", "k"):
                        if catalogue_value(mat, what, wl) is not None:
                            continue             # a catalogue glass already asked at this wavelength: nothing to fetch
                        try:
                            # the reference caches these per wavelength (materials/base.py:98-149), so the
                            # later call in _index_table returns the same object
                            self._add(getattr(mat, what)(float(wl)))
                        except Exception:
                            pass

    def __enter__(self):
        try:
            self._walk()
            if not _Prefetch.force and not any(t.is_cuda for t in self.keep):
                _tls.resolved = None     # host tensors convert directly at no cost
                return self
            groups = {}
            for t in self.keep:
                groups.setdefault((t.device, t.dtype), []).append(t)
            resolved = {}
            for ts in groups.values():
                import torch

                if not any(id(t) in self.arrays for t in ts):
                    vals = torch.stack([t if t.ndim == 0 else t.reshape(()) for t in ts]).detach().double().cpu().numpy()
                    for t, v in zip(ts, vals):
                        resolved[id(t)] = float(v)
                    continue
                flat = torch.cat([t.reshape(-1) for t in ts]).detach().double().cpu().numpy()
                off = 0
                for t in ts:
                    n = t.numel()
                    resolved[id(t)] = flat[off:off + n].reshape(t.shape) if id(t) in self.arrays else float(flat[off])
                    off += n
            _tls.resolved = resolved
            _Prefetch.last_count = len(resolved)
        except Exception:
            _tls.resolved = None
        return self

    def __exit__(self, *exc):
        _tls.resolved = None
        self.keep = []
        return False


def _pose(cs):
    """(t, R) of ``cs.get_effective_transform()`` (coordinate_system.py:145-165).  An un-nested frame is
    read directly -- six scalars and, only if tilted, one 3x3 product -- instead of through the ~20 small
    backend ops of the reference method; nested frames use the reference method."""
    if getattr(cs, "reference_cs", None) is not None:
        t_eff, R_eff = cs.get_effective_transform()
        return _arr(t_eff), _arr(R_eff) + 0.0
    t = np.array([_f(cs.x), _f(cs.y), _f(cs.z)], dtype=np.float64)
    rx, ry, rz = _f(cs.rx), _f(cs.ry), _f(cs.rz)
    if rx == 0.0 and ry == 0.0 and rz == 0.0:
        return t, np.eye(3)
    return t, T.rotation_matrix(rx, ry, rz) + 0.0


def pack_aperture(ap) -> np.ndarray:
    """Postfix program for an aperture tree (see include/olb.h)."""
    name = _cls(ap)
    if name == "RadialAperture":
        return T.aperture_radial(_f(ap.r_max), _f(ap.r_min))
    if name == "OffsetRadialAperture":
        return T.aperture_offset_radial(_f(ap.r_max), _f(ap.r_min), _f(ap.offset_x), _f(ap.offset_y))
    if name == "RectangularAperture":
        return T.aperture_rect(_f(ap.x_min), _f(ap.x_max), _f(ap.y_min), _f(ap.y_max))
    if name == "EllipticalAperture":
        return T.aperture_ellipse(_f(ap.a), _f(ap.b), _f(ap.offset_x), _f(ap.offset_y))
    ops = {"UnionAperture": T.AP_UNION, "IntersectionAperture": T.AP_INTERSECT,
           "DifferenceAperture": T.AP_DIFFERENCE}
    if name in ops:
        return T.aperture_combine(ops[name], pack_aperture(ap.a), pack_aperture(ap.b))
    if name in ("PolygonAperture", "FileAperture"):
        # the exact classes only (a subclass may override contains); the LIVE vertices, which scale() rewrites
        v = _grid_array(ap.vertices)
        if v.ndim != 2 or v.shape[1] != 2 or v.shape[0] < 3:
            raise UnsupportedSurface(f"polygon aperture with vertices of shape {v.shape} (at least 3 x 2)")
        if v.shape[0] > T.MAX_POLYGON_VERTICES:
            raise UnsupportedSurface(f"polygon aperture of {v.shape[0]} vertices: more than {T.MAX_POLYGON_VERTICES} "
                                     "prepared in shared memory")
        if not np.all(np.isfinite(v)):
            raise UnsupportedSurface("polygon aperture with non-finite vertices")
        return T.aperture_polygon(v[:, 0], v[:, 1])
    raise UnsupportedSurface(f"aperture type {name}")


# Catalogue glasses (materials/material.py, material_file.py): n(lambda), k(lambda) are functions of the data file alone --
# nothing an optimiser or a user can change on the object -- so their values at a wavelength are memoised ON the material
# object.  The reference's own per-wavelength cache (materials/base.py:98-149) does this job only while be.grad_mode is off:
# with it on every result "requires grad" (be.array(wavelength) does) and is recomputed -- one dispersion formula, ~10
# element-wise ops, per surface side per call, which on a CUDA device made packing the dominant cost of a small
# differentiable step.  Other material classes (IdealMaterial, AbbeMaterial, ...: parameters an optimiser may drive) are
# always asked.
_CATALOGUE_MATERIALS = ("Material", "MaterialFile")


def catalogue_value(material, what: str, wl: float):
    """Memoised n / k of a catalogue glass at ``wl`` (float), or None for any other material class / a memo miss."""
    if _cls(material) not in _CATALOGUE_MATERIALS:
        return None
    memo = material.__dict__.get("_olb_index_memo")
    return None if memo is None else memo.get((what, float(wl)))


def _remember(material, what: str, wl: float, value: float) -> None:
    if _cls(material) in _CATALOGUE_MATERIALS:
        material.__dict__.setdefault("_olb_index_memo", {})[(what, float(wl))] = float(value)


def _index_table(material, wavelengths, what: str) -> np.ndarray:
    fn = getattr(material, what)
    out = np.empty(len(wavelengths), dtype=np.float64)
    pre = getattr(_tls, "resolved", None)
    for j, wl in enumerate(wavelengths):
        known = catalogue_value(material, what, wl)
        if known is not None:
            out[j] = known
            continue
        v = fn(float(wl))
        if pre is not None and id(v) in pre:
            out[j] = pre[id(v)]
            _remember(material, what, wl, out[j])
            continue
        v = _arr(v)
        if np.iscomplexobj(v):
            raise UnsupportedSurface("complex refractive index")
        out[j] = float(v.reshape(-1)[0])
        _remember(material, what, wl, out[j])
    return out


_GEOM_KINDS = {
    "Plane": T.GEOM_PLANE,
    "StandardGeometry": T.GEOM_STANDARD,
    "EvenAsphere": T.GEOM_EVEN_ASPHERE,
    "OddAsphere": T.GEOM_ODD_ASPHERE,
    "PolynomialGeometry": T.GEOM_POLYNOMIAL,
    "ZernikePolynomialGeometry": T.GEOM_ZERNIKE,
    "ChebyshevPolynomialGeometry": T.GEOM_CHEBYSHEV,
    "BiconicGeometry": T.GEOM_BICONIC,
    "ToroidalGeometry": T.GEOM_TOROIDAL,
    "ForbesQNormalSlopeGeometry": T.GEOM_FORBES_QBFS,
    "ForbesQbfsGeometry": T.GEOM_FORBES_QBFS,       # deprecated alias class (forbes/geometry.py:733-759)
    "ForbesQ2dGeometry": T.GEOM_FORBES_Q2D,
}


def pack_phase_profile(profile) -> tuple[int, np.ndarray, float]:
    """(interaction kind, terms, efficiency) of a ``PhaseInteractionModel``'s profile (optiland/phase/*.py).  Only the
    exact profile classes are accepted: a subclass may override get_phase / get_gradient."""
    name = _cls(profile)
    if name == "ConstantPhaseProfile":
        kind, terms = T.INTERACT_PHASE_CONSTANT, [_f(profile.phase)]
    elif name == "LinearGratingPhaseProfile":
        # the profile's own precomputed K_x / K_y (linear_grating.py:51-54), so the rounding matches
        kind, terms = T.INTERACT_PHASE_LINEAR, [_f(profile._K_x), _f(profile._K_y)]
    elif name == "RadialPhaseProfile":
        coefs = list(profile.coefficients)
        if not coefs:
            raise UnsupportedSurface("RadialPhaseProfile without coefficients")
        if len(coefs) > T.MAX_PHASE_TERMS:
            raise UnsupportedSurface(f"RadialPhaseProfile with more than {T.MAX_PHASE_TERMS} coefficients")
        kind, terms = T.INTERACT_PHASE_RADIAL, [_f(c) for c in coefs]
    else:
        raise UnsupportedSurface(f"phase profile {name}")
    return kind, np.array(terms, dtype=np.float64), _f(profile.efficiency)


def _grid_array(v) -> np.ndarray:
    """A grid-sag or polygon-vertex array, from the prefetched copy when there is one (``_Prefetch``)."""
    pre = getattr(_tls, "resolved", None)
    r = pre.get(id(v)) if pre is not None else None
    return np.asarray(r, dtype=np.float64) if isinstance(r, np.ndarray) else _arr(v)


def pack_grid_sag(spec: T.SurfaceSpec, g) -> None:
    """``GridSagGeometry`` (optiland/geometries/grid_sag.py) -> ``spec``: the node coordinates, the sag table, tol and
    max_iter.  Grids the kernel cannot stage (more than ``T.MAX_GRID_ELEMENTS`` prepared elements), axes that are not
    strictly increasing and non-finite values decline, each with a reason."""
    x, y, z = (_grid_array(getattr(g, k)) for k in ("x_grid", "y_grid", "sag_grid"))
    x, y = x.reshape(-1), y.reshape(-1)
    nx, ny = len(x), len(y)
    if nx < 2 or ny < 2 or z.shape != (ny, nx):
        raise UnsupportedSurface(f"grid sag of shape {z.shape} on {ny} x {nx} nodes (at least 2 x 2)")
    if T.grid_elements(nx, ny) > T.MAX_GRID_ELEMENTS:
        raise UnsupportedSurface(f"grid sag of {ny} x {nx} nodes: more than {T.MAX_GRID_ELEMENTS} prepared elements "
                                 "in shared memory")
    for name, c in (("x", x), ("y", y)):
        if not (np.all(np.isfinite(c)) and np.all(np.diff(c) > 0)):
            raise UnsupportedSurface(f"grid sag {name} coordinates not finite and strictly increasing")
    if not np.all(np.isfinite(z)):
        raise UnsupportedSurface("grid sag with non-finite sag values")
    spec.grid_x, spec.grid_y, spec.grid_sag = x.copy(), y.copy(), z.copy()
    spec.tol = float(g.tol)
    spec.max_iter = int(g.max_iter)


def pack_forbes_q2d(spec: T.SurfaceSpec, g) -> None:
    """``ForbesQ2dGeometry`` (optiland/geometries/forbes/geometry.py:445-731) -> ``spec``: the coefficient lists in the
    reference's own grouping (``cm0_coeffs``, ``ams_coeffs``, ``bms_coeffs``, built by ``_prepare_coeffs`` -- what its sag
    and normal read) and the live ``norm_radius``.  Lists over the caps (``T.Q2D_MAX_M``, ``T.Q2D_MAX_TERMS``) and
    non-finite coefficients decline, each with a reason."""
    ams, bms = list(g.ams_coeffs or []), list(g.bms_coeffs or [])
    if len(ams) != len(bms):
        raise UnsupportedSurface(f"Forbes Q-2D with {len(ams)} cosine and {len(bms)} sine lists")
    if len(ams) > T.Q2D_MAX_M:
        raise UnsupportedSurface(f"Forbes Q-2D with azimuthal order {len(ams)} (max {T.Q2D_MAX_M})")
    lists = [np.array([_f(c) for c in v], dtype=np.float64) for v in [list(g.cm0_coeffs or []), *ams, *bms]]
    if any(len(v) > T.Q2D_MAX_TERMS for v in lists):
        raise UnsupportedSurface(f"Forbes Q-2D with radial order above {T.Q2D_MAX_TERMS - 1}")
    if not all(np.all(np.isfinite(v)) for v in lists):
        raise UnsupportedSurface("Forbes Q-2D with non-finite coefficients")
    norm = _f(g.norm_radius)
    if not (np.isfinite(norm) and norm > 0):
        raise UnsupportedSurface(f"Forbes Q-2D with norm_radius {norm}")
    M = len(ams)
    spec.q2d_cm0, spec.q2d_ams, spec.q2d_bms = lists[0], lists[1:1 + M], lists[1 + M:]
    spec.norm_radius = norm


# what the two kernel variants of Q-2D tables do not carry (olb_trace.cu: FEAT_Q2D_EXCLUDED)
def _q2d_excluded(spec: T.SurfaceSpec) -> str | None:
    if spec.interaction == T.INTERACT_GRATING:
        return "ruled grating"
    if spec.interaction != T.INTERACT_REFRACT:
        return "phase profile"
    if spec.kind == T.GEOM_GRID_SAG:
        return "grid sag"
    if spec.bsdf != T.BSDF_NONE:
        return "BSDF"
    if spec.coating in T.JONES_COATINGS:
        return "thin-film, polarizer or retarder coating"
    if spec.aperture is not None and T.polygon_vertices(spec.aperture):
        return "polygon aperture"
    return None


_GRATING_KINDS = {"PlaneGrating": T.GEOM_PLANE, "StandardGratingGeometry": T.GEOM_STANDARD}


def pack_grating(geometry, iname: str) -> tuple[int, tuple[float, float, float]]:
    """(geometry kind, (order, period in um, groove angle in rad)) of a ruled grating: a ``PlaneGrating`` or a
    ``StandardGratingGeometry`` under a ``DiffractiveInteractionModel`` (optiland/interactions/diffractive_model.py).
    Only these exact classes are accepted, as a pair: a subclass may override the grating vector or the diffraction."""
    gname = _cls(geometry)
    if gname not in _GRATING_KINDS:
        raise UnsupportedSurface(f"{iname} on geometry {gname}")
    if iname != "DiffractiveInteractionModel":
        raise UnsupportedSurface(f"interaction model {iname} on grating geometry {gname}")
    kind = _GRATING_KINDS[gname]
    if kind == T.GEOM_STANDARD and not np.isfinite(_f(geometry.radius)):
        # StandardGratingGeometry has no plane branch (its normal and grating vector are NaN there)
        raise UnsupportedSurface("StandardGratingGeometry with an infinite radius")
    period = _f(geometry.grating_period)
    if not np.isfinite(period) or period == 0:
        # the reference yields NaN directions for these; its own loop reproduces that
        raise UnsupportedSurface(f"grating period {period}")
    return kind, (_f(geometry.grating_order), period, _f(geometry.groove_orientation_angle))


# BaseCoatingPolarized coatings with their own Jones model (optiland/coatings.py:418-580): coating class -> the exact
# Jones class its ``jones`` property must return
_JONES_COATINGS = {"ThinFilmCoating": "JonesThinFilm", "PolarizerCoating": "JonesLinearPolarizer",
                   "RetarderCoating": "JonesLinearRetarder"}


def _jones_axis(jones) -> np.ndarray:
    axis = _arr(jones.axis).astype(np.float64).reshape(-1)
    if axis.size != 3 or not np.all(np.isfinite(axis)) or not np.any(axis != 0):
        raise UnsupportedSurface(f"{_cls(jones)} axis {axis.tolist()}")
    return axis


def _film_materials(coating):
    """The materials a ``ThinFilmCoating`` reads per wavelength: the stack's incident and substrate materials and
    every layer's (thin_film/core.py:_tmm_coh)."""
    stack = coating.jones.stack
    return [stack.incident_material, stack.substrate_material] + [layer.material for layer in stack.layers]


def pack_jones_coating(spec: T.SurfaceSpec, coating, wavelengths) -> None:
    """Thin-film, polarizer or retarder coating -> ``spec`` (include/olb.h OLB_COAT_THIN_FILM ...).  Only the exact
    coating classes with their own Jones classes are accepted: a subclass may override the Jones matrix.  What is read
    is what ``coating.jones.calculate_matrix`` reads: the Jones model's stack, axis and retardance."""
    cname = _cls(coating)
    jones = coating.jones
    if _cls(jones) != _JONES_COATINGS[cname]:
        raise UnsupportedSurface(f"{cname} with Jones model {_cls(jones)}")
    if cname == "ThinFilmCoating":
        stack = jones.stack
        if _cls(stack) != "ThinFilmStack":
            raise UnsupportedSurface(f"thin-film stack class {_cls(stack)}")
        layers = list(stack.layers)
        if len(layers) > T.MAX_FILM_LAYERS:
            raise UnsupportedSurface(f"thin-film stack with more than {T.MAX_FILM_LAYERS} layers")
        if any(_cls(layer) != "Layer" for layer in layers):
            raise UnsupportedSurface("thin-film layer class other than Layer")
        d = np.array([_f(layer.thickness_um) for layer in layers], dtype=np.float64)
        if not np.all(np.isfinite(d)) or np.any(d < 0):
            raise UnsupportedSurface(f"thin-film thicknesses {d.tolist()}")
        spec.coating = T.COAT_THIN_FILM
        spec.film_thickness = d
        n_wl = len(wavelengths)
        spec.film_n = np.array([_index_table(layer.material, wavelengths, "n") for layer in layers]).reshape(-1, n_wl)
        spec.film_k = np.array([_index_table(layer.material, wavelengths, "k") for layer in layers]).reshape(-1, n_wl)
        spec.film_n0 = _index_table(stack.incident_material, wavelengths, "n")
        spec.film_k0 = _index_table(stack.incident_material, wavelengths, "k")
        spec.film_ns = _index_table(stack.substrate_material, wavelengths, "n")
        spec.film_ks = _index_table(stack.substrate_material, wavelengths, "k")
    elif cname == "PolarizerCoating":
        spec.coating = T.COAT_POLARIZER
        spec.jones_axis = _jones_axis(jones)      # normalised once at construction (jones.py:128-130)
    else:
        retardance = _f(jones.retardance)
        if not np.isfinite(retardance):
            raise UnsupportedSurface(f"retardance {retardance}")
        spec.coating = T.COAT_RETARDER
        spec.retardance = retardance
        spec.jones_axis = _jones_axis(jones)


def _mix64(v: int) -> int:
    """SplitMix64's finaliser: a bijection of 64-bit integers that scatters nearby inputs."""
    v &= (1 << 64) - 1
    v = ((v ^ (v >> 30)) * 0xBF58476D1CE4E5B9) & ((1 << 64) - 1)
    v = ((v ^ (v >> 27)) * 0x94D049BB133111EB) & ((1 << 64) - 1)
    return v ^ (v >> 31)


def pack_bsdf(bsdf, position: int = 0):
    """(kind, sigma, key) of a surface's ``bsdf`` (optiland/scatter.py), None without one.  Only the two exact classes
    are accepted: a subclass may override the scattering function.  A 64-bit seed is taken from torch's default
    generator the first time the object is packed and kept on it, so every later trace of the same optic uploads the
    same table (the per-call draws differ through OlbTraceCall.rng_stream), and ``torch.manual_seed`` before the optic
    is built makes its traces repeat.  The Philox key mixes that seed with the surface's ``position`` in the table: one
    BSDF object set on several surfaces draws independently at each of them, as the reference's sequential generator
    does."""
    if bsdf is None:
        return None
    name = _cls(bsdf)
    if name == "LambertianBSDF":
        kind, sigma = T.BSDF_LAMBERTIAN, 0.0
    elif name == "GaussianBSDF":
        kind, sigma = T.BSDF_GAUSSIAN, _f(bsdf.sigma)
        if not math.isfinite(sigma):
            raise UnsupportedSurface(f"bsdf GaussianBSDF with sigma {sigma}")
    else:
        raise UnsupportedSurface(f"bsdf scatter of class {name}")
    seed = bsdf.__dict__.get("_olb_seed")
    if seed is None:
        import torch

        lo, hi = (int(v) for v in torch.randint(0, 1 << 32, (2,), dtype=torch.int64))
        seed = lo | (hi << 32)
        bsdf.__dict__["_olb_seed"] = seed
    return kind, sigma, _mix64(seed + (int(position) + 1) * 0x9E3779B97F4A7C15)


def pack_surface(surface, wavelengths, position: int = 0) -> T.SurfaceSpec:
    """One Optiland ``Surface`` / ``ObjectSurface`` / ``ImageSurface`` -> ``SurfaceSpec``; ``position``: its index in the
    table being packed (it keys a BSDF's draws)."""
    sname = _cls(surface)
    n_wl = len(wavelengths)
    if sname == "ObjectSurface":
        # no physics, still records (optiland/surfaces/object_surface.py:56-93)
        return T.SurfaceSpec(kind=T.GEOM_NOOP, n1=np.ones(n_wl), n2=np.ones(n_wl), k1=np.zeros(n_wl))
    if sname not in ("Surface", "ImageSurface"):
        raise UnsupportedSurface(f"surface class {sname}")

    g = surface.geometry
    gname = _cls(g)
    im = surface.interaction_model
    iname = _cls(im)
    grating = None
    if gname in _GRATING_KINDS or iname == "DiffractiveInteractionModel":
        kind, grating = pack_grating(g, iname)
    elif gname == "GridSagGeometry":
        kind = T.GEOM_GRID_SAG
    elif gname not in _GEOM_KINDS:
        raise UnsupportedSurface(f"geometry {gname}")
    else:
        kind = _GEOM_KINDS[gname]

    if grating is None and iname not in ("RefractiveReflectiveModel", "PhaseInteractionModel"):
        raise UnsupportedSurface(f"interaction model {iname}")
    bsdf = pack_bsdf(getattr(im, "bsdf", None), position)
    phase = pack_phase_profile(im.phase_profile) if iname == "PhaseInteractionModel" else None

    t_eff, R_eff = _pose(g.cs)
    if not (np.all(np.isfinite(t_eff)) and np.all(np.isfinite(R_eff))):
        raise UnsupportedSurface("non-finite pose")

    spec = T.SurfaceSpec(kind=kind, t=t_eff, R=R_eff, reflective=bool(im.is_reflective))
    if bsdf is not None:
        spec.bsdf, spec.bsdf_sigma, spec.bsdf_seed = bsdf
    if phase is not None:
        spec.interaction, spec.phase_terms, spec.phase_efficiency = phase
    if grating is not None:
        spec.interaction = T.INTERACT_GRATING
        spec.grating_order, spec.grating_period, spec.grating_angle = grating
    if kind == T.GEOM_GRID_SAG:
        pack_grid_sag(spec, g)          # (no radius, no conic: the geometry has neither)
    elif kind != T.GEOM_PLANE:
        spec.radius = _f(g.radius)
        spec.conic = _f(g.k)
    if kind in T.NEWTON_KINDS:
        spec.tol = float(g.tol)
        spec.max_iter = int(g.max_iter)
    if kind in (T.GEOM_EVEN_ASPHERE, T.GEOM_ODD_ASPHERE):
        spec.coefficients = np.array([_f(c) for c in g.coefficients], dtype=np.float64)
    elif kind == T.GEOM_POLYNOMIAL:
        C = g.coefficients
        spec.coefficients = np.atleast_2d(np.array([[_f(c) for c in row] for row in C], dtype=np.float64))
    elif kind == T.GEOM_CHEBYSHEV:
        spec.coefficients = np.atleast_2d(_arr(g.coefficients))
        spec.norm_radius = _f(g.norm_x)
        spec.norm_y = _f(g.norm_y)
    elif kind == T.GEOM_BICONIC:
        # radius / k of the base class hold Rx / kx (biconic.py:56-57)
        spec.radius_y = _f(g.Ry)
        spec.conic_y = _f(g.ky)
    elif kind == T.GEOM_TOROIDAL:
        # base class: radius = R_yz, k = 0 (the Newton start sphere, toroidal.py:71-73)
        spec.radius_y = _f(g.R_rot)
        spec.conic_y = _f(g.k_yz)
        spec.coefficients = np.array([_f(c) for c in g.coeffs_poly_y], dtype=np.float64)
    elif kind == T.GEOM_FORBES_QBFS:
        # radial_terms {order: a_n}; missing orders are zero (forbes/geometry.py:258-274)
        terms = {int(n): _f(v) for n, v in (g.radial_terms or {}).items()}
        if any(n < 0 for n in terms):
            raise UnsupportedSurface("Forbes radial term with a negative order")
        spec.coefficients = np.array([terms.get(n, 0.0) for n in range(max(terms) + 1)] if terms else [], dtype=np.float64)
        spec.norm_radius = _f(g.norm_radius)
    elif kind == T.GEOM_FORBES_Q2D:
        pack_forbes_q2d(spec, g)
    elif kind == T.GEOM_ZERNIKE:
        z = g.zernike
        coeffs = [_f(c) for c in z.coeffs]
        terms = []
        for (n, m), c in zip(z.indices, coeffs):
            norm = _f(z._norm_constant(int(n), int(m)))
            # the reference forms coeff * N_nm first (optiland/zernike/base.py:63-68)
            terms.append((float(n), float(m), c * norm, c))
        spec.coefficients = np.array(terms, dtype=np.float64).reshape(-1, 4)
        spec.zernike_norms = np.array([_f(z._norm_constant(int(n), int(m))) for (n, m) in z.indices], dtype=np.float64)
        spec.norm_radius = _f(g.norm_radius)

    if surface.aperture is not None:
        spec.aperture = pack_aperture(surface.aperture)

    mpre, mpost = surface.material_pre, surface.material_post
    for mat in (mpre, mpost):
        # the kernel propagates in straight lines (propagation/homogeneous.py:30-57); a GRIN medium raises
        # NotImplementedError in the reference (propagation/grin.py) and must not be traced as homogeneous here
        pm = getattr(mat, "propagation_model", None)
        if pm is not None and _cls(pm) != "HomogeneousPropagation":
            raise UnsupportedSurface(f"propagation model {_cls(pm)}")
    spec.n1 = _index_table(mpre, wavelengths, "n")
    spec.k1 = _index_table(mpre, wavelengths, "k")
    spec.n2 = _index_table(mpost, wavelengths, "n")

    coating = getattr(im, "coating", None)
    if coating is not None:
        cname = _cls(coating)
        if cname == "SimpleCoating":
            spec.coating = T.COAT_SIMPLE
            spec.coat_t = _f(coating.transmittance)
            spec.coat_r = _f(coating.reflectance)
        elif cname == "FresnelCoating":
            spec.coating = T.COAT_FRESNEL
            spec.coat_n1 = _index_table(coating.material_pre, wavelengths, "n")
            spec.coat_n2 = _index_table(coating.material_post, wavelengths, "n")
        elif cname in _JONES_COATINGS:
            pack_jones_coating(spec, coating, wavelengths)
        else:
            raise UnsupportedSurface(f"coating {cname}")
    spec.__post_init__()
    return spec


def pack_surface_group(surface_group, wavelengths) -> T.SurfaceTable:
    """Whole ``SurfaceGroup`` -> ``SurfaceTable`` tabulated at ``wavelengths`` (micrometres)."""
    wavelengths = np.atleast_1d(np.asarray(wavelengths, dtype=np.float64))
    if len(wavelengths) > T.MAX_WAVELENGTHS:
        raise UnsupportedSurface(f"more than {T.MAX_WAVELENGTHS} distinct wavelengths")
    surfaces = list(surface_group.surfaces)
    if len(surfaces) > T.MAX_SURFACES:
        raise UnsupportedSurface(f"more than {T.MAX_SURFACES} surfaces")
    with _Prefetch(surfaces, wavelengths):
        specs = [pack_surface(s, wavelengths, j) for j, s in enumerate(surfaces)]
        nv = sum(T.polygon_vertices(s.aperture) for s in specs if s.aperture is not None)
        if nv > T.MAX_POLYGON_VERTICES:
            raise UnsupportedSurface(f"polygon apertures with {nv} vertices in all: more than {T.MAX_POLYGON_VERTICES} "
                                     "prepared in shared memory")
        q2d = [s for s in specs if s.kind == T.GEOM_FORBES_Q2D]
        if q2d:
            ne = sum(T.q2d_elements(s.q2d_cm0, s.q2d_ams, s.q2d_bms) for s in q2d)
            if ne > T.MAX_Q2D_ELEMENTS:
                raise UnsupportedSurface(f"Forbes Q-2D surfaces with {ne} prepared elements in all: more than "
                                         f"{T.MAX_Q2D_ELEMENTS} in shared memory")
            for s in specs:
                what = _q2d_excluded(s)
                if what is not None:
                    raise UnsupportedSurface(f"Forbes Q-2D surface beside a {what}")
        return T.SurfaceTable(specs, wavelengths)


def launch_scalars(optic, Hx: float, Hy: float) -> dict:
    """Scalars from which the launch state of ONE field point is a closed form of (Px, Py) -- what
    ``field_definition.get_ray_origins`` (optiland/fields/field_types/angle.py:17-58,
    object_height.py:17-46) and ``ParaxialRayAimer.aim_rays`` (optiland/rays/ray_aiming/paraxial.py:33-106)
    compute per ray.  ``optiland_b200.launch.pupil_affine`` turns them into the kernel's affine form.

    mode 0 (no "mode" key in old fixtures): infinite object, angle field -- the ray origin slides with the
        pupil point.
    mode 1: finite object (angle or object-height field): every ray starts at the field's object point
        (x0, y0, z0) and aims at the paraxial entrance pupil.
    mode 2: finite object, object-space telecentric: target = origin + (Px vx, Py vy, cot(asin NA)).
    mode 3: infinite object, an image-height field type: like mode 0 with the pupil-centre origin (x0, y0, z0) taken
        from the reference's own field definition; finite objects of those field types are mode 1.  ``field_kind`` 0
        marks them: one field point per launch only (``launch.pupil_affine_fields`` refuses per-ray field points)."""
    import optiland.backend as be  # only called where the reference is importable

    fd = optic.fields.field_definition
    name = _cls(fd)
    infinite = bool(optic.object_surface.is_infinite)
    vxf, vyf = optic.fields.get_vig_factor(Hx, Hy)
    vx, vy = 1.0 - _f(vxf), 1.0 - _f(vyf)
    if name == "AngleField" and infinite:
        if optic.obj_space_telecentric:
            raise UnsupportedSurface("launch_scalars: telecentric object space with an angle field")
        return {
            "EPL": _f(optic.paraxial.EPL()),
            "EPD": _f(optic.paraxial.EPD()),
            "offset": _f(fd._get_starting_z_offset(optic)),
            "max_field": _f(optic.fields.max_field),
            "z1": _f(be.to_numpy(optic.surfaces.positions)[1]),
            "vx": vx,
            "vy": vy,
            "Hx": float(Hx),
            "Hy": float(Hy),
        }
    if name in ("ParaxialImageHeightField", "RealImageHeightField"):
        # Image-height field types (fields/field_types/paraxial_image_height.py, real_image_height.py): the object angle /
        # height that lands on the requested image height comes from the reference's own code -- a paraxial unit-ray
        # scaling, or a real chief-ray solve (which itself traces through the capability) -- asked for ONE probe pair
        # of pupil points; the launch then has the same closed form as an angle / object-height field: the origin
        # slides with the pupil point by (EPD/2 vx, EPD/2 vy) for an infinite object and is fixed for a finite one.
        # (The reference solves per RAY, for N copies of the same field point.)
        if optic.obj_space_telecentric:
            raise UnsupportedSurface(f"launch_scalars: telecentric object space with field type {name}")
        pr = be.array([0.0, 1.0])
        xo, yo, zo = (_arr(v).reshape(-1) for v in fd.get_ray_origins(optic, be.array([float(Hx)] * 2), be.array([float(Hy)] * 2), pr, pr, vx, vy))
        EPL, EPD = _f(optic.paraxial.EPL()), _f(optic.paraxial.EPD())
        sx, sy = (EPD / 2 * vx, EPD / 2 * vy) if infinite else (0.0, 0.0)
        tol = 1e-9 * (1.0 + abs(EPD))
        if not (abs(xo[1] - xo[0] - sx) <= tol and abs(yo[1] - yo[0] - sy) <= tol and abs(zo[1] - zo[0]) <= tol
                and all(math.isfinite(float(v)) for v in (xo[0], yo[0], zo[0]))):
            raise UnsupportedSurface(f"launch_scalars: field type {name}: the origin is not the expected function of the pupil point")
        return {"mode": 3.0 if infinite else 1.0, "x0": float(xo[0]), "y0": float(yo[0]), "z0": float(zo[0]), "EPL": EPL, "EPD": EPD,
                "vx": vx, "vy": vy, "Hx": float(Hx), "Hy": float(Hy), "max_field": _f(optic.fields.max_field), "field_kind": 0.0}
    if infinite or name not in ("AngleField", "ObjectHeightField"):
        raise UnsupportedSurface(f"launch_scalars: field type {name} with an {'in' if infinite else ''}finite object")
    # finite object: the origin does not depend on the pupil point; ask the reference's own field definition
    # for it (one probe at the pupil centre), like the refractive indices are asked of its materials
    zero = be.array([0.0])
    x0, y0, z0 = fd.get_ray_origins(optic, float(Hx), float(Hy), zero, zero, vx, vy)
    sc = {"x0": _f(_arr(x0).reshape(-1)[0]), "y0": _f(_arr(y0).reshape(-1)[0]), "z0": _f(_arr(z0).reshape(-1)[0]),
          "vx": vx, "vy": vy, "Hx": float(Hx), "Hy": float(Hy), "max_field": _f(optic.fields.max_field),
          "field_kind": 1.0 if name == "AngleField" else 2.0}
    if optic.obj_space_telecentric:
        if name == "AngleField" or not optic.aperture.supports_telecentric:
            raise UnsupportedSurface("launch_scalars: the reference raises for this telecentric configuration")
        sc.update(mode=2.0, sin=_f(optic.aperture.value))
    else:
        sc.update(mode=1.0, EPL=_f(optic.paraxial.EPL()), EPD=_f(optic.paraxial.EPD()))
    return sc


def _isinf(v) -> bool:
    return math.isinf(_f(v))
