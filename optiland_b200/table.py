"""Host-side surface table: the data contract between Optiland objects and libolb.

A ``SurfaceTable`` is the flattened, plain-data description of what the hot path
reads from a live ``SurfaceGroup`` (reference: SURVEY.md Appendix B; the
attributes read by ``Surface._trace_real``,
``optiland/surfaces/standard_surface.py:232-248``).  It packs into
the ``OlbSurface`` array + ``pool`` of ``include/olb.h``.

Nothing here touches a GPU; the module is shared by the product path
(``optiland_b200.trace``), the Optiland plugin (``optiland_b200.plugin``) and the
test oracle.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np

# ---- enums: keep in sync with include/olb.h --------------------------------
GEOM_NOOP = 0
GEOM_PLANE = 1
GEOM_STANDARD = 2
GEOM_EVEN_ASPHERE = 3
GEOM_ZERNIKE = 4
GEOM_ODD_ASPHERE = 5
GEOM_POLYNOMIAL = 6
GEOM_CHEBYSHEV = 7
GEOM_BICONIC = 8
GEOM_TOROIDAL = 9
GEOM_FORBES_QBFS = 10
GEOM_GRID_SAG = 11
# prepared grid-sag elements of one table (olb_prep.h: nx + ny + nx * ny per surface, e.g. an 89 x 89 grid).  They are
# staged in shared memory with the rest of the table, like the thin-film records below; include/olb.h OLB_MAX_GRID_ELEMENTS
MAX_GRID_ELEMENTS = 8192


def grid_elements(nx: int, ny: int) -> int:
    return nx + ny + nx * ny


GEOM_FORBES_Q2D = 12
# Forbes Q-2D caps (include/olb.h): the highest azimuthal order m, the longest coefficient list (radial orders 0 .. 15),
# and the prepared elements of one table, staged in shared memory with the rest of it (olb_prep.h)
Q2D_MAX_M = 16
Q2D_MAX_TERMS = 16
MAX_Q2D_ELEMENTS = 4096


def q2d_elements(cm0, ams, bms) -> int:
    """Prepared elements of one Q-2D surface (olb_prep.h): a 4-element header, the m = 0 list, and per m a 4-element
    header, the recurrence constants (3 per radial order of the longer list) and both lists."""
    return 4 + len(cm0) + sum(4 + 3 * max(len(a), len(b)) + len(a) + len(b) for a, b in zip(ams, bms))

SF_REFLECT = 1 << 0
SF_ROTATED = 1 << 1
SF_APERTURE = 1 << 2
SF_ABSORBING = 1 << 3
SF_NORECORD = 1 << 4
SF_BSDF = 1 << 5

COAT_NONE = 0
COAT_SIMPLE = 1
COAT_FRESNEL = 2
COAT_THIN_FILM = 3
COAT_POLARIZER = 4
COAT_RETARDER = 5
MAX_FILM_LAYERS = 32
# prepared thin-film records of one table, in elements (olb_prep.h: per surface n_wl records of 4 + 5 L, rounded up to 4,
# plus an 8-element header).  They are staged in shared memory with the rest of the table; 8192 elements (64 KiB in fp64)
# keeps the polarized kernel well inside the per-block limit with room for the surfaces and the P-matrix slots.
MAX_FILM_ELEMENTS = 8192


def film_elements(L: int, n_wl: int) -> int:
    return n_wl * (-(-(4 + 5 * L) // 4) * 4) + 8
JONES_COATINGS = (COAT_THIN_FILM, COAT_POLARIZER, COAT_RETARDER)   # their own Jones model (include/olb.h)
POLARIZING_COATINGS = (COAT_FRESNEL,) + JONES_COATINGS               # need polarized rays

INTERACT_REFRACT = 0
INTERACT_PHASE_CONSTANT = 1
INTERACT_PHASE_LINEAR = 2
INTERACT_PHASE_RADIAL = 3
INTERACT_GRATING = 4
MAX_PHASE_TERMS = 16
_PHASE_TERMS = {INTERACT_PHASE_CONSTANT: 1, INTERACT_PHASE_LINEAR: 2}

AP_RADIAL = 1
AP_OFFSET_RADIAL = 2
AP_RECT = 3
AP_ELLIPSE = 4
AP_POLYGON = 5      # the only variable-length instruction: n, then the n (x, y) pairs (include/olb.h)
# vertices of all the polygons of one table: their prepared edges are staged in shared memory with the rest of the table
# (include/olb.h OLB_MAX_POLYGON_VERTICES)
MAX_POLYGON_VERTICES = 1024
AP_UNION = 16
AP_INTERSECT = 17
AP_DIFFERENCE = 18
_AP_OPERANDS = {AP_RADIAL: 2, AP_OFFSET_RADIAL: 4, AP_RECT: 4, AP_ELLIPSE: 4,
                AP_UNION: 0, AP_INTERSECT: 0, AP_DIFFERENCE: 0}

TF_POLARIZED = 1 << 0
ST_ZERNIKE_RANGE = 1 << 0
ST_CHEBYSHEV_RANGE = 1 << 1
ST_K_PARALLEL_X = 1 << 2
ST_BSDF_ATTEMPTS = 1 << 3
ST_AIM_NAN_START = 1 << 4
ST_AIM_UNCONVERGED = 1 << 5

# BSDF scatter (include/olb.h OLB_SF_BSDF): LambertianBSDF / GaussianBSDF, and the kernel's bound on the draws of one ray
BSDF_NONE = 0
BSDF_LAMBERTIAN = 1
BSDF_GAUSSIAN = 2
BSDF_MAX_ATTEMPTS = 65536

MAX_SURFACES = 64
MAX_WAVELENGTHS = 16

NEWTON_KINDS = (GEOM_EVEN_ASPHERE, GEOM_ZERNIKE, GEOM_ODD_ASPHERE, GEOM_POLYNOMIAL, GEOM_CHEBYSHEV, GEOM_BICONIC,
                GEOM_TOROIDAL, GEOM_FORBES_QBFS, GEOM_FORBES_Q2D)

# numpy mirror of `struct OlbSurface` (192 bytes)
OLB_SURFACE_DTYPE = np.dtype(
    [
        ("kind", "<i4"), ("flags", "<u4"), ("n_coef", "<i4"), ("coef_off", "<i4"),
        ("aper_off", "<i4"), ("aper_len", "<i4"), ("max_iter", "<i4"), ("coating", "<i4"),
        ("media_off", "<i4"), ("aux0", "<i4"), ("interaction", "<i4"), ("phase_off", "<i4"),
        ("t", "<f8", (3,)), ("R", "<f8", (9,)),
        ("radius", "<f8"), ("conic", "<f8"), ("tol", "<f8"),
        ("coat_t", "<f8"), ("coat_r", "<f8"), ("norm_radius", "<f8"),
    ],
    align=False,
)
assert OLB_SURFACE_DTYPE.itemsize == 192


@dataclass
class SurfaceSpec:
    """One surface as the trace loop sees it.  Arrays are fp64 numpy."""

    kind: int = GEOM_PLANE
    t: np.ndarray = field(default_factory=lambda: np.zeros(3))
    R: np.ndarray = field(default_factory=lambda: np.eye(3))
    radius: float = float("inf")
    conic: float = 0.0
    tol: float = 1e-10
    max_iter: int = 100
    # EVEN/ODD: (n,) ; POLYNOMIAL: (rows, cols) ; ZERNIKE: (n_terms, 4) {n, m, c*N_nm, c}
    coefficients: np.ndarray = field(default_factory=lambda: np.zeros(0))
    norm_radius: float = 1.0   # Zernike norm_radius; Chebyshev norm_x
    norm_y: float = 1.0        # Chebyshev norm_y
    radius_y: float = float("inf")  # biconic Ry; toroidal: radius of rotation R_rot
    conic_y: float = 0.0            # biconic ky; toroidal: conic of the Y-Z curve
    reflective: bool = False
    aperture: np.ndarray | None = None  # postfix program, see include/olb.h
    n1: np.ndarray = field(default_factory=lambda: np.ones(1))
    n2: np.ndarray = field(default_factory=lambda: np.ones(1))
    k1: np.ndarray = field(default_factory=lambda: np.zeros(1))
    coating: int = COAT_NONE
    coat_t: float = 1.0
    coat_r: float = 0.0
    coat_n1: np.ndarray | None = None
    coat_n2: np.ndarray | None = None
    record: bool = True
    # ZERNIKE only, host side only (not packed): the normalisation constants N_nm per term, for mapping table
    # gradients back to the coefficients when a coefficient is exactly 0 (c * N_nm then does not reveal N_nm)
    zernike_norms: np.ndarray | None = None
    # phase-profile interaction (PhaseInteractionModel, include/olb.h OLB_INTERACT_*): INTERACT_REFRACT for the
    # refractive / reflective model; otherwise the profile's terms (constant {phi}, linear {Kx, Ky}, radial
    # {a_1 .. a_n}) and its diffraction efficiency
    interaction: int = INTERACT_REFRACT
    phase_terms: np.ndarray = field(default_factory=lambda: np.zeros(0))
    phase_efficiency: float = 1.0
    # ruled grating (DiffractiveInteractionModel, INTERACT_GRATING on a plane or a finite-radius conic): the
    # diffraction order, the period in micrometres and the groove orientation angle in radians
    grating_order: float = 0.0
    grating_period: float = float("inf")
    grating_angle: float = 0.0
    # thin-film coating (COAT_THIN_FILM, include/olb.h): layer thicknesses in micrometres (L,), the layers' n and k
    # (L, n_wl), and the stack's incident / substrate n and k (n_wl,)
    film_thickness: np.ndarray = field(default_factory=lambda: np.zeros(0))
    film_n: np.ndarray = field(default_factory=lambda: np.zeros((0, 1)))
    film_k: np.ndarray = field(default_factory=lambda: np.zeros((0, 1)))
    film_n0: np.ndarray | None = None
    film_k0: np.ndarray | None = None
    film_ns: np.ndarray | None = None
    film_ks: np.ndarray | None = None
    # polarizer / retarder coating (COAT_POLARIZER / COAT_RETARDER): the normalised axis and the retardance in radians
    jones_axis: np.ndarray = field(default_factory=lambda: np.array([1.0, 0.0, 0.0]))
    retardance: float = 0.0
    # grid sag (GEOM_GRID_SAG, include/olb.h): node coordinates (nx,), (ny,) and the sag values (ny, nx), row j at y_j
    grid_x: np.ndarray = field(default_factory=lambda: np.zeros(0))
    grid_y: np.ndarray = field(default_factory=lambda: np.zeros(0))
    grid_sag: np.ndarray = field(default_factory=lambda: np.zeros((0, 0)))
    # BSDF scatter (BSDF_LAMBERTIAN / BSDF_GAUSSIAN, include/olb.h): sigma (Gaussian) and the 64-bit Philox key of the
    # surface's draws
    bsdf: int = BSDF_NONE
    bsdf_sigma: float = 0.0
    bsdf_seed: int = 0
    # Forbes Q-2D (GEOM_FORBES_Q2D, include/olb.h): the reference's grouping of the coefficients -- the m = 0 list and,
    # for m = 1 .. M, the cosine and the sine lists (ForbesQ2dGeometry.cm0_coeffs / ams_coeffs / bms_coeffs), each
    # indexed by the radial order n; norm_radius holds the normalisation radius
    q2d_cm0: np.ndarray = field(default_factory=lambda: np.zeros(0))
    q2d_ams: list = field(default_factory=list)
    q2d_bms: list = field(default_factory=list)

    def __post_init__(self):
        self.t = np.asarray(self.t, dtype=np.float64).reshape(3)
        self.R = np.asarray(self.R, dtype=np.float64).reshape(3, 3)
        self.coefficients = np.asarray(self.coefficients, dtype=np.float64)
        self.n1 = np.atleast_1d(np.asarray(self.n1, dtype=np.float64))
        self.n2 = np.atleast_1d(np.asarray(self.n2, dtype=np.float64))
        self.k1 = np.atleast_1d(np.asarray(self.k1, dtype=np.float64))
        self.phase_terms = np.atleast_1d(np.asarray(self.phase_terms, dtype=np.float64)).ravel()
        if self.aperture is not None:
            self.aperture = np.asarray(self.aperture, dtype=np.float64).ravel()
        if self.coat_n1 is not None:
            self.coat_n1 = np.atleast_1d(np.asarray(self.coat_n1, dtype=np.float64))
        if self.coat_n2 is not None:
            self.coat_n2 = np.atleast_1d(np.asarray(self.coat_n2, dtype=np.float64))
        self.film_thickness = np.atleast_1d(np.asarray(self.film_thickness, dtype=np.float64)).ravel()
        L = len(self.film_thickness)
        self.film_n = np.asarray(self.film_n, dtype=np.float64).reshape(L, -1 if L else len(self.n1))
        self.film_k = np.asarray(self.film_k, dtype=np.float64).reshape(L, -1 if L else len(self.n1))
        for name in ("film_n0", "film_k0", "film_ns", "film_ks"):
            v = getattr(self, name)
            if v is not None:
                setattr(self, name, np.atleast_1d(np.asarray(v, dtype=np.float64)))
        self.jones_axis = np.asarray(self.jones_axis, dtype=np.float64).reshape(3)
        self.grid_x = np.asarray(self.grid_x, dtype=np.float64).ravel()
        self.grid_y = np.asarray(self.grid_y, dtype=np.float64).ravel()
        self.grid_sag = np.atleast_2d(np.asarray(self.grid_sag, dtype=np.float64))
        self.q2d_cm0 = np.asarray(self.q2d_cm0, dtype=np.float64).ravel()
        self.q2d_ams = [np.asarray(a, dtype=np.float64).ravel() for a in self.q2d_ams]
        self.q2d_bms = [np.asarray(b, dtype=np.float64).ravel() for b in self.q2d_bms]

    def q2d_block(self) -> np.ndarray:
        """The pool block of a Q-2D surface (include/olb.h): cm0, {na_m, nb_m} per m, then the lists a_1, b_1, a_2, ..."""
        lens = [float(len(v)) for a, b in zip(self.q2d_ams, self.q2d_bms) for v in (a, b)]
        lists = [v for a, b in zip(self.q2d_ams, self.q2d_bms) for v in (a, b)]
        return np.concatenate([self.q2d_cm0, np.asarray(lens, dtype=np.float64), *lists])

    def coating_block(self) -> np.ndarray:
        """The pool block of a thin-film / polarizer / retarder coating (include/olb.h), empty for other coatings."""
        if self.coating == COAT_THIN_FILM:
            L, n_wl = len(self.film_thickness), len(self.n1)
            per_wl = np.empty((n_wl, 4 + 2 * L))
            per_wl[:, 0], per_wl[:, 1] = self.film_n0, self.film_k0
            per_wl[:, 2], per_wl[:, 3] = self.film_ns, self.film_ks
            per_wl[:, 4::2] = self.film_n.T
            per_wl[:, 5::2] = self.film_k.T
            return np.concatenate([[float(L)], self.film_thickness, per_wl.ravel()])
        if self.coating == COAT_POLARIZER:
            return self.jones_axis.copy()
        if self.coating == COAT_RETARDER:
            return np.concatenate([[self.retardance], self.jones_axis])
        return np.zeros(0)

    @property
    def rotated(self) -> bool:
        return not np.array_equal(self.R, np.eye(3))

    @property
    def absorbing(self) -> bool:
        return bool(np.any(self.k1 > 0))

    @property
    def flags(self) -> int:
        f = 0
        if self.reflective:
            f |= SF_REFLECT
        if self.rotated:
            f |= SF_ROTATED
        if self.aperture is not None:
            f |= SF_APERTURE
        if self.absorbing:
            f |= SF_ABSORBING
        if not self.record:
            f |= SF_NORECORD
        if self.bsdf != BSDF_NONE:
            f |= SF_BSDF
        return f

    def bsdf_block(self) -> np.ndarray:
        """The pool block {kind, sigma, seed_lo, seed_hi} of a BSDF surface (include/olb.h), empty without one."""
        if self.bsdf == BSDF_NONE:
            return np.zeros(0)
        seed = int(self.bsdf_seed)
        return np.array([float(self.bsdf), float(self.bsdf_sigma), float(seed & 0xFFFFFFFF), float(seed >> 32)])


def _polygon_operands(prog: np.ndarray, i: int) -> int:
    """Operand count of the AP_POLYGON instruction at ``prog[i]``: the vertex count and the n (x, y) pairs."""
    nv = prog[i + 1] if i + 1 < len(prog) else 0.0
    if not (nv >= 3 and nv == int(nv)):
        raise ValueError(f"polygon aperture: the vertex count must be an integer >= 3, got {nv!r}")
    nv = int(nv)
    if i + 2 + 2 * nv > len(prog):
        raise ValueError("polygon aperture: vertices outside the program")
    if not np.all(np.isfinite(prog[i + 2: i + 2 + 2 * nv])):
        raise ValueError("polygon aperture: non-finite vertex")
    return 1 + 2 * nv


def polygon_vertices(prog: np.ndarray) -> int:
    """Vertices of all the polygons of a (valid) aperture program."""
    i, total = 0, 0
    while i < len(prog):
        op = int(prog[i])
        nops = _polygon_operands(prog, i) if op == AP_POLYGON else _AP_OPERANDS[op]
        total += (nops - 1) // 2 if op == AP_POLYGON else 0
        i += 1 + nops
    return total


def validate_aperture_program(prog: np.ndarray) -> None:
    """Check a postfix aperture program is well formed (stack depth ends at 1)."""
    i, depth = 0, 0
    n = len(prog)
    while i < n:
        op = int(prog[i]) if np.isfinite(prog[i]) else -1
        if (op not in _AP_OPERANDS and op != AP_POLYGON) or prog[i] != op:
            raise ValueError(f"bad aperture opcode {prog[i]!r} at {i}")
        nops = _polygon_operands(prog, i) if op == AP_POLYGON else _AP_OPERANDS[op]
        if op >= AP_UNION:
            if depth < 2:
                raise ValueError("aperture program stack underflow")
            depth -= 1
        else:
            depth += 1
            if depth > 8:
                raise ValueError("aperture program too deep (max 8)")
        i += 1 + nops
    if i != n or depth != 1:
        raise ValueError("malformed aperture program")


@dataclass
class SurfaceTable:
    """All surfaces of a system + the distinct wavelengths their media are tabulated at."""

    surfaces: list[SurfaceSpec]
    wavelengths: np.ndarray  # (n_wl,) micrometres; exact values that appear in rays.w

    def __post_init__(self):
        self.wavelengths = np.atleast_1d(np.asarray(self.wavelengths, dtype=np.float64))
        n_wl = len(self.wavelengths)
        if not 1 <= n_wl <= MAX_WAVELENGTHS:
            raise ValueError(f"n_wl must be in [1, {MAX_WAVELENGTHS}], got {n_wl}")
        if not 1 <= len(self.surfaces) <= MAX_SURFACES:
            raise ValueError(f"number of surfaces must be in [1, {MAX_SURFACES}]")
        for s in self.surfaces:
            for name in ("n1", "n2", "k1"):
                if len(getattr(s, name)) != n_wl:
                    raise ValueError(f"surface media '{name}' must have {n_wl} entries")
            if s.aperture is not None:
                validate_aperture_program(s.aperture)
            if s.coating == COAT_FRESNEL and (s.coat_n1 is None or s.coat_n2 is None):
                raise ValueError("Fresnel coating needs coat_n1/coat_n2")
            if s.coating == COAT_THIN_FILM:
                L = len(s.film_thickness)
                if L > MAX_FILM_LAYERS:
                    raise ValueError(f"thin film: {L} layers (max {MAX_FILM_LAYERS})")
                if not np.all(np.isfinite(s.film_thickness)) or np.any(s.film_thickness < 0):
                    raise ValueError("thin film: thicknesses must be finite and >= 0")
                if s.film_n.shape != (L, n_wl) or s.film_k.shape != (L, n_wl):
                    raise ValueError(f"thin film: layer indices must be ({L}, {n_wl})")
                for name in ("film_n0", "film_k0", "film_ns", "film_ks"):
                    v = getattr(s, name)
                    if v is None or len(v) != n_wl:
                        raise ValueError(f"thin film: '{name}' must have {n_wl} entries")
                if s.kind == GEOM_NOOP:
                    raise ValueError("thin film on an object surface")
            elif s.coating in (COAT_POLARIZER, COAT_RETARDER):
                if not (np.all(np.isfinite(s.jones_axis)) and np.linalg.norm(s.jones_axis) > 0):
                    raise ValueError("polarizer / retarder: the axis must be finite and non-zero")
                if not np.isfinite(s.retardance):
                    raise ValueError("retarder: non-finite retardance")
                if s.kind == GEOM_NOOP:
                    raise ValueError("polarizer / retarder on an object surface")
            if s.bsdf != BSDF_NONE:
                if s.bsdf not in (BSDF_LAMBERTIAN, BSDF_GAUSSIAN):
                    raise ValueError(f"unknown BSDF kind {s.bsdf}")
                if not np.isfinite(s.bsdf_sigma):
                    raise ValueError(f"BSDF sigma {s.bsdf_sigma} must be finite")
                if not 0 <= int(s.bsdf_seed) < 1 << 64:
                    raise ValueError("BSDF seed must be a 64-bit unsigned integer")
                if s.kind == GEOM_NOOP:
                    raise ValueError("BSDF on an object surface")
            if s.kind == GEOM_GRID_SAG:
                nx, ny = len(s.grid_x), len(s.grid_y)
                if nx < 2 or ny < 2 or s.grid_sag.shape != (ny, nx):
                    raise ValueError(f"grid sag: {nx} x-nodes and {ny} y-nodes (>= 2 each) need ({ny}, {nx}) sag values, "
                                     f"got {s.grid_sag.shape}")
                for name in ("grid_x", "grid_y"):
                    c = getattr(s, name)
                    if not (np.all(np.isfinite(c)) and np.all(np.diff(c) > 0)):
                        raise ValueError(f"grid sag: {name} must be finite and strictly increasing")
                if not np.all(np.isfinite(s.grid_sag)):
                    raise ValueError("grid sag: non-finite sag value")
            if s.kind == GEOM_FORBES_Q2D:
                if len(s.q2d_ams) != len(s.q2d_bms) or len(s.q2d_ams) > Q2D_MAX_M:
                    raise ValueError(f"Forbes Q-2D: {len(s.q2d_ams)} cosine and {len(s.q2d_bms)} sine lists (equal, at most "
                                     f"{Q2D_MAX_M})")
                lists = [s.q2d_cm0, *s.q2d_ams, *s.q2d_bms]
                if any(len(v) > Q2D_MAX_TERMS for v in lists):
                    raise ValueError(f"Forbes Q-2D: a coefficient list longer than {Q2D_MAX_TERMS}")
                if not all(np.all(np.isfinite(v)) for v in lists):
                    raise ValueError("Forbes Q-2D: non-finite coefficient")
                if not (np.isfinite(s.norm_radius) and s.norm_radius > 0):
                    raise ValueError(f"Forbes Q-2D: norm_radius {s.norm_radius} must be positive and finite")
            if s.interaction == INTERACT_GRATING:
                if s.kind not in (GEOM_PLANE, GEOM_STANDARD) or (s.kind == GEOM_STANDARD and not np.isfinite(s.radius)):
                    raise ValueError("grating: only on a plane or a conic with a finite radius")
                if not (np.isfinite(s.grating_period) and s.grating_period != 0):
                    raise ValueError(f"grating: period {s.grating_period} must be finite and non-zero")
                if not (np.isfinite(s.grating_order) and np.isfinite(s.grating_angle)):
                    raise ValueError("grating: non-finite order or angle")
            elif s.interaction != INTERACT_REFRACT:
                nt = len(s.phase_terms)
                if s.interaction not in (INTERACT_PHASE_CONSTANT, INTERACT_PHASE_LINEAR, INTERACT_PHASE_RADIAL):
                    raise ValueError(f"unknown interaction {s.interaction}")
                if nt != _PHASE_TERMS.get(s.interaction, nt) or not 1 <= nt <= MAX_PHASE_TERMS:
                    raise ValueError(f"phase profile: {nt} terms for interaction {s.interaction}")

        film = sum(film_elements(len(s.film_thickness), n_wl) for s in self.surfaces if s.coating == COAT_THIN_FILM)
        if film > MAX_FILM_ELEMENTS:
            raise ValueError(f"thin-film stacks of this table need {film} prepared elements in shared memory "
                             f"(more than {MAX_FILM_ELEMENTS})")
        nv = sum(polygon_vertices(s.aperture) for s in self.surfaces if s.aperture is not None)
        if nv > MAX_POLYGON_VERTICES:
            raise ValueError(f"polygon apertures of this table have {nv} vertices: their prepared edges are staged in "
                             f"shared memory (at most {MAX_POLYGON_VERTICES})")
        grid = sum(grid_elements(len(s.grid_x), len(s.grid_y)) for s in self.surfaces if s.kind == GEOM_GRID_SAG)
        if grid > MAX_GRID_ELEMENTS:
            raise ValueError(f"grid-sag surfaces of this table need {grid} prepared elements in shared memory "
                             f"(more than {MAX_GRID_ELEMENTS})")
        q2d = sum(q2d_elements(s.q2d_cm0, s.q2d_ams, s.q2d_bms) for s in self.surfaces if s.kind == GEOM_FORBES_Q2D)
        if q2d > MAX_Q2D_ELEMENTS:
            raise ValueError(f"Forbes Q-2D surfaces of this table need {q2d} prepared elements in shared memory "
                             f"(more than {MAX_Q2D_ELEMENTS})")

    @property
    def num_surfaces(self) -> int:
        return len(self.surfaces)

    @property
    def n_wl(self) -> int:
        return len(self.wavelengths)

    # ---- packing into the C ABI layout ------------------------------------
    def pack(self) -> tuple[np.ndarray, np.ndarray]:
        """Return (surfaces: OLB_SURFACE_DTYPE[n], pool: float64[m])."""
        n_wl = self.n_wl
        n = len(self.surfaces)
        surf = np.zeros(n, dtype=OLB_SURFACE_DTYPE)
        pool: list[float] = []

        def push(values) -> int:
            off = len(pool)
            pool.extend(np.asarray(values, dtype=np.float64).ravel().tolist())
            # keep every block 16-byte aligned for vector loads
            if len(pool) % 2:
                pool.append(0.0)
            return off

        # integer / offset columns are filled per surface, then every struct field is assigned ONCE for all
        # surfaces (a per-element structured assignment costs ~1 us; this runs on every plugin call)
        ints = {k: [0] * n for k in ("n_coef", "aux0", "coef_off", "aper_off", "aper_len", "media_off", "interaction",
                                     "phase_off")}
        for j, s in enumerate(self.surfaces):
            coef = s.coefficients
            extra_head = None
            if s.kind in (GEOM_POLYNOMIAL, GEOM_CHEBYSHEV):
                coef = np.atleast_2d(coef)
                ints["n_coef"][j] = coef.size
                ints["aux0"][j] = coef.shape[1]
                if s.kind == GEOM_CHEBYSHEV:
                    extra_head = [s.norm_radius, s.norm_y]
            elif s.kind in (GEOM_BICONIC, GEOM_TOROIDAL):
                ints["n_coef"][j] = coef.size
                extra_head = [s.radius_y, s.conic_y]
            elif s.kind == GEOM_ZERNIKE:
                coef = coef.reshape(-1, 4)
                ints["n_coef"][j] = coef.shape[0]
            elif s.kind == GEOM_GRID_SAG:
                # x[nx], y[ny], sag[ny][nx] (include/olb.h): aux0 = nx, n_coef = ny
                coef = np.concatenate([s.grid_x, s.grid_y, s.grid_sag.ravel()])
                ints["n_coef"][j] = len(s.grid_y)
                ints["aux0"][j] = len(s.grid_x)
            elif s.kind == GEOM_FORBES_Q2D:
                # cm0[n0], {na_m, nb_m} x M, the lists (include/olb.h): aux0 = n0, n_coef = M
                coef = s.q2d_block()
                ints["n_coef"][j] = len(s.q2d_ams)
                ints["aux0"][j] = len(s.q2d_cm0)
            else:
                ints["n_coef"][j] = coef.size
            if extra_head is not None:
                ints["coef_off"][j] = push(np.concatenate([np.asarray(extra_head, float), coef.ravel()]))
            else:
                ints["coef_off"][j] = push(coef) if coef.size else 0
            if s.aperture is not None:
                ints["aper_off"][j] = push(s.aperture)
                ints["aper_len"][j] = len(s.aperture)
            cn1 = s.coat_n1 if s.coat_n1 is not None else s.n1
            cn2 = s.coat_n2 if s.coat_n2 is not None else s.n2
            # a BSDF block, then a thin-film / polarizer / retarder block follow the media block directly
            # (pool[media_off + 5 n_wl])
            ints["media_off"][j] = push(np.concatenate([s.n1, s.n2, s.k1, cn1, cn2, s.bsdf_block(), s.coating_block()]))
            assert len(s.n1) == n_wl
            if s.interaction == INTERACT_GRATING:
                # the phase block's framing: "efficiency" 1 (the diffractive model has none), 3 terms {m, d, alpha}
                ints["interaction"][j] = s.interaction
                ints["phase_off"][j] = push(np.array([1.0, 3.0, s.grating_order, s.grating_period, s.grating_angle]))
            elif s.interaction != INTERACT_REFRACT:
                ints["interaction"][j] = s.interaction
                ints["phase_off"][j] = push(np.concatenate([[s.phase_efficiency, float(len(s.phase_terms))], s.phase_terms]))
        for k, v in ints.items():
            surf[k] = v
        sl = self.surfaces
        surf["kind"] = [s.kind for s in sl]
        surf["flags"] = [s.flags for s in sl]
        surf["max_iter"] = [s.max_iter for s in sl]
        surf["coating"] = [s.coating for s in sl]
        if n:
            surf["t"] = np.stack([s.t for s in sl])
            surf["R"] = np.stack([s.R.ravel() for s in sl])
        for k, attr in (("radius", "radius"), ("conic", "conic"), ("tol", "tol"), ("coat_t", "coat_t"),
                        ("coat_r", "coat_r"), ("norm_radius", "norm_radius")):
            surf[k] = [getattr(s, attr) for s in sl]
        if not pool:
            pool.append(0.0)
            pool.append(0.0)
        return surf, np.asarray(pool, dtype=np.float64)

    def packed(self):
        """``pack()`` computed once per table object (a table is not mutated after it is built)."""
        pk = self.__dict__.get("_packed")
        if pk is None:
            pk = self.pack()
            self.__dict__["_packed"] = pk
        return pk

    def content_key(self) -> bytes:
        """Every value the kernels read, as bytes: equal keys <=> identical prepared tables."""
        key = self.__dict__.get("_content_key")
        if key is None:
            surf, pool = self.packed()
            key = surf.tobytes() + pool.tobytes() + np.asarray(self.wavelengths, dtype=np.float64).tobytes()
            self.__dict__["_content_key"] = key
        return key

    # ---- (de)serialisation for the golden fixtures ------------------------
    def to_arrays(self, prefix: str = "tab_") -> dict[str, np.ndarray]:
        surf, pool = self.pack()
        return {
            prefix + "surfaces": surf.view(np.uint8).reshape(len(surf), -1),
            prefix + "pool": pool,
            prefix + "wavelengths": self.wavelengths,
        }

    @classmethod
    def from_arrays(cls, arrays, prefix: str = "tab_") -> "SurfaceTable":
        raw = np.ascontiguousarray(arrays[prefix + "surfaces"], dtype=np.uint8)
        surf = raw.reshape(-1).view(OLB_SURFACE_DTYPE)
        pool = np.asarray(arrays[prefix + "pool"], dtype=np.float64)
        wl = np.asarray(arrays[prefix + "wavelengths"], dtype=np.float64)
        return cls.unpack(surf, pool, wl)

    @classmethod
    def unpack(cls, surf: np.ndarray, pool: np.ndarray, wavelengths: np.ndarray) -> "SurfaceTable":
        n_wl = len(wavelengths)
        specs = []
        for r in surf:
            kind = int(r["kind"])
            n_coef = int(r["n_coef"])
            off = int(r["coef_off"])
            head = None
            if kind == GEOM_ZERNIKE:
                coef = pool[off: off + 4 * n_coef].reshape(-1, 4).copy()
            elif kind == GEOM_POLYNOMIAL:
                cols = max(int(r["aux0"]), 1)
                coef = pool[off: off + n_coef].reshape(-1, cols).copy()
            elif kind == GEOM_CHEBYSHEV:
                cols = max(int(r["aux0"]), 1)
                head = pool[off: off + 2].copy()
                coef = pool[off + 2: off + 2 + n_coef].reshape(-1, cols).copy()
            elif kind in (GEOM_BICONIC, GEOM_TOROIDAL):
                head = pool[off: off + 2].copy()
                coef = pool[off + 2: off + 2 + n_coef].copy()
            elif kind == GEOM_GRID_SAG:
                nx = int(r["aux0"])
                g = pool[off: off + nx + n_coef + nx * n_coef]
                grid = dict(grid_x=g[:nx].copy(), grid_y=g[nx:nx + n_coef].copy(),
                            grid_sag=g[nx + n_coef:].reshape(n_coef, nx).copy())
                coef = np.zeros(0)
            elif kind == GEOM_FORBES_Q2D:
                n0 = int(r["aux0"])
                lens = pool[off + n0: off + n0 + 2 * n_coef].astype(int)
                p = off + n0 + 2 * n_coef
                lists = []
                for ln in lens:
                    lists.append(pool[p: p + ln].copy())
                    p += ln
                grid = dict(q2d_cm0=pool[off: off + n0].copy(), q2d_ams=lists[0::2], q2d_bms=lists[1::2])
                coef = np.zeros(0)
            else:
                coef = pool[off: off + n_coef].copy()
            if kind not in (GEOM_GRID_SAG, GEOM_FORBES_Q2D):
                grid = {}
            flags = int(r["flags"])
            aper = None
            if flags & SF_APERTURE:
                a0 = int(r["aper_off"])
                aper = pool[a0: a0 + int(r["aper_len"])].copy()
            m0 = int(r["media_off"])
            media = pool[m0: m0 + 5 * n_wl].reshape(5, n_wl)
            coating = int(r["coating"])
            cb = m0 + 5 * n_wl
            bsdf = {}
            if flags & SF_BSDF:
                bsdf = dict(bsdf=int(pool[cb]), bsdf_sigma=float(pool[cb + 1]),
                            bsdf_seed=int(pool[cb + 2]) | (int(pool[cb + 3]) << 32))
                cb += 4
            film = {}
            if coating == COAT_THIN_FILM:
                L = int(pool[cb])
                per_wl = pool[cb + 1 + L: cb + 1 + L + n_wl * (4 + 2 * L)].reshape(n_wl, 4 + 2 * L)
                film = dict(film_thickness=pool[cb + 1: cb + 1 + L].copy(), film_n=per_wl[:, 4::2].T.copy(),
                            film_k=per_wl[:, 5::2].T.copy(), film_n0=per_wl[:, 0].copy(), film_k0=per_wl[:, 1].copy(),
                            film_ns=per_wl[:, 2].copy(), film_ks=per_wl[:, 3].copy())
            elif coating == COAT_POLARIZER:
                film = dict(jones_axis=pool[cb: cb + 3].copy())
            elif coating == COAT_RETARDER:
                film = dict(retardance=float(pool[cb]), jones_axis=pool[cb + 1: cb + 4].copy())
            inter = int(r["interaction"])
            phase = {}
            if inter == INTERACT_GRATING:
                p0 = int(r["phase_off"])
                phase = dict(interaction=inter, grating_order=float(pool[p0 + 2]), grating_period=float(pool[p0 + 3]),
                             grating_angle=float(pool[p0 + 4]))
            elif inter != INTERACT_REFRACT:
                p0 = int(r["phase_off"])
                phase = dict(interaction=inter, phase_efficiency=float(pool[p0]),
                             phase_terms=pool[p0 + 2: p0 + 2 + int(pool[p0 + 1])].copy())
            specs.append(
                SurfaceSpec(
                    kind=kind, t=r["t"].copy(), R=r["R"].reshape(3, 3).copy(),
                    radius=float(r["radius"]), conic=float(r["conic"]), tol=float(r["tol"]),
                    max_iter=int(r["max_iter"]), coefficients=coef,
                    norm_radius=float(head[0]) if kind == GEOM_CHEBYSHEV else float(r["norm_radius"]),
                    norm_y=float(head[1]) if kind == GEOM_CHEBYSHEV else 1.0,
                    radius_y=float(head[0]) if kind in (GEOM_BICONIC, GEOM_TOROIDAL) else float("inf"),
                    conic_y=float(head[1]) if kind in (GEOM_BICONIC, GEOM_TOROIDAL) else 0.0,
                    reflective=bool(flags & SF_REFLECT), aperture=aper,
                    n1=media[0].copy(), n2=media[1].copy(), k1=media[2].copy(),
                    coating=coating, coat_t=float(r["coat_t"]), coat_r=float(r["coat_r"]),
                    coat_n1=media[3].copy() if coating == COAT_FRESNEL else None,
                    coat_n2=media[4].copy() if coating == COAT_FRESNEL else None,
                    record=not (flags & SF_NORECORD),
                    **phase,
                    **film,
                    **grid,
                    **bsdf,
                )
            )
        return cls(specs, wavelengths)

    def replace_surface(self, index: int, **changes) -> "SurfaceTable":
        surfaces = list(self.surfaces)
        surfaces[index] = dataclasses.replace(surfaces[index], **changes)
        return SurfaceTable(surfaces, self.wavelengths)


# ---- small constructors used by tests / bench (no Optiland needed) ---------

def aperture_radial(r_max: float, r_min: float = 0.0) -> np.ndarray:
    return np.array([AP_RADIAL, r_max, r_min], dtype=np.float64)


def aperture_offset_radial(r_max, r_min, dx, dy) -> np.ndarray:
    return np.array([AP_OFFSET_RADIAL, r_max, r_min, dx, dy], dtype=np.float64)


def aperture_rect(x_min, x_max, y_min, y_max) -> np.ndarray:
    return np.array([AP_RECT, x_min, x_max, y_min, y_max], dtype=np.float64)


def aperture_ellipse(a, b, dx=0.0, dy=0.0) -> np.ndarray:
    return np.array([AP_ELLIPSE, a, b, dx, dy], dtype=np.float64)


def aperture_polygon(x, y) -> np.ndarray:
    """Vertices (x_k, y_k) of a polygon, closed implicitly; any orientation, self-intersections allowed (even-odd)."""
    xy = np.stack([np.asarray(x, dtype=np.float64).ravel(), np.asarray(y, dtype=np.float64).ravel()], axis=1)
    return np.concatenate([[AP_POLYGON, float(len(xy))], xy.ravel()])


def aperture_combine(op: int, a: Sequence[float], b: Sequence[float]) -> np.ndarray:
    return np.concatenate([np.asarray(a, float), np.asarray(b, float), [float(op)]])


def rotation_matrix(rx: float, ry: float, rz: float) -> np.ndarray:
    """R = Rz @ Ry @ Rx  (reference: optiland/coordinate_system.py:121-143)."""
    cx, sx = np.cos(rx), np.sin(rx)
    cy, sy = np.cos(ry), np.sin(ry)
    cz, sz = np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def zernike_monomials(n: int, m: int, width: int) -> np.ndarray:
    """Monomial expansion of the UNIT Zernike term R_n^|m|(rho) {cos, sin}(|m| phi) (m >= 0: cos, m < 0: sin) as a
    (width, width) table M[i, j] ~ xn^i yn^j -- the Python twin of olb_prep.h::zernike_add_monomials (exact integer
    arithmetic in doubles).  The prepared sag table of a Zernike surface is S = sum_k c_k N_k M_k and its slope table
    D = sum_k c_k M_k (the reference's derivative path omits N_k), so table gradients map back to the coefficients by
    dL/dc_k = N_k <M_k, dL/dS> + <M_k, dL/dD>  (optiland_b200.autograd)."""
    from math import comb, factorial

    ma = abs(m)
    out = np.zeros((width, width), dtype=np.float64)
    for k in range((n - ma) // 2 + 1):
        rc = (-1.0 if k & 1 else 1.0) * factorial(n - k) / (factorial(k) * factorial((n + ma) // 2 - k) * factorial((n - ma) // 2 - k))
        q = (n - ma) // 2 - k
        for a in range(q + 1):
            ca = comb(q, a)
            for j in range(ma + 1):
                imag = (j & 1) != 0
                if (m >= 0) == imag:
                    continue
                sgn = -1.0 if (j >> 1) & 1 else 1.0
                out[2 * a + (ma - j), 2 * (q - a) + j] += rc * ca * comb(ma, j) * sgn
    return out
