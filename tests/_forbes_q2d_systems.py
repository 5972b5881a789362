"""Optical systems with Forbes Q-2D freeform surfaces (Optiland's ``surface_type="forbes_q2d"``, ``ForbesQ2dGeometry``),
built through the reference's own API.  Shared by the fixture generator (``oracle/make_golden_forbes_q2d.py``), the
live tests (``tests/test_forbes_q2d.py``) and the benchmark (``scripts/bench_forbes_q2d.py``); every builder needs the
reference importable and takes its backend module."""
from __future__ import annotations

import numpy as np

WL3 = (0.4861, 0.5876, 0.6563)

# the gallery's Q-2D singlet (docs/gallery/freeform/forbes_surface.ipynb)
GALLERY = {("a", 0, 0): 1.0, ("a", 1, 1): 2.0, ("b", 1, 1): 3.0, ("a", 0, 4): 4.0}


def freeform(M, N, scale, seed, m1_terms=None):
    """Seeded Zemax-style coefficients: every (m, n) with m <= M, n <= N, cosine and (m > 0) sine terms of size
    ``scale`` falling with n; ``m1_terms`` radial orders of m = 1 (at least 4 exercise the reference's extra m = 1
    term)."""
    rng = np.random.default_rng(seed)
    out = {}
    for m in range(M + 1):
        for n in range(N + 1 if m != 1 or m1_terms is None else m1_terms):
            out[("a", m, n)] = float(rng.normal() * scale / (1 + n))
            if m > 0:
                out[("b", m, n)] = float(rng.normal() * scale / (1 + n))
    return out


def _lens(be, epd, fields, wls):
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)

    def done():
        lens.set_aperture(aperture_type="EPD", value=epd)
        lens.fields.set_type(field_type="angle")
        for y in fields:
            lens.fields.add(y=y)
        for w in wls:
            lens.wavelengths.add(value=w, is_primary=(w == wls[len(wls) // 2]))
        return lens

    return lens, done


def q2d_kw(coeffs, norm_radius, **kw):
    return dict(surface_type="forbes_q2d", freeform_coeffs=dict(coeffs), norm_radius=norm_radius, **kw)


def singlet(be, max_iter=100):
    """The gallery singlet: N-BK7, front sphere R 100 at the stop, rear Q-2D (R -100, k -0.8, the gallery's four
    coefficients, norm_radius 10, a radial aperture of 20).  3 fields x 3 wavelengths."""
    lens, done = _lens(be, 20.0, (0.0, 3.0, 5.0), WL3)
    lens.surfaces.add(index=1, radius=100, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=-100, conic=-0.8, thickness=100.0, material="air", aperture=20.0,
                      max_iter=max_iter, tol=1e-10, **q2d_kw(GALLERY, 10.0))
    lens.surfaces.add(index=3)
    return done()


M0_TERMS = {0: 2e-3, 1: -1.5e-3, 2: 8e-4, 3: -3e-4, 5: 1e-4}


def m0_only(be, qbfs=False):
    """An m = 0-only Q-2D rear surface, or (``qbfs=True``) its Q-bfs twin with the same radial terms."""
    lens, done = _lens(be, 16.0, (0.0, 3.0), (0.5876,))
    lens.surfaces.add(index=1, radius=60.0, thickness=6.0, material="N-BK7", is_stop=True)
    if qbfs:
        kw = dict(surface_type="forbes_qbfs", radial_terms=dict(M0_TERMS), norm_radius=9.0)
    else:
        kw = q2d_kw({("a", 0, n): v for n, v in M0_TERMS.items()}, 9.0)
    lens.surfaces.add(index=2, radius=-80.0, conic=-0.5, thickness=70.0, tol=1e-12, **kw)
    lens.surfaces.add(index=3)
    return done()


def high_order(be):
    """High azimuthal and radial orders: m <= 8, n <= 9, and a 6-term m = 1 list."""
    lens, done = _lens(be, 16.0, (0.0, 2.0, 4.0), (0.55,))
    lens.surfaces.add(index=1, radius=70.0, thickness=6.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=-90.0, conic=0.4, thickness=80.0, tol=1e-12,
                      **q2d_kw(freeform(8, 9, 2e-3, 7, m1_terms=6), 9.0))
    lens.surfaces.add(index=3)
    return done()


def vertex_window(be):
    """A Q-2D window at the stop (norm_radius 3 over an 8 mm beam): the fixture's collimated rays are placed on the
    vertex, on the axes and beyond u = 1, not generated."""
    lens, done = _lens(be, 8.0, (0.0,), (0.55,))
    lens.surfaces.add(index=1, radius=40.0, conic=-1.2, thickness=5.0, material="N-BK7", is_stop=True, tol=1e-12,
                      **q2d_kw(freeform(4, 5, 3e-3, 11, m1_terms=5), 3.0))
    lens.surfaces.add(index=2, radius=-30.0, thickness=30.0)
    lens.surfaces.add(index=3)
    return done()


def nested_reflection(be):
    """A reflective Q-2D (a concave freeform mirror), tilted, whose frame is defined inside a tilted, decentred carrier
    frame, followed by a plane."""
    from optiland.coordinate_system import CoordinateSystem

    lens, done = _lens(be, 10.0, (0.0, 3.0), (0.6,))
    lens.surfaces.add(index=1, radius=80.0, thickness=10.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=30.0)
    lens.surfaces.add(index=3, radius=-150.0, conic=-1.0, thickness=-30.0, material="mirror", tol=1e-12,
                      **q2d_kw(freeform(3, 4, 4e-3, 5), 9.0))
    lens.surfaces.add(index=4, radius=be.inf, thickness=0.0)
    done()
    carrier = CoordinateSystem(x=0.2, y=-0.1, z=45.0, rx=0.05, ry=-0.03, rz=0.1)
    lens.surfaces.surfaces[3].geometry.cs = CoordinateSystem(x=0.0, y=0.1, z=-1.0, rx=0.04, reference_cs=carrier)
    return lens


def infinite_radius(be):
    """A Q-2D departure on a plane base (infinite radius: z_base = 0, phi = 1) in front of a lens."""
    lens, done = _lens(be, 10.0, (0.0, 2.0, 4.0), (0.55,))
    lens.surfaces.add(index=1, radius=be.inf, thickness=4.0, material="N-BK7", is_stop=True, tol=1e-12,
                      **q2d_kw(freeform(5, 4, 5e-3, 3, m1_terms=4), 6.0))
    lens.surfaces.add(index=2, radius=-40.0, thickness=40.0)
    lens.surfaces.add(index=3)
    return done()


def aperture_coating(be):
    """A Q-2D surface with an aperture tree (an annulus minus an offset disk) and a SimpleCoating."""
    from optiland import physical_apertures as pa
    from optiland.coatings import SimpleCoating

    lens, done = _lens(be, 12.0, (0.0, 3.0), (0.55,))
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=-70.0, thickness=50.0, coating=SimpleCoating(0.9, 0.05), tol=1e-12,
                      aperture=pa.DifferenceAperture(pa.RadialAperture(r_max=5.5, r_min=0.8),
                                                     pa.OffsetRadialAperture(r_max=1.5, r_min=0.0, offset_x=3.0, offset_y=1.0)),
                      **q2d_kw(freeform(3, 3, 2e-3, 9), 7.0))
    lens.surfaces.add(index=3)
    return done()


def polarized(be, state=None):
    """``singlet`` with Fresnel coatings on every surface (the Q-2D included), unpolarized light by default."""
    from optiland.rays import PolarizationState

    lens = singlet(be)
    lens.surfaces.set_fresnel_coatings()
    lens.set_polarization(state if state is not None else PolarizationState(is_polarized=False))
    return lens


def max_iter_small(be):
    """``singlet`` with max_iter = 2: some rays stop before their Newton iteration has converged."""
    return singlet(be, max_iter=2)


def nan_rays(be):
    """A steep Q-2D rear surface (base R -9) behind a wide beam: the outer rays miss its base sphere (NaN start of the
    Newton iteration), and they stay NaN on every later surface."""
    lens, done = _lens(be, 22.0, (0.0, 4.0), (0.55,))
    lens.surfaces.add(index=1, radius=40.0, thickness=4.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=-9.0, thickness=30.0, tol=1e-12, **q2d_kw(freeform(2, 3, 1e-3, 13), 8.0))
    lens.surfaces.add(index=3)
    return done()


def bench_lens(be, q2d=True, M=6, N=6, m0_only=False):
    """The benchmark lens: an N-BK7 singlet whose rear surface is a Q-2D of order (M, N), or with ``m0_only`` only its
    m = 0 terms; with ``q2d=False`` the Q-bfs twin of those m = 0 terms."""
    lens, done = _lens(be, 20.0, (0.0, 2.0, 4.0), (0.5876,))
    lens.surfaces.add(index=1, radius=60.0, thickness=7.0, material="N-BK7", is_stop=True)
    coeffs = freeform(M, N, 2e-3, 21)
    if m0_only or not q2d:
        coeffs = {k: v for k, v in coeffs.items() if k[1] == 0}
    if q2d:
        kw = q2d_kw(coeffs, 12.5)
    else:
        kw = dict(surface_type="forbes_qbfs", radial_terms={k[2]: v for k, v in coeffs.items()}, norm_radius=12.5)
    lens.surfaces.add(index=2, radius=-90.0, conic=-1.5, thickness=95.0, tol=1e-10, **kw)
    lens.surfaces.add(index=3)
    return done()


BUILDERS = {
    "q2d_singlet": singlet,
    "q2d_m0_only": m0_only,
    "q2d_m0_qbfs_twin": lambda be: m0_only(be, qbfs=True),
    "q2d_high_order": high_order,
    "q2d_vertex": vertex_window,
    "q2d_nested_reflection": nested_reflection,
    "q2d_infinite_radius": infinite_radius,
    "q2d_aperture_coating": aperture_coating,
    "q2d_polarized": polarized,
    "q2d_max_iter": max_iter_small,
    "q2d_nan_rays": nan_rays,
}
