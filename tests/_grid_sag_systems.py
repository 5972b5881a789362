"""Optical systems with grid-sag surfaces (Optiland's ``surface_type="grid_sag"``, ``GridSagGeometry``), built through
the reference's own API.  Shared by the fixture generator (``oracle/make_golden_grid_sag.py``), the live tests
(``tests/test_grid_sag.py``) and the benchmark (``scripts/bench_grid_sag.py``); every builder needs the reference
importable and takes its backend module."""
from __future__ import annotations

import numpy as np

WL3 = (0.4861, 0.5876, 0.6563)


def sphere_sag(x, y, R, k=0.0, coefs=()):
    """Sag of a conic (+ even asphere terms C_i r^(2i+2)) at (x, y)."""
    r2 = x * x + y * y
    z = r2 / (R * (1.0 + np.sqrt(1.0 - (1.0 + k) * r2 / R**2)))
    for i, c in enumerate(coefs):
        z = z + c * r2 ** (i + 1)
    return z


def sampled(xs, ys, fn):
    """(x list, y list, sag rows) of ``fn`` sampled on the nodes: row j at y_j (GridSagGeometry's layout)."""
    X, Y = np.meshgrid(np.asarray(xs, float), np.asarray(ys, float))
    return [float(v) for v in xs], [float(v) for v in ys], fn(X, Y).tolist()


def grid_kw(xs, ys, fn, **kw):
    x, y, z = sampled(xs, ys, fn)
    return dict(surface_type="grid_sag", x_coordinates=x, y_coordinates=y, sag_values=z, **kw)


def _lens(be, epd, fields, wls):
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    return lens, lambda: _finish(lens, epd, fields, wls)


def _finish(lens, epd, fields, wls):
    lens.set_aperture(aperture_type="EPD", value=epd)
    lens.fields.set_type(field_type="angle")
    for y in fields:
        lens.fields.add(y=y)
    for w in wls:
        lens.wavelengths.add(value=w, is_primary=(w == wls[len(wls) // 2]))
    return lens


def singlet(be, n=33, half=6.0, max_iter=100):
    """N-BK7 singlet whose rear surface is an n x n grid over [-half, half]^2 sampled from a sphere (R -60) plus an
    x y^2 departure; a node at 0, so the on-axis chief ray sits on the centre node.  3 fields x 3 wavelengths."""
    lens, done = _lens(be, 10.0, (0.0, 3.0, 5.0), WL3)
    nodes = np.linspace(-half, half, n)
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, thickness=45.0, max_iter=max_iter,
                      **grid_kw(nodes, nodes, lambda X, Y: sphere_sag(X, Y, -60.0) + 2e-4 * X * Y * Y))
    lens.surfaces.add(index=3)
    return done()


def nonuniform(be):
    """A grid with non-uniform x and y spacing (denser towards the edge in x, towards the centre in y) in front of a
    lens; sampled from a tilted toric-like cap."""
    lens, done = _lens(be, 10.0, (0.0, 2.0, 4.0), (0.55,))
    u = np.linspace(-1.0, 1.0, 25)
    xs = 6.5 * np.sign(u) * np.abs(u) ** 0.8
    ys = 6.5 * np.sign(u) * np.abs(u) ** 1.4
    lens.surfaces.add(index=1, thickness=4.0, material="N-BK7", is_stop=True,
                      **grid_kw(xs, ys, lambda X, Y: 0.012 * X * X + 0.008 * Y * Y + 0.01 * X - 3e-4 * X * Y))
    lens.surfaces.add(index=2, radius=-40.0, thickness=40.0)
    lens.surfaces.add(index=3)
    return done()


def nested_reflection(be):
    """A reflective grid (a shallow concave freeform mirror), tilted, whose frame is defined inside a tilted,
    decentred carrier frame, followed by a plane."""
    from optiland.coordinate_system import CoordinateSystem

    lens, done = _lens(be, 10.0, (0.0, 3.0), (0.6,))
    lens.surfaces.add(index=1, radius=80.0, thickness=10.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=30.0)
    nodes = np.linspace(-9.0, 9.0, 37)
    lens.surfaces.add(index=3, thickness=-30.0, material="mirror",
                      **grid_kw(nodes, nodes, lambda X, Y: sphere_sag(X, Y, -150.0) + 1e-4 * X**3))
    lens.surfaces.add(index=4, radius=be.inf, thickness=0.0)
    done()
    carrier = CoordinateSystem(x=0.2, y=-0.1, z=45.0, rx=0.05, ry=-0.03, rz=0.1)
    lens.surfaces.surfaces[3].geometry.cs = CoordinateSystem(x=0.0, y=0.1, z=-1.0, rx=0.04, reference_cs=carrier)
    return lens


def nan_patterns(be):
    """A grid smaller than the beam, placed behind a strongly converging lens: rays whose start point (t = 0, at the
    previous surface) lies outside the grid are NaN from the first iterate, rays that hit beyond the grid are NaN by the
    final test, and rays near the edge whose iterates step outside go NaN on the way."""
    lens, done = _lens(be, 12.0, (0.0, 4.0), (0.55,))
    nodes = np.linspace(-3.0, 3.0, 13)
    lens.surfaces.add(index=1, radius=25.0, thickness=6.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, thickness=20.0, **grid_kw(nodes, nodes, lambda X, Y: sphere_sag(X, Y, -30.0)))
    lens.surfaces.add(index=3)
    return done()


def nodes(be):
    """A plane-parallel grid window at the stop: an on-axis collimated beam whose rays sit exactly on nodes, on grid
    lines and on the inclusive upper edge (the fixture's rays are placed there, not generated)."""
    lens, done = _lens(be, 8.0, (0.0,), (0.55,))
    xs = np.linspace(-4.0, 4.0, 17)
    lens.surfaces.add(index=1, thickness=5.0, material="N-BK7", is_stop=True,
                      **grid_kw(xs, xs, lambda X, Y: 0.01 * X * X - 0.02 * Y * Y + 0.03 * X * Y + 0.05 * np.abs(X)))
    lens.surfaces.add(index=2, radius=-30.0, thickness=30.0)
    lens.surfaces.add(index=3)
    return done()


def aperture_coating(be):
    """A grid surface with an aperture tree (an annulus minus an offset disk) and a SimpleCoating."""
    from optiland import physical_apertures as pa
    from optiland.coatings import SimpleCoating

    lens, done = _lens(be, 12.0, (0.0, 3.0), (0.55,))
    nodes = np.linspace(-7.0, 7.0, 29)
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, thickness=50.0, coating=SimpleCoating(0.9, 0.05),
                      aperture=pa.DifferenceAperture(pa.RadialAperture(r_max=5.5, r_min=0.8),
                                                     pa.OffsetRadialAperture(r_max=1.5, r_min=0.0, offset_x=3.0, offset_y=1.0)),
                      **grid_kw(nodes, nodes, lambda X, Y: sphere_sag(X, Y, -70.0) + 5e-4 * X * Y))
    lens.surfaces.add(index=3)
    return done()


def polarized(be, state=None):
    """``singlet`` with Fresnel coatings on every surface (the grid included), unpolarized light by default."""
    from optiland.rays import PolarizationState

    lens = singlet(be)
    lens.surfaces.set_fresnel_coatings()
    lens.set_polarization(state if state is not None else PolarizationState(is_polarized=False))
    return lens


def doe_on_grid(be):
    """A radial DOE on a grid substrate: the phase interaction uses the geometry's unaligned normal, which for a grid
    points the opposite way to every other geometry's."""
    from optiland.phase import RadialPhaseProfile

    lens, done = _lens(be, 10.0, (0.0, 3.0), WL3)
    nodes = np.linspace(-6.0, 6.0, 25)
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, thickness=45.0, phase_profile=RadialPhaseProfile([-1.2, 3e-4]),
                      **grid_kw(nodes, nodes, lambda X, Y: sphere_sag(X, Y, -80.0)))
    lens.surfaces.add(index=3)
    return done()


def max_iter_small(be):
    """``singlet`` with max_iter = 2: some rays stop before their Newton iteration has converged."""
    return singlet(be, max_iter=2)


def asphere_lens(be, grid=True, n=65):
    """The benchmark lens: an N-BK7 singlet whose rear surface is an even asphere, or (``grid=True``) an n x n grid
    sampled from that asphere over the clear aperture."""
    lens, done = _lens(be, 20.0, (0.0, 2.0, 4.0), (0.5876,))
    lens.surfaces.add(index=1, radius=60.0, thickness=7.0, material="N-BK7", is_stop=True)
    R, k, coefs = -90.0, -1.5, (2e-6, -3e-9)
    if grid:
        nodes = np.linspace(-12.0, 12.0, n)
        lens.surfaces.add(index=2, thickness=95.0, tol=1e-10, **grid_kw(nodes, nodes, lambda X, Y: sphere_sag(X, Y, R, k, coefs)))
    else:
        lens.surfaces.add(index=2, radius=R, conic=k, thickness=95.0, surface_type="even_asphere",
                          coefficients=list(coefs), tol=1e-10)
    lens.surfaces.add(index=3)
    return done()


BUILDERS = {
    "grid_singlet": singlet,
    "grid_nonuniform": nonuniform,
    "grid_nested_reflection": nested_reflection,
    "grid_nan_patterns": nan_patterns,
    "grid_nodes": nodes,
    "grid_aperture_coating": aperture_coating,
    "grid_polarized": polarized,
    "grid_doe": doe_on_grid,
    "grid_max_iter": max_iter_small,
}
