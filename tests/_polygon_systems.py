"""Optical systems with polygon apertures (Optiland's ``PolygonAperture`` and ``FileAperture``), built through the
reference's own API.  Shared by the fixture generator (``oracle/make_golden_polygon.py``), the live tests
(``tests/test_polygon_apertures.py``) and the benchmark (``scripts/bench_polygon_aperture.py``); every builder needs
the reference importable and takes its backend module."""
from __future__ import annotations

import os

import numpy as np

WL3 = (0.4861, 0.5876, 0.6563)
OUTLINE_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "polygon_aperture", "outline_240.txt")


def regular(n, radius, phase=0.0, cx=0.0, cy=0.0):
    """(x, y) of a regular n-gon, counter-clockwise."""
    th = phase + 2.0 * np.pi * np.arange(n) / n
    return cx + radius * np.cos(th), cy + radius * np.sin(th)


def vane(angle, r0, r1, half_width):
    """(x, y) of a thin rectangle from radius r0 to r1 along ``angle``: one spider vane."""
    c, s = np.cos(angle), np.sin(angle)
    u = np.array([r0, r1, r1, r0])
    v = np.array([-half_width, -half_width, half_width, half_width])
    return c * u - s * v, s * u + c * v


def wavy_outline(n, radius=9.0):
    """(x, y) of a closed outline of n vertices with lobes: what a measured mechanical outline looks like."""
    th = 2.0 * np.pi * np.arange(n) / n
    r = radius * (1.0 + 0.07 * np.cos(5 * th) + 0.03 * np.sin(11 * th))
    return r * np.cos(th), r * np.sin(th)


# an L-shaped (concave) stop and a bow-tie whose edges cross at the origin; integer coordinates, so rays can be
# placed exactly on vertices' levels, on edges and on horizontal edges
L_SHAPE = (np.array([-4.0, 4.0, 4.0, 1.0, 1.0, -4.0]), np.array([-4.0, -4.0, 0.0, 0.0, 4.0, 4.0]))
BOW_TIE = (np.array([-4.0, 4.0, -4.0, 4.0]), np.array([-3.0, 3.0, 3.0, -3.0]))


def _poly(xy):
    from optiland import physical_apertures as pa

    return pa.PolygonAperture(x=list(map(float, xy[0])), y=list(map(float, xy[1])))


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


def hexagon_mirror(be):
    """One hexagonal segment: a concave conic mirror whose aperture is a hexagon smaller than the beam."""
    lens, done = _lens(be, 14.0, (0.0, 0.5), (0.55,))
    lens.surfaces.add(index=1, radius=-200.0, conic=-0.9, thickness=-90.0, material="mirror", is_stop=True,
                      aperture=_poly(regular(6, 6.0, phase=0.1)))
    lens.surfaces.add(index=2)
    return done()


def spider_aperture(r_max=10.0, r_min=2.0, half_width=0.15):
    """DifferenceAperture(annulus, union of three vanes at 90, 210 and 330 degrees), the vanes as polygons."""
    from optiland import physical_apertures as pa

    vanes = [_poly(vane(np.deg2rad(a), 0.0, r_max + 1.0, half_width)) for a in (90.0, 210.0, 330.0)]
    return pa.DifferenceAperture(pa.RadialAperture(r_max=r_max, r_min=r_min),
                                 pa.UnionAperture(pa.UnionAperture(vanes[0], vanes[1]), vanes[2]))


def cassegrain(be, aperture="spider", epd=21.0):
    """A two-mirror telescope whose primary carries ``aperture``: "spider" (the difference tree above), "radial" (the
    obscuration alone), "hexagon", an (x, y) outline, or a ready aperture object."""
    from optiland import physical_apertures as pa

    if isinstance(aperture, str):
        aperture = {"spider": spider_aperture, "radial": lambda: pa.RadialAperture(r_max=10.0, r_min=2.0),
                    "hexagon": lambda: _poly(regular(6, 10.0))}[aperture]()
    elif isinstance(aperture, tuple):
        aperture = _poly(aperture)
    lens, done = _lens(be, epd, (0.0, 0.2), (0.55,))
    lens.surfaces.add(index=1, radius=-120.0, conic=-1.05, thickness=-40.0, material="mirror", is_stop=True, aperture=aperture)
    lens.surfaces.add(index=2, radius=-60.0, conic=-2.5, thickness=60.0, material="mirror")
    lens.surfaces.add(index=3)
    return done()


def concave_and_bowtie(be):
    """An L-shaped stop on the front of a singlet and a self-intersecting bow-tie on its back."""
    lens, done = _lens(be, 12.0, (0.0, 3.0), WL3)
    lens.surfaces.add(index=1, radius=60.0, thickness=5.0, material="N-BK7", is_stop=True, aperture=_poly(L_SHAPE))
    lens.surfaces.add(index=2, radius=-80.0, thickness=50.0, aperture=_poly(BOW_TIE))
    lens.surfaces.add(index=3)
    return done()


def clockwise(be):
    """A pentagon given clockwise."""
    x, y = regular(5, 5.0, phase=0.3)
    lens, done = _lens(be, 12.0, (0.0, 3.0), (0.55,))
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True, aperture=_poly((x[::-1], y[::-1])))
    lens.surfaces.add(index=2, radius=-70.0, thickness=45.0)
    lens.surfaces.add(index=3)
    return done()


def nested_tilted(be):
    """A hexagonal fold mirror, tilted and decentred, whose frame is defined inside a tilted carrier frame."""
    from optiland.coordinate_system import CoordinateSystem

    lens, done = _lens(be, 10.0, (0.0, 2.0), (0.6,))
    lens.surfaces.add(index=1, radius=80.0, thickness=10.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=30.0)
    lens.surfaces.add(index=3, radius=be.inf, thickness=-30.0, material="mirror", aperture=_poly(regular(6, 4.0, cx=0.3, cy=-0.2)))
    lens.surfaces.add(index=4, radius=be.inf, thickness=0.0)
    done()
    carrier = CoordinateSystem(x=0.2, y=-0.1, z=45.0, rx=0.05, ry=-0.03, rz=0.1)
    lens.surfaces.surfaces[3].geometry.cs = CoordinateSystem(x=0.0, y=0.1, z=-1.0, rx=0.04, reference_cs=carrier)
    return lens


def asphere_and_grid(be):
    """A triangle on an even asphere, then an octagon on a grid-sag substrate."""
    from tests import _grid_sag_systems as GS

    lens, done = _lens(be, 12.0, (0.0, 3.0), (0.55,))
    lens.surfaces.add(index=1, radius=50.0, conic=-0.5, thickness=5.0, material="N-BK7", is_stop=True,
                      surface_type="even_asphere", coefficients=[1e-5, -2e-8], aperture=_poly(regular(3, 7.0, phase=0.2)))
    nodes = np.linspace(-7.0, 7.0, 29)
    lens.surfaces.add(index=2, thickness=45.0, aperture=_poly(regular(8, 4.5)),
                      **GS.grid_kw(nodes, nodes, lambda X, Y: GS.sphere_sag(X, Y, -70.0) + 3e-4 * X * Y))
    lens.surfaces.add(index=3)
    return done()


def polarized(be):
    """``concave_and_bowtie`` with Fresnel coatings on every surface and unpolarized light."""
    from optiland.rays import PolarizationState

    lens = concave_and_bowtie(be)
    lens.surfaces.set_fresnel_coatings()
    lens.set_polarization(PolarizationState(is_polarized=False))
    return lens


def file_outline(be, path=OUTLINE_FILE):
    """A ``FileAperture`` (a measured outline of 240 vertices, read from a text file) on the front of a singlet."""
    from optiland import physical_apertures as pa

    lens, done = _lens(be, 20.0, (0.0, 2.0), (0.55,))
    lens.surfaces.add(index=1, radius=80.0, thickness=6.0, material="N-BK7", is_stop=True,
                      aperture=pa.FileAperture(path, skip_header=1))
    lens.surfaces.add(index=2, radius=-120.0, thickness=70.0)
    lens.surfaces.add(index=3)
    return done()


def scaled(be):
    """A hexagon built at radius 10 and then ``scale()``d by 0.45: the live ``vertices`` are what clips."""
    lens = clockwise(be)
    ap = _poly(regular(6, 10.0))
    ap.scale(0.45)
    lens.surfaces.surfaces[1].aperture = ap
    return lens


def edge_window(be):
    """The L-shaped stop on a plane window at z = 0: on-axis collimated rays placed on it stay where they are placed."""
    lens, done = _lens(be, 10.0, (0.0,), (0.55,))
    lens.surfaces.add(index=1, radius=be.inf, thickness=3.0, material="N-BK7", is_stop=True, aperture=_poly(L_SHAPE))
    lens.surfaces.add(index=2, radius=be.inf, thickness=10.0, aperture=_poly(BOW_TIE))
    lens.surfaces.add(index=3)
    return done()


def nan_rays(be):
    """A steep front surface that the outer rays miss (NaN in band), then a hexagonal stop: NaN rays are clipped."""
    lens, done = _lens(be, 12.0, (0.0, 4.0), (0.55,))
    lens.surfaces.add(index=1, radius=5.5, thickness=3.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=10.0, aperture=_poly(regular(6, 3.0)))
    lens.surfaces.add(index=3)
    return done()


BUILDERS = {
    "polygon_hexagon_mirror": hexagon_mirror,
    "polygon_cassegrain_spider": cassegrain,
    "polygon_concave_bowtie": concave_and_bowtie,
    "polygon_clockwise": clockwise,
    "polygon_nested_tilted": nested_tilted,
    "polygon_asphere_grid": asphere_and_grid,
    "polygon_polarized": polarized,
    "polygon_file_outline": file_outline,
    "polygon_scaled": scaled,
    "polygon_edge_window": edge_window,
    "polygon_nan_rays": nan_rays,
}
