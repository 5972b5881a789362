"""Optical systems with ruled gratings (Optiland's ``surface_type="grating"``: a ``DiffractiveInteractionModel`` on a
``PlaneGrating`` or a ``StandardGratingGeometry``), built through the reference's own API.  Shared by the fixture
generator (``oracle/make_golden_grating.py``), the live tests (``tests/test_ruled_gratings.py``) and the benchmark
(``scripts/bench_grating.py``); every builder needs the reference importable and takes its backend module."""
from __future__ import annotations

import numpy as np

WL3 = (0.4861, 0.5876, 0.6563)


def spectrograph(be, grating=True):
    """Lens, tilted plane transmission grating (200 lines/mm, first order, grooves turned by 0.2 rad) on the back of
    a glass plate, camera lens: 3 fields x 3 wavelengths.  ``grating=False`` puts a plain plane in the grating's
    place (the same geometry, refraction only)."""
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=80.0, thickness=4.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=-80.0, thickness=10.0)
    lens.surfaces.add(index=3, radius=be.inf, thickness=3.0, material="N-BK7", rx=0.05)
    kw = dict(surface_type="grating", grating_order=1, grating_period=5.0, groove_orientation_angle=0.2) if grating else {}
    lens.surfaces.add(index=4, radius=be.inf, thickness=15.0, rx=0.05, **kw)
    lens.surfaces.add(index=5, radius=60.0, thickness=5.0, material="N-BK7")
    lens.surfaces.add(index=6, radius=-60.0, thickness=40.0)
    lens.surfaces.add(index=7)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    for y in (0.0, 2.0, 3.0):
        lens.fields.add(y=y)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return lens


def curved_transmission(be):
    """A conic transmission grating (R 50, k -0.5, order -1, grooves turned by 0.3 rad): the grating vector follows
    the groove tangent on the curved surface."""
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=be.inf, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=50.0, conic=-0.5, thickness=30.0, surface_type="grating", grating_order=-1,
                      grating_period=5.0, groove_orientation_angle=0.3)
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=15.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=10.0)
    lens.wavelengths.add(value=0.587, is_primary=True)
    return lens


def concave_reflection(be):
    """A concave reflection grating (R 70, order 1, 3 um period, grooves turned by 0.25 rad) with the image plane
    30 mm before it: the reference returns the negative of the reflected direction, so the image is reached at t < 0."""
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=70.0, conic=0.2, thickness=-30.0, material="mirror", surface_type="grating",
                      is_stop=True, grating_order=1, grating_period=3.0, groove_orientation_angle=0.25)
    lens.surfaces.add(index=2)
    lens.set_aperture(aperture_type="EPD", value=15.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=10.0)
    lens.wavelengths.add(value=0.587, is_primary=True)
    return lens


def nested_reflection(be):
    """A tilted plane reflection grating (order -1, 1.5 um period, grooves along x) whose frame is defined inside a
    tilted, decentred carrier frame, followed by a plane."""
    from optiland import optic as _optic
    from optiland.coordinate_system import CoordinateSystem

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=80.0, thickness=10.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=30.0)
    lens.surfaces.add(index=3, radius=be.inf, thickness=-30.0, material="mirror", surface_type="grating",
                      grating_order=-1, grating_period=1.5, groove_orientation_angle=np.pi / 2)
    lens.surfaces.add(index=4, radius=be.inf, thickness=0.0)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=3.0)
    lens.wavelengths.add(value=0.6, is_primary=True)
    carrier = CoordinateSystem(x=0.2, y=-0.1, z=45.0, rx=0.3, ry=-0.05, rz=0.1)
    lens.surfaces.surfaces[3].geometry.cs = CoordinateSystem(x=0.0, y=0.1, z=-1.0, rx=0.1, reference_cs=carrier)
    return lens


def high_orders(be):
    """Second and third orders on a glass-to-air plane grating (1.1 um period): part of the field goes evanescent,
    which the reference leaves as NaN directions with the intensity unchanged."""
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=be.inf, thickness=3.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=2.0, material="N-BK7", surface_type="grating",
                      grating_order=2, grating_period=2.2, groove_orientation_angle=0.1)
    lens.surfaces.add(index=3, radius=be.inf, thickness=20.0, surface_type="grating", grating_order=3,
                      grating_period=3.3, groove_orientation_angle=-0.2)
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=8.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=20.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def aperture_coating(be):
    """A plane grating with an aperture tree (union of an annulus and an offset disk) and a SimpleCoating."""
    from optiland import optic as _optic
    from optiland import physical_apertures as pa
    from optiland.coatings import SimpleCoating

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=60.0, coating=SimpleCoating(0.9, 0.05), surface_type="grating",
                      grating_order=-1, grating_period=4.0, groove_orientation_angle=0.0,
                      aperture=pa.UnionAperture(pa.RadialAperture(r_max=5.0, r_min=1.0),
                                                pa.OffsetRadialAperture(r_max=2.5, r_min=0.0, offset_x=4.5, offset_y=1.0)))
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=14.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=4.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def polarized(be, state=None):
    """``spectrograph`` with Fresnel coatings on every surface (the grating included), unpolarized light by
    default."""
    from optiland.rays import PolarizationState

    lens = spectrograph(be)
    lens.surfaces.set_fresnel_coatings()
    lens.set_polarization(state if state is not None else PolarizationState(is_polarized=False))
    return lens


def grating_and_doe(be):
    """A radial DOE and a plane grating in one system (a spectrograph with a diffractive corrector)."""
    from optiland import optic as _optic
    from optiland.phase import RadialPhaseProfile

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=55.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=10.0, phase_profile=RadialPhaseProfile([-1.2, 3e-4]))
    lens.surfaces.add(index=3, radius=be.inf, thickness=80.0, surface_type="grating", grating_order=1,
                      grating_period=6.0, groove_orientation_angle=0.1, rx=-0.03)
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=3.0)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return lens


BUILDERS = {
    "grating_spectrograph": spectrograph,
    "grating_curved_transmission": curved_transmission,
    "grating_concave_reflection": concave_reflection,
    "grating_nested_reflection": nested_reflection,
    "grating_high_orders": high_orders,
    "grating_aperture_coating": aperture_coating,
    "grating_polarized": polarized,
    "grating_and_doe": grating_and_doe,
}
