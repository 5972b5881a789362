"""Optical systems with phase-profile surfaces (Optiland's ``PhaseInteractionModel``: diffractive optics, gratings),
built through the reference's own API.  Shared by the fixture generator (``oracle/make_golden_phase.py``) and the live
tests (``tests/test_phase_surfaces.py``); every builder needs the reference importable and takes its backend module."""
from __future__ import annotations

import numpy as np

WL3 = (0.4861, 0.5876, 0.6563)


def doe_achromat(be):
    """Hybrid refractive-diffractive achromat: an N-BK7 plano-convex lens whose plane back carries a radial DOE
    (positive diffractive power, opposite dispersion), 3 fields x 3 wavelengths."""
    from optiland import optic as _optic
    from optiland.phase import RadialPhaseProfile

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=55.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=95.0, phase_profile=RadialPhaseProfile([-1.2, 3e-4, -2e-7]))
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=14.0)
    lens.fields.set_type(field_type="angle")
    for y in (0.0, 3.0, 5.0):
        lens.fields.add(y=y)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return lens


def doe_with_plane(be):
    """``doe_achromat`` with the phase surface replaced by a plain plane (the same geometry, refraction only)."""
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=55.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=95.0)
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=14.0)
    lens.fields.set_type(field_type="angle")
    for y in (0.0, 3.0, 5.0):
        lens.fields.add(y=y)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return lens


def radial_on_substrates(be):
    """Radial phase on a conic and on an even-asphere substrate.  Their normals point to -z, so the reference sends
    the transmitted rays BACKWARDS (N < 0): the reversed-ray behaviour the kernel reproduces."""
    from optiland import optic as _optic
    from optiland.phase import RadialPhaseProfile

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=100.0, conic=-0.6, thickness=6.0, material="N-BK7", is_stop=True,
                      phase_profile=RadialPhaseProfile([-2.0, 1e-3]))
    lens.surfaces.add(index=2, radius=-100.0, thickness=-40.0, surface_type="even_asphere", conic=0.2,
                      coefficients=[1e-5, -2e-8], tol=1e-12, phase_profile=RadialPhaseProfile([0.8]))
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=4.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def linear_gratings(be):
    """Two transmission gratings at a grating angle != 0 (orders -1 and 2, efficiency 0.7 on the second) strong enough
    that part of the field goes evanescent there (intensity 0, finite grazing direction)."""
    from optiland import optic as _optic
    from optiland.phase import LinearGratingPhaseProfile

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=be.inf, thickness=3.0, material="N-BK7", is_stop=True,
                      phase_profile=LinearGratingPhaseProfile(period=0.004, angle=0.35, order=-1))
    lens.surfaces.add(index=2, radius=be.inf, thickness=20.0,
                      phase_profile=LinearGratingPhaseProfile(period=0.0012, angle=-0.8, order=2, efficiency=0.7))
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=8.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=20.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def reflective_grating(be):
    """A tilted plane reflection grating (a grating mirror folding the beam) followed by a tilted image plane."""
    from optiland import optic as _optic
    from optiland.phase import LinearGratingPhaseProfile

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=80.0, thickness=10.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=30.0)
    lens.surfaces.add(index=3, radius=be.inf, thickness=-30.0, material="mirror", rx=np.pi / 8,
                      phase_profile=LinearGratingPhaseProfile(period=0.002, angle=np.pi / 2, order=1))
    lens.surfaces.add(index=4, radius=be.inf, thickness=0.0, rx=np.pi / 4)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=3.0)
    lens.wavelengths.add(value=0.6, is_primary=True)
    return lens


def constant_phase(be):
    """A constant phase on a plane inside a singlet: an OPD shift -phi / k0 that depends on the wavelength."""
    from optiland import optic as _optic
    from optiland.phase import ConstantPhaseProfile

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=40.0, thickness=4.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=3.0, material="N-BK7", phase_profile=ConstantPhaseProfile(2.5))
    lens.surfaces.add(index=3, radius=-80.0, thickness=50.0)
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=3.0)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return lens


def phase_aperture_coating(be):
    """A DOE with an aperture tree (union of an annulus and an offset disk) and a SimpleCoating."""
    from optiland import optic as _optic
    from optiland import physical_apertures as pa
    from optiland.coatings import SimpleCoating
    from optiland.phase import RadialPhaseProfile

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=60.0, coating=SimpleCoating(0.9, 0.05),
                      phase_profile=RadialPhaseProfile([-1.5, 2e-4]),
                      aperture=pa.UnionAperture(pa.RadialAperture(r_max=5.0, r_min=1.0),
                                                pa.OffsetRadialAperture(r_max=2.5, r_min=0.0, offset_x=4.5, offset_y=1.0)))
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=14.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=4.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def doe_polarized(be):
    """``doe_achromat`` with Fresnel coatings on every surface (the DOE included) and unpolarized light."""
    from optiland.rays import PolarizationState

    lens = doe_achromat(be)
    lens.surfaces.set_fresnel_coatings()
    lens.set_polarization(PolarizationState(is_polarized=False))
    return lens


BUILDERS = {
    "phase_doe_achromat": doe_achromat,
    "phase_substrates": radial_on_substrates,
    "phase_linear_gratings": linear_gratings,
    "phase_reflective_grating": reflective_grating,
    "phase_constant": constant_phase,
    "phase_aperture_coating": phase_aperture_coating,
    "phase_doe_polarized": doe_polarized,
}
