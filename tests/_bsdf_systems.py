"""Optical systems with BSDF surfaces (Optiland's ``LambertianBSDF`` / ``GaussianBSDF`` set as a surface's ``bsdf``),
built through the reference's own API, and the launch rays traced through them, for the BSDF tests
(``tests/test_bsdf_scatter.py``); every builder needs the reference importable and takes its backend module."""
from __future__ import annotations

import numpy as np

from tests._grid_sag_systems import grid_kw, sphere_sag


def _lens(be):
    from optiland import optic as _optic

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    return lens


def _finish(lens, epd=10.0, wl=0.55):
    lens.set_aperture(aperture_type="EPD", value=epd)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.wavelengths.add(value=wl, is_primary=True)
    return lens


def gaussian_lens(be, sigma=0.1):
    """A singlet whose back surface is a Gaussian diffuser: the scatter sends its rays BACKWARDS (the conic's normal
    points to -z), as the reference does."""
    from optiland.scatter import GaussianBSDF

    lens = _lens(be)
    lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=-60.0, thickness=40.0, bsdf=GaussianBSDF(sigma))
    lens.surfaces.add(index=3)
    return _finish(lens)


def plane_diffuser(be, sigma=0.05):
    """A lens, then a flat Gaussian diffuser (the plane's normal is +z: forward scatter) in front of the detector."""
    from optiland.scatter import GaussianBSDF

    lens = _lens(be)
    lens.surfaces.add(index=1, radius=40.0, thickness=4.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=30.0)
    lens.surfaces.add(index=3, radius=be.inf, thickness=20.0, bsdf=GaussianBSDF(sigma))
    lens.surfaces.add(index=4)
    return _finish(lens)


def lambertian_mirror(be):
    """A concave Lambertian mirror (a white screen)."""
    from optiland.scatter import LambertianBSDF

    lens = _lens(be)
    lens.surfaces.add(index=1, radius=-200.0, thickness=-80.0, material="mirror", is_stop=True, bsdf=LambertianBSDF())
    lens.surfaces.add(index=2)
    return _finish(lens)


def two_bsdf_tilted(be):
    """Two BSDF surfaces in one system: a Gaussian diffuser with a radial aperture (clipped rays are scattered too) and
    a SimpleCoating, then a Lambertian plane tilted and decentred inside a tilted carrier frame."""
    from optiland.coatings import SimpleCoating
    from optiland.coordinate_system import CoordinateSystem
    from optiland.physical_apertures import RadialAperture
    from optiland.scatter import GaussianBSDF, LambertianBSDF

    lens = _lens(be)
    lens.surfaces.add(index=1, radius=30.0, thickness=3.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=-45.0, thickness=25.0, bsdf=GaussianBSDF(0.2), aperture=RadialAperture(r_max=3.0),
                      coating=SimpleCoating(0.8, 0.1))
    lens.surfaces.add(index=3, radius=be.inf, thickness=20.0, bsdf=LambertianBSDF())
    lens.surfaces.add(index=4)
    lens = _finish(lens)
    carrier = CoordinateSystem(x=0.2, y=-0.1, z=28.0, rx=0.05, ry=-0.03, rz=0.1)
    lens.surfaces.surfaces[3].geometry.cs = CoordinateSystem(x=0.0, y=0.1, z=0.0, rx=0.3, ry=0.1, reference_cs=carrier)
    return lens


def grid_diffuser(be):
    """A Gaussian diffuser on a grid-sag surface: its normal points to +z, so the scatter goes forwards."""
    from optiland.scatter import GaussianBSDF

    lens = _lens(be)
    lens.surfaces.add(index=1, radius=80.0, thickness=4.0, material="N-BK7", is_stop=True)
    xs = np.linspace(-8.0, 8.0, 17)
    lens.surfaces.add(index=2, thickness=30.0, bsdf=GaussianBSDF(0.15),
                      **grid_kw(xs, xs, lambda X, Y: sphere_sag(X, Y, -120.0)))
    lens.surfaces.add(index=3)
    return _finish(lens)


def doe_and_grating(be):
    """A Gaussian BSDF on a radial DOE, then a Lambertian BSDF on a ruled plane grating."""
    from optiland.phase import RadialPhaseProfile
    from optiland.scatter import GaussianBSDF, LambertianBSDF

    lens = _lens(be)
    lens.surfaces.add(index=1, radius=be.inf, thickness=20.0, material="N-BK7", is_stop=True,
                      phase_profile=RadialPhaseProfile([-1.2, 3e-4]), bsdf=GaussianBSDF(0.05))
    lens.surfaces.add(index=2, surface_type="grating", radius=be.inf, thickness=30.0, grating_order=1,
                      grating_period=2.0, groove_orientation_angle=0.2, bsdf=LambertianBSDF())
    lens.surfaces.add(index=3)
    return _finish(lens)


def gaussian_sigma(be, sigma):
    """A flat Gaussian diffuser alone (sigma = 0: no scatter beyond the reference's frame arithmetic; a large sigma:
    many rejections per ray)."""
    from optiland.scatter import GaussianBSDF

    lens = _lens(be)
    lens.surfaces.add(index=1, radius=be.inf, thickness=10.0, is_stop=True, bsdf=GaussianBSDF(sigma))
    lens.surfaces.add(index=2)
    return _finish(lens)


def shared_instance(be, sigma=0.1):
    """ONE GaussianBSDF object set on two flat diffusers in series: each surface must draw its own numbers."""
    from optiland.scatter import GaussianBSDF

    d = GaussianBSDF(sigma)
    lens = _lens(be)
    lens.surfaces.add(index=1, radius=be.inf, thickness=10.0, is_stop=True, bsdf=d)
    lens.surfaces.add(index=2, radius=be.inf, thickness=10.0, bsdf=d)
    lens.surfaces.add(index=3)
    return _finish(lens)


BUILDERS = {
    "shared_instance": shared_instance,
    "gaussian_lens": gaussian_lens,
    "plane_diffuser": plane_diffuser,
    "lambertian_mirror": lambertian_mirror,
    "two_bsdf_tilted": two_bsdf_tilted,
    "grid_diffuser": grid_diffuser,
    "doe_and_grating": doe_and_grating,
    "sigma_zero": lambda be: gaussian_sigma(be, 0.0),
    "grazing": lambda be: gaussian_sigma(be, 1.5),
}


def launch_rays(n, seed, spread=0.15, radius=4.0, grazing=False):
    """Launch state at z = -5 (dict of fp64 arrays): positions in a disk, directions within ``spread`` rad of the axis.
    ``grazing``: directions near 80 degrees, including some with L >= 0.999, so that the other arbitrary vector is
    taken.  The last rays are NaN."""
    rng = np.random.default_rng(seed)
    r = radius * np.sqrt(rng.uniform(0, 1, n))
    t = rng.uniform(0, 2 * np.pi, n)
    if grazing:
        th = rng.uniform(1.2, 1.55, n)
    else:
        th = spread * np.sqrt(rng.uniform(0, 1, n))
    ph = rng.uniform(0, 2 * np.pi, n)
    L, M, N = np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)
    if grazing:
        k = n // 8
        L[:k], M[:k], N[:k] = 0.9995, 0.0, np.sqrt(1 - 0.9995**2)
    rays = dict(x=r * np.cos(t), y=r * np.sin(t), z=np.full(n, -5.0), L=L, M=M, N=N, i=np.ones(n), w=np.full(n, 0.55))
    for k in ("x", "L"):
        rays[k][-3:] = np.nan
    return rays
