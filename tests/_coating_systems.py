"""Optical systems with thin-film, polarizer and retarder coatings (Optiland's ``ThinFilmCoating``,
``PolarizerCoating``, ``RetarderCoating``), built through the reference's own API.  Shared by the live tests
(``tests/test_polarization_coatings.py``); every builder needs the reference importable and takes its backend
module.  Each returns an ``Optic`` with its polarization state set."""
from __future__ import annotations

import numpy as np

WL3 = (0.4861, 0.5876, 0.6563)


def bbar(be):
    """The 4-layer MgF2 / TiO2 broadband anti-reflection stack (air -> N-BK7) of the reference's AR-coating tutorial."""
    from optiland.coatings import ThinFilmCoating
    from optiland.materials import IdealMaterial, Material

    mgf2, tio2 = Material("MgF2", reference="Li"), Material("TiO2", reference="Siefke")
    layers = [(mgf2, 94.0, "L1"), (tio2, 117.0, "H1"), (mgf2, 38.0, "L2"), (tio2, 14.0, "H2")]
    return ThinFilmCoating(IdealMaterial(n=1.0), Material("N-BK7", reference="SCHOTT"), layers)


def _state(lens, polarized=False, Ex=1.0, Ey=0.0, phase_x=0.0, phase_y=0.0):
    from optiland.rays import PolarizationState

    if polarized:
        lens.set_polarization(PolarizationState(is_polarized=True, Ex=Ex, Ey=Ey, phase_x=phase_x, phase_y=phase_y))
    else:
        lens.set_polarization(PolarizationState(is_polarized=False))
    return lens


def coated_doublet(be, coating="thin_film", polarized=False):
    """The tutorial's CoatedDoublet (an f/8 cemented-style doublet, 3 fields x 3 wavelengths) with the same coating on
    all four lens surfaces: ``"thin_film"`` (the BBAR stack), ``"fresnel"`` (bare interfaces) or None."""
    from optiland import optic as _optic
    from optiland.coatings import FresnelCoating
    from optiland.materials import IdealMaterial, Material

    c = {"thin_film": lambda: bbar(be),
         "fresnel": lambda: FresnelCoating(IdealMaterial(n=1.0), Material("N-BK7", reference="SCHOTT")),
         None: lambda: None}[coating]
    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=29.32908, thickness=0.7, material="N-BK7", is_stop=True, coating=c())
    lens.surfaces.add(index=2, radius=-20.06842, thickness=0.032, coating=c())
    lens.surfaces.add(index=3, radius=-20.08770, thickness=0.5780, material=("SF2", "schott"), coating=c())
    lens.surfaces.add(index=4, radius=-66.54774, thickness=47.3562, coating=c())
    lens.surfaces.add(index=5)
    lens.set_aperture(aperture_type="imageFNO", value=8.0)
    lens.fields.set_type(field_type="angle")
    for y in (0.0, 0.7, 1.0):
        lens.fields.add(y=y)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    lens.update_paraxial()
    lens.image_solve()
    return _state(lens, polarized)


def qwot_singlet(be):
    """A strongly curved singlet with a single-layer MgF2 quarter-wave coating (at 0.55 um) on both faces, wide field
    and aperture, so the angles of incidence reach about 60 degrees; one linear polarized state at 30 degrees."""
    from optiland import optic as _optic
    from optiland.coatings import ThinFilmCoating
    from optiland.materials import IdealMaterial, Material

    def qw():
        mgf2 = Material("MgF2", reference="Li")
        return ThinFilmCoating(IdealMaterial(n=1.0), IdealMaterial(n=1.5), [(mgf2, 550.0 / (4 * 1.38), "QW")])

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=12.0, thickness=6.0, material="N-BK7", is_stop=True, coating=qw())
    lens.surfaces.add(index=2, radius=-12.0, thickness=10.0, coating=qw())
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=16.0)
    lens.fields.set_type(field_type="angle")
    for y in (0.0, 20.0, 30.0):
        lens.fields.add(y=y)
    lens.wavelengths.add(value=0.55, is_primary=True)
    lens.wavelengths.add(value=0.65)
    return _state(lens, True, Ex=np.cos(np.pi / 6), Ey=np.sin(np.pi / 6))


def absorbing_fold(be):
    """A 45-degree fold mirror (tilted about x) coated with an absorbing layer (n 2.0, k 0.6, 80 nm) over a dielectric
    layer: reflection through the thin-film stack with k > 0."""
    from optiland import optic as _optic
    from optiland.coatings import ThinFilmCoating
    from optiland.materials import IdealMaterial

    film = ThinFilmCoating(IdealMaterial(n=1.0), IdealMaterial(n=1.0),
                           [(IdealMaterial(n=2.0, k=0.6), 80.0, "absorber"), (IdealMaterial(n=1.45), 120.0, "spacer")])
    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=60.0, thickness=5.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=30.0)
    lens.surfaces.add(index=3, radius=be.inf, thickness=-40.0, material="mirror", rx=np.pi / 4, coating=film)
    lens.surfaces.add(index=4, radius=be.inf, thickness=0.0, rx=np.pi / 2)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=5.0)
    lens.wavelengths.add(value=0.6, is_primary=True)
    return _state(lens, True, Ex=1.0, Ey=1.0, phase_y=np.pi / 2)


def zero_layer(be):
    """A stack with no layers (the bare interface of the TMM) on one face and a FresnelCoating on the other."""
    from optiland import optic as _optic
    from optiland.coatings import FresnelCoating, ThinFilmCoating
    from optiland.materials import IdealMaterial, Material

    glass = Material("N-BK7", reference="SCHOTT")
    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=40.0, thickness=5.0, material="N-BK7", is_stop=True,
                      coating=ThinFilmCoating(IdealMaterial(n=1.0), glass, []))
    lens.surfaces.add(index=2, radius=-40.0, thickness=30.0, coating=FresnelCoating(glass, IdealMaterial(n=1.0)))
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=8.0)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return _state(lens, False)


def polarizer_nested(be):
    """A linear polarizer (axis (1, 1, 0.2)) on a tilted plane whose frame sits inside a tilted, decentred carrier
    frame; 45-degree linear input."""
    from optiland import optic as _optic
    from optiland.coatings import PolarizerCoating
    from optiland.coordinate_system import CoordinateSystem

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=50.0, thickness=4.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=20.0)
    lens.surfaces.add(index=3, radius=be.inf, thickness=20.0, coating=PolarizerCoating(axis=(1.0, 1.0, 0.2)))
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=4.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    carrier = CoordinateSystem(x=0.3, y=-0.2, z=30.0, rx=0.2, ry=-0.1, rz=0.15)
    lens.surfaces.surfaces[3].geometry.cs = CoordinateSystem(x=0.0, y=0.1, z=-2.0, rx=0.15, reference_cs=carrier)
    return _state(lens, True, Ex=1.0, Ey=1.0)


def retarders(be):
    """A quarter-wave retarder given by theta (fast axis at 30 degrees) and a half-wave retarder given by an axis, on
    the two faces of a plate; circular-ish input."""
    from optiland import optic as _optic
    from optiland.coatings import RetarderCoating

    qw = RetarderCoating(np.pi / 2, axis=np.pi / 6)    # a scalar axis is the angle theta (jones.py:344-348)
    hw = RetarderCoating(np.pi, axis=(0.3, 1.0, 0.0))
    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=be.inf, thickness=2.0, material="N-BK7", is_stop=True, coating=qw)
    lens.surfaces.add(index=2, radius=-60.0, thickness=20.0, coating=hw)
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=6.0)
    lens.wavelengths.add(value=0.6328, is_primary=True)
    return _state(lens, True, Ex=1.0, Ey=0.5, phase_y=0.7)


def polarizer_refracting(be):
    """A linear polarizer on a refracting conic (air to glass) and a retarder on the refracting back face: there the
    ray bends, so p0 != p1 and the polarizer's J01 != J10 -- the orientation of the general 2x2 Jones block matters."""
    from optiland import optic as _optic
    from optiland.coatings import PolarizerCoating, RetarderCoating

    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=18.0, conic=-0.6, thickness=5.0, material="N-BK7", is_stop=True,
                      coating=PolarizerCoating(axis=(0.6, 0.7, 0.2)))
    lens.surfaces.add(index=2, radius=-40.0, thickness=25.0, coating=RetarderCoating(np.pi / 3, axis=(0.2, 1.0, 0.1)))
    lens.surfaces.add(index=3)
    lens.set_aperture(aperture_type="EPD", value=14.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=10.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return _state(lens, True, Ex=1.0, Ey=1.0, phase_y=0.4)


def mixed(be):
    """Thin film next to a FresnelCoating, a SimpleCoating, an aperture tree and two mirrors (one of them coated with a
    thin-film stack), 3 wavelengths."""
    from optiland import optic as _optic
    from optiland import physical_apertures as pa
    from optiland.coatings import FresnelCoating, SimpleCoating, ThinFilmCoating
    from optiland.materials import IdealMaterial, Material

    glass = Material("N-BK7", reference="SCHOTT")
    enh = ThinFilmCoating(IdealMaterial(n=1.0), IdealMaterial(n=1.0),
                          [(IdealMaterial(n=2.3), 60.0, "H"), (IdealMaterial(n=1.38), 100.0, "L"),
                           (IdealMaterial(n=0.12, k=3.4), 150.0, "metal")])
    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=45.0, thickness=5.0, material="N-BK7", is_stop=True, coating=bbar(be))
    lens.surfaces.add(index=2, radius=-45.0, thickness=20.0, coating=FresnelCoating(glass, IdealMaterial(n=1.0)),
                      aperture=pa.UnionAperture(pa.RadialAperture(r_max=6.0, r_min=1.0),
                                                pa.OffsetRadialAperture(r_max=2.5, r_min=0.0, offset_x=5.0, offset_y=1.0)))
    lens.surfaces.add(index=3, radius=be.inf, thickness=-25.0, material="mirror", rx=np.pi / 8, coating=enh)
    lens.surfaces.add(index=4, radius=-200.0, thickness=30.0, material="mirror", rx=np.pi / 8, coating=SimpleCoating(0.1, 0.9))
    lens.surfaces.add(index=5)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=3.0)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return _state(lens, False)


def film_on_doe_and_grating(be):
    """A thin-film coating on a radial-DOE surface, a polarizer on a ruled transmission grating: the new kernel variant
    on tables with phase and grating surfaces."""
    from optiland import optic as _optic
    from optiland.coatings import PolarizerCoating, ThinFilmCoating
    from optiland.materials import IdealMaterial, Material
    from optiland.phase import RadialPhaseProfile

    glass = Material("N-BK7", reference="SCHOTT")
    film = ThinFilmCoating(glass, IdealMaterial(n=1.0), [(IdealMaterial(n=1.38), 100.0, "L"), (IdealMaterial(n=2.1), 60.0, "H")])
    lens = _optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=80.0, thickness=4.0, material="N-BK7", is_stop=True)
    lens.surfaces.add(index=2, radius=be.inf, thickness=20.0, coating=film, phase_profile=RadialPhaseProfile([-1.5, 2e-4]))
    lens.surfaces.add(index=3, radius=be.inf, thickness=3.0, material="N-BK7")
    lens.surfaces.add(index=4, radius=be.inf, thickness=30.0, surface_type="grating", grating_order=1, grating_period=5.0,
                      groove_orientation_angle=0.2, coating=PolarizerCoating(axis=(1.0, 0.3, 0.0)))
    lens.surfaces.add(index=5)
    lens.set_aperture(aperture_type="EPD", value=10.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=3.0)
    for w in WL3:
        lens.wavelengths.add(value=w, is_primary=(w == 0.5876))
    return _state(lens, True, Ex=0.6, Ey=0.8, phase_y=1.1)


BUILDERS = {"coated_doublet": coated_doublet, "qwot_singlet": qwot_singlet, "absorbing_fold": absorbing_fold,
            "zero_layer": zero_layer, "polarizer_nested": polarizer_nested, "retarders": retarders,
            "polarizer_refracting": polarizer_refracting, "mixed": mixed, "film_on_doe_and_grating": film_on_doe_and_grating}
