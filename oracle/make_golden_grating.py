"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/grating/*.npz from the UNMODIFIED reference: systems with ruled
gratings (Optiland's ``DiffractiveInteractionModel`` on ``PlaneGrating`` / ``StandardGratingGeometry``), built by
``tests/_grating_systems.py``.

    python -m oracle.make_golden_grating

Same layout as ``oracle/make_golden.py`` (``run_case``): the packed table of the live objects, the launch rays the
reference generated, and what its own ``SurfaceGroup.trace`` produced on the NumPy backend in fp64.  The fixtures live
in a subdirectory so that the suites parametrised over every top-level fixture do not pick them up.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from tests import _grating_systems as GS  # noqa: E402  (before the reference's own ``tests`` package is importable)

from oracle import make_golden as MG  # noqa: E402  (imports the reference)
from oracle.make_golden_phase import _rays  # noqa: E402

be = MG.be


def main():
    be.set_backend("numpy")
    os.makedirs(os.path.join(MG.OUT, "grating"), exist_ok=True)
    wl3 = list(GS.WL3)
    three = [(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)]
    specs = {
        "grating_spectrograph": (three, wl3, 1.0),
        "grating_curved_transmission": (three, [0.587], 1.0),
        "grating_concave_reflection": (three, [0.587], 1.0),
        "grating_nested_reflection": (three, [0.6], 1.0),
        "grating_high_orders": ([(0.0, 0.0), (0.5, 0.6), (0.6, -1.0)], [0.55], 1.0),
        "grating_aperture_coating": (three, [0.55], 1.2),
        "grating_and_doe": (three, wl3, 1.0),
    }
    for name, (fields, wls, rmax) in specs.items():
        lens = GS.BUILDERS[name](be)
        rays = _rays(lens, 120, 500 + len(name), fields, wls, rmax)
        MG.run_case("grating/" + name, lens, rays, wls)
    # unpolarized PolarizedRays with Fresnel coatings on every surface, the grating included
    name = "grating_polarized"
    lens = GS.BUILDERS[name](be)
    rays = _rays(lens, 80, 700, three, wl3)
    assert type(rays).__name__ == "PolarizedRays"
    i0 = np.array(rays._i0)
    k0 = np.stack([np.array(rays._L0), np.array(rays._M0), np.array(rays._N0)])
    probe = copy.deepcopy(rays)
    lens2 = GS.BUILDERS[name](be)
    lens2.surfaces.trace(probe)
    probe.update_intensity(lens2.polarization_state)
    MG.run_case("grating/" + name, lens, rays, wl3, polarized=True,
                extra={"i0": i0, "k0": k0, "final_intensity_unpolarized": np.array(probe.i)})


if __name__ == "__main__":
    main()
