"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/phase/*.npz from the UNMODIFIED reference: systems with
phase-profile surfaces (Optiland's ``PhaseInteractionModel``), built by ``tests/_phase_systems.py``.

    python -m oracle.make_golden_phase

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

from tests import _phase_systems as PS  # noqa: E402  (before the reference's own ``tests`` package is importable)

from oracle import make_golden as MG  # noqa: E402  (imports the reference)

be = MG.be


def _rays(lens, n_per, seed, fields, wavelengths, rmax=1.0):
    """Launch rays of every (field, wavelength) pair, interleaved in one batch (trace_generic's call shape)."""
    Px, Py, Hx, Hy, W = [], [], [], [], []
    for j, (hx, hy) in enumerate(fields):
        for k, wl in enumerate(wavelengths):
            px, py = MG.disk(n_per, seed=seed + 10 * j + k, rmax=rmax)
            Px.append(px); Py.append(py)
            Hx.append(np.full(n_per, hx)); Hy.append(np.full(n_per, hy)); W.append(np.full(n_per, wl))
    cat = np.concatenate
    return MG.gen(lens, cat(Hx), cat(Hy), cat(Px), cat(Py), cat(W))


def main():
    be.set_backend("numpy")
    os.makedirs(os.path.join(MG.OUT, "phase"), exist_ok=True)
    wl3 = list(PS.WL3)
    three = [(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)]
    specs = {
        "phase_doe_achromat": (three, wl3, 1.0),
        "phase_substrates": (three, [0.55], 1.0),
        "phase_linear_gratings": ([(0.0, 0.0), (0.5, 0.6), (0.6, -1.0)], [0.55], 1.0),
        "phase_reflective_grating": (three, [0.6], 1.0),
        "phase_constant": ([(0.0, 0.0), (0.0, 1.0)], wl3, 1.0),
        "phase_aperture_coating": (three, [0.55], 1.2),
    }
    for name, (fields, wls, rmax) in specs.items():
        lens = PS.BUILDERS[name](be)
        rays = _rays(lens, 120, 100 + len(name), fields, wls, rmax)
        MG.run_case("phase/" + name, lens, rays, wls)
    # unpolarized PolarizedRays with Fresnel coatings on every surface, the DOE included
    name = "phase_doe_polarized"
    lens = PS.BUILDERS[name](be)
    rays = _rays(lens, 80, 300, three, wl3)
    assert type(rays).__name__ == "PolarizedRays"
    i0 = np.array(rays._i0)
    k0 = np.stack([np.array(rays._L0), np.array(rays._M0), np.array(rays._N0)])
    probe = copy.deepcopy(rays)
    lens2 = PS.BUILDERS[name](be)
    lens2.surfaces.trace(probe)
    probe.update_intensity(lens2.polarization_state)
    MG.run_case("phase/" + name, lens, rays, wl3, polarized=True,
                extra={"i0": i0, "k0": k0, "final_intensity_unpolarized": np.array(probe.i)})


if __name__ == "__main__":
    main()
