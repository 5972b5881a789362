"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/forbes_q2d/*.npz from the UNMODIFIED reference: systems with
Forbes Q-2D surfaces (Optiland's ``ForbesQ2dGeometry``), built by ``tests/_forbes_q2d_systems.py``.

    python -m oracle.make_golden_forbes_q2d

Same layout as ``oracle/make_golden.py`` (``run_case``): the packed table of the live objects, the launch rays the
reference generated (or, for ``q2d_vertex``, rays placed on the vertex, on the axes and beyond the normalisation radius),
and what its own ``SurfaceGroup.trace`` produced on the NumPy backend in fp64.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from tests import _forbes_q2d_systems as QS  # noqa: E402  (before the reference's own ``tests`` package is importable)

from oracle import make_golden as MG  # noqa: E402  (imports the reference)
from oracle.make_golden_phase import _rays  # noqa: E402

be = MG.be


def vertex_rays():
    """Collimated rays at z = -1 on the vertex (both signs of zero), on the x and y axes, on the diagonals, around the
    normalisation radius 3 (u = 1 +- 1e-9, beyond it) and scattered over the 8 mm beam."""
    from optiland.rays import RealRays

    rng = np.random.default_rng(31)
    t = np.linspace(-3.9, 3.9, 27)
    px = [np.array([0.0, -0.0, 0.0, -0.0, 1e-13, 0.0]), t, np.zeros(27), t / np.sqrt(2)]
    py = [np.array([0.0, 0.0, -0.0, -0.0, 0.0, 1e-13]), np.zeros(27), t, -t / np.sqrt(2)]
    ang = rng.uniform(0, 2 * np.pi, 24)
    for rad in (3.0 * (1 - 1e-9), 3.0, 3.0 * (1 + 1e-9), 3.5):
        px.append(rad * np.cos(ang)); py.append(rad * np.sin(ang))
    r = 4.0 * np.sqrt(rng.uniform(0, 1, 120)); a = rng.uniform(0, 2 * np.pi, 120)
    px.append(r * np.cos(a)); py.append(r * np.sin(a))
    x, y = np.concatenate(px), np.concatenate(py)
    n = x.size
    return RealRays(x, y, np.full(n, -1.0), np.zeros(n), np.zeros(n), np.ones(n), np.ones(n), np.full(n, 0.55))


def main():
    be.set_backend("numpy")
    os.makedirs(os.path.join(MG.OUT, "forbes_q2d"), exist_ok=True)
    wl3 = list(QS.WL3)
    three = [(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)]
    specs = {
        "q2d_singlet": (three, wl3, 1.0),
        "q2d_m0_only": ([(0.0, 0.0), (0.0, 1.0)], [0.5876], 1.0),
        "q2d_m0_qbfs_twin": ([(0.0, 0.0), (0.0, 1.0)], [0.5876], 1.0),
        "q2d_high_order": (three, [0.55], 1.0),
        "q2d_nested_reflection": ([(0.0, 0.0), (0.0, 1.0)], [0.6], 1.0),
        "q2d_infinite_radius": (three, [0.55], 1.0),
        "q2d_aperture_coating": ([(0.0, 0.0), (0.0, 1.0)], [0.55], 1.2),
        "q2d_max_iter": (three, wl3, 1.0),
        "q2d_nan_rays": ([(0.0, 0.0), (0.0, 1.0)], [0.55], 1.0),
    }
    for name, (fields, wls, rmax) in specs.items():
        lens = QS.BUILDERS[name](be)
        # (the twins share their launch rays: the same seed)
        rays = _rays(lens, 120, 700 + len(name.replace("_qbfs_twin", "_only")), fields, wls, rmax)
        MG.run_case("forbes_q2d/" + name, lens, rays, wls)
    MG.run_case("forbes_q2d/q2d_vertex", QS.BUILDERS["q2d_vertex"](be), vertex_rays(), [0.55])
    # unpolarized PolarizedRays with Fresnel coatings on every surface, the Q-2D included
    name = "q2d_polarized"
    lens = QS.BUILDERS[name](be)
    rays = _rays(lens, 80, 790, three, wl3)
    assert type(rays).__name__ == "PolarizedRays"
    i0 = np.array(rays._i0)
    k0 = np.stack([np.array(rays._L0), np.array(rays._M0), np.array(rays._N0)])
    probe = copy.deepcopy(rays)
    lens2 = QS.BUILDERS[name](be)
    lens2.surfaces.trace(probe)
    probe.update_intensity(lens2.polarization_state)
    MG.run_case("forbes_q2d/" + name, lens, rays, wl3, polarized=True,
                extra={"i0": i0, "k0": k0, "final_intensity_unpolarized": np.array(probe.i)})


if __name__ == "__main__":
    main()
