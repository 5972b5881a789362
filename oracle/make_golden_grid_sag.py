"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/grid_sag/*.npz from the UNMODIFIED reference: systems with
grid-sag surfaces (Optiland's ``GridSagGeometry``), built by ``tests/_grid_sag_systems.py``.

    python -m oracle.make_golden_grid_sag

Same layout as ``oracle/make_golden.py`` (``run_case``): the packed table of the live objects, the launch rays the
reference generated (or, for ``grid_nodes``, rays placed on the grid's nodes and lines), and what its own
``SurfaceGroup.trace`` produced on the NumPy backend in fp64.  The fixtures live in a subdirectory so that the suites
parametrised over every top-level fixture do not pick them up.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from tests import _grid_sag_systems as GS  # noqa: E402  (before the reference's own ``tests`` package is importable)

from oracle import make_golden as MG  # noqa: E402  (imports the reference)
from oracle.make_golden_phase import _rays  # noqa: E402

be = MG.be


def node_rays():
    """On-axis collimated rays at z = -1 exactly on the 17 x 17 nodes of ``grid_nodes``, on its grid lines, on the
    inclusive upper edges x = 4 / y = 4, and 1e-6 outside the grid (outside in fp32 too)."""
    from optiland.rays import RealRays

    nodes = np.linspace(-4.0, 4.0, 17)
    X, Y = np.meshgrid(nodes, nodes)
    rng = np.random.default_rng(17)
    px = [X.ravel()]
    py = [Y.ravel()]
    u = rng.uniform(-4.0, 4.0, 60)
    px += [rng.choice(nodes, 60), u]                 # on vertical lines / on horizontal lines
    py += [u, rng.choice(nodes, 60)]
    e = rng.uniform(-4.0, 4.0, 20)
    px += [np.full(20, 4.0), e, np.array([4.0, -4.0, 4.0 + 1e-6, -4.0 - 1e-6, 0.0, 0.0])]
    py += [e, np.full(20, 4.0), np.array([4.0, -4.0, 0.0, 0.0, 4.0 + 1e-6, -4.0 - 1e-6])]
    x, y = np.concatenate(px), np.concatenate(py)
    n = x.size
    return RealRays(x, y, np.full(n, -1.0), np.zeros(n), np.zeros(n), np.ones(n), np.ones(n), np.full(n, 0.55))


def main():
    be.set_backend("numpy")
    os.makedirs(os.path.join(MG.OUT, "grid_sag"), exist_ok=True)
    wl3 = list(GS.WL3)
    specs = {
        "grid_singlet": ([(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)], wl3, 1.0),
        "grid_nonuniform": ([(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)], [0.55], 1.0),
        "grid_nested_reflection": ([(0.0, 0.0), (0.0, 1.0)], [0.6], 1.0),
        "grid_nan_patterns": ([(0.0, 0.0), (0.0, 1.0)], [0.55], 1.0),
        "grid_aperture_coating": ([(0.0, 0.0), (0.0, 1.0)], [0.55], 1.2),
        "grid_doe": ([(0.0, 0.0), (0.0, 1.0)], wl3, 1.0),
        "grid_max_iter": ([(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)], wl3, 1.0),
    }
    for name, (fields, wls, rmax) in specs.items():
        lens = GS.BUILDERS[name](be)
        rays = _rays(lens, 120, 900 + len(name), fields, wls, rmax)
        MG.run_case("grid_sag/" + name, lens, rays, wls)
    MG.run_case("grid_sag/grid_nodes", GS.nodes(be), node_rays(), [0.55])
    # unpolarized PolarizedRays with Fresnel coatings on every surface, the grid included
    name = "grid_polarized"
    three = [(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)]
    lens = GS.BUILDERS[name](be)
    rays = _rays(lens, 80, 990, three, wl3)
    assert type(rays).__name__ == "PolarizedRays"
    i0 = np.array(rays._i0)
    k0 = np.stack([np.array(rays._L0), np.array(rays._M0), np.array(rays._N0)])
    probe = copy.deepcopy(rays)
    lens2 = GS.BUILDERS[name](be)
    lens2.surfaces.trace(probe)
    probe.update_intensity(lens2.polarization_state)
    MG.run_case("grid_sag/" + name, lens, rays, wl3, polarized=True,
                extra={"i0": i0, "k0": k0, "final_intensity_unpolarized": np.array(probe.i)})


if __name__ == "__main__":
    main()
