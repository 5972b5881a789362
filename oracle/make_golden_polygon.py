"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/polygon_aperture/*.npz from the UNMODIFIED reference: systems
with polygon apertures (Optiland's ``PolygonAperture`` / ``FileAperture``), built by ``tests/_polygon_systems.py``.

    python -m oracle.make_golden_polygon

Same layout as ``oracle/make_golden.py`` (``run_case``), with one difference: the reference runs on its TORCH backend
(CPU, fp64), not on NumPy.  The plugin stands in for the torch backend, whose point-in-polygon test is the half-open
crossing count the kernel reproduces; the NumPy backend's test is matplotlib's ``Path.contains_points``, which decides
points on an edge differently and is not installed where this runs.  The outline file of ``polygon_file_outline``
(``outline_240.txt``, written here when missing) is a data fixture beside the others.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from tests import _polygon_systems as PS  # noqa: E402  (before the reference's own ``tests`` package is importable)

from oracle import make_golden as MG  # noqa: E402  (imports the reference)
from oracle.make_golden_phase import _rays  # noqa: E402

be = MG.be


def write_outline():
    if os.path.exists(PS.OUTLINE_FILE):
        return
    x, y = PS.wavy_outline(240)
    with open(PS.OUTLINE_FILE, "w") as f:
        f.write("// x y in mm: a lobed mechanical outline, 240 vertices, counter-clockwise\n")
        for a, b in zip(x, y):
            f.write(f"{a:.9f} {b:.9f}\n")


def placed_rays():
    """On-axis collimated rays at z = -1 on the L-shaped stop of ``polygon_edge_window`` (and the bow-tie behind it):
    on every vertex, level with vertices, on vertical, horizontal and slanted edges, at the bow-tie's crossing point,
    one ulp-scale step either side of edges, and NaN."""
    from optiland.rays import RealRays

    rng = np.random.default_rng(23)
    lx, ly = PS.L_SHAPE
    bx, by = PS.BOW_TIE
    px = [lx, bx, rng.uniform(-5, 5, 80), rng.choice(np.concatenate([lx, bx]), 80), rng.uniform(-5, 5, 80)]
    py = [ly, by, rng.choice(np.concatenate([ly, by]), 80), rng.uniform(-5, 5, 80), rng.uniform(-5, 5, 80)]
    t = rng.uniform(0, 1, 40)
    px.append(-4.0 + 8.0 * t)                  # on the bow-tie's slanted edge (-4, -3) -> (4, 3), up to rounding
    py.append(-3.0 + 6.0 * t)
    e = np.array([0.0, 1e-13, -1e-13])
    px.append(np.concatenate([1.0 + e, 4.0 + e, -4.0 + e, np.zeros(3), [np.nan, 0.5, np.nan]]))
    py.append(np.concatenate([np.full(3, 2.0), np.full(3, -2.0), np.full(3, 1.0), e, [0.5, np.nan, np.nan]]))
    x, y = np.concatenate(px), np.concatenate(py)
    n = x.size
    return RealRays(be.array(x), be.array(y), be.full((n,), -1.0), be.zeros(n), be.zeros(n), be.ones(n), be.ones(n),
                    be.full((n,), 0.55))


def main():
    be.set_backend("torch")
    be.set_device("cpu")
    be.set_precision("float64")
    be.grad_mode.disable()
    os.makedirs(os.path.join(MG.OUT, "polygon_aperture"), exist_ok=True)
    write_outline()
    wl3 = list(PS.WL3)
    two = [(0.0, 0.0), (0.0, 1.0)]
    specs = {
        "polygon_hexagon_mirror": (two, [0.55], 1.0),
        "polygon_cassegrain_spider": (two, [0.55], 1.0),
        "polygon_concave_bowtie": ([(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)], wl3, 1.0),
        "polygon_clockwise": (two, [0.55], 1.0),
        "polygon_nested_tilted": (two, [0.6], 1.0),
        "polygon_asphere_grid": (two, [0.55], 1.0),
        "polygon_file_outline": (two, [0.55], 1.0),
        "polygon_scaled": (two, [0.55], 1.0),
        "polygon_nan_rays": (two, [0.55], 1.0),
    }
    for name, (fields, wls, rmax) in specs.items():
        lens = PS.BUILDERS[name](be)
        rays = _rays(lens, 150, 700 + len(name), fields, wls, rmax)
        MG.run_case("polygon_aperture/" + name, lens, rays, wls)
    MG.run_case("polygon_aperture/polygon_edge_window", PS.edge_window(be), placed_rays(), [0.55])
    # unpolarized PolarizedRays with Fresnel coatings on every surface
    name = "polygon_polarized"
    three = [(0.0, 0.0), (0.0, 0.7), (0.3, 1.0)]
    lens = PS.BUILDERS[name](be)
    rays = _rays(lens, 80, 790, three, wl3)
    assert type(rays).__name__ == "PolarizedRays"
    i0 = np.array(rays._i0)
    k0 = np.stack([np.array(rays._L0), np.array(rays._M0), np.array(rays._N0)])
    probe = copy.deepcopy(rays)
    lens2 = PS.BUILDERS[name](be)
    lens2.surfaces.trace(probe)
    probe.update_intensity(lens2.polarization_state)
    MG.run_case("polygon_aperture/" + name, lens, rays, wl3, polarized=True,
                extra={"i0": i0, "k0": k0, "final_intensity_unpolarized": np.array(probe.i)})
    be.set_backend("numpy")


if __name__ == "__main__":
    main()
