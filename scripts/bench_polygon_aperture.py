"""Throughput of polygon apertures on the trace path: a two-mirror telescope (tests/_polygon_systems.py ``cassegrain``)
whose primary carries (a) the radial obscuration only (the control, no polygon), (b) a 6-vertex hexagon, (c) the spider
difference tree (an annulus minus three vanes given as polygons) and (d) a 300-vertex outline such as a FileAperture
reads, at 10 M rays (2 fields, one wavelength), fp32 and fp64, with full per-surface records and endpoint-only.  (b) and
(c) are on the one-bucket side of the prepared table's choice (olb_prep.h PG_LINEAR_MAX), (d) on the bucketed side.
Kernel time from CUDA events over repeated launches (median); the HBM fraction is the bytes the trace must move (computed
from the shapes below) over that time, against the H100 SXM data sheet's 3.35 TB/s.  With --reference the stock
reference's torch-CUDA eager ``SurfaceGroup.trace`` of the same live systems is timed as well, at --ref-rays rays (its
polygon test materialises rays x vertices matrices: 12 GB per fp32 temporary at 10 M rays x 300 vertices).  The systems are built
through the reference's API (staged under oracle/_ref by build()).  Prints one JSON object, with the card's name and
power limit read in the same run.  Without a CUDA device the script fails.

    python scripts/bench_polygon_aperture.py [--rays 10000000] [--reps 20] [--reference]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

from bench_grid_sag import PEAK_BW, bytes_moved, card, time_kernel  # noqa: E402

WL = 0.55


def apertures():
    from tests import _polygon_systems as PS

    return {"radial": "radial", "hexagon": "hexagon", "spider": "spider", "outline300": PS.wavy_outline(300, 9.5)}


def systems(be):
    """({label: table}, launch rays as numpy arrays) of the benchmark telescope."""
    from optiland_b200.pack import pack_surface_group
    from tests import _polygon_systems as PS

    be.set_backend("numpy")
    lenses = {k: PS.cassegrain(be, aperture=a) for k, a in apertures().items()}
    rng = np.random.default_rng(0)
    n = 2 * 8192
    rr, th = np.sqrt(rng.random(n)), 2 * np.pi * rng.random(n)
    Hy = np.repeat([0.0, 1.0], n // 2)
    rays = lenses["radial"].ray_tracer.ray_generator.generate_rays(np.zeros(n), Hy, rr * np.cos(th), rr * np.sin(th), WL)
    r = {k: np.array(getattr(rays, k), dtype=np.float64) for k in ("x", "y", "z", "L", "M", "N", "i", "w")}
    return {k: pack_surface_group(v.surfaces, [WL]) for k, v in lenses.items()}, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--ref-rays", type=int, default=1_000_000)
    args = ap.parse_args()

    import torch

    from oracle.ref_import import import_reference
    from optiland_b200.trace import DeviceTable, RealRays, trace_device

    assert torch.cuda.is_available(), "bench_polygon_aperture.py needs a CUDA device"
    from tests import _polygon_systems  # noqa: F401  (before the reference's own ``tests`` package is importable)

    import_reference()
    import optiland.backend as be

    tables, base = systems(be)
    n = args.rays
    idx = np.random.default_rng(1).integers(0, base["x"].size, size=n)
    jitter = np.random.default_rng(2).uniform(-1e-3, 1e-3, (2, n))      # every ray its own hit point
    rows = tables["radial"].num_surfaces
    res = {"what": "two-mirror telescope, primary aperture: radial obscuration (control) / hexagon / spider difference "
                   "tree / 300-vertex outline; 2 fields, 1 wavelength, 4 surfaces: one trace of N rays, CUDA events, "
                   "median of reps",
           "rays": n, "card": card(), "results": [],
           "note": "ms: median event time of one trace minus that of the RealRays input copy it includes"}
    for dtype in (torch.float32, torch.float64):
        elem = torch.finfo(dtype).bits // 8
        r = {k: torch.from_numpy(v[idx] + (jitter[0] if k == "x" else jitter[1] if k == "y" else 0.0)).to("cuda", dtype)
             for k, v in base.items()}
        for record in (True, False):
            row = {"precision": str(dtype).split(".")[1], "mode": "full_record" if record else "endpoint_only"}
            t_copy, _ = time_kernel(lambda: RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"],
                                                     dtype=dtype, device="cuda"), args.reps)
            for label, tab in tables.items():
                dt = DeviceTable(tab)

                def run():
                    rays = RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype, device="cuda")
                    trace_device(dt, rays, 0, rows, record=record)
                    return rays

                t, t_min = time_kernel(run, args.reps)
                tk = max(t - t_copy, 1e-9)
                b = bytes_moved(n, rows, elem, tab.n_wl, record)
                row[label] = {"ms": 1e3 * tk, "ms_min_incl_copy": 1e3 * t_min, "rays_per_s": n / tk,
                              "hbm_fraction": b / tk / PEAK_BW, "bytes": b}
                if record:      # (the rays' final state is a view of the last record row)
                    row[label]["clipped_fraction"] = float((run().i == 0).double().mean())
            for label in ("hexagon", "spider", "outline300"):
                row[label + "_over_radial_time"] = row[label]["ms"] / row["radial"]["ms"]
            res["results"].append(row)
        del r
        torch.cuda.empty_cache()
    if args.reference:
        res["reference_torch_cuda"] = reference_eager(args.ref_rays, max(3, args.reps // 4))
    print(json.dumps(res), flush=True)


def reference_eager(n, reps):
    """The stock reference's eager torch-CUDA SurfaceGroup.trace of the live telescopes (no plugin) at ``n`` rays."""
    import torch

    from tests import _polygon_systems as PS
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    be.set_backend("torch")
    be.set_device("cuda")
    be.grad_mode.disable()
    out = []
    for prec in ("float32", "float64"):
        be.set_precision(prec)
        for label, a in apertures().items():
            lens = PS.cassegrain(be, aperture=a)
            rng = np.random.default_rng(0)
            rr = np.sqrt(rng.random(n))
            th = 2 * np.pi * rng.random(n)
            Px, Py = be.array(rr * np.cos(th)), be.array(rr * np.sin(th))
            zeros = be.zeros_like(Px)
            ts = []
            for k in range(reps + 1):
                rays = lens.ray_tracer.ray_generator.generate_rays(zeros, zeros, Px, Py, WL)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                lens.surfaces.trace(rays)
                torch.cuda.synchronize()
                if k:
                    ts.append(time.perf_counter() - t0)
            t = float(np.median(ts))
            out.append({"precision": prec, "aperture": label, "rays": n, "ms": 1e3 * t, "ms_per_1M_rays": 1e3 * t * 1e6 / n,
                        "rays_per_s": n / t})
            del lens, rays
            torch.cuda.empty_cache()
    be.set_device("cpu")
    be.set_backend("numpy")
    return out


if __name__ == "__main__":
    main()
