"""Throughput of thin-film coatings on the polarized trace path: the coated doublet of tests/_coating_systems.py
(the reference's AR-coating tutorial system, the 4-layer MgF2 / TiO2 stack on all four lens surfaces), traced as
PolarizedRays with the unpolarized intensity epilogue, at 10 M rays, fp32 and fp64, with full per-surface records and
endpoint-only.  Arms: the thin-film stack, the same system with FresnelCoating (control: the same polarized update
without the stack), and the uncoated system (PolarizedRays, no coating).  Kernel time from CUDA events over repeated
launches; the HBM fraction is the bytes the trace must move (launch state and P matrix in, records or the final state,
P matrix and polarized intensity out) over that time, against the H100 SXM data sheet's 3.35 TB/s.  With --reference
the stock reference's torch-CUDA eager ``SurfaceGroup.trace`` of the thin-film system is timed as well (at --ref-rays
rays).  Needs the staged reference (oracle/_ref) to build the systems.  Prints one JSON object, with the card's name and
power limit.

    python scripts/bench_coating.py [--rays 10000000] [--reps 20] [--reference]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from scripts.bench_grating import PEAK_BW, card, time_kernel  # noqa: E402


def bytes_moved(n, rows, elem, record):
    """Read x, y, z, L, M, N, i, opd, w and the 18-value P matrix; write 8 values per record row with records (else the
    8 final values), the P matrix and the polarized intensity."""
    return n * elem * (9 + 18 + (8 * rows if record else 8) + 18 + 1)


def launch(n, be, lens):
    """n launch rays of the field Hy = 0.7 at the primary wavelength, uniform in the pupil (the reference's own ray
    generator, NumPy backend)."""
    rng = np.random.default_rng(0)
    rr, th = np.sqrt(rng.random(n)), 2 * np.pi * rng.random(n)
    Px, Py = rr * np.cos(th), rr * np.sin(th)
    r = lens.ray_tracer.ray_generator.generate_rays(0.0, 0.7, Px, Py, 0.5876)
    return {k: np.asarray(getattr(r, k), dtype=np.float64) for k in ("x", "y", "z", "L", "M", "N", "i", "w")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--ref-rays", type=int, default=1_000_000)
    args = ap.parse_args()

    import torch

    from optiland_b200.pack import pack_surface_group
    from optiland_b200.trace import DeviceTable, PolarizedRays, trace_device
    from tests import _coating_systems as CS     # (before the reference's own tests package is importable)
    from oracle.ref_import import import_reference

    assert torch.cuda.is_available(), "bench_coating.py needs a CUDA device"
    import_reference()
    import optiland.backend as be

    be.set_backend("numpy")
    lenses = {k: CS.coated_doublet(be, coating=c) for k, c in (("thin_film", "thin_film"), ("fresnel", "fresnel"),
                                                                 ("uncoated", None))}
    tables = {k: pack_surface_group(v.surfaces, [0.5876]) for k, v in lenses.items()}
    n = args.rays
    launch_np = launch(n, be, lenses["thin_film"])
    rows = tables["thin_film"].num_surfaces
    res = {"what": "coated doublet (4 lens surfaces, 6 surfaces), PolarizedRays with the unpolarized intensity epilogue: "
                   "one trace of N rays, CUDA events, median of reps",
           "rays": n, "card": card(), "results": [],
           "note": "ms: median event time of one trace minus that of the PolarizedRays input copy it includes"}
    for dtype in (torch.float32, torch.float64):
        elem = torch.finfo(dtype).bits // 8
        r = {k: torch.from_numpy(v).to("cuda", dtype) for k, v in launch_np.items()}

        def make():
            return PolarizedRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype, device="cuda")

        for record in (True, False):
            row = {"precision": str(dtype).split(".")[1], "mode": "full_record" if record else "endpoint_only"}
            for label, tab in tables.items():
                dt = DeviceTable(tab)

                def run():
                    return trace_device(dt, make(), 0, rows, record=record, polarization="unpolarized")

                t_copy, _ = time_kernel(make, args.reps)
                t, t_min = time_kernel(run, args.reps)
                tk = max(t - t_copy, 1e-9)
                b = bytes_moved(n, rows, elem, record)
                row[label] = {"ms": 1e3 * tk, "ms_min_incl_copy": 1e3 * t_min, "rays_per_s": n / tk,
                              "hbm_fraction": b / tk / PEAK_BW, "bytes": b}
            row["thin_film_over_fresnel_time"] = row["thin_film"]["ms"] / row["fresnel"]["ms"]
            res["results"].append(row)
        del r
        torch.cuda.empty_cache()
    if args.reference:
        res["reference_torch_cuda"] = reference_eager(args.ref_rays, max(3, args.reps // 4))
    print(json.dumps(res), flush=True)


def reference_eager(n, reps):
    """The stock reference's eager torch-CUDA SurfaceGroup.trace of the live thin-film doublet (no plugin)."""
    import torch

    import optiland.backend as be
    from optiland.rays import PolarizedRays

    CS = sys.modules["tests._coating_systems"]

    be.set_backend("torch")
    be.set_device("cuda")
    be.grad_mode.disable()
    out = []
    for prec in ("float32", "float64"):
        be.set_precision(prec)
        lens = CS.coated_doublet(be)
        rng = np.random.default_rng(0)
        rr, th = np.sqrt(rng.random(n)), 2 * np.pi * rng.random(n)
        Px, Py = be.array(rr * np.cos(th)), be.array(rr * np.sin(th))
        ts = []
        for k in range(reps + 1):
            rays = lens.ray_tracer.ray_generator.generate_rays(0.0, 0.7, Px, Py, 0.5876)
            assert isinstance(rays, PolarizedRays)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            lens.surfaces.trace(rays)
            torch.cuda.synchronize()
            if k:
                ts.append(time.perf_counter() - t0)
        t = float(np.median(ts))
        out.append({"precision": prec, "rays": n, "ms": 1e3 * t, "rays_per_s": n / t})
    be.set_device("cpu")
    be.set_backend("numpy")
    return out


if __name__ == "__main__":
    main()
