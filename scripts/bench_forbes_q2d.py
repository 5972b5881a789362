"""Throughput of a Forbes Q-2D freeform on the trace path: an N-BK7 singlet whose rear surface is a Q-2D of order
m, n <= 6 (tests/_forbes_q2d_systems.py ``bench_lens``), at 10 M rays (3 fields, one wavelength), fp32 and fp64, with
full per-surface records and endpoint-only.  Two controls: the same lens with only the Q-2D's m = 0 terms, timed beside
its Q-bfs twin (the same shape), which shows the cost of the Q-2D kernel variant apart from the cost of the m > 0 terms;
and (--reference) the stock reference's torch-CUDA eager ``SurfaceGroup.trace`` of the live Q-2D lens, at --ref-rays rays.
Kernel time from CUDA events over repeated launches (median); the HBM fraction is the bytes the trace must move
(computed from the shapes below) over that time, against the H100 SXM data sheet's 3.35 TB/s.  The systems are built
through the reference's API (staged under oracle/_ref by build()).  Prints one JSON object, with the card's name and power
limit read in the same run.

    python scripts/bench_forbes_q2d.py [--rays 10000000] [--reps 20] [--reference]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

PEAK_BW = 3.35e12


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"], out["max_sm_mhz"] = float(q[0]), float(q[1])
    except Exception as e:  # noqa: BLE001
        out["power_limit_w"] = f"unavailable: {e}"
    return out


def bytes_moved(n, rows, elem, n_wl, record):
    """HBM traffic of one trace: read x, y, z, L, M, N, i, opd (+ w with several wavelengths); write 8 values per
    record row with records (the final state is the last row), else the 8 final values."""
    reads = 8 + (1 if n_wl > 1 else 0)
    writes = 8 * rows if record else 8
    return n * elem * (reads + writes)


def time_kernel(fn, reps):
    import torch

    fn()
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(ts)), float(np.min(ts))


def systems(be):
    """{label: table} of the benchmark lens and its controls, and the launch rays as numpy arrays."""
    from optiland_b200.pack import pack_surface_group
    from tests import _forbes_q2d_systems as QS

    be.set_backend("numpy")
    lenses = {"q2d": QS.bench_lens(be), "q2d_m0_only": QS.bench_lens(be, m0_only=True),
              "qbfs_twin": QS.bench_lens(be, q2d=False)}
    rng = np.random.default_rng(0)
    n = 3 * 4096
    rr, th = np.sqrt(rng.random(n)), 2 * np.pi * rng.random(n)
    Hy = np.repeat([0.0, 0.5, 1.0], n // 3)
    rays = lenses["q2d"].ray_tracer.ray_generator.generate_rays(np.zeros(n), Hy, rr * np.cos(th), rr * np.sin(th), 0.5876)
    r = {k: np.array(getattr(rays, k), dtype=np.float64) for k in ("x", "y", "z", "L", "M", "N", "i", "w")}
    return {k: pack_surface_group(v.surfaces, [0.5876]) for k, v in lenses.items()}, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--ref-rays", type=int, default=100_000)
    args = ap.parse_args()

    import torch

    from oracle.ref_import import import_reference
    from optiland_b200.trace import DeviceTable, RealRays, trace_device

    assert torch.cuda.is_available(), "bench_forbes_q2d.py needs a CUDA device"
    from tests import _forbes_q2d_systems  # noqa: F401  (before the reference's own ``tests`` package is importable)

    import_reference()
    import optiland.backend as be

    tabs, base = systems(be)
    n = args.rays
    idx = np.random.default_rng(1).integers(0, base["x"].size, size=n)
    rows = tabs["q2d"].num_surfaces
    res = {"what": "N-BK7 singlet, rear surface a Forbes Q-2D (m, n <= 6); controls: its m = 0 terms alone as a Q-2D and as "
                   "the Q-bfs twin; 3 fields, 1 wavelength, 4 surfaces: one trace of N rays, CUDA events, median of reps",
           "rays": n, "card": card(), "results": [],
           "note": "ms: median event time of one trace minus that of the RealRays input copy it includes"}
    for dtype in (torch.float32, torch.float64):
        elem = torch.finfo(dtype).bits // 8
        r = {k: torch.from_numpy(v[idx]).to("cuda", dtype) for k, v in base.items()}
        for record in (True, False):
            row = {"precision": str(dtype).split(".")[1], "mode": "full_record" if record else "endpoint_only"}
            for label, tab in tabs.items():
                dt = DeviceTable(tab)

                def run():
                    rays = RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype, device="cuda")
                    return trace_device(dt, rays, 0, rows, record=record)

                # RealRays copies its inputs: time the copy alone and subtract it
                t_copy, _ = time_kernel(lambda: RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"],
                                                         dtype=dtype, device="cuda"), args.reps)
                t, t_min = time_kernel(run, args.reps)
                tk = max(t - t_copy, 1e-9)
                b = bytes_moved(n, rows, elem, tab.n_wl, record)
                row[label] = {"ms": 1e3 * tk, "ms_min_incl_copy": 1e3 * t_min, "rays_per_s": n / tk,
                              "hbm_fraction": b / tk / PEAK_BW, "bytes": b}
            row["q2d_m0_over_qbfs_time"] = row["q2d_m0_only"]["ms"] / row["qbfs_twin"]["ms"]
            row["q2d_over_q2d_m0_time"] = row["q2d"]["ms"] / row["q2d_m0_only"]["ms"]
            res["results"].append(row)
        del r
        torch.cuda.empty_cache()
    if args.reference:
        res["reference_torch_cuda"] = reference_eager(args.ref_rays, max(3, args.reps // 4))
    print(json.dumps(res), flush=True)


def reference_eager(n, reps):
    """The stock reference's eager torch-CUDA SurfaceGroup.trace of the live Q-2D lens (no plugin), per 1 M rays."""
    import torch

    from tests import _forbes_q2d_systems as QS
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    be.set_backend("torch")
    be.set_device("cuda")
    be.grad_mode.disable()
    out = []
    for prec in ("float32", "float64"):
        be.set_precision(prec)
        lens = QS.bench_lens(be)
        rng = np.random.default_rng(0)
        rr = np.sqrt(rng.random(n))
        th = 2 * np.pi * rng.random(n)
        Px, Py = be.array(rr * np.cos(th)), be.array(rr * np.sin(th))
        zeros = be.zeros_like(Px)
        ts = []
        for k in range(reps + 1):
            rays = lens.ray_tracer.ray_generator.generate_rays(zeros, zeros, Px, Py, 0.5876)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            lens.surfaces.trace(rays)
            torch.cuda.synchronize()
            if k:
                ts.append(time.perf_counter() - t0)
        t = float(np.median(ts))
        out.append({"precision": prec, "rays": n, "ms": 1e3 * t, "ms_per_1M_rays": 1e3 * t * 1e6 / n, "rays_per_s": n / t})
    be.set_device("cpu")
    be.set_backend("numpy")
    return out


if __name__ == "__main__":
    main()
