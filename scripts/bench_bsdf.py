"""BSDF scatter on the trace kernel: 10 M rays through a singlet whose back surface is a Gaussian diffuser (and a
Lambertian variant), each against the same system without a BSDF as the control, in fp32 and fp64, with full records
and endpoint only.  Kernel time is the trace kernel's own duration in a torch.profiler run (median of --reps launches
after a warm-up), so the BSDF rows' status word and its read-back are not counted; the share of 3.35 TB/s
(H100 SXM HBM3) is for the bytes the trace must move: the launch state read (8 arrays) plus the record rows (8 arrays
per surface) or the final state (8 arrays) written.  Prints one JSON line per case, then the card's name and power
limit read in the same run.

    python scripts/bench_bsdf.py [--rays 10000000] [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12


def systems():
    from optiland_b200 import table as T

    def lens(bsdf, sigma=0.0):
        return T.SurfaceTable([
            T.SurfaceSpec(kind=T.GEOM_NOOP),
            T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=50.0, n2=[1.5168]),
            T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=-60.0, t=[0, 0, 5.0], n1=[1.5168], bsdf=bsdf, bsdf_sigma=sigma,
                          bsdf_seed=12345 if bsdf else 0),
            T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 45.0]),
        ], [0.55])

    return {"control": lens(T.BSDF_NONE), "gaussian_0.1": lens(T.BSDF_GAUSSIAN, 0.1),
            "lambertian": lens(T.BSDF_LAMBERTIAN)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch

    from optiland_b200.trace import DeviceTable, RealRays, trace_device

    n = args.rays
    rng = np.random.default_rng(1)
    r = 4.0 * np.sqrt(rng.uniform(0, 1, n))
    t = rng.uniform(0, 2 * np.pi, n)
    launch = dict(x=r * np.cos(t), y=r * np.sin(t), z=np.full(n, -5.0), L=np.zeros(n), M=np.zeros(n), N=np.ones(n),
                  i=np.ones(n), w=np.full(n, 0.55))
    for name, table in systems().items():
        dt = DeviceTable(table, "cuda:0")
        S = table.num_surfaces
        for dtype in (torch.float32, torch.float64):
            es = 4 if dtype == torch.float32 else 8
            base = RealRays(*[launch[k] for k in ("x", "y", "z", "L", "M", "N", "i", "w")], dtype=dtype, device="cuda:0")
            for record in (True, False):
                def once():
                    rr = RealRays.__new__(RealRays)
                    for k in ("x", "y", "z", "L", "M", "N", "i", "w", "opd"):
                        setattr(rr, k, getattr(base, k).clone())
                    rr.L0 = rr.M0 = rr.N0 = None
                    return rr
                for rep in range(2):
                    trace_device(dt, once(), 0, S, record=record, rng_stream=rep)
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for rep in range(args.reps):
                        rr = once()        # (the copies are kernels of their own; only trace_kernel is counted)
                        trace_device(dt, rr, 0, S, record=record, rng_stream=rep)
                        del rr
                    torch.cuda.synchronize()
                times = [e.device_time * 1e-6 for e in prof.events() if "trace_kernel" in e.name]
                assert len(times) == args.reps, len(times)
                med = float(np.median(times))
                nbytes = n * es * (8 + 8 * (S if record else 1))
                print(json.dumps({"system": name, "dtype": str(dtype).split(".")[-1],
                                  "records": "full" if record else "endpoint", "rays": n, "kernel_ms": med * 1e3,
                                  "GB_moved": nbytes / 1e9, "hbm_share": nbytes / med / HBM_BPS,
                                  "features": dt.features}), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": q}))


if __name__ == "__main__":
    main()
