"""Robust ray aiming on the device: ``Optic.trace`` of the three sample systems that use ``set_aiming("robust",
cache=True)`` (ProjectionLens120FOV, ProjectionLens160FOV, WideAngle170FOV) at every field, with a 4-ring hexapolar
pupil and a 64 x 64 uniform pupil, once with every solve as one aim launch (``plugin._state["device_aim"] = True``) and
once through the reference's Newton-Broyden loop of subset traces (``False``), alternated in the same run.

* wall time: host clock around ``Optic.trace`` followed by ``torch.cuda.synchronize()``, median of ``--reps`` (the
  aimer's cache is cleared before every trace, so every trace aims);
* ``olb_launch_count`` per trace;
* the aim kernel's own time under ``torch.profiler`` for one solve of 10^6 rays (WideAngle170FOV, half field, a
  converging step of the continuation), median of ``--reps`` launches.

Prints one JSON line per row, then the card's name and power limit read in the same run.

    python scripts/bench_robust_aim.py [--reps 10] [--max-seconds 60]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SAMPLES = ("ProjectionLens120FOV", "ProjectionLens160FOV", "WideAngle170FOV")
PUPILS = ((4, "hexapolar"), (64, "uniform"))


def _find_cached_aimers(lens):
    """Every CachedRayAimer reachable from the optic (the cache would turn repeated traces into look-ups)."""
    from optiland.rays.ray_aiming.cached import CachedRayAimer

    out, seen, todo = [], set(), [lens]
    while todo:
        o = todo.pop()
        if id(o) in seen or not hasattr(o, "__dict__"):
            continue
        seen.add(id(o))
        if isinstance(o, CachedRayAimer):
            out.append(o)
        for v in vars(o).values():
            if hasattr(v, "__dict__") and type(v).__module__.startswith("optiland"):
                todo.append(v)
    return out


def time_trace(P, lens, hx, hy, n, dist, device_aim, lib, torch):
    P._state["device_aim"] = device_aim
    for a in _find_cached_aimers(lens):
        a.clear_cache()
    torch.cuda.synchronize()
    l0 = lib.olb_launch_count()
    t0 = time.perf_counter()
    lens.trace(hx, hy, lens.primary_wavelength, n, dist)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, lib.olb_launch_count() - l0


def kernel_time(P, reps, torch):
    """torch.profiler duration of the aim kernel for one 10^6-ray solve."""
    import optiland.backend as be
    from optiland.samples.objectives import WideAngle170FOV

    from optiland.rays.ray_aiming.robust import RobustRayAimer

    lens = WideAngle170FOV()
    aimer = RobustRayAimer(lens)
    rng = np.random.default_rng(0)
    n = 1_000_000
    r = np.sqrt(rng.uniform(0, 1, n))
    a = rng.uniform(0, 2 * np.pi, n)
    t = 0.25
    Px, Py = be.array(r * np.cos(a) * t), be.array(r * np.sin(a) * t)
    H = (be.array(np.zeros(n)), be.array(np.full(n, 0.5 * t)))
    wl = lens.primary_wavelength
    guess = aimer._paraxial.aim_rays(H, wl, (Px, Py))
    backend = be.__getattr__.__globals__["_backends"]["torch"]     # the plugin's backend (install() registers it)
    solver = P._device_aim_solver(backend, aimer, guess, wl)
    assert solver is not None, "the device aimer declined the benchmark system"
    sol = solver.solve((Px, Py), guess)
    assert sol is not None, "the benchmark solve did not converge"
    for _ in range(3):
        solver.solve((Px, Py), guess)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            solver.solve((Px, Py), guess)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "aim_kernel" in e.name]
    return n, float(np.median(times)) * 1e-3 if times else float("nan"), len(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--max-seconds", type=float, default=60.0,
                    help="per row and path: stop repeating once this much time is spent (the row reports its count)")
    args = ap.parse_args()
    warnings.filterwarnings("ignore")
    import torch

    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be
    from optiland.samples import objectives

    from optiland_b200 import _lib
    from optiland_b200 import plugin as P

    assert torch.cuda.is_available(), "bench_robust_aim needs a CUDA device"
    be.set_backend("torch")
    be.set_device("cuda")
    be.set_precision("float64")
    be.grad_mode.disable()
    P.install()
    lib = _lib.load()
    for name in SAMPLES:
        for n, dist in PUPILS:
            lens = getattr(objectives, name)()
            for f in lens.fields.get_field_coords():
                hx, hy = float(f[0]), float(f[1])
                for dev in (True, False):                     # warm-up: modules, tables, allocator
                    time_trace(P, lens, hx, hy, n, dist, dev, lib, torch)
                res = {True: [], False: []}
                launches = {}
                spent = {True: 0.0, False: 0.0}
                for _ in range(args.reps):
                    for dev in (True, False):
                        if res[dev] and spent[dev] > args.max_seconds:
                            continue
                        dt, nl = time_trace(P, lens, hx, hy, n, dist, dev, lib, torch)
                        res[dev].append(dt)
                        spent[dev] += dt
                        launches[dev] = nl
                row = dict(system=name, field=[hx, hy], pupil=f"{n} {dist}",
                           device_aim_ms=1e3 * float(np.median(res[True])), device_aim_reps=len(res[True]),
                           device_aim_launches=launches[True],
                           reference_loop_ms=1e3 * float(np.median(res[False])), reference_loop_reps=len(res[False]),
                           reference_loop_launches=launches[False])
                row["speedup"] = row["reference_loop_ms"] / row["device_aim_ms"]
                print(json.dumps(row), flush=True)
    P._state["device_aim"] = True
    n, ms, count = kernel_time(P, args.reps, torch)
    print(json.dumps(dict(kernel="aim_kernel", rays=n, median_ms=ms, launches=count)), flush=True)
    P.uninstall()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)


if __name__ == "__main__":
    main()
