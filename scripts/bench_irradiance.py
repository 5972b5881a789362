"""Irradiance binning timing (olb_irradiance_*, optiland_b200/irradiance.py) on the GPU.

Workloads, each in fp32 and fp64 (rays on the detector plane, unrotated frame: x, y and power are read):
  uniform_10M_128     10^7 rays spread over a 128 x 128 grid (610 rays per bin: shared-memory path)
  uniform_1M_128      10^6 rays, same grid (61 per bin: global path); uniform_10k_128  10^4 rays, where launch and host
                      overhead show
  uniform_10M_32      10^7 rays over 32 x 32 (many rays per bin: where the shared path wins by most)
  focus_10M_21        10^7 rays into the four pixels around one vertex of a 21 x 21 grid (a perfect-focus mirror:
                      contention on four bins)
  uniform_10M_1024    10^7 rays over 1024 x 1024 (too large for shared memory: global path only)
For each: the kernel's device time (torch.profiler, median of 20 calls) on the path the library picks and on both paths
forced (OlbIrradiance.path), its share of 3.35 TB/s for the bytes the pass must read (n x 3 values), the time of one
``bin_irradiance`` call (CUDA events, median of 20), and a three-line device baseline (torch.searchsorted +
torch.bincount with fp64 weights).  With ``--reference``: the end-to-end ``IncoherentIrradiance(...)`` (10^6 and 10^7
user rays through a four-surface system, 128 x 128) with the plugin against the stock reference on the same GPU:
median, min and max of 10 runs after 2 warm-up runs (stock: 3 runs after 1).  Prints a markdown table and one JSON line; ``--out DIR`` also writes both there."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from optiland_b200 import _lib  # noqa: E402
from optiland_b200.irradiance import bin_irradiance  # noqa: E402

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def events_median(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def kernel_median_us(fn, reps=20, attempts=3):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    for _ in range(attempts):   # a profiling window occasionally comes back without its kernel records: take another
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        ts = [e.device_time for e in prof.events() if "irradiance_" in e.name and "kernel" in e.name]
        if ts:
            return statistics.median(ts)
    return float("nan")


def baseline(x, y, p, xe_t, ye_t, nx, ny):
    ix = torch.searchsorted(xe_t, x.double(), right=True).sub_(1).clamp_(max=nx - 1)
    iy = torch.searchsorted(ye_t, y.double(), right=True).sub_(1).clamp_(max=ny - 1)
    keep = (p > 0) & (x >= xe_t[0]) & (x <= xe_t[-1]) & (y >= ye_t[0]) & (y <= ye_t[-1])
    return torch.bincount((ix * ny + iy)[keep], weights=p[keep].double(), minlength=nx * ny).reshape(nx, ny)


WORKLOADS = [("uniform_10M_128", 10_000_000, 128, False), ("uniform_1M_128", 1_000_000, 128, False),
             ("uniform_10k_128", 10_000, 128, False), ("uniform_10M_32", 10_000_000, 32, False),
             ("focus_10M_21", 10_000_000, 21, True), ("uniform_10M_1024", 10_000_000, 1024, False)]
SHARED_MAX_BINS = 27 * 1024


def auto_path(nb, n):
    """The path OLB_IRR_PATH_AUTO takes (csrc/olb_irradiance.cu, irr_use_shared)."""
    return "shared" if nb <= SHARED_MAX_BINS and n >= 256 * nb else "global"


def kernel_rows():
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, n, npix, focus in WORKLOADS:
        for dtype in (torch.float32, torch.float64):
            xe = ye = np.linspace(-2.5, 2.5, npix + 1)
            span, c = (0.2, float(xe[npix // 2 + 1])) if focus else (5.0, 0.0)   # focus: around the vertex next to 0
            x = c + (torch.rand(n, generator=g, device="cuda", dtype=dtype) - 0.5) * span
            y = c + (torch.rand(n, generator=g, device="cuda", dtype=dtype) - 0.5) * span
            p = torch.rand(n, generator=g, device="cuda", dtype=dtype)
            out = torch.zeros((npix, npix), dtype=torch.float64, device="cuda")
            call = lambda: bin_irradiance(x, y, p, xe, ye, out=out)  # noqa: E731
            k_us = kernel_median_us(call)
            forced = {}
            for name_, path in (("shared", _lib.IRR_PATH_SHARED), ("global", _lib.IRR_PATH_GLOBAL)):
                if name_ == "global" or npix * npix <= SHARED_MAX_BINS:
                    forced[name_] = kernel_median_us(lambda: bin_irradiance(x, y, p, xe, ye, out=out, path=path))
            c_ms = events_median(call)
            xe_t, ye_t = (torch.tensor(e, device="cuda") for e in (xe, ye))
            b_ms = events_median(lambda: baseline(x, y, p, xe_t, ye_t, npix, npix))
            h = bin_irradiance(x, y, p, xe, ye)
            err = float((h - baseline(x, y, p, xe_t, ye_t, npix, npix)).abs().max() / h.abs().max())
            nbytes = n * 3 * x.element_size()
            rows.append(dict(workload=name, dtype=str(dtype).replace("torch.", ""), n=n, grid=npix,
                             path=auto_path(npix * npix, n), kernel_us=k_us, shared_us=forced.get("shared"),
                             global_us=forced["global"],
                             hbm_share=nbytes / HBM / (k_us * 1e-6), call_ms=c_ms, baseline_ms=b_ms,
                             max_rel_diff_vs_baseline=err))
            del x, y, p
    return rows


def e2e_rows():
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be
    from optiland.analysis import IncoherentIrradiance
    from optiland.optic import Optic
    from optiland.physical_apertures import RectangularAperture
    from optiland.rays import RealRays

    from optiland_b200 import plugin as P

    be.set_backend("torch")
    be.set_device("cuda")
    be.grad_mode.disable()
    rows = []
    for precision in ("float32", "float64"):
        be.set_precision(precision)
        op = Optic()
        op.surfaces.add(index=0, thickness=be.inf)
        op.surfaces.add(index=1, thickness=0, is_stop=True)
        op.surfaces.add(index=2, thickness=10)
        op.surfaces.add(index=3)
        op.surfaces[-1].aperture = RectangularAperture(x_min=-2.5, x_max=2.5, y_min=-2.5, y_max=2.5)
        op.wavelengths.add(0.55)
        op.fields.set_type("angle")
        op.fields.add(y=0)
        op.set_aperture("EPD", 5.0)
        dt = torch.float32 if precision == "float32" else torch.float64
        for n in (1_000_000, 10_000_000):
            g = torch.Generator(device="cuda").manual_seed(2)
            x = (torch.rand(n, generator=g, device="cuda", dtype=dt) - 0.5) * 5
            y = (torch.rand(n, generator=g, device="cuda", dtype=dt) - 0.5) * 5
            z0 = torch.zeros(n, device="cuda", dtype=dt)
            rays = RealRays(x, y, z0, z0, z0, z0 + 1, torch.rand(n, generator=g, device="cuda", dtype=dt), z0 + 0.55)

            def run():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                a = IncoherentIrradiance(op, res=(128, 128), user_initial_rays=rays)
                torch.cuda.synchronize()
                return time.perf_counter() - t0, a.data[0][0][0]

            res = {}
            for arm in ("plugin", "stock"):
                if arm == "plugin":
                    P.install()
                    P.stats(reset=True)
                elif P._state.get("installed"):
                    P.uninstall()
                warm, reps = (2, 10) if arm == "plugin" else (1, 3)
                for _ in range(warm):
                    run()
                ts, irr = [], None
                for _ in range(reps):
                    t, irr = run()
                    ts.append(t)
                res[arm] = (statistics.median(ts), be.to_numpy(irr).astype(np.float64), min(ts), max(ts))
                if arm == "plugin":
                    assert not P.stats(), P.stats()
            g_, w_ = res["plugin"][1], res["stock"][1]
            rows.append(dict(precision=precision, n=n, plugin_ms=res["plugin"][0] * 1e3, stock_ms=res["stock"][0] * 1e3,
                             plugin_min_ms=res["plugin"][2] * 1e3, plugin_max_ms=res["plugin"][3] * 1e3,
                             stock_min_ms=res["stock"][2] * 1e3, stock_max_ms=res["stock"][3] * 1e3,
                             speedup=res["stock"][0] / res["plugin"][0],
                             rel_l1_diff=float(np.abs(g_ - w_).sum() / np.abs(w_).sum())))
    if P._state.get("installed"):
        P.uninstall()
    be.set_precision("float64")
    be.set_device("cpu")
    be.set_backend("numpy")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", action="store_true", help="also time IncoherentIrradiance, plugin against stock")
    ap.add_argument("--out", default=None, help="directory for bench_irradiance.md / .json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_irradiance.py needs a CUDA device")
    gpu = card()
    rows = kernel_rows()
    lines = [f"GPU: {gpu}", "",
             "| workload | dtype | path | kernel (us) | shared forced (us) | global forced (us) | share of 3.35 TB/s "
             "| call (ms) | searchsorted+bincount (ms) |",
             "|---|---|---|---:|---:|---:|---:|---:|---:|"]
    for r in rows:
        sh = "-" if r["shared_us"] is None else f"{r['shared_us']:.1f}"
        lines.append(f"| {r['workload']} | {r['dtype']} | {r['path']} | {r['kernel_us']:.1f} | {sh} | {r['global_us']:.1f} "
                     f"| {100 * r['hbm_share']:.0f} % | {r['call_ms']:.3f} | {r['baseline_ms']:.3f} |")
    e2e = e2e_rows() if args.reference else []
    if e2e:
        lines += ["", "| IncoherentIrradiance, user rays, 128 x 128 | rays | plugin (ms) median [min, max] "
                  "| stock (ms) median [min, max] | speed-up |",
                  "|---|---:|---:|---:|---:|"]
        for r in e2e:
            lines.append(f"| {r['precision']} | {r['n']:.0e} | {r['plugin_ms']:.2f} [{r['plugin_min_ms']:.2f}, "
                         f"{r['plugin_max_ms']:.2f}] | {r['stock_ms']:.0f} [{r['stock_min_ms']:.0f}, {r['stock_max_ms']:.0f}] "
                         f"| {r['speedup']:.0f}x |")
    text = "\n".join(lines)
    print(text)
    result = dict(gpu=gpu, kernel=rows, e2e=e2e)
    print(json.dumps(result))
    if args.out:
        out = args.out
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "bench_irradiance.md"), "w") as f:
            f.write(text + "\n")
        with open(os.path.join(out, "bench_irradiance.json"), "w") as f:
            json.dump(result, f)


if __name__ == "__main__":
    main()
