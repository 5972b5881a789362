"""Time the device-resident trace step (one kernel launch), with and without records."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import WAVELENGTH, load_case  # noqa: E402
from optiland_b200.launch import launch_infinite_angle  # noqa: E402
from optiland_b200.trace import DeviceTable, RealRays, trace_device  # noqa: E402


def main():
    case = sys.argv[1] if len(sys.argv) > 1 else "dgauss_c2"
    n = int(float(sys.argv[2])) if len(sys.argv) > 2 else 10_000_000
    c, sc = load_case()
    if case != "dgauss_c2":
        from tests._util import Case
        c = Case(case)
    dev = torch.device("cuda:0")
    dtab = DeviceTable(c.table, dev)
    S = c.table.num_surfaces
    out = {"case": case, "n": n}
    for dtype, tag, es in ((torch.float32, "f32", 4), (torch.float64, "f64", 8)):
        if case == "dgauss_c2":
            g = torch.Generator(device=dev).manual_seed(0)
            r = torch.rand(n, generator=g, device=dev, dtype=torch.float64).sqrt()
            th = 2 * np.pi * torch.rand(n, generator=g, device=dev, dtype=torch.float64)
            x0, y0, z0, L, M, N = launch_infinite_angle(r * torch.cos(th), r * torch.sin(th), sc)
            base = RealRays(x0, y0, z0, L, M, N, 1.0, WAVELENGTH, dtype=dtype, device=dev)
        else:
            idx = torch.randint(0, c.n, (n,), device=dev)
            rr = {k: torch.from_numpy(v).to(dev)[idx] for k, v in c.rays.items()}
            base = RealRays(rr["x"], rr["y"], rr["z"], rr["L"], rr["M"], rr["N"], rr["i"], rr["w"], dtype=dtype, device=dev)

        def step(record=True):
            rr = RealRays.__new__(RealRays)
            rr.__dict__.update(base.__dict__)
            return trace_device(dtab, rr, 0, S, record=record)

        for record in (True, False):
            def one():
                if record:
                    return step(True)
                # the record-less trace updates the ray arrays in place: give it a private copy
                rr = RealRays.__new__(RealRays)
                rr.__dict__.update(base.__dict__)
                for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
                    setattr(rr, k, getattr(base, k).clone())
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                trace_device(dtab, rr, 0, S, record=False)
                e1.record()
                return e0, e1
            for _ in range(5):
                one()
            torch.cuda.synchronize()
            K = 30
            if record:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(K):
                    one()
                b.record()
                torch.cuda.synchronize()
                ms = a.elapsed_time(b) / K
            else:
                evs = [one() for _ in range(K)]
                torch.cuda.synchronize()
                ms = sum(a.elapsed_time(b) for a, b in evs) / K
            n_loads = 8 if c.table.n_wl == 1 else 9
            gb = es * (n_loads + 8 * S) * n / 1e9
            if record:
                out[tag] = {"ms": round(ms, 4), "GBps": round(gb / ms * 1e3, 1), "Grs_per_s": round(n * (S - 1) / ms / 1e6, 2)}
            else:
                out[tag]["ms_norecord"] = round(ms, 4)
        del base
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
