"""Wavefront data (OPD map + exit-pupil intercepts) for one field of the Double-Gauss, 10 M pupil samples:
  fused      OlbTraceCall.wavefront_*: launch generation + trace + reference-sphere epilogue, 5 values/ray written
  unfused    OlbTraceCall.launch with full records (what Optic.trace does) + the reference's steps 4-5
             (wavefront/strategy.py:179-190) as eager torch ops on the device.
CUDA-event timed; both produce the same numbers (checked)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import load_case  # noqa: E402
from optiland_b200.launch import pupil_affine  # noqa: E402
from optiland_b200.trace import DeviceTable, trace_pupil_device, trace_wavefront_device  # noqa: E402


def eager_epilogue(r, Px, Py, ref):
    xc, yc, zc = ref["center"]
    R, n = ref["radius"], ref["n_image"]
    L, M, N = -r.L, -r.M, -r.N
    a = L**2 + M**2 + N**2
    b = 2 * (L * (r.x - xc) + M * (r.y - yc) + N * (r.z - zc))
    c = r.x**2 + r.y**2 + r.z**2 - 2 * (r.x * xc + r.y * yc + r.z * zc) + xc**2 + yc**2 + zc**2 - R**2
    d = b**2 - 4 * a * c
    d = torch.where(d < 0, torch.zeros_like(d), d)
    t1 = (-b - torch.sqrt(d)) / (2 * a)
    t2 = (-b + torch.sqrt(d)) / (2 * a)
    t = torch.where(t1 < 0, t2, t1)
    opd_img = n * t
    opd = r.opd - opd_img + (ref["tilt"][0] * Px + ref["tilt"][1] * Py)
    opd_wv = (ref["opd_ref"] - opd) / (ref["wavelength_um"] * 1e-3)
    tt = opd_img / n
    return opd_wv, r.x - tt * r.L, r.y - tt * r.M, r.z - tt * r.N


def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 10_000_000
    dev = torch.device("cuda:0")
    c, sc = load_case()
    S = c.table.num_surfaces
    aff = pupil_affine(sc)
    dtab = DeviceTable(c.table, dev)
    out = {"workload": f"double_gauss_13surf_{n}rays_wavefront_data"}
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        g = torch.Generator(device=dev).manual_seed(0)
        r = torch.rand(n, generator=g, device=dev, dtype=torch.float64).sqrt()
        th = 2 * np.pi * torch.rand(n, generator=g, device=dev, dtype=torch.float64)
        Px, Py = (r * torch.cos(th)).to(dtype), (r * torch.sin(th)).to(dtype)
        # reference sphere from the chief ray (Px = Py = 0), fp64
        z0 = torch.zeros(4, device=dev, dtype=torch.float64)
        chief, _ = trace_pupil_device(dtab, z0, z0, aff, 0, S)
        cx, cy, cz = (float(v[0]) for v in (chief.x, chief.y, chief.z))
        ref = {"center": (cx, cy, cz), "radius": 100.0, "n_image": 1.0, "tilt": (0.0, 0.0), "wavelength_um": 0.5876}
        o, *_ = eager_epilogue(chief, z0, z0, {**ref, "opd_ref": 0.0})
        ref["opd_ref"] = float(-o[0] * ref["wavelength_um"] * 1e-3)

        def timed(fn, reps=20):
            res = None
            for _ in range(4):
                res = None
                res = fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                res = None
                res = fn()
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / reps, res

        ms_f, fused = timed(lambda: trace_wavefront_device(dtab, Px, Py, aff, ref))

        def unfused():
            rays, _ = trace_pupil_device(dtab, Px, Py, aff, 0, S)
            return eager_epilogue(rays, Px, Py, ref)

        ms_u, un = timed(unfused, 10)
        d_opd = float((fused["opd"].double() - un[0].double()).abs().max())
        out[tag] = {"fused_ms": round(ms_f, 4), "unfused_ms": round(ms_u, 3), "speedup": ms_u / ms_f,
                    "fused_ray_surfaces_per_s": n * (S - 1) / ms_f * 1e3, "max_abs_dopd_waves_vs_unfused": d_opd}
        del fused, un
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
