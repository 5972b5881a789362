"""Secondary measurements (not the headline bench): the other BASELINE.json configurations at their
full sizes on one GPU -- forward fp32/fp64 with full records, polarized forward, and the
forward+backward step of the autograd configuration.  Prints one JSON line per configuration."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from optiland_b200 import autograd as AG  # noqa: E402
from optiland_b200.trace import DeviceTable, PolarizedRays, RealRays, trace_device  # noqa: E402
from tests._util import Case  # noqa: E402


def timeit(fn, k=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(k):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / k


def resample(c, n, dtype, cls=RealRays):
    dev = torch.device("cuda:0")
    idx = torch.randint(0, c.n, (n,), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    rr = {k: torch.from_numpy(v).to(dev)[idx] for k, v in c.rays.items()}
    return cls(rr["x"], rr["y"], rr["z"], rr["L"], rr["M"], rr["N"], rr["i"], rr["w"], dtype=dtype, device=dev)


def forward_case(name, n, label, cls=RealRays):
    c = Case(name)
    dtab = DeviceTable(c.table, "cuda:0")
    S = c.table.num_surfaces
    out = {"config": label, "system": name, "rays": n, "surfaces": S}
    for dtype, tag, es in ((torch.float32, "f32", 4), (torch.float64, "f64", 8)):
        base = resample(c, n, dtype, cls)

        def step():
            rr = cls.__new__(cls)
            rr.__dict__.update(base.__dict__)
            if cls is PolarizedRays:
                rr.p = None
            trace_device(dtab, rr, 0, S, record=True)

        ms = timeit(step)
        bytes_ = es * ((8 if c.table.n_wl == 1 else 9) + 8 * S) * n + (18 * es * n if cls is PolarizedRays else 0)
        out[tag] = {"ms": round(ms, 4), "ray_surfaces_per_s": round(n * (S - 1) / ms * 1e3, 0),
                    "algorithmic_GBps": round(bytes_ / ms / 1e6, 1)}
        del base
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


def autograd_case(n, name="telephoto_c3_tol1e-6",
                  label="C3 reverse telephoto + 2 even aspheres: forward + backward (d RMS spot / d all parameters)"):
    c = Case(name)
    S = c.table.num_surfaces
    out = {"config": label, "rays": n, "surfaces": S}
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        base = resample(c, n, dtype)
        params = AG.table_to_params(c.table).requires_grad_(True)
        coefs = AG.table_to_coefs(c.table)          # Zernike / polynomial coefficients (None without such surfaces)
        if coefs is not None:
            coefs = coefs.requires_grad_(True)

        def step():
            rr = RealRays.__new__(RealRays)
            rr.__dict__.update(base.__dict__)
            rec = AG.trace_differentiable(c.table, params, rr, rows=(-1,), coefs=coefs)
            x, y = rec["x"], rec["y"]
            m = torch.isfinite(x) & torch.isfinite(y)
            x, y = torch.where(m, x, 0), torch.where(m, y, 0)
            loss = torch.sqrt(torch.mean((x - x.mean()) ** 2 + (y - y.mean()) ** 2))
            params.grad = None
            if coefs is not None:
                coefs.grad = None
            loss.backward()

        ms = timeit(step, k=10)
        out[tag] = {"ms_fwd_bwd": round(ms, 3), "ray_surfaces_per_s": round(n * (S - 1) / ms * 1e3, 0)}
        del base
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


def c5_call_shape_case(n):
    """Config 5's CALL SHAPE: trace_generic-style per-ray (Hx, Hy, Px, Py, wavelength) arrays -> polarized fused launch
    (launch state generated in-kernel, P starts as the identity in shared memory) with (a) full records + P matrices +
    the update_intensity epilogue, (b) records only + intensity epilogue (P never written)."""
    import ctypes as C

    from optiland_b200 import _lib
    from optiland_b200.launch import pupil_affine_fields
    from optiland_b200.trace import _c_launch, _c_polarization, trace_pupil_device

    c = Case("generic_polarized_c5")
    sc = {k[9:]: float(c.z[k]) for k in c.z.files if k.startswith("x_launch_")}
    dtab = DeviceTable(c.table, "cuda:0")
    S = c.table.num_surfaces
    dev = torch.device("cuda:0")
    out = {"config": "C5 call shape: polarized fused launch, 5 fields x 3 wavelengths per-ray arrays", "rays": n, "surfaces": S}
    for dtype, tag, es in ((torch.float32, "f32", 4), (torch.float64, "f64", 8)):
        idx = torch.randint(0, c.n, (n,), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        a = {k: torch.from_numpy(np.ascontiguousarray(c.extra(k))).to(dev)[idx].to(dtype) for k in ("Px", "Py", "Hx", "Hy")}
        w = torch.from_numpy(c.rays["w"]).to(dev)[idx].to(dtype)
        aff = pupil_affine_fields(sc, a["Hx"], a["Hy"])
        ms_full = timeit(lambda: trace_pupil_device(dtab, a["Px"], a["Py"], aff, 0, S, wavelength=w, polarization=None))
        # (b) through the C ABI directly: records + intensity, rays.p = NULL
        vec = 4 if es == 4 else 2
        buf = torch.empty((8, S, n), dtype=dtype, device=dev)
        inten = torch.empty(n, dtype=dtype, device=dev)
        c_rec = _lib.OlbRecords(*[buf[j].data_ptr() for j in range(8)], n)
        la = _c_launch(aff, a["Px"], a["Py"])
        c_pol = _c_polarization(None, inten)
        rays = _lib.OlbRays(w=w.data_ptr())
        call = _lib.OlbTraceCall(first=0, last=S, n_rays=n, flags=_lib.TF_NO_FINAL | _lib.TF_POLARIZED,
                                 rays=C.pointer(rays), rec=C.pointer(c_rec), launch=C.pointer(la), pol=C.pointer(c_pol))
        fn = getattr(dtab.lib, "olb_trace_call_" + tag)
        stream = torch.cuda.current_stream().cuda_stream

        def lean():
            rc = fn(C.byref(dtab.c), C.byref(call), C.c_void_p(stream))
            assert rc == 0, _lib.last_error()

        ms_lean = timeit(lean)
        b_full = es * (5 + 8 * S + 18 + 1) * n
        b_lean = es * (5 + 8 * S + 1) * n
        out[tag] = {"ms_records_P_intensity": round(ms_full, 4), "GBps": round(b_full / ms_full / 1e6, 1),
                    "ms_records_intensity_only": round(ms_lean, 4), "GBps_lean": round(b_lean / ms_lean / 1e6, 1),
                    "ray_surfaces_per_s": round(n * (S - 1) / ms_lean * 1e3, 0)}
        del buf, inten, a, w
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


CASES = {
    "c2": lambda: forward_case("dgauss_c2", 10_000_000, "C2 Double-Gauss 10M rays (resampled fixture rays)"),
    "c3": lambda: forward_case("telephoto_c3_tol1e-6", 4_000_000, "C3 reverse telephoto + 2 even aspheres, 4M rays"),
    "c4": lambda: forward_case("hubble_c4", 16_000_000, "C4 Hubble (conic mirrors + obscuration), 16M rays"),
    "zern": lambda: forward_case("zernike_fringe", 4_000_000, "C5 geometry: Zernike freeform singlet, 4M rays"),
    "c5pol": lambda: forward_case("zernike_polarized_c5", 4_000_000,
                                  "C5: Zernike + Fresnel coatings + polarized, 3 wavelengths, 4M rays/GPU", PolarizedRays),
    "c5shape": lambda: c5_call_shape_case(4_000_000),
    "c3grad": lambda: autograd_case(4_000_000),
    "zerngrad": lambda: autograd_case(4_000_000, "zernike_fringe", "Zernike freeform singlet: forward + backward incl. d/d Zernike "
                                      "coefficients (olb_trace_bwd_* with grad_tables)"),
}

if __name__ == "__main__":
    only = sys.argv[1:] or list(CASES)
    for k in only:
        CASES[k]()
