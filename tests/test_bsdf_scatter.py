"""BSDF scatter (Optiland's ``LambertianBSDF`` / ``GaussianBSDF``) in the trace kernel: the draws, the host
instantiation of the FEAT_BSDF kernel variant (tests/hostcheck/hostcheck_bsdf.cpp) against the reference's own scatter
driven by the same draws, the attempt bound, packing and what stays declined.  GPU tests (marked) compare the kernel
with the host instantiation draw for draw, and check the plugin's reproducibility and independence of calls."""
import numpy as np
import pytest

from oracle.ref_import import reference_available
from optiland_b200 import table as T
from tests import _bsdf_systems as BS

REC = ("x", "y", "z", "L", "M", "N", "intensity", "opd")
# fp32 host instantiation against the reference's fp64 records, worst ray per system in units of the system's scale, with
# the 160 launch rays and the seeds of test_host_instantiation_matches_reference_scatter; the test holds each system to
# 3x its value (rays past that are rejection tests flipped by rounding: a different draw, counted and bounded)
F32_ACHIEVED = {"doe_and_grating": 1.47e-06, "gaussian_lens": 1.58e-07, "grazing": 1.86e-05, "grid_diffuser": 1.61e-07,
                "lambertian_mirror": 3.27e-06, "plane_diffuser": 1.72e-07, "shared_instance": 9.83e-08,
                "sigma_zero": 1.61e-07, "two_bsdf_tilted": 1.23e-04}
# fp32 kernel against the fp32 host instantiation, worst ray per system in units of the scale, with the 4099 rays and the
# seeds of test_gpu_kernel_matches_host_instantiation ("host_path": test_gpu_host_path_chunking), measured on an NVIDIA
# H100 80GB HBM3 (700 W power limit); the GPU tests hold each to 3x
F32_ACHIEVED_GPU = {"doe_and_grating": 7.91e-06, "gaussian_lens": 2.54e-07, "grazing": 8.27e-05, "grid_diffuser": 2.24e-07,
                    "lambertian_mirror": 9.47e-06, "plane_diffuser": 2.12e-07, "shared_instance": 9.54e-08,
                    "sigma_zero": 1.91e-07, "two_bsdf_tilted": 2.25e-05, "host_path": 5.72e-08}
FEAT_BSDF = 1 << 10
needs_ref = pytest.mark.skipif(not reference_available(), reason="reference not staged (build())")


def _numpy_backend():
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    be.set_backend("numpy")
    return be


def _bsdf_of(surface):
    return getattr(surface.interaction_model, "bsdf", None)


def _packed(lens, seed=2024):
    """The host table of a reference system; each BSDF's seed is drawn on first use from torch's generator, seeded here
    so that every run draws the same numbers."""
    import torch

    from optiland_b200.pack import pack_surface_group

    torch.manual_seed(seed)
    return pack_surface_group(lens.surfaces, [0.55])


def _reference_records(lens, table, rays, stream, dtype=np.float64):
    """The reference's NumPy-backend trace of ``rays`` with its own ``scatter`` (the numba function's Python body), each
    ray's ``get_point`` returning that ray's successive draws from the host instantiation with the key ``table`` holds
    for that surface (the scatter calls come in surface order)."""
    import optiland.scatter as sc
    from optiland.rays import RealRays

    from oracle import hostcheck_bsdf as H

    src = [(s.bsdf_seed, s.bsdf, s.bsdf_sigma) for s in table.surfaces if s.bsdf != T.BSDF_NONE]
    calls = []

    def parallel(L, M, N, nx, ny, nz, get_point):
        seed, kind, sigma = src[len(calls)]
        calls.append(seed)
        out = np.empty((len(L), 3))
        for i in range(len(L)):
            state = {"next": 0, "buf": None}

            def point(i=i, state=state):
                a = state["next"]
                if state["buf"] is None or a - state["base"] >= len(state["buf"]):
                    state["buf"] = H.draws(seed, stream, i, 64, kind, sigma, dtype, attempt0=a)
                    state["base"] = a
                state["next"] = a + 1
                x, y = state["buf"][a - state["base"]]
                return float(x), float(y)

            out[i] = sc.scatter.py_func(L[i], M[i], N[i], nx[i], ny[i], nz[i], point)
        return out

    r = RealRays(*[rays[k].copy() for k in ("x", "y", "z", "L", "M", "N", "i", "w")])
    orig = sc.scatter_parallel
    sc.scatter_parallel = parallel
    try:
        with np.errstate(all="ignore"):
            lens.surfaces.trace(r)
    finally:
        sc.scatter_parallel = orig
    assert len(calls) == len(src)
    g = lens.surfaces
    return {k: np.array(getattr(g, k), dtype=np.float64) for k in REC}


def _scale(rec):
    v = np.abs(np.concatenate([rec[k][np.isfinite(rec[k])] for k in ("x", "y", "z")]))
    return max(1.0, float(v.max()))


def _assert_close(got, want, tol, allow_bad=0):
    """Every record equal within ``tol`` with the same NaN pattern, except at most ``allow_bad`` rays."""
    bad = np.zeros(got["x"].shape[1], dtype=bool)
    for k in REC:
        g, w = got[k], want[k]
        nan_g, nan_w = ~np.isfinite(g), ~np.isfinite(w)
        with np.errstate(invalid="ignore"):
            err = np.where(nan_g | nan_w, np.where(nan_g == nan_w, 0.0, np.inf), np.abs(g - w))
        bad |= np.any(err > tol, axis=0)
    assert bad.sum() <= allow_bad, (int(bad.sum()), allow_bad, tol)
    return int(bad.sum())


# ---- the draws -------------------------------------------------------------------------------------------------------

def test_philox_known_answer():
    """The host instantiation's Philox4x32-10 gives Random123's known answers."""
    from oracle import hostcheck_bsdf as H

    assert H.philox([0, 0, 0, 0], [0, 0]) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert H.philox([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_draws_same_in_both_precisions_and_distributed():
    from oracle import hostcheck_bsdf as H

    d64 = np.concatenate([H.draws(99, 3, ray, 50, T.BSDF_GAUSSIAN, 0.3) for ray in range(200)])
    d32 = np.concatenate([H.draws(99, 3, ray, 50, T.BSDF_GAUSSIAN, 0.3, dtype=np.float32) for ray in range(200)])
    assert np.all(np.isfinite(d64)) and np.max(np.abs(d32 - d64)) < 1e-5
    n = len(d64)
    assert abs(d64[:, 0].std() - 0.3) < 5 * 0.3 / np.sqrt(2 * n) and abs(d64[:, 1].mean()) < 5 * 0.3 / np.sqrt(n)
    lam = np.concatenate([H.draws(5, 0, ray, 50, T.BSDF_LAMBERTIAN, 0.0) for ray in range(200)])
    r2 = (lam ** 2).sum(axis=1)
    assert r2.max() <= 1.0 and abs(r2.mean() - 0.5) < 5 * np.sqrt(1 / 12 / len(r2))
    # a different stream, ray or seed draws other numbers
    base = H.draws(99, 3, 7, 4, T.BSDF_GAUSSIAN, 0.3)
    for args in ((99, 4, 7), (99, 3, 8), (100, 3, 7)):
        assert not np.any(H.draws(*args, 4, T.BSDF_GAUSSIAN, 0.3) == base)


# ---- kernel arithmetic against the reference's scatter -------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("name", sorted(BS.BUILDERS))
def test_host_instantiation_matches_reference_scatter(name):
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    be = _numpy_backend()
    lens = BS.BUILDERS[name](be)
    table = _packed(lens)
    assert any(s.bsdf for s in table.surfaces)
    rays = BS.launch_rays(160, 11 + len(name), grazing=name == "grazing")
    stream = 5
    want = _reference_records(lens, table, rays, stream)
    _, got, status = run_hostcheck_bsdf(table, rays, np.float64, stream=stream)
    assert status == 0
    scale = _scale(want)
    _assert_close(got, want, 1e-11 * scale)
    # fp32: the same draws (rounded); a ray whose rejection test flips by rounding takes another draw -- counted
    _, got32, _ = run_hostcheck_bsdf(table, rays, np.float32, stream=stream)
    flips = _assert_close({k: v.astype(np.float64) for k, v in got32.items()}, want, 3 * F32_ACHIEVED[name] * scale,
                          allow_bad=1)
    assert flips <= 1


@needs_ref
def test_nan_rays_and_the_other_arbitrary_vector():
    """NaN rays stay NaN after one draw; rays with L >= 0.999 use (0, 1, 0) (the grazing system covers them)."""
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    be = _numpy_backend()
    lens = BS.BUILDERS["grazing"](be)
    table = _packed(lens)
    rays = BS.launch_rays(64, 3, grazing=True)
    _, rec, _ = run_hostcheck_bsdf(table, rays, np.float64)
    assert np.all(np.isnan(rec["L"][-1, -3:])) and np.all(np.isfinite(rec["L"][1, :8]))


def test_attempt_bound_sets_status_and_nan():
    """An absurd sigma: rays that reject OLB_BSDF_MAX_ATTEMPTS draws leave with a NaN direction and the status bit."""
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, bsdf=T.BSDF_GAUSSIAN, bsdf_sigma=2000.0, bsdf_seed=17),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 5.0])], [0.55])
    rays = BS.launch_rays(24, 2)
    for dtype in (np.float64, np.float32):
        _, rec, status = run_hostcheck_bsdf(tab, rays, dtype)
        assert status & T.ST_BSDF_ATTEMPTS
        lost = np.isnan(rec["L"][1])
        assert lost.sum() > 12        # acceptance ~ 1 / (2 sigma^2) per draw: most rays exhaust the bound
    ok = T.SurfaceTable([tab.surfaces[0], T.SurfaceSpec(kind=T.GEOM_PLANE, bsdf=T.BSDF_GAUSSIAN, bsdf_sigma=0.5,
                                                        bsdf_seed=17)], [0.55])
    assert run_hostcheck_bsdf(ok, rays, np.float64)[2] == 0


def test_draws_key_on_global_ray_index():
    """A ray's draws depend on its index, not on where a chunk starts: two halves with ray0 equal one call."""
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, bsdf=T.BSDF_LAMBERTIAN, bsdf_seed=(1 << 63) + 5),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 5.0])], [0.55])
    rays = BS.launch_rays(40, 4)
    _, whole, _ = run_hostcheck_bsdf(tab, rays, np.float64, stream=9)
    a = {k: v[:17] for k, v in rays.items()}
    b = {k: v[17:] for k, v in rays.items()}
    _, ra, _ = run_hostcheck_bsdf(tab, a, np.float64, stream=9)
    _, rb, _ = run_hostcheck_bsdf(tab, b, np.float64, ray0=17, stream=9)
    for k in REC:
        np.testing.assert_array_equal(np.concatenate([ra[k], rb[k]], axis=1), whole[k])


# ---- host side ------------------------------------------------------------------------------------------------------

def test_table_pack_roundtrip_and_validation():
    s = T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=-30.0, bsdf=T.BSDF_GAUSSIAN, bsdf_sigma=0.25,
                      bsdf_seed=(123 << 32) + 456, coating=T.COAT_SIMPLE, coat_t=0.9)
    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP), s], [0.55])
    assert tab.surfaces[1].flags & T.SF_BSDF
    surf, pool = tab.pack()
    back = T.SurfaceTable.unpack(surf, pool, tab.wavelengths).surfaces[1]
    assert (back.bsdf, back.bsdf_sigma, back.bsdf_seed) == (T.BSDF_GAUSSIAN, 0.25, (123 << 32) + 456)
    m0 = int(surf[1]["media_off"])
    np.testing.assert_array_equal(pool[m0 + 5: m0 + 9], [T.BSDF_GAUSSIAN, 0.25, 456.0, 123.0])
    for bad in (dict(bsdf_sigma=float("inf")), dict(bsdf=7)):
        with pytest.raises(ValueError):
            T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP), T.SurfaceSpec(kind=T.GEOM_PLANE, **dict(dict(bsdf=1), **bad))],
                           [0.55])


def test_upload_preparation_rejects_bad_blocks():
    """The host preparation (the code olb_table_upload runs) refuses a non-finite sigma and non-integer seeds."""
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, bsdf=T.BSDF_GAUSSIAN, bsdf_sigma=0.1)], [0.55])
    surf, pool = tab.pack()
    m0 = int(surf[1]["media_off"])
    rays = BS.launch_rays(4, 1)
    for off, val, msg in ((1, np.nan, "sigma"), (2, 0.5, "seed"), (0, 3.0, "kind")):
        p = pool.copy()
        p[m0 + 5 + off] = val
        bad = T.SurfaceTable(list(tab.surfaces), tab.wavelengths)
        bad.pack = lambda p=p: (surf, p)      # (the Python-side validation would refuse these values first)
        with pytest.raises(AssertionError, match=msg):
            run_hostcheck_bsdf(bad, rays, np.float64)


@needs_ref
def test_pack_accepts_the_two_classes_only():
    from optiland.scatter import GaussianBSDF

    from optiland_b200.pack import UnsupportedSurface, pack_bsdf

    be = _numpy_backend()
    lens = BS.gaussian_lens(be, 0.2)
    b = _bsdf_of(lens.surfaces.surfaces[2])
    kind, sigma, seed = pack_bsdf(b)
    assert (kind, sigma) == (T.BSDF_GAUSSIAN, 0.2) and pack_bsdf(b)[2] == seed    # the seed stays with the object

    class Mine(GaussianBSDF):
        pass

    for obj in (Mine(0.1), object()):
        with pytest.raises(UnsupportedSurface, match="bsdf"):
            pack_bsdf(obj)


def test_batched_tables_decline():
    from optiland_b200 import batch

    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP), T.SurfaceSpec(kind=T.GEOM_PLANE, bsdf=T.BSDF_LAMBERTIAN)],
                         [0.55])
    with pytest.raises(ValueError, match="BSDF"):
        batch.template_params(tab)


# ---- GPU --------------------------------------------------------------------------------------------------------------

def _device_trace(table, rays, dtype, stream):
    import torch

    from optiland_b200.trace import DeviceTable, RealRays, trace_device

    dt = DeviceTable(table, "cuda:0")
    r = RealRays(*[rays[k] for k in ("x", "y", "z", "L", "M", "N", "i", "w")], dtype=dtype, device="cuda:0")
    rec = trace_device(dt, r, 0, table.num_surfaces, record=True, rng_stream=stream)
    torch.cuda.synchronize()
    return dt, {k: rec[k].double().cpu().numpy() for k in REC}


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("name", sorted(BS.BUILDERS))
def test_gpu_kernel_matches_host_instantiation(name):
    import torch

    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    be = _numpy_backend()
    table = _packed(BS.BUILDERS[name](be))
    rays = BS.launch_rays(4099, 31, grazing=name == "grazing")
    _, want, _ = run_hostcheck_bsdf(table, rays, np.float64, stream=77)
    scale = _scale(want)
    dt, got = _device_trace(table, rays, torch.float64, 77)
    assert dt.features & FEAT_BSDF
    # (a scattered ray that leaves nearly parallel to a later surface amplifies the last-ulp differences of the device's
    # and the host's sin / cos / sqrt by 1 / N^2 there: a few rays per thousand may exceed the tolerance)
    _assert_close(got, want, 1e-12 * scale, allow_bad=4)
    _, got32 = _device_trace(table, rays, torch.float32, 77)
    _, want32, _ = run_hostcheck_bsdf(table, rays, np.float32, stream=77)
    _assert_f32_with_flips(got32, {k: v.astype(np.float64) for k, v in want32.items()}, name, scale)


def _assert_f32_with_flips(got, want, name, scale):
    """fp32 kernel against the fp32 host instantiation: every ray within 3x the system's achieved fp32 error, except
    rays whose rejection test flipped by rounding -- they took another draw, so they differ grossly (more than 1e-3 x
    scale) -- and at most one in a thousand of those."""
    tol = 3 * F32_ACHIEVED_GPU[name] * scale
    n = got["x"].shape[1]
    err = np.zeros(n)
    for k in REC:
        g, w = got[k], want[k]
        nan_g, nan_w = ~np.isfinite(g), ~np.isfinite(w)
        with np.errstate(invalid="ignore"):
            e = np.where(nan_g | nan_w, np.where(nan_g == nan_w, 0.0, np.inf), np.abs(g - w))
        err = np.maximum(err, e.max(axis=0))
    bad = err > tol
    flips = err > 1e-3 * scale
    print(f"{name}: fp32 worst non-flipped {np.max(err[~flips]) / scale:.3e} x scale, {int(flips.sum())} flips of {n}")
    assert not np.any(bad & ~flips), (name, np.sort(err[bad & ~flips])[-5:] / scale, tol / scale)
    assert flips.sum() <= n // 1000, int(flips.sum())


@pytest.mark.gpu
def test_gpu_same_stream_repeats_other_stream_differs():
    import torch

    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, bsdf=T.BSDF_GAUSSIAN, bsdf_sigma=0.2, bsdf_seed=3),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 5.0])], [0.55])
    rays = BS.launch_rays(10000, 8)
    _, a = _device_trace(tab, rays, torch.float64, 1)
    _, b = _device_trace(tab, rays, torch.float64, 1)
    _, c = _device_trace(tab, rays, torch.float64, 2)
    np.testing.assert_array_equal(a["L"], b["L"])
    fin = np.isfinite(a["L"][-1])
    assert np.mean(a["L"][-1][fin] != c["L"][-1][fin]) > 0.99


@pytest.mark.gpu
def test_gpu_features_of_tables_without_bsdf_unchanged():
    from optiland_b200.trace import DeviceTable

    base = [T.SurfaceSpec(kind=T.GEOM_NOOP), T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=40.0, n2=[1.5]),
            T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 5.0], n1=[1.5])]
    plain = DeviceTable(T.SurfaceTable(base, [0.55]), "cuda:0")
    assert plain.features == 0
    import dataclasses

    with_b = list(base)
    with_b[1] = dataclasses.replace(base[1], bsdf=T.BSDF_LAMBERTIAN, bsdf_seed=1)
    assert DeviceTable(T.SurfaceTable(with_b, [0.55]), "cuda:0").features == FEAT_BSDF


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_gpu_host_path_chunking(dtype_name):
    import torch

    from oracle.hostcheck_bsdf import run_hostcheck_bsdf
    from optiland_b200.trace import DeviceTable, trace_host

    dtype = getattr(torch, dtype_name)
    npd = np.float64 if dtype == torch.float64 else np.float32
    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP),
                          T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=-40.0, bsdf=T.BSDF_GAUSSIAN, bsdf_sigma=0.1,
                                        bsdf_seed=11),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 20.0])], [0.55])
    n = 50001
    rays = BS.launch_rays(n, 6)
    dt = DeviceTable(tab, "cuda:0")
    h_in = {k: torch.from_numpy(rays[k].astype(npd)).pin_memory() for k in ("x", "y", "z", "L", "M", "N", "i", "w")}
    outs = []
    for chunk in (n, 8192):
        h_out = {k: torch.empty(n, dtype=dtype).pin_memory() for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
        trace_host(dt, h_in, h_out, n, dtype=dtype, chunk=chunk)
        outs.append({k: v.numpy().astype(np.float64) for k, v in h_out.items()})
    for k in outs[0]:
        np.testing.assert_array_equal(outs[0][k], outs[1][k])
    # the host path draws stream 0 with the rays' indices in the whole host array
    fin, _, _ = run_hostcheck_bsdf(tab, rays, npd, stream=0)
    rec = {k: fin[k][None, :].astype(np.float64) for k in ("x", "y", "z", "L", "M", "N")}
    rec.update(intensity=fin["i"][None, :].astype(np.float64), opd=fin["opd"][None, :].astype(np.float64))
    got = {k: outs[0][k][None, :] for k in ("x", "y", "z", "L", "M", "N", "opd")}
    got["intensity"] = outs[0]["i"][None, :]
    if dtype == torch.float64:
        _assert_close(got, rec, 1e-12 * 100.0, allow_bad=n // 1000)
    else:
        _assert_f32_with_flips(got, rec, "host_path", 100.0)


@pytest.mark.gpu
@needs_ref
def test_gpu_plugin_optic_trace_reproducible_and_independent():
    """Unmodified Optic.trace through the plugin: torch.manual_seed before the optic is built repeats the rays bit for
    bit; two successive traces draw independently; nothing declines."""
    import torch

    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin

    be.set_backend("torch")
    be.set_device("cuda")
    be.set_precision("float64")
    be.grad_mode.disable()
    plugin.install()
    plugin.stats(reset=True)
    try:
        def run(seed):
            torch.manual_seed(seed)
            lens = BS.plane_diffuser(be)
            lens.trace(Hx=0.0, Hy=0.0, wavelength=0.55, num_rays=64, distribution="hexapolar")
            first = be.to_numpy(lens.surfaces.L).copy()
            lens.trace(Hx=0.0, Hy=0.0, wavelength=0.55, num_rays=64, distribution="hexapolar")
            return first, be.to_numpy(lens.surfaces.L).copy()

        a1, a2 = run(4)
        b1, b2 = run(4)
        np.testing.assert_array_equal(a1, b1)
        np.testing.assert_array_equal(a2, b2)
        assert np.mean(a1[-1] != a2[-1]) > 0.99
        assert np.all(np.isfinite(a1[-1])) and not plugin.stats(), plugin.stats()
    finally:
        plugin.uninstall()
        be.set_device("cpu")
        be.set_backend("numpy")


# ---- one BSDF object on several surfaces -------------------------------------------------------------------------------

@needs_ref
def test_one_instance_on_two_surfaces_draws_independently():
    """The Philox key depends on the surface's position: a shared GaussianBSDF draws other numbers at each surface (the
    reference's sequential generator does too), so two diffusers in series spread by sqrt(2) sigma, not 2 sigma."""
    from oracle import hostcheck_bsdf as H
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    be = _numpy_backend()
    table = _packed(BS.shared_instance(be, sigma=0.05))
    k1, k2 = (s.bsdf_seed for s in table.surfaces if s.bsdf)
    assert k1 != k2
    assert not np.any(H.draws(k1, 0, 3, 8, T.BSDF_GAUSSIAN, 0.05) == H.draws(k2, 0, 3, 8, T.BSDF_GAUSSIAN, 0.05))
    n = 20000
    rays = dict(x=np.zeros(n), y=np.zeros(n), z=np.full(n, -5.0), L=np.zeros(n), M=np.zeros(n), N=np.ones(n),
                i=np.ones(n), w=np.full(n, 0.55))
    _, rec, _ = run_hostcheck_bsdf(table, rays, np.float64)
    # on-axis rays on a plane: a = (0, 1, 0), b = (-1, 0, 0), so the direction's (M, -L) is the sum of the two draws
    spread = np.std(rec["M"][2])
    assert abs(spread - np.sqrt(2) * 0.05) < 5 * np.sqrt(2) * 0.05 / np.sqrt(2 * n), spread


# ---- the distribution against the reference's own generator ------------------------------------------------------------

def _local_frame(n, L):
    """(a, b) of the reference's scatter for normal ``n`` and a ray with x-cosine ``L``."""
    arb = np.array([1.0, 0.0, 0.0]) if L < 0.999 else np.array([0.0, 1.0, 0.0])
    a = np.cross(n, arb)
    a /= np.linalg.norm(a)
    return a, np.cross(n, a)


@needs_ref
@pytest.mark.parametrize("kind,sigma", [(T.BSDF_LAMBERTIAN, 0.0), (T.BSDF_GAUSSIAN, 0.1), (T.BSDF_GAUSSIAN, 0.5)])
def test_distribution_matches_the_reference_generator(kind, sigma):
    """10^6 rays through a flat diffuser: the local-frame (sx, sy) of the kernel's draws (host instantiation) against
    the reference's NumPy backend with its numba generator, seeded.  The rays come in at 0.3 rad, so the rejection
    loop matters.  Means and second moments agree within 5 standard errors; a two-sample chi-square on a 2-D histogram
    passes at p > 1e-6.  (The reference's parallel scatter loop is compiled without threads here, so one seeded stream
    serves every ray and the test is deterministic.)"""
    import numba
    import optiland.scatter as sc
    from optiland.rays import RealRays
    from scipy import stats

    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    be = _numpy_backend()
    from optiland.scatter import LambertianBSDF

    lens = BS.gaussian_sigma(be, sigma)
    if kind == T.BSDF_LAMBERTIAN:
        lens.surfaces.surfaces[1].interaction_model.bsdf = LambertianBSDF()
    table = _packed(lens)
    n = 1_000_000
    rng = np.random.default_rng(3)
    L0, M0 = np.sin(0.3), 0.0
    rays = dict(x=rng.uniform(-2, 2, n), y=rng.uniform(-2, 2, n), z=np.full(n, -5.0), L=np.full(n, L0),
                M=np.full(n, M0), N=np.full(n, np.cos(0.3)), i=np.ones(n), w=np.full(n, 0.55))
    _, ours, _ = run_hostcheck_bsdf(table, rays, np.float64, stream=1)

    @numba.njit
    def seed(s):
        np.random.seed(s)

    serial = numba.njit(sc.scatter_parallel.py_func)
    seed(12345)
    r = RealRays(*[rays[k].copy() for k in ("x", "y", "z", "L", "M", "N", "i", "w")])
    orig = sc.scatter_parallel
    sc.scatter_parallel = serial
    try:
        lens.surfaces.trace(r)
    finally:
        sc.scatter_parallel = orig
    a, b = _local_frame(np.array([0.0, 0.0, 1.0]), L0)
    samples = []
    for d in ({k: ours[k][1] for k in "LMN"}, {k: np.asarray(getattr(lens.surfaces, k))[1] for k in "LMN"}):
        s = np.stack([d["L"], d["M"], d["N"]], axis=1)
        samples.append((s @ a, s @ b))
    (x1, y1), (x2, y2) = samples
    for f1, f2 in ((x1, x2), (y1, y2), (x1 * x1, x2 * x2), (y1 * y1, y2 * y2), (x1 * y1, x2 * y2)):
        se = np.sqrt(f1.var() / n + f2.var() / n)
        assert abs(f1.mean() - f2.mean()) <= 5 * se, (f1.mean(), f2.mean(), se)
    lo = min(x1.min(), x2.min(), y1.min(), y2.min())
    hi = max(x1.max(), x2.max(), y1.max(), y2.max())
    edges = np.linspace(lo, hi, 25)
    h1 = np.histogram2d(x1, y1, bins=[edges, edges])[0].ravel()
    h2 = np.histogram2d(x2, y2, bins=[edges, edges])[0].ravel()
    keep = (h1 + h2) > 0
    chi2 = np.sum((h1[keep] - h2[keep]) ** 2 / (h1[keep] + h2[keep]))
    p = stats.chi2.sf(chi2, int(keep.sum()) - 1)
    assert p > 1e-6, (chi2, int(keep.sum()), p)


# ---- GPU: the plugin's call shapes against the host instantiation -------------------------------------------------------

STREAM = 4242


@pytest.fixture
def live(monkeypatch):
    """The reference on the torch backend on cuda:0 in fp64 with the plugin installed; every BSDF trace draws stream
    STREAM, so the host instantiation can replay it."""
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin
    from optiland_b200 import trace as TR

    monkeypatch.setattr(TR, "next_rng_stream", lambda: STREAM)
    be.set_backend("torch")
    be.set_device("cuda")
    be.set_precision("float64")
    be.grad_mode.disable()
    plugin.install()
    plugin.stats(reset=True)
    try:
        yield be, plugin
    finally:
        be.grad_mode.disable()
        plugin.uninstall()
        be.set_device("cpu")
        be.set_backend("numpy")


def _np(be, t):
    return np.asarray(be.to_numpy(t), dtype=np.float64)


def _group_records(be, lens):
    return {k: _np(be, getattr(lens.surfaces, k)) for k in REC}


def _replay(table, rec0, first_row=0):
    """Host instantiation over the whole table from the launch state in record row 0 (the object surface's row)."""
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    n = rec0["x"].shape[-1]
    rays = {k: rec0[k][first_row].copy() for k in ("x", "y", "z", "L", "M", "N")}
    rays.update(i=rec0["intensity"][first_row].copy(), w=np.full(n, 0.55), opd=np.zeros(n))
    return run_hostcheck_bsdf(table, rays, np.float64, stream=STREAM)


def _table_of(lens):
    from optiland_b200.pack import pack_surface_group

    return pack_surface_group(lens.surfaces, [0.55])     # (the seeds are already on the BSDF objects)


@pytest.mark.gpu
@needs_ref
def test_gpu_plugin_surface_group_and_surface_trace(live):
    """SurfaceGroup.trace and a single Surface.trace (the aimers' call shape) through the plugin."""
    from optiland.rays import RealRays

    from oracle.hostcheck_bsdf import run_hostcheck_bsdf
    from optiland_b200.pack import pack_surface

    be, plugin = live
    lens = BS.two_bsdf_tilted(be)
    rays = BS.launch_rays(3001, 5)
    r = RealRays(*[be.array(rays[k]) for k in ("x", "y", "z", "L", "M", "N", "i", "w")])
    lens.surfaces.trace(r)
    assert not plugin.stats(), plugin.stats()
    got = _group_records(be, lens)
    _, want, _ = run_hostcheck_bsdf(_table_of(lens), rays, np.float64, stream=STREAM)
    _assert_close(got, want, 1e-12 * _scale(want), allow_bad=3)
    # one surface, as the aimers call it: global rays in front of the Lambertian plane
    surf = lens.surfaces.surfaces[3]
    r1 = RealRays(*[be.array(rays[k]) for k in ("x", "y", "z", "L", "M", "N", "i", "w")])
    surf.trace(r1)
    assert not plugin.stats(), plugin.stats()
    one = T.SurfaceTable([pack_surface(surf, [0.55])], [0.55])
    fin, _, _ = run_hostcheck_bsdf(one, rays, np.float64, stream=STREAM)
    for k in ("L", "M", "N"):
        np.testing.assert_allclose(_np(be, getattr(r1, k)), fin[k], rtol=0, atol=1e-12)


@pytest.mark.gpu
@needs_ref
def test_gpu_plugin_fused_optic_trace_and_trace_generic(live):
    be, plugin = live
    lens = BS.plane_diffuser(be)
    lens.trace(Hx=0.0, Hy=0.0, wavelength=0.55, num_rays=40, distribution="hexapolar")
    got = _group_records(be, lens)
    _, want, _ = _replay(_table_of(lens), got)
    _assert_close(got, want, 1e-12 * _scale(want), allow_bad=2)
    n = 5000
    rng = np.random.default_rng(2)
    Px, Py = (be.array(rng.uniform(-0.7, 0.7, n)) for _ in range(2))
    lens.trace_generic(Hx=be.zeros(n), Hy=be.zeros(n), Px=Px, Py=Py, wavelength=0.55)
    got = _group_records(be, lens)
    _, want, _ = _replay(_table_of(lens), got)
    _assert_close(got, want, 1e-12 * _scale(want), allow_bad=5)
    assert not plugin.stats(), plugin.stats()


@pytest.mark.gpu
@needs_ref
def test_gpu_spot_moments_of_a_bsdf_table(monkeypatch):
    """The fused spot-moment epilogue (no per-ray output) on a BSDF table against the host instantiation's last row."""
    import torch

    from oracle.hostcheck_bsdf import run_hostcheck_bsdf
    from optiland_b200 import trace as TR
    from optiland_b200.trace import DeviceTable, RealRays, trace_moments_device

    monkeypatch.setattr(TR, "next_rng_stream", lambda: STREAM)
    be = _numpy_backend()
    table = _packed(BS.plane_diffuser(be))
    rays = BS.launch_rays(20000, 9)
    _, rec, _ = run_hostcheck_bsdf(table, rays, np.float64, stream=STREAM)
    dt = DeviceTable(table, "cuda:0")
    r = RealRays(*[rays[k] for k in ("x", "y", "z", "L", "M", "N", "i", "w")], dtype=torch.float64, device="cuda:0")
    m = trace_moments_device(dt, 20000, torch.float64, rays=r).cpu().numpy()
    x, y, i = rec["x"][-1] - table.surfaces[-1].t[0], rec["y"][-1] - table.surfaces[-1].t[1], rec["intensity"][-1]
    keep = (i > 0) & np.isfinite(x) & np.isfinite(y)
    assert m[0] == keep.sum()
    np.testing.assert_allclose(m[1:4], [x[keep].sum(), y[keep].sum(), (x[keep] ** 2 + y[keep] ** 2).sum()],
                               rtol=1e-9, atol=1e-9)


@pytest.mark.gpu
@needs_ref
def test_gpu_wavefront_epilogue_of_a_bsdf_table(monkeypatch):
    """The fused wavefront epilogue on a BSDF table: its per-ray OPD against the host instantiation's final state put
    through the epilogue's host arithmetic (hostcheck.cpp wavefront_point)."""
    import torch

    from oracle import hostcheck_api
    from oracle.hostcheck_bsdf import run_hostcheck_bsdf
    from optiland_b200 import trace as TR
    from optiland_b200.launch import launch_from_affine
    from optiland_b200.trace import DeviceTable, trace_wavefront_device

    monkeypatch.setattr(TR, "next_rng_stream", lambda: STREAM)
    be = _numpy_backend()
    table = _packed(BS.plane_diffuser(be, sigma=0.02))
    dt = DeviceTable(table, "cuda:0")
    n = 4096
    rng = np.random.default_rng(4)
    Px, Py = rng.uniform(-0.7, 0.7, n), rng.uniform(-0.7, 0.7, n)
    aff = {"origin0": [0.0, 0.0, -5.0], "origin_scale": [5.0, 5.0], "target0": [0.0, 0.0, 0.0],
           "target_scale": [5.0, 5.0], "intensity": 1.0}
    ref = {"center": [0.0, 0.0, 54.0], "radius": 60.0, "n_image": 1.0, "opd_ref": 0.0, "wavelength_um": 0.55}
    tx, ty = (torch.from_numpy(v).cuda() for v in (Px, Py))
    out = trace_wavefront_device(dt, tx, ty, aff, ref)
    x, y, z, L, M, N = (np.broadcast_to(np.asarray(v, dtype=np.float64), (n,)).copy()
                        for v in launch_from_affine(Px, Py, aff))
    rays = dict(x=x, y=y, z=z, L=L, M=M, N=N, i=np.ones(n), w=np.full(n, 0.55))
    fin, _, _ = run_hostcheck_bsdf(table, rays, np.float64, stream=STREAM)
    want = hostcheck_api.run_wavefront(hostcheck_api.load(), fin, Px, Py, ref)
    got = out["opd"].double().cpu().numpy()
    ok = np.isfinite(want["opd"])
    assert np.array_equal(ok, np.isfinite(got))
    assert np.mean(np.abs(got[ok] - want["opd"][ok]) <= 1e-5) > 0.999


@pytest.mark.gpu
@needs_ref
def test_gpu_irradiance_of_a_diffuser_with_user_rays(live):
    """IncoherentIrradiance with user rays through a diffuser: the plugin's map against np.histogram2d of the host
    instantiation's image-plane intercepts (rays within rounding of a bin edge may land in the neighbour bin)."""
    from optiland.analysis import IncoherentIrradiance
    from optiland.physical_apertures import RectangularAperture
    from optiland.rays import RealRays

    from oracle.hostcheck_bsdf import run_hostcheck_bsdf

    be, plugin = live
    lens = BS.plane_diffuser(be, sigma=0.1)
    lens.surfaces.surfaces[-1].aperture = RectangularAperture(-8.0, 8.0, -8.0, 8.0)     # the detector's size
    n = 200_000
    rays = BS.launch_rays(n, 12)
    for k in ("x", "L"):
        rays[k][-3:] = 0.0
    r = RealRays(*[be.array(rays[k]) for k in ("x", "y", "z", "L", "M", "N", "i", "w")])
    a = IncoherentIrradiance(lens, res=(40, 40), user_initial_rays=r)
    got, xe, ye = a.data[0][0]
    got, xe, ye = _np(be, got), np.asarray(xe, dtype=np.float64), np.asarray(ye, dtype=np.float64)
    assert not plugin.stats(), plugin.stats()
    _, rec, _ = run_hostcheck_bsdf(_table_of(lens), rays, np.float64, stream=STREAM)
    t = _table_of(lens).surfaces[-1].t
    x, y, i = rec["x"][-1] - t[0], rec["y"][-1] - t[1], rec["intensity"][-1]
    keep = i > 0
    want = np.histogram2d(x[keep], y[keep], bins=[xe, ye], weights=i[keep])[0]
    assert got.shape == want.shape
    got = got * ((xe[1] - xe[0]) * (ye[1] - ye[0]))        # the map is power per pixel area
    assert np.isclose(got.sum(), want.sum(), rtol=1e-12) or abs(got.sum() - want.sum()) <= 4
    assert np.abs(got - want).sum() <= 8, np.abs(got - want).sum()


@pytest.mark.gpu
@needs_ref
def test_gpu_plugin_declines_polarized_rays_and_gradients(live):
    """A BSDF with polarized rays, and with gradients wanted, goes back to the reference's path (which then cannot run
    its numba scatter on torch tensors), each with its reason."""
    from optiland.rays import PolarizedRays, RealRays

    be, plugin = live
    lens = BS.plane_diffuser(be)
    rays = BS.launch_rays(64, 1)
    pr = PolarizedRays(*[be.array(rays[k]) for k in ("x", "y", "z", "L", "M", "N", "i", "w")])
    with pytest.raises(Exception):
        lens.surfaces.trace(pr)
    assert "BSDF scatter with polarized rays" in plugin.stats(reset=True)
    be.grad_mode.enable()
    r = RealRays(*[be.array(rays[k]) for k in ("x", "y", "z", "L", "M", "N", "i", "w")])
    with pytest.raises(Exception):
        lens.surfaces.trace(r)
    assert "gradients wanted: BSDF scatter" in plugin.stats(reset=True)
