"""The ray-aiming kernel (``olb_aim_f32`` / ``olb_aim_f64``: ``aim_kernel`` in csrc/olb_trace.cu, the per-ray solve in
csrc/olb_aim.cuh) on the GPU at full batch sizes, ray by ray against its host instantiation
(tests/hostcheck/hostcheck_aim.cpp through ``oracle/hostcheck_aim.py``).

Every kernel variant (closed form, general, superset) runs in both precisions at 1, 31 and 257 rays (two CTAs) and at
one resident wave of 256-thread CTAs plus 7 rays, which exceeds the grid ``launch_aim`` caps at any occupancy, so every
variant runs its grid-stride loop.  Pupil points and fields are drawn per ray from a seeded generator; the guesses are
the reference's paraxial aimer's.  fp64 solves match the fp64 host solve ray by ray; fp32 solves are held against the
fp32 host solve and re-traced in fp64.  Then planted failures, per-ray independence of the batch, the C ABI's argument
checks, and live robust traces through ``CudaEngine``.  The largest differences and residual ratios are recorded as
test properties (``--junitxml``)."""
import ctypes as C

import numpy as np
import pytest

from oracle.ref_import import reference_available
from tests.test_robust_aiming import (KEYS, ROBUST, _aim_inputs, _check_record_arrays, _doe_before_stop, _finite_object,
                                      _host_solve, _numpy_records, _sample, _scale, _tilted_stop, _zernike_stop,
                                      torch_backend)  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not reference_available(), reason="reference not present on this box")]

BLOCK = 256
WL3 = (0.48, 0.55, 0.65)


def _asphere_stop(be):
    """The tilted-stop doublet's layout with an even-asphere stop: the general variant's Newton intercept."""
    from optiland import optic

    lens = optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=45.0, thickness=6.0, material="N-BK7")
    lens.surfaces.add(index=2, radius=-70.0, thickness=5.0)
    lens.surfaces.add(index=3, thickness=45.0, is_stop=True, surface_type="even_asphere", radius=-120.0, conic=-0.6,
                      coefficients=[2e-4, -3e-6])
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=8.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def _with_surface_one(be, **kw):
    """An infinite-object singlet whose front surface takes ``kw``, a plane, and a plane stop behind it."""
    from optiland import optic

    lens = optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, thickness=6.0, material="N-BK7", **kw)
    lens.surfaces.add(index=2, radius=-70.0, thickness=5.0)
    lens.surfaces.add(index=3, thickness=45.0, is_stop=True)
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=6.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def _grid_before_stop(be):
    """A grid-sag front surface sampled from a sphere (R 45) plus an x y^2 departure.  The reference's paraxial aimer
    cannot trace a grid-sag surface (it has no radius), so the guesses are those of the R 45 sphere in its place."""
    from tests._grid_sag_systems import grid_kw, sphere_sag

    nodes = np.linspace(-9.0, 9.0, 37)
    return _with_surface_one(be, **grid_kw(nodes, nodes, lambda X, Y: sphere_sag(X, Y, 45.0) + 2e-4 * X * Y * Y))


def _grid_twin(be):
    return _with_surface_one(be, radius=45.0)


def _polygon_before_stop(be):
    from tests._polygon_systems import _poly, regular

    return _with_surface_one(be, radius=45.0, aperture=_poly(regular(6, 6.5, phase=0.2)))


def _polygon_on_stop(be):
    from tests._polygon_systems import _poly, regular

    lens = _tilted_stop(be)
    lens.surfaces[3].aperture = _poly(regular(7, 5.0, phase=0.1))
    return lens


# name: (builder, kernel variant, wavelengths drawn per ray or None for the primary one)
SYSTEMS = {
    "tilted": (_tilted_stop, "closed form", None),
    "tilted_3wl": (_tilted_stop, "closed form", WL3),
    "finite": (_finite_object, "closed form", None),
    "asphere": (_asphere_stop, "general", None),
    "zernike": (lambda be: _zernike_stop(be, 12.0), "general", None),
    "doe": (_doe_before_stop, "superset", None),
    "grid": (_grid_before_stop, "superset", None),
    "polygon_before": (_polygon_before_stop, "superset", None),
    "polygon_stop": (_polygon_on_stop, "superset", None),
}
SIZES = ("1", "31", "257", "wave+7")
_INPUTS, _HOST = {}, {}


def _n_wave():
    """Threads of one full wave of 256-thread CTAs on this device: more than launch_aim's grid at any occupancy."""
    import torch

    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count * (p.max_threads_per_multi_processor // BLOCK) * BLOCK


def _size(size):
    return _n_wave() + 7 if size == "wave+7" else int(size)


def _inputs(be, name, n, zernike_norm=None):
    """One solve's inputs for ``n`` seeded rays of system ``name`` (cached: the paraxial guesses are the slow part)."""
    key = (name, n, zernike_norm)
    if key not in _INPUTS:
        build, _, wls = SYSTEMS[name]
        lens = build(be) if zernike_norm is None else _zernike_stop(be, zernike_norm)
        rng = np.random.default_rng([n, sorted(SYSTEMS).index(name)])
        r, th = np.sqrt(rng.uniform(0.0, 1.0, n)), rng.uniform(0.0, 2.0 * np.pi, n)
        hx, hy = rng.uniform(-0.2, 0.2, n), rng.uniform(-0.5, 0.5, n)
        wl = None if wls is None else be.array(np.asarray(wls)[rng.integers(0, len(wls), n)])
        a = _aim_inputs(_grid_twin(be) if name == "grid" else lens, hx, hy, 0.8, wl=wl,
                        pupil=(r * np.cos(th), r * np.sin(th)))
        if name == "grid":
            a["table"] = _aim_table(lens, a["table"].wavelengths)
        a["scale"] = _scale(lens)
        _INPUTS[key] = a
    return _INPUTS[key]


def _arrays(a, dtype):
    """The solve's inputs as NumPy arrays of ``dtype``: the six guess arrays, w, Px and Py."""
    import optiland.backend as be

    g = {k: be.to_numpy(be.as_array_1d(v)).astype(dtype) for k, v in zip(KEYS, a["guess"])}
    n = g["x"].size
    g["w"] = np.broadcast_to(be.to_numpy(be.as_array_1d(a["wl"])), (n,)).astype(dtype)
    g["Px"], g["Py"] = be.to_numpy(a["Px"]).astype(dtype), be.to_numpy(a["Py"]).astype(dtype)
    return g


def _host(a, dtype, max_iter=None):
    """Host solve of ``a`` (cached for the untouched inputs): (solution, per-ray status, status word, variant)."""
    def run():
        rs = np.full(int(a["Px"].numel()), -1, dtype=np.int32)
        sol, st, variant = _host_solve(a, dtype=dtype, max_iter=max_iter, ray_status=rs)
        return sol, rs, st, variant

    key = (id(a), np.dtype(dtype).name, max_iter)
    if any(a is v for v in _INPUTS.values()):
        if key not in _HOST:
            _HOST[key] = run()
        return _HOST[key]
    return run()


def _aim_table(lens, wavelengths):
    """The aim table of ``lens`` as ``_aim_inputs`` packs it: surfaces [first, stop]."""
    from optiland_b200 import table as T
    from optiland_b200.pack import pack_surface_group

    full = pack_surface_group(lens.surfaces, np.unique(np.asarray(wavelengths, dtype=np.float64)))
    start = 1 if getattr(lens.object_surface, "is_infinite", False) else 0
    return T.SurfaceTable(full.surfaces[start:lens.surfaces.stop_index + 1], full.wavelengths)


def _dtab(a):
    from optiland_b200.trace import DeviceTable

    if "dtab" not in a:
        a["dtab"] = DeviceTable(a["table"], "cuda:0")
    return a["dtab"]


def _gpu_solve(a, g, max_iter=None, first=0, last=None):
    """One aim launch on copies of the arrays ``g`` (as ``_arrays`` makes them): (solution arrays, status word)."""
    import torch

    from optiland_b200.trace import aim_device

    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to("cuda:0") for k, v in g.items()}
    st = aim_device(_dtab(a), {k: t[k] for k in KEYS + ("w",)}, t["Px"], t["Py"], first,
                    a["table"].num_surfaces if last is None else last, a["r_stop"], a["J"], a["it"].tol,
                    a["it"].max_iter if max_iter is None else max_iter, a["inf"])
    return {k: t[k].cpu().numpy() for k in KEYS}, int(st.item())


def _bits(v):
    return np.ascontiguousarray(v).view(np.int64 if v.dtype == np.float64 else np.int32)


def _moved(a):
    return ("x", "y") if a["inf"] else ("L", "M")


def _residual64(a, sol):
    """|stop-local residual| of each ray of ``sol`` re-traced in fp64 by the host instantiation."""
    import optiland.backend as be

    from oracle.hostcheck_aim import aim_residual

    rays = {k: np.asarray(sol[k], dtype=np.float64) for k in KEYS}
    rays["w"] = np.broadcast_to(be.to_numpy(be.as_array_1d(a["wl"])), rays["x"].shape)
    ex, ey, _ = aim_residual(a["table"], rays, be.to_numpy(a["Px"]), be.to_numpy(a["Py"]), 0, a["table"].num_surfaces,
                             a["r_stop"])
    return np.hypot(ex, ey)


def _fp32_trace_error(a):
    """The largest |fp32 - fp64| stop residual the host instantiation reaches on this table for the fp32 guesses."""
    from oracle.hostcheck_aim import aim_residual

    g = _arrays(a, np.float32)
    px, py = g.pop("Px"), g.pop("Py")
    e32 = aim_residual(a["table"], g, px, py, 0, a["table"].num_surfaces, a["r_stop"], dtype=np.float32)
    g64 = {k: v.astype(np.float64) for k, v in g.items()}
    g64["w"] = _arrays(a, np.float64)["w"]                 # the table's fp64 wavelengths, not their fp32 roundings
    e64 = aim_residual(a["table"], g64, px.astype(np.float64),
                       py.astype(np.float64), 0, a["table"].num_surfaces, a["r_stop"])
    return float(np.nanmax(np.hypot(e32[0] - e64[0], e32[1] - e64[1])))


def _check_fp64(a, g, host, rs, got, st, what, min_converged=0.99):
    """The fp64 bars: the status word is the OR of the host's per-ray bits, the four arrays the solve does not move are
    bit-identical to the guesses, and each ray the host solved (status 0) is within 1e-10 x system scale of it (at
    least ``min_converged`` of the rays in batches of 257 and more).  Returns the largest difference."""
    assert st == int(np.bitwise_or.reduce(rs)), (what, st, np.unique(rs))
    for k in KEYS:
        if k not in _moved(a):
            assert np.array_equal(_bits(got[k]), _bits(g[k])), (what, k)
    ok = rs == 0
    assert rs.size < 257 or ok.mean() >= min_converged, (what, ok.mean())
    worst = 0.0
    for k in _moved(a):
        err = float(np.max(np.abs(got[k][ok] - host[k][ok]), initial=0.0))
        assert err <= 1e-10 * a["scale"], (what, k, err)
        worst = max(worst, err)
    return worst


# ---- the variant matrix ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("name", list(SYSTEMS))
def test_fp64_solve_matches_host_ray_by_ray(torch_backend, record_property, name, size):
    a = _inputs(torch_backend, name, _size(size))
    host, rs, _, variant = _host(a, np.float64)
    assert variant == SYSTEMS[name][1]
    assert a["table"].n_wl == len(np.unique(_arrays(a, np.float64)["w"]))
    g = _arrays(a, np.float64)
    got, st = _gpu_solve(a, g)
    record_property("max_fp64_diff", _check_fp64(a, g, host, rs, got, st, (name, size),
                                                 min_converged=0.3 if name == "doe" else 0.99))


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("name", list(SYSTEMS))
def test_fp32_solve_against_fp32_host(torch_backend, record_property, name, size):
    """Same status word and NaN-start rays as the fp32 host solve, the unmoved arrays untouched, and residuals re-traced
    in fp64 at most 3x the fp32 host solution's plus the fp64 solve's floor.  The fp32 default tolerance (1e-8) lies
    below fp32 resolution, so each solve runs all max_iter steps, and Broyden updates taken on rounding noise make a few
    rays wander chaotically: one ulp of difference in a guess moves ~5 % of the rays' final residuals past the bar, and
    the GPU's contractions of the trace into fused multiply-adds move 10-30 % (H100).  So the per-ray bar must hold for
    most rays, and the bar on the median residual for the batch."""
    a = _inputs(torch_backend, name, _size(size))
    host, rs, hst, variant = _host(a, np.float32)
    assert variant == SYSTEMS[name][1]
    g = _arrays(a, np.float32)
    got, st = _gpu_solve(a, g)
    assert st == hst, (name, size, st, hst)
    for k in KEYS:
        if k not in _moved(a):
            assert np.array_equal(_bits(got[k]), _bits(g[k])), k
    nan_start = (rs & _st().ST_AIM_NAN_START) != 0
    kept = np.all([_bits(got[k]) == _bits(g[k]) for k in _moved(a)], axis=0)
    assert kept[nan_start].all()
    r_gpu, r_host = _residual64(a, got), _residual64(a, host)
    sol64, rs64 = _host(a, np.float64)[:2]
    floor = float(np.max(_residual64(a, sol64)[rs64 == 0], initial=0.0))
    live = ~nan_start & np.isfinite(r_host)
    if not live.any():
        return
    within = np.nan_to_num(r_gpu[live], nan=np.inf) <= 3.0 * r_host[live] + floor
    assert within.mean() >= (0.5 if live.sum() >= 31 else 0.0), (name, size, within.mean())
    med_gpu, med_host = np.median(np.nan_to_num(r_gpu[live], nan=np.inf)), np.median(r_host[live])
    assert med_gpu <= 3.0 * med_host + floor, (name, size, med_gpu, med_host)
    record_property("fp32_median_residual_ratio", float(med_gpu / max(med_host, floor)))
    record_property("fp32_rays_within_per_ray_bar", float(within.mean()))


def _st():
    from optiland_b200 import table as T

    return T


# ---- the first steps: max_iter 0, 1, 2 ---------------------------------------------------------------------------------

@pytest.mark.parametrize("max_iter", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(SYSTEMS))
def test_first_steps_match_host_on_every_ray(torch_backend, record_property, name, dtype, max_iter):
    """max_iter = 0 leaves the guesses bit-identical; one and two steps are deterministic and match the host on every
    ray: fp64 within 1e-10 x scale, fp32 within 3x the fp32 trace error the host reaches on this table over |J| (the
    second fp32 step on 95 % of the rays)."""
    a = _inputs(torch_backend, name, _size("wave+7"))
    host, rs, hst, _ = _host(a, dtype, max_iter)
    g = _arrays(a, dtype)
    got, st = _gpu_solve(a, g, max_iter=max_iter)
    assert st == hst, (st, hst)
    if max_iter == 0:
        assert hst & _st().ST_AIM_UNCONVERGED
        for k in KEYS:
            assert np.array_equal(_bits(got[k]), _bits(g[k])), k
        return
    bar = 1e-10 * a["scale"] if dtype == np.float64 else 3.0 * _fp32_trace_error(a) / abs(a["J"])
    # fp32, second step: it uses the Broyden-updated J, which a near-singular update can make far smaller than J_factor;
    # the fp32 trace error of such a ray is amplified past the bar, so the bar must hold for 95 % of the rays (on an
    # H100: 96.7 % for the DOE system, where even the fp64 solve fails on half of the rays, and 99 % or more elsewhere)
    share = 0.95 if dtype == np.float32 and max_iter == 2 else 1.0
    worst = 0.0
    for k in KEYS:
        if k not in _moved(a):
            assert np.array_equal(_bits(got[k]), _bits(g[k])), k
            continue
        assert np.array_equal(np.isnan(got[k]), np.isnan(host[k])), k
        m = ~np.isnan(host[k])
        err = np.abs(got[k][m].astype(np.float64) - host[k][m])
        within = float(np.mean(err <= bar)) if m.any() else 1.0
        assert within >= share, (name, k, within, float(np.max(err)), bar)
        worst = max(worst, float(np.quantile(err, share, method="higher")) if m.any() else 0.0)
    record_property("max_diff_over_bar", worst / bar)


# ---- planted failures --------------------------------------------------------------------------------------------------

def _planted(n):
    nw = _n_wave()
    return np.array([0, 256, nw, n - 1])


@pytest.mark.parametrize("name", ["tilted", "finite"])
def test_nan_guesses_fail_only_their_own_rays(torch_backend, name):
    be = torch_backend
    a = _inputs(be, name, _size("wave+7"))
    n = int(a["Px"].numel())
    idx = _planted(n)
    k = 0 if a["inf"] else 4                       # x for an infinite object, M for a finite one
    guess = list(a["guess"])
    v = be.to_numpy(be.as_array_1d(guess[k])).copy()
    v[idx] = np.nan
    guess[k] = be.array(v)
    a2 = dict(a, guess=tuple(guess))
    rs0 = _host(a, np.float64)[1]
    host, rs, hst, _ = _host(a2, np.float64)
    # the planted rays fail as NaN starts; every other ray keeps its own outcome (the few unconverged ones included)
    assert (rs[idx] == _st().ST_AIM_NAN_START).all() and np.array_equal(np.delete(rs, idx), np.delete(rs0, idx))
    g = _arrays(a2, np.float64)
    got, st = _gpu_solve(a, g)
    assert st == _st().ST_AIM_NAN_START | int(np.bitwise_or.reduce(np.delete(rs0, idx)))
    for key in KEYS:
        assert np.array_equal(_bits(got[key][idx]), _bits(g[key][idx])), key
    _check_fp64(a, g, host, rs, got, st, name)


def test_wavelength_missing_from_the_table_fails_only_its_rays(torch_backend):
    be = torch_backend
    a = _inputs(be, "tilted_3wl", _size("wave+7"))
    assert a["table"].n_wl == 3
    n = int(a["Px"].numel())
    idx = _planted(n)
    w = be.to_numpy(a["wl"]).copy()
    w[idx] = 0.5
    a2 = dict(a, wl=be.array(w))
    host, rs, hst, _ = _host(a2, np.float64)
    assert hst == _st().ST_AIM_NAN_START and np.array_equal(np.flatnonzero(rs), idx), np.flatnonzero(rs)
    g = _arrays(a2, np.float64)
    got, st = _gpu_solve(a, g)
    assert st == _st().ST_AIM_NAN_START
    for key in KEYS:
        assert np.array_equal(_bits(got[key][idx]), _bits(g[key][idx])), key
    _check_fp64(a, g, host, rs, got, st, "missing wavelength")


def test_zernike_out_of_range_rays_set_the_range_bit(torch_backend):
    a = _inputs(torch_backend, "zernike", _size("wave+7"), zernike_norm=5.0)
    host, rs, hst, variant = _host(a, np.float64)
    assert variant == "general" and hst & _st().ST_ZERNIKE_RANGE and (rs == 0).any()
    g = _arrays(a, np.float64)
    got, st = _gpu_solve(a, g)
    assert st & _st().ST_ZERNIKE_RANGE
    _check_fp64(a, g, host, rs, got, st, "zernike range", min_converged=0.0)


# ---- per-ray independence ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", ["tilted_3wl", "finite", "zernike", "grid"])
def test_rays_are_independent_of_their_batch(torch_backend, name, dtype):
    """Reversing the batch reverses the result bit for bit; [0, k) and [k, n) in two launches give the full launch's."""
    a = _inputs(torch_backend, name, _size("wave+7"))
    g = _arrays(a, dtype)
    full, st = _gpu_solve(a, g)
    rev, st_rev = _gpu_solve(a, {k: v[::-1] for k, v in g.items()})
    assert st_rev == st
    for k in KEYS:
        assert np.array_equal(_bits(rev[k][::-1]), _bits(full[k])), k
    cut = _n_wave() // 2 + 3
    lo, st_lo = _gpu_solve(a, {k: v[:cut] for k, v in g.items()})
    hi, st_hi = _gpu_solve(a, {k: v[cut:] for k, v in g.items()})
    assert st_lo | st_hi == st
    for k in KEYS:
        assert np.array_equal(_bits(np.concatenate([lo[k], hi[k]])), _bits(full[k])), k


# ---- the C ABI ---------------------------------------------------------------------------------------------------------

def _table_of(lens):
    """Every surface of ``lens`` after the object surface, packed at its primary wavelength."""
    import optiland.backend as be

    from optiland_b200 import table as T
    from optiland_b200.pack import pack_surface_group

    full = pack_surface_group(lens.surfaces, np.atleast_1d(be.to_numpy(be.as_array_1d(lens.primary_wavelength))))
    return T.SurfaceTable(full.surfaces[1:], full.wavelengths)


def test_abi_rejects_bad_calls_without_a_launch(torch_backend):
    import torch

    from optiland_b200 import _lib
    from optiland_b200.batch import BatchedTable, template_params
    from optiland_b200.trace import DeviceTable
    from tests import _bsdf_systems, _coating_systems
    from oracle.make_golden import zernike_singlet

    be = torch_backend
    lib = _lib.load()
    a = _inputs(be, "tilted", 31)
    dt = _dtab(a)
    n = 32
    buf = {k: torch.zeros(n + 2, dtype=torch.float64, device="cuda:0") for k in KEYS + ("w", "Px", "Py")}
    status = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    rays = _lib.OlbRays(**{k: buf[k].data_ptr() for k in KEYS + ("w",)})
    nsurf = a["table"].num_surfaces

    def call(table=dt, **kw):
        c = dict(first=0, last=nsurf, n_rays=n, rays=C.pointer(rays), Px=buf["Px"].data_ptr(),
                 Py=buf["Py"].data_ptr(), r_stop=a["r_stop"], J_factor=a["J"], tol=1e-8, max_iter=20, infinite=1,
                 status=status.data_ptr())
        c.update(kw)
        l0 = lib.olb_launch_count()
        rc = lib.olb_aim_f64(C.byref(table.c), C.byref(_lib.OlbAimCall(**c)), None)
        torch.cuda.synchronize()
        return rc, lib.olb_launch_count() - l0

    err = {"arg": -1, "unsupported": -2, "align": -4}
    cases = {
        "NULL status": (dict(status=None), "arg"),
        "misaligned Px": (dict(Px=buf["Px"].data_ptr() + 8), "align"),
        "n_rays < 0": (dict(n_rays=-1), "arg"),
        "first < 0": (dict(first=-1), "arg"),
        "last past the table": (dict(last=nsurf + 1), "arg"),
        "first >= last": (dict(first=nsurf - 1, last=nsurf - 1), "arg"),
        "max_iter < 0": (dict(max_iter=-1), "arg"),
    }
    for what, (kw, e) in cases.items():
        assert call(**kw) == (err[e], 0), what

    batched = BatchedTable(a["table"], np.stack([template_params(a["table"])] * 2))
    assert call(batched) == (err["unsupported"], 0), "batched table"
    others = {"BSDF": _bsdf_systems.gaussian_lens(be), "Fresnel": zernike_singlet(fresnel=True),
              "thin film": _coating_systems.coated_doublet(be, "thin_film")}
    for what, lens in others.items():
        tab = DeviceTable(_table_of(lens), "cuda:0")
        assert call(tab, last=tab.table.num_surfaces) == (err["unsupported"], 0), what
    assert call(n_rays=0) == (0, 0)
    assert int(status.item()) == 0


# ---- live robust traces through CudaEngine -----------------------------------------------------------------------------

def _trace_on_cuda(name, precision, plugin):
    """Optic.trace(0, 0.7, primary, 64, "uniform") of sample ``name`` on cuda:0 in ``precision``, with or without the
    plugin: its records as NumPy arrays, or the exception type it raised."""
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin as P

    be.set_backend("torch")
    be.set_precision(precision)
    be.grad_mode.disable()
    be.set_device("cuda")
    if plugin:
        P.install(engine=P.CudaEngine())
    try:
        lens = _sample(name)
        lens.trace(0.0, 0.7, lens.primary_wavelength, 64, "uniform")
        return {k: be.to_numpy(getattr(lens.surfaces, k)).astype(np.float64)
                for k in ("x", "y", "z", "L", "M", "N", "opd", "intensity")}
    except Exception as e:  # noqa: BLE001  (the outcome is compared with the stock reference's)
        return type(e)
    finally:
        P.uninstall()
        be.set_device("cpu")
        be.set_precision("float64")
        be.set_backend("numpy")


@pytest.mark.parametrize("name", ROBUST)
def test_robust_trace_on_cuda_64x64_uniform_equals_numpy(name):
    """The 3 096 rays of a 64 x 64 uniform pupil (13 CTAs) in each solve of the robust aimer's continuation, fp64,
    against the NumPy reference."""
    want = _numpy_records(name, [(0.0, 0.7)], num_rays=64, distribution="uniform")[0]
    got = _trace_on_cuda(name, "float64", plugin=True)
    assert isinstance(got, dict), got
    assert got["x"].shape[-1] > 12 * BLOCK, got["x"].shape
    _check_record_arrays(got, want, (name, "64x64 uniform"))


@pytest.mark.parametrize("name", ROBUST)
def test_robust_trace_on_cuda_float32_matches_stock_reference(name):
    """At float32 the stock reference returns (its solves cannot meet the 1e-8 tolerance, so its continuation halves
    down to its smallest interval); the plugin must return too, with records as close to the fp64 NumPy records as 3x
    the stock reference's own fp32 error."""
    want = _numpy_records(name, [(0.0, 0.7)], num_rays=64, distribution="uniform")[0]
    stock = _trace_on_cuda(name, "float32", plugin=False)
    got = _trace_on_cuda(name, "float32", plugin=True)
    assert isinstance(stock, dict) == isinstance(got, dict), (stock if not isinstance(stock, dict) else got)
    if not isinstance(stock, dict):
        assert got is stock
        return
    for k, v in want.items():
        assert got[k].shape == stock[k].shape == v.shape, k
        assert np.array_equal(np.isnan(got[k]), np.isnan(stock[k])), k
        m = np.isfinite(stock[k])
        bar = 3.0 * float(np.max(np.abs(stock[k][m] - v[m]), initial=0.0))
        err = float(np.max(np.abs(got[k][m] - v[m]), initial=0.0))
        assert err <= bar, (name, k, err, bar)
