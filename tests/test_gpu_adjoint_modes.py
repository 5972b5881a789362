"""Every instantiation of the adjoint kernel, trace_bwd_kernel<T, ACC, POLY> (optiland_b200/csrc/olb_trace.cu), against
the host instantiation of the same arithmetic (tests/hostcheck).

olb_trace.cu:783-793 picks one of three ways to sum the parameter gradients from the table's shared-memory footprint:
ACC 2 (one fp32 / fp64 accumulator column per thread), ACC 1 (two neighbouring lanes share a column after one shuffle)
and ACC 0 (each surface's values are warp-reduced at once into a shared fp64 block).  POLY compiles the table-gradient
paths of polynomial-family / Forbes / grid-sag surfaces in.  Ordinary systems only reach ACC 1 and ACC 0 when they are
large, so the systems here are small bases padded with transparent planes (a plane with n1 == n2 leaves every ray
alone) until the footprint lands in the wanted mode; some of the planes are tilted, which puts the nine dLoss/dR slots
of a tilted pose into every mode.  One profiled launch per (table, precision) checks that the instantiation that ran
is the one ``adjoint_mode`` predicts; the other GPU tests assert that prediction for the tables they run.

The CPU tests hold the parametrization to the twelve instantiations and the padding to the oracle."""
from __future__ import annotations

import ctypes as C
import dataclasses
import functools
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from optiland_b200 import _lib
from optiland_b200 import table as T
from tests._util import REC, Case

BLOCK = 256                    # threads per CTA of the backward kernel (olb_trace.cu BLOCK)
SMEM_PER_CTA = 113 * 1024      # two resident CTAs per SM must fit (olb_trace.cu:787)
BASES = ("cooke_c1", "zernike_fringe", "tilted_fold")
POLY_BASES = ("zernike_fringe",)
DTYPES = ("float64", "float32")
MODES = (2, 1, 0)
MODE_COMPARISON_SEED = 5       # the bundle test_every_mode_gives_the_same_gradient traces through every padding
# the widest bundle member: its launch offsets from the bundle centre scaled by this, far enough for some rays to miss
# the first curved surface (radius 22, 40 and 50 mm against bundles of 13, 8 and 5.5 mm)
WIDE = {"cooke_c1": 2.5, "zernike_fringe": 6.0, "tilted_fold": 12.0, "litho_telecentric": 2.5}
RAY_KEYS = ("x", "y", "z", "L", "M", "N", "i", "w")
GIN_KEYS = ("x", "y", "z", "L", "M", "N", "i", "opd")


# ---- which instantiation a launch takes --------------------------------------------------------------------------
def adjoint_mode(dtab, dtype) -> tuple[int, bool]:
    """(ACC, POLY) of the trace_bwd_kernel instantiation olb_trace_bwd_* launches for ``dtab`` (an ``OlbDeviceTable``
    or anything with its fields bytes_f64 / bytes_f32, bwd_slots, bwd_supported) in ``dtype``; mirrors
    olb_trace.cu:783-789 (the table staged in shared memory behind a 16-byte barrier, then the accumulators)."""
    wide = _is64(dtype)
    size = 8 if wide else 4
    blob = int(dtab.bytes_f64 if wide else dtab.bytes_f32)
    base = 16 + ((blob + 15) & ~15)
    smem_acc = base + int(dtab.bwd_slots) * BLOCK * size
    smem_pair = base + int(dtab.bwd_slots) * (BLOCK // 2) * size
    acc = 2 if smem_acc <= SMEM_PER_CTA else (1 if smem_pair <= SMEM_PER_CTA else 0)
    return acc, int(dtab.bwd_supported) == 2


def _is64(dtype) -> bool:
    return dtype in ("float64", torch.float64, np.float64)


def _torch_dtype(dtype):
    return torch.float64 if _is64(dtype) else torch.float32


def _np_dtype(dtype):
    return np.float64 if _is64(dtype) else np.float32


@functools.lru_cache(maxsize=1)
def _hc():
    from oracle.hostcheck_api import load

    hc = load()
    for name in ("olbhc_bwd_slots", "olbhc_bwd_level", "olbhc_single_blob"):
        getattr(hc, name).restype = C.c_int
    return hc


def host_table_fields(table: T.SurfaceTable) -> SimpleNamespace:
    """The fields of ``OlbDeviceTable`` that ``adjoint_mode`` reads, from the host preparation of the table (the same
    olb_prep.h the upload runs)."""
    hc = _hc()
    ht = _lib.HostTable(table)
    buf = (C.c_ubyte * (1 << 20))()
    feats, err = C.c_uint(0), C.create_string_buffer(256)
    sizes = [hc.olbhc_single_blob(C.byref(ht.c), which, buf, len(buf), C.byref(feats), err, 256) for which in (0, 1)]
    assert min(sizes) > 0, err.value
    return SimpleNamespace(bytes_f64=sizes[0], bytes_f32=sizes[1], bwd_slots=hc.olbhc_bwd_slots(C.byref(ht.c)),
                           bwd_supported=hc.olbhc_bwd_level(C.byref(ht.c)))


_KERNEL_NAME = re.compile(r"trace_bwd_kernel<\s*(float|double)\s*,\s*(?:\(int\))?\s*(\d+)\s*,\s*(?:\(bool\))?\s*(true|false|1|0)\s*>")
_KERNEL_MANGLED = re.compile(r"trace_bwd_kernelI([fd])Li(\d+)ELb([01])E")
PROFILED: set = set()          # (T, ACC, POLY) of every launch profiled in this session


def parse_instantiation(name: str) -> tuple[str, int, bool]:
    """(T, ACC, POLY) from a trace_bwd_kernel name as the profiler reports it (demangled in either spelling of the
    template arguments, or mangled)."""
    m = _KERNEL_NAME.search(name)
    if m:
        return m.group(1), int(m.group(2)), m.group(3) in ("true", "1")
    m = _KERNEL_MANGLED.search(name)
    assert m, f"cannot read the template arguments of {name!r}"
    return ("double" if m.group(1) == "d" else "float"), int(m.group(2)), m.group(3) == "1"


def profiled_backward(fn) -> tuple[str, int, bool]:
    """Run ``fn`` (one olb_trace_bwd_* call) once under torch.profiler and return the (T, ACC, POLY) of the one
    trace_bwd_kernel launch the session reports.  The session is opened with the device idle and held open a few
    milliseconds past the launch's completion, so that the kernel's activity record is neither stamped near the
    session's edges nor still in flight when it closes; no launch seen, or more than one, fails."""
    import time

    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        time.sleep(0.005)
        fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    names = [e.name for e in prof.events() if "trace_bwd_kernel" in e.name]
    assert len(names) == 1, f"expected one trace_bwd_kernel launch, the profiler saw {names}"
    inst = parse_instantiation(names[0])
    PROFILED.add(inst)
    return inst


# ---- systems ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def base_system(name: str):
    """(table, rays, first real surface) of a fixture at one wavelength: Newton tolerance 1e-13 as in the other adjoint
    tests, and a radial aperture on the second real surface at 80 % of the fixture's own ray height there, so that
    part of every bundle is clipped."""
    c = Case(name)
    assert c.table.n_wl == 1
    surfaces = [dataclasses.replace(s, tol=1e-13) if s.kind in T.NEWTON_KINDS else s for s in c.table.surfaces]
    s0 = next(j for j, s in enumerate(surfaces) if s.kind != T.GEOM_NOOP)
    s_ap = s0 + 1
    r = np.hypot(c.rec["x"][s_ap] - surfaces[s_ap].t[0], c.rec["y"][s_ap] - surfaces[s_ap].t[1])
    surfaces[s_ap] = dataclasses.replace(surfaces[s_ap], aperture=T.aperture_radial(0.8 * float(np.nanmax(r))))
    return T.SurfaceTable(surfaces, c.table.wavelengths), c.rays, s0


def bundle(name: str, n: int, seed: int) -> dict:
    """``n`` rays drawn from the fixture's launch state; launch offsets from the bundle centre (position and direction)
    scaled by 0.5-1 for most rays and by 1.2-WIDE for every seventh, which clips them at the aperture or makes them miss
    a surface."""
    _, r0, _ = base_system(name)
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, r0["x"].size, n)
    f = rng.uniform(0.5, 1.0, n)
    wide = rng.random(n) < 1 / 7
    f[wide] = rng.uniform(1.2, WIDE[name], int(wide.sum()))
    return _widened(r0, pick, f)


def _widened(r0, pick, f):
    out = {k: np.asarray(r0[k], dtype=np.float64)[pick].copy() for k in RAY_KEYS}
    for k in ("x", "y", "L", "M"):
        c = float(np.mean(r0[k]))
        g = f if k in ("x", "y") else 1 + 0.5 * (f - 1)      # directions widen half as fast
        out[k] = c + g * (out[k] - c)
    out["N"] = np.sqrt(1 - out["L"] ** 2 - out["M"] ** 2)
    return out


def _bundle_radius(name: str, dz: float) -> float:
    """Largest distance from the axis of any ray ``bundle`` can draw, from its launch plane to ``dz`` beyond it (the
    extreme scalings 0.5 and WIDE bound it: a ray's position is linear in its scaling)."""
    _, r0, _ = base_system(name)
    m = r0["x"].size
    h = 0.0
    for f in (0.5, WIDE[name]):
        r = _widened(r0, np.arange(m), np.full(m, f))
        for d in (0.0, dz):
            h = max(h, float(np.max(np.hypot(r["x"] + r["L"] / r["N"] * d, r["y"] + r["M"] / r["N"] * d))))
    return h


@functools.lru_cache(maxsize=None)
def _first_surface_front(name: str) -> float:
    """The smallest z at which the first real surface is met by rays of ``bundle`` (its vertex, or where its sag or
    tilt brings it closer to the launch plane): fixture rays at twelve scalings from 0.5 to WIDE, on the oracle."""
    from oracle import trace_oracle as O

    table, r0, s0 = base_system(name)
    m = r0["x"].size
    f = np.repeat(np.linspace(0.5, WIDE[name], 12), m)
    _, rec, _ = O.trace(table, _widened(r0, np.tile(np.arange(m), 12), f))
    z = rec["z"][s0]
    return min(float(table.surfaces[s0].t[2]), float(np.min(z[np.isfinite(z)])))


@functools.lru_cache(maxsize=None)
def padded(name: str, k: int) -> T.SurfaceTable:
    """The base system with ``k`` transparent planes (n1 == n2 == the index there, no aperture) in the first 80 % of the
    gap between the launch plane and the nearest point of the first real surface the bundle meets; every third plane,
    from the second on, is tilted (about x and y in turn).  A tilted plane spans +- h tan(tilt) in z over a bundle of
    radius h; the tilt keeps that under half the spacing so that every ray meets the planes in order, and the last
    plane stays more than a spacing clear of the first real surface (a plane met behind the ray changes its OPD).
    test_padding_leaves_the_rays_alone checks the result on the bundles the comparisons use."""
    table, r0, s0 = base_system(name)
    if k == 0:
        return table
    z0 = float(np.max(r0["z"]))
    gap = _first_surface_front(name) - z0
    assert gap > 0
    spacing = 0.8 * gap / (k + 1)
    h = _bundle_radius(name, gap)
    tilt = min(np.deg2rad(3.0), float(np.arctan(0.5 * spacing / h)))
    nn = table.surfaces[s0].n1.copy()
    planes = []
    for j in range(k):
        R = np.eye(3)
        if j % 3 == 1:
            R = T.rotation_matrix(tilt, 0.0, 0.0) if j % 6 == 1 else T.rotation_matrix(0.0, tilt, 0.0)
        planes.append(T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0.0, 0.0, z0 + spacing * (j + 1)], R=R, n1=nn.copy(), n2=nn.copy()))
    return T.SurfaceTable(table.surfaces[:s0] + planes + table.surfaces[s0:], table.wavelengths)


@functools.lru_cache(maxsize=None)
def planes_for(name: str, dtype: str, mode: int) -> int:
    """The fewest padding planes that put ``name``'s adjoint in ``dtype`` into accumulation mode ``mode``."""
    if name == "litho_telecentric":
        return 0
    for k in range(T.MAX_SURFACES - base_system(name)[0].num_surfaces + 1):
        if adjoint_mode(host_table_fields(padded(name, k)), dtype)[0] == mode:
            return k
    raise AssertionError(f"{name} does not reach ACC {mode} in {dtype}")


def system(name: str, dtype: str, mode: int) -> T.SurfaceTable:
    return padded(name, planes_for(name, dtype, mode))


def modes_of(name: str, dtype: str) -> tuple[int, ...]:
    """The modes padding can reach: the tilted fold's five tilted surfaces already take 64 slots, ACC 1 in fp64."""
    return (1, 0) if (name, dtype) == ("tilted_fold", "float64") else MODES


# (base, dtype, ACC): every instantiation, each from a plain, a polynomial-family and a tilted base; the 44-surface
# lithography lens is a real system that takes ACC 0 unpadded
CASES = [(b, d, m) for b in BASES for d in DTYPES for m in modes_of(b, d)] + [("litho_telecentric", d, 0) for d in DTYPES]
CASE_IDS = [f"{b}-{d}-acc{m}" for b, d, m in CASES]


# ---- device calls ---------------------------------------------------------------------------------------------------
def device_forward(dtab, rays: dict, dtype, first: int = 0, last: int | None = None):
    """Forward records of ``rays`` over [first, last) on the device: (launch-state tensors x y z L M N i opd, (8, rows,
    stride) record buffer)."""
    from optiland_b200.trace import _c_records, _out_buffer, _trace

    tdt = _torch_dtype(dtype)
    last = dtab.table.num_surfaces if last is None else last
    n = rays["x"].size
    ins = [torch.tensor(np.asarray(rays[k] if k in rays else np.zeros(n)), dtype=tdt, device=dtab.device) for k in GIN_KEYS]
    w = torch.tensor(rays["w"], dtype=tdt, device=dtab.device)
    buf = _out_buffer(8, last - first, n, tdt, dtab.device)
    c_rays = _lib.OlbRays(**{k: t.data_ptr() for k, t in zip(GIN_KEYS, ins)}, w=w.data_ptr())
    _trace(dtab, dtab.device, tdt, first, last, n, _lib.TF_NO_FINAL, rays=c_rays, rec=_c_records(buf), own_status=False)
    torch.cuda.synchronize()
    return ins, buf


def device_backward(dtab, dtype, ins, buf, grec, first=0, last=None, lo=0, n=None, mask=(1 << 64) - 1, want_gin=True,
                    null=()):
    """One olb_trace_bwd_* call over rays [lo, lo + n) of the forward buffers (pointers offset into them): returns
    (dLoss/d launch state as a list of 8 tensors or None, grad_params (S, GP_COUNT), grad_tables or None).  ``grec``:
    (8, rows, stride) tensor; the quantities in ``null`` are passed as NULL."""
    tdt = _torch_dtype(dtype)
    es = 8 if _is64(dtype) else 4
    S = dtab.table.num_surfaces
    last = S if last is None else last
    n = ins[0].numel() - lo if n is None else n
    c_in = _lib.OlbRays(**{k: t.data_ptr() + lo * es for k, t in zip(GIN_KEYS, ins)})
    c_rec = _lib.OlbRecords(*[buf[j].data_ptr() + lo * es for j in range(8)], buf.shape[-1])
    c_grec = _lib.OlbRecords(*[None if j in null else grec[j].data_ptr() + lo * es for j in range(8)], grec.shape[-1])
    gin = [torch.zeros(n, dtype=tdt, device=dtab.device) for _ in range(8)] if want_gin else None
    c_gin = _lib.OlbRays(**{k: t.data_ptr() for k, t in zip(GIN_KEYS, gin)}) if want_gin else None
    gpar = torch.zeros((S, _lib.GP_COUNT), dtype=torch.float64, device=dtab.device)
    poly = int(dtab.c.bwd_supported) == 2
    gtab = torch.zeros((S, 2, _lib.GT_DIM, _lib.GT_DIM), dtype=torch.float64, device=dtab.device) if poly else None
    lib = _lib.load()
    rc = getattr(lib, f"olb_trace_bwd_{'f64' if _is64(dtype) else 'f32'}")(
        C.byref(dtab.c), first, last, C.byref(c_in), C.byref(c_rec), C.byref(c_grec),
        C.byref(c_gin) if c_gin is not None else None, C.c_void_p(gpar.data_ptr()),
        C.c_void_p(gtab.data_ptr() if gtab is not None else None), n, C.c_uint64(mask), C.c_void_p(0))
    _lib.check(rc, "olb_trace_bwd")
    torch.cuda.synchronize()
    return gin, gpar, gtab


def random_weights(buf, seed, rows=None):
    """dLoss/d(records): a random linear functional, zero wherever the record is not finite (as the product's losses
    weight rays that miss a surface); ``rows``: only these record rows are weighted."""
    g = torch.Generator(device=buf.device)
    g.manual_seed(seed)
    w = torch.randn(buf.shape, generator=g, device=buf.device, dtype=torch.float64).to(buf.dtype)
    if rows is not None:
        keep = torch.zeros(buf.shape[1], dtype=torch.bool, device=buf.device)
        keep[list(rows)] = True
        w[:, ~keep] = 0
    return torch.where(torch.isfinite(buf), w, torch.zeros((), dtype=buf.dtype, device=buf.device))


def _np(t, n):
    return t[..., :n].double().cpu().numpy()


def _rel(a, b, scale):
    """max |a - b| over entries finite in the reference ``b`` / ``scale``; the NaN patterns must agree."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), "NaN pattern differs"
    m = np.isfinite(b)
    return float(np.max(np.abs(a[m] - b[m]))) / scale if m.any() else 0.0


def _scale(a):
    a = np.asarray(a, dtype=np.float64)
    a = a[np.isfinite(a)]
    return max(float(np.max(np.abs(a))) if a.size else 0.0, 1e-300)


# ---- CPU: the parametrization and the padding ---------------------------------------------------------------------
def test_parametrization_reaches_every_instantiation():
    """Every (base, dtype, ACC) case lands in its mode by the host preparation of its padded table, is backward-
    supported and stays under the surface cap, and the cases cover all twelve (T, ACC, POLY) instantiations."""
    seen = {}
    for name, dtype, mode in CASES:
        table = system(name, dtype, mode)
        f = host_table_fields(table)
        assert f.bwd_supported >= 1, (name, dtype, mode)
        assert table.num_surfaces <= T.MAX_SURFACES
        acc, poly = adjoint_mode(f, dtype)
        assert acc == mode, (name, dtype, mode, acc)
        assert poly == (name in POLY_BASES), (name, poly)
        inst = ("double" if _is64(dtype) else "float", acc, poly)
        seen.setdefault(inst, []).append(f"{name}+{planes_for(name, dtype, mode)} planes ({f.bwd_slots} slots)")
    for inst in sorted(seen):
        print("trace_bwd_kernel<%s, %d, %s>:" % (inst[0], inst[1], str(inst[2]).lower()), ", ".join(seen[inst]))
    assert set(seen) == {(t, a, p) for t in ("double", "float") for a in MODES for p in (False, True)}


def test_mode_rule_on_known_tables():
    """adjoint_mode on footprints either side of the thresholds, and the profiler-name parser on every spelling."""
    f = SimpleNamespace(bytes_f64=1000, bytes_f32=500, bwd_slots=50, bwd_supported=1)
    assert adjoint_mode(f, "float64") == (2, False) and adjoint_mode(f, "float32") == (2, False)
    f.bwd_slots = 100
    assert adjoint_mode(f, "float64") == (1, False) and adjoint_mode(f, "float32") == (2, False)
    f.bwd_slots, f.bwd_supported = 200, 2
    assert adjoint_mode(f, "float64") == (0, True) and adjoint_mode(f, "float32") == (1, True)
    # fp32 pairs: 16 + 512 bytes in front of 224 x 128 x 4 = 114 688 fits in 115 712, one more slot does not
    f.bwd_slots = 224
    assert adjoint_mode(f, "float32")[0] == 1
    f.bwd_slots = 225
    assert adjoint_mode(f, "float32")[0] == 0
    assert parse_instantiation("void olb::trace_bwd_kernel<double, 0, true>(olb::BwdArgs)") == ("double", 0, True)
    assert parse_instantiation("void olb::trace_bwd_kernel<float, (int)1, (bool)0>(olb::BwdArgs)") == ("float", 1, False)
    assert parse_instantiation("_ZN3olb16trace_bwd_kernelIdLi2ELb1EEEvNS_7BwdArgsE") == ("double", 2, True)


@pytest.mark.parametrize("name", BASES)
def test_padding_leaves_the_rays_alone(name):
    """The premise of the padding, on the oracle: for every padded table the GPU tests use, the image row and the
    second real surface's row of the padded system equal the unpadded system's to 1e-12 x scale, with the same NaN
    pattern, on the bundle test_every_mode_gives_the_same_gradient compares the modes on (the other GPU tests compare
    a padded table with itself) -- which clips some rays at the aperture and loses some on a surface."""
    from oracle import trace_oracle as O

    table, _, s0 = base_system(name)
    rays = bundle(name, 4099, seed=MODE_COMPARISON_SEED)
    _, ref, _ = O.trace(table, rays)
    scale = Case(name).scale
    rows = ((-1, -1), (s0 + 1, s0 + 1))
    # Rays whose records move by more than the tolerance when their launch point moves by 1e-14 mm (a few ulps) cannot
    # be held to it through any change of rounding: the tilted fold has 2 such rays of 4099, its mirror meets them where
    # a last-bit change of direction grows a millionfold.  They are held to 1e-6 x scale, which still separates them
    # from a plane met out of order (millimetres of OPD).
    sensitive = np.zeros(rays["x"].size, dtype=bool)
    for dx, dy in ((1e-14, 0.0), (0.0, 1e-14), (-1e-14, 1e-14)):
        _, moved, _ = O.trace(table, dict(rays, x=rays["x"] + dx, y=rays["y"] + dy))
        for row, _ in rows:
            for q in REC:
                a, b = moved[q][row], ref[q][row]
                sensitive |= (np.isnan(a) != np.isnan(b)) | (np.abs(np.nan_to_num(a - b)) > 1e-12 * scale)
    assert sensitive.mean() <= 1e-3, int(sensitive.sum())
    ks = sorted({planes_for(name, d, m) for d in DTYPES for m in modes_of(name, d)} - {0})
    assert ks
    for k in ks:
        _, rec, _ = O.trace(padded(name, k), rays)
        for row_b, row_p in ((-1, -1), (s0 + 1, s0 + 1 + k)):
            for q in REC:
                a, b = rec[q][row_p], ref[q][row_b]
                assert np.array_equal(np.isnan(a), np.isnan(b)), (k, q, row_b)
                err = np.abs(np.where(np.isfinite(b), a - b, 0.0))
                assert np.max(err[~sensitive]) <= 1e-12 * scale, (k, q, row_b)
                assert np.max(err[sensitive], initial=0.0) <= 1e-6 * scale, (k, q, row_b)


@pytest.mark.parametrize("name", BASES + ("litho_telecentric",))
def test_bundles_clip_and_lose_rays(name):
    """Every bundle the GPU tests draw has rays clipped by the aperture (finite, zero intensity) and rays that miss a
    surface (NaN), and most of its rays reach the image."""
    from oracle import trace_oracle as O

    table, _, s0 = base_system(name)
    _, rec, _ = O.trace(table, bundle(name, 4099, seed=MODE_COMPARISON_SEED))
    lost = np.mean(~np.isfinite(rec["x"][-1]))
    clipped = np.mean(np.isfinite(rec["x"][s0 + 1]) & (rec["intensity"][s0 + 1] == 0))
    print(f"[{name}] lost {lost:.3f}, clipped at the aperture {clipped:.3f}")
    assert 0 < lost < 0.3 and clipped > 0


def test_total_internal_reflection_carries_no_gradient():
    """A ray that meets a refracting surface beyond the critical angle keeps a finite intercept there but a NaN
    direction.  It carries no gradient from that surface on: the adjoint of a bundle with such rays is finite, and with
    their weights zeroed it equals the adjoint of the bundle without them.  (Before, the NaN partials of that surface
    times even a zero adjoint turned the parameter gradients of every surface in front of it NaN, for the whole
    bundle.)"""
    from oracle import trace_oracle as O
    from oracle.hostcheck_api import load, run_backward

    table, _, _ = base_system("tilted_fold")
    rays = bundle("tilted_fold", 256, seed=2)
    S = table.num_surfaces
    _, rec, _ = O.trace(table, rays)
    tir = np.any(np.isfinite(rec["x"]) & np.isnan(rec["L"]), axis=0)
    assert 0 < tir.sum() < 256
    rng = np.random.default_rng(12)
    w = {q: rng.normal(size=(S, 256)) * np.isfinite(rec[q]) for q in REC}
    gin, gpar = run_backward(load(), table, rays, rec, w)
    assert np.all(np.isfinite(gpar)) and all(np.all(np.isfinite(gin[k])) for k in GIN_KEYS)
    keep = ~tir
    for q in REC:
        w[q][:, tir] = 0
    gin, gpar = run_backward(load(), table, rays, rec, w)
    gin_k, gpar_k = run_backward(load(), table, {k: v[keep] for k, v in rays.items()}, {q: rec[q][:, keep] for q in REC},
                                 {q: w[q][:, keep] for q in REC})
    assert np.abs(gpar).max() > 0
    assert np.max(np.abs(gpar - gpar_k)) <= 1e-12 * np.abs(gpar).max()
    for k in GIN_KEYS:
        assert np.all(gin[k][tir] == 0)
        assert np.array_equal(gin[k][keep], gin_k[k])


def test_host_adjoint_over_a_surface_range():
    """run_backward over [first, last) (the state in front of ``first`` as input, records of that range) gives the
    parameter gradients of surfaces first .. last-1 that the whole-table adjoint gives when the loss reads only those
    rows, and nothing for the others."""
    from oracle import trace_oracle as O
    from oracle.hostcheck_api import load, run_backward

    table = padded("tilted_fold", 4)
    rays = bundle("tilted_fold", 64, seed=2)
    S = table.num_surfaces
    first, last = 3, S - 1
    _, rec, _ = O.trace(table, rays)
    rng = np.random.default_rng(3)
    w = {q: rng.normal(size=(S, 64)) * np.isfinite(rec[q]) for q in REC}
    for q in REC:
        w[q][:first] = 0
        w[q][last:] = 0
    _, gfull = run_backward(load(), table, rays, rec, w)
    rin = {q: rec[k][first - 1] for q, k in zip(RAY_KEYS[:7], REC[:7])}
    rin["w"] = rays["w"]
    _, gsub = run_backward(load(), table, rin, {q: rec[q][first:last] for q in REC}, {q: w[q][first:last] for q in REC},
                           first=first, last=last)
    assert np.any(gsub[first:last])
    assert not np.any(gsub[:first]) and not np.any(gsub[last:])
    assert np.max(np.abs(gsub[first:last] - gfull[first:last])) <= 1e-12 * np.abs(gfull).max()


# ---- GPU ------------------------------------------------------------------------------------------------------------
# What fp32 achieves against the host instantiation in fp32 (max |kernel - host| / max |host| over the sizes of
# test_each_instantiation_matches_the_host_instantiation), per base and mode, measured on an H100 80GB HBM3 at a 700 W
# power limit and identical over six runs; the test asserts 3x these.  The tilted fold's entries come from a few rays
# of its 4099-ray bundle: the launch-state gradient, which sums nothing across rays, differs from the host as much, and
# its ACC 0 entry went from 2.5e-7 to 1.4e-4 when the padding planes moved by 15 um.  They measure how that system's
# per-ray adjoint amplifies a change of fp32 rounding, not the accumulation, and hold only for this padding.  fp64
# achieves <= 4.6e-15 in every case against the 1e-10 asserted.
FP32_ACHIEVED = {
    ("cooke_c1", 2): dict(params=6.4e-7, launch=8.8e-7),
    ("cooke_c1", 1): dict(params=2.3e-7, launch=5.6e-7),
    ("cooke_c1", 0): dict(params=5.3e-7, launch=5.2e-7),
    ("zernike_fringe", 2): dict(params=2.4e-6, tables=1.5e-7, launch=2.8e-7),
    ("zernike_fringe", 1): dict(params=7.0e-7, tables=3.2e-7, launch=1.2e-6),
    ("zernike_fringe", 0): dict(params=4.4e-7, tables=8.3e-8, launch=8.1e-7),
    ("tilted_fold", 2): dict(params=9.4e-5, launch=1.2e-4),
    ("tilted_fold", 1): dict(params=2.2e-5, launch=4.2e-5),
    ("tilted_fold", 0): dict(params=1.5e-4, launch=1.2e-4),
    ("litho_telecentric", 0): dict(params=6.3e-7, launch=1.1e-6),
}
# test_persistent_loop_visits_every_tile in fp32, same card: the whole bundle against the sum of its chunks, per mode
# (ACC 0 sums each warp's fp32 values in fp64 at once and came out equal; the floor of 1e-13 leaves room for the order
# of the fp64 atomics).  fp64 achieves <= 4e-15 against the 1e-11 asserted (six runs).
FP32_CHUNKS_ACHIEVED = {2: 5.9e-8, 1: 5.6e-8, 0: 0.0}


@pytest.fixture(scope="module")
def report_instantiations():
    yield
    print("\nprofiled trace_bwd_kernel instantiations (%d):" % len(PROFILED),
          ", ".join("<%s, %d, %s>" % (t, a, str(p).lower()) for t, a, p in sorted(PROFILED)))


def _device_table(table):
    from optiland_b200.trace import DeviceTable

    return DeviceTable(table, "cuda:0")


def _expect(dtab, table, dtype, mode, name):
    """The device table's own prediction agrees with the host preparation's and with the case.  Every GPU test below
    runs one of the (table, dtype) pairs of CASES, whose launches test_launch_takes_the_predicted_instantiation
    profiles."""
    pred = adjoint_mode(dtab.c, dtype)
    assert pred == adjoint_mode(host_table_fields(table), dtype)
    assert pred == (mode, name in POLY_BASES), (name, dtype, mode, pred)
    return ("double" if _is64(dtype) else "float", mode, pred[1])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_launch_takes_the_predicted_instantiation(case, report_instantiations):
    """The instantiation depends on the table and the precision only: one profiled launch per case, over the 4099-ray
    bundle (17 CTAs), must be trace_bwd_kernel<T, ACC, POLY> as adjoint_mode predicts it from the device table."""
    name, dtype, mode = case
    table = system(name, dtype, mode)
    dtab = _device_table(table)
    want = _expect(dtab, table, dtype, mode, name)
    ins, buf = device_forward(dtab, bundle(name, 4099, seed=10 + 4099), dtype)
    grec = random_weights(buf, seed=4099)
    assert profiled_backward(lambda: device_backward(dtab, dtype, ins, buf, grec)) == want


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4099])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_each_instantiation_matches_the_host_instantiation(case, n):
    """One live lane, a full warp and one lane, and many CTAs with a ragged last tile: parameter, table (POLY) and
    launch-state gradients of a random linear functional of all 8 records on every row, kernel against the host
    instantiation in the same precision fed the kernel's own records (so the per-ray inputs are identical and only
    the accumulation differs).  fp64: 1e-10 x max |g_host|; fp32: 3x what the H100 achieves (FP32_ACHIEVED).
    test_launch_takes_the_predicted_instantiation checks that the launch is the instantiation named in the id."""
    from oracle.hostcheck_api import load, run_backward

    name, dtype, mode = case
    table = system(name, dtype, mode)
    dtab = _device_table(table)
    poly = _expect(dtab, table, dtype, mode, name)[2]
    rays = bundle(name, n, seed=10 + n)
    ins, buf = device_forward(dtab, rays, dtype)
    grec = random_weights(buf, seed=n)
    gin, gpar, gtab = device_backward(dtab, dtype, ins, buf, grec)
    npd = _np_dtype(dtype)
    hin = {k: ins[j].cpu().numpy() for j, k in enumerate(GIN_KEYS[:7])}
    hin["w"] = rays["w"].astype(npd)
    krec = {k: buf[j, :, :n].cpu().numpy() for j, k in enumerate(REC)}
    hw = {k: grec[j, :, :n].cpu().numpy() for j, k in enumerate(REC)}
    host = run_backward(load(), table, hin, krec, hw, dtype=npd, tables=poly)
    hgin, hpar = host[0], host[1]
    assert np.all(np.isfinite(gpar.cpu().numpy())) and np.all(np.isfinite(hpar))
    errs ={"params": _rel(gpar.cpu().numpy(), hpar, _scale(hpar))}
    if poly:
        errs["tables"] = _rel(gtab.cpu().numpy(), host[2], _scale(host[2]))
        assert np.abs(host[2]).max() > 0
    lscale = max(_scale(hgin[k]) for k in GIN_KEYS)
    errs["launch"] = max(_rel(gin[j].double().cpu().numpy(), hgin[k], lscale) for j, k in enumerate(GIN_KEYS))
    assert np.abs(hpar).max() > 0
    print(f"[adjoint {name} {dtype} acc{mode} n={n}]", {k: f"{v:.3g}" for k, v in errs.items()})
    for k, e in errs.items():
        tol = 1e-10 if _is64(dtype) else 3 * FP32_ACHIEVED[name, mode][k]
        assert e <= tol, (k, e, tol)


def _base_view(name, k, gpar, gtab, s0):
    """Gradients of the base surfaces out of a system padded with ``k`` planes, without the index slots of the medium
    the planes split (its share moves to the planes)."""
    nb = base_system(name)[0].num_surfaces
    idx = [b if b < s0 else b + k for b in range(nb)]
    p = gpar[idx].copy()
    p[s0, _lib.GP_N1] = 0
    if s0 > 0:
        p[s0 - 1, _lib.GP_N2] = 0
    return p, (gtab[idx] if gtab is not None else None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", BASES)
def test_every_mode_gives_the_same_gradient(name):
    """The same base, padded to land in ACC 2, 1 and 0 in fp64: the base surfaces' parameter gradients, table
    gradients and launch-state gradients of a loss on the image row and the second real surface's row agree across the
    three modes to 1e-10 x max |g|.  (GPU against GPU: test_each_instantiation_matches_the_host_instantiation holds the
    per-surface arithmetic to the host.)"""
    base, _, s0 = base_system(name)
    rays = bundle(name, 4099, seed=MODE_COMPARISON_SEED)
    # the same weights in every mode, on the rows of the same two physical surfaces
    base_w = random_weights(device_forward(_device_table(base), rays, "float64")[1], seed=7,
                            rows=(s0 + 1, base.num_surfaces - 1))
    got = {}
    modes = modes_of(name, "float64")
    for mode in modes:
        k = planes_for(name, "float64", mode)
        table = padded(name, k)
        dtab = _device_table(table)
        _expect(dtab, table, "float64", mode, name)
        ins, buf = device_forward(dtab, rays, "float64")
        S = table.num_surfaces
        grec = torch.zeros_like(buf)
        grec[:, s0 + 1 + k] = base_w[:, s0 + 1]
        grec[:, S - 1] = base_w[:, -1]
        grec = torch.where(torch.isfinite(buf), grec, torch.zeros((), dtype=buf.dtype, device=buf.device))
        gin, gpar, gtab = device_backward(dtab, "float64", ins, buf, grec)
        p, t = _base_view(name, k, gpar.cpu().numpy(), gtab.cpu().numpy() if gtab is not None else None, s0)
        got[mode] = (p, t, np.stack([g.cpu().numpy() for g in gin]))
    p2, t2, l2 = got[modes[0]]
    assert np.abs(p2).max() > 0
    for mode in modes[1:]:
        p, t, l = got[mode]
        assert _rel(p, p2, _scale(p2)) <= 1e-10, mode
        if t2 is not None:
            assert np.abs(t2).max() > 0
            assert _rel(t, t2, _scale(t2)) <= 1e-10, mode
        assert _rel(l, l2, _scale(l2)) <= 1e-10, mode


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", MODES)
def test_persistent_loop_visits_every_tile(mode, dtype):
    """600 013 rays: the backward grid is one resident wave, so every CTA walks several tiles.  The gradient over the
    whole bundle equals the sum of the gradients over chunks of at most 32 768 rays (128 tiles: at most one per CTA),
    fp64 to 1e-11 relative, fp32 to 3x what the H100 achieves (FP32_CHUNKS_ACHIEVED); launch-state gradients are per
    ray and equal exactly."""
    name = "cooke_c1"
    table = system(name, dtype, mode)
    dtab = _device_table(table)
    _expect(dtab, table, dtype, mode, name)
    n, chunk = 600_013, 32_768
    ins, buf = device_forward(dtab, bundle(name, n, seed=3), dtype)
    grec = random_weights(buf, seed=4)
    gin, gpar, _ = device_backward(dtab, dtype, ins, buf, grec)
    total = torch.zeros_like(gpar)
    for lo in range(0, n, chunk):
        cg, cp, _ = device_backward(dtab, dtype, ins, buf, grec, lo=lo, n=min(chunk, n - lo))
        total += cp
        for j in range(8):
            a, b = gin[j][lo:lo + cg[j].numel()], cg[j]
            assert torch.equal(torch.isnan(a), torch.isnan(b)) and bool(torch.all((a == b) | torch.isnan(a))), (lo, j)
    full, parts = gpar.cpu().numpy(), total.cpu().numpy()
    e = _rel(parts, full, _scale(full))
    print(f"[persistent {dtype} acc{mode}] chunks vs whole: {e:.3g}")
    assert e <= (1e-11 if _is64(dtype) else max(3 * FP32_CHUNKS_ACHIEVED[mode], 1e-13))


ABI_CASES = [("cooke_c1", "float64", 0), ("cooke_c1", "float64", 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ABI_CASES, ids=[f"{b}-{d}-acc{m}" for b, d, m in ABI_CASES])
def test_sub_range_of_surfaces(case):
    """first > 0 and last < S: the launch state is row first-1 of a whole-table forward, the records come from a
    forward over the same range (which reproduces the whole-table rows), and the gradients equal the host
    instantiation's over that range."""
    from oracle.hostcheck_api import load, run_backward

    name, dtype, mode = case
    table = system(name, dtype, mode)
    dtab = _device_table(table)
    _expect(dtab, table, dtype, mode, name)
    S, n = table.num_surfaces, 4099
    first, last = S // 3, S - 2
    rays = bundle(name, n, seed=6)
    _, full = device_forward(dtab, rays, dtype)
    rin = {k: full[j, first - 1, :n].cpu().numpy() for j, k in enumerate(RAY_KEYS[:7])}
    rin["w"], rin["opd"] = rays["w"], full[7, first - 1, :n].cpu().numpy()
    ins, buf = device_forward(dtab, rin, dtype, first, last)
    assert _rel(_np(buf, n), _np(full[:, first:last], n), 1.0) <= 1e-12 * Case(name).scale
    grec = random_weights(buf, seed=8)
    gin, gpar, _ = device_backward(dtab, dtype, ins, buf, grec, first=first, last=last)
    hin = {k: ins[j].cpu().numpy() for j, k in enumerate(GIN_KEYS[:7])}
    hin["w"] = rays["w"]
    hgin, hpar = run_backward(load(), table, hin, {k: _np(buf[j], n) for j, k in enumerate(REC)},
                              {k: _np(grec[j], n) for j, k in enumerate(REC)}, first=first, last=last)
    assert np.any(hpar[first:last]) and not np.any(gpar.cpu().numpy()[:first])
    assert _rel(gpar.cpu().numpy(), hpar, _scale(hpar)) <= 1e-10
    lscale = max(_scale(hgin[k]) for k in GIN_KEYS)
    for j, k in enumerate(GIN_KEYS):
        assert _rel(gin[j].cpu().numpy(), hgin[k], lscale) <= 1e-10, k


@pytest.mark.gpu
@pytest.mark.parametrize("n", [32, 4099])
@pytest.mark.parametrize("case", ABI_CASES, ids=[f"{b}-{d}-acc{m}" for b, d, m in ABI_CASES])
def test_row_mask_null_entries_and_no_launch_gradient(case, n):
    """Inputs the differentiable trace never passes.  A clear grad_row_mask bit hides a row that holds non-zero data
    (same result as zeroing it); a NULL grad_rec entry acts as zeros; grad_rays_in == NULL leaves the parameter
    gradients unchanged.  With one warp of rays (n = 32) the sums are formed in a fixed order and the results must be
    bit-identical; with many CTAs the fp64 atomics land in any order: 1e-13 x max |g|."""
    name, dtype, mode = case
    table = system(name, dtype, mode)
    dtab = _device_table(table)
    _expect(dtab, table, dtype, mode, name)
    S = table.num_surfaces
    ins, buf = device_forward(dtab, bundle(name, n, seed=9), dtype)
    grec = random_weights(buf, seed=11)
    tol = 0.0 if n <= 32 else 1e-13

    def same(a, b):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        assert np.abs(b).max() > 0
        if tol == 0.0:
            assert np.array_equal(a, b, equal_nan=True)
        else:
            assert _rel(a, b, _scale(b)) <= tol

    hidden = (1, S // 2, S - 2)
    mask = (1 << 64) - 1
    for r in hidden:
        mask &= ~(1 << r)
    assert bool(torch.any(grec[:, list(hidden)] != 0))
    zeroed = grec.clone()
    zeroed[:, list(hidden)] = 0
    g_mask, p_mask, _ = device_backward(dtab, dtype, ins, buf, grec, mask=mask)
    g_zero, p_zero, _ = device_backward(dtab, dtype, ins, buf, zeroed)
    same(p_mask, p_zero)
    for a, b in zip(g_mask, g_zero):
        assert torch.equal(torch.isnan(a), torch.isnan(b)) and bool(torch.all((a == b) | torch.isnan(a)))
    # NULL entries act as zeros: intensity and opd gradients absent
    z2 = grec.clone()
    z2[6:8] = 0
    _, p_null, _ = device_backward(dtab, dtype, ins, buf, grec, null=(6, 7))
    _, p_z2, _ = device_backward(dtab, dtype, ins, buf, z2)
    same(p_null, p_z2)
    # no launch-state gradient wanted
    _, p_with, _ = device_backward(dtab, dtype, ins, buf, grec)
    _, p_without, _ = device_backward(dtab, dtype, ins, buf, grec, want_gin=False)
    same(p_without, p_with)
