"""Polygon apertures (Optiland's ``PolygonAperture`` and ``FileAperture``) on the trace path: the aperture-program
opcode and its prepared form, the kernel arithmetic against fixtures the unmodified reference produced on its torch
backend (tests/golden/polygon_aperture, ``oracle/make_golden_polygon.py``), the plugin with live reference objects, the
adjoint, and what stays declined.  GPU tests are marked; the rest runs on the CPU through the host instantiation of the
device arithmetic with the polygon-table kernel variants (tests/hostcheck/hostcheck_polygon.cpp) and the test engine
built on it (oracle/polygon_engines.py)."""
import ctypes as C
import dataclasses
import glob
import os

import numpy as np
import pytest

from optiland_b200 import table as T
from tests._util import GOLDEN, REC, Case, fp32_errors, max_abs_err

CASES = sorted("polygon_aperture/" + os.path.splitext(os.path.basename(p))[0]
               for p in glob.glob(os.path.join(GOLDEN, "polygon_aperture", "*.npz")))
PLAIN_CASES = [c for c in CASES if "polarized" not in c]
FEAT_POLYGON = 1 << 9
# fp32 records against the reference's fp64 ones: intercepts and OPD in units of the system's scale, direction cosines
F32_POS, F32_DIR = 4e-6, 1e-5


def _pmat(c, dtype=np.complex128):
    return np.tile(np.eye(3, dtype=dtype), (c.n, 1, 1)) if "out_p" in c.z else None


def _window(program, z=0.0):
    """Object surface + a plane at ``z`` that carries ``program``."""
    return T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP),
                           T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, z], aperture=program)], [0.55])


def _rays(x, y):
    n = len(x)
    return {"x": np.asarray(x, float), "y": np.asarray(y, float), "z": np.full(n, -1.0), "L": np.zeros(n), "M": np.zeros(n),
            "N": np.ones(n), "i": np.ones(n), "w": np.full(n, 0.55)}


def _torch_rule(vx, vy, px, py):
    """The reference's torch point-in-polygon test (backend/torch_backend.py path_contains_points) in NumPy, in the
    dtype of its arguments."""
    vxn, vyn = np.roll(vx, -1), np.roll(vy, -1)
    px, py = px[:, None], py[:, None]
    with np.errstate(all="ignore"):
        cond = (vy > py) != (vyn > py)
        slope = (vxn - vx) / (vyn - vy)
        x_int = vx + slope * (py - vy)
        return np.sum(cond & (px < x_int), axis=1) % 2 == 1


def _polygons(program):
    """[(x, y)] of every polygon of an aperture program."""
    out, i = [], 0
    while i < len(program):
        op = int(program[i])
        if op == T.AP_POLYGON:
            n = int(program[i + 1])
            xy = program[i + 2:i + 2 + 2 * n].reshape(n, 2)
            out.append((xy[:, 0], xy[:, 1]))
            i += 2 + 2 * n
        else:
            i += 1 + T._AP_OPERANDS[op]
    return out


def _edge_distance(vx, vy, px, py):
    """Distance of every point to the nearest edge of the closed polygon."""
    ax, ay, bx, by = vx, vy, np.roll(vx, -1), np.roll(vy, -1)
    dx, dy = bx - ax, by - ay
    t = ((px[:, None] - ax) * dx + (py[:, None] - ay) * dy) / np.maximum(dx * dx + dy * dy, 1e-300)
    t = np.clip(t, 0.0, 1.0)
    return np.min(np.hypot(px[:, None] - (ax + t * dx), py[:, None] - (ay + t * dy)), axis=1)


# ---- ABI / table layer -----------------------------------------------------------------------------------------

def test_polygon_program_layout_round_trip_and_validation():
    """{AP_POLYGON, n, x_0, y_0, ...}; it composes with aperture_combine, survives pack / unpack, and malformed
    programs are refused by the table layer."""
    hexa = T.aperture_polygon([1, 0, -1, -1, 0, 1], [0, 1, 1, 0, -1, -1])
    assert list(hexa[:4]) == [T.AP_POLYGON, 6, 1, 0] and len(hexa) == 14
    spider = T.aperture_combine(T.AP_DIFFERENCE, T.aperture_radial(10.0, 2.0),
                                T.aperture_combine(T.AP_UNION, T.aperture_polygon([-0.1, 0.1, 0.1, -0.1], [0, 0, 11, 11]),
                                                   T.aperture_polygon([0, 11, 11, 0], [-0.1, -0.1, 0.1, 0.1])))
    T.validate_aperture_program(spider)
    assert T.polygon_vertices(spider) == 8
    tab = _window(spider)
    surf, pool = tab.pack()
    back = T.SurfaceTable.unpack(surf, pool, tab.wavelengths)
    assert np.array_equal(back.surfaces[1].aperture, spider) and back.content_key() == tab.content_key()
    for bad, word in ((T.aperture_polygon([0, 1], [0, 1]), "integer >= 3"),
                      (T.aperture_polygon([0, 1, np.nan], [0, 1, 0]), "non-finite"),
                      (hexa[:-1], "outside the program"),
                      (np.array([T.AP_POLYGON, 3.5, 0, 0, 1, 0, 0, 1]), "integer >= 3"),
                      (np.concatenate([hexa, hexa]), "malformed")):
        with pytest.raises(ValueError, match=word):
            T.validate_aperture_program(np.asarray(bad, float))


def _upload(tab, mutate=lambda s, p: None):
    """(return code of olb_table_workspace_bytes, its message, feature bits or -1) for a table whose packed arrays
    ``mutate`` edits."""
    from optiland_b200 import _lib
    from oracle.hostcheck_api import load

    surf, pool = tab.pack()
    mutate(surf, pool)
    ht = _lib.HostTable(tab, packed=(surf, pool))
    lib = _lib.load()
    rc = int(lib.olb_table_workspace_bytes(C.byref(ht.c)))
    buf = C.create_string_buffer(256)
    lib.olb_last_error(buf, 256)
    return rc, buf.value.decode(), int(load().olbhc_features(C.byref(ht.c)))


def test_vertex_cap_and_malformed_polygons_are_table_errors():
    """At most MAX_POLYGON_VERTICES vertices per table, refused by the table layer and by the upload; the upload also
    refuses fewer than 3 vertices, non-finite vertices and a truncated vertex list, each with a reason."""
    assert T.MAX_POLYGON_VERTICES == 1024
    th = np.linspace(0, 2 * np.pi, 600, endpoint=False)
    big = T.aperture_polygon(np.cos(th), np.sin(th))
    one = _window(big)
    rc, msg, feat = _upload(one)
    assert rc > 0 and feat & FEAT_POLYGON
    both = T.aperture_combine(T.AP_INTERSECT, big, big)
    with pytest.raises(ValueError, match="shared memory"):
        _window(both)
    two = object.__new__(T.SurfaceTable)          # (past the table layer's own check)
    two.surfaces = [one.surfaces[0], dataclasses.replace(one.surfaces[1], aperture=both)]
    two.wavelengths = one.wavelengths
    rc, msg, feat = _upload(two)
    assert rc == -5 and "1024" in msg and "shared memory" in msg and feat == -1

    tab = _window(T.aperture_polygon([0, 1, 0, -1], [-1, 0, 1, 0]))

    def off(s):
        return int(s["aper_off"][1])

    def two_vertices(s, p):
        p[off(s) + 1] = 2.0

    def fractional(s, p):
        p[off(s) + 1] = 3.5

    def nan_vertex(s, p):
        p[off(s) + 4] = np.nan

    def inf_vertex(s, p):
        p[off(s) + 5] = np.inf

    def truncated(s, p):
        s["aper_len"][1] -= 2

    for mutate, word in ((two_vertices, "vertex count"), (fractional, "vertex count"), (nan_vertex, "non-finite vertex"),
                         (inf_vertex, "non-finite vertex"), (truncated, "outside the program")):
        rc, msg, feat = _upload(tab, mutate)
        assert rc == -5 and word in msg and feat == -1, (mutate.__name__, rc, msg)


def test_tables_without_a_polygon_keep_their_feature_bits():
    c = Case("hubble_c4")
    assert not _upload(c.table)[2] & FEAT_POLYGON


def test_prepared_edges_hold_the_reference_slopes_and_skip_horizontal_edges():
    """Per precision: slope = (vx_next - vx) / (vy_next - vy) computed in the table's precision from the vertices
    rounded to it; horizontal edges are left out; up to 16 vertices one bucket, above that several."""
    from oracle.hostcheck_polygon import polygon_block

    from tests import _polygon_systems as PS

    x, y = PS.L_SHAPE
    for dtype in (np.float64, np.float32):
        nb, ymin, ymax, start, rec = polygon_block(_window(T.aperture_polygon(x * 1.1, y / 3.0)), 1, dtype)
        vx, vy = (x * 1.1).astype(dtype), (y / 3.0).astype(dtype)
        vxn, vyn = np.roll(vx, -1), np.roll(vy, -1)
        keep = vy != vyn
        assert nb == 1 and list(start) == [0, int(keep.sum())] and keep.sum() == 3
        assert (ymin, ymax) == (vy.min(), vy.max())
        want = np.stack([vx[keep], vy[keep], vyn[keep], ((vxn - vx)[keep] / (vyn - vy)[keep]).astype(dtype)], axis=1)
        assert np.array_equal(rec, want.astype(np.float64))
    ox, oy = PS.wavy_outline(300)
    nb, ymin, ymax, start, rec = polygon_block(_window(T.aperture_polygon(ox, oy)), 1)
    assert nb == 300 // 4 and start[0] == 0 and np.all(np.diff(start) > 0) and start[-1] == len(rec) <= 2 * 300
    # a zigzag whose every edge spans the whole height: one bucket per edge would repeat every edge in every bucket,
    # so the bucket count is halved until the records are at most twice the edges
    zx = np.arange(40.0)
    nb, _, _, start, rec = polygon_block(_window(T.aperture_polygon(np.r_[zx, 39.0, 0.0], np.r_[zx % 2, 5.0, 5.0])), 1)
    assert nb < 42 // 4 and len(rec) <= 2 * 42


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", ["outline300", "zigzag", "star", "bowtie", "collinear"])
def test_bucketed_scan_equals_the_reference_rule_point_for_point(shape, dtype):
    """Random points, points level with every vertex, on vertices and on edges: the kernel arithmetic (one bucket or
    many) classifies each exactly as the reference's crossing count over ALL edges does, in fp64 and, from the vertices
    and points rounded to fp32, in fp32."""
    from oracle.hostcheck_polygon import run_hostcheck_polygon

    from tests import _polygon_systems as PS

    rng = np.random.default_rng(len(shape))
    if shape == "outline300":
        vx, vy = PS.wavy_outline(300)
    elif shape == "zigzag":
        zx = np.arange(40.0)
        vx, vy = np.r_[zx, 39.0, 0.0], np.r_[(zx % 2) * 3.0, 5.0, 5.0]
    elif shape == "star":
        th = 2 * np.pi * np.arange(46) / 46
        r = np.where(np.arange(46) % 2, 2.0, 6.0)
        vx, vy = r * np.cos(th), r * np.sin(th)
    elif shape == "bowtie":
        vx, vy = PS.BOW_TIE
    else:      # collinear runs, horizontal edges and a repeated vertex
        vx = np.array([-3, -1, 0, 2, 3, 3, 3, 1, 1, 0, -3, -3, -3.0])
        vy = np.array([-2, -2, -2, -2, -2, 0, 2, 2, 2, 2, 2, 0, 0.0])
    vx, vy = vx.astype(dtype), vy.astype(dtype)
    lo, hi = min(vx.min(), vy.min()) - 1, max(vx.max(), vy.max()) + 1
    n = 4000
    px = np.r_[rng.uniform(lo, hi, n), rng.uniform(lo, hi, n), vx, (vx + np.roll(vx, -1)) / 2, [np.nan, 0.0]]
    py = np.r_[rng.uniform(lo, hi, n), rng.choice(vy, n), vy, (vy + np.roll(vy, -1)) / 2, [0.0, np.nan]]
    px, py = px.astype(dtype), py.astype(dtype)
    out, _, _ = run_hostcheck_polygon(_window(T.aperture_polygon(vx, vy)), _rays(px, py), dtype)
    want = _torch_rule(vx, vy, px, py)
    assert 0.05 < want.mean() < 0.95
    assert np.array_equal(out["i"] != 0, want)


def test_adjoint_and_batched_uploads_cover_polygon_tables():
    """A polygon table is inside the adjoint's scope (its general variant holds the scan).  Batched uploads pass the
    template's aperture program through unchanged -- the polygon is not a batched parameter -- so every system's blob
    holds the same prepared polygon."""
    from optiland_b200 import _lib
    from optiland_b200.batch import template_params
    from oracle.hostcheck_api import load

    c = Case("polygon_aperture/polygon_cassegrain_spider")
    ht = _lib.HostTable(c.table)
    hc = load()
    assert hc.olbhc_bwd_level(C.byref(ht.c)) == 2
    params = np.stack([template_params(c.table)] * 2)
    params[1, 2, _lib.BP_TX + 2] += 0.01
    err = C.create_string_buffer(256)
    feat = C.c_uint(0)
    blobs = []
    for b in range(2):
        out = np.zeros(1 << 16, dtype=np.uint8)
        n = hc.olbhc_batch_blob(C.byref(ht.c), C.c_void_p(params.ctypes.data), 2, b, 0, C.c_void_p(out.ctypes.data),
                                out.size, C.byref(feat), err, 256)
        assert n > 0 and feat.value & FEAT_POLYGON, err.value
        blobs.append(out[:n].copy())
    single = np.zeros(1 << 16, dtype=np.uint8)
    n1 = hc.olbhc_single_blob(C.byref(ht.c), 0, C.c_void_p(single.ctypes.data), single.size, C.byref(feat), err, 256)
    assert n1 == len(blobs[0]) and np.array_equal(single[:n1], blobs[0]) and not np.array_equal(blobs[0], blobs[1])


# ---- kernel arithmetic (host instantiation) vs the reference's fixtures ----------------------------------------

def _check_fp64(c, rec, out=None):
    tol = 1e-11 * c.scale
    for k in REC:
        assert max_abs_err(rec[k], c.rec[k]) <= tol, k      # (max_abs_err also asserts the same NaN pattern)
    assert np.array_equal(rec["intensity"] == 0, c.rec["intensity"] == 0)


def _local_hits(c, s):
    """Reference fp64 hit points on surface ``s`` in its local frame."""
    spec = c.table.surfaces[s]
    p = np.stack([c.rec[k][s] for k in ("x", "y", "z")]) - spec.t[:, None]
    q = spec.R.T @ p
    return q[0], q[1]


def _check_fp32(c, rec):
    """Records at the fp32 tolerance; the clip mask may differ from the reference's only for rays whose fp64 hit point
    lies within the fp32 position error (F32_POS x the system's scale) of a polygon edge."""
    flipped = np.zeros(c.n, bool)
    for s, spec in enumerate(c.table.surfaces):
        differs = (rec["intensity"][s] == 0) != (c.rec["intensity"][s] == 0)
        new = differs & ~flipped
        if new.any():
            assert spec.aperture is not None, s
            x, y = _local_hits(c, s)
            d = np.min([_edge_distance(vx, vy, x[new], y[new]) for vx, vy in _polygons(spec.aperture)], axis=0)
            assert np.all(d <= F32_POS * c.scale), (s, float(d.max()))
        flipped |= differs
    assert flipped.mean() <= 0.02
    keep = {k: np.where(flipped, np.nan, rec[k]) for k in REC}
    want = {k: np.where(flipped, np.nan, c.rec[k]) for k in REC}
    got = fp32_errors(keep, want)
    assert got["pos"] <= F32_POS * c.scale and got["opd"] <= F32_POS * c.scale, got
    assert got["dir"] <= F32_DIR and got["intensity"] <= F32_DIR, got


@pytest.mark.parametrize("name", CASES)
def test_host_arithmetic_fp64_matches_reference_fixture(name):
    """The intensity mask equals the reference's ray for ray, the records to 1e-11 x the system's scale."""
    from oracle.hostcheck_polygon import run_hostcheck_polygon

    c = Case(name)
    out, rec, status = run_hostcheck_polygon(c.table, c.rays, np.float64, pmat=_pmat(c), want_l0=True)
    assert status == 0
    _check_fp64(c, rec, out)
    for k in ("x", "y", "z", "L", "M", "N", "i", "opd", "L0", "M0", "N0"):
        assert max_abs_err(out[k], c.out[k]) <= 1e-11 * c.scale, k


# fp32 records are not compared where fp32 cannot resolve the question: rays placed exactly on edges (edge_window), and
# rays grazing the steep front surface of nan_rays, whose intercepts are ill-conditioned
F32_CASES = [n for n in CASES if "edge_window" not in n and "nan_rays" not in n]


@pytest.mark.parametrize("name", F32_CASES)
def test_host_arithmetic_fp32(name):
    from oracle.hostcheck_polygon import run_hostcheck_polygon

    c = Case(name)
    _, rec, _ = run_hostcheck_polygon(c.table, c.rays, np.float32, pmat=_pmat(c, np.complex64))
    _check_fp32(c, rec)


def test_fixtures_pin_the_reference_behaviours():
    """Rays on vertices, level with vertices, on vertical / horizontal / slanted edges and NaN rays are in the fixtures;
    every fixture clips some rays and passes others; the scaled polygon clips at the scaled size."""
    from tests import _polygon_systems as PS

    c = Case("polygon_aperture/polygon_edge_window")
    x, y = c.rays["x"], c.rays["y"]
    lx, ly = PS.L_SHAPE
    inside = c.rec["intensity"][1] != 0
    assert np.array_equal(inside, _torch_rule(lx, ly, x, y))
    nan = np.isnan(x) | np.isnan(y)
    assert nan.sum() == 3 and not inside[nan].any()
    on_vertex_level = np.isin(y, ly) & ~nan
    assert on_vertex_level.sum() > 40 and inside[on_vertex_level].any() and not inside[on_vertex_level].all()
    assert not inside[(y == 4.0)].any() and inside[(y == -4.0) & (x > -4) & (x < 4)].all()      # half-open in y
    assert not inside[(x == 4.0) & (y > -4) & (y < 0)].any() and inside[(x == -4.0) & (y > -4) & (y < 4)].all()
    for name in CASES:
        i = Case(name).rec["intensity"][-1]
        assert (i == 0).any() and (i != 0).any(), name
    s = Case("polygon_aperture/polygon_scaled")
    vx, vy = _polygons(s.table.surfaces[1].aperture)[0]
    assert np.allclose(np.hypot(vx, vy), 4.5)
    f = Case("polygon_aperture/polygon_file_outline")
    assert len(_polygons(f.table.surfaces[1].aperture)[0][0]) == 240
    n = Case("polygon_aperture/polygon_nan_rays")
    bad = np.isnan(n.rec["x"][2])
    assert bad.any() and not bad.all() and np.all(n.rec["intensity"][2][bad] == 0)


def test_adjoint_matches_finite_differences():
    """The adjoint of the spider Cassegrain (the general variant of surface_backward, on the CPU) against central
    differences of the forward arithmetic for a random linear functional of the records.  The mask is a constant of the
    adjoint, and no ray changes side under these steps."""
    from oracle.hostcheck_api import load, run_backward
    from oracle.hostcheck_polygon import run_hostcheck_polygon

    c = Case("polygon_aperture/polygon_cassegrain_spider")
    table, rays = c.table, {k: v[:150].copy() for k, v in c.rays.items()}
    S, n = table.num_surfaces, 150
    rng = np.random.default_rng(7)
    w = {k: rng.normal(size=(S, n)) for k in REC}

    def loss(tab, r):
        _, rec, _ = run_hostcheck_polygon(tab, r, np.float64)
        return sum(float(np.sum(w[k] * rec[k])) for k in REC)

    _, rec, _ = run_hostcheck_polygon(table, rays, np.float64)
    assert (rec["intensity"][1] == 0).any()
    gin, gpar, _ = run_backward(load(), table, rays, rec, w, tables=True)
    h = 1e-7
    for k in ("x", "y", "L", "i"):
        d = rng.normal(size=n)
        fd = (loss(table, {**rays, k: rays[k] + h * d}) - loss(table, {**rays, k: rays[k] - h * d})) / (2 * h)
        assert fd == pytest.approx(float(np.sum(gin[k] * d)), rel=2e-6, abs=1e-6), k
    for s in (1, 2):
        for q in range(3):
            def with_t(delta, s=s, q=q):
                t = table.surfaces[s].t.copy()
                t[q] += delta
                return loss(table.replace_surface(s, t=t), rays)

            fd = (with_t(h) - with_t(-h)) / (2 * h)
            assert fd == pytest.approx(gpar[s, q], rel=2e-6, abs=1e-6), (s, q)


# ---- live reference objects through the plugin -----------------------------------------------------------------

pytest_ref = pytest.importorskip("oracle.ref_import")
needs_ref = pytest.mark.skipif(not pytest_ref.reference_available(), reason="reference not present on this box")

LIVE_REC = ("x", "y", "z", "L", "M", "N", "opd", "intensity")


@pytest.fixture(params=["devmath", pytest.param("cuda", marks=pytest.mark.gpu)])
def live(request):
    """The reference on its torch backend in fp64 (the backend whose polygon rule the kernel follows), on the CPU for
    the device-math engine and on the GPU for the CUDA engine."""
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin as P

    if request.param == "cuda":
        eng = P.CudaEngine()
    else:
        from oracle.polygon_engines import PolygonDeviceMathEngine

        eng = PolygonDeviceMathEngine()
    be.set_backend("torch")
    be.set_precision("float64")
    be.grad_mode.disable()
    be.set_device("cuda" if request.param == "cuda" else "cpu")
    yield P, eng, be, request.param
    if P._state.get("installed"):
        P.uninstall()
    be.set_backend("torch")
    be.set_precision("float64")
    be.grad_mode.disable()
    be.set_device("cpu")
    be.set_backend("numpy")


def _close(got, want, scale, what):
    assert got.shape == want.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern")
    m = np.isfinite(want)
    assert not m.any() or np.max(np.abs(got[m] - want[m])) <= 1e-11 * scale, (what, float(np.max(np.abs(got[m] - want[m]))))


def _both(P, eng, run):
    """``run()`` on the stock reference, then with the plugin installed over ``eng``."""
    if P._state.get("installed"):
        P.uninstall()
    want = run()
    P.install(engine=eng)
    P.stats(reset=True)
    return want, run()


@needs_ref
@pytest.mark.parametrize("system", ["polygon_hexagon_mirror", "polygon_cassegrain_spider", "polygon_concave_bowtie",
                                    "polygon_nested_tilted", "polygon_asphere_grid", "polygon_file_outline",
                                    "polygon_scaled"])
def test_optic_trace_through_the_plugin_equals_the_reference(live, system):
    """Optic.trace of two fields x every wavelength: each record row and the clip mask equal the stock torch reference,
    one fused launch per trace, no decline (the parent declined with "aperture type PolygonAperture")."""
    from tests import _polygon_systems as PS

    P, eng, be, which = live

    def run():
        lens = PS.BUILDERS[system](be)
        out = []
        for hy in (0.0, 1.0):
            for w in lens.wavelengths.wavelengths:
                r = lens.trace(0.0, hy, float(w.value), 12, "hexapolar")
                out.append(({k: be.to_numpy(getattr(lens.surfaces, k)).astype(np.float64) for k in LIVE_REC},
                            be.to_numpy(r.i).astype(np.float64)))
        return out

    n0 = len(eng.calls)
    want, got = _both(P, eng, run)
    for (w, wi), (g, gi) in zip(want, got):
        scale = max(1.0, float(np.nanmax(np.abs(w["z"]))))
        for k in LIVE_REC:
            _close(g[k], w[k], scale, k)
        assert np.array_equal(g["intensity"] == 0, w["intensity"] == 0)
        _close(gi, wi, 1.0, "i")
    assert not P.stats(), P.stats()
    assert sum(1 for c in eng.calls[n0:] if c and c[0] == "pupil") == len(want), eng.calls[n0:]


@needs_ref
def test_spot_diagram_wavefront_and_trace_generic_run_on_the_kernel(live):
    """trace_generic with per-ray fields, SpotDiagram (the fused launch and spot-moment epilogue) and Wavefront (the
    wavefront epilogue) on the spider Cassegrain equal the stock reference with ``plugin.stats()`` empty."""
    from optiland.analysis import SpotDiagram
    from optiland.wavefront import Wavefront

    from tests import _polygon_systems as PS

    P, eng, be, which = live
    rng = np.random.default_rng(3)
    n = 400
    Hy, Px, Py = rng.uniform(0, 1, n), rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)

    def run():
        lens = PS.cassegrain(be)
        out = {}
        r = lens.trace_generic(be.zeros(n), be.array(Hy), be.array(Px), be.array(Py), 0.55)
        for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
            out["g_" + k] = be.to_numpy(getattr(r, k)).astype(np.float64)
        out["rms"] = np.array([[float(be.to_numpy(v)) for v in row] for row in SpotDiagram(lens).rms_spot_radius()])
        wf = Wavefront(lens, fields=[(0.0, 1.0)], wavelengths=[0.55], num_rays=10, distribution="hexapolar")
        d = wf.get_data((0.0, 1.0), 0.55)
        out["wf_opd"], out["wf_i"] = be.to_numpy(d.opd).astype(np.float64), be.to_numpy(d.intensity).astype(np.float64)
        return out

    want, got = _both(P, eng, run)
    assert (want["g_i"] == 0).any() and (want["wf_i"] == 0).any()
    for k, v in want.items():
        rel = k in ("rms", "wf_opd")
        np.testing.assert_allclose(got[k], v, rtol=1e-8 if rel else 0, atol=1e-8 if rel else 1e-9, err_msg=k)
    assert not P.stats(), P.stats()


@needs_ref
@pytest.mark.gpu
def test_incoherent_irradiance_runs_on_the_kernel():
    """IncoherentIrradiance of the spider Cassegrain on a CUDA torch backend: trace and binning kernels both run, nothing
    declines, and the map equals the stock reference's up to rays within rounding of a pixel edge."""
    import torch

    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be
    from optiland import physical_apertures as pa
    from optiland.analysis import IncoherentIrradiance

    from optiland_b200 import plugin as P
    from tests import _polygon_systems as PS

    be.set_backend("torch")
    be.set_device("cuda")
    be.set_precision("float64")
    be.grad_mode.disable()
    try:
        def run():
            lens = PS.cassegrain(be)
            lens.surfaces[-1].aperture = pa.RectangularAperture(x_min=-0.5, x_max=0.5, y_min=-0.5, y_max=0.5)
            torch.manual_seed(0)
            return IncoherentIrradiance(lens, num_rays=100_000, res=(32, 32), distribution="random").data[0][0]

        want = run()
        eng = P.CudaEngine()
        P.install(engine=eng)
        P.stats(reset=True)
        got = run()
        assert not P.stats(), P.stats()
        assert any(c[0] == "irradiance" for c in eng.calls)
        g, w = got[0].double().cpu().numpy(), want[0].double().cpu().numpy()
        assert w.sum() > 0 and float(np.abs(g - w).sum()) <= 1e-6 * float(np.abs(w).sum()) + 1e-9
    finally:
        if P._state.get("installed"):
            P.uninstall()
        be.set_device("cpu")
        be.set_backend("numpy")


@needs_ref
def test_what_declines(live):
    """A subclass of PolygonAperture (it may override contains), more vertices than the cap, and non-finite vertices
    decline with a reason; so does a polygon whose vertices an optimiser drives while gradients are wanted."""
    import torch
    from optiland import physical_apertures as pa

    from optiland_b200.pack import UnsupportedSurface, pack_surface_group
    from tests import _polygon_systems as PS

    P, eng, be, which = live
    lens = PS.clockwise(be)
    tab = pack_surface_group(lens.surfaces, [0.55])
    assert int(tab.surfaces[1].aperture[0]) == T.AP_POLYGON and T.polygon_vertices(tab.surfaces[1].aperture) == 5
    ap = lens.surfaces.surfaces[1].aperture
    ap.__class__ = type("MyPolygon", (type(ap),), {})
    with pytest.raises(UnsupportedSurface, match="aperture type MyPolygon"):
        pack_surface_group(lens.surfaces, [0.55])
    lens = PS.clockwise(be)
    lens.surfaces.surfaces[1].aperture = pa.PolygonAperture(*PS.wavy_outline(1100))
    with pytest.raises(UnsupportedSurface, match="1024"):
        pack_surface_group(lens.surfaces, [0.55])
    half = pa.PolygonAperture(*PS.wavy_outline(600))
    lens.surfaces.surfaces[1].aperture = pa.UnionAperture(half, pa.PolygonAperture(*PS.wavy_outline(600, 5.0)))
    with pytest.raises(UnsupportedSurface, match="1200 vertices in all"):
        pack_surface_group(lens.surfaces, [0.55])
    bad = pa.PolygonAperture([0.0, 1.0, float("nan")], [0.0, 1.0, 0.0])
    lens.surfaces.surfaces[1].aperture = bad
    with pytest.raises(UnsupportedSurface, match="non-finite"):
        pack_surface_group(lens.surfaces, [0.55])
    # gradients wanted with respect to a vertex: the reference's eager graph
    P.install(engine=eng)
    P.stats(reset=True)
    be.grad_mode.enable()
    try:
        lens = PS.clockwise(be)
        ap = lens.surfaces.surfaces[1].aperture
        ap.vertices = torch.nn.Parameter(ap.vertices.detach().clone())
        n0 = len(eng.calls)
        lens.trace(0.0, 1.0, 0.55, 6, "hexapolar")
        assert "gradients wanted" in " ".join(P.stats()), P.stats()
        assert not any(c and c[0] == "grad" for c in eng.calls[n0:])
    finally:
        be.grad_mode.disable()


def _grad_lens(be):
    from tests import _polygon_systems as PS

    return PS.cassegrain(be)


@needs_ref
def test_autograd_through_a_polygon_stopped_system_matches_the_reference(live):
    """be.grad_mode on: d(RMS spot + OPD)/d(radius, conic, thickness, decenter) of the spider Cassegrain through the plugin
    (forward kernel + adjoint, the mask a constant) against the reference's own eager autograd, to 1e-7 relative."""
    import torch

    P, eng, be, which = live
    P.install(engine=eng)
    P.stats(reset=True)

    def run():
        lens = _grad_lens(be)
        S = lens.surfaces.surfaces
        params = {}
        for name, obj, attr in (("radius1", S[1].geometry, "radius"), ("conic1", S[1].geometry, "k"),
                                ("radius2", S[2].geometry, "radius"), ("tz2", S[2].geometry.cs, "z"),
                                ("dy2", S[2].geometry.cs, "y"), ("tz3", S[3].geometry.cs, "z")):
            params[name] = torch.tensor(float(getattr(obj, attr)), dtype=torch.float64, requires_grad=True,
                                        device=be.get_device())
            setattr(obj, attr, params[name])
        lens.trace(0.0, 1.0, 0.55, 8, "hexapolar")
        x, y, i = lens.surfaces.x[-1, :], lens.surfaces.y[-1, :], lens.surfaces.intensity[-1, :]
        assert bool((i == 0).any())
        wgt = i / i.sum()
        cx, cy = (wgt * x).sum(), (wgt * y).sum()
        loss = torch.sqrt((wgt * ((x - cx) ** 2 + (y - cy) ** 2)).sum()) + 1e-3 * (wgt * lens.surfaces.opd[-1, :]).sum()
        loss.backward()
        return float(loss.detach()), {k: float(v.grad) for k, v in params.items()}

    be.grad_mode.enable()
    try:
        n0 = len(eng.calls)
        got_loss, got = run()
        assert any(c[0] == "grad" for c in eng.calls[n0:]) and not P.stats(), (eng.calls[n0:], P.stats())
        P.uninstall()
        ref_loss, ref = run()
    finally:
        be.grad_mode.disable()
    assert got_loss == pytest.approx(ref_loss, rel=1e-9)
    scale = max(abs(v) for v in ref.values())
    for k in ref:
        assert got[k] == pytest.approx(ref[k], rel=1e-7, abs=1e-9 * scale), (k, got[k], ref[k])


@needs_ref
@pytest.mark.parametrize("block", range(2))
def test_seeded_fuzz_of_random_polygons_and_substrates(block):
    """Random polygons (convex, star-shaped, with collinear runs and horizontal edges, either orientation, alone or in
    a difference tree) x random substrates (conic lens, mirror, asphere, tilted) through the device math equal the stock
    torch reference: 2 blocks x 20 seeds."""
    from oracle.polygon_engines import PolygonDeviceMathEngine
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be
    from optiland import optic as _optic
    from optiland import physical_apertures as pa

    from optiland_b200 import plugin as P

    def polygon(rng):
        kind = rng.integers(0, 4)
        n = int(rng.integers(3, 40))
        th = np.sort(rng.uniform(0, 2 * np.pi, n))
        if kind == 0:                                  # convex
            x, y = 5 * np.cos(th), 4 * np.sin(th)
        elif kind == 1:                                # star-shaped, concave
            r = rng.uniform(2.0, 6.0, n)
            x, y = r * np.cos(th), r * np.sin(th)
        elif kind == 2:                                # staircase on a grid: horizontal edges and collinear runs
            m = int(rng.integers(2, 6))
            k = np.arange(m + 1)
            x = np.r_[np.repeat(k, 2)[1:-1], m, 0.0] * 1.5 - 3.017     # (no vertex level through the chief ray's (0, 0))
            y = np.r_[np.repeat(k, 2)[:-2], m, m] * 1.0 - 2.013
            x = np.r_[x[:1], (x[0] + x[1]) / 2, x[1:]]
            y = np.r_[y[:1], (y[0] + y[1]) / 2, y[1:]]
        else:                                          # self-intersecting
            x, y = rng.uniform(-5, 5, n), rng.uniform(-5, 5, n)
        if rng.random() < 0.5:
            x, y = x[::-1], y[::-1]
        return pa.PolygonAperture(list(map(float, x)), list(map(float, y)))

    def build(seed):
        rng = np.random.default_rng(seed)
        lens = _optic.Optic()
        lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
        ap = polygon(rng)
        if rng.random() < 0.4:
            ap = pa.DifferenceAperture(pa.RadialAperture(r_max=float(rng.uniform(4, 7))), polygon(rng))
        sub = rng.integers(0, 4)
        kw = dict(rx=float(rng.uniform(-0.04, 0.04))) if rng.random() < 0.4 else {}
        if sub == 0:
            lens.surfaces.add(index=1, radius=float(rng.uniform(30, 90)), conic=float(rng.uniform(-1.5, 0.5)), thickness=5.0,
                              material="N-BK7", is_stop=True, aperture=ap, **kw)
            lens.surfaces.add(index=2, radius=-60.0, thickness=40.0)
        elif sub == 1:
            lens.surfaces.add(index=1, radius=-float(rng.uniform(80, 200)), thickness=-40.0, material="mirror", is_stop=True,
                              aperture=ap, **kw)
            lens.surfaces.add(index=2, radius=be.inf, thickness=0.0)
        elif sub == 2:
            lens.surfaces.add(index=1, radius=50.0, conic=-0.3, thickness=5.0, material="N-SF5", is_stop=True,
                              surface_type="even_asphere", coefficients=[float(rng.uniform(-1e-5, 1e-5))], aperture=ap, **kw)
            lens.surfaces.add(index=2, radius=-90.0, thickness=40.0)
        else:
            lens.surfaces.add(index=1, radius=60.0, thickness=4.0, material="N-BK7", is_stop=True)
            lens.surfaces.add(index=2, radius=be.inf, thickness=30.0, aperture=ap, **kw)
        lens.surfaces.add(index=3)
        lens.set_aperture(aperture_type="EPD", value=11.0)
        lens.fields.set_type(field_type="angle")
        lens.fields.add(y=0.0)
        lens.fields.add(y=3.0)
        lens.wavelengths.add(value=0.55, is_primary=True)
        return lens

    def run(seed):
        lens = build(seed)
        lens.trace(0.0, 1.0, 0.55, 9, "hexapolar")
        return {k: be.to_numpy(getattr(lens.surfaces, k)).astype(np.float64) for k in LIVE_REC}

    seeds = range(5000 + 20 * block, 5020 + 20 * block)
    be.set_backend("torch")
    be.set_device("cpu")
    be.set_precision("float64")
    be.grad_mode.disable()
    try:
        want = {s: run(s) for s in seeds}
        P.install(engine=PolygonDeviceMathEngine())
        P.stats(reset=True)
        clipped = 0
        for s in seeds:
            got = run(s)
            scale = max(1.0, float(np.nanmax(np.abs(want[s]["z"]))))
            for k, v in want[s].items():
                _close(got[k], v, scale, (s, k))
            assert np.array_equal(got["intensity"] == 0, v == 0), s
            clipped += int((v[-1] == 0).any() and (v[-1] != 0).any())
        assert not P.stats(), P.stats()
        assert clipped >= 12
    finally:
        if P._state.get("installed"):
            P.uninstall()
        be.set_backend("numpy")


# ---- GPU: the kernel itself ------------------------------------------------------------------------------------

def _np(t):
    return t.double().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", PLAIN_CASES)
def test_kernel_fp64_and_fp32_vs_reference_fixture(name):
    """Through the C ABI on the GPU: fp64 with the reference's mask ray for ray and records to 1e-11 x scale; fp32 with
    records at the fp32 tolerance and a mask that differs only within the fp32 position error of an edge."""
    import torch

    from optiland_b200.trace import RealRays, SurfaceGroup

    c = Case(name)
    r = c.rays
    for dtype in (torch.float64, torch.float32):
        rays = RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)
        sg = SurfaceGroup(c.table)
        sg.trace(rays)
        rec = {k: _np(getattr(sg, k)) for k in REC}
        if dtype == torch.float64:
            _check_fp64(c, rec)
            for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
                assert max_abs_err(_np(getattr(rays, k)), c.out[k]) <= 1e-11 * c.scale, k
        elif name in F32_CASES:
            _check_fp32(c, rec)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_kernel_polarized_fixture(dtype_name):
    import torch

    from optiland_b200.trace import PolarizedRays, SurfaceGroup

    dtype = getattr(torch, dtype_name)
    c = Case("polygon_aperture/polygon_polarized")
    r = c.rays
    rays = PolarizedRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)
    sg = SurfaceGroup(c.table)
    sg.trace(rays)
    rec = {k: _np(getattr(sg, k)) for k in REC}
    if dtype == torch.float64:
        _check_fp64(c, rec)
    else:
        _check_fp32(c, rec)


@pytest.mark.gpu
def test_bucketed_scan_on_the_gpu_equals_the_reference_rule():
    """One million random points and points level with vertices on a 300-vertex outline (many buckets) and on a hexagon
    (one bucket), in fp64 and fp32: the kernel's mask equals the reference's crossing count over all edges exactly."""
    import torch

    from optiland_b200.trace import RealRays, SurfaceGroup
    from tests import _polygon_systems as PS

    rng = np.random.default_rng(1)
    n = 1_000_000
    for vx, vy in (PS.wavy_outline(300), PS.regular(6, 8.0)):
        for dtype, npt in ((torch.float64, np.float64), (torch.float32, np.float32)):
            vx_, vy_ = vx.astype(npt), vy.astype(npt)
            px = rng.uniform(-11, 11, n).astype(npt)
            py = np.r_[rng.uniform(-11, 11, n // 2), rng.choice(vy_, n // 2)].astype(npt)
            r = _rays(px, py)
            rays = RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)
            SurfaceGroup(_window(T.aperture_polygon(vx_, vy_))).trace(rays)
            got = rays.i.cpu().numpy() != 0
            want = np.concatenate([_torch_rule(vx_, vy_, px[k:k + 50_000], py[k:k + 50_000]) for k in range(0, n, 50_000)])
            assert np.array_equal(got, want), (len(vx), dtype)


@pytest.mark.gpu
def test_trace_differentiable_gradients_on_the_gpu():
    """olb_trace_bwd_* (the general variant with the polygon scan) through ``trace_differentiable`` in fp64 and fp32
    against the fp64 gradients of the same adjoint on the CPU (held to finite differences above)."""
    import torch

    from oracle.hostcheck_api import load, run_backward
    from oracle.hostcheck_polygon import run_hostcheck_polygon
    from optiland_b200 import autograd as AG
    from optiland_b200.trace import RealRays

    c = Case("polygon_aperture/polygon_cassegrain_spider")
    table, rays_np = c.table, c.rays
    rng = np.random.default_rng(2)
    w = {k: rng.normal(size=(table.num_surfaces, c.n)) for k in REC}
    _, rec, _ = run_hostcheck_polygon(table, rays_np, np.float64)
    gin, gpar, _ = run_backward(load(), table, rays_np, rec, w, tables=True)
    for dtype in (torch.float64, torch.float32):
        params = AG.table_to_params(table).cuda().requires_grad_(True)
        rr = RealRays(*[rays_np[k] for k in ("x", "y", "z", "L", "M", "N", "i", "w")], dtype=dtype)
        for k in ("x", "y", "L"):
            getattr(rr, k).requires_grad_(True)
        out = AG.trace_differentiable(table, params, rr)
        mask_same = np.array_equal(_np(out["intensity"].detach()) == 0, rec["intensity"] == 0)
        assert mask_same or dtype == torch.float32
        if not mask_same:
            continue
        loss = sum((out[k].double() * torch.from_numpy(w[k]).cuda()).sum() for k in REC)
        loss.backward()
        tol = 1e-8 if dtype == torch.float64 else 2e-2
        assert np.max(np.abs(params.grad.cpu().numpy() - gpar)) <= tol * np.abs(gpar).max(), dtype
        for k in ("x", "y", "L"):
            g = getattr(rr, k).grad.double().cpu().numpy()
            assert np.max(np.abs(g - gin[k])) <= tol * max(1.0, np.abs(gin[k]).max()), (dtype, k)
