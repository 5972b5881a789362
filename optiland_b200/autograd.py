"""Differentiable trace: ``torch.autograd.Function`` over olb_trace_call_* / olb_trace_bwd_*.

The reference obtains gradients by ``loss.backward()`` through the eager graph of every
element-wise op of the trace (optiland/optimization/optimizer/torch/base.py:96-156),
reading record rows as in the ``rms_spot_size`` operand (optimization/operand/ray.py:299-342).  Here
the forward is ONE kernel launch and the backward ONE launch of the hand-derived adjoint
(``olb_math.cuh::surface_backward``); nothing but the launch state and the records is saved.

Parameters enter as one tensor ``params`` of shape (S, GP_COUNT) (fp64) laid out like the C ABI's
gradient block: columns ``GP_TX, GP_TY, GP_TZ`` pose translation, ``GP_CURV`` curvature 1/radius,
``GP_CONIC``, ``GP_N1``, ``GP_N2``, ``GP_COEF + j`` even- / odd-asphere coefficients, ``GP_R + 3 i + j`` the pose
rotation matrix (gradients only for tilted poses).  Callers build it from their own leaf tensors with ordinary
torch ops (e.g. ``params[s, GP_CURV] = 1 / radius``, ``R = Rz(rz) @ Ry(ry) @ Rx(rx)``), so the chain rule to radii,
thicknesses, tilt angles ... is autograd's job.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np
import torch

from . import _lib
from . import table as T
from .trace import _DTYPES, _REC_KEYS, DeviceTable, _c_records, _out_buffer, _trace

GP_TX, GP_TY, GP_TZ, GP_CURV, GP_CONIC, GP_N1, GP_N2, GP_COEF = 0, 1, 2, 3, 4, 5, 6, 7
GP_MAX_COEF = _lib.GP_MAX_COEF
GP_R = _lib.GP_R
GP_COUNT = _lib.GP_COUNT


# kinds whose 1-D coefficient list rides in the GP_COEF columns: even / odd asphere C_j, Forbes Q^bfs a_m (the kernel
# differentiates with respect to the Clenshaw-basis b_m; _TraceFn.backward maps the gradient back, forbes_basis_matrix)
COEF_KINDS = (T.GEOM_EVEN_ASPHERE, T.GEOM_ODD_ASPHERE, T.GEOM_FORBES_QBFS)


def table_to_params(table: T.SurfaceTable) -> torch.Tensor:
    """(S, GP_COUNT) fp64 tensor of the differentiable parameters of ``table`` (one wavelength)."""
    if table.n_wl != 1:
        raise ValueError("differentiable trace supports one wavelength per call")
    p = np.zeros((table.num_surfaces, GP_COUNT))
    for s, spec in enumerate(table.surfaces):
        p[s, GP_TX:GP_TZ + 1] = spec.t
        p[s, GP_CURV] = 0.0 if not np.isfinite(spec.radius) else 1.0 / spec.radius
        p[s, GP_CONIC] = spec.conic
        p[s, GP_N1], p[s, GP_N2] = spec.n1[0], spec.n2[0]
        p[s, GP_R:GP_R + 9] = np.asarray(spec.R, dtype=np.float64).reshape(9)
        if spec.kind in COEF_KINDS:
            k = len(spec.coefficients)
            if k > GP_MAX_COEF:
                raise ValueError(f"more than {GP_MAX_COEF} asphere / Forbes coefficients")
            p[s, GP_COEF:GP_COEF + k] = spec.coefficients
    return torch.from_numpy(p)


POLY_KINDS = (T.GEOM_POLYNOMIAL, T.GEOM_ZERNIKE, T.GEOM_CHEBYSHEV)


def chebyshev_monomials(n: int) -> np.ndarray:
    """(n, n) matrix Tc with T_i(x) = sum_p Tc[i, p] x**p (T_0 = 1, T_1 = x, T_{i+1} = 2 x T_i - T_{i-1}): the
    expansion the table upload applies to a Chebyshev surface (csrc/olb_prep.h)."""
    Tc = np.zeros((n, n))
    if n > 0:
        Tc[0, 0] = 1.0
    if n > 1:
        Tc[1, 1] = 1.0
    for i in range(2, n):
        Tc[i, 1:] = 2.0 * Tc[i - 1, :-1]
        Tc[i] -= Tc[i - 2]
    return Tc


def forbes_basis_matrix(nc: int) -> np.ndarray:
    """Upper-banded (nc, nc) matrix A of the Forbes Q^bfs change of basis ``A b = a`` between the user's coefficients a_m
    and the coefficients b_m the Clenshaw recurrence runs on: A[i, i] = f_i, A[i, i+1] = g_i, A[i, i+2] = h_i
    (G. W. Forbes, Opt. Express 18, 19700 (2010), eqs. A.14-A.16; optiland/geometries/forbes/qpoly.py:56-115;
    the table upload solves it by back-substitution, csrc/olb_prep.h).  The adjoint kernel returns dLoss/db_m in the
    coefficient slots; dLoss/da = A^-T dLoss/db."""
    f, g, h = np.zeros(nc + 2), np.zeros(nc + 2), np.zeros(nc + 2)
    for n in range(nc):
        if n == 0:
            f[0] = 2.0
        elif n == 1:
            g[0] = -0.5
            f[1] = np.sqrt(19.0) / 2.0
        else:
            h[n - 2] = -n * (n - 1) / (2.0 * f[n - 2])
            g[n - 1] = -(1.0 + g[n - 2] * h[n - 2]) / f[n - 1]
            f[n] = np.sqrt(n * (n + 1) + 3.0 - g[n - 1] ** 2 - h[n - 2] ** 2)
    A = np.zeros((nc, nc))
    for i in range(nc):
        A[i, i] = f[i]
        if i + 1 < nc:
            A[i, i + 1] = g[i]
        if i + 2 < nc:
            A[i, i + 2] = h[i]
    return A


def forbes_coef_grads(gb: np.ndarray) -> np.ndarray:
    """dLoss/da_m of a Forbes Q^bfs surface from the kernel's dLoss/db_m (``forbes_basis_matrix``)."""
    nc = len(gb)
    return np.linalg.solve(forbes_basis_matrix(nc).T, gb) if nc else gb


def zernike_norms(spec) -> np.ndarray:
    """N_nm per Zernike term: from the packer when it ran on live objects, else c N / c (1 where c == 0)."""
    if spec.zernike_norms is not None:
        return np.asarray(spec.zernike_norms, dtype=np.float64)
    cf = spec.coefficients.reshape(-1, 4)
    with np.errstate(all="ignore"):
        return np.where(cf[:, 3] != 0, cf[:, 2] / np.where(cf[:, 3] != 0, cf[:, 3], 1.0), 1.0)


def table_to_coefs(table: T.SurfaceTable) -> torch.Tensor | None:
    """(S, K) fp64 tensor of the USER coefficients of the polynomial-family surfaces (Zernike: c_k in term order;
    polynomial and Chebyshev: C_ij row-major), zero-padded to the longest; None when the table has none."""
    rows = []
    for spec in table.surfaces:
        if spec.kind == T.GEOM_ZERNIKE:
            rows.append(spec.coefficients.reshape(-1, 4)[:, 3].copy())
        elif spec.kind in (T.GEOM_POLYNOMIAL, T.GEOM_CHEBYSHEV):
            rows.append(np.atleast_2d(spec.coefficients).ravel().copy())
        else:
            rows.append(np.zeros(0))
    K = max(len(r) for r in rows)
    if K == 0:
        return None
    out = np.zeros((len(rows), K))
    for s, r in enumerate(rows):
        out[s, :len(r)] = r
    return torch.from_numpy(out)


def _coef_maps(table: T.SurfaceTable):
    """Per polynomial-family surface the linear map (table gradients -> coefficient gradients), cached on the table:
    Zernike: stacks N_k M_k and M_k (K, 12, 12); polynomial: the (rows, cols) shape."""
    maps = table.__dict__.get("_coef_maps")
    if maps is None:
        maps = {}
        for s, spec in enumerate(table.surfaces):
            if spec.kind == T.GEOM_ZERNIKE:
                cf = spec.coefficients.reshape(-1, 4)
                M = np.stack([T.zernike_monomials(int(n), int(m), _lib.GT_DIM) for n, m in cf[:, :2]]) if len(cf) else np.zeros((0, 12, 12))
                maps[s] = ("zernike", M * zernike_norms(spec)[:, None, None], M)
            elif spec.kind == T.GEOM_POLYNOMIAL:
                maps[s] = ("polynomial", np.atleast_2d(spec.coefficients).shape)
            elif spec.kind == T.GEOM_CHEBYSHEV:
                shp = np.atleast_2d(spec.coefficients).shape
                Tc = chebyshev_monomials(max(shp))
                maps[s] = ("chebyshev", shp, Tc[:shp[0], :shp[0]], Tc[:shp[1], :shp[1]])
        table.__dict__["_coef_maps"] = maps
    return maps


def tables_to_coef_grads(table: T.SurfaceTable, gtab: np.ndarray, K: int) -> np.ndarray:
    """(S, 2, 12, 12) table gradients of olb_trace_bwd_* (grad_tables) -> (S, K) gradients of the user coefficients."""
    out = np.zeros((table.num_surfaces, K))
    for s, m in _coef_maps(table).items():
        if m[0] == "zernike":
            g = np.tensordot(m[1], gtab[s, 0], axes=2) + np.tensordot(m[2], gtab[s, 1], axes=2)
            out[s, :len(g)] = g
        elif m[0] == "chebyshev":
            # ONE monomial table P_pq = sum_ij C_ij Tc[i, p] Tc[j, q] serves the sag and the slopes
            r, c = m[1]
            g = gtab[s, 0, :r, :c] + gtab[s, 1, :r, :c]
            out[s, :r * c] = (m[2] @ g @ m[3].T).ravel()
        else:
            r, c = m[1]
            out[s, :r * c] = (gtab[s, 0, :r, :c] + gtab[s, 1, :r, :c]).ravel()
    return out


def params_to_table(table: T.SurfaceTable, params: torch.Tensor, coefs: torch.Tensor | None = None) -> T.SurfaceTable:
    """``table`` with its differentiable parameters replaced by the VALUES in ``params`` (and, for polynomial-family
    surfaces, the user coefficients in ``coefs``)."""
    p = params.detach().double().cpu().numpy()
    cv = coefs.detach().double().cpu().numpy() if coefs is not None else None
    specs = []
    for s, spec in enumerate(table.surfaces):
        ch = dict(t=p[s, GP_TX:GP_TZ + 1].copy(), n1=np.array([p[s, GP_N1]]), n2=np.array([p[s, GP_N2]]))
        if spec.kind != T.GEOM_NOOP:
            ch["R"] = p[s, GP_R:GP_R + 9].reshape(3, 3).copy()
        if spec.kind in (T.GEOM_STANDARD,) + COEF_KINDS:
            ch["radius"] = float("inf") if p[s, GP_CURV] == 0 else 1.0 / p[s, GP_CURV]
            ch["conic"] = float(p[s, GP_CONIC])
        if spec.kind in COEF_KINDS:
            ch["coefficients"] = p[s, GP_COEF:GP_COEF + len(spec.coefficients)].copy()
        if spec.kind in POLY_KINDS:
            ch["radius"] = float("inf") if p[s, GP_CURV] == 0 else 1.0 / p[s, GP_CURV]
            ch["conic"] = float(p[s, GP_CONIC])
            if cv is not None:
                if spec.kind == T.GEOM_ZERNIKE:
                    cf = spec.coefficients.reshape(-1, 4).copy()
                    cf[:, 3] = cv[s, :len(cf)]
                    cf[:, 2] = cf[:, 3] * zernike_norms(spec)
                    ch["coefficients"] = cf
                    ch["zernike_norms"] = zernike_norms(spec)
                else:                                   # polynomial, Chebyshev: C_ij row-major
                    shp = np.atleast_2d(spec.coefficients).shape
                    ch["coefficients"] = cv[s, :shp[0] * shp[1]].reshape(shp).copy()
        specs.append(dataclasses.replace(spec, **ch))
    return T.SurfaceTable(specs, table.wavelengths)


class _ParamPacker:
    """``params_to_table(template, params).packed()`` without building SurfaceSpec objects: the template's packed
    arrays (C ABI layout, table.py ``pack``) with the parameter VALUES written in place by a handful of vectorised
    numpy assignments -- the per-step host cost of an optimisation loop (dataclass copies + re-packing otherwise).
    Same bytes as the slow path (tests/test_autograd_cpu.py)."""

    def __init__(self, template: T.SurfaceTable):
        surf, pool = template.packed()
        self.surf0, self.pool0 = surf, pool
        kinds = np.array([s.kind for s in template.surfaces])
        self.rot = np.nonzero(kinds != T.GEOM_NOOP)[0]
        self.curved = np.nonzero(np.isin(kinds, (T.GEOM_STANDARD,) + COEF_KINDS + POLY_KINDS))[0]
        ci, cs, ck = [], [], []
        for s, spec in enumerate(template.surfaces):
            if spec.kind in COEF_KINDS:
                k = len(spec.coefficients)
                ci += list(range(int(surf["coef_off"][s]), int(surf["coef_off"][s]) + k))
                cs += [s] * k
                ck += list(range(GP_COEF, GP_COEF + k))
        self.coef_pool, self.coef_s, self.coef_k = (np.asarray(a, dtype=np.int64) for a in (ci, cs, ck))
        # media block of a surface (one wavelength): n1, n2, k1, coating n1, coating n2  (table.py pack)
        self.media = surf["media_off"].astype(np.int64)
        self.cn1 = np.array([s.coat_n1 is None for s in template.surfaces])
        self.cn2 = np.array([s.coat_n2 is None for s in template.surfaces])

    def __call__(self, p: np.ndarray):
        surf, pool = self.surf0.copy(), self.pool0.copy()
        surf["t"] = p[:, GP_TX:GP_TZ + 1]
        if len(self.rot):
            R = surf["R"]
            R[self.rot] = p[self.rot, GP_R:GP_R + 9]
            surf["R"] = R
            # SurfaceSpec.flags: ROTATED <=> R differs from the identity (table.py)
            fl = surf["flags"]
            is_rot = np.any(R != np.eye(3).reshape(9), axis=1)
            surf["flags"] = np.where(is_rot, fl | T.SF_ROTATED, fl & ~np.uint32(T.SF_ROTATED)).astype(fl.dtype)
        if len(self.curved):
            cv = p[self.curved, GP_CURV]
            rad = surf["radius"]
            with np.errstate(divide="ignore"):
                rad[self.curved] = np.where(cv == 0, np.inf, 1.0 / np.where(cv == 0, 1.0, cv))
            surf["radius"] = rad
            kc = surf["conic"]
            kc[self.curved] = p[self.curved, GP_CONIC]
            surf["conic"] = kc
        if len(self.coef_pool):
            pool[self.coef_pool] = p[self.coef_s, self.coef_k]
        pool[self.media] = p[:, GP_N1]
        pool[self.media + 1] = p[:, GP_N2]
        pool[self.media[self.cn1] + 3] = p[self.cn1, GP_N1]
        pool[self.media[self.cn2] + 4] = p[self.cn2, GP_N2]
        return surf, pool


def _packed_from_params(template: T.SurfaceTable, params: torch.Tensor):
    pk = template.__dict__.get("_param_packer")
    if pk is None:
        pk = template.__dict__["_param_packer"] = _ParamPacker(template)
    return pk(params.detach().double().cpu().numpy())


_forbes_cache: dict = {}


def _forbes_inv_t(nc: int, device) -> torch.Tensor:
    """A^-T of ``forbes_basis_matrix(nc)`` as a device tensor (cached): dLoss/da = A^-T dLoss/db."""
    key = (nc, str(device))
    m = _forbes_cache.get(key)
    if m is None:
        m = _forbes_cache[key] = torch.from_numpy(np.linalg.inv(forbes_basis_matrix(nc)).T.copy()).to(device)
    return m


class _TraceFn(torch.autograd.Function):
    """forward(template, holder, rows, params, x, y, z, L, M, N, i, opd).  ``rows`` = None: the 8 outputs
    are the full (S, N) record arrays; ``rows`` = tuple of row indices: 8 * len(rows) outputs, one (N,)
    tensor per (quantity, row) -- the backward pass then reads gradients only for those rows."""

    @staticmethod
    def forward(ctx, template, device_tables, rows, params, coefs, x, y, z, L, M, N, i, opd):
        ctx.set_materialize_grads(False)
        dtype = x.dtype
        sfx = _DTYPES[dtype]
        if device_tables and isinstance(device_tables[0], DeviceTable):
            # the caller already prepared + uploaded the table that holds exactly the VALUES of ``params``
            # (the plugin packs it from the live objects the parameters were read from)
            dtab = device_tables[0]
            table = dtab.table
        elif coefs is None and template.n_wl == 1:
            # (the DeviceTable's ``table`` stays the TEMPLATE: same structure, the values are those of ``params``)
            table = template
            dtab = DeviceTable(template, x.device, packed=_packed_from_params(template, params))
            device_tables.append(dtab)
        else:
            table = params_to_table(template, params, coefs)
            dtab = DeviceTable(table, x.device)
            device_tables.append(dtab)
        if not dtab.c.bwd_supported:
            raise _lib.OlbError("differentiable trace: table not supported by olb_trace_bwd_* (a geometry other than plane / "
                                "standard / even- and odd-asphere / polynomial / Zernike / Chebyshev / Forbes Q-bfs, a Fresnel coating, several wavelengths in one table)")
        n = x.numel()
        S = table.num_surfaces
        # (a slice / view of a larger tensor may start anywhere: the C ABI wants 16-byte aligned arrays)
        ins = [t.detach().contiguous() for t in (x, y, z, L, M, N, i, opd)]
        ins = [t.clone() if t.data_ptr() % 16 else t for t in ins]
        buf = _out_buffer(8, S, n, dtype, x.device)
        c_rays = _lib.OlbRays(**{k: t.data_ptr() for k, t in zip(("x", "y", "z", "L", "M", "N", "i", "opd"), ins)})
        # (no status word: out-of-range freeform coordinates are not reported on this path)
        _trace(dtab, x.device, dtype, 0, S, n, _lib.TF_NO_FINAL, rays=c_rays, rec=_c_records(buf), own_status=False)
        ctx.dtab, ctx.ins, ctx.buf, ctx.sfx = dtab, ins, buf, sfx
        ctx.rows = None if rows is None else tuple(r % S for r in rows)
        ctx.params_on_device = params.is_cuda
        ctx.coefs_meta = None if coefs is None else (coefs.shape[1], coefs.is_cuda, coefs.dtype)
        ctx.needs_ray_grad = any(t.requires_grad for t in (x, y, z, L, M, N, i, opd))
        if ctx.rows is None:
            return tuple(buf[j, :, :n] for j in range(8))
        return tuple(buf[j, r, :n] for j in range(8) for r in ctx.rows)

    @staticmethod
    def backward(ctx, *grads):
        lib = _lib.load()
        dtab, ins, buf = ctx.dtab, ctx.ins, ctx.buf
        n = ins[0].numel()
        S = buf.shape[1]
        dtype = buf.dtype
        if ctx.rows is None:
            gbufs = [None if g is None else g.to(dtype).contiguous() for g in grads]
            gbufs = [g.clone() if (g is not None and g.data_ptr() % 16) else g for g in gbufs]
            mask = (1 << 64) - 1
        else:
            # dense (S, n) gradient arrays are allocated WITHOUT a fill; only the rows named in the mask
            # are written here and read by the kernel
            nr = len(ctx.rows)
            gbufs, mask = [], 0
            for q, r in enumerate(ctx.rows):       # rows some quantity has a gradient for
                if any(grads[j * nr + q] is not None for j in range(8)):
                    mask |= 1 << r
            for j in range(8):
                gs = grads[j * nr:(j + 1) * nr]
                if all(g is None for g in gs):
                    gbufs.append(None)
                    continue
                gb = torch.empty((S, n), dtype=dtype, device=buf.device)
                for r, g in zip(ctx.rows, gs):
                    if not (mask >> r) & 1:
                        continue                   # the kernel never reads this row
                    if g is None:
                        gb[r].zero_()
                    else:
                        gb[r].copy_(g)
                gbufs.append(gb)
        c_grec = _lib.OlbRecords(*[(g.data_ptr() if g is not None else None) for g in gbufs], n)
        c_rec = _c_records(buf)
        c_in = _lib.OlbRays(**{k: t.data_ptr() for k, t in zip(("x", "y", "z", "L", "M", "N", "i", "opd"), ins)})
        gin = [torch.empty_like(ins[0]) for _ in range(8)] if ctx.needs_ray_grad else None
        c_gin = _lib.OlbRays(**{k: t.data_ptr() for k, t in zip(("x", "y", "z", "L", "M", "N", "i", "opd"), gin)}) if gin else None
        gpar = torch.zeros((S, GP_COUNT), dtype=torch.float64, device=buf.device)
        tables = int(dtab.c.bwd_supported) == 2
        gtab = torch.zeros((S, 2, _lib.GT_DIM, _lib.GT_DIM), dtype=torch.float64, device=buf.device) if tables else None
        with torch.cuda.device(buf.device):
            stream = torch.cuda.current_stream(buf.device).cuda_stream
            # polynomial / Zernike / Chebyshev surfaces: table gradients as well (grad_tables)
            rc = getattr(lib, f"olb_trace_bwd_{ctx.sfx}")(
                C.byref(dtab.c), 0, S, C.byref(c_in), C.byref(c_rec), C.byref(c_grec),
                C.byref(c_gin) if c_gin is not None else None, C.c_void_p(gpar.data_ptr()),
                C.c_void_p(gtab.data_ptr() if gtab is not None else None), n, C.c_uint64(mask & ((1 << 64) - 1)),
                C.c_void_p(stream))
        _lib.check(rc, f"olb_trace_bwd_{ctx.sfx}")
        for s, spec in enumerate(dtab.table.surfaces):
            if spec.kind == T.GEOM_FORBES_QBFS and len(spec.coefficients):
                # the kernel's coefficient slots hold dLoss/db_m (Clenshaw basis): back to the user's a_m, on the device
                nc = len(spec.coefficients)
                gpar[s, GP_COEF:GP_COEF + nc] = _forbes_inv_t(nc, gpar.device) @ gpar[s, GP_COEF:GP_COEF + nc]
        gi = gin if gin is not None else [None] * 8
        gcoef = None
        if ctx.coefs_meta is not None and tables:
            # the tables are linear in the user's coefficients: a few hundred doubles, mapped on the host
            K, on_dev, cdt = ctx.coefs_meta
            gc = torch.from_numpy(tables_to_coef_grads(dtab.table, gtab.cpu().numpy(), K)).to(cdt)
            gcoef = gc.to(buf.device) if on_dev else gc
        return (None, None, None, gpar if ctx.params_on_device else gpar.cpu(), gcoef, *gi)


def trace_differentiable(template: T.SurfaceTable, params: torch.Tensor, rays, rows=None, coefs: torch.Tensor | None = None):
    """Trace ``rays`` (an ``optiland_b200.trace.RealRays``) through ``template`` with parameter VALUES
    taken from ``params`` (and ``coefs``: the user coefficients of polynomial / Zernike / Chebyshev surfaces, ``table_to_coefs``).  Returns a dict of record tensors that are autograd outputs of ``params``
    (and of the ray tensors when they require grad): (S, N) arrays when ``rows`` is None, otherwise
    only the requested rows -- (N,) tensors for a single row, lists of (N,) tensors for several --
    which keeps the backward pass from touching gradients of rows the loss never reads."""
    holder: list = []
    rows_t = None if rows is None else tuple(int(r) for r in rows)
    outs = _TraceFn.apply(template, holder, rows_t, params, coefs, rays.x, rays.y, rays.z, rays.L, rays.M, rays.N, rays.i, rays.opd)
    if rows_t is None:
        return dict(zip(_REC_KEYS, outs))
    nr = len(rows_t)
    if nr == 1:
        return {k: outs[j] for j, k in enumerate(_REC_KEYS)}
    return {k: list(outs[j * nr:(j + 1) * nr]) for j, k in enumerate(_REC_KEYS)}
