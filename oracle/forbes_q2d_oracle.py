"""TEST INFRASTRUCTURE ONLY -- CPU restatement (NumPy, fp64) of Optiland's ``ForbesQ2dGeometry``
(optiland/geometries/forbes/geometry.py:445-672 with the Q-2D recurrences of qpoly.py:286-540), on top of the NumPy oracle
of the trace loop (``oracle/trace_oracle.py``).

``trace`` has the signature and the results of ``trace_oracle.trace``; Q-2D surfaces get their sag and normal from here,
every other surface is traced by ``trace_oracle`` unchanged.  The restatement follows the reference's formulas and their
order of operations, written out from the papers' recurrences (G. W. Forbes, Opt. Express 20, 2483 (2012)); it shares no
code with the kernel's host-side preparation (olb_prep.h).
"""
from __future__ import annotations

from functools import lru_cache
from math import factorial

import numpy as np

from oracle import trace_oracle as O
from optiland_b200 import table as T

_EPS = 1e-12


def _dfact(k: int) -> float:
    out = 1
    while k > 1:
        out *= k
        k -= 2
    return float(out)


@lru_cache(maxsize=None)
def _gamma(n: int, m: int) -> float:
    if n == 1 and m == 2:
        return 3 / 8
    if n == 1 and m > 2:
        return ((2 * (m - 1) + 1) / (2 * (m - 2))) * _gamma(1, m - 1)
    return (n * (2 * m + 2 * (n - 1) - 1) / ((m + n - 3) * (2 * (n - 1) + 1))) * _gamma(n - 1, m)


def _g_raw(n: int, m: int) -> float:
    if n == 0:
        return _dfact(2 * m - 1) / (2 ** (m + 1) * factorial(m - 1))
    if m == 1:
        return -(2 * n**2 - 1) * (n**2 - 1) / (8 * (4 * n**2 - 1)) - (1 / 24 if n == 1 else 0)
    num = (2 * n * (m + n - 1) - m) * ((n + 1) * (2 * m + 2 * n - 1))
    den = (m + 2 * n - 2) * (m + 2 * n - 1) * ((m + 2 * n) * (2 * n + 1))
    return -num / den * _gamma(n, m)


def _f_raw(n: int, m: int) -> float:
    if n == 0 and m == 1:
        return 0.25
    if n == 0:
        return m**2 * _dfact(2 * m - 3) / (2 ** (m + 1) * factorial(m - 1))
    if m == 1:
        return (4 * (n - 1) ** 2 * n**2 + 1) / (8 * (2 * n - 1) ** 2) + (11 / 32 if n == 1 else 0)
    chi = m + n - 2
    num = 2 * n * chi * (3 - 5 * m + 4 * n * chi) + m**2 * (3 - m + 4 * n * chi)
    den = (m + 2 * n - 3) * (m + 2 * n - 2) * ((m + 2 * n - 1) * (2 * n - 1))
    return num / den * _gamma(n, m)


@lru_cache(maxsize=None)
def _fg(n: int, m: int) -> tuple[float, float]:
    f = np.sqrt(_f_raw(0, m)) if n == 0 else np.sqrt(_f_raw(n, m) - _fg(n - 1, m)[1] ** 2)
    return float(f), _g_raw(n, m) / float(f)


_SPECIAL = {(1, 0): (2, -1, 0), (1, 1): (-4 / 3, -8 / 3, -11 / 3), (1, 2): (9 / 5, -24 / 5, 0), (2, 0): (3, -2, 0),
            (3, 0): (5, -4, 0)}


def _abc(n: int, m: int) -> tuple[float, float, float]:
    if (m, n) in _SPECIAL:
        return _SPECIAL[(m, n)]
    d = (4 * n**2 - 1) * (m + n - 2) * (m + 2 * n - 3) or 1e-99
    a = (2 * n - 1) * (m + 2 * n - 2) * (4 * n * (m + n - 2) + (m - 3) * (2 * m - 1)) / d
    b = -2 * (2 * n - 1) * (m + 2 * n - 3) * (m + 2 * n - 2) * (m + 2 * n - 1) / d
    c = n * (2 * n - 3) * (m + 2 * n - 1) * (2 * m + 2 * n - 3) / d
    return a, b, c


def _pnm_basis(cs, m):
    """change_basis_q2d_to_pnm (qpoly.py:355-370)."""
    nmax = len(cs) - 1
    ds = [0.0] * (nmax + 1)
    for n in range(nmax, -1, -1):
        f, g = _fg(n, m)
        ds[n] = cs[n] / f if n == nmax else (cs[n] - g * ds[n + 1]) / f
    return ds


def _q2d_sum(cs, m, usq):
    """clenshaw_q2d_der with j = 1 and q2d_sum_from_alphas (qpoly.py:403-412, 507-584): (S, dS/d(usq))."""
    ds = _pnm_basis(cs, m)
    nmax = len(ds) - 1
    zero = np.zeros_like(usq)
    al = [zero] * (nmax + 3)
    dl = [zero] * (nmax + 3)
    for n in range(nmax, -1, -1):
        a, b, _ = _abc(n, m)
        c = _abc(n + 1, m)[2]
        al[n] = ds[n] + (a + b * usq) * al[n + 1] - c * al[n + 2]
        dl[n] = b * al[n + 1] + (a + b * usq) * dl[n + 1] - c * dl[n + 2]
    S, dS = 0.5 * al[0], 0.5 * dl[0]
    if m == 1 and len(cs) > 3:
        S, dS = S - 2 / 5 * al[3], dS - 2 / 5 * dl[3]
    return S, dS


def _sums(s: T.SurfaceSpec, u, theta):
    """compute_z_zprime_q2d (qpoly.py:462-473): S0, dS0/du, P, dP/du, dP/dtheta."""
    usq = u * u
    zero = np.zeros_like(u)
    S0, dS0 = zero, zero
    if len(s.q2d_cm0):
        S0, d = O._qbfs_sum(list(s.q2d_cm0), usq, want_derivative=True)
        dS0 = d * 2 * u
    P, DR, DT = zero, zero, zero
    for mi, (a, b) in enumerate(zip(s.q2d_ams, s.q2d_bms)):
        m = mi + 1
        sa = sap = sb = sbp = 0.0
        if len(a):
            sa, sap = _q2d_sum(list(a), m, usq)
        if len(b):
            sb, sbp = _q2d_sum(list(b), m, usq)
        cm, sm = np.cos(m * theta), np.sin(m * theta)
        P = P + u**m * (cm * sa + sm * sb)
        DR = DR + u ** (m - 1) * (cm * (2 * usq * sap + m * sa) + sm * (2 * usq * sbp + m * sb))
        DT = DT + m * u**m * (-sa * sm + sb * cm)
    return S0, dS0, P, DR, DT


def q2d_sag(s: T.SurfaceSpec, x, y):
    """ForbesQ2dGeometry.sag (geometry.py:539-571)."""
    with np.errstate(all="ignore"):
        r2 = x**2 + y**2
        if np.isinf(s.radius):
            zb = np.zeros_like(r2)
        else:
            arg = 1 - (1 + s.conic) * r2 / s.radius**2
            zb = r2 / (s.radius * (1 + np.sqrt(np.where(arg < 0, 0, arg))))
        rho = np.sqrt(r2 + _EPS)
        u = rho / s.norm_radius
        theta = np.arctan2(y, np.where(rho < _EPS, x + 1e-12, x))
        S0, _, P, _, _ = _sums(s, u, theta)
        phi, _ = O._forbes_phi(r2, s.radius, s.conic)
        usq = u**2
        dep = usq * (1 - usq) * phi * S0 + phi * P
        return zb + np.where(u > 1, 0.0, dep)


def q2d_vertex_slopes(s: T.SurfaceSpec):
    """_surface_normal_analytical_vertex (geometry.py:596-609)."""
    out = [0.0, 0.0]
    if s.q2d_ams:
        for j, lst in enumerate((s.q2d_ams[0], s.q2d_bms[0])):
            if len(lst):
                out[j] = float(_q2d_sum(list(lst), 1, np.float64(0.0))[0]) / s.norm_radius
    return out


def q2d_slopes(s: T.SurfaceSpec, x, y):
    """_surface_normal_analytical (geometry.py:611-672): (df/dx, df/dy)."""
    vx, vy = q2d_vertex_slopes(s)
    with np.errstate(all="ignore"):
        r2 = x**2 + y**2
        rho = np.sqrt(r2)
        vertex = rho < _EPS
        rs = np.where(vertex, _EPS, rho)
        u = rho / s.norm_radius
        theta = np.arctan2(y, x)
        S0, dS0, P, DR, DT = _sums(s, u, theta)
        phi, dphi = O._forbes_phi(r2, s.radius, s.conic)
        usq = u**2
        dpref = (2 * u - 4 * u**3) / s.norm_radius
        ds0 = (dpref * S0 + (usq - usq**2) * dS0 / s.norm_radius) * phi + (usq - usq**2) * S0 * dphi
        dsr = np.where(u > 1, 0.0, ds0 + dphi * P + phi * DR / s.norm_radius)
        dst = np.where(u > 1, 0.0, phi * DT)
        c, sn = x / rs, y / rs
        if np.isinf(s.radius) or s.radius == 0:
            db = np.zeros_like(rho)
        else:
            cv = 1.0 / s.radius
            arg = 1 - (s.conic + 1) * cv**2 * r2
            db = cv * rho / np.sqrt(np.where(arg > 0, arg, 1e-12))
        fx = db * c + (c * dsr - (sn / rs) * dst)
        fy = db * sn + (sn * dsr + (c / rs) * dst)
        return np.where(vertex, vx, fx), np.where(vertex, vy, fy)


def q2d_normal(s: T.SurfaceSpec, x, y):
    """ForbesQ2dGeometry._surface_normal (geometry.py:573-594)."""
    fx, fy = q2d_slopes(s, x, y)
    with np.errstate(all="ignore"):
        mag = np.sqrt(fx**2 + fy**2 + 1)
        mag = np.where(mag < _EPS, 1.0, mag)
        return fx / mag, fy / mag, -1.0 / mag


def trace(table: T.SurfaceTable, rays: dict, first: int = 0, last: int | None = None, polarized: bool = False):
    """``trace_oracle.trace`` with Q-2D surfaces."""
    orig = O._sag_and_normal_fns

    def fns(s, status):
        if s.kind == T.GEOM_FORBES_Q2D:
            return (lambda x, y: q2d_sag(s, x, y)), (lambda x, y: q2d_normal(s, x, y))
        return orig(s, status)

    O._sag_and_normal_fns = fns
    try:
        return O.trace(table, rays, first, last, polarized=polarized)
    finally:
        O._sag_and_normal_fns = orig
