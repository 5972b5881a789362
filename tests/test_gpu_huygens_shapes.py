"""The Huygens-Fresnel PSF kernel (``olb_huygens_psf_f64``, csrc/olb_psf.cu) in each of its launch shapes.

The launcher runs one thread per image point (``PSF_BLOCK`` = 128 per CTA) and, when there are fewer than 8 CTAs per SM,
splits the pupil sum over ``gridDim.y`` slices of whole ``PSF_TILE`` = 512-point tiles, each slice adding its partial
field with an atomic.  The slice count is ``ceil(8 SMs / CTAs)``, capped by the number of pupil tiles and by 64, and then
recomputed from the rounded-up ``pupil_per_split`` (which can lower it).  Every shape below is chosen from the device's own
SM count so that it lands on one branch of that rule: a single slice (pupil within one tile, or an image that fills the
device), 2 slices, the two shapes of scripts/bench_psf.py, the 64-slice cap, pupils ragged against the tile, a
recomputation that lowers the count, one image point, and complex amplitudes.

The reference is ``oracle.trace_oracle.huygens_fresnel_psf`` restated per image point in ``np.longdouble``.  The bound
per image point is derived from the kernel's operation count (see ``_field_bound``); the atomics make the low bits differ
from run to run, so no test asks for bit-equality between runs.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

PSF_BLOCK = 128                   # olb_psf.cu
PSF_TILE = 512
MAX_SPLITS = 64
CTAS_PER_SM = 8
U64 = 2.0 ** -53
ULD = float(np.finfo(np.longdouble).eps) / 2      # unit roundoff of the reference's arithmetic
PI_LD = np.longdouble("3.14159265358979323846264338327950288")
WAVELENGTH = 0.55e-3              # mm
RP = -80.0                        # pupil sphere radius (mm), negative as in tests/golden/huygens_psf_ref.npz
# C1: the phase in turns, (R - opd) / lambda.  R2 = fma(dx, dx, fma(dy, dy, dz dz)) carries 2u from the rounded
# differences and 3u from its own three roundings (5u); R = R2 rsqrt(R2) then has 2.5u from R2, 2u from rsqrt (1 ulp) and
# u from the product (5.5u); the subtraction, the rounded 1 / lambda and the product add 3u of (R + |opd|).  The reduction
# to [-1/2, 1/2] turns and the doubling are exact.
C1 = 8.5
# sincospi is within 1 ulp (<= 2u) per component: 2 sqrt(2) u of the unit phasor; ar = amp_re q, ai = amp_im q one
# rounding each: sqrt(2) u of |amp q|
C_PHASOR = 2.0 * math.sqrt(2.0) + math.sqrt(2.0)


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _slices(n_img, n_pupil, sms):
    """The launcher's rule (olb_huygens_psf_f64): (slices before the recomputation, slices, pupil points per slice)."""
    grid = -(-n_img // PSF_BLOCK)
    want = CTAS_PER_SM * sms
    splits = 1
    if grid < want:
        splits = -(-want // grid)
        splits = max(1, min(splits, -(-n_pupil // PSF_TILE), MAX_SPLITS))
    first = splits
    per = n_pupil
    if splits > 1:
        per = -(-(-(-n_pupil // splits)) // PSF_TILE) * PSF_TILE
        splits = -(-n_pupil // per)
    return first, splits, per


def _disk(side):
    lin = np.linspace(-1.0, 1.0, side)
    U, V = np.meshgrid(lin, lin, indexing="ij")
    m = U ** 2 + V ** 2 <= 1
    return U[m], V[m]


def _pupil(n_pupil, rng, bench_side=None, complex_amp=False):
    """Pupil points on the sphere |Q| = |Rp| about the image origin, 10 mm aperture: a random disk sample, or the
    bench's grid of ``bench_side``^2 cells inside the unit disk."""
    if bench_side is not None:
        U, V = _disk(bench_side)
    else:
        r = np.sqrt(rng.uniform(0.0, 1.0, n_pupil))
        th = rng.uniform(0.0, 2.0 * np.pi, n_pupil)
        U, V = r * np.cos(th), r * np.sin(th)
    pu, pv = 10.0 * U, 10.0 * V
    pw = -np.sqrt(RP ** 2 - pu ** 2 - pv ** 2)
    amp = rng.uniform(0.5, 1.5, pu.size)
    if complex_amp:
        amp = amp * np.exp(1j * rng.uniform(0.0, 2.0 * np.pi, pu.size))
    opd = 1e-4 * rng.standard_normal(pu.size)
    return pu, pv, pw, amp, opd


def _image(n_img):
    """A raster of n_img points over a 40 um square at z = 0 (row-major, ragged last row)."""
    side = max(1, math.isqrt(n_img - 1) + 1)
    k = np.arange(n_img)
    span = 0.04 / max(side - 1, 1)
    x = -0.02 + span * (k % side)
    y = -0.02 + span * (k // side)
    return x, y, np.zeros(n_img)


def _shape(name, sms):
    """(n_image, n_pupil, bench pupil side or None, complex amplitudes, expected slices) for one launch shape."""
    want = CTAS_PER_SM * sms
    if name == "pupil_in_one_tile":
        return 10 * PSF_BLOCK, PSF_TILE, None, False, 1
    if name == "image_fills_the_device":
        return (want - 1) * PSF_BLOCK + 1, 1025, None, False, 1
    if name == "two_slices":
        return (want * 3 // 4) * PSF_BLOCK - 37, 1025, None, False, 2
    if name in ("bench_128", "bench_256"):
        side = 128 if name == "bench_128" else 256
        n_img = side * side
        return n_img, _disk(side)[0].size, side, False, -(-want // (n_img // PSF_BLOCK))   # 9 and 3 on 132 SMs
    if name == "cap_64":
        return PSF_BLOCK, 65536, None, False, MAX_SPLITS
    if name.startswith("pupil_"):
        n_pup = int(name[6:])
        return 100, n_pup, None, False, -(-n_pup // PSF_TILE)
    if name == "recomputation_lowers":
        # 4 slices asked for, 6 tiles: pupil_per_split = ceil(ceil(2561 / 4) / 512) 512 = 1024 -> 3 slices
        return (2 * sms + 1) * PSF_BLOCK, 5 * PSF_TILE + 1, None, False, 3
    if name == "one_image_point":
        return 1, 8 * PSF_TILE + 1, None, False, 9
    if name == "complex_amplitudes":
        return 1000, 3001, None, True, -(-3001 // PSF_TILE)        # 8 CTAs: capped by the pupil's 6 tiles
    raise KeyError(name)


SHAPES = ["pupil_in_one_tile", "image_fills_the_device", "two_slices", "bench_128", "bench_256", "cap_64",
          "pupil_511", "pupil_512", "pupil_513", "pupil_1025", "recomputation_lowers", "one_image_point",
          "complex_amplitudes"]


def _sample(n_img, psf, rng):
    """Image points checked against the reference: every point of small images; otherwise the first and the last CTA,
    the peak and 256 drawn at random."""
    if n_img <= 4 * PSF_BLOCK:
        return np.arange(n_img)
    last0 = (n_img - 1) // PSF_BLOCK * PSF_BLOCK
    idx = np.concatenate([np.arange(PSF_BLOCK), np.arange(last0, n_img), [int(np.argmax(psf))],
                          rng.integers(0, n_img, 256)])
    return np.unique(idx)


def _reference(ix, iy, iz, pu, pv, pw, amp, opd, sel):
    """Per image point of ``sel``: the field in long double (trace_oracle.huygens_fresnel_psf with the phase reduced
    to a fraction of a turn before the sine and cosine), sum |amp q|, max (R + |opd|) and the condition number of the
    obliquity factor that C2 needs."""
    L = np.longdouble
    u, v, w = pu.astype(L), pv.astype(L), pw.astype(L)
    op = opd.astype(L)
    ar = np.real(amp).astype(L)
    ai = np.imag(amp).astype(L) if np.iscomplexobj(amp) else np.zeros_like(ar)
    aabs = np.abs(amp).astype(np.float64)
    lam = L(WAVELENGTH)
    field = np.empty(sel.size, np.complex128)
    S = np.empty(sel.size)
    Rmax = np.empty(sel.size)
    cq = np.empty(sel.size)
    for j, p in enumerate(sel):
        dx, dy, dz = L(ix[p]) - u, L(iy[p]) - v, L(iz[p]) - w
        R = np.sqrt(dx * dx + dy * dy + dz * dz)
        turns = (R - op) / lam
        ph = 2 * PI_LD * (turns - np.rint(turns))
        dot = (dx * u + dy * v + dz * w) / L(RP)
        x = dot / R
        q = 0.5 * (1 + x) / R
        c, s = np.cos(ph), np.sin(ph)
        field[j] = complex(float(np.sum(q * (ar * c - ai * s))), float(np.sum(q * (ar * s + ai * c))))
        qd = q.astype(np.float64)
        S[j] = float(np.sum(aabs * np.abs(qd)))
        Rmax[j] = float(np.max(R.astype(np.float64) + np.abs(opd)))
        xd = x.astype(np.float64)
        sr = (np.abs(dx * u) + np.abs(dy * v) + np.abs(dz * w)).astype(np.float64) / (abs(RP) * R.astype(np.float64))
        cq[j] = float(np.max((4.0 * sr + 7.5 * np.abs(xd)) / np.abs(1.0 + xd))) + 6.5
    return field, S, Rmax, cq


def _field_bound(S, Rmax, cq, n_chain, u):
    """|field error| per image point at unit roundoff u:

        (C1 u 2 pi max(R + |opd|) / lambda + C2 u + 2 n_chain u) sum |amp q|

    C2 = C_PHASOR + the relative error of q = 0.5 (1 + dot rsqrt(R2)) rsqrt(R2) (``cq``: dot = fma(dx, u, fma(dy, v,
    dz w)) / Rp carries 4u of sum |d_i Q_i| / |Rp| and 2u of |dot|; rsqrt(R2) 4.5u, its products u each; all over
    |1 + dot / R|).  n_chain: the additions on one thread's running sum -- two fused multiply-adds per pupil point of its
    slice -- plus one atomic per slice; a chain of n roundings on a component errs by <= n u sum(|ar cs| + |ai sn|) <=
    sqrt(2) n u sum |amp q|, and the two components together by sqrt(2) times that."""
    return (C1 * u * 2.0 * math.pi * Rmax / WAVELENGTH + (C_PHASOR + cq) * u + 2.0 * n_chain * u) * S


@pytest.mark.parametrize("name", SHAPES)
def test_huygens_psf_against_the_long_double_sum(name):
    from optiland_b200.psf import huygens_fresnel_psf

    sms = _sms()
    n_img, n_pup, side, cplx, expect = _shape(name, sms)
    first, splits, per = _slices(n_img, n_pup, sms)
    assert splits == expect, (name, first, splits, per)
    if name == "recomputation_lowers":
        assert first == 4 and splits == 3
    if name == "pupil_in_one_tile":
        assert n_pup <= PSF_TILE and -(-n_img // PSF_BLOCK) < CTAS_PER_SM * sms
    if name == "image_fills_the_device":
        assert -(-n_img // PSF_BLOCK) == CTAS_PER_SM * sms
    if name == "cap_64":
        assert first == MAX_SPLITS and per * MAX_SPLITS == n_pup
    rng = np.random.default_rng(SHAPES.index(name))
    pu, pv, pw, amp, opd = _pupil(n_pup, rng, side, cplx)
    assert pu.size == n_pup
    ix, iy, iz = _image(n_img)
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (ix, iy, iz, pu, pv, pw, amp, opd)]
    psf_f, field = huygens_fresnel_psf(*dev, WAVELENGTH, RP, return_field=True)
    psf_o = huygens_fresnel_psf(*dev, WAVELENGTH, RP)
    psf_f, psf_o, field = psf_f.cpu().numpy(), psf_o.cpu().numpy(), field.cpu().numpy()
    assert psf_f.shape == psf_o.shape == field.shape == (n_img,)

    sel = _sample(n_img, psf_f, rng)
    ref, S, Rmax, cq = _reference(ix, iy, iz, pu, pv, pw, amp, opd, sel)
    n_chain = 2 * per + (splits if splits > 1 else 0)
    df = _field_bound(S, Rmax, cq, n_chain, U64) + _field_bound(S, Rmax, cq, 2 * n_pup, ULD)
    fa = np.abs(ref)
    # |psf - |ref|^2| <= 2 |ref| df + df^2, plus the kernel's re^2 + im^2 (2u) and the reference's own |.|^2
    dp = 2.0 * fa * df + df * df + (2.0 * U64 + 3.0 * ULD) * fa * fa
    err_f = np.abs(field[sel] - ref)
    assert np.all(err_f <= df), (name, float(np.max(err_f / df)))
    worst = float(np.max(err_f / df))
    for psf in (psf_f, psf_o):
        err_p = np.abs(psf[sel] - fa * fa)
        assert np.all(err_p <= dp), (name, float(np.max(err_p / dp)))
        worst = max(worst, float(np.max(err_p / dp)))
    # every pupil point counts: one term is far above the bound, so a dropped or doubled tile cannot hide in it
    assert np.all(df < 1e-3 * S / n_pup), (name, float(np.max(df * n_pup / S)))
    print(f"{name}: {n_img} image x {n_pup} pupil points, {splits} slice(s), worst error / bound {worst:.3e}")
