"""Host-side mirror of the reference's interface for the hot path.

Names, argument meaning and error behaviour follow the reference so that the parity tests
read like the reference's own:

* ``RealRays``      <- optiland/rays/real_rays.py:23-89   (SoA container, same attribute names)
* ``SurfaceGroup``  <- optiland/surfaces/surface_group.py:27, ``trace(rays, skip=0)`` :245-257 and
  the stacked record properties ``x, y, z, L, M, N, opd, intensity`` :108-153

Everything numeric happens in libolb.so (sm_90a CUDA) through the C ABI; torch is used only
to own device memory and streams.  There is no CPU path: constructing these objects on a
box without CUDA or without the built library raises.
"""
from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import torch

from . import _lib
from . import table as T

_REC_KEYS = ("x", "y", "z", "L", "M", "N", "intensity", "opd")
_DTYPES = {torch.float32: "f32", torch.float64: "f64"}
_CDTYPES = {torch.float32: torch.complex64, torch.float64: torch.complex128}


def _require_cuda():
    if not torch.cuda.is_available():
        raise _lib.OlbError("optiland_b200 needs a CUDA device (sm_90a); there is no CPU fallback")


def _as_dev(v, n, dtype, device):
    t = torch.as_tensor(v, dtype=dtype, device=device)
    if t.ndim == 0:
        t = t.expand(n)
    t = t.reshape(-1).contiguous()
    if t.data_ptr() % 16:
        t = t.clone()
    return t


class RealRays:
    """Device-resident ray batch (structure of arrays), reference attribute names."""

    def __init__(self, x, y, z, L, M, N, intensity, wavelength, dtype=torch.float32, device=None):
        _require_cuda()
        if dtype not in _DTYPES:
            raise ValueError("dtype must be torch.float32 or torch.float64")
        device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        n = max(int(np.size(v)) if not torch.is_tensor(v) else v.numel()
                for v in (x, y, z, L, M, N, intensity, wavelength))
        self.x = _as_dev(x, n, dtype, device)
        self.y = _as_dev(y, n, dtype, device)
        self.z = _as_dev(z, n, dtype, device)
        self.L = _as_dev(L, n, dtype, device)
        self.M = _as_dev(M, n, dtype, device)
        self.N = _as_dev(N, n, dtype, device)
        self.i = _as_dev(intensity, n, dtype, device)
        self.w = _as_dev(wavelength, n, dtype, device)
        self.opd = torch.zeros_like(self.x)
        self.L0 = self.M0 = self.N0 = None
        self.is_normalized = True

    def __len__(self):
        return self.x.numel()

    @property
    def dtype(self):
        return self.x.dtype

    @property
    def device(self):
        return self.x.device


class PolarizedRays(RealRays):
    """``RealRays`` + the 3x3 complex polarization matrix ``p`` per ray, initialised to the identity
    (optiland/rays/polarized_rays.py:17-56).  ``p`` is a complex (N, 3, 3) tensor: the same memory
    layout as the reference's, which is what the C ABI takes."""

    def __init__(self, x, y, z, L, M, N, intensity, wavelength, dtype=torch.float32, device=None):
        super().__init__(x, y, z, L, M, N, intensity, wavelength, dtype=dtype, device=device)
        self.p = None  # identity until the first trace (OLB_TF_POL_IDENTITY: not read from HBM)
        self._i0 = self.i.clone()
        self._L0, self._M0, self._N0 = self.L.clone(), self.M.clone(), self.N.clone()

    def update_intensity(self, state=None):
        """Host-side epilogue of RealRayTracer.trace (polarized_rays.py:57-133, :204-233):
        i = sum |P E0|^2 * i0 / n_fields; ``state`` = (Ex, Ey, phase_x, phase_y) or None (unpolarized)."""
        k = torch.stack([self._L0, self._M0, self._N0], dim=1)
        xh = torch.tensor([1.0, 0.0, 0.0], dtype=k.dtype, device=k.device).expand_as(k)
        pv = torch.linalg.cross(k, xh)
        norms = torch.linalg.norm(pv, dim=1)
        if bool((norms == 0).any()):
            raise ValueError("k-vector parallel to x-axis is not currently supported.")
        pv = pv / norms[:, None]
        sv = torch.linalg.cross(pv, k)
        states = [state] if state is not None else [(1.0, 0.0, 0.0, 0.0), (0.0, 1.0, 0.0, 0.0)]
        inten = torch.zeros_like(self._i0)
        P = self.p
        for Ex, Ey, phx, phy in states:
            ax = complex(np.cos(phx), np.sin(phx)) * Ex
            ay = complex(np.cos(phy), np.sin(phy)) * Ey
            E0 = sv.to(P.dtype) * ax + pv.to(P.dtype) * ay
            E1 = torch.matmul(P, E0[:, :, None])[:, :, 0]
            inten = inten + (E1.abs() ** 2).sum(dim=1)
        self.i = inten * self._i0 / len(states)


class DeviceTable:
    """A ``SurfaceTable`` prepared and resident on one GPU (olb_table_upload)."""

    DEFAULT_WORKSPACE = 48 * 1024

    def __init__(self, table: T.SurfaceTable, device=None, packed=None):
        _require_cuda()
        self.lib = _lib.load()
        self.table = table
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.host = _lib.HostTable(table, packed)   # ``packed``: a (surf, pool) pair the caller already made
        self.c = _lib.OlbDeviceTable()
        # ONE preparation per upload: a generous workspace instead of asking olb_table_workspace_bytes first (which
        # prepares the table just to measure it); the rare table that needs more says so and is retried
        nbytes = self.DEFAULT_WORKSPACE
        for attempt in range(2):
            self.workspace = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
            with torch.cuda.device(self.device):
                stream = torch.cuda.current_stream(self.device).cuda_stream
                rc = self.lib.olb_table_upload(C.byref(self.host.c), self.workspace.data_ptr(), int(nbytes),
                                               C.c_void_p(stream), C.byref(self.c))
            if rc != 0 and attempt == 0 and "workspace too small" in _lib.last_error():
                nbytes = self.lib.olb_table_workspace_bytes(C.byref(self.host.c))
                if nbytes < 0:
                    _lib.check(int(nbytes), "olb_table_workspace_bytes")
                continue
            break
        _lib.check(rc, "olb_table_upload")
        # the upload is asynchronous on the current stream: launches on that stream are ordered behind it; users of
        # OTHER streams (the host-buffer pipeline, side streams) wait on this event first
        self.ready = torch.cuda.Event()
        self.ready.record(torch.cuda.current_stream(self.device))
        self.has_zernike = any(s.kind in (T.GEOM_ZERNIKE, T.GEOM_CHEBYSHEV) for s in table.surfaces)
        self.has_bsdf = any(s.bsdf != T.BSDF_NONE for s in table.surfaces)

    @property
    def features(self) -> int:
        return int(self.c.features)


def _byref(s):
    return C.byref(s) if s is not None else None


def _pointer(s):
    return C.pointer(s) if s is not None else None


def _status_word(dtab: "DeviceTable", device, force: bool = False):
    """Device int32 the kernels OR their OLB_ST_* bits into -- only for tables / call shapes that can raise them."""
    return torch.zeros(1, dtype=torch.int32, device=device) if (dtab.has_zernike or _has_bsdf(dtab) or force) else None


def _has_bsdf(dtab) -> bool:
    """Does the prepared table hold BSDF surfaces?  (Batched tables never do, and have no such attribute.)"""
    return getattr(dtab, "has_bsdf", False)


_STREAM = {"state": None, "next": 0}
_STREAM_LOCK = threading.Lock()


def next_rng_stream() -> int:
    """The Philox counter word of one trace of a table with BSDF surfaces (OlbTraceCall.rng_stream).  A counter: each
    call takes the next value, so successive calls never repeat a stream (up to 2^32 calls).  Its start is drawn from
    torch's default generator whenever that generator's state is not the one this function left behind (first use,
    ``torch.manual_seed``, other draws in between), so ``torch.manual_seed`` makes a sequence of traces repeat bit for
    bit."""
    g = torch.default_generator
    with _STREAM_LOCK:
        st = g.get_state()
        if _STREAM["state"] is None or not torch.equal(st, _STREAM["state"]):
            _STREAM["next"] = int(torch.randint(0, 1 << 32, (1,), dtype=torch.int64).item())
            _STREAM["state"] = g.get_state()
        s = _STREAM["next"]
        _STREAM["next"] = (s + 1) & 0xFFFFFFFF
        return s


def _raise_status(status) -> None:
    """The reference's ValueErrors for out-of-range freeform coordinates, from the kernel's status word; shared by
    every entry point (plain, pupil-launch, wavefront, moments) so that none of them returns extrapolated numbers."""
    if status is None:
        return
    st = int(status.item())
    if st & T.ST_ZERNIKE_RANGE:
        # same exception, same message as optiland/geometries/zernike.py:254-266
        raise ValueError(
            "Zernike coordinates must be normalized to [-1, 1]. Consider updating the normalization "
            "radius to 1.1x the surface aperture.")
    if st & T.ST_CHEBYSHEV_RANGE:
        # optiland/geometries/chebyshev.py:230-244
        raise ValueError(
            "Chebyshev input coordinates must be normalized to [-1, 1]. Consider updating the "
            "normalization factors.")
    if st & T.ST_K_PARALLEL_X:
        # optiland/rays/polarized_rays.py:216-218
        raise ValueError("k-vector parallel to x-axis is not currently supported.")
    if st & T.ST_BSDF_ATTEMPTS:
        # the reference would loop for ever (optiland/scatter.py); the kernel bounds the loop
        raise ValueError(f"BSDF scatter: a ray rejected {T.BSDF_MAX_ATTEMPTS} drawn directions (is the Gaussian sigma "
                         "far above 1?); its direction is NaN")


def _out_buffer(k: int, rows: int, n: int, dtype, device) -> torch.Tensor:
    """Uninitialised (k, rows, stride) output rows of n rays.  The kernel uses vector accesses (4 fp32 / 2 fp64 rays)
    only when every row starts on a vector boundary, so the stride is n when n is a multiple of the vector width and
    otherwise n rounded up to 64 (every row stays 16-byte aligned)."""
    vec = 4 if dtype == torch.float32 else 2
    stride = n if n % vec == 0 else (n + 63) // 64 * 64
    return torch.empty((k, rows, stride), dtype=dtype, device=device)


def _c_records(buf: torch.Tensor):
    """OlbRecords over an (8, rows, stride) buffer."""
    return _lib.OlbRecords(*[buf[j].data_ptr() for j in range(8)], buf.shape[-1])


def _take_last_row(rays, recs):
    """``rays.x`` .. ``rays.opd`` become views of the last record row (with OLB_TF_NO_FINAL the kernel writes the
    final state only there)."""
    rays.x, rays.y, rays.z = recs["x"][-1], recs["y"][-1], recs["z"][-1]
    rays.L, rays.M, rays.N = recs["L"][-1], recs["M"][-1], recs["N"][-1]
    rays.i, rays.opd = recs["intensity"][-1], recs["opd"][-1]
    return rays


def _trace(dtab, device, dtype, first, last, n, flags, rays=None, rec=None, launch=None, center=(0.0, 0.0),
           moments=None, rays_per_system=0, wavefront=None, pol=None, status=None, own_status=True, rng_stream=None):
    """The one forward call of the library (olb_trace_call_f32 / _f64, include/olb.h: OlbTraceCall).  ``rays`` /
    ``rec`` / ``launch`` / ``pol``: ctypes structs or None; ``wavefront``: (OlbWavefrontRef, OlbWavefrontOut) or None;
    ``moments``: device tensor or None.  ``own_status``: the status word is made here (when the table or the call
    shape can set OLB_ST_* bits) and the reference's errors are raised from it; otherwise ``status`` (a caller-owned
    device int32, or None) is passed through unchecked.  ``rng_stream``: the counter word of BSDF scatter draws (tables
    with BSDF surfaces; None draws a fresh one, ``next_rng_stream``)."""
    if _has_bsdf(dtab) and rng_stream is None:
        rng_stream = next_rng_stream()
    if own_status:
        status = _status_word(dtab, device, force=pol is not None)
    ref, out = wavefront if wavefront is not None else (None, None)
    call = _lib.OlbTraceCall(
        first=first, last=last, n_rays=n, flags=flags, rng_stream=int(rng_stream or 0), rays=_pointer(rays),
        rec=_pointer(rec), launch=_pointer(launch),
        center=(float(center[0]), float(center[1])), moments=moments.data_ptr() if moments is not None else None,
        rays_per_system=rays_per_system, wavefront_ref=_pointer(ref), wavefront_out=_pointer(out), pol=_pointer(pol),
        status=status.data_ptr() if status is not None else None)
    sfx = _DTYPES[dtype]
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        rc = getattr(dtab.lib, f"olb_trace_call_{sfx}")(C.byref(dtab.c), C.byref(call), C.c_void_p(stream))
    _lib.check(rc, f"olb_trace_call_{sfx}")
    if own_status:
        _raise_status(status)


def _c_polarization(state, intensity_out=None):
    """OlbPolarization from ``state`` = None / "unpolarized" (the mean of two orthogonal states) or
    (Ex, Ey, phase_x, phase_y) (normalised as PolarizationState does, polarization_state.py:53-56)."""
    c = _lib.OlbPolarization()
    if state is None or state == "unpolarized":
        c.is_polarized = 0
    else:
        Ex, Ey, phx, phy = (float(v) for v in state)
        mag = (Ex * Ex + Ey * Ey) ** 0.5
        c.is_polarized, c.Ex, c.Ey, c.phase_x, c.phase_y = 1, Ex / mag, Ey / mag, phx, phy
    c.intensity = intensity_out.data_ptr() if intensity_out is not None else None
    return c


def trace_device(dtab: DeviceTable, rays: RealRays, first: int, last: int, record: bool = True,
                 want_l0: bool = False, polarization=False, rng_stream=None):
    """One trace of ``rays`` on the device.  Returns the dict of (rows, N) record tensors (or None).

    With ``record`` the final state is NOT written a second time: ``rays.x`` .. ``rays.opd``
    become views of the last record row (OLB_TF_NO_FINAL), saving 32-64 B/ray of HBM traffic.
    The reference never mutates these arrays in place (it re-assigns attributes), so the
    aliasing is not observable through its API.

    ``polarization`` (PolarizedRays only): None / "unpolarized" / (Ex, Ey, phase_x, phase_y) runs
    PolarizedRays.update_intensity as the kernel's epilogue (OlbTraceCall.pol): ``rays.i`` becomes
    sum |P E0|^2 i0 / n_states while the record rows keep the geometric intensity.

    ``rng_stream``: BSDF tables only, the counter word of the scatter draws (None: ``next_rng_stream()``).
    """
    n = len(rays)
    if rays.device != dtab.device:
        raise ValueError(f"rays on {rays.device}, table on {dtab.device}")
    rows = last - first
    recs = None
    c_rec = None
    flags = 0
    if record and rows > 0:
        buf = _out_buffer(8, rows, n, rays.dtype, rays.device)
        recs = {k: buf[j, :, :n] for j, k in enumerate(_REC_KEYS)}
        c_rec = _c_records(buf)
        flags |= _lib.TF_NO_FINAL
    if want_l0:
        rays.L0 = torch.empty_like(rays.x)
        rays.M0 = torch.empty_like(rays.x)
        rays.N0 = torch.empty_like(rays.x)
    p_ptr = None
    if isinstance(rays, PolarizedRays):
        flags |= _lib.TF_POLARIZED
        if rays.p is None:
            rays.p = torch.empty((n, 3, 3), dtype=_CDTYPES[rays.dtype], device=rays.device)
            flags |= _lib.TF_POL_IDENTITY
        else:
            rays.p = rays.p.to(_CDTYPES[rays.dtype]).contiguous()
        p_ptr = torch.view_as_real(rays.p).data_ptr()
    c_rays = _lib.OlbRays(
        x=rays.x.data_ptr(), y=rays.y.data_ptr(), z=rays.z.data_ptr(), L=rays.L.data_ptr(),
        M=rays.M.data_ptr(), N=rays.N.data_ptr(), i=rays.i.data_ptr(),
        w=rays.w.data_ptr() if dtab.table.n_wl > 1 else None, opd=rays.opd.data_ptr(),
        L0=rays.L0.data_ptr() if want_l0 else None, M0=rays.M0.data_ptr() if want_l0 else None,
        N0=rays.N0.data_ptr() if want_l0 else None, p=p_ptr)
    pol_i, c_pol = None, None
    if polarization is not False:
        if not isinstance(rays, PolarizedRays):
            raise ValueError("the intensity epilogue needs PolarizedRays")
        pol_i = torch.empty_like(rays.x)
        c_pol = _c_polarization(polarization, pol_i)
    _trace(dtab, rays.device, rays.dtype, first, last, n, flags, rays=c_rays, rec=c_rec, pol=c_pol, rng_stream=rng_stream)
    if recs is not None:
        _take_last_row(rays, recs)
    if pol_i is not None:
        rays.i = pol_i
    return recs


def aim_device(dtab: DeviceTable, guess: dict, Px: torch.Tensor, Py: torch.Tensor, first: int, last: int,
               r_stop: float, J_factor: float, tol: float, max_iter: int, infinite: bool) -> torch.Tensor:
    """One ray-aiming solve on the device (olb_aim_f32 / _f64, include/olb.h: OlbAimCall).  ``guess``: the launch state
    {"x", "y", "z", "L", "M", "N"} (+ "w" when the table has several wavelengths), 1-D device tensors of one type and
    length, 16-byte aligned; the solution is written into them in place.  ``Px`` / ``Py``: the pupil targets, same type
    and length.  Returns the device int32 status word (OLB_ST_* bits; not checked here, nothing is synchronised)."""
    x = guess["x"]
    n = int(x.numel())
    for t in [guess[k] for k in ("y", "z", "L", "M", "N")] + [Px, Py]:
        if t.dtype != x.dtype or t.device != dtab.device or t.numel() != n:
            raise ValueError("aim: guess and pupil arrays must share one dtype, length and the table's device")
    status = torch.zeros(1, dtype=torch.int32, device=dtab.device)
    w = guess.get("w") if dtab.table.n_wl > 1 else None
    c_rays = _lib.OlbRays(x=x.data_ptr(), y=guess["y"].data_ptr(), z=guess["z"].data_ptr(), L=guess["L"].data_ptr(),
                          M=guess["M"].data_ptr(), N=guess["N"].data_ptr(), w=w.data_ptr() if w is not None else None)
    call = _lib.OlbAimCall(first=first, last=last, n_rays=n, rays=C.pointer(c_rays), Px=Px.data_ptr(), Py=Py.data_ptr(),
                           r_stop=float(r_stop), J_factor=float(J_factor), tol=float(tol), max_iter=int(max_iter),
                           infinite=1 if infinite else 0, status=status.data_ptr())
    sfx = _DTYPES[x.dtype]
    with torch.cuda.device(dtab.device):
        stream = torch.cuda.current_stream(dtab.device).cuda_stream
        rc = getattr(dtab.lib, f"olb_aim_{sfx}")(C.byref(dtab.c), C.byref(call), C.c_void_p(stream))
    _lib.check(rc, f"olb_aim_{sfx}")
    return status


def _aligned(t):
    """Contiguous and 16-byte aligned (a slice of a larger tensor may start anywhere; the C ABI wants aligned arrays)."""
    if t is None:
        return None
    t = t.contiguous()
    return t.clone() if t.data_ptr() % 16 else t


def _c_launch(affine: dict, Px, Py):
    la = _lib.OlbPupilLaunch()
    la.Px, la.Py = Px.data_ptr(), Py.data_ptr()
    la.origin0 = (C.c_double * 3)(*affine["origin0"])
    la.origin_scale = (C.c_double * 2)(*affine["origin_scale"])
    la.target0 = (C.c_double * 3)(*affine["target0"])
    la.target_scale = (C.c_double * 2)(*affine["target_scale"])
    la.intensity = float(affine.get("intensity", 1.0))
    fields = affine.get("fields")
    if fields is not None:      # per-ray field coordinates (Hx, Hy device arrays): launch.pupil_affine_fields
        Hx, Hy = fields
        la.Hx, la.Hy = Hx.data_ptr(), Hy.data_ptr()
        la.field_mode = int(affine["field_mode"])
        la.field_arg = float(affine.get("field_arg", 0.0))
        la.origin_field = (C.c_double * 2)(*affine["origin_field"])
        la.target_field = (C.c_double * 2)(*affine["target_field"])
        vig = affine.get("vig")
        if vig is not None:        # ((n, 4) array of {Hx, Hy, vx, vy} of the defined fields, power): in-kernel lookup
            tab, power = vig
            tab = np.asarray(tab, dtype=np.float64).reshape(-1, 4)
            if len(tab) > 16:
                raise ValueError("more than 16 defined fields with vignetting factors")
            la.n_vig, la.vig_power = len(tab), int(power)
            for j, row in enumerate(tab):
                for q in range(4):
                    la.vig[j][q] = float(row[q])
    return la


def trace_pupil_device(dtab: DeviceTable, Px: torch.Tensor, Py: torch.Tensor, affine: dict, first: int, last: int,
                       wavelength: torch.Tensor | None = None, polarization=False):
    """Launch state generated in-kernel from pupil coordinates (OlbTraceCall.launch, one field or per-ray fields),
    full records.  Returns (rays, records): ``rays`` is a ``RealRays`` view of the last record row.

    ``polarization`` (config 5's call shape): False = RealRays; otherwise PolarizedRays are
    traced -- "matrix": only the P matrices (``rays.p``); None / "unpolarized" / (Ex, Ey, phase_x, phase_y): also the
    intensity epilogue of RealRayTracer.trace in-kernel, ``rays.i`` = sum |P E0|^2 i0 / n_states (the record rows keep
    the geometric intensity, as in the reference)."""
    Px, Py, wavelength = _aligned(Px), _aligned(Py), _aligned(wavelength)
    if affine.get("fields") is not None:
        affine = dict(affine, fields=tuple(_aligned(t) for t in affine["fields"]))
    n, dtype, dev = Px.numel(), Px.dtype, Px.device
    buf = _out_buffer(8, last - first, n, dtype, dev)
    recs = {k: buf[j, :, :n] for j, k in enumerate(_REC_KEYS)}
    la = _c_launch(affine, Px.contiguous(), Py.contiguous())
    out = _lib.OlbRays(w=wavelength.data_ptr() if (wavelength is not None and dtab.table.n_wl > 1) else None)
    flags = _lib.TF_NO_FINAL
    p, inten, c_pol = None, None, None
    if polarization is not False:
        flags |= _lib.TF_POLARIZED
        p = torch.empty((n, 3, 3), dtype=_CDTYPES[dtype], device=dev)
        out.p = torch.view_as_real(p).data_ptr()
        if polarization != "matrix":
            inten = torch.empty(n, dtype=dtype, device=dev)
            c_pol = _c_polarization(polarization, inten)
    _trace(dtab, dev, dtype, first, last, n, flags, rays=out, rec=_c_records(buf), launch=la, pol=c_pol)
    cls = RealRays if p is None else PolarizedRays
    rays = _take_last_row(cls.__new__(cls), recs)
    if p is not None:
        rays.p = p
    if inten is not None:
        rays.i = inten
    rays.w = wavelength
    rays.L0 = rays.M0 = rays.N0 = None
    rays.is_normalized = True
    return rays, recs


WAVEFRONT_KEYS = ("opd", "pupil_x", "pupil_y", "pupil_z", "intensity")


def trace_wavefront_device(dtab: DeviceTable, Px: torch.Tensor, Py: torch.Tensor, affine: dict, ref: dict,
                           wavelength: torch.Tensor | None = None, polarized: bool = False) -> dict:
    """Trace one field's pupil grid and write ONLY the wavefront data (OlbTraceCall.wavefront_*) -- OPD in waves
    against the spherical reference ``ref`` = {center (3), radius, n_image, tilt (2), opd_ref, wavelength_um},
    the exit-pupil intercepts and the image-surface intensity -- no records, no final state
    (optiland/wavefront/strategy.py:152-213).  Returns {key: (N,) tensor} for WAVEFRONT_KEYS."""
    Px, Py, wavelength = _aligned(Px), _aligned(Py), _aligned(wavelength)
    n, dtype, dev = Px.numel(), Px.dtype, Px.device
    buf = _out_buffer(5, 1, n, dtype, dev)[:, 0]
    c_out = _lib.OlbWavefrontOut(*[buf[j].data_ptr() for j in range(5)])
    c_ref = _lib.OlbWavefrontRef()
    c_ref.center = (C.c_double * 3)(*[float(v) for v in ref["center"]])
    c_ref.radius, c_ref.n_image = float(ref["radius"]), float(ref["n_image"])
    c_ref.tilt = (C.c_double * 2)(*[float(v) for v in ref.get("tilt", (0.0, 0.0))])
    c_ref.opd_ref, c_ref.wavelength_um = float(ref["opd_ref"]), float(ref["wavelength_um"])
    la = _c_launch(affine, Px.contiguous(), Py.contiguous())
    rays = _lib.OlbRays(w=wavelength.data_ptr() if (wavelength is not None and dtab.table.n_wl > 1) else None)
    flags = _lib.TF_NO_FINAL
    p = None
    if polarized:
        # PolarizedRays through the wavefront epilogue (config 5).  The strategy reads the GEOMETRIC intensity
        # of the image-surface record (wavefront/strategy.py:181) -- no intensity epilogue -- and hands the
        # polarization ray-tracing matrices on (strategy.py:197-203): `p` is written, 5 + 18 values per ray.
        flags |= _lib.TF_POLARIZED
        p = torch.empty((n, 3, 3), dtype=_CDTYPES[dtype], device=dev)
        rays.p = torch.view_as_real(p).data_ptr()
    _trace(dtab, dev, dtype, 0, dtab.table.num_surfaces, n, flags, rays=rays, launch=la, wavefront=(c_ref, c_out))
    out = {k: buf[j, :n] for j, k in enumerate(WAVEFRONT_KEYS)}
    if p is not None:
        out["p"] = p
    return out


def trace_moments_device(dtab: DeviceTable, n: int, dtype, rays: RealRays | None = None, pupil=None,
                         center=(0.0, 0.0), moments: torch.Tensor | None = None, wavelength=None,
                         status: torch.Tensor | None = None, last: int | None = None, global_xy: bool = False,
                         every_ray: bool = False) -> torch.Tensor:
    """Trace WITHOUT writing any per-ray output and accumulate the spot / OPD moments of the image-surface
    intercepts in-kernel (8 fp64 values on the device; include/olb.h, OlbTraceCall.moments).  Either
    ``rays`` (launch-state arrays, left untouched) or ``pupil`` = (Px, Py, affine).  ``last``: stop after surface
    ``last - 1`` (the moments are of THAT surface); ``global_xy`` / ``every_ray``: OLB_TF_MOMENTS_GLOBAL / _ALL.  ``status``: a caller-owned
    device int32 for the OLB_ST_* bits (a caller that pipelines several launches checks it once at the end with
    ``_raise_status``); by default one is made and checked here for tables that can raise them."""
    dev = dtab.device
    if moments is None:
        moments = torch.zeros(8, dtype=torch.float64, device=dev)
    la = None
    c_rays = _lib.OlbRays()
    if pupil is not None:
        Px, Py, affine = pupil
        Px, Py, wavelength = _aligned(Px), _aligned(Py), _aligned(wavelength)
        la = _c_launch(affine, Px, Py)
        if wavelength is not None and dtab.table.n_wl > 1:
            c_rays.w = wavelength.data_ptr()
    else:
        # the launch arrays are only read (OLB_TF_NO_FINAL): nothing is written back
        for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
            setattr(c_rays, k, getattr(rays, k).data_ptr())
        if dtab.table.n_wl > 1:
            c_rays.w = rays.w.data_ptr()
    flags = _lib.TF_NO_FINAL | (_lib.TF_MOMENTS_GLOBAL if global_xy else 0) | (_lib.TF_MOMENTS_ALL if every_ray else 0)
    _trace(dtab, dev, dtype, 0, dtab.table.num_surfaces if last is None else last, n, flags, rays=c_rays, launch=la,
           center=center, moments=moments, status=status, own_status=status is None)
    return moments


def moments_to_spot(m, center=(0.0, 0.0)) -> dict:
    """count, centroid, RMS radius about the centroid and about ``center``, mean intensity, OPD mean / rms."""
    m = [float(v) for v in (m.cpu() if torch.is_tensor(m) else m)]
    cnt = m[0]
    if cnt == 0:
        return {"count": 0.0}
    mx, my = m[1] / cnt, m[2] / cnt
    var_c = max(m[3] / cnt - mx * mx - my * my, 0.0)
    opd_mean = m[5] / cnt
    return {"count": cnt, "centroid": (center[0] + mx, center[1] + my), "rms_centroid": var_c ** 0.5,
            "rms_center": (m[3] / cnt) ** 0.5, "intensity_sum": m[4], "opd_mean": opd_mean,
            "opd_rms": max(m[6] / cnt - opd_mean * opd_mean, 0.0) ** 0.5}


class SurfaceGroup:
    """The traced part of the reference's ``SurfaceGroup``: ``trace`` + stacked records."""

    def __init__(self, table: T.SurfaceTable, device=None):
        self.table = table
        self.device_table = DeviceTable(table, device)
        self._rec = None

    @property
    def num_surfaces(self) -> int:
        return self.table.num_surfaces

    def trace(self, rays: RealRays, skip: int = 0, stop: int | None = None, record: bool = True):
        """``SurfaceGroup.trace(rays, skip)`` (surface_group.py:245-257); ``stop`` bounds the range
        (exclusive) for the per-surface callers (ray_aiming/iterative.py:366)."""
        last = self.num_surfaces if stop is None else stop
        if not 0 <= skip <= last <= self.num_surfaces:
            raise ValueError("bad surface range")
        self._rec = trace_device(self.device_table, rays, skip, last, record=record)
        return rays

    def trace_pupil(self, Px, Py, affine: dict, wavelength=None):
        """``Optic.trace`` for one field without materialising the launch arrays: pupil coordinates in,
        the launch state (paraxial aiming, optiland/rays/ray_aiming/paraxial.py:33-106) is evaluated
        in-kernel.  ``affine``: see ``optiland_b200.launch.pupil_affine_infinite_angle``."""
        rays, self._rec = trace_pupil_device(self.device_table, Px, Py, affine, 0, self.num_surfaces, wavelength)
        return rays

    def spot_moments(self, rays=None, pupil=None, center=(0.0, 0.0), dtype=None):
        """Fused trace + spot/OPD moments (no per-ray output at all); see ``trace_moments_device``.

        ``rms_centroid`` comes from a second launch whose moments are taken about the first one's centroid: the
        one-pass ``m3/n - mx^2 - my^2`` about ``center`` cancels the spot's offset from it (a micrometre spot 20 mm off
        axis keeps only a few digits), as ``spot.py`` avoids for SpotDiagram."""
        if pupil is not None:
            n, dt = pupil[0].numel(), pupil[0].dtype
        else:
            n, dt = len(rays), rays.dtype
        m = trace_moments_device(self.device_table, n, dtype or dt, rays=rays, pupil=pupil, center=center)
        out = moments_to_spot(m, center)
        cen = out.get("centroid")
        if cen is not None and np.isfinite(cen[0]) and np.isfinite(cen[1]):
            m2 = trace_moments_device(self.device_table, n, dtype or dt, rays=rays, pupil=pupil, center=cen)
            out["rms_centroid"] = moments_to_spot(m2, cen)["rms_centroid"]
        return out

    def _get(self, key):
        if self._rec is None:
            raise RuntimeError("no records: call trace(..., record=True) first")
        return self._rec[key]

    x = property(lambda self: self._get("x"))
    y = property(lambda self: self._get("y"))
    z = property(lambda self: self._get("z"))
    L = property(lambda self: self._get("L"))
    M = property(lambda self: self._get("M"))
    N = property(lambda self: self._get("N"))
    opd = property(lambda self: self._get("opd"))
    intensity = property(lambda self: self._get("intensity"))


def trace_host(dtab: DeviceTable, h_in: dict, h_out: dict, n: int, dtype=torch.float32, chunk: int = 1 << 20,
               scratch: torch.Tensor | None = None, rec=None, first: int = 0, last: int | None = None,
               affine: dict | None = None):
    """olb_trace_host_*: HOST SoA in (pinned tensors x,y,z,L,M,N,i[,w]) -> HOST final state out
    (x,y,z,L,M,N,i,opd); chunks are pipelined H2D / kernel / D2H on three streams.  With ``affine`` the host
    pupil arrays h_in["Px"], h_in["Py"] go in instead (8 B/ray over PCIe) and the launch state is generated on
    the device."""
    lib = dtab.lib
    sfx = _DTYPES[dtype]
    es = 4 if dtype == torch.float32 else 8
    last = dtab.table.num_surfaces if last is None else last
    dtab.ready.synchronize()        # the library's copy / compute streams are not ordered behind the upload's stream
    need = int(lib.olb_host_scratch_bytes(es, chunk))
    if scratch is None or scratch.numel() < need:
        scratch = torch.empty(need, dtype=torch.uint8, device=dtab.device)
    c_out = _lib.OlbRays(**{k: h_out[k].data_ptr() for k in ("x", "y", "z", "L", "M", "N", "i", "opd")})
    la, c_in = None, None
    if affine is not None:
        la = _c_launch(affine, h_in["Px"], h_in["Py"])
        if dtab.table.n_wl > 1:
            # (pupil launch: the per-ray wavelengths travel in h_out.w -- include/olb.h, olb_trace_host_*)
            c_out.w = (h_in["w"] if "w" in h_in else h_out["w"]).data_ptr()
    else:
        c_in = _lib.OlbRays(**{k: h_in[k].data_ptr() for k in ("x", "y", "z", "L", "M", "N", "i")},
                            w=h_in["w"].data_ptr() if "w" in h_in and dtab.table.n_wl > 1 else None)
    c_rec = _c_records(rec) if rec is not None else None
    # BSDF tables: the attempt bound's status bit (the other OLB_ST_* bits are not collected on this path)
    status = torch.zeros(1, dtype=torch.int32, device=dtab.device) if _has_bsdf(dtab) else None
    with torch.cuda.device(dtab.device):
        rc = getattr(lib, f"olb_trace_host_{sfx}")(
            C.byref(dtab.c), first, last, _byref(la), _byref(c_in), C.byref(c_out), _byref(c_rec), n, chunk,
            C.c_void_p(scratch.data_ptr()), scratch.numel(), 0,
            C.c_void_p(status.data_ptr()) if status is not None else None)
    _lib.check(rc, f"olb_trace_host_{sfx}")
    _raise_status(status)
    return scratch
