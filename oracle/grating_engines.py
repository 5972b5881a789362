"""TEST INFRASTRUCTURE ONLY -- stand-ins for optiland_b200.plugin.CudaEngine on boxes without a GPU that also trace
ruled gratings (``DiffractiveInteractionModel``) and phase-profile surfaces: the call shapes of
``oracle/phase_engines._PhaseEngine`` (trace, fused pupil launch, spot moments, wavefront), with the trace done by

``GratingOracleEngine``      the NumPy restatement (``oracle/grating_oracle.py`` on top of ``oracle/phase_oracle.py``);
``GratingDeviceMathEngine``  the DEVICE ARITHMETIC compiled for the host with the kernel variants the launcher picks
                             for grating tables (``oracle/hostcheck_grating.py``, tests/hostcheck/hostcheck_grating.cpp).

The plain ``OracleEngine`` / ``DeviceMathEngine`` ignore ``SurfaceSpec.interaction``: a CPU test that traces live
grating objects through the plugin must install one of these."""
from oracle.phase_engines import PhaseDeviceMathEngine, PhaseOracleEngine


class GratingOracleEngine(PhaseOracleEngine):
    """TEST-ONLY: the NumPy restatement of the reference, ruled gratings and phase-profile surfaces included."""

    def _core(self, table, inp, first, last, pmat):
        from oracle import grating_oracle

        if pmat is not None:
            inp = dict(inp, p=pmat)
        return grating_oracle.trace(table, inp, first, last, polarized=pmat is not None)


class GratingDeviceMathEngine(PhaseDeviceMathEngine):
    """TEST-ONLY: the kernel's own arithmetic on the CPU, ruled gratings and phase-profile surfaces included."""

    def _core(self, table, inp, first, last, pmat):
        import numpy as np

        from oracle.hostcheck_grating import run_hostcheck_grating

        return run_hostcheck_grating(table, inp, np.float64, first, last, pmat=pmat)
