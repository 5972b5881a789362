"""TEST INFRASTRUCTURE ONLY -- a stand-in for optiland_b200.plugin.CudaEngine on boxes without a GPU that also traces
thin-film, polarizer and retarder coatings: the call shapes of ``oracle/phase_engines._PhaseEngine`` (trace, fused
pupil launch, spot moments, wavefront) with the trace done by the DEVICE ARITHMETIC compiled for the host with the
kernel variant the launcher picks for such tables (``oracle/hostcheck_coating.py``,
tests/hostcheck/hostcheck_coating.cpp).  Phase-profile and ruled-grating tables take the same dispatch."""
from oracle.phase_engines import PhaseDeviceMathEngine


class CoatingDeviceMathEngine(PhaseDeviceMathEngine):
    """TEST-ONLY: the kernel's own arithmetic on the CPU, thin-film / polarizer / retarder coatings included."""

    def _core(self, table, inp, first, last, pmat):
        import numpy as np

        from oracle.hostcheck_coating import run_hostcheck_coating

        return run_hostcheck_coating(table, inp, np.float64, first, last, pmat=pmat)
