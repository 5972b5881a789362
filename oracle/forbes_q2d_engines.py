"""TEST INFRASTRUCTURE ONLY -- stand-ins for optiland_b200.plugin.CudaEngine on boxes without a GPU that also trace
Forbes Q-2D surfaces (Optiland's ``ForbesQ2dGeometry``), with the call shapes of ``oracle/phase_engines._PhaseEngine``
(trace, fused pupil launch, spot moments, wavefront):

* ``Q2dOracleEngine``: the NumPy restatement (``oracle/forbes_q2d_oracle.py``);
* ``Q2dDeviceMathEngine``: the DEVICE ARITHMETIC compiled for the host with the two kernel variants the launcher picks for
  Q-2D tables (``oracle/hostcheck_forbes_q2d.py``, tests/hostcheck/hostcheck_forbes_q2d.cpp).

Neither is differentiable: a Q-2D table has no adjoint, so gradient traces decline to the reference's eager path."""
import numpy as np

from oracle.phase_engines import PhaseDeviceMathEngine, PhaseOracleEngine


class Q2dOracleEngine(PhaseOracleEngine):
    """TEST-ONLY: the NumPy restatement of the reference, Q-2D surfaces included."""

    def _core(self, table, inp, first, last, pmat):
        from oracle import forbes_q2d_oracle

        if pmat is not None:
            inp = dict(inp, p=pmat)
        return forbes_q2d_oracle.trace(table, inp, first, last, polarized=pmat is not None)


class Q2dDeviceMathEngine(PhaseDeviceMathEngine):
    """TEST-ONLY: the kernel's own arithmetic on the CPU, Q-2D surfaces included."""

    def _core(self, table, inp, first, last, pmat):
        from oracle.hostcheck_forbes_q2d import run_hostcheck_forbes_q2d

        return run_hostcheck_forbes_q2d(table, inp, np.float64, first, last, pmat=pmat)
