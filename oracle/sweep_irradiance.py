"""pytest plugin (TEST INFRASTRUCTURE), loaded after ``oracle.sweep_plugin``: prints the number of irradiance-binning calls
the installed engine served on a line of its own, ``[olb sweep] irradiance calls: N``."""
from oracle import sweep_plugin


def pytest_terminal_summary(terminalreporter):
    eng = sweep_plugin.ENGINE
    if eng is not None:
        n = sum(1 for c in eng.calls if c and c[0] == "irradiance")
        terminalreporter.write_line(f"[olb sweep] irradiance calls: {n}")
