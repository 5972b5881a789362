"""Measure what the fp32 arithmetic of the trace kernel achieves on the Forbes Q-2D fixtures (tests/golden/forbes_q2d/*.npz)
against the reference's fp64 records, on the CPU instantiation of the device math (tests/hostcheck/hostcheck_forbes_q2d.cpp) and, when a GPU is
present, on the fp32 kernel itself (the larger of the two per quantity), and write tests/golden/forbes_q2d/f32_achieved.json
(or --out).  The parity tests assert the fp32 kernel within 3x of these numbers.

    python scripts/f32_achieved_forbes_q2d.py [--out PATH]
"""
from __future__ import annotations

import glob
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.hostcheck_forbes_q2d import run_hostcheck_forbes_q2d  # noqa: E402
from tests._util import GOLDEN, REC, Case, fp32_errors  # noqa: E402


def measure(name: str) -> dict:
    c = Case(name)
    pmat = None
    if "out_p" in c.z:
        pmat = np.tile(np.eye(3, dtype=np.complex64), (c.n, 1, 1))
    out, rec, _ = run_hostcheck_forbes_q2d(c.table, c.rays, np.float32, pmat=pmat)
    got = fp32_errors(rec, c.rec)
    if pmat is not None:
        got["p"] = float(np.nanmax(np.abs(out["p"].astype(np.complex128) - c.out["p"])))
    for k, v in measure_kernel(c).items():
        got[k] = max(got[k], v)
    return got


def measure_kernel(c) -> dict:
    """The same errors of the H100 kernel (empty without a GPU)."""
    import torch

    if not torch.cuda.is_available():
        return {}
    from optiland_b200.trace import PolarizedRays, RealRays, SurfaceGroup

    r = c.rays
    cls = PolarizedRays if "out_p" in c.z else RealRays
    rays = cls(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=torch.float32)
    sg = SurfaceGroup(c.table)
    sg.trace(rays)
    got = fp32_errors({k: getattr(sg, k).double().cpu().numpy() for k in REC}, c.rec)
    if "out_p" in c.z:
        got["p"] = float(np.nanmax(np.abs(rays.p.to(torch.complex128).cpu().numpy() - c.out["p"])))
    return got


def main():
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(GOLDEN, "forbes_q2d", "f32_achieved.json"))
    args = ap.parse_args()
    names = sorted("forbes_q2d/" + os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "forbes_q2d", "*.npz")))
    cases = {n.split("/", 1)[1]: measure(n) for n in names}
    doc = {"source": "fp32: the larger of the CPU instantiation of the device arithmetic and the H100 kernel, vs the "
                     "reference's fp64 records; max |error| of intercepts (mm), OPD (mm), direction cosines, intensity, "
                     "P-matrix entries",
           "cases": cases}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(doc, f, indent=1, sort_keys=True)
        f.write("\n")
    for k, v in cases.items():
        print(k, v)


if __name__ == "__main__":
    main()
