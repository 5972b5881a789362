"""Measure what the fp32 arithmetic ACHIEVES against the reference's fp64 goldens, per fixture: max |error| of
intercepts (x, y, z), OPD and direction cosines over all record rows.  `tests/golden/f32_achieved.json` holds the
larger of the CPU instantiation of the device math (tests/hostcheck; IEEE sqrt / div) and the H100 kernel (MUFU
approximations); the parity tests assert <= 3x these numbers.

    python scripts/f32_achieved.py                            # host arithmetic (no GPU needed)
    python scripts/f32_achieved.py --gpu f32_achieved_gpu.json  # the kernel, on the GPU (writes the given file)
    python scripts/f32_achieved.py --merge f32_achieved_gpu.json  # fold a GPU measurement in
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "f32_achieved.json")


def errors(rec, want):
    out = {}
    for tag, keys in (("pos", ("x", "y", "z")), ("opd", ("opd",)), ("dir", ("L", "M", "N")), ("intensity", ("intensity",))):
        w = 0.0
        for k in keys:
            a, b = np.asarray(rec[k], dtype=np.float64), want[k]
            m = np.isfinite(a) & np.isfinite(b)
            if m.any():
                w = max(w, float(np.max(np.abs(a[m] - b[m]))))
        out[tag] = w
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", metavar="OUT", default=None)
    ap.add_argument("--merge", default=None)
    args = ap.parse_args()
    from tests._util import POLARIZED_CASES, REAL_CASES, Case

    if args.merge:
        cur = json.load(open(OUT))
        new = json.load(open(args.merge))
        for name, e in new["cases"].items():
            c = cur["cases"].setdefault(name, e)
            for k, v in e.items():
                c[k] = max(c.get(k, 0.0), v)
        cur["sources"] = sorted(set(cur.get("sources", [])) | set(new.get("sources", [])))
        json.dump(cur, open(OUT, "w"), indent=1, sort_keys=True)
        print("merged", args.merge)
        return
    res = {}
    if args.gpu:
        import torch

        from optiland_b200.trace import PolarizedRays, RealRays, SurfaceGroup

        for name in REAL_CASES + POLARIZED_CASES:
            c = Case(name)
            r = c.rays
            cls = PolarizedRays if name in POLARIZED_CASES else RealRays
            rays = cls(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=torch.float32)
            sg = SurfaceGroup(c.table)
            sg.trace(rays)
            rec = {k: getattr(sg, k).double().cpu().numpy() for k in ("x", "y", "z", "L", "M", "N", "opd", "intensity")}
            res[name] = errors(rec, c.rec)
            if name in POLARIZED_CASES:
                res[name]["p"] = float(np.max(np.abs(rays.p.cpu().numpy().astype(np.complex128) - c.out["p"])))
        path = args.gpu
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        json.dump({"cases": res, "sources": [f"{torch.cuda.get_device_name()} kernel (olb_trace_call_f32)"]}, open(path, "w"),
                  indent=1, sort_keys=True)
        print("wrote", path)
    else:
        from oracle.hostcheck_api import load, run_hostcheck

        hc = load()
        for name in REAL_CASES + POLARIZED_CASES:
            c = Case(name)
            pm = np.tile(np.eye(3, dtype=np.complex128), (c.n, 1, 1)) if name in POLARIZED_CASES else None
            out, rec, _ = run_hostcheck(hc, c.table, c.rays, np.float32, pmat=pm)
            res[name] = errors(rec, c.rec)
            if pm is not None:
                res[name]["p"] = float(np.max(np.abs(out["p"].astype(np.complex128) - c.out["p"])))
        json.dump({"cases": res, "sources": ["host instantiation of the device math (tests/hostcheck)"],
                   "unit": "mm (pos, opd), 1 (dir, intensity, p)"}, open(OUT, "w"), indent=1, sort_keys=True)
        print("wrote", OUT)
    for k, v in res.items():
        print(f"{k:28s} " + " ".join(f"{a}={b:.2e}" for a, b in v.items()))


if __name__ == "__main__":
    main()
