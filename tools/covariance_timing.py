"""Wall clock of ctvio_covariance at C2 and C4 (fixed_knot_index 3: the windows have no prior, so the gauge is fixed by
knots), with and without the outputs copied back, next to one LM solve of the same window.  The call ends in a stream
synchronise, so the host clock around it is the call's time; the card name and power limit are read in the same run.
Usage: python tools/covariance_timing.py [--reps N] [--out file.json]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("ctrl-vio_b200")
syn = pkg.synthetic


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def time_calls(f, reps):
    for _ in range(3):
        f()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), float(np.min(t)), float(np.max(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = pkg.load()
    res = {"card": card(), "reps": a.reps, "cases": {}}
    for name, w in (("C2", syn.config_c2()), ("C4", syn.config_c4())):
        opt = pkg.make_options(fixed_knot_index=3, fix_ld=w.fix_ld, ld_lower=w.ld_lower, ld_upper=w.ld_upper)
        est = pkg.setup_estimator(lib, w, options=opt)
        est.Solve(15)
        full = time_calls(lambda: est.Covariance(), a.reps)
        none = time_calls(lambda: est.Covariance(want_cc=False, want_rho=False), a.reps)
        _, _, rcond = est.Covariance(want_cc=False, want_rho=False)
        s = est.Solve(1)
        res["cases"][name] = dict(np=est.np_dim, n_lm=est.n_lm, rcond=rcond, ms_with_outputs=full, ms_without_outputs=none,
                                  solve1_device_ms=s.device_ms)
        print(f"{name}: np {est.np_dim}, nL {est.n_lm}, rcond {rcond:.2e}: covariance {full[0]:.3f} ms median "
              f"(min {full[1]:.3f}, max {full[2]:.3f}) with outputs, {none[0]:.3f} ms without; "
              f"one LM iteration {s.device_ms:.3f} ms on device")
    print("card (name, power limit, max SM clock):", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
