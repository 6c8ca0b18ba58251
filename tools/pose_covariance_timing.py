"""Wall clock of ctvio_pose_covariance at C2 and C4 (gauge_knot_index 3 on windows whose options fix no knots, as the
streaming window's solve does) for n = 1, 64 and 1024 query times, next to the host route it replaces:
ctvio_covariance with the np x np matrix copied back, then the same 12 x 24 projection in numpy.  The host route is
timed with its Jacobians already at hand (random matrices of the right shape, built outside the clock), so it is a
lower bound: a real caller would also have to evaluate the spline Jacobians on the host.  Both calls end in a stream
synchronise, so the host clock around them is their time; the card name and power limit are read in the same run.
Usage: python tools/pose_covariance_timing.py [--reps N] [--out file.json]"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("ctrl-vio_b200")
syn = pkg.synthetic
from covariance_timing import card, time_calls  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = pkg.load()
    rng = np.random.default_rng(0)
    res = {"card": card(), "reps": a.reps, "cases": {}}
    for name, w in (("C2", syn.config_c2()), ("C4", syn.config_c4())):
        opt = pkg.make_options(fixed_knot_index=3, fix_ld=w.fix_ld, ld_lower=w.ld_lower, ld_upper=w.ld_upper)
        est = pkg.setup_estimator(lib, w, options=opt)
        est.Solve(15)
        est.SetOptions(pkg.make_options(fixed_knot_index=-1, fix_ld=w.fix_ld, ld_lower=w.ld_lower,
                                        ld_upper=w.ld_upper))
        nK = est.n_knots
        t_end = w.t0_ns + (nK - 3) * w.dt_ns
        row = {}
        for n in (1, 64, 1024):
            t = np.linspace(w.t0_ns, t_end - 1, n).astype(np.int64) if n > 1 else np.array([t_end - 50_000_000])
            seg = (t - w.t0_ns) // w.dt_ns
            J = rng.standard_normal((n, 12, 24))
            dev = time_calls(lambda: est.PoseCovariance(t, gauge_knot_index=3, camera_frame=True), a.reps)
            _, rcond = est.PoseCovariance(t, gauge_knot_index=3, camera_frame=True)

            def host_route():
                cov = est.Covariance(want_rho=False)[0]
                idx = 6 * seg[:, None] + np.arange(24)[None, :]
                S = cov[idx[:, :, None], idx[:, None, :]]
                return J @ S @ J.transpose(0, 2, 1)
            # the options fix knots 0..3 for the host route (ctvio_covariance has no gauge argument)
            est.SetOptions(opt)
            host = time_calls(host_route, a.reps)
            est.SetOptions(pkg.make_options(fixed_knot_index=-1, fix_ld=w.fix_ld, ld_lower=w.ld_lower,
                                            ld_upper=w.ld_upper))
            row[n] = dict(ms_pose_covariance=dev, ms_covariance_plus_numpy=host, rcond=rcond)
            print(f"{name} n {n:5d}: ctvio_pose_covariance {dev[0]:.3f} ms median (min {dev[1]:.3f}, max {dev[2]:.3f}); "
                  f"ctvio_covariance + numpy projection {host[0]:.3f} ms (min {host[1]:.3f}); rcond {rcond:.2e}")
        res["cases"][name] = dict(np=est.np_dim, n_lm=est.n_lm, n=row)
    print("card (name, power limit, max SM clock):", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
