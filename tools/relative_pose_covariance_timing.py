"""Wall clock of ctvio_relative_pose_covariance at C2 and C4 (gauge_knot_index 3 on windows whose options fix no knots,
as the streaming window's solve does; camera frame) for n = 1, 10 and 1024 pairs (t, t + 100 ms), the spacing of
consecutive keyframes, next to ctvio_covariance without outputs: the formation of Sigma the call shares.  The host route
the call replaces, ctvio_covariance with the np x np matrix copied back and then the same 6 x 36 projection over each
pair's union in numpy, runs once per n, with its Jacobians already at hand (random matrices of the right shape, built
outside the clock), so it is a lower bound.  Each call ends in a stream synchronise, so the host clock around it is its
time.  A separate traced run (torch.profiler) of the n = 1024 call gives relative_pose_cov_kernel's device time.  The
card name and power limit are read in the same run.
Usage: python tools/relative_pose_covariance_timing.py [--reps N] [--out file.json]"""
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

GAP_NS = 100_000_000  # consecutive keyframes of the streaming window


def kernel_us(f):
    """device time (us) of relative_pose_cov_kernel in one traced call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        f()
        torch.cuda.synchronize()
    return sum(ev.time_range.elapsed_us() for ev in prof.events()
               if ev.device_type == torch.autograd.DeviceType.CUDA and "relative_pose_cov_kernel" in ev.name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = pkg.load()
    rng = np.random.default_rng(0)
    res = {"card": card(), "reps": a.reps, "cases": {}}
    for name, w in (("C2", syn.config_c2()), ("C4", syn.config_c4())):
        fixed = pkg.make_options(fixed_knot_index=3, fix_ld=w.fix_ld, ld_lower=w.ld_lower, ld_upper=w.ld_upper)
        free = pkg.make_options(fixed_knot_index=-1, fix_ld=w.fix_ld, ld_lower=w.ld_lower, ld_upper=w.ld_upper)
        est = pkg.setup_estimator(lib, w, options=fixed)
        est.Solve(15)
        nK = est.n_knots
        t_end = w.t0_ns + (nK - 3) * w.dt_ns
        sigma = time_calls(lambda: est.Covariance(want_cc=False, want_rho=False), a.reps)  # fixed knots 0..3
        row = {}
        for n in (1, 10, 1024):
            ta = (np.linspace(w.t0_ns, t_end - 1 - GAP_NS, n).astype(np.int64) if n > 1
                  else np.array([t_end - 1 - GAP_NS], np.int64))
            tb = ta + GAP_NS
            sa, sb = (ta - w.t0_ns) // w.dt_ns, (tb - w.t0_ns) // w.dt_ns
            assert (sb - sa == 2).all()  # every union: knots sa .. sa + 5
            idx = 6 * sa[:, None] + np.arange(36)[None, :]
            G = rng.standard_normal((n, 6, 36))
            est.SetOptions(free)
            call = lambda: est.RelativePoseCovariance(ta, tb, gauge_knot_index=3, camera_frame=True)  # noqa: E731
            dev = time_calls(call, a.reps)
            _, _, rcond = call()
            us = kernel_us(call) if n == 1024 else None

            def host_route():
                cov = est.Covariance(want_rho=False)[0]
                S = cov[idx[:, :, None], idx[:, None, :]]
                return G @ S @ G.transpose(0, 2, 1)
            # the options fix knots 0..3 for the host route (ctvio_covariance has no gauge argument)
            est.SetOptions(fixed)
            host = time_calls(host_route, 1)
            row[n] = dict(ms_relative_pose_covariance=dev, ms_covariance_plus_numpy=host[0], rcond=rcond,
                          us_relative_pose_cov_kernel=us)
            print(f"{name} n {n:5d}: ctvio_relative_pose_covariance {dev[0]:.3f} ms median (min {dev[1]:.3f}, max "
                  f"{dev[2]:.3f}); covariance without outputs {sigma[0]:.3f} ms median; ctvio_covariance + numpy "
                  f"projection {host[0]:.3f} ms (one run); rcond {rcond:.2e}"
                  + ("" if us is None else f"; traced relative_pose_cov_kernel {us:.1f} us"))
        res["cases"][name] = dict(np=est.np_dim, n_lm=est.n_lm, ms_covariance_without_outputs=sigma, n=row)
    print("card (name, power limit, max SM clock):", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
