"""Wall clock of ctvio_point_covariance at C2 and C4 for every landmark of the window (gauge_knot_index 3 on windows
whose options fix no knots, as the streaming window's solve does), next to ctvio_covariance without outputs: the
formation of Sigma the call shares.  Each call ends in a stream synchronise, so the host clock around it is its time.
The call always copies its n x 9 result back; a separate traced run (torch.profiler) splits one call's device time
into point_cov_kernel and the device-to-host copy, so the time without the copy back is the host clock minus that
copy.  The card name and power limit are read in the same run.
Usage: python tools/point_covariance_timing.py [--reps N] [--out file.json]"""
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


def trace_call(f):
    """device time (us) of the point kernel and of the device-to-host copies of one call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        f()
        torch.cuda.synchronize()
    out = dict(us_point_cov_kernel=0.0, us_copy_back=0.0)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "point_cov_kernel" in ev.name:
            out["us_point_cov_kernel"] += ev.time_range.elapsed_us()
        elif "DtoH" in ev.name or "Device -> Pageable" in ev.name or "D2H" in ev.name:
            out["us_copy_back"] += ev.time_range.elapsed_us()
    return out


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
        nL, nK = est.n_lm, est.n_knots
        t_end = w.t0_ns + (nK - 3) * w.dt_ns
        lm = np.arange(nL, dtype=np.int32)
        t = rng.integers(w.t0_ns, t_end, nL).astype(np.int64)
        b = rng.uniform(-0.4, 0.4, (nL, 2))
        sigma = time_calls(lambda: est.Covariance(want_cc=False, want_rho=False), a.reps)  # fixed knots 0..3
        est.SetOptions(free)
        call = lambda: est.PointCovariance(lm, t, b, gauge_knot_index=3)  # noqa: E731
        point = time_calls(call, a.reps)
        _, rcond = call()
        traced = trace_call(call)
        res["cases"][name] = dict(np=est.np_dim, n_lm=nL, rcond=rcond, ms_point_covariance=point,
                                  ms_covariance_without_outputs=sigma, **traced)
        print(f"{name}: np {est.np_dim}, n = nL = {nL}, rcond {rcond:.2e}: point covariance {point[0]:.3f} ms median "
              f"(min {point[1]:.3f}, max {point[2]:.3f}); covariance without outputs {sigma[0]:.3f} ms median; traced "
              f"point_cov_kernel {traced['us_point_cov_kernel']:.1f} us, copy back {traced['us_copy_back']:.1f} us")
    print("card (name, power limit, max SM clock):", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
