"""Host-side cost of the host-buffer path at C2: per-call wall clock of one e2e step (Set* / Add* / Solve / Get*)."""
import importlib, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("ctrl-vio_b200"); syn = pkg.synthetic
lib = pkg.load()
w = syn.config_c2()
est = pkg.Estimator(lib, pkg.make_config(device=0, **w.config_kwargs()))
est.SetOptions(pkg.make_options(fix_ld=w.fix_ld, ld_lower=w.ld_lower, ld_upper=w.ld_upper))
names = ["SetKnots", "SetBiases", "SetInvDepths", "SetLineDelay", "ClearFactors", "AddImage", "AddIMU", "AddBias", "Solve", "GetKnots", "GetBiases", "GetInvDepths", "GetLineDelay"]
acc = np.zeros(len(names)); n = 0
for it in range(30):
    ts = [time.perf_counter()]
    est.SetKnots(w.q0, w.p0); ts.append(time.perf_counter())
    est.SetBiases(w.bias0); ts.append(time.perf_counter())
    est.SetInvDepths(w.rho0); ts.append(time.perf_counter())
    est.SetLineDelay(w.ld0); ts.append(time.perf_counter())
    est.ClearFactors(); ts.append(time.perf_counter())
    est.AddImageFeatureDelayAnalytic(w.ti, w.rowi, w.pi, w.tj, w.rowj, w.pj, w.lm); ts.append(time.perf_counter())
    est.AddIMUMeasurementAnalytic(w.imu_t, w.imu_gyro, w.imu_accel, w.imu_node); ts.append(time.perf_counter())
    est.AddBiasFactor(w.bf_i, w.bf_j, w.bf_sqrt_info); ts.append(time.perf_counter())
    s = est.Solve(15); ts.append(time.perf_counter())
    est.GetKnots(); ts.append(time.perf_counter())
    est.GetBiases(); ts.append(time.perf_counter())
    est.GetInvDepths(); ts.append(time.perf_counter())
    est.GetLineDelay(); ts.append(time.perf_counter())
    if it >= 10:
        acc += np.diff(ts); n += 1
print("per call (us):", {k: round(1e6 * v / n, 1) for k, v in zip(names, acc)})
print("total us", round(1e6 * acc.sum() / n, 1), " solve device ms", s.device_ms)
