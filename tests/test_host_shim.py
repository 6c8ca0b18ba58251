"""The C++ host mirror of ctrlvio::TrajectoryEstimator (ctrl-vio_b200/host/trajectory_estimator.hpp):
compiles against include/ctvio.h with plain g++ (no Eigen / Ceres / ROS), links the C-ABI library, and
 - without a GPU: fails loudly with CTVIO_ERR_NO_DEVICE (no CPU fallback),
 - on an H100: reproduces the oracle's solve through the reference-shaped call sequence."""
import os
import subprocess

import numpy as np
import pytest

from helpers import pkg, rot_angle_between, syn

HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(HERE, "host_shim", "shim_main")


def build_shim():
    src = os.path.join(HERE, "host_shim", "shim_main.cpp")
    hdr = os.path.join(pkg.PKG_DIR, "host", "trajectory_estimator.hpp")
    pkg.load()
    if not os.path.exists(EXE) or max(os.path.getmtime(src), os.path.getmtime(hdr)) > os.path.getmtime(EXE):
        subprocess.run(["g++", "-std=c++17", "-O2", src, "-o", EXE, f"-L{pkg.CSRC_DIR}", "-lctvio_b200",
                        f"-Wl,-rpath,{pkg.CSRC_DIR}"], check=True)
    return EXE


def dump_window(w, path, iters, cycle=None):
    def wv(f, a, dt):
        a = np.ascontiguousarray(a, dt)
        np.array([a.size], np.int64).tofile(f); a.tofile(f)
    with open(path, "wb") as f:
        wv(f, [w.t0_ns, w.dt_ns, iters, int(w.fix_ld)], np.int64)
        wv(f, w.q0, np.float64); wv(f, w.p0, np.float64); wv(f, w.bias0, np.float64); wv(f, w.rho0, np.float64)
        misc = np.concatenate([[w.ld0, w.ld_lower, w.ld_upper, syn.IMAGE_WEIGHT], syn.Q_CtoI, syn.P_CinI, syn.GRAVITY,
                               [1 / syn.SIGMA_G] * 3 + [1 / syn.SIGMA_A] * 3])
        wv(f, misc, np.float64)
        wv(f, w.ti, np.int64); wv(f, w.tj, np.int64); wv(f, w.rowi, np.int32); wv(f, w.rowj, np.int32)
        wv(f, w.pi, np.float64); wv(f, w.pj, np.float64); wv(f, w.lm, np.int32)
        wv(f, w.imu_t, np.int64); wv(f, w.imu_gyro, np.float64); wv(f, w.imu_accel, np.float64); wv(f, w.imu_node, np.int32)
        wv(f, w.bf_i, np.int32); wv(f, w.bf_j, np.int32); wv(f, w.bf_sqrt_info, np.float64)
        if cycle is not None:
            wv(f, cycle["ints"], np.int64)
            wv(f, cycle["img_marg"], np.int32); wv(f, cycle["imu_marg"], np.int32); wv(f, cycle["bias_marg"], np.int32)


def test_host_shim_compiles_and_refuses_without_gpu(tmp_path):
    exe = build_shim()
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("GPU present")
    except ImportError:
        pass
    w = syn.config_c1()
    dump_window(w, tmp_path / "in.bin", 3)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3, (r.returncode, r.stderr)
    assert "no CUDA device" in r.stderr


@pytest.mark.gpu
def test_host_shim_matches_oracle(oracle_lib, tmp_path):
    exe = build_shim()
    w = syn.config_c2(fix_ld=False)
    dump_window(w, tmp_path / "in.bin", 15)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = np.fromfile(tmp_path / "out.bin", np.float64)
    n = w.n_knots
    q = out[:4 * n].reshape(n, 4); p = out[4 * n:7 * n].reshape(n, 3)
    o = pkg.setup_estimator(oracle_lib, w)
    o.Solve(15)
    qo, po = o.GetKnots()
    assert np.abs(p - po).max() / np.abs(po).max() < 1e-5
    assert rot_angle_between(qo, q).max() < 1e-4
    assert abs(out[-1] - o.GetLineDelay()) < 1e-9


@pytest.mark.gpu
def test_host_shim_runs_the_reference_cycle(oracle_lib, tmp_path):
    """InitTrajectory (IMU only, SetFixedIndex, locked biases, Solve(8)) -> UpdateTrajectory (Solve(15)) -> double2vector ->
    UpdateVIOPrior (marg flags, GetResidualSummary, SaveMarginalizationInfo(info&, blocks&)) through the C++ mirror with
    the reference's own argument shapes, against the oracle driven through the same sequence."""
    exe = build_shim()
    w = syn.config_c2(fix_ld=False)
    # the newest control points are copies of control point 24 (ExtendTrajectory), the predictor re-estimates them
    w.q0 = w.q0.copy(); w.p0 = w.p0.copy()
    w.q0[25:] = w.q0[24]; w.p0[25:] = w.p0[24]
    nowk = int((w.kf_times[0] - w.t0_ns) // w.dt_ns); later = int((w.kf_times[1] - w.t0_ns) // w.dt_ns)
    t_min = int(w.t0_ns + 22 * w.dt_ns)
    img_marg = (w.anchor_frame[w.lm] == 0).astype(np.int32)
    imu_marg = (w.imu_t < w.kf_times[1]).astype(np.int32)
    bias_marg = np.zeros(len(w.bf_i), np.int32); bias_marg[0] = 1
    dump_window(w, tmp_path / "in.bin", 15, cycle=dict(ints=[nowk, later, 24, t_min], img_marg=img_marg, imu_marg=imu_marg,
                                                         bias_marg=bias_marg))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), "cycle"], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    out = np.fromfile(tmp_path / "out.bin", np.float64)
    n = w.n_knots; nb = len(w.bias0); nl = len(w.rho0)
    o0 = 7 * n + 6 * nb + nl
    q = out[:4 * n].reshape(n, 4); p = out[4 * n:7 * n].reshape(n, 3)
    ld = out[o0]; pn = int(out[o0 + 1]); nblk = int(out[o0 + 2])
    J = out[o0 + 3:o0 + 3 + pn * pn].reshape(pn, pn); rr = out[o0 + 3 + pn * pn:o0 + 3 + pn * pn + pn]
    summ = out[o0 + 3 + pn * pn + pn:]
    # ---- the oracle through the same sequence ----
    lib = oracle_lib
    e1 = pkg.Estimator(lib, pkg.make_config(**w.config_kwargs()))
    e1.SetOptions(pkg.make_options(fixed_knot_index=24, lock_wb=True, lock_ab=True, fix_ld=False, ld_lower=w.ld_lower, ld_upper=w.ld_upper))
    e1.SetKnots(w.q0, w.p0); e1.SetBiases(w.bias0); e1.SetInvDepths(w.rho0); e1.SetLineDelay(w.ld0)
    m = w.imu_t >= t_min
    e1.AddIMUMeasurementAnalytic(w.imu_t[m], w.imu_gyro[m], w.imu_accel[m], np.full(m.sum(), nb - 1, np.int32))
    e1.Solve(8)
    q1, p1 = e1.GetKnots()
    R0 = syn.qrot(q1[nowk][None], np.eye(3)).T.copy(); t0 = p1[nowk].copy()
    e2 = pkg.setup_estimator(lib, w, options=pkg.make_options(fix_ld=False, ld_lower=w.ld_lower, ld_upper=w.ld_upper))
    e2.SetKnots(q1, p1)
    e2.Solve(15)
    e2.GaugeRealign(nowk, R0, t0)
    q2, p2 = e2.GetKnots()
    assert np.abs(p - p2).max() / np.abs(p2).max() < 1e-5
    assert rot_angle_between(q2, q).max() < 1e-4
    assert abs(ld - e2.GetLineDelay()) < 1e-9
    sel = imu_marg != 0
    e3 = pkg.Estimator(lib, pkg.make_config(**w.config_kwargs()))
    e3.SetOptions(pkg.make_options(fix_ld=False, ld_lower=w.ld_lower, ld_upper=w.ld_upper, is_marg_state=True,
                                   ctrl_to_be_opt_now=nowk, ctrl_to_be_opt_later=later))
    e3.SetKnots(q2, p2); e3.SetBiases(e2.GetBiases()); e3.SetInvDepths(e2.GetInvDepths()); e3.SetLineDelay(e2.GetLineDelay())
    e3.AddImageFeatureDelayAnalytic(w.ti, w.rowi, w.pi, w.tj, w.rowj, w.pj, w.lm, img_marg)
    e3.AddIMUMeasurementAnalytic(w.imu_t[sel], w.imu_gyro[sel], w.imu_accel[sel], w.imu_node[sel], imu_marg[sel])
    e3.AddBiasFactor(w.bf_i[:1], w.bf_j[:1], w.bf_sqrt_info[:1], bias_marg[:1])
    ri, _, _, _ = e3.EvalImageFactors(False, 0.0)
    rm, _, _, _ = e3.EvalImuFactors(False)
    po = e3.SaveMarginalizationInfo()
    assert po is not None and po.n == pn and nblk == len(po.blk_type)
    Ag, Ao = J.T @ J, po.J.T @ po.J
    assert np.allclose(Ag, Ao, atol=1e-6 * np.abs(Ao).max()), np.abs(Ag - Ao).max() / np.abs(Ao).max()
    assert np.allclose(J.T @ rr, po.J.T @ po.r, atol=1e-6 * np.abs(po.J.T @ po.r).max())
    # GetResidualSummary: counts and per-component sums of |r| without the loss
    assert int(summ[0]) == w.n_obs and np.allclose(summ[1:3], np.abs(ri).sum(0), rtol=1e-6)
    assert int(summ[3]) == int(sel.sum()) and np.allclose(summ[4:10], np.abs(rm).sum(0), rtol=1e-6)
    assert int(summ[10]) == 1
