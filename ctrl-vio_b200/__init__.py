"""ctrl-vio_b200 — H100-native sliding-window continuous-time bundle adjustment.

The product is `csrc/libctvio_b200.so` (hand-written sm_90a CUDA behind the C-ABI
of include/ctvio.h).  This Python package is only the host-side mirror used by
tests and bench.py: ctypes binding (`binding.py`), the `Estimator` class with the
reference's `TrajectoryEstimator` method names, and the synthetic window
generator (`synthetic.py`).  There is no CPU fallback: `load()` raises when the
CUDA library has not been built, and `ctvio_create` fails without an H100.

The directory name contains a hyphen (it is the name the build contract asks
for); import it with `importlib.import_module("ctrl-vio_b200")`.
"""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np

from . import binding, synthetic
from .binding import (ABI_SYMBOLS, BLK_BA, BLK_BG, BLK_LD, BLK_POS, BLK_RHO, BLK_ROT, Config, CtvioError, CtvioLib,
                      Estimator, Options, PriorData, Summary)

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(PKG_DIR)
CSRC_DIR = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(CSRC_DIR, "libctvio_b200.so")

_lib = None


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA engine for sm_90a in-tree (csrc/build.sh)."""
    script = os.path.join(CSRC_DIR, "build.sh")
    env = dict(os.environ)
    if force:
        env["CTVIO_FORCE_BUILD"] = "1"
    res = subprocess.run(["bash", script], cwd=CSRC_DIR, env=env, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise CtvioError("building libctvio_b200.so failed")
    return LIB_PATH


def load() -> CtvioLib:
    """Load the CUDA engine; fails loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CtvioError(f"{LIB_PATH} is missing — run __graft_entry__.build() (nvcc, sm_90a). "
                             "There is no CPU fallback for the product path.")
        _lib = CtvioLib(LIB_PATH, "ctvio_")
    return _lib


def make_config(*, t0_ns, dt_ns, q_CtoI, p_CinI, image_weight, gravity, imu_info, rs_padding_ns, cauchy_solve=2.0,
                cauchy_marg=1.0, device=0) -> Config:
    c = Config()
    c.t0_ns = int(t0_ns)
    c.dt_ns = int(dt_ns)
    c.q_CtoI[:] = list(np.asarray(q_CtoI, float))
    c.p_CinI[:] = list(np.asarray(p_CinI, float))
    c.image_weight = float(image_weight)
    c.gravity[:] = list(np.asarray(gravity, float))
    c.imu_info[:] = list(np.asarray(imu_info, float))
    c.rs_padding_ns = int(rs_padding_ns)
    c.cauchy_solve = float(cauchy_solve)
    c.cauchy_marg = float(cauchy_marg)
    c.device = int(device)
    return c


def make_options(*, fixed_knot_index=-1, lock_traj=False, lock_wb=False, lock_ab=False, fix_ld=True, is_marg_state=False,
                 ctrl_to_be_opt_now=0, ctrl_to_be_opt_later=0, ld_lower=0.0, ld_upper=0.0) -> Options:
    o = Options()
    o.fixed_knot_index = int(fixed_knot_index)
    o.lock_traj = int(lock_traj)
    o.lock_wb = int(lock_wb)
    o.lock_ab = int(lock_ab)
    o.fix_ld = int(fix_ld)
    o.is_marg_state = int(is_marg_state)
    o.ctrl_to_be_opt_now = int(ctrl_to_be_opt_now)
    o.ctrl_to_be_opt_later = int(ctrl_to_be_opt_later)
    o.ld_lower = float(ld_lower)
    o.ld_upper = float(ld_upper)
    return o


def setup_estimator(lib: CtvioLib, w: "synthetic.Window", *, device=0, state="init", image_marg=None, imu_marg=None,
                    bias_marg=None, options: Options = None, image_slice=None, with_imu=True) -> Estimator:
    """Build an Estimator for a synthetic window the way TrajectoryManager::UpdateTrajectory
    (src/estimator/trajectory_manager.cpp:317-453 of the reference) builds its problem:
    prior (caller), image factors, IMU factors, bias factors."""
    est = Estimator(lib, make_config(device=device, **w.config_kwargs()))
    if options is None:
        options = make_options(fix_ld=w.fix_ld, ld_lower=w.ld_lower, ld_upper=w.ld_upper)
    est.SetOptions(options)
    if state == "init":
        est.SetKnots(w.q0, w.p0); est.SetBiases(w.bias0); est.SetInvDepths(w.rho0); est.SetLineDelay(w.ld0)
    else:
        est.SetKnots(w.q_gt, w.p_gt); est.SetBiases(w.bias_gt); est.SetInvDepths(w.rho_gt); est.SetLineDelay(w.ld_gt)
    sl = image_slice if image_slice is not None else slice(None)
    if w.n_obs:
        est.AddImageFeatureDelayAnalytic(w.ti[sl], w.rowi[sl], w.pi[sl], w.tj[sl], w.rowj[sl], w.pj[sl], w.lm[sl],
                                         None if image_marg is None else image_marg[sl])
    if with_imu and len(w.imu_t):
        est.AddIMUMeasurementAnalytic(w.imu_t, w.imu_gyro, w.imu_accel, w.imu_node, imu_marg)
    if with_imu and len(w.bf_i):
        est.AddBiasFactor(w.bf_i, w.bf_j, w.bf_sqrt_info, bias_marg)
    return est
