"""ctypes binding of the C-ABI declared in include/ctvio.h.

`CtvioLib(path, prefix)` binds one shared library exporting that ABI under a
symbol prefix; the product library is `libctvio_b200.so` with prefix `ctvio_`.
(The test-suite binds the CPU oracle, which mirrors the ABI under `ctvo_`, with
the same class — the product never does.)

`Estimator` is the host-side mirror of the reference's
`ctrlvio::TrajectoryEstimator` surface (src/estimator/trajectory_estimator.h:76-171):
same method names and argument meaning, batched over numpy arrays, with
pointer identity replaced by index identity.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

ABI_VERSION = 1

BLK_ROT, BLK_POS, BLK_BG, BLK_BA, BLK_LD, BLK_RHO = range(6)
TERM_NAMES = ["NO_CONVERGENCE", "GRADIENT", "PARAMETER", "FUNCTION", "FAILURE", "MIN_RADIUS"]


class CtvioError(RuntimeError):
    pass


class Config(C.Structure):
    """ctvio_config (include/ctvio.h)."""

    _fields_ = [
        ("t0_ns", C.c_int64),
        ("dt_ns", C.c_int64),
        ("q_CtoI", C.c_double * 4),
        ("p_CinI", C.c_double * 3),
        ("image_weight", C.c_double),
        ("gravity", C.c_double * 3),
        ("imu_info", C.c_double * 6),
        ("rs_padding_ns", C.c_int64),
        ("cauchy_solve", C.c_double),
        ("cauchy_marg", C.c_double),
        ("device", C.c_int32),
        ("reserved", C.c_int32),
    ]


class Options(C.Structure):
    """ctvio_options (include/ctvio.h)."""

    _fields_ = [
        ("fixed_knot_index", C.c_int32),
        ("lock_traj", C.c_int32),
        ("lock_wb", C.c_int32),
        ("lock_ab", C.c_int32),
        ("fix_ld", C.c_int32),
        ("is_marg_state", C.c_int32),
        ("ctrl_to_be_opt_now", C.c_int32),
        ("ctrl_to_be_opt_later", C.c_int32),
        ("ld_lower", C.c_double),
        ("ld_upper", C.c_double),
    ]


class Summary(C.Structure):
    """ctvio_summary (include/ctvio.h)."""

    _fields_ = [
        ("iterations", C.c_int32),
        ("num_successful_steps", C.c_int32),
        ("num_unsuccessful_steps", C.c_int32),
        ("termination", C.c_int32),
        ("num_cost_evals", C.c_int32),
        ("num_jacobian_evals", C.c_int32),
        ("num_linear_solves", C.c_int32),
        ("num_line_search_steps", C.c_int32),
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("final_radius", C.c_double),
        ("device_ms", C.c_double),
        ("kernel_launches", C.c_int64),
    ]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["termination_name"] = TERM_NAMES[self.termination] if 0 <= self.termination < len(TERM_NAMES) else "?"
        return d


class ImageMsg(C.Structure):
    """ctvio_image_msg (include/ctvio.h)."""

    _fields_ = [("t_ns", C.c_int64), ("n_points", C.c_int32), ("reserved", C.c_int32)] + [
        (n, C.c_void_p) for n in ("points_xyz", "ch_id", "ch_u", "ch_v", "ch_vx", "ch_vy")]


class ImuMsgs(C.Structure):
    """ctvio_imu_msgs (include/ctvio.h)."""

    _fields_ = [("n", C.c_int32), ("stride_bytes", C.c_int32), ("off_gyro", C.c_int32), ("off_accel", C.c_int32),
                ("data", C.c_void_p)]


class CycleOptions(C.Structure):
    """ctvio_cycle_options (include/ctvio.h)."""

    _fields_ = [
        ("window_size", C.c_int32), ("solve_iterations", C.c_int32), ("predictor_iterations", C.c_int32),
        ("fix_ld", C.c_int32), ("min_parallax", C.c_double), ("init_depth", C.c_double), ("extend_ns", C.c_int64),
        ("ld_lower", C.c_double), ("ld_upper", C.c_double), ("sigma_wb_discrete", C.c_double),
        ("sigma_ab_discrete", C.c_double), ("reanchor", C.c_int32), ("publish_map", C.c_int32),
        ("publish_pose_covariance", C.c_int32), ("publish_odometry_covariance", C.c_int32),
        ("publish_map_covariance", C.c_int32), ("covariance_gauge_knot", C.c_int32),
    ]


class CycleOutputs(C.Structure):
    """ctvio_cycle_outputs (include/ctvio.h)."""

    _fields_ = [("knot_capacity", C.c_int32), ("map_capacity", C.c_int32)] + [
        (n, C.c_void_p) for n in ("q_xyzw", "p_xyz", "line_delay", "map_xyz", "map_feature_id", "map_in_margin_cloud",
                                  "cam_q_xyzw", "cam_p_xyz")]


class CycleResult(C.Structure):
    """ctvio_cycle_result (include/ctvio.h)."""

    _fields_ = [
        ("marg_flag", C.c_int32), ("n_tracked", C.c_int32), ("parallax_num", C.c_int32), ("frame_slot", C.c_int32),
        ("parallax_sum", C.c_double), ("n_frames", C.c_int32), ("n_knots", C.c_int32), ("knot_t0_ns", C.c_int64),
        ("n_landmarks", C.c_int32), ("n_image_factors", C.c_int32), ("n_imu_factors", C.c_int32),
        ("n_predictor_imu", C.c_int32), ("n_triangulated", C.c_int32), ("n_fallback", C.c_int32),
        ("predictor", Summary), ("solve", Summary),
        ("prior_dim", C.c_int32), ("n_removed", C.c_int32), ("n_reanchored", C.c_int32), ("n_map_points", C.c_int32),
        ("n_margin_points", C.c_int32), ("n_knots_after", C.c_int32), ("host_ms", C.c_double),
    ]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k not in ("predictor", "solve")}
        d["predictor"] = self.predictor.as_dict()
        d["solve"] = self.solve.as_dict()
        return d


class CycleCovarianceInfo(C.Structure):
    """ctvio_cycle_covariance_info (include/ctvio.h)."""

    _fields_ = [
        ("requested", C.c_int32), ("available", C.c_int32), ("status", C.c_int32), ("gauge_knot", C.c_int32),
        ("rcond", C.c_double), ("pose_t_ns", C.c_int64), ("n_pairs", C.c_int32), ("n_map_points", C.c_int32),
        ("n_map_points_without_cov", C.c_int32), ("reserved", C.c_int32),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


# every symbol include/ctvio.h declares (without prefix); used by the
# export-completeness test and by the binder.
ABI_SYMBOLS = [
    "last_error", "abi_version", "create", "destroy", "set_options", "set_deterministic",
    "set_knots", "set_biases", "set_inv_depths", "set_line_delay", "set_time_origin",
    "get_knots", "get_biases", "get_inv_depths", "get_line_delay",
    "clear_factors", "add_image_features", "add_imu_measurements", "add_bias_factors", "set_prior",
    "solve", "gauge_realign", "marginalize", "get_prior", "adopt_prior",
    "save_state", "restore_state",
    "eval_image_factors", "eval_imu_factors", "residual_summary", "eval_cost", "normal_equations", "covariance",
    "pose_covariance", "relative_pose_covariance", "point_covariance", "query_trajectory", "triangulate",
    "extend_knots_to", "slide_window", "remap_landmarks", "enable_prior", "ingest_feature_cloud", "add_image_features_from_slots",
    "ingest_imu", "add_imu_from_table", "transfer_stats", "profile_kernels", "measure_fp64_tflops", "measure_fp64_tensor_tflops",
    "selfcheck_solver", "nccl_unique_id", "comm_init", "triangulate_window", "check_keyframe", "slide_window_second_new",
    "feature_table_add", "feature_table_window", "triangulate_window_from_table", "add_image_features_from_table",
    "feature_table_slide", "feature_table_landmarks", "feature_table_map", "feature_table_slide_reanchor",
    "debug_structure", "feature_table_point_covariance", "sync_stats", "cycle_default_options", "odometry_start",
    "process_image", "debug_bias_weights", "cycle_covariances", "odometry_checkpoint", "odometry_restore",
]


# entry points a checker library (the CPU oracle mirrors the ABI under `ctvo_`) need not provide: multi-GPU plumbing and
# the device-residency / wire-format calls, which have no CPU meaning, and the covariances, which the tests form from the
# oracle's normal equations instead
DEVICE_ONLY_SYMBOLS = ("nccl_unique_id", "comm_init", "set_deterministic", "enable_prior", "extend_knots_to", "slide_window", "remap_landmarks",
                       "ingest_feature_cloud", "add_image_features_from_slots", "ingest_imu", "add_imu_from_table",
                       "transfer_stats", "residual_summary", "triangulate_window", "check_keyframe",
                       "slide_window_second_new", "feature_table_add", "feature_table_window", "triangulate_window_from_table",
                       "add_image_features_from_table", "feature_table_slide", "feature_table_landmarks",
                       "feature_table_map", "feature_table_slide_reanchor", "debug_structure", "covariance",
                       "pose_covariance", "relative_pose_covariance", "point_covariance", "feature_table_point_covariance",
                       "sync_stats", "cycle_default_options", "odometry_start", "process_image", "debug_bias_weights",
                       "cycle_covariances", "odometry_checkpoint", "odometry_restore")

# ctypes prototypes of the entry points whose arguments ctypes must convert on its own (include/ctvio.h)
PROTOTYPES = {
    "odometry_checkpoint": [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)],
    "odometry_restore": [C.c_void_p, C.c_void_p, C.c_int64],
}


def _addr(a):
    # (numpy's `.ctypes.data_as(...)` costs more per array than the raw address as a void pointer: the host-buffer
    #  path passes ~25 arrays per window)
    return C.c_void_p(a.__array_interface__["data"][0]) if a is not None else None


_dp = _ip = _lp = _addr


def _f64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None:
        a = a.reshape(shape)
    return a


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


class CtvioLib:
    """One loaded shared library exporting the ctvio C-ABI under `prefix`."""

    def __init__(self, path: str, prefix: str = "ctvio_", optional=()):
        if not os.path.exists(path):
            raise CtvioError(f"shared library not found: {path}")
        self.path = path
        self.prefix = prefix
        self.lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
        self._fn = {}
        for name in ABI_SYMBOLS:
            try:
                self._fn[name] = getattr(self.lib, prefix + name)
            except AttributeError:
                if name in optional:
                    continue
                raise CtvioError(f"{path} does not export {prefix}{name}")
        self._fn["last_error"].restype = C.c_char_p
        for name, f in self._fn.items():
            if name != "last_error":
                f.restype = C.c_int
            if name in PROTOTYPES:
                f.argtypes = PROTOTYPES[name]

    def has(self, name):
        return name in self._fn

    def raw(self, name):
        """Any extra symbol of the library (oracle-only probes etc.)."""
        return getattr(self.lib, self.prefix + name)

    def call(self, name, *args):
        rc = self._fn[name](*args)
        if rc != 0:
            msg = self._fn["last_error"]()
            raise CtvioError(f"{self.prefix}{name} failed ({rc}): {msg.decode() if msg else ''}")
        return rc


@dataclass
class PriorData:
    """MarginalizationInfo payload (marginalization_factor.h:96-131)."""

    n: int = 0
    J: np.ndarray = field(default_factory=lambda: np.zeros((0, 0)))
    r: np.ndarray = field(default_factory=lambda: np.zeros(0))
    blk_type: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    blk_index: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    blk_col: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    blk_x0: np.ndarray = field(default_factory=lambda: np.zeros((0, 4)))


class Estimator:
    """Host-side mirror of ctrlvio::TrajectoryEstimator over the C-ABI.

    Method names follow src/estimator/trajectory_estimator.h:76-171; array
    arguments batch what the reference adds one factor at a time.
    """

    def __init__(self, lib: CtvioLib, cfg: Config):
        self.lib = lib
        self.cfg = cfg
        self.h = C.c_void_p()
        lib.call("create", C.byref(cfg), C.byref(self.h))
        self.n_knots = self.n_bias = self.n_lm = 0
        self.n_img = self.n_imu = self.n_biasf = 0

    def close(self):
        if self.h:
            self.lib.call("destroy", self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- options / state ---------------------------------------------------
    def SetOptions(self, opt: Options):
        self.lib.call("set_options", self.h, C.byref(opt))

    def SetDeterministic(self, on=True):
        self.lib.call("set_deterministic", self.h, C.c_int32(int(on)))

    def SetKnots(self, q, p):
        q = _f64(q, (-1, 4)); p = _f64(p, (-1, 3))
        assert q.shape[0] == p.shape[0]
        self.n_knots = q.shape[0]
        self.lib.call("set_knots", self.h, C.c_int32(self.n_knots), _dp(q), _dp(p))

    def SetBiases(self, b):
        b = _f64(b, (-1, 6))
        self.n_bias = b.shape[0]
        self.lib.call("set_biases", self.h, C.c_int32(self.n_bias), _dp(b))

    def SetInvDepths(self, r):
        r = _f64(r, (-1,))
        self.n_lm = r.shape[0]
        self.lib.call("set_inv_depths", self.h, C.c_int32(self.n_lm), _dp(r))

    def SetTimeOrigin(self, t0_ns):
        """Move the window: knot 0 of the next SetKnots slice sits at t0_ns (on the knot grid)."""
        self.lib.call("set_time_origin", self.h, C.c_int64(int(t0_ns)))

    def SetLineDelay(self, ld):
        self.lib.call("set_line_delay", self.h, C.c_double(ld))

    def GetKnots(self):
        q = np.zeros((self.n_knots, 4)); p = np.zeros((self.n_knots, 3))
        self.lib.call("get_knots", self.h, _dp(q), _dp(p))
        return q, p

    def GetBiases(self):
        b = np.zeros((self.n_bias, 6))
        self.lib.call("get_biases", self.h, _dp(b))
        return b

    def GetInvDepths(self):
        r = np.zeros(self.n_lm)
        self.lib.call("get_inv_depths", self.h, _dp(r))
        return r

    def GetLineDelay(self):
        v = C.c_double()
        self.lib.call("get_line_delay", self.h, C.byref(v))
        return v.value

    # --- factors -------------------------------------------------------------
    def ClearFactors(self):
        self.lib.call("clear_factors", self.h)
        self.n_img = self.n_imu = self.n_biasf = 0

    def AddImageFeatureDelayAnalytic(self, ti, rowi, pi, tj, rowj, pj, landmark, marg=None):
        ti = _i64(ti); tj = _i64(tj); rowi = _i32(rowi); rowj = _i32(rowj)
        pi = _f64(pi, (-1, 2)); pj = _f64(pj, (-1, 2)); landmark = _i32(landmark)
        marg = _i32(marg) if marg is not None else None
        n = ti.shape[0]
        self.lib.call("add_image_features", self.h, C.c_int32(n), _lp(ti), _ip(rowi), _dp(pi), _lp(tj), _ip(rowj),
                      _dp(pj), _ip(landmark), _ip(marg))
        self.n_img += n

    def AddIMUMeasurementAnalytic(self, t, gyro, accel, bias_node, marg=None):
        t = _i64(t); gyro = _f64(gyro, (-1, 3)); accel = _f64(accel, (-1, 3)); bias_node = _i32(bias_node)
        marg = _i32(marg) if marg is not None else None
        n = t.shape[0]
        self.lib.call("add_imu_measurements", self.h, C.c_int32(n), _lp(t), _dp(gyro), _dp(accel), _ip(bias_node),
                      _ip(marg))
        self.n_imu += n

    def AddBiasFactor(self, node_i, node_j, sqrt_info, marg=None):
        node_i = _i32(node_i); node_j = _i32(node_j); sqrt_info = _f64(sqrt_info, (-1, 6))
        marg = _i32(marg) if marg is not None else None
        n = node_i.shape[0]
        self.lib.call("add_bias_factors", self.h, C.c_int32(n), _ip(node_i), _ip(node_j), _dp(sqrt_info), _ip(marg))
        self.n_biasf += n

    def AddMarginalizationFactor(self, prior: Optional[PriorData]):
        if prior is None or prior.n == 0:
            self.lib.call("set_prior", self.h, C.c_int32(0), None, None, C.c_int32(0), None, None, None, None)
            return
        J = _f64(prior.J, (prior.n, prior.n)); r = _f64(prior.r, (prior.n,))
        bt = _i32(prior.blk_type); bi = _i32(prior.blk_index); bc = _i32(prior.blk_col)
        x0 = _f64(prior.blk_x0, (-1, 4))
        self.lib.call("set_prior", self.h, C.c_int32(prior.n), _dp(J), _dp(r), C.c_int32(bt.shape[0]), _ip(bt),
                      _ip(bi), _ip(bc), _dp(x0))

    # --- solve / marginalize ---------------------------------------------------
    def Solve(self, max_iterations=50) -> Summary:
        s = Summary()
        self.lib.call("solve", self.h, C.c_int32(max_iterations), C.byref(s))
        return s

    def GaugeRealign(self, min_idx, R0, t0):
        R0 = _f64(R0, (9,)); t0 = _f64(t0, (3,))
        self.lib.call("gauge_realign", self.h, C.c_int32(min_idx), _dp(R0), _dp(t0))

    def SaveMarginalizationInfo(self) -> Optional[PriorData]:
        n = C.c_int32(); nb = C.c_int32()
        self.lib.call("marginalize", self.h, C.byref(n), C.byref(nb))
        if n.value <= 0:
            return None
        pr = PriorData(n=n.value, J=np.zeros((n.value, n.value)), r=np.zeros(n.value),
                       blk_type=np.zeros(nb.value, np.int32), blk_index=np.zeros(nb.value, np.int32),
                       blk_col=np.zeros(nb.value, np.int32), blk_x0=np.zeros((nb.value, 4)))
        self.lib.call("get_prior", self.h, _dp(pr.J), _dp(pr.r), _ip(pr.blk_type), _ip(pr.blk_index),
                      _ip(pr.blk_col), _dp(pr.blk_x0))
        return pr

    def AdoptPrior(self):
        self.lib.call("adopt_prior", self.h)

    def SaveState(self):
        self.lib.call("save_state", self.h)

    def RestoreState(self):
        self.lib.call("restore_state", self.h)

    # --- probes -------------------------------------------------------------------
    def EvalImageFactors(self, want_jacobians=True, cauchy_scale=0.0):
        n = self.n_img
        r = np.zeros((n, 2)); s = np.zeros((n, 2), np.int32); J = np.zeros((n, 100)); cost = C.c_double()
        self.lib.call("eval_image_factors", self.h, C.c_int32(int(want_jacobians)), C.c_double(cauchy_scale), _dp(r),
                      _ip(s), _dp(J), C.byref(cost))
        return r, s, J, cost.value

    def EvalImuFactors(self, want_jacobians=True):
        n = self.n_imu
        r = np.zeros((n, 6)); s = np.zeros(n, np.int32); J = np.zeros((n, 156)); cost = C.c_double()
        self.lib.call("eval_imu_factors", self.h, C.c_int32(int(want_jacobians)), _dp(r), _ip(s), _dp(J),
                      C.byref(cost))
        return r, s, J, cost.value

    def ResidualSummary(self, prior_n=0):
        """GetResidualSummary: ({type: (count, per-component sums of |r|)})."""
        counts = np.zeros(4, np.int32); sums = np.zeros(18); pr = np.zeros(max(prior_n, 1))
        self.lib.call("residual_summary", self.h, _ip(counts), _dp(sums), _dp(pr) if prior_n else None)
        return {"image": (int(counts[0]), sums[0:2].copy()), "imu": (int(counts[1]), sums[2:8].copy()),
                "bias": (int(counts[2]), sums[8:14].copy()), "prior": (int(counts[3]), pr[:prior_n].copy())}

    def EvalCost(self):
        cost = C.c_double()
        self.lib.call("eval_cost", self.h, C.byref(cost))
        return cost.value

    @property
    def np_dim(self):
        return 6 * self.n_knots + 6 * self.n_bias + 1

    def NormalEquations(self):
        npd = self.np_dim
        H = np.zeros((npd, npd)); g = np.zeros(npd); hl = np.zeros(self.n_lm); gl = np.zeros(self.n_lm)
        cost = C.c_double()
        self.lib.call("normal_equations", self.h, _dp(H), _dp(g), _dp(hl), _dp(gl), C.byref(cost))
        return H, g, hl, gl, cost.value

    def Covariance(self, want_cc=True, want_rho=True):
        """ceres::Covariance of the camera-side block and the inverse depths at the current state (ctvio_covariance):
        (cov_cc [np, np] or None, var_rho [n_lm] or None, rcond).  Raises CtvioError on a rank-deficient window, with
        rcond in the message."""
        npd = self.np_dim
        cc = np.zeros((npd, npd)) if want_cc else None
        vr = np.zeros(self.n_lm) if want_rho else None
        rcond = C.c_double()
        self.lib.call("covariance", self.h, _dp(cc), _dp(vr), C.byref(rcond))
        return cc, vr, rcond.value

    def PoseCovariance(self, t, gauge_knot_index=-1, camera_frame=False):
        """Covariance of (dtheta, dp, domega, dv) at the times t (ctvio_pose_covariance): (cov [n, 12, 12], rcond).
        Knots <= gauge_knot_index are held constant for this call only; camera_frame=True gives the camera's pose and
        velocity.  Raises CtvioError on a rank-deficient window, with rcond in the message."""
        t = _i64(np.atleast_1d(t)); n = t.shape[0]
        cov = np.zeros((n, 12, 12))
        rcond = C.c_double()
        self.lib.call("pose_covariance", self.h, C.c_int32(n), _lp(t), C.c_int32(int(gauge_knot_index)),
                      C.c_int32(int(bool(camera_frame))), _dp(cov), C.byref(rcond))
        return cov, rcond.value

    def RelativePoseCovariance(self, t_a, t_b, gauge_knot_index=-1, camera_frame=False, want_cross=False):
        """Covariance of (dtheta_ab, dp_ab), the pose at t_b in the frame of the pose at t_a, for each pair
        (ctvio_relative_pose_covariance): (cov [n, 6, 6], cross [n, 6, 6] or None, rcond).  cross (want_cross=True) is the
        covariance of the two poses' (dtheta, dp), rows a and columns b.  Knots <= gauge_knot_index are held constant for
        this call only; camera_frame=True gives the camera poses.  Raises CtvioError on a rank-deficient window, with
        rcond in the message."""
        ta = _i64(np.atleast_1d(t_a)); tb = _i64(np.atleast_1d(t_b)); n = ta.shape[0]
        assert tb.shape[0] == n
        cov = np.zeros((n, 6, 6))
        cross = np.zeros((n, 6, 6)) if want_cross else None
        rcond = C.c_double()
        self.lib.call("relative_pose_covariance", self.h, C.c_int32(n), _lp(ta), _lp(tb), C.c_int32(int(gauge_knot_index)),
                      C.c_int32(int(bool(camera_frame))), _dp(cov), _dp(cross), C.byref(rcond))
        return cov, cross, rcond.value

    def PointCovariance(self, landmark, t, bearing, gauge_knot_index=-1):
        """Covariance of the world points of landmarks anchored at the times t with the bearings (x, y)
        (ctvio_point_covariance): (cov [n, 3, 3], rcond).  Knots <= gauge_knot_index are held constant for this call
        only.  Raises CtvioError on a rank-deficient window, with rcond in the message."""
        lm = _i32(np.atleast_1d(landmark)); t = _i64(np.atleast_1d(t)); b = _f64(bearing, (-1, 2))
        n = lm.shape[0]
        assert t.shape[0] == n and b.shape[0] == n
        cov = np.zeros((n, 3, 3))
        rcond = C.c_double()
        self.lib.call("point_covariance", self.h, C.c_int32(n), _ip(lm), _lp(t), _dp(b), C.c_int32(int(gauge_knot_index)),
                      _dp(cov), C.byref(rcond))
        return cov, rcond.value

    def QueryTrajectory(self, t):
        t = _i64(t); n = t.shape[0]
        q = np.zeros((n, 4)); p = np.zeros((n, 3)); w = np.zeros((n, 3)); v = np.zeros((n, 3)); a = np.zeros((n, 3))
        self.lib.call("query_trajectory", self.h, C.c_int32(n), _lp(t), _dp(q), _dp(p), _dp(w), _dp(v), _dp(a))
        return q, p, w, v, a

    def Triangulate(self, Rs, Ps, ric, tic, start_frame, obs_offset, obs_point, depth, window_size=10,
                    init_depth=5.0):
        """FeatureManager::triangulate (feature_manager.cpp:230-275) over CSR-packed landmark observations;
        returns the updated depth array (entries > 0 are kept)."""
        Rs = _f64(Rs, (-1, 9)); Ps = _f64(Ps, (-1, 3)); ric = _f64(ric, (9,)); tic = _f64(tic, (3,))
        start_frame = _i32(start_frame); obs_offset = _i32(obs_offset); obs_point = _f64(obs_point, (-1, 3))
        depth = _f64(depth, (-1,)).copy()
        self.lib.call("triangulate", self.h, C.c_int32(Rs.shape[0]), _dp(Rs), _dp(Ps), _dp(ric), _dp(tic),
                      C.c_int32(start_frame.shape[0]), _ip(start_frame), _ip(obs_offset), _dp(obs_point),
                      C.c_int32(window_size), C.c_double(init_depth), _dp(depth))
        return depth

    # --- device-resident window / wire formats (SURVEY 8f-1, 8f-4) ---------------------
    def ExtendKnotsTo(self, t_ns) -> int:
        n = C.c_int32()
        self.lib.call("extend_knots_to", self.h, C.c_int64(int(t_ns)), C.byref(n))
        self.n_knots = n.value
        return n.value

    def SlideWindow(self, n_drop_knots, n_drop_bias, n_new_bias):
        self.lib.call("slide_window", self.h, C.c_int32(n_drop_knots), C.c_int32(n_drop_bias), C.c_int32(n_new_bias))
        self.n_knots -= n_drop_knots
        self.n_bias += n_new_bias - n_drop_bias

    def SlideWindowSecondNew(self):
        """the MARGIN_SECOND_NEW slide (visual_odometry.cpp:253-278): bias node n-2 takes node n-1's value; knots and
        prior stay."""
        self.lib.call("slide_window_second_new", self.h)

    def CheckKeyframe(self, frame_slots, min_parallax):
        """FeatureManager::addFeatureCheckParallax (feature_manager.cpp:28-87) over resident frame slots, oldest to
        newest, the new image last.  Returns (is_keyframe, n_tracked, parallax_num, parallax_sum)."""
        slots = _i32(frame_slots)
        kf, nt, num = C.c_int32(), C.c_int32(), C.c_int32()
        s = C.c_double()
        self.lib.call("check_keyframe", self.h, C.c_int32(slots.shape[0]), _ip(slots), C.c_double(min_parallax),
                      C.byref(kf), C.byref(nt), C.byref(num), C.byref(s))
        return bool(kf.value), nt.value, num.value, s.value

    def EnablePrior(self, on: bool):
        self.lib.call("enable_prior", self.h, C.c_int32(int(on)))

    def RemapLandmarks(self, old_index, init_inv_depth):
        old_index = _i32(old_index); init = _f64(init_inv_depth, (-1,))
        assert old_index.shape[0] == init.shape[0]
        self.lib.call("remap_landmarks", self.h, C.c_int32(old_index.shape[0]), _ip(old_index), _dp(init))
        self.n_lm = old_index.shape[0]

    def IngestFeatureCloud(self, frame_slot, t_ns, points_xyz, ch_id, ch_u, ch_v, ch_vx, ch_vy):
        """sensor_msgs::PointCloud of the tracker as it is: float32 point triples + five float32 channels."""
        f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
        pts = f32(points_xyz).reshape(-1, 3); ch = [f32(x).reshape(-1) for x in (ch_id, ch_u, ch_v, ch_vx, ch_vy)]
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        self.lib.call("ingest_feature_cloud", self.h, C.c_int32(frame_slot), C.c_int64(int(t_ns)), C.c_int32(pts.shape[0]),
                      fp(pts), *[fp(x) for x in ch])

    def AddImageFeaturesFromSlots(self, slot_i, idx_i, slot_j, idx_j, landmark, marg=None):
        a = [_i32(x) for x in (slot_i, idx_i, slot_j, idx_j, landmark)]
        marg = _i32(marg) if marg is not None else None
        n = a[0].shape[0]
        self.lib.call("add_image_features_from_slots", self.h, C.c_int32(n), *[_ip(x) for x in a], _ip(marg))
        self.n_img += n

    def TriangulateWindow(self, obs_offset, obs_slot, obs_idx, init_depth=5.0):
        """FeatureManager::triangulate of the resident window (feature_manager.cpp:226-338): DLT of every landmark whose
        inverse depth is <= 0 from its observations (frame slot, feature index; the first one the anchor), camera poses
        from the resident spline at each observation's row time.  Returns (n_triangulated, n_fallback)."""
        obs_offset = _i32(obs_offset); obs_slot = _i32(obs_slot); obs_idx = _i32(obs_idx)
        nt, nf = C.c_int32(), C.c_int32()
        self.lib.call("triangulate_window", self.h, C.c_int32(max(obs_offset.shape[0] - 1, 0)), _ip(obs_offset), _ip(obs_slot),
                      _ip(obs_idx), C.c_double(init_depth), C.byref(nt), C.byref(nf))
        return nt.value, nf.value

    # --- resident feature table (FeatureManager's feature list on the device) --------------------------------
    def FeatureTableAdd(self, frame_slot):
        """addFeatureCheckParallax's insertion (feature_manager.cpp:28-59) for the cloud ingested into frame_slot.
        Returns (n_tracked, n_new)."""
        nt, nn = C.c_int32(), C.c_int32()
        self.lib.call("feature_table_add", self.h, C.c_int32(frame_slot), C.byref(nt), C.byref(nn))
        return nt.value, nn.value

    def FeatureTableWindow(self, frame_slots, window_size):
        """setDepth + getDepthVector's numbering over the window's frame slots, oldest to newest; re-lays out the resident
        inverse depths to it.  Returns n_landmarks."""
        slots = _i32(frame_slots)
        n = C.c_int32()
        self.lib.call("feature_table_window", self.h, C.c_int32(slots.shape[0]), _ip(slots), C.c_int32(window_size),
                      C.byref(n))
        self.n_lm = n.value
        return n.value

    def TriangulateWindowFromTable(self, init_depth=5.0):
        """TriangulateWindow over the last FeatureTableWindow's landmarks.  Returns (n_triangulated, n_fallback)."""
        nt, nf = C.c_int32(), C.c_int32()
        self.lib.call("triangulate_window_from_table", self.h, C.c_double(init_depth), C.byref(nt), C.byref(nf))
        return nt.value, nf.value

    def AddImageFeaturesFromTable(self, marg_oldest):
        """one image factor per (landmark, non-anchor observation) of the last window.  Returns n_factors."""
        n = C.c_int32()
        self.lib.call("add_image_features_from_table", self.h, C.c_int32(int(marg_oldest)), C.byref(n))
        self.n_img += n.value
        return n.value

    def FeatureTableSlide(self, frame_slot):
        """removeFailures, then the leaving slot's landmarks and observations leave.  Returns n_removed."""
        n = C.c_int32()
        self.lib.call("feature_table_slide", self.h, C.c_int32(frame_slot), C.byref(n))
        return n.value

    def FeatureTableSlideReanchor(self, frame_slots, marg_old, init_depth=5.0):
        """removeFailures, then SlideWindowOld's removeBackShiftDepth (marg_old: frame_slots[0] leaves, its landmarks are
        re-anchored in the next frame with their depth shifted there) or SlideWindowNew's removeFront (frame_slots[-2]
        leaves, its landmarks seen in the newest frame are re-anchored there).  frame_slots: the window before the slide,
        oldest to newest.  Returns (n_removed, n_reanchored)."""
        slots = _i32(frame_slots)
        nr, na = C.c_int32(), C.c_int32()
        self.lib.call("feature_table_slide_reanchor", self.h, C.c_int32(slots.shape[0]), _ip(slots), C.c_int32(int(marg_old)),
                      C.c_double(init_depth), C.byref(nr), C.byref(na))
        return nr.value, na.value

    def FeatureTableLandmarks(self, n_landmarks=None):
        """(feature id, anchor slot, used_num) of each landmark of the last window"""
        n = self.n_lm if n_landmarks is None else n_landmarks
        ids, anchor, used = (np.zeros(max(n, 0), np.int32) for _ in range(3))
        self.lib.call("feature_table_landmarks", self.h, C.c_int32(n), _ip(ids), _ip(anchor), _ip(used))
        return ids, anchor, used

    def FeatureTablePointCovariance(self, gauge_knot_index=-1):
        """PointCovariance of every landmark of the last window, anchored as the feature table holds it
        (ctvio_feature_table_point_covariance): (cov [n_lm, 3, 3], rcond) in the window's numbering."""
        n = self.n_lm
        cov = np.zeros((n, 3, 3))
        rcond = C.c_double()
        self.lib.call("feature_table_point_covariance", self.h, C.c_int32(n), C.c_int32(int(gauge_knot_index)), _dp(cov),
                      C.byref(rcond))
        return cov, rcond.value

    # capacity of FeatureTableMap's point arrays: every entry the table can hold (16 slots x 1024 features)
    MAP_CAPACITY = 16 * 1024

    def FeatureTableMap(self, frame_slots, window_size):
        """GetLandmarksInWindow / GetMarginCloud / PublishVioKeyFrame (visual_odometry.cpp:310-372) over the window's
        frame slots after the slide, oldest to newest.  Returns (xyz [n, 3], feature ids [n], in_margin_cloud [n] bool,
        camera q xyzw [n_frames, 4], camera p [n_frames, 3]): the stable landmarks in table order, world points, and
        the frames' camera poses at the frame time."""
        slots = _i32(frame_slots)
        cap = self.MAP_CAPACITY
        xyz, ids, marg = np.empty((cap, 3)), np.empty(cap, np.int32), np.empty(cap, np.uint8)
        cq, cp = np.empty((slots.shape[0], 4)), np.empty((slots.shape[0], 3))
        n = C.c_int32()
        self.lib.call("feature_table_map", self.h, C.c_int32(slots.shape[0]), _ip(slots), C.c_int32(window_size),
                      C.c_int32(cap), _dp(xyz), _ip(ids), _ip(marg), C.byref(n), _dp(cq), _dp(cp))
        k = n.value
        return xyz[:k].copy(), ids[:k].copy(), marg[:k].astype(bool), cq, cp

    def IngestImu(self, records: np.ndarray, off_gyro, off_accel, drop_before_ns=0):
        """packed IMUData records (structured / byte array, one record per row)."""
        rec = np.ascontiguousarray(records)
        n = rec.shape[0]
        stride = rec.strides[0] if n else rec.dtype.itemsize
        self.lib.call("ingest_imu", self.h, C.c_int32(n), rec.ctypes.data_as(C.c_void_p), C.c_int32(stride),
                      C.c_int32(off_gyro), C.c_int32(off_accel), C.c_int64(int(drop_before_ns)))

    def AddImuFromTable(self, t_min_ns, t_max_ns, kf_times=None, fixed_node=-1, marg_before_ns=-(1 << 62)) -> int:
        kf = _i64(kf_times) if kf_times is not None else None
        n = C.c_int32()
        self.lib.call("add_imu_from_table", self.h, C.c_int64(int(t_min_ns)), C.c_int64(int(t_max_ns)),
                      C.c_int32(0 if kf is None else kf.shape[0]), _lp(kf), C.c_int32(fixed_node),
                      C.c_int64(int(marg_before_ns)), C.byref(n))
        self.n_imu += n.value
        return n.value

    def TransferStats(self, reset=True):
        a, b = C.c_int64(), C.c_int64()
        self.lib.call("transfer_stats", self.h, C.byref(a), C.byref(b), C.c_int32(int(reset)))
        return a.value, b.value

    def SyncStats(self, reset=True):
        """host waits on the device (stream synchronisations, published-scalar spins) since the last reset"""
        a = C.c_int64()
        self.lib.call("sync_stats", self.h, C.byref(a), C.c_int32(int(reset)))
        return a.value

    # --- the per-image odometry cycle ---------------------------------------------------------------------------
    @staticmethod
    def _image_msg(t_ns, message):
        """(ImageMsg, keep-alive arrays) of a tracker message (points, id, u, v, vx, vy)"""
        pts = np.ascontiguousarray(message[0], np.float32).reshape(-1, 3)
        ch = [np.ascontiguousarray(x, np.float32).reshape(-1) for x in message[1:6]]
        m = ImageMsg(t_ns=int(t_ns), n_points=pts.shape[0])
        m.points_xyz, m.ch_id, m.ch_u, m.ch_v, m.ch_vx, m.ch_vy = (a.ctypes.data for a in [pts] + ch)
        return m, [pts] + ch

    @staticmethod
    def _imu_msgs(records, off_gyro, off_accel):
        if records is None:
            return None, None
        rec = np.ascontiguousarray(records)
        n = rec.shape[0]
        m = ImuMsgs(n=n, stride_bytes=rec.strides[0] if n else rec.dtype.itemsize, off_gyro=off_gyro, off_accel=off_accel,
                    data=rec.ctypes.data if n else None)
        return m, rec

    def _cycle_outputs(self, want_knots, want_map, n_knots_cap):
        out = CycleOutputs()
        keep = {}
        if want_knots:
            keep["q"] = np.zeros((n_knots_cap, 4)); keep["p"] = np.zeros((n_knots_cap, 3)); keep["ld"] = np.zeros(1)
            out.knot_capacity = n_knots_cap
            out.q_xyzw, out.p_xyz, out.line_delay = keep["q"].ctypes.data, keep["p"].ctypes.data, keep["ld"].ctypes.data
        if want_map:
            cap = self.MAP_CAPACITY
            keep["xyz"] = np.empty((cap, 3)); keep["ids"] = np.empty(cap, np.int32); keep["marg"] = np.empty(cap, np.uint8)
            keep["cq"] = np.empty((16, 4)); keep["cp"] = np.empty((16, 3))
            out.map_capacity = cap
            out.map_xyz, out.map_feature_id, out.map_in_margin_cloud = (keep[k].ctypes.data for k in ("xyz", "ids", "marg"))
            out.cam_q_xyzw, out.cam_p_xyz = keep["cq"].ctypes.data, keep["cp"].ctypes.data
        return out, keep

    @staticmethod
    def _cycle_arrays(res, keep):
        arrays = {}
        if "q" in keep:
            n = res.n_knots
            arrays.update(q=keep["q"][:n].copy(), p=keep["p"][:n].copy(), line_delay=float(keep["ld"][0]))
        if "xyz" in keep:
            k, nf = res.n_map_points, res.n_frames - 1
            arrays["map"] = (keep["xyz"][:k].copy(), keep["ids"][:k].copy(), keep["marg"][:k].astype(bool),
                             keep["cq"][:nf].copy(), keep["cp"][:nf].copy())
        return arrays

    def OdometryStart(self, opt: CycleOptions, t0_ns, q, p, messages, frame_times, bg_ba, line_delay, imu_records=None,
                      off_gyro=8, off_accel=32, marg_flag_override=-1, want_knots=True, want_map=True):
        """ctvio_odometry_start: the initializer's window (knots from t0_ns, one tracker message and one bias node per
        frame, the IMU records so far) solved as the first window.  Returns (result dict, arrays dict: q, p, line_delay
        when want_knots; map = (xyz, ids, in_margin, cam_q, cam_p) when want_map)."""
        q = _f64(q, (-1, 4)); p = _f64(p, (-1, 3)); b = _f64(bg_ba, (-1, 6))
        msgs, keep_alive = [], []
        for t, m in zip(frame_times, messages):
            mm, ka = self._image_msg(t, m)
            msgs.append(mm); keep_alive.append(ka)
        frames = (ImageMsg * len(msgs))(*msgs)
        imu, rec = self._imu_msgs(imu_records, off_gyro, off_accel)
        out, keep = self._cycle_outputs(want_knots, want_map, q.shape[0])
        res = CycleResult()
        self.lib.call("odometry_start", self.h, C.byref(opt), C.c_int64(int(t0_ns)), C.c_int32(q.shape[0]), _dp(q), _dp(p),
                      C.c_int32(len(msgs)), frames, _dp(b), C.c_double(line_delay), C.byref(imu) if imu is not None else None,
                      C.c_int32(marg_flag_override), C.byref(out), C.byref(res))
        self._after_cycle(res, opt)
        return res.as_dict(), self._cycle_arrays(res, keep)

    def ProcessImage(self, t_ns, message, imu_records=None, off_gyro=8, off_accel=32, marg_flag_override=-1,
                     want_knots=True, want_map=True):
        """ctvio_process_image: one image of the per-image cycle.  Returns (result dict, arrays dict) as OdometryStart."""
        m, _ka = self._image_msg(t_ns, message)
        imu, rec = self._imu_msgs(imu_records, off_gyro, off_accel)
        # the extension adds at most extend_ns / dt + 1 knots
        out, keep = self._cycle_outputs(want_knots, want_map, self.n_knots + 64)
        res = CycleResult()
        self.lib.call("process_image", self.h, C.byref(m), C.byref(imu) if imu is not None else None,
                      C.c_int32(marg_flag_override), C.byref(out), C.byref(res))
        self._after_cycle(res, None)
        return res.as_dict(), self._cycle_arrays(res, keep)

    def _after_cycle(self, res, opt):
        # the engine's window after the slide (GetKnots / GetBiases / GetInvDepths read it)
        self.n_knots = res.n_knots_after
        self.n_bias = res.n_frames   # (the newest node stands for the next image)
        self.n_lm = res.n_landmarks

    CTVIO_ERR_STATE = -4

    def CycleCovariances(self):
        """ctvio_cycle_covariances: what the last cycle published with its publish_*_covariance options, as
        (cov12 [12, 12] or None, cov6 [n_frames - 1, 6, 6] or None, map_cov9 [n_map_points, 3, 3] or None, info dict).
        The info dict (ctvio_cycle_covariance_info) also carries pose_t_ns, pair_t_ns [n_pairs, 2] and, when nothing is
        available, the reason as "error".  Raises CtvioError when no cycle asked for covariances."""
        info = CycleCovarianceInfo()
        cov12 = np.zeros((12, 12)); cov6 = np.zeros((15, 6, 6)); pair_t = np.zeros((15, 2), np.int64)
        cap = self.MAP_CAPACITY
        cov9 = np.empty((cap, 3, 3))
        t = C.c_int64()
        fn = self.lib._fn["cycle_covariances"]
        rc = fn(self.h, _dp(cov12), C.byref(t), _dp(cov6), _lp(pair_t), C.c_int32(cap), _dp(cov9), C.byref(info))
        d = info.as_dict()
        if rc != 0:
            msg = self.lib._fn["last_error"]().decode()
            if rc != self.CTVIO_ERR_STATE or not info.requested:
                raise CtvioError(f"{self.lib.prefix}cycle_covariances failed ({rc}): {msg}")
            d["error"] = msg
            return None, None, None, d
        a = info.available
        d["pair_t_ns"] = pair_t[:info.n_pairs].copy()
        return (cov12 if a & 1 else None, cov6[:info.n_pairs].copy() if a & 2 else None,
                cov9[:info.n_map_points].copy() if a & 4 else None, d)

    # the blob's header size: the counts section follows it and starts with nK, nB, nL (int32)
    CHECKPOINT_HEADER_BYTES = 40 + 16 * 21

    def Checkpoint(self) -> bytes:
        """ctvio_odometry_checkpoint: the odometry cycle's run as one blob (ctvio_odometry_restore continues it)."""
        n = C.c_int64()
        self.lib.call("odometry_checkpoint", self.h, None, 0, C.byref(n))
        buf = C.create_string_buffer(n.value)
        self.lib.call("odometry_checkpoint", self.h, buf, n.value, C.byref(n))
        return buf.raw[:n.value]

    def Restore(self, blob: bytes):
        """ctvio_odometry_restore: replace this engine's run with the blob's; the next call is ProcessImage."""
        blob = bytes(blob)
        self.lib.call("odometry_restore", self.h, blob, len(blob))
        nK, nB, nL = np.frombuffer(blob, np.int32, 3, self.CHECKPOINT_HEADER_BYTES).tolist()
        self.n_knots, self.n_bias, self.n_lm = nK, nB, nL

    def DebugBiasWeights(self, kf_times, sigma_wb, sigma_ab):
        """(test support) the bias random-walk weights of ctvio_process_image for these keyframe times over the resident
        IMU table: [n_kf - 1, 6]"""
        kf = _i64(kf_times)
        out = np.zeros((kf.shape[0] - 1, 6))
        self.lib.call("debug_bias_weights", self.h, C.c_int32(kf.shape[0]), _lp(kf), C.c_double(sigma_wb),
                      C.c_double(sigma_ab), _dp(out))
        return out

    def DebugStructure(self):
        """the structure the engine built for the current factor set (ctvio_debug_structure), as int64 arrays: desc
        (n_desc x 4), orig, items (x 4), lo, hi, woff, schur_items (x 4), entries (x 5), active, after a
        marginalization that built its blocks pos_cam, pos_lm, marg_img (else None), and imu_items (x 4: start, count,
        start knot, bias node)."""
        n = C.c_int64(0)
        self.lib.call("debug_structure", self.h, None, C.byref(n))
        out = np.zeros(n.value, np.int64)
        self.lib.call("debug_structure", self.h, _lp(out), C.byref(n))
        hdr = out[:16]
        n_f, n_desc, n_items, nL, n_si, n_e, np_, n_marg, n_imu = (int(x) for x in hdr[:9])
        parts = [("desc", (n_desc, 4)), ("orig", (n_f,)), ("items", (n_items, 4)), ("lo", (nL,)), ("hi", (nL,)),
                 ("woff", (nL + 1,)), ("schur_items", (n_si, 4)), ("entries", (n_e, 5)), ("active", (np_ + nL,))]
        if n_marg >= 0:
            parts += [("pos_cam", (np_,)), ("pos_lm", (nL,)), ("marg_img", (n_marg,))]
        parts += [("imu_items", (n_imu, 4))]
        res, o = {"pos_cam": None, "pos_lm": None, "marg_img": None}, 16
        for name, shape in parts:
            k = int(np.prod(shape))
            res[name] = out[o:o + k].reshape(shape)
            o += k
        return res

    def ProfileKernels(self, reps=20, flush_l2=True):
        out = np.zeros(8)
        self.lib.call("profile_kernels", self.h, C.c_int32(reps), C.c_int32(int(flush_l2)), _dp(out))
        names = ["visual", "imu", "small", "reduced_schur", "cholesky_solve", "step_vectors", "apply_table", "visual_cost"]
        return dict(zip(names, out.tolist()))

    def ProfileVisual(self, reps=20, flush_l2=True):
        """K1 only (sharded engines: the other stages involve collectives)."""
        out = np.zeros(8)
        self.lib.call("profile_kernels", self.h, C.c_int32(-reps), C.c_int32(int(flush_l2)), _dp(out))
        return float(out[0])

    def SelfcheckSolver(self, reps=50):
        """(bitwise mismatches over `reps` repeated solves of the same reduced system, relative residual)."""
        mm, res = C.c_int32(), C.c_double()
        self.lib.call("selfcheck_solver", self.h, C.c_int32(reps), C.byref(mm), C.byref(res))
        return mm.value, res.value

    def MeasureFp64Tflops(self):
        v = C.c_double()
        self.lib.call("measure_fp64_tflops", self.h, C.byref(v))
        return v.value

    def MeasureFp64TensorTflops(self):
        v = C.c_double()
        self.lib.call("measure_fp64_tensor_tflops", self.h, C.byref(v))
        return v.value

    # --- multi-GPU -----------------------------------------------------------------
    def NcclUniqueId(self) -> bytes:
        buf = (C.c_uint8 * 128)()
        self.lib.call("nccl_unique_id", buf)
        return bytes(buf)

    def CommInit(self, rank, world_size, unique_id: bytes):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self.lib.call("comm_init", self.h, C.c_int32(rank), C.c_int32(world_size), buf)
