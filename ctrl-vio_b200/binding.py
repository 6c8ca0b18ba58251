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


# every symbol include/ctvio.h declares (without prefix); used by the
# export-completeness test and by the binder.
ABI_SYMBOLS = [
    "last_error", "abi_version", "create", "destroy", "set_options", "set_deterministic",
    "set_knots", "set_biases", "set_inv_depths", "set_line_delay", "set_time_origin",
    "get_knots", "get_biases", "get_inv_depths", "get_line_delay",
    "clear_factors", "add_image_features", "add_imu_measurements", "add_bias_factors", "set_prior",
    "solve", "gauge_realign", "marginalize", "get_prior", "adopt_prior",
    "save_state", "restore_state",
    "eval_image_factors", "eval_imu_factors", "residual_summary", "eval_cost", "normal_equations",
    "query_trajectory", "triangulate",
    "extend_knots_to", "slide_window", "remap_landmarks", "enable_prior", "ingest_feature_cloud", "add_image_features_from_slots",
    "ingest_imu", "add_imu_from_table", "transfer_stats", "profile_kernels", "measure_fp64_tflops", "measure_fp64_tensor_tflops",
    "selfcheck_solver", "nccl_unique_id", "comm_init",
]


# entry points a checker library (the CPU oracle mirrors the ABI under `ctvo_`) need not provide: multi-GPU plumbing and
# the device-residency / wire-format calls, which have no CPU meaning
DEVICE_ONLY_SYMBOLS = ("nccl_unique_id", "comm_init", "set_deterministic", "enable_prior", "extend_knots_to", "slide_window", "remap_landmarks", "enable_prior",
                       "ingest_feature_cloud", "add_image_features_from_slots", "ingest_imu", "add_imu_from_table",
                       "transfer_stats", "residual_summary")


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
