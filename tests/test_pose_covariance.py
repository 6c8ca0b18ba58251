"""ctvio_pose_covariance: the covariance of the pose and velocity at any time, J(t) Sigma_sub J(t)', against references
independent of the engine.

The reference Jacobian J_fd comes from central differences of synthetic.spline_pose / spline_imu, each knot rotation
perturbed on the right (q_k -> q_k Exp(d)), each knot position additively; the rows are dtheta (right perturbation of
R(t), or of the camera's R(t) R_CI), dp, domega (body) and dv (world), the order of ctvio_query_trajectory.  The window
covariances are the cases of test_covariance (CASES): the engine's own Covariance() output for the projection alone,
the fp64 inverse of the oracle's H end to end.
"""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest

from helpers import get_state, pkg, syn
from test_covariance import CASES, RCOND_MIN, U, c3_prior_inputs, gpu_system, make_case, oracle_case, reference
from test_lm_step_regimes import regime_window

st = importlib.import_module("ctrl-vio_b200.streaming")
P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
ERR_INVALID, ERR_STATE, ERR_TIME_RANGE = -1, -4, -6


# ------------------------------------------------------------------------------------------------------------------
# finite-difference reference

def pose_quantities(q, p, t, w, camera):
    """(rotation quaternion, p, omega, v) at the times t: of the body, or of the camera (R R_CI, p + R p_CI)."""
    qt, pt = syn.spline_pose(q, p, t, w.t0_ns, w.dt_ns)
    om, _, v = syn.spline_imu(q, p, t, w.t0_ns, w.dt_ns)
    if camera:
        qc = np.broadcast_to(syn.Q_CtoI, qt.shape)
        pci = np.broadcast_to(syn.P_CinI, pt.shape)
        v = v + syn.qrot(qt, np.cross(om, pci))
        pt = pt + syn.qrot(qt, pci)
        om = syn.qrot(syn.qconj(qc), om)
        qt = syn.qmul(qt, qc)
    return qt, pt, om, v


def fd_jacobian(q, p, t, w, camera=False, h=1e-6):
    """J_fd [n, 12, 24] and the segment of each time: columns 6k + r over knots s..s+3 (r < 3 rotation, else
    position)."""
    t = np.asarray(t, np.int64)
    s = (t - w.t0_ns) // w.dt_ns
    q0 = pose_quantities(q, p, t, w, camera)[0]
    J = np.zeros((len(t), 12, 24))
    for k in range(4):
        for r in range(6):
            out = []
            for sgn in (1.0, -1.0):
                qq, pp = np.repeat(q[None], len(t), 0), np.repeat(p[None], len(t), 0)
                d = np.zeros(3); d[r % 3] = sgn * h
                rows = np.arange(len(t))
                if r < 3:
                    qq[rows, s + k] = syn.qmul(qq[rows, s + k], syn.qexp(d))
                else:
                    pp[rows, s + k] += d
                vals = [pose_quantities(qq[i], pp[i], t[i:i + 1], w, camera) for i in range(len(t))]
                qt = np.concatenate([x[0] for x in vals])
                dth = syn.qlog(syn.qmul(syn.qconj(q0), qt))
                out.append(np.concatenate([dth] + [np.concatenate([x[j] for x in vals]) for j in (1, 2, 3)], 1))
            J[:, :, 6 * k + r] = (out[0] - out[1]) / (2 * h)
    return J, s


def query_times(w, n_knots, n=50):
    """times spread over the window: interior points, knot boundaries, the first and the last valid nanosecond"""
    t_end = w.t0_ns + (n_knots - 3) * w.dt_ns
    inner = np.linspace(w.t0_ns, t_end - 1, n - 12).astype(np.int64)
    bounds = w.t0_ns + np.linspace(0, n_knots - 4, 10).astype(np.int64) * w.dt_ns
    return np.unique(np.concatenate([inner, bounds, [w.t0_ns, t_end - 1]]))


def sub_block(cov, s):
    return np.stack([cov[6 * x:6 * x + 24, 6 * x:6 * x + 24] for x in s])


def project(J, S):
    return np.einsum("nia,nab,njb->nij", J, S, J)


def abs_project(J, S):
    return np.einsum("nia,nab,njb->nij", np.abs(J), np.abs(S), np.abs(J))


FD_ERR = 1e-9  # J_fd's own error (rounding of the central differences), per row: below 5e-10 of the row's largest entry


def fd_error_project(J, S):
    """the part of |J_fd S J_fd' - J S J'| J_fd's own error can make: E |S| |J|' + |J| |S| E' + E |S| E'"""
    A = np.abs(J)
    E = np.broadcast_to(FD_ERR * A.max(axis=2, keepdims=True), A.shape)
    return abs_project(E, S) + np.einsum("nia,nab,njb->nij", E, np.abs(S), A) + np.einsum("nia,nab,njb->nij", A, np.abs(S), E)


# ------------------------------------------------------------------------------------------------------------------
# CPU part

def test_fd_reference_position_columns_are_the_spline_weights():
    """J_fd's position columns are c_k I (dp) and the first-derivative weights (dv) to rounding, in both frames; its
    rotation columns agree between h and h / 2."""
    w = syn.config_c2()
    q, p = w.q0, w.p0
    t = query_times(w, len(q), 12)
    s = (t - w.t0_ns) // w.dt_ns
    u = ((t - w.t0_ns) % w.dt_ns) / w.dt_ns
    inv_dt = 1e9 / w.dt_ns
    c0 = syn._coeffs(u, syn.M_PLAIN, 0, inv_dt)
    c1 = syn._coeffs(u, syn.M_PLAIN, 1, inv_dt)
    for camera in (False, True):
        J, s2 = fd_jacobian(q, p, t, w, camera)
        Jh, _ = fd_jacobian(q, p, t, w, camera, h=0.5e-6)
        assert np.array_equal(s, s2)
        scale = np.abs(J).max(axis=2, keepdims=True)  # per time and row: the omega / v rows carry 1 / dt
        for k in range(4):
            pos = J[:, :, 6 * k + 3:6 * k + 6]
            assert np.abs(pos[:, 3:6] - c0[:, k, None, None] * np.eye(3)).max() < 1e-8
            assert np.abs(pos[:, 9:12] - c1[:, k, None, None] * np.eye(3)).max() < 1e-8 * inv_dt
            assert np.abs(pos[:, 0:3]).max() < 1e-8 and np.abs(pos[:, 6:9]).max() < 1e-8 * inv_dt
            rot, roth = J[:, :, 6 * k:6 * k + 3], Jh[:, :, 6 * k:6 * k + 3]
            assert (np.abs(rot - roth) <= 1e-6 * scale).all(), np.abs(rot - roth).max()


def test_binding_exposes_the_pose_covariance():
    assert "pose_covariance" in pkg.ABI_SYMBOLS and "pose_covariance" in pkg.binding.DEVICE_ONLY_SYMBOLS
    assert hasattr(pkg.Estimator, "PoseCovariance")
    assert "publish_covariance" in st.ResidentRunner.__init__.__code__.co_varnames


def test_host_mirror_call_compiles(tmp_path):
    src = tmp_path / "pose_cov_mirror.cpp"
    src.write_text('#include "' + os.path.join(pkg.PKG_DIR, "host", "trajectory_estimator.hpp") + '"\n'
                   "double f(ctvio_host::TrajectoryEstimator& e) {\n"
                   "  int64_t t[2] = {0, 1};\n"
                   "  double cov[2 * 144];\n"
                   "  return e.GetPoseCovariance(2, t, 3, true, cov);\n"
                   "}\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", str(src)], check=True)


@pytest.fixture(scope="module")
def jac_lib(tmp_path_factory):
    """pose_jacobian / pose_jacobian_column of csrc/spline_eval.cuh built for the host"""
    d = tmp_path_factory.mktemp("posejac")
    src, so = d / "posejac.cpp", d / "libposejac.so"
    src.write_text('#include "' + os.path.join(pkg.CSRC_DIR, "spline_eval.cuh") + '"\n' + r'''
using namespace ctvio;
extern "C" int posejac(int64_t t0, int64_t dt, int nK, const double* q, const double* p, const double* qci,
                       const double* pci, int64_t t, int camera, double* J) {
  SplineParams sp{t0, dt, nK, 1e9 / double(dt)};
  int32_t s; double u;
  if (!spline_index(sp, t, s, u)) return -1;
  KnotPair* tab = new KnotPair[nK];
  for (int k = 0; k + 1 < nK; ++k) make_knot_pair(q, k, tab[k]);
  PoseJacobian pj;
  pose_jacobian<3>(sp, q, p, tab, s, u, pj);
  const M3 R_CI = so3_matrix(Q4{qci[0], qci[1], qci[2], qci[3]});
  for (int c = 0; c < 24; ++c) {
    double col[12];
    pose_jacobian_column(pj, camera != 0, R_CI, V3{pci[0], pci[1], pci[2]}, c, col);
    for (int i = 0; i < 12; ++i) J[i * 24 + c] = col[i];
  }
  delete[] tab;
  return s;
}
''')
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.posejac.restype = C.c_int
    lib.posejac.argtypes = [I64, I64, C.c_int, P, P, P, P, I64, C.c_int, P]
    return lib


def test_device_jacobian_matches_finite_differences(jac_lib):
    """The Jacobian pose_cov_kernel builds (the same inline functions, compiled for the host) against J_fd, in both
    frames, to FD_ERR of each row's largest entry (measured: below 5e-10, the rounding error of the differences)."""
    w = syn.config_c2()
    q, p = np.ascontiguousarray(w.q0), np.ascontiguousarray(w.p0)
    qci, pci = np.ascontiguousarray(syn.Q_CtoI, float), np.ascontiguousarray(syn.P_CinI, float)
    t = query_times(w, len(q), 20)
    for camera in (False, True):
        Jfd, s = fd_jacobian(q, p, t, w, camera)
        for i, ti in enumerate(t):
            J = np.zeros((12, 24))
            assert jac_lib.posejac(w.t0_ns, w.dt_ns, len(q), q.ctypes.data, p.ctypes.data, qci.ctypes.data,
                                   pci.ctypes.data, int(ti), int(camera), J.ctypes.data) == s[i]
            scale = np.abs(Jfd[i]).max(axis=1, keepdims=True)  # per row: the omega / v rows carry 1 / dt
            assert (np.abs(J - Jfd[i]) <= FD_ERR * scale).all(), (camera, i, np.abs(J - Jfd[i]).max())


# ------------------------------------------------------------------------------------------------------------------
# GPU part

def case_window(oracle_lib, name):
    return c3_prior_inputs(oracle_lib)[0] if CASES[name][0] == "c3prior" else regime_window(CASES[name][0])


def cov_bound(est, s, ref):
    """test_covariance's entrywise bound on |Sigma_engine - Sigma_ref| (kappa-based, in the Jacobi-scaled space)"""
    free, sc = s["free"], ref["sc"]
    A, W, hl = gpu_system(est)
    A = np.triu(A) + np.triu(A, 1).T
    nL = len(s["hl"])
    dH = np.block([[A - s["A"], (W[:nL] - s["W"]).T], [W[:nL] - s["W"], np.diag(hl[:nL] - s["hl"])]])
    H = np.block([[s["A"], s["W"].T], [s["W"], np.diag(s["hl"])]])
    keep = np.concatenate([free, s["hl"] > 0])
    sf = 1.0 / (1.0 + np.sqrt(np.diag(H)[keep]))
    K = sf[:, None] * H[np.ix_(keep, keep)] * sf[None, :]
    eta = np.abs(sf[:, None] * dH[np.ix_(keep, keep)] * sf[None, :]).sum(1).max() / np.abs(K).sum(1).max()
    npad = (A.shape[0] + 63) // 64 * 64
    bound = ref["kappa"] * (4 * npad * U + 2 * eta) * ref["kinv_max"]
    d = np.where(free, sc, 0.0)
    return bound * d[:, None] * d[None, :]


def check_psd_symmetric(C):
    assert np.array_equal(C, np.swapaxes(C, 1, 2))
    for c in C:
        lam = np.linalg.eigvalsh(c)
        assert lam[0] >= -1e-12 * max(lam[-1], 0.0), lam


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_pose_covariance_matches_references(oracle_lib, cuda_lib, name):
    """Per case, about 50 times, both frames: C against J_fd Sigma J_fd' (Sigma the engine's Covariance(), the one the
    call forms), the dp block against sum c_k c_l Sigma_{P_k P_l}, and C against J_fd Sigma_ref J_fd' end to end."""
    s = oracle_case(oracle_lib, name)
    ref = reference(s)
    w = case_window(oracle_lib, name)
    est, opt = make_case(cuda_lib, oracle_lib, name)
    est.SetDeterministic(True)
    cov, _, rc0 = est.Covariance(want_rho=False)
    q, p = est.GetKnots()
    t = query_times(w, est.n_knots)
    Sbound = cov_bound(est, s, ref)
    worst = [0.0, 0.0]
    for camera in (False, True):
        C_, rc = est.PoseCovariance(t, camera_frame=camera)
        assert rc == rc0 and C_.shape == (len(t), 12, 12)
        check_psd_symmetric(C_)
        Jfd, seg = fd_jacobian(q, p, t, w, camera)
        S = sub_block(cov, seg)
        # 1. the projection alone
        tol1 = 1e-7 * abs_project(Jfd, S) + fd_error_project(Jfd, S)
        err1 = np.abs(C_ - project(Jfd, S))
        r1 = np.where(tol1 > 0, err1 / np.maximum(tol1, 1e-300), 0.0)
        assert (err1 <= tol1).all(), r1.max()
        if not camera:  # dp = sum_k c_k dP_k: its block is sum c_k c_l Sigma_{P_k P_l}, against a long-double sum
            u = ((t - w.t0_ns) % w.dt_ns).astype(np.float64) / w.dt_ns
            c0 = syn._coeffs(u, syn.M_PLAIN, 0, 1e9 / w.dt_ns).astype(np.longdouble)
            for a in range(3):
                for b in range(3):
                    Skl = S[:, [6 * k + 3 + a for k in range(4)]][:, :, [6 * k + 3 + b for k in range(4)]]
                    Skl = Skl.astype(np.longdouble)
                    pp = np.einsum("nk,nkl,nl->n", c0, Skl, c0)
                    mag = np.einsum("nk,nkl,nl->n", np.abs(c0), np.abs(Skl), np.abs(c0))
                    err = np.abs(C_[:, 3 + a, 3 + b].astype(np.longdouble) - pp)
                    assert (err <= 8 * U * mag).all(), float((err / np.maximum(mag, 1e-300)).max())
        # 2. end to end against the fp64 reference, the covariance bound propagated through |J|
        Sref = sub_block(ref["cov"], seg)
        tol = (abs_project(Jfd, sub_block(Sbound, seg)) + 1e-7 * abs_project(Jfd, np.abs(Sref) + np.abs(S))
               + fd_error_project(Jfd, Sref))
        err = np.abs(C_ - project(Jfd, Sref))
        assert (err <= tol).all(), float((err / np.maximum(tol, 1e-300)).max())
        worst = [max(worst[0], r1.max()), max(worst[1], float((err / np.maximum(tol, 1e-300)).max()))]
    print(f"{name}: {len(t)} times, rcond {rc0:.2e}; worst ratio to bound: projection {worst[0]:.1e}, "
          f"end-to-end ratio to bound {worst[1]:.1e}")


@pytest.mark.gpu
def test_gauge_argument(oracle_lib, cuda_lib):
    """The c2 window without fixed knots is rank deficient (only rcond written); with gauge_knot_index = 3 it matches the
    c2 case, whose options fix knots 0..3."""
    free, _ = make_case(cuda_lib, oracle_lib, "c2", fixed_knot_index=-1)
    fixed, _ = make_case(cuda_lib, oracle_lib, "c2")
    for e in (free, fixed):
        e.SetDeterministic(True)
    w = case_window(oracle_lib, "c2")
    t = query_times(w, free.n_knots)
    f = cuda_lib.lib.ctvio_pose_covariance
    f.argtypes = [P, I32, P, I32, I32, P, P]
    f.restype = C.c_int
    out = np.full((len(t), 12, 12), 123.5)
    rcond = C.c_double(-1.0)
    rc = f(free.h, len(t), t.ctypes.data, -1, 1, out.ctypes.data, C.byref(rcond))
    msg = cuda_lib._fn["last_error"]().decode()
    print(f"no gauge: rc {rc}, rcond {rcond.value:.2e}, '{msg}'")
    assert rc == ERR_STATE and "rank deficient" in msg and (out == 123.5).all()
    assert 0.0 <= rcond.value < RCOND_MIN or "pivot" in msg
    with pytest.raises(pkg.CtvioError, match="rank deficient"):
        free.PoseCovariance(t)
    for camera in (False, True):
        Cg, rg = free.PoseCovariance(t, gauge_knot_index=3, camera_frame=camera)
        Cf, rf = fixed.PoseCovariance(t, camera_frame=camera)
        d = np.sqrt(np.einsum("nii->ni", Cf))
        scale = d[:, :, None] * d[:, None, :]
        err = np.abs(Cg - Cf)
        print(f"camera {camera}: rcond {rg:.3e} vs {rf:.3e}, worst relative {float((err / np.maximum(scale, 1e-300)).max()):.1e}")
        assert (err <= 1e-12 * scale).all()
        assert abs(rg - rf) <= 1e-12 * rf
    # the gauge leaves the solve's options alone: the window is still rank deficient for ctvio_covariance
    with pytest.raises(pkg.CtvioError, match="rank deficient"):
        free.Covariance()


@pytest.mark.gpu
def test_constant_knots_give_exact_zeros(oracle_lib, cuda_lib):
    """masked case (knots 0..12 fixed): segments <= 9 use constant knots only and get exact zero matrices; segments
    10..12 have the free knot 13 and a non-zero covariance (their values are checked in
    test_pose_covariance_matches_references)."""
    est, _ = make_case(cuda_lib, oracle_lib, "masked")
    est.SetDeterministic(True)
    w = case_window(oracle_lib, "masked")
    t = w.t0_ns + np.arange(14, dtype=np.int64) * w.dt_ns + w.dt_ns // 3
    for camera in (False, True):
        Cm, _ = est.PoseCovariance(t, camera_frame=camera)
        assert not Cm[:10].any()
        assert all(Cm[k].any() for k in range(10, 14))
        check_psd_symmetric(Cm)


@pytest.mark.gpu
def test_errors_leave_the_output_untouched(oracle_lib, cuda_lib):
    est, _ = make_case(cuda_lib, oracle_lib, "c2")
    f = cuda_lib.lib.ctvio_pose_covariance
    f.argtypes = [P, I32, P, I32, I32, P, P]
    f.restype = C.c_int
    w = case_window(oracle_lib, "c2")
    t_end = w.t0_ns + (est.n_knots - 3) * w.dt_ns
    good = np.array([w.t0_ns + 5, t_end - 1], np.int64)
    out = np.full((2, 12, 12), 123.5)
    rcond = C.c_double(-7.0)

    def call(h=est.h, n=2, t=good, gauge=-1, cam=0, o=out):
        return f(h, n, None if t is None else t.ctypes.data, gauge, cam, None if o is None else o.ctypes.data,
                 C.byref(rcond))
    cases = [
        (dict(h=None), ERR_INVALID), (dict(n=-1), ERR_INVALID), (dict(t=None), ERR_INVALID),
        (dict(o=None), ERR_INVALID), (dict(cam=2), ERR_INVALID), (dict(cam=-1), ERR_INVALID),
        (dict(gauge=-2), ERR_INVALID), (dict(gauge=est.n_knots), ERR_INVALID),
        (dict(t=np.array([w.t0_ns - 1, t_end - 1], np.int64)), ERR_TIME_RANGE),
        (dict(t=np.array([w.t0_ns, t_end], np.int64)), ERR_TIME_RANGE),
    ]
    for kw, code in cases:
        assert call(**kw) == code, kw
        assert (out == 123.5).all() and rcond.value == -7.0, kw
    assert call(n=0, t=None, o=None) == 0 and rcond.value == -7.0
    assert call(gauge=est.n_knots - 1) == 0  # the whole trajectory constant: every matrix exactly zero
    assert not out.any()
    cfg = pkg.make_config(**w.config_kwargs())
    bare = pkg.Estimator(cuda_lib, cfg)
    with pytest.raises(pkg.CtvioError, match=r"\(-4\)"):
        bare.PoseCovariance(good)


@pytest.mark.gpu
def test_no_side_effects_and_transfer_counts(oracle_lib, cuda_lib):
    """Deterministic mode: a solve after the call is bitwise the solve without it (C3 window with its prior); the call
    moves 8 n bytes up and 1152 n bytes down."""
    runs = []
    w = case_window(oracle_lib, "c3prior")
    for with_cov in (True, False):
        est, _ = make_case(cuda_lib, oracle_lib, "c3prior")
        est.SetDeterministic(True)
        t = query_times(w, est.n_knots, 20)
        if with_cov:
            x0 = get_state(est)
            est.PoseCovariance(t, gauge_knot_index=5, camera_frame=True)
            x1 = get_state(est)
            assert all(np.array_equal(a, b) for a, b in zip(x0[:4], x1[:4])) and x0[4] == x1[4]
            est.TransferStats(reset=True)
            est.PoseCovariance(t)
            assert est.TransferStats() == (8 * len(t), 1152 * len(t))
        s = est.Solve(8)
        runs.append((s, get_state(est)))
    (s1, x1), (s2, x2) = runs
    for fld in ("iterations", "num_successful_steps", "num_unsuccessful_steps", "termination", "initial_cost",
                "final_cost", "final_radius", "num_linear_solves", "num_jacobian_evals"):
        assert getattr(s1, fld) == getattr(s2, fld), fld
    assert all(np.array_equal(a, b) for a, b in zip(x1[:4], x2[:4])) and x1[4] == x2[4]


class PriorRecorder:
    """Stands in for the runner's library: after each marginalization, the fresh prior read with ctvio_get_prior."""

    def __init__(self, lib):
        self._lib = lib
        self.priors = []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def call(self, name, h, *args):
        rc = self._lib.call(name, h, *args)
        if name == "marginalize":
            n, nb = args[0]._obj.value, args[1]._obj.value
            if n > 0:
                J, r, x0 = np.zeros((n, n)), np.zeros(n), np.zeros((nb, 4))
                ty, ix, co = np.zeros(nb, np.int32), np.zeros(nb, np.int32), np.zeros(nb, np.int32)
                self._lib.call("get_prior", h, J.ctypes.data_as(P), r.ctypes.data_as(P), ty.ctypes.data_as(P),
                               ix.ctypes.data_as(P), co.ctypes.data_as(P), x0.ctypes.data_as(P))
                self.priors.append((J, r, ty, ix, co, x0))
        return rc


def bitwise(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.gpu
def test_runner_publish_covariance_only_reads(cuda_lib):
    """Six C5 windows, deterministic: the runner with publish_covariance=True solves, marginalizes and slides exactly as
    the runner without it, and every window's camera-pose covariance is finite, symmetric, PSD, with rcond >= 1e-14."""
    n = 6
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    a = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True)
    b = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, publish_covariance=True)
    covs = []
    for x in (a, b):
        x.est.SetDeterministic(True)
        x.est.lib = PriorRecorder(x.est.lib)
    for _ in range(n):
        a.step()
        b.step()
        covs.append(b.last_pose_cov)
    for rec in b.records:
        print(f"window {rec['window']}: pose_cov_rcond {rec['pose_cov_rcond']:.3e}, ms_pose_cov {rec['ms_pose_cov']:.3f}"
              + (f", {rec['pose_cov_error']}" if "pose_cov_error" in rec else ""))
    for key in ("iterations", "initial_cost", "final_cost", "prior_dim", "n_obs", "n_lm"):
        assert [x[key] for x in a.records] == [x[key] for x in b.records], key
    assert "pose_cov_rcond" not in a.records[0] and a.last_pose_cov is None
    assert bitwise(a.q[:a.ncp], b.q[:b.ncp]) and bitwise(a.p[:a.ncp], b.p[:b.ncp])
    assert bitwise(a.est.GetBiases(), b.est.GetBiases())
    assert bitwise(a.est.GetInvDepths(), b.est.GetInvDepths())
    assert bitwise(a.ld, b.ld)
    pa, pb = a.est.lib.priors, b.est.lib.priors
    assert len(pa) == len(pb) > 0
    assert all(bitwise(x, y) for u, v in zip(pa, pb) for x, y in zip(u, v))
    for rec, c in zip(b.records, covs):
        assert rec["pose_cov_rcond"] >= RCOND_MIN, rec
        assert c.shape == (1, 12, 12) and np.isfinite(c).all() and np.diag(c[0]).min() > 0
        check_psd_symmetric(c)
